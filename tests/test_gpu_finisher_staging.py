"""Staged re-projection of the finishers (lk_fused.cu: fused_finish). While it waits for the last chunk rows, a finisher
forms the IMU-frame points of its first FIN_STAGE points and keeps them in shared memory; the rest of its share, and
every point in direct mode, goes through the loop that loads them after the solve. Either way the world cloud and every
other output must equal those of the kernel without finishers (lk_set_param "finishers" 0) bit for bit: at scan sizes
that put one finisher's share just below, at and just above the staging capacity, at one spare SM (one finisher: most
of its share overflows), in direct mode, and in back-to-back rings at 1 and 3 iterations."""
import numpy as np
import pytest

from test_gpu_finishers import _run_ring, _same, _scans, _sms

pytestmark = pytest.mark.gpu

BLOCK = 256
# lk_fused.cu FIN_STAGE: the record tiles of the hot-image pass (2 x 256 slots x 176 B) less the group sums of the
# finishers' one-hop total (LL_MAX_GROUPS = 20 rows of 32 doubles), over three doubles per point
FIN_STAGE = (2 * BLOCK * 176 - 20 * 32 * 8) // 24
MAX_FINISHERS = 24  # lk_llsync.cuh: LL_MAX_FINISHERS


def _shares(n, sms):
    """Points of each finisher for an n-point scan (lk_api.cu: finishers = min(spare SMs, 24); fused_finish: finisher
    fi, thread t takes points fi * 256 + t + j * step), or None when the scan leaves no SM spare."""
    chunks = -(-n // BLOCK)
    if chunks >= sms:
        return None
    step = min(sms - chunks, MAX_FINISHERS) * BLOCK
    return [sum(max(0, -(-(n - fi * BLOCK - t) // step)) for t in range(BLOCK)) for fi in range(step // BLOCK)]


def _capacity_sizes():
    """The smallest scan sizes at which some finisher's share is FIN_STAGE - 1, FIN_STAGE and FIN_STAGE + 1."""
    sms = _sms()
    out = {}
    for n in range(1, sms * BLOCK):
        s = _shares(n, sms)
        for d in (-1, 0, 1):
            if s is not None and d not in out and FIN_STAGE + d in s:
                out[d] = n
    if len(out) < 3:
        pytest.skip(f"no scan size puts a finisher's share at the staging capacity on {sms} SMs")
    return [out[-1], out[0], out[1]]


@pytest.mark.parametrize("iters", [1, 3])
def test_ring_at_staging_capacity_bitwise(iters):
    sizes = _capacity_sizes() + [(_sms() - 1) * BLOCK]
    cfg, blob, scans = _scans(sizes, stream0=5100)
    ref = _run_ring(cfg, blob, scans, iters, 1, finishers=0)
    assert int(ref["n_eff"].min()) > 0
    out = _run_ring(cfg, blob, scans, iters, 4, finishers=1)
    _same(out, ref)


@pytest.mark.parametrize("edge", [-1, 0, 1])
def test_direct_mode_at_staging_capacity_bitwise(edge):
    from legkilo_b200 import Engine, abi

    n = _capacity_sizes()[edge + 1]
    cfg, blob, scans = _scans([n], stream0=5200)
    args = (abi.default_states(1), abi.init_cov(1), abi.process_cov_Q(cfg), np.zeros(1, abi.CLOCK_DTYPE), scans[0],
            [0, n], [0.0])
    outs = []
    for fin in (0, 1):
        eng = Engine(cfg)
        eng.set_param("finishers", fin)
        eng.map_upload(blob)
        for _ in range(3):  # back to back: the second and third launches follow a fused launch (PDL)
            o = eng.scan_update(*args, iters=3, pinned=True)
        outs.append(o)
    ref, out = outs
    assert int(ref["n_eff"][0]) > 0
    _same(out, ref)
