"""Finishers of the per-scan kernel (lk_fused.cu): a single-bucket scan that leaves SMs idle runs its last exchange, solve,
re-projection, covariance update and stores on extra blocks while the chunk blocks leave at their last row. Whatever
the grid looks like, the results must equal those of the kernel without finishers (lk_set_param "finishers" 0) bit for
bit: a ring of scans of many sizes launched back to back (programmatic dependent launch), every iteration count the
kernel's exchange buffers cycle through, direct mode, and the grid edges: one spare SM, no spare SM (the old path), and
a tiny scan (the cap on the number of finishers)."""
import numpy as np
import pytest
import torch

import scenes
from legkilo_b200 import Engine, abi

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _scans(sizes, stream0=4700):
    """Scans of exactly `sizes` points, drawn from box-room scans (a point and its map lookups are valid wherever it
    appears); the chunk count of a scan is its size over 256, rounded up."""
    cfg, blob, scans = scenes.box_scene(batch=2, stream0=stream0)
    base = np.concatenate(scans)
    rng = np.random.default_rng(stream0)
    return cfg, blob, [base[rng.integers(0, len(base), n)] for n in sizes]


def _ring_sizes():
    s = _sms()
    # typical, one spare SM, no spare SM, tiny (finishers capped), a partial last chunk
    return [28800, (s - 1) * 256, s * 256, 300, 20000 + 77]


def _run_ring(cfg, blob, scans, iters, reps, **params):
    n = len(scans)
    pts = np.concatenate(scans)
    offs = np.concatenate([[0], np.cumsum([len(s) for s in scans])]).astype(np.uint32)
    eng = Engine(cfg)
    for k, v in params.items():
        eng.set_param(k, v)
    eng.map_upload(blob)
    eng.stage(abi.default_states(n), abi.init_cov(n), abi.process_cov_Q(cfg), np.zeros(n, abi.CLOCK_DTYPE), pts, offs, np.zeros(n))
    for rep in range(reps):
        for i in range(n):
            eng.run_range(i, 1, iters=iters)
    eng.sync()
    return eng.fetch()


def _same(out, ref):
    assert out["x"].tobytes() == ref["x"].tobytes()
    assert out["P"].tobytes() == ref["P"].tobytes()
    assert out["clk"].tobytes() == ref["clk"].tobytes()
    assert np.array_equal(out["n_eff"], ref["n_eff"])
    np.testing.assert_array_equal(np.asarray(out["world"]), np.asarray(ref["world"]))


@pytest.mark.parametrize("iters", [1, 2, 3, 4, 5])
def test_ring_back_to_back_bitwise(iters):
    cfg, blob, scans = _scans(_ring_sizes())
    ref = _run_ring(cfg, blob, scans, iters, 1, finishers=0)
    assert int(ref["n_eff"].min()) > 0
    out = _run_ring(cfg, blob, scans, iters, 8, finishers=1)
    _same(out, ref)


@pytest.mark.parametrize("params", [dict(pdl=0), dict(slim_p=0), dict(lane_cache=0)])
def test_ring_launch_modes_bitwise(params):
    cfg, blob, scans = _scans(_ring_sizes(), stream0=4800)
    ref = _run_ring(cfg, blob, scans, 3, 1, finishers=0)
    out = _run_ring(cfg, blob, scans, 3, 4, finishers=1, **params)
    _same(out, ref)


@pytest.mark.parametrize("size", ["typical", "one_spare", "no_spare", "tiny"])
def test_direct_mode_bitwise(size):
    s = _sms()
    n = dict(typical=28800, one_spare=(s - 1) * 256, no_spare=s * 256, tiny=300)[size]
    cfg, blob, scans = _scans([n], stream0=4900)
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
    assert out["x"].tobytes() == ref["x"].tobytes()
    assert out["P"].tobytes() == ref["P"].tobytes()
    assert out["clk"].tobytes() == ref["clk"].tobytes()
    np.testing.assert_array_equal(out["n_eff"], ref["n_eff"])
    np.testing.assert_array_equal(np.asarray(out["world"]), np.asarray(ref["world"]))
