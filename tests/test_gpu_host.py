"""Host-side state of a handle: a staged batch is not disturbed by the one-filter steps, and a map upload whose
allocation fails leaves the handle with no map (not a half-built one)."""
import numpy as np
import pytest

import scenes
from legkilo_b200 import Engine, LkError, abi, synth

pytestmark = pytest.mark.gpu


def _same(a, b):
    for k in ("x", "P", "clk", "world", "n_eff"):
        assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), k


def _unrelated_filter_steps(eng, cfg):
    g = synth.rng(77)
    A = g.standard_normal((30, 30)) * 1e-3
    x = abi.default_states(1)
    P = A @ A.T + 1e-6 * np.eye(30)
    Q = abi.process_cov_Q(cfg)
    clk = np.zeros(1, abi.CLOCK_DTYPE); clk["last_predict_time"] = 3.0; clk["last_update_time"] = 2.995
    eng.predict(x, P.reshape(1, 900), Q, [0.01])
    eng.obs_imu(x, P, Q, clk, synth.imu_stream(3.0, 3.02))
    eng.update_by_points(x, P, g.standard_normal((8, 6)), g.standard_normal(8) * 1e-2, np.full(8, 1e-3))


@pytest.mark.parametrize("batch", [1, 3])  # 1: the per-scan kernel; 3: the throughput kernels
def test_staged_batch_survives_filter_steps(batch):
    cfg, blob, scans = scenes.box_scene(batch=batch)
    eng = Engine(cfg)
    eng.map_upload(blob)
    pts = np.concatenate(scans)
    offs = np.concatenate([[0], np.cumsum([len(s) for s in scans])])
    eng.stage(abi.default_states(batch), abi.init_cov(batch), abi.process_cov_Q(cfg), np.zeros(batch, abi.CLOCK_DTYPE),
              pts, offs, np.zeros(batch))
    eng.run(iters=2)
    a = eng.fetch()
    assert a["n_eff"].min() > 0
    _unrelated_filter_steps(eng, cfg)
    eng.run(iters=2)  # runs again from the staged inputs
    _same(a, eng.fetch())


def test_failed_map_upload_leaves_no_map():
    cfg, blob, scans = scenes.box_scene(batch=1)
    args = (abi.default_states(1), abi.init_cov(1), abi.process_cov_Q(cfg), np.zeros(1, abi.CLOCK_DTYPE), scans[0],
            [0, len(scans[0])], [0.0])
    eng = Engine(cfg)
    eng.map_reserve(0, 1 << 30, 0)  # a node pool of 2^30 nodes: cudaMalloc refuses it without holding any memory
    with pytest.raises(LkError) as e:
        eng.map_upload(blob)
    assert e.value.code == -4  # LK_ERR_OUT_OF_MEMORY
    assert all(v == 0 for v in eng.map_memory().values()), eng.map_memory()
    with pytest.raises(LkError) as e:
        eng.scan_update(*args)
    assert e.value.code == -7  # LK_ERR_NOT_READY
    eng.map_reserve(0, 0, 0)
    eng.map_upload(blob)
    ref = Engine(cfg)
    ref.map_upload(blob)
    _same(eng.scan_update(*args), ref.scan_update(*args))


def test_direct_staged_batch_refuses_other_paths():
    """lk_scan_update on page-locked buffers stages for the per-scan kernel alone (the points stay in the caller's buffer,
    the small inputs ride in the launch): running that batch again through any other path is refused before a kernel
    reads device buffers that were never filled, and the handle keeps working."""
    cfg, blob, scans = scenes.box_scene(batch=1)
    args = (abi.default_states(1), abi.init_cov(1), abi.process_cov_Q(cfg), np.zeros(1, abi.CLOCK_DTYPE), scans[0],
            [0, len(scans[0])], [0.0])
    eng = Engine(cfg)
    eng.map_upload(blob)
    eng.scan_update(*args, iters=2, pinned=True)
    with pytest.raises(LkError) as e:
        eng.run(iters=2, update_map=True)  # the map update runs outside the per-scan kernel (fused_insert is off)
    assert e.value.code == -2, e.value
    eng.set_param("fused", 0)
    with pytest.raises(LkError) as e:
        eng.run(iters=2)
    assert e.value.code == -2, e.value
    eng.set_param("fused", 1)
    ref = Engine(cfg)
    ref.map_upload(blob)
    _same(eng.scan_update(*args, iters=2), ref.scan_update(*args, iters=2))
