"""Edge cases of the boundary on the GPU: empty and far-away scans, ragged batches, argument errors (status codes,
never an exception across the ABI, handle usable afterwards)."""
import numpy as np
import pytest

import lko
import scenes
from legkilo_b200 import Engine, LkError, abi

pytestmark = pytest.mark.gpu
STATE_TOL = 7e-12  # (tests/scenes.py) worst measured on an H100 80GB HBM3: 7.2e-14 sd
COV_TOL = 1.9e-12  # worst measured: 1.9e-14


def _oracle(cfg, blob, pts, x0, P0, iters):
    o = lko.Oracle(cfg)
    o.map_import(blob)
    o.set_filter(x0, P0, abi.process_cov_Q(cfg), np.zeros(1, abi.CLOCK_DTYPE))
    o.set_options(gain_mode=lko.GAIN_INFORMATION, iters=iters, update_map=False)
    r = o.predict_update_point(0.0, pts, debug=False)
    x, P, _, _ = o.get_filter()
    return r, x, P


def test_empty_scan_alone_leaves_the_filter_untouched():
    cfg, blob, _ = scenes.box_scene(batch=1)
    eng = Engine(cfg)
    eng.map_upload(blob)
    x0 = abi.default_states(1); P0 = abi.init_cov(1)
    out = eng.scan_update(x0, P0, abi.process_cov_Q(cfg), np.zeros(1, abi.CLOCK_DTYPE), np.zeros((0, 4), np.float32), [0, 0], [0.0], iters=2)
    assert int(out["n_eff"][0]) == 0
    np.testing.assert_array_equal(out["x"].view(np.float64), x0.view(np.float64))
    np.testing.assert_array_equal(out["P"], P0.reshape(1, 900))


def test_ragged_batch_with_empty_and_far_away_scans():
    """Scan 1 has no points, scan 3 looks at nothing the map knows (no voxel hit => no residual => no update, KILO.cc:180-185);
    their neighbours in the same call are unaffected."""
    cfg, blob, scans = scenes.box_scene(batch=3)
    far = scans[2].copy(); far[:, :3] += np.float32(1000.0)
    pieces = [scans[0], np.zeros((0, 4), np.float32), scans[1], far]
    B = len(pieces)
    pts = np.concatenate(pieces)
    offs = np.concatenate([[0], np.cumsum([len(p) for p in pieces])]).astype(np.uint32)
    x0 = abi.default_states(B); P0 = abi.init_cov(B)
    eng = Engine(cfg)
    eng.map_upload(blob)
    out = eng.scan_update(x0, P0, abi.process_cov_Q(cfg), np.zeros(B, abi.CLOCK_DTYPE), pts, offs, np.zeros(B), iters=2)
    for i in (0, 2):
        ro, xo, Po = _oracle(cfg, blob, pieces[i], x0[i:i + 1], P0[i:i + 1], 2)
        assert int(out["n_eff"][i]) == ro["n_eff"] > 0
        scenes.check_filter(out["x"][i:i + 1], out["P"][i], xo, Po, STATE_TOL, COV_TOL, f"scan {i}")
    for i in (1, 3):
        assert int(out["n_eff"][i]) == 0
        np.testing.assert_array_equal(out["x"][i:i + 1].view(np.float64), x0[i:i + 1].view(np.float64))
        np.testing.assert_array_equal(out["P"][i], P0.reshape(B, 900)[i])
    # the far-away scan is still re-projected (intensity 0: no update happened, KILO.cc:130-133)
    w = out["world"][offs[3]:offs[4]]
    assert np.all(w[:, 3] == 0.0) and np.isfinite(w).all()


def test_argument_errors_are_status_codes_and_the_handle_survives():
    cfg, blob, scans = scenes.box_scene(batch=2)
    eng = Engine(cfg)
    x1 = abi.default_states(1); P1 = abi.init_cov(1); Q = abi.process_cov_Q(cfg); c1 = np.zeros(1, abi.CLOCK_DTYPE)
    s = scans[0]
    with pytest.raises(LkError) as e:  # no map yet
        eng.scan_update(x1, P1, Q, c1, s, [0, len(s)], [0.0])
    assert e.value.code == -7
    with pytest.raises(LkError) as e:  # not a map blob
        eng.map_upload(np.frombuffer(b"\x01" * 4096, np.uint8).copy())
    assert e.value.code < 0
    eng.map_upload(blob)
    with pytest.raises(LkError) as e:  # iterations must be >= 1
        eng.scan_update(x1, P1, Q, c1, s, [0, len(s)], [0.0], iters=0)
    assert e.value.code == -1
    with pytest.raises(LkError) as e:  # offsets must be monotone
        eng.scan_update(abi.default_states(2), abi.init_cov(2), Q, np.zeros(2, abi.CLOCK_DTYPE), s, [0, len(s), len(s) - 5], np.zeros(2))
    assert e.value.code == -1
    with pytest.raises(LkError) as e:  # a map-updating stream is one scan per call
        pts = np.concatenate(scans); offs = [0, len(scans[0]), len(pts)]
        eng.scan_update(abi.default_states(2), abi.init_cov(2), Q, np.zeros(2, abi.CLOCK_DTYPE), pts, offs, np.zeros(2), update_map=True)
    assert e.value.code == -1
    # and the handle still works
    out = eng.scan_update(x1, P1, Q, c1, s, [0, len(s)], [0.0], iters=2)
    ro, xo, Po = _oracle(cfg, blob, s, x1, P1, 2)
    assert int(out["n_eff"][0]) == ro["n_eff"] > 0
    scenes.check_filter(out["x"], out["P"][0], xo, Po, STATE_TOL, COV_TOL)


def test_corrupt_map_blobs_are_rejected():
    """lk_map_upload validates what the kernels later follow blindly: child indices, layers, child masks without children,
    and two roots with one key (the second would be unreachable). A rejected upload leaves the handle usable."""
    cfg, blob, scans = scenes.box_scene(batch=1)
    hd, roots, nodes, aux, pts = abi.parse_map_blob(blob)
    eng = Engine(cfg)

    def bad(mut):
        r, n, a = roots.copy(), nodes.copy(), aux.copy()
        mut(r, n, a)
        with pytest.raises(LkError) as e:
            eng.map_upload(abi.make_map_blob(r, n, a, pts))
        assert e.value.code == -5, e.value  # LK_ERR_BAD_BLOB

    def child_out_of_range(r, n, a):
        n["child_base"][3] = len(n) - 4
    def negative_child(r, n, a):
        n["child_base"][3] = -7
    def mask_without_children(r, n, a):
        n["flags"][5] = (int(n["flags"][5]) | (0x21 << 16)); n["child_base"][5] = -1
    def layer_too_deep(r, n, a):
        n["flags"][7] = (int(n["flags"][7]) & ~0xFF00) | (4 << 8)
    def duplicate_root(r, n, a):
        r["key"][1] = r["key"][0]
    def root_node_out_of_range(r, n, a):
        r["node"][2] = len(n)
    for m in (child_out_of_range, negative_child, mask_without_children, layer_too_deep, duplicate_root, root_node_out_of_range):
        bad(m)
    eng.map_upload(blob)  # the handle survived all of that
    x0 = abi.default_states(1); P0 = abi.init_cov(1)
    out = eng.scan_update(x0, P0, abi.process_cov_Q(cfg), np.zeros(1, abi.CLOCK_DTYPE), scans[0], [0, len(scans[0])], [0.0])
    assert int(out["n_eff"][0]) > 0
