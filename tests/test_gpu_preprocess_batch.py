"""lk_preprocess_scans: voxel-grid down-sampling, time sort and buckets of a whole batch of raw scans in one device call.
Every scan's output must be bitwise what the oracle's single-scan preprocess gives (and so what lk_preprocess_scan gives),
the output must feed lk_scan_update exactly as a batch assembled on the host, errors must leave the handle usable, and a
call that fits the handle's scratch must not allocate."""
import ctypes as C
import functools
import gc

import numpy as np
import pytest

import lko
import scenes
from legkilo_b200 import Engine, LkError, abi, lib, synth

pytestmark = pytest.mark.gpu

CFG = abi.CONFIGS["leg_fusion"]


@pytest.fixture
def engine():
    """Engine factory whose handles are destroyed when the test ends, not whenever the garbage collector gets to them."""
    made = []

    def make(cfg):
        made.append(Engine(cfg))
        return made[-1]
    yield make
    for e in made:
        e.close()


@functools.lru_cache(maxsize=None)
def _pool():
    """Eight raw streaming scans of the box room, VLP-16 and OS64 alternating, at spread-out poses."""
    R, t = abi.extrinsics(CFG)
    sc = synth.BoxScene(ground_half_extent=20.0)
    rv, tv = synth.random_poses(8, 0.2, 2.0, stream=7000)
    return tuple(sc.scan(rotvec=rv[i], trans=tv[i], ext_R=R, ext_t=t, blind=1.5, stream=7001 + i, streaming=True,
                         **(synth.VLP16 if i % 2 == 0 else synth.OS64)) for i in range(8))


def _variant(i):
    """Pool scan i % 8, cut to a length of its own, with NaNs sprinkled at a stride and axis of its own."""
    s = _pool()[i % 8].copy()
    s = s[:len(s) - (i * 7919) % (len(s) // 2)]
    s[(i % 13)::389 + i, i % 3] = np.nan
    return s


def _specials():
    g = synth.rng(7100)
    nan_scan = g.uniform(-5, 5, (500, 4)).astype(np.float32)
    nan_scan[np.arange(500), g.integers(0, 3, 500)] = np.where(np.arange(500) % 2, np.nan, np.inf)
    one_curv = _pool()[1][:20000].copy()
    one_curv[:, 3] = np.float32(0.0625)  # a power of two: every centroid of it is exactly 0.0625 again
    return [np.zeros((0, 4), np.float32), nan_scan, np.array([[1.0, -2.0, 0.5, 0.01]], np.float32), one_curv]


def _batch(n_scans):
    if n_scans == 1:
        return [_variant(3)]
    sp = _specials()
    scans = [_variant(i) for i in range(n_scans - len(sp))]
    for k, s in enumerate(sp):  # in the middle of the batch, where the non-finite runs sit between valid leaves
        scans.insert(1 + k * (len(scans) // len(sp)), s)
    return scans


def _flat(scans):
    so = np.concatenate([[0], np.cumsum([len(s) for s in scans])]).astype(np.uint32)
    return np.concatenate(scans).astype(np.float32), so


def _host_batch(scans, leaf, begins):
    """The same batch laid out on the host from per-scan oracle results and synth.bucketize's times."""
    pts, so, sbp, bo, bt, bc = [], [0], [0], [], [], []
    for s, b in zip(scans, begins):
        p, offs, curv = lko.preprocess_scan(s, leaf)
        _, _, times = synth.bucketize(p, begin_time=float(b))
        bo.append(offs[:-1] + so[-1]); bt.append(times); bc.append(curv); pts.append(p)
        so.append(so[-1] + len(p)); sbp.append(sbp[-1] + len(curv))
    bo.append([so[-1]])
    return dict(pts=np.concatenate(pts), scan_offsets=np.array(so, np.uint32), scan_bucket_ptr=np.array(sbp, np.uint32),
                bucket_offsets=np.concatenate(bo).astype(np.uint32), bucket_times=np.concatenate(bt),
                bucket_curvature=np.concatenate(bc))


@pytest.mark.parametrize("n_scans", [1, 7, 130])
@pytest.mark.parametrize("leaf", [0.3, 0.5])
def test_bitwise_per_scan_against_oracle(leaf, n_scans, engine):
    scans = _batch(n_scans)
    pts, io = _flat(scans)
    begins = 1000.0 + 0.1 * np.arange(n_scans)
    got = engine(CFG).preprocess_scans(pts, io, leaf, begin_times=begins)
    so, sbp = got["scan_offsets"], got["scan_bucket_ptr"]
    assert len(so) == len(sbp) == n_scans + 1 and so[0] == sbp[0] == 0
    assert len(got["pts"]) == so[-1] and len(got["bucket_offsets"]) == sbp[-1] + 1
    for s, scan in enumerate(scans):
        ref_pts, ref_offs, ref_curv = lko.preprocess_scan(scan, leaf)
        a, b, ba, bb = int(so[s]), int(so[s + 1]), int(sbp[s]), int(sbp[s + 1])
        np.testing.assert_array_equal(got["pts"][a:b], ref_pts, err_msg=f"scan {s}")
        np.testing.assert_array_equal(got["bucket_offsets"][ba:bb + 1] - a, ref_offs, err_msg=f"scan {s}")
        np.testing.assert_array_equal(got["bucket_curvature"][ba:bb], ref_curv, err_msg=f"scan {s}")
        _, bz_offs, bz_times = synth.bucketize(ref_pts, begin_time=float(begins[s]))
        np.testing.assert_array_equal(bz_offs, ref_offs)
        np.testing.assert_array_equal(got["bucket_times"][ba:bb], bz_times, err_msg=f"scan {s}")
    if n_scans > 1:  # the special scans: empty, all NaN, one point, one curvature
        n_pts, n_b = np.diff(so), np.diff(sbp)
        sizes = [len(s) for s in scans]
        assert any(z == 0 and n == 0 for z, n in zip(sizes, n_pts))
        assert any(z == 500 and n == 0 and m == 0 for z, n, m in zip(sizes, n_pts, n_b))
        assert any(z == 1 and n == 1 and m == 1 for z, n, m in zip(sizes, n_pts, n_b))
        assert any(z == 20000 and n > 100 and m == 1 for z, n, m in zip(sizes, n_pts, n_b))
    # one call without bucket times gives the same points and buckets
    plain = engine(CFG).preprocess_scans(pts, io, leaf)
    assert plain["bucket_times"] is None
    for k in ("pts", "scan_offsets", "scan_bucket_ptr", "bucket_offsets", "bucket_curvature"):
        np.testing.assert_array_equal(plain[k], got[k], err_msg=k)


def test_single_scan_call_is_the_batch_of_one(engine):
    eng = engine(CFG)
    for i in (0, 1, 2):
        s = _variant(i)
        one = eng.preprocess_scan(s, 0.4)
        b = eng.preprocess_scans(s, [0, len(s)], 0.4)
        np.testing.assert_array_equal(one[0], b["pts"])
        np.testing.assert_array_equal(one[1], b["bucket_offsets"])
        np.testing.assert_array_equal(one[2], b["bucket_curvature"])


def test_offsets_need_not_start_at_zero(engine):
    scans = _batch(7)
    pts, io = _flat(scans)
    pad = np.full((37, 4), 123.0, np.float32)
    eng = engine(CFG)
    a = eng.preprocess_scans(pts, io, 0.5)
    b = eng.preprocess_scans(np.concatenate([pad, pts]), io + 37, 0.5)
    for k in ("pts", "scan_offsets", "scan_bucket_ptr", "bucket_offsets", "bucket_curvature"):
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def test_feeds_scan_update_like_a_host_assembled_batch(engine):
    batch = 5
    cfg, blob, scans = scenes.box_scene(batch=batch, streaming=True, stream0=7200)
    leaf = 0.5
    begins = 100.0 + 0.1 * np.arange(batch)
    pts, io = _flat(scans)
    eng = engine(cfg)
    eng.map_upload(blob)
    dev = eng.preprocess_scans(pts, io, leaf, begin_times=begins)
    host = _host_batch(scans, leaf, begins)
    for k in host:
        np.testing.assert_array_equal(dev[k], host[k], err_msg=k)
    assert (np.diff(dev["scan_bucket_ptr"]) > 20).all()
    x0 = abi.default_states(batch); P0 = abi.init_cov(batch); Q = abi.process_cov_Q(cfg)
    clk0 = np.zeros(batch, abi.CLOCK_DTYPE)
    clk0["last_predict_time"] = begins - 0.01; clk0["last_update_time"] = begins - 0.015
    outs = []
    for d in (dev, host):
        outs.append(eng.scan_update(x0, P0, Q, clk0, d["pts"], d["scan_offsets"], d["bucket_times"],
                                    scan_bucket_ptr=d["scan_bucket_ptr"], bucket_offsets=d["bucket_offsets"], iters=3))
    assert (outs[0]["n_eff"] > 0).all()
    for k in ("x", "P", "clk", "n_eff", "world"):
        assert np.asarray(outs[0][k]).tobytes() == np.asarray(outs[1][k]).tobytes(), k


def _raw_call(eng, n_scans, pts, io, leaf, begin, out):
    return lib().lk_preprocess_scans(eng.h, n_scans, _vp(pts), _vp(io), leaf, _vp(begin), *(_vp(out[k]) for k in (
        "pts", "so", "sbp", "bo", "bc", "bt")))


def _vp(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _out_buffers(n, n_scans, fill=0xA5):
    out = dict(pts=np.zeros((n, 4), np.float32), so=np.zeros(n_scans + 1, np.uint32), sbp=np.zeros(n_scans + 1, np.uint32),
               bo=np.zeros(n + 1, np.uint32), bc=np.zeros(n, np.float32), bt=np.zeros(n))
    for v in out.values():
        v.view(np.uint8)[...] = fill
    return out


def test_errors_leave_the_handle_usable(engine):
    eng = engine(CFG)
    good = _batch(7)
    gpts, gio = _flat(good)
    ref = eng.preprocess_scans(gpts, gio, 0.5)

    def still_works():
        again = eng.preprocess_scans(gpts, gio, 0.5)
        for k in ("pts", "scan_offsets", "scan_bucket_ptr", "bucket_offsets", "bucket_curvature"):
            np.testing.assert_array_equal(again[k], ref[k], err_msg=k)

    with pytest.raises(LkError) as e:
        eng.preprocess_scans(gpts, np.array([0, 10, 5, len(gpts)], np.uint32), 0.5)
    assert e.value.code == -1 and "monotone" in str(e.value)
    still_works()
    for leaf in (0.0, float("nan"), -0.3, float("inf")):
        with pytest.raises(LkError) as e:
            eng.preprocess_scans(gpts, gio, leaf)
        assert e.value.code == -1 and "leaf size" in str(e.value)
        still_works()
    # scan 1 spans 1 km x 1 km: at a 1 mm leaf its leaf index would overflow int32
    g = synth.rng(7300)
    wide = np.zeros((4000, 4), np.float32)
    wide[:, :2] = g.uniform(0, 1000, (4000, 2)); wide[:2, :2] = [[0, 0], [1000, 1000]]
    cube = [g.uniform(0, 1, (300, 4)).astype(np.float32) for _ in range(2)]  # 1 m cubes: 10^9 leaves, just fit
    bad = [cube[0], wide, cube[1]]
    bpts, bio = _flat(bad)
    with pytest.raises(LkError) as e:
        eng.preprocess_scans(bpts, bio, 1e-3)
    assert e.value.code == -1 and "scan 1" in str(e.value)
    still_works()
    # nothing is written by a refused call
    out = _out_buffers(len(bpts), 3)
    before = {k: v.copy() for k, v in out.items()}
    assert _raw_call(eng, 3, bpts, bio, 1e-3, np.zeros(3), out) == -1
    for k in out:
        assert out[k].tobytes() == before[k].tobytes(), k
    still_works()
    # NULL arguments; begin_times and bucket_times only together
    out = _out_buffers(len(gpts), 7)
    assert _raw_call(eng, 7, gpts, gio, 0.5, np.zeros(7), out) == 0
    assert _raw_call(eng, 7, None, gio, 0.5, None, {**out, "bt": None}) == -1
    assert _raw_call(eng, 7, gpts, gio, 0.5, np.zeros(7), {**out, "bt": None}) == -1
    assert _raw_call(eng, 7, gpts, gio, 0.5, None, out) == -1
    for k in ("pts", "so", "sbp", "bo", "bc"):
        assert _raw_call(eng, 7, gpts, gio, 0.5, None, {**out, k: None, "bt": None}) == -1, k
    assert lib().lk_preprocess_scans(None, 7, _vp(gpts), _vp(gio), C.c_float(0.5), None, *(
        _vp(out[k]) for k in ("pts", "so", "sbp", "bo", "bc")), None) == -1
    still_works()


def test_no_scans_and_no_points(engine):
    eng = engine(CFG)
    out = _out_buffers(1, 0)
    assert _raw_call(eng, 0, np.zeros((1, 4), np.float32), np.zeros(1, np.uint32), 0.5, None, {**out, "bt": None}) == 0
    assert out["so"][0] == 0 and out["sbp"][0] == 0 and out["bo"][0] == 0
    r = eng.preprocess_scans(np.zeros((0, 4), np.float32), [0, 0, 0], 0.5, begin_times=[1.0, 2.0])
    assert len(r["pts"]) == 0 and list(r["scan_offsets"]) == [0, 0, 0] and list(r["scan_bucket_ptr"]) == [0, 0, 0]
    assert list(r["bucket_offsets"]) == [0] and len(r["bucket_times"]) == 0
    with pytest.raises(ValueError):
        eng.preprocess_scans(np.zeros((0, 4), np.float32), [], 0.5)
    with pytest.raises(ValueError):
        eng.preprocess_scans(np.zeros((3, 4), np.float32), [0, 4], 0.5)


def test_a_call_that_fits_does_not_allocate(engine):
    import torch
    torch.cuda.init()
    scans = _batch(24)
    full, half = _flat(scans), _flat(scans[:12])
    eng = engine(CFG)
    calls = (("full", lambda: eng.preprocess_scans(*full, 0.3, begin_times=np.zeros(24))),
             ("half", lambda: eng.preprocess_scans(*half, 0.5)),
             ("one", lambda: eng.preprocess_scan(scans[5], 0.3)))
    first = [c() for _, c in calls]  # grows the scratch to the largest call and loads every kernel the calls use
    torch.cuda.synchronize()
    torch.cuda.mem_get_info()
    # device memory is freed by Engine.__del__: no collection may run between the reads
    gc.collect()
    gc.disable()
    try:
        free0, _ = torch.cuda.mem_get_info()
        again = []
        for name, c in calls:  # read after each call on its own: a smaller call must not shrink or regrow the scratch
            again.append(c())
            free, _ = torch.cuda.mem_get_info()
            assert free == free0, (name, free0, free)
    finally:
        gc.enable()
    for k in first[0]:
        np.testing.assert_array_equal(first[0][k], again[0][k], err_msg=k)
    for k in first[1]:
        np.testing.assert_array_equal(first[1][k], again[1][k], err_msg=k)
    a, b = int(first[0]["scan_offsets"][5]), int(first[0]["scan_offsets"][6])
    np.testing.assert_array_equal(again[2][0], first[0]["pts"][a:b])
