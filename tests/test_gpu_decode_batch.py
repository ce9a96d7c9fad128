"""lk_decode_pointcloud2s: PointCloud2 decode of a whole batch of messages in one device call. Every message must be
bitwise what the oracle gives for it alone (points, intensity, offsets, begin / end times), the device must match the
reference-made fixture, the output must chain into lk_preprocess_scans exactly as per-message decodes stitched on the
host, errors must leave the handle usable, and a call that fits the handle's scratch must not allocate."""
import ctypes as C
import functools
import gc

import numpy as np
import pytest

import decode_cases
import lko_decode
from legkilo_b200 import Engine, abi, lib, synth
from test_decode_oracle import GOLDEN, assert_decode_equal

pytestmark = pytest.mark.gpu

CFG = abi.CONFIGS["leg_fusion"]
BLIND, FILTER = 1.5, 3


@pytest.fixture
def engine():
    """Engine factory whose handles are destroyed when the test ends, not whenever the garbage collector gets to them."""
    made = []

    def make():
        made.append(Engine(CFG))
        return made[-1]
    yield make
    for e in made:
        e.close()


@functools.lru_cache(maxsize=None)
def _pool(lt):
    msgs, _ = synth.box_pointcloud2s(8, lt, distinct=8, stream=9700 + 20 * lt)
    return tuple(msgs)


def _specials(lt):
    """An empty message, one point, all inside the blind sphere, shorter than FILTER, all NaN."""
    a = _pool(lt)[0]
    near = a[:300].copy()
    near["x"], near["y"], near["z"] = 0.5, -0.25, 0.125
    nan = a[:200].copy()
    nan["x"] = np.nan
    return [a[:0].copy(), a[7:8].copy(), near, a[100:102].copy(), nan]


def _batch(lt, n_msgs):
    """Pool message m % 8 cut to a length of its own, with the special messages spread through the batch."""
    pool = _pool(lt)
    msgs = [pool[m % 8][(m * 613) % 5000:len(pool[m % 8]) - (m * 7919) % 9000].copy() for m in range(n_msgs)]
    if n_msgs > 1:
        for k, s in enumerate(_specials(lt)):
            msgs[(1 + k * (n_msgs // 5 + 1)) % n_msgs] = s
    stamps = 1.7e9 + 0.1 * np.arange(n_msgs) + 0.013
    return msgs, stamps


def _oracle(msg, lt, stamp, blind=BLIND, fn=FILTER, layout=None, ts=None):
    layout = abi.pc2_layout(lt) if layout is None else layout
    ts = synth.PC2_TIME_SCALE[lt] if ts is None else ts
    if len(msg) == 0:
        return np.zeros((0, 4), np.float32), np.zeros(0, np.float32), np.nan, np.nan
    return lko_decode.decode_pointcloud2(msg.view(np.uint8), layout, blind, fn, ts, stamp)


def _check_batch(got, msgs, refs):
    offs = got["offsets"]
    assert len(offs) == len(msgs) + 1 and offs[0] == 0 and offs[-1] == len(got["pts"])
    for m, ref in enumerate(refs):
        a, b = int(offs[m]), int(offs[m + 1])
        assert_decode_equal((got["pts"][a:b], got["intensity"][a:b], got["begin_times"][m], got["end_times"][m]), ref)


@pytest.mark.parametrize("lt", [1, 2, 3])
@pytest.mark.parametrize("n_msgs", [1, 7, 300])
def test_every_message_equals_the_oracle(engine, lt, n_msgs):
    msgs, stamps = _batch(lt, n_msgs)
    got = engine().decode_pointcloud2s(msgs, abi.pc2_layout(lt), BLIND, FILTER, synth.PC2_TIME_SCALE[lt], stamps=stamps)
    _check_batch(got, msgs, [_oracle(m, lt, s) for m, s in zip(msgs, stamps)])
    if n_msgs > 1:
        empty = np.array([len(m) == 0 for m in msgs])
        assert empty.any() and (np.isnan(got["begin_times"]) == empty).all()
        assert np.isnan(got["pts"][:, 0]).any() and len(got["pts"]) > 1000


def test_stamps_none_is_stamp_zero(engine):
    msgs, _ = _batch(2, 7)
    eng = engine()
    a = eng.decode_pointcloud2s(msgs, abi.pc2_layout(2), BLIND, 1, synth.PC2_TIME_SCALE[2])
    b = eng.decode_pointcloud2s(msgs, abi.pc2_layout(2), BLIND, 1, synth.PC2_TIME_SCALE[2], stamps=np.zeros(7))
    for k in a:
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def test_device_matches_reference_fixture(engine):
    z = np.load(GOLDEN)
    eng = engine()
    for name in [m[0] for m in decode_cases.messages()]:
        layout = decode_cases.layout_of(z[f"{name}__layout"])
        data, ts, stamp = z[f"{name}__data"], float(z[f"{name}__time_scale"]), float(z[f"{name}__stamp"])
        for c, (blind, fn) in enumerate(decode_cases.COMBOS):
            ref = (z[f"{name}__{c}__pts"], z[f"{name}__{c}__intensity"], *z[f"{name}__{c}__times"])
            # the message three times over in one call, each copy at its own stamp (Hesai ignores stamps)
            got = eng.decode_pointcloud2s([data] * 3, layout, blind, fn, ts, stamps=[stamp, stamp, stamp])
            _check_batch(got, [data] * 3, [ref] * 3)


@pytest.mark.parametrize("lt", [1, 2])
def test_chains_into_preprocess_scans(engine, lt):
    """decode_pointcloud2s -> preprocess_scans(offsets, begin_times) against one decode per message, offsets and begin
    times stitched on the host, then preprocess_scans."""
    msgs, stamps = _batch(lt, 24)
    keep = [i for i, m in enumerate(msgs) if len(m)]  # the empty message's NaN begin time is never read, but keep it out
    msgs, stamps = [msgs[i] for i in keep], stamps[keep]
    layout, ts = abi.pc2_layout(lt), synth.PC2_TIME_SCALE[lt]
    eng = engine()
    d = eng.decode_pointcloud2s(msgs, layout, BLIND, 1, ts, stamps=stamps)
    batch = eng.preprocess_scans(d["pts"], d["offsets"], 0.3, begin_times=d["begin_times"])
    pts, begin = [], []
    for m, s in zip(msgs, stamps):
        p, _, first, _ = eng.decode_pointcloud2(m.view(np.uint8), layout, BLIND, 1, ts)
        pts.append(p)
        begin.append(s + first)
    io = np.concatenate([[0], np.cumsum([len(p) for p in pts])]).astype(np.uint32)
    host = eng.preprocess_scans(np.concatenate(pts), io, 0.3, begin_times=np.array(begin))
    for k in host:
        np.testing.assert_array_equal(batch[k], host[k], err_msg=k)
    assert len(batch["bucket_times"]) > 100


@pytest.mark.parametrize("lt", [1, 2, 3])
def test_single_message_call_is_the_batch_of_one(engine, lt):
    msg = _pool(lt)[3]
    eng = engine()
    one = eng.decode_pointcloud2(msg.view(np.uint8), abi.pc2_layout(lt), BLIND, FILTER, synth.PC2_TIME_SCALE[lt])
    b = eng.decode_pointcloud2s([msg], abi.pc2_layout(lt), BLIND, FILTER, synth.PC2_TIME_SCALE[lt])
    assert_decode_equal(one, (b["pts"], b["intensity"], b["begin_times"][0], b["end_times"][0]))
    # n_points == 0 returns at once, times untouched
    ft, lt_, no = C.c_double(-7.0), C.c_double(-8.0), C.c_uint32(99)
    assert lib().lk_decode_pointcloud2(eng.h, None, 0, C.byref(abi.pc2_layout(lt)), BLIND, FILTER, 1.0, None, None,
                                       C.byref(no), C.byref(ft), C.byref(lt_)) == 0
    assert no.value == 0 and ft.value == -7.0 and lt_.value == -8.0


def _raw_call(eng, n_msgs, ptrs, counts, layout, filter_num=1, out_offs=None, pts=None):
    return lib().lk_decode_pointcloud2s(eng.h, n_msgs, ptrs, counts, None, C.byref(layout) if layout is not None else None,
                                        0.0, filter_num, 1.0, pts, None, out_offs, None, None)


def test_argument_errors_leave_the_handle_usable(engine):
    eng = engine()
    lay = abi.pc2_layout(1)
    msg = _pool(1)[0][:64].copy()
    buf = msg.view(np.uint8)
    pts = np.zeros((128, 4), np.float32)
    offs = np.full(3, 12345, np.uint32)
    good_ptrs = (C.c_void_p * 2)(buf.ctypes.data, buf.ctypes.data)
    counts = np.array([64, 64], np.uint32)
    P = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    bad_lay = abi.pc2_layout(1); bad_lay.off_time = bad_lay.point_step - 2
    huge = np.array([2 ** 31, 2 ** 31], np.uint32)  # a uint32 sum wraps to 0
    over = np.array([2 ** 31 - 1, 1], np.uint32)
    cases = [
        ("null out_offsets", lambda: _raw_call(eng, 2, good_ptrs, P(counts), lay, pts=P(pts))),
        ("null layout", lambda: _raw_call(eng, 2, good_ptrs, P(counts), None, out_offs=P(offs), pts=P(pts))),
        ("null data", lambda: _raw_call(eng, 2, None, P(counts), lay, out_offs=P(offs), pts=P(pts))),
        ("null data[1]", lambda: _raw_call(eng, 2, (C.c_void_p * 2)(buf.ctypes.data, None), P(counts), lay, out_offs=P(offs),
                                           pts=P(pts))),
        ("filter_num 0", lambda: _raw_call(eng, 2, good_ptrs, P(counts), lay, filter_num=0, out_offs=P(offs), pts=P(pts))),
        ("layout", lambda: _raw_call(eng, 2, good_ptrs, P(counts), bad_lay, out_offs=P(offs), pts=P(pts))),
        ("2^31 + 2^31", lambda: _raw_call(eng, 2, good_ptrs, P(huge), lay, out_offs=P(offs), pts=P(pts))),
        ("INT_MAX + 1", lambda: _raw_call(eng, 2, good_ptrs, P(over), lay, out_offs=P(offs), pts=P(pts))),
    ]
    ref = eng.decode_pointcloud2s([msg, msg], lay, 0.0, 1, 1.0)
    for name, call in cases:
        assert call() == -1, name  # LK_ERR_INVALID_ARG
        assert (offs == 12345).all(), name  # nothing written
        got = eng.decode_pointcloud2s([msg, msg], lay, 0.0, 1, 1.0)
        for k in ref:
            np.testing.assert_array_equal(got[k], ref[k], err_msg=name)
    assert _raw_call(eng, 2, good_ptrs, P(huge), lay, out_offs=P(offs), pts=P(pts)) == -1
    assert "INT_MAX" in lib().lk_last_error(eng.h).decode()
    # no messages: out_offsets[0] = 0
    offs[:] = 12345
    assert _raw_call(eng, 0, None, None, lay, out_offs=P(offs)) == 0 and offs[0] == 0
    with pytest.raises(ValueError):
        eng.decode_pointcloud2s([buf[:-1]], lay, 0.0, 1, 1.0)
    with pytest.raises(ValueError):
        eng.decode_pointcloud2s([msg, msg], lay, 0.0, 1, 1.0, stamps=[1.0])


def test_a_call_that_fits_does_not_allocate(engine):
    import torch
    torch.cuda.init()
    lt = 1
    layout, ts = abi.pc2_layout(lt), synth.PC2_TIME_SCALE[lt]
    msgs, stamps = _batch(lt, 40)
    eng = engine()
    singles = [m.view(np.uint8) for m in msgs[:6]]
    calls = (("full", lambda: eng.decode_pointcloud2s(msgs, layout, BLIND, FILTER, ts, stamps=stamps)),
             ("half", lambda: eng.decode_pointcloud2s(msgs[:20], layout, 0.0, 1, ts)),
             ("singles", lambda: [eng.decode_pointcloud2(s, layout, BLIND, FILTER, ts) for s in singles]))
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
    for i in (0, 1):
        for k in first[i]:
            np.testing.assert_array_equal(first[i][k], again[i][k], err_msg=k)
    for a, b in zip(first[2], again[2]):
        assert_decode_equal(a, b)
