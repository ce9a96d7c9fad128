"""lk_leg_kinematics: unitree leg states -> kinematic-inertial samples (Kinematics, kinematics.{h,cc}, and the redundancy
drop of RosInterface::kinematicImuCallBack, ros_interface.cc:221-248).

CPU: struct layouts; the restatement (oracle/lko_leg.py) against the reference's own kinematics.cc (oracle/lkref_leg.py,
skipped without it) and against the fixture made from it (tests/golden/ref_leg_kinematics.npz).
GPU: the device path against the restatement and the fixture, track carry across calls, a many-tile stream, edge cases,
and three streaming scans in Kin+IMU mode through lk_process_scan."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

import lko
import lko_leg
import lkref_leg
import scenes
from legkilo_b200 import HEADER_PATH, Engine, LkError, abi, lib, synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_leg_kinematics.npz")
EXACT = ("stamp", "contact", "acc", "gyr")


def _cfg_with(base, **kw):
    c = dict(abi.CONFIGS[base])
    c.update(kw)
    return c


def _track_bytes(t):
    return C.string_at(C.addressof(t), C.sizeof(t))


def _track(contacts, acc_z=0.0, gyr_z=0.0):
    return abi.LkLegTrack((C.c_int32 * 4)(*contacts), acc_z, gyr_z)


def _assert_same(a, b, fk_tol=None):
    """Bitwise on n_out, stamps, contacts, acc, gyr; foot_pos / foot_vel bitwise (fk_tol None) or within
    fk_tol * max(1, |v|)."""
    assert len(a) == len(b)
    for f in EXACT:
        assert a[f].tobytes() == b[f].tobytes(), f
    for f in ("foot_pos", "foot_vel"):
        if fk_tol is None:
            assert a[f].tobytes() == b[f].tobytes(), f
        else:
            err = np.abs(a[f] - b[f]) / np.maximum(1.0, np.abs(b[f]))
            assert err.max(initial=0.0) <= fk_tol, (f, err.max())


def _edge_stream(cfg, n=400, stream=5):
    """Forces exactly at each threshold and on either side of them; the first message's acc.z and gyr.z both 0."""
    s = synth.leg_state_stream(1.0, 1.0 + n / 500.0, 500.0, "leg_fusion", stream)
    up, down = cfg["contact_force_threshold_up"], cfg["contact_force_threshold_down"]
    g = synth.rng(stream + 1000)
    choices = np.array([up, down, up - 1, up + 1, down - 1, down + 1, 0, 2 * max(up, down)])
    s["foot_force"] = choices[g.integers(0, len(choices), size=(len(s), 4))].astype(np.int16)
    s["acc"][0, 2] = 0.0
    s["gyr"][0, 2] = 0.0
    return s


LEG_CFGS = ["leg_fusion", "diter", "hilti", "nclt"]


# ---- CPU ----------------------------------------------------------------------------------------------------------

def test_struct_layouts_match_header():
    hdr = open(HEADER_PATH).read()
    for tag, size in (("lk_leg_cfg; /* 56 B */", 56), ("lk_leg_state; /* 136 B */", 136), ("lk_leg_track; /* 24 B */", 24)):
        assert tag in hdr
    assert C.sizeof(abi.LkLegCfg) == 56 and [f for f, _ in abi.LkLegCfg._fields_] == re.findall(
        r"double (\w+);", hdr[hdr.index("typedef struct lk_leg_cfg"):hdr.index("} lk_leg_cfg;")])
    assert abi.LEG_STATE_DTYPE.itemsize == 136
    assert {k: v[1] for k, v in abi.LEG_STATE_DTYPE.fields.items()} == dict(stamp=0, acc=8, gyr=20, q=32, dq=80, foot_force=128)
    assert C.sizeof(abi.LkLegTrack) == 24 and abi.LkLegTrack.last_acc_z.offset == 16 and abi.LkLegTrack.last_gyr_z.offset == 20


def test_track_default_is_the_reference_initial_state():
    t = abi.LkLegTrack()
    assert lib().lk_leg_track_default(C.byref(t)) == 0
    assert _track_bytes(t) == _track_bytes(abi.leg_track_default())
    assert list(t.in_contact) == [1, 1, 1, 1] and t.last_acc_z == 0.0 and t.last_gyr_z == 0.0


needs_ref = pytest.mark.skipif(not lkref_leg.available(), reason="needs oracle/_ref/liblkref_leg.so or the reference sources")


@needs_ref
@pytest.mark.parametrize("cfg_name", LEG_CFGS)
@pytest.mark.parametrize("redundancy", [True, False])
def test_oracle_matches_reference_stream(cfg_name, redundancy):
    cfg = abi.CONFIGS[cfg_name]
    s = synth.leg_state_stream(5.0, 7.0, 500.0, cfg_name, 60 + LEG_CFGS.index(cfg_name))
    ko, to = lko_leg.leg_kinematics(s, cfg, redundancy=redundancy)
    kr, tr = lkref_leg.leg_kinematics(s, cfg, redundancy=redundancy)
    assert (len(ko) < len(s)) == redundancy
    _assert_same(ko, kr, fk_tol=1e-14)
    assert _track_bytes(to) == _track_bytes(tr)


@needs_ref
@pytest.mark.parametrize("thresholds", [(220.0, 200.0), (40.0, 60.0), (50.0, 50.0)], ids=["up>down", "up<down", "up==down"])
def test_oracle_matches_reference_at_thresholds(thresholds):
    cfg = _cfg_with("leg_fusion", contact_force_threshold_up=thresholds[0], contact_force_threshold_down=thresholds[1])
    s = _edge_stream(cfg)
    ko, to = lko_leg.leg_kinematics(s, cfg)
    kr, tr = lkref_leg.leg_kinematics(s, cfg)
    assert len(ko) < len(s) and ko["stamp"][0] == s["stamp"][1]  # the zero first message equals the zero "previous" one
    _assert_same(ko, kr, fk_tol=1e-14)
    assert _track_bytes(to) == _track_bytes(tr)
    assert 0 < ko["contact"].mean() < 1


def test_oracle_contact_detector_semantics():
    """kinematics.h:16-22 with up < down (diter.yaml:50-51): a force held in (up, down) flips the detector every sample."""
    cfg = _cfg_with("leg_fusion", contact_force_threshold_up=40.0, contact_force_threshold_down=60.0)
    s = synth.leg_state_stream(0.0, 0.02, 500.0, "leg_fusion", 3)
    s["acc"][:, 2] = np.arange(len(s)) + 1.0  # nothing redundant
    s["foot_force"] = 50
    k, t = lko_leg.leg_kinematics(s, cfg)
    assert len(k) == len(s)
    assert (k["contact"][:, 0] == np.arange(len(s)) % 2).all()  # in contact -> 50 < 60 off -> 50 > 40 on -> ...
    assert list(t.in_contact) == [int(len(s) % 2 == 0)] * 4


def test_oracle_matches_reference_golden():
    d = np.load(GOLDEN)
    for name in ("leg_fusion", "diter"):
        s = d[f"{name}_states"].view(abi.LEG_STATE_DTYPE)
        ko, to = lko_leg.leg_kinematics(s, abi.CONFIGS[name])
        _assert_same(ko, d[f"{name}_kin"].view(abi.KINIMU_DTYPE), fk_tol=1e-14)
        assert _track_bytes(to) == d[f"{name}_track"].tobytes()


# ---- GPU ----------------------------------------------------------------------------------------------------------

FK_TOL = 1e-12
# three streaming scans with map updates, the device filter carried from scan to scan, against the oracle's
# (tests/scenes.py; worst measured on an H100 80GB HBM3: 5.2e-9 sd, 4.1e-12)
KIN_CHAIN_STATE_TOL = 5e-7
KIN_CHAIN_COV_TOL = 4e-10


@pytest.fixture(scope="module")
def eng():
    e = Engine(abi.CONFIGS["leg_fusion"])
    yield e
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name", ["leg_fusion", "diter"])
@pytest.mark.parametrize("redundancy", [True, False])
def test_gpu_matches_oracle(eng, cfg_name, redundancy):
    cfg = abi.CONFIGS[cfg_name]
    s = synth.leg_state_stream(5.0, 9.0, 500.0, cfg_name, 70)
    tr0 = _track([1, 0, 0, 1], float(s["acc"][0, 2]), 0.25)
    kg, tg = eng.leg_kinematics(s, cfg, track=tr0, redundancy=redundancy)
    ko, to = lko_leg.leg_kinematics(s, cfg, track=tr0, redundancy=redundancy)
    _assert_same(kg, ko, fk_tol=FK_TOL)
    assert _track_bytes(tg) == _track_bytes(to)


@pytest.mark.gpu
def test_gpu_matches_reference_golden(eng):
    d = np.load(GOLDEN)
    for name in ("leg_fusion", "diter"):
        s = d[f"{name}_states"].view(abi.LEG_STATE_DTYPE)
        kg, tg = eng.leg_kinematics(s, abi.CONFIGS[name])
        _assert_same(kg, d[f"{name}_kin"].view(abi.KINIMU_DTYPE), fk_tol=FK_TOL)
        assert _track_bytes(tg) == d[f"{name}_track"].tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("parts", [1, 2, 7, 50])
def test_gpu_split_calls_carry_the_track(eng, parts):
    cfg = abi.CONFIGS["diter"]
    s = synth.leg_state_stream(2.0, 3.0, 500.0, "diter", 71)
    whole, tw = eng.leg_kinematics(s, cfg)
    cuts = np.linspace(0, len(s), parts + 1).astype(int)
    pieces, tr = [], None
    for a, b in zip(cuts[:-1], cuts[1:]):
        k, tr = eng.leg_kinematics(s[a:b], cfg, track=tr)
        pieces.append(k)
    joined = np.concatenate(pieces)
    assert joined.tobytes() == whole.tobytes()
    assert _track_bytes(tr) == _track_bytes(tw)


@pytest.mark.gpu
def test_gpu_many_tiles_match_oracle(eng):
    cfg = abi.CONFIGS["leg_fusion"]
    s = synth.leg_state_stream(0.0, 1000.0, 500.0, "leg_fusion", 72)
    assert len(s) == 500_000
    kg, tg = eng.leg_kinematics(s, cfg)
    ko, to = lko_leg.leg_kinematics(s, cfg)
    assert 0.5 * len(s) < len(kg) < len(s)
    _assert_same(kg, ko, fk_tol=FK_TOL)
    assert _track_bytes(tg) == _track_bytes(to)


@pytest.mark.gpu
def test_gpu_edge_cases(eng):
    cfg = abi.CONFIGS["leg_fusion"]
    s = synth.leg_state_stream(0.0, 0.2, 500.0, "leg_fusion", 73)
    # n = 0: nothing written, the track unchanged
    tr0 = _track([0, 1, 0, 1], 1.5, -2.5)
    k, t = eng.leg_kinematics(s[:0], cfg, track=tr0)
    assert len(k) == 0 and _track_bytes(t) == _track_bytes(tr0)
    # every message dropped: contacts unchanged, the last raw z pair taken
    d = s.copy(); d["acc"][:, 2] = 1.5; d["gyr"][:, 2] = -2.5
    k, t = eng.leg_kinematics(d, cfg, track=tr0)
    assert len(k) == 0 and _track_bytes(t) == _track_bytes(tr0)
    # redundancy off keeps every message, still tracks the last raw z pair
    k, t = eng.leg_kinematics(d, cfg, track=tr0, redundancy=False)
    ko, to = lko_leg.leg_kinematics(d, cfg, track=tr0, redundancy=False)
    assert len(k) == len(d)
    _assert_same(k, ko, fk_tol=FK_TOL)
    assert _track_bytes(t) == _track_bytes(to)
    # null arguments and a non-finite configuration
    L = lib()
    lc = abi.leg_cfg(cfg); tr = abi.leg_track_default(); no = C.c_uint32(7)
    out = np.zeros(len(s), abi.KINIMU_DTYPE)
    sp, op = s.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)
    n = len(s)
    assert L.lk_leg_kinematics(None, C.byref(lc), sp, n, 1, C.byref(tr), op, C.byref(no)) == -1
    assert L.lk_leg_kinematics(eng.h, None, sp, n, 1, C.byref(tr), op, C.byref(no)) == -1
    assert L.lk_leg_kinematics(eng.h, C.byref(lc), None, n, 1, C.byref(tr), op, C.byref(no)) == -1
    assert L.lk_leg_kinematics(eng.h, C.byref(lc), sp, n, 1, None, op, C.byref(no)) == -1
    assert L.lk_leg_kinematics(eng.h, C.byref(lc), sp, n, 1, C.byref(tr), None, C.byref(no)) == -1
    assert L.lk_leg_kinematics(eng.h, C.byref(lc), sp, n, 1, C.byref(tr), op, None) == -1
    assert L.lk_leg_track_default(None) == -1
    for field in ("leg_offset_x", "leg_thigh_length", "contact_force_threshold_down"):
        for bad in (math.nan, math.inf):
            bc = abi.leg_cfg(cfg); setattr(bc, field, bad)
            with pytest.raises(LkError) as e:
                eng.leg_kinematics(s, bc)
            assert e.value.code == -1
    assert _track_bytes(tr) == _track_bytes(abi.leg_track_default())
    # the handle still works after the refusals
    k, t = eng.leg_kinematics(s, cfg)
    assert len(k) > 0


@pytest.mark.gpu
def test_gpu_three_streaming_scans_kin_imu_mode():
    """Leg states -> lk_leg_kinematics -> lk_process_scan over three consecutive scans, the leg track and the
    unconsumed samples carried from scan to scan; the oracle's kinematics then lko_process_scan alongside."""
    cfg, blob, scans = scenes.box_scene(batch=3, streaming=True, stream0=1300)
    Q = abi.process_cov_Q(cfg)
    x0 = abi.default_states(1)
    x0["vel"][0] = (0.4, -0.2, 0.05); x0["imu_a"][0] = (0.3, 0.1, 9.7); x0["imu_w"][0] = (0.02, -0.03, 0.15)
    P0 = abi.init_cov(1)
    clk = np.zeros(1, abi.CLOCK_DTYPE); clk["last_predict_time"] = 19.995; clk["last_update_time"] = 19.995
    states = synth.leg_state_stream(19.996, 20.33, 500.0, "leg_fusion", 74)

    o = lko.Oracle(cfg); o.map_import(blob); o.set_filter(x0, P0, Q, clk)
    o.set_options(gain_mode=lko.GAIN_INFORMATION, update_map=True, imu_mode_only=False, gravity=9.81, acc_norm=9.79)
    eng = Engine(cfg); eng.map_upload(blob)
    x, P, c = x0, P0, clk
    tg = to = None
    qg = qo = np.zeros(0, abi.KINIMU_DTYPE)
    edges = (0.0, 20.1, 20.2, 20.3)  # the messages that arrive while scan k is taken
    for k in range(3):
        t0 = 20.0 + 0.1 * k
        seg = states[(states["stamp"] > edges[k]) & (states["stamp"] <= edges[k + 1])]
        kg, tg = eng.leg_kinematics(seg, cfg, track=tg)
        ko, to = lko_leg.leg_kinematics(seg, cfg, track=to)
        assert _track_bytes(tg) == _track_bytes(to) and len(kg) == len(ko) > 20
        qg = np.concatenate([qg, kg]); qo = np.concatenate([qo, ko])
        pts, offs, times = synth.bucketize(scans[k], begin_time=t0)
        ro = o.process_scan(t0, pts, kin=qo)
        out = eng.process_scan(x, P, Q, c, pts, offs, times, kin=qg, gravity=9.81, acc_norm=9.79, update_map=True)
        assert out["n_consumed"] == ro["n_consumed"] > 20 and out["n_eff"] == ro["n_eff"] > 0
        qg = qg[out["n_consumed"]:]; qo = qo[ro["n_consumed"]:]
        x, P, c = out["x"], out["P"], out["clk"]
        xo, Po, _, co = o.get_filter()
        scenes.check_filter(x, P, xo, Po, KIN_CHAIN_STATE_TOL, KIN_CHAIN_COV_TOL, f"scan {k}")
    eng.close()
