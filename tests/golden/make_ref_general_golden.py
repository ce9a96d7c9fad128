"""Writes tests/golden/ref_general_*.npz from the reference itself (oracle/_ref/liblkref.so, see make_ref_golden.py), at
general priors: the first-frame map is built from a general pose G (tens of degrees about every axis, keys negative on
some axes), the prior composes G with a small perturbation, and P0 is dense and SPD with attitude / position blocks large
enough that the state term of sigma_l matters (tests/general_prior.py). Writes only new files; the other fixtures are
untouched.

  ref_general_bucket_<cfg>.npz      one KILO::predictUpdatePoint bucket with UpdateVoxelMap (leg_fusion; hilti has a
                                    non-identity extrinsic rotation)
  ref_general_bucket_asym.npz       the leg_fusion bucket with P0 plus a skew part of 1e-6 of its largest entry; the
                                    generator asserts that the skew part changes the reference's output
  ref_general_bucket_far.npz        the leg_fusion bucket with the scene around (1.8e3, -2.6e3, 35) m
  ref_general_stream_<kind>.npz     one KILO::process frame with the inertial (imu) or kinematic-inertial (kin) queue
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in ("leg-kilo_b200/python", "oracle", "tests"):
    sys.path.insert(0, os.path.join(ROOT, p))
import general_prior as gp  # noqa: E402
import lkref  # noqa: E402
import mapcmp  # noqa: E402
import scenes  # noqa: E402
from legkilo_b200 import abi, synth  # noqa: E402

G = synth.exp_so3(gp.G_ROTVEC)
# (state_err, cov_err) by which the reference's output for the skewed P0 must differ from its output for the symmetric part
# (measured: 2.7e-4 sd, 1.2e-3)
SKEW_SEEN = (1e-5, 1e-4)


def _reference(cfg, pw, pb, imu_mode_only=True):
    r = lkref.Reference(cfg, imu_mode_only=imu_mode_only, gravity=9.81, acc_norm=9.79)
    rot_cov, pos_cov = gp.map_covs(G)
    r.build_voxel_map(pw, pb, R=G, rot_cov=rot_cov, pos_cov=pos_cov)
    return r


def bucket(cfg_name, pos=gp.G_POS, asym=False):
    cfg = abi.CONFIGS[cfg_name]
    sc, pw, pb = gp.map_cloud(cfg, G, pos)
    scan = gp.room_scan(cfg, sc, 9100, False)
    g = synth.rng(9150)
    x0 = gp.prior_at(G, pos, g)
    P0 = gp.dense_cov(g)
    if asym:
        P0 = gp.skewed(P0, g)
    clk = np.zeros(1, abi.CLOCK_DTYPE); clk["last_predict_time"] = 99.99; clk["last_update_time"] = 99.985
    pts = np.ascontiguousarray(scan[:500])

    def run(P):
        r = _reference(cfg, pw, pb)
        map0 = mapcmp.digest(r.map_export())
        r.set_filter(x0, P, abi.process_cov_Q(cfg), clk)
        out = r.predict_update_point(100.0, pts)
        return r, map0, out

    r, map0, out = run(P0)
    assert out["n_eff"] > 300, out["n_eff"]
    x, P, _, c = r.get_filter()
    if asym:  # the skew part must be observable in the reference's own output
        Psym = 0.5 * (P0.reshape(30, 30) + P0.reshape(30, 30).T)
        rs, _, _ = run(Psym.ravel())
        xs, Ps, _, _ = rs.get_filter()
        es, eP = scenes.state_err(xs, x, P), scenes.cov_err(Ps, P)
        assert es > SKEW_SEEN[0] and eP > SKEW_SEEN[1], (es, eP)
    name = "asym" if asym else ("far" if pos is gp.FAR_POS else cfg_name)
    np.savez_compressed(os.path.join(HERE, f"ref_general_bucket_{name}.npz"), pw=pw, pb=pb, map0=map0, x0=x0.view(np.float64),
                        P0=P0, clk0=clk.view(np.float64), t=100.0, pts=pts, x=x.view(np.float64), P=P, clk=c.view(np.float64),
                        world=out["world"], n_eff=out["n_eff"], map1=mapcmp.digest(r.map_export()))
    return out["n_eff"]


def stream(kind):
    cfg = abi.CONFIGS["leg_fusion"]
    sc, pw, pb = gp.map_cloud(cfg, G, gp.G_POS)
    scan = gp.room_scan(cfg, sc, 9200, True)
    g = synth.rng(9251)
    x0 = gp.prior_at(G, gp.G_POS, g)
    P0 = gp.dense_cov(g)
    clk = np.zeros(1, abi.CLOCK_DTYPE); clk["last_predict_time"] = 19.995; clk["last_update_time"] = 19.995
    meas = (synth.imu_stream if kind == "imu" else synth.kinimu_stream)(19.996, 20.13)

    def run(P):
        r = _reference(cfg, pw, pb, imu_mode_only=(kind == "imu"))
        map0 = mapcmp.digest(r.map_export())
        r.set_filter(x0, P, abi.process_cov_Q(cfg), clk)
        return r, map0, r.process(20.0, 20.1, scan, **{kind: meas})

    r, map0, out = run(P0)
    assert out["ok"] and out["n_eff"] > 0.5 * len(scan), (out["n_eff"], len(scan))
    x, P, _, c = r.get_filter()
    # At a dense prior, the map update makes a frame of ~50 buckets sensitive: a change of 1e-15 in P0 moves the final
    # state of the reference itself by up to a few 1e-7 of the update step (without UpdateVoxelMap, by 1e-16). The
    # tests compare these fixtures to STREAM_TOLS; the generator checks that three such perturbations stay well inside it.
    for s in (9297, 9298, 9299):
        Pp = P0 * (1.0 + 1e-15 * synth.rng(s).standard_normal(900))
        rp, _, _ = run((0.5 * (Pp.reshape(30, 30) + Pp.reshape(30, 30).T)).ravel())
        xp, Ppp, _, _ = rp.get_filter()
        spread = scenes.state_err(xp, x, P), scenes.cov_err(Ppp, P)
        assert spread[0] < gp.STREAM_TOLS[0] / 4 and spread[1] < gp.STREAM_TOLS[1] / 4, spread
    np.savez_compressed(os.path.join(HERE, f"ref_general_stream_{kind}.npz"), pw=pw, pb=pb, map0=map0, x0=x0.view(np.float64), P0=P0,
                        clk0=clk.view(np.float64), begin=20.0, pts=out["body"], meas=meas.view(np.uint8), x=x.view(np.float64), P=P,
                        clk=c.view(np.float64), world=out["world"], n_eff=out["n_eff"], map1=mapcmp.digest(r.map_export()))
    return out["n_eff"]


if __name__ == "__main__":
    for args in (("leg_fusion",), ("hilti",), ("leg_fusion", gp.G_POS, True), ("leg_fusion", gp.FAR_POS)):
        print("bucket", args[0], "n_eff", bucket(*args))
    for kind in ("imu", "kin"):
        print("stream", kind, "n_eff", stream(kind))
    print("reference-made general-prior fixtures written")
