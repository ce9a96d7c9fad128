"""Inputs of lk_map_insert shared by tests/golden/make_ref_map_insert_golden.py (fixtures made by the reference),
tests/test_map_insert_oracle.py (oracle on CPU) and tests/test_gpu_map_insert.py (device).

A case is a dict of the call's buffers (pts, set_offsets, rot, pos, rot_cov, pos_cov) plus, when it inserts on top of a
map, the first-frame cloud (pw, pb) that map is built from with BuildVoxelMap at the general pose G:
  room_empty    box-room scans at general poses (tests/general_prior.py) with dense covariance blocks, into an empty map;
  room_on_blob  the same kind of trajectory on top of the box room's first-frame map;
  cluttered     volumetric clutter and a dense slab, split over three sets: roots cut into octants, leaves that freeze
                at max_points_num."""
import numpy as np

import general_prior as gp
import lko_insert
from legkilo_b200 import abi, synth

G = synth.exp_so3(gp.G_ROTVEC)
NAMES = ("room_empty", "room_on_blob", "cluttered")
CALL_KEYS = ("pts", "set_offsets", "rot", "pos", "rot_cov", "pos_cov")


def poses(g, n):
    """n placements near G: attitude and position of gp.prior_at, the theta / position blocks of a dense P."""
    rot, pos, rc, pc = [], [], [], []
    for _ in range(n):
        x = gp.prior_at(G, gp.G_POS, g)
        P = gp.dense_cov(g).reshape(30, 30)
        rot.append(x["rot"][0].reshape(3, 3)); pos.append(x["pos"][0]); rc.append(P[:3, :3]); pc.append(P[3:6, 3:6])
    return dict(rot=np.array(rot), pos=np.array(pos), rot_cov=np.array(rc), pos_cov=np.array(pc))


def offsets(sizes):
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)


def room_trajectory(cfg, n_scans, seed, n_az=120):
    """n_scans revolutions in the box room, each placed at its own general pose."""
    sc, pw, pb = gp.map_cloud(cfg, G, gp.G_POS)
    scans = [gp.room_scan(cfg, sc, seed + 2 * i, False, n_az=n_az) for i in range(n_scans)]
    return dict(pw=pw, pb=pb, pts=np.concatenate(scans), set_offsets=offsets([len(s) for s in scans]),
                **poses(synth.rng(seed + 1), n_scans))


def cluttered(seed=9480, n=9000):
    g = synth.rng(seed)
    clutter = np.c_[g.uniform(2.0, 3.5, (n // 3, 2)), g.uniform(-0.5, 0.5, n // 3)]
    slab = np.c_[g.uniform(-3.0, -2.0, (2 * n // 3, 2)), -0.75 + 0.002 * g.standard_normal(2 * n // 3)]
    body = np.concatenate([clutter, slab])[g.permutation(n)]
    pts = np.zeros((n, 4), np.float32)
    pts[:, :3] = body.astype(np.float32)
    return dict(pts=pts, set_offsets=offsets([n // 3, n // 3, n - 2 * (n // 3)]), **poses(g, 3))


def case(name):
    cfg = abi.CONFIGS["leg_fusion"]
    if name == "cluttered":
        return cfg, cluttered()
    c = room_trajectory(cfg, 4, 9400 if name == "room_empty" else 9440)
    if name == "room_empty":
        del c["pw"], c["pb"]
    return cfg, c


def call(c):
    return [c[k] for k in CALL_KEYS]


def start_blob(cfg, c):
    """The map a case inserts on top of, as the oracle's BuildVoxelMap makes it (None: an empty map)."""
    if "pw" not in c:
        return None
    o = lko_insert.Oracle(cfg)
    o.build_voxel_map(c["pw"], c["pb"], R=G, rot_cov=gp.map_covs(G)[0], pos_cov=gp.map_covs(G)[1])
    return o.map_export()


def oracle_insert(cfg, blob, *args):
    o = lko_insert.Oracle(cfg)
    if blob is not None:
        o.map_import(blob)
    o.map_insert(*args)
    return o.map_export()
