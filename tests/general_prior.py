"""Scenes and priors away from the special case the rest of the suite starts from (identity attitude, zero position,
P0 = 1e-6 I): a box room whose first frame was taken from a general pose G (tens of degrees about every axis, metres to
kilometres from the origin), priors that compose G with a small perturbation, and dense SPD covariances whose attitude and
position blocks are large enough for the state term of sigma_l (lk_point.cuh: quad_sym3(Pth, h) + quad_sym3(Ppp, n)) to
be of the order of the body term.

Shared by tests/golden/make_ref_general_golden.py (fixtures made by the reference), tests/test_general_prior.py (oracle
on CPU) and tests/test_gpu_general_prior.py (device)."""
import numpy as np

from legkilo_b200 import abi, synth

HALF, WALL = 3.5, 2.75

# the general pose of the fixtures: tens of degrees about all three axes, negative keys on y
G_ROTVEC = (0.35, -0.6, 1.1)
G_POS = (-37.3, 81.6, 2.4)
FAR_POS = (1800.3, -2600.7, 35.2)

# (state_err, cov_err) tolerances (tests/scenes.py) of a whole streaming frame with map updates at a dense prior. Such a
# frame is sensitive: when P0 changes by 1e-15 the reference itself moves by up to 3.1e-5 sd / 5.2e-8
# (tests/golden/make_ref_general_golden.py checks that these moves stay within a quarter of the tolerances). Measured worst:
# the oracle against the fixtures 2.1e-5 sd / 3.9e-8, the device on an H100 80GB HBM3 3.2e-5 sd / 6.8e-8.
STREAM_TOLS = (1e-3, 2e-6)

# state blocks of the 30-vector (eskf.h): rot, pos, vel, ba, bw, grav, imu_a, imu_w, bv, contact
_SD_REST = (0.02, 0.02, 0.02, 5e-3, 5e-3, 5e-3, 1e-3, 1.2e-3, 0.8e-3, 1e-3, 1e-3, 1e-3, 0.05, 0.05, 0.05, 0.01, 0.01, 0.01,
            1e-3, 1e-3, 1e-3, 1e-3, 1e-3, 1e-3)


def dense_cov(g, rot_sd=(2.5e-3, 3e-3, 3.5e-3), pos_sd=(0.02, 0.03, 0.04), corr=0.6, scale=1.0):
    """A dense SPD 30 x 30 covariance, row-major [900]: distinct standard deviations on the attitude (rad) and position (m)
    blocks, and correlations between every pair of states (the attitude <-> position and {attitude, position} <->
    {vel, ba, bw} cross blocks included) drawn from `g`."""
    sd = scale * np.concatenate([rot_sd, pos_sd, _SD_REST])
    A = g.standard_normal((30, 30))
    C = corr * (A @ A.T) / 30.0 + (1.0 - corr) * np.eye(30)
    d = np.sqrt(np.diag(C))
    C = C / np.outer(d, d)
    P = C * np.outer(sd, sd)
    assert np.linalg.eigvalsh(P).min() > 0
    return P.ravel().copy()


def skewed(P, g, rel=1e-6):
    """P plus an antisymmetric part of `rel` times P's largest entry: the asymmetry P - K H P leaves behind after a real
    update, which makes the row-major convention of the ABI observable."""
    P = np.asarray(P, np.float64).reshape(30, 30)
    S = g.standard_normal((30, 30))
    S = S - S.T
    S *= rel * np.abs(P).max() / np.abs(S).max()
    return (P + S).ravel().copy()


def so3_uniform(g):
    """A rotation drawn uniformly on SO(3) (unit quaternion from a 4-D Gaussian)."""
    q = g.standard_normal(4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def moving_state(G, p):
    """The moving prior of the other reference fixtures (non-zero vel, biases, imu_a / imu_w) at attitude G, position p."""
    x0 = abi.default_states(1)
    x0["rot"][0] = np.asarray(G, np.float64).ravel()
    x0["pos"][0] = p
    x0["vel"][0] = (0.4, -0.2, 0.05)
    x0["imu_w"][0] = (0.02, -0.03, 0.15)
    x0["imu_a"][0] = (0.3, 0.1, 9.7)
    x0["ba"][0] = (0.01, -0.02, 0.03)
    x0["bw"][0] = (1e-3, 2e-3, -1e-3)
    return x0


def prior_at(G, pG, g, rot_sd=3e-3, pos_sd=0.03):
    """x0 = G composed with a small perturbation (attitude and position) drawn from `g`."""
    R = G @ synth.exp_so3(rot_sd * g.standard_normal(3))
    p = np.asarray(pG, np.float64) + G @ (pos_sd * g.standard_normal(3))
    return moving_state(R, p)


def map_cloud(cfg, G, pG, stream=11):
    """The box room's first-frame cloud seen from the general pose (G, pG): body points as the room-centred frame sees
    them, world points = f32(G (Re pb + te) + pG) as KILO::pointLidarToWorld stores them."""
    Re, te = abi.extrinsics(cfg)
    sc = synth.BoxScene(ground_half_extent=HALF, wall=WALL)
    _, pb = sc.map_points(ext_R=Re, ext_t=te, stream=stream)
    pw = ((pb.astype(np.float64) @ Re.T + te) @ np.asarray(G).T + np.asarray(pG, np.float64)).astype(np.float32)
    return sc, pw, pb


def room_scan(cfg, sc, stream, streaming, rotvec=None, trans=None, n_rings=16, n_az=120):
    """One revolution from a pose near the room's centre (the frame G maps to the world)."""
    Re, te = abi.extrinsics(cfg)
    if rotvec is None:
        rv, tv = synth.random_poses(1, 2e-3, 0.02, stream=stream)
        rotvec, trans = rv[0], tv[0]
    return sc.scan(rotvec=rotvec, trans=trans, ext_R=Re, ext_t=te, blind=cfg["blind"], stream=stream + 1, n_rings=n_rings,
                   n_az=n_az, fov_deg=(-15.0, 15.0), streaming=streaming)


def map_covs(G):
    """Non-isotropic attitude / position covariances for BuildVoxelMap (the first frame's P blocks)."""
    A = synth.exp_so3((0.3, 0.2, -0.4))
    return A @ np.diag([1e-6, 2.5e-6, 4e-6]) @ A.T, G @ np.diag([3e-6, 1e-6, 6e-6]) @ G.T


def world_atol(world, floor=5e-6):
    """Float32 world coordinates: `floor` near the origin, two ulps of the coordinate far from it."""
    return floor + 2.0 * np.spacing(np.abs(np.asarray(world, np.float32)[:, :3]))
