"""Seeded synthetic scenes for the BASELINE.json configs (SURVEY.md §8d).

Everything here produces plain numpy arrays that are handed, unchanged, to both the CUDA library
and (in tests / the cpu_baseline leg of bench.py) the CPU oracle — so bit-identical inputs need no
cross-language RNG. Base seed 0x4C4B494C4F ("LKILO").

Point layout everywhere: float32 [n, 4] = (x, y, z, curvature) in the LiDAR body frame, the four
fields of the reference's 48-byte pcl::PointXYZINormal that the hot path reads
(legkilo/src/core/slam/KILO.cc:123-127; curvature = per-point time offset in seconds,
legkilo/src/preprocess/lidar_processing.cc:48).
"""
from __future__ import annotations

import numpy as np

BASE_SEED = 0x4C4B494C4F


def rng(stream: int, seed: int = BASE_SEED) -> np.random.Generator:
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence([seed, stream])))


def exp_so3(v) -> np.ndarray:
    v = np.asarray(v, dtype=np.float64)
    th = np.linalg.norm(v)
    if th < 1e-12:
        return np.eye(3)
    k = v / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * (K @ K)


def world_to_body(pw: np.ndarray, R: np.ndarray, p: np.ndarray, ext_R: np.ndarray, ext_t: np.ndarray) -> np.ndarray:
    """Inverse of pw = R (ext_R pb + ext_t) + p  (KILO.cc:127-129)."""
    pi = (pw - p) @ R  # R^T (pw - p), row-vector form
    return (pi - ext_t) @ ext_R


# ---------------------------------------------------------------------------------------------
# Config 1: planar scene
# ---------------------------------------------------------------------------------------------

def planar_map_points(half_extent: float = 20.0, z: float = -0.75, voxel: float = 0.5, pts_per_voxel: int = 8,
                      sigma: float = 0.01, ext_R=None, ext_t=None, stream: int = 1):
    """Ground plane z=const sampled `pts_per_voxel` per voxel column (first-frame cloud).
    Returns (xyz_world float32 [n,3], xyz_body float32 [n,3]) for BuildVoxelMap with R=I, p=0."""
    ext_R = np.eye(3) if ext_R is None else np.asarray(ext_R, float)
    ext_t = np.zeros(3) if ext_t is None else np.asarray(ext_t, float)
    g = rng(stream)
    nv = int(round(2 * half_extent / voxel))
    ix, iy = np.meshgrid(np.arange(nv), np.arange(nv), indexing="ij")
    base = np.stack([ix.ravel(), iy.ravel()], 1).astype(np.float64) * voxel - half_extent
    base = np.repeat(base, pts_per_voxel, axis=0)
    xy = base + g.uniform(0.02, voxel - 0.02, size=base.shape)
    zz = z + sigma * g.standard_normal(len(xy))
    pw = np.concatenate([xy, zz[:, None]], 1)
    pb = world_to_body(pw, np.eye(3), np.zeros(3), ext_R, ext_t)
    pb32 = pb.astype(np.float32)
    # the reference stores the world cloud as float (KILO.cc:101-103): world = f32(R(ext pb)+p)
    pw32 = ((pb32.astype(np.float64) @ ext_R.T) + ext_t).astype(np.float32)
    return pw32, pb32


def planar_scan(n: int = 2048, radius: float = 15.0, z: float = -0.75, sigma: float = 0.01,
                rotvec=(2e-3, -1e-3, 3e-3), trans=(0.02, -0.01, 0.03), ext_R=None, ext_t=None, stream: int = 2,
                blind: float = 0.0):
    """n points uniform in a disc on the plane as seen from the TRUE pose (Exp(rotvec), trans)."""
    ext_R = np.eye(3) if ext_R is None else np.asarray(ext_R, float)
    ext_t = np.zeros(3) if ext_t is None else np.asarray(ext_t, float)
    g = rng(stream)
    R = exp_so3(rotvec)
    p = np.asarray(trans, float)
    out = np.zeros((0, 3))
    while len(out) < n:
        m = 2 * (n - len(out)) + 16
        r = radius * np.sqrt(g.uniform(0, 1, m))
        a = g.uniform(0, 2 * np.pi, m)
        pw = np.stack([r * np.cos(a), r * np.sin(a), z + sigma * g.standard_normal(m)], 1)
        pb = world_to_body(pw, R, p, ext_R, ext_t)
        keep = np.linalg.norm(pb, axis=1) >= blind
        out = np.concatenate([out, pb[keep]], 0)
    pts = np.zeros((n, 4), np.float32)
    pts[:, :3] = out[:n].astype(np.float32)
    return pts


# ---------------------------------------------------------------------------------------------
# Configs 2-5: box room (ground + 4 walls) ray-cast by a spinning LiDAR
# ---------------------------------------------------------------------------------------------

class BoxScene:
    """Ground plane z=zg over [-E,E]^2 and four walls x=+-W, y=+-W from zg up to z_top.
    Plane offsets sit mid-voxel (…25) so that noisy samples stay inside one root voxel."""

    def __init__(self, ground_half_extent: float = 250.0, wall: float = 15.25, zg: float = -0.75, z_top: float = 6.25,
                 voxel: float = 0.5, rooms=None):
        self.E = float(ground_half_extent)
        self.W = float(wall)
        self.zg = float(zg)
        self.z_top = float(z_top)
        self.voxel = float(voxel)
        # room centres (multiples of the voxel size so every room looks the same on the voxel grid)
        self.rooms = [(0.0, 0.0)] if rooms is None else [(float(a), float(b)) for a, b in rooms]

    @staticmethod
    def room_grid(n_side: int, spacing: float = 62.0):
        """n_side x n_side room centres, `spacing` metres apart, centred on the origin."""
        c = (np.arange(n_side) - (n_side - 1) / 2.0) * spacing
        c = np.round(c / 0.5) * 0.5
        return [(float(a), float(b)) for a in c for b in c]

    # -- first-frame style dense cloud for the map --------------------------------------------
    def map_points(self, pts_per_voxel: int = 8, sigma: float = 0.01, ext_R=None, ext_t=None, stream: int = 11,
                   ground_half_extent: float | None = None):
        ext_R = np.eye(3) if ext_R is None else np.asarray(ext_R, float)
        ext_t = np.zeros(3) if ext_t is None else np.asarray(ext_t, float)
        g = rng(stream)
        v = self.voxel
        E = self.E if ground_half_extent is None else float(ground_half_extent)
        chunks = []
        # ground
        nv = int(round(2 * E / v))
        ix, iy = np.meshgrid(np.arange(nv, dtype=np.int32), np.arange(nv, dtype=np.int32), indexing="ij")
        base = np.stack([ix.ravel(), iy.ravel()], 1).astype(np.float64) * v - E
        base = np.repeat(base, pts_per_voxel, axis=0)
        xy = base + g.uniform(0.02, v - 0.02, size=base.shape)
        zz = self.zg + sigma * g.standard_normal(len(xy))
        chunks.append(np.concatenate([xy, zz[:, None]], 1))
        # walls: cells over (along, height)
        nl = int(round(2 * self.W / v)) + 1
        nh = int(np.ceil((self.z_top - self.zg) / v))
        il, ih = np.meshgrid(np.arange(nl), np.arange(nh), indexing="ij")
        cell = np.stack([il.ravel(), ih.ravel()], 1).astype(np.float64)
        cell = np.repeat(cell, pts_per_voxel, axis=0)
        for (rcx, rcy) in self.rooms:
            rc = (rcx, rcy)
            for axis, sign in ((0, 1), (0, -1), (1, 1), (1, -1)):
                u = cell + g.uniform(0.04, 0.96, size=cell.shape)
                along = -self.W - 0.25 + u[:, 0] * v
                hz = np.floor(self.zg / v) * v + u[:, 1] * v
                off = sign * self.W + sigma * g.standard_normal(len(u))
                ok = (np.abs(along) < self.W) & (hz > self.zg + 0.05) & (hz < self.z_top)
                p = np.zeros((ok.sum(), 3))
                p[:, axis] = rc[axis] + off[ok]
                p[:, 1 - axis] = rc[1 - axis] + along[ok]
                p[:, 2] = hz[ok]
                chunks.append(p)
        pw = np.concatenate(chunks, 0)
        # every point is "seen" from the centre of its nearest room (identity attitude), the way a
        # first frame taken there would see it: body = ext^-1 (world - room centre)
        rc = np.asarray(self.rooms, float)
        near = np.zeros(len(pw), np.int64)
        best = np.full(len(pw), np.inf)
        for i, c in enumerate(rc):
            d2 = (pw[:, 0] - c[0]) ** 2 + (pw[:, 1] - c[1]) ** 2
            m = d2 < best
            near[m] = i
            best[m] = d2[m]
        origin = np.concatenate([rc[near], np.zeros((len(pw), 1))], 1)
        pb = world_to_body(pw - origin, np.eye(3), np.zeros(3), ext_R, ext_t)
        pb32 = pb.astype(np.float32)
        pw32 = (((pb32.astype(np.float64) @ ext_R.T) + ext_t) + origin).astype(np.float32)
        return pw32, pb32

    # -- one LiDAR revolution -------------------------------------------------------------------
    def scan(self, n_rings: int, n_az: int, fov_deg: tuple[float, float], rotvec, trans, ext_R=None, ext_t=None,
             sigma: float = 0.01, blind: float = 1.5, stream: int = 21, scan_period: float = 0.1,
             time_quantum: float = 0.002, streaming: bool = False, room: int = 0):
        """Ray-cast n_rings x n_az rays from the true pose. Returns float32 [n,4]; curvature is
        the 2 ms-quantised time offset (lidar_processing.cc:48) when streaming, else 0."""
        ext_R = np.eye(3) if ext_R is None else np.asarray(ext_R, float)
        ext_t = np.zeros(3) if ext_t is None else np.asarray(ext_t, float)
        g = rng(stream)
        R = exp_so3(rotvec)
        sensor_xy = self.rooms[room]
        p = np.asarray(trans, float) + np.array([sensor_xy[0], sensor_xy[1], 0.0])
        el = np.deg2rad(np.linspace(fov_deg[0], fov_deg[1], n_rings))
        az = (np.arange(n_az) + 0.5) * (2 * np.pi / n_az)
        A, EL = np.meshgrid(az, el, indexing="ij")  # azimuth-major = time order
        d_l = np.stack([np.cos(EL) * np.cos(A), np.cos(EL) * np.sin(A), np.sin(EL)], -1).reshape(-1, 3)
        t_off = np.repeat(np.arange(n_az) / n_az * scan_period, n_rings)
        M = R @ ext_R
        o = R @ ext_t + p
        d = d_l @ M.T
        best = np.full(len(d), np.inf)
        with np.errstate(divide="ignore", invalid="ignore"):
            tg = (self.zg - o[2]) / d[:, 2]
            hit = o[None, :] + tg[:, None] * d
            ok = (tg > 0) & (np.abs(hit[:, 0] - sensor_xy[0]) <= self.W) & (np.abs(hit[:, 1] - sensor_xy[1]) <= self.W)
            best = np.where(ok, np.minimum(best, tg), best)
            for axis, sign in ((0, 1), (0, -1), (1, 1), (1, -1)):
                c = sensor_xy[axis] + sign * self.W
                tw = (c - o[axis]) / d[:, axis]
                hit = o[None, :] + tw[:, None] * d
                ok = (tw > 0) & (np.abs(hit[:, 1 - axis] - sensor_xy[1 - axis]) <= self.W) & (hit[:, 2] >= self.zg) & (
                    hit[:, 2] <= self.z_top)
                best = np.where(ok, np.minimum(best, tw), best)
        valid = np.isfinite(best)
        rng_m = best + sigma * g.standard_normal(len(best))
        valid &= rng_m >= blind
        pb = d_l[valid] * rng_m[valid, None]
        pts = np.zeros((int(valid.sum()), 4), np.float32)
        pts[:, :3] = pb.astype(np.float32)
        if streaming:
            # curvature = round(t / quantum) * quantum as float (lidar_processing.cc:48)
            pts[:, 3] = (np.round(t_off[valid] / time_quantum) * time_quantum).astype(np.float32)
        return pts


VLP16 = dict(n_rings=16, n_az=1800, fov_deg=(-15.0, 15.0))
OS64 = dict(n_rings=64, n_az=2048, fov_deg=(-16.6, 16.6))


# Raw time units of the three drivers' shipped configurations (nclt / diter / hilti .yaml): the time_scale of each.
PC2_TIME_SCALE = {1: 1e-6, 2: 1e-9, 3: 1.0}


def pack_pointcloud2(lidar_type: int, xyz, t, intensity, t0: float = 0.0) -> np.ndarray:
    """One PointCloud2 message's points in the driver layout abi.PC2_DTYPES[lidar_type] (its .view(np.uint8) is the
    message's data). xyz [n, 3], t [n] seconds since the start of the sweep, raw time as the driver writes it
    (lidar_processing.h:10-72): Velodyne float32 microseconds, Ouster uint32 nanoseconds, Hesai float64 absolute
    seconds t0 + t."""
    from . import abi
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    a = np.zeros(len(xyz), abi.PC2_DTYPES[lidar_type])
    a["x"], a["y"], a["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    a["intensity"] = intensity
    t = np.asarray(t, np.float64)
    if lidar_type == 1:
        a["time"] = (t * 1e6).astype(np.float32)
    elif lidar_type == 2:
        a["t"] = np.round(t * 1e9).astype(np.uint32)
    else:
        a["timestamp"] = t0 + t
    return a


def box_pointcloud2s(n_msgs: int, lidar_type: int, lidar=VLP16, distinct: int = 8, stream: int = 9500):
    """n_msgs PointCloud2 messages of box-room sweeps (`distinct` poses, repeated) in the driver layout of `lidar_type`,
    with the ray geometry of `lidar`. Raw point times jitter by up to 1 ms around each ray's firing time, so the decode's
    2 ms rounding has work to do; no blind cut, so points near the sensor stay in. Returns (messages as structured arrays,
    header stamps 1000 + 0.1 s per message)."""
    from . import abi
    R, t = abi.extrinsics(abi.CONFIGS["leg_fusion"])
    sc = BoxScene(ground_half_extent=20.0)
    rv, tv = random_poses(distinct, 0.2, 2.0, stream=stream)
    stamps = 1000.0 + 0.1 * np.arange(n_msgs)
    base = []
    for i in range(distinct):
        g = rng(stream + 1 + distinct + i)
        s = sc.scan(rotvec=rv[i], trans=tv[i], ext_R=R, ext_t=t, blind=0.0, stream=stream + 1 + i, streaming=True, **lidar)
        tt = np.clip(s[:, 3].astype(np.float64) + g.uniform(-1e-3, 1e-3, len(s)), 0.0, None)
        base.append((s[:, :3], tt, g.uniform(0.0, 255.0, len(s)).astype(np.float32)))
    msgs = [pack_pointcloud2(lidar_type, *base[m % distinct], t0=stamps[m]) for m in range(n_msgs)]
    return msgs, stamps


def random_poses(batch: int, rot_sigma: float, trans_sigma: float, stream: int = 31):
    g = rng(stream)
    return rot_sigma * g.standard_normal((batch, 3)), trans_sigma * g.standard_normal((batch, 3))


def bucketize(pts: np.ndarray, begin_time: float = 0.0):
    """Canonical a1 ordering (SURVEY §8a a1): stable sort by curvature, then maximal equal runs
    (KILO.cc:370-378). Returns (sorted pts, bucket_offsets uint32 [nb+1], bucket_times f64 [nb])."""
    order = np.argsort(pts[:, 3], kind="stable")
    s = np.ascontiguousarray(pts[order])
    if len(s) == 0:
        return s, np.zeros(1, np.uint32), np.zeros(0, np.float64)
    brk = np.flatnonzero(s[1:, 3] != s[:-1, 3]) + 1
    offs = np.concatenate([[0], brk, [len(s)]]).astype(np.uint32)
    times = begin_time + s[offs[:-1], 3].astype(np.float64)
    return s, offs, times


# ---------------------------------------------------------------------------------------------
# Inertial / kinematic sample streams (SURVEY §8d config 5)
# ---------------------------------------------------------------------------------------------

def imu_stream(t0: float, t1: float, rate_hz: float = 400.0, stream: int = 41):
    """lk_imu_meas samples on (t0, t1]: gravity-dominated accelerometer, small gyro, white noise."""
    from . import abi
    g = rng(stream)
    n = int(np.floor((t1 - t0) * rate_hz))
    m = np.zeros(n, abi.IMU_DTYPE)
    m["stamp"] = t0 + (np.arange(n) + 1) / rate_hz
    m["acc"] = np.array([0.15, -0.1, 9.79]) + 0.05 * g.standard_normal((n, 3))
    m["gyr"] = np.array([0.01, -0.02, 0.12]) + 0.005 * g.standard_normal((n, 3))
    return m


def kinimu_stream(t0: float, t1: float, rate_hz: float = 400.0, stream: int = 43):
    """lk_kinimu_meas samples (sensor_types.hpp:19-26): 2-4 feet in contact, trotting pattern."""
    from . import abi
    g = rng(stream)
    im = imu_stream(t0, t1, rate_hz, stream)
    n = len(im)
    m = np.zeros(n, abi.KINIMU_DTYPE)
    m["stamp"] = im["stamp"]; m["acc"] = im["acc"]; m["gyr"] = im["gyr"]
    hip = np.array([[0.19, -0.13, -0.3], [0.19, 0.13, -0.3], [-0.19, -0.13, -0.3], [-0.19, 0.13, -0.3]])
    m["foot_pos"] = hip[None] + 0.02 * g.standard_normal((n, 4, 3))
    m["foot_vel"] = 0.05 * g.standard_normal((n, 4, 3))
    phase = (np.arange(n) // 20) % 3
    pat = np.array([[1, 0, 0, 1], [0, 1, 1, 0], [1, 1, 1, 1]], np.int32)
    m["contact"] = pat[phase]
    return m


def leg_state_stream(t0: float, t1: float, rate_hz: float = 500.0, cfg_name: str = "leg_fusion", stream: int = 47):
    """unitree HighState fields (abi.LEG_STATE_DTYPE, message order FL FR RL RR) on (t0, t1] for lk_leg_kinematics:
    joints around a standing pose with a 2 Hz trot (diagonal pairs FL+RR / FR+RL in antiphase), dq the derivative plus
    noise; foot forces that cross both contact thresholds of `cfg_name`, sit between them for stretches and hit each
    exactly now and then; runs of messages that repeat the previous accelerometer z AND gyroscope z (dropped by the
    redundancy check), and some that repeat only one of them (kept)."""
    from . import abi
    cfg = abi.CONFIGS[cfg_name]
    g = rng(stream)
    n = int(np.floor((t1 - t0) * rate_hz))
    m = np.zeros(n, abi.LEG_STATE_DTYPE)
    t = t0 + (np.arange(n) + 1) / rate_hz
    m["stamp"] = t
    w = 2.0 * np.pi * 2.0
    phase = w * t[:, None] + np.array([0.0, np.pi, np.pi, 0.0])[None]  # (n, 4)
    stand = np.array([0.0, 0.8, -1.6]); amp = np.array([0.05, 0.25, 0.35])
    q = stand + amp * np.sin(phase)[:, :, None]
    dq = amp * w * np.cos(phase)[:, :, None] + 0.05 * g.standard_normal((n, 4, 3))
    m["q"] = q.reshape(n, 12).astype(np.float32)
    m["dq"] = dq.reshape(n, 12).astype(np.float32)
    up, down = cfg["contact_force_threshold_up"], cfg["contact_force_threshold_down"]
    lo, hi = min(up, down), max(up, down)
    # stance (sin < 0) well above both thresholds, swing well below, a trapezoid so that the crossing takes a few samples
    mid, half = 0.5 * (lo + hi), 0.5 * (hi - lo) + 60.0
    f = mid + half * np.clip(-2.5 * np.sin(phase), -1.0, 1.0) + 4.0 * g.standard_normal((n, 4))
    # stretches of 10-40 samples strictly between the thresholds
    for leg in range(4):
        for s0 in g.integers(0, max(n, 1), size=max(n // 150, 1)):
            seg = f[s0:s0 + int(g.integers(10, 41)), leg]
            seg[:] = g.uniform(lo + 1.0, hi - 1.0, size=len(seg))
    hit = g.uniform(size=(n, 4))
    f = np.where(hit < 0.02, up, np.where(hit > 0.98, down, f))
    m["foot_force"] = np.clip(np.rint(f), -32768, 32767).astype(np.int16)
    acc = (np.array([0.15, -0.1, 9.79]) + 0.05 * g.standard_normal((n, 3))).astype(np.float32)
    gyr = (np.array([0.01, -0.02, 0.12]) + 0.005 * g.standard_normal((n, 3))).astype(np.float32)
    # repeats: each message copies the previous one's z pair with probability 0.3, so runs form
    rep = g.uniform(size=n) < 0.3
    rep[0] = False
    src = np.maximum.accumulate(np.where(rep, 0, np.arange(n)))
    acc[:, 2] = acc[src, 2]; gyr[:, 2] = gyr[src, 2]
    one = (~rep) & (g.uniform(size=n) < 0.05)  # only the accelerometer z repeats: not redundant
    one[0] = False
    prev = np.flatnonzero(one) - 1
    acc[one, 2] = acc[prev, 2]
    m["acc"] = acc; m["gyr"] = gyr
    return m
