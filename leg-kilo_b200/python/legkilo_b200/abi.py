"""ctypes mirrors of the POD structs in include/legkilo_b200.h, and the reference's four dataset
configurations (values of legkilo/config/{leg_fusion,diter,hilti,nclt}.yaml — data, see
SURVEY.md Appendix B) as ready-made structs."""
from __future__ import annotations

import ctypes as C

import numpy as np

DIM_STATE = 30


class LkState(C.Structure):
    _fields_ = [("rot", C.c_double * 9), ("pos", C.c_double * 3), ("vel", C.c_double * 3), ("ba", C.c_double * 3),
                ("bw", C.c_double * 3), ("grav", C.c_double * 3), ("imu_a", C.c_double * 3),
                ("imu_w", C.c_double * 3), ("bv", C.c_double * 3), ("contact", C.c_double * 3)]


class LkEskfCfg(C.Structure):
    _fields_ = [(n, C.c_double) for n in (
        "vel_process_cov", "imu_acc_process_cov", "imu_gyr_process_cov", "contact_process_cov",
        "acc_bias_process_cov", "gyr_bias_process_cov", "kin_bias_process_cov", "imu_acc_meas_noise",
        "imu_acc_z_meas_noise", "imu_gyr_meas_noise", "kin_meas_noise", "chd_meas_noise", "contact_meas_noise",
        "lidar_point_meas_ratio")]


class LkMapCfg(C.Structure):
    _fields_ = [("max_voxel_size", C.c_double), ("planner_threshold", C.c_double), ("beam_err", C.c_double),
                ("dept_err", C.c_double), ("sigma_num", C.c_double), ("sliding_thresh", C.c_double),
                ("max_layer", C.c_int32), ("max_iterations", C.c_int32), ("max_points_num", C.c_int32),
                ("layer_init_num", C.c_int32 * 5), ("is_pub_plane_map", C.c_int32), ("map_sliding_en", C.c_int32),
                ("half_map_size", C.c_int32), ("reserved", C.c_int32)]


class LkStreamClock(C.Structure):
    _fields_ = [("last_predict_time", C.c_double), ("last_update_time", C.c_double)]


class LkImuMeas(C.Structure):
    _fields_ = [("stamp", C.c_double), ("acc", C.c_double * 3), ("gyr", C.c_double * 3)]


class LkKinImuMeas(C.Structure):
    _fields_ = [("stamp", C.c_double), ("foot_pos", (C.c_double * 3) * 4), ("foot_vel", (C.c_double * 3) * 4),
                ("contact", C.c_int32 * 4), ("acc", C.c_double * 3), ("gyr", C.c_double * 3)]


class LkLegCfg(C.Structure):
    _fields_ = [(n, C.c_double) for n in (
        "leg_offset_x", "leg_offset_y", "leg_calf_length", "leg_thigh_length", "leg_thigh_offset",
        "contact_force_threshold_up", "contact_force_threshold_down")]


class LkLegTrack(C.Structure):
    _fields_ = [("in_contact", C.c_int32 * 4), ("last_acc_z", C.c_float), ("last_gyr_z", C.c_float)]


def leg_track_default() -> LkLegTrack:
    """lk_leg_track_default: every detector in contact, a zero previous message (kinematics.h:12, ros_interface.cc:222)."""
    return LkLegTrack((C.c_int32 * 4)(1, 1, 1, 1), 0.0, 0.0)


class LkPc2Layout(C.Structure):
    _fields_ = [("point_step", C.c_uint32), ("off_x", C.c_uint32), ("off_y", C.c_uint32), ("off_z", C.c_uint32),
                ("off_intensity", C.c_uint32), ("off_time", C.c_uint32), ("lidar_type", C.c_int32), ("reserved", C.c_int32)]


# numpy views of the three driver point layouts (lidar_processing.h:10-72; EIGEN_ALIGN16 structs)
PC2_DTYPES = {
    1: np.dtype({"names": ["x", "y", "z", "intensity", "time", "ring"], "formats": ["f4", "f4", "f4", "f4", "f4", "u2"],
                 "offsets": [0, 4, 8, 16, 20, 24], "itemsize": 32}),
    2: np.dtype({"names": ["x", "y", "z", "intensity", "t", "reflectivity", "ring", "ambient", "range"],
                 "formats": ["f4", "f4", "f4", "f4", "u4", "u2", "u1", "u2", "u4"], "offsets": [0, 4, 8, 16, 20, 24, 26, 28, 32],
                 "itemsize": 48}),
    3: np.dtype({"names": ["x", "y", "z", "intensity", "timestamp", "ring"], "formats": ["f4", "f4", "f4", "f4", "f8", "u2"],
                 "offsets": [0, 4, 8, 16, 24, 32], "itemsize": 48}),
}


def pc2_layout(lidar_type: int) -> LkPc2Layout:
    dt = PC2_DTYPES[lidar_type]
    tname = {1: "time", 2: "t", 3: "timestamp"}[lidar_type]
    f = dt.fields
    return LkPc2Layout(dt.itemsize, f["x"][1], f["y"][1], f["z"][1], f["intensity"][1], f[tname][1], lidar_type, 0)


STATE_DTYPE = np.dtype([("rot", "f8", (9,)), ("pos", "f8", (3,)), ("vel", "f8", (3,)), ("ba", "f8", (3,)),
                        ("bw", "f8", (3,)), ("grav", "f8", (3,)), ("imu_a", "f8", (3,)), ("imu_w", "f8", (3,)),
                        ("bv", "f8", (3,)), ("contact", "f8", (3,))])
CLOCK_DTYPE = np.dtype([("last_predict_time", "f8"), ("last_update_time", "f8")])
IMU_DTYPE = np.dtype([("stamp", "f8"), ("acc", "f8", (3,)), ("gyr", "f8", (3,))])
KINIMU_DTYPE = np.dtype([("stamp", "f8"), ("foot_pos", "f8", (4, 3)), ("foot_vel", "f8", (4, 3)),
                         ("contact", "i4", (4,)), ("acc", "f8", (3,)), ("gyr", "f8", (3,))])
# lk_leg_state: one unitree_legged_msgs::HighState, message index order (legs FL FR RL RR) and types
LEG_STATE_DTYPE = np.dtype([("stamp", "f8"), ("acc", "f4", (3,)), ("gyr", "f4", (3,)), ("q", "f4", (12,)),
                            ("dq", "f4", (12,)), ("foot_force", "i2", (4,))], align=True)
assert STATE_DTYPE.itemsize == C.sizeof(LkState) == 288
assert LEG_STATE_DTYPE.itemsize == 136 and C.sizeof(LkLegCfg) == 56 and C.sizeof(LkLegTrack) == 24
assert KINIMU_DTYPE.itemsize == C.sizeof(LkKinImuMeas)

# map blob dtypes (include/legkilo_b200.h)
MAP_MAGIC = 0x504D4B4C
MAP_HEADER_DTYPE = np.dtype([("magic", "u4"), ("version", "u4"), ("n_roots", "u4"), ("n_nodes", "u4"),
                             ("n_points", "u8"), ("reserved", "u4", (2,))])
MAP_ROOT_DTYPE = np.dtype([("key", "i4", (3,)), ("node", "i4")])
MAP_NODE_DTYPE = np.dtype([("center", "f8", (3,)), ("normal", "f8", (3,)), ("plane_var", "f8", (21,)), ("d", "f4"),
                           ("radius", "f4"), ("flags", "u4"), ("child_base", "i4"), ("pad", "u4", (6,))])
MAP_AUX_DTYPE = np.dtype([("voxel_center", "f8", (3,)), ("quater_length", "f4"), ("pts_base", "u4"),
                          ("pts_count", "i4"), ("pts_cap", "i4"), ("new_points", "i4"), ("parent", "i4"),
                          ("key", "i4", (3,)), ("pad", "i4")])
MAP_POINT_DTYPE = np.dtype([("pw", "f8", (3,)), ("var", "f8", (6,))])
assert MAP_HEADER_DTYPE.itemsize == 32 and MAP_ROOT_DTYPE.itemsize == 16
assert MAP_NODE_DTYPE.itemsize == 256 and MAP_AUX_DTYPE.itemsize == 64 and MAP_POINT_DTYPE.itemsize == 72

# lk_score_poses record (LK_SCORE_*): A = sum h^T h / R (upper triangle, 21) | b = sum h^T z / R (6) | sum R | count |
# sum z^2 / R | 0 0
SCORE_A, SCORE_B, SCORE_SUM_R, SCORE_COUNT, SCORE_SUM_Z2R, SCORE_STRIDE = 0, 21, 27, 28, 29, 32

NODE_IS_PLANE, NODE_INIT_OCTO, NODE_UPDATE_ENABLE = 1, 2, 4
NODE_LAYER_SHIFT, NODE_CHILDMASK_SHIFT = 8, 16


def parse_map_blob(blob: bytes | np.ndarray):
    """Split an lk_map blob into (header, roots, nodes, aux, points) numpy views."""
    buf = np.frombuffer(blob, dtype=np.uint8)
    hd = buf[:32].view(MAP_HEADER_DTYPE)[0]
    assert hd["magic"] == MAP_MAGIC
    o = 32
    nr, nn, npnt = int(hd["n_roots"]), int(hd["n_nodes"]), int(hd["n_points"])
    roots = buf[o:o + 16 * nr].view(MAP_ROOT_DTYPE); o += 16 * nr
    nodes = buf[o:o + 256 * nn].view(MAP_NODE_DTYPE); o += 256 * nn
    aux = buf[o:o + 64 * nn].view(MAP_AUX_DTYPE); o += 64 * nn
    pts = buf[o:o + 72 * npnt].view(MAP_POINT_DTYPE)
    return hd, roots, nodes, aux, pts


def make_map_blob(roots, nodes, aux, points) -> np.ndarray:
    hd = np.zeros(1, MAP_HEADER_DTYPE)
    hd["magic"] = MAP_MAGIC
    hd["version"] = 1
    hd["n_roots"] = len(roots)
    hd["n_nodes"] = len(nodes)
    hd["n_points"] = len(points)
    parts = [hd.view(np.uint8), np.ascontiguousarray(roots).view(np.uint8).ravel(),
             np.ascontiguousarray(nodes).view(np.uint8).ravel(), np.ascontiguousarray(aux).view(np.uint8).ravel(),
             np.ascontiguousarray(points).view(np.uint8).ravel()]
    return np.concatenate(parts)


# ---- reference dataset configurations (legkilo/config/*.yaml) --------------------------------
_COMMON = dict(
    vel_process_cov=20.0, imu_acc_process_cov=500.0, imu_gyr_process_cov=1000.0, contact_process_cov=20.0,
    acc_bias_process_cov=0.001, gyr_bias_process_cov=0.001, kin_bias_process_cov=0.001, kin_meas_noise=0.1,
    chd_meas_noise=0.1, contact_meas_noise=0.001, lidar_point_meas_ratio=10.0,
    max_layer=2, voxel_size=0.5, min_eigen_value=0.01, sigma_num=3.0, beam_err=0.2, dept_err=0.04,
    layer_init_num=(5, 5, 5, 5, 5), max_points_num=50, map_sliding_en=0, half_map_size=100, sliding_thresh=8.0,
    gravity=9.81, blind=1.5, filter_num=3, redundancy=True)

# Kinematics::Config (legkilo/config/*.yaml:45-51)
_LEG_UNITREE = dict(leg_offset_x=0.1881, leg_offset_y=0.04675, leg_calf_length=0.213, leg_thigh_length=0.213,
                    leg_thigh_offset=0.08, contact_force_threshold_up=220.0, contact_force_threshold_down=200.0)
_LEG_DITER = dict(leg_offset_x=0.1934, leg_offset_y=0.0465, leg_calf_length=0.213, leg_thigh_length=0.213,
                  leg_thigh_offset=0.0465, contact_force_threshold_up=40.0, contact_force_threshold_down=60.0)

CONFIGS = {
    "leg_fusion": dict(_COMMON, **_LEG_UNITREE, only_imu_use=False, extrinsic_T=(0.0, 0.0, 0.20),
                       extrinsic_R=(1, 0, 0, 0, 1, 0, 0, 0, 1), voxel_grid_resolution=0.3, lidar_type=1, time_scale=1.0,
                       imu_acc_meas_noise=0.1, imu_acc_z_meas_noise=1.0, imu_gyr_meas_noise=0.01),
    "diter": dict(_COMMON, **_LEG_DITER, only_imu_use=False, extrinsic_T=(0.005, 0.00056, 0.299),
                  extrinsic_R=(1, 0, 0, 0, 1, 0, 0, 0, 1), voxel_grid_resolution=0.5, lidar_type=2, time_scale=1e-9,
                  imu_acc_meas_noise=0.01, imu_acc_z_meas_noise=0.1, imu_gyr_meas_noise=0.001),
    "hilti": dict(_COMMON, **_LEG_UNITREE, only_imu_use=True, extrinsic_T=(-0.001, -0.00855, 0.055),
                  extrinsic_R=(0, -1, 0, -1, 0, 0, 0, 0, -1), voxel_grid_resolution=0.5, lidar_type=3, time_scale=1.0,
                  imu_acc_meas_noise=0.01, imu_acc_z_meas_noise=0.01, imu_gyr_meas_noise=0.01, blind=0.2),
    "nclt": dict(_COMMON, **_LEG_UNITREE, only_imu_use=True, extrinsic_T=(0.0, 0.0, 0.28), extrinsic_R=(1, 0, 0, 0, 1, 0, 0, 0, 1),
                 voxel_grid_resolution=0.5, lidar_type=1, time_scale=1e-6, imu_acc_meas_noise=0.1,
                 imu_acc_z_meas_noise=1.0, imu_gyr_meas_noise=0.01),
}


def eskf_cfg(cfg: dict) -> LkEskfCfg:
    e = LkEskfCfg()
    for name, _ in LkEskfCfg._fields_:
        setattr(e, name, float(cfg[name]))
    return e


def leg_cfg(cfg: dict) -> LkLegCfg:
    """Kinematics::Config (kinematics.h:27-35) of a dataset configuration."""
    c = LkLegCfg()
    for name, _ in LkLegCfg._fields_:
        setattr(c, name, float(cfg[name]))
    return c


def map_cfg(cfg: dict) -> LkMapCfg:
    m = LkMapCfg()
    m.max_voxel_size = cfg["voxel_size"]
    m.planner_threshold = cfg["min_eigen_value"]
    m.beam_err = cfg["beam_err"]
    m.dept_err = cfg["dept_err"]
    m.sigma_num = cfg["sigma_num"]
    m.sliding_thresh = cfg["sliding_thresh"]
    m.max_layer = cfg["max_layer"]
    m.max_iterations = 1
    m.max_points_num = cfg["max_points_num"]
    for i, v in enumerate(cfg["layer_init_num"]):
        m.layer_init_num[i] = v
    m.map_sliding_en = cfg["map_sliding_en"]
    m.half_map_size = cfg["half_map_size"]
    return m


def extrinsics(cfg: dict):
    return (np.asarray(cfg["extrinsic_R"], np.float64).reshape(3, 3).copy(),
            np.asarray(cfg["extrinsic_T"], np.float64).copy())


def default_states(batch: int) -> np.ndarray:
    """State::State() (eskf.cc:5-16) x batch."""
    x = np.zeros(batch, STATE_DTYPE)
    x["rot"] = np.eye(3).ravel()
    x["grav"] = (0.0, 0.0, -9.81)
    return x


def init_cov(batch: int) -> np.ndarray:
    """StateInitial: P0 = 1e-6 * I (state_initial.hpp:69)."""
    return np.tile((1e-6 * np.eye(30)).ravel(), (batch, 1)).reshape(batch, 900).copy()


def process_cov_Q(cfg: dict) -> np.ndarray:
    """ESKF::initProcessCovQ (eskf.cc:47-62)."""
    Q = np.zeros((30, 30))
    for at, key in ((6, "vel_process_cov"), (9, "acc_bias_process_cov"), (12, "gyr_bias_process_cov"),
                    (18, "imu_acc_process_cov"), (21, "imu_gyr_process_cov"), (24, "kin_bias_process_cov"),
                    (27, "contact_process_cov")):
        for k in range(3):
            Q[at + k, at + k] = cfg[key]
    return Q.ravel().copy()
