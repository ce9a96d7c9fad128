"""legkilo_b200 — thin ctypes driver over liblegkilo_b200.so (the C-ABI in include/legkilo_b200.h).

The product is the CUDA library; this module only marshals numpy buffers across the C boundary
for tests and bench.py. It never computes the hot path itself and has no CPU fallback: if the
shared library is missing, or no CUDA device is present, it raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import abi

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.normpath(os.path.join(_PKG, "..", "..", "liblegkilo_b200.so"))
HEADER_PATH = os.path.normpath(os.path.join(_PKG, "..", "..", "..", "include", "legkilo_b200.h"))

_LIB = None


class LkError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"legkilo_b200 error {code}: {msg}")
        self.code = code


def lib():
    """Load the CUDA library. Fails loudly when it has not been built."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). There is no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        vp, i32, u32, dbl = C.c_void_p, C.c_int, C.c_uint32, C.c_double
        L.lk_create.argtypes = [vp, vp, vp, vp, i32, vp]
        L.lk_destroy.argtypes = [vp]
        L.lk_last_error.restype = C.c_char_p
        L.lk_last_error.argtypes = [vp]
        L.lk_init_process_cov.argtypes = [vp, vp]
        L.lk_state_default.argtypes = [vp]
        L.lk_host_alloc.argtypes = [vp, C.c_size_t]
        L.lk_host_free.argtypes = [vp]
        L.lk_set_param.argtypes = [vp, C.c_char_p, dbl]
        L.lk_sync.argtypes = [vp]
        L.lk_map_reserve.argtypes = [vp, C.c_uint64, C.c_uint64, C.c_uint64]
        L.lk_map_upload.argtypes = [vp, vp, C.c_size_t]
        L.lk_map_download.argtypes = [vp, vp, C.c_size_t, vp]
        L.lk_map_build.argtypes = [vp, vp, vp, C.c_size_t, vp, vp, vp]
        L.lk_first_frame.argtypes = [vp, vp, vp, vp, vp, vp, u32, dbl, vp, vp, u32, dbl, vp]
        L.lk_map_insert.argtypes = [vp, u32, vp, vp, vp, vp, vp, vp]
        L.lk_score_poses.argtypes = [vp, u32, vp, vp, u32] + [vp] * 6
        L.lk_refine_poses.argtypes = [vp, u32, vp, vp, u32] + [vp] * 5 + [C.c_int] + [vp] * 3
        L.lk_search_poses.argtypes = [vp, u32] + [vp] * 9 + [C.c_int, vp, vp, u32] + [vp] * 4
        L.lk_map_stats.argtypes = [vp, vp]
        L.lk_map_slide.argtypes = [vp, vp, vp, vp]
        L.lk_map_memory.argtypes = [vp, vp]
        L.lk_tum_line.argtypes = [dbl, vp, vp, C.c_char_p, C.c_size_t]
        L.lk_scan_update.argtypes = [vp, i32] + [vp] * 9 + [i32, i32, vp, vp]
        L.lk_batch_stage.argtypes = [vp, i32] + [vp] * 9
        L.lk_batch_run.argtypes = [vp, i32, i32]
        L.lk_batch_run_range.argtypes = [vp, u32, u32, i32, i32]
        L.lk_timer_start.argtypes = [vp]
        L.lk_timer_stop.argtypes = [vp] * 5
        L.lk_debug_read.argtypes = [vp, i32, vp, C.c_size_t]
        L.lk_batch_fetch.argtypes = [vp] * 6
        L.lk_batch_last_timing.argtypes = [vp] * 5
        L.lk_debug_residuals.argtypes = [vp, vp, vp, vp, u32] + [vp] * 5
        L.lk_predict.argtypes = [vp, i32, vp, vp, vp, vp, i32, i32]
        L.lk_update_by_points.argtypes = [vp, vp, vp, u32, vp, vp, vp]
        L.lk_obs_imu.argtypes = [vp, vp, vp, vp, vp, vp, u32, dbl, dbl]
        L.lk_obs_kinimu.argtypes = [vp, vp, vp, vp, vp, vp, u32, dbl, dbl]
        L.lk_process_scan.argtypes = [vp, vp, vp, vp, vp, vp, u32, vp, vp, u32, vp, vp, u32, dbl, dbl, i32, i32, vp,
                                      vp, vp]
        L.lk_decode_pointcloud2.argtypes = [vp, vp, u32, vp, C.c_float, i32, dbl, vp, vp, vp, vp, vp]
        L.lk_decode_pointcloud2s.argtypes = [vp, u32, vp, vp, vp, vp, C.c_float, i32, dbl] + [vp] * 5
        L.lk_preprocess_scan.argtypes = [vp, vp, u32, C.c_float, vp, vp, vp, vp, vp]
        L.lk_preprocess_scans.argtypes = [vp, u32, vp, vp, C.c_float] + [vp] * 7
        L.lk_leg_track_default.argtypes = [vp]
        L.lk_leg_kinematics.argtypes = [vp, vp, vp, u32, i32, vp, vp, vp]
        _LIB = L
    return _LIB


def tum_line(timestamp, rot, pos) -> str:
    """TrajectorySaver::write (trajectory_saver.hpp:43-50)."""
    rot = np.ascontiguousarray(rot, np.float64).reshape(9); pos = np.ascontiguousarray(pos, np.float64)
    buf = C.create_string_buffer(256)
    n = lib().lk_tum_line(float(timestamp), _p(rot), _p(pos), buf, 256)
    if n < 0:
        raise LkError(n, "lk_tum_line")
    return buf.value.decode()


def _p(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(C.c_void_p)
    return C.cast(a, C.c_void_p)


def pinned_empty(shape, dtype) -> np.ndarray:
    """numpy array over cudaHostAlloc'ed (pinned) memory; freed when the array is collected."""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape)) * dtype.itemsize
    ptr = C.c_void_p()
    rc = lib().lk_host_alloc(C.byref(ptr), max(n, 1))
    if rc:
        raise LkError(rc, "cudaHostAlloc failed")
    buf = (C.c_char * max(n, 1)).from_address(ptr.value)
    arr = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)

    class _Owner:
        def __init__(self, p):
            self.p = p

        def __del__(self):
            try:
                lib().lk_host_free(self.p)
            except Exception:
                pass
    _OWNERS[arr.ctypes.data] = _Owner(ptr)
    return arr


_OWNERS: dict = {}


class Engine:
    """One device context: extrinsics + ESKF / map configuration + the map in HBM.
    Mirrors what KILO owns (legkilo/src/core/slam/KILO.h:48-63)."""

    def __init__(self, cfg: dict, device: int = 0):
        self.cfg = cfg
        self._ec = abi.eskf_cfg(cfg)
        self._mc = abi.map_cfg(cfg)
        R, t = abi.extrinsics(cfg)
        self._R, self._t = R, t
        self.h = C.c_void_p()
        rc = lib().lk_create(C.byref(self._ec), C.byref(self._mc), _p(R), _p(t), device, C.byref(self.h))
        if rc:
            raise LkError(rc, lib().lk_last_error(None).decode())

    def close(self):
        if getattr(self, "h", None) is not None and self.h:
            lib().lk_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _chk(self, rc):
        if rc:
            raise LkError(rc, lib().lk_last_error(self.h).decode())

    def set_param(self, name: str, value: float):
        self._chk(lib().lk_set_param(self.h, name.encode(), float(value)))

    # ---- map ---------------------------------------------------------------------------------
    def map_reserve(self, max_roots: int, max_nodes: int, max_points: int):
        self._chk(lib().lk_map_reserve(self.h, max_roots, max_nodes, max_points))

    def map_upload(self, blob: np.ndarray):
        blob = np.ascontiguousarray(blob, np.uint8)
        self._chk(lib().lk_map_upload(self.h, _p(blob), blob.size))

    def map_download(self) -> np.ndarray:
        sz = C.c_size_t(0)
        self._chk(lib().lk_map_download(self.h, None, 0, C.byref(sz)))
        buf = np.zeros(sz.value, np.uint8)
        self._chk(lib().lk_map_download(self.h, _p(buf), buf.size, C.byref(sz)))
        return buf[:sz.value]

    def map_build(self, xyz_world, xyz_body, R=None, rot_cov=None, pos_cov=None):
        xyz_world = np.ascontiguousarray(xyz_world, np.float32)
        xyz_body = np.ascontiguousarray(xyz_body, np.float32)
        R = np.eye(3) if R is None else np.ascontiguousarray(R, np.float64)
        rot_cov = 1e-6 * np.eye(3) if rot_cov is None else np.ascontiguousarray(rot_cov, np.float64)
        pos_cov = 1e-6 * np.eye(3) if pos_cov is None else np.ascontiguousarray(pos_cov, np.float64)
        self._chk(lib().lk_map_build(self.h, _p(xyz_world), _p(xyz_body), len(xyz_world), _p(R), _p(rot_cov),
                                     _p(pos_cov)))

    def first_frame(self, x, pts, end_time, imu=None, kin=None, gravity=9.81, world=True):
        """lk_first_frame: the first frame of KILO::process (KILO.cc:331-353) on a raw float32 [n, 4] lidar cloud and the
        frame's inertial queue (exactly one of imu / kin): StateInitial, the world cloud at the prior's position and the
        map build. Returns x, P [900], clk, acc_norm and the world cloud (float32 [n, 4], None when world is False)."""
        x = np.array(x, abi.STATE_DTYPE, copy=True).reshape(1)
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
        imu = None if imu is None else np.ascontiguousarray(imu, abi.IMU_DTYPE)
        kin = None if kin is None else np.ascontiguousarray(kin, abi.KINIMU_DTYPE)
        nm = len(imu) if imu is not None else (len(kin) if kin is not None else 0)
        P = np.zeros(900); clk = np.zeros(1, abi.CLOCK_DTYPE); acc_norm = C.c_double(0.0)
        out = np.zeros((len(pts), 4), np.float32) if world else None
        self._chk(lib().lk_first_frame(self.h, _p(x), _p(P), _p(clk), C.byref(acc_norm), _p(pts), len(pts), float(end_time),
                                       _p(imu), _p(kin), nm, float(gravity), _p(out)))
        return dict(x=x, P=P, clk=clk, acc_norm=acc_norm.value, world=out)

    def map_insert(self, pts, set_offsets, rot, pos, rot_cov, pos_cov):
        """lk_map_insert: UpdateVoxelMap of point sets at known poses. pts float32 [n, 4] (lidar frame), set_offsets
        [n_sets + 1]; per set rot [n_sets, 3, 3], pos [n_sets, 3], rot_cov / pos_cov [n_sets, 3, 3]."""
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
        so = np.ascontiguousarray(set_offsets, np.uint32)
        n_sets = len(so) - 1
        rot, pos, rot_cov, pos_cov = (np.ascontiguousarray(a, np.float64).reshape(n_sets, k)
                                      for a, k in ((rot, 9), (pos, 3), (rot_cov, 9), (pos_cov, 9)))
        self._chk(lib().lk_map_insert(self.h, n_sets, _p(pts), _p(so), _p(rot), _p(pos), _p(rot_cov), _p(pos_cov)))

    def score_poses(self, pts, set_offsets, pose_set, rot, pos, rot_cov, pos_cov):
        """lk_score_poses: the sums of the LiDAR update at every candidate pose, against the map, touching nothing.
        pts float32 [n, 4] (lidar frame), set_offsets [n_sets + 1]; per pose pose_set [n_poses], rot [n_poses, 3, 3],
        pos [n_poses, 3]; rot_cov / pos_cov [3, 3] shared by every pose. Returns float64 [n_poses, 32], laid out as
        abi.SCORE_* (A upper triangle | b | sum R | count | sum z^2 / R | 0 0)."""
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
        so = np.ascontiguousarray(set_offsets, np.uint32).reshape(-1)
        if len(so) < 1:
            raise ValueError("set_offsets needs n_sets + 1 entries")
        if len(pts) < int(so[-1]):
            raise ValueError(f"set_offsets ends at point {int(so[-1])}, pts has {len(pts)}")
        ps = np.ascontiguousarray(pose_set, np.uint32).reshape(-1)
        n_poses = len(ps)
        rot = np.ascontiguousarray(rot, np.float64).reshape(n_poses, 9)
        pos = np.ascontiguousarray(pos, np.float64).reshape(n_poses, 3)
        rot_cov = np.ascontiguousarray(rot_cov, np.float64).reshape(9)
        pos_cov = np.ascontiguousarray(pos_cov, np.float64).reshape(9)
        out = np.zeros((n_poses, abi.SCORE_STRIDE))
        self._chk(lib().lk_score_poses(self.h, len(so) - 1, _p(pts), _p(so), n_poses, _p(ps), _p(rot), _p(pos), _p(rot_cov),
                                       _p(pos_cov), _p(out)))
        return out

    def refine_poses(self, pts, set_offsets, pose_set, rot, pos, rot_cov, pos_cov, iters, want_records=True):
        """lk_refine_poses: every candidate pose refined by `iters` steps of the LiDAR update with P's theta / position
        blocks held at rot_cov / pos_cov, against the map, touching nothing. Inputs as score_poses. Returns (rot
        [n_poses, 3, 3], pos [n_poses, 3], records float64 [n_poses, 32] at the refined poses, or None without
        want_records)."""
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
        so = np.ascontiguousarray(set_offsets, np.uint32).reshape(-1)
        if len(so) < 1:
            raise ValueError("set_offsets needs n_sets + 1 entries")
        if len(pts) < int(so[-1]):
            raise ValueError(f"set_offsets ends at point {int(so[-1])}, pts has {len(pts)}")
        ps = np.ascontiguousarray(pose_set, np.uint32).reshape(-1)
        n_poses = len(ps)
        rot = np.ascontiguousarray(rot, np.float64).reshape(n_poses, 9)
        pos = np.ascontiguousarray(pos, np.float64).reshape(n_poses, 3)
        rot_cov = np.ascontiguousarray(rot_cov, np.float64).reshape(9)
        pos_cov = np.ascontiguousarray(pos_cov, np.float64).reshape(9)
        rot_out, pos_out = np.zeros((n_poses, 3, 3)), np.zeros((n_poses, 3))
        rec = np.zeros((n_poses, abi.SCORE_STRIDE)) if want_records else None
        self._chk(lib().lk_refine_poses(self.h, len(so) - 1, _p(pts), _p(so), n_poses, _p(ps), _p(rot), _p(pos),
                                        _p(rot_cov), _p(pos_cov), int(iters), _p(rot_out), _p(pos_out),
                                        None if rec is None else _p(rec)))
        return rot_out, pos_out, rec

    def search_poses(self, pts, set_offsets, att_offsets, att_rot, origin, step, counts, rot_cov, pos_cov, iters,
                     rot_cov_tight, pos_cov_tight, k):
        """lk_search_poses: per set, a lattice of candidate poses (its attitudes att_rot[att_offsets[s]:att_offsets[s + 1]]
        times counts = (nx, ny, nz) positions spaced step from origin[s]) scored with rot_cov / pos_cov, the best k kept,
        refined by `iters` steps, re-scored with rot_cov_tight / pos_cov_tight and ordered by that count, all on the
        device. Returns (rot [n_sets, k, 3, 3], pos [n_sets, k, 3], tight records float64 [n_sets, k, 32], candidate
        index uint32 [n_sets, k])."""
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
        so = np.ascontiguousarray(set_offsets, np.uint32).reshape(-1)
        ao = np.ascontiguousarray(att_offsets, np.uint32).reshape(-1)
        if len(so) < 1 or len(ao) != len(so):
            raise ValueError("set_offsets and att_offsets need n_sets + 1 entries each")
        if len(pts) < int(so[-1]):
            raise ValueError(f"set_offsets ends at point {int(so[-1])}, pts has {len(pts)}")
        n_sets = len(so) - 1
        att = np.ascontiguousarray(att_rot, np.float64).reshape(-1, 9)
        if len(att) < int(ao[-1]):
            raise ValueError(f"att_offsets ends at attitude {int(ao[-1])}, att_rot has {len(att)}")
        org = np.ascontiguousarray(origin, np.float64).reshape(n_sets, 3)
        st = np.ascontiguousarray(step, np.float64).reshape(3)
        cn = np.ascontiguousarray(counts, np.uint32).reshape(3)
        covs = [np.ascontiguousarray(c, np.float64).reshape(9) for c in (rot_cov, pos_cov, rot_cov_tight, pos_cov_tight)]
        k = int(k)
        rot_out, pos_out = np.zeros((n_sets, k, 3, 3)), np.zeros((n_sets, k, 3))
        rec, cand = np.zeros((n_sets, k, abi.SCORE_STRIDE)), np.zeros((n_sets, k), np.uint32)
        self._chk(lib().lk_search_poses(self.h, n_sets, _p(pts), _p(so), _p(ao), _p(att), _p(org), _p(st), _p(cn),
                                        _p(covs[0]), _p(covs[1]), int(iters), _p(covs[2]), _p(covs[3]), k, _p(rot_out),
                                        _p(pos_out), _p(rec), _p(cand)))
        return rot_out, pos_out, rec, cand

    def scorer_scratch(self):
        """lk_debug_read(h, 4): (device bytes, page-locked bytes) the pose scorer holds."""
        out = np.zeros(2, np.uint64)
        self._chk(lib().lk_debug_read(self.h, 4, _p(out), out.nbytes))
        return int(out[0]), int(out[1])

    def map_slide(self, position):
        """VoxelMapManager::mapSliding (voxel_map.cc:552-571). Returns (slid, removed root voxels)."""
        pos = np.ascontiguousarray(position, np.float64)
        slid = C.c_int32(0); removed = C.c_uint64(0)
        self._chk(lib().lk_map_slide(self.h, _p(pos), C.byref(slid), C.byref(removed)))
        return bool(slid.value), int(removed.value)

    def map_stats(self):
        out = np.zeros(4, np.uint64)
        self._chk(lib().lk_map_stats(self.h, _p(out)))
        return dict(roots=int(out[0]), nodes=int(out[1]), points=int(out[2]), planes=int(out[3]))

    def map_memory(self):
        """lk_map_memory: bump-allocated and free-listed nodes / point slots, pool bytes, pool reallocations."""
        out = np.zeros(6, np.uint64)
        self._chk(lib().lk_map_memory(self.h, _p(out)))
        return dict(nodes=int(out[0]), free_nodes=int(out[1]), point_slots=int(out[2]), free_point_slots=int(out[3]),
                    pool_bytes=int(out[4]), reallocs=int(out[5]))

    # ---- hot path ------------------------------------------------------------------------------
    @staticmethod
    def _norm_batch(x, P, clk, pts, scan_offsets, scan_bucket_ptr, bucket_offsets, bucket_times):
        x = np.ascontiguousarray(x, abi.STATE_DTYPE)
        batch = len(x)
        P = np.ascontiguousarray(P, np.float64).reshape(batch, 900)
        clk = np.ascontiguousarray(clk, abi.CLOCK_DTYPE)
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
        scan_offsets = np.ascontiguousarray(scan_offsets, np.uint32)
        if scan_bucket_ptr is None:  # one bucket per scan
            scan_bucket_ptr = np.arange(batch + 1, dtype=np.uint32)
            bucket_offsets = scan_offsets
        scan_bucket_ptr = np.ascontiguousarray(scan_bucket_ptr, np.uint32)
        bucket_offsets = np.ascontiguousarray(bucket_offsets, np.uint32)
        bucket_times = np.ascontiguousarray(bucket_times, np.float64)
        assert len(scan_offsets) == batch + 1 and len(scan_bucket_ptr) == batch + 1
        assert len(bucket_offsets) == scan_bucket_ptr[-1] + 1 and len(bucket_times) == scan_bucket_ptr[-1]
        return x, P, clk, pts, scan_offsets, scan_bucket_ptr, bucket_offsets, bucket_times

    def scan_update(self, x, P, Q, clk, pts, scan_offsets, bucket_times, scan_bucket_ptr=None, bucket_offsets=None,
                    iters=1, update_map=False, want_world=True, pinned=False):
        """lk_scan_update: host buffers in, host buffers out (copies of x / P / clk are returned).
        pinned=True puts the points and the world cloud in page-locked memory (lk_host_alloc), which lets a
        one-scan call run in direct mode (the kernel reads / writes them in place)."""
        x, P, clk, pts, so, sbp, bo, bt = self._norm_batch(x, P, clk, pts, scan_offsets, scan_bucket_ptr,
                                                           bucket_offsets, bucket_times)
        x = x.copy(); P = P.copy(); clk = clk.copy()
        Q = np.ascontiguousarray(Q, np.float64)
        if pinned:
            hp = pinned_empty(pts.shape, np.float32); hp[...] = pts; pts = hp
            world = pinned_empty((len(pts), 4), np.float32) if want_world else None
            if world is not None:
                world[...] = 0
        else:
            world = np.zeros((len(pts), 4), np.float32) if want_world else None
        neff = np.zeros(len(x), np.uint32)
        self._chk(lib().lk_scan_update(self.h, len(x), _p(x), _p(P), _p(Q), _p(clk), _p(pts), _p(so), _p(sbp), _p(bo),
                                       _p(bt), iters, int(update_map), _p(world), _p(neff)))
        return dict(x=x, P=P, clk=clk, world=world, n_eff=neff)

    def stage(self, x, P, Q, clk, pts, scan_offsets, bucket_times, scan_bucket_ptr=None, bucket_offsets=None):
        x, P, clk, pts, so, sbp, bo, bt = self._norm_batch(x, P, clk, pts, scan_offsets, scan_bucket_ptr,
                                                           bucket_offsets, bucket_times)
        Q = np.ascontiguousarray(Q, np.float64)
        self._staged = (len(x), len(pts))
        self._chk(lib().lk_batch_stage(self.h, len(x), _p(x), _p(P), _p(Q), _p(clk), _p(pts), _p(so), _p(sbp), _p(bo),
                                       _p(bt)))

    def run(self, iters=1, update_map=False):
        self._chk(lib().lk_batch_run(self.h, iters, int(update_map)))

    def run_range(self, first, count, iters=1, update_map=False):
        """Asynchronous: enqueue scans [first, first+count) of the staged batch (no host sync)."""
        self._chk(lib().lk_batch_run_range(self.h, first, count, iters, int(update_map)))

    def timer_start(self):
        self._chk(lib().lk_timer_start(self.h))

    def timer_stop(self):
        t = C.c_float(); r = C.c_float(); n = C.c_uint32(); nr = C.c_uint32()
        self._chk(lib().lk_timer_stop(self.h, C.byref(t), C.byref(r), C.byref(n), C.byref(nr)))
        return dict(total_ms=t.value, residual_ms=r.value, launches=n.value, residual_launches=nr.value)

    def sync(self):
        self._chk(lib().lk_sync(self.h))

    def fetch(self, want_world=True):
        batch, npts = self._staged
        x = np.zeros(batch, abi.STATE_DTYPE); P = np.zeros((batch, 900)); clk = np.zeros(batch, abi.CLOCK_DTYPE)
        world = np.zeros((npts, 4), np.float32) if want_world else None
        neff = np.zeros(batch, np.uint32)
        self._chk(lib().lk_batch_fetch(self.h, _p(x), _p(P), _p(clk), _p(world), _p(neff)))
        return dict(x=x, P=P, clk=clk, world=world, n_eff=neff)

    def last_timing(self):
        t = C.c_float(); r = C.c_float(); n = C.c_uint32(); nr = C.c_uint32()
        self._chk(lib().lk_batch_last_timing(self.h, C.byref(t), C.byref(r), C.byref(n), C.byref(nr)))
        return dict(total_ms=t.value, residual_ms=r.value, launches=n.value, residual_launches=nr.value)

    def debug_residuals(self, x, P, pts):
        x = np.ascontiguousarray(x, abi.STATE_DTYPE); P = np.ascontiguousarray(P, np.float64)
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
        n = len(pts)
        ok = np.zeros(n, np.uint8); h = np.zeros((n, 6)); z = np.zeros(n); R = np.zeros(n)
        key = np.zeros((n, 3), np.int32)
        self._chk(lib().lk_debug_residuals(self.h, _p(x), _p(P), _p(pts), n, _p(ok), _p(h), _p(z), _p(R), _p(key)))
        return dict(ok=ok, h=h, z=z, R=R, key=key)

    def update_by_points(self, x, P, h, z, R):
        """ESKF::updateByPoints (eskf.cc:91-113) from explicit rows."""
        x = np.array(x, abi.STATE_DTYPE, copy=True); P = np.array(P, np.float64, copy=True).reshape(900)
        h = np.ascontiguousarray(h, np.float64).reshape(-1, 6); z = np.ascontiguousarray(z, np.float64)
        R = np.ascontiguousarray(R, np.float64)
        self._chk(lib().lk_update_by_points(self.h, _p(x), _p(P), len(z), _p(h), _p(z), _p(R)))
        return x, P

    def obs_imu(self, x, P, Q, clk, imu, gravity=9.81, acc_norm=1.0):
        """KILO::predictUpdateImu per sample (KILO.cc:235-258)."""
        x = np.array(x, abi.STATE_DTYPE, copy=True); P = np.array(P, np.float64, copy=True).reshape(900)
        clk = np.array(clk, abi.CLOCK_DTYPE, copy=True); Q = np.ascontiguousarray(Q, np.float64)
        imu = np.ascontiguousarray(imu, abi.IMU_DTYPE)
        self._chk(lib().lk_obs_imu(self.h, _p(x), _p(P), _p(Q), _p(clk), _p(imu), len(imu), gravity, acc_norm))
        return x, P, clk

    def obs_kinimu(self, x, P, Q, clk, kin, gravity=9.81, acc_norm=1.0):
        """KILO::predictUpdateKinImu per sample (KILO.cc:260-314)."""
        x = np.array(x, abi.STATE_DTYPE, copy=True); P = np.array(P, np.float64, copy=True).reshape(900)
        clk = np.array(clk, abi.CLOCK_DTYPE, copy=True); Q = np.ascontiguousarray(Q, np.float64)
        kin = np.ascontiguousarray(kin, abi.KINIMU_DTYPE)
        self._chk(lib().lk_obs_kinimu(self.h, _p(x), _p(P), _p(Q), _p(clk), _p(kin), len(kin), gravity, acc_norm))
        return x, P, clk

    def process_scan(self, x, P, Q, clk, pts, bucket_offsets, bucket_times, imu=None, kin=None, gravity=9.81, acc_norm=1.0,
                     iters=1, update_map=True):
        """The second lambda of KILO::process (KILO.cc:367-396) for one scan, inertial / kinematic queue
        interleaved on the device."""
        x = np.array(x, abi.STATE_DTYPE, copy=True); P = np.array(P, np.float64, copy=True).reshape(900)
        clk = np.array(clk, abi.CLOCK_DTYPE, copy=True); Q = np.ascontiguousarray(Q, np.float64)
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
        bo = np.ascontiguousarray(bucket_offsets, np.uint32); bt = np.ascontiguousarray(bucket_times, np.float64)
        imu = None if imu is None else np.ascontiguousarray(imu, abi.IMU_DTYPE)
        kin = None if kin is None else np.ascontiguousarray(kin, abi.KINIMU_DTYPE)
        nm = len(imu) if imu is not None else (len(kin) if kin is not None else 0)
        world = np.zeros((len(pts), 4), np.float32); neff = np.zeros(1, np.uint32); ncons = np.zeros(1, np.uint32)
        self._chk(lib().lk_process_scan(self.h, _p(x), _p(P), _p(Q), _p(clk), _p(pts), len(pts), _p(bo), _p(bt), len(bt), _p(imu),
                                        _p(kin), nm, gravity, acc_norm, iters, int(update_map), _p(world), _p(neff), _p(ncons)))
        return dict(x=x, P=P, clk=clk, world=world, n_eff=int(neff[0]), n_consumed=int(ncons[0]))

    def decode_pointcloud2(self, data, layout, blind, filter_num, time_scale):
        """lk_decode_pointcloud2: raw PointCloud2 bytes -> float4 (x, y, z, curvature) + intensity."""
        data = np.ascontiguousarray(data, np.uint8)
        n = data.size // layout.point_step
        pts = np.zeros((n, 4), np.float32); inten = np.zeros(n, np.float32)
        no = np.zeros(1, np.uint32); ft = np.zeros(1); lt = np.zeros(1)
        self._chk(lib().lk_decode_pointcloud2(self.h, _p(data), n, C.byref(layout), blind, filter_num, time_scale, _p(pts),
                                              _p(inten), _p(no), _p(ft), _p(lt)))
        return pts[:no[0]].copy(), inten[:no[0]].copy(), float(ft[0]), float(lt[0])

    def decode_pointcloud2s(self, messages, layout, blind, filter_num, time_scale, stamps=None):
        """lk_decode_pointcloud2s: decode_pointcloud2 of every message of a batch in one call. `messages` is a list of
        uint8 arrays or structured point arrays (viewed as bytes here), each a whole number of layout.point_step points;
        stamps [len(messages)] are the header stamps (None = 0). Returns pts float32 [n, 4], offsets [len(messages) + 1]
        (message m is pts[offsets[m]:offsets[m + 1]]), intensity, begin_times and end_times, ready for
        preprocess_scans(pts, offsets, leaf, begin_times)."""
        step = layout.point_step
        data = [np.ascontiguousarray(m).reshape(-1).view(np.uint8) for m in messages]
        for i, d in enumerate(data):
            if d.size % step:
                raise ValueError(f"message {i} has {d.size} bytes, not a multiple of point_step {step}")
        n_msgs = len(data)
        if stamps is not None:
            stamps = np.ascontiguousarray(stamps, np.float64).reshape(-1)
            if len(stamps) != n_msgs:
                raise ValueError(f"{len(stamps)} stamps for {n_msgs} messages")
        ptrs = (C.c_void_p * max(n_msgs, 1))(*[d.ctypes.data for d in data])
        counts = np.array([d.size // step for d in data], np.uint32)
        cap = max(int(counts.sum(dtype=np.int64)), 1)
        pts = np.zeros((cap, 4), np.float32); inten = np.zeros(cap, np.float32); offs = np.zeros(n_msgs + 1, np.uint32)
        bt = np.zeros(n_msgs); et = np.zeros(n_msgs)
        self._chk(lib().lk_decode_pointcloud2s(self.h, n_msgs, ptrs, _p(counts), _p(stamps), C.byref(layout), blind, filter_num,
                                               time_scale, _p(pts), _p(inten), _p(offs), _p(bt), _p(et)))
        n_out = int(offs[-1])
        return dict(pts=pts[:n_out].copy(), offsets=offs, intensity=inten[:n_out].copy(), begin_times=bt, end_times=et)

    def preprocess_scan(self, pts, leaf):
        """lk_preprocess_scan: voxel-grid centroid filter, stable curvature sort, bucket boundaries."""
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
        n = len(pts)
        out = np.zeros((n, 4), np.float32); offs = np.zeros(n + 1, np.uint32); curv = np.zeros(max(n, 1), np.float32)
        no = np.zeros(1, np.uint32); nb = np.zeros(1, np.uint32)
        self._chk(lib().lk_preprocess_scan(self.h, _p(pts), n, leaf, _p(out), _p(no), _p(offs), _p(curv), _p(nb)))
        return out[:no[0]].copy(), offs[:nb[0] + 1].copy(), curv[:nb[0]].copy()

    def preprocess_scans(self, pts, in_offsets, leaf, begin_times=None):
        """lk_preprocess_scans: preprocess_scan of every scan of a batch in one call. pts float32 [n, 4] (x, y, z,
        curvature), scan s = pts[in_offsets[s]:in_offsets[s + 1]]. Returns the batch layout scan_update / stage take:
        pts, scan_offsets, scan_bucket_ptr, bucket_offsets, bucket_times (begin_times[s] + curvature; None when
        begin_times is None) and bucket_curvature."""
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
        io = np.ascontiguousarray(in_offsets, np.uint32).reshape(-1)
        if len(io) < 1:
            raise ValueError("in_offsets needs n_scans + 1 entries")
        if len(pts) < int(io[-1]):
            raise ValueError(f"in_offsets ends at point {int(io[-1])}, pts has {len(pts)}")
        n_scans = len(io) - 1
        cap = max(int(io[-1]), 1)
        out = np.zeros((cap, 4), np.float32); so = np.zeros(n_scans + 1, np.uint32); sbp = np.zeros(n_scans + 1, np.uint32)
        bo = np.zeros(cap + 1, np.uint32); bc = np.zeros(cap, np.float32)
        bt = None
        if begin_times is not None:
            begin_times = np.ascontiguousarray(begin_times, np.float64)
            assert len(begin_times) == n_scans
            bt = np.zeros(cap)
        self._chk(lib().lk_preprocess_scans(self.h, n_scans, _p(pts), _p(io), leaf, _p(begin_times), _p(out), _p(so), _p(sbp),
                                            _p(bo), _p(bc), _p(bt)))
        n_out, n_b = int(so[-1]), int(sbp[-1])
        return dict(pts=out[:n_out].copy(), scan_offsets=so, scan_bucket_ptr=sbp, bucket_offsets=bo[:n_b + 1].copy(),
                    bucket_times=None if bt is None else bt[:n_b].copy(), bucket_curvature=bc[:n_b].copy())

    def leg_kinematics(self, states, cfg, track=None, redundancy=True):
        """lk_leg_kinematics: unitree HighState fields (abi.LEG_STATE_DTYPE) -> kinematic-inertial samples
        (abi.KINIMU_DTYPE), the redundancy drop and the contact detectors carried by `track` (abi.LkLegTrack; None =
        the reference's initial state). `cfg` is a configuration dict or an abi.LkLegCfg. Returns (kin, new track)."""
        states = np.ascontiguousarray(states, abi.LEG_STATE_DTYPE)
        lc = cfg if isinstance(cfg, abi.LkLegCfg) else abi.leg_cfg(cfg)
        tr = abi.LkLegTrack()
        if track is None:
            self._chk(lib().lk_leg_track_default(C.byref(tr)))
        else:
            C.memmove(C.byref(tr), C.byref(track), C.sizeof(tr))
        out = np.zeros(len(states), abi.KINIMU_DTYPE)
        no = C.c_uint32(0)
        self._chk(lib().lk_leg_kinematics(self.h, C.byref(lc), _p(states), len(states), int(bool(redundancy)), C.byref(tr),
                                          _p(out), C.byref(no)))
        return out[:no.value].copy(), tr

    def predict(self, x, P, Q, dt, prop_state=True, prop_cov=True):
        x = np.array(x, abi.STATE_DTYPE, copy=True); batch = len(x)
        P = np.array(P, np.float64, copy=True).reshape(batch, 900)
        Q = np.ascontiguousarray(Q, np.float64); dt = np.ascontiguousarray(dt, np.float64)
        self._chk(lib().lk_predict(self.h, batch, _p(x), _p(P), _p(Q), _p(dt), int(prop_state), int(prop_cov)))
        return x, P
