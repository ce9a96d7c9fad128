/*
 * legkilo_b200.h — C ABI of the H100-native Leg-KILO LiDAR measurement-update path.
 *
 * This is the drop-in boundary (SURVEY.md §8b). The reference has no FFI: the seam is the C++
 * member call `KILO::process` -> `KILO::predictUpdatePoint` (legkilo/src/core/slam/KILO.cc:316,
 * :108) which in turn drives `ESKF` (legkilo/src/core/slam/eskf.h:46-109) and `VoxelMapManager`
 * (legkilo/src/core/slam/voxel_map.h:180-244). Every entry point below names the reference
 * member it replaces. Plain pointers and sizes only; host pointers unless a name ends in `_dev`;
 * never throws; 0 = success, negative = lk_status error code, message via lk_last_error().
 *
 * All matrices are row-major doubles. The error-state layout is the reference's
 * (legkilo/src/core/slam/eskf.cc:18-29): theta 0-2, pos 3-5, vel 6-8, ba 9-11, bw 12-14,
 * grav 15-17, imu_a 18-20, imu_w 21-23, bv 24-26, contact 27-29.
 */
#ifndef LEGKILO_B200_H_
#define LEGKILO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LK_DIM_STATE 30
#define LK_ABI_VERSION 1

typedef enum lk_status {
    LK_OK = 0,
    LK_ERR_INVALID_ARG = -1,
    LK_ERR_CUDA = -2,
    LK_ERR_NO_DEVICE = -3,
    LK_ERR_OUT_OF_MEMORY = -4,
    LK_ERR_BAD_BLOB = -5,
    LK_ERR_CAPACITY = -6,
    LK_ERR_NOT_READY = -7
} lk_status;

/* = legkilo::State (eskf.h:15-32). rot is row-major R (body -> world). 36 doubles. */
typedef struct lk_state {
    double rot[9];
    double pos[3];
    double vel[3];
    double ba[3];
    double bw[3];
    double grav[3];
    double imu_a[3];
    double imu_w[3];
    double bv[3];
    double contact[3];
} lk_state;

/* = legkilo::ESKF::Config (eskf.h:49-65), same field order. */
typedef struct lk_eskf_cfg {
    double vel_process_cov;
    double imu_acc_process_cov;
    double imu_gyr_process_cov;
    double contact_process_cov;
    double acc_bias_process_cov;
    double gyr_bias_process_cov;
    double kin_bias_process_cov;
    double imu_acc_meas_noise;
    double imu_acc_z_meas_noise;
    double imu_gyr_meas_noise;
    double kin_meas_noise;
    double chd_meas_noise;
    double contact_meas_noise;
    double lidar_point_meas_ratio;
} lk_eskf_cfg;

/* = legkilo::VoxelMapConfig (voxel_map.h:41-57). */
typedef struct lk_map_cfg {
    double max_voxel_size;     /* voxel_size */
    double planner_threshold;  /* min_eigen_value */
    double beam_err;           /* degrees */
    double dept_err;           /* metres */
    double sigma_num;
    double sliding_thresh;     /* read, unused by the reference hot path */
    int32_t max_layer;
    int32_t max_iterations;    /* declared by the reference, never read (voxel_map.h:44) */
    int32_t max_points_num;
    int32_t layer_init_num[5];
    int32_t is_pub_plane_map;
    int32_t map_sliding_en;
    int32_t half_map_size;
    int32_t reserved;
} lk_map_cfg;

/* KILO::last_state_predict_time_ / last_state_update_time_ (KILO.h:56-57), one per scan stream. */
typedef struct lk_stream_clock {
    double last_predict_time;
    double last_update_time;
} lk_stream_clock;

/* One inertial sample for KILO::predictUpdateImu (KILO.cc:235-258). */
typedef struct lk_imu_meas {
    double stamp;
    double acc[3];
    double gyr[3];
} lk_imu_meas;

/* = legkilo::common::KinImuMeas (sensor_types.hpp:19-26); contact as int32 instead of bool. */
typedef struct lk_kinimu_meas {
    double stamp;
    double foot_pos[4][3];
    double foot_vel[4][3];
    int32_t contact[4];
    double acc[3];
    double gyr[3];
} lk_kinimu_meas;

/* ------------------------------------------------------------------------------------------
 * Map blob (lk_map_upload / lk_map_download): an implementation-neutral dump of the voxel map,
 * i.e. of `unordered_map<Vector3i, VoxelOctoTree*>` (voxel_map.h:186) with every octree node's
 * cached plane (VoxelPlane, voxel_map.h:96-119) and retained points (temp_points_, :132).
 * Layout: header | roots[n_roots] | nodes[n_nodes] | aux[n_nodes] | points[n_points].
 * ------------------------------------------------------------------------------------------ */
#define LK_MAP_MAGIC 0x504D4B4Cu /* "LKMP" */

#define LK_NODE_IS_PLANE 0x1u       /* plane_ptr_->is_plane_ */
#define LK_NODE_INIT_OCTO 0x2u      /* init_octo_ */
#define LK_NODE_UPDATE_ENABLE 0x4u  /* update_enable_ */
#define LK_NODE_LAYER_SHIFT 8       /* bits 8..15  : layer_ */
#define LK_NODE_CHILDMASK_SHIFT 16  /* bits 16..23 : leaves_[i] != nullptr */

typedef struct lk_map_blob_header {
    uint32_t magic;
    uint32_t version;
    uint32_t n_roots;
    uint32_t n_nodes;
    uint64_t n_points;
    uint32_t reserved[2];
} lk_map_blob_header; /* 32 B */

typedef struct lk_map_root {
    int32_t key[3]; /* voxelKeyFloor (eigen_types.hpp:89-95) */
    int32_t node;   /* index into nodes[] */
} lk_map_root; /* 16 B */

/* The 232 bytes the residual kernel reads (voxel_map.cc:371-403), padded to 256. */
typedef struct lk_map_node {
    double center[3];    /* VoxelPlane::center_ */
    double normal[3];    /* VoxelPlane::normal_ */
    double plane_var[21]; /* upper triangle of VoxelPlane::plane_var_, row-major (00 01..05 11 12..55) */
    float d;             /* VoxelPlane::d_ (float in the reference) */
    float radius;        /* VoxelPlane::radius_ (float in the reference) */
    uint32_t flags;      /* LK_NODE_* */
    int32_t child_base;  /* index of 8 contiguous child nodes (leaves_[0..7]) or -1 */
    uint32_t pad[6];
} lk_map_node; /* 256 B */

typedef struct lk_map_aux {
    double voxel_center[3]; /* VoxelOctoTree::voxel_center_ */
    float quater_length;    /* VoxelOctoTree::quater_length_ */
    uint32_t pts_base;      /* first retained point in points[] */
    int32_t pts_count;      /* temp_points_.size() */
    int32_t pts_cap;        /* device capacity (ignored on upload) */
    int32_t new_points;     /* new_points_ */
    int32_t parent;         /* parent node index, -1 for a root */
    int32_t key[3];         /* root key (roots only) */
    int32_t pad;
} lk_map_aux; /* 64 B */

typedef struct lk_map_point {
    double pw[3];  /* pointWithVar::point_w */
    double var[6]; /* upper triangle of pointWithVar::var: xx xy xz yy yz zz */
} lk_map_point; /* 72 B */

typedef struct lk_context* lk_handle;

/* ---- lifecycle ------------------------------------------------------------------------- */

/* Replaces KILO::initializeFromYaml's construction of ESKF / VoxelMapManager / extrinsics
 * (KILO.cc:25-84). `device` is the CUDA ordinal. Fails with LK_ERR_NO_DEVICE when no CUDA
 * device is usable — there is no CPU fallback. */
int lk_create(const lk_eskf_cfg* eskf_cfg, const lk_map_cfg* map_cfg, const double ext_rot[9],
              const double ext_t[3], int device, lk_handle* out);
int lk_destroy(lk_handle h);
const char* lk_last_error(lk_handle h); /* h may be NULL: returns the last create-time error */
int lk_abi_version(void);

/* ESKF::initProcessCovQ (eskf.cc:47-62): fills Q[900] from the ESKF config. Host-side helper. */
int lk_init_process_cov(const lk_eskf_cfg* cfg, double* Q900);
/* State::State() (eskf.cc:5-16). */
int lk_state_default(lk_state* x);

/* Page-locked host memory (cudaHostAlloc / cudaFreeHost). A one-scan lk_scan_update whose `pts` and
 * `pts_world_out` live in page-locked memory (from here or cudaHostRegister) runs in DIRECT mode: nothing
 * is staged, the kernel reads the points and stores the world cloud / filter in place (DESIGN.md 3.7). */
int lk_host_alloc(void** p, size_t bytes);
int lk_host_free(void* p);
/* Tuning / diagnostic knobs by name. Results never depend on them beyond floating-point summation order.
 *   "fused"       1 (default) one scan per call runs as ONE persistent kernel; 0 = multi-kernel path
 *   "lane_cache"  1 (default) keep per-lane lookups across the iterations of a bucket (fused kernel)
 *   "direct_io"   1 (default) allow the direct mode of lk_scan_update; "inline_in" 1 = small inputs ride in
 *                 the kernel parameter block in direct mode
 *   "pdl"         1 (default) back-to-back fused launches of one stream use programmatic dependent launch: the
 *                 next scan's blocks run their prologue while the previous scan's last blocks drain
 *   "coop_launch" 1 = launch the fused kernel through cudaLaunchCooperativeKernel (co-residency checked by the
 *                 driver; for devices shared with OTHER processes, see INTEGRATION.md "Sharing a device")
 *   "fast_insert" 1 (default) UpdateVoxelMap of a bucket of <= 4096 points takes two launches instead of five
 *   "fused_insert" 0 (default); 1 = a streaming scan (update_map) runs entirely inside ONE persistent kernel, the map
 *                 insert included (DESIGN.md 3.5; currently slower than the per-bucket kernels)
 *   "slim_p"      1 (default) blocks that never read the full covariance load only the strip they need (fused kernel)
 *   "debug_records" 0 (default) lk_debug_residuals evaluates the hot plane images, as calls with a fixed map do;
 *                 1 = the node records, as calls with update_map do (the two round sigma_plane differently)
 *   "kernel_timing", "trace": measurement / debugging aids
 * Any other name fails with LK_ERR_INVALID_ARG. */
int lk_set_param(lk_handle h, const char* name, double value);

/* Debug read-back (what: 0 = per-chunk partial sums, 1 = scan constants, 2 = %globaltimer trace,
 * 3 = host-side phase times of lk_scan_update [stage, enqueue, wait+fetch, calls] in ns (reading resets)). */
int lk_debug_read(lk_handle h, int what, void* dst, size_t bytes);

/* ---- map ------------------------------------------------------------------------------- */

/* Reserve device capacity for the map (root voxels, octree nodes, retained points). Optional:
 * lk_map_upload / lk_map_build size the map themselves when this was not called. */
int lk_map_reserve(lk_handle h, uint64_t max_roots, uint64_t max_nodes, uint64_t max_points);
/* Replace the device map by a blob (fixtures, replicas on other GPUs, resume). When the new map's storage cannot be
 * allocated (LK_ERR_OUT_OF_MEMORY, or LK_ERR_CAPACITY for pools past their index range) the current map is dropped too:
 * the handle has no map (LK_ERR_NOT_READY) until the next successful upload or build. */
int lk_map_upload(lk_handle h, const void* blob, size_t bytes);
/* Dump the device map. Call with blob==NULL to query the size into *bytes_out. */
int lk_map_download(lk_handle h, void* blob, size_t capacity, size_t* bytes_out);
/* VoxelMapManager::BuildVoxelMap (voxel_map.cc:287-334): first-frame bulk build. As for lk_map_upload, a failed
 * allocation of the map's storage leaves the handle with no map.
 * xyz_world = feats_down_world_ (float xyz, n*3), xyz_body = feats_down_body_ (lidar frame). */
int lk_map_build(lk_handle h, const float* xyz_world, const float* xyz_body, size_t n,
                 const double rot[9], const double rot_cov[9], const double pos_cov[9]);
/* Step 4 of KILO::predictUpdatePoint (KILO.cc:216-231) without the filter: UpdateVoxelMap (voxel_map.cc:336-361) of
 * n_sets point sets, each placed at its own pose. Set s holds pts[set_offsets[s] .. set_offsets[s+1]) (float4, lidar frame,
 * the 4th component ignored) and is placed with rot[9s..] (row-major body->world), pos[3s..], rot_cov[9s..] and
 * pos_cov[9s..] (the theta and position blocks of P, row-major 3x3):
 *   p_i = R_ext p_b + t_ext, p_w = R p_i + p, var = (R R_ext) Sigma_b (R R_ext)^T + (R [p_i]x) rot_cov (R [p_i]x)^T + pos_cov.
 * rot_cov / pos_cov enter through their symmetric parts 0.5 (a_ij + a_ji), as the filter's P blocks do in streaming: a set
 * given the state and P a streaming bucket ended with is placed bitwise as that bucket's insert placed it.
 * Points are inserted in set order, then in their order within the set, exactly as consecutive UpdateVoxelMap calls would.
 * A handle with no map starts from an empty one (as streaming from empty does). This is not lk_map_build: BuildVoxelMap
 * fits each root once after all points, and UpdateVoxelMap refits as points arrive.
 * LK_ERR_INVALID_ARG: a NULL argument with n_sets > 0, set_offsets not monotone, or a non-finite entry of rot, pos, rot_cov
 * or pos_cov. n_sets == 0 does nothing. LK_ERR_CAPACITY: the map pools ran out (the map then holds the points inserted up
 * to the window that overflowed, and some of that window's). A staged batch stays staged. */
int lk_map_insert(lk_handle h, uint32_t n_sets, const float* pts, const uint32_t* set_offsets, const double* rot,
                  const double* pos, const double* rot_cov, const double* pos_cov);
/* Map counters: out[0]=roots, out[1]=nodes, out[2]=retained points, out[3]=plane nodes. */
int lk_map_stats(lk_handle h, uint64_t out[4]);
/* VoxelMapManager::mapSliding + clearMemOutOfMap (voxel_map.cc:552-594; dead code in the reference, needed for unbounded
 * runs): when `position` is at least sliding_thresh away from the position of the last slide (initially the origin,
 * voxel_map.h:201), every root voxel whose key lies outside [k - half_map_size, k + half_map_size] on some axis,
 * k = floor(position / voxel_size) (eigen_types.hpp:89-95), is removed from the map. *slid = 1 when a slide happened,
 * *removed = root voxels dropped. The root table is rebuilt, and the dropped octrees' nodes and standard point tiles
 * go to the map's free lists, from which the next scan that updates the map allocates before it grows the pools. */
int lk_map_slide(lk_handle h, const double position[3], int32_t* slid, uint64_t* removed);
/* Device memory of the map, for long runs that must check it has stopped growing:
 * out[0] = node slots handed out by the bump allocator, out[1] = nodes on the free lists,
 * out[2] = point slots handed out by the bump allocator, out[3] = point slots on the free lists,
 * out[4] = device bytes of the map pools as allocated, out[5] = pool reallocations since the map was created.
 * Storage is recycled where the map stops using it: the point tile of a leaf that freezes at max_points_num, the tile
 * of a node whose points were cut into octants, and whole octrees dropped by lk_map_slide. An entry freed by one
 * launch is reused from the next launch that updates the map on. out[0] - out[1] nodes and out[2] - out[3] slots are
 * held; only tiles of the standard max_points_num + 2 (even) slots are recycled. */
int lk_map_memory(lk_handle h, uint64_t out[6]);

/* ---- the hot path ---------------------------------------------------------------------- */

/* Batched replacement of the bucket loop of KILO::process (KILO.cc:367-396) calling
 * KILO::predictUpdatePoint (KILO.cc:108-233) per bucket, for `batch` independent scans
 * (each with its own state / covariance / clock; all against this handle's map).
 *
 *  x_inout[batch], P_inout[batch*900], clk_inout[batch] : per-scan filter (in/out)
 *  Q[900]                : process covariance shared by the batch (ESKF::Q_)
 *  pts                   : float4 per point (x, y, z, curvature = time offset [s]); points of a
 *                          scan contiguous and already ordered by curvature (stable)
 *  scan_offsets[batch+1] : point range of every scan
 *  scan_bucket_ptr[batch+1], bucket_offsets[nb+1], bucket_times[nb] :
 *                          scan s owns buckets [scan_bucket_ptr[s], scan_bucket_ptr[s+1]);
 *                          bucket b holds points [bucket_offsets[b], bucket_offsets[b+1]) and is
 *                          stamped bucket_times[b] (= begin_time + curvature, KILO.cc:376)
 *  iters                 : residual/solve iterations per bucket (1 = the reference; SURVEY §8d)
 *  update_map            : 1 = insert every bucket into the map after its update
 *                          (UpdateVoxelMap, KILO.cc:231); requires batch == 1 per handle map
 *  pts_world_out         : float4 per point (x, y, z world, intensity 0|255) = cloud_down_world
 *  n_effective_out[batch]: success_pts_size_out (KILO.cc:180) per scan
 */
int lk_scan_update(lk_handle h, int batch, lk_state* x_inout, double* P_inout, const double* Q,
                   lk_stream_clock* clk_inout, const float* pts, const uint32_t* scan_offsets,
                   const uint32_t* scan_bucket_ptr, const uint32_t* bucket_offsets,
                   const double* bucket_times, int iters, int update_map, float* pts_world_out,
                   uint32_t* n_effective_out);

/* The same work split for resident-data measurement: stage copies every input to HBM once,
 * run executes the whole batch from the staged inputs (idempotent: reads staged x/P, writes
 * separate outputs), fetch copies results back. lk_scan_update == stage + run + fetch. */
int lk_batch_stage(lk_handle h, int batch, const lk_state* x, const double* P, const double* Q,
                   const lk_stream_clock* clk, const float* pts, const uint32_t* scan_offsets,
                   const uint32_t* scan_bucket_ptr, const uint32_t* bucket_offsets,
                   const double* bucket_times);
int lk_batch_run(lk_handle h, int iters, int update_map);
int lk_batch_fetch(lk_handle h, lk_state* x_out, double* P_out, lk_stream_clock* clk_out,
                   float* pts_world_out, uint32_t* n_effective_out);
/* Asynchronous form: enqueue the hot path for scans [first, first+count) of the staged batch on
 * the library's stream and return without synchronising (pipelined steps). */
int lk_batch_run_range(lk_handle h, uint32_t first, uint32_t count, int iters, int update_map);
/* CUDA-event timer on the library's stream: start records an event, stop records another,
 * synchronises and reports the elapsed device time, the time inside the residual kernel (when
 * "kernel_timing" is on), and the number of kernels launched in between. */
int lk_timer_start(lk_handle h);
int lk_timer_stop(lk_handle h, float* total_ms, float* residual_kernel_ms, uint32_t* n_kernel_launches,
                  uint32_t* n_residual_launches);
/* Device time of the most recent lk_batch_run (CUDA events on the library's stream), and the
 * number of kernels it launched / time spent in the residual kernel alone. */
int lk_batch_last_timing(lk_handle h, float* total_ms, float* residual_kernel_ms,
                         uint32_t* n_kernel_launches, uint32_t* n_residual_launches);
/* Block until all work queued on the library's stream is done. */
int lk_sync(lk_handle h);

/* Per-point residual rows of ONE bucket at the given state (no update applied): the output of
 * the loop KILO.cc:122-210 — ok flag, h (6), z, R per point. For parity tests of rows a3-a7. */
int lk_debug_residuals(lk_handle h, const lk_state* x, const double* P, const float* pts,
                       uint32_t n, uint8_t* ok_out, double* h_out /*n*6*/, double* z_out,
                       double* R_out, int32_t* key_out /*n*3*/);

/* ---- filter steps outside the point loop (SURVEY §8f rank 1) ---------------------------- */

/* ESKF::predict (eskf.cc:83-89) on `batch` host-resident filters. */
int lk_predict(lk_handle h, int batch, lk_state* x_inout, double* P_inout, const double* Q,
               const double* dt, int prop_state, int prop_cov);
/* ESKF::updateByPoints (eskf.cc:91-113) from explicit rows (n x 6 h, n z, n R). */
int lk_update_by_points(lk_handle h, lk_state* x_inout, double* P_inout, uint32_t n,
                        const double* pt_h, const double* pt_z, const double* pt_R);
/* KILO::predictUpdateImu (KILO.cc:235-258) -> ESKF::updateByImu (eskf.cc:125-135). */
int lk_obs_imu(lk_handle h, lk_state* x_inout, double* P_inout, const double* Q,
               lk_stream_clock* clk_inout, const lk_imu_meas* imu, uint32_t n, double gravity,
               double acc_norm);
/* KILO::predictUpdateKinImu (KILO.cc:260-314) -> ESKF::updateByKinImu (eskf.cc:137-145). */
int lk_obs_kinimu(lk_handle h, lk_state* x_inout, double* P_inout, const double* Q,
                  lk_stream_clock* clk_inout, const lk_kinimu_meas* kin, uint32_t n, double gravity,
                  double acc_norm);

/* KILO::process second lambda (KILO.cc:367-396) for ONE streaming scan with its inertial /
 * kinematic queue interleaved on the device: every sample with stamp < bucket time is applied
 * before the bucket. Exactly one of imu / kin may be non-NULL (imu_mode_only_, KILO.cc:379-390).
 * Consumed sample count is returned in *n_consumed (the rest stays queued at the caller). */
int lk_process_scan(lk_handle h, lk_state* x_inout, double* P_inout, const double* Q,
                    lk_stream_clock* clk_inout, const float* pts, uint32_t n_pts,
                    const uint32_t* bucket_offsets, const double* bucket_times, uint32_t n_buckets,
                    const lk_imu_meas* imu, const lk_kinimu_meas* kin, uint32_t n_meas,
                    double gravity, double acc_norm, int iters, int update_map,
                    float* pts_world_out, uint32_t* n_effective_out, uint32_t* n_consumed);

/* TrajectorySaver::write (trajectory_saver.hpp:43-50): one TUM line "timestamp tx ty tz qx qy qz qw\n", fixed notation,
 * 9 decimals, the quaternion by Eigen's Quaterniond(Matrix3d) rule. rot = row-major body->world. Host-side helper;
 * returns the number of characters written (excluding the NUL) or LK_ERR_CAPACITY. */
int lk_tum_line(double timestamp, const double rot[9], const double pos[3], char* buf, size_t capacity);

/* ---- what feeds the path (SURVEY §8f ranks 2-3) ------------------------------------------- */

/* Field layout of a sensor_msgs/PointCloud2 as pcl::fromROSMsg resolves it by name for the three
 * driver formats of legkilo/src/preprocess/lidar_processing.h:10-72. */
typedef enum lk_lidar_type { LK_LIDAR_VELODYNE = 1, LK_LIDAR_OUSTER = 2, LK_LIDAR_HESAI = 3 } lk_lidar_type;
typedef struct lk_pc2_layout {
    uint32_t point_step;    /* bytes per point */
    uint32_t off_x, off_y, off_z, off_intensity; /* float32 fields */
    uint32_t off_time;      /* velodyne "time" float32 | ouster "t" uint32 | hesai "timestamp" float64 */
    int32_t lidar_type;     /* lk_lidar_type: selects the time field's type and arithmetic */
    int32_t reserved;
} lk_pc2_layout;

/* LidarProcessing::{velodyne,ouster,hesai}Handler (lidar_processing.cc:25-108): every filter_num-th
 * point outside the blind sphere, time offset from the first point rounded to 1/500 s into the
 * `curvature` slot. pts_out: float4 (x, y, z, curvature) x n_points capacity, intensity_out nullable.
 * first_time / last_time: time_scale x the first / last RAW point's time (the caller adds the header
 * stamp as lidar_processing.cc:33-34 does). */
int lk_decode_pointcloud2(lk_handle h, const uint8_t* data, uint32_t n_points, const lk_pc2_layout* layout,
                          float blind, int32_t filter_num, double time_scale, float* pts_out, float* intensity_out,
                          uint32_t* n_out, double* first_time, double* last_time);

/* The two steps between decode and the hot loop (KILO.cc:356-378): pcl::VoxelGrid centroid filter with
 * leaf_size on all axes (PCL 1.8 voxel_grid.hpp: leaf index = floor(p / leaf) - min index, centroid of
 * x, y, z AND curvature in float, leaves emitted in ascending index), then the sort by curvature
 * (stable here; std::sort in the reference) and the maximal equal-curvature runs.
 * Outputs (capacity n_in points / n_in + 1 offsets): pts_out float4, bucket_offsets, bucket_curvature
 * (add lidar_begin_time_ to get bucket times). */
int lk_preprocess_scan(lk_handle h, const float* pts_in, uint32_t n_in, float leaf_size, float* pts_out,
                       uint32_t* n_out, uint32_t* bucket_offsets, float* bucket_curvature, uint32_t* n_buckets);

/* ---- leg kinematics: what feeds lk_obs_kinimu / the kin queue of lk_process_scan ----------- */

/* = legkilo::Kinematics::Config (kinematics.h:27-35), same field order. */
typedef struct lk_leg_cfg {
    double leg_offset_x;
    double leg_offset_y;
    double leg_calf_length;
    double leg_thigh_length;
    double leg_thigh_offset;
    double contact_force_threshold_up;   /* ContactDetector T_on_ */
    double contact_force_threshold_down; /* ContactDetector T_off_ */
} lk_leg_cfg; /* 56 B */

/* The fields of one unitree_legged_msgs::HighState that Kinematics::processing and the redundancy check read, in the
 * MESSAGE's index order (legs FL FR RL RR, kinematics.cc:13-16) and the message's own types. */
typedef struct lk_leg_state {
    double stamp;           /* stamp.toSec() */
    float acc[3];           /* imu.accelerometer */
    float gyr[3];           /* imu.gyroscope */
    float q[12];            /* motorState[0..11].q: hip, thigh, calf of FL, FR, RL, RR */
    float dq[12];           /* motorState[0..11].dq */
    int16_t foot_force[4];  /* footForce (FL FR RL RR) */
} lk_leg_state; /* 136 B */

/* What a caller carries from one lk_leg_kinematics call to the next (like lk_stream_clock): the four
 * ContactDetector states (kinematics.h:10-23) in the project's leg order FR FL RR RL, and imu.accelerometer[2] /
 * imu.gyroscope[2] of the last RAW message, kept or dropped (ros_interface.cc:222, :228, :247). */
typedef struct lk_leg_track {
    int32_t in_contact[4];
    float last_acc_z;
    float last_gyr_z;
} lk_leg_track; /* 24 B */

/* The reference's initial state: every detector in contact (kinematics.h:12), the previous message zero-initialised
 * (the static HighState of ros_interface.cc:222). Host-side helper. */
int lk_leg_track_default(lk_leg_track* t);

/* RosInterface::kinematicImuCallBack (ros_interface.cc:221-248) without its ROS plumbing, over `n` consecutive
 * messages, then Kinematics::processing (kinematics.cc:5-90) on every message it keeps:
 *  - redundancy != 0 drops a message whose imu.accelerometer[2] AND imu.gyroscope[2] both equal (float ==) those of
 *    the previous raw message (ros_interface.cc:225-231); for in[0] that is track_inout's last_acc_z / last_gyr_z.
 *    A dropped message does not advance the contact detectors.
 *  - contact: the detector of leg FR / FL / RR / RL reads footForce[1] / [0] / [3] / [2] (kinematics.cc:17-20) and
 *    switches on when out of contact and force > threshold_up, off when in contact and force < threshold_down.
 *  - foot_pos / foot_vel: forward kinematics and Jacobian times joint rates in fp64 (caculateFootPosVel,
 *    kinematics.cc:54-90), joints of FR / FL / RR / RL from motorState[3..5] / [0..2] / [9..11] / [6..8].
 * The kept samples are written in order to out[0 .. *n_out) (capacity n) and the updated track is written back.
 * n == 0 returns LK_OK with *n_out = 0 and the track unchanged. A NULL h, cfg, track_inout or n_out, a NULL in / out
 * with n > 0, or a non-finite cfg field is LK_ERR_INVALID_ARG.
 * Runs on the device for any n: one thread per message, two device-wide scans (output positions; the contact
 * detectors as a composition of per-message transfer functions), one thread per kept message. n_out, stamps,
 * contacts, acc, gyr and the track are bitwise what the reference computes; foot_pos / foot_vel can differ from a CPU
 * build by a few ulp (device sin / cos against the host libm, and FMA contraction by nvcc). */
int lk_leg_kinematics(lk_handle h, const lk_leg_cfg* cfg, const lk_leg_state* in, uint32_t n, int32_t redundancy,
                      lk_leg_track* track_inout, lk_kinimu_meas* out, uint32_t* n_out);

#ifdef __cplusplus
}
#endif
#endif /* LEGKILO_B200_H_ */
