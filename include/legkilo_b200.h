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
 * 3 = host-side phase times of lk_scan_update [stage, enqueue, wait+fetch, calls] in ns (reading resets),
 * 4 = the scratch the pose scorer holds (lk_score_poses, lk_refine_poses, lk_search_poses): two uint64, device bytes and
 * page-locked bytes). */
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
/* KILO::process's first frame (KILO.cc:331-353): StateInitialByImu / ByKinImu::processing (state_initial.hpp:34-117),
 * cloudLidarToWorld (KILO.cc:89-106) and VoxelMapManager::BuildVoxelMap (voxel_map.cc:287-334) in one call.
 *  pts            : n_pts float4 (x, y, z, w) in the lidar frame, the raw (not down-sampled) cloud as lk_decode_pointcloud2
 *                   writes it; only x, y, z go into the map
 *  imu / kin      : the frame's inertial queue, exactly one non-NULL (imu_mode_only_), n_meas samples
 *  x_inout        : grav = -mean_acc / |mean_acc| * gravity, bw = mean_gyr, rot = I; every other field is left as passed
 *                   (lk_state_default for a fresh stream). The means follow the reference's recurrence: seeded with
 *                   sample 0, then mean += (s - mean) / N over every sample, sample 0 included.
 *  P_out[900]     : 1e-6 I;  clk_out: both times = end_time;  acc_norm_out: |mean_acc| (the acc_norm of later calls)
 *  pts_world_out  : nullable, n_pts float4 (x_w, y_w, z_w, w): p_w = R (R_ext p + t_ext) + pos with R = I and the caller's
 *                   pos, fp64 in the reference's summation order without FMA, rounded to float (bitwise the reference's)
 * The map is built from those world points and the lidar points with rot = I, rot_cov = P[0:3,0:3], pos_cov = P[3:6,3:6],
 * and replaces the handle's map as lk_map_build does (a failed pool allocation leaves the handle with no map).
 * LK_ERR_NOT_READY (nothing written, the map untouched): n_pts == 0 or n_meas == 0 ("Data packet is not ready",
 * KILO.cc:326-329). LK_ERR_INVALID_ARG: a NULL required argument, both imu and kin, or n_pts >= 2^31.
 * LK_ERR_CAPACITY / LK_ERR_OUT_OF_MEMORY as lk_map_build. Outputs are written only on success. */
int lk_first_frame(lk_handle h, lk_state* x_inout, double* P_out, lk_stream_clock* clk_out, double* acc_norm_out,
                   const float* pts, uint32_t n_pts, double end_time,
                   const lk_imu_meas* imu, const lk_kinimu_meas* kin, uint32_t n_meas, double gravity,
                   float* pts_world_out);
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
/* Record of one pose in lk_score_poses (LK_SCORE_STRIDE doubles): the sums the LiDAR update (KILO.cc:187-210) would form.
 *   [LK_SCORE_A, +21)        upper triangle, row-major, of sum h^T h / R over the residual rows (h = [p_i x R^T n, n])
 *   [LK_SCORE_B, +6)         sum h^T z / R
 *   [LK_SCORE_SUM_R]         sum R
 *   [LK_SCORE_COUNT]         number of residual rows (success_pts_size_out, KILO.cc:180)
 *   [LK_SCORE_SUM_Z2R]       sum z^2 / R
 *   the rest of the stride is 0. */
#define LK_SCORE_A 0
#define LK_SCORE_B 21
#define LK_SCORE_SUM_R 27
#define LK_SCORE_COUNT 28
#define LK_SCORE_SUM_Z2R 29
#define LK_SCORE_STRIDE 32
/* n_poses candidate poses of n_sets point sets, scored against the handle's map. No filter, map or staged batch is touched.
 * Set s = pts[set_offsets[s] .. set_offsets[s+1]) (float4, lidar frame, 4th component ignored). Pose m places set
 * pose_set[m] with rot[9m..] (row-major body->world) and pos[3m..]. rot_cov / pos_cov (9 each, shared by every pose) are the
 * theta / position blocks of P that enter the point variance and the gate, through their symmetric parts, as in
 * lk_map_insert. sums_out[LK_SCORE_STRIDE m ..] receives pose m's record (LK_SCORE_*).
 * Every point goes through the rows of KILO::predictUpdatePoint (KILO.cc:122-210) at that pose: transform, body
 * covariance, voxel key, home voxel, then the one neighbour voxel, on the hot plane images (the form lk_debug_residuals
 * evaluates with "debug_records" 0). A pose's record depends only on that pose and its set, not on the other poses of the
 * call, their order or their number.
 * LK_ERR_NOT_READY: the handle has no map. LK_ERR_INVALID_ARG: a NULL argument with n_poses > 0, set_offsets not monotone,
 * pose_set[m] >= n_sets, or a non-finite entry of rot, pos, rot_cov or pos_cov. On any error nothing is written.
 * n_poses == 0 does nothing.
 * Runs on the device with one host synchronisation. Device memory, kept by the handle and grown to the largest call:
 * 16 bytes per point, 488 bytes per pose, 32 bytes per (256-point chunk, tile of up to 16 poses of its set), and at most
 * 64 MB of partial rows (256 bytes per pose and chunk of its set: the poses run in consecutive windows of at most that; a
 * pose whose set alone has more than 262 144 chunks takes a window of its own). Page-locked staging: the larger of the
 * per-pose / per-tile inputs and the records. */
int lk_score_poses(lk_handle h, uint32_t n_sets, const float* pts, const uint32_t* set_offsets, uint32_t n_poses,
                   const uint32_t* pose_set, const double* rot, const double* pos, const double* rot_cov,
                   const double* pos_cov, double* sums_out);
/* n_poses candidate poses of n_sets point sets, each refined against the handle's map by iters steps of the LiDAR update
 * with the pose's covariance held. No filter, map or staged batch is touched. The inputs are those of lk_score_poses, with
 * the same meaning. One step of pose m:
 *   1. its record (LK_SCORE_*) at the current pose, exactly as lk_score_poses forms it;
 *   2. with P66 = blockdiag(sym(rot_cov), sym(pos_cov)): y = (I + A P66)^-1 b, delta = P66 y, i.e. K z of
 *      ESKF::updateByPoints (eskf.cc:91-113) restricted to the pose, in information form, with the reference's N == 1 rule
 *      (A and b scaled by sum R / (sum R + 1e-4) when the count is 1);
 *   3. State::operator+= (eskf.cc:18-29): R <- R Exp(delta_theta), p <- p + delta_p. A count of 0, or a singular
 *      I + A P66, gives a zero step.
 * lk_batch_run(iters) re-applies the gain at every iterate with P held and updates P once, at the end. So the refined pose
 * is the pose lk_batch_run(iters) gives for the one-bucket scan of the pose's set staged at that pose, when P's theta /
 * position blocks are sym(rot_cov) / sym(pos_cov) with a zero cross block between them (no other entry of P reaches the
 * pose) and the bucket time equals the clock (the predict is then the identity); the two differ only in the order in which
 * the record's sums are added.
 * rot_out[9m..] (row-major) / pos_out[3m..] receive pose m's refined pose; they may alias rot / pos. sums_out may be NULL;
 * otherwise sums_out[LK_SCORE_STRIDE m ..] receives the record at the refined pose (one more scoring pass), bitwise what
 * lk_score_poses returns for the refined poses with the same rot_cov / pos_cov.
 * A pose's outputs depend only on that pose, its set, rot_cov, pos_cov and iters, not on the other poses of the call, their
 * order or their number. No convergence test: every pose takes iters steps.
 * LK_ERR_INVALID_ARG: iters < 1, NULL rot_out or pos_out with n_poses > 0, or an input lk_score_poses refuses;
 * LK_ERR_NOT_READY: the handle has no map. On any error nothing is written. n_poses == 0 does nothing.
 * Runs on the device with one host synchronisation, whatever iters. Device memory: the scratch of lk_score_poses, shared
 * with it. Page-locked staging: the larger of the per-pose / per-tile inputs and the refined poses plus the records. */
int lk_refine_poses(lk_handle h, uint32_t n_sets, const float* pts, const uint32_t* set_offsets, uint32_t n_poses,
                    const uint32_t* pose_set, const double* rot, const double* pos, const double* rot_cov,
                    const double* pos_cov, int iters, double* rot_out, double* pos_out, double* sums_out);
/* The search of INTEGRATION.md §5 in one call: a lattice of candidate poses per point set, scored, the best k kept, refined
 * and re-scored, with nothing per candidate leaving the device. No filter, map or staged batch is touched.
 * Set s = pts[set_offsets[s] .. set_offsets[s+1]), as in lk_score_poses. Its candidates are its attitudes
 * att_offsets[s] .. att_offsets[s+1] (row-major 3x3 each in att_rot, body->world) times one position lattice of
 * counts = (nx, ny, nz) points spaced step, anchored at origin[3s..]. With L = nx ny nz, candidate c of set s is
 *   a = c / L, r = c % L, ix = r % nx, iy = (r / nx) % ny, iz = r / (nx ny),
 *   rot = att_rot[9 (att_offsets[s] + a) ..],  pos[j] = origin[3s + j] + (double)i_j * step[j]
 * (the product rounded to double, then the sum: no fused multiply-add).
 * The result is, bitwise, this composition of the other calls, per set s:
 *   1. every candidate of s scored as lk_score_poses scores it, with rot_cov / pos_cov;
 *   2. the k best kept, ordered by (count descending, candidate index ascending), a total order;
 *   3. those refined as lk_refine_poses(iters) refines them, with rot_cov / pos_cov;
 *   4. the refined poses scored as lk_score_poses scores them, with rot_cov_tight / pos_cov_tight;
 *   5. ordered by (tight count descending, rank in step 2 ascending).
 * Entry s k + j of each output is the j-th of step 5: rot_out 9 doubles, pos_out 3, sums_out LK_SCORE_STRIDE (the tight
 * record, LK_SCORE_*), cand_out 1 (its candidate index c). A set's outputs depend only on that set, its candidates, the
 * four blocks, iters and k: not on the other sets, their order or how the call is cut into windows.
 * LK_ERR_NOT_READY: the handle has no map. LK_ERR_INVALID_ARG: a NULL argument with n_sets > 0, set_offsets or att_offsets
 * not monotone, a zero entry of counts, k of 0 or above LK_SEARCH_MAX_K, iters < 1, a non-finite entry of the attitudes,
 * origin, step or any block, or a set with fewer than k candidates or with 2^32 or more. On any error nothing is written.
 * n_sets == 0 does nothing.
 * Runs on the device with one host synchronisation, whatever the number of candidates: they are generated, scored and
 * kept window by window on the device (windows of at most 262 144 candidates and 262 144 partial rows). Device memory,
 * shared with lk_score_poses and lk_refine_poses, kept by the handle and grown to the largest call, does not depend on the
 * number of candidates: at most 16 bytes per point, 72 bytes per set and per attitude, 1 024 bytes per kept pose
 * (n_sets k) plus 32 bytes per (256-point chunk of a set, tile of up to 16 of its kept poses), and 192 MiB for one window
 * (64 MiB of partial rows, 64 MiB of records, 64 MiB for the window's 192-byte pose constants, sums and items), each buffer
 * with up to 1/8 growth slack. Page-locked staging: the larger of (72 bytes per set and per attitude, 16 bytes per kept
 * pose and 32 per (chunk, tile) of them) and 356 bytes per kept pose, plus alignment and 1/4 growth slack.
 * lk_debug_read(h, 4, ...) reads back what is held. */
#define LK_SEARCH_MAX_K 256
int lk_search_poses(lk_handle h, uint32_t n_sets, const float* pts, const uint32_t* set_offsets,
                    const uint32_t* att_offsets, const double* att_rot, const double* origin,
                    const double step[3], const uint32_t counts[3],
                    const double* rot_cov, const double* pos_cov, int iters,
                    const double* rot_cov_tight, const double* pos_cov_tight, uint32_t k,
                    double* rot_out, double* pos_out, double* sums_out, uint32_t* cand_out);
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
 * stamp as lidar_processing.cc:33-34 does). n_points == 0 returns at once with the times untouched.
 * The batch of one of lk_decode_pointcloud2s at stamp 0: no device allocation once the handle's scratch fits. */
int lk_decode_pointcloud2(lk_handle h, const uint8_t* data, uint32_t n_points, const lk_pc2_layout* layout,
                          float blind, int32_t filter_num, double time_scale, float* pts_out, float* intensity_out,
                          uint32_t* n_out, double* first_time, double* last_time);

/* lk_decode_pointcloud2 for n_msgs messages in one call, output in the layout lk_preprocess_scans takes
 * (LidarProcessing::processing, lidar_processing.cc:25-108, per message).
 * In: message m is n_points[m] points of layout->point_step bytes at data[m] (the message's own buffer; nothing needs to
 * be concatenated); stamps[m] = header.stamp.toSec(), stamps NULL = 0 for every message. One layout, blind, filter_num
 * and time_scale for the whole call (a fleet with several drivers makes one call per driver).
 * Each message is decoded exactly as lk_decode_pointcloud2 decodes it alone: i % filter_num counts from the message's own
 * first point, and the time offset is taken from the message's own first raw point.
 * Out (capacities from N = sum of n_points): message m's kept points are pts_out[out_offsets[m] .. out_offsets[m+1]) as
 * float4 (x, y, z, curvature); intensity_out (N, nullable) alongside; out_offsets n_msgs + 1. begin_times / end_times
 * (n_msgs each, nullable) equal lidar_begin_time_ / lidar_end_time_ bitwise:
 *   Velodyne / Ouster: stamps[m] + (double)(float)(time_scale * t_first), and the same with t_last (:31-35, :59-63);
 *   Hesai: time_scale * t_first and time_scale * t_last, no stamp (:87-91).
 * A message with no points yields zero points and NaN times (the reference reads front() of an empty cloud).
 * out_offsets and begin_times are the in_offsets and begin_times of lk_preprocess_scans: the two calls chain with no host
 * work in between.
 * LK_ERR_INVALID_ARG (nothing written, the handle stays usable): a NULL required argument or a NULL data[m] with
 * n_points[m] > 0, filter_num < 1, a layout whose fields do not fit point_step, or a sum of n_points above INT_MAX.
 * n_msgs == 0 writes out_offsets[0] = 0. Runs on the device with two host synchronisations whatever n_msgs is; its
 * device memory is kept by the handle and grown to the largest call. */
int lk_decode_pointcloud2s(lk_handle h, uint32_t n_msgs, const uint8_t* const* data, const uint32_t* n_points,
                           const double* stamps, const lk_pc2_layout* layout, float blind, int32_t filter_num,
                           double time_scale, float* pts_out, float* intensity_out, uint32_t* out_offsets,
                           double* begin_times, double* end_times);

/* The two steps between decode and the hot loop (KILO.cc:356-378): pcl::VoxelGrid centroid filter with
 * leaf_size on all axes (PCL 1.8 voxel_grid.hpp: leaf index = floor(p / leaf) - min index, centroid of
 * x, y, z AND curvature in float, leaves emitted in ascending index), then the sort by curvature
 * (stable here; std::sort in the reference) and the maximal equal-curvature runs.
 * Outputs (capacity n_in points / n_in + 1 offsets): pts_out float4, bucket_offsets, bucket_curvature
 * (add lidar_begin_time_ to get bucket times). */
int lk_preprocess_scan(lk_handle h, const float* pts_in, uint32_t n_in, float leaf_size, float* pts_out,
                       uint32_t* n_out, uint32_t* bucket_offsets, float* bucket_curvature, uint32_t* n_buckets);

/* lk_preprocess_scan for n_scans scans in one call, output in the layout lk_batch_stage / lk_scan_update take.
 * Scan s is pts_in[in_offsets[s] .. in_offsets[s+1]) (float4 x, y, z, curvature). Every scan is filtered with leaf_size
 * on its OWN bounding box (PCL 1.8 semantics, as lk_preprocess_scan), then stable-sorted by curvature and cut into maximal
 * equal-curvature runs; each scan's output is bitwise what lk_preprocess_scan gives for it alone.
 * Out (capacities from N = in_offsets[n_scans]): pts_out N float4; scan_offsets / scan_bucket_ptr n_scans + 1;
 * bucket_offsets N + 1 (global point indices); bucket_curvature N; bucket_times N, written iff begin_times != NULL:
 * bucket_times[b] = begin_times[s] + (double)bucket_curvature[b] (KILO.cc:376). Totals are scan_offsets[n_scans] and
 * scan_bucket_ptr[n_scans]. A scan with no finite point yields zero points and zero buckets.
 * LK_ERR_INVALID_ARG: a NULL argument, in_offsets not monotone, leaf_size not positive and finite, begin_times given
 * without bucket_times or the reverse, or a scan whose leaf index would overflow int32 (lk_last_error names the scan;
 * nothing is written). n_scans == 0 writes scan_offsets[0] = scan_bucket_ptr[0] = bucket_offsets[0] = 0.
 * Runs on the device with a fixed number of host synchronisations (four) whatever n_scans is; its device memory is kept
 * by the handle and grown to the largest call. */
int lk_preprocess_scans(lk_handle h, uint32_t n_scans, const float* pts_in, const uint32_t* in_offsets, float leaf_size,
                        const double* begin_times, float* pts_out, uint32_t* scan_offsets, uint32_t* scan_bucket_ptr,
                        uint32_t* bucket_offsets, float* bucket_curvature, double* bucket_times);

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
