// lk_mapbuild.cu — device-side VoxelMapManager::BuildVoxelMap (voxel_map.cc:287-334): per-point
// covariance, voxel keys, stable grouping by root voxel (radix sort on the packed key, original
// index as tie-break = the reference's insertion order), then one warp per root voxel runs
// init_octo_tree / cut_octo_tree (voxel_map.cc:119-183) with the warp-cooperative plane fit.
#include <cub/cub.cuh>

#include "lk_kernels.h"
#include "lk_plane.cuh"
#include "lk_mapdev.h"

namespace lk {

namespace {

constexpr int KEY_BIAS = 1 << 20;  // keys in [-2^20, 2^20) per axis -> 21 bits each

__host__ __device__ __forceinline__ unsigned long long pack_key(int kx, int ky, int kz) {
    return ((unsigned long long)(uint32_t)(kx + KEY_BIAS) << 42) | ((unsigned long long)(uint32_t)(ky + KEY_BIAS) << 21) |
           (unsigned long long)(uint32_t)(kz + KEY_BIAS);
}
__host__ __device__ __forceinline__ void unpack_key(unsigned long long k, int& kx, int& ky, int& kz) {
    kx = (int)((k >> 42) & 0x1fffffu) - KEY_BIAS;
    ky = (int)((k >> 21) & 0x1fffffu) - KEY_BIAS;
    kz = (int)(k & 0x1fffffu) - KEY_BIAS;
}

struct BuildConst {
    double M[9];     // rot * extR
    double MMt[9];   // M M^T
    double Crot[9];  // rot_cov
    double Cpos[9];  // pos_cov
};

// voxel_map.cc:296-311: pv.point_w from the float world cloud, var from the LIDAR-frame point
// (cross-matrix of the lidar point, no rotation on it — differs from KILO.cc:136-140 on purpose).
__global__ void k_build_points(const float* __restrict__ xyz_world, const float* __restrict__ xyz_body, uint32_t n,
                               BuildConst bc, Globals g, unsigned long long* keys, uint32_t* idx, DevPoint* recs,
                               uint32_t* bad) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    DevPoint p;
    p.pw[0] = (double)xyz_world[3 * i]; p.pw[1] = (double)xyz_world[3 * i + 1]; p.pw[2] = (double)xyz_world[3 * i + 2];
    double bx = (double)xyz_body[3 * i], by = (double)xyz_body[3 * i + 1], bz = (double)xyz_body[3 * i + 2];
    if (bz == 0.0) bz = 0.0001;  // calcBodyCov mutates its argument; the cross-matrix below sees it too (:302-304)
    double r2 = bx * bx + by * by + bz * bz;
    float range = (float)sqrt(r2);
    double range2 = (double)range * (double)range;
    // Sigma_b = rv u u^T + range^2 dv (I - u u^T);  M Sigma_b M^T = (rv - range^2 dv) (Mu)(Mu)^T + range^2 dv M M^T
    double inv = 1.0 / sqrt(r2);
    double ux = bx * inv, uy = by * inv, uz = bz * inv;
    double mu[3] = {bc.M[0] * ux + bc.M[1] * uy + bc.M[2] * uz, bc.M[3] * ux + bc.M[4] * uy + bc.M[5] * uz,
                    bc.M[6] * ux + bc.M[7] * uy + bc.M[8] * uz};
    double a = (double)g.rv - range2 * g.dv, b = range2 * g.dv;
    // (-[pl]x) rot_cov (-[pl]x)^T = [pl]x rot_cov [pl]x^T
    double K[9] = {0, -bz, by, bz, 0, -bx, -by, bx, 0};
    double KC[9], KCKt[9];
    mat3_mul(K, bc.Crot, KC);
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) KCKt[r * 3 + c] = KC[r * 3] * K[c * 3] + KC[r * 3 + 1] * K[c * 3 + 1] + KC[r * 3 + 2] * K[c * 3 + 2];
    const int ut[6][2] = {{0, 0}, {0, 1}, {0, 2}, {1, 1}, {1, 2}, {2, 2}};
#pragma unroll
    for (int q = 0; q < 6; ++q) {
        int r = ut[q][0], c = ut[q][1];
        p.var[q] = a * mu[r] * mu[c] + b * bc.MMt[r * 3 + c] + KCKt[r * 3 + c] + bc.Cpos[r * 3 + c];
    }
    p.pad = 0.0;
    // voxelKeyFloor(point_w, (double)(float)voxel_size)   (eigen_types.hpp:89-95, voxel_map.cc:289)
    double vs = (double)g.voxel_f;
    int kx = (int)floor(p.pw[0] / vs), ky = (int)floor(p.pw[1] / vs), kz = (int)floor(p.pw[2] / vs);
    if (kx < -KEY_BIAS || kx >= KEY_BIAS || ky < -KEY_BIAS || ky >= KEY_BIAS || kz < -KEY_BIAS || kz >= KEY_BIAS) {
        atomicExch(bad, 1u);
        kx = ky = kz = 0;
    }
    keys[i] = pack_key(kx, ky, kz);
    idx[i] = i;
    recs[i] = p;
}

// KILO::cloudLidarToWorld (KILO.cc:89-106) over a raw float4 cloud, one load per point: the body and world xyz that
// k_build_points reads, and the world float4 the node publishes (w copied as pointLidarToWorld copies the intensity).
// p_i = R_ext p + t_ext, p_w = R p_i + pos, each product the reference's s = 0; s += a_k b_k (so 0 + -0.0 = +0.0), no FMA.
__device__ __forceinline__ double row_dot(const double* r, double x, double y, double z) {
    double s = __dadd_rn(0.0, __dmul_rn(r[0], x));
    s = __dadd_rn(s, __dmul_rn(r[1], y));
    return __dadd_rn(s, __dmul_rn(r[2], z));
}

struct WorldPose {
    double Re[9], te[3];  // extrinsics
    double R[9], p[3];    // body -> world
};

__global__ void k_first_frame_points(const float4* __restrict__ pts, uint32_t n, WorldPose wp, float* __restrict__ xyz_body,
                                     float* __restrict__ xyz_world, float4* __restrict__ world4) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 q = pts[i];
    const double x = q.x, y = q.y, z = q.z;
    double pi[3], pw[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) pi[k] = __dadd_rn(row_dot(wp.Re + 3 * k, x, y, z), wp.te[k]);
#pragma unroll
    for (int k = 0; k < 3; ++k) pw[k] = __dadd_rn(row_dot(wp.R + 3 * k, pi[0], pi[1], pi[2]), wp.p[k]);
    const float wx = __double2float_rn(pw[0]), wy = __double2float_rn(pw[1]), wz = __double2float_rn(pw[2]);
    xyz_body[3 * i] = q.x; xyz_body[3 * i + 1] = q.y; xyz_body[3 * i + 2] = q.z;
    xyz_world[3 * i] = wx; xyz_world[3 * i + 1] = wy; xyz_world[3 * i + 2] = wz;
    if (world4) world4[i] = make_float4(wx, wy, wz, q.w);
}

__global__ void k_gather_points(const DevPoint* __restrict__ recs, const uint32_t* __restrict__ idx, uint32_t n,
                                DevPoint* out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = recs[idx[i]];
}

}  // namespace

// ---- octree state machine (shared with the insert kernel through lk_octree.cuh) --------------
}  // namespace lk

#include "lk_octree.cuh"

namespace lk {
namespace {

// One warp per root voxel: create the root (voxel_map.cc:317-327) and run init_octo_tree.
__global__ void __launch_bounds__(128) k_build_roots(MapDev md, Globals g, const unsigned long long* __restrict__ ukeys,
                                                     const uint32_t* __restrict__ counts,
                                                     const uint32_t* __restrict__ starts, uint32_t n_roots,
                                                     const DevPoint* __restrict__ sorted, uint32_t node_first) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    WarpTile* tiles = reinterpret_cast<WarpTile*>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    WarpTile* wt = tiles + warp;
    if (lane == 0) {
        mbar_init(&wt->bar, 1);
        wt->phase = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        fence_proxy_async();
    }
    __syncwarp();
    uint32_t r = blockIdx.x * (blockDim.x >> 5) + warp;
    if (r >= n_roots) return;
    int kx, ky, kz;
    unpack_key(ukeys[r], kx, ky, kz);
    const uint32_t node = node_first + r;
    const int cnt = (int)counts[r];
    if (lane == 0) {
        init_root_node(md, g, node, kx, ky, kz);
        if (!hash_insert_dev(md.slots, md.hash_mask, kx, ky, kz, (int)node)) atomicOr(md.overflow, 4u);
    }
    __syncwarp();
    // BuildVoxelMap pushes every point first (new_points_ += count) and only then runs
    // init_octo_tree on every root (voxel_map.cc:333).
    warp_init_octo_tree(md, g, wt, node, sorted + starts[r], cnt, /*pts_in_pool=*/false, lane);
}

}  // namespace

int map_build_device(MapDevHost& mh, const Globals& g, const float* d_xyz_world, const float* d_xyz_body, uint32_t n,
                     const double* rot, const double* rot_cov, const double* pos_cov, cudaStream_t s,
                     std::string& err) {
    BuildConst bc;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            double m = 0;
            for (int k = 0; k < 3; ++k) m += rot[r * 3 + k] * g.Re[k * 3 + c];
            bc.M[r * 3 + c] = m;
        }
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            double m = 0;
            for (int k = 0; k < 3; ++k) m += bc.M[r * 3 + k] * bc.M[c * 3 + k];
            bc.MMt[r * 3 + c] = m;
        }
    for (int i = 0; i < 9; ++i) {
        bc.Crot[i] = rot_cov[i];
        bc.Cpos[i] = pos_cov[i];
    }
    const size_t nn = std::max<size_t>(n, 1);
    DevBuf b_keys, b_keys_sorted, b_ukeys, b_idx, b_idx_sorted, b_counts, b_starts, b_nruns, b_bad, b_recs, b_sorted, b_tmp;
    LK_CUDA(err, b_keys.alloc(nn * 8));
    LK_CUDA(err, b_keys_sorted.alloc(nn * 8));
    LK_CUDA(err, b_ukeys.alloc(nn * 8));
    LK_CUDA(err, b_idx.alloc(nn * 4));
    LK_CUDA(err, b_idx_sorted.alloc(nn * 4));
    LK_CUDA(err, b_counts.alloc(nn * 4));
    LK_CUDA(err, b_starts.alloc(nn * 4));
    LK_CUDA(err, b_nruns.alloc(16));
    LK_CUDA(err, b_bad.alloc(16));
    LK_CUDA(err, b_recs.alloc(nn * sizeof(DevPoint)));
    LK_CUDA(err, b_sorted.alloc(nn * sizeof(DevPoint)));
    auto* keys = b_keys.as<unsigned long long>();
    auto* keys_sorted = b_keys_sorted.as<unsigned long long>();
    auto* ukeys = b_ukeys.as<unsigned long long>();
    auto* idx = b_idx.as<uint32_t>();
    auto* idx_sorted = b_idx_sorted.as<uint32_t>();
    auto* counts = b_counts.as<uint32_t>();
    auto* starts = b_starts.as<uint32_t>();
    auto* nruns = b_nruns.as<uint32_t>();
    auto* bad = b_bad.as<uint32_t>();
    auto* recs = b_recs.as<DevPoint>();
    auto* sorted = b_sorted.as<DevPoint>();
    size_t tmp_bytes = 0;
    cudaError_t e;
    cudaMemsetAsync(bad, 0, 16, s);
    cudaMemsetAsync(nruns, 0, 16, s);
    uint32_t h_runs = 0;
    if (n) {
        k_build_points<<<(n + 255) / 256, 256, 0, s>>>(d_xyz_world, d_xyz_body, n, bc, g, keys, idx, recs, bad);
        size_t b1 = 0, b2 = 0, b3 = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, b1, keys, keys_sorted, idx, idx_sorted, (int)n, 0, 63, s);
        cub::DeviceRunLengthEncode::Encode(nullptr, b2, keys_sorted, ukeys, counts, nruns, (int)n, s);
        cub::DeviceScan::ExclusiveSum(nullptr, b3, counts, starts, (int)n, s);
        tmp_bytes = std::max(b1, std::max(b2, b3));
        LK_CUDA(err, b_tmp.alloc(std::max<size_t>(tmp_bytes, 16)));
        void* tmp = b_tmp.p;
        // LSD radix sort is stable: equal keys keep ascending original index = insertion order
        cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys, keys_sorted, idx, idx_sorted, (int)n, 0, 63, s);
        cub::DeviceRunLengthEncode::Encode(tmp, tmp_bytes, keys_sorted, ukeys, counts, nruns, (int)n, s);
        k_gather_points<<<(n + 255) / 256, 256, 0, s>>>(recs, idx_sorted, n, sorted);
        uint32_t h_bad = 0;
        cudaMemcpyAsync(&h_runs, nruns, 4, cudaMemcpyDeviceToHost, s);
        cudaMemcpyAsync(&h_bad, bad, 4, cudaMemcpyDeviceToHost, s);
        e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) { err = cudaGetErrorString(e); cudaGetLastError(); return LK_ERR_CUDA; }
        if (h_bad) { err = "point outside the addressable key range (|key| >= 2^20)"; return LK_ERR_INVALID_ARG; }
        cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, counts, starts, (int)h_runs, s);
    }
    // size the map for this build plus the caller's reserve, then run the per-root warps;
    // on pool overflow grow and retry (the bump allocators make a rebuild the simple, safe path)
    const int P2 = g.max_points_num + 2;
    unsigned long long want_points = (unsigned long long)h_runs * P2 + 2ull * n + 4096;
    uint32_t want_nodes = h_runs + h_runs / 4 + 4096;
    int rc = LK_OK;
    for (int attempt = 0; attempt < 6; ++attempt) {
        rc = mh.allocate(h_runs, want_nodes, want_points, s, err);
        if (rc) break;
        if (h_runs) {
            const int warps_per_block = 4;
            size_t smem = warps_per_block * sizeof(WarpTile);
            MapDev md = mh.dev();
            // roots occupy nodes [0, h_runs)
            cudaMemcpyAsync(md.n_nodes, &h_runs, 4, cudaMemcpyHostToDevice, s);
            cudaMemcpyAsync(md.n_roots, &h_runs, 4, cudaMemcpyHostToDevice, s);
            k_build_roots<<<(h_runs + warps_per_block - 1) / warps_per_block, warps_per_block * 32, smem, s>>>(
                md, g, ukeys, counts, starts, h_runs, sorted, 0);
        }
        uint32_t ovf = 0;
        cudaMemcpyAsync(&ovf, mh.dev().overflow, 4, cudaMemcpyDeviceToHost, s);
        e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) { rc = LK_ERR_CUDA; err = std::string("map build kernel: ") + cudaGetErrorString(e); cudaGetLastError(); break; }
        if (!ovf) { rc = mh.sync_counters(s, err); break; }
        if (ovf & 1u) want_nodes *= 2;
        if (ovf & 2u) want_points *= 2;
        if (ovf & 4u) { rc = LK_ERR_CAPACITY; err = "root table overflow during build"; break; }
        rc = LK_ERR_CAPACITY;
        err = "map pools overflowed repeatedly";
    }
    return rc;
}

void launch_first_frame_points(const Globals& g, const float4* d_pts, uint32_t n, const double* rot, const double* pos,
                               float* d_xyz_body, float* d_xyz_world, float4* d_world4, cudaStream_t s) {
    if (!n) return;
    WorldPose wp;
    for (int i = 0; i < 9; ++i) {
        wp.Re[i] = g.Re[i];
        wp.R[i] = rot[i];
    }
    for (int i = 0; i < 3; ++i) {
        wp.te[i] = g.te[i];
        wp.p[i] = pos[i];
    }
    k_first_frame_points<<<(n + 255) / 256, 256, 0, s>>>(d_pts, n, wp, d_xyz_body, d_xyz_world, d_world4);
}

}  // namespace lk
