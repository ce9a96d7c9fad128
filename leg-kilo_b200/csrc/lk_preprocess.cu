// lk_preprocess.cu — what feeds the hot path (SURVEY §8f ranks 2-3), on the device:
//   * wire decode of sensor_msgs/PointCloud2 for the three driver layouts
//     (legkilo/src/preprocess/lidar_processing.cc:25-108): every filter_num-th point, blind-sphere test,
//     time offset rounded to 1/500 s, stable compaction;
//   * pcl::VoxelGrid centroid down-sampling as KILO::process uses it (KILO.cc:82-83, :356-360; PCL 1.8
//     voxel_grid.hpp — the library is absent from /root/reference, its published algorithm is restated),
//     then the sort by curvature and the equal-curvature bucket boundaries (KILO.cc:370-378).
// Sorting / scanning / run-length encoding use CUB (library code, like cuBLAS for a plain GEMM); the
// per-point and per-leaf arithmetic is hand-written and bit-identical to the CPU restatement.
#include <cub/cub.cuh>

#include <climits>
#include <string>

#include "lk_device.cuh"
#include "lk_host.h"

namespace lk {

namespace {

// ---- decode ---------------------------------------------------------------------------------------
__global__ void k_decode_flags(const uint8_t* __restrict__ data, uint32_t n, lk_pc2_layout L, float blind,
                               int filter_num, uint32_t* flags) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t* p = data + (size_t)i * L.point_step;
    float x, y, z;
    memcpy(&x, p + L.off_x, 4); memcpy(&y, p + L.off_y, 4); memcpy(&z, p + L.off_z, 4);
    // blindCheck (lidar_processing.h:94-97): blind*blind > x*x + y*y + z*z, float, no contraction
    const float r2 = __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
    const bool drop = (i % (uint32_t)filter_num) != 0 || (__fmul_rn(blind, blind) > r2);
    flags[i] = drop ? 0u : 1u;
}

__device__ __forceinline__ double raw_time(const uint8_t* p, const lk_pc2_layout& L) {
    if (L.lidar_type == LK_LIDAR_VELODYNE) { float t; memcpy(&t, p + L.off_time, 4); return (double)t; }
    if (L.lidar_type == LK_LIDAR_OUSTER) { uint32_t t; memcpy(&t, p + L.off_time, 4); return (double)t; }
    double t; memcpy(&t, p + L.off_time, 8); return t;
}

__global__ void k_decode_scatter(const uint8_t* __restrict__ data, uint32_t n, lk_pc2_layout L, double time_scale,
                                 const uint32_t* __restrict__ flags, const uint32_t* __restrict__ pos, float4* out,
                                 float* intensity) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !flags[i]) return;
    const uint8_t* p = data + (size_t)i * L.point_step;
    float4 o;
    memcpy(&o.x, p + L.off_x, 4); memcpy(&o.y, p + L.off_y, 4); memcpy(&o.z, p + L.off_z, 4);
    const double t0 = raw_time(data, L), ti = raw_time(p, L);
    if (L.lidar_type == LK_LIDAR_HESAI) {
        // double first / cur; std::round((cur - first) * 500.0f) / 500.0f in double, narrowed on store (:101-104)
        const double first = time_scale * t0, cur = time_scale * ti;
        o.w = (float)(round((cur - first) * (double)500.0f) / (double)500.0f);
    } else {
        // float first / cur (:30, :47-48 / :59, :75-76)
        const float first = (float)(time_scale * t0), cur = (float)(time_scale * ti);
        o.w = __fdiv_rn(roundf(__fmul_rn(__fsub_rn(cur, first), 500.0f)), 500.0f);
    }
    out[pos[i]] = o;
    if (intensity) {
        float v; memcpy(&v, p + L.off_intensity, 4);
        intensity[pos[i]] = v;
    }
}

// ---- voxel grid ---------------------------------------------------------------------------------------
__device__ __forceinline__ int f2ord(float f) { int i = __float_as_int(f); return i >= 0 ? i : i ^ 0x7fffffff; }
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

__global__ void k_minmax(const float4* __restrict__ pts, uint32_t n, int* mm /* [6]: min xyz, max xyz (ordered ints) */) {
    __shared__ int s[6][256];
    int mn[3] = {INT_MAX, INT_MAX, INT_MAX}, mx[3] = {INT_MIN, INT_MIN, INT_MIN};
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float4 p = pts[i];
        if (!isfinite(p.x) || !isfinite(p.y) || !isfinite(p.z)) continue;  // getMinMax3D skips non-finite points
        const int a[3] = {f2ord(p.x), f2ord(p.y), f2ord(p.z)};
        for (int k = 0; k < 3; ++k) { mn[k] = min(mn[k], a[k]); mx[k] = max(mx[k], a[k]); }
    }
    for (int k = 0; k < 3; ++k) { s[k][threadIdx.x] = mn[k]; s[3 + k][threadIdx.x] = mx[k]; }
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o)
            for (int k = 0; k < 3; ++k) {
                s[k][threadIdx.x] = min(s[k][threadIdx.x], s[k][threadIdx.x + o]);
                s[3 + k][threadIdx.x] = max(s[3 + k][threadIdx.x], s[3 + k][threadIdx.x + o]);
            }
        __syncthreads();
    }
    if (threadIdx.x < 3) atomicMin(&mm[threadIdx.x], s[threadIdx.x][0]);
    else if (threadIdx.x < 6) atomicMax(&mm[threadIdx.x], s[threadIdx.x][0]);
}

struct GridParams {
    float inv_leaf;
    int min_b[3];
    int mul[3];
};

__global__ void k_leaf_index(const float4* __restrict__ pts, uint32_t n, GridParams gp, uint32_t* idx, uint32_t* order) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = pts[i];
    // voxel_grid.hpp: ijk = floor(p * inverse_leaf_size) - min_b ; idx = ijk . divb_mul   (non-finite -> last)
    uint32_t v = 0xffffffffu;
    if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
        const int i0 = (int)floorf(__fmul_rn(p.x, gp.inv_leaf)) - gp.min_b[0];
        const int i1 = (int)floorf(__fmul_rn(p.y, gp.inv_leaf)) - gp.min_b[1];
        const int i2 = (int)floorf(__fmul_rn(p.z, gp.inv_leaf)) - gp.min_b[2];
        v = (uint32_t)(i0 * gp.mul[0] + i1 * gp.mul[1] + i2 * gp.mul[2]);
    }
    idx[i] = v;
    order[i] = i;
}

// One thread per leaf: float sums in original point order, divided by float(n) (CentroidPoint of PCL 1.8).
__global__ void k_centroids(const float4* __restrict__ pts, const uint32_t* __restrict__ order, const uint32_t* __restrict__ ukeys,
                            const uint32_t* __restrict__ counts, const uint32_t* __restrict__ starts, uint32_t n_leaves,
                            float4* out, uint32_t* curv_bits, uint32_t* leaf_ids, uint32_t* n_valid) {
    const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= n_leaves) return;
    if (ukeys[l] == 0xffffffffu) return;  // the run of non-finite points
    float sx = 0.f, sy = 0.f, sz = 0.f, sc = 0.f;
    const uint32_t s0 = starts[l], c = counts[l];
    for (uint32_t j = 0; j < c; ++j) {
        const float4 p = pts[order[s0 + j]];
        sx = __fadd_rn(sx, p.x); sy = __fadd_rn(sy, p.y); sz = __fadd_rn(sz, p.z); sc = __fadd_rn(sc, p.w);
    }
    const float fn = (float)c;
    float4 o = make_float4(__fdiv_rn(sx, fn), __fdiv_rn(sy, fn), __fdiv_rn(sz, fn), __fdiv_rn(sc, fn));
    out[l] = o;
    curv_bits[l] = (uint32_t)f2ord(o.w) ^ 0x80000000u;  // order-preserving unsigned key
    leaf_ids[l] = l;
    atomicAdd(n_valid, 1u);
}

__global__ void k_gather_sorted(const float4* __restrict__ cent, const uint32_t* __restrict__ ids, uint32_t n, float4* out,
                                uint32_t* heads) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = cent[ids[i]];
    out[i] = p;
    heads[i] = (i == 0 || cent[ids[i - 1]].w != p.w) ? 1u : 0u;  // maximal equal-curvature runs (KILO.cc:377-378)
}

__global__ void k_bucket_heads(const float4* __restrict__ pts, const uint32_t* __restrict__ heads, const uint32_t* __restrict__ pos,
                               uint32_t n, uint32_t* offsets, float* curv) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !heads[i]) return;
    offsets[pos[i]] = i;
    curv[pos[i]] = pts[i].w;
}

}  // namespace

int decode_pointcloud2_device(const uint8_t* h_data, uint32_t n, const lk_pc2_layout& L, float blind, int filter_num,
                              double time_scale, float* h_pts_out, float* h_intensity_out, uint32_t* n_out, cudaStream_t s,
                              std::string& err) {
    *n_out = 0;
    if (!n) return LK_OK;
    DevBuf d_data, d_flags, d_pos, d_out, d_int, d_tmp;
    const size_t bytes = (size_t)n * L.point_step;
    LK_CUDA(err, d_data.alloc(bytes));
    LK_CUDA(err, d_flags.alloc((size_t)n * 4));
    LK_CUDA(err, d_pos.alloc((size_t)n * 4));
    LK_CUDA(err, d_out.alloc((size_t)n * 16));
    LK_CUDA(err, d_int.alloc((size_t)n * 4));
    LK_CUDA(err, cudaMemcpyAsync(d_data.p, h_data, bytes, cudaMemcpyHostToDevice, s));
    const unsigned g = (n + 255) / 256;
    k_decode_flags<<<g, 256, 0, s>>>(d_data.as<uint8_t>(), n, L, blind, filter_num, d_flags.as<uint32_t>());
    size_t tb = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tb, d_flags.as<uint32_t>(), d_pos.as<uint32_t>(), (int)n, s);
    LK_CUDA(err, d_tmp.alloc(tb));
    cub::DeviceScan::ExclusiveSum(d_tmp.p, tb, d_flags.as<uint32_t>(), d_pos.as<uint32_t>(), (int)n, s);
    k_decode_scatter<<<g, 256, 0, s>>>(d_data.as<uint8_t>(), n, L, time_scale, d_flags.as<uint32_t>(), d_pos.as<uint32_t>(),
                                       d_out.as<float4>(), h_intensity_out ? d_int.as<float>() : nullptr);
    uint32_t last_pos = 0, last_flag = 0;
    LK_CUDA(err, cudaMemcpyAsync(&last_pos, d_pos.as<uint32_t>() + (n - 1), 4, cudaMemcpyDeviceToHost, s));
    LK_CUDA(err, cudaMemcpyAsync(&last_flag, d_flags.as<uint32_t>() + (n - 1), 4, cudaMemcpyDeviceToHost, s));
    LK_CUDA(err, cudaStreamSynchronize(s));
    const uint32_t m = last_pos + last_flag;
    *n_out = m;
    if (m) {
        LK_CUDA(err, cudaMemcpyAsync(h_pts_out, d_out.p, (size_t)m * 16, cudaMemcpyDeviceToHost, s));
        if (h_intensity_out) LK_CUDA(err, cudaMemcpyAsync(h_intensity_out, d_int.p, (size_t)m * 4, cudaMemcpyDeviceToHost, s));
        LK_CUDA(err, cudaStreamSynchronize(s));
    }
    LK_CUDA(err, cudaGetLastError());
    return LK_OK;
}

int preprocess_scan_device(const float* h_pts_in, uint32_t n, float leaf, float* h_pts_out, uint32_t* n_out,
                           uint32_t* h_bucket_offsets, float* h_bucket_curv, uint32_t* n_buckets, cudaStream_t s,
                           std::string& err) {
    *n_out = 0;
    *n_buckets = 0;
    if (!n) { h_bucket_offsets[0] = 0; return LK_OK; }
    DevBuf d_in, d_mm, d_idx, d_ord, d_idx2, d_ord2, d_uk, d_cnt, d_st, d_nr, d_cent, d_cb, d_lid, d_cb2, d_lid2, d_out, d_heads,
        d_pos, d_off, d_curv, d_tmp;
    LK_CUDA(err, d_in.alloc((size_t)n * 16));
    LK_CUDA(err, d_mm.alloc(64));
    LK_CUDA(err, cudaMemcpyAsync(d_in.p, h_pts_in, (size_t)n * 16, cudaMemcpyHostToDevice, s));
    int mm0[6] = {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN};
    LK_CUDA(err, cudaMemcpyAsync(d_mm.p, mm0, sizeof(mm0), cudaMemcpyHostToDevice, s));
    k_minmax<<<std::min<unsigned>((n + 255) / 256, 1184u), 256, 0, s>>>(d_in.as<float4>(), n, d_mm.as<int>());
    int mm[6];
    LK_CUDA(err, cudaMemcpyAsync(mm, d_mm.p, sizeof(mm), cudaMemcpyDeviceToHost, s));
    LK_CUDA(err, cudaStreamSynchronize(s));
    auto ord2f_h = [](int i) { int j = i >= 0 ? i : i ^ 0x7fffffff; float f; std::memcpy(&f, &j, 4); return f; };
    GridParams gp;
    gp.inv_leaf = 1.0f / leaf;  // inverse_leaf_size_ = Ones / leaf_size_ (float)
    int max_b[3], div_b[3];
    for (int k = 0; k < 3; ++k) {
        gp.min_b[k] = (int)std::floor(ord2f_h(mm[k]) * gp.inv_leaf);
        max_b[k] = (int)std::floor(ord2f_h(mm[3 + k]) * gp.inv_leaf);
        div_b[k] = max_b[k] - gp.min_b[k] + 1;
    }
    const long long cells = (long long)div_b[0] * div_b[1] * div_b[2];
    if (cells > (long long)INT_MAX) {  // PCL warns "Leaf size is too small" and returns the cloud unfiltered; we refuse
        err = "voxel grid: leaf size too small for the cloud extent (index would overflow)";
        return LK_ERR_INVALID_ARG;
    }
    gp.mul[0] = 1; gp.mul[1] = div_b[0]; gp.mul[2] = div_b[0] * div_b[1];
    const unsigned g = (n + 255) / 256;
    LK_CUDA(err, d_idx.alloc((size_t)n * 4)); LK_CUDA(err, d_ord.alloc((size_t)n * 4)); LK_CUDA(err, d_idx2.alloc((size_t)n * 4)); LK_CUDA(err, d_ord2.alloc((size_t)n * 4));
    LK_CUDA(err, d_uk.alloc((size_t)n * 4)); LK_CUDA(err, d_cnt.alloc((size_t)n * 4)); LK_CUDA(err, d_st.alloc((size_t)n * 4)); LK_CUDA(err, d_nr.alloc(16));
    k_leaf_index<<<g, 256, 0, s>>>(d_in.as<float4>(), n, gp, d_idx.as<uint32_t>(), d_ord.as<uint32_t>());
    size_t b1 = 0, b2 = 0, b3 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, b1, d_idx.as<uint32_t>(), d_idx2.as<uint32_t>(), d_ord.as<uint32_t>(), d_ord2.as<uint32_t>(), (int)n, 0, 32, s);
    cub::DeviceRunLengthEncode::Encode(nullptr, b2, d_idx2.as<uint32_t>(), d_uk.as<uint32_t>(), d_cnt.as<uint32_t>(), d_nr.as<uint32_t>(), (int)n, s);
    cub::DeviceScan::ExclusiveSum(nullptr, b3, d_cnt.as<uint32_t>(), d_st.as<uint32_t>(), (int)n, s);
    const size_t tb = std::max(b1, std::max(b2, b3));
    LK_CUDA(err, d_tmp.alloc(tb));
    size_t tb2 = tb;
    cub::DeviceRadixSort::SortPairs(d_tmp.p, tb2, d_idx.as<uint32_t>(), d_idx2.as<uint32_t>(), d_ord.as<uint32_t>(), d_ord2.as<uint32_t>(), (int)n, 0, 32, s);
    tb2 = tb;
    cub::DeviceRunLengthEncode::Encode(d_tmp.p, tb2, d_idx2.as<uint32_t>(), d_uk.as<uint32_t>(), d_cnt.as<uint32_t>(), d_nr.as<uint32_t>(), (int)n, s);
    uint32_t n_leaves = 0;
    LK_CUDA(err, cudaMemcpyAsync(&n_leaves, d_nr.p, 4, cudaMemcpyDeviceToHost, s));
    LK_CUDA(err, cudaStreamSynchronize(s));
    tb2 = tb;
    cub::DeviceScan::ExclusiveSum(d_tmp.p, tb2, d_cnt.as<uint32_t>(), d_st.as<uint32_t>(), (int)n_leaves, s);
    LK_CUDA(err, d_cent.alloc((size_t)n_leaves * 16)); LK_CUDA(err, d_cb.alloc((size_t)n_leaves * 4)); LK_CUDA(err, d_lid.alloc((size_t)n_leaves * 4));
    LK_CUDA(err, d_cb2.alloc((size_t)n_leaves * 4)); LK_CUDA(err, d_lid2.alloc((size_t)n_leaves * 4)); LK_CUDA(err, d_out.alloc((size_t)n_leaves * 16));
    LK_CUDA(err, d_heads.alloc((size_t)n_leaves * 4)); LK_CUDA(err, d_pos.alloc((size_t)n_leaves * 4));
    LK_CUDA(err, d_off.alloc(((size_t)n_leaves + 1) * 4)); LK_CUDA(err, d_curv.alloc((size_t)n_leaves * 4));
    LK_CUDA(err, cudaMemsetAsync(d_nr.p, 0, 16, s));
    k_centroids<<<(n_leaves + 127) / 128, 128, 0, s>>>(d_in.as<float4>(), d_ord2.as<uint32_t>(), d_uk.as<uint32_t>(), d_cnt.as<uint32_t>(),
                                                       d_st.as<uint32_t>(), n_leaves, d_cent.as<float4>(), d_cb.as<uint32_t>(),
                                                       d_lid.as<uint32_t>(), d_nr.as<uint32_t>());
    uint32_t n_valid = 0;
    LK_CUDA(err, cudaMemcpyAsync(&n_valid, d_nr.p, 4, cudaMemcpyDeviceToHost, s));
    LK_CUDA(err, cudaStreamSynchronize(s));
    // non-finite points form the LAST run (key 0xffffffff) and were skipped: the first n_valid leaves are the output
    if (n_valid) {
        size_t c1 = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, c1, d_cb.as<uint32_t>(), d_cb2.as<uint32_t>(), d_lid.as<uint32_t>(), d_lid2.as<uint32_t>(), (int)n_valid, 0, 32, s);
        DevBuf d_t2;
        LK_CUDA(err, d_t2.alloc(c1));
        cub::DeviceRadixSort::SortPairs(d_t2.p, c1, d_cb.as<uint32_t>(), d_cb2.as<uint32_t>(), d_lid.as<uint32_t>(), d_lid2.as<uint32_t>(), (int)n_valid, 0, 32, s);
        const unsigned gl = (n_valid + 255) / 256;
        k_gather_sorted<<<gl, 256, 0, s>>>(d_cent.as<float4>(), d_lid2.as<uint32_t>(), n_valid, d_out.as<float4>(), d_heads.as<uint32_t>());
        size_t c2 = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, c2, d_heads.as<uint32_t>(), d_pos.as<uint32_t>(), (int)n_valid, s);
        DevBuf d_t3;
        LK_CUDA(err, d_t3.alloc(c2));
        cub::DeviceScan::ExclusiveSum(d_t3.p, c2, d_heads.as<uint32_t>(), d_pos.as<uint32_t>(), (int)n_valid, s);
        k_bucket_heads<<<gl, 256, 0, s>>>(d_out.as<float4>(), d_heads.as<uint32_t>(), d_pos.as<uint32_t>(), n_valid, d_off.as<uint32_t>(), d_curv.as<float>());
        uint32_t lp = 0, lh = 0;
        LK_CUDA(err, cudaMemcpyAsync(&lp, d_pos.as<uint32_t>() + (n_valid - 1), 4, cudaMemcpyDeviceToHost, s));
        LK_CUDA(err, cudaMemcpyAsync(&lh, d_heads.as<uint32_t>() + (n_valid - 1), 4, cudaMemcpyDeviceToHost, s));
        LK_CUDA(err, cudaStreamSynchronize(s));
        const uint32_t nb = lp + lh;
        LK_CUDA(err, cudaMemcpyAsync(h_pts_out, d_out.p, (size_t)n_valid * 16, cudaMemcpyDeviceToHost, s));
        LK_CUDA(err, cudaMemcpyAsync(h_bucket_offsets, d_off.p, (size_t)nb * 4, cudaMemcpyDeviceToHost, s));
        LK_CUDA(err, cudaMemcpyAsync(h_bucket_curv, d_curv.p, (size_t)nb * 4, cudaMemcpyDeviceToHost, s));
        LK_CUDA(err, cudaStreamSynchronize(s));
        h_bucket_offsets[nb] = n_valid;
        *n_buckets = nb;
    } else {
        h_bucket_offsets[0] = 0;
    }
    *n_out = n_valid;
    LK_CUDA(err, cudaGetLastError());
    return LK_OK;
}

}  // namespace lk
