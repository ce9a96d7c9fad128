// lk_preprocess.cu — what feeds the hot path (SURVEY §8f ranks 2-3), on the device:
//   * wire decode of sensor_msgs/PointCloud2 for the three driver layouts
//     (legkilo/src/preprocess/lidar_processing.cc:25-108): every filter_num-th point, blind-sphere test,
//     time offset rounded to 1/500 s, stable compaction, begin / end times; a batch of messages in one pass
//     (lk_decode_pointcloud2s; lk_decode_pointcloud2 is the batch of one);
//   * pcl::VoxelGrid centroid down-sampling as KILO::process uses it (KILO.cc:82-83, :356-360; PCL 1.8
//     voxel_grid.hpp — the library is absent from /root/reference, its published algorithm is restated),
//     then the sort by curvature and the equal-curvature bucket boundaries (KILO.cc:370-378), for a batch of scans
//     in one pass (lk_preprocess_scans; lk_preprocess_scan is the batch of one).
// Sorting / scanning / run-length encoding use CUB (library code, like cuBLAS for a plain GEMM); the
// per-point and per-leaf arithmetic is hand-written and bit-identical to the CPU restatement.
#include <cub/cub.cuh>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "lk_device.cuh"
#include "lk_host.h"

namespace lk {

namespace {

// ---- decode of a batch of messages ------------------------------------------------------------------
// Message m is points [offs[m], offs[m+1]) of one device buffer (messages lie back to back, one layout), so point i is at
// byte i * point_step. Every rule that depends on the message reads it through msg_of: the filter_num stride counts from
// the message's own first point, and the time offset is taken from the message's own first raw point.
__device__ __forceinline__ uint32_t msg_of(const uint32_t* __restrict__ offs, uint32_t n_msgs, uint32_t i) {
    uint32_t lo = 0, hi = n_msgs;  // the last m with offs[m] <= i (an empty message m has offs[m] == offs[m + 1])
    while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (offs[mid] <= i) lo = mid;
        else hi = mid;
    }
    return lo;
}

__global__ void k_decode_flags(const uint8_t* __restrict__ data, const uint32_t* __restrict__ offs, uint32_t n_msgs, uint32_t n,
                               lk_pc2_layout L, float blind, int filter_num, uint32_t* flags) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t* p = data + (size_t)i * L.point_step;
    float x, y, z;
    memcpy(&x, p + L.off_x, 4); memcpy(&y, p + L.off_y, 4); memcpy(&z, p + L.off_z, 4);
    // blindCheck (lidar_processing.h:94-97): blind*blind > x*x + y*y + z*z, float, no contraction
    const float r2 = __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
    const uint32_t k = i - offs[msg_of(offs, n_msgs, i)];
    const bool drop = (k % (uint32_t)filter_num) != 0 || (__fmul_rn(blind, blind) > r2);
    flags[i] = drop ? 0u : 1u;
}

__device__ __forceinline__ double raw_time(const uint8_t* p, const lk_pc2_layout& L) {
    if (L.lidar_type == LK_LIDAR_VELODYNE) { float t; memcpy(&t, p + L.off_time, 4); return (double)t; }
    if (L.lidar_type == LK_LIDAR_OUSTER) { uint32_t t; memcpy(&t, p + L.off_time, 4); return (double)t; }
    double t; memcpy(&t, p + L.off_time, 8); return t;
}

__global__ void k_decode_scatter(const uint8_t* __restrict__ data, const uint32_t* __restrict__ offs, uint32_t n_msgs, uint32_t n,
                                 lk_pc2_layout L, double time_scale, const uint32_t* __restrict__ flags,
                                 const uint32_t* __restrict__ pos, float4* out, float* intensity) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !flags[i]) return;
    const uint8_t* p = data + (size_t)i * L.point_step;
    float4 o;
    memcpy(&o.x, p + L.off_x, 4); memcpy(&o.y, p + L.off_y, 4); memcpy(&o.z, p + L.off_z, 4);
    const double t0 = raw_time(data + (size_t)offs[msg_of(offs, n_msgs, i)] * L.point_step, L), ti = raw_time(p, L);
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

// Per message m <= n_msgs: its first output point (the exclusive sum at its first raw point; the total past the last
// point), and for m < n_msgs lidar_begin_time_ / lidar_end_time_ (:31-35, :59-63, :87-91), NaN for an empty message.
__global__ void k_decode_msgs(const uint8_t* __restrict__ data, const uint32_t* __restrict__ offs, uint32_t n_msgs, uint32_t n,
                              lk_pc2_layout L, double time_scale, const double* __restrict__ stamps,
                              const uint32_t* __restrict__ flags, const uint32_t* __restrict__ pos, uint32_t* out_offs,
                              double* begin, double* end) {
    const uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m > n_msgs) return;
    const uint32_t a = offs[m];
    out_offs[m] = a < n ? pos[a] : pos[n - 1] + flags[n - 1];
    if (m == n_msgs) return;
    const uint32_t b = offs[m + 1];
    double tb = __longlong_as_double(0x7ff8000000000000ll), te = tb;  // the quiet NaN std::nan("") gives on the host
    if (b > a) {
        const double f = time_scale * raw_time(data + (size_t)a * L.point_step, L);
        const double l = time_scale * raw_time(data + (size_t)(b - 1) * L.point_step, L);
        if (L.lidar_type == LK_LIDAR_HESAI) { tb = f; te = l; }  // no header stamp (:90-91)
        else {
            const double st = stamps ? stamps[m] : 0.0;  // stamp + float first / last point time (:34-35)
            tb = st + (double)(float)f;
            te = st + (double)(float)l;
        }
    }
    begin[m] = tb;
    end[m] = te;
}

// ---- voxel grid, time sort and buckets of a batch of scans -------------------------------------------------
// The 2-D kernels take one scan per blockIdx.x and cut it into gridDim.y slices: scan s is pts[offs[s] .. offs[s + 1]).
// Keys carry the scan in their high word, so one sort keeps every scan apart and orders each one exactly as a sort of
// that scan alone would (CUB's radix sort is stable).
__device__ __forceinline__ int f2ord(float f) { int i = __float_as_int(f); return i >= 0 ? i : i ^ 0x7fffffff; }

constexpr uint32_t kNonFinite = 0xffffffffu;  // leaf index of a non-finite point: its scan's last run

__global__ void k_minmax(const float4* __restrict__ pts, const uint32_t* __restrict__ offs,
                         int* mm /* [6 per scan]: min xyz, max xyz (ordered ints) */) {
    __shared__ int s[6][256];
    const uint32_t scan = blockIdx.x, end = offs[scan + 1];
    const uint32_t first = offs[scan] + blockIdx.y * blockDim.x;
    if (first >= end) return;  // block-uniform
    int mn[3] = {INT_MAX, INT_MAX, INT_MAX}, mx[3] = {INT_MIN, INT_MIN, INT_MIN};
    for (uint32_t i = first + threadIdx.x; i < end; i += gridDim.y * blockDim.x) {
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
    if (threadIdx.x < 3) atomicMin(&mm[6 * scan + threadIdx.x], s[threadIdx.x][0]);
    else if (threadIdx.x < 6) atomicMax(&mm[6 * scan + threadIdx.x], s[threadIdx.x][0]);
}

struct GridParams {
    float inv_leaf;
    int min_b[3];
    int mul[3];
};

__global__ void k_leaf_index(const float4* __restrict__ pts, const uint32_t* __restrict__ offs,
                             const GridParams* __restrict__ grids, uint64_t* key, uint32_t* order) {
    const uint32_t scan = blockIdx.x, end = offs[scan + 1];
    const GridParams gp = grids[scan];
    for (uint32_t i = offs[scan] + blockIdx.y * blockDim.x + threadIdx.x; i < end; i += gridDim.y * blockDim.x) {
        const float4 p = pts[i];
        // voxel_grid.hpp: ijk = floor(p * inverse_leaf_size) - min_b ; idx = ijk . divb_mul   (non-finite -> last)
        uint32_t v = kNonFinite;
        if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
            const int i0 = (int)floorf(__fmul_rn(p.x, gp.inv_leaf)) - gp.min_b[0];
            const int i1 = (int)floorf(__fmul_rn(p.y, gp.inv_leaf)) - gp.min_b[1];
            const int i2 = (int)floorf(__fmul_rn(p.z, gp.inv_leaf)) - gp.min_b[2];
            v = (uint32_t)(i0 * gp.mul[0] + i1 * gp.mul[1] + i2 * gp.mul[2]);
        }
        key[i] = (uint64_t)scan << 32 | v;
        order[i] = i;
    }
}

// One thread per leaf: float sums in original point order, divided by float(n) (CentroidPoint of PCL 1.8). The time-sort
// key is (scan, order-preserving curvature bits); a scan's run of non-finite points gets scan = n_scans instead, so the
// sort moves those runs behind every centroid and the valid leaves end up compacted at the front.
__global__ void k_centroids(const float4* __restrict__ pts, const uint32_t* __restrict__ order, const uint64_t* __restrict__ ukeys,
                            const uint32_t* __restrict__ counts, const uint32_t* __restrict__ starts, uint32_t n_leaves,
                            uint32_t n_scans, float4* out, uint64_t* tkey, uint32_t* leaf_ids) {
    const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= n_leaves) return;
    leaf_ids[l] = l;
    const uint64_t k = ukeys[l];
    if ((uint32_t)k == kNonFinite) { tkey[l] = (uint64_t)n_scans << 32; return; }
    float sx = 0.f, sy = 0.f, sz = 0.f, sc = 0.f;
    const uint32_t s0 = starts[l], c = counts[l];
    for (uint32_t j = 0; j < c; ++j) {
        const float4 p = pts[order[s0 + j]];
        sx = __fadd_rn(sx, p.x); sy = __fadd_rn(sy, p.y); sz = __fadd_rn(sz, p.z); sc = __fadd_rn(sc, p.w);
    }
    const float fn = (float)c;
    float4 o = make_float4(__fdiv_rn(sx, fn), __fdiv_rn(sy, fn), __fdiv_rn(sz, fn), __fdiv_rn(sc, fn));
    out[l] = o;
    tkey[l] = (k & 0xffffffff00000000ull) | ((uint32_t)f2ord(o.w) ^ 0x80000000u);
}

__global__ void k_gather_sorted(const float4* __restrict__ cent, const uint64_t* __restrict__ tkey, const uint32_t* __restrict__ ids,
                                uint32_t n, uint32_t n_scans, float4* out, uint32_t* heads) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t scan = (uint32_t)(tkey[i] >> 32);
    if (scan >= n_scans) { heads[i] = 0u; return; }  // a non-finite run
    const float4 p = cent[ids[i]];
    out[i] = p;
    // maximal equal-curvature runs of one scan (KILO.cc:377-378)
    heads[i] = (i == 0 || (uint32_t)(tkey[i - 1] >> 32) != scan || cent[ids[i - 1]].w != p.w) ? 1u : 0u;
}

// incl = inclusive sum of heads: the bucket a head starts is incl[i] - 1.
__global__ void k_bucket_heads(const float4* __restrict__ pts, const uint64_t* __restrict__ tkey, const uint32_t* __restrict__ heads,
                               const uint32_t* __restrict__ incl, uint32_t n, const double* __restrict__ begin_times,
                               uint32_t* offsets, float* curv, double* times) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !heads[i]) return;
    const uint32_t b = incl[i] - 1u;
    const float c = pts[i].w;
    offsets[b] = i;
    curv[b] = c;
    if (times) times[b] = begin_times[tkey[i] >> 32] + (double)c;  // t_b = lidar_begin_time_ + curvature (KILO.cc:376)
}

// Per scan s <= n_scans: its first output point (the first sorted key of scan >= s) and the buckets before it.
__global__ void k_scan_ptrs(const uint64_t* __restrict__ tkey, const uint32_t* __restrict__ incl, uint32_t n, uint32_t n_scans,
                            uint32_t* scan_offsets, uint32_t* scan_bucket_ptr) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s > n_scans) return;
    const uint64_t k = (uint64_t)s << 32;
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (tkey[mid] < k) lo = mid + 1;
        else hi = mid;
    }
    scan_offsets[s] = lo;
    scan_bucket_ptr[s] = lo ? incl[lo - 1] : 0u;
}

uint32_t bit_width(uint32_t v) { uint32_t b = 0; while (v) { ++b; v >>= 1; } return b; }

size_t align_up(size_t b) { return (b + 255) & ~size_t(255); }

// Device scratch of one lk_preprocess_scans call, one block carved in this order. n points, n_scans scans; every
// per-leaf array is sized by n (a scan has at most as many leaves as points). A later phase reuses an array an earlier
// one is done with: the leaf keys hold the time keys, the point order the leaf ids, the run counts / starts the bucket
// heads / their sum.
struct PreScratch {
    size_t pts, offs, begin, grids, mm, nruns, key, key_s, ukeys, ord, ord_s, cnt, start, cent, out, boff, bcurv, btimes,
        scan_off, scan_bptr, tmp, total;
    PreScratch(uint32_t n, uint32_t n_scans) {
        const int ni = (int)n;
        const int leaf_bits = 32 + (int)bit_width(n_scans - 1), time_bits = 32 + (int)bit_width(n_scans);
        size_t t1 = 0, t2 = 0, t3 = 0, t4 = 0, t5 = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, t1, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const uint32_t*)nullptr,
                                        (uint32_t*)nullptr, ni, 0, leaf_bits);
        cub::DeviceRadixSort::SortPairs(nullptr, t2, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const uint32_t*)nullptr,
                                        (uint32_t*)nullptr, ni, 0, time_bits);
        cub::DeviceRunLengthEncode::Encode(nullptr, t3, (const uint64_t*)nullptr, (uint64_t*)nullptr, (uint32_t*)nullptr,
                                           (uint32_t*)nullptr, ni);
        cub::DeviceScan::ExclusiveSum(nullptr, t4, (const uint32_t*)nullptr, (uint32_t*)nullptr, ni);
        cub::DeviceScan::InclusiveSum(nullptr, t5, (const uint32_t*)nullptr, (uint32_t*)nullptr, ni);
        size_t o = 0;
        auto take = [&o](size_t bytes) { const size_t at = o; o += align_up(bytes); return at; };
        pts = take((size_t)n * 16);
        offs = take(((size_t)n_scans + 1) * 4);
        begin = take((size_t)n_scans * 8);
        grids = take((size_t)n_scans * sizeof(GridParams));
        mm = take((size_t)n_scans * 6 * 4);
        nruns = take(4);
        key = take((size_t)n * 8);
        key_s = take((size_t)n * 8);
        ukeys = take((size_t)n * 8);
        ord = take((size_t)n * 4);
        ord_s = take((size_t)n * 4);
        cnt = take((size_t)n * 4);
        start = take((size_t)n * 4);
        cent = take((size_t)n * 16);
        out = take((size_t)n * 16);
        boff = take((size_t)n * 4);
        bcurv = take((size_t)n * 4);
        btimes = take((size_t)n * 8);
        scan_off = take(((size_t)n_scans + 1) * 4);
        scan_bptr = take(((size_t)n_scans + 1) * 4);
        tmp = take(std::max({t1, t2, t3, t4, t5}));
        total = o;
    }
};


// Device scratch of one lk_decode_pointcloud2s call, one block carved in this order: the raw bytes of n points, the
// message offsets / stamps, keep flags and their exclusive sum, the decoded points, and the per-message outputs.
struct DecScratch {
    size_t data, offs, stamps, flags, pos, out, inten, out_offs, begin, end, tmp, total;
    DecScratch(uint32_t n, uint32_t n_msgs, uint32_t point_step) {
        size_t tb = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, tb, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n);
        size_t o = 0;
        auto take = [&o](size_t bytes) { const size_t at = o; o += align_up(bytes); return at; };
        data = take((size_t)n * point_step);
        offs = take(((size_t)n_msgs + 1) * 4);
        stamps = take((size_t)n_msgs * 8);
        flags = take((size_t)n * 4);
        pos = take((size_t)n * 4);
        out = take((size_t)n * 16);
        inten = take((size_t)n * 4);
        out_offs = take(((size_t)n_msgs + 1) * 4);
        begin = take((size_t)n_msgs * 8);
        end = take((size_t)n_msgs * 8);
        tmp = take(tb);
        total = o;
    }
};

}  // namespace

// lk_decode_pointcloud2s behind its argument checks: n_msgs >= 1, every data[m] with points non-null, the sum of the
// point counts at most INT_MAX. `scratch` is grown to the call's size. Two host synchronisations whatever n_msgs is: the
// per-message offsets and times, then the copy-out of the points.
int decode_pointcloud2s_device(uint32_t n_msgs, const uint8_t* const* h_data, const uint32_t* h_n, const double* h_stamps,
                               const lk_pc2_layout& L, float blind, int filter_num, double time_scale, float* h_pts_out,
                               float* h_intensity_out, uint32_t* h_out_offs, double* h_begin, double* h_end, DevBuf& scratch,
                               cudaStream_t s, std::string& err) {
    std::vector<uint32_t> offs(n_msgs + 1);
    offs[0] = 0;
    for (uint32_t m = 0; m < n_msgs; ++m) offs[m + 1] = offs[m] + h_n[m];
    const uint32_t n = offs[n_msgs];
    if (!n) {
        const double nan = std::nan("");
        for (uint32_t m = 0; m <= n_msgs; ++m) h_out_offs[m] = 0;
        for (uint32_t m = 0; m < n_msgs; ++m) {
            if (h_begin) h_begin[m] = nan;
            if (h_end) h_end[m] = nan;
        }
        return LK_OK;
    }
    const DecScratch D(n, n_msgs, L.point_step);
    LK_CUDA(err, scratch.ensure(D.total));
    char* base_p = static_cast<char*>(scratch.p);
    auto at = [base_p](size_t off) { return reinterpret_cast<void*>(base_p + off); };
    auto* d_data = static_cast<uint8_t*>(at(D.data));
    auto* d_offs = static_cast<uint32_t*>(at(D.offs));
    auto* d_stamps = static_cast<double*>(at(D.stamps));
    auto* d_flags = static_cast<uint32_t*>(at(D.flags));
    auto* d_pos = static_cast<uint32_t*>(at(D.pos));
    auto* d_out = static_cast<float4*>(at(D.out));
    auto* d_int = static_cast<float*>(at(D.inten));
    auto* d_out_offs = static_cast<uint32_t*>(at(D.out_offs));
    auto* d_begin = static_cast<double*>(at(D.begin));
    auto* d_end = static_cast<double*>(at(D.end));
    size_t tb = D.total - D.tmp;

    for (uint32_t m = 0; m < n_msgs; ++m)
        if (h_n[m])
            LK_CUDA(err, cudaMemcpyAsync(d_data + (size_t)offs[m] * L.point_step, h_data[m], (size_t)h_n[m] * L.point_step,
                                         cudaMemcpyHostToDevice, s));
    LK_CUDA(err, cudaMemcpyAsync(d_offs, offs.data(), offs.size() * 4, cudaMemcpyHostToDevice, s));
    if (h_stamps) LK_CUDA(err, cudaMemcpyAsync(d_stamps, h_stamps, (size_t)n_msgs * 8, cudaMemcpyHostToDevice, s));
    const unsigned g = (n + 255) / 256;
    k_decode_flags<<<g, 256, 0, s>>>(d_data, d_offs, n_msgs, n, L, blind, filter_num, d_flags);
    LK_CUDA(err, cub::DeviceScan::ExclusiveSum(at(D.tmp), tb, d_flags, d_pos, (int)n, s));
    k_decode_scatter<<<g, 256, 0, s>>>(d_data, d_offs, n_msgs, n, L, time_scale, d_flags, d_pos, d_out,
                                       h_intensity_out ? d_int : nullptr);
    k_decode_msgs<<<(n_msgs + 256) / 256, 256, 0, s>>>(d_data, d_offs, n_msgs, n, L, time_scale, h_stamps ? d_stamps : nullptr,
                                                      d_flags, d_pos, d_out_offs, d_begin, d_end);
    LK_CUDA(err, cudaGetLastError());
    LK_CUDA(err, cudaMemcpyAsync(h_out_offs, d_out_offs, ((size_t)n_msgs + 1) * 4, cudaMemcpyDeviceToHost, s));
    if (h_begin) LK_CUDA(err, cudaMemcpyAsync(h_begin, d_begin, (size_t)n_msgs * 8, cudaMemcpyDeviceToHost, s));
    if (h_end) LK_CUDA(err, cudaMemcpyAsync(h_end, d_end, (size_t)n_msgs * 8, cudaMemcpyDeviceToHost, s));
    LK_CUDA(err, cudaStreamSynchronize(s));
    const uint32_t n_out = h_out_offs[n_msgs];
    if (n_out) {
        LK_CUDA(err, cudaMemcpyAsync(h_pts_out, d_out, (size_t)n_out * 16, cudaMemcpyDeviceToHost, s));
        if (h_intensity_out) LK_CUDA(err, cudaMemcpyAsync(h_intensity_out, d_int, (size_t)n_out * 4, cudaMemcpyDeviceToHost, s));
        LK_CUDA(err, cudaStreamSynchronize(s));
    }
    return LK_OK;
}

// lk_preprocess_scans behind its argument checks: n_scans >= 1, h_offs non-decreasing. `scratch` is grown to the call's
// size. Four host synchronisations whatever n_scans is: the bounding boxes, the leaf count, the output totals, the copy-out.
int preprocess_scans_device(uint32_t n_scans, const float* h_pts_in, const uint32_t* h_offs, float leaf, const double* h_begin,
                            float* h_pts_out, uint32_t* h_scan_off, uint32_t* h_scan_bptr, uint32_t* h_boff, float* h_bcurv,
                            double* h_btimes, DevBuf& scratch, cudaStream_t s, std::string& err) {
    const uint32_t base = h_offs[0], n = h_offs[n_scans] - base;
    if (n > (uint32_t)INT_MAX) {
        err = "voxel grid: more than INT_MAX points in one call";
        return LK_ERR_INVALID_ARG;
    }
    if (!n) {
        for (uint32_t i = 0; i <= n_scans; ++i) h_scan_off[i] = h_scan_bptr[i] = 0;
        h_boff[0] = 0;
        return LK_OK;
    }
    std::vector<uint32_t> offs(n_scans + 1);
    uint32_t widest = 0;
    for (uint32_t i = 0; i <= n_scans; ++i) offs[i] = h_offs[i] - base;
    for (uint32_t i = 0; i < n_scans; ++i) widest = std::max(widest, offs[i + 1] - offs[i]);
    const PreScratch L(n, n_scans);
    LK_CUDA(err, scratch.ensure(L.total));
    char* base_p = static_cast<char*>(scratch.p);
    auto at = [base_p](size_t off) { return reinterpret_cast<void*>(base_p + off); };
    auto* d_pts = static_cast<float4*>(at(L.pts));
    auto* d_offs = static_cast<uint32_t*>(at(L.offs));
    auto* d_begin = static_cast<double*>(at(L.begin));
    auto* d_grids = static_cast<GridParams*>(at(L.grids));
    auto* d_mm = static_cast<int*>(at(L.mm));
    auto* d_nruns = static_cast<uint32_t*>(at(L.nruns));
    auto* d_key = static_cast<uint64_t*>(at(L.key));      // leaf keys, then time keys
    auto* d_key_s = static_cast<uint64_t*>(at(L.key_s));  // sorted leaf keys, then sorted time keys
    auto* d_ukeys = static_cast<uint64_t*>(at(L.ukeys));
    auto* d_ord = static_cast<uint32_t*>(at(L.ord));      // point order, then leaf ids
    auto* d_ord_s = static_cast<uint32_t*>(at(L.ord_s));  // sorted point order, then leaf ids in time order
    auto* d_cnt = static_cast<uint32_t*>(at(L.cnt));      // points per leaf, then bucket heads
    auto* d_start = static_cast<uint32_t*>(at(L.start));  // first point of each leaf, then the inclusive sum of the heads
    auto* d_cent = static_cast<float4*>(at(L.cent));
    auto* d_out = static_cast<float4*>(at(L.out));
    auto* d_boff = static_cast<uint32_t*>(at(L.boff));
    auto* d_bcurv = static_cast<float*>(at(L.bcurv));
    auto* d_btimes = static_cast<double*>(at(L.btimes));
    auto* d_scan_off = static_cast<uint32_t*>(at(L.scan_off));
    auto* d_scan_bptr = static_cast<uint32_t*>(at(L.scan_bptr));
    void* d_tmp = at(L.tmp);
    const size_t tmp_bytes = L.total - L.tmp;

    // 1. per-scan bounding boxes
    std::vector<int> mm(6 * (size_t)n_scans);
    for (uint32_t i = 0; i < n_scans; ++i)
        for (int k = 0; k < 3; ++k) { mm[6 * i + k] = INT_MAX; mm[6 * i + 3 + k] = INT_MIN; }
    LK_CUDA(err, cudaMemcpyAsync(d_pts, h_pts_in + 4 * (size_t)base, (size_t)n * 16, cudaMemcpyHostToDevice, s));
    LK_CUDA(err, cudaMemcpyAsync(d_offs, offs.data(), offs.size() * 4, cudaMemcpyHostToDevice, s));
    if (h_begin) LK_CUDA(err, cudaMemcpyAsync(d_begin, h_begin, (size_t)n_scans * 8, cudaMemcpyHostToDevice, s));
    LK_CUDA(err, cudaMemcpyAsync(d_mm, mm.data(), mm.size() * 4, cudaMemcpyHostToDevice, s));
    const dim3 per_scan(n_scans, std::min<uint32_t>(std::max<uint32_t>((widest + 2047) / 2048, 1u), 64u));
    k_minmax<<<per_scan, 256, 0, s>>>(d_pts, d_offs, d_mm);
    LK_CUDA(err, cudaMemcpyAsync(mm.data(), d_mm, mm.size() * 4, cudaMemcpyDeviceToHost, s));
    LK_CUDA(err, cudaStreamSynchronize(s));

    // 2. the grid of every scan on its own bounding box; leaf keys (scan, leaf index), stable sort
    auto ord2f_h = [](int i) { int j = i >= 0 ? i : i ^ 0x7fffffff; float f; std::memcpy(&f, &j, 4); return f; };
    std::vector<GridParams> grids(n_scans);
    for (uint32_t i = 0; i < n_scans; ++i) {
        GridParams& gp = grids[i];
        gp = GridParams{};
        gp.inv_leaf = 1.0f / leaf;  // inverse_leaf_size_ = Ones / leaf_size_ (float)
        if (mm[6 * i] == INT_MAX) continue;  // no finite point: every key is the non-finite run's
        int max_b[3], div_b[3];
        for (int k = 0; k < 3; ++k) {
            gp.min_b[k] = (int)std::floor(ord2f_h(mm[6 * i + k]) * gp.inv_leaf);
            max_b[k] = (int)std::floor(ord2f_h(mm[6 * i + 3 + k]) * gp.inv_leaf);
            div_b[k] = max_b[k] - gp.min_b[k] + 1;
        }
        const long long cells = (long long)div_b[0] * div_b[1] * div_b[2];
        if (cells > (long long)INT_MAX) {  // PCL warns "Leaf size is too small" and returns the cloud unfiltered; we refuse
            err = "voxel grid: leaf size too small for the extent of scan " + std::to_string(i) + " (index would overflow)";
            return LK_ERR_INVALID_ARG;
        }
        gp.mul[0] = 1; gp.mul[1] = div_b[0]; gp.mul[2] = div_b[0] * div_b[1];
    }
    LK_CUDA(err, cudaMemcpyAsync(d_grids, grids.data(), grids.size() * sizeof(GridParams), cudaMemcpyHostToDevice, s));
    k_leaf_index<<<per_scan, 256, 0, s>>>(d_pts, d_offs, d_grids, d_key, d_ord);
    size_t tb = tmp_bytes;
    LK_CUDA(err, cub::DeviceRadixSort::SortPairs(d_tmp, tb, d_key, d_key_s, d_ord, d_ord_s, (int)n, 0,
                                                 32 + (int)bit_width(n_scans - 1), s));

    // 3. leaves: runs of equal keys, centroids
    tb = tmp_bytes;
    LK_CUDA(err, cub::DeviceRunLengthEncode::Encode(d_tmp, tb, d_key_s, d_ukeys, d_cnt, d_nruns, (int)n, s));
    uint32_t n_leaves = 0;
    LK_CUDA(err, cudaMemcpyAsync(&n_leaves, d_nruns, 4, cudaMemcpyDeviceToHost, s));
    LK_CUDA(err, cudaStreamSynchronize(s));
    tb = tmp_bytes;
    LK_CUDA(err, cub::DeviceScan::ExclusiveSum(d_tmp, tb, d_cnt, d_start, (int)n_leaves, s));
    const unsigned gl = (n_leaves + 255) / 256;
    k_centroids<<<gl, 256, 0, s>>>(d_pts, d_ord_s, d_ukeys, d_cnt, d_start, n_leaves, n_scans, d_cent, d_key, d_ord);

    // 4. time order (scan, curvature), buckets, per-scan offsets
    tb = tmp_bytes;
    LK_CUDA(err, cub::DeviceRadixSort::SortPairs(d_tmp, tb, d_key, d_key_s, d_ord, d_ord_s, (int)n_leaves, 0,
                                                 32 + (int)bit_width(n_scans), s));
    k_gather_sorted<<<gl, 256, 0, s>>>(d_cent, d_key_s, d_ord_s, n_leaves, n_scans, d_out, d_cnt);
    tb = tmp_bytes;
    LK_CUDA(err, cub::DeviceScan::InclusiveSum(d_tmp, tb, d_cnt, d_start, (int)n_leaves, s));
    k_bucket_heads<<<gl, 256, 0, s>>>(d_out, d_key_s, d_cnt, d_start, n_leaves, d_begin, d_boff, d_bcurv,
                                      h_btimes ? d_btimes : nullptr);
    k_scan_ptrs<<<(n_scans + 256) / 256, 256, 0, s>>>(d_key_s, d_start, n_leaves, n_scans, d_scan_off, d_scan_bptr);
    LK_CUDA(err, cudaGetLastError());
    LK_CUDA(err, cudaMemcpyAsync(h_scan_off, d_scan_off, ((size_t)n_scans + 1) * 4, cudaMemcpyDeviceToHost, s));
    LK_CUDA(err, cudaMemcpyAsync(h_scan_bptr, d_scan_bptr, ((size_t)n_scans + 1) * 4, cudaMemcpyDeviceToHost, s));
    LK_CUDA(err, cudaStreamSynchronize(s));
    const uint32_t n_out = h_scan_off[n_scans], n_buckets = h_scan_bptr[n_scans];
    if (n_out) {
        LK_CUDA(err, cudaMemcpyAsync(h_pts_out, d_out, (size_t)n_out * 16, cudaMemcpyDeviceToHost, s));
        LK_CUDA(err, cudaMemcpyAsync(h_boff, d_boff, (size_t)n_buckets * 4, cudaMemcpyDeviceToHost, s));
        LK_CUDA(err, cudaMemcpyAsync(h_bcurv, d_bcurv, (size_t)n_buckets * 4, cudaMemcpyDeviceToHost, s));
        if (h_btimes) LK_CUDA(err, cudaMemcpyAsync(h_btimes, d_btimes, (size_t)n_buckets * 8, cudaMemcpyDeviceToHost, s));
        LK_CUDA(err, cudaStreamSynchronize(s));
    }
    h_boff[n_buckets] = n_out;
    return LK_OK;
}

}  // namespace lk
