// lk_score.cu — lk_score_poses: the sums the LiDAR update would form, at many candidate poses of each point set, against a
// map that stays fixed for the call; and lk_refine_poses, which steps each pose from those sums. No filter is read or
// written.
//
// k_score: one block per (256-point chunk of a set, tile of up to SCORE_TILE of that set's poses). The block loads its chunk
// once and forms what does not depend on the pose once (lk_point.cuh: body_point, kept in the lane's LaneCache); then, pose
// after pose, one points_pass (lk_pass.cuh) on the hot plane images: world point, both probes, staging, gates and row. The
// lane cache also keeps the voxel keys, their roots and the staged images from one pose to the next: a point that stays in
// its voxel (neighbouring poses of a search grid) skips both probes and both gathers. The map is fixed for the call, so what
// is cached is exactly what a fresh probe would find, and a pose's row does not depend on which poses share its tile.
// Each pose's rows of the chunk are reduced to one partial row (block_row, fixed order).
//
// k_score_sum: one block per pose, its set's partial rows summed in ascending groups (block_sum_partials), so the record of
// a pose depends only on that pose and its set.
//
// k_refine_step (lk_refine_poses): one warp per pose, one pose step from the pose's record: the information-form solve of
// block_solve_state (its column assembly, warp_solve6) with the pose's P66 held, and State::operator+= on R and p, written into
// the pose's ScanConst in place. Steps chain on the device: k_score, k_score_sum, k_refine_step, k_score, ...
//
// PoseScorer (lk_mapdev.h) is the host plan both calls run: the pose table, its tiles and windows, one packed H2D copy, the
// launches of every window, one read-back and one host synchronisation.
#include <algorithm>
#include <cstring>
#include <vector>

#include "lk_kernels.h"
#include "lk_mapdev.h"
#include "lk_pass.cuh"
#include "lk_solve.cuh"

namespace lk {

static_assert(LK_SCORE_A == 0 && LK_SCORE_B == ACC_B && LK_SCORE_SUM_R == ACC_SUMR && LK_SCORE_COUNT == ACC_CNT &&
                  LK_SCORE_SUM_Z2R == NACC && LK_SCORE_STRIDE == PARTIAL_STRIDE,
              "lk_score_poses record layout (include/legkilo_b200.h) = the partial-row layout");

constexpr uint32_t SCORE_CHUNK = 256;  // points per block: one per thread
constexpr uint32_t SCORE_TILE = 16;    // poses per block
// A call keeps at most this many partial rows (256 bytes each) in flight: poses past it run in the next window.
constexpr uint32_t SCORE_WINDOW_ROWS = 1u << 18;  // 64 MB
// One block of k_score: points [start, start + count) of one set against poses [pose0, pose0 + n_poses) of the pose table
// (consecutive poses of that set); pose pose0 + k writes partial row row0 + k * row_stride.
struct ScoreItem {
    uint32_t start, count, pose0, n_poses, row0, row_stride, pad[2];
};
// One block of k_score_sum: partial rows [row0, row0 + n_rows) summed into record `pose` of out.
struct ScoreSum {
    uint32_t row0, n_rows, pose, pad;
};
struct ScoreArgs {
    const float4* pts;
    const ScoreItem* items;
    uint32_t item_first;  // first item of this launch (grid.x = number of items)
    const ScoreSum* sums;
    uint32_t sum_first;
    const ScanConst* sc;  // one per pose, in the order the items address them
    double* partial;      // [rows of the window * PARTIAL_STRIDE]
    double* out;          // [n_poses * PARTIAL_STRIDE], by the caller's pose index
    MapView mv;
    Globals g;
};

namespace {

constexpr int BLOCK = SCORE_CHUNK;  // one point per thread per pass
constexpr int WARPS = BLOCK / 32;
constexpr int SUM_THREADS = 128;
constexpr int REFINE_THREADS = 128;  // four poses per block, one per warp

__global__ void __launch_bounds__(BLOCK, 1) k_score(const __grid_constant__ ScoreArgs a) {
    extern __shared__ __align__(16) unsigned char s_raw[];
    __shared__ ScanConst s_sc;
    __shared__ double s_slice[WARPS * 32];
    PassSmem<BLOCK, true>* ps = reinterpret_cast<PassSmem<BLOCK, true>*>(s_raw);
    const int tid = threadIdx.x;
    const ScoreItem it = a.items[a.item_first + blockIdx.x];
    pass_init(ps);
    LaneCache lc;
    lc.have = 0;
    const float4 pre = (uint32_t)tid < it.count ? __ldg(a.pts + it.start + tid) : make_float4(0.f, 0.f, 0.f, 0.f);
    uint32_t phase = 0;
    for (uint32_t k = 0; k < it.n_poses; ++k) {
        load_scan_const(&s_sc, a.sc + it.pose0 + k);
        __syncthreads();  // also: warp 0 of the previous pose has read s_slice
        double acc[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[i] = 0.0;
        points_pass<BLOCK, false, true>(ps, phase, it.count, s_sc, a.mv, a.g, lc, pre, [&](uint32_t, const Row& row) {
            accumulate_row(row, acc);
            acc[LK_SCORE_SUM_Z2R] += row.z * row.z / row.R;
        });
        double* dst = a.partial + (size_t)(it.row0 + k * it.row_stride) * PARTIAL_STRIDE;
        block_row<WARPS>(acc, s_slice, [&](int i, double v) { dst[i] = v; });
    }
}

__global__ void __launch_bounds__(SUM_THREADS) k_score_sum(const __grid_constant__ ScoreArgs a) {
    __shared__ double s_slice[(SUM_THREADS / 32) * 32];
    __shared__ double s_out[32];
    const ScoreSum ss = a.sums[a.sum_first + blockIdx.x];
    block_sum_partials<SUM_THREADS / 32>(a.partial, ss.row0, ss.row0 + ss.n_rows, s_slice, s_out);
    if (threadIdx.x < 32) a.out[(size_t)ss.pose * PARTIAL_STRIDE + threadIdx.x] = s_out[threadIdx.x];
}

// Entry (i, j) of P66 = blockdiag(Pth, Ppp) from the packed upper triangles (xx xy xz yy yz zz); the cross blocks are 0.
__device__ __forceinline__ double p66_entry(const ScanConst* sc, int i, int j) {
    if ((i < 3) != (j < 3)) return 0.0;
    const int o = i < 3 ? 0 : 3, r = min(i, j) - o, c = max(i, j) - o;
    return (i < 3 ? sc->Pth : sc->Ppp)[r * 3 - r * (r - 1) / 2 + (c - r)];
}

// One step of one pose per warp: ESKF::updateByPoints' K z (eskf.cc:91-113) restricted to the pose, with P66 held, in the
// information form of block_solve_state: y = (I + A P66)^-1 b from the pose's record (the sums at its current pose),
// delta = P66 y, then State::operator+= (eskf.cc:18-29): R <- R Exp(delta_theta), p <- p + delta_p, written back into the
// pose's ScanConst for the next k_score. A count of 0 leaves the pose untouched; a singular M gives a zero step, as in
// block_solve_state.
__global__ void __launch_bounds__(REFINE_THREADS) k_refine_step(const __grid_constant__ ScoreArgs a, ScanConst* sc, uint32_t n) {
    const int lane = threadIdx.x & 31;
    const uint32_t w = blockIdx.x * (REFINE_THREADS / 32) + (threadIdx.x >> 5);
    if (w >= n) return;  // warp-uniform
    const uint32_t pose = a.sum_first + w;
    const double* acc = a.out + (size_t)a.sums[pose].pose * PARTIAL_STRIDE;
    if (!(acc[ACC_CNT] > 0.5)) return;
    ScanConst* s = sc + pose;
    // N == 1 adds 1e-4 to S (eskf.cc:100)  <=>  weights scale by R / (R + 1e-4)
    const double scale = (acc[ACC_CNT] < 1.5) ? acc[ACC_SUMR] / (acc[ACC_SUMR] + 0.0001) : 1.0;
    // Pc: column `lane` of P66 (lanes 0..5), which is also its row: P66 is symmetric
    double Pc[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) Pc[k] = p66_entry(s, k, lane < 6 ? lane : 0);
    // columns of [M | b | A], M = I + A P66, one per lane (0..12), formed as block_solve_state forms them
    double col[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        double ar[6];
#pragma unroll
        for (int k = 0; k < 6; ++k) {
            const int r = i < k ? i : k, c = i < k ? k : i;
            ar[k] = acc[r * 6 - r * (r - 1) / 2 + (c - r)] * scale;
        }
        double m = (i == lane) ? 1.0 : 0.0;
#pragma unroll
        for (int k = 0; k < 6; ++k) m += ar[k] * Pc[k];
        double asel = ar[0];
#pragma unroll
        for (int t = 1; t < 6; ++t) asel = (lane - 7 == t) ? ar[t] : asel;
        const double bsel = acc[ACC_B + i] * scale;
        col[i] = lane < 6 ? m : (lane == 6 ? bsel : (lane < 13 ? asel : 0.0));
    }
    const bool ok = warp_solve6(col, lane);
    double d = 0.0;
#pragma unroll
    for (int k = 0; k < 6; ++k) d += Pc[k] * __shfl_sync(0xffffffffu, ok ? col[k] : 0.0, 6);
    const double d0 = __shfl_sync(0xffffffffu, d, 0), d1 = __shfl_sync(0xffffffffu, d, 1),
                 d2 = __shfl_sync(0xffffffffu, d, 2);
    const double dp = __shfl_sync(0xffffffffu, d, (lane + 26) & 31);  // lanes 9..11: delta_p from lanes 3..5
    double rv = 0.0;
    if (lane < 9) {
        double E[9];
        so3_exp3(d0, d1, d2, E);
        // column j of E picked with compile-time indices (E indexed at run time would live in local memory)
        const int i = lane / 3, j = lane % 3;
        const double e0 = j == 0 ? E[0] : (j == 1 ? E[1] : E[2]);
        const double e1 = j == 0 ? E[3] : (j == 1 ? E[4] : E[5]);
        const double e2 = j == 0 ? E[6] : (j == 1 ? E[7] : E[8]);
        rv = s->R[i * 3] * e0 + s->R[i * 3 + 1] * e1 + s->R[i * 3 + 2] * e2;
    }
    __syncwarp();
    if (lane < 9) s->R[lane] = rv;
    else if (lane < 12) s->p[lane - 9] += dp;
}

}  // namespace

void launch_score(const ScoreArgs& a, uint32_t n_items, uint32_t n_sums, cudaStream_t s) {
    static PerDeviceOnce once;
    const size_t smem = sizeof(PassSmem<BLOCK, true>);
    if (once.first()) cudaFuncSetAttribute(k_score, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (n_items) k_score<<<n_items, BLOCK, smem, s>>>(a);
    if (n_sums) k_score_sum<<<n_sums, SUM_THREADS, 0, s>>>(a);
}

// One pose step (k_refine_step) for poses [sum_first, sum_first + n_sums) of the pose table, from the records a.out holds
// at their current poses; the new R / p are written into sc, the same buffer as a.sc.
void launch_refine_step(const ScoreArgs& a, ScanConst* sc, uint32_t n_sums, cudaStream_t s) {
    constexpr uint32_t per_block = REFINE_THREADS / 32;
    if (n_sums) k_refine_step<<<(n_sums + per_block - 1) / per_block, REFINE_THREADS, 0, s>>>(a, sc, n_sums);
}

int PoseScorer::run(const MapDevHost& mh, const Globals& g, uint32_t n_sets, const float* pts, const uint32_t* set_offsets,
                    uint32_t n_poses, const uint32_t* pose_set, const double* rot, const double* pos, const double* rot_cov,
                    const double* pos_cov, int iters, double* rot_out, double* pos_out, double* sums_out, cudaStream_t st,
                    std::string& err) {
    // The pose table in set order (ord: the caller's pose index of each entry, the caller's order within a set), cut into
    // tiles of consecutive poses of one set, and the tiles into windows of at most SCORE_WINDOW_ROWS partial rows (or one
    // tile); window w is items [win_items[w], win_items[w + 1]) and pose-table entries [win_sums[w], win_sums[w + 1]). Item
    // order: tile-major, so the blocks in flight together score one set at neighbouring poses, and touch neighbouring voxels.
    auto n_chunks = [&](uint32_t s) { return (set_offsets[s + 1] - set_offsets[s] + SCORE_CHUNK - 1) / SCORE_CHUNK; };
    std::vector<uint32_t> first(n_sets + 1, 0), ord(n_poses, 0);
    for (uint32_t m = 0; m < n_poses; ++m) ++first[pose_set[m] + 1];
    for (uint32_t s = 0; s < n_sets; ++s) first[s + 1] += first[s];
    {
        std::vector<uint32_t> fill(first.begin(), first.end() - 1);
        for (uint32_t m = 0; m < n_poses; ++m) ord[fill[pose_set[m]]++] = m;
    }
    std::vector<ScoreItem> items;
    std::vector<ScoreSum> sums(n_poses);
    std::vector<uint32_t> win_items(1, 0), win_sums(1, 0);
    uint32_t rows = 0;
    for (uint32_t s = 0; s < n_sets; ++s) {
        const uint32_t nc = n_chunks(s);
        const uint32_t tile = std::max<uint32_t>(1, std::min<uint32_t>(SCORE_TILE, nc ? SCORE_WINDOW_ROWS / nc : SCORE_TILE));
        for (uint32_t p0 = first[s]; p0 < first[s + 1]; p0 += tile) {
            const uint32_t np = std::min(tile, first[s + 1] - p0);
            if (rows > 0 && (uint64_t)rows + (uint64_t)np * nc > SCORE_WINDOW_ROWS) {
                win_items.push_back((uint32_t)items.size());
                win_sums.push_back(p0);
                rows = 0;
            }
            for (uint32_t c = 0; c < nc; ++c) {
                ScoreItem it;
                it.start = set_offsets[s] - set_offsets[0] + c * SCORE_CHUNK;
                it.count = std::min(SCORE_CHUNK, set_offsets[s + 1] - set_offsets[s] - c * SCORE_CHUNK);
                it.pose0 = p0;
                it.n_poses = np;
                it.row0 = rows + c;
                it.row_stride = nc;
                it.pad[0] = it.pad[1] = 0;
                items.push_back(it);
            }
            for (uint32_t k = 0; k < np; ++k) sums[p0 + k] = ScoreSum{rows + k * nc, nc, ord[p0 + k], 0};
            rows += np * nc;
        }
    }
    win_items.push_back((uint32_t)items.size());
    win_sums.push_back(n_poses);
    uint32_t max_rows = 0;
    for (size_t w = 0; w + 1 < win_sums.size(); ++w)
        for (uint32_t p = win_sums[w]; p < win_sums[w + 1]; ++p) max_rows = std::max(max_rows, sums[p].row0 + sums[p].n_rows);

    // One packed block, items | sums | ScanConst per pose (pose-table order), and one H2D copy. The staging block h_ then
    // receives the read-back: the ScanConst of every pose if rot_out is set, then the records if sums_out is.
    const size_t o_sums = align256(std::max<size_t>(items.size(), 1) * sizeof(ScoreItem));
    const size_t o_sc = o_sums + align256((size_t)n_poses * sizeof(ScoreSum));
    const size_t sc_bytes = (size_t)n_poses * sizeof(ScanConst), small_bytes = o_sc + sc_bytes;
    const size_t out_bytes = (size_t)n_poses * PARTIAL_STRIDE * 8;
    const size_t o_rec = rot_out ? align256(sc_bytes) : 0, back_bytes = o_rec + (sums_out ? out_bytes : 0);
    const uint64_t n_pts = (uint64_t)set_offsets[n_sets] - set_offsets[0];
    LK_CUDA(err, pts_.ensure(std::max<uint64_t>(n_pts, 1) * 16));
    LK_CUDA(err, small_.ensure(small_bytes));
    LK_CUDA(err, partial_.ensure((size_t)std::max<uint32_t>(max_rows, 1) * PARTIAL_STRIDE * 8));
    LK_CUDA(err, out_.ensure(out_bytes));
    LK_CUDA(err, h_.ensure(std::max(small_bytes, back_bytes)));
    char* hb = (char*)h_.p;
    std::memcpy(hb, items.data(), items.size() * sizeof(ScoreItem));
    std::memcpy(hb + o_sums, sums.data(), (size_t)n_poses * sizeof(ScoreSum));
    ScanConst* hs = reinterpret_cast<ScanConst*>(hb + o_sc);
    for (uint32_t p = 0; p < n_poses; ++p) scan_const_at(rot + 9 * (size_t)ord[p], pos + 3 * (size_t)ord[p], rot_cov, pos_cov, hs[p]);
    if (n_pts) LK_CUDA(err, cudaMemcpyAsync(pts_.p, pts + 4 * (size_t)set_offsets[0], n_pts * 16, cudaMemcpyHostToDevice, st));
    LK_CUDA(err, cudaMemcpyAsync(small_.p, hb, small_bytes, cudaMemcpyHostToDevice, st));

    // the pose constants the items read are stepped in place: k_score takes them const, k_refine_step writable
    ScanConst* sc = reinterpret_cast<ScanConst*>((char*)small_.p + o_sc);
    ScoreArgs a;
    std::memset(&a, 0, sizeof(a));
    a.pts = pts_.as<float4>();
    a.items = small_.as<ScoreItem>();
    a.sums = reinterpret_cast<const ScoreSum*>((char*)small_.p + o_sums);
    a.sc = sc;
    a.partial = partial_.as<double>();
    a.out = out_.as<double>();
    a.mv = mh.view();
    a.g = g;
    // window by window, every step of its poses, then (with sums_out) their records at the final poses; the windows reuse
    // the partial rows in stream order, and no launch waits for the host
    for (size_t w = 0; w + 1 < win_items.size(); ++w) {
        a.item_first = win_items[w];
        a.sum_first = win_sums[w];
        const uint32_t n_items = win_items[w + 1] - win_items[w], n_sums = win_sums[w + 1] - win_sums[w];
        for (int it = 0; it < iters; ++it) {
            launch_score(a, n_items, n_sums, st);
            launch_refine_step(a, sc, n_sums, st);
        }
        if (sums_out) launch_score(a, n_items, n_sums, st);
        LK_CUDA(err, cudaGetLastError());
    }
    // the one host synchronisation: the staging block is reused only after its H2D copy (same stream)
    if (rot_out) LK_CUDA(err, cudaMemcpyAsync(hb, sc, sc_bytes, cudaMemcpyDeviceToHost, st));
    if (sums_out) LK_CUDA(err, cudaMemcpyAsync(hb + o_rec, out_.p, out_bytes, cudaMemcpyDeviceToHost, st));
    LK_CUDA(err, cudaStreamSynchronize(st));
    LK_CUDA(err, cudaGetLastError());
    if (rot_out) {
        const ScanConst* hr = reinterpret_cast<const ScanConst*>(hb);
        for (uint32_t p = 0; p < n_poses; ++p) {
            std::memcpy(rot_out + 9 * (size_t)ord[p], hr[p].R, sizeof(hr[p].R));
            std::memcpy(pos_out + 3 * (size_t)ord[p], hr[p].p, sizeof(hr[p].p));
        }
    }
    if (sums_out) std::memcpy(sums_out, hb + o_rec, out_bytes);
    return LK_OK;
}

}  // namespace lk
