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
// lk_search_poses: the candidates of a pose lattice per set, generated on the device window by window (k_search_expand),
// scored by k_score / k_score_sum and merged into each set's running best k (k_search_keep); then the kept poses gathered
// (k_search_gather), refined, re-scored with the tight blocks (k_search_tight) and ranked (k_search_rank).
//
// PoseScorer (lk_mapdev.h) is the host side of the three calls: one plan (plan_windows: tiles and windows from the sets'
// sizes and pose counts), its items formed on the host (host_plan) or on the device (the search's windows), its windows
// run over a ScanConst block already on the device (run_windows), one packed H2D copy, one read-back and one host
// synchronisation.
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

// Item c (chunk c of the set) of a tile: poses [pose0, pose0 + n_poses) of the pose table against chunk c of the set's
// points [pt_start, pt_start + pt_count); pose pose0 + j writes partial row row0 + j * nc + c. The plan of every call forms
// its items so, on the host (lk_score_poses, lk_refine_poses) or on the device (k_search_expand).
__host__ __device__ inline ScoreItem tile_item(uint32_t pt_start, uint32_t pt_count, uint32_t nc, uint32_t pose0,
                                               uint32_t n_poses, uint32_t row0, uint32_t c) {
    ScoreItem it;
    it.start = pt_start + c * SCORE_CHUNK;
    it.count = pt_count - c * SCORE_CHUNK < SCORE_CHUNK ? pt_count - c * SCORE_CHUNK : SCORE_CHUNK;
    it.pose0 = pose0;
    it.n_poses = n_poses;
    it.row0 = row0 + c;
    it.row_stride = nc;
    it.pad[0] = it.pad[1] = 0;
    return it;
}

// lk_search_poses. One per set: the totals of the plan's walk (plan_windows, without windows) before the set, its points
// and chunk count, its tile, its attitudes (att0: the first, relative to att_offsets[0]), its candidates and lattice origin.
struct SearchSet {
    uint64_t poses0, rows0, items0;
    uint32_t pt_start, pt_count, nc, tile, att0, n_cand;
    double origin[3];
};
// One candidate window: candidates [first0, ...) of set0 through [..., end1) of set1; poses0 / rows0 / items0 are the
// walk's totals before it, so the window-local index of anything is its walk index minus these.
struct SearchWindow {
    uint32_t set0, set1, first0, end1, n_poses, n_items;
    uint64_t poses0, rows0, items0;
};
struct SearchLattice {
    uint32_t n[3], pad;
    double step[3];
};
// Per kept pose of the read-back: R (9) | p (3) | record (PARTIAL_STRIDE), doubles.
constexpr int SEARCH_RESULT = 12 + PARTIAL_STRIDE;
struct SearchArgs {
    const SearchSet* sets;
    const double* att;  // row-major 3 x 3 per attitude
    SearchLattice lat;
    ScanConst wide, tight;  // R, p unused: the symmetrised blocks as scan_const_at forms them
    ScanConst* win_sc;      // one window's candidates
    ScoreSum* win_sums;
    ScoreItem* win_items;
    const double* out;  // the records (by ScoreSum::pose)
    uint64_t* best;     // k keys per set, ascending (keep_key)
    uint32_t k;
};

namespace {

constexpr int BLOCK = SCORE_CHUNK;  // one point per thread per pass
constexpr int WARPS = BLOCK / 32;
constexpr int SUM_THREADS = 128;
constexpr int REFINE_THREADS = 128;  // four poses per block, one per warp
constexpr int EXPAND_THREADS = 256;
constexpr int KEEP_THREADS = 1024;  // candidates a keep step sorts

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

// ---- lk_search_poses ----------------------------------------------------------------------------------------------------

// Candidate c of a set with nx * ny * nz lattice positions: attitude a = c / L of the set, position (ix, iy, iz) of
// r = c % L with ix fastest; pos[j] = origin[j] + i_j * step[j], the product rounded, then the sum (no FMA).
__device__ __forceinline__ void lattice_pose(const SearchSet& ss, const double* att, const SearchLattice& l, uint32_t c,
                                             ScanConst& sc) {
    const uint32_t L = l.n[0] * l.n[1] * l.n[2], a = c / L, r = c % L;
    const uint32_t i[3] = {r % l.n[0], (r / l.n[0]) % l.n[1], r / (l.n[0] * l.n[1])};
    const double* R = att + 9 * (size_t)(ss.att0 + a);
#pragma unroll
    for (int q = 0; q < 9; ++q) sc.R[q] = R[q];
#pragma unroll
    for (int j = 0; j < 3; ++j) sc.p[j] = __dadd_rn(ss.origin[j], __dmul_rn((double)i[j], l.step[j]));
}

// The set of window-local pose q / item q: the last set of the window whose first pose (item) in the walk is <= base + q.
template <class First>
__device__ __forceinline__ uint32_t window_set(const SearchWindow& w, uint64_t g, First first) {
    uint32_t lo = w.set0, hi = w.set1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) / 2;
        if (first(mid) <= g) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// One window of the search: the ScanConst and ScoreSum of each candidate in it and its ScoreItems, exactly what the plan
// of lk_score_poses forms for those poses (tile_item, the window's partial rows from 0).
__global__ void __launch_bounds__(EXPAND_THREADS) k_search_expand(const __grid_constant__ SearchArgs a, SearchWindow w) {
    const uint32_t n = max(w.n_poses, w.n_items);
    for (uint32_t q = blockIdx.x * EXPAND_THREADS + threadIdx.x; q < n; q += gridDim.x * EXPAND_THREADS) {
        if (q < w.n_poses) {
            const uint64_t gq = w.poses0 + q;
            const uint32_t s = window_set(w, gq, [&](uint32_t t) { return a.sets[t].poses0; });
            const SearchSet& ss = a.sets[s];
            const uint32_t c = (uint32_t)(gq - ss.poses0);
            ScanConst sc = a.wide;
            lattice_pose(ss, a.att, a.lat, c, sc);
            a.win_sc[q] = sc;
            a.win_sums[q] = ScoreSum{(uint32_t)(ss.rows0 + (uint64_t)c * ss.nc - w.rows0), ss.nc, q, 0};
        }
        if (q < w.n_items) {
            const uint64_t gi = w.items0 + q;
            const uint32_t s = window_set(w, gi, [&](uint32_t t) { return a.sets[t].items0; });
            const SearchSet& ss = a.sets[s];
            const uint64_t li = gi - ss.items0;  // a set's items may pass 2^32, its candidates do not
            const uint32_t ct = (uint32_t)(li / ss.nc) * ss.tile;
            a.win_items[q] = tile_item(ss.pt_start, ss.pt_count, ss.nc, (uint32_t)(ss.poses0 + ct - w.poses0),
                                       min(ss.tile, ss.n_cand - ct), (uint32_t)(ss.rows0 + (uint64_t)ct * ss.nc - w.rows0),
                                       (uint32_t)(li % ss.nc));
        }
    }
}

// Ascending bitonic sort of N keys in shared memory by the block's first N threads (every thread of the block calls it).
template <int N>
__device__ __forceinline__ void block_sort(uint64_t* s) {
    const int tid = threadIdx.x;
    __syncthreads();
#pragma unroll 1
    for (int kk = 2; kk <= N; kk <<= 1)
#pragma unroll 1
        for (int j = kk >> 1; j > 0; j >>= 1) {
            const int o = tid ^ j;
            if (tid < N && o > tid) {
                const uint64_t x = s[tid], y = s[o];
                if ((x > y) == ((tid & kk) == 0)) s[tid] = y, s[o] = x;
            }
            __syncthreads();
        }
}

// Number of keys of sorted s[0, n) below x (upper: at most x).
template <bool UPPER>
__device__ __forceinline__ uint32_t rank_in(const uint64_t* s, uint32_t n, uint64_t x) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) / 2;
        if (UPPER ? s[mid] <= x : s[mid] < x) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// The key of a candidate: count descending, then candidate index ascending, as one ascending 64-bit key.
__device__ __forceinline__ uint64_t keep_key(double count, uint32_t c) {
    return ((uint64_t)(0xffffffffu - (uint32_t)count) << 32) | c;
}

// After one window's records: one block per set of the window merges the set's candidates in it into its running best k
// (sorted keys, best[k s ..]). KEEP_THREADS candidates at a time: those better than the running k-th are sorted and the
// first k merged with the running list (a stable merge: each key's place is its index plus its rank in the other list).
__global__ void __launch_bounds__(KEEP_THREADS) k_search_keep(const __grid_constant__ SearchArgs a, SearchWindow w) {
    __shared__ uint64_t s_key[KEEP_THREADS];
    __shared__ uint64_t s_best[LK_SEARCH_MAX_K], s_next[LK_SEARCH_MAX_K];
    const uint32_t tid = threadIdx.x, k = a.k, s = w.set0 + blockIdx.x;
    const SearchSet ss = a.sets[s];
    const uint32_t c_lo = s == w.set0 ? w.first0 : 0, c_hi = s == w.set1 ? w.end1 : ss.n_cand;
    if (tid < k) s_best[tid] = a.best[(size_t)s * k + tid];
    __syncthreads();
    for (uint64_t c0 = c_lo; c0 < c_hi; c0 += KEEP_THREADS) {
        const uint64_t worst = s_best[k - 1], c = c0 + tid;
        uint64_t key = ~0ull;
        if (c < c_hi) {
            key = keep_key(a.out[(ss.poses0 + c - w.poses0) * PARTIAL_STRIDE + ACC_CNT], (uint32_t)c);
            if (key >= worst) key = ~0ull;
        }
        if (!__syncthreads_or(key != ~0ull)) continue;
        s_key[tid] = key;
        block_sort<KEEP_THREADS>(s_key);
        if (tid < k) {
            const uint64_t x = s_best[tid];
            const uint32_t p = tid + rank_in<false>(s_key, k, x);
            if (p < k) s_next[p] = x;
        } else if (tid < 2 * k) {
            const uint64_t x = s_key[tid - k];
            const uint32_t p = tid - k + rank_in<true>(s_best, k, x);
            if (p < k) s_next[p] = x;
        }
        __syncthreads();
        if (tid < k) s_best[tid] = s_next[tid];
        __syncthreads();
    }
    if (tid < k) a.best[(size_t)s * k + tid] = s_best[tid];
}

// Kept pose g = k s + j (pose-table entry g of the refinement plan): candidate best[g] of set s at the wide blocks.
__global__ void __launch_bounds__(EXPAND_THREADS) k_search_gather(const __grid_constant__ SearchArgs a, ScanConst* sc,
                                                                  uint32_t n) {
    const uint32_t g = blockIdx.x * EXPAND_THREADS + threadIdx.x;
    if (g >= n) return;
    ScanConst t = a.wide;
    lattice_pose(a.sets[g / a.k], a.att, a.lat, (uint32_t)a.best[g], t);
    sc[g] = t;
}

// The tight blocks into every kept pose, its refined R and p kept.
__global__ void __launch_bounds__(EXPAND_THREADS) k_search_tight(const __grid_constant__ SearchArgs a, ScanConst* sc,
                                                                 uint32_t n) {
    const uint32_t g = blockIdx.x * EXPAND_THREADS + threadIdx.x;
    if (g >= n) return;
#pragma unroll
    for (int q = 0; q < 6; ++q) sc[g].Pth[q] = a.tight.Pth[q], sc[g].Ppp[q] = a.tight.Ppp[q];
}

// One block per set: its k kept poses ordered by (tight count descending, keep rank ascending), written as the call's
// outputs: rot (9) | pos (3) | record (PARTIAL_STRIDE) per entry, then the candidate indices.
__global__ void __launch_bounds__(LK_SEARCH_MAX_K) k_search_rank(const __grid_constant__ SearchArgs a, const ScanConst* sc,
                                                                 double* res, uint32_t n_sets) {
    __shared__ uint64_t s_key[LK_SEARCH_MAX_K];
    const uint32_t tid = threadIdx.x, k = a.k, s = blockIdx.x;
    const size_t g0 = (size_t)s * k;
    s_key[tid] = tid < k ? keep_key(a.out[(g0 + tid) * PARTIAL_STRIDE + ACC_CNT], tid) : ~0ull;
    block_sort<LK_SEARCH_MAX_K>(s_key);
    if (tid >= k) return;
    const size_t src = g0 + (uint32_t)s_key[tid], dst = g0 + tid;
    double* o = res + dst * SEARCH_RESULT;
#pragma unroll
    for (int q = 0; q < 9; ++q) o[q] = sc[src].R[q];
#pragma unroll
    for (int q = 0; q < 3; ++q) o[9 + q] = sc[src].p[q];
    for (int q = 0; q < PARTIAL_STRIDE; ++q) o[12 + q] = a.out[src * PARTIAL_STRIDE + q];
    reinterpret_cast<uint32_t*>(res + (size_t)n_sets * k * SEARCH_RESULT)[dst] = (uint32_t)a.best[src];
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

// ---- the plan: tiles and windows -----------------------------------------------------------------------------------------

namespace {

uint32_t n_chunks(const uint32_t* set_offsets, uint32_t s) {
    return (set_offsets[s + 1] - set_offsets[s] + SCORE_CHUNK - 1) / SCORE_CHUNK;
}

// Poses of a set per tile: up to SCORE_TILE, fewer when that many would not fit a window (a set of more than
// SCORE_WINDOW_ROWS chunks: one pose per tile, alone in its window).
uint32_t score_tile(uint32_t nc) {
    return std::max<uint32_t>(1, std::min<uint32_t>(SCORE_TILE, nc ? SCORE_WINDOW_ROWS / nc : SCORE_TILE));
}

// A run of consecutive poses of one set inside one window: poses [first, first + n) of set `set` (in the set's pose order)
// are the window's poses [pose0, pose0 + n), their partial rows start at row0 and their items at item0 (window-local).
struct ScoreRun {
    uint32_t set;
    uint64_t first;
    uint32_t n, pose0, row0, item0;
};

// The plan of a call, a function of the sets' sizes and pose counts only: set after set, its poses (n_poses(s) of them, in
// order) cut into tiles (score_tile) and the tiles into windows of at most SCORE_WINDOW_ROWS partial rows and as many
// poses (or one tile). A tile of np poses of a set of nc chunks is nc items (tile_item) and np * nc partial rows: pose j of
// the tile writes rows row0 + j * nc + c. run(r) for each run, window(rows, poses, items) at the end of each window.
template <class NPoses, class Run, class Window>
void plan_windows(uint32_t n_sets, const uint32_t* set_offsets, NPoses n_poses, Run run, Window window) {
    uint32_t rows = 0, poses = 0, items = 0;
    for (uint32_t s = 0; s < n_sets; ++s) {
        const uint32_t nc = n_chunks(set_offsets, s), tile = score_tile(nc);
        const uint64_t N = n_poses(s);
        for (uint64_t done = 0; done < N;) {
            const uint32_t np = (uint32_t)std::min<uint64_t>(tile, N - done);
            if (poses > 0 && ((uint64_t)rows + (uint64_t)np * nc > SCORE_WINDOW_ROWS || poses + np > SCORE_WINDOW_ROWS)) {
                window(rows, poses, items);
                rows = poses = items = 0;
            }
            // as many whole tiles as fit beside what the window holds, at least one
            uint64_t fit = (SCORE_WINDOW_ROWS - poses) / tile;
            if (nc) fit = std::min<uint64_t>(fit, (SCORE_WINDOW_ROWS - std::min<uint32_t>(rows, SCORE_WINDOW_ROWS)) /
                                                      ((uint64_t)tile * nc));
            const uint32_t n = (uint32_t)std::min<uint64_t>(N - done, std::max<uint64_t>(fit, 1) * tile);
            run(ScoreRun{s, done, n, poses, rows, items});
            rows += n * nc;
            poses += n;
            items += (n + tile - 1) / tile * nc;
            done += n;
        }
    }
    if (poses > 0) window(rows, poses, items);
}

}  // namespace

// lk_score_poses / lk_refine_poses: the plan expanded on the host over the pose table in set order (ord: the caller's
// pose index of each entry, the caller's order within a set). Window w is items [win_items[w], win_items[w + 1]) and
// pose-table entries [win_sums[w], win_sums[w + 1]); returns the most partial rows a window holds. Item order: tile-major,
// so the blocks in flight together score one set at neighbouring poses, and touch neighbouring voxels.
static uint32_t host_plan(uint32_t n_sets, const uint32_t* set_offsets, const uint32_t* first, const uint32_t* ord,
                          std::vector<ScoreItem>& items, std::vector<ScoreSum>& sums, std::vector<uint32_t>& win_items,
                          std::vector<uint32_t>& win_sums) {
    uint32_t max_rows = 0, n_poses = first[n_sets];
    items.clear();
    sums.assign(n_poses, ScoreSum{0, 0, 0, 0});
    win_items.assign(1, 0);
    win_sums.assign(1, 0);
    uint32_t seen = 0;
    plan_windows(
        n_sets, set_offsets, [&](uint32_t s) { return (uint64_t)(first[s + 1] - first[s]); },
        [&](const ScoreRun& r) {
            const uint32_t nc = n_chunks(set_offsets, r.set), tile = score_tile(nc), p0 = first[r.set] + (uint32_t)r.first;
            const uint32_t pt = set_offsets[r.set] - set_offsets[0], cnt = set_offsets[r.set + 1] - set_offsets[r.set];
            for (uint32_t t = 0; t * tile < r.n; ++t)
                for (uint32_t c = 0; c < nc; ++c)
                    items.push_back(tile_item(pt, cnt, nc, p0 + t * tile, std::min(tile, r.n - t * tile), r.row0 + t * tile * nc, c));
            for (uint32_t j = 0; j < r.n; ++j) sums[p0 + j] = ScoreSum{r.row0 + j * nc, nc, ord[p0 + j], 0};
            seen = p0 + r.n;
        },
        [&](uint32_t rows, uint32_t, uint32_t) {
            win_items.push_back((uint32_t)items.size());
            win_sums.push_back(seen);
            max_rows = std::max(max_rows, rows);
        });
    return max_rows;
}

// Every window of a host plan: iters steps of each of its poses, then (score) their records at the final poses; the
// windows reuse the partial rows in stream order, and no launch waits for the host.
static void run_windows(ScoreArgs a, const std::vector<uint32_t>& win_items, const std::vector<uint32_t>& win_sums,
                        ScanConst* sc, int iters, bool score, cudaStream_t st) {
    for (size_t w = 0; w + 1 < win_items.size(); ++w) {
        a.item_first = win_items[w];
        a.sum_first = win_sums[w];
        const uint32_t n_items = win_items[w + 1] - win_items[w], n_sums = win_sums[w + 1] - win_sums[w];
        for (int it = 0; it < iters; ++it) {
            launch_score(a, n_items, n_sums, st);
            launch_refine_step(a, sc, n_sums, st);
        }
        if (score) launch_score(a, n_items, n_sums, st);
    }
}

int PoseScorer::run(const MapDevHost& mh, const Globals& g, uint32_t n_sets, const float* pts, const uint32_t* set_offsets,
                    uint32_t n_poses, const uint32_t* pose_set, const double* rot, const double* pos, const double* rot_cov,
                    const double* pos_cov, int iters, double* rot_out, double* pos_out, double* sums_out, cudaStream_t st,
                    std::string& err) {
    std::vector<uint32_t> first(n_sets + 1, 0), ord(n_poses, 0);
    for (uint32_t m = 0; m < n_poses; ++m) ++first[pose_set[m] + 1];
    for (uint32_t s = 0; s < n_sets; ++s) first[s + 1] += first[s];
    {
        std::vector<uint32_t> fill(first.begin(), first.end() - 1);
        for (uint32_t m = 0; m < n_poses; ++m) ord[fill[pose_set[m]]++] = m;
    }
    std::vector<ScoreItem> items;
    std::vector<ScoreSum> sums;
    std::vector<uint32_t> win_items, win_sums;
    const uint32_t max_rows = host_plan(n_sets, set_offsets, first.data(), ord.data(), items, sums, win_items, win_sums);

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
    run_windows(a, win_items, win_sums, sc, iters, sums_out != nullptr, st);
    LK_CUDA(err, cudaGetLastError());
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

int PoseScorer::search(const MapDevHost& mh, const Globals& g, uint32_t n_sets, const float* pts, const uint32_t* set_offsets,
                       const uint32_t* att_offsets, const double* att_rot, const double* origin, const double* step,
                       const uint32_t* counts, const double* rot_cov, const double* pos_cov, int iters,
                       const double* rot_cov_tight, const double* pos_cov_tight, uint32_t k, double* rot_out,
                       double* pos_out, double* sums_out, uint32_t* cand_out, cudaStream_t st, std::string& err) {
    const uint32_t L = counts[0] * counts[1] * counts[2];  // < 2^32: checked by the caller
    auto n_cand = [&](uint32_t s) { return (uint64_t)(att_offsets[s + 1] - att_offsets[s]) * L; };

    // The per-set table: the walk's totals before each set (without windows), its points, tile and attitudes.
    std::vector<SearchSet> sets(n_sets);
    uint64_t poses = 0, rows = 0, items = 0;
    for (uint32_t s = 0; s < n_sets; ++s) {
        SearchSet& t = sets[s];
        std::memset(&t, 0, sizeof(t));
        t.poses0 = poses, t.rows0 = rows, t.items0 = items;
        t.pt_start = set_offsets[s] - set_offsets[0];
        t.pt_count = set_offsets[s + 1] - set_offsets[s];
        t.nc = n_chunks(set_offsets, s);
        t.tile = score_tile(t.nc);
        t.att0 = att_offsets[s] - att_offsets[0];
        t.n_cand = (uint32_t)n_cand(s);
        for (int j = 0; j < 3; ++j) t.origin[j] = origin[3 * (size_t)s + j];
        poses += t.n_cand;
        rows += (uint64_t)t.n_cand * t.nc;
        items += ((uint64_t)t.n_cand + t.tile - 1) / t.tile * t.nc;
    }
    // The candidate windows, from the same walk as every other call's plan: each window's first set and candidate, its
    // last set and end, and its totals. max_*: what the largest window needs.
    std::vector<SearchWindow> wins;
    SearchWindow cur;
    std::memset(&cur, 0, sizeof(cur));
    bool open = false;
    uint32_t max_poses = 0, max_items = 0, max_rows = 0;
    plan_windows(
        n_sets, set_offsets, n_cand,
        [&](const ScoreRun& r) {
            if (!open) {
                const SearchSet& t = sets[r.set];
                cur.set0 = r.set;
                cur.first0 = (uint32_t)r.first;
                cur.poses0 = t.poses0 + r.first;
                cur.rows0 = t.rows0 + r.first * t.nc;
                cur.items0 = t.items0 + r.first / t.tile * t.nc;
                open = true;
            }
            cur.set1 = r.set;
            cur.end1 = (uint32_t)(r.first + r.n);
        },
        [&](uint32_t rows_w, uint32_t poses_w, uint32_t items_w) {
            cur.n_poses = poses_w, cur.n_items = items_w;
            wins.push_back(cur);
            open = false;
            max_poses = std::max(max_poses, poses_w), max_items = std::max(max_items, items_w);
            max_rows = std::max(max_rows, rows_w);
        });

    // The kept poses' plan: k per set, in set order (pose-table entry k s + j is rank j of set s's keep).
    const uint32_t n_keep = n_sets * k;
    std::vector<uint32_t> first(n_sets + 1), ord(n_keep);
    for (uint32_t s = 0; s <= n_sets; ++s) first[s] = s * k;
    for (uint32_t m = 0; m < n_keep; ++m) ord[m] = m;
    std::vector<ScoreItem> kitems;
    std::vector<ScoreSum> ksums;
    std::vector<uint32_t> win_items, win_sums;
    max_rows = std::max(max_rows, host_plan(n_sets, set_offsets, first.data(), ord.data(), kitems, ksums, win_items, win_sums));

    // Device: sets_ = SearchSet per set | attitudes; win_ = ScanConst | ScoreSum per window pose | ScoreItem per window item;
    // small_ = the kept poses' items | sums | ScanConst | ranked results; best_ = k keys per set.
    const uint32_t n_att = att_offsets[n_sets] - att_offsets[0];
    const size_t o_att = align256((size_t)n_sets * sizeof(SearchSet)), sets_bytes = o_att + (size_t)n_att * 72;
    const size_t o_wsum = align256((size_t)max_poses * sizeof(ScanConst));
    const size_t o_witem = o_wsum + align256((size_t)max_poses * sizeof(ScoreSum));
    const size_t win_bytes = o_witem + (size_t)std::max<uint32_t>(max_items, 1) * sizeof(ScoreItem);
    const size_t o_sums = align256(std::max<size_t>(kitems.size(), 1) * sizeof(ScoreItem));
    const size_t o_sc = o_sums + align256((size_t)n_keep * sizeof(ScoreSum));
    const size_t o_res = o_sc + align256((size_t)n_keep * sizeof(ScanConst));
    const size_t res_bytes = (size_t)n_keep * (SEARCH_RESULT * 8 + 4), small_bytes = o_res + res_bytes;
    const size_t plan_bytes = o_sc;  // what the host stages of small_
    const uint64_t n_pts = (uint64_t)set_offsets[n_sets] - set_offsets[0];
    LK_CUDA(err, pts_.ensure(std::max<uint64_t>(n_pts, 1) * 16));
    LK_CUDA(err, sets_.ensure(sets_bytes));
    LK_CUDA(err, win_.ensure(win_bytes));
    LK_CUDA(err, small_.ensure(small_bytes));
    LK_CUDA(err, partial_.ensure((size_t)std::max<uint32_t>(max_rows, 1) * PARTIAL_STRIDE * 8));
    LK_CUDA(err, out_.ensure((size_t)std::max(max_poses, n_keep) * PARTIAL_STRIDE * 8));
    LK_CUDA(err, best_.ensure((size_t)n_keep * 8));
    const size_t o_hplan = align256(sets_bytes);
    LK_CUDA(err, h_.ensure(std::max(o_hplan + plan_bytes, res_bytes)));
    char* hb = (char*)h_.p;
    std::memcpy(hb, sets.data(), (size_t)n_sets * sizeof(SearchSet));
    std::memcpy(hb + o_att, att_rot + 9 * (size_t)att_offsets[0], (size_t)n_att * 72);
    std::memcpy(hb + o_hplan, kitems.data(), kitems.size() * sizeof(ScoreItem));
    std::memcpy(hb + o_hplan + o_sums, ksums.data(), (size_t)n_keep * sizeof(ScoreSum));
    if (n_pts) LK_CUDA(err, cudaMemcpyAsync(pts_.p, pts + 4 * (size_t)set_offsets[0], n_pts * 16, cudaMemcpyHostToDevice, st));
    LK_CUDA(err, cudaMemcpyAsync(sets_.p, hb, sets_bytes, cudaMemcpyHostToDevice, st));
    LK_CUDA(err, cudaMemcpyAsync(small_.p, hb + o_hplan, plan_bytes, cudaMemcpyHostToDevice, st));
    LK_CUDA(err, cudaMemsetAsync(best_.p, 0xff, (size_t)n_keep * 8, st));

    SearchArgs sa;
    std::memset(&sa, 0, sizeof(sa));
    sa.sets = sets_.as<SearchSet>();
    sa.att = reinterpret_cast<const double*>((char*)sets_.p + o_att);
    for (int j = 0; j < 3; ++j) sa.lat.n[j] = counts[j], sa.lat.step[j] = step[j];
    const double zero[12] = {};
    scan_const_at(zero, zero, rot_cov, pos_cov, sa.wide);
    scan_const_at(zero, zero, rot_cov_tight, pos_cov_tight, sa.tight);
    sa.win_sc = win_.as<ScanConst>();
    sa.win_sums = reinterpret_cast<ScoreSum*>((char*)win_.p + o_wsum);
    sa.win_items = reinterpret_cast<ScoreItem*>((char*)win_.p + o_witem);
    sa.out = out_.as<double>();
    sa.best = best_.as<uint64_t>();
    sa.k = k;

    ScoreArgs a;
    std::memset(&a, 0, sizeof(a));
    a.pts = pts_.as<float4>();
    a.partial = partial_.as<double>();
    a.out = out_.as<double>();
    a.mv = mh.view();
    a.g = g;
    // 1-2. window by window: expand the candidates, score them with the wide blocks, merge them into the running best k
    a.items = sa.win_items;
    a.sums = sa.win_sums;
    a.sc = sa.win_sc;
    for (const SearchWindow& w : wins) {
        const uint32_t n = std::max(w.n_poses, w.n_items);
        k_search_expand<<<std::min<uint32_t>((n + EXPAND_THREADS - 1) / EXPAND_THREADS, 4096), EXPAND_THREADS, 0, st>>>(sa, w);
        launch_score(a, w.n_items, w.n_poses, st);
        k_search_keep<<<w.set1 - w.set0 + 1, KEEP_THREADS, 0, st>>>(sa, w);
    }
    LK_CUDA(err, cudaGetLastError());
    // 3-4. the kept poses through the plan of lk_refine_poses (wide blocks), then scored once with the tight blocks
    ScanConst* sc = reinterpret_cast<ScanConst*>((char*)small_.p + o_sc);
    double* res = reinterpret_cast<double*>((char*)small_.p + o_res);
    const uint32_t kb = (n_keep + EXPAND_THREADS - 1) / EXPAND_THREADS;
    k_search_gather<<<kb, EXPAND_THREADS, 0, st>>>(sa, sc, n_keep);
    a.items = small_.as<ScoreItem>();
    a.sums = reinterpret_cast<const ScoreSum*>((char*)small_.p + o_sums);
    a.sc = sc;
    run_windows(a, win_items, win_sums, sc, iters, false, st);
    k_search_tight<<<kb, EXPAND_THREADS, 0, st>>>(sa, sc, n_keep);
    run_windows(a, win_items, win_sums, sc, 0, true, st);
    // 5. each set's k in order, and the one read-back
    k_search_rank<<<n_sets, LK_SEARCH_MAX_K, 0, st>>>(sa, sc, res, n_sets);
    LK_CUDA(err, cudaGetLastError());
    LK_CUDA(err, cudaMemcpyAsync(hb, res, res_bytes, cudaMemcpyDeviceToHost, st));
    LK_CUDA(err, cudaStreamSynchronize(st));
    LK_CUDA(err, cudaGetLastError());
    const double* hr = reinterpret_cast<const double*>(hb);
    for (uint32_t m = 0; m < n_keep; ++m) {
        const double* o = hr + (size_t)m * SEARCH_RESULT;
        std::memcpy(rot_out + 9 * (size_t)m, o, 72);
        std::memcpy(pos_out + 3 * (size_t)m, o + 9, 24);
        std::memcpy(sums_out + PARTIAL_STRIDE * (size_t)m, o + 12, PARTIAL_STRIDE * 8);
    }
    std::memcpy(cand_out, hr + (size_t)n_keep * SEARCH_RESULT, (size_t)n_keep * 4);
    return LK_OK;
}

size_t PoseScorer::device_bytes() const {
    return pts_.cap + small_.cap + partial_.cap + out_.cap + sets_.cap + win_.cap + best_.cap;
}

size_t PoseScorer::host_bytes() const { return h_.cap; }

}  // namespace lk
