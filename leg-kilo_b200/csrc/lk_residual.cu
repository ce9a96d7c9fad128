// lk_residual.cu — one scan on the multi-kernel path: the per-point pass of lk_pass.cuh (transform -> voxel key ->
// hash probes -> staged records -> plane gates -> residual / Jacobian row, the one neighbour voxel on failure) ->
// block-reduced H^T R^-1 H, H^T R^-1 z; the last block of every scan does the 6x6 information-form Kalman solve and the
// state / covariance update. The same pass writes the per-point rows of lk_debug_residuals.
//
// Follows, row by row (SURVEY.md §8a): a3-a7 as lk_point.cuh (where their restructured algebra is written down),
// a8 eskf.cc:91-113, a9 eskf.cc:18-29. K = P H^T (H P H^T + R)^-1 is evaluated as P[:,0:6] (I + A P66)^-1 with
// A = sum h^T h / R (never the results' meaning).
#include "lk_kernels.h"
#include "lk_pass.cuh"
#include "lk_solve.cuh"

namespace lk {

namespace {

#define LK_TRACE(slot) do { if (a.trace && threadIdx.x == 0) a.trace[(size_t)blockIdx.x * 8 + (slot)] = gtime(); } while (0)
#define LK_TRACE_TAIL(slot) do { if (a.trace && threadIdx.x == 0) a.trace[(size_t)gridDim.x * 8 + (slot)] = gtime(); } while (0)

constexpr int BLOCK = 256;  // 8 warps; one point per thread per pass
constexpr int WARPS = BLOCK / 32;

struct TailSmem {
    BlockFilter f;
    double slice[WARPS * 32];
};

// eskf.cc:91-113 + State::operator+= for one scan; run by the last block to finish that scan.
__device__ void scan_solve(const ResidualArgs& a, uint32_t scan, TailSmem* ts) {
    const int tid = threadIdx.x;
    const ScanStep st = a.step[scan];
    double* xg = a.x + (size_t)scan * 36;
    double* Pg = a.P + (size_t)scan * 900;
    // filter into shared memory (these loads overlap the partial-row loads below)
    for (int e = tid; e < 900; e += BLOCK) ts->f.P[e] = Pg[e];
    if (tid < 36) ts->f.x[tid] = xg[tid];
    block_sum_partials<WARPS>(a.partial, st.chunk_begin, st.chunk_end, ts->slice, ts->f.acc);
    LK_TRACE_TAIL(1);
    const uint32_t n = block_solve_update<BLOCK>(&ts->f, a.last_iter != 0);
    LK_TRACE_TAIL(2);
    if (n > 0) {
        if (tid < 36) xg[tid] = ts->f.x[tid];
        if (a.last_iter)
            for (int e = tid; e < 900; e += BLOCK) Pg[e] = ts->f.P[e];
        if (tid == 0) a.clk[scan].last_update_time = st.t_bucket;  // KILO.cc:212
    }
    if (n > 0 || a.last_iter) scan_const_from(&ts->f, a.sc + scan);
    if (tid == 0) {
        ScanStep* sp = a.step + scan;
        sp->n_eff_last = n;
        if (n > 0) sp->updated = 1;
        if (a.last_iter) a.n_eff[scan] += n;
        a.ticket[scan] = 0;
    }
}

template <bool HOT>
union ResidualSmem {  // the tail runs after the pass: same storage
    PassSmem<BLOCK, HOT> pass;
    TailSmem tail;
};

// One pass over the block's chunk (at most BLOCK points on this path), its rows summed into the chunk's partial row; the last
// block of a scan solves. DEBUG (lk_debug_residuals): the chunk may be longer, so the block walks it in BLOCK-point slices and
// writes every point's row and voxel key instead of summing.
// HOT: the pass stages hot plane images (a map that stays fixed for the call), else node records (lk_pass.cuh: Stage).
template <bool DEBUG, bool HOT>
__global__ void __launch_bounds__(BLOCK, 1) k_residual(const __grid_constant__ ResidualArgs a) {
    extern __shared__ __align__(16) unsigned char s_raw[];
    __shared__ ScanConst s_sc;
    __shared__ uint32_t s_last;
    ResidualSmem<HOT>* rs = reinterpret_cast<ResidualSmem<HOT>*>(s_raw);
    TailSmem* ts = &rs->tail;
    const int tid = threadIdx.x;
    LK_TRACE(0);
    const ChunkDesc cd = a.chunks[a.chunk_first + blockIdx.x];
    load_scan_const(&s_sc, a.sc + cd.scan);
    pass_init(&rs->pass);
    LK_TRACE(1);
    MapView mv;
    mv.slots = a.slots; mv.hash_mask = a.hash_mask; mv.nodes = a.nodes; mv.hot = a.hot;
    double acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.0;
    uint32_t phase = 0;
    if (DEBUG) {
        for (uint32_t off = 0; off < cd.count; off += BLOCK) {
            const uint32_t n = min((uint32_t)BLOCK, cd.count - off);
            const size_t base = (size_t)cd.start + off;
            LaneCache lc;
            lc.have = 0;
            float4 pre = make_float4(0.f, 0.f, 0.f, 0.f);
            if ((uint32_t)tid < n) {  // no row yet; the fallback row of this point may come from another thread, after a barrier
                pre = __ldg(a.pts + base + tid);
                a.dbg_ok[base + tid] = 0;
                for (int k = 0; k < 6; ++k) a.dbg_h[(base + tid) * 6 + k] = 0.0;
                a.dbg_z[base + tid] = 0.0;
                a.dbg_R[base + tid] = 0.0;
            }
            points_pass<BLOCK>(&rs->pass, phase, n, s_sc, mv, a.g, lc, pre, [&](uint32_t idx, const Row& row) {
                const size_t gi = base + idx;
                a.dbg_ok[gi] = 1;
                for (int k = 0; k < 6; ++k) a.dbg_h[gi * 6 + k] = row.h[k];
                a.dbg_z[gi] = row.z;
                a.dbg_R[gi] = row.R;
            });
            if ((uint32_t)tid < n) {
                a.dbg_key[(base + tid) * 3 + 0] = lc.kx;
                a.dbg_key[(base + tid) * 3 + 1] = lc.ky;
                a.dbg_key[(base + tid) * 3 + 2] = lc.kz;
            }
        }
        return;
    }
    const uint32_t n = min((uint32_t)BLOCK, cd.count);
    LaneCache lc;
    lc.have = 0;
    float4 pre = make_float4(0.f, 0.f, 0.f, 0.f);
    if ((uint32_t)tid < n) pre = __ldg(a.pts + cd.start + tid);
    points_pass<BLOCK>(&rs->pass, phase, n, s_sc, mv, a.g, lc, pre, [&](uint32_t, const Row& row) { accumulate_row(row, acc); });
    LK_TRACE(2);

    block_row<WARPS>(acc, ts->slice, [&](int i, double v) {
        a.partial[(size_t)(a.chunk_first + blockIdx.x) * PARTIAL_STRIDE + i] = v;
        __threadfence();
    });
    __syncthreads();
    if (tid == 0) {
        const ScanStep* sp = a.step + cd.scan;
        uint32_t n_chunks = sp->chunk_end - sp->chunk_begin;
        uint32_t t = atomicAdd(a.ticket + cd.scan, 1u);
        s_last = (t == n_chunks - 1) ? 1u : 0u;
    }
    __syncthreads();
    LK_TRACE(3);
    if (s_last) {
        __threadfence();
        LK_TRACE_TAIL(0);
        scan_solve(a, cd.scan, ts);
        LK_TRACE_TAIL(7);
    }
}

// The per-scan solve on its own (after lk_stream2.cu's residual pass): one block per scan.
__global__ void __launch_bounds__(BLOCK) k_scan_tail(const __grid_constant__ ResidualArgs a, const uint32_t scan_first) {
    extern __shared__ __align__(16) unsigned char s_raw[];
    TailSmem* ts = reinterpret_cast<TailSmem*>(s_raw);
    const uint32_t scan = scan_first + blockIdx.x;
    const ScanStep st = a.step[scan];
    if (!st.active || st.chunk_end == st.chunk_begin) return;
    scan_solve(a, scan, ts);
}

}  // namespace

void launch_scan_tail(const ResidualArgs& a, uint32_t scan_first, uint32_t n_scans, cudaStream_t s) {
    if (n_scans == 0) return;
    static PerDeviceOnce once;
    if (once.first()) cudaFuncSetAttribute(k_scan_tail, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TailSmem));
    k_scan_tail<<<n_scans, BLOCK, sizeof(TailSmem), s>>>(a, scan_first);
}

template <bool HOT>
void launch_residual_as(const ResidualArgs& a, uint32_t n_chunks, bool debug, cudaStream_t s) {
    static PerDeviceOnce once;
    const size_t smem = sizeof(ResidualSmem<HOT>);
    if (once.first()) {
        cudaFuncSetAttribute(k_residual<true, HOT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        cudaFuncSetAttribute(k_residual<false, HOT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    }
    if (debug)
        k_residual<true, HOT><<<n_chunks, BLOCK, smem, s>>>(a);
    else
        k_residual<false, HOT><<<n_chunks, BLOCK, smem, s>>>(a);
}

void launch_residual(const ResidualArgs& a, uint32_t n_chunks, bool debug, bool hot, cudaStream_t s) {
    if (n_chunks == 0) return;
    if (hot) launch_residual_as<true>(a, n_chunks, debug, s);
    else launch_residual_as<false>(a, n_chunks, debug, s);
}

// ---- re-projection with the updated state (KILO.cc:216-224) ---------------------------------
namespace {
__global__ void __launch_bounds__(BLOCK) k_reproject(const __grid_constant__ ReprojectArgs a) {
    __shared__ ScanConst s_sc;
    __shared__ uint32_t s_upd;
    const int tid = threadIdx.x;
    const ChunkDesc cd = a.chunks[a.chunk_first + blockIdx.x];
    load_scan_const(&s_sc, a.sc + cd.scan);
    if (tid == 0) s_upd = a.step[cd.scan].updated;
    __syncthreads();
    const float inten = s_upd ? 255.0f : 0.0f;
    for (uint32_t i = tid; i < cd.count; i += BLOCK) {
        PointCtx pc;
        imu_point(__ldg(a.pts + cd.start + i), a.g, pc);
        world_point(pc, s_sc);
        float4 o;
        o.x = (float)pc.pwx; o.y = (float)pc.pwy; o.z = (float)pc.pwz;
        o.w = inten;
        a.world[cd.start + i] = o;
    }
}
}  // namespace

void launch_reproject(const ReprojectArgs& a, uint32_t n_chunks, cudaStream_t s) {
    if (n_chunks == 0) return;
    k_reproject<<<n_chunks, BLOCK, 0, s>>>(a);
}

}  // namespace lk
