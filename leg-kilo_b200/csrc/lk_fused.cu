// lk_fused.cu — the whole bucket loop of ONE scan (KILO.cc:367-396 -> predictUpdatePoint
// KILO.cc:108-233) as a single persistent kernel, one 256-point chunk per block: every block keeps its
// own copy of the filter (state 36 + covariance 900 doubles) in shared memory and repeats the tiny
// serial parts (predict, 6x6 solve, state / covariance update) redundantly, so the only grid-wide
// exchange per iteration is ONE all-reduce of the 29 sums H^T R^-1 H | H^T R^-1 z | sum R | count.
//
// That all-reduce has no barrier: rows travel in the flagged format of lk_llsync.cuh (data and "ready"
// tag in the same 8-byte words), two levels deep — the block of a group's first chunk adds the group's
// LK_GROUP rows and publishes the group row, every block adds the (<= 19) group rows — so a round costs
// two L2 round trips after the slowest block, moves ~10 KB per block instead of every row to every block,
// and the sum has ONE fixed order that the multi-kernel path reproduces (block_sum_partials).
//
// Per-lane cache (lk_pass.cuh: points_pass): a lane keeps its point, voxel keys, lookups and BOTH
// candidate plane records (home + the reference's one fallback neighbour, TMA-staged together) across the
// iterations of a bucket, so iterations 2..n touch no global memory unless a key moved.
//
// Two instantiations keep the instruction footprint of the common case small: OBS = false (no inertial /
// kinematic queue: the scan-at-once and streaming-without-queue shapes) and OBS = true (queue drained
// before every bucket, KILO.cc:379-390). The predict and the queue drain are out of line in both.
// The kernel is PDL-aware (griddepcontrol): launched with programmatic stream serialisation, the next
// scan's blocks become resident and run their prologue (filter load, point prefetch) while this scan's
// last blocks drain; everything that could collide with the previous launch (flagged rows, outputs) sits
// behind griddepcontrol.wait.
//
// Finishers: a single-bucket launch without a queue or insert that leaves SMs idle gets up to LL_MAX_FINISHERS extra
// blocks (FusedArgs::finishers). They follow every exchange and solve like the other blocks (their filter is the same),
// but the chunk blocks — workers — leave at the last exchange as soon as their row is published: the last total, solve,
// re-projection, covariance update and stores run on the finishers (fused_finish), while the workers' SMs already take
// the next launch's blocks, which need none of that work until their own first exchange.
#include "lk_insert.cuh"
#include "lk_kernels.h"
#include "lk_obs.cuh"
#include "lk_pass.cuh"
#include "lk_predict.cuh"
#include "lk_solve.cuh"

namespace lk {

namespace {

#define FT(slot) do { if (a.trace && threadIdx.x == 0 && (slot) < 32) a.trace[(size_t)blockIdx.x * 32 + (slot)] = gtime(); } while (0)
// per-iteration stamps of the first three exchanges i: 14 + i pass done, 2 + 4i block row in shared memory, 3 + 4i all-reduce
// total in shared memory, 4 + 4i solve done (tools/trace_fused.py); 23 / 24 before / after the first griddepcontrol.wait,
// a finisher's 20 re-projection stored, 21 covariance stored, 22 state stored; 31 a block's end
#define FTI(slot) do { if (it_global < 3) FT(slot); } while (0)
// per-bucket stamps of the streaming variants (block 0, first 64 buckets, 8 stamps each, behind the per-block area)
#define FTS(slot) do { if (a.trace && blockIdx.x == 0 && threadIdx.x == 0 && k < 64) a.trace[(size_t)gridDim.x * 32 + (size_t)k * 8 + (slot)] = gtime(); } while (0)
// The all-reduce's hop stamps and poll-round counts (lk_llsync.cuh: LL_HOP_SLOTS per exchange, first three exchanges, 16
// slots per block behind the per-bucket area: 160 blocks fill the 8192-stamp trace area). Unlike FT / FTI they are gated at
// compile time as well as by a.trace: only `make HOP_TRACE=1` (a library of its own, tools/trace_fused.py --hops) compiles
// them in, so the default library's all-reduce has the same instructions whether tracing exists or not.
#ifndef LK_HOP_TRACE
#define LK_HOP_TRACE 0
#endif
#define FT_HOPS() ((LK_HOP_TRACE && a.trace && it_global < 3) \
                       ? a.trace + (size_t)gridDim.x * 32 + 64 * 8 + (size_t)blockIdx.x * 16 + it_global * LL_HOP_SLOTS : nullptr)

constexpr int BLOCK = FB;
constexpr int WARPS = BLOCK / 32;

struct PredictScratch {
    double F[900];
    double T[900];
    double Ps[900];
    ObsScratch obs;  // the IMU / Kin+IMU update follows its predict, so both live here
};

// HOT: the passes stage hot plane images (a map that stays fixed for the launch), else node records (lk_pass.cuh: Stage)
template <bool HOT>
struct FusedSmemT {
    BlockFilter f;
    ScanConst sc;
    double slice[WARPS * 32];
    double clk[2];
    union {  // predict and the point passes never overlap in time
        PredictScratch pr;
        PassSmem<BLOCK, HOT> pass;
    } u;
};
typedef FusedSmemT<true> FusedSmem;  // without the map insert

// with the map insert inside: the plane-fit staging tiles of the warps, with their own mbarriers (initialised once)
struct FusedSmemIns {
    FusedSmemT<false> base;  // the map changes between buckets: node records
    WarpTile wt[WARPS];
    MapDev md;   // copies for the out-of-line insert phase
    Globals g;
};

// Phase 2 of the in-kernel UpdateVoxelMap, out of line: the octree / plane-fit code then gets a register allocation of
// its own (as in the stand-alone insert kernel) instead of spilling inside the persistent kernel's.
__device__ __noinline__ void fused_insert_phase2(FusedSmemIns* si, const uint32_t* touched, const int* iroot, const DevPoint* ipts,
                                                 int* pend, uint32_t n_touched, uint32_t n_bucket) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    MapDev md = si->md;
    WarpTile* wt = si->wt + warp;
    for (uint32_t t = blockIdx.x * (uint32_t)WARPS + (uint32_t)warp; t < n_touched; t += gridDim.x * (uint32_t)WARPS)
        warp_insert_root_scan(md, si->g, wt, __ldcg(&touched[t]), iroot, ipts, n_bucket, pend, lane);
}

static_assert(sizeof(PredictScratch) <= sizeof(((PassSmem<BLOCK, true>*)0)->tile) &&
                  sizeof(PredictScratch) <= sizeof(((PassSmem<BLOCK, false>*)0)->tile),
              "predict scratch must not reach the mbarriers");
static_assert(sizeof(FusedSmemIns) <= 227 * 1024, "one block per SM");
// The block's shared memory plus the 1 KiB the driver reserves per block must fit the 132 KiB carve-out: the remaining
// 124 KiB of L1 then hold the stack frames of all 256 threads (a few hundred bytes each) beside the cached point and table
// reads, so their spill traffic stays in L1. With the node-record tiles (the map-insert variant) it needs 164 KiB or more.
static_assert(sizeof(FusedSmem) + 1024 <= 132 * 1024, "the batch-of-one kernel's stack frames must fit in L1");

// The smallest shared-memory carve-out that holds one block of `smem` bytes, as the percentage
// cudaFuncAttributePreferredSharedMemoryCarveout takes (the driver rounds up to the next carve-out the SM supports). Without
// it the driver may pick a larger carve-out than one block needs, and the L1 left for the stack frames shrinks.
int carveout_percent(size_t smem, int dev) {
    int per_sm = 0, per_block = 0;
    cudaDeviceGetAttribute(&per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
    cudaDeviceGetAttribute(&per_block, cudaDevAttrReservedSharedMemoryPerBlock, dev);
    if (per_sm <= 0) return 100;
    const size_t need = smem + (size_t)per_block;
    const int pct = (int)((need * 100 + (size_t)per_sm - 1) / (size_t)per_sm);
    return pct < 100 ? pct : 100;
}

// KILO.cc:110-115: covariance with dt since the last UPDATE, state with dt since the last PREDICT; F is built
// from the pre-propagation state. Out of line: a scan-at-once call (bucket time == both clocks) never gets here.
template <class SM>
__device__ __noinline__ void fused_predict(SM* sm, const double* Q, double dtc, double dt) {
    if (dtc != 0.0) {
        build_F(sm->u.pr.F, sm->f.x, dtc);
        cov_predict(sm->f.P, sm->u.pr.F, sm->u.pr.T, sm->u.pr.Ps, Q, dtc);
    }
    if (dt != 0.0) {
        if (threadIdx.x == 0) state_predict(sm->f.x, dt);
    }
    // the scratch aliased the record tiles (not the mbarriers, which sit behind them and keep their
    // phases): order these generic-proxy writes before the next bulk copies
    fence_proxy_async();
    __syncthreads();
}

// every queued inertial / kinematic sample older than this bucket (KILO.cc:379-390)
template <class SM>
__device__ __noinline__ void fused_drain_queue(SM* sm, const FusedArgs& a, uint32_t& mi, double t_bucket) {
    bool drained = false;
    while (mi < a.n_meas) {
        const double ts = a.imu ? a.imu[mi].stamp : a.kin[mi].stamp;
        if (!(ts < t_bucket)) break;
        block_predict_to(&sm->f, sm->clk, ts, sm->u.pr.F, sm->u.pr.T, sm->u.pr.Ps, a.Q);
        if (a.imu) block_obs_imu<BLOCK>(&sm->f, &sm->u.pr.obs, a.imu + mi, &a.ecfg, a.gravity, a.acc_norm);
        else block_obs_kinimu<BLOCK>(&sm->f, &sm->u.pr.obs, a.kin + mi, &a.ecfg, a.gravity, a.acc_norm);
        if (threadIdx.x == 0) sm->clk[1] = ts;
        __syncthreads();
        ++mi;
        drained = true;
    }
    if (drained) {  // the scratch aliased the record tiles
        fence_proxy_async();
        __syncthreads();
    }
}

// KILO.cc:216-224: a point of the world cloud at the updated state (pi: the point in the IMU frame, imu_point)
__device__ __forceinline__ float4 world_out(const double* X, double pix, double piy, double piz, bool updated) {
    float4 o;
    o.x = (float)(X[0] * pix + X[1] * piy + X[2] * piz + X[9]);
    o.y = (float)(X[3] * pix + X[4] * piy + X[5] * piz + X[10]);
    o.z = (float)(X[6] * pix + X[7] * piy + X[8] * piz + X[11]);
    o.w = updated ? 255.0f : 0.0f;
    return o;
}

// The state, the clocks, the residual count and the status word of the scan (the covariance is stored by the caller).
template <class SM>
__device__ __forceinline__ void store_state(SM* sm, const FusedArgs& a, uint32_t n_eff) {
    const int tid = threadIdx.x;
    if (tid < 36) a.x[(size_t)a.scan * 36 + tid] = sm->f.x[tid];
    if (tid < 2) reinterpret_cast<double*>(a.clk + a.scan)[tid] = sm->clk[tid];
    if (tid == 0) {
        a.n_eff[a.scan] = n_eff;
        // did any wait of this launch give up (lk_llsync.cuh / lk_async.cuh watchdogs)? The host looks at this word first
        // and only then pays for the detailed read-back
        *a.status = (*reinterpret_cast<volatile uint32_t*>(a.ll.stall) ? 1u : 0u) | (*reinterpret_cast<volatile uint32_t*>(&lk_stall_note[0]) ? 2u : 0u);
    }
}

// A finisher's re-projection inputs, staged while it waits for the last chunk rows (fused_finish): the IMU-frame points
// (pix, piy, piz) of its first FIN_STAGE points, kept in the record tiles behind the group sums of ll_sum_chunk_rows
// (u.pr.F). A finisher's passes have no points, so it never issues a bulk copy into those tiles, and the predict scratch
// is dead by its last exchange.
typedef PassSmem<BLOCK, true> PassHot;
typedef PassSmem<BLOCK, false> PassNodes;
constexpr size_t FIN_GS_BYTES = (size_t)LL_MAX_GROUPS * 32 * sizeof(double);
constexpr uint32_t FIN_STAGE = (uint32_t)((sizeof(PassHot::tile) - FIN_GS_BYTES) / (3 * sizeof(double)));
static_assert(offsetof(PredictScratch, F) == 0 && offsetof(PassHot, tile) == 0 && offsetof(PassNodes, tile) == 0,
              "the group sums and the staging area start at the tiles");
static_assert(FIN_GS_BYTES + 3 * sizeof(double) * FIN_STAGE <= sizeof(PassHot::tile) &&
                  sizeof(PassHot::tile) <= sizeof(PassNodes::tile) && sizeof(PassHot::tile) <= offsetof(PassHot, bar),
              "the finishers' staging area must stay inside the tiles, clear of the mbarriers");

// The epilogue of a launch with finishers, run by each finisher (blocks n_chunks .. gridDim.x - 1) at the scan's last
// exchange: that exchange in one hop from the chunk rows, the last solve, then the re-projection and the covariance update
// split over the finishers, and the stores. The workers have left by then; the filter they would have ended with is the
// one every finisher holds. Out of line, so the workers' register allocation is that of the kernel without it.
template <class SM>
__device__ __noinline__ void fused_finish(SM* sm, const FusedArgs& a, const StepInit& in, uint32_t n_chunks, uint32_t it_global,
                                          bool updated, bool dep_waited) {
    const int tid = threadIdx.x;
    const uint32_t fi = blockIdx.x - n_chunks, nf = gridDim.x - n_chunks;
    if (!dep_waited) asm volatile("griddepcontrol.wait;" ::: "memory");  // the rows / outputs of the previous launch
    // A thread's j-th point of the re-projection is first + j * step. The IMU-frame point does not depend on the state:
    // form it for the first n_st of them now, while the last chunk rows are still on their way, and keep it in shared
    // memory at j * BLOCK + tid (the thread's own slots: no barrier). Direct mode reads the workers' device copy, which
    // is complete only with their last row: it stages nothing.
    constexpr int U = 8;  // a thread's points in batches of U, all loads of a batch issued before the first use
    const uint32_t step = nf * BLOCK;
    const uint32_t first = in.pt_begin + fi * BLOCK + tid;
    double* st = reinterpret_cast<double*>(reinterpret_cast<unsigned char*>(&sm->u) + FIN_GS_BYTES);
    const uint32_t n_pts = first < in.pt_end ? (in.pt_end - first + step - 1) / step : 0u;
    const uint32_t n_st = a.pts_copy ? 0u : min(n_pts, (FIN_STAGE - (uint32_t)tid + BLOCK - 1) / BLOCK);
    for (uint32_t j0 = 0; j0 < n_st; j0 += U) {
        float4 q[U];
#pragma unroll
        for (int u = 0; u < U; ++u)
            if (j0 + u < n_st) q[u] = __ldcg(a.pts + first + (j0 + u) * step);
#pragma unroll
        for (int u = 0; u < U; ++u)
            if (j0 + u < n_st) {
                PointCtx p;
                imu_point(q[u], a.g, p);
                const uint32_t l = (j0 + u) * BLOCK + tid;
                st[l] = p.pix;
                st[FIN_STAGE + l] = p.piy;
                st[2 * FIN_STAGE + l] = p.piz;
            }
    }
    ll_sum_chunk_rows<WARPS>(a.ll, it_global & 1u, a.epoch + it_global, n_chunks, sm->u.pr.F, sm->f.acc);
    FTI(3 + it_global * 4);
    const uint32_t n = block_solve_state(&sm->f);
    FTI(4 + it_global * 4);
    if (n > 0) {
        updated = true;
        if (tid == 0) sm->clk[1] = in.t_bucket;  // KILO.cc:212
    }
    // re-projection (KILO.cc:216-224): the staged points first
    for (uint32_t j = 0; j < n_st; ++j) {
        const uint32_t l = j * BLOCK + tid;
        a.world[first + j * step] = world_out(sm->f.x, st[l], st[FIN_STAGE + l], st[2 * FIN_STAGE + l], updated);
    }
    // then the points beyond the staging area, and in direct mode all of them: from the workers' device copy, stored
    // before their last row (the fence makes those stores visible here); a finisher never reads host memory
    const float4* pts = a.pts;
    if (a.pts_copy) {
        __threadfence();
        pts = a.pts_copy;
    }
    for (uint32_t i0 = first + n_st * step; i0 < in.pt_end; i0 += U * step) {
        float4 q[U];
#pragma unroll
        for (int u = 0; u < U; ++u)
            if (i0 + u * step < in.pt_end) q[u] = __ldcg(pts + i0 + u * step);
#pragma unroll
        for (int u = 0; u < U; ++u)
            if (i0 + u * step < in.pt_end) {
                PointCtx p;
                imu_point(q[u], a.g, p);
                a.world[i0 + u * step] = world_out(sm->f.x, p.pix, p.piy, p.piz, updated);
            }
    }
    FT(20);
    if (n > 0) cov_prep(&sm->f, BLOCK);
    __syncthreads();
    for (uint32_t e = fi * BLOCK + tid; e < 900; e += nf * BLOCK)
        a.P[(size_t)a.scan * 900 + e] = n > 0 ? cov_entry(&sm->f, (int)e) : sm->f.P[e];
    FT(21);
    if (fi == 0) store_state(sm, a, n);
    FT(22);
}

// The all-reduce's shared-memory scratch (ll_allreduce: LL_XS doubles) lives in the pass's point contexts: a pass writes
// every context it reads (points_pass) and ends with a block barrier, and the exchange ends with one before the next pass,
// so the two never overlap. Between buckets the contexts are dead too (the predict scratch and the insert use other
// memory), which covers the barriers of grid_sync.
template <class SM>
__device__ __forceinline__ double* ll_scratch(SM* sm) { return reinterpret_cast<double*>(sm->u.pass.pt); }
static_assert(sizeof(PassHot::pt) >= LL_XS * sizeof(double) && sizeof(PassNodes::pt) >= LL_XS * sizeof(double) &&
                  alignof(PointCtx) >= alignof(double),
              "the all-reduce's scratch must fit in the point contexts");

template <bool INL> struct InlineSel { typedef FusedInline type; };
template <> struct InlineSel<false> { typedef FusedNoInline type; };

// A grid-wide barrier out of the flagged-row all-reduce (every block contributes a zero row). Release side: every thread
// fences its earlier global writes. Acquire side: a gpu-scope fence AFTER the barrier — on this architecture it also
// invalidates the SM's L1 (CCTL.IVALL, see the SASS), so the plain (L1-cached) loads of the next phase cannot be served from
// a line cached before another SM rewrote it; the read-only path (ld.global.nc) is not used on the map in these kernels.
// The next bucket's pass reads the node records the insert just wrote with generic stores through bulk copies (async
// proxy): a proxy fence after the acquire orders the two.
template <class SM>
__device__ __forceinline__ void grid_sync(SM* sm, const FusedArgs& a, uint32_t& sync_idx) {
    __threadfence();
    __syncthreads();
    (void)ll_allreduce<WARPS>(a.ll, sync_idx & 1u, a.epoch + sync_idx, blockIdx.x, gridDim.x, 0.0, ll_scratch(sm));
    ++sync_idx;
    __syncthreads();
    __threadfence();
    fence_proxy_async_global();
}

// OBS: an inertial / kinematic queue is drained before every bucket. INL: the small inputs ride in the parameter block.
// INS: UpdateVoxelMap runs inside the kernel after every bucket (KILO.cc:231): the map is then read through L2.
template <bool OBS, bool INL, bool INS>
__global__ void __launch_bounds__(BLOCK, 1) k_scan_fused(const __grid_constant__ FusedArgs a,
                                                         const __grid_constant__ typename InlineSel<INL>::type inl) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    FusedSmemT<!INS>* sm = reinterpret_cast<FusedSmemT<!INS>*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t scan = a.scan;
    // a.finishers > 0: the last a.finishers blocks of the grid are finishers (fused_finish), the others workers
    const bool finisher = blockIdx.x + a.finishers >= gridDim.x;
    // let the next launch of the stream (if it was launched with programmatic serialisation) start placing its
    // blocks as soon as this grid's blocks are all running; it blocks in griddepcontrol.wait until we are done
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    FT(0);
    // the filter: always reloaded from the staged inputs (idempotent runs); these are inputs, never written by a kernel
    {
        const double* Pin;
        const double* xin;
        const double* cin;
        if constexpr (INL) { Pin = inl.P; xin = inl.x; cin = inl.clk; }
        else { Pin = a.P_in + (size_t)scan * 900; xin = a.x_in + (size_t)scan * 36; cin = reinterpret_cast<const double*>(a.clk_in + scan); }
        if (a.slim_p && !finisher && (a.finishers || blockIdx.x != 0)) {
            // a single-bucket scan without a queue never predicts; blocks that do not store the covariance (all but block
            // 0, or all workers) then only ever read P[:, 0:6]: the 6x6 corner for the solve and the scan constants, the
            // 30x6 strip for delta
            if (tid < 180) sm->f.P[(tid / 6) * 30 + tid % 6] = Pin[(tid / 6) * 30 + tid % 6];
        } else {
            for (int e = tid; e < 900; e += BLOCK) sm->f.P[e] = Pin[e];
        }
        if (tid < 36) sm->f.x[tid] = xin[tid];
        if (tid < 2) sm->clk[tid] = cin[tid];
    }
    if constexpr (INS) {
        FusedSmemIns* si = reinterpret_cast<FusedSmemIns*>(smem_raw);
        WarpTile* wt = si->wt + warp;
        if (lane == 0) {
            mbar_init(&wt->bar, 1);
            wt->phase = 0;
        }
        if (tid == 0) si->md = a.md;
        if (tid < (int)(sizeof(Globals) / 4)) reinterpret_cast<uint32_t*>(&si->g)[tid] = reinterpret_cast<const uint32_t*>(&a.g)[tid];
    }
    pass_init(&sm->u.pass);  // mbarrier init fence + block barrier
    FT(1);
    uint32_t n_eff_total = 0;
    uint32_t phase = 0;
    uint32_t it_global = 0;  // index of the next grid-wide exchange (all-reduce or barrier): tag and buffer parity
    uint32_t cslot = 0;      // which of the two "touched roots" counters the current bucket uses (INS)
    uint32_t mi = 0;  // next inertial / kinematic sample
    bool dep_waited = false;

    for (uint32_t k = 0; k < a.n_steps; ++k) {
        StepInit in;
        if constexpr (INL) in = inl.steps[k];
        else in = a.inits[(size_t)k * a.batch + scan];
        if (!in.active) continue;
        const uint32_t n_chunks = in.chunk_end - in.chunk_begin;  // <= gridDim.x (the host checks)
        // a lane sees the same point in every iteration of the bucket: issue its load now, ahead of the predict
        // (the point may sit in page-locked host memory)
        const uint32_t my_start = in.pt_begin + blockIdx.x * (uint32_t)BLOCK;
        const uint32_t my_count = blockIdx.x < n_chunks ? min((uint32_t)BLOCK, in.pt_end - my_start) : 0u;
        float4 pre = make_float4(0.f, 0.f, 0.f, 0.f);
        if ((uint32_t)tid < my_count) pre = __ldg(a.pts + my_start + tid);
        FTS(0);
        if constexpr (OBS) fused_drain_queue(sm, a, mi, in.t_bucket);
        FTS(1);
        const double dtc = in.t_bucket - sm->clk[1];
        const double dt = in.t_bucket - sm->clk[0];
        if (dtc != 0.0 || dt != 0.0) fused_predict(sm, a.Q, dtc, dt);
        if (tid == 0) sm->clk[0] = in.t_bucket;
        FTS(2);
        bool updated = false, cov_pending = false;
        uint32_t n_last = 0;
        LaneCache lc;
        lc.have = 0;
        const bool more_steps = k + 1 < a.n_steps;
        for (int it = 0; it < a.iters; ++it, ++it_global) {
            scan_const_from(&sm->f, &sm->sc);
            __syncthreads();
            // 1) residual rows of my chunk
            double acc[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) acc[i] = 0.0;
            if (!a.lane_cache && lc.have == 2) lc.have = 1;
            points_pass<BLOCK, INS>(&sm->u.pass, phase, my_count, sm->sc, a.mv, a.g, lc, pre,
                                    [&](uint32_t, const Row& row) { accumulate_row(row, acc); });
            FTI(14 + it_global);
            const double tot = warp_transpose_sum(acc, lane);
            sm->slice[warp * 32 + lane] = tot;
            __syncthreads();
            FTI(2 + it_global * 4);
            if (it == 0) FTS(3);
            const bool last = it == a.iters - 1;
            if (!OBS && !INS && a.finishers && last) {
                // the last exchange of a launch with finishers (a single bucket): a worker publishes its row and leaves, the
                // finishers take it from there; the SMs of the workers go to the next launch
                if (finisher) {
                    fused_finish(sm, a, in, n_chunks, it_global, updated, dep_waited);
                } else {
                    if (!dep_waited) asm volatile("griddepcontrol.wait;" ::: "memory");  // the rows of the previous launch
                    if (a.pts_copy) {  // direct mode: the finishers re-project from a device copy (fused_finish)
                        if ((uint32_t)tid < my_count) a.pts_copy[my_start + tid] = pre;
                        __threadfence();
                        __syncthreads();
                    }
                    if (warp == 0) {
                        double v = 0.0;
#pragma unroll
                        for (int w = 0; w < WARPS; ++w) v += sm->slice[w * 32 + lane];
                        ll_publish_row(a.ll, it_global & 1u, a.epoch + it_global, blockIdx.x, v, lane);
                    }
                }
                FT(31);
                return;
            }
            // 2) all-reduce of the block rows, no grid barrier: warp 0 stores, every warp polls
            double v = 0.0;
            if (warp == 0) {
#pragma unroll
                for (int w = 0; w < WARPS; ++w) v += sm->slice[w * 32 + lane];
                if (!dep_waited) {  // the rows / outputs of the previous launch
                    FT(23);
                    asm volatile("griddepcontrol.wait;" ::: "memory");
                    FT(24);
                }
            }
            const double t = ll_allreduce<WARPS>(a.ll, it_global & 1u, a.epoch + it_global, blockIdx.x, n_chunks, v, ll_scratch(sm),
                                                 FT_HOPS(), a.finishers, it_global >= 2);
            if (warp == 0) sm->f.acc[lane] = t;
            dep_waited = true;
            __syncthreads();
            FTI(3 + it_global * 4);
            if (it == 0) FTS(4);
            // 3) every block solves redundantly (eskf.cc:91-113); the covariance update of the last iteration is
            //    deferred behind the re-projection, and skipped where nobody reads the result
            const uint32_t n = block_solve_state(&sm->f);
            FTI(4 + it_global * 4);
            if (n > 0) {
                updated = true;
                if (tid == 0) sm->clk[1] = in.t_bucket;  // KILO.cc:212
                if (last) cov_pending = INS || more_steps || blockIdx.x == 0;  // the insert needs the updated covariance in every block
            }
            n_last = n;
        }
        n_eff_total += n_last;
        FTS(5);
        if constexpr (!INS) {
            // 4) re-projection with the updated state (KILO.cc:216-224)
            if ((uint32_t)tid < my_count) a.world[my_start + tid] = world_out(sm->f.x, lc.pix, lc.piy, lc.piz, updated);
            FT(20);
            if (cov_pending) block_cov_update<BLOCK>(&sm->f);
        } else {
            // 4') re-projection AND map insert with the updated state and covariance (KILO.cc:216-231). Phase 1, the blocks
            //     that hold the bucket's points: pointWithVar, world cloud, find-or-create of the root voxel.
            if (cov_pending) block_cov_update<BLOCK>(&sm->f);
            __syncthreads();
            scan_const_from(&sm->f, &sm->sc);
            __syncthreads();
            MapDev md = a.md;
            const uint32_t n_bucket = in.pt_end - in.pt_begin;
            if ((uint32_t)tid < my_count) {
                // (without an update the reference inserts the point as the residual loop left it, KILO.cc:127-140, :215: the
                // same formulas at the unchanged state)
                DevPoint p;
                make_insert_point(lc.pix, lc.piy, lc.piz, lc.pbx, lc.pby, lc.pbz, sm->sc, a.g, p);
                const uint32_t li = my_start + tid - in.pt_begin;
                a.ipts[li] = p;
                float4 o;
                o.x = (float)p.pw[0]; o.y = (float)p.pw[1]; o.z = (float)p.pw[2];
                o.w = updated ? 255.0f : 0.0f;
                a.world[my_start + tid] = o;
                a.iroot[li] = insert_register_point(md, a.g, p, a.pend, a.touched, &a.ins_counters[cslot]);
            }
            grid_sync(sm, a, it_global);
            FTS(6);
            // Phase 2, every warp of every block: one touched root at a time, its points in index order
            {
                const uint32_t n_touched = __ldcg(&a.ins_counters[cslot]);
                if (blockIdx.x == 0 && tid == 0) a.ins_counters[cslot ^ 1u] = 0;  // the next bucket's counter
                fused_insert_phase2(reinterpret_cast<FusedSmemIns*>(smem_raw), a.touched, a.iroot, a.ipts, a.pend, n_touched, n_bucket);
                cslot ^= 1u;
            }
            grid_sync(sm, a, it_global);
            FTS(7);
        }
    }
    FT(30);
    if (blockIdx.x == 0) {
        if (!dep_waited) asm volatile("griddepcontrol.wait;" ::: "memory");
        __syncthreads();
        for (int e = tid; e < 900; e += BLOCK) a.P[(size_t)scan * 900 + e] = sm->f.P[e];
        store_state(sm, a, n_eff_total);
    }
    FT(31);
}

template <bool OBS, bool INL, bool INS>
cudaError_t launch_one(const FusedArgs& a, const FusedInline* inl, uint32_t grid, cudaStream_t s, int mode) {
    auto kern = k_scan_fused<OBS, INL, INS>;
    constexpr size_t SMEM = INS ? sizeof(FusedSmemIns) : sizeof(FusedSmem);
    static PerDeviceOnce once;
    if (once.first()) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM);
        if (e != cudaSuccess) return e;
        e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, carveout_percent(SMEM, dev));
        if (e != cudaSuccess) return e;
    }
    typename InlineSel<INL>::type local_inl;
    const typename InlineSel<INL>::type* ip;
    if constexpr (INL) ip = inl;
    else { local_inl.unused = 0; ip = &local_inl; }
    if (mode == FUSED_LAUNCH_COOPERATIVE) {
        void* params[] = {(void*)&a, (void*)ip};
        return cudaLaunchCooperativeKernel((const void*)kern, dim3(grid), dim3(BLOCK), params, SMEM, s);
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(BLOCK);
    cfg.dynamicSmemBytes = SMEM;
    cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = mode == FUSED_LAUNCH_PDL ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, a, *ip);
}

}  // namespace

size_t fused_smem_bytes() { return sizeof(FusedSmem); }

// read and clear this translation unit's watchdog note (lk_async.cuh)
int fused_read_stall(uint32_t out[8]) {
    if (cudaMemcpyFromSymbol(out, lk_stall_note, 32) != cudaSuccess) return -1;
    if (out[0]) {
        const uint32_t z[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        cudaMemcpyToSymbol(lk_stall_note, z, 32);
    }
    return 0;
}

int fused_max_blocks(int device) {
    static int cached[64];
    static bool have[64];
    if (device >= 0 && device < 64 && have[device]) return cached[device];
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    int n = sms < LL_MAX_CHUNKS ? sms : LL_MAX_CHUNKS;  // one block per SM (launch bounds + shared memory)
    if (device >= 0 && device < 64) { cached[device] = n; have[device] = true; }
    return n;
}

// mode: plain <<<>>>, cooperative (the driver checks co-residency and serialises cooperative grids: a gap between
// back-to-back launches) or programmatic stream serialisation (PDL). The non-cooperative launches rely on the
// fact the host enforces — grid <= SM count at one block per SM, i.e. every block fits on the device at once —
// so blocks polling for rows only ever wait for blocks that are resident or become resident as soon as unrelated
// work drains; lk_api.cu serialises fused grids of different handles of one process (see INTEGRATION.md for the
// multi-process caveat and the cooperative knob).
cudaError_t launch_scan_fused(const FusedArgs& a, const FusedInline* inl, uint32_t grid, cudaStream_t s, int mode) {
    const bool obs = a.n_meas > 0;
    if (a.insert) {  // streaming with map insertion: never with inline inputs
        if (inl) return cudaErrorInvalidValue;
        return obs ? launch_one<true, false, true>(a, inl, grid, s, mode) : launch_one<false, false, true>(a, inl, grid, s, mode);
    }
    if (obs) return inl ? launch_one<true, true, false>(a, inl, grid, s, mode) : launch_one<true, false, false>(a, inl, grid, s, mode);
    return inl ? launch_one<false, true, false>(a, inl, grid, s, mode) : launch_one<false, false, false>(a, inl, grid, s, mode);
}

}  // namespace lk
