// lk_pass.cuh — points_pass, one block-wide pass over up to NTHREADS points (one point per thread) through the reference's
// residual sequence (KILO.cc:143-178). The one per-point pass of the per-scan kernel (lk_fused.cu), the single-scan residual
// kernel and the debug rows (lk_residual.cu):
//   1. transform, voxel key, home probe AND the speculative probe of the one neighbour voxel the
//      reference falls back to (KILO.cc:156-178) — both 16-byte table reads are in flight together;
//   2. every lane stages what it evaluates of its home and neighbour roots into shared memory with TMA bulk copies
//      (cp.async.bulk global -> shared, completion on the warp's mbarrier) instead of scattered 128-bit loads:
//      HOT = the 144-byte hot plane images (lk_device.cuh: HotRec), else the first 240 bytes of the node records;
//   3. gates + residual row from the staged slot (conflict-free 128-bit shared loads); with HOT, a root that holds
//      no plane reads its node record and descends into its children (eval_descent, rare);
//   4. points whose home voxel gave no residual are compacted into a block-wide list and their
//      neighbour record is evaluated by the first threads of the block — a few percent of the
//      points fail, but almost every warp holds one, so without compaction every warp would pay
//      the second round.
#pragma once
#include <cstddef>

#include "lk_async.cuh"
#include "lk_point.cuh"

namespace lk {

// What a lane stages per root, and the slot stride of the tiles: an odd number of 16-byte units, so the 128-bit reads of 8
// consecutive lanes fall into 8 disjoint groups of 4 banks.
//   HOT = false: the 15 x 16 bytes of the node record plane_from_smem reads (centre .. flags / child_base), 240-byte slots.
//   HOT = true: the 144 used bytes of the hot image (eval_plane_hot), 176-byte slots.
// The hot image evaluates sigma_plane in the collapsed form a^T Scc a - 2 a^T v + s, which rounds differently from the
// 21-term form of the node record (about 1e-16 relative). A pass over a map that stays fixed for the call takes the hot
// images, like the throughput family; a call that updates the map takes the node records, so that the rounding does not
// compound through the points it inserts (the map-vs-reference parity of the streaming path is bitwise in the form it has).
template <bool HOT> struct Stage;
template <> struct Stage<false> { static constexpr uint32_t BYTES = 240; static constexpr int STRIDE = 240; };
template <> struct Stage<true> { static constexpr uint32_t BYTES = 144; static constexpr int STRIDE = 176; };
static_assert(offsetof(lk_map_node, child_base) + sizeof(int32_t) <= Stage<false>::BYTES && Stage<false>::BYTES % 16 == 0 &&
                  Stage<false>::STRIDE >= (int)Stage<false>::BYTES && Stage<false>::STRIDE % 32 == 16,
              "staged record slots");
static_assert(Stage<true>::BYTES % 16 == 0 && Stage<true>::BYTES <= sizeof(HotRec) && Stage<true>::STRIDE >= (int)Stage<true>::BYTES &&
                  Stage<true>::STRIDE % 32 == 16,
              "staged hot image slots");

__device__ __forceinline__ void accumulate_row(const Row& row, double (&acc)[32]) {
    const double w = 1.0 / row.R;
    int q = 0;
#pragma unroll
    for (int r = 0; r < 6; ++r) {
        const double hw = row.h[r] * w;
#pragma unroll
        for (int c = r; c < 6; ++c) acc[q++] += hw * row.h[c];
        acc[ACC_B + r] += hw * row.z;
    }
    acc[ACC_SUMR] += row.R;
    acc[ACC_CNT] += 1.0;
}

// Linear probing, two slots per step: an even-aligned pair of 16-byte slots shares one 32-byte
// sector, so the second slot is free. `pre` holds the pair at the key's home position (already
// loaded by the caller so several lookups can be in flight together).
struct SlotPair {
    int4 a, b;
};
template <bool COH = false>
__device__ __forceinline__ SlotPair load_pair(const HashSlot* __restrict__ slots, uint32_t i) {
    SlotPair p;
    const int4* q = reinterpret_cast<const int4*>(slots + (i & ~1u));
    p.a = COH ? __ldcg(q) : __ldg(q);
    p.b = COH ? __ldcg(q + 1) : __ldg(q + 1);
    return p;
}
// A slot whose node is -2 / -3 is being published / was poisoned by an insert (lk_insert.cuh); both are negative, so
// the probe treats them as "end of the chain" — the persistent kernel only probes between inserts, never during one.
template <bool COH = false>
__device__ __forceinline__ int resolve_pair(const HashSlot* __restrict__ slots, uint32_t mask, uint32_t i, SlotPair p,
                                            int kx, int ky, int kz) {
    // first step may start on the odd slot of its pair
    if ((i & 1u) == 0) {
        if (p.a.w < 0) return -1;
        if (p.a.x == kx && p.a.y == ky && p.a.z == kz) return p.a.w;
    }
    if (p.b.w < 0) return -1;
    if (p.b.x == kx && p.b.y == ky && p.b.z == kz) return p.b.w;
    uint32_t j = ((i & ~1u) + 2) & mask;
    for (uint32_t probes = 0;; ++probes) {
        if (probes > mask) {  // walked the whole table without meeting an empty slot (see lk_stall_note)
            stall_note(4u, i);
            return -1;
        }
        p = load_pair<COH>(slots, j);
        if (p.a.w < 0) return -1;
        if (p.a.x == kx && p.a.y == ky && p.a.z == kz) return p.a.w;
        if (p.b.w < 0) return -1;
        if (p.b.x == kx && p.b.y == ky && p.b.z == kz) return p.b.w;
        j = (j + 2) & mask;
    }
}

template <int NTHREADS, class PS>
__device__ __forceinline__ bool fallback_pick(const PS* ps, uint32_t& fb_slot) {
    uint32_t n_fb = 0, k = threadIdx.x;
    bool found = false;
#pragma unroll
    for (int w = 0; w < NTHREADS / 32; ++w) {
        const uint32_t c = ps->wcnt[w];
        if (!found && k < c) { fb_slot = (uint32_t)w * 32u + k; found = true; }
        if (!found) k -= c;
        n_fb += c;
    }
    return threadIdx.x < n_fb;
}

// One root through build_single_residual (voxel_map.cc:363-427) from its staged hot image: the plane decides, or, when
// the root holds no plane, the descent into its children.
template <bool COH = false>
__device__ __forceinline__ bool eval_root(const MapNode* __restrict__ nodes, int root, const unsigned char* slot, const PointCtx& pc,
                                          const ScanConst& sc, const Globals& g, Row& row) {
    const int rc = eval_plane_hot(slot, pc, sc, g, row);
    if (rc != 1) return rc == 0;
    return eval_descent<COH>(nodes, root, pc, sc, g, row);
}

// One root from its staged slot, in the form HOT selects.
template <bool COH, bool HOT>
__device__ __forceinline__ bool eval_staged(const MapNode* __restrict__ nodes, int root, const unsigned char* slot, const PointCtx& pc,
                                            const ScanConst& sc, const Globals& g, Row& row) {
    if constexpr (HOT) {
        return eval_root<COH>(nodes, root, slot, pc, sc, g, row);
    } else {
        PlaneRec r;
        plane_from_smem(slot, r);
        return eval_record<COH>(nodes, r, pc, sc, g, row);
    }
}

// =================================================================================================
// The block-wide pass. In the fused per-scan kernel a block keeps one chunk, so a lane sees the same point in every
// iteration of a bucket: the lane keeps everything that does not depend on the state, plus the last voxel key with its
// lookup results; BOTH candidate records — the home voxel's and the one neighbour voxel's the reference falls back to
// (KILO.cc:156-178) — are staged into shared memory by TMA bulk copies issued together, and stay there: when the key
// is unchanged in a later iteration (the map is static within a bucket) the probes AND the gathers are skipped, and
// the fallback round reads its record from shared memory instead of paying another dependent global round trip.
// A kernel that sees each point once starts every pass with a fresh LaneCache (have = 0).
// =================================================================================================
struct LaneCache {
    double pbx, pby, pbz, pix, piy, piz, r2, range2;
    int kx, ky, kz, nx, ny, nz, root, near;
    int have;  // 0 = nothing cached, 1 = point quantities cached, 2 = + keys / root / near / staged records
};

template <int NTHREADS, bool HOT>
struct PassSmem {
    static constexpr int STRIDE = Stage<HOT>::STRIDE;
    __align__(16) unsigned char tile[2][NTHREADS * STRIDE];  // [0] home roots, [1] neighbour roots (Stage<HOT>)
    // Every lane's point context of the current pass. The evaluations read it from here and the descent receives its
    // address, so it never lives in the stack frame (which the L1 left beside this much shared memory cannot hold: every
    // access would go to L2); the fallback round reads the failing lane's context in place, without a copy.
    PointCtx pt[NTHREADS];
    struct __align__(8) Fallback {
        int near;      // the neighbour root (its node record, should a descent be needed)
        uint32_t idx;  // the failing lane: its context is pt[idx], its neighbour's staged slot tile[1] slot idx
    } fb[NTHREADS];
    uint64_t bar[NTHREADS / 32];
    uint32_t wcnt[NTHREADS / 32];
};

template <class PS>
__device__ __forceinline__ void pass_init(PS* ps) {
    const int tid = threadIdx.x;
    if ((tid & 31) == 0) mbar_init(&ps->bar[tid >> 5], 1);
    mbar_init_fence();
    __syncthreads();
}

// `phase` is the warp's mbarrier parity (start at 0, carried between passes). Every row goes to sink(idx, row), `idx` being
// the thread that holds the point: a thread passes its own home row, then the fallback row it evaluated for another
// thread. Both calls follow both evaluations, so nothing the sink keeps (the accumulators) is live across an evaluation.
template <int NTHREADS, bool COH = false, bool HOT, class Sink>
__device__ __forceinline__ void points_pass(PassSmem<NTHREADS, HOT>* ps, uint32_t& phase, uint32_t count, const ScanConst& sc,
                                            const MapView& mv, const Globals& g, LaneCache& lc, float4 pre, Sink sink) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool active = (uint32_t)tid < count;
    PointCtx& pc = ps->pt[tid];
    int root = -1, near = -1;
    bool gather_home = false, gather_near = false;
    if (active) {
        if (lc.have == 0) {
            body_point(pre, g, lc);
            lc.have = 1;
        }
        pc.pbx = lc.pbx; pc.pby = lc.pby; pc.pbz = lc.pbz; pc.pix = lc.pix; pc.piy = lc.piy; pc.piz = lc.piz;
        pc.r2 = lc.r2; pc.range2 = lc.range2;
        world_point(pc, sc);
        float lx, ly, lz;
        voxel_loc(pc, g, lx, ly, lz);
        const int kx = (int)lx, ky = (int)ly, kz = (int)lz;
        int nx, ny, nz;
        neighbour_key(g, lx, ly, lz, kx, ky, kz, nx, ny, nz);
        const bool differs = (nx != kx) || (ny != ky) || (nz != kz);
        const bool same_home = lc.have == 2 && lc.kx == kx && lc.ky == ky && lc.kz == kz;
        if (same_home) {
            root = lc.root;
            near = lc.near;
            if (lc.nx != nx || lc.ny != ny || lc.nz != nz) {  // same home voxel, different neighbour: redo that lookup only
                const uint32_t in = hash_key(nx, ny, nz) & mv.hash_mask;
                near = (root >= 0 && differs) ? resolve_pair<COH>(mv.slots, mv.hash_mask, in, load_pair<COH>(mv.slots, in), nx, ny, nz) : -1;
                gather_near = near >= 0;
            }
        } else {
            // both home pairs are read before either is inspected
            const uint32_t ih = hash_key(kx, ky, kz) & mv.hash_mask, in = hash_key(nx, ny, nz) & mv.hash_mask;
            const SlotPair sh = load_pair<COH>(mv.slots, ih);
            const SlotPair sn = load_pair<COH>(mv.slots, in);
            root = resolve_pair<COH>(mv.slots, mv.hash_mask, ih, sh, kx, ky, kz);
            // the reference only looks at the neighbour when the home voxel exists
            near = (root >= 0 && differs) ? resolve_pair<COH>(mv.slots, mv.hash_mask, in, sn, nx, ny, nz) : -1;
            gather_home = root >= 0;
            gather_near = near >= 0;
        }
        lc.kx = kx; lc.ky = ky; lc.kz = kz; lc.nx = nx; lc.ny = ny; lc.nz = nz;
        lc.root = root; lc.near = near;
        lc.have = 2;
    }
    // ---- stage the roots: one bulk copy per lane and root ---------------------------------------
    constexpr uint32_t BYTES = Stage<HOT>::BYTES;
    unsigned char* home_slot = ps->tile[0] + (size_t)tid * ps->STRIDE;
    unsigned char* near_slot = ps->tile[1] + (size_t)tid * ps->STRIDE;
    auto src = [&](int r) -> const void* {
        if constexpr (HOT) return mv.hot + r;
        else return mv.nodes + r;
    };
    const uint32_t vh = __ballot_sync(0xffffffffu, gather_home), vn = __ballot_sync(0xffffffffu, gather_near);
    if (vh | vn) {
        if (lane == 0) mbar_expect_tx(&ps->bar[warp], BYTES * (uint32_t)(__popc(vh) + __popc(vn)));
        __syncwarp();
        if (gather_home) bulk_g2s(home_slot, src(root), BYTES, &ps->bar[warp]);
        if (gather_near) bulk_g2s(near_slot, src(near), BYTES, &ps->bar[warp]);
        mbar_wait(&ps->bar[warp], phase);
        phase ^= 1u;
    }
    // ---- gates + row -----------------------------------------------------------------------------
    Row row;
    bool ok = false;
    if (root >= 0) ok = eval_staged<COH, HOT>(mv.nodes, root, home_slot, pc, sc, g, row);
    {  // the failing points, listed per warp in lane order (no atomics: the order, hence the sums, are reproducible); entry
       // `tid` of the warp-major concatenation of the lists is handled by thread `tid`; their contexts stay in pt
        const bool want = root >= 0 && !ok && near >= 0;
        const uint32_t m = __ballot_sync(0xffffffffu, want);
        if (lane == 0) ps->wcnt[warp] = (uint32_t)__popc(m);
        if (want) {
            auto& f = ps->fb[(uint32_t)warp * 32u + (uint32_t)__popc(m & ((1u << lane) - 1u))];
            f.near = near;
            f.idx = (uint32_t)tid;
        }
    }
    __syncthreads();
    // ---- fallback round: the neighbour voxel of the points that failed at home, already staged -------
    uint32_t fb_slot = 0, idx = 0;
    Row row2;
    bool ok2 = false;
    if (fallback_pick<NTHREADS>(ps, fb_slot)) {
        const auto f = ps->fb[fb_slot];
        idx = f.idx;
        ok2 = eval_staged<COH, HOT>(mv.nodes, f.near, ps->tile[1] + (size_t)idx * ps->STRIDE, ps->pt[idx], sc, g, row2);
    }
    if (ok) sink((uint32_t)tid, row);
    if (ok2) sink(idx, row2);
    __syncthreads();  // the fallback list is rewritten by the next pass
}

}  // namespace lk
