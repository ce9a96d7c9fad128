// lk_stream2.cu — throughput family of the residual pass (calls with >= 2 scans), two kernels per iteration:
//
// k_residual_stream2: every warp streams its 32-point groups of the block's chunk through a 3-deep software pipeline
//     points(i+3) | key + root-table probe(i+2) | hot-record gather(i+1) -> shared stage | gates + row(i)
// so that, while a group is evaluated from shared memory (voxel_map.cc:363-411, KILO.cc:187-210), the next group's 32 hot
// plane images (lk_device.cuh: HotRec, 144 bytes each) are already in flight (11 cooperative 16-byte async-copy instructions, three
// records each) and the one after has its probe and its points in flight. The 21 terms of A = sum h^T h / R accumulate in shared
// memory, one column per thread. 6 warps x 2 stages per block, 2 blocks per SM, 132 registers, no spills. Points the hot image
// cannot finish — no plane in the home node, or gated out by it — are appended per chunk and warp, in ballot order, to a list in
// global memory.
//
// k_residual_fallback: one block per chunk finishes that list with the full reference sequence (home octree descent, then the ONE
// neighbour voxel, KILO.cc:156-178) — or only the neighbour half when the list entry says a home plane gated the point out — in
// the warp-major order of the lists, and adds its sums to the chunk's partial row. Deterministic order in both kernels, so the
// per-chunk sums are bitwise reproducible and do not depend on how a batch is sharded.
//
// One partial row per chunk; the per-scan solve follows as its own kernel (lk_residual.cu: k_scan_tail).
#include <algorithm>

#include "lk_kernels.h"
#include "lk_pass.cuh"

namespace lk {

namespace {

constexpr int S2_MAXPTS = 4096;  // largest chunk lk_api.cu hands out (3 840 = 6 warps x 20 groups)
// slot of a lane: the 144 used bytes of the plane's hot image (lk_device.cuh: HotRec) | root index at 144 | point at 160.
// 176-byte stride = 11 x 16 B: the 128-bit reads of 8 consecutive lanes fall into 8 disjoint groups of 4 banks.
constexpr int S2_STRIDE = 176, S2_SLOT_ROOT = 144, S2_SLOT_PT = 160, S2_REC_PIECES = 9;
constexpr int S2_STAGE_BYTES = 32 * S2_STRIDE;

struct Probe {  // what stage B leaves for stage C
    float4 pt;
    SlotPair pair;
    int kx, ky, kz;
    uint32_t ih;
};

template <int S2_WARPS>
struct S2Smem {
    static constexpr int FB_CAP = ((S2_MAXPTS / 32 + S2_WARPS - 1) / S2_WARPS) * 32;
    static_assert(S2_WARPS == (int)S2_FB_WARPS && FB_CAP == (int)S2_FB_CAP && S2_MAXPTS <= 0x8000, "fallback list layout (lk_kernels.h)");
    __align__(16) unsigned char st[S2_WARPS][2][S2_STAGE_BYTES];
    double slice[S2_WARPS * 32];
    // A = sum h^T h / R (21 terms) of every thread, [term][thread]: at 168 registers the compiler kept these in local memory,
    // whose footprint (two blocks x 192 threads) does not fit the 28 KB of L1 left beside the stages — every reload was an L2
    // round trip. Conflict-free 8-byte accesses, no synchronisation: a thread owns its column.
    double accA[21][S2_WARPS * 32];
    ScanConst sc;
};
static_assert(2 * (sizeof(S2Smem<6>) + 1024) <= 228 * 1024, "two blocks per SM");

__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait_group() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// One warp instruction of the cooperative gather: the hot images of lanes 3*JJ .. 3*JJ+2, nine 16-byte pieces each
// (lanes 0-8, 9-17, 18-26; lanes 27-31 idle). r >= thr with thr = 0 for a copying lane and INT_MAX for an idle one:
// one predicate, one wide multiply-add for the source address, one predicated copy.
template <int JJ>
__device__ __forceinline__ void gather_triple(int r, const unsigned char* hot_sub, uint32_t dst0, int thr) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t.reg .b64 a;\n\t"
        "setp.ge.s32 p, %0, %3;\n\t"
        "mad.wide.u32 a, %0, 160, %1;\n\t"
        "@p cp.async.cg.shared.global [%2+%4], [a], 16;\n\t}" ::"r"(r),
        "l"(hot_sub), "r"(dst0), "r"(thr), "n"(JJ * 3 * S2_STRIDE)
        : "memory");
}

// accumulate_row (lk_pass.cuh) with the 21 terms of A in shared memory: same products, same order, same contraction.
template <int NT>
__device__ __forceinline__ void accumulate_row_sm(const Row& row, double* colA, double (&rest)[8]) {
    const double w = 1.0 / row.R;
    int q = 0;
#pragma unroll
    for (int r = 0; r < 6; ++r) {
        const double hw = row.h[r] * w;
#pragma unroll
        for (int c = r; c < 6; ++c) {
            colA[q * NT] += hw * row.h[c];
            ++q;
        }
        rest[r] += hw * row.z;
    }
    rest[6] += row.R;
    rest[7] += 1.0;
}

template <int S2_THREADS>
__global__ void __launch_bounds__(S2_THREADS, 2) k_residual_stream2(const __grid_constant__ ResidualArgs a) {
    constexpr int S2_WARPS = S2_THREADS / 32;
    extern __shared__ __align__(16) unsigned char s_raw[];
    S2Smem<S2_WARPS>* sm = reinterpret_cast<S2Smem<S2_WARPS>*>(s_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const ChunkDesc cd = a.chunks[a.chunk_first + blockIdx.x];
    load_scan_const(&sm->sc, a.sc + cd.scan);
    __syncthreads();
    const ScanConst& sc = sm->sc;
    const MapView mv = {a.slots, a.hash_mask, a.nodes, a.hot};
    const Globals& g = a.g;
    const float4* __restrict__ pts = a.pts + cd.start;
    const uint32_t count = cd.count;

    const int third = lane / S2_REC_PIECES, sub = lane % S2_REC_PIECES;  // third == 3: lanes 27-31 never copy
    const uint32_t st_base = smem_u32(&sm->st[warp][0][0]);
    const uint32_t slot_off = (uint32_t)lane * S2_STRIDE;
    const uint32_t copy_off = (uint32_t)(third % 3) * S2_STRIDE + (uint32_t)sub * 16u;
    const unsigned char* hot_sub = reinterpret_cast<const unsigned char*>(a.hot) + sub * 16;
    const int thr = third < 3 ? 0 : 0x7fffffff;
    const int thr_last = third < 2 ? 0 : 0x7fffffff;  // the 11th instruction carries lanes 30, 31 only

    double* colA = &sm->accA[0][tid];
#pragma unroll
    for (int i = 0; i < 21; ++i) colA[i * S2_THREADS] = 0.0;
    double rest[8];  // b (6) | sum R | count
#pragma unroll
    for (int i = 0; i < 8; ++i) rest[i] = 0.0;
    uint32_t nfbw = 0;
    // this warp's list of points to finish with the full reference sequence (k_residual_fallback), in ballot order
    uint16_t* fbw = a.fb_list + ((size_t)(a.chunk_first + blockIdx.x) * S2_FB_WARPS + (uint32_t)warp) * S2_FB_CAP;

    // group i of this warp starts at point (warp + i * S2_WARPS) * 32
    auto first_of = [&](uint32_t i) { return ((uint32_t)warp + i * (uint32_t)S2_WARPS) * 32u; };
    auto stage_A = [&](uint32_t i) {  // points
        const uint32_t p = first_of(i) + (uint32_t)lane;
        return p < count ? __ldg(pts + p) : make_float4(0.f, 0.f, 0.f, 0.f);
    };
    auto stage_B = [&](uint32_t i, float4 pt, Probe& pr) {  // key + probe
        pr.pt = pt;
        if (first_of(i) + (uint32_t)lane < count) {
            PointCtx pc;
            float lx, ly, lz;
            prepare_point(pt, sc, g, pc, lx, ly, lz);
            pr.kx = (int)lx; pr.ky = (int)ly; pr.kz = (int)lz;
            pr.ih = hash_key(pr.kx, pr.ky, pr.kz) & mv.hash_mask;
            pr.pair = load_pair(mv.slots, pr.ih);
        }
    };
    auto stage_C = [&](uint32_t i, const Probe& pr) {  // root -> gather into stage i & 1 (always commits a group)
        if (first_of(i) < count) {
            int root = -1;
            if (first_of(i) + (uint32_t)lane < count) root = resolve_pair(mv.slots, mv.hash_mask, pr.ih, pr.pair, pr.kx, pr.ky, pr.kz);
            const uint32_t stage = st_base + (i & 1u) * (uint32_t)S2_STAGE_BYTES;
            asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(stage + slot_off + S2_SLOT_PT), "f"(pr.pt.x), "f"(pr.pt.y),
                         "f"(pr.pt.z), "f"(pr.pt.w) : "memory");
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(stage + slot_off + S2_SLOT_ROOT), "r"(root) : "memory");
            const uint32_t dst0 = stage + copy_off;
#define LK_G(JJ) gather_triple<JJ>(__shfl_sync(0xffffffffu, root, (3 * JJ + third) & 31), hot_sub, dst0, (JJ) == 10 ? thr_last : thr);
            LK_G(0) LK_G(1) LK_G(2) LK_G(3) LK_G(4) LK_G(5) LK_G(6) LK_G(7) LK_G(8) LK_G(9) LK_G(10)
#undef LK_G
        }
        cp_async_commit();
    };

    const uint32_t n_groups = (count + 31u) >> 5;
    const uint32_t n_mine = n_groups > (uint32_t)warp ? (n_groups - (uint32_t)warp + S2_WARPS - 1) / S2_WARPS : 0;
    // prologue
    Probe pr_c, pr_b;  // pr_c: probed, next to gather; pr_b: being probed
    pr_c.pair.a = make_int4(0, 0, 0, -1); pr_c.pair.b = pr_c.pair.a; pr_c.kx = pr_c.ky = pr_c.kz = 0; pr_c.ih = 0;
    pr_c.pt = make_float4(0.f, 0.f, 0.f, 0.f);
    pr_b = pr_c;
    float4 pt_a;
    {
        stage_B(0, stage_A(0), pr_c);
        pt_a = stage_A(1);
        stage_C(0, pr_c);            // gather(0) in flight
        stage_B(1, pt_a, pr_c);      // probe(1) in flight
        pt_a = stage_A(2);           // points(2) in flight
    }
    for (uint32_t i = 0; i < n_mine; ++i) {
        stage_C(i + 1, pr_c);             // gather(i+1) -> the other stage (its previous reader finished last round)
        stage_B(i + 2, pt_a, pr_b);       // probe(i+2)
        pt_a = stage_A(i + 3);            // points(i+3)
        cp_async_wait_group<1>();         // gather(i) has landed (this lane's copies) ...
        __syncwarp();                     // ... and everybody else's
        {
            const unsigned char* slot = &sm->st[warp][i & 1u][0] + (size_t)lane * S2_STRIDE;
            const int root = *reinterpret_cast<const int*>(slot + S2_SLOT_ROOT);
            bool fail = false;
            int why = 0;
            if (root >= 0) {
                const float4 pt = *reinterpret_cast<const float4*>(slot + S2_SLOT_PT);
                PointCtx pc;
                float lx, ly, lz;
                prepare_point(pt, sc, g, pc, lx, ly, lz);
                Row row;
                const int rc = eval_plane_hot(slot, pc, sc, g, row);
                if (rc == 0) accumulate_row_sm<S2_THREADS>(row, colA, rest);
                else { fail = true; why = rc; }  // finished by k_residual_fallback
            }
            const uint32_t m = __ballot_sync(0xffffffffu, fail);
            if (fail) fbw[nfbw + __popc(m & ((1u << lane) - 1u))] = (uint16_t)((first_of(i) + (uint32_t)lane) | (why == 2 ? 0x8000u : 0u));
            nfbw += __popc(m);
        }
        __syncwarp();  // the stage is rewritten by the gather issued next round
        pr_c = pr_b;
    }
    cp_async_wait_group<0>();
    if (lane == 0) a.fb_cnt[(size_t)(a.chunk_first + blockIdx.x) * S2_FB_WARPS + (uint32_t)warp] = nfbw;
    // register image for the reduction (layout of lk_device.cuh: A | b | sum R | count)
    double acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.0;
#pragma unroll
    for (int i = 0; i < 21; ++i) acc[i] = colA[i * S2_THREADS];
#pragma unroll
    for (int i = 0; i < 6; ++i) acc[ACC_B + i] = rest[i];
    acc[ACC_SUMR] = rest[6];
    acc[ACC_CNT] = rest[7];
    block_row<S2_WARPS>(acc, sm->slice, [&](int i, double v) { a.partial[(size_t)(a.chunk_first + blockIdx.x) * PARTIAL_STRIDE + i] = v; });
}

// The points the pipelined kernel could not finish on the hot images — no plane in the home node (octree descent, voxel_map.cc:412-424)
// or gated out at home (then the one neighbour voxel, KILO.cc:156-178) — with the full reference sequence (point_row), one block
// per chunk, entry e of the warp-major concatenation of the chunk's lists on thread e. A chain of dependent cold reads per point:
// it wants many points in flight and few registers live, which is why it is its own kernel (inside the pipelined kernel it held
// the warps of the pipeline at its long-latency loads). Adds its sums to the chunk's partial row: same stream, after the kernel that wrote the row.
// The second half of KILO.cc:154-178 alone: the ONE neighbour voxel, for a point whose home voxel is known to have failed.
__device__ __forceinline__ bool point_row_neighbour(float4 pt, const ScanConst& sc, const MapView& mv, const Globals& g, Row& row) {
    PointCtx pc;
    float lx, ly, lz;
    prepare_point(pt, sc, g, pc, lx, ly, lz);
    const int kx = (int)lx, ky = (int)ly, kz = (int)lz;
    int nx, ny, nz;
    neighbour_key(g, lx, ly, lz, kx, ky, kz, nx, ny, nz);
    if (nx == kx && ny == ky && nz == kz) return false;  // the same voxel again: the same failure
    const int root = map_find(mv.slots, mv.hash_mask, nx, ny, nz);
    if (root < 0) return false;
    // a plane in the neighbour root (the common case): its hot image decides, as in the pipelined kernel; otherwise the descent
    return eval_root(mv.nodes, root, reinterpret_cast<const unsigned char*>(mv.hot + root), pc, sc, g, row);
}

constexpr int FB_THREADS = 128;
__global__ void __launch_bounds__(FB_THREADS, 8) k_residual_fallback(const __grid_constant__ ResidualArgs a) {
    __shared__ ScanConst s_sc;
    __shared__ double s_slice[(FB_THREADS / 32) * 32];
    const int tid = threadIdx.x;
    const uint32_t c = a.chunk_first + blockIdx.x;
    uint32_t cnt[S2_FB_WARPS], total = 0;
#pragma unroll
    for (uint32_t w = 0; w < S2_FB_WARPS; ++w) { cnt[w] = __ldg(a.fb_cnt + (size_t)c * S2_FB_WARPS + w); total += cnt[w]; }
    if (total == 0) return;  // the same for every thread of the block
    const ChunkDesc cd = a.chunks[c];
    load_scan_const(&s_sc, a.sc + cd.scan);
    __syncthreads();
    const MapView mv = {a.slots, a.hash_mask, a.nodes, a.hot};
    const float4* __restrict__ pts = a.pts + cd.start;
    double acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.0;
    for (uint32_t e = (uint32_t)tid; e < total; e += FB_THREADS) {
        uint32_t k = e, w2 = 0;
#pragma unroll
        for (uint32_t t = 0; t < S2_FB_WARPS - 1; ++t)
            if (w2 == t && k >= cnt[t]) { k -= cnt[t]; w2 = t + 1; }
        const uint32_t ent = __ldg(a.fb_list + ((size_t)c * S2_FB_WARPS + w2) * S2_FB_CAP + k);
        const float4 pt = __ldg(pts + (ent & 0x7fffu));
        Row row;
        // bit 15: the home voxel is a plane that gated the point out — build_single_residual left is_success false there
        // (voxel_map.cc:370-411), so only the neighbour voxel is left to try; otherwise the whole sequence, descent included
        const bool ok = (ent & 0x8000u) ? point_row_neighbour(pt, s_sc, mv, a.g, row) : point_row(pt, s_sc, mv, a.g, row);
        if (ok) accumulate_row(row, acc);
    }
    block_row<FB_THREADS / 32>(acc, s_slice, [&](int i, double v) { a.partial[(size_t)c * PARTIAL_STRIDE + i] += v; });
}

}  // namespace

void launch_residual_stream2(const ResidualArgs& a, uint32_t n_chunks, cudaStream_t s) {
    if (n_chunks == 0) return;
    static PerDeviceOnce once;
    if (once.first()) {
        cudaFuncSetAttribute(k_residual_stream2<192>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(S2Smem<6>));
        cudaFuncSetAttribute(k_residual_stream2<192>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    }
    k_residual_stream2<192><<<n_chunks, 192, sizeof(S2Smem<6>), s>>>(a);
}

void launch_residual_fallback(const ResidualArgs& a, uint32_t n_chunks, cudaStream_t s) {
    if (n_chunks == 0) return;
    k_residual_fallback<<<n_chunks, FB_THREADS, 0, s>>>(a);
}

}  // namespace lk
