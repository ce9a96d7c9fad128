// lk_llsync.cuh — grid-wide all-reduce of one 32-double row per block WITHOUT a barrier: rows travel
// through global memory in a flagged ("low-latency") format — every double is split into two 8-byte
// words {low 32 bits | tag << 32, high 32 bits | tag << 32} stored with ONE 16-byte store. Aligned 8-byte
// stores are single-copy atomic, so a reader that finds the expected tag in both words holds the whole
// value: data and "ready" flag arrive together, there is no release fence, no counter and no second
// round trip to read the rows after a barrier. The tag is a per-handle epoch that grows with every
// (launch, iteration), so stale rows of earlier iterations never match; two buffers alternate by
// iteration parity (a block writes iteration i+2 only after it has seen every row of iteration i+1,
// i.e. after every block has finished reading iteration i).
//
// Who reads. Warp 0 of a block stores its rows; every warp of the block polls a share of the rows it needs
// (ll_poll_rows: row k to warp k % warps), keeps each element it has matched in shared memory and does not load that
// row again, and may have a second poll round in flight while it inspects the first. A word is accepted only when both
// halves carry this exchange's tag, so neither the number of reading warps nor a load that was issued a round earlier can
// make a reader accept a word of the buffer's next use: exchange i+2 of the same buffer writes tag + 2, which never
// matches, whenever the load happens to be performed. A load whose round is never inspected (the warp matched everything
// from the other round) is simply dropped. The block's reads of exchange i end at the block barrier that follows every
// warp's poll; only after it does warp 0 add the rows, and every later store of the block (its chunk row of i+1, a
// leader's group row of i+1 or i+2, a finisher's acknowledgement of i) comes after that barrier in program order.
//
// Every group row is published in LL_REPLICAS copies, and block b polls only copy b % LL_REPLICAS, so
// each copy's lines have ~blocks / LL_REPLICAS readers instead of all of them. The reuse rule above holds
// for every copy, for every block that publishes a chunk row in exchange i+1: a leader writes all copies of
// its group row of i+2 at one point of its program, after the barrier that ends its reads (in its own copy) of every
// group row of i+1; each of those exists only once its group's leader has seen every chunk row of that group for i+1,
// and a block publishes its chunk row of i+1 only after the barrier that ends all its warps' reads of its copy of every
// group row of i. The chain runs through block barriers as well as through each block's warp 0, and a barrier orders
// the other warps' completed loads before warp 0's later stores just as program order orders warp 0's own. Which copy
// a block reads plays no part in that chain. A block with b >= n_chunks of exchange i+1 publishes nothing
// there, so the chain does not order its reads of i before the writes of i+2; it only holds because such a
// block would have to lag a whole pass and solve behind the others. This is as old as the two buffers.
//
// Finishers (lk_fused.cu) are such blocks, made safe by construction: they read a copy of the group rows of
// their own (copy LL_REPLICAS, written only when the launch has finishers) and, after the barrier that ends every warp's
// reads of exchange i, store an acknowledgement word tagged i with release semantics; a leader of exchange i+2 polls
// those words with acquire loads before it writes its group row. A finisher takes the LAST exchange of its launch straight
// from the chunk rows (ll_sum_chunk_rows), which every block then publishes, leaders included; nothing writes rows after
// it within the launch, and the next launch writes rows only behind griddepcontrol.wait.
//
// Summation order (shared with the multi-kernel path, lk_solve.cuh: block_sum_partials):
//   total = sum over groups g ascending of ( sum over the rows of group g ascending ),
//   group g = chunks [g*LK_GROUP, (g+1)*LK_GROUP) of the bucket — a function of the bucket alone.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "lk_async.cuh"

namespace lk {

constexpr int LK_GROUP = 8;          // chunk rows per group (level-1 fan-in)
constexpr int LL_ROW = 32;           // slots (doubles) per row
constexpr int LL_MAX_CHUNKS = 160;   // >= SM count: the fused kernel runs one chunk per block
constexpr int LL_MAX_GROUPS = (LL_MAX_CHUNKS + LK_GROUP - 1) / LK_GROUP;
constexpr int LL_REPLICAS = 4;       // copies of every group row (level-2 readers per copy: blocks / LL_REPLICAS)
constexpr int LL_COPIES = LL_REPLICAS + 1;  // + the finishers' copy
constexpr int LL_MAX_FINISHERS = 24;  // one acknowledgement word per finisher, polled one per lane

struct LLView {
    ulonglong2* chunk_rows;  // [2][LL_MAX_CHUNKS][LL_ROW]
    ulonglong2* group_rows;  // [2][LL_COPIES][LL_MAX_GROUPS][LL_ROW]
    uint32_t* stall;         // [8] watchdog record: [0] != 0 once a poll gave up | block | tag | first row | rows | lane
    uint32_t* acks;          // [2][LL_MAX_FINISHERS] tag of the last exchange each finisher has read
};
constexpr size_t LL_ROWS_BYTES = (size_t)2 * (LL_MAX_CHUNKS + LL_COPIES * LL_MAX_GROUPS) * LL_ROW * sizeof(ulonglong2);
constexpr size_t LL_BYTES = LL_ROWS_BYTES + 64 + 2 * LL_MAX_FINISHERS * sizeof(uint32_t);
// A poll that sees nothing for this many rounds (seconds) gives up, records who waited for what and lets the kernel run
// to its end with garbage sums; the host then reports LK_ERR_CUDA instead of hanging. It means the blocks of the grid were
// not all resident (another process holds SMs: see INTEGRATION.md "Sharing a device") — or a bug.
constexpr uint32_t LL_SPIN_LIMIT = 1u << 23;
// Slots per exchange of the optional hop trace (ll_allreduce's `hops`): [0] own chunk row stored (a leader: level 1 entered),
// [1] level-1 sum complete (leader), [2] group row stored (leader), [3] total in hand, [4] poll rounds: level 1 | level 2 << 32
constexpr int LL_HOP_SLOTS = 5;
// Shared-memory scratch of ll_allreduce, in doubles: the level-1 rows (LK_GROUP), the level-2 rows (LL_MAX_GROUPS), and
// 32 more for the hop trace's per-warp round counts.
constexpr int LL_XS = (LK_GROUP + LL_MAX_GROUPS + 1) * 32;
// Poll rounds a warp keeps in flight (ll_poll_rows); `make POLL_DEPTH=2` builds the other depth for comparison.
#ifndef LL_POLL_DEPTH
#define LL_POLL_DEPTH 1
#endif

__device__ __forceinline__ void ll_store(ulonglong2* p, double v, uint32_t tag) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(v);
    const unsigned long long t = (unsigned long long)tag << 32;
    const unsigned long long w0 = (b & 0xffffffffull) | t, w1 = (b >> 32) | t;
    asm volatile("st.relaxed.gpu.global.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(w0), "l"(w1) : "memory");
}

// Gives up a poll: records who waited for what (the first to give up) so the host can report it.
__device__ __forceinline__ void ll_give_up(uint32_t* stall, uint32_t tag, uint32_t r0, uint32_t n, int lane) {
    if (atomicCAS(stall, 0u, 1u) == 0u) {
        stall[1] = blockIdx.x; stall[2] = tag; stall[3] = r0; stall[4] = n; stall[5] = (uint32_t)lane;
        __threadfence();
    }
}

// Element `lane` of rows [r0, r0 + n) (n <= N), summed in ascending row order starting from 0.0. Every poll round
// issues its loads back to back (independent, so they overlap in the memory system: one L2 round trip per round, not one
// per row) and only then inspects the tags. A row that matched keeps its words and is not loaded again (rows never change
// once published within an epoch), so a round loads only the rows still missing.
// SPLIT < N: two sums in one poll, rows [0, SPLIT) returned and rows [SPLIT, n) in *hi, each from 0.0 in ascending order.
// `rounds` receives the number of poll rounds. One full warp.
template <int N, int SPLIT = N>
__device__ __forceinline__ double ll_sum_rows(const ulonglong2* rows, uint32_t r0, uint32_t n, uint32_t tag, int lane,
                                              uint32_t* stall, uint32_t& rounds, double* hi = nullptr) {
    static_assert(N <= 32, "one bit per row");
    const ulonglong2* p = rows + (size_t)r0 * LL_ROW + lane;
    unsigned long long w0[N], w1[N];
    const unsigned long long want = ((unsigned long long)tag << 32);
    uint32_t spins = 0;
    uint32_t todo = n >= 32u ? 0xffffffffu : (1u << n) - 1u;  // rows not seen yet
    while (true) {
#pragma unroll
        for (int k = 0; k < N; ++k)
            if ((todo >> k) & 1u)
                asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(w0[k]), "=l"(w1[k]) : "l"(p + (size_t)k * LL_ROW));
#pragma unroll
        for (int k = 0; k < N; ++k)
            if (((todo >> k) & 1u) && ((w0[k] & 0xffffffff00000000ull) == want) && ((w1[k] & 0xffffffff00000000ull) == want))
                todo &= ~(1u << k);
        ++spins;
        if (todo == 0u) break;
        if ((spins & 0xfffu) == 0u) {  // watchdog, off the fast path
            if (spins >= LL_SPIN_LIMIT || *reinterpret_cast<volatile uint32_t*>(stall) != 0u) {
                ll_give_up(stall, tag, r0, n, lane);
                break;
            }
        }
    }
    rounds = spins;
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < SPLIT; ++k)
        if ((uint32_t)k < n) s += __longlong_as_double((long long)((w0[k] & 0xffffffffull) | (w1[k] << 32)));
    if constexpr (SPLIT < N) {
        double s2 = 0.0;
#pragma unroll
        for (int k = SPLIT; k < N; ++k)
            if ((uint32_t)k < n) s2 += __longlong_as_double((long long)((w0[k] & 0xffffffffull) | (w1[k] << 32)));
        *hi = s2;
    }
    return s;
}

// Rows [r0 + k0, r0 + n) polled by all NWARPS warps of the block: row r0 + k goes to warp k % NWARPS (at most RPW rows
// per warp, n <= NWARPS * RPW). As soon as both words of element `lane` of a row carry `tag`, the element goes to
// xs[k * 32 + lane] and the row is not loaded again. The caller reads xs after a block barrier. A round issues the loads of
// the warp's missing rows back to back and only then inspects them. DEPTH = 2 keeps two rounds in flight: after the first
// round, which also measures the round trip, the warp issues round k + 1 before it inspects round k, and starts the second
// round half a round trip after the first, so a row that lands just after one round's loads left is seen by the other
// about half a round trip later instead of a whole one. Returns this lane's poll rounds (inspections). All threads call.
template <int NWARPS, int RPW, int DEPTH>
__device__ __forceinline__ uint32_t ll_poll_rows(const ulonglong2* rows, uint32_t r0, uint32_t k0, uint32_t n, uint32_t tag,
                                                 uint32_t* stall, double* xs) {
    static_assert(DEPTH == 1 || DEPTH == 2, "one or two rounds in flight");
    static_assert(NWARPS * RPW <= 32 * 32, "rows per poll");
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const ulonglong2* p = rows + (size_t)(r0 + (uint32_t)warp) * LL_ROW + lane;
    const unsigned long long want = ((unsigned long long)tag << 32);
    uint32_t todo = 0;  // the warp's rows not seen yet: bit j is row warp + j * NWARPS
#pragma unroll
    for (int j = 0; j < RPW; ++j) {
        const uint32_t k = (uint32_t)(warp + j * NWARPS);
        if (k >= k0 && k < n) todo |= 1u << j;
    }
    if (todo == 0u) return 0u;
    unsigned long long a0[RPW], a1[RPW], b0[RPW], b1[RPW];
    auto issue = [&](unsigned long long* w0, unsigned long long* w1) {
#pragma unroll
        for (int j = 0; j < RPW; ++j)
            if ((todo >> j) & 1u)
                asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];"
                             : "=l"(w0[j]), "=l"(w1[j]) : "l"(p + (size_t)j * NWARPS * LL_ROW));
    };
    // every row still missing was loaded by the round being inspected: `todo` only shrinks, and a round loads all of it
    auto inspect = [&](const unsigned long long* w0, const unsigned long long* w1) {
#pragma unroll
        for (int j = 0; j < RPW; ++j)
            if (((todo >> j) & 1u) && ((w0[j] & 0xffffffff00000000ull) == want) && ((w1[j] & 0xffffffff00000000ull) == want)) {
                xs[(size_t)(warp + j * NWARPS) * 32 + lane] = __longlong_as_double((long long)((w0[j] & 0xffffffffull) | (w1[j] << 32)));
                todo &= ~(1u << j);
            }
    };
    uint32_t spins = 0;
    auto watchdog = [&]() -> bool {  // off the fast path
        if ((spins & 0xfffu) == 0u && (spins >= LL_SPIN_LIMIT || *reinterpret_cast<volatile uint32_t*>(stall) != 0u)) {
            ll_give_up(stall, tag, r0 + k0, n - k0, lane);
            return true;
        }
        return false;
    };
    if constexpr (DEPTH == 1) {
        while (true) {
            issue(a0, a1);
            inspect(a0, a1);
            ++spins;
            if (todo == 0u || watchdog()) break;
        }
    } else {
        const long long c0 = clock64();
        issue(a0, a1);
        inspect(a0, a1);
        ++spins;
        if (todo != 0u) {
            const long long c1 = clock64(), half = (c1 - c0) >> 1;
            issue(a0, a1);
            while (clock64() - c1 < half) {}
            while (true) {
                issue(b0, b1);
                inspect(a0, a1);
                ++spins;
                if (todo == 0u || watchdog()) break;
                issue(a0, a1);
                inspect(b0, b1);
                ++spins;
                if (todo == 0u || watchdog()) break;
            }
        }
    }
    return spins;
}

// Waits until finishers [0, fin) have acknowledged exchange `tag` (a group leader, before it rewrites the buffers that
// exchange used). One full warp, fin <= 32.
__device__ __forceinline__ void ll_wait_acks(const uint32_t* acks, uint32_t fin, uint32_t tag, int lane, uint32_t* stall) {
    uint32_t spins = 0;
    bool mine = (uint32_t)lane >= fin;
    while (!__all_sync(0xffffffffu, mine)) {
        if (!mine) {
            uint32_t w;
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(w) : "l"(acks + lane) : "memory");
            mine = w == tag;
        }
        if ((++spins & 0xfffu) == 0u && (spins >= LL_SPIN_LIMIT || *reinterpret_cast<volatile uint32_t*>(stall) != 0u)) {
            ll_give_up(stall, tag, 0, fin, lane);
            break;
        }
    }
}

// The all-reduce. All threads of the block call; `v` = this block's row element `lane`, read in warp 0 only. Block b owns
// chunk b of the n_chunks chunks of the bucket (blocks with b >= n_chunks contribute nothing but still receive the
// total). Returns, in warp 0, the total of element `lane` in the fixed grouped order (the other warps get 0.0). Level 1:
// rows travel through global memory in the flagged format, the group's first block (its leader) polls the group's other
// rows with one warp per row, and warp 0 adds them to its own; level 2: warp 0 publishes the group row in LL_REPLICAS
// copies, and every block polls its copy of the (<= 20) group rows with all its warps (ll_poll_rows); after a block
// barrier warp 0 adds them. Only warp 0 stores rows, so a caller that must order those stores (griddepcontrol.wait) does
// so in warp 0. `xs` is LL_XS doubles of shared memory the call may overwrite. `hops` (nullptr: no trace) receives
// LL_HOP_SLOTS stamps and counts. `fin` > 0: the launch has `fin` finishers, blocks n_chunks .. n_chunks + fin - 1;
// leaders also write the finishers' copy, and when `acks_due` (exchange tag - 2 is of this launch) first wait for every
// finisher to have read it.
template <int NWARPS, int DEPTH = LL_POLL_DEPTH>
__device__ __forceinline__ double ll_allreduce(const LLView& ll, uint32_t parity, uint32_t tag, uint32_t b, uint32_t n_chunks,
                                               double v, double* xs, unsigned long long* hops = nullptr, uint32_t fin = 0,
                                               bool acks_due = false) {
    static_assert(LK_GROUP <= NWARPS && 2 * NWARPS <= 64, "one level-1 row per warp; the round counts fit their slots");
    constexpr int RPW2 = (LL_MAX_GROUPS + NWARPS - 1) / NWARPS;  // level-2 rows per warp
    constexpr size_t COPY = (size_t)LL_MAX_GROUPS * LL_ROW;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    ulonglong2* crows = ll.chunk_rows + (size_t)parity * LL_MAX_CHUNKS * LL_ROW;
    ulonglong2* grows = ll.group_rows + (size_t)parity * LL_COPIES * COPY;
    uint32_t* acks = ll.acks + (size_t)parity * LL_MAX_FINISHERS;
    double* xs1 = xs;                      // level 1: element `lane` of the group's row k at xs1[k * 32 + lane], k >= 1
    double* xs2 = xs + LK_GROUP * 32;      // level 2: group row g at xs2[g * 32 + lane]
    uint32_t* rw = reinterpret_cast<uint32_t*>(xs + (LK_GROUP + LL_MAX_GROUPS) * 32);  // hop trace: rounds per warp
    const uint32_t n_groups = (n_chunks + LK_GROUP - 1) / LK_GROUP;
    uint32_t r1 = 0, r2 = 0;
    if (b < n_chunks) {
        if ((b % LK_GROUP) == 0) {
            if (hops && threadIdx.x == 0) hops[0] = gtime();
            const uint32_t n = min((uint32_t)LK_GROUP, n_chunks - b);
            r1 = ll_poll_rows<NWARPS, 1, DEPTH>(crows, b, 1, n, tag, ll.stall, xs1);
            __syncthreads();
            if (warp == 0) {
                double s = 0.0;
                s += v;
#pragma unroll
                for (uint32_t k = 1; k < (uint32_t)LK_GROUP; ++k)
                    if (k < n) s += xs1[k * 32 + lane];
                if (hops && lane == 0) hops[1] = gtime();
                ulonglong2* g = grows + (size_t)(b / LK_GROUP) * LL_ROW + lane;
                if (fin && acks_due) ll_wait_acks(acks, fin, tag - 2u, lane, ll.stall);
#pragma unroll
                for (int r = 0; r < LL_REPLICAS; ++r) ll_store(g + (size_t)r * COPY, s, tag);
                if (fin) ll_store(g + (size_t)LL_REPLICAS * COPY, s, tag);
                if (hops && lane == 0) hops[2] = gtime();
            }
        } else if (warp == 0) {
            ll_store(crows + (size_t)b * LL_ROW + lane, v, tag);
            if (hops && lane == 0) hops[0] = gtime();
        }
    }
    const bool finisher = fin && b >= n_chunks;
    r2 = ll_poll_rows<NWARPS, RPW2, DEPTH>(grows + (size_t)(finisher ? LL_REPLICAS : b % LL_REPLICAS) * COPY, 0, 0, n_groups, tag,
                                           ll.stall, xs2);
    if (hops) {
        r1 = __reduce_max_sync(0xffffffffu, r1);
        r2 = __reduce_max_sync(0xffffffffu, r2);
        if (lane == 0) {
            rw[2 * warp] = r1;
            rw[2 * warp + 1] = r2;
        }
    }
    __syncthreads();  // every warp's reads of this exchange are done, and its rows are in xs2
    double t = 0.0;
    if (warp == 0) {
        if (finisher && lane == 0) asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(acks + (b - n_chunks)), "r"(tag) : "memory");
        for (uint32_t g = 0; g < n_groups; ++g) t += xs2[g * 32 + lane];
        if (hops) {
            r1 = lane < NWARPS ? rw[2 * lane] : 0u;
            r2 = lane < NWARPS ? rw[2 * lane + 1] : 0u;
            r1 = __reduce_max_sync(0xffffffffu, r1);
            r2 = __reduce_max_sync(0xffffffffu, r2);
            if (lane == 0) {
                hops[3] = gtime();
                hops[4] = (unsigned long long)r1 | ((unsigned long long)r2 << 32);
            }
        }
    }
    return t;
}

// The last exchange of a launch with finishers, the worker side: block b < n_chunks publishes its chunk row (a leader
// too) and is done with the exchange. Warp 0 calls, all 32 lanes.
__device__ __forceinline__ void ll_publish_row(const LLView& ll, uint32_t parity, uint32_t tag, uint32_t b, double v, int lane) {
    ll_store(ll.chunk_rows + ((size_t)parity * LL_MAX_CHUNKS + b) * LL_ROW + lane, v, tag);
}

// The last exchange of a launch with finishers, the finisher side: the total of the n_chunks chunk rows in one hop, in
// the grouped order of ll_allreduce (each group summed from 0.0 in ascending row order, then the group sums in ascending
// order). Warp w polls the group pairs w, w + NWARPS, ... (groups 2p and 2p + 1: up to 2 * LK_GROUP consecutive rows) in
// one poll that keeps the rows it has seen, and stores the two group sums in gs[g * 32 + lane] (LL_MAX_GROUPS * 32
// doubles); result in out[0..31]. All threads of the block call. It keeps a poll of its own rather than ll_poll_rows:
// that one stages every row in shared memory, and up to LL_MAX_CHUNKS rows (40 KB) would take the room in which a
// finisher stages its re-projection inputs (lk_fused.cu: fused_finish).
template <int NWARPS>
__device__ __forceinline__ void ll_sum_chunk_rows(const LLView& ll, uint32_t parity, uint32_t tag, uint32_t n_chunks, double* gs,
                                                  double* out) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const ulonglong2* crows = ll.chunk_rows + (size_t)parity * LL_MAX_CHUNKS * LL_ROW;
    const uint32_t n_groups = (n_chunks + LK_GROUP - 1) / LK_GROUP;
    for (uint32_t g = 2u * (uint32_t)warp; g < n_groups; g += 2u * NWARPS) {
        uint32_t rounds;
        double hi;
        gs[g * 32 + lane] = ll_sum_rows<2 * LK_GROUP, LK_GROUP>(crows, g * LK_GROUP, min(2u * LK_GROUP, n_chunks - g * LK_GROUP),
                                                                 tag, lane, ll.stall, rounds, &hi);
        if (g + 1 < n_groups) gs[(g + 1) * 32 + lane] = hi;
    }
    __syncthreads();
    if (tid < 32) {
        double t = 0.0;
        for (uint32_t g = 0; g < n_groups; ++g) t += gs[g * 32 + tid];
        out[tid] = t;
    }
    __syncthreads();
}

}  // namespace lk
