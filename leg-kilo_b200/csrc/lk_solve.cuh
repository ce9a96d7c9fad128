// lk_solve.cuh — block-level pieces of ESKF::updateByPoints (eskf.cc:91-113) in information form,
// operating on a filter (state 36 + covariance 900 doubles) held in shared memory:
//   K = P H^T (H P H^T + R)^-1  ==  P[:,0:6] (I + A P66)^-1,  A = sum h^T h / R, b = sum h^T z / R
// (SURVEY §8a a8, Appendix A.5), followed by State::operator+= (eskf.cc:18-29) and, on the last
// iteration, P <- P - K H P[0:6,:] (no symmetrisation, as the reference).
#pragma once
#include "lk_llsync.cuh"
#include "lk_point.cuh"

namespace lk {

struct BlockFilter {
    double x[36];
    double P[900];
    double acc[32];   // reduced A (21) | b (6) | sumR | count
    double A[36];
    double M[36];
    double y[6];
    double W[36];
    double delta[30];
    double Prow[180];
    double KH[180];
};

// Deterministic sum of the per-chunk partial rows [c0, c1) in the grouped order every path shares (lk_llsync.cuh):
//   total = sum over groups g ascending of ( sum over the rows of group g ascending ), LK_GROUP rows per group.
// Warp w forms the sum of group g0 + w (all loads of a group issued before the first add), the group sums are then
// added in ascending order. `slice` must hold nwarps*32 doubles. Result in out[0..31]. All threads of the block call.
template <int NWARPS>
__device__ __forceinline__ void block_sum_partials(const double* partial, uint32_t c0, uint32_t c1, double* slice,
                                                   double* out) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t n = c1 - c0, ng = (n + LK_GROUP - 1) / LK_GROUP;
    double tot = 0.0;
    for (uint32_t g0 = 0; g0 < ng; g0 += NWARPS) {
        const uint32_t g = g0 + (uint32_t)warp;
        if (g < ng) {
            const uint32_t r0 = c0 + g * LK_GROUP, m = min((uint32_t)LK_GROUP, c1 - r0);
            const double* p = partial + (size_t)r0 * PARTIAL_STRIDE + lane;
            double v[LK_GROUP];
#pragma unroll
            for (int k = 0; k < LK_GROUP; ++k) v[k] = ((uint32_t)k < m) ? __ldcg(p + (size_t)k * PARTIAL_STRIDE) : 0.0;
            double s = 0.0;
#pragma unroll
            for (int k = 0; k < LK_GROUP; ++k)
                if ((uint32_t)k < m) s += v[k];
            slice[warp * 32 + lane] = s;
        }
        __syncthreads();
        if (tid < 32) {
#pragma unroll
            for (int w = 0; w < NWARPS; ++w)
                if (g0 + (uint32_t)w < ng) tot += slice[w * 32 + tid];
        }
        __syncthreads();
    }
    if (tid < 32) out[tid] = tot;
    __syncthreads();
}

// The state half of the update. f->acc holds the reduced sums. Returns the residual count. All threads call.
// Warp 0 carries the whole serial chain (A, M = I + A P66, Gauss-Jordan, delta, State (+)) with warp-level
// synchronisation only, and leaves W = M^-1 A in f->W for the covariance half; ends with a block barrier.
__device__ __forceinline__ uint32_t block_solve_state(BlockFilter* f, unsigned long long* clk = nullptr) {
#define LK_SC(i) do { if (clk && threadIdx.x == 0) clk[i] = (unsigned long long)clock64(); } while (0)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const double cnt = f->acc[ACC_CNT];
    LK_SC(0);
    if (cnt > 0.5) {
        if (warp == 0) {
            // N == 1 adds 1e-4 to S (eskf.cc:100)  <=>  weights scale by R / (R + 1e-4)
            const double scale = (cnt < 1.5) ? f->acc[ACC_SUMR] / (f->acc[ACC_SUMR] + 0.0001) : 1.0;
            // columns of [M | b | A], M = I + A P66, one per lane (0..12). Branch-free: every lane forms the six
            // scaled entries of row i of A from the packed upper triangle (compile-time indices, broadcast reads),
            // lanes 0..5 run the dot product with their column of P66, the others select.
            double Pc[6];
#pragma unroll
            for (int k = 0; k < 6; ++k) Pc[k] = f->P[k * 30 + (lane < 6 ? lane : 0)];
            LK_SC(1);
            double col[6];
#pragma unroll
            for (int i = 0; i < 6; ++i) {
                double ar[6];
#pragma unroll
                for (int k = 0; k < 6; ++k) {
                    const int r = i < k ? i : k, c = i < k ? k : i;
                    ar[k] = f->acc[r * 6 - r * (r - 1) / 2 + (c - r)] * scale;
                }
                double m = (i == lane) ? 1.0 : 0.0;
#pragma unroll
                for (int k = 0; k < 6; ++k) m += ar[k] * Pc[k];
                double asel = ar[0];
#pragma unroll
                for (int t = 1; t < 6; ++t) asel = (lane - 7 == t) ? ar[t] : asel;
                const double bsel = f->acc[ACC_B + i] * scale;
                col[i] = lane < 6 ? m : (lane == 6 ? bsel : (lane < 13 ? asel : 0.0));
            }
            LK_SC(2);
            const bool okl = warp_solve6(col, lane);
            LK_SC(3);
            double y[6];
#pragma unroll
            for (int i = 0; i < 6; ++i) {
                y[i] = __shfl_sync(0xffffffffu, okl ? col[i] : 0.0, 6);
                if (lane >= 7 && lane < 13) f->W[i * 6 + (lane - 7)] = okl ? col[i] : 0.0;
            }
            double d = 0.0;
            if (lane < 30) {
#pragma unroll
                for (int k = 0; k < 6; ++k) d += f->P[lane * 30 + k] * y[k];
            }
            LK_SC(4);
            // State::operator+= : Exp(delta_theta) is formed by every lane from the broadcast angles
            const double d0 = __shfl_sync(0xffffffffu, d, 0), d1 = __shfl_sync(0xffffffffu, d, 1),
                         d2 = __shfl_sync(0xffffffffu, d, 2);
            double rv = 0.0;
            if (lane < 9) {
                double E[9];
                so3_exp3(d0, d1, d2, E);
                // column j of E picked with compile-time indices: E indexed at run time would live in local memory
                const int i = lane / 3, j = lane % 3;
                const double e0 = j == 0 ? E[0] : (j == 1 ? E[1] : E[2]);
                const double e1 = j == 0 ? E[3] : (j == 1 ? E[4] : E[5]);
                const double e2 = j == 0 ? E[6] : (j == 1 ? E[7] : E[8]);
                rv = f->x[i * 3] * e0 + f->x[i * 3 + 1] * e1 + f->x[i * 3 + 2] * e2;
            }
            __syncwarp();
            if (lane < 9) f->x[lane] = rv;
            if (lane >= 3 && lane < 30) f->x[6 + lane] += d;  // delta[3..29] -> x[9..35]
            LK_SC(5);
        }
        __syncthreads();
        LK_SC(6);
    }
#undef LK_SC
    return (uint32_t)(cnt + 0.5);
}

// The covariance half: P <- P - (P6 W) P[0:6,:]   (eskf.cc:112, no symmetrisation), in two steps every caller shares:
// cov_prep fills KH = P6 W and Prow = P[0:6,:] (threads [0, nthreads) of the block), then entry e is cov_entry(f, e).
__device__ __forceinline__ void cov_prep(BlockFilter* f, int nthreads) {
    for (int e = threadIdx.x; e < 180; e += nthreads) {
        f->Prow[e] = f->P[e];  // rows 0..5 are contiguous
        int i = e / 6, j = e % 6;
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < 6; ++k) s += f->P[i * 30 + k] * f->W[k * 6 + j];
        f->KH[e] = s;
    }
}

__device__ __forceinline__ double cov_entry(const BlockFilter* f, int e) {
    int i = e / 30, j = e % 30;
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < 6; ++k) s += f->KH[i * 6 + k] * f->Prow[k * 30 + j];
    return f->P[e] - s;
}

// The whole update in shared memory. All threads call.
template <int NTHREADS>
__device__ __forceinline__ void block_cov_update(BlockFilter* f) {
    cov_prep(f, NTHREADS);
    __syncthreads();
    for (int e = threadIdx.x; e < 900; e += NTHREADS) f->P[e] = cov_entry(f, e);
    __syncthreads();
}

// Both halves (the covariance only after the last iteration). Returns the residual count.
template <int NTHREADS>
__device__ __forceinline__ uint32_t block_solve_update(BlockFilter* f, bool last_iter, unsigned long long* clk = nullptr) {
    const uint32_t n = block_solve_state(f, clk);
    if (n > 0 && last_iter) block_cov_update<NTHREADS>(f);
    return n;
}

// ScanConst from a shared-memory filter. Threads 0..23.
__device__ __forceinline__ void scan_const_from(const BlockFilter* f, ScanConst* sc) {
    const int tid = threadIdx.x;
    if (tid < 9) sc->R[tid] = f->x[tid];
    else if (tid < 12) sc->p[tid - 9] = f->x[tid];
    else if (tid < 24) {
        // entry q of the upper triangle xx xy xz yy yz zz: (i, j) computed, not read from a table indexed at run time
        // (which would live in local memory)
        const int q = (tid - 12) % 6, o = (tid < 18) ? 0 : 3;
        const int i = (q < 3 ? 0 : (q < 5 ? 1 : 2)) + o, j = (q < 3 ? q : (q < 5 ? q - 2 : 2)) + o;
        const double v = 0.5 * (f->P[i * 30 + j] + f->P[j * 30 + i]);
        if (tid < 18) sc->Pth[q] = v; else sc->Ppp[q] = v;
    }
}

}  // namespace lk
