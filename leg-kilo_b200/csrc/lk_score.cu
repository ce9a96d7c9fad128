// lk_score.cu — lk_score_poses: the sums the LiDAR update would form, at many candidate poses of each point set, against a
// map that stays fixed for the call. No filter is read or written and nothing is solved.
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
#include "lk_kernels.h"
#include "lk_pass.cuh"
#include "lk_solve.cuh"

namespace lk {

static_assert(LK_SCORE_A == 0 && LK_SCORE_B == ACC_B && LK_SCORE_SUM_R == ACC_SUMR && LK_SCORE_COUNT == ACC_CNT &&
                  LK_SCORE_SUM_Z2R == NACC && LK_SCORE_STRIDE == PARTIAL_STRIDE,
              "lk_score_poses record layout (include/legkilo_b200.h) = the partial-row layout");

namespace {

constexpr int BLOCK = SCORE_CHUNK;  // one point per thread per pass
constexpr int WARPS = BLOCK / 32;
constexpr int SUM_THREADS = 128;

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

}  // namespace

void launch_score(const ScoreArgs& a, uint32_t n_items, uint32_t n_sums, cudaStream_t s) {
    static PerDeviceOnce once;
    const size_t smem = sizeof(PassSmem<BLOCK, true>);
    if (once.first()) cudaFuncSetAttribute(k_score, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (n_items) k_score<<<n_items, BLOCK, smem, s>>>(a);
    if (n_sums) k_score_sum<<<n_sums, SUM_THREADS, 0, s>>>(a);
}

}  // namespace lk
