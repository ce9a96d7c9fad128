// lk_kernels.h — host-callable launchers of the device kernels (one translation unit each).
#pragma once
#include <cuda_runtime.h>

#include "lk_device.cuh"
#include "lk_llsync.cuh"
#include "lk_plane.cuh"

namespace lk {

// Per (step, scan) description of the bucket processed in that step; built on the host at
// stage time from scan_offsets / bucket_offsets / bucket_times.
struct StepInit {
    uint32_t chunk_begin, chunk_end;
    uint32_t pt_begin, pt_end;
    double t_bucket;
    uint32_t active;
    uint32_t pad;
};

struct ResidualArgs {
    const float4* pts;
    const HashSlot* slots;
    uint32_t hash_mask;
    const MapNode* nodes;
    const HotRec* hot;        // hot images of the nodes (throughput kernel)
    const ChunkDesc* chunks;  // chunk table of the whole staged batch
    uint32_t chunk_first;     // first chunk of this launch (grid.x = number of chunks)
    ScanConst* sc;            // [batch]
    ScanStep* step;           // [batch]
    double* partial;          // [total_chunks * PARTIAL_STRIDE]
    uint32_t* ticket;         // [batch]
    double* x;                // [batch * 36]
    double* P;                // [batch * 900]
    lk_stream_clock* clk;     // [batch]
    uint32_t* n_eff;          // [batch] accumulated success_pts_size_out
    int last_iter;
    // debug (lk_debug_residuals): per-point rows instead of accumulation
    uint8_t* dbg_ok;
    double* dbg_h;
    double* dbg_z;
    double* dbg_R;
    int32_t* dbg_key;
    unsigned long long* trace;  // optional %globaltimer stamps: 8 per block + 8 for the tail
    // throughput family: the points whose home voxel gave no residual on the hot images, per chunk and warp in ballot order
    // (chunk-relative indices), finished by k_residual_fallback with the full reference sequence
    uint16_t* fb_list;  // [total_chunks][S2_FB_WARPS][S2_FB_CAP]
    uint32_t* fb_cnt;   // [total_chunks][S2_FB_WARPS]
    Globals g;
};
constexpr uint32_t S2_FB_WARPS = 6, S2_FB_CAP = 704;

// Every chunk of the launch holds at most 256 points (one point per thread, one pass), except with debug
// (lk_debug_residuals), where a block walks its chunk in 256-point slices and writes per-point rows. hot: the map stays fixed
// for the call, so the pass stages hot plane images instead of node records (lk_pass.cuh: Stage)
void launch_residual(const ResidualArgs& a, uint32_t n_chunks, bool debug, bool hot, cudaStream_t s);
// throughput family: pipelined residual pass (lk_stream2.cu) writing one partial row per chunk, then the per-scan
// solve for scans [scan_first, scan_first + n_scans) (lk_residual.cu)
void launch_residual_stream2(const ResidualArgs& a, uint32_t n_chunks, cudaStream_t s);
void launch_residual_fallback(const ResidualArgs& a, uint32_t n_chunks, cudaStream_t s);
void launch_scan_tail(const ResidualArgs& a, uint32_t scan_first, uint32_t n_scans, cudaStream_t s);

struct PredictArgs {
    const StepInit* init;  // [batch] for this step
    ScanStep* step;        // [batch]
    ScanConst* sc;         // [batch]
    double* x;             // [batch*36]
    double* P;             // [batch*900]
    const double* Q;       // [900]
    lk_stream_clock* clk;  // [batch]
    uint32_t* ticket;
    uint32_t* n_eff;
    const double* x_in;   // staged inputs, read when reset != 0
    const double* P_in;
    const lk_stream_clock* clk_in;
    int reset;            // re-load the filter from the staged inputs first (only on a scan's first step)
    int scan_first;  // first scan of the range this launch covers
    int batch;       // scans in the range (grid.x)
};
void launch_predict_prepare(const PredictArgs& a, cudaStream_t s);
void launch_obs_predict_prepare(const PredictArgs& a, const lk_imu_meas* imu, const lk_kinimu_meas* kin, uint32_t n,
                                const lk_eskf_cfg& cfg, double gravity, double acc_norm, cudaStream_t s);

// Plain ESKF::predict on `batch` filters with explicit dt (lk_predict).
void launch_predict_dt(double* x, double* P, const double* Q, const double* dt, int batch, int prop_state,
                       int prop_cov, cudaStream_t s);

struct ReprojectArgs {
    const float4* pts;
    float4* world;
    const ChunkDesc* chunks;
    uint32_t chunk_first;
    const ScanConst* sc;
    const ScanStep* step;
    Globals g;
};
void launch_reproject(const ReprojectArgs& a, uint32_t n_chunks, cudaStream_t s);


void launch_filter_obs(double* x, double* P, const double* Q, lk_stream_clock* clk, const lk_imu_meas* imu,
                       const lk_kinimu_meas* kin, uint32_t n, const lk_eskf_cfg& cfg, double gravity, double acc_norm,
                       cudaStream_t s);
void launch_update_by_points(double* x, double* P, uint32_t n, const double* h, const double* z, const double* r,
                             cudaStream_t s);

// ---- fused per-scan persistent kernel (lk_fused.cu) -------------------------------------------
constexpr int FUSED_INLINE_STEPS = 64;
// Small inputs carried in the kernel's parameter block (direct mode: no staging copy before the launch).
struct FusedInline {
    double x[36];
    double P[900];
    double clk[2];
    StepInit steps[FUSED_INLINE_STEPS];
};
struct FusedNoInline {
    int unused;
};

struct FusedArgs {
    const float4* pts;    // device memory, or page-locked host memory read in place (each point is read once)
    float4* world;
    const StepInit* inits;  // [n_steps][batch] (unused with inline inputs)
    int batch;
    uint32_t n_steps;
    uint32_t scan;
    const double* x_in;
    const double* P_in;
    const lk_stream_clock* clk_in;
    const double* Q;
    double* x;
    double* P;
    lk_stream_clock* clk;
    uint32_t* n_eff;
    uint32_t* status;  // one word next to the outputs: non-zero when a device-side wait of this launch gave up
    LLView ll;       // flagged rows of the barrier-free all-reduce (lk_llsync.cuh)
    uint32_t epoch;  // tag of this launch's first exchange; the launch uses epoch .. epoch + n_steps * (iters + 2) - 1
    int iters;
    int lane_cache;  // keep per-lane lookups / staged records across the iterations of a bucket
    int slim_p;        // blocks other than 0 load only P[:, 0:6] (valid when the scan has one bucket, no queue, no predict)
    // > 0 (one active bucket, no queue, no insert): the last `finishers` blocks of the grid run the scan's epilogue and the
    // others leave at their last row (lk_fused.cu)
    uint32_t finishers;
    float4* pts_copy;  // with finishers and points in host memory: device copy of the points the workers make for them
    MapView mv;
    const lk_imu_meas* imu;      // queued samples interleaved with the buckets (exactly one of imu / kin, or none)
    const lk_kinimu_meas* kin;
    uint32_t n_meas;
    double gravity, acc_norm;
    lk_eskf_cfg ecfg;
    unsigned long long* trace;  // optional: 32 %globaltimer stamps per block
    Globals g;
    // in-kernel UpdateVoxelMap after every bucket (streaming): the device map and the per-bucket scratch of lk_insert.cu
    int insert;
    MapDev md;
    DevPoint* ipts;          // [largest bucket]
    int* iroot;              // [largest bucket]
    int* pend;               // [node_cap * 3]
    uint32_t* touched;       // [largest bucket]
    uint32_t* ins_counters;  // [2] touched-root counters used alternately by consecutive buckets (both zero at launch)
};
enum { FUSED_LAUNCH_PLAIN = 0, FUSED_LAUNCH_COOPERATIVE = 1, FUSED_LAUNCH_PDL = 2 };
size_t fused_smem_bytes();
int fused_max_blocks(int device);
int fused_read_stall(uint32_t out[8]);  // watchdog note of the fused kernels (lk_async.cuh: lk_stall_note)
// inl != null: the filter inputs and the step table ride in the parameter block
cudaError_t launch_scan_fused(const FusedArgs& a, const FusedInline* inl, uint32_t grid, cudaStream_t s, int mode);

// Per-device "already done" latch for cudaFuncSetAttribute-style one-time setup (function attributes are per device).
struct PerDeviceOnce {
    bool done[64] = {};
    bool first() {
        int d = 0;
        cudaGetDevice(&d);
        if (d < 0 || d >= 64) return true;
        if (done[d]) return false;
        done[d] = true;
        return true;
    }
};

}  // namespace lk
