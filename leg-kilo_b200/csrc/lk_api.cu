// lk_api.cu — the extern "C" boundary (include/legkilo_b200.h): context, device memory,
// staging, launch sequencing. No CPU fallback anywhere: without a CUDA device lk_create fails.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <chrono>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "lk_host.h"
#include "lk_kernels.h"
#include "lk_mapdev.h"

using namespace lk;

namespace {

thread_local std::string g_create_error;

struct DevView {  // a typed window into somebody else's device allocation
    void* p = nullptr;
    template <class T>
    T* as() const { return reinterpret_cast<T*>(p); }
};

// The packed small inputs of a staged batch (one page-locked block, one H2D copy), byte offsets of
// chunks | inits | x | P | clk | Q | chunksL | initsL, each 256-byte aligned.
struct InBlock {
    size_t chunks = 0, inits = 0, x = 0, P = 0, clk = 0, Q = 0, chunksL = 0, initsL = 0, bytes = 0;
    InBlock() = default;
    InBlock(int batch, size_t n_chunks, size_t n_inits, size_t n_chunksL, size_t n_initsL)
        : inits(align256(std::max<size_t>(n_chunks, 1) * sizeof(ChunkDesc))),
          x(inits + align256(std::max<size_t>(n_inits, 1) * sizeof(StepInit))),
          P(x + align256((size_t)batch * sizeof(lk_state))),
          clk(P + align256((size_t)batch * 900 * 8)),
          Q(clk + align256((size_t)batch * sizeof(lk_stream_clock))),
          chunksL(Q + align256(900 * 8)),
          initsL(chunksL + align256(n_chunksL * sizeof(ChunkDesc))),
          bytes(initsL + align256(n_initsL * sizeof(StepInit))) {}
};

// The small outputs (one device block, or in direct mode the page-locked block the kernel stores into; one D2H copy),
// byte offsets of x | P | clk | n_eff | status word, each 256-byte aligned.
struct OutBlock {
    size_t x = 0, P = 0, clk = 0, n_eff = 0, status = 0, bytes = 0;
    OutBlock() = default;
    explicit OutBlock(int batch)
        : P(align256((size_t)batch * sizeof(lk_state))),
          clk(P + align256((size_t)batch * 900 * 8)),
          n_eff(clk + align256((size_t)batch * sizeof(lk_stream_clock))),
          status(n_eff + align256((size_t)batch * 4)),
          bytes(status + 256) {}
};

}  // namespace

struct lk_context {
    int device = 0;
    cudaStream_t stream = nullptr;
    std::string err;
    lk_eskf_cfg ec;
    lk_map_cfg mc;
    Globals g;

    // map
    MapDevHost map;
    double last_slide_position[3] = {0.0, 0.0, 0.0};  // VoxelMapManager::last_slide_position (voxel_map.h:201)

    // staged batch
    int batch = 0;
    uint64_t total_pts = 0;
    uint32_t total_chunks = 0, n_steps = 0, max_chunk_pts = 0;
    std::vector<ChunkDesc> h_chunks, h_chunksL;
    InBlock in;    // layout of small_in / h_small_in
    OutBlock out;  // layout of small_out / h_small_out
    DevBuf pts, world, sc, step, partial, ticket, fb_list, fb_cnt;
    // small per-call inputs / outputs travel as ONE packed copy each way (pinned staging blocks)
    DevBuf small_in, small_out, fx, fP, fQ, fclk;
    PinnedBuf h_small_in, h_small_out;
    DevView chunks, stepinit, x_in, P_in, clk_in, Q, x, P, clk, n_eff, status;
    DevBuf dbg_ok, dbg_h, dbg_z, dbg_R, dbg_key, tmp, trace, bar;
    MapInserter inserter;  // UpdateVoxelMap: update_map runs and lk_map_insert
    PoseScorer scorer;     // lk_score_poses and lk_refine_poses
    int trace_on = 0;
    uint32_t trace_seq = 0;  // fused launches traced since the trace was switched on or last read back
    int lane_cache = 1;
    int use_fused = 1;      // batch-of-one runs go through the persistent per-scan kernel
    FusedInline inl;         // parameter-block image of the small inputs (direct mode)
    DevBuf ll;               // flagged rows of the fused kernel's all-reduce (lk_llsync.cuh), zero-filled once
    uint32_t ll_epoch = 1;   // next unused tag (0 = the fill value, never used)
    bool prev_fused = false;  // the last operation enqueued on `stream` was a fused launch (PDL is only used then)
    uint32_t fused_launches = 0, fused_launches_since_check = 0;
    // direct mode of lk_scan_update (one scan, page-locked caller buffers): the kernel reads the points and
    // writes the world cloud / the filter in place, the small inputs ride in the kernel's parameter block
    int direct_io = 1, inline_in = 1, coop_launch = 0, pdl = 1, n_sms = 132, slim_p = 1;
    int finishers = 1;  // per-scan kernel: run a single-bucket scan's epilogue on the SMs its chunks leave idle (lk_fused.cu)
    int fast_insert = 1;  // update_map: two-launch insert for small buckets, re-projection folded into it
    int fused_insert = 0;  // 1 = update_map of one scan with small buckets: UpdateVoxelMap inside the persistent kernel (one
                           // launch per scan; the serial per-root insert chain holds every other SM at the grid barrier)
    int debug_records = 0;  // 1 = lk_debug_residuals stages node records (the form update_map calls evaluate), not hot images
    bool direct = false, direct_ran = false, inline_ok = false;
    const float4* direct_pts = nullptr;
    float4* direct_world = nullptr;
    double hprof[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // host-side ns of lk_scan_update: stage | enqueue | wait+fetch | calls
    DevBuf Qc;                     // process noise kept on the device between calls
    DevBuf leg_scratch;            // lk_leg_kinematics: inputs, flags, scans and outputs of the last call's size
    DevBuf pre_scratch;            // lk_preprocess_scan(s): points, keys, leaves and buckets of the largest call
    DevBuf dec_scratch;            // lk_decode_pointcloud2(s): raw bytes, flags and decoded points of the largest call
    std::vector<double> Q_shadow;  // what Qc holds

    // timing
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    std::vector<cudaEvent_t> kev;
    float last_total_ms = 0, last_residual_ms = 0;
    uint32_t last_launches = 0, last_residual_launches = 0;
    uint32_t acc_launches = 0, acc_residual_launches = 0;
    size_t nev = 0;
    int kernel_timing = 1;
    std::vector<StepInit> h_inits;
    std::vector<uint32_t> h_scan_pts;
    std::vector<uint32_t> h_scan_chunks;  // per scan: the most chunks of one of its buckets (at least 1)
    // the throughput family's chunk table (same buckets, larger chunks); aliases the first one when equal
    std::vector<StepInit> h_initsL;
    DevView chunksL, stepinitL;
    uint32_t total_chunksL = 0;

    ~lk_context() {  // the buffers free themselves after this
        for (cudaEvent_t e : kev) cudaEventDestroy(e);
        if (ev0) cudaEventDestroy(ev0);
        if (ev1) cudaEventDestroy(ev1);
        if (stream) cudaStreamDestroy(stream);
    }
};

namespace {

// Every field of a PointCloud2 layout lies inside point_step (the time field is 8 bytes for Hesai, 4 otherwise).
bool pc2_layout_fits(const lk_pc2_layout& L) {
    const uint32_t tsz = L.lidar_type == LK_LIDAR_HESAI ? 8u : 4u;
    return L.lidar_type >= 1 && L.lidar_type <= 3 && L.off_x + 4 <= L.point_step && L.off_y + 4 <= L.point_step &&
           L.off_z + 4 <= L.point_step && L.off_intensity + 4 <= L.point_step && L.off_time + tsz <= L.point_step;
}

bool all_finite(const double* v, size_t n) { return std::all_of(v, v + n, [](double x) { return std::isfinite(x); }); }

int fail(lk_handle h, int code, const std::string& msg) {
    if (h) h->err = msg;
    else g_create_error = msg;
    return code;
}

// One per device: the stream of the most recent fused launch of this process (see run_range_impl).
struct FusedGate {
    std::mutex m;
    cudaStream_t last = nullptr;
    cudaEvent_t ev = nullptr;
};
FusedGate& fused_gate(int device) {
    static FusedGate gates[64];
    return gates[(device >= 0 && device < 64) ? device : 0];
}

// Start of every entry point that enqueues work: the handle's device, and the next fused launch must not chain by PDL
// (programmatic dependent launch) onto what this call enqueues: PDL may only overlap a fused launch with the previous one.
void enter(lk_handle h) {
    cudaSetDevice(h->device);
    h->prev_fused = false;
}

void fill_globals(lk_context* c, const double* extR, const double* extT) {
    Globals& g = c->g;
    for (int i = 0; i < 9; ++i) g.Re[i] = extR[i];
    for (int i = 0; i < 3; ++i) g.te[i] = extT[i];
    g.voxel = c->mc.max_voxel_size;
    int ex = 0;
    double m = std::frexp(g.voxel, &ex);
    g.voxel_pow2 = (m == 0.5 && g.voxel > 0) ? 1 : 0;
    g.inv_voxel = 1.0 / g.voxel;
    g.sigma_num = c->mc.sigma_num;
    g.ratio = c->ec.lidar_point_meas_ratio;
    // calcBodyCov(pb, dept_err (float range_inc), beam_err (float degree_inc)) — voxel_map.cc:22-27
    float range_inc = (float)c->mc.dept_err;
    float degree_inc = (float)c->mc.beam_err;
    g.rv = range_inc * range_inc;
    double sd = std::sin((double)degree_inc * 0.017453293);  // PCL DEG2RAD
    g.dv = sd * sd;
    g.voxel_f = (float)c->mc.max_voxel_size;
    g.planer_threshold = (float)c->mc.planner_threshold;
    g.max_layer = c->mc.max_layer;
    g.max_points_num = c->mc.max_points_num;
    for (int i = 0; i < 5; ++i) g.layer_init_num[i] = c->mc.layer_init_num[i];
    c->map.tile_slots = (uint32_t)((std::max(g.max_points_num, 0) + 2 + 1) & ~1);  // lk_octree.cuh: std_tile
}

// the trace buffer ((1 << 16) * 8 doubles' worth of %globaltimer stamps): TRACE_AREAS areas of TRACE_AREA stamps, one per
// traced fused launch (a launch writes 32 per block plus, streaming with the insert inside, 64 x 8 per-bucket stamps)
constexpr size_t TRACE_AREA = 8192;
constexpr size_t TRACE_AREAS = 64;

// Chunking is a function of the bucket and of the kernel family alone, so results are bitwise independent
// of how a batch is sharded across GPUs (SURVEY §4 multi-GPU invariant).
//   latency family (one scan per call): buckets up to 132 x 256 points use one point per thread (256-point
//     chunks, one per SM: the fused kernel); larger ones the throughput family's chunks;
//   throughput family (>= 2 scans per call): 3 840-point chunks as soon as a bucket exceeds 2 048 points —
//     every warp then streams 20 groups and the per-chunk reduce is amortised.
constexpr uint32_t LATENCY_MAX_BUCKET = 132u * 256u;  // one 256-point chunk per SM of an H100: the fused kernel's reach
uint32_t chunk_size_for(uint32_t n, bool throughput, uint32_t big = 3840u) {
    if (throughput) return n <= 2048u ? 256u : big;
    return n <= LATENCY_MAX_BUCKET ? 256u : big;
}

cudaEvent_t kev_get(lk_context* c, size_t i) {
    while (c->kev.size() <= i) {
        cudaEvent_t e;
        cudaEventCreate(&e);
        c->kev.push_back(e);
    }
    return c->kev[i];
}

ResidualArgs residual_args(lk_context* c, const ChunkDesc* chunks) {
    ResidualArgs a;
    std::memset(&a, 0, sizeof(a));
    const MapDev md = c->map.dev();
    a.pts = c->pts.as<float4>();
    a.slots = md.slots;
    a.hash_mask = md.hash_mask;
    a.nodes = md.nodes;
    a.hot = md.hot;
    a.chunks = chunks;
    a.sc = c->sc.as<ScanConst>();
    a.step = c->step.as<ScanStep>();
    a.partial = c->partial.as<double>();
    a.ticket = c->ticket.as<uint32_t>();
    a.x = c->x.as<double>();
    a.P = c->P.as<double>();
    a.clk = c->clk.as<lk_stream_clock>();
    a.n_eff = c->n_eff.as<uint32_t>();
    a.trace = c->trace_on ? c->trace.as<unsigned long long>() : nullptr;
    a.fb_list = c->fb_list.as<uint16_t>();
    a.fb_cnt = c->fb_cnt.as<uint32_t>();
    a.g = c->g;
    return a;
}

// The predict / prepare launch of one step for scans [first, first + count); reset: re-load the staged filter first.
PredictArgs predict_args(lk_context* c, const StepInit* init, int reset, uint32_t first, uint32_t count) {
    PredictArgs a;
    a.init = init;
    a.step = c->step.as<ScanStep>();
    a.sc = c->sc.as<ScanConst>();
    a.x = c->x.as<double>();
    a.P = c->P.as<double>();
    a.Q = c->Q.as<double>();
    a.clk = c->clk.as<lk_stream_clock>();
    a.ticket = c->ticket.as<uint32_t>();
    a.n_eff = c->n_eff.as<uint32_t>();
    a.x_in = c->x_in.as<double>();
    a.P_in = c->P_in.as<double>();
    a.clk_in = c->clk_in.as<lk_stream_clock>();
    a.reset = reset;
    a.scan_first = (int)first;
    a.batch = (int)count;
    return a;
}

// Does a run of `count` scans from `first` take ONE launch of the per-scan kernel (lk_fused.cu)? One scan whose buckets
// have one chunk per block and at most as many chunks as the kernel has blocks; a map insert must then run inside it.
bool per_scan_kernel(const lk_context* h, uint32_t first, uint32_t count, bool update_map, bool fused_insert) {
    return count == 1 && h->use_fused && h->max_chunk_pts <= 256 && (!update_map || fused_insert) &&
           h->h_scan_chunks[first] <= (uint32_t)fused_max_blocks(h->device);
}

// Point the output views at a block laid out as h->out (device memory, or page-locked memory in direct mode).
void point_outputs(lk_context* h, char* base) {
    h->x.p = base + h->out.x;
    h->P.p = base + h->out.P;
    h->clk.p = base + h->out.clk;
    h->n_eff.p = base + h->out.n_eff;
    h->status.p = base + h->out.status;
}

// After a synchronisation: did a fused launch give up waiting for its peers (lk_llsync.cuh watchdog)?
int check_stall(lk_handle h) {
    if (!h->ll.p || !h->fused_launches_since_check) return LK_OK;
    h->fused_launches_since_check = 0;
    uint32_t st[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    LK_CUDA(h->err, cudaMemcpy(st, (char*)h->ll.p + LL_ROWS_BYTES, sizeof(st), cudaMemcpyDeviceToHost));
    uint32_t note[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (fused_read_stall(note) == 0 && note[0]) {
        char m2[256];
        static const char* what[] = {"", "a bulk copy never completed its mbarrier", "a root-table slot was never published",
                                     "octree deeper than max_layer", "root table has no empty slot"};
        std::snprintf(m2, sizeof(m2), "per-scan kernel watchdog: %s (block %u, thread %u, detail %u)", what[note[0] < 5 ? note[0] : 0],
                      note[1], note[2], note[3]);
        return fail(h, LK_ERR_CUDA, m2);
    }
    if (!st[0]) return LK_OK;
    LK_CUDA(h->err, cudaMemset((char*)h->ll.p + LL_ROWS_BYTES, 0, 64));
    char msg[320];
    std::snprintf(msg, sizeof(msg), "per-scan kernel: block %u gave up waiting for rows [%u, %u) of exchange tag %u (lane %u): the grid was "
                  "not fully resident (device shared with another process?)", st[1], st[3], st[3] + st[4], st[2], st[5]);
    return fail(h, LK_ERR_CUDA, msg);
}

// StateInitialByImu / ByKinImu::processing (state_initial.hpp:34-117): the running means seeded with sample 0, which the
// loop then visits again with N = 1; acc / gyr at the same offsets in both sample types.
template <class Meas>
void state_initial(const Meas* m, uint32_t n, double gravity, lk_state* x, double* acc_norm) {
    double ma[3], mw[3];
    for (int k = 0; k < 3; ++k) {
        ma[k] = m[0].acc[k];
        mw[k] = m[0].gyr[k];
    }
    int N = 1;
    for (uint32_t i = 0; i < n; ++i, ++N)
        for (int k = 0; k < 3; ++k) {
            ma[k] += (m[i].acc[k] - ma[k]) / N;
            mw[k] += (m[i].gyr[k] - mw[k]) / N;
        }
    double s = 0.0;
    for (int k = 0; k < 3; ++k) s += ma[k] * ma[k];
    *acc_norm = std::sqrt(s);
    for (int k = 0; k < 3; ++k) {
        x->grav[k] = -ma[k] / *acc_norm * gravity;
        x->bw[k] = mw[k];
    }
    for (int i = 0; i < 9; ++i) x->rot[i] = (i % 4 == 0) ? 1.0 : 0.0;
}

}  // namespace

extern "C" {

int lk_abi_version(void) { return LK_ABI_VERSION; }

const char* lk_last_error(lk_handle h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int lk_create(const lk_eskf_cfg* eskf_cfg, const lk_map_cfg* map_cfg, const double ext_rot[9], const double ext_t[3],
              int device, lk_handle* out) {
    if (!eskf_cfg || !map_cfg || !ext_rot || !ext_t || !out) return fail(nullptr, LK_ERR_INVALID_ARG, "null argument");
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        return fail(nullptr, LK_ERR_NO_DEVICE,
                    std::string("no CUDA device: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "count == 0") +
                        " (this library has no CPU fallback)");
    }
    if (device < 0 || device >= n) return fail(nullptr, LK_ERR_INVALID_ARG, "device ordinal out of range");
    if (map_cfg->max_layer < 0 || map_cfg->max_layer > 4) return fail(nullptr, LK_ERR_INVALID_ARG, "max_layer must be 0..4");
    if (!(map_cfg->max_voxel_size > 0)) return fail(nullptr, LK_ERR_INVALID_ARG, "voxel size must be positive");
    e = cudaSetDevice(device);
    if (e != cudaSuccess) return fail(nullptr, LK_ERR_CUDA, cudaGetErrorString(e));
    lk_context* c = new lk_context;
    c->device = device;
    c->ec = *eskf_cfg;
    c->mc = *map_cfg;
    fill_globals(c, ext_rot, ext_t);
    cudaDeviceGetAttribute(&c->n_sms, cudaDevAttrMultiProcessorCount, device);
    e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) {
        c->stream = nullptr;
        delete c;
        return fail(nullptr, LK_ERR_CUDA, cudaGetErrorString(e));
    }
    cudaEventCreate(&c->ev0);
    cudaEventCreate(&c->ev1);
    *out = c;
    return LK_OK;
}

int lk_destroy(lk_handle h) {
    if (!h) return LK_OK;
    enter(h);
    cudaStreamSynchronize(h->stream);
    {
        FusedGate& gate = fused_gate(h->device);
        std::lock_guard<std::mutex> lock(gate.m);
        if (gate.last == h->stream) gate.last = nullptr;
    }
    delete h;
    return LK_OK;
}

int lk_init_process_cov(const lk_eskf_cfg* c, double* Q) {
    if (!c || !Q) return LK_ERR_INVALID_ARG;
    for (int i = 0; i < 900; ++i) Q[i] = 0.0;
    const double d[7] = {c->vel_process_cov,     c->acc_bias_process_cov, c->gyr_bias_process_cov, c->imu_acc_process_cov,
                         c->imu_gyr_process_cov, c->kin_bias_process_cov, c->contact_process_cov};
    const int at[7] = {6, 9, 12, 18, 21, 24, 27};
    for (int b = 0; b < 7; ++b)
        for (int k = 0; k < 3; ++k) Q[(at[b] + k) * 30 + at[b] + k] = d[b];
    return LK_OK;
}

int lk_state_default(lk_state* x) {
    if (!x) return LK_ERR_INVALID_ARG;
    std::memset(x, 0, sizeof(*x));
    x->rot[0] = x->rot[4] = x->rot[8] = 1.0;
    x->grav[2] = -9.81;
    return LK_OK;
}

int lk_leg_track_default(lk_leg_track* t) {
    if (!t) return LK_ERR_INVALID_ARG;
    for (int k = 0; k < 4; ++k) t->in_contact[k] = 1;  // ContactDetector::in_contact_{true} (kinematics.h:12)
    t->last_acc_z = 0.0f;                                // the zero-initialised static HighState (ros_interface.cc:222)
    t->last_gyr_z = 0.0f;
    return LK_OK;
}

int lk_host_alloc(void** p, size_t bytes) {
    if (!p) return LK_ERR_INVALID_ARG;
    cudaError_t e = cudaHostAlloc(p, bytes, cudaHostAllocDefault);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return LK_ERR_OUT_OF_MEMORY;
    }
    return LK_OK;
}

int lk_host_free(void* p) {
    if (p) cudaFreeHost(p);
    return LK_OK;
}

int lk_set_param(lk_handle h, const char* name, double value) {
    if (!h || !name) return LK_ERR_INVALID_ARG;
    using IntKnob = int lk_context::*;
    static const struct {
        const char* name;
        IntKnob knob;
    } knobs[] = {{"kernel_timing", &lk_context::kernel_timing}, {"fused", &lk_context::use_fused},
                 {"lane_cache", &lk_context::lane_cache},       {"fast_insert", &lk_context::fast_insert},
                 {"fused_insert", &lk_context::fused_insert},   {"coop_launch", &lk_context::coop_launch},
                 {"pdl", &lk_context::pdl},                     {"slim_p", &lk_context::slim_p},
                 {"direct_io", &lk_context::direct_io},         {"inline_in", &lk_context::inline_in},
                 {"debug_records", &lk_context::debug_records}, {"finishers", &lk_context::finishers}};
    for (const auto& k : knobs)
        if (!std::strcmp(name, k.name)) {
            h->*k.knob = (int)value;
            return LK_OK;
        }
    if (!std::strcmp(name, "trace")) {
        h->trace_on = (int)value;
        if (h->trace_on) {
            enter(h);
            LK_CUDA(h->err, h->trace.ensure((size_t)(1 << 16) * 8 * 8));
            LK_CUDA(h->err, cudaMemset(h->trace.p, 0, (size_t)(1 << 16) * 8 * 8));
        }
        h->trace_seq = 0;
        return LK_OK;
    }
    return fail(h, LK_ERR_INVALID_ARG, std::string("unknown parameter ") + name);
}

// Debug read-back of internal device buffers: what = 0 partial sums, 1 scan constants (the header lists the rest).
int lk_debug_read(lk_handle h, int what, void* dst, size_t bytes) {
    if (!h || !dst) return LK_ERR_INVALID_ARG;
    if (what == 3) {  // host-side phase times of lk_scan_update (ns, accumulated) — reading resets them
        std::memcpy(dst, h->hprof, std::min(bytes, sizeof(h->hprof)));
        std::memset(h->hprof, 0, sizeof(h->hprof));
        return LK_OK;
    }
    if (what == 4) {  // the pose scorer's scratch: device bytes, page-locked bytes
        const uint64_t held[2] = {h->scorer.device_bytes(), h->scorer.host_bytes()};
        std::memcpy(dst, held, std::min(bytes, sizeof(held)));
        return LK_OK;
    }
    enter(h);
    DevBuf* b = what == 0 ? &h->partial : (what == 1 ? &h->sc : &h->trace);
    if (what == 2) h->trace_seq = 0;
    if (bytes > b->cap) bytes = b->cap;
    LK_CUDA(h->err, cudaMemcpy(dst, b->p, bytes, cudaMemcpyDeviceToHost));
    return LK_OK;
}

int lk_sync(lk_handle h) {
    if (!h) return LK_ERR_INVALID_ARG;
    enter(h);
    LK_CUDA(h->err, cudaStreamSynchronize(h->stream));
    return check_stall(h);
}

// ---- map ------------------------------------------------------------------------------------

int lk_map_reserve(lk_handle h, uint64_t max_roots, uint64_t max_nodes, uint64_t max_points) {
    if (!h) return LK_ERR_INVALID_ARG;
    h->map.reserve_roots = max_roots;
    h->map.reserve_nodes = max_nodes;
    h->map.reserve_points = max_points;
    return LK_OK;
}

int lk_map_upload(lk_handle h, const void* blob, size_t bytes) {
    if (!h || !blob) return fail(h, LK_ERR_INVALID_ARG, "null argument");
    enter(h);
    return map_upload_blob(h->map, h->g, blob, bytes, h->stream, h->err);
}

int lk_map_stats(lk_handle h, uint64_t out[4]) {
    if (!h || !out) return LK_ERR_INVALID_ARG;
    enter(h);
    uint64_t planes = 0, live = 0;
    const int rc = map_count_planes(h->map, &planes, &live, h->stream, h->err);
    if (rc) return rc;
    out[0] = h->map.n_roots;
    out[1] = h->map.n_nodes;
    out[2] = live;
    out[3] = planes;
    return LK_OK;
}

int lk_map_memory(lk_handle h, uint64_t out[6]) {
    if (!h || !out) return LK_ERR_INVALID_ARG;
    enter(h);
    MapDevHost& m = h->map;
    const int rc = m.ready() ? m.sync_counters(h->stream, h->err) : LK_OK;
    if (rc) return rc;
    out[0] = m.n_nodes;
    out[1] = 8 * m.free_entries(FREE_GROUPS) + m.free_entries(FREE_SINGLES);
    out[2] = m.n_points;
    out[3] = (uint64_t)m.tile_slots * m.free_entries(FREE_TILES);
    out[4] = m.pool_bytes();
    out[5] = m.reallocs;
    return LK_OK;
}

int lk_map_slide(lk_handle h, const double position[3], int32_t* slid, uint64_t* removed) {
    if (!h || !position) return fail(h, LK_ERR_INVALID_ARG, "null argument");
    if (slid) *slid = 0;
    if (removed) *removed = 0;
    enter(h);
    // voxel_map.cc:553: (position_last_ - last_slide_position).norm() < sliding_thresh -> nothing to do
    double d2 = 0.0;
    for (int k = 0; k < 3; ++k) d2 += (position[k] - h->last_slide_position[k]) * (position[k] - h->last_slide_position[k]);
    if (std::sqrt(d2) < h->mc.sliding_thresh) return LK_OK;
    for (int k = 0; k < 3; ++k) h->last_slide_position[k] = position[k];
    int lo[3], hi[3];
    for (int k = 0; k < 3; ++k) {
        const int key = (int)std::floor(position[k] / h->mc.max_voxel_size);  // voxelKeyFloor (eigen_types.hpp:89-95)
        lo[k] = key - h->mc.half_map_size;
        hi[k] = key + h->mc.half_map_size;
    }
    const int rc = map_clear_outside(h->map, lo, hi, removed, h->stream, h->err);
    if (rc) return rc;
    if (slid) *slid = 1;
    return LK_OK;
}

int lk_tum_line(double timestamp, const double rot[9], const double pos[3], char* buf, size_t capacity) {
    if (!rot || !pos || !buf) return LK_ERR_INVALID_ARG;
    // Eigen::Quaterniond(Matrix3d) (Eigen/src/Geometry/Quaternion.h, quaternionbase_assign_impl<Other, 3, 3>), m(i, j) = rot[3 i + j]
    auto m = [&](int i, int j) { return rot[3 * i + j]; };
    double q[4];  // x y z w
    double t = m(0, 0) + m(1, 1) + m(2, 2);
    if (t > 0.0) {
        t = std::sqrt(t + 1.0);
        q[3] = 0.5 * t;
        t = 0.5 / t;
        q[0] = (m(2, 1) - m(1, 2)) * t;
        q[1] = (m(0, 2) - m(2, 0)) * t;
        q[2] = (m(1, 0) - m(0, 1)) * t;
    } else {
        int i = 0;
        if (m(1, 1) > m(0, 0)) i = 1;
        if (m(2, 2) > m(i, i)) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        t = std::sqrt(m(i, i) - m(j, j) - m(k, k) + 1.0);
        q[i] = 0.5 * t;
        t = 0.5 / t;
        q[3] = (m(k, j) - m(j, k)) * t;
        q[j] = (m(j, i) + m(i, j)) * t;
        q[k] = (m(k, i) + m(i, k)) * t;
    }
    const int n = std::snprintf(buf, capacity, "%.9f %.9f %.9f %.9f %.9f %.9f %.9f %.9f\n", timestamp, pos[0], pos[1], pos[2], q[0], q[1],
                                q[2], q[3]);
    if (n < 0 || (size_t)n >= capacity) return LK_ERR_CAPACITY;
    return n;
}

int lk_map_download(lk_handle h, void* blob, size_t capacity, size_t* bytes_out) {
    if (!h) return LK_ERR_INVALID_ARG;
    enter(h);
    return map_download_blob(h->map, blob, capacity, bytes_out, h->stream, h->err);
}

int lk_map_build(lk_handle h, const float* xyz_world, const float* xyz_body, size_t n, const double* rot,
                 const double* rot_cov, const double* pos_cov) {
    if (!h || !rot || !rot_cov || !pos_cov || (n && (!xyz_world || !xyz_body))) return fail(h, LK_ERR_INVALID_ARG, "null argument");
    if (n >= (1ull << 31)) return fail(h, LK_ERR_CAPACITY, "too many points for one build");
    enter(h);
    cudaStream_t s = h->stream;
    LK_CUDA(h->err, h->pts.ensure(std::max<size_t>(n, 1) * 12));
    LK_CUDA(h->err, h->world.ensure(std::max<size_t>(n, 1) * 12));
    if (n) {
        LK_CUDA(h->err, cudaMemcpyAsync(h->world.p, xyz_world, n * 12, cudaMemcpyHostToDevice, s));
        LK_CUDA(h->err, cudaMemcpyAsync(h->pts.p, xyz_body, n * 12, cudaMemcpyHostToDevice, s));
    }
    h->batch = 0;  // the staging buffers were borrowed
    std::string err;
    int rc = map_build_device(h->map, h->g, h->world.as<float>(), h->pts.as<float>(), (uint32_t)n, rot, rot_cov, pos_cov, s, err);
    return rc ? fail(h, rc, err) : LK_OK;
}

int lk_first_frame(lk_handle h, lk_state* x_inout, double* P_out, lk_stream_clock* clk_out, double* acc_norm_out,
                   const float* pts, uint32_t n_pts, double end_time, const lk_imu_meas* imu, const lk_kinimu_meas* kin,
                   uint32_t n_meas, double gravity, float* pts_world_out) {
    if (!h || !x_inout || !P_out || !clk_out || !acc_norm_out || (n_pts && !pts))
        return fail(h, LK_ERR_INVALID_ARG, "null argument");
    if (imu && kin) return fail(h, LK_ERR_INVALID_ARG, "pass either imu or kin samples, not both (imu_mode_only_, KILO.cc:379)");
    if (n_meas && !imu && !kin) return fail(h, LK_ERR_INVALID_ARG, "n_meas > 0 without samples");
    if (n_pts >= (1u << 31)) return fail(h, LK_ERR_INVALID_ARG, "too many points for one build");
    if (!n_pts || !n_meas) return fail(h, LK_ERR_NOT_READY, "data packet is not ready: empty cloud or inertial queue (KILO.cc:326-329)");
    enter(h);
    lk_state x = *x_inout;
    double acc_norm = 0.0;
    if (imu) state_initial(imu, n_meas, gravity, &x, &acc_norm);
    else state_initial(kin, n_meas, gravity, &x, &acc_norm);
    // P = 1e-6 I (state_initial.hpp:68); BuildVoxelMap takes rot = I and P's rotation / position blocks (KILO.cc:337)
    const double C[9] = {1e-6, 0.0, 0.0, 0.0, 1e-6, 0.0, 0.0, 0.0, 1e-6};
    cudaStream_t s = h->stream;
    const size_t n = n_pts;
    // h->pts = raw float4 | body xyz, h->world = world float4 | world xyz
    LK_CUDA(h->err, h->pts.ensure(n * 28));
    LK_CUDA(h->err, h->world.ensure(n * 28));
    h->batch = 0;  // the staging buffers were borrowed
    float4* d_in = h->pts.as<float4>();
    float* d_body = reinterpret_cast<float*>(d_in + n);
    float4* d_world4 = h->world.as<float4>();
    float* d_world = reinterpret_cast<float*>(d_world4 + n);
    LK_CUDA(h->err, cudaMemcpyAsync(d_in, pts, n * 16, cudaMemcpyHostToDevice, s));
    launch_first_frame_points(h->g, d_in, (uint32_t)n, x.rot, x.pos, d_body, d_world, pts_world_out ? d_world4 : nullptr, s);
    std::string err;
    const int rc = map_build_device(h->map, h->g, d_world, d_body, (uint32_t)n, x.rot, C, C, s, err);
    if (rc) return fail(h, rc, err);
    if (pts_world_out) {
        LK_CUDA(h->err, cudaMemcpyAsync(pts_world_out, d_world4, n * 16, cudaMemcpyDeviceToHost, s));
        LK_CUDA(h->err, cudaStreamSynchronize(s));
    }
    *x_inout = x;
    for (int i = 0; i < LK_DIM_STATE * LK_DIM_STATE; ++i) P_out[i] = (i % (LK_DIM_STATE + 1) == 0) ? 1e-6 : 0.0;
    clk_out->last_predict_time = clk_out->last_update_time = end_time;  // KILO.cc:350-351
    *acc_norm_out = acc_norm;
    return LK_OK;
}

// ---- batch staging / run / fetch ----------------------------------------------------------------

// Device-visible alias of a page-locked host pointer (cudaHostAlloc / cudaHostRegister), else null.
static void* pinned_device_ptr(const void* p) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    return at.type == cudaMemoryTypeHost ? at.devicePointer : nullptr;
}

static int stage_impl(lk_handle h, int batch, const lk_state* x, const double* P, const double* Q,
                      const lk_stream_clock* clk, const float* pts, const uint32_t* scan_offsets,
                      const uint32_t* scan_bucket_ptr, const uint32_t* bucket_offsets, const double* bucket_times,
                      bool sync_after, bool want_direct = false, float* world_out = nullptr) {
    if (!h) return LK_ERR_INVALID_ARG;
    enter(h);
    h->direct = h->direct_ran = h->inline_ok = false;
    if (batch <= 0 || !x || !P || !Q || !clk || !scan_offsets || !scan_bucket_ptr || !bucket_offsets || !bucket_times)
        return fail(h, LK_ERR_INVALID_ARG, "null / empty batch argument");
    const uint64_t total = scan_offsets[batch];
    if (total && !pts) return fail(h, LK_ERR_INVALID_ARG, "pts is null");
    // host-side tables: chunks grouped by step (bucket rank inside its scan)
    uint32_t max_buckets = 0;
    for (int s = 0; s < batch; ++s) {
        if (scan_offsets[s + 1] < scan_offsets[s]) return fail(h, LK_ERR_INVALID_ARG, "scan_offsets not monotone");
        uint32_t nb = scan_bucket_ptr[s + 1] - scan_bucket_ptr[s];
        max_buckets = std::max(max_buckets, nb);
        for (uint32_t b = scan_bucket_ptr[s]; b < scan_bucket_ptr[s + 1]; ++b) {
            if (bucket_offsets[b + 1] < bucket_offsets[b] || bucket_offsets[b] < scan_offsets[s] ||
                bucket_offsets[b + 1] > scan_offsets[s + 1])
                return fail(h, LK_ERR_INVALID_ARG, "bucket_offsets outside their scan");
        }
    }
    // 60 groups split evenly over the pipelined kernel's 6 warps
    const uint32_t big_chunk = 3840u;
    auto build_tables = [&](bool throughput, std::vector<ChunkDesc>& chunks, std::vector<StepInit>& inits) {
        chunks.clear();
        inits.assign((size_t)max_buckets * batch, StepInit());
        for (uint32_t k = 0; k < max_buckets; ++k) {
            for (int s = 0; s < batch; ++s) {
                StepInit& in = inits[(size_t)k * batch + s];
                std::memset(&in, 0, sizeof(in));
                in.chunk_begin = in.chunk_end = (uint32_t)chunks.size();
                uint32_t nb = scan_bucket_ptr[s + 1] - scan_bucket_ptr[s];
                if (k >= nb) continue;
                uint32_t b = scan_bucket_ptr[s] + k;
                uint32_t p0 = bucket_offsets[b], p1 = bucket_offsets[b + 1];
                in.active = 1;
                in.pt_begin = p0;
                in.pt_end = p1;
                in.t_bucket = bucket_times[b];
                in.chunk_begin = (uint32_t)chunks.size();
                uint32_t cs = chunk_size_for(p1 - p0, throughput, big_chunk);
                for (uint32_t q = p0; q < p1; q += cs) {
                    ChunkDesc cd;
                    cd.scan = (uint32_t)s;
                    cd.start = q;
                    cd.count = std::min(cs, p1 - q);
                    cd.pad = 0;
                    chunks.push_back(cd);
                }
                in.chunk_end = (uint32_t)chunks.size();
            }
        }
    };
    std::vector<ChunkDesc>& chunks = h->h_chunks;
    std::vector<ChunkDesc>& chunksL = h->h_chunksL;
    std::vector<StepInit>& inits = h->h_inits;
    build_tables(false, chunks, inits);
    bool twoTables = false;
    if (batch >= 2) {
        for (uint32_t b = 0; b < scan_bucket_ptr[batch] && !twoTables; ++b) {
            const uint32_t n = bucket_offsets[b + 1] - bucket_offsets[b];
            twoTables = chunk_size_for(n, true, big_chunk) != chunk_size_for(n, false);
        }
    }
    if (twoTables) build_tables(true, chunksL, h->h_initsL);
    else { chunksL.clear(); h->h_initsL.clear(); }
    h->batch = batch;
    h->h_scan_pts.assign(batch, 0);
    h->h_scan_chunks.assign(batch, 1);
    for (int s2 = 0; s2 < batch; ++s2) {
        h->h_scan_pts[s2] = scan_offsets[s2 + 1] - scan_offsets[s2];
        for (uint32_t k = 0; k < max_buckets; ++k) {
            const StepInit& in = inits[(size_t)k * batch + s2];
            h->h_scan_chunks[s2] = std::max(h->h_scan_chunks[s2], in.chunk_end - in.chunk_begin);
        }
    }
    h->total_pts = total;
    h->total_chunks = (uint32_t)chunks.size();
    h->max_chunk_pts = 0;
    for (const ChunkDesc& cd : chunks) h->max_chunk_pts = std::max(h->max_chunk_pts, cd.count);
    h->n_steps = max_buckets;

    LK_CUDA(h->err, h->pts.ensure(std::max<size_t>(total, 1) * 16));
    LK_CUDA(h->err, h->world.ensure(std::max<size_t>(total, 1) * 16));
    LK_CUDA(h->err, h->sc.ensure((size_t)batch * sizeof(ScanConst)));
    LK_CUDA(h->err, h->step.ensure((size_t)batch * sizeof(ScanStep)));
    LK_CUDA(h->err, h->partial.ensure(2 * std::max<size_t>(std::max(chunks.size(), chunksL.size()), 1) * PARTIAL_STRIDE * 8));
    if (batch >= 2 || h->max_chunk_pts > 256) {  // the throughput family's per-chunk fallback lists
        const size_t nch = std::max<size_t>(std::max(chunks.size(), chunksL.size()), 1);
        LK_CUDA(h->err, h->fb_list.ensure(nch * S2_FB_WARPS * S2_FB_CAP * sizeof(uint16_t)));
        LK_CUDA(h->err, h->fb_cnt.ensure(nch * S2_FB_WARPS * sizeof(uint32_t)));
    }
    if (!h->ll.p) {
        LK_CUDA(h->err, h->ll.ensure(LL_BYTES));
        LK_CUDA(h->err, cudaMemsetAsync(h->ll.p, 0, LL_BYTES, h->stream));
        h->ll_epoch = 1;
    }
    LK_CUDA(h->err, h->ticket.ensure((size_t)batch * 4));
    // ---- small inputs: one pinned block, one H2D copy ------------------------------------------
    const InBlock& in = h->in = InBlock(batch, chunks.size(), inits.size(), chunksL.size(), h->h_initsL.size());
    LK_CUDA(h->err, h->small_in.ensure(in.bytes));
    LK_CUDA(h->err, h->h_small_in.ensure(in.bytes));
    char* hs = (char*)h->h_small_in.p;
    if (!chunks.empty()) std::memcpy(hs + in.chunks, chunks.data(), chunks.size() * sizeof(ChunkDesc));
    if (!inits.empty()) std::memcpy(hs + in.inits, inits.data(), inits.size() * sizeof(StepInit));
    std::memcpy(hs + in.x, x, (size_t)batch * sizeof(lk_state));
    std::memcpy(hs + in.P, P, (size_t)batch * 900 * 8);
    std::memcpy(hs + in.clk, clk, (size_t)batch * sizeof(lk_stream_clock));
    std::memcpy(hs + in.Q, Q, 900 * 8);
    if (twoTables) {
        std::memcpy(hs + in.chunksL, chunksL.data(), chunksL.size() * sizeof(ChunkDesc));
        std::memcpy(hs + in.initsL, h->h_initsL.data(), h->h_initsL.size() * sizeof(StepInit));
    }
    char* ds = (char*)h->small_in.p;
    h->chunks.p = ds + in.chunks; h->stepinit.p = ds + in.inits; h->x_in.p = ds + in.x; h->P_in.p = ds + in.P;
    h->clk_in.p = ds + in.clk; h->Q.p = ds + in.Q;
    h->chunksL.p = twoTables ? ds + in.chunksL : ds + in.chunks;
    h->stepinitL.p = twoTables ? ds + in.initsL : ds + in.inits;
    h->total_chunksL = twoTables ? (uint32_t)chunksL.size() : (uint32_t)chunks.size();
    // ---- small outputs: one device block, fetched with one D2H copy ------------------------------
    h->out = OutBlock(batch);
    LK_CUDA(h->err, h->small_out.ensure(h->out.bytes));
    LK_CUDA(h->err, h->h_small_out.ensure(h->out.bytes));
    point_outputs(h, (char*)h->small_out.p);
    std::memset((char*)h->h_small_out.p + h->out.status, 0, 4);
    cudaStream_t s = h->stream;
    if (want_direct && h->direct_io && batch == 1 && h->lane_cache && total && h->map.ready() &&
        per_scan_kernel(h, 0, 1, false, false)) {
        const void* dp = pinned_device_ptr(pts);
        void* dw = (dp && world_out) ? pinned_device_ptr(world_out) : nullptr;
        if (dp && (dw || !world_out)) {
            h->direct = true;
            h->direct_pts = (const float4*)dp;
            h->direct_world = dw ? (float4*)dw : h->world.as<float4>();
            point_outputs(h, (char*)h->h_small_out.p);  // page-locked: the kernel stores the filter straight into it
            if (h->inline_in && max_buckets <= (uint32_t)FUSED_INLINE_STEPS) {
                if (h->Q_shadow.size() != 900 || std::memcmp(h->Q_shadow.data(), Q, 900 * 8) != 0) {
                    LK_CUDA(h->err, h->Qc.ensure(900 * 8));
                    h->Q_shadow.assign(Q, Q + 900);
                    LK_CUDA(h->err, cudaMemcpyAsync(h->Qc.p, h->Q_shadow.data(), 900 * 8, cudaMemcpyHostToDevice, s));
                    LK_CUDA(h->err, cudaStreamSynchronize(s));
                }
                h->inline_ok = true;
                h->Q.p = h->Qc.p;
            }
        }
    }
    if (total && !h->direct) LK_CUDA(h->err, cudaMemcpyAsync(h->pts.p, pts, total * 16, cudaMemcpyHostToDevice, s));
    if (!h->inline_ok) LK_CUDA(h->err, cudaMemcpyAsync(h->small_in.p, h->h_small_in.p, in.bytes, cudaMemcpyHostToDevice, s));
    if (!sync_after) return LK_OK;
    LK_CUDA(h->err, cudaStreamSynchronize(s));  // the host tables above go out of scope
    return LK_OK;
}

int lk_batch_stage(lk_handle h, int batch, const lk_state* x, const double* P, const double* Q,
                   const lk_stream_clock* clk, const float* pts, const uint32_t* scan_offsets,
                   const uint32_t* scan_bucket_ptr, const uint32_t* bucket_offsets, const double* bucket_times) {
    return stage_impl(h, batch, x, P, Q, clk, pts, scan_offsets, scan_bucket_ptr, bucket_offsets, bucket_times, true);
}

int lk_timer_start(lk_handle h) {
    if (!h) return LK_ERR_INVALID_ARG;
    enter(h);
    h->nev = 0;
    h->acc_launches = 0;
    h->acc_residual_launches = 0;
    LK_CUDA(h->err, cudaEventRecord(h->ev0, h->stream));
    return LK_OK;
}

int lk_timer_stop(lk_handle h, float* total_ms, float* residual_kernel_ms, uint32_t* n_kernel_launches,
                  uint32_t* n_residual_launches) {
    if (!h) return LK_ERR_INVALID_ARG;
    enter(h);
    LK_CUDA(h->err, cudaEventRecord(h->ev1, h->stream));
    LK_CUDA(h->err, cudaStreamSynchronize(h->stream));
    LK_CUDA(h->err, cudaGetLastError());
    {
        const int rc = check_stall(h);
        if (rc) return rc;
    }
    LK_CUDA(h->err, cudaEventElapsedTime(&h->last_total_ms, h->ev0, h->ev1));
    float rms = 0;
    for (size_t i = 0; i + 1 < h->nev; i += 2) {
        float ms = 0;
        cudaEventElapsedTime(&ms, h->kev[i], h->kev[i + 1]);
        rms += ms;
    }
    h->last_residual_ms = rms;
    h->last_launches = h->acc_launches;
    h->last_residual_launches = h->acc_residual_launches;
    if (total_ms) *total_ms = h->last_total_ms;
    if (residual_kernel_ms) *residual_kernel_ms = rms;
    if (n_kernel_launches) *n_kernel_launches = h->last_launches;
    if (n_residual_launches) *n_residual_launches = h->last_residual_launches;
    return LK_OK;
}

namespace {
// The inertial / kinematic-inertial samples lk_process_scan applies between the buckets of its scan.
struct MeasQueue {
    const lk_imu_meas* d_imu = nullptr;
    const lk_kinimu_meas* d_kin = nullptr;
    const double* stamps = nullptr;  // host copy of the stamps
    uint32_t n = 0;
    double gravity = 9.81, acc_norm = 1.0;
};
}  // namespace

// The per-scan kernel's arguments for scan `first` of the staged batch; `insert`: UpdateVoxelMap runs inside it.
static FusedArgs fused_args(lk_handle h, uint32_t first, int iters, bool insert, const MeasQueue* mq) {
    FusedArgs fa;
    std::memset(&fa, 0, sizeof(fa));
    fa.pts = h->direct ? h->direct_pts : h->pts.as<float4>();
    fa.world = h->direct ? h->direct_world : h->world.as<float4>();
    fa.inits = h->stepinit.as<StepInit>();
    fa.batch = h->batch;
    fa.n_steps = h->n_steps;
    fa.scan = first;
    fa.x_in = h->x_in.as<double>();
    fa.P_in = h->P_in.as<double>();
    fa.clk_in = h->clk_in.as<lk_stream_clock>();
    fa.Q = h->Q.as<double>();
    fa.x = h->x.as<double>();
    fa.P = h->P.as<double>();
    fa.clk = h->clk.as<lk_stream_clock>();
    fa.n_eff = h->n_eff.as<uint32_t>();
    fa.status = h->status.as<uint32_t>();
    fa.ll.chunk_rows = h->ll.as<ulonglong2>();
    fa.ll.group_rows = h->ll.as<ulonglong2>() + (size_t)2 * LL_MAX_CHUNKS * LL_ROW;
    fa.ll.stall = reinterpret_cast<uint32_t*>((char*)h->ll.p + LL_ROWS_BYTES);
    fa.ll.acks = reinterpret_cast<uint32_t*>((char*)h->ll.p + LL_ROWS_BYTES + 64);
    fa.epoch = h->ll_epoch;
    fa.iters = iters;
    fa.lane_cache = h->lane_cache;
    {
        // "no predict": one bucket whose time equals both clocks of the staged filter
        const lk_stream_clock* ck = reinterpret_cast<const lk_stream_clock*>((const char*)h->h_small_in.p + h->in.clk) + first;
        const StepInit& in0 = h->h_inits[first];
        fa.slim_p = h->slim_p && h->n_steps == 1 && !mq && in0.active && in0.t_bucket == ck->last_predict_time &&
                    in0.t_bucket == ck->last_update_time;
    }
    fa.mv = h->map.view();
    if (mq) {
        fa.imu = mq->d_imu;
        fa.kin = mq->d_kin;
        fa.n_meas = mq->n;
        fa.gravity = mq->gravity;
        fa.acc_norm = mq->acc_norm;
    }
    {
        // finishers: one active bucket without a queue or insert, and SMs the chunks leave idle
        const StepInit& in0 = h->h_inits[first];
        const uint32_t sms = (uint32_t)fused_max_blocks(h->device), chunks = h->h_scan_chunks[first];
        if (h->finishers && !insert && fa.n_meas == 0 && h->n_steps == 1 && in0.active && in0.chunk_end - in0.chunk_begin == chunks &&
            chunks > 0 && iters >= 1 && chunks < sms) {  // the kernel's workers are then blocks [0, chunks)
            fa.finishers = std::min(sms - chunks, (uint32_t)LL_MAX_FINISHERS);
            // a finisher never reads host memory: in direct mode the workers copy their points to the staging buffer
            if (h->direct) fa.pts_copy = h->pts.as<float4>();
        }
    }
    fa.ecfg = h->ec;
    // back-to-back launches trace into consecutive areas (TRACE_AREA stamps each, TRACE_AREAS of them, cycling), so the
    // overlap of one launch with the next can be read back; the first launch after lk_debug_read starts again at area 0
    fa.trace = h->trace_on ? h->trace.as<unsigned long long>() + (size_t)(h->trace_seq++ % TRACE_AREAS) * TRACE_AREA : nullptr;
    fa.g = h->g;
    if (insert) {
        fa.insert = 1;
        fa.md = h->map.dev();
        h->inserter.fused_scratch(fa);
    }
    return fa;
}

// One scan: the whole bucket loop in ONE persistent kernel, one chunk per block (lk_fused.cu). With the map insert
// inside, every SM gets a block: the buckets' points sit in the first few, but the insert phase hands one touched root
// voxel to every warp of the grid.
static int run_fused(lk_handle h, uint32_t first, int iters, bool insert, const MeasQueue* mq, bool timed) {
    cudaStream_t s = h->stream;
    FusedInline* inl = nullptr;
    if (h->inline_ok) {  // the staged filter and step table ride in the parameter block
        const char* hs = (const char*)h->h_small_in.p;
        inl = &h->inl;
        std::memcpy(inl->x, hs + h->in.x, sizeof(inl->x));
        std::memcpy(inl->P, hs + h->in.P, sizeof(inl->P));
        std::memcpy(inl->clk, hs + h->in.clk, sizeof(inl->clk));
        std::memcpy(inl->steps, h->h_inits.data(), h->h_inits.size() * sizeof(StepInit));
    }
    // tags of the flagged rows: one per (step, iteration); restart (with a cleared buffer) long before the 32-bit wrap
    const uint32_t need = h->n_steps * ((uint32_t)iters + 2u) + 1u;  // + two barriers per bucket with the insert inside
    if (h->ll_epoch > 0xE0000000u || need > 0x10000000u) {
        if (need > 0x10000000u) return fail(h, LK_ERR_INVALID_ARG, "steps x iters too large for one launch");
        LK_CUDA(h->err, cudaMemsetAsync(h->ll.p, 0, LL_BYTES, s));
        h->ll_epoch = 1;
        h->prev_fused = false;
    }
    const FusedArgs fa = fused_args(h, first, iters, insert, mq);
    const uint32_t grid = insert ? (uint32_t)fused_max_blocks(h->device) : h->h_scan_chunks[first] + fa.finishers;
    h->ll_epoch += need;
    if (insert) h->prev_fused = false;  // the insert counters were cleared by a memset on the stream
    if (timed) { cudaEventRecord(kev_get(h, h->nev++), s); h->prev_fused = false; }
    const int mode = h->coop_launch ? FUSED_LAUNCH_COOPERATIVE : ((h->pdl && h->prev_fused) ? FUSED_LAUNCH_PDL : FUSED_LAUNCH_PLAIN);
    {
        // Blocks of this kernel poll for each other's rows: two such grids must never share the device half
        // resident. Launches of one stream are ordered by the stream; launches of different handles of this
        // process are ordered here (the later one waits for everything the earlier stream has queued).
        FusedGate& gate = fused_gate(h->device);
        std::lock_guard<std::mutex> lock(gate.m);
        if (gate.last && gate.last != s) {
            if (!gate.ev) LK_CUDA(h->err, cudaEventCreateWithFlags(&gate.ev, cudaEventDisableTiming));
            LK_CUDA(h->err, cudaEventRecord(gate.ev, gate.last));
            LK_CUDA(h->err, cudaStreamWaitEvent(s, gate.ev, 0));
        }
        gate.last = s;
        LK_CUDA(h->err, launch_scan_fused(fa, inl, grid, s, mode));
    }
    h->prev_fused = true;
    ++h->fused_launches_since_check;
    if (timed) { cudaEventRecord(kev_get(h, h->nev++), s); h->prev_fused = false; }
    ++h->acc_launches;
    ++h->acc_residual_launches;
    h->direct_ran = h->direct;
    return LK_OK;
}

// The multi-kernel path: per bucket a predict launch, the residual / solve launches of every iteration, and the
// re-projection and map insert. >= 2 scans per call use the throughput family and its chunk table (see chunk_size_for).
static int run_kernels(lk_handle h, uint32_t first, uint32_t count, int iters, bool update_map, const MeasQueue* mq,
                       bool timed) {
    cudaStream_t s = h->stream;
    const int batch = h->batch;
    const bool big = count >= 2 && !h->h_initsL.empty();
    const std::vector<StepInit>& tin = big ? h->h_initsL : h->h_inits;
    const ChunkDesc* d_chunks = big ? h->chunksL.as<ChunkDesc>() : h->chunks.as<ChunkDesc>();
    const StepInit* d_inits = big ? h->stepinitL.as<StepInit>() : h->stepinit.as<StepInit>();
    uint32_t mi = 0;
    if (mq) {  // the queue is applied BEFORE bucket 0 as well, so the filter is re-loaded here, not in the kernel
        LK_CUDA(h->err, cudaMemcpyAsync(h->x.as<lk_state>() + first, h->x_in.as<lk_state>() + first, sizeof(lk_state), cudaMemcpyDeviceToDevice, s));
        LK_CUDA(h->err, cudaMemcpyAsync(h->P.as<double>() + (size_t)first * 900, h->P_in.as<double>() + (size_t)first * 900, 900 * 8, cudaMemcpyDeviceToDevice, s));
        LK_CUDA(h->err, cudaMemcpyAsync(h->clk.as<lk_stream_clock>() + first, h->clk_in.as<lk_stream_clock>() + first, sizeof(lk_stream_clock), cudaMemcpyDeviceToDevice, s));
        LK_CUDA(h->err, cudaMemsetAsync(h->n_eff.as<uint32_t>() + first, 0, 4, s));
    }
    for (uint32_t k = 0; k < h->n_steps; ++k) {
        const StepInit* hin = tin.data() + (size_t)k * batch;
        uint32_t c0 = hin[first].chunk_begin, c1 = hin[first + count - 1].chunk_end;
        uint32_t m_obs0 = mi, m_obs1 = mi;  // samples with stamp < bucket time (KILO.cc:379-390)
        if (mq && hin[first].active) {
            while (m_obs1 < mq->n && mq->stamps[m_obs1] < hin[first].t_bucket) ++m_obs1;
            mi = m_obs1;
        }
        const PredictArgs pa = predict_args(h, d_inits + (size_t)k * batch, (k == 0 && !mq) ? 1 : 0, first, count);
        if (mq && count == 1 && hin[first].active)  // the queue drain and the bucket's predict share one launch and one copy of the filter
            launch_obs_predict_prepare(pa, mq->d_imu ? mq->d_imu + m_obs0 : nullptr, mq->d_kin ? mq->d_kin + m_obs0 : nullptr,
                                       m_obs1 - m_obs0, h->ec, mq->gravity, mq->acc_norm, s);
        else
            launch_predict_prepare(pa, s);
        ++h->acc_launches;
        for (int it = 0; it < iters; ++it) {
            ResidualArgs ra = residual_args(h, d_chunks);
            ra.chunk_first = c0;
            ra.last_iter = (it == iters - 1) ? 1 : 0;
            if (timed) cudaEventRecord(kev_get(h, h->nev++), s);
            // latency variant only for a single scan: the kernel family must not depend on how a batch is
            // sharded (bitwise-reproducible sums)
            if (count >= 2 || h->max_chunk_pts > 256) {
                launch_residual_stream2(ra, c1 - c0, s);
                launch_residual_fallback(ra, c1 - c0, s);
                launch_scan_tail(ra, first, count, s);
                if (c1 > c0) h->acc_launches += 2;
            } else {
                launch_residual(ra, c1 - c0, false, !update_map, s);
            }
            if (timed) cudaEventRecord(kev_get(h, h->nev++), s);
            if (c1 > c0) { ++h->acc_launches; ++h->acc_residual_launches; }
        }
        // KILO.cc:231 — the map insert runs always, even when no update happened. With fast_insert its first phase also
        // stores the re-projected cloud, so the re-projection kernel only runs without it.
        const bool insert = update_map && c1 > c0;
        const bool insert_reprojects = insert && h->fast_insert;
        if (!insert_reprojects) {
            ReprojectArgs rp;
            rp.pts = h->pts.as<float4>();
            rp.world = h->world.as<float4>();
            rp.chunks = d_chunks;
            rp.chunk_first = c0;
            rp.sc = h->sc.as<ScanConst>();
            rp.step = h->step.as<ScanStep>();
            rp.g = h->g;
            launch_reproject(rp, c1 - c0, s);
            if (c1 > c0) ++h->acc_launches;
        }
        if (insert) {
            const StepInit& in = hin[first];
            h->acc_launches += h->inserter.bucket(h->map, h->g, h->pts.as<float4>(), d_chunks, c0, c1 - c0, in.pt_begin,
                                                  in.pt_end - in.pt_begin, h->sc.as<ScanConst>(), h->step.as<ScanStep>(), s,
                                                  insert_reprojects ? h->world.as<float4>() : nullptr);
        }
    }
    LK_CUDA(h->err, cudaGetLastError());
    return LK_OK;
}

// Enqueue the hot path for scans [first, first+count) of the staged batch; no host sync unless update_map.
// timed: bracket the residual launches with events for lk_timer_stop.
static int run_range_impl(lk_handle h, uint32_t first, uint32_t count, int iters, int update_map, const MeasQueue* mq,
                          bool timed) {
    if (!h) return LK_ERR_INVALID_ARG;
    if (h->batch <= 0) return fail(h, LK_ERR_NOT_READY, "lk_batch_run before lk_batch_stage");
    if (iters < 1) return fail(h, LK_ERR_INVALID_ARG, "iters must be >= 1");
    if (count == 0 || first + count > (uint32_t)h->batch) return fail(h, LK_ERR_INVALID_ARG, "scan range outside the staged batch");
    if (update_map && count != 1)
        return fail(h, LK_ERR_INVALID_ARG, "update_map inserts into this handle's map: run one scan (stream) per call");
    uint32_t max_bucket = 0;
    if (update_map) {
        for (uint32_t k = 0; k < h->n_steps; ++k) {
            const StepInit& in = h->h_inits[(size_t)k * h->batch + first];
            max_bucket = std::max(max_bucket, in.pt_end - in.pt_begin);
        }
        const int rc = h->inserter.begin(h->map, h->g, h->h_scan_pts[first], max_bucket, h->stream, h->err);
        if (rc) return rc;
    }
    if (!h->map.ready()) return fail(h, LK_ERR_NOT_READY, "no map: call lk_map_upload or lk_map_build first");
    // update_map inside the persistent kernel: buckets of up to 4 096 points (the root-per-point scan of its insert phase)
    const bool fused_ins = update_map && h->fast_insert && h->fused_insert && max_bucket <= 4096u;
    const bool fused = per_scan_kernel(h, first, count, update_map, fused_ins);
    if (!fused) h->prev_fused = false;
    // direct staging filled only what the per-scan kernel reads (caller buffers, parameter block), not pts / small_in
    if (!fused && h->direct)
        return fail(h, LK_ERR_CUDA, "batch staged by lk_scan_update for the per-scan kernel: re-stage it to run it another way");
    int rc = fused ? run_fused(h, first, iters, update_map, mq, timed) : run_kernels(h, first, count, iters, update_map, mq, timed);
    if (rc || !update_map) return rc;
    // update_map: the caller observes a finished insert; a per-scan kernel that gave up waiting reports that, not the pools
    h->prev_fused = false;
    rc = h->map.sync_counters(h->stream, h->err);
    if (!rc && fused) rc = check_stall(h);
    return rc ? rc : h->inserter.finish(h->map, h->err);
}

int lk_map_insert(lk_handle h, uint32_t n_sets, const float* pts, const uint32_t* set_offsets, const double* rot,
                  const double* pos, const double* rot_cov, const double* pos_cov) {
    if (!h) return LK_ERR_INVALID_ARG;
    if (n_sets == 0) return LK_OK;
    if (!pts || !set_offsets || !rot || !pos || !rot_cov || !pos_cov) return fail(h, LK_ERR_INVALID_ARG, "null argument");
    for (uint32_t s = 0; s < n_sets; ++s) {
        if (set_offsets[s + 1] < set_offsets[s]) return fail(h, LK_ERR_INVALID_ARG, "set_offsets not monotone");
        if (!all_finite(rot + 9 * (size_t)s, 9) || !all_finite(rot_cov + 9 * (size_t)s, 9) ||
            !all_finite(pos_cov + 9 * (size_t)s, 9) || !all_finite(pos + 3 * (size_t)s, 3))
            return fail(h, LK_ERR_INVALID_ARG, "non-finite pose or covariance");
    }
    enter(h);
    return h->inserter.insert_sets(h->map, h->g, n_sets, pts, set_offsets, rot, pos, rot_cov, pos_cov, h->stream, h->err);
}

// The inputs lk_score_poses and lk_refine_poses share, checked as the header documents for both (n_poses > 0).
static int score_check(lk_handle h, uint32_t n_sets, const float* pts, const uint32_t* set_offsets, uint32_t n_poses,
                       const uint32_t* pose_set, const double* rot, const double* pos, const double* rot_cov,
                       const double* pos_cov) {
    if (!pts || !set_offsets || !pose_set || !rot || !pos || !rot_cov || !pos_cov)
        return fail(h, LK_ERR_INVALID_ARG, "null argument");
    for (uint32_t s = 0; s < n_sets; ++s)
        if (set_offsets[s + 1] < set_offsets[s]) return fail(h, LK_ERR_INVALID_ARG, "set_offsets not monotone");
    for (uint32_t m = 0; m < n_poses; ++m)
        if (pose_set[m] >= n_sets) return fail(h, LK_ERR_INVALID_ARG, "pose_set names a set past n_sets");
    if (!all_finite(rot_cov, 9) || !all_finite(pos_cov, 9) || !all_finite(rot, 9 * (size_t)n_poses) ||
        !all_finite(pos, 3 * (size_t)n_poses))
        return fail(h, LK_ERR_INVALID_ARG, "non-finite pose or covariance");
    if (!h->map.ready()) return fail(h, LK_ERR_NOT_READY, "no map: call lk_map_upload or lk_map_build first");
    return LK_OK;
}

int lk_score_poses(lk_handle h, uint32_t n_sets, const float* pts, const uint32_t* set_offsets, uint32_t n_poses,
                   const uint32_t* pose_set, const double* rot, const double* pos, const double* rot_cov,
                   const double* pos_cov, double* sums_out) {
    if (!h) return LK_ERR_INVALID_ARG;
    if (n_poses == 0) return LK_OK;
    if (!sums_out) return fail(h, LK_ERR_INVALID_ARG, "null argument");
    if (int rc = score_check(h, n_sets, pts, set_offsets, n_poses, pose_set, rot, pos, rot_cov, pos_cov)) return rc;
    enter(h);
    return h->scorer.run(h->map, h->g, n_sets, pts, set_offsets, n_poses, pose_set, rot, pos, rot_cov, pos_cov, 0, nullptr,
                         nullptr, sums_out, h->stream, h->err);
}

int lk_refine_poses(lk_handle h, uint32_t n_sets, const float* pts, const uint32_t* set_offsets, uint32_t n_poses,
                    const uint32_t* pose_set, const double* rot, const double* pos, const double* rot_cov,
                    const double* pos_cov, int iters, double* rot_out, double* pos_out, double* sums_out) {
    if (!h) return LK_ERR_INVALID_ARG;
    if (n_poses == 0) return LK_OK;
    if (!rot_out || !pos_out) return fail(h, LK_ERR_INVALID_ARG, "null argument");
    if (iters < 1) return fail(h, LK_ERR_INVALID_ARG, "iters < 1");
    if (int rc = score_check(h, n_sets, pts, set_offsets, n_poses, pose_set, rot, pos, rot_cov, pos_cov)) return rc;
    enter(h);
    return h->scorer.run(h->map, h->g, n_sets, pts, set_offsets, n_poses, pose_set, rot, pos, rot_cov, pos_cov, iters, rot_out,
                         pos_out, sums_out, h->stream, h->err);
}

int lk_search_poses(lk_handle h, uint32_t n_sets, const float* pts, const uint32_t* set_offsets, const uint32_t* att_offsets,
                    const double* att_rot, const double* origin, const double step[3], const uint32_t counts[3],
                    const double* rot_cov, const double* pos_cov, int iters, const double* rot_cov_tight,
                    const double* pos_cov_tight, uint32_t k, double* rot_out, double* pos_out, double* sums_out,
                    uint32_t* cand_out) {
    if (!h) return LK_ERR_INVALID_ARG;
    if (n_sets == 0) return LK_OK;
    if (!pts || !set_offsets || !att_offsets || !att_rot || !origin || !step || !counts || !rot_cov || !pos_cov ||
        !rot_cov_tight || !pos_cov_tight || !rot_out || !pos_out || !sums_out || !cand_out)
        return fail(h, LK_ERR_INVALID_ARG, "null argument");
    for (uint32_t s = 0; s < n_sets; ++s) {
        if (set_offsets[s + 1] < set_offsets[s]) return fail(h, LK_ERR_INVALID_ARG, "set_offsets not monotone");
        if (att_offsets[s + 1] < att_offsets[s]) return fail(h, LK_ERR_INVALID_ARG, "att_offsets not monotone");
    }
    if (!counts[0] || !counts[1] || !counts[2]) return fail(h, LK_ERR_INVALID_ARG, "a zero lattice count");
    if (k == 0 || k > LK_SEARCH_MAX_K) return fail(h, LK_ERR_INVALID_ARG, "k outside 1 .. LK_SEARCH_MAX_K");
    if (iters < 1) return fail(h, LK_ERR_INVALID_ARG, "iters < 1");
    if (!all_finite(att_rot + 9 * (size_t)att_offsets[0], 9 * (size_t)(att_offsets[n_sets] - att_offsets[0])) ||
        !all_finite(origin, 3 * (size_t)n_sets) || !all_finite(step, 3) || !all_finite(rot_cov, 9) ||
        !all_finite(pos_cov, 9) || !all_finite(rot_cov_tight, 9) || !all_finite(pos_cov_tight, 9))
        return fail(h, LK_ERR_INVALID_ARG, "non-finite attitude, origin, step or covariance");
    for (uint32_t s = 0; s < n_sets; ++s) {  // attitudes x lattice, stopping once past 2^32 (no factor reaches 2^32)
        uint64_t n = att_offsets[s + 1] - att_offsets[s];
        for (int j = 0; j < 3 && n < (1ull << 32); ++j) n *= counts[j];
        if (n >= (1ull << 32)) return fail(h, LK_ERR_INVALID_ARG, "a set with 2^32 or more candidates");
        if (n < k) return fail(h, LK_ERR_INVALID_ARG, "a set with fewer than k candidates");
    }
    if (!h->map.ready()) return fail(h, LK_ERR_NOT_READY, "no map: call lk_map_upload or lk_map_build first");
    enter(h);
    return h->scorer.search(h->map, h->g, n_sets, pts, set_offsets, att_offsets, att_rot, origin, step, counts, rot_cov,
                            pos_cov, iters, rot_cov_tight, pos_cov_tight, k, rot_out, pos_out, sums_out, cand_out, h->stream,
                            h->err);
}

int lk_batch_run_range(lk_handle h, uint32_t first, uint32_t count, int iters, int update_map) {
    if (!h) return LK_ERR_INVALID_ARG;
    // not enter(): prev_fused is kept, so that back-to-back fused launches of one stream chain by PDL
    cudaSetDevice(h->device);
    return run_range_impl(h, first, count, iters, update_map, nullptr, h->kernel_timing != 0);
}

int lk_batch_run(lk_handle h, int iters, int update_map) {
    if (!h) return LK_ERR_INVALID_ARG;
    if (h->batch <= 0) return fail(h, LK_ERR_NOT_READY, "lk_batch_run before lk_batch_stage");
    int rc = lk_timer_start(h);
    if (rc) return rc;
    rc = lk_batch_run_range(h, 0, (uint32_t)h->batch, iters, update_map);
    if (rc) return rc;
    return lk_timer_stop(h, nullptr, nullptr, nullptr, nullptr);
}

int lk_batch_fetch(lk_handle h, lk_state* x_out, double* P_out, lk_stream_clock* clk_out, float* pts_world_out,
                   uint32_t* n_effective_out) {
    if (!h) return LK_ERR_INVALID_ARG;
    if (h->batch <= 0) return fail(h, LK_ERR_NOT_READY, "nothing staged");
    enter(h);
    cudaStream_t s = h->stream;
    const int batch = h->batch;
    const bool small = x_out || P_out || clk_out || n_effective_out;
    if (!h->direct_ran) {  // direct mode: the kernel already stored both into page-locked host memory
        if (small) LK_CUDA(h->err, cudaMemcpyAsync(h->h_small_out.p, h->small_out.p, h->out.bytes, cudaMemcpyDeviceToHost, s));
        if (pts_world_out && h->total_pts)
            LK_CUDA(h->err, cudaMemcpyAsync(pts_world_out, h->world.p, h->total_pts * 16, cudaMemcpyDeviceToHost, s));
    } else if (pts_world_out && h->direct_world == h->world.as<float4>() && h->total_pts) {
        LK_CUDA(h->err, cudaMemcpyAsync(pts_world_out, h->world.p, h->total_pts * 16, cudaMemcpyDeviceToHost, s));
    }
    LK_CUDA(h->err, cudaStreamSynchronize(s));
    LK_CUDA(h->err, cudaGetLastError());
    const char* ho = (const char*)h->h_small_out.p;
    if (small && h->fused_launches_since_check) {
        // the per-scan kernel leaves one status word with its outputs: only a non-zero one is worth the detailed read-back
        uint32_t st;
        std::memcpy(&st, ho + h->out.status, 4);
        if (st) {
            const int rc = check_stall(h);
            if (rc) return rc;
        }
        h->fused_launches_since_check = 0;
    }
    if (x_out) std::memcpy(x_out, ho + h->out.x, (size_t)batch * sizeof(lk_state));
    if (P_out) std::memcpy(P_out, ho + h->out.P, (size_t)batch * 900 * 8);
    if (clk_out) std::memcpy(clk_out, ho + h->out.clk, (size_t)batch * sizeof(lk_stream_clock));
    if (n_effective_out) std::memcpy(n_effective_out, ho + h->out.n_eff, (size_t)batch * 4);
    return LK_OK;
}

int lk_batch_last_timing(lk_handle h, float* total_ms, float* residual_kernel_ms, uint32_t* n_kernel_launches,
                         uint32_t* n_residual_launches) {
    if (!h) return LK_ERR_INVALID_ARG;
    if (total_ms) *total_ms = h->last_total_ms;
    if (residual_kernel_ms) *residual_kernel_ms = h->last_residual_ms;
    if (n_kernel_launches) *n_kernel_launches = h->last_launches;
    if (n_residual_launches) *n_residual_launches = h->last_residual_launches;
    return LK_OK;
}

int lk_scan_update(lk_handle h, int batch, lk_state* x_inout, double* P_inout, const double* Q,
                   lk_stream_clock* clk_inout, const float* pts, const uint32_t* scan_offsets,
                   const uint32_t* scan_bucket_ptr, const uint32_t* bucket_offsets, const double* bucket_times, int iters,
                   int update_map, float* pts_world_out, uint32_t* n_effective_out) {
    // one packed H2D (+ the points), the kernels, one packed D2H (+ the world cloud), ONE host sync
    using clock = std::chrono::steady_clock;
    const auto t0 = clock::now();
    int rc = stage_impl(h, batch, x_inout, P_inout, Q, clk_inout, pts, scan_offsets, scan_bucket_ptr, bucket_offsets,
                        bucket_times, false, !update_map, pts_world_out);
    if (rc) return rc;
    const auto t1 = clock::now();
    h->nev = 0;
    rc = run_range_impl(h, 0, (uint32_t)batch, iters, update_map, nullptr, false);
    if (rc) return rc;
    const auto t2 = clock::now();
    rc = lk_batch_fetch(h, x_inout, P_inout, clk_inout, pts_world_out, n_effective_out);
    const auto t3 = clock::now();
    h->hprof[0] += std::chrono::duration<double, std::nano>(t1 - t0).count();
    h->hprof[1] += std::chrono::duration<double, std::nano>(t2 - t1).count();
    h->hprof[2] += std::chrono::duration<double, std::nano>(t3 - t2).count();
    h->hprof[3] += 1.0;
    return rc;
}

int lk_debug_residuals(lk_handle h, const lk_state* x, const double* P, const float* pts, uint32_t n, uint8_t* ok_out,
                       double* h_out, double* z_out, double* R_out, int32_t* key_out) {
    if (!h || !x || !P || (!pts && n)) return fail(h, LK_ERR_INVALID_ARG, "null argument");
    if (!h->map.ready()) return fail(h, LK_ERR_NOT_READY, "no map");
    std::vector<double> Q(900, 0.0);
    lk_stream_clock clk = {0.0, 0.0};
    uint32_t so[2] = {0, n}, sb[2] = {0, 1}, bo[2] = {0, n};
    double bt[1] = {0.0};
    int rc = lk_batch_stage(h, 1, x, P, Q.data(), &clk, pts, so, sb, bo, bt);
    if (rc) return rc;
    cudaStream_t s = h->stream;
    size_t nn = std::max<size_t>(n, 1);
    LK_CUDA(h->err, h->dbg_ok.ensure(nn));
    LK_CUDA(h->err, h->dbg_h.ensure(nn * 48));
    LK_CUDA(h->err, h->dbg_z.ensure(nn * 8));
    LK_CUDA(h->err, h->dbg_R.ensure(nn * 8));
    LK_CUDA(h->err, h->dbg_key.ensure(nn * 12));
    launch_predict_prepare(predict_args(h, h->stepinit.as<StepInit>(), 1, 0, 1), s);
    ResidualArgs ra = residual_args(h, h->chunks.as<ChunkDesc>());
    ra.chunk_first = 0;
    ra.dbg_ok = h->dbg_ok.as<uint8_t>();
    ra.dbg_h = h->dbg_h.as<double>();
    ra.dbg_z = h->dbg_z.as<double>();
    ra.dbg_R = h->dbg_R.as<double>();
    ra.dbg_key = h->dbg_key.as<int32_t>();
    launch_residual(ra, h->total_chunks, true, !h->debug_records, s);
    LK_CUDA(h->err, cudaGetLastError());
    if (n) {
        if (ok_out) LK_CUDA(h->err, cudaMemcpyAsync(ok_out, h->dbg_ok.p, n, cudaMemcpyDeviceToHost, s));
        if (h_out) LK_CUDA(h->err, cudaMemcpyAsync(h_out, h->dbg_h.p, (size_t)n * 48, cudaMemcpyDeviceToHost, s));
        if (z_out) LK_CUDA(h->err, cudaMemcpyAsync(z_out, h->dbg_z.p, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
        if (R_out) LK_CUDA(h->err, cudaMemcpyAsync(R_out, h->dbg_R.p, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
        if (key_out) LK_CUDA(h->err, cudaMemcpyAsync(key_out, h->dbg_key.p, (size_t)n * 12, cudaMemcpyDeviceToHost, s));
    }
    LK_CUDA(h->err, cudaStreamSynchronize(s));
    return LK_OK;
}

// ---- filter steps ---------------------------------------------------------------------------------

int lk_predict(lk_handle h, int batch, lk_state* x_inout, double* P_inout, const double* Q, const double* dt,
               int prop_state, int prop_cov) {
    if (!h || batch <= 0 || !x_inout || !P_inout || !Q || !dt) return fail(h, LK_ERR_INVALID_ARG, "null argument");
    enter(h);
    cudaStream_t s = h->stream;
    LK_CUDA(h->err, h->fx.ensure((size_t)batch * sizeof(lk_state)));
    LK_CUDA(h->err, h->fP.ensure((size_t)batch * 900 * 8));
    LK_CUDA(h->err, h->fQ.ensure(900 * 8));
    LK_CUDA(h->err, h->tmp.ensure((size_t)batch * 8));
    LK_CUDA(h->err, cudaMemcpyAsync(h->fx.p, x_inout, (size_t)batch * sizeof(lk_state), cudaMemcpyHostToDevice, s));
    LK_CUDA(h->err, cudaMemcpyAsync(h->fP.p, P_inout, (size_t)batch * 900 * 8, cudaMemcpyHostToDevice, s));
    LK_CUDA(h->err, cudaMemcpyAsync(h->fQ.p, Q, 900 * 8, cudaMemcpyHostToDevice, s));
    LK_CUDA(h->err, cudaMemcpyAsync(h->tmp.p, dt, (size_t)batch * 8, cudaMemcpyHostToDevice, s));
    launch_predict_dt(h->fx.as<double>(), h->fP.as<double>(), h->fQ.as<double>(), h->tmp.as<double>(), batch, prop_state,
                      prop_cov, s);
    LK_CUDA(h->err, cudaGetLastError());
    LK_CUDA(h->err, cudaMemcpyAsync(x_inout, h->fx.p, (size_t)batch * sizeof(lk_state), cudaMemcpyDeviceToHost, s));
    LK_CUDA(h->err, cudaMemcpyAsync(P_inout, h->fP.p, (size_t)batch * 900 * 8, cudaMemcpyDeviceToHost, s));
    LK_CUDA(h->err, cudaStreamSynchronize(s));
    return LK_OK;
}

// The one-filter steps below work on fx / fP / fQ / fclk and leave a staged batch untouched.
namespace {
int filter_upload(lk_handle h, const lk_state* x, const double* P, const double* Q, const lk_stream_clock* clk) {
    cudaStream_t s = h->stream;
    LK_CUDA(h->err, h->fx.ensure(sizeof(lk_state)));
    LK_CUDA(h->err, h->fP.ensure(900 * 8));
    LK_CUDA(h->err, h->fQ.ensure(900 * 8));
    LK_CUDA(h->err, h->fclk.ensure(sizeof(lk_stream_clock)));
    LK_CUDA(h->err, cudaMemcpyAsync(h->fx.p, x, sizeof(lk_state), cudaMemcpyHostToDevice, s));
    LK_CUDA(h->err, cudaMemcpyAsync(h->fP.p, P, 900 * 8, cudaMemcpyHostToDevice, s));
    if (Q) LK_CUDA(h->err, cudaMemcpyAsync(h->fQ.p, Q, 900 * 8, cudaMemcpyHostToDevice, s));
    if (clk) LK_CUDA(h->err, cudaMemcpyAsync(h->fclk.p, clk, sizeof(lk_stream_clock), cudaMemcpyHostToDevice, s));
    return LK_OK;
}
int filter_download(lk_handle h, lk_state* x, double* P, lk_stream_clock* clk) {
    cudaStream_t s = h->stream;
    LK_CUDA(h->err, cudaGetLastError());
    LK_CUDA(h->err, cudaMemcpyAsync(x, h->fx.p, sizeof(lk_state), cudaMemcpyDeviceToHost, s));
    LK_CUDA(h->err, cudaMemcpyAsync(P, h->fP.p, 900 * 8, cudaMemcpyDeviceToHost, s));
    if (clk) LK_CUDA(h->err, cudaMemcpyAsync(clk, h->fclk.p, sizeof(lk_stream_clock), cudaMemcpyDeviceToHost, s));
    LK_CUDA(h->err, cudaStreamSynchronize(s));
    return LK_OK;
}
}  // namespace

int lk_update_by_points(lk_handle h, lk_state* x_inout, double* P_inout, uint32_t n, const double* pt_h, const double* pt_z,
                        const double* pt_R) {
    if (!h || !x_inout || !P_inout || (n && (!pt_h || !pt_z || !pt_R))) return fail(h, LK_ERR_INVALID_ARG, "null argument");
    enter(h);
    if (n == 0) return LK_OK;  // KILO.cc:188: no residual, no update
    int rc = filter_upload(h, x_inout, P_inout, nullptr, nullptr);
    if (rc) return rc;
    cudaStream_t s = h->stream;
    LK_CUDA(h->err, h->dbg_h.ensure((size_t)n * 48));
    LK_CUDA(h->err, h->dbg_z.ensure((size_t)n * 8));
    LK_CUDA(h->err, h->dbg_R.ensure((size_t)n * 8));
    LK_CUDA(h->err, cudaMemcpyAsync(h->dbg_h.p, pt_h, (size_t)n * 48, cudaMemcpyHostToDevice, s));
    LK_CUDA(h->err, cudaMemcpyAsync(h->dbg_z.p, pt_z, (size_t)n * 8, cudaMemcpyHostToDevice, s));
    LK_CUDA(h->err, cudaMemcpyAsync(h->dbg_R.p, pt_R, (size_t)n * 8, cudaMemcpyHostToDevice, s));
    launch_update_by_points(h->fx.as<double>(), h->fP.as<double>(), n, h->dbg_h.as<double>(), h->dbg_z.as<double>(),
                            h->dbg_R.as<double>(), s);
    return filter_download(h, x_inout, P_inout, nullptr);
}

int lk_obs_imu(lk_handle h, lk_state* x_inout, double* P_inout, const double* Q, lk_stream_clock* clk_inout,
               const lk_imu_meas* imu, uint32_t n, double gravity, double acc_norm) {
    if (!h || !x_inout || !P_inout || !Q || !clk_inout || (n && !imu)) return fail(h, LK_ERR_INVALID_ARG, "null argument");
    enter(h);
    if (n == 0) return LK_OK;
    int rc = filter_upload(h, x_inout, P_inout, Q, clk_inout);
    if (rc) return rc;
    LK_CUDA(h->err, h->tmp.ensure((size_t)n * sizeof(lk_imu_meas)));
    LK_CUDA(h->err, cudaMemcpyAsync(h->tmp.p, imu, (size_t)n * sizeof(lk_imu_meas), cudaMemcpyHostToDevice, h->stream));
    launch_filter_obs(h->fx.as<double>(), h->fP.as<double>(), h->fQ.as<double>(), h->fclk.as<lk_stream_clock>(),
                      h->tmp.as<lk_imu_meas>(), nullptr, n, h->ec, gravity, acc_norm, h->stream);
    return filter_download(h, x_inout, P_inout, clk_inout);
}

int lk_obs_kinimu(lk_handle h, lk_state* x_inout, double* P_inout, const double* Q, lk_stream_clock* clk_inout,
                  const lk_kinimu_meas* kin, uint32_t n, double gravity, double acc_norm) {
    if (!h || !x_inout || !P_inout || !Q || !clk_inout || (n && !kin)) return fail(h, LK_ERR_INVALID_ARG, "null argument");
    enter(h);
    if (n == 0) return LK_OK;
    int rc = filter_upload(h, x_inout, P_inout, Q, clk_inout);
    if (rc) return rc;
    LK_CUDA(h->err, h->tmp.ensure((size_t)n * sizeof(lk_kinimu_meas)));
    LK_CUDA(h->err, cudaMemcpyAsync(h->tmp.p, kin, (size_t)n * sizeof(lk_kinimu_meas), cudaMemcpyHostToDevice, h->stream));
    launch_filter_obs(h->fx.as<double>(), h->fP.as<double>(), h->fQ.as<double>(), h->fclk.as<lk_stream_clock>(), nullptr,
                      h->tmp.as<lk_kinimu_meas>(), n, h->ec, gravity, acc_norm, h->stream);
    return filter_download(h, x_inout, P_inout, clk_inout);
}

int lk_process_scan(lk_handle h, lk_state* x_inout, double* P_inout, const double* Q, lk_stream_clock* clk_inout,
                    const float* pts, uint32_t n_pts, const uint32_t* bucket_offsets, const double* bucket_times,
                    uint32_t n_buckets, const lk_imu_meas* imu, const lk_kinimu_meas* kin, uint32_t n_meas, double gravity,
                    double acc_norm, int iters, int update_map, float* pts_world_out, uint32_t* n_effective_out,
                    uint32_t* n_consumed) {
    if (!h || !x_inout || !P_inout || !Q || !clk_inout || !bucket_offsets || (n_buckets && !bucket_times))
        return fail(h, LK_ERR_INVALID_ARG, "null argument");
    if (imu && kin) return fail(h, LK_ERR_INVALID_ARG, "pass either imu or kin samples, not both (imu_mode_only_, KILO.cc:379)");
    if (n_meas && !imu && !kin) return fail(h, LK_ERR_INVALID_ARG, "n_meas > 0 without samples");
    uint32_t so[2] = {0, n_pts}, sb[2] = {0, n_buckets};
    int rc = stage_impl(h, 1, x_inout, P_inout, Q, clk_inout, pts, so, sb, bucket_offsets, bucket_times, false);
    if (rc) return rc;
    MeasQueue mq;
    std::vector<double> stamps(n_meas);
    if (n_meas) {
        const size_t bytes = (size_t)n_meas * (imu ? sizeof(lk_imu_meas) : sizeof(lk_kinimu_meas));
        LK_CUDA(h->err, h->tmp.ensure(bytes));
        LK_CUDA(h->err, cudaMemcpyAsync(h->tmp.p, imu ? (const void*)imu : (const void*)kin, bytes, cudaMemcpyHostToDevice, h->stream));
        for (uint32_t i = 0; i < n_meas; ++i) stamps[i] = imu ? imu[i].stamp : kin[i].stamp;
        mq.d_imu = imu ? h->tmp.as<lk_imu_meas>() : nullptr;
        mq.d_kin = kin ? h->tmp.as<lk_kinimu_meas>() : nullptr;
        mq.stamps = stamps.data();
        mq.n = n_meas;
    }
    mq.gravity = gravity;
    mq.acc_norm = acc_norm;
    h->nev = 0;
    rc = run_range_impl(h, 0, 1, iters, update_map, &mq, false);
    if (rc) return rc;
    if (n_consumed) {  // samples older than the LAST bucket were applied; the rest stays queued at the caller
        uint32_t c = 0;
        if (n_buckets)
            while (c < n_meas && stamps[c] < bucket_times[n_buckets - 1]) ++c;
        *n_consumed = c;
    }
    return lk_batch_fetch(h, x_inout, P_inout, clk_inout, pts_world_out, n_effective_out);
}

int lk_decode_pointcloud2(lk_handle h, const uint8_t* data, uint32_t n_points, const lk_pc2_layout* layout, float blind,
                          int32_t filter_num, double time_scale, float* pts_out, float* intensity_out, uint32_t* n_out,
                          double* first_time, double* last_time) {
    if (!h || !layout || !n_out || (n_points && (!data || !pts_out))) return fail(h, LK_ERR_INVALID_ARG, "null argument");
    if (filter_num < 1) return fail(h, LK_ERR_INVALID_ARG, "filter_num must be >= 1");
    if (!pc2_layout_fits(*layout)) return fail(h, LK_ERR_INVALID_ARG, "field layout does not fit point_step");
    *n_out = 0;
    if (!n_points) return LK_OK;
    enter(h);
    uint32_t out_offs[2];
    const int rc = decode_pointcloud2s_device(1, &data, &n_points, nullptr, *layout, blind, filter_num, time_scale, pts_out,
                                              intensity_out, out_offs, first_time, last_time, h->dec_scratch, h->stream, h->err);
    if (rc) return rc;
    *n_out = out_offs[1];
    return LK_OK;
}

int lk_decode_pointcloud2s(lk_handle h, uint32_t n_msgs, const uint8_t* const* data, const uint32_t* n_points,
                           const double* stamps, const lk_pc2_layout* layout, float blind, int32_t filter_num,
                           double time_scale, float* pts_out, float* intensity_out, uint32_t* out_offsets,
                           double* begin_times, double* end_times) {
    if (!h || !layout || !out_offsets || (n_msgs && (!data || !n_points || !pts_out)))
        return fail(h, LK_ERR_INVALID_ARG, "null argument");
    if (filter_num < 1) return fail(h, LK_ERR_INVALID_ARG, "filter_num must be >= 1");
    if (!pc2_layout_fits(*layout)) return fail(h, LK_ERR_INVALID_ARG, "field layout does not fit point_step");
    uint64_t total = 0;  // 64 bits: a uint32 sum of {2^31, 2^31} wraps to 0
    for (uint32_t m = 0; m < n_msgs; ++m) {
        if (n_points[m] && !data[m])
            return fail(h, LK_ERR_INVALID_ARG, "null data for message " + std::to_string(m) + " with points");
        total += n_points[m];
    }
    if (total > (uint64_t)INT_MAX) return fail(h, LK_ERR_INVALID_ARG, "more than INT_MAX points in one call");
    if (!n_msgs) {
        out_offsets[0] = 0;
        return LK_OK;
    }
    enter(h);
    return decode_pointcloud2s_device(n_msgs, data, n_points, stamps, *layout, blind, filter_num, time_scale, pts_out,
                                      intensity_out, out_offsets, begin_times, end_times, h->dec_scratch, h->stream, h->err);
}

int lk_preprocess_scan(lk_handle h, const float* pts_in, uint32_t n_in, float leaf_size, float* pts_out, uint32_t* n_out,
                       uint32_t* bucket_offsets, float* bucket_curvature, uint32_t* n_buckets) {
    if (!h || !n_out || !n_buckets || !bucket_offsets || (n_in && (!pts_in || !pts_out || !bucket_curvature)))
        return fail(h, LK_ERR_INVALID_ARG, "null argument");
    if (!(leaf_size > 0)) return fail(h, LK_ERR_INVALID_ARG, "leaf size must be positive");
    *n_out = 0;
    *n_buckets = 0;
    enter(h);
    const uint32_t offs[2] = {0, n_in};
    uint32_t scan_off[2], scan_bptr[2];
    const int rc = preprocess_scans_device(1, pts_in, offs, leaf_size, nullptr, pts_out, scan_off, scan_bptr, bucket_offsets,
                                           bucket_curvature, nullptr, h->pre_scratch, h->stream, h->err);
    if (rc) return rc;
    *n_out = scan_off[1];
    *n_buckets = scan_bptr[1];
    return LK_OK;
}

int lk_preprocess_scans(lk_handle h, uint32_t n_scans, const float* pts_in, const uint32_t* in_offsets, float leaf_size,
                        const double* begin_times, float* pts_out, uint32_t* scan_offsets, uint32_t* scan_bucket_ptr,
                        uint32_t* bucket_offsets, float* bucket_curvature, double* bucket_times) {
    if (!h || !pts_in || !in_offsets || !pts_out || !scan_offsets || !scan_bucket_ptr || !bucket_offsets || !bucket_curvature)
        return fail(h, LK_ERR_INVALID_ARG, "null argument");
    if (!begin_times != !bucket_times) return fail(h, LK_ERR_INVALID_ARG, "begin_times and bucket_times go together");
    if (!(leaf_size > 0) || !std::isfinite(leaf_size)) return fail(h, LK_ERR_INVALID_ARG, "leaf size must be positive and finite");
    for (uint32_t s = 0; s < n_scans; ++s)
        if (in_offsets[s + 1] < in_offsets[s]) return fail(h, LK_ERR_INVALID_ARG, "in_offsets not monotone");
    if (!n_scans) {
        scan_offsets[0] = scan_bucket_ptr[0] = bucket_offsets[0] = 0;
        return LK_OK;
    }
    enter(h);
    return preprocess_scans_device(n_scans, pts_in, in_offsets, leaf_size, begin_times, pts_out, scan_offsets, scan_bucket_ptr,
                                   bucket_offsets, bucket_curvature, bucket_times, h->pre_scratch, h->stream, h->err);
}

int lk_leg_kinematics(lk_handle h, const lk_leg_cfg* cfg, const lk_leg_state* in, uint32_t n, int32_t redundancy,
                      lk_leg_track* track_inout, lk_kinimu_meas* out, uint32_t* n_out) {
    if (!h || !cfg || !track_inout || !n_out || (n && (!in || !out))) return fail(h, LK_ERR_INVALID_ARG, "null argument");
    const double f[7] = {cfg->leg_offset_x,     cfg->leg_offset_y,     cfg->leg_calf_length,           cfg->leg_thigh_length,
                         cfg->leg_thigh_offset, cfg->contact_force_threshold_up, cfg->contact_force_threshold_down};
    for (double v : f)
        if (!std::isfinite(v)) return fail(h, LK_ERR_INVALID_ARG, "non-finite leg configuration");
    *n_out = 0;
    if (!n) return LK_OK;
    enter(h);
    LK_CUDA(h->err, h->leg_scratch.ensure(leg_kinematics_scratch_bytes(n)));
    return leg_kinematics_device(*cfg, in, n, redundancy, track_inout, out, n_out, h->leg_scratch.p, h->stream, h->err);
}

}  // extern "C"
