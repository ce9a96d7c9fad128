// lk_insert.cu — device-side VoxelMapManager::UpdateVoxelMap (voxel_map.cc:336-361) for one
// bucket: step 4 of KILO::predictUpdatePoint (KILO.cc:215-231).
//
// The reference inserts the bucket's points one after another; points only interact when they
// fall into the same ROOT voxel (every octree node belongs to exactly one root). So:
//   P1  per point: world point + covariance with the UPDATED state (KILO.cc:218-228), insert key
//       (voxelKeyFloor), find-or-create the root (CAS on the open-addressed table), count the
//       point on its root, first toucher registers the root;
//   P2  per touched root: reserve a slice of the pending list;
//   P3  per point: drop the point index into its root's slice;
//   P4  one warp per touched root: order the slice by point index (= the reference's insertion
//       order) and run UpdateOctoTree sequentially on it, with the warp-cooperative plane refit.
// Small buckets (the 2 ms buckets of streaming mode: a few hundred points) skip P2 / P3 and the sort: the
// warp of a touched root simply scans the bucket's root-per-point array in index order (P4S), and P1 also
// stores the re-projected world point (KILO.cc:216-224), so a bucket costs two launches instead of six.
#include "lk_kernels.h"
#include "lk_mapdev.h"
#include "lk_insert.cuh"
#include "lk_point.cuh"

namespace lk {

namespace {

struct InsertArgs {
    MapDev md;
    Globals g;
    const float4* pts;
    const ChunkDesc* chunks;
    uint32_t chunk_first;
    const ScanConst* sc;
    const ScanStep* step;
    DevPoint* ipts;      // [bucket points] DevPoint per point
    int* iroot;          // [bucket points] root node per point (-1 = dropped)
    uint32_t pt_base;    // absolute index of the first point covered by this launch's scratch
    int* pend;           // [node_cap * 3] count | offset | fill
    uint32_t* touched;   // [bucket points]
    uint32_t* counters;  // [0] n_touched  [1] list bump
    uint32_t* list;      // [2 * bucket points]  (second half = sort scratch)
    uint32_t n_pts;
    float4* world;       // non-null: P1 also writes cloud_down_world (x, y, z, intensity 0 | 255)
    uint32_t cslot;      // which of the two n_touched counters this bucket uses (small-bucket path)
};

// P1 — also the re-projection's covariance half (KILO.cc:225-228).
__global__ void __launch_bounds__(256) k_insert_p1(const __grid_constant__ InsertArgs a) {
    __shared__ ScanConst s_sc;
    const int tid = threadIdx.x;
    const ChunkDesc cd = a.chunks[a.chunk_first + blockIdx.x];
    load_scan_const(&s_sc, a.sc + cd.scan);
    __syncthreads();
    const Globals& g = a.g;
    MapDev md = a.md;
    for (uint32_t i = tid; i < cd.count; i += blockDim.x) {
        PointCtx pc;
        body_point(__ldg(a.pts + cd.start + i), g, pc);
        DevPoint p;
        make_insert_point(pc.pix, pc.piy, pc.piz, pc.pbx, pc.pby, pc.pbz, s_sc, g, p);
        const uint32_t li = cd.start + i - a.pt_base;
        a.ipts[li] = p;
        if (a.world) {
            float4 o;
            o.x = (float)p.pw[0]; o.y = (float)p.pw[1]; o.z = (float)p.pw[2];
            o.w = a.step[cd.scan].updated ? 255.0f : 0.0f;
            a.world[cd.start + i] = o;
        }
        a.iroot[li] = insert_register_point(md, g, p, a.pend, a.touched, &a.counters[a.cslot]);
    }
}

__global__ void k_insert_p2(const __grid_constant__ InsertArgs a) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.counters[0]) return;
    const uint32_t root = a.touched[t];
    const int cnt = a.pend[root * 3];
    a.pend[root * 3 + 1] = (int)atomicAdd(&a.counters[1], (uint32_t)cnt);
    a.pend[root * 3 + 2] = 0;
}

__global__ void k_insert_p3(const __grid_constant__ InsertArgs a) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n_pts) return;
    const int root = a.iroot[i];
    if (root < 0) return;
    const int slot = atomicAdd(&a.pend[root * 3 + 2], 1);
    a.list[a.pend[root * 3 + 1] + slot] = i;
}

__global__ void __launch_bounds__(128) k_insert_p4(const __grid_constant__ InsertArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    WarpTile* tiles = reinterpret_cast<WarpTile*>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    WarpTile* wt = tiles + warp;
    if (lane == 0) {
        mbar_init(&wt->bar, 1);
        wt->phase = 0;
        mbar_init_fence();
    }
    __syncwarp();
    const uint32_t t = blockIdx.x * (blockDim.x >> 5) + warp;
    if (t >= a.counters[0]) return;
    const uint32_t root = a.touched[t];
    const int cnt = a.pend[root * 3];
    const int off = a.pend[root * 3 + 1];
    uint32_t* src = a.list + off;
    uint32_t* dst = a.list + a.n_pts + off;
    // rank sort by point index = the order UpdateVoxelMap walks input_points
    for (int j = lane; j < cnt; j += 32) {
        const uint32_t v = src[j];
        int rank = 0;
        for (int k = 0; k < cnt; ++k) rank += (src[k] < v) ? 1 : 0;
        dst[rank] = v;
    }
    __syncwarp();
    MapDev md = a.md;
    for (int j = 0; j < cnt; ++j) {
        const DevPoint p = a.ipts[dst[j]];
        warp_update_octo_tree(md, a.g, wt, root, p, lane);
    }
    __syncwarp();
    if (lane == 0) a.pend[root * 3] = 0;
}

// P4S — small buckets: one warp per touched root walks the bucket's root-per-point array in index order
// (= the order UpdateVoxelMap walks input_points) and inserts its own points; no slices, no sort.
__global__ void __launch_bounds__(128) k_insert_p4_scan(const __grid_constant__ InsertArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    WarpTile* tiles = reinterpret_cast<WarpTile*>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    WarpTile* wt = tiles + warp;
    if (lane == 0) {
        mbar_init(&wt->bar, 1);
        wt->phase = 0;
        mbar_init_fence();
    }
    __syncwarp();
    if (blockIdx.x == 0 && threadIdx.x == 0) a.counters[a.cslot ^ 1u] = 0;  // the next bucket's counter
    const uint32_t t = blockIdx.x * (blockDim.x >> 5) + warp;
    if (t >= a.counters[a.cslot]) return;
    const uint32_t root = a.touched[t];
    MapDev md = a.md;
    warp_insert_root_scan(md, a.g, wt, root, a.iroot, a.ipts, a.n_pts, a.pend, lane);
}

// insert_sets runs its input through the slice-and-sort insert in windows of at most this many points (DESIGN §3.5): per
// window, the headroom begin reserves for a streaming scan of as many points, and scratch of a fixed size.
constexpr uint32_t MAP_INSERT_WINDOW = 32768u;

}  // namespace

int MapInserter::begin(MapDevHost& mh, const Globals& g, uint64_t n, uint32_t max_bucket, cudaStream_t s, std::string& err) {
    int rc = mh.ready() ? mh.sync_counters(s, err) : LK_OK;
    // Worst case of UpdateVoxelMap per inserted point (lk_octree.cuh): a new root (1 node, one tile); per octree level one
    // cut (8 nodes) whose children each get a tile — at most threshold + 1 of them hold a point when the cut fires.
    // Reserving the bound makes a mid-insert overflow impossible: no point is ever dropped (the pools only grow when a
    // scan could actually exceed them: 80 GB of HBM is the budget).
    if (!rc) {
        int thr = 0;
        for (int l = 0; l < 5; ++l) thr = std::max(thr, g.layer_init_num[l]);
        const uint64_t tile = mh.tile_slots;
        const uint64_t per_pt_nodes = 1 + 8ull * (uint64_t)std::max(g.max_layer, 0);
        const uint64_t per_pt_slots = tile * (1 + (uint64_t)std::max(g.max_layer, 0) * (uint64_t)std::min(8, thr + 1)) + 2;
        rc = mh.ensure_headroom(n + 16, per_pt_nodes * n + 64, per_pt_slots * n + 64, s, err);
    }
    if (!rc) rc = mh.push_counters(s, err);  // also makes what earlier launches freed available to this insert
    if (rc) return rc;
    if (pend_nodes_ < mh.node_cap) {
        LK_CUDA(err, pend_.ensure((size_t)mh.node_cap * 3 * sizeof(int)));
        LK_CUDA(err, cudaMemsetAsync(pend_.p, 0, pend_.cap, s));
        pend_nodes_ = mh.node_cap;
    }
    const size_t mb = std::max<uint32_t>(max_bucket, 1);
    LK_CUDA(err, pts_.ensure(mb * sizeof(DevPoint)));
    LK_CUDA(err, root_.ensure(mb * 4));
    LK_CUDA(err, touched_.ensure(mb * 4));
    LK_CUDA(err, list_.ensure(2 * mb * 4));
    LK_CUDA(err, counters_.ensure(64));
    LK_CUDA(err, cudaMemsetAsync(counters_.p, 0, 64, s));
    parity_ = 0;
    return LK_OK;
}

int MapInserter::bucket(const MapDevHost& mh, const Globals& g, const float4* pts, const ChunkDesc* chunks,
                        uint32_t chunk_first, uint32_t n_chunks, uint32_t pt_begin, uint32_t n_pts, const ScanConst* sc,
                        const ScanStep* step, cudaStream_t s, float4* world) {
    if (!n_pts || !n_chunks) return LK_OK;
    uint32_t* counters = counters_.as<uint32_t>();
    InsertArgs a;
    a.md = mh.dev();
    a.g = g;
    a.pts = pts;
    a.chunks = chunks;
    a.chunk_first = chunk_first;
    a.sc = sc;
    a.step = step;
    a.ipts = pts_.as<DevPoint>();
    a.iroot = root_.as<int>();
    a.pt_base = pt_begin;
    a.pend = pend_.as<int>();
    a.touched = touched_.as<uint32_t>();
    a.counters = counters;
    a.list = list_.as<uint32_t>();
    a.n_pts = n_pts;
    a.world = world;
    a.cslot = 0;
    const int wpb = 4;
    if (world && n_pts <= 4096u) {
        // counters[2 + parity] is this bucket's n_touched; P4S zeroes the other one for the next bucket (begin zeroed both)
        a.counters = counters + 2;
        a.cslot = parity_;
        parity_ ^= 1u;
        k_insert_p1<<<n_chunks, 256, 0, s>>>(a);
        k_insert_p4_scan<<<(n_pts + wpb - 1) / wpb, wpb * 32, wpb * sizeof(WarpTile), s>>>(a);
        return 2;
    }
    cudaMemsetAsync(counters, 0, 8, s);
    k_insert_p1<<<n_chunks, 256, 0, s>>>(a);
    k_insert_p2<<<(n_pts + 255) / 256, 256, 0, s>>>(a);
    k_insert_p3<<<(n_pts + 255) / 256, 256, 0, s>>>(a);
    k_insert_p4<<<(n_pts + wpb - 1) / wpb, wpb * 32, wpb * sizeof(WarpTile), s>>>(a);
    return 5;
}

int MapInserter::finish(const MapDevHost& mh, std::string& err) const {
    uint32_t ovf = 0;
    LK_CUDA(err, cudaMemcpy(&ovf, mh.dev().overflow, 4, cudaMemcpyDeviceToHost));
    if (ovf) err = "map pools exhausted during UpdateVoxelMap (raise lk_map_reserve)";
    return ovf ? LK_ERR_CAPACITY : LK_OK;
}

void MapInserter::fused_scratch(FusedArgs& fa) const {
    fa.ipts = pts_.as<DevPoint>();
    fa.iroot = root_.as<int>();
    fa.pend = pend_.as<int>();
    fa.touched = touched_.as<uint32_t>();
    fa.ins_counters = counters_.as<uint32_t>() + 2;
}

int MapInserter::insert_sets(MapDevHost& mh, const Globals& g, uint32_t n_sets, const float* pts, const uint32_t* set_offsets,
                             const double* rot, const double* pos, const double* rot_cov, const double* pos_cov,
                             cudaStream_t st, std::string& err) {
    const uint32_t W = MAP_INSERT_WINDOW;
    // a window holds points of at most W sets, and its chunks are 256 points each plus one partial chunk per set
    const uint32_t max_sets = std::min(n_sets, W);
    const size_t sc_off = align256(((size_t)W / 256u + max_sets) * sizeof(ChunkDesc));
    const size_t small_bytes = sc_off + (size_t)max_sets * sizeof(ScanConst);
    LK_CUDA(err, win_pts_.ensure((size_t)W * 16));
    LK_CUDA(err, win_small_.ensure(small_bytes));
    LK_CUDA(err, h_win_.ensure(small_bytes));
    ChunkDesc* hc = reinterpret_cast<ChunkDesc*>(h_win_.p);
    ScanConst* hs = reinterpret_cast<ScanConst*>((char*)h_win_.p + sc_off);
    const ChunkDesc* dc = reinterpret_cast<const ChunkDesc*>(win_small_.p);
    const ScanConst* ds = reinterpret_cast<const ScanConst*>((char*)win_small_.p + sc_off);
    const uint64_t end = set_offsets[n_sets];
    uint32_t s = 0;
    for (uint64_t p0 = set_offsets[0]; p0 < end;) {
        const uint64_t p1 = std::min<uint64_t>(end, p0 + W);
        const uint32_t n = (uint32_t)(p1 - p0);
        int rc = begin(mh, g, n, W, st, err);
        if (rc) return rc;
        // the window's chunks; ChunkDesc.scan = the set's row in the window's table of placements
        uint32_t nc = 0, nsc = 0;
        while (set_offsets[s + 1] <= p0) ++s;
        for (uint32_t t = s; t < n_sets && set_offsets[t] < p1; ++t) {
            const uint64_t a = std::max<uint64_t>(set_offsets[t], p0), b = std::min<uint64_t>(set_offsets[t + 1], p1);
            if (a >= b) continue;
            scan_const_at(rot + 9 * (size_t)t, pos + 3 * (size_t)t, rot_cov + 9 * (size_t)t, pos_cov + 9 * (size_t)t, hs[nsc]);
            for (uint64_t q = a; q < b; q += 256) {
                ChunkDesc& cd = hc[nc++];
                cd.scan = nsc;
                cd.start = (uint32_t)(q - p0);
                cd.count = (uint32_t)std::min<uint64_t>(256, b - q);
                cd.pad = 0;
            }
            ++nsc;
        }
        LK_CUDA(err, cudaMemcpyAsync(win_pts_.p, pts + 4 * p0, (size_t)n * 16, cudaMemcpyHostToDevice, st));
        // (h_win_ is free again: the previous window's sync_counters waited for its copies)
        LK_CUDA(err, cudaMemcpyAsync(win_small_.p, hc, (size_t)nc * sizeof(ChunkDesc), cudaMemcpyHostToDevice, st));
        LK_CUDA(err, cudaMemcpyAsync((char*)win_small_.p + sc_off, hs, (size_t)nsc * sizeof(ScanConst), cudaMemcpyHostToDevice, st));
        bucket(mh, g, win_pts_.as<float4>(), dc, 0, nc, 0, n, ds, nullptr, st);
        LK_CUDA(err, cudaGetLastError());
        rc = mh.sync_counters(st, err);
        if (!rc) rc = finish(mh, err);
        if (rc) return rc;
        p0 = p1;
    }
    return LK_OK;
}

}  // namespace lk
