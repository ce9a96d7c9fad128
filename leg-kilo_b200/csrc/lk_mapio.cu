// lk_mapio.cu — device map storage management and the blob import / export
// (lk_map_upload / lk_map_download of include/legkilo_b200.h).
#include <algorithm>
#include <cstring>
#include <vector>

#include "lk_kernels.h"
#include "lk_mapdev.h"
#include "lk_octree.cuh"

namespace lk {

namespace {

__global__ void k_hash_clear(HashSlot* slots, uint64_t capacity) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < capacity) {
        HashSlot s;
        s.kx = 0; s.ky = 0; s.kz = 0; s.node = -1;
        slots[i] = s;
    }
}

__global__ void k_hash_insert_roots(HashSlot* slots, uint32_t mask, const lk_map_root* roots, uint32_t n, uint32_t* ovf) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    lk_map_root r = roots[i];
    if (!hash_insert_dev(slots, mask, r.key[0], r.key[1], r.key[2], r.node)) atomicOr(ovf, 4u);
}

__global__ void k_hash_dump(const HashSlot* slots, uint64_t capacity, lk_map_root* roots, uint32_t* counter) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= capacity) return;
    HashSlot s = slots[i];
    if (s.node >= 0) {
        uint32_t o = atomicAdd(counter, 1u);
        lk_map_root r;
        r.key[0] = s.kx; r.key[1] = s.ky; r.key[2] = s.kz; r.node = s.node;
        roots[o] = r;
    }
}

// every root key must resolve to its own node: a second root with the same key is unreachable (and means a corrupt blob)
__global__ void k_check_roots(const HashSlot* slots, uint32_t mask, const lk_map_root* roots, uint32_t n, uint32_t* ovf) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    lk_map_root r = roots[i];
    if (hash_find_dev(slots, mask, r.key[0], r.key[1], r.key[2]) != r.node) atomicOr(ovf, 8u);
}

// hot images of nodes [0, n) from their node records (after a blob upload)
__global__ void k_hot_from_nodes(const MapNode* nodes, HotRec* hot, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) hot_from_node(nodes[i], hot[i]);
}

__global__ void k_count_planes(const MapNode* nodes, const MapAux* aux, uint32_t n, unsigned long long* out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (nodes[i].flags & LK_NODE_IS_PLANE) atomicAdd(out, 1ull);
    if (aux[i].pts_count > 0) atomicAdd(out + 1, (unsigned long long)aux[i].pts_count);
}

// The storage of the octrees under dropped roots goes back to the free lists: one thread per root walks the subtree
// through child_base and the child mask, pushes the standard tiles still held, every 8-node child group and the root
// node, and resets each node to the empty state (hot record included). The nodes are unreachable: the table no longer
// holds their keys.
__global__ void k_free_subtrees(MapDev md, const lk_map_root* gone, uint32_t n, int tile) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t root = (uint32_t)gone[i].node;
    free_push(md, FREE_SINGLES, root);
    uint32_t stack[8 * 6];  // depth-first: at most 7 pending siblings per level below the root (layer <= 4)
    int sp = 0;
    stack[sp++] = root;
    while (sp > 0) {
        const uint32_t nd = stack[--sp];
        const uint32_t flags = md.nodes[nd].flags;
        const int cb = md.nodes[nd].child_base;
        const MapAux& a = md.aux[nd];
        if (a.pts_cap == tile && a.pts_base != NO_TILE) free_push(md, FREE_TILES, a.pts_base);
        if (cb >= 0) {
            free_push(md, FREE_GROUPS, (uint32_t)cb);
            const uint32_t mask = (flags >> LK_NODE_CHILDMASK_SHIFT) & 0xffu;
            for (int c = 0; c < 8; ++c) {
                if (!((mask >> c) & 1u)) node_reset(md, (uint32_t)cb + c, 0, -1);
                else if (sp < 8 * 6) stack[sp++] = (uint32_t)cb + c;
            }
        }
        node_reset(md, nd, 0, -1);
    }
}

uint64_t next_pow2(uint64_t v) {
    uint64_t p = 1;
    while (p < v) p <<= 1;
    return p;
}

}  // namespace

constexpr size_t COUNTER_BYTES = 128;
constexpr int FREE_CTR = 16;  // first counter word of the free lists

void MapDevHost::release() {
    for (DevBuf* b : {&slots, &nodes, &aux, &hot, &points, &counters}) b->reset();
    hash_cap = node_cap = point_cap = 0;
    n_roots = n_nodes = 0;
    n_points = 0;
    for (int l = 0; l < 3; ++l) {
        free_items[l].reset();
        free_cap[l] = 0;
        free_avail[l] = 0; free_base[l] = free_top[l] = 0;
    }
    reallocs = 0;
}

// Grow the free-list arrays to twice the entries the pools can hold. keep: copy the entries of the old arrays (the
// mirrors are those of a sync after the last launch); else the lists start empty.
int MapDevHost::size_free_lists(bool keep, cudaStream_t s, std::string& err) {
    const uint64_t want[3] = {2 * (point_cap / std::max<uint32_t>(tile_slots, 2)) + 2, 2 * (node_cap / 8) + 2, 2 * node_cap + 2};
    for (int l = 0; l < 3; ++l) {
        if (!keep) { free_avail[l] = 0; free_base[l] = free_top[l] = 0; }
        if (want[l] <= free_cap[l]) continue;
        DevBuf p;
        LK_CUDA(err, p.alloc(want[l] * sizeof(uint32_t)));
        const uint64_t used = keep ? std::min<uint64_t>(free_top[l], free_cap[l]) : 0;
        if (used) LK_CUDA(err, cudaMemcpyAsync(p.p, free_items[l].p, used * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
        LK_CUDA(err, cudaStreamSynchronize(s));
        free_items[l] = std::move(p);
        free_cap[l] = want[l];
    }
    return LK_OK;
}

uint64_t MapDevHost::free_entries(int l) const {
    return (uint64_t)std::max(free_avail[l], 0) + (std::min<uint64_t>(free_top[l], free_cap[l]) - free_base[l]);
}

uint64_t MapDevHost::pool_bytes() const {
    uint64_t b = hash_cap * sizeof(HashSlot) + node_cap * (sizeof(MapNode) + sizeof(MapAux) + sizeof(HotRec)) +
                 point_cap * sizeof(DevPoint) + (counters.p ? COUNTER_BYTES : 0);
    for (int l = 0; l < 3; ++l) b += free_cap[l] * sizeof(uint32_t);
    return b;
}

MapDev MapDevHost::dev() const {
    MapDev d;
    uint32_t* ctr = counters.as<uint32_t>();
    d.slots = slots.as<HashSlot>();
    d.hash_mask = (uint32_t)(hash_cap - 1);
    d.nodes = nodes.as<MapNode>();
    d.aux = aux.as<MapAux>();
    d.hot = hot.as<HotRec>();
    d.points = points.as<DevPoint>();
    d.node_cap = (uint32_t)node_cap;
    d.point_cap = point_cap;
    d.n_nodes = ctr;
    d.n_roots = ctr + 1;
    d.overflow = ctr + 2;
    d.n_points = reinterpret_cast<unsigned long long*>(ctr + 4);
    for (int l = 0; l < 3; ++l) {
        d.free_items[l] = free_items[l].as<uint32_t>();
        d.free_cap[l] = (uint32_t)std::min<uint64_t>(free_cap[l], 0xffffffffu);
    }
    d.free_ctr = ctr ? ctr + FREE_CTR : nullptr;
    return d;
}

MapView MapDevHost::view() const {
    const MapDev d = dev();
    return {d.slots, d.hash_mask, d.nodes, d.hot};
}

int MapDevHost::allocate(uint64_t roots, uint64_t nnodes, uint64_t npoints, cudaStream_t s, std::string& err) {
    // Pools that are large enough are kept; a pool that is not is freed before its replacement is allocated. Any
    // failure drops the whole map, so no caller goes ahead on a half-built one.
    auto build = [&]() -> int {
        uint64_t want_hash = next_pow2(std::max<uint64_t>(1024, 4 * (roots + reserve_roots)));  // load factor <= 0.25
        if (want_hash > (1ull << 31)) { err = "root table too large"; return LK_ERR_CAPACITY; }
        uint64_t want_nodes = std::max<uint64_t>(nnodes + reserve_nodes, 64);
        uint64_t want_points = std::max<uint64_t>(npoints + reserve_points, 64);
        if (want_nodes >= (1ull << 31)) { err = "node pool too large"; return LK_ERR_CAPACITY; }
        if (want_points >= (1ull << 32)) { err = "point pool too large"; return LK_ERR_CAPACITY; }
        if (!counters.p) LK_CUDA(err, counters.alloc(COUNTER_BYTES));
        if (want_hash != hash_cap) {
            hash_cap = 0;
            LK_CUDA(err, slots.alloc(want_hash * sizeof(HashSlot)));
            hash_cap = want_hash;
        }
        if (want_nodes > node_cap) {
            nodes.reset(); aux.reset(); hot.reset(); node_cap = 0;
            LK_CUDA(err, nodes.alloc(want_nodes * sizeof(MapNode)));
            LK_CUDA(err, aux.alloc(want_nodes * sizeof(MapAux)));
            LK_CUDA(err, hot.alloc(want_nodes * sizeof(HotRec)));
            node_cap = want_nodes;
        }
        if (want_points > point_cap) {
            point_cap = 0;
            LK_CUDA(err, points.alloc(want_points * sizeof(DevPoint)));
            point_cap = want_points;
        }
        int rc = size_free_lists(false, s, err);  // a new map starts with empty free lists
        if (rc) return rc;
        k_hash_clear<<<(unsigned)((hash_cap + 255) / 256), 256, 0, s>>>(slots.as<HashSlot>(), hash_cap);
        LK_CUDA(err, cudaMemsetAsync(counters.p, 0, COUNTER_BYTES, s));
        LK_CUDA(err, cudaGetLastError());
        return LK_OK;
    };
    const int rc = build();
    if (rc) {
        release();
        return rc;
    }
    n_roots = n_nodes = 0;
    n_points = 0;
    reallocs = 0;
    return LK_OK;
}

int MapDevHost::ensure_headroom(uint64_t extra_roots, uint64_t extra_nodes, uint64_t extra_points, cudaStream_t s,
                                std::string& err) {
    if (!ready()) return allocate(extra_roots, extra_nodes, extra_points, s, err);
    // nodes
    if (n_nodes + extra_nodes > node_cap) {
        uint64_t want = std::max<uint64_t>(n_nodes + extra_nodes, node_cap + node_cap / 2);
        if (want >= (1ull << 31)) { err = "node pool too large"; return LK_ERR_CAPACITY; }
        DevBuf nn, na, nh;
        LK_CUDA(err, nn.alloc(want * sizeof(MapNode)));
        LK_CUDA(err, na.alloc(want * sizeof(MapAux)));
        LK_CUDA(err, nh.alloc(want * sizeof(HotRec)));
        LK_CUDA(err, cudaMemcpyAsync(nn.p, nodes.p, (size_t)n_nodes * sizeof(MapNode), cudaMemcpyDeviceToDevice, s));
        LK_CUDA(err, cudaMemcpyAsync(na.p, aux.p, (size_t)n_nodes * sizeof(MapAux), cudaMemcpyDeviceToDevice, s));
        LK_CUDA(err, cudaMemcpyAsync(nh.p, hot.p, (size_t)n_nodes * sizeof(HotRec), cudaMemcpyDeviceToDevice, s));
        LK_CUDA(err, cudaStreamSynchronize(s));
        nodes = std::move(nn); aux = std::move(na); hot = std::move(nh); node_cap = want;
        ++reallocs;
    }
    if (n_points + extra_points > point_cap) {
        uint64_t want = std::max<uint64_t>(n_points + extra_points, point_cap + point_cap / 2);
        if (want >= (1ull << 32)) { err = "point pool too large"; return LK_ERR_CAPACITY; }
        DevBuf np;
        LK_CUDA(err, np.alloc(want * sizeof(DevPoint)));
        LK_CUDA(err, cudaMemcpyAsync(np.p, points.p, (size_t)n_points * sizeof(DevPoint), cudaMemcpyDeviceToDevice, s));
        LK_CUDA(err, cudaStreamSynchronize(s));
        points = std::move(np); point_cap = want;
        ++reallocs;
    }
    int rc = size_free_lists(true, s, err);
    if (rc) return rc;
    if (4 * (n_roots + extra_roots) > hash_cap) {
        // rehash: dump roots, rebuild a bigger table
        uint64_t want = next_pow2(4 * (n_roots + extra_roots) + 4 * reserve_roots);
        if (want > (1ull << 31)) { err = "root table too large"; return LK_ERR_CAPACITY; }
        DevBuf tmp, ns;
        LK_CUDA(err, tmp.alloc(std::max<size_t>(n_roots, 1) * sizeof(lk_map_root)));
        uint32_t* cnt = counters.as<uint32_t>() + 8;
        LK_CUDA(err, cudaMemsetAsync(cnt, 0, 4, s));
        k_hash_dump<<<(unsigned)((hash_cap + 255) / 256), 256, 0, s>>>(slots.as<HashSlot>(), hash_cap, tmp.as<lk_map_root>(), cnt);
        LK_CUDA(err, ns.alloc(want * sizeof(HashSlot)));
        k_hash_clear<<<(unsigned)((want + 255) / 256), 256, 0, s>>>(ns.as<HashSlot>(), want);
        if (n_roots)
            k_hash_insert_roots<<<(n_roots + 255) / 256, 256, 0, s>>>(ns.as<HashSlot>(), (uint32_t)(want - 1), tmp.as<lk_map_root>(),
                                                                     n_roots, counters.as<uint32_t>() + 2);
        LK_CUDA(err, cudaStreamSynchronize(s));
        slots = std::move(ns); hash_cap = want;
        ++reallocs;
    }
    return LK_OK;
}

int MapDevHost::sync_counters(cudaStream_t s, std::string& err) {
    uint32_t h[FREE_CTR + 9] = {};
    LK_CUDA(err, cudaMemcpyAsync(h, counters.p, sizeof(h), cudaMemcpyDeviceToHost, s));
    LK_CUDA(err, cudaStreamSynchronize(s));
    n_nodes = h[0];
    n_roots = h[1];
    unsigned long long np;
    std::memcpy(&np, &h[4], 8);
    n_points = np;
    for (int l = 0; l < 3; ++l) {
        free_avail[l] = (int32_t)h[FREE_CTR + 3 * l];
        free_base[l] = h[FREE_CTR + 3 * l + 1];
        free_top[l] = h[FREE_CTR + 3 * l + 2];
    }
    return LK_OK;
}

int MapDevHost::push_counters(cudaStream_t s, std::string& err) {
    // Promote: the entries pushed since the last push, [base, top), join the available ones. Pops left a hole
    // [avail, base); the last min(hole, pending) entries move into it (disjoint ranges, order is irrelevant).
    for (int l = 0; l < 3; ++l) {
        const uint32_t a = (uint32_t)std::max(free_avail[l], 0);
        const uint32_t b = free_base[l];
        const uint32_t t = (uint32_t)std::min<uint64_t>(free_top[l], free_cap[l]);
        const uint32_t pend = t - b, k = std::min(b - a, pend);
        uint32_t* items = free_items[l].as<uint32_t>();
        if (k) LK_CUDA(err, cudaMemcpyAsync(items + a, items + (t - k), (size_t)k * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
        free_avail[l] = (int32_t)(a + pend);
        free_base[l] = free_top[l] = a + pend;
    }
    uint32_t h[FREE_CTR + 9] = {n_nodes, n_roots};
    unsigned long long np = n_points;
    std::memcpy(&h[4], &np, 8);
    for (int l = 0; l < 3; ++l) {
        h[FREE_CTR + 3 * l] = (uint32_t)free_avail[l];
        h[FREE_CTR + 3 * l + 1] = free_base[l];
        h[FREE_CTR + 3 * l + 2] = free_top[l];
    }
    LK_CUDA(err, cudaMemcpyAsync(counters.p, h, sizeof(h), cudaMemcpyHostToDevice, s));
    LK_CUDA(err, cudaStreamSynchronize(s));
    return LK_OK;
}

int map_upload_blob(MapDevHost& mh, const Globals& g, const void* blob, size_t bytes, cudaStream_t s, std::string& err) {
    if (bytes < sizeof(lk_map_blob_header)) { err = "blob shorter than its header"; return LK_ERR_BAD_BLOB; }
    lk_map_blob_header hd;
    std::memcpy(&hd, blob, sizeof(hd));
    if (hd.magic != LK_MAP_MAGIC || hd.version != 1) { err = "bad magic / version"; return LK_ERR_BAD_BLOB; }
    size_t need = sizeof(hd) + (size_t)hd.n_roots * sizeof(lk_map_root) + (size_t)hd.n_nodes * (sizeof(lk_map_node) + sizeof(lk_map_aux)) +
                  (size_t)hd.n_points * sizeof(lk_map_point);
    if (bytes < need) { err = "blob truncated"; return LK_ERR_BAD_BLOB; }
    const char* p = (const char*)blob + sizeof(hd);
    const lk_map_root* roots = (const lk_map_root*)p;
    p += (size_t)hd.n_roots * sizeof(lk_map_root);
    const lk_map_node* nodes = (const lk_map_node*)p;
    p += (size_t)hd.n_nodes * sizeof(lk_map_node);
    const lk_map_aux* aux = (const lk_map_aux*)p;
    p += (size_t)hd.n_nodes * sizeof(lk_map_aux);
    const lk_map_point* pts = (const lk_map_point*)p;
    for (uint32_t r = 0; r < hd.n_roots; ++r)
        if (roots[r].node < 0 || (uint32_t)roots[r].node >= hd.n_nodes) { err = "root node index out of range"; return LK_ERR_BAD_BLOB; }

    // Re-pack retained points into growable 80-byte tiles. A node may still take points when it is
    // not initialised, or is an update-enabled leaf (plane, or non-plane at max_layer).
    std::vector<lk_map_aux> aux2(aux, aux + hd.n_nodes);
    std::vector<DevPoint> dpts;
    const int P2 = g.max_points_num + 2;
    uint64_t slots_needed = 0;
    for (uint32_t i = 0; i < hd.n_nodes; ++i) {
        const lk_map_node& n = nodes[i];
        lk_map_aux& a = aux2[i];
        if ((uint64_t)a.pts_base + (uint64_t)std::max(a.pts_count, 0) > hd.n_points) { err = "node point range out of bounds"; return LK_ERR_BAD_BLOB; }
        int layer = (n.flags >> LK_NODE_LAYER_SHIFT) & 0xff;
        const uint32_t cmask = (n.flags >> LK_NODE_CHILDMASK_SHIFT) & 0xffu;
        // the residual kernels follow child_base / the child mask without further checks
        if (layer > g.max_layer || layer > 4) { err = "node layer exceeds max_layer"; return LK_ERR_BAD_BLOB; }
        if (n.child_base < -1 || (n.child_base >= 0 && (uint64_t)n.child_base + 8 > hd.n_nodes)) { err = "node child_base out of range"; return LK_ERR_BAD_BLOB; }
        if (cmask && n.child_base < 0) { err = "node has a child mask but no children"; return LK_ERR_BAD_BLOB; }
        bool init = n.flags & LK_NODE_INIT_OCTO, plane = n.flags & LK_NODE_IS_PLANE, upd = n.flags & LK_NODE_UPDATE_ENABLE;
        bool interior = init && !plane && layer < g.max_layer;
        bool can_grow = !init || (upd && !interior);
        int cnt = interior ? 0 : std::max(a.pts_count, 0);
        int cap = 0;
        if (cnt > 0) cap = ((std::max(cnt + 1, can_grow ? P2 : cnt) + 1) & ~1);
        a.pts_count = cnt;
        a.pts_cap = cap;
        const uint32_t src = a.pts_base;
        a.pts_base = (uint32_t)slots_needed;
        if (cap) {
            size_t at = dpts.size();
            dpts.resize(at + cap);
            std::memset(&dpts[at], 0, sizeof(DevPoint) * cap);
            for (int j = 0; j < cnt; ++j) {
                std::memcpy(dpts[at + j].pw, pts[src + j].pw, 24);
                std::memcpy(dpts[at + j].var, pts[src + j].var, 48);
            }
        }
        slots_needed += cap;
    }
    int rc = mh.allocate(hd.n_roots, hd.n_nodes, slots_needed, s, err);
    if (rc) return rc;
    DevBuf d_roots;
    LK_CUDA(err, d_roots.alloc(std::max<size_t>(hd.n_roots, 1) * sizeof(lk_map_root)));
    const MapDev md = mh.dev();
    cudaError_t e = cudaSuccess;
    if (hd.n_nodes) {
        e = cudaMemcpyAsync(md.nodes, nodes, (size_t)hd.n_nodes * sizeof(MapNode), cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(md.aux, aux2.data(), (size_t)hd.n_nodes * sizeof(MapAux), cudaMemcpyHostToDevice, s);
    }
    if (e == cudaSuccess && !dpts.empty()) e = cudaMemcpyAsync(md.points, dpts.data(), dpts.size() * sizeof(DevPoint), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && hd.n_roots) {
        e = cudaMemcpyAsync(d_roots.p, roots, (size_t)hd.n_roots * sizeof(lk_map_root), cudaMemcpyHostToDevice, s);
        k_hash_insert_roots<<<(hd.n_roots + 255) / 256, 256, 0, s>>>(md.slots, md.hash_mask, d_roots.as<lk_map_root>(), hd.n_roots, md.overflow);
        k_check_roots<<<(hd.n_roots + 255) / 256, 256, 0, s>>>(md.slots, md.hash_mask, d_roots.as<lk_map_root>(), hd.n_roots, md.overflow);
    }
    if (e == cudaSuccess && hd.n_nodes) k_hot_from_nodes<<<(hd.n_nodes + 255) / 256, 256, 0, s>>>(md.nodes, md.hot, hd.n_nodes);
    uint32_t ovf = 0;
    if (e == cudaSuccess) e = cudaMemcpyAsync(&ovf, md.overflow, 4, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { cudaGetLastError(); err = cudaGetErrorString(e); return LK_ERR_CUDA; }
    if (ovf & 8u) { err = "duplicate root keys in the blob"; return LK_ERR_BAD_BLOB; }
    if (ovf) { err = "root table overflow"; return LK_ERR_CAPACITY; }
    mh.n_roots = hd.n_roots;
    mh.n_nodes = hd.n_nodes;
    mh.n_points = slots_needed;
    return mh.push_counters(s, err);
}

int map_download_blob(MapDevHost& mh, void* blob, size_t capacity, size_t* bytes_out, cudaStream_t s, std::string& err) {
    if (!mh.ready()) {
        lk_map_blob_header hd;
        std::memset(&hd, 0, sizeof(hd));
        hd.magic = LK_MAP_MAGIC; hd.version = 1;
        if (bytes_out) *bytes_out = sizeof(hd);
        if (blob) {
            if (capacity < sizeof(hd)) { err = "blob buffer too small"; return LK_ERR_CAPACITY; }
            std::memcpy(blob, &hd, sizeof(hd));
        }
        return LK_OK;
    }
    int rc = mh.sync_counters(s, err);
    if (rc) return rc;
    std::vector<lk_map_aux> aux(mh.n_nodes);
    if (mh.n_nodes) LK_CUDA(err, cudaMemcpyAsync(aux.data(), mh.aux.p, (size_t)mh.n_nodes * sizeof(MapAux), cudaMemcpyDeviceToHost, s));
    LK_CUDA(err, cudaStreamSynchronize(s));
    uint64_t live = 0;
    for (auto& a : aux) live += (uint64_t)std::max(a.pts_count, 0);
    size_t need = sizeof(lk_map_blob_header) + (size_t)mh.n_roots * sizeof(lk_map_root) +
                  (size_t)mh.n_nodes * (sizeof(lk_map_node) + sizeof(lk_map_aux)) + (size_t)live * sizeof(lk_map_point);
    if (bytes_out) *bytes_out = need;
    if (!blob) return LK_OK;
    if (capacity < need) { err = "blob buffer too small"; return LK_ERR_CAPACITY; }
    lk_map_blob_header hd;
    std::memset(&hd, 0, sizeof(hd));
    hd.magic = LK_MAP_MAGIC; hd.version = 1;
    hd.n_roots = mh.n_roots; hd.n_nodes = mh.n_nodes; hd.n_points = live;
    char* p = (char*)blob;
    std::memcpy(p, &hd, sizeof(hd));
    p += sizeof(hd);
    DevBuf d_roots;
    LK_CUDA(err, d_roots.alloc(std::max<size_t>(mh.n_roots, 1) * sizeof(lk_map_root)));
    uint32_t* cnt = mh.counters.as<uint32_t>() + 8;
    cudaMemsetAsync(cnt, 0, 4, s);
    k_hash_dump<<<(unsigned)((mh.hash_cap + 255) / 256), 256, 0, s>>>(mh.slots.as<HashSlot>(), mh.hash_cap, d_roots.as<lk_map_root>(), cnt);
    cudaError_t e = cudaMemcpyAsync(p, d_roots.p, (size_t)mh.n_roots * sizeof(lk_map_root), cudaMemcpyDeviceToHost, s);
    p += (size_t)mh.n_roots * sizeof(lk_map_root);
    if (e == cudaSuccess && mh.n_nodes) e = cudaMemcpyAsync(p, mh.nodes.p, (size_t)mh.n_nodes * sizeof(MapNode), cudaMemcpyDeviceToHost, s);
    p += (size_t)mh.n_nodes * sizeof(MapNode);
    lk_map_aux* out_aux = (lk_map_aux*)p;
    p += (size_t)mh.n_nodes * sizeof(MapAux);
    lk_map_point* out_pts = (lk_map_point*)p;
    std::vector<DevPoint> dpts((size_t)mh.n_points);
    if (e == cudaSuccess && mh.n_points) e = cudaMemcpyAsync(dpts.data(), mh.points.p, (size_t)mh.n_points * sizeof(DevPoint), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { cudaGetLastError(); err = cudaGetErrorString(e); return LK_ERR_CUDA; }
    uint64_t at = 0;
    for (uint32_t i = 0; i < mh.n_nodes; ++i) {
        lk_map_aux a = aux[i];
        int cnt_i = std::max(a.pts_count, 0);
        for (int j = 0; j < cnt_i; ++j) {
            std::memcpy(out_pts[at + j].pw, dpts[(size_t)a.pts_base + j].pw, 24);
            std::memcpy(out_pts[at + j].var, dpts[(size_t)a.pts_base + j].var, 48);
        }
        a.pts_base = (uint32_t)at;
        a.pts_count = cnt_i;
        out_aux[i] = a;
        at += cnt_i;
    }
    return LK_OK;
}

int map_clear_outside(MapDevHost& mh, const int lo[3], const int hi[3], uint64_t* removed, cudaStream_t s, std::string& err) {
    if (removed) *removed = 0;
    if (!mh.ready()) return LK_OK;
    int rc = mh.sync_counters(s, err);
    if (rc) return rc;
    if (mh.n_roots == 0) return LK_OK;
    DevBuf d_roots, d_cnt;
    LK_CUDA(err, d_roots.alloc((size_t)mh.n_roots * sizeof(lk_map_root)));
    LK_CUDA(err, d_cnt.alloc(4));
    LK_CUDA(err, cudaMemsetAsync(d_cnt.p, 0, 4, s));
    const MapDev md = mh.dev();
    lk_map_root* dr = d_roots.as<lk_map_root>();
    k_hash_dump<<<(unsigned)((mh.hash_cap + 255) / 256), 256, 0, s>>>(md.slots, mh.hash_cap, dr, d_cnt.as<uint32_t>());
    std::vector<lk_map_root> roots(mh.n_roots);
    uint32_t n = 0;
    cudaError_t e = cudaMemcpyAsync(&n, d_cnt.p, 4, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e == cudaSuccess && n) e = cudaMemcpy(roots.data(), dr, (size_t)std::min(n, mh.n_roots) * sizeof(lk_map_root), cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) { cudaGetLastError(); err = cudaGetErrorString(e); return LK_ERR_CUDA; }
    n = std::min(n, mh.n_roots);
    // kept roots first, dropped ones after them
    std::vector<lk_map_root> gone;
    uint32_t keep = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const lk_map_root& r = roots[i];
        const bool out = r.key[0] > hi[0] || r.key[0] < lo[0] || r.key[1] > hi[1] || r.key[1] < lo[1] || r.key[2] > hi[2] || r.key[2] < lo[2];
        if (!out) roots[keep++] = r;
        else gone.push_back(r);
    }
    if (removed) *removed = n - keep;
    if (keep != n) {
        std::copy(gone.begin(), gone.end(), roots.begin() + keep);
        e = cudaMemcpyAsync(dr, roots.data(), (size_t)n * sizeof(lk_map_root), cudaMemcpyHostToDevice, s);
        k_hash_clear<<<(unsigned)((mh.hash_cap + 255) / 256), 256, 0, s>>>(md.slots, mh.hash_cap);
        if (keep) k_hash_insert_roots<<<(keep + 255) / 256, 256, 0, s>>>(md.slots, md.hash_mask, dr, keep, md.overflow);
        // their storage is recycled by the next launch that grows the map
        k_free_subtrees<<<(n - keep + 127) / 128, 128, 0, s>>>(md, dr + keep, n - keep, (int)mh.tile_slots);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    }
    if (e != cudaSuccess) { cudaGetLastError(); err = cudaGetErrorString(e); return LK_ERR_CUDA; }
    if (keep == n) return LK_OK;
    rc = mh.sync_counters(s, err);  // the free lists as the kernel left them
    if (rc) return rc;
    mh.n_roots = keep;
    return mh.push_counters(s, err);
}

int map_count_planes(MapDevHost& mh, uint64_t* planes, uint64_t* live_points, cudaStream_t s, std::string& err) {
    *planes = 0;
    *live_points = 0;
    if (!mh.ready()) return LK_OK;
    int rc = mh.sync_counters(s, err);
    if (rc) return rc;
    unsigned long long* out = reinterpret_cast<unsigned long long*>(mh.counters.as<uint32_t>() + 10);
    LK_CUDA(err, cudaMemsetAsync(out, 0, 16, s));
    if (mh.n_nodes) k_count_planes<<<(mh.n_nodes + 255) / 256, 256, 0, s>>>(mh.nodes.as<MapNode>(), mh.aux.as<MapAux>(), mh.n_nodes, out);
    unsigned long long h[2] = {0, 0};
    LK_CUDA(err, cudaMemcpyAsync(h, out, 16, cudaMemcpyDeviceToHost, s));
    LK_CUDA(err, cudaStreamSynchronize(s));
    *planes = h[0];
    *live_points = h[1];
    return LK_OK;
}

}  // namespace lk
