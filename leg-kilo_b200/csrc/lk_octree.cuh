// lk_octree.cuh — the VoxelOctoTree state machine on device (voxel_map.h:129-176):
//   init_octo_tree  voxel_map.cc:119-137     cut_octo_tree  voxel_map.cc:139-183
//   UpdateOctoTree  voxel_map.cc:185-241     root creation  voxel_map.cc:317-327 / :348-357
// One warp owns one root voxel at a time, so every node of that tree is mutated by exactly one
// warp; lane 0 does the scalar bookkeeping, all lanes cooperate on fits, partitions and copies.
#pragma once
#include "lk_plane.cuh"

namespace lk {

__device__ __forceinline__ bool hash_insert_dev(HashSlot* slots, uint32_t mask, int kx, int ky, int kz, int node) {
    uint32_t i = hash_key(kx, ky, kz) & mask;
    for (uint32_t probe = 0; probe <= mask; ++probe) {
        int* nodep = &slots[i].node;
        int old = atomicCAS(nodep, -1, -2);  // -2 = claimed, key words being written
        if (old == -1) {
            slots[i].kx = kx; slots[i].ky = ky; slots[i].kz = kz;
            __threadfence();
            atomicExch(nodep, node);
            return true;
        }
        i = (i + 1) & mask;
    }
    return false;
}

__device__ __forceinline__ int hash_find_dev(const HashSlot* slots, uint32_t mask, int kx, int ky, int kz) {
    uint32_t i = hash_key(kx, ky, kz) & mask;
    for (;;) {
        int4 s = *reinterpret_cast<const int4*>(slots + i);
        if (s.w == -1) return -1;
        if (s.w >= 0 && s.x == kx && s.y == ky && s.z == kz) return s.w;
        i = (i + 1) & mask;
    }
}

__device__ __forceinline__ int even_up(int v) { return (v + 1) & ~1; }

// keep the node's hot image (lk_device.cuh: HotRec) in step with a plane fit; lane 0 wrote the node record
__device__ __forceinline__ void hot_after_fit(MapDev& md, uint32_t nd, bool is_plane, int lane) {
    if (lane == 0) {
        if (is_plane) hot_fill(md.nodes[nd], md.hot[nd]);
        else md.hot[nd].radius = -1.0f;
    }
}

__device__ __forceinline__ void node_reset(MapDev& md, uint32_t nd, int layer, int parent) {
    MapNode* n = md.nodes + nd;
    double* z = reinterpret_cast<double*>(n);
#pragma unroll
    for (int i = 0; i < 32; ++i) z[i] = 0.0;
    n->flags = LK_NODE_UPDATE_ENABLE | ((uint32_t)layer << LK_NODE_LAYER_SHIFT);  // ctor: update_enable_ = true
    n->child_base = -1;
    md.hot[nd].radius = -1.0f;  // no plane yet
    MapAux* a = md.aux + nd;
    a->pts_base = 0; a->pts_count = 0; a->pts_cap = 0; a->new_points = 0; a->parent = parent;
    a->key[0] = a->key[1] = a->key[2] = 0; a->pad = 0;
}

// voxel_map.cc:320-326 — single lane.
__device__ __forceinline__ void init_root_node(MapDev& md, const Globals& g, uint32_t nd, int kx, int ky, int kz) {
    node_reset(md, nd, 0, -1);
    MapAux* a = md.aux + nd;
    a->voxel_center[0] = (0.5 + kx) * (double)g.voxel_f;
    a->voxel_center[1] = (0.5 + ky) * (double)g.voxel_f;
    a->voxel_center[2] = (0.5 + kz) * (double)g.voxel_f;
    a->quater_length = g.voxel_f / 4;
    a->key[0] = kx; a->key[1] = ky; a->key[2] = kz;
}

// ---- free lists (MapDev::free_*) ---------------------------------------------------------------
// An entry pushed during a launch stays pending until the host promotes it between launches (MapDevHost::push_counters),
// so nothing freed by a launch is handed out again by the same launch: the warps of one launch that mutate different
// roots, and the in-kernel insert across its grid barriers, keep the ordering they have with bump-only allocation.
// Pops only read [0, avail), which no launch writes; a pop that finds the list empty leaves avail <= 0 (the host clamps).
__device__ __forceinline__ bool free_pop(const MapDev& md, int l, uint32_t& v) {
    const int a = atomicSub(reinterpret_cast<int*>(md.free_ctr + 3 * l), 1);
    if (a <= 0) return false;
    v = md.free_items[l][a - 1];
    return true;
}

__device__ __forceinline__ void free_push(const MapDev& md, int l, uint32_t v) {
    const uint32_t t = atomicAdd(md.free_ctr + 3 * l + 2, 1u);
    if (t < md.free_cap[l]) md.free_items[l][t] = v;  // sized for twice the pool: never full in practice, a leak if so
}

__device__ __forceinline__ int std_tile(const Globals& g) { return even_up(g.max_points_num + 2); }

// Bump-allocate `n` point slots (n even). Lane 0 only. Returns base or ~0ull on overflow.
__device__ __forceinline__ unsigned long long alloc_points(MapDev& md, uint32_t n) {
    unsigned long long b = atomicAdd(md.n_points, (unsigned long long)n);
    if (b + n > md.point_cap) {
        atomicOr(md.overflow, 2u);
        return ~0ull;
    }
    return b;
}

// `cap` point slots for one node: a standard tile comes off the free list when it holds one, anything else is bumped.
__device__ __forceinline__ unsigned long long alloc_slots(MapDev& md, const Globals& g, int cap) {
    uint32_t v;
    if (cap == std_tile(g) && free_pop(md, FREE_TILES, v)) return v;
    return alloc_points(md, (uint32_t)cap);
}

// Node `nd` will never read its points again (frozen leaf, cut parent): a standard tile goes back to the free list.
// pts_cap keeps its value, so lk_map_download reports the node exactly as before; pts_base = NO_TILE says the tile
// is gone (a slide must not return it twice). Lane 0 only.
__device__ __forceinline__ void release_tile(MapDev& md, const Globals& g, uint32_t nd) {
    MapAux* a = md.aux + nd;
    if (a->pts_cap == std_tile(g) && a->pts_base != NO_TILE) free_push(md, FREE_TILES, a->pts_base);
    a->pts_base = NO_TILE;
}

__device__ __forceinline__ int alloc_nodes8(MapDev& md) {
    uint32_t v;
    if (free_pop(md, FREE_GROUPS, v)) return (int)v;
    uint32_t b = atomicAdd(md.n_nodes, 8u);
    if (b + 8 > md.node_cap) {
        atomicOr(md.overflow, 1u);
        return -1;
    }
    return (int)b;
}

__device__ __forceinline__ void copy_point(DevPoint* dst, const DevPoint* src) {
    const double2* s = reinterpret_cast<const double2*>(src);
    double2* d = reinterpret_cast<double2*>(dst);
#pragma unroll
    for (int i = 0; i < 5; ++i) d[i] = s[i];
}

// Give node `nd` pool storage holding points [src, src+cnt) with room to grow. Warp-wide.
__device__ inline bool retain_points(MapDev& md, const Globals& g, uint32_t nd, const DevPoint* src, int cnt,
                                     bool in_pool, int lane) {
    if (in_pool) return true;
    int cap = even_up(max(cnt + 1, g.max_points_num + 2));
    unsigned long long base = 0;
    if (lane == 0) base = alloc_slots(md, g, cap);
    base = __shfl_sync(0xffffffffu, base, 0);
    if (base == ~0ull) return false;
    for (int j = lane; j < cnt; j += 32) copy_point(md.points + base + j, src + j);
    if (lane == 0) {
        MapAux* a = md.aux + nd;
        a->pts_base = (uint32_t)base;
        a->pts_count = cnt;
        a->pts_cap = cap;
    }
    __syncwarp();
    return true;
}

__device__ __forceinline__ int octant_of(const DevPoint* p, const double* vc) {
    return 4 * (p->pw[0] > vc[0] ? 1 : 0) + 2 * (p->pw[1] > vc[1] ? 1 : 0) + (p->pw[2] > vc[2] ? 1 : 0);
}

// Child creation (voxel_map.cc:151-157 / :220-226). Lane 0.
__device__ __forceinline__ void init_child_node(MapDev& md, uint32_t parent, uint32_t child, int oct) {
    const MapAux* pa = md.aux + parent;
    int layer = (int)((md.nodes[parent].flags >> LK_NODE_LAYER_SHIFT) & 0xffu) + 1;
    node_reset(md, child, layer, (int)parent);
    MapAux* a = md.aux + child;
    const int xyz[3] = {(oct >> 2) & 1, (oct >> 1) & 1, oct & 1};
#pragma unroll
    for (int k = 0; k < 3; ++k) a->voxel_center[k] = pa->voxel_center[k] + (double)((float)(2 * xyz[k] - 1) * pa->quater_length);
    a->quater_length = pa->quater_length / 2;
}

// cut_octo_tree's distribution loop (voxel_map.cc:144-160): stable partition of the node's points
// into octant children. Returns the child base (or -1). cnt_out[8] receives the child counts.
__device__ inline int warp_cut(MapDev& md, const Globals& g, uint32_t nd, const DevPoint* src, int cnt, int* cnt_out,
                               int lane) {
    double vc[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) vc[k] = md.aux[nd].voxel_center[k];
    int counts[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) counts[c] = 0;
    for (int j0 = 0; j0 < cnt; j0 += 32) {
        int j = j0 + lane;
        int o = (j < cnt) ? octant_of(src + j, vc) : -1;
#pragma unroll
        for (int c = 0; c < 8; ++c) counts[c] += __popc(__ballot_sync(0xffffffffu, o == c));
    }
    // a child of the standard size takes a tile of its own (recyclable); the larger ones share one bump block
    const int tile = std_tile(g);
    int caps[8], offs[8], total = 0;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        caps[c] = counts[c] > 0 ? even_up(max(counts[c] + 1, g.max_points_num + 2)) : 0;
        offs[c] = total;
        if (caps[c] != tile) total += caps[c];
        cnt_out[c] = counts[c];
    }
    int cbase = -1;
    unsigned long long pbase = 0;
    if (lane == 0) {
        cbase = md.nodes[nd].child_base;
        if (cbase < 0) cbase = alloc_nodes8(md);
        pbase = (cbase >= 0 && total > 0) ? alloc_points(md, (uint32_t)total) : 0;
    }
    cbase = __shfl_sync(0xffffffffu, cbase, 0);
    pbase = __shfl_sync(0xffffffffu, pbase, 0);
    if (cbase < 0 || pbase == ~0ull) return -1;
    bool mine = false;  // lane c < 8 allocates child c's own tile
#pragma unroll
    for (int c = 0; c < 8; ++c) mine |= lane == c && caps[c] == tile;
    unsigned long long own = mine ? alloc_slots(md, g, tile) : 0;
    bool failed = false;
    unsigned long long cpb[8], my_pb = 0;  // first slot of each child's points; lane c < 8: child c's
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const unsigned long long t = __shfl_sync(0xffffffffu, own, c);
        cpb[c] = (caps[c] == tile) ? t : pbase + offs[c];
        failed |= cpb[c] == ~0ull;
        if (lane == c) my_pb = cpb[c];
    }
    if (failed) return -1;
    int run[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) run[c] = 0;
    const uint32_t lt = (1u << lane) - 1u;
    for (int j0 = 0; j0 < cnt; j0 += 32) {
        int j = j0 + lane;
        int o = (j < cnt) ? octant_of(src + j, vc) : -1;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            uint32_t m = __ballot_sync(0xffffffffu, o == c);
            if (o == c) copy_point(md.points + cpb[c] + run[c] + __popc(m & lt), src + j);
            run[c] += __popc(m);
        }
    }
    __syncwarp();
    if (lane < 8) {
        const int c = lane;
        uint32_t child = (uint32_t)cbase + c;
        const bool existed = (md.nodes[nd].flags >> (LK_NODE_CHILDMASK_SHIFT + c)) & 1u;
        if (!existed) {
            init_child_node(md, nd, child, c);
            MapAux* a = md.aux + child;
            a->pts_base = (uint32_t)my_pb;
            a->pts_count = counts[c];
            a->pts_cap = caps[c];
            a->new_points = counts[c];  // new_points_++ per pushed point (:159)
        }
    }
    __syncwarp();
    if (lane == 0) {
        uint32_t mask = 0;
#pragma unroll
        for (int c = 0; c < 8; ++c)
            if (counts[c] > 0) mask |= 1u << c;
        MapNode* n = md.nodes + nd;
        n->child_base = cbase;
        n->flags |= mask << LK_NODE_CHILDMASK_SHIFT;
    }
    __syncwarp();
    return cbase;
}

// init_octo_tree on node `root_nd` whose `cnt` points sit at `src` (voxel_map.cc:119-137), with the
// recursion of cut_octo_tree (:161-182) unrolled through a small per-warp stack.
__device__ inline void warp_init_octo_tree(MapDev& md, const Globals& g, WarpTile* wt, uint32_t root_nd,
                                           const DevPoint* src0, int cnt0, bool pts_in_pool, int lane) {
    uint32_t stack[40];
    int sp = 0;
    stack[sp++] = root_nd;
    bool first = true;
    while (sp > 0) {
        const uint32_t nd = stack[--sp];
        const DevPoint* src;
        int cnt;
        bool in_pool;
        if (first) {
            src = src0; cnt = cnt0; in_pool = pts_in_pool;
            first = false;
        } else {
            src = md.points + md.aux[nd].pts_base;
            cnt = md.aux[nd].pts_count;
            in_pool = true;
        }
        const uint32_t flags0 = md.nodes[nd].flags;
        const int layer = (int)((flags0 >> LK_NODE_LAYER_SHIFT) & 0xffu);
        const int thr = g.layer_init_num[layer];
        __syncwarp();
        if (cnt > thr) {
            const bool is_plane = warp_fit_plane(wt, src, cnt, md.nodes + nd, g.planer_threshold, lane);
            hot_after_fit(md, nd, is_plane, lane);
            if (is_plane) {
                if (cnt > g.max_points_num) {  // freeze and free (:126-130)
                    if (lane == 0) {
                        md.nodes[nd].flags = (flags0 | LK_NODE_IS_PLANE | LK_NODE_INIT_OCTO) & ~LK_NODE_UPDATE_ENABLE;
                        md.aux[nd].pts_count = 0;
                        md.aux[nd].new_points = 0;
                        if (in_pool) release_tile(md, g, nd);
                    }
                } else {
                    retain_points(md, g, nd, src, cnt, in_pool, lane);
                    if (lane == 0) {
                        md.nodes[nd].flags = flags0 | LK_NODE_IS_PLANE | LK_NODE_INIT_OCTO;
                        md.aux[nd].new_points = 0;
                    }
                }
            } else {
                if (layer >= g.max_layer) {  // cut_octo_tree returns at once: stays a leaf (:140-143)
                    retain_points(md, g, nd, src, cnt, in_pool, lane);
                    if (lane == 0) {
                        md.nodes[nd].flags = (flags0 | LK_NODE_INIT_OCTO) & ~LK_NODE_IS_PLANE;
                        md.aux[nd].new_points = 0;
                    }
                } else {
                    int ccnt[8];
                    int cbase = warp_cut(md, g, nd, src, cnt, ccnt, lane);
                    if (lane == 0) {
                        md.nodes[nd].flags = (md.nodes[nd].flags | LK_NODE_INIT_OCTO) & ~LK_NODE_IS_PLANE;
                        md.aux[nd].pts_count = 0;  // the parent never looks at its own points again
                        md.aux[nd].new_points = 0;
                        // warp_cut copied them out before its last __syncwarp; the bulk build's sorted scratch is no tile
                        if (in_pool && cbase >= 0) release_tile(md, g, nd);
                    }
                    if (cbase >= 0) {
                        const int thr_c = g.layer_init_num[layer + 1 < 5 ? layer + 1 : 4];
                        for (int c = 7; c >= 0; --c)
                            if (ccnt[c] > thr_c && sp < 40) stack[sp++] = (uint32_t)cbase + c;
                    }
                }
            }
        } else {
            // below the init threshold: keep collecting (only reachable for the first node)
            retain_points(md, g, nd, src, cnt, in_pool, lane);
            if (lane == 0) md.aux[nd].new_points = cnt;
        }
        __syncwarp();
    }
}

// Append one point to a node's retained list (temp_points_.push_back). Warp-wide; lane 0 writes.
__device__ inline void warp_append(MapDev& md, const Globals& g, uint32_t nd, const DevPoint& p, int lane) {
    if (lane == 0) {
        MapAux* a = md.aux + nd;
        if (a->pts_cap == 0) {
            const int cap = std_tile(g);
            unsigned long long b = alloc_slots(md, g, cap);
            if (b != ~0ull) {
                a->pts_base = (uint32_t)b;
                a->pts_cap = cap;
                a->pts_count = 0;
            }
        }
        if (a->pts_count < a->pts_cap) {
            md.points[a->pts_base + a->pts_count] = p;
            a->pts_count += 1;
        } else if (a->pts_cap > 0) {
            atomicOr(md.overflow, 8u);  // list full: only possible for a leaf that freezes right now
        }
        a->new_points += 1;
    }
    __syncwarp();
}

// VoxelOctoTree::UpdateOctoTree(pv) starting at root `nd` (voxel_map.cc:185-241). Warp-wide.
__device__ inline void warp_update_octo_tree(MapDev& md, const Globals& g, WarpTile* wt, uint32_t nd, const DevPoint& p,
                                             int lane) {
    for (int depth = 0;; ++depth) {
        __syncwarp();
        if (depth > 8) {  // deeper than any max_layer: the tree is corrupt (see lk_stall_note)
            stall_note(3u, nd);
            return;
        }
        const uint32_t flags = md.nodes[nd].flags;
        const int layer = (int)((flags >> LK_NODE_LAYER_SHIFT) & 0xffu);
        if (!(flags & LK_NODE_INIT_OCTO)) {
            warp_append(md, g, nd, p, lane);
            const int cnt = md.aux[nd].pts_count;
            if (cnt > g.layer_init_num[layer])
                warp_init_octo_tree(md, g, wt, nd, md.points + md.aux[nd].pts_base, cnt, true, lane);
            return;
        }
        const bool leaf_branch = (flags & LK_NODE_IS_PLANE) || layer >= g.max_layer;
        if (leaf_branch) {
            if (flags & LK_NODE_UPDATE_ENABLE) {
                warp_append(md, g, nd, p, lane);
                const int cnt = md.aux[nd].pts_count;
                const int newp = md.aux[nd].new_points;
                if (newp > 5) {  // update_size_threshold_ = 5 (voxel_map.h:157)
                    const bool pl = warp_fit_plane(wt, md.points + md.aux[nd].pts_base, cnt, md.nodes + nd,
                                                   g.planer_threshold, lane);
                    hot_after_fit(md, nd, pl, lane);
                    if (lane == 0) {
                        uint32_t f = md.nodes[nd].flags;
                        md.nodes[nd].flags = pl ? (f | LK_NODE_IS_PLANE) : (f & ~LK_NODE_IS_PLANE);
                        md.aux[nd].new_points = 0;
                    }
                    __syncwarp();
                }
                // freeze test: plane branch ">=" (:199), max-layer branch ">" (:232). The branch was
                // chosen on the flags BEFORE a possible refit, exactly as the reference's if/else.
                const bool freeze = (flags & LK_NODE_IS_PLANE) ? (cnt >= g.max_points_num) : (cnt > g.max_points_num);
                if (freeze && lane == 0) {
                    md.nodes[nd].flags &= ~LK_NODE_UPDATE_ENABLE;
                    md.aux[nd].pts_count = 0;
                    md.aux[nd].new_points = 0;
                    release_tile(md, g, nd);  // the points are dropped (:206): update_enable is off for good
                }
            }
            return;
        }
        // initialised, not a plane, above max_layer: route to the octant child (:208-227)
        double vc[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) vc[k] = md.aux[nd].voxel_center[k];
        const int oct = octant_of(&p, vc);
        int cbase = md.nodes[nd].child_base;
        if (cbase < 0) {
            if (lane == 0) {
                cbase = alloc_nodes8(md);
                if (cbase >= 0) {
                    for (int c = 0; c < 8; ++c) node_reset(md, (uint32_t)cbase + c, layer + 1, (int)nd);
                    md.nodes[nd].child_base = cbase;
                }
            }
            cbase = __shfl_sync(0xffffffffu, cbase, 0);
            if (cbase < 0) return;
        }
        if (!((flags >> (LK_NODE_CHILDMASK_SHIFT + oct)) & 1u)) {
            if (lane == 0) {
                init_child_node(md, nd, (uint32_t)cbase + oct, oct);
                md.nodes[nd].flags |= 1u << (LK_NODE_CHILDMASK_SHIFT + oct);
            }
            __syncwarp();
        }
        nd = (uint32_t)cbase + oct;
    }
}

}  // namespace lk
