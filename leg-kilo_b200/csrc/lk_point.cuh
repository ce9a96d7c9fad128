// lk_point.cuh — the per-point steps of rows a3-a7 of SURVEY.md §8a, each written once: the LiDAR point in the IMU and body
// frames, the float voxel key and the one neighbour voxel, the node record and its plane, the gates and the row, the octree
// descent. The block-wide pass (lk_pass.cuh) and the throughput family (lk_stream2.cu) are built from them, and point_row runs
// one point through the whole sequence straight from global memory for the throughput family's fallback kernel. Also the
// warp-level reduction / 6x6 solve primitives.
//
// Follows: a3 KILO.cc:127-140 + voxel_map.cc:22-40, a4 KILO.cc:143-149, a5 voxel_map.cc:363-427,
// a6 KILO.cc:156-178, a7 KILO.cc:187-210. Algebra is restructured (never the results' meaning):
//   * calcBodyCov's A*A^T is range^2 (I - u u^T) because {b1, b2, u} is orthonormal, so
//     n^T M Sigma_b M^T n = rv (u.w)^2 + range^2 dv (|w|^2 - (u.w)^2), w = M^T n;
//   * n^T (R[pi]x) P_tt (R[pi]x)^T n = h_t^T P_tt h_t with h_t = pi x (R^T n), the Jacobian row itself.
#pragma once
#include "lk_device.cuh"

namespace lk {

struct PlaneRec {
    double c[3], n[3], pv[21];
    float d, radius;
    uint32_t flags;
    int child_base;
};

// The first 15 x 16 bytes of a node record (lk_map_node: centre .. flags / child_base), the 232 bytes the path needs.
__device__ __forceinline__ void unpack_plane(const double2 (&v)[15], PlaneRec& r) {
    r.c[0] = v[0].x; r.c[1] = v[0].y; r.c[2] = v[1].x;
    r.n[0] = v[1].y; r.n[1] = v[2].x; r.n[2] = v[2].y;
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        r.pv[2 * i] = v[3 + i].x;
        r.pv[2 * i + 1] = v[3 + i].y;
    }
    r.pv[20] = v[13].x;
    long long dr = __double_as_longlong(v[13].y);
    r.d = __int_as_float((int)(dr & 0xffffffffll));
    r.radius = __int_as_float((int)(dr >> 32));
    long long fc = __double_as_longlong(v[14].x);
    r.flags = (uint32_t)(fc & 0xffffffffll);
    r.child_base = (int)(fc >> 32);
}

// From global memory, 15 x 128-bit loads. COH = the map may be written by this very kernel (persistent per-scan kernel with
// the map insert inside): read through L2 instead of the non-coherent path.
template <bool COH = false>
__device__ __forceinline__ void load_plane(const MapNode* __restrict__ nd, PlaneRec& r) {
    const double2* q = reinterpret_cast<const double2*>(nd);
    double2 v[15];
#pragma unroll
    for (int i = 0; i < 15; ++i) v[i] = COH ? __ldcg(q + i) : __ldg(q + i);
    unpack_plane(v, r);
}

// From a record staged in shared memory (lk_pass.cuh: Stage<false>).
__device__ __forceinline__ void plane_from_smem(const unsigned char* slot, PlaneRec& r) {
    const double2* q = reinterpret_cast<const double2*>(slot);
    double2 v[15];
#pragma unroll
    for (int i = 0; i < 15; ++i) v[i] = q[i];
    unpack_plane(v, r);
}

struct PointCtx {
    double pbx, pby, pbz;  // lidar-frame point as calcBodyCov sees it (z == 0 -> 1e-4)
    double pix, piy, piz;  // IMU frame
    double pwx, pwy, pwz;  // world
    double r2;             // |pb|^2
    double range2;         // (double)(float range)^2   (voxel_map.cc:24)
};

struct Row {
    double h[6];
    double z;
    double R;
};

// The LiDAR point in the IMU frame, pi = Re pb + te (KILO.cc:127-140). P: anything with pix / piy / piz.
template <class P>
__device__ __forceinline__ void imu_point(float4 pt, const Globals& g, P& p) {
    const double bx = (double)pt.x, by = (double)pt.y, bz = (double)pt.z;
    p.pix = g.Re[0] * bx + g.Re[1] * by + g.Re[2] * bz + g.te[0];
    p.piy = g.Re[3] * bx + g.Re[4] * by + g.Re[5] * bz + g.te[1];
    p.piz = g.Re[6] * bx + g.Re[7] * by + g.Re[8] * bz + g.te[2];
}

// The point as calcBodyCov sees it: pb with z == 0 -> 1e-4, a mutation made AFTER pi / pw were formed (voxel_map.cc:23,
// KILO.cc:134), |pb|^2 and the float range squared (voxel_map.cc:24). P: PointCtx or LaneCache.
template <class P>
__device__ __forceinline__ void body_terms(float4 pt, P& p) {
    const double bx = (double)pt.x, by = (double)pt.y, bz = (double)pt.z;
    p.pbx = bx; p.pby = by; p.pbz = (bz == 0.0) ? 0.0001 : bz;
    p.r2 = p.pbx * p.pbx + p.pby * p.pby + p.pbz * p.pbz;
    const float range = (float)sqrt(p.r2);
    p.range2 = (double)range * (double)range;
}

// Everything of a point that does not depend on the state.
template <class P>
__device__ __forceinline__ void body_point(float4 pt, const Globals& g, P& p) {
    imu_point(pt, g, p);
    body_terms(pt, p);
}

// pw = R pi + p at the state of sc
__device__ __forceinline__ void world_point(PointCtx& pc, const ScanConst& sc) {
    pc.pwx = sc.R[0] * pc.pix + sc.R[1] * pc.piy + sc.R[2] * pc.piz + sc.p[0];
    pc.pwy = sc.R[3] * pc.pix + sc.R[4] * pc.piy + sc.R[5] * pc.piz + sc.p[1];
    pc.pwz = sc.R[6] * pc.pix + sc.R[7] * pc.piy + sc.R[8] * pc.piz + sc.p[2];
}

// voxel key in float: quotient, -1 shift for negatives; the caller truncates (KILO.cc:143-148)
__device__ __forceinline__ void voxel_loc(const PointCtx& pc, const Globals& g, float& lx, float& ly, float& lz) {
    if (g.voxel_pow2) {
        lx = (float)(pc.pwx * g.inv_voxel); ly = (float)(pc.pwy * g.inv_voxel); lz = (float)(pc.pwz * g.inv_voxel);
    } else {
        lx = (float)(pc.pwx / g.voxel); ly = (float)(pc.pwy / g.voxel); lz = (float)(pc.pwz / g.voxel);
    }
    if (lx < 0) lx = (float)((double)lx - 1.0);
    if (ly < 0) ly = (float)((double)ly - 1.0);
    if (lz < 0) lz = (float)((double)lz - 1.0);
}

// the ONE neighbour the reference falls back to: loc in VOXEL units against a centre in METRES (the reference's
// own unit mismatch, KILO.cc:158-172)
__device__ __forceinline__ void neighbour_key(const Globals& g, float lx, float ly, float lz, int kx, int ky, int kz, int& nx,
                                              int& ny, int& nz) {
    const double q = (double)(g.voxel_f / 4.0f);
    const double cx = (0.5 + kx) * (double)g.voxel_f, cy = (0.5 + ky) * (double)g.voxel_f, cz = (0.5 + kz) * (double)g.voxel_f;
    nx = kx; ny = ky; nz = kz;
    if ((double)lx > cx + q) nx++; else if ((double)lx < cx - q) nx--;
    if ((double)ly > cy + q) ny++; else if ((double)ly < cy - q) ny--;
    if ((double)lz > cz + q) nz++; else if ((double)lz < cz - q) nz--;
}

// The whole per-point preparation of a pass that sees the point once: body_point, pw and the float voxel key.
__device__ __forceinline__ void prepare_point(float4 pt, const ScanConst& sc, const Globals& g, PointCtx& pc, float& lx,
                                              float& ly, float& lz) {
    body_point(pt, g, pc);
    world_point(pc, sc);
    voxel_loc(pc, g, lx, ly, lz);
}

__device__ __forceinline__ double quad_sym3(const double* S, double a, double b, double c) {
    return S[0] * a * a + S[3] * b * b + S[5] * c * c + 2.0 * (S[1] * a * b + S[2] * a * c + S[4] * b * c);
}

// What follows the first gate of build_single_residual's plane branch (voxel_map.cc:382-411) and the row of KILO.cc:192-209,
// for a plane with normal n, s = n.pw + d, dis = |s| in float and sigma_plane = J_nq Sigma_plane J_nq^T.
__device__ __forceinline__ bool plane_row(double n0, double n1, double n2, double s, float dis, double sigma_pl, const PointCtx& pc,
                                          const ScanConst& sc, const Globals& g, bool need_prob, double& prob, Row& row) {
    // q = R^T n ; h_theta = pi x q ; w = (R Re)^T n = Re^T q
    const double qx = sc.R[0] * n0 + sc.R[3] * n1 + sc.R[6] * n2;
    const double qy = sc.R[1] * n0 + sc.R[4] * n1 + sc.R[7] * n2;
    const double qz = sc.R[2] * n0 + sc.R[5] * n1 + sc.R[8] * n2;
    const double hx = pc.piy * qz - pc.piz * qy;
    const double hy = pc.piz * qx - pc.pix * qz;
    const double hz = pc.pix * qy - pc.piy * qx;
    const double wx = g.Re[0] * qx + g.Re[3] * qy + g.Re[6] * qz;
    const double wy = g.Re[1] * qx + g.Re[4] * qy + g.Re[7] * qz;
    const double wz = g.Re[2] * qx + g.Re[5] * qy + g.Re[8] * qz;
    const double uw = pc.pbx * wx + pc.pby * wy + pc.pbz * wz;
    const double ww = wx * wx + wy * wy + wz * wz;
    const double uw2 = uw * uw / pc.r2;  // (u.w)^2
    const double body = (double)g.rv * uw2 + pc.range2 * g.dv * (ww - uw2);
    const double state = quad_sym3(sc.Pth, hx, hy, hz) + quad_sym3(sc.Ppp, n0, n1, n2);
    const double sigma_l = sigma_pl + body + state;

    // gate 2: dis_to_plane < sigma_num * sqrt(sigma_l)   (voxel_map.cc:387), squared with an exact
    // fallback at the boundary so the decision equals the reference's comparison.
    const double lhs = (double)dis * (double)dis;
    const double rhs = g.sigma_num * g.sigma_num * sigma_l;
    bool pass;
    if (lhs < rhs * (1.0 - 1e-12)) pass = true;
    else if (lhs > rhs * (1.0 + 1e-12)) pass = false;
    else pass = (double)dis < g.sigma_num * sqrt(sigma_l);
    if (!pass) return false;
    if (need_prob) {
        const double this_prob = 1.0 / sqrt(sigma_l) * exp(-0.5 * (double)dis * (double)dis / sigma_l);
        if (!(this_prob > prob)) return true;  // is_success without replacing the candidate
        prob = this_prob;
    }
    row.h[0] = hx; row.h[1] = hy; row.h[2] = hz;
    row.h[3] = n0; row.h[4] = n1; row.h[5] = n2;
    row.z = -(double)(float)s;  // dis_to_plane_ is float (voxel_map.h:92)
    row.R = g.ratio * (sigma_pl + body);
    return true;
}

// build_single_residual's plane branch (voxel_map.cc:370-411) + the row of KILO.cc:192-209, on a node record.
__device__ __forceinline__ bool eval_plane(const PlaneRec& r, const PointCtx& pc, const ScanConst& sc,
                                           const Globals& g, bool need_prob, double& prob, Row& row) {
    double s = r.n[0] * pc.pwx + r.n[1] * pc.pwy + r.n[2] * pc.pwz + (double)r.d;
    float dis = (float)fabs(s);
    double ax = pc.pwx - r.c[0], ay = pc.pwy - r.c[1], az = pc.pwz - r.c[2];
    float dc = (float)(ax * ax + ay * ay + az * az);
    float rd = sqrtf(__fsub_rn(dc, __fmul_rn(dis, dis)));  // float arithmetic as in the reference
    if (!((double)rd <= 3.0 * (double)r.radius)) return false;

    // J_nq Sigma_plane J_nq^T, J_nq = [(pw - c)^T, -n^T]
    const double J0 = ax, J1 = ay, J2 = az, J3 = -r.n[0], J4 = -r.n[1], J5 = -r.n[2];
    const double* pv = r.pv;
    double t0 = pv[0] * J0 + 2.0 * (pv[1] * J1 + pv[2] * J2 + pv[3] * J3 + pv[4] * J4 + pv[5] * J5);
    double t1 = pv[6] * J1 + 2.0 * (pv[7] * J2 + pv[8] * J3 + pv[9] * J4 + pv[10] * J5);
    double t2 = pv[11] * J2 + 2.0 * (pv[12] * J3 + pv[13] * J4 + pv[14] * J5);
    double t3 = pv[15] * J3 + 2.0 * (pv[16] * J4 + pv[17] * J5);
    double t4 = pv[18] * J4 + 2.0 * (pv[19] * J5);
    double t5 = pv[20] * J5;
    double sigma_pl = J0 * t0 + J1 * t1 + J2 * t2 + J3 * t3 + J4 * t4 + J5 * t5;
    return plane_row(r.n[0], r.n[1], r.n[2], s, dis, sigma_pl, pc, sc, g, need_prob, prob, row);
}

// eval_plane (need_prob = false) on a staged hot image (lk_device.cuh: HotRec, 144 bytes, 16-byte aligned, nine 128-bit
// loads): sigma_plane = a^T Scc a - 2 a^T v + s. Everything else as eval_plane.
// Returns 0 = row produced, 1 = the node holds no plane (octree descent needed), 2 = a plane, but the point is gated out.
__device__ __forceinline__ int eval_plane_hot(const unsigned char* slot, const PointCtx& pc, const ScanConst& sc, const Globals& g,
                                              Row& row) {
    const double2* q = reinterpret_cast<const double2*>(slot);
    const float2 dr = *reinterpret_cast<const float2*>(q + 8);
    if (dr.y < 0.0f) return 1;  // no plane in this node
    const double2 v0 = q[0], v1 = q[1], v2 = q[2];
    const double c0 = v0.x, c1 = v0.y, c2 = v1.x, n0 = v1.y, n1 = v2.x, n2 = v2.y;
    const double s = n0 * pc.pwx + n1 * pc.pwy + n2 * pc.pwz + (double)dr.x;
    const float dis = (float)fabs(s);
    const double ax = pc.pwx - c0, ay = pc.pwy - c1, az = pc.pwz - c2;
    const float dc = (float)(ax * ax + ay * ay + az * az);
    const float rd = sqrtf(__fsub_rn(dc, __fmul_rn(dis, dis)));
    if (!((double)rd <= 3.0 * (double)dr.y)) return 2;
    const double2 v3 = q[3], v4 = q[4], v5 = q[5], v6 = q[6], v7 = q[7];
    const double scc[6] = {v3.x, v3.y, v4.x, v4.y, v5.x, v5.y};
    const double sigma_pl = quad_sym3(scc, ax, ay, az) - 2.0 * (ax * v6.x + ay * v6.y + az * v7.x) + v7.y;
    double prob = 0.0;
    return plane_row(n0, n1, n2, s, dis, sigma_pl, pc, sc, g, false, prob, row) ? 0 : 2;
}

__device__ __forceinline__ int map_find(const HashSlot* __restrict__ slots, uint32_t mask, int kx, int ky, int kz) {
    uint32_t i = hash_key(kx, ky, kz) & mask;
    for (;;) {
        int4 s = __ldg(reinterpret_cast<const int4*>(slots + i));
        if (s.w < 0) return -1;
        if (s.x == kx && s.y == ky && s.z == kz) return s.w;
        i = (i + 1) & mask;
    }
}

// Rare path of build_single_residual (voxel_map.cc:412-424): the root is not a plane, so every
// initialised plane among ALL children of non-plane nodes down to max_layer is a candidate and the
// most probable one wins. Kept out of line so the common path does not carry its registers.
template <bool COH = false>
static __device__ __noinline__ bool visit_subtree(const MapNode* __restrict__ nodes, int child_base, uint32_t cmask,
                                           const PointCtx* pcp, const ScanConst* scp, const Globals* gp, double* probp,
                                           Row* rowp) {
    const PointCtx& pc = *pcp;
    const ScanConst& sc = *scp;
    const Globals& g = *gp;
    bool ok = false;
    int st_base[4];
    uint32_t st_mask[4];
    int sp = 1;
    st_base[0] = child_base;
    st_mask[0] = cmask;
    double prob = *probp;
    Row row = *rowp;
    while (sp > 0) {
        uint32_t m = st_mask[sp - 1];
        if (m == 0) { --sp; continue; }
        int c = __ffs(m) - 1;  // child order 0..7 as the reference's loop
        st_mask[sp - 1] = m & (m - 1);
        int layer = sp;  // children of a layer-(sp-1) node
        PlaneRec cr;
        load_plane<COH>(nodes + st_base[sp - 1] + c, cr);
        if (cr.flags & LK_NODE_IS_PLANE) {
            if (eval_plane(cr, pc, sc, g, true, prob, row)) ok = true;
        } else if (layer < g.max_layer && sp < 4) {
            uint32_t cm = (cr.flags >> LK_NODE_CHILDMASK_SHIFT) & 0xffu;
            if (cr.child_base >= 0 && cm) {
                st_base[sp] = cr.child_base;
                st_mask[sp] = cm;
                ++sp;
            }
        }
    }
    *probp = prob;
    *rowp = row;
    return ok;
}

// One root through build_single_residual (voxel_map.cc:363-427) from its node record: the plane decides, or, when the root
// holds no plane, every plane among its children competes (voxel_map.cc:412-424).
template <bool COH = false>
__device__ __forceinline__ bool eval_record(const MapNode* __restrict__ nodes, const PlaneRec& r, const PointCtx& pc,
                                            const ScanConst& sc, const Globals& g, Row& row) {
    double prob = 0.0;
    if (r.flags & LK_NODE_IS_PLANE) return eval_plane(r, pc, sc, g, false, prob, row);
    const uint32_t cmask = (r.flags >> LK_NODE_CHILDMASK_SHIFT) & 0xffu;
    if (g.max_layer >= 1 && r.child_base >= 0 && cmask) return visit_subtree<COH>(nodes, r.child_base, cmask, &pc, &sc, &g, &prob, &row);
    return false;
}

// Root `root` holds no plane (eval_plane_hot returned 1): the descent of eval_record, with the root's flags and child base
// from one dependent read of its node record (rare). The guard is eval_record's, written out again: shared through an
// inlined helper, the compiler places the early returns differently and the batch-of-one scan kernels' code changes.
template <bool COH = false>
__device__ __forceinline__ bool eval_descent(const MapNode* __restrict__ nodes, int root, const PointCtx& pc, const ScanConst& sc,
                                             const Globals& g, Row& row) {
    if (g.max_layer < 1) return false;
    const uint2* fcp = reinterpret_cast<const uint2*>(&nodes[root].flags);
    const uint2 fc = COH ? __ldcg(fcp) : __ldg(fcp);
    const uint32_t cmask = (fc.x >> LK_NODE_CHILDMASK_SHIFT) & 0xffu;
    const int child_base = (int)fc.y;
    if (child_base < 0 || !cmask) return false;
    double prob = 0.0;
    return visit_subtree<COH>(nodes, child_base, cmask, &pc, &sc, &g, &prob, &row);
}

// One point through rows a3-a7. Returns true when a residual row was produced.
__device__ __forceinline__ bool point_row(float4 pt, const ScanConst& sc, const MapView& a, const Globals& g, Row& row) {
    PointCtx pc;
    imu_point(pt, g, pc);
    world_point(pc, sc);
    float lx, ly, lz;
    voxel_loc(pc, g, lx, ly, lz);
    const int kx = (int)lx, ky = (int)ly, kz = (int)lz;
    int root = map_find(a.slots, a.hash_mask, kx, ky, kz);  // issue the probe before the fp64 work below
    if (root < 0) return false;
    body_terms(pt, pc);

    // home voxel first; on failure ONE (possibly diagonal) neighbour (KILO.cc:156-178). This loop keeps its own copies of
    // eval_record's choice and of neighbour_key: written with them, the fallback kernel's code changed and the batched
    // throughput workload measured 0.55 % slower (1.557 against 1.565 x 10^10 point-iterations/s, three alternating runs each,
    // spread 0.1 %, one H100 80GB HBM3 at a 700 W power limit).
    double prob = 0.0;
    bool ok = false;
    int nx = kx, ny = ky, nz = kz;
#pragma unroll 1
    for (int attempt = 0; attempt < 2; ++attempt) {
        PlaneRec r;
        load_plane(a.nodes + root, r);
        if (r.flags & LK_NODE_IS_PLANE) {
            ok = eval_plane(r, pc, sc, g, false, prob, row);
        } else {
            uint32_t cmask = (r.flags >> LK_NODE_CHILDMASK_SHIFT) & 0xffu;
            if (g.max_layer >= 1 && r.child_base >= 0 && cmask)
                ok = visit_subtree(a.nodes, r.child_base, cmask, &pc, &sc, &g, &prob, &row);
        }
        if (ok || attempt == 1) break;
        // loc in VOXEL units against a centre in METRES: the reference's own unit mismatch
        double q = (double)(g.voxel_f / 4.0f);
        double cx = (0.5 + kx) * (double)g.voxel_f, cy = (0.5 + ky) * (double)g.voxel_f, cz = (0.5 + kz) * (double)g.voxel_f;
        if ((double)lx > cx + q) nx++; else if ((double)lx < cx - q) nx--;
        if ((double)ly > cy + q) ny++; else if ((double)ly < cy - q) ny--;
        if ((double)lz > cz + q) nz++; else if ((double)lz < cz - q) nz--;
        if (nx == kx && ny == ky && nz == kz) break;
        root = map_find(a.slots, a.hash_mask, nx, ny, nz);
        if (root < 0) break;
    }
    return ok;
}

// One exchange step of warp_transpose_sum. The offset must be a compile-time constant: a loop over halving offsets has no
// trip count the compiler can find, stays rolled, and the array it indexes then lives in local memory.
template <int OFF>
__device__ __forceinline__ void warp_transpose_step(double (&v)[32], int lane) {
    const bool upper = (lane & OFF) != 0;
#pragma unroll
    for (int i = 0; i < OFF; ++i) {
        double send = upper ? v[i] : v[i + OFF];
        double keep = upper ? v[i + OFF] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);
    }
}

// Sum of 32 per-lane values over the warp with value/lane transposition: after the 5 exchange
// steps lane L holds the warp total of value L (31 exchanges instead of 32 x 5 shuffles).
__device__ __forceinline__ double warp_transpose_sum(double (&v)[32], int lane) {
    warp_transpose_step<16>(v, lane);
    warp_transpose_step<8>(v, lane);
    warp_transpose_step<4>(v, lane);
    warp_transpose_step<2>(v, lane);
    warp_transpose_step<1>(v, lane);
    return v[0];
}

// The block's sum of every thread's 32 accumulators in one fixed order: the warp's transposing tree, one row per warp in
// `slice` (WARPS * 32 doubles), the warps' rows added in warp order by warp 0, whose lane i hands the sum of accumulator i
// to store(i, v).
template <int WARPS, class Store>
__device__ __forceinline__ void block_row(double (&acc)[32], double* slice, Store store) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    slice[warp * 32 + lane] = warp_transpose_sum(acc, lane);
    __syncthreads();
    if (tid < 32) {
        double v = 0.0;
#pragma unroll
        for (int w = 0; w < WARPS; ++w) v += slice[w * 32 + tid];
        store(tid, v);
    }
}

// 6 x 6 solve [M | b | A] -> [I | y | W] by Gauss-Jordan with partial pivoting, one column per
// lane (lanes 0..12), executed by one full warp. Returns false on a zero pivot.
__device__ __forceinline__ bool warp_solve6(double (&col)[6], int lane) {
    bool ok = true;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        double ck[6];
#pragma unroll
        for (int i = 0; i < 6; ++i) ck[i] = __shfl_sync(0xffffffffu, col[i], k);
        int piv = k;
        double best = fabs(ck[k]);
#pragma unroll
        for (int i = k + 1; i < 6; ++i) {
            double a = fabs(ck[i]);
            if (a > best) { best = a; piv = i; }
        }
        if (best == 0.0) ok = false;
#pragma unroll
        for (int i = k + 1; i < 6; ++i)
            if (piv == i) {
                double t = col[k]; col[k] = col[i]; col[i] = t;
                t = ck[k]; ck[k] = ck[i]; ck[i] = t;
            }
        const double inv = 1.0 / ck[k];
        col[k] *= inv;
#pragma unroll
        for (int i = 0; i < 6; ++i)
            if (i != k) col[i] -= ck[i] * col[k];
    }
    return ok;
}

}  // namespace lk
