// lk_insert.cuh — the device pieces of VoxelMapManager::UpdateVoxelMap (voxel_map.cc:336-361) shared by the insert
// kernels (lk_insert.cu) and the persistent per-scan kernel (lk_fused.cu), so that both build bit-identical maps:
//   * the inserted point: world position and covariance with the UPDATED state (KILO.cc:216-228);
//   * find-or-create of the root voxel (CAS on the open-addressed table);
//   * one warp applying UpdateOctoTree to the points of ONE root in their index order (the reference's insertion order).
#pragma once
#include "lk_octree.cuh"

namespace lk {

__device__ __forceinline__ int hash_find_or_create(MapDev& md, const Globals& g, int kx, int ky, int kz) {
    uint32_t i = hash_key(kx, ky, kz) & md.hash_mask;
    for (uint32_t probe = 0; probe <= md.hash_mask; ++probe) {
        int* nodep = &md.slots[i].node;
        int node = *(volatile int*)nodep;
        if (node == -1) {
            int old = atomicCAS(nodep, -1, -2);
            if (old == -1) {
                md.slots[i].kx = kx; md.slots[i].ky = ky; md.slots[i].kz = kz;
                uint32_t nd;
                if (!free_pop(md, FREE_SINGLES, nd)) nd = atomicAdd(md.n_nodes, 1u);  // a slid-out root's node first
                if (nd >= md.node_cap) {
                    atomicOr(md.overflow, 1u);
                    __threadfence();
                    atomicExch(nodep, -3);  // poisoned slot: key present, no node
                    return -1;
                }
                init_root_node(md, g, nd, kx, ky, kz);
                atomicAdd(md.n_roots, 1u);
                __threadfence();
                atomicExch(nodep, (int)nd);
                return (int)nd;
            }
            node = old;
        }
        for (uint32_t spins = 0; node == -2; ++spins) {  // another thread is publishing this slot
            node = *(volatile int*)nodep;
            if (spins > (1u << 26)) { stall_note(2u, i); return -1; }
        }
        __threadfence();
        const int sx = *(volatile int*)&md.slots[i].kx, sy = *(volatile int*)&md.slots[i].ky, sz = *(volatile int*)&md.slots[i].kz;
        if (sx == kx && sy == ky && sz == kz) return node >= 0 ? node : -1;
        i = (i + 1) & md.hash_mask;
    }
    atomicOr(md.overflow, 4u);
    return -1;
}

// pointWithVar of one bucket point after the update (KILO.cc:218-228): pw = R pi + p, var = M Sigma_b M^T + G P_tt G^T + P_pp
// with M = R Re, G = R [pi]x. (bx, by, bz) = the LiDAR-frame point as calcBodyCov saw it (z == 0 -> 1e-4).
__device__ __forceinline__ void make_insert_point(double pix, double piy, double piz, double bx, double by, double bz,
                                                  const ScanConst& sc, const Globals& g, DevPoint& p) {
    const double* R = sc.R;
    p.pw[0] = R[0] * pix + R[1] * piy + R[2] * piz + sc.p[0];
    p.pw[1] = R[3] * pix + R[4] * piy + R[5] * piz + sc.p[1];
    p.pw[2] = R[6] * pix + R[7] * piy + R[8] * piz + sc.p[2];
    const double r2 = bx * bx + by * by + bz * bz;
    const float range = (float)sqrt(r2);
    const double range2 = (double)range * (double)range;
    const double inv = 1.0 / sqrt(r2);
    const double ux = bx * inv, uy = by * inv, uz = bz * inv;
    // M = R Re ; mu = M u
    double M[9];
    mat3_mul(R, g.Re, M);
    const double mu[3] = {M[0] * ux + M[1] * uy + M[2] * uz, M[3] * ux + M[4] * uy + M[5] * uz, M[6] * ux + M[7] * uy + M[8] * uz};
    double MMt[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) MMt[r * 3 + c] = M[r * 3] * M[c * 3] + M[r * 3 + 1] * M[c * 3 + 1] + M[r * 3 + 2] * M[c * 3 + 2];
    const double ca = (double)g.rv - range2 * g.dv, cb = range2 * g.dv;
    // G = R [pi]x ; G P_tt G^T
    const double K[9] = {0, -piz, piy, piz, 0, -pix, -piy, pix, 0};
    double G[9], GP[9];
    mat3_mul(R, K, G);
    const double* S = sc.Pth;
    const double Pt[9] = {S[0], S[1], S[2], S[1], S[3], S[4], S[2], S[4], S[5]};
    mat3_mul(G, Pt, GP);
    const double* Sp = sc.Ppp;
    const double Pp[9] = {Sp[0], Sp[1], Sp[2], Sp[1], Sp[3], Sp[4], Sp[2], Sp[4], Sp[5]};
    const int ut[6][2] = {{0, 0}, {0, 1}, {0, 2}, {1, 1}, {1, 2}, {2, 2}};
#pragma unroll
    for (int q = 0; q < 6; ++q) {
        const int r = ut[q][0], c = ut[q][1];
        p.var[q] = ca * mu[r] * mu[c] + cb * MMt[r * 3 + c] + (GP[r * 3] * G[c * 3] + GP[r * 3 + 1] * G[c * 3 + 1] + GP[r * 3 + 2] * G[c * 3 + 2]) +
                   Pp[r * 3 + c];
    }
    p.pad = 0.0;
}

// voxelKeyFloor(point_w, (double)(float)voxel_size) (voxel_map.cc:337,343), find-or-create the root, count the point on it;
// the first point of a root registers it in `touched`. Returns the root node (-1 = dropped: pools exhausted).
__device__ __forceinline__ int insert_register_point(MapDev& md, const Globals& g, const DevPoint& p, int* pend, uint32_t* touched,
                                                     uint32_t* n_touched) {
    const double vs = (double)g.voxel_f;
    const int kx = (int)floor(p.pw[0] / vs), ky = (int)floor(p.pw[1] / vs), kz = (int)floor(p.pw[2] / vs);
    const int root = hash_find_or_create(md, g, kx, ky, kz);
    if (root >= 0) {
        const int c = atomicAdd(&pend[root * 3], 1);
        if (c == 0) touched[atomicAdd(n_touched, 1u)] = (uint32_t)root;
    }
    return root;
}

// One warp, one touched root: walk the bucket's root-per-point array in index order (= the order UpdateVoxelMap walks
// input_points) and insert the root's own points. iroot / ipts are read through L2 (they were written by other blocks).
__device__ __forceinline__ void warp_insert_root_scan(MapDev& md, const Globals& g, WarpTile* wt, uint32_t root, const int* iroot,
                                                      const DevPoint* ipts, uint32_t n_pts, int* pend, int lane) {
    const int cnt = __ldcg(&pend[root * 3]);
    int done = 0;
    for (uint32_t base = 0; base < n_pts && done < cnt; base += 32) {
        const uint32_t j = base + (uint32_t)lane;
        const int r = j < n_pts ? __ldcg(iroot + j) : -1;
        uint32_t m = __ballot_sync(0xffffffffu, r == (int)root);
        while (m) {
            const int b = __ffs(m) - 1;
            m &= m - 1;
            DevPoint p;
            const double2* s2 = reinterpret_cast<const double2*>(ipts + base + (uint32_t)b);
            double2* d2 = reinterpret_cast<double2*>(&p);
#pragma unroll
            for (int q = 0; q < 5; ++q) d2[q] = __ldcg(s2 + q);
            warp_update_octo_tree(md, g, wt, root, p, lane);
            ++done;
        }
    }
    __syncwarp();
    if (lane == 0) pend[root * 3] = 0;
}

}  // namespace lk
