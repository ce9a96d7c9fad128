// lk_plane.cuh — warp-cooperative plane fit (VoxelOctoTree::init_plane, voxel_map.cc:42-117) and
// the octree initialisation / subdivision state machine (init_octo_tree :119-137, cut_octo_tree
// :139-183) shared by the bulk build and the incremental insert kernels.
//
// A leaf's retained points live in an HBM pool as 80-byte records (16-byte aligned so that a tile
// is one TMA bulk copy, cp.async.bulk global->shared completing on an mbarrier); a warp stages a
// tile in shared memory, reduces the moments with shuffles, every lane solves the same 3x3
// symmetric eigenproblem (Jacobi), and the 6x6 plane covariance is accumulated lane-parallel over
// the tile and shuffle-reduced.
#pragma once
#include "lk_async.cuh"
#include "lk_device.cuh"

namespace lk {

struct __align__(16) DevPoint {  // pointWithVar::point_w + var (voxel_map.h:59-78), padded to 80 B
    double pw[3];
    double var[6];  // xx xy xz yy yz zz
    double pad;
};

struct MapDev {
    HashSlot* slots;
    uint32_t hash_mask;
    MapNode* nodes;
    MapAux* aux;
    HotRec* hot;  // one per node (lk_device.cuh)
    DevPoint* points;
    uint32_t node_cap;
    unsigned long long point_cap;
    uint32_t* n_nodes;             // bump allocator of nodes
    unsigned long long* n_points;  // bump allocator of point slots
    uint32_t* n_roots;
    uint32_t* overflow;  // bit0 nodes, bit1 points, bit2 hash
    // Free lists of recycled storage (lk_octree.cuh: free_pop / free_push): standard point tiles (their first slot),
    // 8-node child groups (their first node) and single root nodes. free_ctr[3 l .. 3 l + 2] = avail | base | top of
    // list l: [0, avail) may be popped, pushes land at [top, ...), and the host promotes [base, top) between launches.
    uint32_t* free_items[3];
    uint32_t free_cap[3];
    uint32_t* free_ctr;
};

enum { FREE_TILES = 0, FREE_GROUPS = 1, FREE_SINGLES = 2 };
constexpr uint32_t NO_TILE = 0xffffffffu;  // aux.pts_base of a node whose tile went back to the free list

constexpr int TILE_PTS = 64;  // points per staged tile (5 120 B)

// ---- 3x3 symmetric eigen-decomposition (cyclic Jacobi), every lane redundantly -----------------
// C = {xx, xy, xz, yy, yz, zz}; returns eigenvalues w[3] and unit eigenvectors as columns of V.
__device__ inline void eig_sym3(const double* C, double* w, double* V) {
    double A[3][3] = {{C[0], C[1], C[2]}, {C[1], C[3], C[4]}, {C[2], C[4], C[5]}};
    double Q[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int sweep = 0; sweep < 32; ++sweep) {
        double off = fabs(A[0][1]) + fabs(A[0][2]) + fabs(A[1][2]);
        double diag = fabs(A[0][0]) + fabs(A[1][1]) + fabs(A[2][2]);
        if (off <= 1e-300 || off <= 1e-22 * diag) break;
#pragma unroll
        for (int p = 0; p < 2; ++p)
#pragma unroll
            for (int q = p + 1; q < 3; ++q) {
                if (A[p][q] == 0.0) continue;
                double theta = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
                double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    double akp = A[k][p], akq = A[k][q];
                    A[k][p] = c * akp - s * akq;
                    A[k][q] = s * akp + c * akq;
                }
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    double apk = A[p][k], aqk = A[q][k];
                    A[p][k] = c * apk - s * aqk;
                    A[q][k] = s * apk + c * aqk;
                }
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    double qkp = Q[k][p], qkq = Q[k][q];
                    Q[k][p] = c * qkp - s * qkq;
                    Q[k][q] = s * qkp + c * qkq;
                }
            }
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        w[i] = A[i][i];
        double n = sqrt(Q[0][i] * Q[0][i] + Q[1][i] * Q[1][i] + Q[2][i] * Q[2][i]);
#pragma unroll
        for (int k = 0; k < 3; ++k) V[k * 3 + i] = Q[k][i] / n;
    }
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Per-warp staging area.
struct __align__(16) WarpTile {
    DevPoint pts[TILE_PTS];
    uint64_t bar;
    uint32_t phase;
    uint32_t pad;
};

// Stage points [first, first+cnt) of `src` into the warp's tile through TMA.
__device__ __forceinline__ void tile_load(WarpTile* wt, const DevPoint* src, int cnt, int lane) {
    __syncwarp();
    if (lane == 0) {
        uint32_t bytes = (uint32_t)cnt * (uint32_t)sizeof(DevPoint);
        mbar_expect_tx(&wt->bar, bytes);
        bulk_g2s(wt->pts, src, bytes, &wt->bar);
    }
    __syncwarp();
    uint32_t ph = wt->phase;
    mbar_wait(&wt->bar, ph);
    __syncwarp();
    if (lane == 0) wt->phase = ph ^ 1u;
    __syncwarp();
}

// init_plane over `n` points at `src` (HBM, 16-B aligned). Writes the plane fields of `node`
// when it is a plane. Returns is_plane. All 32 lanes must call.
__device__ inline bool warp_fit_plane(WarpTile* wt, const DevPoint* src, int n, MapNode* node, float planer_threshold,
                                      int lane) {
    // ---- pass 1: centre and covariance  (voxel_map.cc:49-54) -----------------------------------
    double m[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) m[i] = 0.0;
    const bool single = n <= TILE_PTS;
    for (int t0 = 0; t0 < n; t0 += TILE_PTS) {
        int cnt = min(TILE_PTS, n - t0);
        tile_load(wt, src + t0, cnt, lane);
        for (int j = lane; j < cnt; j += 32) {
            const double x = wt->pts[j].pw[0], y = wt->pts[j].pw[1], z = wt->pts[j].pw[2];
            m[0] += x; m[1] += y; m[2] += z;
            m[3] += x * x; m[4] += x * y; m[5] += x * z; m[6] += y * y; m[7] += y * z; m[8] += z * z;
        }
    }
#pragma unroll
    for (int i = 0; i < 9; ++i) m[i] = warp_sum(m[i]);
    const double N = (double)n;
    const double cx = m[0] / N, cy = m[1] / N, cz = m[2] / N;
    double Cv[6] = {m[3] / N - cx * cx, m[4] / N - cx * cy, m[5] / N - cx * cz,
                    m[6] / N - cy * cy, m[7] / N - cy * cz, m[8] / N - cz * cz};
    double w[3], V[9];
    eig_sym3(Cv, w, V);
    int imin = 0, imax = 0;  // first extremum, as minCoeff / maxCoeff (voxel_map.cc:60-61)
    if (w[1] < w[imin]) imin = 1;
    if (w[2] < w[imin]) imin = 2;
    if (w[1] > w[imax]) imax = 1;
    if (w[2] > w[imax]) imax = 2;
    if (!(w[imin] < (double)planer_threshold)) return false;

    // ---- pass 2: plane covariance  (voxel_map.cc:74-92) -----------------------------------------
    // J_i = [E F_i ; I/N], E F_i = sum_{m != min} a_m e_m [ (d.e_m) e_min + (d.e_min) e_m ]^T,
    // a_m = 1 / (N (l_min - l_m)), d = p_i - c.
    double emin[3] = {V[0 * 3 + imin], V[1 * 3 + imin], V[2 * 3 + imin]};
    double acc[21];
#pragma unroll
    for (int i = 0; i < 21; ++i) acc[i] = 0.0;
    const double invN = 1.0 / N;
    for (int t0 = 0; t0 < n; t0 += TILE_PTS) {
        int cnt = min(TILE_PTS, n - t0);
        if (!single) tile_load(wt, src + t0, cnt, lane);
        for (int j = lane; j < cnt; j += 32) {
            const DevPoint& p = wt->pts[j];
            const double dx = p.pw[0] - cx, dy = p.pw[1] - cy, dz = p.pw[2] - cz;
            const double dmin = dx * emin[0] + dy * emin[1] + dz * emin[2];
            double G[9];
#pragma unroll
            for (int i = 0; i < 9; ++i) G[i] = 0.0;
#pragma unroll
            for (int mm = 0; mm < 3; ++mm) {
                if (mm == imin) continue;
                const double em[3] = {V[0 * 3 + mm], V[1 * 3 + mm], V[2 * 3 + mm]};
                const double a = 1.0 / (N * (w[imin] - w[mm]));
                const double dm = dx * em[0] + dy * em[1] + dz * em[2];
                double row[3];
#pragma unroll
                for (int k = 0; k < 3; ++k) row[k] = a * (dm * emin[k] + dmin * em[k]);
#pragma unroll
                for (int r = 0; r < 3; ++r)
#pragma unroll
                    for (int k = 0; k < 3; ++k) G[r * 3 + k] += em[r] * row[k];
            }
            const double S[9] = {p.var[0], p.var[1], p.var[2], p.var[1], p.var[3], p.var[4], p.var[2], p.var[4], p.var[5]};
            double GS[9];
            mat3_mul(G, S, GS);
            // upper triangle of [[G S G^T, G S / N], [.., S / N^2]]
            int q = 0;
#pragma unroll
            for (int r = 0; r < 3; ++r) {
#pragma unroll
                for (int c = r; c < 3; ++c) acc[q++] += GS[r * 3] * G[c * 3] + GS[r * 3 + 1] * G[c * 3 + 1] + GS[r * 3 + 2] * G[c * 3 + 2];
#pragma unroll
                for (int c = 0; c < 3; ++c) acc[q++] += GS[r * 3 + c] * invN;
            }
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
                for (int c = r; c < 3; ++c) acc[q++] += S[r * 3 + c] * invN * invN;
        }
    }
#pragma unroll
    for (int i = 0; i < 21; ++i) acc[i] = warp_sum(acc[i]);
    if (lane == 0) {
        node->center[0] = cx; node->center[1] = cy; node->center[2] = cz;
        node->normal[0] = emin[0]; node->normal[1] = emin[1]; node->normal[2] = emin[2];
#pragma unroll
        for (int i = 0; i < 21; ++i) node->plane_var[i] = acc[i];
        node->radius = (float)sqrt(w[imax]);
        node->d = (float)(-(emin[0] * cx + emin[1] * cy + emin[2] * cz));
    }
    return true;
}

}  // namespace lk
