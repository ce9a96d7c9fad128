// lk_device.cuh — device-side types and small dense math shared by the kernels of the
// H100-native Leg-KILO LiDAR update path. sm_90a only; fp64 throughout with the reference's
// float temporaries reproduced where they decide something (SURVEY.md §8a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/legkilo_b200.h"

namespace lk {

// ---- map in HBM --------------------------------------------------------------------------
// Open-addressed table of root voxels: 16-byte slots, linear probing, empty <=> node < 0.
struct __align__(16) HashSlot {
    int kx, ky, kz;
    int node;
};

__host__ __device__ __forceinline__ uint32_t hash_key(int x, int y, int z) {
    uint32_t h = (uint32_t)x * 73856093u ^ (uint32_t)y * 19349669u ^ (uint32_t)z * 83492791u;
    h ^= h >> 15;
    h *= 0x2c1b3c6du;
    h ^= h >> 12;
    h *= 0x297a2d39u;
    h ^= h >> 15;
    return h;
}

typedef lk_map_node MapNode;   // 256 B, first 232 B are what the residual kernel reads
typedef lk_map_aux MapAux;     // 64 B
typedef lk_map_point MapPoint; // 72 B

// Hot image of a plane, 160-byte stride (five 32-byte sectors, 144 bytes used): what the throughput kernel gathers per
// point instead of the 256-byte node record. With J = [a, -n], a = pw - c:
//     J Sigma_plane J^T = a^T Scc a - 2 a^T (Scn n) + n^T Snn n = a^T Scc a - 2 a^T v + s,
// so the 21 covariance terms collapse to Scc (6), v = Scn n (3) and s = n^T Snn n (1), which do not depend on the point.
// radius < 0 <=> the node holds no plane (the kernel then takes the full reference sequence on the node records).
struct __align__(32) HotRec {
    double c[3], n[3];
    double scc[6];  // xx xy xz yy yz zz of the centre block of plane_var
    double v[3];
    double s;
    float d, radius;
    uint32_t pad[6];
};
static_assert(sizeof(HotRec) == 160, "hot record stride");

__host__ __device__ inline void hot_fill(const lk_map_node& nd, HotRec& h) {  // nd holds a plane
    const double* pv = nd.plane_var;  // upper triangle, row-major: row r starts at r*6 - r(r-1)/2
    const double n0 = nd.normal[0], n1 = nd.normal[1], n2 = nd.normal[2];
    for (int i = 0; i < 3; ++i) { h.c[i] = nd.center[i]; h.n[i] = nd.normal[i]; }
    h.scc[0] = pv[0]; h.scc[1] = pv[1]; h.scc[2] = pv[2]; h.scc[3] = pv[6]; h.scc[4] = pv[7]; h.scc[5] = pv[11];
    // Scn rows: (0,3..5) = pv[3..5], (1,3..5) = pv[8..10], (2,3..5) = pv[12..14]
    h.v[0] = pv[3] * n0 + pv[4] * n1 + pv[5] * n2;
    h.v[1] = pv[8] * n0 + pv[9] * n1 + pv[10] * n2;
    h.v[2] = pv[12] * n0 + pv[13] * n1 + pv[14] * n2;
    // Snn: (3,3) pv[15] (3,4) pv[16] (3,5) pv[17] (4,4) pv[18] (4,5) pv[19] (5,5) pv[20]
    h.s = pv[15] * n0 * n0 + pv[18] * n1 * n1 + pv[20] * n2 * n2 + 2.0 * (pv[16] * n0 * n1 + pv[17] * n0 * n2 + pv[19] * n1 * n2);
    h.d = nd.d;
    h.radius = nd.radius;
}
__host__ __device__ inline void hot_from_node(const lk_map_node& nd, HotRec& h) {
    if (nd.flags & LK_NODE_IS_PLANE) hot_fill(nd, h);
    else h.radius = -1.0f;
}

struct MapView {  // what the residual path reads of the map
    const HashSlot* slots;
    uint32_t hash_mask;
    const MapNode* nodes;  // full records: the octree descent below a root that holds no plane
    const HotRec* hot;     // plane images of the nodes: what the per-point passes gather
};

// ---- per-call constants (kernel parameter space) ------------------------------------------
struct Globals {
    double Re[9];      // extrinsic rotation  (KILO::ext_rot_)
    double te[3];      // extrinsic translation
    double voxel;      // max_voxel_size_ as double (KILO.cc:145)
    double inv_voxel;  // exact reciprocal when voxel is a power of two, else unused
    double sigma_num;
    double ratio;      // lidar_point_meas_ratio
    double dv;         // sin(DEG2RAD(beam_err))^2 with PCL's DEG2RAD constant (voxel_map.cc:27)
    float voxel_f;     // (float)max_voxel_size_ (voxel_map.cc:289,337)
    float rv;          // range_inc*range_inc in float (voxel_map.cc:25)
    float planer_threshold;  // (float)min_eigen_value
    int voxel_pow2;
    int max_layer;
    int max_points_num;
    int layer_init_num[5];
};

// What every residual thread needs of one scan's filter at the current linearisation point.
struct ScanConst {
    double R[9];    // rot
    double p[3];    // pos
    double Pth[6];  // sym(P[0:3,0:3]) upper: xx xy xz yy yz zz
    double Ppp[6];  // sym(P[3:6,3:6]) upper
};

// The ScanConst of a pose given without a filter (lk_map_insert, lk_score_poses), as scan_const_from fills it from one: R, p
// and the symmetric parts of the theta / position blocks of P (row-major 3 x 3 each).
inline void scan_const_at(const double* R, const double* p, const double* Pt, const double* Pp, ScanConst& sc) {
    for (int i = 0; i < 9; ++i) sc.R[i] = R[i];
    for (int i = 0; i < 3; ++i) sc.p[i] = p[i];
    const int ut[6][2] = {{0, 0}, {0, 1}, {0, 2}, {1, 1}, {1, 2}, {2, 2}};
    for (int q = 0; q < 6; ++q) {
        const int i = ut[q][0], j = ut[q][1];
        sc.Pth[q] = 0.5 * (Pt[i * 3 + j] + Pt[j * 3 + i]);
        sc.Ppp[q] = 0.5 * (Pp[i * 3 + j] + Pp[j * 3 + i]);
    }
}

// The block's copy of one scan's constants, one double per thread; the caller synchronises before reading it.
__device__ __forceinline__ void load_scan_const(ScanConst* dst, const ScanConst* src) {
    const int tid = threadIdx.x;
    if (tid < (int)(sizeof(ScanConst) / sizeof(double)))
        reinterpret_cast<double*>(dst)[tid] = reinterpret_cast<const double*>(src)[tid];
}

// 32 doubles per chunk partial: A upper (21) | b (6) | sumR | count | pad
constexpr int NACC = 29;
constexpr int ACC_B = 21, ACC_SUMR = 27, ACC_CNT = 28;
constexpr int PARTIAL_STRIDE = 32;

struct ChunkDesc {
    uint32_t scan;   // scan index in the batch
    uint32_t start;  // first point (absolute)
    uint32_t count;  // points in this chunk
    uint32_t pad;
};

// Per-scan bookkeeping of the current bucket step.
struct ScanStep {
    uint32_t chunk_begin, chunk_end;  // chunks of this scan's current bucket
    uint32_t pt_begin, pt_end;        // point range of the current bucket
    double t_bucket;
    uint32_t active;  // 0 => scan has no bucket in this step
    uint32_t updated; // any iteration of this bucket produced an update
    uint32_t n_eff_last;  // residual count of the most recent iteration
    uint32_t pad;
};

// ---- tiny dense helpers ----------------------------------------------------------------------
__device__ __forceinline__ void mat3_mul(const double* A, const double* B, double* C) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) C[i * 3 + j] = A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j] + A[i * 3 + 2] * B[6 + j];
}

// math_utils.hpp:55-68 — Exp(v1,v2,v3) with the reference's 1e-5 identity threshold.
__device__ __forceinline__ void so3_exp3(double v1, double v2, double v3, double* E) {
    double norm = sqrt(v1 * v1 + v2 * v2 + v3 * v3);
    E[0] = 1; E[1] = 0; E[2] = 0; E[3] = 0; E[4] = 1; E[5] = 0; E[6] = 0; E[7] = 0; E[8] = 1;
    if (norm > 0.00001) {
        double kx = v1 / norm, ky = v2 / norm, kz = v3 / norm;
        double s, c;
        sincos(norm, &s, &c);
        double c1 = 1.0 - c;
        double K[9] = {0, -kz, ky, kz, 0, -kx, -ky, kx, 0};
        double K2[9];
        mat3_mul(K, K, K2);
#pragma unroll
        for (int i = 0; i < 9; ++i) E[i] += s * K[i] + c1 * K2[i];
    }
}

// math_utils.hpp:20-32 — Exp(vec) with the 1e-7 threshold (used by getFx).
__device__ __forceinline__ void so3_exp_vec(double v1, double v2, double v3, double* E) {
    double norm = sqrt(v1 * v1 + v2 * v2 + v3 * v3);
    E[0] = 1; E[1] = 0; E[2] = 0; E[3] = 0; E[4] = 1; E[5] = 0; E[6] = 0; E[7] = 0; E[8] = 1;
    if (norm > 0.0000001) {
        double kx = v1 / norm, ky = v2 / norm, kz = v3 / norm;
        double s, c;
        sincos(norm, &s, &c);
        double c1 = 1.0 - c;
        double K[9] = {0, -kz, ky, kz, 0, -kx, -ky, kx, 0};
        double K2[9];
        mat3_mul(K, K, K2);
#pragma unroll
        for (int i = 0; i < 9; ++i) E[i] += s * K[i] + c1 * K2[i];
    }
}

// State::operator+= (eskf.cc:18-29) on the 36-double lk_state layout.
__device__ __forceinline__ void state_boxplus(double* x36, const double* d30) {
    double E[9], Rn[9];
    so3_exp3(d30[0], d30[1], d30[2], E);
    mat3_mul(x36, E, Rn);
#pragma unroll
    for (int i = 0; i < 9; ++i) x36[i] = Rn[i];
#pragma unroll
    for (int i = 0; i < 27; ++i) x36[9 + i] += d30[3 + i];
}

// In-place LU with partial pivoting of an n x n system with m right-hand sides (n <= 18).
// M is n x n row-major (stride n), B is n x m row-major. Single thread.
template <int MAXN>
__device__ inline bool lu_solve_small(double* M, double* B, int n, int m) {
    for (int k = 0; k < n; ++k) {
        int piv = k;
        double best = fabs(M[k * n + k]);
        for (int i = k + 1; i < n; ++i) {
            double v = fabs(M[i * n + k]);
            if (v > best) { best = v; piv = i; }
        }
        if (best == 0.0) return false;
        if (piv != k) {
            for (int j = 0; j < n; ++j) { double t = M[k * n + j]; M[k * n + j] = M[piv * n + j]; M[piv * n + j] = t; }
            for (int j = 0; j < m; ++j) { double t = B[k * m + j]; B[k * m + j] = B[piv * m + j]; B[piv * m + j] = t; }
        }
        double inv = 1.0 / M[k * n + k];
        for (int i = k + 1; i < n; ++i) {
            double l = M[i * n + k] * inv;
            if (l != 0.0) {
                for (int j = k + 1; j < n; ++j) M[i * n + j] -= l * M[k * n + j];
                for (int j = 0; j < m; ++j) B[i * m + j] -= l * B[k * m + j];
            }
        }
    }
    for (int i = n - 1; i >= 0; --i) {
        double inv = 1.0 / M[i * n + i];
        for (int j = 0; j < m; ++j) {
            double s = B[i * m + j];
            for (int k = i + 1; k < n; ++k) s -= M[i * n + k] * B[k * m + j];
            B[i * m + j] = s * inv;
        }
    }
    return true;
}

}  // namespace lk
