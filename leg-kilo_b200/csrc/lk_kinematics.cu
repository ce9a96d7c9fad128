// lk_kinematics.cu — leg states to kinematic-inertial samples on the device (lk_leg_kinematics):
//   * the redundancy drop of RosInterface::kinematicImuCallBack (legkilo/src/interface/ros1/ros_interface.cc:225-231),
//   * the four ContactDetectors of Kinematics (legkilo/src/preprocess/kinematics.h:10-23, kinematics.cc:17-20),
//   * forward kinematics and foot velocity (caculateFootPosVel, kinematics.cc:54-90) with the leg remap (:13-33).
// The shape is decode_pointcloud2_device's: flags, device-wide scans, scatter. The detectors are sequential, but a
// detector is a map bool -> bool fixed by the force alone, and those four maps form a monoid under composition, so the
// state in front of every message is an inclusive scan of the per-message maps applied to the carried-in state.
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <string>

#include "lk_device.cuh"
#include "lk_host.h"

namespace lk {

namespace {

// A detector map is 2 bits, (f(false), f(true)) in bits (0, 1); four legs (FR FL RR RL) pack into one byte.
constexpr uint8_t kLegIdentity = 0xAA;  // f(s) = s on every leg

__host__ __device__ __forceinline__ int leg_apply(uint8_t code, int leg, int s) { return (code >> (2 * leg + s)) & 1; }

// (b o a): a first, then b. Associative, not commutative; CUB keeps the operands in sequence order.
struct LegCompose {
    __host__ __device__ __forceinline__ uint8_t operator()(uint8_t a, uint8_t b) const {
        uint8_t r = 0;
        for (int leg = 0; leg < 4; ++leg)
            for (int s = 0; s < 2; ++s) r |= (uint8_t)(leg_apply(b, leg, leg_apply(a, leg, s)) << (2 * leg + s));
        return r;
    }
};

// project leg (FR FL RR RL) -> message leg (FL FR RL RR), the footForce index and motorState index / 3
// (kinematics.cc:17-33): the legs swap in pairs
__host__ __device__ __forceinline__ int msg_leg(int leg) { return leg ^ 1; }

__global__ void k_leg_flags(const lk_leg_state* __restrict__ in, uint32_t n, int redundancy, float acc_z0, float gyr_z0,
                            double up, double down, uint32_t* __restrict__ keep, uint8_t* __restrict__ code) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float az = in[i].acc[2], gz = in[i].gyr[2];
    const float paz = i ? in[i - 1].acc[2] : acc_z0, pgz = i ? in[i - 1].gyr[2] : gyr_z0;
    const bool k = !redundancy || !(az == paz && gz == pgz);  // ros_interface.cc:226-227 (float ==)
    keep[i] = k ? 1u : 0u;
    uint8_t c = kLegIdentity;
    if (k) {
        c = 0;
#pragma unroll
        for (int leg = 0; leg < 4; ++leg) {
            const double val = (double)in[i].foot_force[msg_leg(leg)];
            const int off = val > up ? 1 : 0;      // !in_contact_ && val > T_on_  -> true
            const int on = (val < down) ? 0 : 1;   //  in_contact_ && val < T_off_ -> false
            c |= (uint8_t)((off | (on << 1)) << (2 * leg));
        }
    }
    code[i] = c;
}

struct LegResult {
    uint32_t n_out;
    int32_t in_contact[4];
    float last_acc_z, last_gyr_z;
};

__global__ void k_leg_scatter(const lk_leg_state* __restrict__ in, uint32_t n, lk_leg_cfg cfg, int4 contact0,
                              const uint32_t* __restrict__ keep, const uint32_t* __restrict__ pos,
                              const uint8_t* __restrict__ scode, lk_kinimu_meas* __restrict__ out, LegResult* res) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int c0[4] = {contact0.x, contact0.y, contact0.z, contact0.w};
    if (i == n - 1) {  // the new track: the detectors after the last message, the last raw message's z values
        res->n_out = pos[i] + keep[i];
#pragma unroll
        for (int leg = 0; leg < 4; ++leg) res->in_contact[leg] = leg_apply(scode[i], leg, c0[leg]);
        res->last_acc_z = in[i].acc[2];
        res->last_gyr_z = in[i].gyr[2];
    }
    if (!keep[i]) return;
    const lk_leg_state& m = in[i];
    lk_kinimu_meas o;
    o.stamp = m.stamp;
    for (int k = 0; k < 3; ++k) { o.acc[k] = (double)m.acc[k]; o.gyr[k] = (double)m.gyr[k]; }
    const uint8_t sc = scode[i];
    const double ox = cfg.leg_offset_x, oy = cfg.leg_offset_y, lc = cfg.leg_calf_length, lt = cfg.leg_thigh_length,
                 d = cfg.leg_thigh_offset;
#pragma unroll
    for (int leg = 0; leg < 4; ++leg) {
        o.contact[leg] = leg_apply(sc, leg, c0[leg]);
        const int j = 3 * msg_leg(leg);
        const double a0 = (double)m.q[j], a1 = (double)m.q[j + 1], a2 = (double)m.q[j + 2];
        const double v0 = (double)m.dq[j], v1 = (double)m.dq[j + 1], v2 = (double)m.dq[j + 2];
        const int lfoot = (leg == 0 || leg == 2) ? 1 : -1, ffoot = leg < 2 ? 1 : -1;
        const double s1 = sin(a0), s2 = sin(a1), s23 = sin(a1 + a2);
        const double c1 = cos(a0), c2 = cos(a1), c23 = cos(a1 + a2);
        o.foot_pos[leg][0] = -lt * s2 - lc * s23 + ffoot * ox;
        o.foot_pos[leg][1] = lfoot * d * c1 + lc * s1 * c23 + lt * c2 * s1 + lfoot * oy;
        o.foot_pos[leg][2] = lfoot * d * s1 - lc * c1 * c23 - lt * c1 * c2;
        const double j01 = -lc * c23 - lt * c2, j02 = -lc * c23;
        const double j10 = lt * c1 * c2 - lfoot * d * s1 + lc * c1 * c23, j11 = -s1 * (lc * s23 + lt * s2),
                     j12 = -lc * s23 * s1;
        const double j20 = lt * c2 * s1 + lfoot * d * c1 + lc * s1 * c23, j21 = c1 * (lc * s23 + lt * s2),
                     j22 = lc * s23 * c1;
        o.foot_vel[leg][0] = j01 * v1 + j02 * v2;
        o.foot_vel[leg][1] = j10 * v0 + j11 * v1 + j12 * v2;
        o.foot_vel[leg][2] = j20 * v0 + j21 * v1 + j22 * v2;
    }
    out[pos[i]] = o;
}

size_t align_up(size_t b) { return (b + 255) & ~size_t(255); }

struct LegScratch {  // one device block, carved in this order
    size_t in, keep, pos, code, scode, out, res, tmp, total;
    explicit LegScratch(uint32_t n) {
        size_t t1 = 0, t2 = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, t1, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n);
        cub::DeviceScan::InclusiveScan(nullptr, t2, (const uint8_t*)nullptr, (uint8_t*)nullptr, LegCompose(), (int)n);
        size_t o = 0;
        in = o; o += align_up((size_t)n * sizeof(lk_leg_state));
        keep = o; o += align_up((size_t)n * 4);
        pos = o; o += align_up((size_t)n * 4);
        code = o; o += align_up(n);
        scode = o; o += align_up(n);
        out = o; o += align_up((size_t)n * sizeof(lk_kinimu_meas));
        res = o; o += align_up(sizeof(LegResult));
        tmp = o; o += align_up(std::max(t1, t2));
        total = o;
    }
};

}  // namespace

size_t leg_kinematics_scratch_bytes(uint32_t n) { return n ? LegScratch(n).total : 0; }

// `scratch` holds leg_kinematics_scratch_bytes(n) bytes of device memory. n > 0.
int leg_kinematics_device(const lk_leg_cfg& cfg, const lk_leg_state* h_in, uint32_t n, int redundancy,
                          lk_leg_track* track, lk_kinimu_meas* h_out, uint32_t* n_out, void* scratch, cudaStream_t s,
                          std::string& err) {
    const LegScratch L(n);
    char* base = static_cast<char*>(scratch);
    auto* d_in = reinterpret_cast<lk_leg_state*>(base + L.in);
    auto* d_keep = reinterpret_cast<uint32_t*>(base + L.keep);
    auto* d_pos = reinterpret_cast<uint32_t*>(base + L.pos);
    auto* d_code = reinterpret_cast<uint8_t*>(base + L.code);
    auto* d_scode = reinterpret_cast<uint8_t*>(base + L.scode);
    auto* d_out = reinterpret_cast<lk_kinimu_meas*>(base + L.out);
    auto* d_res = reinterpret_cast<LegResult*>(base + L.res);
    void* d_tmp = base + L.tmp;
    size_t tb = L.total - L.tmp;
    LK_CUDA(err, cudaMemcpyAsync(d_in, h_in, (size_t)n * sizeof(lk_leg_state), cudaMemcpyHostToDevice, s));
    const unsigned g = (n + 255) / 256;
    k_leg_flags<<<g, 256, 0, s>>>(d_in, n, redundancy, track->last_acc_z, track->last_gyr_z,
                                  cfg.contact_force_threshold_up, cfg.contact_force_threshold_down, d_keep, d_code);
    LK_CUDA(err, cub::DeviceScan::ExclusiveSum(d_tmp, tb, d_keep, d_pos, (int)n, s));
    tb = L.total - L.tmp;
    LK_CUDA(err, cub::DeviceScan::InclusiveScan(d_tmp, tb, d_code, d_scode, LegCompose(), (int)n, s));
    const int4 c0 = make_int4(track->in_contact[0] != 0, track->in_contact[1] != 0, track->in_contact[2] != 0,
                              track->in_contact[3] != 0);
    k_leg_scatter<<<g, 256, 0, s>>>(d_in, n, cfg, c0, d_keep, d_pos, d_scode, d_out, d_res);
    LK_CUDA(err, cudaGetLastError());
    LegResult r;
    LK_CUDA(err, cudaMemcpyAsync(&r, d_res, sizeof(r), cudaMemcpyDeviceToHost, s));
    LK_CUDA(err, cudaStreamSynchronize(s));
    if (r.n_out)
        LK_CUDA(err, cudaMemcpyAsync(h_out, d_out, (size_t)r.n_out * sizeof(lk_kinimu_meas), cudaMemcpyDeviceToHost, s));
    LK_CUDA(err, cudaStreamSynchronize(s));
    *n_out = r.n_out;
    for (int leg = 0; leg < 4; ++leg) track->in_contact[leg] = r.in_contact[leg];
    track->last_acc_z = r.last_acc_z;
    track->last_gyr_z = r.last_gyr_z;
    return LK_OK;
}

}  // namespace lk
