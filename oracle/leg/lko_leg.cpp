// oracle/leg/lko_leg.cpp — TEST INFRASTRUCTURE ONLY (see oracle/README.md).
//
// CPU restatement of the reference's leg-kinematics step, the input of the kinematic-inertial path: ContactDetector and
// Kinematics (legkilo/src/preprocess/kinematics.h:10-58, kinematics.cc:5-90) under the reference's names, written from
// their behaviour, and the redundancy drop of RosInterface::kinematicImuCallBack (interface/ros1/ros_interface.cc:
// 221-248). Pinned against the reference's own kinematics.cc (oracle/ref_leg/, tests/test_leg_kinematics.py) and the
// fixture tests/golden/ref_leg_kinematics.npz made from it. Kept apart from liblko.so: a library of its own, so the
// restatement of the hot path is untouched by it.
#include <cmath>
#include <cstdint>
#include <vector>

#include "../../include/legkilo_b200.h"

namespace lko_leg {

class ContactDetector {  // kinematics.h:10-23: hysteresis on the foot force, starts in contact
    double T_on_, T_off_;
    bool in_contact_ = true;

   public:
    ContactDetector(double ton, double toff) : T_on_(ton), T_off_(toff) {}
    // switch on above T_on_ while out of contact, off below T_off_ while in contact (kinematics.h:16-22)
    bool update(double val) {
        in_contact_ = in_contact_ ? !(val < T_off_) : (val > T_on_);
        return in_contact_;
    }
    // carried between calls (lk_leg_track); the reference keeps the detector alive instead
    bool state() const { return in_contact_; }
    void set_state(bool s) { in_contact_ = s; }
};

class Kinematics {  // kinematics.h:25-58
   public:
    explicit Kinematics(const lk_leg_cfg& c)
        : ox_(c.leg_offset_x), oy_(c.leg_offset_y), lc_(c.leg_calf_length), lt_(c.leg_thigh_length),
          d_(c.leg_thigh_offset),
          contacts_(4, ContactDetector(c.contact_force_threshold_up, c.contact_force_threshold_down)) {}

    // kinematics.cc:5-35 on the fields of HighState that lk_leg_state carries (message order, message types).
    // Leg k of the project (FR FL RR RL) is leg k ^ 1 of the message (FL FR RL RR): its footForce entry and its three
    // motorState entries (kinematics.cc:13-33).
    void processing(const lk_leg_state& msg, lk_kinimu_meas& out) {
        out.stamp = msg.stamp;
        for (int a = 0; a < 3; ++a) {
            out.acc[a] = (double)msg.acc[a];
            out.gyr[a] = (double)msg.gyr[a];
        }
        for (int k = 0; k < 4; ++k) {
            const int u = k ^ 1;
            out.contact[k] = contacts_[k].update((double)msg.foot_force[u]) ? 1 : 0;
            double q[3], dq[3];
            for (int a = 0; a < 3; ++a) {
                q[a] = (double)msg.q[3 * u + a];
                dq[a] = (double)msg.dq[3 * u + a];
            }
            caculateFootPosVel(k, q, dq, out.foot_pos[k], out.foot_vel[k]);
        }
    }

    // kinematics.cc:54-90 for one leg: hip roll q[0], thigh q[1], knee q[2]. Same operations in the same order as
    // the reference (left-to-right sums, no contraction: see Makefile).
    void caculateFootPosVel(int k, const double q[3], const double dq[3], double p[3], double v[3]) const {
        const double side = (k == 0 || k == 2) ? 1.0 : -1.0;  // lfoot
        const double fore = k < 2 ? 1.0 : -1.0;               // ffoot
        const double sr = std::sin(q[0]), cr = std::cos(q[0]);
        const double st = std::sin(q[1]), ct = std::cos(q[1]);
        const double sk = std::sin(q[1] + q[2]), ck = std::cos(q[1] + q[2]);
        const double sd = side * d_;

        p[0] = ((-lt_) * st - lc_ * sk) + fore * ox_;
        p[1] = ((sd * cr + lc_ * sr * ck) + lt_ * ct * sr) + side * oy_;
        p[2] = (sd * sr - lc_ * cr * ck) - lt_ * cr * ct;

        // Jacobian rows; its (0, 0) entry is zero and drops out of the sum
        const double J01 = (-lc_) * ck - lt_ * ct, J02 = (-lc_) * ck;
        const double J10 = (lt_ * cr * ct - sd * sr) + lc_ * cr * ck;
        const double J11 = (-sr) * (lc_ * sk + lt_ * st), J12 = (-lc_) * sk * sr;
        const double J20 = (lt_ * ct * sr + sd * cr) + lc_ * sr * ck;
        const double J21 = cr * (lc_ * sk + lt_ * st), J22 = lc_ * sk * cr;
        v[0] = J01 * dq[1] + J02 * dq[2];
        v[1] = (J10 * dq[0] + J11 * dq[1]) + J12 * dq[2];
        v[2] = (J20 * dq[0] + J21 * dq[1]) + J22 * dq[2];
    }

    double ox_, oy_, lc_, lt_, d_;
    std::vector<ContactDetector> contacts_;
};

}  // namespace lko_leg

extern "C" {

// lk_leg_kinematics on the CPU: kinematicImuCallBack's redundancy drop (ros_interface.cc:225-231, the previous raw
// message updated on both paths, :228 and :247) and Kinematics::processing of every kept message. Returns n_out.
uint32_t lko_leg_kinematics(const lk_leg_cfg* cfg, const lk_leg_state* in, uint32_t n, int32_t redundancy,
                            lk_leg_track* track, lk_kinimu_meas* out) {
    lko_leg::Kinematics kin(*cfg);
    for (int k = 0; k < 4; ++k) kin.contacts_[k].set_state(track->in_contact[k] != 0);
    float last_acc_z = track->last_acc_z, last_gyr_z = track->last_gyr_z;
    uint32_t m = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const bool drop = redundancy && in[i].acc[2] == last_acc_z && in[i].gyr[2] == last_gyr_z;
        last_acc_z = in[i].acc[2];
        last_gyr_z = in[i].gyr[2];
        if (drop) continue;
        kin.processing(in[i], out[m++]);
    }
    for (int k = 0; k < 4; ++k) track->in_contact[k] = kin.contacts_[k].state() ? 1 : 0;
    track->last_acc_z = last_acc_z;
    track->last_gyr_z = last_gyr_z;
    return m;
}

}  // extern "C"
