// oracle/ref_leg/ref_leg_capi.cpp — TEST INFRASTRUCTURE ONLY.
//
// C entry point (ctypes) over the REFERENCE's own legkilo/src/preprocess/kinematics.cc, compiled unmodified by
// oracle/ref_leg/Makefile into oracle/_ref/liblkref_leg.so. One legkilo::Kinematics instance is driven over the whole
// sequence, from its initial state (every detector in contact). The redundancy drop lives in ROS code
// (RosInterface::kinematicImuCallBack, interface/ros1/ros_interface.cc:225-231, :247) that is not compiled here; the
// rule is restated below. Uses the product's POD structs (include/legkilo_b200.h) so tests hand both the same buffers.
#include <cstring>

#include <unitree_legged_msgs/HighState.h>

#include "preprocess/kinematics.h"

#include "../../include/legkilo_b200.h"

using namespace legkilo;

extern "C" {

// Returns the number of kept messages; track_out receives the detectors after the sequence (read back from the last
// kept output, which is what the detectors hold) and the z values of the last raw message.
uint32_t lkref_leg_kinematics(const lk_leg_cfg* c, const lk_leg_state* in, uint32_t n, int32_t redundancy,
                              lk_kinimu_meas* out, lk_leg_track* track_out) {
    Kinematics::Config cfg{c->leg_offset_x,     c->leg_offset_y,
                           c->leg_calf_length,  c->leg_thigh_length,
                           c->leg_thigh_offset, c->contact_force_threshold_up,
                           c->contact_force_threshold_down};
    Kinematics kin(cfg);
    unitree_legged_msgs::HighState last{};  // `static unitree_legged_msgs::HighState last_highstate_msg` (:222)
    int32_t contact[4] = {1, 1, 1, 1};
    uint32_t m = 0;
    for (uint32_t i = 0; i < n; ++i) {
        unitree_legged_msgs::HighState msg{};
        msg.stamp = ros::Time(in[i].stamp);
        for (int k = 0; k < 3; ++k) {
            msg.imu.accelerometer[k] = in[i].acc[k];
            msg.imu.gyroscope[k] = in[i].gyr[k];
        }
        for (int j = 0; j < 12; ++j) {
            msg.motorState[j].q = in[i].q[j];
            msg.motorState[j].dq = in[i].dq[j];
        }
        for (int k = 0; k < 4; ++k) msg.footForce[k] = in[i].foot_force[k];
        // ros_interface.cc:225-231: equal acc.z and gyr.z to the previous raw message -> drop, remember it anyway
        const bool drop = redundancy && msg.imu.accelerometer[2] == last.imu.accelerometer[2] &&
                          msg.imu.gyroscope[2] == last.imu.gyroscope[2];
        last = msg;
        if (drop) continue;
        common::KinImuMeas meas;
        kin.processing(msg, meas);
        lk_kinimu_meas& o = out[m++];
        o.stamp = meas.time_stamp_;
        std::memcpy(o.foot_pos, meas.foot_pos_, sizeof(o.foot_pos));
        std::memcpy(o.foot_vel, meas.foot_vel_, sizeof(o.foot_vel));
        for (int k = 0; k < 4; ++k) o.contact[k] = contact[k] = meas.contact_[k] ? 1 : 0;
        for (int k = 0; k < 3; ++k) {
            o.acc[k] = meas.acc_[k];
            o.gyr[k] = meas.gyr_[k];
        }
    }
    if (track_out) {
        for (int k = 0; k < 4; ++k) track_out->in_contact[k] = contact[k];
        track_out->last_acc_z = last.imu.accelerometer[2];
        track_out->last_gyr_z = last.imu.gyroscope[2];
    }
    return m;
}

}  // extern "C"
