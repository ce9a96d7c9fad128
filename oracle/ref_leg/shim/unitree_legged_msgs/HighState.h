// Stand-in for the generated unitree_legged_msgs/HighState.h: only the fields Kinematics::processing reads, with the
// types of unitree_legged_msgs/msg/{HighState,IMU,MotorState}.msg (fixed-size message arrays as plain arrays).
#pragma once
#include <cstdint>
#include <ros/ros.h>
namespace unitree_legged_msgs {
struct IMU { float gyroscope[3]; float accelerometer[3]; };
struct MotorState { float q; float dq; };
struct HighState {
    ros::Time stamp;
    IMU imu;
    MotorState motorState[20];
    int16_t footForce[4];
};
}  // namespace unitree_legged_msgs
