// Stand-in for sensor_msgs/PointCloud2 (test infrastructure; see ../../../ref/shim/Eigen/Dense for the rationale): the
// message fields fromROSMsg reads.
#pragma once
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include <ros/ros.h>

namespace sensor_msgs {
struct PointField {
    enum { INT8 = 1, UINT8 = 2, INT16 = 3, UINT16 = 4, INT32 = 5, UINT32 = 6, FLOAT32 = 7, FLOAT64 = 8 };
    std::string name;
    uint32_t offset = 0;
    uint8_t datatype = 0;
    uint32_t count = 1;
};
struct PointCloud2 {
    std_msgs::Header header;
    uint32_t height = 1, width = 0;
    std::vector<PointField> fields;
    bool is_bigendian = false;
    uint32_t point_step = 0, row_step = 0;
    std::vector<uint8_t> data;
    bool is_dense = true;
    typedef std::shared_ptr<PointCloud2> Ptr;
    typedef std::shared_ptr<const PointCloud2> ConstPtr;
};
}  // namespace sensor_msgs
