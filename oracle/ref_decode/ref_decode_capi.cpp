// oracle/ref_decode/ref_decode_capi.cpp — TEST INFRASTRUCTURE ONLY.
//
// C entry point (ctypes) over the REFERENCE's own legkilo/src/preprocess/lidar_processing.cc, compiled unmodified by
// oracle/ref_decode/Makefile into oracle/_ref/liblkref_decode.so. Each call wraps the raw point bytes in a
// sensor_msgs::PointCloud2 whose fields are named as the driver publishes them (lidar_processing.h:20-71), with the given
// header stamp, and runs one LidarProcessing::processing on it. Uses the product's lk_pc2_layout (include/legkilo_b200.h)
// so tests hand both the same buffers.
#include <cmath>
#include <cstring>
#include <memory>

#include "preprocess/lidar_processing.h"

#include "../../include/legkilo_b200.h"

using namespace legkilo;

extern "C" {

// Returns the number of points kept; pts_out = float4 (x, y, z, curvature), intensity_out alongside, begin / end =
// lidar_begin_time_ / lidar_end_time_. An empty message is not handed to the reference (it reads front() of an empty
// cloud): it keeps no point and gets NaN times.
uint32_t lkref_decode_pointcloud2(const uint8_t* data, uint32_t n, const lk_pc2_layout* L, float blind, int32_t filter_num,
                                  double time_scale, double stamp, float* pts_out, float* intensity_out, double* begin_time,
                                  double* end_time) {
    if (!n) {
        *begin_time = *end_time = std::nan("");
        return 0;
    }
    auto msg = std::make_shared<sensor_msgs::PointCloud2>();
    msg->header.stamp = ros::Time(stamp);
    msg->height = 1;
    msg->width = n;
    msg->point_step = L->point_step;
    msg->row_step = n * L->point_step;
    using F = sensor_msgs::PointField;
    auto field = [&](const char* name, uint32_t off, uint8_t type) {
        F f;
        f.name = name;
        f.offset = off;
        f.datatype = type;
        msg->fields.push_back(f);
    };
    field("x", L->off_x, F::FLOAT32);
    field("y", L->off_y, F::FLOAT32);
    field("z", L->off_z, F::FLOAT32);
    field("intensity", L->off_intensity, F::FLOAT32);
    if (L->lidar_type == LK_LIDAR_VELODYNE) field("time", L->off_time, F::FLOAT32);
    else if (L->lidar_type == LK_LIDAR_OUSTER) field("t", L->off_time, F::UINT32);
    else field("timestamp", L->off_time, F::FLOAT64);
    msg->data.assign(data, data + (size_t)n * L->point_step);

    LidarProcessing::Config cfg;
    cfg.blind_ = blind;
    cfg.filter_num_ = filter_num;
    cfg.lidar_type_ = static_cast<common::LidarType>(L->lidar_type);
    cfg.time_scale_ = time_scale;
    LidarProcessing lp(cfg);
    common::LidarScan scan;
    const sensor_msgs::PointCloud2::ConstPtr cmsg = msg;
    lp.processing(cmsg, scan);

    const auto& pts = scan.cloud_->points;
    for (size_t i = 0; i < pts.size(); ++i) {
        pts_out[4 * i] = pts[i].x;
        pts_out[4 * i + 1] = pts[i].y;
        pts_out[4 * i + 2] = pts[i].z;
        pts_out[4 * i + 3] = pts[i].curvature;
        if (intensity_out) intensity_out[i] = pts[i].intensity;
    }
    *begin_time = scan.lidar_begin_time_;
    *end_time = scan.lidar_end_time_;
    return (uint32_t)pts.size();
}

}  // extern "C"
