// Stand-in for pcl_conversions::fromROSMsg and for the point-registration macros the driver point structs of
// preprocess/lidar_processing.h use (test infrastructure; see ../../../ref/shim/Eigen/Dense for the rationale).
// lidar_processing.h includes this header before it declares those structs, so the macros are defined here rather than
// in the shared stand-ins of pcl/point_types.h and Eigen.
//
// fromROSMsg resolves every registered field BY NAME among the message's fields, as PCL does: a point struct's member
// receives the bytes of the message field of the same name, wherever that field lies in the message's point_step. A
// registered field the message lacks keeps its zero value (PCL warns and leaves it).
#pragma once
#include <cstddef>
#include <cstring>
#include <string>
#include <vector>

#include <pcl/point_cloud.h>
#include <sensor_msgs/PointCloud2.h>

#ifndef EIGEN_ALIGN16
#define EIGEN_ALIGN16 alignas(16)
#endif
// PCL's 16-byte x / y / z / padding union: the fields after it start at byte 16.
#define PCL_ADD_POINT4D float x, y, z, data_pad_4d_;

namespace lk_shim {
struct FieldDesc {
    std::string name;
    size_t offset, size;
    FieldDesc(const char* n, size_t o, size_t s) : name(n), offset(o), size(s) {}
};
template <class PointT>
struct PointFields;  // one specialisation per POINT_CLOUD_REGISTER_POINT_STRUCT
}  // namespace lk_shim

// POINT_CLOUD_REGISTER_POINT_STRUCT(T, (type, member, name)(type, member, name)...): the sequence is walked by two
// alternating macros, each of which emits one element and names the other to consume the next parenthesised group; the
// name left over after the last group is pasted with _END into an empty macro. Elements are parenthesised calls, not
// braced lists, so that their commas stay inside parentheses when the whole expansion passes through LK_SHIM_CAT.
#define LK_SHIM_CAT(a, b) LK_SHIM_CAT_I(a, b)
#define LK_SHIM_CAT_I(a, b) a##b
#define LK_SHIM_FIELD_0(type, member, name) \
    v.push_back(::lk_shim::FieldDesc(#name, offsetof(Point, member), sizeof(type))); LK_SHIM_FIELD_1
#define LK_SHIM_FIELD_1(type, member, name) \
    v.push_back(::lk_shim::FieldDesc(#name, offsetof(Point, member), sizeof(type))); LK_SHIM_FIELD_0
#define LK_SHIM_FIELD_0_END
#define LK_SHIM_FIELD_1_END
#define POINT_CLOUD_REGISTER_POINT_STRUCT(T, seq)                    \
    namespace lk_shim {                                              \
    template <>                                                      \
    struct PointFields<T> {                                          \
        static std::vector<FieldDesc> get() {                        \
            using Point = T;                                         \
            std::vector<FieldDesc> v;                                \
            LK_SHIM_CAT(LK_SHIM_FIELD_0 seq, _END)                   \
            return v;                                                \
        }                                                            \
    };                                                               \
    }

namespace pcl {
template <class PointT>
void fromROSMsg(const sensor_msgs::PointCloud2& msg, PointCloud<PointT>& cloud) {
    struct Copy {
        size_t dst, src, size;
    };
    std::vector<Copy> map;
    for (const lk_shim::FieldDesc& f : lk_shim::PointFields<PointT>::get())
        for (const sensor_msgs::PointField& mf : msg.fields)
            if (mf.name == f.name) {
                map.push_back(Copy{f.offset, mf.offset, f.size});
                break;
            }
    cloud.points.assign((size_t)msg.width * msg.height, PointT());
    for (uint32_t r = 0; r < msg.height; ++r)
        for (uint32_t c = 0; c < msg.width; ++c) {
            const uint8_t* src = msg.data.data() + (size_t)r * msg.row_step + (size_t)c * msg.point_step;
            char* dst = reinterpret_cast<char*>(&cloud.points[(size_t)r * msg.width + c]);
            for (const Copy& m : map) std::memcpy(dst + m.dst, src + m.src, m.size);
        }
    cloud.width = msg.width;
    cloud.height = msg.height;
    cloud.is_dense = msg.is_dense;
}
}  // namespace pcl
