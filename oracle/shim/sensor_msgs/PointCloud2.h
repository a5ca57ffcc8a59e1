// ORACLE / TEST INFRASTRUCTURE ONLY -- not part of the product path.
//
// Minimal stand-in for <sensor_msgs/PointCloud2.h>: the message's fields as ROS defines them (sensor_msgs/PointField.msg,
// sensor_msgs/PointCloud2.msg).  ConstPtr is a std::shared_ptr where ROS uses boost::shared_ptr.
#pragma once
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include <ros/ros.h>

namespace sensor_msgs {
struct PointField {
    enum : uint8_t { INT8 = 1, UINT8 = 2, INT16 = 3, UINT16 = 4, INT32 = 5, UINT32 = 6, FLOAT32 = 7, FLOAT64 = 8 };
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
    typedef std::shared_ptr<const PointCloud2> ConstPtr;
};
}  // namespace sensor_msgs
