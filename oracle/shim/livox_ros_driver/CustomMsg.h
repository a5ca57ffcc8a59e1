// ORACLE / TEST INFRASTRUCTURE ONLY -- not part of the product path.
//
// Minimal stand-in for the Livox driver's message (livox_ros_driver/msg/CustomPoint.msg, CustomMsg.msg): the fields in
// the message's order, so a CustomPoint is 20 bytes (u32, 3 x f32, 3 x u8, padding).
#pragma once
#include <cstdint>
#include <memory>
#include <vector>

#include <ros/ros.h>

namespace livox_ros_driver {
struct CustomPoint {
    uint32_t offset_time = 0;
    float x = 0.f, y = 0.f, z = 0.f;
    uint8_t reflectivity = 0, tag = 0, line = 0;
};
struct CustomMsg {
    std_msgs::Header header;
    uint64_t timebase = 0;
    uint32_t point_num = 0;
    uint8_t lidar_id = 0;
    uint8_t rsvd[3] = {0, 0, 0};
    std::vector<CustomPoint> points;
    typedef std::shared_ptr<const CustomMsg> ConstPtr;
};
}  // namespace livox_ros_driver
