// ORACLE / TEST INFRASTRUCTURE ONLY -- not part of the product path.
//
// Minimal stand-in for <ros/ros.h> so that the reference's src/preprocess.{h,cpp} compile unmodified without ROS.
// Only what preprocess.cpp names is provided: ros::Time (header stamps, Preprocess::pub_func), ros::Publisher
// (members of Preprocess, never used) and the headers roscpp would bring in (<cmath>, <vector>, OpenMP's omp_get_wtime).
#pragma once
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <memory>
#include <string>
#include <vector>

#include <omp.h>

namespace ros {
struct Time {
    uint32_t sec = 0, nsec = 0;
    double toSec() const { return double(sec) + 1e-9 * double(nsec); }
};
struct Publisher {};
}  // namespace ros

namespace std_msgs {
struct Header {
    uint32_t seq = 0;
    ros::Time stamp;
    std::string frame_id;
};
}  // namespace std_msgs
