// ============================================================================
// ORACLE -- TEST INFRASTRUCTURE ONLY (see oracle/fastlio_oracle.cpp header).
//
// extern "C" wrapper around the reference's own Preprocess::process (src/preprocess.cpp:44-87), compiled unmodified
// together with it against the shims under oracle/shim.  Built by oracle/preprocess_ref.py into
// oracle/_ref/libpreprocess_ref.so; nothing from the reference is copied here.
//
// The raw frame is what the sensor driver publishes: n rows of point_step bytes, with the fields at the byte offsets of
// off8 = (x, y, z, intensity, time, ring, tag, line), -1 = absent.  The field types are those of the reference's structs
// (the fl_preprocess_params_t convention, include/fastlio_b200.h):
//   AVIA (1)   livox_ros_driver::CustomMsg: offset_time u32 (time), x/y/z f32, reflectivity u8 (intensity), tag u8, line u8
//   VELO16 (2) velodyne_ros::Point:         x/y/z/intensity/time f32, ring u16
//   OUST64 (3) ouster_ros::Point:           x/y/z/intensity f32, t u32 (time)
//   MARSIM (4) pcl::PointXYZI:              x/y/z/intensity f32
// Avia rows are decoded into a CustomMsg as the driver's deserialiser would; the others travel as a PointCloud2 whose
// fields list the present offsets, and the shim's fromROSMsg decodes them.
// ============================================================================
#include "preprocess.h"

#include <chrono>
#include <cstring>

namespace {

enum { F_X, F_Y, F_Z, F_I, F_T, F_RING, F_TAG, F_LINE };

template <class T>
T field(const uint8_t* row, int off) {
    T v = 0;
    if (off >= 0) std::memcpy(&v, row + off, sizeof(T));
    return v;
}

struct Frame {
    livox_ros_driver::CustomMsg::ConstPtr livox;
    sensor_msgs::PointCloud2::ConstPtr cloud;
};

Frame make_frame(int lidar_type, const uint8_t* raw, int n, int point_step, const int* off) {
    Frame fr;
    if (lidar_type == AVIA) {
        auto m = std::make_shared<livox_ros_driver::CustomMsg>();
        m->point_num = uint32_t(n);
        m->points.resize(n);
        for (int i = 0; i < n; i++) {
            const uint8_t* r = raw + size_t(i) * point_step;
            livox_ros_driver::CustomPoint& p = m->points[i];
            p.offset_time = field<uint32_t>(r, off[F_T]);
            p.x = field<float>(r, off[F_X]);
            p.y = field<float>(r, off[F_Y]);
            p.z = field<float>(r, off[F_Z]);
            p.reflectivity = field<uint8_t>(r, off[F_I]);
            p.tag = field<uint8_t>(r, off[F_TAG]);
            p.line = field<uint8_t>(r, off[F_LINE]);
        }
        fr.livox = m;
        return fr;
    }
    auto m = std::make_shared<sensor_msgs::PointCloud2>();
    m->width = uint32_t(n);
    m->point_step = uint32_t(point_step);
    m->row_step = uint32_t(n) * uint32_t(point_step);
    m->data.assign(raw, raw + size_t(n) * point_step);
    typedef sensor_msgs::PointField PF;
    auto add = [&](const char* name, int o, uint8_t type) {
        if (o < 0) return;
        PF f;
        f.name = name;
        f.offset = uint32_t(o);
        f.datatype = type;
        m->fields.push_back(f);
    };
    add("x", off[F_X], PF::FLOAT32);
    add("y", off[F_Y], PF::FLOAT32);
    add("z", off[F_Z], PF::FLOAT32);
    add("intensity", off[F_I], PF::FLOAT32);
    if (lidar_type == VELO16) {
        add("time", off[F_T], PF::FLOAT32);
        add("ring", off[F_RING], PF::UINT16);
    } else if (lidar_type == OUST64) {
        add("t", off[F_T], PF::UINT32);
    }
    fr.cloud = m;
    return fr;
}

}  // namespace

extern "C" {

// Preprocess::set(false, lidar_type, blind, point_filter_num) with N_SCANS, SCAN_RATE and time_unit as laserMapping.cpp
// reads them (:781-787), then one process() call on the frame.  Writes min(|pl_surf|, cap) rows of (x, y, z, intensity)
// and curvature; returns |pl_surf|.  *seconds (may be NULL) receives the wall time of process() alone.
int ref_preprocess(int lidar_type, int n_scans, int scan_rate, int time_unit, int point_filter_num, double blind,
                   const uint8_t* raw, int n, int point_step, const int* off8, float* out_xyzi, float* out_ms, int cap,
                   double* seconds) {
    Preprocess p;
    p.set(false, lidar_type, blind, point_filter_num);
    p.N_SCANS = n_scans;
    p.SCAN_RATE = scan_rate;
    p.time_unit = time_unit;
    Frame fr = make_frame(lidar_type, raw, n, point_step, off8);
    PointCloudXYZI::Ptr out(new PointCloudXYZI());
    const auto t0 = std::chrono::steady_clock::now();
    if (fr.livox) p.process(fr.livox, out);
    else p.process(fr.cloud, out);
    const auto t1 = std::chrono::steady_clock::now();
    if (seconds) *seconds = std::chrono::duration<double>(t1 - t0).count();
    const int m = int(out->size());
    for (int i = 0; i < m && i < cap; i++) {
        const PointType& q = out->points[i];
        out_xyzi[4 * i + 0] = q.x;
        out_xyzi[4 * i + 1] = q.y;
        out_xyzi[4 * i + 2] = q.z;
        out_xyzi[4 * i + 3] = q.intensity;
        out_ms[i] = q.curvature;
    }
    return m;
}

}  // extern "C"
