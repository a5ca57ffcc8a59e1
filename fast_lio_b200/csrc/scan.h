// Scan front end: the steps between the raw LiDAR points and the measurement update, kept in HBM.
//   sort by offset time + per-point de-skew     ImuProcess::UndistortPcl   src/IMU_Processing.hpp:232-234, 312-346
//   voxel-grid down-sampling                    pcl::VoxelGrid::filter     src/laserMapping.cpp:904-905
// and the sliding local-map cube that produces the delete boxes (host arithmetic only)
//   LocalMapCube                                lasermap_fov_segment()     src/laserMapping.cpp:229-277
#pragma once
#include "map.h"

namespace fl {

constexpr int POSE_DOUBLES = 22;   // msg/Pose6D.msg: offset_time, acc[3], gyr[3], vel[3], pos[3], rot[9]

class ScanFrontEnd {
public:
    explicit ScanFrontEnd(Map* map) : map_(map) {}
    ~ScanFrontEnd();
    int init();
    // raw scan: n x (x,y,z,intensity) and the per-point offset time in ms (PointType::curvature), host memory
    int upload(const float* xyzi, const float* offset_ms, int n);
    // stable sort by offset time (:234), then backward propagation of every point to the frame end (:312-346).
    // poses: n_pose x 22 doubles = IMUpose; x26_end: kf_state.get_x() after the last predict (:303)
    int undistort(const double* poses, int n_pose, const double* x26_end);
    // feats_undistort -> feats_down_body; *n_out = number of occupied voxels (one 4-byte read-back)
    int voxel_downsample(float leaf, int* n_out);
    int download(int which, float* out_xyzi, int cap, int* n);   // which 0: raw / undistorted, 1: down-sampled
    const float4* down_device() const { return down_.as<float4>(); }
    int down_count() const { return n_down_; }
    int raw_count() const { return n_raw_; }
    Map* map() const { return map_; }

    // Device forms (fl_scan_*_device): enqueued on the caller's stream `st`, counts kept in device memory and read there, grids
    // sized from n_max, no host synchronisation and no allocation, so they may be captured into a CUDA graph.  They use buffers of
    // their own, sized by reserve_device (synchronous) for up to n_max points and n_pose_max IMU poses.
    int reserve_device(int n_max, int n_pose_max);
    int upload_on_stream(const float* d_xyzi, const float* d_offset_ms, const int* d_n, int n_max, cudaStream_t st);
    int undistort_on_stream(const double* d_poses, const int* d_n_pose, int n_pose_max, const double* d_x26_end, cudaStream_t st);
    int voxel_downsample_on_stream(float leaf, int* d_n_out, cudaStream_t st);
    // every host-form call first: takes over the device forms' cloud and counts when they produced the current one
    int settle();
    // the device forms' down-sampled cloud, its count in device memory, and its row bound (the n_max of their last upload)
    const float4* down_dev() const;
    const int* down_count_dev() const;
    int dev_n_max() const { return dev_n_max_; }
    bool dev_down_ready() const { return dev_down_; }      // a device-form down-sample ran since the last upload

private:
    static constexpr size_t UNDISTORT_SMEM_MAX = 200 * 1024;     // IMU poses in k_undistort's shared memory
    int undistort_smem(size_t smem);
    int cub_fits(int n, const char* what) const;
    Map* map_;
    int n_raw_ = 0, n_down_ = 0;
    DeviceBuffer raw_, raw_alt_, time_, time_alt_, down_, keys_, keys_alt_, vals_, vals_alt_, heads_, pos_, cub_tmp_, ctl_, poses_;
    int* h_count_ = nullptr;        // pinned
    size_t undistort_smem_ = 48 * 1024;
    // device forms: uploaded (d_raw_, d_time_) -> time-sorted and de-skewed (d_sraw_, d_stime_) -> down-sampled (d_down_)
    DeviceBuffer d_raw_, d_time_, d_sraw_, d_stime_, d_down_, d_keys_, d_keys_alt_, d_vals_, d_vals_alt_, d_heads_, d_pos_, d_cub_, d_ctl_;
    void* h_dctl_ = nullptr;        // pinned copy of the device forms' control block (settle)
    int res_n_max_ = 0, res_pose_max_ = 0, dev_n_max_ = 0;
    bool dev_used_ = false, dev_uploaded_ = false, dev_undistorted_ = false, dev_down_ = false;
};

// lasermap_fov_segment() without its globals: LocalMap_Points (:229) and Localmap_Initialized (:230) live here.
class LocalMapCube {
public:
    LocalMapCube(double cube_len, float det_range) : cube_len_(cube_len), det_range_(det_range) {}
    // returns the number of delete boxes written to boxes6 (<= 3, each min xyz / max xyz) -- cub_needrm
    int slide(const double pos_lid[3], float* boxes6);
    bool initialized() const { return init_; }
    void get(float* box6) const;

private:
    double cube_len_;
    float det_range_;
    float lo_[3] = {0, 0, 0}, hi_[3] = {0, 0, 0};
    bool init_ = false;
};

}  // namespace fl
