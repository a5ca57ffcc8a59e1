// Scan front end: the steps between the raw LiDAR points and the measurement update, kept in HBM.
//   sort by offset time + per-point de-skew     ImuProcess::UndistortPcl   src/IMU_Processing.hpp:232-234, 312-346
//   voxel-grid down-sampling                    pcl::VoxelGrid::filter     src/laserMapping.cpp:904-905
// and the sliding local-map cube that produces the delete boxes (on the host, or on the device from the state there)
//   LocalMapCube                                lasermap_fov_segment()     src/laserMapping.cpp:229-277
#pragma once
#include "lie.cuh"
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
    // that cloud in FL_FRAME_LIDAR / IMU / WORLD with the state x26 (host memory), at most cap rows; *n = the cloud's size
    int frame(int which, int frame, const double* x26, float* out_xyzi, int cap, int* n);
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
    // the device forms' cloud `which` in a frame, appended at *d_n_io of d_out (cap rows) when it fits; d_status2 = (status, n)
    int frame_on_stream(int which, int frame, const double* d_x26, float* d_out, int* d_n_io, int cap, int* d_status2, cudaStream_t st);
    // every host-form call first: takes over the device forms' cloud and counts when they produced the current one
    int settle();
    // the device forms' down-sampled cloud, its count in device memory, and its row bound (the n_max of their last upload)
    const float4* down_dev() const;
    const int* down_count_dev() const;
    int dev_n_max() const { return dev_n_max_; }
    bool dev_down_ready() const { return dev_down_; }      // a device-form down-sample ran since the last upload
    int reserved_n_max() const { return dev_used_ ? res_n_max_ : -1; }      // the rows reserve_device sized (-1: not yet)

private:
    static constexpr size_t UNDISTORT_SMEM_MAX = 200 * 1024;     // IMU poses in k_undistort's shared memory
    int undistort_smem(size_t smem);
    int cub_fits(int n, const char* what) const;
    Map* map_;
    int n_raw_ = 0, n_down_ = 0;
    DeviceBuffer raw_, raw_alt_, time_, time_alt_, down_, keys_, keys_alt_, vals_, vals_alt_, heads_, pos_, cub_tmp_, ctl_, poses_;
    DeviceBuffer frame_out_, frame_x_;      // the host form of frame(): its rows before the read-back, and its state
    int* h_count_ = nullptr;        // pinned
    size_t undistort_smem_ = 48 * 1024;
    // device forms: uploaded (d_raw_, d_time_) -> time-sorted and de-skewed (d_sraw_, d_stime_) -> down-sampled (d_down_)
    DeviceBuffer d_raw_, d_time_, d_sraw_, d_stime_, d_down_, d_keys_, d_keys_alt_, d_vals_, d_vals_alt_, d_heads_, d_pos_, d_cub_, d_ctl_;
    void* h_dctl_ = nullptr;        // pinned copy of the device forms' control block (settle)
    int res_n_max_ = 0, res_pose_max_ = 0, dev_n_max_ = 0;
    bool dev_used_ = false, dev_uploaded_ = false, dev_undistorted_ = false, dev_down_ = false;
};

// The scan front end of many scans in one call (fl_scan_batch_run_device): slot s of the packed [n_scans][n_max] buffers goes through
// the device forms' steps -- upload, stable time sort, de-skew, voxel grid -- with the kernels of ScanFrontEnd's stages run per slot,
// and one cub sort or scan over every slot at once where ScanFrontEnd runs one per scan.  The buffers are fixed between reserves.
class ScanBatch {
public:
    explicit ScanBatch(Map* map) : map_(map) {}
    ~ScanBatch();
    int reserve(int n_scans_max, int n_max, int n_pose_max);       // synchronous, grow-only
    int run_on_stream(const fl_scan_raw_t* d_raws, int n_scans, int n_max, int n_pose_max, int undistort, float leaf, int* d_status2,
                      cudaStream_t st);
    int refs(int which, const fl_scan_ref_t** out, int* n_max) const;
    int download(int which, int slot, float* out_xyzi, int cap, int* n);
    Map* map() const { return map_; }

private:
    static constexpr size_t UNDISTORT_SMEM_MAX = 200 * 1024;       // as ScanFrontEnd's
    static constexpr int SLOTS_MAX = 65535;                          // the grids' y dimension
    int cub_bytes(int rows, int end_bit, size_t* bytes) const;
    Map* map_;
    int res_slots_ = 0, res_n_max_ = 0, res_pose_max_ = 0;
    bool reserved_ = false;
    size_t undistort_smem_ = 48 * 1024;
    // rows as uploaded -> time-sorted and de-skewed -> down-sampled, each [n_scans][n_max]; the radix keys and values of both sorts,
    // the heads and their positions; per slot a BatchSlot (scan.cu); the two ref tables [2][n_scans_max] and their counts
    DeviceBuffer raw_, sraw_, down_, keys_, keys_alt_, vals_, vals_alt_, heads_, pos_, cub_, slots_, refs_, counts_;
};

// LocalMap_Points (:229) and Localmap_Initialized (:230)
struct CubeBox {
    float lo[3], hi[3];
    int init;
};
// The cube arithmetic of lasermap_fov_segment() (:236-270), shared by the host form and the device form's one-thread kernel.
// Slides `c` for the LiDAR position pos and returns the number of delete boxes written to boxes6 (<= 3, each min xyz / max xyz)
// -- cub_needrm.  The arithmetic keeps the reference's types: cube corners are float (BoxPointType, ikd_Tree.h:42-45), the
// position and cube_len are double, MOV_THRESHOLD (1.5f) and DET_RANGE are float (laserMapping.cpp:77-78).
FL_HD int cube_slide(CubeBox& c, const double pos[3], double cube_len, float det_range, float* boxes6) {
    const float margin = 1.5f * det_range;
    if (!c.init) {                                     // :238-245: first call only centres the cube
        for (int a = 0; a < 3; a++) {
            c.lo[a] = float(pos[a] - cube_len / 2.0);
            c.hi[a] = float(pos[a] + cube_len / 2.0);
        }
        c.init = 1;
        return 0;
    }
    int dir[3];                                        // 0: stay, 1: towards the low face, 2: towards the high face
    bool near_edge = false;
    for (int a = 0; a < 3; a++) {
        const float to_lo = float(fabs(pos[a] - double(c.lo[a])));
        const float to_hi = float(fabs(pos[a] - double(c.hi[a])));
        dir[a] = to_lo <= margin ? 1 : (to_hi <= margin ? 2 : 0);    // the low face wins (:259-264)
        near_edge = near_edge || dir[a] != 0;
    }
    if (!near_edge) return 0;
    const double shift = (cube_len - 2.0 * 1.5f * det_range) * 0.5 * 0.9, floor_ = double(det_range * (1.5f - 1));
    const float step = float(shift < floor_ ? floor_ : shift);        // std::max (:256)
    int nb = 0;
    float new_lo[3], new_hi[3];
    for (int a = 0; a < 3; a++) {
        new_lo[a] = c.lo[a]; new_hi[a] = c.hi[a];
        if (dir[a] == 0) continue;
        float* b = boxes6 + nb * 6;                    // the slab the cube leaves behind, spanning the OLD cube on the other axes
        for (int k = 0; k < 3; k++) { b[k] = c.lo[k]; b[3 + k] = c.hi[k]; }
        if (dir[a] == 1) {
            new_hi[a] = c.hi[a] - step; new_lo[a] = c.lo[a] - step;
            b[a] = c.hi[a] - step;
        } else {
            new_hi[a] = c.hi[a] + step; new_lo[a] = c.lo[a] + step;
            b[3 + a] = c.lo[a] + step;
        }
        nb++;
    }
    for (int a = 0; a < 3; a++) { c.lo[a] = new_lo[a]; c.hi[a] = new_hi[a]; }
    return nb;
}

// lasermap_fov_segment() without its globals.  The host form slides the cube in host memory; the device form
// (fl_localmap_segment_device) keeps it in a small buffer on the map's device, allocated by its first call, and from then on that
// copy is the cube: host-form calls read it back and write it again (synchronously).
class LocalMapCube {
public:
    LocalMapCube(double cube_len, float det_range) : cube_len_(cube_len), det_range_(det_range) {}
    ~LocalMapCube();
    // returns the number of delete boxes written to boxes6 (<= 3) -- cub_needrm
    int slide(const double pos_lid[3], float* boxes6) { return cube_slide(c_, pos_lid, cube_len_, det_range_, boxes6); }
    bool initialized() const { return c_.init != 0; }
    void get(float* box6) const;

    // Device form: pos_lid from the state x26 on the device, the cube slid there, then Map::enqueue_delete of its boxes,
    // all-or-nothing; out3 = (|cub_needrm|, kdtree_delete_counter, status).  The first call (outside capture) allocates the
    // buffer and uploads the host cube.  Call with the map's lock held.
    int segment_on_stream(Map* map, const double* d_x26, const int* d_n_scan, float* d_boxes18, int* d_out3, cudaStream_t st);
    Map* device_map() const { return dmap_; }
    // the device cube into the host's copy / the host's copy into the device cube (synchronous, on the map's stream)
    int pull();
    int push();

private:
    double cube_len_;
    float det_range_;
    CubeBox c_ = {{0, 0, 0}, {0, 0, 0}, 0};
    Map* dmap_ = nullptr;
    DeviceBuffer dev_;              // SegState (scan.cu)
};

}  // namespace fl
