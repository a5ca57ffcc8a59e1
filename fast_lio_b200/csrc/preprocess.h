// Sensor preprocessing on the device: Preprocess::process of the reference (src/preprocess.cpp) with feature extraction
// off, for the four LiDAR types the launch files run (fl_preprocess_device, include/fastlio_b200.h).
#pragma once
#include <cuda_runtime.h>

#include "map.h"

namespace fl {

struct PpParams {
    int type, n_scans, pfn, step;
    int off[8];          // x, y, z, intensity, time, ring, tag, line; -1 = absent
    float scale;         // time_unit_scale (preprocess.cpp:52-69)
    double bb;           // blind * blind
    double omega_l;      // 0.361 * SCAN_RATE (preprocess.cpp:297)
    int key_bits;        // bits of the ring sort keys (rings 0..n_scans-1, n_scans = padding)
};

class Preprocessor {
public:
    Preprocessor(int device, const PpParams& p, int n_raw_max) : dev_(device), p_(p), n_raw_max_(n_raw_max) {}
    ~Preprocessor();
    int init();
    int device() const { return dev_; }
    // fl_preprocess_device
    int run_device(const void* d_raw, const int* d_n, int n_max, float* d_xyzi, float* d_ms, int* d_out2, float* d_last, cudaStream_t st);
    // fl_preprocess: returns the kept count
    int run_host(const void* raw, int n, float* xyzi, float* ms, int cap, float* last_ms);

private:
    int enqueue(const void* d_raw, const int* d_n, int n_max, float* d_xyzi, float* d_ms, int* d_out2, float* d_last, cudaStream_t st);
    size_t cub_bytes(int n) const;

    int dev_;
    PpParams p_;
    int n_raw_max_;
    cudaStream_t stream_ = nullptr;       // the host form's
    cudaEvent_t ev_ = nullptr;            // the last device-form call outside capture; the host form waits for it
    DeviceBuffer d_keep_, d_pos_, d_tm_, d_valid_, d_keys_, d_keys_alt_, d_vals_, d_vals_alt_, d_yaw_, d_tri_, d_tri_alt_,
        d_yaw_fp_, d_ctl_, d_cub_;
    // the host form's device copies
    DeviceBuffer d_raw_, d_n_, d_xyzi_, d_ms_, d_out_;
};

// Preprocess::process of many frames in one call (fl_preprocess_batch_run_device): slot s owns rows [s n_max, (s + 1) n_max) of
// the packed scratch and rows [s n_raw_max, (s + 1) n_raw_max) of the outputs; each of Preprocessor's steps runs per slot on grids
// of (row blocks, slots), and each cub call runs once over every slot's rows.  Everything is sized at creation.
class PreprocessBatch {
public:
    static constexpr int SLOTS_MAX = 65535;         // the grids' y dimension
    PreprocessBatch(int device, const PpParams& p, int n_slots_max, int n_raw_max)
        : dev_(device), p_(p), slots_max_(n_slots_max), n_raw_max_(n_raw_max) {}
    ~PreprocessBatch();
    int init();
    int run_device(const fl_preprocess_raw_t* d_raws, int n_slots, int n_max, int* d_status2, cudaStream_t st);
    void outputs(float** xyzi, float** ms, int** out2, float** last, int* n_raw_max) const;
    int download(int slot, float* xyzi, float* ms, int cap, float* last, int* n);

private:
    size_t cub_bytes(int rows) const;
    int dev_;
    PpParams p_;
    int slots_max_, n_raw_max_, sort_bits_ = 0;     // sort_bits_: the Velodyne ring sort's, key_bits + the bits of n_slots_max
    cudaStream_t stream_ = nullptr;                 // download's
    cudaEvent_t ev_ = nullptr;                      // the last call outside capture; download waits for it
    // per packed row: the flags, positions, times and the Velodyne sort's keys, values, yaws and maps; per slot its PbSlot
    // (preprocess.cu) and yaw_fp [slot][ring]
    DeviceBuffer keep_, pos_, tm_, valid_, keys_, keys_alt_, vals_, vals_alt_, yaw_, tri_, tri_alt_, yaw_fp_, slots_, cub_;
    DeviceBuffer xyzi_, ms_, out2_, last_;          // the outputs
};

}  // namespace fl
