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

}  // namespace fl
