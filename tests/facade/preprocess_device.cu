// A plain CUDA program on the C ABI: Preprocess::process of an Ouster-like frame through fl_preprocess_device, captured once
// into a CUDA graph and replayed for two frame sizes, against the host form fl_preprocess.  Prints "preprocess_device ok".
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include <cuda_runtime.h>

#include "fastlio_b200.h"

#define CHECK(x)                                                                          \
    do {                                                                                  \
        long long _r = (long long)(x);                                                    \
        if (_r < 0) { printf("%s:%d: %s -> %lld (%s)\n", __FILE__, __LINE__, #x, _r, fl_last_error()); return 1; } \
    } while (0)
#define CUCHECK(x)                                                                        \
    do {                                                                                  \
        cudaError_t _e = (x);                                                             \
        if (_e != cudaSuccess) { printf("%s:%d: %s\n", __FILE__, __LINE__, cudaGetErrorString(_e)); return 1; } \
    } while (0)

int main() {
    const int step = 48, n_max = 4096;       // ouster_ros::Point
    fl_preprocess_params_t p;
    memset(&p, 0, sizeof p);
    p.lidar_type = FL_LIDAR_OUST64; p.n_scans = 64; p.scan_rate = 10; p.time_unit = 3; p.point_filter_num = 2; p.blind = 0.5;
    p.point_step = step;
    p.off_x = 0; p.off_y = 4; p.off_z = 8; p.off_intensity = 16; p.off_time = 20; p.off_ring = -1; p.off_tag = -1; p.off_line = -1;
    fl_preprocess_t* h = nullptr;
    CHECK(fl_preprocess_create(&h, 0, &p, n_max));

    std::vector<uint8_t> raw((size_t)n_max * step, 0);
    for (int i = 0; i < n_max; i++) {
        float v[4] = {0.001f * (float)(i % 997) - 0.3f, 0.5f + 0.01f * (float)(i % 13), -0.2f, (float)i};
        uint32_t t = 100000000u / n_max * (uint32_t)i;
        memcpy(&raw[(size_t)i * step], v, 12);
        memcpy(&raw[(size_t)i * step + 16], &v[3], 4);
        memcpy(&raw[(size_t)i * step + 20], &t, 4);
    }
    uint8_t* d_raw; int* d_n; float *d_xyzi, *d_ms, *d_last; int* d_out2;
    CUCHECK(cudaMalloc(&d_raw, raw.size()));
    CUCHECK(cudaMalloc(&d_n, sizeof(int)));
    CUCHECK(cudaMalloc(&d_xyzi, sizeof(float) * 4 * n_max));
    CUCHECK(cudaMalloc(&d_ms, sizeof(float) * n_max));
    CUCHECK(cudaMalloc(&d_out2, sizeof(int) * 2));
    CUCHECK(cudaMalloc(&d_last, sizeof(float)));
    CUCHECK(cudaMemcpy(d_raw, raw.data(), raw.size(), cudaMemcpyHostToDevice));
    cudaStream_t st;
    CUCHECK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    cudaGraph_t g;
    cudaGraphExec_t ge;
    CUCHECK(cudaStreamBeginCapture(st, cudaStreamCaptureModeGlobal));
    CHECK(fl_preprocess_device(h, d_raw, d_n, n_max, d_xyzi, d_ms, d_out2, d_last, st));
    CUCHECK(cudaStreamEndCapture(st, &g));
    CUCHECK(cudaGraphInstantiate(&ge, g, 0));

    for (int n : {n_max, 1234}) {
        CUCHECK(cudaMemcpyAsync(d_n, &n, sizeof(int), cudaMemcpyHostToDevice, st));
        CUCHECK(cudaGraphLaunch(ge, st));
        int out2[2];
        float last = -1.f;
        CUCHECK(cudaMemcpyAsync(out2, d_out2, sizeof out2, cudaMemcpyDeviceToHost, st));
        CUCHECK(cudaMemcpyAsync(&last, d_last, sizeof last, cudaMemcpyDeviceToHost, st));
        CUCHECK(cudaStreamSynchronize(st));
        std::vector<float> hx(4 * n_max), hm(n_max), dx(4 * n_max), dm(n_max);
        float hlast = -2.f;
        const int k = fl_preprocess(h, raw.data(), n, hx.data(), hm.data(), n_max, &hlast);
        CHECK(k);
        CUCHECK(cudaMemcpy(dx.data(), d_xyzi, sizeof(float) * 4 * k, cudaMemcpyDeviceToHost));
        CUCHECK(cudaMemcpy(dm.data(), d_ms, sizeof(float) * k, cudaMemcpyDeviceToHost));
        if (out2[0] != k || out2[1] != 0 || memcmp(dx.data(), hx.data(), sizeof(float) * 4 * k) ||
            memcmp(dm.data(), hm.data(), sizeof(float) * k) || last != hlast || k < n / 2 - 64 || k > (n + 1) / 2) {
            printf("mismatch at n = %d: device kept %d, host %d\n", n, out2[0], k);
            return 1;
        }
    }
    cudaGraphExecDestroy(ge);
    cudaGraphDestroy(g);
    cudaStreamDestroy(st);
    cudaFree(d_raw); cudaFree(d_n); cudaFree(d_xyzi); cudaFree(d_ms); cudaFree(d_out2); cudaFree(d_last);
    CHECK(fl_preprocess_destroy(h));
    printf("preprocess_device ok\n");
    return 0;
}
