// Shared helpers for the sm_90a kernels of the FAST-LIO2 measurement-update path.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/fastlio_b200.h"   // FL_OK / FL_ERR_* status codes

namespace fl {

// ----------------------------------------------------------------------------- errors
// No exceptions cross the C ABI: every host entry point returns an int status and
// records a message retrievable through fl_last_error().
void set_last_error(const char* fmt, ...);

#define FL_CUDA(expr)                                                                   \
    do {                                                                                \
        cudaError_t _e = (expr);                                                        \
        if (_e != cudaSuccess) {                                                        \
            ::fl::set_last_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,          \
                                 cudaGetErrorString(_e));                               \
            return FL_ERR_CUDA;                                                   \
        }                                                                               \
    } while (0)

#define FL_CHECK(expr)                      \
    do {                                    \
        int _s = (expr);                    \
        if (_s != FL_OK) return _s;   \
    } while (0)

// ----------------------------------------------------------------------------- constants
constexpr int LEAF = 32;            // slots per leaf bucket == warp width (one coalesced 512 B load)
constexpr int FAN = 32;             // children per internal node (one lane per child box)
constexpr int MAX_LEVELS = 7;       // 32^7 leaves -- far beyond 80 GB of HBM
constexpr int KNN_K = 5;            // NUM_MATCH_POINTS, reference include/common_lib.h:26
constexpr unsigned FULL = 0xffffffffu;

constexpr int NRED = 78 + 12 + 2;   // upper triangle of H^T H (12x12), H^T h, effct, sum |res|

// ----------------------------------------------------------------------------- exact float helpers
// The reference computes squared distances in float32 on x86-64 without FMA contraction
// (ikd_Tree.cpp:1683-1709).  To obtain bit-identical distances (hence identical neighbour
// sets) every parity-critical float expression is written with explicitly rounded intrinsics.
__device__ __forceinline__ float sq_dist3(float ax, float ay, float az, float bx, float by, float bz) {
    float dx = __fsub_rn(ax, bx), dy = __fsub_rn(ay, by), dz = __fsub_rn(az, bz);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// calc_box_dist (ikd_Tree.cpp:1691-1709): squared distance from a point to an AABB
__device__ __forceinline__ float box_dist3(float qx, float qy, float qz, float lx, float ly, float lz,
                                           float hx, float hy, float hz) {
    // per axis at most one of (q < lo), (q > hi) holds, and (q - lo)^2 == (lo - q)^2 exactly, so
    // max(lo - q, q - hi, 0)^2 summed x, y, z reproduces the reference's value bit for bit
    const float dx = fmaxf(fmaxf(__fsub_rn(lx, qx), __fsub_rn(qx, hx)), 0.0f);
    const float dy = fmaxf(fmaxf(__fsub_rn(ly, qy), __fsub_rn(qy, hy)), 0.0f);
    const float dz = fmaxf(fmaxf(__fsub_rn(lz, qz), __fsub_rn(qz, hz)), 0.0f);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// ----------------------------------------------------------------------------- float atomics
__device__ __forceinline__ void atomic_min_float(float* addr, float v) {
    // works for any finite / infinite floats (no NaN)
    if (v >= 0.0f) atomicMin((int*)addr, __float_as_int(v));
    else atomicMax((unsigned int*)addr, __float_as_uint(v));
}
__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
    if (v >= 0.0f) atomicMax((int*)addr, __float_as_int(v));
    else atomicMin((unsigned int*)addr, __float_as_uint(v));
}

}  // namespace fl
