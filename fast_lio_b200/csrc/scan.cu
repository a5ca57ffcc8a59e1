// Scan front end kernels (see scan.h).  Everything runs on the map's stream, so a scan goes
// raw -> de-skewed -> down-sampled -> iEKF update -> map_incremental without leaving HBM.
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

#include <cub/cub.cuh>

#include "common.cuh"
#include "lie.cuh"
#include "measure.cuh"
#include "scan.h"

namespace fl {

void set_last_error(const char* fmt, ...);

namespace {

struct VgCtl {
    float mn[3], mx[3];
    int total;          // number of output points
    int passthrough;    // PCL's "leaf size too small" exit: output = input
};

// The device forms' control block: their voxel grid, and what the host forms need to take the cloud over (ScanFrontEnd::settle).
// Every device-form stage sets src, so the host forms see the result of whichever device-form stage ran last.
struct ScanDevCtl {
    VgCtl vg;           // vg.total: the device forms' feats_down_size
    int n_raw;          // *n_device of their last upload, clamped to [0, n_max]
    int src;            // 1: a device-form stage ran since the host forms last took the cloud over (settle clears it)
    int stage;          // 1: their cloud was de-skewed (it is in the sorted buffers), 0: as uploaded
    int down;           // 1: they down-sampled it since their upload
};

// ------------------------------------------------------------------------------------------------ de-skew
struct EndState {
    D3 pos, offT;
    Q4 rot_inv, offR, offR_inv;
};

// Exp(ang_vel, dt) as the reference evaluates it (include/so3_math.h:37-58): Rodrigues with the
// normalised axis, I + sin(a) K + ((1 - cos a) K) K.
__device__ __forceinline__ M33 rodrigues(const D3& w, double dt) {
    const double n = norm3(w);
    if (!(n > 0.0000001)) return eye33();
    const D3 a = d3(w.x / n, w.y / n, w.z / n);
    const M33 K = hat3(a);
    const double ang = n * dt;
    double s, c;
    sincos(ang, &s, &c);
    const double c1 = 1.0 - c;
    M33 cK;
#pragma unroll
    for (int i = 0; i < 9; i++) cK.m[i] = c1 * K.m[i];
    const M33 cKK = mul33(cK, K);
    const M33 I = eye33();
    M33 r;
#pragma unroll
    for (int i = 0; i < 9; i++) r.m[i] = (I.m[i] + s * K.m[i]) + cKK.m[i];
    return r;
}

// One point, one IMU segment [head, tail] (IMU_Processing.hpp:327-341).
__device__ __forceinline__ void compensate(float4& p, double t, const double* head, const double* tail, const EndState& e) {
    const double dt = t - head[0];
    M33 R_imu;
#pragma unroll
    for (int i = 0; i < 9; i++) R_imu.m[i] = head[13 + i];
    const D3 vel = ld3(head + 7), pos = ld3(head + 10), acc = ld3(tail + 1), gyr = ld3(tail + 4);
    const M33 R_i = mul33(R_imu, rodrigues(gyr, dt));
    const D3 P_i = d3(p.x, p.y, p.z);
    const D3 T_ei = d3(((pos.x + vel.x * dt) + ((0.5 * acc.x) * dt) * dt) - e.pos.x,
                       ((pos.y + vel.y * dt) + ((0.5 * acc.y) * dt) * dt) - e.pos.y,
                       ((pos.z + vel.z * dt) + ((0.5 * acc.z) * dt) * dt) - e.pos.z);
    const D3 inner = mul33v(R_i, qrot(e.offR, P_i) + e.offT) + T_ei;
    const D3 out = qrot(e.offR_inv, qrot(e.rot_inv, inner) - e.offT);
    p.x = float(out.x); p.y = float(out.y); p.z = float(out.z);
}

__device__ __forceinline__ EndState end_state(const double* x_end) {
    EndState e;
    e.pos = ld3(x_end);
    e.rot_inv = qconj(ldq(x_end + 3));
    e.offR = ldq(x_end + 7);
    e.offR_inv = qconj(e.offR);
    e.offT = ld3(x_end + 11);
    return e;
}

// The reference sweeps points and IMU segments backwards together (:314-345).  For time-sorted points that
// is: point i belongs to the LAST segment kp whose head is strictly older than the point; points older than
// every head stay untouched.  One quirk is kept: the sweep `break`s on the first point and then re-tests
// it against every earlier segment, so point 0 is compensated once per earlier segment that is older than it.
// Device forms: n and n_pose are the row bounds, the counts are min(*n_dev, n) and *n_pose_dev clamped to [0, n_pose], and
// the kernel marks the device forms' cloud as de-skewed and current (dc: null in the host form).
// Row i of the sorted cloud, at time t (s), through the segments of the n_pose poses in s_pose; written back only when it moved.
// k_batch_undistort's form of k_undistort's loop below, which keeps its own copy: calling this helper there flips one branch of
// its SASS (tests/golden/sass_scan_kernels_sm90a.json pins it).
__device__ __forceinline__ void undistort_row(float4* __restrict__ pts, int i, double t, const double* s_pose, int n_pose, const EndState& e) {
    float4 p = pts[i];
    bool touched = false;
    for (int kp = n_pose - 1; kp >= 1; kp--) {
        const double* head = s_pose + (kp - 1) * POSE_DOUBLES;
        if (t > head[0]) {
            compensate(p, t, head, head + POSE_DOUBLES, e);
            touched = true;
            if (i != 0) break;
        }
    }
    if (touched) pts[i] = p;
}

__global__ void k_undistort(float4* __restrict__ pts, const float* __restrict__ t_ms, int n,
                            const double* __restrict__ poses, int n_pose, const double* __restrict__ x_end,
                            const int* __restrict__ n_dev, const int* __restrict__ n_pose_dev, ScanDevCtl* dc) {
    extern __shared__ double s_pose[];
    if (n_dev) n = min(*n_dev, n);
    if (n_pose_dev) n_pose = min(max(*n_pose_dev, 0), n_pose);
    if (dc && blockIdx.x == 0 && threadIdx.x == 0) { dc->stage = 1; dc->src = 1; }
    for (int i = threadIdx.x; i < n_pose * POSE_DOUBLES; i += blockDim.x) s_pose[i] = poses[i];
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    EndState e;
    e.pos = ld3(x_end);
    e.rot_inv = qconj(ldq(x_end + 3));
    e.offR = ldq(x_end + 7);
    e.offR_inv = qconj(e.offR);
    e.offT = ld3(x_end + 11);
    const double t = double(t_ms[i]) / double(1000);
    float4 p = pts[i];
    bool touched = false;
    for (int kp = n_pose - 1; kp >= 1; kp--) {
        const double* head = s_pose + (kp - 1) * POSE_DOUBLES;
        if (t > head[0]) {
            compensate(p, t, head, head + POSE_DOUBLES, e);
            touched = true;
            if (i != 0) break;
        }
    }
    if (touched) pts[i] = p;
}

// ------------------------------------------------------------------------------------------------ voxel grid
// The `*_dev` counts of the kernels below: n is the row bound (n_max), the count min(*n_dev, n); null in the host forms.
__device__ __forceinline__ int dev_count(const int* n_dev, int n) { return n_dev ? min(*n_dev, n) : n; }

// dc (device forms, null in the host form): the down-sampled cloud is theirs and current
__global__ void k_vg_reset(VgCtl* c, ScanDevCtl* dc) {
    if (threadIdx.x < 3) { c->mn[threadIdx.x] = FLT_MAX; c->mx[threadIdx.x] = -FLT_MAX; }
    if (threadIdx.x == 3) { c->total = 0; c->passthrough = 0; }
    if (threadIdx.x == 4 && dc) { dc->down = 1; dc->src = 1; }
}

// fl_scan_upload_device: the first n = *n_dev (clamped to [0, n_max]) rows, and the offset time 0x7FFFFFFF (a NaN) in rows
// [n, n_max).  cub's float twiddle maps that pattern to 0xFFFFFFFF, the largest key, and the sort is stable, so the padding rows
// sort after the real ones and the first n rows of the n_max-row time sort are those of the n-row sort, NaN times included.
__global__ void k_upload_n(const float4* __restrict__ xyzi, const float* __restrict__ t_ms, const int* __restrict__ n_dev, int n_max,
                           float4* __restrict__ raw, float* __restrict__ time, ScanDevCtl* c) {
    const int n = min(max(*n_dev, 0), n_max);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) { c->n_raw = n; c->src = 1; c->stage = 0; c->down = 0; }
    if (i >= n_max) return;
    if (i < n) { raw[i] = xyzi[i]; time[i] = t_ms[i]; }
    else time[i] = __int_as_float(0x7FFFFFFF);
}

// getMinMax3D (pcl/common/impl/common.hpp) over a dense cloud: the block's rows i = block * blockDim.x + threadIdx.x, strided by
// blocks * blockDim.x, into c's bounds
__device__ __forceinline__ void vg_minmax_block(const float4* __restrict__ pts, int n, VgCtl* c, int block, int blocks) {
    float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int i = block * blockDim.x + threadIdx.x; i < n; i += blocks * blockDim.x) {
        const float4 p = pts[i];
        mn[0] = fminf(mn[0], p.x); mx[0] = fmaxf(mx[0], p.x);
        mn[1] = fminf(mn[1], p.y); mx[1] = fmaxf(mx[1], p.y);
        mn[2] = fminf(mn[2], p.z); mx[2] = fmaxf(mx[2], p.z);
    }
#pragma unroll
    for (int a = 0; a < 3; a++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
            mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
        }
    }
    // one set of atomics per BLOCK: all of them hit the same six words, so every atomic that is saved is latency saved
    __shared__ float s_mn[8][3], s_mx[8][3];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) {
#pragma unroll
        for (int a = 0; a < 3; a++) { s_mn[warp][a] = mn[a]; s_mx[warp][a] = mx[a]; }
    }
    __syncthreads();
    if (threadIdx.x < 3) {
        const int a = threadIdx.x;
        float lo = s_mn[0][a], hi = s_mx[0][a];
        for (int w = 1; w < (int)(blockDim.x >> 5); w++) { lo = fminf(lo, s_mn[w][a]); hi = fmaxf(hi, s_mx[w][a]); }
        atomic_min_float(&c->mn[a], lo);
        atomic_max_float(&c->mx[a], hi);
    }
}

__global__ void k_vg_minmax(const float4* __restrict__ pts, int n, VgCtl* c, const int* __restrict__ n_dev) {
    vg_minmax_block(pts, dev_count(n_dev, n), c, blockIdx.x, gridDim.x);
}

struct VgGrid {
    float inv;
    int min_b[3], mul[3];
    bool overflow;
};
// pcl::VoxelGrid::applyFilter: leaf-size check, min_b_/div_b_/divb_mul_
__device__ __forceinline__ VgGrid vg_grid(const VgCtl* c, float leaf) {
    VgGrid g;
    g.inv = __fdiv_rn(1.0f, leaf);
    long long d[3];
    int div_b[3];
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const float mn = c->mn[a], mx = c->mx[a];
        d[a] = (long long)(__fmul_rn(__fsub_rn(mx, mn), g.inv)) + 1;
        g.min_b[a] = int(floorf(__fmul_rn(mn, g.inv)));
        div_b[a] = int(floorf(__fmul_rn(mx, g.inv))) - g.min_b[a] + 1;
    }
    g.overflow = d[0] * d[1] * d[2] > (long long)INT_MAX;
    g.mul[0] = 1; g.mul[1] = div_b[0]; g.mul[2] = div_b[0] * div_b[1];
    return g;
}

// A real row's voxel key: its cell's index in the grid, or in passthrough mode its row index i, which makes the "cell" the point
// itself and turns the rest of the pipeline into a copy
__device__ __forceinline__ unsigned vg_key(const float4& p, const VgGrid& g, int i) {
    const int i0 = int(__fsub_rn(floorf(__fmul_rn(p.x, g.inv)), float(g.min_b[0])));
    const int i1 = int(__fsub_rn(floorf(__fmul_rn(p.y, g.inv)), float(g.min_b[1])));
    const int i2 = int(__fsub_rn(floorf(__fmul_rn(p.z, g.inv)), float(g.min_b[2])));
    return g.overflow ? unsigned(i) : unsigned(i0 * g.mul[0] + i1 * g.mul[1] + i2 * g.mul[2]);
}

// Padding rows (device forms) get the key 0xFFFFFFFF.  Real keys are below 2^31 (the overflow test bounds the grid, passthrough
// keys are row indices), and a real key equal to it would still precede the padding rows in the stable sort.
__global__ void k_vg_keys(const float4* __restrict__ pts, int n, float leaf, VgCtl* c, unsigned* __restrict__ keys, int* __restrict__ vals,
                          const int* __restrict__ n_dev) {
    const VgGrid g = vg_grid(c, leaf);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) c->passthrough = g.overflow ? 1 : 0;
    if (i >= n) return;
    if (i >= dev_count(n_dev, n)) { keys[i] = 0xFFFFFFFFu; vals[i] = i; return; }
    keys[i] = vg_key(pts[i], g, i);
    vals[i] = i;
}

// padding rows are no heads, so the exclusive scan over n_max rows gives the real rows the positions of the n-row scan
__global__ void k_vg_heads(const unsigned* __restrict__ keys, int n, int* __restrict__ heads, const int* __restrict__ n_dev) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) heads[i] = (i < dev_count(n_dev, n) && (i == 0 || keys[i] != keys[i - 1])) ? 1 : 0;
}

// CentroidPoint per occupied cell: float sums in ascending input index (the radix sort is stable), then / count.
// One thread per cell walks its run; raw scans put a handful of points into a cell.  The run of head row i among rows [0, n):
template <class Key>
__device__ __forceinline__ float4 vg_run(const float4* __restrict__ pts, const Key* __restrict__ keys, const int* __restrict__ vals, int i, int n) {
    const Key key = keys[i];
    float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f;
    int j = i;
    do {
        const float4 p = pts[vals[j]];
        sx = __fadd_rn(sx, p.x); sy = __fadd_rn(sy, p.y); sz = __fadd_rn(sz, p.z); si = __fadd_rn(si, p.w);
        j++;
    } while (j < n && keys[j] == key);
    const float cnt = float(j - i);
    return make_float4(__fdiv_rn(sx, cnt), __fdiv_rn(sy, cnt), __fdiv_rn(sz, cnt), __fdiv_rn(si, cnt));
}

__global__ void k_vg_centroid(const float4* __restrict__ pts, const unsigned* __restrict__ keys, const int* __restrict__ vals,
                              const int* __restrict__ heads, const int* __restrict__ pos, int n, float4* __restrict__ out, VgCtl* c,
                              const int* __restrict__ n_dev) {
    n = dev_count(n_dev, n);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (i == n - 1) c->total = pos[i] + heads[i];
    if (!heads[i]) return;
    out[pos[i]] = vg_run(pts, keys, vals, i, n);
}

// ------------------------------------------------------------------------------------------------ clouds in a frame
// The loops of publish_frame_world / publish_frame_body / the map's first Build (laserMapping.cpp:200-220, :177-186): row i of the
// cloud into row pos + i of out, in FL_FRAME_LIDAR as stored, in FL_FRAME_IMU as p_this = R_LI p + t_LI and in FL_FRAME_WORLD as
// rot p_this + pos -- body_to_world, the arithmetic of the update and k_map_incremental -- with the intensity passed through.
// Device form: n = *n_dev clamped to [0, n], pos = *n_io, and nothing is written unless 0 <= pos and pos + n <= cap (k_frame_commit
// then reports why); host form: n_dev and n_io null, pos 0.
__global__ void k_frame(const float4* __restrict__ src, int n, const int* __restrict__ n_dev, const double* __restrict__ x, int frame,
                        float4* __restrict__ out, const int* __restrict__ n_io, int cap) {
    if (n_dev) n = min(max(*n_dev, 0), n);
    const int pos = n_io ? *n_io : 0;
    if (pos < 0 || pos > cap || n > cap - pos) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float4 p = src[i];
    if (frame != FL_FRAME_LIDAR) {
        float wx, wy, wz;
        const D3 p_this = body_to_world(load_pose(x), p, wx, wy, wz);
        if (frame == FL_FRAME_IMU) { p.x = (float)p_this.x; p.y = (float)p_this.y; p.z = (float)p_this.z; }
        else { p.x = wx; p.y = wy; p.z = wz; }
    }
    out[pos + i] = p;
}

// after k_frame: status2 = (FL_OK, n) and *n_io advanced by n, or (FL_ERR_ARG / FL_ERR_CAPACITY, n) with *n_io as it was
__global__ void k_frame_commit(const int* __restrict__ n_dev, int n_max, int* __restrict__ n_io, int cap, int* __restrict__ status2) {
    const int n = min(max(*n_dev, 0), n_max);
    const int pos = *n_io;
    const int st = (pos < 0 || pos > cap) ? FL_ERR_ARG : (n > cap - pos ? FL_ERR_CAPACITY : FL_OK);
    if (st == FL_OK) *n_io = pos + n;
    status2[0] = st;
    status2[1] = n;
}


// ------------------------------------------------------------------------------------------------ many scans (ScanBatch)
// Slot s owns rows [s * n_max, (s + 1) * n_max) of every packed buffer; the grids are (row blocks, slots), so blockIdx.y is the slot.
struct BatchSlot {
    VgCtl vg;           // the slot's voxel grid; vg.total: its feats_down_size
    int n;              // its count c, 0 for a refused slot
    int err;            // FL_OK or its refusal
};

// cub's radix key for a float (its RadixSortTwiddle): -0.0 folded onto +0.0, then the sign-dependent flip.  Below the slot index
// in bits 32 and up, one sort orders every slot's rows by time as the single form's sort orders the scan's, stably.
__device__ __forceinline__ unsigned twiddle_f32(float t) {
    unsigned b = __float_as_uint(t);
    if (b == 0x80000000u) b = 0u;
    return b ^ ((b & 0x80000000u) ? 0xFFFFFFFFu : 0x80000000u);
}
// the float a sorted key stands for; -0.0 comes back as +0.0, which k_undistort's arithmetic cannot tell apart (the time only
// enters through t > head[0], true for neither zero against any head, and t - head[0] of a point older than its head)
__device__ __forceinline__ float untwiddle_f32(unsigned k) { return __uint_as_float(k ^ ((k & 0x80000000u) ? 0x80000000u : 0xFFFFFFFFu)); }

__device__ __forceinline__ bool misaligned(const void* p, unsigned align) { return (reinterpret_cast<uintptr_t>(p) & (align - 1)) != 0; }

// fl_scan_batch_run_device's first step, k_upload_n per slot: the slot's refusal is decided, its first c rows are copied into the
// packed buffer and, when de-skewing, their time keys written, the padding rows carrying the padding time (0x7FFFFFFF, whose key
// 0xFFFFFFFF sorts after every real row of the slot).  Thread 0 of each slot resets its voxel grid and writes its ref-table
// entries; block (0, 0) also sets the counts of the slots [n_scans, n_scans_max) to -1.
__global__ void k_batch_gather(const fl_scan_raw_t* __restrict__ raws, int n_scans, int n_scans_max, int n_max, int n_pose_max, int undistort,
                               float4* __restrict__ raw, unsigned long long* __restrict__ keys, const float4* sraw, const float4* down,
                               BatchSlot* __restrict__ slots, fl_scan_ref_t* __restrict__ refs, int* __restrict__ counts) {
    const int s = blockIdx.y;
    const fl_scan_raw_t r = raws[s];
    int err = FL_OK, c = 0;
    if (!r.n || misaligned(r.n, 4)) err = FL_ERR_ARG;
    else {
        c = *r.n;
        if (c < 0) err = FL_ERR_ARG;
        else if (c > n_max) err = FL_ERR_CAPACITY;
        else if (c > 0 && (!r.xyzi || misaligned(r.xyzi, 16) || !r.offset_ms || misaligned(r.offset_ms, 4))) err = FL_ERR_ARG;
        else if (undistort) {
            if (!r.x26_end || misaligned(r.x26_end, 8) || misaligned(r.n_pose, 4)) err = FL_ERR_ARG;
            else if (r.n_pose && min(max(*r.n_pose, 0), n_pose_max) >= 2 && (!r.imu_pose22 || misaligned(r.imu_pose22, 8))) err = FL_ERR_ARG;
        }
    }
    if (err != FL_OK) c = 0;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const size_t row = (size_t)s * n_max + i;
    if (i == 0) {
        BatchSlot& b = slots[s];
        for (int a = 0; a < 3; a++) { b.vg.mn[a] = FLT_MAX; b.vg.mx[a] = -FLT_MAX; }
        b.vg.total = 0; b.vg.passthrough = 0;
        b.n = c; b.err = err;
        const size_t base = (size_t)s * n_max;
        refs[s].body_xyzi = reinterpret_cast<const float*>((undistort ? sraw : raw) + base);
        refs[s].n = counts + s;
        refs[n_scans_max + s].body_xyzi = reinterpret_cast<const float*>(down + base);
        refs[n_scans_max + s].n = counts + n_scans_max + s;
        counts[s] = err == FL_OK ? c : -1;
        counts[n_scans_max + s] = -1;                       // k_batch_commit writes feats_down_size
    }
    if (s == 0 && blockIdx.x == 0)
        for (int t = n_scans + threadIdx.x; t < n_scans_max; t += blockDim.x) counts[t] = counts[n_scans_max + t] = -1;
    if (i >= n_max) return;
    if (i < c) raw[row] = reinterpret_cast<const float4*>(r.xyzi)[i];
    if (undistort) keys[row] = ((unsigned long long)s << 32) | (i < c ? twiddle_f32(r.offset_ms[i]) : 0xFFFFFFFFu);
}

// k_undistort per slot over the time-sorted rows: each block belongs to one slot and loads that slot's poses into shared memory
__global__ void k_batch_undistort(float4* __restrict__ pts, const unsigned long long* __restrict__ keys, int n_max,
                                  const fl_scan_raw_t* __restrict__ raws, int n_pose_max, const BatchSlot* __restrict__ slots) {
    extern __shared__ double s_pose[];
    const int s = blockIdx.y;
    if (slots[s].err != FL_OK) return;
    const fl_scan_raw_t r = raws[s];
    const int n_pose = r.n_pose ? min(max(*r.n_pose, 0), n_pose_max) : 0;
    if (n_pose < 2) return;                                 // no segment: the points stay as sorted
    const int n = slots[s].n;
    for (int i = threadIdx.x; i < n_pose * POSE_DOUBLES; i += blockDim.x) s_pose[i] = r.imu_pose22[i];
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const EndState e = end_state(r.x26_end);
    const size_t base = (size_t)s * n_max;
    undistort_row(pts + base, i, double(untwiddle_f32(unsigned(keys[base + i]))) / double(1000), s_pose, n_pose, e);
}

__global__ void k_batch_minmax(const float4* __restrict__ pts, int n_max, BatchSlot* slots) {
    const int s = blockIdx.y;
    vg_minmax_block(pts + (size_t)s * n_max, slots[s].n, &slots[s].vg, blockIdx.x, gridDim.x);
}

// k_vg_keys per slot, the slot index above the 32-bit key; the values are global rows
__global__ void k_batch_keys(const float4* __restrict__ pts, int n_max, float leaf, BatchSlot* slots, unsigned long long* __restrict__ keys,
                             int* __restrict__ vals) {
    const int s = blockIdx.y;
    const VgGrid g = vg_grid(&slots[s].vg, leaf);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) slots[s].vg.passthrough = g.overflow ? 1 : 0;
    if (i >= n_max) return;
    const size_t row = (size_t)s * n_max + i;
    keys[row] = ((unsigned long long)s << 32) | (i < slots[s].n ? vg_key(pts[row], g, i) : 0xFFFFFFFFu);
    vals[row] = (int)row;
}

// k_vg_heads per slot: the heads restart at each slot's first row, padding rows are none
__global__ void k_batch_heads(const unsigned long long* __restrict__ keys, int n_max, const BatchSlot* __restrict__ slots, int* __restrict__ heads) {
    const int s = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_max) return;
    const size_t row = (size_t)s * n_max + i;
    heads[row] = (i < slots[s].n && (i == 0 || keys[row] != keys[row - 1])) ? 1 : 0;
}

// k_vg_centroid per slot: positions of the one exclusive scan over every slot, less the slot's first; rows at s * n_max + position
__global__ void k_batch_centroid(const float4* __restrict__ pts, const unsigned long long* __restrict__ keys, const int* __restrict__ vals,
                                 const int* __restrict__ heads, const int* __restrict__ pos, int n_max, float4* __restrict__ out, BatchSlot* slots) {
    const int s = blockIdx.y;
    const int n = slots[s].n;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const size_t base = (size_t)s * n_max;
    const int at = pos[base + i] - pos[base];
    if (i == n - 1) slots[s].vg.total = at + heads[base + i];
    if (!heads[base + i]) return;
    out[base + at] = vg_run(pts, keys + base, vals + base, i, n);
}

// status2 = (FL_OK, feats_down_size) and the count of ref table 1, or (refusal, 0) and -1
__global__ void k_batch_commit(const BatchSlot* __restrict__ slots, int n_scans, int n_scans_max, int* __restrict__ counts, int* __restrict__ status2) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_scans) return;
    const int err = slots[s].err, total = err == FL_OK ? slots[s].vg.total : 0;
    counts[n_scans_max + s] = err == FL_OK ? total : -1;
    status2[2 * s] = err;
    status2[2 * s + 1] = total;
}

}  // namespace

// ================================================================================================ ScanFrontEnd
ScanFrontEnd::~ScanFrontEnd() {
    cudaSetDevice(map_->device());
    DeviceBuffer* all[] = {&raw_, &raw_alt_, &time_, &time_alt_, &down_, &keys_, &keys_alt_, &vals_, &vals_alt_, &heads_, &pos_, &cub_tmp_, &ctl_, &poses_,
                           &frame_out_, &frame_x_,
                           &d_raw_, &d_time_, &d_sraw_, &d_stime_, &d_down_, &d_keys_, &d_keys_alt_, &d_vals_, &d_vals_alt_, &d_heads_, &d_pos_,
                           &d_cub_, &d_ctl_};
    for (DeviceBuffer* b : all) b->release();
    if (h_count_) cudaFreeHost(h_count_);
    if (h_dctl_) cudaFreeHost(h_dctl_);
}

// k_undistort's dynamic shared memory above the default 48 KB: the attribute only grows, so a launch the host form or
// fl_scan_reserve allowed stays allowed (a captured graph keeps launching with the size of capture time)
int ScanFrontEnd::undistort_smem(size_t smem) {
    if (smem <= undistort_smem_) return FL_OK;
    FL_CUDA(cudaFuncSetAttribute(k_undistort, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    undistort_smem_ = smem;
    return FL_OK;
}

int ScanFrontEnd::init() {
    FL_CUDA(cudaSetDevice(map_->device()));
    FL_CHECK(ctl_.reserve(sizeof(VgCtl)));
    FL_CUDA(cudaMallocHost(&h_count_, sizeof(int)));
    return FL_OK;
}

int ScanFrontEnd::upload(const float* xyzi, const float* offset_ms, int n) {
    if (n < 0 || (n > 0 && (!xyzi || !offset_ms))) { set_last_error("scan upload: bad arguments"); return FL_ERR_ARG; }
    FL_CUDA(cudaSetDevice(map_->device()));
    const size_t m = (size_t)std::max(1, n);
    FL_CHECK(raw_.reserve(sizeof(float4) * m));
    FL_CHECK(time_.reserve(sizeof(float) * m));
    if (n > 0) {
        FL_CUDA(cudaMemcpyAsync(raw_.ptr, xyzi, sizeof(float4) * (size_t)n, cudaMemcpyHostToDevice, map_->stream()));
        FL_CUDA(cudaMemcpyAsync(time_.ptr, offset_ms, sizeof(float) * (size_t)n, cudaMemcpyHostToDevice, map_->stream()));
    }
    n_raw_ = n;
    n_down_ = 0;
    dev_uploaded_ = dev_undistorted_ = dev_down_ = false;      // the device forms' cloud is no longer the scan's
    return FL_OK;
}

int ScanFrontEnd::undistort(const double* poses, int n_pose, const double* x26_end) {
    if (n_pose < 0 || (n_pose > 0 && !poses) || !x26_end) { set_last_error("undistort: bad arguments"); return FL_ERR_ARG; }
    dev_uploaded_ = dev_undistorted_ = dev_down_ = false;      // the host forms now hold the scan's cloud: device forms upload anew
    const int n = n_raw_;
    if (n == 0) return FL_OK;
    FL_CUDA(cudaSetDevice(map_->device()));
    cudaStream_t st = map_->stream();
    // sort(pcl_out.points.begin(), pcl_out.points.end(), time_list)  (:234) -- stable here
    FL_CHECK(raw_alt_.reserve(sizeof(float4) * (size_t)n));
    FL_CHECK(time_alt_.reserve(sizeof(float) * (size_t)n));
    size_t tmp = 0;
    FL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp, time_.as<float>(), time_alt_.as<float>(), raw_.as<float4>(), raw_alt_.as<float4>(), n, 0, 32, st));
    FL_CHECK(cub_tmp_.reserve(tmp));
    FL_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp_.ptr, tmp, time_.as<float>(), time_alt_.as<float>(), raw_.as<float4>(), raw_alt_.as<float4>(), n, 0, 32, st));
    std::swap(raw_, raw_alt_);
    std::swap(time_, time_alt_);
    if (n_pose < 2) return FL_OK;                       // no segment: the backward sweep has nothing to walk
    const size_t np = (size_t)n_pose * POSE_DOUBLES;
    const size_t smem = sizeof(double) * np;
    if (smem > UNDISTORT_SMEM_MAX) { set_last_error("undistort: %d IMU poses do not fit shared memory", n_pose); return FL_ERR_CAPACITY; }
    // a few KB from pageable host memory: the runtime stages them before returning, the caller's arrays are free at once
    FL_CHECK(poses_.reserve(sizeof(double) * (np + XLEN)));
    FL_CUDA(cudaMemcpyAsync(poses_.ptr, poses, sizeof(double) * np, cudaMemcpyHostToDevice, st));
    FL_CUDA(cudaMemcpyAsync(poses_.as<double>() + np, x26_end, sizeof(double) * XLEN, cudaMemcpyHostToDevice, st));
    FL_CHECK(undistort_smem(smem));
    const int block = 128;
    k_undistort<<<(n + block - 1) / block, block, smem, st>>>(raw_.as<float4>(), time_.as<float>(), n, poses_.as<double>(), n_pose,
                                                              poses_.as<double>() + (size_t)n_pose * POSE_DOUBLES, nullptr, nullptr, nullptr);
    FL_CUDA(cudaGetLastError());
    return FL_OK;
}

int ScanFrontEnd::voxel_downsample(float leaf, int* n_out) {
    if (n_out) *n_out = 0;
    if (!(leaf > 0.f)) { set_last_error("voxel_downsample: leaf size must be > 0"); return FL_ERR_ARG; }
    dev_uploaded_ = dev_undistorted_ = dev_down_ = false;      // the host forms now hold the scan's cloud: device forms upload anew
    const int n = n_raw_;
    n_down_ = 0;
    if (n == 0) return FL_OK;
    FL_CUDA(cudaSetDevice(map_->device()));
    cudaStream_t st = map_->stream();
    FL_CHECK(down_.reserve(sizeof(float4) * (size_t)n));
    FL_CHECK(keys_.reserve(sizeof(unsigned) * (size_t)n));
    FL_CHECK(keys_alt_.reserve(sizeof(unsigned) * (size_t)n));
    FL_CHECK(vals_.reserve(sizeof(int) * (size_t)n));
    FL_CHECK(vals_alt_.reserve(sizeof(int) * (size_t)n));
    FL_CHECK(heads_.reserve(sizeof(int) * (size_t)n));
    FL_CHECK(pos_.reserve(sizeof(int) * (size_t)n));
    VgCtl* ctl = ctl_.as<VgCtl>();
    const int block = 256, grid = (n + block - 1) / block;
    k_vg_reset<<<1, 32, 0, st>>>(ctl, nullptr);
    k_vg_minmax<<<std::min(grid, 132), block, 0, st>>>(raw_.as<float4>(), n, ctl, nullptr);
    k_vg_keys<<<grid, block, 0, st>>>(raw_.as<float4>(), n, leaf, ctl, keys_.as<unsigned>(), vals_.as<int>(), nullptr);
    size_t tmp_sort = 0, tmp_scan = 0;
    FL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, keys_.as<unsigned>(), keys_alt_.as<unsigned>(), vals_.as<int>(), vals_alt_.as<int>(), n, 0, 32, st));
    FL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_scan, heads_.as<int>(), pos_.as<int>(), n, st));
    FL_CHECK(cub_tmp_.reserve(std::max(tmp_sort, tmp_scan)));
    FL_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp_.ptr, tmp_sort, keys_.as<unsigned>(), keys_alt_.as<unsigned>(), vals_.as<int>(), vals_alt_.as<int>(), n, 0, 32, st));
    k_vg_heads<<<grid, block, 0, st>>>(keys_alt_.as<unsigned>(), n, heads_.as<int>(), nullptr);
    FL_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp_.ptr, tmp_scan, heads_.as<int>(), pos_.as<int>(), n, st));
    k_vg_centroid<<<grid, block, 0, st>>>(raw_.as<float4>(), keys_alt_.as<unsigned>(), vals_alt_.as<int>(), heads_.as<int>(), pos_.as<int>(), n,
                                          down_.as<float4>(), ctl, nullptr);
    FL_CUDA(cudaGetLastError());
    FL_CUDA(cudaMemcpyAsync(h_count_, &ctl->total, sizeof(int), cudaMemcpyDeviceToHost, st));
    FL_CUDA(cudaStreamSynchronize(st));
    n_down_ = *h_count_;
    if (n_out) *n_out = n_down_;
    return FL_OK;
}

int ScanFrontEnd::download(int which, float* out_xyzi, int cap, int* n) {
    const int have = which == 0 ? n_raw_ : n_down_;
    if (n) *n = have;
    if (which != 0 && which != 1) { set_last_error("scan download: which must be 0 or 1"); return FL_ERR_ARG; }
    const int take = std::min(have, cap);
    if (take <= 0) return FL_OK;
    if (!out_xyzi) { set_last_error("scan download: null buffer"); return FL_ERR_ARG; }
    FL_CUDA(cudaSetDevice(map_->device()));
    const void* src = which == 0 ? raw_.ptr : down_.ptr;
    FL_CUDA(cudaMemcpyAsync(out_xyzi, src, sizeof(float4) * (size_t)take, cudaMemcpyDeviceToHost, map_->stream()));
    FL_CUDA(cudaStreamSynchronize(map_->stream()));
    return FL_OK;
}

// the current cloud through k_frame into frame_out_, then read back (the kernel of the device form, so the bytes are the same)
int ScanFrontEnd::frame(int which, int frame, const double* x26, float* out_xyzi, int cap, int* n) {
    const int have = which == 0 ? n_raw_ : n_down_;
    if (n) *n = have;
    if ((which != 0 && which != 1) || frame < FL_FRAME_LIDAR || frame > FL_FRAME_WORLD || (frame != FL_FRAME_LIDAR && !x26)) {
        set_last_error("scan frame: which must be 0 or 1, frame FL_FRAME_LIDAR / IMU / WORLD, and x26 non-null outside FL_FRAME_LIDAR");
        return FL_ERR_ARG;
    }
    const int take = std::min(have, cap);
    if (take <= 0) return FL_OK;
    if (!out_xyzi) { set_last_error("scan frame: null buffer"); return FL_ERR_ARG; }
    FL_CUDA(cudaSetDevice(map_->device()));
    cudaStream_t st = map_->stream();
    FL_CHECK(frame_out_.reserve(sizeof(float4) * (size_t)take));
    FL_CHECK(frame_x_.reserve(sizeof(double) * XLEN));
    if (frame != FL_FRAME_LIDAR) FL_CUDA(cudaMemcpyAsync(frame_x_.ptr, x26, sizeof(double) * XLEN, cudaMemcpyHostToDevice, st));
    const int block = 256;
    k_frame<<<(take + block - 1) / block, block, 0, st>>>(which == 0 ? raw_.as<float4>() : down_.as<float4>(), take, nullptr,
                                                          frame_x_.as<double>(), frame, frame_out_.as<float4>(), nullptr, take);
    FL_CUDA(cudaGetLastError());
    FL_CUDA(cudaMemcpyAsync(out_xyzi, frame_out_.ptr, sizeof(float4) * (size_t)take, cudaMemcpyDeviceToHost, st));
    FL_CUDA(cudaStreamSynchronize(st));
    return FL_OK;
}

// ------------------------------------------------------------------------------------------------ device forms
// They own a fixed set of buffers, sized here and never by the calls themselves, and never swap them: a captured graph keeps
// reading and writing the buffers of capture time, whatever host-form calls (which grow and swap their own buffers) ran since.
int ScanFrontEnd::reserve_device(int n_max, int n_pose_max) {
    if (n_max < 0 || n_pose_max < 0) { set_last_error("scan reserve: n_max and n_pose_max must be >= 0"); return FL_ERR_ARG; }
    const size_t smem = sizeof(double) * POSE_DOUBLES * (size_t)n_pose_max;
    if (smem > UNDISTORT_SMEM_MAX) { set_last_error("scan reserve: %d IMU poses do not fit shared memory", n_pose_max); return FL_ERR_CAPACITY; }
    FL_CUDA(cudaSetDevice(map_->device()));
    const size_t m = (size_t)std::max(1, n_max);
    FL_CHECK(d_raw_.reserve(sizeof(float4) * m));
    FL_CHECK(d_sraw_.reserve(sizeof(float4) * m));
    FL_CHECK(d_down_.reserve(sizeof(float4) * m));
    FL_CHECK(d_time_.reserve(sizeof(float) * m));
    FL_CHECK(d_stime_.reserve(sizeof(float) * m));
    FL_CHECK(d_keys_.reserve(sizeof(unsigned) * m));
    FL_CHECK(d_keys_alt_.reserve(sizeof(unsigned) * m));
    FL_CHECK(d_vals_.reserve(sizeof(int) * m));
    FL_CHECK(d_vals_alt_.reserve(sizeof(int) * m));
    FL_CHECK(d_heads_.reserve(sizeof(int) * m));
    FL_CHECK(d_pos_.reserve(sizeof(int) * m));
    size_t t_time = 0, t_vg = 0, t_scan = 0;
    FL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t_time, (const float*)nullptr, (float*)nullptr, (const float4*)nullptr, (float4*)nullptr, (int)m));
    FL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t_vg, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr, (int*)nullptr, (int)m));
    FL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, t_scan, (const int*)nullptr, (int*)nullptr, (int)m));
    FL_CHECK(d_cub_.reserve(std::max(t_time, std::max(t_vg, t_scan))));
    if (!d_ctl_.ptr) {
        FL_CHECK(d_ctl_.reserve(sizeof(ScanDevCtl)));
        FL_CUDA(cudaMemsetAsync(d_ctl_.ptr, 0, sizeof(ScanDevCtl), map_->stream()));
        FL_CUDA(cudaMallocHost(&h_dctl_, sizeof(ScanDevCtl)));
    }
    FL_CHECK(undistort_smem(smem));
    FL_CUDA(cudaStreamSynchronize(map_->stream()));
    res_n_max_ = std::max(res_n_max_, n_max);
    res_pose_max_ = std::max(res_pose_max_, n_pose_max);
    dev_used_ = true;
    return FL_OK;
}

const float4* ScanFrontEnd::down_dev() const { return d_down_.as<float4>(); }
const int* ScanFrontEnd::down_count_dev() const { return &d_ctl_.as<ScanDevCtl>()->vg.total; }

// cub's temporary storage for `n` rows within what reserve_device sized
int ScanFrontEnd::cub_fits(int n, const char* what) const {
    size_t t_time = 0, t_vg = 0, t_scan = 0;
    FL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t_time, (const float*)nullptr, (float*)nullptr, (const float4*)nullptr, (float4*)nullptr, n));
    FL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t_vg, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr, (int*)nullptr, n));
    FL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, t_scan, (const int*)nullptr, (int*)nullptr, n));
    if (std::max(t_time, std::max(t_vg, t_scan)) > d_cub_.bytes) {
        set_last_error("%s: %d rows exceed what fl_scan_reserve sized", what, n);
        return FL_ERR_CAPACITY;
    }
    return FL_OK;
}

int ScanFrontEnd::upload_on_stream(const float* d_xyzi, const float* d_offset_ms, const int* d_n, int n_max, cudaStream_t st) {
    const int dev = map_->device();
    if (n_max < 0 || !device_ptr(d_n, dev, 4) || (n_max > 0 && (!device_ptr(d_xyzi, dev, 16) || !device_ptr(d_offset_ms, dev, 4)))) {
        set_last_error("scan upload_device: n_max < 0, or a buffer is not device memory on device %d (points 16-byte, offset times and "
                       "n 4-byte aligned)", dev);
        return FL_ERR_ARG;
    }
    if (!d_ctl_.ptr || n_max > res_n_max_) {
        set_last_error("scan upload_device: n_max = %d exceeds the %d rows fl_scan_reserve sized", n_max, d_ctl_.ptr ? res_n_max_ : 0);
        return FL_ERR_CAPACITY;
    }
    FL_CUDA(cudaSetDevice(dev));
    bool joined = false;
    FL_CHECK(map_->query_begin(st, &joined));
    const int block = 256;
    k_upload_n<<<std::max(1, (n_max + block - 1) / block), block, 0, st>>>(reinterpret_cast<const float4*>(d_xyzi), d_offset_ms, d_n, n_max,
                                                                            d_raw_.as<float4>(), d_time_.as<float>(), d_ctl_.as<ScanDevCtl>());
    FL_CHECK(map_->query_end(st, joined));
    dev_n_max_ = n_max;
    dev_uploaded_ = true;
    dev_undistorted_ = false;
    dev_down_ = false;
    return FL_OK;
}

int ScanFrontEnd::undistort_on_stream(const double* d_poses, const int* d_n_pose, int n_pose_max, const double* d_x26_end, cudaStream_t st) {
    const int dev = map_->device();
    if (n_pose_max < 0 || !device_ptr(d_n_pose, dev, 4) || !device_ptr(d_x26_end, dev, 8) || (n_pose_max > 0 && !device_ptr(d_poses, dev, 8))) {
        set_last_error("scan undistort_device: n_pose_max < 0, or a buffer is not device memory on device %d (poses and x 8-byte, "
                       "n_pose 4-byte aligned)", dev);
        return FL_ERR_ARG;
    }
    if (!dev_uploaded_) { set_last_error("scan undistort_device: no fl_scan_upload_device since the last host-form upload"); return FL_ERR_STATE; }
    const size_t smem = sizeof(double) * POSE_DOUBLES * (size_t)n_pose_max;
    if (n_pose_max > res_pose_max_ || smem > UNDISTORT_SMEM_MAX) {
        set_last_error("scan undistort_device: n_pose_max = %d exceeds the %d poses fl_scan_reserve sized", n_pose_max, res_pose_max_);
        return FL_ERR_CAPACITY;
    }
    const int n = dev_n_max_;
    FL_CHECK(cub_fits(n, "scan undistort_device"));
    FL_CUDA(cudaSetDevice(dev));
    bool joined = false;
    FL_CHECK(map_->query_begin(st, &joined));
    // the stable time sort of n_max rows (the padding rows last, see k_upload_n), then the backward pass over the first n
    size_t tmp = d_cub_.bytes;
    FL_CUDA(cub::DeviceRadixSort::SortPairs(d_cub_.ptr, tmp, d_time_.as<float>(), d_stime_.as<float>(), d_raw_.as<float4>(), d_sraw_.as<float4>(),
                                            n, 0, 32, st));
    const int block = 128;
    ScanDevCtl* c = d_ctl_.as<ScanDevCtl>();
    k_undistort<<<std::max(1, (n + block - 1) / block), block, smem, st>>>(d_sraw_.as<float4>(), d_stime_.as<float>(), n, d_poses, n_pose_max,
                                                                           d_x26_end, &c->n_raw, d_n_pose, c);
    FL_CHECK(map_->query_end(st, joined));
    dev_undistorted_ = true;
    return FL_OK;
}

int ScanFrontEnd::voxel_downsample_on_stream(float leaf, int* d_n_out, cudaStream_t st) {
    const int dev = map_->device();
    if (!(leaf > 0.f)) { set_last_error("voxel_downsample_device: leaf size must be > 0"); return FL_ERR_ARG; }
    if (d_n_out && !device_ptr(d_n_out, dev, 4)) { set_last_error("voxel_downsample_device: n_out must be 4-byte aligned device memory on device %d", dev); return FL_ERR_ARG; }
    if (!dev_uploaded_) { set_last_error("voxel_downsample_device: no fl_scan_upload_device since the last host-form upload"); return FL_ERR_STATE; }
    const int n = dev_n_max_;
    FL_CHECK(cub_fits(n, "voxel_downsample_device"));
    FL_CUDA(cudaSetDevice(dev));
    bool joined = false;
    FL_CHECK(map_->query_begin(st, &joined));
    ScanDevCtl* c = d_ctl_.as<ScanDevCtl>();
    VgCtl* ctl = &c->vg;
    const int* cnt = &c->n_raw;
    const float4* src = dev_undistorted_ ? d_sraw_.as<float4>() : d_raw_.as<float4>();
    unsigned *keys = d_keys_.as<unsigned>(), *keys_alt = d_keys_alt_.as<unsigned>();
    int *vals = d_vals_.as<int>(), *vals_alt = d_vals_alt_.as<int>(), *heads = d_heads_.as<int>(), *pos = d_pos_.as<int>();
    const int block = 256, grid = std::max(1, (n + block - 1) / block);
    k_vg_reset<<<1, 32, 0, st>>>(ctl, c);
    k_vg_minmax<<<std::min(grid, 132), block, 0, st>>>(src, n, ctl, cnt);
    k_vg_keys<<<grid, block, 0, st>>>(src, n, leaf, ctl, keys, vals, cnt);
    size_t tmp = d_cub_.bytes;
    FL_CUDA(cub::DeviceRadixSort::SortPairs(d_cub_.ptr, tmp, keys, keys_alt, vals, vals_alt, n, 0, 32, st));
    k_vg_heads<<<grid, block, 0, st>>>(keys_alt, n, heads, cnt);
    tmp = d_cub_.bytes;
    FL_CUDA(cub::DeviceScan::ExclusiveSum(d_cub_.ptr, tmp, heads, pos, n, st));
    k_vg_centroid<<<grid, block, 0, st>>>(src, keys_alt, vals_alt, heads, pos, n, d_down_.as<float4>(), ctl, cnt);
    FL_CUDA(cudaGetLastError());
    if (d_n_out) FL_CUDA(cudaMemcpyAsync(d_n_out, &ctl->total, sizeof(int), cudaMemcpyDeviceToDevice, st));
    FL_CHECK(map_->query_end(st, joined));
    dev_down_ = true;
    return FL_OK;
}

int ScanFrontEnd::frame_on_stream(int which, int frame, const double* d_x26, float* d_out, int* d_n_io, int cap, int* d_status2,
                                  cudaStream_t st) {
    const int dev = map_->device();
    if ((which != 0 && which != 1) || frame < FL_FRAME_LIDAR || frame > FL_FRAME_WORLD || cap < 0) {
        set_last_error("scan frame_device: which must be 0 or 1, frame FL_FRAME_LIDAR / IMU / WORLD, and cap >= 0");
        return FL_ERR_ARG;
    }
    if (!device_ptr(d_out, dev, 16) || !device_ptr(d_n_io, dev, 4) || !device_ptr(d_status2, dev, 4) ||
        ((frame != FL_FRAME_LIDAR || d_x26) && !device_ptr(d_x26, dev, 8))) {
        set_last_error("scan frame_device: a buffer is not device memory on device %d (out 16-byte, x 8-byte, n_io and status "
                       "4-byte aligned; x may be null only for FL_FRAME_LIDAR)", dev);
        return FL_ERR_ARG;
    }
    if (!dev_uploaded_) { set_last_error("scan frame_device: no fl_scan_upload_device since the last host-form upload, undistort or down-sample"); return FL_ERR_STATE; }
    if (which == 1 && !dev_down_) { set_last_error("scan frame_device: no fl_scan_voxel_downsample_device since the last device-form upload"); return FL_ERR_STATE; }
    const int n = dev_n_max_;
    ScanDevCtl* c = d_ctl_.as<ScanDevCtl>();
    const float4* src = which == 1 ? d_down_.as<float4>() : dev_undistorted_ ? d_sraw_.as<float4>() : d_raw_.as<float4>();
    const int* cnt = which == 1 ? &c->vg.total : &c->n_raw;
    FL_CUDA(cudaSetDevice(dev));
    bool joined = false;
    FL_CHECK(map_->query_begin(st, &joined));
    const int block = 256;
    k_frame<<<std::max(1, (n + block - 1) / block), block, 0, st>>>(src, n, cnt, d_x26, frame, reinterpret_cast<float4*>(d_out), d_n_io, cap);
    k_frame_commit<<<1, 1, 0, st>>>(cnt, n, d_n_io, cap, d_status2);
    FL_CUDA(cudaGetLastError());
    return map_->query_end(st, joined);
}

// Host forms after device forms: when the device forms produced the current cloud (their upload ran after the host forms' last
// one, directly or in a graph replay), its counts are read back and its clouds copied into the host forms' buffers, so the host
// forms continue from exactly the state the host-form chain would have left.  One read-back per host-form call once the device
// forms are in use; none before.
int ScanFrontEnd::settle() {
    if (!dev_used_) return FL_OK;
    FL_CUDA(cudaSetDevice(map_->device()));
    cudaStream_t st = map_->stream();
    FL_CUDA(cudaMemcpyAsync(h_dctl_, d_ctl_.ptr, sizeof(ScanDevCtl), cudaMemcpyDeviceToHost, st));
    FL_CUDA(cudaStreamSynchronize(st));
    const ScanDevCtl h = *static_cast<const ScanDevCtl*>(h_dctl_);
    if (!h.src) return FL_OK;
    const int n = h.n_raw;
    FL_CHECK(raw_.reserve(sizeof(float4) * (size_t)std::max(1, n)));
    FL_CHECK(time_.reserve(sizeof(float) * (size_t)std::max(1, n)));
    if (n > 0) {
        FL_CUDA(cudaMemcpyAsync(raw_.ptr, h.stage ? d_sraw_.ptr : d_raw_.ptr, sizeof(float4) * (size_t)n, cudaMemcpyDeviceToDevice, st));
        FL_CUDA(cudaMemcpyAsync(time_.ptr, h.stage ? d_stime_.ptr : d_time_.ptr, sizeof(float) * (size_t)n, cudaMemcpyDeviceToDevice, st));
    }
    n_raw_ = n;
    n_down_ = h.down ? h.vg.total : 0;
    if (n_down_ > 0) {
        FL_CHECK(down_.reserve(sizeof(float4) * (size_t)n_down_));
        FL_CUDA(cudaMemcpyAsync(down_.ptr, d_down_.ptr, sizeof(float4) * (size_t)n_down_, cudaMemcpyDeviceToDevice, st));
    }
    FL_CUDA(cudaMemsetAsync(&d_ctl_.as<ScanDevCtl>()->src, 0, sizeof(int), st));
    return FL_OK;
}

// ================================================================================================ ScanBatch
ScanBatch::~ScanBatch() {
    cudaSetDevice(map_->device());
    DeviceBuffer* all[] = {&raw_, &sraw_, &down_, &keys_, &keys_alt_, &vals_, &vals_alt_, &heads_, &pos_, &cub_, &slots_, &refs_, &counts_};
    for (DeviceBuffer* b : all) b->release();
}

namespace {
// the bits the slot index takes above the 32-bit keys of n_scans slots
int slot_bits(int n_scans) {
    int b = 0;
    while ((1ll << b) < (long long)n_scans) b++;
    return b;
}
}  // namespace

// cub's temporary storage for both sorts and the scan over `rows` packed rows, the sorts on bits [0, end_bit)
int ScanBatch::cub_bytes(int rows, int end_bit, size_t* bytes) const {
    using U64 = unsigned long long;
    size_t t_time = 0, t_vg = 0, t_scan = 0;
    FL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t_time, (const U64*)nullptr, (U64*)nullptr, (const float4*)nullptr, (float4*)nullptr, rows, 0, end_bit));
    FL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t_vg, (const U64*)nullptr, (U64*)nullptr, (const int*)nullptr, (int*)nullptr, rows, 0, end_bit));
    FL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, t_scan, (const int*)nullptr, (int*)nullptr, rows));
    *bytes = std::max(t_time, std::max(t_vg, t_scan));
    return FL_OK;
}

int ScanBatch::reserve(int n_scans_max, int n_max, int n_pose_max) {
    if (n_scans_max < 0 || n_max < 0 || n_pose_max < 0) {
        set_last_error("scan batch reserve: n_scans_max, n_max and n_pose_max must be >= 0");
        return FL_ERR_ARG;
    }
    const int S = std::max(res_slots_, n_scans_max), m = std::max(res_n_max_, n_max), np = std::max(res_pose_max_, n_pose_max);
    const size_t smem = sizeof(double) * POSE_DOUBLES * (size_t)np;
    if (smem > UNDISTORT_SMEM_MAX || S > SLOTS_MAX || (long long)S * m > (long long)INT_MAX) {
        set_last_error("scan batch reserve: %d IMU poses (shared memory holds %d), %d slots (at most %d) or %lld rows (at most INT_MAX)", np,
                       (int)(UNDISTORT_SMEM_MAX / (sizeof(double) * POSE_DOUBLES)), S, SLOTS_MAX, (long long)S * m);
        return FL_ERR_CAPACITY;
    }
    if (reserved_ && S == res_slots_ && m == res_n_max_ && np == res_pose_max_) return FL_OK;
    FL_CUDA(cudaSetDevice(map_->device()));
    FL_CUDA(cudaStreamSynchronize(map_->stream()));
    const size_t rows = (size_t)std::max(1, S * m), slots = (size_t)std::max(1, S);
    FL_CHECK(raw_.reserve(sizeof(float4) * rows));
    FL_CHECK(sraw_.reserve(sizeof(float4) * rows));
    FL_CHECK(down_.reserve(sizeof(float4) * rows));
    FL_CHECK(keys_.reserve(sizeof(unsigned long long) * rows));
    FL_CHECK(keys_alt_.reserve(sizeof(unsigned long long) * rows));
    FL_CHECK(vals_.reserve(sizeof(int) * rows));
    FL_CHECK(vals_alt_.reserve(sizeof(int) * rows));
    FL_CHECK(heads_.reserve(sizeof(int) * rows));
    FL_CHECK(pos_.reserve(sizeof(int) * rows));
    size_t tmp = 0;
    FL_CHECK(cub_bytes((int)rows, 32 + slot_bits(S), &tmp));
    FL_CHECK(cub_.reserve(tmp));
    FL_CHECK(slots_.reserve(sizeof(BatchSlot) * slots));
    FL_CHECK(refs_.reserve(sizeof(fl_scan_ref_t) * 2 * slots));
    FL_CHECK(counts_.reserve(sizeof(int) * 2 * slots));
    // table 0 then table 1, n_scans_max entries each; every entry starts as a slot with no rows (count -1)
    std::vector<fl_scan_ref_t> t(2 * slots);
    for (size_t s = 0; s < slots; s++) {
        t[s].body_xyzi = reinterpret_cast<const float*>(raw_.as<float4>() + s * m);
        t[s].n = counts_.as<int>() + s;
        t[slots + s].body_xyzi = reinterpret_cast<const float*>(down_.as<float4>() + s * m);
        t[slots + s].n = counts_.as<int>() + slots + s;
    }
    FL_CUDA(cudaMemcpyAsync(refs_.ptr, t.data(), sizeof(fl_scan_ref_t) * 2 * slots, cudaMemcpyHostToDevice, map_->stream()));
    FL_CUDA(cudaMemsetAsync(counts_.ptr, 0xFF, sizeof(int) * 2 * slots, map_->stream()));
    if (smem > undistort_smem_) {
        FL_CUDA(cudaFuncSetAttribute(k_batch_undistort, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        undistort_smem_ = smem;
    }
    FL_CUDA(cudaStreamSynchronize(map_->stream()));
    res_slots_ = (int)slots;
    res_n_max_ = m;
    res_pose_max_ = np;
    reserved_ = true;
    return FL_OK;
}

int ScanBatch::run_on_stream(const fl_scan_raw_t* d_raws, int n_scans, int n_max, int n_pose_max, int undistort, float leaf, int* d_status2,
                             cudaStream_t st) {
    const int dev = map_->device();
    if (n_scans < 0 || n_max < 0 || n_pose_max < 0 || !(leaf > 0.f) || (undistort != 0 && undistort != 1) ||
        (n_scans > 0 && (!device_ptr(d_raws, dev, 8) || !device_ptr(d_status2, dev, 4)))) {
        set_last_error("scan batch run_device: n_scans, n_max or n_pose_max < 0, leaf not > 0, undistort not 0 or 1, or a buffer is not "
                       "device memory on device %d (table 8-byte, status 4-byte aligned)", dev);
        return FL_ERR_ARG;
    }
    if (!reserved_) { set_last_error("scan batch run_device: call fl_scan_batch_reserve first"); return FL_ERR_STATE; }
    const size_t smem = sizeof(double) * POSE_DOUBLES * (size_t)n_pose_max;
    if (n_scans > res_slots_ || n_max > res_n_max_ || n_pose_max > res_pose_max_ || smem > UNDISTORT_SMEM_MAX ||
        (long long)n_scans * n_max > (long long)INT_MAX) {
        set_last_error("scan batch run_device: %d slots, %d rows or %d poses exceed the %d, %d and %d fl_scan_batch_reserve sized", n_scans,
                       n_max, n_pose_max, res_slots_, res_n_max_, res_pose_max_);
        return FL_ERR_CAPACITY;
    }
    if (n_scans == 0) return FL_OK;
    // the sorts' bits follow the reserved slot count, not n_scans, so cub's passes (and launches) are the same for every n_scans
    const int rows = n_scans * n_max, end_bit = 32 + slot_bits(res_slots_);
    size_t need = 0;
    FL_CHECK(cub_bytes(rows, end_bit, &need));
    if (need > cub_.bytes) { set_last_error("scan batch run_device: %d rows exceed what fl_scan_batch_reserve sized", rows); return FL_ERR_CAPACITY; }
    FL_CUDA(cudaSetDevice(dev));
    bool joined = false;
    FL_CHECK(map_->query_begin(st, &joined));
    using U64 = unsigned long long;
    BatchSlot* slots = slots_.as<BatchSlot>();
    float4 *raw = raw_.as<float4>(), *sraw = sraw_.as<float4>(), *down = down_.as<float4>();
    U64 *keys = keys_.as<U64>(), *keys_alt = keys_alt_.as<U64>();
    int *vals = vals_.as<int>(), *vals_alt = vals_alt_.as<int>(), *heads = heads_.as<int>(), *pos = pos_.as<int>(), *counts = counts_.as<int>();
    const int block = 256, gx = std::max(1, (n_max + block - 1) / block);
    k_batch_gather<<<dim3(gx, n_scans), block, 0, st>>>(d_raws, n_scans, res_slots_, n_max, n_pose_max, undistort, raw, keys, sraw, down, slots,
                                                        refs_.as<fl_scan_ref_t>(), counts);
    const float4* src = raw;
    if (undistort && rows > 0) {
        // the stable time sort of every slot at once (slot index above cub's float key), then the backward pass per slot
        size_t tmp = cub_.bytes;
        FL_CUDA(cub::DeviceRadixSort::SortPairs(cub_.ptr, tmp, keys, keys_alt, raw, sraw, rows, 0, end_bit, st));
        const int ub = 128;
        k_batch_undistort<<<dim3((n_max + ub - 1) / ub, n_scans), ub, smem, st>>>(sraw, keys_alt, n_max, d_raws, n_pose_max, slots);
        src = sraw;
    }
    if (rows > 0) {
        k_batch_minmax<<<dim3(std::min(gx, 32), n_scans), block, 0, st>>>(src, n_max, slots);
        k_batch_keys<<<dim3(gx, n_scans), block, 0, st>>>(src, n_max, leaf, slots, keys, vals);
        size_t tmp = cub_.bytes;
        FL_CUDA(cub::DeviceRadixSort::SortPairs(cub_.ptr, tmp, keys, keys_alt, vals, vals_alt, rows, 0, end_bit, st));
        k_batch_heads<<<dim3(gx, n_scans), block, 0, st>>>(keys_alt, n_max, slots, heads);
        tmp = cub_.bytes;
        FL_CUDA(cub::DeviceScan::ExclusiveSum(cub_.ptr, tmp, heads, pos, rows, st));
        k_batch_centroid<<<dim3(gx, n_scans), block, 0, st>>>(src, keys_alt, vals_alt, heads, pos, n_max, down, slots);
    }
    k_batch_commit<<<(n_scans + 127) / 128, 128, 0, st>>>(slots, n_scans, res_slots_, counts, d_status2);
    FL_CUDA(cudaGetLastError());
    return map_->query_end(st, joined);
}

int ScanBatch::refs(int which, const fl_scan_ref_t** out, int* n_max) const {
    if ((which != 0 && which != 1) || !out) { set_last_error("scan batch get_refs: which must be 0 or 1, and out non-null"); return FL_ERR_ARG; }
    if (!reserved_) { set_last_error("scan batch get_refs: call fl_scan_batch_reserve first"); return FL_ERR_STATE; }
    *out = refs_.as<fl_scan_ref_t>() + (size_t)which * res_slots_;
    if (n_max) *n_max = res_n_max_;
    return FL_OK;
}

// the slot's entry of the table (where the last call put its rows) and its count, then the rows
int ScanBatch::download(int which, int slot, float* out_xyzi, int cap, int* n) {
    if (n) *n = 0;
    if (which != 0 && which != 1) { set_last_error("scan batch download: which must be 0 or 1"); return FL_ERR_ARG; }
    if (!reserved_) { set_last_error("scan batch download: call fl_scan_batch_reserve first"); return FL_ERR_STATE; }
    if (slot < 0 || slot >= res_slots_) { set_last_error("scan batch download: slot %d outside [0, %d)", slot, res_slots_); return FL_ERR_ARG; }
    FL_CUDA(cudaSetDevice(map_->device()));
    cudaStream_t st = map_->stream();
    fl_scan_ref_t r;
    int c = 0;
    const size_t e = (size_t)which * res_slots_ + slot;
    FL_CUDA(cudaMemcpyAsync(&r, refs_.as<fl_scan_ref_t>() + e, sizeof(r), cudaMemcpyDeviceToHost, st));
    FL_CUDA(cudaMemcpyAsync(&c, counts_.as<int>() + e, sizeof(int), cudaMemcpyDeviceToHost, st));
    FL_CUDA(cudaStreamSynchronize(st));
    c = std::max(c, 0);
    if (n) *n = c;
    const int take = std::min(c, cap);
    if (take <= 0) return FL_OK;
    if (!out_xyzi) { set_last_error("scan batch download: null buffer"); return FL_ERR_ARG; }
    FL_CUDA(cudaMemcpyAsync(out_xyzi, r.body_xyzi, sizeof(float4) * (size_t)take, cudaMemcpyDeviceToHost, st));
    FL_CUDA(cudaStreamSynchronize(st));
    return FL_OK;
}

// ================================================================================================ LocalMapCube
// The host form slides through cube_slide (scan.h); so does the device form's one-thread kernel below.
namespace {
// the device form's state: the committed cube, the cube the slide proposes, cub_needrm and its size, the delete's status2
struct SegState {
    CubeBox cube, next;
    float boxes[18];
    int nb;
    int st2[2];
};
// pos_lid = pos + rot * offset_T_L_I (laserMapping.cpp:890, Eigen's _transformVector), then the slide of a copy of the cube.
// An empty scan (*n_scan <= 0) is skipped before the segment (:892-896): nothing is proposed.
__global__ void k_seg_slide(SegState* s, const double* __restrict__ x, const int* __restrict__ n_scan, double cube_len, float det_range) {
    s->next = s->cube;
    s->nb = 0;
    if (n_scan && *n_scan <= 0) return;
    const D3 p = ld3(x + X_POS) + qrot(ldq(x + X_ROT), ld3(x + X_OFFT));
    const double pos[3] = {p.x, p.y, p.z};
    s->nb = cube_slide(s->next, pos, cube_len, det_range, s->boxes);
}
// the new cube is committed only when the delete went through; out3 = (|cub_needrm|, kdtree_delete_counter, status)
__global__ void k_seg_commit(SegState* s, float* __restrict__ boxes18, int* __restrict__ out3) {
    const int st = s->st2[0];
    if (st != FL_ERR_CAPACITY) s->cube = s->next;
    out3[0] = s->nb; out3[1] = s->st2[1]; out3[2] = st;
    if (boxes18) for (int i = 0; i < 18; i++) boxes18[i] = i < s->nb * 6 ? s->boxes[i] : 0.f;
}
}  // namespace

LocalMapCube::~LocalMapCube() {
    if (dev_.ptr && dmap_) cudaSetDevice(dmap_->device());
    dev_.release();
}

int LocalMapCube::pull() {
    if (!dev_.ptr) return FL_OK;
    FL_CUDA(cudaSetDevice(dmap_->device()));
    FL_CUDA(cudaMemcpyAsync(&c_, &dev_.as<SegState>()->cube, sizeof(CubeBox), cudaMemcpyDeviceToHost, dmap_->stream()));
    FL_CUDA(cudaStreamSynchronize(dmap_->stream()));
    return FL_OK;
}
int LocalMapCube::push() {
    if (!dev_.ptr) return FL_OK;
    FL_CUDA(cudaSetDevice(dmap_->device()));
    FL_CUDA(cudaMemcpyAsync(&dev_.as<SegState>()->cube, &c_, sizeof(CubeBox), cudaMemcpyHostToDevice, dmap_->stream()));
    FL_CUDA(cudaStreamSynchronize(dmap_->stream()));
    return FL_OK;
}

int LocalMapCube::segment_on_stream(Map* map, const double* d_x26, const int* d_n_scan, float* d_boxes18, int* d_out3, cudaStream_t st) {
    if (dmap_ && dmap_ != map) { set_last_error("fl_localmap_segment_device: the cube lives on another map"); return FL_ERR_ARG; }
    const int dev = map->device();
    if (!device_ptr(d_x26, dev, 8) || !device_ptr(d_out3, dev, 4) || (d_n_scan && !device_ptr(d_n_scan, dev, 4)) ||
        (d_boxes18 && !device_ptr(d_boxes18, dev, 4))) {
        set_last_error("fl_localmap_segment_device: a buffer is not device memory on device %d (x 8-byte, the others 4-byte aligned)", dev);
        return FL_ERR_ARG;
    }
    FL_CUDA(cudaSetDevice(dev));
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    FL_CUDA(cudaStreamGetCaptureInfo(st, &cs));
    if (!dev_.ptr) {
        if (cs != cudaStreamCaptureStatusNone) {
            set_last_error("fl_localmap_segment_device: the first call allocates the cube on the device; make it outside capture");
            return FL_ERR_STATE;
        }
        FL_CHECK(dev_.reserve(sizeof(SegState)));
        dmap_ = map;                                   // from here on the device copy is the cube (the caller retains the map)
        FL_CUDA(cudaMemsetAsync(dev_.ptr, 0, sizeof(SegState), map->stream()));
        FL_CHECK(push());                              // the host form's cube so far
    }
    FL_CHECK(map->delete_prepare(st));
    bool joined = false;
    FL_CHECK(map->mutation_begin(st, &joined));
    SegState* s = dev_.as<SegState>();
    k_seg_slide<<<1, 1, 0, st>>>(s, d_x26, d_n_scan, cube_len_, det_range_);
    FL_CHECK(map->enqueue_delete(s->boxes, &s->nb, 3, s->st2, st));   // if (cub_needrm.size() > 0) Delete_Point_Boxes (:275)
    k_seg_commit<<<1, 1, 0, st>>>(s, d_boxes18, d_out3);
    FL_CUDA(cudaGetLastError());
    return map->mutation_end(st, joined);
}

void LocalMapCube::get(float* box6) const {
    for (int a = 0; a < 3; a++) { box6[a] = c_.lo[a]; box6[3 + a] = c_.hi[a]; }
}

}  // namespace fl
