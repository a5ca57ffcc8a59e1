// Preprocess::process on the device (see preprocess.h).  Every per-row decision is a kernel over n_max rows whose rows
// past the device count n count nothing; the three steps that couple rows are cub calls over the same n_max rows:
//   - Avia's valid_num, an inclusive sum of the valid flags (preprocess.cpp:165-168);
//   - Velodyne's per-ring time recurrence without point times (:420-441): a stable radix sort of the rows by ring, an
//     inclusive scan by ring of the maps c -> (lo < c) ? hi : lo, and a scatter back (DESIGN §4c);
//   - the order-preserving compaction into pl_surf, an exclusive sum of the kept flags.
// No host synchronisation, allocation or launch sized from a device value, so a call can be captured into a CUDA graph.
#include <cmath>
#include <cstring>

#include <cub/cub.cuh>

#include "common.cuh"
#include "preprocess.h"

namespace fl {

namespace {

enum { F_X, F_Y, F_Z, F_I, F_T, F_RING, F_TAG, F_LINE };
enum { AVIA = 1, VELO16 = 2, OUST64 = 3, MARSIM = 4 };
constexpr int BLOCK = 256;

struct PpCtl {
    int dropped;        // rows with ring >= N_SCANS on the Velodyne yaw path
};

// (t, a, b): c -> (t < c) ? b : a.  One Velodyne row is (lo, lo, hi), a ring's first row the constant 0.
struct Tri {
    float t, a, b;
};
__device__ __forceinline__ float tri_apply(const Tri& f, float c) { return f.t < c ? f.b : f.a; }
// second o first = (first.t, second(first.a), second(first.b)); cub passes the earlier aggregate first
struct TriCompose {
    __device__ __forceinline__ Tri operator()(const Tri& first, const Tri& second) const {
        return Tri{first.t, tri_apply(second, first.a), tri_apply(second, first.b)};
    }
};

// a field of the reference's type at a byte offset that may be unaligned; an absent field (-1) reads as 0
template <class T>
__device__ __forceinline__ T rd(const unsigned char* row, int off) {
    T v = 0;
    if (off >= 0) memcpy(&v, row + off, sizeof(T));
    return v;
}

// x*x + y*y + z*z in float (the reference's PointType arithmetic), left to right, without contraction
__device__ __forceinline__ float range2(float x, float y, float z) {
    return __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
}

__device__ __forceinline__ int clamp_n(const int* n_dev, int n_max) { return min(max(*n_dev, 0), n_max); }

// Per-row decisions that need no other row.  keep: the row's own tests (Ouster, MARSIM, Velodyne); valid: Avia's;
// tm: the row's offset time in ms (PointType::curvature); keys / vals / yaw: the Velodyne yaw path's sort input.
__global__ void k_pp_mark(const unsigned char* __restrict__ raw, const int* __restrict__ n_dev, int n_max, PpParams P,
                          int* __restrict__ keep, int* __restrict__ valid, float* __restrict__ tm, unsigned* __restrict__ keys,
                          int* __restrict__ vals, float* __restrict__ yaw, PpCtl* ctl) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_max) return;
    const int n = clamp_n(n_dev, n_max);
    const bool in = i < n;
    const unsigned char* row = raw + (size_t)i * P.step;
    float x = 0.f, y = 0.f, z = 0.f;
    if (in) { x = rd<float>(row, P.off[F_X]); y = rd<float>(row, P.off[F_Y]); z = rd<float>(row, P.off[F_Z]); }
    const double r = (double)range2(x, y, z);
    switch (P.type) {
    case AVIA: {           // :165, the loop starts at row 1
        const unsigned tag = in ? rd<unsigned char>(row, P.off[F_TAG]) & 0x30u : 0u;
        const int line = in ? rd<unsigned char>(row, P.off[F_LINE]) : 0;
        valid[i] = in && i >= 1 && line < P.n_scans && (tag == 0x10u || tag == 0x00u);
        tm[i] = in ? __fdiv_rn((float)rd<unsigned>(row, P.off[F_T]), 1000000.f) : 0.f;      // :174
        break;
    }
    case OUST64:           // :259-272; a row exactly at blind^2 is kept
        keep[i] = in && i % P.pfn == 0 && !(r < P.bb);
        tm[i] = in ? __fmul_rn((float)rd<unsigned>(row, P.off[F_T]), P.scale) : 0.f;
        break;
    case MARSIM:           // :465-479: no decimation, curvature 0
        keep[i] = in && !(r < P.bb);
        tm[i] = 0.f;
        break;
    default: {             // VELO16 :305-322, :403-452
        const bool given = n > 0 && rd<float>(raw + (size_t)(n - 1) * P.step, P.off[F_T]) > 0.f;
        keep[i] = in && i % P.pfn == 0 && r > P.bb;
        tm[i] = in ? __fmul_rn(rd<float>(row, P.off[F_T]), P.scale) : 0.f;
        const int ring = in ? rd<unsigned short>(row, P.off[F_RING]) : 0;
        const bool yaw_row = in && !given && ring < P.n_scans;
        if (in && !given && ring >= P.n_scans) atomicAdd(&ctl->dropped, 1);
        keys[i] = yaw_row ? (unsigned)ring : (unsigned)P.n_scans;
        vals[i] = i;
        // the reference's atan2(float, float) is atan2f; the device rounds the double atan2 to float (DESIGN §4c)
        yaw[i] = (float)atan2((double)y, (double)x);
        break;
    }
    }
}

// Avia :166-182 after valid_num: a row is selected when valid_num % point_filter_num == 0; the duplicate test compares with
// row i-1 only when that row was selected (pl_full is cleared and resized each call), else with PCL's zero point.
__global__ void k_pp_avia_keep(const unsigned char* __restrict__ raw, int n_max, PpParams P, const int* __restrict__ valid,
                               const int* __restrict__ vnum, int* __restrict__ keep) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_max) return;
    const bool sel = valid[i] && vnum[i] % P.pfn == 0;
    if (!sel) { keep[i] = 0; return; }
    const bool psel = i >= 1 && valid[i - 1] && vnum[i - 1] % P.pfn == 0;
    const unsigned char* row = raw + (size_t)i * P.step;
    const float x = rd<float>(row, P.off[F_X]), y = rd<float>(row, P.off[F_Y]), z = rd<float>(row, P.off[F_Z]);
    float px = 0.f, py = 0.f, pz = 0.f;
    if (psel) {
        const unsigned char* prow = row - P.step;
        px = rd<float>(prow, P.off[F_X]); py = rd<float>(prow, P.off[F_Y]); pz = rd<float>(prow, P.off[F_Z]);
    }
    const bool is_new = (double)fabsf(__fsub_rn(x, px)) > 1e-7 || (double)fabsf(__fsub_rn(y, py)) > 1e-7 ||
                        (double)fabsf(__fsub_rn(z, pz)) > 1e-7;
    keep[i] = is_new && (double)range2(x, y, z) > P.bb;
}

// The first row of each ring (in raw order, so the first of its run after the stable sort) sets yaw_fp (:425-433).
__global__ void k_pp_velo_head(const unsigned* __restrict__ keys, const int* __restrict__ vals, const float* __restrict__ yaw,
                               int n_max, PpParams P, double* __restrict__ yaw_fp) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_max) return;
    const unsigned k = keys[p];
    if (k < (unsigned)P.n_scans && (p == 0 || keys[p - 1] != k)) yaw_fp[k] = (double)yaw[vals[p]] * 57.2957;
}

// One map per sorted row: lo and hi = float(double(lo) + 360 / omega_l) (:436-443); the first row of a ring, and padding, 0.
__global__ void k_pp_velo_tri(const unsigned* __restrict__ keys, const int* __restrict__ vals, const float* __restrict__ yaw,
                              int n_max, PpParams P, const double* __restrict__ yaw_fp, Tri* __restrict__ tri) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_max) return;
    const unsigned k = keys[p];
    if (k >= (unsigned)P.n_scans || p == 0 || keys[p - 1] != k) { tri[p] = Tri{0.f, 0.f, 0.f}; return; }
    const double y = (double)yaw[vals[p]] * 57.2957, fp = yaw_fp[k];
    const float lo = (float)(y <= fp ? (fp - y) / P.omega_l : (fp - y + 360.0) / P.omega_l);
    tri[p] = Tri{lo, lo, (float)((double)lo + 360.0 / P.omega_l)};
}

// Back to raw order: a ring's first row is never output (its `continue` comes before the decimation, :431), a ring >= N_SCANS
// is dropped (the reference's undefined behaviour), the others take the scanned time.  Nothing changes with point times.
__global__ void k_pp_velo_out(const unsigned* __restrict__ keys, const int* __restrict__ vals, const Tri* __restrict__ tri,
                              const unsigned char* __restrict__ raw, const int* __restrict__ n_dev, int n_max, PpParams P,
                              int* __restrict__ keep, float* __restrict__ tm) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_max) return;
    const int n = clamp_n(n_dev, n_max);
    if (n == 0 || rd<float>(raw + (size_t)(n - 1) * P.step, P.off[F_T]) > 0.f) return;
    const unsigned k = keys[p];
    const int idx = vals[p];
    if (k >= (unsigned)P.n_scans || p == 0 || keys[p - 1] != k) { keep[idx] = 0; return; }
    tm[idx] = tri_apply(tri[p], 0.f);
}

// pl_surf: the kept rows in raw order.  out2 = (kept, dropped rings); last = pl_surf.back().curvature (0 when nothing is kept).
__global__ void k_pp_scatter(const unsigned char* __restrict__ raw, int n_max, PpParams P, const int* __restrict__ keep,
                             const int* __restrict__ pos, const float* __restrict__ tm, const PpCtl* __restrict__ ctl,
                             float4* __restrict__ xyzi, float* __restrict__ ms, int* __restrict__ out2, float* __restrict__ last) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int total = n_max > 0 ? pos[n_max - 1] + keep[n_max - 1] : 0;
    if (i == 0) {
        out2[0] = total;
        out2[1] = ctl->dropped;
        if (last && total == 0) *last = 0.f;
    }
    if (i >= n_max || !keep[i]) return;
    const unsigned char* row = raw + (size_t)i * P.step;
    const float in = P.type == AVIA ? (float)rd<unsigned char>(row, P.off[F_I]) : rd<float>(row, P.off[F_I]);
    const int o = pos[i];
    xyzi[o] = make_float4(rd<float>(row, P.off[F_X]), rd<float>(row, P.off[F_Y]), rd<float>(row, P.off[F_Z]), in);
    ms[o] = tm[i];
    if (last && o == total - 1) *last = tm[i];
}

}  // namespace

Preprocessor::~Preprocessor() {
    cudaSetDevice(dev_);
    for (DeviceBuffer* b : {&d_keep_, &d_pos_, &d_tm_, &d_valid_, &d_keys_, &d_keys_alt_, &d_vals_, &d_vals_alt_, &d_yaw_, &d_tri_,
                            &d_tri_alt_, &d_yaw_fp_, &d_ctl_, &d_cub_, &d_raw_, &d_n_, &d_xyzi_, &d_ms_, &d_out_})
        b->release();
    if (ev_) cudaEventDestroy(ev_);
    if (stream_) cudaStreamDestroy(stream_);
}

size_t Preprocessor::cub_bytes(int n) const {
    size_t a = 0, b = 0, c = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, a, (const int*)nullptr, (int*)nullptr, n);
    if (p_.type == VELO16) {
        cub::DeviceRadixSort::SortPairs(nullptr, b, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr, (int*)nullptr, n, 0,
                                        p_.key_bits);
        cub::DeviceScan::InclusiveScanByKey(nullptr, c, (const unsigned*)nullptr, (const Tri*)nullptr, (Tri*)nullptr, TriCompose(), n);
    }
    return std::max(a, std::max(b, c));
}

int Preprocessor::init() {
    FL_CUDA(cudaSetDevice(dev_));
    FL_CUDA(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
    FL_CUDA(cudaEventCreateWithFlags(&ev_, cudaEventDisableTiming));
    const size_t m = (size_t)std::max(1, n_raw_max_);
    FL_CHECK(d_keep_.reserve(sizeof(int) * m));
    FL_CHECK(d_pos_.reserve(sizeof(int) * m));
    FL_CHECK(d_tm_.reserve(sizeof(float) * m));
    if (p_.type == AVIA) FL_CHECK(d_valid_.reserve(sizeof(int) * m));
    if (p_.type == VELO16) {
        FL_CHECK(d_keys_.reserve(sizeof(unsigned) * m));
        FL_CHECK(d_keys_alt_.reserve(sizeof(unsigned) * m));
        FL_CHECK(d_vals_.reserve(sizeof(int) * m));
        FL_CHECK(d_vals_alt_.reserve(sizeof(int) * m));
        FL_CHECK(d_yaw_.reserve(sizeof(float) * m));
        FL_CHECK(d_tri_.reserve(sizeof(Tri) * m));
        FL_CHECK(d_tri_alt_.reserve(sizeof(Tri) * m));
        FL_CHECK(d_yaw_fp_.reserve(sizeof(double) * p_.n_scans));
    }
    FL_CHECK(d_ctl_.reserve(sizeof(PpCtl)));
    FL_CHECK(d_cub_.reserve(std::max<size_t>(1, cub_bytes((int)m))));
    FL_CHECK(d_raw_.reserve(m * p_.step));
    FL_CHECK(d_n_.reserve(sizeof(int)));
    FL_CHECK(d_xyzi_.reserve(sizeof(float4) * m));
    FL_CHECK(d_ms_.reserve(sizeof(float) * m));
    FL_CHECK(d_out_.reserve(sizeof(int) * 2 + sizeof(float)));
    return FL_OK;
}

int Preprocessor::enqueue(const void* d_raw, const int* d_n, int n_max, float* d_xyzi, float* d_ms, int* d_out2, float* d_last,
                          cudaStream_t st) {
    const unsigned char* raw = static_cast<const unsigned char*>(d_raw);
    const int grid = std::max(1, (n_max + BLOCK - 1) / BLOCK);
    size_t tmp = d_cub_.bytes;
    int* keep = d_keep_.as<int>();
    int* pos = d_pos_.as<int>();
    float* tm = d_tm_.as<float>();
    PpCtl* ctl = d_ctl_.as<PpCtl>();
    FL_CUDA(cudaMemsetAsync(ctl, 0, sizeof(PpCtl), st));
    k_pp_mark<<<grid, BLOCK, 0, st>>>(raw, d_n, n_max, p_, keep, d_valid_.as<int>(), tm, d_keys_.as<unsigned>(), d_vals_.as<int>(),
                                      d_yaw_.as<float>(), ctl);
    FL_CUDA(cudaGetLastError());
    if (n_max > 0 && p_.type == AVIA) {
        FL_CUDA(cub::DeviceScan::InclusiveSum(d_cub_.ptr, tmp, d_valid_.as<int>(), pos, n_max, st));
        k_pp_avia_keep<<<grid, BLOCK, 0, st>>>(raw, n_max, p_, d_valid_.as<int>(), pos, keep);
        FL_CUDA(cudaGetLastError());
    }
    if (n_max > 0 && p_.type == VELO16) {
        unsigned* keys = d_keys_alt_.as<unsigned>();
        int* vals = d_vals_alt_.as<int>();
        FL_CUDA(cub::DeviceRadixSort::SortPairs(d_cub_.ptr, tmp, d_keys_.as<unsigned>(), keys, d_vals_.as<int>(), vals, n_max, 0,
                                                p_.key_bits, st));
        tmp = d_cub_.bytes;
        k_pp_velo_head<<<grid, BLOCK, 0, st>>>(keys, vals, d_yaw_.as<float>(), n_max, p_, d_yaw_fp_.as<double>());
        k_pp_velo_tri<<<grid, BLOCK, 0, st>>>(keys, vals, d_yaw_.as<float>(), n_max, p_, d_yaw_fp_.as<double>(), d_tri_.as<Tri>());
        FL_CUDA(cudaGetLastError());
        FL_CUDA(cub::DeviceScan::InclusiveScanByKey(d_cub_.ptr, tmp, keys, d_tri_.as<Tri>(), d_tri_alt_.as<Tri>(), TriCompose(), n_max,
                                                    cub::Equality(), st));
        k_pp_velo_out<<<grid, BLOCK, 0, st>>>(keys, vals, d_tri_alt_.as<Tri>(), raw, d_n, n_max, p_, keep, tm);
        FL_CUDA(cudaGetLastError());
    }
    if (n_max > 0) {
        tmp = d_cub_.bytes;
        FL_CUDA(cub::DeviceScan::ExclusiveSum(d_cub_.ptr, tmp, keep, pos, n_max, st));
    }
    k_pp_scatter<<<grid, BLOCK, 0, st>>>(raw, n_max, p_, keep, pos, tm, ctl, reinterpret_cast<float4*>(d_xyzi), d_ms, d_out2, d_last);
    FL_CUDA(cudaGetLastError());
    return FL_OK;
}

int Preprocessor::run_device(const void* d_raw, const int* d_n, int n_max, float* d_xyzi, float* d_ms, int* d_out2, float* d_last,
                             cudaStream_t st) {
    if (n_max < 0 || !device_ptr(d_n, dev_, 4) || !device_ptr(d_out2, dev_, 4) || (d_last && !device_ptr(d_last, dev_, 4)) ||
        (n_max > 0 && (!device_ptr(d_raw, dev_, 1) || !device_ptr(d_xyzi, dev_, 16) || !device_ptr(d_ms, dev_, 4)))) {
        set_last_error("preprocess_device: n_max < 0, or a buffer is not device memory on device %d (xyzi 16-byte, offset times, "
                       "n, out2 and last_ms 4-byte aligned)", dev_);
        return FL_ERR_ARG;
    }
    if (n_max > n_raw_max_) {
        set_last_error("preprocess_device: n_max = %d exceeds the handle's n_raw_max = %d", n_max, n_raw_max_);
        return FL_ERR_CAPACITY;
    }
    FL_CUDA(cudaSetDevice(dev_));
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    FL_CUDA(cudaStreamGetCaptureInfo(st, &cs));
    FL_CHECK(enqueue(d_raw, d_n, n_max, d_xyzi, d_ms, d_out2, d_last, st));
    if (cs == cudaStreamCaptureStatusNone) FL_CUDA(cudaEventRecord(ev_, st));
    return FL_OK;
}

int Preprocessor::run_host(const void* raw, int n, float* xyzi, float* ms, int cap, float* last_ms) {
    if (n < 0 || cap < 0 || (n > 0 && !raw) || (cap > 0 && (!xyzi || !ms))) {
        set_last_error("preprocess: n < 0, cap < 0, or a null buffer");
        return FL_ERR_ARG;
    }
    if (n > n_raw_max_) {
        set_last_error("preprocess: %d rows exceed the handle's n_raw_max = %d", n, n_raw_max_);
        return FL_ERR_CAPACITY;
    }
    FL_CUDA(cudaSetDevice(dev_));
    FL_CUDA(cudaStreamWaitEvent(stream_, ev_, 0));      // the workspace is shared with the device form
    if (n > 0) FL_CUDA(cudaMemcpyAsync(d_raw_.ptr, raw, (size_t)n * p_.step, cudaMemcpyHostToDevice, stream_));
    FL_CUDA(cudaMemcpyAsync(d_n_.ptr, &n, sizeof(int), cudaMemcpyHostToDevice, stream_));
    int* out2 = d_out_.as<int>();
    float* last = reinterpret_cast<float*>(out2 + 2);
    FL_CHECK(enqueue(d_raw_.ptr, d_n_.as<int>(), n, d_xyzi_.as<float>(), d_ms_.as<float>(), out2, last, stream_));
    int h_out[3] = {0, 0, 0};
    FL_CUDA(cudaMemcpyAsync(h_out, out2, sizeof(h_out), cudaMemcpyDeviceToHost, stream_));
    FL_CUDA(cudaStreamSynchronize(stream_));
    const int kept = h_out[0], m = std::min(kept, cap);
    if (m > 0) {
        FL_CUDA(cudaMemcpyAsync(xyzi, d_xyzi_.ptr, sizeof(float4) * m, cudaMemcpyDeviceToHost, stream_));
        FL_CUDA(cudaMemcpyAsync(ms, d_ms_.ptr, sizeof(float) * m, cudaMemcpyDeviceToHost, stream_));
        FL_CUDA(cudaStreamSynchronize(stream_));
    }
    if (last_ms) memcpy(last_ms, &h_out[2], sizeof(float));
    return kept;
}

}  // namespace fl
