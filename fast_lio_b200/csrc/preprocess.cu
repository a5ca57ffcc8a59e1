// Preprocess::process on the device (see preprocess.h).  Every per-row decision is a kernel over n_max rows whose rows
// past the device count n count nothing; the three steps that couple rows are cub calls over the same n_max rows:
//   - Avia's valid_num, an inclusive sum of the valid flags (preprocess.cpp:165-168);
//   - Velodyne's per-ring time recurrence without point times (:420-441): a stable radix sort of the rows by ring, an
//     inclusive scan by ring of the maps c -> (lo < c) ? hi : lo, and a scatter back (DESIGN §4c);
//   - the order-preserving compaction into pl_surf, an exclusive sum of the kept flags.
// No host synchronisation, allocation or launch sized from a device value, so a call can be captured into a CUDA graph.
#include <cmath>
#include <cstring>
#include <vector>

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

// Velodyne :305-322: a frame of n > 0 rows gives point times when its last row's time is positive
__device__ __forceinline__ bool velo_timed(const unsigned char* __restrict__ raw, int n, const PpParams& P) {
    return rd<float>(raw + (size_t)(n - 1) * P.step, P.off[F_T]) > 0.f;
}

// Per-row decisions that need no other row, for row i of a frame of n rows at raw, stored at index o of the per-row arrays.
// keep: the row's own tests (Ouster, MARSIM, Velodyne); valid: Avia's; tm: the row's offset time in ms (PointType::curvature);
// keys / vals / yaw: the Velodyne yaw path's sort input, key_hi above the ring key and the value o; dropped counts rings >= N_SCANS.
__device__ __forceinline__ void pp_mark_row(const unsigned char* __restrict__ raw, int n, int i, int o, unsigned key_hi, const PpParams& P,
                                            int* __restrict__ keep, int* __restrict__ valid, float* __restrict__ tm,
                                            unsigned* __restrict__ keys, int* __restrict__ vals, float* __restrict__ yaw, int* dropped) {
    const bool in = i < n;
    const unsigned char* row = raw + (size_t)i * P.step;
    float x = 0.f, y = 0.f, z = 0.f;
    if (in) { x = rd<float>(row, P.off[F_X]); y = rd<float>(row, P.off[F_Y]); z = rd<float>(row, P.off[F_Z]); }
    const double r = (double)range2(x, y, z);
    switch (P.type) {
    case AVIA: {           // :165, the loop starts at row 1
        const unsigned tag = in ? rd<unsigned char>(row, P.off[F_TAG]) & 0x30u : 0u;
        const int line = in ? rd<unsigned char>(row, P.off[F_LINE]) : 0;
        valid[o] = in && i >= 1 && line < P.n_scans && (tag == 0x10u || tag == 0x00u);
        tm[o] = in ? __fdiv_rn((float)rd<unsigned>(row, P.off[F_T]), 1000000.f) : 0.f;      // :174
        break;
    }
    case OUST64:           // :259-272; a row exactly at blind^2 is kept
        keep[o] = in && i % P.pfn == 0 && !(r < P.bb);
        tm[o] = in ? __fmul_rn((float)rd<unsigned>(row, P.off[F_T]), P.scale) : 0.f;
        break;
    case MARSIM:           // :465-479: no decimation, curvature 0
        keep[o] = in && !(r < P.bb);
        tm[o] = 0.f;
        break;
    default: {             // VELO16 :305-322, :403-452
        const bool given = n > 0 && velo_timed(raw, n, P);
        keep[o] = in && i % P.pfn == 0 && r > P.bb;
        tm[o] = in ? __fmul_rn(rd<float>(row, P.off[F_T]), P.scale) : 0.f;
        const int ring = in ? rd<unsigned short>(row, P.off[F_RING]) : 0;
        const bool yaw_row = in && !given && ring < P.n_scans;
        if (in && !given && ring >= P.n_scans) atomicAdd(dropped, 1);
        keys[o] = key_hi | (yaw_row ? (unsigned)ring : (unsigned)P.n_scans);
        vals[o] = o;
        // the reference's atan2(float, float) is atan2f; the device rounds the double atan2 to float (DESIGN §4c)
        yaw[o] = (float)atan2((double)y, (double)x);
        break;
    }
    }
}

__global__ void k_pp_mark(const unsigned char* __restrict__ raw, const int* __restrict__ n_dev, int n_max, PpParams P,
                          int* __restrict__ keep, int* __restrict__ valid, float* __restrict__ tm, unsigned* __restrict__ keys,
                          int* __restrict__ vals, float* __restrict__ yaw, PpCtl* ctl) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_max) return;
    pp_mark_row(raw, clamp_n(n_dev, n_max), i, i, 0u, P, keep, valid, tm, keys, vals, yaw, &ctl->dropped);
}

// Avia :166-182 after valid_num: a row is selected when valid_num % point_filter_num == 0; the duplicate test compares with
// row i-1 only when that row was selected (pl_full is cleared and resized each call), else with PCL's zero point.
// a selected row: new against the previous row when that one was selected (psel), else against the zero point; outside blind
__device__ __forceinline__ bool avia_keep_row(const unsigned char* row, bool psel, const PpParams& P) {
    const float x = rd<float>(row, P.off[F_X]), y = rd<float>(row, P.off[F_Y]), z = rd<float>(row, P.off[F_Z]);
    float px = 0.f, py = 0.f, pz = 0.f;
    if (psel) {
        const unsigned char* prow = row - P.step;
        px = rd<float>(prow, P.off[F_X]); py = rd<float>(prow, P.off[F_Y]); pz = rd<float>(prow, P.off[F_Z]);
    }
    const bool is_new = (double)fabsf(__fsub_rn(x, px)) > 1e-7 || (double)fabsf(__fsub_rn(y, py)) > 1e-7 ||
                        (double)fabsf(__fsub_rn(z, pz)) > 1e-7;
    return is_new && (double)range2(x, y, z) > P.bb;
}

__global__ void k_pp_avia_keep(const unsigned char* __restrict__ raw, int n_max, PpParams P, const int* __restrict__ valid,
                               const int* __restrict__ vnum, int* __restrict__ keep) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_max) return;
    const bool sel = valid[i] && vnum[i] % P.pfn == 0;
    if (!sel) { keep[i] = 0; return; }
    const bool psel = i >= 1 && valid[i - 1] && vnum[i - 1] % P.pfn == 0;
    // avia_keep_row's body: calling it moves this kernel's instruction schedule, so it keeps its own copy
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

// a yaw in degrees as the reference scales it (:425-433)
__device__ __forceinline__ double yaw_deg(float yaw) { return (double)yaw * 57.2957; }

// lo and hi = float(double(lo) + 360 / omega_l) of a row at yaw (radians) on a ring whose first row's yaw is fp (degrees), :436-443
__device__ __forceinline__ Tri velo_tri(float yaw, double fp, const PpParams& P) {
    const double y = yaw_deg(yaw);
    const float lo = (float)(y <= fp ? (fp - y) / P.omega_l : (fp - y + 360.0) / P.omega_l);
    return Tri{lo, lo, (float)((double)lo + 360.0 / P.omega_l)};
}

// The first row of each ring (in raw order, so the first of its run after the stable sort) sets yaw_fp (:425-433).
__global__ void k_pp_velo_head(const unsigned* __restrict__ keys, const int* __restrict__ vals, const float* __restrict__ yaw,
                               int n_max, PpParams P, double* __restrict__ yaw_fp) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_max) return;
    const unsigned k = keys[p];
    if (k < (unsigned)P.n_scans && (p == 0 || keys[p - 1] != k)) yaw_fp[k] = yaw_deg(yaw[vals[p]]);
}

// One map per sorted row: lo and hi = float(double(lo) + 360 / omega_l) (:436-443); the first row of a ring, and padding, 0.
__global__ void k_pp_velo_tri(const unsigned* __restrict__ keys, const int* __restrict__ vals, const float* __restrict__ yaw,
                              int n_max, PpParams P, const double* __restrict__ yaw_fp, Tri* __restrict__ tri) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_max) return;
    const unsigned k = keys[p];
    if (k >= (unsigned)P.n_scans || p == 0 || keys[p - 1] != k) { tri[p] = Tri{0.f, 0.f, 0.f}; return; }
    tri[p] = velo_tri(yaw[vals[p]], yaw_fp[k], P);
}

// Back to raw order: a ring's first row is never output (its `continue` comes before the decimation, :431), a ring >= N_SCANS
// is dropped (the reference's undefined behaviour), the others take the scanned time.  Nothing changes with point times.
__global__ void k_pp_velo_out(const unsigned* __restrict__ keys, const int* __restrict__ vals, const Tri* __restrict__ tri,
                              const unsigned char* __restrict__ raw, const int* __restrict__ n_dev, int n_max, PpParams P,
                              int* __restrict__ keep, float* __restrict__ tm) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_max) return;
    const int n = clamp_n(n_dev, n_max);
    if (n == 0 || velo_timed(raw, n, P)) return;
    const unsigned k = keys[p];
    const int idx = vals[p];
    if (k >= (unsigned)P.n_scans || p == 0 || keys[p - 1] != k) { keep[idx] = 0; return; }
    tm[idx] = tri_apply(tri[p], 0.f);
}

// a kept row of pl_surf: x, y, z and the intensity (Avia's reflectivity byte as a float)
__device__ __forceinline__ float4 pp_point(const unsigned char* __restrict__ row, const PpParams& P) {
    const float in = P.type == AVIA ? (float)rd<unsigned char>(row, P.off[F_I]) : rd<float>(row, P.off[F_I]);
    return make_float4(rd<float>(row, P.off[F_X]), rd<float>(row, P.off[F_Y]), rd<float>(row, P.off[F_Z]), in);
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
    const float4 v = pp_point(raw + (size_t)i * P.step, P);
    const int o = pos[i];
    xyzi[o] = v;
    ms[o] = tm[i];
    if (last && o == total - 1) *last = tm[i];
}


// ------------------------------------------------------------------------------------------------ many frames (PreprocessBatch)
// Slot s owns packed rows [s * n_max, (s + 1) * n_max) of the scratch and output rows [s * stride, ...), stride the handle's
// n_raw_max; the grids are (row blocks, slots), so blockIdx.y is the slot.  Positions of the cub scans over every slot are taken
// less the slot's first, which makes them the single form's positions within the frame.
struct PbSlot {
    int n;              // its count c, 0 for a refused slot
    int err;            // FL_OK or its refusal
    int dropped;        // as PpCtl's
    int given;          // Velodyne: the frame gives point times
};

__device__ __forceinline__ bool misaligned(const void* p, unsigned align) { return (reinterpret_cast<uintptr_t>(p) & (align - 1)) != 0; }

// k_pp_mark per slot: every block decides its slot's refusal (a refused slot is a frame of 0 rows) and thread 0 of the slot
// records it; the ring keys carry the slot above key_bits
__global__ void k_ppb_mark(const fl_preprocess_raw_t* __restrict__ raws, int n_max, PpParams P, PbSlot* slots, int* __restrict__ keep,
                           int* __restrict__ valid, float* __restrict__ tm, unsigned* __restrict__ keys, int* __restrict__ vals,
                           float* __restrict__ yaw) {
    const int s = blockIdx.y;
    const fl_preprocess_raw_t r = raws[s];
    int err = FL_OK, c = 0;
    if (!r.n_raw || misaligned(r.n_raw, 4)) err = FL_ERR_ARG;
    else {
        c = *r.n_raw;
        if (c < 0) err = FL_ERR_ARG;
        else if (c > n_max) err = FL_ERR_CAPACITY;
        else if (c > 0 && !r.raw) err = FL_ERR_ARG;
    }
    if (err != FL_OK) c = 0;
    const unsigned char* raw = static_cast<const unsigned char*>(r.raw);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) {
        slots[s].n = c;
        slots[s].err = err;
        slots[s].given = P.type == VELO16 && c > 0 && velo_timed(raw, c, P);
    }
    if (i >= n_max) return;
    pp_mark_row(raw, c, i, s * n_max + i, (unsigned)s << P.key_bits, P, keep, valid, tm, keys, vals, yaw, &slots[s].dropped);
}

// k_pp_avia_keep per slot: valid_num is the inclusive sum over every slot less the slot's count before its first row, and the
// previous row is looked at only inside the slot
__global__ void k_ppb_avia_keep(const fl_preprocess_raw_t* __restrict__ raws, int n_max, PpParams P, const int* __restrict__ valid,
                                const int* __restrict__ vsum, int* __restrict__ keep) {
    const int s = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_max) return;
    const int b = s * n_max, r = b + i;
    const int base = vsum[b] - valid[b];
    if (!(valid[r] && (vsum[r] - base) % P.pfn == 0)) { keep[r] = 0; return; }
    const bool psel = i >= 1 && valid[r - 1] && (vsum[r - 1] - base) % P.pfn == 0;
    keep[r] = avia_keep_row(static_cast<const unsigned char*>(raws[s].raw) + (size_t)i * P.step, psel, P);
}

// k_pp_velo_head / k_pp_velo_tri / k_pp_velo_out over the slot-prefixed ring sort: a key (slot, ring) runs inside its slot's
// region, yaw_fp is [slot][ring], and the values are packed rows
__global__ void k_ppb_velo_head(const unsigned* __restrict__ keys, const int* __restrict__ vals, const float* __restrict__ yaw,
                                int n_max, PpParams P, double* __restrict__ yaw_fp) {
    const int s = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_max) return;
    const int p = s * n_max + i;
    const unsigned k = keys[p], ring = k & ((1u << P.key_bits) - 1u);
    if (ring < (unsigned)P.n_scans && (i == 0 || keys[p - 1] != k)) yaw_fp[(size_t)s * P.n_scans + ring] = yaw_deg(yaw[vals[p]]);
}

__global__ void k_ppb_velo_tri(const unsigned* __restrict__ keys, const int* __restrict__ vals, const float* __restrict__ yaw,
                               int n_max, PpParams P, const double* __restrict__ yaw_fp, Tri* __restrict__ tri) {
    const int s = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_max) return;
    const int p = s * n_max + i;
    const unsigned k = keys[p], ring = k & ((1u << P.key_bits) - 1u);
    if (ring >= (unsigned)P.n_scans || i == 0 || keys[p - 1] != k) { tri[p] = Tri{0.f, 0.f, 0.f}; return; }
    tri[p] = velo_tri(yaw[vals[p]], yaw_fp[(size_t)s * P.n_scans + ring], P);
}

__global__ void k_ppb_velo_out(const unsigned* __restrict__ keys, const int* __restrict__ vals, const Tri* __restrict__ tri, int n_max,
                               PpParams P, const PbSlot* __restrict__ slots, int* __restrict__ keep, float* __restrict__ tm) {
    const int s = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_max || slots[s].n == 0 || slots[s].given) return;
    const int p = s * n_max + i;
    const unsigned k = keys[p], ring = k & ((1u << P.key_bits) - 1u);
    const int idx = vals[p];
    if (ring >= (unsigned)P.n_scans || i == 0 || keys[p - 1] != k) { keep[idx] = 0; return; }
    tm[idx] = tri_apply(tri[p], 0.f);
}

// the slot's |pl_surf| from the exclusive sum of the kept flags over every slot
__device__ __forceinline__ int slot_total(const int* __restrict__ keep, const int* __restrict__ pos, int b, int n_max) {
    return pos[b + n_max - 1] + keep[b + n_max - 1] - pos[b];
}

// k_pp_scatter per slot, into the slot's output region; last_ms of a slot that keeps nothing is k_ppb_commit's
__global__ void k_ppb_scatter(const fl_preprocess_raw_t* __restrict__ raws, int n_max, int stride, PpParams P, const int* __restrict__ keep,
                              const int* __restrict__ pos, const float* __restrict__ tm, float4* __restrict__ xyzi, float* __restrict__ ms,
                              float* __restrict__ last) {
    const int s = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_max) return;
    const int b = s * n_max, r = b + i;
    if (!keep[r]) return;
    const int o = pos[r] - pos[b];
    const size_t out = (size_t)s * stride + o;
    xyzi[out] = pp_point(static_cast<const unsigned char*>(raws[s].raw) + (size_t)i * P.step, P);
    ms[out] = tm[r];
    if (o == slot_total(keep, pos, b, n_max) - 1) last[s] = tm[r];
}

// per slot of the handle: out2 = (|pl_surf|, dropped) and status2 = (FL_OK, |pl_surf|), or (-1, 0) and (refusal, 0); slots the
// call does not cover get out2 = (-1, 0); last_ms is 0 wherever k_ppb_scatter wrote none
__global__ void k_ppb_commit(const PbSlot* __restrict__ slots, int n_slots, int n_slots_max, int n_max, const int* __restrict__ keep,
                             const int* __restrict__ pos, int* __restrict__ out2, float* __restrict__ last, int* __restrict__ status2) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_slots_max) return;
    const int err = s < n_slots ? slots[s].err : FL_ERR_ARG;
    const int total = err == FL_OK && n_max > 0 ? slot_total(keep, pos, s * n_max, n_max) : 0;
    out2[2 * s] = err == FL_OK ? total : -1;
    out2[2 * s + 1] = err == FL_OK ? slots[s].dropped : 0;
    if (total == 0) last[s] = 0.f;
    if (s < n_slots) {
        status2[2 * s] = err;
        status2[2 * s + 1] = total;
    }
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


// ================================================================================================ PreprocessBatch
PreprocessBatch::~PreprocessBatch() {
    cudaSetDevice(dev_);
    for (DeviceBuffer* b : {&keep_, &pos_, &tm_, &valid_, &keys_, &keys_alt_, &vals_, &vals_alt_, &yaw_, &tri_, &tri_alt_, &yaw_fp_,
                            &slots_, &cub_, &xyzi_, &ms_, &out2_, &last_})
        b->release();
    if (ev_) cudaEventDestroy(ev_);
    if (stream_) cudaStreamDestroy(stream_);
}

// cub's temporary storage for the scans over `rows` packed rows and, on the Velodyne path, the ring sort on sort_bits_ bits
size_t PreprocessBatch::cub_bytes(int rows) const {
    size_t a = 0, b = 0, c = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, a, (const int*)nullptr, (int*)nullptr, rows);
    if (p_.type == VELO16) {
        cub::DeviceRadixSort::SortPairs(nullptr, b, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr, (int*)nullptr, rows, 0,
                                        sort_bits_);
        cub::DeviceScan::InclusiveScanByKey(nullptr, c, (const unsigned*)nullptr, (const Tri*)nullptr, (Tri*)nullptr, TriCompose(), rows);
    }
    return std::max(a, std::max(b, c));
}

int PreprocessBatch::init() {
    FL_CUDA(cudaSetDevice(dev_));
    FL_CUDA(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
    FL_CUDA(cudaEventCreateWithFlags(&ev_, cudaEventDisableTiming));
    // the slot index above the ring key: as many bits as n_slots_max needs, so the sort's passes (and launches) are the same
    // for every n_slots
    int slot_bits = 0;
    while ((1ll << slot_bits) < (long long)slots_max_) slot_bits++;
    sort_bits_ = p_.key_bits + slot_bits;
    const size_t S = (size_t)std::max(1, slots_max_), rows = std::max<size_t>(1, (size_t)slots_max_ * n_raw_max_);
    FL_CHECK(keep_.reserve(sizeof(int) * rows));
    FL_CHECK(pos_.reserve(sizeof(int) * rows));
    FL_CHECK(tm_.reserve(sizeof(float) * rows));
    if (p_.type == AVIA) FL_CHECK(valid_.reserve(sizeof(int) * rows));
    if (p_.type == VELO16) {
        FL_CHECK(keys_.reserve(sizeof(unsigned) * rows));
        FL_CHECK(keys_alt_.reserve(sizeof(unsigned) * rows));
        FL_CHECK(vals_.reserve(sizeof(int) * rows));
        FL_CHECK(vals_alt_.reserve(sizeof(int) * rows));
        FL_CHECK(yaw_.reserve(sizeof(float) * rows));
        FL_CHECK(tri_.reserve(sizeof(Tri) * rows));
        FL_CHECK(tri_alt_.reserve(sizeof(Tri) * rows));
        FL_CHECK(yaw_fp_.reserve(sizeof(double) * S * p_.n_scans));
    }
    FL_CHECK(slots_.reserve(sizeof(PbSlot) * S));
    FL_CHECK(cub_.reserve(std::max<size_t>(1, cub_bytes((int)rows))));
    FL_CHECK(xyzi_.reserve(sizeof(float4) * rows));
    FL_CHECK(ms_.reserve(sizeof(float) * rows));
    FL_CHECK(out2_.reserve(sizeof(int) * 2 * S));
    FL_CHECK(last_.reserve(sizeof(float) * S));
    // before any call every slot reads as uncovered: out2 = (-1, 0), last_ms 0
    std::vector<int> o(2 * S);
    for (size_t s = 0; s < S; s++) { o[2 * s] = -1; o[2 * s + 1] = 0; }
    FL_CUDA(cudaMemcpyAsync(out2_.ptr, o.data(), sizeof(int) * 2 * S, cudaMemcpyHostToDevice, stream_));
    FL_CUDA(cudaMemsetAsync(last_.ptr, 0, sizeof(float) * S, stream_));
    FL_CUDA(cudaStreamSynchronize(stream_));
    return FL_OK;
}

int PreprocessBatch::run_device(const fl_preprocess_raw_t* d_raws, int n_slots, int n_max, int* d_status2, cudaStream_t st) {
    if (n_slots < 0 || n_max < 0 || (n_slots > 0 && (!device_ptr(d_raws, dev_, 8) || !device_ptr(d_status2, dev_, 4)))) {
        set_last_error("preprocess batch run_device: n_slots or n_max < 0, or a buffer is not device memory on device %d (table "
                       "8-byte, status2 4-byte aligned)", dev_);
        return FL_ERR_ARG;
    }
    if (n_slots > slots_max_ || n_max > n_raw_max_) {
        set_last_error("preprocess batch run_device: %d slots or %d rows exceed the handle's n_slots_max = %d and n_raw_max = %d",
                       n_slots, n_max, slots_max_, n_raw_max_);
        return FL_ERR_CAPACITY;
    }
    if (n_slots == 0) return FL_OK;
    const int rows = n_slots * n_max, gx = std::max(1, (n_max + BLOCK - 1) / BLOCK);
    if (cub_bytes(rows) > cub_.bytes) { set_last_error("preprocess batch run_device: %d rows exceed cub's storage", rows); return FL_ERR_CAPACITY; }
    FL_CUDA(cudaSetDevice(dev_));
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    FL_CUDA(cudaStreamGetCaptureInfo(st, &cs));
    const dim3 grid(gx, n_slots);
    PbSlot* slots = slots_.as<PbSlot>();
    int *keep = keep_.as<int>(), *pos = pos_.as<int>(), *valid = valid_.as<int>();
    float* tm = tm_.as<float>();
    size_t tmp = cub_.bytes;
    FL_CUDA(cudaMemsetAsync(slots, 0, sizeof(PbSlot) * n_slots, st));
    k_ppb_mark<<<grid, BLOCK, 0, st>>>(d_raws, n_max, p_, slots, keep, valid, tm, keys_.as<unsigned>(), vals_.as<int>(), yaw_.as<float>());
    FL_CUDA(cudaGetLastError());
    if (rows > 0 && p_.type == AVIA) {
        FL_CUDA(cub::DeviceScan::InclusiveSum(cub_.ptr, tmp, valid, pos, rows, st));
        k_ppb_avia_keep<<<grid, BLOCK, 0, st>>>(d_raws, n_max, p_, valid, pos, keep);
        FL_CUDA(cudaGetLastError());
    }
    if (rows > 0 && p_.type == VELO16) {
        unsigned* keys = keys_alt_.as<unsigned>();
        int* vals = vals_alt_.as<int>();
        tmp = cub_.bytes;
        FL_CUDA(cub::DeviceRadixSort::SortPairs(cub_.ptr, tmp, keys_.as<unsigned>(), keys, vals_.as<int>(), vals, rows, 0, sort_bits_, st));
        k_ppb_velo_head<<<grid, BLOCK, 0, st>>>(keys, vals, yaw_.as<float>(), n_max, p_, yaw_fp_.as<double>());
        k_ppb_velo_tri<<<grid, BLOCK, 0, st>>>(keys, vals, yaw_.as<float>(), n_max, p_, yaw_fp_.as<double>(), tri_.as<Tri>());
        FL_CUDA(cudaGetLastError());
        tmp = cub_.bytes;
        FL_CUDA(cub::DeviceScan::InclusiveScanByKey(cub_.ptr, tmp, keys, tri_.as<Tri>(), tri_alt_.as<Tri>(), TriCompose(), rows,
                                                    cub::Equality(), st));
        k_ppb_velo_out<<<grid, BLOCK, 0, st>>>(keys, vals, tri_alt_.as<Tri>(), n_max, p_, slots, keep, tm);
        FL_CUDA(cudaGetLastError());
    }
    if (rows > 0) {
        tmp = cub_.bytes;
        FL_CUDA(cub::DeviceScan::ExclusiveSum(cub_.ptr, tmp, keep, pos, rows, st));
        k_ppb_scatter<<<grid, BLOCK, 0, st>>>(d_raws, n_max, n_raw_max_, p_, keep, pos, tm, xyzi_.as<float4>(), ms_.as<float>(),
                                               last_.as<float>());
    }
    k_ppb_commit<<<(slots_max_ + 127) / 128, 128, 0, st>>>(slots, n_slots, slots_max_, n_max, keep, pos, out2_.as<int>(), last_.as<float>(),
                                                          d_status2);
    FL_CUDA(cudaGetLastError());
    if (cs == cudaStreamCaptureStatusNone) FL_CUDA(cudaEventRecord(ev_, st));
    return FL_OK;
}

void PreprocessBatch::outputs(float** xyzi, float** ms, int** out2, float** last, int* n_raw_max) const {
    if (xyzi) *xyzi = xyzi_.as<float>();
    if (ms) *ms = ms_.as<float>();
    if (out2) *out2 = out2_.as<int>();
    if (last) *last = last_.as<float>();
    if (n_raw_max) *n_raw_max = n_raw_max_;
}

int PreprocessBatch::download(int slot, float* xyzi, float* ms, int cap, float* last, int* n) {
    *n = 0;
    if (slot < 0 || slot >= slots_max_ || cap < 0) {
        set_last_error("preprocess batch download: slot %d outside [0, %d), or cap < 0", slot, slots_max_);
        return FL_ERR_ARG;
    }
    FL_CUDA(cudaSetDevice(dev_));
    FL_CUDA(cudaStreamWaitEvent(stream_, ev_, 0));
    int o2[2] = {0, 0};
    float l = 0.f;
    FL_CUDA(cudaMemcpyAsync(o2, out2_.as<int>() + 2 * (size_t)slot, sizeof(o2), cudaMemcpyDeviceToHost, stream_));
    FL_CUDA(cudaMemcpyAsync(&l, last_.as<float>() + slot, sizeof(float), cudaMemcpyDeviceToHost, stream_));
    FL_CUDA(cudaStreamSynchronize(stream_));
    const int c = std::max(o2[0], 0), take = std::min(c, cap);
    if (take > 0 && (!xyzi || !ms)) { set_last_error("preprocess batch download: null buffer"); return FL_ERR_ARG; }
    if (take > 0) {
        const size_t base = (size_t)slot * n_raw_max_;
        FL_CUDA(cudaMemcpyAsync(xyzi, xyzi_.as<float4>() + base, sizeof(float4) * take, cudaMemcpyDeviceToHost, stream_));
        FL_CUDA(cudaMemcpyAsync(ms, ms_.as<float>() + base, sizeof(float) * take, cudaMemcpyDeviceToHost, stream_));
        FL_CUDA(cudaStreamSynchronize(stream_));
    }
    if (last) *last = l;
    *n = c;
    return FL_OK;
}

}  // namespace fl
