// Relocalisation: recover the pose of one scan on the map from many hypotheses, on the caller's stream.
//
//   k_reloc_expand : the hypotheses of a grid around a prior (reloc.cuh), one thread per state component.
//   k_reloc_screen : one thread per (hypothesis, screened scan point): the update's FP64 body->world transform (measure.cuh),
//                    then the exact nearest neighbour of the float32 world point from the map's own search (knn_block: the cell
//                    directory, the BVH walk for what it cannot prove) -- the search fl_map_nearest_search runs for k <= 5.
//                    The point is an inlier when that neighbour lies within r (d2 <= md2): an integer count per hypothesis.
//   k_reloc_keys   : the 64-bit rank key of each hypothesis, sorted by cub's radix sort.
//   k_reloc_gather : the states of the first `keep` keys, and P, into the survivors' slots of the batched update.
//   k_reloc_rank   : the survivors' rows from their batch status and last pass log, and the winner.
#include <algorithm>
#include <climits>
#include <cmath>

#include <cub/device/device_radix_sort.cuh>

#include "filter.h"
#include "map.cuh"
#include "measure.cuh"
#include "reloc.cuh"

namespace fl {

constexpr int RELOC_THREADS = 256;
constexpr int RELOC_MAX_LOGS = 16;         // the pass logs per survivor: max_iter + 1 <= 16 (Filter::set_params)

__global__ void __launch_bounds__(RELOC_THREADS) k_reloc_expand(const double* __restrict__ prior, fl_reloc_grid_t g,
                                                                 double* __restrict__ out, long long total) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    out[t] = reloc_component(prior, g, t / XLEN, (int)(t % XLEN));
}

// Block b screens points [chunk * RELOC_THREADS, ...) of the screened set (scan rows i * stride) from hypothesis b / chunks.  The
// inlier test is the gate of fl_map_nearest_search at k = 1: the nearest neighbour's d2 <= md2.  Its squared distance does not
// depend on the tie rule, so the map's deterministic mode needs no kernel of its own here.  (That gate reads the first entry
// after knn_fetch's tie ordering, which swaps only entries whose d2 differ by less than 1e-10: for md2 >= 1e-6 such entries are
// bit-equal or both far below md2, so the count is the same.)
__global__ void __launch_bounds__(RELOC_THREADS) k_reloc_screen(MapView m, const float4* __restrict__ body, int nq, int stride,
                                                                 int chunks, const double* __restrict__ x26, float md2,
                                                                 int* __restrict__ inliers) {
    __shared__ WalkPool pool;
    if (threadIdx.x == 0) pool.n[0] = pool.n[1] = 0;
    const int h = (int)(blockIdx.x / chunks);
    const long long j = (long long)(blockIdx.x % chunks) * RELOC_THREADS + threadIdx.x;
    const long long i = j * stride;
    const PoseS s = load_pose(x26 + (size_t)h * XLEN);
    float wx = 0.f, wy = 0.f, wz = 0.f;
    if (i < nq) body_to_world(s, __ldg(&body[i]), wx, wy, wz);
    const bool active = i < nq && isfinite(wx) && isfinite(wy) && isfinite(wz);    // a non-finite query finds nothing
    __syncthreads();
    int phase = 0;
    TBest kb;
    knn_block(m, active, wx, wy, wz, kb, pool, phase);
    const int n = __syncthreads_count(active && kb.idx[0] >= 0 && kb.d[0] <= md2);
    if (threadIdx.x == 0 && n) atomicAdd(&inliers[h], n);
}

// key = ((screened - inliers) << 32) | h: ascending order is most inliers first, ties to the lowest h
__global__ void k_reloc_keys(const int* __restrict__ inliers, int n_hyp, int screened, unsigned long long* __restrict__ keys) {
    const int h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h < n_hyp) keys[h] = ((unsigned long long)(unsigned)(screened - inliers[h]) << 32) | (unsigned)h;
}

// block s: survivor s (rank s) -- its hypothesis's state and the caller's P into slot s of the batch
__global__ void __launch_bounds__(RELOC_THREADS) k_reloc_gather(const unsigned long long* __restrict__ keys,
                                                                 const double* __restrict__ x26_hyp, const double* __restrict__ P,
                                                                 double* __restrict__ x_s, double* __restrict__ P_s) {
    const int s = blockIdx.x;
    const unsigned h = (unsigned)keys[s];
    for (int c = threadIdx.x; c < NDOF * NDOF; c += RELOC_THREADS) P_s[(size_t)s * NDOF * NDOF + c] = P[c];
    if (threadIdx.x < XLEN) x_s[(size_t)s * XLEN + threadIdx.x] = x26_hyp[(size_t)h * XLEN + threadIdx.x];
}

// One block.  Row s: survivor s's hypothesis, inliers, batch status, passes, and its last pass's effct and res_sum.  The winner:
// a qualifying row (FL_OK, last-pass effct >= min_effct) with the largest effct, then the smallest res_sum / effct, then the
// earliest rank; its x and P go to x_out / P_out only when there is one.
__global__ void __launch_bounds__(RELOC_THREADS) k_reloc_rank(const unsigned long long* __restrict__ keys,
                                                               const int* __restrict__ inliers, const int* __restrict__ status2,
                                                               const PassLog* __restrict__ logs, int log_stride, int keep,
                                                               int min_effct, const double* __restrict__ x_s,
                                                               const double* __restrict__ P_s, fl_reloc_row_t* __restrict__ rows_out,
                                                               double* __restrict__ x_out, double* __restrict__ P_out,
                                                               int* __restrict__ status4) {
    __shared__ int win;
    if (threadIdx.x == 0) {
        int best = -1, best_effct = 0;
        double best_ratio = 0.0;
        for (int s = 0; s < keep; s++) {
            fl_reloc_row_t r;
            r.hyp = (int)(unsigned)keys[s];
            r.inliers = inliers[r.hyp];
            r.status = status2[2 * s];
            r.passes = status2[2 * s + 1];
            r.effct = 0; r.pad = 0; r.res_sum = 0.0;
            if (r.passes > 0) {
                const PassLog& l = logs[(size_t)s * log_stride + r.passes - 1];
                r.effct = l.effct;
                r.res_sum = l.res_sum;
            }
            if (rows_out) rows_out[s] = r;
            if (r.status != FL_OK || r.passes < 1 || r.effct < min_effct) continue;
            const double ratio = r.res_sum / (double)r.effct;
            if (best < 0 || r.effct > best_effct || (r.effct == best_effct && ratio < best_ratio)) {
                best = s; best_effct = r.effct; best_ratio = ratio;
            }
        }
        win = best;
        const int h = best >= 0 ? (int)(unsigned)keys[best] : -1;
        status4[0] = best >= 0 ? FL_OK : FL_ERR_STATE;
        status4[1] = h;
        status4[2] = best >= 0 ? best_effct : 0;
        status4[3] = best >= 0 ? inliers[h] : 0;
    }
    __syncthreads();
    const int s = win;
    if (s < 0) return;
    for (int c = threadIdx.x; c < NDOF * NDOF; c += RELOC_THREADS) P_out[c] = P_s[(size_t)s * NDOF * NDOF + c];
    if (threadIdx.x < XLEN) x_out[threadIdx.x] = x_s[(size_t)s * XLEN + threadIdx.x];
}

static size_t sort_temp_bytes(int n) {
    size_t bytes = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, n, 0, 64);
    return bytes;
}

// ----------------------------------------------------------------------------- fl_reloc_expand_grid_device
int reloc_expand_grid(const double* d_prior, const fl_reloc_grid_t* g, double* d_hyp, cudaStream_t st) {
    cudaPointerAttributes a;
    if (!d_prior || cudaPointerGetAttributes(&a, d_prior) != cudaSuccess) {
        cudaGetLastError();
        set_last_error("reloc_expand_grid_device: the prior is not device memory");
        return FL_ERR_ARG;
    }
    const int dev = a.device;
    if (!g || !device_ptr(d_prior, dev, 8) || !device_ptr(d_hyp, dev, 8)) {
        set_last_error("reloc_expand_grid_device: a null grid, or the prior and the hypotheses are not 8-byte aligned memory of one device");
        return FL_ERR_ARG;
    }
    long long H = 1;
    for (int k = 0; k < 4; k++) {
        if (g->n[k] < 1 || !(g->step[k] >= 0.0) || !isfinite(g->step[k])) {
            set_last_error("reloc_expand_grid_device: axis %d has n = %d, step = %g (n >= 1, finite step >= 0)", k, g->n[k], g->step[k]);
            return FL_ERR_ARG;
        }
        H *= g->n[k];
        if (H > INT_MAX) { set_last_error("reloc_expand_grid_device: more than INT_MAX hypotheses"); return FL_ERR_CAPACITY; }
    }
    int prev = 0;
    FL_CUDA(cudaGetDevice(&prev));
    FL_CUDA(cudaSetDevice(dev));
    const long long total = H * XLEN;
    k_reloc_expand<<<(unsigned)((total + RELOC_THREADS - 1) / RELOC_THREADS), RELOC_THREADS, 0, st>>>(d_prior, *g, d_hyp, total);
    const cudaError_t e = cudaGetLastError();
    cudaSetDevice(prev);
    FL_CUDA(e);
    return FL_OK;
}

// ----------------------------------------------------------------------------- Filter: relocalisation
int Filter::reserve_reloc(int nq_max, int n_hyp_max, int keep_max) {
    if (nq_max < 1 || n_hyp_max < 1 || keep_max < 1) {
        set_last_error("reserve_reloc: nq_max, n_hyp_max and keep_max must be >= 1");
        return FL_ERR_ARG;
    }
    FL_CHECK(reserve_batch(nq_max));
    FL_CUDA(cudaSetDevice(map_->device()));
    const int hyp = std::max(n_hyp_max, reloc_hyp_max_), keep = std::max(keep_max, reloc_keep_max_);
    FL_CHECK(r_keys_.reserve(sizeof(unsigned long long) * 2 * (size_t)hyp));
    FL_CHECK(r_temp_.reserve(std::max<size_t>(1, sort_temp_bytes(hyp))));
    FL_CHECK(r_inl_.reserve(sizeof(int) * (size_t)hyp));
    FL_CHECK(r_x_.reserve(sizeof(double) * XLEN * (size_t)keep));
    FL_CHECK(r_P_.reserve(sizeof(double) * NDOF * NDOF * (size_t)keep));
    FL_CHECK(r_status_.reserve(sizeof(int) * 2 * (size_t)keep));
    FL_CHECK(r_logs_.reserve(sizeof(PassLog) * RELOC_MAX_LOGS * (size_t)keep));
    reloc_nq_max_ = std::max(reloc_nq_max_, nq_max);
    reloc_hyp_max_ = hyp;
    reloc_keep_max_ = keep;
    return FL_OK;
}

int Filter::relocalize_on_stream(const float* d_body, int nq, int n_hyp, const double* d_x26_hyp, const double* d_P, double R,
                                 const fl_reloc_params_t* prm, double* d_x_out, double* d_P_out, int* d_inliers,
                                 fl_reloc_row_t* d_rows, int* d_status4, cudaStream_t st) {
    const int dev = map_->device();
    if (!prm || nq < 1 || n_hyp < 1 || prm->keep < 1 || prm->stride < 1 || !(prm->r_inlier > 0.f)) {
        set_last_error("relocalize_device: null params, or nq, n_hyp, keep or stride < 1, or r_inlier not > 0");
        return FL_ERR_ARG;
    }
    if (!device_ptr(d_body, dev, 16) || !device_ptr(d_x26_hyp, dev, 8) || !device_ptr(d_P, dev, 8) || !device_ptr(d_x_out, dev, 8) ||
        !device_ptr(d_P_out, dev, 8) || !device_ptr(d_status4, dev, 4) || (d_inliers && !device_ptr(d_inliers, dev, 4)) ||
        (d_rows && !device_ptr(d_rows, dev, 8))) {
        set_last_error("relocalize_device: a buffer is not device memory on device %d (scan 16-byte, x, P and rows 8-byte, inliers "
                       "and status 4-byte aligned)", dev);
        return FL_ERR_ARG;
    }
    FL_CHECK(device_form_scope("relocalize_device", true));
    if (reloc_nq_max_ < 0) { set_last_error("relocalize_device: call fl_filter_reserve_reloc first"); return FL_ERR_STATE; }
    if (nq > reloc_nq_max_ || n_hyp > reloc_hyp_max_ || prm->keep > reloc_keep_max_) {
        set_last_error("relocalize_device: nq %d, n_hyp %d or keep %d exceed the %d, %d, %d fl_filter_reserve_reloc sized", nq, n_hyp,
                       prm->keep, reloc_nq_max_, reloc_hyp_max_, reloc_keep_max_);
        return FL_ERR_CAPACITY;
    }
    const int keep = std::min(prm->keep, n_hyp);
    int workers = 0, slots = 0, waves = 0;
    FL_CHECK(batch_plan(nq, keep, &workers, &slots, &waves));      // the batch below cannot refuse once work is enqueued
    size_t temp = r_temp_.bytes;
    if (sort_temp_bytes(n_hyp) > temp) {
        set_last_error("relocalize_device: the sort needs more temporary storage than fl_filter_reserve_reloc sized");
        return FL_ERR_CAPACITY;
    }
    FL_CUDA(cudaSetDevice(dev));
    bool joined = false;
    FL_CHECK(map_->query_begin(st, &joined));
    const int screened = (nq + prm->stride - 1) / prm->stride;
    const int chunks = (screened + RELOC_THREADS - 1) / RELOC_THREADS;
    int* inl = r_inl_.as<int>();
    unsigned long long* keys_in = r_keys_.as<unsigned long long>();
    unsigned long long* keys = keys_in + reloc_hyp_max_;
    FL_CUDA(cudaMemsetAsync(inl, 0, sizeof(int) * (size_t)n_hyp, st));
    k_reloc_screen<<<(unsigned)((long long)chunks * n_hyp), RELOC_THREADS, 0, st>>>(
        map_->view(), reinterpret_cast<const float4*>(d_body), nq, prm->stride, chunks, d_x26_hyp, prm->r_inlier * prm->r_inlier, inl);
    FL_CUDA(cudaGetLastError());
    k_reloc_keys<<<(n_hyp + RELOC_THREADS - 1) / RELOC_THREADS, RELOC_THREADS, 0, st>>>(inl, n_hyp, screened, keys_in);
    FL_CUDA(cudaGetLastError());
    FL_CUDA(cub::DeviceRadixSort::SortKeys(r_temp_.ptr, temp, keys_in, keys, n_hyp, 0, 64, st));
    k_reloc_gather<<<keep, RELOC_THREADS, 0, st>>>(keys, d_x26_hyp, d_P, r_x_.as<double>(), r_P_.as<double>());
    FL_CUDA(cudaGetLastError());
    FL_CHECK(update_batch_on_stream(d_body, nq, keep, r_x_.as<double>(), r_P_.as<double>(), R, r_status_.as<int>(),
                                    r_logs_.as<PassLog>(), st));
    k_reloc_rank<<<1, RELOC_THREADS, 0, st>>>(keys, inl, r_status_.as<int>(), r_logs_.as<PassLog>(), max_iter_ + 1, keep,
                                              prm->min_effct, r_x_.as<double>(), r_P_.as<double>(), d_rows, d_x_out, d_P_out, d_status4);
    FL_CUDA(cudaGetLastError());
    if (d_inliers) FL_CUDA(cudaMemcpyAsync(d_inliers, inl, sizeof(int) * (size_t)n_hyp, cudaMemcpyDeviceToDevice, st));
    return map_->query_end(st, joined);
}

}  // namespace fl
