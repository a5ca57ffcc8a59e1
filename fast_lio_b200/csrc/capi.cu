// extern "C" boundary (include/fastlio_b200.h).  Thin: argument checks, handle plumbing,
// status codes.  No torch types, no exceptions.
#include <atomic>
#include <chrono>
#include <cstring>
#include <mutex>
#include <new>

#include "../../include/fastlio_b200.h"
#include "filter.h"
#include "preprocess.h"
#include "scan.h"

namespace fl {
const char* last_error();
int nccl_unique_id(void* out128);
}  // namespace fl

// A map handle is shared by the filters and scan front ends created on it: they keep it alive, so destroying the
// handles in any order is safe (fl_map_destroy only drops the caller's reference).
struct fl_map {
    fl::Map* impl;
    std::mutex mu;
    std::atomic<int> refs{1};
};
static void map_retain(fl_map* m) { m->refs.fetch_add(1, std::memory_order_relaxed); }
static void map_release(fl_map* m) {
    if (m->refs.fetch_sub(1, std::memory_order_acq_rel) == 1) {
        delete m->impl;
        delete m;
    }
}
struct fl_filter {
    fl::Filter* impl;
    fl_map* map;
    fl::DeviceBuffer flush;
};

struct fl_scan {
    fl::ScanFrontEnd* impl;
    fl_map* map;
};
struct fl_scan_batch {
    fl::ScanBatch* impl;
    fl_map* map;
};
struct fl_localmap {
    fl::LocalMapCube cube;
    fl_map* map = nullptr;          // the map of the device form (retained), whose device holds the cube from then on
};

static_assert(sizeof(fl_pass_log_t) == sizeof(fl::PassLog), "pass-log layouts must match");

extern "C" {

const char* fl_last_error(void) { return fl::last_error(); }
int fl_version(void) { return 100; }
int fl_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

int fl_host_register(const void* ptr, unsigned long long bytes) {
    if (!ptr || !bytes) return FL_ERR_ARG;
    FL_CUDA(cudaHostRegister(const_cast<void*>(ptr), (size_t)bytes, cudaHostRegisterDefault));
    return FL_OK;
}
int fl_host_unregister(const void* ptr) {
    if (!ptr) return FL_ERR_ARG;
    FL_CUDA(cudaHostUnregister(const_cast<void*>(ptr)));
    return FL_OK;
}

// ------------------------------------------------------------------------------------ map
int fl_map_create(fl_map_t** out, int device, float downsample_size) {
    if (!out) { fl::set_last_error("fl_map_create: null out"); return FL_ERR_ARG; }
    *out = nullptr;
    int n = fl_device_count();
    if (n <= 0) { fl::set_last_error("fl_map_create: no CUDA device visible (this library has no CPU path)"); return FL_ERR_CUDA; }
    if (device < 0 || device >= n) { fl::set_last_error("fl_map_create: device %d out of range [0, %d)", device, n); return FL_ERR_ARG; }
    fl_map* m = new (std::nothrow) fl_map();
    if (!m) return FL_ERR_CAPACITY;
    m->impl = new (std::nothrow) fl::Map(device, downsample_size);
    if (!m->impl) { delete m; return FL_ERR_CAPACITY; }
    int rc = m->impl->init();
    if (rc != FL_OK) { delete m->impl; delete m; return rc; }
    *out = m;
    return FL_OK;
}
int fl_map_destroy(fl_map_t* m) {
    if (!m) return FL_OK;
    map_release(m);
    return FL_OK;
}
// Every call that may enqueue work on the handle's stream touch()es the map: the next device-buffer query joins that work.
#define MAP_GUARD(m)                                                             \
    if (!(m) || !(m)->impl) { fl::set_last_error("null map handle"); return FL_ERR_ARG; } \
    std::lock_guard<std::mutex> _lk((m)->mu);                                    \
    (m)->impl->touch()
// the device-buffer queries: stream-ordered on the caller's stream, they leave the handle's stream's frontier as it is
#define MAP_QUERY_GUARD(m)                                                       \
    if (!(m) || !(m)->impl) { fl::set_last_error("null map handle"); return FL_ERR_ARG; } \
    std::lock_guard<std::mutex> _lk((m)->mu)
// host forms settle the device forms' mutations first (Map::settle): a read-only call refreshes the host's view of the map, any
// other call also runs the re-pack / re-list they deferred
#define MAP_READ_GUARD(m)                                                        \
    MAP_GUARD(m);                                                                \
    { const int _rc = (m)->impl->settle(false); if (_rc != FL_OK) return _rc; }
#define MAP_MUTATE_GUARD(m)                                                      \
    MAP_GUARD(m);                                                                \
    { const int _rc = (m)->impl->settle(true); if (_rc != FL_OK) return _rc; }

int fl_map_set_downsample(fl_map_t* m, float v) { MAP_GUARD(m); m->impl->set_downsample(v); return FL_OK; }
int fl_map_build(fl_map_t* m, const float* pts, int n) { MAP_MUTATE_GUARD(m); return m->impl->build(pts, n); }
int fl_map_size(fl_map_t* m) { MAP_READ_GUARD(m); return m->impl->size(); }
int fl_map_validnum(fl_map_t* m) { MAP_READ_GUARD(m); return m->impl->validnum(); }
int fl_map_knn(fl_map_t* m, const float* q, int nq, int k, float* out_pts, float* out_d2, int* out_cnt) {
    MAP_READ_GUARD(m);
    if (nq > 0 && (!q || !out_pts || !out_d2 || !out_cnt)) { fl::set_last_error("fl_map_knn: null buffer"); return FL_ERR_ARG; }
    return m->impl->knn(q, nq, k, out_pts, out_d2, out_cnt);
}
int fl_map_nearest_search(fl_map_t* m, const float* q, int nq, int k, float max_dist, float* out_pts, float* out_d2, int* out_cnt) {
    MAP_READ_GUARD(m);
    if (nq > 0 && (!q || !out_pts || !out_d2 || !out_cnt)) { fl::set_last_error("fl_map_nearest_search: null buffer"); return FL_ERR_ARG; }
    return m->impl->nearest_search(q, nq, k, max_dist, out_pts, out_d2, out_cnt);
}
int fl_map_add_points(fl_map_t* m, const float* pts, int n, int downsample_on) {
    MAP_MUTATE_GUARD(m);
    int added = 0;
    int rc = m->impl->add_points(pts, n, downsample_on != 0, &added);
    return rc == FL_OK ? added : rc;
}
int fl_map_delete_boxes(fl_map_t* m, const float* boxes6, int nb) {
    MAP_MUTATE_GUARD(m);
    int deleted = 0;
    int rc = m->impl->delete_boxes(boxes6, nb, &deleted);
    return rc == FL_OK ? deleted : rc;
}
int fl_map_add_boxes(fl_map_t* m, const float* boxes6, int nb) {
    MAP_MUTATE_GUARD(m);
    int revived = 0;
    int rc = m->impl->add_boxes(boxes6, nb, &revived);
    return rc == FL_OK ? revived : rc;
}
int fl_map_acquire_removed(fl_map_t* m, float* out, int cap) {
    MAP_READ_GUARD(m);
    int n = 0;
    int rc = m->impl->acquire_removed(out, cap, &n);
    return rc == FL_OK ? n : rc;
}
int fl_map_flatten(fl_map_t* m, float* out, int cap) {
    MAP_READ_GUARD(m);
    int n = 0;
    int rc = m->impl->flatten(out, cap, &n);
    return rc == FL_OK ? n : rc;
}
int fl_map_box_search(fl_map_t* m, const float* boxes6, int nb, int* out_offsets, float* out_xyzi, int cap) {
    MAP_READ_GUARD(m);
    long long total = 0;
    int rc = m->impl->range_search(false, boxes6, nb, out_offsets, out_xyzi, cap, &total);
    return rc == FL_OK ? (int)total : rc;
}
int fl_map_radius_search(fl_map_t* m, const float* centers_xyzr, int nq, int* out_offsets, float* out_xyzi, int cap) {
    MAP_READ_GUARD(m);
    long long total = 0;
    int rc = m->impl->range_search(true, centers_xyzr, nq, out_offsets, out_xyzi, cap, &total);
    return rc == FL_OK ? (int)total : rc;
}
int fl_map_nearest_search_device(fl_map_t* m, const float* q_xyzi_device, int nq, int k, float max_dist,
                                 float* out_pts_device, float* out_d2_device, int* out_cnt_device, void* stream) {
    MAP_QUERY_GUARD(m);
    return m->impl->nearest_search_device(q_xyzi_device, nq, k, max_dist, out_pts_device, out_d2_device, out_cnt_device,
                                          static_cast<cudaStream_t>(stream));
}
int fl_map_range_workspace_bytes(fl_map_t* m, int nq, long long max_pairs, unsigned long long* out_bytes) {
    MAP_QUERY_GUARD(m);
    return m->impl->range_workspace_bytes(nq, max_pairs, out_bytes);
}
int fl_map_box_search_device(fl_map_t* m, const float* boxes6_device, int nb, int* out_offsets_device, float* out_xyzi_device,
                             long long cap, void* workspace_device, unsigned long long workspace_bytes, long long* status2_device,
                             void* stream) {
    MAP_QUERY_GUARD(m);
    return m->impl->range_search_device(false, boxes6_device, nb, out_offsets_device, out_xyzi_device, cap, workspace_device,
                                        workspace_bytes, status2_device, static_cast<cudaStream_t>(stream));
}
int fl_map_radius_search_device(fl_map_t* m, const float* centers_xyzr_device, int nq, int* out_offsets_device, float* out_xyzi_device,
                                long long cap, void* workspace_device, unsigned long long workspace_bytes, long long* status2_device,
                                void* stream) {
    MAP_QUERY_GUARD(m);
    return m->impl->range_search_device(true, centers_xyzr_device, nq, out_offsets_device, out_xyzi_device, cap, workspace_device,
                                        workspace_bytes, status2_device, static_cast<cudaStream_t>(stream));
}
int fl_map_build_device(fl_map_t* m, const float* pts_xyzi_device, int n, void* stream) {
    MAP_MUTATE_GUARD(m);
    return m->impl->build_from_caller(pts_xyzi_device, n, static_cast<cudaStream_t>(stream));
}
int fl_map_add_points_device(fl_map_t* m, const float* pts_xyzi_device, int n, int downsample_on, void* stream) {
    MAP_MUTATE_GUARD(m);
    int added = 0;
    int rc = m->impl->add_points_from_caller(pts_xyzi_device, n, downsample_on != 0, static_cast<cudaStream_t>(stream), &added);
    return rc == FL_OK ? added : rc;
}
// Device form: never settles (the host's view catches up at the next host-form call or fl_map_maintain)
int fl_map_add_points_async(fl_map_t* m, const float* pts_xyzi_device, const int* n_device, int n_max, int downsample_on,
                            int* status2_device, void* stream) {
    MAP_GUARD(m);
    return m->impl->add_points_async_checked(pts_xyzi_device, n_device, n_max, downsample_on != 0, status2_device,
                                             static_cast<cudaStream_t>(stream));
}
// Device form of Delete_Point_Boxes: never settles either
int fl_map_delete_boxes_async(fl_map_t* m, const float* boxes6_device, const int* nb_device, int nb_max, int* status2_device,
                              void* stream) {
    MAP_GUARD(m);
    return m->impl->delete_boxes_async_checked(boxes6_device, nb_device, nb_max, status2_device, static_cast<cudaStream_t>(stream));
}
int fl_map_maintain(fl_map_t* m, int* layout_changed) {
    MAP_GUARD(m);
    int changed = 0;
    const int rc = m->impl->settle(true, &changed);
    if (layout_changed) *layout_changed = changed;
    return rc;
}
int fl_map_tree_range(fl_map_t* m, float* box6) { MAP_READ_GUARD(m); if (!box6) return FL_ERR_ARG; return m->impl->tree_range(box6); }
int fl_map_rebuild(fl_map_t* m) { MAP_MUTATE_GUARD(m); return m->impl->rebuild(); }
int fl_map_stats(fl_map_t* m, int* out4) {
    MAP_READ_GUARD(m);
    if (!out4) return FL_ERR_ARG;
    out4[0] = m->impl->view().n_main; out4[1] = m->impl->overflow_leaves();
    out4[2] = m->impl->view().n_levels; out4[3] = m->impl->rebuild_count();
    return FL_OK;
}

int fl_map_set_cell_directory(fl_map_t* m, int on, float cell_size) {
    MAP_MUTATE_GUARD(m);
    m->impl->set_cell_directory(on != 0, cell_size > 0.f ? cell_size : 0.f);
    return m->impl->build_directory();
}
int fl_map_set_deterministic(fl_map_t* m, int on) {
    MAP_GUARD(m);
    return m->impl->set_deterministic(on != 0);
}
int fl_map_get_deterministic(fl_map_t* m, int* on) {
    MAP_GUARD(m);
    if (!on) { fl::set_last_error("fl_map_get_deterministic: null output"); return FL_ERR_ARG; }
    *on = m->impl->deterministic() ? 1 : 0;
    return FL_OK;
}
int fl_map_dir_stats(fl_map_t* m, int* out6) {
    MAP_READ_GUARD(m);
    if (!out6) return FL_ERR_ARG;
    return m->impl->dir_stats(out6);
}

// ------------------------------------------------------------------------------------ filter
#define FILTER_GUARD(f)                                                                        \
    if (!(f) || !(f)->impl) { fl::set_last_error("null filter handle"); return FL_ERR_ARG; }   \
    std::lock_guard<std::mutex> _lk((f)->map->mu);                                             \
    (f)->map->impl->touch()
// the filter's host forms settle the map first, with its deferred re-pack / re-list (Map::settle)
#define FILTER_HOST_GUARD(f)                                                                   \
    FILTER_GUARD(f);                                                                           \
    { const int _rc = (f)->map->impl->settle(true); if (_rc != FL_OK) return _rc; }

int fl_filter_create(fl_filter_t** out, fl_map_t* map, int max_points) {
    if (!out || !map || !map->impl) { fl::set_last_error("fl_filter_create: null argument"); return FL_ERR_ARG; }
    *out = nullptr;
    fl_filter* f = new (std::nothrow) fl_filter();
    if (!f) return FL_ERR_CAPACITY;
    f->map = map;
    f->impl = new (std::nothrow) fl::Filter(map->impl, max_points);
    if (!f->impl) { delete f; return FL_ERR_CAPACITY; }
    int rc = f->impl->init();
    if (rc != FL_OK) { delete f->impl; delete f; return rc; }
    map_retain(map);
    *out = f;
    return FL_OK;
}
int fl_filter_destroy(fl_filter_t* f) {
    if (!f) return FL_OK;
    f->flush.release();
    delete f->impl;
    map_release(f->map);
    delete f;
    return FL_OK;
}
int fl_filter_set_params(fl_filter_t* f, int max_iter, const double* limit23, int extr) { FILTER_GUARD(f); return f->impl->set_params(max_iter, limit23, extr); }
int fl_filter_set_solver(fl_filter_t* f, int mode) { FILTER_GUARD(f); if (mode < 0 || mode > 1) return FL_ERR_ARG; f->impl->set_solver(mode); return FL_OK; }
int fl_filter_set_fused(fl_filter_t* f, int on) { FILTER_GUARD(f); f->impl->set_fused(on != 0); return FL_OK; }
int fl_filter_set_search(fl_filter_t* f, int mode) { FILTER_GUARD(f); if (mode < 0 || mode > 1) return FL_ERR_ARG; f->impl->set_search_mode(mode); return FL_OK; }
int fl_filter_update(fl_filter_t* f, const float* body, int nq, double* x26, double* P, double R, double* solve_time_s) {
    FILTER_HOST_GUARD(f);
    return f->impl->update(body, nq, x26, P, R, solve_time_s);
}
int fl_filter_map_incremental(fl_filter_t* f, double fsm, int ekf_inited, int* out3) {
    FILTER_HOST_GUARD(f);
    int a = 0, b = 0, c = 0;
    int rc = f->impl->map_incremental(fsm, ekf_inited, &a, &b, &c);
    if (out3) { out3[0] = a; out3[1] = b; out3[2] = c; }
    return rc;
}
int fl_filter_map_incremental_device(fl_filter_t* f, double fsm, int ekf_inited, int* out4_device, void* stream) {
    FILTER_GUARD(f);
    return f->impl->map_incremental_on_stream(fsm, ekf_inited, out4_device, static_cast<cudaStream_t>(stream));
}
int fl_filter_get_nearest(fl_filter_t* f, float* out_pts, int* out_cnt, int nq) { FILTER_GUARD(f); return f->impl->get_nearest(out_pts, out_cnt, nq); }
int fl_filter_get_selected(fl_filter_t* f, unsigned char* out, int nq) { FILTER_GUARD(f); if (!out) return FL_ERR_ARG; return f->impl->get_selected(out, nq); }
int fl_filter_get_pass_logs(fl_filter_t* f, fl_pass_log_t* out, int cap) {
    FILTER_GUARD(f);
    if (!out || cap < 0) return FL_ERR_ARG;
    int n = 0;
    int rc = f->impl->get_pass_logs(reinterpret_cast<fl::PassLog*>(out), cap, &n);
    return rc == FL_OK ? n : rc;
}
// Device-buffer forms: the guard touch()es the map, so the join in Map::query_begin also orders this call after an earlier
// device-form update of the filter on another caller stream (they share the filter's buffers).
int fl_filter_update_device(fl_filter_t* f, const float* body_xyzi_device, int nq, double* x26_device, double* P_device, double R,
                            int* status2_device, void* stream) {
    FILTER_GUARD(f);
    return f->impl->update_on_stream(body_xyzi_device, nq, x26_device, P_device, R, status2_device, static_cast<cudaStream_t>(stream));
}
static_assert(sizeof(fl_pass_log_t) == sizeof(fl::PassLog) && offsetof(fl_pass_log_t, x_after) == offsetof(fl::PassLog, x_after),
              "fl_pass_log_t is fl::PassLog");
int fl_filter_reserve_batch(fl_filter_t* f, int nq_max) { FILTER_GUARD(f); return f->impl->reserve_batch(nq_max); }
int fl_filter_batch_plan(fl_filter_t* f, int nq, int n_hyp, int* out3) {
    FILTER_GUARD(f);
    if (!out3) { fl::set_last_error("fl_filter_batch_plan: null out3"); return FL_ERR_ARG; }
    return f->impl->batch_plan(nq, n_hyp, &out3[0], &out3[1], &out3[2]);
}
int fl_filter_update_batch_device(fl_filter_t* f, const float* body_xyzi_device, int nq, int n_hyp, double* x26_device, double* P_device,
                                  double R, int* status2_device, fl_pass_log_t* logs_device, void* stream) {
    FILTER_GUARD(f);
    return f->impl->update_batch_on_stream(body_xyzi_device, nq, n_hyp, x26_device, P_device, R, status2_device,
                                           reinterpret_cast<fl::PassLog*>(logs_device), static_cast<cudaStream_t>(stream));
}
int fl_reloc_expand_grid_device(const double* x26_prior_device, const fl_reloc_grid_t* grid, double* x26_hyp_device, void* stream) {
    return fl::reloc_expand_grid(x26_prior_device, grid, x26_hyp_device, static_cast<cudaStream_t>(stream));
}
int fl_filter_reserve_reloc(fl_filter_t* f, int nq_max, int n_hyp_max, int keep_max) {
    FILTER_GUARD(f);
    return f->impl->reserve_reloc(nq_max, n_hyp_max, keep_max);
}
int fl_filter_relocalize_device(fl_filter_t* f, const float* body_xyzi_device, int nq, int n_hyp, const double* x26_hyp_device,
                                const double* P_device, double R, const fl_reloc_params_t* params, double* x26_out_device,
                                double* P_out_device, int* inliers_device, fl_reloc_row_t* rows_device, int* status4_device,
                                void* stream) {
    FILTER_GUARD(f);
    return f->impl->relocalize_on_stream(body_xyzi_device, nq, n_hyp, x26_hyp_device, P_device, R, params, x26_out_device, P_out_device,
                                         inliers_device, rows_device, status4_device, static_cast<cudaStream_t>(stream));
}
int fl_filter_get_nearest_device(fl_filter_t* f, float* out_pts_device, int* out_cnt_device, int nq, void* stream) {
    FILTER_GUARD(f);
    return f->impl->get_nearest_on_stream(out_pts_device, out_cnt_device, nq, static_cast<cudaStream_t>(stream));
}
int fl_filter_get_selected_device(fl_filter_t* f, unsigned char* out_device, int nq, void* stream) {
    FILTER_GUARD(f);
    return f->impl->get_selected_on_stream(out_device, nq, static_cast<cudaStream_t>(stream));
}
int fl_filter_upload_scan(fl_filter_t* f, const float* body, int nq) { FILTER_GUARD(f); return f->impl->upload_scan(body, nq); }
int fl_filter_upload_state(fl_filter_t* f, const double* x26, const double* P, double R) {
    FILTER_GUARD(f);
    if (!x26 || !P) return FL_ERR_ARG;
    return f->impl->upload_state(x26, P, R);
}
int fl_filter_run(fl_filter_t* f) { FILTER_HOST_GUARD(f); return f->impl->run_passes(); }
int fl_filter_download_state(fl_filter_t* f, double* x26, double* P, int* n_pass) { FILTER_GUARD(f); return f->impl->download_state(x26, P, n_pass); }
int fl_filter_sync(fl_filter_t* f) { FILTER_GUARD(f); return f->impl->sync(); }
int fl_filter_debug_prof(fl_filter_t* f, long long* out16) {
    FILTER_GUARD(f);
    if (!out16) return FL_ERR_ARG;
    FL_CUDA(cudaMemcpy(out16, f->impl->ctl_device()->prof, sizeof(long long) * 16, cudaMemcpyDeviceToHost));
    for (int i = 0; i < 4; i++) out16[12 + i] = f->impl->host_ns()[i];       // host-side ns of the last fl_filter_update
    return FL_OK;
}
int fl_filter_gpu_launches(fl_filter_t* f) { FILTER_GUARD(f); return f->impl->gpu_launches(); }

int fl_filter_time_resident(fl_filter_t* f, int reps, int flush_l2, float* ms_total) {
    FILTER_GUARD(f);
    if (reps < 1 || !ms_total) return FL_ERR_ARG;
    fl::Filter* F = f->impl;
    cudaStream_t st = F->stream();
    FL_CUDA(cudaSetDevice(F->map()->device()));
    const size_t flush_bytes = 256u << 20;       // > 50 MB of H100 L2
    if (flush_l2) FL_CHECK(f->flush.reserve(flush_bytes));
    cudaEvent_t e0, e1;
    FL_CUDA(cudaEventCreate(&e0));
    FL_CUDA(cudaEventCreate(&e1));
    float total = 0.f;
    for (int r = 0; r < reps; r++) {
        FL_CHECK(F->restore_state());
        if (flush_l2) FL_CUDA(cudaMemsetAsync(f->flush.ptr, r & 0xff, flush_bytes, st));
        FL_CHECK(F->p2p_barrier());           // multi-GPU: all ranks enter the timed step together (no-op on one GPU)
        FL_CUDA(cudaEventRecord(e0, st));
        int rc = F->run_passes();
        if (rc != FL_OK) { cudaEventDestroy(e0); cudaEventDestroy(e1); return rc; }
        FL_CUDA(cudaEventRecord(e1, st));
        FL_CUDA(cudaEventSynchronize(e1));
        float ms = 0.f;
        FL_CUDA(cudaEventElapsedTime(&ms, e0, e1));
        total += ms;
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    *ms_total = total;
    return FL_OK;
}

// Wall time of `reps` whole fl_filter_update calls made back to back from native code -- what a C++ application
// (the reference is one) sees per scan: host buffers in, host buffers out, every copy inside.  Each repetition starts
// from the same prior, like the bench's resident loop.
int fl_filter_time_e2e(fl_filter_t* f, const float* body, int nq, const double* x26, const double* P, double R, int reps,
                       double* seconds, double* x26_out, double* P_out) {
    if (!f || !x26 || !P || !seconds || reps < 1) return FL_ERR_ARG;
    double x[fl::XLEN], Pw[fl::NDOF * fl::NDOF];
    const auto t0 = std::chrono::steady_clock::now();
    for (int r = 0; r < reps; r++) {
        memcpy(x, x26, sizeof(x));
        memcpy(Pw, P, sizeof(Pw));
        int rc = fl_filter_update(f, body, nq, x, Pw, R, nullptr);
        if (rc != FL_OK) return rc;
    }
    *seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    if (x26_out) memcpy(x26_out, x, sizeof(x));
    if (P_out) memcpy(P_out, Pw, sizeof(Pw));
    return FL_OK;
}

// Device time of the dominant phase alone: the kNN of one searching pass (k_update's search_only launch; k_search_c / k_search on the legacy path).
int fl_filter_time_search_pass(fl_filter_t* f, int reps, int flush_l2, float* ms_total) {
    FILTER_GUARD(f);
    if (reps < 1 || !ms_total) return FL_ERR_ARG;
    fl::Filter* F = f->impl;
    cudaStream_t st = F->stream();
    FL_CUDA(cudaSetDevice(F->map()->device()));
    const size_t flush_bytes = 256u << 20;
    if (flush_l2) FL_CHECK(f->flush.reserve(flush_bytes));
    cudaEvent_t e0, e1;
    FL_CUDA(cudaEventCreate(&e0));
    FL_CUDA(cudaEventCreate(&e1));
    float total = 0.f;
    for (int r = 0; r < reps; r++) {
        FL_CHECK(F->restore_state());
        if (flush_l2) FL_CUDA(cudaMemsetAsync(f->flush.ptr, r & 0xff, flush_bytes, st));
        FL_CUDA(cudaEventRecord(e0, st));
        int rc = F->launch_search_only();
        if (rc != FL_OK) { cudaEventDestroy(e0); cudaEventDestroy(e1); return rc; }
        FL_CUDA(cudaEventRecord(e1, st));
        FL_CUDA(cudaEventSynchronize(e1));
        float ms = 0.f;
        FL_CUDA(cudaEventElapsedTime(&ms, e0, e1));
        total += ms;
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    // leave the control block as uploaded
    FL_CHECK(F->restore_state());
    *ms_total = total;
    return FL_OK;
}

// ------------------------------------------------------------------------------------ scan front end
#define SCAN_GUARD(s)                                                                        \
    if (!(s) || !(s)->impl) { fl::set_last_error("null scan handle"); return FL_ERR_ARG; }   \
    std::lock_guard<std::mutex> _lk((s)->map->mu);                                             \
    (s)->map->impl->touch()

int fl_scan_create(fl_scan_t** out, fl_map_t* map) {
    if (!out) return FL_ERR_ARG;
    *out = nullptr;
    if (!map || !map->impl) { fl::set_last_error("fl_scan_create: null map handle"); return FL_ERR_ARG; }
    fl_scan* s = new (std::nothrow) fl_scan();
    if (!s) return FL_ERR_CAPACITY;
    s->map = map;
    s->impl = new (std::nothrow) fl::ScanFrontEnd(map->impl);
    if (!s->impl) { delete s; return FL_ERR_CAPACITY; }
    int rc = s->impl->init();
    if (rc != FL_OK) { delete s->impl; delete s; return rc; }
    map_retain(map);
    *out = s;
    return FL_OK;
}
int fl_scan_destroy(fl_scan_t* s) {
    if (!s) return FL_OK;
    delete s->impl;
    map_release(s->map);
    delete s;
    return FL_OK;
}
// the host forms first take over the cloud and counts of the device forms when those produced the current cloud
#define SCAN_HOST_GUARD(s)                                                                   \
    SCAN_GUARD(s);                                                                           \
    { const int _rc = (s)->impl->settle(); if (_rc != FL_OK) return _rc; }
int fl_scan_upload(fl_scan_t* s, const float* xyzi, const float* offset_ms, int n) { SCAN_HOST_GUARD(s); return s->impl->upload(xyzi, offset_ms, n); }
int fl_scan_undistort(fl_scan_t* s, const double* imu_pose22, int n_pose, const double* x26_end) {
    SCAN_HOST_GUARD(s);
    return s->impl->undistort(imu_pose22, n_pose, x26_end);
}
int fl_scan_voxel_downsample(fl_scan_t* s, float leaf_size) {
    SCAN_HOST_GUARD(s);
    int n = 0;
    int rc = s->impl->voxel_downsample(leaf_size, &n);
    return rc == FL_OK ? n : rc;
}
int fl_scan_download(fl_scan_t* s, int which, float* out_xyzi, int cap) {
    SCAN_HOST_GUARD(s);
    int n = 0;
    int rc = s->impl->download(which, out_xyzi, cap, &n);
    return rc == FL_OK ? n : rc;
}
int fl_filter_update_scan(fl_filter_t* f, fl_scan_t* s, double* x26, double* P, double R, double* solve_time_s) {
    FILTER_HOST_GUARD(f);
    if (!s || !s->impl || s->map != f->map) { fl::set_last_error("fl_filter_update_scan: the scan must live on the filter's map"); return FL_ERR_ARG; }
    { const int rc = s->impl->settle(); if (rc != FL_OK) return rc; }
    return f->impl->update_device(s->impl->down_device(), s->impl->down_count(), x26, P, R, solve_time_s);
}
// Device forms: the guard touch()es the map, so Map::query_begin orders them after everything enqueued on the handle's stream.
int fl_scan_reserve(fl_scan_t* s, int n_max, int n_pose_max) { SCAN_GUARD(s); return s->impl->reserve_device(n_max, n_pose_max); }
int fl_scan_upload_device(fl_scan_t* s, const float* xyzi_device, const float* offset_ms_device, const int* n_device, int n_max, void* stream) {
    SCAN_GUARD(s);
    return s->impl->upload_on_stream(xyzi_device, offset_ms_device, n_device, n_max, static_cast<cudaStream_t>(stream));
}
int fl_scan_undistort_device(fl_scan_t* s, const double* imu_pose22_device, const int* n_pose_device, int n_pose_max, const double* x26_end_device,
                             void* stream) {
    SCAN_GUARD(s);
    return s->impl->undistort_on_stream(imu_pose22_device, n_pose_device, n_pose_max, x26_end_device, static_cast<cudaStream_t>(stream));
}
int fl_scan_voxel_downsample_device(fl_scan_t* s, float leaf_size, int* n_out_device, void* stream) {
    SCAN_GUARD(s);
    return s->impl->voxel_downsample_on_stream(leaf_size, n_out_device, static_cast<cudaStream_t>(stream));
}
int fl_filter_update_scan_device(fl_filter_t* f, fl_scan_t* s, double* x26_device, double* P_device, double R, int* status2_device, void* stream) {
    FILTER_GUARD(f);
    if (!s || !s->impl || s->map != f->map) { fl::set_last_error("fl_filter_update_scan_device: the scan must live on the filter's map"); return FL_ERR_ARG; }
    if (!s->impl->dev_down_ready()) {
        fl::set_last_error("fl_filter_update_scan_device: no fl_scan_voxel_downsample_device since the scan's last upload");
        return FL_ERR_STATE;
    }
    return f->impl->update_scan_on_stream(s->impl->down_dev(), s->impl->down_count_dev(), s->impl->dev_n_max(), x26_device, P_device, R,
                                          status2_device, static_cast<cudaStream_t>(stream));
}
static_assert(sizeof(fl_scan_ref_t) == 16, "fl_scan_ref_t is two device pointers");
int fl_scan_get_ref(fl_scan_t* s, fl_scan_ref_t* out, int* n_max) {
    SCAN_GUARD(s);
    if (!out) { fl::set_last_error("fl_scan_get_ref: null out"); return FL_ERR_ARG; }
    const int m = s->impl->reserved_n_max();
    if (m < 0) { fl::set_last_error("fl_scan_get_ref: call fl_scan_reserve first"); return FL_ERR_STATE; }
    out->body_xyzi = reinterpret_cast<const float*>(s->impl->down_dev());
    out->n = s->impl->down_count_dev();
    if (n_max) *n_max = m;
    return FL_OK;
}
int fl_filter_update_scans_device(fl_filter_t* f, const fl_scan_ref_t* scans_device, int n_scans, int nq_max, double* x26_device,
                                  double* P_device, double R, int* status2_device, fl_pass_log_t* logs_device, void* stream) {
    FILTER_GUARD(f);
    return f->impl->update_scans_on_stream(scans_device, n_scans, nq_max, x26_device, P_device, R, status2_device,
                                           reinterpret_cast<fl::PassLog*>(logs_device), static_cast<cudaStream_t>(stream));
}
// ------------------------------------------------------------------------------------ scan front end of many scans
static_assert(sizeof(fl_scan_raw_t) == 48, "fl_scan_raw_t is six device pointers");
#define BATCH_GUARD(b)                                                                             \
    if (!(b) || !(b)->impl) { fl::set_last_error("null scan batch handle"); return FL_ERR_ARG; }   \
    std::lock_guard<std::mutex> _lk((b)->map->mu);                                                   \
    (b)->map->impl->touch()
int fl_scan_batch_create(fl_scan_batch_t** out, fl_map_t* map) {
    if (!out) return FL_ERR_ARG;
    *out = nullptr;
    if (!map || !map->impl) { fl::set_last_error("fl_scan_batch_create: null map handle"); return FL_ERR_ARG; }
    fl_scan_batch* b = new (std::nothrow) fl_scan_batch();
    if (!b) return FL_ERR_CAPACITY;
    b->map = map;
    b->impl = new (std::nothrow) fl::ScanBatch(map->impl);
    if (!b->impl) { delete b; return FL_ERR_CAPACITY; }
    map_retain(map);
    *out = b;
    return FL_OK;
}
int fl_scan_batch_destroy(fl_scan_batch_t* b) {
    if (!b) return FL_OK;
    delete b->impl;
    map_release(b->map);
    delete b;
    return FL_OK;
}
int fl_scan_batch_reserve(fl_scan_batch_t* b, int n_scans_max, int n_max, int n_pose_max) {
    BATCH_GUARD(b);
    return b->impl->reserve(n_scans_max, n_max, n_pose_max);
}
int fl_scan_batch_run_device(fl_scan_batch_t* b, const fl_scan_raw_t* raws_device, int n_scans, int n_max, int n_pose_max, int undistort,
                             float leaf_size, int* status2_device, void* stream) {
    BATCH_GUARD(b);
    return b->impl->run_on_stream(raws_device, n_scans, n_max, n_pose_max, undistort, leaf_size, status2_device,
                                  static_cast<cudaStream_t>(stream));
}
int fl_scan_batch_get_refs(fl_scan_batch_t* b, int which, const fl_scan_ref_t** refs_device, int* n_max) {
    BATCH_GUARD(b);
    return b->impl->refs(which, refs_device, n_max);
}
int fl_scan_batch_download(fl_scan_batch_t* b, int which, int slot, float* out_xyzi, int cap) {
    BATCH_GUARD(b);
    int n = 0;
    const int rc = b->impl->download(which, slot, out_xyzi, cap, &n);
    return rc == FL_OK ? n : rc;
}
// publish_frame_world / publish_frame_body / pointBodyToWorld                     laserMapping.cpp:177-220, :478-549, :909-921
int fl_scan_frame(fl_scan_t* s, int which, int frame, const double* x26, float* out_xyzi, int cap) {
    SCAN_HOST_GUARD(s);
    int n = 0;
    int rc = s->impl->frame(which, frame, x26, out_xyzi, cap, &n);
    return rc == FL_OK ? n : rc;
}
int fl_scan_frame_device(fl_scan_t* s, int which, int frame, const double* x26_device, float* out_xyzi_device, int* n_io_device, int cap,
                         int* status2_device, void* stream) {
    SCAN_GUARD(s);
    return s->impl->frame_on_stream(which, frame, x26_device, out_xyzi_device, n_io_device, cap, status2_device, static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------------------------ local-map cube
int fl_localmap_create(fl_localmap_t** out, double cube_len, float det_range) {
    if (!out) return FL_ERR_ARG;
    *out = nullptr;
    if (!(cube_len > 0.0) || !(det_range > 0.f)) { fl::set_last_error("fl_localmap_create: cube_len and det_range must be > 0"); return FL_ERR_ARG; }
    fl_localmap* l = new (std::nothrow) fl_localmap{fl::LocalMapCube(cube_len, det_range)};
    if (!l) return FL_ERR_CAPACITY;
    *out = l;
    return FL_OK;
}
int fl_localmap_destroy(fl_localmap_t* l) {
    if (!l) return FL_OK;
    fl_map* m = l->map;
    delete l;
    if (m) map_release(m);
    return FL_OK;
}
int fl_localmap_segment(fl_localmap_t* l, fl_map_t* map, const double* pos_lid, float* boxes6_out, int* n_deleted) {
    if (n_deleted) *n_deleted = 0;
    if (!l || !pos_lid) { fl::set_last_error("fl_localmap_segment: null argument"); return FL_ERR_ARG; }
    float boxes[18];
    int nb = 0;
    if (l->map) {                                     // the device form's cube is the cube: read it, slide, write it back
        std::lock_guard<std::mutex> lk(l->map->mu);
        int rc = l->cube.pull();
        if (rc == FL_OK) { nb = l->cube.slide(pos_lid, boxes); rc = l->cube.push(); }
        if (rc != FL_OK) return rc;
    } else {
        nb = l->cube.slide(pos_lid, boxes);
    }
    if (boxes6_out) for (int i = 0; i < nb * 6; i++) boxes6_out[i] = boxes[i];
    if (nb > 0 && map) {                              // if (cub_needrm.size() > 0) ikdtree.Delete_Point_Boxes(cub_needrm)  (:275)
        int deleted = fl_map_delete_boxes(map, boxes, nb);
        if (deleted < 0) return deleted;
        if (n_deleted) *n_deleted = deleted;
    }
    return nb;
}
int fl_localmap_get(fl_localmap_t* l, float* box6) {
    if (!l || !box6) return FL_ERR_ARG;
    if (l->map) {
        std::lock_guard<std::mutex> lk(l->map->mu);
        const int rc = l->cube.pull();
        if (rc != FL_OK) return rc;
    }
    if (!l->cube.initialized()) { fl::set_last_error("fl_localmap_get: the cube is placed by the first fl_localmap_segment call"); return FL_ERR_STATE; }
    l->cube.get(box6);
    return FL_OK;
}
// Device form: the guard touch()es the map, so the call is ordered after everything enqueued on the map's stream
int fl_localmap_segment_device(fl_localmap_t* l, fl_map_t* map, const double* x26_device, const int* n_scan_device,
                               float* boxes18_device, int* out3_device, void* stream) {
    if (!l) { fl::set_last_error("fl_localmap_segment_device: null cube handle"); return FL_ERR_ARG; }
    if (l->map && l->map != map) { fl::set_last_error("fl_localmap_segment_device: the cube lives on another map"); return FL_ERR_ARG; }
    MAP_GUARD(map);
    const int rc = l->cube.segment_on_stream(map->impl, x26_device, n_scan_device, boxes18_device, out3_device,
                                             static_cast<cudaStream_t>(stream));
    // the cube moved to the map's device (even when a later step of the call failed): from now on it is the cube, and the map
    // stays alive as long as the handle
    if (!l->map && l->cube.device_map()) { l->map = map; map_retain(map); }
    return rc;
}

// ------------------------------------------------------------------------------------ sensor preprocessing
struct fl_preprocessor {
    fl::Preprocessor* impl;
    std::mutex mu;
};

// fl_preprocess_params_t -> PpParams, with the checks of fl_preprocess_create (and of its batched form); `who` names the caller
static int pp_params(const char* who, int device, const fl_preprocess_params_t* pp, int n_raw_max, fl::PpParams* out) {
    if (!pp) { fl::set_last_error("%s: null parameters", who); return FL_ERR_ARG; }
    const fl_preprocess_params_t& p = *pp;
    if (p.lidar_type < FL_LIDAR_AVIA || p.lidar_type > FL_LIDAR_MARSIM || p.time_unit < 0 || p.time_unit > 3 || p.n_scans < 1 ||
        p.n_scans > 128 || p.point_filter_num < 1 || p.point_step < 1 || n_raw_max < 0 ||
        (p.lidar_type == FL_LIDAR_VELO16 && p.scan_rate < 1)) {
        fl::set_last_error("%s: bad lidar_type %d, time_unit %d, n_scans %d, scan_rate %d, point_filter_num %d, "
                           "point_step %d or n_raw_max %d", who, p.lidar_type, p.time_unit, p.n_scans, p.scan_rate, p.point_filter_num,
                           p.point_step, n_raw_max);
        return FL_ERR_ARG;
    }
    fl::PpParams q{};
    q.type = p.lidar_type;
    q.n_scans = p.n_scans;
    q.pfn = p.point_filter_num;
    q.step = p.point_step;
    const int offs[8] = {p.off_x, p.off_y, p.off_z, p.off_intensity, p.off_time, p.off_ring, p.off_tag, p.off_line};
    // the bytes each field occupies for this type (0: the type does not read it)
    const int avia[8] = {4, 4, 4, 1, 4, 0, 1, 1}, velo[8] = {4, 4, 4, 4, 4, 2, 0, 0}, oust[8] = {4, 4, 4, 4, 4, 0, 0, 0},
              sim[8] = {4, 4, 4, 4, 0, 0, 0, 0};
    const int* size = p.lidar_type == FL_LIDAR_AVIA ? avia : p.lidar_type == FL_LIDAR_VELO16 ? velo : p.lidar_type == FL_LIDAR_OUST64 ? oust : sim;
    for (int k = 0; k < 8; k++) {
        q.off[k] = size[k] ? offs[k] : -1;
        if (size[k] && (offs[k] < -1 || (offs[k] >= 0 && offs[k] + size[k] > p.point_step))) {
            fl::set_last_error("%s: field %d at offset %d does not fit point_step %d", who, k, offs[k], p.point_step);
            return FL_ERR_ARG;
        }
    }
    static const float scale[4] = {1.e3f, 1.f, 1.e-3f, 1.e-6f};     // preprocess.cpp:52-69
    q.scale = scale[p.time_unit];
    q.bb = p.blind * p.blind;
    q.omega_l = 0.361 * p.scan_rate;
    q.key_bits = 1;
    while ((1 << q.key_bits) <= p.n_scans) q.key_bits++;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) {
        cudaGetLastError();
        fl::set_last_error("%s: no CUDA device %d", who, device);
        return FL_ERR_ARG;
    }
    *out = q;
    return FL_OK;
}

int fl_preprocess_create(fl_preprocess_t** out, int device, const fl_preprocess_params_t* pp, int n_raw_max) {
    if (!out) return FL_ERR_ARG;
    *out = nullptr;
    fl::PpParams q{};
    FL_CHECK(pp_params("fl_preprocess_create", device, pp, n_raw_max, &q));
    fl_preprocess_t* h = new (std::nothrow) fl_preprocess_t();
    if (!h) return FL_ERR_CAPACITY;
    h->impl = new (std::nothrow) fl::Preprocessor(device, q, n_raw_max);
    if (!h->impl) { delete h; return FL_ERR_CAPACITY; }
    const int rc = h->impl->init();
    if (rc != FL_OK) { delete h->impl; delete h; return rc; }
    *out = h;
    return FL_OK;
}
int fl_preprocess_destroy(fl_preprocess_t* h) {
    if (!h) return FL_OK;
    delete h->impl;
    delete h;
    return FL_OK;
}
int fl_preprocess_device(fl_preprocess_t* h, const void* raw_device, const int* n_raw_device, int n_raw_max, float* xyzi_out_device,
                         float* offset_ms_out_device, int* out2_device, float* last_ms_device, void* stream) {
    if (!h || !h->impl) { fl::set_last_error("null preprocess handle"); return FL_ERR_ARG; }
    std::lock_guard<std::mutex> lk(h->mu);
    return h->impl->run_device(raw_device, n_raw_device, n_raw_max, xyzi_out_device, offset_ms_out_device, out2_device, last_ms_device,
                               static_cast<cudaStream_t>(stream));
}
int fl_preprocess(fl_preprocess_t* h, const void* raw_host, int n_raw, float* xyzi_out, float* offset_ms_out, int cap, float* last_ms) {
    if (!h || !h->impl) { fl::set_last_error("null preprocess handle"); return FL_ERR_ARG; }
    std::lock_guard<std::mutex> lk(h->mu);
    return h->impl->run_host(raw_host, n_raw, xyzi_out, offset_ms_out, cap, last_ms);
}
// ------------------------------------------------------------------------------------ preprocessing of many frames
static_assert(sizeof(fl_preprocess_raw_t) == 16, "fl_preprocess_raw_t is two device pointers");
struct fl_preprocess_batch {
    fl::PreprocessBatch* impl;
    std::mutex mu;
};
int fl_preprocess_batch_create(fl_preprocess_batch_t** out, int device, const fl_preprocess_params_t* pp, int n_slots_max, int n_raw_max) {
    if (!out) return FL_ERR_ARG;
    *out = nullptr;
    fl::PpParams q{};
    FL_CHECK(pp_params("fl_preprocess_batch_create", device, pp, n_raw_max, &q));
    if (n_slots_max < 0) { fl::set_last_error("fl_preprocess_batch_create: n_slots_max %d < 0", n_slots_max); return FL_ERR_ARG; }
    if (n_slots_max > fl::PreprocessBatch::SLOTS_MAX || (long long)n_slots_max * n_raw_max > (long long)INT_MAX) {
        fl::set_last_error("fl_preprocess_batch_create: %d slots (at most %d) or %lld rows (at most INT_MAX)", n_slots_max,
                           fl::PreprocessBatch::SLOTS_MAX, (long long)n_slots_max * n_raw_max);
        return FL_ERR_CAPACITY;
    }
    fl_preprocess_batch_t* b = new (std::nothrow) fl_preprocess_batch_t();
    if (!b) return FL_ERR_CAPACITY;
    b->impl = new (std::nothrow) fl::PreprocessBatch(device, q, n_slots_max, n_raw_max);
    if (!b->impl) { delete b; return FL_ERR_CAPACITY; }
    const int rc = b->impl->init();
    if (rc != FL_OK) { delete b->impl; delete b; return rc; }
    *out = b;
    return FL_OK;
}
int fl_preprocess_batch_destroy(fl_preprocess_batch_t* b) {
    if (!b) return FL_OK;
    delete b->impl;
    delete b;
    return FL_OK;
}
#define PP_BATCH_GUARD(b)                                                                              \
    if (!(b) || !(b)->impl) { fl::set_last_error("null preprocess batch handle"); return FL_ERR_ARG; } \
    std::lock_guard<std::mutex> _lk((b)->mu)
int fl_preprocess_batch_run_device(fl_preprocess_batch_t* b, const fl_preprocess_raw_t* raws_device, int n_slots, int n_max,
                                   int* status2_device, void* stream) {
    PP_BATCH_GUARD(b);
    return b->impl->run_device(raws_device, n_slots, n_max, status2_device, static_cast<cudaStream_t>(stream));
}
int fl_preprocess_batch_get_outputs(fl_preprocess_batch_t* b, float** xyzi, float** offset_ms, int** out2, float** last_ms, int* n_raw_max) {
    PP_BATCH_GUARD(b);
    b->impl->outputs(xyzi, offset_ms, out2, last_ms, n_raw_max);
    return FL_OK;
}
int fl_preprocess_batch_download(fl_preprocess_batch_t* b, int slot, float* out_xyzi, float* out_offset_ms, int cap, float* last_ms) {
    PP_BATCH_GUARD(b);
    int n = 0;
    const int rc = b->impl->download(slot, out_xyzi, out_offset_ms, cap, last_ms, &n);
    return rc == FL_OK ? n : rc;
}

// ------------------------------------------------------------------------------------ multi-GPU
int fl_comm_unique_id(void* out128) { if (!out128) return FL_ERR_ARG; return fl::nccl_unique_id(out128); }
int fl_filter_comm_init(fl_filter_t* f, int nranks, int rank, const void* id128) {
    FILTER_GUARD(f);
    if (nranks > 1 && !id128) return FL_ERR_ARG;
    return f->impl->comm_init(nranks, rank, id128);
}
int fl_filter_p2p_handle(fl_filter_t* f, void* out64) { FILTER_GUARD(f); if (!out64) return FL_ERR_ARG; return f->impl->p2p_local_handle(out64); }
int fl_filter_p2p_connect(fl_filter_t* f, int nranks, int rank, const void* handles) { FILTER_GUARD(f); return f->impl->p2p_connect(nranks, rank, handles); }
int fl_filter_set_shard(fl_filter_t* f, int q_begin, int q_end) { FILTER_GUARD(f); return f->impl->set_shard(q_begin, q_end); }

}  // extern "C"
