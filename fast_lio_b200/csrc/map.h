// Host-side owner of the device point map (the H100 counterpart of KD_TREE<PointType>,
// reference include/ikd-Tree/ikd_Tree.h:48-341).  All methods return fl::Status.
#pragma once
#include <algorithm>
#include <vector>

#include "map.cuh"

namespace fl {

struct DeviceBuffer {
    void* ptr = nullptr;
    size_t bytes = 0;
    int reserve(size_t want);      // grow-only (x1.5), contents NOT preserved
    void release();
    template <class T> T* as() const { return static_cast<T*>(ptr); }
};

// true: p is device memory of `device` (or managed memory allocated against it), aligned to `align` bytes
bool device_ptr(const void* p, int device, size_t align);

class Map {
public:
    Map(int device, float downsample_size);
    ~Map();
    int init();

    // KD_TREE::Build (ikd_Tree.cpp:409-423).  pts: n x (x, y, z, intensity), host memory.
    int build(const float* pts_xyzi, int n);
    // same, from points already resident on this device
    int build_device(const float4* d_pts_xyzi, int n);
    // KD_TREE::Nearest_Search, batched (ikd_Tree.cpp:426-461); host buffers
    int knn(const float* q_xyzi, int nq, int k, float* out_pts, float* out_d2, int* out_cnt);
    // KD_TREE::Nearest_Search(point, k, .., max_dist), batched, 1 <= k <= KNN_KMAX (fl_map_nearest_search); host buffers
    int nearest_search(const float* q_xyzi, int nq, int k, float max_dist, float* out_pts, float* out_d2, int* out_cnt);
    // KD_TREE::Delete_Point_Boxes (ikd_Tree.cpp:632-658); returns the number of points invalidated in *deleted
    int delete_boxes(const float* boxes6, int nb, int* deleted);
    // KD_TREE::Add_Points (ikd_Tree.cpp:478-573); *added = the reference's return value
    int add_points(const float* pts_xyzi, int n, bool downsample_on, int* added);
    int add_points_device(const float4* d_pts_xyzi, int n, bool downsample_on, int* added);
    // KD_TREE::Add_Point_Boxes (ikd_Tree.cpp:576-603) / acquire_removed_points (:661-676)
    int add_boxes(const float* boxes6, int nb, int* revived);
    int acquire_removed(float* out_xyzi, int cap, int* n_out);
    // all valid points, unordered (flatten(Root_Node, ..., NOT_RECORD), ikd_Tree.cpp:1627-1658)
    int flatten(float* out_xyzi, int cap, int* n_out);
    // KD_TREE::Box_Search (ikd_Tree.cpp:464-468, radius = false; queries: nq x (min xyz, max xyz)) and KD_TREE::Radius_Search
    // (:470-475, radius = true; queries: nq x (x, y, z, r)), batched.  Host buffers.  The points of query i are
    // out_xyzi[out_offsets[i] .. out_offsets[i + 1]) (only the first `cap` of all are written); *total = out_offsets[nq].
    int range_search(bool radius, const float* queries, int nq, int* out_offsets, float* out_xyzi, int cap, long long* total);

    // Device-buffer forms (fl_map_*_device): stream-ordered on the caller's stream `st`, no host synchronisation, capturable.
    int nearest_search_device(const float* q_xyzi, int nq, int k, float max_dist, float* out_pts, float* out_d2, int* out_cnt, cudaStream_t st);
    int range_workspace_bytes(int nq, long long max_pairs, unsigned long long* out) const;
    int range_search_device(bool radius, const float* queries, int nq, int* out_offsets, float* out_xyzi, long long cap,
                            void* workspace, unsigned long long workspace_bytes, long long* status2, cudaStream_t st);
    // Build / Add_Points from caller device memory, read in order on `st` (synchronous, like the host forms)
    int build_from_caller(const float* d_pts_xyzi, int n, cudaStream_t st);
    int add_points_from_caller(const float* d_pts_xyzi, int n, bool downsample_on, cudaStream_t st, int* added);
    // every call that may enqueue work on the handle's stream marks it, so the next device query joins that work
    void touch() { front_stale_ = true; }
    // the join of every device-buffer call on a caller's stream `st` (map queries, fl_filter_update_device): outside capture,
    // query_begin makes `st` wait for the handle's stream and query_end makes the handle's stream wait for `st`
    int query_begin(cudaStream_t st, bool* joined);
    int query_end(cudaStream_t st, bool joined);
    // Device forms of Add_Points (fl_map_add_points_async, fl_filter_map_incremental_device): enqueued on the caller's stream `st`,
    // the point counts read from device memory when `st` reaches them, no host synchronisation, no allocation (except the one
    // documented case in async_prepare), grids sized from n_max.  A one-thread plan kernel checks the headroom first; when the
    // batch might not fit, nothing is changed and the status is FL_ERR_CAPACITY.
    //   async_prepare: the host's bound of the headroom for one more call of up to n_max points.  Outside capture a call that
    //     might not fit settles the map and grows it first (synchronously); on a capturing stream it is FL_ERR_CAPACITY.
    //   mutation_begin / mutation_end: the join of a device-form mutation (everything enqueued on the handle so far comes first)
    int async_prepare(int n_max, cudaStream_t st, const char* what);
    int mutation_begin(cudaStream_t st, bool* joined);
    int mutation_end(cudaStream_t st, bool joined);
    // one or two Add_Points (list a with downsample_a, then list b plain; b may be null) of up to n_max points each, counts
    // *na / *nb in device memory (clamped to [0, n_max]), all-or-nothing together.  out: status2 = (status, added) when
    // list_counts is null, else out4 = (list_counts[0], list_counts[1], added, status)
    int add_points_async(const float4* pa, const int* na, bool downsample_a, const float4* pb, const int* nb, int n_max,
                         const int* list_counts, int* out, cudaStream_t st);
    // the public fl_map_add_points_async: argument checks, async_prepare, the join, add_points_async
    int add_points_async_checked(const float* d_pts, const int* d_n, int n_max, bool downsample_on, int* d_status2, cudaStream_t st);
    // Device form of Delete_Point_Boxes (fl_map_delete_boxes_async), with the conventions of the Add_Points forms above.
    //   delete_prepare: outside capture, room in the removed-points record by the host's bound (the one synchronous case)
    //   enqueue_delete: up to nb_max boxes (min xyz, max xyz) at `boxes`, count *nb_dev (clamped to [0, nb_max]); a one-thread
    //     plan checks the record's room first.  status2 = (status, deleted).  Between mutation_begin and mutation_end.
    int delete_prepare(cudaStream_t st);
    int enqueue_delete(const float* boxes, const int* nb_dev, int nb_max, int* status2, cudaStream_t st);
    int delete_boxes_async_checked(const float* d_boxes, const int* d_nb, int nb_max, int* d_status2, cudaStream_t st);
    // Host-form calls settle first.  Read-only ones (full = false) refresh the host's mirror of the device counters (one read-back
    // when a device-form mutation may have run); the others (full = true) also run the re-pack / re-list the device forms deferred,
    // by the host form's rules.  *layout_changed: buffers or leaves moved since the last report (captured graphs are stale).
    int settle(bool full, int* layout_changed = nullptr);
    // re-sort every valid point into fresh, evenly filled leaves (ikd-Tree's Rebuild, ikd_Tree.cpp:736-764)
    int rebuild();
    // re-list every live slot in the hashed cell directory (map.cuh); done by build / rebuild, and when inserts crowd it
    int build_directory();
    void set_cell_directory(bool on, float cell_size) { dir_enabled_ = on; cell_override_ = cell_size; }
    int dir_rebuild_count() const { return n_dir_rebuilds_; }
    int dir_stats(int* out6) const;
    // recompute every AABB from the valid points (after deletions)
    int refit();
    // the same launches on `st`; gate (may be null): every kernel returns at once when *gate is 0 on the device
    int refit_on(cudaStream_t st, const int* gate);

    int size() const { return n_valid_ + n_tomb_; }       // KD_TREE::size()  (valid + lazily deleted; settle(false) first)
    int validnum() const { return n_valid_; }             // KD_TREE::validnum()
    void set_downsample(float v) { downsample_ = v; }
    // the keyed tie rule of k-NN and down-sampling (map.cuh, "tie rules") and flatten's sorted rows; waits for the stream first
    int set_deterministic(bool on);
    bool deterministic() const { return det_; }
    float downsample() const { return downsample_; }
    int tree_range(float* box6);

    const MapView& view() const { return v_; }
    cudaStream_t stream() const { return stream_; }
    int device() const { return device_; }
    int rebuild_count() const { return n_rebuilds_; }
    int overflow_leaves() const;

    int fill_ = 24;            // slots populated per leaf at (re)build time; the rest absorb inserts
    int min_pool_ = 65536;     // minimum overflow-pool size in leaves (32 MB)
    float rebuild_overflow_frac_ = 0.05f;   // rebuild when overflow leaves exceed this fraction of main leaves

private:
    // workspace of a range query: byte offsets from its first 256-byte boundary (range_workspace), room for max_pairs pairs
    struct RangeWorkspace { size_t q, lcnt, loff, ctl, part, cub, cub_bytes, pairs, pcnt, poff, bytes; long long max_pairs; };
    int range_workspace(int nq, long long max_pairs, RangeWorkspace& w) const;
    void range_layout(int nq, long long max_pairs, size_t cub_bytes, RangeWorkspace& w) const;
    int scan_blocks() const { return 2 * std::max(n_sm_, 1); }      // grid of the device-length scan
    // the two stages of every range query, enqueued on `st` over the workspace at `base`: count (writes status2), then emit
    int range_count(bool radius, int nq, const RangeWorkspace& w, char* base, long long* status2, cudaStream_t st);
    int range_emit(bool radius, int nq, const RangeWorkspace& w, char* base, int* out_offsets, float4* out, long long cap, cudaStream_t st);
    // the kernel and grid of every nearest search; knn_host runs it on host buffers
    void launch_knn(bool gated, const float4* q, int nq, int k, float md2, float4* p, float* d2, int* cnt, cudaStream_t st);
    int knn_host(bool gated, const float* q_xyzi, int nq, int k, float md2, float* out_pts, float* out_d2, int* out_cnt);
    int wait_for_caller(cudaStream_t st, const char* what);

    int ensure_capacity(int n_points);
    int build_from_sorted(const float4* d_src, int n);
    int insert_device(const float4* d_pts, int n);
    int maybe_rebuild();
    int add_points_host(const float4* d_pts, int n, bool downsample_on, int* added);
    // the host's n_valid_ / n_tomb_ into the device counters the device forms keep (after every host-form mutation)
    int publish_counts();
    // the removed-points record: room for every valid point on top of what it holds (synchronous), and its capacity in points
    int removed_room();
    int removed_cap() const;
    // device forms: one Add_Points of the batch at pts, effective count at counters_[slot], after the plan kernel
    int enqueue_add(const float4* pts, int slot, bool downsample_on, int n_max, cudaStream_t st);
    int enqueue_insert(const float4* pts, const int* n_dev, int n_max, cudaStream_t st);
    bool async_fits(long long n_max) const;
    int async_grow(int n_max, bool pool);
    int async_scratch(int n_max, bool may_allocate);

    // device forms: pending_ = unsettled device-form mutations; captured_ = one was captured into a graph, so replays may
    // mutate the map at any time and every settle reads back; ub_n_ = points the device forms may have inserted since the last
    // settle (the host's bound of the headroom they used)
    bool pending_ = false, captured_ = false, async_used_ = false, layout_dirty_ = false;
    // owed by the next full settle (fl_map_maintain, a host-form mutation): the deferred re-pack / re-list (due_) and room for a
    // refused call (refused_).  Read-only settles only add to them.
    bool due_ = false, refused_ = false;
    long long ub_n_ = 0;
    int async_n_max_ = 0;
    DeviceBuffer a_keys_in_, a_keys_out_, a_vals_in_, a_vals_out_, a_groups_, a_ins_, a_slots_, a_fix_, a_cub_, cellcnt_;

    int device_;
    float downsample_;
    cudaStream_t stream_ = nullptr;
    MapView v_;
    int n_valid_ = 0, n_tomb_ = 0, n_rebuilds_ = 0;
    bool built_ = false;

    DeviceBuffer pts_, payload_, next_, counters_, dir_tab_, dir_lists_, removed_, ins_slots_, dir_fix_;
    bool record_removed_ = false;
    int n_removed_ = 0;
    bool dir_enabled_ = true;
    bool det_ = false;          // fl_map_set_deterministic
    float cell_override_ = 0.f;           // 0: cell edge = 2 x downsample size
    size_t dir_min_cap_ = 0, dir_min_pool_ = 0;
    int n_dir_rebuilds_ = 0;
    DeviceBuffer ebox_[MAX_LEVELS];
    DeviceBuffer segid_, segtab_[2], bbox_;        // k-d partition build scratch
    DeviceBuffer src_, keys_in_, keys_out_, vals_in_, vals_out_, cub_tmp_, scratch_, scratch2_, scratch3_;
    // host-buffer range search: the workspace (laid out for range_ws_pairs_ pairs, the most of any call so far) and status2 + output
    DeviceBuffer range_ws_, range_out_;
    long long range_ws_pairs_ = 0;
    int n_sm_ = 0;                  // multiprocessors of the device (grid sizing)
    int* h_counters_ = nullptr;     // pinned mirror of the device counters
    // device-buffer queries: ev_front_ marks the handle's stream for callers to wait on (re-recorded when front_stale_),
    // ev_caller_ a caller's stream for the handle's stream to wait on
    cudaEvent_t ev_front_ = nullptr, ev_caller_ = nullptr;
    bool front_stale_ = true;
};

}  // namespace fl
