// Host-side owner of the per-scan iterated-EKF measurement update on the device: the H100
// counterpart of esekfom::esekf<state_ikfom,12,input_ikfom>::update_iterated_dyn_share_modified
// (reference include/IKFoM_toolkit/esekfom/esekfom.hpp:1619-1931) with h_share_model
// (reference src/laserMapping.cpp:638-754) bound as a fused device measurement model.
#pragma once
#include "lie.cuh"
#include "map.h"
#include "upd_plan.h"

namespace fl {

// Per-pass record, same layout as the oracle's OraclePassLog (tests compare them field by field).
struct PassLog {
    int searched, valid, effct, converged;
    double res_sum;
    double HtH[144];
    double Hth[12];
    double x_after[XLEN];
};

// Device-resident control block of one update (what the reference keeps in locals of
// update_iterated_dyn_share_modified and in members x_, P_ of esekf).
struct FilterCtl {
    int iter;            // loop variable i, starts at -1            (esekfom.hpp:1633)
    int t;               // converged-step counter                   (esekfom.hpp:1624)
    int converge;        // dyn_share.converge: run the kNN on the next pass
    int done;            // the update has returned
    int n_pass;          // passes executed so far
    int max_iter;        // maximum_iter
    int extrinsic_est;   // extrinsic_est_en (laserMapping.cpp:739)
    int error;           // device-side failure: 1 singular system, 2 a peer never delivered its sums, 3 a block gave up waiting
    int ticket;          // k_residual: blocks finished so far (the last one reduces and solves)
    int gen;             // k_update: passes published so far (the workers of the next pass spin on it)
    double R;            // LASER_POINT_COV passed as R
    double limit[NDOF];
    double x[XLEN];
    double x_prop[XLEN];
    double P[NDOF * NDOF];
    double P_prop[NDOF * NDOF];
    long long prof[16];  // clock64() stamps of the last solve_pass (thread 0), for tuning
    double x_search[XLEN];   // the state the last searching pass used (Nearest_Points belong to it)
    FilterCtl* host_mirror;  // page-locked, device-mapped copy on the host: the pass that ends the update stores the result there
};

struct ScanView {
    const float4* body;      // [Q] body-frame points (x, y, z, intensity)      feats_down_body
    float4* nearest;         // [Q * 5] neighbours of the last search pass      Nearest_Points
    int* nearest_cnt;        // [Q]
    unsigned char* selected; // [Q] point_selected_surf (persists across passes, trap T3)
    float4* normvec;         // [Q] (n, pd2)                                    normvec
    float4* plane;           // [Q] pabcd of the last search pass's plane fit (reused by the passes that do not search)
    double* srange;          // [Q] sqrt(|p_body|) of the score (laserMapping.cpp:681), cached by the searching passes
    int q_begin, q_end;      // this rank's shard of the scan
    int Q;
};

struct NcclApi;
struct UpdArgs;
struct StateIn;
struct ScanSlot;

// Peer-memory exchange of the per-pass sums (fused into k_residual's solver block): every rank owns a
// mailbox [2 epoch parities][nranks][96] values, each two epoch-tagged 8-byte words; peers store into it over NVLink.
constexpr int P2P_MAX_RANKS = 8;
struct P2PState {
    double* peer_mail[P2P_MAX_RANKS];                 // mailbox of rank r (mapped through CUDA IPC)
    unsigned long long* peer_flag[P2P_MAX_RANKS];     // its flag array
    unsigned long long* peer_bar[P2P_MAX_RANKS];      // rank r's barrier slots (k_p2p_barrier: aligns the ranks before a timed step)
    unsigned long long epoch;                         // passes exchanged so far (identical on all ranks)
    unsigned long long bar_epoch;                     // barriers passed so far
    int nranks, rank;
};

class Filter {
public:
    Filter(Map* map, int max_points);
    ~Filter();
    int init();
    int set_params(int max_iter, const double* limit23, int extrinsic_est_en);
    void set_search_mode(int mode) { search_mode_ = mode; }
    void set_pdl(bool on) { pdl_ = on; }
    void set_solver(int mode) { solver_ = mode; }       // 1 (default): one ne x ne solve; 0: the reference's two 23x23 inversions, literally

    // whole update with host buffers (scan H2D, state H2D, passes, state D2H)
    int update(const float* body_xyzi, int nq, double* x26, double* P, double R, double* solve_time_s);
    // same with feats_down_body already in HBM on the map's device (ScanFrontEnd::down_device())
    int update_device(const float4* d_body, int nq, double* x26, double* P, double R, double* solve_time_s);
    // pieces, for device-resident benchmarking / pipelines
    int upload_scan(const float* body_xyzi, int nq);
    int set_scan_device(const float4* d_body, int nq);
    int upload_state(const double* x26, const double* P, double R, bool snapshot = true);
    int restore_state();                               // device-side copy of the last uploaded state -> control block
    int run_passes();                                  // enqueue every pass on the stream (no sync)
    int launch_search_only();
    int launch_residual_only();
    int download_state(double* x26, double* P, int* n_pass);
    int sync();
    // the whole update on caller device buffers, enqueued on the caller's stream `st` (fl_filter_update_device): the scan is
    // copied into body_, a state-in kernel sets the control block up from x26 / P, k_update runs the passes and a state-out
    // kernel writes x26 / P (on success) and status2 = (status, passes).  No host synchronisation, no allocation.
    int update_on_stream(const float* d_body, int nq, double* d_x26, double* d_P, double R, int* d_status2, cudaStream_t st);
    // Nearest_Points / point_selected_surf of the last update into caller device buffers, on `st`
    int get_nearest_on_stream(float* d_pts, int* d_cnt, int nq, cudaStream_t st);
    int get_selected_on_stream(unsigned char* d_out, int nq, cudaStream_t st);
    // update_on_stream on a scan bound in place (the scan front end's down-sampled cloud, fl_filter_update_scan_device) whose
    // point count is read from device memory: d_n is copied into the filter's own count, grids follow n_max (k_update_n)
    int update_scan_on_stream(const float4* d_body, const int* d_n, int n_max, double* d_x26, double* d_P, double R, int* d_status2, cudaStream_t st);
    // the largest scan the per-point buffers hold without growing (max_points at create, or the largest scan since)
    int capacity() const;
    // One scan from n_hyp priors (fl_filter_update_batch_device), each exactly as update_on_stream would run it, in waves of
    // `slots` hypotheses per k_update_batch launch.  The batch has buffers of its own (b_*): the scan's copy, per slot a control
    // block, a publication block and partial rows, and caches of slots x nq rows, so the filter's own state, scan binding and
    // results stay those of its last single update.  The map's walk counter (fl_map_dir_stats) does count the batch's walks.
    // reserve_batch sizes them for every nq <= nq_max (grow-only, synchronous; a grow moves them); batch_plan gives the workers
    // per hypothesis, the slots per wave and the waves for nq points and n_hyp hypotheses.
    int reserve_batch(int nq_max);
    int batch_plan(int nq, int n_hyp, int* workers, int* slots, int* waves) const;
    int update_batch_on_stream(const float* d_body, int nq, int n_hyp, double* d_x26, double* d_P, double R, int* d_status2,
                               PassLog* d_logs, cudaStream_t st);
    // The batch with a scan per slot (fl_filter_update_scans_device): slot s runs the table entry d_refs[s] in place, on the batch's
    // buffers, in waves planned at nq_max (UR_BATCH on scans_caps_); k_scans_state_in validates each entry and count on the device.
    int update_scans_on_stream(const fl_scan_ref_t* d_refs, int n_scans, int nq_max, double* d_x26, double* d_P, double R,
                               int* d_status2, PassLog* d_logs, cudaStream_t st);
    // Relocalisation (fl_filter_relocalize_device, reloc.cu): screen n_hyp states by inliers (k_reloc_screen), rank them (cub radix
    // sort), run update_batch_on_stream from the first `keep` and choose one (k_reloc_rank).  Its own buffers (r_*) hold the
    // counts, the keys and the survivors' x, P, status and logs; reserve_reloc sizes them and calls reserve_batch (grow-only).
    int reserve_reloc(int nq_max, int n_hyp_max, int keep_max);
    int relocalize_on_stream(const float* d_body, int nq, int n_hyp, const double* d_x26_hyp, const double* d_P, double R,
                             const fl_reloc_params_t* prm, double* d_x_out, double* d_P_out, int* d_inliers, fl_reloc_row_t* d_rows,
                             int* d_status4, cudaStream_t st);

    // map_incremental (laserMapping.cpp:427-474) on the device: classify every scan point with the final
    // state and its cached neighbours, then Add_Points(PointToAdd, true) + Add_Points(PointNoNeedDownsample, false)
    int map_incremental(double filter_size_map_min, int ekf_inited, int* n_to_add, int* n_no_downsample, int* added);
    // the same on the caller's stream `st` (fl_filter_map_incremental_device): the classification and the compaction of the bound
    // scan, then both Add_Points as one all-or-nothing device-form call of the map (Map::add_points_async, n_max = the scan's
    // size); out4 = (|PointToAdd|, |PointNoNeedDownsample|, Add_Points(PointToAdd, true), status).  No host synchronisation.
    int map_incremental_on_stream(double filter_size_map_min, int ekf_inited, int* d_out4, cudaStream_t st);
    int get_nearest(float* out_pts, int* out_cnt, int nq);
    // multi-GPU: Nearest_Points of the points outside this rank's shard (searched by their own rank during the update) are
    // recomputed here, with the state of the last searching pass, before anything reads the whole scan's neighbours
    int complete_neighbours();
    int get_selected(unsigned char* out, int nq);
    int get_pass_logs(PassLog* out, int cap, int* n);
    // multi-GPU: scan points sharded across ranks, map replicated, one all-reduce per pass
    int comm_init(int nranks, int rank, const void* nccl_unique_id_128);
    int set_shard(int q_begin, int q_end);             // default: the whole scan
    // fused all-reduce over NVLink peer memory instead of NCCL (one kernel per pass)
    int p2p_local_handle(void* out64);
    int p2p_connect(int nranks, int rank, const void* handles64);
    int p2p_barrier();                                 // device-side rendezvous of all ranks on the stream (no-op on one rank)

    // 1 (default): the whole update in one persistent fused kernel (k_update, update.cuh); 0: the two-kernels-per-pass chain
    // (k_search / k_search_c + k_residual) it grew out of, kept for A/B and for solver mode 0
    void set_fused(bool on) { fused_ = on; }
    bool fused() const { return fused_ && solver_ == 1; }
    int gpu_launches() const { return launches_; }
    const long long* host_ns() const { return host_ns_; }
    const float4* nearest_device() const { return scan_.nearest; }
    const ScanView& scan() const { return scan_; }
    cudaStream_t stream() const { return map_->stream(); }
    Map* map() const { return map_; }
    const FilterCtl* ctl_device() const { return ctl_.as<FilterCtl>(); }

private:
    int reserve(int nq);
    int update_any(const float* body_xyzi, const float4* d_body, int nq, double* x26, double* P, double R, double* solve_time_s);
    Map* map_;
    int max_points_;
    int max_iter_ = 4;
    double limit_[NDOF];
    int extrinsic_est_ = 0;
    int solver_ = 1;
    bool mirror_ = true;               // the last pass stores the result into the page-locked host block itself
    bool pdl_ = true;                  // programmatic dependent launch between the kernels of a scan
    int search_occ_ = 5;               // resident k_search blocks per SM the kernel is compiled for
    int search_mode_ = 1;              // 1 (default): one lane per query through the cell directory (k_search_c); 0: one warp per query through the BVH (k_search)
    ScanView scan_;
    DeviceBuffer srange_;
    DeviceBuffer body_, nearest_, nearest_cnt_, selected_, normvec_, plane_, partials_, red_, ctl_, ctl0_, logs_;
    DeviceBuffer mi_world_, mi_flag_add_, mi_flag_no_, mi_list_add_, mi_list_no_, mi_tmp_, mi_counts_;
    FilterCtl* h_ctl_ = nullptr;       // pinned staging
    cudaEvent_t ev0_ = nullptr, ev1_ = nullptr;
    int sms_ = 0, search_grid_max_ = 0, max_resid_grid_ = 0, resid_grid_ = 1;
    bool fused_ = true;
    DeviceBuffer pub_;                 // k_update's publication block
    unsigned launch_nonce_ = 0;
    UpdCaps upd_caps_ = {};                      // co-resident blocks of every update kernel on this device (init)
    UpdCaps scans_caps_ = {};                    // upd_caps_ with UK_BATCH's count lowered to k_update_scans' if that is smaller
    int launch_update(int max_passes, int mode, int search_only) { return launch_update(max_passes, mode, search_only, stream()); }
    int launch_update(int max_passes, int mode, int search_only, cudaStream_t st);
    UpdPlan plan(UpdRoute r, int rows, int n_hyp = 0) const;       // plan_update here, FASTLIO_B200_PAIR read at every plan
    // the only launch of an update kernel: n is the count of the _n forms, log_stride k_update_batch's, grid.y = p.slots,
    // slots k_update_scans' table (p.scans)
    cudaError_t launch_plan(const UpdPlan& p, const UpdArgs& a, cudaStream_t st, const int* n = nullptr, int log_stride = 0,
                            const ScanSlot* slots = nullptr);
    StateIn state_in_args(double R) const;       // k_state_in / k_batch_state_in's setup besides the caller's x26 / P
    // the device forms cover a single-rank filter (and the update a fused, solver-1 one); FL_ERR_STATE otherwise
    int device_form_scope(const char* what, bool update) const;
    // the UpdArgs of a launch of k_update / k_update_n
    UpdArgs upd_args(int max_passes, int mode, int search_only);
    // binds the scan without recording the binding on the device (set_scan_device: the host forms' binding, recorded)
    int bind_scan(const float4* d_body, int nq);
    // device-count binding (update_scan_on_stream): the bound scan's count lives in d_bind_[0] and scan_.Q / q_end hold the row
    // bound q_max_ until a host-form call reads the count back (read_binding); set_scan_device ends it
    bool dev_count_ = false;
    int q_max_ = 0;
    const float4* scan_body_ = nullptr;      // the scan front end's cloud of the last update_scan_on_stream
    // d_bind_ = (size, BIND_*): the binding the stream work recorded last, written by the device forms (in their graphs too) and,
    // once a device form has run (stream_bound_), by the host forms' binds; read_binding restores it for the host forms
    bool stream_bound_ = false;
    DeviceBuffer d_bind_;
    DeviceBuffer rows_;                // k_update_wave / k_update_n_wave: the tagged partial rows (one per worker block)
    int read_binding();
    int batch_nq_max_ = -1;            // the nq_max reserve_batch sized the batch buffers for (-1: not yet)
    DeviceBuffer b_body_, b_ctl_, b_pub_, b_partials_, b_nearest_, b_nearest_cnt_, b_selected_, b_plane_, b_srange_;
    DeviceBuffer b_slots_;             // update_scans_on_stream: one wave's ScanSlot table (k_scans_state_in)
    int reloc_nq_max_ = -1, reloc_hyp_max_ = 0, reloc_keep_max_ = 0;     // what reserve_reloc sized (-1: not yet)
    DeviceBuffer r_keys_, r_temp_, r_inl_, r_x_, r_P_, r_status_, r_logs_;
    int launches_ = 0;
    long long host_ns_[4] = {0, 0, 0, 0};
    bool shard_set_ = false;
    bool neighbours_complete_ = true;
    // NCCL (resolved lazily with dlopen so that single-GPU use needs no NCCL at all)
    NcclApi* nccl_ = nullptr;
    void* comm_ = nullptr;
    int nranks_ = 1, rank_ = 0;
    DeviceBuffer mailbox_, p2p_;
    void* peer_ptr_[P2P_MAX_RANKS] = {nullptr};
    bool p2p_on_ = false;
};

// fl_reloc_expand_grid_device (reloc.cu): the grid's hypotheses around d_prior, on the device that holds it
int reloc_expand_grid(const double* d_prior, const fl_reloc_grid_t* g, double* d_hyp, cudaStream_t st);

}  // namespace fl
