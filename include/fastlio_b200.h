/* fastlio_b200.h -- C ABI of the H100-native FAST-LIO2 measurement-update path.
 *
 * The reference (hku-mars/FAST_LIO) has no FFI layer: the hot path is reached through two
 * C++ class APIs used by src/laserMapping.cpp.  This header is the extern "C" boundary that
 * sits underneath drop-in facades of those two classes (include/ikd-Tree/ikd_Tree.h and
 * include/IKFoM_toolkit/esekfom/esekfom.hpp in this repository); each entry point cites
 * the reference interface it replaces (paths relative to the reference tree).
 *
 * Conventions: opaque handles; caller-owned HOST buffers unless a name says _device;
 * every function returns an int status (0 = ok, <0 = error, see FL_ERR_*) except the
 * counting queries; no exceptions cross the boundary; fl_last_error() returns a
 * thread-local message.  One CUDA stream per map handle; handles are thread-compatible
 * (serialise calls on one handle), distinct handles are independent.
 *
 * Point layout everywhere: 4 floats (x, y, z, intensity) -- the fields of
 * pcl::PointXYZINormal (include/common_lib.h:37) that the path reads.
 * State layout (26 doubles): pos(3) rot(x,y,z,w) offset_R_L_I(x,y,z,w) offset_T_L_I(3)
 * vel(3) bg(3) ba(3) grav(3)  == state_ikfom (include/use-ikfom.hpp:12-21), quaternions in
 * Eigen coeffs() order.  Covariance: 23 x 23 doubles, row-major, DOF order of state_ikfom.
 */
#ifndef FASTLIO_B200_H
#define FASTLIO_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define FL_OK 0
#define FL_ERR_CUDA (-1)
#define FL_ERR_ARG (-2)
#define FL_ERR_NCCL (-3)
#define FL_ERR_STATE (-4)
#define FL_ERR_CAPACITY (-5)

typedef struct fl_map fl_map_t;        /* replaces KD_TREE<PointType>          include/ikd-Tree/ikd_Tree.h:48-341 */
typedef struct fl_filter fl_filter_t;  /* replaces esekfom::esekf<state_ikfom,12,input_ikfom> + h_share_model */

/* Same layout as the oracle's per-pass log; used by the parity tests. */
typedef struct fl_pass_log {
    int searched, valid, effct, converged;
    double res_sum;
    double HtH[144];
    double Hth[12];
    double x_after[26];
} fl_pass_log_t;

const char* fl_last_error(void);
/* Page-lock a caller-owned, long-lived host buffer (e.g. the scan buffer reused every scan) so that
 * fl_filter_update / fl_map_add_points copy from it by DMA; unregister before freeing it. */
int fl_host_register(const void* ptr, unsigned long long bytes);
int fl_host_unregister(const void* ptr);
int fl_device_count(void);
int fl_version(void);

/* ------------------------------------------------------------------ map: KD_TREE<PointType> */
/* KD_TREE::KD_TREE(delete_param, balance_param, box_length)          ikd_Tree.h:309, ikd_Tree.cpp:9-18
 * (the two rebuild criteria have no counterpart: leaves are re-packed by fl_map_rebuild / automatically) */
int fl_map_create(fl_map_t** out, int device, float downsample_size);
int fl_map_destroy(fl_map_t* m);   /* drops the caller's reference; filters / scans created on the map keep it alive until they go */
/* KD_TREE::set_downsample_param                                      ikd_Tree.h:319-322 */
int fl_map_set_downsample(fl_map_t* m, float downsample_size);
/* KD_TREE::Build(PointVector)                                        ikd_Tree.cpp:409-423 */
int fl_map_build(fl_map_t* m, const float* pts_xyzi, int n);
/* KD_TREE::size() / validnum()                                       ikd_Tree.cpp:70-97, 140-163 */
int fl_map_size(fl_map_t* m);
int fl_map_validnum(fl_map_t* m);
/* KD_TREE::Nearest_Search, batched over nq queries, k <= 5           ikd_Tree.cpp:426-461
 * out_pts: nq*k*4 floats (ascending distance), out_d2: nq*k floats, out_cnt: nq ints.  Safe for
 * concurrent host callers on one handle (internally serialised). */
int fl_map_knn(fl_map_t* m, const float* q_xyzi, int nq, int k, float* out_pts, float* out_d2, int* out_cnt);
/* KD_TREE::Nearest_Search(point, k_nearest, Nearest_Points, Point_Distance, max_dist), batched
 *                                                                    ikd_Tree.cpp:426-461, Search :1062-1244
 * The layout of fl_map_knn: out_pts nq*k*4 floats, out_d2 nq*k floats, out_cnt nq ints; entries j >= out_cnt[i] are
 * (0, 0, 0, 0) with d2 = +inf.  1 <= k <= 32, else FL_ERR_ARG (so is a null buffer with nq > 0).
 * With md2 = max_dist * max_dist rounded to float32 (:1067), a point is a candidate when its float32 squared distance (x, y, z
 * summed in that order, bit-identical to the reference's) is <= md2; the answer is the min(k, #candidates) nearest
 * candidates.  So max_dist = +inf applies no gate, a negative max_dist acts as |max_dist|, 0 finds only coincident points
 * and NaN finds nothing, as in the reference.  A query with a non-finite coordinate finds nothing.
 * Order: ascending d2; adjacent entries whose d2 differ by less than 1e-10 are ordered by ascending x (PointType_CMP,
 * ikd_Tree.h:102-108).  Where the k-th and the (k+1)-th candidates tie, the reference keeps whichever its traversal found
 * first; this map keeps one deterministically (the same bytes on every call for the same map and queries).
 * k <= 5 runs the search of fl_map_knn and cuts its answer at md2; 6 <= k <= 32 runs one warp per query.  Serialised on the
 * handle like the other map calls. */
int fl_map_nearest_search(fl_map_t* m, const float* q_xyzi, int nq, int k, float max_dist,
                          float* out_pts, float* out_d2, int* out_cnt);
/* KD_TREE::Add_Points(PointVector&, bool downsample_on) -> int       ikd_Tree.cpp:478-573
 * returns the reference's return value (>= 0) or an error (< 0) */
int fl_map_add_points(fl_map_t* m, const float* pts_xyzi, int n, int downsample_on);
/* KD_TREE::Delete_Point_Boxes(vector<BoxPointType>&) -> int          ikd_Tree.cpp:632-658
 * boxes6: nb * (min xyz, max xyz); returns the number of points invalidated or an error (< 0) */
int fl_map_delete_boxes(fl_map_t* m, const float* boxes6, int nb);
/* KD_TREE::Add_Point_Boxes(vector<BoxPointType>&)                     ikd_Tree.cpp:576-603 (Add_by_range :854-934)
 * points that Delete_Point_Boxes removed, lie in the boxes and have not been overwritten by later inserts come back
 * (points removed by the down-sampling of Add_Points do not, as in the reference); returns how many, or an error (< 0) */
int fl_map_add_boxes(fl_map_t* m, const float* boxes6, int nb);
/* KD_TREE::acquire_removed_points(PointVector&)                       ikd_Tree.cpp:661-676 (called at laserMapping.cpp:225)
 * the points removed by Delete_Point_Boxes since the previous call (the reference hands them over when it rebuilds the
 * subtree, this map at once); the first call starts the record and returns 0.  Returns the number of points (writes at
 * most cap of them), or an error (< 0).  Call with cap >= the return value of the deletes since the last call. */
int fl_map_acquire_removed(fl_map_t* m, float* out_xyzi, int cap);
/* KD_TREE::flatten(Root_Node, Storage, NOT_RECORD): all valid points  ikd_Tree.cpp:1627-1658
 * returns the number of valid points (writes at most cap of them) or an error (< 0) */
int fl_map_flatten(fl_map_t* m, float* out_xyzi, int cap);
/* KD_TREE::Box_Search(const BoxPointType&, PointVector&), batched     ikd_Tree.cpp:464-468 (Search_by_range :1247-1289)
 * boxes6: nb x (min xyz, max xyz); a point is found when min <= p < max on every axis.
 * KD_TREE::Radius_Search(PointType, float, PointVector&), batched     ikd_Tree.cpp:470-475 (Search_by_radius :1292-1332)
 * centers_xyzr: nq x (x, y, z, radius); a point is found when its float32 squared distance (x, y, z summed in that order)
 * is <= radius * radius rounded to float32 -- the test of :1308.  The reference decides leaves and whole subtrees by
 * sqrtf(d2) <= radius instead, so the two answers may differ on points with d2 > fl(r * r) and sqrtf(d2) <= r.
 * Both: CSR output.  out_offsets[nq + 1] is always written; the points of query i are out_xyzi[4 * out_offsets[i] ..
 * 4 * out_offsets[i + 1]), in an order that is deterministic but unrelated to the reference's.  At most cap points are
 * written (out_xyzi may be NULL when cap is 0).  Returns the total number of points found (call again with cap >= it)
 * or an error (< 0): FL_ERR_ARG for a null buffer, FL_ERR_CAPACITY for a total above INT_MAX.  NaN input, a negative
 * radius and an empty or inverted box find nothing. */
int fl_map_box_search(fl_map_t* m, const float* boxes6, int nb, int* out_offsets, float* out_xyzi, int cap);
int fl_map_radius_search(fl_map_t* m, const float* centers_xyzr, int nq, int* out_offsets, float* out_xyzi, int cap);

/* ---- device-buffer forms of the queries and of Build / Add_Points
 * Every *_device pointer is device memory on the map's device (or managed memory allocated against it); point and query
 * buffers of 4 floats are 16-byte aligned.  `stream` is a cudaStream_t passed as void* (NULL: the legacy default stream).
 * The queries return an enqueue status (FL_OK, FL_ERR_ARG, FL_ERR_CUDA); their answers stay on the device and are complete
 * when `stream` reaches them.  They never synchronise the host, allocate, or size a launch from a value produced on the
 * device, so they may be captured into a CUDA graph.  A host pointer, a pointer to another device, a null buffer with
 * nq > 0 or a misaligned one returns FL_ERR_ARG before anything is enqueued.
 * Ordering: outside stream capture a query first waits for everything already enqueued on the handle's stream (a
 * fl_filter_run still in flight, a scan step, a mutation), and the handle's stream then waits for the query, so a later
 * Add_Points, Delete_Point_Boxes, rebuild or filter launch does not overwrite the map under it.  Two queries on two caller
 * streams with no other call on the handle between them do not wait for each other.  While `stream` is capturing, the
 * call joins nothing: the caller orders replays against mutations ("mutators must not overlap searches"), and a captured
 * graph holds the map's layout of capture time, so capture again after any call that changes the map. */
/* KD_TREE::Nearest_Search(point, k_nearest, Nearest_Points, Point_Distance, max_dist), batched, on device buffers
 *                                                                    ikd_Tree.cpp:426-461, Search :1062-1244
 * Writes exactly the bytes fl_map_nearest_search returns for the same map and queries: points, d2, counts, the (0, 0, 0, 0) /
 * +inf padding; a non-finite query and a NaN max_dist find nothing.  fl_map_dir_stats counts its walked queries the same way.
 * k <= 5 runs fl_map_knn's search with the non-finite queries moved to the origin and the cut at md2 on the device;
 * 6 <= k <= 32 the one-warp-per-query search.  k outside [1, 32] is FL_ERR_ARG; nq = 0 writes nothing. */
int fl_map_nearest_search_device(fl_map_t* m, const float* q_xyzi_device, int nq, int k, float max_dist,
                                 float* out_pts_device, float* out_d2_device, int* out_cnt_device, void* stream);
/* Bytes of caller-provided workspace for a range query of nq queries and up to max_pairs (query, main leaf) pairs.  The only
 * sizing rule: a workspace of W bytes holds the largest max_pairs whose size is <= W. */
int fl_map_range_workspace_bytes(fl_map_t* m, int nq, long long max_pairs, unsigned long long* out_bytes);
/* KD_TREE::Box_Search / Radius_Search, batched, on device buffers     ikd_Tree.cpp:464-475 (Search_by_range :1247-1289,
 * Search_by_radius :1292-1332).  The rules, the offsets and the points (in the same order) of fl_map_box_search /
 * fl_map_radius_search.  status2_device[1] always receives the number of (query, leaf) pairs needed; status2_device[0]:
 *   -1            the pairs did not fit the workspace: the offsets are all zero and no point is written;
 *   > INT_MAX     the total (the counterpart of FL_ERR_CAPACITY): the offsets are all zero and no point is written;
 *   otherwise     the total: out_offsets[nb + 1] is written in full and at most cap points (out_xyzi may be NULL when cap = 0).
 * Read the status when convenient and retry with a larger workspace or cap.  Nothing outside the given buffers is written.
 * nb = 0 writes out_offsets[0] = 0 and status (0, 0).  The workspace is the caller's (the handle's scratch is not used), and
 * a workspace may not be shared by two queries in flight. */
int fl_map_box_search_device(fl_map_t* m, const float* boxes6_device, int nb, int* out_offsets_device, float* out_xyzi_device,
                             long long cap, void* workspace_device, unsigned long long workspace_bytes, long long* status2_device,
                             void* stream);
int fl_map_radius_search_device(fl_map_t* m, const float* centers_xyzr_device, int nq, int* out_offsets_device, float* out_xyzi_device,
                                long long cap, void* workspace_device, unsigned long long workspace_bytes, long long* status2_device,
                                void* stream);
/* KD_TREE::Build / Add_Points from device memory                      ikd_Tree.cpp:409-423 / :478-573
 * Synchronous, with the return values of fl_map_build / fl_map_add_points; the input is read after the work already
 * enqueued on `stream`, and may be reused when the call returns.  Cannot be called on a capturing stream (FL_ERR_ARG). */
int fl_map_build_device(fl_map_t* m, const float* pts_xyzi_device, int n, void* stream);
int fl_map_add_points_device(fl_map_t* m, const float* pts_xyzi_device, int n, int downsample_on, void* stream);
/* KD_TREE::Add_Points on the caller's stream                          ikd_Tree.cpp:478-573
 * n is read from *n_device when `stream` reaches the call; the caller promises 0 <= *n_device <= n_max (a larger value is
 * clamped to n_max).  status2_device[0]: FL_OK; 1 = maintenance due (the insert was applied, and the host form would have
 * re-packed the leaves or re-listed the directory at this point: call fl_map_maintain); FL_ERR_CAPACITY = the call did not fit
 * the map's headroom and NOTHING was changed.  status2_device[1]: the reference's return value, 0 on a refusal.
 * Like the device-buffer queries above: never synchronises, allocates, re-packs, re-lists or sizes a launch from a device value
 * (grids follow n_max), so it may be captured into a CUDA graph and replayed with other counts.  A plan kernel checks, before
 * anything is written, that the batch fits the room left (overflow leaves, cell table below 90 % load, halo-list pool); every
 * other kernel of the call then runs over the count the plan let through.  The one exception to "never synchronises": outside
 * capture, when the host's bound of the headroom (overflow leaves and table cells for the points of every device-form call since
 * the map was last settled, plus n_max; the list pool is checked on the device only) says the call might not fit, the call first
 * settles the map (a wait for the stream) and grows it if it has no room either, synchronously, as the host form would.  On
 * a capturing stream that case is FL_ERR_CAPACITY with nothing captured (so is a first call with this n_max: make the call once
 * outside capture before capturing it).
 * Ordering: outside capture `stream` first waits for everything enqueued on the handle (device queries joined from other
 * streams included), and the handle's stream then waits for the call, so later calls on the map see the insert.  Inside capture
 * nothing is joined (the rules of the queries above).  Host, wrong-device, null or misaligned pointers are FL_ERR_ARG and
 * nothing is enqueued.  The host-form calls settle first: read-only ones (size, validnum, flatten, tree_range, the queries,
 * fl_map_stats, fl_map_dir_stats) read the device's counters back once and change no layout, so a captured graph stays valid
 * across them (synchronise graph replays before them); mutations and the filter's host forms also run the deferred re-pack /
 * re-list. */
int fl_map_add_points_async(fl_map_t* m, const float* pts_xyzi_device, const int* n_device, int n_max, int downsample_on,
                            int* status2_device, void* stream);
/* KD_TREE::Delete_Point_Boxes on the caller's stream                   ikd_Tree.cpp:632-658
 * boxes6_device: nb_max x (min xyz, max xyz); nb read from *nb_device (clamped to [0, nb_max]) when `stream` reaches the call.
 * status2_device = (status, deleted): FL_OK, 1 = maintenance due (the points were deleted, and the host form would have re-packed
 * the leaves here: call fl_map_maintain), FL_ERR_CAPACITY = nothing changed; deleted = the return value of fl_map_delete_boxes (0
 * on a refusal).  The contract of fl_map_add_points_async: the same joins, capture rules, argument refusals (boxes 4-byte
 * aligned, may be NULL when nb_max = 0), no host synchronisation, allocation or launch sized from a device value.  The pass over
 * the slots reads the map's used leaves on the device (inserts replayed since the last settle included), and the AABBs are refit
 * only when a point was deleted: the launches are the same either way.  After a settle the map is exactly what
 * fl_map_delete_boxes leaves.  Once fl_map_acquire_removed has started the removed-points record, a one-thread plan checks
 * before any slot is touched that the record has room for every valid point on top of what it holds (the host form grows it to
 * that before each delete); without room the call is refused, and fl_map_maintain (which sizes a started record for the next
 * delete, and reports the layout changed when the record is allocated or moves) makes room.  The host's bound of the room is the
 * record's count and the valid points at the last settle plus the points of device-form inserts since.  Outside capture, when
 * that bound says the record might be short, the call first settles the map and grows the record (the one synchronous case);
 * on a capturing stream it is FL_ERR_CAPACITY with nothing captured (call fl_map_maintain first).  Starting the record
 * (fl_map_acquire_removed) reports a layout change at the next fl_map_maintain: deletes captured before it do not record. */
int fl_map_delete_boxes_async(fl_map_t* m, const float* boxes6_device, const int* nb_device, int nb_max, int* status2_device,
                              void* stream);
/* Settles the host's view of the map and runs the re-pack / directory re-list that device-form mutations deferred (by the host
 * form's rules), and grows the map for a device-form call it refused (FL_ERR_CAPACITY).  *layout_changed (may be NULL) = 1 when
 * buffers or leaves moved since the last report: graphs captured before must be captured again.  Synchronous.  A status of 1 or a
 * refusal stays owed to this call when read-only host calls (validnum, size, ...) run in between; calls refused for lack of room
 * keep being refused until it runs. */
int fl_map_maintain(fl_map_t* m, int* layout_changed);
/* KD_TREE::tree_range()                                              ikd_Tree.cpp:100-137 */
int fl_map_tree_range(fl_map_t* m, float* box6);
/* KD_TREE::Rebuild of the whole tree (ikd_Tree.cpp:736-764): re-sorts all valid points into fresh leaves */
int fl_map_rebuild(fl_map_t* m);
/* introspection: [0] main leaves [1] overflow leaves [2] internal levels [3] rebuilds so far */
int fl_map_stats(fl_map_t* m, int* out4);
/* The k-NN fast path: a hashed directory of cubic cells over the same points (no reference counterpart; the results are
 * those of KD_TREE::Nearest_Search either way).  on = 0 answers every query through the BVH walk; cell_size <= 0 picks
 * 2 x downsample_size.  Takes effect immediately (the directory is re-listed). */
int fl_map_set_cell_directory(fl_map_t* m, int on, float cell_size);
/* Deterministic mode (off by default; no reference counterpart).  With it on, every answer that reaches the caller or the
 * filter's state is a function of the SET of valid points -- compared as (x, y, z, intensity) bits -- not of the slots they
 * occupy, which racing inserts, deletes and re-lists make differ from run to run.  For maps holding the same valid points,
 * whatever the history of Build / Add_Points / Delete_Point_Boxes / Add_Point_Boxes / maintenance that produced them:
 *   - k-NN (fl_map_knn, fl_map_nearest_search and its _device form, every k and max_dist, and the neighbours every update
 *     kernel finds): the returned set is the k smallest under the total order (d2, x, y, z, intensity), d2 the float32 the
 *     kernels compute and the other keys breaking its bit-equal ties, each compared as an order-preserving integer of its bits
 *     (-0 below +0).  The order is the usual one: ascending d2, candidates within 1e-10 by x (PointType_CMP), and entries equal
 *     on both by (y, z, intensity).  The output bytes are equal across such maps.
 *   - Add_Points with down-sampling: of the valid points of a voxel at equal distance from its centre, the one with the
 *     smallest (x, y, z, intensity) counts as the nearest; batch points keep their input order.  The same prior point set and
 *     batch give the same resulting point set and return value.
 *   - Updates (fl_filter_update, its _device, _scan_device and _batch_device forms, map_incremental in both forms) read the
 *     map only through these two rules, so x, P, pass logs, Nearest_Points and selected are equal bit for bit across such
 *     maps and from run to run.  The update runs the fused kernels only: a filter on solver mode 0 or the two-kernels-per-pass
 *     chain (fl_filter_set_fused 0) fails with FL_ERR_STATE.
 *   - fl_map_flatten returns its rows sorted by (x, y, z, intensity) bits, so a map written to disk is byte-stable.
 * Not covered: the row order of Box_Search / Radius_Search (their sets are already equal), the order of
 * fl_map_acquire_removed, slot layout, fl_map_size (it counts lazily deleted slots) and sharded filters beyond what the
 * same rules give them.  The mode differs from the reference only where the reference itself is arbitrary: bit-equal d2 and x
 * at the k-th place, and equal distances to a voxel centre.
 * The setter waits for the handle's stream, then switches; it takes no stream, so it cannot be called from inside a capture.
 * Filters and scans created on the map follow its mode at every launch; a captured graph keeps the kernels of capture time,
 * so capture again after switching (as after fl_filter_set_params).  A null handle (or output) is FL_ERR_ARG. */
int fl_map_set_deterministic(fl_map_t* m, int on);
int fl_map_get_deterministic(fl_map_t* m, int* on);
/* [0] cells [1] external buckets [2] crowded cells (queries touching them use the BVH walk) [3] table capacity
 * [4] directory re-lists triggered by inserts [5] queries answered by the BVH walk since the last call (-1: directory off) */
int fl_map_dir_stats(fl_map_t* m, int* out6);

/* ------------------------------------------------------------------ filter: esekf + h_share_model */
/* esekf::esekf + esekf::init_dyn_share(f, f_x, f_w, h_share_model, maximum_iteration, limit)
 *                                                                   esekfom.hpp:238-254, laserMapping.cpp:826-828 */
int fl_filter_create(fl_filter_t** out, fl_map_t* map, int max_points);
int fl_filter_destroy(fl_filter_t* f);
/* maximum_iter, limit[23], extrinsic_est_en (laserMapping.cpp:739,789) */
int fl_filter_set_params(fl_filter_t* f, int max_iter, const double* limit23, int extrinsic_est_en);
/* 1 (default): the gain of esekfom.hpp:1782-1809 through one 6x6 (12x12 with extrinsic estimation) solve,
 *    algebraically identical (DESIGN.md section 4);
 * 0: the information form with two 23x23 inversions exactly as written in the reference (validation) */
int fl_filter_set_solver(fl_filter_t* f, int mode);
/* kNN of the search passes: 1 (default) one lane per scan point through the map's cell directory, the BVH walk for
 * whatever that cannot prove; 0 one warp per scan point through the BVH walk only -- same neighbours, same distances */
int fl_filter_set_search(fl_filter_t* f, int mode);
/* 1 (default): the whole update in ONE persistent kernel launch (h_share_model fused with the search, the Kalman step
 * in the kernel's solver block); 0: the two-kernels-per-pass chain it grew out of (A/B; solver mode 0 always uses it) */
int fl_filter_set_fused(fl_filter_t* f, int on);
/* esekf::update_iterated_dyn_share_modified(R, solve_time) with feats_down_body bound
 *                                                                   esekfom.hpp:1619-1931, laserMapping.cpp:638-754, :960
 * x26 / P: in = kf.get_x()/get_P() before the update, out = after.  solve_time_s (may be NULL)
 * is incremented by the device time of the update, like the reference's out-parameter. */
int fl_filter_update(fl_filter_t* f, const float* body_xyzi, int nq, double* x26, double* P, double R, double* solve_time_s);
/* map_incremental() (laserMapping.cpp:427-474) without leaving the device: classifies the bound scan with the
 * updated state and the cached neighbours, then performs the two Add_Points calls (:470-471).
 * out3 (may be NULL): [0] |PointToAdd| [1] |PointNoNeedDownsample| [2] return value of Add_Points(PointToAdd, true) */
int fl_filter_map_incremental(fl_filter_t* f, double filter_size_map_min, int flg_EKF_inited, int* out3);
/* Nearest_Points after the update (laserMapping.cpp:102, read by map_incremental :438-460) */
int fl_filter_get_nearest(fl_filter_t* f, float* out_pts, int* out_cnt, int nq);
/* point_selected_surf after the update (laserMapping.cpp:76) */
int fl_filter_get_selected(fl_filter_t* f, unsigned char* out, int nq);
/* per-pass H^T H, H^T h, effct_feat_num, total_residual, state -- for parity tests / the reference's debug log */
int fl_filter_get_pass_logs(fl_filter_t* f, fl_pass_log_t* out, int cap);
/* pieces of fl_filter_update for pipelines that keep the scan resident in HBM */
int fl_filter_upload_scan(fl_filter_t* f, const float* body_xyzi, int nq);
int fl_filter_upload_state(fl_filter_t* f, const double* x26, const double* P, double R);
int fl_filter_run(fl_filter_t* f);                 /* enqueue all passes, asynchronous */
int fl_filter_download_state(fl_filter_t* f, double* x26, double* P, int* n_pass);   /* synchronises */
int fl_filter_sync(fl_filter_t* f);
/* device time in milliseconds of `reps` back-to-back resident updates from the uploaded state
 * (CUDA events on the handle's stream); optionally flushes L2 between repetitions */
int fl_filter_time_resident(fl_filter_t* f, int reps, int flush_l2, float* ms_total);
/* wall-clock seconds of `reps` consecutive fl_filter_update(body, nq, copy of x26, copy of P, R) calls issued from
 * native code (the per-scan cost a C++ caller such as laserMapping.cpp sees); x26_out / P_out (may be NULL): last result */
int fl_filter_time_e2e(fl_filter_t* f, const float* body_xyzi, int nq, const double* x26, const double* P, double R, int reps,
                       double* seconds, double* x26_out, double* P_out);
/* device time of `reps` launches of the dominant kernel alone (k_search: the kNN of the first pass of an update) */
int fl_filter_time_search_pass(fl_filter_t* f, int reps, int flush_l2, float* ms_total);
int fl_filter_gpu_launches(fl_filter_t* f);
/* clock64() stamps of the last on-device Kalman step (tuning aid; layout in scripts/profile_once.py) */
int fl_filter_debug_prof(fl_filter_t* f, long long* out16);

/* ---- device-buffer form of the update (the conventions of the map's *_device block above)
 * esekf::update_iterated_dyn_share_modified on device buffers      esekfom.hpp:1619-1931, laserMapping.cpp:638-754
 * x26_device (26 doubles) and P_device (23 x 23, row-major) are read when the update starts and overwritten when it ends, like
 * the reference's x_ / P_, but only when it succeeds.  status2_device[0] receives FL_OK, or FL_ERR_STATE for a singular system
 * or a block that gave up waiting; status2_device[1] the number of passes run.  On success x and P hold exactly the bytes
 * fl_filter_update returns for the same map, scan, prior, R and parameters; fl_filter_get_pass_logs, get_nearest,
 * get_selected, download_state and map_incremental afterwards see this update as they would see fl_filter_update's.
 * The scan is copied into the filter's own buffer on `stream`: the caller may reuse or free body_xyzi_device once `stream`
 * has passed the call.  The call never synchronises the host, never allocates and never sizes a launch from a device value;
 * nq above the filter's capacity (max_points at create, or the largest scan it has bound since) is FL_ERR_CAPACITY and
 * enqueues nothing.  solve_time is not reported: time the call with events on `stream`.
 * Ordering: outside stream capture, `stream` first waits for everything enqueued on the handle's stream (including an
 * earlier device-form update of this filter on another stream), and the handle's stream then waits for the update, so a
 * later host-form call on the filter or the map (map_incremental, get_pass_logs, Add_Points, Delete_Point_Boxes) sees its
 * result and cannot change the map under it.  While `stream` is capturing nothing is joined: order replays against other
 * calls on the filter and the map yourself (synchronise a replay before a host-form call on the filter).  A captured graph
 * keeps the map's layout, the filter's buffers, nq and the parameters (max_iter, limit, extrinsic_est_en, R) of capture time;
 * capture again after any of them changes.
 * A host pointer, a pointer to another device, a null pointer (the scan may be null when nq = 0) or a misaligned one (scan
 * 16 bytes, x and P 8, status 4) is FL_ERR_ARG; a sharded filter (set_shard, comm_init with nranks > 1, p2p_connect), solver
 * mode 0 or fused 0 is FL_ERR_STATE: the device form runs k_update only.  Nothing is enqueued on a refusal. */
int fl_filter_update_device(fl_filter_t* f, const float* body_xyzi_device, int nq, double* x26_device, double* P_device, double R,
                            int* status2_device, void* stream);
/* Nearest_Points / point_selected_surf of the last update (the bytes of fl_filter_get_nearest / get_selected), copied into
 * device buffers on `stream` with the update's ordering rules; 0 <= nq <= the bound scan's size.  Not for sharded filters. */
int fl_filter_get_nearest_device(fl_filter_t* f, float* out_pts_device, int* out_cnt_device, int nq, void* stream);
int fl_filter_get_selected_device(fl_filter_t* f, unsigned char* out_device, int nq, void* stream);
/* map_incremental() (laserMapping.cpp:427-474) on the caller's stream, after the last update of this filter (host or device
 * form): out4_device = (|PointToAdd|, |PointNoNeedDownsample|, Add_Points(PointToAdd, true), status), the first three the values
 * of fl_filter_map_incremental's out3, the status that of fl_map_add_points_async for both inserts, which are all-or-nothing
 * together (FL_ERR_CAPACITY: neither list was inserted).  n_max is the bound scan's size.  The conventions, ordering and capture
 * rules of fl_map_add_points_async; per scan, fl_filter_update_device then this call may be captured into one graph.  A sharded
 * filter is FL_ERR_STATE and a null, host or misaligned out4 FL_ERR_ARG, with nothing enqueued. */
int fl_filter_map_incremental_device(fl_filter_t* f, double filter_size_map_min, int flg_EKF_inited, int* out4_device, void* stream);

/* ---- batched form of the update: one scan from many priors (relocalisation, multi-hypothesis evaluation)
 * esekf::update_iterated_dyn_share_modified run from n_hyp priors     esekfom.hpp:1619-1931, laserMapping.cpp:638-754
 * Hypothesis h receives exactly the x, P, status pair and pass logs [0, passes) that fl_filter_update_device gives for the prior
 * (x26_device[h], P_device[h]) on the same map, scan, R and parameters; log entries from `passes` on are not written, and, as in
 * fl_filter_get_pass_logs, an entry of a pass without effective points leaves HtH and Hth as they were.  x26_device is
 * [n_hyp][26], P_device [n_hyp][23 * 23], status2_device [n_hyp][2], logs_device (may be NULL) [n_hyp][max_iter + 1].
 * The hypotheses run in waves: one launch holds `hypotheses per wave` of them, each with the workers of the single form, and a
 * wave lasts as long as its slowest hypothesis.  fl_filter_batch_plan writes out3 = (workers per hypothesis, hypotheses per
 * wave, waves) for nq points and n_hyp hypotheses (FL_ERR_CAPACITY if one hypothesis does not fit the co-resident grid).
 * The batch uses buffers of its own: afterwards fl_filter_get_nearest / get_selected / get_pass_logs / download_state,
 * map_incremental (both forms) and the *_device getters return what they returned before it.  fl_map_dir_stats does count its
 * BVH walks.  There is no per-hypothesis Nearest_Points / point_selected_surf.
 * fl_filter_reserve_batch sizes those buffers for every nq <= nq_max (a few MB); nq_max above the filter's capacity is
 * FL_ERR_CAPACITY.  Synchronous and grow-only, like fl_scan_reserve; a grow moves the buffers, so capture graphs of the batch
 * again after it.
 * The conventions, ordering and capture rules of fl_filter_update_device: the scan is copied on `stream`, so the caller may free
 * it once `stream` has passed the call; no host synchronisation, allocation or launch sized from a device value.  n_hyp = 0
 * returns FL_OK and enqueues nothing.  FL_ERR_ARG: nq or n_hyp < 0; a host, wrong-device, null or misaligned pointer (scan 16
 * bytes, x and P 8, status 4, logs 8; the scan may be null when nq = 0, the outputs when n_hyp = 0).  FL_ERR_STATE: no
 * fl_filter_reserve_batch yet, or a sharded, solver-0 or fused-0 filter.  FL_ERR_CAPACITY: nq above the reserved nq_max.
 * Nothing is enqueued on a refusal.  A filter runs one batch at a time: order batch calls on one filter on one stream (or
 * join their streams). */
int fl_filter_reserve_batch(fl_filter_t* f, int nq_max);
int fl_filter_batch_plan(fl_filter_t* f, int nq, int n_hyp, int* out3);
int fl_filter_update_batch_device(fl_filter_t* f, const float* body_xyzi_device, int nq, int n_hyp, double* x26_device,
                                  double* P_device, double R, int* status2_device, fl_pass_log_t* logs_device, void* stream);

/* ---- relocalisation: recover the pose of one scan on the map from many hypotheses
 * Three stages on the caller's stream, none of which synchronises the host or sizes a launch from a device value, so a whole
 * relocalisation can be captured into a CUDA graph and replayed.
 *
 * fl_reloc_expand_grid_device: hypotheses from a grid around a prior.  x26_prior_device is one state (26 doubles), x26_hyp_device
 * receives H = n[0] n[1] n[2] n[3] states [H][26], hypothesis h = ((i_yaw n[2] + i_z) n[1] + i_y) n[0] + i_x.  The offset on axis
 * a is (i_a - (n[a] - 1) / 2.0) step[a]: axes 0-2 add it to pos in the world frame (m), axis 3 turns rot by that yaw (rad) about
 * u = -grav / |grav| of the prior, rot = q_yaw * rot_prior (the world z axis is not the gravity axis in general).  Every other
 * component is the prior's.  The kernel runs on the device that holds x26_prior_device.  Each count must be >= 1 and each step
 * finite and >= 0, else FL_ERR_ARG (so are a null grid, host, null or misaligned (8-byte) pointers, and x26_hyp_device on another
 * device); H above INT_MAX is FL_ERR_CAPACITY.  Nothing is enqueued on a refusal.  Callers with hypotheses of their own (GNSS,
 * place recognition) skip this stage. */
typedef struct fl_reloc_grid {
    int n[4];            /* x, y, z, yaw */
    double step[4];      /* m, m, m, rad */
} fl_reloc_grid_t;
int fl_reloc_expand_grid_device(const double* x26_prior_device, const fl_reloc_grid_t* grid, double* x26_hyp_device, void* stream);

/* fl_filter_relocalize_device: screen, refine and choose.
 *   1. Screen (k_reloc_screen): every scan point i with i % stride == 0 is taken to the world by hypothesis h with the update's
 *      FP64 transform and rounded to float32, exactly as the update's search queries; it is an inlier when the map holds a point
 *      within r_inlier of it (d2 <= r_inlier * r_inlier in float32: the answer of fl_map_nearest_search with k = 1 and
 *      max_dist = r_inlier).  inliers[h] counts them; the counts are integers, the same in both modes of the map.
 *   2. The hypotheses are ranked by the 64-bit key ((screened - inliers[h]) << 32) | h, ascending: most inliers first, ties to
 *      the lowest h.  The first min(keep, n_hyp) survive.
 *   3. Refine: fl_filter_update_batch_device runs the scan from each survivor's state, in rank order, all with the one P_device
 *      and R; a survivor qualifies when its status is FL_OK and the last pass's effct is >= min_effct.  The winner is the
 *      qualifying survivor with the largest last-pass effct, then the smallest res_sum / effct, then the earliest rank.
 * x26_out_device and P_out_device receive the winner's updated x and P, the bytes fl_filter_update_device gives from the winner's
 * state with P_device; when none qualifies they are left as they were.  status4_device = (FL_OK, or FL_ERR_STATE when none
 * qualifies; the winning h or -1; its last-pass effct or 0; its inliers or 0).  inliers_device [n_hyp] and rows_device
 * [min(keep, n_hyp)] may be NULL; row s is survivor s: its h, inliers, batch status and passes, and the effct and res_sum of its
 * last pass (0 when it ran none).
 * fl_filter_reserve_reloc sizes the buffers of the call for scans of up to nq_max points, n_hyp_max hypotheses and keep_max
 * survivors (it calls fl_filter_reserve_batch(nq_max)); synchronous and grow-only, a grow moves the buffers (capture again).
 * Refusals enqueue nothing, also on a capturing stream.  FL_ERR_ARG: nq or n_hyp < 1, keep < 1, stride < 1, r_inlier not > 0,
 * a null params, or a host, wrong-device, null or misaligned pointer (scan 16 bytes; hypotheses, P, x_out, P_out and rows 8;
 * inliers and status 4; inliers and rows may be NULL).  FL_ERR_STATE: no fl_filter_reserve_reloc yet, or a sharded, solver-0 or fused-0 filter.  FL_ERR_CAPACITY:
 * nq, n_hyp or keep above what was reserved.  The conventions, ordering and capture rules of fl_filter_update_batch_device; like
 * the batch, the call leaves the filter's own results (getters, map_incremental) as they were: to go on mapping from the winner,
 * run fl_filter_update_device from x26_out_device, then map_incremental. */
typedef struct fl_reloc_params {
    int keep;            /* survivors of the screen that run the update */
    int stride;          /* screen every stride-th scan point */
    float r_inlier;      /* m */
    int min_effct;       /* effective points a survivor's last pass needs to qualify */
} fl_reloc_params_t;
typedef struct fl_reloc_row {
    int hyp, inliers, status, passes, effct, pad;
    double res_sum;
} fl_reloc_row_t;
int fl_filter_reserve_reloc(fl_filter_t* f, int nq_max, int n_hyp_max, int keep_max);
int fl_filter_relocalize_device(fl_filter_t* f, const float* body_xyzi_device, int nq, int n_hyp, const double* x26_hyp_device,
                                const double* P_device, double R, const fl_reloc_params_t* params, double* x26_out_device,
                                double* P_out_device, int* inliers_device, fl_reloc_row_t* rows_device, int* status4_device,
                                void* stream);

/* ------------------------------------------------------------------ scan front end (SURVEY.md §8f rows 3-4)
 * The two steps that produce feats_down_body, kept in HBM on the map's device and stream so that a scan goes
 * raw -> de-skewed -> down-sampled -> update -> map_incremental with one upload. */
typedef struct fl_scan fl_scan_t;      /* replaces the feats_undistort / feats_down_body clouds   laserMapping.cpp:122-124 */
int fl_scan_create(fl_scan_t** out, fl_map_t* map);
int fl_scan_destroy(fl_scan_t* s);
/* Measures.lidar (common_lib.h:47-58): n x (x,y,z,intensity) + PointType::curvature = offset time in ms */
int fl_scan_upload(fl_scan_t* s, const float* xyzi, const float* offset_ms, int n);
/* ImuProcess::UndistortPcl, the sort (:234) and the backward pass (:312-346)         IMU_Processing.hpp:216-346
 * imu_pose22: IMUpose, n_pose x Pose6D (msg/Pose6D.msg: offset_time, acc[3], gyr[3], vel[3], pos[3], rot[9] row-major),
 * filled by the caller's forward propagation (:244-301, esekf::predict stays on the host);
 * x26_end: kf_state.get_x() after the last predict (:303).  Points stay in HBM, time-sorted (stable). */
int fl_scan_undistort(fl_scan_t* s, const double* imu_pose22, int n_pose, const double* x26_end);
/* downSizeFilterSurf.setInputCloud(feats_undistort); .filter(*feats_down_body)         laserMapping.cpp:904-905
 * = pcl::VoxelGrid<PointType> with leaf (l,l,l) (laserMapping.cpp:811): centroid of every occupied cell, output in
 * ascending cell index.  Returns feats_down_size (>= 0) or an error (< 0). */
int fl_scan_voxel_downsample(fl_scan_t* s, float leaf_size);
/* which 0: the raw / de-skewed cloud, 1: the down-sampled cloud; returns the cloud's size (writes at most cap points) */
int fl_scan_download(fl_scan_t* s, int which, float* out_xyzi, int cap);
/* fl_filter_update on the down-sampled cloud of `s` without a host hop */
int fl_filter_update_scan(fl_filter_t* f, fl_scan_t* s, double* x26, double* P, double R, double* solve_time_s);

/* ---- device-buffer forms of the scan front end and of the update on it (the conventions of the map's *_device block above)
 * Per scan, fl_localmap_segment_device -> upload -> undistort -> voxel_downsample -> fl_filter_update_scan_device ->
 * fl_filter_map_incremental_device run on the caller's stream with every point count in device memory, so one CUDA graph
 * captured with an upper bound n_max replays a whole scan of any size up to it.  Only esekf::predict stays on the host between
 * replays.
 * None of them synchronises the host, allocates, or sizes a launch from a device value: grids follow n_max (the n_max of the
 * last fl_scan_upload_device) and the kernels stop at the device counts.  Host, wrong-device, null or misaligned pointers are
 * FL_ERR_ARG; an n_max or n_pose_max above what fl_scan_reserve sized is FL_ERR_CAPACITY; nothing is enqueued on a refusal.
 * Ordering: outside capture `stream` first waits for everything enqueued on the map's stream and the map's stream then waits
 * for the call (Map::query_begin / query_end); inside capture nothing is joined.
 * They use buffers of their own, which host-form calls never move, so a graph stays valid across host-form calls on the scan;
 * capture again after fl_scan_reserve grows them.  Each call's outputs equal, byte for byte, those of its host form at the device
 * count n; rows from n up to n_max of the device-form buffers are unspecified.
 * Host forms after device forms: fl_scan_upload / undistort / voxel_downsample / download and fl_filter_update_scan first read
 * the device counts back (once per call, and only once the device forms are in use).  Every device-form stage marks its result
 * as the scan's current one on the device, so when a device-form stage ran after the host forms last took the cloud over
 * (directly or in a graph replay: synchronise replays before host-form calls), the host forms continue from the state the
 * host-form chain would have left.  A host-form undistort or voxel_downsample replaces the cloud: the device-form stages then
 * need a new fl_scan_upload_device (FL_ERR_STATE before it).  Likewise fl_filter_get_nearest / get_selected / map_incremental /
 * get_pass_logs read back which update bound the filter's scan last (a device form, also in a graph replay, or a host form)
 * and run over that scan and its count. */
/* Sizes every device-form buffer, cub's temporary storage for both sorts, and k_undistort's shared memory for up to n_max points
 * and n_pose_max IMU poses (grow-only).  Synchronous.  FL_ERR_CAPACITY when n_pose_max poses exceed the shared memory
 * fl_scan_undistort allows. */
int fl_scan_reserve(fl_scan_t* s, int n_max, int n_pose_max);
/* Measures.lidar (common_lib.h:47-58) from device memory: the first *n_device points (clamped to [0, n_max]) of xyzi_device
 * (4 floats each) and offset_ms_device (PointType::curvature) are copied into the scan, so the caller may reuse its buffers once
 * `stream` has passed the call. */
int fl_scan_upload_device(fl_scan_t* s, const float* xyzi_device, const float* offset_ms_device, const int* n_device, int n_max,
                          void* stream);
/* ImuProcess::UndistortPcl, the sort (:234) and the backward pass (:312-346)         IMU_Processing.hpp:216-346
 * The cloud of the last fl_scan_upload_device, sorted by offset time (stable, over n_max rows whose padding sorts last) and
 * de-skewed with the first *n_pose_device (clamped to [0, n_pose_max]) poses of imu_pose22_device (n_pose_max x 22 doubles, the
 * layout of fl_scan_undistort) and x26_end_device (26 doubles), which are read when `stream` reaches the call.  Fewer than two
 * poses leave the points as sorted, as in fl_scan_undistort.  FL_ERR_STATE without a device-form upload since the last
 * host-form upload, undistort or voxel_downsample. */
int fl_scan_undistort_device(fl_scan_t* s, const double* imu_pose22_device, const int* n_pose_device, int n_pose_max,
                             const double* x26_end_device, void* stream);
/* downSizeFilterSurf.filter(*feats_down_body)                                        laserMapping.cpp:904-905
 * fl_scan_voxel_downsample of the device forms' cloud (de-skewed or as uploaded).  feats_down_size stays in the scan for
 * fl_filter_update_scan_device, and is also copied to n_out_device (may be NULL).  FL_ERR_STATE without a device-form upload since the
 * last host-form upload, undistort or voxel_downsample. */
int fl_scan_voxel_downsample_device(fl_scan_t* s, float leaf_size, int* n_out_device, void* stream);
/* esekf::update_iterated_dyn_share_modified with feats_down_body bound      esekfom.hpp:1619-1931, laserMapping.cpp:638-754, :960
 * fl_filter_update_scan on device buffers: the contract of fl_filter_update_device for x26_device, P_device and status2_device,
 * on the device forms' down-sampled cloud of `s` (bound in place, like fl_filter_update_scan) with its count read on the device.
 * Grids follow the scan's n_max; fl_filter_map_incremental_device afterwards also runs over the device count with n_max = the
 * scan's n_max.  A sharded, solver-0 or fused-0 filter, or a scan without fl_scan_voxel_downsample_device since its last upload,
 * is FL_ERR_STATE; a filter capacity below the scan's n_max FL_ERR_CAPACITY; a scan on another map FL_ERR_ARG. */
int fl_filter_update_scan_device(fl_filter_t* f, fl_scan_t* s, double* x26_device, double* P_device, double R, int* status2_device,
                                 void* stream);

/* ---- batched form of the update over many scans: each slot its own scan and prior, one shared map (a fleet localising on a
 * prior map, offline re-registration of a recorded sequence)
 * esekf::update_iterated_dyn_share_modified run for n_scans (scan, prior) pairs    esekfom.hpp:1619-1931, laserMapping.cpp:638-754
 * scans_device is a device table of n_scans fl_scan_ref_t.  For slot s the count c = *scans_device[s].n is read when `stream`
 * reaches the call.  Per slot: if 0 <= c <= nq_max and the body is non-null and 16-byte aligned (null is allowed when c = 0),
 * x26_device[s], P_device[s], status2_device[s] and logs_device[s][0, passes) receive exactly the bytes fl_filter_update_device
 * gives for rows [0, c) of that body from the prior (x26_device[s], P_device[s]) on the same map, R and parameters; log entries
 * from `passes` on are not written.  A refused slot: c < 0, a null or misaligned body with c > 0, or a null or misaligned
 * (4-byte) count pointer gives status2_device[s] = (FL_ERR_ARG, 0); c > nq_max gives (FL_ERR_CAPACITY, 0).  Its x, P and logs
 * are not touched, and no other slot's result depends on it.  x26_device is [n_scans][26], P_device [n_scans][23 * 23],
 * status2_device [n_scans][2], logs_device (may be NULL) [n_scans][max_iter + 1].
 * The slots run in waves planned at nq_max: fl_filter_batch_plan(f, nq_max, n_scans, out3) gives (workers per slot, slots per
 * wave, waves), and a wave lasts as long as its slowest slot.  The call uses the buffers of fl_filter_reserve_batch(f, >= nq_max)
 * and, like fl_filter_update_batch_device, leaves the filter's own results as they were: the getters, map_incremental (both
 * forms) and the next single update.  Calls that use the batch's buffers of one filter must be ordered on one stream.
 * The scans are read in place, not copied: their rows and counts must stay as they are until `stream` has passed the call.
 * Several slots may reference the same or overlapping rows.
 * The conventions, ordering and capture rules of fl_filter_update_batch_device; the map's deterministic mode is followed.
 * n_scans = 0 returns FL_OK and enqueues nothing.  Refusals enqueue nothing, also on a capturing stream.  FL_ERR_ARG: n_scans or
 * nq_max < 0; a host, wrong-device, null or misaligned pointer (table 8 bytes, x and P 8, status 4, logs 8).  FL_ERR_STATE: no
 * fl_filter_reserve_batch yet, or a sharded, solver-0 or fused-0 filter.  FL_ERR_CAPACITY: nq_max above the reserved nq_max,
 * or one slot does not fit the co-resident grid.
 * fl_scan_get_ref writes the device forms' feats_down_body and feats_down_size of a scan front end as a table entry, and *n_max
 * (may be NULL) the rows fl_scan_reserve sized.  The entry is valid until an fl_scan_reserve that grows the scan (capture
 * again after it).  FL_ERR_STATE before fl_scan_reserve; a null out is FL_ERR_ARG.  Per robot, fl_scan_upload_device ->
 * undistort_device -> voxel_downsample_device, then one fl_filter_update_scans_device over every robot's entry, can be captured
 * into one graph. */
typedef struct fl_scan_ref {
    const float* body_xyzi;   /* device: the scan's rows (x, y, z, intensity), 16-byte aligned */
    const int* n;             /* device: its row count, read when the stream reaches the call */
} fl_scan_ref_t;              /* 16 bytes */
int fl_scan_get_ref(fl_scan_t* s, fl_scan_ref_t* out, int* n_max);
int fl_filter_update_scans_device(fl_filter_t* f, const fl_scan_ref_t* scans_device, int n_scans, int nq_max, double* x26_device,
                                  double* P_device, double R, int* status2_device, fl_pass_log_t* logs_device, void* stream);

/* ---- batched scan front end: UndistortPcl and the voxel grid of many scans in one call, into the table the batched update reads
 * (a fleet's raw scans in, every robot's feats_down_body out, then one fl_filter_update_scans_device)
 * raws_device is a device table of n_scans fl_scan_raw_t.  For slot s the count c = *raws_device[s].n is read when `stream`
 * reaches the call.  If 0 <= c <= n_max and the slot's pointers are valid, the slot's feats_undistort (which 0) and
 * feats_down_body (which 1) rows and its feats_down_size equal, byte for byte, what one fl_scan_t gives for the same inputs:
 * undistort 1: fl_scan_upload_device -> fl_scan_undistort_device -> fl_scan_voxel_downsample_device; undistort 0: upload ->
 * voxel_downsample (the cloud in upload order).  status2_device[s] = (FL_OK, feats_down_size).
 * A refused slot: a null or misaligned (4-byte) n; c < 0; a null or misaligned xyzi (16-byte) or offset_ms (4-byte) with c > 0; with
 * undistort 1 a null or misaligned (8-byte) x26_end, a misaligned n_pose, or a null or misaligned (8-byte) imu_pose22 while
 * *n_pose, clamped to [0, n_pose_max], is >= 2 (a null n_pose is no pose) -- each (FL_ERR_ARG, 0); c > n_max (FL_ERR_CAPACITY, 0).
 * Its counts in both ref tables are -1, which fl_filter_update_scans_device refuses with (FL_ERR_ARG, 0); no other slot depends
 * on it.  The inputs are copied on `stream`: the caller may reuse them once `stream` has passed the call.  Slots may share or
 * overlap their inputs, and may point at fl_preprocess_device outputs (n = &out2_device[0]) or at the slots of a
 * fl_preprocess_batch_t's outputs (below).
 * The outputs live in the handle: per slot a region of n_max rows and a count.  fl_scan_batch_get_refs gives the device table of
 * n_scans_max fl_scan_ref_t for `which` (0 or 1), to hand straight to fl_filter_update_scans_device(f, refs, n_scans, *n_max, ...);
 * slots the last call did not cover have the count -1.  The table's address stays valid until a reserve that grows the handle
 * (capture again after one); its entries are written by each call.  fl_scan_batch_download copies slot `slot`'s rows of the last
 * call into host memory (synchronous, at most cap rows) and returns the slot's count, 0 for a refused slot.
 * The conventions, ordering and capture rules of the scan front end's device forms: no host synchronisation, no allocation, grids
 * follow n_scans x n_max, and the number of launches does not depend on n_scans.  n_scans = 0 returns FL_OK and enqueues nothing.
 * Refusals enqueue nothing, also on a capturing stream.  FL_ERR_ARG: n_scans, n_max or n_pose_max < 0, leaf_size not > 0,
 * undistort not 0 or 1, a host, wrong-device, null or misaligned table (8-byte) or status (4-byte).  FL_ERR_STATE: no
 * fl_scan_batch_reserve yet.  FL_ERR_CAPACITY: n_scans, n_max or n_pose_max above what was reserved, or n_scans x n_max above
 * INT_MAX.  fl_scan_batch_reserve (synchronous, grow-only) sizes the buffers, cub's temporary storage and k_undistort's shared
 * memory; FL_ERR_CAPACITY when n_pose_max poses exceed the 200 KB of shared memory fl_scan_undistort allows, n_scans_max is
 * above 65535 or n_scans_max x n_max above INT_MAX. */
typedef struct fl_scan_raw {
    const float* xyzi;          /* device: rows (x, y, z, intensity), 16-byte aligned -- Measures.lidar */
    const float* offset_ms;     /* device: PointType::curvature per row, 4-byte aligned */
    const int* n;               /* device: the row count, read when the stream reaches the call */
    const double* imu_pose22;   /* device: IMUpose, n_pose x 22 doubles (fl_scan_undistort's layout); may be NULL when undistort is 0 */
    const int* n_pose;          /* device: the pose count, clamped to [0, n_pose_max] as fl_scan_undistort_device does */
    const double* x26_end;      /* device: kf_state.get_x() after the last predict (26 doubles); may be NULL when undistort is 0 */
} fl_scan_raw_t;                /* 48 bytes */
typedef struct fl_scan_batch fl_scan_batch_t;
int fl_scan_batch_create(fl_scan_batch_t** out, fl_map_t* map);
int fl_scan_batch_destroy(fl_scan_batch_t* b);
int fl_scan_batch_reserve(fl_scan_batch_t* b, int n_scans_max, int n_max, int n_pose_max);
int fl_scan_batch_run_device(fl_scan_batch_t* b, const fl_scan_raw_t* raws_device, int n_scans, int n_max, int n_pose_max,
                             int undistort, float leaf_size, int* status2_device, void* stream);
int fl_scan_batch_get_refs(fl_scan_batch_t* b, int which, const fl_scan_ref_t** refs_device, int* n_max);
int fl_scan_batch_download(fl_scan_batch_t* b, int which, int slot, float* out_xyzi, int cap);

/* ---- the scan's clouds in a frame: the clouds a FAST-LIO user consumes after map_incremental (laserMapping.cpp:980-982)
 * which (as in fl_scan_download): 0 feats_undistort (de-skewed, or as uploaded), 1 feats_down_body.  Per row, float (x, y, z,
 * intensity), the intensity passed through; the coordinates in FP64 with Eigen's _transformVector order, then rounded to float:
 *   FL_FRAME_LIDAR  the rows as stored (fl_scan_download)
 *   FL_FRAME_IMU    offset_R_L_I * p + offset_T_L_I                     RGBpointBodyLidarToIMU :211-220, publish_frame_body :532-549
 *   FL_FRAME_WORLD  rot * (offset_R_L_I * p + offset_T_L_I) + pos       RGBpointBodyToWorld :200-209, publish_frame_world :478-529,
 *                                                                        pointBodyToWorld :177-186 (the first scan's Build :909-921)
 * with the state x26 (26 doubles) -- the arithmetic of the update and of map_incremental. */
#define FL_FRAME_LIDAR 0
#define FL_FRAME_IMU 1
#define FL_FRAME_WORLD 2
/* Host form: the current cloud (after the device forms' one, as the other host forms take it over), x26 in host memory (unused
 * for FL_FRAME_LIDAR, may be NULL there).  Writes at most cap rows and returns the cloud's size; synchronous, the conventions of
 * fl_scan_download. */
int fl_scan_frame(fl_scan_t* s, int which, int frame, const double* x26, float* out_xyzi, int cap);
/* Device form, on `stream` (the conventions of the device forms above; capturable).  When `stream` reaches the call it reads the
 * cloud's device count n, x26_device and the append position *n_io_device.  If 0 <= *n_io_device and *n_io_device + n <= cap it
 * writes rows [*n_io_device, *n_io_device + n) of out_xyzi_device and advances *n_io_device by n; otherwise it writes no row and
 * leaves *n_io_device as it was.  status2_device = (status, n): FL_OK, FL_ERR_CAPACITY (the cloud did not fit) or FL_ERR_ARG
 * (*n_io_device outside [0, cap]).  Rows outside the written range are never touched.  Publishing: zero *n_io_device before
 * each scan (a memset node in the graph).  Accumulating (pcl_wait_save += , :521): keep appending, and drain out_xyzi_device on
 * the host every pcd_save_interval scans, then zero *n_io_device.
 * Refusals enqueue nothing, also on a capturing stream.  FL_ERR_ARG: a bad which or frame; cap < 0; a host, wrong-device or
 * misaligned pointer (out 16 bytes, x26 8, n_io and status2 4); a null x26_device for FL_FRAME_IMU or FL_FRAME_WORLD.
 * FL_ERR_STATE: which 0 without a device-form upload since the last host-form upload, undistort or voxel_downsample; which 1
 * without a device-form voxel_downsample since that upload.  The output equals fl_scan_frame's byte for byte at the same count. */
int fl_scan_frame_device(fl_scan_t* s, int which, int frame, const double* x26_device, float* out_xyzi_device, int* n_io_device,
                         int cap, int* status2_device, void* stream);

/* ------------------------------------------------------------------ local-map cube (SURVEY.md §8f row 2)
 * lasermap_fov_segment()                                            laserMapping.cpp:229-277
 * LocalMap_Points / Localmap_Initialized (:229-230) live in the handle; cube_len = cube_side_length (:774),
 * det_range = mapping/det_range (:775). */
typedef struct fl_localmap fl_localmap_t;
int fl_localmap_create(fl_localmap_t** out, double cube_len, float det_range);
int fl_localmap_destroy(fl_localmap_t* l);
/* One call per scan with pos_lid (:236).  Returns |cub_needrm| (0..3); boxes6_out (may be NULL, room for 3 boxes)
 * receives cub_needrm; with map != NULL also runs ikdtree.Delete_Point_Boxes(cub_needrm) (:275) and stores
 * kdtree_delete_counter in *n_deleted (may be NULL). */
int fl_localmap_segment(fl_localmap_t* l, fl_map_t* map, const double* pos_lid, float* boxes6_out, int* n_deleted);
int fl_localmap_get(fl_localmap_t* l, float* box6);   /* LocalMap_Points as (min xyz, max xyz) */
/* lasermap_fov_segment()                                             laserMapping.cpp:229-277
 * pos_lid = pos + rot * offset_T_L_I (:890) from x26_device (26 doubles) when `stream` reaches the call; the cube lives on the
 * map's device.  n_scan_device (may be NULL): when it holds 0 nothing happens (the loop skips an empty scan before the
 * segment, :892-896).  boxes18_device (may be NULL) receives cub_needrm (3 boxes; those past |cub_needrm| are zero);
 * out3_device = (|cub_needrm|, kdtree_delete_counter, status) with the statuses of fl_map_delete_boxes_async.  On
 * FL_ERR_CAPACITY neither the map nor the cube changed (out3[0] and the boxes are what the call would have deleted), so the next
 * call decides again from the unmoved cube.  The slide uses the arithmetic of fl_localmap_segment, and the delete is that of
 * fl_map_delete_boxes_async with its conventions, ordering and capture rules; the launches are the same whether or not the cube
 * moves.  The first call allocates the cube on the map's device and takes over the cube of the host form so far: it must be
 * made outside capture (FL_ERR_STATE on a capturing stream, nothing captured).  A handle used with a second map is FL_ERR_ARG;
 * host, wrong-device, null (x26, out3) or misaligned pointers (x26 8-byte, the others 4-byte) are FL_ERR_ARG; nothing is
 * enqueued on a refusal.  From the first call on, fl_localmap_segment and fl_localmap_get read the device cube back (and the
 * former writes it again), synchronously: synchronise graph replays before those host-form calls. */
int fl_localmap_segment_device(fl_localmap_t* l, fl_map_t* map, const double* x26_device, const int* n_scan_device,
                               float* boxes18_device, int* out3_device, void* stream);

/* ------------------------------------------------------------------ sensor preprocessing (DESIGN §4c)
 * Preprocess::process (src/preprocess.cpp:44-87) with feature_enabled = 0, as every launch file runs it: the raw points of one
 * LiDAR message in, Measures.lidar (pl_surf, the input of fl_scan_upload[_device]) out.  Paths: avia_handler :161-186,
 * velodyne_handler :284-322 + :399-455, oust64_handler :253-279, sim_handler :458-481.  Feature extraction (give_feature)
 * is not provided. */
#define FL_LIDAR_AVIA 1          /* enum LID_TYPE, preprocess.h:16 */
#define FL_LIDAR_VELO16 2
#define FL_LIDAR_OUST64 3
#define FL_LIDAR_MARSIM 4
/* The raw layout: point_step bytes per point and the byte offset of each field (PointField.offset for a PointCloud2; the
 * offsets of livox_ros_driver::CustomPoint for Avia), -1 where the field is absent (it then reads as 0, as PCL's fromROSMsg
 * leaves a field it cannot match).  Offsets need no alignment.  Each type's fields have the types of the reference's structs:
 *   AVIA   livox CustomPoint:       time = offset_time u32 (ns), x/y/z f32, intensity = reflectivity u8, tag u8, line u8
 *   VELO16 velodyne_ros::Point:     x/y/z/intensity f32, time f32 (in time_unit), ring u16            preprocess.h:41-57
 *   OUST64 ouster_ros::Point:       x/y/z/intensity f32, time = t u32 (in time_unit)                  preprocess.h:59-84
 *   MARSIM pcl::PointXYZI:          x/y/z/intensity f32
 * Fields a type does not read are ignored.  The scalars are the ROS parameters laserMapping.cpp:778-787 reads into Preprocess. */
typedef struct fl_preprocess_params {
    int lidar_type;          /* FL_LIDAR_* */
    int n_scans;             /* preprocess/scan_line: N_SCANS, 1..128 (Avia: line < N_SCANS; Velodyne: rings per ring scan) */
    int scan_rate;           /* preprocess/scan_rate: SCAN_RATE in Hz (Velodyne without point times; >= 1 there) */
    int time_unit;           /* preprocess/timestamp_unit: 0 s, 1 ms, 2 us, 3 ns (Velodyne and Ouster) */
    int point_filter_num;    /* point_filter_num >= 1 (MARSIM ignores it, as the reference does) */
    double blind;            /* preprocess/blind in m */
    int point_step;          /* bytes per raw point, >= 1 */
    int off_x, off_y, off_z, off_intensity, off_time, off_ring, off_tag, off_line;
} fl_preprocess_params_t;
typedef struct fl_preprocessor fl_preprocess_t;  /* replaces Preprocess (p_pre, laserMapping.cpp:140) */
/* A handle on `device` for raw frames of up to n_raw_max points: holds the parameters and a workspace sized once (cub's
 * temporary storage, per-row and per-ring scratch, the host form's device copies).  FL_ERR_ARG for a bad type, unit, n_scans,
 * scan_rate, point_filter_num or point_step, or a field that does not fit point_step. */
int fl_preprocess_create(fl_preprocess_t** out, int device, const fl_preprocess_params_t* params, int n_raw_max);
int fl_preprocess_destroy(fl_preprocess_t* h);
/* p_pre->process(msg, ptr) in the LiDAR callback                      laserMapping.cpp:291, :327
 * On the caller's stream: the first *n_raw_device (clamped to [0, n_raw_max]) points of raw_device (n_raw_max x point_step
 * bytes) -> pl_surf in raw order: xyzi_out_device (4 floats per row: x, y, z, intensity) and offset_ms_out_device
 * (PointType::curvature, the offset time in ms), exactly fl_scan_upload_device's inputs.  out2_device = (|pl_surf|, rows
 * dropped for a ring >= n_scans on the Velodyne path without point times, which is undefined behaviour in the reference);
 * last_ms_device (may be NULL) = pl_surf.points.back().curvature, which sync_packages (:381-399) reads for lidar_end_time
 * (0 when nothing is kept).  Rows past |pl_surf| are not written.  The Velodyne offset times derived from the yaw use
 * float(atan2(double, double)) where the reference uses atan2f (DESIGN §4c); everything else is bit-exact.
 * No host synchronisation, allocation or launch sized from a device value, so the call can be captured into a CUDA graph.
 * Host, wrong-device, null or misaligned pointers (xyzi 16-byte; offset times, n, out2, last_ms 4-byte) are FL_ERR_ARG; an
 * n_raw_max above the handle's FL_ERR_CAPACITY; nothing is enqueued on a refusal.  Calls on one handle share its workspace:
 * enqueue them in one stream order, and synchronise graph replays before a host-form call. */
int fl_preprocess_device(fl_preprocess_t* h, const void* raw_device, const int* n_raw_device, int n_raw_max, float* xyzi_out_device,
                         float* offset_ms_out_device, int* out2_device, float* last_ms_device, void* stream);
/* The host form: the same launches on the handle's own stream, after the handle's last device-form call outside capture.
 * Writes min(|pl_surf|, cap) rows, *last_ms (may be NULL) as above; returns |pl_surf| (>= 0) or an error (< 0). */
int fl_preprocess(fl_preprocess_t* h, const void* raw_host, int n_raw, float* xyzi_out, float* offset_ms_out, int cap, float* last_ms);

/* ---- batched preprocessing: Preprocess::process of many raw frames in one call (a fleet's driver points in, every robot's
 * pl_surf out, ready for fl_scan_batch_run_device)
 * One parameter set per handle: every slot is a frame of the handle's LiDAR type and layout (a mixed fleet makes one handle and
 * one call per sensor model).  fl_preprocess_batch_create validates params as fl_preprocess_create does; it sizes everything
 * once for n_slots_max frames of up to n_raw_max points.  FL_ERR_CAPACITY when n_slots_max is above 65535 or n_slots_max x
 * n_raw_max above INT_MAX; FL_ERR_ARG for bad parameters or a negative size.
 * raws_device is a device table of n_slots fl_preprocess_raw_t.  For slot s the count c = *raws_device[s].n_raw is read when
 * `stream` reaches the call.  If 0 <= c <= n_max and the slot's pointers are valid, the slot's rows [0, |pl_surf|) of xyzi and
 * offset_ms, out2[s] = (|pl_surf|, dropped rings) and last_ms[s] equal, byte for byte, what fl_preprocess_device writes for the
 * same frame with the device count c; status2_device[s] = (FL_OK, |pl_surf|).  A refused slot: a null or misaligned (4-byte)
 * n_raw, c < 0, or a null raw with c > 0 -- (FL_ERR_ARG, 0); c > n_max -- (FL_ERR_CAPACITY, 0) (where fl_preprocess_device
 * clamps: a count above the bound means the caller's buffer overflowed).  It writes no row, gets out2[s] = (-1, 0) and
 * last_ms[s] = 0, so fl_scan_batch_run_device (c < 0) and then fl_filter_update_scans_device refuse it too; no other slot
 * depends on it.  Slots [n_slots, n_slots_max) get out2 = (-1, 0) and last_ms = 0.  Slots may share or overlap their raw
 * buffers; the inputs may be reused once `stream` has passed the call.
 * The outputs live in the handle, at addresses fixed at creation (fl_preprocess_batch_get_outputs, any pointer may be NULL):
 * xyzi [n_slots_max][n_raw_max][4], offset_ms [n_slots_max][n_raw_max], out2 [n_slots_max][2], last_ms [n_slots_max]; the slot
 * stride is the handle's n_raw_max, not the call's n_max, so a fl_scan_raw_t table over them (xyzi + s n_raw_max 4, offset_ms +
 * s n_raw_max, n = out2 + 2 s) is built once and read in place by fl_scan_batch_run_device.  fl_preprocess_batch_download
 * copies slot `slot`'s rows of the last call into host memory (synchronous, at most cap rows; last_ms may be NULL), after the
 * handle's last call outside capture (synchronise graph replays first), and returns the slot's |pl_surf|, 0 for a refused slot.
 * No host synchronisation, no allocation, no launch sized from a device value, and the number of launches does not depend on
 * n_slots (the ring sort's bits are fixed by n_slots_max), so the call can be captured into a CUDA graph.  n_slots = 0 returns
 * FL_OK and enqueues nothing.  Refusals enqueue nothing, also on a capturing stream.  FL_ERR_ARG: n_slots or n_max < 0; a host,
 * wrong-device, null or misaligned table (8-byte) or status2 (4-byte).  FL_ERR_CAPACITY: n_slots above n_slots_max, n_max above
 * n_raw_max.  Calls on one handle share its workspace: enqueue them in one stream order. */
typedef struct fl_preprocess_raw {
    const void* raw;            /* device: the driver's points, point_step bytes each, no alignment required */
    const int* n_raw;           /* device: the row count, read when the stream reaches the call */
} fl_preprocess_raw_t;          /* 16 bytes */
typedef struct fl_preprocess_batch fl_preprocess_batch_t;
int fl_preprocess_batch_create(fl_preprocess_batch_t** out, int device, const fl_preprocess_params_t* params, int n_slots_max,
                               int n_raw_max);
int fl_preprocess_batch_destroy(fl_preprocess_batch_t* b);
int fl_preprocess_batch_run_device(fl_preprocess_batch_t* b, const fl_preprocess_raw_t* raws_device, int n_slots, int n_max,
                                   int* status2_device, void* stream);
int fl_preprocess_batch_get_outputs(fl_preprocess_batch_t* b, float** xyzi, float** offset_ms, int** out2, float** last_ms,
                                    int* n_raw_max);
int fl_preprocess_batch_download(fl_preprocess_batch_t* b, int slot, float* out_xyzi, float* out_offset_ms, int cap, float* last_ms);

/* ------------------------------------------------------------------ multi-GPU (no reference counterpart)
 * scan points are sharded across ranks, the map is replicated, the 92 normal-equation doubles
 * are all-reduced once per pass (NCCL over NVLink) and every rank solves redundantly. */
int fl_comm_unique_id(void* out128);
int fl_filter_comm_init(fl_filter_t* f, int nranks, int rank, const void* unique_id128);
int fl_filter_set_shard(fl_filter_t* f, int q_begin, int q_end);
/* Same exchange without NCCL, fused into the residual kernel: each rank exports its mailbox as a 64-byte CUDA-IPC
 * handle (fl_filter_p2p_handle), the application all-gathers the handles, fl_filter_p2p_connect maps the peers.
 * Per pass every rank stores its 92 sums straight into its peers' mailboxes over NVLink as epoch-tagged 8-byte words
 * (the data is the flag) and adds the slots of its own mailbox in rank order: every rank ends with the same bits. */
int fl_filter_p2p_handle(fl_filter_t* f, void* out64);
int fl_filter_p2p_connect(fl_filter_t* f, int nranks, int rank, const void* handles /* nranks x 64 bytes */);

#ifdef __cplusplus
}
#endif
#endif /* FASTLIO_B200_H */
