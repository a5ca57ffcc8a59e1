// Drop-in facade: KD_TREE<PointType> with the call surface of the reference's
// include/ikd-Tree/ikd_Tree.h (hku-mars/ikd-Tree @ e2e3f4e), served by the H100 device map
// through the C ABI in fastlio_b200.h.  Put this directory in front of the reference's
// include path and link libfastlio_b200.so; src/laserMapping.cpp compiles unchanged.
//
// Header-only; needs the PointType headers the reference already uses (pcl/point_types.h,
// Eigen::aligned_allocator).  Only x, y, z, intensity of a point live in the map
// (the fields FAST-LIO reads back: laserMapping.cpp:438-460, 680); normals/curvature of
// points returned by a search are zero.
//
//   reference member                         this facade
//   ---------------------------------------  ------------------------------------------------
//   KD_TREE(delete, balance, box_length)     fl_map_create (criteria have no counterpart)
//   set_downsample_param / Initialize...     fl_map_set_downsample
//   Build(PointVector)                       fl_map_build
//   Nearest_Search(p, k, out, dist, max)     fl_map_knn, one query per call (thread-safe, slow:
//                                            the fused filter path never calls it -- see
//                                            IKFoM_toolkit/esekfom/esekfom_b200.hpp)
//   Add_Points(PointVector&, bool)           fl_map_add_points        (same return value)
//   Delete_Point_Boxes(vector<Box>&)         fl_map_delete_boxes      (same return value)
//   size() / validnum() / tree_range()       fl_map_size / fl_map_validnum / fl_map_tree_range
//   flatten(root, Storage, type)             fl_map_flatten (all valid points)
//   Box_Search(box, Storage)                 fl_map_box_search, one box per call (same point set; order differs)
//   Radius_Search(p, r, Storage)             fl_map_radius_search, one sphere per call: the literal test of
//                                            ikd_Tree.cpp:1308, d2 <= r * r; the reference may differ on points with
//                                            d2 > fl(r * r) and sqrtf(d2) <= r (it decides leaves by sqrtf)
//   (extension) Box_Search_Batch /           the same, all queries in one call
//               Radius_Search_Batch
//   (extension) Nearest_Search_K(p, k, out,  fl_map_nearest_search: any 1 <= k <= 32, max_dist applied on the device
//               dist, max) / _K_Batch        (d2 <= fl(max_dist * max_dist)); one query per call / all queries in one call
//   Delete_Points(PointVector&)              fl_map_delete_boxes with 2e-6 m boxes (same_point EPSS)
//   Add_Point_Boxes(vector<Box>&)            fl_map_add_boxes: box-deleted points not yet overwritten come back
//   acquire_removed_points(PointVector&)     fl_map_acquire_removed: the points removed by Delete_Point_Boxes since the last call
//                                            (the reference hands them over when it rebuilds the subtree; here at once)
//   Root_Node                                non-null once built (laserMapping.cpp:909 tests it)
//   (extension) set_deterministic(bool)      fl_map_set_deterministic: k-NN answers, the down-sampling survivor and the
//                                            update depend only on the map's point set; FASTLIO_B200_DETERMINISTIC=1 turns
//                                            it on at construction
//
// Limits and failure reporting (the reference's members return void / int and cannot fail):
//   * k_nearest <= 5 (NUM_MATCH_POINTS, include/common_lib.h:26 -- the only k FAST-LIO uses).  A larger k is an error:
//     the call prints a diagnostic once, returns no neighbours and sets failed().  Nearest_Search_K takes 1 <= k <= 32;
//     outside that range it returns no neighbours and sets failed().
//   * the CUDA device is chosen by KD_TREE::set_default_device(i) before construction, else by the environment variable
//     FASTLIO_B200_DEVICE, else device 0 (the reference's tree is a global object, laserMapping.cpp:120).
//   * ok() tells whether the device map exists (no GPU / out of memory at construction); failed() whether any call on
//     this object has failed since clear_failed(); last_error() returns the library's message.
#pragma once
#include <stdlib.h>
#include <math.h>
#include <stdio.h>

#include <algorithm>
#include <memory>
#include <vector>

#include <pcl/point_types.h>

#include "../fastlio_b200.h"

struct BoxPointType {
    float vertex_min[3];
    float vertex_max[3];
};

enum delete_point_storage_set { NOT_RECORD, DELETE_POINTS_REC, MULTI_THREAD_REC };

template <typename PointType>
class KD_TREE {
public:
    using PointVector = std::vector<PointType, Eigen::aligned_allocator<PointType>>;
    using Ptr = std::shared_ptr<KD_TREE<PointType>>;
    struct KD_TREE_NODE { int unused; };

    KD_TREE(float delete_param = 0.5, float balance_param = 0.6, float box_length = 0.2) : downsample_size_(box_length) {
        (void)delete_param; (void)balance_param;
        int dev = default_device();
        if (dev < 0) { const char* e = getenv("FASTLIO_B200_DEVICE"); dev = e ? atoi(e) : 0; }
        device_ = dev;
        if (fl_map_create(&map_, dev, box_length) != FL_OK) {
            fprintf(stderr, "KD_TREE(H100): cannot create the device map on CUDA device %d: %s\n", dev, fl_last_error());
            map_ = nullptr;
            failed_ = true;
        } else if (const char* d = getenv("FASTLIO_B200_DETERMINISTIC")) {
            if (d[0] == '1') set_deterministic(true);
        }
    }
    // extension: the deterministic mode (fl_map_set_deterministic); FASTLIO_B200_DETERMINISTIC=1 turns it on at construction
    void set_deterministic(bool on) { if (map_) check(fl_map_set_deterministic(map_, on ? 1 : 0), "set_deterministic"); }
    bool deterministic() const {
        int on = 0;
        return map_ && fl_map_get_deterministic(map_, &on) == FL_OK && on;
    }
    // extension: device selection and failure reporting (see the header comment)
    static void set_default_device(int device) { default_device() = device; }
    int device() const { return device_; }
    bool ok() const { return map_ != nullptr; }
    bool failed() const { return failed_; }
    void clear_failed() { failed_ = false; }
    static const char* last_error() { return fl_last_error(); }
    ~KD_TREE() { if (map_) fl_map_destroy(map_); }
    KD_TREE(const KD_TREE&) = delete;
    KD_TREE& operator=(const KD_TREE&) = delete;

    void Set_delete_criterion_param(float) {}
    void Set_balance_criterion_param(float) {}
    void set_downsample_param(float v) { downsample_size_ = v; if (map_) fl_map_set_downsample(map_, v); }
    void InitializeKDTree(float delete_param = 0.5, float balance_param = 0.7, float box_length = 0.2) {
        (void)delete_param; (void)balance_param;
        set_downsample_param(box_length);
    }
    int size() { return map_ ? fl_map_size(map_) : 0; }
    int validnum() { return map_ ? fl_map_validnum(map_) : 0; }
    void root_alpha(float& alpha_bal, float& alpha_del) { alpha_bal = 0.5f; alpha_del = 0.0f; }

    void Build(PointVector point_cloud) {
        std::vector<float> buf;
        pack(point_cloud, buf);
        check(fl_map_build(map_, buf.data(), (int)point_cloud.size()), "Build");
        Root_Node = point_cloud.empty() ? nullptr : &root_token_;
    }

    void Nearest_Search(PointType point, int k_nearest, PointVector& Nearest_Points, std::vector<float>& Point_Distance,
                        float max_dist = INFINITY) {
        Nearest_Points.clear();
        Point_Distance.clear();
        if (!check_k(k_nearest)) return;
        const int k = k_nearest;
        float q[4] = {point.x, point.y, point.z, 0.f};
        float pts[20], d2[5];
        int cnt = 0;
        if (check(fl_map_knn(map_, q, 1, k, pts, d2, &cnt), "Nearest_Search") != FL_OK) return;
        const float md2 = max_dist * max_dist;
        for (int i = 0; i < cnt; i++) {
            if (d2[i] > md2) break;
            Nearest_Points.push_back(unpack(&pts[4 * i]));
            Point_Distance.push_back(d2[i]);
        }
    }

    // extension: all queries in one launch (what a batched caller should use)
    void Nearest_Search_Batch(const PointVector& queries, int k_nearest, std::vector<PointVector>& out_points,
                              std::vector<std::vector<float>>& out_dist) {
        out_points.clear();
        out_dist.clear();
        if (!check_k(k_nearest)) return;
        const int nq = (int)queries.size(), k = k_nearest;
        std::vector<float> q, pts((size_t)nq * k * 4), d2((size_t)nq * k);
        std::vector<int> cnt(nq);
        pack(queries, q);
        out_points.assign(nq, PointVector());
        out_dist.assign(nq, std::vector<float>());
        if (nq == 0 || check(fl_map_knn(map_, q.data(), nq, k, pts.data(), d2.data(), cnt.data()), "Nearest_Search_Batch") != FL_OK) return;
        for (int i = 0; i < nq; i++)
            for (int j = 0; j < cnt[i]; j++) {
                out_points[i].push_back(unpack(&pts[((size_t)i * k + j) * 4]));
                out_dist[i].push_back(d2[(size_t)i * k + j]);
            }
    }

    // extension: KD_TREE::Nearest_Search for any 1 <= k_nearest <= 32, with max_dist applied by the device search
    void Nearest_Search_K(PointType point, int k_nearest, PointVector& Nearest_Points, std::vector<float>& Point_Distance,
                          float max_dist = INFINITY) {
        std::vector<PointVector> p;
        std::vector<std::vector<float>> d;
        Nearest_Search_K_Batch(PointVector(1, point), k_nearest, p, d, max_dist);
        Nearest_Points.swap(p[0]);
        Point_Distance.swap(d[0]);
    }
    void Nearest_Search_K_Batch(const PointVector& queries, int k_nearest, std::vector<PointVector>& out_points,
                                std::vector<std::vector<float>>& out_dist, float max_dist = INFINITY) {
        const int nq = (int)queries.size();
        out_points.assign(nq, PointVector());
        out_dist.assign(nq, std::vector<float>());
        const int k = std::max(k_nearest, 1);
        std::vector<float> q, pts((size_t)nq * k * 4), d2((size_t)nq * k);
        std::vector<int> cnt(std::max(nq, 1));
        pack(queries, q);
        if (check(fl_map_nearest_search(map_, q.data(), nq, k_nearest, max_dist, pts.data(), d2.data(), cnt.data()), "Nearest_Search_K") != FL_OK) return;
        for (int i = 0; i < nq; i++)
            for (int j = 0; j < cnt[i]; j++) {
                out_points[i].push_back(unpack(&pts[((size_t)i * k + j) * 4]));
                out_dist[i].push_back(d2[(size_t)i * k + j]);
            }
    }

    void Box_Search(const BoxPointType& box, PointVector& Storage) {
        Storage.clear();
        float b[6];
        box6(box, b);
        range_search(fl_map_box_search, b, 1, &Storage, "Box_Search");
    }
    void Radius_Search(PointType point, const float radius, PointVector& Storage) {
        Storage.clear();
        const float q[4] = {point.x, point.y, point.z, radius};
        range_search(fl_map_radius_search, q, 1, &Storage, "Radius_Search");
    }
    // extension: all boxes / spheres in one call (out[i] = Box_Search(boxes[i]) / Radius_Search(centers[i], radii[i]))
    void Box_Search_Batch(const std::vector<BoxPointType>& boxes, std::vector<PointVector>& out) {
        std::vector<float> b(boxes.size() * 6);
        for (size_t i = 0; i < boxes.size(); i++) box6(boxes[i], &b[6 * i]);
        out.assign(boxes.size(), PointVector());
        if (!boxes.empty()) range_search(fl_map_box_search, b.data(), (int)boxes.size(), out.data(), "Box_Search_Batch");
    }
    void Radius_Search_Batch(const PointVector& centers, const std::vector<float>& radii, std::vector<PointVector>& out) {
        out.assign(centers.size(), PointVector());
        if (radii.size() != centers.size() && radii.size() != 1) { check(FL_ERR_ARG, "Radius_Search_Batch (one radius, or one per centre)"); return; }
        std::vector<float> q(centers.size() * 4);
        for (size_t i = 0; i < centers.size(); i++) {
            q[4 * i] = centers[i].x; q[4 * i + 1] = centers[i].y; q[4 * i + 2] = centers[i].z;
            q[4 * i + 3] = radii.size() == 1 ? radii[0] : radii[i];
        }
        if (!centers.empty()) range_search(fl_map_radius_search, q.data(), (int)centers.size(), out.data(), "Radius_Search_Batch");
    }
    void Radius_Search_Batch(const PointVector& centers, float radius, std::vector<PointVector>& out) {
        Radius_Search_Batch(centers, std::vector<float>(1, radius), out);
    }

    int Add_Points(PointVector& PointToAdd, bool downsample_on) {
        std::vector<float> buf;
        pack(PointToAdd, buf);
        int rc = fl_map_add_points(map_, buf.data(), (int)PointToAdd.size(), downsample_on ? 1 : 0);
        if (rc < 0) { check(rc, "Add_Points"); return 0; }
        if (!PointToAdd.empty()) Root_Node = &root_token_;
        return rc;
    }
    void Add_Point_Boxes(std::vector<BoxPointType>& BoxPoints) {
        std::vector<float> boxes;
        for (const auto& b : BoxPoints) {
            for (int a = 0; a < 3; a++) boxes.push_back(b.vertex_min[a]);
            for (int a = 0; a < 3; a++) boxes.push_back(b.vertex_max[a]);
        }
        if (!boxes.empty()) check(std::min(0, fl_map_add_boxes(map_, boxes.data(), (int)BoxPoints.size())), "Add_Point_Boxes");
    }
    void Delete_Points(PointVector& PointToDel) {
        std::vector<float> boxes;
        for (const auto& p : PointToDel) {
            const float c[3] = {p.x, p.y, p.z};
            for (int a = 0; a < 3; a++) boxes.push_back(c[a] - 1e-6f);
            for (int a = 0; a < 3; a++) boxes.push_back(nextafterf(c[a] + 1e-6f, INFINITY));
        }
        if (!boxes.empty()) check(std::min(0, fl_map_delete_boxes(map_, boxes.data(), (int)PointToDel.size())), "Delete_Points");
    }
    int Delete_Point_Boxes(std::vector<BoxPointType>& BoxPoints) {
        std::vector<float> boxes;
        for (const auto& b : BoxPoints) {
            for (int a = 0; a < 3; a++) boxes.push_back(b.vertex_min[a]);
            for (int a = 0; a < 3; a++) boxes.push_back(b.vertex_max[a]);
        }
        int rc = fl_map_delete_boxes(map_, boxes.data(), (int)BoxPoints.size());
        if (rc < 0) { check(rc, "Delete_Point_Boxes"); return 0; }
        removed_pending_ += rc;
        return rc;
    }
    void flatten(KD_TREE_NODE*, PointVector& Storage, delete_point_storage_set) {
        const int n = validnum();
        std::vector<float> buf((size_t)std::max(n, 1) * 4);
        const int got = fl_map_flatten(map_, buf.data(), n);
        if (got < 0) { check(got, "flatten"); return; }
        for (int i = 0; i < got; i++) Storage.push_back(unpack(&buf[(size_t)i * 4]));
    }
    void acquire_removed_points(PointVector& removed_points) {
        // history of the points Delete_Point_Boxes removed since the previous call (the very first call starts the record)
        std::vector<float> buf((size_t)std::max(removed_pending_, 1) * 4);
        const int n = fl_map_acquire_removed(map_, buf.data(), removed_pending_);
        if (n < 0) { check(n, "acquire_removed_points"); return; }
        for (int i = 0; i < std::min(n, removed_pending_); i++) removed_points.push_back(unpack(&buf[(size_t)i * 4]));
        removed_pending_ = 0;
    }
    BoxPointType tree_range() {
        BoxPointType r;
        float b[6] = {0, 0, 0, 0, 0, 0};
        if (map_) fl_map_tree_range(map_, b);
        for (int a = 0; a < 3; a++) { r.vertex_min[a] = b[a]; r.vertex_max[a] = b[3 + a]; }
        return r;
    }

    PointVector PCL_Storage;
    KD_TREE_NODE* Root_Node = nullptr;
    int max_queue_size = 0;

    // extension: the device map, to bind the fused measurement update (esekfom_b200.hpp)
    fl_map_t* handle() const { return map_; }

private:
    static void pack(const PointVector& v, std::vector<float>& out) {
        out.resize(v.size() * 4);
        for (size_t i = 0; i < v.size(); i++) { out[4 * i] = v[i].x; out[4 * i + 1] = v[i].y; out[4 * i + 2] = v[i].z; out[4 * i + 3] = intensity_of(v[i], 0); }
    }
    template <class P> static auto intensity_of(const P& p, int) -> decltype(p.intensity, 0.f) { return p.intensity; }
    template <class P> static float intensity_of(const P&, long) { return 0.f; }
    template <class P> static auto set_intensity(P& p, float v, int) -> decltype(p.intensity, void()) { p.intensity = v; }
    template <class P> static void set_intensity(P&, float, long) {}
    static PointType unpack(const float* f) {
        PointType p;
        p.x = f[0]; p.y = f[1]; p.z = f[2];
        set_intensity(p, f[3], 0);
        return p;
    }
    static void box6(const BoxPointType& b, float* out) {
        for (int a = 0; a < 3; a++) { out[a] = b.vertex_min[a]; out[3 + a] = b.vertex_max[a]; }
    }
    // one batched range call; query i's points are appended to out[i].  The buffer kept between calls usually has room; when
    // the total is larger, the call is repeated once with room for it.
    void range_search(int (*fn)(fl_map_t*, const float*, int, int*, float*, int), const float* q, int nq, PointVector* out, const char* what) {
        std::vector<int> offsets((size_t)nq + 1);
        if (range_buf_.empty()) range_buf_.resize(4 * 4096);
        int total = fn(map_, q, nq, offsets.data(), range_buf_.data(), (int)(range_buf_.size() / 4));
        if (total > (int)(range_buf_.size() / 4)) {
            range_buf_.resize((size_t)total * 4);
            total = fn(map_, q, nq, offsets.data(), range_buf_.data(), total);
        }
        if (check(std::min(0, total), what) < 0) return;
        for (int i = 0; i < nq; i++) {
            out[i].reserve(out[i].size() + (size_t)(offsets[i + 1] - offsets[i]));
            for (int j = offsets[i]; j < offsets[i + 1]; j++) out[i].push_back(unpack(&range_buf_[(size_t)j * 4]));
        }
    }
    int check(int rc, const char* what) {
        if (rc < 0) { failed_ = true; fprintf(stderr, "KD_TREE(H100)::%s failed: %s\n", what, fl_last_error()); }
        return rc;
    }
    bool check_k(int k) {
        if (k >= 1 && k <= 5) return true;
        failed_ = true;
        static bool told = false;
        if (!told) { told = true; fprintf(stderr, "KD_TREE(H100)::Nearest_Search: k_nearest = %d is not supported (1 <= k <= 5, NUM_MATCH_POINTS)\n", k); }
        return false;
    }
    static int& default_device() { static int d = -1; return d; }
    int device_ = 0;
    int removed_pending_ = 0;      // points deleted by boxes since the last acquire_removed_points
    std::vector<float> range_buf_; // host buffer of the range searches, grown to the largest answer seen
    bool failed_ = false;
    fl_map_t* map_ = nullptr;
    float downsample_size_;
    KD_TREE_NODE root_token_{0};
};
