// ============================================================================
// ORACLE -- TEST INFRASTRUCTURE ONLY (see oracle/fastlio_oracle.cpp header).
//
// extern "C" wrapper around the reference's own KD_TREE::Nearest_Search with
// its max_dist argument (include/ikd-Tree/ikd_Tree.cpp:426-461).  It is linked
// against oracle/_ref/libikdtree_ref.so, which holds the reference's explicit
// instantiation of KD_TREE<pcl::PointXYZINormal>, and acts on the tree handles
// that library's ref_kdtree_create returns.  Built by oracle/knn_ref.py into
// oracle/_ref/libikdtree_knn.so; nothing from the reference is copied here.
// ============================================================================
#include <ikd_Tree.h>

#include <cmath>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef pcl::PointXYZINormal PointType;
typedef KD_TREE<PointType> Tree;
typedef Tree::PointVector PointVector;

extern "C" {

// One public call per query, in the layout of fl_map_nearest_search (include/fastlio_b200.h): out_pts4 nq*k*4 floats,
// out_d2 nq*k, out_cnt nq; entries past the count are (0, 0, 0, 0) with d2 = +inf.  nthreads > 1 runs the queries in an
// OpenMP loop.
void ref_kdtree_nearest_search(void* h, const float* q4, int nq, int k, float max_dist, float* out_pts4, float* out_d2,
                               int* out_cnt, int nthreads) {
    Tree* t = static_cast<Tree*>(h);
#ifdef _OPENMP
    if (nthreads > 0) omp_set_num_threads(nthreads);
#pragma omp parallel for schedule(dynamic, 64) if (nthreads > 1)
#endif
    for (int i = 0; i < nq; i++) {
        PointType q;
        q.x = q4[size_t(i) * 4]; q.y = q4[size_t(i) * 4 + 1]; q.z = q4[size_t(i) * 4 + 2];
        PointVector near;
        std::vector<float> d2;
        t->Nearest_Search(q, k, near, d2, max_dist);
        const int cnt = int(near.size());
        for (int j = 0; j < k; j++) {
            float* o = &out_pts4[(size_t(i) * k + j) * 4];
            if (j < cnt) { o[0] = near[j].x; o[1] = near[j].y; o[2] = near[j].z; o[3] = near[j].intensity; out_d2[size_t(i) * k + j] = d2[j]; }
            else { o[0] = o[1] = o[2] = o[3] = 0.f; out_d2[size_t(i) * k + j] = INFINITY; }
        }
        out_cnt[i] = cnt;
    }
}

}  // extern "C"
