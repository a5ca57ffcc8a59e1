// ============================================================================
// ORACLE -- TEST INFRASTRUCTURE ONLY (see oracle/fastlio_oracle.cpp header).
//
// extern "C" wrapper around the reference's own KD_TREE::Box_Search and
// KD_TREE::Radius_Search (include/ikd-Tree/ikd_Tree.cpp:464-475).  It is linked
// against oracle/_ref/libikdtree_ref.so, which holds the reference's explicit
// instantiation of KD_TREE<pcl::PointXYZINormal>, and acts on the tree handles
// that library's ref_kdtree_create returns.  Built by oracle/range_ref.py into
// oracle/_ref/libikdtree_range.so; nothing from the reference is copied here.
// ============================================================================
#include <ikd_Tree.h>

#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef pcl::PointXYZINormal PointType;
typedef KD_TREE<PointType> Tree;
typedef Tree::PointVector PointVector;

// One public call per query, the answers concatenated in query order in the CSR layout of fl_map_box_search /
// fl_map_radius_search (include/fastlio_b200.h).  nthreads > 1 runs the queries in an OpenMP loop, each into its own
// vector; the concatenation is the same.  Returns the total, writes at most cap points.
template <class F>
static int range_batch(int nq, int* out_offsets, float* out4, int cap, int nthreads, F one) {
    std::vector<PointVector> res(nq);
#ifdef _OPENMP
    if (nthreads > 0) omp_set_num_threads(nthreads);
#pragma omp parallel for schedule(dynamic, 16) if (nthreads > 1)
#endif
    for (int i = 0; i < nq; i++) one(i, res[i]);
    int total = 0;
    for (int i = 0; i < nq; i++) {
        out_offsets[i] = total;
        for (const PointType& p : res[i]) {
            if (total < cap) {
                float* o = &out4[size_t(total) * 4];
                o[0] = p.x; o[1] = p.y; o[2] = p.z; o[3] = p.intensity;
            }
            total++;
        }
    }
    out_offsets[nq] = total;
    return total;
}

extern "C" {

int ref_kdtree_box_search(void* h, const float* boxes6, int nb, int* out_offsets, float* out4, int cap, int nthreads) {
    Tree* t = static_cast<Tree*>(h);
    return range_batch(nb, out_offsets, out4, cap, nthreads, [&](int i, PointVector& v) {
        BoxPointType b;
        for (int a = 0; a < 3; a++) { b.vertex_min[a] = boxes6[size_t(i) * 6 + a]; b.vertex_max[a] = boxes6[size_t(i) * 6 + 3 + a]; }
        t->Box_Search(b, v);
    });
}

int ref_kdtree_radius_search(void* h, const float* centers4, int nq, int* out_offsets, float* out4, int cap, int nthreads) {
    Tree* t = static_cast<Tree*>(h);
    return range_batch(nq, out_offsets, out4, cap, nthreads, [&](int i, PointVector& v) {
        PointType c;
        c.x = centers4[size_t(i) * 4]; c.y = centers4[size_t(i) * 4 + 1]; c.z = centers4[size_t(i) * 4 + 2];
        t->Radius_Search(c, centers4[size_t(i) * 4 + 3], v);
    });
}

}  // extern "C"
