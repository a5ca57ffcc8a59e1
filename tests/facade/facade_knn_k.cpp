// EXECUTES the k-nearest queries of the KD_TREE<PointType> facade on a GPU (tests/test_gpu_knn_k.py builds and runs it):
// Nearest_Search_K one query per call, then Nearest_Search_K_Batch over all of them, for each (k, max_dist) pair.
//   usage: facade_knn_k <in.bin> <out.bin>
//   in : int32 n_map, nq, npairs; float32 map[n_map*4], queries[nq*4]; npairs x (int32 k, float32 max_dist)
//   out: per pair two result sets (one query per call, batched), each int32 counts[nq] followed by, query after query,
//        float32 points[cnt*4] (x, y, z, intensity) and float32 d2[cnt]
#include <ikd-Tree/ikd_Tree.h>

#include <cstdio>
#include <vector>

typedef pcl::PointXYZINormal PointType;
typedef KD_TREE<PointType>::PointVector PointVector;

template <class T> static bool rd(FILE* f, T* p, size_t n) { return fread(p, sizeof(T), n, f) == n; }

static void write_set(FILE* f, const std::vector<PointVector>& pts, const std::vector<std::vector<float>>& d2) {
    for (const auto& v : pts) { const int n = (int)v.size(); fwrite(&n, sizeof(int), 1, f); }
    for (size_t i = 0; i < pts.size(); i++) {
        for (const auto& p : pts[i]) { const float o[4] = {p.x, p.y, p.z, p.intensity}; fwrite(o, sizeof(float), 4, f); }
        fwrite(d2[i].data(), sizeof(float), d2[i].size(), f);
    }
}

int main(int argc, char** argv) {
    if (argc < 3) { fprintf(stderr, "usage: facade_knn_k in out\n"); return 2; }
    FILE* fi = fopen(argv[1], "rb");
    if (!fi) { perror("in"); return 2; }
    int hdr[3];
    if (!rd(fi, hdr, 3)) return 2;
    const int n_map = hdr[0], nq = hdr[1], npairs = hdr[2];
    std::vector<float> map((size_t)n_map * 4), qs((size_t)nq * 4);
    if (!rd(fi, map.data(), map.size()) || !rd(fi, qs.data(), qs.size())) return 2;
    std::vector<int> ks(npairs);
    std::vector<float> mds(npairs);
    for (int i = 0; i < npairs; i++) if (!rd(fi, &ks[i], 1) || !rd(fi, &mds[i], 1)) return 2;
    fclose(fi);

    KD_TREE<PointType> ikdtree(0.5f, 0.6f, 0.5f);
    if (!ikdtree.ok()) { fprintf(stderr, "no device map: %s\n", KD_TREE<PointType>::last_error()); return 3; }
    PointVector cloud(n_map);
    for (int i = 0; i < n_map; i++) { cloud[i].x = map[4 * i]; cloud[i].y = map[4 * i + 1]; cloud[i].z = map[4 * i + 2]; cloud[i].intensity = map[4 * i + 3]; }
    ikdtree.Build(cloud);
    PointVector queries(nq);
    for (int i = 0; i < nq; i++) { queries[i].x = qs[4 * i]; queries[i].y = qs[4 * i + 1]; queries[i].z = qs[4 * i + 2]; }

    FILE* fo = fopen(argv[2], "wb");
    if (!fo) { perror("out"); return 2; }
    for (int c = 0; c < npairs; c++) {
        std::vector<PointVector> one_p(nq), batch_p;
        std::vector<std::vector<float>> one_d(nq), batch_d;
        for (int i = 0; i < nq; i++) {
            one_p[i].push_back(PointType());           // Nearest_Search_K replaces what the vectors held
            one_d[i].push_back(-1.f);
            ikdtree.Nearest_Search_K(queries[i], ks[c], one_p[i], one_d[i], mds[c]);
        }
        ikdtree.Nearest_Search_K_Batch(queries, ks[c], batch_p, batch_d, mds[c]);
        write_set(fo, one_p, one_d);
        write_set(fo, batch_p, batch_d);
    }
    fclose(fo);
    if (ikdtree.failed()) { fprintf(stderr, "a KD_TREE call failed: %s\n", KD_TREE<PointType>::last_error()); return 6; }
    // an unsupported k is reported, not clamped
    std::vector<float> d;
    PointVector p;
    ikdtree.Nearest_Search_K(queries.empty() ? PointType() : queries[0], 33, p, d);
    if (!ikdtree.failed() || !p.empty()) { fprintf(stderr, "k = 33 was not refused\n"); return 7; }
    printf("facade_knn_k ok: %d queries, %d (k, max_dist) pairs\n", nq, npairs);
    return 0;
}
