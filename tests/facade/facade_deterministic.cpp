// EXECUTES the deterministic mode of the KD_TREE<PointType> facade on a GPU (tests/test_gpu_deterministic.py builds and runs it):
// the mode as FASTLIO_B200_DETERMINISTIC set it at construction, then set_deterministic(false / true) and their effect; the map
// is built from the first half of the points and the rest added (Add_Points without down-sampling), so its slot layout differs
// from a plain Build of the same points.
//   usage: facade_deterministic <in.bin> <out.bin>
//   in : int32 n_map, nq, k; float32 map[n_map*4], queries[nq*4]
//   out: int32 mode at construction; int32 counts[nq]; then query after query float32 points[cnt*4] (x, y, z, intensity);
//        int32 n_flat; float32 flatten rows[n_flat*4]
#include <ikd-Tree/ikd_Tree.h>

#include <cstdio>
#include <vector>

typedef pcl::PointXYZINormal PointType;
typedef KD_TREE<PointType>::PointVector PointVector;

template <class T> static bool rd(FILE* f, T* p, size_t n) { return fread(p, sizeof(T), n, f) == n; }

int main(int argc, char** argv) {
    if (argc < 3) { fprintf(stderr, "usage: facade_deterministic in out\n"); return 2; }
    FILE* fi = fopen(argv[1], "rb");
    if (!fi) { perror("in"); return 2; }
    int hdr[3];
    if (!rd(fi, hdr, 3)) return 2;
    const int n_map = hdr[0], nq = hdr[1], k = hdr[2];
    std::vector<float> map((size_t)n_map * 4), qs((size_t)nq * 4);
    if (!rd(fi, map.data(), map.size()) || !rd(fi, qs.data(), qs.size())) return 2;
    fclose(fi);

    KD_TREE<PointType> ikdtree(0.5f, 0.6f, 0.5f);
    if (!ikdtree.ok()) { fprintf(stderr, "no device map: %s\n", KD_TREE<PointType>::last_error()); return 3; }
    const int at_construction = ikdtree.deterministic() ? 1 : 0;
    // the setter switches both ways and the getter follows it
    ikdtree.set_deterministic(!at_construction);
    if (ikdtree.deterministic() == (at_construction != 0)) { fprintf(stderr, "set_deterministic did not switch\n"); return 4; }
    ikdtree.set_deterministic(at_construction != 0);
    if (ikdtree.deterministic() != (at_construction != 0)) { fprintf(stderr, "set_deterministic did not switch back\n"); return 4; }

    PointVector first, rest;
    for (int i = 0; i < n_map; i++) {
        PointType p;
        p.x = map[4 * i]; p.y = map[4 * i + 1]; p.z = map[4 * i + 2]; p.intensity = map[4 * i + 3];
        (i < n_map / 2 ? first : rest).push_back(p);
    }
    ikdtree.Build(first);
    ikdtree.Add_Points(rest, false);
    PointVector queries(nq);
    for (int i = 0; i < nq; i++) { queries[i].x = qs[4 * i]; queries[i].y = qs[4 * i + 1]; queries[i].z = qs[4 * i + 2]; }
    std::vector<PointVector> pts;
    std::vector<std::vector<float>> d2;
    ikdtree.Nearest_Search_K_Batch(queries, k, pts, d2);
    PointVector flat;
    ikdtree.flatten(ikdtree.Root_Node, flat, NOT_RECORD);
    if (ikdtree.failed()) { fprintf(stderr, "a KD_TREE call failed: %s\n", KD_TREE<PointType>::last_error()); return 6; }

    FILE* fo = fopen(argv[2], "wb");
    if (!fo) { perror("out"); return 2; }
    fwrite(&at_construction, sizeof(int), 1, fo);
    for (const auto& v : pts) { const int n = (int)v.size(); fwrite(&n, sizeof(int), 1, fo); }
    for (const auto& v : pts)
        for (const auto& p : v) { const float o[4] = {p.x, p.y, p.z, p.intensity}; fwrite(o, sizeof(float), 4, fo); }
    const int nf = (int)flat.size();
    fwrite(&nf, sizeof(int), 1, fo);
    for (const auto& p : flat) { const float o[4] = {p.x, p.y, p.z, p.intensity}; fwrite(o, sizeof(float), 4, fo); }
    fclose(fo);
    printf("facade_deterministic ok: mode %d at construction, %d queries, %d points\n", at_construction, nq, nf);
    return 0;
}
