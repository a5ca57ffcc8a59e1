// EXECUTES the range queries of the KD_TREE<PointType> facade on a GPU (tests/test_gpu_range_search.py builds and runs it):
// Box_Search / Radius_Search one query per call, then Box_Search_Batch / Radius_Search_Batch over all of them.
//   usage: facade_range <in.bin> <out.bin>
//   in : int32 n_map, nb, nq; float32 map[n_map*4], boxes[nb*6], spheres[nq*4] (x, y, z, radius)
//   out: four result sets (Box_Search, Radius_Search, Box_Search_Batch, Radius_Search_Batch), each
//        int32 counts[n] followed by float32 points[sum(counts)*4] (x, y, z, intensity), query after query
#include <ikd-Tree/ikd_Tree.h>

#include <cstdio>
#include <vector>

typedef pcl::PointXYZINormal PointType;
typedef KD_TREE<PointType>::PointVector PointVector;

template <class T> static bool rd(FILE* f, T* p, size_t n) { return fread(p, sizeof(T), n, f) == n; }

static void write_set(FILE* f, const std::vector<PointVector>& res) {
    for (const auto& v : res) { const int n = (int)v.size(); fwrite(&n, sizeof(int), 1, f); }
    for (const auto& v : res)
        for (const auto& p : v) { const float o[4] = {p.x, p.y, p.z, p.intensity}; fwrite(o, sizeof(float), 4, f); }
}

int main(int argc, char** argv) {
    if (argc < 3) { fprintf(stderr, "usage: facade_range in out\n"); return 2; }
    FILE* fi = fopen(argv[1], "rb");
    if (!fi) { perror("in"); return 2; }
    int hdr[3];
    if (!rd(fi, hdr, 3)) return 2;
    const int n_map = hdr[0], nb = hdr[1], nq = hdr[2];
    std::vector<float> map((size_t)n_map * 4), boxes((size_t)nb * 6), spheres((size_t)nq * 4);
    if (!rd(fi, map.data(), map.size()) || !rd(fi, boxes.data(), boxes.size()) || !rd(fi, spheres.data(), spheres.size())) return 2;
    fclose(fi);

    KD_TREE<PointType> ikdtree(0.5f, 0.6f, 0.5f);
    if (!ikdtree.ok()) { fprintf(stderr, "no device map: %s\n", KD_TREE<PointType>::last_error()); return 3; }
    PointVector cloud(n_map);
    for (int i = 0; i < n_map; i++) { cloud[i].x = map[4 * i]; cloud[i].y = map[4 * i + 1]; cloud[i].z = map[4 * i + 2]; cloud[i].intensity = map[4 * i + 3]; }
    ikdtree.Build(cloud);

    std::vector<BoxPointType> bv(nb);
    for (int i = 0; i < nb; i++)
        for (int a = 0; a < 3; a++) { bv[i].vertex_min[a] = boxes[6 * i + a]; bv[i].vertex_max[a] = boxes[6 * i + 3 + a]; }
    PointVector centers(nq);
    std::vector<float> radii(nq);
    for (int i = 0; i < nq; i++) { centers[i].x = spheres[4 * i]; centers[i].y = spheres[4 * i + 1]; centers[i].z = spheres[4 * i + 2]; radii[i] = spheres[4 * i + 3]; }

    std::vector<PointVector> box_one(nb), rad_one(nq), box_batch, rad_batch;
    for (int i = 0; i < nb; i++) {
        box_one[i].push_back(PointType());            // Box_Search replaces what Storage held
        ikdtree.Box_Search(bv[i], box_one[i]);
    }
    for (int i = 0; i < nq; i++) ikdtree.Radius_Search(centers[i], radii[i], rad_one[i]);
    ikdtree.Box_Search_Batch(bv, box_batch);
    ikdtree.Radius_Search_Batch(centers, radii, rad_batch);
    if (ikdtree.failed()) { fprintf(stderr, "a KD_TREE call failed: %s\n", KD_TREE<PointType>::last_error()); return 6; }

    FILE* fo = fopen(argv[2], "wb");
    if (!fo) { perror("out"); return 2; }
    write_set(fo, box_one); write_set(fo, rad_one); write_set(fo, box_batch); write_set(fo, rad_batch);
    fclose(fo);
    printf("facade_range ok: %d boxes, %d spheres\n", nb, nq);
    return 0;
}
