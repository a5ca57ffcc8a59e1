// A plain C/CUDA caller of the device-buffer map queries: it cudaMallocs its buffers, enqueues the device entries on its own
// stream, and compares their answers with the host entries on the same map.  Input file: 4 ints (map points, kNN queries,
// boxes, spheres), then the map (x, y, z, i), the kNN queries (x, y, z, i), the boxes (min xyz, max xyz), the spheres
// (x, y, z, r), all float32.  Prints "all equal" and exits 0 when every answer matches.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "fastlio_b200.h"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(2); } } while (0)
#define OK(x) do { int r_ = (x); if (r_ < 0) { printf("%s: %d %s\n", #x, r_, fl_last_error()); exit(3); } } while (0)

static int failures = 0;
static void expect(bool ok, const char* what) { if (!ok) { printf("MISMATCH: %s\n", what); failures++; } }

template <class T> static T* to_device(const std::vector<T>& h) {
    T* d = nullptr;
    CK(cudaMalloc(&d, sizeof(T) * (h.size() ? h.size() : 1)));
    if (!h.empty()) CK(cudaMemcpy(d, h.data(), sizeof(T) * h.size(), cudaMemcpyHostToDevice));
    return d;
}
template <class T> static std::vector<T> to_host(const T* d, size_t n, cudaStream_t st) {
    std::vector<T> h(n);
    if (n) CK(cudaMemcpyAsync(h.data(), d, sizeof(T) * n, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return h;
}

static void range(fl_map_t* m, bool radius, const std::vector<float>& q, int nq, cudaStream_t st) {
    std::vector<int> off_h(nq + 1);
    int total = radius ? fl_map_radius_search(m, q.data(), nq, off_h.data(), nullptr, 0) : fl_map_box_search(m, q.data(), nq, off_h.data(), nullptr, 0);
    OK(total);
    std::vector<float> pts_h(4 * (size_t)total + 4);
    OK(radius ? fl_map_radius_search(m, q.data(), nq, off_h.data(), pts_h.data(), total) : fl_map_box_search(m, q.data(), nq, off_h.data(), pts_h.data(), total));
    float* dq = to_device(q);
    int* doff = nullptr; float* dpts = nullptr; long long* dst = nullptr; void* ws = nullptr;
    CK(cudaMalloc(&doff, sizeof(int) * (nq + 1)));
    CK(cudaMalloc(&dpts, sizeof(float) * 4 * ((size_t)total + 1)));
    CK(cudaMalloc(&dst, 2 * sizeof(long long)));
    unsigned long long wb = 0;
    OK(fl_map_range_workspace_bytes(m, nq, 16, &wb));          // deliberately small: the first call reports the pairs needed
    CK(cudaMalloc(&ws, wb));
    OK(radius ? fl_map_radius_search_device(m, dq, nq, doff, dpts, total, ws, wb, dst, st) : fl_map_box_search_device(m, dq, nq, doff, dpts, total, ws, wb, dst, st));
    std::vector<long long> s = to_host(dst, 2, st);
    if (s[0] == -1) {
        CK(cudaFree(ws));
        OK(fl_map_range_workspace_bytes(m, nq, s[1], &wb));
        CK(cudaMalloc(&ws, wb));
        OK(radius ? fl_map_radius_search_device(m, dq, nq, doff, dpts, total, ws, wb, dst, st) : fl_map_box_search_device(m, dq, nq, doff, dpts, total, ws, wb, dst, st));
        s = to_host(dst, 2, st);
    }
    expect(s[0] == total, radius ? "radius total" : "box total");
    std::vector<int> off_d = to_host(doff, nq + 1, st);
    std::vector<float> pts_d = to_host(dpts, 4 * (size_t)total, st);
    expect(off_d == off_h, radius ? "radius offsets" : "box offsets");
    expect(memcmp(pts_d.data(), pts_h.data(), sizeof(float) * 4 * (size_t)total) == 0, radius ? "radius points" : "box points");
    CK(cudaFree(dq)); CK(cudaFree(doff)); CK(cudaFree(dpts)); CK(cudaFree(dst)); CK(cudaFree(ws));
}

int main(int argc, char** argv) {
    if (argc < 2) { printf("usage: device_queries in.bin\n"); return 1; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { printf("cannot open %s\n", argv[1]); return 1; }
    int hdr[4];
    if (fread(hdr, sizeof(int), 4, f) != 4) return 1;
    const int n = hdr[0], nq = hdr[1], nb = hdr[2], ns = hdr[3];
    std::vector<float> map(4 * (size_t)n), q(4 * (size_t)nq), boxes(6 * (size_t)nb), spheres(4 * (size_t)ns);
    if (fread(map.data(), sizeof(float), map.size(), f) != map.size() || fread(q.data(), sizeof(float), q.size(), f) != q.size() ||
        fread(boxes.data(), sizeof(float), boxes.size(), f) != boxes.size() || fread(spheres.data(), sizeof(float), spheres.size(), f) != spheres.size())
        return 1;
    fclose(f);

    cudaStream_t st;
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    fl_map_t* m = nullptr;
    OK(fl_map_create(&m, 0, 0.5f));
    float* dmap = to_device(map);
    OK(fl_map_build_device(m, dmap, n, st));

    float* dq = to_device(q);
    const int ks[] = {1, 5, 8, 32};
    const float mds[] = {INFINITY, 1.0f};
    float *dp = nullptr, *dd = nullptr; int* dc = nullptr;
    CK(cudaMalloc(&dp, sizeof(float) * 4 * 32 * (size_t)nq));
    CK(cudaMalloc(&dd, sizeof(float) * 32 * (size_t)nq));
    CK(cudaMalloc(&dc, sizeof(int) * (size_t)nq));
    for (int k : ks) {
        for (float md : mds) {
            std::vector<float> hp(4 * (size_t)k * nq), hd((size_t)k * nq);
            std::vector<int> hc(nq);
            OK(fl_map_nearest_search(m, q.data(), nq, k, md, hp.data(), hd.data(), hc.data()));
            OK(fl_map_nearest_search_device(m, dq, nq, k, md, dp, dd, dc, st));
            std::vector<float> gp = to_host(dp, hp.size(), st), gd = to_host(dd, hd.size(), st);
            std::vector<int> gc = to_host(dc, hc.size(), st);
            expect(memcmp(gp.data(), hp.data(), sizeof(float) * hp.size()) == 0 && memcmp(gd.data(), hd.data(), sizeof(float) * hd.size()) == 0 &&
                   gc == hc, "nearest search");
        }
    }
    range(m, false, boxes, nb, st);
    range(m, true, spheres, ns, st);

    // Add_Points from device memory, then the map equals one mutated from the host
    fl_map_t* h = nullptr;
    OK(fl_map_create(&h, 0, 0.5f));
    OK(fl_map_build(h, map.data(), n));
    std::vector<float> add(q.begin(), q.begin() + 4 * (size_t)(nq / 2));
    for (size_t i = 0; i < add.size(); i++) if (!std::isfinite(add[i])) add[i] = 0.f;
    float* dadd = to_device(add);
    const int ra = fl_map_add_points_device(m, dadd, nq / 2, 1, st), rb = fl_map_add_points(h, add.data(), nq / 2, 1);
    expect(ra == rb && ra >= 0, "add_points return value");
    expect(fl_map_validnum(m) == fl_map_validnum(h), "validnum after add_points");

    CK(cudaFree(dmap)); CK(cudaFree(dq)); CK(cudaFree(dp)); CK(cudaFree(dd)); CK(cudaFree(dc)); CK(cudaFree(dadd));
    fl_map_destroy(m);
    fl_map_destroy(h);
    CK(cudaStreamDestroy(st));
    if (failures) { printf("%d mismatches\n", failures); return 4; }
    printf("all equal\n");
    return 0;
}
