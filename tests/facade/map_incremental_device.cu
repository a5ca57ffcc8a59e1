// A plain C/CUDA caller of the whole scan on the device: it cudaMallocs the scan, the state, the covariance and the status words,
// runs fl_filter_update_device + fl_filter_map_incremental_device once on its own stream, captures the two into a CUDA graph and
// replays the graph over the remaining scans (each copied into the captured scan buffer), and compares every scan with
// fl_filter_update + fl_filter_map_incremental on a twin map and filter: x, P, the three counts, validnum, and at the end, after
// fl_map_maintain, the point sets.  Input file: 4 ints (map points, points per scan, scans, max_iter), one double (R), the map
// and the scans (x, y, z, i) as float32, then x26, P (23 x 23) and limit[23] as float64.  Prints "all equal" and exits 0 when
// every result matches.
#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "fastlio_b200.h"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(2); } } while (0)
#define OK(x) do { int r_ = (x); if (r_ < 0) { printf("%s: %d %s\n", #x, r_, fl_last_error()); exit(3); } } while (0)

static int failures = 0;
static void expect(bool ok, const char* what, int scan) { if (!ok) { printf("MISMATCH: %s (scan %d)\n", what, scan); failures++; } }

static std::vector<std::array<unsigned, 4>> sorted_points(fl_map_t* m) {
    const int n = fl_map_validnum(m);
    std::vector<std::array<unsigned, 4>> rows((size_t)std::max(n, 1));
    OK(fl_map_flatten(m, reinterpret_cast<float*>(rows.data()), n));
    rows.resize((size_t)n);
    std::sort(rows.begin(), rows.end());
    return rows;
}

int main(int argc, char** argv) {
    if (argc < 2) { printf("usage: map_incremental_device in.bin\n"); return 1; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { printf("cannot open %s\n", argv[1]); return 1; }
    int hdr[4];
    double R = 0.0;
    if (fread(hdr, sizeof(int), 4, f) != 4 || fread(&R, sizeof(double), 1, f) != 1) return 1;
    const int n = hdr[0], nq = hdr[1], n_scans = hdr[2], max_iter = hdr[3];
    std::vector<float> map(4 * (size_t)n), scans(4 * (size_t)nq * n_scans);
    std::vector<double> x0(26), P0(23 * 23), limit(23);
    if (fread(map.data(), sizeof(float), map.size(), f) != map.size() || fread(scans.data(), sizeof(float), scans.size(), f) != scans.size() ||
        fread(x0.data(), sizeof(double), 26, f) != 26 || fread(P0.data(), sizeof(double), P0.size(), f) != P0.size() ||
        fread(limit.data(), sizeof(double), 23, f) != 23)
        return 1;
    fclose(f);

    cudaStream_t st;
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    fl_map_t *md = nullptr, *mh = nullptr;
    OK(fl_map_create(&md, 0, 0.5f));
    OK(fl_map_create(&mh, 0, 0.5f));
    OK(fl_map_build(md, map.data(), n));
    OK(fl_map_build(mh, map.data(), n));
    fl_filter_t *fd = nullptr, *fh = nullptr;
    OK(fl_filter_create(&fd, md, nq));
    OK(fl_filter_create(&fh, mh, nq));
    OK(fl_filter_set_params(fd, max_iter, limit.data(), 0));
    OK(fl_filter_set_params(fh, max_iter, limit.data(), 0));

    float* d_scan = nullptr;
    double *d_x = nullptr, *d_P = nullptr;
    int *d_status = nullptr, *d_out4 = nullptr;
    CK(cudaMalloc(&d_scan, sizeof(float) * 4 * (size_t)nq));
    CK(cudaMalloc(&d_x, sizeof(double) * 26));
    CK(cudaMalloc(&d_P, sizeof(double) * 23 * 23));
    CK(cudaMalloc(&d_status, sizeof(int) * 2));
    CK(cudaMalloc(&d_out4, sizeof(int) * 4));
    CK(cudaMemcpyAsync(d_x, x0.data(), sizeof(double) * 26, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_P, P0.data(), sizeof(double) * 23 * 23, cudaMemcpyHostToDevice, st));
    std::vector<double> xh(x0), Ph(P0);

    cudaGraphExec_t exec = nullptr;
    for (int s = 0; s < n_scans; s++) {
        const float* scan = scans.data() + 4 * (size_t)nq * s;
        CK(cudaMemcpyAsync(d_scan, scan, sizeof(float) * 4 * (size_t)nq, cudaMemcpyHostToDevice, st));
        if (s == 0) {                        // once outside capture, then capture the pair
            OK(fl_filter_update_device(fd, d_scan, nq, d_x, d_P, R, d_status, st));
            OK(fl_filter_map_incremental_device(fd, 0.5, 1, d_out4, st));
            CK(cudaStreamSynchronize(st));
            cudaGraph_t g;
            CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeGlobal));
            OK(fl_filter_update_device(fd, d_scan, nq, d_x, d_P, R, d_status, st));
            OK(fl_filter_map_incremental_device(fd, 0.5, 1, d_out4, st));
            CK(cudaStreamEndCapture(st, &g));
            CK(cudaGraphInstantiate(&exec, g, 0));
            CK(cudaGraphDestroy(g));
        } else {
            CK(cudaGraphLaunch(exec, st));
        }
        OK(fl_filter_update(fh, scan, nq, xh.data(), Ph.data(), R, nullptr));
        int out3[3] = {0, 0, 0};
        OK(fl_filter_map_incremental(fh, 0.5, 1, out3));
        std::vector<double> xd(26), Pd(23 * 23);
        int sd[2] = {-1, -1}, o4[4] = {-1, -1, -1, -1};
        CK(cudaMemcpyAsync(xd.data(), d_x, sizeof(double) * 26, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(Pd.data(), d_P, sizeof(double) * 23 * 23, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(sd, d_status, sizeof(sd), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(o4, d_out4, sizeof(o4), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        expect(memcmp(xd.data(), xh.data(), sizeof(double) * 26) == 0 && memcmp(Pd.data(), Ph.data(), sizeof(double) * 23 * 23) == 0, "x, P", s);
        expect(sd[0] == FL_OK, "update status", s);
        expect(o4[0] == out3[0] && o4[1] == out3[1] && o4[2] == out3[2], "map_incremental counts", s);
        expect(o4[3] == FL_OK || o4[3] == 1, "map_incremental status", s);
        expect(fl_map_validnum(md) == fl_map_validnum(mh), "validnum", s);      // a read-only host call between two replays
    }
    int changed = 0;
    OK(fl_map_maintain(md, &changed));
    expect(sorted_points(md) == sorted_points(mh), "point sets", n_scans);
    CK(cudaGraphExecDestroy(exec));
    CK(cudaFree(d_scan)); CK(cudaFree(d_x)); CK(cudaFree(d_P)); CK(cudaFree(d_status)); CK(cudaFree(d_out4));
    OK(fl_filter_destroy(fd)); OK(fl_filter_destroy(fh));
    OK(fl_map_destroy(md)); OK(fl_map_destroy(mh));
    CK(cudaStreamDestroy(st));
    if (failures) { printf("%d mismatches\n", failures); return 4; }
    printf("all equal\n");
    return 0;
}
