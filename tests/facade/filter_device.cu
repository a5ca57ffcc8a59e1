// A plain C/CUDA caller of the device-buffer update: it cudaMallocs the scan, the state, the covariance and the status, runs
// fl_filter_update_device on its own stream, then captures the update into a CUDA graph and replays it from two priors, and
// compares every result with fl_filter_update on the same inputs.  Input file: 3 ints (map points, scan points, max_iter),
// one double (R), the map and the scan (x, y, z, i) as float32, then x26, P (23 x 23) and limit[23] as float64.  Prints
// "all equal" and exits 0 when every result matches.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "fastlio_b200.h"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(2); } } while (0)
#define OK(x) do { int r_ = (x); if (r_ < 0) { printf("%s: %d %s\n", #x, r_, fl_last_error()); exit(3); } } while (0)

static int failures = 0;
static void expect(bool ok, const char* what) { if (!ok) { printf("MISMATCH: %s\n", what); failures++; } }

// the device result (x, P, status) against fl_filter_update from the same prior on a second filter
static void check(fl_filter_t* ref, const std::vector<float>& scan, int nq, const std::vector<double>& x0, const std::vector<double>& P0,
                  double R, const double* dx, const double* dP, const int* ds, cudaStream_t st, const char* what) {
    std::vector<double> xh(x0), Ph(P0);
    OK(fl_filter_update(ref, scan.data(), nq, xh.data(), Ph.data(), R, nullptr));
    int n_pass = 0;
    OK(fl_filter_download_state(ref, nullptr, nullptr, &n_pass));
    std::vector<double> xd(26), Pd(23 * 23);
    int sd[2] = {-1, -1};
    CK(cudaMemcpyAsync(xd.data(), dx, sizeof(double) * 26, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(Pd.data(), dP, sizeof(double) * 23 * 23, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(sd, ds, sizeof(sd), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    expect(memcmp(xd.data(), xh.data(), sizeof(double) * 26) == 0 && memcmp(Pd.data(), Ph.data(), sizeof(double) * 23 * 23) == 0, what);
    expect(sd[0] == FL_OK && sd[1] == n_pass, what);
}

int main(int argc, char** argv) {
    if (argc < 2) { printf("usage: filter_device in.bin\n"); return 1; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { printf("cannot open %s\n", argv[1]); return 1; }
    int hdr[3];
    double R = 0.0;
    if (fread(hdr, sizeof(int), 3, f) != 3 || fread(&R, sizeof(double), 1, f) != 1) return 1;
    const int n = hdr[0], nq = hdr[1], max_iter = hdr[2];
    std::vector<float> map(4 * (size_t)n), scan(4 * (size_t)nq);
    std::vector<double> x0(26), P0(23 * 23), limit(23);
    if (fread(map.data(), sizeof(float), map.size(), f) != map.size() || fread(scan.data(), sizeof(float), scan.size(), f) != scan.size() ||
        fread(x0.data(), sizeof(double), 26, f) != 26 || fread(P0.data(), sizeof(double), P0.size(), f) != P0.size() ||
        fread(limit.data(), sizeof(double), 23, f) != 23)
        return 1;
    fclose(f);

    cudaStream_t st;
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    fl_map_t* m = nullptr;
    OK(fl_map_create(&m, 0, 0.5f));
    OK(fl_map_build(m, map.data(), n));
    fl_filter_t *fd = nullptr, *fh = nullptr;
    OK(fl_filter_create(&fd, m, nq));
    OK(fl_filter_create(&fh, m, nq));
    OK(fl_filter_set_params(fd, max_iter, limit.data(), 0));
    OK(fl_filter_set_params(fh, max_iter, limit.data(), 0));

    float* dscan = nullptr; double *dx = nullptr, *dP = nullptr; int* ds = nullptr;
    CK(cudaMalloc(&dscan, sizeof(float) * scan.size()));
    CK(cudaMalloc(&dx, sizeof(double) * 26));
    CK(cudaMalloc(&dP, sizeof(double) * 23 * 23));
    CK(cudaMalloc(&ds, sizeof(int) * 2));
    CK(cudaMemcpyAsync(dscan, scan.data(), sizeof(float) * scan.size(), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(dx, x0.data(), sizeof(double) * 26, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(dP, P0.data(), sizeof(double) * 23 * 23, cudaMemcpyHostToDevice, st));

    // one update on the program's own stream
    OK(fl_filter_update_device(fd, dscan, nq, dx, dP, R, ds, st));
    check(fh, scan, nq, x0, P0, R, dx, dP, ds, st, "update on the caller's stream");

    // the same update captured once and replayed from two priors
    cudaGraph_t graph;
    cudaGraphExec_t exec;
    CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeGlobal));
    OK(fl_filter_update_device(fd, dscan, nq, dx, dP, R, ds, st));
    CK(cudaStreamEndCapture(st, &graph));
    CK(cudaGraphInstantiate(&exec, graph, 0));
    for (int rep = 0; rep < 2; rep++) {
        std::vector<double> xr(x0), Pr(P0);
        xr[0] += 0.03 * (rep + 1); xr[2] -= 0.02 * rep;
        for (double& v : Pr) v *= 1.0 + 0.5 * rep;
        CK(cudaMemcpyAsync(dx, xr.data(), sizeof(double) * 26, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(dP, Pr.data(), sizeof(double) * 23 * 23, cudaMemcpyHostToDevice, st));
        CK(cudaGraphLaunch(exec, st));
        check(fh, scan, nq, xr, Pr, R, dx, dP, ds, st, rep == 0 ? "graph replay 1" : "graph replay 2");
    }
    CK(cudaGraphExecDestroy(exec));
    CK(cudaGraphDestroy(graph));

    CK(cudaFree(dscan)); CK(cudaFree(dx)); CK(cudaFree(dP)); CK(cudaFree(ds));
    fl_filter_destroy(fd);
    fl_filter_destroy(fh);
    fl_map_destroy(m);
    CK(cudaStreamDestroy(st));
    if (failures) { printf("%d mismatches\n", failures); return 4; }
    printf("all equal\n");
    return 0;
}
