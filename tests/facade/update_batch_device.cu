// A plain C/CUDA caller of the batched update: it cudaMallocs the scan and H priors, runs fl_filter_update_batch_device on its
// own stream, then captures the call with cudaStreamBeginCapture and replays it from a second set of priors, and compares every
// hypothesis with fl_filter_update_device from the same prior on a second filter.  Input file: that of filter_device.cu (3 ints:
// map points, scan points, max_iter; one double R; the map and the scan as float32 x, y, z, i; x26, P and limit[23] as float64).
// The priors are the file's, shifted by a few centimetres and scaled.  Prints "all equal" and exits 0 when every result matches.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "fastlio_b200.h"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(2); } } while (0)
#define OK(x) do { int r_ = (x); if (r_ < 0) { printf("%s: %d %s\n", #x, r_, fl_last_error()); exit(3); } } while (0)

static int failures = 0;
static void expect(bool ok, const char* what, int h) { if (!ok) { printf("MISMATCH: %s, hypothesis %d\n", what, h); failures++; } }

static void make_priors(const std::vector<double>& x0, const std::vector<double>& P0, int H, int set, std::vector<double>& X, std::vector<double>& P) {
    X.resize(26 * (size_t)H); P.resize(529 * (size_t)H);
    for (int h = 0; h < H; h++) {
        for (int i = 0; i < 26; i++) X[26 * (size_t)h + i] = x0[i];
        X[26 * (size_t)h + 0] += 0.01 * ((h * 7 + set) % 11 - 5);
        X[26 * (size_t)h + 1] -= 0.008 * ((h * 3 + 2 * set) % 7 - 3);
        for (int i = 0; i < 529; i++) P[529 * (size_t)h + i] = P0[i] * (1.0 + 0.1 * ((h + set) % 4));
    }
}

// every hypothesis of the batch result in (dx, dP, ds) against fl_filter_update_device on `ref` from the same prior
static void check(fl_filter_t* ref, const float* dscan, int nq, int H, const std::vector<double>& X, const std::vector<double>& P, double R,
                  const double* dx, const double* dP, const int* ds, cudaStream_t st, const char* what) {
    std::vector<double> xb(26 * (size_t)H), Pb(529 * (size_t)H);
    std::vector<int> sb(2 * (size_t)H);
    CK(cudaMemcpyAsync(xb.data(), dx, sizeof(double) * xb.size(), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(Pb.data(), dP, sizeof(double) * Pb.size(), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(sb.data(), ds, sizeof(int) * sb.size(), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    double *rx = nullptr, *rP = nullptr; int* rs = nullptr;
    CK(cudaMalloc(&rx, sizeof(double) * 26)); CK(cudaMalloc(&rP, sizeof(double) * 529)); CK(cudaMalloc(&rs, sizeof(int) * 2));
    for (int h = 0; h < H; h++) {
        CK(cudaMemcpyAsync(rx, &X[26 * (size_t)h], sizeof(double) * 26, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(rP, &P[529 * (size_t)h], sizeof(double) * 529, cudaMemcpyHostToDevice, st));
        OK(fl_filter_update_device(ref, dscan, nq, rx, rP, R, rs, st));
        double xh[26], Ph[529]; int sh[2];
        CK(cudaMemcpyAsync(xh, rx, sizeof(xh), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(Ph, rP, sizeof(Ph), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(sh, rs, sizeof(sh), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        expect(memcmp(xh, &xb[26 * (size_t)h], sizeof(xh)) == 0 && memcmp(Ph, &Pb[529 * (size_t)h], sizeof(Ph)) == 0, what, h);
        expect(sh[0] == FL_OK && sh[0] == sb[2 * h] && sh[1] == sb[2 * h + 1], what, h);
    }
    CK(cudaFree(rx)); CK(cudaFree(rP)); CK(cudaFree(rs));
}

int main(int argc, char** argv) {
    if (argc < 2) { printf("usage: update_batch_device in.bin\n"); return 1; }
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
    fl_filter_t *fb = nullptr, *fh = nullptr;
    OK(fl_filter_create(&fb, m, nq));
    OK(fl_filter_create(&fh, m, nq));
    OK(fl_filter_set_params(fb, max_iter, limit.data(), 0));
    OK(fl_filter_set_params(fh, max_iter, limit.data(), 0));
    OK(fl_filter_reserve_batch(fb, nq));
    int plan[3];
    OK(fl_filter_batch_plan(fb, nq, 1, plan));
    const int H = plan[1] + 3;                        // two waves
    OK(fl_filter_batch_plan(fb, nq, H, plan));
    if (plan[2] != 2) { printf("expected two waves, plan (%d, %d, %d)\n", plan[0], plan[1], plan[2]); return 5; }

    float* dscan = nullptr; double *dx = nullptr, *dP = nullptr; int* ds = nullptr;
    CK(cudaMalloc(&dscan, sizeof(float) * scan.size()));
    CK(cudaMalloc(&dx, sizeof(double) * 26 * H));
    CK(cudaMalloc(&dP, sizeof(double) * 529 * H));
    CK(cudaMalloc(&ds, sizeof(int) * 2 * H));
    CK(cudaMemcpyAsync(dscan, scan.data(), sizeof(float) * scan.size(), cudaMemcpyHostToDevice, st));
    std::vector<double> X, P;

    // one batch on the program's own stream
    make_priors(x0, P0, H, 0, X, P);
    CK(cudaMemcpyAsync(dx, X.data(), sizeof(double) * X.size(), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(dP, P.data(), sizeof(double) * P.size(), cudaMemcpyHostToDevice, st));
    OK(fl_filter_update_batch_device(fb, dscan, nq, H, dx, dP, R, ds, nullptr, st));
    check(fh, dscan, nq, H, X, P, R, dx, dP, ds, st, "batch on the caller's stream");

    // the batch captured once and replayed from two more sets of priors
    cudaGraph_t graph;
    cudaGraphExec_t exec;
    CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeGlobal));
    OK(fl_filter_update_batch_device(fb, dscan, nq, H, dx, dP, R, ds, nullptr, st));
    CK(cudaStreamEndCapture(st, &graph));
    CK(cudaGraphInstantiate(&exec, graph, 0));
    for (int rep = 1; rep <= 2; rep++) {
        make_priors(x0, P0, H, rep, X, P);
        CK(cudaMemcpyAsync(dx, X.data(), sizeof(double) * X.size(), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(dP, P.data(), sizeof(double) * P.size(), cudaMemcpyHostToDevice, st));
        CK(cudaGraphLaunch(exec, st));
        check(fh, dscan, nq, H, X, P, R, dx, dP, ds, st, rep == 1 ? "graph replay 1" : "graph replay 2");
    }
    CK(cudaGraphExecDestroy(exec));
    CK(cudaGraphDestroy(graph));

    CK(cudaFree(dscan)); CK(cudaFree(dx)); CK(cudaFree(dP)); CK(cudaFree(ds));
    fl_filter_destroy(fb);
    fl_filter_destroy(fh);
    fl_map_destroy(m);
    CK(cudaStreamDestroy(st));
    if (failures) { printf("%d mismatches\n", failures); return 4; }
    printf("all equal\n");
    return 0;
}
