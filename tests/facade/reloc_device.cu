// A plain C/CUDA caller of the relocalisation: it cudaMallocs the scan and a prior, expands a grid of hypotheses around the prior
// with fl_reloc_expand_grid_device and runs fl_filter_relocalize_device on its own stream; then it captures both calls with
// cudaStreamBeginCapture and replays the graph from two priors, comparing every output with the uncaptured calls.  Input file:
// that of filter_device.cu (3 ints: map points, scan points, max_iter; one double R; the map and the scan as float32 x, y, z, i;
// x26, P and limit[23] as float64).  Prints "all equal" and exits 0 when every result matches.
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

struct Out {
    std::vector<double> x, P, hyp;
    std::vector<int> inl, st;
    std::vector<fl_reloc_row_t> rows;
};

static Out download(const double* dx, const double* dP, const double* dhyp, const int* dinl, const fl_reloc_row_t* drows, const int* dst,
                    int H, int keep, cudaStream_t st) {
    Out o;
    o.x.resize(26); o.P.resize(529); o.hyp.resize(26 * (size_t)H); o.inl.resize(H); o.st.resize(4); o.rows.resize(keep);
    CK(cudaMemcpyAsync(o.x.data(), dx, sizeof(double) * 26, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(o.P.data(), dP, sizeof(double) * 529, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(o.hyp.data(), dhyp, sizeof(double) * o.hyp.size(), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(o.inl.data(), dinl, sizeof(int) * H, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(o.st.data(), dst, sizeof(int) * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(o.rows.data(), drows, sizeof(fl_reloc_row_t) * keep, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return o;
}

static bool same(const Out& a, const Out& b) {
    return memcmp(a.x.data(), b.x.data(), sizeof(double) * 26) == 0 && memcmp(a.P.data(), b.P.data(), sizeof(double) * 529) == 0 &&
           memcmp(a.hyp.data(), b.hyp.data(), sizeof(double) * a.hyp.size()) == 0 && a.inl == b.inl && a.st == b.st &&
           memcmp(a.rows.data(), b.rows.data(), sizeof(fl_reloc_row_t) * a.rows.size()) == 0;
}

int main(int argc, char** argv) {
    if (argc < 2) { printf("usage: reloc_device in.bin\n"); return 1; }
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
    fl_filter_t* fr = nullptr;
    OK(fl_filter_create(&fr, m, nq));
    OK(fl_filter_set_params(fr, max_iter, limit.data(), 0));
    const fl_reloc_grid_t grid = {{5, 5, 1, 7}, {0.5, 0.5, 0.0, 0.05}};
    const int H = 5 * 5 * 7, keep = 8;
    const fl_reloc_params_t prm = {keep, 2, 0.3f, 10};
    OK(fl_filter_reserve_reloc(fr, nq, H, keep));

    float* dscan = nullptr;
    double *dprior = nullptr, *dP = nullptr, *dhyp = nullptr, *dx = nullptr, *dPo = nullptr;
    int *dinl = nullptr, *dst = nullptr;
    fl_reloc_row_t* drows = nullptr;
    CK(cudaMalloc(&dscan, sizeof(float) * scan.size()));
    CK(cudaMalloc(&dprior, sizeof(double) * 26));
    CK(cudaMalloc(&dP, sizeof(double) * 529));
    CK(cudaMalloc(&dhyp, sizeof(double) * 26 * H));
    CK(cudaMalloc(&dx, sizeof(double) * 26));
    CK(cudaMalloc(&dPo, sizeof(double) * 529));
    CK(cudaMalloc(&dinl, sizeof(int) * H));
    CK(cudaMalloc(&dst, sizeof(int) * 4));
    CK(cudaMalloc(&drows, sizeof(fl_reloc_row_t) * keep));
    CK(cudaMemcpyAsync(dscan, scan.data(), sizeof(float) * scan.size(), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(dP, P0.data(), sizeof(double) * 529, cudaMemcpyHostToDevice, st));

    // the prior of replay r: the file's, moved by r * (0.4, -0.3) m
    auto set_prior = [&](int r) {
        std::vector<double> x = x0;
        x[0] += 0.4 * r; x[1] -= 0.3 * r;
        CK(cudaMemcpyAsync(dprior, x.data(), sizeof(double) * 26, cudaMemcpyHostToDevice, st));
        CK(cudaMemsetAsync(dx, 0, sizeof(double) * 26, st));
        CK(cudaMemsetAsync(dPo, 0, sizeof(double) * 529, st));
    };
    auto calls = [&]() {
        OK(fl_reloc_expand_grid_device(dprior, &grid, dhyp, st));
        OK(fl_filter_relocalize_device(fr, dscan, nq, H, dhyp, dP, R, &prm, dx, dPo, dinl, drows, dst, st));
    };
    std::vector<Out> want;
    for (int r = 0; r < 2; r++) {
        set_prior(r);
        calls();
        want.push_back(download(dx, dPo, dhyp, dinl, drows, dst, H, keep, st));
        if (want.back().st[0] != FL_OK) { printf("no winner from prior %d\n", r); failures++; }
    }

    cudaGraph_t graph;
    cudaGraphExec_t exec;
    CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeGlobal));
    calls();
    CK(cudaStreamEndCapture(st, &graph));
    CK(cudaGraphInstantiate(&exec, graph, 0));
    for (int r : {1, 0, 1}) {
        set_prior(r);
        CK(cudaGraphLaunch(exec, st));
        expect(same(download(dx, dPo, dhyp, dinl, drows, dst, H, keep, st), want[r]), r ? "graph replay from prior 1" : "graph replay from prior 0");
    }
    CK(cudaGraphExecDestroy(exec));
    CK(cudaGraphDestroy(graph));

    CK(cudaFree(dscan)); CK(cudaFree(dprior)); CK(cudaFree(dP)); CK(cudaFree(dhyp)); CK(cudaFree(dx)); CK(cudaFree(dPo));
    CK(cudaFree(dinl)); CK(cudaFree(dst)); CK(cudaFree(drows));
    fl_filter_destroy(fr);
    fl_map_destroy(m);
    CK(cudaStreamDestroy(st));
    if (failures) { printf("%d mismatches\n", failures); return 4; }
    printf("all equal\n");
    return 0;
}
