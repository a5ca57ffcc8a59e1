// A plain C/CUDA caller of the batched scan front end: a fleet of robots on one shared map.  One fl_scan_batch_run_device de-skews
// and down-samples every robot's raw scan, and one fl_filter_update_scans_device then updates every robot from its own state with
// the batch's fl_scan_batch_get_refs table.  Both calls are captured into one graph with cudaStreamBeginCapture on the program's
// stream and replayed once per step, each robot's x and P chained from step to step.  A second filter runs the same steps robot by
// robot with fl_filter_update_scan_device on single front ends (fl_scan_t), and the states and statuses must match byte for byte.
// Input file: the layout of update_scans_device.cu.  Prints "all equal" and exits 0 when every state matches.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "fastlio_b200.h"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(2); } } while (0)
#define OK(x) do { int r_ = (x); if (r_ < 0) { printf("%s: %d %s\n", #x, r_, fl_last_error()); exit(3); } } while (0)

struct Raw {
    std::vector<float> xyzi, t_ms;
    std::vector<double> poses, x_end;
};

int main(int argc, char** argv) {
    if (argc < 2) { printf("usage: scan_batch_device in.bin\n"); return 1; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { printf("cannot open %s\n", argv[1]); return 1; }
    int hdr[6];
    double R = 0.0;
    if (fread(hdr, sizeof(int), 6, f) != 6 || fread(&R, sizeof(double), 1, f) != 1) return 1;
    const int n_map = hdr[0], robots = hdr[1], steps = hdr[2], n_raw = hdr[3], n_pose = hdr[4], max_iter = hdr[5];
    std::vector<float> map(4 * (size_t)n_map);
    std::vector<double> x0(26 * (size_t)robots), P0(529);
    if (fread(map.data(), sizeof(float), map.size(), f) != map.size() || fread(x0.data(), sizeof(double), x0.size(), f) != x0.size() ||
        fread(P0.data(), sizeof(double), 529, f) != 529)
        return 1;
    std::vector<Raw> raw((size_t)robots * steps);
    for (Raw& r : raw) {
        r.xyzi.resize(4 * (size_t)n_raw); r.t_ms.resize(n_raw); r.poses.resize(22 * (size_t)n_pose); r.x_end.resize(26);
        if (fread(r.xyzi.data(), sizeof(float), r.xyzi.size(), f) != r.xyzi.size() || fread(r.t_ms.data(), sizeof(float), n_raw, f) != (size_t)n_raw ||
            fread(r.poses.data(), sizeof(double), r.poses.size(), f) != r.poses.size() || fread(r.x_end.data(), sizeof(double), 26, f) != 26)
            return 1;
    }
    fclose(f);
    const float leaf = 0.5f;

    cudaStream_t st;
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    fl_map_t* m = nullptr;
    OK(fl_map_create(&m, 0, 0.5f));
    OK(fl_map_build(m, map.data(), n_map));
    fl_filter_t *fg = nullptr, *ft = nullptr;
    OK(fl_filter_create(&fg, m, n_raw));
    OK(fl_filter_create(&ft, m, n_raw));
    OK(fl_filter_set_params(fg, max_iter, nullptr, 0));
    OK(fl_filter_set_params(ft, max_iter, nullptr, 0));
    OK(fl_filter_reserve_batch(fg, n_raw));

    // the fleet's batch and the twins' front ends; the batch's table of down-sampled clouds
    fl_scan_batch_t* batch = nullptr;
    OK(fl_scan_batch_create(&batch, m));
    OK(fl_scan_batch_reserve(batch, robots, n_raw, n_pose));
    const fl_scan_ref_t* dref = nullptr;
    int n_max = 0;
    OK(fl_scan_batch_get_refs(batch, 1, &dref, &n_max));
    if (n_max != n_raw) { printf("fl_scan_batch_get_refs: n_max %d, expected %d\n", n_max, n_raw); return 5; }
    std::vector<fl_scan_t*> twins(robots);
    for (int r = 0; r < robots; r++) { OK(fl_scan_create(&twins[r], m)); OK(fl_scan_reserve(twins[r], n_raw, n_pose)); }
    fl_scan_raw_t* draw = nullptr;
    float *dxyzi = nullptr, *dtms = nullptr; double *dposes = nullptr, *dxend = nullptr, *dx = nullptr, *dP = nullptr;
    int *dn = nullptr, *dnp = nullptr, *ds = nullptr, *dbs = nullptr;
    CK(cudaMalloc(&draw, sizeof(fl_scan_raw_t) * robots));
    CK(cudaMalloc(&dbs, sizeof(int) * 2 * robots));
    CK(cudaMalloc(&dxyzi, sizeof(float) * 4 * (size_t)n_raw * robots));
    CK(cudaMalloc(&dtms, sizeof(float) * (size_t)n_raw * robots));
    CK(cudaMalloc(&dposes, sizeof(double) * 22 * (size_t)n_pose * robots));
    CK(cudaMalloc(&dxend, sizeof(double) * 26 * robots));
    CK(cudaMalloc(&dx, sizeof(double) * 26 * robots));
    CK(cudaMalloc(&dP, sizeof(double) * 529 * robots));
    CK(cudaMalloc(&dn, sizeof(int) * robots));
    CK(cudaMalloc(&dnp, sizeof(int) * robots));
    CK(cudaMalloc(&ds, sizeof(int) * 2 * robots));
    std::vector<int> counts(robots, n_raw), pcounts(robots, n_pose);
    CK(cudaMemcpy(dn, counts.data(), sizeof(int) * robots, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dnp, pcounts.data(), sizeof(int) * robots, cudaMemcpyHostToDevice));
    std::vector<fl_scan_raw_t> raws(robots);
    for (int r = 0; r < robots; r++)
        raws[r] = {dxyzi + 4 * (size_t)n_raw * r, dtms + (size_t)n_raw * r, dn + r, dposes + 22 * (size_t)n_pose * r, dnp + r, dxend + 26 * (size_t)r};
    CK(cudaMemcpy(draw, raws.data(), sizeof(fl_scan_raw_t) * robots, cudaMemcpyHostToDevice));
    std::vector<double> Pall(529 * (size_t)robots);
    for (int r = 0; r < robots; r++) memcpy(&Pall[529 * (size_t)r], P0.data(), sizeof(double) * 529);
    CK(cudaMemcpy(dx, x0.data(), sizeof(double) * x0.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dP, Pall.data(), sizeof(double) * Pall.size(), cudaMemcpyHostToDevice));
    // the twin chain's states and per-robot inputs
    double *tx = nullptr, *tP = nullptr; int* ts = nullptr;
    CK(cudaMalloc(&tx, sizeof(double) * 26 * robots));
    CK(cudaMalloc(&tP, sizeof(double) * 529 * robots));
    CK(cudaMalloc(&ts, sizeof(int) * 2));
    CK(cudaMemcpy(tx, x0.data(), sizeof(double) * x0.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(tP, Pall.data(), sizeof(double) * Pall.size(), cudaMemcpyHostToDevice));

    auto fill = [&](int k) {
        for (int r = 0; r < robots; r++) {
            const Raw& w = raw[(size_t)r * steps + k];
            CK(cudaMemcpyAsync(dxyzi + 4 * (size_t)n_raw * r, w.xyzi.data(), sizeof(float) * w.xyzi.size(), cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(dtms + (size_t)n_raw * r, w.t_ms.data(), sizeof(float) * n_raw, cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(dposes + 22 * (size_t)n_pose * r, w.poses.data(), sizeof(double) * w.poses.size(), cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(dxend + 26 * (size_t)r, w.x_end.data(), sizeof(double) * 26, cudaMemcpyHostToDevice, st));
        }
        CK(cudaStreamSynchronize(st));
    };
    auto front = [&](fl_scan_t* s, int r) {
        OK(fl_scan_upload_device(s, dxyzi + 4 * (size_t)n_raw * r, dtms + (size_t)n_raw * r, dn + r, n_raw, st));
        OK(fl_scan_undistort_device(s, dposes + 22 * (size_t)n_pose * r, dnp + r, n_pose, dxend + 26 * (size_t)r, st));
        OK(fl_scan_voxel_downsample_device(s, leaf, nullptr, st));
    };

    // warm-up outside capture on throw-away states, then one capture of the whole fleet step
    double *wx = nullptr, *wP = nullptr;
    CK(cudaMalloc(&wx, sizeof(double) * 26 * robots));
    CK(cudaMalloc(&wP, sizeof(double) * 529 * robots));
    CK(cudaMemcpy(wx, x0.data(), sizeof(double) * x0.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(wP, Pall.data(), sizeof(double) * Pall.size(), cudaMemcpyHostToDevice));
    fill(0);
    OK(fl_scan_batch_run_device(batch, draw, robots, n_raw, n_pose, 1, leaf, dbs, st));
    OK(fl_filter_update_scans_device(fg, dref, robots, n_raw, wx, wP, R, ds, nullptr, st));
    CK(cudaStreamSynchronize(st));
    cudaGraph_t graph;
    cudaGraphExec_t exec;
    CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeGlobal));
    OK(fl_scan_batch_run_device(batch, draw, robots, n_raw, n_pose, 1, leaf, dbs, st));
    OK(fl_filter_update_scans_device(fg, dref, robots, n_raw, dx, dP, R, ds, nullptr, st));
    CK(cudaStreamEndCapture(st, &graph));
    CK(cudaGraphInstantiate(&exec, graph, 0));

    int failures = 0;
    std::vector<double> gx(26), gP(529), hx(26), hP(529);
    for (int k = 0; k < steps; k++) {
        fill(k);
        CK(cudaGraphLaunch(exec, st));
        for (int r = 0; r < robots; r++) {            // the twin chain: one robot at a time
            front(twins[r], r);
            OK(fl_filter_update_scan_device(ft, twins[r], tx + 26 * (size_t)r, tP + 529 * (size_t)r, R, ts, st));
            int s2[2], g2[2], b2[2];
            CK(cudaMemcpyAsync(s2, ts, sizeof(s2), cudaMemcpyDeviceToHost, st));
            CK(cudaMemcpyAsync(b2, dbs + 2 * r, sizeof(b2), cudaMemcpyDeviceToHost, st));
            CK(cudaMemcpyAsync(g2, ds + 2 * r, sizeof(g2), cudaMemcpyDeviceToHost, st));
            CK(cudaMemcpyAsync(gx.data(), dx + 26 * (size_t)r, sizeof(double) * 26, cudaMemcpyDeviceToHost, st));
            CK(cudaMemcpyAsync(gP.data(), dP + 529 * (size_t)r, sizeof(double) * 529, cudaMemcpyDeviceToHost, st));
            CK(cudaMemcpyAsync(hx.data(), tx + 26 * (size_t)r, sizeof(double) * 26, cudaMemcpyDeviceToHost, st));
            CK(cudaMemcpyAsync(hP.data(), tP + 529 * (size_t)r, sizeof(double) * 529, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            if (b2[0] != FL_OK || b2[1] <= 0 || g2[0] != FL_OK || s2[0] != FL_OK || g2[1] != s2[1] || memcmp(gx.data(), hx.data(), sizeof(double) * 26) != 0 ||
                memcmp(gP.data(), hP.data(), sizeof(double) * 529) != 0) {
                printf("MISMATCH: step %d, robot %d (status %d/%d, passes %d/%d)\n", k, r, g2[0], s2[0], g2[1], s2[1]);
                failures++;
            }
        }
    }
    CK(cudaGraphExecDestroy(exec));
    CK(cudaGraphDestroy(graph));
    for (void* p : {(void*)draw, (void*)dbs, (void*)dxyzi, (void*)dtms, (void*)dposes, (void*)dxend, (void*)dx, (void*)dP, (void*)dn, (void*)dnp,
                    (void*)ds, (void*)tx, (void*)tP, (void*)ts, (void*)wx, (void*)wP})
        CK(cudaFree(p));
    for (int r = 0; r < robots; r++) fl_scan_destroy(twins[r]);
    fl_scan_batch_destroy(batch);
    fl_filter_destroy(fg);
    fl_filter_destroy(ft);
    fl_map_destroy(m);
    CK(cudaStreamDestroy(st));
    if (failures) { printf("%d mismatches\n", failures); return 4; }
    printf("all equal\n");
    return 0;
}
