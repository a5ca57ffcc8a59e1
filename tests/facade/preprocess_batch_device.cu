// A plain C/CUDA caller of the batched preprocess: a fleet step from the drivers' raw Livox points.  One
// fl_preprocess_batch_run_device turns every robot's raw frame into pl_surf in the handle's outputs, one fl_scan_batch_run_device
// reads those slots in place through a fl_scan_raw_t table built once, and one fl_filter_update_scans_device updates every robot.
// The three calls are captured into one graph with cudaStreamBeginCapture, at 1 and at 64 robots on the same handles: the graphs
// must have the same number of nodes, and every robot's statuses must be FL_OK after a replay.  The map and the frames are
// generated here (a floor and two walls, frames sampled from them around the origin); the frames are small enough after the
// voxel grid that the update runs every robot in one wave, as its launches follow its waves.  Prints "preprocess_batch_device ok".
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "fastlio_b200.h"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(2); } } while (0)
#define OK(x) do { int r_ = (x); if (r_ < 0) { printf("%s: %d %s\n", #x, r_, fl_last_error()); exit(3); } } while (0)

static unsigned long long g_rng = 88172645463325252ull;
static double uni() {                        // xorshift64, [0, 1)
    g_rng ^= g_rng << 13; g_rng ^= g_rng >> 7; g_rng ^= g_rng << 17;
    return (double)(g_rng >> 11) / 9007199254740992.0;
}

// a point of the scene within `span` of the origin: the floor z = -1.5 or the walls x = 4.5, y = 4.5
static void scene_point(float* p, double span) {
    const double a = (uni() * 2 - 1) * span, b = (uni() * 2 - 1) * span, w = uni();
    if (w < 0.6) { p[0] = (float)a; p[1] = (float)b; p[2] = -1.5f; }
    else if (w < 0.8) { p[0] = 4.5f; p[1] = (float)a; p[2] = (float)(-1.5 + 3.0 * uni()); }
    else { p[0] = (float)a; p[1] = 4.5f; p[2] = (float)(-1.5 + 3.0 * uni()); }
}

int main() {
    const int S_MAX = 64, N_RAW = 8192, max_iter = 4;
    const int step = 20;                     // livox_ros_driver::CustomPoint
    // the map: 40 000 points of the scene
    std::vector<float> map(4 * 40000);
    for (int i = 0; i < 40000; i++) { scene_point(&map[4 * i], 8.0); map[4 * i + 3] = 1.f; }
    // one raw Avia frame per robot: row 0 a dummy, then points of the scene, tag 0x10, lines 0-5, offset times in ns
    std::vector<unsigned char> raw((size_t)S_MAX * N_RAW * step, 0);
    std::vector<int> counts(S_MAX);
    for (int r = 0; r < S_MAX; r++) {
        const int n = 3000 + (int)(uni() * 4000);
        counts[r] = n;
        for (int i = 0; i < n; i++) {
            unsigned char* row = &raw[((size_t)r * N_RAW + i) * step];
            float p[3] = {0.f, 0.f, 0.f};
            if (i > 0) scene_point(p, 4.0);
            const unsigned t = (unsigned)((long long)i * 100000000ll / n);
            memcpy(row, &t, 4);
            memcpy(row + 4, p, 12);
            row[16] = (unsigned char)(i % 256); row[17] = 0x10; row[18] = (unsigned char)(i % 6);
        }
    }

    cudaStream_t st;
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    fl_map_t* m = nullptr;
    OK(fl_map_create(&m, 0, 0.5f));
    OK(fl_map_build(m, map.data(), 40000));
    fl_filter_t* f = nullptr;
    OK(fl_filter_create(&f, m, N_RAW));
    OK(fl_filter_set_params(f, max_iter, nullptr, 0));
    // the largest nq_max whose plan runs 64 robots in one wave (a frame down-samples to at most ~450 points: 0.5 m voxels of an
    // 8 m x 8 m floor and two 8 m x 3 m walls)
    OK(fl_filter_reserve_batch(f, 4096));
    int NQ_MAX = 0;
    for (int nq = 4096; nq >= 512 && !NQ_MAX; nq /= 2) {
        int plan[3];
        OK(fl_filter_batch_plan(f, nq, S_MAX, plan));
        if (plan[2] == 1) NQ_MAX = nq;
    }
    if (!NQ_MAX) { printf("no nq_max of 512 or more runs %d robots in one wave\n", S_MAX); return 4; }

    fl_preprocess_params_t pp = {FL_LIDAR_AVIA, 6, 10, 3, 1, 0.5, step, 4, 8, 12, 16, 0, -1, 17, 18};
    fl_preprocess_batch_t* pb = nullptr;
    OK(fl_preprocess_batch_create(&pb, 0, &pp, S_MAX, N_RAW));
    float *xyzi = nullptr, *ms = nullptr, *last = nullptr;
    int* out2 = nullptr;
    int n_raw_max = 0;
    OK(fl_preprocess_batch_get_outputs(pb, &xyzi, &ms, &out2, &last, &n_raw_max));
    if (n_raw_max != N_RAW) { printf("n_raw_max %d, expected %d\n", n_raw_max, N_RAW); return 5; }
    fl_scan_batch_t* sb = nullptr;
    OK(fl_scan_batch_create(&sb, m));
    OK(fl_scan_batch_reserve(sb, S_MAX, N_RAW, 0));
    const fl_scan_ref_t* refs = nullptr;
    OK(fl_scan_batch_get_refs(sb, 1, &refs, nullptr));

    // device inputs: the raw frames and counts, the two tables, the states and the statuses
    unsigned char* draw = nullptr;
    int *dn = nullptr, *dps = nullptr, *dss = nullptr, *dus = nullptr;
    fl_preprocess_raw_t* dpraw = nullptr;
    fl_scan_raw_t* dsraw = nullptr;
    double *dx = nullptr, *dP = nullptr;
    CK(cudaMalloc(&draw, raw.size()));
    CK(cudaMalloc(&dn, sizeof(int) * S_MAX));
    CK(cudaMalloc(&dps, sizeof(int) * 2 * S_MAX));
    CK(cudaMalloc(&dss, sizeof(int) * 2 * S_MAX));
    CK(cudaMalloc(&dus, sizeof(int) * 2 * S_MAX));
    CK(cudaMalloc(&dpraw, sizeof(fl_preprocess_raw_t) * S_MAX));
    CK(cudaMalloc(&dsraw, sizeof(fl_scan_raw_t) * S_MAX));
    CK(cudaMalloc(&dx, sizeof(double) * 26 * S_MAX));
    CK(cudaMalloc(&dP, sizeof(double) * 529 * S_MAX));
    CK(cudaMemcpy(draw, raw.data(), raw.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dn, counts.data(), sizeof(int) * S_MAX, cudaMemcpyHostToDevice));
    std::vector<fl_preprocess_raw_t> praw(S_MAX);
    std::vector<fl_scan_raw_t> sraw(S_MAX);
    for (int r = 0; r < S_MAX; r++) {
        praw[r].raw = draw + (size_t)r * N_RAW * step;
        praw[r].n_raw = dn + r;
        sraw[r] = fl_scan_raw_t{xyzi + (size_t)r * N_RAW * 4, ms + (size_t)r * N_RAW, out2 + 2 * r, nullptr, nullptr, nullptr};
    }
    CK(cudaMemcpy(dpraw, praw.data(), sizeof(fl_preprocess_raw_t) * S_MAX, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dsraw, sraw.data(), sizeof(fl_scan_raw_t) * S_MAX, cudaMemcpyHostToDevice));
    std::vector<double> x(26 * S_MAX, 0.0), P(529 * S_MAX, 0.0);
    for (int r = 0; r < S_MAX; r++) {
        double* xr = &x[26 * r];
        xr[6] = 1.0; xr[10] = 1.0; xr[25] = -9.81;           // rot and offset_R_L_I the identity (x, y, z, w), gravity -z
        for (int i = 0; i < 23; i++) P[529 * r + 24 * i] = 1e-3;
    }

    size_t nodes[2] = {0, 0};
    const int sizes[2] = {1, S_MAX};
    for (int k = 0; k < 2; k++) {
        const int S = sizes[k];
        CK(cudaMemcpy(dx, x.data(), sizeof(double) * x.size(), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(dP, P.data(), sizeof(double) * P.size(), cudaMemcpyHostToDevice));
        CK(cudaMemset(dus, 0xFF, sizeof(int) * 2 * S_MAX));
        cudaGraph_t g;
        cudaGraphExec_t ge;
        CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        OK(fl_preprocess_batch_run_device(pb, dpraw, S, N_RAW, dps, st));
        OK(fl_scan_batch_run_device(sb, dsraw, S, N_RAW, 0, 0, 0.5f, dss, st));
        OK(fl_filter_update_scans_device(f, refs, S, NQ_MAX, dx, dP, 0.001, dus, nullptr, st));
        CK(cudaStreamEndCapture(st, &g));
        CK(cudaGraphGetNodes(g, nullptr, &nodes[k]));
        CK(cudaGraphInstantiate(&ge, g, 0));
        CK(cudaGraphLaunch(ge, st));
        CK(cudaStreamSynchronize(st));
        std::vector<int> ps(2 * S), ss(2 * S), us(2 * S);
        CK(cudaMemcpy(ps.data(), dps, sizeof(int) * 2 * S, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(ss.data(), dss, sizeof(int) * 2 * S, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(us.data(), dus, sizeof(int) * 2 * S, cudaMemcpyDeviceToHost));
        for (int r = 0; r < S; r++) {
            if (ps[2 * r] != FL_OK || ps[2 * r + 1] <= 0 || ss[2 * r] != FL_OK || ss[2 * r + 1] <= 0 || us[2 * r] != FL_OK) {
                printf("S = %d robot %d: preprocess (%d, %d), scan batch (%d, %d), update (%d, %d)\n", S, r, ps[2 * r], ps[2 * r + 1],
                       ss[2 * r], ss[2 * r + 1], us[2 * r], us[2 * r + 1]);
                return 6;
            }
        }
        CK(cudaGraphExecDestroy(ge));
        CK(cudaGraphDestroy(g));
        printf("S = %d: %zu graph nodes (nq_max %d)\n", S, nodes[k], NQ_MAX);
    }
    if (nodes[0] != nodes[1]) { printf("node counts differ: %zu at S = 1, %zu at S = %d\n", nodes[0], nodes[1], S_MAX); return 7; }

    OK(fl_preprocess_batch_destroy(pb));
    OK(fl_scan_batch_destroy(sb));
    OK(fl_filter_destroy(f));
    OK(fl_map_destroy(m));
    CK(cudaFree(draw)); CK(cudaFree(dn)); CK(cudaFree(dps)); CK(cudaFree(dss)); CK(cudaFree(dus));
    CK(cudaFree(dpraw)); CK(cudaFree(dsraw)); CK(cudaFree(dx)); CK(cudaFree(dP));
    CK(cudaStreamDestroy(st));
    printf("preprocess_batch_device ok\n");
    return 0;
}
