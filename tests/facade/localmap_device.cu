// A plain C/CUDA caller of the whole per-scan chain of laserMapping.cpp on the device: lasermap_fov_segment (the cube slid from the
// state on the device, Delete_Point_Boxes) -> raw points -> de-skew -> down-sample -> update -> map_incremental, every count in
// device memory.  The first scan runs the device forms on the program's own stream; the chain
// is then captured into one CUDA graph (cudaStreamBeginCapture) with the upper bound n_max, and the graph is replayed for every
// other scan, whatever its size and IMU pose count (the inputs are copied into the captured buffers first).  Every scan is
// compared with the host forms on a twin map, cube, scan and filter (the host-form segment with pos_lid computed here in the
// order of Eigen's _transformVector): cub_needrm, kdtree_delete_counter, x, P and the three counts of map_incremental; at the end,
// after fl_map_maintain, the point sets and the cubes.  Between scans the program stands in for esekf::predict: it moves the
// updated state by predict_dx along x and copies it into the captured x.  Input file: 5 ints (map points, scans, n_max,
// n_pose_max, max_iter), R (double), leaf (float), cube_len (double), det_range (float), predict_dx (double), the map (x, y,
// z, i float32), x26 and P (23 x 23) as float64, then per scan: n and n_pose (ints), xyzi (n x 4
// float32), offset times (n float32), the IMU poses (n_pose x 22 float64) and x26_end (26 float64).  Prints "all equal" and
// exits 0 when every result matches.
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
#define RD(p, sz, n) do { if (fread((p), (sz), (n), f) != (size_t)(n)) { printf("short input\n"); return 1; } } while (0)

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
    if (argc < 2) { printf("usage: localmap_device in.bin\n"); return 1; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { printf("cannot open %s\n", argv[1]); return 1; }
    int hdr[5];
    double R = 0.0;
    float leaf = 0.f;
    double cube_len = 0.0;
    float det_range = 0.f;
    RD(hdr, sizeof(int), 5); RD(&R, sizeof(double), 1); RD(&leaf, sizeof(float), 1);
    double predict_dx = 0.0;
    RD(&cube_len, sizeof(double), 1); RD(&det_range, sizeof(float), 1); RD(&predict_dx, sizeof(double), 1);
    const int n_map = hdr[0], n_scans = hdr[1], n_max = hdr[2], n_pose_max = hdr[3], max_iter = hdr[4];
    std::vector<float> map_pts((size_t)n_map * 4);
    RD(map_pts.data(), sizeof(float), map_pts.size());
    double xh[26], Ph[529];
    RD(xh, sizeof(double), 26); RD(Ph, sizeof(double), 529);

    fl_map_t *mh = nullptr, *md = nullptr;
    OK(fl_map_create(&mh, 0, 0.5f)); OK(fl_map_create(&md, 0, 0.5f));
    OK(fl_map_build(mh, map_pts.data(), n_map)); OK(fl_map_build(md, map_pts.data(), n_map));
    fl_filter_t *fh = nullptr, *fd = nullptr;
    OK(fl_filter_create(&fh, mh, n_max)); OK(fl_filter_create(&fd, md, n_max));
    OK(fl_filter_set_params(fh, max_iter, nullptr, 0)); OK(fl_filter_set_params(fd, max_iter, nullptr, 0));
    fl_scan_t *sh = nullptr, *sd = nullptr;
    OK(fl_scan_create(&sh, mh)); OK(fl_scan_create(&sd, md));
    OK(fl_scan_reserve(sd, n_max, n_pose_max));
    fl_localmap_t *lh = nullptr, *ld = nullptr;
    OK(fl_localmap_create(&lh, cube_len, det_range)); OK(fl_localmap_create(&ld, cube_len, det_range));

    float *d_xyzi, *d_t;
    double *d_poses, *d_xend, *d_x, *d_P;
    int *d_n, *d_npose, *d_status, *d_out4, *d_seg3;
    float* d_boxes;
    CK(cudaMalloc(&d_xyzi, sizeof(float) * 4 * n_max)); CK(cudaMalloc(&d_t, sizeof(float) * n_max));
    CK(cudaMalloc(&d_poses, sizeof(double) * 22 * n_pose_max)); CK(cudaMalloc(&d_xend, sizeof(double) * 26));
    CK(cudaMalloc(&d_x, sizeof(double) * 26)); CK(cudaMalloc(&d_P, sizeof(double) * 529));
    CK(cudaMalloc(&d_n, sizeof(int))); CK(cudaMalloc(&d_npose, sizeof(int)));
    CK(cudaMalloc(&d_status, sizeof(int) * 2)); CK(cudaMalloc(&d_out4, sizeof(int) * 4));
    CK(cudaMalloc(&d_seg3, sizeof(int) * 3)); CK(cudaMalloc(&d_boxes, sizeof(float) * 18));
    CK(cudaMemcpy(d_x, xh, sizeof(xh), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_P, Ph, sizeof(Ph), cudaMemcpyHostToDevice));
    cudaStream_t st;
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    void* s = (void*)st;
    auto chain = [&]() {
        OK(fl_localmap_segment_device(ld, md, d_x, d_n, d_boxes, d_seg3, s));      // reads the predicted x (:890, :913)
        OK(fl_scan_upload_device(sd, d_xyzi, d_t, d_n, n_max, s));
        OK(fl_scan_undistort_device(sd, d_poses, d_npose, n_pose_max, d_xend, s));
        OK(fl_scan_voxel_downsample_device(sd, leaf, nullptr, s));
        OK(fl_filter_update_scan_device(fd, sd, d_x, d_P, R, d_status, s));
        OK(fl_filter_map_incremental_device(fd, 0.5, 1, d_out4, s));
    };
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    int slides = 0;
    for (int k = 0; k < n_scans; k++) {
        int nn[2];
        RD(nn, sizeof(int), 2);
        const int n = nn[0], n_pose = nn[1];
        std::vector<float> xyzi((size_t)std::max(n, 1) * 4), t((size_t)std::max(n, 1));
        std::vector<double> poses((size_t)std::max(n_pose, 1) * 22), xend(26);
        RD(xyzi.data(), sizeof(float), (size_t)n * 4); RD(t.data(), sizeof(float), n);
        RD(poses.data(), sizeof(double), (size_t)n_pose * 22); RD(xend.data(), sizeof(double), 26);
        // host forms on the twin: pos_lid = pos + rot * offset_T_L_I (:890), Eigen's _transformVector
        const double* q = xh + 3;
        const double* v = xh + 11;
        double uv[3] = {q[1] * v[2] - q[2] * v[1], q[2] * v[0] - q[0] * v[2], q[0] * v[1] - q[1] * v[0]};
        for (int a = 0; a < 3; a++) uv[a] = uv[a] + uv[a];
        const double c[3] = {q[1] * uv[2] - q[2] * uv[1], q[2] * uv[0] - q[0] * uv[2], q[0] * uv[1] - q[1] * uv[0]};
        double pos[3];
        for (int a = 0; a < 3; a++) pos[a] = xh[a] + ((v[a] + uv[a] * q[3]) + c[a]);
        float boxes_h[18] = {0};
        int deleted_h = 0;
        const int nb_h = fl_localmap_segment(lh, mh, pos, boxes_h, &deleted_h);
        OK(nb_h);
        slides += nb_h > 0;
        OK(fl_scan_upload(sh, xyzi.data(), t.data(), n));
        OK(fl_scan_undistort(sh, poses.data(), n_pose, xend.data()));
        OK(fl_scan_voxel_downsample(sh, leaf));
        OK(fl_filter_update_scan(fh, sh, xh, Ph, R, nullptr));
        int out3[3];
        OK(fl_filter_map_incremental(fh, 0.5, 1, out3));
        // device forms: inputs into the captured buffers, then the chain (scan 0) or a replay
        CK(cudaMemcpyAsync(d_xyzi, xyzi.data(), sizeof(float) * 4 * n, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_t, t.data(), sizeof(float) * n, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_n, &n, sizeof(int), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_poses, poses.data(), sizeof(double) * 22 * n_pose, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_npose, &n_pose, sizeof(int), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_xend, xend.data(), sizeof(double) * 26, cudaMemcpyHostToDevice, st));
        if (k == 0) {
            chain();
        } else {
            if (!exec) {
                CK(cudaStreamSynchronize(st));
                OK(fl_map_maintain(md, nullptr));           // settles the host's bound of the map's headroom before capturing
                CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
                chain();
                CK(cudaStreamEndCapture(st, &graph));
                CK(cudaGraphInstantiate(&exec, graph, 0));
            }
            CK(cudaGraphLaunch(exec, st));
        }
        double x[26], P[529];
        int status[2], out4[4], seg3[3];
        float boxes_d[18];
        CK(cudaMemcpyAsync(x, d_x, sizeof(x), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(P, d_P, sizeof(P), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(status, d_status, sizeof(status), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(out4, d_out4, sizeof(out4), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(seg3, d_seg3, sizeof(seg3), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(boxes_d, d_boxes, sizeof(boxes_d), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        expect(seg3[0] == nb_h && seg3[1] == deleted_h, "cub_needrm size / kdtree_delete_counter", k);
        expect(seg3[2] == FL_OK || seg3[2] == 1, "segment status", k);
        expect(memcmp(boxes_d, boxes_h, sizeof(float) * 6 * nb_h) == 0, "cub_needrm", k);
        expect(status[0] == FL_OK, "update status", k);
        expect(memcmp(x, xh, sizeof(x)) == 0, "x", k);
        expect(memcmp(P, Ph, sizeof(P)) == 0, "P", k);
        expect(out4[0] == out3[0] && out4[1] == out3[1] && out4[2] == out3[2], "map_incremental counts", k);
        expect(out4[3] == FL_OK || out4[3] == 1, "map_incremental status", k);
        int moved = 0;
        if (out4[3] == 1 || seg3[2] == 1) OK(fl_map_maintain(md, &moved));
        if (moved && exec) { cudaGraphExecDestroy(exec); cudaGraphDestroy(graph); exec = nullptr; graph = nullptr; }   // capture again
        xh[0] += predict_dx;                                // the prediction of the next scan, on the host
        CK(cudaMemcpyAsync(d_x, xh, sizeof(xh), cudaMemcpyHostToDevice, st));
    }
    int changed = 0;
    OK(fl_map_maintain(md, &changed));
    expect(fl_map_validnum(md) == fl_map_validnum(mh), "validnum", n_scans);
    expect(sorted_points(md) == sorted_points(mh), "map points", n_scans);
    float cube_h[6], cube_d[6];
    OK(fl_localmap_get(lh, cube_h)); OK(fl_localmap_get(ld, cube_d));
    expect(memcmp(cube_h, cube_d, sizeof(cube_h)) == 0, "cube", n_scans);
    expect(slides > 0, "the cube never slid", n_scans);
    if (exec) { cudaGraphExecDestroy(exec); cudaGraphDestroy(graph); }
    cudaStreamDestroy(st);
    cudaFree(d_xyzi); cudaFree(d_t); cudaFree(d_poses); cudaFree(d_xend); cudaFree(d_x); cudaFree(d_P);
    cudaFree(d_n); cudaFree(d_npose); cudaFree(d_status); cudaFree(d_out4); cudaFree(d_seg3); cudaFree(d_boxes);
    fl_localmap_destroy(lh); fl_localmap_destroy(ld);
    fl_scan_destroy(sh); fl_scan_destroy(sd); fl_filter_destroy(fh); fl_filter_destroy(fd); fl_map_destroy(mh); fl_map_destroy(md);
    if (failures) { printf("%d mismatches\n", failures); return 4; }
    printf("all equal (%d slides)\n", slides);
    return 0;
}
