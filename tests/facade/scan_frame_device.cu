// A plain C/CUDA caller of the per-scan chain with its published clouds: upload -> de-skew -> down-sample -> update ->
// map_incremental, then a memset of the publish positions and three fl_scan_frame_device calls with the updated state -- the
// dense world cloud (publish_frame_world), the dense IMU-frame cloud (publish_frame_body) and the dense world cloud appended to
// an accumulation buffer (pcl_wait_save).  The first scan runs on the program's own stream, then the whole sequence is captured
// once (cudaStreamBeginCapture) and replayed for every other scan.  Every scan is compared with the host forms on a twin map,
// scan and filter followed by fl_scan_frame; at the end the accumulated cloud is compared with the concatenation of the host
// forms' world clouds.  Input file: that of frontend_device.cu.  Prints "all equal" and exits 0 when every result matches.
#include <cuda_runtime.h>

#include <algorithm>
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

int main(int argc, char** argv) {
    if (argc < 2) { printf("usage: scan_frame_device in.bin\n"); return 1; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { printf("cannot open %s\n", argv[1]); return 1; }
    int hdr[5];
    double R = 0.0;
    float leaf = 0.f;
    RD(hdr, sizeof(int), 5); RD(&R, sizeof(double), 1); RD(&leaf, sizeof(float), 1);
    const int n_map = hdr[0], n_scans = hdr[1], n_max = hdr[2], n_pose_max = hdr[3], max_iter = hdr[4];
    const int cap_save = n_max * n_scans;
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

    float *d_xyzi, *d_t, *d_world, *d_imu, *d_save;
    double *d_poses, *d_xend, *d_x, *d_P;
    int *d_n, *d_npose, *d_status, *d_out4, *d_pub, *d_nsave, *d_fst;
    CK(cudaMalloc(&d_xyzi, sizeof(float) * 4 * n_max)); CK(cudaMalloc(&d_t, sizeof(float) * n_max));
    CK(cudaMalloc(&d_world, sizeof(float) * 4 * n_max)); CK(cudaMalloc(&d_imu, sizeof(float) * 4 * n_max));
    CK(cudaMalloc(&d_save, sizeof(float) * 4 * cap_save));
    CK(cudaMalloc(&d_poses, sizeof(double) * 22 * n_pose_max)); CK(cudaMalloc(&d_xend, sizeof(double) * 26));
    CK(cudaMalloc(&d_x, sizeof(double) * 26)); CK(cudaMalloc(&d_P, sizeof(double) * 529));
    CK(cudaMalloc(&d_n, sizeof(int))); CK(cudaMalloc(&d_npose, sizeof(int)));
    CK(cudaMalloc(&d_status, sizeof(int) * 2)); CK(cudaMalloc(&d_out4, sizeof(int) * 4));
    CK(cudaMalloc(&d_pub, sizeof(int) * 2)); CK(cudaMalloc(&d_nsave, sizeof(int))); CK(cudaMalloc(&d_fst, sizeof(int) * 6));
    CK(cudaMemset(d_nsave, 0, sizeof(int)));
    CK(cudaMemcpy(d_x, xh, sizeof(xh), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_P, Ph, sizeof(Ph), cudaMemcpyHostToDevice));
    cudaStream_t st;
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    void* s = (void*)st;
    auto chain = [&]() {
        OK(fl_scan_upload_device(sd, d_xyzi, d_t, d_n, n_max, s));
        OK(fl_scan_undistort_device(sd, d_poses, d_npose, n_pose_max, d_xend, s));
        OK(fl_scan_voxel_downsample_device(sd, leaf, nullptr, s));
        OK(fl_filter_update_scan_device(fd, sd, d_x, d_P, R, d_status, s));
        OK(fl_filter_map_incremental_device(fd, 0.5, 1, d_out4, s));
        CK(cudaMemsetAsync(d_pub, 0, sizeof(int) * 2, st));                                     // this scan's clouds start at row 0
        OK(fl_scan_frame_device(sd, 0, FL_FRAME_WORLD, d_x, d_world, d_pub, n_max, d_fst, s));        // publish_frame_world
        OK(fl_scan_frame_device(sd, 0, FL_FRAME_IMU, d_x, d_imu, d_pub + 1, n_max, d_fst + 2, s));    // publish_frame_body
        OK(fl_scan_frame_device(sd, 0, FL_FRAME_WORLD, d_x, d_save, d_nsave, cap_save, d_fst + 4, s)); // pcl_wait_save +=
    };
    std::vector<float> saved;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    for (int k = 0; k < n_scans; k++) {
        int nn[2];
        RD(nn, sizeof(int), 2);
        const int n = nn[0], n_pose = nn[1];
        std::vector<float> xyzi((size_t)std::max(n, 1) * 4), t((size_t)std::max(n, 1));
        std::vector<double> poses((size_t)std::max(n_pose, 1) * 22), xend(26);
        RD(xyzi.data(), sizeof(float), (size_t)n * 4); RD(t.data(), sizeof(float), n);
        RD(poses.data(), sizeof(double), (size_t)n_pose * 22); RD(xend.data(), sizeof(double), 26);
        // host forms on the twin, then the clouds with the updated state
        OK(fl_scan_upload(sh, xyzi.data(), t.data(), n));
        OK(fl_scan_undistort(sh, poses.data(), n_pose, xend.data()));
        OK(fl_scan_voxel_downsample(sh, leaf));
        OK(fl_filter_update_scan(fh, sh, xh, Ph, R, nullptr));
        int out3[3];
        OK(fl_filter_map_incremental(fh, 0.5, 1, out3));
        std::vector<float> hw((size_t)std::max(n, 1) * 4), hi((size_t)std::max(n, 1) * 4);
        const int nw = fl_scan_frame(sh, 0, FL_FRAME_WORLD, xh, hw.data(), n);
        const int ni = fl_scan_frame(sh, 0, FL_FRAME_IMU, xh, hi.data(), n);
        OK(nw); OK(ni);
        saved.insert(saved.end(), hw.begin(), hw.begin() + (size_t)nw * 4);
        // device forms: inputs into the captured buffers, then the sequence (scan 0) or a replay
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
        int status[2], out4[4], fst[6], pub[2];
        std::vector<float> dw((size_t)std::max(n, 1) * 4), di((size_t)std::max(n, 1) * 4);
        CK(cudaMemcpyAsync(x, d_x, sizeof(x), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(P, d_P, sizeof(P), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(status, d_status, sizeof(status), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(out4, d_out4, sizeof(out4), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(fst, d_fst, sizeof(fst), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(pub, d_pub, sizeof(pub), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(dw.data(), d_world, sizeof(float) * 4 * nw, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(di.data(), d_imu, sizeof(float) * 4 * ni, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        expect(status[0] == FL_OK, "update status", k);
        expect(memcmp(x, xh, sizeof(x)) == 0, "x", k);
        expect(memcmp(P, Ph, sizeof(P)) == 0, "P", k);
        expect(out4[0] == out3[0] && out4[1] == out3[1] && out4[2] == out3[2], "map_incremental counts", k);
        expect(fst[0] == FL_OK && fst[1] == nw && fst[2] == FL_OK && fst[3] == ni && fst[4] == FL_OK && fst[5] == nw, "frame statuses", k);
        expect(pub[0] == nw && pub[1] == ni, "publish positions", k);
        expect(memcmp(dw.data(), hw.data(), sizeof(float) * 4 * nw) == 0, "world cloud", k);
        expect(memcmp(di.data(), hi.data(), sizeof(float) * 4 * ni) == 0, "IMU-frame cloud", k);
        int moved = 0;
        if (out4[3] == 1) OK(fl_map_maintain(md, &moved));
        if (moved && exec) { cudaGraphExecDestroy(exec); cudaGraphDestroy(graph); exec = nullptr; graph = nullptr; }   // capture again
    }
    int nsave = -1;
    CK(cudaMemcpy(&nsave, d_nsave, sizeof(int), cudaMemcpyDeviceToHost));
    expect((size_t)nsave * 4 == saved.size(), "accumulated rows", n_scans);
    std::vector<float> ds(saved.size() + 4);
    CK(cudaMemcpy(ds.data(), d_save, sizeof(float) * saved.size(), cudaMemcpyDeviceToHost));
    expect(memcmp(ds.data(), saved.data(), sizeof(float) * saved.size()) == 0, "accumulated cloud", n_scans);
    if (exec) { cudaGraphExecDestroy(exec); cudaGraphDestroy(graph); }
    cudaStreamDestroy(st);
    cudaFree(d_xyzi); cudaFree(d_t); cudaFree(d_world); cudaFree(d_imu); cudaFree(d_save); cudaFree(d_poses); cudaFree(d_xend);
    cudaFree(d_x); cudaFree(d_P); cudaFree(d_n); cudaFree(d_npose); cudaFree(d_status); cudaFree(d_out4); cudaFree(d_pub);
    cudaFree(d_nsave); cudaFree(d_fst);
    fl_scan_destroy(sh); fl_scan_destroy(sd); fl_filter_destroy(fh); fl_filter_destroy(fd); fl_map_destroy(mh); fl_map_destroy(md);
    if (failures) { printf("%d mismatches\n", failures); return 4; }
    printf("all equal\n");
    return 0;
}
