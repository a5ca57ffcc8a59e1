// Test harness for the FP64 manifold arithmetic (lie.cuh), the per-point measurement model (measure.cuh) and the
// Gauss-Jordan solvers (gj.cuh).
//
// mh_eval runs one lie.cuh or measure.cuh function over a batch of inputs, either in a kernel (one thread per input) or on the host,
// from the same FL_HD code; mh_gj runs one Gauss-Jordan routine per block over a batch of systems.  Built with the
// library's nvcc flags (tests/manifold_harness.py), so it measures the arithmetic the library ships.
#include "../../fast_lio_b200/csrc/gj.cuh"
#include "../../fast_lio_b200/csrc/lie.cuh"
#include "../../fast_lio_b200/csrc/measure.cuh"

namespace fl {
void set_last_error(const char*, ...) {}
}
using namespace fl;

enum Fn {
    F_COS_SINC_SQRT, F_SO3_EXP, F_SO3_LOG, F_A_MATRIX, F_S2_BX, F_S2_BOXPLUS, F_S2_BOXMINUS, F_S2_NX_YY, F_S2_MX,
    F_S2_CONGRUENCE, F_STATE_BOXPLUS, F_STATE_BOXMINUS, F_ESTI_PLANE, F_MEASURE, F_COUNT
};
// inputs / outputs per evaluation, in doubles
static const int kWidth[F_COUNT][2] = {{1, 2}, {3, 4}, {4, 3}, {3, 9}, {3, 6}, {5, 3}, {6, 2}, {3, 6}, {5, 6},
                                       {8, 4}, {49, 26}, {52, 23}, {16, 5}, {47, 38}};

// Floats travel exactly in the double arrays.
FL_HD void esti_plane_eval(const double* in, double* out) {      // in: 5 x 3 points, threshold; out: ok, pabcd
    float pt[KNN_K][3], pabcd[4];
    for (int j = 0; j < KNN_K; j++) for (int c = 0; c < 3; c++) pt[j][c] = (float)in[3 * j + c];
    out[0] = esti_plane_dev(pabcd, pt, (float)in[15]) ? 1.0 : 0.0;
    for (int c = 0; c < 4; c++) out[1 + c] = pabcd[c];
}

// One scan point through the measurement model in the order of measure_fused (update.cuh), every stage evaluated whatever
// the gates before it decided.  in: x26, body point (3), 5 x 3 neighbours, neighbour count, 5th squared distance, extr.
// out: world point (3), kNN gate, plane ok, score gate, pabcd (4), pd2, score, row (12, jacobian_row_at), z, and the row
// and z of jacobian_row (the split kernels' form).
template <bool EXTR>
FL_HD void measure_eval(const double* in, double* out) {
    const PoseS s = load_pose(in);
    const float4 pb = make_float4((float)in[26], (float)in[27], (float)in[28], 0.f);
    float pn[KNN_K][3];
    for (int j = 0; j < KNN_K; j++) for (int c = 0; c < 3; c++) pn[j][c] = (float)in[29 + 3 * j + c];
    float wx, wy, wz;
    const D3 p_this = body_to_world(s, pb, wx, wy, wz);
    const bool gate = knn_gate((int)in[44], (float)in[45]);
    float pabcd[4];
    const bool ok = esti_plane_dev(pabcd, pn, 0.1f);
    const float pd2 = plane_residual(pabcd, wx, wy, wz);
    float score;
    const bool scored = score_gate(pd2, sqrt(norm3(d3(pb.x, pb.y, pb.z))), score);
    const float4 nv = make_float4(pabcd[0], pabcd[1], pabcd[2], pd2);
    double h[12] = {0.0}, h2[12] = {0.0}, z, z2;
    jacobian_row_at<EXTR>(s, pb, p_this, nv, h, z);
    jacobian_row<EXTR>(s, pb, nv, h2, z2);
    out[0] = wx; out[1] = wy; out[2] = wz;
    out[3] = gate; out[4] = ok; out[5] = scored;
    for (int c = 0; c < 4; c++) out[6 + c] = pabcd[c];
    out[10] = pd2; out[11] = score;
    for (int c = 0; c < 12; c++) { out[12 + c] = h[c]; out[25 + c] = h2[c]; }
    out[24] = z; out[37] = z2;
}

FL_HD void eval(int fn, const double* in, double* out) {
    switch (fn) {
    case F_COS_SINC_SQRT: cos_sinc_sqrt(in[0], out[0], out[1]); break;
    case F_SO3_EXP: stq(out, so3_exp(ld3(in))); break;
    case F_SO3_LOG: st3(out, so3_log(ldq(in))); break;
    case F_A_MATRIX: { const M33 a = A_matrix(ld3(in)); for (int i = 0; i < 9; i++) out[i] = a.m[i]; } break;
    case F_S2_BX: S2_Bx(ld3(in), out); break;
    case F_S2_BOXPLUS: st3(out, S2_boxplus(ld3(in), in[3], in[4])); break;
    case F_S2_BOXMINUS: S2_boxminus(ld3(in), ld3(in + 3), out[0], out[1]); break;
    case F_S2_NX_YY: S2_Nx_yy(ld3(in), out); break;
    case F_S2_MX: S2_Mx(ld3(in), in[3], in[4], out); break;
    case F_S2_CONGRUENCE: S2_congruence(ld3(in), ld3(in + 3), in[6], in[7], out); break;
    case F_STATE_BOXPLUS: for (int i = 0; i < XLEN; i++) out[i] = in[i]; state_boxplus(out, in + XLEN); break;
    case F_STATE_BOXMINUS: state_boxminus(in, in + XLEN, out); break;
    case F_ESTI_PLANE: esti_plane_eval(in, out); break;
    case F_MEASURE: if (in[46] != 0.0) measure_eval<true>(in, out); else measure_eval<false>(in, out); break;
    }
}

__global__ void k_eval(int fn, int count, int nin, int nout, const double* in, double* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) eval(fn, in + (size_t)i * nin, out + (size_t)i * nout);
}

// Gauss-Jordan variants; every one solves A X = B for the n x nc system [A | B] (row stride ld) of its block.
enum Gj { G_ELIMINATE, G_WARP, G_WARP_REG6, G_WARP_REG12, G_COLS6, G_COLS12 };

template <int N>
__device__ bool run_cols(double* a, int nc, int ld, int* row_k, int lane) {
    double c[N];
    for (int r = 0; r < N; r++) c[r] = lane < nc ? a[r * ld + lane] : 0.0;
    const bool ok = gj_cols<N>(c, row_k, lane);
    for (int r = 0; r < N; r++) if (lane < nc) a[r * ld + lane] = c[r];
    __syncwarp();
    return ok;
}

// x: n x (nc - n) solution; map: the routine's row map (row_of[k] = physical row of unknown k, or for gj_cols
// row_k[r] = unknown of physical row r); ok: the routine's return value
__global__ void k_gj(int variant, int n, int nc, int ld, const double* in, double* x, int* map, int* ok) {
    __shared__ double a[32 * 64];
    __shared__ int rmap[32], row_of[32];
    __shared__ int s_ok;
    const size_t sys = blockIdx.x;
    for (int e = threadIdx.x; e < n * ld; e += blockDim.x) a[e] = in[sys * n * ld + e];
    for (int e = threadIdx.x; e < 32; e += blockDim.x) rmap[e] = -1;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    if (variant == G_ELIMINATE) {
        const bool r = gj_eliminate(a, n, nc, ld, rmap);
        if (threadIdx.x == 0) s_ok = r;
    } else if (threadIdx.x < 32) {
        bool r = false;
        switch (variant) {
        case G_WARP: r = gj_warp(a, n, nc, ld, rmap, lane); break;
        case G_WARP_REG6: r = gj_warp_reg<6>(a, nc, ld, rmap, lane); break;
        case G_WARP_REG12: r = gj_warp_reg<12>(a, nc, ld, rmap, lane); break;
        case G_COLS6: r = run_cols<6>(a, nc, ld, rmap, lane); break;
        case G_COLS12: r = run_cols<12>(a, nc, ld, rmap, lane); break;
        }
        if (lane == 0) s_ok = r;
    }
    __syncthreads();
    const bool cols = variant == G_COLS6 || variant == G_COLS12;
    if (threadIdx.x < n) {
        map[sys * n + threadIdx.x] = rmap[threadIdx.x];
        if (cols) { const int k = rmap[threadIdx.x]; if (k >= 0 && k < n) row_of[k] = threadIdx.x; }
        else row_of[threadIdx.x] = rmap[threadIdx.x];
    }
    if (threadIdx.x == 0) ok[sys] = s_ok;
    __syncthreads();
    if (!s_ok) return;
    const int m = nc - n;
    for (int e = threadIdx.x; e < n * m; e += blockDim.x) {
        const int k = e / m, j = e % m, r = row_of[k];
        x[sys * n * m + e] = cols ? a[r * ld + n + j] : a[r * ld + n + j] / a[r * ld + k];
    }
}

extern "C" {

int mh_width(int fn, int which) { return fn >= 0 && fn < F_COUNT && (which == 0 || which == 1) ? kWidth[fn][which] : -1; }

// Evaluates function `fn` over `count` inputs; on the device when `device` != 0.  Returns 0 or a cudaError_t.
int mh_eval(int fn, int count, const double* in, double* out, int device) {
    if (mh_width(fn, 0) < 0 || count < 0) return -1;
    const int nin = kWidth[fn][0], nout = kWidth[fn][1];
    if (!device) {
        for (int i = 0; i < count; i++) eval(fn, in + (size_t)i * nin, out + (size_t)i * nout);
        return 0;
    }
    if (count == 0) return 0;
    double *din = nullptr, *dout = nullptr;
    cudaError_t e = cudaMalloc(&din, sizeof(double) * nin * count);
    if (e == cudaSuccess) e = cudaMalloc(&dout, sizeof(double) * nout * count);
    if (e == cudaSuccess) e = cudaMemcpy(din, in, sizeof(double) * nin * count, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) { k_eval<<<(count + 127) / 128, 128>>>(fn, count, nin, nout, din, dout); e = cudaGetLastError(); }
    if (e == cudaSuccess) e = cudaMemcpy(out, dout, sizeof(double) * nout * count, cudaMemcpyDeviceToHost);
    cudaFree(din);
    cudaFree(dout);
    return (int)e;
}

// Runs Gauss-Jordan variant `variant` on `count` systems of n x ld doubles with `threads` threads per block.
int mh_gj(int variant, int count, int n, int nc, int ld, int threads, const double* in, double* x, int* map, int* ok) {
    if (n < 1 || n > 32 || nc <= n || nc > 64 || ld < nc || n * ld > 32 * 64 || threads < 32 || threads % 32 || count < 1) return -1;
    if (variant != G_ELIMINATE && (nc > 32 || (variant == G_WARP && n > 12) || ((variant == G_WARP_REG6 || variant == G_COLS6) && n != 6) ||
                                   ((variant == G_WARP_REG12 || variant == G_COLS12) && n != 12)))
        return -1;
    const size_t na = (size_t)count * n * ld, nx = (size_t)count * n * (nc - n);
    double *din = nullptr, *dx = nullptr;
    int *dmap = nullptr, *dok = nullptr;
    cudaError_t e = cudaMalloc(&din, sizeof(double) * na);
    if (e == cudaSuccess) e = cudaMalloc(&dx, sizeof(double) * nx);
    if (e == cudaSuccess) e = cudaMalloc(&dmap, sizeof(int) * count * n);
    if (e == cudaSuccess) e = cudaMalloc(&dok, sizeof(int) * count);
    if (e == cudaSuccess) e = cudaMemcpy(din, in, sizeof(double) * na, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemset(dx, 0, sizeof(double) * nx);
    if (e == cudaSuccess) { k_gj<<<count, threads>>>(variant, n, nc, ld, din, dx, dmap, dok); e = cudaGetLastError(); }
    if (e == cudaSuccess) e = cudaMemcpy(x, dx, sizeof(double) * nx, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(map, dmap, sizeof(int) * count * n, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(ok, dok, sizeof(int) * count, cudaMemcpyDeviceToHost);
    cudaFree(din);
    cudaFree(dx);
    cudaFree(dmap);
    cudaFree(dok);
    return (int)e;
}

}  // extern "C"
