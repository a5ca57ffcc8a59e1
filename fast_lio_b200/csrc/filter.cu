// The per-scan iterated-EKF measurement update of FAST-LIO2 on the device.  Per pass, two kernels:
//
//   k_search   : the kNN half of h_share_model (reference src/laserMapping.cpp:656-672): body->world transform and
//                k = 5 nearest-neighbour search in the device map, one warp per scan point; works only on the passes
//                for which the filter asks for a search (decided on the device).
//   k_residual : the rest of h_share_model (:674-752) -- 5-point plane fit (esti_plane, include/common_lib.h:225-257),
//                residual gating, Jacobian row -- folded straight into the FP64 normal equations H^T H (12x12) /
//                H^T h (12) that update_iterated_dyn_share_modified consumes (esekfom.hpp:1784,1804), one deterministic
//                partial per block; block 0 is the solver block and runs esekfom.hpp:1651-1927 (boxminus, manifold
//                congruences on P, the Kalman gain algebra, boxplus, convergence bookkeeping, final covariance).
//
// The kernels of a scan are chained with programmatic dependent launch; the whole multi-pass update runs without a
// host round trip.  Multi-GPU: scan points are sharded, the 92 sums are exchanged inside k_residual over peer memory
// (or with NCCL between k_residual and k_solve_only).
#include <dlfcn.h>

#include <algorithm>
#include <chrono>
#include <cstdlib>

#include <cub/device/device_select.cuh>

#include "filter.h"
#include "gj.cuh"
#include "measure.cuh"

namespace fl {

constexpr int PSTRIDE = 96;          // doubles per partial row (NRED = 92 padded)
// peer mailbox: [2 parities][P2P_MAX_RANKS slots][PSTRIDE values] x two tagged 8-byte words per value
constexpr size_t P2P_MAIL_BYTES = sizeof(unsigned long long) * 2 * 2 * P2P_MAX_RANKS * PSTRIDE;
constexpr int SEARCH_THREADS = 256;
constexpr int SEARCH_C_THREADS = 256;
constexpr int RESID_THREADS = 256;
constexpr int MAX_LOGS = 16;

// Programmatic dependent launch (sm_90+): a kernel launched with the programmatic-serialization attribute
// may start while its predecessor in the stream is still running; pdl_wait() blocks until the predecessor
// has completed and flushed, pdl_launch() lets the successor begin its own launch early.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ int tri12(int a, int b) { return a * 12 - (a * (a - 1)) / 2 + (b - a); }   // a <= b

// Per-point part of h_share_model after the search (laserMapping.cpp:674-692).
// Returns true when the point contributes a row.
template <bool EXTR>
__device__ __forceinline__ bool measure_point(const ScanView& sc, int q, const PoseS& s, bool searched, double* h, double& z, float& absres) {
    if (!sc.selected[q]) return false;                                   // :674
    sc.selected[q] = 0;                                                  // :677
    const float4 pb = __ldg(&sc.body[q]);
    float wx, wy, wz;
    body_to_world(s, pb, wx, wy, wz);
    float pabcd[4];
    if (searched) {
        float pn[KNN_K][3];
#pragma unroll
        for (int j = 0; j < KNN_K; j++) { const float4 p = sc.nearest[(size_t)q * KNN_K + j]; pn[j][0] = p.x; pn[j][1] = p.y; pn[j][2] = p.z; }
        if (!esti_plane_dev(pabcd, pn, 0.1f)) return false;              // :678
        sc.plane[q] = make_float4(pabcd[0], pabcd[1], pabcd[2], pabcd[3]);
    } else {
        // A pass that does not search fits the plane to the SAME five neighbours (Nearest_Points persists, T3) and
        // only points whose fit succeeded last time are still selected: the fit is a pure function of the
        // neighbours, so its result is reused instead of recomputed.
        const float4 pl = sc.plane[q];
        pabcd[0] = pl.x; pabcd[1] = pl.y; pabcd[2] = pl.z; pabcd[3] = pl.w;
    }
    const float pd2 = plane_residual(pabcd, wx, wy, wz);                 // :680
    float score;
    if (!score_gate(pd2, sqrt(norm3(d3(pb.x, pb.y, pb.z))), score)) return false;    // :681-683
    sc.selected[q] = 1;
    const float4 nv = make_float4(pabcd[0], pabcd[1], pabcd[2], pd2);
    sc.normvec[q] = nv;
    absres = fabsf(pd2);                                                 // res_last
    jacobian_row<EXTR>(s, pb, nv, h, z);
    return true;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}

// Fold the rows held by the 32 lanes into the lane-distributed accumulators: output o of the
// NRED-vector lives in lane (o & 31), register acc[o >> 5].  The 32 rows are staged in the warp's
// slice of shared memory and every lane accumulates its own outputs over the 32 rows (one LDS pair +
// one FP64 multiply-add per row), instead of one 5-step shuffle butterfly per output.
template <bool EXTR> struct RowStage { static constexpr int NC = EXTR ? 12 : 6; static constexpr int RS = NC + 2; };   // h[NC], z, pad

template <bool EXTR>
__device__ __forceinline__ void warp_accumulate(bool contrib, const double* h, double z, float absres, double (&acc)[3],
                                                int lane, double* stage /* this warp's 32 x RS doubles */) {
    constexpr int NC = RowStage<EXTR>::NC, RS = RowStage<EXTR>::RS;
    constexpr int NPAIR = NC * (NC + 1) / 2;
    const unsigned any = __ballot_sync(FULL, contrib);
    if (!any) return;
#pragma unroll
    for (int a = 0; a < NC; a++) stage[lane * RS + a] = contrib ? h[a] : 0.0;
    stage[lane * RS + NC] = contrib ? z : 0.0;
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 3; j++) {
        const int t = lane + 32 * j;                      // t-th output of this pass: pairs (a<=b) row-major, then H^T h
        if (t < NPAIR + NC) {
            int a, b, o;
            if (t < NPAIR) {
                a = 0; int rem = t;
                while (rem >= NC - a) { rem -= NC - a; a++; }
                b = a + rem;
                o = a * 12 - (a * (a - 1)) / 2 + (b - a);  // position in the 12-wide upper triangle
            } else { a = t - NPAIR; b = NC; o = 78 + a; }
            double v = 0.0;
#pragma unroll 8
            for (int i = 0; i < 32; i++) v += stage[i * RS + a] * stage[i * RS + b];
            // hand the sum to the lane/register that owns output o
            // (t and o coincide lane-wise only when NC == 12; otherwise route through shared memory)
            stage[32 * RS + t] = v;
            (void)o;
        }
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 3; j++) {
        const int o = lane + 32 * j;                      // output owned by (lane, j)
        if (o < 90) {
            int t = -1;
            if (o < 78) {
                // invert tri12: find (a, b) of the 12-wide triangle
                int a = 0, rem = o;
                while (rem >= 12 - a) { rem -= 12 - a; a++; }
                const int b = a + rem;
                if (b < NC) t = a * NC - (a * (a - 1)) / 2 + (b - a);
            } else if (o - 78 < NC) t = NPAIR + (o - 78);
            if (t >= 0) acc[j] += stage[32 * RS + t];
        }
    }
    {
        const double v = (double)__popc(any);
        if (lane == (90 & 31)) acc[90 >> 5] += v;
        double r = contrib ? (double)absres : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(FULL, r, o);
        if (lane == (91 & 31)) acc[91 >> 5] += r;
    }
    __syncwarp();
}

// the search of one scan point by one warp, results stored as h_share_model leaves them (laserMapping.cpp:670-671)
__device__ __forceinline__ void search_point(const MapView& m, const ScanView& sc, int q, float qx, float qy, float qz, int lane) {
    KBest kb;
    knn_query(m, qx, qy, qz, kb, lane);
    float4 p;
    const int cnt = knn_fetch_warp(m, kb, p, lane);
    if (lane < KNN_K) sc.nearest[(size_t)q * KNN_K + lane] = p;
    if (lane == KNN_K - 1) {
        sc.nearest_cnt[q] = cnt;
        sc.selected[q] = knn_gate(cnt, kb.d) ? 1 : 0;                         // laserMapping.cpp:671
    }
}

// k_search -- the kNN half of h_share_model (laserMapping.cpp:667-672).  One warp per scan
// point, a contiguous run of points per warp: the lanes first transform the warp's points to the
// world frame thread-parallel (FP64, laserMapping.cpp:656-661), then the warp walks the map once
// per point.  Runs only when the filter asks for a search (ekfom_data.converge, decided on the
// device); few registers, so that many warps hide the latency of the dependent tree loads.
template <int MINB>
__global__ void __launch_bounds__(SEARCH_THREADS, MINB) k_search(MapView m, ScanView sc, const FilterCtl* __restrict__ ctl) {
    pdl_wait();                 // the previous pass's Kalman step (or the upload) is complete and visible
    pdl_launch();               // k_residual may start: its solver block prepares while we search
    if (ctl->done || !ctl->converge) return;
    if (blockIdx.x == 0 && threadIdx.x < XLEN) const_cast<FilterCtl*>(ctl)->x_search[threadIdx.x] = ctl->x[threadIdx.x];
    const int lane = threadIdx.x & 31;
    const int gwarp = (blockIdx.x * SEARCH_THREADS + threadIdx.x) >> 5;
    const int nwarps = (gridDim.x * SEARCH_THREADS) >> 5;
    const int q0 = sc.q_begin, q1 = sc.q_end;
    // balanced split: every warp gets floor or ceil of (points / warps) -- with a ceil-sized run per warp the last
    // ~10 % of the warps (whole SMs' worth) would sit idle while the others carry their points
    const long long nq = q1 - q0;
    const int wq0 = q0 + (int)(nq * gwarp / nwarps);
    const int wq1 = q0 + (int)(nq * (gwarp + 1) / nwarps);
    for (int base = wq0; base < wq1; base += 32) {
        const int myq = base + lane;
        float wx = 0.f, wy = 0.f, wz = 0.f;
        if (myq < wq1) {
            const PoseS s = load_pose(ctl->x);
            body_to_world(s, __ldg(&sc.body[myq]), wx, wy, wz);
        }
        const int cnt_chunk = min(32, wq1 - base);
        for (int l = 0; l < cnt_chunk; l++) {
            const float qx = __shfl_sync(FULL, wx, l), qy = __shfl_sync(FULL, wy, l), qz = __shfl_sync(FULL, wz, l);
            search_point(m, sc, base + l, qx, qy, qz, lane);
        }
    }
}

// ============================================================================= solve
struct SolveShared {
    double red[PSTRIDE];
    double HTH[144];
    double Hth[12];
    double wred[8 * PSTRIDE];     // per-warp partial sums (worker blocks: block partial; solver block: cross-block reduction)
    // ---- from here to stage_end: reused by the worker blocks as row-staging area (see k_residual)
    double P[NDOF * NDOF];        // P_propagated after the manifold congruence (esekfom.hpp:1657-1699)
    double L[NDOF * NDOF];        // scratch, then L_ of the final covariance step
    double aug[NDOF * 2 * NDOF];  // augmented system for Gauss-Jordan
    double Kx[NDOF * 12];         // K_x[:, 0:12]   (columns 12..22 are zero in every branch)
    double Kh[NDOF];
    double dx[NDOF], dx_new[NDOF], dxu[NDOF];
    double J[2][9];               // A_matrix(.)^T of the two SO3 blocks (rot, offset_R_L_I)
    double M2[4];                 // Nx * Mx of the S2 block (grav)
    double xnew[XLEN];
    double rows[22 * 13];         // small-m branch: [h_x row (12) | h]
    double PHt[NDOF * 22];        // small-m branch
    double T[22 * 13];            // S^{-1} [h_x | h]  /  (I + M A11)^{-1} [H^T h | H^T H]
    double stage_pad[760];        // tops the staging area up to 8 warps x (32 x 14 + 96) doubles
    double stage_end[1];
    int row_of[32], m_rows, finish, over, prep_ok;
    int row_idx[22];
};

// rows {3..5, 6..8, 21..22} of dst := J * (same rows of src), first `ncols` columns
__device__ void apply_rows(double* dst, const double* src, const double* J3, const double* J6, const double* M2, int ncols, int ld) {
    const int i = threadIdx.x;
    if (i < ncols) {
#pragma unroll
        for (int b = 0; b < 2; b++) {
            const int idx = b == 0 ? 3 : 6;
            const double* J = b == 0 ? J3 : J6;
            const double v0 = src[idx * ld + i], v1 = src[(idx + 1) * ld + i], v2 = src[(idx + 2) * ld + i];
            dst[idx * ld + i] = J[0] * v0 + J[1] * v1 + J[2] * v2;
            dst[(idx + 1) * ld + i] = J[3] * v0 + J[4] * v1 + J[5] * v2;
            dst[(idx + 2) * ld + i] = J[6] * v0 + J[7] * v1 + J[8] * v2;
        }
        const double a = src[21 * ld + i], bq = src[22 * ld + i];
        dst[21 * ld + i] = M2[0] * a + M2[1] * bq;
        dst[22 * ld + i] = M2[2] * a + M2[3] * bq;
    }
}
// columns {3..5, 6..8, 21..22} of the 23x23 `mat` := (row block) * J^T, for every row
__device__ void apply_cols(double* mat, const double* J3, const double* J6, const double* M2, int first_thread) {
    const int i = (int)threadIdx.x - first_thread;
    if (i >= 0 && i < NDOF) {
#pragma unroll
        for (int b = 0; b < 2; b++) {
            const int idx = b == 0 ? 3 : 6;
            const double* J = b == 0 ? J3 : J6;
            const double v0 = mat[i * NDOF + idx], v1 = mat[i * NDOF + idx + 1], v2 = mat[i * NDOF + idx + 2];
            mat[i * NDOF + idx] = J[0] * v0 + J[1] * v1 + J[2] * v2;
            mat[i * NDOF + idx + 1] = J[3] * v0 + J[4] * v1 + J[5] * v2;
            mat[i * NDOF + idx + 2] = J[6] * v0 + J[7] * v1 + J[8] * v2;
        }
        const double a = mat[i * NDOF + 21], bq = mat[i * NDOF + 22];
        mat[i * NDOF + 21] = a * M2[0] + bq * M2[1];
        mat[i * NDOF + 22] = a * M2[2] + bq * M2[3];
    }
}

// ----------------------------------------------------------------------------- the Kalman step of one pass
// Split in two so that the part that does not depend on this pass's residuals can run while the
// other blocks are still computing them:
//   solve_prepare : dx = x [-] x_prop, the manifold congruence blocks, P := T P_prop T^T
//                   (esekfom.hpp:1651-1699) and, for the reference-form solver, (P/R)^{-1};
//   solve_finish  : gain, dx_, boxplus, convergence bookkeeping, final covariance
//                   (esekfom.hpp:1715-1927), from the reduced normal equations in S.red.
// Both are block-wide (blockDim a multiple of 32 and >= 160: solve_finish copies H^T H one
// entry per thread; gj_eliminate takes any multiple of 32).  The scalar manifold work is spread over the first lanes
// of different warps so that the FP64 chains (and their instruction fetches) overlap.
#define STAMP(i) do { if (threadIdx.x == 0) ctl->prof[i] = clock64(); } while (0)

template <int SOLVER>
__device__ __noinline__ void solve_prepare(SolveShared& S, const FilterCtl* ctl) {
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5;
    constexpr int n = NDOF;
    if (lane == 0) {
        if (warp < 2) {                 // SO3 blocks: rot (idx 3), offset_R_L_I (idx 6)
            const int idx = warp == 0 ? 3 : 6, xo = warp == 0 ? X_ROT : X_OFFR;
            const D3 l = so3_log(qmul(qconj(ldq(ctl->x_prop + xo)), ldq(ctl->x + xo)));            // SOn.hpp:237-239
            const M33 J = transpose33(A_matrix(l));                                                 // T5
#pragma unroll 1
            for (int i = 0; i < 9; i++) S.J[warp][i] = J.m[i];
            const D3 seg = mul33v(J, l);
            S.dx[idx] = l.x; S.dx[idx + 1] = l.y; S.dx[idx + 2] = l.z;
            S.dx_new[idx] = seg.x; S.dx_new[idx + 1] = seg.y; S.dx_new[idx + 2] = seg.z;
        } else if (warp == 2) {         // S2 block: grav (idx 21)
            double d0, d1;
            S2_boxminus(ld3(ctl->x + X_GRAV), ld3(ctl->x_prop + X_GRAV), d0, d1);
            S2_congruence(ld3(ctl->x + X_GRAV), ld3(ctl->x_prop + X_GRAV), d0, d1, S.M2);
            S.dx[21] = d0; S.dx[22] = d1;
            S.dx_new[21] = S.M2[0] * d0 + S.M2[1] * d1;
            S.dx_new[22] = S.M2[2] * d0 + S.M2[3] * d1;
        }
    }
    if (warp == 3 && lane < 15) {       // vect blocks: pos, offset_T_L_I, vel, bg, ba
        const int b = lane / 3, c = lane % 3;
        const int dof = b == 0 ? 0 : 9 + 3 * (b - 1);
        const int xo = b == 0 ? X_POS : (b == 1 ? X_OFFT : (b == 2 ? X_VEL : (b == 3 ? X_BG : X_BA)));
        const double d = ctl->x[xo + c] - ctl->x_prop[xo + c];
        S.dx[dof + c] = d; S.dx_new[dof + c] = d;
    }
#pragma unroll 1
    for (int e = tid; e < n * n; e += nt) S.P[e] = ctl->P_prop[e];
    __syncthreads();
    // The reference interleaves row/column products per block (rows3, cols3, rows6, cols6, rows21,
    // cols21); the blocks act on disjoint index sets, so P := T P T^T either way.
    apply_rows(S.P, S.P, S.J[0], S.J[1], S.M2, n, n);
    __syncthreads();
    apply_cols(S.P, S.J[0], S.J[1], S.M2, 0);
    __syncthreads();
    S.prep_ok = 1;
    if constexpr (SOLVER == 0) {
        // first half of esekfom.hpp:1782:  P_temp = (P/R)^{-1}  -> S.L  (independent of H)
        const double R = ctl->R;
#pragma unroll 1
        for (int e = tid; e < n * 2 * n; e += nt) {
            const int i = e / (2 * n), j = e % (2 * n);
            S.aug[e] = j < n ? S.P[i * n + j] / R : (j - n == i ? 1.0 : 0.0);
        }
        __syncthreads();
        const bool ok = gj_eliminate(S.aug, n, 2 * n, 2 * n, S.row_of);
        if (ok) {
#pragma unroll 1
            for (int e = tid; e < n * n; e += nt) {
                const int k = e / n, j = e % n;
                const int pr = S.row_of[k];
                S.L[e] = S.aug[pr * 2 * n + n + j] / S.aug[pr * 2 * n + k];
            }
        }
        __syncthreads();
        if (tid == 0) S.prep_ok = ok ? 1 : 0;
        __syncthreads();
    }
}

// small-m branch, esekfom.hpp:1715-1744 (T6):  K = P H^T (H P H^T / R + I)^{-1} / R ;  K_h = K h ;  K_x = K H.
// Cold path (fewer than 23 effective points), kept out of line.
__device__ __noinline__ bool solve_gain_small_m(SolveShared& S, const FilterCtl* ctl, const ScanView& sc, int extr, double R) {
    const int tid = threadIdx.x, nt = blockDim.x;
    constexpr int n = NDOF;
    bool ok = true;
        //   K = P H^T (H P H^T / R + I)^{-1} / R ;  K_h = K h ;  K_x = K H
        // the m (< 23) Jacobian rows are rebuilt, in point order, from what k_residual left per point
        if (tid == 0) {
            int mrows = 0;
            for (int q = sc.q_begin; q < sc.q_end && mrows < 22; q++) if (sc.selected[q]) S.row_idx[mrows++] = q;
            S.m_rows = mrows;
        }
        __syncthreads();
        const int mr = S.m_rows;
        if (tid < mr) {
            const PoseS ps = load_pose(ctl->x);
            double h[12]; double z;
            for (int a = 0; a < 12; a++) h[a] = 0.0;
            const int q = S.row_idx[tid];
            if (extr) jacobian_row<true>(ps, sc.body[q], sc.normvec[q], h, z);
            else jacobian_row<false>(ps, sc.body[q], sc.normvec[q], h, z);
            for (int a = 0; a < 12; a++) S.rows[tid * 13 + a] = h[a];
            S.rows[tid * 13 + 12] = z;
        }
        __syncthreads();
#pragma unroll 1
        for (int e = tid; e < n * mr; e += nt) {                 // PHt = P H^T  (23 x m)
            const int i = e / mr, r = e % mr;
            double v = 0.0;
            for (int k = 0; k < 12; k++) v += S.P[i * n + k] * S.rows[r * 13 + k];
            S.PHt[i * 22 + r] = v;
        }
        __syncthreads();
        const int ld = mr + 13;
#pragma unroll 1
        for (int e = tid; e < mr * ld; e += nt) {                // [H P H^T / R + I | h_x | h]
            const int r = e / ld, c2 = e % ld;
            double v;
            if (c2 < mr) {
                v = 0.0;
                for (int k = 0; k < 12; k++) v += S.rows[r * 13 + k] * S.PHt[k * 22 + c2];
                v = v / R + (r == c2 ? 1.0 : 0.0);
            } else {
                v = S.rows[r * 13 + (c2 - mr)];
            }
            S.aug[r * ld + c2] = v;
        }
        __syncthreads();
        ok = gj_eliminate(S.aug, mr, ld, ld, S.row_of);
        if (ok) {
#pragma unroll 1
            for (int e = tid; e < mr * 13; e += nt) {            // T = S^{-1} [h_x | h]
                const int k = e / 13, j = e % 13;
                const int pr = S.row_of[k];
                S.T[e] = S.aug[pr * ld + mr + j] / S.aug[pr * ld + k];
            }
            __syncthreads();
#pragma unroll 1
            for (int e = tid; e < n * 13; e += nt) {             // [K_x | K_h] = PHt T / R
                const int i = e / 13, j = e % 13;
                double v = 0.0;
                for (int k = 0; k < mr; k++) v += S.PHt[i * 22 + k] * S.T[k * 13 + j];
                v /= R;
                if (j < 12) S.Kx[i * 12 + j] = v; else S.Kh[i] = v;
            }
        }
    return ok;
}

template <int SOLVER, bool EXTR>
__device__ __noinline__ void solve_finish(SolveShared& S, FilterCtl* ctl, const ScanView& sc, PassLog* logs, bool rows_local) {
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5;
    constexpr int n = NDOF;
    STAMP(1);
    if (tid < 144) { const int a = tid / 12, b = tid % 12; S.HTH[tid] = S.red[a <= b ? tri12(a, b) : tri12(b, a)]; }
    if (tid < 12) S.Hth[tid] = S.red[78 + tid];
    const int effct = (int)(S.red[90] + 0.5);
    const int it = ctl->iter, max_iter = ctl->max_iter, n_pass = ctl->n_pass;
    const int searched = ctl->converge;
    const int t_in = ctl->t;
    constexpr int extr = EXTR ? 1 : 0;
    const double R = ctl->R;
    PassLog* lg = (logs && n_pass < MAX_LOGS) ? &logs[n_pass] : nullptr;
    // ------------------------------------------------------------------ invalid pass (laserMapping.cpp:708-713, esekfom.hpp:1638-1641)
    if (effct < 1) {
        if (tid == 0) {
            if (lg) {
                lg->searched = searched; lg->effct = 0; lg->res_sum = 0.0; lg->valid = 0;
                lg->converged = searched; for (int i = 0; i < XLEN; i++) lg->x_after[i] = ctl->x[i];
            }
            ctl->n_pass = n_pass + 1;
            ctl->iter = it + 1;
            if (it + 1 >= max_iter) ctl->done = 1;
        }
        return;
    }
    __syncthreads();
    if (lg) {
        if (tid < 144) lg->HtH[tid] = S.HTH[tid];
        if (tid < 12) lg->Hth[tid] = S.Hth[tid];
        if (tid == 0) { lg->searched = searched; lg->effct = effct; lg->res_sum = S.red[91]; lg->valid = 1; }
    }
    bool ok = S.prep_ok != 0;
    constexpr int ne = EXTR ? 12 : 6;       // with extrinsic_est_en == false, columns 6..11 of h_x are zero
    if (!ok) {
        // fall through to the error exit below
    } else if (effct < n && rows_local) {
        // the small-m form rebuilds the (< 23) Jacobian rows from this rank's points: only valid when all of them are here.  With
        // the scan sharded over ranks the information form below is used instead -- the same gain by the matrix-inversion lemma,
        // from the all-reduced sums alone (ADVICE r1)
        ok = solve_gain_small_m(S, ctl, sc, extr, R);
    } else if constexpr (SOLVER == 0) {
        // -------------------------------------------------------------- information form exactly as the reference, esekfom.hpp:1782-1809
        //   P_temp = (P/R)^{-1} (S.L, from solve_prepare);  P_temp[0:12,0:12] += H^T H;  P_inv = P_temp^{-1}
#pragma unroll 1
        for (int e = tid; e < n * 2 * n; e += nt) {
            const int i = e / (2 * n), j = e % (2 * n);
            double v;
            if (j < n) { v = S.L[i * n + j]; if (i < 12 && j < 12) v += S.HTH[i * 12 + j]; }
            else v = (j - n == i) ? 1.0 : 0.0;
            S.aug[e] = v;
        }
        __syncthreads();
        ok = gj_eliminate(S.aug, n, 2 * n, 2 * n, S.row_of);
        if (ok) {
            // P_inv[:, 0:12] first (one division per entry), then
            // K_h = P_inv[:, 0:12] H^T h ;  K_x[:, 0:12] = P_inv[:, 0:12] H^T H
#pragma unroll 1
            for (int e = tid; e < n * 12; e += nt) {
                const int i = e / 12, a = e % 12;
                const int pr = S.row_of[i];
                S.L[i * 12 + a] = S.aug[pr * 2 * n + n + a] / S.aug[pr * 2 * n + i];
            }
            __syncthreads();
#pragma unroll 1
            for (int e = tid; e < n * 13; e += nt) {
                const int i = e / 13, j = e % 13;
                double v = 0.0;
                for (int a = 0; a < 12; a++) v += S.L[i * 12 + a] * (j < 12 ? S.HTH[a * 12 + j] : S.Hth[a]);
                if (j < 12) S.Kx[i * 12 + j] = v; else S.Kh[i] = v;
            }
        }
    } else {
        // -------------------------------------------------------------- the same gain through one small solve.
        // With A = P/R and E = [I_12; 0]:  (A^{-1} + E M E^T)^{-1} E = A E (I + M A_11)^{-1}, hence
        //   [K_h | K_x[:, 0:12]] = (P[:, 0:12] / R) (I + H^T H P_11 / R)^{-1} [H^T h | H^T H]
        // -- algebraically identical to esekfom.hpp:1782-1809 without the two 23x23 inversions.
        // Rows/columns ne..11 of H^T H are zero when the extrinsic columns are (ne = 6): the system
        // is then block upper-triangular and only its leading ne x ne block needs eliminating.
        constexpr int ld = ne + ne + 1;                   // <= 25 columns: one lane each
        const double Rinv = 1.0 / R;
        const int nwarps = nt >> 5;
#pragma unroll 1
        for (int r = warp; r < ne; r += nwarps) {
            if (lane < ld) {
                double v;
                if (lane < ne) {
                    v = 0.0;
#pragma unroll
                    for (int k = 0; k < ne; k++) v += S.HTH[r * 12 + k] * (S.P[k * n + lane] * Rinv);
                    v += (r == lane ? 1.0 : 0.0);
                } else if (lane == ne) v = S.Hth[r];
                else v = S.HTH[r * 12 + (lane - ne - 1)];
                S.aug[r * ld + lane] = v;
            }
        }
        __syncthreads();
        if (warp == 0) {
            const bool w_ok = gj_warp_reg<ne>(S.aug, ld, ld, S.row_of, lane);
            if (lane == 0) S.m_rows = w_ok ? 1 : 0;
        }
        __syncthreads();
        ok = S.m_rows != 0;
        if (ok) {
#pragma unroll 1
            for (int k = warp; k < ne; k += nwarps) {
                if (lane <= ne) {
                    const int pr = S.row_of[k];
                    S.T[k * 13 + lane] = S.aug[pr * ld + ne + lane] / S.aug[pr * ld + k];   // column 0: for H^T h, 1..ne: for H^T H
                }
            }
            __syncthreads();
#pragma unroll 1
            for (int i = warp; i < n; i += nwarps) {
                if (lane < 13) {
                    double v = 0.0;
                    if (lane <= ne) {
#pragma unroll
                        for (int a = 0; a < ne; a++) v += (S.P[i * n + a] * Rinv) * S.T[a * 13 + lane];
                    }
                    if (lane == 0) S.Kh[i] = v; else S.Kx[i * 12 + (lane - 1)] = v;
                }
            }
        }
    }
    __syncthreads();
    STAMP(4);
    if (!ok) {
        if (tid == 0) { ctl->error = 1; ctl->done = 1; ctl->n_pass = n_pass + 1; }
        return;
    }
    // ------------------------------------------------------------------ esekfom.hpp:1815-1817
    if (tid < n) {
        double v = S.Kh[tid];
#pragma unroll
        for (int j = 0; j < 12; j++) v += S.Kx[tid * 12 + j] * S.dx_new[j];
        const double d = v - S.dx_new[tid];                   // K_h + (K_x - I) dx_new
        S.dxu[tid] = d;
        const unsigned over = __ballot_sync(0x7fffffu, fabs(d) > ctl->limit[tid]);
        if (tid == 0) S.over = over ? 1 : 0;
    }
    __syncthreads();
    STAMP(5);
    // esekfom.hpp:1818-1834 (S.over is complete: it was written before the barrier above)
    int converge = S.over ? 0 : 1;
    int t = t_in;
    if (converge) t++;
    if (!t && it == max_iter - 2) converge = 1;               // T2: force a re-search on the last pass
    const int finish = (t > 1 || it == max_iter - 1) ? 1 : 0;
    // x_.boxplus(dx_) and -- only when this pass is the last -- the congruence blocks at dx_
    // for the final covariance (esekfom.hpp:1817, 1836-1876)
    if (lane == 0) {
        if (warp < 2) {
            const int idx = warp == 0 ? 3 : 6, xo = warp == 0 ? X_ROT : X_OFFR;
            const D3 d = d3(S.dxu[idx], S.dxu[idx + 1], S.dxu[idx + 2]);
            stq(S.xnew + xo, qmul(ldq(ctl->x + xo), so3_exp(d)));                                   // SOn.hpp:233-236
            if (finish) {
                const M33 J = transpose33(A_matrix(d));
#pragma unroll 1
                for (int i = 0; i < 9; i++) S.J[warp][i] = J.m[i];
            }
        } else if (warp == 2) {
            const D3 g = S2_boxplus(ld3(ctl->x + X_GRAV), S.dxu[21], S.dxu[22]);
            st3(S.xnew + X_GRAV, g);
            if (finish) S2_congruence(g, ld3(ctl->x_prop + X_GRAV), S.dxu[21], S.dxu[22], S.M2);
        }
    }
    if (warp == 3 && lane < 15) {
        const int b = lane / 3, c = lane % 3;
        const int dof = b == 0 ? 0 : 9 + 3 * (b - 1);
        const int xo = b == 0 ? X_POS : (b == 1 ? X_OFFT : (b == 2 ? X_VEL : (b == 3 ? X_BG : X_BA)));
        S.xnew[xo + c] = ctl->x[xo + c] + S.dxu[dof + c];                                           // vect.hpp:117-119
    }
    __syncthreads();
    STAMP(6);
    if (tid < XLEN) { ctl->x[tid] = S.xnew[tid]; if (lg) lg->x_after[tid] = S.xnew[tid]; }
    if (tid == 0) {
        ctl->t = t;
        ctl->converge = converge;
        ctl->n_pass = n_pass + 1;
        ctl->iter = it + 1;
        if (finish) ctl->done = 1;
        if (lg) lg->converged = converge;
    }
    if (!finish) {
        // the reference leaves P_ = congruence-transformed P_propagated between passes
#pragma unroll 1
        for (int e = tid; e < n * n; e += nt) ctl->P[e] = S.P[e];
        STAMP(7);
        return;
    }
    // ------------------------------------------------------------------ final covariance, esekfom.hpp:1834-1927
#pragma unroll 1
    for (int e = tid; e < n * n; e += nt) S.L[e] = S.P[e];
    __syncthreads();
    apply_rows(S.L, S.P, S.J[0], S.J[1], S.M2, n, n);          // L rows from P rows
    __syncthreads();
    apply_rows(S.Kx, S.Kx, S.J[0], S.J[1], S.M2, 12, 12);      // K_x rows, first 12 columns  (threads 0..11)
    apply_cols(S.L, S.J[0], S.J[1], S.M2, 32);                 // threads 32..54
    apply_cols(S.P, S.J[0], S.J[1], S.M2, 64);                 // threads 64..86  (L rows no longer read P)
    __syncthreads();
#pragma unroll 1
    for (int e = tid; e < n * n; e += nt) {                     // P_ = L_ - K_x[:, 0:12] P_[0:12, :]
        const int i = e / n, j = e % n;
        double v = 0.0;
#pragma unroll
        for (int a = 0; a < 12; a++) v += S.Kx[i * 12 + a] * S.P[a * n + j];
        ctl->P[e] = S.L[e] - v;
    }
    STAMP(7);
}

// k_search_c -- the same search through the map's hashed cell directory: one LANE per scan point finds its cell's halo list (every
// point of the 3x3x3 block of cells around it), scores it and proves its five neighbours exact; the few points it cannot prove
// (nothing nearby, over-full cells) are pooled per block and walked through the BVH by its warps (knn_block, map.cuh).  Same neighbours, same
// distances, bit for bit.
__global__ void __maxnreg__(96) k_search_c(MapView m, ScanView sc, const FilterCtl* __restrict__ ctl) {
    __shared__ WalkPool pool;
    pdl_wait();
    pdl_launch();
    if (ctl->done || !ctl->converge) return;
    if (blockIdx.x == 0 && threadIdx.x < XLEN) const_cast<FilterCtl*>(ctl)->x_search[threadIdx.x] = ctl->x[threadIdx.x];
    if (threadIdx.x == 0) pool.n[0] = pool.n[1] = 0;
    __syncthreads();
    int phase = 0;
    const int q = sc.q_begin + blockIdx.x * SEARCH_C_THREADS + threadIdx.x;
    const bool active = q < sc.q_end;
    float wx = 0.f, wy = 0.f, wz = 0.f;
    if (active) {
        const PoseS s = load_pose(ctl->x);
        body_to_world(s, __ldg(&sc.body[q]), wx, wy, wz);
    }
    TBest kb;
    knn_block(m, active, wx, wy, wz, kb, pool, phase);
    if (!active) return;
    float4 p[KNN_K];
    const int cnt = knn_fetch(m, kb, p);
#pragma unroll
    for (int j = 0; j < KNN_K; j++) sc.nearest[(size_t)q * KNN_K + j] = p[j];
    sc.nearest_cnt[q] = cnt;
    sc.selected[q] = knn_gate(cnt, kb.d[KNN_K - 1]) ? 1 : 0;                         // laserMapping.cpp:671
}

// k_residual -- everything of h_share_model after the search (laserMapping.cpp:674-752), one
// thread per scan point, every pass: plane fit on the cached neighbours, gating, Jacobian row;
// the rows never reach memory -- they are folded into the FP64 normal equations with warp
// shuffles and one deterministic partial per block.
//
// Block 0 is the solver block: it owns no scan points.  While the other blocks work it runs the
// H-independent half of the Kalman step (solve_prepare), then waits for their tickets, reduces
// the partials in a fixed order and
//   mode 0: finishes the Kalman step of this pass on the spot (single GPU -- no extra launch),
//   mode 1: publishes the 92 sums for the all-reduce across ranks (k_solve_only follows).
// Waiting cannot deadlock: block 0 holds no resource another block needs in order to run.
__device__ __forceinline__ void mirror_result(const FilterCtl* ctl);

template <bool EXTR, int SOLVER>
__global__ void __launch_bounds__(RESID_THREADS) k_residual(ScanView sc, FilterCtl* ctl, double* __restrict__ partials,
                                                             double* red_g, int mode, PassLog* logs, P2PState* p2p) {
    __shared__ SolveShared S;
    // ctl was written by the previous pass's k_residual, which completed before this pass's k_search
    // passed its own pdl_wait(): it may be read before pdl_wait() here
    pdl_launch();               // the next pass's k_search may queue up (it waits for us at its pdl_wait)
    if (ctl->done) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int NW = RESID_THREADS / 32;
    const int nwork = (int)gridDim.x - 1;
    if (blockIdx.x > 0) {
        pdl_wait();             // this pass's k_search has published the neighbours
        const int wb = (int)blockIdx.x - 1;
        const PoseS s = load_pose(ctl->x);
        const bool searched = ctl->converge != 0;      // what this pass's k_search saw (laserMapping.cpp:667)
        double acc[3] = {0.0, 0.0, 0.0};
        // worker blocks do not use the solver's matrices: their storage stages the warps' rows
        constexpr int STAGE = 32 * RowStage<EXTR>::RS + 96;
        static_assert(offsetof(SolveShared, stage_end) - offsetof(SolveShared, P) >= sizeof(double) * NW * STAGE, "staging area too small");
        double* stage = S.P + warp * STAGE;
        const int q0 = sc.q_begin, q1 = sc.q_end;
        for (int base = q0 + wb * RESID_THREADS + warp * 32; base < q1; base += nwork * RESID_THREADS) {
            const int q = base + lane;
            double h[12]; double z = 0.0; float ar = 0.f;
            bool contrib = false;
            if (q < q1) contrib = measure_point<EXTR>(sc, q, s, searched, h, z, ar);
            warp_accumulate<EXTR>(contrib, h, z, ar, acc, lane, stage);
        }
        double (*wacc)[PSTRIDE] = reinterpret_cast<double (*)[PSTRIDE]>(S.wred);     // NW x 96 doubles
#pragma unroll
        for (int j = 0; j < 3; j++) wacc[warp][lane + 32 * j] = acc[j];
        __syncthreads();
        if (threadIdx.x < PSTRIDE) {
            double v = 0.0;
#pragma unroll
            for (int w = 0; w < NW; w++) v += wacc[w][threadIdx.x];
            partials[(size_t)wb * PSTRIDE + threadIdx.x] = v;
        }
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0) atomicAdd(&ctl->ticket, 1);
        return;
    }
    // ------------------------------------------------------------------ solver block
    STAMP(0);
    if (mode != 1) solve_prepare<SOLVER>(S, ctl);
    pdl_wait();
    STAMP(8);
    if (threadIdx.x == 0) {
        while (atomicAdd(&ctl->ticket, 0) < nwork) __nanosleep(64);
        ctl->ticket = 0;
    }
    __syncthreads();
    __threadfence();
    STAMP(9);
    {   // fixed-order reduction of the block partials: warp w takes rows w, w+NW, ...; lanes take outputs
        double a0 = 0.0, a1 = 0.0, a2 = 0.0;
#pragma unroll 8
        for (int b = warp; b < nwork; b += NW) {
            const double* row = partials + (size_t)b * PSTRIDE;
            a0 += __ldcg(&row[lane]); a1 += __ldcg(&row[lane + 32]); a2 += __ldcg(&row[lane + 64]);
        }
        double (*wacc)[PSTRIDE] = reinterpret_cast<double (*)[PSTRIDE]>(S.wred);
        wacc[warp][lane] = a0; wacc[warp][lane + 32] = a1; wacc[warp][lane + 64] = a2;
        __syncthreads();
        if (threadIdx.x < PSTRIDE) {
            double v = 0.0;
#pragma unroll
            for (int w = 0; w < NW; w++) v += wacc[w][threadIdx.x];
            S.red[threadIdx.x] = v;
            if (mode == 1 && threadIdx.x < NRED) red_g[threadIdx.x] = v;
        }
        __syncthreads();
    }
    if (mode == 1) return;
    if (mode == 2) {
        // ---- all-reduce over peer memory, fused.  Low-latency protocol: every 8-byte word that crosses NVLink carries
        // half a double and the 32-bit epoch, so the data IS the flag -- no fence, no separate flag round trip.  Each rank
        // stores its 92 sums into its slot of every rank's mailbox (its own included) and then reads the slots of its own
        // mailbox in rank order, spinning on a word until it shows this epoch: every rank adds the same numbers in the
        // same order and ends with the bit-identical sum.  Two parities: a rank can be at most one exchange ahead.
        const int nr = p2p->nranks, me = p2p->rank;
        const unsigned long long epoch = p2p->epoch + 1;
        const unsigned long long tag = (epoch & 0xffffffffull) << 32;
        const int par = (int)(epoch & 1ull);
        for (int idx = threadIdx.x; idx < nr * PSTRIDE; idx += RESID_THREADS) {
            const int r = idx / PSTRIDE, o = idx - r * PSTRIDE;
            const unsigned long long bits = (unsigned long long)__double_as_longlong(S.red[o]);
            unsigned long long* dst = reinterpret_cast<unsigned long long*>(p2p->peer_mail[r]) + (((size_t)par * nr + me) * PSTRIDE + o) * 2;
            asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(dst), "l"(tag | (bits & 0xffffffffull)) : "memory");
            asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(dst + 1), "l"(tag | (bits >> 32)) : "memory");
        }
        __syncthreads();                                  // S.red has been sent before it is overwritten with the sum
        if (threadIdx.x < PSTRIDE) {
            const unsigned long long* mail = reinterpret_cast<const unsigned long long*>(p2p->peer_mail[me]) + (size_t)par * nr * PSTRIDE * 2;
            double v = 0.0;
            bool late = false;
            for (int r = 0; r < nr; r++) {
                const unsigned long long* src = mail + ((size_t)r * PSTRIDE + threadIdx.x) * 2;
                unsigned long long lo = 0, hi = 0;
                const long long t0 = clock64();
                while (true) {
                    asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(lo) : "l"(src) : "memory");
                    asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(hi) : "l"(src + 1) : "memory");
                    if ((lo & 0xffffffff00000000ull) == tag && (hi & 0xffffffff00000000ull) == tag) break;
                    if (clock64() - t0 > 4000000000ll) { late = true; break; }      // ~2 s: a dead peer must not hang the GPU
                }
                v += __longlong_as_double((long long)((hi << 32) | (lo & 0xffffffffull)));
            }
            S.red[threadIdx.x] = v;
            if (late) ctl->error = 2;
        }
        if (threadIdx.x == 0) p2p->epoch = epoch;
        __syncthreads();
        if (ctl->error == 2) {                  // a peer never delivered: end the update here instead of solving with garbage
            if (threadIdx.x == 0) { ctl->done = 1; ctl->n_pass = ctl->n_pass + 1; }
            mirror_result(ctl);
            return;
        }
    }
    solve_finish<SOLVER, EXTR>(S, ctl, sc, logs, mode == 0);
    mirror_result(ctl);
}

// The pass that ends the update stores the result (header, state, covariance) straight into the caller-visible
// page-locked mirror over PCIe: the host then only waits for the stream instead of queueing a device-to-host copy
// behind the last kernel.  Block-wide; the block's own writes to ctl are visible after the barrier.
// mirror_copy: the copy alone, by threads 0 .. nthreads-1, after the caller's barrier.
__device__ __forceinline__ void mirror_copy(const FilterCtl* ctl, int nthreads) {
    if (!ctl->done || !ctl->host_mirror) return;
    constexpr int ND = (int)(offsetof(FilterCtl, P_prop) / sizeof(double));
    static_assert(offsetof(FilterCtl, P_prop) % sizeof(double) == 0, "mirror copies 8-byte words");
    const double* src = reinterpret_cast<const double*>(ctl);
    double* dst = reinterpret_cast<double*>(ctl->host_mirror);
    for (int i = threadIdx.x; i < ND; i += nthreads) dst[i] = src[i];
}
__device__ __forceinline__ void mirror_result(const FilterCtl* ctl) {
    __syncthreads();
    mirror_copy(ctl, blockDim.x);
}

// multi-GPU: the Kalman step from the all-reduced sums
template <bool EXTR, int SOLVER>
__global__ void __launch_bounds__(RESID_THREADS) k_solve_only(FilterCtl* ctl, const double* __restrict__ red_g, ScanView sc,
                                                              PassLog* logs) {
    __shared__ SolveShared S;
    pdl_wait();
    pdl_launch();
    if (ctl->done) return;
    solve_prepare<SOLVER>(S, ctl);
    if (threadIdx.x < NRED) S.red[threadIdx.x] = red_g[threadIdx.x];
    __syncthreads();
    solve_finish<SOLVER, EXTR>(S, ctl, sc, logs, false);        // multi-GPU: the rows live on several ranks
    mirror_result(ctl);
}
#undef STAMP

// Device-side rendezvous over the peer mailboxes: every rank raises its slot in every peer's barrier array and waits
// for all slots of its own.  Used by the benchmark to start a timed step on all ranks together (the first exchange
// of a pass would otherwise absorb -- and bill -- whatever skew the untimed L2 flush and the host loops left).
__global__ void k_p2p_barrier(P2PState* p2p) {
    const int nr = p2p->nranks, me = p2p->rank;
    const unsigned long long epoch = p2p->bar_epoch + 1;
    if ((int)threadIdx.x < nr) {
        asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p2p->peer_bar[threadIdx.x] + me), "l"(epoch) : "memory");
        const unsigned long long* mine = p2p->peer_bar[me] + threadIdx.x;
        unsigned long long seen = 0;
        const long long t0 = clock64();
        do {
            asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(mine) : "memory");
            if (seen >= epoch) break;
            __nanosleep(32);
        } while (clock64() - t0 < 4000000000ll);
    }
    __syncthreads();
    if (threadIdx.x == 0) p2p->bar_epoch = epoch;
}

}  // namespace fl
#include "update.cuh"
namespace fl {

// ============================================================================= map_incremental
// laserMapping.cpp:427-474: which scan points enter the map, and how.  One thread per point.
__global__ void k_map_incremental(ScanView sc, const FilterCtl* __restrict__ ctl, double fsm, int ekf_inited,
                                  float4* __restrict__ world, unsigned char* __restrict__ flag_add, unsigned char* __restrict__ flag_no) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= sc.Q) return;
    const PoseS s = load_pose(ctl->x);                                   // state_point after the update (:961)
    const float4 pb = __ldg(&sc.body[q]);
    float w[3];
    body_to_world(s, pb, w[0], w[1], w[2]);                              // pointBodyToWorld :177-186
    world[q] = make_float4(w[0], w[1], w[2], pb.w);
    int cls = 0;                                                         // 0: PointToAdd, 1: PointNoNeedDownsample, 2: neither
    const int cnt = sc.nearest_cnt[q];
    if (cnt > 0 && ekf_inited) {                                         // :438
        float mid[3];
#pragma unroll
        for (int a = 0; a < 3; a++) mid[a] = (float)(floor((double)w[a] / fsm) * fsm + 0.5 * fsm);     // :444-446
        const float dist = sq_dist3(w[0], w[1], w[2], mid[0], mid[1], mid[2]);                           // :447 calc_dist (common_lib.h:219-222)
        const float4 n0 = sc.nearest[(size_t)q * KNN_K];
        if ((double)fabsf(__fsub_rn(n0.x, mid[0])) > 0.5 * fsm && (double)fabsf(__fsub_rn(n0.y, mid[1])) > 0.5 * fsm &&
            (double)fabsf(__fsub_rn(n0.z, mid[2])) > 0.5 * fsm) {        // :448
            cls = 1;
        } else {
            bool need_add = true;
            if (cnt >= KNN_K) {                                          // :454
                for (int j = 0; j < KNN_K; j++) {
                    const float4 nj = sc.nearest[(size_t)q * KNN_K + j];
                    if (sq_dist3(nj.x, nj.y, nj.z, mid[0], mid[1], mid[2]) < dist) { need_add = false; break; }      // :455
                }
            }
            cls = need_add ? 0 : 2;
        }
    }
    flag_add[q] = cls == 0;
    flag_no[q] = cls == 1;
}

// ============================================================================= device-buffer update (fl_filter_update_device)
// What upload_state sets up on the host, from kernel arguments and the caller's x26 / P in HBM.
struct StateIn {
    double limit[NDOF];
    double R;
    int max_iter, extrinsic_est;
};
constexpr int STATE_THREADS = 256;
// which call bound the filter's scan last, as stream work records it (Filter::d_bind_[1]): a host-form call (its size is the
// host's), fl_filter_update_device (the filter's copy of the caller's scan), fl_filter_update_scan_device (the scan front end's cloud)
constexpr int BIND_HOST = 0, BIND_COPY = 1, BIND_SCAN = 2;

// Also clears k_update's publication block: its workers take a word as current when its tag equals pub_tag(nonce, pass), and
// every replay of a captured graph passes the same nonce, so words left by the previous replay would otherwise look current.
// And it clears `done` in the page-locked mirror, so download_state / get_pass_logs fetch this update's control block instead
// of trusting a result an earlier host-form update mirrored there.
// bind (fl_filter_update_device, null otherwise) receives the binding of this update: (nq, BIND_COPY), see Filter::read_binding.
// state_in: the control block and the publication block of one update, by the STATE_THREADS threads of one block.
__device__ __forceinline__ void state_in(FilterCtl* ctl, unsigned long long* pub, const double* __restrict__ x26,
                                         const double* __restrict__ P, const StateIn& s) {
    const int t = threadIdx.x;
    for (int i = t; i < NDOF * NDOF; i += STATE_THREADS) { const double v = P[i]; ctl->P[i] = v; ctl->P_prop[i] = v; }   // P_propagated = P_
    if (t < XLEN) { const double v = x26[t]; ctl->x[t] = v; ctl->x_prop[t] = v; ctl->x_search[t] = 0.0; }                 // x_propagated = x_
    if (t < NDOF) ctl->limit[t] = s.limit[t];
    if (t < 16) ctl->prof[t] = 0;
    if (t < PUB_WORDS) pub[t] = 0ull;              // tag 0 is never current: pub_tag(nonce, pass) has pass >= 1 there
    if (t == 0) {
        // esekfom.hpp:1621-1631, as upload_state
        ctl->iter = -1; ctl->t = 0; ctl->converge = 1; ctl->done = 0; ctl->n_pass = 0; ctl->error = 0; ctl->ticket = 0; ctl->gen = 0;
        ctl->max_iter = s.max_iter; ctl->extrinsic_est = s.extrinsic_est; ctl->R = s.R;
        ctl->host_mirror = nullptr;
    }
}
__global__ void __launch_bounds__(STATE_THREADS) k_state_in(FilterCtl* ctl, unsigned long long* pub, FilterCtl* mirror,
                                                            const double* __restrict__ x26, const double* __restrict__ P, StateIn s,
                                                            int* __restrict__ bind, int nq) {
    pdl_launch();           // k_update may begin launching: its pdl_wait() holds it until this grid is complete and flushed
    state_in(ctl, pub, x26, P, s);
    if (threadIdx.x == 0) {
        mirror->done = 0;
        if (bind) { bind[0] = nq; bind[1] = BIND_COPY; }
    }
}
// fl_filter_update_batch_device: block b sets up slot b of a wave from prior b of x26 / P (the wave's first prior) -- the
// batch's own control and publication blocks; the filter's page-locked mirror and its binding are not touched.
__global__ void __launch_bounds__(STATE_THREADS) k_batch_state_in(FilterCtl* ctl, unsigned long long* pub, const double* __restrict__ x26,
                                                                  const double* __restrict__ P, StateIn s) {
    pdl_launch();           // as k_state_in: k_update_batch waits in pdl_wait() for this grid
    const int b = (int)blockIdx.x;
    state_in(ctl + b, pub + (size_t)b * BATCH_PUB_WORDS, x26 + (size_t)b * XLEN, P + (size_t)b * NDOF * NDOF, s);
}

// fl_filter_update_scan_device: the scan's count, clamped to [0, n_max], becomes the filter's own (bind[0]), with the binding
// BIND_SCAN.  k_update_n reads bind[0] before its pdl_wait(): this kernel completes before k_state_in, its predecessor, starts.
__global__ void k_count_in(const int* __restrict__ n, int n_max, int* __restrict__ bind) {
    bind[0] = min(max(*n, 0), n_max);
    bind[1] = BIND_SCAN;
}

// x26 / P receive the result only when the update succeeded; status2 = (FL_OK or the error download_state reports, passes run)
__device__ __forceinline__ void state_out(const FilterCtl* __restrict__ ctl, double* __restrict__ x26, double* __restrict__ P,
                                          int* __restrict__ status2) {
    const int t = threadIdx.x;
    const int e = ctl->error;
    if (e == 0) {
        for (int i = t; i < NDOF * NDOF; i += STATE_THREADS) P[i] = ctl->P[i];
        if (t < XLEN) x26[t] = ctl->x[t];
    }
    if (t == 0) { status2[0] = e == 0 ? FL_OK : (e == 2 ? FL_ERR_NCCL : FL_ERR_STATE); status2[1] = ctl->n_pass; }
}
__global__ void __launch_bounds__(STATE_THREADS) k_state_out(const FilterCtl* __restrict__ ctl, double* __restrict__ x26,
                                                             double* __restrict__ P, int* __restrict__ status2) {
    state_out(ctl, x26, P, status2);
}
// block b: slot b of a wave into prior b of x26 / P / status2 (the wave's first)
__global__ void __launch_bounds__(STATE_THREADS) k_batch_state_out(const FilterCtl* __restrict__ ctl, double* __restrict__ x26,
                                                                   double* __restrict__ P, int* __restrict__ status2) {
    const int b = (int)blockIdx.x;
    state_out(ctl + b, x26 + (size_t)b * XLEN, P + (size_t)b * NDOF * NDOF, status2 + 2 * b);
}

// map_incremental over n_max rows with the count in device memory: rows [*n, n_max) are neither PointToAdd nor PointNoNeedDownsample
__global__ void k_flags_clear(unsigned char* __restrict__ flag_add, unsigned char* __restrict__ flag_no, const int* __restrict__ n, int n_max) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < n_max && q >= *n) { flag_add[q] = 0; flag_no[q] = 0; }
}

// ============================================================================= NCCL (lazy)
struct NcclUniqueId { char internal[128]; };
struct NcclApi {
    void* lib = nullptr;
    int (*GetUniqueId)(NcclUniqueId*) = nullptr;
    int (*CommInitRank)(void**, int, NcclUniqueId, int) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
static NcclApi* load_nccl() {
    static NcclApi api;
    if (api.lib) return &api;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* nm : names) { api.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL); if (api.lib) break; }
    if (!api.lib) { set_last_error("NCCL: cannot dlopen libnccl.so.2: %s", dlerror()); return nullptr; }
    api.GetUniqueId = (int (*)(NcclUniqueId*))dlsym(api.lib, "ncclGetUniqueId");
    api.CommInitRank = (int (*)(void**, int, NcclUniqueId, int))dlsym(api.lib, "ncclCommInitRank");
    api.AllReduce = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))dlsym(api.lib, "ncclAllReduce");
    api.CommDestroy = (int (*)(void*))dlsym(api.lib, "ncclCommDestroy");
    api.GetErrorString = (const char* (*)(int))dlsym(api.lib, "ncclGetErrorString");
    if (!api.GetUniqueId || !api.CommInitRank || !api.AllReduce || !api.CommDestroy) {
        set_last_error("NCCL: missing symbols in libnccl");
        api.lib = nullptr;
        return nullptr;
    }
    return &api;
}
int nccl_unique_id(void* out128) {
    NcclApi* api = load_nccl();
    if (!api) return FL_ERR_NCCL;
    NcclUniqueId id;
    int rc = api->GetUniqueId(&id);
    if (rc != 0) { set_last_error("ncclGetUniqueId failed: %d", rc); return FL_ERR_NCCL; }
    memcpy(out128, &id, 128);
    return FL_OK;
}

// ============================================================================= Filter (host)
Filter::Filter(Map* map, int max_points) : map_(map), max_points_(max_points) {
    memset(&scan_, 0, sizeof(scan_));
    for (int i = 0; i < NDOF; i++) limit_[i] = 0.001;      // epsi, laserMapping.cpp:826-827
}
Filter::~Filter() {
    cudaSetDevice(map_->device());
    if (comm_ && nccl_) nccl_->CommDestroy(comm_);
    for (int r = 0; r < P2P_MAX_RANKS; r++) if (peer_ptr_[r]) cudaIpcCloseMemHandle(peer_ptr_[r]);
    mailbox_.release(); p2p_.release();
    body_.release(); nearest_.release(); nearest_cnt_.release(); selected_.release(); normvec_.release(); plane_.release(); srange_.release();
    partials_.release(); red_.release(); ctl_.release(); ctl0_.release(); logs_.release(); pub_.release(); rows_.release();
    mi_world_.release(); mi_flag_add_.release(); mi_flag_no_.release(); mi_list_add_.release(); mi_list_no_.release(); mi_tmp_.release(); mi_counts_.release();
    d_bind_.release();
    b_body_.release(); b_ctl_.release(); b_pub_.release(); b_partials_.release();
    b_nearest_.release(); b_nearest_cnt_.release(); b_selected_.release(); b_plane_.release(); b_srange_.release();
    if (h_ctl_) cudaFreeHost(h_ctl_);
    if (ev0_) cudaEventDestroy(ev0_);
    if (ev1_) cudaEventDestroy(ev1_);
}

int Filter::init() {
    FL_CUDA(cudaSetDevice(map_->device()));
    if (const char* e = getenv("FASTLIO_B200_NO_PDL")) pdl_ = !(e[0] == '1');      // A/B switches for tuning
    if (const char* e = getenv("FASTLIO_B200_NO_MIRROR")) mirror_ = !(e[0] == '1');
    if (const char* e = getenv("FASTLIO_B200_SEARCH")) search_mode_ = atoi(e) ? 1 : 0;
    FL_CHECK(ctl_.reserve(sizeof(FilterCtl)));
    FL_CHECK(ctl0_.reserve(sizeof(FilterCtl)));
    FL_CHECK(red_.reserve(sizeof(double) * PSTRIDE));
    FL_CHECK(logs_.reserve(sizeof(PassLog) * MAX_LOGS));
    FL_CHECK(pub_.reserve(512));
    FL_CUDA(cudaMemsetAsync(pub_.ptr, 0, 512, stream()));
    FL_CUDA(cudaMallocHost(&h_ctl_, sizeof(FilterCtl)));
    memset(h_ctl_, 0, sizeof(FilterCtl));
    FL_CUDA(cudaMemsetAsync(ctl_.ptr, 0, sizeof(FilterCtl), stream()));
    FL_CUDA(cudaMemsetAsync(ctl0_.ptr, 0, sizeof(FilterCtl), stream()));
    FL_CUDA(cudaMemsetAsync(logs_.ptr, 0, sizeof(PassLog) * MAX_LOGS, stream()));
    // k_search: as many co-resident blocks as fit (queries are spread over all of them);
    // k_residual: one thread per point, at most max_resid_grid_ blocks (one partial row each)
    int dev = map_->device(), occ = 0;
    FL_CUDA(cudaDeviceGetAttribute(&sms_, cudaDevAttrMultiProcessorCount, dev));
    if (const char* e = getenv("FASTLIO_B200_SEARCH_OCC")) search_occ_ = atoi(e);      // A/B: 4 (62 regs), 5 (<= 51) or 6 (<= 42) blocks per SM
    if (search_occ_ == 6) FL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_search<6>, SEARCH_THREADS, 0));
    else if (search_occ_ == 5) FL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_search<5>, SEARCH_THREADS, 0));
    else FL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_search<4>, SEARCH_THREADS, 0));
    search_grid_max_ = sms_ * std::max(1, occ);
    if (const char* e = getenv("FASTLIO_B200_LEGACY")) fused_ = !(e[0] == '1');      // A/B: the split kernels of round 1
    // co-resident blocks of every update kernel (the solver block and its workers wait for each other).  The one-thread k_update
    // forms count at least one block per SM; a k_update_n form runs its host form's tiles, so it is capped at that form's grid.
    const void* const upd_fn[UK_COUNT][2] = {      // [UpdKernel][EXTR]
        {(const void*)k_update<false, 1>, (const void*)k_update<true, 1>}, {(const void*)k_update<false, 2>, (const void*)k_update<true, 2>},
        {(const void*)k_update_n<false, 1>, (const void*)k_update_n<true, 1>}, {(const void*)k_update_n<false, 2>, (const void*)k_update_n<true, 2>},
        {(const void*)k_update_wave<false>, (const void*)k_update_wave<true>}, {(const void*)k_update_n_wave<false>, (const void*)k_update_n_wave<true>},
        {(const void*)k_update_batch<false>, (const void*)k_update_batch<true>}};
    const void* const upd_fn_det[UK_COUNT][2] = {  // the keyed-tie-rule forms: a kernel's cap holds for both of its forms
        {(const void*)k_update_det<false, 1>, (const void*)k_update_det<true, 1>}, {(const void*)k_update_det<false, 2>, (const void*)k_update_det<true, 2>},
        {(const void*)k_update_n_det<false, 1>, (const void*)k_update_n_det<true, 1>}, {(const void*)k_update_n_det<false, 2>, (const void*)k_update_n_det<true, 2>},
        {(const void*)k_update_wave_det<false>, (const void*)k_update_wave_det<true>}, {(const void*)k_update_n_wave_det<false>, (const void*)k_update_n_wave_det<true>},
        {(const void*)k_update_batch_det<false>, (const void*)k_update_batch_det<true>}};
    upd_caps_.threads = UPD_THREADS;
    upd_caps_.wave_smem = (int)sizeof(WavePoint);      // a wave block's tile of points in dynamic shared memory
    for (int k = 0; k < UK_COUNT; k++)
        for (int e = 0; e < 2; e++) {
            const int smem = k == UK_WAVE || k == UK_N_WAVE ? upd_caps_.wave_smem : 0;
            if (smem) FL_CUDA(cudaFuncSetAttribute(upd_fn[k][e], cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
            if (smem) FL_CUDA(cudaFuncSetAttribute(upd_fn_det[k][e], cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
            FL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, upd_fn[k][e], upd_kernel_pair(k) * UPD_THREADS, smem));
            int occ_det = 0;
            FL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_det, upd_fn_det[k][e], upd_kernel_pair(k) * UPD_THREADS, smem));
            occ = std::min(occ, occ_det);
            int& cap = upd_caps_.blocks[k][e];
            cap = sms_ * (k == UK_UPDATE1 || k == UK_N1 ? std::max(1, occ) : occ);
            const int host = k == UK_N1 ? UK_UPDATE1 : k == UK_N2 ? UK_UPDATE2 : k == UK_N_WAVE ? UK_WAVE : -1;
            if (host >= 0) cap = std::min(cap, upd_caps_.blocks[host][e]);
        }
    {
        const int* wave = upd_caps_.blocks[UK_WAVE];
        const size_t bytes = sizeof(unsigned long long) * 2 * PSTRIDE * (size_t)std::max(1, std::max(wave[0], wave[1]));
        FL_CHECK(rows_.reserve(bytes));
        FL_CUDA(cudaMemsetAsync(rows_.ptr, 0, bytes, stream()));     // tag 0: never current (row_tag)
    }
    FL_CHECK(d_bind_.reserve(2 * sizeof(int)));
    FL_CUDA(cudaMemsetAsync(d_bind_.ptr, 0, 2 * sizeof(int), stream()));
    FL_CHECK(partials_.reserve(sizeof(double) * PSTRIDE * (size_t)std::max(upd_caps_.blocks[UK_UPDATE1][0], upd_caps_.blocks[UK_UPDATE1][1])));
    max_resid_grid_ = sms_;
    FL_CHECK(partials_.reserve(sizeof(double) * PSTRIDE * (size_t)max_resid_grid_));
    FL_CHECK(reserve(std::max(1, max_points_)));
    return FL_OK;
}

int Filter::reserve(int nq) {
    FL_CHECK(body_.reserve(sizeof(float4) * (size_t)nq));
    FL_CHECK(nearest_.reserve(sizeof(float4) * KNN_K * (size_t)nq));
    { const size_t had = nearest_cnt_.bytes; FL_CHECK(nearest_cnt_.reserve(sizeof(int) * (size_t)nq)); if (nearest_cnt_.bytes != had) FL_CUDA(cudaMemsetAsync(nearest_cnt_.ptr, 0, nearest_cnt_.bytes, stream())); }
    FL_CHECK(selected_.reserve((size_t)nq));
    FL_CHECK(normvec_.reserve(sizeof(float4) * (size_t)nq));
    scan_.nearest = nearest_.as<float4>();
    scan_.nearest_cnt = nearest_cnt_.as<int>();
    scan_.selected = selected_.as<unsigned char>();
    scan_.normvec = normvec_.as<float4>();
    FL_CHECK(plane_.reserve(sizeof(float4) * (size_t)nq));
    scan_.plane = plane_.as<float4>();
    FL_CHECK(srange_.reserve(sizeof(double) * (size_t)nq));
    scan_.srange = srange_.as<double>();
    // map_incremental's buffers, so that its device form never allocates for a scan within capacity()
    FL_CHECK(mi_world_.reserve(sizeof(float4) * (size_t)nq));
    FL_CHECK(mi_flag_add_.reserve((size_t)nq));
    FL_CHECK(mi_flag_no_.reserve((size_t)nq));
    FL_CHECK(mi_list_add_.reserve(sizeof(float4) * (size_t)nq));
    FL_CHECK(mi_list_no_.reserve(sizeof(float4) * (size_t)nq));
    FL_CHECK(mi_counts_.reserve(sizeof(int) * 2));
    size_t tmp = 0;
    FL_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp, (const float4*)nullptr, (const unsigned char*)nullptr, (float4*)nullptr, (int*)nullptr, nq));
    FL_CHECK(mi_tmp_.reserve(tmp));
    return FL_OK;
}

int Filter::set_params(int max_iter, const double* limit23, int extrinsic_est_en) {
    if (max_iter < 1 || max_iter + 1 > MAX_LOGS) { set_last_error("set_params: max_iter must be in [1, %d]", MAX_LOGS - 1); return FL_ERR_ARG; }
    max_iter_ = max_iter;
    if (limit23) for (int i = 0; i < NDOF; i++) limit_[i] = limit23[i];
    extrinsic_est_ = extrinsic_est_en ? 1 : 0;
    return FL_OK;
}

int Filter::set_scan_device(const float4* d_body, int nq) {
    FL_CHECK(bind_scan(d_body, nq));
    // once a device form has bound the scan, stream work records the binding: from here on the host's (read_binding)
    if (stream_bound_) FL_CUDA(cudaMemsetAsync(d_bind_.as<int>() + 1, 0, sizeof(int), stream()));
    return FL_OK;
}
int Filter::bind_scan(const float4* d_body, int nq) {
    if (nq < 0) { set_last_error("scan: nq < 0"); return FL_ERR_ARG; }
    FL_CUDA(cudaSetDevice(map_->device()));
    FL_CHECK(reserve(std::max(1, nq)));
    scan_.body = d_body;
    scan_.Q = nq;
    if (!shard_set_) { scan_.q_begin = 0; scan_.q_end = nq; }
    dev_count_ = false;
    // per-scan state of the reference's globals: point_selected_surf is rewritten for every point
    // on the first (always searching) pass, Nearest_Points likewise
    return FL_OK;
}

int Filter::upload_scan(const float* body_xyzi, int nq) {
    if (nq < 0 || (nq > 0 && !body_xyzi)) { set_last_error("scan: bad arguments"); return FL_ERR_ARG; }
    FL_CUDA(cudaSetDevice(map_->device()));
    FL_CHECK(reserve(std::max(1, nq)));
    if (nq > 0) FL_CUDA(cudaMemcpyAsync(body_.ptr, body_xyzi, sizeof(float4) * (size_t)nq, cudaMemcpyHostToDevice, stream()));
    return set_scan_device(body_.as<float4>(), nq);
}

int Filter::set_shard(int q_begin, int q_end) {
    if (q_begin < 0 || q_end < q_begin) { set_last_error("set_shard: bad range"); return FL_ERR_ARG; }
    scan_.q_begin = q_begin; scan_.q_end = q_end;
    shard_set_ = true;
    return FL_OK;
}

int Filter::upload_state(const double* x26, const double* P, double R, bool snapshot) {
    FL_CUDA(cudaSetDevice(map_->device()));
    // h_ctl_ is the source of the upload below AND the block the device mirrors its result into: nothing queued earlier
    // on the stream may still be reading or writing it when it is rewritten
    FL_CUDA(cudaStreamSynchronize(stream()));
    // what update_iterated_dyn_share_modified sets up before its loop (esekfom.hpp:1621-1631)
    FilterCtl& c = *h_ctl_;
    c.iter = -1; c.t = 0; c.converge = 1; c.done = 0; c.n_pass = 0; c.error = 0; c.ticket = 0; c.gen = 0;
    c.max_iter = max_iter_;
    c.host_mirror = (mirror_ && !snapshot) ? h_ctl_ : nullptr;      // whole-update calls only: resident pipelines fetch the result when they want it
    c.extrinsic_est = extrinsic_est_;
    c.R = R;
    for (int i = 0; i < NDOF; i++) c.limit[i] = limit_[i];
    memcpy(c.x, x26, sizeof(double) * XLEN);
    memcpy(c.x_prop, x26, sizeof(double) * XLEN);                     // x_propagated = x_
    memcpy(c.P, P, sizeof(double) * NDOF * NDOF);
    memcpy(c.P_prop, P, sizeof(double) * NDOF * NDOF);                // P_propagated = P_
    FL_CUDA(cudaMemcpyAsync(ctl_.ptr, h_ctl_, sizeof(FilterCtl), cudaMemcpyHostToDevice, stream()));
    // the resident-timing entry points restart every repetition from this snapshot
    if (snapshot) FL_CUDA(cudaMemcpyAsync(ctl0_.ptr, ctl_.ptr, sizeof(FilterCtl), cudaMemcpyDeviceToDevice, stream()));
    return FL_OK;
}

int Filter::restore_state() {
    FL_CUDA(cudaSetDevice(map_->device()));
    FL_CUDA(cudaMemcpyAsync(ctl_.ptr, ctl0_.ptr, sizeof(FilterCtl), cudaMemcpyDeviceToDevice, stream()));
    return FL_OK;
}

template <class... KArgs, class... Args>
static cudaError_t launch_pdl_smem(void (*kernel)(KArgs...), dim3 grid, int block, size_t smem, cudaStream_t st, bool pdl, Args... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid; cfg.blockDim = dim3((unsigned)block); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl ? 1 : 0;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
template <class... KArgs, class... Args>
static cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, int block, cudaStream_t st, bool pdl, Args... args) {
    return launch_pdl_smem(kernel, grid, block, 0, st, pdl, args...);
}

// Nearest_Points of the points other ranks own: the same search, with the state the last searching pass used, on this rank's
// (identical) map replica -- bit-identical to what the owning rank cached.
int Filter::complete_neighbours() {
    if (neighbours_complete_ || (scan_.q_begin <= 0 && scan_.q_end >= scan_.Q)) { neighbours_complete_ = true; return FL_OK; }
    FL_CUDA(cudaSetDevice(map_->device()));
    const int keep_b = scan_.q_begin, keep_e = scan_.q_end;
    const int ranges[2][2] = {{0, keep_b}, {keep_e, scan_.Q}};
    for (int r = 0; r < 2; r++) {
        if (ranges[r][1] <= ranges[r][0]) continue;
        scan_.q_begin = ranges[r][0]; scan_.q_end = ranges[r][1];
        UpdArgs a = upd_args(1, 0, 1);
        a.dbg = 0; a.pose_from_search = 1;
        cudaError_t e = launch_plan(plan(UR_NEIGHBOURS, scan_.q_end - scan_.q_begin), a, stream());
        if (e != cudaSuccess) { scan_.q_begin = keep_b; scan_.q_end = keep_e; set_last_error("complete_neighbours: %s", cudaGetErrorString(e)); return FL_ERR_CUDA; }
    }
    scan_.q_begin = keep_b; scan_.q_end = keep_e;
    neighbours_complete_ = true;
    return FL_OK;
}

int Filter::run_passes() {
    FL_CUDA(cudaSetDevice(map_->device()));
    if (scan_.q_end > scan_.Q) { set_last_error("shard exceeds the scan"); return FL_ERR_ARG; }
    neighbours_complete_ = false;
    launches_ = 0;
    if (!fused() && map_->deterministic()) {
        set_last_error("update: the deterministic map mode runs k_update only; this filter uses %s",
                       solver_ != 1 ? "solver mode 0" : "the two-kernels-per-pass chain (fused 0)");
        return FL_ERR_STATE;
    }
    if (fused()) {
        cudaStream_t st = stream();
        if (nranks_ > 1 && !p2p_on_) {
            // NCCL between the measurement and the solve: one pass per launch pair
            for (int pass = 0; pass <= max_iter_; pass++) {
                FL_CHECK(launch_update(1, 1, 0));
                int rc = nccl_->AllReduce(red_.ptr, red_.ptr, NRED, /*ncclDouble*/ 8, /*ncclSum*/ 0, comm_, st);
                if (rc != 0) { set_last_error("ncclAllReduce failed: %d", rc); return FL_ERR_NCCL; }
                FL_CHECK(launch_update(1, 3, 0));
                launches_ += 2;
            }
        } else {
            FL_CHECK(launch_update(max_iter_ + 1, nranks_ > 1 ? 2 : 0, 0));
            launches_ = 1;
        }
        FL_CUDA(cudaGetLastError());
        return FL_OK;
    }
    for (int pass = 0; pass <= max_iter_; pass++) {
        FL_CHECK(launch_search_only());
        FL_CHECK(launch_residual_only());
        launches_ += 2;
        if (nranks_ > 1 && !p2p_on_) {
            cudaStream_t st = stream();
            int rc = nccl_->AllReduce(red_.ptr, red_.ptr, NRED, /*ncclDouble*/ 8, /*ncclSum*/ 0, comm_, st);
            if (rc != 0) { set_last_error("ncclAllReduce failed: %d", rc); return FL_ERR_NCCL; }
            FilterCtl* c = ctl_.as<FilterCtl>(); double* rg = red_.as<double>(); PassLog* lg = logs_.as<PassLog>();
            if (extrinsic_est_) { if (solver_) k_solve_only<true, 1><<<1, RESID_THREADS, 0, st>>>(c, rg, scan_, lg); else k_solve_only<true, 0><<<1, RESID_THREADS, 0, st>>>(c, rg, scan_, lg); }
            else { if (solver_) k_solve_only<false, 1><<<1, RESID_THREADS, 0, st>>>(c, rg, scan_, lg); else k_solve_only<false, 0><<<1, RESID_THREADS, 0, st>>>(c, rg, scan_, lg); }
            launches_++;
        }
    }
    FL_CUDA(cudaGetLastError());
    return FL_OK;
}

// the fused persistent kernel: blockIdx 0 solves, the others measure; every block must be co-resident (they wait for each other)
UpdArgs Filter::upd_args(int max_passes, int mode, int search_only) {
    UpdArgs a;
    a.m = map_->view();
    if (search_mode_ == 0) a.m.dir.cap = 0;                  // A/B: every query through the BVH walk
    a.sc = scan_; a.ctl = ctl_.as<FilterCtl>(); a.partials = partials_.as<double>(); a.red_g = red_.as<double>();
    a.logs = logs_.as<PassLog>(); a.p2p = p2p_.as<P2PState>();
    a.mode = mode; a.max_passes = max_passes; a.search_only = search_only;
    a.pub = pub_.as<unsigned long long>(); a.nonce = ++launch_nonce_;
    { const char* e = getenv("FASTLIO_B200_DBG"); a.dbg = e ? atoi(e) : 0; }
    a.pose_from_search = 0;
    return a;
}

int Filter::launch_update(int max_passes, int mode, int search_only, cudaStream_t st) {
    FL_CUDA(cudaSetDevice(map_->device()));
    FL_CUDA(launch_plan(plan((UpdRoute)mode, scan_.q_end - scan_.q_begin), upd_args(max_passes, mode, search_only), st));
    return FL_OK;
}

UpdPlan Filter::plan(UpdRoute r, int rows, int n_hyp) const {
    const char* e = getenv("FASTLIO_B200_PAIR");
    return plan_update(upd_caps_, r, rows, extrinsic_est_, e && e[0] == '1', n_hyp, map_->deterministic());
}

template <bool E>
static cudaError_t launch_upd_kernel(const UpdPlan& p, bool pdl, cudaStream_t st, const UpdArgs& a, const int* n, unsigned long long* rows, int log_stride) {
    const dim3 grid((unsigned)p.grid_x, (unsigned)p.slots);
    if (p.det) switch (p.kernel) {           // the keyed tie rule (fl_map_set_deterministic)
    case UK_UPDATE1: return launch_pdl(k_update_det<E, 1>, grid, p.block, st, pdl, a);
    case UK_UPDATE2: return launch_pdl(k_update_det<E, 2>, grid, p.block, st, pdl, a);
    case UK_N1: return launch_pdl(k_update_n_det<E, 1>, grid, p.block, st, pdl, a, n);
    case UK_N2: return launch_pdl(k_update_n_det<E, 2>, grid, p.block, st, pdl, a, n);
    case UK_WAVE: return launch_pdl_smem(k_update_wave_det<E>, grid, p.block, p.smem, st, pdl, a, rows);
    case UK_N_WAVE: return launch_pdl_smem(k_update_n_wave_det<E>, grid, p.block, p.smem, st, pdl, a, n, rows);
    case UK_BATCH: return launch_pdl(k_update_batch_det<E>, grid, p.block, st, pdl, a, log_stride);
    default: return cudaErrorInvalidValue;
    }
    switch (p.kernel) {
    case UK_UPDATE1: return launch_pdl(k_update<E, 1>, grid, p.block, st, pdl, a);
    case UK_UPDATE2: return launch_pdl(k_update<E, 2>, grid, p.block, st, pdl, a);
    case UK_N1: return launch_pdl(k_update_n<E, 1>, grid, p.block, st, pdl, a, n);
    case UK_N2: return launch_pdl(k_update_n<E, 2>, grid, p.block, st, pdl, a, n);
    case UK_WAVE: return launch_pdl_smem(k_update_wave<E>, grid, p.block, p.smem, st, pdl, a, rows);
    case UK_N_WAVE: return launch_pdl_smem(k_update_n_wave<E>, grid, p.block, p.smem, st, pdl, a, n, rows);
    case UK_BATCH: return launch_pdl(k_update_batch<E>, grid, p.block, st, pdl, a, log_stride);
    default: return cudaErrorInvalidValue;
    }
}
cudaError_t Filter::launch_plan(const UpdPlan& p, const UpdArgs& a, cudaStream_t st, const int* n, int log_stride) {
    return (extrinsic_est_ ? launch_upd_kernel<true> : launch_upd_kernel<false>)(p, pdl_ && p.pdl, st, a, n, rows_.as<unsigned long long>(), log_stride);
}

int Filter::launch_search_only() {
    FL_CUDA(cudaSetDevice(map_->device()));
    const int nq = scan_.q_end - scan_.q_begin;
    if (fused()) return launch_update(1, 0, 1);
    if (search_mode_ == 1) {
        const int cgrid = std::max(1, (nq + SEARCH_C_THREADS - 1) / SEARCH_C_THREADS);
        FL_CUDA(launch_pdl(k_search_c, cgrid, SEARCH_C_THREADS, stream(), pdl_, map_->view(), scan_, (const FilterCtl*)ctl_.as<FilterCtl>()));
        return FL_OK;
    }
    const int sgrid = std::max(1, std::min(search_grid_max_, (nq * 32 + SEARCH_THREADS - 1) / SEARCH_THREADS));
    const FilterCtl* cc = ctl_.as<FilterCtl>();
    if (search_occ_ == 6) FL_CUDA(launch_pdl(k_search<6>, sgrid, SEARCH_THREADS, stream(), pdl_, map_->view(), scan_, cc));
    else if (search_occ_ == 5) FL_CUDA(launch_pdl(k_search<5>, sgrid, SEARCH_THREADS, stream(), pdl_, map_->view(), scan_, cc));
    else FL_CUDA(launch_pdl(k_search<4>, sgrid, SEARCH_THREADS, stream(), pdl_, map_->view(), scan_, cc));
    return FL_OK;
}
int Filter::launch_residual_only() {
    FL_CUDA(cudaSetDevice(map_->device()));
    const int nq = scan_.q_end - scan_.q_begin;
    // worker blocks (one thread per point, grid-stride beyond max_resid_grid_ - 1 blocks) + the solver block 0
    resid_grid_ = std::min(max_resid_grid_ - 1, (nq + RESID_THREADS - 1) / RESID_THREADS) + 1;
    const int mode = nranks_ > 1 ? (p2p_on_ ? 2 : 1) : 0;
    P2PState* p2p = p2p_.as<P2PState>();
    FilterCtl* c = ctl_.as<FilterCtl>(); double* pp = partials_.as<double>(); double* rg = red_.as<double>(); PassLog* lg = logs_.as<PassLog>();
    cudaStream_t st = stream();
    if (extrinsic_est_) {
        if (solver_) FL_CUDA(launch_pdl(k_residual<true, 1>, resid_grid_, RESID_THREADS, st, pdl_, scan_, c, pp, rg, mode, lg, p2p));
        else FL_CUDA(launch_pdl(k_residual<true, 0>, resid_grid_, RESID_THREADS, st, pdl_, scan_, c, pp, rg, mode, lg, p2p));
    } else {
        if (solver_) FL_CUDA(launch_pdl(k_residual<false, 1>, resid_grid_, RESID_THREADS, st, pdl_, scan_, c, pp, rg, mode, lg, p2p));
        else FL_CUDA(launch_pdl(k_residual<false, 0>, resid_grid_, RESID_THREADS, st, pdl_, scan_, c, pp, rg, mode, lg, p2p));
    }
    FL_CUDA(cudaGetLastError());
    return FL_OK;
}
int Filter::sync() {
    FL_CUDA(cudaSetDevice(map_->device()));
    FL_CUDA(cudaStreamSynchronize(stream()));
    return FL_OK;
}

int Filter::download_state(double* x26, double* P, int* n_pass) {
    FL_CUDA(cudaSetDevice(map_->device()));
    FL_CUDA(cudaStreamSynchronize(stream()));
    if (!(mirror_ && h_ctl_->done)) {                   // nothing ran since the upload (or the mirror is off): fetch the block
        FL_CUDA(cudaMemcpyAsync(h_ctl_, ctl_.ptr, offsetof(FilterCtl, P_prop), cudaMemcpyDeviceToHost, stream()));
        FL_CUDA(cudaStreamSynchronize(stream()));
    }
    if (h_ctl_->error) {
        const int e = h_ctl_->error;
        set_last_error(e == 2 ? "update: a peer rank never delivered its sums (peer-memory exchange timed out)"
                              : (e == 3 ? "update: a block gave up waiting for the solver / the workers on the device" : "update: singular system on device"));
        return e == 2 ? FL_ERR_NCCL : FL_ERR_STATE;
    }
    if (x26) memcpy(x26, h_ctl_->x, sizeof(double) * XLEN);
    if (P) memcpy(P, h_ctl_->P, sizeof(double) * NDOF * NDOF);
    if (n_pass) *n_pass = h_ctl_->n_pass;
    return FL_OK;
}

int Filter::update(const float* body_xyzi, int nq, double* x26, double* P, double R, double* solve_time_s) {
    return update_any(body_xyzi, nullptr, nq, x26, P, R, solve_time_s);
}
int Filter::update_device(const float4* d_body, int nq, double* x26, double* P, double R, double* solve_time_s) {
    if (nq > 0 && !d_body) { set_last_error("update: null device scan"); return FL_ERR_ARG; }
    return update_any(nullptr, d_body, nq, x26, P, R, solve_time_s);
}
int Filter::update_any(const float* body_xyzi, const float4* d_body, int nq, double* x26, double* P, double R, double* solve_time_s) {
    if (!x26 || !P) { set_last_error("update: null state"); return FL_ERR_ARG; }
    FL_CUDA(cudaSetDevice(map_->device()));
    if (solve_time_s && !ev0_) { FL_CUDA(cudaEventCreate(&ev0_)); FL_CUDA(cudaEventCreate(&ev1_)); }
    if (solve_time_s) FL_CUDA(cudaEventRecord(ev0_, stream()));
    const auto h0 = std::chrono::steady_clock::now();
    if (d_body) FL_CHECK(set_scan_device(d_body, nq));
    else FL_CHECK(upload_scan(body_xyzi, nq));
    FL_CHECK(upload_state(x26, P, R, false));
    const auto h1 = std::chrono::steady_clock::now();
    FL_CHECK(run_passes());
    if (solve_time_s) FL_CUDA(cudaEventRecord(ev1_, stream()));
    const auto h2 = std::chrono::steady_clock::now();
    FL_CHECK(download_state(x26, P, nullptr));
    const auto h3 = std::chrono::steady_clock::now();
    // host-side anatomy of the last call (tuning aid, fl_filter_debug_prof slots 12..15): ns spent enqueueing the uploads,
    // enqueueing the passes, and waiting for the result
    host_ns_[0] = std::chrono::duration_cast<std::chrono::nanoseconds>(h1 - h0).count();
    host_ns_[1] = std::chrono::duration_cast<std::chrono::nanoseconds>(h2 - h1).count();
    host_ns_[2] = std::chrono::duration_cast<std::chrono::nanoseconds>(h3 - h2).count();
    host_ns_[3] = std::chrono::duration_cast<std::chrono::nanoseconds>(h3 - h0).count();
    if (solve_time_s) {
        float ms = 0.f;
        FL_CUDA(cudaEventElapsedTime(&ms, ev0_, ev1_));
        *solve_time_s += ms * 1e-3;                       // the reference accumulates into solve_time (esekfom.hpp:1926)
    }
    return FL_OK;
}

// ----------------------------------------------------------------------------- device-buffer forms
int Filter::capacity() const {
    size_t c = body_.bytes / sizeof(float4);
    c = std::min(c, nearest_.bytes / (sizeof(float4) * KNN_K));
    c = std::min(c, nearest_cnt_.bytes / sizeof(int));
    c = std::min(c, selected_.bytes);
    c = std::min(c, normvec_.bytes / sizeof(float4));
    c = std::min(c, plane_.bytes / sizeof(float4));
    c = std::min(c, srange_.bytes / sizeof(double));
    c = std::min(c, mi_world_.bytes / sizeof(float4));
    c = std::min(c, std::min(mi_flag_add_.bytes, mi_flag_no_.bytes));
    c = std::min(c, std::min(mi_list_add_.bytes, mi_list_no_.bytes) / sizeof(float4));
    return (int)std::min<size_t>(c, INT_MAX);
}

int Filter::device_form_scope(const char* what, bool update) const {
    if (shard_set_ || nranks_ > 1 || p2p_on_) {
        set_last_error("%s: a sharded filter (set_shard / comm_init / p2p_connect) has no device-buffer form", what);
        return FL_ERR_STATE;
    }
    if (update && !fused()) {
        set_last_error("%s: the device-buffer form runs k_update only; this filter uses %s", what,
                       solver_ != 1 ? "solver mode 0" : "the two-kernels-per-pass chain (fused 0)");
        return FL_ERR_STATE;
    }
    return FL_OK;
}

StateIn Filter::state_in_args(double R) const {
    StateIn s;
    for (int i = 0; i < NDOF; i++) s.limit[i] = limit_[i];
    s.R = R; s.max_iter = max_iter_; s.extrinsic_est = extrinsic_est_;
    return s;
}

int Filter::update_on_stream(const float* d_body, int nq, double* d_x26, double* d_P, double R, int* d_status2, cudaStream_t st) {
    const int dev = map_->device();
    if (nq < 0 || (nq > 0 && !device_ptr(d_body, dev, 16)) || !device_ptr(d_x26, dev, 8) || !device_ptr(d_P, dev, 8) ||
        !device_ptr(d_status2, dev, 4)) {
        set_last_error("update_device: nq < 0, or a buffer is not device memory on device %d (scan 16-byte, x and P 8-byte, "
                       "status 4-byte aligned)", dev);
        return FL_ERR_ARG;
    }
    FL_CHECK(device_form_scope("update_device", true));
    if (nq > capacity()) {
        set_last_error("update_device: %d points exceed the filter's capacity of %d (max_points, or the largest scan so far)", nq, capacity());
        return FL_ERR_CAPACITY;
    }
    FL_CUDA(cudaSetDevice(dev));
    bool joined = false;
    FL_CHECK(map_->query_begin(st, &joined));
    FL_CHECK(bind_scan(body_.as<float4>(), nq));             // within capacity: binds, allocates nothing
    stream_bound_ = true;
    if (nq > 0) FL_CUDA(cudaMemcpyAsync(body_.ptr, d_body, sizeof(float4) * (size_t)nq, cudaMemcpyDeviceToDevice, st));
    k_state_in<<<1, STATE_THREADS, 0, st>>>(ctl_.as<FilterCtl>(), pub_.as<unsigned long long>(), h_ctl_, d_x26, d_P, state_in_args(R),
                                            d_bind_.as<int>(), nq);
    FL_CUDA(cudaGetLastError());
    // run_passes's fused single-rank branch, on `st`
    neighbours_complete_ = false;
    FL_CHECK(launch_update(max_iter_ + 1, 0, 0, st));
    launches_ = 1;
    k_state_out<<<1, STATE_THREADS, 0, st>>>(ctl_.as<FilterCtl>(), d_x26, d_P, d_status2);
    return map_->query_end(st, joined);
}

int Filter::update_scan_on_stream(const float4* d_body, const int* d_n, int n_max, double* d_x26, double* d_P, double R, int* d_status2,
                                  cudaStream_t st) {
    const int dev = map_->device();
    if (!device_ptr(d_x26, dev, 8) || !device_ptr(d_P, dev, 8) || !device_ptr(d_status2, dev, 4)) {
        set_last_error("update_scan_device: a buffer is not device memory on device %d (x and P 8-byte, status 4-byte aligned)", dev);
        return FL_ERR_ARG;
    }
    FL_CHECK(device_form_scope("update_scan_device", true));
    if (n_max > capacity()) {
        set_last_error("update_scan_device: the scan's n_max of %d exceeds the filter's capacity of %d (max_points, or the largest scan so far)",
                       n_max, capacity());
        return FL_ERR_CAPACITY;
    }
    FL_CUDA(cudaSetDevice(dev));
    bool joined = false;
    FL_CHECK(map_->query_begin(st, &joined));
    FL_CHECK(bind_scan(d_body, n_max));                      // within capacity: binds, allocates nothing
    dev_count_ = true;
    q_max_ = n_max;
    scan_body_ = d_body;
    stream_bound_ = true;
    // the count is the filter's own from here on (later host-form calls read it back)
    k_count_in<<<1, 1, 0, st>>>(d_n, n_max, d_bind_.as<int>());
    k_state_in<<<1, STATE_THREADS, 0, st>>>(ctl_.as<FilterCtl>(), pub_.as<unsigned long long>(), h_ctl_, d_x26, d_P, state_in_args(R), nullptr, 0);
    FL_CUDA(cudaGetLastError());
    neighbours_complete_ = false;
    // k_update_n over the row bound: the workers of the host form at n_max rows (tile t to block t, as at the count), one or
    // two threads per point as the host form picks at n_max -- both forms give the same bytes
    FL_CUDA(launch_plan(plan(UR_DEVICE_COUNT, n_max), upd_args(max_iter_ + 1, 0, 0), st, d_bind_.as<int>()));
    launches_ = 1;
    k_state_out<<<1, STATE_THREADS, 0, st>>>(ctl_.as<FilterCtl>(), d_x26, d_P, d_status2);
    return map_->query_end(st, joined);
}

// ----------------------------------------------------------------------------- batched update (fl_filter_update_batch_device)
// Each hypothesis runs with the single form's workers, so its tiles, partial rows and sums are those of fl_filter_update_device;
// a wave holds as many hypotheses as fit the co-resident k_update_batch grid (plan_update, UR_BATCH).
int Filter::batch_plan(int nq, int n_hyp, int* workers, int* slots, int* waves) const {
    if (nq < 0 || n_hyp < 0) { set_last_error("batch_plan: nq and n_hyp must be >= 0"); return FL_ERR_ARG; }
    const UpdPlan p = plan(UR_BATCH, nq, n_hyp);
    if (!p.slots) {
        set_last_error("batch_plan: a hypothesis takes %d blocks, %d k_update_batch blocks are co-resident", p.grid_x,
                       upd_caps_.blocks[UK_BATCH][extrinsic_est_ ? 1 : 0]);
        return FL_ERR_CAPACITY;
    }
    *workers = p.workers;
    *slots = p.slots;
    *waves = p.waves;
    return FL_OK;
}

int Filter::reserve_batch(int nq_max) {
    if (nq_max < 0) { set_last_error("reserve_batch: nq_max must be >= 0"); return FL_ERR_ARG; }
    if (nq_max > capacity()) {
        set_last_error("reserve_batch: %d points exceed the filter's capacity of %d (max_points, or the largest scan so far)", nq_max, capacity());
        return FL_ERR_CAPACITY;
    }
    FL_CUDA(cudaSetDevice(map_->device()));
    // the largest wave of any nq <= nq_max, under either extrinsic_est_en: slots(workers) * the largest nq with those workers
    // (a wave has at most cap slots, the zero-point scan's, and at most cap blocks, so at most cap partial rows)
    size_t rows = 1;
    int cap = 1;
    for (int e = 0; e < 2; e++) {
        const int wmax = plan_update(upd_caps_, UR_BATCH, nq_max, e, false).workers;
        for (int w = 0; w <= wmax; w++) {
            const int nq_hi = w == wmax ? nq_max : std::min(nq_max, UPD_THREADS * w);
            const UpdPlan p = plan_update(upd_caps_, UR_BATCH, nq_hi, e, false);     // w workers
            if (!p.slots) break;
            rows = std::max(rows, (size_t)p.slots * (size_t)nq_hi);
        }
        cap = std::max(cap, upd_caps_.blocks[UK_BATCH][e]);
    }
    FL_CHECK(b_body_.reserve(sizeof(float4) * (size_t)std::max(1, nq_max)));
    FL_CHECK(b_ctl_.reserve(sizeof(FilterCtl) * (size_t)cap));
    FL_CHECK(b_pub_.reserve(sizeof(unsigned long long) * BATCH_PUB_WORDS * (size_t)cap));
    FL_CHECK(b_partials_.reserve(sizeof(double) * PSTRIDE * (size_t)cap));
    FL_CHECK(b_nearest_.reserve(sizeof(float4) * KNN_K * rows));
    FL_CHECK(b_nearest_cnt_.reserve(sizeof(int) * rows));
    FL_CHECK(b_selected_.reserve(rows));
    FL_CHECK(b_plane_.reserve(sizeof(float4) * rows));
    FL_CHECK(b_srange_.reserve(sizeof(double) * rows));
    FL_CUDA(cudaMemsetAsync(b_ctl_.ptr, 0, b_ctl_.bytes, stream()));
    FL_CUDA(cudaMemsetAsync(b_pub_.ptr, 0, b_pub_.bytes, stream()));
    FL_CUDA(cudaStreamSynchronize(stream()));
    batch_nq_max_ = std::max(batch_nq_max_, nq_max);
    return FL_OK;
}

int Filter::update_batch_on_stream(const float* d_body, int nq, int n_hyp, double* d_x26, double* d_P, double R, int* d_status2,
                                   PassLog* d_logs, cudaStream_t st) {
    const int dev = map_->device();
    if (nq < 0 || n_hyp < 0 || (nq > 0 && !device_ptr(d_body, dev, 16)) ||
        (n_hyp > 0 && (!device_ptr(d_x26, dev, 8) || !device_ptr(d_P, dev, 8) || !device_ptr(d_status2, dev, 4) ||
                       (d_logs && !device_ptr(d_logs, dev, 8))))) {
        set_last_error("update_batch_device: nq or n_hyp < 0, or a buffer is not device memory on device %d (scan 16-byte, x, P and "
                       "logs 8-byte, status 4-byte aligned)", dev);
        return FL_ERR_ARG;
    }
    FL_CHECK(device_form_scope("update_batch_device", true));
    if (batch_nq_max_ < 0) { set_last_error("update_batch_device: call fl_filter_reserve_batch first"); return FL_ERR_STATE; }
    if (nq > batch_nq_max_) {
        set_last_error("update_batch_device: %d points exceed the %d fl_filter_reserve_batch sized", nq, batch_nq_max_);
        return FL_ERR_CAPACITY;
    }
    int workers = 0, slots = 0, waves = 0;
    FL_CHECK(batch_plan(nq, n_hyp, &workers, &slots, &waves));      // FL_ERR_CAPACITY where one hypothesis does not fit
    if (n_hyp == 0) return FL_OK;
    UpdPlan p = plan(UR_BATCH, nq, n_hyp);
    FL_CUDA(cudaSetDevice(dev));
    bool joined = false;
    FL_CHECK(map_->query_begin(st, &joined));
    if (nq > 0) FL_CUDA(cudaMemcpyAsync(b_body_.ptr, d_body, sizeof(float4) * (size_t)nq, cudaMemcpyDeviceToDevice, st));
    ScanView sc;
    memset(&sc, 0, sizeof(sc));
    sc.body = b_body_.as<float4>();
    sc.nearest = b_nearest_.as<float4>(); sc.nearest_cnt = b_nearest_cnt_.as<int>(); sc.selected = b_selected_.as<unsigned char>();
    sc.plane = b_plane_.as<float4>(); sc.srange = b_srange_.as<double>();
    sc.q_begin = 0; sc.q_end = sc.Q = nq;
    const StateIn s = state_in_args(R);
    const int log_stride = max_iter_ + 1;
    FilterCtl* ctl = b_ctl_.as<FilterCtl>();
    unsigned long long* pub = b_pub_.as<unsigned long long>();
    for (int w = 0; w < waves; w++) {
        const int h0 = w * slots, n = std::min(slots, n_hyp - h0);
        double* x = d_x26 + (size_t)h0 * XLEN;
        double* P = d_P + (size_t)h0 * NDOF * NDOF;
        k_batch_state_in<<<n, STATE_THREADS, 0, st>>>(ctl, pub, x, P, s);
        FL_CUDA(cudaGetLastError());
        UpdArgs a = upd_args(max_iter_ + 1, 0, 0);    // the map view, the search A/B switch and a fresh nonce, as the single form
        a.sc = sc; a.ctl = ctl; a.partials = b_partials_.as<double>(); a.pub = pub;
        a.logs = d_logs ? d_logs + (size_t)h0 * log_stride : nullptr;
        p.slots = n;                                  // grid.y: the hypotheses of this wave (the last may be partial)
        FL_CUDA(launch_plan(p, a, st, nullptr, log_stride));
        k_batch_state_out<<<n, STATE_THREADS, 0, st>>>(ctl, x, P, d_status2 + 2 * (size_t)h0);
        FL_CUDA(cudaGetLastError());
    }
    return map_->query_end(st, joined);
}

// Host forms after a device form: the binding the stream work recorded last is read back (once per call), so a host form after a
// graph replay runs over the replay's scan even when a host-form update was called between the capture and the replay.
int Filter::read_binding() {
    if (!stream_bound_) return FL_OK;
    FL_CUDA(cudaSetDevice(map_->device()));
    int b[2] = {0, BIND_HOST};
    FL_CUDA(cudaStreamSynchronize(stream()));
    FL_CUDA(cudaMemcpyAsync(b, d_bind_.ptr, sizeof(b), cudaMemcpyDeviceToHost, stream()));
    FL_CUDA(cudaStreamSynchronize(stream()));
    if (b[1] == BIND_HOST || shard_set_) return FL_OK;      // the host's binding stands (device forms refuse sharded filters)
    if (b[1] == BIND_SCAN) {                                // the scan front end's cloud, the count on the device
        scan_.body = scan_body_;
        dev_count_ = true;
        scan_.Q = scan_.q_end = std::max(0, std::min(b[0], q_max_));
    } else {                                                // fl_filter_update_device's copy of the caller's scan
        scan_.body = body_.as<float4>();
        dev_count_ = false;
        scan_.Q = scan_.q_end = b[0];
    }
    scan_.q_begin = 0;
    return FL_OK;
}

int Filter::get_nearest_on_stream(float* d_pts, int* d_cnt, int nq, cudaStream_t st) {
    const int dev = map_->device();
    if (nq < 0 || nq > scan_.Q) { set_last_error("get_nearest_device: nq must be in [0, %d] (the bound scan)", scan_.Q); return FL_ERR_ARG; }
    if (nq > 0 && (!device_ptr(d_pts, dev, 16) || !device_ptr(d_cnt, dev, 4))) {
        set_last_error("get_nearest_device: the buffers must be device memory on device %d (points 16-byte aligned)", dev);
        return FL_ERR_ARG;
    }
    FL_CHECK(device_form_scope("get_nearest_device", false));
    if (nq == 0) return FL_OK;
    FL_CUDA(cudaSetDevice(dev));
    bool joined = false;
    FL_CHECK(map_->query_begin(st, &joined));
    FL_CUDA(cudaMemcpyAsync(d_pts, scan_.nearest, sizeof(float4) * KNN_K * (size_t)nq, cudaMemcpyDeviceToDevice, st));
    FL_CUDA(cudaMemcpyAsync(d_cnt, scan_.nearest_cnt, sizeof(int) * (size_t)nq, cudaMemcpyDeviceToDevice, st));
    return map_->query_end(st, joined);
}

int Filter::get_selected_on_stream(unsigned char* d_out, int nq, cudaStream_t st) {
    const int dev = map_->device();
    if (nq < 0 || nq > scan_.Q) { set_last_error("get_selected_device: nq must be in [0, %d] (the bound scan)", scan_.Q); return FL_ERR_ARG; }
    if (nq > 0 && !device_ptr(d_out, dev, 1)) { set_last_error("get_selected_device: the buffer must be device memory on device %d", dev); return FL_ERR_ARG; }
    FL_CHECK(device_form_scope("get_selected_device", false));
    if (nq == 0) return FL_OK;
    FL_CUDA(cudaSetDevice(dev));
    bool joined = false;
    FL_CHECK(map_->query_begin(st, &joined));
    FL_CUDA(cudaMemcpyAsync(d_out, scan_.selected, (size_t)nq, cudaMemcpyDeviceToDevice, st));
    return map_->query_end(st, joined);
}

int Filter::map_incremental(double fsm, int ekf_inited, int* n_to_add, int* n_no_downsample, int* added) {
    if (n_to_add) *n_to_add = 0;
    if (n_no_downsample) *n_no_downsample = 0;
    if (added) *added = 0;
    FL_CHECK(read_binding());
    const int nq = scan_.Q;
    if (nq <= 0) return FL_OK;
    if (!(fsm > 0.0)) { set_last_error("map_incremental: filter_size_map_min must be > 0"); return FL_ERR_ARG; }
    FL_CUDA(cudaSetDevice(map_->device()));
    FL_CHECK(complete_neighbours());          // sharded update: every rank must classify the WHOLE scan the same way
    cudaStream_t st = stream();
    FL_CHECK(mi_world_.reserve(sizeof(float4) * (size_t)nq));
    FL_CHECK(mi_flag_add_.reserve((size_t)nq));
    FL_CHECK(mi_flag_no_.reserve((size_t)nq));
    FL_CHECK(mi_list_add_.reserve(sizeof(float4) * (size_t)nq));
    FL_CHECK(mi_list_no_.reserve(sizeof(float4) * (size_t)nq));
    FL_CHECK(mi_counts_.reserve(sizeof(int) * 2));
    k_map_incremental<<<(nq + 255) / 256, 256, 0, st>>>(scan_, ctl_.as<FilterCtl>(), fsm, ekf_inited, mi_world_.as<float4>(),
                                                       mi_flag_add_.as<unsigned char>(), mi_flag_no_.as<unsigned char>());
    FL_CUDA(cudaGetLastError());
    // order-preserving compaction: Add_Points is sequential in the batch order (ikd_Tree.cpp:487)
    size_t tmp = 0;
    FL_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp, mi_world_.as<float4>(), mi_flag_add_.as<unsigned char>(), mi_list_add_.as<float4>(),
                                       mi_counts_.as<int>(), nq, st));
    FL_CHECK(mi_tmp_.reserve(tmp));
    tmp = mi_tmp_.bytes;
    FL_CUDA(cub::DeviceSelect::Flagged(mi_tmp_.ptr, tmp, mi_world_.as<float4>(), mi_flag_add_.as<unsigned char>(), mi_list_add_.as<float4>(),
                                       mi_counts_.as<int>(), nq, st));
    tmp = mi_tmp_.bytes;
    FL_CUDA(cub::DeviceSelect::Flagged(mi_tmp_.ptr, tmp, mi_world_.as<float4>(), mi_flag_no_.as<unsigned char>(), mi_list_no_.as<float4>(),
                                       mi_counts_.as<int>() + 1, nq, st));
    int counts[2] = {0, 0};
    FL_CUDA(cudaMemcpyAsync(counts, mi_counts_.ptr, sizeof(counts), cudaMemcpyDeviceToHost, st));
    FL_CUDA(cudaStreamSynchronize(st));
    if (n_to_add) *n_to_add = counts[0];
    if (n_no_downsample) *n_no_downsample = counts[1];
    int a = 0, b = 0;
    FL_CHECK(map_->add_points_device(mi_list_add_.as<float4>(), counts[0], true, &a));      // :470
    FL_CHECK(map_->add_points_device(mi_list_no_.as<float4>(), counts[1], false, &b));      // :471
    if (added) *added = a;
    return FL_OK;
}

int Filter::map_incremental_on_stream(double fsm, int ekf_inited, int* d_out4, cudaStream_t st) {
    const int dev = map_->device();
    if (!device_ptr(d_out4, dev, 4)) { set_last_error("map_incremental_device: out4 must be 4-byte aligned device memory on device %d", dev); return FL_ERR_ARG; }
    if (!(fsm > 0.0)) { set_last_error("map_incremental_device: filter_size_map_min must be > 0"); return FL_ERR_ARG; }
    FL_CHECK(device_form_scope("map_incremental_device", false));
    const int nq = dev_count_ ? q_max_ : scan_.Q;              // after update_scan_device: the row bound, the count on the device
    FL_CUDA(cudaSetDevice(dev));
    size_t tmp = 0;
    FL_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp, (const float4*)nullptr, (const unsigned char*)nullptr, (float4*)nullptr, (int*)nullptr, nq, st));
    if (nq > capacity() || tmp > mi_tmp_.bytes) {
        set_last_error("map_incremental_device: the bound scan of %d points exceeds the filter's capacity of %d", nq, capacity());
        return FL_ERR_CAPACITY;
    }
    if (nq <= 0) {                                      // the host form inserts nothing either: (0, 0, 0, FL_OK)
        bool joined = false;
        FL_CHECK(map_->query_begin(st, &joined));
        FL_CUDA(cudaMemsetAsync(d_out4, 0, 4 * sizeof(int), st));
        return map_->query_end(st, joined);
    }
    FL_CHECK(map_->async_prepare(nq, st, "map_incremental_device"));
    bool joined = false;
    FL_CHECK(map_->mutation_begin(st, &joined));
    ScanView sv = scan_;
    sv.Q = nq;
    k_map_incremental<<<(nq + 255) / 256, 256, 0, st>>>(sv, ctl_.as<FilterCtl>(), fsm, ekf_inited, mi_world_.as<float4>(),
                                                       mi_flag_add_.as<unsigned char>(), mi_flag_no_.as<unsigned char>());
    // rows from the device count on enter neither list, so the compactions below give the count-n host form's lists
    if (dev_count_) k_flags_clear<<<(nq + 255) / 256, 256, 0, st>>>(mi_flag_add_.as<unsigned char>(), mi_flag_no_.as<unsigned char>(), d_bind_.as<int>(), nq);
    FL_CUDA(cudaGetLastError());
    tmp = mi_tmp_.bytes;
    FL_CUDA(cub::DeviceSelect::Flagged(mi_tmp_.ptr, tmp, mi_world_.as<float4>(), mi_flag_add_.as<unsigned char>(), mi_list_add_.as<float4>(),
                                       mi_counts_.as<int>(), nq, st));
    tmp = mi_tmp_.bytes;
    FL_CUDA(cub::DeviceSelect::Flagged(mi_tmp_.ptr, tmp, mi_world_.as<float4>(), mi_flag_no_.as<unsigned char>(), mi_list_no_.as<float4>(),
                                       mi_counts_.as<int>() + 1, nq, st));
    const int* counts = mi_counts_.as<int>();
    FL_CHECK(map_->add_points_async(mi_list_add_.as<float4>(), counts, true, mi_list_no_.as<float4>(), counts + 1, nq, counts, d_out4, st));   // :470-471
    return map_->mutation_end(st, joined);
}

int Filter::get_nearest(float* out_pts, int* out_cnt, int nq) {
    FL_CHECK(read_binding());
    if (nq > scan_.Q) { set_last_error("get_nearest: nq exceeds the bound scan"); return FL_ERR_ARG; }
    FL_CUDA(cudaSetDevice(map_->device()));
    FL_CHECK(complete_neighbours());
    if (out_pts) FL_CUDA(cudaMemcpyAsync(out_pts, scan_.nearest, sizeof(float4) * KNN_K * (size_t)nq, cudaMemcpyDeviceToHost, stream()));
    if (out_cnt) FL_CUDA(cudaMemcpyAsync(out_cnt, scan_.nearest_cnt, sizeof(int) * (size_t)nq, cudaMemcpyDeviceToHost, stream()));
    FL_CUDA(cudaStreamSynchronize(stream()));
    return FL_OK;
}
int Filter::get_selected(unsigned char* out, int nq) {
    FL_CHECK(read_binding());
    if (nq > scan_.Q) { set_last_error("get_selected: nq exceeds the bound scan"); return FL_ERR_ARG; }
    if (scan_.q_begin > 0 || scan_.q_end < nq) {
        set_last_error("get_selected: point_selected_surf of points outside this rank's shard [%d, %d) lives on the rank that owns them", scan_.q_begin, scan_.q_end);
        return FL_ERR_STATE;
    }
    FL_CUDA(cudaSetDevice(map_->device()));
    FL_CUDA(cudaMemcpyAsync(out, scan_.selected, (size_t)nq, cudaMemcpyDeviceToHost, stream()));
    FL_CUDA(cudaStreamSynchronize(stream()));
    return FL_OK;
}
int Filter::get_pass_logs(PassLog* out, int cap, int* n) {
    FL_CHECK(read_binding());
    FL_CUDA(cudaSetDevice(map_->device()));
    FL_CUDA(cudaStreamSynchronize(stream()));
    if (!(mirror_ && h_ctl_->done)) {                   // nothing ran since the upload (or the mirror is off): fetch the block
        FL_CUDA(cudaMemcpyAsync(h_ctl_, ctl_.ptr, offsetof(FilterCtl, P_prop), cudaMemcpyDeviceToHost, stream()));
        FL_CUDA(cudaStreamSynchronize(stream()));
    }
    const int np = std::min(std::min(h_ctl_->n_pass, MAX_LOGS), cap);
    if (np > 0) {
        FL_CUDA(cudaMemcpyAsync(out, logs_.ptr, sizeof(PassLog) * (size_t)np, cudaMemcpyDeviceToHost, stream()));
        FL_CUDA(cudaStreamSynchronize(stream()));
    }
    if (n) *n = np;
    return FL_OK;
}

int Filter::p2p_local_handle(void* out64) {
    FL_CUDA(cudaSetDevice(map_->device()));
    const size_t bytes = P2P_MAIL_BYTES + sizeof(unsigned long long) * 2 * P2P_MAX_RANKS;   // mail, (unused) flags, barrier slots
    if (!mailbox_.ptr) {
        FL_CHECK(mailbox_.reserve(bytes));
        FL_CUDA(cudaMemset(mailbox_.ptr, 0, mailbox_.bytes));
    }
    cudaIpcMemHandle_t h;
    FL_CUDA(cudaIpcGetMemHandle(&h, mailbox_.ptr));
    static_assert(sizeof(h) == 64, "CUDA IPC handle size");
    memcpy(out64, &h, 64);
    return FL_OK;
}

int Filter::p2p_connect(int nranks, int rank, const void* handles64) {
    if (nranks < 1 || nranks > P2P_MAX_RANKS || rank < 0 || rank >= nranks || !handles64) { set_last_error("p2p_connect: bad arguments"); return FL_ERR_ARG; }
    if (!mailbox_.ptr) { set_last_error("p2p_connect: call p2p_local_handle first"); return FL_ERR_STATE; }
    FL_CUDA(cudaSetDevice(map_->device()));
    P2PState st;
    memset(&st, 0, sizeof(st));
    st.nranks = nranks; st.rank = rank; st.epoch = 0;
    for (int r = 0; r < nranks; r++) {
        void* base = mailbox_.ptr;
        if (r != rank) {
            cudaIpcMemHandle_t h;
            memcpy(&h, (const char*)handles64 + 64 * r, 64);
            FL_CUDA(cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess));
            peer_ptr_[r] = base;
        }
        st.peer_mail[r] = (double*)base;
        st.peer_flag[r] = (unsigned long long*)((char*)base + P2P_MAIL_BYTES);
        st.peer_bar[r] = st.peer_flag[r] + P2P_MAX_RANKS;
    }
    // NOTE the mailbox stride uses P2P_MAX_RANKS rows per parity only for the allocation size; rows are indexed [par * nranks + r]
    FL_CHECK(p2p_.reserve(sizeof(P2PState)));
    FL_CUDA(cudaMemcpy(p2p_.ptr, &st, sizeof(st), cudaMemcpyHostToDevice));
    nranks_ = nranks; rank_ = rank;
    p2p_on_ = nranks > 1;
    return FL_OK;
}

int Filter::p2p_barrier() {
    if (!p2p_on_) return FL_OK;
    FL_CUDA(cudaSetDevice(map_->device()));
    k_p2p_barrier<<<1, 32, 0, stream()>>>(p2p_.as<P2PState>());
    FL_CUDA(cudaGetLastError());
    return FL_OK;
}

int Filter::comm_init(int nranks, int rank, const void* id128) {
    if (nranks < 1 || rank < 0 || rank >= nranks) { set_last_error("comm_init: bad rank/size"); return FL_ERR_ARG; }
    nranks_ = nranks; rank_ = rank;
    if (nranks == 1) return FL_OK;
    FL_CUDA(cudaSetDevice(map_->device()));
    nccl_ = load_nccl();
    if (!nccl_) return FL_ERR_NCCL;
    NcclUniqueId id;
    memcpy(&id, id128, 128);
    int rc = nccl_->CommInitRank(&comm_, nranks, id, rank);
    if (rc != 0) { set_last_error("ncclCommInitRank failed: %d (%s)", rc, nccl_->GetErrorString ? nccl_->GetErrorString(rc) : "?"); return FL_ERR_NCCL; }
    return FL_OK;
}

}  // namespace fl
