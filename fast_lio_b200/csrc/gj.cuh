// Gauss-Jordan eliminations in shared memory used by the on-device Kalman step.
#pragma once
#include "common.cuh"

namespace fl {

// Gauss-Jordan with logical partial pivoting on the n x nc system [A | B] in shared memory
// (row stride ld), n <= 32, nc <= 64, any blockDim that is a multiple of 32.  Every thread
// re-derives the pivot of the step from shared memory; the pivot row and the factors of the step
// are staged before a barrier, after which warps (rows) and lanes (columns) update [A | B] in
// place, so a step costs two barriers.  On return
//   (A^{-1} B)[k][j] = a[row_of[k]][n + j] / a[row_of[k]][k].
__device__ bool gj_eliminate(double* a, int n, int nc, int ld, int* row_of) {
    __shared__ double prow[64], fcol[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    unsigned used = 0;
    bool ok = true;
    for (int k = 0; k < n; k++) {
        int p = -1; double best = 0.0;
        for (int r = 0; r < n; r++) {
            if (used >> r & 1u) continue;
            const double v = fabs(a[r * ld + k]);
            if (v > best) { best = v; p = r; }
        }
        if (p < 0) { ok = false; break; }              // uniform: every thread sees the same column
        const double inv = 1.0 / a[p * ld + k];
        for (int j = threadIdx.x; j < nc; j += blockDim.x) prow[j] = a[p * ld + j];
        for (int i = threadIdx.x; i < n; i += blockDim.x) fcol[i] = a[i * ld + k] * inv;
        __syncthreads();
        for (int i = warp; i < n; i += nwarps) {
            if (i == p) continue;
            const double f = fcol[i];
            for (int j = lane; j < nc; j += 32) a[i * ld + j] = a[i * ld + j] - f * prow[j];
        }
        if (threadIdx.x == 0) row_of[k] = p;
        used |= 1u << p;
        __syncthreads();
    }
    return ok;
}

// Gauss-Jordan for a small system (n <= 12, nc <= 32) by ONE warp, warp-synchronous: lanes own
// columns.  Column k is left untouched below/above the pivot (it is never read again), which
// removes the read/write hazard inside a step; columns < k are final and skipped.  Same result access as gj_eliminate.
__device__ bool gj_warp(double* a, int n, int nc, int ld, int* row_of, int lane) {
    unsigned used = 0;
#pragma unroll 1
    for (int k = 0; k < n; k++) {
        int p = -1; double best = 0.0;
#pragma unroll 1
        for (int r = 0; r < n; r++) {
            if (used >> r & 1u) continue;
            const double v = fabs(a[r * ld + k]);
            if (v > best) { best = v; p = r; }
        }
        if (p < 0) return false;
        const double inv = 1.0 / a[p * ld + k];
        if (lane < nc && lane > k) {                      // columns <= k are final (their pivots must stay)
            const double apj = a[p * ld + lane];
#pragma unroll 1
            for (int i = 0; i < n; i++) {
                if (i == p) continue;
                a[i * ld + lane] -= (a[i * ld + k] * inv) * apj;
            }
        }
        if (lane == 0) row_of[k] = p;
        used |= 1u << p;
        __syncwarp();
    }
    return true;
}

// Register-resident variant for N = 6 / 12: lane j keeps column j of [A | B] (nc <= 32 columns) in
// registers, the pivot column is broadcast with shuffles; the rows of a step are unrolled, the
// steps are not -- no shared-memory traffic, no dependent LDS chains, small code.
template <int N>
__device__ __forceinline__ bool gj_warp_reg(double* a, int nc, int ld, int* row_of, int lane) {
    __syncwarp();
    double c[N];
#pragma unroll
    for (int r = 0; r < N; r++) c[r] = lane < nc ? a[r * ld + lane] : 0.0;
    unsigned used = 0;
    bool ok = true;
#pragma unroll 1                                   // one compact step body, re-executed N times (instruction-cache friendly)
    for (int k = 0; k < N; k++) {
        int p = 0; double best = -1.0;
#pragma unroll
        for (int r = 0; r < N; r++) {
            const double v = fabs(c[r]);
            const bool cand = !((used >> r) & 1u) && v > best;
            best = cand ? v : best; p = cand ? r : p;
        }
        p = __shfl_sync(FULL, p, k);
        best = __shfl_sync(FULL, best, k);
        if (!(best > 0.0)) ok = false;
        double apj = 0.0;
#pragma unroll
        for (int r = 0; r < N; r++) apj = (r == p) ? c[r] : apj;
        const double inv = 1.0 / __shfl_sync(FULL, apj, k);
#pragma unroll
        for (int r = 0; r < N; r++) {
            const double ck = __shfl_sync(FULL, c[r], k);
            if (r != p && lane > k) c[r] -= (ck * inv) * apj;
        }
        used |= 1u << p;
        if (lane == 0) row_of[k] = p;
        __syncwarp();
    }
#pragma unroll
    for (int r = 0; r < N; r++) if (lane < nc) a[r * ld + lane] = c[r];
    __syncwarp();
    return ok;
}

// Gauss-Jordan with partial pivoting on [A | B], ne rows, one COLUMN per lane, rows in registers.  The pivot row is scaled to a
// unit pivot as it is chosen, so after the last step the solution row of unknown k is physical row `r` with row_k[r] == k.
template <int N>
__device__ __forceinline__ bool gj_cols(double (&c)[N], int* row_k, int lane) {
    unsigned used = 0;
    bool ok = true;
#pragma unroll 1
    for (int k = 0; k < N; k++) {
        int p = 0; double best = -1.0;
#pragma unroll
        for (int r = 0; r < N; r++) {
            const double v = fabs(c[r]);
            const bool cand = !((used >> r) & 1u) && v > best;
            best = cand ? v : best; p = cand ? r : p;
        }
        p = __shfl_sync(FULL, p, k);
        best = __shfl_sync(FULL, best, k);
        if (!(best > 0.0)) ok = false;
        double apj = 0.0;
#pragma unroll
        for (int r = 0; r < N; r++) apj = (r == p) ? c[r] : apj;
        const double inv = 1.0 / __shfl_sync(FULL, apj, k);
        apj *= inv;                                        // the scaled pivot row, this lane's column
#pragma unroll
        for (int r = 0; r < N; r++) {
            const double ck = __shfl_sync(FULL, c[r], k);
            if (r == p) c[r] = apj;
            else if (lane > k) c[r] -= ck * apj;
        }
        used |= 1u << p;
        if (lane == 0) row_k[p] = k;
    }
    __syncwarp();
    return ok;
}

}  // namespace fl
