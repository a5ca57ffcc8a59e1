// The solver pass of the wave kernels (k_update_wave, k_update_n_wave and their _det twins): sol_pass with a shorter chain from
// the rows summed to the publication.  Every double is the same operation on the same operands in the same order as in
// sol_pass (the library builds with --fmad=false and IEEE division, so a value kept in a register equals the one sol_pass
// stores and reloads), so the bits are sol_pass's: FASTLIO_B200_PAIR=1 runs k_update<EXTR, 1> with sol_pass, and the tests
// compare the two byte for byte.  What is shorter, all in warp 0:
//   * the sums: sol_gather ends after one barrier; warp 0 adds the warps' sums of the row slots itself (sol_reduce's order, from
//     +0.0), stores them at their entries of S.red and reads H^T H from it, while warps 1..3 expand S.HTH for the log off the chain;
//   * the gain: gj_cols_wave broadcasts the pivot column once per step and every lane picks the pivot itself, so a step has
//     no shuffle that waits on another; the dx_ factors, dx_new and the limits are loaded before the solve;
//   * dx_ reaches the pose lanes by shuffles instead of shared memory and a __syncwarp.
// The bookkeeping after the publication is sol_pass's.
#pragma once

namespace fl {

// gj_cols with the same pivots and the same operations: every lane takes column k with one round of independent shuffles and
// chooses the pivot itself (the first unused row with the strictly largest |c|), so the reciprocal no longer waits on the
// pivot's and the pivot value's shuffles, and the factors of the step are already there when it completes.
template <int N>
__device__ __forceinline__ bool gj_cols_wave(double (&c)[N], int* row_k, int lane) {
    unsigned used = 0;
    bool ok = true;
#pragma unroll 1
    for (int k = 0; k < N; k++) {
        double ck[N];
#pragma unroll
        for (int r = 0; r < N; r++) ck[r] = __shfl_sync(FULL, c[r], k);
        int p = 0; double best = -1.0;
#pragma unroll
        for (int r = 0; r < N; r++) {
            const double v = fabs(ck[r]);
            const bool cand = !((used >> r) & 1u) && v > best;
            best = cand ? v : best; p = cand ? r : p;
        }
        if (!(best > 0.0)) ok = false;
        double apk = 0.0, apj = 0.0;
#pragma unroll
        for (int r = 0; r < N; r++) { apk = (r == p) ? ck[r] : apk; apj = (r == p) ? c[r] : apj; }
        const double inv = 1.0 / apk;
        apj *= inv;
#pragma unroll
        for (int r = 0; r < N; r++) {
            if (r == p) c[r] = apj;
            else if (lane > k) c[r] -= ck[r] * apj;
        }
        used |= 1u << p;
        if (lane == 0) row_k[p] = k;
    }
    __syncwarp();
    return ok;
}

// sol_pass with the warp-0 chain above; the solver warps come from sol_gather, whose barrier left the warps' sums in S.wred
template <bool EXTR>
__device__ void sol_pass_wave(SolverSm& S, FilterCtl* ctl, PassLog* logs, unsigned long long* pub, unsigned tag_next) {
    constexpr int NE = EXTR ? 12 : 6;
    constexpr int n = NDOF;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const double Rinv = 1.0 / S.R;
    if (warp == 0) {
        // the same sums as sol_reduce's S.red: lane l forms those of row slots l, l + 32, ... (wave_row.cuh) and stores each at
        // its entry; the entries no slot carries hold +0.0
        constexpr int J = WaveRow<EXTR>::W / 32, S_EFFCT = wave_slot<EXTR>(90);
        double r[J];
#pragma unroll
        for (int j = 0; j < J; j++) r[j] = 0.0;
#pragma unroll
        for (int w = 0; w < UPD_WARPS; w++) {
#pragma unroll
            for (int j = 0; j < J; j++) r[j] += S.wred[w][lane + 32 * j];
        }
#pragma unroll
        for (int j = 0; j < J; j++) {
            if (lane + 32 * j < WaveRow<EXTR>::LIVE) S.red[wave_entry<EXTR>(lane + 32 * j)] = r[j];
        }
        const int effct = (int)(__shfl_sync(FULL, r[S_EFFCT / 32], S_EFFCT % 32) + 0.5);
        const int late = S.late;
        // known before the solve: u (below), the dx_ factors Pt[lane, :ne] / R, dx_new and the limit of this lane
        const int ln = lane < n ? lane : 0;
        double f[NE];
#pragma unroll
        for (int a = 0; a < NE; a++) f[a] = S.Pt[ln * n + a] * Rinv;
        const double dxn_l = S.dxn[ln], lim = S.limit[ln];
        __syncwarp();                                      // S.red
        bool ok = true;
        int finish = 0;
        if (effct >= 1 && !late) {
            // the columns of sol_pass, with H^T H read from the packed sums
            double c[NE], u[NE];
#pragma unroll
            for (int k = 0; k < NE; k++) {
                const double pk = S.Pt[k * n + (lane < NE ? lane : 0)] * Rinv;
                u[k] = lane < NE ? pk : (lane == NE ? S.dxn[k] : (k == lane - NE - 1 ? 1.0 : 0.0));
            }
#pragma unroll
            for (int r = 0; r < NE; r++) {
                double v = lane < NE ? (r == lane ? 1.0 : 0.0) : (lane == NE ? S.red[78 + r] : 0.0);
#pragma unroll
                for (int k = 0; k < NE; k++) v = fma(S.red[r <= k ? r * 12 - (r * (r - 1)) / 2 + (k - r) : k * 12 - (k * (k - 1)) / 2 + (r - k)], u[k], v);
                c[r] = lane <= 2 * NE ? v : 0.0;
            }
            ok = gj_cols_wave<NE>(c, S.row_k, lane);
            if (lane == 0) ctl->prof[4] = clock64();
            if (lane >= NE && lane <= 2 * NE) {
#pragma unroll
                for (int r = 0; r < NE; r++) S.Wm[S.row_k[r] * 13 + (lane - NE)] = c[r];
            }
            __syncwarp();
            // dx_ = (P[:, :ne] / R) v - dx_new                                                          (:1815)
            double d = 0.0;
            if (lane < n) {
#pragma unroll
                for (int a = 0; a < NE; a++) d = fma(f[a], S.Wm[a * 13], d);
                d -= dxn_l;
                S.dxu[lane] = d;
            }
            // the pose lanes' components: lanes 0 / 1 the rotations (dof 3..5, 6..8), lanes 2..7 pos and offset_T (dof 0..2, 9..11)
            const int src = lane < 2 ? 3 + 3 * lane : (lane < 5 ? lane - 2 : (lane < 8 ? lane + 4 : 0));
            const double d0 = __shfl_sync(FULL, d, src), d1 = __shfl_sync(FULL, d, src + 1), d2 = __shfl_sync(FULL, d, src + 2);
            const unsigned over = __ballot_sync(FULL, lane < n && fabs(d) > lim);                      // :1818-1825
            int converge = over ? 0 : 1;
            int t = S.t;
            if (converge) t++;
            if (!t && S.iter == S.max_iter - 2) converge = 1;
            finish = (t > 1 || S.iter == S.max_iter - 1) ? 1 : 0;
            if (lane == 0) ctl->prof[6] = clock64();
            if (ok) {
                if (lane < 2) {
                    const int xo = lane == 0 ? X_ROT : X_OFFR;
                    stq(S.xnew + xo, qmul(ldq(S.x + xo), so3_exp(d3(d0, d1, d2))));
                } else if (lane < 8) {
                    const int xo = lane < 5 ? X_POS + lane - 2 : X_OFFT + lane - 5;
                    S.xnew[xo] = S.x[xo] + d0;
                }
                __syncwarp();
                if (lane == 0) ctl->prof[10] = clock64();
                pub_publish(pub, tag_next, S.xnew, converge, finish, lane);
                if (lane == 0) {
                    ctl->prof[5] = clock64();
                    S.searched = S.converge; S.t = t; S.converge = converge;
                }
            }
        }
        if (lane == 0) { S.effct = effct; S.ok = ok ? 1 : 0; S.finish = finish; }
        if (effct < 1 || !ok || late) {
            if (lane == 0) {
                if (effct < 1 && !late) { S.iter++; if (S.iter >= S.max_iter) S.done = 1; S.searched = S.converge; }
                else { S.error = late ? (late == 2 ? 3 : 2) : 1; S.done = 1; }
            }
            __syncwarp();
            pub_publish(pub, tag_next, S.x, S.converge, S.done, lane);
        }
    }
    sol_sync();
    PassLog* lg = (logs && S.n_pass < MAX_LOGS) ? &logs[S.n_pass] : nullptr;
    if (S.effct < 1 || !S.ok || S.late) {
        if (tid == 0) {
            if (lg && S.effct < 1 && !S.late) {
                lg->searched = S.searched; lg->effct = 0; lg->res_sum = 0.0; lg->valid = 0; lg->converged = S.converge;
                for (int i = 0; i < XLEN; i++) lg->x_after[i] = S.x[i];
            }
            S.n_pass++;
            ctl->iter = S.iter; ctl->n_pass = S.n_pass; ctl->done = S.done; ctl->error = S.error;
        }
        sol_sync();
        return;
    }
    // ------------------------------------------------------------------ after the publication
    const int finish = S.finish;
    // [+] on the rest of the state; on the last pass also the congruence blocks at dx_ (:1836-1876)
    if (warp == 1 && lane < 2 && finish) {
        const int idx = lane == 0 ? 3 : 6;
        const M33 J = transpose33(A_matrix(d3(S.dxu[idx], S.dxu[idx + 1], S.dxu[idx + 2])));
#pragma unroll 1
        for (int i = 0; i < 9; i++) S.J[lane][i] = J.m[i];
    }
    if (warp == 2 && lane == 0) {
        const D3 g = S2_boxplus(ld3(S.x + X_GRAV), S.dxu[21], S.dxu[22]);                           // S2.hpp:136-142
        st3(S.xnew + X_GRAV, g);
        if (finish) S2_congruence_B(g, ld3(S.xprop + X_GRAV), S.Bprop, S.dxu[21], S.dxu[22], S.M2);
    }
    if (warp == 3 && lane < 9) {
        const int b = lane / 3, c = lane % 3;
        const int dof = 12 + 3 * b, xo = b == 0 ? X_VEL : (b == 1 ? X_BG : X_BA);
        S.xnew[xo + c] = S.x[xo + c] + S.dxu[dof + c];
    }
    if (lg) {
        if (tid >= 64 && tid < 64 + 144) lg->HtH[tid - 64] = S.HTH[tid - 64];
        if (tid >= 224 && tid < 236) lg->Hth[tid - 224] = S.red[78 + tid - 224];
        if (tid == 255) { lg->searched = S.searched; lg->effct = S.effct; lg->res_sum = S.red[91]; lg->valid = 1; lg->converged = S.converge; }
    }
    if (finish && warp >= 4) {
        // final covariance (:1834-1927):  P = T2 (Pt - (Pt[:, :ne] / R) W Pt[:ne, :]) T2^T.  The part that needs neither the new
        // state nor the congruence at dx_ is formed by warps 4..7 while warps 1..3 are still busy with those.
        const int t4 = tid - 128;
#pragma unroll 1
        for (int e = t4; e < NE * n; e += 128) {
            const int a = e / n, j = e - a * n;
            double v = 0.0;
#pragma unroll
            for (int b = 0; b < NE; b++) v = fma(S.Wm[a * 13 + 1 + b], S.Pt[b * n + j], v);
            S.Y[e] = v;
        }
        asm volatile("bar.sync 1, 128;" ::: "memory");
#pragma unroll 1
        for (int e = t4; e < n * n; e += 128) {
            const int i = e / n, j = e - i * n;
            double v = 0.0;
#pragma unroll
            for (int a = 0; a < NE; a++) v = fma(S.Pt[i * n + a] * Rinv, S.Y[a * n + j], v);
            S.W1[e] = S.Pt[e] - v;
        }
    }
    sol_sync();
    if (tid < XLEN) { ctl->x[tid] = S.xnew[tid]; if (lg) lg->x_after[tid] = S.xnew[tid]; }
    if (tid == 32) { ctl->t = S.t; ctl->converge = S.converge; ctl->iter = S.iter + 1; ctl->n_pass = S.n_pass + 1; ctl->done = finish; }
    if (!finish) {
        // the reference leaves P_ = congruence-transformed P_propagated between passes
#pragma unroll 1
        for (int e = tid; e < n * n; e += UPD_THREADS) ctl->P[e] = S.Pt[e];
    } else {
#pragma unroll 1
        for (int e = tid; e < n * n; e += UPD_THREADS) {            // rows
            const int i = e / n, j = e - i * n;
            double v;
            if (i >= 3 && i < 9) {
                const int b = i >= 6, base = 3 + 3 * b, r = i - base;
                v = S.J[b][3 * r] * S.W1[base * n + j] + S.J[b][3 * r + 1] * S.W1[(base + 1) * n + j] + S.J[b][3 * r + 2] * S.W1[(base + 2) * n + j];
            } else if (i >= 21) {
                const int r = i - 21;
                v = S.M2[2 * r] * S.W1[21 * n + j] + S.M2[2 * r + 1] * S.W1[22 * n + j];
            } else v = S.W1[e];
            S.Pt[e] = v;
        }
        sol_sync();
#pragma unroll 1
        for (int e = tid; e < n * n; e += UPD_THREADS) {            // columns
            const int i = e / n, j = e - i * n;
            const double* row = &S.Pt[i * n];
            double v;
            if (j >= 3 && j < 9) {
                const int b = j >= 6, base = 3 + 3 * b, r = j - base;
                v = S.J[b][3 * r] * row[base] + S.J[b][3 * r + 1] * row[base + 1] + S.J[b][3 * r + 2] * row[base + 2];
            } else if (j >= 21) {
                const int r = j - 21;
                v = S.M2[2 * r] * row[21] + S.M2[2 * r + 1] * row[22];
            } else v = row[j];
            ctl->P[e] = v;
        }
    }
    sol_sync();
    if (tid < XLEN) S.x[tid] = S.xnew[tid];
    if (tid == 32) { S.iter++; S.n_pass++; S.done = finish; }
    sol_sync();
}

}  // namespace fl
