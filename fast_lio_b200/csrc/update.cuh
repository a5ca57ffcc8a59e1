// k_update -- the whole iterated-EKF measurement update of one scan in ONE persistent kernel launch.
//
//   worker blocks (1 .. gridDim.x-1), one lane per scan point, every pass:
//       h_share_model (reference src/laserMapping.cpp:638-754) fused end to end -- body->world transform, k = 5 nearest
//       neighbours (cell directory + BVH walk, map.cuh) on the passes that search, 5-point plane fit straight from the
//       registers that hold the neighbours (esti_plane, include/common_lib.h:225-257), residual gating, Jacobian row --
//       folded into the FP64 normal equations H^T H / H^T h with one deterministic partial per block.  The rows never
//       reach memory; the neighbours are written once (map_incremental reads them, laserMapping.cpp:438-460).
//   solver block (0):
//       update_iterated_dyn_share_modified (reference include/IKFoM_toolkit/esekfom/esekfom.hpp:1619-1931) for the same
//       pass: while the workers measure it prepares everything that depends only on the state (x [-] x_prop, the manifold
//       congruence T P_prop T^T, :1651-1699); when their tickets are in it reduces the partials in a fixed order, forms
//       the gain in one warp with the system in registers, applies [+], decides convergence and PUBLISHES the new pose
//       (release store of a generation counter) -- the workers of the next pass spin on that counter, there is no
//       kernel boundary between passes.  Covariance bookkeeping and the pass log happen after the publication, off the
//       critical path.
//
// Gain.  The reference's information form (:1782-1809)   K_h = (H^T H + (P/R)^-1)^-1 H^T h,  K_x = (...)^-1 H^T H
// is evaluated through the matrix-inversion lemma on the only block H touches (ne = 6 columns, 12 with extrinsic
// estimation):   [K_h | K_x[:, :ne]] = (P[:, :ne] / R) (I + H^T H P_11 / R)^-1 [H^T h | H^T H]   -- no 23x23 inverse.
// Only  dx_ = K_h + (K_x - I) dx_new  is needed to advance the state, i.e. ONE extra right-hand side
//   v = (I + H^T H P_11 / R)^-1 (H^T h + H^T H dx_new[:ne]),   dx_ = (P[:, :ne] / R) v - dx_new,
// and K_x itself only for the covariance of the pass that ends the update (:1834-1927), which collapses to
//   P_final = T2 (P - (P[:, :ne] / R) W P[:ne, :]) T2^T,   W = (I + H^T H P_11 / R)^-1 H^T H,   T2 = congruence at dx_.
// The small-m branch of the reference (:1715-1744, fewer than 23 rows) is the same gain by the same lemma; this kernel
// uses the one form for every m >= 1 (which also makes the multi-GPU solve independent of how the rows are sharded).
// fl_filter_set_solver(0) runs the reference's two formulas literally through the legacy kernels (validation).
#pragma once

namespace fl {

constexpr int UPD_THREADS = 256;
constexpr int UPD_WARPS = UPD_THREADS / 32;

struct UpdArgs {
    MapView m;
    ScanView sc;
    FilterCtl* ctl;
    double* partials;      // [worker blocks][PSTRIDE]
    double* red_g;         // [PSTRIDE] sums of this rank (mode 1 out, mode 3 in)
    PassLog* logs;
    P2PState* p2p;
    unsigned long long* pub;   // publication block (32 words, own 256-byte line pair): the pose of the next pass as tagged words
    unsigned nonce;        // unique per launch: stale words of an earlier launch can never look current
    int mode;              // 0: single GPU; 1: workers + reduction only (ncclAllReduce follows); 2: peer-memory exchange; 3: solver only, sums from red_g
    int max_passes;        // passes this launch may run (persistent: max_iter + 1; NCCL chain: 1)
    int search_only;       // 1: the kNN phase of one searching pass alone (neighbours + gate), for timing
    int dbg;               // tuning switches (FASTLIO_B200_DBG)
    int pose_from_search;  // search_only: transform with ctl->x_search (the state of the last searching pass) instead of ctl->x
};

struct SolverSm {
    double Pp[NDOF * NDOF];        // P_propagated (fixed for the update)
    double Pt[NDOF * NDOF];        // T P_prop T^T of the current pass   (esekfom.hpp:1657-1699)
    double W1[NDOF * NDOF];        // scratch
    double Y[12 * NDOF];           // W P[:ne, :]
    double Wm[12 * 13];            // row k: [v_k | W_k,0..ne-1]
    double HTH[144];
    double wred[UPD_WARPS][PSTRIDE];
    double red[PSTRIDE];
    double x[XLEN], xprop[XLEN], xnew[XLEN];
    double dx[NDOF], dxn[NDOF], dxu[NDOF], limit[NDOF];
    double J[2][9], M2[4];
    double Bprop[6];               // S2_Bx(x_propagated.grav): fixed for the update
    double R;
    int iter, t, converge, done, n_pass, max_iter, error;
    int effct, ok, finish, searched, late;
    int row_k[12];                 // pivot row -> elimination step
};
template <bool EXTR> struct WorkerSm {
    static constexpr int STAGE = 32 * RowStage<EXTR>::RS + 96;
    double stage[UPD_WARPS][STAGE];
    double wred[UPD_WARPS][PSTRIDE];
    WalkPool walks;
    unsigned pose_bits[28];
    unsigned flags;
    int abort;
};

__device__ __forceinline__ int ld_acquire(const int* p) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(int* p, int v) { asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
constexpr long long SPIN_LIMIT = 3000000000ll;       // ~1.5 s of SM clocks: a wedged peer must not hang the GPU

// Publication of a pass's result to the worker blocks WITHOUT a fence: every 8-byte word carries 32 bits of payload and a
// 32-bit tag (launch nonce, pass number) -- the data is the flag.  Words 0..27: the 14 doubles of the pose h_share_model
// reads (pos, rot, offset_R_L_I, offset_T_L_I = x[0..13]) as halves; word 28: bit 0 converge, bit 1 done.
constexpr int PUB_WORDS = 29;
__device__ __forceinline__ unsigned pub_tag(unsigned nonce, int pass) { return (nonce << 8) | (unsigned)(pass & 0xff); }
__device__ __forceinline__ void pub_store(unsigned long long* p, unsigned tag, unsigned payload) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(((unsigned long long)tag << 32) | payload) : "memory");
}
__device__ __forceinline__ unsigned long long pub_load(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
// warp 0 of the solver block: x[0..13] and the flags, tagged for `pass`
__device__ __forceinline__ void pub_publish(unsigned long long* pub, unsigned tag, const double* x, int converge, int done, int lane) {
    if (lane < 28) {
        const unsigned long long bits = (unsigned long long)__double_as_longlong(x[lane >> 1]);
        pub_store(pub + lane, tag, (lane & 1) ? (unsigned)(bits >> 32) : (unsigned)bits);
    } else if (lane == 28) {
        pub_store(pub + 28, tag, (converge ? 1u : 0u) | (done ? 2u : 0u));
    }
}

// ============================================================================= paired search (PAIR = 2)
// In a 512-thread worker block, thread t < 256 owns point tile + t exactly as in the 256-thread block, and thread t + 256 is
// its search partner: on a searching pass both score the query's halo list, the owner its first ceil(n / 2) 8-candidate chunks
// and the partner the rest, so each thread runs about half the dependent round trips of cell_scan_list.  Each keeps the k best
// of its chunks in a TBest, and the owner then inserts the partner's k best, in order, into its own.  That is exactly
// cell_scan_list's answer: TBest keeps the first of two equal distances and refuses a slot it holds, so a whole-list scan ends
// with the k smallest distinct slots by (d2, first listing); the owner's list is that scan's state after the first half, and a
// listing of the second half that is not among the partner's k best has k distinct slots ahead of it in that half and so cannot
// be in the answer (tests/test_update_pair_merge.py checks the rule on the CPU).

// cell_scan_list over the chunks [c0, c1) of the halo list [start, start + cnt)
template <bool DET>
__device__ __forceinline__ void cell_scan_chunks(const MapView& m, int start, int cnt, int c0, int c1, float qx, float qy, float qz, TBestT<DET>& kb) {
    const int4* list = reinterpret_cast<const int4*>(m.dir.lists + start);
    int4 ia = make_int4(0, 0, 0, 0), ib = make_int4(0, 0, 0, 0);
    if (c0 < c1) {
        ia = __ldg(&list[2 * c0]);
        if (cnt - 8 * c0 > 4) ib = __ldg(&list[2 * c0 + 1]);
    }
#pragma unroll 1
    for (int c = c0; c < c1; c++) {
        const int n8 = cnt - 8 * c;                                            // candidates left, >= 1
        float4 p0, p1, p2, p3, p4, p5, p6, p7;
        p1 = p2 = p3 = p4 = p5 = p6 = p7 = make_float4(0.f, 0.f, 0.f, 0.f);  // flag 0: not a live point
        p0 = __ldg(&m.pts[ia.x]);
        if (n8 > 1) p1 = __ldg(&m.pts[ia.y]);
        if (n8 > 2) p2 = __ldg(&m.pts[ia.z]);
        if (n8 > 3) p3 = __ldg(&m.pts[ia.w]);
        if (n8 > 4) p4 = __ldg(&m.pts[ib.x]);
        if (n8 > 5) p5 = __ldg(&m.pts[ib.y]);
        if (n8 > 6) p6 = __ldg(&m.pts[ib.z]);
        if (n8 > 7) p7 = __ldg(&m.pts[ib.w]);
        int4 na = ia, nb = ib;
        if (c + 1 < c1) {
            na = __ldg(&list[2 * c + 2]);
            if (n8 > 12) nb = __ldg(&list[2 * c + 3]);
        }
        cell_consider(m, p0, ia.x, qx, qy, qz, kb);
        cell_consider(m, p1, ia.y, qx, qy, qz, kb);
        cell_consider(m, p2, ia.z, qx, qy, qz, kb);
        cell_consider(m, p3, ia.w, qx, qy, qz, kb);
        cell_consider(m, p4, ib.x, qx, qy, qz, kb);
        cell_consider(m, p5, ib.y, qx, qy, qz, kb);
        cell_consider(m, p6, ib.z, qx, qy, qz, kb);
        cell_consider(m, p7, ib.w, qx, qy, qz, kb);
        ia = na; ib = nb;
    }
}

// the partner's list, handed to its owner through the owner warp's `stage` slice (unused during the search)
struct PairXch {
    float d[KNN_K][32];
    int idx[KNN_K][32];
};

// The owner's merge: its TBest holds what cell_scan_list holds after the owner's chunks; the partner's entries go in after
// them, in the partner's order, through the same insert (equal distances keep their arrival order, a held slot is refused).
// DET: the insert ranks by the keyed order, so the merge is the k smallest of both lists under it -- the answer of the whole
// list's scan, since a listing the partner dropped has k distinct slots ahead of it under that order.
template <bool DET>
__device__ __forceinline__ void pair_merge(const MapView& m, const PairXch& X, int lane, TBestT<DET>& kb) {
#pragma unroll
    for (int j = 0; j < KNN_K; j++) {
        const float d = X.d[j][lane];
        const int i = X.idx[j][lane];
        if (i >= 0 && kb.admits(m, d, i)) kb.insert(d, i, m);
    }
}

// owner warp w and partner warp w + 8 only
__device__ __forceinline__ void pair_sync(int warp) { asm volatile("bar.sync %0, 64;" ::"r"(1 + (warp & (UPD_WARPS - 1))) : "memory"); }

// knn_block for the 512-thread block: every thread calls it; kb is the answer for owners (threadIdx.x < UPD_THREADS), the
// partner's kb is undefined.  The thread search is the paired scan above; what it cannot prove goes through the same walk pool,
// walked by all 16 warps, and pool overflow is walked by the owner's warp.  `stage` is the owner warp's stage slice.
template <bool DET>
__device__ __forceinline__ void knn_block_pair(const MapView& m, bool active, float qx, float qy, float qz, TBestT<DET>& kb, WalkPool& W,
                                               int& phase, double* stage) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const bool owner = threadIdx.x < UPD_THREADS;
    const CellDir& D = m.dir;
    kb.init();
    int ix = 0, iy = 0, iz = 0;
    bool listed = false;                             // the query's halo list was scored (by both threads of the pair)
    if (active && D.cap != 0u) {
        const float inv = D.inv_cell;
        ix = cell_coord(qx, inv); iy = cell_coord(qy, inv); iz = cell_coord(qz, inv);
        if (!(abs(ix) >= CELL_CLAMP - 1 || abs(iy) >= CELL_CLAMP - 1 || abs(iz) >= CELL_CLAMP - 1)) {
            int start, cnt;
            if (cell_list(D, cell_key(ix, iy, iz), start, cnt) > 0) {
                const int nchunks = (cnt + 7) >> 3, h = (nchunks + 1) >> 1;
                cell_scan_chunks(m, start, cnt, owner ? 0 : h, owner ? h : nchunks, qx, qy, qz, kb);
                listed = true;
            }
        }
    }
    PairXch& X = *reinterpret_cast<PairXch*>(stage);
    pair_sync(warp);                                 // the owner warp is done with its stage slice (previous tile)
    if (!owner) {
#pragma unroll
        for (int j = 0; j < KNN_K; j++) { X.d[j][lane] = kb.d[j]; X.idx[j][lane] = kb.idx[j]; }
    }
    pair_sync(warp);
    bool exact = true;
    if (owner && active) {
        exact = false;
        if (listed) {
            pair_merge(m, X, lane, kb);
            if (kb.idx[KNN_K - 1] >= 0) {
                const float g = cell_block_dist(D, qx, qy, qz, ix, iy, iz);
                exact = kb.d[KNN_K - 1] < g * g;
            }
        }
    }
    // from here on: knn_block's pool, with the pool filled by the owners only
    int mine_slot = -1;
    int* counter = &W.n[phase & 1];
    if (owner && active && !exact) {
        mine_slot = atomicAdd(counter, 1);
        if (mine_slot < WALK_POOL) {
            W.who[mine_slot] = (int)threadIdx.x; W.x[mine_slot] = qx; W.y[mine_slot] = qy; W.z[mine_slot] = qz;
            const bool full = kb.idx[KNN_K - 1] >= 0;
#pragma unroll
            for (int j = 0; j < KNN_K; j++) { W.rd[mine_slot][j] = full ? kb.d[j] : INFINITY; W.ri[mine_slot][j] = full ? kb.idx[j] : -1; }
        }
    }
    __syncthreads();
    const int total = *counter, n = min(total, WALK_POOL);
    if (threadIdx.x == 0) W.n[(phase + 1) & 1] = 0;
    phase++;
    for (int i = warp; i < n; i += nwarps) {
        KBestT<DET> w;
        w.init();
        if (lane < KNN_K) { w.d = W.rd[i][lane]; w.idx = W.ri[i][lane]; }
        w.w = __shfl_sync(FULL, w.d, KNN_K - 1);
        w.n = w.w < INFINITY ? KNN_K : 0;
        knn_query_from(m, W.x[i], W.y[i], W.z[i], w, lane);
        __syncwarp();
        if (lane < KNN_K) { W.rd[i][lane] = w.d; W.ri[i][lane] = w.idx; }
    }
    unsigned todo = __ballot_sync(FULL, mine_slot >= WALK_POOL);      // partner warps never pool: todo == 0 there
    while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        KBestT<DET> w;
        knn_query(m, __shfl_sync(FULL, qx, src), __shfl_sync(FULL, qy, src), __shfl_sync(FULL, qz, src), w, lane);
#pragma unroll
        for (int j = 0; j < KNN_K; j++) {
            const float dj = __shfl_sync(FULL, w.d, j);
            const int ij = __shfl_sync(FULL, w.idx, j);
            if (lane == src) { kb.d[j] = dj; kb.idx[j] = ij; }
        }
    }
    __syncthreads();
    if (mine_slot >= 0 && mine_slot < WALK_POOL) {
#pragma unroll
        for (int j = 0; j < KNN_K; j++) { kb.d[j] = W.rd[mine_slot][j]; kb.idx[j] = W.ri[mine_slot][j]; }
    }
    if (threadIdx.x == 0 && total && m.dir.cap && m.dir.n_walked) atomicAdd(m.dir.n_walked, total);
}

// ============================================================================= workers
// Everything of h_share_model for one scan point (laserMapping.cpp:650-692), one thread per point.  Block-collective on a
// searching pass (the queries the directory cannot prove are walked through the BVH by all warps of the block, knn_block).  On a searching pass the five neighbours go from the search's registers
// straight into the plane fit; they are stored once (map_incremental reads them, laserMapping.cpp:438-460).  Returns true when
// the point contributes a row.  PAIR = 2: the partner threads (threadIdx.x >= UPD_THREADS) call it on searching passes only,
// for the paired search, and return false.
template <bool EXTR, int PAIR, bool DET>
__device__ __forceinline__ bool measure_fused(const MapView& m, const ScanView& sc, int q, bool active, const PoseS& s, bool searched,
                                              bool search_only, WalkPool& walks, int& phase, double* stage, double* h, double& z, float& absres) {
    float4 pb = make_float4(0.f, 0.f, 0.f, 0.f);
    float wx = 0.f, wy = 0.f, wz = 0.f;
    D3 p_this = d3(0.0, 0.0, 0.0);
    if (active) {
        pb = __ldg(&sc.body[q]);
        p_this = body_to_world(s, pb, wx, wy, wz);                          // :656-661 (also the lever arm of the Jacobian, :733)
    }
    bool sel = false;
    float pabcd[4] = {0.f, 0.f, 0.f, 0.f};
    if (searched) {                                                         // :667
        TBestT<DET> kb;
        if constexpr (PAIR == 1) {
            knn_block(m, active, wx, wy, wz, kb, walks, phase);                    // :670 (block-wide: two barriers)
        } else {
            knn_block_pair(m, active, wx, wy, wz, kb, walks, phase, stage);
            if (threadIdx.x >= UPD_THREADS) return false;
        }
        if (active) {
            float4 p[KNN_K];
            const int cnt = knn_fetch(m, kb, p);
#pragma unroll
            for (int j = 0; j < KNN_K; j++) sc.nearest[(size_t)q * KNN_K + j] = p[j];
            sc.nearest_cnt[q] = cnt;
            sel = knn_gate(cnt, kb.d[KNN_K - 1]);                           // :671
            if (search_only) { sc.selected[q] = sel ? 1 : 0; return false; }
            if (sel) {
                float pn[KNN_K][3];
#pragma unroll
                for (int j = 0; j < KNN_K; j++) { pn[j][0] = p[j].x; pn[j][1] = p[j].y; pn[j][2] = p[j].z; }
                sel = esti_plane_dev(pabcd, pn, 0.1f);                      // :678
                if (sel) sc.plane[q] = make_float4(pabcd[0], pabcd[1], pabcd[2], pabcd[3]);
            }
        }
    } else if (active) {
        // a pass that does not search fits the plane to the SAME five neighbours (Nearest_Points persists, T3) and only
        // points whose fit and score succeeded last time are still selected: the fit is reused, not recomputed
        sel = sc.selected[q] != 0;                                          // :674
        if (sel) { const float4 pl = sc.plane[q]; pabcd[0] = pl.x; pabcd[1] = pl.y; pabcd[2] = pl.z; pabcd[3] = pl.w; }
    }
    bool contrib = false;
    if (active && sel) {
        const float pd2 = plane_residual(pabcd, wx, wy, wz);                                    // :680
        // sqrt(p_body.norm()) depends on the point alone: computed on the searching passes, cached for the others
        double srange;
        if (searched) { srange = sqrt(norm3(d3(pb.x, pb.y, pb.z))); sc.srange[q] = srange; }
        else srange = sc.srange[q];
        float score;
        if (score_gate(pd2, srange, score)) {                                                   // :681-683
            contrib = true;
            absres = fabsf(pd2);                                                                // res_last
            jacobian_row_at<EXTR>(s, pb, p_this, make_float4(pabcd[0], pabcd[1], pabcd[2], pd2), h, z);    // :723-751
        }
    }
    if (active) sc.selected[q] = contrib ? 1 : 0;                                               // :677, :685
    return contrib;
}

// ============================================================================= solver
// The solver runs on threads 0..255 of block 0 whatever the block size (in a 512-thread block the others leave at once), so its
// barriers name those 256 threads.
__device__ __forceinline__ void sol_sync() { asm volatile("bar.sync 2, 256;" ::: "memory"); }

// once per launch: the control block into shared memory
__device__ void sol_load(SolverSm& S, const FilterCtl* ctl) {
    const int tid = threadIdx.x;
    for (int e = tid; e < NDOF * NDOF; e += UPD_THREADS) S.Pp[e] = __ldcg(&ctl->P_prop[e]);
    if (tid < XLEN) { S.x[tid] = __ldcg(&ctl->x[tid]); S.xprop[tid] = __ldcg(&ctl->x_prop[tid]); }
    if (tid >= 32 && tid < 32 + NDOF) S.limit[tid - 32] = __ldcg(&ctl->limit[tid - 32]);
    if (tid == 64) {
        S.R = __ldcg(&ctl->R);
        S.iter = __ldcg(&ctl->iter); S.t = __ldcg(&ctl->t); S.converge = __ldcg(&ctl->converge); S.done = __ldcg(&ctl->done);
        S.n_pass = __ldcg(&ctl->n_pass); S.max_iter = __ldcg(&ctl->max_iter); S.error = 0; S.late = 0;
    }
    sol_sync();
    if (tid == 0) S2_Bx(ld3(S.xprop + X_GRAV), S.Bprop);
    sol_sync();
}

// the state-only half of a pass (esekfom.hpp:1651-1699): dx = x [-] x_prop, dx_new, the congruence blocks, Pt = T P_prop T^T
__device__ void sol_prepare(SolverSm& S) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int n = NDOF;
    if (lane == 0) {
        if (warp < 2) {                 // SO3 blocks: rot (idx 3), offset_R_L_I (idx 6)
            const int idx = warp == 0 ? 3 : 6, xo = warp == 0 ? X_ROT : X_OFFR;
            const D3 l = so3_log(qmul(qconj(ldq(S.xprop + xo)), ldq(S.x + xo)));                    // SOn.hpp:237-239
            const M33 J = transpose33(A_matrix(l));                                                 // T5
#pragma unroll 1
            for (int i = 0; i < 9; i++) S.J[warp][i] = J.m[i];
            const D3 seg = mul33v(J, l);
            S.dx[idx] = l.x; S.dx[idx + 1] = l.y; S.dx[idx + 2] = l.z;
            S.dxn[idx] = seg.x; S.dxn[idx + 1] = seg.y; S.dxn[idx + 2] = seg.z;
        } else if (warp == 2) {         // S2 block: grav (idx 21)
            double d0, d1;
            S2_boxminus_B(ld3(S.x + X_GRAV), ld3(S.xprop + X_GRAV), S.Bprop, d0, d1);
            S2_congruence_B(ld3(S.x + X_GRAV), ld3(S.xprop + X_GRAV), S.Bprop, d0, d1, S.M2);
            S.dx[21] = d0; S.dx[22] = d1;
            S.dxn[21] = S.M2[0] * d0 + S.M2[1] * d1;
            S.dxn[22] = S.M2[2] * d0 + S.M2[3] * d1;
        }
    }
    if (warp == 3 && lane < 15) {       // vect blocks: pos, offset_T_L_I, vel, bg, ba
        const int b = lane / 3, c = lane % 3;
        const int dof = b == 0 ? 0 : 9 + 3 * (b - 1);
        const int xo = b == 0 ? X_POS : (b == 1 ? X_OFFT : (b == 2 ? X_VEL : (b == 3 ? X_BG : X_BA)));
        const double d = S.x[xo + c] - S.xprop[xo + c];
        S.dx[dof + c] = d; S.dxn[dof + c] = d;
    }
    sol_sync();
    // W1 = P_prop T^T  (columns of the SO3 / S2 blocks), then Pt = T W1 (their rows): T P T^T as :1659-1699 apply it block by block
#pragma unroll 1
    for (int e = tid; e < n * n; e += UPD_THREADS) {
        const int i = e / n, j = e - i * n;
        const double* row = &S.Pp[i * n];
        double v;
        if (j >= 3 && j < 9) {
            const int b = j >= 6, base = 3 + 3 * b, r = j - base;
            v = S.J[b][3 * r] * row[base] + S.J[b][3 * r + 1] * row[base + 1] + S.J[b][3 * r + 2] * row[base + 2];
        } else if (j >= 21) {
            const int r = j - 21;
            v = S.M2[2 * r] * row[21] + S.M2[2 * r + 1] * row[22];
        } else v = row[j];
        S.W1[e] = v;
    }
    sol_sync();
#pragma unroll 1
    for (int e = tid; e < n * n; e += UPD_THREADS) {
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
}

// fixed-order reduction of the workers' block partials into S.red
__device__ void sol_reduce(SolverSm& S, const double* __restrict__ partials, int nwork) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double a0 = 0.0, a1 = 0.0, a2 = 0.0;
    for (int b = warp; b < nwork; b += 8 * UPD_WARPS) {          // eight rows per step: 24 loads in flight, then summed in row order
        double v[8][3];
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int bb = b + k * UPD_WARPS;
            const double* row = partials + (size_t)bb * PSTRIDE;
            v[k][0] = v[k][1] = v[k][2] = 0.0;
            if (bb < nwork) { v[k][0] = __ldcg(&row[lane]); v[k][1] = __ldcg(&row[lane + 32]); v[k][2] = __ldcg(&row[lane + 64]); }
        }
#pragma unroll
        for (int k = 0; k < 8; k++) { a0 += v[k][0]; a1 += v[k][1]; a2 += v[k][2]; }
    }
    S.wred[warp][lane] = a0; S.wred[warp][lane + 32] = a1; S.wred[warp][lane + 64] = a2;
    sol_sync();
    if (tid < PSTRIDE) {
        double v = 0.0;
#pragma unroll
        for (int w = 0; w < UPD_WARPS; w++) v += S.wred[w][tid];
        S.red[tid] = v;
        if (tid < 78) {                       // H^T H in full 12 x 12 form for the gain (tid -> (a <= b) of the packed upper triangle)
            int a = 0, rem = tid;
            while (rem >= 12 - a) { rem -= 12 - a; a++; }
            const int b = a + rem;
            S.HTH[a * 12 + b] = v; S.HTH[b * 12 + a] = v;
        }
    }
    sol_sync();
}
// the same expansion for sums that did not come through sol_reduce (peer exchange, NCCL)
__device__ void sol_expand(SolverSm& S) {
    const int tid = threadIdx.x;
    if (tid < 144) { const int a = tid / 12, b = tid - a * 12; S.HTH[tid] = S.red[a <= b ? tri12(a, b) : tri12(b, a)]; }
    sol_sync();
}

// all-reduce of S.red over the peer mailboxes (see k_residual / DESIGN.md section 5): every rank stores its sums into its slot
// of every rank's mailbox as epoch-tagged words and adds the slots of its own mailbox in rank order
__device__ void sol_exchange(SolverSm& S, P2PState* p2p) {
    const int nr = p2p->nranks, me = p2p->rank;
    const unsigned long long epoch = p2p->epoch + 1;
    const unsigned long long tag = (epoch & 0xffffffffull) << 32;
    const int par = (int)(epoch & 1ull);
    for (int idx = threadIdx.x; idx < nr * PSTRIDE; idx += UPD_THREADS) {
        const int r = idx / PSTRIDE, o = idx - r * PSTRIDE;
        const unsigned long long bits = (unsigned long long)__double_as_longlong(S.red[o]);
        unsigned long long* dst = reinterpret_cast<unsigned long long*>(p2p->peer_mail[r]) + (((size_t)par * nr + me) * PSTRIDE + o) * 2;
        asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(dst), "l"(tag | (bits & 0xffffffffull)) : "memory");
        asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(dst + 1), "l"(tag | (bits >> 32)) : "memory");
    }
    sol_sync();                                  // S.red has been sent before it is overwritten with the sum
    if (threadIdx.x < PSTRIDE) {
        const unsigned long long* mail = reinterpret_cast<const unsigned long long*>(p2p->peer_mail[me]) + (size_t)par * nr * PSTRIDE * 2;
        double v = 0.0;
        bool late = false;
        for (int r = 0; r < nr && !late; r++) {
            const unsigned long long* src = mail + ((size_t)r * PSTRIDE + threadIdx.x) * 2;
            unsigned long long lo = 0, hi = 0;
            const long long t0 = clock64();
            while (true) {
                asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(lo) : "l"(src) : "memory");
                asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(hi) : "l"(src + 1) : "memory");
                if ((lo & 0xffffffff00000000ull) == tag && (hi & 0xffffffff00000000ull) == tag) break;
                if (clock64() - t0 > SPIN_LIMIT) { late = true; break; }
            }
            v += __longlong_as_double((long long)((hi << 32) | (lo & 0xffffffffull)));
        }
        S.red[threadIdx.x] = v;
        if (late) S.late = 1;
    }
    if (threadIdx.x == 0) p2p->epoch = epoch;
    sol_sync();
}

// The H-dependent half of a pass (esekfom.hpp:1782-1834).  The critical path -- gain, dx_, convergence, [+] on the pose the
// measurement model reads, publication -- runs in WARP 0 ALONE, with the system in registers and no block barrier; everything
// else ([+] on velocity / biases / gravity, the log, the covariance bookkeeping and, on the pass that ends the update, the final
// covariance) follows the publication.
template <bool EXTR>
__device__ void sol_pass(SolverSm& S, FilterCtl* ctl, PassLog* logs, unsigned long long* pub, unsigned tag_next) {
    constexpr int NE = EXTR ? 12 : 6;
    constexpr int n = NDOF;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const double Rinv = 1.0 / S.R;
    if (warp == 0) {
        const int effct = (int)(S.red[90] + 0.5);
        bool ok = true;
        int finish = 0;
        if (effct >= 1 && !S.late) {
            // lane j <= 2 NE holds column j of [A | rhs | H^T H] as  base + H^T H u:
            //   j < NE   : A = I + H^T H P_11 / R          u = P_11[:, j] / R       base = e_j
            //   j == NE  : H^T h + H^T H dx_new[:ne]       u = dx_new[:ne]          base = H^T h
            //   j > NE   : H^T H                           u = e_(j - NE - 1)       base = 0
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
                for (int k = 0; k < NE; k++) v = fma(S.HTH[r * 12 + k], u[k], v);
                c[r] = lane <= 2 * NE ? v : 0.0;
            }
            ok = gj_cols<NE>(c, S.row_k, lane);
            if (lane == 0) ctl->prof[4] = clock64();
            if (lane >= NE && lane <= 2 * NE) {
#pragma unroll
                for (int r = 0; r < NE; r++) S.Wm[S.row_k[r] * 13 + (lane - NE)] = c[r];
            }
            __syncwarp();
            // dx_ = K_h + (K_x - I) dx_new = (P[:, :ne] / R) v - dx_new                                  (:1815)
            double d = 0.0;
            if (lane < n) {
#pragma unroll
                for (int a = 0; a < NE; a++) d = fma(S.Pt[lane * n + a] * Rinv, S.Wm[a * 13], d);
                d -= S.dxn[lane];
                S.dxu[lane] = d;
            }
            const unsigned over = __ballot_sync(FULL, lane < n && fabs(d) > S.limit[lane]);              // :1818-1825
            int converge = over ? 0 : 1;
            int t = S.t;
            if (converge) t++;
            if (!t && S.iter == S.max_iter - 2) converge = 1;               // T2: force a re-search on the last pass (:1829-1832)
            finish = (t > 1 || S.iter == S.max_iter - 1) ? 1 : 0;           // :1834
            __syncwarp();
            if (lane == 0) ctl->prof[6] = clock64();
            if (ok) {
                // x_.boxplus(dx_) on the pose (:1817): lanes 0 / 1 the two rotations (one instruction stream), lanes 2..7 pos, offset_T
                if (lane < 2) {
                    const int idx = lane == 0 ? 3 : 6, xo = lane == 0 ? X_ROT : X_OFFR;
                    stq(S.xnew + xo, qmul(ldq(S.x + xo), so3_exp(d3(S.dxu[idx], S.dxu[idx + 1], S.dxu[idx + 2]))));   // SOn.hpp:233-236
                } else if (lane < 8) {
                    const int b = (lane - 2) / 3, cc = (lane - 2) % 3;
                    const int dof = b == 0 ? 0 : 9, xo = b == 0 ? X_POS : X_OFFT;
                    S.xnew[xo + cc] = S.x[xo + cc] + S.dxu[dof + cc];                                                  // vect.hpp:117-119
                }
                __syncwarp();
                if (lane == 0) ctl->prof[10] = clock64();
                pub_publish(pub, tag_next, S.xnew, converge, finish, lane);
                if (lane == 0) { ctl->prof[5] = clock64(); S.searched = S.converge; S.t = t; S.converge = converge; }
            }
        }
        if (lane == 0) { S.effct = effct; S.ok = ok ? 1 : 0; S.finish = finish; }
        if (effct < 1 || !ok || S.late) {
            // ---- invalid pass (laserMapping.cpp:708-713, esekfom.hpp:1638-1641: `continue`) or a device-side failure
            if (lane == 0) {
                if (effct < 1 && !S.late) { S.iter++; if (S.iter >= S.max_iter) S.done = 1; S.searched = S.converge; }
                else { S.error = S.late ? (S.late == 2 ? 3 : 2) : 1; S.done = 1; }     // 2: a peer never delivered; 3: the workers never reported; 1: singular system
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

// ============================================================================= the kernel
// PAIR = 1: one thread per point, 256 threads, two blocks per SM.  PAIR = 2: the same 256-point tiles, dealt the same way, with a
// search partner per point (knn_block_pair): 512 threads, one block per SM, the same 128-register cap.  Warps 8..15 only help
// on the searching passes and otherwise just join the block barriers; the tiles, the partial rows and every sum are those of
// PAIR = 1, so both forms give the same bytes.
// The body is shared by k_update (the scan's points [q_begin, q_end)) and k_update_n (a point count in device memory): q1 is
// the end of the points the workers measure.
template <bool EXTR, int PAIR, bool DET = false>
__device__ __forceinline__ void update_body(const UpdArgs& a, const int q1) {
    static_assert(PAIR == 1 || PAIR == 2, "one or two threads per point");
    static_assert(sizeof(PairXch) <= sizeof(double) * WorkerSm<EXTR>::STAGE, "the partner's list fits the owner warp's stage slice");
    __shared__ __align__(16) unsigned char smem_raw[sizeof(SolverSm) > sizeof(WorkerSm<EXTR>) ? sizeof(SolverSm) : sizeof(WorkerSm<EXTR>)];
    FilterCtl* ctl = a.ctl;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nwork = (int)gridDim.x - 1;
    pdl_wait();
    pdl_launch();
    if (blockIdx.x > 0) {
        // ------------------------------------------------------------------ worker block
        WorkerSm<EXTR>& Wk = *reinterpret_cast<WorkerSm<EXTR>*>(smem_raw);
        const int wb = (int)blockIdx.x - 1;
        if (tid == 0) { Wk.abort = 0; Wk.walks.n[0] = Wk.walks.n[1] = 0; }
        __syncthreads();
        int walk_phase = 0;
        for (int p = 0; p < a.max_passes; p++) {
            PoseS s;
            bool searched;
            if (p == 0) {
                // the state this launch starts from is in the control block (uploaded / left by the previous launch)
                if (__ldcg(&ctl->done) && !a.search_only) return;      // (a search-only launch may follow a finished update)
                searched = __ldcg(&ctl->converge) != 0 || a.search_only;      // dyn_share.converge (laserMapping.cpp:667)
                s = load_pose(a.pose_from_search ? ctl->x_search : ctl->x);
            } else {
                // later passes: wait for the solver block's publication of pass p (tagged words, see pub_publish)
                const unsigned tag = pub_tag(a.nonce, p);
                if (tid == 0) {
                    const long long t0 = clock64();
                    while ((unsigned)(pub_load(a.pub + 28) >> 32) != tag) {
                        if (clock64() - t0 > SPIN_LIMIT) { Wk.abort = 1; atomicExch(&ctl->error, 3); break; }
                        __nanosleep((a.dbg & 1) ? 2000 : 100);
                    }
                }
                __syncthreads();
                if (Wk.abort) return;
                if (tid < PUB_WORDS) {
                    unsigned long long w = pub_load(a.pub + tid);
                    const long long t0 = clock64();
                    while ((unsigned)(w >> 32) != tag && clock64() - t0 < SPIN_LIMIT) w = pub_load(a.pub + tid);
                    if (tid < 28) Wk.pose_bits[tid] = (unsigned)w; else Wk.flags = (unsigned)w;
                }
                __syncthreads();
                if (Wk.flags & 2u) return;
                searched = (Wk.flags & 1u) != 0;
                double x14[14];
#pragma unroll
                for (int i = 0; i < 14; i++) x14[i] = __longlong_as_double((long long)(((unsigned long long)Wk.pose_bits[2 * i + 1] << 32) | Wk.pose_bits[2 * i]));
                s.pos = d3(x14[X_POS], x14[X_POS + 1], x14[X_POS + 2]);
                s.rot.x = x14[X_ROT]; s.rot.y = x14[X_ROT + 1]; s.rot.z = x14[X_ROT + 2]; s.rot.w = x14[X_ROT + 3];
                s.offR.x = x14[X_OFFR]; s.offR.y = x14[X_OFFR + 1]; s.offR.z = x14[X_OFFR + 2]; s.offR.w = x14[X_OFFR + 3];
                s.offT = d3(x14[X_OFFT], x14[X_OFFT + 1], x14[X_OFFT + 2]);
            }
            double acc[3] = {0.0, 0.0, 0.0};
            const bool owner = PAIR == 1 || tid < UPD_THREADS;
            double* stage = Wk.stage[warp & (UPD_WARPS - 1)];          // a partner warp hands its lists over in its owner's slice
            // tiles of UPD_THREADS consecutive points, dealt round-robin to the worker blocks -- the same tiles every pass (a point's
            // cached neighbours, plane and flag are only ever touched by its own thread)
            const int q0 = a.sc.q_begin;
            for (int tile = q0 + wb * UPD_THREADS; tile < q1; tile += nwork * UPD_THREADS) {
                const int q = tile + (tid & (UPD_THREADS - 1));
                double h[12]; double z = 0.0; float ar = 0.f;
                bool contrib = false;
                if (owner || searched)
                    contrib = measure_fused<EXTR, PAIR, DET>(a.m, a.sc, q, q < q1, s, searched, a.search_only != 0, Wk.walks, walk_phase, stage, h, z, ar);
                if (owner && !a.search_only) warp_accumulate<EXTR>(contrib, h, z, ar, acc, lane, stage);
            }
            if (a.search_only) return;
            if (owner) {
#pragma unroll
                for (int j = 0; j < 3; j++) Wk.wred[warp][lane + 32 * j] = acc[j];
            }
            __syncthreads();
            if (tid < PSTRIDE) {
                double v = 0.0;
#pragma unroll
                for (int w = 0; w < UPD_WARPS; w++) v += Wk.wred[w][tid];
                __stcg(&a.partials[(size_t)wb * PSTRIDE + tid], v);
            }
            __syncthreads();                                // the block's partial is written ...
            if (tid == 0) asm volatile("red.release.gpu.global.add.s32 [%0], 1;" ::"l"(&ctl->ticket) : "memory");      // ... and ordered before the ticket (release)
            if (a.mode == 1) return;
        }
        return;
    }
    // ------------------------------------------------------------------ solver block
    if (a.search_only) return;
    if (tid >= UPD_THREADS) return;                  // PAIR = 2: the solver is the first 256 threads (sol_sync)
    SolverSm& S = *reinterpret_cast<SolverSm*>(smem_raw);
    sol_load(S, ctl);
    int p = 0;
    for (; p < a.max_passes && !S.done; p++) {
        if (tid == 0) ctl->prof[0] = clock64();
        if (S.converge && tid < XLEN) ctl->x_search[tid] = S.x[tid];      // this pass searches: Nearest_Points will belong to this state
        if (a.mode != 1) sol_prepare(S);                 // overlaps the workers' measurement
        if (tid == 0) ctl->prof[8] = clock64();
        if (a.mode != 3) {
            if (tid == 0) {
                const long long t0 = clock64();
                while (ld_acquire(&ctl->ticket) < nwork * (p + 1)) {        // tickets only grow within a launch
                    if (clock64() - t0 > SPIN_LIMIT) { S.late = 2; break; }
                }
            }
            sol_sync();
            if (tid == 0) ctl->prof[9] = clock64();
            sol_reduce(S, a.partials, nwork);
            if (a.mode == 1) {
                if (tid < NRED) a.red_g[tid] = S.red[tid];
                if (tid == 0) ctl->ticket = 0;
                return;
            }
        } else {
            if (tid < PSTRIDE) S.red[tid] = tid < NRED ? a.red_g[tid] : 0.0;
            sol_sync();
            sol_expand(S);
        }
        if (a.mode == 2) { sol_exchange(S, a.p2p); sol_expand(S); }
        if (tid == 0) ctl->prof[1] = clock64();
        sol_pass<EXTR>(S, ctl, a.logs, a.pub, pub_tag(a.nonce, p + 1));
        if (tid == 0) ctl->prof[7] = clock64();
    }
    if (tid == 0) { ctl->error = S.error | ctl->error; ctl->ticket = 0; }
    sol_sync();
    mirror_copy(ctl, UPD_THREADS);
}

template <bool EXTR, int PAIR>
__global__ void __launch_bounds__(UPD_THREADS * PAIR, 3 - PAIR) k_update(UpdArgs a) {
    update_body<EXTR, PAIR>(a, a.sc.q_end);
}

// fl_filter_update_scan_device: the points [q_begin, min(*n, q_end)), q_end the row bound the grid was sized for.  The tiles
// below the count go to the blocks the host form gives them; blocks beyond write +0.0 partial rows, which leave sol_reduce's
// fixed-order sums (they start from +0.0) unchanged, so the result is the host form's at count *n.  *n is written before the
// kernel ahead of this one starts (fl_filter_update_scan_device copies it before k_state_in), so it may be read ahead of
// pdl_wait().
template <bool EXTR, int PAIR>
__global__ void __launch_bounds__(UPD_THREADS * PAIR, 3 - PAIR) k_update_n(UpdArgs a, const int* __restrict__ n) {
    update_body<EXTR, PAIR>(a, min(*n, a.sc.q_end));
}

// fl_filter_update_batch_device: one scan from gridDim.y priors in one launch.  Slot blockIdx.y is a whole k_update<EXTR, 1> grid
// of its own -- blockIdx.x and gridDim.x mean what they mean there, so the slot has the solver block, the workers, the tiles and
// the fixed-order sums of the single form -- with its own control block, publication block, partial rows, pass logs and
// per-point caches; the map and the scan are shared.  The slot's caches are rows [s Q, (s + 1) Q) of flat arrays, its partial
// rows start at s (gridDim.x - 1), its publication block is BATCH_PUB_WORDS words, its log entries start at s log_stride.
// Footprint: the registers (128) and shared memory of k_update<EXTR, 1>, so the same co-resident grid; the slot's pointers are
// values here rather than kernel parameters, so ptxas spills a little more (sm_90a, nvcc 12.9: stack 336 / 392 bytes against
// 288 for EXTR false / true, spill stores + loads 508 / 716 bytes against 352 / 496).
constexpr int BATCH_PUB_WORDS = 32;      // 256 bytes per slot
template <bool EXTR, bool DET = false>
__device__ __forceinline__ void update_batch_body(UpdArgs& a, int log_stride) {
    const int s = (int)blockIdx.y;
    const size_t rows = (size_t)s * (size_t)a.sc.Q;
    a.ctl += s;
    a.partials += (size_t)s * (gridDim.x - 1) * PSTRIDE;
    a.pub += (size_t)s * BATCH_PUB_WORDS;
    if (a.logs) a.logs += (size_t)s * log_stride;
    a.sc.nearest += rows * KNN_K;
    a.sc.nearest_cnt += rows;
    a.sc.selected += rows;
    a.sc.plane += rows;
    a.sc.srange += rows;
    update_body<EXTR, 1, DET>(a, a.sc.q_end);
}
template <bool EXTR>
__global__ void __launch_bounds__(UPD_THREADS, 2) k_update_batch(UpdArgs a, int log_stride) {
    update_batch_body<EXTR>(a, log_stride);
}

// ============================================================================= one tile per worker block: k_update_wave
// The single-GPU update (mode 0) when every tile of the scan has a worker block of its own, which is exactly when plan_update
// picks two threads per point: the 512-thread block, the paired search and the tiles of k_update<EXTR, 2>, so the same bytes.
// Thread t < 256 owns point tile + t for the whole launch, which removes three things from every pass's chain:
//   * the point's state stays in shared memory (WavePoint): the body point, sqrt(|p_body|), the plane and the selected flag; a
//     pass that does not search no longer reloads selected -> plane -> srange from L2 (the memory copies are still written);
//   * the pickup of the solver's publication: lanes 0..28 of warp 0 spin on their own tagged word, then one barrier;
//   * the partial rows go out as tagged words (row_tag: 32 bits of payload, 32 of tag, as pub_store), with no ticket; each
//     solver warp spins on and sums its own rows as they arrive, in sol_reduce's order.
// A graph replay keeps the launch nonce it was captured with, so the rows are tagged with an epoch kept in device memory
// (word WAVE_EPOCH of the publication block, outside the control block that restore_state rewinds): each launch tags with
// the stored epoch + 1 and the solver stores it when the update ends, so no row of an earlier launch is ever current.
// Stamps in ctl->prof besides k_update's clock64 ones, in %globaltimer ns so they compare across SMs, for the pass that ends
// the update: [11] the solver has summed every partial row, [2] its publication is visible on the solver's SM (an otherwise
// idle thread of block 0 polls for it), [3] the last worker block has picked it up.  Each is read by a thread nothing waits
// for: a %globaltimer read costs several hundred cycles on H100.
struct WavePoint {                 // dynamic shared memory of a worker block: its tile's points
    float4 body[UPD_THREADS];
    float4 plane[UPD_THREADS];
    double srange[UPD_THREADS];
    unsigned char sel[UPD_THREADS];
};
constexpr int WAVE_EPOCH = 32;     // word of the publication block (a 128-byte line of its own)
__device__ __forceinline__ unsigned row_tag(unsigned epoch, int pass) { return pub_tag(epoch, pass + 1); }     // never 0
__device__ __forceinline__ unsigned long long globaltimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ ulonglong2 row_load(const unsigned long long* p) {
    ulonglong2 v;
    asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ bool row_current(ulonglong2 v, unsigned tag) { return (unsigned)(v.x >> 32) == tag && (unsigned)(v.y >> 32) == tag; }
__device__ __forceinline__ double row_value(ulonglong2 v) { return __longlong_as_double((long long)((v.y << 32) | (v.x & 0xffffffffull))); }

// measure_fused<EXTR, 2> with the point's state in `pt` (slot threadIdx.x % 256); the same outputs in memory
template <bool EXTR, bool DET>
__device__ __forceinline__ bool measure_wave(const MapView& m, const ScanView& sc, int q, bool active, const PoseS& s, bool searched,
                                             bool search_only, WalkPool& walks, int& phase, double* stage, WavePoint& pt, double* h,
                                             double& z, float& absres) {
    const int i = threadIdx.x & (UPD_THREADS - 1);
    float4 pb = make_float4(0.f, 0.f, 0.f, 0.f);
    float wx = 0.f, wy = 0.f, wz = 0.f;
    D3 p_this = d3(0.0, 0.0, 0.0);
    if (active) {
        pb = pt.body[i];
        p_this = body_to_world(s, pb, wx, wy, wz);
    }
    bool sel = false;
    float pabcd[4] = {0.f, 0.f, 0.f, 0.f};
    if (searched) {
        TBestT<DET> kb;
        knn_block_pair(m, active, wx, wy, wz, kb, walks, phase, stage);
        if (threadIdx.x >= UPD_THREADS) return false;
        if (active) {
            float4 p[KNN_K];
            const int cnt = knn_fetch(m, kb, p);
#pragma unroll
            for (int j = 0; j < KNN_K; j++) sc.nearest[(size_t)q * KNN_K + j] = p[j];
            sc.nearest_cnt[q] = cnt;
            sel = knn_gate(cnt, kb.d[KNN_K - 1]);
            if (search_only) { sc.selected[q] = sel ? 1 : 0; return false; }
            if (sel) {
                float pn[KNN_K][3];
#pragma unroll
                for (int j = 0; j < KNN_K; j++) { pn[j][0] = p[j].x; pn[j][1] = p[j].y; pn[j][2] = p[j].z; }
                sel = esti_plane_dev(pabcd, pn, 0.1f);
                if (sel) { const float4 pl = make_float4(pabcd[0], pabcd[1], pabcd[2], pabcd[3]); sc.plane[q] = pl; pt.plane[i] = pl; }
            }
        }
    } else if (active) {
        sel = pt.sel[i] != 0;
        if (sel) { const float4 pl = pt.plane[i]; pabcd[0] = pl.x; pabcd[1] = pl.y; pabcd[2] = pl.z; pabcd[3] = pl.w; }
    }
    bool contrib = false;
    if (active && sel) {
        const float pd2 = plane_residual(pabcd, wx, wy, wz);
        const double srange = pt.srange[i];
        if (searched) sc.srange[q] = srange;
        float score;
        if (score_gate(pd2, srange, score)) {
            contrib = true;
            absres = fabsf(pd2);
            jacobian_row_at<EXTR>(s, pb, p_this, make_float4(pabcd[0], pabcd[1], pabcd[2], pd2), h, z);
        }
    }
    if (active) { sc.selected[q] = contrib ? 1 : 0; pt.sel[i] = contrib ? 1 : 0; }
    return contrib;
}

// sol_reduce over tagged rows: warp w takes the rows w, w + 8, ... of pass `tag` GATHER_ROWS at a time, spins until each of them
// is current (every poll reloads all the stale words of the batch at once: one round trip) and sums them in ascending order from
// +0.0 (sol_reduce's order; the +0.0 rows it adds past nwork change no sum)
constexpr int GATHER_ROWS = 8;
__device__ void sol_gather(SolverSm& S, FilterCtl* ctl, const unsigned long long* __restrict__ rows, int nwork, unsigned tag) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double a0 = 0.0, a1 = 0.0, a2 = 0.0;
    bool late = false;
    const long long t0 = clock64();
    for (int b = warp; b < nwork; b += GATHER_ROWS * UPD_WARPS) {
        const unsigned long long* base = rows + (size_t)b * PSTRIDE * 2 + 2 * lane;
        ulonglong2 v[GATHER_ROWS][3];
#pragma unroll
        for (int k = 0; k < GATHER_ROWS; k++) {
#pragma unroll
            for (int j = 0; j < 3; j++) v[k][j] = make_ulonglong2(0ull, 0ull);
            if (b + k * UPD_WARPS < nwork) {
#pragma unroll
                for (int j = 0; j < 3; j++) v[k][j] = row_load(base + (size_t)k * UPD_WARPS * PSTRIDE * 2 + 64 * j);
            }
        }
        while (true) {
            bool stale = false;
#pragma unroll
            for (int k = 0; k < GATHER_ROWS; k++) {
#pragma unroll
                for (int j = 0; j < 3; j++) stale |= b + k * UPD_WARPS < nwork && !row_current(v[k][j], tag);
            }
            if (!stale) break;
            if (clock64() - t0 > SPIN_LIMIT) { late = true; break; }
#pragma unroll
            for (int k = 0; k < GATHER_ROWS; k++) {
#pragma unroll
                for (int j = 0; j < 3; j++) {
                    if (b + k * UPD_WARPS < nwork && !row_current(v[k][j], tag)) v[k][j] = row_load(base + (size_t)k * UPD_WARPS * PSTRIDE * 2 + 64 * j);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < GATHER_ROWS; k++) {
            if (b + k * UPD_WARPS < nwork) { a0 += row_value(v[k][0]); a1 += row_value(v[k][1]); a2 += row_value(v[k][2]); }
        }
        if (late) break;
    }
    S.wred[warp][lane] = a0; S.wred[warp][lane + 32] = a1; S.wred[warp][lane + 64] = a2;
    if (late) S.late = 2;
    sol_sync();
    if (tid == 0) ctl->prof[9] = clock64();
    if (tid < PSTRIDE) {
        double v = 0.0;
#pragma unroll
        for (int w = 0; w < UPD_WARPS; w++) v += S.wred[w][tid];
        S.red[tid] = v;
        if (tid < 78) {
            int a = 0, rem = tid;
            while (rem >= 12 - a) { rem -= 12 - a; a++; }
            const int b = a + rem;
            S.HTH[a * 12 + b] = v; S.HTH[b * 12 + a] = v;
        }
    }
    sol_sync();
    if (tid == 128) ctl->prof[11] = (long long)globaltimer();         // a warp the gain does not wait for
}

// update_body<EXTR, 2> for mode 0 with one tile per worker block (gridDim.x - 1 >= the tiles of [q_begin, q1)); rows: the
// partial rows as tagged words, [worker block][PSTRIDE][2]
template <bool EXTR, bool DET = false>
__device__ __forceinline__ void update_wave_body(const UpdArgs& a, unsigned long long* __restrict__ rows, const int q1) {
    static_assert(sizeof(PairXch) <= sizeof(double) * WorkerSm<EXTR>::STAGE, "the partner's list fits the owner warp's stage slice");
    __shared__ __align__(16) unsigned char smem_raw[sizeof(SolverSm) > sizeof(WorkerSm<EXTR>) ? sizeof(SolverSm) : sizeof(WorkerSm<EXTR>)];
    extern __shared__ __align__(16) unsigned char wave_dyn[];
    __shared__ volatile int solver_ended;
    FilterCtl* ctl = a.ctl;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nwork = (int)gridDim.x - 1;
    pdl_wait();
    pdl_launch();
    const unsigned epoch = (unsigned)__ldcg(a.pub + WAVE_EPOCH) + 1u;
    if (blockIdx.x > 0) {
        // ------------------------------------------------------------------ worker block
        WorkerSm<EXTR>& Wk = *reinterpret_cast<WorkerSm<EXTR>*>(smem_raw);
        WavePoint& pt = *reinterpret_cast<WavePoint*>(wave_dyn);
        const int wb = (int)blockIdx.x - 1;
        const int i = tid & (UPD_THREADS - 1), q = a.sc.q_begin + wb * UPD_THREADS + i;
        const bool active = q < q1, owner = tid < UPD_THREADS;
        if (tid == 0) { Wk.abort = 0; Wk.walks.n[0] = Wk.walks.n[1] = 0; }
        int walk_phase = 0;
        double* stage = Wk.stage[warp & (UPD_WARPS - 1)];
        for (int p = 0; p < a.max_passes; p++) {
            PoseS s;
            bool searched;
            if (p == 0) {
                // the state this launch starts from, and the tile's points, loaded together
                const bool done = __ldcg(&ctl->done) != 0;
                searched = __ldcg(&ctl->converge) != 0 || a.search_only;
                s = load_pose(a.pose_from_search ? ctl->x_search : ctl->x);
                if (owner && active) {
                    const float4 pb = __ldg(&a.sc.body[q]);
                    pt.body[i] = pb;
                    pt.srange[i] = sqrt(norm3(d3(pb.x, pb.y, pb.z)));       // sqrt(p_body.norm()) of the score, for every pass
                    if (!searched) {                                        // the fit and the flag of an earlier launch
                        pt.sel[i] = a.sc.selected[q];
                        if (pt.sel[i]) { pt.plane[i] = a.sc.plane[q]; pt.srange[i] = a.sc.srange[q]; }
                    }
                }
                __syncthreads();
                if (done && !a.search_only) return;
            } else {
                const unsigned tag = pub_tag(a.nonce, p);
                if (warp == 0 && lane < PUB_WORDS) {
                    unsigned long long w = pub_load(a.pub + lane);
                    const long long t0 = clock64();
                    while ((unsigned)(w >> 32) != tag) {
                        if (clock64() - t0 > SPIN_LIMIT) { Wk.abort = 1; atomicExch(&ctl->error, 3); break; }
                        w = pub_load(a.pub + lane);
                    }
                    if (lane < 28) Wk.pose_bits[lane] = (unsigned)w; else Wk.flags = (unsigned)w;
                }
                __syncthreads();
                if (Wk.abort) return;
                if (Wk.flags & 2u) {
                    // reading %globaltimer takes hundreds of cycles: stamped only where nothing waits for it
                    if (tid == 0) atomicMax(reinterpret_cast<unsigned long long*>(&ctl->prof[3]), globaltimer());
                    return;
                }
                searched = (Wk.flags & 1u) != 0;
                double x14[14];
#pragma unroll
                for (int k = 0; k < 14; k++) x14[k] = __longlong_as_double((long long)(((unsigned long long)Wk.pose_bits[2 * k + 1] << 32) | Wk.pose_bits[2 * k]));
                s.pos = d3(x14[X_POS], x14[X_POS + 1], x14[X_POS + 2]);
                s.rot.x = x14[X_ROT]; s.rot.y = x14[X_ROT + 1]; s.rot.z = x14[X_ROT + 2]; s.rot.w = x14[X_ROT + 3];
                s.offR.x = x14[X_OFFR]; s.offR.y = x14[X_OFFR + 1]; s.offR.z = x14[X_OFFR + 2]; s.offR.w = x14[X_OFFR + 3];
                s.offT = d3(x14[X_OFFT], x14[X_OFFT + 1], x14[X_OFFT + 2]);
            }
            double acc[3] = {0.0, 0.0, 0.0};
            double h[12]; double z = 0.0; float ar = 0.f;
            bool contrib = false;
            if (owner || searched)
                contrib = measure_wave<EXTR, DET>(a.m, a.sc, q, active, s, searched, a.search_only != 0, Wk.walks, walk_phase, stage, pt, h, z, ar);
            if (owner && !a.search_only) warp_accumulate<EXTR>(contrib, h, z, ar, acc, lane, stage);
            if (a.search_only) return;
            if (owner) {
#pragma unroll
                for (int j = 0; j < 3; j++) Wk.wred[warp][lane + 32 * j] = acc[j];
            }
            __syncthreads();
            if (tid < PSTRIDE) {
                double v = 0.0;
#pragma unroll
                for (int w = 0; w < UPD_WARPS; w++) v += Wk.wred[w][tid];
                const unsigned long long bits = (unsigned long long)__double_as_longlong(v);
                unsigned long long* dst = rows + ((size_t)wb * PSTRIDE + tid) * 2;
                const unsigned tag = row_tag(epoch, p);
                pub_store(dst, tag, (unsigned)bits);
                pub_store(dst + 1, tag, (unsigned)(bits >> 32));
            }
        }
        return;
    }
    // ------------------------------------------------------------------ solver block
    if (a.search_only) return;
    if (tid == 0) solver_ended = 0;
    __syncthreads();
    if (tid >= UPD_THREADS) {
        // one thread stamps the publications as they become visible on this SM
        if (tid == UPD_THREADS) {
            for (int p = 1; p <= a.max_passes; p++) {
                const unsigned tag = pub_tag(a.nonce, p);
                unsigned long long w;
                while ((unsigned)((w = pub_load(a.pub + 28)) >> 32) != tag) if (solver_ended) return;
                ctl->prof[2] = (long long)globaltimer();
                if (w & 2u) return;
            }
        }
        return;
    }
    SolverSm& S = *reinterpret_cast<SolverSm*>(smem_raw);
    sol_load(S, ctl);
    for (int p = 0; p < a.max_passes && !S.done; p++) {
        if (tid == 0) ctl->prof[0] = clock64();
        if (S.converge && tid < XLEN) ctl->x_search[tid] = S.x[tid];
        sol_prepare(S);
        if (tid == 0) ctl->prof[8] = clock64();
        sol_gather(S, ctl, rows, nwork, row_tag(epoch, p));
        if (tid == 0) ctl->prof[1] = clock64();
        sol_pass<EXTR>(S, ctl, a.logs, a.pub, pub_tag(a.nonce, p + 1));
        if (tid == 0) ctl->prof[7] = clock64();
    }
    if (tid == 0) {
        ctl->error = S.error | ctl->error; ctl->ticket = 0;
        a.pub[WAVE_EPOCH] = epoch;
        solver_ended = 1;
    }
    sol_sync();
    mirror_copy(ctl, UPD_THREADS);
}

template <bool EXTR>
__global__ void __launch_bounds__(2 * UPD_THREADS, 1) k_update_wave(UpdArgs a, unsigned long long* rows) {
    update_wave_body<EXTR>(a, rows, a.sc.q_end);
}
// k_update_n's form: the point count in device memory (read before pdl_wait, see k_update_n)
template <bool EXTR>
__global__ void __launch_bounds__(2 * UPD_THREADS, 1) k_update_n_wave(UpdArgs a, const int* __restrict__ n, unsigned long long* rows) {
    update_wave_body<EXTR>(a, rows, min(*n, a.sc.q_end));
}

// ============================================================================= the keyed tie rule (fl_map_set_deterministic)
// Every update kernel above again, searching the map under the keyed order (map.cuh, "tie rules"): same bounds, same shared
// memory, same tiles and sums, so the launch plan's grids hold for them.  Kernels of their own, so the default ones keep their code.
template <bool EXTR, int PAIR>
__global__ void __launch_bounds__(UPD_THREADS * PAIR, 3 - PAIR) k_update_det(UpdArgs a) {
    update_body<EXTR, PAIR, true>(a, a.sc.q_end);
}
template <bool EXTR, int PAIR>
__global__ void __launch_bounds__(UPD_THREADS * PAIR, 3 - PAIR) k_update_n_det(UpdArgs a, const int* __restrict__ n) {
    update_body<EXTR, PAIR, true>(a, min(*n, a.sc.q_end));
}
template <bool EXTR>
__global__ void __launch_bounds__(UPD_THREADS, 2) k_update_batch_det(UpdArgs a, int log_stride) {
    update_batch_body<EXTR, true>(a, log_stride);
}
template <bool EXTR>
__global__ void __launch_bounds__(2 * UPD_THREADS, 1) k_update_wave_det(UpdArgs a, unsigned long long* rows) {
    update_wave_body<EXTR, true>(a, rows, a.sc.q_end);
}
template <bool EXTR>
__global__ void __launch_bounds__(2 * UPD_THREADS, 1) k_update_n_wave_det(UpdArgs a, const int* __restrict__ n, unsigned long long* rows) {
    update_wave_body<EXTR, true>(a, rows, min(*n, a.sc.q_end));
}

}  // namespace fl
