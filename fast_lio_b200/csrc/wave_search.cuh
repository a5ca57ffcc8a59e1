// The k-NN search of k_update_wave / k_update_n_wave (and their _det twins): knn_block_pair, with the BVH walks of the queries
// the halo list does not prove called out of line (wave_walk).  The walk is rare -- a few dozen queries per update on config 2 --
// but inlined twice into measure_wave its six-level descent dominates the kernel's code and its register allocation; out of line,
// the path every point takes is compiled without it.  The answers are the same bits: the same walk from the same seed.
#pragma once

namespace fl {

// knn_query_from for one pooled query; the map is passed by value so that the call does not need the kernel parameters' address
template <bool DET>
__device__ __noinline__ void wave_walk(const MapView m, float qx, float qy, float qz, KBestT<DET>& kb, int lane) {
    knn_query_from(m, qx, qy, qz, kb, lane);
}

// knn_block_pair with its walks through wave_walk
template <bool DET>
__device__ __forceinline__ void knn_block_wave(const MapView& m, bool active, float qx, float qy, float qz, TBestT<DET>& kb, WalkPool& W,
                                               int& phase, double* stage) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const bool owner = threadIdx.x < UPD_THREADS;
    const CellDir& D = m.dir;
    kb.init();
    int ix = 0, iy = 0, iz = 0;
    bool listed = false;
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
    pair_sync(warp);
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
        wave_walk(m, W.x[i], W.y[i], W.z[i], w, lane);
        __syncwarp();
        if (lane < KNN_K) { W.rd[i][lane] = w.d; W.ri[i][lane] = w.idx; }
    }
    unsigned todo = __ballot_sync(FULL, mine_slot >= WALK_POOL);
    while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        KBestT<DET> w;
        w.init();
        wave_walk(m, __shfl_sync(FULL, qx, src), __shfl_sync(FULL, qy, src), __shfl_sync(FULL, qz, src), w, lane);
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

}  // namespace fl
