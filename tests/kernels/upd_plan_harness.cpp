// ctypes front of fast_lio_b200/csrc/upd_plan.h (tests/test_update_plan.py), built with g++ alone: the header needs no CUDA.
#include "../../fast_lio_b200/csrc/upd_plan.h"

extern "C" int up_kernel_count() { return fl::UK_COUNT; }

// blocks: [UK_COUNT][2] co-resident blocks; in: n rows of (route, rows, extr, one_thread, n_hyp); out: n rows of
// (kernel, workers, pair, grid_x, slots, waves, block, smem, pdl)
extern "C" void up_plan(const int* blocks, int threads, int wave_smem, int n, const int* in, int* out) {
    fl::UpdCaps c;
    for (int k = 0; k < fl::UK_COUNT; k++)
        for (int e = 0; e < 2; e++) c.blocks[k][e] = blocks[2 * k + e];
    c.threads = threads;
    c.wave_smem = wave_smem;
    for (int i = 0; i < n; i++) {
        const int* a = in + 5 * i;
        const fl::UpdPlan p = fl::plan_update(c, (fl::UpdRoute)a[0], a[1], a[2] != 0, a[3] != 0, a[4]);
        const int v[9] = {p.kernel, p.workers, p.pair, p.grid_x, p.slots, p.waves, p.block, p.smem, p.pdl ? 1 : 0};
        for (int j = 0; j < 9; j++) out[9 * i + j] = v[j];
    }
}
