// Which update kernel a launch of the iterated-EKF update runs, on how many worker blocks, with one or two threads per point:
// the rule of every route in one place.  Plain C++ without CUDA, so tests/test_update_plan.py checks it on the host.
#pragma once
#include <algorithm>

namespace fl {

// k_update<EXTR, 1|2>, k_update_n<EXTR, 1|2> (the count in device memory), k_update_wave, k_update_n_wave, k_update_batch
enum UpdKernel { UK_UPDATE1, UK_UPDATE2, UK_N1, UK_N2, UK_WAVE, UK_N_WAVE, UK_BATCH, UK_COUNT };
inline int upd_kernel_pair(int k) { return k == UK_UPDATE2 || k == UK_N2 || k == UK_WAVE || k == UK_N_WAVE ? 2 : 1; }

// 0..3: UpdArgs::mode over the scan bound on the host (Filter::launch_update, search-only launches included in mode 0), then
// update_scan_on_stream (the count in device memory), complete_neighbours and update_batch_on_stream
enum UpdRoute { UR_MODE0, UR_MODE1, UR_MODE2, UR_MODE3, UR_DEVICE_COUNT, UR_NEIGHBOURS, UR_BATCH };

struct UpdCaps {
    int blocks[UK_COUNT][2];   // co-resident blocks of each kernel on the device, [kernel][EXTR]
    int threads;               // points per tile (UPD_THREADS)
    int wave_smem;             // dynamic shared memory of the wave kernels (sizeof(WavePoint))
};

struct UpdPlan {
    UpdKernel kernel;
    int workers, pair;         // worker blocks (block 0 solves), threads per point
    int grid_x, slots, waves;  // workers + 1; batch: hypotheses per wave (0: one does not fit) and waves for n_hyp, else 1 and 1
    int block, smem;           // threads per block, dynamic shared memory bytes
    bool pdl;                  // may overlap its predecessor (programmatic dependent launch, when the filter has it on)
    bool det;                  // the keyed-tie-rule instantiation of `kernel` (the map's deterministic mode)
    bool scans;                // UK_BATCH with a scan per slot (k_update_scans): never set here, the filter sets it
};

// Every co-resident block works (a searching pass wants many warps in flight), one thread per point in full warps.  Two threads
// per point when the tiles all fit the co-resident 512-thread grid, so the tiles, workers and partial rows are those of the
// one-thread form; larger scans keep one thread per point rather than idle half the warps on passes that do not search, and
// one_thread (FASTLIO_B200_PAIR=1) forces it.  The paired mode-0 update runs the wave kernel when its grid fits.  det picks the
// keyed-tie-rule instantiation of the same kernel: same grid, block and shared memory (its caps are those of both forms).
inline UpdPlan plan_update(const UpdCaps& c, UpdRoute r, int rows, bool extr, bool one_thread, int n_hyp = 0, bool det = false) {
    auto cap = [&](UpdKernel k) { return c.blocks[k][extr ? 1 : 0]; };
    const int tiles = (rows + c.threads - 1) / c.threads;
    UpdPlan p{};
    p.workers = std::max(0, std::min(cap(UK_UPDATE1) - 1, tiles));
    p.pair = !one_thread && tiles >= 1 && tiles <= cap(UK_UPDATE2) - 1 ? 2 : 1;
    p.slots = p.waves = 1;
    p.pdl = true;
    if (r == UR_DEVICE_COUNT) {            // the host form's choice at the row bound, against the _n forms' grids
        if (tiles > cap(UK_N2) - 1) p.pair = 1;
        p.workers = std::max(0, std::min(cap(UK_N1) - 1, tiles));
        p.kernel = p.pair == 1 ? UK_N1 : p.workers + 1 <= cap(UK_N_WAVE) ? UK_N_WAVE : UK_N2;
    } else if (r == UR_NEIGHBOURS) {       // at least one worker, no PDL, never the wave kernel
        p.workers = std::max(1, p.workers);
        p.kernel = p.pair == 1 ? UK_UPDATE1 : UK_UPDATE2;
        p.pdl = false;
    } else if (r == UR_BATCH) {            // the single form's workers per hypothesis, one thread per point
        p.pair = 1;
        p.kernel = UK_BATCH;
        p.slots = p.workers + 1 <= cap(UK_BATCH) ? cap(UK_BATCH) / (p.workers + 1) : 0;
        p.waves = p.slots ? (n_hyp + p.slots - 1) / p.slots : 0;
    } else {                               // mode 3 is the solver block alone, with the block size of the pair choice
        if (r == UR_MODE3) p.workers = 0;
        p.kernel = p.pair == 1 ? UK_UPDATE1 : r == UR_MODE0 && p.workers + 1 <= cap(UK_WAVE) ? UK_WAVE : UK_UPDATE2;
    }
    p.grid_x = p.workers + 1;
    p.block = p.pair * c.threads;
    p.smem = p.kernel == UK_WAVE || p.kernel == UK_N_WAVE ? c.wave_smem : 0;
    p.det = det;
    return p;
}

}  // namespace fl
