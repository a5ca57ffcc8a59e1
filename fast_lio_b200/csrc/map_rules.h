// When the map re-packs its leaves, re-lists its cell directory and grows for a batch: the rules of the host-form mutations
// (Map::maybe_rebuild, relist_if_due, grow_for_batch, async_fits) and of the device forms' one-thread kernels (k_plan,
// k_async_account, k_delete_account), which must agree for the device forms to give the host forms' answers.  Plain C++ on
// plain integers, FL_HD so that both sides call the same code; tests/test_map_rules.py checks it on the host.
#pragma once
#include <limits.h>
#include <stddef.h>

#include "lie.cuh"

namespace fl {

// --------------------------------------------------------------------------------------------- re-pack (ikd-Tree's Rebuild)
// The most overflow leaves the main leaves may chain before a re-pack: a fraction of them, at least 64
FL_HD int chain_limit(float overflow_frac, int n_main) {
    const int c = (int)(overflow_frac * n_main);
    return c > 64 ? c : 64;
}
// Too chained, or too sparse: more than 1024 lazily deleted points and more of them than valid ones (ikd-Tree's delete
// criterion, alpha_del = 0.5)
FL_HD bool repack_due(int leaf_used, int n_main, int max_chained, int tombs, int valid) {
    return leaf_used - n_main > max_chained || (tombs > 1024 && tombs > valid);
}

// --------------------------------------------------------------------------------------------- re-list (the cell directory)
// After inserts: the table or the list pool ran out (dir_error), or too many cells are crowded (their queries walk the BVH)
FL_HD bool relist_due(int dir_error, int crowded, int cells) {
    const int limit = cells / 1024;
    return dir_error || crowded > (limit > 64 ? limit : 64);
}

// --------------------------------------------------------------------------------------------- headroom for a batch of n points
// Worst case, each point takes one fresh overflow leaf and claims its 27 halo cells fresh.  The counts are non-negative ints
// and n far below 2^50, so no sum or product here leaves long long, and the size_t some callers used gives the same results.
FL_HD bool leaves_fit(long long leaf_used, long long leaf_cap, long long n) { return leaf_used + n <= leaf_cap; }
FL_HD long long cells_after(long long cells, long long n) { return cells + 27 * n; }
// the table at most 90 % loaded, so that probing does not degenerate (cap 0: the directory is off)
FL_HD bool table_fits(long long cells, long long cap, long long n) { return !cap || cells_after(cells, n) * 10 <= cap * 9; }
FL_HD bool batch_fits(long long leaf_used, long long leaf_cap, long long cells, long long cap, long long n) {
    return leaves_fit(leaf_used, leaf_cap, n) && table_fits(cells, cap, n);
}

// --------------------------------------------------------------------------------------------- growth: the new minimums
// The overflow pool (in leaves) for a batch the leaves might not hold: the batch and 1024 to spare.  The clamp keeps the int
// defined for any n.  It binds only far above 0x7fffffff / LEAF leaves, where Map::ensure_capacity refuses the re-pack anyway.
FL_HD int pool_min_for_batch(int min_pool, long long n) {
    const long long want = n + 1024 > min_pool ? n + 1024 : min_pool;
    return (int)(want < INT_MAX / 2 ? want : INT_MAX / 2);
}
// The table for a batch that might load it above 90 %: twice the cells it would have, and 16384 to spare
FL_HD size_t dir_cap_min_for_batch(size_t min_cap, long long cells, long long n) {
    const size_t want = (size_t)cells_after(cells, n) * 2 + 16384;
    return want > min_cap ? want : min_cap;
}
// The table after an insert found it full: 1.5 times the current one
FL_HD size_t dir_cap_min_after_error(size_t min_cap, size_t cap) {
    const size_t want = cap + cap / 2;
    return want > min_cap ? want : min_cap;
}
// The list pool after it ran out: twice the last minimum, and at least `at_least`
FL_HD size_t list_pool_min_grown(size_t min_pool, size_t at_least) {
    return min_pool * 2 > at_least ? min_pool * 2 : at_least;
}

}  // namespace fl
