// ctypes front of fast_lio_b200/csrc/map_rules.h (tests/test_map_rules.py), built with g++ alone: the header needs no CUDA.
#include "../../fast_lio_b200/csrc/map_rules.h"

extern "C" {
int mr_chain_limit(float frac, int n_main) { return fl::chain_limit(frac, n_main); }
int mr_repack_due(int leaf_used, int n_main, int max_chained, int tombs, int valid) {
    return fl::repack_due(leaf_used, n_main, max_chained, tombs, valid);
}
int mr_relist_due(int dir_error, int crowded, int cells) { return fl::relist_due(dir_error, crowded, cells); }
int mr_leaves_fit(long long leaf_used, long long leaf_cap, long long n) { return fl::leaves_fit(leaf_used, leaf_cap, n); }
int mr_table_fits(long long cells, long long cap, long long n) { return fl::table_fits(cells, cap, n); }
int mr_batch_fits(long long leaf_used, long long leaf_cap, long long cells, long long cap, long long n) {
    return fl::batch_fits(leaf_used, leaf_cap, cells, cap, n);
}
int mr_pool_min_for_batch(int min_pool, long long n) { return fl::pool_min_for_batch(min_pool, n); }
size_t mr_dir_cap_min_for_batch(size_t min_cap, long long cells, long long n) { return fl::dir_cap_min_for_batch(min_cap, cells, n); }
size_t mr_dir_cap_min_after_error(size_t min_cap, size_t cap) { return fl::dir_cap_min_after_error(min_cap, cap); }
size_t mr_list_pool_min_grown(size_t min_pool, size_t at_least) { return fl::list_pool_min_grown(min_pool, at_least); }
}
