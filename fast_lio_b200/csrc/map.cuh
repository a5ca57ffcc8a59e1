// Device-side view of the point map and the warp-cooperative traversals over it.
//
// The reference's ikd-Tree (include/ikd-Tree/ikd_Tree.{h,cpp}) is a pointer-chasing
// binary k-d tree with 176-byte nodes (ikd_Tree.h:59-82) and ~33 dependent node visits
// per query.  Here the map is a flattened, implicit 32-ary bounding-volume hierarchy over
// a k-d partition of the points:
//
//   level 0   leaf buckets: 32 slots of float4 (x, y, z, flag) = 512 B, one coalesced
//             warp load.  At (re)build time the points are split top-down at the median
//             of the longest axis -- the rule of KD_TREE::BuildTree (ikd_Tree.cpp:679-733)
//             -- until each cell holds `fill` points; the free slots absorb inserts.
//   level k   entity e of level k (a leaf for k = 0, an internal node otherwise) has its
//             AABB in ebox[k][e] (two float4: lo, hi).  Node j of level k+1 owns entities
//             32j .. 32j+31 of level k: five binary k-d levels collapse into one 32-wide
//             node, there are no child pointers, and a warp tests all children of a node
//             with one box per lane.
//
// A query is served by one warp: every lane holds the query, the k best candidates live
// one per lane (lanes 0..k-1, ascending), candidates are ranked with the hardware warp
// reduction (redux.sync) and the traversal state of each level lives in registers (the
// recursion over the <= 7 levels is unrolled at compile time): no stack in memory.
#pragma once
#include <limits.h>

#include "common.cuh"

namespace fl {

// ----------------------------------------------------------------------------- cell directory
// A hashed directory of cubic cells over the SAME leaf slots, arranged so that a k-NN query is ONE look-up: the entry of cell
// (ix, iy, iz) = floor(p * inv_cell) lists the slot indices of every point that lies in the 3x3x3 block of cells around it
// (its "halo list", contiguous in HBM).  A thread finds its query's cell, scores the listed points and proves the result exact
// from the distance to the faces of that block; whatever it cannot prove -- nothing nearby, an over-full cell -- goes through the
// warp-cooperative BVH walk below, so the result is always the exact answer of KD_TREE::Nearest_Search (ikd_Tree.cpp:426-461).
// Every point is listed in the 27 cells around it (HBM is plentiful: ~130 bytes of directory per point).  Validity lives in the
// slot's flag only: a deleted point keeps its listings and is skipped.  A slot re-used by a later insert is listed again under
// its new point's cells and keeps the old listings: a list may therefore name a slot twice, or name a slot whose point lies
// outside the block -- both harmless (any live point is a legitimate candidate; the k-best list never takes a slot twice) and
// packed away by the next re-list.
constexpr int CELL_OFF = 1 << 20;                  // 21 bits per axis
constexpr int CELL_CLAMP = (1 << 20) - 4;
constexpr int HALO_MAX = 2048;                     // a cell whose block holds more points than this sends its queries to the BVH walk
constexpr int HALO_NEW_CAP = 64;                   // room of a list created by an insert (lists made by a re-list get count + 25 %)

struct __align__(16) CellEntry {
    unsigned long long key;      // 0 = free, else cell_key()
    int start;                   // first index of the list in `lists` (multiple of 4); < 0: over-full, use the BVH walk
    unsigned cnt_cap;            // low 16 bits: points listed, high 16 bits: room
};
struct CellDir {
    CellEntry* tab;              // [cap]
    int* lists;                  // [lists_cap]
    unsigned cap;                // 0: directory disabled
    int lists_cap;
    float cell, inv_cell;
    int* n_walked;               // statistics: queries that went through the BVH walk
};

struct MapView {
    CellDir dir;
    float4* pts;                     // [leaf_cap * 32]  (x, y, z, as_float(flag)); flag 1 = valid
    float* payload;                  // [leaf_cap * 32]  intensity of the point in that slot
    int* next;                       // [leaf_cap]       overflow chain of a leaf, -1 = none
    float4* ebox[MAX_LEVELS];        // [count * 2]      AABB (lo, hi) of each entity of level k
    int count[MAX_LEVELS + 1];       // entities per level; count[n_levels] == 1 (the root)
    int n_levels;                    // number of internal levels (>= 1)
    int n_main;                      // leaves addressed by the implicit tree (== count[0])
    int leaf_cap;                    // allocated leaves (main + overflow pool)
};

// slot flag (bits of pts[].w): never used / live point / being written by an insert / deleted by Delete_Point_Boxes (Add_Point_Boxes
// may revive it) / deleted by the down-sampling of Add_Points.  Deleted points keep their listing in the cell directory.
constexpr int SLOT_FREE = 0, SLOT_VALID = 1, SLOT_BUSY = 2, SLOT_TOMB = 3, SLOT_TOMB_DS = 4;
__device__ __forceinline__ bool slot_valid(const float4& p) { return __float_as_int(p.w) == SLOT_VALID; }
// ----------------------------------------------------------------------------- k-best list
// Squared distances are non-negative floats, so their bit patterns order like the values and
// +inf (0x7f800000) can serve as the "no candidate" marker of the integer warp reductions.
constexpr unsigned INF_BITS = 0x7f800000u;

// ----------------------------------------------------------------------------- tie rules
// Every k-best list below takes a tie rule as its template parameter DET:
//   false (the default): a candidate enters only if strictly closer than the k-th best, so of two points at bit-equal squared
//          distances the one visited first wins -- the reference's rule (ikd_Tree.cpp:1088), whose visiting order here is the
//          slot order of leaves and halo lists, which racing inserts make run-dependent;
//   true  (fl_map_set_deterministic): candidates are ranked by the total order (d2, x, y, z, intensity), the coordinates and
//          the intensity compared as order-preserving integers of their bits (key_less), so the k best are a function of the
//          SET of valid points.  The key is read from the map (m.pts / m.payload) only when a candidate's d2 equals an entry's,
//          the rare path: nothing extra is carried in registers.
__device__ __forceinline__ unsigned ord_bits(float f) {            // float order, with -0 below +0
    const unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
// (x, y, z, intensity) of the point in slot a strictly below that of slot b.  NC: read-only (non-coherent) loads, for kernels that
// write no slot; the down-sampling kernel, whose warps retire slots while others read, uses plain loads (NC = false).
template <bool NC = true>
__device__ __forceinline__ float4 map_pt(const MapView& m, int i) { if constexpr (NC) return __ldg(&m.pts[i]); else return m.pts[i]; }
template <bool NC = true>
__device__ __forceinline__ float map_payload(const MapView& m, int i) { if constexpr (NC) return __ldg(&m.payload[i]); else return m.payload[i]; }
template <bool NC = true>
__device__ __forceinline__ bool key_less(const MapView& m, int a, int b) {
    const float4 pa = map_pt<NC>(m, a), pb = map_pt<NC>(m, b);
    if (pa.x != pb.x || __float_as_uint(pa.x) != __float_as_uint(pb.x)) return ord_bits(pa.x) < ord_bits(pb.x);
    if (pa.y != pb.y || __float_as_uint(pa.y) != __float_as_uint(pb.y)) return ord_bits(pa.y) < ord_bits(pb.y);
    if (pa.z != pb.z || __float_as_uint(pa.z) != __float_as_uint(pb.z)) return ord_bits(pa.z) < ord_bits(pb.z);
    return ord_bits(map_payload<NC>(m, a)) < ord_bits(map_payload<NC>(m, b));
}
// candidate (nd, slot nidx) ranks before the entry (d, slot idx; idx < 0: empty) under the keyed order
__device__ __forceinline__ bool key_before(const MapView& m, float nd, int nidx, float d, int idx) {
    if (nd != d) return nd < d;
    return idx >= 0 && key_less(m, nidx, idx);
}
// y, z, intensity (p.w) of a below those of b: the keyed order of two fetched neighbours with equal x
__device__ __forceinline__ bool yzi_less(const float4& a, const float4& b) {
    if (ord_bits(a.y) != ord_bits(b.y)) return ord_bits(a.y) < ord_bits(b.y);
    if (ord_bits(a.z) != ord_bits(b.z)) return ord_bits(a.z) < ord_bits(b.z);
    return ord_bits(a.w) < ord_bits(b.w);
}
// The lane of `tied` (lanes whose candidates have bit-equal d2) that holds the smallest key; p: the lane's point, slot its slot
template <bool NC = true>
__device__ __forceinline__ int warp_key_min(const MapView& m, unsigned tied, const float4& p, int slot, int lane) {
    if ((tied & (tied - 1)) == 0) return __ffs(tied) - 1;
    bool in = (tied >> lane) & 1u;
    unsigned v = __reduce_min_sync(FULL, in ? ord_bits(p.x) : 0xffffffffu);
    in = in && ord_bits(p.x) == v;
    v = __reduce_min_sync(FULL, in ? ord_bits(p.y) : 0xffffffffu);
    in = in && ord_bits(p.y) == v;
    v = __reduce_min_sync(FULL, in ? ord_bits(p.z) : 0xffffffffu);
    in = in && ord_bits(p.z) == v;
    unsigned t = __ballot_sync(FULL, in);
    if (t & (t - 1)) {
        const unsigned ki = in ? ord_bits(map_payload<NC>(m, slot)) : 0xffffffffu;
        v = __reduce_min_sync(FULL, ki);
        t = __ballot_sync(FULL, in && ki == v);
    }
    return __ffs(t) - 1;
}

// Lane j < K holds the j-th best (distance, slot); other lanes hold +inf.  Mirrors MANUAL_HEAP
// + PointType_CMP (ikd_Tree.h:93-201) in effect: a candidate enters only if strictly closer
// than the current k-th best (ikd_Tree.cpp:1088); `w` caches that k-th best, warp-uniform.
// DET: the keyed order instead (see the tie rules above).
template <bool DET>
struct KBestT {
    static constexpr bool det = DET;
    float d;
    int idx;
    float w;
    int n;          // entries filled so far (warp-uniform)
    __device__ __forceinline__ void init() { d = INFINITY; idx = -1; w = INFINITY; n = 0; }
    __host__ __device__ static constexpr int cap() { return KNN_K; }
    __device__ __forceinline__ static constexpr bool gated(unsigned) { return false; }       // no distance gate
    // nd, nidx warp-uniform, nd < w (DET: or nd == w and a key below the k-th entry's)
    __device__ __forceinline__ void insert(float nd, int nidx, int lane, const MapView& m) {
        const float up_d = __shfl_up_sync(FULL, d, 1);
        const int up_i = __shfl_up_sync(FULL, idx, 1);
        if constexpr (!DET) {
            if (lane < KNN_K && nd < d) {
                const bool take_prev = lane > 0 && nd < up_d;
                d = take_prev ? up_d : nd;
                idx = take_prev ? up_i : nidx;
            }
        } else {
            const bool lt = lane < KNN_K && key_before(m, nd, nidx, d, idx);
            const bool up_lt = __shfl_up_sync(FULL, (int)lt, 1) != 0;
            if (lt) {
                const bool take_prev = lane > 0 && up_lt;
                d = take_prev ? up_d : nd;
                idx = take_prev ? up_i : nidx;
            }
        }
        w = __shfl_sync(FULL, d, KNN_K - 1);
    }
};
using KBest = KBestT<false>;

// The same list for a runtime k (1..32, lanes 0..k-1) with the distance gate of Nearest_Search's max_dist
// (ikd_Tree.cpp:1067-1088): a point is admitted while the list is not full when d2 <= md2, and once it is full when d2 is
// strictly below the k-th best.  gate = nextafterf(md2, +inf), so "strictly below w = min(k-th best, gate)" says both.
// Every box of the walk is pruned against w as well, which is the reference's box_dist > md2 cut-off.
constexpr int KNN_KMAX = 32;
template <bool DET>
struct KBestKT {
    static constexpr bool det = DET;
    float d;
    int idx;
    float w;
    int n;
    int k;
    float gate;
    __device__ __forceinline__ void init(int k_, float gate_) { d = INFINITY; idx = -1; w = gate_; n = 0; k = k_; gate = gate_; }
    __device__ __forceinline__ int cap() const { return k; }
    // while the list is not full, w is the gate: the first leaf of a query stops at it
    __device__ __forceinline__ bool gated(unsigned best) const { return best >= __float_as_uint(w); }
    __device__ __forceinline__ void insert(float nd, int nidx, int lane, const MapView& m) {
        const float up_d = __shfl_up_sync(FULL, d, 1);
        const int up_i = __shfl_up_sync(FULL, idx, 1);
        if constexpr (!DET) {
            if (lane < k && nd < d) {
                const bool take_prev = lane > 0 && nd < up_d;
                d = take_prev ? up_d : nd;
                idx = take_prev ? up_i : nidx;
            }
        } else {
            const bool lt = lane < k && key_before(m, nd, nidx, d, idx);
            const bool up_lt = __shfl_up_sync(FULL, (int)lt, 1) != 0;
            if (lt) {
                const bool take_prev = lane > 0 && up_lt;
                d = take_prev ? up_d : nd;
                idx = take_prev ? up_i : nidx;
            }
        }
        w = fminf(__shfl_sync(FULL, d, k - 1), gate);
    }
};
using KBestK = KBestKT<false>;

// Visit one leaf bucket (and its overflow chain): each lane scores one slot, then the
// (at most K) improving candidates are extracted in ascending order.
template <class KB = KBest>
__device__ __forceinline__ void knn_leaf(const MapView& m, int leaf, float qx, float qy, float qz,
                                         KB& kb, int lane) {
    while (leaf >= 0) {
        const float4 p = __ldg(&m.pts[leaf * LEAF + lane]);
        const int nxt = __ldg(&m.next[leaf]);
        unsigned key = slot_valid(p) ? __float_as_uint(sq_dist3(qx, qy, qz, p.x, p.y, p.z)) : INF_BITS;
        if (kb.n == 0) {
            // empty list (the first leaf of a query): the r-th smallest goes straight to lane r -- no merge
            unsigned best = INF_BITS;
#pragma unroll
            for (int r = 0; r < kb.cap(); r++) {
                best = __reduce_min_sync(FULL, key);
                if (best == INF_BITS || kb.gated(best)) break;
                int src;
                if constexpr (KB::det) src = warp_key_min(m, __ballot_sync(FULL, key == best), p, leaf * LEAF + lane, lane);
                else src = __ffs(__ballot_sync(FULL, key == best)) - 1;
                if (lane == r) { kb.d = __uint_as_float(best); kb.idx = leaf * LEAF + src; }
                if (lane == src) key = INF_BITS;
                kb.n = r + 1;
            }
            if (kb.n == kb.cap()) kb.w = __uint_as_float(best);
            leaf = nxt;
            continue;
        }
#pragma unroll 1
        while (true) {
            const unsigned best = __reduce_min_sync(FULL, key);
            int src, cidx;
            if constexpr (!KB::det) {
                if (best >= __float_as_uint(kb.w)) break;       // nothing strictly closer than the k-th best is left (covers the marker)
                src = __ffs(__ballot_sync(FULL, key == best)) - 1;
                cidx = leaf * LEAF + src;
            } else {
                if (best > __float_as_uint(kb.w) || best == INF_BITS) break;
                src = warp_key_min(m, __ballot_sync(FULL, key == best), p, leaf * LEAF + lane, lane);
                cidx = leaf * LEAF + src;
                if (best == __float_as_uint(kb.w)) {            // rare: ties the k-th best -- enters only with a smaller key
                    const int kth = __shfl_sync(FULL, kb.idx, kb.cap() - 1);
                    if (kth < 0 || !key_less(m, cidx, kth)) break;      // the smallest tied key does not: no tied point does
                }
            }
            // a walk seeded with candidates found elsewhere (knn_block) meets them again here: never list a slot twice
            if (!__any_sync(FULL, lane < kb.cap() && kb.idx == cidx)) kb.insert(__uint_as_float(best), cidx, lane, m);
            if (lane == src) key = INF_BITS;
        }
        leaf = nxt;
    }
}

// Visit node `node` of level L (its children are entities of level L-1).  Children are
// taken nearest-first and re-tested against the shrinking k-th best distance after each
// return -- the pruning rule of KD_TREE::Search (ikd_Tree.cpp:1097-1243).  The ordering key is
// the box distance with its low 5 mantissa bits traded for the lane id; a child is skipped only
// when even that rounded-DOWN distance is not below the k-th best, so pruning never drops a
// child that could matter (it may visit one whose distance ties the bound within 2^-18).  Under the keyed
// rule a point at exactly the k-th distance can still enter, so a child is skipped only when its rounded-down
// distance is strictly above the bound.
template <int L, class KB = KBest>
__device__ __forceinline__ void knn_node(const MapView& m, int node, float qx, float qy, float qz,
                                         KB& kb, int lane) {
    const int e = node * FAN + lane;
    unsigned key = 0xffffffffu;
    if (e < m.count[L - 1]) {
        const float4 lo = __ldg(&m.ebox[L - 1][2 * e]);
        const float4 hi = __ldg(&m.ebox[L - 1][2 * e + 1]);
        key = (__float_as_uint(box_dist3(qx, qy, qz, lo.x, lo.y, lo.z, hi.x, hi.y, hi.z)) & ~31u) | (unsigned)lane;
    }
#pragma unroll 1
    while (true) {
        const unsigned best = __reduce_min_sync(FULL, key);
        // keyed: a box at exactly the bound may hold a winner; one at +inf (an empty entity, or nothing left) never does
        if (KB::det ? (best & ~31u) > __float_as_uint(kb.w) || (best & ~31u) >= INF_BITS : (best & ~31u) >= __float_as_uint(kb.w)) break;
        const int c = best & 31;
        if (lane == c) key = 0xffffffffu;
        if constexpr (L == 1) knn_leaf<KB>(m, node * FAN + c, qx, qy, qz, kb, lane);
        else knn_node<L - 1, KB>(m, node * FAN + c, qx, qy, qz, kb, lane);
    }
}

// The root owns up to 64 entities (two per lane), which saves the two nearly empty top levels a
// strict 32-ary hierarchy would have (1 M points: 41 667 leaves -> 1 303 -> 41 -> root).
constexpr int ROOT_FAN = 64;

template <int L, class KB = KBest>
__device__ __forceinline__ void knn_root(const MapView& m, float qx, float qy, float qz, KB& kb, int lane) {
    const int cnt = m.count[L - 1];
    unsigned k0 = 0xffffffffu, k1 = 0xffffffffu;
    if (lane < cnt) {
        const float4 lo = __ldg(&m.ebox[L - 1][2 * lane]), hi = __ldg(&m.ebox[L - 1][2 * lane + 1]);
        k0 = (__float_as_uint(box_dist3(qx, qy, qz, lo.x, lo.y, lo.z, hi.x, hi.y, hi.z)) & ~63u) | (unsigned)lane;
    }
    if (lane + 32 < cnt) {
        const float4 lo = __ldg(&m.ebox[L - 1][2 * (lane + 32)]), hi = __ldg(&m.ebox[L - 1][2 * (lane + 32) + 1]);
        k1 = (__float_as_uint(box_dist3(qx, qy, qz, lo.x, lo.y, lo.z, hi.x, hi.y, hi.z)) & ~63u) | (unsigned)(lane + 32);
    }
#pragma unroll 1
    while (true) {
        const unsigned best = __reduce_min_sync(FULL, min(k0, k1));
        if (KB::det ? (best & ~63u) > __float_as_uint(kb.w) || (best & ~63u) >= INF_BITS : (best & ~63u) >= __float_as_uint(kb.w)) break;
        const int c = best & 63;
        if (lane == (c & 31)) { if (c < 32) k0 = 0xffffffffu; else k1 = 0xffffffffu; }
        if constexpr (L == 1) knn_leaf<KB>(m, c, qx, qy, qz, kb, lane);
        else knn_node<L - 1, KB>(m, c, qx, qy, qz, kb, lane);
    }
}

// Exact k-nearest-neighbour search for one query by one warp, continuing from the list in kb (empty after kb.init(), or seeded
// with live points and their true distances).
template <class KB = KBest>
__device__ __forceinline__ void knn_query_from(const MapView& m, float qx, float qy, float qz, KB& kb, int lane) {
    switch (m.n_levels) {
        case 1: knn_root<1, KB>(m, qx, qy, qz, kb, lane); break;
        case 2: knn_root<2, KB>(m, qx, qy, qz, kb, lane); break;
        case 3: knn_root<3, KB>(m, qx, qy, qz, kb, lane); break;
        case 4: knn_root<4, KB>(m, qx, qy, qz, kb, lane); break;
        case 5: knn_root<5, KB>(m, qx, qy, qz, kb, lane); break;
        default: knn_root<6, KB>(m, qx, qy, qz, kb, lane); break;
    }
}

template <bool DET = false>
__device__ __forceinline__ void knn_query(const MapView& m, float qx, float qy, float qz, KBestT<DET>& kb, int lane) {
    kb.init();
    knn_query_from(m, qx, qy, qz, kb, lane);
}

// ----------------------------------------------------------------------------- box query
// Half-open membership test of Search_by_range / Delete_by_range (ikd_Tree.cpp:796,1263):
//   vertex_min <= p < vertex_max  on every axis.
__device__ __forceinline__ bool in_box(const float4& p, const float* bmin, const float* bmax) {
    return bmin[0] <= p.x && bmax[0] > p.x && bmin[1] <= p.y && bmax[1] > p.y && bmin[2] <= p.z && bmax[2] > p.z;
}
// AABB-vs-box rejection, the negation of ikd_Tree.cpp:1253-1258
__device__ __forceinline__ bool box_overlaps(const float4& lo, const float4& hi, const float* bmin, const float* bmax) {
    if (bmax[0] <= lo.x || bmin[0] > hi.x) return false;
    if (bmax[1] <= lo.y || bmin[1] > hi.y) return false;
    if (bmax[2] <= lo.z || bmin[2] > hi.z) return false;
    return true;
}

// Functor interface: f.leaf(leaf_index) is called warp-uniformly for every main leaf whose
// AABB overlaps the box (the functor walks the overflow chain itself).
template <int L, class F>
__device__ __forceinline__ void box_node(const MapView& m, int node, const float* bmin, const float* bmax, F& f, int lane) {
    const int e = node * FAN + lane;
    bool hit = false;
    if (e < m.count[L - 1]) {
        const float4 lo = __ldg(&m.ebox[L - 1][2 * e]);
        const float4 hi = __ldg(&m.ebox[L - 1][2 * e + 1]);
        hit = box_overlaps(lo, hi, bmin, bmax);
    }
    unsigned mask = __ballot_sync(FULL, hit);
    while (mask) {
        const int c = __ffs(mask) - 1;
        mask &= mask - 1;
        if constexpr (L == 1) f.leaf(node * FAN + c);
        else box_node<L - 1, F>(m, node * FAN + c, bmin, bmax, f, lane);
    }
}
template <int L, class F>
__device__ __forceinline__ void box_root(const MapView& m, const float* bmin, const float* bmax, F& f, int lane) {
    const int cnt = m.count[L - 1];
#pragma unroll
    for (int half = 0; half < 2; half++) {
        const int e = lane + 32 * half;
        bool hit = false;
        if (e < cnt) {
            const float4 lo = __ldg(&m.ebox[L - 1][2 * e]), hi = __ldg(&m.ebox[L - 1][2 * e + 1]);
            hit = box_overlaps(lo, hi, bmin, bmax);
        }
        unsigned mask = __ballot_sync(FULL, hit);
        while (mask) {
            const int c = __ffs(mask) - 1 + 32 * half;
            mask &= mask - 1;
            if constexpr (L == 1) f.leaf(c);
            else box_node<L - 1, F>(m, c, bmin, bmax, f, lane);
        }
    }
}
template <class F>
__device__ __forceinline__ void box_query(const MapView& m, const float* bmin, const float* bmax, F& f, int lane) {
    switch (m.n_levels) {
        case 1: box_root<1, F>(m, bmin, bmax, f, lane); break;
        case 2: box_root<2, F>(m, bmin, bmax, f, lane); break;
        case 3: box_root<3, F>(m, bmin, bmax, f, lane); break;
        case 4: box_root<4, F>(m, bmin, bmax, f, lane); break;
        case 5: box_root<5, F>(m, bmin, bmax, f, lane); break;
        default: box_root<6, F>(m, bmin, bmax, f, lane); break;
    }
}

}  // namespace fl

// ============================================================================= cell directory: search
// One THREAD per query:
//   1. one hashed look-up finds the entry of the query's cell;
//   2. the points of its halo list (everything in the 3x3x3 block of cells around the query) are scored eight at a time, loads
//      first; the k best are kept in registers;
//   3. every point OUTSIDE the block is at least g = (distance from the query to the block's faces) away, so the k best found
//      are final when the k-th squared distance is strictly below g^2 (strict: the reference keeps the first of two
//      equidistant candidates, ikd_Tree.cpp:1088) -- tests/cell_directory_model.py pins the rule on the CPU.
// Anything else (no entry: nothing within a cell's width; fewer than k points; an over-full cell; coordinates beyond the key
// range) is NOT answered here: knn_block() pools those queries per block and its warps walk them through the BVH (knn_query_from).
// Squared distances use the same explicitly rounded float32 arithmetic as the BVH walk (sq_dist3): either route returns
// bit-identical distances.  All margins shrink the proven radius, never the searched set.
namespace fl {

__device__ __forceinline__ int cell_coord(float x, float inv_cell) {
    const float f = floorf(__fmul_rn(x, inv_cell));
    return (int)fminf(fmaxf(f, -(float)CELL_CLAMP), (float)CELL_CLAMP);
}
__host__ __device__ __forceinline__ unsigned long long cell_key(int ix, int iy, int iz) {
    return (1ull << 63) | ((unsigned long long)(unsigned)(ix + CELL_OFF) << 42) | ((unsigned long long)(unsigned)(iy + CELL_OFF) << 21) |
           (unsigned long long)(unsigned)(iz + CELL_OFF);
}
__device__ __forceinline__ unsigned cell_slot(unsigned long long key, unsigned cap) {
    const unsigned long long h = key * 0x9E3779B97F4A7C15ull;
    return __umulhi((unsigned)(h >> 32) ^ (unsigned)h, cap);
}

template <bool DET>
struct TBestT {                      // k best of one thread, ascending; empty entries: (+inf, -1)
    float d[KNN_K];
    int idx[KNN_K];
    __device__ __forceinline__ void init() {
#pragma unroll
        for (int i = 0; i < KNN_K; i++) { d[i] = INFINITY; idx[i] = -1; }
    }
    // the candidate ranks before the k-th entry: it enters the list
    __device__ __forceinline__ bool admits(const MapView& m, float nd, int nidx) const {
        if constexpr (DET) return key_before(m, nd, nidx, d[KNN_K - 1], idx[KNN_K - 1]);
        else return nd < d[KNN_K - 1];
    }
    // admits(nd, nidx); equal distances keep their arrival order (DET: their key order)
    __device__ __forceinline__ void insert(float nd, int nidx, const MapView& m) {
        // a halo list may name a slot twice (a slot re-used by a later insert keeps its old listings): never keep it twice
        bool dup = false;
#pragma unroll
        for (int i = 0; i < KNN_K; i++) dup |= idx[i] == nidx;
        if (dup) return;
        if constexpr (!DET) {
#pragma unroll
            for (int i = KNN_K - 1; i > 0; i--) {
                const bool shift = nd < d[i - 1];
                const bool here = !shift && nd < d[i];
                d[i] = shift ? d[i - 1] : (here ? nd : d[i]);
                idx[i] = shift ? idx[i - 1] : (here ? nidx : idx[i]);
            }
            if (nd < d[0]) { d[0] = nd; idx[0] = nidx; }
        } else {
            bool lt[KNN_K];
#pragma unroll
            for (int i = 0; i < KNN_K; i++) lt[i] = key_before(m, nd, nidx, d[i], idx[i]);
#pragma unroll
            for (int i = KNN_K - 1; i > 0; i--) {
                const bool shift = lt[i - 1];
                const bool here = !shift && lt[i];
                d[i] = shift ? d[i - 1] : (here ? nd : d[i]);
                idx[i] = shift ? idx[i - 1] : (here ? nidx : idx[i]);
            }
            if (lt[0]) { d[0] = nd; idx[0] = nidx; }
        }
    }
};
using TBest = TBestT<false>;

// the entry of cell `key`: (start, cnt) of its halo list.  Returns 1: usable; 0: no entry (no point within a cell's width of
// that cell); -1: over-full (or being set up) -- the BVH walk must answer
__device__ __forceinline__ int cell_list(const CellDir& D, unsigned long long key, int& start, int& cnt) {
    const uint4* tab = reinterpret_cast<const uint4*>(D.tab);
    unsigned s = cell_slot(key, D.cap);
    uint4 e;
    unsigned probes = 0;
    while (true) {
        e = __ldg(&tab[s]);
        const unsigned long long k = (unsigned long long)e.x | ((unsigned long long)e.y << 32);
        if (k == key) break;
        if (k == 0ull || ++probes >= D.cap) return 0;
        s = (s + 1 == D.cap) ? 0u : s + 1;
    }
    start = (int)e.z; cnt = (int)(e.w & 0xffffu);
    const int room = (int)(e.w >> 16);
    return (start >= 0 && cnt <= room && cnt > 0) ? 1 : -1;
}

// one candidate (a deleted point keeps its listings: it is skipped by its flag)
template <bool DET>
__device__ __forceinline__ void cell_consider(const MapView& m, const float4& p, int idx, float qx, float qy, float qz, TBestT<DET>& kb) {
    if (slot_valid(p)) {
        const float dd = sq_dist3(qx, qy, qz, p.x, p.y, p.z);
        if (kb.admits(m, dd, idx)) kb.insert(dd, idx, m);
    }
}

// Score the halo list [start, start + cnt), eight candidates at a time: their point loads are issued together and the indices of
// the next eight are fetched while these are scored (a scan is only a few warps per SM: the chain of dependent loads of one
// thread IS the run time -- probe, first indices, then one round trip per eight candidates).
template <bool DET>
__device__ __forceinline__ void cell_scan_list(const MapView& m, int start, int cnt, float qx, float qy, float qz, TBestT<DET>& kb) {
    const int4* list = reinterpret_cast<const int4*>(m.dir.lists + start);
    const int nchunks = (cnt + 7) >> 3;
    int4 ia = __ldg(&list[0]), ib = make_int4(0, 0, 0, 0);
    if (cnt > 4) ib = __ldg(&list[1]);
#pragma unroll 1
    for (int c = 0; c < nchunks; c++) {
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
        if (n8 > 8) na = __ldg(&list[2 * c + 2]);
        if (n8 > 12) nb = __ldg(&list[2 * c + 3]);
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

// A lower bound g on the distance from the query, in cell (ix, iy, iz), to every point outside the 3x3x3 block of cells around
// that cell.  The distances from the query to the faces of its own cell are shrunk by more than any rounding of the cell
// arithmetic.
__device__ __forceinline__ float cell_block_dist(const CellDir& D, float qx, float qy, float qz, int ix, int iy, int iz) {
    const float c = D.cell;
    const float marg = 4e-6f * (fmaxf(fmaxf(fabsf(qx), fabsf(qy)), fabsf(qz)) + 2.f * c);
    const float lox = fmaxf(qx - (float)ix * c - marg, 0.f), hix = fmaxf((float)(ix + 1) * c - qx - marg, 0.f);
    const float loy = fmaxf(qy - (float)iy * c - marg, 0.f), hiy = fmaxf((float)(iy + 1) * c - qy - marg, 0.f);
    const float loz = fmaxf(qz - (float)iz * c - marg, 0.f), hiz = fmaxf((float)(iz + 1) * c - qz - marg, 0.f);
    const float c1 = c - marg;
    const float gx = fminf(lox, hix) + c1, gy = fminf(loy, hiy) + c1, gz = fminf(loz, hiz) + c1;      // distance to the block's nearest face, per axis
    return fminf(fminf(gx, gy), gz);
}

// k-NN of one query by one thread.  Returns true when kb is PROVEN to be the exact answer.  The proof is strict: a point
// outside the block is farther than the k-th best, so it can neither be closer nor tie it (the keyed rule admits ties).
template <bool DET>
__device__ __forceinline__ bool cell_knn(const MapView& m, float qx, float qy, float qz, TBestT<DET>& kb) {
    const CellDir& D = m.dir;
    kb.init();
    if (D.cap == 0u) return false;
    const float inv = D.inv_cell;
    const int ix = cell_coord(qx, inv), iy = cell_coord(qy, inv), iz = cell_coord(qz, inv);
    if (abs(ix) >= CELL_CLAMP - 1 || abs(iy) >= CELL_CLAMP - 1 || abs(iz) >= CELL_CLAMP - 1) return false;
    // ---- 1. + 2. the halo list of the query's cell: every point of the 3x3x3 block of cells around it
    int start, cnt;
    if (cell_list(D, cell_key(ix, iy, iz), start, cnt) <= 0) return false;
    cell_scan_list(m, start, cnt, qx, qy, qz, kb);
    if (kb.idx[KNN_K - 1] < 0) return false;
    // ---- 3. proof: every point outside the block is at least g away
    const float g = cell_block_dist(D, qx, qy, qz, ix, iy, iz);
    return kb.d[KNN_K - 1] < g * g;
}

// Exact k-NN for the queries of a thread block (one per thread; `active` masks the tail).  The thread search answers what it can
// prove.  The rest -- typically a handful of queries in sparse corners of the map, often neighbours in the scan and therefore
// in the same warp -- is pooled in shared memory and walked through the BVH by ALL warps of the block, one query per warp at a
// time (a cold walk is ~10 dependent memory round trips: five of them in one warp would make that warp the kernel's tail).
// Block-wide: every thread of the block must call it (two barriers); `phase` is the caller's call counter (block-uniform,
// starts at 0 with W.n[0] == W.n[1] == 0).
constexpr int WALK_POOL = 64;
struct WalkPool {
    int n[2];                      // the counter of the current call and, being cleared, that of the next (see knn_block)
    int who[WALK_POOL];
    float x[WALK_POOL], y[WALK_POOL], z[WALK_POOL];
    float rd[WALK_POOL][KNN_K];    // in: the k candidates the thread search found (a bound for the walk; +inf / -1 when it found fewer); out: the answer
    int ri[WALK_POOL][KNN_K];
};
template <bool DET>
__device__ __forceinline__ void knn_block(const MapView& m, bool active, float qx, float qy, float qz, TBestT<DET>& kb, WalkPool& W, int& phase) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    bool exact = true;
    if (active) exact = cell_knn(m, qx, qy, qz, kb);
    else kb.init();
    int mine = -1;
    int* counter = &W.n[phase & 1];
    if (active && !exact) {
        mine = atomicAdd(counter, 1);
        if (mine < WALK_POOL) {
            W.who[mine] = (int)threadIdx.x; W.x[mine] = qx; W.y[mine] = qy; W.z[mine] = qz;
            const bool full = kb.idx[KNN_K - 1] >= 0;         // seed only with a complete list (its k-th distance bounds the walk)
#pragma unroll
            for (int j = 0; j < KNN_K; j++) { W.rd[mine][j] = full ? kb.d[j] : INFINITY; W.ri[mine][j] = full ? kb.idx[j] : -1; }
        }
    }
    __syncthreads();
    const int total = *counter, n = min(total, WALK_POOL);
    if (threadIdx.x == 0) W.n[(phase + 1) & 1] = 0;     // nobody touches the other counter before the next call's first barrier
    phase++;
    for (int i = warp; i < n; i += nwarps) {
        // the walk starts from what the thread search found: with the k-th distance as its bound it only enters boxes that cut
        // the known ball (a handful of dependent loads instead of a full descent)
        KBestT<DET> w;
        w.init();
        if (lane < KNN_K) { w.d = W.rd[i][lane]; w.idx = W.ri[i][lane]; }
        w.w = __shfl_sync(FULL, w.d, KNN_K - 1);
        w.n = w.w < INFINITY ? KNN_K : 0;
        knn_query_from(m, W.x[i], W.y[i], W.z[i], w, lane);
        __syncwarp();
        if (lane < KNN_K) { W.rd[i][lane] = w.d; W.ri[i][lane] = w.idx; }
    }
    // more unproven queries than the pool holds (a scan far from the map): their own warp walks them
    unsigned todo = __ballot_sync(FULL, mine >= WALK_POOL);
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
    if (mine >= 0 && mine < WALK_POOL) {
#pragma unroll
        for (int j = 0; j < KNN_K; j++) { kb.d[j] = W.rd[mine][j]; kb.idx[j] = W.ri[mine][j]; }
    }
    if (threadIdx.x == 0 && total && m.dir.cap && m.dir.n_walked) atomicAdd(m.dir.n_walked, total);
}

// The neighbours as the caller sees them: coordinates + intensity, nearest first; candidates whose squared distances
// differ by less than 1e-10 are ordered by x like PointType_CMP does for the reference's heap (ikd_Tree.h:102-108).  DET: those
// with equal x as well by (y, z, intensity), so the order is a function of the neighbours alone.
template <bool DET>
__device__ __forceinline__ int knn_fetch(const MapView& m, TBestT<DET>& kb, float4 (&p)[KNN_K]) {
    int cnt = 0;
#pragma unroll
    for (int j = 0; j < KNN_K; j++) {
        p[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (kb.idx[j] >= 0) { p[j] = __ldg(&m.pts[kb.idx[j]]); p[j].w = __ldg(&m.payload[kb.idx[j]]); cnt++; }
    }
    bool tie = false;
#pragma unroll
    for (int j = 0; j + 1 < KNN_K; j++) tie |= kb.idx[j + 1] >= 0 && fabsf(kb.d[j + 1] - kb.d[j]) < 1e-10f;
    if (tie) {
#pragma unroll
        for (int pass = 0; pass < KNN_K - 1; pass++) {
#pragma unroll
            for (int j = 0; j + 1 < KNN_K - pass; j++) {
                if (kb.idx[j + 1] >= 0 && fabsf(kb.d[j + 1] - kb.d[j]) < 1e-10f &&
                    (p[j + 1].x < p[j].x || (DET && p[j + 1].x == p[j].x && yzi_less(p[j + 1], p[j])))) {
                    const float4 tp = p[j]; p[j] = p[j + 1]; p[j + 1] = tp;
                    const float td = kb.d[j]; kb.d[j] = kb.d[j + 1]; kb.d[j + 1] = td;
                    const int ti = kb.idx[j]; kb.idx[j] = kb.idx[j + 1]; kb.idx[j + 1] = ti;
                }
            }
        }
    }
    return cnt;
}

// the same for the warp-cooperative list of the BVH walk (lane j < K holds neighbour j)
template <class KB = KBest>
__device__ __forceinline__ int knn_fetch_warp(const MapView& m, KB& kb, float4& p, int lane) {
    const bool have = lane < kb.cap() && kb.idx >= 0;
    p = make_float4(0.f, 0.f, 0.f, 0.f);
    if (have) { p = __ldg(&m.pts[kb.idx]); p.w = __ldg(&m.payload[kb.idx]); }
    const int cnt = __popc(__ballot_sync(FULL, have));
    const float dn = __shfl_down_sync(FULL, kb.d, 1);
    const bool tie = lane + 1 < cnt && fabsf(dn - kb.d) < 1e-10f;
    if (__any_sync(FULL, tie)) {                    // odd-even transposition over the (at most K) entries
#pragma unroll
        for (int pass = 0; pass < kb.cap(); pass++) {
            const int partner = ((lane + pass) & 1) ? lane - 1 : lane + 1;
            const int pl = min(max(partner, 0), 31);
            const float od = __shfl_sync(FULL, kb.d, pl);
            const int oi = __shfl_sync(FULL, kb.idx, pl);
            const float ox = __shfl_sync(FULL, p.x, pl), oy = __shfl_sync(FULL, p.y, pl), oz = __shfl_sync(FULL, p.z, pl), ow = __shfl_sync(FULL, p.w, pl);
            const bool both = partner >= 0 && lane < cnt && partner < cnt;
            if (both && fabsf(od - kb.d) < 1e-10f) {
                const bool lower = lane < partner;                                    // the lower lane keeps the smaller x
                bool take = lower ? (ox < p.x) : (ox > p.x);
                if constexpr (KB::det) {
                    const float4 o = make_float4(ox, oy, oz, ow);
                    if (ox == p.x) take = lower ? yzi_less(o, p) : yzi_less(p, o);
                }
                if (take) { kb.d = od; kb.idx = oi; p = make_float4(ox, oy, oz, ow); }
            }
        }
    }
    return cnt;
}

// Seed of a runtime-k query (KBestK, empty on entry) from the cell directory, by one warp: lane 0 finds the query's cell, the
// warp scores its halo list 32 entries at a time and merges the admissible points like knn_leaf does.  Returns true when the
// list is PROVEN to be the exact answer: every point outside the block is at least g away (cell_block_dist), so the list is
// final when it holds k entries and the k-th is below g^2, or when md2 < g^2 (every admissible point lies in the block, however
// few there are).  Otherwise the list seeds the BVH walk (knn_query_from), which only adds what the block did not hold.
template <bool DET>
__device__ __forceinline__ bool knn_seed_k(const MapView& m, float qx, float qy, float qz, float md2, KBestKT<DET>& kb, int lane) {
    const CellDir& D = m.dir;
    if (D.cap == 0u) return false;
    const float inv = D.inv_cell;
    const int ix = cell_coord(qx, inv), iy = cell_coord(qy, inv), iz = cell_coord(qz, inv);
    if (abs(ix) >= CELL_CLAMP - 1 || abs(iy) >= CELL_CLAMP - 1 || abs(iz) >= CELL_CLAMP - 1) return false;
    int start = 0, cnt = 0, ok = 0;
    if (lane == 0) ok = cell_list(D, cell_key(ix, iy, iz), start, cnt);
    ok = __shfl_sync(FULL, ok, 0);
    if (ok <= 0) return false;
    start = __shfl_sync(FULL, start, 0);
    cnt = __shfl_sync(FULL, cnt, 0);
#pragma unroll 1
    for (int b = 0; b < cnt; b += 32) {
        unsigned key = INF_BITS;
        int slot = -1;
        float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
        if (b + lane < cnt) {
            slot = __ldg(&D.lists[start + b + lane]);
            p = __ldg(&m.pts[slot]);
            if (slot_valid(p)) key = __float_as_uint(sq_dist3(qx, qy, qz, p.x, p.y, p.z));
        }
#pragma unroll 1
        while (true) {
            const unsigned best = __reduce_min_sync(FULL, key);
            int src, cidx;
            if constexpr (!DET) {
                if (best >= __float_as_uint(kb.w)) break;
                src = __ffs(__ballot_sync(FULL, key == best)) - 1;
                cidx = __shfl_sync(FULL, slot, src);
            } else {                                    // the keyed rule, as in knn_leaf
                if (best > __float_as_uint(kb.w) || best == INF_BITS) break;
                src = warp_key_min(m, __ballot_sync(FULL, key == best), p, slot, lane);
                cidx = __shfl_sync(FULL, slot, src);
                if (best == __float_as_uint(kb.w)) {
                    const int kth = __shfl_sync(FULL, kb.idx, kb.k - 1);
                    if (kth < 0 || !key_less(m, cidx, kth)) break;
                }
            }
            // a list may name a slot twice: never list it twice
            if (!__any_sync(FULL, lane < kb.k && kb.idx == cidx)) kb.insert(__uint_as_float(best), cidx, lane, m);
            if (lane == src) key = INF_BITS;
        }
    }
    kb.n = __popc(__ballot_sync(FULL, kb.idx >= 0));
    const float g = cell_block_dist(D, qx, qy, qz, ix, iy, iz);
    const float g2 = g * g;
    return __shfl_sync(FULL, kb.d, kb.k - 1) < g2 || md2 < g2;
}

}  // namespace fl
