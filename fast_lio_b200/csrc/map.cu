// Device point map: build / refit / search / box-delete / incremental insert.
// H100-native replacement for the subset of KD_TREE<PointType> that FAST-LIO's
// laserMapping.cpp calls (reference include/ikd-Tree/ikd_Tree.cpp).  See map.cuh for the
// memory layout and DESIGN.md for the rationale.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdlib>
#include <vector>

#include "map.h"

namespace fl {

// ============================================================================= errors
static thread_local char g_last_error[512] = "";
void set_last_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
    va_end(ap);
}
const char* last_error() { return g_last_error; }

// ============================================================================= DeviceBuffer
int DeviceBuffer::reserve(size_t want) {
    if (want <= bytes) return FL_OK;
    size_t grow = std::max(want, bytes + bytes / 2);
    if (ptr) { FL_CUDA(cudaFree(ptr)); ptr = nullptr; bytes = 0; }
    FL_CUDA(cudaMalloc(&ptr, grow));
    bytes = grow;
    return FL_OK;
}
void DeviceBuffer::release() {
    if (ptr) cudaFree(ptr);
    ptr = nullptr; bytes = 0;
}

// counters_ layout
enum Counter { C_LEAF_USED = 0, C_DELETED, C_ADDED, C_GROUPS, C_NINSERT, C_TOMB, C_ERROR, C_COMPACT,
               C_DIR_CELLS, C_DIR_POOL, C_DIR_CROWDED, C_DIR_ERROR, C_DIR_WALKED, C_REMOVED, C_REVIVED, C_NFIX,
               // device forms of Add_Points: validnum / lazily deleted points (n_valid_, n_tomb_ on the device), the batch
               // sizes as read (RA, RB) and as applied (NA, NB: 0 when the plan refused), the plan's counts, its verdict, and
               // "maintenance due" (the host form would have re-packed or re-listed); C_REFUSED: a call was refused since the last
               // fl_map_maintain (sticky, unlike C_SKIP), C_NEED: the list-pool need the plan last computed
               C_VALID, C_TOMBS, C_RA, C_RB, C_NA, C_NB, C_MISS, C_FIXES, C_SKIP, C_DUE, C_REFUSED, C_NEED,
               // device form of Delete_Point_Boxes: the box count the plan let through (0 when it refused), and its verdict
               C_DEL_NB, C_DEL_SKIP, C_COUNT = 32 };

// ============================================================================= kernels
// ----------------------------------------------------------------------------- k-d partition build
// Top-down, level-synchronous: every level (1) bounds each segment, (2) sorts all points by
// (segment, coordinate on the segment's longest axis) with one radix sort, (3) splits each
// segment at a leaf boundary.  A segment owns a contiguous range of sorted points [p0, p1) and a
// contiguous range of leaves [a, b); splits are placed on 32^k-aligned leaf boundaries so that
// the five binary levels below any 32-wide node are exactly its children.
struct Segment { int p0, p1, a, b; };

__device__ __forceinline__ unsigned flip_float(float f) {
    const unsigned u = __float_as_uint(f);
    return u ^ ((u >> 31) ? 0xffffffffu : 0x80000000u);
}
// split leaf of a segment covering leaves [a, b), b - a >= 2
// pmax = leaves under one child of the root: above it the root's (up to 64) children are split
// evenly instead of on powers of 32
__host__ __device__ __forceinline__ int split_leaf(int a, int b, long long pmax) {
    const int span = b - a;
    long long p = 1;
    while (p * FAN < span && p * FAN <= pmax) p *= FAN;
    const int nch = (int)((span + p - 1) / p);
    return a + (int)((nch / 2) * p);
}

__global__ void k_kd_init(int n, unsigned* __restrict__ idx, int* __restrict__ segid, Segment* seg, int n_leaves) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { idx[i] = (unsigned)i; segid[i] = 0; }
    if (i == 0) { seg[0].p0 = 0; seg[0].p1 = n; seg[0].a = 0; seg[0].b = n_leaves; }
}
__global__ void k_kd_bbox_init(float* __restrict__ bbox, int nseg) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nseg * 6) bbox[i] = (i % 6) < 3 ? INFINITY : -INFINITY;
}
__global__ void k_kd_bbox(const float4* __restrict__ src, const unsigned* __restrict__ idx, const int* __restrict__ segid,
                          int n, float* __restrict__ bbox) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const bool live = r < n;
    int s = -1;
    float v[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};
    if (live) {
        s = segid[r];
        const float4 p = src[idx[r]];
        v[0] = v[3] = p.x; v[1] = v[4] = p.y; v[2] = v[5] = p.z;
    }
    // positions are ordered by segment: usually the whole warp shares one segment
    const int s0 = __shfl_sync(FULL, s, 0);
    if (__all_sync(FULL, s == s0)) {
        if (s0 < 0) return;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
            for (int a = 0; a < 3; a++) {
                v[a] = fminf(v[a], __shfl_xor_sync(FULL, v[a], o));
                v[3 + a] = fmaxf(v[3 + a], __shfl_xor_sync(FULL, v[3 + a], o));
            }
        }
        if (lane < 3) atomic_min_float(&bbox[s0 * 6 + lane], lane == 0 ? v[0] : (lane == 1 ? v[1] : v[2]));
        else if (lane < 6) atomic_max_float(&bbox[s0 * 6 + lane], lane == 3 ? v[3] : (lane == 4 ? v[4] : v[5]));
    } else if (live) {
#pragma unroll
        for (int a = 0; a < 3; a++) { atomic_min_float(&bbox[s * 6 + a], v[a]); atomic_max_float(&bbox[s * 6 + 3 + a], v[3 + a]); }
    }
}
__global__ void k_kd_keys(const float4* __restrict__ src, const unsigned* __restrict__ idx, const int* __restrict__ segid, int n,
                          const float* __restrict__ bbox, unsigned long long* __restrict__ keys, unsigned* __restrict__ vals) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const int s = segid[r];
    const float* b = &bbox[s * 6];
    // longest axis, first one wins ties (ikd_Tree.cpp:704-707)
    const float ex = b[3] - b[0], ey = b[4] - b[1], ez = b[5] - b[2];
    int axis = 0; float best = ex;
    if (ey > best) { best = ey; axis = 1; }
    if (ez > best) { axis = 2; }
    const unsigned id = idx[r];
    const float4 p = src[id];
    const float c = axis == 0 ? p.x : (axis == 1 ? p.y : p.z);
    keys[r] = ((unsigned long long)(unsigned)s << 32) | flip_float(c);
    vals[r] = id;
}
__global__ void k_kd_split(const Segment* __restrict__ in, Segment* __restrict__ out, int nseg, int fill, long long pmax) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= nseg) return;
    const Segment g = in[s];
    Segment l = g, r;
    r.p0 = r.p1 = g.p1; r.a = r.b = g.b;
    if (g.b - g.a >= 2) {
        const int m = split_leaf(g.a, g.b, pmax);
        long long cut = (long long)g.p0 + (long long)(m - g.a) * fill;
        if (cut > g.p1) cut = g.p1;
        l.p1 = (int)cut; l.b = m;
        r.p0 = (int)cut; r.p1 = g.p1; r.a = m; r.b = g.b;
    }
    out[2 * s] = l;
    out[2 * s + 1] = r;
}
__global__ void k_kd_assign(const unsigned long long* __restrict__ sorted_keys, int n, const Segment* __restrict__ next_seg,
                            int* __restrict__ segid) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const int s = (int)(sorted_keys[r] >> 32);
    segid[r] = 2 * s + (r >= next_seg[2 * s].p1 ? 1 : 0);
}

// Scatter the partitioned points into their leaf buckets; clear every other slot, the overflow
// pool and the chains.
__global__ void k_clear_leaves(MapView m) {
    const long long total = (long long)m.leaf_cap * LEAF;
    for (long long slot = blockIdx.x * (long long)blockDim.x + threadIdx.x; slot < total;
         slot += (long long)gridDim.x * blockDim.x) {
        m.pts[slot] = make_float4(0.f, 0.f, 0.f, __int_as_float(0));
        m.payload[slot] = 0.f;
        if ((slot % LEAF) == 0) m.next[slot / LEAF] = -1;
    }
}
__global__ void k_fill_leaves(MapView m, const float4* __restrict__ src, const unsigned* __restrict__ idx,
                              const int* __restrict__ segid, const Segment* __restrict__ seg, int n) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const Segment g = seg[segid[r]];
    const float4 p = src[idx[r]];
    const long long slot = (long long)g.a * LEAF + (r - g.p0);
    m.pts[slot] = make_float4(p.x, p.y, p.z, __int_as_float(1));
    m.payload[slot] = p.w;
}

// One warp per main leaf: AABB of the valid points of the leaf and of its overflow chain.  gate (may be null): the device form of
// Delete_Point_Boxes refits only when its deleted count there is non-zero, as the host form does.
__global__ void k_refit_leaves(MapView m, const int* __restrict__ gate) {
    if (gate && *gate == 0) return;
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    for (int leaf = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; leaf < m.n_main; leaf += warps) {
        float lx = INFINITY, ly = INFINITY, lz = INFINITY, hx = -INFINITY, hy = -INFINITY, hz = -INFINITY;
        int l = leaf;
        while (l >= 0) {
            const float4 p = m.pts[l * LEAF + lane];
            if (slot_valid(p)) {
                lx = fminf(lx, p.x); ly = fminf(ly, p.y); lz = fminf(lz, p.z);
                hx = fmaxf(hx, p.x); hy = fmaxf(hy, p.y); hz = fmaxf(hz, p.z);
            }
            l = m.next[l];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lx = fminf(lx, __shfl_xor_sync(FULL, lx, o)); ly = fminf(ly, __shfl_xor_sync(FULL, ly, o));
            lz = fminf(lz, __shfl_xor_sync(FULL, lz, o)); hx = fmaxf(hx, __shfl_xor_sync(FULL, hx, o));
            hy = fmaxf(hy, __shfl_xor_sync(FULL, hy, o)); hz = fmaxf(hz, __shfl_xor_sync(FULL, hz, o));
        }
        if (lane == 0) {
            m.ebox[0][2 * leaf] = make_float4(lx, ly, lz, 0.f);
            m.ebox[0][2 * leaf + 1] = make_float4(hx, hy, hz, 0.f);
        }
    }
}

// One warp per entity of level k (k >= 1): union of its <= 32 children boxes.
__global__ void k_refit_level(MapView m, int k, const int* __restrict__ gate) {
    if (gate && *gate == 0) return;
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    for (int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < m.count[k]; e += warps) {
        const int c = e * FAN + lane;
        float lx = INFINITY, ly = INFINITY, lz = INFINITY, hx = -INFINITY, hy = -INFINITY, hz = -INFINITY;
        if (c < m.count[k - 1]) {
            const float4 lo = m.ebox[k - 1][2 * c], hi = m.ebox[k - 1][2 * c + 1];
            lx = lo.x; ly = lo.y; lz = lo.z; hx = hi.x; hy = hi.y; hz = hi.z;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lx = fminf(lx, __shfl_xor_sync(FULL, lx, o)); ly = fminf(ly, __shfl_xor_sync(FULL, ly, o));
            lz = fminf(lz, __shfl_xor_sync(FULL, lz, o)); hx = fmaxf(hx, __shfl_xor_sync(FULL, hx, o));
            hy = fmaxf(hy, __shfl_xor_sync(FULL, hy, o)); hz = fmaxf(hz, __shfl_xor_sync(FULL, hz, o));
        }
        if (lane == 0) {
            m.ebox[k][2 * e] = make_float4(lx, ly, lz, 0.f);
            m.ebox[k][2 * e + 1] = make_float4(hx, hy, hz, 0.f);
        }
    }
}

// ----------------------------------------------------------------------------- cell directory (map.cuh)
// find the entry of `key`, claiming a free one if the cell is new; returns its table index (0xffffffff: table full)
__device__ __forceinline__ unsigned dir_claim(const CellDir& D, unsigned long long key, int* counters, bool* fresh = nullptr) {
    unsigned s = cell_slot(key, D.cap);
    for (unsigned probes = 0; probes < D.cap; probes++) {
        const unsigned long long old = atomicCAS(&D.tab[s].key, 0ull, key);
        if (old == 0ull) { atomicAdd(&counters[C_DIR_CELLS], 1); if (fresh) *fresh = true; return s; }
        if (old == key) return s;
        s = (s + 1 == D.cap) ? 0u : s + 1;
    }
    atomicExch(&counters[C_DIR_ERROR], 1);      // table full (the host sizes it so that this cannot happen)
    return 0xffffffffu;
}
__device__ __forceinline__ unsigned dir_find(const CellDir& D, unsigned long long key) {
    unsigned s = cell_slot(key, D.cap);
    for (unsigned probes = 0; probes < D.cap; probes++) {
        const unsigned long long k = D.tab[s].key;
        if (k == key) return s;
        if (k == 0ull) break;
        s = (s + 1 == D.cap) ? 0u : s + 1;
    }
    return 0xffffffffu;
}
// the 27 cells whose halo lists a point belongs to: neighbour t of its own cell
__device__ __forceinline__ unsigned long long halo_key(const CellDir& D, const float4& p, int t) {
    return cell_key(cell_coord(p.x, D.inv_cell) + t % 3 - 1, cell_coord(p.y, D.inv_cell) + (t / 3) % 3 - 1, cell_coord(p.z, D.inv_cell) + t / 9 - 1);
}
__device__ __forceinline__ bool same_cell(const CellDir& D, const float4& a, const float4& b) {
    return cell_coord(a.x, D.inv_cell) == cell_coord(b.x, D.inv_cell) && cell_coord(a.y, D.inv_cell) == cell_coord(b.y, D.inv_cell) &&
           cell_coord(a.z, D.inv_cell) == cell_coord(b.z, D.inv_cell);
}

// (re)list, three passes so that no thread ever waits for another:
//   1. every live slot claims its 27 cells and counts itself in each (cnt_cap holds a plain count);
//   2. every cell gets room for its count + 25 % (a multiple of 4 indices) out of the list pool, counts restart;
//   3. every live slot appends its index to its 27 lists.
__global__ void k_halo_count(MapView m, int n_leaf_used, int* counters) {
    const long long total = (long long)n_leaf_used * LEAF;
    for (long long slot = blockIdx.x * (long long)blockDim.x + threadIdx.x; slot < total; slot += (long long)gridDim.x * blockDim.x) {
        const float4 p = m.pts[slot];
        if (!slot_valid(p)) continue;
#pragma unroll 1
        for (int t = 0; t < 27; t++) {
            const unsigned e = dir_claim(m.dir, halo_key(m.dir, p, t), counters);
            if (e != 0xffffffffu) atomicAdd(&m.dir.tab[e].cnt_cap, 1u);
        }
    }
}
__global__ void k_halo_alloc(MapView m, int* counters) {
    for (unsigned e = blockIdx.x * blockDim.x + threadIdx.x; e < m.dir.cap; e += gridDim.x * blockDim.x) {
        CellEntry& E = m.dir.tab[e];
        if (E.key == 0ull) continue;
        const int cnt = (int)E.cnt_cap;
        if (cnt > HALO_MAX) { E.start = -1; E.cnt_cap = 0u; atomicAdd(&counters[C_DIR_CROWDED], 1); continue; }
        const int room = (cnt + max(8, cnt / 4) + 3) & ~3;
        const int start = atomicAdd(&counters[C_DIR_POOL], room);
        if (start + room > m.dir.lists_cap) { E.start = -1; E.cnt_cap = 0u; atomicExch(&counters[C_DIR_ERROR], 1); continue; }
        E.start = start;
        E.cnt_cap = (unsigned)room << 16;
    }
}
__global__ void k_halo_fill(MapView m, int n_leaf_used) {
    const long long total = (long long)n_leaf_used * LEAF;
    for (long long slot = blockIdx.x * (long long)blockDim.x + threadIdx.x; slot < total; slot += (long long)gridDim.x * blockDim.x) {
        const float4 p = m.pts[slot];
        if (!slot_valid(p)) continue;
#pragma unroll 1
        for (int t = 0; t < 27; t++) {
            const unsigned e = dir_find(m.dir, halo_key(m.dir, p, t));
            if (e == 0xffffffffu) continue;
            CellEntry& E = m.dir.tab[e];
            if (E.start < 0) continue;
            const unsigned old = atomicAdd(&E.cnt_cap, 1u);
            const int pos = (int)(old & 0xffffu), room = (int)(old >> 16);
            if (pos < room) m.dir.lists[E.start + pos] = (int)slot;
        }
    }
}
// The batch size of a kernel of Add_Points: n (host form), or *n_dev clamped to [0, n] (device forms: n is the n_max the grid
// was sized from, *n_dev the count some earlier kernel of the call left in device memory).
__device__ __forceinline__ int batch_count(int n, const int* __restrict__ n_dev) {
    return n_dev ? min(max(*n_dev, 0), n) : n;
}
// incremental, two kernels (claim, then append) so that nobody waits for a list that is still being set up.
// One warp per inserted point, lane t < 27 its t-th cell.  slots[i] < 0: the point could not be placed.
__global__ void __launch_bounds__(256) k_halo_claim(MapView m, const float4* __restrict__ pts, const int* __restrict__ slots, int n,
                                                     const int* __restrict__ n_dev, int* counters) {
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    n = batch_count(n, n_dev);
    for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        if (slots[i] < 0 || lane >= 27) continue;
        bool fresh = false;
        const unsigned e = dir_claim(m.dir, halo_key(m.dir, pts[i], lane), counters, &fresh);
        if (e == 0xffffffffu || !fresh) continue;
        CellEntry& E = m.dir.tab[e];
        const int start = atomicAdd(&counters[C_DIR_POOL], HALO_NEW_CAP);
        if (start + HALO_NEW_CAP > m.dir.lists_cap) { E.start = -1; E.cnt_cap = 0u; atomicExch(&counters[C_DIR_ERROR], 1); continue; }
        E.start = start;
        E.cnt_cap = (unsigned)HALO_NEW_CAP << 16;
    }
}
__global__ void __launch_bounds__(256) k_halo_append(MapView m, const float4* __restrict__ pts, const int* __restrict__ slots, int n,
                                                      const int* __restrict__ n_dev, int* counters, unsigned* __restrict__ fix, int fix_cap) {
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    n = batch_count(n, n_dev);
    for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        const int slot = slots[i];
        if (slot < 0 || lane >= 27) continue;
        const unsigned e = dir_find(m.dir, halo_key(m.dir, pts[i], lane));
        if (e == 0xffffffffu) { atomicExch(&counters[C_DIR_ERROR], 1); continue; }
        CellEntry& E = m.dir.tab[e];
        if (E.start < 0) continue;                                   // already over-full
        const unsigned old = atomicAdd(&E.cnt_cap, 1u);
        const int pos = (int)(old & 0xffffu), room = (int)(old >> 16);
        if (pos < room) m.dir.lists[E.start + pos] = slot;
        else {                                                       // no room: queue the cell for k_halo_fix (a new, larger list)
            atomicSub(&E.cnt_cap, 1u);
            if (atomicExch(&E.start, -1) >= 0) {
                const int at = atomicAdd(&counters[C_NFIX], 1);
                if (at < fix_cap) fix[at] = e; else atomicAdd(&counters[C_DIR_CROWDED], 1);
            }
        }
    }
}

// Lists that ran out of room are made anew, larger, by one warp each: the live points of the cell's 3x3x3 block are found through
// the BVH (box query over the block, exact membership by cell coordinate), counted, then listed.  The old list is abandoned in the
// pool (the next global re-list packs it away).  A cell whose block holds more than HALO_MAX points stays with the BVH walk.
struct HaloGather {
    const MapView& m; int lane; int cx, cy, cz; int* out; int cnt = 0;
    __device__ HaloGather(const MapView& m_, int lane_, int cx_, int cy_, int cz_, int* out_) : m(m_), lane(lane_), cx(cx_), cy(cy_), cz(cz_), out(out_) {}
    __device__ __forceinline__ void leaf(int l) {
        const float inv = m.dir.inv_cell;
        while (l >= 0) {
            const int slot = l * LEAF + lane;
            const float4 p = m.pts[slot];
            const bool in = slot_valid(p) && abs(cell_coord(p.x, inv) - cx) <= 1 && abs(cell_coord(p.y, inv) - cy) <= 1 && abs(cell_coord(p.z, inv) - cz) <= 1;
            const unsigned mask = __ballot_sync(FULL, in);
            if (out && in) { const int at = cnt + __popc(mask & ((1u << lane) - 1)); out[at] = slot; }
            cnt += __popc(mask);
            l = m.next[l];
        }
    }
};
__global__ void __launch_bounds__(256) k_halo_fix(MapView m, const unsigned* __restrict__ fix, int fix_cap, int* counters) {
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    const int n = min(counters[C_NFIX], fix_cap);
    for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        CellEntry& E = m.dir.tab[fix[i]];
        const unsigned long long key = E.key;
        const int cx = (int)((key >> 42) & 0x1fffffu) - CELL_OFF, cy = (int)((key >> 21) & 0x1fffffu) - CELL_OFF, cz = (int)(key & 0x1fffffu) - CELL_OFF;
        const float c = m.dir.cell, pad = 1e-3f * c;
        const float bmin[3] = {(cx - 1) * c - pad, (cy - 1) * c - pad, (cz - 1) * c - pad};
        const float bmax[3] = {(cx + 2) * c + pad, (cy + 2) * c + pad, (cz + 2) * c + pad};
        HaloGather count(m, lane, cx, cy, cz, nullptr);
        box_query(m, bmin, bmax, count, lane);
        const int cnt = count.cnt;
        int start = -1, room = 0;
        if (cnt <= HALO_MAX) {
            room = (cnt + max(16, cnt / 2) + 3) & ~3;
            if (lane == 0) start = atomicAdd(&counters[C_DIR_POOL], room);
            start = __shfl_sync(FULL, start, 0);
            if (start + room > m.dir.lists_cap) { start = -1; if (lane == 0) atomicExch(&counters[C_DIR_ERROR], 1); }
        }
        if (start < 0) { if (lane == 0) atomicAdd(&counters[C_DIR_CROWDED], 1); continue; }      // stays with the BVH walk
        HaloGather fill(m, lane, cx, cy, cz, m.dir.lists + start);
        box_query(m, bmin, bmax, fill, lane);
        __syncwarp();
        if (lane == 0) { E.cnt_cap = ((unsigned)room << 16) | (unsigned)fill.cnt; __threadfence(); E.start = start; }
    }
}

// Batched Nearest_Search: one lane per query (cell directory), BVH walk by the warp for what that cannot prove.
// GATED (fl_map_nearest_search for k <= KNN_K, both forms): a query with a non-finite coordinate is searched at the origin
// (so fl_map_dir_stats counts it as a walk from there) and finds nothing; every other row keeps its leading entries with
// d2 <= md2.  Dropped entries are (0, 0, 0, 0) with d2 = +inf.
template <bool GATED, bool DET = false>
__device__ __forceinline__ void knn_batch(const MapView& m, const float4* __restrict__ q, int nq, int k, float md2,
                                          float4* __restrict__ out_pts, float* __restrict__ out_d2, int* __restrict__ out_cnt,
                                          WalkPool& pool) {
    if (threadIdx.x == 0) pool.n[0] = pool.n[1] = 0;
    __syncthreads();
    int phase = 0;
    const int stride = gridDim.x * blockDim.x;
    for (int base = blockIdx.x * blockDim.x; base < nq; base += stride) {          // block-uniform trip count (knn_block has barriers)
        const int i = base + threadIdx.x;
        const bool active = i < nq;
        float4 qq = make_float4(0.f, 0.f, 0.f, 0.f);
        if (active) qq = __ldg(&q[i]);
        bool finite = true;
        if constexpr (GATED) {
            finite = isfinite(qq.x) && isfinite(qq.y) && isfinite(qq.z);
            if (!finite) qq.x = qq.y = qq.z = 0.f;
        }
        TBestT<DET> kb;
        knn_block(m, active, qq.x, qq.y, qq.z, kb, pool, phase);
        if (active) {
            float4 p[KNN_K];
            const int cnt = knn_fetch(m, kb, p);
            int c = min(k, cnt);
            if constexpr (GATED) {
                int g = 0;
#pragma unroll
                for (int j = 0; j < KNN_K; j++) g += (finite && g == j && j < c && kb.d[j] <= md2) ? 1 : 0;
                c = g;
#pragma unroll
                for (int j = 0; j < KNN_K; j++) {
                    if (j >= c) { p[j] = make_float4(0.f, 0.f, 0.f, 0.f); kb.d[j] = INFINITY; }
                }
            }
#pragma unroll
            for (int j = 0; j < KNN_K; j++) {
                if (j < k) { out_pts[(size_t)i * k + j] = p[j]; out_d2[(size_t)i * k + j] = kb.d[j]; }
            }
            out_cnt[i] = c;
        }
        __syncthreads();
    }
}
__global__ void __launch_bounds__(128) k_knn_batch(MapView m, const float4* __restrict__ q, int nq, int k,
                                                    float4* __restrict__ out_pts, float* __restrict__ out_d2,
                                                    int* __restrict__ out_cnt) {
    __shared__ WalkPool pool;
    knn_batch<false>(m, q, nq, k, 0.f, out_pts, out_d2, out_cnt, pool);
}
__global__ void __launch_bounds__(128) k_knn_batch_gated(MapView m, const float4* __restrict__ q, int nq, int k, float md2,
                                                          float4* __restrict__ out_pts, float* __restrict__ out_d2,
                                                          int* __restrict__ out_cnt) {
    __shared__ WalkPool pool;
    knn_batch<true>(m, q, nq, k, md2, out_pts, out_d2, out_cnt, pool);
}

// the keyed tie rule (fl_map_set_deterministic, map.cuh "tie rules"): kernels of their own, so the default ones keep their code
__global__ void __launch_bounds__(128) k_knn_batch_det(MapView m, const float4* __restrict__ q, int nq, int k,
                                                        float4* __restrict__ out_pts, float* __restrict__ out_d2,
                                                        int* __restrict__ out_cnt) {
    __shared__ WalkPool pool;
    knn_batch<false, true>(m, q, nq, k, 0.f, out_pts, out_d2, out_cnt, pool);
}
__global__ void __launch_bounds__(128) k_knn_batch_gated_det(MapView m, const float4* __restrict__ q, int nq, int k, float md2,
                                                              float4* __restrict__ out_pts, float* __restrict__ out_d2,
                                                              int* __restrict__ out_cnt) {
    __shared__ WalkPool pool;
    knn_batch<true, true>(m, q, nq, k, md2, out_pts, out_d2, out_cnt, pool);
}

// Nearest_Search(point, k, .., max_dist) for 6 <= k <= 32: one warp per query, the k-best list one entry per lane (KBestK),
// seeded from the cell directory (knn_seed_k) and completed by the BVH walk where the seed is not proven.  A query with a
// non-finite coordinate, or a NaN md2, finds nothing.  Lane j writes entry j of the row.
template <bool DET>
__device__ __forceinline__ void knn_k(const MapView& m, const float4* __restrict__ q, int nq, int k, float md2,
                                      float4* __restrict__ out_pts, float* __restrict__ out_d2, int* __restrict__ out_cnt) {
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    const float gate = nextafterf(md2, INFINITY);
    int walked = 0;
    for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < nq; i += warps) {
        const float4 qq = __ldg(&q[i]);
        KBestKT<DET> kb;
        kb.init(k, gate);
        if (isfinite(qq.x) && isfinite(qq.y) && isfinite(qq.z) && !isnan(md2) && !knn_seed_k(m, qq.x, qq.y, qq.z, md2, kb, lane)) {
            walked++;
            knn_query_from(m, qq.x, qq.y, qq.z, kb, lane);
        }
        float4 p;
        const int cnt = knn_fetch_warp(m, kb, p, lane);
        if (lane < k) { out_pts[(size_t)i * k + lane] = p; out_d2[(size_t)i * k + lane] = kb.d; }
        if (lane == 0) out_cnt[i] = cnt;
    }
    if (lane == 0 && walked && m.dir.cap && m.dir.n_walked) atomicAdd(m.dir.n_walked, walked);
}
__global__ void __launch_bounds__(256) k_knn_k(MapView m, const float4* __restrict__ q, int nq, int k, float md2,
                                                float4* __restrict__ out_pts, float* __restrict__ out_d2, int* __restrict__ out_cnt) {
    knn_k<false>(m, q, nq, k, md2, out_pts, out_d2, out_cnt);
}
__global__ void __launch_bounds__(256) k_knn_k_det(MapView m, const float4* __restrict__ q, int nq, int k, float md2,
                                                    float4* __restrict__ out_pts, float* __restrict__ out_d2, int* __restrict__ out_cnt) {
    knn_k<true>(m, q, nq, k, md2, out_pts, out_d2, out_cnt);
}

// Delete_Point_Boxes: every slot tests itself against the boxes (half-open, ikd_Tree.cpp:796).
// A flat pass over the leaf array is bandwidth-trivial on HBM3e (16 B per slot) and needs
// no tree descent, no lazy flags and no push-down.  nb_dev / used_dev (may be null): the box count and the used-leaf count read
// from device memory (the device form: the host's mirror of the used leaves misses those device-form inserts claimed since the
// map last settled); the grid is then sized without them.
__global__ void k_delete_boxes(MapView m, const float* __restrict__ boxes, int nb, int n_leaf_used, int* counters,
                               float4* __restrict__ removed, int removed_cap, const int* __restrict__ nb_dev,
                               const int* __restrict__ used_dev) {
    if (nb_dev) nb = *nb_dev;
    if (used_dev) n_leaf_used = *used_dev;
    if (nb <= 0) return;
    const long long total = (long long)n_leaf_used * LEAF;
    const int lane = threadIdx.x & 31;
    int local = 0;
    for (long long base = (blockIdx.x * (long long)blockDim.x + threadIdx.x) - lane; base < total; base += (long long)gridDim.x * blockDim.x) {
        const long long slot = base + lane;
        float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
        bool hit = false;
        if (slot < total) {
            p = m.pts[slot];
            if (slot_valid(p)) for (int b = 0; b < nb && !hit; b++) hit = in_box(p, &boxes[b * 6], &boxes[b * 6 + 3]);
            if (hit) { m.pts[slot].w = __int_as_float(SLOT_TOMB); local++; }
        }
        if (removed) {                                     // history for acquire_removed_points (ikd_Tree.cpp:661-676)
            const unsigned mask = __ballot_sync(FULL, hit);
            int off = 0;
            if (lane == 0 && mask) off = atomicAdd(&counters[C_REMOVED], __popc(mask));
            off = __shfl_sync(FULL, off, 0);
            const int at = off + __popc(mask & ((1u << lane) - 1));
            if (hit && at < removed_cap) { p.w = m.payload[slot]; removed[at] = p; }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(FULL, local, o);
    if (lane == 0 && local) atomicAdd(&counters[C_DELETED], local);
}
// Delete_Point_Boxes on the caller's stream.  The plan, before any slot is touched: the box count, and room in the removed-points
// record for every valid point on top of what it holds (the host form grows the record to that before each delete).  Without
// room nothing is deleted; the next full settle (fl_map_maintain) grows the record, as it does whenever the record is started.
// A delete refusal leaves C_REFUSED alone: that flag makes the settle grow the map and its directory for the Add_Points forms.
__global__ void k_delete_plan(int* counters, const int* __restrict__ nb_dev, int nb_max, bool record, int removed_cap) {
    const int nb = min(max(*nb_dev, 0), nb_max);
    const bool ok = nb == 0 || !record || (long long)counters[C_REMOVED] + counters[C_VALID] <= removed_cap;
    counters[C_DEL_NB] = ok ? nb : 0;
    counters[C_DEL_SKIP] = !ok;
    counters[C_DELETED] = 0;
}
// after the delete: the host form's bookkeeping (delete_boxes) and its maybe_rebuild, which here only marks maintenance as due
__global__ void k_delete_account(MapView m, int* counters, int chain_limit) {
    const int d = counters[C_DELETED];
    if (d == 0) return;
    counters[C_VALID] -= d;
    counters[C_TOMBS] += d;
    const int tombs = counters[C_TOMBS];
    if ((tombs > 1024 && tombs > counters[C_VALID]) || counters[C_LEAF_USED] - m.n_main > chain_limit) counters[C_DUE] = 1;
}
// status2 = (status, deleted)
__global__ void k_delete_status(const int* __restrict__ counters, int* __restrict__ out) {
    out[0] = counters[C_DEL_SKIP] ? FL_ERR_CAPACITY : (counters[C_DUE] ? 1 : FL_OK);
    out[1] = counters[C_DELETED];
}
// Add_Point_Boxes (ikd_Tree.cpp:576-603 -> Add_by_range :854-934): points deleted by Delete_Point_Boxes that lie in the boxes
// and have not been overwritten since come back (points removed by down-sampling do not, as in the reference)
__global__ void k_revive_boxes(MapView m, const float* __restrict__ boxes, int nb, int n_leaf_used, int* counters) {
    const long long total = (long long)n_leaf_used * LEAF;
    int local = 0;
    for (long long slot = blockIdx.x * (long long)blockDim.x + threadIdx.x; slot < total; slot += (long long)gridDim.x * blockDim.x) {
        const float4 p = m.pts[slot];
        if (__float_as_int(p.w) != SLOT_TOMB) continue;
        bool hit = false;
        for (int b = 0; b < nb && !hit; b++) hit = in_box(p, &boxes[b * 6], &boxes[b * 6 + 3]);
        if (hit) { m.pts[slot].w = __int_as_float(SLOT_VALID); local++; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(FULL, local, o);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(&counters[C_REVIVED], local);
}

// Compaction of every valid point (x, y, z, intensity) -- flatten() and the input of rebuild().
__global__ void k_compact(MapView m, int n_leaf_used, float4* __restrict__ out, int* counters) {
    const long long total = (long long)n_leaf_used * LEAF;
    const int lane = threadIdx.x & 31;
    for (long long base = (blockIdx.x * (long long)blockDim.x + threadIdx.x) - lane; base < total;
         base += (long long)gridDim.x * blockDim.x) {
        const long long slot = base + lane;
        float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
        bool v = false;
        if (slot < total) { p = m.pts[slot]; v = slot_valid(p); }
        const unsigned mask = __ballot_sync(FULL, v);
        int off = 0;
        if (lane == 0 && mask) off = atomicAdd(&counters[C_COMPACT], __popc(mask));
        off = __shfl_sync(FULL, off, 0);
        if (v) {
            p.w = m.payload[slot];
            out[off + __popc(mask & ((1u << lane) - 1))] = p;
        }
    }
}

// fl_map_flatten in the deterministic mode: the compacted rows sorted by (x, y, z, intensity) as order-preserving integers of their
// bits (ord_bits), by two stable 64-bit radix sorts, least significant half first: (z, intensity), then (x, y).
__global__ void k_flatten_keys(const float4* __restrict__ rows, const unsigned* __restrict__ perm, int n, bool xy,
                               unsigned long long* __restrict__ keys, unsigned* __restrict__ vals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned r = perm ? perm[i] : (unsigned)i;
    const float4 p = rows[r];
    keys[i] = xy ? ((unsigned long long)ord_bits(p.x) << 32) | ord_bits(p.y) : ((unsigned long long)ord_bits(p.z) << 32) | ord_bits(p.w);
    vals[i] = r;
}
__global__ void k_gather_rows(const float4* __restrict__ rows, const unsigned* __restrict__ perm, int n, float4* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = rows[perm[i]];
}

// ----------------------------------------------------------------------------- Add_Points
// Voxel of a point exactly as Add_Points computes it (ikd_Tree.cpp:491-499): float division,
// float floor, float multiply.
struct VoxelBox { float bmin[3], bmax[3], mid[3]; };
__device__ __forceinline__ void voxel_box(const float4& p, float ds, VoxelBox& vb) {
    const float c[3] = {p.x, p.y, p.z};
#pragma unroll
    for (int a = 0; a < 3; a++) {
        vb.bmin[a] = __fmul_rn(floorf(__fdiv_rn(c[a], ds)), ds);
        vb.bmax[a] = __fadd_rn(vb.bmin[a], ds);
        // mid = min + (max - min) / 2.0  evaluated in double, stored to float (ikd_Tree.cpp:497-499)
        vb.mid[a] = (float)((double)vb.bmin[a] + (double)__fsub_rn(vb.bmax[a], vb.bmin[a]) / 2.0);
    }
}
__device__ __forceinline__ unsigned long long voxel_key(const float4& p, float ds) {
    unsigned long long key = 0;
    const float c[3] = {p.x, p.y, p.z};
#pragma unroll
    for (int a = 0; a < 3; a++) {
        float f = floorf(__fdiv_rn(c[a], ds)) + 1048576.0f;
        f = f < 0.f ? 0.f : (f > 2097151.f ? 2097151.f : f);
        key = (key << 21) | (unsigned long long)(unsigned)f;
    }
    return key;
}
// Real keys use bits 0-62 (and reach 2^63 - 1 where the coordinates clamp).  Device forms sort all n_max rows: rows past the
// batch get PAD_KEY, which sorts after every real key, so the first n sorted rows are those of the host form's sort of n rows.
constexpr unsigned long long PAD_KEY = 1ull << 63;
__global__ void k_voxel_keys(const float4* __restrict__ pts, int n, float ds, unsigned long long* __restrict__ keys,
                             unsigned* __restrict__ vals, const int* __restrict__ n_dev) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { keys[i] = i < batch_count(n, n_dev) ? voxel_key(pts[i], ds) : PAD_KEY; vals[i] = (unsigned)i; }
}
__global__ void k_group_heads(const unsigned long long* __restrict__ keys, int n, int* __restrict__ group_start, int* counters,
                              const int* __restrict__ n_dev) {
    int r = blockIdx.x * blockDim.x + threadIdx.x;
    n = batch_count(n, n_dev);
    if (r < n && (r == 0 || keys[r] != keys[r - 1])) group_start[atomicAdd(&counters[C_GROUPS], 1)] = r;
}

// pass 1: count the valid points inside the voxel and find the one closest to its centre.  DET (fl_map_set_deterministic): of
// points at bit-equal distances the one with the smallest (x, y, z, intensity) counts as the closest (map.cuh, "tie rules")
template <bool DET = false>
struct BoxScan {
    const MapView& m; const VoxelBox& vb; int lane;
    int count = 0; float best_d = INFINITY; int best_slot = -1;
    __device__ BoxScan(const MapView& m_, const VoxelBox& vb_, int lane_) : m(m_), vb(vb_), lane(lane_) {}
    __device__ __forceinline__ void leaf(int l) {
        while (l >= 0) {
            const int slot = l * LEAF + lane;
            const float4 p = m.pts[slot];
            const bool in = slot_valid(p) && in_box(p, vb.bmin, vb.bmax);
            const unsigned mask = __ballot_sync(FULL, in);
            if (mask) {
                count += __popc(mask);
                const float d = in ? sq_dist3(p.x, p.y, p.z, vb.mid[0], vb.mid[1], vb.mid[2]) : INFINITY;
                const unsigned key = in ? __float_as_uint(d) : 0xffffffffu;
                const unsigned best = __reduce_min_sync(FULL, key);
                if constexpr (!DET) {
                    if (__uint_as_float(best) < best_d) {       // strict: the first one found wins ties (ikd_Tree.cpp:508)
                        best_d = __uint_as_float(best);
                        best_slot = l * LEAF + (__ffs(__ballot_sync(FULL, key == best)) - 1);
                    }
                } else if (__uint_as_float(best) <= best_d) {
                    const int cand = l * LEAF + warp_key_min<false>(m, __ballot_sync(FULL, key == best), p, slot, lane);
                    if (__uint_as_float(best) < best_d || key_less<false>(m, cand, best_slot)) { best_d = __uint_as_float(best); best_slot = cand; }
                }
            }
            l = m.next[l];
        }
    }
};
struct BoxKill {       // pass 2: invalidate every valid point inside the voxel except `keep`
    const MapView& m; const VoxelBox& vb; int lane; int keep;
    __device__ BoxKill(const MapView& m_, const VoxelBox& vb_, int lane_, int keep_) : m(m_), vb(vb_), lane(lane_), keep(keep_) {}
    __device__ __forceinline__ void leaf(int l) {
        while (l >= 0) {
            const int slot = l * LEAF + lane;
            const float4 p = m.pts[slot];
            if (slot_valid(p) && in_box(p, vb.bmin, vb.bmax) && slot != keep) m.pts[slot].w = __int_as_float(SLOT_TOMB_DS);
            l = m.next[l];
        }
    }
};

__device__ __forceinline__ bool same_point(const float4& a, const float4& b) {   // ikd_Tree.cpp:1676-1680, EPSS = 1e-6
    return fabs((double)a.x - (double)b.x) < 1e-6 && fabs((double)a.y - (double)b.y) < 1e-6 && fabs((double)a.z - (double)b.z) < 1e-6;
}

// One warp per touched voxel (device forms: rows past the batch carry PAD_KEY, which no group's key equals, so a group never
// runs into them and n may be n_max).  Reproduces the sequential per-point semantics of
// Add_Points(downsample_on = true) (ikd_Tree.cpp:489-521) for all batch points that fall
// into the voxel, in their original order (the sort is stable).
template <bool DET>
__device__ __forceinline__ void downsample_resolve(const MapView& m, const float4* __restrict__ batch,
                                                   const unsigned long long* __restrict__ keys,
                                                   const unsigned* __restrict__ vals, int n,
                                                   const int* __restrict__ group_start, float ds,
                                                   float4* __restrict__ insert_list, int* counters) {
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    const int n_groups = counters[C_GROUPS];
    for (int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; g < n_groups; g += warps) {
        const int r0 = group_start[g];
        const unsigned long long key = keys[r0];
        const float4 first = batch[vals[r0]];
        VoxelBox vb;
        voxel_box(first, ds, vb);
        BoxScan<DET> scan(m, vb, lane);
        box_query(m, vb.bmin, vb.bmax, scan, lane);
        // ---- sequential resolution (warp-uniform scalar work)
        int cur_count = scan.count;
        float cur_d = scan.best_d;
        int cur_slot = scan.best_slot;        // >= 0: existing map point; -1: none / a batch point
        int cur_batch = -1;                   // index into batch[] if the current best is a new point
        float4 cur_pt = make_float4(0.f, 0.f, 0.f, 0.f);
        if (cur_slot >= 0) cur_pt = m.pts[cur_slot];
        bool modified = false;
        int added = 0;
        for (int r = r0; r < n && keys[r] == key; r++) {
            const int bi = (int)vals[r];
            const float4 p = batch[bi];
            const float d_new = sq_dist3(p.x, p.y, p.z, vb.mid[0], vb.mid[1], vb.mid[2]);
            const bool cur_wins = cur_count > 0 && cur_d < d_new;       // tmp_dist < min_dist
            const bool same = !cur_wins || same_point(p, cur_pt);
            if (cur_count > 1 || same) {
                modified = true;
                added++;
                if (!cur_wins) { cur_d = d_new; cur_slot = -1; cur_batch = bi; cur_pt = p; }
                cur_count = 1;
            }
        }
        if (modified) {
            const int keep = cur_slot;            // existing survivor stays in place (== delete + re-add of the same point)
            BoxKill kill(m, vb, lane, keep);
            box_query(m, vb.bmin, vb.bmax, kill, lane);
            if (lane == 0) {
                const int killed = scan.count - (keep >= 0 ? 1 : 0);
                if (killed) atomicAdd(&counters[C_TOMB], killed);
                if (keep < 0) insert_list[atomicAdd(&counters[C_NINSERT], 1)] = batch[cur_batch];
                atomicAdd(&counters[C_ADDED], added);
            }
        }
    }
}
__global__ void __launch_bounds__(256) k_downsample_resolve(MapView m, const float4* __restrict__ batch,
                                                             const unsigned long long* __restrict__ keys,
                                                             const unsigned* __restrict__ vals, int n,
                                                             const int* __restrict__ group_start, float ds,
                                                             float4* __restrict__ insert_list, int* counters) {
    downsample_resolve<false>(m, batch, keys, vals, n, group_start, ds, insert_list, counters);
}
__global__ void __launch_bounds__(256) k_downsample_keyed(MapView m, const float4* __restrict__ batch,
                                                                 const unsigned long long* __restrict__ keys,
                                                                 const unsigned* __restrict__ vals, int n,
                                                                 const int* __restrict__ group_start, float ds,
                                                                 float4* __restrict__ insert_list, int* counters) {
    downsample_resolve<true>(m, batch, keys, vals, n, group_start, ds, insert_list, counters);
}

// One warp per new point: descend towards the nearest child box to the home leaf, claim a free slot there or
// in its overflow chain (allocating a chain leaf from the pool if needed), publish the point
// and grow the AABBs on the root path with float atomics ("partial refit").
__global__ void __launch_bounds__(256) k_insert(MapView m, const float4* __restrict__ pts, int n, const int* __restrict__ n_dev, int* counters,
                                                 int* __restrict__ slot_out) {
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    n = batch_count(n, n_dev);
    for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        const float4 p = pts[i];
        int node = 0;
        for (int k = m.n_levels - 1; k >= 0; k--) {
            const bool root = (k == m.n_levels - 1);
            unsigned key = 0xffffffffu;
#pragma unroll
            for (int half = 0; half < 2; half++) {
                if (half == 1 && !root) break;
                const int c = lane + 32 * half;
                const int e = root ? c : node * FAN + c;
                if (e < m.count[k]) {
                    const float4 lo = m.ebox[k][2 * e], hi = m.ebox[k][2 * e + 1];
                    // empty entities have inverted boxes (distance +inf): they are the last resort
                    const float d = box_dist3(p.x, p.y, p.z, lo.x, lo.y, lo.z, hi.x, hi.y, hi.z);
                    key = min(key, (min(__float_as_uint(d), 0x7f800000u) & ~63u) | (unsigned)c);
                }
            }
            const unsigned best = __reduce_min_sync(FULL, key);
            node = (root ? 0 : node * FAN) + (int)(best & 63u);
        }
        const int home = node;
        int leaf = home;
        bool placed = false;
        while (!placed) {
            const float4 cur = m.pts[leaf * LEAF + lane];
            const int w = __float_as_int(cur.w);
            unsigned freem = __ballot_sync(FULL, w == SLOT_FREE || w == SLOT_TOMB || w == SLOT_TOMB_DS);      // never used, or a deleted point's
            while (freem && !placed) {
                const int s = __ffs(freem) - 1;
                const int seen = __shfl_sync(FULL, w, s);
                int old = 0;
                if (lane == 0) old = atomicCAS((int*)&m.pts[leaf * LEAF + s].w, seen, SLOT_BUSY);
                old = __shfl_sync(FULL, old, 0);
                if (old == seen) {
                    if (lane == 0) {
                        m.payload[leaf * LEAF + s] = p.w;
                        m.pts[leaf * LEAF + s] = make_float4(p.x, p.y, p.z, __int_as_float(SLOT_VALID));
                        slot_out[i] = leaf * LEAF + s;
                    }
                    placed = true;
                } else {
                    freem &= ~(1u << s);
                }
            }
            if (placed) break;
            int nxt = 0;
            if (lane == 0) {
                nxt = atomicAdd(&m.next[leaf], 0);
                if (nxt < 0) {
                    int fresh = atomicAdd(&counters[C_LEAF_USED], 1);
                    if (fresh >= m.leaf_cap) { atomicExch(&counters[C_ERROR], 1); nxt = -2; }
                    else {
                        int old = atomicCAS(&m.next[leaf], -1, fresh);
                        nxt = (old == -1) ? fresh : old;       // lost the race: follow the winner (the fresh leaf stays unused)
                    }
                }
            }
            nxt = __shfl_sync(FULL, nxt, 0);
            if (nxt < 0) break;                                    // pool exhausted (host guarantees this cannot happen)
            leaf = nxt;
        }
        if (!placed) { if (lane == 0) slot_out[i] = -1; continue; }
        // grow the boxes of the home leaf and of its ancestors
        int e = home;
        const float c3[3] = {p.x, p.y, p.z};
        for (int k = 0; k < m.n_levels; k++) {
            if (lane < 3) atomic_min_float(&((float*)&m.ebox[k][2 * e])[lane], c3[lane]);
            else if (lane < 6) atomic_max_float(&((float*)&m.ebox[k][2 * e + 1])[lane - 3], c3[lane - 3]);
            e /= FAN;
        }
    }
}

// ----------------------------------------------------------------------------- Add_Points on the caller's stream
// The device forms cannot re-pack or re-list after the fact (the pinned searches would answer from incomplete halo lists in
// between), so a plan decides before anything is written whether the whole call fits the room left, and every kernel of the call
// then runs over the count the plan let through: 0 when it refused.
constexpr int HALO_FIX_MAX = (HALO_MAX + HALO_MAX / 2 + 3) & ~3;      // the largest list k_halo_fix makes

__global__ void k_plan_begin(int* counters, const int* __restrict__ na, const int* __restrict__ nb, int n_max) {
    counters[C_RA] = min(max(*na, 0), n_max);
    counters[C_RB] = nb ? min(max(*nb, 0), n_max) : 0;
    counters[C_MISS] = 0;
    counters[C_FIXES] = 0;
}
// The list-pool need of a batch, counted over every (point, halo cell) pair of the batch (a superset of what the inserts append).
// k_plan_count: a pair whose cell has no entry yet may claim a fresh list (HALO_NEW_CAP); the pairs of a listed cell are counted
// in cellcnt (one int per table entry, all zero between calls).  k_plan_reset, after the counts of both lists: the first pair of
// a cell to take its count back to zero judges the cell.  Its list overflows when the count exceeds the free places; k_halo_fix
// then makes one new list (per insert) for the live points of the block, which are all listed already or in this batch, so at
// most L = listed + count of them.  C_FIXES: the need of those lists, in units of 16 ints.
__global__ void __launch_bounds__(256) k_plan_count(MapView m, const float4* __restrict__ pts, int n, const int* __restrict__ n_dev,
                                                     int* counters, int* __restrict__ cellcnt) {
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    n = batch_count(n, n_dev);
    for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        bool miss = false;
        if (lane < 27) {
            const unsigned e = dir_find(m.dir, halo_key(m.dir, pts[i], lane));
            if (e == 0xffffffffu) miss = true;
            else if (m.dir.tab[e].start >= 0) atomicAdd(&cellcnt[e], 1);
        }
        const unsigned mm = __ballot_sync(FULL, miss);
        if (lane == 0 && mm) atomicAdd(&counters[C_MISS], __popc(mm));
    }
}
__global__ void __launch_bounds__(256) k_plan_reset(MapView m, const float4* __restrict__ pts, int n, const int* __restrict__ n_dev,
                                                     int* counters, int* __restrict__ cellcnt, int inserts) {
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    n = batch_count(n, n_dev);
    for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        if (lane >= 27) continue;
        const unsigned e = dir_find(m.dir, halo_key(m.dir, pts[i], lane));
        if (e == 0xffffffffu) continue;
        const int t = atomicExch(&cellcnt[e], 0);
        const CellEntry E = m.dir.tab[e];
        if (t == 0 || E.start < 0) continue;
        const int listed = (int)(E.cnt_cap & 0xffffu), free_ = (int)(E.cnt_cap >> 16) - listed;
        if (t <= free_) continue;
        const int L = listed + t;
        const int room = min(HALO_FIX_MAX, (L + max(16, L / 2) + 3) & ~3);
        const int fixes = 1 + (inserts > 1 && t > free_ + 16);            // a second insert overflows the new list's >= 16 free places
        atomicAdd(&counters[C_FIXES], fixes * ((room + 15) / 16));
    }
}
// The host form's guards before an insert, for the whole call at once, in terms of the batch size (nothing is tombstoned yet):
// overflow leaves for one fresh leaf per point, the table below 90 % load, the list pool for the counted need.  The fix list is
// sized for 27 entries per point and cannot overflow.
__global__ void k_plan(MapView m, int* counters) {
    const long long n = (long long)counters[C_RA] + counters[C_RB];
    bool ok = counters[C_LEAF_USED] + n <= m.leaf_cap;
    if (m.dir.cap) {
        ok = ok && ((long long)counters[C_DIR_CELLS] + 27 * n) * 10 <= (long long)m.dir.cap * 9;
        const long long miss = counters[C_MISS];
        // fresh cells: a fresh list of HALO_NEW_CAP each, and a new list for each (per insert) that more than HALO_NEW_CAP pairs hit
        const long long need = miss * HALO_NEW_CAP + 16ll * counters[C_FIXES] + 2 * (miss / (HALO_NEW_CAP + 1)) * HALO_FIX_MAX;
        ok = ok && counters[C_DIR_POOL] + need <= m.dir.lists_cap;
        counters[C_NEED] = (int)min(need, (long long)INT_MAX);
    }
    counters[C_SKIP] = !ok;
    if (!ok) counters[C_REFUSED] = 1;
    counters[C_NA] = ok ? counters[C_RA] : 0;
    counters[C_NB] = ok ? counters[C_RB] : 0;
    counters[C_ADDED] = counters[C_GROUPS] = counters[C_NINSERT] = counters[C_TOMB] = 0;
}
// After one Add_Points of the call: the host form's bookkeeping of n_valid_ / n_tomb_ (add_points_host) and its decisions after
// the insert (insert_device's re-list of a full or crowded directory, maybe_rebuild), which here only mark maintenance as due.
__global__ void k_async_account(MapView m, int* counters, int slot, bool downsample_on, int chain_limit) {
    const int batch = counters[slot];
    if (batch == 0) return;
    int inserted = batch;
    if (downsample_on) {
        const int tomb = counters[C_TOMB];
        inserted = counters[C_NINSERT];
        counters[C_VALID] -= tomb;
        counters[C_TOMBS] += tomb;
    }
    counters[C_VALID] += inserted;
    bool due = false;
    if (inserted > 0 && m.dir.cap) due = counters[C_DIR_ERROR] || counters[C_DIR_CROWDED] > max(64, counters[C_DIR_CELLS] / 1024);
    if (downsample_on) counters[C_TOMBS] = max(0, counters[C_TOMBS] - inserted);
    const int tombs = counters[C_TOMBS];
    due = due || counters[C_LEAF_USED] - m.n_main > chain_limit || (tombs > 1024 && tombs > counters[C_VALID]) || counters[C_ERROR];
    if (due) counters[C_DUE] = 1;
}
// status2 = (status, added), or out4 = (list_counts[0], list_counts[1], added, status)
__global__ void k_async_status(const int* __restrict__ counters, const int* __restrict__ list_counts, int* __restrict__ out) {
    const bool skip = counters[C_SKIP] != 0;
    const int st = skip ? FL_ERR_CAPACITY : (counters[C_DUE] ? 1 : FL_OK);
    const int added = skip ? 0 : counters[C_ADDED];
    if (list_counts) { out[0] = list_counts[0]; out[1] = list_counts[1]; out[2] = added; out[3] = st; }
    else { out[0] = st; out[1] = added; }
}
__global__ void k_set_counts(int* counters, int valid, int tomb, int due) {
    counters[C_VALID] = valid;
    counters[C_TOMBS] = tomb;
    counters[C_DUE] = due;
}

// ----------------------------------------------------------------------------- Box_Search / Radius_Search
// A query is a box (min xyz, max xyz) or a sphere (x, y, z, r).  One warp per query would stall on a single whole-map box, so
// the work is spread over (query, main leaf) pairs: k_range_leaves lists, per query, the main leaves whose AABB can hold an
// answer, then one warp per pair decides membership slot by slot with the exact rule (k_range_count_dev, k_range_fill_dev).
// The pruning may widen the searched set, never narrow it.  The host-buffer and device-buffer forms run the same kernels
// (Map::range_count, Map::range_emit).
struct RangeQuery {
    float bmin[3], bmax[3];      // pruning box: the query box itself, or the sphere's AABB padded outward
    float c[3], r2, r2_pad;      // sphere: centre, fl(r * r) (the rule of Search_by_radius, ikd_Tree.cpp:1308) and a padded bound
    bool valid;                  // false: NaN input, negative radius or an empty box -- no answer
};
template <bool RADIUS>
__device__ __forceinline__ RangeQuery range_query(const float* __restrict__ q, int i) {
    RangeQuery Q;
    if constexpr (RADIUS) {
        const float4 s = __ldg(reinterpret_cast<const float4*>(q) + i);
        Q.c[0] = s.x; Q.c[1] = s.y; Q.c[2] = s.z;
        Q.valid = !isnan(s.x) && !isnan(s.y) && !isnan(s.z) && s.w >= 0.f;       // NaN radius fails the comparison
        Q.r2 = __fmul_rn(s.w, s.w);
        Q.r2_pad = __fmul_rn(Q.r2, 1.0001f);
        // every point with sq_dist3 <= r2 lies within r (1 + a few ulps) of the centre on each axis; the pad is far wider
        const float pad = __fadd_rn(__fadd_rn(__fmul_rn(s.w, 1.0001f), 1e-6f * fmaxf(fmaxf(fabsf(s.x), fabsf(s.y)), fabsf(s.z))), 1e-30f);
#pragma unroll
        for (int a = 0; a < 3; a++) { Q.bmin[a] = __fsub_rn(Q.c[a], pad); Q.bmax[a] = __fadd_rn(Q.c[a], pad); }
    } else {
        bool ok = true;
#pragma unroll
        for (int a = 0; a < 3; a++) {
            Q.bmin[a] = __ldg(&q[6 * (size_t)i + a]);
            Q.bmax[a] = __ldg(&q[6 * (size_t)i + 3 + a]);
            ok &= Q.bmin[a] < Q.bmax[a];                     // false for NaN and for an inverted or empty box
        }
        Q.valid = ok;
        Q.c[0] = Q.c[1] = Q.c[2] = Q.r2 = Q.r2_pad = 0.f;
    }
    return Q;
}
// the per-point rule: Search_by_range's half-open box (ikd_Tree.cpp:1263), or Search_by_radius's calc_dist(p, q) <= r * r (:1308)
template <bool RADIUS>
__device__ __forceinline__ bool range_hit(const float4& p, const RangeQuery& Q) {
    if (!slot_valid(p)) return false;
    if constexpr (RADIUS) return sq_dist3(Q.c[0], Q.c[1], Q.c[2], p.x, p.y, p.z) <= Q.r2;
    else return in_box(p, Q.bmin, Q.bmax);
}

template <bool RADIUS>
struct RangeLeaves {             // box_query functor: counts (out == nullptr) or lists the candidate leaves of query q
    const MapView& m; const RangeQuery& Q; int2* out; int q; int lane; int n = 0;
    __device__ RangeLeaves(const MapView& m_, const RangeQuery& Q_, int2* out_, int q_, int lane_) : m(m_), Q(Q_), out(out_), q(q_), lane(lane_) {}
    __device__ __forceinline__ void leaf(int l) {
        if constexpr (RADIUS) {
            // box_dist3 <= sq_dist3 of every point in the box (both are monotone in the exact distances), so this drop is exact
            const float4 lo = __ldg(&m.ebox[0][2 * l]), hi = __ldg(&m.ebox[0][2 * l + 1]);
            if (box_dist3(Q.c[0], Q.c[1], Q.c[2], lo.x, lo.y, lo.z, hi.x, hi.y, hi.z) > Q.r2_pad) return;
        }
        if (out && lane == 0) out[n] = make_int2(q, l);
        n++;
    }
};
// One warp per query.  Count pass (pairs == nullptr): cnt[i] = candidate leaves.  Fill pass: the (query, leaf) pairs at
// off[i], in ascending leaf order (box_query visits children in lane order).
template <bool RADIUS>
__device__ __forceinline__ void range_leaves(const MapView& m, const float* __restrict__ q, int nq, long long* __restrict__ cnt,
                                             const long long* __restrict__ off, int2* __restrict__ pairs) {
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < nq; i += warps) {
        const RangeQuery Q = range_query<RADIUS>(q, i);
        if (!Q.valid) { if (lane == 0 && !pairs) cnt[i] = 0; continue; }
        RangeLeaves<RADIUS> f(m, Q, pairs ? pairs + off[i] : nullptr, i, lane);
        box_query(m, Q.bmin, Q.bmax, f, lane);
        if (lane == 0 && !pairs) cnt[i] = f.n;
    }
}
template <bool RADIUS>
__global__ void __launch_bounds__(256) k_range_leaves(MapView m, const float* __restrict__ q, int nq, long long* __restrict__ cnt,
                                                      const long long* __restrict__ off, int2* __restrict__ pairs) {
    range_leaves<RADIUS>(m, q, nq, cnt, off, pairs);
}
// the fill pass of the device-buffer form: the pairs are listed only when all off[nq] of them fit the caller's workspace
template <bool RADIUS>
__global__ void __launch_bounds__(256) k_range_leaves_bounded(MapView m, const float* __restrict__ q, int nq, const long long* __restrict__ off,
                                                              int2* __restrict__ pairs, long long max_pairs) {
    if (off[nq] > max_pairs) return;
    range_leaves<RADIUS>(m, q, nq, nullptr, off, pairs);
}
// One warp per (query, leaf) pair: the leaf and its overflow chain, one slot per lane.  Count pass (out == nullptr): cnt[w] =
// points found.  Fill pass: (x, y, z, intensity) of each at off[w] + the prefix popcount, the first `cap` of all only.
template <bool RADIUS>
__device__ __forceinline__ void range_points(const MapView& m, const float* __restrict__ q, const int2* __restrict__ pairs, long long npairs,
                                             long long* __restrict__ cnt, const long long* __restrict__ off, float4* __restrict__ out, long long cap) {
    const int lane = threadIdx.x & 31;
    const long long warps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < npairs; w += warps) {
        const long long base = out ? off[w] : 0;
        if (out && base >= cap) continue;
        const int2 pr = pairs[w];
        const RangeQuery Q = range_query<RADIUS>(q, pr.x);
        int leaf = pr.y, n = 0;
        while (leaf >= 0) {
            const float4 p = __ldg(&m.pts[leaf * LEAF + lane]);
            const int nxt = __ldg(&m.next[leaf]);
            const bool hit = range_hit<RADIUS>(p, Q);
            const unsigned mask = __ballot_sync(FULL, hit);
            if (out && hit) {
                const long long at = base + n + __popc(mask & ((1u << lane) - 1));
                if (at < cap) out[at] = make_float4(p.x, p.y, p.z, __ldg(&m.payload[leaf * LEAF + lane]));
            }
            n += __popc(mask);
            leaf = nxt;
        }
        if (!out && lane == 0) cnt[w] = n;
    }
}

// No kernel reads a count back to the host: the number of pairs and of points stay in device memory (the control words
// below), and every kernel runs a grid sized from host-known bounds and loops up to them.
enum RangeCtl { RS_PAIRS = 0,       // pairs listed: off[nq] when it fits the workspace, else 0
                RS_FILL,            // pairs whose points are written: RS_PAIRS, or 0 when nothing may be written
                RS_OK,              // 1: the offsets are written in full
                RS_CTL_COUNT };
__global__ void k_range_plan(const long long* __restrict__ leaf_off, int nq, long long max_pairs, long long* __restrict__ ctl) {
    const long long np = leaf_off[nq];
    ctl[RS_PAIRS] = np <= max_pairs ? np : 0;
}
template <bool RADIUS>
__global__ void __launch_bounds__(256) k_range_count_dev(MapView m, const float* __restrict__ q, const int2* __restrict__ pairs,
                                                         const long long* __restrict__ npairs, long long* __restrict__ cnt) {
    range_points<RADIUS>(m, q, pairs, *npairs, cnt, nullptr, nullptr, 0);
}
template <bool RADIUS>
__global__ void __launch_bounds__(256) k_range_fill_dev(MapView m, const float* __restrict__ q, const int2* __restrict__ pairs,
                                                        const long long* __restrict__ npairs, const long long* __restrict__ off,
                                                        float4* __restrict__ out, long long cap) {
    range_points<RADIUS>(m, q, pairs, *npairs, nullptr, off, out, cap);
}
// status2 = (points found, pairs needed), or (-1, pairs needed) when the pairs did not fit; decides what may be written
__global__ void k_range_status(const long long* __restrict__ leaf_off, const long long* __restrict__ point_off, int nq, long long max_pairs,
                               long long* __restrict__ ctl, long long* __restrict__ status2) {
    const long long np = leaf_off[nq];
    long long total = -1;
    bool ok = false;
    if (np <= max_pairs) {
        total = point_off[ctl[RS_PAIRS]];
        ok = total <= INT_MAX;                 // above: the counterpart of FL_ERR_CAPACITY, the total alone is reported
    }
    ctl[RS_FILL] = ok ? ctl[RS_PAIRS] : 0;
    ctl[RS_OK] = ok;
    status2[0] = total;
    status2[1] = np;
}
__global__ void k_range_offsets_dev(const long long* __restrict__ leaf_off, const long long* __restrict__ point_off, int nq,
                                    const long long* __restrict__ ctl, int* __restrict__ offsets) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= nq) offsets[i] = ctl[RS_OK] ? (int)point_off[leaf_off[i]] : 0;
}

// Exclusive prefix sum whose length lives in device memory: out[0 .. n] with out[n] the total, n = *len.  CUB's scans take a host
// count, and scanning the whole capacity would make every call pay for the workspace rather than for the answer.  A fixed grid
// of gridDim.x blocks splits [0, n) into contiguous chunks: (1) each block sums its chunk, (2) one block scans the partial sums,
// (3) each block scans its chunk from its partial.  Integer sums: the result equals CUB's ExclusiveSum exactly.
constexpr int DSCAN_THREADS = 256;
using DScanReduce = cub::BlockReduce<long long, DSCAN_THREADS>;
using DScanBlock = cub::BlockScan<long long, DSCAN_THREADS>;
__device__ __forceinline__ void dscan_chunk(long long n, long long& lo, long long& hi) {
    const long long per = (n + gridDim.x - 1) / gridDim.x;
    lo = min(n, (long long)blockIdx.x * per);
    hi = min(n, lo + per);
}
__global__ void __launch_bounds__(DSCAN_THREADS) k_dscan_reduce(const long long* __restrict__ in, const long long* __restrict__ len,
                                                                long long* __restrict__ part) {
    __shared__ typename DScanReduce::TempStorage tmp;
    long long lo, hi;
    dscan_chunk(*len, lo, hi);
    long long s = 0;
    for (long long i = lo + threadIdx.x; i < hi; i += DSCAN_THREADS) s += in[i];
    s = DScanReduce(tmp).Sum(s);
    if (threadIdx.x == 0) part[blockIdx.x] = s;
}
// one block: part[0 .. nb) becomes its exclusive scan, part[nb] the total
__global__ void __launch_bounds__(DSCAN_THREADS) k_dscan_partials(long long* __restrict__ part, int nb) {
    __shared__ typename DScanBlock::TempStorage tmp;
    long long carry = 0;
    for (int base = 0; base < nb; base += DSCAN_THREADS) {
        const int i = base + threadIdx.x;
        long long y, tile;
        DScanBlock(tmp).ExclusiveSum(i < nb ? part[i] : 0ll, y, tile);
        if (i < nb) part[i] = carry + y;
        carry += tile;
        __syncthreads();
    }
    if (threadIdx.x == 0) part[nb] = carry;
}
__global__ void __launch_bounds__(DSCAN_THREADS) k_dscan_down(const long long* __restrict__ in, const long long* __restrict__ len,
                                                              const long long* __restrict__ part, long long* __restrict__ out) {
    __shared__ typename DScanBlock::TempStorage tmp;
    const long long n = *len;
    long long lo, hi;
    dscan_chunk(n, lo, hi);
    long long carry = part[blockIdx.x];
    for (long long base = lo; base < hi; base += DSCAN_THREADS) {       // block-uniform trip count
        const long long i = base + threadIdx.x;
        long long y, tile;
        DScanBlock(tmp).ExclusiveSum(i < hi ? in[i] : 0ll, y, tile);
        if (i < hi) out[i] = carry + y;
        carry += tile;
        __syncthreads();
    }
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) out[n] = part[gridDim.x];
}

// ============================================================================= host
static inline int blocks_for(long long threads, int block, int cap = 132 * 16) {      // 16 blocks on each of the H100 SXM's 132 SMs
    long long b = (threads + block - 1) / block;
    return (int)std::max<long long>(1, std::min<long long>(b, cap));
}

// Blocks for a grid-stride kernel over `threads` threads: no more than the device keeps resident at once.
template <class K>
static int resident_blocks(K kernel, int block, long long threads, int n_sm) {
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, block, 0) != cudaSuccess || per_sm < 1) { cudaGetLastError(); per_sm = 1; }
    const long long want = (threads + block - 1) / block;
    return (int)std::max<long long>(1, std::min<long long>(want, (long long)std::max(n_sm, 1) * per_sm));
}

Map::Map(int device, float downsample_size) : device_(device), downsample_(downsample_size) { memset(&v_, 0, sizeof(v_)); }

Map::~Map() {
    cudaSetDevice(device_);
    pts_.release(); payload_.release(); next_.release(); counters_.release(); dir_tab_.release(); dir_lists_.release(); removed_.release(); ins_slots_.release(); dir_fix_.release();
    for (int k = 0; k < MAX_LEVELS; k++) ebox_[k].release();
    segid_.release(); segtab_[0].release(); segtab_[1].release(); bbox_.release();
    src_.release(); keys_in_.release(); keys_out_.release(); vals_in_.release(); vals_out_.release();
    cub_tmp_.release(); scratch_.release(); scratch2_.release(); scratch3_.release();
    range_ws_.release(); range_out_.release();
    a_keys_in_.release(); a_keys_out_.release(); a_vals_in_.release(); a_vals_out_.release(); a_groups_.release(); a_ins_.release();
    a_slots_.release(); a_fix_.release(); a_cub_.release(); cellcnt_.release();
    if (h_counters_) cudaFreeHost(h_counters_);
    if (ev_front_) cudaEventDestroy(ev_front_);
    if (ev_caller_) cudaEventDestroy(ev_caller_);
    if (stream_) cudaStreamDestroy(stream_);
}

int Map::init() {
    FL_CUDA(cudaSetDevice(device_));
    FL_CUDA(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
    FL_CUDA(cudaDeviceGetAttribute(&n_sm_, cudaDevAttrMultiProcessorCount, device_));
    FL_CUDA(cudaEventCreateWithFlags(&ev_front_, cudaEventDisableTiming));
    FL_CUDA(cudaEventCreateWithFlags(&ev_caller_, cudaEventDisableTiming));
    FL_CHECK(counters_.reserve(sizeof(int) * C_COUNT));
    FL_CUDA(cudaMemsetAsync(counters_.ptr, 0, sizeof(int) * C_COUNT, stream_));
    FL_CUDA(cudaMallocHost(&h_counters_, sizeof(int) * C_COUNT));
    memset(h_counters_, 0, sizeof(int) * C_COUNT);
    if (const char* e = getenv("FASTLIO_B200_NO_CELLDIR")) dir_enabled_ = !(e[0] == '1');      // A/B: BVH walk only
    if (const char* e = getenv("FASTLIO_B200_CELL")) cell_override_ = (float)atof(e);           // A/B: cell edge in metres
    // an empty map: one empty leaf under a one-level root, so that every kernel is well defined
    FL_CHECK(src_.reserve(sizeof(float4)));
    return build_from_sorted(src_.as<float4>(), 0);
}

int Map::ensure_capacity(int n_points) {
    const int n_main = std::max(1, (n_points + fill_ - 1) / fill_);
    // overflow pool: half the main leaves, never less than 64k leaves (32 MB) -- enough for
    // any single Add_Points batch to take one fresh leaf per point in the worst case
    const long long want = (long long)n_main + std::max<long long>(n_main / 2, min_pool_);
    if (want > 0x7fffffff / LEAF) { set_last_error("map too large: %d points", n_points); return FL_ERR_CAPACITY; }
    if (want > v_.leaf_cap || !pts_.ptr) {
        FL_CHECK(pts_.reserve(sizeof(float4) * LEAF * (size_t)want));
        FL_CHECK(payload_.reserve(sizeof(float) * LEAF * (size_t)want));
        FL_CHECK(next_.reserve(sizeof(int) * (size_t)want));
        v_.leaf_cap = (int)std::min<size_t>({pts_.bytes / (sizeof(float4) * LEAF), payload_.bytes / (sizeof(float) * LEAF),
                                              next_.bytes / sizeof(int)});
        v_.pts = pts_.as<float4>(); v_.payload = payload_.as<float>(); v_.next = next_.as<int>();
    }
    // level geometry
    v_.n_main = n_main;
    v_.count[0] = n_main;
    int k = 0;
    while (true) {
        const int c = v_.count[k];
        FL_CHECK(ebox_[k].reserve(sizeof(float4) * 2 * (size_t)c));
        v_.ebox[k] = ebox_[k].as<float4>();
        k++;
        if (c <= ROOT_FAN) { v_.count[k] = 1; break; }          // the root owns up to 64 entities of level k-1
        v_.count[k] = (c + FAN - 1) / FAN;
        if (k >= MAX_LEVELS) { set_last_error("too many tree levels"); return FL_ERR_CAPACITY; }
    }
    v_.n_levels = k;
    return FL_OK;
}

int Map::refit() {
    FL_CUDA(cudaSetDevice(device_));
    return refit_on(stream_, nullptr);
}
int Map::refit_on(cudaStream_t st, const int* gate) {
    k_refit_leaves<<<blocks_for((long long)v_.n_main * 32, 256), 256, 0, st>>>(v_, gate);
    for (int k = 1; k < v_.n_levels; k++)
        k_refit_level<<<blocks_for((long long)v_.count[k] * 32, 256), 256, 0, st>>>(v_, k, gate);
    FL_CUDA(cudaGetLastError());
    return FL_OK;
}

static int kd_depth(int span, long long pmax) {
    if (span <= 1) return 0;
    const int m = split_leaf(0, span, pmax);
    return 1 + std::max(kd_depth(m, pmax), kd_depth(span - m, pmax));
}

// d_src: n points (x, y, z, intensity) on the device, any order.
int Map::build_from_sorted(const float4* d_src, int n) {
    FL_CUDA(cudaSetDevice(device_));
    FL_CHECK(ensure_capacity(n));
    k_clear_leaves<<<blocks_for((long long)v_.leaf_cap * LEAF, 256), 256, 0, stream_>>>(v_);
    if (n > 0) {
        const int L = v_.n_main;
        long long pmax = 1;
        for (int k = 1; k < v_.n_levels; k++) pmax *= FAN;            // leaves under one child of the root
        const int depth = kd_depth(L, pmax);
        const size_t max_seg = (size_t)1 << depth;
        FL_CHECK(keys_in_.reserve(sizeof(unsigned long long) * (size_t)n));
        FL_CHECK(keys_out_.reserve(sizeof(unsigned long long) * (size_t)n));
        FL_CHECK(vals_in_.reserve(sizeof(unsigned) * (size_t)n));
        FL_CHECK(vals_out_.reserve(sizeof(unsigned) * (size_t)n));
        FL_CHECK(segid_.reserve(sizeof(int) * (size_t)n));
        FL_CHECK(segtab_[0].reserve(sizeof(Segment) * max_seg));
        FL_CHECK(segtab_[1].reserve(sizeof(Segment) * max_seg));
        FL_CHECK(bbox_.reserve(sizeof(float) * 6 * max_seg));
        unsigned* idx = vals_out_.as<unsigned>();          // current order of the points
        unsigned* idx_tmp = vals_in_.as<unsigned>();
        int* segid = segid_.as<int>();
        const int nb = blocks_for(n, 256, 1 << 30);
        k_kd_init<<<nb, 256, 0, stream_>>>(n, idx, segid, segtab_[0].as<Segment>(), L);
        int cur = 0;
        for (int lvl = 0; lvl < depth; lvl++) {
            const int nseg = 1 << lvl;
            k_kd_bbox_init<<<blocks_for((long long)nseg * 6, 256, 1 << 30), 256, 0, stream_>>>(bbox_.as<float>(), nseg);
            k_kd_bbox<<<nb, 256, 0, stream_>>>(d_src, idx, segid, n, bbox_.as<float>());
            k_kd_keys<<<nb, 256, 0, stream_>>>(d_src, idx, segid, n, bbox_.as<float>(), keys_in_.as<unsigned long long>(), idx_tmp);
            size_t tmp = 0;
            const int end_bit = 32 + std::max(1, lvl);
            FL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp, keys_in_.as<unsigned long long>(), keys_out_.as<unsigned long long>(),
                                                    idx_tmp, idx, n, 0, end_bit, stream_));
            FL_CHECK(cub_tmp_.reserve(tmp));
            tmp = cub_tmp_.bytes;
            FL_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp_.ptr, tmp, keys_in_.as<unsigned long long>(), keys_out_.as<unsigned long long>(),
                                                    idx_tmp, idx, n, 0, end_bit, stream_));
            k_kd_split<<<blocks_for(nseg, 256, 1 << 30), 256, 0, stream_>>>(segtab_[cur].as<Segment>(), segtab_[cur ^ 1].as<Segment>(), nseg, fill_, pmax);
            k_kd_assign<<<nb, 256, 0, stream_>>>(keys_out_.as<unsigned long long>(), n, segtab_[cur ^ 1].as<Segment>(), segid);
            cur ^= 1;
        }
        k_fill_leaves<<<nb, 256, 0, stream_>>>(v_, d_src, idx, segid, segtab_[cur].as<Segment>(), n);
    }
    FL_CUDA(cudaGetLastError());
    h_counters_[C_LEAF_USED] = v_.n_main;
    FL_CUDA(cudaMemcpyAsync(&counters_.as<int>()[C_LEAF_USED], &h_counters_[C_LEAF_USED], sizeof(int), cudaMemcpyHostToDevice, stream_));
    FL_CHECK(refit());
    FL_CUDA(cudaStreamSynchronize(stream_));
    n_valid_ = n;
    n_tomb_ = 0;
    built_ = true;
    layout_dirty_ = true;
    FL_CHECK(publish_counts());
    return build_directory();
}

// (Re)list the cell directory over the live slots.  Pass 1 counts into a table sized from the point count (re-sized when the
// cells turn out to be more numerous than guessed: load factor below ~0.6); the list pool is then sized from the counts.
int Map::build_directory() {
    FL_CUDA(cudaSetDevice(device_));
    if (!dir_enabled_) { v_.dir.cap = 0; return FL_OK; }
    const float cell = cell_override_ > 0.f ? cell_override_ : (downsample_ > 0.f ? 2.f * downsample_ : 1.f);
    const int used = h_counters_[C_LEAF_USED];
    size_t want_cap = std::max<size_t>(dir_min_cap_, std::max<size_t>(16384, (size_t)n_valid_ * 4));
    int* d_cnt = counters_.as<int>();
    const int nb = blocks_for((long long)used * LEAF, 256);
    for (int attempt = 0; attempt < 6; attempt++) {
        if (want_cap > 0xfffffff0ull / 2) { set_last_error("cell directory too large"); return FL_ERR_CAPACITY; }
        FL_CHECK(dir_tab_.reserve(sizeof(CellEntry) * want_cap));
        v_.dir.tab = dir_tab_.as<CellEntry>();
        v_.dir.cap = (unsigned)(dir_tab_.bytes / sizeof(CellEntry));
        v_.dir.cell = cell;
        v_.dir.inv_cell = 1.0f / cell;
        v_.dir.n_walked = &d_cnt[C_DIR_WALKED];
        FL_CUDA(cudaMemsetAsync(dir_tab_.ptr, 0, sizeof(CellEntry) * (size_t)v_.dir.cap, stream_));
        FL_CUDA(cudaMemsetAsync(&d_cnt[C_DIR_CELLS], 0, sizeof(int) * 4, stream_));      // CELLS, POOL, CROWDED, ERROR
        k_halo_count<<<nb, 256, 0, stream_>>>(v_, used, d_cnt);
        FL_CUDA(cudaGetLastError());
        FL_CUDA(cudaMemcpyAsync(&h_counters_[C_DIR_CELLS], &d_cnt[C_DIR_CELLS], sizeof(int) * 4, cudaMemcpyDeviceToHost, stream_));
        FL_CUDA(cudaStreamSynchronize(stream_));
        const size_t cells = (size_t)h_counters_[C_DIR_CELLS];
        if (h_counters_[C_DIR_ERROR] || cells * 10 > (size_t)v_.dir.cap * 6) { want_cap = std::max(want_cap * 2, cells * 5 / 2 + 16384); continue; }
        // lists: 27 listings per point + 25 % + 8 per cell (rounded to 4), plus room for the lists inserts will create
        const size_t pool = (size_t)n_valid_ * 27 + (size_t)n_valid_ * 27 / 4 + cells * 12 + std::max<size_t>(dir_min_pool_, std::max<size_t>((size_t)HALO_NEW_CAP * 262144, (size_t)n_valid_ * 6));
        if (pool > 0x7ffffff0ull) { set_last_error("cell directory: list pool too large"); return FL_ERR_CAPACITY; }
        FL_CHECK(dir_lists_.reserve(sizeof(int) * pool));
        v_.dir.lists = dir_lists_.as<int>();
        v_.dir.lists_cap = (int)std::min<size_t>(dir_lists_.bytes / sizeof(int), 0x7ffffff0ull);
        // the slack at the end of a list is read (and ignored) by the 16-byte loads of the search: keep it defined
        FL_CUDA(cudaMemsetAsync(dir_lists_.ptr, 0, sizeof(int) * (size_t)v_.dir.lists_cap, stream_));
        k_halo_alloc<<<blocks_for(v_.dir.cap, 256), 256, 0, stream_>>>(v_, d_cnt);
        k_halo_fill<<<nb, 256, 0, stream_>>>(v_, used);
        FL_CUDA(cudaGetLastError());
        FL_CUDA(cudaMemcpyAsync(&h_counters_[C_DIR_CELLS], &d_cnt[C_DIR_CELLS], sizeof(int) * 4, cudaMemcpyDeviceToHost, stream_));
        FL_CUDA(cudaStreamSynchronize(stream_));
        if (h_counters_[C_DIR_ERROR]) { dir_min_pool_ = std::max<size_t>(dir_min_pool_ * 2, (size_t)HALO_NEW_CAP * 262144); continue; }
        layout_dirty_ = true;
        if (async_used_) {          // the plan's per-entry counters (k_plan_count): one int per table entry, all zero
            FL_CHECK(cellcnt_.reserve(sizeof(int) * (size_t)v_.dir.cap));
            FL_CUDA(cudaMemsetAsync(cellcnt_.ptr, 0, cellcnt_.bytes, stream_));
        }
        return FL_OK;
    }
    set_last_error("cell directory: could not size the table");
    return FL_ERR_CAPACITY;
}

int Map::dir_stats(int* out6) const {
    // [5]: queries answered by the BVH walk since the last call (0 when the directory is off: every query walks)
    int walked = 0;
    if (v_.dir.cap) {
        cudaSetDevice(device_);
        cudaMemcpyAsync(&walked, &counters_.as<int>()[C_DIR_WALKED], sizeof(int), cudaMemcpyDeviceToHost, stream_);
        cudaMemsetAsync(&counters_.as<int>()[C_DIR_WALKED], 0, sizeof(int), stream_);
        cudaStreamSynchronize(stream_);
    }
    out6[0] = h_counters_[C_DIR_CELLS]; out6[1] = h_counters_[C_DIR_POOL]; out6[2] = h_counters_[C_DIR_CROWDED];
    out6[3] = (int)v_.dir.cap; out6[4] = n_dir_rebuilds_; out6[5] = v_.dir.cap ? walked : -1;
    return FL_OK;
}

int Map::build_device(const float4* d_pts_xyzi, int n) {
    if (n < 0) { set_last_error("build: n < 0"); return FL_ERR_ARG; }
    return build_from_sorted(d_pts_xyzi, n);
}

int Map::build(const float* pts_xyzi, int n) {
    if (n < 0 || (n > 0 && !pts_xyzi)) { set_last_error("build: bad arguments"); return FL_ERR_ARG; }
    FL_CUDA(cudaSetDevice(device_));
    FL_CHECK(src_.reserve(sizeof(float4) * (size_t)std::max(n, 1)));
    if (n > 0) FL_CUDA(cudaMemcpyAsync(src_.ptr, pts_xyzi, sizeof(float4) * (size_t)n, cudaMemcpyHostToDevice, stream_));
    return build_from_sorted(src_.as<float4>(), n);
}

// The one launch of a batched nearest search on `st`: fl_map_knn's k_knn_batch (ungated), or fl_map_nearest_search's
// k_knn_batch_gated (k <= KNN_K) or k_knn_k.
void Map::launch_knn(bool gated, const float4* q, int nq, int k, float md2, float4* p, float* d2, int* cnt, cudaStream_t st) {
    if (det_) {                  // the keyed tie rule
        if (!gated) k_knn_batch_det<<<blocks_for(nq, 128, 1 << 20), 128, 0, st>>>(v_, q, nq, k, p, d2, cnt);
        else if (k <= KNN_K) k_knn_batch_gated_det<<<blocks_for(nq, 128, 1 << 20), 128, 0, st>>>(v_, q, nq, k, md2, p, d2, cnt);
        else k_knn_k_det<<<resident_blocks(k_knn_k_det, 256, (long long)nq * 32, n_sm_), 256, 0, st>>>(v_, q, nq, k, md2, p, d2, cnt);
        return;
    }
    if (!gated) k_knn_batch<<<blocks_for(nq, 128, 1 << 20), 128, 0, st>>>(v_, q, nq, k, p, d2, cnt);
    else if (k <= KNN_K) k_knn_batch_gated<<<blocks_for(nq, 128, 1 << 20), 128, 0, st>>>(v_, q, nq, k, md2, p, d2, cnt);
    else k_knn_k<<<resident_blocks(k_knn_k, 256, (long long)nq * 32, n_sm_), 256, 0, st>>>(v_, q, nq, k, md2, p, d2, cnt);
}

// host buffers: the queries in through scratch_, launch_knn on the handle's stream, the three outputs back
int Map::knn_host(bool gated, const float* q_xyzi, int nq, int k, float md2, float* out_pts, float* out_d2, int* out_cnt) {
    FL_CUDA(cudaSetDevice(device_));
    const size_t qb = sizeof(float4) * (size_t)nq, pb = sizeof(float4) * (size_t)nq * k, db = sizeof(float) * (size_t)nq * k, cb = sizeof(int) * (size_t)nq;
    FL_CHECK(scratch_.reserve(qb + pb + db + cb));
    char* base = scratch_.as<char>();
    float4* d_q = (float4*)base; float4* d_p = (float4*)(base + qb); float* d_d = (float*)(base + qb + pb); int* d_c = (int*)(base + qb + pb + db);
    FL_CUDA(cudaMemcpyAsync(d_q, q_xyzi, qb, cudaMemcpyHostToDevice, stream_));
    launch_knn(gated, d_q, nq, k, md2, d_p, d_d, d_c, stream_);
    FL_CUDA(cudaGetLastError());
    FL_CUDA(cudaMemcpyAsync(out_pts, d_p, pb, cudaMemcpyDeviceToHost, stream_));
    FL_CUDA(cudaMemcpyAsync(out_d2, d_d, db, cudaMemcpyDeviceToHost, stream_));
    FL_CUDA(cudaMemcpyAsync(out_cnt, d_c, cb, cudaMemcpyDeviceToHost, stream_));
    FL_CUDA(cudaStreamSynchronize(stream_));
    return FL_OK;
}

int Map::knn(const float* q_xyzi, int nq, int k, float* out_pts, float* out_d2, int* out_cnt) {
    if (nq < 0 || k < 1 || k > KNN_K) { set_last_error("knn: k must be in [1, %d]", KNN_K); return FL_ERR_ARG; }
    if (nq == 0) return FL_OK;
    return knn_host(false, q_xyzi, nq, k, 0.f, out_pts, out_d2, out_cnt);
}

int Map::nearest_search(const float* q_xyzi, int nq, int k, float max_dist, float* out_pts, float* out_d2, int* out_cnt) {
    if (nq < 0 || k < 1 || k > KNN_KMAX) { set_last_error("nearest_search: k must be in [1, %d]", KNN_KMAX); return FL_ERR_ARG; }
    if (nq == 0) return FL_OK;
    return knn_host(true, q_xyzi, nq, k, max_dist * max_dist, out_pts, out_d2, out_cnt);      // md2 in float32, as ikd_Tree.cpp:1067
}

int Map::overflow_leaves() const { return h_counters_ ? h_counters_[C_LEAF_USED] - v_.n_main : 0; }

int Map::delete_boxes(const float* boxes6, int nb, int* deleted) {
    if (deleted) *deleted = 0;
    if (nb < 0 || (nb > 0 && !boxes6)) { set_last_error("delete_boxes: bad arguments"); return FL_ERR_ARG; }
    if (nb == 0) return FL_OK;
    FL_CUDA(cudaSetDevice(device_));
    FL_CHECK(scratch_.reserve(sizeof(float) * 6 * (size_t)nb));
    FL_CUDA(cudaMemcpyAsync(scratch_.ptr, boxes6, sizeof(float) * 6 * (size_t)nb, cudaMemcpyHostToDevice, stream_));
    FL_CUDA(cudaMemsetAsync(&counters_.as<int>()[C_DELETED], 0, sizeof(int), stream_));
    const int used = h_counters_[C_LEAF_USED];
    if (record_removed_) FL_CHECK(removed_room());
    k_delete_boxes<<<blocks_for((long long)used * LEAF, 256), 256, 0, stream_>>>(v_, scratch_.as<float>(), nb, used, counters_.as<int>(),
                                                                                   record_removed_ ? removed_.as<float4>() : nullptr,
                                                                                   removed_cap(), nullptr, nullptr);
    FL_CUDA(cudaGetLastError());
    FL_CUDA(cudaMemcpyAsync(&h_counters_[C_DELETED], &counters_.as<int>()[C_DELETED], sizeof(int), cudaMemcpyDeviceToHost, stream_));
    FL_CUDA(cudaStreamSynchronize(stream_));
    const int d = h_counters_[C_DELETED];
    if (record_removed_) n_removed_ += d;
    if (d > 0) {
        n_valid_ -= d; n_tomb_ += d;
        FL_CHECK(refit());          // tighten every AABB ("box-delete by refit")
        FL_CHECK(maybe_rebuild());
        FL_CHECK(publish_counts());
    }
    if (deleted) *deleted = d;
    return FL_OK;
}

// Room in the removed-points record for the worst case of one more delete: every valid point on top of what it holds.  A record
// that is allocated or moves leaves graphs captured before stale (they hold no record, or the old one).  Synchronous; the map
// must be settled.
int Map::removed_room() {
    const size_t want = (size_t)n_removed_ + (size_t)n_valid_;
    if (want * sizeof(float4) <= removed_.bytes && removed_.ptr) return FL_OK;
    DeviceBuffer bigger;
    FL_CHECK(bigger.reserve(sizeof(float4) * std::max<size_t>(want + want / 2, 1)));
    if (n_removed_) FL_CUDA(cudaMemcpyAsync(bigger.ptr, removed_.ptr, sizeof(float4) * (size_t)n_removed_, cudaMemcpyDeviceToDevice, stream_));
    FL_CUDA(cudaStreamSynchronize(stream_));
    layout_dirty_ = true;
    removed_.release();
    removed_ = bigger;
    return FL_OK;
}
int Map::removed_cap() const { return (int)std::min<size_t>(removed_.bytes / sizeof(float4), 0x7fffffff); }

// Delete_Point_Boxes of up to nb_max boxes at `boxes`, count at *nb_dev, on `st`; status2 = (status, deleted).  The plan decides
// first (k_delete_plan); the pass over the slots reads the used leaves from the device counters, and the refit runs only when a
// point went away.  Every grid is fixed on the host: the same launches whether or not anything is deleted.
int Map::enqueue_delete(const float* boxes, const int* nb_dev, int nb_max, int* status2, cudaStream_t st) {
    int* d_cnt = counters_.as<int>();
    const int chain_limit = std::max(64, (int)(rebuild_overflow_frac_ * v_.n_main));
    k_delete_plan<<<1, 1, 0, st>>>(d_cnt, nb_dev, nb_max, record_removed_, removed_cap());
    const int g = resident_blocks(k_delete_boxes, 256, (long long)v_.leaf_cap * LEAF, n_sm_);
    k_delete_boxes<<<g, 256, 0, st>>>(v_, boxes, nb_max, 0, d_cnt, record_removed_ ? removed_.as<float4>() : nullptr, removed_cap(),
                                      &d_cnt[C_DEL_NB], &d_cnt[C_LEAF_USED]);
    k_delete_account<<<1, 1, 0, st>>>(v_, d_cnt, chain_limit);
    FL_CHECK(refit_on(st, &d_cnt[C_DELETED]));          // tighten every AABB, when something was deleted
    k_delete_status<<<1, 1, 0, st>>>(d_cnt, status2);
    FL_CUDA(cudaGetLastError());
    return FL_OK;
}

// Room in the removed-points record by the host's bound (deletes move points from the valid count to the record, device-form
// inserts since the last settle add at most ub_n_ valid points).  Outside capture, when it might be short, the map settles and
// the record grows (synchronously).  On a capturing stream such a call is FL_ERR_CAPACITY and captures nothing, as
// async_prepare does: a graph captured with no record, or too small a one, would refuse every delete until captured again.
// Replays that fill the record later are refused by the plan.
int Map::delete_prepare(cudaStream_t st) {
    if (!record_removed_) return FL_OK;
    const size_t bound = (size_t)n_removed_ + (size_t)n_valid_ + (size_t)ub_n_;
    if (bound * sizeof(float4) <= removed_.bytes && removed_.ptr) return FL_OK;
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    FL_CUDA(cudaStreamGetCaptureInfo(st, &cs));
    if (cs != cudaStreamCaptureStatusNone) {
        set_last_error("delete_boxes_async: the removed-points record might not hold this delete; call fl_map_maintain (or the call "
                       "once outside capture) first");
        return FL_ERR_CAPACITY;
    }
    FL_CHECK(settle(false));
    return removed_room();
}

int Map::delete_boxes_async_checked(const float* d_boxes, const int* d_nb, int nb_max, int* d_status2, cudaStream_t st) {
    if (nb_max < 0 || !device_ptr(d_nb, device_, 4) || !device_ptr(d_status2, device_, 4) || (nb_max > 0 && !device_ptr(d_boxes, device_, 4))) {
        set_last_error("delete_boxes_async: nb_max < 0, or a buffer is not 4-byte aligned device memory on device %d", device_);
        return FL_ERR_ARG;
    }
    FL_CUDA(cudaSetDevice(device_));
    if (nb_max == 0) {                                  // nothing can be deleted: (FL_OK, 0)
        bool joined = false;
        FL_CHECK(query_begin(st, &joined));
        FL_CUDA(cudaMemsetAsync(d_status2, 0, 2 * sizeof(int), st));
        return query_end(st, joined);
    }
    FL_CHECK(delete_prepare(st));
    bool joined = false;
    FL_CHECK(mutation_begin(st, &joined));
    FL_CHECK(enqueue_delete(d_boxes, d_nb, nb_max, d_status2, st));
    return mutation_end(st, joined);
}

// KD_TREE::acquire_removed_points (ikd_Tree.cpp:661-676): the points Delete_Point_Boxes removed since the last call.  Recording
// starts with the first call (the reference's caller asks before every box delete, laserMapping.cpp:273-275).
int Map::acquire_removed(float* out_xyzi, int cap, int* n_out) {
    FL_CUDA(cudaSetDevice(device_));
    const int n = n_removed_;
    if (n_out) *n_out = n;
    if (!record_removed_) {
        record_removed_ = true;
        layout_dirty_ = true;           // device-form deletes captured before record nothing: capture them again
        FL_CUDA(cudaMemsetAsync(&counters_.as<int>()[C_REMOVED], 0, sizeof(int), stream_));
        return FL_OK;
    }
    if (n > 0 && out_xyzi && cap > 0)
        FL_CUDA(cudaMemcpyAsync(out_xyzi, removed_.ptr, sizeof(float4) * (size_t)std::min(n, cap), cudaMemcpyDeviceToHost, stream_));
    FL_CUDA(cudaMemsetAsync(&counters_.as<int>()[C_REMOVED], 0, sizeof(int), stream_));
    FL_CUDA(cudaStreamSynchronize(stream_));
    n_removed_ = 0;
    return FL_OK;
}

// KD_TREE::Add_Point_Boxes (ikd_Tree.cpp:576-603)
int Map::add_boxes(const float* boxes6, int nb, int* revived) {
    if (revived) *revived = 0;
    if (nb < 0 || (nb > 0 && !boxes6)) { set_last_error("add_boxes: bad arguments"); return FL_ERR_ARG; }
    if (nb == 0) return FL_OK;
    FL_CUDA(cudaSetDevice(device_));
    FL_CHECK(scratch_.reserve(sizeof(float) * 6 * (size_t)nb));
    FL_CUDA(cudaMemcpyAsync(scratch_.ptr, boxes6, sizeof(float) * 6 * (size_t)nb, cudaMemcpyHostToDevice, stream_));
    FL_CUDA(cudaMemsetAsync(&counters_.as<int>()[C_REVIVED], 0, sizeof(int), stream_));
    const int used = h_counters_[C_LEAF_USED];
    k_revive_boxes<<<blocks_for((long long)used * LEAF, 256), 256, 0, stream_>>>(v_, scratch_.as<float>(), nb, used, counters_.as<int>());
    FL_CUDA(cudaGetLastError());
    FL_CUDA(cudaMemcpyAsync(&h_counters_[C_REVIVED], &counters_.as<int>()[C_REVIVED], sizeof(int), cudaMemcpyDeviceToHost, stream_));
    FL_CUDA(cudaStreamSynchronize(stream_));
    const int r = h_counters_[C_REVIVED];
    if (r > 0) {
        n_valid_ += r; n_tomb_ = std::max(0, n_tomb_ - r);
        FL_CHECK(refit());          // the boxes were tightened when the points went away
        FL_CHECK(publish_counts());
    }
    if (revived) *revived = r;
    return FL_OK;
}

int Map::set_deterministic(bool on) {
    FL_CUDA(cudaSetDevice(device_));
    FL_CUDA(cudaStreamSynchronize(stream_));     // work already queued on the handle's stream runs under the mode it was queued in
    det_ = on;
    return FL_OK;
}

int Map::flatten(float* out_xyzi, int cap, int* n_out) {
    FL_CUDA(cudaSetDevice(device_));
    FL_CHECK(src_.reserve(sizeof(float4) * (size_t)std::max(1, n_valid_)));
    FL_CUDA(cudaMemsetAsync(&counters_.as<int>()[C_COMPACT], 0, sizeof(int), stream_));
    const int used = h_counters_[C_LEAF_USED];
    k_compact<<<blocks_for((long long)used * LEAF, 256), 256, 0, stream_>>>(v_, used, src_.as<float4>(), counters_.as<int>());
    FL_CUDA(cudaGetLastError());
    FL_CUDA(cudaMemcpyAsync(&h_counters_[C_COMPACT], &counters_.as<int>()[C_COMPACT], sizeof(int), cudaMemcpyDeviceToHost, stream_));
    FL_CUDA(cudaStreamSynchronize(stream_));
    const int n = h_counters_[C_COMPACT];
    if (n != n_valid_) { set_last_error("flatten: %d valid points on device, host expected %d", n, n_valid_); return FL_ERR_STATE; }
    if (n_out) *n_out = n;
    const float4* rows = src_.as<float4>();
    if (det_ && out_xyzi && cap > 0 && n > 1) {
        FL_CHECK(keys_in_.reserve(sizeof(unsigned long long) * (size_t)n));
        FL_CHECK(keys_out_.reserve(sizeof(unsigned long long) * (size_t)n));
        FL_CHECK(vals_in_.reserve(sizeof(unsigned) * (size_t)n));
        FL_CHECK(vals_out_.reserve(sizeof(unsigned) * (size_t)n));
        FL_CHECK(scratch3_.reserve(sizeof(float4) * (size_t)n));
        size_t tmp = 0;
        FL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp, keys_in_.as<unsigned long long>(), keys_out_.as<unsigned long long>(),
                                                vals_in_.as<unsigned>(), vals_out_.as<unsigned>(), n, 0, 64, stream_));
        FL_CHECK(cub_tmp_.reserve(tmp));
        for (int xy = 0; xy < 2; xy++) {
            k_flatten_keys<<<blocks_for(n, 256, 1 << 30), 256, 0, stream_>>>(rows, xy ? vals_out_.as<unsigned>() : nullptr, n, xy != 0,
                                                                             keys_in_.as<unsigned long long>(), vals_in_.as<unsigned>());
            tmp = cub_tmp_.bytes;
            FL_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp_.ptr, tmp, keys_in_.as<unsigned long long>(), keys_out_.as<unsigned long long>(),
                                                    vals_in_.as<unsigned>(), vals_out_.as<unsigned>(), n, 0, 64, stream_));
        }
        k_gather_rows<<<blocks_for(n, 256, 1 << 30), 256, 0, stream_>>>(rows, vals_out_.as<unsigned>(), n, scratch3_.as<float4>());
        FL_CUDA(cudaGetLastError());
        rows = scratch3_.as<float4>();
    }
    if (out_xyzi && cap > 0) {
        FL_CUDA(cudaMemcpyAsync(out_xyzi, rows, sizeof(float4) * (size_t)std::min(n, cap), cudaMemcpyDeviceToHost, stream_));
        FL_CUDA(cudaStreamSynchronize(stream_));
    }
    return FL_OK;
}

// Host buffers: the queries in, the count stage on the handle's stream, one read of status2, the emit stage, the answer out.
// The workspace holds the most pairs laid out by any earlier call on the handle, and at least max(4 nq, 1024); a call that
// needs more pairs than that runs the count stage a second time, in a workspace grown to exactly what it needs.
int Map::range_search(bool radius, const float* queries, int nq, int* out_offsets, float* out_xyzi, int cap, long long* total) {
    if (total) *total = 0;
    const char* what = radius ? "radius_search" : "box_search";
    if (nq < 0 || cap < 0 || !out_offsets || (nq > 0 && !queries) || (cap > 0 && !out_xyzi)) {
        set_last_error("%s: bad arguments (null buffer or negative size)", what);
        return FL_ERR_ARG;
    }
    memset(out_offsets, 0, sizeof(int) * ((size_t)nq + 1));
    if (nq == 0) return FL_OK;
    FL_CUDA(cudaSetDevice(device_));
    // range_out_: status2, the CSR offsets, then the points (grown for those only after status2 has been read)
    const size_t ob = 16 + ((sizeof(int) * ((size_t)nq + 1) + 15) & ~(size_t)15);
    FL_CHECK(range_out_.reserve(ob));
    long long status2[2] = {0, 0};
    RangeWorkspace w;
    auto count = [&](long long max_pairs) -> int {
        FL_CHECK(range_workspace(nq, max_pairs, w));
        FL_CHECK(range_ws_.reserve(w.bytes));
        range_ws_pairs_ = std::max(range_ws_pairs_, max_pairs);
        FL_CUDA(cudaMemcpyAsync(range_ws_.as<char>() + w.q, queries, sizeof(float) * (radius ? 4 : 6) * (size_t)nq, cudaMemcpyHostToDevice, stream_));
        FL_CHECK(range_count(radius, nq, w, range_ws_.as<char>(), range_out_.as<long long>(), stream_));
        FL_CUDA(cudaMemcpyAsync(status2, range_out_.ptr, sizeof(status2), cudaMemcpyDeviceToHost, stream_));
        FL_CUDA(cudaStreamSynchronize(stream_));
        return FL_OK;
    };
    FL_CHECK(count(std::max({range_ws_pairs_, 4ll * nq, 1024ll})));
    if (status2[0] == -1) {                 // the pairs did not fit the workspace
        if (status2[1] > INT_MAX) { set_last_error("%s: %lld (query, leaf) pairs exceed INT_MAX; split the batch", what, status2[1]); return FL_ERR_CAPACITY; }
        FL_CHECK(count(status2[1]));
    }
    const long long n = status2[0];
    if (n > INT_MAX) { set_last_error("%s: %lld points found exceed INT_MAX; split the batch", what, n); return FL_ERR_CAPACITY; }
    const long long m = std::min<long long>(n, cap);
    FL_CHECK(range_out_.reserve(ob + sizeof(float4) * (size_t)m));
    int* d_offsets = reinterpret_cast<int*>(range_out_.as<char>() + 16);
    float4* d_pts = reinterpret_cast<float4*>(range_out_.as<char>() + ob);
    FL_CHECK(range_emit(radius, nq, w, range_ws_.as<char>(), d_offsets, d_pts, m, stream_));
    FL_CUDA(cudaMemcpyAsync(out_offsets, d_offsets, sizeof(int) * ((size_t)nq + 1), cudaMemcpyDeviceToHost, stream_));
    if (m > 0) FL_CUDA(cudaMemcpyAsync(out_xyzi, d_pts, sizeof(float4) * (size_t)m, cudaMemcpyDeviceToHost, stream_));
    FL_CUDA(cudaStreamSynchronize(stream_));
    if (total) *total = n;
    return FL_OK;
}

// ----------------------------------------------------------------------------- device-buffer forms
bool device_ptr(const void* p, int device, size_t align) {
    if (!p || (reinterpret_cast<uintptr_t>(p) % align) != 0) return false;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) && a.device == device;
}

// Outside stream capture the caller's stream first waits for everything enqueued on the handle's stream (a filter run, a
// mutation); the event is recorded anew only when that stream may have received work since the last query (touch()), so
// queries on two caller streams do not wait for each other.  While `st` is capturing nothing is joined.
int Map::query_begin(cudaStream_t st, bool* joined) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    FL_CUDA(cudaStreamGetCaptureInfo(st, &cs));
    *joined = cs == cudaStreamCaptureStatusNone;
    if (!*joined) return FL_OK;
    if (front_stale_) { FL_CUDA(cudaEventRecord(ev_front_, stream_)); front_stale_ = false; }
    FL_CUDA(cudaStreamWaitEvent(st, ev_front_, 0));
    return FL_OK;
}
// ... and afterwards the handle's stream waits for the query, so no later mutation overwrites the map under it
int Map::query_end(cudaStream_t st, bool joined) {
    FL_CUDA(cudaGetLastError());
    if (!joined) return FL_OK;
    FL_CUDA(cudaEventRecord(ev_caller_, st));
    FL_CUDA(cudaStreamWaitEvent(stream_, ev_caller_, 0));
    return FL_OK;
}
// a synchronous call that reads caller device memory: its work on the handle's stream starts after what `st` holds
int Map::wait_for_caller(cudaStream_t st, const char* what) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    FL_CUDA(cudaStreamGetCaptureInfo(st, &cs));
    if (cs != cudaStreamCaptureStatusNone) { set_last_error("%s: synchronous, cannot be called on a capturing stream", what); return FL_ERR_ARG; }
    FL_CUDA(cudaEventRecord(ev_caller_, st));
    FL_CUDA(cudaStreamWaitEvent(stream_, ev_caller_, 0));
    return FL_OK;
}

int Map::build_from_caller(const float* d_pts_xyzi, int n, cudaStream_t st) {
    if (n < 0 || (n > 0 && !device_ptr(d_pts_xyzi, device_, 16))) {
        set_last_error("build_device: n < 0, or the points are not 16-byte aligned device memory on device %d", device_);
        return FL_ERR_ARG;
    }
    FL_CUDA(cudaSetDevice(device_));
    FL_CHECK(wait_for_caller(st, "build_device"));
    return build_device(reinterpret_cast<const float4*>(d_pts_xyzi), n);
}

int Map::add_points_from_caller(const float* d_pts_xyzi, int n, bool downsample_on, cudaStream_t st, int* added) {
    if (added) *added = 0;
    if (n < 0 || (n > 0 && !device_ptr(d_pts_xyzi, device_, 16))) {
        set_last_error("add_points_device: n < 0, or the points are not 16-byte aligned device memory on device %d", device_);
        return FL_ERR_ARG;
    }
    if (n == 0) return FL_OK;
    FL_CUDA(cudaSetDevice(device_));
    FL_CHECK(wait_for_caller(st, "add_points_device"));
    return add_points_device(reinterpret_cast<const float4*>(d_pts_xyzi), n, downsample_on, added);
}

int Map::nearest_search_device(const float* q_xyzi, int nq, int k, float max_dist, float* out_pts, float* out_d2, int* out_cnt, cudaStream_t st) {
    if (nq < 0 || k < 1 || k > KNN_KMAX) { set_last_error("nearest_search_device: k must be in [1, %d]", KNN_KMAX); return FL_ERR_ARG; }
    if (nq > 0 && (!device_ptr(q_xyzi, device_, 16) || !device_ptr(out_pts, device_, 16) || !device_ptr(out_d2, device_, 4) ||
                   !device_ptr(out_cnt, device_, 4))) {
        set_last_error("nearest_search_device: every buffer must be device memory on device %d (queries and points 16-byte aligned)", device_);
        return FL_ERR_ARG;
    }
    if (nq == 0) return FL_OK;
    FL_CUDA(cudaSetDevice(device_));
    bool joined = false;
    FL_CHECK(query_begin(st, &joined));
    launch_knn(true, reinterpret_cast<const float4*>(q_xyzi), nq, k, max_dist * max_dist,      // md2 in float32, as ikd_Tree.cpp:1067
               reinterpret_cast<float4*>(out_pts), out_d2, out_cnt, st);
    return query_end(st, joined);
}

// The one layout of a range query's workspace: byte offsets from the first 256-byte boundary of the caller's buffer.
int Map::range_workspace(int nq, long long max_pairs, RangeWorkspace& w) const {
    size_t cub_bytes = 0;
    FL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, (long long*)nullptr, (long long*)nullptr, (long long)nq + 1));
    range_layout(nq, max_pairs, cub_bytes, w);
    return FL_OK;
}
void Map::range_layout(int nq, long long max_pairs, size_t cub_bytes, RangeWorkspace& w) const {
    size_t at = 0;
    auto take = [&at](size_t bytes) { const size_t o = at; at = (at + bytes + 255) & ~(size_t)255; return o; };
    w.q = take(sizeof(float) * 6 * (size_t)nq);                     // a copy of the queries (boxes or spheres), 16-byte aligned
    w.lcnt = take(sizeof(long long) * ((size_t)nq + 1));            // candidate leaves per query
    w.loff = take(sizeof(long long) * ((size_t)nq + 1));            // their offsets; loff[nq] = the pairs needed
    w.ctl = take(sizeof(long long) * RS_CTL_COUNT);
    w.part = take(sizeof(long long) * ((size_t)scan_blocks() + 1)); // partial sums of the device-length scan
    w.cub = take(cub_bytes);
    w.cub_bytes = cub_bytes;
    w.pairs = take(sizeof(int2) * (size_t)max_pairs);               // (query, leaf)
    w.pcnt = take(sizeof(long long) * (size_t)max_pairs);           // points per pair
    w.poff = take(sizeof(long long) * ((size_t)max_pairs + 1));     // their offsets
    w.max_pairs = max_pairs;
    w.bytes = at + 256;                                             // room to align the caller's pointer
}

int Map::range_workspace_bytes(int nq, long long max_pairs, unsigned long long* out) const {
    if (nq < 0 || max_pairs < 0 || max_pairs > (1ll << 40) || !out) { set_last_error("range_workspace_bytes: bad arguments"); return FL_ERR_ARG; }
    FL_CUDA(cudaSetDevice(device_));
    RangeWorkspace w;
    FL_CHECK(range_workspace(nq, max_pairs, w));
    *out = w.bytes;
    return FL_OK;
}

// Count stage, on the queries already copied to base + w.q: the candidate leaves, the pairs (only when they all fit), the
// points of each pair and their offsets, then status2 = (points found, pairs needed), or (-1, pairs needed).
int Map::range_count(bool radius, int nq, const RangeWorkspace& w, char* base, long long* status2, cudaStream_t st) {
    const float* d_q = reinterpret_cast<const float*>(base + w.q);
    long long* lcnt = reinterpret_cast<long long*>(base + w.lcnt);
    long long* loff = reinterpret_cast<long long*>(base + w.loff);
    long long* ctl = reinterpret_cast<long long*>(base + w.ctl);
    long long* part = reinterpret_cast<long long*>(base + w.part);
    int2* pairs = reinterpret_cast<int2*>(base + w.pairs);
    long long* pcnt = reinterpret_cast<long long*>(base + w.pcnt);
    long long* poff = reinterpret_cast<long long*>(base + w.poff);
    // 1. candidate leaves per query and their offsets (CUB over the host-known nq + 1); loff[nq] = the pairs needed
    FL_CUDA(cudaMemsetAsync(lcnt + nq, 0, sizeof(long long), st));
    const int qb = resident_blocks(radius ? k_range_leaves<true> : k_range_leaves<false>, 256, (long long)nq * 32, n_sm_);
    if (radius) k_range_leaves<true><<<qb, 256, 0, st>>>(v_, d_q, nq, lcnt, nullptr, nullptr);
    else k_range_leaves<false><<<qb, 256, 0, st>>>(v_, d_q, nq, lcnt, nullptr, nullptr);
    size_t cub_bytes = w.cub_bytes;
    FL_CUDA(cub::DeviceScan::ExclusiveSum(base + w.cub, cub_bytes, lcnt, loff, (long long)nq + 1, st));
    k_range_plan<<<1, 1, 0, st>>>(loff, nq, w.max_pairs, ctl);
    // 2. the pairs, the points of each, their offsets by the device-length scan
    const int lb = resident_blocks(radius ? k_range_leaves_bounded<true> : k_range_leaves_bounded<false>, 256, (long long)nq * 32, n_sm_);
    if (radius) k_range_leaves_bounded<true><<<lb, 256, 0, st>>>(v_, d_q, nq, loff, pairs, w.max_pairs);
    else k_range_leaves_bounded<false><<<lb, 256, 0, st>>>(v_, d_q, nq, loff, pairs, w.max_pairs);
    const int cb = resident_blocks(radius ? k_range_count_dev<true> : k_range_count_dev<false>, 256, w.max_pairs * 32, n_sm_);
    if (radius) k_range_count_dev<true><<<cb, 256, 0, st>>>(v_, d_q, pairs, ctl + RS_PAIRS, pcnt);
    else k_range_count_dev<false><<<cb, 256, 0, st>>>(v_, d_q, pairs, ctl + RS_PAIRS, pcnt);
    k_dscan_reduce<<<scan_blocks(), DSCAN_THREADS, 0, st>>>(pcnt, ctl + RS_PAIRS, part);
    k_dscan_partials<<<1, DSCAN_THREADS, 0, st>>>(part, scan_blocks());
    k_dscan_down<<<scan_blocks(), DSCAN_THREADS, 0, st>>>(pcnt, ctl + RS_PAIRS, part, poff);
    // 3. the status words
    k_range_status<<<1, 1, 0, st>>>(loff, poff, nq, w.max_pairs, ctl, status2);
    FL_CUDA(cudaGetLastError());
    return FL_OK;
}

// Emit stage, after the count stage on the same workspace: the CSR offsets (zeros unless status2 reported a total within
// INT_MAX) and the first `cap` points.
int Map::range_emit(bool radius, int nq, const RangeWorkspace& w, char* base, int* out_offsets, float4* out, long long cap, cudaStream_t st) {
    const float* d_q = reinterpret_cast<const float*>(base + w.q);
    const long long* loff = reinterpret_cast<const long long*>(base + w.loff);
    const long long* ctl = reinterpret_cast<const long long*>(base + w.ctl);
    const int2* pairs = reinterpret_cast<const int2*>(base + w.pairs);
    const long long* poff = reinterpret_cast<const long long*>(base + w.poff);
    k_range_offsets_dev<<<(nq + 256) / 256, 256, 0, st>>>(loff, poff, nq, ctl, out_offsets);
    if (cap > 0) {
        const int fb = resident_blocks(radius ? k_range_fill_dev<true> : k_range_fill_dev<false>, 256, w.max_pairs * 32, n_sm_);
        if (radius) k_range_fill_dev<true><<<fb, 256, 0, st>>>(v_, d_q, pairs, ctl + RS_FILL, poff, out, cap);
        else k_range_fill_dev<false><<<fb, 256, 0, st>>>(v_, d_q, pairs, ctl + RS_FILL, poff, out, cap);
    }
    FL_CUDA(cudaGetLastError());
    return FL_OK;
}

int Map::range_search_device(bool radius, const float* queries, int nq, int* out_offsets, float* out_xyzi, long long cap,
                             void* workspace, unsigned long long workspace_bytes, long long* status2, cudaStream_t st) {
    const char* what = radius ? "radius_search_device" : "box_search_device";
    if (nq < 0 || cap < 0) { set_last_error("%s: negative size", what); return FL_ERR_ARG; }
    if (!device_ptr(out_offsets, device_, 4) || !device_ptr(status2, device_, 8) || (nq > 0 && !device_ptr(queries, device_, 4)) ||
        (nq > 0 && !device_ptr(workspace, device_, 1)) || (cap > 0 && !device_ptr(out_xyzi, device_, 16))) {
        set_last_error("%s: every buffer must be device memory on device %d (points 16-byte aligned)", what, device_);
        return FL_ERR_ARG;
    }
    FL_CUDA(cudaSetDevice(device_));
    RangeWorkspace w;
    if (nq > 0) {                       // the most pairs the workspace holds
        FL_CHECK(range_workspace(nq, 0, w));
        if (workspace_bytes < w.bytes) {
            set_last_error("%s: a workspace of %llu bytes is below the %zu that %d queries need", what, workspace_bytes, w.bytes, nq);
            return FL_ERR_ARG;
        }
        // 24 bytes per pair; the 256-byte rounding of the three per-pair arrays moves the size by less than 64 pairs' worth
        const long long est = (long long)std::min<unsigned long long>((workspace_bytes - w.bytes) / (sizeof(int2) + 2 * sizeof(long long)), 1ull << 40);
        long long max_pairs;
        for (max_pairs = est + 64; max_pairs > 0; max_pairs--) {
            range_layout(nq, max_pairs, w.cub_bytes, w);
            if (w.bytes <= workspace_bytes) break;
        }
        range_layout(nq, max_pairs, w.cub_bytes, w);
    }
    bool joined = false;
    FL_CHECK(query_begin(st, &joined));
    if (nq == 0) {
        FL_CUDA(cudaMemsetAsync(out_offsets, 0, sizeof(int), st));
        FL_CUDA(cudaMemsetAsync(status2, 0, 2 * sizeof(long long), st));
        return query_end(st, joined);
    }
    char* base = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
    FL_CUDA(cudaMemcpyAsync(base + w.q, queries, sizeof(float) * (radius ? 4 : 6) * (size_t)nq, cudaMemcpyDeviceToDevice, st));
    FL_CHECK(range_count(radius, nq, w, base, status2, st));
    FL_CHECK(range_emit(radius, nq, w, base, out_offsets, reinterpret_cast<float4*>(out_xyzi), cap, st));
    return query_end(st, joined);
}

int Map::rebuild() {
    FL_CUDA(cudaSetDevice(device_));
    FL_CHECK(src_.reserve(sizeof(float4) * (size_t)std::max(1, n_valid_)));
    FL_CUDA(cudaMemsetAsync(&counters_.as<int>()[C_COMPACT], 0, sizeof(int), stream_));
    const int used = h_counters_[C_LEAF_USED];
    k_compact<<<blocks_for((long long)used * LEAF, 256), 256, 0, stream_>>>(v_, used, src_.as<float4>(), counters_.as<int>());
    FL_CUDA(cudaGetLastError());
    n_rebuilds_++;
    return build_from_sorted(src_.as<float4>(), n_valid_);
}

int Map::maybe_rebuild() {
    const int overflow = h_counters_[C_LEAF_USED] - v_.n_main;
    const bool too_chained = overflow > std::max(64, (int)(rebuild_overflow_frac_ * v_.n_main));
    const bool too_sparse = n_tomb_ > 1024 && n_tomb_ > n_valid_;       // ikd-Tree's delete criterion (alpha_del = 0.5)
    if (too_chained || too_sparse) return rebuild();
    return FL_OK;
}

int Map::insert_device(const float4* d_pts, int n) {
    if (n <= 0) return FL_OK;
    // worst case one fresh overflow leaf per point: guarantee the pool can take the batch
    if ((long long)h_counters_[C_LEAF_USED] + n > v_.leaf_cap) {
        min_pool_ = std::max(min_pool_, n + 1024);
        FL_CHECK(rebuild());            // re-packs the leaves and re-sizes the pool
    }
    if (v_.dir.cap) {
        // the insert kernels cope with a full table / an exhausted list pool (they flag it, the directory is re-listed below);
        // re-list beforehand only when the table could get so full that probing degenerates
        const size_t cells = (size_t)h_counters_[C_DIR_CELLS] + (size_t)n * 27;
        if (cells * 10 > (size_t)v_.dir.cap * 9) {
            dir_min_cap_ = std::max(dir_min_cap_, cells * 2 + 16384);
            n_dir_rebuilds_++;
            FL_CHECK(build_directory());
        }
    }
    FL_CHECK(ins_slots_.reserve(sizeof(int) * (size_t)n));
    k_insert<<<blocks_for((long long)n * 32, 256), 256, 0, stream_>>>(v_, d_pts, n, nullptr, counters_.as<int>(), ins_slots_.as<int>());
    if (v_.dir.cap) {
        k_halo_claim<<<blocks_for((long long)n * 32, 256), 256, 0, stream_>>>(v_, d_pts, ins_slots_.as<int>(), n, nullptr, counters_.as<int>());
        FL_CHECK(dir_fix_.reserve(sizeof(unsigned) * 65536));
        FL_CUDA(cudaMemsetAsync(&counters_.as<int>()[C_NFIX], 0, sizeof(int), stream_));
        k_halo_append<<<blocks_for((long long)n * 32, 256), 256, 0, stream_>>>(v_, d_pts, ins_slots_.as<int>(), n, nullptr, counters_.as<int>(),
                                                                                 dir_fix_.as<unsigned>(), 65536);
        k_halo_fix<<<296, 256, 0, stream_>>>(v_, dir_fix_.as<unsigned>(), 65536, counters_.as<int>());
    }
    FL_CUDA(cudaGetLastError());
    FL_CUDA(cudaMemcpyAsync(h_counters_, counters_.ptr, sizeof(int) * C_COUNT, cudaMemcpyDeviceToHost, stream_));
    FL_CUDA(cudaStreamSynchronize(stream_));
    if (h_counters_[C_ERROR]) { set_last_error("insert: overflow pool exhausted"); return FL_ERR_CAPACITY; }
    n_valid_ += n;
    // directory: out of room, or too many over-full cells (their queries walk the BVH) -> re-list the live slots
    if (v_.dir.cap) {
        const bool crowded = h_counters_[C_DIR_CROWDED] > std::max(64, h_counters_[C_DIR_CELLS] / 1024);
        if (h_counters_[C_DIR_ERROR]) {
            dir_min_cap_ = std::max(dir_min_cap_, (size_t)v_.dir.cap + (size_t)v_.dir.cap / 2);
            dir_min_pool_ = std::max<size_t>(dir_min_pool_ * 2, (size_t)HALO_NEW_CAP * 262144);
        }
        if (h_counters_[C_DIR_ERROR] || crowded) { n_dir_rebuilds_++; FL_CHECK(build_directory()); }
    }
    return FL_OK;
}

int Map::add_points_device(const float4* d_pts, int n, bool downsample_on, int* added) {
    FL_CHECK(add_points_host(d_pts, n, downsample_on, added));
    return publish_counts();
}

int Map::add_points_host(const float4* d_pts, int n, bool downsample_on, int* added) {
    if (added) *added = 0;
    if (n < 0) { set_last_error("add_points: n < 0"); return FL_ERR_ARG; }
    if (n == 0) return FL_OK;
    FL_CUDA(cudaSetDevice(device_));
    if (!downsample_on) {                                   // ikd_Tree.cpp:549-568: plain inserts, return value 0
        FL_CHECK(insert_device(d_pts, n));
        return maybe_rebuild();
    }
    FL_CHECK(keys_in_.reserve(sizeof(unsigned long long) * (size_t)n));
    FL_CHECK(keys_out_.reserve(sizeof(unsigned long long) * (size_t)n));
    FL_CHECK(vals_in_.reserve(sizeof(unsigned) * (size_t)n));
    FL_CHECK(vals_out_.reserve(sizeof(unsigned) * (size_t)n));
    FL_CHECK(scratch2_.reserve(sizeof(int) * (size_t)n));          // group starts
    FL_CHECK(scratch3_.reserve(sizeof(float4) * (size_t)n));       // insert list
    int* d_cnt = counters_.as<int>();
    FL_CUDA(cudaMemsetAsync(&d_cnt[C_ADDED], 0, sizeof(int) * 4, stream_));   // ADDED, GROUPS, NINSERT, TOMB
    k_voxel_keys<<<blocks_for(n, 256, 1 << 30), 256, 0, stream_>>>(d_pts, n, downsample_, keys_in_.as<unsigned long long>(), vals_in_.as<unsigned>(), nullptr);
    size_t tmp = 0;
    FL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp, keys_in_.as<unsigned long long>(), keys_out_.as<unsigned long long>(),
                                            vals_in_.as<unsigned>(), vals_out_.as<unsigned>(), n, 0, 63, stream_));
    FL_CHECK(cub_tmp_.reserve(tmp));
    tmp = cub_tmp_.bytes;
    FL_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp_.ptr, tmp, keys_in_.as<unsigned long long>(), keys_out_.as<unsigned long long>(),
                                            vals_in_.as<unsigned>(), vals_out_.as<unsigned>(), n, 0, 63, stream_));
    k_group_heads<<<blocks_for(n, 256, 1 << 30), 256, 0, stream_>>>(keys_out_.as<unsigned long long>(), n, scratch2_.as<int>(), d_cnt, nullptr);
    (det_ ? k_downsample_keyed : k_downsample_resolve)<<<blocks_for((long long)n * 32, 256), 256, 0, stream_>>>(
        v_, d_pts, keys_out_.as<unsigned long long>(), vals_out_.as<unsigned>(), n, scratch2_.as<int>(), downsample_,
        scratch3_.as<float4>(), d_cnt);
    FL_CUDA(cudaGetLastError());
    FL_CUDA(cudaMemcpyAsync(h_counters_, counters_.ptr, sizeof(int) * C_COUNT, cudaMemcpyDeviceToHost, stream_));
    FL_CUDA(cudaStreamSynchronize(stream_));
    const int n_ins = h_counters_[C_NINSERT], n_tomb = h_counters_[C_TOMB];
    if (added) *added = h_counters_[C_ADDED];
    n_valid_ -= n_tomb; n_tomb_ += n_tomb;
    FL_CHECK(insert_device(scratch3_.as<float4>(), n_ins));
    // tombstoned slots are reused by later inserts; they stop counting once re-occupied
    n_tomb_ = std::max(0, n_tomb_ - n_ins);
    return maybe_rebuild();
}

int Map::add_points(const float* pts_xyzi, int n, bool downsample_on, int* added) {
    if (added) *added = 0;
    if (n < 0 || (n > 0 && !pts_xyzi)) { set_last_error("add_points: bad arguments"); return FL_ERR_ARG; }
    if (n == 0) return FL_OK;
    FL_CUDA(cudaSetDevice(device_));
    FL_CHECK(scratch_.reserve(sizeof(float4) * (size_t)n));
    FL_CUDA(cudaMemcpyAsync(scratch_.ptr, pts_xyzi, sizeof(float4) * (size_t)n, cudaMemcpyHostToDevice, stream_));
    return add_points_device(scratch_.as<float4>(), n, downsample_on, added);
}

// ----------------------------------------------------------------------------- device forms of Add_Points
int Map::publish_counts() {
    k_set_counts<<<1, 1, 0, stream_>>>(counters_.as<int>(), n_valid_, n_tomb_, due_ ? 1 : 0);
    FL_CUDA(cudaGetLastError());
    return FL_OK;
}

int Map::settle(bool full, int* layout_changed) {
    FL_CUDA(cudaSetDevice(device_));
    if (pending_ || captured_) {
        // the device forms' work reached the handle's stream through mutation_end; graph replays the caller has synchronised
        FL_CUDA(cudaMemcpyAsync(h_counters_, counters_.ptr, sizeof(int) * C_COUNT, cudaMemcpyDeviceToHost, stream_));
        FL_CUDA(cudaStreamSynchronize(stream_));
        n_valid_ = h_counters_[C_VALID];
        n_tomb_ = h_counters_[C_TOMBS];
        if (record_removed_) n_removed_ = h_counters_[C_REMOVED];
        ub_n_ = 0;
        // what is owed survives read-only settles: only a full settle does it and clears it
        due_ = due_ || h_counters_[C_DUE] != 0;
        refused_ = refused_ || h_counters_[C_REFUSED] != 0;
        pending_ = false;
    }
    if (full && (due_ || refused_)) {
        // what the host form would have done after its inserts (insert_device, maybe_rebuild), then room for a refused call
        if (v_.dir.cap) {
            const bool crowded = h_counters_[C_DIR_CROWDED] > std::max(64, h_counters_[C_DIR_CELLS] / 1024);
            if (h_counters_[C_DIR_ERROR]) {
                dir_min_cap_ = std::max(dir_min_cap_, (size_t)v_.dir.cap + (size_t)v_.dir.cap / 2);
                dir_min_pool_ = std::max<size_t>(dir_min_pool_ * 2, (size_t)HALO_NEW_CAP * 262144);
            }
            if (h_counters_[C_DIR_ERROR] || crowded) { n_dir_rebuilds_++; FL_CHECK(build_directory()); }
        }
        FL_CHECK(maybe_rebuild());
        if (refused_) FL_CHECK(async_grow(async_n_max_, true));
        due_ = refused_ = false;
        h_counters_[C_REFUSED] = 0;
        FL_CUDA(cudaMemsetAsync(&counters_.as<int>()[C_REFUSED], 0, sizeof(int), stream_));
        FL_CHECK(publish_counts());          // C_DUE = 0
        FL_CUDA(cudaStreamSynchronize(stream_));
    }
    // room in the started removed-points record for the next delete (a device-form delete refused for it, a record started by
    // fl_map_acquire_removed and not sized yet), as the host form grows it before each delete
    if (full && record_removed_) FL_CHECK(removed_room());
    if (layout_changed) { *layout_changed = layout_dirty_ ? 1 : 0; layout_dirty_ = false; }
    return FL_OK;
}

// the host's bound: the call fits when the points of every device-form call since the last settle and n_max more could each take
// one fresh leaf and claim 27 fresh cells with the table below 90 % load -- insert_device's two guards.  The list pool's need
// has no useful bound on the host (up to 27 fresh lists per point); the plan kernel checks it on the device.
bool Map::async_fits(long long n_max) const {
    const long long n = ub_n_ + n_max;
    if (h_counters_[C_LEAF_USED] + n > v_.leaf_cap) return false;
    return !v_.dir.cap || (h_counters_[C_DIR_CELLS] + 27 * n) * 10 <= (long long)v_.dir.cap * 9;
}

// Room for one call of n_max points, by insert_device's rules (a re-pack with a larger overflow pool, a re-list with a larger
// table); after a refused call (pool = true) also a re-list with a larger list pool when the need the plan last computed does
// not fit it.  Synchronous; the map must be settled.
int Map::async_grow(int n_max, bool pool) {
    const long long n = std::max(n_max, 1);
    if (h_counters_[C_LEAF_USED] + n > v_.leaf_cap) {
        min_pool_ = (int)std::min<long long>(std::max<long long>(min_pool_, n + 1024), INT_MAX / 2);
        FL_CHECK(rebuild());
    }
    if (v_.dir.cap) {
        const long long cells = (long long)h_counters_[C_DIR_CELLS] + 27 * n;
        const bool grow_cap = cells * 10 > (long long)v_.dir.cap * 9;
        const long long need = std::max<long long>(h_counters_[C_NEED], 0);
        const bool grow_pool = pool && (long long)h_counters_[C_DIR_POOL] + need > v_.dir.lists_cap;
        if (grow_cap) dir_min_cap_ = std::max(dir_min_cap_, (size_t)cells * 2 + 16384);
        if (grow_pool) dir_min_pool_ = std::max<size_t>(dir_min_pool_ * 2, 2 * (size_t)need);
        if (grow_cap || grow_pool) { n_dir_rebuilds_++; FL_CHECK(build_directory()); }
    }
    FL_CUDA(cudaStreamSynchronize(stream_));
    return publish_counts();
}

// Scratch of a device-form call of n_max points (its own buffers: a host-form call never moves what a graph captured)
int Map::async_scratch(int n_max, bool may_allocate) {
    const size_t n = (size_t)std::max(n_max, 1);
    size_t sort_bytes = 0;
    FL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                            (unsigned*)nullptr, (unsigned*)nullptr, (int)n, 0, 64, stream_));
    struct Want { DeviceBuffer* b; size_t bytes; } want[] = {
        {&a_keys_in_, sizeof(unsigned long long) * n}, {&a_keys_out_, sizeof(unsigned long long) * n}, {&a_vals_in_, sizeof(unsigned) * n},
        {&a_vals_out_, sizeof(unsigned) * n}, {&a_groups_, sizeof(int) * n}, {&a_ins_, sizeof(float4) * n}, {&a_slots_, sizeof(int) * n},
        {&a_fix_, sizeof(unsigned) * 27 * n}, {&a_cub_, sort_bytes}, {&cellcnt_, sizeof(int) * (size_t)v_.dir.cap}};
    bool short_ = false;
    for (const Want& w : want) short_ = short_ || w.b->bytes < w.bytes;
    if (!short_) return FL_OK;
    if (!may_allocate) return FL_ERR_CAPACITY;
    FL_CUDA(cudaStreamSynchronize(stream_));          // nothing in flight may still use a buffer that moves
    for (const Want& w : want) {
        if (w.b->bytes >= w.bytes) continue;
        if (w.b->ptr) layout_dirty_ = true;
        FL_CHECK(w.b->reserve(w.bytes));
        if (w.b == &cellcnt_) FL_CUDA(cudaMemsetAsync(cellcnt_.ptr, 0, cellcnt_.bytes, stream_));
    }
    return FL_OK;
}

int Map::async_prepare(int n_max, cudaStream_t st, const char* what) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    FL_CUDA(cudaStreamGetCaptureInfo(st, &cs));
    const bool capturing = cs != cudaStreamCaptureStatusNone;
    async_used_ = true;
    async_n_max_ = std::max(async_n_max_, n_max);
    if (capturing) {
        if (!async_fits(n_max)) {
            set_last_error("%s: %d points might not fit the map's headroom; call fl_map_maintain (or the call once outside capture) first", what, n_max);
            return FL_ERR_CAPACITY;
        }
        if (async_scratch(n_max, false) != FL_OK) {
            set_last_error("%s: no scratch for %d points yet; make the call once outside capture first", what, n_max);
            return FL_ERR_CAPACITY;
        }
        return FL_OK;
    }
    if (!async_fits(n_max)) {                  // the one synchronous case: settle, and grow when the settled map has no room either
        FL_CHECK(settle(false));
        if (!async_fits(n_max)) FL_CHECK(async_grow(n_max, false));
    }
    return async_scratch(n_max, true);
}

int Map::mutation_begin(cudaStream_t st, bool* joined) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    FL_CUDA(cudaStreamGetCaptureInfo(st, &cs));
    *joined = cs == cudaStreamCaptureStatusNone;
    if (!*joined) { captured_ = true; return FL_OK; }
    // a mutation waits for everything enqueued on the handle so far, device queries joined from other streams included
    FL_CUDA(cudaEventRecord(ev_front_, stream_));
    FL_CUDA(cudaStreamWaitEvent(st, ev_front_, 0));
    return FL_OK;
}
int Map::mutation_end(cudaStream_t st, bool joined) {
    pending_ = true;
    touch();
    return query_end(st, joined);
}

int Map::enqueue_insert(const float4* pts, const int* n_dev, int n_max, cudaStream_t st) {
    const int g = blocks_for((long long)n_max * 32, 256);
    int* d_cnt = counters_.as<int>();
    k_insert<<<g, 256, 0, st>>>(v_, pts, n_max, n_dev, d_cnt, a_slots_.as<int>());
    if (v_.dir.cap) {
        const int fix_cap = (int)std::min<long long>(27ll * n_max, INT_MAX);
        k_halo_claim<<<g, 256, 0, st>>>(v_, pts, a_slots_.as<int>(), n_max, n_dev, d_cnt);
        FL_CUDA(cudaMemsetAsync(&d_cnt[C_NFIX], 0, sizeof(int), st));
        k_halo_append<<<g, 256, 0, st>>>(v_, pts, a_slots_.as<int>(), n_max, n_dev, d_cnt, a_fix_.as<unsigned>(), fix_cap);
        k_halo_fix<<<296, 256, 0, st>>>(v_, a_fix_.as<unsigned>(), fix_cap, d_cnt);
    }
    FL_CUDA(cudaGetLastError());
    return FL_OK;
}

// add_points_host on the device: the batch's count at counters_[slot]
int Map::enqueue_add(const float4* pts, int slot, bool downsample_on, int n_max, cudaStream_t st) {
    int* d_cnt = counters_.as<int>();
    const int chain_limit = std::max(64, (int)(rebuild_overflow_frac_ * v_.n_main));
    if (downsample_on) {
        unsigned long long* ki = a_keys_in_.as<unsigned long long>();
        unsigned long long* ko = a_keys_out_.as<unsigned long long>();
        k_voxel_keys<<<blocks_for(n_max, 256, 1 << 30), 256, 0, st>>>(pts, n_max, downsample_, ki, a_vals_in_.as<unsigned>(), &d_cnt[slot]);
        size_t tmp = a_cub_.bytes;
        FL_CUDA(cub::DeviceRadixSort::SortPairs(a_cub_.ptr, tmp, ki, ko, a_vals_in_.as<unsigned>(), a_vals_out_.as<unsigned>(), n_max, 0, 64, st));
        k_group_heads<<<blocks_for(n_max, 256, 1 << 30), 256, 0, st>>>(ko, n_max, a_groups_.as<int>(), d_cnt, &d_cnt[slot]);
        (det_ ? k_downsample_keyed : k_downsample_resolve)<<<blocks_for((long long)n_max * 32, 256), 256, 0, st>>>(
            v_, pts, ko, a_vals_out_.as<unsigned>(), n_max, a_groups_.as<int>(), downsample_, a_ins_.as<float4>(), d_cnt);
        FL_CHECK(enqueue_insert(a_ins_.as<float4>(), &d_cnt[C_NINSERT], n_max, st));
    } else {
        FL_CHECK(enqueue_insert(pts, &d_cnt[slot], n_max, st));
    }
    k_async_account<<<1, 1, 0, st>>>(v_, d_cnt, slot, downsample_on, chain_limit);
    FL_CUDA(cudaGetLastError());
    return FL_OK;
}

int Map::add_points_async(const float4* pa, const int* na, bool downsample_a, const float4* pb, const int* nb, int n_max,
                          const int* list_counts, int* out, cudaStream_t st) {
    int* d_cnt = counters_.as<int>();
    k_plan_begin<<<1, 1, 0, st>>>(d_cnt, na, nb, n_max);
    if (v_.dir.cap) {
        const int g = blocks_for((long long)n_max * 32, 256);
        const float4* lists[2] = {pa, pb};
        for (int l = 0; l < 2; l++)
            if (lists[l]) k_plan_count<<<g, 256, 0, st>>>(v_, lists[l], n_max, &d_cnt[l ? C_RB : C_RA], d_cnt, cellcnt_.as<int>());
        for (int l = 0; l < 2; l++)
            if (lists[l]) k_plan_reset<<<g, 256, 0, st>>>(v_, lists[l], n_max, &d_cnt[l ? C_RB : C_RA], d_cnt, cellcnt_.as<int>(), pb ? 2 : 1);
    }
    k_plan<<<1, 1, 0, st>>>(v_, d_cnt);
    FL_CHECK(enqueue_add(pa, C_NA, downsample_a, n_max, st));
    if (pb) FL_CHECK(enqueue_add(pb, C_NB, false, n_max, st));
    k_async_status<<<1, 1, 0, st>>>(d_cnt, list_counts, out);
    FL_CUDA(cudaGetLastError());
    ub_n_ += n_max;
    return FL_OK;
}

int Map::add_points_async_checked(const float* d_pts, const int* d_n, int n_max, bool downsample_on, int* d_status2, cudaStream_t st) {
    if (n_max < 0 || !device_ptr(d_n, device_, 4) || !device_ptr(d_status2, device_, 4) || (n_max > 0 && !device_ptr(d_pts, device_, 16))) {
        set_last_error("add_points_async: n_max < 0, or a buffer is not device memory on device %d (points 16-byte, n and status "
                       "4-byte aligned)", device_);
        return FL_ERR_ARG;
    }
    FL_CUDA(cudaSetDevice(device_));
    if (n_max == 0) {                                   // nothing can be inserted: (FL_OK, 0)
        bool joined = false;
        FL_CHECK(query_begin(st, &joined));
        FL_CUDA(cudaMemsetAsync(d_status2, 0, 2 * sizeof(int), st));
        return query_end(st, joined);
    }
    FL_CHECK(async_prepare(n_max, st, "add_points_async"));
    bool joined = false;
    FL_CHECK(mutation_begin(st, &joined));
    FL_CHECK(add_points_async(reinterpret_cast<const float4*>(d_pts), d_n, downsample_on, nullptr, nullptr, n_max, nullptr, d_status2, st));
    return mutation_end(st, joined);
}

int Map::tree_range(float* box6) {
    FL_CUDA(cudaSetDevice(device_));
    // union of the top-level entity boxes
    const int k = v_.n_levels - 1;
    const int c = v_.count[k];
    std::vector<float4> h(2 * (size_t)c);
    FL_CUDA(cudaMemcpyAsync(h.data(), v_.ebox[k], sizeof(float4) * 2 * (size_t)c, cudaMemcpyDeviceToHost, stream_));
    FL_CUDA(cudaStreamSynchronize(stream_));
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = 0; i < c; i++) {
        lo[0] = std::min(lo[0], h[2 * i].x); lo[1] = std::min(lo[1], h[2 * i].y); lo[2] = std::min(lo[2], h[2 * i].z);
        hi[0] = std::max(hi[0], h[2 * i + 1].x); hi[1] = std::max(hi[1], h[2 * i + 1].y); hi[2] = std::max(hi[2], h[2 * i + 1].z);
    }
    if (n_valid_ == 0) for (int a = 0; a < 3; a++) lo[a] = hi[a] = 0.f;        // memset(&range, 0, ...) ikd_Tree.cpp:114
    for (int a = 0; a < 3; a++) { box6[a] = lo[a]; box6[3 + a] = hi[a]; }
    return FL_OK;
}

}  // namespace fl
