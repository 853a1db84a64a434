// Candidate pruning for the sweep: a (y, z) cell grid UNDER the x-sorted order.
//
// The reference's sweep tests every j in the x-window (i, end_i) of interval i.  In 3D-dense scenes that window holds thousands of
// candidates of which a handful overlap in y and z (100k-cube stack: ~1 500 candidates, ~4 hits; 1M spheres: ~5 000 candidates,
// ~2 hits).  The set of pairs and their order are properties of the x-sorted RANKS only, so the search may use any index that finds
// exactly the pairs {i < j < end_i, y/z overlap}:
//   * every interval is binned by the (y, z) cell of its min corner; the cell edge per axis is the largest "small" extent on that axis
//     (extents above 4x the mean are "large"), so a small j that overlaps i lies in the cell range [cell(min_i - edge), cell(max_i)]
//     (with the extents rounded up and min_i - edge rounded down: see query_lo);
//   * one stable radix sort of the ranks by cell id groups the ranks per cell IN RANK ORDER, so the x-window of i is a contiguous
//     sub-range of each cell list (two binary searches);
//   * large intervals share one extra list (cell id 0xFFFF) that every i scans inside its x-window;
//   * hits of one i come out cell by cell, so each i's segment of the pair buffer is sorted by rank j afterwards (segments are a few
//     entries long), then `materialize_pairs` writes the ABI columns.  Count pass -> exclusive scan -> emit pass keep the i order.
// Intervals that are wide in x (more than SW_WIDE candidates) still go through sweep_wide_kernel (brute force over their window).
#pragma once

namespace avn {
namespace {

constexpr int CG_MAX_AXIS = 1024;        // cells per axis
constexpr uint32_t CG_LARGE = 0xFFFFu;   // cell id of the large-interval list
constexpr int CG_MAX_CELLS = 0xFFFF;     // ids 0 .. 0xFFFE
constexpr int CG_GROUP = 16;             // lanes per interval in the cell sweep

template <class S>
struct CellGrid {
    S y0, z0, inv_cy, inv_cz, edge_y, edge_z;   // origin, 1/cell edge, small-extent bound per axis
    int ny, nz;
};

template <class S> __device__ __forceinline__ int cell_coord(S v, S v0, S inv_c, int n) {
    S t = (v - v0) * inv_c;
    int c = t > S(0) ? (t < S(n) ? int(t) : n - 1) : 0;   // clamps; NaN cannot occur (non-finite AABBs never reach the intervals)
    return c;
}

// directed rounding: query_lo(min_i, edge) <= min_i - edge <= max_j - extent_up(j) <= min_j for every small j overlapping i (cell_coord is monotone)
__device__ __forceinline__ float sub_dir(float a, float b, bool up) { return up ? __fsub_ru(a, b) : __fsub_rd(a, b); }
__device__ __forceinline__ double sub_dir(double a, double b, bool up) { return up ? __dsub_ru(a, b) : __dsub_rd(a, b); }
template <class S> __device__ __forceinline__ S extent_up(S lo, S hi) { return sub_dir(hi, lo, true); }     // decides small / large and the edge
template <class S> __device__ __forceinline__ S query_lo(S v, S edge) { return sub_dir(v, edge, false); }

// per-block partial reductions of yz_stats
template <class S>
struct YzPartial { S min_y, max_y, min_z, max_z, max_ey, max_ez; double sum_ey, sum_ez; };
constexpr int YZ_BLOCKS = 296;

// min/max of the min corners, sum and max of the extents: one partial per block ...
template <class S>
__global__ void __launch_bounds__(256) yz_stats(const Vec4<S>* __restrict__ yz, int n, YzPartial<S>* __restrict__ partial) {
    __shared__ YzPartial<S> s_part[8];
    S mny = S(INFINITY), mxy = S(-INFINITY), mnz = S(INFINITY), mxz = S(-INFINITY), mey = 0, mez = 0;
    double sey = 0, sez = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        Vec4<S> v = yz[i];
        S ey = v.y - v.x, ez = v.w - v.z;
        mny = avn_min(mny, v.x); mxy = avn_max(mxy, v.x); mnz = avn_min(mnz, v.z); mxz = avn_max(mxz, v.z);
        mey = avn_max(mey, ey); mez = avn_max(mez, ez);
        sey += double(ey); sez += double(ez);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mny = avn_min(mny, __shfl_xor_sync(0xffffffffu, mny, o)); mxy = avn_max(mxy, __shfl_xor_sync(0xffffffffu, mxy, o));
        mnz = avn_min(mnz, __shfl_xor_sync(0xffffffffu, mnz, o)); mxz = avn_max(mxz, __shfl_xor_sync(0xffffffffu, mxz, o));
        mey = avn_max(mey, __shfl_xor_sync(0xffffffffu, mey, o)); mez = avn_max(mez, __shfl_xor_sync(0xffffffffu, mez, o));
        sey += __shfl_xor_sync(0xffffffffu, sey, o); sez += __shfl_xor_sync(0xffffffffu, sez, o);
    }
    if ((threadIdx.x & 31) == 0) {
        YzPartial<S> p; p.min_y = mny; p.max_y = mxy; p.min_z = mnz; p.max_z = mxz; p.max_ey = mey; p.max_ez = mez; p.sum_ey = sey; p.sum_ez = sez;
        s_part[threadIdx.x >> 5] = p;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        YzPartial<S> p = s_part[0];
        for (int k = 1; k < 8; ++k) {
            const YzPartial<S>& q = s_part[k];
            p.min_y = avn_min(p.min_y, q.min_y); p.max_y = avn_max(p.max_y, q.max_y); p.min_z = avn_min(p.min_z, q.min_z); p.max_z = avn_max(p.max_z, q.max_z);
            p.max_ey = avn_max(p.max_ey, q.max_ey); p.max_ez = avn_max(p.max_ez, q.max_ez); p.sum_ey += q.sum_ey; p.sum_ez += q.sum_ez;
        }
        partial[blockIdx.x] = p;
    }
}
// ... one thread folds the partials (into partial[0]) and derives the "large" thresholds 4 x mean extent (stored in grid->edge_*) ...
template <class S>
__global__ void yz_fold(YzPartial<S>* __restrict__ partial, int nparts, int n, CellGrid<S>* __restrict__ grid) {
    // one warp: lanes stride the partials, then a shuffle reduction
    YzPartial<S> p = partial[threadIdx.x < nparts ? threadIdx.x : 0];
    for (int k = threadIdx.x + 32; k < nparts; k += 32) {
        const YzPartial<S>& q = partial[k];
        p.min_y = avn_min(p.min_y, q.min_y); p.max_y = avn_max(p.max_y, q.max_y); p.min_z = avn_min(p.min_z, q.min_z); p.max_z = avn_max(p.max_z, q.max_z);
        p.max_ey = avn_max(p.max_ey, q.max_ey); p.max_ez = avn_max(p.max_ez, q.max_ez); p.sum_ey += q.sum_ey; p.sum_ez += q.sum_ez;
    }
    if (threadIdx.x >= nparts) { p.sum_ey = 0; p.sum_ez = 0; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        p.min_y = avn_min(p.min_y, __shfl_xor_sync(0xffffffffu, p.min_y, o)); p.max_y = avn_max(p.max_y, __shfl_xor_sync(0xffffffffu, p.max_y, o));
        p.min_z = avn_min(p.min_z, __shfl_xor_sync(0xffffffffu, p.min_z, o)); p.max_z = avn_max(p.max_z, __shfl_xor_sync(0xffffffffu, p.max_z, o));
        p.max_ey = avn_max(p.max_ey, __shfl_xor_sync(0xffffffffu, p.max_ey, o)); p.max_ez = avn_max(p.max_ez, __shfl_xor_sync(0xffffffffu, p.max_ez, o));
        p.sum_ey += __shfl_xor_sync(0xffffffffu, p.sum_ey, o); p.sum_ez += __shfl_xor_sync(0xffffffffu, p.sum_ez, o);
    }
    if (threadIdx.x != 0) return;
    partial[0] = p;
    grid->edge_y = S(4) * S(p.sum_ey / n);
    grid->edge_z = S(4) * S(p.sum_ez / n);
}
// ... a second pass finds the largest extent that is still "small" (<= the threshold) on each axis: that is the cell edge ...
template <class S>
__global__ void __launch_bounds__(256) yz_small_max(const Vec4<S>* __restrict__ yz, int n, const CellGrid<S>* __restrict__ grid, S* __restrict__ out /*[2*gridDim.x]*/) {
    __shared__ S s_y[8], s_z[8];
    const S thr_y = grid->edge_y, thr_z = grid->edge_z;
    S my = 0, mz = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        Vec4<S> v = yz[i];
        S ey = extent_up(v.x, v.y), ez = extent_up(v.z, v.w);
        if (ey <= thr_y) my = avn_max(my, ey);
        if (ez <= thr_z) mz = avn_max(mz, ez);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { my = avn_max(my, __shfl_xor_sync(0xffffffffu, my, o)); mz = avn_max(mz, __shfl_xor_sync(0xffffffffu, mz, o)); }
    if ((threadIdx.x & 31) == 0) { s_y[threadIdx.x >> 5] = my; s_z[threadIdx.x >> 5] = mz; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < 8; ++k) { my = avn_max(my, s_y[k]); mz = avn_max(mz, s_z[k]); }
        out[2 * blockIdx.x] = my; out[2 * blockIdx.x + 1] = mz;
    }
}
// ... and one thread turns everything into the grid parameters
template <class S>
__global__ void yz_grid(const YzPartial<S>* __restrict__ partial, const S* __restrict__ small_max, int nparts, int n, CellGrid<S>* __restrict__ grid) {
    const YzPartial<S> p = partial[0];
    S edge_y = 0, edge_z = 0;
    for (int k = threadIdx.x; k < nparts; k += 32) { edge_y = avn_max(edge_y, small_max[2 * k]); edge_z = avn_max(edge_z, small_max[2 * k + 1]); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { edge_y = avn_max(edge_y, __shfl_xor_sync(0xffffffffu, edge_y, o)); edge_z = avn_max(edge_z, __shfl_xor_sync(0xffffffffu, edge_z, o)); }
    if (threadIdx.x != 0) return;
    // extents above 4 x mean are "large"; when every interval exceeds its axis threshold (impossible for a mean) edge stays 0 = all large
    S range_y = p.max_y - p.min_y, range_z = p.max_z - p.min_z;
    S cy = avn_max(edge_y, range_y / S(CG_MAX_AXIS)), cz = avn_max(edge_z, range_z / S(CG_MAX_AXIS));
    int ny = cy > S(0) ? int(range_y / cy) + 1 : 1, nz = cz > S(0) ? int(range_z / cz) + 1 : 1;
    ny = max(1, min(ny, CG_MAX_AXIS)); nz = max(1, min(nz, CG_MAX_AXIS));
    while ((long long)ny * nz > CG_MAX_CELLS) {   // coarsen the finer axis until the ids fit 16 bits (cells only get larger: still exact)
        if (ny >= nz) { ny = (ny + 1) / 2; cy = cy * S(2); } else { nz = (nz + 1) / 2; cz = cz * S(2); }
    }
    CellGrid<S> g;
    g.y0 = p.min_y; g.z0 = p.min_z; g.inv_cy = cy > S(0) ? S(1) / cy : S(0); g.inv_cz = cz > S(0) ? S(1) / cz : S(0);
    g.edge_y = edge_y; g.edge_z = edge_z; g.ny = ny; g.nz = nz;
    *grid = g;
}

// number of cells in the query range of an interval with y/z bounds yi (the cells a small overlapping j can live in)
template <class S> __device__ __forceinline__ long long query_cell_count(const CellGrid<S>& g, Vec4<S> yi) {
    const int cy_lo = cell_coord(query_lo(yi.x, g.edge_y), g.y0, g.inv_cy, g.ny), cy_hi = cell_coord(yi.y, g.y0, g.inv_cy, g.ny);
    const int cz_lo = cell_coord(query_lo(yi.z, g.edge_z), g.z0, g.inv_cz, g.nz), cz_hi = cell_coord(yi.w, g.z0, g.inv_cz, g.nz);
    return (long long)(cy_hi - cy_lo + 1) * (cz_hi - cz_lo + 1);
}

template <class S>
__global__ void cell_keys(const Vec4<S>* __restrict__ yz, int n, const CellGrid<S>* __restrict__ grid, uint32_t* __restrict__ keys,
                          uint32_t* __restrict__ vals) {
    int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const CellGrid<S> g = *grid;
    Vec4<S> v = yz[r];
    const bool large = extent_up(v.x, v.y) > g.edge_y || extent_up(v.z, v.w) > g.edge_z;   // the same extents as yz_small_max
    keys[r] = large ? CG_LARGE : uint32_t(cell_coord(v.x, g.y0, g.inv_cy, g.ny) * g.nz + cell_coord(v.z, g.z0, g.inv_cz, g.nz));
    vals[r] = uint32_t(r);
}

// [start, end) of every cell in the sorted key array (cells that do not occur keep start = 0x7fffffff > end = 0)
__global__ void cell_bounds(const uint32_t* __restrict__ sorted_keys, int n, int* __restrict__ cstart, int* __restrict__ cend) {
    int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    uint32_t k = sorted_keys[p];
    if (p == 0 || sorted_keys[p - 1] != k) cstart[k] = p;
    if (p == n - 1 || sorted_keys[p + 1] != k) cend[k] = p + 1;
}

// first position in ranks[lo, hi) whose value is > key (upper bound) / >= key (lower bound)
__device__ __forceinline__ int ub_rank(const uint32_t* __restrict__ ranks, int lo, int hi, uint32_t key) {
    while (lo < hi) { int mid = (lo + hi) >> 1; if (ranks[mid] > key) hi = mid; else lo = mid + 1; }
    return lo;
}
__device__ __forceinline__ int lb_rank(const uint32_t* __restrict__ ranks, int lo, int hi, uint32_t key) {
    while (lo < hi) { int mid = (lo + hi) >> 1; if (ranks[mid] >= key) hi = mid; else lo = mid + 1; }
    return lo;
}

template <class S>
struct CellSweep {
    const CellGrid<S>* grid;
    const uint32_t* cranks;   // ranks grouped by cell, ascending inside a cell
    const int* cstart; const int* cend;   // [0x10000]
    uint64_t capacity;        // entries of the pair buffer the emit pass may write (the count pass runs first; a larger total re-runs)
};

// CG_GROUP lanes per interval i.  The lanes stride over the cells of i's query range (+ one lane-strided pass over the large list);
// per cell: the x-window (i, end_i) as a sub-range of the cell's rank list, then the exact tests of broad_phase.rs:394-428.
// EMIT = false: counts[i].  EMIT = true: pairs[offsets[i] ...] = (i, j), unordered inside the segment.
template <class S, bool EMIT>
__global__ void __launch_bounds__(256) sweep_cells_kernel(const __grid_constant__ Sweep<S> s, const __grid_constant__ CellSweep<S> cs,
                                                          uint32_t* __restrict__ counts, const uint64_t* __restrict__ offsets, uint2* __restrict__ pairs) {
    const int lane = threadIdx.x & (CG_GROUP - 1);
    const unsigned gmask = CG_GROUP == 32 ? 0xffffffffu : (((1u << CG_GROUP) - 1u) << ((threadIdx.x & 31) & ~(CG_GROUP - 1)));
    const long long groups = (long long)gridDim.x * (blockDim.x / CG_GROUP);
    const CellGrid<S> g = *cs.grid;
    for (long long i64 = (long long)blockIdx.x * (blockDim.x / CG_GROUP) + threadIdx.x / CG_GROUP; i64 < s.n; i64 += groups) {
        const int i = int(i64);
        if (s.is_wide[i]) continue;   // group-uniform
        if (EMIT && offsets[i + 1] == offsets[i]) continue;   // the count pass found nothing for this interval (the usual case in steady state)
        const int e = s.end[i];
        uint32_t mine = 0;            // hits found by this lane
        uint64_t base = 0;
        Vec4<S> yi; uint4 mi = make_uint4(0, 0, 0, 0); uint32_t fi = 0;
        if (e > i + 1) {
            yi = s.yz[i]; mi = s.meta[i]; fi = s.flags[i];
            if (EMIT) base = offsets[i];
        }
        // two passes when emitting: first count per lane to get lane offsets inside the segment, then write
        for (int pass = 0; pass < (EMIT ? 2 : 1); ++pass) {
            uint32_t wr = 0;
            if (EMIT && pass == 1) {   // exclusive prefix of `mine` over the group's lanes
                uint32_t x = mine;
#pragma unroll
                for (int o = 1; o < CG_GROUP; o <<= 1) {
                    uint32_t y = __shfl_up_sync(gmask, x, o, CG_GROUP);
                    if (lane >= o) x += y;
                }
                wr = x - mine;
            }
            if (e > i + 1) {
                const int cy_lo = cell_coord(query_lo(yi.x, g.edge_y), g.y0, g.inv_cy, g.ny), cy_hi = cell_coord(yi.y, g.y0, g.inv_cy, g.ny);
                const int cz_lo = cell_coord(query_lo(yi.z, g.edge_z), g.z0, g.inv_cz, g.nz), cz_hi = cell_coord(yi.w, g.z0, g.inv_cz, g.nz);
                const int wz = cz_hi - cz_lo + 1, ncell = (cy_hi - cy_lo + 1) * wz;
                if (ncell > e - i - 1) {
                    // more cells than x-candidates (a big footprint with a short window): test the window directly, lane-strided
                    for (int j = i + 1 + lane; j < e; j += CG_GROUP) {
                        const Vec4<S> yj = s.yz[j];
                        if ((yi.x > yj.y || yi.y < yj.x) || (yi.z > yj.w || yi.w < yj.z)) continue;
                        uint32_t pf; uint4 mj;
                        if (!pair_filters(s, mi, fi, j, pf, mj)) continue;
                        if (EMIT && pass == 1 && base + wr < cs.capacity) pairs[base + wr] = make_uint2(uint32_t(i), uint32_t(j));
                        ++wr;
                    }
                } else {
                for (int q = lane; q < ncell; q += CG_GROUP) {
                    const int cell = (cy_lo + q / wz) * g.nz + (cz_lo + q % wz);
                    int lo = cs.cstart[cell], hi = cs.cend[cell];
                    if (lo >= hi) continue;
                    lo = ub_rank(cs.cranks, lo, hi, uint32_t(i));
                    hi = lb_rank(cs.cranks, lo, hi, uint32_t(e));
                    for (int p = lo; p < hi; ++p) {
                        const int j = int(cs.cranks[p]);
                        const Vec4<S> yj = s.yz[j];
                        if ((yi.x > yj.y || yi.y < yj.x) || (yi.z > yj.w || yi.w < yj.z)) continue;
                        uint32_t pf; uint4 mj;
                        if (!pair_filters(s, mi, fi, j, pf, mj)) continue;
                        if (EMIT && pass == 1 && base + wr < cs.capacity) pairs[base + wr] = make_uint2(uint32_t(i), uint32_t(j));
                        ++wr;
                    }
                }
                {   // large intervals: lane-strided over the part of their list inside the x-window
                    int lo = cs.cstart[CG_LARGE], hi = cs.cend[CG_LARGE];
                    if (lo < hi) {
                        lo = ub_rank(cs.cranks, lo, hi, uint32_t(i));
                        hi = lb_rank(cs.cranks, lo, hi, uint32_t(e));
                        for (int p = lo + lane; p < hi; p += CG_GROUP) {
                            const int j = int(cs.cranks[p]);
                            const Vec4<S> yj = s.yz[j];
                            if ((yi.x > yj.y || yi.y < yj.x) || (yi.z > yj.w || yi.w < yj.z)) continue;
                            uint32_t pf; uint4 mj;
                            if (!pair_filters(s, mi, fi, j, pf, mj)) continue;
                            if (EMIT && pass == 1 && base + wr < cs.capacity) pairs[base + wr] = make_uint2(uint32_t(i), uint32_t(j));
                            ++wr;
                        }
                    }
                }
                }
            }
            if (pass == 0) mine = wr;
        }
        if (!EMIT) {
            uint32_t tot = mine;
#pragma unroll
            for (int o = CG_GROUP / 2; o > 0; o >>= 1) tot += __shfl_xor_sync(gmask, tot, o, CG_GROUP);
            if (lane == 0) counts[i] = tot;
        }
    }
}

// sort every non-wide interval's segment of the pair buffer by rank j (insertion sort: segments are a few entries long)
__global__ void segment_sort(const uint64_t* __restrict__ offsets, const uint8_t* __restrict__ is_wide, int n, uint2* __restrict__ pairs, uint64_t capacity) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || is_wide[i]) return;
    const uint64_t b = offsets[i], e = offsets[i + 1];
    if (e > capacity || e - b < 2) return;   // (too small a buffer: the host grows it and runs again) / nothing to sort
    for (uint64_t p = b + 1; p < e; ++p) {
        uint2 v = pairs[p];
        uint64_t q = p;
        while (q > b && pairs[q - 1].y > v.y) { pairs[q] = pairs[q - 1]; --q; }
        pairs[q] = v;
    }
}

// (rank i, rank j) -> the ABI columns of the emitted pair (broad_phase.rs:443-468)
template <class S>
__global__ void materialize_pairs(const __grid_constant__ Sweep<S> s, const uint2* __restrict__ pairs, const uint64_t* __restrict__ total_ptr, uint64_t capacity,
                                  uint32_t* __restrict__ out_c1, uint32_t* __restrict__ out_c2, uint32_t* __restrict__ out_b1,
                                  uint32_t* __restrict__ out_b2, uint8_t* __restrict__ out_flags) {
    const uint64_t total = *total_ptr;   // the count pass's result, still on the device: no host round trip between count and emit
    if (total > capacity) return;
    for (uint64_t p = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; p < total; p += uint64_t(gridDim.x) * blockDim.x) {
    const uint2 ij = pairs[p];
    const uint4 mi = s.meta[ij.x], mj = s.meta[ij.y];
    const uint32_t u = uint32_t(s.flags[ij.x]) | uint32_t(s.flags[ij.y]);
    out_c1[p] = mi.x; out_c2[p] = mj.x; out_b1[p] = mi.y; out_b2[p] = mj.y;
    out_flags[p] = uint8_t(((u & AVN_AABB_CONTACT_EVENTS) ? AVN_PAIR_CONTACT_EVENTS : 0u) | ((u & AVN_AABB_MODIFY_CONTACTS) ? AVN_PAIR_MODIFY_CONTACTS : 0u) |
                           ((u & AVN_AABB_GENERATE_CONSTRAINTS) ? AVN_PAIR_GENERATE_CONSTRAINTS : 0u) | ((u & AVN_AABB_CUSTOM_FILTER) ? AVN_PAIR_NEEDS_HOOK : 0u));
    }
}

}  // namespace
}  // namespace avn
