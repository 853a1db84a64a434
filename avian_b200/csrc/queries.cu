// Spatial queries on the device: the collider tree of SpatialQueryPipeline::update (spatial_query/pipeline.rs:96-133) rebuilt by every
// update as an LBVH, and batched cast_ray / ray_hits / aabb_intersections_with_aabb against it (pipeline.rs:156-216, 690-729).
// The per-shape arithmetic is csrc/query_math.hpp — the same header the host fixture's brute force compiles — evaluated in double and rounded
// to the column scalar on store, so every answer equals the brute force over all colliders bit for bit (tests/test_gpu_query.py).
//
// Update (no host round trip):
//   1. per collider: tight AABB in double; its f32 culling bounds (outward + one ulp, qm::culling_bounds); the centre; the scene bounds of
//      the centres by ordered-integer atomics.  A collider with a non-finite pose or dims or a zero quaternion (qm::collider_valid) gets the
//      key 0xFFFFFFFF and stays out of the tree.
//   2. 30-bit Morton codes of the centres; stable radix sort of (code, index), 4 passes of device_prims.cuh's rs_histogram / rs_scatter.
//   3. Karras' hierarchy over the m finite colliders (m is counted on the device): equal codes split on the index bits, so a node's common
//      prefix length lies in [2, 63] and strictly grows downwards: depth <= 62, which the fixed traversal stack of Q_STACK entries holds.
//   4. bottom-up refit: the second child to arrive at a node merges the two boxes (atom.acq_rel: the first arrival's box store is released
//      by its increment and acquired by the second's, the counter discipline of the wavefront solver, DESIGN.md §3.1).
// Queries: one thread per query, a stack traversal that culls against the f32 bounds (double slab test clipped to [0, max_distance]) and
// runs the exact test at the leaves.  cast_ray keeps the lexicographic minimum (t, collider); ray_hits and aabb_intersections use the broad
// phase's count -> exclusive scan -> emit -> per-segment sort pattern into CSR lists.
// Shape casts (pipeline.rs:335-554) cull against the node boxes grown by the cast shape's AABB half size, nearer child first for the closest
// hit; project_point (570-615) prunes on the squared point-box distance; point and shape intersections (628-683, 744-826) use the same CSR
// pattern.  Their geometry is the shape-cast part of query_math.hpp.
// Move and slide (character_controller/move_and_slide.rs): q_move runs csrc/move_math.hpp's loop per character over this tree (TreeScene).
// Capsules and convex hulls (DESIGN.md §7j, §7l): every kernel that evaluates a collider's or a query's shape is a template over the shape
// level G: 0 = cuboids and spheres, 1 = + capsules, 2 = + convex hulls (csrc/hull_query_math.hpp, over the context's hull table, which the
// tree carries).  The host launches the lowest level that covers the tree (remembered across AVN_QUERY_SHAPES_UNCHANGED updates) and the
// batch; the G = 0 and G = 1 instances compile the code they had before hulls were queried.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

#include "context.hpp"
#include "device_prims.cuh"
#include "hull_query_math.hpp"
#include "query_math.hpp"
#include "move_math.hpp"

namespace avn {
namespace {

constexpr int Q_STACK = 64;
// node prefix lengths: [2, 31] for distinct 30-bit codes, 32 + [1, 31] for equal codes split on index bits -> at most 62 internal levels;
// a pop pushes two children, so the stack holds at most (levels - 1) pending siblings + 2 entries
static_assert(62 - 1 + 2 <= Q_STACK, "LBVH depth bound exceeds the traversal stack");
constexpr uint32_t Q_INVALID_KEY = 0xFFFFFFFFu;
constexpr int Q_THREADS = 128;

struct __align__(16) NodeBox { float4 lo, hi; };   // .w unused

template <class S>
struct Tree {
    int n;                                           // colliders passed to the update
    const int* m;                                    // colliders in the tree (finite ones), on the device
    const uint8_t* shape; const S* dims; const S* pos; const S* rot; const uint32_t* memb;
    const S* tmn; const S* tmx;                      // tight AABBs rounded to S
    const NodeBox* nodes;                            // [2m - 1]: internal nodes [0, m - 1), leaf k at m - 1 + k; root = 0
    const int2* child;                               // [m - 1]
    const uint32_t* leaf;                            // [m] sorted position -> collider
    hm::Table hulls;                                 // the context's hull table (count 0: none); read by the G = 2 instances only
};

template <class S>
struct Rays {
    int n;
    const S* o; const S* d; const S* maxd;
    const uint8_t* solid; const uint32_t* max_hits; const uint32_t* mask; const uint32_t* xoff; const uint32_t* xs;
};

template <class S> __device__ __forceinline__ nm::V3 ld3(const S* p, size_t i) { return {double(p[3 * i]), double(p[3 * i + 1]), double(p[3 * i + 2])}; }
template <class S> __device__ __forceinline__ nm::Q ldq(const S* p, size_t i) {
    return {double(p[4 * i]), double(p[4 * i + 1]), double(p[4 * i + 2]), double(p[4 * i + 3])};
}

// the geometry of shape level G (0: cuboid / sphere, 1: + capsule, 2: + convex hull over the tree's table)
template <int G, class S>
__device__ __forceinline__ void g_aabb(const Tree<S>& t, int shape, nm::V3 he, nm::V3 p, nm::Q q, nm::V3& mn, nm::V3& mx) {
    if constexpr (G == 2) qh::collider_aabb(t.hulls, shape, he, p, q, mn, mx);
    else qm::collider_aabb<G == 1>(shape, he, p, q, mn, mx);
}
template <int G, class S>
__device__ __forceinline__ bool g_ray(const Tree<S>& t, int shape, nm::V3 he, nm::V3 p, nm::Q q, nm::V3 o, nm::V3 d, double maxd, bool solid, double& th, nm::V3& nh) {
    if constexpr (G == 2) return qh::ray_collider(t.hulls, shape, he, p, q, o, d, maxd, solid, th, nh);
    else return qm::ray_collider<G == 1>(shape, he, p, q, o, d, maxd, solid, th, nh);
}
template <int G, class S>
__device__ __forceinline__ nm::V3 g_half_size(const Tree<S>& t, int shape, nm::V3 he, const nm::M3& r) {
    if constexpr (G == 2) return qh::half_size(t.hulls, shape, he, r);
    else return qm::half_size<G == 1>(shape, he, r);
}
template <int G, class S>
__device__ __forceinline__ bool g_cast(const Tree<S>& t, int sa, nm::V3 ha, nm::V3 ca, nm::Q qa, nm::V3 d, double maxd, uint32_t flags, int sb, nm::V3 hb, nm::V3 cb,
                                       nm::Q qb, double& th, int& axis) {
    if constexpr (G == 2) return qh::cast_collider(t.hulls, sa, ha, ca, qa, d, maxd, flags, sb, hb, cb, qb, th, axis);
    else return qm::cast_collider<G == 1>(sa, ha, ca, qa, d, maxd, flags, sb, hb, cb, qb, th, axis);
}
template <int G, class S>
__device__ __forceinline__ void g_cast_output(const Tree<S>& t, int sa, nm::V3 ha, nm::V3 ca, nm::Q qa, nm::V3 d, uint32_t flags, int sb, nm::V3 hb, nm::V3 cb, nm::Q qb,
                                              double th, int axis, qm::ShapeContact& h) {
    if constexpr (G == 2) qh::cast_output(t.hulls, sa, ha, ca, qa, d, flags, sb, hb, cb, qb, th, axis, h);
    else qm::cast_output<G == 1>(sa, ha, ca, qa, d, flags, sb, hb, cb, qb, th, axis, h);
}
template <int G, class S>
__device__ __forceinline__ double g_project(const Tree<S>& t, int shape, nm::V3 he, nm::V3 c, nm::Q q, nm::V3 p, bool solid, nm::V3& proj, bool& inside) {
    if constexpr (G == 2) return qh::project_point(t.hulls, shape, he, c, q, p, solid, proj, inside);
    else return qm::project_point<G == 1>(shape, he, c, q, p, solid, proj, inside);
}
template <int G, class S>
__device__ __forceinline__ bool g_contains(const Tree<S>& t, int shape, nm::V3 he, nm::V3 c, nm::Q q, nm::V3 p) {
    if constexpr (G == 2) return qh::contains_point(t.hulls, shape, he, c, q, p);
    else return qm::contains_point<G == 1>(shape, he, c, q, p);
}
template <int G, class S>
__device__ __forceinline__ bool g_intersect(const Tree<S>& t, int sa, nm::V3 ha, nm::V3 ca, nm::Q qa, int sb, nm::V3 hb, nm::V3 cb, nm::Q qb) {
    if constexpr (G == 2) return qh::shapes_intersect(t.hulls, sa, ha, ca, qa, sb, hb, cb, qb);
    else return qm::shapes_intersect<G == 1>(sa, ha, ca, qa, sb, hb, cb, qb);
}

__device__ __forceinline__ uint32_t f_ord(float f) { const uint32_t u = __float_as_uint(f); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
__device__ __forceinline__ float f_unord(uint32_t u) { return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u); }

__device__ __forceinline__ uint32_t atom_add_acq_rel(uint32_t* p, uint32_t v) {
    uint32_t old;
    asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
    return old;
}

__device__ __forceinline__ float f32_clamped(double x) { return float(fmin(fmax(x, -double(FLT_MAX)), double(FLT_MAX))); }

// 1. per collider: validity, tight AABB (rounded to S), f32 culling box, centre; scene bounds of the centres
template <class S, int G>
__global__ void __launch_bounds__(256) q_prepare(const __grid_constant__ Tree<S> t, S* __restrict__ tmn, S* __restrict__ tmx, NodeBox* __restrict__ cbox,
                                                 float4* __restrict__ centre, uint8_t* __restrict__ valid, int* __restrict__ m, uint32_t* __restrict__ sb) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    bool ok = false;
    float cx = 0, cy = 0, cz = 0;
    if (i < t.n) {
        const nm::V3 he = ld3(t.dims, i), p = ld3(t.pos, i);
        const nm::Q q = ldq(t.rot, i);
        ok = qm::collider_valid(he, p, q);
        if (ok) {
            nm::V3 mn, mx;
            g_aabb<G>(t, t.shape[i], he, p, q, mn, mx);
            tmn[3 * i] = S(mn.x); tmn[3 * i + 1] = S(mn.y); tmn[3 * i + 2] = S(mn.z);
            tmx[3 * i] = S(mx.x); tmx[3 * i + 1] = S(mx.y); tmx[3 * i + 2] = S(mx.z);
            NodeBox b;
            if constexpr (G == 2) {                      // a hull culls against its bounding ball's box (hull_query_math.hpp)
                nm::V3 lo, hi;
                qh::cull_box(t.hulls, t.shape[i], he, p, mn, mx, lo, hi);
                qm::culling_bounds(lo.x, hi.x, b.lo.x, b.hi.x);
                qm::culling_bounds(lo.y, hi.y, b.lo.y, b.hi.y);
                qm::culling_bounds(lo.z, hi.z, b.lo.z, b.hi.z);
            } else {
                qm::culling_bounds(mn.x, mx.x, b.lo.x, b.hi.x);
                qm::culling_bounds(mn.y, mx.y, b.lo.y, b.hi.y);
                qm::culling_bounds(mn.z, mx.z, b.lo.z, b.hi.z);
            }
            b.lo.w = b.hi.w = 0.f;
            cbox[i] = b;
            // the f32 centre only places the collider on the Morton curve: clamped, so a finite pose beyond the f32 range keeps finite
            // scene bounds (its culling box is then infinite, which is conservative)
            cx = f32_clamped((mn.x + mx.x) * 0.5); cy = f32_clamped((mn.y + mx.y) * 0.5); cz = f32_clamped((mn.z + mx.z) * 0.5);
        }
        valid[i] = ok ? 1 : 0;
        centre[i] = make_float4(cx, cy, cz, 0.f);
    }
    const unsigned full = 0xffffffffu;
    const unsigned ballot = __ballot_sync(full, ok);
    const uint32_t mnx = __reduce_min_sync(full, ok ? f_ord(cx) : 0xffffffffu), mny = __reduce_min_sync(full, ok ? f_ord(cy) : 0xffffffffu),
                   mnz = __reduce_min_sync(full, ok ? f_ord(cz) : 0xffffffffu);
    const uint32_t mxx = __reduce_max_sync(full, ok ? f_ord(cx) : 0u), mxy = __reduce_max_sync(full, ok ? f_ord(cy) : 0u),
                   mxz = __reduce_max_sync(full, ok ? f_ord(cz) : 0u);
    if ((threadIdx.x & 31) == 0 && ballot) {
        atomicAdd(m, __popc(ballot));
        atomicMin(&sb[0], mnx); atomicMin(&sb[1], mny); atomicMin(&sb[2], mnz);
        atomicMax(&sb[3], mxx); atomicMax(&sb[4], mxy); atomicMax(&sb[5], mxz);
    }
}

__device__ __forceinline__ uint32_t expand10(uint32_t v) {
    v &= 0x3ffu;
    v = (v * 0x00010001u) & 0xFF0000FFu;
    v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u;
    v = (v * 0x00000005u) & 0x49249249u;
    return v;
}
__device__ __forceinline__ uint32_t grid10(float c, float lo, float hi) {
    const float ext = hi - lo;
    const float u = ext > 0.f ? (c - lo) / ext : 0.f;
    return uint32_t(fminf(fmaxf(u * 1024.f, 0.f), 1023.f));
}

// 2. Morton keys (finite colliders) or the key that sorts last (the rest)
__global__ void q_codes(int n, const float4* __restrict__ centre, const uint8_t* __restrict__ valid, const uint32_t* __restrict__ sb,
                        uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    vals[i] = uint32_t(i);
    if (!valid[i]) { keys[i] = Q_INVALID_KEY; return; }
    const float4 c = centre[i];
    const uint32_t x = grid10(c.x, f_unord(sb[0]), f_unord(sb[3])), y = grid10(c.y, f_unord(sb[1]), f_unord(sb[4])),
                   z = grid10(c.z, f_unord(sb[2]), f_unord(sb[5]));
    keys[i] = (expand10(x) << 2) | (expand10(y) << 1) | expand10(z);
}

// 3. Karras (2012) hierarchy: internal node i covers a key range; equal keys compare on their index bits (32 + clz)
__device__ __forceinline__ int q_delta(const uint32_t* keys, int m, int i, long long j) {
    if (j < 0 || j >= m) return -1;
    const uint32_t a = keys[i], b = keys[j];
    return a == b ? 32 + __clz(uint32_t(i) ^ uint32_t(j)) : __clz(a ^ b);
}
__global__ void q_karras(const int* __restrict__ m_ptr, int n, const uint32_t* __restrict__ keys, int2* __restrict__ child, int* __restrict__ parent) {
    const int m = *m_ptr;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) parent[0] = -1;
    if (i >= m - 1 || i >= n) return;
    const int d = q_delta(keys, m, i, i + 1) > q_delta(keys, m, i, i - 1) ? 1 : -1;
    const int dmin = q_delta(keys, m, i, (long long)i - d);
    long long lmax = 2;
    while (q_delta(keys, m, i, i + lmax * d) > dmin) lmax *= 2;
    long long l = 0;
    for (long long s = lmax / 2; s >= 1; s /= 2)
        if (q_delta(keys, m, i, i + (l + s) * d) > dmin) l += s;
    const long long j = i + l * d;
    const int dnode = q_delta(keys, m, i, j);
    long long s = 0;
    for (long long w = (l + 1) / 2;; w = (w + 1) / 2) {
        if (q_delta(keys, m, i, i + (s + w) * d) > dnode) s += w;
        if (w == 1) break;
    }
    const int gamma = int(i + s * d + (d < 0 ? -1 : 0));
    const int lo = int(i < j ? i : j), hi = int(i < j ? j : i);
    const int left = lo == gamma ? (m - 1) + gamma : gamma;
    const int right = hi == gamma + 1 ? (m - 1) + gamma + 1 : gamma + 1;
    child[i] = make_int2(left, right);
    parent[left] = i;
    parent[right] = i;
}

// 4. leaves and bottom-up refit: the second child to arrive at a node merges
__global__ void q_refit(const int* __restrict__ m_ptr, const uint32_t* __restrict__ leaf, const NodeBox* __restrict__ cbox, const int* __restrict__ parent,
                        const int2* __restrict__ child, uint32_t* __restrict__ arrived, NodeBox* nodes) {
    const int m = *m_ptr;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= m) return;
    int node = (m - 1) + k;
    NodeBox b = cbox[leaf[k]];
    nodes[node] = b;
    for (;;) {
        const int p = parent[node];
        if (p < 0) return;
        if (atom_add_acq_rel(&arrived[p], 1u) == 0) return;   // first arrival: its box is published by this increment
        const int2 c = child[p];
        const NodeBox o = nodes[c.x == node ? c.y : c.x];       // the sibling's box, released by the other arrival
        b.lo = make_float4(fminf(b.lo.x, o.lo.x), fminf(b.lo.y, o.lo.y), fminf(b.lo.z, o.lo.z), 0.f);
        b.hi = make_float4(fmaxf(b.hi.x, o.hi.x), fmaxf(b.hi.y, o.hi.y), fmaxf(b.hi.z, o.hi.z), 0.f);
        nodes[p] = b;
        node = p;
    }
}

// stack traversal: visit(box) decides whether to descend, leaf(collider) runs the exact test
template <class S, class Visit, class Leaf>
__device__ __forceinline__ void traverse(const Tree<S>& t, int m, Visit visit, Leaf leaf) {
    if (m <= 0) return;
    int stack[Q_STACK];
    int sp = 0;
    stack[sp++] = 0;
    while (sp > 0) {
        const int nd = stack[--sp];
        const NodeBox b = t.nodes[nd];
        if (!visit(b)) continue;
        if (nd >= m - 1) {
            leaf(t.leaf[nd - (m - 1)]);
        } else {
            const int2 c = t.child[nd];
            stack[sp++] = c.y;
            stack[sp++] = c.x;
        }
    }
}

template <class S>
struct RayIn {
    nm::V3 o, d;
    double maxd;
    bool solid, ok;
    uint32_t mask;
    const uint32_t* xs;
    uint32_t nx;
};
template <class S>
__device__ __forceinline__ RayIn<S> load_ray(const Rays<S>& r, int i) {
    RayIn<S> q;
    q.o = ld3(r.o, i);
    q.d = ld3(r.d, i);
    q.maxd = double(r.maxd[i]);
    q.solid = r.solid ? r.solid[i] != 0 : true;
    q.mask = r.mask ? r.mask[i] : 0xffffffffu;
    q.xs = r.xoff ? r.xs + r.xoff[i] : nullptr;
    q.nx = r.xoff ? r.xoff[i + 1] - r.xoff[i] : 0u;
    q.ok = qm::ray_finite(q.o, q.d, q.maxd);
    return q;
}
template <int G, class S>
__device__ __forceinline__ bool ray_leaf(const Tree<S>& t, const RayIn<S>& q, uint32_t c, double& th, nm::V3& nh) {
    const uint32_t memb = t.memb ? t.memb[c] : 1u;
    if (!qm::passes_filter(memb, q.mask, q.xs, q.nx, c)) return false;
    return g_ray<G>(t, t.shape[c], ld3(t.dims, c), ld3(t.pos, c), ldq(t.rot, c), q.o, q.d, q.maxd, q.solid, th, nh);
}
__device__ __forceinline__ bool ray_visit(const NodeBox& b, nm::V3 o, nm::V3 d, double tclip) {
    return qm::ray_box_entry(&b.lo.x, &b.hi.x, o, d, tclip) != INFINITY;
}

// closest-hit traversal: a node's two children are tested when the node is popped, against the ray clipped to the best hit so far; a leaf
// child runs the exact test at once, internal children go on the stack nearer-entry last, so the nearer subtree is searched first and the
// best distance shrinks early.  The answer does not depend on this order (lexicographic minimum of (t, collider)).
template <class S, class Leaf>
__device__ __forceinline__ void traverse_closest(const Tree<S>& t, int m, nm::V3 o, nm::V3 d, double maxd, const double& best_t, Leaf leaf) {
    if (m <= 0) return;
    if (qm::ray_box_entry(&t.nodes[0].lo.x, &t.nodes[0].hi.x, o, d, maxd) == INFINITY) return;
    if (m == 1) { leaf(t.leaf[0]); return; }
    int stack[Q_STACK];
    int sp = 0;
    stack[sp++] = 0;
    while (sp > 0) {
        const int2 c = t.child[stack[--sp]];
        const double clip = nm::smin(maxd, best_t);
        const NodeBox ba = t.nodes[c.x], bb = t.nodes[c.y];
        const double ta = qm::ray_box_entry(&ba.lo.x, &ba.hi.x, o, d, clip), tb = qm::ray_box_entry(&bb.lo.x, &bb.hi.x, o, d, clip);
        const bool b_first = tb < ta;
        const int near = b_first ? c.y : c.x, far = b_first ? c.x : c.y;
        const double tn = b_first ? tb : ta, tf = b_first ? ta : tb;
        if (tn == INFINITY) continue;
        if (near >= m - 1) leaf(t.leaf[near - (m - 1)]);
        // the far child: a leaf is tested now (against the clip the near leaf may just have tightened), an internal node waits
        if (tf != INFINITY && tf <= best_t) {
            if (far >= m - 1) leaf(t.leaf[far - (m - 1)]);
            else stack[sp++] = far;
        }
        if (near < m - 1) stack[sp++] = near;
    }
}

template <class S, int G>
__global__ void __launch_bounds__(Q_THREADS) q_cast_ray(const __grid_constant__ Tree<S> t, const __grid_constant__ Rays<S> r, int32_t* __restrict__ out_c,
                                                         S* __restrict__ out_t, S* __restrict__ out_n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= r.n) return;
    const RayIn<S> q = load_ray(r, i);
    double best_t = INFINITY;
    uint32_t best_c = 0xffffffffu;
    nm::V3 best_n{0, 0, 0};
    if (q.ok)
        traverse_closest(t, *t.m, q.o, q.d, q.maxd, best_t, [&](uint32_t c) {
            double th;
            nm::V3 nh;
            if (ray_leaf<G>(t, q, c, th, nh) && qm::hit_before(th, c, best_t, best_c)) { best_t = th; best_c = c; best_n = nh; }
        });
    const bool hit = best_c != 0xffffffffu;
    out_c[i] = hit ? int32_t(best_c) : -1;
    out_t[i] = hit ? S(best_t) : S(0);
    out_n[3 * i] = S(best_n.x); out_n[3 * i + 1] = S(best_n.y); out_n[3 * i + 2] = S(best_n.z);
}

// ray_hits count pass: every hit, and the part of it the ray keeps (max_hits)
template <class S, int G>
__global__ void __launch_bounds__(Q_THREADS) q_ray_count(const __grid_constant__ Tree<S> t, const __grid_constant__ Rays<S> r, uint32_t* __restrict__ full,
                                                          uint32_t* __restrict__ kept) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= r.n) return;
    const RayIn<S> q = load_ray(r, i);
    uint32_t cnt = 0;
    if (q.ok)
        traverse(t, *t.m, [&](const NodeBox& b) { return ray_visit(b, q.o, q.d, q.maxd); },
                 [&](uint32_t c) { double th; nm::V3 nh; if (ray_leaf<G>(t, q, c, th, nh)) ++cnt; });
    full[i] = cnt;
    const uint32_t mh = r.max_hits ? r.max_hits[i] : 0xffffffffu;
    kept[i] = cnt < mh ? cnt : mh;
}

// in-place sort of one segment: insertion sort when short, heap sort otherwise (the keys of a segment are distinct)
template <class Less, class Swap>
__device__ void sort_segment(uint32_t n, Less less, Swap swp) {
    if (n < 2) return;
    if (n <= 16) {
        for (uint32_t i = 1; i < n; ++i)
            for (uint32_t j = i; j > 0 && less(j, j - 1); --j) swp(j, j - 1);
        return;
    }
    auto sift = [&](uint32_t root, uint32_t end) {
        for (;;) {
            uint32_t c = 2 * root + 1;
            if (c >= end) return;
            if (c + 1 < end && less(c, c + 1)) ++c;
            if (!less(root, c)) return;
            swp(root, c);
            root = c;
        }
    };
    for (uint32_t s = n / 2; s-- > 0;) sift(s, n);
    for (uint32_t e = n - 1; e > 0; --e) { swp(0, e); sift(0, e); }
}

// ray_hits emit pass: all hits into the scratch segment, sorted by (t, collider), the first `kept` written out with their normals
template <class S, int G>
__global__ void __launch_bounds__(Q_THREADS) q_ray_emit(const __grid_constant__ Tree<S> t, const __grid_constant__ Rays<S> r, const uint64_t* __restrict__ full_off,
                                                         const uint64_t* __restrict__ kept_off, double* __restrict__ tmp_t, uint32_t* __restrict__ tmp_c,
                                                         uint32_t* __restrict__ out_c, S* __restrict__ out_t, S* __restrict__ out_n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= r.n) return;
    const RayIn<S> q = load_ray(r, i);
    if (!q.ok) return;
    const uint64_t base = full_off[i];
    const uint32_t n = uint32_t(full_off[i + 1] - base), keep = uint32_t(kept_off[i + 1] - kept_off[i]);
    if (keep == 0) return;
    double* ts = tmp_t + base;
    uint32_t* cs = tmp_c + base;
    uint32_t w = 0;
    traverse(t, *t.m, [&](const NodeBox& b) { return ray_visit(b, q.o, q.d, q.maxd); },
             [&](uint32_t c) {
                 double th;
                 nm::V3 nh;
                 if (ray_leaf<G>(t, q, c, th, nh) && w < n) { ts[w] = th; cs[w] = c; ++w; }
             });
    sort_segment(
        w, [&](uint32_t a, uint32_t b) { return qm::hit_before(ts[a], cs[a], ts[b], cs[b]); },
        [&](uint32_t a, uint32_t b) { const double x = ts[a]; ts[a] = ts[b]; ts[b] = x; const uint32_t y = cs[a]; cs[a] = cs[b]; cs[b] = y; });
    const uint64_t o = kept_off[i];
    for (uint32_t k = 0; k < keep && k < w; ++k) {
        const uint32_t c = cs[k];
        double th;
        nm::V3 nh{0, 0, 0};
        ray_leaf<G>(t, q, c, th, nh);    // the same exact test again: the normal of this hit
        out_c[o + k] = c;
        if (out_t) out_t[o + k] = S(ts[k]);
        if (out_n) { out_n[3 * (o + k)] = S(nh.x); out_n[3 * (o + k) + 1] = S(nh.y); out_n[3 * (o + k) + 2] = S(nh.z); }
    }
}

// aabb_intersections: count, then emit + sort ascending by collider
template <class S, bool EMIT>
__global__ void __launch_bounds__(Q_THREADS) q_aabb(const __grid_constant__ Tree<S> t, int n, const S* __restrict__ qmn, const S* __restrict__ qmx,
                                                     uint32_t* __restrict__ counts, const uint64_t* __restrict__ off, uint32_t* __restrict__ out_c) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const S a[3] = {qmn[3 * i], qmn[3 * i + 1], qmn[3 * i + 2]}, b[3] = {qmx[3 * i], qmx[3 * i + 1], qmx[3 * i + 2]};
    const double ad[3] = {double(a[0]), double(a[1]), double(a[2])}, bd[3] = {double(b[0]), double(b[1]), double(b[2])};
    uint32_t w = 0;
    uint32_t* seg = EMIT ? out_c + off[i] : nullptr;
    traverse(t, *t.m,
             [&](const NodeBox& nb) {
                 const double lo[3] = {nb.lo.x, nb.lo.y, nb.lo.z}, hi[3] = {nb.hi.x, nb.hi.y, nb.hi.z};
                 return qm::aabb_overlap(ad, bd, lo, hi);
             },
             [&](uint32_t c) {
                 if (!qm::aabb_overlap(a, b, t.tmn + 3 * size_t(c), t.tmx + 3 * size_t(c))) return;
                 if (EMIT) seg[w] = c;
                 ++w;
             });
    if (!EMIT) { counts[i] = w; return; }
    sort_segment(w, [&](uint32_t x, uint32_t y) { return seg[x] < seg[y]; }, [&](uint32_t x, uint32_t y) { const uint32_t v = seg[x]; seg[x] = seg[y]; seg[y] = v; });
}

// ---- shape casts, point projection, point and shape intersections ----------------------------------------------------------------------
template <class S>
struct Shapes {
    int n;
    const uint8_t* shape; const S* dims; const S* pos; const S* rot; const S* d; const S* maxd;
    const uint32_t* flags; const uint32_t* max_hits; const uint32_t* mask; const uint32_t* xoff; const uint32_t* xs;
};
template <class S>
struct Points {
    int n;
    const S* p; const uint8_t* solid; const uint32_t* mask; const uint32_t* xoff; const uint32_t* xs;
};

// one query shape.  ext: the f32 half size of its tight AABB, rounded up plus one ulp (qm::culling_bounds of [-e, e]); lo / hi: its culling box
struct ShapeIn {
    int shape;
    nm::V3 he, c, d;
    nm::Q q;
    double maxd;
    uint32_t flags, mask, nx;
    const uint32_t* xs;
    float ext[3], lo[3], hi[3];
    bool ok;
};
template <int G, class S>
__device__ __forceinline__ ShapeIn load_shape(const Tree<S>& t, const Shapes<S>& s, int i, bool cast) {
    ShapeIn q;
    q.shape = s.shape[i];
    q.he = ld3(s.dims, i);
    q.c = ld3(s.pos, i);
    q.q = ldq(s.rot, i);
    q.d = cast ? ld3(s.d, i) : nm::V3{0, 0, 0};
    q.maxd = cast ? double(s.maxd[i]) : 0.0;
    q.flags = cast && s.flags ? s.flags[i] : 0u;
    q.mask = s.mask ? s.mask[i] : 0xffffffffu;
    q.xs = s.xoff ? s.xs + s.xoff[i] : nullptr;
    q.nx = s.xoff ? s.xoff[i + 1] - s.xoff[i] : 0u;
    q.ok = cast ? qm::cast_finite(q.he, q.c, q.q, q.d, q.maxd) : qm::collider_valid(q.he, q.c, q.q);
    if (q.ok) {
        const nm::V3 e = g_half_size<G>(t, q.shape, q.he, qm::rot_mat(q.q));
        for (int k = 0; k < 3; ++k) {
            float l, h;
            qm::culling_bounds(-nm::comp(e, k), nm::comp(e, k), l, h);
            q.ext[k] = h;
            qm::culling_bounds(nm::comp(q.c, k) - nm::comp(e, k), nm::comp(q.c, k) + nm::comp(e, k), q.lo[k], q.hi[k]);
        }
    }
    return q;
}

// where the cast shape's centre enters a node box grown by the shape's half size, clipped to [0, tmax]; INFINITY when it never does.
// The swept shape can touch a collider in the node only while its AABB overlaps the node box, i.e. while its centre is in the grown box.
__device__ __forceinline__ double grown_entry(const NodeBox& b, const float* ext, nm::V3 o, nm::V3 d, double tmax) {
    const float lo[3] = {b.lo.x, b.lo.y, b.lo.z}, hi[3] = {b.hi.x, b.hi.y, b.hi.z};
    double t0 = 0, t1 = tmax;
    for (int k = 0; k < 3; ++k) {
        const double ok = nm::comp(o, k), dk = nm::comp(d, k), l = double(lo[k]) - double(ext[k]), h = double(hi[k]) + double(ext[k]);
        if (dk == 0) {
            if (ok < l || ok > h) return INFINITY;
            continue;
        }
        double a = (l - ok) / dk, c = (h - ok) / dk;
        if (a > c) { const double s = a; a = c; c = s; }
        t0 = nm::smax(t0, a);
        t1 = nm::smin(t1, c);
    }
    return t0 <= t1 ? t0 : INFINITY;
}

// nearest-first traversal with a shrinking bound: key(box) orders and culls (a node is searched while key <= bound; with CULL_INF a key of
// INFINITY also culls), leaf(collider) runs the exact test and may lower bound.  The nearer child is searched first; the answer does not
// depend on the order (the leaf keeps a lexicographic minimum).
template <bool CULL_INF, class S, class Key, class Leaf>
__device__ __forceinline__ void traverse_nearest(const Tree<S>& t, int m, const double& bound, Key key, Leaf leaf) {
    auto pass = [&](double k) { return (!CULL_INF || k != INFINITY) && k <= bound; };
    if (m <= 0 || !pass(key(t.nodes[0]))) return;
    if (m == 1) { leaf(t.leaf[0]); return; }
    int stack[Q_STACK];
    int sp = 0;
    stack[sp++] = 0;
    while (sp > 0) {
        const int2 c = t.child[stack[--sp]];
        const double ka = key(t.nodes[c.x]), kb = key(t.nodes[c.y]);
        const bool b_first = kb < ka;
        const int near = b_first ? c.y : c.x, far = b_first ? c.x : c.y;
        const double kn = b_first ? kb : ka, kf = b_first ? ka : kb;
        if (!pass(kn)) continue;
        if (near >= m - 1) leaf(t.leaf[near - (m - 1)]);
        if (pass(kf)) {
            if (far >= m - 1) leaf(t.leaf[far - (m - 1)]);
            else stack[sp++] = far;
        }
        if (near < m - 1) stack[sp++] = near;
    }
}

template <int G, class S>
__device__ __forceinline__ bool cast_leaf(const Tree<S>& t, const ShapeIn& q, uint32_t c, double& th, int& axis) {
    const uint32_t memb = t.memb ? t.memb[c] : 1u;
    if (!qm::passes_filter(memb, q.mask, q.xs, q.nx, c)) return false;
    return g_cast<G>(t, q.shape, q.he, q.c, q.q, q.d, q.maxd, q.flags, t.shape[c], ld3(t.dims, c), ld3(t.pos, c), ldq(t.rot, c), th, axis);
}
template <int G, class S>
__device__ __forceinline__ void cast_store(const Tree<S>& t, const ShapeIn& q, uint32_t c, double th, int axis, size_t o, S* p1, S* p2, S* n1, S* n2) {
    qm::ShapeContact h;
    g_cast_output<G>(t, q.shape, q.he, q.c, q.q, q.d, q.flags, t.shape[c], ld3(t.dims, c), ld3(t.pos, c), ldq(t.rot, c), th, axis, h);
    const nm::V3 v[4] = {h.p1, h.p2, h.n1, h.n2};
    S* dst[4] = {p1, p2, n1, n2};
    for (int k = 0; k < 4; ++k)
        if (dst[k]) { dst[k][3 * o] = S(v[k].x); dst[k][3 * o + 1] = S(v[k].y); dst[k][3 * o + 2] = S(v[k].z); }
}
__device__ __forceinline__ bool cast_visit(const NodeBox& b, const ShapeIn& q) { return grown_entry(b, q.ext, q.c, q.d, q.maxd) != INFINITY; }

// cast_shape: the lexicographic minimum of (t, collider)
template <class S, int G>
__global__ void __launch_bounds__(Q_THREADS) q_cast_shape(const __grid_constant__ Tree<S> t, const __grid_constant__ Shapes<S> s, int32_t* __restrict__ out_c,
                                                           S* __restrict__ out_t, S* __restrict__ p1, S* __restrict__ p2, S* __restrict__ n1, S* __restrict__ n2) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= s.n) return;
    const ShapeIn q = load_shape<G>(t, s, i, true);
    double best_t = INFINITY;
    uint32_t best_c = 0xffffffffu;
    int best_axis = -1;
    if (q.ok)
        traverse_nearest<true>(t, *t.m, best_t, [&](const NodeBox& b) { return grown_entry(b, q.ext, q.c, q.d, q.maxd); },
                               [&](uint32_t c) {
                                   double th;
                                   int ax;
                                   if (cast_leaf<G>(t, q, c, th, ax) && qm::hit_before(th, c, best_t, best_c)) { best_t = th; best_c = c; best_axis = ax; }
                               });
    const bool hit = best_c != 0xffffffffu;
    out_c[i] = hit ? int32_t(best_c) : -1;
    out_t[i] = hit ? S(best_t) : S(0);
    if (hit) {
        cast_store<G>(t, q, best_c, best_t, best_axis, size_t(i), p1, p2, n1, n2);
    } else {
        for (int k = 0; k < 3; ++k) p1[3 * i + k] = p2[3 * i + k] = n1[3 * i + k] = n2[3 * i + k] = S(0);
    }
}

// shape_hits count pass: every hit, and the part of it the query keeps (max_hits)
template <class S, int G>
__global__ void __launch_bounds__(Q_THREADS) q_shape_count(const __grid_constant__ Tree<S> t, const __grid_constant__ Shapes<S> s, uint32_t* __restrict__ full,
                                                            uint32_t* __restrict__ kept) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= s.n) return;
    const ShapeIn q = load_shape<G>(t, s, i, true);
    uint32_t cnt = 0;
    if (q.ok)
        traverse(t, *t.m, [&](const NodeBox& b) { return cast_visit(b, q); },
                 [&](uint32_t c) { double th; int ax; if (cast_leaf<G>(t, q, c, th, ax)) ++cnt; });
    full[i] = cnt;
    const uint32_t mh = s.max_hits ? s.max_hits[i] : 0xffffffffu;
    kept[i] = cnt < mh ? cnt : mh;
}

// shape_hits emit pass: all hits into the scratch segment, sorted by (t, collider), the first `kept` written out with their contacts
template <class S, int G>
__global__ void __launch_bounds__(Q_THREADS) q_shape_emit(const __grid_constant__ Tree<S> t, const __grid_constant__ Shapes<S> s, const uint64_t* __restrict__ full_off,
                                                           const uint64_t* __restrict__ kept_off, double* __restrict__ tmp_t, uint32_t* __restrict__ tmp_c,
                                                           uint32_t* __restrict__ out_c, S* __restrict__ out_t, S* __restrict__ p1, S* __restrict__ p2,
                                                           S* __restrict__ n1, S* __restrict__ n2) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= s.n) return;
    const ShapeIn q = load_shape<G>(t, s, i, true);
    if (!q.ok) return;
    const uint64_t base = full_off[i];
    const uint32_t n = uint32_t(full_off[i + 1] - base), keep = uint32_t(kept_off[i + 1] - kept_off[i]);
    if (keep == 0) return;
    double* ts = tmp_t + base;
    uint32_t* cs = tmp_c + base;
    uint32_t w = 0;
    traverse(t, *t.m, [&](const NodeBox& b) { return cast_visit(b, q); },
             [&](uint32_t c) {
                 double th;
                 int ax;
                 if (cast_leaf<G>(t, q, c, th, ax) && w < n) { ts[w] = th; cs[w] = c; ++w; }
             });
    sort_segment(
        w, [&](uint32_t a, uint32_t b) { return qm::hit_before(ts[a], cs[a], ts[b], cs[b]); },
        [&](uint32_t a, uint32_t b) { const double x = ts[a]; ts[a] = ts[b]; ts[b] = x; const uint32_t y = cs[a]; cs[a] = cs[b]; cs[b] = y; });
    const uint64_t o = kept_off[i];
    for (uint32_t k = 0; k < keep && k < w; ++k) {
        const uint32_t c = cs[k];
        double th = 0;
        int ax = -1;
        cast_leaf<G>(t, q, c, th, ax);    // the same exact test again: the axis of this hit
        out_c[o + k] = c;
        if (out_t) out_t[o + k] = S(ts[k]);
        cast_store<G>(t, q, c, ts[k], ax, size_t(o + k), p1, p2, n1, n2);
    }
}

// project_point: the lexicographic minimum of (distance, collider); a node is pruned when its squared distance exceeds the best so far
template <class S, int G>
__global__ void __launch_bounds__(Q_THREADS) q_project_point(const __grid_constant__ Tree<S> t, const __grid_constant__ Points<S> pts, int32_t* __restrict__ out_c,
                                                              S* __restrict__ out_p, uint8_t* __restrict__ out_in) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pts.n) return;
    const nm::V3 p = ld3(pts.p, i);
    const bool solid = pts.solid ? pts.solid[i] != 0 : true;
    const uint32_t mask = pts.mask ? pts.mask[i] : 0xffffffffu;
    const uint32_t* xs = pts.xoff ? pts.xs + pts.xoff[i] : nullptr;
    const uint32_t nx = pts.xoff ? pts.xoff[i + 1] - pts.xoff[i] : 0u;
    double best_d = INFINITY, bound = INFINITY;
    uint32_t best_c = 0xffffffffu;
    nm::V3 best_p{0, 0, 0};
    bool best_in = false;
    if (qm::finite3(p))
        traverse_nearest<false>(t, *t.m, bound, [&](const NodeBox& b) { return qm::point_box_d2(&b.lo.x, &b.hi.x, p); },
                                [&](uint32_t c) {
                                    const uint32_t memb = t.memb ? t.memb[c] : 1u;
                                    if (!qm::passes_filter(memb, mask, xs, nx, c)) return;
                                    nm::V3 pr;
                                    bool in;
                                    const double dd = g_project<G>(t, t.shape[c], ld3(t.dims, c), ld3(t.pos, c), ldq(t.rot, c), p, solid, pr, in);
                                    if (qm::hit_before(dd, c, best_d, best_c)) { best_d = dd; best_c = c; best_p = pr; best_in = in; bound = dd * dd; }
                                });
    const bool hit = best_c != 0xffffffffu;
    out_c[i] = hit ? int32_t(best_c) : -1;
    out_p[3 * i] = S(best_p.x); out_p[3 * i + 1] = S(best_p.y); out_p[3 * i + 2] = S(best_p.z);
    out_in[i] = hit && best_in ? 1 : 0;
}

// point_intersections: count, then emit + sort ascending by collider
template <class S, bool EMIT, int G>
__global__ void __launch_bounds__(Q_THREADS) q_point_isect(const __grid_constant__ Tree<S> t, const __grid_constant__ Points<S> pts, uint32_t* __restrict__ counts,
                                                            const uint64_t* __restrict__ off, uint32_t* __restrict__ out_c) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pts.n) return;
    const nm::V3 p = ld3(pts.p, i);
    const uint32_t mask = pts.mask ? pts.mask[i] : 0xffffffffu;
    const uint32_t* xs = pts.xoff ? pts.xs + pts.xoff[i] : nullptr;
    const uint32_t nx = pts.xoff ? pts.xoff[i + 1] - pts.xoff[i] : 0u;
    uint32_t w = 0;
    uint32_t* seg = EMIT ? out_c + off[i] : nullptr;
    if (qm::finite3(p))
        traverse(t, *t.m, [&](const NodeBox& b) { return qm::point_box_d2(&b.lo.x, &b.hi.x, p) == 0; },
                 [&](uint32_t c) {
                     const uint32_t memb = t.memb ? t.memb[c] : 1u;
                     if (!qm::passes_filter(memb, mask, xs, nx, c)) return;
                     if (!g_contains<G>(t, t.shape[c], ld3(t.dims, c), ld3(t.pos, c), ldq(t.rot, c), p)) return;
                     if (EMIT) seg[w] = c;
                     ++w;
                 });
    if (!EMIT) { counts[i] = w; return; }
    sort_segment(w, [&](uint32_t x, uint32_t y) { return seg[x] < seg[y]; }, [&](uint32_t x, uint32_t y) { const uint32_t v = seg[x]; seg[x] = seg[y]; seg[y] = v; });
}

// shape_intersections: count, then emit + sort ascending by collider
template <class S, bool EMIT, int G>
__global__ void __launch_bounds__(Q_THREADS) q_shape_isect(const __grid_constant__ Tree<S> t, const __grid_constant__ Shapes<S> s, uint32_t* __restrict__ counts,
                                                            const uint64_t* __restrict__ off, uint32_t* __restrict__ out_c) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= s.n) return;
    const ShapeIn q = load_shape<G>(t, s, i, false);
    uint32_t w = 0;
    uint32_t* seg = EMIT ? out_c + off[i] : nullptr;
    if (q.ok)
        traverse(t, *t.m,
                 [&](const NodeBox& b) { return qm::aabb_overlap(q.lo, q.hi, &b.lo.x, &b.hi.x); },
                 [&](uint32_t c) {
                     const uint32_t memb = t.memb ? t.memb[c] : 1u;
                     if (!qm::passes_filter(memb, q.mask, q.xs, q.nx, c)) return;
                     if (!g_intersect<G>(t, q.shape, q.he, q.c, q.q, t.shape[c], ld3(t.dims, c), ld3(t.pos, c), ldq(t.rot, c))) return;
                     if (EMIT) seg[w] = c;
                     ++w;
                 });
    if (!EMIT) { counts[i] = w; return; }
    sort_segment(w, [&](uint32_t x, uint32_t y) { return seg[x] < seg[y]; }, [&](uint32_t x, uint32_t y) { const uint32_t v = seg[x]; seg[x] = seg[y]; seg[y] = v; });
}

// ---- move and slide (csrc/move_math.hpp): one thread per character runs the whole loop against the tree ------------------------------
template <class S>
struct Movers {
    int n;
    const uint8_t* shape; const S* dims; const S* pos; const S* rot; const S* vel;
    const uint32_t* mask; const uint32_t* xoff; const uint32_t* xs; const uint32_t* poff; const S* planes;
    const uint8_t* ignored;                          // [tree n] or NULL
};

// the cast leaf of a move, out of line: the shape-cast geometry is instanced once in the move kernel, not at each inlined call site
template <int G, class S>
__device__ __noinline__ bool move_cast_leaf(const Tree<S>& t, uint32_t c, int shape, nm::V3 he, nm::V3 ctr, nm::Q q, nm::V3 d, double maxd, double& th, int& axis) {
    return g_cast<G>(t, shape, he, ctr, q, d, maxd, qm::CAST_IGNORE_ORIGIN_PENETRATION, t.shape[c], ld3(t.dims, c), ld3(t.pos, c), ldq(t.rot, c), th, axis);
}

// the scene of move_math.hpp over the tree, with one character's filter
template <class S, int G>
struct TreeScene {
    const Tree<S>& t;
    int m;
    uint32_t mask, nx;
    const uint32_t* xs;
    const uint8_t* ignored;

    __device__ bool pass(uint32_t c) const {
        const uint32_t memb = t.memb ? t.memb[c] : 1u;
        return qm::passes_filter(memb, mask, xs, nx, c) && !(ignored && ignored[c]);
    }
    __device__ void collider(uint32_t c, int& s, nm::V3& he, nm::V3& p, nm::Q& q) const {
        s = t.shape[c]; he = ld3(t.dims, c); p = ld3(t.pos, c); q = ldq(t.rot, c);
    }
    __device__ const hm::Table& hulls() const { return t.hulls; }
    // the closest filtered cast: nearest-first over the node boxes grown by the shape's half size (as q_cast_shape)
    __device__ bool cast(int shape, nm::V3 he, nm::V3 ctr, nm::Q q, nm::V3 d, double maxd, double& t_out, uint32_t& c_out, int& axis_out) const {
        float ext[3];
        const nm::V3 e = g_half_size<G>(t, shape, he, qm::rot_mat(q));
        for (int k = 0; k < 3; ++k) {
            float l;
            qm::culling_bounds(-nm::comp(e, k), nm::comp(e, k), l, ext[k]);
        }
        double best_t = INFINITY;
        uint32_t best_c = 0xffffffffu;
        int best_axis = -1;
        traverse_nearest<true>(t, m, best_t, [&](const NodeBox& b) { return grown_entry(b, ext, ctr, d, maxd); },
                               [&](uint32_t c) {
                                   if (!pass(c)) return;
                                   double th;
                                   int ax;
                                   if (move_cast_leaf<G>(t, c, shape, he, ctr, q, d, maxd, th, ax) && qm::hit_before(th, c, best_t, best_c)) {
                                       best_t = th; best_c = c; best_axis = ax;
                                   }
                               });
        if (best_c == 0xffffffffu) return false;
        t_out = best_t; c_out = best_c; axis_out = best_axis;
        return true;
    }
    // fn(collider) in ascending index: each walk keeps the MOVE_WINDOW smallest passing indices above the last one handled, in a sorted
    // window, and notes whether it had to leave any out; the window is handled outside the walk, and the next walk starts above it
    template <class F>
    __device__ void candidates(const S lo[3], const S hi[3], F fn) const {
        const double lod[3] = {double(lo[0]), double(lo[1]), double(lo[2])}, hid[3] = {double(hi[0]), double(hi[1]), double(hi[2])};
        uint32_t after = 0;
        bool first = true;
        for (;;) {
            uint32_t win[mv::MOVE_WINDOW];
            int nw = 0;
            bool more = false;
            traverse(t, m,
                     [&](const NodeBox& nb) {
                         const double blo[3] = {nb.lo.x, nb.lo.y, nb.lo.z}, bhi[3] = {nb.hi.x, nb.hi.y, nb.hi.z};
                         return qm::aabb_overlap(lod, hid, blo, bhi);
                     },
                     [&](uint32_t c) {
                         if (!first && c <= after) return;
                         if (nw == mv::MOVE_WINDOW && c > win[nw - 1]) { more = true; return; }
                         if (!qm::aabb_overlap(lo, hi, t.tmn + 3 * size_t(c), t.tmx + 3 * size_t(c)) || !pass(c)) return;
                         if (nw == mv::MOVE_WINDOW) { more = true; --nw; }
                         int j = nw++;
                         for (; j > 0 && win[j - 1] > c; --j) win[j] = win[j - 1];
                         win[j] = c;
                     });
NM_ROLLED
            for (int k = 0; k < nw; ++k) fn(win[k]);
            if (!more || nw == 0) return;
            after = win[nw - 1];
            first = false;
        }
    }
};

template <class S>
struct MoveHits {
    int32_t* c; S* d; S* t; S* p; S* n;
    size_t base;
    __device__ void sweep(uint32_t it, uint32_t col, S safe, S toi, mv::T3<S> p1, mv::T3<S> n1) {
        const size_t o = base + it;
        if (c) c[o] = int32_t(col);
        if (d) d[o] = safe;
        if (t) t[o] = toi;
        if (p) { p[3 * o] = p1.x; p[3 * o + 1] = p1.y; p[3 * o + 2] = p1.z; }
        if (n) { n[3 * o] = n1.x; n[3 * o + 1] = n1.y; n[3 * o + 2] = n1.z; }
    }
};

template <class S, int G>
__global__ void __launch_bounds__(Q_THREADS) q_move(const __grid_constant__ Tree<S> t, const __grid_constant__ Movers<S> mb, const __grid_constant__ mv::Config<S> cfg,
                                                     S* __restrict__ out_pos, S* __restrict__ out_vel, int32_t* __restrict__ hc, S* __restrict__ hd,
                                                     S* __restrict__ ht, S* __restrict__ hp, S* __restrict__ hn) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= mb.n) return;
    MoveHits<S> hits{hc, hd, ht, hp, hn, size_t(i) * cfg.iterations};
    for (uint32_t it = 0; it < cfg.iterations; ++it) {
        const size_t o = hits.base + it;
        if (hc) hc[o] = -1;
        if (hd) hd[o] = S(0);
        if (ht) ht[o] = S(0);
        for (int k = 0; k < 3; ++k) {
            if (hp) hp[3 * o + k] = S(0);
            if (hn) hn[3 * o + k] = S(0);
        }
    }
    const mv::Body b{int(mb.shape[i]), ld3(mb.dims, i), ldq(mb.rot, i)};
    mv::T3<S> pos{mb.pos[3 * i], mb.pos[3 * i + 1], mb.pos[3 * i + 2]}, vel{mb.vel[3 * i], mb.vel[3 * i + 1], mb.vel[3 * i + 2]};
    if (qm::collider_valid(b.he, mv::to_v3(pos), b.q) && qm::finite3(mv::to_v3(vel))) {
        mv::T3<float> init[mv::MAX_PLANES];
        int ni = 0;
        if (mb.poff)
            for (uint32_t k = mb.poff[i]; k < mb.poff[i + 1]; ++k)
                init[ni++] = mv::plane_dir(mv::T3<S>{mb.planes[3 * k], mb.planes[3 * k + 1], mb.planes[3 * k + 2]});
        const TreeScene<S, G> sc{t, *t.m, mb.mask ? mb.mask[i] : 0xffffffffu, mb.xoff ? mb.xoff[i + 1] - mb.xoff[i] : 0u,
                              mb.xoff ? mb.xs + mb.xoff[i] : nullptr, mb.ignored};
        mv::move_and_slide<G>(sc, cfg, b, pos, vel, init, ni, hits);
    }
    out_pos[3 * i] = pos.x; out_pos[3 * i + 1] = pos.y; out_pos[3 * i + 2] = pos.z;
    out_vel[3 * i] = vel.x; out_vel[3 * i + 1] = vel.y; out_vel[3 * i + 2] = vel.z;
}

template <class S>
class Queries final : public QueriesBase {
   public:
    Queries(cudaStream_t stream, ErrorSink* err) : stream_(stream), err_(err) {}

    AvnStatus update(const AvnQueryColliders* c, uint32_t flags) override {
        const bool keep_shapes = (flags & AVN_QUERY_SHAPES_UNCHANGED) != 0;
        bool saw_capsule = false, saw_hull = false;
        uint32_t max_hull = 0;
        const uint32_t hc = hull_count();   // the kept column's check below reads it too
        if (const char* why = qm::check_colliders(c, !keep_shapes, sizeof(S) == 8, true, &saw_capsule, &hc, &saw_hull, &max_hull))
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_query_update: %s", why);
        if (keep_shapes && (!built_ || c->count != uint32_t(n_)))
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_query_update: AVN_QUERY_SHAPES_UNCHANGED needs a previous update of the same count");
        if (keep_shapes && hull_ && max_hull_ >= hc)   // the kept column's hulls against the current table
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_query_update: the kept shape column names convex hull %u, and the hull table holds %u", max_hull_, hc);
        const int n = int(c->count);
        built_ = false;
        n_ = n;
        if (!keep_shapes) {                      // AVN_QUERY_SHAPES_UNCHANGED keeps the shape column, and with it whether it holds a capsule or a hull
            caps_ = saw_capsule;
            hull_ = saw_hull;
            max_hull_ = max_hull;
        }
        gen_ = hulls_ ? hulls_->generation : 0;  // the hull bounds below are built from this table
        const size_t nn = size_t(std::max(n, 1));
        AVN_CUDA(pos_.ensure(3 * nn * sizeof(S)));
        AVN_CUDA(rot_.ensure(4 * nn * sizeof(S)));
        AVN_CUDA(shape_.ensure(nn));
        AVN_CUDA(dims_.ensure(3 * nn * sizeof(S)));
        AVN_CUDA(memb_.ensure(nn * sizeof(uint32_t)));
        AVN_CUDA(tmn_.ensure(3 * nn * sizeof(S)));
        AVN_CUDA(tmx_.ensure(3 * nn * sizeof(S)));
        AVN_CUDA(cbox_.ensure(nn * sizeof(NodeBox)));
        AVN_CUDA(centre_.ensure(nn * sizeof(float4)));
        AVN_CUDA(valid_.ensure(nn));
        AVN_CUDA(k0_.ensure(nn * 4)); AVN_CUDA(k1_.ensure(nn * 4)); AVN_CUDA(v0_.ensure(nn * 4)); AVN_CUDA(v1_.ensure(nn * 4));
        const int nblocks = int((nn + RS_TILE - 1) / RS_TILE);
        AVN_CUDA(hist_.ensure(size_t(256) * nblocks * 4));
        AVN_CUDA(nodes_.ensure((2 * nn) * sizeof(NodeBox)));
        AVN_CUDA(child_.ensure(nn * sizeof(int2)));
        AVN_CUDA(parent_.ensure(2 * nn * sizeof(int)));
        AVN_CUDA(arrived_.ensure(nn * sizeof(uint32_t)));
        AVN_CUDA(meta_.ensure(64));
        if (n > 0) {
            AVN_CUDA(cudaMemcpyAsync(pos_.p, c->position, 3 * size_t(n) * sizeof(S), cudaMemcpyHostToDevice, stream_));
            AVN_CUDA(cudaMemcpyAsync(rot_.p, c->rotation, 4 * size_t(n) * sizeof(S), cudaMemcpyHostToDevice, stream_));
            if (!keep_shapes) {
                AVN_CUDA(cudaMemcpyAsync(shape_.p, c->shape, size_t(n), cudaMemcpyHostToDevice, stream_));
                AVN_CUDA(cudaMemcpyAsync(dims_.p, c->dims, 3 * size_t(n) * sizeof(S), cudaMemcpyHostToDevice, stream_));
                has_memb_ = c->memberships != nullptr;
                if (has_memb_) AVN_CUDA(cudaMemcpyAsync(memb_.p, c->memberships, size_t(n) * sizeof(uint32_t), cudaMemcpyHostToDevice, stream_));
            }
        }
        // meta: [0] = m (colliders in the tree), [1..6] = ordered-integer scene bounds of the centres (min x y z, max x y z)
        int* d_m = meta_.as<int>();
        uint32_t* sb = meta_.as<uint32_t>() + 1;
        AVN_CUDA(cudaMemsetAsync(d_m, 0, 4, stream_));
        AVN_CUDA(cudaMemsetAsync(sb, 0xff, 12, stream_));
        AVN_CUDA(cudaMemsetAsync(sb + 3, 0, 12, stream_));
        const Tree<S> t = tree();
        if (n > 0) {
            const unsigned g = unsigned((n + 255) / 256);
            const int lv = level(false, false);
            auto prepare = lv == 2 ? q_prepare<S, 2> : lv == 1 ? q_prepare<S, 1> : q_prepare<S, 0>;
            prepare<<<g, 256, 0, stream_>>>(t, tmn_.as<S>(), tmx_.as<S>(), cbox_.as<NodeBox>(), centre_.as<float4>(), valid_.as<uint8_t>(), d_m, sb);
            q_codes<<<g, 256, 0, stream_>>>(n, centre_.as<float4>(), valid_.as<uint8_t>(), sb, k0_.as<uint32_t>(), v0_.as<uint32_t>());
            uint32_t *ka = k0_.as<uint32_t>(), *kb = k1_.as<uint32_t>(), *va = v0_.as<uint32_t>(), *vb = v1_.as<uint32_t>();
            for (int pass = 0; pass < 4; ++pass) {
                rs_histogram<uint32_t><<<nblocks, RS_THREADS, 0, stream_>>>(ka, n, 8 * pass, hist_.as<uint32_t>(), nblocks);
                if (nblocks <= RS_FUSE_MAX_BLOCKS) {
                    rs_scatter<uint32_t, true><<<nblocks, RS_THREADS, 0, stream_>>>(ka, va, n, 8 * pass, hist_.as<uint32_t>(), nblocks, kb, vb);
                } else {
                    rs_scan<<<1, 1024, 0, stream_>>>(hist_.as<uint32_t>(), 256 * nblocks);
                    rs_scatter<uint32_t, false><<<nblocks, RS_THREADS, 0, stream_>>>(ka, va, n, 8 * pass, hist_.as<uint32_t>(), nblocks, kb, vb);
                }
                std::swap(ka, kb);
                std::swap(va, vb);
            }
            // four passes: sorted keys and collider indices are back in k0_ / v0_
            AVN_CUDA(cudaMemsetAsync(arrived_.p, 0, size_t(n) * sizeof(uint32_t), stream_));
            q_karras<<<g, 256, 0, stream_>>>(d_m, n, k0_.as<uint32_t>(), child_.as<int2>(), parent_.as<int>());
            q_refit<<<g, 256, 0, stream_>>>(d_m, v0_.as<uint32_t>(), cbox_.as<NodeBox>(), parent_.as<int>(), child_.as<int2>(), arrived_.as<uint32_t>(),
                                            nodes_.as<NodeBox>());
            AVN_CUDA(cudaGetLastError());
        }
        AVN_CUDA(cudaStreamSynchronize(stream_));
        built_ = true;
        return AVN_OK;
    }

    AvnStatus cast_ray(const AvnRayBatch* r, AvnRayClosest* out) override {
        AvnStatus st = rays_in(r, "avn_query_cast_ray");
        if (st != AVN_OK) return st;
        if (!out || !out->collider || !out->distance || !out->normal)
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_query_cast_ray: collider, distance and normal outputs are required");
        const int n = int(r->count);
        if (n == 0) return AVN_OK;
        AVN_CUDA(oc_.ensure(size_t(n) * 4));
        AVN_CUDA(ot_.ensure(size_t(n) * sizeof(S)));
        AVN_CUDA(on_.ensure(3 * size_t(n) * sizeof(S)));
        const unsigned g = unsigned((n + Q_THREADS - 1) / Q_THREADS);
        const int lv = level(false, false);
        auto cast = lv == 2 ? q_cast_ray<S, 2> : lv == 1 ? q_cast_ray<S, 1> : q_cast_ray<S, 0>;
        cast<<<g, Q_THREADS, 0, stream_>>>(tree(), rays_, oc_.as<int32_t>(), ot_.as<S>(), on_.as<S>());
        AVN_CUDA(cudaGetLastError());
        AVN_CUDA(cudaMemcpyAsync(out->collider, oc_.p, size_t(n) * 4, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(out->distance, ot_.p, size_t(n) * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(out->normal, on_.p, 3 * size_t(n) * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        return AVN_OK;
    }

    AvnStatus ray_hits(const AvnRayBatch* r, AvnHitList* out) override {
        AvnStatus st = rays_in(r, "avn_query_ray_hits");
        if (st != AVN_OK) return st;
        if ((st = list_out(out, "avn_query_ray_hits")) != AVN_OK) return st;
        const int n = int(r->count);
        AVN_CUDA(full_.ensure(size_t(n + 1) * 4));
        AVN_CUDA(kept_.ensure(size_t(n + 1) * 4));
        AVN_CUDA(full_off_.ensure(size_t(n + 1) * 8));
        AVN_CUDA(kept_off_.ensure(size_t(n + 1) * 8));
        const Tree<S> t = tree();
        const unsigned g = unsigned((n + Q_THREADS - 1) / Q_THREADS);
        const int lv = level(false, false);
        if (n > 0) {
            auto count = lv == 2 ? q_ray_count<S, 2> : lv == 1 ? q_ray_count<S, 1> : q_ray_count<S, 0>;
            count<<<g, Q_THREADS, 0, stream_>>>(t, rays_, full_.as<uint32_t>(), kept_.as<uint32_t>());
        }
        uint64_t tot[2];
        if ((st = scan(full_.as<uint32_t>(), n, full_off_.as<uint64_t>())) != AVN_OK) return st;
        if ((st = scan(kept_.as<uint32_t>(), n, kept_off_.as<uint64_t>())) != AVN_OK) return st;
        AVN_CUDA(cudaMemcpyAsync(&tot[0], full_off_.as<uint64_t>() + n, 8, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(&tot[1], kept_off_.as<uint64_t>() + n, 8, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        out->count = tot[1];
        if (tot[1] > out->capacity)
            return err_->fail(AVN_ERR_CAPACITY, "avn_query_ray_hits: %llu hits, capacity %llu", (unsigned long long)tot[1], (unsigned long long)out->capacity);
        const size_t nf = size_t(std::max<uint64_t>(tot[0], 1)), nk = size_t(std::max<uint64_t>(tot[1], 1));
        AVN_CUDA(tmp_t_.ensure(nf * 8));
        AVN_CUDA(tmp_c_.ensure(nf * 4));
        AVN_CUDA(oc_.ensure(nk * 4));
        AVN_CUDA(ot_.ensure(nk * sizeof(S)));
        AVN_CUDA(on_.ensure(3 * nk * sizeof(S)));
        if (n > 0 && tot[1] > 0) {
            auto emit = lv == 2 ? q_ray_emit<S, 2> : lv == 1 ? q_ray_emit<S, 1> : q_ray_emit<S, 0>;
            emit<<<g, Q_THREADS, 0, stream_>>>(t, rays_, full_off_.as<uint64_t>(), kept_off_.as<uint64_t>(), tmp_t_.as<double>(), tmp_c_.as<uint32_t>(),
                                               oc_.as<uint32_t>(), ot_.as<S>(), on_.as<S>());
            AVN_CUDA(cudaGetLastError());
        }
        return list_download(out, n, kept_off_.as<uint64_t>(), tot[1], true);
    }

    AvnStatus aabb_intersections(uint32_t count, const void* mn, const void* mx, AvnHitList* out) override {
        if (!built_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_query_aabb_intersections before any avn_query_update");
        if (AvnStatus st = stale("avn_query_aabb_intersections")) return st;
        if (count && (!mn || !mx)) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_query_aabb_intersections: min and max are required");
        AvnStatus st = list_out(out, "avn_query_aabb_intersections");
        if (st != AVN_OK) return st;
        const int n = int(count);
        const size_t nn = size_t(std::max(n, 1));
        AVN_CUDA(qmn_.ensure(3 * nn * sizeof(S)));
        AVN_CUDA(qmx_.ensure(3 * nn * sizeof(S)));
        AVN_CUDA(full_.ensure((nn + 1) * 4));
        AVN_CUDA(kept_off_.ensure((nn + 1) * 8));
        if (n > 0) {
            AVN_CUDA(cudaMemcpyAsync(qmn_.p, mn, 3 * size_t(n) * sizeof(S), cudaMemcpyHostToDevice, stream_));
            AVN_CUDA(cudaMemcpyAsync(qmx_.p, mx, 3 * size_t(n) * sizeof(S), cudaMemcpyHostToDevice, stream_));
        }
        const Tree<S> t = tree();
        const unsigned g = unsigned((n + Q_THREADS - 1) / Q_THREADS);
        if (n > 0) q_aabb<S, false><<<g, Q_THREADS, 0, stream_>>>(t, n, qmn_.as<S>(), qmx_.as<S>(), full_.as<uint32_t>(), nullptr, nullptr);
        if ((st = scan(full_.as<uint32_t>(), n, kept_off_.as<uint64_t>())) != AVN_OK) return st;
        uint64_t total = 0;
        AVN_CUDA(cudaMemcpyAsync(&total, kept_off_.as<uint64_t>() + n, 8, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        out->count = total;
        if (total > out->capacity)
            return err_->fail(AVN_ERR_CAPACITY, "avn_query_aabb_intersections: %llu hits, capacity %llu", (unsigned long long)total, (unsigned long long)out->capacity);
        AVN_CUDA(oc_.ensure(size_t(std::max<uint64_t>(total, 1)) * 4));
        if (n > 0 && total > 0) {
            q_aabb<S, true><<<g, Q_THREADS, 0, stream_>>>(t, n, qmn_.as<S>(), qmx_.as<S>(), nullptr, kept_off_.as<uint64_t>(), oc_.as<uint32_t>());
            AVN_CUDA(cudaGetLastError());
        }
        return list_download(out, n, kept_off_.as<uint64_t>(), total, false);
    }

    AvnStatus cast_shape(const AvnShapeBatch* s, AvnShapeClosest* out) override {
        AvnStatus st = shapes_in(s, true, "avn_query_cast_shape");
        if (st != AVN_OK) return st;
        if (!out || (s->count && (!out->collider || !out->distance || !out->point1 || !out->point2 || !out->normal1 || !out->normal2)))
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_query_cast_shape: collider, distance, point1, point2, normal1 and normal2 outputs are required");
        const int n = int(s->count);
        if (n == 0) return AVN_OK;
        AVN_CUDA(oc_.ensure(size_t(n) * 4));
        AVN_CUDA(ot_.ensure(size_t(n) * sizeof(S)));
        for (DevBuf* b : {&op1_, &op2_, &on1_, &on2_}) AVN_CUDA(b->ensure(3 * size_t(n) * sizeof(S)));
        const int lv = level(shapes_caps_, shapes_hull_);
        auto cast = lv == 2 ? q_cast_shape<S, 2> : lv == 1 ? q_cast_shape<S, 1> : q_cast_shape<S, 0>;
        cast<<<unsigned((n + Q_THREADS - 1) / Q_THREADS), Q_THREADS, 0, stream_>>>(tree(), shapes_, oc_.as<int32_t>(), ot_.as<S>(), op1_.as<S>(), op2_.as<S>(),
                                                                                 on1_.as<S>(), on2_.as<S>());
        AVN_CUDA(cudaGetLastError());
        AVN_CUDA(cudaMemcpyAsync(out->collider, oc_.p, size_t(n) * 4, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(out->distance, ot_.p, size_t(n) * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        void* dst[4] = {out->point1, out->point2, out->normal1, out->normal2};
        const DevBuf* src[4] = {&op1_, &op2_, &on1_, &on2_};
        for (int k = 0; k < 4; ++k) AVN_CUDA(cudaMemcpyAsync(dst[k], src[k]->p, 3 * size_t(n) * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        return AVN_OK;
    }

    AvnStatus shape_hits(const AvnShapeBatch* s, AvnShapeHitList* out) override {
        AvnStatus st = shapes_in(s, true, "avn_query_shape_hits");
        if (st != AVN_OK) return st;
        if (!out || !out->offsets || (out->capacity && !out->collider))
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_query_shape_hits: offsets and (with a capacity) collider are required");
        const int n = int(s->count);
        AVN_CUDA(full_.ensure(size_t(n + 1) * 4));
        AVN_CUDA(kept_.ensure(size_t(n + 1) * 4));
        AVN_CUDA(full_off_.ensure(size_t(n + 1) * 8));
        AVN_CUDA(kept_off_.ensure(size_t(n + 1) * 8));
        const Tree<S> t = tree();
        const unsigned g = unsigned((n + Q_THREADS - 1) / Q_THREADS);
        const int lv = level(shapes_caps_, shapes_hull_);
        if (n > 0) {
            auto count = lv == 2 ? q_shape_count<S, 2> : lv == 1 ? q_shape_count<S, 1> : q_shape_count<S, 0>;
            count<<<g, Q_THREADS, 0, stream_>>>(t, shapes_, full_.as<uint32_t>(), kept_.as<uint32_t>());
        }
        uint64_t tot[2];
        if ((st = scan(full_.as<uint32_t>(), n, full_off_.as<uint64_t>())) != AVN_OK) return st;
        if ((st = scan(kept_.as<uint32_t>(), n, kept_off_.as<uint64_t>())) != AVN_OK) return st;
        AVN_CUDA(cudaMemcpyAsync(&tot[0], full_off_.as<uint64_t>() + n, 8, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(&tot[1], kept_off_.as<uint64_t>() + n, 8, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        out->count = tot[1];
        if (tot[1] > out->capacity)
            return err_->fail(AVN_ERR_CAPACITY, "avn_query_shape_hits: %llu hits, capacity %llu", (unsigned long long)tot[1], (unsigned long long)out->capacity);
        const size_t nf = size_t(std::max<uint64_t>(tot[0], 1)), nk = size_t(std::max<uint64_t>(tot[1], 1));
        AVN_CUDA(tmp_t_.ensure(nf * 8));
        AVN_CUDA(tmp_c_.ensure(nf * 4));
        AVN_CUDA(oc_.ensure(nk * 4));
        AVN_CUDA(ot_.ensure(nk * sizeof(S)));
        for (DevBuf* b : {&op1_, &op2_, &on1_, &on2_}) AVN_CUDA(b->ensure(3 * nk * sizeof(S)));
        if (n > 0 && tot[1] > 0) {
            auto emit = lv == 2 ? q_shape_emit<S, 2> : lv == 1 ? q_shape_emit<S, 1> : q_shape_emit<S, 0>;
            emit<<<g, Q_THREADS, 0, stream_>>>(t, shapes_, full_off_.as<uint64_t>(), kept_off_.as<uint64_t>(), tmp_t_.as<double>(), tmp_c_.as<uint32_t>(),
                                               oc_.as<uint32_t>(), ot_.as<S>(), op1_.as<S>(), op2_.as<S>(), on1_.as<S>(), on2_.as<S>());
            AVN_CUDA(cudaGetLastError());
        }
        AVN_CUDA(cudaMemcpyAsync(out->offsets, kept_off_.as<uint64_t>(), size_t(n + 1) * 8, cudaMemcpyDeviceToHost, stream_));
        if (tot[1]) {
            const size_t k = tot[1];
            AVN_CUDA(cudaMemcpyAsync(out->collider, oc_.p, k * 4, cudaMemcpyDeviceToHost, stream_));
            if (out->distance) AVN_CUDA(cudaMemcpyAsync(out->distance, ot_.p, k * sizeof(S), cudaMemcpyDeviceToHost, stream_));
            void* dst[4] = {out->point1, out->point2, out->normal1, out->normal2};
            const DevBuf* src[4] = {&op1_, &op2_, &on1_, &on2_};
            for (int j = 0; j < 4; ++j)
                if (dst[j]) AVN_CUDA(cudaMemcpyAsync(dst[j], src[j]->p, 3 * k * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        }
        AVN_CUDA(cudaStreamSynchronize(stream_));
        return AVN_OK;
    }

    AvnStatus project_point(const AvnPointBatch* p, AvnPointProjection* out) override {
        AvnStatus st = points_in(p, "avn_query_project_point");
        if (st != AVN_OK) return st;
        if (!out || (p->count && (!out->collider || !out->point || !out->is_inside)))
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_query_project_point: collider, point and is_inside outputs are required");
        const int n = int(p->count);
        if (n == 0) return AVN_OK;
        AVN_CUDA(oc_.ensure(size_t(n) * 4));
        AVN_CUDA(op1_.ensure(3 * size_t(n) * sizeof(S)));
        AVN_CUDA(oin_.ensure(size_t(n)));
        const int lv = level(false, false);
        auto project = lv == 2 ? q_project_point<S, 2> : lv == 1 ? q_project_point<S, 1> : q_project_point<S, 0>;
        project<<<unsigned((n + Q_THREADS - 1) / Q_THREADS), Q_THREADS, 0, stream_>>>(tree(), points_, oc_.as<int32_t>(), op1_.as<S>(), oin_.as<uint8_t>());
        AVN_CUDA(cudaGetLastError());
        AVN_CUDA(cudaMemcpyAsync(out->collider, oc_.p, size_t(n) * 4, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(out->point, op1_.p, 3 * size_t(n) * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(out->is_inside, oin_.p, size_t(n), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        return AVN_OK;
    }

    AvnStatus point_intersections(const AvnPointBatch* p, AvnHitList* out) override {
        AvnStatus st = points_in(p, "avn_query_point_intersections");
        if (st != AVN_OK) return st;
        if ((st = list_out(out, "avn_query_point_intersections")) != AVN_OK) return st;
        const int n = int(p->count);
        const int lv = level(false, false);
        return intersections(n, out, "avn_query_point_intersections", [&](const Tree<S>& t, unsigned g, uint32_t* counts, const uint64_t* off, uint32_t* oc) {
            if (counts)
                (lv == 2 ? q_point_isect<S, false, 2> : lv == 1 ? q_point_isect<S, false, 1> : q_point_isect<S, false, 0>)<<<g, Q_THREADS, 0, stream_>>>(t, points_, counts, nullptr, nullptr);
            else
                (lv == 2 ? q_point_isect<S, true, 2> : lv == 1 ? q_point_isect<S, true, 1> : q_point_isect<S, true, 0>)<<<g, Q_THREADS, 0, stream_>>>(t, points_, nullptr, off, oc);
        });
    }

    AvnStatus shape_intersections(const AvnShapeBatch* s, AvnHitList* out) override {
        AvnStatus st = shapes_in(s, false, "avn_query_shape_intersections");
        if (st != AVN_OK) return st;
        if ((st = list_out(out, "avn_query_shape_intersections")) != AVN_OK) return st;
        const int n = int(s->count);
        const int lv = level(shapes_caps_, shapes_hull_);
        return intersections(n, out, "avn_query_shape_intersections", [&](const Tree<S>& t, unsigned g, uint32_t* counts, const uint64_t* off, uint32_t* oc) {
            if (counts)
                (lv == 2 ? q_shape_isect<S, false, 2> : lv == 1 ? q_shape_isect<S, false, 1> : q_shape_isect<S, false, 0>)<<<g, Q_THREADS, 0, stream_>>>(t, shapes_, counts, nullptr, nullptr);
            else
                (lv == 2 ? q_shape_isect<S, true, 2> : lv == 1 ? q_shape_isect<S, true, 1> : q_shape_isect<S, true, 0>)<<<g, Q_THREADS, 0, stream_>>>(t, shapes_, nullptr, off, oc);
        });
    }

    AvnStatus move_and_slide(const AvnMoveConfig* cfg, const AvnMoveBatch* b, AvnMoveResult* out) override {
        if (!built_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_move_and_slide before any avn_query_update");
        if (AvnStatus st = stale("avn_move_and_slide")) return st;
        bool batch_caps = false, batch_hull = false;
        const uint32_t hull_n = hull_count();
        if (const char* why = mv::check_move(cfg, b, sizeof(S) == 8, uint32_t(n_), true, &batch_caps, &hull_n, &batch_hull))
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_move_and_slide: %s", why);
        if (!out || (b->count && (!out->position || !out->velocity)))
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_move_and_slide: position and velocity outputs are required");
        out->kernel_ms = 0.f;
        const size_t n = b->count;
        if (n == 0) return AVN_OK;
        Movers<S> mb{};
        mb.n = int(n);
        AvnStatus st;
#define UPM(buf, host, cnt, T, dst) if ((st = up<T>(buf, host, cnt, &dst)) != AVN_OK) return st
        UPM(s_shape_, b->shape, n, uint8_t, mb.shape);
        UPM(s_dims_, b->dims, 3 * n, S, mb.dims);
        UPM(s_pos_, b->position, 3 * n, S, mb.pos);
        UPM(s_rot_, b->rotation, 4 * n, S, mb.rot);
        UPM(s_d_, b->velocity, 3 * n, S, mb.vel);
        UPM(s_mask_, b->mask, n, uint32_t, mb.mask);
        UPM(s_xoff_, b->exclude_offsets, n + 1, uint32_t, mb.xoff);
        if (b->exclude_offsets) UPM(s_xs_, b->exclude_count ? b->exclude : nullptr, b->exclude_count, uint32_t, mb.xs);
        UPM(m_poff_, b->plane_offsets, n + 1, uint32_t, mb.poff);
        if (b->plane_offsets) UPM(m_planes_, b->planes, 3 * size_t(b->plane_offsets[n]), S, mb.planes);
        UPM(m_ignored_, cfg->ignored, size_t(n_), uint8_t, mb.ignored);
#undef UPM
        const size_t nh = n * cfg->move_and_slide_iterations;
        AVN_CUDA(op1_.ensure(3 * n * sizeof(S)));
        AVN_CUDA(op2_.ensure(3 * n * sizeof(S)));
        int32_t* hc = nullptr;
        S *hd = nullptr, *ht = nullptr, *hp = nullptr, *hn = nullptr;
        if (nh) {
            if (out->hit_collider) { AVN_CUDA(oc_.ensure(nh * 4)); hc = oc_.as<int32_t>(); }
            if (out->hit_distance) { AVN_CUDA(ot_.ensure(nh * sizeof(S))); hd = ot_.as<S>(); }
            if (out->hit_toi) { AVN_CUDA(m_toi_.ensure(nh * sizeof(S))); ht = m_toi_.as<S>(); }
            if (out->hit_point) { AVN_CUDA(on1_.ensure(3 * nh * sizeof(S))); hp = on1_.as<S>(); }
            if (out->hit_normal) { AVN_CUDA(on2_.ensure(3 * nh * sizeof(S))); hn = on2_.as<S>(); }
        }
        if (!ev_[0]) {
            AVN_CUDA(cudaEventCreate(&ev_[0]));
            AVN_CUDA(cudaEventCreate(&ev_[1]));
        }
        AVN_CUDA(cudaEventRecord(ev_[0], stream_));
        const int lv = level(batch_caps, batch_hull);
        auto move = lv == 2 ? q_move<S, 2> : lv == 1 ? q_move<S, 1> : q_move<S, 0>;
        move<<<unsigned((n + Q_THREADS - 1) / Q_THREADS), Q_THREADS, 0, stream_>>>(tree(), mb, mv::config_of<S>(cfg), op1_.as<S>(), op2_.as<S>(), hc, hd, ht, hp, hn);
        AVN_CUDA(cudaGetLastError());
        AVN_CUDA(cudaEventRecord(ev_[1], stream_));
        AVN_CUDA(cudaMemcpyAsync(out->position, op1_.p, 3 * n * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(out->velocity, op2_.p, 3 * n * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        if (hc) AVN_CUDA(cudaMemcpyAsync(out->hit_collider, hc, nh * 4, cudaMemcpyDeviceToHost, stream_));
        if (hd) AVN_CUDA(cudaMemcpyAsync(out->hit_distance, hd, nh * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        if (ht) AVN_CUDA(cudaMemcpyAsync(out->hit_toi, ht, nh * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        if (hp) AVN_CUDA(cudaMemcpyAsync(out->hit_point, hp, 3 * nh * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        if (hn) AVN_CUDA(cudaMemcpyAsync(out->hit_normal, hn, 3 * nh * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        AVN_CUDA(cudaEventElapsedTime(&out->kernel_ms, ev_[0], ev_[1]));
        return AVN_OK;
    }

    void attach_hulls(const HullTable* hulls) override { hulls_ = hulls; }

    ~Queries() override {
        for (cudaEvent_t e : ev_)
            if (e) cudaEventDestroy(e);
    }

   private:
    // count -> scan -> (capacity check) -> emit of a collider-only CSR list; launch(t, grid, counts, nullptr, nullptr) counts,
    // launch(t, grid, nullptr, offsets, out) emits
    template <class Launch>
    AvnStatus intersections(int n, AvnHitList* out, const char* what, Launch launch) {
        const size_t nn = size_t(std::max(n, 1));
        AVN_CUDA(full_.ensure((nn + 1) * 4));
        AVN_CUDA(kept_off_.ensure((nn + 1) * 8));
        const Tree<S> t = tree();
        const unsigned g = unsigned((n + Q_THREADS - 1) / Q_THREADS);
        if (n > 0) launch(t, g, full_.as<uint32_t>(), nullptr, nullptr);
        AvnStatus st = scan(full_.as<uint32_t>(), n, kept_off_.as<uint64_t>());
        if (st != AVN_OK) return st;
        uint64_t total = 0;
        AVN_CUDA(cudaMemcpyAsync(&total, kept_off_.as<uint64_t>() + n, 8, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        out->count = total;
        if (total > out->capacity)
            return err_->fail(AVN_ERR_CAPACITY, "%s: %llu hits, capacity %llu", what, (unsigned long long)total, (unsigned long long)out->capacity);
        AVN_CUDA(oc_.ensure(size_t(std::max<uint64_t>(total, 1)) * 4));
        if (n > 0 && total > 0) {
            launch(t, g, nullptr, kept_off_.as<uint64_t>(), oc_.as<uint32_t>());
            AVN_CUDA(cudaGetLastError());
        }
        return list_download(out, n, kept_off_.as<uint64_t>(), total, false);
    }

    // validate on the host, then upload the shape columns into shapes_ (cast: the cast-only columns too)
    AvnStatus shapes_in(const AvnShapeBatch* s, bool cast, const char* what) {
        if (!built_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "%s before any avn_query_update", what);
        if (AvnStatus st = stale(what)) return st;
        const uint32_t hc = hull_count();
        if (const char* why = qm::check_shapes(s, cast, sizeof(S) == 8, true, &shapes_caps_, &hc, &shapes_hull_))
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "%s: %s", what, why);
        const size_t n = s->count;
        shapes_ = Shapes<S>{};
        shapes_.n = int(n);
        if (n == 0) return AVN_OK;
        AvnStatus st;
#define UPS(buf, host, cnt, T, dst) if ((st = up<T>(buf, host, cnt, &dst)) != AVN_OK) return st
        UPS(s_shape_, s->shape, n, uint8_t, shapes_.shape);
        UPS(s_dims_, s->dims, 3 * n, S, shapes_.dims);
        UPS(s_pos_, s->position, 3 * n, S, shapes_.pos);
        UPS(s_rot_, s->rotation, 4 * n, S, shapes_.rot);
        if (cast) {
            UPS(s_d_, s->direction, 3 * n, S, shapes_.d);
            UPS(s_maxd_, s->max_distance, n, S, shapes_.maxd);
            UPS(s_flags_, s->flags, n, uint32_t, shapes_.flags);
            UPS(s_mh_, s->max_hits, n, uint32_t, shapes_.max_hits);
        }
        UPS(s_mask_, s->mask, n, uint32_t, shapes_.mask);
        UPS(s_xoff_, s->exclude_offsets, n + 1, uint32_t, shapes_.xoff);
        if (s->exclude_offsets) UPS(s_xs_, s->exclude_count ? s->exclude : nullptr, s->exclude_count, uint32_t, shapes_.xs);
#undef UPS
        return AVN_OK;
    }
    AvnStatus points_in(const AvnPointBatch* p, const char* what) {
        if (!built_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "%s before any avn_query_update", what);
        if (AvnStatus st = stale(what)) return st;
        if (const char* why = qm::check_points(p)) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "%s: %s", what, why);
        const size_t n = p->count;
        points_ = Points<S>{};
        points_.n = int(n);
        if (n == 0) return AVN_OK;
        AvnStatus st;
#define UPP(buf, host, cnt, T, dst) if ((st = up<T>(buf, host, cnt, &dst)) != AVN_OK) return st
        UPP(r_o_, p->point, 3 * n, S, points_.p);
        UPP(r_solid_, p->solid, n, uint8_t, points_.solid);
        UPP(r_mask_, p->mask, n, uint32_t, points_.mask);
        UPP(r_xoff_, p->exclude_offsets, n + 1, uint32_t, points_.xoff);
        if (p->exclude_offsets) UPP(r_xs_, p->exclude_count ? p->exclude : nullptr, p->exclude_count, uint32_t, points_.xs);
#undef UPP
        return AVN_OK;
    }

    Tree<S> tree() const {
        Tree<S> t{};
        t.n = n_;
        t.m = meta_.as<int>();
        t.shape = shape_.as<uint8_t>(); t.dims = dims_.as<S>(); t.pos = pos_.as<S>(); t.rot = rot_.as<S>();
        t.memb = has_memb_ ? memb_.as<uint32_t>() : nullptr;
        t.tmn = tmn_.as<S>(); t.tmx = tmx_.as<S>();
        t.nodes = nodes_.as<NodeBox>(); t.child = child_.as<int2>(); t.leaf = v0_.as<uint32_t>();
        t.hulls = hulls_ && hulls_->set ? hulls_->dev : hm::Table{};
        return t;
    }
    uint32_t hull_count() const { return hulls_ ? hulls_->count() : 0u; }
    // the instance that covers the tree and the batch: 2 with a hull, 1 with a capsule, else 0
    int level(bool batch_caps, bool batch_hull) const { return hull_ || batch_hull ? 2 : (caps_ || batch_caps ? 1 : 0); }
    // a tree holding a hull was bounded with the table of its update: refused once avn_set_convex_hulls has replaced that table
    AvnStatus stale(const char* what) {
        if (hull_ && (!hulls_ || hulls_->generation != gen_))
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "%s: the convex hull table was replaced after the avn_query_update whose tree holds a hull: update again", what);
        return AVN_OK;
    }

    // validate on the host, then upload the ray columns into rays_
    AvnStatus rays_in(const AvnRayBatch* r, const char* what) {
        if (!built_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "%s before any avn_query_update", what);
        if (AvnStatus st = stale(what)) return st;
        if (const char* why = qm::check_rays(r)) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "%s: %s", what, why);
        if (r->count >= 0x7fffffffu) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "%s: too many rays", what);
        const size_t n = r->count;
        rays_ = Rays<S>{};
        rays_.n = int(n);
        if (n == 0) return AVN_OK;
        AvnStatus st;
#define UPR(buf, host, cnt, T, dst) if ((st = up<T>(buf, host, cnt, &dst)) != AVN_OK) return st
        UPR(r_o_, r->origin, 3 * n, S, rays_.o);
        UPR(r_d_, r->direction, 3 * n, S, rays_.d);
        UPR(r_maxd_, r->max_distance, n, S, rays_.maxd);
        UPR(r_solid_, r->solid, n, uint8_t, rays_.solid);
        UPR(r_mh_, r->max_hits, n, uint32_t, rays_.max_hits);
        UPR(r_mask_, r->mask, n, uint32_t, rays_.mask);
        UPR(r_xoff_, r->exclude_offsets, n + 1, uint32_t, rays_.xoff);
        if (r->exclude_offsets) UPR(r_xs_, r->exclude_count ? r->exclude : nullptr, r->exclude_count, uint32_t, rays_.xs);
#undef UPR
        return AVN_OK;
    }
    AvnStatus list_out(AvnHitList* out, const char* what) {
        if (!out || !out->offsets || (out->capacity && !out->collider))
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "%s: offsets and (with a capacity) collider are required", what);
        return AVN_OK;
    }
    // exclusive scan of n counts -> offsets[0..n], offsets[n] = total
    AvnStatus scan(const uint32_t* counts, int n, uint64_t* offsets) {
        if (n == 0) {
            AVN_CUDA(cudaMemsetAsync(offsets, 0, 8, stream_));
            return AVN_OK;
        }
        const int sblocks = (n + 1023) / 1024;
        AVN_CUDA(block_sums_.ensure(size_t(sblocks) * 8));
        scan_block_sums<<<sblocks, 1024, 0, stream_>>>(counts, n, block_sums_.as<uint64_t>());
        scan_block_offsets<<<1, 1024, 0, stream_>>>(block_sums_.as<uint64_t>(), sblocks, offsets + n);
        scan_apply<<<sblocks, 1024, 0, stream_>>>(counts, n, block_sums_.as<uint64_t>(), offsets);
        AVN_CUDA(cudaGetLastError());
        return AVN_OK;
    }
    AvnStatus list_download(AvnHitList* out, int n, const uint64_t* d_off, uint64_t total, bool ray) {
        AVN_CUDA(cudaMemcpyAsync(out->offsets, d_off, size_t(n + 1) * 8, cudaMemcpyDeviceToHost, stream_));
        if (total) {
            AVN_CUDA(cudaMemcpyAsync(out->collider, oc_.p, total * 4, cudaMemcpyDeviceToHost, stream_));
            if (ray && out->distance) AVN_CUDA(cudaMemcpyAsync(out->distance, ot_.p, total * sizeof(S), cudaMemcpyDeviceToHost, stream_));
            if (ray && out->normal) AVN_CUDA(cudaMemcpyAsync(out->normal, on_.p, 3 * total * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        }
        AVN_CUDA(cudaStreamSynchronize(stream_));
        return AVN_OK;
    }
    template <class T> AvnStatus up(DevBuf& buf, const void* host, size_t count, const T** dev) {
        *dev = nullptr;
        if (!host || count == 0) return AVN_OK;
        AVN_CUDA(buf.ensure(count * sizeof(T)));
        AVN_CUDA(cudaMemcpyAsync(buf.p, host, count * sizeof(T), cudaMemcpyHostToDevice, stream_));
        *dev = buf.as<T>();
        return AVN_OK;
    }

    cudaStream_t stream_;
    ErrorSink* err_;
    bool built_ = false, has_memb_ = false;
    bool caps_ = false;                              // the tree's shape column holds a capsule
    bool shapes_caps_ = false;                       // the last shape batch holds a capsule
    bool hull_ = false;                              // the tree's shape column holds a convex hull
    bool shapes_hull_ = false;                       // the last shape batch holds a convex hull
    uint32_t max_hull_ = 0;                          // the largest hull index of the tree's shape column
    uint64_t gen_ = 0;                               // the hull table generation the tree was built with
    const HullTable* hulls_ = nullptr;               // the context's table (attach_hulls)
    int n_ = 0;
    Rays<S> rays_{};
    Shapes<S> shapes_{};
    Points<S> points_{};
    DevBuf s_shape_, s_dims_, s_pos_, s_rot_, s_d_, s_maxd_, s_flags_, s_mh_, s_mask_, s_xoff_, s_xs_, op1_, op2_, on1_, on2_, oin_;
    DevBuf pos_, rot_, shape_, dims_, memb_, tmn_, tmx_, cbox_, centre_, valid_, k0_, k1_, v0_, v1_, hist_, nodes_, child_, parent_, arrived_, meta_;
    DevBuf r_o_, r_d_, r_maxd_, r_solid_, r_mh_, r_mask_, r_xoff_, r_xs_;
    DevBuf full_, kept_, full_off_, kept_off_, block_sums_, tmp_t_, tmp_c_, oc_, ot_, on_, qmn_, qmx_;
    DevBuf m_poff_, m_planes_, m_ignored_, m_toi_;
    cudaEvent_t ev_[2] = {nullptr, nullptr};
};

}  // namespace

QueriesBase* make_queries(uint32_t scalar_bits, cudaStream_t stream, ErrorSink* err) {
    if (scalar_bits == 32) return new Queries<float>(stream, err);
    if (scalar_bits == 64) return new Queries<double>(stream, err);
    return nullptr;
}

}  // namespace avn
