// Spatial-query geometry for cuboid / sphere colliders, written once for the host fixture (g++, -ffp-contract=off) and for the device
// (nvcc, -fmad=false): the same expressions in the same order, IEEE double throughout, so both evaluate to the same bits.
//
// What this is: OUR ray and AABB arithmetic.  The reference delegates it to parry3d 0.25 (Cuboid / Ball ray casts, compute_aabb), which is
// not vendored, so there is no parity claim against parry — the claim is that the device (csrc/queries.cu, tree traversal) and the host
// brute force (host/host_api.cpp, every collider) report the same hits bit for bit.
// Reference call sites: spatial_query/pipeline.rs:96-133 (update: compute_aabb per collider), 156-216 (cast_ray, ray_hits),
// 700-729 (aabb_intersections_with_aabb), query_filter.rs:97-101 (SpatialQueryFilter::test).
//
// Conventions (ours, not parry's; repeated in include/avian_b200.h and DESIGN.md §7d):
//   * Tight collider AABB, as compute_aabb(isometry): cuboid centre ± |R|·half_extents, sphere centre ± radius.  Rounded to the column
//     scalar for output and for the exact AABB test.
//   * A ray is origin + t·direction; distances t are in units of |direction| (the caller passes a unit Dir3).
//   * A hit counts when 0 <= t <= max_distance.
//   * Shapes are closed: a point on the surface is inside.  Origin inside and `solid` -> t = 0, normal 0.  Origin inside and hollow ->
//     the exit parameter with the outward normal at the exit.
//   * The rotation is the quaternion's, normalised (rot_mat): the AABB and the ray test see the same box for a quaternion of any length.
//   * Ray vs cuboid: the ray goes into the cuboid's frame (components along the rotated axes), then a slab test.  A direction component that
//     is exactly 0 is handled on its own, with no 0·inf: the ray misses when the origin is outside that slab, else the axis is unconstrained.
//     The normal is the outward face normal of the entering axis (the largest entering parameter, ties to the lowest axis index) rotated
//     back to world; for a hollow exit, of the exiting axis (the smallest exit parameter, ties to the lowest axis index).
//   * Ray vs sphere: closed form of |o + t·d - c|² = r²; the normal is the unit vector from the centre to the hit point.
//   * Filter: a collider passes when (memberships & mask) != 0 and it is not in the ray's excluded list.
//   * AABB test: inclusive compares on all three axes (Aabb::intersects) against the tight AABB, with no filter.
//   * A collider with a non-finite pose or dims, or a zero rotation quaternion, is never reported (negative dims are refused); a ray with a non-finite origin, direction or max_distance hits nothing.
#pragma once
#include <cmath>
#include <cstdint>

#include "narrow_math.hpp"

namespace qm {

using nm::S;
using nm::V3;
using nm::Q;

NM_HD inline bool finite3(V3 v) { return std::isfinite(v.x) && std::isfinite(v.y) && std::isfinite(v.z); }

// a collider the queries can report: finite pose and dims and a rotation quaternion that can be normalised
NM_HD inline bool collider_valid(V3 he, V3 p, Q q) {
    return finite3(he) && finite3(p) && std::isfinite(q.x) && std::isfinite(q.y) && std::isfinite(q.z) && std::isfinite(q.w) &&
           q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w > 0;
}

// The rotation of q as a proper rotation matrix (columns = world directions of the local axes).  nm::to_mat(q) is |q|²·R, so it is divided
// by |q|² here: a quaternion rounded to f32 from a unit one has |q|² - 1 of about 1e-7, and the AABB and the ray test must describe the
// same box, not one scaled by |q|² and the other by 1/|q|².
NM_HD inline nm::M3 rot_mat(Q q) {
    const S s = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
    const nm::M3 r = nm::to_mat(q);
    nm::M3 m;
    for (int k = 0; k < 3; ++k) m.c[k] = V3{r.c[k].x / s, r.c[k].y / s, r.c[k].z / s};
    return m;
}

// compute_aabb(isometry): cuboid centre ± |R|·he (R = rotation matrix, columns = world directions of the local axes), sphere centre ± r
NM_HD inline void collider_aabb(int shape, V3 he, V3 p, Q q, V3& mn, V3& mx) {
    V3 e;
    if (shape == nm::SHAPE_SPHERE) {
        e = V3{he.x, he.x, he.x};
    } else {
        const nm::M3 r = rot_mat(q);
        e = V3{fabs(r.c[0].x) * he.x + fabs(r.c[1].x) * he.y + fabs(r.c[2].x) * he.z,
               fabs(r.c[0].y) * he.x + fabs(r.c[1].y) * he.y + fabs(r.c[2].y) * he.z,
               fabs(r.c[0].z) * he.x + fabs(r.c[1].z) * he.y + fabs(r.c[2].z) * he.z};
    }
    mn = p - e;
    mx = p + e;
}

// Aabb::intersects: inclusive on all three axes
template <class T>
NM_HD inline bool aabb_overlap(const T* amn, const T* amx, const T* bmn, const T* bmx) {
    return amn[0] <= bmx[0] && amx[0] >= bmn[0] && amn[1] <= bmx[1] && amx[1] >= bmn[1] && amn[2] <= bmx[2] && amx[2] >= bmn[2];
}

// ray vs cuboid in its own frame.  Returns false on a miss; t and n (world) otherwise, before the [0, max_distance] acceptance.
NM_HD inline bool ray_cuboid(V3 he, V3 p, Q q, V3 o, V3 d, bool solid, S& t, V3& n) {
    const nm::M3 r = rot_mat(q);
    const V3 rel = o - p;
    S tmin = -INFINITY, tmax = INFINITY;
    int ein = -1, eout = -1;
    S sin_ = 0, sout = 0;
    for (int k = 0; k < 3; ++k) {
        const S lo = nm::dot(rel, r.c[k]), ld = nm::dot(d, r.c[k]), h = nm::comp(he, k);
        if (ld == 0) {                       // parallel to this slab: in it or not, no parameter
            if (lo < -h || lo > h) return false;
            continue;
        }
        const S t1 = (-h - lo) / ld, t2 = (h - lo) / ld;
        const S tn = ld > 0 ? t1 : t2, tf = ld > 0 ? t2 : t1;
        const S sn = ld > 0 ? -1 : 1;        // outward normal sign of the face the ray enters through
        if (tn > tmin) { tmin = tn; ein = k; sin_ = sn; }
        if (tf < tmax) { tmax = tf; eout = k; sout = -sn; }
    }
    if (tmin > tmax) return false;
    if (tmin > 0) {                          // origin outside: the entering face
        t = tmin;
        n = r.c[ein] * sin_;
        return true;
    }
    if (tmax < 0) return false;              // the whole box lies behind the origin
    if (solid) { t = 0; n = V3{0, 0, 0}; return true; }
    if (eout < 0) return false;              // zero direction from inside: no exit
    t = tmax;
    n = r.c[eout] * sout;
    return true;
}

// ray vs sphere, closed form: a t² + 2 b t + c = 0 with a = d·d, b = (o - centre)·d, c = |o - centre|² - r²
NM_HD inline bool ray_sphere(S radius, V3 centre, V3 o, V3 d, bool solid, S& t, V3& n) {
    const V3 oc = o - centre;
    const S a = nm::dot(d, d), b = nm::dot(oc, d), c = nm::dot(oc, oc) - radius * radius;
    const bool inside = c <= 0;
    if (inside && solid) { t = 0; n = V3{0, 0, 0}; return true; }
    if (a == 0) return false;                // zero direction: never reaches the surface
    const S disc = b * b - a * c;
    if (disc < 0) return false;
    const S sq = sqrt(disc);
    if (inside) {
        t = (-b + sq) / a;                   // the exit
    } else {
        t = (-b - sq) / a;                   // the entry (both roots share a sign: negative = behind the origin)
        if (t < 0) return false;
    }
    const V3 h = oc + d * t;
    const S l = nm::len(h);
    n = l > 0 ? h * (1 / l) : V3{0, 0, 0};
    return true;
}

// one collider, acceptance included: hit when 0 <= t <= max_distance
NM_HD inline bool ray_collider(int shape, V3 he, V3 p, Q q, V3 o, V3 d, S max_distance, bool solid, S& t, V3& n) {
    const bool hit = shape == nm::SHAPE_SPHERE ? ray_sphere(he.x, p, o, d, solid, t, n) : ray_cuboid(he, p, q, o, d, solid, t, n);
    return hit && t >= 0 && t <= max_distance;
}

NM_HD inline bool ray_finite(V3 o, V3 d, S max_distance) { return finite3(o) && finite3(d) && std::isfinite(max_distance); }

// SpatialQueryFilter::test (query_filter.rs:97-101): layer mask and the excluded entities
NM_HD inline bool passes_filter(uint32_t memberships, uint32_t mask, const uint32_t* exclude, uint32_t exclude_count, uint32_t collider) {
    if ((memberships & mask) == 0) return false;
    for (uint32_t k = 0; k < exclude_count; ++k)
        if (exclude[k] == collider) return false;
    return true;
}

// (t, collider) lexicographic order: the closest hit and the order of a ray's hit list, independent of how the colliders were visited
NM_HD inline bool hit_before(S ta, uint32_t ca, S tb, uint32_t cb) { return ta < tb || (ta == tb && ca < cb); }

// ---- culling bounds of the device tree: f32, strictly larger than the tight double AABB -------------------------------------------------
// Each bound is rounded to f32 outward, then moved out by one f32 ulp of the larger of the axis' two bound magnitudes, so that even a bound
// that is exactly representable (a half extent of 0.5 at an integer position) or exactly 0 gets room for the rounding of the exact tests.
NM_HD inline float f32_down(double x) { float f = float(x); if (double(f) > x) f = nextafterf(f, -INFINITY); return f; }
NM_HD inline float f32_up(double x) { float f = float(x); if (double(f) < x) f = nextafterf(f, INFINITY); return f; }
NM_HD inline void culling_bounds(double lo, double hi, float& out_lo, float& out_hi) {
    const float l = f32_down(lo), h = f32_up(hi);
    const float m = fabsf(l) > fabsf(h) ? fabsf(l) : fabsf(h);
    const float u = std::isfinite(m) ? nextafterf(m, INFINITY) - m : 0.0f;
    out_lo = f32_down(double(l) - double(u));
    out_hi = f32_up(double(h) + double(u));
}

// where the ray enters a box, its parameter interval clipped to [0, tmax_clip]; INFINITY when that interval is empty.  The same
// zero-direction rule as ray_cuboid.  Used only to cull and to order the traversal.
NM_HD inline S ray_box_entry(const float* lo, const float* hi, V3 o, V3 d, S tmax_clip) {
    S t0 = 0, t1 = tmax_clip;
    for (int k = 0; k < 3; ++k) {
        const S ok = nm::comp(o, k), dk = nm::comp(d, k), l = lo[k], h = hi[k];
        if (dk == 0) {
            if (ok < l || ok > h) return INFINITY;
            continue;
        }
        S a = (l - ok) / dk, b = (h - ok) / dk;
        if (a > b) { S s = a; a = b; b = s; }
        t0 = nm::smax(t0, a);
        t1 = nm::smin(t1, b);
    }
    return t0 <= t1 ? t0 : INFINITY;
}

}  // namespace qm

// ---- host-side validation shared by the ABI (before any upload) and the host fixture --------------------------------------------------
#include "../../include/avian_b200.h"
namespace qm {
// NULL when the batch is usable; the reason otherwise
inline const char* check_rays(const AvnRayBatch* r) {
    if (!r) return "ray batch is required";
    if (r->count == 0) return nullptr;
    if (!r->origin || !r->direction || !r->max_distance) return "rays: origin, direction and max_distance are required";
    if (r->exclude_offsets) {           // (NULL: no ray excludes anything; exclude is then ignored)
        if (r->exclude_count && !r->exclude) return "rays: exclude_count > 0 needs exclude";
        for (uint32_t i = 0; i < r->count; ++i)
            if (r->exclude_offsets[i] > r->exclude_offsets[i + 1]) return "rays: exclude_offsets must be monotone";
        if (r->exclude_offsets[r->count] > r->exclude_count) return "rays: exclude_offsets run past exclude_count";
    }
    return nullptr;
}
inline const char* check_colliders(const AvnQueryColliders* c, bool shapes_required, bool f64) {
    if (!c) return "colliders are required";
    if (c->count >= 0x80000000u) return "colliders: at most 2^31 - 1";
    if (c->count == 0) return nullptr;
    if (!c->position || !c->rotation) return "colliders: position and rotation are required";
    if (shapes_required) {
        if (!c->shape || !c->dims) return "colliders: shape and dims are required";
        for (uint32_t i = 0; i < c->count; ++i) {
            if (c->shape[i] > AVN_SHAPE_SPHERE) return "colliders: unknown shape (only AVN_SHAPE_CUBOID and AVN_SHAPE_SPHERE)";
            for (int k = 0; k < (c->shape[i] == AVN_SHAPE_SPHERE ? 1 : 3); ++k) {
                const double v = f64 ? static_cast<const double*>(c->dims)[3 * size_t(i) + k] : static_cast<const float*>(c->dims)[3 * size_t(i) + k];
                if (v < 0) return "colliders: negative half extent or radius";
            }
        }
    }
    return nullptr;
}
}  // namespace qm
