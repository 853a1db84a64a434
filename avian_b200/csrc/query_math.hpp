// Spatial-query geometry for cuboid / sphere / capsule colliders, written once for the host fixture (g++, -ffp-contract=off) and for the device
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
//   * Capsules (DESIGN.md §7j): dims = [radius, half_length, unused], the segment from (0, -hl, 0) to (0, +hl, 0) of the collider frame, every
//     rotation through rot_mat.  AABB: the two posed segment ends, componentwise min / max, grown by the radius.  Ray vs capsule, closed form:
//     the infinite cylinder's quadratic (a = |d x u|², discriminant a r² - |(o - c) x u x (d x u)|², Lagrange's identity) kept when the root's
//     axial coordinate lies within [-hl, hl], and the two end spheres (a r² - |(o - e) x d|²); the smallest valid root (the largest exit for a
//     hollow ray from inside).  Normal: unit(hit - closest point of the segment).  half_length = 0 is a sphere, radius = 0 a closed segment.
//   Every capsule routine is out of line (NM_COLD) and compiled only into the CAPS = true instances of the templates below, so the cuboid /
//   sphere code is what it was before capsules were queried.
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

// capsule AABB: the segment ends p ∓ u·hl (u = rot_mat(q)'s local y), componentwise min / max, grown by the radius
NM_HD inline void capsule_aabb(V3 he, V3 p, Q q, V3& mn, V3& mx) {
    const V3 u = rot_mat(q).c[1];
    const V3 a = p - u * he.y, b = p + u * he.y;
    mn = V3{nm::smin(a.x, b.x) - he.x, nm::smin(a.y, b.y) - he.x, nm::smin(a.z, b.z) - he.x};
    mx = V3{nm::smax(a.x, b.x) + he.x, nm::smax(a.y, b.y) + he.x, nm::smax(a.z, b.z) + he.x};
}

// compute_aabb(isometry): cuboid centre ± |R|·he (R = rotation matrix, columns = world directions of the local axes), sphere centre ± r,
// capsule_aabb (CAPS only)
template <bool CAPS = false>
NM_HD inline void collider_aabb(int shape, V3 he, V3 p, Q q, V3& mn, V3& mx) {
    if (CAPS && shape == nm::SHAPE_CAPSULE) { capsule_aabb(he, p, q, mn, mx); return; }
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

// ray vs capsule: oc = origin - segment centre, u = unit axis, h = half length, r = radius.  Closed: a point at distance <= r from the segment is
// inside.  Outside: the smallest entry of the lateral surface (root kept when its axial coordinate lies in [-h, h]) and of the two end spheres;
// ties go to the lateral surface, then the -h end.  Inside and hollow: the largest exit of the same three (the capsule is convex, so the last
// exit is the capsule's).  The normal is unit(hit - closest segment point), 0 on the segment itself (radius 0).
NM_COLD inline bool ray_capsule_rel(V3 oc, V3 u, S h, S r, V3 d, bool solid, S& t, V3& n) {
    const S r2 = r * r;
    const S s0 = nm::smax(-h, nm::smin(h, nm::dot(oc, u)));
    const V3 e0 = oc - u * s0;
    const bool inside = nm::dot(e0, e0) <= r2;
    if (inside && solid) { t = 0; n = V3{0, 0, 0}; return true; }
    const S a = nm::dot(d, d);
    if (a == 0) return false;                // zero direction: never reaches the surface
    S best = inside ? -INFINITY : INFINITY;
    bool found = false;
    // lateral surface: |(oc + t d) x u|² = r²
    const V3 w = nm::cross(oc, u), v = nm::cross(d, u);
    const S al = nm::dot(v, v);
    if (al > 0) {
        const V3 x = nm::cross(w, v);
        const S disc = al * r2 - nm::dot(x, x);
        if (disc >= 0) {
            const S sq = sqrt(disc), b = nm::dot(w, v);
            const S tc = inside ? (-b + sq) / al : (-b - sq) / al;
            const S ax = nm::dot(oc + d * tc, u);
            if (ax >= -h && ax <= h && (inside || tc >= 0)) { best = tc; found = true; }
        }
    }
NM_ROLLED
    for (int i = 0; i < 2; ++i) {            // the end spheres at -h, +h
        const V3 oe = oc - u * (i == 0 ? -h : h);
        const V3 x = nm::cross(oe, d);
        const S disc = a * r2 - nm::dot(x, x);
        if (disc < 0) continue;
        const S sq = sqrt(disc), b = nm::dot(oe, d);
        if (inside) {
            const S te = (-b + sq) / a;
            if (te > best) { best = te; found = true; }
        } else {
            const S ts = (-b - sq) / a;
            if (ts >= 0 && ts < best) { best = ts; found = true; }
        }
    }
    if (!found || best < 0) return false;
    t = best;
    const V3 hp = oc + d * t;
    const V3 e = hp - u * nm::smax(-h, nm::smin(h, nm::dot(hp, u)));
    const S l = nm::len(e);
    n = l > 0 ? e * (1 / l) : V3{0, 0, 0};
    return true;
}
NM_HD inline bool ray_capsule(V3 he, V3 p, Q q, V3 o, V3 d, bool solid, S& t, V3& n) {
    return ray_capsule_rel(o - p, rot_mat(q).c[1], he.y, he.x, d, solid, t, n);
}

// one collider, acceptance included: hit when 0 <= t <= max_distance
template <bool CAPS = false>
NM_HD inline bool ray_collider(int shape, V3 he, V3 p, Q q, V3 o, V3 d, S max_distance, bool solid, S& t, V3& n) {
    const bool hit = CAPS && shape == nm::SHAPE_CAPSULE ? ray_capsule(he, p, q, o, d, solid, t, n)
                   : shape == nm::SHAPE_SPHERE          ? ray_sphere(he.x, p, o, d, solid, t, n)
                                                        : ray_cuboid(he, p, q, o, d, solid, t, n);
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

// ---- shape casts, point projection, point and shape intersections (cuboid / sphere / capsule) ------------------------------------------
// Reference call sites: spatial_query/pipeline.rs:315-615 (cast_shape, shape_hits, project_point), 617-683 (point_intersections), 731-826
// (shape_intersections), shape_caster.rs:335-400 (ShapeCaster::cast).  The reference hands the arithmetic to parry3d; these conventions are ours.
//
//   * Shape cast.  The cast shape A (pose c, q) moves along d; t is in units of |d|, as for rays.  The time of impact (TOI) with a collider B is
//     the smallest t in [0, max_distance] at which the closed shapes intersect.  target_distance is always 0 (the ABI refuses anything else).
//       - sphere-sphere: a solid ray cast of c against the sphere of radius rA + rB at B's centre.  The discriminant is evaluated as
//         a (rA + rB)² - |oc × d|² (Lagrange's identity), so it does not cancel for small radii.
//       - sphere-cuboid, cuboid-sphere: the sphere's centre (moving with +d, or with -d when the cuboid is cast) against the box rounded by
//         the radius, in the box's frame.  The times where the point crosses a slab face ±h_k split [0, inf) into at most 7 segments; on each
//         the squared distance to the box is one quadratic in t, and the first t where it reaches r² is its smaller root (the same identity
//         for the discriminant).  A segment whose every coordinate lies inside its slab is a hit at its start, which makes a radius-0 sphere
//         exact at the slab faces (the ray-like cast).
//       - cuboid-cuboid: a moving separating-axis test over the 15 axes in the fixed order A's 3 faces, B's 3 faces, A_i × B_j (i major);
//         an axis that is exactly zero is skipped.  On each axis the overlap is an interval of t (unnormalised); t_enter = the largest start
//         (ties to the lowest axis), t_exit = the smallest end.  Hit when t_enter <= t_exit, t_exit >= 0 and max(t_enter, 0) <= max_distance.
//     Origin penetration: TOI 0 (the shapes touch or overlap at t = 0).  Its normal is the axis of least penetration for boxes (depth / |axis|,
//     ties to the lowest axis), nm::box_sphere's inside rule for a sphere centre inside a box (the face of least depth, ties to the lowest
//     axis, + side when the coordinate is 0), the centre difference for two spheres (+y when the centres coincide).
//     Outputs (ShapeHitData, shape_caster.rs:562-592), world space: point1 / normal1 on the hit collider (normal1 outward, so it points towards
//     the cast shape), point2 / normal2 = -normal1 on the cast shape at its TOI pose.  Spheres: the centre-to-centre / closest-point
//     direction.  Box-box on a face axis: the face of the other box most anti-parallel to that face (the incident face) is clipped against the
//     reference face's side planes (nm::box_face / nm::clip_poly, as the narrow phase does); the witness is the clipped vertex nearest to the
//     reference plane (the first such vertex on a tie), projected onto that plane for the reference box's point.  Box-box on an edge axis: the
//     closest points of the two supporting edges.
//     AVN_CAST_IGNORE_ORIGIN_PENETRATION drops a TOI-0 collider when d · normal1 > 0 (the cast moves away from it);
//     AVN_CAST_NO_CONTACT_ON_PENETRATION writes the points and normals of a TOI-0 hit as 0.
//   * Point projection: cuboid = clamp in its frame, sphere = centre + r · unit(p - centre).  Closed shapes: the surface counts as inside.
//     Inside and solid -> the point itself, is_inside.  Inside and hollow -> the nearest face of a cuboid (ties to the lowest axis, then the
//     + side) or the sphere surface along p - centre (+y at the centre).  Distance = |projection - p|; the closest collider is the
//     lexicographic minimum of (distance, collider index).
//   * Point intersections: closed containment.  Shape intersections: exact separating-axis test for two cuboids (touching intersects; no bias),
//     closest point for sphere-cuboid, centre distance for two spheres.  Both apply the filter.
//   * A query shape with a non-finite pose, dims, direction or max_distance, or a zero quaternion, hits nothing; a point that is not finite
//     projects onto nothing and lies in nothing.  A sphere of radius 0 is legal.
//   * Capsules (CAPS = true instances only; DESIGN.md §7j).  Every cast kind with a capsule is an exact TOI on [0, max_distance]:
//       - sphere-capsule, capsule-sphere: a solid ray cast of the sphere's centre (+d, or -d when the capsule is cast) against the capsule grown
//         to rA + rB (ray_capsule_rel).
//       - capsule-capsule: the origin moving along d against the parallelogram P = (cB - cA) + {uB s - uA σ} grown by R = rA + rB
//         (seg_seg_toi): the minimum of the four edge casts (an end point of one segment against the other capsule of radius R, as a ray vs
//         capsule) and of the two faces of P offset by ±R along uA x uB, a face hit counting only inside P.  Parallel axes (uA x uB = 0) have
//         no face; the edge casts cover them.
//       - capsule-cuboid, cuboid-capsule: the capsule's two end points against the box rounded by r (point_rounded_box_toi) and the segment
//         against the box's 12 edges as segment-segment casts of radius r.  Exact: two convex shapes first touch at a feature pair, and a
//         segment's interior first touches a face's interior only when the two are parallel, when its end points touch at the same t.
//     Overlap at t = 0 (TOI 0): the closest-feature distance of the pair is at most the summed radii (segment-segment, segment-point,
//     segment-box with 0 when the segment meets the closed box).
//     Outputs: nm::capsule_round / nm::box_capsule at the TOI pose with no distance limit, so the normals and the fallbacks for coincident or
//     crossing axes are the narrow phase's (§7h).  A contact that is a continuum (parallel segments, a capsule lying on a face) has two
//     witnesses there; the first is reported: the end of the overlap at the lower parameter along the capsule's axis (A's axis for two
//     capsules).
//   * Capsule projection: the closest segment point + r · unit(p - closest); a point on the axis goes along the capsule's local +x.  Inside and
//     hollow: to the surface along p - closest.  Containment: dist(p, segment) <= r.  Intersections: capsule-sphere and capsule-capsule compare
//     the segment distance with the summed radii, capsule-cuboid the exact segment-box distance (0 when the segment meets the box) with r.

constexpr uint32_t CAST_IGNORE_ORIGIN_PENETRATION = 0x1u;   // = AVN_CAST_IGNORE_ORIGIN_PENETRATION
constexpr uint32_t CAST_NO_CONTACT_ON_PENETRATION = 0x2u;   // = AVN_CAST_NO_CONTACT_ON_PENETRATION

// half size of the tight AABB of a shape (collider_aabb's e; for a capsule |u|·hl + r, u = r.c[1])
template <bool CAPS = false>
NM_HD inline V3 half_size(int shape, V3 he, const nm::M3& r) {
    if (CAPS && shape == nm::SHAPE_CAPSULE)
        return V3{fabs(r.c[1].x) * he.y + he.x, fabs(r.c[1].y) * he.y + he.x, fabs(r.c[1].z) * he.y + he.x};
    if (shape == nm::SHAPE_SPHERE) return V3{he.x, he.x, he.x};
    return V3{fabs(r.c[0].x) * he.x + fabs(r.c[1].x) * he.y + fabs(r.c[2].x) * he.z,
              fabs(r.c[0].y) * he.x + fabs(r.c[1].y) * he.y + fabs(r.c[2].y) * he.z,
              fabs(r.c[0].z) * he.x + fabs(r.c[1].z) * he.y + fabs(r.c[2].z) * he.z};
}

NM_HD inline V3 to_local(const nm::M3& r, V3 v) { return V3{nm::dot(v, r.c[0]), nm::dot(v, r.c[1]), nm::dot(v, r.c[2])}; }
NM_HD inline V3 to_world(const nm::M3& r, V3 v) { return r.c[0] * v.x + r.c[1] * v.y + r.c[2] * v.z; }
NM_HD inline V3 clamp_box(V3 p, V3 h) {
    return V3{nm::smax(-h.x, nm::smin(h.x, p.x)), nm::smax(-h.y, nm::smin(h.y, p.y)), nm::smax(-h.z, nm::smin(h.z, p.z))};
}
NM_HD inline bool in_box(V3 p, V3 h) { return fabs(p.x) <= h.x && fabs(p.y) <= h.y && fabs(p.z) <= h.z; }
// squared distance from a local point to the box [-h, h]
NM_HD inline S box_d2(V3 p, V3 h) { const V3 e = p - clamp_box(p, h); return nm::dot(e, e); }

// the feature of the box [-h, h] nearest to the local point p: on_box and the outward unit normal there.  Outside: the clamp and the
// direction to p.  Inside (or on the surface with p == clamp): nm::box_sphere's inside rule, the face of least depth h_k - |p_k| (ties to the
// lowest axis, + side when p_k >= 0), on_box = p moved onto that face.
NM_HD inline void box_feature(V3 p, V3 h, V3& on_box, V3& n) {
    on_box = clamp_box(p, h);
    const V3 e = p - on_box;
    const S l = nm::len(e);
    if (l > 0) { n = e * (1 / l); return; }
    int ax = 0;
    S best = INFINITY;
    for (int k = 0; k < 3; ++k) {
        const S v = nm::comp(h, k) - fabs(nm::comp(p, k));
        if (v < best) { best = v; ax = k; }
    }
    const S sg = nm::comp(p, ax) >= 0 ? 1 : -1;
    n = V3{ax == 0 ? sg : 0, ax == 1 ? sg : 0, ax == 2 ? sg : 0};
    on_box = p;
    if (ax == 0) on_box.x = sg * h.x; else if (ax == 1) on_box.y = sg * h.y; else on_box.z = sg * h.z;
}

// sphere-sphere TOI: centre c moving along d against a sphere of radius R at p
NM_HD inline bool sphere_sphere_toi(V3 c, V3 d, V3 p, S R, S& t) {
    const V3 oc = c - p;
    const S cc = nm::dot(oc, oc) - R * R;
    if (cc <= 0) { t = 0; return true; }
    const S a = nm::dot(d, d), b = nm::dot(oc, d);
    if (a == 0 || b >= 0) return false;                  // not moving, or moving away from the centre
    const V3 x = nm::cross(oc, d);
    const S disc = a * (R * R) - nm::dot(x, x);
    if (disc < 0) return false;
    t = (-b - sqrt(disc)) / a;
    if (t < 0) t = 0;
    return true;
}

// rounded-box TOI: the local point p moving along v against the box [-h, h] rounded by r; t = 0 when it already lies within r
NM_HD inline bool point_rounded_box_toi(V3 p, V3 v, V3 h, S r, S maxd, S& t) {
    const S r2 = r * r;
    if (box_d2(p, h) <= r2) { t = 0; return true; }
    S bp[6];
    int nb = 0;
    for (int k = 0; k < 3; ++k) {
        const S pk = nm::comp(p, k), vk = nm::comp(v, k), hk = nm::comp(h, k);
        if (vk == 0) continue;
        const S a = (-hk - pk) / vk, b = (hk - pk) / vk;
        if (a > 0) bp[nb++] = a;
        if (b > 0) bp[nb++] = b;
    }
    for (int i = 1; i < nb; ++i)
        for (int j = i; j > 0 && bp[j] < bp[j - 1]; --j) { const S s = bp[j]; bp[j] = bp[j - 1]; bp[j - 1] = s; }
    S lo = 0;
    for (int i = 0; i <= nb; ++i) {
        const S hi = i < nb ? bp[i] : INFINITY;
        if (lo > maxd) return false;
        if (!(hi > lo)) continue;
        const S mid = hi == INFINITY ? lo + 1 : lo + (hi - lo) * 0.5;
        // per axis on this segment: the offset o_k of the face the point is outside of (p_k -/+ h_k), or inside the slab
        S o[3], w[3];
        bool out[3];
        S A = 0, B = 0, C = 0;
        for (int k = 0; k < 3; ++k) {
            const S pk = nm::comp(p, k), vk = nm::comp(v, k), hk = nm::comp(h, k), x = pk + mid * vk;
            out[k] = x > hk || x < -hk;
            o[k] = x > hk ? pk - hk : pk + hk;
            w[k] = vk;
            if (!out[k]) continue;
            A += vk * vk;
            B += o[k] * vk;
            C += o[k] * o[k];
        }
        if (A == 0) {
            if (C <= r2) { t = lo; return t <= maxd; }   // every moving coordinate inside its slab: within reach from the segment's start
        } else {
            // B² - A (C - r²) = A r² - sum over pairs of outside axes (o_i w_j - o_j w_i)²
            S disc = A * r2;
            for (int a = 0; a < 3; ++a)
                for (int b = a + 1; b < 3; ++b) {
                    if (!out[a] || !out[b]) continue;
                    const S x = o[a] * w[b] - o[b] * w[a];
                    disc = disc - x * x;
                }
            if (disc >= 0) {
                const S sq = sqrt(disc), rs = (-B - sq) / A, rl = (-B + sq) / A;
                if (rs <= hi && rl >= lo) { t = nm::smax(rs, lo); return t <= maxd; }
            }
        }
        lo = hi;
    }
    return false;
}

// the 15 separating axes of two boxes in the fixed order: A's faces, B's faces, A_i × B_j
NM_HD inline V3 sat_axis(const nm::M3& ra, const nm::M3& rb, int k) {
    if (k < 3) return ra.c[k];
    if (k < 6) return rb.c[k - 3];
    k -= 6;
    return nm::cross(ra.c[k / 3], rb.c[k % 3]);
}
NM_HD inline bool is_zero3(V3 v) { return v.x == 0 && v.y == 0 && v.z == 0; }
NM_HD inline S box_extent(const nm::M3& r, V3 he, V3 L) {
    return fabs(nm::dot(r.c[0], L)) * he.x + fabs(nm::dot(r.c[1], L)) * he.y + fabs(nm::dot(r.c[2], L)) * he.z;
}

// moving SAT: box A (ra, ha, ca) along d against box B.  axis = the entering axis, or at TOI 0 the axis of least penetration
NM_HD inline bool box_box_toi(const nm::M3& ra, V3 ha, V3 ca, V3 d, const nm::M3& rb, V3 hb, V3 cb, S maxd, S& t, int& axis) {
    const V3 s = cb - ca;
    S t_in = -INFINITY, t_out = INFINITY;
    int ax = -1;
    for (int k = 0; k < 15; ++k) {
        const V3 L = sat_axis(ra, rb, k);
        if (is_zero3(L)) continue;
        const S s0 = nm::dot(L, s), v = nm::dot(L, d), rho = box_extent(ra, ha, L) + box_extent(rb, hb, L);
        if (v == 0) {
            if (fabs(s0) > rho) return false;
            continue;
        }
        const S t1 = (s0 - rho) / v, t2 = (s0 + rho) / v;
        const S a = nm::smin(t1, t2), b = nm::smax(t1, t2);
        if (a > t_in) { t_in = a; ax = k; }
        if (b < t_out) t_out = b;
    }
    if (!(t_in <= t_out) || t_out < 0 || nm::smax(t_in, 0) > maxd) return false;
    if (t_in > 0) { t = t_in; axis = ax; return true; }
    t = 0;
    S best = INFINITY;
    for (int k = 0; k < 15; ++k) {
        const V3 L = sat_axis(ra, rb, k);
        if (is_zero3(L)) continue;
        const S pen = (box_extent(ra, ha, L) + box_extent(rb, hb, L) - fabs(nm::dot(L, s))) / nm::len(L);
        if (pen < best) { best = pen; axis = k; }
    }
    return true;
}

struct ShapeContact { V3 p1, p2, n1, n2; };

// witnesses of two boxes touching on SAT axis `axis`; n = unit normal from A to B
NM_HD inline void box_box_witness(const nm::Box& A, const nm::Box& B, int axis, V3 n, ShapeContact& c) {
    c.n1 = -n;
    c.n2 = n;
    if (axis >= 6) {                                     // edge-edge: closest points of the supporting edges
        const int i = (axis - 6) / 3, j = (axis - 6) % 3;
        const V3 ea = A.r.c[i], eb = B.r.c[j];
        V3 pa = A.c, pb = B.c;
        for (int k = 0; k < 3; ++k) {
            if (k != i) pa = pa + A.r.c[k] * (nm::comp(A.he, k) * (nm::dot(A.r.c[k], n) > 0 ? 1 : -1));
            if (k != j) pb = pb + B.r.c[k] * (nm::comp(B.he, k) * (nm::dot(B.r.c[k], n) < 0 ? 1 : -1));
        }
        const V3 r = pa - pb;
        const S a = nm::dot(ea, ea), e = nm::dot(eb, eb), f = nm::dot(eb, r), cc = nm::dot(ea, r), b = nm::dot(ea, eb);
        const S den = a * e - b * b;
        S s = den > 0 ? (b * f - cc * e) / den : 0;
        S u = (b * s + f) / e;
        const S ha = nm::comp(A.he, i), hb = nm::comp(B.he, j);
        s = nm::smax(-ha, nm::smin(ha, s));
        u = nm::smax(-hb, nm::smin(hb, u));
        c.p2 = pa + ea * s;
        c.p1 = pb + eb * u;
        return;
    }
    const bool ref_is_a = axis < 3;
    const nm::Box& R = ref_is_a ? A : B;
    const nm::Box& I = ref_is_a ? B : A;
    const int ra = axis % 3;
    const V3 rn = ref_is_a ? n : -n;                     // outward normal of the reference face
    int ia = 0;
    S ib = -1;
    for (int k = 0; k < 3; ++k) {
        const S v = fabs(nm::dot(I.r.c[k], rn));
        if (v > ib) { ib = v; ia = k; }
    }
    V3 poly[16], tmp[16];
    nm::box_face(I, ia, nm::dot(I.r.c[ia], rn) > 0 ? -1 : 1, poly);
    int np = 4;
    const int side[2] = {(ra + 1) % 3, (ra + 2) % 3};
    for (int a = 0; a < 2 && np > 0; ++a) {
        const V3 sn = R.r.c[side[a]];
        const S he = nm::comp(R.he, side[a]);
        np = nm::clip_poly(poly, np, sn, nm::dot(sn, R.c) + he, tmp);
        np = nm::clip_poly(tmp, np, -sn, -nm::dot(sn, R.c) + he, poly);
    }
    const S face_d = nm::dot(rn, R.c) + nm::comp(R.he, ra);
    V3 w;
    if (np > 0) {
        int best = 0;
        for (int k = 1; k < np; ++k)
            if (nm::dot(rn, poly[k]) < nm::dot(rn, poly[best])) best = k;
        w = poly[best];
    } else {                                             // clipped away by rounding: the incident box's support point towards the face
        w = I.c;
        for (int k = 0; k < 3; ++k) w = w + I.r.c[k] * (nm::comp(I.he, k) * (nm::dot(I.r.c[k], rn) > 0 ? -1 : 1));
    }
    const V3 on_ref = w - rn * (nm::dot(rn, w) - face_d);
    if (ref_is_a) { c.p2 = on_ref; c.p1 = w; } else { c.p1 = on_ref; c.p2 = w; }
}

// ---- capsule casts, contacts, projection and intersections (out of line: only the CAPS instances call them) ------------------------------

// squared distance from p (relative to the segment's centre) to the segment of unit axis u, half length h; the clamped parameter in s
NM_HD inline S segment_point_d2(V3 p, V3 u, S h, S& s) {
    s = nm::smax(-h, nm::smin(h, nm::dot(p, u)));
    const V3 e = p - u * s;
    return nm::dot(e, e);
}

// whether the segment of C meets the closed box b: its parameter interval clipped by the three slabs is not empty
NM_HD inline bool segment_meets_box(const nm::Box& b, const nm::Capsule& C) {
    S lo = -C.h, hi = C.h;
NM_ROLLED
    for (int k = 0; k < 3; ++k) {
        const S a = nm::dot(b.r.c[k], C.c - b.c), g = nm::dot(b.r.c[k], C.u), he = nm::comp(b.he, k);
        if (g == 0) {
            if (fabs(a) > he) return false;
            continue;
        }
        const S s0 = (-he - a) / g, s1 = (he - a) / g;
        lo = nm::smax(lo, nm::smin(s0, s1));
        hi = nm::smin(hi, nm::smax(s0, s1));
    }
    return lo <= hi;
}

// the exact distance between C's segment and the box b: 0 when they meet, else nm::segment_box_closest
NM_COLD inline S segment_box_distance(const nm::Box& b, const nm::Capsule& C) {
    if (segment_meets_box(b, C)) return 0;
    V3 on_seg, on_box;
    return nm::segment_box_closest(b, C, on_seg, on_box);
}

// The origin moving along d against P = c + {ub s - ua σ : |s| <= hb, |σ| <= ha} grown by R: the first t >= 0 at which the segment
// (0, ua, ha) moved by d t comes within R of the segment (c, ub, hb).  t = 0 when it already is.
NM_COLD inline bool seg_seg_toi(V3 c, V3 ua, S ha, V3 ub, S hb, S R, V3 d, S& t) {
    S s, u;
    nm::segment_closest(V3{0, 0, 0}, ua, ha, c, ub, hb, s, u);
    const V3 g = (c + ub * u) - ua * s;
    if (nm::dot(g, g) <= R * R) { t = 0; return true; }
    S best = INFINITY;
    V3 n;
NM_ROLLED
    for (int i = 0; i < 4; ++i) {            // the edges of P: B's ends -hb, +hb along ua, A's ends -ha, +ha along ub
        const bool b_end = i < 2;
        const S sg = (i & 1) ? 1 : -1;
        const V3 e = b_end ? c + ub * (sg * hb) : c - ua * (sg * ha);
        S ti;
        if (ray_capsule_rel(-e, b_end ? ua : ub, b_end ? ha : hb, R, d, true, ti, n) && ti < best) best = ti;
    }
    const V3 m = nm::cross(ua, ub);
    const S lm2 = nm::dot(m, m);
    if (lm2 > 0) {                           // the faces of P offset by ±R, entered from the side d comes from
        const V3 mn = m * (1 / sqrt(lm2));
        const S dn = nm::dot(d, mn);
        if (dn != 0) {
            const S tf = (nm::dot(c, mn) - (dn > 0 ? R : -R)) / dn;
            if (tf >= 0 && tf < best) {
                const V3 y = d * tf - c;
                const S yb = nm::dot(y, ub), ya = nm::dot(y, ua), cab = nm::dot(ua, ub);
                const S sb = (yb - cab * ya) / lm2, sa = (cab * yb - ya) / lm2;
                if (fabs(sb) <= hb && fabs(sa) <= ha) best = tf;
            }
        }
    }
    if (best == INFINITY) return false;
    t = best;
    return true;
}

// capsule C moving along v against the box b (rotation r): the end points against the rounded box, the segment against the 12 edges
NM_COLD inline bool capsule_box_toi(const nm::Capsule& C, const nm::Box& b, V3 v, S maxd, S& t) {
    if (segment_box_distance(b, C) <= C.r) { t = 0; return true; }
    S best = INFINITY;
    const V3 lv = to_local(b.r, v);
NM_ROLLED
    for (int i = 0; i < 2; ++i) {
        S ti;
        const V3 e = C.c + C.u * (i == 0 ? -C.h : C.h);
        if (point_rounded_box_toi(to_local(b.r, e - b.c), lv, b.he, C.r, maxd, ti) && ti < best) best = ti;
    }
NM_ROLLED
    for (int ei = 0; ei < 12; ++ei) {
        const int k = ei >> 2, m = ei & 3, u = (k + 1) % 3, w = (k + 2) % 3;
        const V3 ec = b.c + b.r.c[u] * (m & 1 ? nm::comp(b.he, u) : -nm::comp(b.he, u)) + b.r.c[w] * (m & 2 ? nm::comp(b.he, w) : -nm::comp(b.he, w));
        S ti;
        if (seg_seg_toi(ec - C.c, C.u, C.h, b.r.c[k], nm::comp(b.he, k), C.r, v, ti) && ti < best) best = ti;
    }
    if (best == INFINITY) return false;
    t = best;
    return true;
}

NM_HD inline nm::Capsule capsule_of(V3 he, V3 c, Q q) { return nm::Capsule{c, rot_mat(q).c[1], he.y, he.x}; }

// radius of a sphere about the centre that holds the shape
NM_HD inline S bounding_radius(int shape, V3 he) {
    if (shape == nm::SHAPE_CAPSULE) return he.x + he.y;
    if (shape == nm::SHAPE_SPHERE) return he.x;
    return nm::len(he);
}

// the TOI of a pair with at least one capsule (A moves along d).  First a conservative cull: the two bounding spheres, grown by 1e-6
// relative, never meet on [0, maxd] -> no hit (the constructions below are exact; the cull only skips them for far pairs).
NM_COLD inline bool capsule_cast_toi(int sa, V3 ha, V3 ca, Q qa, V3 d, S maxd, int sb, V3 hb, V3 cb, Q qb, S& t) {
    S tb;
    if (!sphere_sphere_toi(ca, d, cb, (bounding_radius(sa, ha) + bounding_radius(sb, hb)) * (1 + 1e-6), tb) || tb > maxd) return false;
    V3 n;
    if (sa == nm::SHAPE_SPHERE) return ray_capsule_rel(ca - cb, rot_mat(qb).c[1], hb.y, ha.x + hb.x, d, true, t, n);
    if (sb == nm::SHAPE_SPHERE) return ray_capsule_rel(cb - ca, rot_mat(qa).c[1], ha.y, ha.x + hb.x, -d, true, t, n);
    if (sa == nm::SHAPE_CAPSULE && sb == nm::SHAPE_CAPSULE)
        return seg_seg_toi(cb - ca, rot_mat(qa).c[1], ha.y, rot_mat(qb).c[1], hb.y, ha.x + hb.x, d, t);
    if (sa == nm::SHAPE_CAPSULE) return capsule_box_toi(capsule_of(ha, ca, qa), nm::Box{cb, rot_mat(qb), hb}, d, maxd, t);
    return capsule_box_toi(capsule_of(hb, cb, qb), nm::Box{ca, rot_mat(qa), ha}, -d, maxd, t);
}

// the contact of a capsule pair with A at `at`: the narrow phase's closest features with no distance limit, the first witness pair
NM_COLD inline void capsule_cast_contact(int sa, V3 ha, V3 at, Q qa, int sb, V3 hb, V3 cb, Q qb, ShapeContact& c) {
    nm::Contacts pts;
    pts.clear();
    V3 n{0, 1, 0};
    bool a_first;                            // whether pts / n run from A to B (else from B to A)
    if (sa == nm::SHAPE_CAPSULE && sb != nm::SHAPE_CUBOID) {
        const nm::Capsule A = capsule_of(ha, at, qa);
        if (sb == nm::SHAPE_CAPSULE) nm::capsule_round(A, cb, rot_mat(qb).c[1], hb.y, hb.x, INFINITY, n, pts);
        else nm::capsule_round(A, cb, A.u, 0, hb.x, INFINITY, n, pts);
        a_first = true;
    } else if (sa == nm::SHAPE_SPHERE) {     // B is the capsule
        const nm::Capsule B = capsule_of(hb, cb, qb);
        nm::capsule_round(B, at, B.u, 0, ha.x, INFINITY, n, pts);
        a_first = false;
    } else if (sa == nm::SHAPE_CAPSULE) {    // B is a cuboid: box_capsule runs from the box to the capsule
        nm::box_capsule(nm::Box{cb, rot_mat(qb), hb}, capsule_of(ha, at, qa), INFINITY, n, pts);
        a_first = false;
    } else {                                 // A is a cuboid, B the capsule
        nm::box_capsule(nm::Box{at, rot_mat(qa), ha}, capsule_of(hb, cb, qb), INFINITY, n, pts);
        a_first = true;
    }
    if (a_first) { c.n2 = n; c.n1 = -n; c.p2 = pts.p[0].a; c.p1 = pts.p[0].b; }
    else { c.n1 = n; c.n2 = -n; c.p1 = pts.p[0].a; c.p2 = pts.p[0].b; }
}

// project_point against a capsule
NM_COLD inline S capsule_project(V3 he, V3 c, Q q, V3 p, bool solid, V3& proj, bool& inside) {
    const nm::M3 r = rot_mat(q);
    S s;
    const V3 rel = p - c;
    const S l2 = segment_point_d2(rel, r.c[1], he.y, s);
    inside = l2 <= he.x * he.x;
    if (inside && solid) { proj = p; return 0; }
    const V3 foot = r.c[1] * s, e = rel - foot;
    const S l = sqrt(l2);
    proj = c + (l > 0 ? foot + e * (he.x / l) : foot + r.c[0] * he.x);
    return nm::len(proj - p);
}

// closed intersection of a pair with at least one capsule
NM_COLD inline bool capsule_intersect(int sa, V3 ha, V3 ca, Q qa, int sb, V3 hb, V3 cb, Q qb) {
    const bool a_cap = sa == nm::SHAPE_CAPSULE;
    const int so = a_cap ? sb : sa;
    const V3 hc = a_cap ? ha : hb, ho = a_cap ? hb : ha, cc = a_cap ? ca : cb, co = a_cap ? cb : ca;
    const Q qc = a_cap ? qa : qb, qo = a_cap ? qb : qa;
    const nm::Capsule C = capsule_of(hc, cc, qc);
    if (so == nm::SHAPE_SPHERE) {
        S s;
        const S R = hc.x + ho.x;
        return segment_point_d2(co - cc, C.u, C.h, s) <= R * R;
    }
    if (so == nm::SHAPE_CAPSULE) {
        S s, t;
        const V3 uo = rot_mat(qo).c[1];
        nm::segment_closest(cc, C.u, C.h, co, uo, ho.y, s, t);
        const V3 e = (co + uo * t) - (cc + C.u * s);
        const S R = hc.x + ho.x;
        return nm::dot(e, e) <= R * R;
    }
    return segment_box_distance(nm::Box{co, rot_mat(qo), ho}, C) <= C.r;
}

// The TOI of cast shape A against collider B (before the origin-penetration flag); axis: the box-box SAT axis the cast chose
template <bool CAPS = false>
NM_HD inline bool cast_toi(int sa, V3 ha, V3 ca, Q qa, V3 d, S maxd, int sb, V3 hb, V3 cb, Q qb, S& t, int& axis) {
    axis = -1;
    bool hit;
    if (CAPS && (sa == nm::SHAPE_CAPSULE || sb == nm::SHAPE_CAPSULE)) {
        hit = capsule_cast_toi(sa, ha, ca, qa, d, maxd, sb, hb, cb, qb, t);
    } else if (sa == nm::SHAPE_SPHERE && sb == nm::SHAPE_SPHERE) {
        hit = sphere_sphere_toi(ca, d, cb, ha.x + hb.x, t);
    } else if (sa == nm::SHAPE_SPHERE) {                 // the sphere's centre moves with +d against B's rounded box
        const nm::M3 r = rot_mat(qb);
        hit = point_rounded_box_toi(to_local(r, ca - cb), to_local(r, d), hb, ha.x, maxd, t);
    } else if (sb == nm::SHAPE_SPHERE) {                 // B's centre moves with -d against A's rounded box
        const nm::M3 r = rot_mat(qa);
        hit = point_rounded_box_toi(to_local(r, cb - ca), to_local(r, -d), ha, hb.x, maxd, t);
    } else {
        hit = box_box_toi(rot_mat(qa), ha, ca, d, rot_mat(qb), hb, cb, maxd, t, axis);
    }
    return hit && t <= maxd;
}

// points and normals of a cast hit at TOI t (A at ca + d t)
template <bool CAPS = false>
NM_HD inline void cast_contact(int sa, V3 ha, V3 ca, Q qa, V3 d, int sb, V3 hb, V3 cb, Q qb, S t, int axis, ShapeContact& c) {
    const V3 at = ca + d * t;
    if (CAPS && (sa == nm::SHAPE_CAPSULE || sb == nm::SHAPE_CAPSULE)) {
        capsule_cast_contact(sa, ha, at, qa, sb, hb, cb, qb, c);
    } else if (sa == nm::SHAPE_SPHERE && sb == nm::SHAPE_SPHERE) {
        const V3 e = at - cb;
        const S l = nm::len(e);
        c.n1 = l > 0 ? e * (1 / l) : V3{0, 1, 0};
        c.n2 = -c.n1;
        c.p1 = cb + c.n1 * hb.x;
        c.p2 = at + c.n2 * ha.x;
    } else if (sa == nm::SHAPE_SPHERE) {
        const nm::M3 r = rot_mat(qb);
        V3 on, n;
        box_feature(to_local(r, at - cb), hb, on, n);
        c.n1 = to_world(r, n);
        c.n2 = -c.n1;
        c.p1 = cb + to_world(r, on);
        c.p2 = at + c.n2 * ha.x;
    } else if (sb == nm::SHAPE_SPHERE) {
        const nm::M3 r = rot_mat(qa);
        V3 on, n;
        box_feature(to_local(r, cb - at), ha, on, n);
        c.n2 = to_world(r, n);
        c.n1 = -c.n2;
        c.p2 = at + to_world(r, on);
        c.p1 = cb + c.n1 * hb.x;
    } else {
        const nm::Box A{at, rot_mat(qa), ha}, B{cb, rot_mat(qb), hb};
        const V3 L = sat_axis(A.r, B.r, axis);
        // from A to B along the axis: the side B is entered from (t > 0), the side B's centre lies on (t = 0)
        const S side = t > 0 ? nm::dot(L, d) : nm::dot(L, cb - at);
        const V3 n = L * ((side >= 0 ? 1 : -1) / nm::len(L));
        box_box_witness(A, B, axis, n, c);
    }
}

// one collider, acceptance included: the TOI in [0, max_distance] and the origin-penetration flag
template <bool CAPS = false>
NM_HD inline bool cast_collider(int sa, V3 ha, V3 ca, Q qa, V3 d, S maxd, uint32_t flags, int sb, V3 hb, V3 cb, Q qb, S& t, int& axis) {
    if (!cast_toi<CAPS>(sa, ha, ca, qa, d, maxd, sb, hb, cb, qb, t, axis)) return false;
    if (t == 0 && (flags & CAST_IGNORE_ORIGIN_PENETRATION)) {
        ShapeContact c;
        cast_contact<CAPS>(sa, ha, ca, qa, d, sb, hb, cb, qb, t, axis, c);
        if (nm::dot(d, c.n1) > 0) return false;
    }
    return true;
}

// the outputs of a hit: its contact, or zeros for a TOI-0 hit with AVN_CAST_NO_CONTACT_ON_PENETRATION
template <bool CAPS = false>
NM_HD inline void cast_output(int sa, V3 ha, V3 ca, Q qa, V3 d, uint32_t flags, int sb, V3 hb, V3 cb, Q qb, S t, int axis, ShapeContact& c) {
    if (t == 0 && (flags & CAST_NO_CONTACT_ON_PENETRATION)) {
        c.p1 = c.p2 = c.n1 = c.n2 = V3{0, 0, 0};
        return;
    }
    cast_contact<CAPS>(sa, ha, ca, qa, d, sb, hb, cb, qb, t, axis, c);
}

NM_HD inline bool cast_finite(V3 he, V3 c, Q q, V3 d, S maxd) { return collider_valid(he, c, q) && finite3(d) && std::isfinite(maxd); }

// project_point against one collider: the projection, inside or not; returns |projection - p|
template <bool CAPS = false>
NM_HD inline S project_point(int shape, V3 he, V3 c, Q q, V3 p, bool solid, V3& proj, bool& inside) {
    if (CAPS && shape == nm::SHAPE_CAPSULE) return capsule_project(he, c, q, p, solid, proj, inside);
    if (shape == nm::SHAPE_SPHERE) {
        const V3 e = p - c;
        const S l2 = nm::dot(e, e);
        inside = l2 <= he.x * he.x;
        if (inside && solid) { proj = p; return 0; }
        const S l = sqrt(l2);
        proj = l > 0 ? c + e * (he.x / l) : c + V3{0, he.x, 0};
    } else {
        const nm::M3 r = rot_mat(q);
        const V3 lp = to_local(r, p - c);
        inside = in_box(lp, he);
        if (inside && solid) { proj = p; return 0; }
        V3 on = clamp_box(lp, he);
        if (inside) {                                    // the nearest face: ties to the lowest axis, then the + side
            int ax = 0;
            S best = INFINITY;
            for (int k = 0; k < 3; ++k) {
                const S v = nm::comp(he, k) - fabs(nm::comp(lp, k));
                if (v < best) { best = v; ax = k; }
            }
            const S sg = nm::comp(lp, ax) >= 0 ? 1 : -1;
            if (ax == 0) on.x = sg * he.x; else if (ax == 1) on.y = sg * he.y; else on.z = sg * he.z;
        }
        proj = c + to_world(r, on);
    }
    return nm::len(proj - p);
}

// closed containment
template <bool CAPS = false>
NM_HD inline bool contains_point(int shape, V3 he, V3 c, Q q, V3 p) {
    if (CAPS && shape == nm::SHAPE_CAPSULE) {
        S s;
        return segment_point_d2(p - c, rot_mat(q).c[1], he.y, s) <= he.x * he.x;
    }
    if (shape == nm::SHAPE_SPHERE) {
        const V3 e = p - c;
        return nm::dot(e, e) <= he.x * he.x;
    }
    return in_box(to_local(rot_mat(q), p - c), he);
}

// closed intersection of two posed shapes
template <bool CAPS = false>
NM_HD inline bool shapes_intersect(int sa, V3 ha, V3 ca, Q qa, int sb, V3 hb, V3 cb, Q qb) {
    if (CAPS && (sa == nm::SHAPE_CAPSULE || sb == nm::SHAPE_CAPSULE)) return capsule_intersect(sa, ha, ca, qa, sb, hb, cb, qb);
    if (sa == nm::SHAPE_SPHERE && sb == nm::SHAPE_SPHERE) {
        const V3 e = ca - cb;
        const S R = ha.x + hb.x;
        return nm::dot(e, e) <= R * R;
    }
    if (sa == nm::SHAPE_SPHERE || sb == nm::SHAPE_SPHERE) {
        const bool a_sphere = sa == nm::SHAPE_SPHERE;
        const nm::M3 r = rot_mat(a_sphere ? qb : qa);
        const V3 lp = to_local(r, a_sphere ? ca - cb : cb - ca);
        const S rad = a_sphere ? ha.x : hb.x;
        return box_d2(lp, a_sphere ? hb : ha) <= rad * rad;
    }
    const nm::M3 ra = rot_mat(qa), rb = rot_mat(qb);
    const V3 s = cb - ca;
    for (int k = 0; k < 15; ++k) {
        const V3 L = sat_axis(ra, rb, k);
        if (is_zero3(L)) continue;
        if (fabs(nm::dot(L, s)) > box_extent(ra, ha, L) + box_extent(rb, hb, L)) return false;
    }
    return true;
}

// squared distance from a point to a culling box (0 inside)
NM_HD inline S point_box_d2(const float* lo, const float* hi, V3 p) {
    S s = 0;
    for (int k = 0; k < 3; ++k) {
        const S x = nm::comp(p, k), e = x < lo[k] ? S(lo[k]) - x : (x > hi[k] ? x - S(hi[k]) : 0);
        s += e * e;
    }
    return s;
}

}  // namespace qm

// ---- host-side validation shared by the ABI (before any upload) and the host fixture --------------------------------------------------
#include "../../include/avian_b200.h"
#include "shape_column.hpp"
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
// the dims a shape reads: a cuboid's three half extents, a sphere's radius, a capsule's radius and half length
inline int shape_dims_read(uint8_t shape) { return shape == AVN_SHAPE_SPHERE ? 1 : (shape == AVN_SHAPE_CAPSULE ? 2 : 3); }
// capsules: whether AVN_SHAPE_CAPSULE is accepted; saw_capsule (optional): set when the column holds one.  hull_count (the hull instances'
// callers): AVN_SHAPE_CONVEX_HULL is accepted too, its index checked by avn::check_shape_column against *hull_count (0: no table);
// saw_hull / max_hull (optional): whether the column holds a hull, and the largest index it names.
inline const char* check_colliders(const AvnQueryColliders* c, bool shapes_required, bool f64, bool capsules = false, bool* saw_capsule = nullptr,
                                   const uint32_t* hull_count = nullptr, bool* saw_hull = nullptr, uint32_t* max_hull = nullptr) {
    if (saw_capsule) *saw_capsule = false;
    if (saw_hull) *saw_hull = false;
    if (max_hull) *max_hull = 0;
    if (!c) return "colliders are required";
    if (c->count >= 0x80000000u) return "colliders: at most 2^31 - 1";
    if (c->count == 0) return nullptr;
    if (!c->position || !c->rotation) return "colliders: position and rotation are required";
    if (shapes_required) {
        if (!c->shape || !c->dims) return "colliders: shape and dims are required";
        for (uint32_t i = 0; i < c->count; ++i) {
            if (hull_count && c->shape[i] == AVN_SHAPE_CONVEX_HULL) continue;   // its index: below
            if (!capsules && c->shape[i] > AVN_SHAPE_SPHERE) return "colliders: unknown shape (only AVN_SHAPE_CUBOID and AVN_SHAPE_SPHERE)";
            if (c->shape[i] > AVN_SHAPE_CAPSULE) return "colliders: unknown shape (only AVN_SHAPE_CUBOID, AVN_SHAPE_SPHERE and AVN_SHAPE_CAPSULE)";
            for (int k = 0; k < shape_dims_read(c->shape[i]); ++k) {
                const double v = f64 ? static_cast<const double*>(c->dims)[3 * size_t(i) + k] : static_cast<const float*>(c->dims)[3 * size_t(i) + k];
                if (v < 0) return "colliders: negative half extent, radius or half length";
            }
            if (saw_capsule && c->shape[i] == AVN_SHAPE_CAPSULE) *saw_capsule = true;
        }
        size_t at;
        if (hull_count)
            if (const char* why = avn::check_shape_column(c->shape, c->dims, c->count, f64 ? 64 : 32, &at, nullptr, hull_count, saw_hull, max_hull))
                return why;
    }
    return nullptr;
}
// the exclusion CSR of a shape or point batch
inline const char* check_exclusions(uint32_t count, uint32_t exclude_count, const uint32_t* offsets, const uint32_t* exclude) {
    if (!offsets) return nullptr;       // (NULL: no query excludes anything; exclude is then ignored)
    if (exclude_count && !exclude) return "exclude_count > 0 needs exclude";
    for (uint32_t i = 0; i < count; ++i)
        if (offsets[i] > offsets[i + 1]) return "exclude_offsets must be monotone";
    if (offsets[count] > exclude_count) return "exclude_offsets run past exclude_count";
    return nullptr;
}
// cast: the batch feeds a shape cast (direction and max_distance required, target_distance must be 0); hull_count / saw_hull: as check_colliders
inline const char* check_shapes(const AvnShapeBatch* s, bool cast, bool f64, bool capsules = false, bool* saw_capsule = nullptr,
                                const uint32_t* hull_count = nullptr, bool* saw_hull = nullptr) {
    if (saw_capsule) *saw_capsule = false;
    if (saw_hull) *saw_hull = false;
    if (!s) return "shape batch is required";
    if (s->count >= 0x7fffffffu) return "shapes: too many shapes";
    if (s->count == 0) return nullptr;
    if (!s->shape || !s->dims || !s->position || !s->rotation) return "shapes: shape, dims, position and rotation are required";
    if (cast && (!s->direction || !s->max_distance)) return "shapes: direction and max_distance are required for a cast";
    for (uint32_t i = 0; i < s->count; ++i) {
        const bool hull = hull_count && s->shape[i] == AVN_SHAPE_CONVEX_HULL;   // its index: below
        if (!hull && !capsules && s->shape[i] > AVN_SHAPE_SPHERE) return "shapes: unknown shape (only AVN_SHAPE_CUBOID and AVN_SHAPE_SPHERE)";
        if (!hull && s->shape[i] > AVN_SHAPE_CAPSULE) return "shapes: unknown shape (only AVN_SHAPE_CUBOID, AVN_SHAPE_SPHERE and AVN_SHAPE_CAPSULE)";
        for (int k = 0; !hull && k < shape_dims_read(s->shape[i]); ++k) {
            const double v = f64 ? static_cast<const double*>(s->dims)[3 * size_t(i) + k] : static_cast<const float*>(s->dims)[3 * size_t(i) + k];
            if (v < 0) return "shapes: negative half extent, radius or half length";
        }
        if (saw_capsule && s->shape[i] == AVN_SHAPE_CAPSULE) *saw_capsule = true;
        if (cast && s->target_distance) {
            const double td = f64 ? static_cast<const double*>(s->target_distance)[i] : static_cast<const float*>(s->target_distance)[i];
            if (td != 0) return "shapes: target_distance must be 0 (a cast with a target distance is not supported)";
        }
    }
    size_t at;
    if (hull_count)
        if (const char* why = avn::check_shape_column(s->shape, s->dims, s->count, f64 ? 64 : 32, &at, nullptr, hull_count, saw_hull)) return why;
    if (const char* why = check_exclusions(s->count, s->exclude_count, s->exclude_offsets, s->exclude)) return why;
    return nullptr;
}
inline const char* check_points(const AvnPointBatch* p) {
    if (!p) return "point batch is required";
    if (p->count >= 0x7fffffffu) return "points: too many points";
    if (p->count == 0) return nullptr;
    if (!p->point) return "points: point is required";
    return check_exclusions(p->count, p->exclude_count, p->exclude_offsets, p->exclude);
}
}  // namespace qm
