// Spatial-query geometry for convex hull colliders and query shapes (DESIGN.md §7l), written once for the host fixture (g++, -ffp-contract=off)
// and for the device (nvcc, -fmad=false) like query_math.hpp and hull_math.hpp, on which it builds: IEEE double throughout, the same
// expressions in the same order, so csrc/queries.cu's hull instances and the host brute force report the same bits.  parry is not vendored:
// there is no parity claim against parry, only this contract.
//
// What "the hull" is (repeated in DESIGN.md §7l):
//   * The ray test, containment, the projection from inside and the faces of a rounded hull use the table's face planes (Newell normal, mean
//     offset; hull_table.hpp): a point is inside when no face plane has it above (closed).
//   * A hull's extent along a separating axis is the maximum (minimum) over its posed vertices.
//   * The tight AABB is the posed vertices' min / max (rounded to the column scalar for output and the AABB test).  Vertices lie up to
//     AVN_HULL_REL_TOL x size off their planes, so the tree culls a hull against the box of its bounding ball instead: the table's radius about
//     the collider's position, grown by CULL_GROW of itself.  That box holds the vertices and, with room to spare, the face-plane polytope
//     (it exceeds the vertex hull by at most a few tolerances near a vertex).  half_size, which culls casts, is the same symmetric bound.
//   * Every hull is posed through qm::rot_mat (hm::table_hull_at); a cuboid paired with a hull becomes hm::box_hull's 8-vertex hull.
// The entry points below take the hull table and forward every pair without a hull to query_math.hpp's CAPS = true geometry, so a hull
// instance gives the capsule instance's bits on cuboids, spheres and capsules.  Every hull routine is out of line (NM_COLD) and compiled only
// into the hull instances.
#pragma once
#include <cmath>
#include <cstdint>

#include "hull_math.hpp"
#include "query_math.hpp"

namespace qh {

using nm::S;
using nm::V3;
using nm::Q;
using nm::M3;
using hm::Hull;
using hm::Table;

constexpr int SHAPE_HULL = hm::SHAPE_CONVEX_HULL;
constexpr S CULL_GROW = 1e-3;     // culling ball: the hull radius grown by this much of itself

NM_HD inline uint32_t hull_index(V3 he) { return uint32_t(he.x); }
NM_HD inline M3 identity() { M3 m; m.c[0] = V3{1, 0, 0}; m.c[1] = V3{0, 1, 0}; m.c[2] = V3{0, 0, 1}; return m; }
NM_HD inline bool is_poly(int shape) { return shape == SHAPE_HULL || shape == nm::SHAPE_CUBOID; }

// a hull or a cuboid (as hm::box_hull, storage in bh) posed at (c, r)
NM_HD inline Hull polytope(const Table& t, hm::BoxHull& bh, int shape, V3 he, V3 c, const M3& r) {
    if (shape == SHAPE_HULL) return hm::table_hull_at(t, hull_index(he), c, r);
    Hull H = hm::box_hull(bh, he, c, Q{0, 0, 0, 1});
    H.r = r;
    return H;
}

// ---- AABB and culling bounds -------------------------------------------------------------------------------------------------------------
NM_COLD inline void hull_aabb(const Table& t, V3 he, V3 p, Q q, V3& mn, V3& mx) {
    const Hull H = hm::table_hull_at(t, hull_index(he), p, qm::rot_mat(q));
    mn = mx = hm::vtx(H, 0);
NM_ROLLED
    for (int k = 1; k < H.nv; ++k) {
        const V3 v = hm::vtx(H, k);
        mn = V3{nm::smin(mn.x, v.x), nm::smin(mn.y, v.y), nm::smin(mn.z, v.z)};
        mx = V3{nm::smax(mx.x, v.x), nm::smax(mx.y, v.y), nm::smax(mx.z, v.z)};
    }
}
NM_HD inline S cull_radius(const Table& t, V3 he) { return t.radius[hull_index(he)] * (1 + CULL_GROW); }

// the tight AABB (qm::collider_aabb for the other shapes)
NM_HD inline void collider_aabb(const Table& t, int shape, V3 he, V3 p, Q q, V3& mn, V3& mx) {
    if (shape == SHAPE_HULL) { hull_aabb(t, he, p, q, mn, mx); return; }
    qm::collider_aabb<true>(shape, he, p, q, mn, mx);
}
// the box the tree culls against (before qm::culling_bounds): the tight AABB, the bounding ball's box for a hull
NM_HD inline void cull_box(const Table& t, int shape, V3 he, V3 p, V3 mn, V3 mx, V3& lo, V3& hi) {
    if (shape == SHAPE_HULL) {
        const S R = cull_radius(t, he);
        lo = V3{p.x - R, p.y - R, p.z - R};
        hi = V3{p.x + R, p.y + R, p.z + R};
        return;
    }
    lo = mn;
    hi = mx;
}
// a conservative half size about the shape's position (casts cull with it)
NM_HD inline V3 half_size(const Table& t, int shape, V3 he, const M3& r) {
    if (shape == SHAPE_HULL) { const S R = cull_radius(t, he); return V3{R, R, R}; }
    return qm::half_size<true>(shape, he, r);
}
NM_HD inline S bounding_radius(const Table& t, int shape, V3 he) { return shape == SHAPE_HULL ? t.radius[hull_index(he)] : qm::bounding_radius(shape, he); }

// ---- ray vs hull: Cyrus-Beck over the face planes in the hull's frame, ray_cuboid's rules -------------------------------------------------
NM_COLD inline bool ray_hull(const Table& t, V3 he, V3 p, Q q, V3 o, V3 d, bool solid, S& tt, V3& n) {
    const M3 r = qm::rot_mat(q);
    const Hull H = hm::table_hull_at(t, hull_index(he), V3{0, 0, 0}, identity());
    const V3 lo = qm::to_local(r, o - p), ld = qm::to_local(r, d);
    S tmin = -INFINITY, tmax = INFINITY;
    int ein = -1, eout = -1;
NM_ROLLED
    for (int f = 0; f < H.nf; ++f) {
        const V3 nf{H.pl[4 * f], H.pl[4 * f + 1], H.pl[4 * f + 2]};
        const S h = nm::dot(nf, lo) - H.pl[4 * f + 3], den = nm::dot(nf, ld);
        if (den == 0) {                      // parallel to this plane: above it misses, below it leaves the face unconstrained
            if (h > 0) return false;
            continue;
        }
        const S tf = -h / den;
        if (den < 0) {
            if (tf > tmin) { tmin = tf; ein = f; }
        } else if (tf < tmax) {
            tmax = tf; eout = f;
        }
    }
    if (tmin > tmax) return false;
    if (tmin > 0) {
        tt = tmin;
        n = qm::to_world(r, V3{H.pl[4 * ein], H.pl[4 * ein + 1], H.pl[4 * ein + 2]});
        return true;
    }
    if (tmax < 0) return false;
    if (solid) { tt = 0; n = V3{0, 0, 0}; return true; }
    if (eout < 0) return false;
    tt = tmax;
    n = qm::to_world(r, V3{H.pl[4 * eout], H.pl[4 * eout + 1], H.pl[4 * eout + 2]});
    return true;
}
NM_HD inline bool ray_collider(const Table& t, int shape, V3 he, V3 p, Q q, V3 o, V3 d, S max_distance, bool solid, S& tt, V3& n) {
    if (shape == SHAPE_HULL) return ray_hull(t, he, p, q, o, d, solid, tt, n) && tt >= 0 && tt <= max_distance;
    return qm::ray_collider<true>(shape, he, p, q, o, d, max_distance, solid, tt, n);
}

// ---- points ----------------------------------------------------------------------------------------------------------------------------
// the largest signed distance of the local point x to a face plane of H (ties to the lowest face), and that face
NM_HD inline S max_plane(const Hull& H, V3 x, int& fb) {
    S hb = -INFINITY;
    fb = 0;
NM_ROLLED
    for (int f = 0; f < H.nf; ++f) {
        const S h = nm::dot(hm::fnormal(H, f), x) - hm::foffset(H, f);
        if (h > hb) { hb = h; fb = f; }
    }
    return hb;
}
NM_COLD inline bool hull_contains(const Table& t, V3 he, V3 c, Q q, V3 p) {
    const Hull H = hm::table_hull_at(t, hull_index(he), V3{0, 0, 0}, identity());
    int fb;
    return max_plane(H, qm::to_local(qm::rot_mat(q), p - c), fb) <= 0;
}
// outside: hm::point_hull_closest; inside and solid: p; inside and hollow: onto the plane of the face of largest signed distance
NM_COLD inline S hull_project(const Table& t, V3 he, V3 c, Q q, V3 p, bool solid, V3& proj, bool& inside) {
    const M3 r = qm::rot_mat(q);
    const Hull H = hm::table_hull_at(t, hull_index(he), V3{0, 0, 0}, identity());
    const V3 lp = qm::to_local(r, p - c);
    int fb;
    const S hb = max_plane(H, lp, fb);
    inside = hb <= 0;
    if (inside && solid) { proj = p; return 0; }
    V3 on;
    if (inside) on = lp - hm::fnormal(H, fb) * hb;
    else hm::point_hull_closest(H, lp, on);
    proj = c + qm::to_world(r, on);
    return nm::len(proj - p);
}
NM_HD inline S project_point(const Table& t, int shape, V3 he, V3 c, Q q, V3 p, bool solid, V3& proj, bool& inside) {
    if (shape == SHAPE_HULL) return hull_project(t, he, c, q, p, solid, proj, inside);
    return qm::project_point<true>(shape, he, c, q, p, solid, proj, inside);
}
NM_HD inline bool contains_point(const Table& t, int shape, V3 he, V3 c, Q q, V3 p) {
    if (shape == SHAPE_HULL) return hull_contains(t, he, c, q, p);
    return qm::contains_point<true>(shape, he, c, q, p);
}

// ---- two polytopes: the separating axes ------------------------------------------------------------------------------------------------
// Axis k of the pair (A, B) in the fixed order: A's faces, B's faces, then edge pair (i, j) of A's edge i and B's edge j at nf_A + nf_B +
// i ne_B + j.  An edge pair is an axis when its arcs cross on the Gauss map (hm::minkowski_face) and the cross product of the unit edge
// directions is at least 1e-9 long (hm::hull_hull's rule); the axis is that cross product, not normalised.
NM_HD inline int axis_count(const Hull& A, const Hull& B) { return A.nf + B.nf + A.ne * B.ne; }
NM_HD inline V3 axis_vec(const Hull& A, const Hull& B, int k) {
    if (k < A.nf) return hm::fnormal(A, k);
    if (k < A.nf + B.nf) return hm::fnormal(B, k - A.nf);
    k -= A.nf + B.nf;
    V3 ma, ua, mb, ub;
    S ha, hb;
    hm::edge_seg(A, k / B.ne, ma, ua, ha);
    hm::edge_seg(B, k % B.ne, mb, ub, hb);
    return nm::cross(ua, ub);
}
NM_HD inline bool sat_axis(const Hull& A, const Hull& B, int k, V3& L) {
    if (k >= A.nf + B.nf) {
        const int e = k - A.nf - B.nf, i = e / B.ne, j = e % B.ne;
        if (!hm::minkowski_face(hm::fnormal(A, int(A.edge[4 * i + 2])), hm::fnormal(A, int(A.edge[4 * i + 3])), -hm::fnormal(B, int(B.edge[4 * j + 2])),
                                -hm::fnormal(B, int(B.edge[4 * j + 3]))))
            return false;
    }
    L = axis_vec(A, B, k);
    return k < A.nf + B.nf || !(nm::len(L) < 1e-9);
}
// [lo, hi] of the posed vertices along L
NM_HD inline void extent(const Hull& H, V3 L, S& lo, S& hi) {
    lo = INFINITY;
    hi = -INFINITY;
NM_ROLLED
    for (int k = 0; k < H.nv; ++k) {
        const S x = nm::dot(L, hm::vtx(H, k));
        lo = nm::smin(lo, x);
        hi = nm::smax(hi, x);
    }
}

// Moving SAT: A moves along d against B (both posed at t = 0), box_box_toi's interval, tie and hit rules.  axis = the entering axis, or at
// TOI 0 the axis of least penetration (depth min(hi_A - lo_B, hi_B - lo_A) / |L|, ties to the lowest axis).
NM_COLD inline bool poly_toi(const Hull& A, const Hull& B, V3 d, S maxd, S& tt, int& axis) {
    S t_in = -INFINITY, t_out = INFINITY;
    int ax = -1;
    const int n = axis_count(A, B);
NM_ROLLED
    for (int k = 0; k < n; ++k) {
        V3 L;
        if (!sat_axis(A, B, k, L)) continue;
        S alo, ahi, blo, bhi;
        extent(A, L, alo, ahi);
        extent(B, L, blo, bhi);
        const S v = nm::dot(L, d);
        if (v == 0) {
            if (blo - ahi > 0 || bhi - alo < 0) return false;
            continue;
        }
        const S t1 = (blo - ahi) / v, t2 = (bhi - alo) / v;
        const S a = nm::smin(t1, t2), b = nm::smax(t1, t2);
        if (a > t_in) { t_in = a; ax = k; }
        if (b < t_out) t_out = b;
    }
    if (!(t_in <= t_out) || t_out < 0 || nm::smax(t_in, 0) > maxd) return false;
    if (t_in > 0) { tt = t_in; axis = ax; return true; }
    tt = 0;
    S best = INFINITY;
NM_ROLLED
    for (int k = 0; k < n; ++k) {
        V3 L;
        if (!sat_axis(A, B, k, L)) continue;
        S alo, ahi, blo, bhi;
        extent(A, L, alo, ahi);
        extent(B, L, blo, bhi);
        const S pen = nm::smin(ahi - blo, bhi - alo) / nm::len(L);
        if (pen < best) { best = pen; axis = k; }
    }
    return true;
}
// static SAT: touching intersects, no bias
NM_COLD inline bool poly_intersect(const Hull& A, const Hull& B) {
    const int n = axis_count(A, B);
NM_ROLLED
    for (int k = 0; k < n; ++k) {
        V3 L;
        if (!sat_axis(A, B, k, L)) continue;
        S alo, ahi, blo, bhi;
        extent(A, L, alo, ahi);
        extent(B, L, blo, bhi);
        if (blo - ahi > 0 || bhi - alo < 0) return false;
    }
    return true;
}

// Witnesses of two polytopes touching on axis k (A at its TOI pose).  The normal runs from A to B: along the entering axis the side A
// moves to (t > 0); at TOI 0 the side of least penetration.  Face axis: the face of the other polytope most anti-parallel to the reference
// face (the first on a tie) clipped by the reference face's side planes (hm::clip_bounded); the witness is the clipped vertex nearest the
// reference plane (the first on a tie), projected onto that plane for the reference polytope's point.  When the reference face does not face
// the other polytope, or clipping leaves nothing, the witness is the other polytope's support vertex towards the reference (the first on a
// tie), projected onto the reference polytope's support plane.  Edge axis: the closest points of the two edges.
NM_COLD inline void poly_witness(const Hull& A, const Hull& B, int k, V3 d, S tt, qm::ShapeContact& c) {
    const V3 L = axis_vec(A, B, k);
    S side;
    if (tt > 0) {
        side = nm::dot(L, d);
    } else {
        S alo, ahi, blo, bhi;
        extent(A, L, alo, ahi);
        extent(B, L, blo, bhi);
        side = ahi - blo <= bhi - alo ? 1 : -1;
    }
    const V3 n = L * ((side >= 0 ? 1 : -1) / nm::len(L));
    c.n1 = -n;
    c.n2 = n;
    if (k >= A.nf + B.nf) {
        const int e = k - A.nf - B.nf;
        V3 ma, ua, mb, ub;
        S ha, hb, s, u;
        hm::edge_seg(A, e / B.ne, ma, ua, ha);
        hm::edge_seg(B, e % B.ne, mb, ub, hb);
        nm::segment_closest(ma, ua, ha, mb, ub, hb, s, u);
        c.p2 = ma + ua * s;
        c.p1 = mb + ub * u;
        return;
    }
    const bool ref_is_a = k < A.nf;
    const Hull& R = ref_is_a ? A : B;
    const Hull& I = ref_is_a ? B : A;
    const int rf = ref_is_a ? k : k - A.nf;
    const V3 rn = ref_is_a ? n : -n;                     // from the reference polytope towards the other
    V3 poly[hm::MAX_CLIP], tmp[hm::MAX_CLIP];
    int np = 0;
    const V3 fn = hm::fnormal(R, rf);
    if (nm::dot(fn, rn) > 0) {
        int inc = 0;
        S ib = INFINITY;
NM_ROLLED
        for (int f = 0; f < I.nf; ++f) {
            const S v = nm::dot(hm::fnormal(I, f), fn);
            if (v < ib) { ib = v; inc = f; }
        }
        np = hm::fsize(I, inc);
NM_ROLLED
        for (int i = 0; i < np; ++i) poly[i] = hm::fvtx(I, inc, i);
        const int m = hm::fsize(R, rf);
NM_ROLLED
        for (int i = 0; i < m && np > 0; ++i) {
            const V3 a = hm::fvtx(R, rf, i), b = hm::fvtx(R, rf, (i + 1) % m);
            const V3 sn = nm::cross(b - a, fn);
            np = hm::clip_bounded(poly, np, sn, nm::dot(sn, a), tmp);
NM_ROLLED
            for (int q = 0; q < np; ++q) poly[q] = tmp[q];
        }
    }
    V3 w, pn;
    S plane_d;
    if (np > 0) {                                        // the reference face's plane
        int best = 0;
NM_ROLLED
        for (int q = 1; q < np; ++q)
            if (nm::dot(fn, poly[q]) < nm::dot(fn, poly[best])) best = q;
        w = poly[best];
        pn = fn;
        plane_d = hm::foffset(R, rf);
    } else {                                             // the reference polytope's support plane along rn
        int bi = 0, br = 0;
NM_ROLLED
        for (int q = 1; q < I.nv; ++q)
            if (nm::dot(rn, hm::vtx(I, q)) < nm::dot(rn, hm::vtx(I, bi))) bi = q;
NM_ROLLED
        for (int q = 1; q < R.nv; ++q)
            if (nm::dot(rn, hm::vtx(R, q)) > nm::dot(rn, hm::vtx(R, br))) br = q;
        w = hm::vtx(I, bi);
        pn = rn;
        plane_d = nm::dot(rn, hm::vtx(R, br));
    }
    const V3 on_ref = w - pn * (nm::dot(pn, w) - plane_d);
    if (ref_is_a) { c.p2 = on_ref; c.p1 = w; } else { c.p1 = on_ref; c.p2 = w; }
}

// ---- spheres and capsules against a hull (in the hull's frame: H posed at the origin with the identity) ----------------------------------
// The first t >= 0 at which the local point x0 moving along v reaches the hull rounded by r, with no overlap at t = 0 (the caller tests
// that): the face planes offset by r, a hit counting only when its foot lies in the face polygon (hm::in_face), and every edge as a capsule
// of radius r (qm::ray_capsule_rel).  The rounded hull is the union of those pieces, so the minimum is exact.  INFINITY when none is reached.
NM_HD inline S rounded_hull_toi(const Hull& H, V3 x0, V3 v, S r) {
    S best = INFINITY;
NM_ROLLED
    for (int f = 0; f < H.nf; ++f) {
        const V3 n = hm::fnormal(H, f);
        const S dn = nm::dot(n, v);
        if (!(dn < 0)) continue;
        const S tf = (hm::foffset(H, f) + r - nm::dot(n, x0)) / dn;
        if (!(tf >= 0) || !(tf < best)) continue;
        if (hm::in_face(H, f, n, x0 + v * tf - n * r)) best = tf;
    }
NM_ROLLED
    for (int e = 0; e < H.ne; ++e) {
        V3 m, u, nn;
        S h, te;
        hm::edge_seg(H, e, m, u, h);
        if (qm::ray_capsule_rel(x0 - m, u, h, r, v, true, te, nn) && te < best) best = te;
    }
    return best;
}
// the point x lies in the hull or within r of it
NM_HD inline bool point_near_hull(const Hull& H, V3 x, S r) {
    int fb;
    if (max_plane(H, x, fb) <= 0) return true;
    V3 on;
    return hm::point_hull_closest(H, x, on) <= r * r;
}
// the segment (c, u, h) clipped by the face half-spaces is not empty
NM_HD inline bool segment_meets_hull(const Hull& H, V3 c, V3 u, S h) {
    S lo = -h, hi = h;
NM_ROLLED
    for (int f = 0; f < H.nf; ++f) {
        const V3 n = hm::fnormal(H, f);
        const S a = nm::dot(n, c) - hm::foffset(H, f), g = nm::dot(n, u);
        if (g == 0) {
            if (a > 0) return false;
            continue;
        }
        if (g > 0) hi = nm::smin(hi, -a / g); else lo = nm::smax(lo, -a / g);
    }
    return lo <= hi;
}
// the segment meets the hull or comes within r of it (end points against the hull, the segment against every edge)
NM_HD inline bool segment_near_hull(const Hull& H, V3 c, V3 u, S h, S r) {
    if (segment_meets_hull(H, c, u, h)) return true;
    V3 on;
    if (hm::point_hull_closest(H, c - u * h, on) <= r * r || hm::point_hull_closest(H, c + u * h, on) <= r * r) return true;
NM_ROLLED
    for (int e = 0; e < H.ne; ++e) {
        V3 m, ue;
        S he, s, t;
        hm::edge_seg(H, e, m, ue, he);
        nm::segment_closest(c, u, h, m, ue, he, s, t);
        const V3 g = (c + u * s) - (m + ue * t);
        if (nm::dot(g, g) <= r * r) return true;
    }
    return false;
}
// the point of the segment (c, u, h) nearest the hull, which it does not meet: the nearer end point, or the segment's point nearest an edge
NM_HD inline V3 segment_closest_point(const Hull& H, V3 c, V3 u, S h) {
    V3 on, best_p = c - u * h;
    S best = hm::point_hull_closest(H, best_p, on);
    const S d1 = hm::point_hull_closest(H, c + u * h, on);
    if (d1 < best) { best = d1; best_p = c + u * h; }
NM_ROLLED
    for (int e = 0; e < H.ne; ++e) {
        V3 m, ue;
        S he, s, t;
        hm::edge_seg(H, e, m, ue, he);
        nm::segment_closest(c, u, h, m, ue, he, s, t);
        const V3 g = (c + u * s) - (m + ue * t);
        if (nm::dot(g, g) < best) { best = nm::dot(g, g); best_p = c + u * s; }
    }
    return best_p;
}
// a capsule (c, u, h, r) moving along v against the hull: its two end points against the rounded hull, the segment against every edge
// (qm::seg_seg_toi of radius r); capsule_box_toi's argument for any hull
NM_HD inline S capsule_hull_toi(const Hull& H, V3 c, V3 u, S h, S r, V3 v) {
    S best = nm::smin(rounded_hull_toi(H, c - u * h, v, r), rounded_hull_toi(H, c + u * h, v, r));
NM_ROLLED
    for (int e = 0; e < H.ne; ++e) {
        V3 m, ue;
        S he, te;
        hm::edge_seg(H, e, m, ue, he);
        if (qm::seg_seg_toi(m - c, u, h, ue, he, r, v, te) && te < best) best = te;
    }
    return best;
}

// ---- the pairs with at least one hull --------------------------------------------------------------------------------------------------
// The TOI of cast shape A against collider B: the bounding-sphere cull of §7j (table radius for a hull), then the moving SAT for two
// polytopes, or the sphere's centre / the capsule against the other shape's rounded hull in the hull's frame (+d when the hull is the
// collider, -d when it is cast).  Overlap at t = 0 is TOI 0.
NM_COLD inline bool hull_cast_toi(const Table& t, int sa, V3 ha, V3 ca, Q qa, V3 d, S maxd, int sb, V3 hb, V3 cb, Q qb, S& tt, int& axis) {
    S tb;
    if (!qm::sphere_sphere_toi(ca, d, cb, (bounding_radius(t, sa, ha) + bounding_radius(t, sb, hb)) * (1 + 1e-6), tb) || tb > maxd) return false;
    if (is_poly(sa) && is_poly(sb)) {
        hm::BoxHull ba, bb;
        const Hull A = polytope(t, ba, sa, ha, V3{0, 0, 0}, qm::rot_mat(qa)), B = polytope(t, bb, sb, hb, cb - ca, qm::rot_mat(qb));
        return poly_toi(A, B, d, maxd, tt, axis);
    }
    const bool a_hull = sa == SHAPE_HULL;
    const int so = a_hull ? sb : sa;
    const V3 hh = a_hull ? ha : hb, ho = a_hull ? hb : ha;
    const M3 rh = qm::rot_mat(a_hull ? qa : qb);
    const Hull H = hm::table_hull_at(t, hull_index(hh), V3{0, 0, 0}, identity());
    const V3 rel = qm::to_local(rh, a_hull ? cb - ca : ca - cb), v = qm::to_local(rh, a_hull ? -d : d);
    S best;
    if (so == nm::SHAPE_SPHERE) {
        if (point_near_hull(H, rel, ho.x)) { tt = 0; return true; }
        best = rounded_hull_toi(H, rel, v, ho.x);
    } else {
        const V3 u = qm::to_local(rh, qm::rot_mat(a_hull ? qb : qa).c[1]);
        if (segment_near_hull(H, rel, u, ho.y, ho.x)) { tt = 0; return true; }
        best = capsule_hull_toi(H, rel, u, ho.y, ho.x, v);
    }
    if (best == INFINITY) return false;
    tt = best;
    return true;
}

// the contact of a pair with at least one hull, A at `at`
NM_COLD inline void hull_cast_contact(const Table& t, int sa, V3 ha, V3 at, Q qa, V3 d, int sb, V3 hb, V3 cb, Q qb, S tt, int axis, qm::ShapeContact& c) {
    if (is_poly(sa) && is_poly(sb)) {
        hm::BoxHull ba, bb;
        const Hull A = polytope(t, ba, sa, ha, at, qm::rot_mat(qa)), B = polytope(t, bb, sb, hb, cb, qm::rot_mat(qb));
        poly_witness(A, B, axis, d, tt, c);
        return;
    }
    // hm::hull_sphere / hm::hull_capsule at the TOI pose with no distance limit, the first witness; their normal runs from the hull
    const bool a_hull = sa == SHAPE_HULL;
    const int so = a_hull ? sb : sa;
    const V3 ho = a_hull ? hb : ha, po = a_hull ? cb : at;
    const Hull H = hm::table_hull_at(t, hull_index(a_hull ? ha : hb), a_hull ? at : cb, qm::rot_mat(a_hull ? qa : qb));
    hm::Raw raw;
    raw.n = 0;
    V3 n{0, 1, 0};
    if (so == nm::SHAPE_SPHERE) {
        hm::hull_sphere(H, po, ho.x, INFINITY, n, raw);
    } else {
        const nm::Capsule C = qm::capsule_of(ho, po, a_hull ? qb : qa);
        hm::hull_capsule(H, C, INFINITY, n, raw);
        if (!(std::isfinite(n.x) && std::isfinite(n.y) && std::isfinite(n.z))) {
            // a segment that touches the hull at distance 0 from outside (radius 0): hm::hull_capsule's direction is 0 / 0.  The sphere rule
            // at the segment's closest point instead: the closest point, or the face of largest signed distance when they coincide.
            raw.n = 0;
            hm::hull_sphere(H, segment_closest_point(H, C.c, C.u, C.h), C.r, INFINITY, n, raw);
        }
    }
    const V3 on_hull = raw.n ? raw.p[0].a : H.c, on_other = raw.n ? raw.p[0].b : po;
    if (a_hull) { c.n2 = n; c.n1 = -n; c.p2 = on_hull; c.p1 = on_other; }
    else { c.n1 = n; c.n2 = -n; c.p1 = on_hull; c.p2 = on_other; }
}

// closed intersection of a pair with at least one hull
NM_COLD inline bool hull_intersect(const Table& t, int sa, V3 ha, V3 ca, Q qa, int sb, V3 hb, V3 cb, Q qb) {
    if (is_poly(sa) && is_poly(sb)) {
        hm::BoxHull ba, bb;
        return poly_intersect(polytope(t, ba, sa, ha, V3{0, 0, 0}, qm::rot_mat(qa)), polytope(t, bb, sb, hb, cb - ca, qm::rot_mat(qb)));
    }
    const bool a_hull = sa == SHAPE_HULL;
    const int so = a_hull ? sb : sa;
    const V3 hh = a_hull ? ha : hb, ho = a_hull ? hb : ha;
    const M3 rh = qm::rot_mat(a_hull ? qa : qb);
    const Hull H = hm::table_hull_at(t, hull_index(hh), V3{0, 0, 0}, identity());
    const V3 rel = qm::to_local(rh, a_hull ? cb - ca : ca - cb);
    if (so == nm::SHAPE_SPHERE) return point_near_hull(H, rel, ho.x);
    return segment_near_hull(H, rel, qm::to_local(rh, qm::rot_mat(a_hull ? qb : qa).c[1]), ho.y, ho.x);
}

// ---- the entry points of the hull instances: query_math.hpp's with the table ------------------------------------------------------------
NM_HD inline bool cast_toi(const Table& t, int sa, V3 ha, V3 ca, Q qa, V3 d, S maxd, int sb, V3 hb, V3 cb, Q qb, S& tt, int& axis) {
    if (sa == SHAPE_HULL || sb == SHAPE_HULL) {
        axis = -1;
        return hull_cast_toi(t, sa, ha, ca, qa, d, maxd, sb, hb, cb, qb, tt, axis) && tt <= maxd;
    }
    return qm::cast_toi<true>(sa, ha, ca, qa, d, maxd, sb, hb, cb, qb, tt, axis);
}
NM_HD inline void cast_contact(const Table& t, int sa, V3 ha, V3 ca, Q qa, V3 d, int sb, V3 hb, V3 cb, Q qb, S tt, int axis, qm::ShapeContact& c) {
    if (sa == SHAPE_HULL || sb == SHAPE_HULL) hull_cast_contact(t, sa, ha, ca + d * tt, qa, d, sb, hb, cb, qb, tt, axis, c);
    else qm::cast_contact<true>(sa, ha, ca, qa, d, sb, hb, cb, qb, tt, axis, c);
}
NM_HD inline bool cast_collider(const Table& t, int sa, V3 ha, V3 ca, Q qa, V3 d, S maxd, uint32_t flags, int sb, V3 hb, V3 cb, Q qb, S& tt, int& axis) {
    if (!cast_toi(t, sa, ha, ca, qa, d, maxd, sb, hb, cb, qb, tt, axis)) return false;
    if (tt == 0 && (flags & qm::CAST_IGNORE_ORIGIN_PENETRATION)) {
        qm::ShapeContact c;
        cast_contact(t, sa, ha, ca, qa, d, sb, hb, cb, qb, tt, axis, c);
        if (nm::dot(d, c.n1) > 0) return false;
    }
    return true;
}
NM_HD inline void cast_output(const Table& t, int sa, V3 ha, V3 ca, Q qa, V3 d, uint32_t flags, int sb, V3 hb, V3 cb, Q qb, S tt, int axis, qm::ShapeContact& c) {
    if (tt == 0 && (flags & qm::CAST_NO_CONTACT_ON_PENETRATION)) {
        c.p1 = c.p2 = c.n1 = c.n2 = V3{0, 0, 0};
        return;
    }
    cast_contact(t, sa, ha, ca, qa, d, sb, hb, cb, qb, tt, axis, c);
}
NM_HD inline bool shapes_intersect(const Table& t, int sa, V3 ha, V3 ca, Q qa, int sb, V3 hb, V3 cb, Q qb) {
    if (sa == SHAPE_HULL || sb == SHAPE_HULL) return hull_intersect(t, sa, ha, ca, qa, sb, hb, cb, qb);
    return qm::shapes_intersect<true>(sa, ha, ca, qa, sb, hb, cb, qb);
}

}  // namespace qh
