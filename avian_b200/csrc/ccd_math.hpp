// Swept continuous collision detection (solve_swept_ccd, dynamics/ccd/mod.rs:523-780) for cuboid / sphere / capsule / convex hull colliders: the pair time of impact,
// the per-pair filters and the delta arithmetic, written once for the host fixture (g++, -ffp-contract=off) and for the device pass
// (csrc/ccd.cu, nvcc -fmad=false): the same expressions in the same order, so both evaluate to the same bits.
//
// What this is: OUR time-of-impact arithmetic.  The reference delegates it to parry3d's cast_shapes / cast_shapes_nonlinear, which is not
// vendored, so there is no parity claim against parry — the claim is that the device pass and the host brute force agree bit for bit, and
// that the TOIs satisfy the contract below (tests/test_ccd_cpu.py checks it against an independent float64 distance reference).
//
// Conventions (ours; repeated in include/avian_b200.h and DESIGN.md §7e):
//   * A collider sits at its body's origin and its pose is the body's pose before the step (Position / Rotation).  Velocities are the
//     SolverBody velocities after the substeps.  Geometry is evaluated in IEEE double; the TOI is rounded once to the column scalar.
//   * Linear mode: shape 1 moves with d = v1 - v2 on [0, dt], shape 2 stays still: qm::cast_toi (sphere-sphere, sphere-cuboid as a point
//     against the rounded box, cuboid-cuboid by the moving 15-axis SAT).  Touching or overlapping at t = 0 is a TOI of 0.
//   * Non-linear mode (conservative advancement): com_i(t) = c_i + v_i t, q_i(t) = from_scaled_axis(w_i t) * q_i, the origin follows the
//     com (origin = com - q(t) * local_com).  Each iteration takes the exact distance d and the unit direction n from A to B (15-axis SAT
//     overlap test, then nm::box_box_closest; nm::box_point_closest; the closed form for two spheres) and stops with a hit at t when
//     d <= eps.  Otherwise it advances t by d / mu, mu = max(0, -(v2 - v1).n) + |w1| R1 + |w2| R2, R_i = the shape's farthest point from its
//     com.  mu = 0 or t > t_max: no hit.  After CCD_MAX_ITERATIONS iterations it reports the current t, which lies before the contact.
//     The iterates do not depend on t_max, so evaluating every candidate against dt and keeping the minimum equals the reference's
//     sequential scan with a shrinking bound.
//   * eps = CCD_EPS_PER_LENGTH_UNIT * PhysicsLengthUnit.
//   * Shape level G (DESIGN.md §7e): G = 0 cuboids and spheres, G = 1 adds capsules, G = 2 adds convex hulls over the hull table (the
//     table pointer of the G = 2 entry points; the lower levels take none).  Every branch of a level is out of line and comes first, so a
//     pair without the level's shape evaluates exactly as at the level below, bit for bit.
//   * Capsules (G >= 1): dims = [radius, half length, ·], the segment along the collider's local y (rot_mat(q(t)).c[1], as qm::capsule_of).
//     Linear mode: qm::cast_toi<true>'s exact capsule casts.  Non-linear mode: capsule_distance (point-segment, nm::segment_closest, or 0
//     when qm::segment_meets_box and else nm::segment_box_closest, less the radii; the swapped orders negate n), and
//     R = |(|lc.x|, |lc.y| + half length, |lc.z|)| + radius.
//   * Convex hulls (G = 2): dims = [hull index, ·, ·], posed by hm::table_hull_at with pose_at's rotation matrix.  Linear mode: qh::cast_toi
//     (the exact hull casts of the spatial queries).  Non-linear mode: hull_distance (0 when qh::poly_intersect, else hm::hull_hull_closest
//     for a hull and a hull or a cuboid as hm::box_hull; 0 when qh::point_near_hull, else sqrt(hm::point_hull_closest) less the radius for
//     a sphere; 0 when qh::segment_near_hull, else the distance of qh::segment_closest_point to the hull less the radius for a capsule; the
//     swapped orders negate n), and R = max_k |v_k - lc| over the hull-local vertices + AVN_HULL_REL_TOL x the local vertex-box diagonal:
//     the face planes, which the distance reads, can stand out of the vertex hull by that tolerance.
//   * sin / cos of from_scaled_axis come from ccd_sincos below (Cody-Waite reduction, Taylor polynomials, no libm), so the host and the
//     device round identically in f64 too; otherwise the expression tree is avn_math.cuh's q_from_scaled_axis and qmul.
#pragma once
#include <cmath>
#include <cstdint>

#include "hull_query_math.hpp"
#include "query_math.hpp"

namespace ccd {

using nm::S;
using nm::V3;
using nm::Q;

constexpr int CCD_MAX_ITERATIONS = 64;
constexpr double CCD_EPS_PER_LENGTH_UNIT = 1e-4;
constexpr int MODE_LINEAR = 0, MODE_NON_LINEAR = 1;   // AvnSweepMode

// sin and cos of x in double: x = k pi/2 + r with |r| <= pi/4 (fdlibm's two-part pi/2: k * PIO2_1 is exact for |k| < 2^20), Taylor
// polynomials of degree 17 / 18 in r (truncation below 1e-19), quadrant by k mod 4.  Accurate to a few ulp for |x| < 1e6.
NM_HD inline void ccd_sincos(double x, double& s, double& c) {
    const double PIO2_1 = 1.57079632673412561417e+00, PIO2_1T = 6.07710050650619224932e-11, INV_PIO2 = 6.36619772367581382433e-01;
    const double k = rint(x * INV_PIO2);
    const double r = (x - k * PIO2_1) - k * PIO2_1T;
    const double r2 = r * r;
    double ps = 1.0 / 355687428096000.0;   // 1/17!
    ps = ps * r2 - 1.0 / 1307674368000.0;
    ps = ps * r2 + 1.0 / 6227020800.0;
    ps = ps * r2 - 1.0 / 39916800.0;
    ps = ps * r2 + 1.0 / 362880.0;
    ps = ps * r2 - 1.0 / 5040.0;
    ps = ps * r2 + 1.0 / 120.0;
    ps = ps * r2 - 1.0 / 6.0;
    const double sr = r + r * (r2 * ps);
    double pc = 1.0 / 6402373705728000.0;  // 1/18!
    pc = pc * r2 - 1.0 / 20922789888000.0;
    pc = pc * r2 + 1.0 / 87178291200.0;
    pc = pc * r2 - 1.0 / 479001600.0;
    pc = pc * r2 + 1.0 / 3628800.0;
    pc = pc * r2 - 1.0 / 40320.0;
    pc = pc * r2 + 1.0 / 720.0;
    pc = pc * r2 - 1.0 / 24.0;
    pc = pc * r2 + 0.5;
    const double cr = 1.0 - r2 * pc;
    const long long q = ((static_cast<long long>(k) % 4) + 4) % 4;
    if (q == 0) { s = sr; c = cr; }
    else if (q == 1) { s = cr; c = -sr; }
    else if (q == 2) { s = -sr; c = -cr; }
    else { s = -cr; c = sr; }
}

// vectors and quaternions in the column scalar T (float or double), with avn_math.cuh's expression trees
template <class T> struct V3T { T x, y, z; };
template <class T> struct QT { T x, y, z, w; };
template <class T> NM_HD inline T dot3(V3T<T> a, V3T<T> b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
template <class T> NM_HD inline V3T<T> sub3(V3T<T> a, V3T<T> b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
template <class T> NM_HD inline V3T<T> scale3(V3T<T> a, T s) { return {a.x * s, a.y * s, a.z * s}; }

// Quat::from_scaled_axis (avn_math.cuh q_from_scaled_axis with ccd_sincos: f32 evaluates sin / cos of the f32 half angle in double and rounds)
template <class T> NM_HD inline QT<T> from_scaled_axis(V3T<T> v) {
    const T l = static_cast<T>(sqrt(static_cast<double>(dot3(v, v))));   // correctly rounded sqrt in either type
    if (l == T(0)) return {T(0), T(0), T(0), T(1)};
    const V3T<T> a{v.x / l, v.y / l, v.z / l};
    double s, c;
    ccd_sincos(static_cast<double>(l * T(0.5)), s, c);
    const T ts = static_cast<T>(s), tc = static_cast<T>(c);
    return {a.x * ts, a.y * ts, a.z * ts, tc};
}
// Quat::mul_quat: f32 in glam's SSE2 lane association, f64 left to right (avn_math.cuh qmul)
NM_HD inline QT<float> qmul(QT<float> a, QT<float> b) {
    return {(a.w * b.x + a.x * b.w) + (a.y * b.z - a.z * b.y), (a.w * b.y - a.x * b.z) + (a.y * b.w + a.z * b.x),
            (a.w * b.z + a.x * b.y) + (a.z * b.w - a.y * b.x), (a.w * b.w - a.x * b.x) + (-(a.y * b.y) - a.z * b.z)};
}
NM_HD inline QT<double> qmul(QT<double> a, QT<double> b) {
    return {a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x,
            a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}

// One body of a pair: its collider's shape, the pre-step pose, the local centre of mass and the SolverBody velocities, in double.
struct Motion {
    int shape;   // nm::SHAPE_*
    V3 he;       // half extents / radius in .x
    V3 p;        // Position (the collider's origin)
    Q q;         // Rotation
    V3 lc;       // local centre of mass
    V3 v, w;     // linear / angular velocity
};

// a hull's farthest vertex from the centre of mass, plus the table's tolerance (see the header comment)
NM_COLD inline S hull_motion_radius(const hm::Table& t, const Motion& m) {
    const uint32_t h = qh::hull_index(m.he), v0 = t.voff[h], nv = t.voff[h + 1] - v0;
    const double* v = t.vert + 3 * size_t(v0);
    V3 lo{v[0], v[1], v[2]}, hi = lo;
    S r2 = 0;
NM_ROLLED
    for (uint32_t k = 0; k < nv; ++k) {
        const V3 p{v[3 * k], v[3 * k + 1], v[3 * k + 2]}, e = p - m.lc;
        r2 = nm::smax(r2, nm::dot(e, e));
        lo = V3{nm::smin(lo.x, p.x), nm::smin(lo.y, p.y), nm::smin(lo.z, p.z)};
        hi = V3{nm::smax(hi.x, p.x), nm::smax(hi.y, p.y), nm::smax(hi.z, p.z)};
    }
    return sqrt(r2) + hm::REL_TOL * nm::len(hi - lo);
}

// farthest point of the shape from its centre of mass (a capsule: the farther end of its segment, plus the radius; a hull:
// hull_motion_radius with the table ht, G = 2 only)
template <int G = 0>
NM_HD inline S motion_radius(const Motion& m, const hm::Table* ht = nullptr) {
    if constexpr (G == 2)
        if (m.shape == hm::SHAPE_CONVEX_HULL) return hull_motion_radius(*ht, m);
    if (G >= 1 && m.shape == nm::SHAPE_CAPSULE) return nm::len(V3{fabs(m.lc.x), fabs(m.lc.y) + m.he.y, fabs(m.lc.z)}) + m.he.x;
    if (m.shape == nm::SHAPE_SPHERE) return nm::len(m.lc) + m.he.x;
    const V3 e{fabs(m.lc.x) + m.he.x, fabs(m.lc.y) + m.he.y, fabs(m.lc.z) + m.he.z};
    return nm::len(e);
}

// the pose at time t of the non-linear motion: origin and rotation matrix
NM_HD inline void pose_at(const Motion& m, S t, V3& origin, nm::M3& r) {
    const QT<double> dq = from_scaled_axis<double>({m.w.x * t, m.w.y * t, m.w.z * t});
    const QT<double> q = qmul(dq, QT<double>{m.q.x, m.q.y, m.q.z, m.q.w});
    const Q qt{q.x, q.y, q.z, q.w};
    const V3 com = (m.p + nm::rot(m.q, m.lc)) + m.v * t;
    origin = com - nm::rot(qt, m.lc);
    r = qm::rot_mat(qt);
}

// shape_distance of a pair with at least one capsule C (A when A is one) and the other shape O: the segment's distance to O's centre, to O's
// segment (nm::segment_closest) or to O's box (0 when the segment meets it, else nm::segment_box_closest), less the radii
NM_COLD inline S capsule_distance(int sa, V3 ha, V3 ca, const nm::M3& ra, int sb, V3 hb, V3 cb, const nm::M3& rb, V3& n) {
    n = V3{0, 1, 0};
    const bool a_cap = sa == nm::SHAPE_CAPSULE;
    const int so = a_cap ? sb : sa;
    const V3 hc = a_cap ? ha : hb, ho = a_cap ? hb : ha, co = a_cap ? cb : ca;
    const nm::M3& rc = a_cap ? ra : rb;
    const nm::M3& ro = a_cap ? rb : ra;
    const nm::Capsule C{a_cap ? ca : cb, rc.c[1], hc.y, hc.x};
    V3 e;        // from C's closest point to O's
    S l, radii = C.r;
    if (so == nm::SHAPE_CUBOID) {
        const nm::Box b{co, ro, ho};
        if (qm::segment_meets_box(b, C)) return 0;
        V3 on_seg, on_box;
        l = nm::segment_box_closest(b, C, on_seg, on_box);
        e = on_box - on_seg;
    } else {
        S s, t = 0;
        const V3 uo = ro.c[1];
        if (so == nm::SHAPE_CAPSULE) nm::segment_closest(C.c, C.u, C.h, co, uo, ho.y, s, t);
        else qm::segment_point_d2(co - C.c, C.u, C.h, s);
        e = (co + uo * t) - (C.c + C.u * s);
        l = nm::len(e);
        radii = radii + ho.x;
    }
    if (l > 0) n = (a_cap ? e : -e) * (1 / l);
    return nm::smax(l - radii, 0);
}

// shape_distance of a pair with at least one hull H (A when A is one) and the other shape O (see the header comment)
NM_COLD inline S hull_distance(const hm::Table& t, int sa, V3 ha, V3 ca, const nm::M3& ra, int sb, V3 hb, V3 cb, const nm::M3& rb, V3& n) {
    n = V3{0, 1, 0};
    const bool a_hull = sa == hm::SHAPE_CONVEX_HULL;
    const int so = a_hull ? sb : sa;
    if (qh::is_poly(so)) {
        hm::BoxHull ba, bb;
        const hm::Hull A = qh::polytope(t, ba, sa, ha, ca, ra), B = qh::polytope(t, bb, sb, hb, cb, rb);
        if (qh::poly_intersect(A, B)) return 0;
        V3 on_a, on_b;
        const S l = hm::hull_hull_closest(A, B, on_a, on_b);
        if (l > 0) n = (on_b - on_a) * (1 / l);
        return nm::smax(l, 0);
    }
    const hm::Hull H = hm::table_hull_at(t, qh::hull_index(a_hull ? ha : hb), a_hull ? ca : cb, a_hull ? ra : rb);
    const V3 ho = a_hull ? hb : ha, co = a_hull ? cb : ca;
    V3 x = co;   // the point of O nearest the hull: the sphere's centre, or the capsule segment's point nearest it
    if (so == nm::SHAPE_SPHERE) {
        if (qh::point_near_hull(H, co, ho.x)) return 0;
    } else {
        const V3 u = (a_hull ? rb : ra).c[1];
        if (qh::segment_near_hull(H, co, u, ho.y, ho.x)) return 0;
        x = qh::segment_closest_point(H, co, u, ho.y);
    }
    V3 on;
    const S l = sqrt(hm::point_hull_closest(H, x, on));
    if (l > 0) n = (a_hull ? x - on : on - x) * (1 / l);
    return nm::smax(l - ho.x, 0);
}

// Distance between the closed shapes A and B (0 when they overlap or touch) and the unit direction n from A to B.  Out of line and rolled,
// like nm::box_box_closest which it calls.  G >= 1: pairs with a capsule go to capsule_distance (the G = 0 instance has no such branch);
// pairs with a hull never come here (nonlinear_toi sends them to hull_distance).
template <int G = 0>
NM_COLD inline S shape_distance(int sa, V3 ha, V3 ca, const nm::M3& ra, int sb, V3 hb, V3 cb, const nm::M3& rb, V3& n) {
    if (G >= 1 && (sa == nm::SHAPE_CAPSULE || sb == nm::SHAPE_CAPSULE)) return capsule_distance(sa, ha, ca, ra, sb, hb, cb, rb, n);
    n = V3{0, 1, 0};
    if (sa == nm::SHAPE_SPHERE && sb == nm::SHAPE_SPHERE) {
        const V3 e = cb - ca;
        const S l = nm::len(e);
        if (l > 0) n = e * (1 / l);
        return nm::smax(l - ha.x - hb.x, 0);
    }
    if (sa == nm::SHAPE_SPHERE || sb == nm::SHAPE_SPHERE) {
        const bool box_a = sb == nm::SHAPE_SPHERE;
        const nm::Box box = box_a ? nm::Box{ca, ra, ha} : nm::Box{cb, rb, hb};
        const V3 centre = box_a ? cb : ca;
        const S r = box_a ? hb.x : ha.x;
        V3 on;
        const S l = sqrt(nm::box_point_closest(box, centre, on));
        if (l > 0) n = (box_a ? centre - on : on - centre) * (1 / l);
        return nm::smax(l - r, 0);
    }
    const V3 s = cb - ca;
    bool separated = false;
NM_ROLLED
    for (int k = 0; k < 15 && !separated; ++k) {
        const V3 L = qm::sat_axis(ra, rb, k);
        if (qm::is_zero3(L)) continue;
        separated = fabs(nm::dot(L, s)) > qm::box_extent(ra, ha, L) + qm::box_extent(rb, hb, L);
    }
    if (!separated) return 0;
    V3 on_a, on_b;
    const S l = nm::box_box_closest(nm::Box{ca, ra, ha}, nm::Box{cb, rb, hb}, on_a, on_b);
    if (l > 0) n = (on_b - on_a) * (1 / l);
    return l;
}

// conservative advancement on [0, t_max]; see the header comment.  *iterations (optional): the distance evaluations it took; a hit reported
// with CCD_MAX_ITERATIONS of them stopped at the cap, before reaching eps.  ht: the hull table (G = 2)
template <int G = 0>
NM_HD inline bool nonlinear_toi(const Motion& A, const Motion& B, S t_max, S eps, S& toi, int* iterations = nullptr, const hm::Table* ht = nullptr) {
    const V3 rel = B.v - A.v;
    const S spin = nm::len(A.w) * motion_radius<G>(A, ht) + nm::len(B.w) * motion_radius<G>(B, ht);
    S t = 0;
NM_ROLLED
    for (int it = 0; it < CCD_MAX_ITERATIONS; ++it) {
        V3 ca, cb, n;
        nm::M3 ra, rb;
        pose_at(A, t, ca, ra);
        pose_at(B, t, cb, rb);
        S d;
        if constexpr (G == 2)
            d = A.shape == hm::SHAPE_CONVEX_HULL || B.shape == hm::SHAPE_CONVEX_HULL ? hull_distance(*ht, A.shape, A.he, ca, ra, B.shape, B.he, cb, rb, n)
                                                                                     : shape_distance<1>(A.shape, A.he, ca, ra, B.shape, B.he, cb, rb, n);
        else
            d = shape_distance<G>(A.shape, A.he, ca, ra, B.shape, B.he, cb, rb, n);
        if (iterations) *iterations = it + 1;
        if (d != d) return false;
        if (d <= eps) { toi = t; return true; }
        const S mu = nm::smax(0, -nm::dot(rel, n)) + spin;
        if (!(mu > 0)) return false;
        t = t + d / mu;
        if (!(t <= t_max)) return false;
    }
    toi = t;
    return true;
}

// shape 1 moving with v1 - v2 against shape 2 at rest (qm::cast_toi; qh::cast_toi with the hull table at G = 2)
template <int G = 0>
NM_HD inline bool linear_toi(const Motion& A, const Motion& B, S t_max, S& toi, const hm::Table* ht = nullptr) {
    int axis;
    if constexpr (G == 2) return qh::cast_toi(*ht, A.shape, A.he, A.p, A.q, A.v - B.v, t_max, B.shape, B.he, B.p, B.q, toi, axis);
    else return qm::cast_toi<G == 1>(A.shape, A.he, A.p, A.q, A.v - B.v, t_max, B.shape, B.he, B.p, B.q, toi, axis);
}

// compute_ccd_toi (ccd/mod.rs:692-780) against the bound dt: the TOI rounded to T, with the reference's fallback when it is exactly 0 (shape 2
// replaced by a ball of radius prediction_distance at body 2's pose); T(-1) when the shapes never come within reach on [0, dt].  The caller
// accepts the value when 0 < toi < min_toi.  G: the shape level (G = 0 treats every shape as a cuboid or a sphere); ht: the hull table (G = 2).
template <class T, int G = 0>
NM_HD inline T pair_toi(int mode, const Motion& A, const Motion& B, T dt, S eps, S prediction_distance, const hm::Table* ht = nullptr) {
    S t = 0;
    const bool hit = mode == MODE_LINEAR ? linear_toi<G>(A, B, S(dt), t, ht) : nonlinear_toi<G>(A, B, S(dt), eps, t, nullptr, ht);
    if (!hit) return T(-1);
    const T tt = static_cast<T>(t);
    if (tt != T(0)) return tt;
    Motion ball = B;
    ball.shape = nm::SHAPE_SPHERE;
    ball.he = V3{prediction_distance, 0, 0};
    const bool hit2 = mode == MODE_LINEAR ? linear_toi<G>(A, ball, S(dt), t, ht) : nonlinear_toi<G>(A, ball, S(dt), eps, t, nullptr, ht);
    return hit2 ? static_cast<T>(t) : T(-1);
}

// the velocity filter of solve_swept_ccd (ccd/mod.rs:581-594): true when the pair is skipped
template <class T> NM_HD inline bool below_thresholds(V3T<T> v1, V3T<T> w1, V3T<T> v2, V3T<T> w2, T linear_threshold, T angular_threshold) {
    const V3T<T> dw = sub3(w1, w2), dv = sub3(v1, v2);
    return dot3(dw, dw) < angular_threshold * angular_threshold && dot3(dv, dv) < linear_threshold * linear_threshold;
}

// the overshoot applied to the minimum TOI (ccd/mod.rs:634)
template <class T> NM_HD inline T overshoot(T min_toi) { return min_toi * T(1.0001); }

// the write of one CCD record onto a body's deltas (ccd/mod.rs:636-670): delta_position is overwritten, delta_rotation composed
template <class T> NM_HD inline void apply_record(T m, V3T<T> v, V3T<T> w, V3T<T>& dp, QT<T>& dq) {
    dp = V3T<T>{m * v.x, m * v.y, m * v.z};
    dq = qmul(from_scaled_axis<T>(V3T<T>{w.x * m, w.y * m, w.z * m}), dq);
}

}  // namespace ccd
