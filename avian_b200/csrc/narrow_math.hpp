// Contact-manifold geometry for cuboid / sphere / capsule pairs, written once for the host fixture (g++, -ffp-contract=off) and for the device
// (nvcc, -fmad=false): the same expressions in the same order, IEEE double throughout, so both evaluate to the same bits.
//
// What this is: OUR manifold generator (SAT + face clipping for boxes, closed forms for spheres).  The reference delegates this
// arithmetic to parry3d 0.25, which is not vendored (SURVEY.md §8f #1), so there is no parity claim against parry — the claim is
// fixture-level: whatever consumes these manifolds (oracle or CUDA solver) gets identical inputs.
// Reference call sites: collider/parry/contact_query.rs:156-261 (contact_manifolds), contact_types/mod.rs:478-566 (prune_points),
// narrow_phase/system_param.rs:663-681,736-756 (speculative margin, point keep rule).
#pragma once
#include <cmath>

#if defined(__CUDACC__)
#define NM_HD __host__ __device__
#define NM_COLD __host__ __device__ __noinline__
#define NM_ROLLED _Pragma("unroll 1")
#else
#define NM_HD
#define NM_COLD
#define NM_ROLLED
#endif

namespace nm {

using S = double;  // geometry is evaluated in double and rounded to the column scalar type on export

struct V3 { S x, y, z; };
NM_HD inline V3 operator+(V3 a, V3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
NM_HD inline V3 operator-(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
NM_HD inline V3 operator-(V3 a) { return {-a.x, -a.y, -a.z}; }
NM_HD inline V3 operator*(V3 a, S s) { return {a.x * s, a.y * s, a.z * s}; }
NM_HD inline S dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
NM_HD inline V3 cross(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
NM_HD inline S len(V3 a) { return sqrt(dot(a, a)); }
NM_HD inline S comp(V3 a, int i) { return i == 0 ? a.x : (i == 1 ? a.y : a.z); }
// std::max / std::min semantics (the first argument wins ties), usable on the device
NM_HD inline S smax(S a, S b) { return a < b ? b : a; }
NM_HD inline S smin(S a, S b) { return b < a ? b : a; }

struct Q { S x, y, z, w; };
NM_HD inline V3 rot(Q q, V3 v) {
    V3 b{q.x, q.y, q.z};
    S b2 = dot(b, b);
    return v * (q.w * q.w - b2) + b * (dot(v, b) * 2) + cross(b, v) * (q.w * 2);
}
struct M3 { V3 c[3]; };  // columns = world directions of the local axes
NM_HD inline M3 to_mat(Q q) { return {{rot(q, {1, 0, 0}), rot(q, {0, 1, 0}), rot(q, {0, 0, 1})}}; }

enum ShapeType { SHAPE_CUBOID = 0, SHAPE_SPHERE = 1, SHAPE_CAPSULE = 2 };
struct Box { V3 c; M3 r; V3 he; };

// witness points of a contact: on shape A, on shape B (world axes, origin at A's position: see collide).  A quad clipped by four planes
// has at most 8 vertices.
constexpr int MAX_RAW_POINTS = 8;
struct Witness { V3 a, b; };
struct Contacts {
    int n;
    Witness p[MAX_RAW_POINTS];
    NM_HD void clear() { n = 0; }
    NM_HD void push(V3 on_a, V3 on_b) { p[n].a = on_a; p[n].b = on_b; ++n; }
};

// the face of `b` on the `sign` side of local axis `axis`: 4 corners (world)
NM_HD inline void box_face(const Box& b, int axis, S sign, V3 out[4]) {
    int u = (axis + 1) % 3, v = (axis + 2) % 3;
    V3 n = b.r.c[axis] * (sign * comp(b.he, axis));
    V3 eu = b.r.c[u] * comp(b.he, u), ev = b.r.c[v] * comp(b.he, v);
    V3 fc = b.c + n;
    out[0] = fc + eu + ev; out[1] = fc - eu + ev; out[2] = fc - eu - ev; out[3] = fc + eu - ev;
}

NM_HD inline int clip_poly(const V3* in, int n, V3 plane_n, S plane_d, V3* out) {  // keep dot(n,p) <= d
    int m = 0;
    for (int i = 0; i < n; ++i) {
        V3 a = in[i], b = in[(i + 1) % n];
        S da = dot(plane_n, a) - plane_d, db = dot(plane_n, b) - plane_d;
        if (da <= 0) out[m++] = a;
        if ((da < 0 && db > 0) || (da > 0 && db < 0)) out[m++] = a + (b - a) * (da / (da - db));
    }
    return m;
}

NM_HD inline S box_radius(const Box& b, V3 n) {
    return fabs(dot(b.r.c[0], n)) * b.he.x + fabs(dot(b.r.c[1], n)) * b.he.y + fabs(dot(b.r.c[2], n)) * b.he.z;
}

// Closest points of the segments p + u*s, |s| <= hu and q + w*t, |t| <= hw: clamp s, recompute t from it, and when t has to be clamped
// recompute s from the clamped t (dependent clamping, Ericson, Real-Time Collision Detection §5.1.9).  Returns true when the pair is not
// interior to both segments: an end is active, or the segments are too close to parallel for an interior pair to be defined.
NM_HD inline bool segment_closest(V3 p, V3 u, S hu, V3 q, V3 w, S hw, S& s, S& t) {
    V3 r = p - q;
    S a = dot(u, u), e = dot(w, w), f = dot(w, r), c = dot(u, r), b = dot(u, w);
    S den = a * e - b * b;
    S s0 = den > 1e-12 ? (b * f - c * e) / den : 0;
    s = smax(-hu, smin(hu, s0));
    bool end = den <= 1e-12 || s != s0;
    t = (b * s + f) / e;
    if (t < -hw || t > hw) {
        t = t < -hw ? -hw : hw;
        s = smax(-hu, smin(hu, (b * t - c) / a));
        end = true;
    }
    return end;
}

// The point of box b closest to p (p itself when inside); returns the squared distance.
NM_HD inline S box_point_closest(const Box& b, V3 p, V3& on) {
    V3 d = p - b.c;
    on = b.c;
    for (int k = 0; k < 3; ++k) on = on + b.r.c[k] * smax(-comp(b.he, k), smin(comp(b.he, k), dot(d, b.r.c[k])));
    V3 e = p - on;
    return dot(e, e);
}

// The closest pair of points of two disjoint boxes: the minimum over every vertex against the other box and every edge against every
// edge.  Returns the distance.  box_box uses it only for separated pairs whose SAT feature misses the closest features: a rare branch,
// kept out of line and rolled so that its 16 + 144 candidates are not unrolled into the kernels that inline box_box (fully inlined,
// they took 255 registers and spilled).  The call still costs registers: see DESIGN.md §7 for the ptxas figures.
NM_COLD inline S box_box_closest(const Box& A, const Box& B, V3& on_a, V3& on_b) {
    S best = 1e300;
NM_ROLLED
    for (int side = 0; side < 2; ++side) {
        const Box& P = side == 0 ? A : B;
        const Box& O = side == 0 ? B : A;
NM_ROLLED
        for (int m = 0; m < 8; ++m) {
            V3 v = P.c + P.r.c[0] * (m & 1 ? P.he.x : -P.he.x) + P.r.c[1] * (m & 2 ? P.he.y : -P.he.y) + P.r.c[2] * (m & 4 ? P.he.z : -P.he.z);
            V3 on;
            S d2 = box_point_closest(O, v, on);
            if (d2 < best) { best = d2; on_a = side == 0 ? v : on; on_b = side == 0 ? on : v; }
        }
    }
    // edge k of a box, number m: the segment along axis k through the centre offset by the signs of m on the other two axes
    auto edge_mid = [](const Box& b, int k, int m) {
        int u = (k + 1) % 3, v = (k + 2) % 3;
        return b.c + b.r.c[u] * (m & 1 ? comp(b.he, u) : -comp(b.he, u)) + b.r.c[v] * (m & 2 ? comp(b.he, v) : -comp(b.he, v));
    };
NM_ROLLED
    for (int ei = 0; ei < 12; ++ei) {
        const int i = ei >> 2, mi = ei & 3;
        V3 pa = edge_mid(A, i, mi);
NM_ROLLED
        for (int ej = 0; ej < 12; ++ej) {
            const int j = ej >> 2, mj = ej & 3;
            V3 pb = edge_mid(B, j, mj);
            S s, t;
            segment_closest(pa, A.r.c[i], comp(A.he, i), pb, B.r.c[j], comp(B.he, j), s, t);
            V3 qa = pa + A.r.c[i] * s, qb = pb + B.r.c[j] * t, e = qb - qa;
            S d2 = dot(e, e);
            if (d2 < best) { best = d2; on_a = qa; on_b = qb; }
        }
    }
    return sqrt(best);
}

// A separated pair as its closest points (from box_box_closest): one witness pair, the normal along it (from A to B).  False when it
// is beyond max_dist.
NM_HD inline bool closest_pair(V3 on_a, V3 on_b, S dist, S max_dist, V3& normal, Contacts& pts) {
    pts.clear();
    if (dist > max_dist) return false;
    if (dist > 1e-12) normal = (on_b - on_a) * (1 / dist);
    pts.push(on_a, on_b);
    return true;
}

// How much farther than the true distance the nearest clipped point of a separated face contact may be before the closest feature pair
// replaces the clipped polygon: a face contact whose nearest point is the closest feature (a box resting or landing flat) keeps its
// polygon, and a box whose nearest corner or edge hangs past the reference face gets that corner or edge instead.
constexpr S FACE_GAP_SLACK = 1e-4;

// SAT over the 15 axes, then either the closest points of the two supporting edges or the incident face clipped against the
// reference face's side planes.  Returns false when the boxes are farther apart than max_dist.  normal points from A to B.
// Separated pairs whose SAT feature does not give the closest points (the edges' closest points lie at an end, or the clipped face
// lies farther than FACE_GAP_SLACK beyond the true distance) report their closest feature pair instead.  Overlapping pairs whose edges'
// closest points lie at an end use the best face axis.
NM_HD inline bool box_box(const Box& A, const Box& B, S max_dist, V3& normal, Contacts& pts) {
    pts.clear();
    V3 d = B.c - A.c;
    S best_sep = -1e300;
    int best_kind = -1, best_i = 0, best_j = 0;
    V3 best_n{0, 1, 0};
    auto consider = [&](V3 n, int kind, int i, int j, S bias) {
        S l = len(n);
        if (l < 1e-9) return;
        n = n * (1 / l);
        if (dot(n, d) < 0) n = -n;
        S sep = dot(n, d) - box_radius(A, n) - box_radius(B, n);
        // face axes are preferred over edge axes by a small bias, earlier axes win ties: stable feature choice
        if (sep - bias > best_sep + 1e-9) { best_sep = sep - bias; best_kind = kind; best_i = i; best_j = j; best_n = n; }
    };
    for (int i = 0; i < 3; ++i) consider(A.r.c[i], 0, i, 0, 0);
    for (int i = 0; i < 3; ++i) consider(B.r.c[i], 1, i, 0, 0);
    const S face_sep = best_sep;
    const int face_kind = best_kind, face_i = best_i;
    const V3 face_n = best_n;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) consider(cross(A.r.c[i], B.r.c[j]), 2, i, j, 1e-4);
    S sep = best_kind == 2 ? best_sep + 1e-4 : best_sep;
    if (sep > max_dist) return false;
    normal = best_n;
    if (best_kind == 2) {
        // edge-edge: closest points of the two supporting edges
        V3 ea = A.r.c[best_i], eb = B.r.c[best_j];
        V3 pa = A.c, pb = B.c;
        for (int k = 0; k < 3; ++k) {
            if (k != best_i) pa = pa + A.r.c[k] * (comp(A.he, k) * (dot(A.r.c[k], normal) > 0 ? 1 : -1));
            if (k != best_j) pb = pb + B.r.c[k] * (comp(B.he, k) * (dot(B.r.c[k], normal) < 0 ? 1 : -1));
        }
        S s, t;
        if (!segment_closest(pa, ea, comp(A.he, best_i), pb, eb, comp(B.he, best_j), s, t)) {
            pts.push(pa + ea * s, pb + eb * t);
            return true;
        }
        // an end is active: the edges are not the closest features
        if (sep > 0) {
            V3 on_a, on_b;
            S dist = box_box_closest(A, B, on_a, on_b);
            return closest_pair(on_a, on_b, dist, max_dist, normal, pts);
        }
        sep = face_sep; best_kind = face_kind; best_i = face_i; normal = face_n;
    }
    // face contact: reference box R (face axis), incident box I
    const bool ref_is_a = best_kind == 0;
    const Box& R = ref_is_a ? A : B;
    const Box& I = ref_is_a ? B : A;
    V3 rn = ref_is_a ? normal : -normal;  // outward normal of the reference face
    // incident face: the face of I most anti-parallel to rn
    int inc_axis = 0;
    S inc_best = -1;
    for (int k = 0; k < 3; ++k) {
        S v = fabs(dot(I.r.c[k], rn));
        if (v > inc_best) { inc_best = v; inc_axis = k; }
    }
    S isign = dot(I.r.c[inc_axis], rn) > 0 ? -1 : 1;
    V3 poly[16], tmp[16];
    box_face(I, inc_axis, isign, poly);
    int np = 4;
    int u = (best_i + 1) % 3, v = (best_i + 2) % 3;
    const int axes[2] = {u, v};
    for (int a = 0; a < 2 && np > 0; ++a) {
        V3 sn = R.r.c[axes[a]];
        S he = comp(R.he, axes[a]);
        np = clip_poly(poly, np, sn, dot(sn, R.c) + he, tmp);
        np = clip_poly(tmp, np, -sn, -dot(sn, R.c) + he, poly);
    }
    S face_d = dot(rn, R.c) + comp(R.he, best_i) * 1.0;
    S nearest = 1e300;
    for (int k = 0; k < np; ++k) {
        S dist = dot(rn, poly[k]) - face_d;  // signed distance of the incident point above the reference face
        if (dist > max_dist) continue;
        nearest = smin(nearest, dist);
        V3 on_ref = poly[k] - rn * dist;
        // drop near-duplicates
        bool dup = false;
        for (int q = 0; q < pts.n; ++q) {
            V3 e = (ref_is_a ? pts.p[q].b : pts.p[q].a) - poly[k];
            if (dot(e, e) < 1e-12) { dup = true; break; }
        }
        if (dup) continue;
        if (pts.n == MAX_RAW_POINTS) break;
        if (ref_is_a) pts.push(on_ref, poly[k]); else pts.push(poly[k], on_ref);
    }
    // separated, and the clipped face does not reach down to the SAT separation: the closest features may lie outside the reference
    // face's prism (a corner hanging past its edge), so compare with the true distance
    if (sep > 0 && nearest > sep + FACE_GAP_SLACK) {
        V3 on_a, on_b;
        S dist = box_box_closest(A, B, on_a, on_b);
        if (nearest > dist + FACE_GAP_SLACK) return closest_pair(on_a, on_b, dist, max_dist, normal, pts);
    }
    return pts.n != 0;
}

// keep at most 4 points: deepest, farthest from it, farthest from that segment on each side (cf. prune_points,
// contact_types/mod.rs:478-566, itself after Jolt's PruneContactPoints); survivors stay in their original order
NM_HD inline void prune4(Contacts& pts, V3 n) {
    if (pts.n <= 4) return;
    auto depth = [&](int i) { return dot(pts.p[i].a - pts.p[i].b, n); };
    int p0 = 0;
    for (int i = 1; i < pts.n; ++i) if (depth(i) > depth(p0) + 1e-12) p0 = i;
    int p1 = p0;
    S best = -1;
    for (int i = 0; i < pts.n; ++i) { V3 e = pts.p[i].a - pts.p[p0].a; S v = dot(e, e); if (v > best) { best = v; p1 = i; } }
    V3 dir = cross(pts.p[p1].a - pts.p[p0].a, n);
    int p2 = p0, p3 = p0;
    S mx = 0, mn = 0;
    for (int i = 0; i < pts.n; ++i) {
        S v = dot(pts.p[i].a - pts.p[p0].a, dir);
        if (v > mx) { mx = v; p2 = i; }
        if (v < mn) { mn = v; p3 = i; }
    }
    bool keep[MAX_RAW_POINTS] = {false, false, false, false, false, false, false, false};
    keep[p0] = keep[p1] = keep[p2] = keep[p3] = true;
    int m = 0;
    for (int i = 0; i < pts.n; ++i)
        if (keep[i]) pts.p[m++] = pts.p[i];
    pts.n = m;
}

NM_HD inline bool sphere_sphere(V3 ca, S ra, V3 cb, S rb, S max_dist, V3& normal, Contacts& pts) {
    pts.clear();
    V3 d = cb - ca;
    S l = len(d);
    if (l - ra - rb > max_dist) return false;
    normal = l > 1e-12 ? d * (1 / l) : V3{0, 1, 0};
    pts.push(ca + normal * ra, cb - normal * rb);
    return true;
}

NM_HD inline bool box_sphere(const Box& A, V3 cs, S rs, S max_dist, V3& normal, Contacts& pts) {  // normal from box to sphere
    pts.clear();
    V3 d = cs - A.c;
    V3 local{dot(d, A.r.c[0]), dot(d, A.r.c[1]), dot(d, A.r.c[2])};
    V3 cl{smax(-A.he.x, smin(A.he.x, local.x)), smax(-A.he.y, smin(A.he.y, local.y)), smax(-A.he.z, smin(A.he.z, local.z))};
    V3 on_box = A.c + A.r.c[0] * cl.x + A.r.c[1] * cl.y + A.r.c[2] * cl.z;
    V3 e = cs - on_box;
    S l = len(e);
    // inside is decided on the local coordinates: an f32 quaternion is unit only to an ulp, so rebuilding the centre from them misses
    // it by ~1e-8 and the distance alone cannot tell a centre inside from one just outside
    const bool inside = fabs(local.x) <= A.he.x && fabs(local.y) <= A.he.y && fabs(local.z) <= A.he.z;
    if (!inside && l > 1e-9) {
        if (l - rs > max_dist) return false;
        normal = e * (1 / l);
    } else {  // centre inside the box: push out through the nearest face
        int ax = 0; S best = 1e300;
        for (int k = 0; k < 3; ++k) { S v = comp(A.he, k) - fabs(comp(local, k)); if (v < best) { best = v; ax = k; } }
        S sgn = comp(local, ax) >= 0 ? 1 : -1;
        normal = A.r.c[ax] * sgn;
        on_box = cs + normal * best;
    }
    pts.push(on_box, cs - normal * rs);
    return true;
}

// ---- capsules (DESIGN.md §7h): dims = [radius, half_length, unused], the segment from (0, -half_length, 0) to (0, +half_length, 0) of the
// collider frame grown by the radius.  Every capsule routine is out of line and rolled, and returns through pts and its return value, so the
// cuboid and sphere pairs compile to the code they had before capsules existed.  A capsule pair has at most 2 points.

// Two directions count as parallel (two-point manifolds) when the sine of their angle is at most this (about 0.06 degrees).
constexpr S CAPSULE_PARALLEL_SIN = 1e-3;
// e_k x s axes of the segment-box SAT shorter than this (an edge direction parallel to the segment) are skipped
constexpr S CAPSULE_EDGE_AXIS_MIN = 1e-6;

struct Capsule { V3 c, u; S h, r; };   // centre, unit axis, half length, radius

// u x e_k, normalised, with e_k the first world axis least aligned with the unit vector u: the fallback normal when two axes or a centre and an
// axis coincide (perpendicular to u, so a witness grown from an interior segment point stays on the capsule's surface)
NM_HD inline V3 capsule_perpendicular(V3 u) {
    const V3 e = (fabs(u.x) <= fabs(u.y) && fabs(u.x) <= fabs(u.z)) ? V3{1, 0, 0} : (fabs(u.y) <= fabs(u.z) ? V3{0, 1, 0} : V3{0, 0, 1});
    const V3 n = cross(u, e);
    return n * (1 / len(n));
}

// Capsule A against a round shape B: the segment q + w*t, |t| <= hw, grown by rb (a sphere: hw = 0, w = A.u).  Normal from A to B.
// The closest points of the two segments grown by the radii.  Distance 0: n = +-unit(A.u x w), the sign that points from A's centre to
// B's (u x w itself on a tie); parallel axes (and a sphere centre on A's axis) take capsule_perpendicular(A.u).  Parallel capsules whose
// projections on A's axis overlap get one point at each end of the overlap.
NM_COLD inline bool capsule_round(const Capsule& A, V3 q, V3 w, S hw, S rb, S max_dist, V3& normal, Contacts& pts) {
    S s, t;
    segment_closest(A.c, A.u, A.h, q, w, hw, s, t);
    const V3 p = A.c + A.u * s, qq = q + w * t, d = qq - p;
    const S l = len(d);
    if (l - A.r - rb > max_dist) return false;
    const V3 x = cross(A.u, w);
    const S lx = len(x);
    const bool parallel = !(hw > 0) || lx <= CAPSULE_PARALLEL_SIN;
    if (l > 1e-12) {
        normal = d * (1 / l);
    } else if (!parallel) {
        normal = x * (1 / lx);
        if (dot(normal, q - A.c) < 0) normal = -normal;
    } else {
        normal = capsule_perpendicular(A.u);
    }
    if (hw > 0 && parallel) {
        const S t0 = dot(q - w * hw - A.c, A.u), t1 = dot(q + w * hw - A.c, A.u);
        const S lo = smax(-A.h, smin(t0, t1)), hi = smin(A.h, smax(t0, t1));
        if (lo < hi) {
NM_ROLLED
            for (int i = 0; i < 2; ++i) {
                const V3 pi = A.c + A.u * (i == 0 ? lo : hi);
                const S ti = smax(-hw, smin(hw, dot(pi - q, w)));
                pts.push(pi + normal * A.r, q + w * ti - normal * rb);
            }
            return true;
        }
    }
    pts.push(p + normal * A.r, qq - normal * rb);
    return true;
}

// The closest points of a segment disjoint from box b: the two end points against the box and the segment against the 12 edges.  Returns the
// distance.
NM_COLD inline S segment_box_closest(const Box& b, const Capsule& C, V3& on_seg, V3& on_box) {
    S best = 1e300;
NM_ROLLED
    for (int i = 0; i < 2; ++i) {
        const V3 p = C.c + C.u * (i == 0 ? -C.h : C.h);
        V3 on;
        const S d2 = box_point_closest(b, p, on);
        if (d2 < best) { best = d2; on_seg = p; on_box = on; }
    }
NM_ROLLED
    for (int ei = 0; ei < 12; ++ei) {
        const int k = ei >> 2, m = ei & 3, u = (k + 1) % 3, v = (k + 2) % 3;
        const V3 e = b.c + b.r.c[u] * (m & 1 ? comp(b.he, u) : -comp(b.he, u)) + b.r.c[v] * (m & 2 ? comp(b.he, v) : -comp(b.he, v));
        S s, t;
        segment_closest(C.c, C.u, C.h, e, b.r.c[k], comp(b.he, k), s, t);
        const V3 qs = C.c + C.u * s, qe = e + b.r.c[k] * t, d = qs - qe;
        const S d2 = dot(d, d);
        if (d2 < best) { best = d2; on_seg = qs; on_box = qe; }
    }
    return sqrt(best);
}

// The part [lo, hi] of C's segment (parameter along C.u) inside the side planes of b's faces on local axis k.  False when it is empty.
NM_HD inline bool capsule_face_clip(const Box& b, int k, const Capsule& C, S& lo, S& hi) {
    lo = -C.h; hi = C.h;
NM_ROLLED
    for (int i = 1; i < 3; ++i) {
        const int j = (k + i) % 3;
        const S a = dot(b.r.c[j], C.c - b.c), g = dot(b.r.c[j], C.u), he = comp(b.he, j);
        if (fabs(g) < 1e-12) {
            if (fabs(a) > he) return false;
            continue;
        }
        const S s0 = (-he - a) / g, s1 = (he - a) / g;
        lo = smax(lo, smin(s0, s1));
        hi = smin(hi, smax(s0, s1));
    }
    return lo <= hi;
}

// Box b against capsule C (the segment grown by C.r); normal from the box to the capsule.  A segment disjoint from the box: its exact closest
// points.  A segment that meets the box: the least-overlap axis of the 6-axis SAT (face normals, then e_k x u; an edge axis has to beat the faces
// by 1e-4, as in box_box), with the closest points of the segment and that box edge, or the segment clipped to the face's side planes and its
// deepest clipped point.  Either way, a normal within CAPSULE_PARALLEL_SIN of a face normal with the segment parallel to that face gives the
// two ends of the clipped segment.
NM_COLD inline bool box_capsule(const Box& b, const Capsule& C, S max_dist, V3& normal, Contacts& pts) {
    const V3 d = C.c - b.c;
    S max_sep = -1e300, best = -1e300, face_best = -1e300;
    int best_k = 0, face_k = 0;
    bool best_edge = false;
    V3 best_n{0, 1, 0}, face_n{0, 1, 0};
NM_ROLLED
    for (int i = 0; i < 6; ++i) {
        V3 n = i < 3 ? b.r.c[i] : cross(b.r.c[i - 3], C.u);
        const S l = len(n);
        if (l < CAPSULE_EDGE_AXIS_MIN) continue;
        n = n * (1 / l);
        if (dot(n, d) < 0) n = -n;
        const S sep = dot(n, d) - box_radius(b, n) - C.h * fabs(dot(C.u, n));
        max_sep = smax(max_sep, sep);
        const S biased = i < 3 ? sep : sep - 1e-4;
        if (biased > best + 1e-9) { best = biased; best_k = i % 3; best_edge = i >= 3; best_n = n; }
        if (i < 3 && sep > face_best + 1e-9) { face_best = sep; face_k = i; face_n = n; }
    }
    int fk = -1;   // the face whose normal the contact normal is, or -1
    if (max_sep > 0) {   // the segment misses the box
        V3 on_seg, on_box;
        const S dist = segment_box_closest(b, C, on_seg, on_box);
        if (dist - C.r > max_dist) return false;
        normal = (on_seg - on_box) * (1 / dist);
NM_ROLLED
        for (int k = 0; k < 3; ++k)
            if (fabs(dot(normal, b.r.c[k])) >= 1 - 0.5 * CAPSULE_PARALLEL_SIN * CAPSULE_PARALLEL_SIN) fk = k;
        if (fk < 0 || fabs(dot(C.u, b.r.c[fk])) > CAPSULE_PARALLEL_SIN) {
            pts.push(on_box, on_seg - normal * C.r);
            return true;
        }
        normal = b.r.c[fk] * (dot(normal, b.r.c[fk]) < 0 ? -1 : 1);
    } else {
        if (best_edge) {
            const V3 n = best_n;
            V3 e = b.c;
NM_ROLLED
            for (int j = 0; j < 3; ++j)
                if (j != best_k) e = e + b.r.c[j] * (comp(b.he, j) * (dot(b.r.c[j], n) > 0 ? 1 : -1));
            S s, t;
            if (!segment_closest(C.c, C.u, C.h, e, b.r.c[best_k], comp(b.he, best_k), s, t)) {
                normal = n;
                pts.push(e + b.r.c[best_k] * t, C.c + C.u * s - n * C.r);
                return true;
            }
            // an end is active: the edge is not the deepest feature, the best face axis is used
        }
        fk = face_k;
        normal = face_n;
    }
    // face contact on face fk (outward normal `normal`): the segment clipped to the face's side planes
    const S face_d = dot(normal, b.c) + comp(b.he, fk);
    S lo, hi;
    if (!capsule_face_clip(b, fk, C, lo, hi)) {   // the segment passes beside the face: its deepest end point
        lo = hi = dot(C.u, normal) > 0 ? -C.h : C.h;
    } else if (fabs(dot(C.u, normal)) > CAPSULE_PARALLEL_SIN || !(lo < hi)) {   // one point: the deepest clipped point
        lo = hi = dot(C.u, normal) > 0 ? lo : hi;
    }
NM_ROLLED
    for (int i = 0; i < (lo < hi ? 2 : 1); ++i) {
        const V3 q = C.c + C.u * (i == 0 ? lo : hi);
        pts.push(q - normal * (dot(normal, q) - face_d), q - normal * C.r);
    }
    return true;
}

// A pair with at least one capsule: the capsule goes first (A's unless only B is one), the result is swapped back as in collide.  Returns the
// normal (from A to B); pts.n == 0 when the pair is farther apart than max_dist.
NM_COLD inline V3 capsule_pair(int type_a, V3 dims_a, Q qa, int type_b, V3 dims_b, V3 pb, Q qb, S max_dist, Contacts& pts) {
    pts.clear();
    const bool cap_b = type_a != SHAPE_CAPSULE;
    const int to = cap_b ? type_a : type_b;
    const V3 dc = cap_b ? dims_b : dims_a, dn = cap_b ? dims_a : dims_b;
    const Q qc = cap_b ? qb : qa, qo = cap_b ? qa : qb;
    const V3 pc = cap_b ? pb : V3{0, 0, 0}, po = cap_b ? V3{0, 0, 0} : pb;
    const Capsule C{pc, rot(qc, {0, 1, 0}), dc.y, dc.x};
    V3 normal{0, 1, 0};
    bool flip;
    if (to == SHAPE_CUBOID) {
        const Box X{po, to_mat(qo), dn};
        box_capsule(X, C, max_dist, normal, pts);
        flip = !cap_b;   // box_capsule reports from the box to the capsule
    } else {
        if (to == SHAPE_CAPSULE) capsule_round(C, po, rot(qo, {0, 1, 0}), dn.y, dn.x, max_dist, normal, pts);
        else capsule_round(C, po, C.u, 0, dn.x, max_dist, normal, pts);
        flip = cap_b;
    }
    if (flip) {
        normal = -normal;
NM_ROLLED
        for (int k = 0; k < pts.n; ++k) { V3 t = pts.p[k].a; pts.p[k].a = pts.p[k].b; pts.p[k].b = t; }
    }
    return normal;
}

// One collider pair -> normal (from A to B) and at most 4 witness pairs.  he = half extents of a cuboid, radius in he.x of a sphere, [radius,
// half length] of a capsule.
// The geometry runs in a frame centred on A, so the result does not depend on where the pair is in the world (the header's absolute
// thresholds, e.g. prune4's 1e-12 depth tie, would otherwise meet the rounding of world coordinates): the witnesses are relative to pa.
// CAPSULES = false compiles the cuboid / sphere pairs alone: the device kernels that run those leave every pair with a capsule to a kernel
// of its own (narrow.cu, contacts.cu), so their code and registers are what they were before capsules existed.
template <bool CAPSULES = true>
NM_HD inline bool collide(int type_a, V3 he_a, V3 pa, Q qa, int type_b, V3 he_b, V3 pb, Q qb, S max_dist, V3& normal, Contacts& pts) {
    pb = pb - pa;
    pa = V3{0, 0, 0};
    bool hit;
    if (type_a == SHAPE_CUBOID && type_b == SHAPE_CUBOID) {
        Box A{pa, to_mat(qa), he_a}, B{pb, to_mat(qb), he_b};
        hit = box_box(A, B, max_dist, normal, pts);
        if (hit) prune4(pts, normal);
    } else if (type_a == SHAPE_SPHERE && type_b == SHAPE_SPHERE) {
        hit = sphere_sphere(pa, he_a.x, pb, he_b.x, max_dist, normal, pts);
    } else if (CAPSULES && (type_a == SHAPE_CAPSULE || type_b == SHAPE_CAPSULE)) {
        normal = capsule_pair(type_a, he_a, qa, type_b, he_b, pb, qb, max_dist, pts);
        hit = pts.n != 0;
    } else if (type_a == SHAPE_CUBOID) {
        Box A{pa, to_mat(qa), he_a};
        hit = box_sphere(A, pb, he_b.x, max_dist, normal, pts);
    } else {
        Box B{pb, to_mat(qb), he_b};
        hit = box_sphere(B, pa, he_a.x, max_dist, normal, pts);
        if (hit) {
            normal = -normal;
            for (int k = 0; k < pts.n; ++k) { V3 t = pts.p[k].a; pts.p[k].a = pts.p[k].b; pts.p[k].b = t; }
        }
    }
    return hit;
}

// A manifold point as the solver's input columns want it (ContactPoint, contact_types/mod.rs:603-660): anchors relative to each body's
// centre of mass, penetration, normal speed.  Without body frames a collider sits at its body's origin and the centre of mass at that origin.
struct PointOut { V3 anchor1, anchor2; S penetration, normal_speed; };

// The body frames of a pair (update_contacts, narrow_phase/system_param.rs:540-570): offset = collider position - body position,
// com = body rotation * local centre of mass.
struct PairFrames { V3 offset1, com1, offset2, com2; };

// From the witness pairs of collide (relative to pa) to the manifold's points: the speculative keep rule of
// narrow_phase/system_param.rs:748-756.  rel = v2 - v1, eff_margin = dt * |rel| (margin = MAX).  Returns the number of points written
// to out[0..4).  FRAMES: every anchor is moved from its collider to its body's centre of mass, (anchor + offset) - com in the reference's
// order (system_param.rs:731-735), before the normal speed and the keep rule read it.
template <bool FRAMES>
NM_HD inline int manifold_points_in(const Contacts& pts, V3 normal, V3 pa, V3 pb, V3 rel, V3 w1, V3 w2, S dt, S eff_margin, const PairFrames* fr,
                                    PointOut out[4]) {
    int m = 0;
    for (int k = 0; k < pts.n && m < 4; ++k) {
        PointOut pt;
        pt.anchor1 = pts.p[k].a;
        pt.anchor2 = pts.p[k].b - (pb - pa);
        if (FRAMES) {
            pt.anchor1 = (pt.anchor1 + fr->offset1) - fr->com1;
            pt.anchor2 = (pt.anchor2 + fr->offset2) - fr->com2;
        }
        pt.penetration = dot(pts.p[k].a - pts.p[k].b, normal);
        V3 rv = rel + cross(w2, pt.anchor2) - cross(w1, pt.anchor1);
        pt.normal_speed = dot(rv, normal);
        bool keep = -pt.penetration < eff_margin || (pt.normal_speed * dt - pt.penetration < eff_margin);
        if (!keep) continue;
        out[m++] = pt;
    }
    return m;
}
NM_HD inline int manifold_points(const Contacts& pts, V3 normal, V3 pa, V3 pb, V3 rel, V3 w1, V3 w2, S dt, S eff_margin, PointOut out[4]) {
    return manifold_points_in<false>(pts, normal, pa, pb, rel, w1, w2, dt, eff_margin, nullptr, out);
}
NM_HD inline int manifold_points(const Contacts& pts, V3 normal, V3 pa, V3 pb, V3 rel, V3 w1, V3 w2, S dt, S eff_margin, const PairFrames& fr,
                                 PointOut out[4]) {
    return manifold_points_in<true>(pts, normal, pa, pb, rel, w1, w2, dt, eff_margin, &fr, out);
}

// ContactManifold::match_contacts with unknown feature ids (contact_types/mod.rs:426-470): a new point inherits the warm-start impulses
// of the first old point whose two anchors both lie within the distance threshold (squared: thr2) of its own, in either body order.
// Returns the index of that old point or -1.
NM_HD inline int match_point(V3 anchor1, V3 anchor2, const V3* old_anchor1, const V3* old_anchor2, int n_old, S thr2) {
    for (int k = 0; k < n_old; ++k) {
        V3 e11 = anchor1 - old_anchor1[k], e22 = anchor2 - old_anchor2[k], e12 = anchor1 - old_anchor2[k], e21 = anchor2 - old_anchor1[k];
        if ((dot(e11, e11) < thr2 && dot(e22, e22) < thr2) || (dot(e12, e12) < thr2 && dot(e21, e21) < thr2)) return k;
    }
    return -1;
}

}  // namespace nm
