// Convex hull colliders (DESIGN.md §7k): the table's checks and derived data, and the contact geometry of every pair with a hull, written once
// for the host fixture (g++, -ffp-contract=off) and for the device (nvcc, -fmad=false) like narrow_math.hpp, on which it builds: IEEE double
// throughout, the same expressions in the same order, so the device and the fixture produce the same bits.  parry3d's ConvexPolyhedron and
// its contact routines are not vendored (SURVEY.md §8f #1), so there is no parity claim against parry: the claim is the §7 contract.
#pragma once
#include <cstdint>
#include <utility>
#include <vector>

#include "../../include/avian_b200.h"
#include "hull_table.hpp"
#include "narrow_math.hpp"

namespace hm {

using nm::S;
using nm::V3;
using nm::M3;
using nm::Q;
using nm::Witness;
using nm::dot;
using nm::cross;
using nm::len;
using nm::smax;
using nm::smin;

constexpr int SHAPE_CONVEX_HULL = AVN_SHAPE_CONVEX_HULL;
constexpr int MAX_VERTICES = int(AVN_HULL_MAX_VERTICES), MAX_FACES = int(AVN_HULL_MAX_FACES), MAX_FACE_VERTICES = int(AVN_HULL_MAX_FACE_VERTICES);
// A convex incident face clipped by the side planes of a convex reference face gains at most one vertex per plane.
constexpr int MAX_CLIP = 2 * MAX_FACE_VERTICES;
constexpr S REL_TOL = AVN_HULL_REL_TOL;

// ---- the table -------------------------------------------------------------------------------------------------------------------------
// Derived in double on the host (derive_hulls) and uploaded as is; the layout is Table's (hull_table.hpp).
struct HullSet {
    std::vector<double> vert, plane, centre, radius;   // [V][3], [F][4], [H][3] vertex mean, [H] max |v|
    std::vector<uint32_t> voff, foff, loff, loop, eoff, edge;
};

inline Table view(const HullSet& s) {
    return Table{uint32_t(s.radius.size()), s.vert.data(), s.plane.data(), s.centre.data(), s.radius.data(), s.voff.data(), s.foff.data(),
                 s.loff.data(), s.loop.data(), s.eoff.data(), s.edge.data()};
}

// Checks one table (the ABI's AvnConvexHulls, vertices as doubles) and derives the rest.  Returns NULL or the reason, with the offending hull
// in *at.  Nothing is written to *out unless the table is accepted.
inline const char* derive_hulls(uint32_t H, const uint32_t* voff, const double* vert, const uint32_t* foff, const uint32_t* loff, const uint32_t* loop,
                                HullSet* out, uint32_t* at) {
    *at = 0;
    if (H > AVN_HULL_MAX_COUNT) return "more than AVN_HULL_MAX_COUNT hulls";
    if (!voff || !vert || !foff || !loff || !loop) return "vertex_offsets, vertices, face_offsets, loop_offsets and loop are required";
    if (voff[0] != 0 || foff[0] != 0 || loff[0] != 0) return "offsets must start at 0";
    HullSet s;
    s.voff.assign(voff, voff + H + 1);
    s.foff.assign(foff, foff + H + 1);
    s.eoff.push_back(0);
    for (uint32_t h = 0; h < H; ++h) {
        *at = h;
        if (voff[h + 1] < voff[h] || foff[h + 1] < foff[h]) return "offsets must not decrease";
        const uint32_t nv = voff[h + 1] - voff[h], nf = foff[h + 1] - foff[h];
        if (nv > uint32_t(MAX_VERTICES)) return "more than AVN_HULL_MAX_VERTICES vertices";
        if (nf > uint32_t(MAX_FACES)) return "more than AVN_HULL_MAX_FACES faces";
        if (nv < 4 || nf < 4) return "a closed convex surface has at least 4 vertices and 4 faces";
        const double* v = vert + 3 * size_t(voff[h]);
        auto P = [&](uint32_t k) { return V3{v[3 * k], v[3 * k + 1], v[3 * k + 2]}; };
        V3 lo = P(0), hi = P(0), c{0, 0, 0};
        double radius = 0;
        for (uint32_t k = 0; k < nv; ++k) {
            const V3 p = P(k);
            lo = V3{smin(lo.x, p.x), smin(lo.y, p.y), smin(lo.z, p.z)};
            hi = V3{smax(hi.x, p.x), smax(hi.y, p.y), smax(hi.z, p.z)};
            c = c + p;
            radius = smax(radius, len(p));
        }
        c = c * (1.0 / nv);
        const double size = len(hi - lo), tol = REL_TOL * size;
        if (!(size > 0)) return "a hull's vertices coincide";
        for (uint32_t i = 0; i < nv; ++i)
            for (uint32_t j = i + 1; j < nv; ++j)
                if (len(P(i) - P(j)) <= tol) return "two vertices coincide";
        // directed edges: each once, and its reverse once
        std::vector<int32_t> owner(size_t(nv) * nv, -1);
        uint32_t directed = 0;
        for (uint32_t f = foff[h]; f < foff[h + 1]; ++f) {
            if (loff[f + 1] < loff[f]) return "offsets must not decrease";
            const uint32_t m = loff[f + 1] - loff[f];
            if (m < 3) return "a face loop has fewer than 3 vertices";
            if (m > uint32_t(MAX_FACE_VERTICES)) return "more than AVN_HULL_MAX_FACE_VERTICES vertices on a face";
            const uint32_t* L = loop + loff[f];
            for (uint32_t i = 0; i < m; ++i) {
                if (L[i] >= nv) return "a face loop names a vertex past the hull's vertices";
                for (uint32_t j = i + 1; j < m; ++j)
                    if (L[i] == L[j]) return "a face loop repeats a vertex";
            }
            for (uint32_t i = 0; i < m; ++i) {
                int32_t& o = owner[size_t(L[i]) * nv + L[(i + 1) % m]];
                if (o >= 0) return "a directed edge appears twice: the surface is not manifold or a face is wound inward";
                o = int32_t(f - foff[h]);
                ++directed;
            }
        }
        for (uint32_t a = 0; a < nv; ++a)
            for (uint32_t b = 0; b < nv; ++b)
                if ((owner[size_t(a) * nv + b] >= 0) != (owner[size_t(b) * nv + a] >= 0)) return "an edge has no reverse: the surface is open";
        const uint32_t E = directed / 2;
        if (int64_t(nv) - int64_t(E) + int64_t(nf) != 2) return "V - E + F != 2: the surface is not a sphere";
        // planes (Newell), planarity, area, winding, convexity
        for (uint32_t f = foff[h]; f < foff[h + 1]; ++f) {
            const uint32_t m = loff[f + 1] - loff[f];
            const uint32_t* L = loop + loff[f];
            V3 n{0, 0, 0}, fc{0, 0, 0};
            for (uint32_t i = 0; i < m; ++i) {
                const V3 a = P(L[i]), b = P(L[(i + 1) % m]);
                n = n + V3{(a.y - b.y) * (a.z + b.z), (a.z - b.z) * (a.x + b.x), (a.x - b.x) * (a.y + b.y)};
                fc = fc + a;
            }
            const double l = len(n);   // twice the area
            if (!(0.5 * l > tol * tol)) return "a face has zero area";
            n = n * (1 / l);
            const double d = dot(n, fc * (1.0 / m));
            for (uint32_t i = 0; i < m; ++i)
                if (fabs(dot(n, P(L[i])) - d) > tol) return "a face is not planar";
            if (!(dot(n, c) - d < -tol)) return "a face is wound inward (its normal points into the hull)";
            for (uint32_t k = 0; k < nv; ++k)
                if (dot(n, P(k)) - d > tol) return "the hull is not convex: a vertex lies above a face plane";
            s.plane.insert(s.plane.end(), {n.x, n.y, n.z, d});
            s.loff.push_back(uint32_t(s.loop.size()));
            s.loop.insert(s.loop.end(), L, L + m);
        }
        for (uint32_t a = 0; a < nv; ++a)
            for (uint32_t b = a + 1; b < nv; ++b)
                if (owner[size_t(a) * nv + b] >= 0)
                    s.edge.insert(s.edge.end(), {a, b, uint32_t(owner[size_t(a) * nv + b]), uint32_t(owner[size_t(b) * nv + a])});
        s.eoff.push_back(uint32_t(s.edge.size() / 4));
        s.vert.insert(s.vert.end(), v, v + 3 * size_t(nv));
        s.centre.insert(s.centre.end(), {c.x, c.y, c.z});
        s.radius.push_back(radius);
    }
    s.loff.push_back(uint32_t(s.loop.size()));   // rebuilt in face order: loff indexes s.loop whatever the caller's layout
    *out = std::move(s);
    return nullptr;
}

// ---- geometry ---------------------------------------------------------------------------------------------------------------------------
// One hull in world axes.  The cuboid of a hull-cuboid pair is an 8-vertex, 6-face hull built in local arrays (BoxHull).
struct Hull {
    const double* v; const double* pl; const uint32_t* loff; const uint32_t* loop; const uint32_t* edge;
    int nv, nf, ne;
    M3 r; V3 c;        // pose
    V3 mid;            // the vertex mean, world
    S radius;
};

NM_HD inline V3 xf(const M3& r, V3 v) { return r.c[0] * v.x + r.c[1] * v.y + r.c[2] * v.z; }
NM_HD inline V3 vtx(const Hull& H, int k) { return H.c + xf(H.r, V3{H.v[3 * k], H.v[3 * k + 1], H.v[3 * k + 2]}); }
NM_HD inline V3 fnormal(const Hull& H, int f) { return xf(H.r, V3{H.pl[4 * f], H.pl[4 * f + 1], H.pl[4 * f + 2]}); }
NM_HD inline S foffset(const Hull& H, int f) { return dot(fnormal(H, f), H.c) + H.pl[4 * f + 3]; }
NM_HD inline int fsize(const Hull& H, int f) { return int(H.loff[f + 1] - H.loff[f]); }
NM_HD inline V3 fvtx(const Hull& H, int f, int i) { return vtx(H, int(H.loop[H.loff[f] + uint32_t(i)])); }

NM_HD inline Hull table_hull(const Table& t, uint32_t h, V3 c, Q q) {
    Hull H;
    const uint32_t v0 = t.voff[h], f0 = t.foff[h], e0 = t.eoff[h];
    H.v = t.vert + 3 * size_t(v0);
    H.pl = t.plane + 4 * size_t(f0);
    H.loff = t.loff + f0;
    H.loop = t.loop;
    H.edge = t.edge + 4 * size_t(e0);
    H.nv = int(t.voff[h + 1] - v0); H.nf = int(t.foff[h + 1] - f0); H.ne = int(t.eoff[h + 1] - e0);
    H.r = nm::to_mat(q); H.c = c;
    H.mid = c + xf(H.r, V3{t.centre[3 * h], t.centre[3 * h + 1], t.centre[3 * h + 2]});
    H.radius = t.radius[h];
    return H;
}

// table_hull posed by a given rotation matrix (the spatial queries pose every shape through qm::rot_mat, the normalised rotation)
NM_HD inline Hull table_hull_at(const Table& t, uint32_t h, V3 c, const M3& r) {
    Hull H;
    const uint32_t v0 = t.voff[h], f0 = t.foff[h], e0 = t.eoff[h];
    H.v = t.vert + 3 * size_t(v0);
    H.pl = t.plane + 4 * size_t(f0);
    H.loff = t.loff + f0;
    H.loop = t.loop;
    H.edge = t.edge + 4 * size_t(e0);
    H.nv = int(t.voff[h + 1] - v0); H.nf = int(t.foff[h + 1] - f0); H.ne = int(t.eoff[h + 1] - e0);
    H.r = r; H.c = c;
    H.mid = c + xf(r, V3{t.centre[3 * h], t.centre[3 * h + 1], t.centre[3 * h + 2]});
    H.radius = t.radius[h];
    return H;
}

// A cuboid as a hull: vertex m = (+-he.x, +-he.y, +-he.z) with the sign of bit 0 / 1 / 2 of m; faces +x, -x, +y, -y, +z, -z.
struct BoxHull {
    double v[24], pl[24];
    uint32_t loff[7], loop[24], edge[48];
};
NM_HD inline Hull box_hull(BoxHull& b, V3 he, V3 c, Q q) {
    const uint32_t loops[24] = {1, 3, 7, 5, 0, 4, 6, 2, 2, 6, 7, 3, 0, 1, 5, 4, 4, 5, 7, 6, 0, 2, 3, 1};
    for (int m = 0; m < 8; ++m) {
        b.v[3 * m] = m & 1 ? he.x : -he.x; b.v[3 * m + 1] = m & 2 ? he.y : -he.y; b.v[3 * m + 2] = m & 4 ? he.z : -he.z;
    }
    for (int f = 0; f < 6; ++f) {
        const int k = f >> 1;
        const double s = f & 1 ? -1.0 : 1.0;
        b.pl[4 * f] = k == 0 ? s : 0.0; b.pl[4 * f + 1] = k == 1 ? s : 0.0; b.pl[4 * f + 2] = k == 2 ? s : 0.0;
        b.pl[4 * f + 3] = nm::comp(he, k);
        b.loff[f] = uint32_t(4 * f);
    }
    b.loff[6] = 24;
    for (int i = 0; i < 24; ++i) b.loop[i] = loops[i];
    // the unique edges in the order derive_hulls gives them: by (v0 < v1), with the faces of v0 -> v1 and v1 -> v0
    int ne = 0;
    for (uint32_t a = 0; a < 8; ++a)
        for (uint32_t c2 = a + 1; c2 < 8; ++c2) {
            int fab = -1, fba = -1;
            for (int f = 0; f < 6; ++f)
                for (int i = 0; i < 4; ++i) {
                    const uint32_t x = loops[4 * f + i], y = loops[4 * f + (i + 1) % 4];
                    if (x == a && y == c2) fab = f;
                    if (x == c2 && y == a) fba = f;
                }
            if (fab < 0) continue;
            b.edge[4 * ne] = a; b.edge[4 * ne + 1] = c2; b.edge[4 * ne + 2] = uint32_t(fab); b.edge[4 * ne + 3] = uint32_t(fba);
            ++ne;
        }
    Hull H;
    H.v = b.v; H.pl = b.pl; H.loff = b.loff; H.loop = b.loop; H.edge = b.edge;
    H.nv = 8; H.nf = 6; H.ne = 12;
    H.r = nm::to_mat(q); H.c = c; H.mid = c;
    H.radius = len(he);
    return H;
}

// The raw witness pairs of a hull contact before the reduction to 4: a clipped face has at most MAX_CLIP vertices.
struct Raw {
    int n;
    Witness p[MAX_CLIP];
    NM_HD void push(V3 on_a, V3 on_b) { p[n].a = on_a; p[n].b = on_b; ++n; }
};

// prune4's rule (narrow_math.hpp) over the raw buffer, written into the shared Contacts: the deepest point, the farthest from it, the
// farthest on either side of that segment, survivors in their original order.
NM_HD inline void reduce4(const Raw& raw, V3 n, nm::Contacts& pts) {
    pts.clear();
    if (raw.n <= 4) {
        for (int i = 0; i < raw.n; ++i) pts.push(raw.p[i].a, raw.p[i].b);
        return;
    }
    auto depth = [&](int i) { return dot(raw.p[i].a - raw.p[i].b, n); };
    int p0 = 0;
    for (int i = 1; i < raw.n; ++i) if (depth(i) > depth(p0) + 1e-12) p0 = i;
    int p1 = p0;
    S best = -1;
    for (int i = 0; i < raw.n; ++i) { V3 e = raw.p[i].a - raw.p[p0].a; S v = dot(e, e); if (v > best) { best = v; p1 = i; } }
    V3 dir = cross(raw.p[p1].a - raw.p[p0].a, n);
    int p2 = p0, p3 = p0;
    S mx = 0, mn = 0;
    for (int i = 0; i < raw.n; ++i) {
        S v = dot(raw.p[i].a - raw.p[p0].a, dir);
        if (v > mx) { mx = v; p2 = i; }
        if (v < mn) { mn = v; p3 = i; }
    }
    for (int i = 0; i < raw.n; ++i)
        if (i == p0 || i == p1 || i == p2 || i == p3) pts.push(raw.p[i].a, raw.p[i].b);
}

// Is q (on the plane of face f) inside the face's polygon?  Every side plane: dot(e x n, q - v0) <= 0.
NM_HD inline bool in_face(const Hull& H, int f, V3 n, V3 q) {
    const int m = fsize(H, f);
NM_ROLLED
    for (int i = 0; i < m; ++i) {
        const V3 a = fvtx(H, f, i), b = fvtx(H, f, (i + 1) % m);
        if (dot(cross(b - a, n), q - a) > 0) return false;
    }
    return true;
}

// The point of hull H closest to p, outside H; returns the squared distance.  Faces p projects into, then every edge (its ends included).
NM_COLD inline S point_hull_closest(const Hull& H, V3 p, V3& on) {
    S best = 1e300;
NM_ROLLED
    for (int f = 0; f < H.nf; ++f) {
        const V3 n = fnormal(H, f);
        const S h = dot(n, p) - foffset(H, f);
        if (!(h > 0)) continue;
        const V3 q = p - n * h;
        if (h * h < best && in_face(H, f, n, q)) { best = h * h; on = q; }
    }
NM_ROLLED
    for (int e = 0; e < H.ne; ++e) {
        const V3 a = vtx(H, int(H.edge[4 * e])), b = vtx(H, int(H.edge[4 * e + 1])), ab = b - a;
        const S t = smax(0.0, smin(1.0, dot(p - a, ab) / dot(ab, ab)));
        const V3 q = a + ab * t, d = p - q;
        const S d2 = dot(d, d);
        if (d2 < best) { best = d2; on = q; }
    }
    return best;
}

// An edge as nm::segment_closest wants it: centre, unit direction, half length.
NM_HD inline void edge_seg(const Hull& H, int e, V3& mid, V3& u, S& h) {
    const V3 a = vtx(H, int(H.edge[4 * e])), b = vtx(H, int(H.edge[4 * e + 1])), ab = b - a;
    const S l = len(ab);
    mid = (a + b) * 0.5; u = ab * (1 / l); h = 0.5 * l;
}

// The closest points of two disjoint hulls by feature enumeration: every vertex against every face of the other hull it projects into, and
// every edge against every edge.  Returns the distance.  Rare (separated pairs whose SAT feature is not the closest one): out of line, rolled.
NM_COLD inline S hull_hull_closest(const Hull& A, const Hull& B, V3& on_a, V3& on_b) {
    S best = 1e300;
NM_ROLLED
    for (int side = 0; side < 2; ++side) {
        const Hull& P = side == 0 ? A : B;
        const Hull& O = side == 0 ? B : A;
NM_ROLLED
        for (int k = 0; k < P.nv; ++k) {
            const V3 v = vtx(P, k);
NM_ROLLED
            for (int f = 0; f < O.nf; ++f) {
                const V3 n = fnormal(O, f);
                const S h = dot(n, v) - foffset(O, f);
                if (!(h >= 0) || !(h * h < best)) continue;
                const V3 q = v - n * h;
                if (!in_face(O, f, n, q)) continue;
                best = h * h;
                on_a = side == 0 ? v : q; on_b = side == 0 ? q : v;
            }
        }
    }
NM_ROLLED
    for (int i = 0; i < A.ne; ++i) {
        V3 ma, ua; S ha;
        edge_seg(A, i, ma, ua, ha);
NM_ROLLED
        for (int j = 0; j < B.ne; ++j) {
            V3 mb, ub; S hb;
            edge_seg(B, j, mb, ub, hb);
            S s, t;
            nm::segment_closest(ma, ua, ha, mb, ub, hb, s, t);
            const V3 qa = ma + ua * s, qb = mb + ub * t, e = qb - qa;
            const S d2 = dot(e, e);
            if (d2 < best) { best = d2; on_a = qa; on_b = qb; }
        }
    }
    return sqrt(best);
}

// nm::clip_poly with the output bounded by MAX_CLIP: a convex polygon gains at most one vertex per plane, but rounding can flip the side of
// points lying on the plane, and the fixed buffers must hold whatever comes out.
NM_HD inline int clip_bounded(const V3* in, int n, V3 plane_n, S plane_d, V3* out) {
    int m = 0;
NM_ROLLED
    for (int i = 0; i < n; ++i) {
        const V3 a = in[i], b = in[(i + 1) % n];
        const S da = dot(plane_n, a) - plane_d, db = dot(plane_n, b) - plane_d;
        if (da <= 0 && m < MAX_CLIP) out[m++] = a;
        if (((da < 0 && db > 0) || (da > 0 && db < 0)) && m < MAX_CLIP) out[m++] = a + (b - a) * (da / (da - db));
    }
    return m;
}

// Do the arcs of edge (a, b) of A and edge (c, d) of B (c, d: B's face normals negated) cross on the Gauss map?  Only then is the pair's
// cross product a face of the Minkowski difference, a candidate separating axis (Gregorius, "The Separating Axis Test between Convex
// Polyhedra", GDC 2013).
NM_HD inline bool minkowski_face(V3 a, V3 b, V3 c, V3 d) {
    const V3 bxa = cross(b, a), dxc = cross(d, c);
    const S cba = dot(c, bxa), dba = dot(d, bxa), adc = dot(a, dxc), bdc = dot(b, dxc);
    return cba * dba < 0 && adc * bdc < 0 && cba * bdc > 0;
}

// SAT over A's face normals, B's face normals and the edge pairs that pass minkowski_face, then the closest points of the two supporting
// edges or the incident face clipped against the reference face's side planes: box_box (narrow_math.hpp) for any two hulls, with its bias,
// tie rule and fallbacks.  normal from A to B.
NM_COLD inline bool hull_hull(const Hull& A, const Hull& B, S max_dist, V3& normal, Raw& pts) {
    pts.n = 0;
    S best_sep = -1e300;
    int best_kind = -1, best_i = 0, best_j = 0;
    V3 best_n{0, 1, 0};
NM_ROLLED
    for (int side = 0; side < 2; ++side) {
        const Hull& R = side == 0 ? A : B;
        const Hull& O = side == 0 ? B : A;
NM_ROLLED
        for (int f = 0; f < R.nf; ++f) {
            const V3 n = fnormal(R, f);
            const S d = foffset(R, f);
            S sep = 1e300;
NM_ROLLED
            for (int k = 0; k < O.nv; ++k) sep = smin(sep, dot(n, vtx(O, k)) - d);
            if (sep > best_sep + 1e-9) { best_sep = sep; best_kind = side; best_i = f; best_n = side == 0 ? n : -n; }
        }
    }
    const S face_sep = best_sep;
    const int face_kind = best_kind, face_i = best_i;
    const V3 face_n = best_n;
NM_ROLLED
    for (int i = 0; i < A.ne; ++i) {
        const V3 a = fnormal(A, int(A.edge[4 * i + 2])), b = fnormal(A, int(A.edge[4 * i + 3]));
        V3 ma, ua; S ha;
        edge_seg(A, i, ma, ua, ha);
NM_ROLLED
        for (int j = 0; j < B.ne; ++j) {
            if (!minkowski_face(a, b, -fnormal(B, int(B.edge[4 * j + 2])), -fnormal(B, int(B.edge[4 * j + 3])))) continue;
            V3 mb, ub; S hb;
            edge_seg(B, j, mb, ub, hb);
            V3 n = cross(ua, ub);
            const S l = len(n);
            if (l < 1e-9) continue;
            n = n * (1 / l);
            if (dot(n, ma - A.mid) < 0) n = -n;
            const S sep = dot(n, mb - ma);
            if (sep - 1e-4 > best_sep + 1e-9) { best_sep = sep - 1e-4; best_kind = 2; best_i = i; best_j = j; best_n = n; }
        }
    }
    S sep = best_kind == 2 ? best_sep + 1e-4 : best_sep;
    if (sep > max_dist) return false;
    normal = best_n;
    if (best_kind == 2) {
        V3 ma, ua, mb, ub; S ha, hb, s, t;
        edge_seg(A, best_i, ma, ua, ha);
        edge_seg(B, best_j, mb, ub, hb);
        if (!nm::segment_closest(ma, ua, ha, mb, ub, hb, s, t)) {
            pts.push(ma + ua * s, mb + ub * t);
            return true;
        }
        if (sep > 0) {   // an end is active: the edges are not the closest features
            V3 on_a, on_b;
            const S dist = hull_hull_closest(A, B, on_a, on_b);
            if (dist > max_dist) return false;
            if (dist > 1e-12) normal = (on_b - on_a) * (1 / dist);
            pts.push(on_a, on_b);
            return true;
        }
        sep = face_sep; best_kind = face_kind; best_i = face_i; normal = face_n;
    }
    // face contact: reference hull R (face best_i), incident hull I
    const bool ref_is_a = best_kind == 0;
    const Hull& R = ref_is_a ? A : B;
    const Hull& I = ref_is_a ? B : A;
    const V3 rn = ref_is_a ? normal : -normal;
    int inc = 0;
    S inc_best = 1e300;
NM_ROLLED
    for (int f = 0; f < I.nf; ++f) {
        const S v = dot(fnormal(I, f), rn);
        if (v < inc_best) { inc_best = v; inc = f; }
    }
    V3 poly[MAX_CLIP], tmp[MAX_CLIP];
    int np = fsize(I, inc);
NM_ROLLED
    for (int i = 0; i < np; ++i) poly[i] = fvtx(I, inc, i);
    const int m = fsize(R, best_i);
NM_ROLLED
    for (int i = 0; i < m && np > 0; ++i) {
        const V3 a = fvtx(R, best_i, i), b = fvtx(R, best_i, (i + 1) % m);
        const V3 sn = cross(b - a, rn);
        np = clip_bounded(poly, np, sn, dot(sn, a), tmp);
NM_ROLLED
        for (int k = 0; k < np; ++k) poly[k] = tmp[k];
    }
    const S face_d = foffset(R, best_i);
    S nearest = 1e300;
NM_ROLLED
    for (int k = 0; k < np; ++k) {
        const S dist = dot(rn, poly[k]) - face_d;
        if (dist > max_dist) continue;
        nearest = smin(nearest, dist);
        const V3 on_ref = poly[k] - rn * dist;
        bool dup = false;
NM_ROLLED
        for (int q = 0; q < pts.n; ++q) {
            const V3 e = (ref_is_a ? pts.p[q].b : pts.p[q].a) - poly[k];
            if (dot(e, e) < 1e-12) { dup = true; break; }
        }
        if (dup) continue;
        if (ref_is_a) pts.push(on_ref, poly[k]); else pts.push(poly[k], on_ref);
    }
    if (sep > 0 && nearest > sep + nm::FACE_GAP_SLACK) {
        V3 on_a, on_b;
        const S dist = hull_hull_closest(A, B, on_a, on_b);
        if (nearest > dist + nm::FACE_GAP_SLACK) {
            pts.n = 0;
            if (dist > max_dist) return false;
            if (dist > 1e-12) normal = (on_b - on_a) * (1 / dist);
            pts.push(on_a, on_b);
            return true;
        }
    }
    return pts.n != 0;
}

// Hull A against a sphere (centre cs, radius rs); normal from the hull to the sphere.  A centre outside: its closest point on the hull.  A
// centre inside (no face plane below it): pushed out through the face of largest signed distance.
NM_COLD inline bool hull_sphere(const Hull& A, V3 cs, S rs, S max_dist, V3& normal, Raw& pts) {
    pts.n = 0;
    int fb = 0;
    S hb = -1e300;
NM_ROLLED
    for (int f = 0; f < A.nf; ++f) {
        const S h = dot(fnormal(A, f), cs) - foffset(A, f);
        if (h > hb) { hb = h; fb = f; }
    }
    V3 on;
    if (hb > 0) {
        const S l = sqrt(point_hull_closest(A, cs, on));
        if (l - rs > max_dist) return false;
        normal = l > 1e-9 ? (cs - on) * (1 / l) : fnormal(A, fb);
    } else {
        normal = fnormal(A, fb);
        on = cs - normal * hb;
    }
    pts.push(on, cs - normal * rs);
    return true;
}

// Hull A against capsule C; normal from the hull to the capsule.  box_capsule (narrow_math.hpp) for any hull: a segment disjoint from the hull
// gives its exact closest points; one that meets it the least-overlap axis of a SAT over the face normals and the edge x axis directions (an
// edge axis has to beat the faces by 1e-4), with the closest points of the segment and that edge, or the segment clipped to the face's side
// planes (two points when it lies within CAPSULE_PARALLEL_SIN of the face's plane).
NM_COLD inline bool hull_capsule(const Hull& A, const nm::Capsule& C, S max_dist, V3& normal, Raw& pts) {
    pts.n = 0;
    const V3 p0 = C.c - C.u * C.h, p1 = C.c + C.u * C.h;
    S max_sep = -1e300, best = -1e300, face_best = -1e300;
    int best_i = 0, face_k = 0;
    bool best_edge = false;
    V3 best_n{0, 1, 0}, face_n{0, 1, 0};
NM_ROLLED
    for (int f = 0; f < A.nf; ++f) {
        const V3 n = fnormal(A, f);
        const S sep = smin(dot(n, p0), dot(n, p1)) - foffset(A, f);
        max_sep = smax(max_sep, sep);
        if (sep > best + 1e-9) { best = sep; best_i = f; best_edge = false; best_n = n; }
        if (sep > face_best + 1e-9) { face_best = sep; face_k = f; face_n = n; }
    }
NM_ROLLED
    for (int e = 0; e < A.ne; ++e) {
        // e x u is a face of the Minkowski difference only when the arc of the edge's face normals crosses the great circle normal to the
        // axis; the edge is then the hull's support along the axis, oriented into the arc
        const V3 fa = fnormal(A, int(A.edge[4 * e + 2])), fb = fnormal(A, int(A.edge[4 * e + 3]));
        if (!(dot(fa, C.u) * dot(fb, C.u) < 0)) continue;
        V3 m, u; S h;
        edge_seg(A, e, m, u, h);
        V3 n = cross(u, C.u);
        const S l = len(n);
        if (l < nm::CAPSULE_EDGE_AXIS_MIN) continue;
        n = n * (1 / l);
        if (dot(n, fa + fb) < 0) n = -n;
        const S sep = smin(dot(n, p0), dot(n, p1)) - dot(n, m);
        max_sep = smax(max_sep, sep);
        if (sep - 1e-4 > best + 1e-9) { best = sep - 1e-4; best_i = e; best_edge = true; best_n = n; }
    }
    int fk = -1;
    if (max_sep > 0) {   // the segment misses the hull: its exact closest points (end points against the hull, the segment against every edge)
        V3 on_seg = p0, on_hull;
        S d2 = point_hull_closest(A, p0, on_hull);
        V3 oh;
        const S d2b = point_hull_closest(A, p1, oh);
        if (d2b < d2) { d2 = d2b; on_seg = p1; on_hull = oh; }
NM_ROLLED
        for (int e = 0; e < A.ne; ++e) {
            V3 m, u; S h, s, t;
            edge_seg(A, e, m, u, h);
            nm::segment_closest(C.c, C.u, C.h, m, u, h, s, t);
            const V3 qs = C.c + C.u * s, qe = m + u * t, d = qs - qe;
            if (dot(d, d) < d2) { d2 = dot(d, d); on_seg = qs; on_hull = qe; }
        }
        const S dist = sqrt(d2);
        if (dist - C.r > max_dist) return false;
        normal = (on_seg - on_hull) * (1 / dist);
NM_ROLLED
        for (int f = 0; f < A.nf; ++f)
            if (dot(normal, fnormal(A, f)) >= 1 - 0.5 * nm::CAPSULE_PARALLEL_SIN * nm::CAPSULE_PARALLEL_SIN) fk = f;
        if (fk < 0 || fabs(dot(C.u, fnormal(A, fk))) > nm::CAPSULE_PARALLEL_SIN) {
            pts.push(on_hull, on_seg - normal * C.r);
            return true;
        }
        normal = fnormal(A, fk);
    } else {
        if (best_edge) {
            V3 m, u; S h, s, t;
            edge_seg(A, best_i, m, u, h);
            if (!nm::segment_closest(C.c, C.u, C.h, m, u, h, s, t)) {
                normal = best_n;
                pts.push(m + u * t, C.c + C.u * s - best_n * C.r);
                return true;
            }
        }
        fk = face_k;
        normal = face_n;
    }
    // face contact on face fk: the segment clipped to the face's side planes
    const S face_d = foffset(A, fk);
    S lo = -C.h, hi = C.h;
    bool inside = true;
    const int m = fsize(A, fk);
NM_ROLLED
    for (int i = 0; i < m; ++i) {
        const V3 a = fvtx(A, fk, i), b = fvtx(A, fk, (i + 1) % m);
        V3 sn = cross(b - a, normal);
        sn = sn * (1 / len(sn));
        const S g = dot(sn, C.u), s0 = dot(sn, C.c - a);
        if (fabs(g) < 1e-12) {
            if (s0 > 0) inside = false;
            continue;
        }
        if (g > 0) hi = smin(hi, -s0 / g); else lo = smax(lo, -s0 / g);
    }
    if (!inside || !(lo <= hi)) {
        lo = hi = dot(C.u, normal) > 0 ? -C.h : C.h;
    } else if (fabs(dot(C.u, normal)) > nm::CAPSULE_PARALLEL_SIN || !(lo < hi)) {
        lo = hi = dot(C.u, normal) > 0 ? lo : hi;
    }
NM_ROLLED
    for (int i = 0; i < (lo < hi ? 2 : 1); ++i) {
        const V3 q = C.c + C.u * (i == 0 ? lo : hi);
        pts.push(q - normal * (dot(normal, q) - face_d), q - normal * C.r);
    }
    return true;
}

// A pair with at least one hull, in the frame centred on A like nm::collide: the hull goes first (A's unless only B is one), the result is
// reduced to at most 4 points in that order and swapped back.  dims of a hull: [index, -, -]; the caller has checked the index.  Returns the
// normal (from A to B) through `normal`; false when the pair is farther apart than max_dist.
NM_COLD inline bool collide(const Table& t, int type_a, V3 dims_a, V3 pa, Q qa, int type_b, V3 dims_b, V3 pb, Q qb, S max_dist, V3& normal,
                            nm::Contacts& out) {
    out.clear();
    pb = pb - pa;
    const bool swap = type_a != SHAPE_CONVEX_HULL;
    const int to = swap ? type_a : type_b;
    const V3 dh = swap ? dims_b : dims_a, dn = swap ? dims_a : dims_b;
    const Q qh = swap ? qb : qa, qo = swap ? qa : qb;
    const V3 ph = swap ? pb : V3{0, 0, 0}, po = swap ? V3{0, 0, 0} : pb;
    const Hull X = table_hull(t, uint32_t(dh.x), ph, qh);
    Raw raw;
    raw.n = 0;
    V3 n{0, 1, 0};
    bool hit;
    if (to == SHAPE_CONVEX_HULL || to == nm::SHAPE_CUBOID) {
        BoxHull bh;
        const Hull Y = to == SHAPE_CONVEX_HULL ? table_hull(t, uint32_t(dn.x), po, qo) : box_hull(bh, dn, po, qo);
        const S gap = len(po - ph) - X.radius - Y.radius;   // bounding spheres about the hulls' origins: farther than max_dist apart, no contact
        hit = gap <= max_dist && hull_hull(X, Y, max_dist, n, raw);
    } else if (to == nm::SHAPE_SPHERE) {
        hit = hull_sphere(X, po, dn.x, max_dist, n, raw);
    } else {
        const nm::Capsule C{po, nm::rot(qo, {0, 1, 0}), dn.y, dn.x};
        hit = hull_capsule(X, C, max_dist, n, raw);
    }
    if (!hit) return false;
    reduce4(raw, n, out);
    if (swap) {
        n = -n;
NM_ROLLED
        for (int k = 0; k < out.n; ++k) { V3 w = out.p[k].a; out.p[k].a = out.p[k].b; out.p[k].b = w; }
    }
    normal = n;
    return out.n != 0;
}

}  // namespace hm
