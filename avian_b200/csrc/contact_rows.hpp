// One row of the device-resident contact store (csrc/contacts.cu): geometry + match_contacts for the contact edge `e`.  Written once for the
// device kernel (one thread per row) and for the host fixture (avh_rows_narrow: the CPU tests run this very function over numpy rows), like
// narrow_math.hpp which it builds on.
#pragma once
#include <cstdint>

#include "hull_math.hpp"
#include "narrow_math.hpp"

namespace avn {

template <class S>
struct EdgeRows {
    int E;
    uint32_t* c1; uint32_t* c2; uint32_t* b1; uint32_t* b2; uint8_t* live;
    uint8_t* count; uint8_t* disjoint; S* normal; S* a1; S* a2; S* pen; S* ns;
    uint8_t* prev_count; double* prev_a1; double* prev_a2;
    S* ws_n_in; S* ws_t_in; S* ws_n_out; S* ws_t_out; S* nimp_in; S* nimp_out;
    const uint8_t* asleep;   // the row sleeps with an island (NULL = no row does): it is left completely alone
};

template <class S>
struct NarrowEdgeArgs {
    EdgeRows<S> r;
    const uint8_t* shape; const S* dims; const S* pos; const S* rot; const S* lv; const S* av; const S* amin; const S* amax;
    double dt, tol, thr2;
    int match;
};

template <class S> NM_HD inline nm::V3 ldd3(const S* p, size_t i) { return {double(p[3 * i]), double(p[3 * i + 1]), double(p[3 * i + 2])}; }
template <class S> NM_HD inline void std3(S* p, size_t i, nm::V3 v) { p[3 * i] = S(v.x); p[3 * i + 1] = S(v.y); p[3 * i + 2] = S(v.z); }

// The body frames of avn_contacts_set_body_frames on the device (or over host arrays): [B] rows like the velocity columns.
template <class S>
struct BodyFrameCols { const S* pos; const S* rot; const S* com; };   // Position [B][3], Rotation [B][4], local centre of mass [B][3] (NULL = 0)

// The frames of the pair (collider ca at pa on body ba, collider cb at pb on body bb).  rot * com is nm::rot, the expression tree of
// avn::qrot (avn_math.cuh), which the solver's writeback uses for the same product, evaluated in double like the rest of the row.
template <class S>
NM_HD inline nm::PairFrames pair_frames(const BodyFrameCols<S>& f, uint32_t ba, nm::V3 pa, uint32_t bb, nm::V3 pb) {
    nm::PairFrames fr;
    fr.offset1 = pa - ldd3(f.pos, ba);
    fr.offset2 = pb - ldd3(f.pos, bb);
    fr.com1 = nm::V3{0, 0, 0};
    fr.com2 = nm::V3{0, 0, 0};
    if (f.com) {
        const nm::Q q1{double(f.rot[4 * size_t(ba)]), double(f.rot[4 * size_t(ba) + 1]), double(f.rot[4 * size_t(ba) + 2]), double(f.rot[4 * size_t(ba) + 3])};
        const nm::Q q2{double(f.rot[4 * size_t(bb)]), double(f.rot[4 * size_t(bb) + 1]), double(f.rot[4 * size_t(bb) + 2]), double(f.rot[4 * size_t(bb) + 3])};
        fr.com1 = nm::rot(q1, ldd3(f.com, ba));
        fr.com2 = nm::rot(q2, ldd3(f.com, bb));
    }
    return fr;
}

// A live row that names a capsule: the device runs it in a kernel of its own (narrow_capsule_edges_kernel), see nm::collide.
template <class S>
NM_HD inline bool capsule_row(const NarrowEdgeArgs<S>& a, int e) {
    return a.shape && a.r.live[e] && (a.shape[a.r.c1[e]] == nm::SHAPE_CAPSULE || a.shape[a.r.c2[e]] == nm::SHAPE_CAPSULE);
}

// A live row that names a convex hull: the device runs it in a kernel of its own (narrow_hull_edges_kernel), see hm::collide.
template <class S>
NM_HD inline bool hull_row(const NarrowEdgeArgs<S>& a, int e) {
    return a.shape && a.r.live[e] && (a.shape[a.r.c1[e]] == hm::SHAPE_CONVEX_HULL || a.shape[a.r.c2[e]] == hm::SHAPE_CONVEX_HULL);
}

// geometry + match_contacts for every live row (same arithmetic as avh_raw_manifolds + avh_match_raw of the host fixture).  CAPSULES = false:
// the row holds no capsule (the cuboid / sphere kernel).  FRAMES: the anchors are moved to the bodies' centres of mass by the frames `f`
// (nm::manifold_points); without it `f` is not read and the row compiles to what it was before body frames existed.  HULLS: the row names a
// convex hull and runs hm::collide over the hull table `t` (CAPSULES is then not read).
template <class S, bool CAPSULES = true, bool FRAMES = false, bool HULLS = false>
NM_HD inline void narrow_edge_row(const NarrowEdgeArgs<S>& a, int e, const BodyFrameCols<S>& f = BodyFrameCols<S>{}, const hm::Table* t = nullptr) {
    const EdgeRows<S>& r = a.r;
    if (r.asleep && r.asleep[e]) return;   // update_contacts runs over active_pairs only (narrow_phase/system_param.rs:437)
    if (!r.live[e]) { r.count[e] = 0; r.disjoint[e] = 0; return; }
    const uint32_t ca = r.c1[e], cb = r.c2[e], ba = r.b1[e], bb = r.b2[e];
    int np = 0;
    nm::V3 normal{0, 0, 0};
    nm::PointOut out[4];
    bool disjoint = false;
    {
        const nm::V3 mina = ldd3(a.amin, ca), maxa = ldd3(a.amax, ca), minb = ldd3(a.amin, cb), maxb = ldd3(a.amax, cb);
        disjoint = (mina.x > maxb.x || maxa.x < minb.x || mina.y > maxb.y || maxa.y < minb.y || mina.z > maxb.z || maxa.z < minb.z);
    }
    r.disjoint[e] = disjoint ? 1 : 0;
    if (!disjoint) {
        const nm::V3 pa = ldd3(a.pos, ca), pb = ldd3(a.pos, cb);
        const nm::Q qa{double(a.rot[4 * size_t(ca)]), double(a.rot[4 * size_t(ca) + 1]), double(a.rot[4 * size_t(ca) + 2]), double(a.rot[4 * size_t(ca) + 3])};
        const nm::Q qb{double(a.rot[4 * size_t(cb)]), double(a.rot[4 * size_t(cb) + 1]), double(a.rot[4 * size_t(cb) + 2]), double(a.rot[4 * size_t(cb) + 3])};
        const nm::V3 v1 = ldd3(a.lv, ba), v2 = ldd3(a.lv, bb), w1 = ldd3(a.av, ba), w2 = ldd3(a.av, bb);
        const nm::V3 rel = v2 - v1;
        const double eff_margin = a.dt * nm::len(rel);
        const double max_dist = nm::smax(eff_margin, a.tol);
        nm::Contacts pts;
        const int ta = a.shape ? a.shape[ca] : nm::SHAPE_CUBOID, tb = a.shape ? a.shape[cb] : nm::SHAPE_CUBOID;
        if (HULLS ? hm::collide(*t, ta, ldd3(a.dims, ca), pa, qa, tb, ldd3(a.dims, cb), pb, qb, max_dist, normal, pts)
                  : nm::collide<CAPSULES>(ta, ldd3(a.dims, ca), pa, qa, tb, ldd3(a.dims, cb), pb, qb, max_dist, normal, pts)) {
            if (FRAMES) np = nm::manifold_points(pts, normal, pa, pb, rel, w1, w2, a.dt, eff_margin, pair_frames(f, ba, pa, bb, pb), out);
            else np = nm::manifold_points(pts, normal, pa, pb, rel, w1, w2, a.dt, eff_margin, out);
        } else
            normal = nm::V3{0, 0, 0};
    }
    // match_contacts against the manifold of the previous step: the impulses the last solve left (ws_*_out) move to the matching new points
    const int oc = r.prev_count[e];
    nm::V3 oa1[4], oa2[4];
    S on[4], otx[4], oty[4];
    for (int k = 0; k < oc; ++k) {
        const size_t q = size_t(e) * 4 + k;
        oa1[k] = nm::V3{r.prev_a1[3 * q], r.prev_a1[3 * q + 1], r.prev_a1[3 * q + 2]};
        oa2[k] = nm::V3{r.prev_a2[3 * q], r.prev_a2[3 * q + 1], r.prev_a2[3 * q + 2]};
        on[k] = r.ws_n_out[q]; otx[k] = r.ws_t_out[2 * q]; oty[k] = r.ws_t_out[2 * q + 1];
    }
    r.count[e] = uint8_t(np);
    std3(r.normal, size_t(e), normal);
    for (int k = 0; k < 4; ++k) {
        const size_t q = size_t(e) * 4 + k;
        S vn = S(0), vx = S(0), vy = S(0);
        if (k < np) {
            const int j = a.match ? nm::match_point(out[k].anchor1, out[k].anchor2, oa1, oa2, oc, a.thr2) : -1;
            if (j >= 0) { vn = on[j]; vx = otx[j]; vy = oty[j]; }
            std3(r.a1, q, out[k].anchor1);
            std3(r.a2, q, out[k].anchor2);
            r.pen[q] = S(out[k].penetration);
            r.ns[q] = S(out[k].normal_speed);
            r.prev_a1[3 * q] = out[k].anchor1.x; r.prev_a1[3 * q + 1] = out[k].anchor1.y; r.prev_a1[3 * q + 2] = out[k].anchor1.z;
            r.prev_a2[3 * q] = out[k].anchor2.x; r.prev_a2[3 * q + 1] = out[k].anchor2.y; r.prev_a2[3 * q + 2] = out[k].anchor2.z;
        } else {
            std3(r.a1, q, nm::V3{0, 0, 0});
            std3(r.a2, q, nm::V3{0, 0, 0});
            r.pen[q] = S(0);
            r.ns[q] = S(0);
        }
        r.ws_n_in[q] = vn;
        r.ws_t_in[2 * q] = vx;
        r.ws_t_in[2 * q + 1] = vy;
        // "out" always holds the latest impulses of the row: the matched ones now, the solved ones once store_contact_impulses has run
        // for the rows of the constraint graph (rows outside the graph keep the matched values, like the reference's ContactPoints)
        r.ws_n_out[q] = vn;
        r.ws_t_out[2 * q] = vx;
        r.ws_t_out[2 * q + 1] = vy;
    }
    r.prev_count[e] = uint8_t(np);
}


}  // namespace avn
