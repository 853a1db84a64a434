// libavian_host.so — the host-side FIXTURE that stands in for the parts of an avian3d app that stay on the CPU
// around the GPU hot path, so the hot path can be exercised and benchmarked without Bevy:
//   * swept collider AABBs        (restates update_aabb for cuboids/spheres/capsules, collider/backend.rs:498-625)
//   * ContactGraph bookkeeping    (pair set, lowest-free ContactId, contact_graph.rs:521-631; id_pool.rs:43-52)
//   * a narrow phase for cuboid / sphere / capsule / convex hull pairs (SAT + face clipping; the reference delegates this arithmetic
//     to parry3d 0.25, which is not vendored, so this is OUR manifold generator: a fixture, identical for the
//     oracle and the GPU path, not a parity claim), contact matching (contact_types/mod.rs:426-470),
//     the status-change loop and ConstraintGraph push/pop colouring (narrow_phase/system_param.rs:136-389,
//     constraint_graph.rs:163-296)
//   * export of the manifolds as per-colour columns in the layout of AvnManifoldColumns.
//   * spatial queries by brute force over every collider (csrc/query_math.hpp): the checker of the device tree (csrc/queries.cu).
//   * swept CCD as the reference's sequential loop (csrc/ccd_math.hpp): the checker of the device pass (csrc/ccd.cu).
//   * move and slide by brute force over every collider (csrc/move_math.hpp): the checker of the move kernel (csrc/queries.cu).
// It contains no solver or broad-phase code: those are the GPU library (product) or oracle/ (tests).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <queue>
#include <unordered_map>
#include <vector>

#include "../../include/avian_b200.h"
#include "../csrc/narrow_math.hpp"
#include "../csrc/hull_math.hpp"
#include "../csrc/hull_query_math.hpp"
#include "../csrc/contact_rows.hpp"
#include "../csrc/query_math.hpp"
#include "../csrc/ccd_math.hpp"
#include "../csrc/move_math.hpp"

namespace {

using namespace nm;  // S = double, V3, Q, M3, Box, Contacts: the manifold geometry shared with the device (csrc/narrow_math.hpp)

inline Q qmul(Q a, Q b) {
    return {a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x,
            a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}
inline Q q_from_scaled_axis(V3 v) {
    S l = len(v);
    if (l == 0) return {0, 0, 0, 1};
    S s = std::sin(l * 0.5) / l;
    return {v.x * s, v.y * s, v.z * s, std::cos(l * 0.5)};
}
template <class T> struct ColR {  // typed reader over a void* column of float or double
    const void* p; bool f64;
    S at(size_t i) const { return f64 ? static_cast<const double*>(p)[i] : S(static_cast<const float*>(p)[i]); }
    V3 v3(size_t i) const { return {at(3 * i), at(3 * i + 1), at(3 * i + 2)}; }
    Q q(size_t i) const { return {at(4 * i), at(4 * i + 1), at(4 * i + 2), at(4 * i + 3)}; }
};
using Col = ColR<void>;
struct ColW {
    void* p; bool f64;
    void set(size_t i, S v) const { if (f64) static_cast<double*>(p)[i] = v; else static_cast<float*>(p)[i] = float(v); }
    void set3(size_t i, V3 v) const { set(3 * i, v.x); set(3 * i + 1, v.y); set(3 * i + 2, v.z); }
};

struct Shape { int type; V3 he; S friction, restitution; };

struct Point {
    V3 anchor1, anchor2;  // world-space offsets from each body's centre of mass
    S penetration, normal_speed;
    S ws_normal = 0, ws_tx = 0, ws_ty = 0, normal_impulse = 0;
};
struct Manifold { V3 normal; std::vector<Point> pts; };
struct Handle { int color; uint32_t local; };

struct Pair {
    uint32_t collider1, collider2, body1, body2;
    uint8_t flags;                 // AVN_PAIR_*
    bool alive = false, touching = false, static1 = false, static2 = false;
    bool asleep = false;           // in ContactGraph::sleeping_pairs (avh_sleep_edges): out of the ConstraintGraph, skipped by the narrow phase
    std::vector<Manifold> manifolds;
    std::vector<Handle> handles;   // ContactEdge::constraint_handles
};

// ConstraintGraph (constraint_graph.rs:39-296)
struct Color {
    std::vector<uint8_t> body_set;
    std::vector<std::pair<uint32_t, uint32_t>> handles;  // (contact id, manifold index)
    bool get(uint32_t i) const { return i < body_set.size() && body_set[i]; }
    void set(uint32_t i) { if (i >= body_set.size()) body_set.resize(size_t(i) + 1, 0); body_set[i] = 1; }
    void unset(uint32_t i) { if (i < body_set.size()) body_set[i] = 0; }
};

struct Pipeline {
    uint32_t n = 0;
    std::vector<Shape> shapes;
    std::vector<uint32_t> order;          // AabbIntervals persistent order (positions -> collider index)
    std::vector<Pair> pairs;              // indexed by ContactId (stable graph edges)
    std::priority_queue<uint32_t, std::vector<uint32_t>, std::greater<uint32_t>> free_ids;  // IdPool: lowest free id
    std::unordered_map<uint64_t, uint32_t> pair_set;  // PairKey -> ContactId
    std::vector<uint32_t> active;         // ContactGraph::active_pairs order
    std::vector<uint8_t> sensor;          // Sensor per collider (empty = none)
    struct Event { uint32_t c1, c2, b1, b2; uint8_t flags; };
    std::vector<Event> started, ended;    // CollisionStart / CollisionEnd of the last status loop (ended: the removals' first)
    std::vector<Event> pending_ended;     // CollisionEnds of removals since the last status loop
    Color colors[AVN_GRAPH_COLOR_COUNT];
    S contact_tolerance = 0.005, length_unit = 1.0;
    // export bookkeeping: the (contact id, manifold, point) of every exported point, in column order
    struct Ref { uint32_t id, mi, pi; };
    std::vector<Ref> export_refs;
};

inline uint64_t pair_key(uint32_t a, uint32_t b) { return a < b ? (uint64_t(a) << 32) | b : (uint64_t(b) << 32) | a; }

// ---- ConstraintGraph::push_manifold / pop_manifold -----------------------------------------------------------
void push_manifold(Pipeline& P, uint32_t id) {
    Pair& pr = P.pairs[id];
    int color = AVN_COLOR_OVERFLOW;
    if (!pr.static1 && !pr.static2) {
        for (int i = 0; i < AVN_DYNAMIC_COLOR_COUNT; ++i) {
            Color& c = P.colors[i];
            if (c.get(pr.body1) || c.get(pr.body2)) continue;
            c.set(pr.body1); c.set(pr.body2); color = i; break;
        }
    } else if (!pr.static1) {
        for (int i = AVN_COLOR_OVERFLOW - 1; i >= 1; --i) {
            Color& c = P.colors[i];
            if (c.get(pr.body1)) continue;
            c.set(pr.body1); color = i; break;
        }
    } else if (!pr.static2) {
        for (int i = AVN_COLOR_OVERFLOW - 1; i >= 1; --i) {
            Color& c = P.colors[i];
            if (c.get(pr.body2)) continue;
            c.set(pr.body2); color = i; break;
        }
    }
    Color& c = P.colors[color];
    uint32_t manifold_index = uint32_t(pr.handles.size());
    pr.handles.push_back({color, uint32_t(c.handles.size())});
    c.handles.push_back({id, manifold_index});
}
void pop_manifold(Pipeline& P, uint32_t id) {
    Pair& pr = P.pairs[id];
    if (pr.handles.empty()) return;
    Handle h = pr.handles.back();
    pr.handles.pop_back();
    Color& c = P.colors[h.color];
    if (h.color != AVN_COLOR_OVERFLOW) { c.unset(pr.body1); c.unset(pr.body2); }
    uint32_t moved = uint32_t(c.handles.size()) - 1;
    c.handles[h.local] = c.handles[moved];
    c.handles.pop_back();
    if (moved != h.local) {
        auto mh = c.handles[h.local];
        P.pairs[mh.first].handles[mh.second].local = h.local;
    }
}

// The row function of the device-resident contact store (csrc/contact_rows.hpp, what csrc/contacts.cu runs one thread per row) over host
// arrays: every live row gets its manifold, matched impulses and history exactly as on the device.  Column layouts as in contacts.cu.
template <class T>
static void rows_narrow(uint32_t E, uint32_t* c1, uint32_t* c2, uint32_t* b1, uint32_t* b2, uint8_t* live, uint8_t* count, uint8_t* disjoint, void* normal, void* a1,
                        void* a2, void* pen, void* ns, uint8_t* prev_count, double* prev_a1, double* prev_a2, void* ws_n_in, void* ws_t_in, void* ws_n_out,
                        void* ws_t_out, const uint8_t* shape, const void* dims, const void* pos, const void* rot, const void* lv, const void* av,
                        const void* amin, const void* amax, double dt, double tol, double length_unit, uint32_t match, const void* body_pos = nullptr,
                        const void* body_rot = nullptr, const void* body_com = nullptr, const hm::HullSet* hulls = nullptr) {
    avn::NarrowEdgeArgs<T> a{};
    a.r.E = int(E);
    a.r.c1 = c1; a.r.c2 = c2; a.r.b1 = b1; a.r.b2 = b2; a.r.live = live; a.r.count = count; a.r.disjoint = disjoint;
    a.r.normal = static_cast<T*>(normal); a.r.a1 = static_cast<T*>(a1); a.r.a2 = static_cast<T*>(a2); a.r.pen = static_cast<T*>(pen); a.r.ns = static_cast<T*>(ns);
    a.r.prev_count = prev_count; a.r.prev_a1 = prev_a1; a.r.prev_a2 = prev_a2;
    a.r.ws_n_in = static_cast<T*>(ws_n_in); a.r.ws_t_in = static_cast<T*>(ws_t_in); a.r.ws_n_out = static_cast<T*>(ws_n_out); a.r.ws_t_out = static_cast<T*>(ws_t_out);
    a.r.nimp_in = nullptr; a.r.nimp_out = nullptr;
    a.shape = shape; a.dims = static_cast<const T*>(dims); a.pos = static_cast<const T*>(pos); a.rot = static_cast<const T*>(rot);
    a.lv = static_cast<const T*>(lv); a.av = static_cast<const T*>(av); a.amin = static_cast<const T*>(amin); a.amax = static_cast<const T*>(amax);
    a.dt = dt; a.tol = tol; a.thr2 = (0.1 * length_unit) * (0.1 * length_unit); a.match = match ? 1 : 0;
    const avn::BodyFrameCols<T> f{static_cast<const T*>(body_pos), static_cast<const T*>(body_rot), static_cast<const T*>(body_com)};
    const hm::Table t = hulls ? hm::view(*hulls) : hm::Table{};
    for (uint32_t e = 0; e < E; ++e) {
        if (hulls && avn::hull_row(a, int(e))) {   // what narrow_hull_edges_kernel runs
            if (body_pos) avn::narrow_edge_row<T, true, true, true>(a, int(e), f, &t);
            else avn::narrow_edge_row<T, true, false, true>(a, int(e), f, &t);
        } else if (body_pos) avn::narrow_edge_row<T, true, true>(a, int(e), f);
        else avn::narrow_edge_row<T>(a, int(e));
    }
}

// The geometry of one pair with the fixture's dispatch: a pair with a convex hull goes to hm::collide over the table (no table: no contact;
// the Python wrappers check the indices), every other pair to nm::collide.
bool collide_any(const hm::HullSet* hulls, int ta, V3 da, V3 pa, Q qa, int tb, V3 db, V3 pb, Q qb, S max_dist, V3& normal, Contacts& pts) {
    if (ta == hm::SHAPE_CONVEX_HULL || tb == hm::SHAPE_CONVEX_HULL) {
        pts.clear();
        return hulls && hm::collide(hm::view(*hulls), ta, da, pa, qa, tb, db, pb, qb, max_dist, normal, pts);
    }
    return collide(ta, da, pa, qa, tb, db, pb, qb, max_dist, normal, pts);
}

// The body frames of a pair over host columns in either scalar (what contact_rows.hpp's pair_frames computes from device columns)
nm::PairFrames host_pair_frames(bool f64, const void* body_pos, const void* body_rot, const void* body_com, uint32_t ba, V3 pa, uint32_t bb, V3 pb) {
    if (f64) return avn::pair_frames(avn::BodyFrameCols<double>{static_cast<const double*>(body_pos), static_cast<const double*>(body_rot),
                                                                static_cast<const double*>(body_com)}, ba, pa, bb, pb);
    return avn::pair_frames(avn::BodyFrameCols<float>{static_cast<const float*>(body_pos), static_cast<const float*>(body_rot),
                                                      static_cast<const float*>(body_com)}, ba, pa, bb, pb);
}

}  // namespace

extern "C" {

struct AvhPipeline;  // opaque = Pipeline

AvhPipeline* avh_create(uint32_t n_bodies) {
    Pipeline* p = new Pipeline();
    p->n = n_bodies;
    p->shapes.assign(n_bodies, Shape{SHAPE_CUBOID, {0.5, 0.5, 0.5}, 0.5, 0.0});
    return reinterpret_cast<AvhPipeline*>(p);
}
void avh_destroy(AvhPipeline* h) { delete reinterpret_cast<Pipeline*>(h); }

// shape_type[n], dims[n][3] (half extents, or radius in [0]), friction[n], restitution[n] — doubles
void avh_set_shapes(AvhPipeline* h, const int32_t* shape_type, const double* dims, const double* friction, const double* restitution) {
    Pipeline& P = *reinterpret_cast<Pipeline*>(h);
    for (uint32_t i = 0; i < P.n; ++i)
        P.shapes[i] = Shape{shape_type[i], {dims[3 * i], dims[3 * i + 1], dims[3 * i + 2]}, friction[i], restitution[i]};
}

// update_aabb (collider/backend.rs:498-625) for the default configuration: speculative margin = MAX, no collision
// margin, collider at the body origin.  AABB = merge(aabb(start pose), aabb(end pose)) grown by contact_tolerance.
void avh_update_aabbs(AvhPipeline* h, uint32_t scalar_bits, const void* position, const void* rotation, const void* linvel, const void* angvel,
                      double dt, void* out_min, void* out_max, const void* hull_table) {
    const hm::HullSet* hulls = static_cast<const hm::HullSet*>(hull_table);
    Pipeline& P = *reinterpret_cast<Pipeline*>(h);
    const bool f64 = scalar_bits == 64;
    Col pos{position, f64}, rt{rotation, f64}, lv{linvel, f64}, av{angvel, f64};
    ColW omin{out_min, f64}, omax{out_max, f64};
    const S tol = P.contact_tolerance * P.length_unit;
    for (uint32_t i = 0; i < P.n; ++i) {
        const Shape& sh = P.shapes[i];
        V3 p0 = pos.v3(i), v = lv.v3(i), w = av.v3(i);
        Q q0 = rt.q(i);
        Q q1 = qmul(q_from_scaled_axis(w * dt), q0);
        S l2 = q1.x * q1.x + q1.y * q1.y + q1.z * q1.z + q1.w * q1.w, k = 0.5 * (3 - l2);
        q1 = {q1.x * k, q1.y * k, q1.z * k, q1.w * k};
        V3 p1 = p0 + v * dt;
        V3 lo{1e300, 1e300, 1e300}, hi{-1e300, -1e300, -1e300};
        for (int e = 0; e < 2; ++e) {
            V3 c = e ? p1 : p0;
            V3 ext;
            if (sh.type == SHAPE_CAPSULE) {   // Capsule::aabb: the segment's end points moved by the pose (nalgebra's quaternion product), loosened by the radius
                const Q q = e ? q1 : q0;
                const V3 b{q.x, q.y, q.z};
                V3 ends[2];
                for (int i = 0; i < 2; ++i) {
                    const V3 v{0, i ? sh.he.y : -sh.he.y, 0};
                    const V3 t = cross(b, v) * 2.0;
                    ends[i] = ((v + cross(b, t)) + t * q.w) + c;
                }
                lo = {std::min(lo.x, std::min(ends[0].x, ends[1].x) - sh.he.x), std::min(lo.y, std::min(ends[0].y, ends[1].y) - sh.he.x),
                      std::min(lo.z, std::min(ends[0].z, ends[1].z) - sh.he.x)};
                hi = {std::max(hi.x, std::max(ends[0].x, ends[1].x) + sh.he.x), std::max(hi.y, std::max(ends[0].y, ends[1].y) + sh.he.x),
                      std::max(hi.z, std::max(ends[0].z, ends[1].z) + sh.he.x)};
                continue;
            }
            if (sh.type == hm::SHAPE_CONVEX_HULL && hulls) {   // ConvexPolyhedron::aabb: every vertex moved by the pose (the product above)
                const Q q = e ? q1 : q0;
                const V3 b{q.x, q.y, q.z};
                const uint32_t hi_ = uint32_t(sh.he.x);
                for (uint32_t k = hulls->voff[hi_]; k < hulls->voff[hi_ + 1]; ++k) {
                    const V3 v{hulls->vert[3 * k], hulls->vert[3 * k + 1], hulls->vert[3 * k + 2]};
                    const V3 t = cross(b, v) * 2.0;
                    const V3 w = ((v + cross(b, t)) + t * q.w) + c;
                    lo = {std::min(lo.x, w.x), std::min(lo.y, w.y), std::min(lo.z, w.z)};
                    hi = {std::max(hi.x, w.x), std::max(hi.y, w.y), std::max(hi.z, w.z)};
                }
                continue;
            }
            if (sh.type == SHAPE_SPHERE) {
                ext = {sh.he.x, sh.he.x, sh.he.x};
            } else {
                M3 m = to_mat(e ? q1 : q0);
                ext = {std::fabs(m.c[0].x) * sh.he.x + std::fabs(m.c[1].x) * sh.he.y + std::fabs(m.c[2].x) * sh.he.z,
                       std::fabs(m.c[0].y) * sh.he.x + std::fabs(m.c[1].y) * sh.he.y + std::fabs(m.c[2].y) * sh.he.z,
                       std::fabs(m.c[0].z) * sh.he.x + std::fabs(m.c[1].z) * sh.he.y + std::fabs(m.c[2].z) * sh.he.z};
            }
            lo = {std::min(lo.x, c.x - ext.x), std::min(lo.y, c.y - ext.y), std::min(lo.z, c.z - ext.z)};
            hi = {std::max(hi.x, c.x + ext.x), std::max(hi.y, c.y + ext.y), std::max(hi.z, c.z + ext.z)};
        }
        omin.set3(i, {lo.x - tol, lo.y - tol, lo.z - tol});
        omax.set3(i, {hi.x + tol, hi.y + tol, hi.z + tol});
    }
}

// AabbIntervals persistent order (broad_phase.rs:296-315).  order[] holds collider indices.
uint32_t avh_get_order(AvhPipeline* h, uint32_t* out) {
    Pipeline& P = *reinterpret_cast<Pipeline*>(h);
    if (P.order.size() != P.n) {  // first use: add_new_aabb_intervals appends in spawn order
        P.order.resize(P.n);
        for (uint32_t i = 0; i < P.n; ++i) P.order[i] = i;
    }
    if (out) std::memcpy(out, P.order.data(), sizeof(uint32_t) * P.n);
    return P.n;
}
void avh_set_order(AvhPipeline* h, const uint32_t* order) {
    Pipeline& P = *reinterpret_cast<Pipeline*>(h);
    P.order.assign(order, order + P.n);
}

uint64_t avh_existing_pairs(AvhPipeline* h, uint64_t* out, uint64_t capacity) {
    Pipeline& P = *reinterpret_cast<Pipeline*>(h);
    uint64_t k = 0;
    for (uint32_t id : P.active) {
        if (out && k < capacity) out[k] = pair_key(P.pairs[id].collider1, P.pairs[id].collider2);
        ++k;
    }
    return k;
}

// ContactGraph::add_edge_and_key_with for each emitted pair, in list order (broad_phase.rs:443-471)
void avh_add_pairs(AvhPipeline* h, const uint32_t* c1, const uint32_t* c2, const uint32_t* b1, const uint32_t* b2, const uint8_t* flags, uint64_t count) {
    Pipeline& P = *reinterpret_cast<Pipeline*>(h);
    for (uint64_t k = 0; k < count; ++k) {
        uint64_t key = pair_key(c1[k], c2[k]);
        if (P.pair_set.count(key)) continue;
        uint32_t id;
        if (!P.free_ids.empty()) { id = P.free_ids.top(); P.free_ids.pop(); }
        else { id = uint32_t(P.pairs.size()); P.pairs.emplace_back(); }
        Pair& pr = P.pairs[id];
        pr = Pair{};
        pr.collider1 = c1[k]; pr.collider2 = c2[k]; pr.body1 = b1[k]; pr.body2 = b2[k]; pr.flags = flags[k]; pr.alive = true;
        // a pair that involves a sensor never generates constraints (narrow_phase/system_param.rs:583-599)
        if (!P.sensor.empty() && (P.sensor[c1[k]] || P.sensor[c2[k]])) pr.flags &= uint8_t(~AVN_PAIR_GENERATE_CONSTRAINTS);
        P.pair_set[key] = id;
        P.active.push_back(id);
    }
}

// the manifolds in the constraint graph; *out_points = their points
static uint32_t graph_size(const Pipeline& P, uint32_t* out_points) {
    uint32_t M = 0, Pn = 0;
    for (int c = 0; c < AVN_GRAPH_COLOR_COUNT; ++c)
        for (auto& hnd : P.colors[c].handles) { ++M; Pn += uint32_t(P.pairs[hnd.first].manifolds[hnd.second].pts.size()); }
    if (out_points) *out_points = Pn;
    return M;
}
uint32_t avh_graph_size(AvhPipeline* h, uint32_t* out_points) { return graph_size(*reinterpret_cast<Pipeline*>(h), out_points); }

// The second half of NarrowPhase::update: status changes in ascending ContactId (system_param.rs:136-389) -> ContactGraph removals and
// ConstraintGraph push / pop.  Returns the number of manifolds in the constraint graph; *out_points = their points.
static uint32_t apply_status_changes(Pipeline& P, std::vector<uint32_t>& changed, const std::vector<uint8_t>& disjoint, const std::vector<uint8_t>& started,
                                     const std::vector<uint8_t>& stopped, const std::vector<int>& count_change, uint32_t* out_points) {
    std::sort(changed.begin(), changed.end());
    P.started.clear();
    P.ended.swap(P.pending_ended);
    P.pending_ended.clear();
    for (uint32_t id : changed) {
        Pair& pr = P.pairs[id];
        const bool gen = pr.flags & AVN_PAIR_GENERATE_CONSTRAINTS;
        const Pipeline::Event ev{pr.collider1, pr.collider2, pr.body1, pr.body2, uint8_t(pr.flags & 0x0f)};
        if (disjoint[id] && pr.touching) P.ended.push_back(ev);   // CollisionEnd (system_param.rs:155-170)
        else if (!disjoint[id] && started[id]) P.started.push_back(ev);
        else if (!disjoint[id] && stopped[id]) P.ended.push_back(ev);
        if (disjoint[id]) {
            if (gen) while (!pr.handles.empty()) pop_manifold(P, id);
            P.pair_set.erase(pair_key(pr.collider1, pr.collider2));
            auto it = std::find(P.active.begin(), P.active.end(), id);  // remove_edge_by_id: swap_remove (contact_graph.rs:615-628)
            if (it != P.active.end()) { *it = P.active.back(); P.active.pop_back(); }
            pr = Pair{};
            P.free_ids.push(id);
        } else if (started[id]) {
            pr.touching = true;
            if (gen) for (size_t k = 0; k < pr.manifolds.size(); ++k) push_manifold(P, id);
        } else if (stopped[id]) {
            pr.touching = false;
            if (gen) while (!pr.handles.empty()) pop_manifold(P, id);
        } else if (pr.touching && gen && count_change[id] > 0) {
            for (int k = 0; k < count_change[id]; ++k) push_manifold(P, id);
        } else if (pr.touching && gen && count_change[id] < 0) {
            for (int k = 0; k < -count_change[id]; ++k) pop_manifold(P, id);
        }
    }
    return graph_size(P, out_points);
}

// remove_collider (narrow_phase/mod.rs:399-459) for each listed collider: every pair that names one of them, in ascending ContactId (the device's
// stated order), queues a CollisionEnd when it was touching, leaves the ConstraintGraph and the ContactGraph.
void avh_remove_colliders(AvhPipeline* h, uint32_t n, const uint32_t* colliders) {
    Pipeline& P = *reinterpret_cast<Pipeline*>(h);
    std::vector<uint8_t> gone(P.n, 0);
    for (uint32_t k = 0; k < n; ++k) if (colliders[k] < P.n) gone[colliders[k]] = 1;
    for (uint32_t id = 0; id < P.pairs.size(); ++id) {
        Pair& pr = P.pairs[id];
        if (!pr.alive || !(gone[pr.collider1] || gone[pr.collider2])) continue;
        if (pr.touching) P.pending_ended.push_back({pr.collider1, pr.collider2, pr.body1, pr.body2, uint8_t(pr.flags & 0x0f)});
        while (!pr.handles.empty()) pop_manifold(P, id);
        P.pair_set.erase(pair_key(pr.collider1, pr.collider2));
        auto it = std::find(P.active.begin(), P.active.end(), id);
        if (it != P.active.end()) { *it = P.active.back(); P.active.pop_back(); }
        pr = Pair{};
        P.free_ids.push(id);
    }
}

// ContactGraph::sleep_entity_with / wake_entity_with (contact_graph.rs:702-826) for the listed ContactIds, in ascending id (the device's stated
// order): a pair put to sleep leaves the ConstraintGraph and keeps its manifolds and impulses; a woken pair that is touching and generates
// constraints is pushed again.  Which edges follow which island is the caller's business.
void avh_sleep_edges(AvhPipeline* h, uint32_t n, const uint32_t* ids) {
    Pipeline& P = *reinterpret_cast<Pipeline*>(h);
    std::vector<uint32_t> list(ids, ids + n);
    std::sort(list.begin(), list.end());
    for (uint32_t id : list) {
        Pair& pr = P.pairs[id];
        if (!pr.alive || pr.asleep) continue;
        pr.asleep = true;
        while (!pr.handles.empty()) pop_manifold(P, id);
    }
}
void avh_wake_edges(AvhPipeline* h, uint32_t n, const uint32_t* ids) {
    Pipeline& P = *reinterpret_cast<Pipeline*>(h);
    std::vector<uint32_t> list(ids, ids + n);
    std::sort(list.begin(), list.end());
    for (uint32_t id : list) {
        Pair& pr = P.pairs[id];
        if (!pr.alive || !pr.asleep) continue;
        pr.asleep = false;
        if (pr.touching && (pr.flags & AVN_PAIR_GENERATE_CONSTRAINTS))
            for (size_t k = 0; k < pr.manifolds.size(); ++k) push_manifold(P, id);
    }
}
// per live pair: ContactId, touching, asleep (arrays sized avh_pair_count(); may be NULL to count)
uint32_t avh_edge_states(AvhPipeline* h, uint32_t* ids, uint8_t* touching, uint8_t* asleep) {
    Pipeline& P = *reinterpret_cast<Pipeline*>(h);
    uint32_t n = 0;
    for (uint32_t id = 0; id < P.pairs.size(); ++id) {
        const Pair& pr = P.pairs[id];
        if (!pr.alive) continue;
        if (ids) { ids[n] = id; touching[n] = pr.touching; asleep[n] = pr.asleep; }
        ++n;
    }
    return n;
}

// The Sensor column (NULL = none): the On<Add, Sensor> / On<Remove, Sensor> observers run remove_collider for every collider whose flag changed.
void avh_set_sensors(AvhPipeline* h, const uint8_t* sensor) {
    Pipeline& P = *reinterpret_cast<Pipeline*>(h);
    std::vector<uint8_t> now(P.n, 0);
    if (sensor) for (uint32_t c = 0; c < P.n; ++c) now[c] = sensor[c] ? 1 : 0;
    std::vector<uint32_t> changed;
    for (uint32_t c = 0; c < P.n; ++c)
        if (now[c] != (P.sensor.empty() ? 0 : P.sensor[c])) changed.push_back(c);
    P.sensor = std::find(now.begin(), now.end(), uint8_t(1)) != now.end() ? now : std::vector<uint8_t>();
    avh_remove_colliders(h, uint32_t(changed.size()), changed.data());
}

// The started (which = 0) or ended (which = 1) list of the last status loop; arrays may be NULL.  Returns the length of the list.
uint32_t avh_events(AvhPipeline* h, uint32_t which, uint32_t* c1, uint32_t* c2, uint32_t* b1, uint32_t* b2, uint8_t* flags) {
    Pipeline& P = *reinterpret_cast<Pipeline*>(h);
    const auto& list = which ? P.ended : P.started;
    for (size_t i = 0; i < list.size(); ++i) {
        if (c1) c1[i] = list[i].c1;
        if (c2) c2[i] = list[i].c2;
        if (b1) b1[i] = list[i].b1;
        if (b2) b2[i] = list[i].b2;
        if (flags) flags[i] = list[i].flags;
    }
    return uint32_t(list.size());
}

// The touching pairs in ascending ContactId with their manifold reduced in slot order in the column type (what avn_contacts_report computes
// from the stored impulses).  Arrays sized by a first call with contact_id == NULL.  Returns the number of entries.
}  // extern "C"
template <class T>
static uint32_t report_rows(Pipeline& P, uint32_t events_only, uint32_t* contact_id, uint32_t* c1, uint32_t* c2, uint32_t* b1, uint32_t* b2, uint8_t* flags,
                            uint8_t* point_count, T* normal, T* total, T* mx, T* deep) {
    uint32_t n = 0;
    for (uint32_t id = 0; id < P.pairs.size(); ++id) {
        const Pair& pr = P.pairs[id];
        if (!pr.alive || !pr.touching || (events_only && !(pr.flags & AVN_PAIR_CONTACT_EVENTS))) continue;
        if (contact_id) {
            contact_id[n] = id; c1[n] = pr.collider1; c2[n] = pr.collider2; b1[n] = pr.body1; b2[n] = pr.body2; flags[n] = uint8_t(pr.flags & 0x0f);
            const Manifold* m = pr.manifolds.empty() ? nullptr : &pr.manifolds[0];
            const int cnt = m ? int(m->pts.size()) : 0;
            point_count[n] = uint8_t(cnt);
            T tot = T(0), big = T(0), d = T(0);
            for (int k = 0; k < cnt; ++k) {
                const T v = T(m->pts[k].normal_impulse);
                tot = tot + v;
                if (v > big) big = v;
                const T p = T(m->pts[k].penetration);
                if (k == 0 || p >= d) d = p;
            }
            const V3 nv = m ? m->normal : V3{0, 0, 0};
            normal[3 * n] = T(nv.x); normal[3 * n + 1] = T(nv.y); normal[3 * n + 2] = T(nv.z);
            total[n] = tot; mx[n] = big; deep[n] = d;
        }
        ++n;
    }
    return n;
}
extern "C" {
uint32_t avh_report(AvhPipeline* h, uint32_t scalar_bits, uint32_t events_only, uint32_t* contact_id, uint32_t* c1, uint32_t* c2, uint32_t* b1, uint32_t* b2,
                    uint8_t* flags, uint8_t* point_count, void* normal, void* total, void* mx, void* deep) {
    Pipeline& P = *reinterpret_cast<Pipeline*>(h);
    if (scalar_bits == 64)
        return report_rows<double>(P, events_only, contact_id, c1, c2, b1, b2, flags, point_count, static_cast<double*>(normal), static_cast<double*>(total),
                                   static_cast<double*>(mx), static_cast<double*>(deep));
    return report_rows<float>(P, events_only, contact_id, c1, c2, b1, b2, flags, point_count, static_cast<float*>(normal), static_cast<float*>(total),
                              static_cast<float*>(mx), static_cast<float*>(deep));
}

// NarrowPhase::update (narrow_phase/system_param.rs:114-400) with the fixture manifold generator.
// kind[n] = AvnBodyKind.  Returns the number of exported manifolds; *out_points = number of points.
uint32_t avh_narrow_phase(AvhPipeline* h, uint32_t scalar_bits, const uint8_t* kind, const void* position, const void* rotation, const void* linvel,
                          const void* angvel, const void* aabb_min, const void* aabb_max, double dt, uint32_t match_contacts, uint32_t* out_points,
                          const void* body_pos, const void* body_rot, const void* body_com, const void* hull_table) {
    Pipeline& P = *reinterpret_cast<Pipeline*>(h);
    const hm::HullSet* hulls = static_cast<const hm::HullSet*>(hull_table);
    const bool f64 = scalar_bits == 64;
    Col pos{position, f64}, rt{rotation, f64}, lv{linvel, f64}, av{angvel, f64}, amin{aabb_min, f64}, amax{aabb_max, f64};
    const S tol = P.contact_tolerance * P.length_unit;
    std::vector<uint32_t> changed;  // contact ids whose status changed
    std::vector<uint8_t> disjoint(P.pairs.size(), 0), started(P.pairs.size(), 0), stopped(P.pairs.size(), 0);
    std::vector<int> count_change(P.pairs.size(), 0);
    Contacts pts;
    for (uint32_t id : P.active) {
        Pair& pr = P.pairs[id];
        if (pr.asleep) continue;   // update_contacts runs over active_pairs only
        const uint32_t a = pr.collider1, b = pr.collider2;
        V3 mina = amin.v3(a), maxa = amax.v3(a), minb = amin.v3(b), maxb = amax.v3(b);
        bool overlap = !(mina.x > maxb.x || maxa.x < minb.x || mina.y > maxb.y || maxa.y < minb.y || mina.z > maxb.z || maxa.z < minb.z);
        if (!overlap) { disjoint[id] = 1; changed.push_back(id); continue; }
        pr.static1 = kind[pr.body1] == AVN_BODY_STATIC;
        pr.static2 = kind[pr.body2] == AVN_BODY_STATIC;
        const Shape& sa = P.shapes[a];
        const Shape& sb = P.shapes[b];
        V3 v1 = lv.v3(pr.body1), v2 = lv.v3(pr.body2), w1 = av.v3(pr.body1), w2 = av.v3(pr.body2);
        V3 rel = v2 - v1;
        S eff_margin = dt * len(rel);  // effective speculative margin (system_param.rs:663-681) with margin = MAX
        S max_dist = std::max(eff_margin, tol);
        std::vector<Manifold> old = std::move(pr.manifolds);
        pr.manifolds.clear();
        V3 normal;
        V3 pa = pos.v3(a), pb = pos.v3(b);
        const bool hit = collide_any(hulls, sa.type, sa.he, pa, rt.q(a), sb.type, sb.he, pb, rt.q(b), max_dist, normal, pts);
        if (hit) {
            PointOut out[4];
            const int np = body_pos ? manifold_points(pts, normal, pa, pb, rel, w1, w2, dt, eff_margin,
                                                      host_pair_frames(f64, body_pos, body_rot, body_com, pr.body1, pa, pr.body2, pb), out)
                                    : manifold_points(pts, normal, pa, pb, rel, w1, w2, dt, eff_margin, out);
            if (np > 0) {
                Manifold m;
                m.normal = normal;
                for (int k = 0; k < np; ++k) {
                    Point pt;
                    pt.anchor1 = out[k].anchor1;
                    pt.anchor2 = out[k].anchor2;
                    pt.penetration = out[k].penetration;
                    pt.normal_speed = out[k].normal_speed;
                    m.pts.push_back(pt);
                }
                pr.manifolds.push_back(std::move(m));
            }
        }
        bool touching = !pr.manifolds.empty();
        if (touching && match_contacts && pr.manifolds.size() <= 4) {
            // ContactManifold::match_contacts with unknown feature ids (contact_types/mod.rs:426-470)
            const S thr2 = (0.1 * P.length_unit) * (0.1 * P.length_unit);
            for (Manifold& m : pr.manifolds)
                for (const Manifold& om : old) {
                    V3 oa1[8], oa2[8];
                    const int n_old = int(std::min<size_t>(om.pts.size(), 8));
                    for (int k = 0; k < n_old; ++k) { oa1[k] = om.pts[k].anchor1; oa2[k] = om.pts[k].anchor2; }
                    for (Point& c : m.pts) {
                        const int k = match_point(c.anchor1, c.anchor2, oa1, oa2, n_old, thr2);
                        if (k >= 0) { c.ws_normal = om.pts[k].ws_normal; c.ws_tx = om.pts[k].ws_tx; c.ws_ty = om.pts[k].ws_ty; }
                    }
                }
        }
        count_change[id] = int(pr.manifolds.size()) - int(old.size());
        if (touching && !pr.touching) { started[id] = 1; changed.push_back(id); }
        else if (!touching && pr.touching) { stopped[id] = 1; changed.push_back(id); }
        else if (count_change[id] != 0) changed.push_back(id);
    }
    return apply_status_changes(P, changed, disjoint, started, stopped, count_change, out_points);
}

// Export the manifolds grouped by colour in manifold_handles order (what prepare_contact_constraints walks,
// solver/plugin.rs:389-434).  Arrays are sized from avh_narrow_phase's return values.
void avh_export_manifolds(AvhPipeline* h, uint32_t scalar_bits, uint32_t* color_offsets /*[25]*/, int32_t* body1, int32_t* body2, void* normal,
                          void* friction, void* restitution, uint32_t* point_offsets, void* anchor1, void* anchor2, void* penetration,
                          void* normal_speed, void* ws_normal, void* ws_tangent) {
    Pipeline& P = *reinterpret_cast<Pipeline*>(h);
    const bool f64 = scalar_bits == 64;
    ColW wn{normal, f64}, wf{friction, f64}, wr{restitution, f64}, wa1{anchor1, f64}, wa2{anchor2, f64}, wp{penetration, f64}, ws{normal_speed, f64},
        wwn{ws_normal, f64}, wwt{ws_tangent, f64};
    P.export_refs.clear();
    uint32_t m = 0, p = 0;
    for (int c = 0; c < AVN_GRAPH_COLOR_COUNT; ++c) {
        color_offsets[c] = m;
        for (auto& hnd : P.colors[c].handles) {
            const Pair& pr = P.pairs[hnd.first];
            const Manifold& mf = pr.manifolds[hnd.second];
            body1[m] = int32_t(pr.body1);
            body2[m] = int32_t(pr.body2);
            wn.set3(m, mf.normal);
            wf.set(m, (P.shapes[pr.collider1].friction + P.shapes[pr.collider2].friction) * 0.5);
            wr.set(m, (P.shapes[pr.collider1].restitution + P.shapes[pr.collider2].restitution) * 0.5);
            point_offsets[m] = p;
            for (uint32_t k = 0; k < mf.pts.size(); ++k) {
                const Point& pt = mf.pts[k];
                wa1.set3(p, pt.anchor1); wa2.set3(p, pt.anchor2);
                wp.set(p, pt.penetration); ws.set(p, pt.normal_speed);
                wwn.set(p, pt.ws_normal); wwt.set(2 * p, pt.ws_tx); wwt.set(2 * p + 1, pt.ws_ty);
                P.export_refs.push_back({hnd.first, hnd.second, k});
                ++p;
            }
            ++m;
        }
    }
    color_offsets[AVN_GRAPH_COLOR_COUNT] = m;
    point_offsets[m] = p;
}

// store_contact_impulses' destination: ContactPoint::{warm_start_*, normal_impulse} (solver/plugin.rs:741-750)
void avh_store_impulses(AvhPipeline* h, uint32_t scalar_bits, const void* ws_normal, const void* ws_tangent, const void* normal_impulse) {
    Pipeline& P = *reinterpret_cast<Pipeline*>(h);
    const bool f64 = scalar_bits == 64;
    Col n{ws_normal, f64}, t{ws_tangent, f64}, ni{normal_impulse, f64};
    for (size_t p = 0; p < P.export_refs.size(); ++p) {
        auto r = P.export_refs[p];
        Point& pt = P.pairs[r.id].manifolds[r.mi].pts[r.pi];
        pt.ws_normal = n.at(p); pt.ws_tx = t.at(2 * p); pt.ws_ty = t.at(2 * p + 1); pt.normal_impulse = ni.at(p);
    }
}

// The geometry stage alone for an explicit list of pairs, in the layout of AvnRawManifolds (4 point slots per pair): the CPU side of the
// device narrow-phase test.  scalar_bits selects the column type; evaluation is in double either way (csrc/narrow_math.hpp).
void avh_raw_manifolds(uint32_t scalar_bits, uint32_t pair_count, const uint32_t* c1, const uint32_t* c2, const uint32_t* b1, const uint32_t* b2,
                       const uint8_t* shape, const void* dims, const void* position, const void* rotation, const void* linvel, const void* angvel,
                       const void* aabb_min, const void* aabb_max, double dt, double tol, uint8_t* point_count, uint8_t* disjoint, void* normal,
                       void* anchor1, void* anchor2, void* penetration, void* normal_speed, double* anchor1_f64, double* anchor2_f64, const void* body_pos,
                       const void* body_rot, const void* body_com, const void* hull_table) {
    const hm::HullSet* hulls = static_cast<const hm::HullSet*>(hull_table);
    const bool f64 = scalar_bits == 64;
    Col dm{dims, f64}, pos{position, f64}, rt{rotation, f64}, lv{linvel, f64}, av{angvel, f64}, amin{aabb_min, f64}, amax{aabb_max, f64};
    ColW on{normal, f64}, oa1{anchor1, f64}, oa2{anchor2, f64}, op{penetration, f64}, os{normal_speed, f64};
    for (uint32_t k = 0; k < pair_count; ++k) {
        const uint32_t a = c1[k], b = c2[k];
        point_count[k] = 0;
        on.set3(k, V3{0, 0, 0});
        for (int p = 0; p < 4; ++p) { oa1.set3(4 * size_t(k) + p, V3{0, 0, 0}); oa2.set3(4 * size_t(k) + p, V3{0, 0, 0}); op.set(4 * size_t(k) + p, 0); os.set(4 * size_t(k) + p, 0); }
        if (aabb_min) {
            V3 mina = amin.v3(a), maxa = amax.v3(a), minb = amin.v3(b), maxb = amax.v3(b);
            bool overlap = !(mina.x > maxb.x || maxa.x < minb.x || mina.y > maxb.y || maxa.y < minb.y || mina.z > maxb.z || maxa.z < minb.z);
            if (disjoint) disjoint[k] = overlap ? 0 : 1;
            if (!overlap) continue;
        } else if (disjoint) {
            disjoint[k] = 0;
        }
        V3 pa = pos.v3(a), pb = pos.v3(b);
        V3 v1 = lv.v3(b1[k]), v2 = lv.v3(b2[k]), w1 = av.v3(b1[k]), w2 = av.v3(b2[k]);
        V3 rel = v2 - v1;
        S eff_margin = dt * len(rel);
        S max_dist = smax(eff_margin, tol);
        V3 nrm;
        Contacts pts;
        int ta = shape ? shape[a] : SHAPE_CUBOID, tb = shape ? shape[b] : SHAPE_CUBOID;
        if (!collide_any(hulls, ta, dm.v3(a), pa, rt.q(a), tb, dm.v3(b), pb, rt.q(b), max_dist, nrm, pts)) continue;
        PointOut out[4];
        int np = body_pos ? manifold_points(pts, nrm, pa, pb, rel, w1, w2, dt, eff_margin, host_pair_frames(f64, body_pos, body_rot, body_com, b1[k], pa, b2[k], pb), out)
                          : manifold_points(pts, nrm, pa, pb, rel, w1, w2, dt, eff_margin, out);
        point_count[k] = uint8_t(np);
        on.set3(k, nrm);
        for (int p = 0; p < np; ++p) {
            oa1.set3(4 * size_t(k) + p, out[p].anchor1);
            oa2.set3(4 * size_t(k) + p, out[p].anchor2);
            if (anchor1_f64)   // unrounded anchors: what the next step's match_contacts compares (the fixture matches in double)
                for (int c = 0; c < 3; ++c) {
                    anchor1_f64[(4 * size_t(k) + p) * 3 + c] = comp(out[p].anchor1, c);
                    anchor2_f64[(4 * size_t(k) + p) * 3 + c] = comp(out[p].anchor2, c);
                }
            op.set(4 * size_t(k) + p, out[p].penetration);
            os.set(4 * size_t(k) + p, out[p].normal_speed);
        }
    }
}

// ---- the graphs and the per-row state in the contact store's terms (SURVEY.md 8f #1/#3): ContactId-indexed edges, 4 point slots per row ----
// The active contact edges in ContactGraph order: edge id (ContactId), colliders, bodies.  Arrays sized avh_pair_count().
uint32_t avh_active_edges(AvhPipeline* h, uint32_t* ids, uint32_t* c1, uint32_t* c2, uint32_t* b1, uint32_t* b2) {
    Pipeline& P = *reinterpret_cast<Pipeline*>(h);
    uint32_t n = 0;
    for (uint32_t id : P.active) {
        const Pair& pr = P.pairs[id];
        ids[n] = id; c1[n] = pr.collider1; c2[n] = pr.collider2; b1[n] = pr.body1; b2[n] = pr.body2;
        ++n;
    }
    return n;
}

// The constraint graph as a colour-major list of edge ids (manifold_handles order) with the per-edge material (what the solver's prepare
// needs besides the geometry).  Arrays sized by the number of manifolds in the graph.
void avh_export_edges(AvhPipeline* h, uint32_t* color_offsets /*[25]*/, uint32_t* edge, int32_t* body1, int32_t* body2, double* friction, double* restitution) {
    Pipeline& P = *reinterpret_cast<Pipeline*>(h);
    uint32_t m = 0;
    for (int c = 0; c < AVN_GRAPH_COLOR_COUNT; ++c) {
        color_offsets[c] = m;
        for (auto& hnd : P.colors[c].handles) {
            const Pair& pr = P.pairs[hnd.first];
            edge[m] = hnd.first;
            body1[m] = int32_t(pr.body1);
            body2[m] = int32_t(pr.body2);
            friction[m] = (P.shapes[pr.collider1].friction + P.shapes[pr.collider2].friction) * 0.5;
            restitution[m] = (P.shapes[pr.collider1].restitution + P.shapes[pr.collider2].restitution) * 0.5;
            ++m;
        }
    }
    color_offsets[AVN_GRAPH_COLOR_COUNT] = m;
}

// match_contacts on edge-indexed resident state (what the device keeps between steps): for edge ids[i] with new_count[i] points whose anchors
// (double, unrounded: the fixture matches in double) are new_a1/new_a2[i][4][3], carry the warm-start impulses over from the matching old
// points and make the new points the resident ones.  ws_n[E][4], ws_t[E][4][2] in the column scalar type.
void avh_match_raw(uint32_t scalar_bits, uint32_t n, const uint32_t* ids, const uint8_t* new_count, const double* new_a1, const double* new_a2,
                   double length_unit, uint32_t match_contacts, uint8_t* prev_count, double* prev_a1, double* prev_a2, void* ws_n, void* ws_t) {
    const bool f64 = scalar_bits == 64;
    Col rn{ws_n, f64}, rtg{ws_t, f64};
    ColW wn{ws_n, f64}, wt{ws_t, f64};
    const S thr2 = (0.1 * length_unit) * (0.1 * length_unit);
    for (uint32_t i = 0; i < n; ++i) {
        const size_t e = ids[i];
        const int nc = new_count[i], oc = prev_count[e];
        V3 oa1[4], oa2[4];
        S on[4], otx[4], oty[4];
        for (int k = 0; k < oc; ++k) {
            oa1[k] = V3{prev_a1[(e * 4 + k) * 3], prev_a1[(e * 4 + k) * 3 + 1], prev_a1[(e * 4 + k) * 3 + 2]};
            oa2[k] = V3{prev_a2[(e * 4 + k) * 3], prev_a2[(e * 4 + k) * 3 + 1], prev_a2[(e * 4 + k) * 3 + 2]};
            on[k] = rn.at(e * 4 + k); otx[k] = rtg.at((e * 4 + k) * 2); oty[k] = rtg.at((e * 4 + k) * 2 + 1);
        }
        for (int k = 0; k < 4; ++k) {
            S vn = 0, vx = 0, vy = 0;
            if (k < nc) {
                const V3 a1{new_a1[(size_t(i) * 4 + k) * 3], new_a1[(size_t(i) * 4 + k) * 3 + 1], new_a1[(size_t(i) * 4 + k) * 3 + 2]};
                const V3 a2{new_a2[(size_t(i) * 4 + k) * 3], new_a2[(size_t(i) * 4 + k) * 3 + 1], new_a2[(size_t(i) * 4 + k) * 3 + 2]};
                const int j = match_contacts ? match_point(a1, a2, oa1, oa2, oc, thr2) : -1;
                if (j >= 0) { vn = on[j]; vx = otx[j]; vy = oty[j]; }
                for (int c = 0; c < 3; ++c) { prev_a1[(e * 4 + k) * 3 + c] = comp(a1, c); prev_a2[(e * 4 + k) * 3 + c] = comp(a2, c); }
            }
            wn.set(e * 4 + k, vn);
            wt.set((e * 4 + k) * 2, vx);
            wt.set((e * 4 + k) * 2 + 1, vy);
        }
        prev_count[e] = uint8_t(nc);
    }
}

// csrc/contact_rows.hpp over host arrays (see rows_narrow above)
void avh_rows_narrow(uint32_t scalar_bits, uint32_t E, uint32_t* c1, uint32_t* c2, uint32_t* b1, uint32_t* b2, uint8_t* live, uint8_t* count, uint8_t* disjoint,
                     void* normal, void* a1, void* a2, void* pen, void* ns, uint8_t* prev_count, double* prev_a1, double* prev_a2, void* ws_n_in, void* ws_t_in,
                     void* ws_n_out, void* ws_t_out, const uint8_t* shape, const void* dims, const void* pos, const void* rot, const void* lv, const void* av,
                     const void* amin, const void* amax, double dt, double tol, double length_unit, uint32_t match) {
    if (scalar_bits == 64)
        rows_narrow<double>(E, c1, c2, b1, b2, live, count, disjoint, normal, a1, a2, pen, ns, prev_count, prev_a1, prev_a2, ws_n_in, ws_t_in, ws_n_out, ws_t_out,
                            shape, dims, pos, rot, lv, av, amin, amax, dt, tol, length_unit, match);
    else
        rows_narrow<float>(E, c1, c2, b1, b2, live, count, disjoint, normal, a1, a2, pen, ns, prev_count, prev_a1, prev_a2, ws_n_in, ws_t_in, ws_n_out, ws_t_out,
                           shape, dims, pos, rot, lv, av, amin, amax, dt, tol, length_unit, match);
}
// avh_rows_narrow with body frames: body_pos [B][3], body_rot [B][4], body_com [B][3] (NULL = 0) in the column scalar.  avh_rows_narrow_hulls:
// the same with the hull table (avh_hulls_create) as the trailing argument; body_pos NULL = no frames.
void avh_rows_narrow_framed(uint32_t scalar_bits, uint32_t E, uint32_t* c1, uint32_t* c2, uint32_t* b1, uint32_t* b2, uint8_t* live, uint8_t* count,
                            uint8_t* disjoint, void* normal, void* a1, void* a2, void* pen, void* ns, uint8_t* prev_count, double* prev_a1, double* prev_a2,
                            void* ws_n_in, void* ws_t_in, void* ws_n_out, void* ws_t_out, const uint8_t* shape, const void* dims, const void* pos,
                            const void* rot, const void* lv, const void* av, const void* amin, const void* amax, double dt, double tol, double length_unit,
                            uint32_t match, const void* body_pos, const void* body_rot, const void* body_com) {
    if (scalar_bits == 64)
        rows_narrow<double>(E, c1, c2, b1, b2, live, count, disjoint, normal, a1, a2, pen, ns, prev_count, prev_a1, prev_a2, ws_n_in, ws_t_in, ws_n_out, ws_t_out,
                            shape, dims, pos, rot, lv, av, amin, amax, dt, tol, length_unit, match, body_pos, body_rot, body_com);
    else
        rows_narrow<float>(E, c1, c2, b1, b2, live, count, disjoint, normal, a1, a2, pen, ns, prev_count, prev_a1, prev_a2, ws_n_in, ws_t_in, ws_n_out, ws_t_out,
                           shape, dims, pos, rot, lv, av, amin, amax, dt, tol, length_unit, match, body_pos, body_rot, body_com);
}
void avh_rows_narrow_hulls(uint32_t scalar_bits, uint32_t E, uint32_t* c1, uint32_t* c2, uint32_t* b1, uint32_t* b2, uint8_t* live, uint8_t* count,
                           uint8_t* disjoint, void* normal, void* a1, void* a2, void* pen, void* ns, uint8_t* prev_count, double* prev_a1, double* prev_a2,
                           void* ws_n_in, void* ws_t_in, void* ws_n_out, void* ws_t_out, const uint8_t* shape, const void* dims, const void* pos,
                           const void* rot, const void* lv, const void* av, const void* amin, const void* amax, double dt, double tol, double length_unit,
                           uint32_t match, const void* body_pos, const void* body_rot, const void* body_com, const void* hull_table) {
    const hm::HullSet* hulls = static_cast<const hm::HullSet*>(hull_table);
    if (scalar_bits == 64)
        rows_narrow<double>(E, c1, c2, b1, b2, live, count, disjoint, normal, a1, a2, pen, ns, prev_count, prev_a1, prev_a2, ws_n_in, ws_t_in, ws_n_out, ws_t_out,
                            shape, dims, pos, rot, lv, av, amin, amax, dt, tol, length_unit, match, body_pos, body_rot, body_com, hulls);
    else
        rows_narrow<float>(E, c1, c2, b1, b2, live, count, disjoint, normal, a1, a2, pen, ns, prev_count, prev_a1, prev_a2, ws_n_in, ws_t_in, ws_n_out, ws_t_out,
                           shape, dims, pos, rot, lv, av, amin, amax, dt, tol, length_unit, match, body_pos, body_rot, body_com, hulls);
}

// The convex hull table of the fixture: avn_set_convex_hulls' checks and derivation (csrc/hull_math.hpp, the same routine), vertices already
// widened to double from the column scalar.  Returns the table, or NULL with the reason in err.  The fixture functions take it as their
// optional trailing argument.
void* avh_hulls_create(uint32_t hull_count, const uint32_t* vertex_offsets, const double* vertices, const uint32_t* face_offsets, const uint32_t* loop_offsets,
                       const uint32_t* loop, char* err, uint32_t err_size) {
    hm::HullSet* s = new hm::HullSet();
    uint32_t at = 0;
    if (const char* why = hm::derive_hulls(hull_count, vertex_offsets, vertices, face_offsets, loop_offsets, loop, s, &at)) {
        snprintf(err, err_size, "hull %u: %s", at, why);
        delete s;
        return nullptr;
    }
    return s;
}
void avh_hulls_destroy(void* hulls) { delete static_cast<hm::HullSet*>(hulls); }
// table queries the tests read: counts, and the derived columns (plane [F][4], edge [E][4], centre [H][3], radius [H])
void avh_hulls_info(const void* hulls, uint32_t* counts /*[4]: H, V, F, E*/, double* plane, uint32_t* edge, uint32_t* eoff, double* centre, double* radius) {
    const hm::HullSet& s = *static_cast<const hm::HullSet*>(hulls);
    counts[0] = uint32_t(s.radius.size()); counts[1] = uint32_t(s.vert.size() / 3); counts[2] = uint32_t(s.plane.size() / 4); counts[3] = uint32_t(s.edge.size() / 4);
    if (plane) std::copy(s.plane.begin(), s.plane.end(), plane);
    if (edge) std::copy(s.edge.begin(), s.edge.end(), edge);
    if (eoff) std::copy(s.eoff.begin(), s.eoff.end(), eoff);
    if (centre) std::copy(s.centre.begin(), s.centre.end(), centre);
    if (radius) std::copy(s.radius.begin(), s.radius.end(), radius);
}

uint32_t avh_pair_count(AvhPipeline* h) { return uint32_t(reinterpret_cast<Pipeline*>(h)->active.size()); }

}  // extern "C"

// ---- spatial queries, brute force over every collider (the checker of csrc/queries.cu; same header, same conventions) ----------------
// Arguments are the ABI structs of avn_query_*; the colliders are passed with every call.  Returns an AvnStatus; avh_query_error() says why.
// scalar_bits: 32 or 64 selects the column type; OR-ed with AVH_CAPSULES (0x100) it also accepts capsule colliders, query shapes and
// characters.  Without that bit a capsule is refused as an unknown shape, as it was before capsules were queried.  OR-ed with AVH_HULLS
// (0x200) it accepts capsules and convex hulls, whose indices the hull table of the avh_*_hulls variants (avh_hulls_create) must hold;
// without it a hull is refused as an unknown shape.  The geometry is always csrc/hull_query_math.hpp's, which gives the CAPS = true bits of
// csrc/query_math.hpp on cuboids, spheres and capsules, and those give the CAPS = false bits on cuboids and spheres.
namespace {
constexpr uint32_t AVH_CAPSULES = 0x100u, AVH_HULLS = 0x200u;
bool bits_f64(uint32_t scalar_bits) { return (scalar_bits & 0xffu) == 64; }
bool bits_hulls(uint32_t scalar_bits) { return (scalar_bits & AVH_HULLS) != 0; }
bool bits_caps(uint32_t scalar_bits) { return (scalar_bits & (AVH_CAPSULES | AVH_HULLS)) != 0; }
uint32_t hull_count(const hm::HullSet* h) { return h ? uint32_t(h->radius.size()) : 0u; }
// the collider column check of the brute force: capsules with AVH_CAPSULES, hulls too with AVH_HULLS
const char* check_query_colliders(uint32_t bits, const AvnQueryColliders* c, const hm::HullSet* h) {
    const uint32_t hc = hull_count(h);
    return qm::check_colliders(c, true, bits_f64(bits), bits_caps(bits), nullptr, bits_hulls(bits) ? &hc : nullptr);
}
thread_local char g_query_error[256];
int query_fail(AvnStatus st, const char* why) {
    snprintf(g_query_error, sizeof g_query_error, "%s", why);
    return st;
}

struct QueryScene {
    const AvnQueryColliders* c; bool f64;
    Col dims, pos, rot;
    hm::Table t;   // the hull table (count 0: none; the checks refuse a hull without one)
    QueryScene(const AvnQueryColliders* cc, bool f, const hm::HullSet* h = nullptr)
        : c(cc), f64(f), dims{cc->dims, f}, pos{cc->position, f}, rot{cc->rotation, f}, t(h ? hm::view(*h) : hm::Table{}) {}
    bool valid(uint32_t i) const { return qm::collider_valid(dims.v3(i), pos.v3(i), rot.q(i)); }
    uint32_t memb(uint32_t i) const { return c->memberships ? c->memberships[i] : 1u; }
};
struct RayView {
    V3 o, d; S maxd; bool solid, ok; uint32_t mask; const uint32_t* xs; uint32_t nx;
};
RayView ray_at(const AvnRayBatch* r, bool f64, uint32_t i) {
    Col o{r->origin, f64}, d{r->direction, f64}, m{r->max_distance, f64};
    RayView v;
    v.o = o.v3(i); v.d = d.v3(i); v.maxd = m.at(i);
    v.solid = r->solid ? r->solid[i] != 0 : true;
    v.mask = r->mask ? r->mask[i] : 0xffffffffu;
    v.xs = r->exclude_offsets ? r->exclude + r->exclude_offsets[i] : nullptr;
    v.nx = r->exclude_offsets ? r->exclude_offsets[i + 1] - r->exclude_offsets[i] : 0u;
    v.ok = qm::ray_finite(v.o, v.d, v.maxd);
    return v;
}
struct RayHit { S t; uint32_t c; V3 n; };
// every hit of one ray, sorted by (t, collider)
void all_hits(const QueryScene& sc, const RayView& v, std::vector<RayHit>& out) {
    out.clear();
    if (!v.ok) return;
    for (uint32_t c = 0; c < sc.c->count; ++c) {
        if (!sc.valid(c) || !qm::passes_filter(sc.memb(c), v.mask, v.xs, v.nx, c)) continue;
        RayHit h{0, c, V3{0, 0, 0}};
        if (qh::ray_collider(sc.t, sc.c->shape[c], sc.dims.v3(c), sc.pos.v3(c), sc.rot.q(c), v.o, v.d, v.maxd, v.solid, h.t, h.n)) out.push_back(h);
    }
    std::sort(out.begin(), out.end(), [](const RayHit& a, const RayHit& b) { return qm::hit_before(a.t, a.c, b.t, b.c); });
}
template <class T>
void query_aabbs(const QueryScene& sc, uint32_t n, const T* mn, const T* mx, std::vector<std::vector<uint32_t>>& per) {
    for (uint32_t c = 0; c < sc.c->count; ++c) {
        if (!sc.valid(c)) continue;
        V3 a, b;
        qh::collider_aabb(sc.t, sc.c->shape[c], sc.dims.v3(c), sc.pos.v3(c), sc.rot.q(c), a, b);
        const T tmn[3] = {T(a.x), T(a.y), T(a.z)}, tmx[3] = {T(b.x), T(b.y), T(b.z)};
        for (uint32_t i = 0; i < n; ++i)
            if (qm::aabb_overlap(mn + 3 * size_t(i), mx + 3 * size_t(i), tmn, tmx)) per[i].push_back(c);
    }
}

int query_inputs(uint32_t scalar_bits, const AvnQueryColliders* c, const AvnRayBatch* r, const hm::HullSet* h) {
    if (const char* why = check_query_colliders(scalar_bits, c, h)) return query_fail(AVN_ERR_INVALID_ARGUMENT, why);
    if (r)
        if (const char* why = qm::check_rays(r)) return query_fail(AVN_ERR_INVALID_ARGUMENT, why);
    return AVN_OK;
}

int query_cast_ray(uint32_t scalar_bits, const AvnQueryColliders* c, const AvnRayBatch* r, AvnRayClosest* out, const hm::HullSet* hs) {
    if (int st = query_inputs(scalar_bits, c, r, hs)) return st;
    if (!out || (r->count && (!out->collider || !out->distance || !out->normal))) return query_fail(AVN_ERR_INVALID_ARGUMENT, "outputs are required");
    const bool f64 = bits_f64(scalar_bits);
    const QueryScene sc(c, f64, hs);
    ColW ot{out->distance, f64}, on{out->normal, f64};
    std::vector<RayHit> hits;
    for (uint32_t i = 0; i < r->count; ++i) {
        all_hits(sc, ray_at(r, f64, i), hits);
        out->collider[i] = hits.empty() ? -1 : int32_t(hits[0].c);
        ot.set(i, hits.empty() ? 0 : hits[0].t);
        on.set3(i, hits.empty() ? V3{0, 0, 0} : hits[0].n);
    }
    return AVN_OK;
}

int query_ray_hits(uint32_t scalar_bits, const AvnQueryColliders* c, const AvnRayBatch* r, AvnHitList* out, const hm::HullSet* hs) {
    if (int st = query_inputs(scalar_bits, c, r, hs)) return st;
    if (!out || !out->offsets || (out->capacity && !out->collider)) return query_fail(AVN_ERR_INVALID_ARGUMENT, "offsets and collider are required");
    const bool f64 = bits_f64(scalar_bits);
    const QueryScene sc(c, f64, hs);
    std::vector<std::vector<RayHit>> per(r->count);
    uint64_t total = 0;
    for (uint32_t i = 0; i < r->count; ++i) {
        all_hits(sc, ray_at(r, f64, i), per[i]);
        const uint32_t mh = r->max_hits ? r->max_hits[i] : 0xffffffffu;
        if (per[i].size() > mh) per[i].resize(mh);
        total += per[i].size();
    }
    out->count = total;
    if (total > out->capacity) return query_fail(AVN_ERR_CAPACITY, "capacity");
    ColW ot{out->distance, f64}, on{out->normal, f64};
    uint64_t k = 0;
    for (uint32_t i = 0; i < r->count; ++i) {
        out->offsets[i] = k;
        for (const RayHit& h : per[i]) {
            out->collider[k] = h.c;
            if (out->distance) ot.set(k, h.t);
            if (out->normal) on.set3(k, h.n);
            ++k;
        }
    }
    out->offsets[r->count] = k;
    return AVN_OK;
}

int query_aabb_intersections(uint32_t scalar_bits, const AvnQueryColliders* c, uint32_t n, const void* mn, const void* mx, AvnHitList* out,
                             const hm::HullSet* hs) {
    if (int st = query_inputs(scalar_bits, c, nullptr, hs)) return st;
    if (n && (!mn || !mx)) return query_fail(AVN_ERR_INVALID_ARGUMENT, "min and max are required");
    if (!out || !out->offsets || (out->capacity && !out->collider)) return query_fail(AVN_ERR_INVALID_ARGUMENT, "offsets and collider are required");
    const QueryScene sc(c, bits_f64(scalar_bits), hs);
    std::vector<std::vector<uint32_t>> per(n);
    if (bits_f64(scalar_bits)) query_aabbs(sc, n, static_cast<const double*>(mn), static_cast<const double*>(mx), per);
    else query_aabbs(sc, n, static_cast<const float*>(mn), static_cast<const float*>(mx), per);
    uint64_t total = 0;
    for (const auto& v : per) total += v.size();
    out->count = total;
    if (total > out->capacity) return query_fail(AVN_ERR_CAPACITY, "capacity");
    uint64_t k = 0;
    for (uint32_t i = 0; i < n; ++i) {
        out->offsets[i] = k;
        for (uint32_t col : per[i]) out->collider[k++] = col;
    }
    out->offsets[n] = k;
    return AVN_OK;
}
}  // namespace

// The brute force's entry points: avh_query_* as before, and avh_query_*_hulls with the fixture's hull table (avh_hulls_create, or NULL) as
// the trailing argument, which AVH_HULLS in scalar_bits enables.  Callers that pass the old argument lists keep reading the same functions.
extern "C" {

const char* avh_query_error() { return g_query_error; }

int avh_query_cast_ray(uint32_t bits, const AvnQueryColliders* c, const AvnRayBatch* r, AvnRayClosest* out) { return query_cast_ray(bits, c, r, out, nullptr); }
int avh_query_cast_ray_hulls(uint32_t bits, const AvnQueryColliders* c, const AvnRayBatch* r, AvnRayClosest* out, const void* h) {
    return query_cast_ray(bits, c, r, out, static_cast<const hm::HullSet*>(h));
}
int avh_query_ray_hits(uint32_t bits, const AvnQueryColliders* c, const AvnRayBatch* r, AvnHitList* out) { return query_ray_hits(bits, c, r, out, nullptr); }
int avh_query_ray_hits_hulls(uint32_t bits, const AvnQueryColliders* c, const AvnRayBatch* r, AvnHitList* out, const void* h) {
    return query_ray_hits(bits, c, r, out, static_cast<const hm::HullSet*>(h));
}
int avh_query_aabb_intersections(uint32_t bits, const AvnQueryColliders* c, uint32_t n, const void* mn, const void* mx, AvnHitList* out) {
    return query_aabb_intersections(bits, c, n, mn, mx, out, nullptr);
}
int avh_query_aabb_intersections_hulls(uint32_t bits, const AvnQueryColliders* c, uint32_t n, const void* mn, const void* mx, AvnHitList* out, const void* h) {
    return query_aabb_intersections(bits, c, n, mn, mx, out, static_cast<const hm::HullSet*>(h));
}

}  // extern "C"

// ---- shape casts, point projection, point and shape intersections, brute force over every collider ------------------------------------
namespace {
struct ShapeView {
    int shape; V3 he, c, d; Q q; S maxd; uint32_t flags, mask; const uint32_t* xs; uint32_t nx; bool ok;
};
ShapeView shape_at(const AvnShapeBatch* s, bool f64, uint32_t i, bool cast) {
    Col dims{s->dims, f64}, pos{s->position, f64}, rot{s->rotation, f64}, dir{s->direction, f64}, md{s->max_distance, f64};
    ShapeView v;
    v.shape = s->shape[i];
    v.he = dims.v3(i); v.c = pos.v3(i); v.q = rot.q(i);
    v.d = cast ? dir.v3(i) : V3{0, 0, 0};
    v.maxd = cast ? md.at(i) : 0;
    v.flags = cast && s->flags ? s->flags[i] : 0u;
    v.mask = s->mask ? s->mask[i] : 0xffffffffu;
    v.xs = s->exclude_offsets ? s->exclude + s->exclude_offsets[i] : nullptr;
    v.nx = s->exclude_offsets ? s->exclude_offsets[i + 1] - s->exclude_offsets[i] : 0u;
    v.ok = cast ? qm::cast_finite(v.he, v.c, v.q, v.d, v.maxd) : qm::collider_valid(v.he, v.c, v.q);
    return v;
}
struct CastHit { S t; uint32_t c; int axis; };
// every hit of one cast, sorted by (t, collider)
void all_cast_hits(const QueryScene& sc, const ShapeView& v, std::vector<CastHit>& out) {
    out.clear();
    if (!v.ok) return;
    for (uint32_t c = 0; c < sc.c->count; ++c) {
        if (!sc.valid(c) || !qm::passes_filter(sc.memb(c), v.mask, v.xs, v.nx, c)) continue;
        CastHit h{0, c, -1};
        if (qh::cast_collider(sc.t, v.shape, v.he, v.c, v.q, v.d, v.maxd, v.flags, sc.c->shape[c], sc.dims.v3(c), sc.pos.v3(c), sc.rot.q(c), h.t, h.axis))
            out.push_back(h);
    }
    std::sort(out.begin(), out.end(), [](const CastHit& a, const CastHit& b) { return qm::hit_before(a.t, a.c, b.t, b.c); });
}
qm::ShapeContact cast_contact_of(const QueryScene& sc, const ShapeView& v, const CastHit& h) {
    qm::ShapeContact k;
    qh::cast_output(sc.t, v.shape, v.he, v.c, v.q, v.d, v.flags, sc.c->shape[h.c], sc.dims.v3(h.c), sc.pos.v3(h.c), sc.rot.q(h.c), h.t, h.axis, k);
    return k;
}
int shape_inputs(uint32_t scalar_bits, const AvnQueryColliders* c, const AvnShapeBatch* s, bool cast, const hm::HullSet* h) {
    if (const char* why = check_query_colliders(scalar_bits, c, h)) return query_fail(AVN_ERR_INVALID_ARGUMENT, why);
    const uint32_t hc = hull_count(h);
    if (const char* why = qm::check_shapes(s, cast, bits_f64(scalar_bits), bits_caps(scalar_bits), nullptr, bits_hulls(scalar_bits) ? &hc : nullptr))
        return query_fail(AVN_ERR_INVALID_ARGUMENT, why);
    return AVN_OK;
}
int point_inputs(uint32_t scalar_bits, const AvnQueryColliders* c, const AvnPointBatch* p, const hm::HullSet* h) {
    if (const char* why = check_query_colliders(scalar_bits, c, h)) return query_fail(AVN_ERR_INVALID_ARGUMENT, why);
    if (const char* why = qm::check_points(p)) return query_fail(AVN_ERR_INVALID_ARGUMENT, why);
    return AVN_OK;
}
int write_list(AvnHitList* out, const std::vector<std::vector<uint32_t>>& per) {
    uint64_t total = 0;
    for (const auto& v : per) total += v.size();
    out->count = total;
    if (total > out->capacity) return query_fail(AVN_ERR_CAPACITY, "capacity");
    uint64_t k = 0;
    for (size_t i = 0; i < per.size(); ++i) {
        out->offsets[i] = k;
        for (uint32_t col : per[i]) out->collider[k++] = col;
    }
    out->offsets[per.size()] = k;
    return AVN_OK;
}

int query_cast_shape(uint32_t scalar_bits, const AvnQueryColliders* c, const AvnShapeBatch* s, AvnShapeClosest* out, const hm::HullSet* hs) {
    if (int st = shape_inputs(scalar_bits, c, s, true, hs)) return st;
    if (!out || (s->count && (!out->collider || !out->distance || !out->point1 || !out->point2 || !out->normal1 || !out->normal2)))
        return query_fail(AVN_ERR_INVALID_ARGUMENT, "outputs are required");
    const bool f64 = bits_f64(scalar_bits);
    const QueryScene sc(c, f64, hs);
    ColW ot{out->distance, f64}, p1{out->point1, f64}, p2{out->point2, f64}, n1{out->normal1, f64}, n2{out->normal2, f64};
    std::vector<CastHit> hits;
    for (uint32_t i = 0; i < s->count; ++i) {
        const ShapeView v = shape_at(s, f64, i, true);
        all_cast_hits(sc, v, hits);
        qm::ShapeContact k{};
        if (!hits.empty()) k = cast_contact_of(sc, v, hits[0]);
        out->collider[i] = hits.empty() ? -1 : int32_t(hits[0].c);
        ot.set(i, hits.empty() ? 0 : hits[0].t);
        p1.set3(i, k.p1); p2.set3(i, k.p2); n1.set3(i, k.n1); n2.set3(i, k.n2);
    }
    return AVN_OK;
}

int query_shape_hits(uint32_t scalar_bits, const AvnQueryColliders* c, const AvnShapeBatch* s, AvnShapeHitList* out, const hm::HullSet* hs) {
    if (int st = shape_inputs(scalar_bits, c, s, true, hs)) return st;
    if (!out || !out->offsets || (out->capacity && !out->collider)) return query_fail(AVN_ERR_INVALID_ARGUMENT, "offsets and collider are required");
    const bool f64 = bits_f64(scalar_bits);
    const QueryScene sc(c, f64, hs);
    std::vector<std::vector<CastHit>> per(s->count);
    uint64_t total = 0;
    for (uint32_t i = 0; i < s->count; ++i) {
        all_cast_hits(sc, shape_at(s, f64, i, true), per[i]);
        const uint32_t mh = s->max_hits ? s->max_hits[i] : 0xffffffffu;
        if (per[i].size() > mh) per[i].resize(mh);
        total += per[i].size();
    }
    out->count = total;
    if (total > out->capacity) return query_fail(AVN_ERR_CAPACITY, "capacity");
    ColW ot{out->distance, f64}, p1{out->point1, f64}, p2{out->point2, f64}, n1{out->normal1, f64}, n2{out->normal2, f64};
    uint64_t k = 0;
    for (uint32_t i = 0; i < s->count; ++i) {
        out->offsets[i] = k;
        const ShapeView v = shape_at(s, f64, i, true);
        for (const CastHit& h : per[i]) {
            const qm::ShapeContact w = cast_contact_of(sc, v, h);
            out->collider[k] = h.c;
            if (out->distance) ot.set(k, h.t);
            if (out->point1) p1.set3(k, w.p1);
            if (out->point2) p2.set3(k, w.p2);
            if (out->normal1) n1.set3(k, w.n1);
            if (out->normal2) n2.set3(k, w.n2);
            ++k;
        }
    }
    out->offsets[s->count] = k;
    return AVN_OK;
}

int query_project_point(uint32_t scalar_bits, const AvnQueryColliders* c, const AvnPointBatch* p, AvnPointProjection* out, const hm::HullSet* hs) {
    if (int st = point_inputs(scalar_bits, c, p, hs)) return st;
    if (!out || (p->count && (!out->collider || !out->point || !out->is_inside))) return query_fail(AVN_ERR_INVALID_ARGUMENT, "outputs are required");
    const bool f64 = bits_f64(scalar_bits);
    const QueryScene sc(c, f64, hs);
    Col pc{p->point, f64};
    ColW op{out->point, f64};
    for (uint32_t i = 0; i < p->count; ++i) {
        const V3 x = pc.v3(i);
        const bool solid = p->solid ? p->solid[i] != 0 : true;
        const uint32_t mask = p->mask ? p->mask[i] : 0xffffffffu;
        const uint32_t* xs = p->exclude_offsets ? p->exclude + p->exclude_offsets[i] : nullptr;
        const uint32_t nx = p->exclude_offsets ? p->exclude_offsets[i + 1] - p->exclude_offsets[i] : 0u;
        S best_d = INFINITY;
        uint32_t best_c = 0xffffffffu;
        V3 best_p{0, 0, 0};
        bool best_in = false;
        if (qm::finite3(x))
            for (uint32_t col = 0; col < c->count; ++col) {
                if (!sc.valid(col) || !qm::passes_filter(sc.memb(col), mask, xs, nx, col)) continue;
                V3 pr;
                bool in;
                const S d = qh::project_point(sc.t, c->shape[col], sc.dims.v3(col), sc.pos.v3(col), sc.rot.q(col), x, solid, pr, in);
                if (qm::hit_before(d, col, best_d, best_c)) { best_d = d; best_c = col; best_p = pr; best_in = in; }
            }
        const bool hit = best_c != 0xffffffffu;
        out->collider[i] = hit ? int32_t(best_c) : -1;
        op.set3(i, best_p);
        out->is_inside[i] = hit && best_in ? 1 : 0;
    }
    return AVN_OK;
}

int query_point_intersections(uint32_t scalar_bits, const AvnQueryColliders* c, const AvnPointBatch* p, AvnHitList* out, const hm::HullSet* hs) {
    if (int st = point_inputs(scalar_bits, c, p, hs)) return st;
    if (!out || !out->offsets || (out->capacity && !out->collider)) return query_fail(AVN_ERR_INVALID_ARGUMENT, "offsets and collider are required");
    const bool f64 = bits_f64(scalar_bits);
    const QueryScene sc(c, f64, hs);
    Col pc{p->point, f64};
    std::vector<std::vector<uint32_t>> per(p->count);
    for (uint32_t i = 0; i < p->count; ++i) {
        const V3 x = pc.v3(i);
        if (!qm::finite3(x)) continue;
        const uint32_t mask = p->mask ? p->mask[i] : 0xffffffffu;
        const uint32_t* xs = p->exclude_offsets ? p->exclude + p->exclude_offsets[i] : nullptr;
        const uint32_t nx = p->exclude_offsets ? p->exclude_offsets[i + 1] - p->exclude_offsets[i] : 0u;
        for (uint32_t col = 0; col < c->count; ++col)
            if (sc.valid(col) && qm::passes_filter(sc.memb(col), mask, xs, nx, col) &&
                qh::contains_point(sc.t, c->shape[col], sc.dims.v3(col), sc.pos.v3(col), sc.rot.q(col), x))
                per[i].push_back(col);
    }
    return write_list(out, per);
}

int query_shape_intersections(uint32_t scalar_bits, const AvnQueryColliders* c, const AvnShapeBatch* s, AvnHitList* out, const hm::HullSet* hs) {
    if (int st = shape_inputs(scalar_bits, c, s, false, hs)) return st;
    if (!out || !out->offsets || (out->capacity && !out->collider)) return query_fail(AVN_ERR_INVALID_ARGUMENT, "offsets and collider are required");
    const bool f64 = bits_f64(scalar_bits);
    const QueryScene sc(c, f64, hs);
    std::vector<std::vector<uint32_t>> per(s->count);
    for (uint32_t i = 0; i < s->count; ++i) {
        const ShapeView v = shape_at(s, f64, i, false);
        if (!v.ok) continue;
        for (uint32_t col = 0; col < c->count; ++col)
            if (sc.valid(col) && qm::passes_filter(sc.memb(col), v.mask, v.xs, v.nx, col) &&
                qh::shapes_intersect(sc.t, v.shape, v.he, v.c, v.q, c->shape[col], sc.dims.v3(col), sc.pos.v3(col), sc.rot.q(col)))
                per[i].push_back(col);
    }
    return write_list(out, per);
}
}  // namespace

extern "C" {

#define AVH_QUERY_PAIR(name, Batch, Out)                                                                                              \
    int avh_query_##name(uint32_t bits, const AvnQueryColliders* c, const Batch* b, Out* out) { return query_##name(bits, c, b, out, nullptr); } \
    int avh_query_##name##_hulls(uint32_t bits, const AvnQueryColliders* c, const Batch* b, Out* out, const void* h) {                   \
        return query_##name(bits, c, b, out, static_cast<const hm::HullSet*>(h));                                                     \
    }
AVH_QUERY_PAIR(cast_shape, AvnShapeBatch, AvnShapeClosest)
AVH_QUERY_PAIR(shape_hits, AvnShapeBatch, AvnShapeHitList)
AVH_QUERY_PAIR(project_point, AvnPointBatch, AvnPointProjection)
AVH_QUERY_PAIR(point_intersections, AvnPointBatch, AvnHitList)
AVH_QUERY_PAIR(shape_intersections, AvnShapeBatch, AvnHitList)
#undef AVH_QUERY_PAIR

}  // extern "C"

// ---- move and slide, brute force over every collider (the checker of q_move in csrc/queries.cu; same header, csrc/move_math.hpp) ------
namespace {
template <class T>
struct HostMoveScene {
    const QueryScene& sc;
    const uint8_t* valid; const T* tmn; const T* tmx;   // per collider: in the scene, tight AABB rounded to T
    uint32_t mask, nx;
    const uint32_t* xs;
    const uint8_t* ignored;

    bool pass(uint32_t c) const { return qm::passes_filter(sc.memb(c), mask, xs, nx, c) && !(ignored && ignored[c]); }
    void collider(uint32_t c, int& s, V3& he, V3& p, Q& q) const { s = sc.c->shape[c]; he = sc.dims.v3(c); p = sc.pos.v3(c); q = sc.rot.q(c); }
    const hm::Table& hulls() const { return sc.t; }
    bool cast(int shape, V3 he, V3 ctr, Q q, V3 d, double maxd, double& t_out, uint32_t& c_out, int& axis_out) const {
        double best_t = INFINITY;
        uint32_t best_c = 0xffffffffu;
        int best_axis = -1;
        for (uint32_t c = 0; c < sc.c->count; ++c) {
            if (!valid[c] || !pass(c)) continue;
            double th;
            int ax;
            if (qh::cast_collider(sc.t, shape, he, ctr, q, d, maxd, qm::CAST_IGNORE_ORIGIN_PENETRATION, sc.c->shape[c], sc.dims.v3(c), sc.pos.v3(c), sc.rot.q(c), th, ax) &&
                qm::hit_before(th, c, best_t, best_c)) {
                best_t = th; best_c = c; best_axis = ax;
            }
        }
        if (best_c == 0xffffffffu) return false;
        t_out = best_t; c_out = best_c; axis_out = best_axis;
        return true;
    }
    template <class F>
    void candidates(const T lo[3], const T hi[3], F fn) const {
        for (uint32_t c = 0; c < sc.c->count; ++c)
            if (valid[c] && qm::aabb_overlap(lo, hi, tmn + 3 * size_t(c), tmx + 3 * size_t(c)) && pass(c)) fn(c);
    }
};

template <class T>
struct HostMoveHits {
    int32_t* c; void* d; void* t; void* p; void* n;
    size_t base;
    void sweep(uint32_t it, uint32_t col, T safe, T toi, mv::T3<T> p1, mv::T3<T> n1) {
        const size_t o = base + it;
        if (c) c[o] = int32_t(col);
        if (d) static_cast<T*>(d)[o] = safe;
        if (t) static_cast<T*>(t)[o] = toi;
        if (p) { T* q = static_cast<T*>(p) + 3 * o; q[0] = p1.x; q[1] = p1.y; q[2] = p1.z; }
        if (n) { T* q = static_cast<T*>(n) + 3 * o; q[0] = n1.x; q[1] = n1.y; q[2] = n1.z; }
    }
};

template <class T>
void move_all(const AvnQueryColliders* c, const AvnMoveConfig* cfg, const AvnMoveBatch* b, AvnMoveResult* out, const hm::HullSet* hs) {
    const QueryScene sc(c, sizeof(T) == 8, hs);
    const uint32_t C = c->count;
    std::vector<uint8_t> valid(C);
    std::vector<T> tmn(3 * size_t(C)), tmx(3 * size_t(C));
    for (uint32_t k = 0; k < C; ++k) {
        valid[k] = sc.valid(k);
        if (!valid[k]) continue;
        V3 a, e;
        qh::collider_aabb(sc.t, c->shape[k], sc.dims.v3(k), sc.pos.v3(k), sc.rot.q(k), a, e);
        tmn[3 * k] = T(a.x); tmn[3 * k + 1] = T(a.y); tmn[3 * k + 2] = T(a.z);
        tmx[3 * k] = T(e.x); tmx[3 * k + 1] = T(e.y); tmx[3 * k + 2] = T(e.z);
    }
    const mv::Config<T> mc = mv::config_of<T>(cfg);
    const T* dims = static_cast<const T*>(b->dims);
    const T* pos = static_cast<const T*>(b->position);
    const T* rot = static_cast<const T*>(b->rotation);
    const T* vel = static_cast<const T*>(b->velocity);
    const T* planes = static_cast<const T*>(b->planes);
    T* opos = static_cast<T*>(out->position);
    T* ovel = static_cast<T*>(out->velocity);
    const uint32_t iters = cfg->move_and_slide_iterations;
    for (uint32_t i = 0; i < b->count; ++i) {
        HostMoveHits<T> hits{out->hit_collider, out->hit_distance, out->hit_toi, out->hit_point, out->hit_normal, size_t(i) * iters};
        for (uint32_t it = 0; it < iters; ++it) hits.sweep(it, 0xffffffffu, T(0), T(0), mv::T3<T>{0, 0, 0}, mv::T3<T>{0, 0, 0});
        const mv::Body bd{int(b->shape[i]), V3{S(dims[3 * i]), S(dims[3 * i + 1]), S(dims[3 * i + 2])},
                          Q{S(rot[4 * i]), S(rot[4 * i + 1]), S(rot[4 * i + 2]), S(rot[4 * i + 3])}};
        mv::T3<T> p{pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]}, v{vel[3 * i], vel[3 * i + 1], vel[3 * i + 2]};
        if (qm::collider_valid(bd.he, mv::to_v3(p), bd.q) && qm::finite3(mv::to_v3(v))) {
            mv::T3<float> init[mv::MAX_PLANES];
            int ni = 0;
            if (b->plane_offsets)
                for (uint32_t k = b->plane_offsets[i]; k < b->plane_offsets[i + 1]; ++k)
                    init[ni++] = mv::plane_dir(mv::T3<T>{planes[3 * k], planes[3 * k + 1], planes[3 * k + 2]});
            const HostMoveScene<T> ms{sc, valid.data(), tmn.data(), tmx.data(), b->mask ? b->mask[i] : 0xffffffffu,
                                      b->exclude_offsets ? b->exclude_offsets[i + 1] - b->exclude_offsets[i] : 0u,
                                      b->exclude_offsets ? b->exclude + b->exclude_offsets[i] : nullptr, cfg->ignored};
            mv::move_and_slide<2>(ms, mc, bd, p, v, init, ni, hits);
        }
        opos[3 * i] = p.x; opos[3 * i + 1] = p.y; opos[3 * i + 2] = p.z;
        ovel[3 * i] = v.x; ovel[3 * i + 1] = v.y; ovel[3 * i + 2] = v.z;
    }
}
int move_and_slide_all(uint32_t scalar_bits, const AvnQueryColliders* c, const AvnMoveConfig* cfg, const AvnMoveBatch* b, AvnMoveResult* out, const hm::HullSet* hs) {
    if (const char* why = check_query_colliders(scalar_bits, c, hs)) return query_fail(AVN_ERR_INVALID_ARGUMENT, why);
    const uint32_t hc = hull_count(hs);
    if (const char* why = mv::check_move(cfg, b, bits_f64(scalar_bits), c->count, bits_caps(scalar_bits), nullptr, bits_hulls(scalar_bits) ? &hc : nullptr))
        return query_fail(AVN_ERR_INVALID_ARGUMENT, why);
    if (!out || (b->count && (!out->position || !out->velocity))) return query_fail(AVN_ERR_INVALID_ARGUMENT, "position and velocity outputs are required");
    out->kernel_ms = 0.f;
    if (bits_f64(scalar_bits)) move_all<double>(c, cfg, b, out, hs);
    else move_all<float>(c, cfg, b, out, hs);
    return AVN_OK;
}
}  // namespace

extern "C" {

// MoveAndSlide::move_and_slide for every character of the batch against every collider: the same output as avn_move_and_slide.
// avh_move_and_slide_hulls: the same with the hull table (AVH_HULLS).
int avh_move_and_slide(uint32_t scalar_bits, const AvnQueryColliders* c, const AvnMoveConfig* cfg, const AvnMoveBatch* b, AvnMoveResult* out) {
    return move_and_slide_all(scalar_bits, c, cfg, b, out, nullptr);
}
int avh_move_and_slide_hulls(uint32_t scalar_bits, const AvnQueryColliders* c, const AvnMoveConfig* cfg, const AvnMoveBatch* b, AvnMoveResult* out,
                             const void* hull_table) {
    return move_and_slide_all(scalar_bits, c, cfg, b, out, static_cast<const hm::HullSet*>(hull_table));
}

// test infrastructure: the shared project_velocity (velocity_project.rs:122-324) on one velocity, normals as f32 Dirs
void avh_move_project_velocity(uint32_t scalar_bits, const void* v, const float* normals, uint32_t n, void* out) {
    std::vector<mv::T3<float>> ns(n);
    for (uint32_t k = 0; k < n; ++k) ns[k] = mv::T3<float>{normals[3 * k], normals[3 * k + 1], normals[3 * k + 2]};
    if (scalar_bits == 64) {
        const double* x = static_cast<const double*>(v);
        const mv::T3<double> r = mv::project_velocity(mv::T3<double>{x[0], x[1], x[2]}, ns.data(), int(n));
        double* o = static_cast<double*>(out);
        o[0] = r.x; o[1] = r.y; o[2] = r.z;
    } else {
        const float* x = static_cast<const float*>(v);
        const mv::T3<float> r = mv::project_velocity(mv::T3<float>{x[0], x[1], x[2]}, ns.data(), int(n));
        float* o = static_cast<float*>(out);
        o[0] = r.x; o[1] = r.y; o[2] = r.z;
    }
}

// test infrastructure: one intersection of the move (character a against collider b, double columns): the deepest penetration rounded to
// the column scalar and the f32 plane normal -manifold.normal; 0 when the pair has no point within `prediction`
int avh_move_contact(uint32_t scalar_bits, int sa, const double* ha, const double* pa, const double* qa, int sb, const double* hb, const double* pb,
                     const double* qb, double prediction, float* normal, double* penetration) {
    const V3 A{ha[0], ha[1], ha[2]}, PA{pa[0], pa[1], pa[2]}, B{hb[0], hb[1], hb[2]}, PB{pb[0], pb[1], pb[2]};
    const Q QA{qa[0], qa[1], qa[2], qa[3]}, QB{qb[0], qb[1], qb[2], qb[3]};
    mv::T3<float> n{0, 0, 0};
    bool hit;
    if (scalar_bits == 64) {
        double pen = 0;
        hit = mv::contact_plane<double, true>(sa, A, PA, QA, sb, B, PB, QB, prediction, n, pen);
        *penetration = pen;
    } else {
        float pen = 0;
        hit = mv::contact_plane<float, true>(sa, A, PA, QA, sb, B, PB, QB, prediction, n, pen);
        *penetration = pen;
    }
    normal[0] = n.x; normal[1] = n.y; normal[2] = n.z;
    return hit ? 1 : 0;
}
// the same through the hull instance's contact planes (mv::contact_plane_hulls) with the fixture's hull table
int avh_move_contact_hulls(uint32_t scalar_bits, int sa, const double* ha, const double* pa, const double* qa, int sb, const double* hb, const double* pb,
                           const double* qb, double prediction, float* normal, double* penetration, const void* hull_table) {
    if (!hull_table) return 0;   // no table: no contact plane, as the other *_hulls variants refuse
    const hm::Table t = hm::view(*static_cast<const hm::HullSet*>(hull_table));
    const V3 A{ha[0], ha[1], ha[2]}, PA{pa[0], pa[1], pa[2]}, B{hb[0], hb[1], hb[2]}, PB{pb[0], pb[1], pb[2]};
    const Q QA{qa[0], qa[1], qa[2], qa[3]}, QB{qb[0], qb[1], qb[2], qb[3]};
    mv::T3<float> n{0, 0, 0};
    bool hit;
    if (scalar_bits == 64) {
        double pen = 0;
        hit = mv::contact_plane_hulls<double>(t, sa, A, PA, QA, sb, B, PB, QB, prediction, n, pen);
        *penetration = pen;
    } else {
        float pen = 0;
        hit = mv::contact_plane_hulls<float>(t, sa, A, PA, QA, sb, B, PB, QB, prediction, n, pen);
        *penetration = pen;
    }
    normal[0] = n.x; normal[1] = n.y; normal[2] = n.z;
    return hit ? 1 : 0;
}

}  // extern "C"

// ---- swept CCD: solve_swept_ccd (dynamics/ccd/mod.rs:523-687) as the reference's sequential loop over the configured bodies, each scanning the
//      live rows that hold its collider in ascending ContactId with the strict `<` — the checker of csrc/ccd.cu -------------------------------
namespace {

template <class T>
ccd::Motion ccd_motion(const T* shape_dims, const uint8_t* shape, uint32_t c, const T* pos, const T* rot, const T* com, ccd::V3T<T> v, ccd::V3T<T> w, uint32_t b) {
    ccd::Motion m;
    m.shape = shape ? shape[c] : SHAPE_CUBOID;
    m.he = V3{S(shape_dims[3 * c]), S(shape_dims[3 * c + 1]), S(shape_dims[3 * c + 2])};
    m.p = V3{S(pos[3 * b]), S(pos[3 * b + 1]), S(pos[3 * b + 2])};
    m.q = Q{S(rot[4 * b]), S(rot[4 * b + 1]), S(rot[4 * b + 2]), S(rot[4 * b + 3])};
    m.lc = com ? V3{S(com[3 * b]), S(com[3 * b + 1]), S(com[3 * b + 2])} : V3{0, 0, 0};
    m.v = V3{S(v.x), S(v.y), S(v.z)};
    m.w = V3{S(w.x), S(w.y), S(w.z)};
    return m;
}

template <class T>
int ccd_solve(double dt_d, double length_unit, uint32_t B, const uint8_t* kind, const T* pos, const T* rot, const T* com, const T* lv, const T* av, T* dpos,
              T* drot, const uint8_t* shape, const T* dims, uint32_t rows, const uint32_t* c1, const uint32_t* c2, const uint32_t* b1, const uint32_t* b2,
              const uint8_t* live, const AvnCcdConfig* cfg, T* out_min, int32_t* out_body, int32_t* out_contact, uint32_t* out_cand, uint32_t* out_hits,
              const hm::Table* ht) {
    const T dt = T(dt_d);
    const S eps = ccd::CCD_EPS_PER_LENGTH_UNIT * length_unit;
    auto kind_of = [&](uint32_t b) { return kind ? kind[b] : uint8_t(AVN_BODY_DYNAMIC); };
    auto has_sb = [&](uint32_t b) { return b < B && kind_of(b) != AVN_BODY_STATIC; };
    auto vel = [&](uint32_t b, const T* col) { return has_sb(b) ? ccd::V3T<T>{col[3 * b], col[3 * b + 1], col[3 * b + 2]} : ccd::V3T<T>{T(0), T(0), T(0)}; };
    std::unordered_map<uint32_t, size_t> slot_of_body;
    for (size_t k = 0; k < cfg->count; ++k) slot_of_body[uint32_t(cfg->body[k])] = k;
    auto mode_of = [&](size_t k) { return cfg->mode ? int(cfg->mode[k]) : ccd::MODE_NON_LINEAR; };
    // each CCD collider's rows in ascending ContactId (the visiting order whose first minimum the strict `<` keeps)
    std::unordered_map<uint32_t, std::vector<uint32_t>> adjacency;
    for (size_t k = 0; k < cfg->count; ++k) adjacency[cfg->collider[k]];
    for (uint32_t e = 0; e < rows; ++e) {
        if (!live[e]) continue;
        auto a = adjacency.find(c1[e]);
        if (a != adjacency.end()) a->second.push_back(e);
        if (c2[e] != c1[e] && (a = adjacency.find(c2[e])) != adjacency.end()) a->second.push_back(e);
    }
    for (size_t k = 0; k < cfg->count; ++k) {
        const uint32_t body1 = uint32_t(cfg->body[k]), own = cfg->collider[k];
        T min_toi = dt;
        int32_t hit = -1, hit_row = -1;
        uint32_t cand = 0, hits = 0;
        if (has_sb(body1)) {
            const T lthr = T(cfg->linear_threshold ? cfg->linear_threshold[k] : 0.0), athr = T(cfg->angular_threshold ? cfg->angular_threshold[k] : 0.0);
            const bool include_dynamic = cfg->include_dynamic ? cfg->include_dynamic[k] != 0 : true;
            for (const uint32_t e : adjacency[own]) {
                const bool first = c1[e] == own;
                const uint32_t other = first ? c2[e] : c1[e], body2 = first ? b2[e] : b1[e];
                if (body2 >= B || body2 == body1) continue;
                if (!include_dynamic && kind_of(body2) == AVN_BODY_DYNAMIC) continue;
                const ccd::V3T<T> v1 = vel(body1, lv), w1 = vel(body1, av), v2 = vel(body2, lv), w2 = vel(body2, av);
                if (ccd::below_thresholds<T>(v1, w1, v2, w2, lthr, athr)) continue;
                const auto it = slot_of_body.find(body2);
                const int mode = (mode_of(k) == ccd::MODE_LINEAR && (it == slot_of_body.end() || mode_of(it->second) == ccd::MODE_LINEAR)) ? ccd::MODE_LINEAR
                                                                                                                                      : ccd::MODE_NON_LINEAR;
                ++cand;
                const ccd::Motion A = ccd_motion(dims, shape, own, pos, rot, com, v1, w1, body1), Bm = ccd_motion(dims, shape, other, pos, rot, com, v2, w2, body2);
                const T t = ht ? ccd::pair_toi<T, 2>(mode, A, Bm, dt, eps, cfg->prediction_distance, ht) : ccd::pair_toi<T, 1>(mode, A, Bm, dt, eps, cfg->prediction_distance);
                if (t > T(0) && t < dt) ++hits;
                if (t > T(0) && t < min_toi) { min_toi = t; hit = int32_t(body2); hit_row = int32_t(e); }
            }
        }
        if (out_min) out_min[k] = min_toi;
        if (out_body) out_body[k] = hit;
        if (out_contact) out_contact[k] = hit_row;
        if (out_cand) out_cand[k] = cand;
        if (out_hits) out_hits[k] = hits;
        if (hit < 0 || !dpos || !drot) continue;
        // application, in list order (ccd/mod.rs:620-670)
        const T m = ccd::overshoot(min_toi);
        for (int side = 0; side < 2; ++side) {
            const uint32_t b = side == 0 ? body1 : uint32_t(hit);
            if (!has_sb(b)) continue;   // the dummy SolverBody: writes are discarded
            ccd::V3T<T> dp{dpos[3 * b], dpos[3 * b + 1], dpos[3 * b + 2]};
            ccd::QT<T> dq{drot[4 * b], drot[4 * b + 1], drot[4 * b + 2], drot[4 * b + 3]};
            ccd::apply_record(m, vel(b, lv), vel(b, av), dp, dq);
            dpos[3 * b] = dp.x; dpos[3 * b + 1] = dp.y; dpos[3 * b + 2] = dp.z;
            drot[4 * b] = dq.x; drot[4 * b + 1] = dq.y; drot[4 * b + 2] = dq.z; drot[4 * b + 3] = dq.w;
        }
    }
    return 0;
}

ccd::Motion motion_from(const double* m) {   // shape, he[3], p[3], q[4], local com[3], v[3], w[3]
    ccd::Motion r;
    r.shape = int(m[0]);
    r.he = V3{m[1], m[2], m[3]}; r.p = V3{m[4], m[5], m[6]}; r.q = Q{m[7], m[8], m[9], m[10]}; r.lc = V3{m[11], m[12], m[13]};
    r.v = V3{m[14], m[15], m[16]}; r.w = V3{m[17], m[18], m[19]};
    return r;
}

// avh_ccd_solve(_hulls): the refusals, then the loop (G = 2 with the table under AVN_CCD_HULLS, else G = 1)
int ccd_solve_any(uint32_t scalar_bits, double dt, double length_unit, uint32_t body_count, const uint8_t* kind, const void* position, const void* rotation,
                  const void* com, const void* linvel, const void* angvel, void* delta_position, void* delta_rotation, const uint8_t* shape, const void* dims,
                  uint32_t rows, const uint32_t* c1, const uint32_t* c2, const uint32_t* b1, const uint32_t* b2, const uint8_t* live, const AvnCcdConfig* cfg,
                  void* min_toi, int32_t* hit_body, int32_t* hit_contact, uint32_t* candidates, uint32_t* hits, const hm::HullSet* hulls) {
    if (!cfg || (cfg->count && (!cfg->body || !cfg->collider))) return -1;
    if (cfg->count && (cfg->flags & ~(AVN_CCD_CAPSULES | AVN_CCD_HULLS))) return AVN_ERR_INVALID_ARGUMENT;
    // without AVN_CCD_CAPSULES a configuration with a row that names a capsule is refused, as the device refuses it
    if (cfg->count && shape && !(cfg->flags & AVN_CCD_CAPSULES))
        for (uint32_t r = 0; r < rows; ++r)
            if ((!live || live[r]) && (shape[c1[r]] == SHAPE_CAPSULE || shape[c2[r]] == SHAPE_CAPSULE)) return AVN_ERR_UNSUPPORTED;
    // the same for convex hulls without AVN_CCD_HULLS; with it, a row naming a hull the table does not hold (or no table) is refused, as the
    // contact step refuses the column
    const bool sweep_hulls = (cfg->flags & AVN_CCD_HULLS) != 0;
    if (cfg->count && shape)
        for (uint32_t r = 0; r < rows; ++r) {
            if (live && !live[r]) continue;
            for (const uint32_t c : {c1[r], c2[r]}) {
                if (shape[c] != hm::SHAPE_CONVEX_HULL) continue;
                if (!sweep_hulls) return AVN_ERR_UNSUPPORTED;
                const double h = scalar_bits == 64 ? static_cast<const double*>(dims)[3 * size_t(c)] : double(static_cast<const float*>(dims)[3 * size_t(c)]);
                if (!hulls || !(h >= 0 && h < double(hull_count(hulls))) || h != double(uint32_t(h))) return AVN_ERR_INVALID_ARGUMENT;
            }
        }
    hm::Table t{};
    if (hulls) t = hm::view(*hulls);
    const hm::Table* ht = sweep_hulls && hulls ? &t : nullptr;
    if (scalar_bits == 64)
        return ccd_solve<double>(dt, length_unit, body_count, kind, static_cast<const double*>(position), static_cast<const double*>(rotation),
                                 static_cast<const double*>(com), static_cast<const double*>(linvel), static_cast<const double*>(angvel),
                                 static_cast<double*>(delta_position), static_cast<double*>(delta_rotation), shape, static_cast<const double*>(dims), rows, c1, c2,
                                 b1, b2, live, cfg, static_cast<double*>(min_toi), hit_body, hit_contact, candidates, hits, ht);
    return ccd_solve<float>(dt, length_unit, body_count, kind, static_cast<const float*>(position), static_cast<const float*>(rotation),
                            static_cast<const float*>(com), static_cast<const float*>(linvel), static_cast<const float*>(angvel),
                            static_cast<float*>(delta_position), static_cast<float*>(delta_rotation), shape, static_cast<const float*>(dims), rows, c1, c2, b1,
                            b2, live, cfg, static_cast<float*>(min_toi), hit_body, hit_contact, candidates, hits, ht);
}

}  // namespace

extern "C" {

// solve_swept_ccd over the given contact rows.  Velocities: the SolverBody velocities after the substeps; delta_position / delta_rotation
// ([B][3] / [B][4], in/out, may be NULL): the substeps' deltas, onto which the pass writes.  Returns -1 for an invalid configuration,
// AVN_ERR_INVALID_ARGUMENT for an unknown cfg->flags bit, and AVN_ERR_UNSUPPORTED for a live row that names a capsule without
// AVN_CCD_CAPSULES or a convex hull without AVN_CCD_HULLS.  The geometry is the G = 1 instance: with no capsule in a pair it is the device's
// G = 0 TOI, bit for bit.
int avh_ccd_solve(uint32_t scalar_bits, double dt, double length_unit, uint32_t body_count, const uint8_t* kind, const void* position, const void* rotation,
                  const void* com, const void* linvel, const void* angvel, void* delta_position, void* delta_rotation, const uint8_t* shape, const void* dims,
                  uint32_t rows, const uint32_t* c1, const uint32_t* c2, const uint32_t* b1, const uint32_t* b2, const uint8_t* live, const AvnCcdConfig* cfg,
                  void* min_toi, int32_t* hit_body, int32_t* hit_contact, uint32_t* candidates, uint32_t* hits) {
    return ccd_solve_any(scalar_bits, dt, length_unit, body_count, kind, position, rotation, com, linvel, angvel, delta_position, delta_rotation, shape, dims,
                         rows, c1, c2, b1, b2, live, cfg, min_toi, hit_body, hit_contact, candidates, hits, nullptr);
}
// The same with the fixture's hull table (avh_hulls_create, may be NULL).  Under AVN_CCD_HULLS with a table the geometry is the G = 2
// instance, which gives the G = 1 bits on pairs without a hull; a live row naming a hull the table does not hold is AVN_ERR_INVALID_ARGUMENT.
int avh_ccd_solve_hulls(uint32_t scalar_bits, double dt, double length_unit, uint32_t body_count, const uint8_t* kind, const void* position,
                        const void* rotation, const void* com, const void* linvel, const void* angvel, void* delta_position, void* delta_rotation,
                        const uint8_t* shape, const void* dims, uint32_t rows, const uint32_t* c1, const uint32_t* c2, const uint32_t* b1, const uint32_t* b2,
                        const uint8_t* live, const AvnCcdConfig* cfg, void* min_toi, int32_t* hit_body, int32_t* hit_contact, uint32_t* candidates,
                        uint32_t* hits, const void* hull_table) {
    return ccd_solve_any(scalar_bits, dt, length_unit, body_count, kind, position, rotation, com, linvel, angvel, delta_position, delta_rotation, shape, dims,
                         rows, c1, c2, b1, b2, live, cfg, min_toi, hit_body, hit_contact, candidates, hits, static_cast<const hm::HullSet*>(hull_table));
}

// One pair's compute_ccd_toi against the bound dt (ccd::pair_toi, fallback included), rounded to the column scalar and returned as a double;
// -1 = no hit.  Motions: 20 doubles each (shape, half extents / radius / capsule radius and half length, position, rotation, local com,
// linear and angular velocity).  Capsules (shape 2) are accepted.
double avh_ccd_pair_toi(uint32_t scalar_bits, int mode, const double* a, const double* b, double dt, double eps, double prediction_distance) {
    if (scalar_bits == 64) return ccd::pair_toi<double, 1>(mode, motion_from(a), motion_from(b), dt, eps, prediction_distance);
    return double(ccd::pair_toi<float, 1>(mode, motion_from(a), motion_from(b), float(dt), eps, prediction_distance));
}
// The same at G = 2 with the fixture's hull table (convex hulls, shape 3, dims[0] = the hull index); NULL table: avh_ccd_pair_toi
double avh_ccd_pair_toi_hulls(uint32_t scalar_bits, int mode, const double* a, const double* b, double dt, double eps, double prediction_distance,
                              const void* hull_table) {
    if (!hull_table) return avh_ccd_pair_toi(scalar_bits, mode, a, b, dt, eps, prediction_distance);
    const hm::Table t = hm::view(*static_cast<const hm::HullSet*>(hull_table));
    if (scalar_bits == 64) return ccd::pair_toi<double, 2>(mode, motion_from(a), motion_from(b), dt, eps, prediction_distance, &t);
    return double(ccd::pair_toi<float, 2>(mode, motion_from(a), motion_from(b), float(dt), eps, prediction_distance, &t));
}

// The raw non-linear TOI in double (no rounding, no fallback): 1 and *toi on a hit, 0 otherwise; *iterations = distance evaluations.
int avh_ccd_nonlinear_toi(const double* a, const double* b, double t_max, double eps, double* toi, int* iterations) {
    double t = 0;
    const bool hit = ccd::nonlinear_toi<1>(motion_from(a), motion_from(b), t_max, eps, t, iterations);
    *toi = t;
    return hit ? 1 : 0;
}
// The same at G = 2 with the fixture's hull table; NULL table: avh_ccd_nonlinear_toi
int avh_ccd_nonlinear_toi_hulls(const double* a, const double* b, double t_max, double eps, double* toi, int* iterations, const void* hull_table) {
    if (!hull_table) return avh_ccd_nonlinear_toi(a, b, t_max, eps, toi, iterations);
    const hm::Table t = hm::view(*static_cast<const hm::HullSet*>(hull_table));
    double tt = 0;
    const bool hit = ccd::nonlinear_toi<2>(motion_from(a), motion_from(b), t_max, eps, tt, iterations, &t);
    *toi = tt;
    return hit ? 1 : 0;
}
// test infrastructure: ccd::motion_radius of one motion (G = 2 with the table, G = 1 without)
double avh_ccd_motion_radius(const double* m, const void* hull_table) {
    if (!hull_table) return ccd::motion_radius<1>(motion_from(m));
    const hm::Table t = hm::view(*static_cast<const hm::HullSet*>(hull_table));
    return ccd::motion_radius<2>(motion_from(m), &t);
}

// Quat::from_scaled_axis and the delta write of one record, in the column scalar (tests)
void avh_ccd_apply_record(uint32_t scalar_bits, double m, const double* v, const double* w, double* dp, double* dq) {
    if (scalar_bits == 64) {
        ccd::V3T<double> p{dp[0], dp[1], dp[2]};
        ccd::QT<double> q{dq[0], dq[1], dq[2], dq[3]};
        ccd::apply_record<double>(m, {v[0], v[1], v[2]}, {w[0], w[1], w[2]}, p, q);
        dp[0] = p.x; dp[1] = p.y; dp[2] = p.z; dq[0] = q.x; dq[1] = q.y; dq[2] = q.z; dq[3] = q.w;
        return;
    }
    ccd::V3T<float> p{float(dp[0]), float(dp[1]), float(dp[2])};
    ccd::QT<float> q{float(dq[0]), float(dq[1]), float(dq[2]), float(dq[3])};
    ccd::apply_record<float>(float(m), {float(v[0]), float(v[1]), float(v[2])}, {float(w[0]), float(w[1]), float(w[2])}, p, q);
    dp[0] = p.x; dp[1] = p.y; dp[2] = p.z; dq[0] = q.x; dq[1] = q.y; dq[2] = q.z; dq[3] = q.w;
}

}  // extern "C"
