// MoveAndSlide (character_controller/move_and_slide.rs, velocity_project.rs) for cuboid / sphere / capsule characters, written once for the host
// fixture (g++, -ffp-contract=off) and for the device (nvcc, -fmad=false), the query_math.hpp / ccd_math.hpp arrangement: the per-character
// algorithm is a template over a "scene" that answers two questions, and both builds evaluate the same expressions in the same order.
//   * sc.cast(shape, he, c, q, d, maxd, t, collider, axis): the closest filtered shape cast (AVN_CAST_IGNORE_ORIGIN_PENETRATION), the
//     lexicographic minimum of (t, collider index).  Host: every collider.  Device: the collider tree (csrc/queries.cu).
//   * sc.candidates(lo, hi, fn): fn(collider) for every filtered collider whose tight AABB (rounded to the column scalar) meets [lo, hi], in
//     ascending collider index.  Host: a loop over every collider.  Device: tree walks that each collect the K = MOVE_WINDOW smallest
//     indices above the last one handled.
//   * sc.collider(c, shape, he, p, q): the collider's columns.
// The filter is the character's: (memberships & mask) != 0, not in its exclusion list, and not marked in the config's `ignored` column
// (sensors, colliders without a body: the reference's `colliders` query is With<ColliderOf>, Without<Sensor>).
//
// Precision (the reference's, kept): the loop runs in the column scalar T (Scalar); `Dir` is f32 in both builds, so the sweep direction
// (Dir::new_and_length(sweep.f32())), every plane normal and the plane-similarity dot product are f32, widened to T where the reference
// calls adjust_precision().  The shape cast and the contact geometry are query_math.hpp / narrow_math.hpp in double, rounded to T on use.
//
// Stated deviations (include/avian_b200.h, DESIGN.md §7g):
//   * on_hit cannot run on the device: every hit is accepted and nothing edits the normal, position or velocity.
//   * the closest sweep hit is the lowest (t, collider index), not the first hit in tree order (the cast_shape rule).
//   * intersections are visited in ascending collider index, not tree order (plane pruning and Gauss-Seidel depend on the order).
//   * the reported hit distance is the TOI; the reference's MoveHitData::collision_distance is the requested movement length (:777).
// Capsules and hulls (DESIGN.md §7j, §7l): the loop is a template over the shape level G.  G = 1 compiles the capsule casts of query_math.hpp
// and the capsule pairs of nm::collide into the sweep and the intersections; G = 0 is the cuboid / sphere loop as it was before capsule
// characters.  G = 2 adds convex hulls: the casts of hull_query_math.hpp and hm::collide for the pairs with a hull, with the scene's hull
// table (sc.hulls()).  queries.cu picks the instance on the host; the host fixture runs G = 2, which gives the G = 1 bits on cuboids, spheres
// and capsules.
#pragma once
#include <cmath>
#include <cstdint>

#include "hull_query_math.hpp"
#include "narrow_math.hpp"
#include "query_math.hpp"

namespace mv {

using nm::Q;
using nm::V3;

constexpr int MAX_PLANES = 32;      // = AVN_MOVE_MAX_PLANES; the plane buffer holds MAX_PLANES + 1 (the sweep hit's plane is pushed unchecked)
constexpr int MOVE_WINDOW = 16;     // K: candidates per tree walk, and the depenetration list kept in local memory
constexpr double DOT_EPSILON = 0.005;
constexpr double MIN_DISTANCE = 1e-4;

template <class T> struct T3 { T x, y, z; };
template <class T> NM_HD inline T3<T> add(T3<T> a, T3<T> b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
template <class T> NM_HD inline T3<T> sub(T3<T> a, T3<T> b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
template <class T> NM_HD inline T3<T> neg(T3<T> a) { return {-a.x, -a.y, -a.z}; }
template <class T> NM_HD inline T3<T> scale(T s, T3<T> a) { return {s * a.x, s * a.y, s * a.z}; }   // glam's scalar * vector
template <class T> NM_HD inline T3<T> divs(T3<T> a, T s) { return {a.x / s, a.y / s, a.z / s}; }
template <class T> NM_HD inline T dot(T3<T> a, T3<T> b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <class T> NM_HD inline T3<T> cross(T3<T> a, T3<T> b) { return {a.y * b.z - b.y * a.z, a.z * b.x - b.z * a.x, a.x * b.y - b.x * a.y}; }
template <class T> NM_HD inline T3<T> wide(T3<float> a) { return {T(a.x), T(a.y), T(a.z)}; }   // adjust_precision()
template <class T> NM_HD inline T3<float> narrow(T3<T> a) { return {float(a.x), float(a.y), float(a.z)}; }   // .f32()
template <class T> NM_HD inline V3 to_v3(T3<T> a) { return V3{double(a.x), double(a.y), double(a.z)}; }
template <class T> NM_HD inline T3<T> from_v3(V3 a) { return {T(a.x), T(a.y), T(a.z)}; }
template <class T> NM_HD inline T smax0(T a) { return a < T(0) ? T(0) : a; }   // Scalar::max(x, 0.0) for a non-NaN x
// Scalar::total_cmp(a, b) == Less for non-NaN values: -0 sorts below +0
template <class T> NM_HD inline bool total_lt(T a, T b) { return a < b || (a == b && std::signbit(a) && !std::signbit(b)); }

template <class T>
struct Config {                      // MoveAndSlideConfig / DepenetrationConfig, in the column scalar
    T dt, length_unit, skin_width, max_depenetration_error, penetration_rejection_threshold, plane_similarity_dot_threshold;
    uint32_t iterations, depenetration_iterations, max_planes;
};

// ---- project_velocity (velocity_project.rs:122-324): the GJK-like projection of v onto the cone of the planes' halfspaces -------------
template <class T>
NM_HD inline T3<T> project_velocity(T3<T> v, const T3<float>* normals, int n) {
    const T eps = T(DOT_EPSILON);
    const T3<T> x0 = neg(v);
    int kind = 0;                    // 0 = origin, 1 = Ray(n1), 2 = Wedge(n1, n2)
    T3<float> n1{0, 0, 0}, n2{0, 0, 0};
    T3<T> sv = x0;
    int iters = 0;
    for (;;) {
        if (dot(sv, sv) < eps * eps) break;
        if (n == 0) break;
        int bi = 0;
        T best = dot(wide<T>(normals[0]), sv);
        for (int k = 1; k < n; ++k) {                    // max_by keeps the last of equal maxima
            const T d = dot(wide<T>(normals[k]), sv);
            if (!total_lt(d, best)) { best = d; bi = k; }
        }
        if (best <= eps) break;
        const T3<float> nd = normals[bi];
        const T3<T> ndv = wide<T>(nd);
        if (kind == 0) {
            const T d = dot(ndv, x0);
            sv = sub(x0, scale(d, ndv));
            n1 = nd;
            kind = 1;
        } else if (kind == 1) {
            const T3<T> c = cross(ndv, wide<T>(n1));
            const T d = dot(x0, c);
            sv = divs(scale(d, c), dot(c, c));
            if (d > T(0)) { n2 = n1; n1 = nd; } else { n2 = nd; }
            kind = 2;
        } else {
            const T3<T> c1 = cross(wide<T>(n1), ndv);
            const T c1sq = dot(c1, c1), d1 = dot(x0, c1);
            const T3<T> c2 = cross(ndv, wide<T>(n2));
            const T c2sq = dot(c2, c2), d2 = dot(x0, c2);
            if (d1 <= T(0) && d2 <= T(0)) { sv = T3<T>{0, 0, 0}; break; }   // inside the solid wedge
            if (d1 * std::fabs(d1) * c2sq > d2 * std::fabs(d2) * c1sq) {
                sv = divs(scale(d1, c1), c1sq);
                n2 = nd;
            } else {
                sv = divs(scale(d2, c2), c2sq);
                n1 = nd;
            }
        }
        if (++iters >= 10) break;
    }
    return neg(sv);
}

// ---- one intersection (intersections, move_and_slide.rs:1032-1078): the contact of the character with one collider -----------------------
// nm::collide(character, collider) -> the deepest point (max_by: the last of equal penetrations) and the plane normal -manifold.normal as
// an f32 Dir.  False when the pair has no point within the prediction distance.  Kept out of line: it holds the narrow phase's box-box
// generator, and the move kernel calls it from two places.  CAPS = false leaves the capsule pairs out (nm::collide<false>): that instance
// never sees a capsule.
template <class T, bool CAPS = false>
NM_COLD inline bool contact_plane(int sa, V3 ha, V3 pa, Q qa, int sb, V3 hb, V3 pb, Q qb, double prediction, T3<float>& normal, T& penetration) {
    V3 n;
    nm::Contacts pts;
    if (!nm::collide<CAPS>(sa, ha, pa, qa, sb, hb, pb, qb, prediction, n, pts) || pts.n == 0) return false;
    T best = T(nm::dot(pts.p[0].a - pts.p[0].b, n));
    for (int k = 1; k < pts.n; ++k) {
        const T p = T(nm::dot(pts.p[k].a - pts.p[k].b, n));
        if (!(p < best)) best = p;
    }
    penetration = best;
    normal = T3<float>{float(-n.x), float(-n.y), float(-n.z)};
    return true;
}
// the same for the hull instance: a pair with a convex hull goes through hm::collide (either order), every other pair through
// nm::collide<true>
template <class T>
NM_COLD inline bool contact_plane_hulls(const hm::Table& ht, int sa, V3 ha, V3 pa, Q qa, int sb, V3 hb, V3 pb, Q qb, double prediction, T3<float>& normal,
                                        T& penetration) {
    V3 n;
    nm::Contacts pts;
    const bool hit = sa == hm::SHAPE_CONVEX_HULL || sb == hm::SHAPE_CONVEX_HULL ? hm::collide(ht, sa, ha, pa, qa, sb, hb, pb, qb, prediction, n, pts)
                                                                                 : nm::collide<true>(sa, ha, pa, qa, sb, hb, pb, qb, prediction, n, pts);
    if (!hit || pts.n == 0) return false;
    T best = T(nm::dot(pts.p[0].a - pts.p[0].b, n));
    for (int k = 1; k < pts.n; ++k) {
        const T p = T(nm::dot(pts.p[k].a - pts.p[k].b, n));
        if (!(p < best)) best = p;
    }
    penetration = best;
    normal = T3<float>{float(-n.x), float(-n.y), float(-n.z)};
    return true;
}

// a configured plane as a Dir (Dir::new on its f32 value); the ABI refuses zero and non-finite planes
template <class T> NM_HD inline T3<float> plane_dir(T3<T> p) { const T3<float> f = narrow(p); return divs(f, std::sqrt(dot(f, f))); }

// the character: shape, dims, rotation (double), fixed for the whole move
struct Body { int shape; V3 he; Q q; };

// the character's tight AABB at pos, rounded to T, grown by `grow` (Aabb::grow)
template <int G, class T, class Scene>
NM_HD inline void grown_aabb(const Scene& sc, const Body& b, T3<T> pos, T grow, T lo[3], T hi[3]) {
    V3 mn, mx;
    if constexpr (G == 2) qh::collider_aabb(sc.hulls(), b.shape, b.he, to_v3(pos), b.q, mn, mx);
    else qm::collider_aabb<G == 1>(b.shape, b.he, to_v3(pos), b.q, mn, mx);
    lo[0] = T(mn.x) - grow; lo[1] = T(mn.y) - grow; lo[2] = T(mn.z) - grow;
    hi[0] = T(mx.x) + grow; hi[1] = T(mx.y) + grow; hi[2] = T(mx.z) + grow;
}

// every intersection plane at pos with prediction distance `pred`, in ascending collider index: fn(normal, penetration)
template <class T, int G, class Scene, class Fn>
NM_HD inline void intersections(const Scene& sc, const Body& b, T3<T> pos, T pred, Fn fn) {
    T lo[3], hi[3];
    grown_aabb<G>(sc, b, pos, pred, lo, hi);
    const V3 p = to_v3(pos);
    sc.candidates(lo, hi, [&](uint32_t c) {
        int s;
        V3 he, cp;
        Q cq;
        sc.collider(c, s, he, cp, cq);
        T3<float> n;
        T pen;
        bool hit;
        if constexpr (G == 2) hit = contact_plane_hulls<T>(sc.hulls(), b.shape, b.he, p, b.q, s, he, cp, cq, double(pred), n, pen);
        else hit = contact_plane<T, G == 1>(b.shape, b.he, p, b.q, s, he, cp, cq, double(pred), n, pen);
        if (hit) fn(n, pen);
    });
}

// depenetrate + depenetrate_intersections (:868-897, :982-1009): Gauss-Seidel over the (normal, penetration + skin) list.  The list is
// kept when it has at most MOVE_WINDOW entries; a longer one is evaluated again, in the same order, in every iteration.
template <int G, class T, class Scene>
NM_HD inline T3<T> depenetrate(const Scene& sc, const Config<T>& cfg, const Body& b, T3<T> pos) {
    T3<T> fixup{0, 0, 0};
    if (cfg.depenetration_iterations == 0) return fixup;
    const T skin = cfg.length_unit * cfg.skin_width;
    const T reject = cfg.length_unit * cfg.penetration_rejection_threshold;
    const T target = cfg.length_unit * cfg.max_depenetration_error;
    T3<float> ln[MOVE_WINDOW];
    T ld[MOVE_WINDOW];
    uint32_t count = 0;
    intersections<T, G>(sc, b, pos, skin, [&](T3<float> n, T pen) {
        if (count < uint32_t(MOVE_WINDOW)) { ln[count] = n; ld[count] = pen + skin; }
        ++count;
    });
    const bool kept = count <= uint32_t(MOVE_WINDOW);
    T total = T(0);
    auto relax = [&](T3<float> n, T dist) {
        if (dist > reject) return;
        const T3<T> nv = wide<T>(n);
        const T err = smax0(dist - dot(fixup, nv));
        total += err;
        fixup = add(fixup, scale(err, nv));
    };
NM_ROLLED
    for (uint32_t it = 0; it < cfg.depenetration_iterations; ++it) {
        total = T(0);
        if (kept) {
            for (uint32_t k = 0; k < count; ++k) relax(ln[k], ld[k]);
        } else {
            intersections<T, G>(sc, b, pos, skin, [&](T3<float> n, T pen) { relax(n, pen + skin); });
        }
        if (total < target) break;
    }
    return fixup;
}

// MoveAndSlide::move_and_slide (:464-609) with an on_hit that accepts every hit.  pos / vel: in, out.  init: the configured planes
// (MoveAndSlideConfig::planes) as f32 Dirs, n_init <= max_planes.  hits.sweep(iteration, collider, safe distance, toi, point1, normal1) is
// called for every iteration that hit something.
template <int G = 0, class T, class Scene, class Hits>
NM_HD inline void move_and_slide(const Scene& sc, const Config<T>& cfg, const Body& b, T3<T>& pos, T3<T>& vel, const T3<float>* init, int n_init,
                                 Hits& hits) {
    T time_left = cfg.dt;
    const T skin = cfg.length_unit * cfg.skin_width;
    pos = add(pos, depenetrate<G>(sc, cfg, b, pos));
    T3<float> planes[MAX_PLANES + 1];
NM_ROLLED
    for (uint32_t it = 0; it < cfg.iterations; ++it) {
        const T3<T> sweep = scale(time_left, vel);
        // Dir::new_and_length(sweep.f32())
        const T3<float> sf = narrow(sweep);
        const float lf = std::sqrt(dot(sf, sf));
        if (!(std::isfinite(lf) && lf > 0.0f)) break;
        const T3<float> dir = divs(sf, lf);
        const T distance = T(lf);
        if (distance < T(MIN_DISTANCE)) break;
        // cast_move (:745-784): the closest hit of the cast along dir up to distance, ignoring origin penetration moving away
        double toi;
        uint32_t c;
        int axis;
        const V3 p = to_v3(pos), d = to_v3(dir);
        if (!sc.cast(b.shape, b.he, p, b.q, d, double(distance), toi, c, axis)) {
            pos = add(pos, sweep);
            break;
        }
        int cs;
        V3 che, cp;
        Q cq;
        sc.collider(c, cs, che, cp, cq);
        qm::ShapeContact hc;
        if constexpr (G == 2) qh::cast_output(sc.hulls(), b.shape, b.he, p, b.q, d, qm::CAST_IGNORE_ORIGIN_PENETRATION, cs, che, cp, cq, toi, axis, hc);
        else qm::cast_output<G == 1>(b.shape, b.he, p, b.q, d, qm::CAST_IGNORE_ORIGIN_PENETRATION, cs, che, cp, cq, toi, axis, hc);
        const T3<T> normal1 = from_v3<T>(hc.n1);
        const T hit_distance = T(toi);
        // pull_back (:789-793)
        const T pd = dot(wide<T>(dir), neg(normal1));
        const T safe = smax0(hit_distance - skin / (pd < T(DOT_EPSILON) ? T(DOT_EPSILON) : pd));
        hits.sweep(it, c, safe, hit_distance, from_v3<T>(hc.p1), normal1);
        time_left -= time_left * (safe / distance);
        pos = add(pos, scale(safe, wide<T>(dir)));
        // planes: the configured ones, the sweep hit's (pushed without the max_planes check), then the contacts at 2 * skin
        int np = 0;
        for (int k = 0; k < n_init; ++k) planes[np++] = init[k];
        planes[np++] = narrow(normal1);
        const T3<T> v = vel;
        intersections<T, G>(sc, b, pos, skin * T(2), [&](T3<float> n, T) {
            for (int k = 0; k < np; ++k) {
                if (T(dot(n, planes[k])) >= cfg.plane_similarity_dot_threshold) {
                    // similar: keep the more blocking normal
                    if (dot(wide<T>(n), v) < dot(wide<T>(planes[k]), v)) planes[k] = n;
                    return;
                }
            }
            if (uint32_t(np) >= cfg.max_planes) return;     // the reference's callback result is ignored: later contacts are still tested
            planes[np++] = n;
        });
        vel = project_velocity(vel, planes, np);
    }
    pos = add(pos, depenetrate<G>(sc, cfg, b, pos));
}

}  // namespace mv

// ---- host-side validation shared by the ABI (before any upload) and the host fixture --------------------------------------------------
#include "../../include/avian_b200.h"
namespace mv {
// NULL when the call is usable; the reason otherwise.  collider_count: the colliders of the scene (the tree's, the host's)
// capsules: whether AVN_SHAPE_CAPSULE characters are accepted; saw_capsule (optional): set when the batch holds one.  hull_count / saw_hull:
// hull characters, as qm::check_colliders takes hull colliders
inline const char* check_move(const AvnMoveConfig* cfg, const AvnMoveBatch* b, bool f64, uint32_t collider_count, bool capsules = false,
                              bool* saw_capsule = nullptr, const uint32_t* hull_count = nullptr, bool* saw_hull = nullptr) {
    if (saw_capsule) *saw_capsule = false;
    if (saw_hull) *saw_hull = false;
    if (!cfg) return "config is required";
    if (!b) return "batch is required";
    const double vals[6] = {cfg->delta_time, cfg->length_unit, cfg->skin_width, cfg->max_depenetration_error, cfg->penetration_rejection_threshold,
                            cfg->plane_similarity_dot_threshold};
    for (double v : vals)
        if (std::isnan(v)) return "config: NaN value";
    if (cfg->max_planes > uint32_t(MAX_PLANES)) return "config: max_planes above AVN_MOVE_MAX_PLANES";
    if (cfg->ignored && cfg->collider_count != collider_count) return "config: collider_count of `ignored` does not match the colliders";
    if (b->count >= 0x7fffffffu) return "batch: too many characters";
    if (b->count == 0) return nullptr;
    if (!b->shape || !b->dims || !b->position || !b->rotation || !b->velocity) return "batch: shape, dims, position, rotation and velocity are required";
    for (uint32_t i = 0; i < b->count; ++i) {
        if (hull_count && b->shape[i] == AVN_SHAPE_CONVEX_HULL) continue;   // its index: below
        if (!capsules && b->shape[i] > AVN_SHAPE_SPHERE) return "batch: unknown shape (only AVN_SHAPE_CUBOID and AVN_SHAPE_SPHERE)";
        if (b->shape[i] > AVN_SHAPE_CAPSULE) return "batch: unknown shape (only AVN_SHAPE_CUBOID, AVN_SHAPE_SPHERE and AVN_SHAPE_CAPSULE)";
        for (int k = 0; k < qm::shape_dims_read(b->shape[i]); ++k) {
            const double v = f64 ? static_cast<const double*>(b->dims)[3 * size_t(i) + k] : static_cast<const float*>(b->dims)[3 * size_t(i) + k];
            if (v < 0) return "batch: negative half extent, radius or half length";
        }
        if (saw_capsule && b->shape[i] == AVN_SHAPE_CAPSULE) *saw_capsule = true;
    }
    size_t at;
    if (hull_count)
        if (const char* why = avn::check_shape_column(b->shape, b->dims, b->count, f64 ? 64 : 32, &at, nullptr, hull_count, saw_hull)) return why;
    if (const char* why = qm::check_exclusions(b->count, b->exclude_count, b->exclude_offsets, b->exclude)) return why;
    if (b->plane_offsets) {
        if (b->plane_offsets[0] != 0) return "batch: plane_offsets must start at 0";
        for (uint32_t i = 0; i < b->count; ++i) {
            if (b->plane_offsets[i] > b->plane_offsets[i + 1]) return "batch: plane_offsets must be monotone";
            if (b->plane_offsets[i + 1] - b->plane_offsets[i] > cfg->max_planes) return "batch: more initial planes than max_planes";
        }
        const uint32_t np = b->plane_offsets[b->count];
        if (np && !b->planes) return "batch: plane_offsets without planes";
        for (uint32_t k = 0; k < 3 * np; k += 3) {
            double v[3];
            for (int j = 0; j < 3; ++j) v[j] = f64 ? static_cast<const double*>(b->planes)[k + j] : static_cast<const float*>(b->planes)[k + j];
            if (!std::isfinite(v[0]) || !std::isfinite(v[1]) || !std::isfinite(v[2])) return "batch: non-finite initial plane";
            const T3<float> f{float(v[0]), float(v[1]), float(v[2])};
            const float l = std::sqrt(dot(f, f));
            if (!(l > 0.0f) || !std::isfinite(l)) return "batch: zero initial plane";
        }
    }
    return nullptr;
}

template <class T>
inline Config<T> config_of(const AvnMoveConfig* c) {
    return Config<T>{T(c->delta_time), T(c->length_unit), T(c->skin_width), T(c->max_depenetration_error), T(c->penetration_rejection_threshold),
                     T(c->plane_similarity_dot_threshold), c->move_and_slide_iterations, c->depenetration_iterations, c->max_planes};
}
}  // namespace mv
