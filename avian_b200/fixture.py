"""ctypes wrapper of libavian_host.so (avian_b200/host/host_api.cpp): the CPU-side fixture around the hot path —
swept AABBs, contact graph, narrow-phase manifolds for cuboids/spheres, constraint-graph colouring.
None of this is the hot path; it produces the INPUTS the hot path consumes (identical for oracle and GPU)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _build, api

_vp = C.c_void_p
_lib = None

SHAPE_CUBOID, SHAPE_SPHERE, SHAPE_CAPSULE, SHAPE_CONVEX_HULL = 0, 1, 2, 3


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(str(_build.build_host()))
        lib.avh_create.argtypes = [C.c_uint32]
        lib.avh_create.restype = _vp
        lib.avh_destroy.argtypes = [_vp]
        lib.avh_set_shapes.argtypes = [_vp, _vp, _vp, _vp, _vp]
        lib.avh_update_aabbs.argtypes = [_vp, C.c_uint32, _vp, _vp, _vp, _vp, C.c_double, _vp, _vp, _vp]
        lib.avh_get_order.argtypes = [_vp, _vp]
        lib.avh_get_order.restype = C.c_uint32
        lib.avh_set_order.argtypes = [_vp, _vp]
        lib.avh_existing_pairs.argtypes = [_vp, _vp, C.c_uint64]
        lib.avh_existing_pairs.restype = C.c_uint64
        lib.avh_add_pairs.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, C.c_uint64]
        lib.avh_narrow_phase.argtypes = [_vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_double, C.c_uint32, C.POINTER(C.c_uint32), _vp, _vp, _vp, _vp]
        lib.avh_narrow_phase.restype = C.c_uint32
        lib.avh_export_manifolds.argtypes = [_vp, C.c_uint32] + [_vp] * 13
        lib.avh_store_impulses.argtypes = [_vp, C.c_uint32, _vp, _vp, _vp]
        lib.avh_raw_manifolds.argtypes = [C.c_uint32, C.c_uint32] + [_vp] * 12 + [C.c_double, C.c_double] + [_vp] * 13
        lib.avh_active_edges.argtypes = [_vp] * 6
        lib.avh_active_edges.restype = C.c_uint32
        lib.avh_export_edges.argtypes = [_vp] * 7
        lib.avh_export_edges.restype = None
        lib.avh_match_raw.argtypes = [C.c_uint32, C.c_uint32, _vp, _vp, _vp, _vp, C.c_double, C.c_uint32, _vp, _vp, _vp, _vp, _vp]
        lib.avh_match_raw.restype = None
        lib.avh_rows_narrow.argtypes = [C.c_uint32, C.c_uint32] + [_vp] * 27 + [C.c_double, C.c_double, C.c_double, C.c_uint32]
        lib.avh_rows_narrow.restype = None
        lib.avh_rows_narrow_framed.argtypes = lib.avh_rows_narrow.argtypes + [_vp] * 3
        lib.avh_rows_narrow_framed.restype = None
        lib.avh_rows_narrow_hulls.argtypes = lib.avh_rows_narrow_framed.argtypes + [_vp]
        lib.avh_rows_narrow_hulls.restype = None
        lib.avh_hulls_create.argtypes = [C.c_uint32, _vp, _vp, _vp, _vp, _vp, C.c_char_p, C.c_uint32]
        lib.avh_hulls_create.restype = _vp
        lib.avh_hulls_destroy.argtypes = [_vp]
        lib.avh_hulls_destroy.restype = None
        lib.avh_hulls_info.argtypes = [_vp] * 7
        lib.avh_hulls_info.restype = None
        lib.avh_raw_manifolds.restype = None
        lib.avh_remove_colliders.argtypes = [_vp, C.c_uint32, _vp]
        lib.avh_remove_colliders.restype = None
        for fn in (lib.avh_sleep_edges, lib.avh_wake_edges):
            fn.argtypes = [_vp, C.c_uint32, _vp]
            fn.restype = None
        lib.avh_graph_size.argtypes = [_vp, C.POINTER(C.c_uint32)]
        lib.avh_graph_size.restype = C.c_uint32
        lib.avh_edge_states.argtypes = [_vp, _vp, _vp, _vp]
        lib.avh_edge_states.restype = C.c_uint32
        lib.avh_set_sensors.argtypes = [_vp, _vp]
        lib.avh_set_sensors.restype = None
        lib.avh_events.argtypes = [_vp, C.c_uint32] + [_vp] * 5
        lib.avh_events.restype = C.c_uint32
        lib.avh_report.argtypes = [_vp, C.c_uint32, C.c_uint32] + [_vp] * 11
        lib.avh_report.restype = C.c_uint32
        lib.avh_pair_count.argtypes = [_vp]
        lib.avh_pair_count.restype = C.c_uint32
        P = C.POINTER
        lib.avh_query_error.argtypes = []
        lib.avh_query_error.restype = C.c_char_p
        lib.avh_query_cast_ray.argtypes = [C.c_uint32, P(api.AvnQueryColliders), P(api.AvnRayBatch), P(api.AvnRayClosest)]
        lib.avh_query_ray_hits.argtypes = [C.c_uint32, P(api.AvnQueryColliders), P(api.AvnRayBatch), P(api.AvnHitList)]
        lib.avh_query_aabb_intersections.argtypes = [C.c_uint32, P(api.AvnQueryColliders), C.c_uint32, _vp, _vp, P(api.AvnHitList)]
        lib.avh_query_cast_shape.argtypes = [C.c_uint32, P(api.AvnQueryColliders), P(api.AvnShapeBatch), P(api.AvnShapeClosest)]
        lib.avh_query_shape_hits.argtypes = [C.c_uint32, P(api.AvnQueryColliders), P(api.AvnShapeBatch), P(api.AvnShapeHitList)]
        lib.avh_query_project_point.argtypes = [C.c_uint32, P(api.AvnQueryColliders), P(api.AvnPointBatch), P(api.AvnPointProjection)]
        lib.avh_query_point_intersections.argtypes = [C.c_uint32, P(api.AvnQueryColliders), P(api.AvnPointBatch), P(api.AvnHitList)]
        lib.avh_query_shape_intersections.argtypes = [C.c_uint32, P(api.AvnQueryColliders), P(api.AvnShapeBatch), P(api.AvnHitList)]
        for f in (lib.avh_query_cast_ray, lib.avh_query_ray_hits, lib.avh_query_aabb_intersections, lib.avh_query_cast_shape, lib.avh_query_shape_hits,
                  lib.avh_query_project_point, lib.avh_query_point_intersections, lib.avh_query_shape_intersections):
            f.restype = C.c_int
        lib.avh_move_and_slide.argtypes = [C.c_uint32, P(api.AvnQueryColliders), P(api.AvnMoveConfig), P(api.AvnMoveBatch), P(api.AvnMoveResult)]
        lib.avh_move_and_slide.restype = C.c_int
        for name in ("query_cast_ray", "query_ray_hits", "query_aabb_intersections", "query_cast_shape", "query_shape_hits", "query_project_point",
                     "query_point_intersections", "query_shape_intersections", "move_and_slide"):   # the same with the hull table
            f = getattr(lib, f"avh_{name}_hulls")
            f.argtypes = getattr(lib, f"avh_{name}").argtypes + [_vp]
            f.restype = C.c_int
        lib.avh_move_project_velocity.argtypes = [C.c_uint32, _vp, _vp, C.c_uint32, _vp]
        lib.avh_move_project_velocity.restype = None
        lib.avh_move_contact.argtypes = [C.c_uint32, C.c_int, _vp, _vp, _vp, C.c_int, _vp, _vp, _vp, C.c_double, _vp, _vp]
        lib.avh_move_contact.restype = C.c_int
        lib.avh_move_contact_hulls.argtypes = lib.avh_move_contact.argtypes + [_vp]
        lib.avh_move_contact_hulls.restype = C.c_int
        lib.avh_ccd_solve.argtypes = [C.c_uint32, C.c_double, C.c_double, C.c_uint32] + [_vp] * 10 + [C.c_uint32] + [_vp] * 5 + [P(api.AvnCcdConfig)] + [_vp] * 5
        lib.avh_ccd_solve.restype = C.c_int
        lib.avh_ccd_pair_toi.argtypes = [C.c_uint32, C.c_int, _vp, _vp, C.c_double, C.c_double, C.c_double]
        lib.avh_ccd_pair_toi.restype = C.c_double
        lib.avh_ccd_nonlinear_toi.argtypes = [_vp, _vp, C.c_double, C.c_double, P(C.c_double), P(C.c_int)]
        lib.avh_ccd_nonlinear_toi.restype = C.c_int
        lib.avh_ccd_solve_hulls.argtypes = lib.avh_ccd_solve.argtypes + [_vp]
        lib.avh_ccd_solve_hulls.restype = C.c_int
        lib.avh_ccd_pair_toi_hulls.argtypes = lib.avh_ccd_pair_toi.argtypes + [_vp]
        lib.avh_ccd_pair_toi_hulls.restype = C.c_double
        lib.avh_ccd_nonlinear_toi_hulls.argtypes = lib.avh_ccd_nonlinear_toi.argtypes + [_vp]
        lib.avh_ccd_nonlinear_toi_hulls.restype = C.c_int
        lib.avh_ccd_motion_radius.argtypes = [_vp, _vp]
        lib.avh_ccd_motion_radius.restype = C.c_double
        lib.avh_ccd_apply_record.argtypes = [C.c_uint32, C.c_double, _vp, _vp, _vp, _vp]
        lib.avh_ccd_apply_record.restype = None
        _lib = lib
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data


def body_frame_columns(scalar, frames: dict | None):
    """(position, rotation, center_of_mass) of a body-frames dict (api.Context.contacts_set_body_frames' columns) in the column scalar;
    (None, None, None) without frames."""
    if frames is None:
        return None, None, None
    dt_ = np.dtype(scalar)
    col = lambda k, w: None if frames.get(k) is None else np.ascontiguousarray(frames[k], dtype=dt_).reshape(-1, w)
    return col("position", 3), col("rotation", 4), col("center_of_mass", 3)


class HullTable:
    """The fixture's convex hull table: avn_set_convex_hulls' checks and derivation (csrc/hull_math.hpp) over an api.ConvexHulls whose vertices
    are rounded to the column scalar, as the library stores them.  Raises ValueError with the library's reason for a table it refuses."""

    def __init__(self, scalar, hulls: "api.ConvexHulls"):
        self.lib = _load()
        self.hulls = hulls
        self.count = hulls.count
        v = np.ascontiguousarray(np.asarray(hulls.vertices, dtype=scalar).astype(np.float64))
        cols = [np.ascontiguousarray(a, dtype=np.uint32) for a in (hulls.vertex_offsets, hulls.face_offsets, hulls.loop_offsets, hulls.loop)]
        err = C.create_string_buffer(256)
        self.h = self.lib.avh_hulls_create(self.count, _p(cols[0]), _p(v), _p(cols[1]), _p(cols[2]), _p(cols[3]), err, 256)
        if not self.h:
            raise ValueError(err.value.decode())

    def __del__(self):
        if getattr(self, "h", None):
            self.lib.avh_hulls_destroy(self.h)
            self.h = None

    def derived(self) -> dict:
        """the derived columns: plane [F,4] (unit outward normal, offset), edge [E,4] (v0, v1, face of v0->v1, face of v1->v0; hull-local),
        edge_offsets [H+1], centre [H,3] (vertex mean), radius [H]"""
        counts = np.zeros(4, dtype=np.uint32)
        self.lib.avh_hulls_info(self.h, _p(counts), None, None, None, None, None)
        H, _, F, E = (int(x) for x in counts)
        out = {"plane": np.zeros((F, 4)), "edge": np.zeros((E, 4), dtype=np.uint32), "edge_offsets": np.zeros(H + 1, dtype=np.uint32),
               "centre": np.zeros((H, 3)), "radius": np.zeros(H)}
        self.lib.avh_hulls_info(self.h, _p(counts), *(_p(out[k]) for k in ("plane", "edge", "edge_offsets", "centre", "radius")))
        return out


def _hull_table(scalar, hulls) -> "HullTable | None":
    if hulls is None or isinstance(hulls, HullTable):
        return hulls
    return HullTable(scalar, hulls)


def check_hull_indices(shape, dims, hulls) -> None:
    """What avn_update_aabbs / avn_narrow_phase / avn_contacts_step refuse: a hull collider without a table, or an index the table does not hold."""
    if shape is None:
        return
    hull = np.asarray(shape) == SHAPE_CONVEX_HULL
    if not hull.any():
        return
    if hulls is None:
        raise ValueError("a convex hull collider, and no hull table")
    idx = np.asarray(dims, dtype=np.float64).reshape(-1, 3)[hull, 0]
    if not (np.all(idx >= 0) and np.all(idx < hulls.count) and np.all(idx == np.floor(idx))):
        raise ValueError("a convex hull's index must be integral, not negative and below the hull table's count")


def raw_manifolds(scalar, dt: float, contact_tolerance: float, pairs, colliders: dict, lin_vel: np.ndarray, ang_vel: np.ndarray,
                  f64_anchors: bool = False, frames: dict | None = None, hulls=None) -> dict:
    """The geometry stage of the fixture's narrow phase for an explicit pair list (same columns as Context.narrow_phase).
    f64_anchors adds the unrounded anchors (what match_contacts compares on the next step).  frames: the body frames (dict position,
    rotation, center_of_mass=None, [B] rows), as Context.contacts_set_body_frames sets them; the anchors are then relative to the bodies'
    centres of mass.  hulls: the convex hull table (api.ConvexHulls or HullTable) the hull colliders index."""
    lib = _load()
    dt_ = np.dtype(scalar)
    hulls = _hull_table(dt_, hulls)
    check_hull_indices(colliders.get("shape"), colliders.get("dims"), hulls)
    fp, fr, fc = body_frame_columns(dt_, frames)
    c1, c2, b1, b2 = (np.ascontiguousarray(x, dtype=np.uint32) for x in pairs)
    n = int(c1.shape[0])
    cols = {k: (None if colliders.get(k) is None else np.ascontiguousarray(colliders[k], dtype=(np.uint8 if k == "shape" else dt_)))
            for k in ("shape", "dims", "position", "rotation", "aabb_min", "aabb_max")}
    lv, av = np.ascontiguousarray(lin_vel, dtype=dt_), np.ascontiguousarray(ang_vel, dtype=dt_)
    out = {"point_count": np.zeros(n, dtype=np.uint8), "disjoint": np.zeros(n, dtype=np.uint8), "normal": np.zeros((n, 3), dtype=dt_),
           "anchor1": np.zeros((n, 4, 3), dtype=dt_), "anchor2": np.zeros((n, 4, 3), dtype=dt_), "penetration": np.zeros((n, 4), dtype=dt_),
           "normal_speed": np.zeros((n, 4), dtype=dt_)}
    a1d = np.zeros((n, 4, 3), dtype=np.float64) if f64_anchors else None
    a2d = np.zeros((n, 4, 3), dtype=np.float64) if f64_anchors else None
    lib.avh_raw_manifolds(32 if dt_ == np.float32 else 64, n, _p(c1), _p(c2), _p(b1), _p(b2), _p(cols["shape"]), _p(cols["dims"]), _p(cols["position"]),
                          _p(cols["rotation"]), _p(lv), _p(av), _p(cols["aabb_min"]), _p(cols["aabb_max"]), float(dt), float(contact_tolerance),
                          *(_p(out[k]) for k in ("point_count", "disjoint", "normal", "anchor1", "anchor2", "penetration", "normal_speed")), _p(a1d), _p(a2d),
                          _p(fp), _p(fr), _p(fc), hulls.h if hulls is not None else None)
    if f64_anchors:
        out["anchor1_f64"], out["anchor2_f64"] = a1d, a2d
    return out


# ---- spatial queries by brute force over every collider (csrc/query_math.hpp, csrc/hull_query_math.hpp): what the device tree must reproduce
# bit for bit.  capsules=True accepts capsule colliders and query shapes (characters for move_and_slide); without it a capsule is refused as an
# unknown shape.  hulls=<HullTable or api.ConvexHulls> accepts convex hulls that index it, and capsules with them; without it a hull is
# refused as an unknown shape.  The device accepts capsules with no flag, and hulls with the context's table.
def _query_check(lib, st: int) -> None:
    if st != api.OK:
        raise api.AvianError(st, lib.avh_query_error().decode())


CAPSULE_BIT = 0x100   # OR-ed into scalar_bits: the brute force accepts capsule colliders, query shapes and characters
HULL_BIT = 0x200      # OR-ed into scalar_bits: convex hulls too, with the table of the avh_*_hulls entry points


def _bits(dt, capsules: bool, hulls=None) -> int:
    return (32 if dt == np.float32 else 64) | (CAPSULE_BIT if capsules else 0) | (HULL_BIT if hulls is not None else 0)


def _call(lib, name: str, dt, capsules: bool, hulls, *args) -> int:
    """avh_<name>, or avh_<name>_hulls with the table when hulls is given"""
    if hulls is None:
        return getattr(lib, f"avh_{name}")(_bits(dt, capsules), *args)
    return getattr(lib, f"avh_{name}_hulls")(_bits(dt, capsules, hulls), *args, hulls.h)


def query_cast_ray(scalar, colliders: "api.QueryColliders", rays: "api.Rays", capsules: bool = False, hulls=None) -> dict:
    """The closest hit of every ray (same output as Context.cast_ray)."""
    lib, dt = _load(), np.dtype(scalar)
    hulls = _hull_table(dt, hulls)
    c, keep_c = colliders.as_struct(dt)
    r, keep_r = rays.as_struct(dt)
    n = rays.count
    out = {"collider": np.zeros(n, dtype=np.int32), "distance": np.zeros(n, dtype=dt), "normal": np.zeros((n, 3), dtype=dt)}
    o = api.AvnRayClosest(*(_p(out[k]) for k in ("collider", "distance", "normal")))
    _query_check(lib, _call(lib, "query_cast_ray", dt, capsules, hulls, C.byref(c), C.byref(r), C.byref(o)))
    return out


def query_ray_hits(scalar, colliders: "api.QueryColliders", rays: "api.Rays", capsules: bool = False, hulls=None) -> dict:
    """Every ray's max_hits nearest hits in (t, collider) order as CSR (same output as Context.ray_hits)."""
    lib, dt = _load(), np.dtype(scalar)
    hulls = _hull_table(dt, hulls)
    c, keep_c = colliders.as_struct(dt)
    r, keep_r = rays.as_struct(dt)
    h, out = api.hit_list(rays.count, 0, dt, True)
    st = _call(lib, "query_ray_hits", dt, capsules, hulls, C.byref(c), C.byref(r), C.byref(h))
    if st == api.ERR_CAPACITY:
        h, out = api.hit_list(rays.count, int(h.count), dt, True)
        st = _call(lib, "query_ray_hits", dt, capsules, hulls, C.byref(c), C.byref(r), C.byref(h))
    _query_check(lib, st)
    return api.hit_list_result(h, out)


def query_aabb_intersections(scalar, colliders: "api.QueryColliders", aabb_min, aabb_max, capsules: bool = False, hulls=None) -> dict:
    """Per query box the colliders whose tight AABB it touches, ascending (same output as Context.aabb_intersections)."""
    lib, dt = _load(), np.dtype(scalar)
    hulls = _hull_table(dt, hulls)
    c, keep_c = colliders.as_struct(dt)
    mn = np.ascontiguousarray(aabb_min, dtype=dt).reshape(-1, 3)
    mx = np.ascontiguousarray(aabb_max, dtype=dt).reshape(-1, 3)
    n = int(mn.shape[0])
    h, out = api.hit_list(n, 0, dt, False)
    st = _call(lib, "query_aabb_intersections", dt, capsules, hulls, C.byref(c), n, _p(mn), _p(mx), C.byref(h))
    if st == api.ERR_CAPACITY:
        h, out = api.hit_list(n, int(h.count), dt, False)
        st = _call(lib, "query_aabb_intersections", dt, capsules, hulls, C.byref(c), n, _p(mn), _p(mx), C.byref(h))
    _query_check(lib, st)
    return api.hit_list_result(h, out)


def query_cast_shape(scalar, colliders: "api.QueryColliders", shapes: "api.ShapeQueries", capsules: bool = False, hulls=None) -> dict:
    """The closest hit of every cast (same output as Context.cast_shape)."""
    lib, dt = _load(), np.dtype(scalar)
    hulls = _hull_table(dt, hulls)
    c, keep_c = colliders.as_struct(dt)
    s, keep_s = shapes.as_struct(dt)
    o, out = api.shape_closest(shapes.count, dt)
    _query_check(lib, _call(lib, "query_cast_shape", dt, capsules, hulls, C.byref(c), C.byref(s), C.byref(o)))
    return out


def query_shape_hits(scalar, colliders: "api.QueryColliders", shapes: "api.ShapeQueries", capsules: bool = False, hulls=None) -> dict:
    """Every cast's max_hits nearest hits in (t, collider) order as CSR (same output as Context.shape_hits)."""
    lib, dt = _load(), np.dtype(scalar)
    hulls = _hull_table(dt, hulls)
    c, keep_c = colliders.as_struct(dt)
    s, keep_s = shapes.as_struct(dt)
    h, out = api.shape_hit_list(shapes.count, 0, dt)
    st = _call(lib, "query_shape_hits", dt, capsules, hulls, C.byref(c), C.byref(s), C.byref(h))
    if st == api.ERR_CAPACITY:
        h, out = api.shape_hit_list(shapes.count, int(h.count), dt)
        st = _call(lib, "query_shape_hits", dt, capsules, hulls, C.byref(c), C.byref(s), C.byref(h))
    _query_check(lib, st)
    return api.hit_list_result(h, out)


def query_project_point(scalar, colliders: "api.QueryColliders", points: "api.Points", capsules: bool = False, hulls=None) -> dict:
    """The closest collider of every point and the projection onto it (same output as Context.project_point)."""
    lib, dt = _load(), np.dtype(scalar)
    hulls = _hull_table(dt, hulls)
    c, keep_c = colliders.as_struct(dt)
    p, keep_p = points.as_struct(dt)
    o, out = api.point_projection(points.count, dt)
    _query_check(lib, _call(lib, "query_project_point", dt, capsules, hulls, C.byref(c), C.byref(p), C.byref(o)))
    return out


def _query_list(fn, scalar, colliders, batch, capsules: bool, hulls=None) -> dict:
    lib, dt = _load(), np.dtype(scalar)
    hulls = _hull_table(dt, hulls)
    c, keep_c = colliders.as_struct(dt)
    b, keep_b = batch.as_struct(dt)
    n = batch.count
    h, out = api.hit_list(n, 0, dt, False)
    st = _call(lib, fn, dt, capsules, hulls, C.byref(c), C.byref(b), C.byref(h))
    if st == api.ERR_CAPACITY:
        h, out = api.hit_list(n, int(h.count), dt, False)
        st = _call(lib, fn, dt, capsules, hulls, C.byref(c), C.byref(b), C.byref(h))
    _query_check(lib, st)
    return api.hit_list_result(h, out)


def query_point_intersections(scalar, colliders: "api.QueryColliders", points: "api.Points", capsules: bool = False, hulls=None) -> dict:
    """Per point the colliders containing it, ascending (same output as Context.point_intersections)."""
    return _query_list("query_point_intersections", scalar, colliders, points, capsules, hulls)


def query_shape_intersections(scalar, colliders: "api.QueryColliders", shapes: "api.ShapeQueries", capsules: bool = False, hulls=None) -> dict:
    """Per query shape the colliders it intersects, ascending (same output as Context.shape_intersections)."""
    return _query_list("query_shape_intersections", scalar, colliders, shapes, capsules, hulls)


# ---- move and slide by brute force over every collider (csrc/move_math.hpp): what the device kernel must reproduce bit for bit
def move_and_slide(scalar, colliders: "api.QueryColliders", config: "api.MoveConfig", batch: "api.MoveBatch", capsules: bool = False,
                   hulls=None) -> dict:
    """MoveAndSlide::move_and_slide for every character (same output as Context.move_and_slide; kernel_ms is 0)."""
    lib, dt = _load(), np.dtype(scalar)
    hulls = _hull_table(dt, hulls)
    c, keep_c = colliders.as_struct(dt)
    m, keep_m = config.as_struct()
    b, keep_b = batch.as_struct(dt)
    o, out = api.move_result(batch.count, config.move_and_slide_iterations, dt)
    _query_check(lib, _call(lib, "move_and_slide", dt, capsules, hulls, C.byref(c), C.byref(m), C.byref(b), C.byref(o)))
    out["kernel_ms"] = 0.0
    return out


def project_velocity(scalar, v, normals) -> np.ndarray:
    """The shared project_velocity (velocity_project.rs:122-324) on one velocity; normals are rounded to f32 (Dir)."""
    lib, dt = _load(), np.dtype(scalar)
    x = np.ascontiguousarray(v, dtype=dt).reshape(3)
    ns = np.ascontiguousarray(normals, dtype=np.float32).reshape(-1, 3)
    out = np.zeros(3, dtype=dt)
    lib.avh_move_project_velocity(32 if dt == np.float32 else 64, _p(x), _p(ns) if ns.size else None, int(ns.shape[0]), _p(out))
    return out


def move_contact(scalar, shape_a: int, dims_a, pos_a, rot_a, shape_b: int, dims_b, pos_b, rot_b, prediction: float, hulls=None):
    """One intersection of a move: (f32 plane normal, deepest penetration) of character a against collider b, or None.  hulls: the table
    that hull shapes index (the hull instance's contact planes)."""
    lib = _load()
    d = lambda a, k: np.ascontiguousarray(a, dtype=np.float64).reshape(k)
    cols = [d(dims_a, 3), d(pos_a, 3), d(rot_a, 4), d(dims_b, 3), d(pos_b, 3), d(rot_b, 4)]
    n, pen = np.zeros(3, dtype=np.float32), np.zeros(1, dtype=np.float64)
    args = (32 if np.dtype(scalar) == np.float32 else 64, int(shape_a), _p(cols[0]), _p(cols[1]), _p(cols[2]), int(shape_b),
            _p(cols[3]), _p(cols[4]), _p(cols[5]), float(prediction), _p(n), _p(pen))
    if hulls is None:
        hit = lib.avh_move_contact(*args)
    else:
        table = _hull_table(np.dtype(scalar), hulls)   # held for the call: the table is freed with it
        hit = lib.avh_move_contact_hulls(*args, table.h)
    return (n, float(pen[0])) if hit else None


class HostPipeline:
    """Contact graph + narrow-phase fixture + constraint graph for a fixed set of colliders.  Without collider_body: one collider per body,
    collider Entity::index() == body Entity::index() == row in the body columns.  collider_body ([C], a collider table): the body of every
    collider; the AABB update and the narrow phase then take the colliders' world poses (and their velocities) separately."""

    def __init__(self, shape_type: np.ndarray, dims: np.ndarray, friction: np.ndarray, restitution: np.ndarray, scalar=np.float32,
                 collider_body: np.ndarray | None = None, hulls=None):
        """hulls: the convex hull table (api.ConvexHulls or HullTable) that hull colliders index."""
        self.lib = _load()
        self.hulls = _hull_table(scalar, hulls)
        check_hull_indices(shape_type, dims, self.hulls)
        self.collider_body = None if collider_body is None else np.ascontiguousarray(collider_body, dtype=np.uint32)
        self.n = int(shape_type.shape[0])
        self.scalar = np.dtype(scalar)
        self.bits = 32 if self.scalar == np.float32 else 64
        dims = np.asarray(dims, dtype=self.scalar).astype(np.float64)      # shapes carry the world's scalar type (Collider is f32 in an f32 build)
        self.h = self.lib.avh_create(self.n)
        st = np.ascontiguousarray(shape_type, dtype=np.int32)
        dm = np.ascontiguousarray(dims, dtype=np.float64)
        fr = np.ascontiguousarray(friction, dtype=np.float64)
        rs = np.ascontiguousarray(restitution, dtype=np.float64)
        self.lib.avh_set_shapes(self.h, _p(st), _p(dm), _p(fr), _p(rs))

    def __del__(self):
        if getattr(self, "h", None):
            self.lib.avh_destroy(self.h)
            self.h = None

    def update_aabbs(self, bodies: api.Bodies, dt: float, colliders: dict | None = None):
        """colliders (a collider table): dict position, rotation, linear_velocity, angular_velocity per collider; None = the body columns."""
        mn = np.empty((self.n, 3), dtype=self.scalar)
        mx = np.empty((self.n, 3), dtype=self.scalar)
        c = {"position": bodies.position, "rotation": bodies.rotation, "linear_velocity": bodies.linear_velocity, "angular_velocity": bodies.angular_velocity}
        if colliders is not None:
            c = {k: np.ascontiguousarray(colliders[k], dtype=self.scalar) for k in c}
        self.lib.avh_update_aabbs(self.h, self.bits, _p(c["position"]), _p(c["rotation"]), _p(c["linear_velocity"]), _p(c["angular_velocity"]), dt,
                                  _p(mn), _p(mx), self.hulls.h if self.hulls is not None else None)
        return mn, mx

    def intervals(self, bodies: api.Bodies, aabb_min: np.ndarray, aabb_max: np.ndarray, with_existing: bool = True) -> api.Aabbs:
        """AabbIntervals in the persistent order + the pair set, as the broad phase's input columns."""
        order = np.empty(self.n, dtype=np.uint32)
        self.lib.avh_get_order(self.h, _p(order))
        body = order.copy() if self.collider_body is None else np.ascontiguousarray(self.collider_body[order])
        flags = np.where(bodies.kind[body] == api.BODY_STATIC, api.AABB_IS_INACTIVE, 0).astype(np.uint8) | np.uint8(api.AABB_GENERATE_CONSTRAINTS)
        existing = None
        if with_existing:
            cnt = int(self.lib.avh_existing_pairs(self.h, None, 0))
            if cnt:
                existing = np.empty(cnt, dtype=np.uint64)
                self.lib.avh_existing_pairs(self.h, _p(existing), cnt)
        return api.Aabbs(collider=order.copy(), body=body, aabb_min=np.ascontiguousarray(aabb_min[order]),
                         aabb_max=np.ascontiguousarray(aabb_max[order]), flags=np.ascontiguousarray(flags),
                         order_out=np.empty(self.n, dtype=np.uint32), existing_pairs=existing)

    def commit_broadphase(self, aabbs: api.Aabbs, pairs: api.PairList) -> None:
        """Persist the sorted interval order and add the new pairs to the contact graph (broad_phase.rs:443-471)."""
        new_order = np.ascontiguousarray(aabbs.collider[aabbs.order_out])
        self.lib.avh_set_order(self.h, _p(new_order))
        n = int(pairs.count)
        if n:
            c1, c2, b1, b2, fl = (np.ascontiguousarray(x[:n]) for x in (pairs.collider1, pairs.collider2, pairs.body1, pairs.body2, pairs.flags))
            self.lib.avh_add_pairs(self.h, _p(c1), _p(c2), _p(b1), _p(b2), _p(fl), n)

    def narrow_phase(self, bodies: api.Bodies, aabb_min: np.ndarray, aabb_max: np.ndarray, dt: float, match_contacts: bool = True,
                     colliders: dict | None = None) -> api.Manifolds:
        """colliders: the collider table's world poses (dict position, rotation, [C] rows); the anchors are then relative to the bodies'
        centres of mass (bodies.position / rotation / center_of_mass are the body frames).  None: one collider per body."""
        pts = C.c_uint32(0)
        kind = np.ascontiguousarray(bodies.kind, dtype=np.uint8)
        if colliders is None:
            pos, rot, frames = bodies.position, bodies.rotation, (None, None, None)
        else:
            pos, rot = (np.ascontiguousarray(colliders[k], dtype=self.scalar) for k in ("position", "rotation"))
            frames = body_frame_columns(self.scalar, {"position": bodies.position, "rotation": bodies.rotation, "center_of_mass": bodies.center_of_mass})
        m = int(self.lib.avh_narrow_phase(self.h, self.bits, _p(kind), _p(pos), _p(rot), _p(bodies.linear_velocity),
                                          _p(bodies.angular_velocity), _p(aabb_min), _p(aabb_max), dt, 1 if match_contacts else 0, C.byref(pts),
                                          *(_p(f) for f in frames), self.hulls.h if self.hulls is not None else None))
        return self.export_manifolds(m, int(pts.value))

    def export_manifolds(self, m: int | None = None, p: int | None = None) -> api.Manifolds:
        """The constraint graph's manifolds grouped by colour (m manifolds with p points; None = ask the graph, e.g. after wake_edges)."""
        if m is None:
            pts = C.c_uint32(0)
            m = int(self.lib.avh_graph_size(self.h, C.byref(pts)))
            p = int(pts.value)
        s = self.scalar
        man = api.Manifolds(
            color_offsets=np.zeros(api.GRAPH_COLOR_COUNT + 1, dtype=np.uint32), body1=np.zeros(m, dtype=np.int32), body2=np.zeros(m, dtype=np.int32),
            normal=np.zeros((m, 3), dtype=s), friction=np.zeros(m, dtype=s), restitution=np.zeros(m, dtype=s),
            point_offsets=np.zeros(m + 1, dtype=np.uint32), anchor1=np.zeros((p, 3), dtype=s), anchor2=np.zeros((p, 3), dtype=s),
            penetration=np.zeros(p, dtype=s), normal_speed=np.zeros(p, dtype=s), warm_start_normal_impulse=np.zeros(p, dtype=s),
            warm_start_tangent_impulse=np.zeros((p, 2), dtype=s), normal_impulse=np.zeros(p, dtype=s))
        self.lib.avh_export_manifolds(self.h, self.bits, _p(man.color_offsets), _p(man.body1), _p(man.body2), _p(man.normal), _p(man.friction),
                                      _p(man.restitution), _p(man.point_offsets), _p(man.anchor1), _p(man.anchor2), _p(man.penetration),
                                      _p(man.normal_speed), _p(man.warm_start_normal_impulse), _p(man.warm_start_tangent_impulse))
        return man

    # ---- the graphs in the contact store's terms: ContactId-indexed edges (SURVEY.md 8f #1/#3)
    def active_edges(self):
        n = self.pair_count
        ids, c1, c2, b1, b2 = (np.zeros(n, dtype=np.uint32) for _ in range(5))
        k = int(self.lib.avh_active_edges(self.h, _p(ids), _p(c1), _p(c2), _p(b1), _p(b2)))
        return ids[:k], c1[:k], c2[:k], b1[:k], b2[:k]

    def export_edges(self, m: int):
        """The constraint graph as a colour-major list of edge ids + per-edge bodies and material."""
        co = np.zeros(api.GRAPH_COLOR_COUNT + 1, dtype=np.uint32)
        edge, b1, b2 = np.zeros(m, dtype=np.uint32), np.zeros(m, dtype=np.int32), np.zeros(m, dtype=np.int32)
        fr, re = np.zeros(m, dtype=np.float64), np.zeros(m, dtype=np.float64)
        self.lib.avh_export_edges(self.h, _p(co), _p(edge), _p(b1), _p(b2), _p(fr), _p(re))
        return co, edge, b1, b2, fr, re

    def store_impulses(self, man: api.Manifolds) -> None:
        self.lib.avh_store_impulses(self.h, self.bits, _p(man.warm_start_normal_impulse), _p(man.warm_start_tangent_impulse), _p(man.normal_impulse))

    # ---- the pipeline's output to the application: what avn_contacts_set_sensors / _remove_colliders / _events / _report do on the device
    def set_sensors(self, sensor) -> None:
        """The Sensor column (None = none); remove_collider for every collider whose flag changed."""
        col = None if sensor is None else np.ascontiguousarray(sensor, dtype=bool).astype(np.uint8)
        self.lib.avh_set_sensors(self.h, _p(col))

    def remove_colliders(self, colliders) -> None:
        ids = np.ascontiguousarray(colliders, dtype=np.uint32)
        self.lib.avh_remove_colliders(self.h, int(ids.shape[0]), _p(ids))

    def sleep_edges(self, ids) -> None:
        """ContactGraph::sleep_entity_with for these ContactIds (ascending): out of the ConstraintGraph, skipped by the narrow phase."""
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        self.lib.avh_sleep_edges(self.h, int(ids.shape[0]), _p(ids))

    def wake_edges(self, ids) -> None:
        """ContactGraph::wake_entity_with for these ContactIds (ascending): touching, constraint-generating pairs are pushed again."""
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        self.lib.avh_wake_edges(self.h, int(ids.shape[0]), _p(ids))

    def edge_states(self) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
        """(ContactId, touching, asleep) of every live pair, ascending ContactId."""
        n = int(self.lib.avh_edge_states(self.h, None, None, None))
        ids, t, a = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint8), np.zeros(n, dtype=np.uint8)
        if n:
            self.lib.avh_edge_states(self.h, _p(ids), _p(t), _p(a))
        return ids, t.astype(bool), a.astype(bool)

    def events(self) -> tuple[dict, dict]:
        """(started, ended) of the last status loop, as Context.contacts_events returns them."""
        lists = []
        for which in (0, 1):
            n = int(self.lib.avh_events(self.h, which, None, None, None, None, None))
            out = {k: np.zeros(n, dtype=d) for k, d in api.EVENT_COLUMNS}
            self.lib.avh_events(self.h, which, *(_p(out[k]) for k, _ in api.EVENT_COLUMNS))
            lists.append(out)
        return lists[0], lists[1]

    def report(self, events_only: bool = False) -> dict:
        """The touching pairs in ascending ContactId from the stored impulses, as Context.contacts_report returns them."""
        eo = 1 if events_only else 0
        n = int(self.lib.avh_report(self.h, self.bits, eo, *([None] * 11)))
        _, out = api.contact_report(n, self.scalar)
        out = {k: v[:n].copy() for k, v in out.items()}
        self.lib.avh_report(self.h, self.bits, eo, *(_p(out[k]) for k, _ in api.AvnContactReport._fields_[2:]))
        return out

    @property
    def pair_count(self) -> int:
        return int(self.lib.avh_pair_count(self.h))


# ---- swept CCD (csrc/ccd_math.hpp): the host brute force the device pass is compared with ----------------------------------------------------
def ccd_motion(shape: int, dims, position, rotation, linear_velocity=(0, 0, 0), angular_velocity=(0, 0, 0), com=(0, 0, 0)) -> np.ndarray:
    """One body of a CCD pair as the 20 doubles avh_ccd_pair_toi takes."""
    return np.concatenate([[float(shape)], np.asarray(dims, float).reshape(3), np.asarray(position, float).reshape(3), np.asarray(rotation, float).reshape(4),
                           np.asarray(com, float).reshape(3), np.asarray(linear_velocity, float).reshape(3), np.asarray(angular_velocity, float).reshape(3)])


def ccd_pair_toi(scalar, mode: int, a: np.ndarray, b: np.ndarray, dt: float, eps: float = 1e-4, prediction_distance: float = float("inf"),
                 hulls=None) -> float:
    """compute_ccd_toi of one pair against the bound dt, rounded to the column scalar (-1 = no hit).  hulls: the hull table (HullTable or
    api.ConvexHulls) that convex hull motions (shape 3, dims[0] = index) index; the shape level then includes hulls."""
    a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    bits = 32 if np.dtype(scalar) == np.float32 else 64
    args = (bits, int(mode), a.ctypes.data, b.ctypes.data, float(dt), float(eps), float(prediction_distance))
    if hulls is None:
        return _load().avh_ccd_pair_toi(*args)
    table = _hull_table(scalar, hulls)   # held until the call returns: the table is freed with it
    return _load().avh_ccd_pair_toi_hulls(*args, table.h)


def ccd_nonlinear_toi(a: np.ndarray, b: np.ndarray, t_max: float, eps: float = 1e-4, iterations: bool = False, hulls=None):
    """The raw conservative-advancement TOI in double, or None; with iterations=True, (TOI or None, distance evaluations).  hulls: as
    ccd_pair_toi (a table built from api.ConvexHulls keeps the vertices in double)."""
    a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    t, its = C.c_double(), C.c_int(0)
    args = (a.ctypes.data, b.ctypes.data, float(t_max), float(eps), C.byref(t), C.byref(its))
    table = _hull_table(np.float64, hulls)
    hit = _load().avh_ccd_nonlinear_toi(*args) if table is None else _load().avh_ccd_nonlinear_toi_hulls(*args, table.h)
    out = t.value if hit else None
    return (out, its.value) if iterations else out


def ccd_motion_radius(a: np.ndarray, hulls=None) -> float:
    """The spin bound R of one motion (its farthest point from the centre of mass, csrc/ccd_math.hpp motion_radius)."""
    a = np.ascontiguousarray(a, dtype=np.float64)
    table = _hull_table(np.float64, hulls)
    return _load().avh_ccd_motion_radius(a.ctypes.data, None if table is None else table.h)


def ccd_apply_record(scalar, m: float, v, w, dp, dq):
    """The delta write of one CCD record (overwrite dp, compose from_scaled_axis(w m) onto dq) in the column scalar; returns (dp, dq)."""
    v, w = np.ascontiguousarray(v, dtype=np.float64), np.ascontiguousarray(w, dtype=np.float64)
    dp, dq = np.array(dp, dtype=np.float64), np.array(dq, dtype=np.float64)
    _load().avh_ccd_apply_record(32 if np.dtype(scalar) == np.float32 else 64, float(m), v.ctypes.data, w.ctypes.data, dp.ctypes.data, dq.ctypes.data)
    return dp, dq


def ccd_solve(scalar, dt: float, length_unit: float, bodies: dict, shape, dims, rows: dict, cfg: dict, delta_position=None, delta_rotation=None,
              hulls=None) -> dict:
    """solve_swept_ccd over the contact rows (dict c1, c2, b1, b2, live) by the reference's sequential loop.  bodies: dict kind, position,
    rotation, linear_velocity, angular_velocity (SolverBody velocities after the substeps), center_of_mass (optional).  cfg: the keyword
    arguments of api.ccd_config, plus capsules=True for api.CCD_CAPSULES and hulls=True for api.CCD_HULLS (as Context.ccd_configure takes
    them).  hulls: the hull table (HullTable or api.ConvexHulls) the hull colliders index.  delta_position / delta_rotation are updated in
    place when given.  Returns what Context.ccd_download returns."""
    lib, dt_ = _load(), np.dtype(scalar)
    hulls = _hull_table(dt_, hulls)
    col = lambda a, t=dt_: None if a is None else np.ascontiguousarray(a, dtype=t)
    kind = col(bodies.get("kind"), np.uint8)
    pos, rot, com, lv, av = (col(bodies.get(k)) for k in ("position", "rotation", "center_of_mass", "linear_velocity", "angular_velocity"))
    B = int(pos.shape[0])
    sh, dm = col(shape, np.uint8), col(dims)
    c1, c2, b1, b2 = (col(rows[k], np.uint32) for k in ("c1", "c2", "b1", "b2"))
    live = col(rows["live"], np.uint8)
    cfg = dict(cfg)
    cfg["flags"] = cfg.get("flags", 0) | (api.CCD_CAPSULES if cfg.pop("capsules", False) else 0) | (api.CCD_HULLS if cfg.pop("hulls", False) else 0)
    conf, keep = api.ccd_config(**cfg)
    n = int(conf.count)
    out = {"min_toi": np.zeros(n, dtype=dt_), "hit_body": np.zeros(n, dtype=np.int32), "hit_contact": np.zeros(n, dtype=np.int32),
           "candidates": np.zeros(n, dtype=np.uint32), "hits": np.zeros(n, dtype=np.uint32)}
    for a in (delta_position, delta_rotation):
        assert a is None or (a.dtype == dt_ and a.flags["C_CONTIGUOUS"])
    args = (32 if dt_ == np.float32 else 64, float(dt), float(length_unit), B, _p(kind), _p(pos), _p(rot), _p(com), _p(lv), _p(av),
            _p(delta_position), _p(delta_rotation), _p(sh), _p(dm), int(c1.shape[0]), _p(c1), _p(c2), _p(b1), _p(b2), _p(live), C.byref(conf),
            *(_p(out[k]) for k in ("min_toi", "hit_body", "hit_contact", "candidates", "hits")))
    st = lib.avh_ccd_solve(*args) if hulls is None else lib.avh_ccd_solve_hulls(*args, hulls.h)
    if st == api.ERR_UNSUPPORTED:
        raise api.AvianError(st, "avh_ccd_solve: a contact row names a capsule and the configuration does not set CCD_CAPSULES, "
                                 "or a convex hull and it does not set CCD_HULLS")
    if st != 0:
        raise ValueError("avh_ccd_solve: invalid configuration (an unknown flag bit included), or a contact row names a convex hull the hull "
                         "table does not hold")
    return out
