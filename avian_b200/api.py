"""ctypes binding of include/avian_b200.h — the same C ABI the Rust shim binds (INTEGRATION.md).

Nothing here computes: arrays go in as numpy buffers, the CUDA library does the work.  If the library or a
CUDA device is missing the constructors raise — there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import _build

GRAPH_COLOR_COUNT = 24
COLOR_OVERFLOW = 23
DYNAMIC_COLOR_COUNT = 20
MAX_MANIFOLD_POINTS = 4
NO_BODY = -1
BODY_DYNAMIC, BODY_KINEMATIC, BODY_STATIC = 0, 1, 2
JOINT_FIXED, JOINT_REVOLUTE, JOINT_SPHERICAL, JOINT_PRISMATIC, JOINT_DISTANCE = range(5)
JOINT_TYPE_COUNT = 5
AABB_IS_INACTIVE, AABB_CONTACT_EVENTS, AABB_GENERATE_CONSTRAINTS, AABB_CUSTOM_FILTER, AABB_MODIFY_CONTACTS = 1, 2, 4, 8, 16
PAIR_CONTACT_EVENTS, PAIR_MODIFY_CONTACTS, PAIR_GENERATE_CONSTRAINTS, PAIR_NEEDS_HOOK = 1, 2, 4, 8
CFG_FAST_TRIG = 1
OK, ERR_INVALID_ARGUMENT, ERR_CUDA, ERR_OUT_OF_MEMORY, ERR_UNSUPPORTED, ERR_CAPACITY, ERR_NCCL = 0, -1, -2, -3, -4, -5, -6
# AvnShape; a capsule's dims are [radius, half length, unused] with its segment along the collider's local y
SHAPE_CUBOID, SHAPE_SPHERE, SHAPE_CAPSULE = 0, 1, 2

_vp = C.c_void_p


class AvnConfig(C.Structure):
    _fields_ = [("abi_version", C.c_uint32), ("device", C.c_int32), ("scalar_bits", C.c_uint32), ("flags", C.c_uint32)]


class AvnStepParams(C.Structure):
    _fields_ = [
        ("dt", C.c_double), ("h", C.c_double), ("substeps", C.c_uint32), ("restitution_iterations", C.c_uint32),
        ("gravity", C.c_double * 3), ("contact_damping_ratio", C.c_double), ("contact_frequency_factor", C.c_double),
        ("max_overlap_solve_speed", C.c_double), ("warm_start_coefficient", C.c_double), ("restitution_threshold", C.c_double),
        ("length_unit", C.c_double), ("match_contacts", C.c_uint32), ("solver_iterations", C.c_uint32),
    ]


class AvnBodyColumns(C.Structure):
    _fields_ = [("count", C.c_uint32), ("_pad", C.c_uint32)] + [
        (n, _vp) for n in (
            "kind", "position", "rotation", "linear_velocity", "angular_velocity", "inverse_mass", "inverse_inertia_local",
            "center_of_mass", "locked_axes", "dominance", "linear_damping", "angular_damping", "gravity_scale",
            "linear_acceleration", "angular_acceleration", "max_linear_speed", "max_angular_speed", "integration_flags")]


class AvnManifoldColumns(C.Structure):
    _fields_ = [("count", C.c_uint32), ("point_count", C.c_uint32), ("color_offsets", C.c_uint32 * (GRAPH_COLOR_COUNT + 1))] + [
        (n, _vp) for n in (
            "body1", "body2", "normal", "friction", "restitution", "tangent_velocity", "point_offsets", "anchor1", "anchor2",
            "penetration", "normal_speed", "warm_start_normal_impulse", "warm_start_tangent_impulse", "normal_impulse")]


class AvnJointColumns(C.Structure):
    _fields_ = [("count", C.c_uint32), ("_pad", C.c_uint32)] + [
        (n, _vp) for n in (
            "body1", "body2", "local_anchor1", "local_anchor2", "local_basis1", "local_basis2", "axis", "limit_enabled",
            "limit_min", "limit_max", "limit2_min", "limit2_max", "compliance0", "compliance1", "compliance2",
            "damping_enabled", "damping_linear", "damping_angular", "force", "torque")]


class AvnJointSet(C.Structure):
    _fields_ = [("types", AvnJointColumns * JOINT_TYPE_COUNT)]


class AvnAabbColumns(C.Structure):
    _fields_ = [("count", C.c_uint32), ("retained_count", C.c_uint32)] + [
        (n, _vp) for n in ("collider", "body", "aabb_min", "aabb_max", "memberships", "filters", "flags", "order_out")] + [
        ("existing_pairs", _vp), ("existing_pair_count", C.c_uint64), ("joint_disabled_body_pairs", _vp), ("joint_disabled_pair_count", C.c_uint64)]


class AvnPairList(C.Structure):
    _fields_ = [("capacity", C.c_uint64), ("count", C.c_uint64)] + [(n, _vp) for n in ("collider1", "collider2", "body1", "body2", "flags")]


class AvnAabbParams(C.Structure):
    _fields_ = [("dt", C.c_double), ("contact_tolerance", C.c_double), ("default_speculative_margin", C.c_double)]


class AvnColliderColumns(C.Structure):
    _fields_ = [("count", C.c_uint32), ("_pad", C.c_uint32)] + [
        (n, _vp) for n in ("shape", "dims", "position", "rotation", "linear_velocity", "angular_velocity", "collision_margin", "speculative_margin",
                           "aabb_min", "aabb_max")]


class AvnTimings(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("h2d_ms", "prepare_ms", "substep_loop_ms", "finalize_ms", "d2h_ms", "broad_phase_ms", "total_ms")] + [
        (n, C.c_uint32) for n in ("kernel_launches", "contact_constraint_count", "joint_levels", "active_colors", "launch_mode")]


class AvianError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"avian_b200 error {status}: {message}")
        self.status = status


def _ptr(a):
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"], "column must be C-contiguous"
    return a.ctypes.data


def default_step_params(dt: float = 1.0 / 60.0, substeps: int = 6, gravity=(0.0, -9.81, 0.0), scalar=np.float32, **kw) -> AvnStepParams:
    """SolverConfig / Gravity / SubstepCount defaults of the reference (solver/plugin.rs:291-302,
    integrator/mod.rs:158-162, solver/schedule.rs:187-191).  dt, h are derived like the reference derives them:
    Duration arithmetic in integer nanoseconds (solver/schedule.rs:195-200, SURVEY H9)."""
    p = AvnStepParams()
    dt_ns = round(dt * 1e9)                       # Duration::from_secs_f64 rounds to the nearest ns
    h_ns = round(dt_ns / 1e9 / substeps * 1e9)    # Duration::div_f64 = from_secs_f64(as_secs_f64() / rhs)
    p.dt = dt_ns / 1e9
    p.h = h_ns / 1e9
    p.substeps = substeps
    p.restitution_iterations = 1
    p.gravity[0], p.gravity[1], p.gravity[2] = gravity
    p.contact_damping_ratio = 10.0
    p.contact_frequency_factor = 1.5
    p.max_overlap_solve_speed = 4.0
    p.warm_start_coefficient = 1.0
    p.restitution_threshold = 1.0
    p.length_unit = 1.0
    p.match_contacts = 1
    p.solver_iterations = 1
    for k, v in kw.items():
        setattr(p, k, v)
    return p


@dataclass
class Bodies:
    """Host columns of the rigid bodies (numpy, dtype = scalar type).  Mirrors AvnBodyColumns."""
    kind: np.ndarray
    position: np.ndarray
    rotation: np.ndarray
    linear_velocity: np.ndarray
    angular_velocity: np.ndarray
    inverse_mass: np.ndarray
    inverse_inertia_local: np.ndarray
    center_of_mass: np.ndarray | None = None
    locked_axes: np.ndarray | None = None
    dominance: np.ndarray | None = None
    linear_damping: np.ndarray | None = None
    angular_damping: np.ndarray | None = None
    gravity_scale: np.ndarray | None = None
    linear_acceleration: np.ndarray | None = None
    angular_acceleration: np.ndarray | None = None
    max_linear_speed: np.ndarray | None = None
    max_angular_speed: np.ndarray | None = None
    integration_flags: np.ndarray | None = None

    @property
    def count(self) -> int:
        return int(self.position.shape[0])

    def as_struct(self) -> AvnBodyColumns:
        s = AvnBodyColumns()
        s.count = self.count
        for name, _ in AvnBodyColumns._fields_[2:]:
            setattr(s, name, _ptr(getattr(self, name)))
        return s

    def copy(self) -> "Bodies":
        return Bodies(**{k: (None if v is None else v.copy()) for k, v in self.__dict__.items()})


@dataclass
class Manifolds:
    color_offsets: np.ndarray          # uint32[25]
    body1: np.ndarray                  # int32[M]
    body2: np.ndarray
    normal: np.ndarray                 # [M,3]
    friction: np.ndarray
    restitution: np.ndarray
    point_offsets: np.ndarray          # uint32[M+1]
    anchor1: np.ndarray                # [P,3]
    anchor2: np.ndarray
    penetration: np.ndarray
    normal_speed: np.ndarray
    warm_start_normal_impulse: np.ndarray
    warm_start_tangent_impulse: np.ndarray   # [P,2]
    normal_impulse: np.ndarray
    tangent_velocity: np.ndarray | None = None

    @property
    def count(self) -> int:
        return int(self.body1.shape[0])

    def as_struct(self) -> AvnManifoldColumns:
        s = AvnManifoldColumns()
        s.count = self.count
        s.point_count = int(self.penetration.shape[0])
        for i in range(GRAPH_COLOR_COUNT + 1):
            s.color_offsets[i] = int(self.color_offsets[i])
        for name, _ in AvnManifoldColumns._fields_[3:]:
            setattr(s, name, _ptr(getattr(self, name)))
        return s

    def copy(self) -> "Manifolds":
        return Manifolds(**{k: (None if v is None else v.copy()) for k, v in self.__dict__.items()})


@dataclass
class Joints:
    """One typed joint array (AvnJointColumns)."""
    body1: np.ndarray
    body2: np.ndarray
    local_anchor1: np.ndarray
    local_anchor2: np.ndarray
    local_basis1: np.ndarray | None = None
    local_basis2: np.ndarray | None = None
    axis: np.ndarray | None = None
    limit_enabled: np.ndarray | None = None
    limit_min: np.ndarray | None = None
    limit_max: np.ndarray | None = None
    limit2_min: np.ndarray | None = None
    limit2_max: np.ndarray | None = None
    compliance0: np.ndarray | None = None
    compliance1: np.ndarray | None = None
    compliance2: np.ndarray | None = None
    damping_enabled: np.ndarray | None = None
    damping_linear: np.ndarray | None = None
    damping_angular: np.ndarray | None = None
    force: np.ndarray | None = None
    torque: np.ndarray | None = None

    @property
    def count(self) -> int:
        return int(self.body1.shape[0])

    def fill(self, s: AvnJointColumns) -> None:
        s.count = self.count
        for name, _ in AvnJointColumns._fields_[2:]:
            setattr(s, name, _ptr(getattr(self, name)))

    def copy(self) -> "Joints":
        return Joints(**{k: (None if v is None else v.copy()) for k, v in self.__dict__.items()})


@dataclass
class JointSet:
    types: dict = field(default_factory=dict)   # AvnJointType -> Joints

    def as_struct(self) -> AvnJointSet:
        s = AvnJointSet()
        for t, j in self.types.items():
            j.fill(s.types[t])
        return s

    def copy(self) -> "JointSet":
        return JointSet({t: j.copy() for t, j in self.types.items()})

    @property
    def count(self) -> int:
        return sum(j.count for j in self.types.values())


@dataclass
class Aabbs:
    collider: np.ndarray     # uint32[C]
    body: np.ndarray         # uint32[C]
    aabb_min: np.ndarray     # [C,3]
    aabb_max: np.ndarray
    flags: np.ndarray        # uint8[C]
    memberships: np.ndarray | None = None
    filters: np.ndarray | None = None
    order_out: np.ndarray | None = None
    existing_pairs: np.ndarray | None = None          # uint64
    joint_disabled_body_pairs: np.ndarray | None = None
    retained_count: int | None = None                 # out: entries of order_out (intervals with a non-finite AABB are dropped)

    def as_struct(self) -> AvnAabbColumns:
        s = AvnAabbColumns()
        s.count = int(self.collider.shape[0])
        for name in ("collider", "body", "aabb_min", "aabb_max", "memberships", "filters", "flags", "order_out"):
            setattr(s, name, _ptr(getattr(self, name)))
        s.existing_pairs = _ptr(self.existing_pairs)
        s.existing_pair_count = 0 if self.existing_pairs is None else int(self.existing_pairs.shape[0])
        s.joint_disabled_body_pairs = _ptr(self.joint_disabled_body_pairs)
        s.joint_disabled_pair_count = 0 if self.joint_disabled_body_pairs is None else int(self.joint_disabled_body_pairs.shape[0])
        return s


@dataclass
class PairList:
    collider1: np.ndarray
    collider2: np.ndarray
    body1: np.ndarray
    body2: np.ndarray
    flags: np.ndarray
    count: int = 0

    @staticmethod
    def empty(capacity: int) -> "PairList":
        u = lambda: np.zeros(capacity, dtype=np.uint32)
        return PairList(u(), u(), u(), u(), np.zeros(capacity, dtype=np.uint8))

    def as_struct(self) -> AvnPairList:
        s = AvnPairList()
        s.capacity = int(self.collider1.shape[0])
        for name in ("collider1", "collider2", "body1", "body2", "flags"):
            setattr(s, name, _ptr(getattr(self, name)))
        return s

    def trimmed(self) -> "PairList":
        n = self.count
        return PairList(self.collider1[:n], self.collider2[:n], self.body1[:n], self.body2[:n], self.flags[:n], n)


class AvnNarrowParams(C.Structure):
    _fields_ = [("dt", C.c_double), ("contact_tolerance", C.c_double)]


class AvnContactGraphConfig(C.Structure):
    _fields_ = [("body_count", C.c_uint32), ("collider_count", C.c_uint32), ("body_kind", _vp), ("friction", _vp), ("restitution", _vp)]


class AvnContactStep(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("rows_high_water", "rows_live", "pairs_added", "pairs_removed", "started_touching", "stopped_touching",
                                         "manifold_count", "colouring_rounds", "any_restitution", "_pad")] + [("color_offsets", C.c_uint32 * (GRAPH_COLOR_COUNT + 1))]


CONTACTS_TAKE_BROADPHASE_PAIRS, CONTACTS_SHAPES_UNCHANGED = 1, 2
BODIES_STATIC_UNCHANGED = 1


class AvnIslandsConfig(C.Structure):
    _fields_ = [("body_count", C.c_uint32), ("joint_count", C.c_uint32), ("body_kind", _vp), ("sleep_threshold_linear", _vp), ("sleep_threshold_angular", _vp),
                ("sleeping_disabled", _vp), ("joint_body1", _vp), ("joint_body2", _vp), ("time_to_sleep", C.c_float), ("length_unit", C.c_float)]


class AvnIslandsStep(C.Structure):
    _fields_ = [("delta_secs", C.c_float), ("_pad", C.c_uint32), ("linear_velocity", _vp), ("angular_velocity", _vp), ("wake", _vp), ("island", _vp),
                ("sleeping", _vp), ("sleep_timer", _vp)] + [(n, C.c_uint32) for n in ("island_count", "sleeping_islands", "islands_put_to_sleep", "islands_woken",
                                                                                     "split_bodies", "merges")]


class AvnIslandsWake(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("islands_woken", "rows_woken", "rows_asleep", "bodies_asleep", "manifold_count", "colouring_rounds")] + [
        ("color_offsets", C.c_uint32 * (GRAPH_COLOR_COUNT + 1))]


class AvnNarrowInput(C.Structure):
    _fields_ = [("pair_count", C.c_uint32), ("collider_count", C.c_uint32), ("body_count", C.c_uint32), ("_pad", C.c_uint32)] + [
        (n, _vp) for n in ("collider1", "collider2", "body1", "body2", "shape", "dims", "position", "rotation", "linear_velocity", "angular_velocity",
                           "aabb_min", "aabb_max")]


class AvnBodyFrames(C.Structure):
    _fields_ = [("body_count", C.c_uint32), ("_pad", C.c_uint32)] + [(n, _vp) for n in ("position", "rotation", "center_of_mass")]


class AvnConvexHulls(C.Structure):
    _fields_ = [("hull_count", C.c_uint32), ("_pad", C.c_uint32)] + [(n, _vp) for n in ("vertex_offsets", "vertices", "face_offsets", "loop_offsets", "loop")]


class AvnRawManifolds(C.Structure):
    _fields_ = [(n, _vp) for n in ("point_count", "disjoint", "normal", "anchor1", "anchor2", "penetration", "normal_speed")]


class AvnBoundary(C.Structure):
    _fields_ = [("count", C.c_uint32), ("record_count", C.c_uint32), ("rank", C.c_uint32), ("world", C.c_uint32),
                ("body", _vp), ("source", _vp), ("owner_rank", _vp)]


class AvnQueryColliders(C.Structure):
    _fields_ = [("count", C.c_uint32), ("_pad", C.c_uint32)] + [(n, _vp) for n in ("shape", "dims", "position", "rotation", "memberships")]


class AvnRayBatch(C.Structure):
    _fields_ = [("count", C.c_uint32), ("exclude_count", C.c_uint32)] + [
        (n, _vp) for n in ("origin", "direction", "max_distance", "solid", "max_hits", "mask", "exclude_offsets", "exclude")]


class AvnRayClosest(C.Structure):
    _fields_ = [(n, _vp) for n in ("collider", "distance", "normal")]


class AvnHitList(C.Structure):
    _fields_ = [("capacity", C.c_uint64), ("count", C.c_uint64)] + [(n, _vp) for n in ("offsets", "collider", "distance", "normal")]


class AvnShapeBatch(C.Structure):
    _fields_ = [("count", C.c_uint32), ("exclude_count", C.c_uint32)] + [
        (n, _vp) for n in ("shape", "dims", "position", "rotation", "direction", "max_distance", "target_distance", "flags", "max_hits", "mask",
                           "exclude_offsets", "exclude")]


class AvnPointBatch(C.Structure):
    _fields_ = [("count", C.c_uint32), ("exclude_count", C.c_uint32)] + [(n, _vp) for n in ("point", "solid", "mask", "exclude_offsets", "exclude")]


class AvnShapeClosest(C.Structure):
    _fields_ = [(n, _vp) for n in ("collider", "distance", "point1", "point2", "normal1", "normal2")]


class AvnShapeHitList(C.Structure):
    _fields_ = [("capacity", C.c_uint64), ("count", C.c_uint64)] + [
        (n, _vp) for n in ("offsets", "collider", "distance", "point1", "point2", "normal1", "normal2")]


class AvnPointProjection(C.Structure):
    _fields_ = [(n, _vp) for n in ("collider", "point", "is_inside")]


class AvnMoveConfig(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("delta_time", "length_unit", "skin_width", "max_depenetration_error", "penetration_rejection_threshold",
                                          "plane_similarity_dot_threshold")] + [
        (n, C.c_uint32) for n in ("move_and_slide_iterations", "depenetration_iterations", "max_planes", "collider_count")] + [("ignored", _vp)]


class AvnMoveBatch(C.Structure):
    _fields_ = [("count", C.c_uint32), ("exclude_count", C.c_uint32)] + [
        (n, _vp) for n in ("shape", "dims", "position", "rotation", "velocity", "mask", "exclude_offsets", "exclude", "plane_offsets", "planes")]


class AvnMoveResult(C.Structure):
    _fields_ = [(n, _vp) for n in ("position", "velocity", "hit_collider", "hit_distance", "hit_toi", "hit_point", "hit_normal")] + [
        ("kernel_ms", C.c_float), ("_pad", C.c_uint32)]


class AvnCollisionEvents(C.Structure):
    _fields_ = [("capacity", C.c_uint64), ("count", C.c_uint64)] + [(n, _vp) for n in ("collider1", "collider2", "body1", "body2", "flags")]


class AvnContactReport(C.Structure):
    _fields_ = [("capacity", C.c_uint64), ("count", C.c_uint64)] + [
        (n, _vp) for n in ("contact_id", "collider1", "collider2", "body1", "body2", "flags", "point_count", "normal", "total_normal_impulse",
                           "max_normal_impulse", "max_penetration")]


REPORT_EVENTS_ONLY = 0x1


class AvnCcdConfig(C.Structure):
    _fields_ = [("count", C.c_uint32), ("flags", C.c_uint32)] + [(n, _vp) for n in ("body", "collider", "mode", "include_dynamic", "linear_threshold",
                                                                                   "angular_threshold")] + [("prediction_distance", C.c_double)]


class AvnCcdResult(C.Structure):
    _fields_ = [(n, _vp) for n in ("min_toi", "hit_body", "hit_contact", "candidates", "hits")] + [("pass_ms", C.c_float), ("total_candidates", C.c_uint32)]


SWEEP_LINEAR, SWEEP_NON_LINEAR = 0, 1
CCD_CAPSULES = 0x1   # AvnCcdConfig.flags: capsule colliders take part in swept CCD
CCD_HULLS = 0x4      # AvnCcdConfig.flags: convex hull colliders take part in swept CCD


def ccd_config(body, collider, mode=None, include_dynamic=None, linear_threshold=None, angular_threshold=None,
               prediction_distance: float = float("inf"), flags: int = 0) -> tuple["AvnCcdConfig", tuple]:
    """An AvnCcdConfig over numpy copies of the columns (returned alongside: they must outlive the struct's use).  flags: CCD_CAPSULES and
    CCD_HULLS bits, or 0."""
    cols = (np.ascontiguousarray(body, dtype=np.int32), np.ascontiguousarray(collider, dtype=np.uint32),
            None if mode is None else np.ascontiguousarray(mode, dtype=np.uint8),
            None if include_dynamic is None else np.ascontiguousarray(include_dynamic, dtype=np.uint8),
            None if linear_threshold is None else np.ascontiguousarray(linear_threshold, dtype=np.float64),
            None if angular_threshold is None else np.ascontiguousarray(angular_threshold, dtype=np.float64))
    return AvnCcdConfig(int(cols[0].shape[0]), int(flags), *(_ptr(a) for a in cols), float(prediction_distance)), cols


QUERY_SHAPES_UNCHANGED = 1
MAX_HITS_ALL = 0xFFFFFFFF
CAST_IGNORE_ORIGIN_PENETRATION = 0x1
CAST_NO_CONTACT_ON_PENETRATION = 0x2


def bind_abi(lib: C.CDLL, prefix: str = "avn") -> None:
    """Declare argument/return types of every entry point of include/avian_b200.h on `lib`."""
    P = C.POINTER
    sig = {
        "create": ([P(AvnConfig), P(_vp)], C.c_int),
        "destroy": ([_vp], None),
        "last_error": ([_vp], C.c_char_p),
        "abi_version": ([], C.c_uint32),
        "alloc_pinned": ([_vp, C.c_size_t, P(_vp)], C.c_int),
        "free_pinned": ([_vp, _vp], C.c_int),
        "solver_step": ([_vp, P(AvnStepParams), P(AvnBodyColumns), P(AvnManifoldColumns), P(AvnJointSet)], C.c_int),
        "solver_upload": ([_vp, P(AvnStepParams), P(AvnBodyColumns), P(AvnManifoldColumns), P(AvnJointSet)], C.c_int),
        "solver_run": ([_vp], C.c_int),
        "solver_download": ([_vp], C.c_int),
        "broadphase": ([_vp, P(AvnAabbColumns), P(AvnPairList)], C.c_int),
        "broadphase_upload": ([_vp, P(AvnAabbColumns)], C.c_int),
        "broadphase_run": ([_vp], C.c_int),
        "broadphase_download": ([_vp, P(AvnPairList)], C.c_int),
        "get_timings": ([_vp, P(AvnTimings)], C.c_int),
        "joint_levels": ([P(AvnBodyColumns), P(AvnJointSet), _vp, P(C.c_uint32)], C.c_int),
        "update_aabbs": ([_vp, P(AvnAabbParams), P(AvnColliderColumns)], C.c_int),
        "solver_run_range": ([_vp, C.c_uint32, C.c_uint32, C.c_uint32], C.c_int),
        "solver_set_boundary": ([_vp, P(AvnBoundary)], C.c_int),
        "solver_boundary_snapshot": ([_vp], C.c_int),
        "solver_boundary_pack": ([_vp, _vp], C.c_int),
        "solver_boundary_apply": ([_vp, _vp], C.c_int),
        "solver_needs_restitution": ([_vp, P(C.c_int)], C.c_int),
        "get_stream": ([_vp, P(_vp)], C.c_int),
        "solver_step_partitioned": ([_vp], C.c_int),
        "comm_unique_id": ([_vp, _vp], C.c_int),
        "comm_init": ([_vp, C.c_uint32, C.c_uint32, _vp], C.c_int),
        "comm_destroy": ([_vp], C.c_int),
        "comm_all_gather": ([_vp, _vp, _vp, C.c_size_t], C.c_int),
        "narrow_phase": ([_vp, P(AvnNarrowParams), P(AvnNarrowInput), P(AvnRawManifolds)], C.c_int),
        "contacts_download_impulses": ([_vp, C.c_uint32, _vp, _vp, _vp], C.c_int),
        "contacts_configure": ([_vp, P(AvnContactGraphConfig)], C.c_int),
        "contacts_step": ([_vp, P(AvnNarrowParams), P(AvnNarrowInput), C.c_uint32, C.c_double, C.c_uint32, P(AvnContactStep)], C.c_int),
        "contacts_set_body_frames": ([_vp, P(AvnBodyFrames)], C.c_int),
        "set_convex_hulls": ([_vp, P(AvnConvexHulls)], C.c_int),
        "solver_upload_resident": ([_vp, P(AvnStepParams), P(AvnBodyColumns), P(AvnJointSet)], C.c_int),
        "broadphase_download_order": ([_vp, P(C.c_uint64)], C.c_int),
        "contacts_download_graph": ([_vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp, _vp], C.c_int),
        "solver_prefetch_bodies": ([_vp, P(AvnBodyColumns), C.c_uint32], C.c_int),
        "islands_configure": ([_vp, P(AvnIslandsConfig)], C.c_int),
        "islands_step": ([_vp, P(AvnIslandsStep)], C.c_int),
        "islands_apply": ([_vp, C.c_uint32], C.c_int),
        "islands_wake": ([_vp, _vp, P(AvnIslandsWake)], C.c_int),
        "contacts_download_sleeping": ([_vp, C.c_uint32, _vp, C.c_uint32, _vp], C.c_int),
        "query_update": ([_vp, P(AvnQueryColliders), C.c_uint32], C.c_int),
        "query_cast_ray": ([_vp, P(AvnRayBatch), P(AvnRayClosest)], C.c_int),
        "query_ray_hits": ([_vp, P(AvnRayBatch), P(AvnHitList)], C.c_int),
        "query_aabb_intersections": ([_vp, C.c_uint32, _vp, _vp, P(AvnHitList)], C.c_int),
        "query_cast_shape": ([_vp, P(AvnShapeBatch), P(AvnShapeClosest)], C.c_int),
        "query_shape_hits": ([_vp, P(AvnShapeBatch), P(AvnShapeHitList)], C.c_int),
        "query_project_point": ([_vp, P(AvnPointBatch), P(AvnPointProjection)], C.c_int),
        "query_point_intersections": ([_vp, P(AvnPointBatch), P(AvnHitList)], C.c_int),
        "query_shape_intersections": ([_vp, P(AvnShapeBatch), P(AvnHitList)], C.c_int),
        "ccd_configure": ([_vp, P(AvnCcdConfig)], C.c_int),
        "ccd_download": ([_vp, P(AvnCcdResult)], C.c_int),
        "contacts_set_sensors": ([_vp, C.c_uint32, _vp], C.c_int),
        "contacts_remove_colliders": ([_vp, C.c_uint32, _vp], C.c_int),
        "contacts_events": ([_vp, P(AvnCollisionEvents), P(AvnCollisionEvents)], C.c_int),
        "contacts_report": ([_vp, C.c_uint32, P(AvnContactReport)], C.c_int),
        "move_and_slide": ([_vp, P(AvnMoveConfig), P(AvnMoveBatch), P(AvnMoveResult)], C.c_int),
    }
    for name, (argtypes, restype) in sig.items():
        fn = getattr(lib, f"{prefix}_{name}")
        fn.argtypes = argtypes
        fn.restype = restype


ABI_SYMBOLS = [
    "avn_create", "avn_destroy", "avn_last_error", "avn_abi_version", "avn_alloc_pinned", "avn_free_pinned", "avn_solver_step",
    "avn_solver_upload", "avn_solver_run", "avn_solver_download", "avn_broadphase", "avn_broadphase_upload", "avn_broadphase_run",
    "avn_broadphase_download", "avn_get_timings", "avn_joint_levels", "avn_update_aabbs", "avn_solver_run_range", "avn_solver_set_boundary",
    "avn_solver_boundary_snapshot", "avn_solver_boundary_pack", "avn_solver_boundary_apply", "avn_solver_needs_restitution", "avn_get_stream",
    "avn_solver_step_partitioned", "avn_comm_unique_id", "avn_comm_init", "avn_comm_destroy", "avn_comm_all_gather", "avn_narrow_phase", "avn_contacts_download_impulses",
    "avn_contacts_configure", "avn_contacts_step", "avn_solver_upload_resident", "avn_broadphase_download_order", "avn_contacts_download_graph",
    "avn_solver_prefetch_bodies", "avn_islands_configure", "avn_islands_step", "avn_query_update", "avn_query_cast_ray", "avn_query_ray_hits",
    "avn_query_aabb_intersections", "avn_query_cast_shape", "avn_query_shape_hits", "avn_query_project_point", "avn_query_point_intersections",
    "avn_query_shape_intersections", "avn_ccd_configure", "avn_ccd_download", "avn_contacts_set_sensors", "avn_contacts_remove_colliders",
    "avn_contacts_events", "avn_contacts_report", "avn_islands_apply", "avn_islands_wake", "avn_contacts_download_sleeping",
    "avn_move_and_slide", "avn_contacts_set_body_frames", "avn_set_convex_hulls"]

RUN_PREPARE, RUN_RESTITUTION, RUN_FINALIZE = 1, 2, 4
COMM_ID_BYTES = 128
BOUNDARY_RECORD_SCALARS = 16


SHAPE_CONVEX_HULL = 3
HULL_MAX_VERTICES, HULL_MAX_FACES, HULL_MAX_FACE_VERTICES = 64, 128, 32


@dataclass
class ConvexHulls:
    """A convex hull table (AvnConvexHulls): what parry's ConvexPolyhedron holds for each hull, in CSR columns.  vertices [V,3] hull-local and
    already scaled; each face a loop of hull-local vertex indices, counter-clockwise seen from outside.  A collider with shape
    SHAPE_CONVEX_HULL names its hull by index in dims[0]."""
    vertex_offsets: np.ndarray   # uint32 [H+1]
    vertices: np.ndarray         # float64 [V,3]
    face_offsets: np.ndarray     # uint32 [H+1]
    loop_offsets: np.ndarray     # uint32 [F+1]
    loop: np.ndarray             # uint32 [L]

    @property
    def count(self) -> int:
        return int(self.vertex_offsets.shape[0]) - 1

    @staticmethod
    def from_polyhedra(hulls) -> "ConvexHulls":
        """hulls: a list of (vertices [v,3], faces: list of vertex-index loops)."""
        vo, fo, lo, verts, loop = [0], [0], [0], [], []
        for v, faces in hulls:
            v = np.asarray(v, dtype=np.float64).reshape(-1, 3)
            verts.append(v)
            vo.append(vo[-1] + v.shape[0])
            for f in faces:
                loop.extend(int(i) for i in f)
                lo.append(len(loop))
            fo.append(fo[-1] + len(faces))
        u32 = lambda a: np.ascontiguousarray(a, dtype=np.uint32)
        return ConvexHulls(u32(vo), np.ascontiguousarray(np.concatenate(verts) if verts else np.zeros((0, 3))), u32(fo), u32(lo), u32(loop))

    def polyhedron(self, h: int):
        """(vertices, faces) of hull h"""
        v = self.vertices[self.vertex_offsets[h]:self.vertex_offsets[h + 1]]
        faces = [self.loop[self.loop_offsets[f]:self.loop_offsets[f + 1]] for f in range(self.face_offsets[h], self.face_offsets[h + 1])]
        return v, faces

    def as_struct(self, scalar) -> tuple["AvnConvexHulls", tuple]:
        """the ABI struct with the vertices in the column scalar, and the arrays it points into (keep them alive while it is used)"""
        keep = (np.ascontiguousarray(self.vertex_offsets, dtype=np.uint32), np.ascontiguousarray(self.vertices, dtype=scalar),
                np.ascontiguousarray(self.face_offsets, dtype=np.uint32), np.ascontiguousarray(self.loop_offsets, dtype=np.uint32),
                np.ascontiguousarray(self.loop, dtype=np.uint32))
        return AvnConvexHulls(self.count, 0, *(_ptr(a) for a in keep)), keep


@dataclass
class Colliders:
    """Collider columns of avn_update_aabbs (AvnColliderColumns)."""
    shape: np.ndarray            # uint8[C]
    dims: np.ndarray             # [C,3]
    position: np.ndarray
    rotation: np.ndarray
    linear_velocity: np.ndarray | None = None
    angular_velocity: np.ndarray | None = None
    collision_margin: np.ndarray | None = None
    speculative_margin: np.ndarray | None = None
    aabb_min: np.ndarray | None = None
    aabb_max: np.ndarray | None = None

    def as_struct(self) -> "AvnColliderColumns":
        n = int(self.position.shape[0])
        if self.aabb_min is None:
            self.aabb_min = np.zeros((n, 3), dtype=self.position.dtype)
            self.aabb_max = np.zeros((n, 3), dtype=self.position.dtype)
        s = AvnColliderColumns()
        s.count = n
        for name, _ in AvnColliderColumns._fields_[2:]:
            setattr(s, name, _ptr(getattr(self, name)))
        return s


@dataclass
class QueryColliders:
    """Collider columns of avn_query_update (AvnQueryColliders); collider index = row."""
    shape: np.ndarray                    # uint8[C] SHAPE_CUBOID / SHAPE_SPHERE
    dims: np.ndarray                     # [C,3] half extents / radius in [0]
    position: np.ndarray                 # [C,3]
    rotation: np.ndarray                 # [C,4] (x, y, z, w)
    memberships: np.ndarray | None = None   # uint32[C] CollisionLayers::memberships (None = 1)

    def as_struct(self, scalar) -> tuple["AvnQueryColliders", list]:
        """The struct and the arrays it points into (keep them alive for the call)."""
        dt = np.dtype(scalar)
        keep = [np.ascontiguousarray(self.shape, dtype=np.uint8), np.ascontiguousarray(self.dims, dtype=dt).reshape(-1, 3),
                np.ascontiguousarray(self.position, dtype=dt).reshape(-1, 3), np.ascontiguousarray(self.rotation, dtype=dt).reshape(-1, 4),
                None if self.memberships is None else np.ascontiguousarray(self.memberships, dtype=np.uint32)]
        return AvnQueryColliders(int(keep[2].shape[0]), 0, *(_ptr(a) for a in keep)), keep


@dataclass
class Rays:
    """A batch of rays (AvnRayBatch).  exclude: per ray an iterable of collider indices it ignores (SpatialQueryFilter::excluded_entities,
    RayCaster::ignore_self), or None."""
    origin: np.ndarray                   # [n,3]
    direction: np.ndarray                # [n,3] unit
    max_distance: np.ndarray             # [n]
    solid: np.ndarray | None = None      # bool/uint8[n] (None = all solid)
    max_hits: np.ndarray | None = None   # uint32[n] (None = all; MAX_HITS_ALL = all)
    mask: np.ndarray | None = None       # uint32[n] SpatialQueryFilter::mask (None = all layers)
    exclude: list | None = None

    @property
    def count(self) -> int:
        return int(np.asarray(self.origin).reshape(-1, 3).shape[0])

    def as_struct(self, scalar) -> tuple["AvnRayBatch", list]:
        dt, n = np.dtype(scalar), self.count
        o = np.ascontiguousarray(self.origin, dtype=dt).reshape(-1, 3)
        d = np.ascontiguousarray(self.direction, dtype=dt).reshape(-1, 3)
        md = np.ascontiguousarray(np.broadcast_to(np.asarray(self.max_distance, dtype=dt), (n,)))
        opt = lambda a, t: None if a is None else np.ascontiguousarray(a, dtype=t)
        solid, mh, mask = opt(self.solid, np.uint8), opt(self.max_hits, np.uint32), opt(self.mask, np.uint32)
        xoff = xs = None
        if self.exclude is not None:
            lists = [np.asarray(list(e), dtype=np.uint32) for e in self.exclude]
            xoff = np.zeros(n + 1, dtype=np.uint32)
            xoff[1:] = np.cumsum([len(e) for e in lists])
            xs = np.ascontiguousarray(np.concatenate(lists) if lists else np.zeros(0, dtype=np.uint32), dtype=np.uint32)
        keep = [o, d, md, solid, mh, mask, xoff, xs]
        st = AvnRayBatch(n, 0 if xs is None else int(xs.shape[0]), *(_ptr(a) if a is None or a.size else None for a in keep))
        if xoff is not None:
            st.exclude_offsets = xoff.ctypes.data
            st.exclude = xs.ctypes.data if xs.size else None
        return st, keep


def _exclusion_csr(exclude, n: int):
    """per query an iterable of excluded collider indices -> (offsets[n+1], indices), or (None, None)"""
    if exclude is None:
        return None, None
    lists = [np.asarray(list(e), dtype=np.uint32) for e in exclude]
    xoff = np.zeros(n + 1, dtype=np.uint32)
    xoff[1:] = np.cumsum([len(e) for e in lists])
    xs = np.ascontiguousarray(np.concatenate(lists) if lists else np.zeros(0, dtype=np.uint32), dtype=np.uint32)
    return xoff, xs


@dataclass
class ShapeQueries:
    """A batch of query shapes (AvnShapeBatch): cuboids / spheres with a pose, for shape casts (direction, max_distance, flags, max_hits)
    and shape intersections (which ignore the cast columns).  exclude: per shape an iterable of collider indices it ignores, or None."""
    shape: np.ndarray                        # uint8[n] SHAPE_CUBOID / SHAPE_SPHERE
    dims: np.ndarray                         # [n,3] half extents / radius in [0]
    position: np.ndarray                     # [n,3]
    rotation: np.ndarray                     # [n,4] (x, y, z, w)
    direction: np.ndarray | None = None      # [n,3] casts
    max_distance: np.ndarray | None = None   # [n] casts
    target_distance: np.ndarray | None = None   # [n] casts: must be 0 (None = 0)
    flags: np.ndarray | None = None          # uint32[n] CAST_* (None = 0)
    max_hits: np.ndarray | None = None       # uint32[n] shape_hits (None = all)
    mask: np.ndarray | None = None           # uint32[n] (None = all layers)
    exclude: list | None = None

    @property
    def count(self) -> int:
        return int(np.asarray(self.position).reshape(-1, 3).shape[0])

    def as_struct(self, scalar) -> tuple["AvnShapeBatch", list]:
        dt, n = np.dtype(scalar), self.count
        col = lambda a, w: None if a is None else np.ascontiguousarray(a, dtype=dt).reshape(-1, w)
        per = lambda a: None if a is None else np.ascontiguousarray(np.broadcast_to(np.asarray(a, dtype=dt), (n,)))
        opt = lambda a, t: None if a is None else np.ascontiguousarray(a, dtype=t)
        xoff, xs = _exclusion_csr(self.exclude, n)
        keep = [opt(self.shape, np.uint8), col(self.dims, 3), col(self.position, 3), col(self.rotation, 4), col(self.direction, 3),
                per(self.max_distance), per(self.target_distance), opt(self.flags, np.uint32), opt(self.max_hits, np.uint32),
                opt(self.mask, np.uint32), xoff, xs]
        st = AvnShapeBatch(n, 0 if xs is None else int(xs.shape[0]), *(_ptr(a) if a is None or a.size else None for a in keep))
        if xoff is not None:
            st.exclude_offsets = xoff.ctypes.data
            st.exclude = xs.ctypes.data if xs.size else None
        return st, keep


@dataclass
class Points:
    """A batch of query points (AvnPointBatch).  solid: project_point only."""
    point: np.ndarray                    # [n,3]
    solid: np.ndarray | None = None      # bool/uint8[n] (None = all solid)
    mask: np.ndarray | None = None       # uint32[n] (None = all layers)
    exclude: list | None = None

    @property
    def count(self) -> int:
        return int(np.asarray(self.point).reshape(-1, 3).shape[0])

    def as_struct(self, scalar) -> tuple["AvnPointBatch", list]:
        dt, n = np.dtype(scalar), self.count
        opt = lambda a, t: None if a is None else np.ascontiguousarray(a, dtype=t)
        xoff, xs = _exclusion_csr(self.exclude, n)
        keep = [np.ascontiguousarray(self.point, dtype=dt).reshape(-1, 3), opt(self.solid, np.uint8), opt(self.mask, np.uint32), xoff, xs]
        st = AvnPointBatch(n, 0 if xs is None else int(xs.shape[0]), *(_ptr(a) if a is None or a.size else None for a in keep))
        if xoff is not None:
            st.exclude_offsets = xoff.ctypes.data
            st.exclude = xs.ctypes.data if xs.size else None
        return st, keep


MOVE_MAX_PLANES = 32
COS_5_DEGREES = 0.99619469809


@dataclass
class MoveConfig:
    """MoveAndSlideConfig (AvnMoveConfig), the reference's defaults.  ignored: uint8[C] per collider of the tree, nonzero = not an obstacle
    (sensors, colliders without a body); None = every collider is one."""
    delta_time: float = 1.0 / 60.0
    length_unit: float = 1.0
    skin_width: float = 0.01
    max_depenetration_error: float = 0.0001
    penetration_rejection_threshold: float = 0.5
    plane_similarity_dot_threshold: float = COS_5_DEGREES
    move_and_slide_iterations: int = 4
    depenetration_iterations: int = 16
    max_planes: int = 20
    ignored: np.ndarray | None = None
    collider_count: int | None = None      # None = len(ignored)

    def as_struct(self) -> tuple["AvnMoveConfig", list]:
        ig = None if self.ignored is None else np.ascontiguousarray(self.ignored, dtype=np.uint8)
        cc = self.collider_count if self.collider_count is not None else (0 if ig is None else int(ig.shape[0]))
        st = AvnMoveConfig(float(self.delta_time), float(self.length_unit), float(self.skin_width), float(self.max_depenetration_error),
                           float(self.penetration_rejection_threshold), float(self.plane_similarity_dot_threshold), int(self.move_and_slide_iterations),
                           int(self.depenetration_iterations), int(self.max_planes), int(cc), _ptr(ig))
        return st, [ig]


@dataclass
class MoveBatch:
    """Characters of one avn_move_and_slide call (AvnMoveBatch).  exclude: per character an iterable of collider indices it ignores (its own
    collider, as the reference's docs tell users to); planes: per character an array [k,3] of initial planes (MoveAndSlideConfig::planes),
    or None."""
    shape: np.ndarray                        # uint8[n] SHAPE_CUBOID / SHAPE_SPHERE
    dims: np.ndarray                         # [n,3] half extents / radius in [0]
    position: np.ndarray                     # [n,3]
    rotation: np.ndarray                     # [n,4] (x, y, z, w)
    velocity: np.ndarray                     # [n,3] desired velocity
    mask: np.ndarray | None = None           # uint32[n] (None = all layers)
    exclude: list | None = None
    planes: list | None = None

    @property
    def count(self) -> int:
        return int(np.asarray(self.position).reshape(-1, 3).shape[0])

    def as_struct(self, scalar) -> tuple["AvnMoveBatch", list]:
        dt, n = np.dtype(scalar), self.count
        col = lambda a, w: np.ascontiguousarray(a, dtype=dt).reshape(-1, w)
        opt = lambda a, t: None if a is None else np.ascontiguousarray(a, dtype=t)
        xoff, xs = _exclusion_csr(self.exclude, n)
        poff = pl = None
        if self.planes is not None:
            lists = [np.zeros((0, 3)) if p is None else np.asarray(p, dtype=np.float64).reshape(-1, 3) for p in self.planes]
            poff = np.zeros(n + 1, dtype=np.uint32)
            poff[1:] = np.cumsum([len(p) for p in lists])
            pl = np.ascontiguousarray(np.concatenate(lists) if lists else np.zeros((0, 3)), dtype=dt).reshape(-1, 3)
        keep = [opt(self.shape, np.uint8), col(self.dims, 3), col(self.position, 3), col(self.rotation, 4), col(self.velocity, 3),
                opt(self.mask, np.uint32), xoff, xs, poff, pl]
        st = AvnMoveBatch(n, 0 if xs is None else int(xs.shape[0]), *(_ptr(a) if a is None or a.size else None for a in keep))
        if xoff is not None:
            st.exclude_offsets = xoff.ctypes.data
            st.exclude = xs.ctypes.data if xs.size else None
        if poff is not None:
            st.plane_offsets = poff.ctypes.data
        return st, keep


MOVE_HIT_FIELDS = ("hit_collider", "hit_distance", "hit_toi", "hit_point", "hit_normal")


def move_result(n: int, iterations: int, scalar) -> tuple["AvnMoveResult", dict]:
    """An AvnMoveResult over fresh numpy arrays: position, velocity [n,3]; hit_collider, hit_distance, hit_toi [n,iterations];
    hit_point, hit_normal [n,iterations,3]."""
    it = int(iterations)
    out = {"position": np.zeros((n, 3), dtype=scalar), "velocity": np.zeros((n, 3), dtype=scalar), "hit_collider": np.zeros((n, it), dtype=np.int32),
           "hit_distance": np.zeros((n, it), dtype=scalar), "hit_toi": np.zeros((n, it), dtype=scalar),
           "hit_point": np.zeros((n, it, 3), dtype=scalar), "hit_normal": np.zeros((n, it, 3), dtype=scalar)}
    return AvnMoveResult(*(_ptr(out[k]) if out[k].size else None for k in ("position", "velocity") + MOVE_HIT_FIELDS), 0.0, 0), out


SHAPE_HIT_FIELDS = ("point1", "point2", "normal1", "normal2")


def shape_closest(n: int, scalar) -> tuple["AvnShapeClosest", dict]:
    out = {"collider": np.zeros(n, dtype=np.int32), "distance": np.zeros(n, dtype=scalar)}
    out.update({k: np.zeros((n, 3), dtype=scalar) for k in SHAPE_HIT_FIELDS})
    return AvnShapeClosest(*(_ptr(out[k]) for k in ("collider", "distance") + SHAPE_HIT_FIELDS)), out


def shape_hit_list(n: int, capacity: int, scalar) -> tuple["AvnShapeHitList", dict]:
    """An AvnShapeHitList over fresh numpy arrays (offsets[n+1], collider, distance, point1, point2, normal1, normal2)."""
    cap = max(int(capacity), 0)
    m = max(cap, 1)
    out = {"offsets": np.zeros(n + 1, dtype=np.uint64), "collider": np.zeros(m, dtype=np.uint32), "distance": np.zeros(m, dtype=scalar)}
    out.update({k: np.zeros((m, 3), dtype=scalar) for k in SHAPE_HIT_FIELDS})
    return AvnShapeHitList(cap, 0, *(_ptr(out[k]) for k in ("offsets", "collider", "distance") + SHAPE_HIT_FIELDS)), out


def point_projection(n: int, scalar) -> tuple["AvnPointProjection", dict]:
    out = {"collider": np.zeros(n, dtype=np.int32), "point": np.zeros((n, 3), dtype=scalar), "is_inside": np.zeros(n, dtype=np.uint8)}
    return AvnPointProjection(*(_ptr(out[k]) for k in ("collider", "point", "is_inside"))), out


def hit_list(n: int, capacity: int, scalar, ray: bool) -> tuple["AvnHitList", dict]:
    """An AvnHitList over fresh numpy arrays (offsets[n+1], collider, and for rays distance / normal)."""
    cap = max(int(capacity), 0)
    out = {"offsets": np.zeros(n + 1, dtype=np.uint64), "collider": np.zeros(max(cap, 1), dtype=np.uint32)}
    if ray:
        out["distance"] = np.zeros(max(cap, 1), dtype=scalar)
        out["normal"] = np.zeros((max(cap, 1), 3), dtype=scalar)
    return AvnHitList(cap, 0, _ptr(out["offsets"]), _ptr(out["collider"]), _ptr(out.get("distance")), _ptr(out.get("normal"))), out


def hit_list_result(h: "AvnHitList", out: dict) -> dict:
    total = int(h.count)
    return {k: (v if k == "offsets" else v[:total]) for k, v in out.items()}


EVENT_COLUMNS = (("collider1", np.uint32), ("collider2", np.uint32), ("body1", np.uint32), ("body2", np.uint32), ("flags", np.uint8))


def collision_events(capacity: int) -> tuple["AvnCollisionEvents", dict]:
    """An AvnCollisionEvents over fresh numpy arrays of `capacity` entries (returned alongside: they must outlive the struct's use)."""
    cap = max(int(capacity), 0)
    out = {k: np.zeros(max(cap, 1), dtype=d) for k, d in EVENT_COLUMNS}
    return AvnCollisionEvents(cap, 0, *(_ptr(out[k]) for k, _ in EVENT_COLUMNS)), out


def contact_report(capacity: int, scalar) -> tuple["AvnContactReport", dict]:
    """An AvnContactReport over fresh numpy arrays of `capacity` entries, scalars in `scalar` (returned alongside: they must outlive the
    struct's use)."""
    cap = max(int(capacity), 1)
    out = {k: np.zeros(cap, dtype=np.uint32) for k in ("contact_id", "collider1", "collider2", "body1", "body2")}
    out.update({"flags": np.zeros(cap, dtype=np.uint8), "point_count": np.zeros(cap, dtype=np.uint8), "normal": np.zeros((cap, 3), dtype=scalar)})
    out.update({k: np.zeros(cap, dtype=scalar) for k in ("total_normal_impulse", "max_normal_impulse", "max_penetration")})
    r = AvnContactReport(max(int(capacity), 0), 0, *(_ptr(out[n]) for n, _ in AvnContactReport._fields_[2:]))
    return r, out


def aabb_params(dt: float, contact_tolerance: float = 0.005, default_speculative_margin: float = float("inf")) -> "AvnAabbParams":
    """NarrowPhaseConfig defaults (narrow_phase/mod.rs:247-255) times PhysicsLengthUnit = 1."""
    return AvnAabbParams(dt, contact_tolerance, default_speculative_margin)


def joint_levels(bodies: "Bodies", joints: "JointSet"):
    """avn_joint_levels: (level per joint in the reference's global order, number of levels).  Host-only."""
    lib = load_library()
    b, j = bodies.as_struct(), joints.as_struct()
    out = np.zeros(joints.count, dtype=np.uint32)
    n = C.c_uint32(0)
    st = lib.avn_joint_levels(C.byref(b), C.byref(j), _ptr(out), C.byref(n))
    if st != OK:
        raise AvianError(st, lib.avn_last_error(None).decode())
    return out, int(n.value)

_lib = None


def load_library() -> C.CDLL:
    """Load (building if needed) libavian_b200.so.  Raises if it cannot be had: no fallback."""
    global _lib
    if _lib is None:
        path = _build.build_cuda()
        lib = C.CDLL(str(path))
        bind_abi(lib)
        _lib = lib
    return _lib


class Context:
    """An AvnContext: one CUDA device, one stream, persistent device buffers."""

    def __init__(self, device: int = 0, scalar=np.float32, flags: int = 0):
        self.lib = load_library()
        self.device = int(device)
        self.scalar = np.dtype(scalar)
        cfg = AvnConfig(self.lib.avn_abi_version(), device, 32 if self.scalar == np.float32 else 64, flags)
        h = _vp()
        st = self.lib.avn_create(C.byref(cfg), C.byref(h))
        if st != OK:
            raise AvianError(st, self.lib.avn_last_error(None).decode())
        self.handle = h
        self._pinned: list[int] = []
        self._keep = None

    def close(self) -> None:
        if getattr(self, "handle", None):
            for p in self._pinned:
                self.lib.avn_free_pinned(self.handle, _vp(p))
            self._pinned.clear()
            self.lib.avn_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _check(self, st: int) -> None:
        if st != OK:
            raise AvianError(st, self.lib.avn_last_error(self.handle).decode())

    def _check_list(self, st: int, h: "AvnHitList") -> None:
        """A CSR query's status: on AVN_ERR_CAPACITY the error carries the required count as .required"""
        if st == ERR_CAPACITY:
            e = AvianError(st, self.lib.avn_last_error(self.handle).decode())
            e.required = int(h.count)
            raise e
        self._check(st)

    def pinned(self, shape, dtype) -> np.ndarray:
        """A numpy array backed by page-locked memory from avn_alloc_pinned (lives as long as the context)."""
        dtype = np.dtype(dtype)
        n = int(np.prod(shape)) * dtype.itemsize
        p = _vp()
        self._check(self.lib.avn_alloc_pinned(self.handle, max(n, 1), C.byref(p)))
        self._pinned.append(p.value)
        buf = (C.c_byte * max(n, 1)).from_address(p.value)
        return np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)

    def pin_like(self, a: np.ndarray | None) -> np.ndarray | None:
        if a is None:
            return None
        out = self.pinned(a.shape, a.dtype)
        out[...] = a
        return out

    # ---- solver stage ------------------------------------------------------------------------------------
    def _solver_args(self, params, bodies: Bodies, manifolds: Manifolds | None, joints: JointSet | None):
        b = bodies.as_struct()
        m = manifolds.as_struct() if manifolds is not None and manifolds.count else None
        j = joints.as_struct() if joints is not None and joints.count else None
        self._keep = (params, bodies, manifolds, joints, b, m, j)
        return (C.byref(params), C.byref(b), C.byref(m) if m is not None else None, C.byref(j) if j is not None else None)

    def solver_step(self, params, bodies, manifolds=None, joints=None) -> None:
        self._check(self.lib.avn_solver_step(self.handle, *self._solver_args(params, bodies, manifolds, joints)))

    def solver_upload(self, params, bodies, manifolds=None, joints=None) -> None:
        self._check(self.lib.avn_solver_upload(self.handle, *self._solver_args(params, bodies, manifolds, joints)))

    def solver_run(self) -> None:
        self._check(self.lib.avn_solver_run(self.handle))

    def solver_download(self) -> None:
        self._check(self.lib.avn_solver_download(self.handle))

    # ---- broad phase -------------------------------------------------------------------------------------
    def broadphase(self, aabbs: Aabbs, capacity: int | None = None) -> PairList:
        """Runs the sweep; grows the output list and retries once when the capacity guess was too small."""
        cap = capacity if capacity is not None else max(1024, 16 * int(aabbs.collider.shape[0]))
        a = aabbs.as_struct()
        self._keep_bp = (aabbs, a)
        self._check(self.lib.avn_broadphase_upload(self.handle, C.byref(a)))
        self._check(self.lib.avn_broadphase_run(self.handle))
        out = PairList.empty(cap)
        s = out.as_struct()
        st = self.lib.avn_broadphase_download(self.handle, C.byref(s))
        if st == ERR_CAPACITY:
            out = PairList.empty(int(s.count))
            s = out.as_struct()
            st = self.lib.avn_broadphase_download(self.handle, C.byref(s))
        self._check(st)
        out.count = int(s.count)
        aabbs.retained_count = int(a.retained_count)
        return out.trimmed()

    def broadphase_upload(self, aabbs: Aabbs) -> None:
        a = aabbs.as_struct()
        self._keep_bp = (aabbs, a)
        self._check(self.lib.avn_broadphase_upload(self.handle, C.byref(a)))

    def broadphase_run(self) -> None:
        self._check(self.lib.avn_broadphase_run(self.handle))

    def broadphase_download(self, out: PairList) -> PairList:
        s = out.as_struct()
        self._check(self.lib.avn_broadphase_download(self.handle, C.byref(s)))
        out.count = int(s.count)
        self._keep_bp[0].retained_count = int(self._keep_bp[1].retained_count)
        return out

    # ---- x-slab partition (include/avian_b200.h "one coupled scene over several GPUs")
    def solver_run_range(self, first: int, count: int, flags: int) -> None:
        self._check(self.lib.avn_solver_run_range(self.handle, first, count, flags))

    def solver_set_boundary(self, body: np.ndarray, source: np.ndarray, owner_rank: np.ndarray, record_count: int, rank: int, world: int) -> None:
        body, source, owner_rank = (np.ascontiguousarray(x, dtype=np.int32) for x in (body, source, owner_rank))
        assert source.size == body.shape[0] * world
        b = AvnBoundary(int(body.shape[0]), int(record_count), int(rank), int(world), _ptr(body), _ptr(source), _ptr(owner_rank))
        self._check(self.lib.avn_solver_set_boundary(self.handle, C.byref(b)))

    def solver_boundary_snapshot(self) -> None:
        self._check(self.lib.avn_solver_boundary_snapshot(self.handle))

    def solver_boundary_pack(self, device_ptr: int) -> None:
        self._check(self.lib.avn_solver_boundary_pack(self.handle, _vp(device_ptr)))

    def solver_boundary_apply(self, device_ptr: int) -> None:
        self._check(self.lib.avn_solver_boundary_apply(self.handle, _vp(device_ptr)))

    def solver_needs_restitution(self) -> bool:
        out = C.c_int(0)
        self._check(self.lib.avn_solver_needs_restitution(self.handle, C.byref(out)))
        return bool(out.value)

    # ---- communicator (NCCL inside the library; one process per GPU)
    def comm_unique_id(self) -> bytes:
        buf = C.create_string_buffer(COMM_ID_BYTES)
        self._check(self.lib.avn_comm_unique_id(self.handle, C.cast(buf, _vp)))
        return buf.raw

    def comm_init(self, rank: int, world: int, unique_id: bytes | None = None) -> None:
        buf = None if unique_id is None else C.create_string_buffer(bytes(unique_id), COMM_ID_BYTES)
        self._check(self.lib.avn_comm_init(self.handle, rank, world, None if buf is None else C.cast(buf, _vp)))

    def comm_destroy(self) -> None:
        self._check(self.lib.avn_comm_destroy(self.handle))

    def comm_all_gather(self, send_device_ptr: int, recv_device_ptr: int, bytes_per_rank: int) -> None:
        self._check(self.lib.avn_comm_all_gather(self.handle, _vp(send_device_ptr), _vp(recv_device_ptr), bytes_per_rank))

    def solver_step_partitioned(self) -> None:
        """The partitioned solver stage of this rank (after solver_upload + solver_set_boundary); then solver_download."""
        self._check(self.lib.avn_solver_step_partitioned(self.handle))

    def stream(self) -> int:
        """The context's cudaStream_t as an integer (torch.cuda.ExternalStream(ptr) orders a collective with the launches)."""
        out = _vp()
        self._check(self.lib.avn_get_stream(self.handle, C.byref(out)))
        return int(out.value or 0)

    # ---- the ContactGraph + ConstraintGraph on the device (include/avian_b200.h avn_contacts_configure / _step)
    def contacts_configure(self, body_kind, collider_count: int, friction=None, restitution=None) -> None:
        kind = np.ascontiguousarray(body_kind, dtype=np.uint8)
        fr = None if friction is None else np.ascontiguousarray(friction, dtype=np.float64)
        re = None if restitution is None else np.ascontiguousarray(restitution, dtype=np.float64)
        cfg = AvnContactGraphConfig(int(kind.shape[0]), int(collider_count), _ptr(kind), _ptr(fr), _ptr(re))
        self._check(self.lib.avn_contacts_configure(self.handle, C.byref(cfg)))

    def solver_prefetch_bodies(self, bodies: Bodies, static_unchanged: bool = False) -> None:
        """avn_solver_prefetch_bodies: the body columns of the next solver upload start moving to the device now (second stream)."""
        b = bodies.as_struct()
        self._keep_prefetch = (bodies, b)
        self._check(self.lib.avn_solver_prefetch_bodies(self.handle, C.byref(b), BODIES_STATIC_UNCHANGED if static_unchanged else 0))

    def contacts_step(self, dt: float, contact_tolerance: float, colliders: dict, lin_vel, ang_vel, match_contacts: bool = True, take_pairs: bool = True,
                      length_unit: float = 1.0, shapes_unchanged: bool = False) -> dict:
        """avn_contacts_step: (the last broad phase's new pairs ->) rows, geometry + matching, status loop, graphs, colour-major list — all on the
        device.  Returns the step's counters and the colour offsets of the list."""
        dt_ = self.scalar
        cols = {k: (None if colliders.get(k) is None else np.ascontiguousarray(colliders[k], dtype=(np.uint8 if k == "shape" else dt_)))
                for k in ("shape", "dims", "position", "rotation", "aabb_min", "aabb_max")}
        lv, av = np.ascontiguousarray(lin_vel, dtype=dt_), np.ascontiguousarray(ang_vel, dtype=dt_)
        inp = AvnNarrowInput(0, int(cols["position"].shape[0]), int(lv.shape[0]), 0, None, None, None, None, _ptr(cols["shape"]), _ptr(cols["dims"]),
                             _ptr(cols["position"]), _ptr(cols["rotation"]), _ptr(lv), _ptr(av), _ptr(cols["aabb_min"]), _ptr(cols["aabb_max"]))
        prm = AvnNarrowParams(float(dt), float(contact_tolerance))
        out = AvnContactStep()
        self._check(self.lib.avn_contacts_step(self.handle, C.byref(prm), C.byref(inp), 1 if match_contacts else 0, float(length_unit),
                                               (CONTACTS_TAKE_BROADPHASE_PAIRS if take_pairs else 0) | (CONTACTS_SHAPES_UNCHANGED if shapes_unchanged else 0),
                                               C.byref(out)))
        st = {n: int(getattr(out, n)) for n, _ in AvnContactStep._fields_ if n not in ("_pad", "color_offsets")}
        st["color_offsets"] = np.array(list(out.color_offsets), dtype=np.uint32)
        return st

    def contacts_set_body_frames(self, position=None, rotation=None, center_of_mass=None, body_count: int | None = None) -> None:
        """avn_contacts_set_body_frames: the body Position / Rotation ([B] rows, like the velocity columns) and local centre of mass (None = 0)
        that every later contacts_step / narrow_phase measures its anchors from, until the next call.  position=None and rotation=None clear
        them (a collider at its body's origin, the centre of mass at that origin).  body_count defaults to the rows of `position`."""
        if position is None and rotation is None and center_of_mass is None and body_count is None:
            self._keep_frames = None
            self._check(self.lib.avn_contacts_set_body_frames(self.handle, None))
            return
        dt_ = self.scalar
        col = lambda a, w: None if a is None else np.ascontiguousarray(a, dtype=dt_).reshape(-1, w)
        pos, rot, com = col(position, 3), col(rotation, 4), col(center_of_mass, 3)
        n = int(body_count if body_count is not None else (pos.shape[0] if pos is not None else 0))
        f = AvnBodyFrames(n, 0, _ptr(pos), _ptr(rot), _ptr(com))
        self._keep_frames = (pos, rot, com, f)
        self._check(self.lib.avn_contacts_set_body_frames(self.handle, C.byref(f)))

    def set_convex_hulls(self, hulls: "ConvexHulls | None") -> None:
        """avn_set_convex_hulls: the hull table every later update_aabbs / narrow_phase / contacts_step, query_update, spatial query and
        move_and_slide reads (None clears it).  Replacing or clearing it makes every query and move_and_slide against a tree that holds a
        hull refuse until the next query_update.  Raises AvianError (AVN_ERR_INVALID_ARGUMENT) for a table the library refuses; a refused
        call changes nothing."""
        if hulls is None:
            self._check(self.lib.avn_set_convex_hulls(self.handle, None))
            return
        st, keep = hulls.as_struct(self.scalar)
        self._check(self.lib.avn_set_convex_hulls(self.handle, C.byref(st)))

    def solver_step_resident(self, params, bodies: Bodies, joints: JointSet | None = None) -> None:
        """avn_solver_upload_resident + run + download: manifolds AND constraint graph come from the contact store on the device."""
        b = bodies.as_struct()
        j = joints.as_struct() if joints is not None and joints.count else None
        self._keep = (params, bodies, joints, b, j)
        self._check(self.lib.avn_solver_upload_resident(self.handle, C.byref(params), C.byref(b), C.byref(j) if j is not None else None))
        self._check(self.lib.avn_solver_run(self.handle))
        self._check(self.lib.avn_solver_download(self.handle))

    def broadphase_download_order(self) -> int:
        n = C.c_uint64(0)
        self._check(self.lib.avn_broadphase_download_order(self.handle, C.byref(n)))
        self._keep_bp[0].retained_count = int(self._keep_bp[1].retained_count)
        return int(n.value)

    def contacts_download_graph(self, capacity: int, manifold_count: int) -> dict:
        out = {"collider1": np.zeros(capacity, dtype=np.uint32), "collider2": np.zeros(capacity, dtype=np.uint32), "live": np.zeros(capacity, dtype=np.uint8),
               "touching": np.zeros(capacity, dtype=np.uint8), "colour": np.zeros(capacity, dtype=np.int8), "edge": np.zeros(manifold_count, dtype=np.uint32)}
        # edge_list receives the WHOLE colour-major list of the last step: only ask for it with a buffer of that size
        ptrs = [out[k].ctypes.data for k in ("collider1", "collider2", "live", "touching", "colour")] + [out["edge"].ctypes.data if manifold_count else None]
        self._check(self.lib.avn_contacts_download_graph(self.handle, int(capacity), *ptrs))
        return out

    # ---- persistent islands + sleeping decisions (include/avian_b200.h avn_islands_configure / _step)
    def islands_configure(self, body_kind, joints=None, thr_lin=None, thr_ang=None, disabled=None, time_to_sleep: float = 0.5, length_unit: float = 1.0) -> None:
        kind = np.ascontiguousarray(body_kind, dtype=np.uint8)
        f32 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float32)
        tl, ta = f32(thr_lin), f32(thr_ang)
        dis = None if disabled is None else np.ascontiguousarray(disabled, dtype=np.uint8)
        j1 = j2 = None
        nj = 0
        if joints is not None and len(joints):
            jj = np.ascontiguousarray(joints, dtype=np.uint32).reshape(-1, 2)
            j1, j2, nj = np.ascontiguousarray(jj[:, 0]), np.ascontiguousarray(jj[:, 1]), int(jj.shape[0])
        cfg = AvnIslandsConfig(int(kind.shape[0]), nj, _ptr(kind), _ptr(tl), _ptr(ta), _ptr(dis), _ptr(j1), _ptr(j2), float(time_to_sleep), float(length_unit))
        self._check(self.lib.avn_islands_configure(self.handle, C.byref(cfg)))
        self._isl_B = int(kind.shape[0])

    def islands_step(self, delta_secs: float, lin_vel, ang_vel, wake=None) -> dict:
        B = self._isl_B
        lv, av = np.ascontiguousarray(lin_vel, dtype=self.scalar), np.ascontiguousarray(ang_vel, dtype=self.scalar)
        wk = None if wake is None else np.ascontiguousarray(wake, dtype=np.uint8)
        out = {"island": np.zeros(B, dtype=np.uint32), "sleeping": np.zeros(B, dtype=np.uint8), "sleep_timer": np.zeros(B, dtype=np.float32)}
        st = AvnIslandsStep(float(delta_secs), 0, _ptr(lv), _ptr(av), _ptr(wk), _ptr(out["island"]), _ptr(out["sleeping"]), _ptr(out["sleep_timer"]))
        self._check(self.lib.avn_islands_step(self.handle, C.byref(st)))
        for n in ("island_count", "sleeping_islands", "islands_put_to_sleep", "islands_woken", "split_bodies", "merges"):
            out[n] = int(getattr(st, n))
        return out

    # ---- applied sleeping (include/avian_b200.h avn_islands_apply / _wake)
    def islands_apply(self, enable: bool = True) -> None:
        """avn_islands_apply: from now on the library plays SleepIslands / WakeIslands on its rows, graphs and solver stage."""
        self._check(self.lib.avn_islands_apply(self.handle, 1 if enable else 0))

    def islands_wake(self, wake=None) -> dict:
        """avn_islands_wake: between contacts_step and solver_step_resident.  Returns the counters and the colour offsets after the wake."""
        wk = None if wake is None else np.ascontiguousarray(wake, dtype=np.uint8)
        out = AvnIslandsWake()
        self._check(self.lib.avn_islands_wake(self.handle, _ptr(wk), C.byref(out)))
        st = {n: int(getattr(out, n)) for n, _ in AvnIslandsWake._fields_ if n != "color_offsets"}
        st["color_offsets"] = np.array(list(out.color_offsets), dtype=np.uint32)
        return st

    def contacts_download_sleeping(self, capacity: int, body_count: int) -> dict:
        out = {"row_asleep": np.zeros(capacity, dtype=np.uint8), "body_asleep": np.zeros(body_count, dtype=np.uint8)}
        self._check(self.lib.avn_contacts_download_sleeping(self.handle, int(capacity), _ptr(out["row_asleep"]) if capacity else None, int(body_count),
                                                            _ptr(out["body_asleep"]) if body_count else None))
        return out

    # ---- swept CCD (include/avian_b200.h avn_ccd_*): solve_swept_ccd inside the device-resident solver stage
    def ccd_configure(self, body=None, collider=None, mode=None, include_dynamic=None, linear_threshold=None, angular_threshold=None,
                      prediction_distance: float = float("inf"), capsules: bool = False, hulls: bool = False) -> None:
        """avn_ccd_configure: the SweptCcd bodies in query order and their own colliders; body=None clears the configuration.  capsules=True
        sets AVN_CCD_CAPSULES: capsule colliders are swept (without it a contact store that holds one is refused).  hulls=True sets
        AVN_CCD_HULLS: convex hull colliders are swept over the context's hull table (set_convex_hulls); without it a contact store that holds
        one is refused.  A solver_run after set_convex_hulls has replaced the table fails until the next contacts_step."""
        if body is None or len(body) == 0:
            self._check(self.lib.avn_ccd_configure(self.handle, None))
            self._ccd_n = 0
            return
        cfg, cols = ccd_config(body, collider, mode, include_dynamic, linear_threshold, angular_threshold, prediction_distance,
                               (CCD_CAPSULES if capsules else 0) | (CCD_HULLS if hulls else 0))
        self._check(self.lib.avn_ccd_configure(self.handle, C.byref(cfg)))
        self._ccd_n = int(cfg.count)

    def ccd_download(self) -> dict:
        """avn_ccd_download: per configured body the last step's min_toi, hit_body, hit_contact, candidates, hits; plus pass_ms, total_candidates."""
        n = getattr(self, "_ccd_n", 0)
        out = {"min_toi": np.zeros(n, dtype=self.scalar), "hit_body": np.zeros(n, dtype=np.int32), "hit_contact": np.zeros(n, dtype=np.int32),
               "candidates": np.zeros(n, dtype=np.uint32), "hits": np.zeros(n, dtype=np.uint32)}
        r = AvnCcdResult(*(_ptr(out[k]) for k in ("min_toi", "hit_body", "hit_contact", "candidates", "hits")), 0.0, 0)
        self._check(self.lib.avn_ccd_download(self.handle, C.byref(r)))
        out["pass_ms"], out["total_candidates"] = float(r.pass_ms), int(r.total_candidates)
        return out

    # ---- the pipeline's output to the application (include/avian_b200.h avn_contacts_set_sensors / _remove_colliders / _events / _report)
    def contacts_set_sensors(self, sensor, collider_count: int | None = None) -> None:
        """avn_contacts_set_sensors: the Sensor flag per collider (None = no sensor; then collider_count is required)."""
        col = None if sensor is None else np.ascontiguousarray(sensor, dtype=bool).astype(np.uint8)
        n = int(col.shape[0]) if collider_count is None else int(collider_count)
        self._check(self.lib.avn_contacts_set_sensors(self.handle, n, _ptr(col)))

    def contacts_remove_colliders(self, colliders) -> None:
        """avn_contacts_remove_colliders: remove_collider for each listed collider (despawned, disabled)."""
        ids = np.ascontiguousarray(colliders, dtype=np.uint32)
        self._check(self.lib.avn_contacts_remove_colliders(self.handle, int(ids.shape[0]), _ptr(ids)))

    def contacts_events(self, capacity: int | None = None) -> tuple[dict, dict]:
        """avn_contacts_events: (started, ended) of the last avn_contacts_step, each a dict of numpy columns collider1, collider2, body1, body2,
        flags.  capacity=None retries once with the required sizes; an explicit capacity that is too small raises AvianError(ERR_CAPACITY)
        with .required = (started, ended)."""
        cap = 256 if capacity is None else int(capacity)
        (s, so), (e, eo) = collision_events(cap), collision_events(cap)
        st = self.lib.avn_contacts_events(self.handle, C.byref(s), C.byref(e))
        if st == ERR_CAPACITY and capacity is None:
            (s, so), (e, eo) = collision_events(int(s.count)), collision_events(int(e.count))
            st = self.lib.avn_contacts_events(self.handle, C.byref(s), C.byref(e))
        if st == ERR_CAPACITY:
            err = AvianError(st, self.lib.avn_last_error(self.handle).decode())
            err.required = (int(s.count), int(e.count))
            raise err
        self._check(st)
        return ({k: v[:int(s.count)] for k, v in so.items()}, {k: v[:int(e.count)] for k, v in eo.items()})

    def contacts_report(self, events_only: bool = False, capacity: int | None = None) -> dict:
        """avn_contacts_report: one entry per touching pair in ascending ContactId (contact_id, collider1, collider2, body1, body2, flags,
        point_count, normal, total_normal_impulse, max_normal_impulse, max_penetration).  Capacity protocol as contacts_events."""
        cap = 1024 if capacity is None else int(capacity)
        flags = REPORT_EVENTS_ONLY if events_only else 0
        r, out = contact_report(cap, self.scalar)
        st = self.lib.avn_contacts_report(self.handle, flags, C.byref(r))
        if st == ERR_CAPACITY and capacity is None:
            r, out = contact_report(int(r.count), self.scalar)
            st = self.lib.avn_contacts_report(self.handle, flags, C.byref(r))
        if st == ERR_CAPACITY:
            err = AvianError(st, self.lib.avn_last_error(self.handle).decode())
            err.required = int(r.count)
            raise err
        self._check(st)
        return {k: v[:int(r.count)] for k, v in out.items()}

    def contacts_download_impulses(self, capacity: int):
        """avn_contacts_download_impulses: (warm_start_normal [capacity, 4], warm_start_tangent [capacity, 4, 2], normal_impulse [capacity, 4]) of the
        rows as the last solve left them; rows beyond the store's stay zero."""
        wn, wt, ni = (np.zeros((capacity, 4), dtype=self.scalar), np.zeros((capacity, 4, 2), dtype=self.scalar), np.zeros((capacity, 4), dtype=self.scalar))
        self._check(self.lib.avn_contacts_download_impulses(self.handle, int(capacity), wn.ctypes.data, wt.ctypes.data, ni.ctypes.data))
        return wn, wt, ni

    def narrow_phase(self, dt: float, contact_tolerance: float, pairs, colliders: dict, lin_vel: np.ndarray, ang_vel: np.ndarray) -> dict:
        """avn_narrow_phase: pairs = (collider1, collider2, body1, body2) uint32 arrays; colliders = dict(shape, dims, position, rotation,
        aabb_min=None, aabb_max=None).  Returns the raw manifold columns (4 point slots per pair)."""
        c1, c2, b1, b2 = (np.ascontiguousarray(x, dtype=np.uint32) for x in pairs)
        n, dt_ = int(c1.shape[0]), self.scalar
        cols = {k: (None if colliders.get(k) is None else np.ascontiguousarray(colliders[k], dtype=(np.uint8 if k == "shape" else dt_)))
                for k in ("shape", "dims", "position", "rotation", "aabb_min", "aabb_max")}
        lv, av = np.ascontiguousarray(lin_vel, dtype=dt_), np.ascontiguousarray(ang_vel, dtype=dt_)
        inp = AvnNarrowInput(n, int(cols["position"].shape[0]), int(lv.shape[0]), 0, _ptr(c1), _ptr(c2), _ptr(b1), _ptr(b2), _ptr(cols["shape"]),
                             _ptr(cols["dims"]), _ptr(cols["position"]), _ptr(cols["rotation"]), _ptr(lv), _ptr(av), _ptr(cols["aabb_min"]),
                             _ptr(cols["aabb_max"]))
        out = {"point_count": np.zeros(n, dtype=np.uint8), "disjoint": np.zeros(n, dtype=np.uint8), "normal": np.zeros((n, 3), dtype=dt_),
               "anchor1": np.zeros((n, 4, 3), dtype=dt_), "anchor2": np.zeros((n, 4, 3), dtype=dt_), "penetration": np.zeros((n, 4), dtype=dt_),
               "normal_speed": np.zeros((n, 4), dtype=dt_)}
        raw = AvnRawManifolds(*(_ptr(out[k]) for k in ("point_count", "disjoint", "normal", "anchor1", "anchor2", "penetration", "normal_speed")))
        prm = AvnNarrowParams(float(dt), float(contact_tolerance))
        self._check(self.lib.avn_narrow_phase(self.handle, C.byref(prm), C.byref(inp), C.byref(raw)))
        return out

    def update_aabbs(self, params: "AvnAabbParams", colliders: "Colliders") -> None:
        c = colliders.as_struct()
        self._keep_aabb = (params, colliders, c)
        self._check(self.lib.avn_update_aabbs(self.handle, C.byref(params), C.byref(c)))

    def timings(self) -> dict:
        t = AvnTimings()
        self._check(self.lib.avn_get_timings(self.handle, C.byref(t)))
        return {n: getattr(t, n) for n, _ in AvnTimings._fields_ if n != "_pad"}

    # ---- spatial queries (include/avian_b200.h avn_query_*): SpatialQueryPipeline on the device
    def query_update(self, colliders: "QueryColliders", shapes_unchanged: bool = False) -> None:
        """avn_query_update: rebuild the collider tree from these poses (shape, dims and memberships stay on the device with shapes_unchanged)."""
        c, keep = colliders.as_struct(self.scalar)
        self._check(self.lib.avn_query_update(self.handle, C.byref(c), QUERY_SHAPES_UNCHANGED if shapes_unchanged else 0))

    def cast_ray(self, rays: "Rays") -> dict:
        """avn_query_cast_ray: per ray the closest hit — collider (-1 = none), distance, normal."""
        r, keep = rays.as_struct(self.scalar)
        n = rays.count
        out = {"collider": np.zeros(n, dtype=np.int32), "distance": np.zeros(n, dtype=self.scalar), "normal": np.zeros((n, 3), dtype=self.scalar)}
        o = AvnRayClosest(*(_ptr(out[k]) for k in ("collider", "distance", "normal")))
        self._check(self.lib.avn_query_cast_ray(self.handle, C.byref(r), C.byref(o)))
        return out

    def ray_hits(self, rays: "Rays", capacity: int | None = None) -> dict:
        """avn_query_ray_hits: CSR offsets[n+1], collider, distance, normal.  capacity=None sizes the output from the required count;
        an explicit capacity that is too small raises AvianError(ERR_CAPACITY) with .required."""
        r, keep = rays.as_struct(self.scalar)
        h, out = hit_list(rays.count, 4 * rays.count if capacity is None else capacity, self.scalar, True)
        st = self.lib.avn_query_ray_hits(self.handle, C.byref(r), C.byref(h))
        if st == ERR_CAPACITY and capacity is None:
            h, out = hit_list(rays.count, int(h.count), self.scalar, True)
            st = self.lib.avn_query_ray_hits(self.handle, C.byref(r), C.byref(h))
        self._check_list(st, h)
        return hit_list_result(h, out)

    def aabb_intersections(self, aabb_min, aabb_max, capacity: int | None = None) -> dict:
        """avn_query_aabb_intersections: per query box the colliders whose tight AABB it touches (CSR offsets[n+1], collider)."""
        mn = np.ascontiguousarray(aabb_min, dtype=self.scalar).reshape(-1, 3)
        mx = np.ascontiguousarray(aabb_max, dtype=self.scalar).reshape(-1, 3)
        n = int(mn.shape[0])
        h, out = hit_list(n, 4 * n if capacity is None else capacity, self.scalar, False)
        st = self.lib.avn_query_aabb_intersections(self.handle, n, _ptr(mn), _ptr(mx), C.byref(h))
        if st == ERR_CAPACITY and capacity is None:
            h, out = hit_list(n, int(h.count), self.scalar, False)
            st = self.lib.avn_query_aabb_intersections(self.handle, n, _ptr(mn), _ptr(mx), C.byref(h))
        self._check_list(st, h)
        return hit_list_result(h, out)

    def cast_shape(self, shapes: "ShapeQueries") -> dict:
        """avn_query_cast_shape: per query shape the closest hit — collider (-1 = none), distance, point1, point2, normal1, normal2."""
        s, keep = shapes.as_struct(self.scalar)
        o, out = shape_closest(shapes.count, self.scalar)
        self._check(self.lib.avn_query_cast_shape(self.handle, C.byref(s), C.byref(o)))
        return out

    def shape_hits(self, shapes: "ShapeQueries", capacity: int | None = None) -> dict:
        """avn_query_shape_hits: CSR offsets[n+1], collider, distance, point1, point2, normal1, normal2 (per shape its max_hits nearest).
        capacity=None sizes the output from the required count; a capacity that is too small raises AvianError(ERR_CAPACITY) with .required."""
        s, keep = shapes.as_struct(self.scalar)
        h, out = shape_hit_list(shapes.count, 4 * shapes.count if capacity is None else capacity, self.scalar)
        st = self.lib.avn_query_shape_hits(self.handle, C.byref(s), C.byref(h))
        if st == ERR_CAPACITY and capacity is None:
            h, out = shape_hit_list(shapes.count, int(h.count), self.scalar)
            st = self.lib.avn_query_shape_hits(self.handle, C.byref(s), C.byref(h))
        self._check_list(st, h)
        return hit_list_result(h, out)

    def project_point(self, points: "Points") -> dict:
        """avn_query_project_point: per point the closest collider (-1 = none), the projection and is_inside."""
        p, keep = points.as_struct(self.scalar)
        o, out = point_projection(points.count, self.scalar)
        self._check(self.lib.avn_query_project_point(self.handle, C.byref(p), C.byref(o)))
        return out

    def point_intersections(self, points: "Points", capacity: int | None = None) -> dict:
        """avn_query_point_intersections: per point the colliders containing it (CSR offsets[n+1], collider ascending)."""
        p, keep = points.as_struct(self.scalar)
        n = points.count
        h, out = hit_list(n, 4 * n if capacity is None else capacity, self.scalar, False)
        st = self.lib.avn_query_point_intersections(self.handle, C.byref(p), C.byref(h))
        if st == ERR_CAPACITY and capacity is None:
            h, out = hit_list(n, int(h.count), self.scalar, False)
            st = self.lib.avn_query_point_intersections(self.handle, C.byref(p), C.byref(h))
        self._check_list(st, h)
        return hit_list_result(h, out)

    def move_and_slide(self, config: "MoveConfig", batch: "MoveBatch") -> dict:
        """avn_move_and_slide against the tree of the last query_update: position, velocity (MoveAndSlideOutput), per iteration the sweep
        hit (hit_collider -1 = none, hit_distance = safe distance, hit_toi, hit_point, hit_normal) and kernel_ms."""
        c, keep_c = config.as_struct()
        b, keep_b = batch.as_struct(self.scalar)
        o, out = move_result(batch.count, config.move_and_slide_iterations, self.scalar)
        self._check(self.lib.avn_move_and_slide(self.handle, C.byref(c), C.byref(b), C.byref(o)))
        out["kernel_ms"] = float(o.kernel_ms)
        return out

    def shape_intersections(self, shapes: "ShapeQueries", capacity: int | None = None) -> dict:
        """avn_query_shape_intersections: per query shape the colliders it intersects (CSR offsets[n+1], collider ascending)."""
        s, keep = shapes.as_struct(self.scalar)
        n = shapes.count
        h, out = hit_list(n, 4 * n if capacity is None else capacity, self.scalar, False)
        st = self.lib.avn_query_shape_intersections(self.handle, C.byref(s), C.byref(h))
        if st == ERR_CAPACITY and capacity is None:
            h, out = hit_list(n, int(h.count), self.scalar, False)
            st = self.lib.avn_query_shape_intersections(self.handle, C.byref(s), C.byref(h))
        self._check_list(st, h)
        return hit_list_result(h, out)
