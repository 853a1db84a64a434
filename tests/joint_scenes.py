"""Seeded joint scenes for the XPBD joint stage: bodies and joints in the input format of tests/golden/handworked/worked.py, no contacts.

`family(name)` gives the scene dict; `columns(scene, dtype)` the ABI columns (tests/test_handworked.py's `_build`); `census(scene)` counts,
from the scene data, the branches of `solve_joint_item`, `damp_joint_item` and `project_velocity_item` and the body sides and schedule
shapes the scene reaches.  The branch predicates are evaluated on the prepared geometry (every body at its input pose), where each
special joint is placed well inside its branch, so the first substep takes it there.

* `features` (4 substeps), `features_sub12` (12 substeps): every type; limits on and off; the revolute angle limit with its obtuse branch with
  and without the `phi > pi` wrap; spherical swing and twist limits, the twist with `dot(a1, a2) <= -0.5` (`max_corr = h`); the prismatic
  slider limit; distance joints below min, above max and inside; the `<= eps` exits of align_orientation (an aligned fixed joint), point_solve
  (coincident anchors), the prismatic and distance corrections and the spherical normalisations (parallel and opposite swing axes); compliance
  zero and non-zero; damping on and off; static bodies by index on side 1, side 2 and both; positive and negative dominance with a dominated
  body also written by an equal-dominance joint; a moving kinematic body under damping; off-origin centres of mass, full local inverse
  inertia, LockedAxes; several damped joints of one type whose static end is on the same side (joint_damping's dummy carry); random joints
  of all five types over a shared pool, so levels interleave the types.
* `hub` (1 substep): a kinematic body shared by 48 joints that all sit in one level (no damping: the hub is only ever the dominated side).
* `chain` (1 substep): 2 500 damped spherical links from a static anchor, one level per link in the solve and the damping schedule.
* `wide` (1 substep): 70 000 distance joints from one static body, one level wider than the megakernel grid (grid x 128 slots).
"""
from __future__ import annotations

import math

import numpy as np

from avian_b200 import api

from test_handworked import _build

DYNAMIC, KINEMATIC, STATIC = api.BODY_DYNAMIC, api.BODY_KINEMATIC, api.BODY_STATIC
FIXED, REVOLUTE, SPHERICAL, PRISMATIC, DISTANCE = (api.JOINT_FIXED, api.JOINT_REVOLUTE, api.JOINT_SPHERICAL, api.JOINT_PRISMATIC,
                                                   api.JOINT_DISTANCE)
DEFAULT_AXIS = {FIXED: (0, 0, 1), REVOLUTE: (0, 0, 1), SPHERICAL: (0, 1, 0), PRISMATIC: (1, 0, 0), DISTANCE: (0, 0, 1)}
LIMIT_KEY = {REVOLUTE: "angle_limit", SPHERICAL: "swing_limit", PRISMATIC: "limits"}


def params(substeps, dt=1.0 / 60.0):
    dt_ns = round(dt * 1e9)                                   # Duration arithmetic in integer nanoseconds (solver/schedule.rs:195-200)
    h_ns = round(dt_ns / 1e9 / substeps * 1e9)
    return {"dt": dt_ns / 1e9, "h": h_ns / 1e9, "substeps": substeps, "gravity": [0.0, -9.81, 0.0], "contact_damping_ratio": 10.0,
            "contact_frequency_factor": 1.5, "max_overlap_solve_speed": 4.0, "warm_start_coefficient": 1.0, "restitution_threshold": 1.0,
            "restitution_iterations": 1, "length_unit": 1.0, "match_contacts": 1}


def axis_angle(axis, angle):
    n = math.sqrt(sum(x * x for x in axis))
    s = math.sin(angle / 2) / n
    return [axis[0] * s, axis[1] * s, axis[2] * s, math.cos(angle / 2)]


IDENTITY = [0.0, 0.0, 0.0, 1.0]


def _unit(rng):
    v = rng.normal(size=3)
    return v / np.linalg.norm(v)


def _unit4(rng):
    q = rng.normal(size=4)
    return q / np.linalg.norm(q)


def _conj(q):
    return np.array([-q[0], -q[1], -q[2], q[3]])


def _mul(q, r):
    x0, y0, z0, w0 = q
    x1, y1, z1, w1 = r
    return np.array([w0 * x1 + x0 * w1 + y0 * z1 - z0 * y1, w0 * y1 - x0 * z1 + y0 * w1 + z0 * x1, w0 * z1 + x0 * y1 - y0 * x1 + z0 * w1,
                     w0 * w1 - x0 * x1 - y0 * y1 - z0 * z1])


def _rot(q, v):
    b, w = np.array(q[:3]), q[3]
    return v * (w * w - b @ b) + 2 * b * (v @ b) + 2 * w * np.cross(b, v)


class _Scene:
    def __init__(self, seed, substeps):
        self.rng = np.random.default_rng(seed)
        self.bodies, self.joints = [], []
        self.params = params(substeps)

    def body(self, kind, pos, rot=IDENTITY, v=(0, 0, 0), w=(0, 0, 0), inv_mass=1.0, inv_inertia=(4.0, 0, 0, 4.0, 0, 4.0), **kw):
        if kind == STATIC:
            v, w, inv_mass, inv_inertia = (0, 0, 0), (0, 0, 0), 0.0, (0,) * 6
        elif kind == KINEMATIC:
            inv_mass, inv_inertia = 0.0, (0,) * 6
        b = {"kind": int(kind), "position": [float(x) for x in pos], "rotation": [float(x) for x in rot], "linear_velocity": [float(x) for x in v],
             "angular_velocity": [float(x) for x in w], "inverse_mass": float(inv_mass), "inverse_inertia_local": [float(x) for x in inv_inertia]}
        b.update(kw)
        self.bodies.append(b)
        return len(self.bodies) - 1

    def random_body(self, near=None, spread=1.5):
        """a dynamic body with what the joint stage reads per body drawn at random: pose (within 0.8 of body `near`, when given), velocities,
        mass, full or diagonal local inverse inertia, centre-of-mass offset, LockedAxes, dominance"""
        r = self.rng
        centre = np.zeros(3) if near is None else np.array(self.bodies[near]["position"])
        spread = spread if near is None else 0.8
        q = r.normal(size=4)
        q /= np.linalg.norm(q)
        d = r.uniform(0.5, 6.0, 3)
        if r.random() < 0.5:
            a = r.normal(size=4)
            a /= np.linalg.norm(a)
            x, y, z, ww = a
            R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - ww * z), 2 * (x * z + ww * y)],
                          [2 * (x * y + ww * z), 1 - 2 * (x * x + z * z), 2 * (y * z - ww * x)],
                          [2 * (x * z - ww * y), 2 * (y * z + ww * x), 1 - 2 * (x * x + y * y)]])
            M = R @ np.diag(d) @ R.T
            il = [M[0, 0], M[0, 1], M[0, 2], M[1, 1], M[1, 2], M[2, 2]]
        else:
            il = [d[0], 0.0, 0.0, d[1], 0.0, d[2]]
        return self.body(DYNAMIC, centre + r.uniform(-spread, spread, 3), q, r.uniform(-1, 1, 3), r.uniform(-2, 2, 3), r.uniform(0.3, 2.0), il,
                         center_of_mass=[float(x) for x in r.uniform(-0.15, 0.15, 3)],
                         locked_axes=int(r.choice([0, 0, 0, 0, 0x20, 0x12, 0x04, 0x07])), dominance=int(r.choice([0, 0, 0, 0, 1, -1])))

    def joint(self, t, b1, b2, a1=(0, 0, 0), a2=(0, 0, 0), **kw):
        j = {"type": int(t), "body1": int(b1), "body2": int(b2), "local_anchor1": [float(x) for x in a1], "local_anchor2": [float(x) for x in a2]}
        if t == DISTANCE:
            j.setdefault("limit_min", 0.0)
            j.setdefault("limit_max", 0.0)
        j.update(kw)
        self.joints.append(j)
        return j

    def random_joint(self, t, b1, b2, damping_share=0.4, **override):
        """a joint of type t between b1 and b2 that starts a few centimetres and a few degrees off its rest pose (random anchors, bases
        and axis, then body 2's anchor and basis fitted to body 1's), with random limits, compliances and damping"""
        r = self.rng
        kw = {"compliance0": float(r.choice([0.0, 1e-4])), "compliance1": float(r.choice([0.0, 1e-3])), "compliance2": float(r.choice([0.0, 1e-3]))}
        P1, Q1 = np.array(self.bodies[b1]["position"]), np.array(self.bodies[b1]["rotation"])
        P2, Q2 = np.array(self.bodies[b2]["position"]), np.array(self.bodies[b2]["rotation"])
        a1 = r.uniform(-0.4, 0.4, 3)
        # world anchors p + R la coincide up to a few centimetres (distance joints: up to a metre, against limits near that length)
        off = r.normal(size=3) * 0.03 if t != DISTANCE else _unit(r) * r.uniform(0.3, 1.0)
        a2 = _rot(_conj(Q2), P1 + _rot(Q1, a1) - P2 + off)
        if t != DISTANCE:
            basis1 = _unit4(r) if r.random() < 0.5 else np.array(IDENTITY)
            # body 2's basis = its rotation undone, body 1's frame, and a turn of up to ~0.15 rad
            kw["local_basis1"] = [float(x) for x in basis1]
            kw["local_basis2"] = [float(x) for x in _mul(_mul(_conj(Q2), _mul(Q1, basis1)), axis_angle(_unit(r), r.uniform(0.0, 0.15)))]
            if r.random() < 0.5:
                kw["axis"] = [float(x) for x in _unit(r)]
        if t in LIMIT_KEY and r.random() < 0.6:
            kw[LIMIT_KEY[t]] = [float(r.uniform(-0.3, -0.01)), float(r.uniform(0.01, 0.3))]
        if t == SPHERICAL and r.random() < 0.6:
            kw["twist_limit"] = [float(r.uniform(-0.2, -0.01)), float(r.uniform(0.01, 0.2))]
        if t == DISTANCE:
            lo = float(np.linalg.norm(off) + r.uniform(-0.1, 0.1))
            kw["limit_min"], kw["limit_max"] = lo, lo + float(r.choice([0.0, r.uniform(0.0, 0.1)]))
        if r.random() < damping_share:
            kw["damping"] = [float(r.uniform(0.0, 2.0)), float(r.uniform(0.0, 3.0))]
        kw.update(override)
        return self.joint(t, b1, b2, a1, a2, **kw)

    def done(self):
        # worked.py solves type by type in table order; the ABI columns are per type: keep the list type-major like both
        self.joints.sort(key=lambda j: j["type"])
        return {"params": self.params, "bodies": self.bodies, "joints": self.joints}


def _features(seed, substeps):
    s = _Scene(seed, substeps)
    B = s.body
    still = dict(gravity_scale=0.0)                   # no motion before the joint pass: the "exact" joints stay exactly where they are put
    st = [B(STATIC, (x, 3.0, 0.0), axis_angle((1, 0, 0), 0.1 * x)) for x in range(4)]
    # -- the revolute angle limit: obtuse branch with and without the phi > pi wrap, a limit that holds, one beyond a limit (acute)
    for ang, lim in ((-2.5, [-0.5, 0.5]), (2.5, [-0.5, 0.5]), (0.2, [-0.5, 0.5]), (0.9, [-0.4, 0.4])):
        b = B(DYNAMIC, (0.6, 3.0, 0.0), axis_angle((0, 0, 1), ang), w=(0.1, -0.2, 0.3))
        s.joint(REVOLUTE, st[0], b, (0.3, 0, 0), (-0.3, 0, 0), angle_limit=lim, compliance1=0.0, compliance2=1e-4)
    # -- spherical swing / twist: beyond both limits, the twist with dot(a1, a2) <= -0.5 (swing axes 2.3 rad apart), limits that hold
    for rot in (axis_angle((0, 0, 1), 1.0), axis_angle((1, 0, 0), 2.3), axis_angle((0, 1, 0), 0.1)):
        b = B(DYNAMIC, (0.0, 2.2, 0.3), rot, w=(0.3, 0.0, -0.2), inv_mass=0.8)
        s.joint(SPHERICAL, st[1], b, (0, -0.4, 0), (0, 0.4, 0), swing_limit=[-0.4, 0.4], twist_limit=[-0.3, 0.3], compliance1=1e-4)
    # the spherical normalisation exits, on bodies that sit on their static partner and do not move: equal swing axes (|a1 x a2| = 0) and,
    # through a half turn about the twist axis in local_basis2, opposite swing axes (|a1 + a2| = 0)
    b = B(DYNAMIC, s.bodies[st[2]]["position"], s.bodies[st[2]]["rotation"], **still)
    s.joint(SPHERICAL, st[2], b, swing_limit=[-0.4, 0.4])
    b = B(DYNAMIC, s.bodies[st[3]]["position"], s.bodies[st[3]]["rotation"], **still)
    s.joint(SPHERICAL, st[3], b, local_basis2=[0.0, 1.0, 0.0, 0.0], twist_limit=[-0.3, 0.3])
    # -- fixed: aligned (align_orientation's angle <= eps) with coincident anchors (point_solve's |sep| = 0), and a misaligned one
    p = s.bodies[st[0]]["position"]
    b = B(DYNAMIC, p, s.bodies[st[0]]["rotation"], **still)
    s.joint(FIXED, st[0], b, compliance1=1e-4)
    b = B(DYNAMIC, (0.1, 2.4, 0.4), axis_angle((1, 1, 0), 0.4))
    s.joint(FIXED, st[2], b, (0, -0.3, 0), (0, 0.3, 0.1), compliance0=1e-4)
    # -- prismatic: beyond the slider limit, within it and on the axis (no correction), limit off
    for off, lim, still_kw in (((0.8, 0.05, -0.03), [-0.2, 0.3], {}), ((0.2, 0.0, 0.0), [-0.2, 0.3], still), ((0.5, 0.1, 0.0), None, {})):
        b = B(DYNAMIC, np.array(s.bodies[st[0]]["position"]) + off, IDENTITY, **still_kw)   # st[0] is not rotated: the offsets are exact
        s.joint(PRISMATIC, st[0], b, **({"limits": lim} if lim else {}), compliance1=1e-5)
    # -- distance: below min, above max, inside, coincident anchors
    for d, lo, hi, still_kw in ((0.3, 0.6, 0.8, {}), (1.2, 0.6, 0.8, {}), (0.7, 0.6, 0.8, {}), (0.0, 0.0, 0.5, still)):
        b = B(DYNAMIC, (9.0 + d, 0.0, 0.0), v=(0.0, 0.1, 0.0), **still_kw)
        a = B(STATIC, (9.0, 0.0, 0.0)) if d else None
        if d:
            s.joint(DISTANCE, a, b, limit_min=lo, limit_max=hi, compliance0=float(d > 1.0) * 1e-4)
        else:
            s.joint(DISTANCE, b, B(STATIC, (9.0, 0.0, 0.0)), limit_min=lo, limit_max=hi)   # static on side 2
    # -- static on both sides
    s.joint(REVOLUTE, st[2], st[3], (0.5, 0, 0), (-0.5, 0, 0), damping=[0.5, 1.0])
    # -- dominance: x (dominance -1) is dominated by y (0) in one joint and written by z (-1) in the next; w (+1) dominates x
    x = B(DYNAMIC, (-3.0, 0.0, 0.0), w=(0.0, 1.0, 0.0), dominance=-1)
    y = B(DYNAMIC, (-2.2, 0.1, 0.0), dominance=0)
    z = B(DYNAMIC, (-3.0, -0.8, 0.2), dominance=-1)
    w_ = B(DYNAMIC, (-3.9, 0.0, 0.0), dominance=1)
    s.joint(SPHERICAL, x, y, (0.4, 0, 0), (-0.4, 0, 0))
    s.joint(SPHERICAL, z, x, (0, 0.4, 0), (0, -0.4, 0), damping=[0.3, 0.6])
    s.joint(REVOLUTE, w_, x, (0.45, 0, 0), (-0.45, 0, 0))
    # -- a moving kinematic body under damping, on either side
    k = B(KINEMATIC, (-6.0, 1.0, 0.0), v=(0.5, 0.0, -0.2), w=(0.0, 0.8, 0.3))
    s.random_joint(DISTANCE, k, s.random_body(near=k), damping=[1.0, 2.0])
    s.random_joint(FIXED, s.random_body(near=k), k, damping=[0.7, 1.5])
    # -- joint_damping's dummy carry: damped joints of one type whose static end is on the same side, on different static bodies
    for t in (REVOLUTE, DISTANCE):
        for i in range(3):
            s.random_joint(t, st[i], s.random_body(near=st[i]), damping=[0.6 + 0.2 * i, 1.0 + i])
        for i in range(2):
            s.random_joint(t, s.random_body(near=st[3 - i]), st[3 - i], damping=[0.4, 2.0 + i])
    # -- random joints of every type over a shared pool: the levels interleave the five types
    pool = [s.random_body() for _ in range(40)]
    for t in (FIXED, REVOLUTE, SPHERICAL, PRISMATIC, DISTANCE):
        for _ in range(14):
            b1, b2 = s.rng.choice(pool, 2, replace=False)
            s.random_joint(t, b1, b2)
    return s.done()


def _hub(seed):
    s = _Scene(seed, 1)
    hub = s.body(KINEMATIC, (0.0, 0.0, 0.0), axis_angle((1, 1, 1), 0.3), v=(0.2, 0.0, 0.1), w=(0.0, 0.5, 0.0))
    for i in range(48):
        t = (SPHERICAL, REVOLUTE, FIXED, DISTANCE)[i % 4]
        b = s.random_body()
        s.bodies[b]["dominance"] = 0
        s.random_joint(t, hub, b, damping_share=0.0) if i % 2 else s.random_joint(t, b, hub, damping_share=0.0)
    return s.done()


def _chain(seed, links=2500):
    s = _Scene(seed, 1)
    prev = s.body(STATIC, (0.0, 0.0, 0.0))
    for i in range(links):
        b = s.body(DYNAMIC, (0.0, -0.5 * (i + 1), 0.0), axis_angle((0, 0, 1), 0.01 * (i % 7)), w=(0.0, 0.0, 0.2), inv_mass=1.0)
        s.joint(SPHERICAL, prev, b, (0, -0.25, 0), (0, 0.25, 0), compliance0=1e-6, damping=[0.2, 0.5],
                **({"swing_limit": [-0.05, 0.05]} if i % 3 == 0 else {}))
        prev = b
    return s.done()


def _wide(seed, n=70000):
    s = _Scene(seed, 1)
    anchor = s.body(STATIC, (0.0, 10.0, 0.0))
    r = s.rng
    pos = r.uniform(-1.0, 1.0, (n, 3)) + np.array([0.0, 9.0, 0.0])
    vel = r.uniform(-1.0, 1.0, (n, 3))
    for i in range(n):
        b = s.body(DYNAMIC, pos[i], IDENTITY, vel[i], (0, 0, 0), 1.0)
        s.joint(DISTANCE, anchor, b, (0, 0, 0), (0.1, 0.0, 0.0), limit_min=0.9, limit_max=1.1)
    return s.done()


FAMILIES = {
    "features": lambda: _features(1, 4),
    "features_sub12": lambda: _features(2, 12),
    "hub": lambda: _hub(3),
    "chain": lambda: _chain(4),
    "wide": lambda: _wide(5),
}
_cache: dict = {}


def family(name: str) -> dict:
    if name not in _cache:
        _cache[name] = FAMILIES[name]()
    return _cache[name]


def columns(scene: dict, dtype):
    """(params, api.Bodies, api.JointSet, where): where[k] = (k, type, index in that type's columns) of joint k of the scene"""
    prm, b, _, j, where = _build(scene, dtype)
    return prm, b, j, where


SHAPE_KEYS = ("solve_levels", "damp_levels", "widest_level", "types_in_one_level", "hub_joints")


def _levels(items, n_res):
    """order-preserving levels: item (r1, r2) goes one past the last level of any earlier item on r1 or r2 (None = no resource)"""
    last, out = [0] * n_res, []
    for r1, r2 in items:
        lv = max([last[r] for r in (r1, r2) if r is not None] + [0])
        for r in (r1, r2):
            if r is not None:
                last[r] = lv + 1
        out.append(lv)
    return out


def _np_rot(q, v):
    return _rot(np.array(q, dtype=float), np.array(v, dtype=float))


def census(scene: dict) -> dict:
    """counts, from the scene data, of the branches, body sides and schedule shapes the scene reaches (module docstring).  The joint
    geometry is evaluated at the input poses, with the reference's formulas (prepare + the first solve of each joint)."""
    bodies, joints = scene["bodies"], scene["joints"]
    kind = [b["kind"] for b in bodies]
    has_sb = [k != STATIC for k in kind]
    dom = [b.get("dominance", 0) if k == DYNAMIC else 128 for b, k in zip(bodies, kind)]
    c = {k: 0 for k in ("fixed", "revolute", "spherical", "prismatic", "distance", "angle_limit_beyond", "angle_limit_holds", "angle_obtuse",
                        "angle_wrap", "swing_limit", "twist_limit", "twist_max_corr_h", "slider_limit", "limit_off", "distance_below",
                        "distance_above", "distance_inside", "align_exit", "point_exit", "prismatic_exit", "distance_exit", "swing_norm_exit",
                        "twist_norm_exit", "compliance_zero", "compliance_nonzero", "damped", "undamped", "static_side1", "static_side2",
                        "static_both", "dominance_pos", "dominance_neg", "dominated_and_written", "kinematic_damped_moving",
                        "com_offset", "full_inertia", "locked_axes", "dummy_carry_side1", "dummy_carry_side2")}
    names = ("fixed", "revolute", "spherical", "prismatic", "distance")
    eps = np.finfo(np.float64).eps
    pos = [np.array(b["position"]) for b in bodies]
    rot = [np.array(b["rotation"]) for b in bodies]
    per_side = {}
    written_by, dominated_in = set(), set()
    for j in joints:
        t, i1, i2 = j["type"], j["body1"], j["body2"]
        c[names[t]] += 1
        comp = [j.get(k, 0.0) for k in ("compliance0", "compliance1", "compliance2")]
        c["compliance_zero"] += any(x == 0 for x in comp)
        c["compliance_nonzero"] += any(x != 0 for x in comp)
        damped = j.get("damping") is not None
        c["damped" if damped else "undamped"] += 1
        c["static_side1"] += (not has_sb[i1]) and has_sb[i2]
        c["static_side2"] += has_sb[i1] and not has_sb[i2]
        c["static_both"] += not has_sb[i1] and not has_sb[i2]
        rel = dom[i1] - dom[i2]
        for i, dominated in ((i1, rel > 0), (i2, rel < 0)):
            if kind[i] == DYNAMIC:
                (dominated_in if dominated else written_by).add(i)
        if damped:
            for side, i in ((1, i1), (2, i2)):
                if not has_sb[i]:
                    per_side[(t, side)] = per_side.get((t, side), 0) + 1
                if kind[i] == KINEMATIC and (any(bodies[i]["linear_velocity"]) or any(bodies[i]["angular_velocity"])):
                    c["kinematic_damped_moving"] += 1
        la1, la2 = np.array(j["local_anchor1"]), np.array(j["local_anchor2"])
        sep = (pos[i2] + _np_rot(rot[i2], la2)) - (pos[i1] + _np_rot(rot[i1], la1))
        f1 = _mul(rot[i1], np.array(j.get("local_basis1", IDENTITY)))
        f2 = _mul(rot[i2], np.array(j.get("local_basis2", IDENTITY)))
        axis = np.array(j.get("axis", DEFAULT_AXIS[t]), dtype=float)
        if t in (FIXED, PRISMATIC):
            c["align_exit"] += bool(np.linalg.norm(_mul(f1, _conj(f2))[:3]) <= eps)
        if t in (FIXED, REVOLUTE, SPHERICAL):
            c["point_exit"] += bool(sep @ sep == 0)
        lim = j.get(LIMIT_KEY.get(t, ""))
        if t in LIMIT_KEY and lim is None and not (t == SPHERICAL and j.get("twist_limit") is not None):
            c["limit_off"] += 1
        if t == REVOLUTE and lim is not None:
            ortho = _any_orthonormal(axis)
            a1, b1, b2 = _np_rot(f1, axis), _np_rot(f1, ortho), _np_rot(f2, ortho)
            phi = math.asin(max(-1.0, min(1.0, np.cross(b1, b2) @ a1)))
            if b1 @ b2 < 0:
                c["angle_obtuse"] += 1
                phi = math.pi - phi
            if phi > math.pi:
                c["angle_wrap"] += 1
                phi -= 2 * math.pi
            c["angle_limit_beyond" if (phi < lim[0] or phi > lim[1]) else "angle_limit_holds"] += 1
        if t == SPHERICAL:
            swing = _any_orthonormal(axis)
            a1, a2 = _np_rot(f1, swing), _np_rot(f2, swing)
            if lim is not None:
                c["swing_limit"] += 1
                c["swing_norm_exit"] += bool(np.linalg.norm(np.cross(a1, a2)) <= eps)
            if j.get("twist_limit") is not None:
                c["twist_limit"] += 1
                c["twist_norm_exit"] += bool(np.linalg.norm(a1 + a2) <= eps)
                c["twist_max_corr_h"] += bool(a1 @ a2 <= -0.5)
        if t == PRISMATIC:
            a1 = _np_rot(f1, axis)
            a = sep @ a1
            off_axis = sep - a * a1
            beyond = lim is not None and (a < lim[0] or a > lim[1])
            c["slider_limit"] += beyond
            c["prismatic_exit"] += bool(not beyond and np.linalg.norm(off_axis) == 0)
        if t == DISTANCE:
            d = float(np.linalg.norm(sep))
            if d * d <= eps:
                c["distance_exit"] += 1
            else:
                c["distance_below" if d < j["limit_min"] else ("distance_above" if d > j["limit_max"] else "distance_inside")] += 1
    c["dummy_carry_side1"] = sum(1 for (t, side), n in per_side.items() if side == 1 and n >= 2)
    c["dummy_carry_side2"] = sum(1 for (t, side), n in per_side.items() if side == 2 and n >= 2)
    c["dominated_and_written"] = len(written_by & dominated_in)
    c["dominance_pos"] = sum(1 for b, k in zip(bodies, kind) if k == DYNAMIC and b.get("dominance", 0) > 0)
    c["dominance_neg"] = sum(1 for b, k in zip(bodies, kind) if k == DYNAMIC and b.get("dominance", 0) < 0)
    c["com_offset"] = sum(1 for b in bodies if any(b.get("center_of_mass", [0, 0, 0])))
    c["full_inertia"] = sum(1 for b in bodies if any(b["inverse_inertia_local"][k] for k in (1, 2, 4)))
    c["locked_axes"] = sum(1 for b in bodies if b.get("locked_axes", 0))
    # the level schedules (avian_b200/csrc/joint_schedule.hpp): a body orders the solve iff a joint writes it; damping writes every
    # SolverBody and the two dummies of each type
    any_damping = any(j.get("damping") is not None for j in joints)
    conflict = [False] * len(bodies)
    for j in joints:
        rel = dom[j["body1"]] - dom[j["body2"]]
        conflict[j["body1"]] |= has_sb[j["body1"]] and (any_damping or not rel > 0)
        conflict[j["body2"]] |= has_sb[j["body2"]] and (any_damping or not rel < 0)
    lv = _levels([tuple(i if conflict[i] else None for i in (j["body1"], j["body2"])) for j in joints], len(bodies))
    B = len(bodies)
    dl = _levels([(j["body1"] if has_sb[j["body1"]] else B + 2 * j["type"], j["body2"] if has_sb[j["body2"]] else B + 2 * j["type"] + 1)
                  for j in joints if j.get("damping") is not None], B + 10)
    c["solve_levels"] = max(lv) + 1 if lv else 0
    c["damp_levels"] = max(dl) + 1 if dl else 0
    c["widest_level"] = int(np.bincount(lv).max()) if lv else 0
    types_per_level = {}
    for j, l in zip(joints, lv):
        types_per_level.setdefault(l, set()).add(j["type"])
    c["types_in_one_level"] = max((len(v) for v in types_per_level.values()), default=0)
    hubs = [i for i in range(B) if kind[i] == KINEMATIC]
    c["hub_joints"] = max((sum(1 for j, l in zip(joints, lv) if l == 0 and i in (j["body1"], j["body2"])) for i in hubs), default=0)
    return c


def _any_orthonormal(v):   # glam Vec3::any_orthonormal_vector
    sign = math.copysign(1.0, v[2])
    a = -1.0 / (sign + v[2])
    b = v[0] * v[1] * a
    return np.array([b, sign + v[1] * v[1] * a, -v[1]])
