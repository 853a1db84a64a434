"""Seeded solver inputs for the wavefront feature tests: `api.Bodies` / `api.Manifolds` built directly, without the narrow phase.

The geometry is only plausible (unit normals, anchors inside a unit body, penetrations of a few centimetres, some separated / speculative
points); what the generator controls is everything the solver stage reads per body and per manifold, and the shape of the colouring:

* bodies: isotropic, diagonal and full (off-diagonal) local inverse inertia, every LockedAxes bit, integration_flags 0..3, finite and
  infinite speed limits, damping, gravity scale, accelerations, centre-of-mass offsets, positive and negative dominance;
* kinds: dynamic, kinematic (shared by many manifolds), static by index and static as AVN_NO_BODY, kinematic-static and kinematic-kinematic
  manifolds (both sides non-dynamic: the solver skips them, the colouring does not);
* manifolds: 1..4 points (or at most one point for the sphere-only variant), friction 0 and > 0 with a tangent velocity, restitution with
  normal speeds on both sides of the threshold;
* optional columns: each one can be left out (None);
* schedule shapes: colour lengths around the 32-wide chunk, empty colours between full ones, a hub body in all 23 colours.

The manifolds are coloured in ascending index by the reference's rule (ConstraintGraph::push_manifold, solver/constraint_graph.rs:163-238):
a pair of two non-static bodies takes the lowest colour in 0..19 free on both; a pair with a static side takes the highest colour in
22..1 free on the other body; static bodies (kind static, or no body at all) carry no colour bits, kinematic bodies do; what finds no
free colour goes to the overflow colour 23.  A candidate that would overflow is left out, so the overflow colour stays empty and the
wavefront schedule is selectable.  The manifolds are then laid out colour by colour, in index order within a colour.

`Scene.columns(dtype)` gives the ABI columns, `Scene.worked()` the dict `tests/golden/handworked/worked.py` evaluates (the same values,
rounded into the working precision the same way).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from avian_b200 import api

DYNAMIC, KINEMATIC, STATIC = api.BODY_DYNAMIC, api.BODY_KINEMATIC, api.BODY_STATIC
OVERFLOW, DYNAMIC_COLOURS = 23, 20
OPTIONAL_BODY = ("center_of_mass", "locked_axes", "dominance", "linear_damping", "angular_damping", "gravity_scale", "linear_acceleration",
                 "angular_acceleration", "max_linear_speed", "max_angular_speed", "integration_flags")


def push_colour(bits, b1, b2, s1, s2):
    """the colour of one manifold by the rule in the module docstring; updates the colour bits of its non-static bodies"""
    if not s1 and not s2:
        for c in range(DYNAMIC_COLOURS):
            if not (bits[b1] >> c) & 1 and not (bits[b2] >> c) & 1:
                bits[b1] |= 1 << c
                bits[b2] |= 1 << c
                return c
        return OVERFLOW
    if s1 and s2:
        return OVERFLOW
    b = b2 if s1 else b1
    for c in range(OVERFLOW - 1, 0, -1):
        if not (bits[b] >> c) & 1:
            bits[b] |= 1 << c
            return c
    return OVERFLOW


@dataclass
class Scene:
    params: dict
    bodies: dict                      # column name -> float64 / integer numpy array (optional columns may be None)
    manifolds: dict                   # column name -> numpy array, laid out by colour; "points" is the per-manifold point count
    colour: np.ndarray                # colour of every manifold (after the layout)
    hub: int | None = None

    @property
    def body_count(self) -> int:
        return int(self.bodies["position"].shape[0])

    def step_params(self) -> api.AvnStepParams:
        p = self.params
        prm = api.default_step_params()
        prm.dt, prm.h, prm.substeps = p["dt"], p["h"], p["substeps"]
        for k in ("restitution_iterations", "contact_damping_ratio", "contact_frequency_factor", "max_overlap_solve_speed", "warm_start_coefficient",
                  "restitution_threshold", "length_unit", "match_contacts", "solver_iterations"):
            setattr(prm, k, p[k])
        prm.gravity[0], prm.gravity[1], prm.gravity[2] = p["gravity"]
        return prm

    def columns(self, dtype):
        """(params, api.Bodies, api.Manifolds) in the scalar type `dtype`"""
        s = np.dtype(dtype)
        bd = self.bodies
        cast = lambda a: None if a is None else (a.astype(s) if a.dtype.kind == "f" else a.copy())
        bodies = api.Bodies(**{k: cast(v) for k, v in bd.items()})
        md = self.manifolds
        co = np.zeros(api.GRAPH_COLOR_COUNT + 1, dtype=np.uint32)
        co[1:] = np.cumsum(np.bincount(self.colour, minlength=api.GRAPH_COLOR_COUNT))
        P = int(md["anchor1"].shape[0])
        man = api.Manifolds(
            color_offsets=co, body1=md["body1"].astype(np.int32), body2=md["body2"].astype(np.int32), normal=md["normal"].astype(s),
            friction=md["friction"].astype(s), restitution=md["restitution"].astype(s),
            point_offsets=np.concatenate([[0], np.cumsum(md["points"])]).astype(np.uint32), anchor1=md["anchor1"].astype(s),
            anchor2=md["anchor2"].astype(s), penetration=md["penetration"].astype(s), normal_speed=md["normal_speed"].astype(s),
            warm_start_normal_impulse=md["warm_start_normal_impulse"].astype(s), warm_start_tangent_impulse=md["warm_start_tangent_impulse"].astype(s),
            normal_impulse=np.zeros(P, dtype=s), tangent_velocity=cast(md.get("tangent_velocity")))
        return self.step_params(), bodies, man

    def worked(self) -> dict:
        """the same scene as worked.py's input dict (an absent optional column is an absent key)"""
        bd, md = self.bodies, self.manifolds
        bodies = []
        for i in range(self.body_count):
            b = {"kind": int(bd["kind"][i])}
            for k in ("position", "rotation", "linear_velocity", "angular_velocity", "inverse_inertia_local"):
                b[k] = [float(x) for x in bd[k][i]]
            b["inverse_mass"] = float(bd["inverse_mass"][i])
            for k in OPTIONAL_BODY:
                v = bd.get(k)
                if v is None:
                    continue
                if k in ("max_linear_speed", "max_angular_speed"):
                    b[k] = float(v[i])           # +inf reaches worked.py as inf: `l2 > inf * inf` never clamps, as in the reference
                elif v.ndim == 2:
                    b[k] = [float(x) for x in v[i]]
                elif v.dtype.kind == "f":
                    b[k] = float(v[i])
                else:
                    b[k] = int(v[i])
            bodies.append(b)
        po = np.concatenate([[0], np.cumsum(md["points"])])
        tv = md.get("tangent_velocity")
        manifolds = []
        for k in range(len(md["body1"])):
            pts = [{"anchor1": [float(x) for x in md["anchor1"][p]], "anchor2": [float(x) for x in md["anchor2"][p]],
                    "penetration": float(md["penetration"][p]), "normal_speed": float(md["normal_speed"][p]),
                    "warm_start_normal_impulse": float(md["warm_start_normal_impulse"][p]),
                    "warm_start_tangent_impulse": [float(x) for x in md["warm_start_tangent_impulse"][p]]} for p in range(po[k], po[k + 1])]
            m = {"body1": int(md["body1"][k]), "body2": int(md["body2"][k]), "normal": [float(x) for x in md["normal"][k]],
                 "friction": float(md["friction"][k]), "restitution": float(md["restitution"][k]), "points": pts}
            if tv is not None:
                m["tangent_velocity"] = [float(x) for x in tv[k]]
            manifolds.append(m)
        co = [0] + np.cumsum(np.bincount(self.colour, minlength=api.GRAPH_COLOR_COUNT)).tolist()
        return {"params": dict(self.params), "bodies": bodies, "manifolds": manifolds, "color_offsets": co}


def step_params_dict(substeps=4, solver_iterations=1, restitution_iterations=1, match_contacts=1, warm_start_coefficient=1.0, dt=1.0 / 60.0):
    dt_ns = round(dt * 1e9)                                   # Duration arithmetic in integer nanoseconds (solver/schedule.rs:195-200)
    h_ns = round(dt_ns / 1e9 / substeps * 1e9)
    return {"dt": dt_ns / 1e9, "h": h_ns / 1e9, "substeps": substeps, "gravity": [0.0, -9.81, 0.0], "contact_damping_ratio": 10.0,
            "contact_frequency_factor": 1.5, "max_overlap_solve_speed": 4.0, "warm_start_coefficient": warm_start_coefficient,
            "restitution_threshold": 1.0, "restitution_iterations": restitution_iterations, "length_unit": 1.0, "match_contacts": match_contacts,
            "solver_iterations": solver_iterations}


def _unit(rng, n):
    v = rng.normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _quats(rng, n):
    q = rng.normal(size=(n, 4))
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def _inverse_inertia(rng, kinds):
    """per body: isotropic, diagonal anisotropic or a full symmetric tensor R diag R^T (m00, m01, m02, m11, m12, m22)"""
    out = np.zeros((len(kinds), 6))
    for i, k in enumerate(kinds):
        if k != DYNAMIC:
            continue
        d = rng.uniform(0.5, 8.0, 3)
        form = rng.integers(3)
        if form == 0:
            out[i] = [d[0], 0, 0, d[0], 0, d[0]]
        elif form == 1:
            out[i] = [d[0], 0, 0, d[1], 0, d[2]]
        else:
            q = _quats(rng, 1)[0]
            x, y, z, w = q
            R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                          [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                          [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
            M = R @ np.diag(d) @ R.T
            out[i] = [M[0, 0], M[0, 1], M[0, 2], M[1, 1], M[1, 2], M[2, 2]]
    return out


def _bodies(rng, kinds, optional):
    """body columns; `optional` = True (all optional columns), False (none) or a set of names"""
    n = len(kinds)
    dyn = kinds == DYNAMIC
    bd = {"kind": kinds.astype(np.uint8), "position": rng.uniform(-20, 20, (n, 3)), "rotation": _quats(rng, n),
          "linear_velocity": rng.uniform(-2, 2, (n, 3)), "angular_velocity": rng.uniform(-3, 3, (n, 3)),
          "inverse_mass": np.where(dyn, rng.uniform(0.2, 2.0, n), 0.0), "inverse_inertia_local": _inverse_inertia(rng, kinds)}
    static = kinds == STATIC
    bd["linear_velocity"][static] = 0.0
    bd["angular_velocity"][static] = 0.0
    # every LockedAxes pattern: none, single bits, all rotation (no gyroscopic torque), all six, random
    locked = rng.choice([0, 0, 0, 0x20, 0x10, 0x08, 0x04, 0x02, 0x01, 0x07, 0x38, 0x3F, 0x22, 0x15], n)
    flags = rng.choice([0, 0, 0, 0, 1, 2, 3], n)
    max_lin = np.where(rng.random(n) < 0.5, rng.uniform(0.3, 2.5, n), np.inf)
    max_ang = np.where(rng.random(n) < 0.5, rng.uniform(0.5, 3.0, n), np.inf)
    cols = {
        "center_of_mass": rng.uniform(-0.2, 0.2, (n, 3)), "locked_axes": locked.astype(np.uint8),
        "dominance": np.where(dyn, rng.choice([0, 0, 0, 1, -1, 3, -4], n), 0).astype(np.int8),
        "linear_damping": rng.choice([0.0, 0.3, 2.0], n), "angular_damping": rng.choice([0.0, 0.5, 3.0], n),
        "gravity_scale": rng.choice([1.0, 1.0, 0.0, 0.5, -1.5], n), "linear_acceleration": rng.uniform(-5, 5, (n, 3)),
        "angular_acceleration": rng.uniform(-4, 4, (n, 3)), "max_linear_speed": max_lin, "max_angular_speed": max_ang,
        "integration_flags": flags.astype(np.uint8)}
    for k in OPTIONAL_BODY:
        on = optional is True or (optional and k in optional)
        bd[k] = cols[k] if on else None
    return bd


def _colour(candidates, is_static, n_bodies):
    """colours the candidate pairs in ascending index; drops the ones that would overflow; returns (kept pairs, their colours)"""
    bits = [0] * (n_bodies + 1)            # slot n_bodies stands for AVN_NO_BODY (never used: static sides carry no bits)
    kept, colours = [], []
    for b1, b2 in candidates:
        s1 = b1 < 0 or is_static[b1]
        s2 = b2 < 0 or is_static[b2]
        c = push_colour(bits, b1, b2, s1, s2)
        if c == OVERFLOW:
            continue
        kept.append((b1, b2))
        colours.append(c)
    return kept, np.array(colours, dtype=np.int64)


def _manifolds(rng, pairs, colours, max_points, tangent_velocity, friction_share=0.6, restitution_share=0.5):
    """the manifold and point columns of the coloured pairs, laid out by colour (stable within a colour)"""
    order = np.argsort(colours, kind="stable")
    pairs = [pairs[i] for i in order]
    colours = colours[order]
    M = len(pairs)
    npts = rng.integers(1, max_points + 1, M) if max_points > 1 else np.ones(M, dtype=np.int64)
    P = int(npts.sum())
    md = {"body1": np.array([p[0] for p in pairs], dtype=np.int32).reshape(M), "body2": np.array([p[1] for p in pairs], dtype=np.int32).reshape(M),
          "normal": _unit(rng, M), "friction": np.where(rng.random(M) < friction_share, rng.uniform(0.1, 0.9, M), 0.0),
          "restitution": np.where(rng.random(M) < restitution_share, rng.uniform(0.1, 0.8, M), 0.0), "points": npts,
          "anchor1": rng.uniform(-0.5, 0.5, (P, 3)), "anchor2": rng.uniform(-0.5, 0.5, (P, 3)),
          # penetration < 0: separated by up to 5 cm (speculative branch); > 0: up to 2 cm overlap (bias branch)
          "penetration": rng.uniform(-0.05, 0.02, P),
          # the restitution threshold is 1 m/s: approach speeds on both sides of it
          "normal_speed": rng.uniform(-3.0, 0.5, P),
          "warm_start_normal_impulse": np.where(rng.random(P) < 0.7, rng.uniform(0.0, 0.3, P), 0.0),
          "warm_start_tangent_impulse": rng.uniform(-0.05, 0.05, (P, 2))}
    if tangent_velocity:
        md["tangent_velocity"] = np.where(rng.random((M, 1)) < 0.5, rng.uniform(-0.5, 0.5, (M, 3)), 0.0)
    return md, colours


def generate(seed: int, *, dynamic: int, kinematic: int = 0, static: int = 0, pairs: int = 0, static_contacts=0, no_body_contacts=0,
             kinematic_pairs: int = 0, hub: str | None = None, colour_shape=None, max_points: int = 4, optional=True, tangent_velocity=True,
             **params) -> Scene:
    """One scene.  Bodies are laid out dynamic, kinematic, static (a hub, when asked for, is body 0).  Candidate manifolds, in index order:
    the hub's 20 dynamic neighbours and 3 static contacts; the `colour_shape` static contacts; `pairs` random pairs among dynamic and
    kinematic bodies; `kinematic_pairs` kinematic-kinematic and kinematic-static pairs; `static_contacts` dynamic-static pairs through a
    static body index and `no_body_contacts` through AVN_NO_BODY.  `params` go to step_params_dict.

    hub: "dynamic" or "kinematic" — body 0 meets 20 dynamic bodies (colours 0..19) and 3 static bodies (colours 22, 21, 20).
    colour_shape: per-body counts of static contacts; the j-th contact of a body takes colour 22 - j, so colour 22 - j holds as many
    manifolds as there are counts greater than j."""
    rng = np.random.default_rng(seed)
    n_dyn, n_kin, n_st = dynamic, kinematic, static
    kinds = np.array([DYNAMIC] * n_dyn + [KINEMATIC] * n_kin + [STATIC] * n_st, dtype=np.int64)
    hub_index = None
    if hub is not None:
        assert n_dyn >= 21 and n_st >= 3
        hub_index = 0
        kinds[0] = DYNAMIC if hub == "dynamic" else KINEMATIC
    B = len(kinds)
    is_static = kinds == STATIC
    dyn_ids = np.flatnonzero(kinds == DYNAMIC)
    kin_ids = np.flatnonzero(kinds == KINEMATIC)
    st_ids = np.flatnonzero(is_static)
    movable = np.flatnonzero(~is_static)
    cand = []
    if hub_index is not None:
        nb = [int(x) for x in dyn_ids if x != hub_index][:20]
        cand += [(hub_index, b) if k % 2 else (b, hub_index) for k, b in enumerate(nb)]
        cand += [(hub_index, int(st_ids[k])) for k in range(3)]
    if colour_shape is not None:
        # the j-th static contact of a body takes colour 22 - j; every third one goes through a static body index
        ids = [int(x) for x in dyn_ids if x != hub_index]
        for j in range(max(colour_shape)):
            for b, count in zip(ids, colour_shape):
                if count > j:
                    cand.append((int(st_ids[j % len(st_ids)]), b) if (b + j) % 3 == 0 and len(st_ids) else (b, -1))
    for _ in range(pairs):
        a, b = rng.choice(movable, 2, replace=False)
        cand.append((int(a), int(b)))
    for _ in range(kinematic_pairs):
        if len(kin_ids) >= 2 and rng.random() < 0.5:
            a, b = rng.choice(kin_ids, 2, replace=False)
            cand.append((int(a), int(b)))
        elif len(kin_ids) and len(st_ids):
            cand.append((int(rng.choice(kin_ids)), int(rng.choice(st_ids)) if rng.random() < 0.5 else -1))
    for _ in range(static_contacts):
        d = int(rng.choice(dyn_ids))
        s = int(rng.choice(st_ids))
        cand.append((d, s) if rng.random() < 0.5 else (s, d))
    for _ in range(no_body_contacts):
        d = int(rng.choice(dyn_ids))
        cand.append((d, -1) if rng.random() < 0.5 else (-1, d))
    kept, colours = _colour(cand, is_static, B)
    bd = _bodies(rng, kinds, optional)
    if hub_index is not None and bd.get("dominance") is not None:
        bd["dominance"][hub_index] = 0
    md, colours = _manifolds(rng, kept, colours, max_points, tangent_velocity and optional is not False)
    return Scene(params=step_params_dict(**params), bodies=bd, manifolds=md, colour=colours, hub=hub_index)


def colouring_errors(scene: Scene) -> list[str]:
    """what is wrong with a scene's colouring: a non-static body twice in one colour, an overflow entry, a colour out of range"""
    kinds = scene.bodies["kind"]
    md = scene.manifolds
    errs = []
    for c in range(api.GRAPH_COLOR_COUNT):
        seen = set()
        for k in np.flatnonzero(scene.colour == c):
            if c == OVERFLOW:
                errs.append(f"manifold {k} in the overflow colour")
            for b in (int(md["body1"][k]), int(md["body2"][k])):
                if b < 0 or kinds[b] == STATIC:
                    continue
                if b in seen:
                    errs.append(f"body {b} twice in colour {c}")
                seen.add(b)
    if np.any(np.diff(scene.colour) < 0):
        errs.append("manifolds not laid out by colour")
    return errs


def colours_of(scene: Scene, body: int) -> set[int]:
    md = scene.manifolds
    on = (md["body1"] == body) | (md["body2"] == body)
    return set(int(c) for c in scene.colour[on])


# ---- the scene families ------------------------------------------------------------------------------------------------------------------
# name -> keyword arguments of generate().  Small and medium: worked.py evaluates them on the CPU within seconds.
FAMILIES = {
    # every feature at once, 33 bodies (one past a 32-item chunk), four-point manifolds
    "mixed_b33": dict(seed=1, dynamic=24, kinematic=4, static=5, pairs=40, static_contacts=12, no_body_contacts=6, kinematic_pairs=6,
                      substeps=4, solver_iterations=2, restitution_iterations=3),
    # every optional column absent: the defaults of the ABI
    "absent_b32": dict(seed=2, dynamic=26, kinematic=2, static=4, pairs=36, static_contacts=10, no_body_contacts=4, kinematic_pairs=3,
                       optional=False, substeps=4, solver_iterations=1, match_contacts=0),
    # one hub in all 23 colours; its rank in colour 22 is the largest the colouring allows
    "hub_dynamic_b31": dict(seed=3, dynamic=26, kinematic=2, static=3, pairs=10, static_contacts=4, hub="dynamic", substeps=12,
                            solver_iterations=1, warm_start_coefficient=0.75),
    "hub_kinematic_b33": dict(seed=4, dynamic=27, kinematic=2, static=4, pairs=12, static_contacts=4, kinematic_pairs=4, hub="kinematic",
                              substeps=4, solver_iterations=3, restitution_iterations=2),
    # one body: every manifold meets AVN_NO_BODY (colours 22 down)
    "single_b1": dict(seed=10, dynamic=1, no_body_contacts=6, substeps=1, solver_iterations=2, restitution_iterations=4),
    # colour lengths 64, 33, 32, 31, 1 in colours 22..18, dynamic colours 0.. below, colours in between empty; B = 1000 + 17
    "shapes_b1017": dict(seed=6, dynamic=1000, kinematic=9, static=8, pairs=70,
                         colour_shape=[5] + [4] * 30 + [3] + [2] + [1] * 31, substeps=4, solver_iterations=1, restitution_iterations=2),
    # sphere-only: at most one point per manifold (the MAXP = 1 kernel instances)
    "spheres_b33": dict(seed=7, dynamic=25, kinematic=3, static=5, pairs=40, static_contacts=12, no_body_contacts=6, kinematic_pairs=4,
                        max_points=1, substeps=4, solver_iterations=2, restitution_iterations=2),
}


def family(name: str) -> Scene:
    return generate(**FAMILIES[name])


def feature_census(scene: Scene) -> dict:
    """counts of the features a scene exercises (the tests assert that each family really contains what it is meant to)"""
    bd, md = scene.bodies, scene.manifolds
    kinds = bd["kind"]
    il = bd["inverse_inertia_local"]
    dyn = kinds == DYNAMIC
    off_diag = dyn & ((il[:, 1] != 0) | (il[:, 2] != 0) | (il[:, 4] != 0))
    aniso = dyn & ((il[:, 0] != il[:, 3]) | (il[:, 3] != il[:, 5]) | off_diag)
    locked = bd["locked_axes"] if bd.get("locked_axes") is not None else np.zeros(len(kinds), dtype=np.uint8)
    gyro = aniso & ((locked & 7) != 7)

    def side_kind(b):
        return np.where(b < 0, STATIC, kinds[np.maximum(b, 0)])
    k1, k2 = side_kind(md["body1"]), side_kind(md["body2"])
    both_nondyn = (k1 != DYNAMIC) & (k2 != DYNAMIC)
    return {"gyroscopic": int(gyro.sum()), "off_diagonal": int(off_diag.sum()), "both_non_dynamic": int(both_nondyn.sum()),
            "no_body": int(((md["body1"] < 0) | (md["body2"] < 0)).sum()),
            "static_index": int((((k1 == STATIC) & (md["body1"] >= 0)) | ((k2 == STATIC) & (md["body2"] >= 0))).sum()),
            "kinematic_dynamic": int((((k1 == KINEMATIC) & (k2 == DYNAMIC)) | ((k2 == KINEMATIC) & (k1 == DYNAMIC))).sum()),
            "max_points": int(md["points"].max()), "colours": int(len(set(scene.colour.tolist())))}
