#!/usr/bin/env python
"""Derives tests/golden/handworked/vectors.json: inputs of a few tiny scenes and the results of the hand-worked evaluation (worked.py).

Provenance: produced by worked.py — an independent Python/numpy restatement written from the Rust source — NOT by oracle/ and not by the
CUDA library.  Re-run:  python tests/golden/handworked/derive.py   (pure numpy; no GPU, no compiled code)

Scenes (every branch named is hit at least once, checked by the asserts at the bottom):
  box_on_ground       cube resting 1 cm inside a static ground, 4 points, friction 0.5, warm-start impulses, sliding and spinning:
                      non_dynamic softness, bias branch, relax branch, friction with and without the Coulomb clamp
  sphere_bounce       two dynamic bodies closing at 30 m/s from 0.2 m apart: speculative branch (separation > 0), no friction part,
                      restitution 0.5 above the threshold
  tumbling_body       no constraints: damping, gravity scale, gyroscopic torque of an anisotropic body, centre-of-mass offset in writeback
  distance_pendulum   a body on a distance joint to a static anchor: point correction, velocity projection, JointForces (dt vs h!)
  revolute_pair       two dynamic bodies, misaligned hinge axes: align_orientation then the point constraint
  fixed_pair          fixed joint with a rotation error: fixed-angle constraint then the point constraint
  spherical_dominant  spherical joint (point only) where body 1 has higher Dominance: its inertia is treated as infinite
  revolute_limited    revolute joint bent beyond its angle limit (AngleLimit::compute_correction: asin, clamp, from_axis_angle) + JointDamping
  spherical_limited   spherical joint beyond its swing AND twist limits
  locked_on_kinematic a body with LockedAxes (translation X, rotation Y) in contact with a moving kinematic body
  prismatic_slider    prismatic joint beyond its slider limit and off its axis, with a rotation error: fixed-angle constraint, then the limit
                      along the free axis and the two zero limits along glam's any_orthogonal_vector axes
  damped_static_pair  two damped distance joints, each from a different static body to a spinning body: joint_damping's dummy_body1 carries
                      the first joint's angular increment into the second
  sap_six             six intervals swept by hand (ties on min.x with -0.0/+0.0, touching y bounds, same body, layer mismatch, both inactive)
"""
import json
import math
from pathlib import Path

import numpy as np

import worked as W

HERE = Path(__file__).resolve().parent


def params(substeps, dt=1.0 / 60.0, **kw):
    dt_ns = round(dt * 1e9)                               # Duration arithmetic in integer nanoseconds (solver/schedule.rs:195-200)
    h_ns = round(dt_ns / 1e9 / substeps * 1e9)
    p = {"dt": dt_ns / 1e9, "h": h_ns / 1e9, "substeps": substeps, "gravity": [0.0, -9.81, 0.0], "contact_damping_ratio": 10.0,
         "contact_frequency_factor": 1.5, "max_overlap_solve_speed": 4.0, "warm_start_coefficient": 1.0, "restitution_threshold": 1.0,
         "restitution_iterations": 1, "length_unit": 1.0, "match_contacts": 1}
    p.update(kw)
    return p


def body(kind, pos, rot=(0, 0, 0, 1), v=(0, 0, 0), w=(0, 0, 0), inv_mass=1.0, inv_inertia=(6.0, 0, 0, 6.0, 0, 6.0), **kw):
    n = math.sqrt(sum(x * x for x in rot))
    b = {"kind": kind, "position": list(pos), "rotation": [x / n for x in rot], "linear_velocity": list(v), "angular_velocity": list(w),
         "inverse_mass": inv_mass, "inverse_inertia_local": list(inv_inertia)}
    b.update(kw)
    return b


def axis_angle(axis, angle):
    n = math.sqrt(sum(x * x for x in axis))
    s = math.sin(angle / 2) / n
    return (axis[0] * s, axis[1] * s, axis[2] * s, math.cos(angle / 2))


SCENES = {}

pts = []
for sx, sz, wn, wt in [(0.5, 0.5, 0.04, (0.01, -0.005)), (-0.5, 0.5, 0.03, (0.0, 0.002)), (-0.5, -0.5, 0.05, (-0.004, 0.0)), (0.5, -0.5, 0.02, (0.001, 0.001))]:
    pts.append({"anchor1": [sx, -0.5, sz], "anchor2": [sx, 0.5, sz], "penetration": 0.01, "normal_speed": -0.2, "warm_start_normal_impulse": wn,
                "warm_start_tangent_impulse": list(wt)})
SCENES["box_on_ground"] = {
    "params": params(2),
    "bodies": [body(W.DYNAMIC, (0, 0.49, 0), v=(0.3, -0.2, 0.1), w=(0.05, 0.4, -0.1))],
    "manifolds": [{"body1": 0, "body2": -1, "normal": [0, -1, 0], "friction": 0.5, "restitution": 0.0, "points": pts}],
    "color_offsets": [0] * 23 + [1, 1],                    # dynamic-vs-static: colour 22 (constraint_graph.rs:196-207)
}

SCENES["sphere_bounce"] = {
    "params": params(2),
    "bodies": [body(W.DYNAMIC, (0, 0, 0), inv_mass=0.5, inv_inertia=(5.0, 0, 0, 5.0, 0, 5.0)),
               body(W.DYNAMIC, (0, 1.2, 0), v=(0, -30.0, 0), inv_mass=2.0, inv_inertia=(20.0, 0, 0, 20.0, 0, 20.0), gravity_scale=0.0)],
    "manifolds": [{"body1": 0, "body2": 1, "normal": [0, 1, 0], "friction": 0.0, "restitution": 0.5,
                   "points": [{"anchor1": [0, 0.5, 0], "anchor2": [0, -0.5, 0], "penetration": -0.2, "normal_speed": -30.0,
                               "warm_start_normal_impulse": 0.0, "warm_start_tangent_impulse": [0.0, 0.0]}]}],
    "color_offsets": [0] + [1] * 24,                       # dynamic-vs-dynamic: colour 0
}

SCENES["tumbling_body"] = {
    "params": params(3),
    "bodies": [body(W.DYNAMIC, (1, 2, 3), rot=axis_angle((1, 2, -1), 0.7), v=(0.5, 1.0, -0.25), w=(1.0, 2.0, 3.0), inv_mass=0.8,
                    inv_inertia=(2.0, 0, 0, 1.0, 0, 0.5), center_of_mass=[0.1, -0.05, 0.2], linear_damping=0.3, angular_damping=0.1, gravity_scale=0.5)],
}

SCENES["distance_pendulum"] = {
    "params": params(2),
    "bodies": [body(W.STATIC, (0, 2, 0), inv_mass=0.0, inv_inertia=(0,) * 6),
               body(W.DYNAMIC, (1.2, 2, 0), rot=axis_angle((0, 0, 1), 0.3), v=(0, 0, 0.5), w=(0.2, 0, 0.1), inv_mass=0.5,
                    inv_inertia=(3.0, 0, 0, 3.0, 0, 3.0))],
    "joints": [{"type": W.DISTANCE, "body1": 0, "body2": 1, "local_anchor1": [0, 0, 0], "local_anchor2": [0.1, 0.2, 0], "limit_min": 1.0,
                "limit_max": 1.0, "compliance0": 0.0}],
}

SCENES["revolute_pair"] = {
    "params": params(2),
    "bodies": [body(W.DYNAMIC, (0, 0, 0), w=(0.1, -0.2, 0.3), inv_mass=1.0, inv_inertia=(4.0, 0, 0, 4.0, 0, 4.0)),
               body(W.DYNAMIC, (1.05, 0.02, -0.01), rot=axis_angle((1, 0.2, 0), 0.25), v=(0.1, 0, 0), inv_mass=2.0,
                    inv_inertia=(9.0, 0, 0, 9.0, 0, 9.0))],
    "joints": [{"type": W.REVOLUTE, "body1": 0, "body2": 1, "local_anchor1": [0.5, 0, 0], "local_anchor2": [-0.5, 0, 0], "axis": [0, 0, 1],
                "compliance0": 0.0, "compliance1": 0.0}],
}

SCENES["fixed_pair"] = {
    "params": params(2),
    "bodies": [body(W.DYNAMIC, (0, 1, 0), rot=axis_angle((0, 1, 0), 0.1), inv_mass=1.0, inv_inertia=(6.0, 0, 0, 6.0, 0, 6.0)),
               body(W.DYNAMIC, (0, 0.1, 0.03), rot=axis_angle((1, 1, 0), -0.15), w=(0, 0.5, 0), inv_mass=1.5, inv_inertia=(7.0, 0, 0, 7.0, 0, 7.0))],
    "joints": [{"type": W.FIXED, "body1": 0, "body2": 1, "local_anchor1": [0, -0.5, 0], "local_anchor2": [0, 0.5, 0], "compliance0": 0.0,
                "compliance1": 1e-4}],
}

SCENES["spherical_dominant"] = {
    "params": params(2),
    "bodies": [body(W.DYNAMIC, (0, 0, 0), inv_mass=1.0, dominance=1),
               body(W.DYNAMIC, (0.9, -0.4, 0.1), v=(0, 0.3, 0), inv_mass=1.0, inv_inertia=(8.0, 0, 0, 8.0, 0, 8.0))],
    "joints": [{"type": W.SPHERICAL, "body1": 0, "body2": 1, "local_anchor1": [0.5, 0, 0], "local_anchor2": [-0.5, 0.2, 0], "compliance0": 0.0}],
}

SCENES["revolute_limited"] = {      # the hinge is bent 1.2 rad, the limit allows [-0.5, 0.5]: align + angle limit + point, with joint damping
    "params": params(2),
    "bodies": [body(W.DYNAMIC, (0, 0, 0), inv_mass=1.0, inv_inertia=(4.0, 0, 0, 4.0, 0, 4.0)),
               body(W.DYNAMIC, (0.9, 0.35, 0), rot=axis_angle((0, 0, 1), 1.2), w=(0, 0, 1.5), inv_mass=1.0, inv_inertia=(5.0, 0, 0, 5.0, 0, 5.0))],
    "joints": [{"type": W.REVOLUTE, "body1": 0, "body2": 1, "local_anchor1": [0.5, 0, 0], "local_anchor2": [-0.5, 0, 0], "axis": [0, 0, 1],
                "angle_limit": [-0.5, 0.5], "compliance0": 0.0, "compliance1": 0.0, "compliance2": 0.0, "damping": [0.8, 2.0]}],
}

SCENES["spherical_limited"] = {     # swing 1.0 rad against a 0.4 limit, twist 0.9 rad against 0.3: point, swing limit, twist limit
    "params": params(2),
    "bodies": [body(W.DYNAMIC, (0, 0, 0), inv_mass=0.5, inv_inertia=(3.0, 0, 0, 3.0, 0, 3.0)),
               body(W.DYNAMIC, (0.3, 0.9, 0.1), rot=tuple(W.quat_mul(np.array(axis_angle((0, 0, 1), 1.0)), np.array(axis_angle((0, 1, 0), 0.9)))),
                    w=(0.3, 0.0, -0.2), inv_mass=1.0, inv_inertia=(6.0, 0, 0, 6.0, 0, 6.0))],
    "joints": [{"type": W.SPHERICAL, "body1": 0, "body2": 1, "local_anchor1": [0, 0.5, 0], "local_anchor2": [0, -0.5, 0], "axis": [0, 1, 0],
                "swing_limit": [-0.4, 0.4], "twist_limit": [-0.3, 0.3], "compliance0": 0.0, "compliance1": 0.0, "compliance2": 0.0}],
}

SCENES["prismatic_slider"] = {      # slid 0.5 along the free axis against a [-0.2, 0.3] limit, 0.08 / 0.05 off it, tilted: fixed angle + three axes
    "params": params(2),
    "bodies": [body(W.DYNAMIC, (0, 1, 0), rot=axis_angle((0, 1, 0), 0.2), inv_mass=1.0, inv_inertia=(5.0, 0, 0, 5.0, 0, 5.0)),
               body(W.DYNAMIC, (0.52, 1.08, -0.05), rot=axis_angle((1, 0, 1), 0.15), v=(0.2, 0, 0), w=(0, 0.3, 0.1), inv_mass=2.0,
                    inv_inertia=(9.0, 0, 0, 9.0, 0, 9.0))],
    "joints": [{"type": W.PRISMATIC, "body1": 0, "body2": 1, "local_anchor1": [0.1, 0, 0], "local_anchor2": [-0.1, 0, 0], "axis": [1, 0, 0],
                "limits": [-0.2, 0.3], "compliance0": 0.0, "compliance1": 1e-5}],
}

SCENES["damped_static_pair"] = {    # two damped distance joints, each hanging a spinning body from a DIFFERENT static body: joint_damping's
    "params": params(2),            # dummy_body1 takes the first joint's delta_omega and hands it to the second (one dummy per type and substep)
    "bodies": [body(W.STATIC, (0, 2, 0), inv_mass=0.0, inv_inertia=(0,) * 6),
               body(W.DYNAMIC, (0.9, 2, 0.1), w=(0.5, 2.0, -1.0), inv_mass=1.0, inv_inertia=(4.0, 0, 0, 4.0, 0, 4.0)),
               body(W.DYNAMIC, (3.1, 1.2, 0), rot=axis_angle((0, 1, 1), 0.4), v=(0, 0.2, 0), w=(-1.5, 0.3, 2.5), inv_mass=0.5,
                    inv_inertia=(3.0, 0, 0, 3.0, 0, 3.0)),
               body(W.STATIC, (3, 2, 0), rot=axis_angle((1, 0, 0), 0.3), inv_mass=0.0, inv_inertia=(0,) * 6)],
    "joints": [{"type": W.DISTANCE, "body1": 0, "body2": 1, "local_anchor1": [0, 0, 0], "local_anchor2": [-0.4, 0, 0], "limit_min": 0.5,
                "limit_max": 0.5, "compliance0": 0.0, "damping": [0.5, 3.0]},
               {"type": W.DISTANCE, "body1": 3, "body2": 2, "local_anchor1": [0, -0.2, 0], "local_anchor2": [0, 0.3, 0], "limit_min": 0.2,
                "limit_max": 0.4, "compliance0": 0.0, "damping": [1.0, 4.0]}],
}

kp = []
for sx, sz, wn in [(0.4, 0.4, 0.02), (-0.4, 0.4, 0.0), (-0.4, -0.4, 0.03), (0.4, -0.4, 0.01)]:
    kp.append({"anchor1": [sx, -0.5, sz], "anchor2": [sx + 0.2, 0.25, sz - 0.1], "penetration": 0.004, "normal_speed": -0.05, "warm_start_normal_impulse": wn,
               "warm_start_tangent_impulse": [0.002, -0.001]})
SCENES["locked_on_kinematic"] = {   # a body with translation X and rotation Y locked riding a moving kinematic platform: per-axis inverse mass, cleared inertia
    "params": params(2),            # rows, locked increments, the kinematic side dominant (2x softness frequency) and integrated but never pushed
    "bodies": [body(W.DYNAMIC, (0, 0.996, 0), v=(0.0, -0.1, 0.05), w=(0.2, 0.0, -0.1), inv_mass=1.0, inv_inertia=(6.0, 0, 0, 6.0, 0, 6.0), locked_axes=0b100_010),
               body(W.KINEMATIC, (-0.2, 0.25, 0.1), v=(0.6, 0.0, 0.3), w=(0, 0.2, 0), inv_mass=0.0, inv_inertia=(0,) * 6)],
    "manifolds": [{"body1": 0, "body2": 1, "normal": [0, -1, 0], "friction": 0.6, "restitution": 0.0, "points": kp}],
    "color_offsets": [0] + [1] * 24,   # both bodies have a SolverBody: the dynamic-dynamic rule, colour 0 (constraint_graph.rs:184-195)
}

SAP = {
    "intervals": [
        {"collider": 10, "body": 10, "min": [2.0, 0.0, 0.0], "max": [3.0, 1.0, 1.0], "memberships": 1, "filters": 0xFFFFFFFF, "inactive": True},
        {"collider": 11, "body": 11, "min": [-0.0, 0.0, 0.0], "max": [1.5, 1.0, 1.0], "memberships": 1, "filters": 0xFFFFFFFF, "inactive": False},
        {"collider": 12, "body": 12, "min": [0.0, 0.5, 0.0], "max": [2.0, 1.5, 1.0], "memberships": 1, "filters": 0xFFFFFFFF, "inactive": False},
        {"collider": 13, "body": 11, "min": [1.0, 0.0, 0.0], "max": [2.5, 1.0, 1.0], "memberships": 1, "filters": 0xFFFFFFFF, "inactive": False},
        {"collider": 14, "body": 14, "min": [1.5, 0.0, 0.0], "max": [1.8, 1.0, 1.0], "memberships": 2, "filters": 2, "inactive": False},
        {"collider": 15, "body": 15, "min": [1.5, 1.0, 0.0], "max": [4.0, 2.0, 1.0], "memberships": 1, "filters": 0xFFFFFFFF, "inactive": True},
    ],
    # Worked by hand against broad_phase.rs:373-474 (the derivation is in DESIGN.md §5 and in tests/test_handworked.py):
    # insertion sort by min.x, swapping only on strict '>': 2.0 | -0.0 | 0.0 | 1.0 | 1.5 | 1.5  ->  rows [1, 2, 3, 4, 5, 0]
    # (-0.0 and 0.0 tie and keep their order, so do the two 1.5s).
    "expected_order": [1, 2, 3, 4, 5, 0],
    # sweep: 11: 12 yes | 13 same body | 14 layers | 15 yes (x: 1.5 > 1.5 is false, y touches at 1.0) | 10 break (2.0 > 1.5)
    #        12: 13 yes | 14 layers | 15 yes | 10 yes (2.0 > 2.0 is false; only 10 is inactive)
    #        13: 14 layers | 15 yes | 10 yes        14: 15 layers | 10 break        15: 10 both inactive
    "expected_pairs": [[11, 12], [11, 15], [12, 13], [12, 15], [12, 10], [13, 15], [13, 10]],
}


def main():
    vectors = {"scenes": {}, "sap_six": SAP}
    for name, sc in SCENES.items():
        out32 = W.step(sc, np.float32)
        out64 = W.step(sc, np.float64)
        # the f32 evaluation must agree with the f64 evaluation of the same scene to f32 accuracy: a guard against a scene sitting on a
        # branch boundary (then the two would differ grossly and the scene would be a bad known-answer case)
        for key in ("position", "linear_velocity"):
            for a, b in zip(out32[key], out64[key]):
                assert np.allclose(a, b, rtol=2e-4, atol=2e-4), (name, key, a, b)
        vectors["scenes"][name] = {"input": sc, "expected_f32": out32, "expected_f64": out64}
        print(name, "ok:", {k: out32[k] for k in ("linear_velocity",)})
    pairs, order = W.sweep_and_prune(SAP["intervals"])
    assert [list(p) for p in pairs] == SAP["expected_pairs"], pairs
    assert order == SAP["expected_order"], order
    # branch coverage of the scenes (hand-checked facts the vectors rely on)
    b = vectors["scenes"]["box_on_ground"]["expected_f32"]
    assert sum(x > 0 for x in b["warm_start_normal_impulse"]) >= 2, "box_on_ground: at least two points must carry load"
    assert any(abs(t[0]) + abs(t[1]) > 0 for t in b["warm_start_tangent_impulse"]), "box_on_ground: friction must act"
    s = vectors["scenes"]["sphere_bounce"]["expected_f32"]
    assert s["linear_velocity"][1][1] > 0, "sphere_bounce: restitution must reverse the approach"
    assert s["normal_impulse"][0] > 0
    for nm in ("revolute_limited", "spherical_limited"):
        t = vectors["scenes"][nm]["expected_f32"]["joint_torque"][0]
        assert sum(abs(x) for x in t) > 1.0, f"{nm}: the limits must act"
    lk = vectors["scenes"]["locked_on_kinematic"]["expected_f32"]
    assert lk["linear_velocity"][0][0] == 0.0 and lk["angular_velocity"][0][1] == 0.0, "locked_on_kinematic: the locked axes must not move"
    assert lk["linear_velocity"][1] == [0.6000000238418579, 0.0, 0.30000001192092896], "the kinematic body keeps its velocity"
    assert abs(lk["linear_velocity"][0][2] - 0.05) > 1e-3 and sum(lk["warm_start_normal_impulse"]) > 0, "friction and the normal part must act"
    pz = vectors["scenes"]["prismatic_slider"]["expected_f32"]
    assert abs(pz["joint_force"][0][0]) > 1.0 and sum(abs(x) for x in pz["joint_torque"][0]) > 0.1, "prismatic_slider: limit and angle constraint must act"
    d = vectors["scenes"]["distance_pendulum"]["expected_f32"]
    assert abs(d["joint_force"][0][0]) > 1.0, "distance_pendulum: the joint must pull"
    (HERE / "vectors.json").write_text(json.dumps(vectors, indent=1))
    print("wrote", HERE / "vectors.json")


if __name__ == "__main__":
    main()
