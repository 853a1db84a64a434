"""The hand-worked restatement (tests/golden/handworked/worked.py) against the C++ oracle on the generated joint scenes of
tests/joint_scenes.py: every joint type and limit branch, the `<= eps` exits, compliance, damping, static / kinematic / dominated body sides,
the dummy bodies of joint_damping, and level schedules of one level, thousands of levels and one level wider than the megakernel grid.

Bars: f64 element-wise relative error <= 1e-10 (floor 1) on every column.  f32, with worked.py following glam's SSE2 quaternion product as
the oracle does: positions and rotations at the hand-worked bar of tests/test_handworked.py (1e-5); velocities, joint forces and torques at
1e-5 / h.  Those columns are position differences divided by the substep (project_velocity, JointForces = sum(lambda) * substeps / dt^2),
so the last-bit differences that remain between the two f32 evaluations on generic (rotated-basis, many-substep) joints reach them
multiplied by 1/h: up to 6e-4 in velocity and 2e-3 in force at h = 1/720 s, against the hand-worked bar's 1e-5.

`wide` has 70 000 independent joints: worked.py evaluates every 97th of them (each joint with its own body and the shared static anchor is
a scene of its own, since nothing writes the anchor) and the oracle the whole scene."""
import importlib.util
from pathlib import Path

import numpy as np
import pytest

import joint_scenes as JS
import oracle_lib
from helpers import rel_err

HERE = Path(__file__).resolve().parent / "golden" / "handworked"
_spec = importlib.util.spec_from_file_location("handworked_worked", HERE / "worked.py")
W = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(W)

F64_RTOL = 1e-10
F32_RTOL = 1e-5       # tests/test_handworked.py KAT_RTOL
WIDE_STRIDE = 97


def worked_subset(scene, dtype, joints=None):
    """worked.py on `scene`, or on the sub-scene of the joints `joints` (with every body: untouched bodies only integrate)"""
    if joints is not None:
        scene = dict(scene, joints=[scene["joints"][k] for k in joints])
    return W.step(scene, dtype, quat_product="sse2")


def compare(scene, b, j, where, dtype, rtol, joints=None, derived_rtol=None):
    """element-wise relative error of the oracle / device columns (b, j) against worked.py; raises on any column above `rtol` (velocities,
    joint forces and torques: above `derived_rtol`, default `rtol`)"""
    out = worked_subset(scene, dtype, joints)
    rows = np.arange(len(scene["bodies"]))
    if joints is not None:     # the bodies of the evaluated joints
        rows = np.unique([scene["joints"][k][s] for k in joints for s in ("body1", "body2")])
    errs = {}
    for key in ("position", "rotation", "linear_velocity"):
        errs[key] = rel_err(getattr(b, key)[rows], np.array(out[key])[rows])
    moving = [i for i in rows if out["angular_velocity"][i] is not None]
    errs["angular_velocity"] = rel_err(b.angular_velocity[moving], np.array([out["angular_velocity"][i] for i in moving]))
    ks = range(len(scene["joints"])) if joints is None else joints
    pos = {k: n for n, k in enumerate(ks)}
    f = [j.types[t].force[i] for k, t, i in where if k in pos]
    tq = [j.types[t].torque[i] for k, t, i in where if k in pos]
    errs["joint_force"] = rel_err(np.array(f), np.array([out["joint_force"][pos[k]] for k, _, _ in where if k in pos]))
    errs["joint_torque"] = rel_err(np.array(tq), np.array([out["joint_torque"][pos[k]] for k, _, _ in where if k in pos]))
    derived = rtol if derived_rtol is None else derived_rtol
    bad = {k: v for k, v in errs.items() if not v <= (rtol if k in ("position", "rotation") else derived)}
    assert not bad, f"worked.py disagrees: {bad}"
    return errs


def worked_joints(name):
    """the joints worked.py evaluates for family `name` (None = all)"""
    return list(range(0, len(JS.family(name)["joints"]), WIDE_STRIDE)) if name == "wide" else None


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", list(JS.FAMILIES))
def test_worked_agrees_with_oracle(name, dtype):
    scene = JS.family(name)
    prm, b, j, where = JS.columns(scene, dtype)
    oracle_lib.solver_step(prm, b, None, j)
    assert np.isfinite(b.position).all() and np.isfinite(b.angular_velocity).all()
    if dtype == np.float64:
        compare(scene, b, j, where, dtype, F64_RTOL, worked_joints(name))
    else:
        compare(scene, b, j, where, dtype, F32_RTOL, worked_joints(name), derived_rtol=F32_RTOL / scene["params"]["h"])


def test_families_cover_the_branches():
    """together the families reach every branch, body side and schedule shape tests/joint_scenes.py names (counted from the scene data)"""
    census = {n: JS.census(JS.family(n)) for n in JS.FAMILIES}
    total = {k: sum(c[k] for c in census.values()) for k in census["features"]}
    missing = sorted(k for k, v in total.items() if k not in JS.SHAPE_KEYS and v == 0)
    assert missing == [], missing
    for name in ("features", "features_sub12"):
        assert census[name]["types_in_one_level"] == 5, "a level interleaves the five types"
    assert census["hub"]["solve_levels"] == 1 and census["hub"]["hub_joints"] >= 32
    assert census["chain"]["solve_levels"] >= 2500 and census["chain"]["damp_levels"] >= 2500
    assert census["wide"]["solve_levels"] == 1 and census["wide"]["widest_level"] > 132 * 4 * 128, "wider than the largest megakernel grid"
    assert {JS.family(n)["params"]["substeps"] for n in JS.FAMILIES} >= {1, 4, 12}
