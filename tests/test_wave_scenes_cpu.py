"""The extended hand-worked restatement (tests/golden/handworked/worked.py) against the C++ oracle on the generated scenes of
tests/wave_scenes.py: gyroscopic bodies with full local inverse inertia, locked axes, custom-integration markers, speed limits,
accelerations, dominance, kinematic hubs, static bodies by index and as AVN_NO_BODY, several solver iterations.  For these features the
oracle was, until now, only checked against the kernels it was written beside; worked.py is an independent reading of the reference.

Bars: f64 element-wise relative error <= 1e-10 (floor 1); f32 the hand-worked bar of tests/test_handworked.py.  Also: worked.py still
reproduces every committed vector of vectors.json exactly, and the generated colourings are what they claim to be."""
import importlib.util
import json
from pathlib import Path

import numpy as np
import pytest

import oracle_lib
import wave_scenes as WS
from helpers import rel_err

HERE = Path(__file__).resolve().parent / "golden" / "handworked"
_spec = importlib.util.spec_from_file_location("handworked_worked", HERE / "worked.py")
W = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(W)

F64_RTOL = 1e-10
F32_RTOL = 1e-5       # tests/test_handworked.py KAT_RTOL
BODY_OUT = ("position", "rotation", "linear_velocity", "angular_velocity")
POINT_OUT = ("warm_start_normal_impulse", "warm_start_tangent_impulse", "normal_impulse")
# worked.py evaluates the small and medium families; shapes_b1017 (1 017 bodies) is checked on the GPU only
CPU_FAMILIES = [f for f in WS.FAMILIES if f != "shapes_b1017"]


def test_worked_reproduces_committed_vectors_exactly():
    """the extension (clamps, markers, accelerations, solver iterations, the general inverse) changed nothing worked.py computed"""
    vectors = json.loads((HERE / "vectors.json").read_text())
    for name, sc in vectors["scenes"].items():
        for dtype, key in ((np.float32, "expected_f32"), (np.float64, "expected_f64")):
            got = json.loads(json.dumps(W.step(sc["input"], dtype)))
            assert got == sc[key], f"{name} {key}"


def worked_vs_columns(scene, dtype):
    """worked.py's result of `scene`, reshaped into the ABI's columns (bodies; points of the manifolds the solver keeps)"""
    # the oracle and the kernels take glam's SSE2 association of the f32 quaternion product (oracle/oracle_math.hpp)
    out = W.step(scene.worked(), dtype, quat_product="sse2")
    md = scene.manifolds
    kinds = scene.bodies["kind"]
    side = lambda b: np.where(b < 0, WS.STATIC, kinds[np.maximum(b, 0)])
    solved = (side(md["body1"]) == WS.DYNAMIC) | (side(md["body2"]) == WS.DYNAMIC)
    point_solved = np.repeat(solved, md["points"])
    return out, point_solved


def compare_with_worked(scene, b, m, dtype, rtol):
    """element-wise relative error of the columns (b, m) against worked.py, per column"""
    out, point_solved = worked_vs_columns(scene, dtype)
    errs = {}
    for key in ("position", "rotation", "linear_velocity"):
        errs[key] = rel_err(getattr(b, key), np.array(out[key]))
    dyn_or_kin = [i for i, av in enumerate(out["angular_velocity"]) if av is not None]
    errs["angular_velocity"] = rel_err(b.angular_velocity[dyn_or_kin], np.array([out["angular_velocity"][i] for i in dyn_or_kin]))
    for key in POINT_OUT:
        errs[key] = rel_err(getattr(m, key)[point_solved], np.array(out[key]).reshape(getattr(m, key)[point_solved].shape))
    bad = {k: v for k, v in errs.items() if not v <= rtol}
    assert not bad, f"worked.py disagrees: {bad}"
    return errs


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", CPU_FAMILIES)
def test_worked_agrees_with_oracle(name, dtype):
    scene = WS.family(name)
    prm, b, m = scene.columns(dtype)
    oracle_lib.solver_step(prm, b, m)
    compare_with_worked(scene, b, m, dtype, F64_RTOL if dtype == np.float64 else F32_RTOL)
    assert np.isfinite(b.position).all() and np.isfinite(b.angular_velocity).all()
    assert (m.normal_impulse > 0).any(), "the contacts carry load"


@pytest.mark.parametrize("name", list(WS.FAMILIES))
def test_generated_colourings_are_valid(name):
    scene = WS.family(name)
    assert WS.colouring_errors(scene) == []
    c = WS.feature_census(scene)
    assert c["max_points"] == (1 if name.startswith("spheres") else 4)
    if scene.hub is not None:
        assert WS.colours_of(scene, scene.hub) == set(range(23)), "the hub sits in all 23 colours"
        md = scene.manifolds
        on = np.flatnonzero((md["body1"] == scene.hub) | (md["body2"] == scene.hub))
        assert len(on) == 23
    if name == "shapes_b1017":
        lengths = np.bincount(scene.colour, minlength=24)
        assert scene.body_count == 1017
        assert [int(x) for x in lengths[18:23]] == [1, 31, 32, 33, 64]
        assert (lengths[4:18] == 0).all() and lengths[0] > 0, "empty colours between non-empty ones"
    if name == "single_b1":
        assert scene.body_count == 1 and c["no_body"] == scene.manifolds["body1"].shape[0]


def test_families_cover_the_features():
    """together the families contain every feature the GPU file claims to pin"""
    census = {n: WS.feature_census(WS.family(n)) for n in WS.FAMILIES}
    total = {k: sum(c[k] for c in census.values()) for k in census["mixed_b33"]}
    for k in ("gyroscopic", "off_diagonal", "both_non_dynamic", "no_body", "static_index", "kinematic_dynamic"):
        assert total[k] > 0, k
    s = WS.family("mixed_b33")
    bd = s.bodies
    assert set(np.unique(bd["integration_flags"])) == {0, 1, 2, 3}
    assert {0x07, 0x3F} <= set(np.unique(bd["locked_axes"]).tolist())
    assert np.isinf(bd["max_linear_speed"]).any() and np.isfinite(bd["max_linear_speed"]).any()
    assert (bd["dominance"] > 0).any() and (bd["dominance"] < 0).any()
    ns = s.manifolds["normal_speed"]
    assert (ns < -1.0).any() and (ns > -1.0).any(), "normal speeds on both sides of the restitution threshold"
    assert (s.manifolds["friction"] == 0).any() and (s.manifolds["friction"] > 0).any()
    assert all(WS.family("absent_b32").bodies[k] is None for k in WS.OPTIONAL_BODY)
