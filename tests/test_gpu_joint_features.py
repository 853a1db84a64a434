"""The XPBD joint stage on the device (the joint phases of step_megakernel and of the per-phase launches) on the generated joint scenes of
tests/joint_scenes.py: every joint type and limit branch, the `<= eps` exits, compliance, damping with joint_damping's dummy bodies, static,
kinematic and dominated body sides, and level schedules of one level, thousands of levels and one level wider than the megakernel grid.

Per scene and scalar type:
  * the default context runs the barrier megakernel (the wavefront schedule is never taken with joints);
  * barrier megakernel == per-phase launches, bit for bit, on the four body columns and on joint force and torque;
  * f32: the device equals the C++ oracle bit for bit;
  * f64: the device is within 1e-10 (element-wise, floor 1) of the oracle and of tests/golden/handworked/worked.py.  Not bit for bit: the
    device's double sin / cos / asin are not the host libm's correctly rounded ones, and an ulp there reaches the last bits of the result."""
import numpy as np
import pytest

import joint_scenes as JS
import oracle_lib
from helpers import rel_err
from test_gpu_wave_features import _env
from test_joint_scenes_cpu import F64_RTOL, compare, worked_joints

from avian_b200 import api

pytestmark = pytest.mark.gpu

BODY_COLUMNS = ("position", "rotation", "linear_velocity", "angular_velocity")
LAUNCH_BARRIER = 1


def _columns(b, j):
    out = {name: getattr(b, name) for name in BODY_COLUMNS}
    for t, jt in sorted(j.types.items()):
        out[f"force{t}"], out[f"torque{t}"] = jt.force, jt.torque
    return out


def _step(scene, dtype, **env):
    prm, b, j, where = JS.columns(scene, dtype)
    with _env(**env):
        ctx = api.Context(device=0, scalar=dtype)
    with ctx:
        ctx.solver_step(prm, b, None, j)
        t = ctx.timings()
    return b, j, where, t


def _differ(a, b):
    return [k for k in a if not np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8))]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", list(JS.FAMILIES))
def test_joint_features(name, dtype):
    scene = JS.family(name)
    b, j, where, t = _step(scene, dtype)
    assert t["launch_mode"] == LAUNCH_BARRIER, f"the default context runs launch mode {t['launch_mode']}"
    census = JS.census(scene)
    assert t["joint_levels"] == census["solve_levels"]
    bp, jp, _, tp = _step(scene, dtype, AVN_LAUNCH_MODE="phases")
    got = _columns(b, j)
    assert _differ(got, _columns(bp, jp)) == [], "barrier megakernel != per-phase launches"
    prm, bo, jo, _ = JS.columns(scene, dtype)
    oracle_lib.solver_step(prm, bo, None, jo)
    want = _columns(bo, jo)
    differ = _differ(got, want)
    print(f"[joint-features] {name} {np.dtype(dtype).name}: {len(got) - len(differ)}/{len(got)} columns bit-identical to the oracle {differ or ''}")
    if dtype == np.float32:
        assert differ == [], f"f32 device != oracle in {differ}"
    else:
        for k in got:
            assert rel_err(got[k], want[k]) <= F64_RTOL, k
        compare(scene, b, j, where, np.float64, F64_RTOL, worked_joints(name))
