"""The wavefront solver stage (step_megakernel, launch mode 2) on the body features and schedule shapes the cube-stack scenes never reach:
gyroscopic bodies with full local inverse inertia, every LockedAxes bit, custom-integration markers, speed limits, accelerations, damping,
positive and negative dominance, kinematic hubs, static bodies by index and as AVN_NO_BODY, manifolds with no dynamic side, colour
lengths around the 32-item chunk, empty colours, a body in all 23 colours (tests/wave_scenes.py builds them).

Per scene and scalar type:
  * the default context picks the wavefront (launch mode 2);
  * wave == barrier == phases, bit for bit, on every body and impulse column;
  * f32: the device equals the C++ oracle bit for bit;
  * f64: the device is within 1e-10 (element-wise, floor 1) of tests/golden/handworked/worked.py, the independent restatement.
Then: a scene large enough that every warp takes several chunks; every compiled megakernel instance (AVN_MEGA_BPS 2/3/4, MAXP 1/4); the
wave / barrier switch at widest colour = 2 * grid * 128.  AVN_* variables are set only while a context is created (and, for the debug
line, while it steps) and restored afterwards."""
import os
import re
from contextlib import contextmanager

import numpy as np
import pytest

from avian_b200 import api

import oracle_lib
import wave_scenes as WS
from helpers import rel_err
from test_wave_scenes_cpu import CPU_FAMILIES, F64_RTOL, compare_with_worked

pytestmark = pytest.mark.gpu

BODY_COLUMNS = ("position", "rotation", "linear_velocity", "angular_velocity")
POINT_COLUMNS = ("warm_start_normal_impulse", "warm_start_tangent_impulse", "normal_impulse")
LAUNCH_BARRIER, LAUNCH_WAVE = 1, 2
DEBUG_LINE = re.compile(r"\[avn\] megakernel bps=(\d) maxp=(\d): (\d+) blocks/SM resident, grid (\d+)")


@contextmanager
def _env(**env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _step(cols, dtype, **env):
    """one solver stage of copies of `cols` in a fresh context created under `env`; returns (bodies, manifolds, launch mode)"""
    prm, b, m = cols
    b, m = b.copy(), m.copy()
    with _env(**env):
        ctx = api.Context(device=0, scalar=dtype)
    with ctx:
        ctx.solver_step(prm, b, m)
        mode = ctx.timings()["launch_mode"]
    return b, m, mode


def _oracle(cols):
    prm, b, m = cols
    b, m = b.copy(), m.copy()
    oracle_lib.solver_step(prm, b, m)
    return b, m


def _bit_identical(got, want):
    """names of the columns of (bodies, manifolds) `got` that differ from `want` in any bit"""
    (bg, mg), (bw, mw) = got, want
    out = []
    for name in BODY_COLUMNS:
        if not np.array_equal(getattr(bg, name).view(np.uint8), getattr(bw, name).view(np.uint8)):
            out.append(name)
    for name in POINT_COLUMNS:
        if not np.array_equal(getattr(mg, name).view(np.uint8), getattr(mw, name).view(np.uint8)):
            out.append(name)
    return out


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", list(WS.FAMILIES))
def test_wave_features(name, dtype):
    scene = WS.family(name)
    cols = scene.columns(dtype)
    bd, md, mode = _step(cols, dtype)
    assert mode == LAUNCH_WAVE, f"the default context runs launch mode {mode}"
    wave, barrier, phases = (_step(cols, dtype, AVN_LAUNCH_MODE=m) for m in ("wave", "barrier", "phases"))
    assert (wave[2], barrier[2]) == (LAUNCH_WAVE, LAUNCH_BARRIER)
    assert _bit_identical((bd, md), wave[:2]) == []
    assert _bit_identical(wave[:2], barrier[:2]) == [], "wave != barrier"
    assert _bit_identical(wave[:2], phases[:2]) == [], "wave != phases"
    want = _oracle(cols)
    differ = _bit_identical((bd, md), want)
    print(f"[wave-features] {name} {np.dtype(dtype).name}: {7 - len(differ)}/7 columns bit-identical to the oracle {differ or ''}")
    if dtype == np.float32:
        assert differ == [], f"f32 device != oracle in {differ}"
    else:
        for col in BODY_COLUMNS:
            assert rel_err(getattr(bd, col), getattr(want[0], col)) <= F64_RTOL, col
        for col in POINT_COLUMNS:
            assert rel_err(getattr(md, col), getattr(want[1], col)) <= F64_RTOL, col
        if name in CPU_FAMILIES:
            compare_with_worked(scene, bd, md, np.float64, F64_RTOL)
    assert (md.normal_impulse > 0).any()


def test_past_the_warp_count():
    """~60 000 bodies and ~110 000 manifolds: at f32 / 3 blocks per SM the grid has about 50 000 lanes, so every warp takes several
    chunks of bodies and of manifolds in every pass"""
    scene = WS.generate(seed=11, dynamic=60000, kinematic=600, static=400, pairs=80000, static_contacts=20000, no_body_contacts=8000,
                        kinematic_pairs=2000, substeps=4, solver_iterations=2, restitution_iterations=2)
    assert WS.colouring_errors(scene) == []
    cols = scene.columns(np.float32)
    assert scene.body_count + len(scene.colour) > 3 * 50688
    wave = _step(cols, np.float32)
    barrier = _step(cols, np.float32, AVN_LAUNCH_MODE="barrier")
    assert (wave[2], barrier[2]) == (LAUNCH_WAVE, LAUNCH_BARRIER)
    assert _bit_identical(wave[:2], barrier[:2]) == [], "wave != barrier"
    assert _bit_identical(wave[:2], _oracle(cols)) == [], "device != oracle"


def _debug_lines(capfd):
    return [tuple(int(x) for x in m.groups()) for m in DEBUG_LINE.finditer(capfd.readouterr().err)]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("bps", [2, 3, 4])
@pytest.mark.parametrize("name,maxp", [("mixed_b33", 4), ("spheres_b33", 1)])
def test_every_megakernel_instance(name, maxp, bps, dtype, capfd):
    """each of the twelve compiled step_megakernel<S, BPS, MAXP> gives the bits of the default instance; the debug line names the one
    that ran (the last selection before the step)"""
    cols = WS.family(name).columns(dtype)
    default = _step(cols, dtype)
    capfd.readouterr()
    with _env(AVN_MEGA_BPS=bps, AVN_DEBUG_GRID=1):
        got = _step(cols, dtype)
    lines = _debug_lines(capfd)
    assert lines, "no [avn] megakernel line"
    ran_bps, ran_maxp, per_sm, grid = lines[-1]
    assert (ran_bps, ran_maxp) == (bps, maxp) and per_sm > 0 and grid > 0
    assert got[2] == default[2] == LAUNCH_WAVE
    assert _bit_identical(got[:2], default[:2]) == []


def test_wave_barrier_switch(capfd):
    """one colour of exactly 2 * grid * 128 single-point manifolds (every one against AVN_NO_BODY) runs the wavefront; one more
    manifold and the default context takes the barrier schedule.  Both equal the oracle bit for bit."""
    probe = WS.family("spheres_b33").columns(np.float32)
    capfd.readouterr()
    with _env(AVN_DEBUG_GRID=1):
        _step(probe, np.float32)
    lines = [x for x in _debug_lines(capfd) if x[1] == 1]
    assert lines
    grid = lines[-1][3]
    limit = 2 * grid * 128
    for n, mode in ((limit, LAUNCH_WAVE), (limit + 1, LAUNCH_BARRIER)):
        scene = WS.generate(seed=12, dynamic=n, colour_shape=[1] * n, max_points=1, substeps=2)
        assert np.bincount(scene.colour).max() == n and (scene.manifolds["body2"] == api.NO_BODY).all()
        cols = scene.columns(np.float32)
        with _env(AVN_DEBUG_GRID=1):
            got = _step(cols, np.float32)
        assert got[2] == mode, (n, got[2])
        assert _bit_identical(got[:2], _oracle(cols)) == [], n
