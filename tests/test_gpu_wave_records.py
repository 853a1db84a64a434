"""The wavefront contact item computes the velocity-independent coefficients of every point's normal impulse before it waits for the
velocities, solves all three cases of the normal part with one branch-free expression, and stores each impulse record as soon as it is
final.  A record is written by the previous pass of the same manifold (relax of the previous substep, or the previous biased iteration) and
read by the next.  These tests pin the wavefront schedule bit for bit against the barrier schedule across those writers: several solver
iterations, restitution, records crossing avn_solver_run_range launches, and a body whose 16 manifolds give it the largest ranks."""
import os

import numpy as np
import pytest

from avian_b200 import api, scenes

from helpers import advance_to_solver_input

pytestmark = pytest.mark.gpu

BODY_COLUMNS = ("position", "rotation", "linear_velocity", "angular_velocity")
POINT_COLUMNS = ("warm_start_normal_impulse", "warm_start_tangent_impulse", "normal_impulse")


def _context(mode):
    """a fresh context whose solver runs the `mode` schedule ("wave" or "barrier"); the mode is read when the context is created"""
    os.environ["AVN_LAUNCH_MODE"] = mode
    try:
        return api.Context(device=0)
    finally:
        os.environ.pop("AVN_LAUNCH_MODE", None)


def _step(mode, prm, b, m):
    with _context(mode) as ctx:
        bb, mm = b.copy(), m.copy()
        ctx.solver_step(prm, bb, mm)
        return bb, mm, ctx.timings()


def _assert_same(got, want, what):
    (bg, mg), (bw, mw) = got, want
    for name in BODY_COLUMNS:
        assert np.array_equal(getattr(bg, name), getattr(bw, name)), (what, name)
    for name in POINT_COLUMNS:
        assert np.array_equal(getattr(mg, name), getattr(mw, name)), (what, name)


def _pile_with_restitution():
    """a brick pile with friction and restitution 0.4, pushed down so that the restitution pass has work"""
    _, (prm, b, m, j) = advance_to_solver_input(scenes.cube_stack(7, 5, 7, brick=True, restitution=0.4), steps=2, substeps=4)
    b.linear_velocity[:, 1] -= 2.0
    assert (m.friction > 0).all() and (m.restitution > 0).any()
    return prm, b, m


@pytest.mark.parametrize("iters", [1, 2, 3])
def test_wave_equals_barrier_over_solver_iterations(iters):
    """solve(s, it > 0) reads the records that solve(s, it - 1) wrote; solve(s, 0) and warm(s) those of relax(s - 1)"""
    prm, b, m = _pile_with_restitution()
    prm.solver_iterations = iters
    bw, mw, tw = _step("wave", prm, b, m)
    bb, mb, tb = _step("barrier", prm, b, m)
    assert tw["launch_mode"] == 2 and tb["launch_mode"] == 1   # AVN_LAUNCH_MEGA_WAVE, AVN_LAUNCH_MEGA_BARRIER
    assert (mw.normal_impulse > 0).any()
    _assert_same((bw, mw), (bb, mb), f"iters={iters}")


@pytest.mark.parametrize("iters", [1, 2])
def test_wave_run_range_one_substep_per_launch(iters):
    """records written by the relax of substep s - 1 in one launch are read by substep s in the next one"""
    prm, b, m = _pile_with_restitution()
    prm.solver_iterations = iters
    one = _step("wave", prm, b, m)
    with _context("wave") as ctx:
        b2, m2 = b.copy(), m.copy()
        ctx.solver_upload(prm, b2, m2, None)
        n = int(prm.substeps)
        for s in range(n):
            ctx.solver_run_range(s, 1, api.RUN_PREPARE if s == 0 else 0)
        ctx.solver_run_range(n, 0, api.RUN_RESTITUTION)
        ctx.solver_run_range(n, 0, api.RUN_FINALIZE)
        ctx.solver_download()
        assert ctx.timings()["launch_mode"] == 2
    _assert_same((b2, m2), one[:2], f"run_range iters={iters}")


@pytest.mark.parametrize("iters", [1, 3])
def test_wave_equals_barrier_with_max_rank_events(iters):
    """a plate on a 4 x 4 field of cubes carries 16 manifolds: its events reach rank 15 of k = 16 in every pass"""
    cubes = np.array([[1.5 * ix, 0.49, 1.5 * iz] for ix in range(4) for iz in range(4)])
    pos = np.concatenate([[[2.25, -0.5, 2.25]], cubes, [[2.25, 1.22, 2.25]]])
    he = np.concatenate([[[20.0, 0.5, 20.0]], np.full((16, 3), 0.5), [[3.5, 0.25, 3.5]]])
    kind = np.concatenate([[api.BODY_STATIC], np.full(17, api.BODY_DYNAMIC)])
    rot = np.tile(np.array([0.0, 0.0, 0.0, 1.0]), (18, 1))
    sc = scenes._assemble("plate_on_cubes", pos, rot, kind, he, np.full(18, scenes.SHAPE_CUBOID), np.float32)
    _, (prm, b, m, j) = advance_to_solver_input(sc, steps=3, substeps=4)
    prm.solver_iterations = iters
    plate = b.count - 1
    assert int((m.body1 == plate).sum() + (m.body2 == plate).sum()) >= 16
    bw, mw, tw = _step("wave", prm, b, m)
    bb, mb, _ = _step("barrier", prm, b, m)
    assert tw["launch_mode"] == 2
    _assert_same((bw, mw), (bb, mb), f"plate iters={iters}")
