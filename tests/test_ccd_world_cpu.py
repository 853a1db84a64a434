"""Swept CCD through a stepped World on the oracle's solver stage (tests/oracle_ccd.py): a plank spinning in place at a small static sphere,
and a 300 m/s sphere at a thin wall.  No GPU."""
from __future__ import annotations

import numpy as np
import pytest

from avian_b200 import api, plugins, scenes
from avian_b200.fixture import SHAPE_CUBOID, SHAPE_SPHERE
from oracle_ccd import oracle_ccd_plugins

DT = 1.0 / 60.0


def world(scene, ccd=None):
    return plugins.World(scene, oracle_ccd_plugins(gravity=plugins.Gravity(0.0, 0.0, 0.0)), substeps=4, ccd=ccd)


def spinning_plank(scalar):
    """Body 0: a plank of half length 2 spinning at 60 rad/s about z (1 rad per step); body 1: a static sphere of radius 0.1 at 0.5 rad, radius
    1.5 — inside the disc the plank sweeps, touched when the plank has turned 0.4 rad."""
    pos = np.array([[0, 0, 0], [1.5 * np.cos(0.5), 1.5 * np.sin(0.5), 0]])
    return scenes._assemble("plank", pos, np.tile([0, 0, 0, 1.0], (2, 1)), np.array([api.BODY_DYNAMIC, api.BODY_STATIC]),
                            np.array([[2.0, 0.05, 0.05], [0.1, 0, 0]]), np.array([SHAPE_CUBOID, SHAPE_SPHERE]), scalar,
                            angvel=np.array([[0, 0, 60.0], [0, 0, 0]]))


def angle_z(q):
    return 2 * np.arctan2(float(q[2]), float(q[3]))


@pytest.mark.parametrize("scalar", [np.float32, np.float64])
def test_spinning_plank(scalar):
    free = world(spinning_plank(scalar))
    free.step()
    assert abs(angle_z(free.bodies.rotation[0]) - 1.0) < 1e-3          # without CCD it turns through the sphere
    lin = world(spinning_plank(scalar), ccd=dict(body=[0], collider=[0], mode=[api.SWEEP_LINEAR]))
    lin.step()
    assert lin.plugins.get("SolverPlugin").last_ccd[0][1] == -1          # a linear sweep of a plank at rest sees nothing
    assert abs(angle_z(lin.bodies.rotation[0]) - 1.0) < 1e-3
    nl = world(spinning_plank(scalar), ccd=dict(body=[0], collider=[0]))
    nl.step()
    toi, hit, _ = nl.plugins.get("SolverPlugin").last_ccd[0]
    assert hit == 1 and abs(60.0 * float(toi) - 0.4) < 1e-3               # the non-linear sweep stops at the sphere
    # ccd/mod.rs:646-648 composes the TOI rotation onto the substeps' delta rotation instead of replacing it, so the plank ends at
    # 1 + 0.4 rad, and delta_position is overwritten with m * v = 0
    m = float(toi) * 1.0001
    assert abs(angle_z(nl.bodies.rotation[0]) - (1.0 + 60.0 * m)) < 1e-3
    assert np.abs(nl.bodies.position[0]).max() == 0


@pytest.mark.parametrize("mode", [None, api.SWEEP_LINEAR, api.SWEEP_NON_LINEAR])
def test_fast_sphere_stops_at_thin_wall(mode):
    # With the default speculative margin (Scalar::MAX) the narrow phase already gives the 300 m/s sphere a speculative contact with the wall,
    # so the substeps stop it there; CCD, reading the velocity after the substeps, then finds nothing left to sweep — as in the reference.
    s = np.float32
    scene = scenes._assemble("bullet", np.array([[0, 0, 0], [4.0, 0, 0]]), np.tile([0, 0, 0, 1.0], (2, 1)), np.array([api.BODY_DYNAMIC, api.BODY_STATIC]),
                             np.array([[0.05, 0, 0], [0.02, 3, 3]]), np.array([SHAPE_SPHERE, SHAPE_CUBOID]), s, linvel=np.array([[300.0, 0, 0], [0, 0, 0]]))
    w = world(scene, ccd=None if mode is None else dict(body=[0], collider=[0], mode=[mode]))
    w.step()
    contact_x = 4.0 - 0.02 - 0.05
    assert abs(float(w.bodies.position[0, 0]) - contact_x) < 1e-3
    if mode is not None:
        assert w.plugins.get("SolverPlugin").last_ccd[0][1] == -1


def test_world_refuses_ccd_without_a_ccd_solver():
    import oracle_lib
    w = plugins.World(spinning_plank(np.float32), oracle_lib.oracle_plugins(), ccd=dict(body=[0], collider=[0]))
    with pytest.raises(ValueError):
        w.step()
