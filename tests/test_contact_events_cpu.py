"""Collision events, sensors, removal of colliders and contact reports in the host fixture (avian_b200/host/host_api.cpp), the bit-exact
comparison for the device pipeline (tests/test_gpu_contact_events.py).  Hand-checked scenarios, each with its event lists written out step by
step; stepped by the ordinary World with the CPU oracle's broad phase and solver."""
import ctypes as C
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
from avian_b200 import api, plugins, scenes  # noqa: E402
import oracle_lib  # noqa: E402

GEN, EVENTS = api.PAIR_GENERATE_CONSTRAINTS, api.PAIR_CONTACT_EVENTS


def test_struct_layouts_match_the_header():
    names = ["AvnCollisionEvents", "AvnContactReport"]
    src = '#include <stdio.h>\n#include "avian_b200.h"\nint main(){' + "".join(f'printf("{n} %zu\\n", sizeof({n}));' for n in names) + "return 0;}"
    with tempfile.TemporaryDirectory() as d:
        (Path(d) / "s.c").write_text(src)
        subprocess.run(["gcc", "-I", str(ROOT / "include"), "-o", f"{d}/s", f"{d}/s.c"], check=True)
        out = subprocess.run([f"{d}/s"], capture_output=True, text=True, check=True).stdout
    sizes = dict(line.split() for line in out.strip().splitlines())
    for n in names:
        assert int(sizes[n]) == C.sizeof(getattr(api, n)), n


def _events(w):
    """(started, ended) of the last step as lists of (collider1, collider2, flags)"""
    f = lambda d: [(int(a), int(b), int(fl)) for a, b, fl in zip(d["collider1"], d["collider2"], d["flags"])]
    s, e = w.events
    return f(s), f(e)


def _timeline(w, steps, first=0):
    out = {}
    for i in range(first, first + steps):
        w.step()
        s, e = _events(w)
        if s or e:
            out[i] = (s, e)
    return out


def _boxes(pos, he, kind, shape=None, restitution=0.0):
    n = len(pos)
    return scenes._assemble("events", np.array(pos, dtype=float), np.tile([0, 0, 0, 1.0], (n, 1)), np.array(kind), np.array(he, dtype=float),
                            np.full(n, scenes.SHAPE_CUBOID) if shape is None else np.array(shape), np.float32, restitution=restitution)


def test_a_cube_bouncing_on_a_plate():
    """a cube dropped 0.5 above a plate (restitution 0.9), events enabled on both: it starts touching, bounces off (end), lands again (start),
    bounces again (end).  Every entry carries CONTACT_EVENTS | GENERATE_CONSTRAINTS."""
    sc = _boxes([[0, -0.5, 0], [0, 1.0, 0]], [[5, 0.5, 5], [0.5, 0.5, 0.5]], [api.BODY_STATIC, api.BODY_DYNAMIC], restitution=0.9)
    w = plugins.World(sc, oracle_lib.oracle_plugins(), substeps=4, events_enabled=[True, True])
    pair = (0, 1, EVENTS | GEN)
    assert _timeline(w, 50) == {19: ([pair], []), 21: ([], [pair]), 46: ([pair], []), 48: ([], [pair])}


def test_a_sphere_falling_through_a_sensor_box():
    """a dynamic sphere falls through a static sensor box: one start when it enters, one end when it leaves; the pair never generates
    constraints (no manifold is coloured), so the free fall is bit for bit the free fall of the same sphere without the box."""
    shape = [scenes.SHAPE_CUBOID, scenes.SHAPE_SPHERE]
    sc = _boxes([[0, 0, 0], [0, 3.0, 0]], [[1, 1, 1], [0.5, 0.5, 0.5]], [api.BODY_STATIC, api.BODY_DYNAMIC], shape)
    alone = _boxes([[0, 3.0, 0]], [[0.5, 0.5, 0.5]], [api.BODY_DYNAMIC], shape[1:])
    w = plugins.World(sc, oracle_lib.oracle_plugins(), substeps=4, sensor=[True, False])
    wf = plugins.World(alone, oracle_lib.oracle_plugins(), substeps=4)
    seen = {}
    for i in range(60):
        w.step(); wf.step()
        assert np.array_equal(w.bodies.linear_velocity[1], wf.bodies.linear_velocity[0]), f"step {i}"
        assert np.array_equal(w.bodies.position[1], wf.bodies.position[0]), f"step {i}"
        assert w.last_manifolds.count == 0, f"step {i}: a sensor pair took a colour"
        s, e = _events(w)
        if s or e:
            seen[i] = (s, e)
        if i == 40:
            r = w.report()
            assert r["contact_id"].tolist() == [0] and r["flags"].tolist() == [0] and r["total_normal_impulse"].tolist() == [0.0]
    assert seen == {33: ([(0, 1, 0)], []), 58: ([], [(0, 1, 0)])}


def _two_resting_cubes():
    return _boxes([[0, -0.5, 0], [0, 0.499, 0], [3, 0.499, 0]], [[10, 0.5, 10], [0.5, 0.5, 0.5], [0.5, 0.5, 0.5]],
                  [api.BODY_STATIC, api.BODY_DYNAMIC, api.BODY_DYNAMIC])


def test_a_collider_removed_while_touching():
    """two cubes resting on the ground (ContactIds 0 and 1), events enabled on cube 1: removing cube 1 queues one CollisionEnd, frees its row,
    and the next broad phase finds the pair again as a new pair that takes the lowest free ContactId (0) and starts touching at once."""
    w = plugins.World(_two_resting_cubes(), oracle_lib.oracle_plugins(), substeps=4, events_enabled=[False, True, False])
    assert _timeline(w, 8) == {0: ([(0, 1, EVENTS | GEN), (0, 2, GEN)], [])}
    w.remove_colliders([1])
    ids, c1, c2, _, _ = w.pipeline.active_edges()
    assert ids.tolist() == [1] and c2.tolist() == [2], "the removed collider's row is gone"
    assert w.pipeline.export_edges(1)[1].tolist() == [1], "and its manifold left the constraint graph"
    w.step()
    assert _events(w) == ([(0, 1, EVENTS | GEN)], [(0, 1, EVENTS | GEN)])       # the queued end first, then the re-found pair starts
    ids, c1, c2, _, _ = w.pipeline.active_edges()
    assert dict(zip(ids.tolist(), c2.tolist())) == {0: 1, 1: 2}
    assert _timeline(w, 3, 9) == {}
    r = w.report()
    assert r["contact_id"].tolist() == [0, 1] and (r["total_normal_impulse"] > 0).all() and (r["point_count"] == 4).all()
    assert w.report(events_only=True)["contact_id"].tolist() == [0]


def test_a_resting_cube_turned_into_a_sensor_falls():
    """a sensor toggled on for a cube resting on the ground: its rows are removed at once (one end) and found again as sensor rows
    (GENERATE_CONSTRAINTS clear) on the next step; nothing holds the cube any more, so it falls through the ground at g."""
    w = plugins.World(_two_resting_cubes(), oracle_lib.oracle_plugins(), substeps=4)
    _timeline(w, 8)
    v0 = w.bodies.linear_velocity[1, 1]
    w.set_sensors([False, True, False])
    w.step()
    assert _events(w) == ([(0, 1, 0)], [(0, 1, GEN)])
    assert w.last_manifolds.count == 1, "only the other cube's manifold is in the constraint graph"
    vy = [float(v0), float(w.bodies.linear_velocity[1, 1])]
    for _ in range(4):
        w.step()
        assert _events(w) == ([], [])
        vy.append(float(w.bodies.linear_velocity[1, 1]))
    dv = np.diff(vy[1:])
    assert np.allclose(dv, -9.81 / 60, rtol=1e-4), dv                   # free fall
    assert w.report()["flags"].tolist() == [0, GEN] and w.report()["total_normal_impulse"][0] == 0
    w.set_sensors(None)                                                  # and back: a solid pair again, pushed out of the ground
    w.step()
    assert _events(w) == ([(0, 1, GEN)], [(0, 1, 0)])
    assert w.last_manifolds.count == 2
