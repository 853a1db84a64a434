"""Compound bodies on the device: avn_narrow_phase with body frames equals the host fixture bit for bit, DeviceGraphWorld equals World step
for step on compound piles (with collision events), and the refusals of avn_contacts_set_body_frames leave the context as it was."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
from avian_b200 import api, fixture, plugins, scenes  # noqa: E402
from compound_scenes import DT, TOL, soup  # noqa: E402
from test_gpu_graph import _check_graphs, _check_impulses  # noqa: E402

pytestmark = pytest.mark.gpu
SCALARS = [np.float32, np.float64]
COLS = ("position", "rotation", "linear_velocity", "angular_velocity")
OUT = ("point_count", "disjoint", "normal", "anchor1", "anchor2", "penetration", "normal_speed")


@pytest.mark.parametrize("scalar", SCALARS)
def test_device_narrow_phase_with_frames_equals_the_fixture(gpu_ctx, scalar):
    pairs, cols, lv, av, frames = soup(scalar, 31, n=3000)
    # a third of the pairs get frame-less bodies inside the same call: the body at its collider's pose, the centre of mass at the origin
    plain_pairs = np.arange(3000) % 3 == 0
    for key in ("position", "rotation"):
        frames[key][0::2][plain_pairs] = cols[key][0::2][plain_pairs]
        frames[key][1::2][plain_pairs] = cols[key][1::2][plain_pairs]
    frames["center_of_mass"][0::2][plain_pairs] = 0
    frames["center_of_mass"][1::2][plain_pairs] = 0
    with api.Context(device=0, scalar=scalar) as ctx:
        plain = ctx.narrow_phase(DT, TOL, pairs, cols, lv, av)
        ctx.contacts_set_body_frames(frames["position"], frames["rotation"], frames["center_of_mass"])
        dev = ctx.narrow_phase(DT, TOL, pairs, cols, lv, av)
        ctx.contacts_set_body_frames()
        again = ctx.narrow_phase(DT, TOL, pairs, cols, lv, av)
    host = fixture.raw_manifolds(scalar, DT, TOL, pairs, cols, lv, av, frames=frames)
    want_plain = fixture.raw_manifolds(scalar, DT, TOL, pairs, cols, lv, av)
    for k in OUT:
        assert np.array_equal(dev[k], host[k]), k
        assert np.array_equal(plain[k], want_plain[k]) and np.array_equal(again[k], want_plain[k]), k
    assert (host["point_count"] > 0).sum() > 500
    for k in OUT:   # the frame-less subset has the frame-less path's values (a + 0 may turn -0 into +0, so ==, not bits)
        assert (dev[k][plain_pairs] == want_plain[k][plain_pairs]).all(), k
    assert (host["point_count"][plain_pairs] > 0).sum() > 150


def _thrown(sc):
    """the pile's bodies start moving down at 4 m/s (as test_gpu_capsules' f64 pile): they meet the ground and each other within the run"""
    sc.bodies.linear_velocity[1:, 1] = -4.0
    return sc


def _compound_scenes():
    return [(lambda: scenes.compound_pile(300, seed=1), 120), (lambda: _thrown(scenes.compound_pile(300, seed=2, scalar=np.float64)), 120),
            (lambda: scenes.compound_pile(300, seed=3, single_share=0.5), 120)]


@pytest.mark.parametrize("scene_fn,steps", _compound_scenes())
def test_device_graph_world_equals_the_world_on_compound_piles(gpu_ctx, scene_fn, steps):
    sc_a, sc_b = scene_fn(), scene_fn()
    scalar = sc_a.bodies.position.dtype
    with api.Context(device=0, scalar=scalar) as ctx_a, api.Context(device=0, scalar=scalar) as ctx_b:
        wa = plugins.World(sc_a, plugins.PhysicsPlugins(ctx_a), substeps=4)
        wb = plugins.DeviceGraphWorld(sc_b, plugins.PhysicsPlugins(ctx_b), ctx_b, substeps=4)
        started = 0
        for i in range(steps):
            wa.step(); wb.step()
            _check_graphs(wa, wb, ctx_b, i)
            _check_impulses(wa, wb, ctx_b, i)
            for k in COLS:
                assert np.array_equal(getattr(wa.bodies, k), getattr(wb.bodies, k)), f"step {i}: {k}"
            started += wb.stats["started_touching"]
        assert started > 0


def test_events_of_a_compound_name_each_touching_part(gpu_ctx):
    sc_a, sc_b = scenes.compound_pile(40, seed=4), scenes.compound_pile(40, seed=4)
    ev = np.zeros(sc_a.collider_body.shape[0], dtype=bool)
    ev[sc_a.collider_body == 1] = True          # CollisionEventsEnabled on every part of body 1
    with api.Context(device=0) as ctx_a, api.Context(device=0) as ctx_b:
        wa = plugins.World(sc_a, plugins.PhysicsPlugins(ctx_a), events_enabled=ev)
        wb = plugins.DeviceGraphWorld(sc_b, plugins.PhysicsPlugins(ctx_b), ctx_b, events_enabled=ev)
        seen = set()
        for i in range(120):
            wa.step(); wb.step()
            for la, lb in zip(wa.events, wb.events):
                assert set(la) == set(lb)
                for k in la:
                    assert np.array_equal(la[k], lb[k]), (i, k)
            st = wb.events[0]
            for c1, c2, b1, b2 in zip(st["collider1"], st["collider2"], st["body1"], st["body2"]):
                assert sc_a.collider_body[c1] == b1 and sc_a.collider_body[c2] == b2
                if b1 == 1: seen.add(int(c1))
                if b2 == 1: seen.add(int(c2))
        assert len(seen) >= 2, seen   # several parts of the one body report their own pairs


def test_refusals_leave_the_context_unchanged(gpu_ctx):
    sc = scenes.compound_pile(30, seed=6)
    with api.Context(device=0) as ctx_a, api.Context(device=0) as ctx_b:
        wa = plugins.DeviceGraphWorld(sc, plugins.PhysicsPlugins(ctx_a), ctx_a)
        wb = plugins.DeviceGraphWorld(scenes.compound_pile(30, seed=6), plugins.PhysicsPlugins(ctx_b), ctx_b)
        for _ in range(20):
            wa.step(); wb.step()
        b = wb.bodies
        with pytest.raises(api.AvianError) as e:
            ctx_b.contacts_set_body_frames(b.position, None)
        assert e.value.status == api.ERR_INVALID_ARGUMENT
        ctx_b.contacts_set_body_frames(b.position[:-1], b.rotation[:-1])      # accepted; the step refuses the body count
        with pytest.raises(api.AvianError) as e:
            colliders = {"shape": wb._shape, "dims": wb._dims, "position": wb.collider_pose["position"], "rotation": wb.collider_pose["rotation"],
                         "aabb_min": wb.aabb_min, "aabb_max": wb.aabb_max}
            ctx_b.contacts_step(wb.params.dt, 0.005, colliders, b.linear_velocity, b.angular_velocity, take_pairs=False)
        assert e.value.status == api.ERR_INVALID_ARGUMENT
        with pytest.raises(api.AvianError) as e:
            ctx_b.ccd_configure(body=[1], collider=[1])
        assert e.value.status == api.ERR_UNSUPPORTED
        for _ in range(20):
            wa.step(); wb.step()
            for k in COLS:
                assert np.array_equal(getattr(wa.bodies, k), getattr(wb.bodies, k)), k
    single = scenes.cube_stack(2, 1, 2)
    with api.Context(device=0) as ctx:
        w = plugins.DeviceGraphWorld(single, plugins.PhysicsPlugins(ctx), ctx, ccd={"body": [1], "collider": [1]})
        w.step()
        with pytest.raises(api.AvianError) as e:
            ctx.contacts_set_body_frames(single.bodies.position, single.bodies.rotation)
        assert e.value.status == api.ERR_UNSUPPORTED
        w.step()   # the refused call left the context as it was: the step still runs without frames
