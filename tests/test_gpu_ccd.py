"""Swept CCD on the device (avn_ccd_*): the pass inside the device-resident solver stage against the host brute force (avh_ccd_solve), bit for
bit — min_toi, hit body, ContactId, counters and the delta_position it writes — plus the refusals and the unchanged single launch."""
from __future__ import annotations

import numpy as np
import pytest

from avian_b200 import api, fixture, plugins, scenes
from avian_b200.fixture import SHAPE_CUBOID, SHAPE_SPHERE
from helpers import advance_to_solver_input, assert_bodies_close
from oracle_ccd import oracle_ccd_plugins
from test_ccd_world_cpu import spinning_plank

pytestmark = pytest.mark.gpu


def pile_with_projectiles(scalar, n_side=6, layers=4, projectiles=40, seed=0, kinematic_target=False, standoff=(4.0, 6.0)):
    """A cube pile on a static ground (body 0) with fast spheres and cubes fired at it from all sides, and one thin plank spinning in place."""
    base = scenes.cube_stack(n_side, layers, n_side, brick=False, scalar=scalar)
    b = base.bodies
    rng = np.random.default_rng(seed)
    n0 = b.count
    centre = np.array([n_side * 0.55, layers * 0.5, n_side * 0.55])
    d = rng.normal(size=(projectiles, 3))
    d[:, 1] = np.abs(d[:, 1])
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    ppos = centre + d * rng.uniform(standoff[0], standoff[1], (projectiles, 1))
    pvel = -d * rng.uniform(200.0, 400.0, (projectiles, 1))
    pshape = np.where(np.arange(projectiles) % 2 == 0, SHAPE_SPHERE, SHAPE_CUBOID)
    pdims = np.where(pshape[:, None] == SHAPE_SPHERE, np.array([[0.15, 0, 0]]), np.array([[0.15, 0.15, 0.15]]))
    plank_pos = centre + np.array([0, layers * 0.5 + 2.0, 0])
    pos = np.concatenate([b.position.astype(np.float64), ppos, plank_pos[None]])
    rot = np.concatenate([b.rotation.astype(np.float64), np.tile([0, 0, 0, 1.0], (projectiles + 1, 1))])
    kind = np.concatenate([b.kind, np.zeros(projectiles, np.uint8), [api.BODY_KINEMATIC if kinematic_target else api.BODY_DYNAMIC]])
    shape = np.concatenate([base.shape_type, pshape, [SHAPE_CUBOID]])
    dims = np.concatenate([base.dims, pdims, [[2.0, 0.05, 0.05]]])
    linvel = np.concatenate([b.linear_velocity.astype(np.float64), pvel, [[0, 0, 0]]])
    angvel = np.concatenate([b.angular_velocity.astype(np.float64), np.zeros((projectiles, 3)), [[0, 60.0, 0]]])
    scene = scenes._assemble("ccd_pile", pos, rot, kind, dims, shape, scalar, linvel=linvel, angvel=angvel)
    ccd_bodies = np.arange(n0, n0 + projectiles + 1)
    return scene, ccd_bodies


def step_and_check(ctx, world, cfg, scalar):
    """One DeviceGraphWorld step with CCD configured; the device's decisions against the host brute force on the same rows and velocities."""
    pre_pos, pre_rot = world.bodies.position.copy(), world.bodies.rotation.copy()
    world.step()
    got = ctx.ccd_download()
    cap = int(world.stats["rows_high_water"])
    g = ctx.contacts_download_graph(cap, 0)
    rows = dict(c1=g["collider1"], c2=g["collider2"], b1=g["collider1"], b2=g["collider2"], live=g["live"])   # colliders are bodies here
    b = world.bodies
    # restitution is 0 in these scenes: the downloaded velocities are the SolverBody velocities the pass read
    bodies = dict(kind=b.kind, position=pre_pos, rotation=pre_rot, center_of_mass=b.center_of_mass, linear_velocity=b.linear_velocity,
                  angular_velocity=b.angular_velocity)
    dp = np.zeros((b.count, 3), scalar)
    dq = np.tile(np.array([0, 0, 0, 1], scalar), (b.count, 1))
    want = fixture.ccd_solve(scalar, float(world.params.dt), 1.0, bodies, world.scene.shape_type.astype(np.uint8), world.scene.dims, rows, cfg, dp, dq)
    for k in ("min_toi", "hit_body", "hit_contact", "candidates", "hits"):
        assert np.array_equal(got[k].view(np.uint8), want[k].view(np.uint8)), k
    assert got["total_candidates"] == int(want["candidates"].sum())
    # every body the pass wrote ends at its pre-step position + the pass's delta_position (centre of mass at the origin)
    hit = np.unique(np.concatenate([np.asarray(cfg["body"])[want["hit_body"] >= 0], want["hit_body"][want["hit_body"] >= 0]]))
    hit = hit[b.kind[hit] != api.BODY_STATIC]
    assert np.array_equal(b.position[hit], pre_pos[hit] + dp[hit])
    return got


@pytest.mark.parametrize("scalar", [np.float32, np.float64])
@pytest.mark.parametrize("kinematic_target", [False, True])
def test_device_pass_equals_host_brute_force(scalar, kinematic_target):
    scene, ccd = pile_with_projectiles(scalar, kinematic_target=kinematic_target)
    cfg = mixed_config(ccd)
    with api.Context(device=0, scalar=scalar) as ctx:
        w = plugins.DeviceGraphWorld(scene, plugins.PhysicsPlugins(ctx), ctx, substeps=4)
        ctx.ccd_configure(**cfg)
        hits = 0
        for _ in range(4):
            got = step_and_check(ctx, w, cfg, scalar)
            hits += int((got["hit_body"] >= 0).sum())
        assert hits > 0


def mixed_config(ccd, seed=1):
    n = ccd.shape[0]
    rng = np.random.default_rng(seed)
    return dict(body=ccd, collider=ccd, mode=rng.integers(0, 2, n), include_dynamic=rng.integers(0, 2, n) | (np.arange(n) % 3 != 0),
                linear_threshold=rng.choice([0.0, 1.0, 1000.0], n), angular_threshold=rng.choice([0.0, 0.5], n))


@pytest.mark.parametrize("case", ["plank", "pile", "kinematic"])
def test_device_world_beside_oracle_world(case):
    """DeviceGraphWorld(ccd) stepped beside World(oracle solver stage + solve_swept_ccd as tests/ccd_reference.py restates it): the CCD
    decisions are bit-identical every step, the bodies — whose rotations carry the composed delta_rotation — agree within the parity bar."""
    scalar = np.float32
    if case == "plank":
        scene_fn, cfg = (lambda: spinning_plank(scalar)), dict(body=[0], collider=[0])
    else:
        scene_fn = lambda: pile_with_projectiles(scalar, kinematic_target=case == "kinematic")[0]
        cfg = mixed_config(pile_with_projectiles(scalar)[1])
    with api.Context(device=0, scalar=scalar) as ctx:
        dev = plugins.DeviceGraphWorld(scene_fn(), plugins.PhysicsPlugins(ctx), ctx, substeps=4, ccd=cfg)
        ref = plugins.World(scene_fn(), oracle_ccd_plugins(), substeps=4, ccd=cfg)
        hits = 0
        for step in range(3):
            dev.step()
            ref.step()
            got = ctx.ccd_download()
            want = ref.plugins.get("SolverPlugin").last_ccd
            assert np.array_equal(got["min_toi"], np.array([w[0] for w in want], scalar)), step
            assert np.array_equal(got["hit_body"], np.array([w[1] for w in want])), step
            assert np.array_equal(got["hit_contact"], np.array([w[2] for w in want])), step
            assert_bodies_close(dev.bodies, ref.bodies, what=f"{case} step {step}: ")
            hits += int((got["hit_body"] >= 0).sum())
        assert hits > 0


def test_equal_tois_go_to_the_lowest_contact_id():
    # the spinning plank of test_ccd_world_cpu with a second sphere at the point reflected through the plank's centre: the plank's two ends
    # reach the two spheres at the same TOI bits (the geometry is symmetric under negation)
    scalar = np.float32
    base = spinning_plank(scalar)
    pos = np.concatenate([base.bodies.position.astype(np.float64), -base.bodies.position[1:2].astype(np.float64)])
    scene = scenes._assemble("tie", pos, np.tile([0, 0, 0, 1.0], (3, 1)), np.array([api.BODY_DYNAMIC, api.BODY_STATIC, api.BODY_STATIC]),
                             np.concatenate([base.dims, base.dims[1:2]]), np.array([SHAPE_CUBOID, SHAPE_SPHERE, SHAPE_SPHERE]), scalar,
                             angvel=np.array([[0, 0, 60.0], [0, 0, 0], [0, 0, 0]]))
    cfg = dict(body=[0], collider=[0])
    with api.Context(device=0, scalar=scalar) as ctx:
        w = plugins.DeviceGraphWorld(scene, plugins.PhysicsPlugins(ctx), ctx, substeps=4, ccd=cfg)
        got = step_and_check(ctx, w, cfg, scalar)
        g = ctx.contacts_download_graph(int(w.stats["rows_high_water"]), 0)
        ids = [e for e in range(g["live"].shape[0]) if g["live"][e] and 0 in (g["collider1"][e], g["collider2"][e])]
        assert len(ids) == 2 and got["hits"][0] == 2 and got["hit_contact"][0] == min(ids)


def test_large_scene_and_refusals():
    scalar = np.float32
    # ~100k cubes and 10 000 projectiles just outside the stack's bounding sphere
    scene, ccd = pile_with_projectiles(scalar, n_side=46, layers=47, projectiles=10000, seed=3, standoff=(45.0, 50.0))
    n = ccd.shape[0]
    cfg = dict(body=ccd, collider=ccd, mode=np.arange(n) % 2)
    with api.Context(device=0, scalar=scalar) as ctx:
        w = plugins.DeviceGraphWorld(scene, plugins.PhysicsPlugins(ctx), ctx, substeps=4)
        w.step()
        single = ctx.timings()["kernel_launches"]
        ctx.ccd_configure(**cfg)
        for _ in range(2):
            step_and_check(ctx, w, cfg, scalar)
        assert ctx.timings()["kernel_launches"] > single
        # refusals while configured
        with pytest.raises(api.AvianError) as e:
            ctx.solver_run_range(0, 1, api.RUN_PREPARE)
        assert e.value.status == api.ERR_UNSUPPORTED
        _, (prm, bodies, m, _) = advance_to_solver_input(scenes.cube_stack(3, 2, 3), steps=1, substeps=4)
        with pytest.raises(api.AvianError) as e:
            ctx.solver_step(prm, bodies, m)    # host manifolds: no ContactGraph on the device
        assert e.value.status == api.ERR_UNSUPPORTED
        ctx.solver_upload(prm, bodies, m)
        with pytest.raises(api.AvianError) as e:
            ctx.solver_run()
        assert e.value.status == api.ERR_UNSUPPORTED
        with pytest.raises(api.AvianError) as e:
            ctx.solver_step_partitioned()
        assert e.value.status == api.ERR_UNSUPPORTED
        for bad in (dict(body=[0, 0], collider=[1, 2]), dict(body=[scene.bodies.count], collider=[0]), dict(body=[1], collider=[10 ** 7]),
                    dict(body=[1], collider=[1], mode=[7]), dict(body=[1], collider=[1], linear_threshold=[np.nan])):
            with pytest.raises(api.AvianError) as e:
                ctx.ccd_configure(**bad)
            assert e.value.status == api.ERR_INVALID_ARGUMENT
        # clearing the configuration brings back the single launch
        ctx.ccd_configure(None)
        w.step()
        assert ctx.timings()["kernel_launches"] == single
