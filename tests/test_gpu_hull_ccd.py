"""Swept CCD with convex hull colliders on the device (avn_ccd_configure with AVN_CCD_HULLS): the G = 2 TOI kernel against the host brute
force (avh_ccd_solve_hulls) bit for bit on a hull pile under fire and on the 100k-cube stack, the device world beside the oracle world, a
spinning hull blade, the flag leaving hull-free scenes byte for byte as they were, and the refusals: a replaced hull table, and the calls
that leave the context as it was."""
from __future__ import annotations

import numpy as np
import pytest

import hull_query_reference as hq
from avian_b200 import api, fixture, plugins, scenes
from avian_b200.fixture import SHAPE_CAPSULE, SHAPE_CUBOID, SHAPE_SPHERE
from helpers import assert_bodies_close
from oracle_hull_ccd import oracle_hull_ccd_plugins
from test_gpu_ccd import mixed_config, pile_with_projectiles

pytestmark = pytest.mark.gpu
SCALARS = [np.float32, np.float64]
HULL = api.SHAPE_CONVEX_HULL
PDIMS = {SHAPE_CAPSULE: [0.1, 0.25, 0.0], SHAPE_SPHERE: [0.15, 0.0, 0.0], SHAPE_CUBOID: [0.15, 0.15, 0.15]}


def polyhedra(hulls):
    return [] if hulls is None else [hq.table_poly(hulls, h) for h in range(hulls.count)]


def extend(base, name, pos, rot, kind, shape, dims, linvel, angvel, extra_polys=(), scalar=np.float32):
    """base plus the given bodies; the base bodies keep their mass properties, a new hull body gets a 0.15 m cube's, and extra_polys are
    appended to the base's hull table (new hull indices count from the base table's size)"""
    b = base.bodies
    polys = polyhedra(base.hulls) + list(extra_polys)
    hulls = api.ConvexHulls.from_polyhedra(polys) if polys else None
    mass_dims = np.where((shape == HULL)[:, None], 0.15, dims)
    sc = scenes._assemble(name, np.concatenate([b.position.astype(np.float64), pos]), np.concatenate([b.rotation.astype(np.float64), rot]),
                          np.concatenate([b.kind, kind]), np.concatenate([np.where((base.shape_type == HULL)[:, None], 0.5, base.dims), mass_dims]),
                          np.concatenate([base.shape_type, np.where(shape == HULL, SHAPE_CUBOID, shape)]), scalar,
                          linvel=np.concatenate([b.linear_velocity.astype(np.float64), linvel]),
                          angvel=np.concatenate([b.angular_velocity.astype(np.float64), angvel]), hulls=hulls)
    sc.bodies.angular_velocity = sc.bodies.angular_velocity.copy()
    sc.shape_type = np.ascontiguousarray(np.concatenate([base.shape_type, shape]), dtype=np.int32)
    sc.dims = np.ascontiguousarray(np.concatenate([base.dims, dims]))
    sc.bodies.inverse_mass[:b.count] = b.inverse_mass
    sc.bodies.inverse_inertia_local[:b.count] = b.inverse_inertia_local
    return sc


def hull_pile_with_projectiles(scalar, n=120, layers=3, projectiles=36, seed=0, kinematic_bat=False):
    """scenes.hull_pile on its static ground (body 0) with hull, cuboid, sphere and capsule projectiles fired at random pile bodies from
    3-5 m at 250-400 m/s, and one long hull bat (a 4 x 0.1 x 0.1 box as an 8-vertex hull) spinning at 60 rad/s just above the pile's top.
    Returns the scene and the CCD bodies (the projectiles and the bat)."""
    base = scenes.hull_pile(n, seed=8, layers=layers, scalar=scalar)
    b = base.bodies
    rng = np.random.default_rng(seed)
    aim = b.position[1 + rng.integers(0, n, projectiles)].astype(np.float64)
    d = rng.normal(size=(projectiles, 3))
    d[:, 1] = np.abs(d[:, 1])
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    ppos = aim + d * rng.uniform(3.0, 5.0, (projectiles, 1))
    pvel = -d * rng.uniform(250.0, 400.0, (projectiles, 1))
    pshape = np.array([HULL, SHAPE_CUBOID, SHAPE_SPHERE, SHAPE_CAPSULE])[np.arange(projectiles) % 4]
    H = base.hulls.count
    pdims = np.array([[float(rng.integers(H)), 0, 0] if s == HULL else PDIMS[s] for s in pshape])
    q = rng.normal(size=(projectiles, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    top = b.position[1:].astype(np.float64)
    bat_pos = top[np.argmax(top[:, 1])] + np.array([0.0, 1.0, 0.0])
    bat = scenes.convex_hull_of(np.array([[sx * 2.0, sy * 0.05, sz * 0.05] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)]))
    sc = extend(base, "hull_ccd_pile", np.concatenate([ppos, bat_pos[None]]), np.concatenate([q, [[0, 0, 0, 1.0]]]),
                np.concatenate([np.zeros(projectiles, np.uint8), [api.BODY_KINEMATIC if kinematic_bat else api.BODY_DYNAMIC]]),
                np.concatenate([pshape, [HULL]]), np.concatenate([pdims, [[float(H), 0, 0]]]), np.concatenate([pvel, [[0, 0, 0]]]),
                np.concatenate([np.zeros((projectiles, 3)), [[0, 60.0, 0]]]), extra_polys=[bat], scalar=scalar)
    return sc, np.arange(b.count, b.count + projectiles + 1)


def hull_config(ccd, seed=1):
    cfg = mixed_config(ccd, seed)
    cfg["mode"] = (np.arange(ccd.shape[0]) % 2).astype(np.uint8)   # half Linear, half NonLinear
    cfg["capsules"] = True
    cfg["hulls"] = True
    return cfg


def step_and_check(ctx, world, cfg, scalar):
    """one DeviceGraphWorld step with CCD configured; the device's decisions against avh_ccd_solve_hulls on the same rows and velocities"""
    pre_pos, pre_rot = world.bodies.position.copy(), world.bodies.rotation.copy()
    world.step()
    got = ctx.ccd_download()
    g = ctx.contacts_download_graph(int(world.stats["rows_high_water"]), 0)
    rows = dict(c1=g["collider1"], c2=g["collider2"], b1=g["collider1"], b2=g["collider2"], live=g["live"])   # colliders are bodies here
    b = world.bodies
    bodies = dict(kind=b.kind, position=pre_pos, rotation=pre_rot, center_of_mass=b.center_of_mass, linear_velocity=b.linear_velocity,
                  angular_velocity=b.angular_velocity)
    dp = np.zeros((b.count, 3), scalar)
    dq = np.tile(np.array([0, 0, 0, 1], scalar), (b.count, 1))
    want = fixture.ccd_solve(scalar, float(world.params.dt), 1.0, bodies, world.scene.shape_type.astype(np.uint8), world.scene.dims, rows, cfg, dp, dq,
                             hulls=world.scene.hulls)
    for k in ("min_toi", "hit_body", "hit_contact", "candidates", "hits"):
        assert np.array_equal(got[k].view(np.uint8), want[k].view(np.uint8)), k
    assert got["total_candidates"] == int(want["candidates"].sum())
    hit = np.unique(np.concatenate([np.asarray(cfg["body"])[want["hit_body"] >= 0], want["hit_body"][want["hit_body"] >= 0]]))
    hit = hit[b.kind[hit] != api.BODY_STATIC]
    assert np.array_equal(b.position[hit], pre_pos[hit] + dp[hit])
    return got


@pytest.mark.parametrize("scalar", SCALARS)
@pytest.mark.parametrize("kinematic_bat", [False, True])
def test_device_pass_equals_host_brute_force(scalar, kinematic_bat):
    scene, ccd = hull_pile_with_projectiles(scalar, kinematic_bat=kinematic_bat)
    cfg = hull_config(ccd)
    with api.Context(device=0, scalar=scalar) as ctx:
        w = plugins.DeviceGraphWorld(scene, plugins.PhysicsPlugins(ctx), ctx, substeps=4)
        ctx.ccd_configure(**cfg)
        hits = hull_hits = 0
        for _ in range(4):
            got = step_and_check(ctx, w, cfg, scalar)
            hit = got["hit_body"] >= 0
            hits += int(hit.sum())
            hull_hits += int((hit & ((scene.shape_type[ccd] == HULL) | (scene.shape_type[np.maximum(got["hit_body"], 0)] == HULL))).sum())
        assert hits > 0 and hull_hits > 0


def test_device_world_beside_oracle_world():
    """DeviceGraphWorld(ccd={..., hulls}) beside World(oracle solver stage + solve_swept_ccd): the CCD decisions bit-identical every step,
    the bodies within the parity bar."""
    scalar = np.float32
    make = lambda: hull_pile_with_projectiles(scalar, n=40, layers=2, projectiles=12, seed=2)
    scene0, ccd = make()
    cfg = hull_config(ccd)
    with api.Context(device=0, scalar=scalar) as ctx:
        dev = plugins.DeviceGraphWorld(make()[0], plugins.PhysicsPlugins(ctx), ctx, substeps=4, ccd=cfg)
        ref = plugins.World(make()[0], oracle_hull_ccd_plugins(scene0.hulls), substeps=4, ccd=cfg)
        hits = 0
        for step in range(30):
            dev.step()
            ref.step()
            got = ctx.ccd_download()
            want = ref.plugins.get("SolverPlugin").last_ccd
            assert np.array_equal(got["min_toi"], np.array([w[0] for w in want], scalar)), step
            assert np.array_equal(got["hit_body"], np.array([w[1] for w in want])), step
            assert np.array_equal(got["hit_contact"], np.array([w[2] for w in want])), step
            assert_bodies_close(dev.bodies, ref.bodies, what=f"hull ccd step {step}: ")
            hits += int((got["hit_body"] >= 0).sum())
        assert hits > 0


def test_hull_projectiles_into_the_100k_stack():
    """1 000 hull projectiles (half Linear, half NonLinear) at the 100k-cube stack: the device pass equals the host brute force"""
    scalar = np.float32
    base = scenes.cube_stack(46, 47, 46, brick=False)
    p = base.bodies.position[1:].astype(np.float64)
    centre = 0.5 * (p.min(axis=0) + p.max(axis=0))
    radius = 0.5 * float(np.linalg.norm(p.max(axis=0) - p.min(axis=0)))
    n = 1000
    rng = np.random.default_rng(0)
    d = rng.normal(size=(n, 3))
    d[:, 1] = np.abs(d[:, 1])
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    ico = scenes.regular_solids(0.2)[2]
    sc = extend(base, "hull_ccd_stack", centre + d * rng.uniform(radius + 1.0, radius + 5.0, (n, 1)), q, np.zeros(n, np.uint8), np.full(n, HULL),
                np.tile([0.0, 0, 0], (n, 1)), -d * rng.uniform(200.0, 400.0, (n, 1)), np.zeros((n, 3)), extra_polys=[ico], scalar=scalar)
    ccd = np.arange(base.bodies.count, base.bodies.count + n)
    cfg = dict(body=ccd, collider=ccd, mode=(np.arange(n) % 2).astype(np.uint8), hulls=True)
    with api.Context(device=0, scalar=scalar) as ctx:
        w = plugins.DeviceGraphWorld(sc, plugins.PhysicsPlugins(ctx), ctx, substeps=4, ccd=cfg)
        hits = 0
        for _ in range(3):
            got = step_and_check(ctx, w, cfg, scalar)
            hits += int((got["hit_body"] >= 0).sum())
        assert hits > 0


@pytest.mark.parametrize("scalar", SCALARS)
def test_spinning_hull_blade_stops_at_the_known_angle(scalar):
    # a 4 m blade (an 8-vertex hull, 2 m each side of its centre) spinning at 60 rad/s about z meets a static ball of radius 0.1 at 1.5 m and
    # 0.5 rad: the pass stops it where its edge first reaches the ball, 0.4 rad into the step (test_ccd_cpu.test_spinning_plank_and_fast_sphere)
    blade = scenes.convex_hull_of(np.array([[sx * 2.0, sy * 0.05, sz * 0.05] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)]))
    empty = scenes._assemble("empty", np.zeros((0, 3)), np.zeros((0, 4)), np.zeros(0, np.uint8), np.zeros((0, 3)), np.zeros(0, np.int32), scalar)
    sc = extend(empty, "hull_blade", np.array([[0, 0, 0], [1.5 * np.cos(0.5), 1.5 * np.sin(0.5), 0]]), np.array([[0, 0, 0, 1.0], [0, 0, 0, 1.0]]),
                np.array([api.BODY_KINEMATIC, api.BODY_STATIC], np.uint8), np.array([HULL, SHAPE_SPHERE]), np.array([[0.0, 0, 0], [0.1, 0, 0]]),
                np.zeros((2, 3)), np.array([[0, 0, 60.0], [0, 0, 0]]), extra_polys=[blade], scalar=scalar)
    cfg = dict(body=np.array([0]), collider=np.array([0]), mode=np.array([api.SWEEP_NON_LINEAR], np.uint8), hulls=True)
    with api.Context(device=0, scalar=scalar) as ctx:
        w = plugins.DeviceGraphWorld(sc, plugins.PhysicsPlugins(ctx), ctx, substeps=4, ccd=cfg)
        got = step_and_check(ctx, w, cfg, scalar)
        assert got["hit_body"][0] == 1
        assert abs(60.0 * float(got["min_toi"][0]) - 0.4) < 1e-3


@pytest.mark.parametrize("scalar", SCALARS)
def test_flag_without_hulls_changes_nothing(scalar):
    """With AVN_CCD_HULLS set and no hull in the scene the pass runs the G = 0 kernel: results and bodies byte-identical."""
    outs = []
    for hulls in (False, True):
        scene, ccd = pile_with_projectiles(scalar)
        cfg = dict(mixed_config(ccd), hulls=hulls)
        with api.Context(device=0, scalar=scalar) as ctx:
            w = plugins.DeviceGraphWorld(scene, plugins.PhysicsPlugins(ctx), ctx, substeps=4, ccd=cfg)
            res = []
            for _ in range(3):
                w.step()
                r = ctx.ccd_download()
                res.append({k: np.asarray(r[k]).copy() for k in ("min_toi", "hit_body", "hit_contact", "candidates", "hits")})
                res.append({k: getattr(w.bodies, k).copy() for k in ("position", "rotation", "linear_velocity", "angular_velocity")})
            outs.append(res)
    for a, b in zip(*outs):
        for k in a:
            assert np.array_equal(np.ascontiguousarray(a[k]).view(np.uint8), np.ascontiguousarray(b[k]).view(np.uint8)), k


def test_replaced_table_is_refused_until_the_next_contact_step():
    scalar = np.float32
    scene, ccd = hull_pile_with_projectiles(scalar, n=60, layers=2, projectiles=8)
    cfg = hull_config(ccd)
    with api.Context(device=0, scalar=scalar) as ctx:
        w = plugins.DeviceGraphWorld(scene, plugins.PhysicsPlugins(ctx), ctx, substeps=4, ccd=cfg)
        w.step()
        prev = ctx.ccd_download()
        bodies = {k: getattr(w.bodies, k).copy() for k in ("position", "rotation", "linear_velocity", "angular_velocity")}
        ctx.set_convex_hulls(scene.hulls)          # the same hulls, a new table: not the one the last contact step read
        with pytest.raises(api.AvianError) as e:
            ctx.solver_step_resident(w.params, w.bodies, w.joints)
        assert e.value.status == api.ERR_INVALID_ARGUMENT
        # nothing ran: the pass's results (its device time included) and the bodies are the last step's
        again = ctx.ccd_download()
        for k in prev:
            assert np.array_equal(np.asarray(again[k]), np.asarray(prev[k])), k
        for k, v in bodies.items():
            assert np.array_equal(getattr(w.bodies, k), v), k
        # a fresh contact step reads the new table: the step runs, and the pass equals the host
        step_and_check(ctx, w, cfg, scalar)


def test_refusals_leave_the_context_unchanged():
    scalar = np.float32
    scene, ccd = hull_pile_with_projectiles(scalar, n=60, layers=2, projectiles=8)
    with api.Context(device=0, scalar=scalar) as ctx:
        w = plugins.DeviceGraphWorld(scene, plugins.PhysicsPlugins(ctx), ctx, substeps=4)
        w.step()
        # without AVN_CCD_HULLS (whatever AVN_CCD_CAPSULES says) the store's hulls are refused as before
        for extra in (dict(), dict(capsules=True)):
            with pytest.raises(api.AvianError) as e:
                ctx.ccd_configure(body=ccd, collider=ccd, **extra)
            assert e.value.status == api.ERR_UNSUPPORTED
        # the store holds capsules too: the hull bit alone is refused
        with pytest.raises(api.AvianError) as e:
            ctx.ccd_configure(body=ccd, collider=ccd, hulls=True)
        assert e.value.status == api.ERR_UNSUPPORTED
        # unknown bits, 0x2 among them
        for flags in (0x2, 0x3, 0x6, 0x7):
            c, keep = api.ccd_config(ccd, ccd, flags=flags)
            with pytest.raises(api.AvianError) as e:
                ctx._check(ctx.lib.avn_ccd_configure(ctx.handle, api.C.byref(c)))
            assert e.value.status == api.ERR_INVALID_ARGUMENT
        # none of that configured anything: the world steps without CCD, and a download still has nothing to give
        w.step()
        with pytest.raises(api.AvianError):
            ctx.ccd_download()
        ctx.ccd_configure(body=ccd, collider=ccd, capsules=True, hulls=True)
        w.step()
        assert ctx.ccd_download()["total_candidates"] > 0
