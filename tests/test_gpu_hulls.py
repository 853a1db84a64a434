"""Convex hull colliders on the device: avn_narrow_phase equals the host fixture's manifolds bit for bit (and so meets the contract that
tests/test_hull_geometry_cpu.py checks on them) on a soup that runs every narrow kernel in one call, with and without body frames;
avn_update_aabbs equals the column-type restatement of ConvexPolyhedron::aabb (single pose and swept) and the oracle on the other shapes;
DeviceGraphWorld equals World step for step on a hull pile and on a pile of convex decompositions; collision events name each hull part with its
body; and the refusals (swept CCD with a hull, shape 3 without a table, a refused table) leave the context as it was."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
from avian_b200 import api, fixture, plugins, scenes  # noqa: E402
import hull_reference as ref  # noqa: E402
import oracle_lib  # noqa: E402
from test_gpu_graph import _check_graphs, _check_impulses  # noqa: E402
from test_hull_geometry_cpu import BOX, CAP, DT, HULL, HULLS, MAX_DIST, SCALARS, SPH, check_contract, soup  # noqa: E402

pytestmark = pytest.mark.gpu
COLS = ("position", "rotation", "linear_velocity", "angular_velocity")
OUT = ("point_count", "disjoint", "normal", "anchor1", "anchor2", "penetration", "normal_speed")


def _columns(scalar, pairs):
    n = len(pairs)
    cols = {"shape": np.array([s for p in pairs for s in (p[0], p[4])], dtype=np.uint8)}
    for key, ia, ib in (("dims", 1, 5), ("position", 2, 6), ("rotation", 3, 7)):
        cols[key] = np.ascontiguousarray([np.asarray(v, float) for p in pairs for v in (p[ia], p[ib])], dtype=scalar)
    c1, c2 = np.arange(0, 2 * n, 2, dtype=np.uint32), np.arange(1, 2 * n, 2, dtype=np.uint32)
    lv = np.zeros((2 * n, 3), dtype=scalar)
    lv[1::2, 0] = MAX_DIST / DT
    return (c1, c2, c1, c2), cols, lv, np.zeros((2 * n, 3), dtype=scalar)


def _mixed_pairs():
    """hull pairs of every kind in both orders, mixed with cuboid, sphere and capsule pairs, so every narrow kernel runs in one call"""
    rng = np.random.default_rng(1)
    pairs = []
    for shape_b in (HULL, BOX, SPH, CAP):
        pairs += soup(200 + shape_b, shape_b, 150)
    for _ in range(300):
        sa, sb = rng.choice([BOX, SPH, CAP]), rng.choice([BOX, SPH, CAP])
        q = rng.normal(size=(2, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
        da, db = rng.uniform(0.2, 1.0, 3), rng.uniform(0.2, 1.0, 3)
        pairs.append((sa, da, rng.uniform(-2, 2, 3), q[0], sb, db, rng.uniform(-2, 2, 3), q[1]))
    return [pairs[i] for i in rng.permutation(len(pairs))]


@pytest.mark.parametrize("scalar", SCALARS)
def test_device_narrow_phase_equals_the_fixture(gpu_ctx, scalar):
    pairs = _mixed_pairs()
    pr, cols, lv, av = _columns(scalar, pairs)
    n = 2 * len(pairs)
    rng = np.random.default_rng(2)
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    frames = {"position": (cols["position"].astype(np.float64) + rng.uniform(-0.3, 0.3, (n, 3))).astype(scalar), "rotation": q.astype(scalar),
              "center_of_mass": rng.uniform(-0.2, 0.2, (n, 3)).astype(scalar)}
    with api.Context(device=0, scalar=scalar) as ctx:
        ctx.set_convex_hulls(HULLS)
        dev = ctx.narrow_phase(DT, 1e-3, pr, cols, lv, av)
        ctx.contacts_set_body_frames(frames["position"], frames["rotation"], frames["center_of_mass"])
        dev_f = ctx.narrow_phase(DT, 1e-3, pr, cols, lv, av)
    host = fixture.raw_manifolds(scalar, DT, 1e-3, pr, cols, lv, av, f64_anchors=True, hulls=HULLS)
    host_f = fixture.raw_manifolds(scalar, DT, 1e-3, pr, cols, lv, av, frames=frames, hulls=HULLS)
    for k in OUT:
        assert np.array_equal(dev[k], host[k]), k
        assert np.array_equal(dev_f[k], host_f[k]), k
    hull_pairs = [k for k, p in enumerate(pairs) if HULL in (p[0], p[4])]
    assert (host["point_count"][hull_pairs] > 0).sum() > 200
    check_contract(scalar, [pairs[k] for k in hull_pairs], {k: v[hull_pairs] for k, v in host.items()})


@pytest.mark.parametrize("scalar", SCALARS)
def test_device_aabbs_equal_the_references(gpu_ctx, scalar):
    rng = np.random.default_rng(3)
    n = 6000
    shape = rng.integers(0, 4, n).astype(np.uint8)
    dims = rng.uniform(0.05, 1.5, (n, 3))
    dims[shape == CAP, 2] = 0.0
    dims[shape == HULL] = 0.0
    dims[shape == HULL, 0] = rng.integers(0, HULLS.count, int((shape == HULL).sum()))
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    cols = dict(shape=shape, dims=dims.astype(scalar), position=rng.uniform(-100, 100, (n, 3)).astype(scalar), rotation=q.astype(scalar))
    prm = api.AvnAabbParams(1.0 / 60.0, 0.005, 0.0)     # speculative margin 0: the pose's own AABB
    dev = api.Colliders(**cols)
    with api.Context(device=0, scalar=scalar) as ctx:
        ctx.set_convex_hulls(HULLS)
        ctx.update_aabbs(prm, dev)
    other = (shape == BOX) | (shape == SPH)
    orc = api.Colliders(**{k: v[other] for k, v in cols.items()})
    oracle_lib.update_aabbs(prm, orc)
    assert np.array_equal(dev.aabb_min[other], orc.aabb_min) and np.array_equal(dev.aabb_max[other], orc.aabb_max)
    g = np.dtype(scalar).type(0.005)
    for i in np.nonzero(shape == HULL)[0]:
        v, _ = HULLS.polyhedron(int(dims[i, 0]))
        mn, mx = ref.hull_aabb(scalar, v, cols["position"][i], cols["rotation"][i])
        assert np.array_equal(dev.aabb_min[i], mn - g) and np.array_equal(dev.aabb_max[i], mx + g), i


@pytest.mark.parametrize("scalar", SCALARS)
def test_device_swept_hull_aabbs(gpu_ctx, scalar):
    rng = np.random.default_rng(4)
    n = 3000
    dims = np.zeros((n, 3)); dims[:, 0] = rng.integers(0, HULLS.count, n)
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    base = dict(shape=np.full(n, HULL, np.uint8), dims=dims.astype(scalar), position=rng.uniform(-100, 100, (n, 3)).astype(scalar),
                rotation=q.astype(scalar), linear_velocity=rng.normal(0, 20, (n, 3)).astype(scalar))
    dt, tol = 1.0 / 60.0, 0.005
    margins = rng.uniform(0.0, 0.5, n).astype(scalar)
    for margin in (None, margins):
        cols = api.Colliders(**base, speculative_margin=margin)
        with api.Context(device=0, scalar=scalar) as ctx:
            ctx.set_convex_hulls(HULLS)
            ctx.update_aabbs(api.AvnAabbParams(dt, tol, float("inf")), cols)
        for i in range(n):
            m = float("inf") if margin is None else float(margin[i])
            v, _ = HULLS.polyhedron(int(dims[i, 0]))
            mn, mx = ref.swept_hull_aabb(scalar, v, base["position"][i], base["rotation"][i], base["linear_velocity"][i], dt, m, tol)
            assert np.array_equal(cols.aabb_min[i], mn) and np.array_equal(cols.aabb_max[i], mx), (i, margin is None)


def _thrown(sc):
    sc.bodies.linear_velocity[1:, 1] = -4.0
    return sc


def _hull_scenes():
    return [(lambda: scenes.hull_pile(300, seed=4), 120), (lambda: _thrown(scenes.hull_pile(200, seed=5, scalar=np.float64)), 120),
            (lambda: scenes.decomposed_pile(150, seed=6), 120)]


@pytest.mark.parametrize("scene_fn,steps", _hull_scenes())
def test_device_graph_world_equals_the_world_on_hull_scenes(gpu_ctx, scene_fn, steps):
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


def test_events_of_a_decomposition_name_each_touching_part(gpu_ctx):
    sc_a, sc_b = scenes.decomposed_pile(30, seed=7), scenes.decomposed_pile(30, seed=7)
    ev = np.zeros(sc_a.collider_body.shape[0], dtype=bool)
    ev[np.isin(sc_a.collider_body, [1, 2, 3])] = True
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
                for c, b in ((c1, b1), (c2, b2)):
                    if b in (1, 2, 3):
                        seen.add(int(c))
        assert len(seen) >= 4, seen


def test_refusals_leave_the_context_unchanged(gpu_ctx):
    with api.Context(device=0) as ctx_a, api.Context(device=0) as ctx_b:
        wa = plugins.DeviceGraphWorld(scenes.hull_pile(60, seed=8), plugins.PhysicsPlugins(ctx_a), ctx_a)
        wb = plugins.DeviceGraphWorld(scenes.hull_pile(60, seed=8), plugins.PhysicsPlugins(ctx_b), ctx_b)
        for _ in range(10):
            wa.step(); wb.step()
        b = wb.bodies
        colliders = {"shape": wb._shape, "dims": wb._dims, "position": b.position, "rotation": b.rotation, "aabb_min": wb.aabb_min,
                     "aabb_max": wb.aabb_max}
        # swept CCD refuses a contact store that holds a hull, with or without the capsule flag
        for caps in (False, True):
            with pytest.raises(api.AvianError) as e:
                ctx_b.ccd_configure(body=[1], collider=[1], capsules=caps)
            assert e.value.status == api.ERR_UNSUPPORTED
        # a refused table leaves the table as it was
        tet = scenes.regular_solids(0.5)[0]
        with pytest.raises(api.AvianError) as e:
            ctx_b.set_convex_hulls(api.ConvexHulls.from_polyhedra([(tet[0], [list(f) for f in tet[1]][:3])]))
        assert e.value.status == api.ERR_INVALID_ARGUMENT
        # an index past the table: every entry point refuses before anything is copied
        bad = wb._dims.copy()
        bad[np.nonzero(wb._shape == HULL)[0][0], 0] = wb.scene.hulls.count
        for fn in (lambda: ctx_b.contacts_step(wb.params.dt, 0.005, dict(colliders, dims=bad), b.linear_velocity, b.angular_velocity, take_pairs=False),
                   lambda: ctx_b.update_aabbs(api.AvnAabbParams(wb.params.dt, 0.005, float("inf")),
                                              api.Colliders(shape=wb._shape, dims=bad, position=b.position, rotation=b.rotation)),
                   lambda: ctx_b.narrow_phase(wb.params.dt, 0.005, (np.array([1], np.uint32),) * 2 + (np.array([1], np.uint32),) * 2,
                                              dict(colliders, dims=bad), b.linear_velocity, b.angular_velocity)):
            with pytest.raises(api.AvianError) as e:
                fn()
            assert e.value.status == api.ERR_INVALID_ARGUMENT
        for _ in range(10):
            wa.step(); wb.step()
            for k in COLS:
                assert np.array_equal(getattr(wa.bodies, k), getattr(wb.bodies, k)), k
    # shape 3 with no table set
    sc = scenes.hull_pile(20, seed=9)
    with api.Context(device=0) as ctx:
        cols = api.Colliders(shape=sc.shape_type.astype(np.uint8), dims=sc.dims.astype(np.float32), position=sc.bodies.position,
                             rotation=sc.bodies.rotation)
        with pytest.raises(api.AvianError) as e:
            ctx.update_aabbs(api.AvnAabbParams(DT, 0.005, float("inf")), cols)
        assert e.value.status == api.ERR_INVALID_ARGUMENT
        ctx.set_convex_hulls(sc.hulls)
        ctx.update_aabbs(api.AvnAabbParams(DT, 0.005, float("inf")), cols)
        ctx.set_convex_hulls(None)
        with pytest.raises(api.AvianError):
            ctx.update_aabbs(api.AvnAabbParams(DT, 0.005, float("inf")), cols)
    # swept CCD configured before the first contact step: the step that brings the hulls in makes the solver stage refuse
    with api.Context(device=0) as ctx:
        w = plugins.DeviceGraphWorld(scenes.hull_pile(20, seed=10), plugins.PhysicsPlugins(ctx), ctx, ccd={"body": [1], "collider": [1]})
        with pytest.raises(api.AvianError) as e:
            w.step()
        assert e.value.status == api.ERR_UNSUPPORTED
