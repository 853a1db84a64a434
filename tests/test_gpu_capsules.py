"""Capsule colliders on the device: avn_narrow_phase equals the host fixture's manifolds bit for bit (and so meets the contract that
tests/test_capsule_geometry_cpu.py checks on them), avn_update_aabbs equals the column-type restatement of Capsule::aabb and the oracle on the
other shapes, DeviceGraphWorld equals World step for step on capsule scenes (with and without sleeping), and the refusals leave the context
as it was."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
from avian_b200 import api, fixture, plugins, scenes  # noqa: E402
import capsule_reference as ref  # noqa: E402
import oracle_lib  # noqa: E402
from test_capsule_geometry_cpu import BOX, CAP, DT, MAX_DIST, SCALARS, SPH, check_contract, log_piles, soup  # noqa: E402
from test_gpu_graph import _check_graphs, _check_impulses  # noqa: E402
from test_gpu_sleeping import _Pair  # noqa: E402

pytestmark = pytest.mark.gpu
COLS = ("position", "rotation", "linear_velocity", "angular_velocity")


def _columns(scalar, pairs):
    n = len(pairs)
    cols = {"shape": np.array([s for p in pairs for s in (p[0], p[4])], dtype=np.uint8)}
    for key, ia, ib in (("dims", 1, 5), ("position", 2, 6), ("rotation", 3, 7)):
        cols[key] = np.ascontiguousarray([np.asarray(v, float) for p in pairs for v in (p[ia], p[ib])], dtype=scalar)
    c1, c2 = np.arange(0, 2 * n, 2, dtype=np.uint32), np.arange(1, 2 * n, 2, dtype=np.uint32)
    lv = np.zeros((2 * n, 3), dtype=scalar)
    lv[1::2, 0] = MAX_DIST / DT
    return (c1, c2, c1, c2), cols, lv, np.zeros((2 * n, 3), dtype=scalar)


@pytest.mark.parametrize("scalar", SCALARS)
def test_device_narrow_phase_equals_the_fixture(gpu_ctx, scalar):
    rng = np.random.default_rng(1)
    # the three capsule pair types in both orders, mixed with cuboid and sphere pairs so both kernels run in one call
    pairs = []
    for shape_b in (CAP, SPH, BOX):
        for p in soup(100 + shape_b, shape_b, 400):
            pairs.append(p if rng.uniform() < 0.5 else (p[4], p[5], p[6], p[7], p[0], p[1], p[2], p[3]))
    for _ in range(300):
        sa, sb = rng.choice([BOX, SPH]), rng.choice([BOX, SPH])
        q = rng.normal(size=(2, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
        pairs.append((sa, rng.uniform(0.2, 1.0, 3), rng.uniform(-2, 2, 3), q[0], sb, rng.uniform(0.2, 1.0, 3), rng.uniform(-2, 2, 3), q[1]))
    order = rng.permutation(len(pairs))
    pairs = [pairs[i] for i in order]
    pr, cols, lv, av = _columns(scalar, pairs)
    with api.Context(device=0, scalar=scalar) as ctx:
        dev = ctx.narrow_phase(DT, 1e-3, pr, cols, lv, av)
    host = fixture.raw_manifolds(scalar, DT, 1e-3, pr, cols, lv, av, f64_anchors=True)
    for k in ("point_count", "normal", "anchor1", "anchor2", "penetration", "normal_speed"):
        assert np.array_equal(dev[k], host[k]), k
    capsule_pairs = [k for k, p in enumerate(pairs) if CAP in (p[0], p[4])]
    sub = {k: v[capsule_pairs] for k, v in host.items()}
    check_contract(scalar, [pairs[k] for k in capsule_pairs], sub)


@pytest.mark.parametrize("scalar", SCALARS)
def test_device_aabbs_equal_the_references(gpu_ctx, scalar):
    rng = np.random.default_rng(2)
    n = 20_000
    shape = rng.integers(0, 3, n).astype(np.uint8)
    dims = rng.uniform(0.05, 1.5, (n, 3))
    dims[shape == CAP, 2] = 0.0
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    cols = dict(shape=shape, dims=dims.astype(scalar), position=rng.uniform(-100, 100, (n, 3)).astype(scalar), rotation=q.astype(scalar))
    prm = api.AvnAabbParams(1.0 / 60.0, 0.005, 0.0)     # speculative margin 0: the pose's own AABB
    dev = api.Colliders(**cols)
    with api.Context(device=0, scalar=scalar) as ctx:
        ctx.update_aabbs(prm, dev)
    orc = api.Colliders(**cols)
    oracle_lib.update_aabbs(prm, orc)
    other = shape != CAP
    assert np.array_equal(dev.aabb_min[other], orc.aabb_min[other]) and np.array_equal(dev.aabb_max[other], orc.aabb_max[other])
    g = np.dtype(scalar).type(0.005)
    for i in np.nonzero(shape == CAP)[0]:
        mn, mx = ref.capsule_aabb(scalar, cols["dims"][i], cols["position"][i], cols["rotation"][i])
        assert np.array_equal(dev.aabb_min[i], mn - g) and np.array_equal(dev.aabb_max[i], mx + g), i


@pytest.mark.parametrize("scalar", SCALARS)
def test_device_swept_capsule_aabbs(gpu_ctx, scalar):
    """the swept path (two poses merged), which the default configuration (speculative margin = MAX) runs: bit for bit against the
    column-type restatement with linear velocities, under the default and under per-collider finite margins that clamp the sweep; with
    angular velocities as well, the box holds both poses' boxes (the end rotation goes through the device's sin / cos)"""
    rng = np.random.default_rng(3)
    n = 5_000
    dims = np.stack([rng.uniform(0.05, 0.5, n), rng.uniform(0.0, 1.5, n), np.zeros(n)], axis=1).astype(scalar)
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    base = dict(shape=np.full(n, CAP, np.uint8), dims=dims, position=rng.uniform(-100, 100, (n, 3)).astype(scalar), rotation=q.astype(scalar),
                linear_velocity=rng.normal(0, 20, (n, 3)).astype(scalar))
    dt, tol = 1.0 / 60.0, 0.005
    margins = rng.uniform(0.0, 0.5, n).astype(scalar)
    for margin in (None, margins):
        cols = api.Colliders(**base, speculative_margin=margin)
        with api.Context(device=0, scalar=scalar) as ctx:
            ctx.update_aabbs(api.AvnAabbParams(dt, tol, float("inf")), cols)
        for i in range(n):
            m = float("inf") if margin is None else float(margin[i])
            mn, mx = ref.swept_capsule_aabb(scalar, dims[i], base["position"][i], base["rotation"][i], base["linear_velocity"][i], dt, m, tol)
            assert np.array_equal(cols.aabb_min[i], mn) and np.array_equal(cols.aabb_max[i], mx), (i, margin is None)
    av = rng.normal(0, 5, (n, 3)).astype(scalar)
    cols = api.Colliders(**base, angular_velocity=av)
    with api.Context(device=0, scalar=scalar) as ctx:
        ctx.update_aabbs(api.AvnAabbParams(dt, tol, float("inf")), cols)
    slack = 64 * np.finfo(scalar).eps * 200
    for i in range(0, n, 7):
        p0, r0 = base["position"][i].astype(np.float64), base["rotation"][i].astype(np.float64)
        w = av[i].astype(np.float64) * dt
        ang = np.linalg.norm(w)
        dq = np.concatenate([w / ang * np.sin(ang / 2), [np.cos(ang / 2)]]) if ang > 0 else np.array([0, 0, 0, 1.0])
        r1 = np.array([dq[3] * r0[0] + dq[0] * r0[3] + dq[1] * r0[2] - dq[2] * r0[1], dq[3] * r0[1] - dq[0] * r0[2] + dq[1] * r0[3] + dq[2] * r0[0],
                       dq[3] * r0[2] + dq[0] * r0[1] - dq[1] * r0[0] + dq[2] * r0[3], dq[3] * r0[3] - dq[0] * r0[0] - dq[1] * r0[1] - dq[2] * r0[2]])
        p1 = p0 + base["linear_velocity"][i].astype(np.float64) * dt
        for p, r in ((p0, r0), (p1, r1)):
            e0, e1 = ref.capsule_segment(p, r, float(dims[i, 1]))
            lo, hi = np.minimum(e0, e1) - float(dims[i, 0]) - tol, np.maximum(e0, e1) + float(dims[i, 0]) + tol
            assert np.all(cols.aabb_min[i] <= lo + slack) and np.all(cols.aabb_max[i] >= hi - slack), i


def _thrown_pile(n, seed, layers, scalar):
    """a capsule pile whose bodies start moving down at 4 m/s: they meet the ground and each other within the run"""
    sc = scenes.capsule_pile(n, seed=seed, layers=layers, scalar=scalar)
    sc.bodies.linear_velocity[1:, 1] = -4.0
    return sc


def _capsule_scenes():
    return [
        (lambda: scenes.capsule_pile(400, seed=4, layers=4), 150),
        (lambda: scenes.ragdoll_field(9, pitch=1.2, drop_height=0.5, limbs="capsule"), 120),
        (lambda: _thrown_pile(200, 5, 3, np.float64), 120),
    ]


@pytest.mark.parametrize("scene_fn,steps", _capsule_scenes())
def test_device_graph_world_equals_the_world_on_capsule_scenes(gpu_ctx, scene_fn, steps):
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


def _check_but_timers(wa, wb, ctx_b, step):
    """test_gpu_sleeping._check without the per-body sleep timers (compared on their own in test_sleep_timers_of_a_cube_and_sphere_pile):
    ContactIds, live / touching / asleep rows, asleep bodies, island labels, Sleeping flags, colours, bodies"""
    g = wa.graph()
    st = wb.stats
    hw = st["rows_high_water"]
    assert st["rows_live"] == g["ids"].shape[0], f"step {step}: live pairs"
    d = ctx_b.contacts_download_graph(hw, wb.wake_stats["manifold_count"])
    sl = ctx_b.contacts_download_sleeping(hw, wb.n)
    live = np.zeros(hw, dtype=bool); live[g["ids"]] = True
    assert np.array_equal(d["live"].astype(bool), live), f"step {step}: ContactIds in use"
    touching = np.zeros(hw, dtype=bool); touching[g["sid"]] = g["touching"]
    asleep = np.zeros(hw, dtype=bool); asleep[g["sid"]] = g["asleep"]
    assert np.array_equal(d["touching"].astype(bool), touching), f"step {step}: touching"
    assert np.array_equal(sl["row_asleep"].astype(bool), asleep), f"step {step}: asleep rows"
    assert np.array_equal(sl["body_asleep"].astype(bool), wa.body_asleep), f"step {step}: asleep bodies"
    for k in ("island", "sleeping_flags"):
        assert np.array_equal(getattr(wa, k), getattr(wb, k)), f"step {step}: {k}"
    colour = np.full(hw, -1, dtype=np.int8)
    for c in range(api.GRAPH_COLOR_COUNT):
        colour[g["edge"][g["color_offsets"][c]:g["color_offsets"][c + 1]]] = c
    assert np.array_equal(d["colour"], colour), f"step {step}: colours"
    for k in COLS:
        assert np.array_equal(getattr(wa.bodies, k), getattr(wb.bodies, k)), f"step {step}: {k}"


def _sleeping_pair(scene_fn, ctx_a, ctx_b):
    from sleeping_world import SleepingWorld
    n = int(scene_fn().bodies.count)
    sl = dict(time_to_sleep=0.2, thr_lin=np.full(n, 0.5, np.float32), thr_ang=np.full(n, 0.5, np.float32))
    wa = SleepingWorld(scene_fn(), plugins.PhysicsPlugins(ctx_a), sl, substeps=4, events_enabled=np.ones(n, dtype=bool))
    wb = plugins.DeviceGraphWorld(scene_fn(), plugins.PhysicsPlugins(ctx_b), ctx_b, sleeping=sl, substeps=4, events_enabled=np.ones(n, dtype=bool))
    return wa, wb


def _step_pair(wa, wb):
    wa.broad_phase(); wa.narrow_phase(); wa.solve(); wa.step_index += 1
    wb.step()


TIMER_DIVERGENCE = ("the device's per-body sleep timers and sleeping_world's diverge on random piles with sleeping applied, and the islands and "
                    "asleep rows follow a few steps later; the same happens on cube / sphere piles with no capsule at the commit before capsules "
                    "existed (test_sleep_timers_of_a_cube_and_sphere_pile), so it is tracked separately (DESIGN.md §7h)")


@pytest.mark.xfail(strict=True, reason=TIMER_DIVERGENCE)
@pytest.mark.parametrize("seed", [6, 7, 8])
def test_capsule_pile_with_sleeping_and_events_equals_the_reference_world(gpu_ctx, seed):
    """scenes.capsule_pile with sleeping applied and collision events on, against sleeping_world, every step: rows, islands, Sleeping flags,
    colours, events and bodies bit for bit.  Expected to fail until the timer divergence is fixed; the resting log piles below meet the same
    bar today."""
    scene_fn = lambda: scenes.capsule_pile(120, seed=seed, layers=2)   # noqa: E731
    with api.Context(device=0) as ctx_a, api.Context(device=0) as ctx_b:
        wa, wb = _sleeping_pair(scene_fn, ctx_a, ctx_b)
        slept = started = 0
        for i in range(150):
            _step_pair(wa, wb)
            _check_but_timers(wa, wb, ctx_b, i)
            assert wa.events is not None and wb.events is not None
            for x, y in zip(wa.events, wb.events):
                for k in x:
                    assert np.array_equal(x[k], y[k]), f"step {i}: events {k}"
            slept += wb.islands["islands_put_to_sleep"]
            started += len(wb.events[0]["collider1"])
        assert started > 0 and slept > 0, (started, slept)


@pytest.mark.xfail(strict=True, reason=TIMER_DIVERGENCE)
def test_sleep_timers_of_a_cube_and_sphere_pile(gpu_ctx):
    """the same divergence with no capsule in the scene: the capsule kernels never launch, and every kernel this pile runs is the one of the
    commit before capsules (byte-identical bench outputs); the first divergence (step 34, bodies 21 and 60) is the same there"""
    scene_fn = lambda: scenes.capsule_pile(120, seed=6, layers=2, capsule_share=0.0, sphere_share=0.5)   # noqa: E731
    with api.Context(device=0) as ctx_a, api.Context(device=0) as ctx_b:
        wa, wb = _sleeping_pair(scene_fn, ctx_a, ctx_b)
        for i in range(60):
            _step_pair(wa, wb)
            assert np.array_equal(wa.sleep_timer, wb.sleep_timer), f"step {i}: sleep timers"


def test_capsule_piles_with_sleeping_equal_the_reference_world(gpu_ctx):
    """four log-cabin capsule piles with sleeping applied and collision events on: they land, come to rest and fall asleep"""
    scene_fn = lambda: log_piles(4)   # noqa: E731
    n = int(scene_fn().bodies.count)
    sleeping = dict(time_to_sleep=0.2, thr_lin=np.full(n, 0.5, np.float32), thr_ang=np.full(n, 0.5, np.float32))
    with api.Context(device=0) as ctx_a, api.Context(device=0) as ctx_b:
        p = _Pair(scene_fn, ctx_a, ctx_b, sleeping, events_enabled=np.ones(n, dtype=bool))
        for _ in range(150):
            p.step()
        assert p.slept > 0, "nothing went to sleep"


def _pile_world(ctx, **kw):
    return plugins.DeviceGraphWorld(scenes.capsule_pile(100, seed=8, layers=2), plugins.PhysicsPlugins(ctx), ctx, substeps=4, **kw)


def test_refusals_leave_the_context_unchanged(gpu_ctx):
    with api.Context(device=0) as ctx_a, api.Context(device=0) as ctx_b:
        wa, wb = _pile_world(ctx_a), _pile_world(ctx_b)
        for _ in range(20):
            wa.step(); wb.step()
        b = wb.bodies
        good = dict(shape=wb._shape, dims=wb._dims, position=b.position, rotation=b.rotation, aabb_min=wb.aabb_min, aabb_max=wb.aabb_max)
        cap = int(np.nonzero(wb._shape == CAP)[0][0])
        bad_shape = wb._shape.copy(); bad_shape[3] = 3
        bad_dims = wb._dims.copy(); bad_dims[cap, 0] = -0.1
        bad_len = wb._dims.copy(); bad_len[cap, 1] = -0.5
        for cols in (dict(good, shape=bad_shape), dict(good, dims=bad_dims), dict(good, dims=bad_len)):
            with pytest.raises(api.AvianError) as e:
                ctx_b.contacts_step(wb.params.dt, 0.005, cols, b.linear_velocity, b.angular_velocity, take_pairs=False)
            assert e.value.status == api.ERR_INVALID_ARGUMENT, str(e.value)
            pr = (np.array([cap], np.uint32), np.array([0], np.uint32), np.array([cap], np.uint32), np.array([0], np.uint32))
            with pytest.raises(api.AvianError) as e:
                ctx_b.narrow_phase(wb.params.dt, 0.005, pr, {k: cols[k] for k in ("shape", "dims", "position", "rotation")}, b.linear_velocity, b.angular_velocity)
            assert e.value.status == api.ERR_INVALID_ARGUMENT, str(e.value)
            with pytest.raises(api.AvianError) as e:
                ctx_b.update_aabbs(api.AvnAabbParams(wb.params.dt, 0.005, float("inf")),
                                   api.Colliders(shape=cols["shape"], dims=cols["dims"], position=b.position, rotation=b.rotation))
            assert e.value.status == api.ERR_INVALID_ARGUMENT, str(e.value)
        for i in range(20):     # the next valid steps are those of the world that saw no refused call
            wa.step(); wb.step()
            for k in COLS:
                assert np.array_equal(getattr(wa.bodies, k), getattr(wb.bodies, k)), f"step {i}: {k}"
    # swept CCD with a capsule in the shape column: the step's solver stage is refused before anything runs, the bodies stay as they were
    with api.Context(device=0) as ctx:
        w = _pile_world(ctx, ccd=dict(body=np.array([1], dtype=np.uint32), collider=np.array([1], dtype=np.uint32)))
        before = {k: getattr(w.bodies, k).copy() for k in COLS}
        with pytest.raises(api.AvianError) as e:
            w.step()
        assert e.value.status == api.ERR_UNSUPPORTED and "capsule" in str(e.value), str(e.value)
        for k in COLS:
            assert np.array_equal(getattr(w.bodies, k), before[k]), k
    # configuring swept CCD once the contact store holds capsules is refused as well; with the configuration cleared the world steps on
    with api.Context(device=0) as ctx:
        w = _pile_world(ctx)
        w.step()
        with pytest.raises(api.AvianError) as e:
            ctx.ccd_configure(body=np.array([1], dtype=np.uint32), collider=np.array([1], dtype=np.uint32))
        assert e.value.status == api.ERR_UNSUPPORTED and "capsule" in str(e.value), str(e.value)
        w.step()


def test_host_ccd_refuses_capsules():
    bodies = dict(kind=np.array([api.BODY_STATIC, api.BODY_DYNAMIC], np.uint8), position=np.array([[0, -0.5, 0], [0, 1, 0]], np.float32),
                  rotation=np.array([[0, 0, 0, 1.0]] * 2, np.float32), linear_velocity=np.array([[0, -50, 0]] * 2, np.float32),
                  angular_velocity=np.zeros((2, 3), np.float32))
    rows = dict(c1=np.array([0]), c2=np.array([1]), b1=np.array([0]), b2=np.array([1]), live=np.array([1]))
    with pytest.raises(api.AvianError) as e:
        fixture.ccd_solve(np.float32, 1 / 60, 1.0, bodies, np.array([BOX, CAP]), np.array([[5, 0.5, 5], [0.2, 0.5, 0]]), rows,
                          dict(body=np.array([1]), collider=np.array([1])))
    assert e.value.status == api.ERR_UNSUPPORTED
