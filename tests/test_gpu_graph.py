"""The ContactGraph and the ConstraintGraph on the device (SURVEY.md 8f #3; avn_contacts_configure / avn_contacts_step /
avn_solver_upload_resident): DeviceGraphWorld against the ordinary GPU World, whose graphs live in the host fixture (a restatement of
contact_graph.rs:521-631 and constraint_graph.rs:163-296).  Every step: the same ContactId for every pair, the same colour for every manifold,
the overflow colour in the same list order, the impulses the solve leaves in the rows, and the bodies bit for bit — i.e. nothing of the
contact pipeline needs the host any more."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
from avian_b200 import api, plugins, scenes  # noqa: E402

pytestmark = pytest.mark.gpu


def _tumble(w, seed=5):
    rng = np.random.default_rng(seed)
    dyn = w.bodies.kind == api.BODY_DYNAMIC
    w.bodies.linear_velocity[dyn] = rng.normal(0, 2.0, size=(int(dyn.sum()), 3)).astype(w.scalar)
    w.bodies.angular_velocity[dyn] = rng.normal(0, 3.0, size=(int(dyn.sum()), 3)).astype(w.scalar)


def _plate_on_cubes(n_side):
    """a plate resting on n_side^2 cubes: the plate collects n_side^2 manifolds — more than the 23 colours hold for n_side = 5 (overflow colour)"""
    cubes = np.array([[1.5 * ix, 0.49, 1.5 * iz] for ix in range(n_side) for iz in range(n_side)])
    mid, n = 0.75 * (n_side - 1), n_side * n_side
    pos = np.concatenate([[[mid, -0.5, mid]], cubes, [[mid, 1.22, mid]]])
    he = np.concatenate([[[20.0, 0.5, 20.0]], np.full((n, 3), 0.5), [[0.75 * n_side + 0.5, 0.25, 0.75 * n_side + 0.5]]])
    kind = np.concatenate([[api.BODY_STATIC], np.full(n + 1, api.BODY_DYNAMIC)])
    rot = np.tile(np.array([0.0, 0.0, 0.0, 1.0]), (n + 2, 1))
    return scenes._assemble(f"plate_on_{n}_cubes", pos, rot, kind, he, np.full(n + 2, scenes.SHAPE_CUBOID), np.float32)


def _host_graph(w):
    """the fixture's graphs: pairs by ContactId and the colour-major edge list"""
    p = w.pipeline
    ids, c1, c2, _, _ = p.active_edges()
    m = w.last_manifolds.count if w.last_manifolds is not None else 0
    co, edge, *_ = p.export_edges(m)
    return ids, c1, c2, co, edge


def _check_graphs(wa, wb, ctx_b, step):
    ids, c1, c2, co, edge = _host_graph(wa)
    st = wb.stats
    assert st["rows_live"] == ids.shape[0], f"step {step}: live pairs {st['rows_live']} != {ids.shape[0]}"
    assert st["manifold_count"] == edge.shape[0], f"step {step}: manifolds {st['manifold_count']} != {edge.shape[0]}"
    assert np.array_equal(st["color_offsets"], co), f"step {step}: colour offsets\n{st['color_offsets']}\n{co}"
    hw = st["rows_high_water"]
    g = ctx_b.contacts_download_graph(hw, st["manifold_count"])
    live = np.zeros(hw, dtype=bool); live[ids] = True
    assert np.array_equal(g["live"].astype(bool), live), f"step {step}: the ContactIds in use differ"
    assert np.array_equal(g["collider1"][ids], c1) and np.array_equal(g["collider2"][ids], c2), f"step {step}: a pair sits in another row"
    colour = np.full(hw, -1, dtype=np.int8)
    for c in range(api.GRAPH_COLOR_COUNT):
        colour[edge[co[c]:co[c + 1]]] = c
    assert np.array_equal(g["colour"], colour), f"step {step}: colours differ for rows {np.nonzero(g['colour'] != colour)[0][:10]}"
    for c in range(api.GRAPH_COLOR_COUNT):        # same members per colour; the overflow colour (solved serially) in the same ORDER
        mine, theirs = g["edge"][co[c]:co[c + 1]], edge[co[c]:co[c + 1]]
        if c == api.COLOR_OVERFLOW:
            assert np.array_equal(mine, theirs), f"step {step}: overflow colour order"
        else:
            assert np.array_equal(mine, np.sort(theirs)), f"step {step}: colour {c}"


def _check_impulses(wa, wb, ctx_b, step):
    """store_contact_impulses into the rows: the rows of the World's colour-major ContactIds hold the World's manifold columns, point by point"""
    ma = wa.last_manifolds
    if ma is None or not ma.count:
        return
    _, _, _, _, edge = _host_graph(wa)
    wn, _, ni = ctx_b.contacts_download_impulses(wb.stats["rows_high_water"])
    slot = np.arange(4)[None, :] < np.diff(ma.point_offsets.astype(np.int64))[:, None]
    assert np.array_equal(wn[edge][slot], ma.warm_start_normal_impulse), f"step {step}: warm-start impulses"
    assert np.array_equal(ni[edge][slot], ma.normal_impulse), f"step {step}: normal impulses"


@pytest.mark.parametrize("scene_fn,steps,substeps,kick", [
    (lambda: scenes.cubes_example(4), 70, 4, True),                   # tumbling cubes: pairs appear, separate, ContactIds are reused
    (lambda: scenes.cube_stack(6, 5, 5, brick=True), 12, 4, False),   # a settling brick pile: contacts start and stop touching
    (lambda: _plate_on_cubes(5), 25, 4, False),                       # 25 manifolds on one body: the overflow colour
    (lambda: scenes.falling_spheres(400, seed=3, box=(6.0, 4.0, 6.0), scalar=np.float64), 30, 4, False),   # f64, sphere contacts
    (lambda: scenes.ragdoll_field(9, pitch=1.2, drop_height=0.5), 40, 4, False),                          # joints next to the contacts
])
def test_device_graphs_equal_the_host_graphs(gpu_ctx, scene_fn, steps, substeps, kick):
    sc_a, sc_b = scene_fn(), scene_fn()
    scalar = sc_a.bodies.position.dtype
    with api.Context(device=0, scalar=scalar) as ctx_a, api.Context(device=0, scalar=scalar) as ctx_b:
        wa = plugins.World(sc_a, plugins.PhysicsPlugins(ctx_a), substeps=substeps)
        wb = plugins.DeviceGraphWorld(sc_b, plugins.PhysicsPlugins(ctx_b), ctx_b, substeps=substeps)
        if kick:
            _tumble(wa); _tumble(wb)
        added = removed = started = stopped = 0
        for i in range(steps):
            wa.step(); wb.step()
            _check_graphs(wa, wb, ctx_b, i)
            _check_impulses(wa, wb, ctx_b, i)
            for k in ("position", "rotation", "linear_velocity", "angular_velocity"):
                assert np.array_equal(getattr(wa.bodies, k), getattr(wb.bodies, k)), f"step {i}: {k}"
            st = wb.stats
            added += st["pairs_added"]; removed += st["pairs_removed"]; started += st["started_touching"]; stopped += st["stopped_touching"]
        assert added > 0 and started > 0
        if kick:
            assert removed > 0 and stopped > 0, "the scene was meant to separate pairs and reuse their ContactIds"


def test_overflow_colour_is_exercised(gpu_ctx):
    sc = _plate_on_cubes(5)
    with api.Context(device=0) as ctx:
        w = plugins.DeviceGraphWorld(sc, plugins.PhysicsPlugins(ctx), ctx, substeps=4)
        for _ in range(6):
            w.step()
        co = w.stats["color_offsets"]
        assert co[api.COLOR_OVERFLOW + 1] - co[api.COLOR_OVERFLOW] >= 2, co


def test_first_frame_of_a_pile_and_the_steady_state(gpu_ctx):
    """~10k cubes: the first frame colours every manifold at once (a deep dependency wavefront), later steps only touch what changed."""
    sc = scenes.cube_stack(23, 20, 22, brick=True)
    with api.Context(device=0) as ctx_a, api.Context(device=0) as ctx_b:
        wa = plugins.World(scenes.cube_stack(23, 20, 22, brick=True), plugins.PhysicsPlugins(ctx_a), substeps=8)
        wb = plugins.DeviceGraphWorld(sc, plugins.PhysicsPlugins(ctx_b), ctx_b, substeps=8)
        rounds = []
        for i in range(3):
            wa.step(); wb.step()
            rounds.append(wb.stats["colouring_rounds"])
            _check_graphs(wa, wb, ctx_b, i)
            for k in ("position", "linear_velocity"):
                assert np.array_equal(getattr(wa.bodies, k), getattr(wb.bodies, k)), f"step {i}: {k}"
        assert wb.stats["manifold_count"] > 30_000
        print("colouring rounds per step:", rounds)


def test_pairs_outside_the_configured_counts_are_refused(gpu_ctx):
    """the rows are gathered through on the device: a new pair that names a body or collider beyond avn_contacts_configure's counts is not
    added and the step reports AVN_ERR_INVALID_ARGUMENT instead of reading out of bounds"""
    sc = scenes.cube_stack(3, 2, 3, brick=True)
    with api.Context(device=0) as ctx:
        w = plugins.DeviceGraphWorld(sc, plugins.PhysicsPlugins(ctx), ctx, substeps=2)
        mn, mx = w.pipeline.update_aabbs(w.bodies, w.params.dt)
        aabbs = w.intervals(mn, mx)
        aabbs.body = aabbs.body.copy(); aabbs.body[3] = 9999          # a collider whose ColliderOf::body is not among the configured bodies
        with pytest.raises(api.AvianError) as e:
            w.step_from(aabbs, mn, mx)
        assert e.value.status == api.ERR_INVALID_ARGUMENT and "not added" in str(e.value), str(e.value)
        # and a step whose inputs outgrow the configuration is refused up front
        ctx.contacts_configure(w.bodies.kind[:5], 5, sc.friction[:5], sc.restitution[:5])
        with pytest.raises(api.AvianError) as e:
            w.step()
        assert e.value.status == api.ERR_INVALID_ARGUMENT
