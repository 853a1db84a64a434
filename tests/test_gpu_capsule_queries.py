"""Capsules in the device spatial queries and move and slide (H100): every avn_query_* entry point and avn_move_and_slide against the
capsule-enabled host brute force (fixture.query_* / fixture.move_and_slide with capsules=True, the same csrc/query_math.hpp and
csrc/move_math.hpp over every collider), bit for bit, f32 and f64.  Trees and batches without a capsule run the kernels' CAPS = false
instances; the existing GPU query tests pin those."""
from __future__ import annotations

import math

import numpy as np
import pytest

from avian_b200 import api, fixture, plugins, scenes
from move_scenes import random_characters, random_colliders, random_quats

pytestmark = pytest.mark.gpu
SCALARS = [np.float32, np.float64]
IDENT = [0.0, 0.0, 0.0, 1.0]
CUB, SPH, CAP = fixture.SHAPE_CUBOID, fixture.SHAPE_SPHERE, fixture.SHAPE_CAPSULE
MOVE_OUTPUTS = ("position", "velocity", "hit_collider", "hit_distance", "hit_toi", "hit_point", "hit_normal")


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({1: np.uint8, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def assert_same(dev: dict, host: dict, what: str = "", keys=None):
    for k in (keys or host):
        if k == "kernel_ms":
            continue
        assert dev[k].shape == host[k].shape, f"{what}{k}: {dev[k].shape} vs {host[k].shape}"
        a, b = _bits(dev[k]), _bits(host[k])
        assert np.array_equal(a, b), f"{what}{k} differs at rows {np.nonzero((a != b).reshape(a.shape[0], -1).any(axis=1))[0][:10]}"


def unit(v):
    v = np.asarray(v, dtype=np.float64)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def mixed_dims(rng, shape):
    n = shape.shape[0]
    dims = rng.uniform(0.2, 1.5, (n, 3))
    caps = shape == CAP
    dims[caps, 0] = rng.uniform(0.1, 0.8, caps.sum())
    dims[caps, 1] = rng.uniform(0.0, 1.5, caps.sum())
    return dims


def mixed_scene(rng, n, extent=20.0):
    shape = rng.integers(0, 3, n).astype(np.uint8)                  # a third each: cuboids, spheres, capsules
    return api.QueryColliders(shape=shape, dims=mixed_dims(rng, shape), position=rng.uniform(-extent, extent, (n, 3)), rotation=random_quats(rng, n),
                              memberships=np.where(rng.random(n) < 0.2, 2, 1).astype(np.uint32))


def mixed_shapes(rng, m, extent=20.0, cast=True, **kw):
    shape = rng.integers(0, 3, m).astype(np.uint8)
    dims = mixed_dims(rng, shape) * 0.6
    extra = dict(direction=unit(rng.normal(size=(m, 3))), max_distance=rng.uniform(2, 30, m)) if cast else {}
    return api.ShapeQueries(shape=shape, dims=dims, position=rng.uniform(-extent, extent, (m, 3)), rotation=random_quats(rng, m), **extra, **kw)


def check_all(ctx, s, cols, rays=None, casts=None, points=None, isect=None, boxes=None, what=""):
    """device == capsule-enabled brute force for every batch given"""
    ctx.query_update(cols)
    H = dict(capsules=True)
    if rays is not None:
        assert_same(ctx.cast_ray(rays), fixture.query_cast_ray(s, cols, rays, **H), what + "cast_ray ")
        assert_same(ctx.ray_hits(rays), fixture.query_ray_hits(s, cols, rays, **H), what + "ray_hits ")
    if boxes is not None:
        assert_same(ctx.aabb_intersections(*boxes), fixture.query_aabb_intersections(s, cols, *boxes, **H), what + "aabb_intersections ")
    if casts is not None:
        assert_same(ctx.cast_shape(casts), fixture.query_cast_shape(s, cols, casts, **H), what + "cast_shape ")
        assert_same(ctx.shape_hits(casts), fixture.query_shape_hits(s, cols, casts, **H), what + "shape_hits ")
    if points is not None:
        assert_same(ctx.project_point(points), fixture.query_project_point(s, cols, points, **H), what + "project_point ")
        assert_same(ctx.point_intersections(points), fixture.query_point_intersections(s, cols, points, **H), what + "point_intersections ")
    if isect is not None:
        assert_same(ctx.shape_intersections(isect), fixture.query_shape_intersections(s, cols, isect, **H), what + "shape_intersections ")


@pytest.fixture(scope="module", params=SCALARS, ids=["f32", "f64"])
def qctx(request):
    ctx = api.Context(device=0, scalar=request.param)
    yield ctx, request.param
    ctx.close()


def test_random_mixed_scene(qctx):
    ctx, s = qctx
    rng = np.random.default_rng(41)
    n, m = 10_000, 2_000
    cols = mixed_scene(rng, n)
    excl = [rng.integers(0, n, size=rng.integers(0, 3)).tolist() for _ in range(m)]
    mask = np.where(rng.random(m) < 0.2, 1, 0xFFFFFFFF).astype(np.uint32)
    o = rng.uniform(-22, 22, (m, 3))
    rays = api.Rays(origin=o, direction=unit(rng.normal(size=(m, 3))), max_distance=rng.uniform(2, 40, m), solid=rng.random(m) < 0.5,
                    max_hits=rng.integers(0, 8, m).astype(np.uint32), mask=mask, exclude=excl)
    casts = mixed_shapes(rng, m, flags=rng.integers(0, 4, m).astype(np.uint32), mask=mask, exclude=excl, max_hits=rng.integers(0, 8, m).astype(np.uint32))
    pts = api.Points(point=rng.uniform(-22, 22, (m, 3)), solid=rng.random(m) < 0.5, mask=mask, exclude=excl)
    isect = mixed_shapes(rng, m, cast=False, mask=mask, exclude=excl)
    c = rng.uniform(-20, 20, (m, 3))
    boxes = ((c - 1.0).astype(s), (c + 1.0).astype(s))
    check_all(ctx, s, cols, rays, casts, pts, isect, boxes, what="mixed ")
    r = ctx.cast_shape(casts)
    hit = r["collider"] >= 0
    assert hit.sum() > m // 3
    assert (cols.shape[r["collider"][hit]] == CAP).sum() > 50 and (casts.shape[hit] == CAP).sum() > 50
    # a cuboid / sphere batch against the capsule tree, and a capsule batch against a tree without capsules (SHAPES_UNCHANGED keeps the flag)
    plain = mixed_shapes(rng, 500)
    plain.shape[plain.shape == CAP] = SPH
    check_all(ctx, s, cols, casts=plain, what="plain-batch ")
    ctx.query_update(cols, shapes_unchanged=True)
    assert_same(ctx.cast_shape(plain), fixture.query_cast_shape(s, cols, plain, capsules=True), "unchanged ")
    boxes_only = api.QueryColliders(shape=np.where(cols.shape == CAP, CUB, cols.shape).astype(np.uint8), dims=cols.dims, position=cols.position,
                                    rotation=cols.rotation)
    check_all(ctx, s, boxes_only, casts=casts, isect=isect, what="capsule-batch ")


def test_grazing_rays(qctx):
    """tangent to the cylinder (and one ulp past it), through the seam, end-on along the axis, from inside, solid and hollow"""
    ctx, s = qctx
    k = 40
    g = np.arange(k, dtype=float) * 4.0
    cols = api.QueryColliders(shape=np.full(k, CAP, np.uint8), dims=np.tile([0.5, 1.0, 0.0], (k, 1)), position=np.stack([g, np.zeros(k), np.zeros(k)], 1),
                              rotation=np.tile(IDENT, (k, 1)))
    up = float(np.nextafter(0.5, 1.0))
    o, d, solid = [], [], []
    for x in g:
        for oo, dd in (([x, 5.0, 0.5], [0, -1.0, 0]), ([x - 1.5, 0.3, 0.5], [1.0, 0, 0]), ([x - 1.5, 0.3, up], [1.0, 0, 0]),
                           ([x - 1.5, 1.0, 0.0], [1.0, 0, 0]), ([x, 5.0, 0.0], [0, -1.0, 0]), ([x + 0.1, 0.2, 0.0], [1.0, 0, 0]),
                           ([x + 0.1, 0.2, 0.0], [0, 1.0, 0]), ([x, 0.0, 0.0], [0, 0, 1.0])):
            o.append(oo); d.append(dd)
            solid.append(len(solid) % 2 == 0)
    rays = api.Rays(origin=np.array(o), direction=np.array(d), max_distance=np.full(len(o), 1.6), solid=np.array(solid, np.uint8))
    pts = api.Points(point=np.array(o), solid=np.array(solid, np.uint8))
    check_all(ctx, s, cols, rays=rays, points=pts, what="grazing ")


def settled_capsule_pile(steps=60):
    with api.Context(device=0) as ctx:
        w = plugins.DeviceGraphWorld(scenes.capsule_pile(3000, seed=5, layers=4), plugins.PhysicsPlugins(ctx), ctx, substeps=4)
        for _ in range(steps):
            w.step()
        return plugins.SpatialQueryPlugin.colliders(w)


def stack_cols():
    sc = scenes.cube_stack(51, 40, 50, brick=True)
    return api.QueryColliders(shape=sc.shape_type.astype(np.uint8), dims=sc.dims, position=np.asarray(sc.bodies.position, np.float64),
                              rotation=np.asarray(sc.bodies.rotation, np.float64))


def down_casts(lo, hi, y, k, rng):
    o = np.stack([rng.uniform(lo[0], hi[0], k), np.full(k, y), rng.uniform(lo[1], hi[1], k)], 1)
    shape = np.where(np.arange(k) % 3 == 0, SPH, CAP).astype(np.uint8)
    dims = np.tile([0.4, 0.5, 0.0], (k, 1))                         # the reference's character capsule: radius 0.4, length 1.0
    rot = random_quats(rng, k)
    rot[: k // 2] = IDENT
    return api.ShapeQueries(shape=shape, dims=dims, position=o, rotation=rot, direction=np.tile([0.0, -1.0, 0.0], (k, 1)),
                            max_distance=np.full(k, 200.0), max_hits=np.full(k, 4, np.uint32))


def test_casts_and_projections_onto_a_settled_capsule_pile(qctx):
    ctx, s = qctx
    cols = settled_capsule_pile()
    rng = np.random.default_rng(42)
    lo, hi = cols.position[:, [0, 2]].min(0), cols.position[:, [0, 2]].max(0)
    casts = down_casts(lo, hi, float(cols.position[:, 1].max()) + 5, 600, rng)
    c = cols.position[rng.integers(0, cols.shape.shape[0], 600)]
    pts = api.Points(point=c + rng.uniform(-0.6, 0.6, c.shape), solid=rng.random(600) < 0.5)
    rays = api.Rays(origin=casts.position, direction=casts.direction, max_distance=casts.max_distance)
    check_all(ctx, s, cols, rays=rays, casts=casts, points=pts, isect=api.ShapeQueries(shape=casts.shape, dims=casts.dims, position=c, rotation=casts.rotation),
              what="pile ")
    assert (ctx.cast_shape(casts)["collider"] >= 0).mean() > 0.5


def test_capsule_casts_onto_the_100k_stack_sample(qctx):
    """100k casts on the device, a sample of them against the brute force over all 100k colliders"""
    ctx, s = qctx
    cols = stack_cols()
    rng = np.random.default_rng(43)
    lo, hi = cols.position[1:, [0, 2]].min(0), cols.position[1:, [0, 2]].max(0)
    casts = down_casts(lo, hi, float(cols.position[1:, 1].max()) + 3, 100_000, rng)
    ctx.query_update(cols)
    dev = ctx.cast_shape(casts)
    assert (dev["collider"] >= 0).mean() > 0.9
    idx = np.sort(rng.choice(casts.count, 24, replace=False))
    sub = api.ShapeQueries(shape=casts.shape[idx], dims=casts.dims[idx], position=casts.position[idx], rotation=casts.rotation[idx],
                           direction=casts.direction[idx], max_distance=casts.max_distance[idx])
    want = fixture.query_cast_shape(s, cols, sub, capsules=True)
    assert_same({k: v[idx] for k, v in dev.items()}, want, "stack sample ")
    # projections onto the stack from capsule-shaped neighbourhoods: points near the top faces
    pts = api.Points(point=np.stack([casts.position[idx, 0], np.full(idx.size, float(cols.position[1:, 1].max()) + 0.7), casts.position[idx, 2]], 1))
    assert_same(ctx.project_point(pts), fixture.query_project_point(s, cols, pts, capsules=True), "stack project ")


def _world_check(ctx_q, s, w, rng, what):
    cols = plugins.SpatialQueryPlugin.colliders(w)
    n = cols.shape.shape[0]
    lo, hi = cols.position.min(0), cols.position.max(0)
    k = 400
    o = rng.uniform(lo - 2, hi + 2, (k, 3))
    o[:, 1] = hi[1] + 4
    rays = plugins.SpatialQueryPlugin.ray_casters(o, unit(rng.normal(size=(k, 3)) * [0.3, 1.0, 0.3] - [0, 2.0, 0]), np.full(k, 40.0),
                                                  max_hits=np.full(k, 3), owner=rng.integers(-1, n, k))
    sp = plugins.SpatialQueryPlugin(ctx_q)
    sp.update_pipeline(w)
    assert_same(sp.raycast(rays), fixture.query_ray_hits(s, cols, rays, capsules=True), what + "raycast ")
    shape = np.where(np.arange(k) % 2 == 0, CAP, SPH).astype(np.uint8)
    casters = plugins.SpatialQueryPlugin.shape_casters(shape, np.tile([0.4 * 0.99, 0.5 * 0.99, 0.0], (k, 1)), o, np.tile(IDENT, (k, 1)),
                                                       np.tile([0.0, -1.0, 0.0], (k, 1)), max_hits=np.full(k, 2), owner=rng.integers(-1, n, k))
    assert_same(sp.shapecast(casters), fixture.query_shape_hits(s, cols, casters, capsules=True), what + "shapecast ")


@pytest.mark.parametrize("scene", ["capsule_pile", "compound_pile"])
def test_plugin_queries_follow_the_device_world(scene):
    """SpatialQueryPlugin ray casts and ShapeCaster casts (a slightly shrunk character capsule, as the reference's ground detection) after
    DeviceGraphWorld steps on the shipped capsule and compound scenes"""
    make = {"capsule_pile": lambda: scenes.capsule_pile(800, seed=9, layers=3), "compound_pile": lambda: scenes.compound_pile(300, seed=4)}[scene]
    rng = np.random.default_rng(44)
    with api.Context(device=0) as ctx, api.Context(device=0) as qc:
        w = plugins.DeviceGraphWorld(make(), plugins.PhysicsPlugins(ctx), ctx, substeps=4)
        for step in range(40):
            w.step()
            if step in (0, 19, 39):
                _world_check(qc, np.float32, w, rng, f"{scene} step {step} ")


# ---- move and slide ------------------------------------------------------------------------------------------------------------------------
def assert_move_same(got, want, what=""):
    for k in MOVE_OUTPUTS:
        a, b = np.ascontiguousarray(got[k]), np.ascontiguousarray(want[k])
        assert a.shape == b.shape, (what, k)
        bad = np.flatnonzero((a.view(np.uint8).reshape(a.shape[0], -1) != b.view(np.uint8).reshape(b.shape[0], -1)).any(axis=1))
        assert bad.size == 0, f"{what} {k}: {bad.size} characters differ, first {bad[:5]}: {a[bad[0]]} vs {b[bad[0]]}"


def take(b: "api.MoveBatch", idx) -> "api.MoveBatch":
    pick = lambda a: None if a is None else np.asarray(a)[idx]
    lst = lambda a: None if a is None else [a[i] for i in idx]
    return api.MoveBatch(shape=pick(b.shape), dims=pick(b.dims), position=pick(b.position), rotation=pick(b.rotation), velocity=pick(b.velocity),
                         mask=pick(b.mask), exclude=lst(b.exclude), planes=lst(b.planes))


CONFIGS = {
    "default": api.MoveConfig(),
    "0-iterations": api.MoveConfig(move_and_slide_iterations=0),
    "1-iteration": api.MoveConfig(move_and_slide_iterations=1),
    "8-iterations": api.MoveConfig(move_and_slide_iterations=8, length_unit=2.0),
    "no-depenetration": api.MoveConfig(depenetration_iterations=0),
    "max-planes-3": api.MoveConfig(max_planes=3, plane_similarity_dot_threshold=0.9),
}


@pytest.fixture(scope="module")
def capsule_move_scene():
    rng = np.random.default_rng(2025)
    cols, ignored = random_colliders(rng, 6_000, 20.0)
    caps = rng.random(cols.shape.shape[0]) < 0.33
    cols.shape[caps] = CAP
    cols.dims[caps, 0] = rng.uniform(0.15, 0.7, caps.sum())
    batch = random_characters(rng, 1_200, 20.0, 6_000)
    batch.shape[np.arange(batch.count) % 3 != 2] = CAP                # capsule and mixed characters
    return cols, ignored, batch


@pytest.mark.parametrize("scalar", SCALARS, ids=lambda s: np.dtype(s).name)
@pytest.mark.parametrize("name", list(CONFIGS))
def test_capsule_characters_match_host(capsule_move_scene, name, scalar):
    cols, ignored, batch = capsule_move_scene
    cfg = CONFIGS[name]
    cfg.ignored = ignored
    if name != "default":
        batch = take(batch, np.arange(400))
    with api.Context(device=0, scalar=scalar) as ctx:
        ctx.query_update(cols)
        got = ctx.move_and_slide(cfg, batch)
    want = fixture.move_and_slide(scalar, cols, cfg, batch, capsules=True)
    assert_move_same(got, want, name)
    if cfg.move_and_slide_iterations:
        assert (want["hit_collider"] >= 0).sum() > 40


@pytest.mark.parametrize("scalar", SCALARS, ids=lambda s: np.dtype(s).name)
def test_capsule_characters_in_a_dense_pile(scalar):
    """every character's grown AABB holds more than three windows of K = 16 candidates"""
    rng = np.random.default_rng(8)
    n = 3000
    shape = np.where(np.arange(n) % 2 == 0, CAP, SPH).astype(np.uint8)
    cols = api.QueryColliders(shape=shape, dims=np.tile([0.06, 0.05, 0.0], (n, 1)), position=rng.uniform(-1.2, 1.2, (n, 3)), rotation=random_quats(rng, n))
    m = 200
    batch = api.MoveBatch(shape=np.full(m, CAP, np.uint8), dims=np.tile([0.3, 0.2, 0.0], (m, 1)), position=rng.uniform(-0.8, 0.8, (m, 3)),
                          rotation=random_quats(rng, m), velocity=rng.normal(size=(m, 3)) * 20)
    cfg = api.MoveConfig(penetration_rejection_threshold=2.0, depenetration_iterations=4)
    with api.Context(device=0, scalar=scalar) as ctx:
        ctx.query_update(cols)
        g = 0.3 + 0.2 + 0.02
        cand = ctx.aabb_intersections((batch.position - g).astype(scalar), (batch.position + g).astype(scalar))
        assert np.diff(cand["offsets"].astype(np.int64)).min() > 3 * 16
        got = ctx.move_and_slide(cfg, batch)
    assert_move_same(got, fixture.move_and_slide(scalar, cols, cfg, batch, capsules=True), "pile")


@pytest.mark.parametrize("scalar", SCALARS, ids=lambda s: np.dtype(s).name)
def test_capsule_walkers_on_the_100k_stack(scalar):
    rng = np.random.default_rng(4)
    cols = stack_cols()
    n = 100_000
    top = float(cols.position[1:, 1].max()) + 0.5
    lo, hi = cols.position[1:, [0, 2]].min(axis=0), cols.position[1:, [0, 2]].max(axis=0)
    pos = np.stack([rng.uniform(lo[0], hi[0], n), top + 0.9 + rng.uniform(-0.05, 0.05, n), rng.uniform(lo[1], hi[1], n)], 1)
    a = rng.uniform(0, 2 * math.pi, n)
    vel = np.stack([np.cos(a) * 6, rng.uniform(-10, 0, n), np.sin(a) * 6], 1)
    planes = [np.array([[0.0, 1.0, 0.0]]) if i % 2 else None for i in range(n)]
    batch = api.MoveBatch(shape=np.full(n, CAP, np.uint8), dims=np.tile([0.4, 0.5, 0.0], (n, 1)), position=pos, rotation=np.tile(IDENT, (n, 1)),
                          velocity=vel, planes=planes)
    cfg = api.MoveConfig()
    with api.Context(device=0, scalar=scalar) as ctx:
        ctx.query_update(cols)
        got = ctx.move_and_slide(cfg, batch)
    for k in ("position", "velocity"):
        assert np.isfinite(got[k]).all(), k
    assert (got["hit_collider"] >= 0).sum() > 10_000
    idx = np.sort(rng.choice(n, 500, replace=False))
    want = fixture.move_and_slide(scalar, cols, cfg, take(batch, idx), capsules=True)
    assert_move_same({k: got[k][idx] for k in MOVE_OUTPUTS}, want, "stack sample")
