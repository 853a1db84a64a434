"""Convex hulls in the device spatial queries and move and slide (H100): every avn_query_* entry point and avn_move_and_slide against the
hull-enabled host brute force (fixture.query_* / fixture.move_and_slide with hulls=, the same csrc/hull_query_math.hpp and csrc/move_math.hpp
over every collider), bit for bit, f32 and f64.  Trees and batches without a hull run the kernels' lower instances; the existing GPU query
tests pin those."""
from __future__ import annotations

import numpy as np
import pytest

from avian_b200 import api, fixture, plugins, scenes
from move_scenes import random_characters, random_colliders, random_quats

pytestmark = pytest.mark.gpu
SCALARS = [np.float32, np.float64]
IDENT = [0.0, 0.0, 0.0, 1.0]
CUB, SPH, CAP, HULL = fixture.SHAPE_CUBOID, fixture.SHAPE_SPHERE, fixture.SHAPE_CAPSULE, fixture.SHAPE_CONVEX_HULL
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


def hull_table():
    """the 28 hulls of scenes.hull_pile: 24 random Qhull polyhedra, the regular solids and a 32-sided prism"""
    return scenes.hull_pile(4).hulls


def mixed_dims(rng, shape, n_hulls, scale=1.0):
    n = shape.shape[0]
    dims = rng.uniform(0.2, 1.5, (n, 3)) * scale
    caps = shape == CAP
    dims[caps, 0] = rng.uniform(0.1, 0.8, caps.sum()) * scale
    dims[caps, 1] = rng.uniform(0.0, 1.5, caps.sum()) * scale
    hull = shape == HULL
    dims[hull] = 0.0
    dims[hull, 0] = rng.integers(0, n_hulls, hull.sum())
    return dims


def mixed_scene(rng, n, n_hulls, extent=20.0):
    shape = rng.integers(0, 4, n).astype(np.uint8)                  # a quarter each: cuboids, spheres, capsules, hulls
    return api.QueryColliders(shape=shape, dims=mixed_dims(rng, shape, n_hulls), position=rng.uniform(-extent, extent, (n, 3)),
                              rotation=random_quats(rng, n), memberships=np.where(rng.random(n) < 0.2, 2, 1).astype(np.uint32))


def mixed_shapes(rng, m, n_hulls, extent=20.0, cast=True, **kw):
    shape = rng.integers(0, 4, m).astype(np.uint8)
    dims = mixed_dims(rng, shape, n_hulls, 0.6)
    extra = dict(direction=unit(rng.normal(size=(m, 3))), max_distance=rng.uniform(2, 30, m)) if cast else {}
    return api.ShapeQueries(shape=shape, dims=dims, position=rng.uniform(-extent, extent, (m, 3)), rotation=random_quats(rng, m), **extra, **kw)


def check_all(ctx, s, cols, hulls, rays=None, casts=None, points=None, isect=None, boxes=None, what=""):
    """device == hull-enabled brute force for every batch given"""
    ctx.query_update(cols)
    H = dict(hulls=hulls)
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
    ctx.set_convex_hulls(hull_table())
    yield ctx, request.param
    ctx.close()


def test_random_mixed_scene(qctx):
    """10k colliders (hulls, cuboids, spheres, capsules) with masks and exclusions, hull and mixed query shapes"""
    ctx, s = qctx
    hulls = fixture.HullTable(s, hull_table())
    rng = np.random.default_rng(71)
    n, m = 10_000, 1_500
    cols = mixed_scene(rng, n, hulls.count)
    excl = [list(rng.choice(n, size=int(rng.integers(0, 4)), replace=False)) for _ in range(m)]
    masks = rng.choice(np.array([0xFFFFFFFF, 1, 2], np.uint32), m)
    o = rng.uniform(-22, 22, (m, 3))
    rays = api.Rays(origin=o, direction=unit(rng.normal(size=(m, 3))), max_distance=rng.uniform(1, 40, m), solid=rng.random(m) < 0.5,
                    max_hits=rng.integers(0, 6, m).astype(np.uint32), mask=masks, exclude=excl)
    flags = rng.choice(np.array([0, api.CAST_IGNORE_ORIGIN_PENETRATION, api.CAST_NO_CONTACT_ON_PENETRATION], np.uint32), m)
    casts = mixed_shapes(rng, m, hulls.count, flags=flags, max_hits=rng.integers(0, 5, m).astype(np.uint32), mask=masks, exclude=excl)
    pts = api.Points(point=np.concatenate([o[: m // 2], cols.position[: m // 2] + rng.uniform(-0.5, 0.5, (m // 2, 3))]),
                     solid=rng.random(m) < 0.5, mask=masks, exclude=excl)
    isect = mixed_shapes(rng, m, hulls.count, cast=False, mask=masks, exclude=excl)
    boxes = (o - 1.5, o + rng.uniform(0.5, 3.0, (m, 3)))
    check_all(ctx, s, cols, hulls, rays=rays, casts=casts, points=pts, isect=isect, boxes=boxes, what="mixed ")
    hit = ctx.cast_shape(casts)["collider"]
    assert (cols.shape[hit[hit >= 0]] == HULL).sum() > 50
    assert ((casts.shape == HULL) & (hit >= 0)).sum() > 50
    # the same tree again with AVN_QUERY_SHAPES_UNCHANGED and moved poses: the kept column still holds hulls
    cols2 = api.QueryColliders(shape=cols.shape, dims=cols.dims, position=cols.position + 0.25, rotation=cols.rotation, memberships=cols.memberships)
    ctx.query_update(cols2, shapes_unchanged=True)
    assert_same(ctx.cast_shape(casts), fixture.query_cast_shape(s, cols2, casts, hulls=hulls), "unchanged ")
    assert_same(ctx.cast_ray(rays), fixture.query_cast_ray(s, cols2, rays, hulls=hulls), "unchanged ")


def _cube_hull_and_tetra():
    cube = np.array([[(1 if m & 1 else -1), (1 if m & 2 else -1), (1 if m & 4 else -1)] for m in range(8)], float) * 0.5
    tet = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], float) - 0.25
    return api.ConvexHulls.from_polyhedra([(cube, [[1, 3, 7, 5], [0, 4, 6, 2], [2, 6, 7, 3], [0, 1, 5, 4], [4, 5, 7, 6], [0, 2, 3, 1]]),
                                           (tet, [[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]])])


@pytest.mark.parametrize("scalar", SCALARS, ids=lambda s: np.dtype(s).name)
def test_grazing_rays(scalar):
    """rays along faces, through edges and vertices, and one ulp outside, on exactly planar hulls (the tight-bound case is
    test_face_planes_outside_the_vertex_box)"""
    table = _cube_hull_and_tetra()
    hulls = fixture.HullTable(scalar, table)
    pos = np.array([[0.0, 0.0, 0.0], [3.0, 0.0, 0.0], [6.25, 0.25, 0.25], [-3.0, 2.0, 1.0]])
    rot = np.array([IDENT, IDENT, IDENT, [0.0, 0.0, np.sin(0.4), np.cos(0.4)]])
    cols = api.QueryColliders(shape=np.array([HULL, HULL, HULL, HULL], np.uint8), dims=np.array([[0, 0, 0], [0, 0, 0], [1, 0, 0], [1, 0, 0]], float),
                              position=pos, rotation=rot)
    eps = np.finfo(scalar).eps
    o, d = [], []
    for cx in (0.0, 3.0):
        for lvl in (0.5, 0.5 * (1 + eps), 0.5 * (1 - eps), -0.5, 0.0):
            o += [[cx - 5, lvl, 0.0], [cx - 5, lvl, lvl], [cx, lvl, -5], [cx + lvl, 5, lvl]]
            d += [[1, 0, 0], [1, 0, 0], [0, 0, 1], [0, -1, 0]]
        o += [[cx - 5, -5, -5], [cx + 5, 5, 5], [cx - 5, 0.5, 0.5 + eps]]
        d += [unit([1, 1, 1]), unit([-1, -1, -1]), [1, 0, 0]]
    # the tetrahedron (vertex mean at 6.25, 0.25, 0.25): through its vertices, along its faces, from inside
    for v in ([6.0, 0.0, 0.0], [7.0, 0.0, 0.0], [6.0, 1.0, 0.0], [6.0, 0.0, 1.0]):
        o += [np.add(v, [0, 0, -3]), np.add(v, [-3, 0, 0]), [6.25, 0.25, 0.25]]
        d += [[0, 0, 1], [1, 0, 0], unit(np.subtract(v, [6.25, 0.25, 0.25]))]
    o += [[6.0, -3.0, 0.5], [6.5, 0.5, -3.0], [6.0, 0.0, -3.0]]
    d += [[0, 1, 0], [0, 0, 1], unit([1, 0, 3])]
    n = len(o)
    rays = api.Rays(origin=np.array(o, float), direction=np.array(d, float), max_distance=np.full(n, 20.0), solid=np.arange(n) % 2 == 0)
    pts = api.Points(point=np.concatenate([np.array(o, float), pos + 0.5 * (1 + eps), pos - 0.5]), solid=np.arange(n + 8) % 2 == 0)
    casts = api.ShapeQueries(shape=np.array([SPH, CAP, HULL, CUB] * (n // 4 + 1), np.uint8)[:n], dims=np.tile([0.0, 0.0, 0.0], (n, 1)),
                             position=np.array(o, float), rotation=np.tile(IDENT, (n, 1)), direction=np.array(d, float), max_distance=np.full(n, 20.0))
    casts.dims[casts.shape == HULL, 0] = 1
    casts.dims[casts.shape == CUB] = 0.05
    with api.Context(device=0, scalar=scalar) as ctx:
        ctx.set_convex_hulls(table)
        check_all(ctx, scalar, cols, hulls, rays=rays, points=pts, casts=casts, what="grazing ")
        assert (ctx.cast_ray(rays)["collider"] >= 0).sum() > n // 2


def _twisted_cube():
    """a unit cube with vertex 7 moved 1e-6 inwards along x: within AVN_HULL_REL_TOL of planar, so the table accepts it, and the +x face's
    Newell plane passes about 2.5e-7 outside the vertex box near the opposite corner (vertex 1)"""
    cube = np.array([[(1 if m & 1 else -1), (1 if m & 2 else -1), (1 if m & 4 else -1)] for m in range(8)], float) * 0.5
    cube[7, 0] -= 1e-6
    return api.ConvexHulls.from_polyhedra([(cube, [[1, 3, 7, 5], [0, 4, 6, 2], [2, 6, 7, 3], [0, 1, 5, 4], [4, 5, 7, 6], [0, 2, 3, 1]])])


@pytest.mark.parametrize("scalar", SCALARS, ids=lambda s: np.dtype(s).name)
def test_face_planes_outside_the_vertex_box(scalar):
    """The face-plane polytope of a hull whose vertices lie within tolerance of its planes sticks out of the vertex box.  Rays, sphere casts
    and points that pass just outside the f32 culling box of the vertex AABB, but inside the +x face plane, hit in the brute force; the
    device finds them only because the tree culls a hull against its bounding ball (qh::cull_box, qh::half_size).  With the tight AABB as
    the culling box the device misses them and this test fails."""
    table = _twisted_cube()
    hulls = fixture.HullTable(scalar, table)
    cols = api.QueryColliders(shape=np.array([HULL], np.uint8), dims=np.zeros((1, 3)), position=np.zeros((1, 3)), rotation=np.array([IDENT]))
    beyond = 0.5 + 2 * np.spacing(np.float32(0.5))            # past the f32 culling box of the vertex box's x max (0.5)
    dx = np.array([1.3e-7, 1.6e-7, 2e-7, 2.4e-7])
    ys = np.linspace(-0.5, 0.5, 41)
    x, y = np.meshgrid(0.5 + dx, ys, indexing="ij")
    x, y = x.ravel(), y.ravel()
    k = x.size
    o = np.concatenate([np.stack([x, y, np.full(k, -3.0)], 1), np.stack([x, np.full(k, -3.0), y], 1)])   # along +z and +y, parallel to the +x face
    d = np.concatenate([np.tile([0.0, 0.0, 1.0], (k, 1)), np.tile([0.0, 1.0, 0.0], (k, 1))])
    n = o.shape[0]
    rays = api.Rays(origin=o, direction=d, max_distance=np.full(n, 10.0), solid=np.arange(n) % 2 == 0)
    # spheres of radius 0.1 the same distance outside the face, moving the other way (towards where the tilted plane leans out)
    r = 0.1
    oc = o + [r, 0.0, 0.0]
    oc[:k, 2] = 3.0
    oc[k:, 1] = 3.0
    casts = api.ShapeQueries(shape=np.full(n, SPH, np.uint8), dims=np.tile([r, 0.0, 0.0], (n, 1)), position=oc, rotation=np.tile(IDENT, (n, 1)),
                             direction=-d, max_distance=np.full(n, 10.0))
    pts = api.Points(point=np.stack([x, y, np.full(k, -0.499)], 1), solid=np.arange(k) % 2 == 0)
    host_rays = fixture.query_cast_ray(scalar, cols, rays, hulls=hulls)
    host_casts = fixture.query_cast_shape(scalar, cols, casts, hulls=hulls)
    host_pts = fixture.query_point_intersections(scalar, cols, pts, hulls=hulls)
    ox = rays.origin[:, 0].astype(scalar).astype(np.float64)
    cx = casts.position[:, 0].astype(scalar).astype(np.float64) - r
    assert ((host_rays["collider"] == 0) & (ox > beyond)).sum() >= 10
    assert ((host_casts["collider"] == 0) & (cx > beyond)).sum() >= 10
    assert ((np.diff(host_pts["offsets"].astype(np.int64)) == 1) & (pts.point[:, 0].astype(scalar) > beyond)).sum() >= 5
    with api.Context(device=0, scalar=scalar) as ctx:
        ctx.set_convex_hulls(table)
        check_all(ctx, scalar, cols, hulls, rays=rays, casts=casts, points=pts, what="twisted ")


def _settled(make, steps=40):
    sc = make()
    with api.Context(device=0) as ctx:
        w = plugins.DeviceGraphWorld(sc, plugins.PhysicsPlugins(ctx), ctx, substeps=4)
        for _ in range(steps):
            w.step()
        return sc, plugins.SpatialQueryPlugin.colliders(w)


@pytest.mark.parametrize("make", [lambda: scenes.hull_pile(1500, layers=4), lambda: scenes.decomposed_pile(600, layers=3)], ids=["hull_pile", "decomposed_pile"])
def test_plugin_queries_on_settled_hull_scenes(make):
    """SpatialQueryPlugin ray casts and ShapeCaster casts (a slightly shrunk character capsule, and hulls of the table) after DeviceGraphWorld
    steps, against the brute force; the query context holds the scene's table"""
    sc, cols = _settled(make)
    s = np.float32
    hulls = fixture.HullTable(s, sc.hulls)
    rng = np.random.default_rng(5)
    k = 500
    lo, hi = cols.position[:, [0, 2]].min(0), cols.position[:, [0, 2]].max(0)
    o = np.stack([rng.uniform(lo[0], hi[0], k), np.full(k, float(cols.position[:, 1].max()) + 4), rng.uniform(lo[1], hi[1], k)], 1)
    with api.Context(device=0) as qc:
        qc.set_convex_hulls(sc.hulls)
        sp = plugins.SpatialQueryPlugin(qc)
        qc.query_update(cols)
        rays = plugins.SpatialQueryPlugin.ray_casters(o, unit(rng.normal(size=(k, 3)) * [0.3, 1.0, 0.3] - [0, 2.0, 0]), np.full(k, 40.0))
        assert_same(sp.raycast(rays), fixture.query_ray_hits(s, cols, rays, hulls=hulls), "raycast ")
        shape = np.where(np.arange(k) % 2 == 0, CAP, HULL).astype(np.uint8)
        dims = np.tile([0.4 * 0.99, 0.5 * 0.99, 0.0], (k, 1))
        dims[shape == HULL] = 0.0
        dims[shape == HULL, 0] = rng.integers(0, hulls.count, (shape == HULL).sum())
        casters = plugins.SpatialQueryPlugin.shape_casters(shape, dims, o, random_quats(rng, k), np.tile([0.0, -1.0, 0.0], (k, 1)))
        got = sp.shapecast(casters)
        assert_same(got, fixture.query_shape_hits(s, cols, casters, hulls=hulls), "shapecast ")
        assert (got["collider"] >= 0).sum() > k // 2
        c = cols.position[rng.integers(0, cols.shape.shape[0], k)]
        pts = api.Points(point=c + rng.uniform(-0.3, 0.3, c.shape), solid=rng.random(k) < 0.5)
        check_all(qc, s, cols, hulls, points=pts, isect=api.ShapeQueries(shape=shape, dims=dims, position=c, rotation=casters.rotation), what="pile ")


@pytest.mark.parametrize("scalar", SCALARS, ids=lambda s: np.dtype(s).name)
def test_hull_casts_onto_the_100k_stack_sample(scalar):
    """100k hull casts onto the 100k-cube stack on the device; a sample of them against the brute force"""
    sc = scenes.cube_stack(51, 40, 50, brick=True)
    cols = api.QueryColliders(shape=sc.shape_type.astype(np.uint8), dims=sc.dims, position=np.asarray(sc.bodies.position, np.float64),
                              rotation=np.asarray(sc.bodies.rotation, np.float64))
    table = hull_table()
    hulls = fixture.HullTable(scalar, table)
    rng = np.random.default_rng(9)
    k = 100_000
    lo, hi = cols.position[:, [0, 2]].min(0), cols.position[:, [0, 2]].max(0)
    o = np.stack([rng.uniform(lo[0], hi[0], k), np.full(k, float(cols.position[:, 1].max()) + 5), rng.uniform(lo[1], hi[1], k)], 1)
    casts = api.ShapeQueries(shape=np.full(k, HULL, np.uint8), dims=np.stack([rng.integers(0, hulls.count, k), np.zeros(k), np.zeros(k)], 1).astype(float),
                             position=o, rotation=random_quats(rng, k), direction=np.tile([0.0, -1.0, 0.0], (k, 1)), max_distance=np.full(k, 200.0))
    with api.Context(device=0, scalar=scalar) as ctx:
        ctx.set_convex_hulls(table)
        ctx.query_update(cols)
        got = ctx.cast_shape(casts)
        idx = rng.choice(k, 300, replace=False)
        sub = api.ShapeQueries(shape=casts.shape[idx], dims=casts.dims[idx], position=o[idx], rotation=casts.rotation[idx], direction=casts.direction[idx],
                               max_distance=casts.max_distance[idx])
        want = fixture.query_cast_shape(scalar, cols, sub, hulls=hulls)
        assert_same({kk: v[idx] for kk, v in got.items()}, want, "stack ")
        assert (got["collider"] >= 0).mean() > 0.9


def assert_move_same(got, want, what=""):
    assert_same(got, want, what, MOVE_OUTPUTS)


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
def hull_move_scene():
    """a dense hull pile: hull obstacles among the mixed colliders, hull, capsule and box characters"""
    rng = np.random.default_rng(2026)
    table = hull_table()
    n_h = 28
    cols, ignored = random_colliders(rng, 3_000, 8.0)
    hull = rng.random(cols.shape.shape[0]) < 0.5
    cols.shape[hull] = HULL
    cols.dims[hull] = 0.0
    cols.dims[hull, 0] = rng.integers(0, n_h, hull.sum())
    batch = random_characters(rng, 600, 8.0, 3_000)
    kind = np.arange(batch.count) % 3
    batch.shape[kind == 0] = HULL
    batch.dims[kind == 0] = 0.0
    batch.dims[kind == 0, 0] = rng.integers(0, n_h, (kind == 0).sum())
    batch.shape[kind == 1] = CAP
    return table, cols, ignored, batch


@pytest.mark.parametrize("scalar", SCALARS, ids=lambda s: np.dtype(s).name)
@pytest.mark.parametrize("name", list(CONFIGS))
def test_hull_characters_match_host(hull_move_scene, name, scalar):
    table, cols, ignored, batch = hull_move_scene
    cfg = CONFIGS[name]
    cfg.ignored = ignored
    if name != "default":
        batch = take(batch, np.arange(200))
    with api.Context(device=0, scalar=scalar) as ctx:
        ctx.set_convex_hulls(table)
        ctx.query_update(cols)
        got = ctx.move_and_slide(cfg, batch)
    want = fixture.move_and_slide(scalar, cols, cfg, batch, hulls=fixture.HullTable(scalar, table))
    assert_move_same(got, want, name)
    if cfg.move_and_slide_iterations:
        hc = want["hit_collider"]
        assert (hc >= 0).sum() > 40
        assert (cols.shape[hc[hc >= 0]] == HULL).sum() > 10


@pytest.mark.parametrize("scalar", SCALARS, ids=lambda s: np.dtype(s).name)
def test_replacing_the_table_refuses_the_hull_tree(scalar):
    """a tree holding a hull is refused once avn_set_convex_hulls replaces the table, plain and under AVN_QUERY_SHAPES_UNCHANGED, until the
    next update; a tree without hulls is not affected"""
    table = hull_table()
    rng = np.random.default_rng(3)
    cols = mixed_scene(rng, 500, 28)
    plain = api.QueryColliders(shape=np.zeros(500, np.uint8), dims=np.full((500, 3), 0.3), position=cols.position, rotation=cols.rotation)
    rays = api.Rays(origin=cols.position[:50] + 3, direction=unit(rng.normal(size=(50, 3))), max_distance=np.full(50, 10.0))
    batch = random_characters(rng, 20, 20.0, 500)
    with api.Context(device=0, scalar=scalar) as ctx:
        with pytest.raises(api.AvianError, match="no hull table"):
            ctx.query_update(cols)
        ctx.set_convex_hulls(table)
        ctx.query_update(cols)
        ctx.cast_ray(rays)
        ctx.set_convex_hulls(table)                           # the same contents, a new table
        for call in (lambda: ctx.cast_ray(rays), lambda: ctx.move_and_slide(api.MoveConfig(), batch),
                     lambda: ctx.aabb_intersections(cols.position[:5] - 1, cols.position[:5] + 1)):
            with pytest.raises(api.AvianError, match="update again"):
                call()
        ctx.query_update(cols, shapes_unchanged=True)        # rebuilt from the current table
        assert_same(ctx.cast_ray(rays), fixture.query_cast_ray(scalar, cols, rays, hulls=fixture.HullTable(scalar, table)), "after update ")
        ctx.set_convex_hulls(_cube_hull_and_tetra())          # 2 hulls: the kept column names indices up to 27
        with pytest.raises(api.AvianError, match="hull table holds"):
            ctx.query_update(cols, shapes_unchanged=True)
        with pytest.raises(api.AvianError, match="below the hull table's count"):
            ctx.query_update(cols)
        ctx.query_update(plain)
        ctx.set_convex_hulls(None)
        ctx.cast_ray(rays)                                    # no hull in the tree: the table does not matter
        shapes = api.ShapeQueries(shape=np.full(3, HULL, np.uint8), dims=np.zeros((3, 3)), position=cols.position[:3], rotation=cols.rotation[:3],
                                  direction=np.tile([1.0, 0, 0], (3, 1)), max_distance=np.full(3, 5.0))
        with pytest.raises(api.AvianError, match="no hull table"):
            ctx.cast_shape(shapes)
