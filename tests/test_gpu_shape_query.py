"""Shape casts, point projection and point / shape intersections on the device (csrc/queries.cu) against the host brute force over every
collider (fixture.query_*, the same csrc/query_math.hpp): collider, distance, point and normal bits of every hit, CSR offsets and contents,
f32 and f64."""
import numpy as np
import pytest

from avian_b200 import api, fixture, plugins, scenes

pytestmark = pytest.mark.gpu
SCALARS = [np.float32, np.float64]
IDENT = [0.0, 0.0, 0.0, 1.0]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({1: np.uint8, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def assert_same(dev: dict, host: dict, what: str = ""):
    assert set(dev) == set(host), what
    for k in host:
        assert dev[k].shape == host[k].shape, f"{what}{k}: {dev[k].shape} vs {host[k].shape}"
        a, b = _bits(dev[k]), _bits(host[k])
        assert np.array_equal(a, b), f"{what}{k} differs at rows {np.nonzero((a != b).reshape(a.shape[0], -1).any(axis=1))[0][:10]}"


def unit(v):
    v = np.asarray(v, dtype=np.float64)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def random_quats(rng, n):
    return unit(rng.normal(size=(n, 4)))


def random_scene(rng, n, extent=20.0):
    shape = (rng.random(n) < 0.4).astype(np.uint8)
    return api.QueryColliders(shape=shape, dims=rng.uniform(0.2, 1.5, size=(n, 3)), position=rng.uniform(-extent, extent, size=(n, 3)),
                              rotation=random_quats(rng, n))


def random_shapes(rng, m, extent=20.0, cast=True, **kw):
    shape = (rng.random(m) < 0.5).astype(np.uint8)
    dims = rng.uniform(0.05, 1.0, size=(m, 3))
    extra = {}
    if cast:
        extra = dict(direction=unit(rng.normal(size=(m, 3))), max_distance=rng.uniform(2, 30, m))
    return api.ShapeQueries(shape=shape, dims=dims, position=rng.uniform(-extent, extent, (m, 3)), rotation=random_quats(rng, m), **extra, **kw)


def check(ctx, s, cols, casts=None, points=None, isect=None, what="", update=True):
    """device == brute force for the calls that get a batch; returns the device shape hits"""
    if update:
        ctx.query_update(cols)
    dev = None
    if casts is not None:
        assert_same(ctx.cast_shape(casts), fixture.query_cast_shape(s, cols, casts), what + "cast_shape ")
        dev = ctx.shape_hits(casts)
        assert_same(dev, fixture.query_shape_hits(s, cols, casts), what + "shape_hits ")
    if points is not None:
        assert_same(ctx.project_point(points), fixture.query_project_point(s, cols, points), what + "project_point ")
        assert_same(ctx.point_intersections(points), fixture.query_point_intersections(s, cols, points), what + "point_intersections ")
    if isect is not None:
        assert_same(ctx.shape_intersections(isect), fixture.query_shape_intersections(s, cols, isect), what + "shape_intersections ")
    return dev


@pytest.fixture(scope="module", params=SCALARS, ids=["f32", "f64"])
def qctx(request):
    ctx = api.Context(device=0, scalar=request.param)
    yield ctx, request.param
    ctx.close()


def test_random_boxes_and_spheres(qctx):
    ctx, s = qctx
    rng = np.random.default_rng(17)
    n, m = 10_000, 3_000
    cols = random_scene(rng, n)
    cols.memberships = np.where(rng.random(n) < 0.2, 2, 1).astype(np.uint32)
    excl = [rng.integers(0, n, size=rng.integers(0, 3)).tolist() for _ in range(m)]
    mask = np.where(rng.random(m) < 0.2, 1, 0xFFFFFFFF).astype(np.uint32)
    flags = rng.integers(0, 4, m).astype(np.uint32)
    casts = random_shapes(rng, m, flags=flags, mask=mask, exclude=excl, max_hits=rng.integers(0, 8, m).astype(np.uint32))
    pts = api.Points(point=rng.uniform(-22, 22, (m, 3)), solid=rng.random(m) < 0.5, mask=mask, exclude=excl)
    isect = random_shapes(rng, m, cast=False, mask=mask, exclude=excl)
    dev = check(ctx, s, cols, casts, pts, isect)
    assert dev["collider"].shape[0] > m // 2
    r = ctx.cast_shape(casts)
    assert (r["distance"][r["collider"] >= 0] == 0).sum() > 10          # some origin penetrations
    assert (ctx.project_point(pts)["is_inside"] == 1).sum() > 10
    assert ctx.point_intersections(pts)["collider"].size > 10 and ctx.shape_intersections(isect)["collider"].size > m


def test_casts_onto_a_settled_cube_stack(qctx):
    """straight down onto the stack: exact face-face contacts, equal TOIs on neighbouring cubes (ties by index)"""
    ctx, s = qctx
    w = plugins.World(scenes.cube_stack(12, 10, 12, brick=True, scalar=s), plugins.PhysicsPlugins(ctx), substeps=4)
    for _ in range(2):
        w.step()
    cols = plugins.SpatialQueryPlugin.colliders(w)
    n = int(w.bodies.count)
    gx, gz = np.meshgrid(np.linspace(-1, 13, 30), np.linspace(-1, 13, 30), indexing="ij")
    k = gx.size
    o = np.stack([gx.ravel(), np.full(k, 30.0), gz.ravel()], 1)
    shape = (np.arange(k) % 2).astype(np.uint8)
    down = api.ShapeQueries(shape=shape, dims=np.full((k, 3), 0.5), position=o, rotation=np.tile(IDENT, (k, 1)), direction=np.tile([0.0, -1.0, 0.0], (k, 1)),
                            max_distance=np.full(k, 60.0), max_hits=np.full(k, 5, np.uint32))
    rng = np.random.default_rng(3)
    c = np.asarray(w.bodies.position[rng.integers(1, n, 800)], dtype=np.float64)
    pts = api.Points(point=c + rng.uniform(-0.6, 0.6, c.shape), solid=rng.random(800) < 0.5)
    isect = api.ShapeQueries(shape=(np.arange(800) % 2).astype(np.uint8), dims=np.full((800, 3), 0.4), position=c, rotation=random_quats(rng, 800))
    dev = check(ctx, s, cols, down, pts, isect, what="stack ")
    assert (np.diff(dev["offsets"]) > 0).mean() > 0.8


def test_sliding_along_faces_and_tangent_spheres(qctx):
    """casts that slide exactly along box faces (a touching face plane all the way) and spheres passing tangent to spheres and edges"""
    ctx, s = qctx
    g = np.arange(-4, 5, 2.0)
    P = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    nb = P.shape[0]
    shape = np.zeros(nb, np.uint8)
    shape[1::3] = 1
    cols = api.QueryColliders(shape=shape, dims=np.full((nb, 3), 0.5), position=P, rotation=np.tile(IDENT, (nb, 1)))
    items = []
    for i in range(nb):
        for ax in range(3):
            d = np.zeros(3)
            d[ax] = 1.0
            off = np.zeros(3)
            off[(ax + 1) % 3] = 1.0                      # a half-size box / radius-0.5 sphere sits exactly on the face plane
            items.append((0, 0.5, P[i] + off - 3 * d, d))
            items.append((1, 0.5, P[i] + off - 3 * d, d))
            off2 = off.copy()
            off2[(ax + 2) % 3] = 1.0 - np.sqrt(0.5)     # near an edge: sphere tangent to the edge cylinder
            items.append((1, 0.5 * np.sqrt(2), P[i] + 0.5 * off2 - 3 * d, d))
    k = len(items)
    casts = api.ShapeQueries(shape=np.array([t[0] for t in items], np.uint8), dims=np.array([[t[1]] * 3 for t in items]),
                             position=np.array([t[2] for t in items]), rotation=np.tile(IDENT, (k, 1)), direction=np.array([t[3] for t in items]),
                             max_distance=np.full(k, 8.0), flags=(np.arange(k) % 4).astype(np.uint32))
    isect = api.ShapeQueries(shape=casts.shape, dims=casts.dims, position=casts.position + 3 * casts.direction, rotation=casts.rotation)
    pts = api.Points(point=P + 0.5, solid=np.arange(nb) % 2 == 0)
    dev = check(ctx, s, cols, casts, pts, isect, what="sliding ")
    assert dev["collider"].size > k // 2


def test_coincident_colliders_zero_and_one(qctx):
    ctx, s = qctx
    n = 400
    cols = api.QueryColliders(shape=(np.arange(n) % 2).astype(np.uint8), dims=np.full((n, 3), 0.5), position=np.tile([1.0, 2.0, 3.0], (n, 1)),
                              rotation=np.tile(IDENT, (n, 1)))
    rng = np.random.default_rng(5)
    m = 64
    d = unit(rng.normal(size=(m, 3)))
    casts = api.ShapeQueries(shape=(np.arange(m) % 2).astype(np.uint8), dims=np.full((m, 3), 0.25), position=np.array([1.0, 2.0, 3.0]) - 5 * d,
                             rotation=random_quats(rng, m), direction=d, max_distance=np.full(m, 10.0))
    pts = api.Points(point=np.array([1.0, 2.0, 3.0]) + rng.uniform(-1, 1, (m, 3)), solid=rng.random(m) < 0.5)
    dev = check(ctx, s, cols, casts, pts, api.ShapeQueries(shape=casts.shape, dims=casts.dims, position=pts.point, rotation=casts.rotation))
    assert np.array_equal(np.diff(dev["offsets"]), np.full(m, n))
    empty = api.QueryColliders(shape=np.zeros(0, np.uint8), dims=np.zeros((0, 3)), position=np.zeros((0, 3)), rotation=np.zeros((0, 4)))
    dev = check(ctx, s, empty, casts, pts, casts)
    assert dev["collider"].size == 0 and (ctx.project_point(pts)["collider"] == -1).all()
    one = api.QueryColliders(shape=np.zeros(1, np.uint8), dims=np.full((1, 3), 0.5), position=np.zeros((1, 3)), rotation=np.array([IDENT]))
    down = api.ShapeQueries(shape=np.array([1], np.uint8), dims=np.full((1, 3), 0.25), position=np.array([[0.0, 5.0, 0.0]]), rotation=np.array([IDENT]),
                            direction=np.array([[0.0, -1.0, 0.0]]), max_distance=np.array([10.0]))
    dev = check(ctx, s, one, down, pts, casts)
    assert dev["collider"].tolist() == [0] and float(dev["distance"][0]) == 4.25


def test_non_finite_and_zero_quaternion_query_shapes(qctx):
    ctx, s = qctx
    rng = np.random.default_rng(9)
    cols = random_scene(rng, 2000, extent=10.0)
    m = 600
    casts = random_shapes(rng, m, extent=10.0)
    bad = np.arange(0, m, 7)
    for j, i in enumerate(bad):
        col = [casts.position, casts.dims, casts.rotation, casts.direction][j % 4]
        col[i, j % col.shape[1]] = [np.nan, np.inf][j % 2]          # (a negative half extent, -inf included, is refused)
    casts.rotation[3::50] = 0.0
    casts.max_distance[5::60] = np.inf
    pts = api.Points(point=rng.uniform(-10, 10, (m, 3)))
    pts.point[::11, 2] = np.nan
    isect = api.ShapeQueries(shape=casts.shape, dims=casts.dims, position=casts.position, rotation=casts.rotation)
    check(ctx, s, cols, casts, pts, isect)
    nohit = np.concatenate([bad, np.arange(3, m, 50), np.arange(5, m, 60)])
    assert (ctx.cast_shape(casts)["collider"][nohit] == -1).all()
    assert (ctx.project_point(pts)["collider"][::11] == -1).all()


def test_max_hits_capacity_before_update_and_second_update(qctx):
    ctx, s = qctx
    fresh = api.Context(device=0, scalar=s)
    one = api.ShapeQueries(shape=np.array([1], np.uint8), dims=np.full((1, 3), 0.25), position=np.array([[0.0, 20.0, 0.0]]), rotation=np.array([IDENT]),
                           direction=np.array([[0.0, -1.0, 0.0]]), max_distance=np.array([50.0]))
    for call in (lambda: fresh.cast_shape(one), lambda: fresh.shape_hits(one), lambda: fresh.shape_intersections(one),
                 lambda: fresh.project_point(api.Points(point=np.zeros((1, 3)))), lambda: fresh.point_intersections(api.Points(point=np.zeros((1, 3))))):
        with pytest.raises(api.AvianError) as e:
            call()
        assert e.value.status == api.ERR_INVALID_ARGUMENT
    fresh.close()
    n = 10
    cols = api.QueryColliders(shape=(np.arange(n) % 2).astype(np.uint8), dims=np.full((n, 3), 0.25),
                              position=np.column_stack([np.zeros(n), np.arange(n, dtype=float), np.zeros(n)]), rotation=np.tile(IDENT, (n, 1)))
    ctx.query_update(cols)
    two = api.ShapeQueries(shape=np.array([1, 0], np.uint8), dims=np.full((2, 3), 0.25), position=np.array([[0.0, 20.0, 0.0]] * 2),
                           rotation=np.tile(IDENT, (2, 1)), direction=np.array([[0.0, -1.0, 0.0]] * 2), max_distance=np.array([50.0, 50.0]))
    with pytest.raises(api.AvianError) as e:
        ctx.shape_hits(two, capacity=5)
    assert e.value.status == api.ERR_CAPACITY and e.value.required == 2 * n
    column = api.ShapeQueries(shape=np.array([0], np.uint8), dims=np.array([[0.1, 20.0, 0.1]]), position=np.zeros((1, 3)), rotation=np.array([IDENT]))
    with pytest.raises(api.AvianError) as e:
        ctx.shape_intersections(column, capacity=3)
    assert e.value.status == api.ERR_CAPACITY and e.value.required == n
    with pytest.raises(api.AvianError) as e:
        ctx.point_intersections(api.Points(point=np.column_stack([np.zeros(n), np.arange(n, dtype=float), np.zeros(n)])), capacity=n - 1)
    assert e.value.status == api.ERR_CAPACITY and e.value.required == n
    assert ctx.shape_hits(two, capacity=2 * n)["collider"].tolist() == list(range(n - 1, -1, -1)) * 2
    for mh, want in ((0, 0), (1, 1), (api.MAX_HITS_ALL, n)):
        two.max_hits = np.full(2, mh, np.uint32)
        h = ctx.shape_hits(two)
        assert np.diff(h["offsets"]).tolist() == [want, want]
        assert_same(h, fixture.query_shape_hits(s, cols, two), f"max_hits={mh} ")
    # max_hits 1 == the closest cast
    two.max_hits = np.ones(2, np.uint32)
    h, r = ctx.shape_hits(two), ctx.cast_shape(two)
    for k in ("distance", "point1", "point2", "normal1", "normal2"):
        assert np.array_equal(_bits(h[k]), _bits(r[k]))
    # the poses move: a second update with the shapes kept answers for the new poses
    cols.position[:, 0] = 5.0
    cols.position[3] = [0.0, 3.0, 0.0]
    ctx.query_update(cols, shapes_unchanged=True)
    r = ctx.cast_shape(two)
    assert r["collider"].tolist() == [3, 3] and float(r["distance"][0]) == 16.5
    rng = np.random.default_rng(2)
    check(ctx, s, cols, random_shapes(rng, 200, extent=6.0), api.Points(point=rng.uniform(-6, 6, (200, 3))), random_shapes(rng, 200, 6.0, cast=False),
          update=False)


def test_radius_zero_sphere_cast_matches_cast_ray(qctx):
    ctx, s = qctx
    rng = np.random.default_rng(12)
    cols = random_scene(rng, 3000, extent=15.0)
    ctx.query_update(cols)
    m = 2000
    o, d = rng.uniform(-17, 17, (m, 3)), unit(rng.normal(size=(m, 3)))
    ray = ctx.cast_ray(api.Rays(origin=o, direction=d, max_distance=np.full(m, 40.0)))
    sc = ctx.cast_shape(api.ShapeQueries(shape=np.ones(m, np.uint8), dims=np.zeros((m, 3)), position=o, rotation=np.tile(IDENT, (m, 1)), direction=d,
                                         max_distance=np.full(m, 40.0)))
    assert np.array_equal(sc["collider"], ray["collider"]) and (ray["collider"] >= 0).sum() > 200
    hit = (ray["collider"] >= 0) & (ray["distance"] > 0)
    eps = np.finfo(s).eps
    assert np.allclose(sc["distance"][hit], ray["distance"][hit], rtol=0, atol=16 * eps * 16)
    assert np.allclose(sc["normal1"][hit], ray["normal"][hit], atol=16 * eps)


def test_shape_caster_plugin_follows_device_graph_world(qctx):
    ctx, s = qctx
    w = plugins.DeviceGraphWorld(scenes.cube_stack(8, 6, 8, brick=True, scalar=s), plugins.PhysicsPlugins(ctx), ctx, substeps=4)
    sq = plugins.SpatialQueryPlugin(ctx)
    rng = np.random.default_rng(1)
    n = int(w.bodies.count)
    memb = np.where(rng.random(n) < 0.1, 2, 1).astype(np.uint32)
    k = 300
    owner = rng.integers(-1, n, k)
    for step in range(3):
        w.step()
        sq.update_pipeline(w, memb, shapes_unchanged=step > 0)
        o = np.where(owner[:, None] >= 0, np.asarray(w.bodies.position[np.maximum(owner, 0)], dtype=np.float64), rng.uniform(-2, 10, (k, 3)))
        enabled = rng.random(k) < 0.8
        casts = sq.shape_casters((rng.random(k) < 0.5).astype(np.uint8), rng.uniform(0.1, 0.4, (k, 3)), o, random_quats(rng, k), unit(rng.normal(size=(k, 3))),
                                 max_distance=20.0, max_hits=None if step == 0 else rng.integers(0, 6, k), enabled=enabled, owner=owner,
                                 ignore_origin_penetration=rng.random(k) < 0.5)
        hits = sq.shapecast(casts)
        assert_same(hits, fixture.query_shape_hits(s, sq.colliders(w, memb), casts), f"step {step} ")
        offs = hits["offsets"].astype(np.int64)
        own = [hits["collider"][offs[i]:offs[i + 1]] for i in range(k)]
        assert all(owner[i] not in own[i] for i in range(k))            # ignore_self
        assert all(len(own[i]) == 0 for i in np.nonzero(~enabled)[0])
        if step == 0:
            assert all(len(h) <= 1 for h in own) and sum(len(h) for h in own) > k // 4      # default max_hits 1
