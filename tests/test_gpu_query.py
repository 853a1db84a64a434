"""Spatial queries on the device (csrc/queries.cu) against the host brute force over every collider (fixture.query_*, the same
csrc/query_math.hpp): collider, distance bits and normal bits of every hit, CSR offsets and contents, f32 and f64.  Equality here means the
tree culls conservatively and the tie rule makes the answer independent of the tree."""
import numpy as np
import pytest

from avian_b200 import api, fixture, plugins, scenes

pytestmark = pytest.mark.gpu
SCALARS = [np.float32, np.float64]


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
    dims = rng.uniform(0.2, 1.5, size=(n, 3))
    pos = rng.uniform(-extent, extent, size=(n, 3))
    return api.QueryColliders(shape=shape, dims=dims, position=pos, rotation=random_quats(rng, n))


def check(ctx, scalar, cols, rays, boxes=None, what=""):
    """device == brute force for all three queries; returns the device ray hits"""
    ctx.query_update(cols)
    assert_same(ctx.cast_ray(rays), fixture.query_cast_ray(scalar, cols, rays), what + "cast_ray ")
    dev = ctx.ray_hits(rays)
    assert_same(dev, fixture.query_ray_hits(scalar, cols, rays), what + "ray_hits ")
    if boxes is not None:
        assert_same(ctx.aabb_intersections(*boxes), fixture.query_aabb_intersections(scalar, cols, *boxes), what + "aabb ")
    return dev


@pytest.fixture(scope="module", params=SCALARS, ids=["f32", "f64"])
def qctx(request):
    ctx = api.Context(device=0, scalar=request.param)
    yield ctx, request.param
    ctx.close()


def test_random_boxes_and_spheres(qctx):
    ctx, s = qctx
    rng = np.random.default_rng(7)
    n, m = 10_000, 4_000
    cols = random_scene(rng, n)
    cols.memberships = np.where(rng.random(n) < 0.2, 2, 1).astype(np.uint32)
    excl = [rng.integers(0, n, size=rng.integers(0, 3)).tolist() for _ in range(m)]
    rays = api.Rays(origin=rng.uniform(-25, 25, size=(m, 3)), direction=unit(rng.normal(size=(m, 3))), max_distance=rng.uniform(5, 60, size=m),
                    solid=rng.random(m) < 0.5, mask=np.where(rng.random(m) < 0.2, 1, 0xFFFFFFFF).astype(np.uint32), exclude=excl)
    c = rng.uniform(-20, 20, size=(2000, 3))
    h = rng.uniform(0, 3, size=(2000, 3))
    dev = check(ctx, s, cols, rays, (c - h, c + h))
    assert dev["collider"].shape[0] > m      # the scene is dense enough that rays hit several colliders


def test_settled_cube_stack(qctx):
    ctx, s = qctx
    w = plugins.World(scenes.cube_stack(22, 20, 22, brick=True, scalar=s), plugins.PhysicsPlugins(ctx), substeps=4)
    for _ in range(2):
        w.step()
    cols = plugins.SpatialQueryPlugin.colliders(w)
    n = int(w.bodies.count)
    assert n > 9000
    rng = np.random.default_rng(3)
    gx, gz = np.meshgrid(np.linspace(-1, 24, 50), np.linspace(-1, 24, 50), indexing="ij")
    down = api.Rays(origin=np.stack([gx.ravel(), np.full(gx.size, 40.0), gz.ravel()], 1), direction=np.tile([0.0, -1.0, 0.0], (gx.size, 1)),
                    max_distance=np.full(gx.size, 100.0))
    check(ctx, s, cols, down, what="down ")
    k = 1500
    inside = api.Rays(origin=np.asarray(w.bodies.position[rng.integers(1, n, k)], dtype=np.float64) + rng.uniform(-0.3, 0.3, (k, 3)),
                      direction=unit(rng.normal(size=(k, 3))), max_distance=np.full(k, 30.0), solid=rng.random(k) < 0.5)
    c = np.asarray(w.bodies.position[rng.integers(1, n, 1000)], dtype=np.float64)
    check(ctx, s, cols, inside, (c - 0.6, c + 0.6), what="inside ")


def test_grazing_rays_edges_corners_tangents(qctx):
    """rays through box edges and corners (axis-aligned at integer / half-integer bounds, and rotated) and tangent to spheres: the culling
    bounds must not lose a hit the exact test reports"""
    ctx, s = qctx
    rng = np.random.default_rng(11)
    g = np.arange(-4, 5, 2.0)
    P = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    nb = P.shape[0]
    rot = np.tile([0.0, 0.0, 0.0, 1.0], (nb, 1))
    rot[::3] = random_quats(rng, len(rot[::3]))
    shape = np.zeros(nb, np.uint8)
    shape[1::4] = 1
    dims = np.full((nb, 3), 0.5)
    cols = api.QueryColliders(shape=shape, dims=dims, position=P, rotation=rot)
    origins, dirs = [], []
    signs = np.array([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)], dtype=np.float64)
    for i in range(nb):
        if shape[i] == 1:     # tangent: a ray at distance r from the centre
            for _ in range(4):
                d = unit(rng.normal(size=3))
                perp = unit(np.cross(d, rng.normal(size=3)))
                origins.append(P[i] + 0.5 * perp - 6 * d); dirs.append(d)
            continue
        q = rot[i]
        R = np.array([[1 - 2 * (q[1] ** 2 + q[2] ** 2), 2 * (q[0] * q[1] - q[2] * q[3]), 2 * (q[0] * q[2] + q[1] * q[3])],
                      [2 * (q[0] * q[1] + q[2] * q[3]), 1 - 2 * (q[0] ** 2 + q[2] ** 2), 2 * (q[1] * q[2] - q[0] * q[3])],
                      [2 * (q[0] * q[2] - q[1] * q[3]), 2 * (q[1] * q[2] + q[0] * q[3]), 1 - 2 * (q[0] ** 2 + q[1] ** 2)]])
        for sg in signs[:4]:
            corner = P[i] + R @ (0.5 * sg)
            d = unit(rng.normal(size=3))
            origins.append(corner - 6 * d); dirs.append(d)                    # through a corner
            edge = P[i] + R @ (0.5 * sg * np.array([1.0, 1.0, 0.0]))
            origins.append(edge - 6 * R[:, 2]); dirs.append(R[:, 2])           # along an edge
            origins.append(edge - 6 * R[:, 0]); dirs.append(R[:, 0])     # across the edge line, in a face plane
    rays = api.Rays(origin=np.array(origins), direction=np.array(dirs), max_distance=np.full(len(origins), 12.0),
                    solid=np.arange(len(origins)) % 2 == 0)
    dev = check(ctx, s, cols, rays, (P - 0.5, P + 0.5), what="grazing ")
    assert dev["collider"].shape[0] > len(origins) // 2


def rotation_matrix(q):
    """the rotation of q / |q| (what csrc/query_math.hpp's rot_mat evaluates)"""
    x, y, z, w = np.asarray(q, dtype=np.float64) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def test_rotated_boxes_at_the_origin_non_unit_quaternions(qctx):
    """Rotated cuboids centred at the origin with half extents just under a power of two, so that a bound's f32 ulp is as small as it gets
    relative to the box, and quaternions that are unit only to f32 precision (|q|^2 - 1 of about 1e-7): the culling box must still cover
    every point the exact ray test accepts.  Rays parallel to an axis pass through (just inside) each corner."""
    ctx, s = qctx
    rng = np.random.default_rng(21)
    n = 300
    q = random_quats(rng, n).astype(np.float32).astype(np.float64)            # unit, rounded to f32: |q|^2 != 1
    q[::2] *= 1.0 + rng.choice([-1.0, 1.0], size=(len(q[::2]), 1)) * 1e-7   # and some further off, both ways
    he = np.exp2(rng.integers(-1, 3, size=(n, 3))) * (1.0 - rng.uniform(1e-4, 3e-2, size=(n, 3)))
    cols = api.QueryColliders(shape=np.zeros(n, np.uint8), dims=he, position=np.zeros((n, 3)), rotation=q)
    origins, dirs = [], []
    signs = np.array([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)], dtype=np.float64)
    for i in range(n):
        R = rotation_matrix(q[i])
        for sg in signs:
            corner = R @ (sg * he[i] * (1.0 - 1e-9))
            for ax in range(3):
                d = np.zeros(3)
                d[ax] = 1.0
                origins.append(corner - 10.0 * d); dirs.append(d)
    rays = api.Rays(origin=np.array(origins), direction=np.array(dirs), max_distance=np.full(len(origins), 30.0))
    c = np.array(origins[::7]) + 10.0 * np.array(dirs[::7])
    dev = check(ctx, s, cols, rays, (c, c), what="origin boxes ")
    assert (np.diff(dev["offsets"]) > 0).mean() > 0.9


def test_all_colliders_at_one_position(qctx):
    """equal Morton codes everywhere: the hierarchy splits on index bits (the depth bound); every ray hits all of them"""
    ctx, s = qctx
    n = 600
    cols = api.QueryColliders(shape=(np.arange(n) % 2).astype(np.uint8), dims=np.full((n, 3), 0.5), position=np.tile([1.0, 2.0, 3.0], (n, 1)),
                              rotation=np.tile([0.0, 0.0, 0.0, 1.0], (n, 1)))
    rng = np.random.default_rng(5)
    m = 64
    d = unit(rng.normal(size=(m, 3)))
    rays = api.Rays(origin=np.array([1.0, 2.0, 3.0]) - 5 * d, direction=d, max_distance=np.full(m, 10.0))
    dev = check(ctx, s, cols, rays, (np.array([[0.0, 1.0, 2.0]]), np.array([[1.0, 2.0, 3.0]])))
    assert np.array_equal(np.diff(dev["offsets"]), np.full(m, n))


def test_ground_slab_spanning_the_scene(qctx):
    ctx, s = qctx
    rng = np.random.default_rng(2)
    n = 2000
    cols = random_scene(rng, n, extent=50.0)
    cols.position[:, 1] = np.abs(cols.position[:, 1]) + 2.0
    cols.shape[0], cols.dims[0], cols.position[0], cols.rotation[0] = 0, [500.0, 0.5, 500.0], [0.0, -0.5, 0.0], [0, 0, 0, 1]
    m = 3000
    rays = api.Rays(origin=np.column_stack([rng.uniform(-60, 60, m), rng.uniform(0, 60, m), rng.uniform(-60, 60, m)]),
                    direction=unit(rng.normal(size=(m, 3)) - [0, 1.0, 0]), max_distance=np.full(m, 200.0))
    c = rng.uniform(-60, 60, (500, 3))
    check(ctx, s, cols, rays, (c - 1, c + 1))


def test_zero_and_one_collider(qctx):
    ctx, s = qctx
    rays = api.Rays(origin=np.array([[0.0, 5.0, 0.0], [3.0, 5.0, 0.0]]), direction=np.array([[0.0, -1.0, 0.0]] * 2), max_distance=np.full(2, 10.0))
    empty = api.QueryColliders(shape=np.zeros(0, np.uint8), dims=np.zeros((0, 3)), position=np.zeros((0, 3)), rotation=np.zeros((0, 4)))
    dev = check(ctx, s, empty, rays, (np.zeros((1, 3)), np.ones((1, 3))))
    assert dev["collider"].size == 0
    one = api.QueryColliders(shape=np.zeros(1, np.uint8), dims=np.full((1, 3), 0.5), position=np.zeros((1, 3)), rotation=np.array([[0.0, 0, 0, 1]]))
    dev = check(ctx, s, one, rays, (np.zeros((1, 3)), np.ones((1, 3))))
    assert dev["collider"].tolist() == [0] and float(dev["distance"][0]) == 4.5


def test_non_finite_colliders_and_rays_are_never_reported(qctx):
    ctx, s = qctx
    rng = np.random.default_rng(9)
    n = 3000
    cols = random_scene(rng, n, extent=10.0)
    bad = rng.choice(n, 60, replace=False)
    for j, i in enumerate(bad):
        col = [cols.position, cols.dims, cols.rotation][j % 3]
        col[i, j % col.shape[1]] = [np.nan, np.inf, -np.inf][j % 3]
    m = 2000
    o = rng.uniform(-12, 12, (m, 3))
    o[::97, 1] = np.nan
    mdist = np.full(m, 30.0)
    mdist[5::101] = np.inf
    rays = api.Rays(origin=o, direction=unit(rng.normal(size=(m, 3))), max_distance=mdist)
    c = rng.uniform(-10, 10, (800, 3))
    dev = check(ctx, s, cols, rays, (c - 2, c + 2))
    assert not np.isin(dev["collider"], bad).any()
    nohit = np.concatenate([np.arange(0, m, 97), np.arange(5, m, 101)])
    assert (np.diff(dev["offsets"])[nohit] == 0).all()
    assert not np.isin(ctx.aabb_intersections(np.full((1, 3), -1e6), np.full((1, 3), 1e6))["collider"], bad).any()


def test_max_hits_masks_excludes_and_closest_agrees(qctx):
    ctx, s = qctx
    rng = np.random.default_rng(4)
    n, m = 4000, 2000
    cols = random_scene(rng, n, extent=12.0)
    cols.memberships = (1 << rng.integers(0, 3, n)).astype(np.uint32)
    o, d = rng.uniform(-14, 14, (m, 3)), unit(rng.normal(size=(m, 3)))
    mask = (rng.integers(1, 8, m)).astype(np.uint32)
    excl = [rng.integers(0, n, rng.integers(0, 4)).tolist() for _ in range(m)]
    base = dict(origin=o, direction=d, max_distance=np.full(m, 40.0), mask=mask, exclude=excl, solid=rng.random(m) < 0.5)
    ctx.query_update(cols)
    full = None
    for mh in (0, 1, 3, api.MAX_HITS_ALL):
        rays = api.Rays(max_hits=np.full(m, mh, np.uint32), **base)
        dev = ctx.ray_hits(rays)
        assert_same(dev, fixture.query_ray_hits(s, cols, rays), f"max_hits={mh} ")
        cnt = np.diff(dev["offsets"]).astype(np.int64)
        if mh == api.MAX_HITS_ALL:
            full = dev
        else:
            assert (cnt <= mh).all()
        if mh == 1:
            closest = ctx.cast_ray(rays)
            hit = cnt == 1
            assert np.array_equal(closest["collider"] >= 0, hit)
            assert np.array_equal(closest["collider"][hit], dev["collider"].astype(np.int32))
            assert np.array_equal(_bits(closest["distance"][hit]), _bits(dev["distance"]))
            assert np.array_equal(_bits(closest["normal"][hit]), _bits(dev["normal"]))
    # masks and exclusions really filter: no reported collider is excluded or outside the ray's mask
    offs = full["offsets"].astype(np.int64)
    for i in range(0, m, 7):
        hits = full["collider"][offs[i]:offs[i + 1]]
        assert not np.isin(hits, excl[i]).any() and ((cols.memberships[hits] & mask[i]) != 0).all()
    assert (np.diff(offs) > 3).any()
    # per ray sorted by (distance, collider)
    for i in range(0, m, 5):
        t, c = full["distance"][offs[i]:offs[i + 1]], full["collider"][offs[i]:offs[i + 1]]
        assert all((t[k], c[k]) < (t[k + 1], c[k + 1]) for k in range(len(t) - 1))


def test_capacity_before_update_and_second_update(qctx):
    ctx, s = qctx
    fresh = api.Context(device=0, scalar=s)
    rays = api.Rays(origin=np.array([[0.0, 5.0, 0.0]]), direction=np.array([[0.0, -1.0, 0.0]]), max_distance=np.array([10.0]))
    with pytest.raises(api.AvianError) as e:
        fresh.cast_ray(rays)
    assert e.value.status == api.ERR_INVALID_ARGUMENT
    with pytest.raises(api.AvianError) as e:
        fresh.aabb_intersections(np.zeros((1, 3)), np.ones((1, 3)))
    assert e.value.status == api.ERR_INVALID_ARGUMENT
    fresh.close()
    n = 10
    cols = api.QueryColliders(shape=np.zeros(n, np.uint8), dims=np.full((n, 3), 0.25), position=np.column_stack([np.zeros(n), np.arange(n, dtype=float), np.zeros(n)]),
                              rotation=np.tile([0.0, 0, 0, 1], (n, 1)))
    ctx.query_update(cols)
    down = api.Rays(origin=np.array([[0.0, 20.0, 0.0], [0.0, 20.0, 0.0]]), direction=np.array([[0.0, -1.0, 0.0]] * 2), max_distance=np.array([50.0, 50.0]))
    with pytest.raises(api.AvianError) as e:
        ctx.ray_hits(down, capacity=5)
    assert e.value.status == api.ERR_CAPACITY and e.value.required == 2 * n
    with pytest.raises(api.AvianError) as e:
        ctx.aabb_intersections(np.full((3, 3), -100.0), np.full((3, 3), 100.0), capacity=29)
    assert e.value.status == api.ERR_CAPACITY and e.value.required == 3 * n
    assert ctx.ray_hits(down, capacity=2 * n)["collider"].tolist() == list(range(n - 1, -1, -1)) * 2
    # the poses move: a second update answers for the new poses
    cols.position[:, 0] = 5.0
    cols.position[3] = [0.0, 3.0, 0.0]
    ctx.query_update(cols, shapes_unchanged=True)
    r = ctx.cast_ray(down)
    assert r["collider"].tolist() == [3, 3] and float(r["distance"][0]) == 16.75
    assert_same(ctx.ray_hits(down), fixture.query_ray_hits(s, cols, down))


def test_spatial_query_plugin_follows_device_graph_world(qctx):
    ctx, s = qctx
    w = plugins.DeviceGraphWorld(scenes.cube_stack(8, 6, 8, brick=True, scalar=s), plugins.PhysicsPlugins(ctx), ctx, substeps=4)
    sq = plugins.SpatialQueryPlugin(ctx)
    rng = np.random.default_rng(1)
    n = int(w.bodies.count)
    memb = np.where(rng.random(n) < 0.1, 2, 1).astype(np.uint32)
    k = 400
    owner = rng.integers(-1, n, k)
    for step in range(3):
        w.step()
        sq.update_pipeline(w, memb, shapes_unchanged=step > 0)
        o = np.where(owner[:, None] >= 0, np.asarray(w.bodies.position[np.maximum(owner, 0)], dtype=np.float64), rng.uniform(-2, 10, (k, 3)))
        rays = sq.ray_casters(o, unit(rng.normal(size=(k, 3))), np.full(k, 20.0), max_hits=rng.integers(0, 6, k), enabled=rng.random(k) < 0.8,
                              owner=owner, solid=rng.random(k) < 0.5)
        hits = sq.raycast(rays)
        assert_same(hits, fixture.query_ray_hits(s, sq.colliders(w, memb), rays), f"step {step} ")
        offs = hits["offsets"].astype(np.int64)
        own = [hits["collider"][offs[i]:offs[i + 1]] for i in range(k)]
        assert all(owner[i] not in own[i] for i in range(k))            # ignore_self
        assert all(len(own[i]) == 0 for i in np.nonzero(rays.max_hits == 0)[0])
