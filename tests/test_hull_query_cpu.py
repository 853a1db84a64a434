"""Convex hulls in the spatial queries and in move and slide, on the host (no GPU): the fixture's brute force (csrc/hull_query_math.hpp and
csrc/move_math.hpp, the headers the device runs, with the hull table) against the independent float64 restatement of
tests/hull_query_reference.py (linear programs for rays and polytope casts, bisection for spheres and capsules), the unit cube as an 8-vertex
hull against the cuboid results, a hand-worked tetrahedron, move_reference's loop, and the refused inputs."""
from __future__ import annotations

import numpy as np
import pytest

from avian_b200 import api, fixture, scenes
import hull_query_reference as hqr
import hull_reference as hr
import move_reference as mref
from capsule_reference import capsule_segment
from move_scenes import random_quats

CUB, SPH, CAP, HULL = fixture.SHAPE_CUBOID, fixture.SHAPE_SPHERE, fixture.SHAPE_CAPSULE, fixture.SHAPE_CONVEX_HULL
IDENT = [0.0, 0.0, 0.0, 1.0]
F64 = np.float64
CUBE = np.array([[(1 if m & 1 else -1), (1 if m & 2 else -1), (1 if m & 4 else -1)] for m in range(8)], float) * 0.5
TET = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], float)
TET_FACES = [[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]]


@pytest.fixture(scope="module")
def table():
    return scenes.hull_pile(4).hulls


def unit(v):
    v = np.asarray(v, float)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def cols(*items):
    """items: (shape, dims, position, rotation)"""
    sh, dm, ps, rt = zip(*items)
    return api.QueryColliders(shape=np.array(sh, np.uint8), dims=np.array([np.broadcast_to(np.asarray(d, float), 3) for d in dm]),
                              position=np.array(ps, float), rotation=np.array(rt, float))


def shapes(items, d=None, maxd=None, flags=None):
    sh, dm, ps, rt = zip(*items)
    kw = {}
    if d is not None:
        kw = dict(direction=np.array(d, float).reshape(-1, 3), max_distance=np.full(len(sh), maxd), flags=None if flags is None else np.full(len(sh), flags, np.uint32))
    return api.ShapeQueries(shape=np.array(sh, np.uint8), dims=np.array([np.broadcast_to(np.asarray(x, float), 3) for x in dm]), position=np.array(ps, float),
                            rotation=np.array(rt, float), **kw)


def world_poly(table, shape, dims, pos, rot):
    if shape == HULL:
        V, F = hqr.table_poly(table, int(dims[0]))
        return hr.posed(V, pos, rot), F
    return hr.box_poly(dims, pos, rot)


def test_ray_vs_linear_program(table):
    """rays at random posed hulls: the TOI against the LP over the face half-spaces, the normal a face normal whose plane holds the hit"""
    rng = np.random.default_rng(1)
    n = 60
    idx = rng.integers(0, table.count, n)
    pos = rng.uniform(-2, 2, (n, 3))
    rot = random_quats(rng, n)
    o = pos + unit(rng.normal(size=(n, 3))) * 1.5
    d = unit(pos + rng.normal(size=(n, 3)) * 0.15 - o)
    hits = 0
    for i in range(n):
        c = cols((HULL, [idx[i], 0, 0], pos[i], rot[i]))
        r = fixture.query_cast_ray(F64, c, api.Rays(origin=o[i:i + 1], direction=d[i:i + 1], max_distance=np.array([5.0])), hulls=table)
        V, F = world_poly(table, HULL, [idx[i]], pos[i], rot[i])
        want = hqr.ray_lp(o[i], d[i], V, F, 5.0)
        got = float(r["distance"][0]) if r["collider"][0] >= 0 else None
        assert (got is None) == (want is None), (i, got, want)
        if got is None:
            continue
        hits += 1
        assert got == pytest.approx(want, abs=1e-9)
        nrm = r["normal"][0]
        x = o[i] + got * d[i]
        assert min(np.linalg.norm(nrm - pn) + abs(pn @ x - pc) for pn, pc in hr.planes(V, F)) < 1e-9
        assert nrm @ d[i] < 0
    assert hits > n // 2


def _cast_pairs(rng, table, n):
    for i in range(n):
        sa, sb = [(HULL, HULL), (HULL, CUB), (CUB, HULL)][i % 3]
        da = [rng.integers(0, table.count), 0, 0] if sa == HULL else rng.uniform(0.1, 0.3, 3)
        db = [rng.integers(0, table.count), 0, 0] if sb == HULL else rng.uniform(0.1, 0.3, 3)
        pb = rng.uniform(-1, 1, 3)
        pa = pb + unit(rng.normal(size=3)) * 1.2
        d = unit(pb + rng.normal(size=3) * 0.2 - pa)
        yield (sa, da, pa, random_quats(rng, 1)[0]), (sb, db, pb, random_quats(rng, 1)[0]), d


def test_polytope_casts_vs_linear_program(table):
    """hull-hull, hull-cuboid and cuboid-hull casts: the TOI against the LP; the witnesses lie on the two shapes at the TOI pose, normal1 is a
    unit vector that points from the collider towards the cast shape"""
    rng = np.random.default_rng(2)
    hits = 0
    for a, b, d in _cast_pairs(rng, table, 45):
        r = fixture.query_cast_shape(F64, cols(b), shapes([a], d, 3.0), hulls=table)
        VA, FA = world_poly(table, *a)
        VB, FB = world_poly(table, *b)
        want = hqr.poly_cast_lp(VA, FA, VB, FB, d, 3.0)
        got = float(r["distance"][0]) if r["collider"][0] >= 0 else None
        assert (got is None) == (want is None), (got, want)
        if got is None:
            continue
        hits += 1
        assert got == pytest.approx(want, abs=1e-8)
        if got == 0:
            continue
        n1, p1, p2 = r["normal1"][0], r["point1"][0], r["point2"][0]
        assert np.linalg.norm(n1) == pytest.approx(1.0, abs=1e-12)
        assert abs(hr.point_distance(p1, VB, FB)) < 1e-7
        assert abs(hr.point_distance(p2, VA + got * d, FA)) < 1e-7
        assert n1 @ d < 1e-9
    assert hits > 20


def test_sphere_and_capsule_casts_vs_bisection(table):
    """a sphere or a capsule cast at a hull and a hull cast at a sphere or a capsule: the TOI against the bisected reference distance; the
    witnesses at distance r and 0 of the two shapes"""
    rng = np.random.default_rng(3)
    hits = 0
    for i in range(24):
        h = [rng.integers(0, table.count), 0, 0]
        ph, qh = rng.uniform(-1, 1, 3), random_quats(rng, 1)[0]
        other = SPH if i % 2 == 0 else CAP
        do = [rng.uniform(0.05, 0.25), rng.uniform(0.0, 0.3), 0.0]
        po = ph + unit(rng.normal(size=3)) * 1.3
        qo = random_quats(rng, 1)[0]
        d = unit(ph + rng.normal(size=3) * 0.2 - po)
        hull_cast = i % 4 >= 2
        if hull_cast:    # the hull moves along -d onto the other shape: the same relative motion
            r = fixture.query_cast_shape(F64, cols((other, do, po, qo)), shapes([(HULL, h, ph, qh)], -d, 3.0), hulls=table)
        else:
            r = fixture.query_cast_shape(F64, cols((HULL, h, ph, qh)), shapes([(other, do, po, qo)], d, 3.0), hulls=table)
        V, F = world_poly(table, HULL, h, ph, qh)
        if other == SPH:
            want = hqr.sphere_cast(po, do[0], d, V, F, 3.0)
        else:
            p0, p1 = capsule_segment(po, qo, do[1])
            want = hqr.capsule_cast(p0, p1, do[0], d, V, F, 3.0)
        got = float(r["distance"][0]) if r["collider"][0] >= 0 else None
        assert (got is None) == (want is None), (i, got, want)
        if got is None:
            continue
        hits += 1
        assert got == pytest.approx(want, abs=1e-7)
        on_hull = r["point2"][0] if hull_cast else r["point1"][0]
        shift = -got * d if hull_cast else np.zeros(3)
        assert abs(hr.point_distance(on_hull, V + shift, F)) < 1e-7
    assert hits > 10


def test_projection_containment_and_intersections(table):
    """project_point, point_intersections and shape_intersections against the reference distances, with touching and a one-ulp gap"""
    rng = np.random.default_rng(4)
    h = [5, 0, 0]
    ph, qh = np.array([0.3, -0.2, 0.1]), random_quats(rng, 1)[0]
    c = cols((HULL, h, ph, qh))
    V, F = world_poly(table, HULL, h, ph, qh)
    x = ph + rng.normal(size=(80, 3)) * 0.25
    for solid in (True, False):
        r = fixture.query_project_point(F64, c, api.Points(point=x, solid=np.full(80, solid)), hulls=table)
        for i in range(80):
            want, inside = hqr.project(x[i], V, F, solid)
            assert bool(r["is_inside"][i]) == inside
            assert np.allclose(r["point"][i], want, atol=1e-9)
    inside = fixture.query_point_intersections(F64, c, api.Points(point=x), hulls=table)
    counts = np.diff(inside["offsets"].astype(np.int64))
    assert np.array_equal(counts == 1, [hr.point_distance(p, V, F) <= 0 for p in x])
    # a sphere touching the hull's top vertex, and one ulp above touching
    top = V[np.argmax(V[:, 1])]
    for gap, want in ((0.0, 1), (np.spacing(top[1] + 0.2) * 4, 0)):
        s = shapes([(SPH, [0.2, 0, 0], top + [0.0, 0.2 + gap, 0.0], IDENT)])
        got = fixture.query_shape_intersections(F64, c, s, hulls=table)
        assert int(got["offsets"][1]) == want, gap
    # polytopes: a cuboid resting on the hull's top vertex, and lifted by a few ulps
    for gap, want in ((0.0, 1), (np.spacing(top[1] + 0.25) * 4, 0)):
        s = shapes([(CUB, [0.5, 0.25, 0.5], top + [0.0, 0.25 + gap, 0.0], IDENT)])
        got = fixture.query_shape_intersections(F64, c, s, hulls=table)
        assert int(got["offsets"][1]) == want, gap
    # capsules against the reference segment distance
    for k in range(30):
        p, q = ph + rng.normal(size=3) * 0.4, random_quats(rng, 1)[0]
        dm = [rng.uniform(0.02, 0.1), rng.uniform(0.0, 0.2), 0.0]
        p0, p1 = capsule_segment(p, q, dm[1])
        want = hr.segment_distance(p0, p1, V, F) <= dm[0]
        got = fixture.query_shape_intersections(F64, c, shapes([(CAP, dm, p, q)]), hulls=table)
        assert int(got["offsets"][1]) == int(want)


def test_unit_cube_hull_equals_the_cuboid():
    """the unit cube as an 8-vertex hull against the existing cuboid results: TOIs within tolerance, the same normals away from ties"""
    table = api.ConvexHulls.from_polyhedra([(CUBE, hr.CUBE_FACES)])
    rng = np.random.default_rng(5)
    q = random_quats(rng, 1)[0]
    hull, box = cols((HULL, [0, 0, 0], [0.1, 0.2, 0.3], q)), cols((CUB, [0.5, 0.5, 0.5], [0.1, 0.2, 0.3], q))
    n = 200
    o = unit(rng.normal(size=(n, 3))) * 2
    d = unit(rng.normal(size=(n, 3)) * 0.3 - o)
    rays = api.Rays(origin=o, direction=d, max_distance=np.full(n, 5.0))
    a = fixture.query_cast_ray(F64, hull, rays, hulls=table)
    b = fixture.query_cast_ray(F64, box, rays)
    assert np.array_equal(a["collider"], b["collider"])
    assert np.allclose(a["distance"], b["distance"], atol=1e-12)
    assert np.allclose(a["normal"], b["normal"], atol=1e-12)
    for s, dm in ((SPH, [0.2, 0, 0]), (CAP, [0.1, 0.2, 0]), (CUB, [0.2, 0.1, 0.3])):
        casts = api.ShapeQueries(shape=np.full(n, s, np.uint8), dims=np.tile(dm, (n, 1)), position=o, rotation=random_quats(rng, n), direction=d,
                                 max_distance=np.full(n, 5.0))
        a = fixture.query_cast_shape(F64, hull, casts, hulls=table)
        b = fixture.query_cast_shape(F64, box, casts, capsules=True)
        assert np.array_equal(a["collider"], b["collider"]), s
        assert np.allclose(a["distance"], b["distance"], atol=1e-9), s
        hit = a["collider"] >= 0
        assert hit.sum() > n // 3
        # the same normal except where the contact is a tie between features (edge or corner first contact)
        same = np.isclose(np.einsum("ij,ij->i", a["normal1"], b["normal1"]), 1.0, atol=1e-9)
        assert same[hit].mean() > 0.9, s
    pts = api.Points(point=rng.normal(size=(n, 3)) * 0.6, solid=rng.random(n) < 0.5)
    a = fixture.query_project_point(F64, hull, pts, hulls=table)
    b = fixture.query_project_point(F64, box, pts)
    assert np.array_equal(a["is_inside"], b["is_inside"])
    assert np.allclose(a["point"], b["point"], atol=1e-12)


def test_tetrahedron_hand_worked():
    """a ray hits the unit tetrahedron through a vertex, an edge and a face; a hollow ray from inside exits through the slanted face"""
    table = api.ConvexHulls.from_polyhedra([(TET, TET_FACES)])
    c = cols((HULL, [0, 0, 0], [0, 0, 0], IDENT))

    def ray(o, d, solid=True):
        r = fixture.query_cast_ray(F64, c, api.Rays(origin=np.array([o], float), direction=unit([d])[None].reshape(1, 3), max_distance=np.array([10.0]),
                                                    solid=np.array([solid], np.uint8)), hulls=table)
        return int(r["collider"][0]), float(r["distance"][0]), r["normal"][0]

    k, t, n = ray([2.0, 0.0, 0.0], [-1, 0, 0])                       # the vertex (1, 0, 0), along the edge on the x axis
    assert k == 0 and t == pytest.approx(1.0) and np.allclose(n, unit([1, 1, 1]))
    k, t, n = ray([0.5, 0.0, -1.0], [0, 0, 1])                       # the edge (0,0,0)-(1,0,0) on the y = 0 face
    assert k == 0 and t == pytest.approx(1.0) and np.allclose(n, [0, 0, -1])
    k, t, n = ray([0.2, 0.2, -1.0], [0, 0, 1])                       # the face z = 0
    assert k == 0 and t == pytest.approx(1.0) and np.allclose(n, [0, 0, -1])
    k, t, n = ray([2.0, 2.0, 2.0], [-1, -1, -1])                     # the slanted face x + y + z = 1
    assert k == 0 and t == pytest.approx(np.sqrt(3) * 5 / 3) and np.allclose(n, unit([1, 1, 1]))
    k, t, n = ray([0.1, 0.1, 0.1], [1, 1, 1], solid=False)           # hollow from inside: exits through x + y + z = 1
    assert k == 0 and t == pytest.approx(np.sqrt(3) * 0.7 / 3) and np.allclose(n, unit([1, 1, 1]))
    k, t, n = ray([0.1, 0.1, 0.1], [1, 1, 1], solid=True)
    assert k == 0 and t == 0 and np.all(n == 0)
    k, t, n = ray([1.0 + 1e-9, 0.0, -2.0], [0, 0, 1])                # just past the vertex: a miss
    assert k == -1


def _patched_move_reference(monkeypatch, table):
    """tests/move_reference.py's loop with the hull table: its casts and contact planes through the hull-enabled fixture, its candidate
    boxes the posed vertices' (a capsule's: the segment ends grown by the radius)"""
    shim = type("shim", (), {})()
    shim.SHAPE_SPHERE = fixture.SHAPE_SPHERE
    shim.query_cast_shape = lambda s, c, q: fixture.query_cast_shape(s, c, q, hulls=table)
    shim.move_contact = lambda *a: fixture.move_contact(*a, hulls=table)
    monkeypatch.setattr(mref, "fixture", shim)
    old = mref._aabb

    def aabb(shape, he, p, q):
        if shape == CAP:
            p0, p1 = capsule_segment(np.asarray(p, float), np.asarray(q, float), he[1])
            return np.minimum(p0, p1) - he[0], np.maximum(p0, p1) + he[0]
        if shape != HULL:
            return old(shape, he, p, q)
        V, _ = hqr.table_poly(table, int(he[0]))
        W = hr.posed(V, p, q)
        return W.min(0), W.max(0)
    monkeypatch.setattr(mref, "_aabb", aabb)


def test_hull_characters_and_obstacles_vs_move_reference(monkeypatch, table):
    rng = np.random.default_rng(6)
    n = 60
    shape = rng.choice([CUB, SPH, CAP, HULL], n).astype(np.uint8)
    dims = rng.uniform(0.2, 0.5, (n, 3))
    dims[shape == HULL] = 0.0
    dims[shape == HULL, 0] = rng.integers(0, table.count, (shape == HULL).sum())
    c = api.QueryColliders(shape=shape, dims=dims, position=rng.uniform(-2, 2, (n, 3)), rotation=random_quats(rng, n))
    _patched_move_reference(monkeypatch, table)
    scene = mref.Scene(c)
    cfg = api.MoveConfig()
    m = 24
    cshape = np.where(np.arange(m) % 2 == 0, HULL, CAP).astype(np.uint8)
    cdims = np.tile([0.25, 0.3, 0.0], (m, 1))
    cdims[cshape == HULL] = 0.0
    cdims[cshape == HULL, 0] = rng.integers(0, table.count, (cshape == HULL).sum())
    pos, rot = rng.uniform(-2, 2, (m, 3)), np.tile(IDENT, (m, 1))
    vel = unit(rng.normal(size=(m, 3))) * 60
    batch = api.MoveBatch(shape=cshape, dims=cdims, position=pos, rotation=rot, velocity=vel)
    got = fixture.move_and_slide(F64, c, cfg, batch, hulls=table)
    hits = 0
    for i in range(m):
        p, v, hl = mref.move_one(scene, cfg, int(cshape[i]), cdims[i], pos[i], rot[i], vel[i])
        assert np.allclose(got["position"][i], p, atol=1e-9), i
        assert np.allclose(got["velocity"][i], v, atol=1e-9), i
        for it, col, safe, toi in hl:
            assert got["hit_collider"][i, it] == col
            assert got["hit_toi"][i, it] == pytest.approx(toi, abs=1e-12)
            hits += 1
    assert hits > 5


def test_refusals(table):
    hc = cols((HULL, [1, 0, 0], [0, 0, 0], IDENT), (CUB, [0.5, 0.5, 0.5], [2, 0, 0], IDENT))
    rays = api.Rays(origin=np.array([[0.0, 5.0, 0.0]]), direction=np.array([[0.0, -1.0, 0.0]]), max_distance=np.array([10.0]))
    with pytest.raises(api.AvianError, match="unknown shape"):              # shape 3 without the hull bit, as before hulls were queried
        fixture.query_cast_ray(F64, hc, rays)
    with pytest.raises(api.AvianError, match="unknown shape"):
        fixture.query_cast_ray(F64, hc, rays, capsules=True)
    lib = fixture._load()
    c, keep = hc.as_struct(F64)
    r, keep_r = rays.as_struct(F64)
    o_arr = {"collider": np.zeros(1, np.int32), "distance": np.zeros(1), "normal": np.zeros((1, 3))}
    o = api.AvnRayClosest(*(o_arr[k].ctypes.data for k in ("collider", "distance", "normal")))
    import ctypes as C
    assert lib.avh_query_cast_ray_hulls(64 | fixture.HULL_BIT, C.byref(c), C.byref(r), C.byref(o), None) == api.ERR_INVALID_ARGUMENT   # no table
    assert b"no hull table" in lib.avh_query_error()
    bad = cols((HULL, [table.count, 0, 0], [0, 0, 0], IDENT))
    with pytest.raises(api.AvianError, match="below the hull table's count"):
        fixture.query_cast_ray(F64, bad, rays, hulls=table)
    with pytest.raises(api.AvianError, match="below the hull table's count"):
        fixture.query_cast_ray(F64, cols((HULL, [0.5, 0, 0], [0, 0, 0], IDENT)), rays, hulls=table)
    with pytest.raises(api.AvianError, match="below the hull table's count"):
        fixture.query_cast_shape(F64, hc, shapes([(HULL, [-1, 0, 0], [0, 3, 0], IDENT)], [0, -1, 0], 5.0), hulls=table)
    with pytest.raises(api.AvianError, match="below the hull table's count"):
        fixture.query_cast_shape(F64, hc, shapes([(HULL, [table.count, 0, 0], [0, 3, 0], IDENT)], [0, -1, 0], 5.0), hulls=table)
    with pytest.raises(api.AvianError, match="below the hull table's count"):
        fixture.move_and_slide(F64, hc, api.MoveConfig(), api.MoveBatch(shape=np.array([HULL], np.uint8), dims=np.array([[99.0, 0, 0]]),
                                                                       position=np.zeros((1, 3)), rotation=np.array([IDENT]), velocity=np.ones((1, 3))), hulls=table)
    assert fixture.query_cast_ray(F64, hc, rays, hulls=table)["collider"][0] == 0
