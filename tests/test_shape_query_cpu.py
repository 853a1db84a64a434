"""Shape casts, point projection and point / shape intersections on the host: hand-worked answers with closed forms, an independent numpy
check of the time of impact (an overlap predicate written here, bisected), the witness properties of random hits, the ABI struct layouts and
the inputs the host path refuses.  The fixture's brute force runs csrc/query_math.hpp, the header the device uses."""
import ctypes as C
import subprocess
import tempfile
from pathlib import Path

import numpy as np
import pytest

from avian_b200 import api, fixture

ROOT = Path(__file__).resolve().parent.parent
IDENT = [0.0, 0.0, 0.0, 1.0]
SCALARS = [np.float32, np.float64]
TOL = {np.float32: 2e-6, np.float64: 1e-12}
S2 = np.sqrt(0.5)


def colliders(*items, memberships=None):
    """items: (shape, dims, position, rotation)"""
    sh, dm, ps, rt = zip(*items)
    return api.QueryColliders(shape=np.array(sh, np.uint8), dims=np.array([np.broadcast_to(d, 3) for d in dm], float), position=np.array(ps, float),
                              rotation=np.array(rt, float), memberships=None if memberships is None else np.array(memberships, np.uint32))


def shapes(*items, direction=None, max_distance=100.0, flags=None, **kw):
    sh, dm, ps, rt = zip(*items)
    n = len(sh)
    return api.ShapeQueries(shape=np.array(sh, np.uint8), dims=np.array([np.broadcast_to(d, 3) for d in dm], float), position=np.array(ps, float),
                            rotation=np.array(rt, float), direction=None if direction is None else np.array(direction, float).reshape(n, 3),
                            max_distance=np.broadcast_to(np.asarray(max_distance, float), (n,)).copy(),
                            flags=None if flags is None else np.broadcast_to(np.asarray(flags, np.uint32), (n,)).copy(), **kw)


def cast1(scalar, cols, item, d, maxd=100.0, flags=0):
    r = fixture.query_cast_shape(scalar, cols, shapes(item, direction=[d], max_distance=maxd, flags=flags))
    return int(r["collider"][0]), float(r["distance"][0]), {k: r[k][0].astype(np.float64) for k in ("point1", "point2", "normal1", "normal2")}


def quat(axis, angle):
    a = np.asarray(axis, float) / np.linalg.norm(axis)
    return list(a * np.sin(angle / 2)) + [np.cos(angle / 2)]


def rot(q):
    x, y, z, w = np.asarray(q, float) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


BOX = (0, 1.0, [0.0, 0.0, 0.0], IDENT)
BALL = (1, [1.0, 0, 0], [0.0, 0.0, 0.0], IDENT)
SMALL_BALL = lambda p: (1, [0.5, 0, 0], p, IDENT)
SMALL_BOX = lambda p, q=IDENT: (0, 0.5, p, q)
DOWN = [0.0, -1.0, 0.0]
R02 = np.sqrt(0.2)
# (name, collider, cast shape, direction, t, normal1, point1)
CASES = [
    ("sphere_sphere_head_on", BALL, SMALL_BALL([-5.0, 0, 0]), [1, 0, 0], 3.5, [-1, 0, 0], [-1, 0, 0]),
    ("sphere_sphere_offset", BALL, SMALL_BALL([-5.0, 1.0, 0]), [1, 0, 0], 5 - np.sqrt(1.25), [-np.sqrt(1.25) / 1.5, 1 / 1.5, 0],
     [-np.sqrt(1.25) / 1.5, 1 / 1.5, 0]),
    ("sphere_onto_box_face", BOX, SMALL_BALL([0.2, 5, 0.3]), DOWN, 3.5, [0, 1, 0], [0.2, 1, 0.3]),
    # the centre passes the edge x = y = 1 at 0.3 in x: cylinder of radius 0.5 around the edge, (0.3)² + (y - 1)² = 0.25
    ("sphere_along_edge", BOX, SMALL_BALL([1.3, 5, 0]), DOWN, 3.6, [0.6, 0.8, 0], [1, 1, 0]),
    # over the corner (1, 1, 1) by (0.2, ., 0.1): sphere of radius 0.5 around the corner
    ("sphere_onto_corner", BOX, SMALL_BALL([1.2, 5, 1.1]), DOWN, 4 - R02, [0.4, 2 * R02, 0.2], [1, 1, 1]),
    ("box_sphere_cast_box", BALL, SMALL_BOX([0.0, 5, 0]), DOWN, 3.5, [0, 1, 0], [0, 1, 0]),
    ("box_box_face_face", BOX, SMALL_BOX([0.3, 5, -0.2]), DOWN, 3.5, [0, 1, 0], None),
    # B turned 45° about z (top edge along z at height sqrt 2 / 2), A turned 45° about x (bottom edge along x): edge meets edge
    ("box_box_edge_edge", SMALL_BOX([0.0, 0, 0], quat([0, 0, 1], np.pi / 4)), SMALL_BOX([0.0, 5, 0], quat([1, 0, 0], np.pi / 4)), DOWN, 5 - np.sqrt(2),
     [0, 1, 0], [0, S2, 0]),
]


@pytest.mark.parametrize("scalar", SCALARS, ids=["f32", "f64"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_hand_worked_times_of_impact(case, scalar):
    name, col, item, d, want_t, want_n, want_p = case
    c, t, h = cast1(scalar, colliders(col), item, d)
    tol = TOL[scalar] * 4
    assert c == 0
    assert abs(t - want_t) <= tol * max(1.0, want_t), (t, want_t)
    n = np.asarray(want_n, float) / np.linalg.norm(want_n)
    assert np.allclose(h["normal1"], n, atol=tol) and np.allclose(h["normal2"], -n, atol=tol)
    if want_p is not None:
        assert np.allclose(h["point1"], want_p, atol=tol) and np.allclose(h["point2"], want_p, atol=tol)
    # the shapes touch at the reported points
    assert np.linalg.norm(h["point1"] - h["point2"]) <= tol * 10


def test_face_face_witness_lies_in_the_touching_square():
    c, t, h = cast1(np.float64, colliders(BOX), SMALL_BOX([0.3, 5, -0.2]), DOWN)
    for p in (h["point1"], h["point2"]):
        assert p[1] == pytest.approx(1.0, abs=1e-12)
        assert -0.2 - 1e-12 <= p[0] <= 0.8 + 1e-12 and -0.7 - 1e-12 <= p[2] <= 0.3 + 1e-12


def test_miss_by_one_ulp_past_an_edge_and_max_distance_at_the_toi():
    cols = colliders(BOX)
    # tangent to the edge cylinder x = y = 1 (radius 0.5) at x = 1.5: a hit at t = 4, one ulp further out a miss
    c, t, _ = cast1(np.float64, cols, SMALL_BALL([1.5, 5, 0]), DOWN)
    assert c == 0 and t == pytest.approx(4.0, abs=1e-12)
    assert cast1(np.float64, cols, SMALL_BALL([float(np.nextafter(1.5, 2.0)), 5, 0]), DOWN)[0] == -1
    ball = colliders(BALL)
    assert cast1(np.float64, ball, SMALL_BALL([-5.0, 0, 0]), [1, 0, 0], maxd=3.5)[:2] == (0, 3.5)
    assert cast1(np.float64, ball, SMALL_BALL([-5.0, 0, 0]), [1, 0, 0], maxd=float(np.nextafter(3.5, 0.0)))[0] == -1
    # a box on the same face: max_distance exactly at the TOI
    assert cast1(np.float64, cols, SMALL_BOX([0.0, 5, 0]), DOWN, maxd=3.5)[:2] == (0, 3.5)
    assert cast1(np.float64, cols, SMALL_BOX([0.0, 5, 0]), DOWN, maxd=float(np.nextafter(3.5, 0.0)))[0] == -1


@pytest.mark.parametrize("scalar", SCALARS, ids=["f32", "f64"])
def test_origin_penetration(scalar):
    cols = colliders(BOX, (1, [1.0, 0, 0], [10.0, 0, 0], IDENT), (0, 1.0, [20.0, 0, 0], IDENT))
    # each cast shape overlaps one collider at t = 0 with normal1 = +y
    for item, want_c in ((SMALL_BALL([0.0, 1.2, 0]), 0), (SMALL_BOX([10.0, 1.2, 0]), 1), (SMALL_BOX([20.0, 1.3, 0.1]), 2),
                         (SMALL_BALL([20.0, 0.9, 0.0]), 2)):
        for d, moving_away in ((DOWN, False), ([0.0, 1.0, 0.0], True)):
            c, t, h = cast1(scalar, cols, item, d)
            assert (c, t) == (want_c, 0.0)
            assert np.allclose(h["normal1"], [0, 1, 0], atol=TOL[scalar]) and np.allclose(h["normal2"], [0, -1, 0], atol=TOL[scalar])
            c, t, h = cast1(scalar, cols, item, d, flags=api.CAST_IGNORE_ORIGIN_PENETRATION)
            assert c == (-1 if moving_away else want_c)
            c, t, h = cast1(scalar, cols, item, d, flags=api.CAST_NO_CONTACT_ON_PENETRATION)
            assert (c, t) == (want_c, 0.0) and all(not v.any() for v in h.values())
    # coincident sphere centres: the fixed +y normal
    c, t, h = cast1(np.float64, colliders(BALL), SMALL_BALL([0.0, 0, 0]), [1, 0, 0])
    assert (c, t) == (0, 0.0) and h["normal1"].tolist() == [0, 1, 0]


# ---- an independent check of the geometry: overlap predicates written here, bisected for the TOI -----------------------------------
def box_point_dist(c, R, he, p):
    local = R.T @ (np.asarray(p) - c)
    return np.linalg.norm(local - np.clip(local, -he, he))


def overlap(a, b):
    """a, b: (shape, he, centre, R); closed shapes"""
    (sa, ha, ca, Ra), (sb, hb, cb, Rb) = a, b
    if sa == 1 and sb == 1:
        return np.linalg.norm(ca - cb) <= ha[0] + hb[0]
    if sa == 1 or sb == 1:
        (sp, box) = (a, b) if sa == 1 else (b, a)
        return box_point_dist(box[2], box[3], box[1], sp[2]) <= sp[1][0]
    axes = [Ra[:, i] for i in range(3)] + [Rb[:, i] for i in range(3)] + [np.cross(Ra[:, i], Rb[:, j]) for i in range(3) for j in range(3)]
    for L in axes:
        if np.linalg.norm(L) < 1e-12:
            continue
        ra = np.sum(np.abs(Ra.T @ L) * ha)
        rb = np.sum(np.abs(Rb.T @ L) * hb)
        if abs(L @ (cb - ca)) > ra + rb:
            return False
    return True


def random_pair(rng, kind):
    sa, sb = kind
    ha = rng.uniform(0.3, 1.2, 3) if sa == 0 else np.array([rng.uniform(0.2, 1.0), 0, 0])
    hb = rng.uniform(0.3, 1.2, 3) if sb == 0 else np.array([rng.uniform(0.2, 1.0), 0, 0])
    qa, qb = rng.normal(size=4), rng.normal(size=4)
    qa, qb = qa / np.linalg.norm(qa), qb / np.linalg.norm(qb)
    cb = rng.uniform(-1, 1, 3)
    ca = cb + rng.normal(size=3) * 4 + np.array([0, 5.0, 0])
    d = (cb + rng.uniform(-1.2, 1.2, 3)) - ca        # aimed near B: most casts hit, some graze past
    d /= np.linalg.norm(d)
    return (sa, ha, ca, qa), (sb, hb, cb, qb), d


KINDS = [(0, 0), (1, 0), (0, 1), (1, 1)]


def cast_pair(a, b, d):
    (sa, ha, ca, qa), (sb, hb, cb, qb) = a, b
    cols = api.QueryColliders(shape=np.array([sb], np.uint8), dims=hb[None], position=cb[None], rotation=qb[None])
    q = api.ShapeQueries(shape=np.array([sa], np.uint8), dims=ha[None], position=ca[None], rotation=qa[None], direction=d[None], max_distance=np.array([50.0]))
    r = fixture.query_cast_shape(np.float64, cols, q)
    return int(r["collider"][0]), float(r["distance"][0]), {k: r[k][0] for k in ("point1", "point2", "normal1", "normal2")}


@pytest.mark.parametrize("kind", KINDS, ids=["box_box", "sphere_box", "box_sphere", "sphere_sphere"])
def test_toi_agrees_with_bisected_numpy_overlap(kind):
    rng = np.random.default_rng(100 + 10 * kind[0] + kind[1])
    hits = misses = 0
    for _ in range(150):
        a, b, d = random_pair(rng, kind)
        c, t, _ = cast_pair(a, b, d)
        posed = lambda s, t_: (s[0], s[1], s[2] + d * t_, rot(s[3]))
        A, B = lambda t_: posed(a, t_), (b[0], b[1], b[2], rot(b[3]))
        if c < 0:
            misses += 1
            assert not any(overlap(A(x), B) for x in np.linspace(0, 50, 2001))
            continue
        hits += 1
        if overlap(A(0.0), B):                           # origin penetration
            assert t == 0
            continue
        assert t > 0
        assert overlap(A(t * (1 + 1e-9)), B), "not touching just after the TOI"
        assert not overlap(A(t * (1 - 1e-9)), B), "already touching just before the TOI"
        # bisection of the predicate lands on the same t
        lo, hi = 0.0, t * (1 + 1e-6)
        for _ in range(80):
            mid = 0.5 * (lo + hi)
            lo, hi = (lo, mid) if overlap(A(mid), B) else (mid, hi)
        assert abs(hi - t) <= 1e-9 * t
    assert hits > 100 and misses > 0


def surface_dist(s, p):
    """distance of p from the surface of s = (shape, he, centre, R)"""
    sh, he, c, R = s
    if sh == 1:
        return abs(np.linalg.norm(p - c) - he[0])
    local = R.T @ (p - c)
    out = np.linalg.norm(local - np.clip(local, -he, he))
    return out if out > 0 else np.min(he - np.abs(local))


def shape_dist(s, p):
    sh, he, c, R = s
    if sh == 1:
        return max(np.linalg.norm(p - c) - he[0], 0.0)
    return box_point_dist(c, R, he, p)


@pytest.mark.parametrize("kind", KINDS, ids=["box_box", "sphere_box", "box_sphere", "sphere_sphere"])
def test_witness_properties_of_random_hits(kind):
    rng = np.random.default_rng(200 + 10 * kind[0] + kind[1])
    checked = 0
    for _ in range(150):
        a, b, d = random_pair(rng, kind)
        c, t, h = cast_pair(a, b, d)
        if c < 0 or t == 0:
            continue
        checked += 1
        A = (a[0], a[1], a[2] + d * t, rot(a[3]))
        B = (b[0], b[1], b[2], rot(b[3]))
        size = max(np.max(a[1]), np.max(b[1]), 1.0)
        tol = 1e-9 * size
        assert surface_dist(B, h["point1"]) <= tol and surface_dist(A, h["point2"]) <= tol
        assert np.linalg.norm(h["point1"] - h["point2"]) <= tol
        for n, s, p in ((h["normal1"], B, h["point1"]), (h["normal2"], A, h["point2"])):
            assert abs(np.linalg.norm(n) - 1) <= 1e-12
            # outward: a step along the normal leaves the shape by exactly its length (the normal lies in the normal cone there)
            assert abs(shape_dist(s, p + 1e-4 * n) - 1e-4) <= 1e-8
        assert np.allclose(h["normal2"], -h["normal1"])
        assert d @ h["normal1"] <= 1e-12
    assert checked > 100


def test_radius_zero_sphere_is_the_ray_cast():
    rng = np.random.default_rng(6)
    n = 300
    cols = api.QueryColliders(shape=(rng.random(n) < 0.4).astype(np.uint8), dims=rng.uniform(0.2, 1.5, (n, 3)), position=rng.uniform(-10, 10, (n, 3)),
                              rotation=rng.normal(size=(n, 4)))
    m = 500
    o, d = rng.uniform(-12, 12, (m, 3)), rng.normal(size=(m, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    ray = fixture.query_cast_ray(np.float64, cols, api.Rays(origin=o, direction=d, max_distance=np.full(m, 40.0)))
    q = api.ShapeQueries(shape=np.ones(m, np.uint8), dims=np.zeros((m, 3)), position=o, rotation=np.tile(IDENT, (m, 1)), direction=d, max_distance=np.full(m, 40.0))
    sc = fixture.query_cast_shape(np.float64, cols, q)
    assert np.array_equal(sc["collider"], ray["collider"]) and (sc["collider"] >= 0).sum() > 100
    hit = ray["collider"] >= 0
    # the formulas differ (ray_sphere's b² - ac cancels near tangency): a few ulp of the scene's coordinates (|x| < 16)
    assert np.allclose(sc["distance"][hit], ray["distance"][hit], rtol=0, atol=16 * np.spacing(16.0))
    outside = hit & (ray["distance"] > 0)
    assert np.allclose(sc["normal1"][outside], ray["normal"][outside], atol=1e-12)


# ---- point projection and intersections --------------------------------------------------------------------------------------------
def project(scalar, cols, p, solid=True):
    r = fixture.query_project_point(scalar, cols, api.Points(point=np.array([p], float), solid=np.array([solid])))
    return int(r["collider"][0]), r["point"][0].astype(np.float64), bool(r["is_inside"][0])


@pytest.mark.parametrize("scalar", SCALARS, ids=["f32", "f64"])
def test_projection_cases(scalar):
    box, ball = colliders(BOX), colliders((1, [1.0, 0, 0], [0.0, 0, 0], IDENT))
    tol = TOL[scalar]
    c, p, inside = project(scalar, box, [3.0, 0.5, -2.0])
    assert (c, inside) == (0, False) and np.allclose(p, [1, 0.5, -1], atol=tol)
    c, p, inside = project(scalar, box, [0.25, 0.5, -0.125])
    assert (c, inside) == (0, True) and np.allclose(p, [0.25, 0.5, -0.125], atol=tol)
    c, p, inside = project(scalar, box, [0.25, 0.5, -0.125], solid=False)        # nearest face: +y (depth 0.5)
    assert (c, inside) == (0, True) and np.allclose(p, [0.25, 1, -0.125], atol=tol)
    c, p, inside = project(scalar, box, [1.0, 0.5, 0.0], solid=False)             # on the surface: inside, projects onto itself
    assert (c, inside) == (0, True) and np.allclose(p, [1, 0.5, 0], atol=tol)
    assert project(scalar, box, [0.0, 0.0, 0.0], solid=False)[1].tolist() == [1, 0, 0]      # centre: lowest axis, + side
    assert project(scalar, box, [0.0, -0.5, -0.5], solid=False)[1].tolist() == [0, -1, -0.5]   # y and z tie at depth 0.5: y, - side
    assert project(scalar, box, [0.5, 0.0, 0.5], solid=False)[1].tolist() == [1, 0, 0.5]      # x and z tie: x, + side
    c, p, inside = project(scalar, ball, [0.0, 3.0, 4.0])
    assert (c, inside) == (0, False) and np.allclose(p, [0, 0.6, 0.8], atol=tol)
    c, p, inside = project(scalar, ball, [0.0, 0.3, 0.4], solid=False)
    assert (c, inside) == (0, True) and np.allclose(p, [0, 0.6, 0.8], atol=tol)
    assert project(scalar, ball, [0.0, 0.0, 0.0], solid=False)[1].tolist() == [0, 1, 0]     # sphere centre: +y
    # the closest of several; equal distances go to the lower index; a masked-out collider is skipped
    two = colliders(BOX, (0, 1.0, [4.0, 0, 0], IDENT), memberships=[1, 2])
    assert project(scalar, two, [2.0, 0.0, 0.0])[0] == 0
    r = fixture.query_project_point(scalar, two, api.Points(point=np.array([[2.0, 0, 0], [2.0, 0, 0]]), mask=np.array([2, 1], np.uint32),
                                                            exclude=[[], [0]]))
    assert r["collider"].tolist() == [1, -1]


@pytest.mark.parametrize("scalar", SCALARS, ids=["f32", "f64"])
def test_touching_intersects_and_a_one_ulp_gap_does_not(scalar):
    up = lambda x: float(np.nextafter(scalar(x), scalar(np.inf)))
    cols = colliders(BOX, (1, [1.0, 0, 0], [10.0, 0, 0], IDENT))
    items = [SMALL_BOX([1.5, 0, 0]), SMALL_BOX([up(1.5), 0, 0]), (1, [1.0, 0, 0], [12.0, 0, 0], IDENT), (1, [1.0, 0, 0], [up(12.0), 0, 0], IDENT),
             SMALL_BALL([1.5, 0, 0]), SMALL_BALL([up(1.5), 0, 0]), SMALL_BOX([11.5, 0, 0]), SMALL_BOX([up(11.5), 0, 0])]
    r = fixture.query_shape_intersections(scalar, cols, shapes(*items))
    assert np.diff(r["offsets"]).tolist() == [1, 0, 1, 0, 1, 0, 1, 0]
    assert r["collider"].tolist() == [0, 1, 0, 1]
    pts = api.Points(point=np.array([[1.0, 1.0, 1.0], [up(1.0), 0, 0], [10.0, 1.0, 0.0], [10.0, up(1.0), 0.0], [0.5, 0.5, 0.5]]))
    r = fixture.query_point_intersections(scalar, cols, pts)
    assert np.diff(r["offsets"]).tolist() == [1, 0, 1, 0, 1]
    # rotated boxes: an edge against a face, and the filter
    turned = SMALL_BOX([0.0, 1.0 + S2 * 0.5, 0.0], quat([0, 0, 1], np.pi / 4))
    r = fixture.query_shape_intersections(scalar, colliders(BOX, memberships=[4]), shapes(turned, turned, mask=np.array([4, 1], np.uint32)))
    assert r["offsets"].tolist() == [0, 1, 1]


def test_refused_inputs():
    cols = colliders(BOX)
    good = shapes(SMALL_BALL([0.0, 5, 0]), direction=[DOWN])
    assert fixture.query_cast_shape(np.float64, cols, good)["collider"].tolist() == [0]
    cases = [(shapes((0, [1.0, -0.5, 1.0], [0, 5, 0], IDENT), direction=[DOWN]), "negative"),
             (shapes((1, [-1.0, 0, 0], [0, 5, 0], IDENT), direction=[DOWN]), "negative"),
             (shapes((2, 1.0, [0, 5, 0], IDENT), direction=[DOWN]), "unknown shape"),
             (shapes(SMALL_BALL([0.0, 5, 0]), direction=[DOWN], target_distance=np.array([0.1])), "target_distance")]
    for scalar in SCALARS:
        for q, why in cases:
            for fn in (fixture.query_cast_shape, fixture.query_shape_hits):
                with pytest.raises(api.AvianError) as e:
                    fn(scalar, cols, q)
                assert e.value.status == api.ERR_INVALID_ARGUMENT and why in str(e.value)
        with pytest.raises(api.AvianError):
            fixture.query_shape_intersections(scalar, cols, cases[2][0])
    # intersections ignore the cast columns: a target distance does not matter there
    assert fixture.query_shape_intersections(np.float64, cols, shapes(SMALL_BALL([0.0, 1.2, 0]), target_distance=np.array([0.1])))["collider"].tolist() == [0]
    lib = fixture._load()
    q = shapes(SMALL_BALL([0.0, 5, 0]), SMALL_BALL([0.0, 5, 0]), direction=[DOWN, DOWN], exclude=[[0], []])
    s, keep = q.as_struct(np.float64)
    c, keep_c = cols.as_struct(np.float64)
    o, out = api.shape_closest(2, np.float64)
    keep[10][:] = [0, 1, 0]                      # exclude_offsets not monotone
    assert lib.avh_query_cast_shape(64, C.byref(c), C.byref(s), C.byref(o)) == api.ERR_INVALID_ARGUMENT
    assert b"monotone" in lib.avh_query_error()
    keep[10][:] = [0, 1, 2]                      # past exclude_count
    assert lib.avh_query_cast_shape(64, C.byref(c), C.byref(s), C.byref(o)) == api.ERR_INVALID_ARGUMENT
    assert b"past exclude_count" in lib.avh_query_error()
    p = api.Points(point=np.zeros((2, 3)), exclude=[[0], []])
    pb, keep_p = p.as_struct(np.float64)
    keep_p[3][:] = [0, 2, 1]
    h, _ = api.hit_list(2, 4, np.float64, False)
    assert lib.avh_query_point_intersections(64, C.byref(c), C.byref(pb), C.byref(h)) == api.ERR_INVALID_ARGUMENT


def test_non_finite_query_shapes_hit_nothing():
    cols = colliders(BOX)
    bad = [SMALL_BALL([np.nan, 5, 0]), (1, [np.inf, 0, 0], [0, 5, 0], IDENT), SMALL_BOX([0, 5, 0], [0.0, 0, 0, 0]), SMALL_BOX([0, 5, 0], [np.nan, 0, 0, 1])]
    r = fixture.query_cast_shape(np.float64, cols, shapes(*bad, direction=[DOWN] * 4))
    assert r["collider"].tolist() == [-1] * 4
    r = fixture.query_cast_shape(np.float64, cols, shapes(SMALL_BALL([0, 5, 0]), SMALL_BALL([0, 5, 0]), direction=[[np.nan, -1, 0], DOWN],
                                                          max_distance=[100.0, np.inf]))
    assert r["collider"].tolist() == [-1, -1]
    assert fixture.query_shape_intersections(np.float64, cols, shapes(*bad))["collider"].size == 0
    r = fixture.query_project_point(np.float64, cols, api.Points(point=np.array([[np.nan, 0, 0], [0, np.inf, 0]])))
    assert r["collider"].tolist() == [-1, -1]


def test_shape_struct_layouts_match_the_header():
    """sizeof of every new spatial-query ABI struct, compiled from the header with gcc, equals the ctypes mirror"""
    names = ["AvnShapeBatch", "AvnPointBatch", "AvnShapeClosest", "AvnShapeHitList", "AvnPointProjection"]
    src = '#include <stdio.h>\n#include "avian_b200.h"\nint main(){' + "".join(f'printf("{n} %zu\\n", sizeof({n}));' for n in names) + "return 0;}"
    with tempfile.TemporaryDirectory() as d:
        (Path(d) / "s.c").write_text(src)
        subprocess.run(["gcc", "-I", str(ROOT / "include"), "-o", f"{d}/s", f"{d}/s.c"], check=True)
        out = subprocess.run([f"{d}/s"], capture_output=True, text=True, check=True).stdout
    sizes = dict(line.split() for line in out.strip().splitlines())
    for n in names:
        assert int(sizes[n]) == C.sizeof(getattr(api, n)), n
