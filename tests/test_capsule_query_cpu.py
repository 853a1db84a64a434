"""Capsules in the spatial queries and in move and slide, on the host (no GPU): the fixture's brute force (csrc/query_math.hpp and
csrc/move_math.hpp, the headers the device runs, with the capsule bit set) against the independent float64 restatement of
tests/capsule_reference.py and tests/capsule_query_reference.py, hand-worked grazing rays and closed forms, the bisected overlap predicate for the five capsule cast kinds, and the
refused inputs."""
from __future__ import annotations

import math
import types

import numpy as np
import pytest

from avian_b200 import api, fixture
import capsule_query_reference as cqr
import capsule_reference as cr
import move_reference as mref
from move_scenes import random_characters, random_colliders

CUB, SPH, CAP = fixture.SHAPE_CUBOID, fixture.SHAPE_SPHERE, fixture.SHAPE_CAPSULE
IDENT = [0.0, 0.0, 0.0, 1.0]
SCALARS = [np.float32, np.float64]
TOL = {np.float32: 2e-6, np.float64: 1e-12}


def cols(*items, memberships=None):
    """items: (shape, dims, position, rotation)"""
    sh, dm, ps, rt = zip(*items)
    return api.QueryColliders(shape=np.array(sh, np.uint8), dims=np.array([np.broadcast_to(np.asarray(d, float), 3) for d in dm]),
                              position=np.array(ps, float), rotation=np.array(rt, float),
                              memberships=None if memberships is None else np.array(memberships, np.uint32))


def rays(o, d, maxd=100.0, solid=None):
    o, d = np.atleast_2d(np.asarray(o, float)), np.atleast_2d(np.asarray(d, float))
    return api.Rays(origin=o, direction=d, max_distance=np.full(len(o), maxd), solid=None if solid is None else np.asarray(solid, np.uint8))


def ray1(scalar, c, o, d, solid=True, maxd=100.0):
    r = fixture.query_cast_ray(scalar, c, rays(o, d, maxd, [solid]), capsules=True)
    return int(r["collider"][0]), float(r["distance"][0]), r["normal"][0].astype(float)


def cast1(scalar, c, item, d, maxd=100.0, flags=0):
    sh, dm, ps, rt = item
    q = api.ShapeQueries(shape=np.array([sh], np.uint8), dims=np.broadcast_to(np.asarray(dm, float), 3)[None].copy(), position=np.array([ps], float),
                         rotation=np.array([rt], float), direction=np.array([d], float), max_distance=np.array([maxd]),
                         flags=np.array([flags], np.uint32))
    r = fixture.query_cast_shape(scalar, c, q, capsules=True)
    return int(r["collider"][0]), float(r["distance"][0]), {k: r[k][0].astype(np.float64) for k in ("point1", "point2", "normal1", "normal2")}


def unit_quat(rng):
    q = rng.normal(size=4)
    return q / np.linalg.norm(q)


def capsule_ends(dims, pos, rot):
    return cr.capsule_segment(pos, rot, dims[1])


# ---- ray casts ------------------------------------------------------------------------------------------------------------------------------
def test_ray_capsule_soup_matches_the_restatement():
    rng = np.random.default_rng(31)
    hits = checked = 0
    for _ in range(20):
        dims = np.array([rng.uniform(0.1, 1.0), rng.uniform(0.0, 1.5), 0.0])
        pos, rot = rng.uniform(-3, 3, 3), unit_quat(rng)
        c = cols((CAP, dims, pos, rot))
        p0, p1 = capsule_ends(dims, pos, rot)
        for _ in range(25):
            o = pos + rng.normal(size=3) * 3
            d = (pos + rng.uniform(-1.5, 1.5, 3)) - o
            d /= np.linalg.norm(d)
            solid = bool(rng.random() < 0.5)
            got_c, got_t, got_n = ray1(np.float64, c, o, d, solid)
            want = cqr.ray_capsule(o, d, p0, p1, dims[0], solid)
            # skip rays that graze the surface within the restatement's own resolution
            dmin = min(cqr.segment_distance(o + d * t, p0, p1) for t in np.linspace(0, 20, 2001))
            if abs(dmin - dims[0]) < 1e-6 or abs(cqr.segment_distance(o, p0, p1) - dims[0]) < 1e-9:
                continue
            checked += 1
            assert (got_c == 0) == (want is not None), (o, d, solid)
            if want is None:
                continue
            hits += 1
            assert abs(got_t - want[0]) <= 1e-9 * max(1.0, want[0])
            assert np.allclose(got_n, want[1], atol=1e-7)
            if got_t > 0:
                # the hit lies on the surface: its distance to the segment at 50 digits is the radius to rounding
                assert abs(cqr.mp_point_segment_distance(o + d * got_t, p0, p1) - dims[0]) <= 1e-12 * max(1.0, got_t)
    assert checked > 400 and hits > 100


@pytest.mark.parametrize("scalar", SCALARS, ids=["f32", "f64"])
def test_grazing_rays(scalar):
    c = cols((CAP, [0.5, 1.0, 0.0], [0.0, 0.0, 0.0], IDENT))
    tol = TOL[scalar] * 4
    # tangent to the cylinder (the discriminant is exactly 0), and one ulp outside it
    col, t, n = ray1(scalar, c, [-5.0, 0.3, 0.5], [1.0, 0, 0])
    assert col == 0 and abs(t - 5.0) <= tol * 5 and np.allclose(n, [0, 0, 1], atol=1e-3)
    if scalar == np.float64:
        assert ray1(scalar, c, [-5.0, 0.3, float(np.nextafter(0.5, 1.0))], [1.0, 0, 0])[0] == -1
    # through the cylinder / cap seam (y = half length)
    col, t, n = ray1(scalar, c, [-5.0, 1.0, 0.0], [1.0, 0, 0])
    assert col == 0 and abs(t - 4.5) <= tol * 5 and np.allclose(n, [-1, 0, 0], atol=tol)
    # end-on along the axis: the cap's pole
    col, t, n = ray1(scalar, c, [0.0, 5.0, 0.0], [0.0, -1.0, 0])
    assert col == 0 and abs(t - 3.5) <= tol * 5 and np.allclose(n, [0, 1, 0], atol=tol)
    # from inside: solid -> t = 0 with a zero normal; hollow -> the exit
    assert ray1(scalar, c, [0.1, 0.2, 0.0], [1.0, 0, 0], solid=True)[:2] == (0, 0.0)
    col, t, n = ray1(scalar, c, [0.1, 0.2, 0.0], [1.0, 0, 0], solid=False)
    assert col == 0 and abs(t - 0.4) <= tol and np.allclose(n, [1, 0, 0], atol=tol)
    col, t, n = ray1(scalar, c, [0.0, 0.0, 0.0], [0.0, 1.0, 0], solid=False)
    assert col == 0 and abs(t - 1.5) <= tol and np.allclose(n, [0, 1, 0], atol=tol)
    # radius 0: a closed bare segment, hit where the ray crosses it
    seg = cols((CAP, [0.0, 1.0, 0.0], [0.0, 0.0, 0.0], IDENT))
    col, t, n = ray1(scalar, seg, [-2.0, 0.5, 0.0], [1.0, 0, 0])
    assert col == 0 and abs(t - 2.0) <= tol


def _ulps(a, b):
    return abs(a - b) / np.spacing(max(abs(a), abs(b), 1.0))


def test_zero_half_length_is_the_sphere_and_a_point_capsule_is_the_ray():
    """half_length = 0 gives the sphere's ray casts, and a capsule of radius 0 and half length 0 cast as a shape gives the ray cast, within 64
    ulps of max(1, t) (1e-9 relative for rays grazing a sphere's rim, where the sphere's own b² - a c discriminant cancels): the closed forms
    differ (Lagrange discriminants, the rounded-box edges) but describe the same set."""
    rng = np.random.default_rng(32)
    n = 60
    r = rng.uniform(0.2, 1.0, n)
    pos, rot = rng.uniform(-6, 6, (n, 3)), np.array([unit_quat(rng) for _ in range(n)])
    as_caps = api.QueryColliders(shape=np.full(n, CAP, np.uint8), dims=np.stack([r, np.zeros(n), np.zeros(n)], 1), position=pos, rotation=rot)
    as_balls = api.QueryColliders(shape=np.full(n, SPH, np.uint8), dims=np.stack([r, np.zeros(n), np.zeros(n)], 1), position=pos, rotation=rot)
    m = 300
    o, d = rng.uniform(-8, 8, (m, 3)), rng.normal(size=(m, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    a = fixture.query_cast_ray(np.float64, as_caps, rays(o, d, 30.0), capsules=True)
    b = fixture.query_cast_ray(np.float64, as_balls, rays(o, d, 30.0))
    assert (a["collider"] >= 0).sum() > 30
    for i in range(m):
        if a["collider"][i] != b["collider"][i]:
            # only a grazing ray may tip over: it passes within rounding of the surface
            c = max(a["collider"][i], b["collider"][i])
            x = o[i] - pos[c]
            assert abs(np.linalg.norm(np.cross(x, d[i])) - r[c]) < 1e-9
            continue
        if a["collider"][i] < 0:
            continue
        c = a["collider"][i]
        # well inside the silhouette (closest approach <= 0.9 r) the two forms agree to 64 ulps; nearer the rim the sphere's b² - a c form
        # cancels, and the bound is 1e-9 relative
        if np.linalg.norm(np.cross(o[i] - pos[c], d[i])) <= 0.9 * r[c]:
            assert _ulps(a["distance"][i], b["distance"][i]) <= 64
        else:
            assert abs(a["distance"][i] - b["distance"][i]) <= 1e-9 * max(1.0, b["distance"][i])
    # a point capsule cast against a mixed scene is the ray cast
    k = 80
    mixed = api.QueryColliders(shape=rng.integers(0, 3, k).astype(np.uint8), dims=np.stack([rng.uniform(0.2, 1.0, k), rng.uniform(0.0, 1.2, k),
                               rng.uniform(0.2, 1.0, k)], 1), position=rng.uniform(-6, 6, (k, 3)), rotation=np.array([unit_quat(rng) for _ in range(k)]))
    q = api.ShapeQueries(shape=np.full(m, CAP, np.uint8), dims=np.zeros((m, 3)), position=o, rotation=np.tile(IDENT, (m, 1)), direction=d,
                         max_distance=np.full(m, 30.0))
    sc = fixture.query_cast_shape(np.float64, mixed, q, capsules=True)
    rc = fixture.query_cast_ray(np.float64, mixed, rays(o, d, 30.0), capsules=True)
    agree = 0
    for i in range(m):
        if sc["collider"][i] == rc["collider"][i]:
            agree += 1
            if rc["collider"][i] >= 0:
                assert _ulps(sc["distance"][i], rc["distance"][i]) <= 64
    assert agree >= m - 2 and (rc["collider"] >= 0).sum() > 50


# ---- shape casts: the five capsule kinds against the bisected overlap predicate ---------------------------------------------------------
KINDS = [(SPH, CAP), (CAP, SPH), (CAP, CAP), (CAP, CUB), (CUB, CAP)]
KIND_IDS = ["sphere_capsule", "capsule_sphere", "capsule_capsule", "capsule_cuboid", "cuboid_capsule"]


def random_dims(rng, s):
    if s == CUB:
        return rng.uniform(0.3, 1.2, 3)
    if s == SPH:
        return np.array([rng.uniform(0.2, 1.0), 0, 0])
    return np.array([rng.uniform(0.15, 0.8), rng.uniform(0.0, 1.2), 0])


def random_pair(rng, kind):
    sa, sb = kind
    ha, hb = random_dims(rng, sa), random_dims(rng, sb)
    qa, qb = unit_quat(rng), unit_quat(rng)
    if rng.random() < 0.25:                                      # parallel axes and axis-aligned boxes: the continuum contacts
        qa = qb = np.array(IDENT)
    cb = rng.uniform(-1, 1, 3)
    ca = cb + rng.normal(size=3) * 4 + np.array([0, 5.0, 0])
    d = (cb + rng.uniform(-1.2, 1.2, 3)) - ca
    d /= np.linalg.norm(d)
    return (sa, ha, ca, qa), (sb, hb, cb, qb), d


def touching(a, b, t, d):
    (sa, ha, ca, qa), (sb, hb, cb, qb) = a, b
    if sa != CAP and sb != CAP:
        raise AssertionError("a capsule kind")
    return cr.capsule_depth(sa, ha, ca + d * t, qa, sb, hb, cb, qb)[0] <= 0.0


def cast_pair(a, b, d, maxd=50.0):
    (sa, ha, ca, qa), (sb, hb, cb, qb) = a, b
    return cast1(np.float64, cols((sb, hb, cb, qb)), (sa, ha, ca, qa), d, maxd)


@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
def test_toi_agrees_with_bisected_overlap(kind):
    rng = np.random.default_rng(300 + 10 * kind[0] + kind[1])
    hits = misses = 0
    for _ in range(120):
        a, b, d = random_pair(rng, kind)
        c, t, _ = cast_pair(a, b, d)
        if c < 0:
            misses += 1
            assert not any(touching(a, b, x, d) for x in np.linspace(0, 50, 401))
            continue
        hits += 1
        if touching(a, b, 0.0, d):
            assert t == 0
            continue
        assert t > 0
        assert touching(a, b, t * (1 + 1e-9), d), "not touching just after the TOI"
        assert not touching(a, b, t * (1 - 1e-9), d), "already touching just before the TOI"
        lo, hi = 0.0, t * (1 + 1e-6)
        for _ in range(60):
            mid = 0.5 * (lo + hi)
            lo, hi = (lo, mid) if touching(a, b, mid, d) else (mid, hi)
        assert abs(hi - t) <= 1e-9 * t + 1e-15
    assert hits > 70 and misses > 0


def shape_dist(s, p):
    sh, he, c, q = s
    if sh == CAP:
        p0, p1 = capsule_ends(he, c, q)
        return max(cqr.segment_distance(p, p0, p1) - he[0], 0.0)
    if sh == SPH:
        return max(np.linalg.norm(p - c) - he[0], 0.0)
    return cr.point_box(p, np.asarray(c, float), cr.quat_matrix(q), np.asarray(he, float))[0]


@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
def test_witness_properties_of_random_hits(kind):
    rng = np.random.default_rng(400 + 10 * kind[0] + kind[1])
    checked = 0
    for _ in range(120):
        a, b, d = random_pair(rng, kind)
        c, t, h = cast_pair(a, b, d)
        if c < 0 or t == 0:
            continue
        checked += 1
        A = (a[0], a[1], a[2] + d * t, a[3])
        tol = 1e-9 * max(np.max(a[1]), np.max(b[1]), 1.0)
        assert cr.surface_distance(b[0], b[1], b[2], b[3], h["point1"]) <= tol
        assert cr.surface_distance(A[0], A[1], A[2], A[3], h["point2"]) <= tol
        assert np.linalg.norm(h["point1"] - h["point2"]) <= tol
        for n, s, p in ((h["normal1"], b, h["point1"]), (h["normal2"], A, h["point2"])):
            assert abs(np.linalg.norm(n) - 1) <= 1e-12
            assert abs(shape_dist(s, p + 1e-4 * n) - 1e-4) <= 1e-8
        assert np.allclose(h["normal2"], -h["normal1"])
        assert d @ h["normal1"] <= 1e-12
    assert checked > 70


@pytest.mark.parametrize("scalar", SCALARS, ids=["f32", "f64"])
def test_origin_penetration_and_flags(scalar):
    c = cols((CUB, 1.0, [0.0, 0, 0], IDENT), (CAP, [0.5, 1.0, 0], [10.0, 0, 0], IDENT))
    lying = [0.0, 0.0, math.sin(math.pi / 4), math.cos(math.pi / 4)]         # axis along -x
    for item, want in (((CAP, [0.3, 0.5, 0], [0.0, 1.2, 0.0], lying), 0), ((SPH, [0.5, 0, 0], [10.0, 1.8, 0.0], IDENT), 1),
                       ((CAP, [0.3, 0.5, 0], [10.0, 2.0, 0.0], IDENT), 1)):
        for d, away in (([0.0, -1.0, 0.0], False), ([0.0, 1.0, 0.0], True)):
            col, t, h = cast1(scalar, c, item, d)
            assert (col, t) == (want, 0.0)
            assert np.allclose(h["normal1"], [0, 1, 0], atol=TOL[scalar] * 10) and np.allclose(h["normal2"], [0, -1, 0], atol=TOL[scalar] * 10)
            assert cast1(scalar, c, item, d, flags=api.CAST_IGNORE_ORIGIN_PENETRATION)[0] == (-1 if away else want)
            col, t, h = cast1(scalar, c, item, d, flags=api.CAST_NO_CONTACT_ON_PENETRATION)
            assert (col, t) == (want, 0.0) and all(not v.any() for v in h.values())


def test_capsule_lying_on_a_face_reports_the_lower_end():
    """the continuum witness rule: a horizontal capsule landing flat on a box face reports the clipped segment's end at the lower parameter"""
    lying = [0.0, 0.0, math.sin(math.pi / 4), math.cos(math.pi / 4)]         # local +y along world -x
    c, t, h = cast1(np.float64, cols((CUB, 1.0, [0.0, 0, 0], IDENT)), (CAP, [0.25, 0.5, 0], [0.2, 4.0, 0.0], lying), [0.0, -1.0, 0])
    assert c == 0 and t == pytest.approx(2.75, abs=1e-12)
    assert np.allclose(h["normal1"], [0, 1, 0], atol=1e-12)
    assert np.allclose(h["point1"], [0.7, 1.0, 0.0], atol=1e-12) and np.allclose(h["point2"], [0.7, 1.0, 0.0], atol=1e-12)


# ---- projection, containment, intersections ----------------------------------------------------------------------------------------------
def test_projection_and_containment_match_the_restatement():
    rng = np.random.default_rng(33)
    for _ in range(30):
        dims = np.array([rng.uniform(0.1, 1.0), rng.uniform(0.0, 1.5), 0.0])
        pos, rot = rng.uniform(-3, 3, 3), unit_quat(rng)
        c = cols((CAP, dims, pos, rot))
        p0, p1 = capsule_ends(dims, pos, rot)
        x_axis = cr.quat_rotate(rot, [1.0, 0, 0])
        m = 40
        pts = pos + rng.normal(size=(m, 3)) * 1.5
        pts[0] = pos                                                           # the centre, on the axis: projected along local +x
        for solid in (True, False):
            r = fixture.query_project_point(np.float64, c, api.Points(point=pts, solid=np.full(m, solid, np.uint8)), capsules=True)
            np.testing.assert_allclose(r["point"][0], pos if solid else pos + x_axis * dims[0], atol=1e-12 * (1 + np.abs(pos).max()))
            for i in range(1, m):
                want, inside = cqr.project_capsule(pts[i], p0, p1, dims[0], x_axis, solid)
                sd = cqr.segment_distance(pts[i], p0, p1)
                if abs(sd - dims[0]) < 1e-9 or sd < 1e-6:                     # on the surface, or so near the axis the direction is rounding
                    continue
                assert bool(r["is_inside"][i]) == inside
                np.testing.assert_allclose(r["point"][i], want, atol=1e-12 * (1 + np.abs(pos).max()))
        inside = fixture.query_point_intersections(np.float64, c, api.Points(point=pts), capsules=True)
        for i in range(m):
            dd = cqr.segment_distance(pts[i], p0, p1) - dims[0]
            if abs(dd) > 1e-9:
                assert (inside["offsets"][i + 1] > inside["offsets"][i]) == (dd < 0)


def _isect(c, item):
    sh, dm, ps, rt = item
    q = api.ShapeQueries(shape=np.array([sh], np.uint8), dims=np.broadcast_to(np.asarray(dm, float), 3)[None].copy(), position=np.array([ps], float),
                         rotation=np.array([rt], float))
    return fixture.query_shape_intersections(np.float64, c, q, capsules=True)["collider"].tolist()


def test_touching_intersects_and_a_one_ulp_gap_does_not():
    c = cols((CAP, [0.5, 1.0, 0.0], [0.0, 0, 0], IDENT))
    up = float(np.nextafter(1.0, 2.0))
    for item, gap in (((SPH, [0.5, 0, 0], [1.0, 0.3, 0.0], IDENT), ((SPH, [0.5, 0, 0], [up, 0.3, 0.0], IDENT))),
                      ((CAP, [0.5, 0.7, 0], [1.0, 0.4, 0.0], IDENT), ((CAP, [0.5, 0.7, 0], [up, 0.4, 0.0], IDENT))),
                      ((CUB, 0.5, [1.0, 0.2, 0.0], IDENT), ((CUB, 0.5, [up, 0.2, 0.0], IDENT)))):
        assert _isect(c, item) == [0], item
        assert _isect(c, gap) == [], gap
    # the other way round: the capsule is the query shape
    assert _isect(cols((CUB, 0.5, [1.0, 0.2, 0.0], IDENT)), (CAP, [0.5, 1.0, 0.0], [0.0, 0, 0], IDENT)) == [0]
    assert _isect(cols((CUB, 0.5, [up, 0.2, 0.0], IDENT)), (CAP, [0.5, 1.0, 0.0], [0.0, 0, 0], IDENT)) == []
    # point containment on the cylinder and on the cap
    for p, gap in (([0.5, 0.3, 0.0], [float(np.nextafter(0.5, 1.0)), 0.3, 0.0]), ([0.0, 1.5, 0.0], [0.0, float(np.nextafter(1.5, 2.0)), 0.0])):
        r = fixture.query_point_intersections(np.float64, c, api.Points(point=np.array([p, gap])), capsules=True)
        assert r["offsets"].tolist() == [0, 1, 1]


def test_shape_intersections_match_the_restatement():
    rng = np.random.default_rng(34)
    n = 60
    shape = rng.integers(0, 3, n).astype(np.uint8)
    dims = np.stack([random_dims(rng, s) for s in shape])
    c = api.QueryColliders(shape=shape, dims=dims, position=rng.uniform(-4, 4, (n, 3)), rotation=np.array([unit_quat(rng) for _ in range(n)]))
    m = 40
    qs = rng.integers(0, 3, m).astype(np.uint8)
    qs[: m // 2] = CAP
    qd = np.stack([random_dims(rng, s) for s in qs])
    qp, qr = rng.uniform(-4, 4, (m, 3)), np.array([unit_quat(rng) for _ in range(m)])
    got = fixture.query_shape_intersections(np.float64, c, api.ShapeQueries(shape=qs, dims=qd, position=qp, rotation=qr), capsules=True)
    seen = 0
    for i in range(m):
        lst = set(got["collider"][got["offsets"][i]:got["offsets"][i + 1]].tolist())
        for j in range(n):
            if qs[i] != CAP and shape[j] != CAP:
                continue
            dist = cr.capsule_depth(qs[i], qd[i], qp[i], qr[i], shape[j], dims[j], c.position[j], c.rotation[j])[0]
            if 0 < dist < 1e-9:
                continue
            seen += 1
            assert (j in lst) == (dist <= 0), (i, j)
    assert seen > 500


# ---- move and slide with capsule characters --------------------------------------------------------------------------------------------
def box(pos, half, rot=IDENT):
    return (CUB, np.asarray(half, float), np.asarray(pos, float), np.asarray(rot, float))


def capsule_character(pos, vel, radius=0.5, half_length=0.5, **kw):
    return api.MoveBatch(shape=np.array([CAP], np.uint8), dims=np.array([[radius, half_length, 0.0]]), position=np.array([pos], float),
                         rotation=np.array([IDENT]), velocity=np.array([vel], float), **kw)


def move(scalar, c, cfg, batch):
    return fixture.move_and_slide(scalar, c, cfg, batch, capsules=True)


def mtol(scalar, lu=1.0):
    return (2e-4 if scalar == np.float32 else 1e-6) * max(lu, 1.0) * 10


MCASES = [(lu, s) for lu in (1.0, 10.0) for s in SCALARS]
mids = lambda c: f"lu{int(c[0])}-{np.dtype(c[1]).name}"


@pytest.mark.parametrize("case", MCASES, ids=mids)
def test_capsule_head_on_wall_stops_at_the_pull_back_distance(case):
    lu, sc = case
    r = move(sc, cols(box((2.0, 0, 0), (0.5, 5, 5))), api.MoveConfig(length_unit=lu), capsule_character((0, 0, 0), (120, 0, 0)))
    skin = 0.01 * lu
    np.testing.assert_allclose(r["position"][0], [1.0 - skin, 0, 0], atol=mtol(sc))
    np.testing.assert_allclose(r["velocity"][0], [0, 0, 0], atol=mtol(sc))
    assert r["hit_collider"][0, 0] == 0
    np.testing.assert_allclose(r["hit_toi"][0, 0], 1.0, atol=mtol(sc))
    np.testing.assert_allclose(r["hit_normal"][0, 0], [-1, 0, 0], atol=mtol(sc))


def _rotz(deg):
    a = math.radians(deg) / 2
    return (0.0, 0.0, math.sin(a), math.cos(a))


@pytest.mark.parametrize("case", MCASES, ids=mids)
def test_capsule_ramp_projects_up_the_ramp_with_v_cos_theta(case):
    """the -x face of a big box tilted back by 30 degrees about z: the upright capsule's support along the face normal n is r + hl |n_y|"""
    lu, sc = case
    theta = 30.0
    q = _rotz(-(90 - theta))
    R = cr.quat_matrix(q)
    ax, n = R[:, 0], -R[:, 0]
    c = cols(box(np.array([3.0, 0, 0]) + 50.0 * ax, (50, 50, 50), q))
    v = np.array([240.0, 0, 0])
    r = move(sc, c, api.MoveConfig(length_unit=lu), capsule_character((0, 0, 0), v))
    support = 0.5 + 0.5 * abs(n[1])
    skin = 0.01 * lu
    t1 = (-3.0 * n[0] - support) / -n[0]
    safe = t1 - skin / -n[0]
    time_left = (1 / 60) * (1 - safe / 4.0)
    vp = v - (v @ n) * n
    got = r["velocity"][0].astype(float)
    np.testing.assert_allclose(np.linalg.norm(got), 240 * math.cos(math.radians(theta)), rtol=1e-5)
    np.testing.assert_allclose(got / np.linalg.norm(got), [math.cos(math.radians(theta)), math.sin(math.radians(theta)), 0], atol=1e-5)
    np.testing.assert_allclose(r["position"][0], np.array([safe, 0, 0]) + time_left * vp, atol=mtol(sc, lu))


@pytest.mark.parametrize("case", MCASES, ids=mids)
def test_capsule_floor_wall_corner_projects_onto_the_edge(case):
    lu, sc = case
    skin = 0.01 * lu
    c = cols(box((0, -50.0, 0), (50, 50, 50)), box((51.0, 0, 0), (50, 50, 50)))
    start = np.array([1.0 - 0.5 - skin, 1.0 + skin, 0.0])                  # radius 0.5 from the wall, half length + radius above the floor
    r = move(sc, c, api.MoveConfig(length_unit=lu), capsule_character(start, (60, -60, 60)))
    np.testing.assert_allclose(r["velocity"][0], [0, 0, 60], atol=mtol(sc) * 60)
    np.testing.assert_allclose(r["position"][0], start + [0, 0, 1.0], atol=mtol(sc, lu))


@pytest.mark.parametrize("case", MCASES, ids=mids)
def test_capsule_embedded_start_is_pushed_out_by_depth_plus_skin(case):
    lu, sc = case
    d = 0.02 * lu
    r = move(sc, cols(box((0, -50.0, 0), (50, 50, 50))), api.MoveConfig(length_unit=lu), capsule_character((0, 1.0 - d, 0), (0, 0, 0)))
    np.testing.assert_allclose(r["position"][0], [0, 1.0 + 0.01 * lu, 0], atol=mtol(sc, lu))


def _capsule_aabb(shape, he, p, q):
    if shape != CAP:
        return _plain_aabb(shape, he, p, q)
    p0, p1 = cr.capsule_segment(p, np.asarray(q, float) / np.linalg.norm(q), he[1])
    return np.minimum(p0, p1) - he[0], np.maximum(p0, p1) + he[0]


_plain_aabb = mref._aabb


def capsule_scene(rng, n, extent):
    c, ignored = random_colliders(rng, n, extent)
    caps = rng.random(n) < 0.3
    c.shape[caps] = CAP
    c.dims[caps, 0] = rng.uniform(0.15, 0.6, caps.sum())
    return c, ignored


@pytest.mark.parametrize("cfg", [api.MoveConfig(), api.MoveConfig(move_and_slide_iterations=8, max_planes=3, length_unit=2.0),
                                 api.MoveConfig(depenetration_iterations=0)], ids=["default", "8-iterations", "no-depenetration"])
def test_capsule_loop_matches_the_restatement(cfg, monkeypatch):
    """tests/move_reference.py's loop with the capsule-enabled fixture for its casts and a capsule-aware candidate box"""
    shim = types.SimpleNamespace(**{k: getattr(fixture, k) for k in dir(fixture) if not k.startswith("__")})
    shim.query_cast_shape = lambda scalar, c, q: fixture.query_cast_shape(scalar, c, q, capsules=True)
    monkeypatch.setattr(mref, "fixture", shim)
    monkeypatch.setattr(mref, "_aabb", _capsule_aabb)
    rng = np.random.default_rng(12)
    c, ignored = capsule_scene(rng, 60, 3.0)
    cfg.ignored = ignored
    batch = random_characters(rng, 150, 3.0, 60)
    batch.shape[np.arange(150) % 3 != 2] = CAP                                # two thirds capsules, the rest cuboids and spheres
    got = fixture.move_and_slide(np.float64, c, cfg, batch, capsules=True)
    scene = mref.Scene(c, ignored)
    hits = 0
    for i in range(batch.count):
        p, v, h = mref.move_one(scene, cfg, int(batch.shape[i]), batch.dims[i], batch.position[i], batch.rotation[i], batch.velocity[i],
                                int(batch.mask[i]), batch.exclude[i], [] if batch.planes[i] is None else batch.planes[i])
        np.testing.assert_allclose(got["position"][i], p, atol=1e-9, err_msg=f"character {i}")
        np.testing.assert_allclose(got["velocity"][i], v, atol=1e-8, err_msg=f"character {i}")
        want_c = np.full(cfg.move_and_slide_iterations, -1)
        for it, col, safe, toi in h:
            want_c[it] = col
            np.testing.assert_allclose([got["hit_distance"][i, it], got["hit_toi"][i, it]], [safe, toi], atol=1e-9)
        np.testing.assert_array_equal(got["hit_collider"][i], want_c)
        hits += len(h)
    assert hits > 40


# ---- refusals ---------------------------------------------------------------------------------------------------------------------------------
def test_refused_inputs():
    good = cols((CAP, [0.5, 1.0, 0.0], [0.0, 0, 0], IDENT))
    r = rays([-5.0, 0, 0], [1.0, 0, 0])
    assert fixture.query_cast_ray(np.float64, good, r, capsules=True)["collider"].tolist() == [0]
    with pytest.raises(api.AvianError, match="unknown shape"):
        fixture.query_cast_ray(np.float64, good, r)                           # without the capsule bit a capsule is still refused
    for dims in ([-0.5, 1.0, 0.0], [0.5, -1.0, 0.0]):
        for scalar in SCALARS:
            with pytest.raises(api.AvianError, match="negative"):
                fixture.query_cast_ray(scalar, cols((CAP, dims, [0.0, 0, 0], IDENT)), r, capsules=True)
    # dims[2] is not read: a negative third entry is accepted
    assert fixture.query_cast_ray(np.float64, cols((CAP, [0.5, 1.0, -3.0], [0.0, 0, 0], IDENT)), r, capsules=True)["collider"].tolist() == [0]
    with pytest.raises(api.AvianError, match="unknown shape"):
        fixture.query_cast_ray(np.float64, cols((3, [0.5, 1.0, 0.0], [0.0, 0, 0], IDENT)), r, capsules=True)
    with pytest.raises(api.AvianError, match="negative"):
        cast1(np.float64, good, (CAP, [0.5, -0.1, 0], [0.0, 5, 0], IDENT), [0, -1.0, 0])
    with pytest.raises(api.AvianError, match="unknown shape"):
        cast1(np.float64, good, (3, [0.5, 0.1, 0], [0.0, 5, 0], IDENT), [0, -1.0, 0])
    cfg = api.MoveConfig()
    with pytest.raises(api.AvianError, match="negative"):
        move(np.float64, good, cfg, capsule_character((5.0, 0, 0), (1, 0, 0), half_length=-0.5))
    bad = capsule_character((5.0, 0, 0), (1, 0, 0))
    bad.shape = np.array([3], np.uint8)
    with pytest.raises(api.AvianError, match="unknown shape"):
        move(np.float64, good, cfg, bad)
    with pytest.raises(api.AvianError, match="unknown shape"):
        fixture.move_and_slide(np.float64, good, cfg, capsule_character((5.0, 0, 0), (1, 0, 0)))
