"""Convex hull colliders in the host fixture (csrc/hull_math.hpp through avh_raw_manifolds, the AABB update, the table checks, scenes' mass
properties) against the independent float64 restatement of tests/hull_reference.py: the contact contract of DESIGN.md §7 on seeded soups of
hull-hull, hull-cuboid, hull-sphere and hull-capsule pairs in both orders, symmetry and invariance, a cuboid written as a hull against the
cuboid path, the refusals, and CPU worlds with the oracle solver."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
from avian_b200 import api, fixture, plugins, scenes  # noqa: E402
import capsule_reference as cref  # noqa: E402
import hull_reference as ref  # noqa: E402
import oracle_lib  # noqa: E402

BOX, SPH, CAP, HULL = fixture.SHAPE_CUBOID, fixture.SHAPE_SPHERE, fixture.SHAPE_CAPSULE, fixture.SHAPE_CONVEX_HULL
DT, MAX_DIST = 1.0 / 60.0, 0.5
SCALARS = [np.float32, np.float64]


def hull_set(seed=5, random_hulls=6):
    """a table of seeded random hulls, the regular solids, the 32-sided prism and the unit-half-extent cube written as a hull (the last one)"""
    rng = np.random.default_rng(seed)
    polys = [scenes.convex_hull_of(rng.normal(size=(int(rng.integers(8, 20)), 3)) * rng.uniform(0.3, 0.8)) for _ in range(random_hulls)]
    polys += scenes.regular_solids(0.6)
    cube = np.array([[(1 if m & 1 else -1), (1 if m & 2 else -1), (1 if m & 4 else -1)] for m in range(8)], float) * 0.5
    polys.append((cube, ref.CUBE_FACES))
    return api.ConvexHulls.from_polyhedra(polys)


HULLS = hull_set()
CUBE = HULLS.count - 1


def shape_poly(scalar, hulls, shape, dims, pos, rot):
    if shape == HULL:
        v, f = hulls.polyhedron(int(dims[0]))
        return ref.posed(np.asarray(v, dtype=scalar).astype(np.float64), pos, rot), [list(x) for x in f]
    return ref.box_poly(dims, pos, rot)


def exact(scalar, hulls, p):
    """(distance, depth) of a pair from the reference: depth > 0 overlapping"""
    sa, da, pa, qa, sb, db, pb, qb = p
    if sa not in (HULL, BOX):
        sa, da, pa, qa, sb, db, pb, qb = sb, db, pb, qb, sa, da, pa, qa
    V, F = shape_poly(scalar, hulls, sa, da, pa, qa)
    if sb in (HULL, BOX):
        W, G = shape_poly(scalar, hulls, sb, db, pb, qb)
        sep, overlap = ref.sat(V, F, W, G)
        return (ref.distance(V, F, W, G), 0.0) if sep > 0 else (0.0, overlap)
    if sb == SPH:
        d = ref.point_distance(np.asarray(pb), V, F) - db[0]
        return (d, 0.0) if d > 0 else (0.0, -d)
    p0, p1 = cref.capsule_segment(pb, qb, db[1])
    d = ref.segment_distance(p0, p1, V, F)
    if d > 0:
        return (d - db[0], 0.0) if d > db[0] else (0.0, db[0] - d)
    return 0.0, ref.segment_depth(p0, p1, db[0], V, F)


def surface_distance(scalar, hulls, shape, dims, pos, rot, x):
    if shape in (HULL, BOX):
        V, F = shape_poly(scalar, hulls, shape, dims, pos, rot)
        return abs(ref.point_distance(x, V, F))
    if shape == SPH:
        return abs(np.linalg.norm(x - pos) - dims[0])
    p0, p1 = cref.capsule_segment(pos, rot, dims[1])
    return abs(np.linalg.norm(x - cref.point_segment(x, p0, p1)) - dims[0])


def collide(scalar, pairs, hulls=HULLS, moving=True):
    n = len(pairs)
    cols = {"shape": np.array([s for p in pairs for s in (p[0], p[4])], dtype=np.uint8)}
    for key, ia, ib in (("dims", 1, 5), ("position", 2, 6), ("rotation", 3, 7)):
        cols[key] = np.ascontiguousarray([np.asarray(v, float) for p in pairs for v in (p[ia], p[ib])], dtype=scalar)
    c1, c2 = np.arange(0, 2 * n, 2, dtype=np.uint32), np.arange(1, 2 * n, 2, dtype=np.uint32)
    lv = np.zeros((2 * n, 3), dtype=scalar)
    if moving:
        lv[1::2, 0] = MAX_DIST / DT
    return fixture.raw_manifolds(scalar, DT, 1e-3, (c1, c2, c1, c2), cols, lv, np.zeros((2 * n, 3), dtype=scalar), f64_anchors=True, hulls=hulls)


def as_f64(scalar, p):
    return tuple(np.asarray(v, dtype=scalar).astype(np.float64) if not np.isscalar(v) else v for v in p)


def scale_of(p):
    return 1.0 + np.abs(np.asarray(p[2])).max() + np.abs(np.asarray(p[6])).max() + 4.0


def check_contract(scalar, pairs, out, hulls=HULLS):
    """DESIGN.md §7's contract (items 1-5, 8) on every pair; returns the classes met"""
    eps = np.finfo(scalar).eps
    met = set()
    for k, p in enumerate(pairs):
        p = as_f64(scalar, p)
        tol = 64 * eps * scale_of(p)
        D, depth = exact(scalar, hulls, p)
        n = int(out["point_count"][k])
        nrm = out["normal"][k].astype(np.float64)
        a = np.asarray(p[2]) + out["anchor1_f64"][k, :n]
        b = np.asarray(p[6]) + out["anchor2_f64"][k, :n]
        pen = out["penetration"][k, :n].astype(np.float64)
        assert n <= 4, f"pair {k}: {n} points"
        if depth == 0.0 and D > MAX_DIST:
            assert n == 0, f"pair {k}: {n} points at distance {D} beyond the margin"
            met.add("beyond")
            continue
        if depth == 0.0 and D > MAX_DIST - 1e-6:
            continue
        assert n >= 1, f"pair {k}: no point at distance {D}, depth {depth}"
        assert abs(np.linalg.norm(nrm) - 1.0) <= 64 * eps, f"pair {k}: |n| = {np.linalg.norm(nrm)}"
        for i in range(n):
            assert surface_distance(scalar, hulls, p[0], p[1], p[2], p[3], a[i]) <= tol, f"pair {k} point {i}: a is off A's surface"
            assert surface_distance(scalar, hulls, p[4], p[5], p[6], p[7], b[i]) <= tol, f"pair {k} point {i}: b is off B's surface"
            assert np.linalg.norm(np.cross(b[i] - a[i], nrm)) <= tol, f"pair {k} point {i}: b - a is not along n"
            assert abs(pen[i] - (a[i] - b[i]) @ nrm) <= tol, f"pair {k} point {i}: penetration"
        if depth > 0.0:
            assert abs(pen.max() - depth) <= 1e-4 + tol, f"pair {k}: deepest {pen.max()} vs SAT overlap {depth}"
            met.add("deep" if depth > 0.1 else "shallow")
        else:
            slack = 1e-4 + tol
            assert -pen.max() <= D + slack, f"pair {k}: smallest gap {-pen.max()} vs distance {D}"
            met.add("separated")
    return met


def _rot(rng):
    q = rng.normal(size=4)
    return q / np.linalg.norm(q)


def soup(seed, shape_b, count=120, hulls=HULLS):
    """a hull (A) against shape_b at random orientations and offsets from deep to beyond the margin; a third of the pairs share A's
    orientation (parallel faces), and half the pairs are written B first"""
    rng = np.random.default_rng(seed)
    pairs = []
    for i in range(count):
        ia = int(rng.integers(0, hulls.count))
        ra = float(np.abs(hulls.polyhedron(ia)[0]).max()) * np.sqrt(3)
        if shape_b == HULL:
            db = np.array([float(rng.integers(0, hulls.count)), 0.0, 0.0])
            rb = float(np.abs(hulls.polyhedron(int(db[0]))[0]).max()) * np.sqrt(3)
        elif shape_b == BOX:
            db = rng.uniform(0.1, 0.8, size=3); rb = np.linalg.norm(db)
        elif shape_b == SPH:
            db = np.array([rng.uniform(0.05, 0.6), 0, 0]); rb = db[0]
        else:
            db = np.array([rng.uniform(0.05, 0.4), rng.uniform(0.0, 0.8), 0]); rb = db[0] + db[1]
        qa = _rot(rng)
        qb = qa.copy() if i % 3 == 1 else _rot(rng)
        off = rng.normal(size=3); off /= np.linalg.norm(off)
        off *= rng.uniform(0.0, ra + rb + MAX_DIST + 0.3)
        pa = rng.uniform(-3, 3, size=3)
        p = (HULL, np.array([float(ia), 0.0, 0.0]), pa, qa, shape_b, db, pa + off, qb)
        pairs.append(p if i % 2 == 0 else (p[4], p[5], p[6], p[7], p[0], p[1], p[2], p[3]))
    return pairs


@pytest.mark.parametrize("scalar", SCALARS)
@pytest.mark.parametrize("shape_b", [HULL, BOX, SPH, CAP])
def test_seeded_soups_meet_the_contract(scalar, shape_b):
    pairs = soup(31 + shape_b, shape_b)
    met = check_contract(scalar, pairs, collide(scalar, pairs))
    assert {"separated", "beyond"} <= met and met & {"deep", "shallow"}, met


@pytest.mark.parametrize("shape_b", [HULL, BOX, SPH, CAP])
def test_swap_translation_and_rotation(shape_b):
    scalar = np.float64
    grid = lambda x: np.round(np.asarray(x) * 2.0 ** 20) / 2.0 ** 20   # positions on a grid the translation keeps exact
    pairs = [(p[0], p[1], grid(p[2]), p[3], p[4], p[5], grid(p[6]), p[7]) for p in soup(41 + shape_b, shape_b, 60)]
    out = collide(scalar, pairs)
    swapped = [(p[4], p[5], p[6], p[7], p[0], p[1], p[2], p[3]) for p in pairs]
    sw = collide(scalar, swapped)
    moved = [(p[0], p[1], p[2] + 5000.0, p[3], p[4], p[5], p[6] + 5000.0, p[7]) for p in pairs]
    mv = collide(scalar, moved)
    for k in ("point_count", "normal", "anchor1", "anchor2", "penetration", "normal_speed"):   # translation keeps every bit
        assert np.array_equal(out[k], mv[k]), k
    for k in range(len(pairs)):
        n = int(out["point_count"][k])
        if n == 0 or int(sw["point_count"][k]) == 0:
            assert n == int(sw["point_count"][k]) or abs(out["penetration"][k].max()) < 1e-3, k
            continue
        # swapping negates the normal and keeps the deepest point (up to the face-axis bias when the SAT feature changes)
        assert abs(out["penetration"][k, :n].max() - sw["penetration"][k, :int(sw["point_count"][k])].max()) <= 1e-4 + 1e-9, k
        if abs(out["normal"][k] @ -sw["normal"][k] - 1) < 1e-9:
            assert np.allclose(out["normal"][k], -sw["normal"][k], atol=1e-12)
    # rotating both shapes about A keeps whether they touch, the deepest point and, where the same feature is chosen (the rotated normal is
    # the rotation of the original one: away from near-ties between axes), the point count
    rng = np.random.default_rng(3)
    counted = 0
    for p, k in zip(pairs, range(len(pairs))):
        r = _rot(rng)
        R = cref.quat_matrix(r)
        rp = (p[0], p[1], p[2], _qmul(r, p[3]), p[4], p[5], p[2] + R @ (np.asarray(p[6]) - p[2]), _qmul(r, p[7]))
        ro = collide(scalar, [rp], moving=False)
        base = collide(scalar, [p], moving=False)
        nb, nr = int(base["point_count"][0]), int(ro["point_count"][0])
        assert (nb == 0) == (nr == 0), k
        if nb == 0:
            continue
        assert abs(base["penetration"][0, :nb].max() - ro["penetration"][0, :nr].max()) <= 1e-4 + 1e-9, k
        if np.linalg.norm(R @ base["normal"][0] - ro["normal"][0]) < 1e-6:
            assert nb == nr, (k, nb, nr)
            counted += 1
    assert counted >= 10, counted


def _qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw,
                     aw * bw - ax * bx - ay * by - az * bz])


def test_cube_hull_matches_the_cuboid_path():
    """the unit cube written as an 8-vertex hull against the box_box path: the same normal and point count away from near-ties, depths
    within the face-axis bias"""
    rng = np.random.default_rng(8)
    hull_pairs, box_pairs = [], []
    for i in range(200):
        db = rng.uniform(0.2, 0.8, 3)
        qa, qb = _rot(rng), _rot(rng)
        off = rng.normal(size=3); off *= rng.uniform(0.3, 1.6) / np.linalg.norm(off)
        hull_pairs.append((HULL, np.array([float(CUBE), 0, 0]), np.zeros(3), qa, BOX, db, off, qb))
        box_pairs.append((BOX, np.full(3, 0.5), np.zeros(3), qa, BOX, db, off, qb))
    h, b = collide(np.float64, hull_pairs), collide(np.float64, box_pairs)
    same = 0
    for k in range(200):
        nh, nb = int(h["point_count"][k]), int(b["point_count"][k])
        assert (nh == 0) == (nb == 0), k
        if nh == 0:
            continue
        assert abs(h["penetration"][k, :nh].max() - b["penetration"][k, :nb].max()) <= 1e-4 + 1e-9, k
        if np.allclose(h["normal"][k], b["normal"][k], atol=1e-9):
            same += 1
            if h["penetration"][k, :nh].max() > -1e-3:
                assert nh == nb, k
    assert same >= 180, same


@pytest.mark.parametrize("scalar", SCALARS)
def test_hull_aabbs_contain_every_posed_vertex(scalar):
    rng = np.random.default_rng(12)
    n = 300
    shape = np.full(n, HULL, dtype=np.int32)
    dims = np.zeros((n, 3)); dims[:, 0] = rng.integers(0, HULLS.count, n)
    pos = rng.uniform(-50, 50, (n, 3)); rot = np.array([_rot(rng) for _ in range(n)])
    bodies = api.Bodies(kind=np.full(n, api.BODY_DYNAMIC, np.uint8), position=pos.astype(scalar), rotation=rot.astype(scalar),
                        linear_velocity=rng.normal(0, 3, (n, 3)).astype(scalar), angular_velocity=np.zeros((n, 3), scalar),
                        inverse_mass=np.ones(n, scalar), inverse_inertia_local=np.zeros((n, 6), scalar))
    pipe = fixture.HostPipeline(shape, dims, np.full(n, 0.5), np.zeros(n), scalar=scalar, hulls=HULLS)
    mn, mx = pipe.update_aabbs(bodies, DT)
    slack = 64 * np.finfo(scalar).eps * 100
    for i in range(n):
        v, _ = HULLS.polyhedron(int(dims[i, 0]))
        for p in (bodies.position[i].astype(float), bodies.position[i].astype(float) + bodies.linear_velocity[i].astype(float) * DT):
            w = ref.posed(np.asarray(v, dtype=scalar).astype(float), p, bodies.rotation[i].astype(float))
            assert np.all(mn[i] <= w.min(axis=0) + slack) and np.all(mx[i] >= w.max(axis=0) - slack), i


def test_derived_table():
    t = fixture.HullTable(np.float64, HULLS).derived()
    eo = t["edge_offsets"]
    for h in range(HULLS.count):
        v, faces = HULLS.polyhedron(h)
        pl = ref.planes(np.asarray(v), [list(f) for f in faces])
        f0 = int(HULLS.face_offsets[h])
        for j, (n, d) in enumerate(pl):
            assert np.allclose(t["plane"][f0 + j, :3], n, atol=1e-12) and abs(t["plane"][f0 + j, 3] - d) < 1e-12
        es = t["edge"][eo[h]:eo[h + 1]]
        assert [tuple(e[:2]) for e in es] == ref.edges(faces)
        assert len(v) - len(es) + len(faces) == 2
        assert np.allclose(t["centre"][h], np.mean(v, axis=0)) and abs(t["radius"][h] - np.linalg.norm(v, axis=1).max()) < 1e-12


def _bad_tables():
    v, f = scenes.regular_solids(0.5)[0]   # tetrahedron
    f = [list(x) for x in f]
    k = np.arange(80) + 0.5   # 80 points of a Fibonacci sphere, all on the hull
    z, phi = 1 - 2 * k / 80, np.pi * (1 + 5 ** 0.5) * k
    big = scenes.convex_hull_of(np.stack([np.sqrt(1 - z * z) * np.cos(phi), np.sqrt(1 - z * z) * np.sin(phi), z], axis=1))
    iv, i_f = scenes.regular_solids(0.5)[2]   # icosahedron
    dent = iv.copy(); dent[0] *= 0.3          # one vertex pushed in past its neighbours' plane: its triangles still face out, a dent
    cube = np.array([[(1 if m & 1 else -1), (1 if m & 2 else -1), (1 if m & 4 else -1)] for m in range(8)], float) * 0.5
    warped = cube.copy(); warped[7] = [0.5, 0.5, 0.6]
    flat = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0.0]])
    return {   # case: (polyhedron, a fragment of the reason)
        "open": ((v, f[:3]), "V - E + F|no reverse|at least 4"),
        "non-manifold": ((v, f + [f[0]]), "appears twice"),
        "short loop": ((v, f[:3] + [[0, 1]]), "fewer than 3"),
        "repeated vertex": ((v, f[:3] + [[0, 0, 1]]), "repeats a vertex"),
        "inward face": ((v, f[:3] + [f[3][::-1]]), "appears twice"),
        "all inward": ((v, [x[::-1] for x in f]), "wound inward"),
        "flat": ((flat, [[0, 1, 2, 3], [3, 2, 1, 0], [0, 1, 2], [0, 2, 3]]), "directed edge|at least 4|wound inward|V - E"),
        "non-convex": ((dent, [list(x) for x in i_f]), "not convex"),
        "non-planar": ((warped, ref.CUBE_FACES), "not planar"),
        "zero area": (_zero_area(v, f), "zero area"),
        "coincident vertices": ((np.concatenate([v, v[:1]]), f), "coincide"),
        "too many vertices": (big, "AVN_HULL_MAX_VERTICES"),
        "face too large": (_big_face(), "AVN_HULL_MAX_FACE_VERTICES"),
        "index out of range": ((v, f[:3] + [[0, 1, 9]]), "past the hull's vertices"),
    }


def _zero_area(v, f):
    """the tetrahedron with the midpoint M of one edge AB added and a sliver face (B, A, M) of zero area, first in the list: the face across
    the edge from the sliver is split into (B, M, Y) and (M, A, Y), so the surface stays closed and V - E + F = 2"""
    a, b, x = f[0]
    f2 = next(g for g in f if any(g[i] == b and g[(i + 1) % 3] == a for i in range(3)))
    y = next(i for i in f2 if i not in (a, b))
    m = len(v)
    faces = [[b, a, m]] + [g for g in f if g is not f2] + [[b, m, y], [m, a, y]]
    return np.concatenate([v, [(v[a] + v[b]) / 2]]), faces


def _big_face():
    k = 33
    a = 2 * np.pi * np.arange(k) / k
    ring = np.stack([np.cos(a), np.zeros(k), np.sin(a)], axis=1)
    v = np.concatenate([ring, [[0, 1.0, 0]]])
    faces = [list(range(k))[::-1]] + [[i, (i + 1) % k, k] for i in range(k)]
    return v, scenes._orient(v, faces)


@pytest.mark.parametrize("case", list(_bad_tables()))
def test_table_refusals(case):
    good = [scenes.regular_solids(0.5)[1]]
    poly, why = _bad_tables()[case]
    with pytest.raises(ValueError, match=f"hull 1: .*({why})"):
        fixture.HullTable(np.float64, api.ConvexHulls.from_polyhedra(good + [poly]))
    fixture.HullTable(np.float64, api.ConvexHulls.from_polyhedra(good))   # the good one alone is accepted


def test_shape_three_needs_a_table():
    pairs = soup(1, SPH, 4)
    with pytest.raises(ValueError):
        collide(np.float64, pairs, hulls=None)
    too_few = api.ConvexHulls.from_polyhedra([scenes.regular_solids(0.5)[0]])
    with pytest.raises(ValueError):
        collide(np.float64, [(HULL, np.array([1.0, 0, 0]), np.zeros(3), np.array([0, 0, 0, 1.0]), SPH, np.array([0.3, 0, 0]), np.ones(3),
                              np.array([0, 0, 0, 1.0]))], hulls=too_few)


def test_mass_properties():
    he = np.array([0.3, 0.5, 0.7])
    cube = np.array([[(1 if m & 1 else -1), (1 if m & 2 else -1), (1 if m & 4 else -1)] for m in range(8)], float) * he
    m, com, inertia = scenes.hull_mass(cube + [1.0, 2.0, 3.0], ref.CUBE_FACES, density=2.0)
    mc, ic = scenes._cuboid_mass(he[None, :], density=2.0)
    assert np.isclose(m, mc[0]) and np.allclose(com, [1.0, 2.0, 3.0]) and np.allclose(inertia, np.diag(ic[0]), atol=1e-12)
    v, f = scenes.regular_solids(1.0)[0]
    a = np.linalg.norm(v[0] - v[1])
    m, com, inertia = scenes.hull_mass(v, f)
    assert np.isclose(m, a ** 3 / (6 * np.sqrt(2))) and np.allclose(com, 0, atol=1e-12)
    assert np.allclose(inertia, np.eye(3) * m * a * a / 20.0, atol=1e-12)


def _world(scene, steps, substeps=4):
    w = plugins.World(scene, oracle_lib.oracle_plugins(), substeps=substeps)
    for _ in range(steps):
        w.step()
    return w


def _single(poly, pos, rot, scalar=np.float64):
    """one hull body above the ground cuboid"""
    v, f, m, inertia = scenes._centred(*poly)
    hulls = api.ConvexHulls.from_polyhedra([(v, f)])
    sc = scenes._assemble("hull", np.array([[0, -0.5, 0], pos]), np.array([[0, 0, 0, 1.0], rot]), np.array([api.BODY_STATIC, api.BODY_DYNAMIC]),
                          np.array([[20, 0.5, 20], [0.5, 0.5, 0.5]]), np.array([BOX, HULL]), scalar, hulls=hulls)
    sc.dims[1] = 0.0
    scenes._set_hull_mass(sc, [(v, f, m, inertia)])
    return scenes._own_velocities(sc)


def test_hull_cube_rests_like_a_cuboid():
    cube = np.array([[(1 if m & 1 else -1), (1 if m & 2 else -1), (1 if m & 4 else -1)] for m in range(8)], float) * 0.5
    w = _world(_single((cube, ref.CUBE_FACES), [0, 0.55, 0], [0, 0, 0, 1.0]), 90)
    sc = scenes._assemble("box", np.array([[0, -0.5, 0], [0, 0.55, 0]]), np.array([[0, 0, 0, 1.0]] * 2), np.array([api.BODY_STATIC, api.BODY_DYNAMIC]),
                          np.array([[20, 0.5, 20], [0.5, 0.5, 0.5]]), np.array([BOX, BOX]), np.float64)
    wb = _world(scenes._own_velocities(sc), 90)
    assert np.allclose(w.bodies.position[1], wb.bodies.position[1], atol=2e-3), (w.bodies.position[1], wb.bodies.position[1])
    assert np.linalg.norm(w.bodies.linear_velocity[1]) < 0.05


def test_tetrahedron_settles_on_a_face():
    tet = scenes.regular_solids(0.4)[0]
    q = np.array([0.3, 0.1, 0.2, 0.9]); q /= np.linalg.norm(q)
    w = _world(_single(tet, [0, 0.6, 0], q), 240)
    v, f, _, _ = scenes._centred(*tet)
    wv = ref.posed(v, w.bodies.position[1], w.bodies.rotation[1])
    low = np.sort(wv[:, 1])
    assert np.linalg.norm(w.bodies.linear_velocity[1]) < 0.05 and np.linalg.norm(w.bodies.angular_velocity[1]) < 0.2
    assert low[2] - low[0] < 0.02 and low[3] - low[0] > 0.2, low   # three vertices down: resting on a face


def test_small_hull_pile_comes_to_rest():
    sc = scenes.hull_pile(40, seed=2, layers=2, scalar=np.float64)
    w = _world(sc, 300)
    dyn = sc.bodies.kind == api.BODY_DYNAMIC
    assert np.all(w.bodies.position[dyn, 1] > -0.05)
    flat = dyn & np.isin(sc.shape_type, [HULL, BOX])   # spheres and capsules may still roll (no rolling friction)
    assert np.abs(w.bodies.linear_velocity[flat]).max() < 0.05 and np.abs(w.bodies.angular_velocity[flat]).max() < 0.3


@pytest.mark.parametrize("tips", [False, True])
def test_decomposed_l_block_rests_or_tips(tips):
    sc = scenes.decomposed_l_block(upright_x=-1.05 if tips else -0.4)
    w = _world(sc, 180)
    q = w.bodies.rotation[1]
    tilt = np.degrees(2 * np.arccos(min(1.0, abs(q[3]))))
    # tipping turns the block about the foot's edge until the upright's lower corner meets the ground (about 17 degrees)
    assert (tilt > 10 if tips else tilt < 1), tilt


def test_host_ccd_refuses_hulls():
    """the host brute force refuses a row that names a hull, with or without the capsule flag, as the device refuses the contact store"""
    bodies = dict(kind=np.array([api.BODY_STATIC, api.BODY_DYNAMIC], np.uint8), position=np.array([[0, -0.5, 0], [0, 1, 0]], np.float32),
                  rotation=np.array([[0, 0, 0, 1.0]] * 2, np.float32), linear_velocity=np.array([[0, -50, 0]] * 2, np.float32),
                  angular_velocity=np.zeros((2, 3), np.float32))
    rows = dict(c1=np.array([0]), c2=np.array([1]), b1=np.array([0]), b2=np.array([1]), live=np.array([1]))
    for caps in (False, True):
        with pytest.raises(api.AvianError) as e:
            fixture.ccd_solve(np.float32, 1 / 60, 1.0, bodies, np.array([BOX, HULL]), np.array([[5, 0.5, 5], [0, 0, 0]]), rows,
                              dict(body=np.array([1]), collider=np.array([1]), capsules=caps))
        assert e.value.status == api.ERR_UNSUPPORTED


@pytest.mark.parametrize("scalar", SCALARS)
@pytest.mark.parametrize("framed", [False, True])
def test_the_row_function_with_hulls_equals_the_geometry_stage(scalar, framed):
    """avh_rows_narrow_hulls (csrc/contact_rows.hpp, the function narrow_hull_edges_kernel runs per row, and the cuboid / sphere / capsule rows
    beside them) gives the geometry stage's manifolds, with and without body frames; run twice, the second pass matches the first pass's
    points and carries their impulses over"""
    rng = np.random.default_rng(17)
    pairs = []
    for shape_b in (HULL, BOX, SPH, CAP):
        pairs += soup(60 + shape_b, shape_b, 60)
    for _ in range(40):
        q = rng.normal(size=(2, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
        pairs.append((BOX, rng.uniform(0.2, 0.8, 3), rng.uniform(-1, 1, 3), q[0], CAP, np.array([0.2, 0.4, 0.0]), rng.uniform(-1, 1, 3), q[1]))
    E, s = len(pairs), np.dtype(scalar)
    cols = {"shape": np.array([x for p in pairs for x in (p[0], p[4])], dtype=np.uint8)}
    for key, ia, ib in (("dims", 1, 5), ("position", 2, 6), ("rotation", 3, 7)):
        cols[key] = np.ascontiguousarray([np.asarray(v, float) for p in pairs for v in (p[ia], p[ib])], dtype=s)
    c1, c2 = np.arange(0, 2 * E, 2, dtype=np.uint32), np.arange(1, 2 * E, 2, dtype=np.uint32)
    lv = np.zeros((2 * E, 3), dtype=s); lv[1::2, 0] = MAX_DIST / DT
    av = rng.normal(0, 0.5, (2 * E, 3)).astype(s)
    frames = None
    if framed:
        q = rng.normal(size=(2 * E, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
        frames = {"position": (cols["position"].astype(np.float64) + rng.uniform(-0.3, 0.3, (2 * E, 3))).astype(s), "rotation": q.astype(s),
                  "center_of_mass": rng.uniform(-0.2, 0.2, (2 * E, 3)).astype(s)}
    want = fixture.raw_manifolds(s, DT, 1e-3, (c1, c2, c1, c2), cols, lv, av, frames=frames, hulls=HULLS)
    table = fixture.HullTable(s, HULLS)
    z = lambda *sh, d=s: np.zeros(sh, dtype=d)
    live, count, disjoint = np.ones(E, dtype=np.uint8), z(E, d=np.uint8), z(E, d=np.uint8)
    normal, a1, a2, pen, ns = z(E, 3), z(E, 4, 3), z(E, 4, 3), z(E, 4), z(E, 4)
    prev_count, prev_a1, prev_a2 = z(E, d=np.uint8), z(E, 4, 3, d=np.float64), z(E, 4, 3, d=np.float64)
    ws_n_in, ws_t_in, ws_n_out, ws_t_out = z(E, 4), z(E, 4, 2), z(E, 4), z(E, 4, 2)
    big = np.full((2 * E, 3), 1e6, dtype=s)   # AABBs that always overlap
    p = fixture._p
    fp, fr, fc = (None, None, None) if frames is None else (frames["position"], frames["rotation"], frames["center_of_mass"])

    def run():
        fixture._load().avh_rows_narrow_hulls(
            32 if s == np.float32 else 64, E, p(c1), p(c2), p(c1), p(c2), p(live), p(count), p(disjoint), p(normal), p(a1), p(a2), p(pen), p(ns),
            p(prev_count), p(prev_a1), p(prev_a2), p(ws_n_in), p(ws_t_in), p(ws_n_out), p(ws_t_out), p(cols["shape"]), p(cols["dims"]),
            p(cols["position"]), p(cols["rotation"]), p(lv), p(av), p(-big), p(big), DT, 1e-3, 1.0, 1, p(fp), p(fr), p(fc), table.h)

    run()
    assert np.array_equal(count, want["point_count"])
    for got, k in ((normal, "normal"), (a1, "anchor1"), (a2, "anchor2"), (pen, "penetration"), (ns, "normal_speed")):
        assert np.array_equal(got, want[k]), k
    hull_rows = np.array([HULL in (q[0], q[4]) for q in pairs])
    assert (count[hull_rows] > 0).sum() > 50 and (count[~hull_rows] > 0).sum() > 10
    # the solve's impulses, then the same rows again: a point inherits the impulse of the first previous point whose two anchors lie within
    # 0.1 of its own, in either body order (match_contacts), which is at the latest the point itself
    ws_n_out[:] = np.arange(E * 4, dtype=s).reshape(E, 4) + 1
    old_a1, old_a2, old_n = prev_a1.copy(), prev_a2.copy(), count.copy()
    run()
    near = lambda x, y: float((x - y) @ (x - y)) < 0.01
    for e in range(E):
        for k in range(int(count[e])):
            j = next(j for j in range(int(old_n[e])) if (near(old_a1[e, k], old_a1[e, j]) and near(old_a2[e, k], old_a2[e, j]))
                     or (near(old_a1[e, k], old_a2[e, j]) and near(old_a2[e, k], old_a1[e, j])))
            assert ws_n_in[e, k] == 4 * e + j + 1, (e, k)
