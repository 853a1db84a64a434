"""Capsule colliders in the host fixture (csrc/narrow_math.hpp through avh_raw_manifolds, the AABB update, scenes' mass properties) against
the independent float64 restatement of tests/capsule_reference.py: the contact contract of DESIGN.md §7h on seeded soups of every pair type,
hand-worked pairs with exact values, symmetry and invariance, the degenerate capsules, and a CPU World with the oracle solver."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
from avian_b200 import api, fixture, plugins, scenes  # noqa: E402
import capsule_reference as ref  # noqa: E402
import oracle_lib  # noqa: E402

BOX, SPH, CAP = fixture.SHAPE_CUBOID, fixture.SHAPE_SPHERE, fixture.SHAPE_CAPSULE
DT, MAX_DIST = 1.0 / 60.0, 0.5          # a relative speed of 30 along x makes the speculative margin dt * 30 = 0.5
SCALARS = [np.float32, np.float64]
IDENT = np.array([0.0, 0.0, 0.0, 1.0])


def qaxis(axis, angle):
    a = np.asarray(axis, float) / np.linalg.norm(axis)
    return np.concatenate([a * np.sin(angle / 2), [np.cos(angle / 2)]])


Z90 = qaxis([0, 0, 1], np.pi / 2)      # maps the capsule axis y onto -x


def collide(scalar, pairs, moving=True):
    """pairs: list of (shape_a, dims_a, pos_a, rot_a, shape_b, dims_b, pos_b, rot_b) -> raw manifolds of every pair (A = collider 2k)"""
    n = len(pairs)
    shape = np.array([s for p in pairs for s in (p[0], p[4])], dtype=np.uint8)
    cols = {"shape": shape}
    for key, ia, ib in (("dims", 1, 5), ("position", 2, 6), ("rotation", 3, 7)):
        cols[key] = np.ascontiguousarray([np.asarray(v, float) for p in pairs for v in (p[ia], p[ib])], dtype=scalar)
    c1, c2 = np.arange(0, 2 * n, 2, dtype=np.uint32), np.arange(1, 2 * n, 2, dtype=np.uint32)
    lv = np.zeros((2 * n, 3), dtype=scalar)
    if moving:
        lv[1::2, 0] = MAX_DIST / DT
    out = fixture.raw_manifolds(scalar, DT, 1e-3, (c1, c2, c1, c2), cols, lv, np.zeros((2 * n, 3), dtype=scalar), f64_anchors=True)
    out["cols"] = cols
    return out


def as_f64(scalar, p):
    """a pair with its values rounded to the column type (what the fixture reads), back in float64"""
    return tuple(v if np.isscalar(v) or isinstance(v, (int, np.integer)) else np.asarray(v, dtype=scalar).astype(np.float64) for v in p)


def witnesses(out, k, p):
    n = int(out["point_count"][k])
    a = np.asarray(p[2]) + out["anchor1_f64"][k, :n]
    b = np.asarray(p[6]) + out["anchor2_f64"][k, :n]
    return n, out["normal"][k].astype(np.float64), a, b, out["penetration"][k, :n].astype(np.float64)


def scale_of(p):
    return 1.0 + np.abs(np.asarray(p[2])).max() + np.abs(np.asarray(p[6])).max() + np.abs(p[1]).sum() + np.abs(p[5]).sum()


def check_contract(scalar, pairs, out):
    """DESIGN.md §7h's contract on every pair; returns the classes met"""
    eps = np.finfo(scalar).eps
    met = set()
    for k, p in enumerate(pairs):
        p = as_f64(scalar, p)
        tol = 64 * eps * scale_of(p)
        D, depth = ref.capsule_depth(*p)
        n, nrm, a, b, pen = witnesses(out, k, p)
        assert n <= 2, f"pair {k}: {n} points"
        if depth == 0.0 and D > MAX_DIST:
            assert n == 0, f"pair {k}: {n} points at distance {D} beyond the margin"
            met.add("beyond")
            continue
        if depth == 0.0 and D > MAX_DIST - 1e-6:
            continue
        assert n >= 1, f"pair {k}: no point at distance {D}, depth {depth}"
        assert abs(np.linalg.norm(nrm) - 1.0) <= 8 * eps, f"pair {k}: |n| = {np.linalg.norm(nrm)}"
        assert nrm @ (np.asarray(p[6]) - np.asarray(p[2])) >= -tol or depth > 0, f"pair {k}: the normal points from B to A"
        for i in range(n):
            assert ref.surface_distance(p[0], p[1], p[2], p[3], a[i]) <= tol, f"pair {k} point {i}: a is off A's surface"
            assert ref.surface_distance(p[4], p[5], p[6], p[7], b[i]) <= tol, f"pair {k} point {i}: b is off B's surface"
            assert np.linalg.norm(np.cross(b[i] - a[i], nrm)) <= tol, f"pair {k} point {i}: b - a is not along n"
            assert abs(pen[i] - (a[i] - b[i]) @ nrm) <= tol, f"pair {k} point {i}: penetration"
        if depth > 0.0:
            slack = 1e-4 + tol if BOX in (p[0], p[4]) else tol
            assert abs(pen.max() - depth) <= slack, f"pair {k}: deepest {pen.max()} vs exact depth {depth}"
            met.add("deep" if depth > 0.1 else "shallow")
        else:
            assert -pen.max() <= D + tol, f"pair {k}: smallest gap {-pen.max()} vs distance {D}"
            met.add("separated")
    return met


def soup(seed, shape_b, count=300):
    """capsule (A) against shape_b at random orientations and offsets from deep to beyond the margin, plus parallel, crossed and end-on pairs"""
    rng = np.random.default_rng(seed)
    pairs = []
    for i in range(count):
        ra, ha = rng.uniform(0.05, 0.5), rng.uniform(0.0, 1.0)
        if shape_b == BOX:
            db = rng.uniform(0.1, 1.0, size=3)
        elif shape_b == SPH:
            db = np.array([rng.uniform(0.05, 0.6), 0, 0])
        else:
            db = np.array([rng.uniform(0.05, 0.5), rng.uniform(0.0, 1.0), 0])
        qa = rng.normal(size=4); qa /= np.linalg.norm(qa)
        qb = rng.normal(size=4); qb /= np.linalg.norm(qb)
        kind = i % 5
        reach = ra + ha + np.abs(db).sum()
        off = rng.normal(size=3); off /= np.linalg.norm(off)
        off *= rng.uniform(0.0, reach + MAX_DIST + 0.3)
        if kind == 1:                  # parallel: the same orientation (a capsule along a box face's plane)
            qb = qa.copy()
        elif kind == 2 and shape_b == CAP:   # crossed: perpendicular axes
            qb = _compose(qa, qaxis([1, 0, 0], np.pi / 2))
            off = ref.quat_rotate(qa, [0, 0, 1]) * rng.uniform(0.0, ra + db[0] + 0.4)
        elif kind == 3:                # end-on: B along A's axis
            off = ref.quat_rotate(qa, [0, 1, 0]) * rng.uniform(ha, ha + ra + np.abs(db).max() + 0.3)
        elif kind == 4 and shape_b == BOX:   # deep: the segment inside the box
            db = np.full(3, ha + ra + 0.2)
            off = rng.uniform(-0.1, 0.1, size=3)
        pa = rng.uniform(-3, 3, size=3)
        pairs.append((CAP, np.array([ra, ha, 0.0]), pa, qa, shape_b, db, pa + off, qb))
    return pairs


def _compose(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw,
                     aw * bw - ax * bx - ay * by - az * bz])


@pytest.mark.parametrize("scalar", SCALARS)
@pytest.mark.parametrize("shape_b", [CAP, SPH, BOX])
def test_seeded_soups_meet_the_contract(scalar, shape_b):
    pairs = soup(11 + shape_b, shape_b)
    met = check_contract(scalar, pairs, collide(scalar, pairs))
    assert {"beyond", "separated", "shallow", "deep"} <= met, met
    # the other order: B against the capsule
    swapped = [(p[4], p[5], p[6], p[7], p[0], p[1], p[2], p[3]) for p in pairs]
    check_contract(scalar, swapped, collide(scalar, swapped))


def test_reference_segment_distance_against_50_digits():
    rng = np.random.default_rng(3)
    worst = 0.0
    for _ in range(200):
        p0, p1, q0, q1 = rng.uniform(-2, 2, size=(4, 3))
        if rng.uniform() < 0.3:
            q1 = q0 + (p1 - p0) * rng.uniform(0.2, 2)   # parallel
        d = ref.segment_segment(p0, p1, q0, q1)[0]
        worst = max(worst, abs(d - ref.mp_segment_distance(p0, p1, q0, q1)))
    assert worst < 1e-13, worst


def one(scalar, p, moving=False):
    out = collide(scalar, [p], moving)
    return witnesses(out, 0, as_f64(scalar, p))


@pytest.mark.parametrize("scalar", SCALARS)
def test_hand_worked_pairs(scalar):
    tol = 64 * np.finfo(scalar).eps * 4
    box = (BOX, np.array([2.0, 0.5, 2.0]), np.zeros(3), IDENT)
    # a capsule lying on a box face, its axis 0.25 above the face: two points of penetration r - 0.25 at the segment's ends
    n, nrm, a, b, pen = one(scalar, box + (CAP, np.array([0.3, 0.8, 0.0]), np.array([0.0, 0.75, 0.0]), Z90))
    assert n == 2 and np.allclose(nrm, [0, 1, 0], atol=tol) and np.allclose(pen, 0.05, atol=tol)
    assert np.allclose(sorted(a[:, 0]), [-0.8, 0.8], atol=tol) and np.allclose(a[:, 1], 0.5, atol=tol)
    # standing on the box: one point under its cap
    n, nrm, a, b, pen = one(scalar, box + (CAP, np.array([0.3, 0.8, 0.0]), np.array([0.0, 0.5 + 0.8 + 0.3 - 0.02, 0.0]), IDENT))
    assert n == 1 and np.allclose(nrm, [0, 1, 0], atol=tol) and np.allclose(pen, 0.02, atol=tol) and np.allclose(a[0], [0, 0.5, 0], atol=tol)
    # crossed capsules: the normal along u x w (y x -x = +z), apart and with intersecting axes
    for d in (0.3, 0.0):
        n, nrm, a, b, pen = one(scalar, (CAP, np.array([0.2, 1.0, 0]), np.zeros(3), IDENT, CAP, np.array([0.25, 1.0, 0]), np.array([0, 0, d]), Z90))
        assert n == 1 and np.allclose(nrm, [0, 0, 1], atol=tol) and np.allclose(pen, 0.45 - d, atol=tol), (nrm, pen)
    # parallel capsules half overlapping: points at the ends of the overlap
    n, nrm, a, b, pen = one(scalar, (CAP, np.array([0.3, 1.0, 0]), np.zeros(3), IDENT, CAP, np.array([0.3, 1.0, 0]), np.array([0.5, 1.0, 0]), IDENT))
    assert n == 2 and np.allclose(nrm, [1, 0, 0], atol=tol) and np.allclose(pen, 0.1, atol=tol) and np.allclose(sorted(a[:, 1]), [0, 1], atol=tol)
    # capsule against a sphere at the cap and at the side
    n, nrm, a, b, pen = one(scalar, (CAP, np.array([0.3, 1.0, 0]), np.zeros(3), IDENT, SPH, np.array([0.2, 0, 0]), np.array([0, 1.45, 0]), IDENT))
    assert n == 1 and np.allclose(nrm, [0, 1, 0], atol=tol) and np.allclose(pen, 0.05, atol=tol) and np.allclose(a[0], [0, 1.3, 0], atol=tol)
    n, nrm, a, b, pen = one(scalar, (CAP, np.array([0.3, 1.0, 0]), np.zeros(3), IDENT, SPH, np.array([0.2, 0, 0]), np.array([0.45, 0.3, 0]), IDENT))
    assert n == 1 and np.allclose(nrm, [1, 0, 0], atol=tol) and np.allclose(pen, 0.05, atol=tol) and np.allclose(a[0], [0.3, 0.3, 0], atol=tol)


@pytest.mark.parametrize("scalar", SCALARS)
def test_swap_negates_the_normal_and_keeps_the_deepest_point(scalar):
    for shape_b in (CAP, SPH, BOX):
        pairs = soup(40 + shape_b, shape_b, 120)
        ab = collide(scalar, pairs)
        ba = collide(scalar, [(p[4], p[5], p[6], p[7], p[0], p[1], p[2], p[3]) for p in pairs])
        for k, p in enumerate(pairs):
            if ab["point_count"][k] == 0 or ba["point_count"][k] == 0:
                continue
            tol = 64 * np.finfo(scalar).eps * scale_of(as_f64(scalar, p))
            assert np.allclose(ab["normal"][k], -ba["normal"][k], rtol=0, atol=tol), k
            assert abs(ab["penetration"][k, :ab["point_count"][k]].max() - ba["penetration"][k, :ba["point_count"][k]].max()) <= tol, k


@pytest.mark.parametrize("scalar", SCALARS)
def test_translation_keeps_every_bit_and_rotation_keeps_the_counts(scalar):
    rng = np.random.default_rng(5)
    for shape_b in (CAP, SPH, BOX):
        pairs = []
        for p in soup(60 + shape_b, shape_b, 100):
            # positions on a 1/1024 grid: a translation by 1e4 is exact in f32 and f64, so pb - pa is the same
            pairs.append(p[:2] + (np.round(np.asarray(p[2]) * 1024) / 1024,) + p[3:6] + (np.round(np.asarray(p[6]) * 1024) / 1024,) + p[7:])
        base = collide(scalar, pairs)
        moved = collide(scalar, [p[:2] + (p[2] + 1e4,) + p[3:6] + (p[6] + 1e4,) + p[7:] for p in pairs])
        for key in ("point_count", "normal", "anchor1", "anchor2", "penetration", "normal_speed"):
            assert np.array_equal(base[key], moved[key]), key
        R = rng.normal(size=4); R /= np.linalg.norm(R)
        turned = collide(scalar, [(p[0], p[1], ref.quat_rotate(R, p[2]), _compose(R, p[3]), p[4], p[5], ref.quat_rotate(R, p[6]), _compose(R, p[7]))
                                  for p in pairs], moving=False)
        still = collide(scalar, pairs, moving=False)
        differ = np.nonzero(turned["point_count"] != still["point_count"])[0]
        assert differ.size == 0, f"point counts changed under rotation for pairs {differ}"


@pytest.mark.parametrize("scalar", SCALARS)
def test_zero_half_length_is_a_sphere_and_zero_radius_a_segment(scalar):
    rng = np.random.default_rng(9)
    for shape_b in (SPH, BOX, CAP):
        pairs = [p[:1] + (np.array([p[1][0], 0.0, 0.0]),) + p[2:] for p in soup(80 + shape_b, shape_b, 150)]
        if shape_b == CAP:
            pairs = [p[:5] + (np.array([p[5][0], 0.0, 0.0]),) + p[6:] for p in pairs]
        spheres = [(SPH,) + p[1:4] + ((SPH,) if p[4] == CAP else (p[4],)) + p[5:] for p in pairs]
        c, s = collide(scalar, pairs), collide(scalar, spheres)
        assert np.array_equal(c["point_count"], s["point_count"])
        for k, p in enumerate(pairs):
            m = int(c["point_count"][k])
            if m == 0:
                continue
            tol = 64 * np.finfo(scalar).eps * scale_of(as_f64(scalar, p))
            assert np.allclose(c["normal"][k], s["normal"][k], atol=tol), k
            assert np.allclose(c["anchor1_f64"][k, :m], s["anchor1_f64"][k, :m], atol=tol), k
            assert np.allclose(c["anchor2_f64"][k, :m], s["anchor2_f64"][k, :m], atol=tol), k
        segments = [p[:1] + (np.array([0.0, p[1][1] + 0.1, 0.0]),) + p[2:] for p in soup(90 + shape_b, shape_b, 150)]
        check_contract(scalar, segments, collide(scalar, segments))


@pytest.mark.parametrize("scalar", SCALARS)
def test_the_fixture_aabb_holds_the_capsule(scalar):
    rng = np.random.default_rng(13)
    n = 200
    dims = np.stack([rng.uniform(0.05, 0.5, n), rng.uniform(0.0, 1.5, n), np.zeros(n)], axis=1)
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    pos = rng.uniform(-50, 50, size=(n, 3))
    sc = scenes._assemble("capsules", pos, q, np.full(n, api.BODY_DYNAMIC), dims, np.full(n, CAP), scalar)
    pipe = fixture.HostPipeline(sc.shape_type, sc.dims, sc.friction, sc.restitution, scalar=scalar)
    mn, mx = pipe.update_aabbs(sc.bodies, 1.0 / 60.0)
    tol = 64 * np.finfo(scalar).eps * 60
    for i in range(n):
        d, p, r = sc.dims[i], sc.bodies.position[i].astype(np.float64), sc.bodies.rotation[i].astype(np.float64)
        e0, e1 = ref.capsule_segment(p, r, d[1])
        lo, hi = np.minimum(e0, e1) - d[0], np.maximum(e0, e1) + d[0]
        grow = 5e-3   # contact_tolerance * length_unit
        assert np.all(np.abs(mn[i] - (lo - grow)) <= tol) and np.all(np.abs(mx[i] - (hi + grow)) <= tol), i
        # the reference in the column type, operation by operation, agrees with the float64 box
        rmn, rmx = ref.capsule_aabb(scalar, sc.dims[i], sc.bodies.position[i], sc.bodies.rotation[i])
        assert np.all(np.abs(rmn - lo) <= tol) and np.all(np.abs(rmx - hi) <= tol), i
        # sampled surface points lie inside
        v = rng.normal(size=(64, 3)); v /= np.linalg.norm(v, axis=1, keepdims=True)
        t = rng.uniform(0, 1, size=(64, 1))
        pts = e0 + (e1 - e0) * t + v * d[0]
        assert np.all(pts >= mn[i] - tol) and np.all(pts <= mx[i] + tol), i


def test_capsule_mass_closed_form():
    from scipy.integrate import quad
    for r, h in ((0.3, 0.0), (0.2, 0.7), (1e-4, 1.0), (0.5, 2.0)):
        m, inertia = scenes._capsule_mass(np.array([r]), np.array([h]))
        rho = lambda y: r if abs(y) <= h else np.sqrt(max(r * r - (abs(y) - h) ** 2, 0.0))   # noqa: E731
        lim = h + r
        mq = quad(lambda y: np.pi * rho(y) ** 2, -lim, lim, points=[-h, h])[0]
        iy = quad(lambda y: np.pi * rho(y) ** 4 / 2, -lim, lim, points=[-h, h])[0]
        ix = quad(lambda y: np.pi * rho(y) ** 4 / 4 + np.pi * rho(y) ** 2 * y * y, -lim, lim, points=[-h, h])[0]
        assert np.allclose([m[0], inertia[0, 0], inertia[0, 1], inertia[0, 2]], [mq, ix, iy, ix], rtol=1e-8), (r, h)
    # the sphere limit and the thin-rod limit
    m, i = scenes._capsule_mass(np.array([0.4]), np.array([0.0]))
    ms = 4 / 3 * np.pi * 0.4 ** 3
    assert np.allclose(m, ms) and np.allclose(i, 0.4 * ms * 0.16)
    m, i = scenes._capsule_mass(np.array([1e-6]), np.array([1.0]))
    assert np.allclose(i[0, 0], m[0] * 4.0 / 12.0, rtol=1e-5) and i[0, 1] < 1e-12


def _world(sc, substeps=6):
    return plugins.World(sc, oracle_lib.oracle_plugins(), substeps=substeps)


def _single(pos, rot, dims, scalar=np.float32):
    p = np.array([[0.0, -0.5, 0.0], pos])
    q = np.array([IDENT, rot])
    he = np.array([[10.0, 0.5, 10.0], dims])
    return scenes._assemble("capsule", p, q, np.array([api.BODY_STATIC, api.BODY_DYNAMIC]), he, np.array([BOX, CAP]), scalar)


def test_a_capsule_dropped_flat_rests_on_two_contacts():
    r = 0.25
    w = _world(_single([0.0, r + 0.3, 0.0], Z90, [r, 0.6, 0.0]))
    for _ in range(180):
        w.step()
    y = float(w.bodies.position[1, 1])
    assert abs(y - r) <= 0.01 * r, y
    assert w.last_manifolds.count == 1 and int(np.diff(w.last_manifolds.point_offsets)[0]) == 2
    assert np.abs(w.bodies.linear_velocity[1]).max() < 1e-2


def test_a_standing_capsule_stays_upright():
    w = _world(_single([0.0, 0.8 + 0.2 + 0.01, 0.0], IDENT, [0.2, 0.8, 0.0]))
    for _ in range(180):
        w.step()
    up = ref.quat_rotate(w.bodies.rotation[1].astype(np.float64), [0, 1, 0])
    assert up[1] > 0.999, up
    assert abs(float(w.bodies.position[1, 1]) - 1.0) < 0.01


def log_piles(count=1, n_layers=4, r=0.2, h=0.6, pitch=3.0):
    """`count` log-cabin piles of capsules side by side on a static ground (4 layers of 3 by default, axes crossing from layer to layer):
    each comes to rest as an island of its own"""
    pos, rot = [[0.0, -0.5, 0.0]], [IDENT]
    for c in range(count):
        for k in range(n_layers):
            for j in (-1, 0, 1):
                off = 0.5 * j
                pos.append([c * pitch + off, r + k * (2 * r - 0.002), 0.0] if k % 2 else [c * pitch, r + k * (2 * r - 0.002), off])
                rot.append(qaxis([1, 0, 0], np.pi / 2) if k % 2 else Z90)
    n = len(pos)
    he = np.concatenate([[[10.0 + count * pitch, 0.5, 10.0]], np.tile([r, h, 0.0], (n - 1, 1))])
    return scenes._assemble(f"log_piles_{count}", np.array(pos), np.array(rot), np.concatenate([[api.BODY_STATIC], np.full(n - 1, api.BODY_DYNAMIC)]),
                            he, np.concatenate([[BOX], np.full(n - 1, CAP)]), np.float32)


def test_a_resting_pile_gains_no_energy():
    """a log-cabin pile of capsules comes to rest and its kinetic energy does not grow"""
    n_layers, r = 4, 0.2
    sc = log_piles(1, n_layers, r)
    w = _world(sc, substeps=8)
    inv_m = sc.bodies.inverse_mass.astype(np.float64)
    inertia = 1.0 / np.where(inv_m[:, None] > 0, sc.bodies.inverse_inertia_local.astype(np.float64)[:, [0, 3, 5]], 1.0)

    def kinetic():
        v = w.bodies.linear_velocity.astype(np.float64)[1:]
        om = np.array([ref.quat_rotate(q * [-1, -1, -1, 1], o) for q, o in zip(w.bodies.rotation.astype(np.float64), w.bodies.angular_velocity)])[1:]
        return float((0.5 / inv_m[1:] * (v * v).sum(axis=1)).sum() + 0.5 * (inertia[1:] * om * om).sum())

    for _ in range(120):
        w.step()
    energies = []
    for _ in range(120):
        w.step()
        energies.append(kinetic())
    assert max(energies) <= energies[0] * 1.1 + 1e-5, energies[::10]
    assert energies[-1] < 1e-3, energies[-1]
    assert float(w.bodies.position[1:, 1].max()) > (n_layers - 1) * 2 * r, "the pile collapsed"
