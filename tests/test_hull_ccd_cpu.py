"""Swept CCD with convex hull colliders, without a GPU: the hull branches of csrc/ccd_math.hpp (pair_toi / nonlinear_toi at shape level
G = 2) against the independent float64 hull distances of tests/hull_reference.py, the linear mode against the hull shape casts of the
spatial queries and tests/hull_query_reference.py's linear program, the spin bound against the face-plane polytope, and the host brute
force's control flow with AVN_CCD_HULLS against tests/ccd_reference.py."""
from __future__ import annotations

import numpy as np
import pytest

import ccd_reference as ref
import hull_query_reference as hq
import hull_reference as hr
import test_capsule_ccd_cpu as caps
import test_ccd_cpu as cpu
from avian_b200 import api, fixture, scenes

DT, EPS = cpu.DT, cpu.EPS
CUBOID, SPHERE, CAPSULE, HULL = fixture.SHAPE_CUBOID, fixture.SHAPE_SPHERE, fixture.SHAPE_CAPSULE, api.SHAPE_CONVEX_HULL
PAIRS = [(HULL, HULL), (HULL, CUBOID), (CUBOID, HULL), (HULL, SPHERE), (SPHERE, HULL), (HULL, CAPSULE), (CAPSULE, HULL)]
SCALARS = [np.float32, np.float64]


def hull_set(seed=5, kinds=6):
    """seeded random hulls (Qhull over 8-16 points) and the regular solids, as scenes.hull_pile builds its table"""
    rng = np.random.default_rng(seed)
    polys = [scenes.convex_hull_of(rng.normal(size=(int(rng.integers(8, 17)), 3)) * rng.uniform(0.3, 0.8)) for _ in range(kinds)]
    polys += scenes.regular_solids(0.6)
    return api.ConvexHulls.from_polyhedra(polys)


HULLS = hull_set()


def table(scalar=np.float64, hulls=HULLS):
    return fixture.HullTable(scalar, hulls)


def poly(m, t, hulls=HULLS):
    """(world vertices, faces) of the polytope of a hull or cuboid motion record at time t"""
    c, R = cpu.pose(m, t)
    if m[0] == CUBOID:
        V, F = hr.box_poly(m[1:4], np.zeros(3), np.array([0, 0, 0, 1.0]))
    else:
        V, F = hq.table_poly(hulls, int(m[1]))
    return np.asarray(V, float) @ R.T + c, F


def distance(a, b, t, hulls=HULLS):
    """exact float64 distance of two shapes at time t (0 when they overlap): tests/hull_reference.py for a pair with a hull"""
    if a[0] != HULL and b[0] != HULL:
        return caps.distance(a, b, t)
    if a[0] != HULL:
        a, b = b, a
    V, F = poly(a, t, hulls)
    if b[0] in (HULL, CUBOID):
        W, G = poly(b, t, hulls)
        if hr.sat(V, F, W, G)[0] <= 0:
            return 0.0
        return hr.distance(V, F, W, G)
    p0, p1, r = caps.core(b, t)
    if b[0] == SPHERE:
        return max(hr.point_distance(p0, V, F) - r, 0.0)
    return max(hr.segment_distance(p0, p1, V, F) - r, 0.0)


def dims_of(rng, shape, hulls=HULLS):
    if shape == HULL:
        return np.array([float(rng.integers(hulls.count)), 0, 0])
    return caps.dims_of(rng, shape)


def random_pair(rng, spin=True, kinds=None):
    """a moving, spinning pair with at least one hull whose swept volumes may meet within DT; off-origin centres of mass on both sides"""
    sa, sb = PAIRS[rng.integers(len(PAIRS))] if kinds is None else kinds
    pb = rng.normal(size=3) * 2.5
    va = pb * rng.uniform(0, 90) + rng.normal(size=3) * 10
    a = fixture.ccd_motion(sa, dims_of(rng, sa), np.zeros(3), caps.rq(rng), va, rng.normal(size=3) * (40 if spin else 0), rng.normal(size=3) * 0.05)
    b = fixture.ccd_motion(sb, dims_of(rng, sb), pb, caps.rq(rng), rng.normal(size=3) * 5, rng.normal(size=3) * (20 if spin else 0),
                           rng.normal(size=3) * 0.05)
    return a, b


# ---- the non-linear contract -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [1, 2])
def test_nonlinear_toi_contract(seed):
    rng = np.random.default_rng(seed)
    t64 = table()
    hits = misses = capped = 0
    kinds = set()
    for _ in range(90):
        a, b = random_pair(rng)
        if distance(a, b, 0.0) <= EPS:
            continue
        t, its = fixture.ccd_nonlinear_toi(a, b, DT, EPS, iterations=True, hulls=t64)
        samples = np.linspace(0.0, DT if t is None else t, 24, endpoint=t is None)
        d = np.array([distance(a, b, s) for s in samples])
        if t is None:
            misses += 1
            assert (d > 0).all(), "no hit reported, yet the shapes touch on [0, dt]"
            continue
        hits += 1
        kinds.add((int(a[0]), int(b[0])))
        assert (d > 0).all(), "contact before the reported TOI (tunnelling)"
        if its == 64:
            capped += 1
            continue
        assert distance(a, b, t) <= EPS + 1e-9
    assert hits > 12 and misses > 3 and capped <= hits // 4
    assert len(kinds) == len(PAIRS), kinds


@pytest.mark.parametrize("scalar", SCALARS)
def test_pair_toi_rounds_the_nonlinear_toi_and_both_orders_agree(scalar):
    rng = np.random.default_rng(4)
    t64 = table(scalar)
    n = 0
    for _ in range(80):
        a, b = random_pair(rng)
        got = fixture.ccd_pair_toi(scalar, api.SWEEP_NON_LINEAR, a, b, DT, EPS, hulls=t64)
        raw = fixture.ccd_nonlinear_toi(a, b, DT, EPS, hulls=t64)
        if raw is None:
            assert got == -1.0
            continue
        if scalar(raw) == 0:
            continue   # the fallback's domain
        assert got == float(scalar(raw))
        # the swapped order sweeps the same pair: the distance and its direction are symmetric, the iterates nearly so
        back = fixture.ccd_nonlinear_toi(b, a, DT, EPS, hulls=t64)
        assert back is not None and abs(back - raw) <= 1e-3 * DT
        n += 1
    assert n > 10


# ---- the linear mode -------------------------------------------------------------------------------------------------------------------
def cast(scalar, a, b, hulls):
    """shape A along v1 - v2 against collider B at rest, as a hull spatial-query cast with max distance dt"""
    cols = api.QueryColliders(shape=np.array([b[0]], np.uint8), dims=b[1:4][None], position=b[4:7][None], rotation=b[7:11][None])
    shapes = api.ShapeQueries(shape=np.array([a[0]], np.uint8), dims=a[1:4][None], position=a[4:7][None], rotation=a[7:11][None],
                              direction=(a[14:17] - b[14:17])[None], max_distance=np.array([DT]))
    got = fixture.query_cast_shape(np.float64, cols, shapes, hulls=hulls)
    return None if got["collider"][0] < 0 else float(got["distance"][0])


@pytest.mark.parametrize("scalar", SCALARS)
def test_linear_toi_is_the_hull_cast_of_the_relative_motion(scalar):
    rng = np.random.default_rng(3)
    t64 = table()
    n = lp = 0
    for _ in range(250):
        a, b = random_pair(rng, spin=False)
        want = fixture.ccd_pair_toi(scalar, api.SWEEP_LINEAR, a, b, DT, hulls=t64)
        t = cast(scalar, a, b, t64)
        if t is None:
            assert want == -1.0
            continue
        if scalar(t) == 0:
            continue   # the zero-TOI fallback, below
        assert want == float(scalar(t))
        n += 1
        if a[0] in (HULL, CUBOID) and b[0] in (HULL, CUBOID):
            # two polytopes: the linear program of tests/hull_query_reference.py
            VA, FA = poly(dict_static(a), 0.0)
            VB, FB = poly(dict_static(b), 0.0)
            ref_t = hq.poly_cast_lp(VA, FA, VB, FB, a[14:17] - b[14:17], DT)
            assert ref_t is not None and abs(ref_t - t) <= 1e-7 + 1e-6 * t
            lp += 1
    assert n > 20 and lp > 5


def dict_static(m):
    """a motion record with its velocities cleared (its pose at t = 0 for any t)"""
    s = m.copy()
    s[14:20] = 0
    return s


def test_zero_toi_fallback_is_a_hull_sphere_pair():
    t64 = table()
    a = fixture.ccd_motion(HULL, (2, 0, 0), (0, 0, 0), (0, 0, 0, 1), (30.0, 0, 0))
    b = fixture.ccd_motion(HULL, (3, 0, 0), (0.3, 0, 0), (0, 0, 0, 1))   # overlapping at t = 0
    ball = b.copy()
    ball[0], ball[1:4] = SPHERE, (0.05, 0, 0)
    for mode in (api.SWEEP_LINEAR, api.SWEEP_NON_LINEAR):
        got = fixture.ccd_pair_toi(np.float64, mode, a, b, DT, EPS, 0.05, hulls=t64)
        want = fixture.ccd_pair_toi(np.float64, mode, a, ball, DT, EPS, 0.05, hulls=t64)
        assert got == want


# ---- known answers ---------------------------------------------------------------------------------------------------------------------
def box_hulls(he):
    V, F = hr.box_poly(he, np.zeros(3), np.array([0, 0, 0, 1.0]))
    return api.ConvexHulls.from_polyhedra([(V, F)])


def test_spinning_plank_as_a_hull():
    # test_ccd_world_cpu.test_spinning_plank's plank as an 8-vertex hull: the touch at 0.4 rad, and no linear hit (it does not translate)
    hulls = box_hulls((2.0, 0.05, 0.05))
    plank = fixture.ccd_motion(HULL, (0, 0, 0), (0, 0, 0), (0, 0, 0, 1), (0, 0, 0), (0, 0, 60.0))
    target = fixture.ccd_motion(SPHERE, (0.1, 0, 0), (1.5 * np.cos(0.5), 1.5 * np.sin(0.5), 0), (0, 0, 0, 1))
    for scalar in SCALARS:
        t_h = table(scalar, hulls)
        assert fixture.ccd_pair_toi(scalar, api.SWEEP_LINEAR, plank, target, DT, hulls=t_h) == -1.0
        t = fixture.ccd_pair_toi(scalar, api.SWEEP_NON_LINEAR, plank, target, DT, hulls=t_h)
        assert 0 < t < DT and abs(60.0 * t - 0.4) < 1e-3
        assert distance(plank, target, float(t), hulls) <= EPS * 1.1


@pytest.mark.parametrize("mode", [api.SWEEP_LINEAR, api.SWEEP_NON_LINEAR])
def test_tetrahedron_falls_vertex_first_onto_a_slab(mode):
    # a regular tetrahedron of circumradius 0.5 with one vertex straight down, 2 m above a slab's top, falling at 50 m/s: the vertex
    # reaches the top at t = 2 / 50 minus the eps of the non-linear stop
    R = 0.5
    top = np.array([0, 0, 1.0])
    base = [np.array([np.cos(a), np.sin(a), 0]) * (2 * np.sqrt(2) / 3) + np.array([0, 0, -1 / 3]) for a in (0, 2 * np.pi / 3, 4 * np.pi / 3)]
    V = np.array([top] + base) * R
    V = V[:, [0, 2, 1]] * np.array([1, -1, 1])       # vertex 0 now points down (-y)
    V, F = scenes.convex_hull_of(V)
    hulls = api.ConvexHulls.from_polyhedra([(V, F)])
    low = V[:, 1].min()
    tet = fixture.ccd_motion(HULL, (0, 0, 0), (0, 2.0 - low, 0), (0, 0, 0, 1), (0, -50.0, 0))
    slab = fixture.ccd_motion(CUBOID, (3, 0.1, 3), (0, -0.1, 0), (0, 0, 0, 1))
    want = 2.0 / 50.0
    for scalar in SCALARS:
        t = fixture.ccd_pair_toi(scalar, mode, tet, slab, 0.1, EPS, hulls=table(scalar, hulls))
        tol = 1e-6 if mode == api.SWEEP_LINEAR else EPS / 50.0 + 1e-6
        assert want - tol <= t <= want + 1e-6, (t, want)


@pytest.mark.parametrize("mode", [api.SWEEP_LINEAR, api.SWEEP_NON_LINEAR])
def test_unit_cube_hull_matches_the_cuboid(mode):
    hulls = box_hulls((0.5, 0.5, 0.5))
    t64 = table(np.float64, hulls)
    rng = np.random.default_rng(17)
    n = 0
    for _ in range(120):
        a, b = random_pair(rng, spin=mode == api.SWEEP_NON_LINEAR, kinds=(CUBOID, [CUBOID, SPHERE, CAPSULE][rng.integers(3)]))
        a[1:4] = 0.5
        h = a.copy()
        h[0], h[1:4] = HULL, (0, 0, 0)
        t_box = fixture.ccd_pair_toi(np.float64, mode, a, b, DT, EPS)
        t_hull = fixture.ccd_pair_toi(np.float64, mode, h, b, DT, EPS, hulls=t64)
        assert (t_box < 0) == (t_hull < 0), (t_box, t_hull)
        if t_box > 0:
            n += 1
            assert abs(t_box - t_hull) <= (1e-9 + 1e-7 * t_box if mode == api.SWEEP_LINEAR else 2e-3 * DT)
    assert n > 10


# ---- the spin bound --------------------------------------------------------------------------------------------------------------------
def test_motion_radius_bounds_vertices_and_face_plane_polytope():
    from scipy.spatial import HalfspaceIntersection
    d = table().derived()
    rng = np.random.default_rng(9)
    for h in range(HULLS.count):
        V, F = hq.table_poly(HULLS, h)
        pl = d["plane"][int(HULLS.face_offsets[h]):int(HULLS.face_offsets[h + 1])]
        hs = np.concatenate([pl[:, :3], -pl[:, 3:4]], axis=1)        # n . x - d <= 0
        P = HalfspaceIntersection(hs, np.asarray(V).mean(axis=0)).intersections
        for lc in (np.zeros(3), rng.normal(size=3) * 0.1):
            R = fixture.ccd_motion_radius(fixture.ccd_motion(HULL, (h, 0, 0), (0, 0, 0), (0, 0, 0, 1), com=lc), hulls=table())
            assert np.linalg.norm(V - lc, axis=1).max() <= R
            assert np.linalg.norm(P - lc, axis=1).max() <= R
    # the other shapes keep their bounds
    for shape, dims in ((CUBOID, (0.3, 0.2, 0.1)), (SPHERE, (0.4, 0, 0)), (CAPSULE, (0.1, 0.5, 0))):
        m = fixture.ccd_motion(shape, dims, (0, 0, 0), (0, 0, 0, 1), com=(0.05, 0, 0))
        assert fixture.ccd_motion_radius(m, hulls=table()) == fixture.ccd_motion_radius(m)


# ---- control flow and refusals ---------------------------------------------------------------------------------------------------------
def hull_world(rng, n, scalar, capsules=True):
    bodies, shape, dims, rows = caps.capsule_world(rng, n, scalar)
    hull = rng.random(n) < 0.5
    shape = np.where(hull, HULL, shape if capsules else np.minimum(shape, SPHERE)).astype(np.uint8)
    dims = dims.astype(np.float64)
    dims[hull] = 0
    dims[hull, 0] = rng.integers(0, HULLS.count, hull.sum())
    dims[shape == SPHERE] = [0.3, 0, 0]
    return bodies, shape, dims.astype(scalar), rows


def run_both(scalar, bodies, shape, dims, rows, cfg, prediction=np.inf):
    """avh_ccd_solve_hulls against tests/ccd_reference.py's loop over the G = 2 pair TOIs: the same decisions and the same bits"""
    n = bodies["position"].shape[0]
    t_s = table(scalar)
    dp0 = np.zeros((n, 3), scalar)
    dq0 = np.tile(np.array([0, 0, 0, 1], scalar), (n, 1))
    dp_f, dq_f = dp0.copy(), dq0.copy()
    got = fixture.ccd_solve(scalar, DT, 1.0, bodies, shape, dims, rows, dict(cfg, prediction_distance=prediction), dp_f, dq_f, hulls=t_s)

    def motion(b, c):
        still = bodies["kind"][b] == 2
        return fixture.ccd_motion(shape[c], dims[c], bodies["position"][b], bodies["rotation"][b], (0, 0, 0) if still else bodies["linear_velocity"][b],
                                  (0, 0, 0) if still else bodies["angular_velocity"][b])

    def pair_toi(mode, b1, c1, b2, c2):
        return fixture.ccd_pair_toi(scalar, mode, motion(b1, c1), motion(b2, c2), DT, EPS, prediction, hulls=t_s)

    def apply(m, v, w, dp, dq):
        p, q = fixture.ccd_apply_record(scalar, float(m), v, w, dp, dq)
        return p.astype(scalar), q.astype(scalar)

    k = len(cfg["body"])
    ccd_bodies = [dict(body=int(cfg["body"][i]), collider=int(cfg["collider"][i]), mode=int(cfg["mode"][i]), include_dynamic=bool(cfg["include_dynamic"][i]),
                       linear_threshold=cfg["linear_threshold"][i], angular_threshold=cfg["angular_threshold"][i]) for i in range(k)]
    live_rows = [(int(e), int(rows["c1"][e]), int(rows["c2"][e]), int(rows["b1"][e]), int(rows["b2"][e])) for e in range(len(rows["c1"])) if rows["live"][e]]
    dp_r, dq_r = dp0.copy(), dq0.copy()
    want, writes = ref.solve_swept_ccd(scalar, DT, ccd_bodies, live_rows, bodies["kind"], bodies["linear_velocity"], bodies["angular_velocity"], dp_r, dq_r,
                                       pair_toi, apply)
    assert np.array_equal(got["min_toi"], np.array([w[0] for w in want], scalar))
    assert np.array_equal(got["hit_body"], np.array([w[1] for w in want]))
    assert np.array_equal(got["hit_contact"], np.array([w[2] for w in want]))
    assert np.array_equal(dp_f.view(np.uint8), dp_r.view(np.uint8)) and np.array_equal(dq_f.view(np.uint8), dq_r.view(np.uint8))
    return got, writes


def world_config(rng, n, k=10):
    body = rng.choice(n, size=k, replace=False)
    return dict(body=body, collider=body, mode=rng.integers(0, 2, k), include_dynamic=rng.integers(0, 2, k),
                linear_threshold=rng.choice([0.0, 50.0, 200.0], k), angular_threshold=rng.choice([0.0, 20.0, 80.0], k), capsules=True, hulls=True)


@pytest.mark.parametrize("scalar", SCALARS)
@pytest.mark.parametrize("seed", [41, 42])
def test_control_flow_matches_reference(scalar, seed):
    rng = np.random.default_rng(seed)
    bodies, shape, dims, rows = hull_world(rng, 24, scalar)
    cfg = world_config(rng, 24)
    got, writes = run_both(scalar, bodies, shape, dims, rows, cfg)
    hull_hits = [int(b) for b, h in zip(cfg["body"], got["hit_body"]) if h >= 0 and (shape[b] == HULL or shape[h] == HULL)]
    assert hull_hits and len(writes) >= 1, "no pair with a hull was hit"
    run_both(scalar, bodies, shape, dims, rows, cfg, prediction=0.05)


def test_flags_and_refusals():
    rng = np.random.default_rng(43)
    scalar = np.float32
    bodies, shape, dims, rows = hull_world(rng, 16, scalar)
    cfg = world_config(rng, 16, 8)
    t_s = table(scalar)
    fixture.ccd_solve(scalar, DT, 1.0, bodies, shape, dims, rows, cfg, hulls=t_s)
    # without AVN_CCD_HULLS the hull rows are refused as before, with or without AVN_CCD_CAPSULES and with or without a table
    for extra in (dict(hulls=False), dict(hulls=False, capsules=False)):
        for h in (None, t_s):
            with pytest.raises(api.AvianError) as e:
                fixture.ccd_solve(scalar, DT, 1.0, bodies, shape, dims, rows, dict(cfg, **extra), hulls=h)
            assert e.value.status == api.ERR_UNSUPPORTED
    # a store with hulls and capsules needs both bits
    assert (shape == CAPSULE).any()
    with pytest.raises(api.AvianError) as e:
        fixture.ccd_solve(scalar, DT, 1.0, bodies, shape, dims, rows, dict(cfg, capsules=False), hulls=t_s)
    assert e.value.status == api.ERR_UNSUPPORTED
    # the flag with no table, or an index past the table: refused as the contact step refuses the column
    with pytest.raises(ValueError):
        fixture.ccd_solve(scalar, DT, 1.0, bodies, shape, dims, rows, cfg)
    bad = dims.copy()
    bad[shape == HULL, 0] = HULLS.count
    with pytest.raises(ValueError):
        fixture.ccd_solve(scalar, DT, 1.0, bodies, shape, bad, rows, cfg, hulls=t_s)
    # 0x2 stays an unknown bit, alone and beside the known ones
    for flags in (0x2, 0x3, 0x6, 0x7):
        with pytest.raises(ValueError):
            fixture.ccd_solve(scalar, DT, 1.0, bodies, shape, dims, rows, dict(body=[0], collider=[0], flags=flags), hulls=t_s)


@pytest.mark.parametrize("scalar", SCALARS)
def test_flag_without_hulls_changes_nothing(scalar):
    rng = np.random.default_rng(12)
    bodies, shape, dims, rows = caps.capsule_world(rng, 24, scalar)
    body = rng.choice(24, size=10, replace=False)
    cfg = dict(body=body, collider=body, mode=rng.integers(0, 2, 10), capsules=True)
    plain = fixture.ccd_solve(scalar, DT, 1.0, bodies, shape, dims, rows, cfg)
    flagged = fixture.ccd_solve(scalar, DT, 1.0, bodies, shape, dims, rows, dict(cfg, hulls=True), hulls=table(scalar))
    for k in plain:
        assert np.array_equal(plain[k].view(np.uint8), flagged[k].view(np.uint8)), k


def test_header_flag_and_reference_config():
    from avian_b200 import _build
    text = (_build.REPO / "include" / "avian_b200.h").read_text()
    assert "#define AVN_CCD_HULLS 0x4u" in text
    assert api.CCD_HULLS == 0x4
    cfg, _ = api.ccd_config([1], [1], flags=api.CCD_CAPSULES | api.CCD_HULLS)
    assert cfg.flags == 0x5
    import oracle_ccd
    assert oracle_ccd.bodies_as_ref_config(dict(body=[3], collider=[4])) == oracle_ccd.bodies_as_ref_config(dict(body=[3], collider=[4], hulls=True))
