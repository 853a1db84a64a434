"""Swept CCD without a GPU: the TOI geometry of csrc/ccd_math.hpp against tests/narrow_reference.py's float64 distances, and the host brute force's
control flow (avh_ccd_solve) against tests/ccd_reference.py, a plain-Python restatement of solve_swept_ccd."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import ccd_reference as ref
import narrow_reference as nr
from avian_b200 import api, fixture

DT = 1.0 / 60.0
EPS = 1e-4
CUBOID, SPHERE = 0, 1


def qmul(a, b):
    return np.array([a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1], a[3] * b[1] - a[0] * b[2] + a[1] * b[3] + a[2] * b[0],
                     a[3] * b[2] + a[0] * b[1] - a[1] * b[0] + a[2] * b[3], a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2]])


def pose(m, t):
    """The non-linear motion of a 20-double motion record at time t, in float64 (origin follows the com)."""
    he, p, q, lc, v, w = m[1:4], m[4:7], m[7:11], m[11:14], m[14:17], m[17:20]
    a = w * t
    ang = np.linalg.norm(a)
    dq = np.array([0, 0, 0, 1.0]) if ang == 0 else np.concatenate([a / ang * np.sin(ang / 2), [np.cos(ang / 2)]])
    qt = qmul(dq, q)
    com = p + nr.rotation(q) @ lc + v * t
    R = nr.rotation(qt)
    return com - R @ lc, R


def distance(a, b, t):
    """Exact float64 distance of the two shapes at time t (0 when they overlap)."""
    ca, Ra = pose(a, t)
    cb, Rb = pose(b, t)
    if a[0] == SPHERE and b[0] == SPHERE:
        return max(nr.sphere_sphere(ca, a[1], cb, b[1])[1], 0.0)
    if a[0] == SPHERE or b[0] == SPHERE:
        (cbx, Rbx, hbx), (cs, rs) = ((ca, Ra, a[1:4]), (cb, b[1])) if b[0] == SPHERE else ((cb, Rb, b[1:4]), (ca, a[1]))
        return max(nr.sphere_box(cbx, Rbx, np.asarray(hbx), cs, rs)[1], 0.0)
    if nr.sat(ca, Ra, a[1:4], cb, Rb, b[1:4])[0] >= 0:
        return 0.0
    return nr.box_box_distance(ca, Ra, a[1:4], cb, Rb, b[1:4])[0]


def random_pair(rng, spin=True):
    """A moving, spinning pair whose swept volumes may meet within DT."""
    def rq():
        q = rng.normal(size=4)
        return q / np.linalg.norm(q)
    shapes = rng.integers(0, 2, size=2)
    dims = [np.array([rng.uniform(0.1, 0.6), 0, 0]) if s == SPHERE else rng.uniform(0.05, 1.5, 3) for s in shapes]
    pa = np.zeros(3)
    pb = rng.normal(size=3) * 2.5
    va = (pb - pa) * rng.uniform(0, 90) + rng.normal(size=3) * 10
    wa = rng.normal(size=3) * (40 if spin else 0)
    wb = rng.normal(size=3) * (20 if spin else 0)
    a = fixture.ccd_motion(shapes[0], dims[0], pa, rq(), va, wa, rng.normal(size=3) * 0.05)
    b = fixture.ccd_motion(shapes[1], dims[1], pb, rq(), rng.normal(size=3) * 5, wb)
    return a, b


@pytest.mark.parametrize("seed", [1, 2])
def test_nonlinear_toi_contract(seed):
    rng = np.random.default_rng(seed)
    hits = misses = 0
    for _ in range(150):
        a, b = random_pair(rng)
        if distance(a, b, 0.0) <= EPS:
            continue
        t = fixture.ccd_nonlinear_toi(a, b, DT, EPS)
        samples = np.linspace(0.0, DT if t is None else t, 200, endpoint=t is None)
        d = np.array([distance(a, b, s) for s in samples])
        if t is None:
            misses += 1
            assert (d > 0).all(), "no hit reported, yet the shapes touch on [0, dt]"
        else:
            hits += 1
            assert (d > 0).all(), "contact before the reported TOI (tunnelling)"
            assert distance(a, b, t) <= EPS + 1e-9
    assert hits > 10 and misses > 10


def test_nonlinear_without_spin_agrees_with_linear():
    # never later than the linear TOI, and whenever the advancement reached eps the true distance there is <= eps.  (Within eps / |v_rel| of the
    # linear TOI holds only for head-on approaches: a glancing one closes the distance slower than |v_rel|.)  A run that hits the iteration cap
    # reports an earlier t (DESIGN.md §7e); those are counted apart
    rng = np.random.default_rng(7)
    n = capped = head_on = 0
    for _ in range(300):
        a, b = random_pair(rng, spin=False)
        lin = fixture.ccd_pair_toi(np.float64, api.SWEEP_LINEAR, a, b, DT)
        if lin <= 0:
            continue
        nl, its = fixture.ccd_nonlinear_toi(a, b, DT, EPS, iterations=True)
        assert nl is not None
        assert nl <= lin + 1e-12
        if its == 64:
            capped += 1
            continue
        assert distance(a, b, nl) <= EPS + 1e-9
        speed = np.linalg.norm(a[14:17] - b[14:17])
        head_on += nl >= lin - EPS / speed - 1e-12
        n += 1
    assert n > 20 and capped <= n // 5 and head_on >= n // 2


@pytest.mark.parametrize("scalar", [np.float32, np.float64])
def test_rounded_nonlinear_toi_contract(scalar):
    """The value the pass uses: pair_toi rounded to the column scalar.  Never later than contact (no contact on [0, toi]), and within eps plus
    the rounding of t (|v_rel| + spin radius times half an ulp of t) of touching there."""
    rng = np.random.default_rng(5)
    hits = 0
    for _ in range(150):
        a, b = random_pair(rng)
        if distance(a, b, 0.0) <= EPS:
            continue
        t = fixture.ccd_pair_toi(scalar, api.SWEEP_NON_LINEAR, a, b, DT, EPS)
        if not 0 < t < DT:
            continue
        hits += 1
        raw = fixture.ccd_nonlinear_toi(a, b, DT, EPS)
        rate = np.linalg.norm(a[14:17] - b[14:17]) + 4 * (np.linalg.norm(a[17:20]) + np.linalg.norm(b[17:20]))
        slack = rate * abs(t - raw)
        assert min(distance(a, b, s) for s in np.linspace(0.0, min(t, raw), 100)) > 0 or slack > 0
        assert distance(a, b, t) <= EPS + slack + 1e-9
    assert hits > 10


@pytest.mark.parametrize("scalar", [np.float32, np.float64])
def test_linear_toi_is_the_shape_cast_of_the_relative_motion(scalar):
    rng = np.random.default_rng(3)
    n = 0
    for _ in range(200):
        a, b = random_pair(rng, spin=False)
        want = fixture.ccd_pair_toi(scalar, api.SWEEP_LINEAR, a, b, DT)
        # the same pair as a spatial-query cast: shape A along v1 - v2 against collider B, max distance dt
        cols = api.QueryColliders(shape=np.array([b[0]], np.uint8), dims=b[1:4][None], position=b[4:7][None], rotation=b[7:11][None])
        shapes = api.ShapeQueries(shape=np.array([a[0]], np.uint8), dims=a[1:4][None], position=a[4:7][None], rotation=a[7:11][None],
                                  direction=(a[14:17] - b[14:17])[None], max_distance=np.array([DT]))
        got = fixture.query_cast_shape(np.float64, cols, shapes)
        if got["collider"][0] < 0:
            assert want == -1.0
            continue
        t = scalar(got["distance"][0])
        if t == 0:
            continue   # the fallback's domain
        assert want == float(t)
        n += 1
    assert n > 10


def test_spinning_plank_and_fast_sphere():
    plank = fixture.ccd_motion(CUBOID, (2.0, 0.05, 0.05), (0, 0, 0), (0, 0, 0, 1), (0, 0, 0), (0, 0, 60.0))
    # the plank's end sweeps 1 rad in dt: a small sphere at 0.5 rad, radius 1.5, lies inside the swept disc
    target = fixture.ccd_motion(SPHERE, (0.1, 0, 0), (1.5 * np.cos(0.5), 1.5 * np.sin(0.5), 0), (0, 0, 0, 1))
    assert fixture.ccd_pair_toi(np.float32, api.SWEEP_LINEAR, plank, target, DT) == -1.0     # linear: passes through
    t = fixture.ccd_pair_toi(np.float32, api.SWEEP_NON_LINEAR, plank, target, DT)
    assert 0 < t < DT and abs(60.0 * t - 0.4) < 1e-3                                          # touches at 0.4 rad
    assert distance(plank, target, t * 1.0001) <= EPS * 1.1 or distance(plank, target, t) <= EPS
    bullet = fixture.ccd_motion(SPHERE, (0.05, 0, 0), (0, 0, 0), (0, 0, 0, 1), (300.0, 0, 0))
    wall = fixture.ccd_motion(CUBOID, (0.02, 3, 3), (4.0, 0, 0), (0, 0, 0, 1))
    for mode in (api.SWEEP_LINEAR, api.SWEEP_NON_LINEAR):
        t = fixture.ccd_pair_toi(np.float64, mode, bullet, wall, DT)
        assert abs(t * 300.0 - (4.0 - 0.02 - 0.05)) <= 1e-3


# ---- control flow ------------------------------------------------------------------------------------------------------------------------
def random_world(rng, n, scalar):
    kind = rng.choice([0, 0, 0, 1, 2], size=n).astype(np.uint8)
    shape = rng.integers(0, 2, size=n).astype(np.uint8)
    dims = np.where(shape[:, None] == SPHERE, np.array([[0.3, 0, 0]]), rng.uniform(0.2, 0.8, (n, 3))).astype(scalar)
    pos = (rng.normal(size=(n, 3)) * 4).astype(scalar)
    q = rng.normal(size=(n, 4))
    rot = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(scalar)
    lv = (-pos * rng.uniform(20, 80, (n, 1)) + rng.normal(size=(n, 3)) * 30).astype(scalar)   # converging on the origin
    av = (rng.normal(size=(n, 3)) * 30).astype(scalar)
    lv[kind == 2] = 0
    av[kind == 2] = 0
    pairs = [(i, j) for i in range(n) for j in range(i + 1, n) if rng.random() < 0.5]
    rows = {"c1": np.array([p[0] for p in pairs], np.uint32), "c2": np.array([p[1] for p in pairs], np.uint32)}
    rows["b1"], rows["b2"] = rows["c1"].copy(), rows["c2"].copy()
    rows["live"] = (rng.random(len(pairs)) < 0.9).astype(np.uint8)
    return dict(kind=kind, position=pos, rotation=rot, linear_velocity=lv, angular_velocity=av), shape, dims, rows


def run_both(scalar, bodies, shape, dims, rows, cfg, prediction=np.inf):
    n = bodies["position"].shape[0]
    dp0 = np.zeros((n, 3), scalar)
    dq0 = np.tile(np.array([0, 0, 0, 1], scalar), (n, 1))
    dp_f, dq_f = dp0.copy(), dq0.copy()
    got = fixture.ccd_solve(scalar, DT, 1.0, bodies, shape, dims, rows, dict(cfg, prediction_distance=prediction), dp_f, dq_f)

    def motion(b, c):
        return fixture.ccd_motion(shape[c], dims[c], bodies["position"][b], bodies["rotation"][b],
                                  bodies["linear_velocity"][b] if bodies["kind"][b] != 2 else (0, 0, 0),
                                  bodies["angular_velocity"][b] if bodies["kind"][b] != 2 else (0, 0, 0))

    def pair_toi(mode, b1, c1, b2, c2):
        return fixture.ccd_pair_toi(scalar, mode, motion(b1, c1), motion(b2, c2), DT, EPS, prediction)

    def apply(m, v, w, dp, dq):
        p, q = fixture.ccd_apply_record(scalar, float(m), v, w, dp, dq)
        return p.astype(scalar), q.astype(scalar)

    ccd_bodies = [dict(body=int(b), collider=int(c), mode=int(cfg["mode"][k]) if cfg.get("mode") is not None else ref.NON_LINEAR,
                       include_dynamic=bool(cfg["include_dynamic"][k]) if cfg.get("include_dynamic") is not None else True,
                       linear_threshold=cfg["linear_threshold"][k] if cfg.get("linear_threshold") is not None else 0.0,
                       angular_threshold=cfg["angular_threshold"][k] if cfg.get("angular_threshold") is not None else 0.0)
                  for k, (b, c) in enumerate(zip(cfg["body"], cfg["collider"]))]
    order = np.arange(len(rows["c1"]))   # ascending ContactId: the fixture's (and the device's) tie rule
    live_rows = [(int(e), int(rows["c1"][e]), int(rows["c2"][e]), int(rows["b1"][e]), int(rows["b2"][e])) for e in order if rows["live"][e]]
    dp_r, dq_r = dp0.copy(), dq0.copy()
    want, writes = ref.solve_swept_ccd(scalar, DT, ccd_bodies, live_rows, bodies["kind"], bodies["linear_velocity"], bodies["angular_velocity"], dp_r, dq_r,
                                       pair_toi, apply)
    assert np.array_equal(got["min_toi"], np.array([w[0] for w in want], scalar))
    assert np.array_equal(got["hit_body"], np.array([w[1] for w in want]))
    assert np.array_equal(got["hit_contact"], np.array([w[2] for w in want]))
    assert np.array_equal(dp_f.view(np.uint8), dp_r.view(np.uint8)) and np.array_equal(dq_f.view(np.uint8), dq_r.view(np.uint8))
    return got, writes, dp_f, dq_f


@pytest.mark.parametrize("scalar", [np.float32, np.float64])
@pytest.mark.parametrize("seed", [11, 12, 13])
def test_control_flow_matches_reference(scalar, seed):
    rng = np.random.default_rng(seed)
    bodies, shape, dims, rows = random_world(rng, 24, scalar)
    k = 10
    body = rng.choice(24, size=k, replace=False)
    cfg = dict(body=body, collider=body, mode=rng.integers(0, 2, k), include_dynamic=rng.integers(0, 2, k),
               linear_threshold=rng.choice([0.0, 50.0, 200.0], k), angular_threshold=rng.choice([0.0, 20.0, 80.0], k))
    got, writes, _, _ = run_both(scalar, bodies, shape, dims, rows, cfg)
    assert (got["hit_body"] >= 0).sum() >= 2 and len(writes) >= 2
    # finite prediction distance: the fallback can produce hits
    run_both(scalar, bodies, shape, dims, rows, cfg, prediction=0.05)


def two_body_scene(scalar, kind2, v1=(300.0, 0, 0)):
    bodies = dict(kind=np.array([0, kind2], np.uint8), position=np.array([[0, 0, 0], [4.0, 0, 0]], scalar),
                  rotation=np.array([[0, 0, 0, 1], [0, 0, 0, 1]], scalar), linear_velocity=np.array([v1, [-10.0, 0, 0] if kind2 != 2 else [0, 0, 0]], scalar),
                  angular_velocity=np.zeros((2, 3), scalar))
    rows = dict(c1=np.array([0], np.uint32), c2=np.array([1], np.uint32), b1=np.array([0], np.uint32), b2=np.array([1], np.uint32), live=np.array([1], np.uint8))
    return bodies, np.array([SPHERE, CUBOID], np.uint8), np.array([[0.1, 0, 0], [0.02, 2, 2]], scalar), rows


@pytest.mark.parametrize("kind2", [0, 1, 2])
def test_static_kinematic_dynamic_body2_and_overshoot(kind2):
    s = np.float32
    bodies, shape, dims, rows = two_body_scene(s, kind2)
    got, writes, dp, dq = run_both(s, bodies, shape, dims, rows, dict(body=[0], collider=[0]))
    t = got["min_toi"][0]
    assert got["hit_body"][0] == 1 and 0 < t < s(DT)
    m = s(t * s(1.0001))
    assert np.array_equal(dp[0], m * bodies["linear_velocity"][0])
    assert [b for b, _ in writes] == ([0] if kind2 == 2 else [0, 1])   # a static body 2 is the dummy: not written, a kinematic one is
    if kind2 == 0:   # include_dynamic = 0 skips a dynamic body 2
        got, _, _, _ = run_both(s, bodies, shape, dims, rows, dict(body=[0], collider=[0], include_dynamic=[0]))
        assert got["hit_body"][0] == -1 and got["min_toi"][0] == s(DT)


def test_thresholds_and_mixed_modes():
    s = np.float64
    bodies, shape, dims, rows = two_body_scene(s, 0)
    # both comparisons must hold to skip: |w1 - w2|^2 = 0 < 0 fails, so a linear threshold alone skips nothing
    got, _, _, _ = run_both(s, bodies, shape, dims, rows, dict(body=[0], collider=[0], linear_threshold=[400.0]))
    assert got["hit_body"][0] == 1 and got["candidates"][0] == 1
    got, _, _, _ = run_both(s, bodies, shape, dims, rows, dict(body=[0], collider=[0], linear_threshold=[400.0], angular_threshold=[1.0]))
    assert got["hit_body"][0] == -1 and got["candidates"][0] == 0
    got, _, _, _ = run_both(s, bodies, shape, dims, rows, dict(body=[0], collider=[0], linear_threshold=[300.0], angular_threshold=[1.0]))
    assert got["candidates"][0] == 1   # |v1 - v2| = 310
    # body 1 Linear, body 2 NonLinear: the pair sweeps NonLinear; body 2 Linear too: Linear
    a = fixture.ccd_motion(SPHERE, dims[0], bodies["position"][0], bodies["rotation"][0], bodies["linear_velocity"][0])
    b = fixture.ccd_motion(CUBOID, dims[1], bodies["position"][1], bodies["rotation"][1], bodies["linear_velocity"][1])
    lin, nl = (fixture.ccd_pair_toi(s, m, a, b, DT, EPS) for m in (api.SWEEP_LINEAR, api.SWEEP_NON_LINEAR))
    assert lin != nl
    got, _, _, _ = run_both(s, bodies, shape, dims, rows, dict(body=[0, 1], collider=[0, 1], mode=[api.SWEEP_LINEAR, api.SWEEP_NON_LINEAR]))
    assert got["min_toi"][0] == nl
    got, _, _, _ = run_both(s, bodies, shape, dims, rows, dict(body=[0, 1], collider=[0, 1], mode=[api.SWEEP_LINEAR, api.SWEEP_LINEAR]))
    assert got["min_toi"][0] == lin


@pytest.mark.parametrize("scalar", [np.float32, np.float64])
def test_zero_toi_fallback(scalar):
    bodies, shape, dims, rows = two_body_scene(scalar, 2)
    bodies["position"][1] = (0.1, 0, 0)   # the sphere starts inside the wall: TOI 0
    got, _, _, _ = run_both(scalar, bodies, shape, dims, rows, dict(body=[0], collider=[0]))
    assert got["hit_body"][0] == -1      # infinite prediction distance: the ball retry gives 0 as well
    got, _, _, _ = run_both(scalar, bodies, shape, dims, rows, dict(body=[0], collider=[0]), prediction=0.5)
    assert got["hit_body"][0] == -1      # the ball of radius 0.5 around the wall's origin already holds the sphere at t = 0
    bodies["position"][0] = (-1.0, 0, 0)
    bodies["position"][1] = (0.0, 0, 0)
    dims[1] = (3.0, 2, 2)                 # overlapping at t = 0, the small ball around the wall's origin is ahead
    got, _, _, _ = run_both(scalar, bodies, shape, dims, rows, dict(body=[0], collider=[0]), prediction=0.2)
    assert got["hit_body"][0] == 1 and 0 < got["min_toi"][0] < scalar(DT)


def test_equal_tois_keep_the_first_contact():
    s = np.float32
    bodies = dict(kind=np.array([0, 2, 2], np.uint8), position=np.array([[0, 0, 0], [3, 1, 0], [3, -1, 0]], s),
                  rotation=np.tile(np.array([0, 0, 0, 1], s), (3, 1)), linear_velocity=np.array([[300, 0, 0], [0, 0, 0], [0, 0, 0]], s),
                  angular_velocity=np.zeros((3, 3), s))
    shape = np.array([CUBOID, CUBOID, CUBOID], np.uint8)
    dims = np.array([[0.5, 0.5, 0.5], [0.5, 0.5, 0.5], [0.5, 0.5, 0.5]], s)
    rows = dict(c1=np.array([0, 0], np.uint32), c2=np.array([2, 1], np.uint32), b1=np.array([0, 0], np.uint32), b2=np.array([2, 1], np.uint32),
                live=np.array([1, 1], np.uint8))
    got, _, _, _ = run_both(s, bodies, shape, dims, rows, dict(body=[0], collider=[0], mode=[api.SWEEP_LINEAR]))
    assert got["hits"][0] == 2 and got["hit_contact"][0] == 0 and got["hit_body"][0] == 2


def test_visiting_order_changes_a_shared_target():
    s = np.float32
    # three projectiles converge on one dynamic body: its delta_position is the last writer's, its delta_rotation the ordered composition
    n = 4
    bodies = dict(kind=np.zeros(n, np.uint8), position=np.array([[0, 0, 0], [-3, 0, 0], [3, 0, 0], [0, 3, 0]], s),
                  rotation=np.tile(np.array([0, 0, 0, 1], s), (n, 1)),
                  linear_velocity=np.array([[1, 2, 3], [300, 0, 0], [-300, 0, 0], [0, -300, 0]], s),
                  angular_velocity=np.array([[5, 1, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0]], s))
    shape = np.full(n, SPHERE, np.uint8)
    dims = np.tile(np.array([[0.5, 0, 0]], s), (n, 1))
    rows = dict(c1=np.array([0, 0, 0], np.uint32), c2=np.array([1, 2, 3], np.uint32), b1=np.array([0, 0, 0], np.uint32), b2=np.array([1, 2, 3], np.uint32),
                live=np.ones(3, np.uint8))
    a = run_both(s, bodies, shape, dims, rows, dict(body=[1, 2, 3], collider=[1, 2, 3], mode=[0, 0, 0]))
    b = run_both(s, bodies, shape, dims, rows, dict(body=[3, 1, 2], collider=[3, 1, 2], mode=[0, 0, 0]))
    assert sorted(a[0]["min_toi"]) == sorted(b[0]["min_toi"])    # the TOIs do not depend on the order
    assert not np.array_equal(a[2][0], b[2][0])                  # the shared target's delta does


def test_struct_sizes():
    assert C.sizeof(api.AvnCcdConfig) == 64
    assert C.sizeof(api.AvnCcdResult) == 48
    assert "avn_ccd_configure" in api.ABI_SYMBOLS and "avn_ccd_download" in api.ABI_SYMBOLS
