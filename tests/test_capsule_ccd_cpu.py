"""Swept CCD with capsule colliders, without a GPU: the capsule branches of csrc/ccd_math.hpp (pair_toi / nonlinear_toi with CAPS = true)
against tests/capsule_reference.py's float64 distances, the linear mode against the capsule shape casts of the spatial queries, and the host
brute force's control flow with AVN_CCD_CAPSULES against tests/ccd_reference.py."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import capsule_reference as cr
import ccd_reference as ref
import test_ccd_cpu as cpu
from avian_b200 import api, fixture

DT, EPS = cpu.DT, cpu.EPS
CUBOID, SPHERE, CAPSULE = fixture.SHAPE_CUBOID, fixture.SHAPE_SPHERE, fixture.SHAPE_CAPSULE
PAIRS = [(CAPSULE, CAPSULE), (CAPSULE, SPHERE), (SPHERE, CAPSULE), (CAPSULE, CUBOID), (CUBOID, CAPSULE)]


def core(m, t):
    """(segment end 0, segment end 1, radius) of a capsule or a sphere of a 20-double motion record at time t"""
    c, R = cpu.pose(m, t)
    u = R[:, 1] * (m[2] if m[0] == CAPSULE else 0.0)
    return c - u, c + u, m[1]


def distance(a, b, t):
    """Exact float64 distance of the two shapes at time t (0 when they overlap), from the definitions of tests/capsule_reference.py."""
    if a[0] != CAPSULE and b[0] != CAPSULE:
        return cpu.distance(a, b, t)
    if a[0] != CAPSULE:
        a, b = b, a
    p0, p1, r = core(a, t)
    if b[0] == CUBOID:
        cb, Rb = cpu.pose(b, t)
        return max(cr.segment_box(p0, p1, cb, Rb, np.asarray(b[1:4]))[0] - r, 0.0)
    q0, q1, rb = core(b, t)
    return max(cr.segment_segment(p0, p1, q0, q1)[0] - r - rb, 0.0)


def rq(rng):
    q = rng.normal(size=4)
    return q / np.linalg.norm(q)


def dims_of(rng, shape):
    if shape == SPHERE:
        return np.array([rng.uniform(0.1, 0.6), 0, 0])
    if shape == CUBOID:
        return rng.uniform(0.05, 1.5, 3)
    if rng.random() < 0.3:   # long and thin
        return np.array([rng.uniform(0.01, 0.05), rng.uniform(1.0, 3.0), 0])
    return np.array([rng.uniform(0.05, 0.5), rng.uniform(0.0, 1.2), 0])


def random_pair(rng, spin=True, kinds=None):
    """A moving, spinning pair with at least one capsule whose swept volumes may meet within DT; off-origin centres of mass on both sides."""
    sa, sb = PAIRS[rng.integers(len(PAIRS))] if kinds is None else kinds
    pb = rng.normal(size=3) * 2.5
    va = pb * rng.uniform(0, 90) + rng.normal(size=3) * 10
    a = fixture.ccd_motion(sa, dims_of(rng, sa), np.zeros(3), rq(rng), va, rng.normal(size=3) * (40 if spin else 0), rng.normal(size=3) * 0.05)
    b = fixture.ccd_motion(sb, dims_of(rng, sb), pb, rq(rng), rng.normal(size=3) * 5, rng.normal(size=3) * (20 if spin else 0),
                           rng.normal(size=3) * 0.05)
    return a, b


# ---- the non-linear contract -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [1, 2])
def test_nonlinear_toi_contract(seed):
    rng = np.random.default_rng(seed)
    hits = misses = capped = 0
    kinds = set()
    for _ in range(200):
        a, b = random_pair(rng)
        if distance(a, b, 0.0) <= EPS:
            continue
        t, its = fixture.ccd_nonlinear_toi(a, b, DT, EPS, iterations=True)
        samples = np.linspace(0.0, DT if t is None else t, 150, endpoint=t is None)
        d = np.array([distance(a, b, s) for s in samples])
        if t is None:
            misses += 1
            assert (d > 0).all(), "no hit reported, yet the shapes touch on [0, dt]"
            continue
        hits += 1
        kinds.add((int(a[0]), int(b[0])))
        assert (d > 0).all(), "contact before the reported TOI (tunnelling)"
        if its == 64:
            capped += 1     # stopped at the cap: t lies before the contact, the distance there may exceed eps
            continue
        assert distance(a, b, t) <= EPS + 1e-9
    assert hits > 20 and misses > 10 and capped <= hits // 5
    assert len(kinds) == len(PAIRS), kinds


def test_nonlinear_without_spin_is_never_later_than_linear():
    rng = np.random.default_rng(7)
    n = capped = 0
    for _ in range(300):
        a, b = random_pair(rng, spin=False)
        lin = fixture.ccd_pair_toi(np.float64, api.SWEEP_LINEAR, a, b, DT)
        if lin <= 0:
            continue
        nl, its = fixture.ccd_nonlinear_toi(a, b, DT, EPS, iterations=True)
        assert nl is not None and nl <= lin + 1e-12
        if its == 64:
            capped += 1
            continue
        assert distance(a, b, nl) <= EPS + 1e-9
        n += 1
    assert n > 20 and capped <= n // 5


# ---- the linear mode -------------------------------------------------------------------------------------------------------------------
def cast(a, b, dims_b=None, shape_b=None):
    """shape A along v1 - v2 against collider B at rest, as a capsule-enabled spatial-query cast with max distance dt (float64)"""
    sb = b[0] if shape_b is None else shape_b
    hb = b[1:4] if dims_b is None else np.asarray(dims_b, float)
    cols = api.QueryColliders(shape=np.array([sb], np.uint8), dims=hb[None], position=b[4:7][None], rotation=b[7:11][None])
    shapes = api.ShapeQueries(shape=np.array([a[0]], np.uint8), dims=a[1:4][None], position=a[4:7][None], rotation=a[7:11][None],
                              direction=(a[14:17] - b[14:17])[None], max_distance=np.array([DT]))
    got = fixture.query_cast_shape(np.float64, cols, shapes, capsules=True)
    return None if got["collider"][0] < 0 else float(got["distance"][0])


def static_distance(a, b, t):
    """the linear mode's motion: A translated by (v1 - v2) t, B at rest, no rotation"""
    a2 = a.copy()
    a2[4:7] = a[4:7] + (a[14:17] - b[14:17]) * t
    a2[14:20] = 0
    b2 = b.copy()
    b2[14:20] = 0
    return distance(a2, b2, 0.0)


def first_contact(a, b, hi):
    """bisection on the reference's exact overlap predicate for the first t in [0, hi] at which the shapes touch (the overlap set of a
    translation against a convex shape is one interval, and hi lies inside it)"""
    lo = 0.0
    for _ in range(80):
        mid = 0.5 * (lo + hi)
        if static_distance(a, b, mid) > 0:
            lo = mid
        else:
            hi = mid
    return hi


@pytest.mark.parametrize("scalar", [np.float32, np.float64])
def test_linear_toi_is_the_capsule_cast_of_the_relative_motion(scalar):
    rng = np.random.default_rng(3)
    n = grazing = fallback = 0
    for _ in range(300):
        a, b = random_pair(rng, spin=False)
        want = fixture.ccd_pair_toi(scalar, api.SWEEP_LINEAR, a, b, DT)
        t = cast(a, b)
        if t is None:
            assert want == -1.0
            assert all(static_distance(a, b, s) > 0 for s in np.linspace(0.0, DT, 60))
            continue
        if scalar(t) == 0:
            # the zero-TOI fallback: shape 2 replaced by a ball of radius prediction_distance at its pose
            got = fixture.ccd_pair_toi(scalar, api.SWEEP_LINEAR, a, b, DT, EPS, 0.05)
            tb = cast(a, b, dims_b=(0.05, 0, 0), shape_b=SPHERE)
            assert got == (-1.0 if tb is None else float(scalar(tb)))
            fallback += 1
            continue
        assert want == float(scalar(t))
        n += 1
        # against the reference: no overlap before the TOI, the first contact (by bisection) within the rounding of t
        assert static_distance(a, b, t * (1 - 1e-7)) > 0
        hi = t * (1 + 1e-6) + 1e-12
        if static_distance(a, b, hi) > 0:
            grazing += 1      # the sweep only touches: the interval of contact is shorter than the probe
            assert static_distance(a, b, t) <= 1e-6
            continue
        assert abs(first_contact(a, b, hi) - want) <= 1e-9 + 1e-6 * t
    assert n > 20 and fallback > 0 and grazing <= n // 10


# ---- degenerate capsules ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [api.SWEEP_LINEAR, api.SWEEP_NON_LINEAR])
def test_zero_half_length_is_a_sphere(mode):
    rng = np.random.default_rng(21)
    n = 0
    for _ in range(150):
        a, b = random_pair(rng, kinds=(CAPSULE, [CUBOID, SPHERE, CAPSULE][rng.integers(3)]), spin=mode == api.SWEEP_NON_LINEAR)
        a[2] = 0.0                                  # half length 0: a ball of the capsule's radius
        s = a.copy()
        s[0] = SPHERE
        s[2] = 0.0
        t_cap = fixture.ccd_pair_toi(np.float64, mode, a, b, DT, EPS)
        t_sph = fixture.ccd_pair_toi(np.float64, mode, s, b, DT, EPS)
        assert (t_cap < 0) == (t_sph < 0)
        if t_cap > 0:
            n += 1
            assert abs(t_cap - t_sph) <= 1e-9 + 1e-6 * t_sph
    assert n > 10


@pytest.mark.parametrize("shape_b", [CUBOID, SPHERE, CAPSULE])
def test_zero_radius_is_a_bare_segment(shape_b):
    rng = np.random.default_rng(22 + shape_b)
    n = 0
    for _ in range(100):
        a, b = random_pair(rng, kinds=(CAPSULE, shape_b))
        a[1] = 0.0
        if distance(a, b, 0.0) <= EPS:
            continue
        t = fixture.ccd_nonlinear_toi(a, b, DT, EPS)
        if t is None:
            continue
        n += 1
        assert min(distance(a, b, s) for s in np.linspace(0.0, t, 100)) > 0
        assert distance(a, b, t) <= EPS + 1e-9 or fixture.ccd_nonlinear_toi(a, b, DT, EPS, iterations=True)[1] == 64
    assert n > 5


# ---- known answers ---------------------------------------------------------------------------------------------------------------------
def test_capsule_bullet_stops_before_the_wall():
    bullet = fixture.ccd_motion(CAPSULE, (0.05, 0.2, 0), (0, 0, 0), (0, 0, 0, 1), (300.0, 0, 0))   # axis y, flying along x
    wall = fixture.ccd_motion(CUBOID, (0.02, 3, 3), (4.0, 0, 0), (0, 0, 0, 1))
    for scalar in (np.float32, np.float64):
        for mode in (api.SWEEP_LINEAR, api.SWEEP_NON_LINEAR):
            t = fixture.ccd_pair_toi(scalar, mode, bullet, wall, DT)
            assert 0 < t < DT
            front = t * 300.0 + 0.05
            assert abs(front - (4.0 - 0.02)) <= 1e-3 and front <= 4.0 - 0.02 + 1e-6


def test_spinning_capsule_bat_and_small_sphere():
    s = np.sin(-np.pi / 4)
    bat = fixture.ccd_motion(CAPSULE, (0.05, 2.0, 0), (0, 0, 0), (0, 0, s, np.cos(-np.pi / 4)), (0, 0, 0), (0, 0, 60.0))   # axis along +x
    target = fixture.ccd_motion(SPHERE, (0.1, 0, 0), (1.5 * np.cos(0.5), 1.5 * np.sin(0.5), 0), (0, 0, 0, 1))
    assert fixture.ccd_pair_toi(np.float32, api.SWEEP_LINEAR, bat, target, DT) == -1.0      # linear: the bat does not translate
    t = fixture.ccd_pair_toi(np.float32, api.SWEEP_NON_LINEAR, bat, target, DT)
    assert 0 < t < DT and abs(60.0 * t - (0.5 - np.arcsin(0.1))) < 1e-3                     # the axis comes within 0.15 of the centre
    assert distance(bat, target, t) <= EPS
    # the swapped order sweeps the same pair
    t2 = fixture.ccd_pair_toi(np.float32, api.SWEEP_NON_LINEAR, target, bat, DT)
    assert abs(t2 - t) <= 1e-6


def test_motion_radius_bounds_the_capsule():
    # the spin bound of a capsule with its centre of mass off the segment's centre: every surface point stays within it.  A capsule
    # spinning about its far centre of mass reaches a sphere exactly when the far end does
    a = fixture.ccd_motion(CAPSULE, (0.1, 1.0, 0), (0, 0, 0), (0, 0, 0, 1), (0, 0, 0), (0, 0, 30.0), com=(0, -0.8, 0))
    # the +y end is 1.8 from the com, its cap reaches 1.9: a ball of radius 0.05 centred 1.95 from the com meets only the cap's tip
    ang = 0.3
    c = np.array([0, -0.8, 0]) + 1.95 * np.array([-np.sin(ang), np.cos(ang), 0])
    target = fixture.ccd_motion(SPHERE, (0.05, 0, 0), c, (0, 0, 0, 1))
    t = fixture.ccd_nonlinear_toi(a, target, DT, EPS)
    # the approach is tangential (d ~ 11.7 (ang - w t)^2), so eps = 1e-4 is reached about 3e-3 rad before the touch
    assert t is not None and 0 <= ang - 30.0 * t < 4e-3 and distance(a, target, t) <= EPS
    assert min(distance(a, target, s) for s in np.linspace(0.0, t, 200)) > 0


# ---- control flow and refusals ---------------------------------------------------------------------------------------------------------
def capsule_world(rng, n, scalar):
    bodies, shape, dims, rows = cpu.random_world(rng, n, scalar)
    shape = rng.integers(0, 3, size=n).astype(np.uint8)
    caps = np.stack([rng.uniform(0.1, 0.4, n), rng.uniform(0.0, 1.0, n), np.zeros(n)], axis=1)
    dims = np.where(shape[:, None] == SPHERE, np.array([[0.3, 0, 0]]),
                    np.where(shape[:, None] == CAPSULE, caps, rng.uniform(0.2, 0.8, (n, 3)))).astype(scalar)
    return bodies, shape, dims, rows


@pytest.mark.parametrize("scalar", [np.float32, np.float64])
@pytest.mark.parametrize("seed", [31, 32, 33])
def test_control_flow_matches_reference(scalar, seed):
    rng = np.random.default_rng(seed)
    bodies, shape, dims, rows = capsule_world(rng, 24, scalar)
    k = 10
    body = rng.choice(24, size=k, replace=False)
    cfg = dict(body=body, collider=body, mode=rng.integers(0, 2, k), include_dynamic=rng.integers(0, 2, k),
               linear_threshold=rng.choice([0.0, 50.0, 200.0], k), angular_threshold=rng.choice([0.0, 20.0, 80.0], k), capsules=True)
    got, writes, _, _ = cpu.run_both(scalar, bodies, shape, dims, rows, cfg)
    capsule_hits = [int(b) for b, h in zip(body, got["hit_body"]) if h >= 0 and (shape[b] == CAPSULE or shape[h] == CAPSULE)]
    assert capsule_hits and len(writes) >= 1, "no pair with a capsule was hit"
    cpu.run_both(scalar, bodies, shape, dims, rows, cfg, prediction=0.05)
    # without the flag the same world is refused
    with pytest.raises(api.AvianError) as e:
        fixture.ccd_solve(scalar, DT, 1.0, bodies, shape, dims, rows, dict(cfg, capsules=False))
    assert e.value.status == api.ERR_UNSUPPORTED


def test_flag_without_capsules_changes_nothing():
    rng = np.random.default_rng(12)
    bodies, shape, dims, rows = cpu.random_world(rng, 24, np.float32)
    body = rng.choice(24, size=10, replace=False)
    cfg = dict(body=body, collider=body, mode=rng.integers(0, 2, 10))
    plain = fixture.ccd_solve(np.float32, DT, 1.0, bodies, shape, dims, rows, cfg)
    flagged = fixture.ccd_solve(np.float32, DT, 1.0, bodies, shape, dims, rows, dict(cfg, capsules=True))
    for k in plain:
        assert np.array_equal(plain[k].view(np.uint8), flagged[k].view(np.uint8)), k


def test_unknown_flag_bits_are_refused():
    rng = np.random.default_rng(13)
    bodies, shape, dims, rows = capsule_world(rng, 8, np.float32)
    for flags in (0x2, 0x3, 0x80000000):
        with pytest.raises(ValueError):
            fixture.ccd_solve(np.float32, DT, 1.0, bodies, shape, dims, rows, dict(body=[0], collider=[0], flags=flags))


def test_config_layout():
    assert C.sizeof(api.AvnCcdConfig) == 64 and api.AvnCcdConfig.flags.offset == 4 and api.AvnCcdConfig.flags.size == 4
    cfg, _ = api.ccd_config([1], [1], flags=api.CCD_CAPSULES)
    assert cfg.flags == api.CCD_CAPSULES == 1
    # the C example and the header agree on the bit
    from avian_b200 import _build
    text = (_build.REPO / "include" / "avian_b200.h").read_text()
    assert "#define AVN_CCD_CAPSULES 0x1u" in text


def test_reference_config_ignores_the_capsules_key():
    import oracle_ccd
    a = oracle_ccd.bodies_as_ref_config(dict(body=[3], collider=[4]))
    b = oracle_ccd.bodies_as_ref_config(dict(body=[3], collider=[4], capsules=True))
    assert a == b
    assert ref.NON_LINEAR == api.SWEEP_NON_LINEAR
