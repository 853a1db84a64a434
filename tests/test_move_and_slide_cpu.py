"""Move and slide on the host (no GPU): fixture.move_and_slide — the brute force over every collider that the device kernel must equal bit
for bit — against hand-worked closed forms, the reference's projection agreement test, and an independent Python restatement of
move_and_slide.rs (tests/move_reference.py).  Also the ABI layouts and the refused inputs."""
from __future__ import annotations

import ctypes as C
import math
import subprocess
import tempfile
from pathlib import Path

import numpy as np
import pytest

from avian_b200 import api, fixture
import move_reference as ref
from move_scenes import random_characters, random_colliders

ROOT = Path(__file__).resolve().parents[1]
ID = np.array([[0.0, 0.0, 0.0, 1.0]])
SCALARS = [np.float32, np.float64]


def box(pos, half, rot=(0.0, 0.0, 0.0, 1.0)):
    return (fixture.SHAPE_CUBOID, np.asarray(half, float), np.asarray(pos, float), np.asarray(rot, float))


def colliders(*items, memberships=None):
    return api.QueryColliders(shape=np.array([i[0] for i in items], np.uint8), dims=np.array([i[1] for i in items]),
                              position=np.array([i[2] for i in items]), rotation=np.array([i[3] for i in items]), memberships=memberships)


def character(shape, pos, vel, **kw):
    return api.MoveBatch(shape=np.array([shape], np.uint8), dims=np.array([[0.5, 0.5, 0.5]]), position=np.array([pos], float), rotation=ID,
                         velocity=np.array([vel], float), **kw)


def run(scalar, cols, cfg, batch):
    return fixture.move_and_slide(scalar, cols, cfg, batch)


def tol(scalar, lu=1.0):
    return (2e-4 if scalar == np.float32 else 1e-6) * max(lu, 1.0) * 10


def quat_axis(axis, deg):
    a = math.radians(deg) / 2
    v = np.asarray(axis, float) * math.sin(a)
    return (v[0], v[1], v[2], math.cos(a))


SHAPES = [fixture.SHAPE_SPHERE, fixture.SHAPE_CUBOID]
CASES = [(s, lu, dt) for s in SHAPES for lu in (1.0, 10.0) for dt in SCALARS]
ids = lambda c: f"{'sphere' if c[0] else 'cuboid'}-lu{int(c[1])}-{np.dtype(c[2]).name}"


@pytest.mark.parametrize("case", CASES, ids=ids)
def test_free_flight(case):
    shape, lu, sc = case
    cols = colliders(box((50, 50, 50), (1, 1, 1)))
    cfg = api.MoveConfig(length_unit=lu)
    r = run(sc, cols, cfg, character(shape, (0, 0, 0), (6, -3, 12)))
    np.testing.assert_allclose(r["position"][0], np.array([6, -3, 12]) / 60, atol=tol(sc))
    np.testing.assert_array_equal(r["velocity"][0], np.array([6, -3, 12], sc))
    assert (r["hit_collider"] == -1).all()


@pytest.mark.parametrize("case", CASES, ids=ids)
def test_head_on_wall_stops_at_the_pull_back_distance(case):
    shape, lu, sc = case
    cols = colliders(box((2.0, 0, 0), (0.5, 5, 5)))         # face at x = 1.5, gap 1.0 to the character's surface
    cfg = api.MoveConfig(length_unit=lu)
    r = run(sc, cols, cfg, character(shape, (0, 0, 0), (120, 0, 0)))
    skin = 0.01 * lu
    np.testing.assert_allclose(r["position"][0], [1.0 - skin, 0, 0], atol=tol(sc))
    np.testing.assert_allclose(r["velocity"][0], [0, 0, 0], atol=tol(sc))
    assert r["hit_collider"][0, 0] == 0 and (r["hit_collider"][0, 1:] == -1).all()
    np.testing.assert_allclose(r["hit_toi"][0, 0], 1.0, atol=tol(sc))
    np.testing.assert_allclose(r["hit_distance"][0, 0], 1.0 - skin, atol=tol(sc))
    np.testing.assert_allclose(r["hit_normal"][0, 0], [-1, 0, 0], atol=tol(sc))


def _slope(shape, lu, sc, axis, deg):
    """A plane through (3, 0, 0) whose outward normal n is the -x face of a big box rotated by deg about axis; the character moves along +x
    at 240 m/s for 1/60 s.  Closed form: first touch at t1 = (D0 - support) / (-n_x), pull-back by skin / (-n_x), the rest of the time
    along v - (v.n) n."""
    q = quat_axis(axis, deg)
    R = np.array(_rot(q))
    ax, n = R[:, 0], -R[:, 0]
    cols = colliders(box(np.array([3.0, 0, 0]) + 50.0 * ax, (50, 50, 50), q))
    cfg = api.MoveConfig(length_unit=lu)
    v = np.array([240.0, 0, 0])
    r = run(sc, cols, cfg, character(shape, (0, 0, 0), v))
    support = 0.5 if shape == fixture.SHAPE_SPHERE else 0.5 * np.abs(n).sum()
    skin = 0.01 * lu
    d0 = -3.0 * n[0]
    t1 = (d0 - support) / -n[0]
    safe = t1 - skin / -n[0]
    time_left = (1 / 60) * (1 - safe / 4.0)
    vp = v - (v @ n) * n
    return r, np.array([safe, 0, 0]) + time_left * vp, vp


def _rot(q):
    x, y, z, w = q
    return [[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
            [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]]


@pytest.mark.parametrize("case", CASES, ids=ids)
def test_45_degree_wall_slides(case):
    shape, lu, sc = case
    r, want_pos, want_vel = _slope(shape, lu, sc, (0, 1, 0), 45)
    np.testing.assert_allclose(r["position"][0], want_pos, atol=tol(sc, lu))
    np.testing.assert_allclose(r["velocity"][0], want_vel, atol=tol(sc) * 240)
    assert r["hit_collider"][0, 0] == 0 and r["hit_collider"][0, 1] == -1


@pytest.mark.parametrize("case", CASES, ids=ids)
def test_ramp_projects_up_the_ramp_with_v_cos_theta(case):
    shape, lu, sc = case
    theta = 30.0
    r, want_pos, want_vel = _slope(shape, lu, sc, (0, 0, 1), -(90 - theta))   # the -x face tilted back: a ramp rising along +x
    v = r["velocity"][0].astype(float)
    np.testing.assert_allclose(np.linalg.norm(v), 240 * math.cos(math.radians(theta)), rtol=1e-5)
    np.testing.assert_allclose(v / np.linalg.norm(v), [math.cos(math.radians(theta)), math.sin(math.radians(theta)), 0], atol=1e-5)
    np.testing.assert_allclose(r["position"][0], want_pos, atol=tol(sc, lu))


def _corner(shape, lu, sc, walls, vel, **cfgkw):
    skin = 0.01 * lu
    items = [box((0, -50.0, 0), (50, 50, 50))]                  # floor, top at y = 0
    if walls >= 1:
        items.append(box((51.0, 0, 0), (50, 50, 50)))           # wall, face at x = 1
    if walls >= 2:
        items.append(box((0, 0, 51.0), (50, 50, 50)))           # wall, face at z = 1
    start = (1.0 - 0.5 - skin, 0.5 + skin, 1.0 - 0.5 - skin if walls >= 2 else 0.0)
    return run(sc, colliders(*items), api.MoveConfig(length_unit=lu, **cfgkw), character(shape, start, vel)), np.array(start)


@pytest.mark.parametrize("case", CASES, ids=ids)
def test_floor_wall_corner_projects_onto_the_edge(case):
    shape, lu, sc = case
    r, start = _corner(shape, lu, sc, 1, (60, -60, 60))
    np.testing.assert_allclose(r["velocity"][0], [0, 0, 60], atol=tol(sc) * 60)
    np.testing.assert_allclose(r["position"][0], start + [0, 0, 1.0], atol=tol(sc, lu))


@pytest.mark.parametrize("case", CASES, ids=ids)
def test_three_plane_corner_projects_to_zero(case):
    shape, lu, sc = case
    r, start = _corner(shape, lu, sc, 2, (60, -60, 60))
    assert np.linalg.norm(r["velocity"][0]) <= ref.DOT_EPSILON * 2
    np.testing.assert_allclose(r["position"][0], start, atol=tol(sc, lu))


@pytest.mark.parametrize("case", CASES, ids=ids)
def test_max_planes_one_keeps_only_the_sweep_plane(case):
    shape, lu, sc = case
    r, _ = _corner(shape, lu, sc, 1, (60, -60, 60), move_and_slide_iterations=1, max_planes=1)
    hit = r["hit_collider"][0, 0]                                       # floor and wall are hit at the same TOI up to rounding
    assert hit in (0, 1)
    np.testing.assert_allclose(r["velocity"][0], [60, 0, 60] if hit == 0 else [0, -60, 60], atol=tol(sc) * 60)
    r, _ = _corner(shape, lu, sc, 1, (60, -60, 60), move_and_slide_iterations=1)
    np.testing.assert_allclose(r["velocity"][0], [0, 0, 60], atol=tol(sc) * 60)


@pytest.mark.parametrize("case", CASES, ids=ids)
def test_embedded_start_is_pushed_out_by_depth_plus_skin(case):
    shape, lu, sc = case
    d = 0.02 * lu
    cols = colliders(box((0, -50.0, 0), (50, 50, 50)))
    r = run(sc, cols, api.MoveConfig(length_unit=lu), character(shape, (0, 0.5 - d, 0), (0, 0, 0)))
    np.testing.assert_allclose(r["position"][0], [0, 0.5 + 0.01 * lu, 0], atol=tol(sc, lu))


@pytest.mark.parametrize("case", CASES, ids=ids)
def test_embedding_deeper_than_the_rejection_threshold_is_left_alone(case):
    shape, lu, sc = case
    d = 0.3                                                             # + skin > 0.5 * lu only at lu = 1: use a threshold below it
    cols = colliders(box((0, -50.0, 0), (50, 50, 50)))
    r = run(sc, cols, api.MoveConfig(length_unit=lu, penetration_rejection_threshold=0.2 / lu), character(shape, (0, 0.5 - d, 0), (0, 0, 0)))
    np.testing.assert_array_equal(r["position"][0], np.array([0, 0.5 - d, 0], sc))


@pytest.mark.parametrize("case", CASES, ids=ids)
def test_initial_ground_plane_removes_the_downward_part(case):
    shape, lu, sc = case
    cols = colliders(box((2.0, 0, 0), (0.5, 5, 5)))
    r = run(sc, cols, api.MoveConfig(length_unit=lu), character(shape, (0, 0, 0), (120, -30, 20), planes=[[[0, 1, 0]]]))
    v = r["velocity"][0]
    assert v[1] >= -ref.DOT_EPSILON
    np.testing.assert_allclose(v, [0, 0, 20], atol=tol(sc) * 120)
    r2 = run(sc, cols, api.MoveConfig(length_unit=lu), character(shape, (0, 0, 0), (120, -30, 20)))
    assert r2["velocity"][0][1] < -1.0                                  # without the plane the wall alone keeps it


@pytest.mark.parametrize("case", CASES, ids=ids)
def test_tiny_motion_only_depenetrates(case):
    shape, lu, sc = case
    cols = colliders(box((0, -50.0, 0), (50, 50, 50)))
    v = (0.003, 0, 0)                                                   # |v dt| = 5e-5 < MIN_DISTANCE
    r = run(sc, cols, api.MoveConfig(length_unit=lu), character(shape, (0, 0.45, 0), v))
    np.testing.assert_allclose(r["position"][0], [0, 0.5 + 0.01 * lu, 0], atol=tol(sc, lu))
    np.testing.assert_array_equal(r["velocity"][0], np.array(v, sc))
    assert (r["hit_collider"] == -1).all()


@pytest.mark.parametrize("case", CASES, ids=ids)
def test_excluded_masked_and_ignored_colliders_are_passed_through(case):
    shape, lu, sc = case
    cfg = api.MoveConfig(length_unit=lu)
    free = run(sc, colliders(box((50, 50, 50), (1, 1, 1))), cfg, character(shape, (0, 0, 0), (120, 0, 0)))
    wall = colliders(box((50, 50, 50), (1, 1, 1)), box((2.0, 0, 0), (0.5, 5, 5)), memberships=np.array([1, 2], np.uint32))
    blocked = run(sc, wall, cfg, character(shape, (0, 0, 0), (120, 0, 0)))
    assert blocked["hit_collider"][0, 0] == 1
    for kw, c in (({"exclude": [[1]]}, cfg), ({"mask": np.array([1], np.uint32)}, cfg),
                  ({}, api.MoveConfig(length_unit=lu, ignored=np.array([0, 1], np.uint8)))):
        r = run(sc, wall, c, character(shape, (0, 0, 0), (120, 0, 0), **kw))
        for k in ("position", "velocity", "hit_collider"):
            np.testing.assert_array_equal(r[k], free[k])


# ---- project_velocity against the reference's agreement test (velocity_project.rs:337-406) --------------------------------------------
def _quasi_random_directions(n):
    plastic = 1.32471795724475
    ip, ip2 = 1.0 / plastic, 1.0 / plastic / plastic
    i = j = 0.0
    out = []
    for _ in range(n):
        phi = 2.0 * math.pi * j
        z = 2.0 * i - 1.0
        rho = math.sqrt(1.0 - z * z)
        out.append((rho * math.cos(phi), rho * math.sin(phi), z))
        i, j = (i + ip) % 1.0, (j + ip2) % 1.0
    return np.array(out)


AGREEMENT_NORMALS = [(0, 0, 1), (2, 0, 1), (-2, 0, 1), (0, 2, 1), (0, -2, 1), (1.5, 1.5, 1), (1.5, -1.5, 1), (-1.5, 1.5, 1), (-1.5, -1.5, 1),
                     (1, 1.75, 1), (1, -1.75, 1), (-1, 1.75, 1), (-1, -1.75, 1), (1.75, 1, 1), (1.75, -1, 1), (-1.75, 1, 1), (-1.75, -1, 1)]


@pytest.mark.parametrize("scalar", SCALARS, ids=lambda s: np.dtype(s).name)
def test_project_velocity_agrees_with_brute_force(scalar):
    normals = [np.array(n, np.float32) / np.float32(np.linalg.norm(np.array(n, np.float32))) for n in AGREEMENT_NORMALS]
    dirs = _quasi_random_directions(1000)
    for k in range(1, len(normals) + 1):
        sel = normals[:k]
        for v in dirs:
            got = fixture.project_velocity(scalar, v, np.array(sel)).astype(np.float64)
            for n in sel:
                assert -(got @ n.astype(np.float64)) <= ref.DOT_EPSILON + 1e-6, (k, v)
            brute = ref.project_velocity_bruteforce(v, sel)
            assert np.linalg.norm(got - v) - np.linalg.norm(brute - v) <= ref.DOT_EPSILON + 1e-6, (k, v)


def test_project_velocity_matches_the_python_restatement():
    rng = np.random.default_rng(5)
    for _ in range(500):
        ns = rng.normal(size=(int(rng.integers(0, 8)), 3))
        ns = (ns / np.linalg.norm(ns, axis=1, keepdims=True)).astype(np.float32)
        v = rng.normal(size=3) * 10
        np.testing.assert_allclose(fixture.project_velocity(np.float64, v, ns), ref.project_velocity(v, list(ns)), atol=1e-9)


# ---- the whole loop against the independent restatement ---------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", [api.MoveConfig(), api.MoveConfig(move_and_slide_iterations=8, max_planes=3, length_unit=2.0),
                                 api.MoveConfig(depenetration_iterations=0)], ids=["default", "8-iterations", "no-depenetration"])
def test_loop_matches_the_restatement(cfg):
    rng = np.random.default_rng(11)
    cols, ignored = random_colliders(rng, 60, 3.0)
    cfg.ignored = ignored
    batch = random_characters(rng, 200, 3.0, 60)
    got = fixture.move_and_slide(np.float64, cols, cfg, batch)
    scene = ref.Scene(cols, ignored)
    hits = 0
    for i in range(batch.count):
        p, v, h = ref.move_one(scene, cfg, int(batch.shape[i]), batch.dims[i], batch.position[i], batch.rotation[i], batch.velocity[i],
                               int(batch.mask[i]), batch.exclude[i], [] if batch.planes[i] is None else batch.planes[i])
        np.testing.assert_allclose(got["position"][i], p, atol=1e-9, err_msg=f"character {i}")
        np.testing.assert_allclose(got["velocity"][i], v, atol=1e-8, err_msg=f"character {i}")
        want_c = np.full(cfg.move_and_slide_iterations, -1)
        for it, c, safe, toi in h:
            want_c[it] = c
            np.testing.assert_allclose([got["hit_distance"][i, it], got["hit_toi"][i, it]], [safe, toi], atol=1e-9)
        np.testing.assert_array_equal(got["hit_collider"][i], want_c)
        hits += len(h)
    assert hits > 50


# ---- ABI ---------------------------------------------------------------------------------------------------------------------------------
def test_move_struct_layouts_match_the_header():
    names = ["AvnMoveConfig", "AvnMoveBatch", "AvnMoveResult"]
    fields = {n: [f[0] for f in getattr(api, n)._fields_ if not f[0].startswith("_")] for n in names}
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "avian_b200.h"\nint main(){'
    src += "".join(f'printf("{n} %zu\\n", sizeof({n}));' for n in names)
    src += "".join(f'printf("{n}.{f} %zu\\n", offsetof({n}, {f}));' for n in names for f in fields[n])
    src += 'printf("AVN_MOVE_MAX_PLANES %d\\n", AVN_MOVE_MAX_PLANES);return 0;}'
    with tempfile.TemporaryDirectory() as d:
        (Path(d) / "s.c").write_text(src)
        subprocess.run(["gcc", "-I", str(ROOT / "include"), "-o", f"{d}/s", f"{d}/s.c"], check=True)
        out = subprocess.run([f"{d}/s"], capture_output=True, text=True, check=True).stdout
    got = dict(line.split() for line in out.strip().splitlines())
    for n in names:
        assert int(got[n]) == C.sizeof(getattr(api, n)), n
        for f in fields[n]:
            assert int(got[f"{n}.{f}"]) == getattr(api, n).__dict__[f].offset, (n, f)
    assert int(got["AVN_MOVE_MAX_PLANES"]) == api.MOVE_MAX_PLANES


def _refused(cols, cfg, batch, what):
    with pytest.raises(api.AvianError) as e:
        fixture.move_and_slide(np.float64, cols, cfg, batch)
    assert e.value.status == api.ERR_INVALID_ARGUMENT and what in str(e.value), str(e.value)


def test_refused_inputs():
    cols = colliders(box((2.0, 0, 0), (0.5, 5, 5)), box((5.0, 0, 0), (0.5, 5, 5)))
    ok = lambda **kw: character(fixture.SHAPE_SPHERE, (0, 0, 0), (1, 0, 0), **kw)
    cfg = api.MoveConfig()
    fixture.move_and_slide(np.float64, cols, cfg, ok())
    bad = ok()
    bad.dims = np.array([[-0.5, 0.5, 0.5]])
    _refused(cols, cfg, bad, "negative")
    bad = ok()
    bad.shape = np.array([7], np.uint8)
    _refused(cols, cfg, bad, "unknown shape")
    b = ok()
    s, keep = b.as_struct(np.float64)
    xoff = np.array([0, 5], np.uint32)
    xs = np.array([0], np.uint32)
    s.exclude_offsets, s.exclude, s.exclude_count = xoff.ctypes.data, xs.ctypes.data, 1
    c, kc = cols.as_struct(np.float64)
    m, km = cfg.as_struct()
    o, out = api.move_result(1, 4, np.float64)
    lib = fixture._load()
    assert lib.avh_move_and_slide(64, C.byref(c), C.byref(m), C.byref(s), C.byref(o)) == api.ERR_INVALID_ARGUMENT
    assert b"exclude_offsets" in lib.avh_query_error()
    _refused(cols, api.MoveConfig(max_planes=api.MOVE_MAX_PLANES + 1), ok(), "max_planes")
    _refused(cols, api.MoveConfig(max_planes=2), ok(planes=[[[0, 1, 0]] * 3]), "more initial planes")
    _refused(cols, cfg, ok(planes=[[[0, math.inf, 0]]]), "non-finite initial plane")
    _refused(cols, cfg, ok(planes=[[[0, 0, 0]]]), "zero initial plane")
    for field in ("delta_time", "length_unit", "skin_width", "max_depenetration_error", "penetration_rejection_threshold",
                  "plane_similarity_dot_threshold"):
        _refused(cols, api.MoveConfig(**{field: math.nan}), ok(), "NaN")
    _refused(cols, api.MoveConfig(ignored=np.zeros(3, np.uint8)), ok(), "ignored")


@pytest.mark.parametrize("scalar", SCALARS, ids=lambda s: np.dtype(s).name)
def test_non_finite_characters_are_returned_unmoved(scalar):
    cols = colliders(box((2.0, 0, 0), (0.5, 5, 5)))
    n = 4
    batch = api.MoveBatch(shape=np.ones(n, np.uint8), dims=np.full((n, 3), 0.5), position=np.zeros((n, 3)), rotation=np.tile(ID, (n, 1)),
                          velocity=np.tile([120.0, 0, 0], (n, 1)))
    batch.position[0, 1] = math.nan
    batch.velocity[1, 2] = math.inf
    batch.rotation[2] = 0.0
    batch.dims[3, 0] = math.inf
    r = fixture.move_and_slide(scalar, cols, api.MoveConfig(), batch)
    np.testing.assert_array_equal(r["position"], batch.position.astype(scalar))
    np.testing.assert_array_equal(r["velocity"], batch.velocity.astype(scalar))
    assert (r["hit_collider"] == -1).all() and not r["hit_distance"].any()
