"""Move and slide on the device (H100): avn_move_and_slide against the host brute force (fixture.move_and_slide, the same
csrc/move_math.hpp over every collider), bit for bit on every output, f32 and f64."""
from __future__ import annotations

import math

import numpy as np
import pytest

from avian_b200 import api, fixture, scenes
from move_scenes import random_characters, random_colliders, random_quats

pytestmark = pytest.mark.gpu
SCALARS = [np.float32, np.float64]
OUTPUTS = ("position", "velocity", "hit_collider", "hit_distance", "hit_toi", "hit_point", "hit_normal")


def assert_bitwise(got, want, what=""):
    for k in OUTPUTS:
        a, b = np.ascontiguousarray(got[k]), np.ascontiguousarray(want[k])
        assert a.shape == b.shape, (what, k)
        bad = np.flatnonzero((a.view(np.uint8).reshape(a.shape[0], -1) != b.view(np.uint8).reshape(b.shape[0], -1)).any(axis=1))
        assert bad.size == 0, f"{what} {k}: {bad.size} characters differ, first {bad[:5]}: {a[bad[0]]} vs {b[bad[0]]}"


def take(b: "api.MoveBatch", idx) -> "api.MoveBatch":
    pick = lambda a: None if a is None else np.asarray(a)[idx]
    lst = lambda a: None if a is None else [a[i] for i in idx]
    return api.MoveBatch(shape=pick(b.shape), dims=pick(b.dims), position=pick(b.position), rotation=pick(b.rotation), velocity=pick(b.velocity),
                         mask=pick(b.mask), exclude=lst(b.exclude), planes=lst(b.planes))


def rows(r: dict, idx) -> dict:
    return {k: r[k][idx] for k in OUTPUTS}


CONFIGS = {
    "default": api.MoveConfig(),
    "0-iterations": api.MoveConfig(move_and_slide_iterations=0),
    "1-iteration": api.MoveConfig(move_and_slide_iterations=1),
    "8-iterations": api.MoveConfig(move_and_slide_iterations=8, length_unit=2.0),
    "no-depenetration": api.MoveConfig(depenetration_iterations=0),
    "max-planes-3": api.MoveConfig(max_planes=3, plane_similarity_dot_threshold=0.9),   # characters carry up to 3 initial planes
}


@pytest.fixture(scope="module")
def random_scene():
    rng = np.random.default_rng(2024)
    cols, ignored = random_colliders(rng, 10_000, 22.0)
    batch = random_characters(rng, 3_000, 22.0, 10_000)
    return cols, ignored, batch


@pytest.mark.parametrize("scalar", SCALARS, ids=lambda s: np.dtype(s).name)
@pytest.mark.parametrize("name", list(CONFIGS))
def test_random_scene_matches_host(random_scene, name, scalar):
    cols, ignored, batch = random_scene
    cfg = CONFIGS[name]
    cfg.ignored = ignored
    if name != "default":                        # the host brute force is the slow side: the other configs on a third of the characters
        batch = take(batch, np.arange(1_000))
    with api.Context(device=0, scalar=scalar) as ctx:
        ctx.query_update(cols)
        got = ctx.move_and_slide(cfg, batch)
    want = fixture.move_and_slide(scalar, cols, cfg, batch)
    assert_bitwise(got, want, name)
    if cfg.move_and_slide_iterations:
        assert (want["hit_collider"] >= 0).sum() > 100, "the scene should make the characters hit something"


@pytest.mark.parametrize("scalar", SCALARS, ids=lambda s: np.dtype(s).name)
def test_dense_pile_windows_match_host(scalar):
    """Every character's grown AABB meets many times K = 16 candidates: the windowed walks and the depenetration list that does not fit."""
    rng = np.random.default_rng(7)
    n = 3000
    cols = api.QueryColliders(shape=np.ones(n, np.uint8), dims=np.full((n, 3), 0.08), position=rng.uniform(-1.2, 1.2, (n, 3)),
                              rotation=np.tile([0.0, 0.0, 0.0, 1.0], (n, 1)))
    m = 200
    batch = api.MoveBatch(shape=(np.arange(m) % 2).astype(np.uint8), dims=np.full((m, 3), 0.4), position=rng.uniform(-0.8, 0.8, (m, 3)),
                          rotation=random_quats(rng, m), velocity=rng.normal(size=(m, 3)) * 20)
    cfg = api.MoveConfig(penetration_rejection_threshold=2.0, depenetration_iterations=4)
    with api.Context(device=0, scalar=scalar) as ctx:
        ctx.query_update(cols)
        grown = 0.4 + 0.02                       # within every character's grown AABB (spheres of radius 0.4, cuboids of half size 0.4)
        cand = ctx.aabb_intersections((batch.position - grown).astype(scalar), (batch.position + grown).astype(scalar))
        counts = np.diff(cand["offsets"].astype(np.int64))
        assert counts.min() > 3 * 16, counts.min()
        got = ctx.move_and_slide(cfg, batch)
    assert_bitwise(got, fixture.move_and_slide(scalar, cols, cfg, batch), "pile")


def stack_world():
    sc = scenes.cube_stack(51, 40, 50, brick=True)
    return api.QueryColliders(shape=sc.shape_type.astype(np.uint8), dims=sc.dims, position=np.asarray(sc.bodies.position, np.float64),
                              rotation=np.asarray(sc.bodies.rotation, np.float64))


def walkers(rng, cols, n):
    """characters on top of the stack (some sunk a little into it), walking in random directions, half of them with a ground plane"""
    top = float(cols.position[1:, 1].max()) + 0.5
    lo, hi = cols.position[1:, [0, 2]].min(axis=0), cols.position[1:, [0, 2]].max(axis=0)
    shape = (rng.random(n) < 0.5).astype(np.uint8)
    dims = np.tile([0.3, 0.5, 0.3], (n, 1))
    half = np.where(shape == fixture.SHAPE_SPHERE, 0.3, 0.5)
    pos = np.stack([rng.uniform(lo[0], hi[0], n), top + half + rng.uniform(-0.05, 0.05, n), rng.uniform(lo[1], hi[1], n)], 1)
    a = rng.uniform(0, 2 * math.pi, n)
    vel = np.stack([np.cos(a) * 6, rng.uniform(-10, 0, n), np.sin(a) * 6], 1)
    planes = [np.array([[0.0, 1.0, 0.0]]) if i % 2 else None for i in range(n)]
    return api.MoveBatch(shape=shape, dims=dims, position=pos, rotation=np.tile([0.0, 0.0, 0.0, 1.0], (n, 1)), velocity=vel, planes=planes)


@pytest.mark.parametrize("scalar", SCALARS, ids=lambda s: np.dtype(s).name)
def test_walkers_on_the_100k_stack(scalar):
    rng = np.random.default_rng(3)
    cols = stack_world()
    batch = walkers(rng, cols, 100_000)
    cfg = api.MoveConfig()
    with api.Context(device=0, scalar=scalar) as ctx:
        ctx.query_update(cols)
        got = ctx.move_and_slide(cfg, batch)
    for k in ("position", "velocity"):
        assert np.isfinite(got[k]).all(), k
    assert (got["hit_collider"] >= 0).sum() > 10_000
    idx = np.sort(rng.choice(batch.count, 500, replace=False))
    want = fixture.move_and_slide(scalar, cols, cfg, take(batch, idx))
    assert_bitwise(rows(got, idx), want, "stack sample")


@pytest.mark.parametrize("scalar", SCALARS, ids=lambda s: np.dtype(s).name)
def test_non_finite_characters_and_the_call_before_any_update(scalar):
    cols = api.QueryColliders(shape=np.zeros(1, np.uint8), dims=np.array([[0.5, 5, 5]]), position=np.array([[2.0, 0, 0]]),
                              rotation=np.array([[0.0, 0, 0, 1]]))
    n = 5
    batch = api.MoveBatch(shape=np.ones(n, np.uint8), dims=np.full((n, 3), 0.5), position=np.zeros((n, 3)), rotation=np.tile([0.0, 0, 0, 1], (n, 1)),
                          velocity=np.tile([120.0, 0, 0], (n, 1)))
    batch.position[0, 1] = math.nan
    batch.velocity[1, 2] = math.inf
    batch.rotation[2] = 0.0
    batch.dims[3, 0] = math.inf
    cfg = api.MoveConfig()
    with api.Context(device=0, scalar=scalar) as ctx:
        with pytest.raises(api.AvianError) as e:
            ctx.move_and_slide(cfg, batch)
        assert e.value.status == api.ERR_INVALID_ARGUMENT
        ctx.query_update(cols)
        got = ctx.move_and_slide(cfg, batch)
        with pytest.raises(api.AvianError):
            ctx.move_and_slide(api.MoveConfig(ignored=np.zeros(2, np.uint8)), batch)
        with pytest.raises(api.AvianError):
            ctx.move_and_slide(api.MoveConfig(max_planes=api.MOVE_MAX_PLANES + 1), batch)
    assert_bitwise(got, fixture.move_and_slide(scalar, cols, cfg, batch), "non-finite")
    np.testing.assert_array_equal(got["position"][:4], batch.position[:4].astype(scalar))
    np.testing.assert_array_equal(got["velocity"][:4], batch.velocity[:4].astype(scalar))
    assert (got["hit_collider"][:4] == -1).all() and got["hit_collider"][4, 0] == 0
