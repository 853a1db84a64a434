"""Device narrow phase, the stand-alone geometry stage (SURVEY.md 8f #1): avn_narrow_phase against the host fixture's generator — the same
header (csrc/narrow_math.hpp) compiled by g++ and by nvcc — bit for bit: point counts, normals, anchors, penetrations, normal speeds and the
disjoint flags, on random cuboid / sphere soups (face, edge and vertex contacts, deep overlaps, near misses) in f32 and f64.  The contact
store runs the same geometry on its rows inside avn_contacts_step (tests/test_gpu_graph.py)."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
from avian_b200 import api, fixture  # noqa: E402

pytestmark = pytest.mark.gpu


def soup(n, seed, scalar, spheres=0.3, box=6.0):
    rng = np.random.default_rng(seed)
    pos = rng.uniform(0, box, size=(n, 3))
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[: n // 5] = (0, 0, 0, 1)                                   # some axis-aligned boxes: exact face-face and parallel-edge cases
    shape = (rng.random(n) < spheres).astype(np.uint8)
    dims = rng.uniform(0.2, 0.8, size=(n, 3))
    he = np.where(shape[:, None] == 1, dims[:, :1], np.abs(dims).max(axis=1, keepdims=True) * 1.8)
    cols = {"shape": shape, "dims": dims.astype(scalar), "position": pos.astype(scalar), "rotation": q.astype(scalar),
            "aabb_min": (pos - he).astype(scalar), "aabb_max": (pos + he).astype(scalar)}
    lv, av = rng.normal(0, 1.5, size=(n, 3)).astype(scalar), rng.normal(0, 2.0, size=(n, 3)).astype(scalar)
    # candidate pairs: everything within 2 units (plus some far ones for the disjoint flag)
    d = np.linalg.norm(pos[:, None] - pos[None], axis=2)
    i, j = np.nonzero(np.triu(d < 2.0, k=1))
    far = rng.integers(0, n, size=(50, 2))
    far = far[far[:, 0] != far[:, 1]]
    c1 = np.concatenate([i, far[:, 0]]).astype(np.uint32)
    c2 = np.concatenate([j, far[:, 1]]).astype(np.uint32)
    return cols, lv, av, (c1, c2, c1.copy(), c2.copy())


@pytest.mark.parametrize("scalar", [np.float32, np.float64])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_device_manifolds_equal_the_fixture(scalar, seed):
    cols, lv, av, pairs = soup(600, seed, scalar)
    want = fixture.raw_manifolds(scalar, 1.0 / 60.0, 0.005, pairs, cols, lv, av)
    with api.Context(device=0, scalar=scalar) as ctx:
        got = ctx.narrow_phase(1.0 / 60.0, 0.005, pairs, cols, lv, av)
    assert int((want["point_count"] > 0).sum()) > 300 and int((want["point_count"] == 4).sum()) > 10 and int(want["disjoint"].sum()) > 5
    for k in want:
        assert np.array_equal(got[k], want[k]), k


def test_without_aabbs_and_empty_input(gpu_ctx):
    cols, lv, av, pairs = soup(100, 9, np.float32)
    cols["aabb_min"] = cols["aabb_max"] = None
    want = fixture.raw_manifolds(np.float32, 1.0 / 60.0, 0.005, pairs, cols, lv, av)
    got = gpu_ctx.narrow_phase(1.0 / 60.0, 0.005, pairs, cols, lv, av)
    for k in want:
        assert np.array_equal(got[k], want[k]), k
    empty = tuple(np.zeros(0, dtype=np.uint32) for _ in range(4))
    assert gpu_ctx.narrow_phase(1.0 / 60.0, 0.005, empty, cols, lv, av)["point_count"].shape == (0,)
    bad = (np.array([1000], dtype=np.uint32),) * 4
    with pytest.raises(api.AvianError):
        gpu_ctx.narrow_phase(1.0 / 60.0, 0.005, bad, cols, lv, av)
