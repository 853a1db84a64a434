"""Spatial queries on the host: hand-worked answers (computed here with plain numpy, independently of csrc/query_math.hpp) that the fixture's
brute force must reproduce, the ABI struct layouts of the query entry points, and the inputs the host path refuses."""
import ctypes as C
import subprocess
import tempfile
from pathlib import Path

import numpy as np
import pytest

from avian_b200 import api, fixture

ROOT = Path(__file__).resolve().parent.parent
S2 = np.sqrt(0.5)
IDENT = [0.0, 0.0, 0.0, 1.0]
ROT_Z45 = [0.0, 0.0, np.sin(np.pi / 8), np.cos(np.pi / 8)]
TOL = {np.float32: 1e-6, np.float64: 1e-12}


def colliders(*items, memberships=None):
    """items: (shape, dims, position, rotation)"""
    sh, dm, ps, rt = zip(*items)
    return api.QueryColliders(shape=np.array(sh, np.uint8), dims=np.array([np.broadcast_to(d, 3) for d in dm], float), position=np.array(ps, float),
                              rotation=np.array(rt, float), memberships=None if memberships is None else np.array(memberships, np.uint32))


def cast(scalar, cols, o, d, maxd=100.0, solid=True, mask=None, exclude=None):
    rays = api.Rays(origin=np.array([o], float), direction=np.array([d], float), max_distance=np.array([maxd]), solid=np.array([solid]),
                    mask=None if mask is None else np.array([mask], np.uint32), exclude=None if exclude is None else [exclude])
    r = fixture.query_cast_ray(scalar, cols, rays)
    return int(r["collider"][0]), float(r["distance"][0]), r["normal"][0].astype(np.float64)


BOX = (0, 1.0, [0.0, 0.0, 0.0], IDENT)
SPHERE = (1, [1.0, 0.0, 0.0], [0.0, 0.0, 0.0], IDENT)

# (name, colliders, ray kwargs, expected collider, expected t, expected normal)
CASES = [
    ("box_axis_aligned", [BOX], dict(o=[-5, 0.2, 0.3], d=[1, 0, 0]), 0, 4.0, [-1, 0, 0]),
    # rotated 45 deg about z: at height y = 0.3 the ray meets the face -x s + y c = 1 first (x = 0.3 - sqrt 2)
    ("box_rotated_45", [(0, 1.0, [0, 0, 0], ROT_Z45)], dict(o=[-5, 0.3, 0.1], d=[1, 0, 0]), 0, 5.3 - np.sqrt(2), [-S2, S2, 0]),
    ("sphere_front", [SPHERE], dict(o=[-5, 0.6, 0], d=[1, 0, 0]), 0, 4.2, [-0.8, 0.6, 0]),
    ("sphere_tangent", [SPHERE], dict(o=[-5, 1.0, 0], d=[1, 0, 0]), 0, 5.0, [0, 1, 0]),
    ("sphere_miss", [SPHERE], dict(o=[-5, 1.01, 0], d=[1, 0, 0]), -1, 0.0, [0, 0, 0]),
    ("box_inside_solid", [BOX], dict(o=[0.2, 0, 0], d=[1, 0, 0]), 0, 0.0, [0, 0, 0]),
    ("box_inside_hollow", [BOX], dict(o=[0.2, 0, 0], d=[1, 0, 0], solid=False), 0, 0.8, [1, 0, 0]),
    ("sphere_inside_solid", [SPHERE], dict(o=[0, 0.6, 0], d=[1, 0, 0]), 0, 0.0, [0, 0, 0]),
    ("sphere_inside_hollow", [SPHERE], dict(o=[0, 0.6, 0], d=[1, 0, 0], solid=False), 0, 0.8, [0.8, 0.6, 0]),
    ("at_max_distance", [BOX], dict(o=[-5, 0, 0], d=[1, 0, 0], maxd=4.0), 0, 4.0, [-1, 0, 0]),
    ("beyond_max_distance", [BOX], dict(o=[-5, 0, 0], d=[1, 0, 0], maxd=float(np.nextafter(np.float32(4.0), np.float32(0.0)))), -1, 0.0, [0, 0, 0]),
    ("zero_components_inside_slabs", [BOX], dict(o=[0.5, -0.5, -5], d=[0, 0, 1]), 0, 4.0, [0, 0, -1]),
    ("zero_components_on_slab_face", [BOX], dict(o=[1.0, 1.0, -5], d=[0, 0, 1]), 0, 4.0, [0, 0, -1]),
    ("zero_components_outside_slab", [BOX], dict(o=[1.5, 0, -5], d=[0, 0, 1]), -1, 0.0, [0, 0, 0]),
    # through the edge x = y = -1: x and y enter at the same t, the tie goes to the lowest axis
    ("edge_tie_lowest_axis", [BOX], dict(o=[-2, -2, 0], d=[S2, S2, 0]), 0, np.sqrt(2), [-1, 0, 0]),
    ("box_behind", [BOX], dict(o=[5, 0, 0], d=[1, 0, 0]), -1, 0.0, [0, 0, 0]),
    # two boxes on the ray: the near one (x in [-1, 1]) is on layer 2 only, the far one (x in [4, 6]) on layer 1
    ("mask_excludes_nearest", [BOX, (0, 1.0, [5, 0, 0], IDENT)], dict(o=[-5, 0, 0], d=[1, 0, 0], mask=1), 1, 9.0, [-1, 0, 0]),
    ("excluded_entity", [BOX, (0, 1.0, [5, 0, 0], IDENT)], dict(o=[-5, 0, 0], d=[1, 0, 0], exclude=[0]), 1, 9.0, [-1, 0, 0]),
    ("equal_distance_lowest_index", [(1, [1.0, 0, 0], [0, 0, 0], IDENT), BOX], dict(o=[-5, 0, 0], d=[1, 0, 0]), 0, 4.0, [-1, 0, 0]),
]


@pytest.mark.parametrize("scalar", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_hand_worked_ray_casts(case, scalar):
    name, items, ray, want_c, want_t, want_n = case
    cols = colliders(*items, memberships=[2, 1] if name == "mask_excludes_nearest" else None)
    c, t, n = cast(scalar, cols, **ray)
    assert c == want_c
    assert abs(t - want_t) <= TOL[scalar] * max(1.0, abs(want_t))
    assert np.allclose(n, want_n, rtol=0, atol=TOL[scalar])


@pytest.mark.parametrize("scalar", [np.float32, np.float64], ids=["f32", "f64"])
def test_hand_worked_ray_hits_and_aabbs(scalar):
    cols = colliders(BOX, (1, [1.0, 0, 0], [5, 0, 0], IDENT), (0, 1.0, [10, 0, 0], IDENT))
    rays = api.Rays(origin=np.array([[-5.0, 0, 0]] * 4), direction=np.array([[1.0, 0, 0]] * 4), max_distance=np.full(4, 100.0),
                    max_hits=np.array([api.MAX_HITS_ALL, 2, 0, 1], np.uint32))
    h = fixture.query_ray_hits(scalar, cols, rays)
    assert h["offsets"].tolist() == [0, 3, 5, 5, 6]
    assert h["collider"].tolist() == [0, 1, 2, 0, 1, 0]
    assert np.allclose(h["distance"], [4, 9, 14, 4, 9, 4], atol=TOL[scalar])
    assert np.allclose(h["normal"], [[-1, 0, 0]] * 6, atol=TOL[scalar])
    # Aabb::intersects is inclusive: touching the box [-1, 1]^3 at a corner counts, a gap of 1e-3 does not
    q = fixture.query_aabb_intersections(scalar, cols, [[1, 1, 1], [1.001, 1.001, 1.001], [-20, -0.5, -0.5]], [[2, 2, 2], [2, 2, 2], [20, 0.5, 0.5]])
    assert q["offsets"].tolist() == [0, 1, 1, 4]
    assert q["collider"].tolist() == [0, 0, 1, 2]


def test_non_finite_inputs_hit_nothing():
    cols = colliders(BOX, (0, 1.0, [np.nan, 0, 0], IDENT), (0, [1.0, np.inf, 1.0], [0, 0, 0], IDENT))
    assert cast(np.float64, cols, o=[-5, 0, 0], d=[1, 0, 0], exclude=[0])[0] == -1
    assert cast(np.float64, cols, o=[np.nan, 0, 0], d=[1, 0, 0])[0] == -1
    assert cast(np.float64, cols, o=[-5, 0, 0], d=[1, 0, 0], maxd=np.inf)[0] == -1
    q = fixture.query_aabb_intersections(np.float64, cols, [[-1e9] * 3], [[1e9] * 3])
    assert q["collider"].tolist() == [0]


def test_aabb_and_ray_test_describe_the_same_box_for_non_unit_quaternions():
    """the tight AABB covers every point the exact ray test accepts, whatever |q|: for each axis, the corner of the box that is extreme
    along it (just inside, by 1e-9 relative) is on a ray that hits the box and lies inside the collider's AABB (a zero-size AABB query there
    reports it).  Both use the normalised rotation; with |q|^2 R they differ by about 2 |1 - |q|^2| of the extent."""
    rng = np.random.default_rng(3)
    for trial in range(40):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        q *= np.sqrt(1.0 + (1e-7 if trial % 2 else -1e-7) * (1 + trial % 3))
        he = rng.uniform(0.2, 2.0, 3)
        cols = colliders((0, he, [0.0, 0.0, 0.0], q))
        x, y, z, w = q / np.linalg.norm(q)
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                      [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                      [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
        for j in range(3):
            corner = R @ (np.sign(R[j]) * he * (1.0 - 1e-9))
            d = np.zeros(3)
            d[(j + 1) % 3] = 1.0
            c, t, _ = cast(np.float64, cols, o=corner - 5.0 * d, d=d)     # passes through a point inside the box
            assert c == 0 and 0 < t <= 5.0, (trial, j)
            q_hit = fixture.query_aabb_intersections(np.float64, cols, [corner], [corner])
            assert q_hit["collider"].tolist() == [0], (trial, j)


def test_degenerate_rotation_is_never_reported():
    cols = colliders(BOX, (0, 1.0, [0, 0, 0], [0.0, 0.0, 0.0, 0.0]), (1, [1.0, 0, 0], [0, 0, 0], [0.0, 0.0, 0.0, 0.0]))
    assert cast(np.float64, cols, o=[-5, 0, 0], d=[1, 0, 0], exclude=[0])[0] == -1
    assert fixture.query_aabb_intersections(np.float64, cols, [[-1, -1, -1]], [[1, 1, 1]])["collider"].tolist() == [0]


def test_refused_inputs():
    cols = colliders(BOX, BOX)
    rays = api.Rays(origin=np.zeros((2, 3)), direction=np.array([[1.0, 0, 0]] * 2), max_distance=np.ones(2), exclude=[[0], [1]])
    r, keep = rays.as_struct(np.float64)
    keep[6][:] = [0, 2, 1]                     # exclude_offsets not monotone
    c, keep_c = cols.as_struct(np.float64)
    lib = fixture._load()
    out = api.AvnRayClosest(*(a.ctypes.data for a in (np.zeros(2, np.int32), np.zeros(2), np.zeros((2, 3)))))
    assert lib.avh_query_cast_ray(64, C.byref(c), C.byref(r), C.byref(out)) == api.ERR_INVALID_ARGUMENT
    assert b"monotone" in lib.avh_query_error()
    keep[6][:] = [0, 1, 3]                     # past exclude_count
    assert lib.avh_query_cast_ray(64, C.byref(c), C.byref(r), C.byref(out)) == api.ERR_INVALID_ARGUMENT
    bad = colliders(BOX, (2, 1.0, [0, 0, 0], IDENT))
    with pytest.raises(api.AvianError) as e:
        fixture.query_ray_hits(np.float64, bad, api.Rays(origin=np.zeros((1, 3)), direction=np.array([[1.0, 0, 0]]), max_distance=np.ones(1)))
    assert e.value.status == api.ERR_INVALID_ARGUMENT and "unknown shape" in str(e.value)
    with pytest.raises(api.AvianError):
        fixture.query_aabb_intersections(np.float32, bad, np.zeros((1, 3)), np.ones((1, 3)))
    for neg in (colliders(BOX, (0, [1.0, -0.5, 1.0], [0, 0, 0], IDENT)), colliders((1, [-1.0, 0, 0], [0, 0, 0], IDENT))):
        for scalar in (np.float32, np.float64):
            with pytest.raises(api.AvianError) as e:
                fixture.query_cast_ray(scalar, neg, api.Rays(origin=np.zeros((1, 3)), direction=np.array([[1.0, 0, 0]]), max_distance=np.ones(1)))
            assert e.value.status == api.ERR_INVALID_ARGUMENT and "negative" in str(e.value)


def test_query_struct_layouts_match_the_header():
    """sizeof of every spatial-query ABI struct, compiled from the header with gcc, equals the ctypes mirror"""
    names = ["AvnQueryColliders", "AvnRayBatch", "AvnRayClosest", "AvnHitList"]
    src = '#include <stdio.h>\n#include "avian_b200.h"\nint main(){' + "".join(f'printf("{n} %zu\\n", sizeof({n}));' for n in names) + "return 0;}"
    with tempfile.TemporaryDirectory() as d:
        (Path(d) / "s.c").write_text(src)
        subprocess.run(["gcc", "-I", str(ROOT / "include"), "-o", f"{d}/s", f"{d}/s.c"], check=True)
        out = subprocess.run([f"{d}/s"], capture_output=True, text=True, check=True).stdout
    sizes = dict(line.split() for line in out.strip().splitlines())
    for n in names:
        assert int(sizes[n]) == C.sizeof(getattr(api, n)), n
