"""Bodies with several colliders, offset from the body origin, and a centre of mass off the origin, in the host fixture: the anchor
transform of update_contacts against an independent restatement (tests/compound_reference.py), zero frames against the frame-less path,
a scene re-expressed from other body origins stepping like the original, the physics of compound bodies, and the ABI mirror."""
import copy
import ctypes as C
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
from avian_b200 import api, fixture, plugins, scenes  # noqa: E402
import compound_reference as ref  # noqa: E402
import oracle_lib  # noqa: E402
from compound_scenes import DT, TOL, soup  # noqa: E402

SCALARS = [np.float32, np.float64]


@pytest.mark.parametrize("scalar", SCALARS)
@pytest.mark.parametrize("with_com", [True, False])
def test_row_transform_matches_the_restatement(scalar, with_com):
    """anchors, normal speeds and keep decisions of the framed fixture equal the restatement applied to the frame-less witnesses, on the
    points the keep rule's first clause keeps either way (the decisions away from the threshold)"""
    pairs, cols, lv, av, frames = soup(scalar, 3 + with_com, with_com=with_com)
    plain = fixture.raw_manifolds(scalar, DT, TOL, pairs, cols, lv, av, f64_anchors=True)
    framed = fixture.raw_manifolds(scalar, DT, TOL, pairs, cols, lv, av, frames=frames)
    c1, c2, b1, b2 = pairs
    eps = np.finfo(scalar).eps
    com = frames["center_of_mass"] if with_com else np.zeros_like(frames["position"])
    checked = 0
    for k in range(c1.shape[0]):
        n = int(plain["point_count"][k])
        pen = plain["penetration"][k, :n].astype(np.float64)
        m = DT * np.linalg.norm(lv[b2[k]].astype(float) - lv[b1[k]].astype(float))
        if n == 0 or not (-pen < m * 0.999).all():
            continue
        assert framed["point_count"][k] == n, k
        a1 = ref.transform(plain["anchor1_f64"][k, :n], cols["position"][c1[k]], frames["position"][b1[k]], frames["rotation"][b1[k]], com[b1[k]])
        a2 = ref.transform(plain["anchor2_f64"][k, :n], cols["position"][c2[k]], frames["position"][b2[k]], frames["rotation"][b2[k]], com[b2[k]])
        scale = 4.0 + np.abs(frames["position"][[b1[k], b2[k]]]).max()
        assert np.abs(framed["anchor1"][k, :n] - a1).max() <= 64 * eps * scale, k
        assert np.abs(framed["anchor2"][k, :n] - a2).max() <= 64 * eps * scale, k
        ns = ref.normal_speed(a1, a2, framed["normal"][k], lv[b1[k]], av[b1[k]], lv[b2[k]], av[b2[k]])
        assert np.abs(framed["normal_speed"][k, :n] - ns).max() <= 256 * eps * scale * 10.0, k
        assert ref.keep(pen, ns, DT, lv[b1[k]], lv[b2[k]]).all()
        assert np.array_equal(framed["penetration"][k, :n], plain["penetration"][k, :n])
        checked += 1
    assert checked > 100


@pytest.mark.parametrize("scalar", SCALARS)
def test_zero_frames_equal_the_frameless_path(scalar):
    pairs, cols, lv, av, frames = soup(scalar, 9, zero_frames=True)
    plain = fixture.raw_manifolds(scalar, DT, TOL, pairs, cols, lv, av)
    framed = fixture.raw_manifolds(scalar, DT, TOL, pairs, cols, lv, av, frames=frames)
    for k in plain:
        assert (framed[k] == plain[k]).all(), k


@pytest.mark.parametrize("scalar", SCALARS)
def test_the_row_function_with_frames_equals_the_geometry_stage(scalar):
    """avh_rows_narrow_framed (csrc/contact_rows.hpp, what the device runs per row) gives the geometry stage's framed manifolds"""
    pairs, cols, lv, av, frames = soup(scalar, 21)
    want = fixture.raw_manifolds(scalar, DT, TOL, pairs, cols, lv, av, frames=frames)
    c1, c2, b1, b2 = (np.ascontiguousarray(x) for x in pairs)
    E, s = int(c1.shape[0]), np.dtype(scalar)
    z = lambda *sh, d=s: np.zeros(sh, dtype=d)
    live, count, disjoint = np.ones(E, dtype=np.uint8), z(E, d=np.uint8), z(E, d=np.uint8)
    normal, a1, a2, pen, ns = z(E, 3), z(E, 4, 3), z(E, 4, 3), z(E, 4), z(E, 4)
    prev_count, prev_a1, prev_a2 = z(E, d=np.uint8), z(E, 4, 3, d=np.float64), z(E, 4, 3, d=np.float64)
    ws = [z(E, 4), z(E, 4, 2), z(E, 4), z(E, 4, 2)]
    big = np.full((cols["position"].shape[0], 3), 1e6, dtype=s)   # AABBs that always overlap
    lo = -big
    p = fixture._p
    fixture._load().avh_rows_narrow_framed(
        32 if s == np.float32 else 64, E, p(c1), p(c2), p(b1), p(b2), p(live), p(count), p(disjoint), p(normal), p(a1), p(a2), p(pen), p(ns),
        p(prev_count), p(prev_a1), p(prev_a2), *(p(w) for w in ws), p(cols["shape"]), p(cols["dims"]), p(cols["position"]), p(cols["rotation"]),
        p(lv), p(av), p(lo), p(big), DT, TOL, 1.0, 1, p(frames["position"]), p(frames["rotation"]), p(frames["center_of_mass"]))
    assert np.array_equal(count, want["point_count"])
    for got, k in ((normal, "normal"), (a1, "anchor1"), (a2, "anchor2"), (pen, "penetration"), (ns, "normal_speed")):
        assert np.array_equal(got, want[k]), k


def _com_world(b):
    return b.position.astype(np.float64) + ref.qrot(b.rotation, b.center_of_mass)


def test_reexpressed_body_origins_step_like_the_original():
    """a single-collider scene whose body origins move off their colliders by d_i (centre of mass = d_i) gives the same contact counts and
    the same centre-of-mass poses and velocities for 60 steps.  Collider and centre of mass share their local point here, so the anchor
    transform's two terms cancel: this pins the World's pose propagation and the writeback about the centre of mass; the transform itself is
    pinned by the restatement above and by the L-block and dumbbell below.  In f32, on one layer of cubes resting on the ground, where the
    rounding of the re-expressed poses stays near 1e-6 (the oracle's f64 build leaves the velocity columns at zero after a step)."""
    sc = scenes.cube_stack(4, 1, 4, scalar=np.float32)
    rng = np.random.default_rng(5)
    d = rng.uniform(-0.4, 0.4, size=(sc.bodies.count, 3))
    sc2 = scenes.with_collider_table(copy.deepcopy(sc), offset=d)
    wa = plugins.World(sc, oracle_lib.oracle_plugins())
    wb = plugins.World(sc2, oracle_lib.oracle_plugins())
    for i in range(60):
        wa.step(); wb.step()
        ma, mb = wa.last_manifolds, wb.last_manifolds
        assert ma.count == mb.count, i   # contact counts; a point near the keep threshold may go either way in f32
        assert np.abs(_com_world(wb.bodies) - wa.bodies.position).max() < 2e-5, i
        for k in ("rotation", "linear_velocity", "angular_velocity"):
            assert np.abs(getattr(wb.bodies, k) - getattr(wa.bodies, k)).max() < 2e-5, (i, k)
    assert ma.count > 0


def _lblock(com_shift):
    """an L-block (a foot along x and an upright at its -x end) on the ground, its centre of mass moved by com_shift along x"""
    parts = [(scenes.SHAPE_CUBOID, (0.5, 0.1, 0.3), (0.5, 0.1, 0.0), (0, 0, 0, 1.0)), (scenes.SHAPE_CUBOID, (0.1, 0.6, 0.3), (0.1, 0.8, 0.0), (0, 0, 0, 1.0))]
    M, c, I = scenes.compound_mass(parts)
    Ii = np.linalg.inv(I)
    com = c + np.array([com_shift, 0.0, 0.0])
    s = np.float32
    b = api.Bodies(kind=np.array([api.BODY_STATIC, api.BODY_DYNAMIC], np.uint8), position=np.array([[0, -0.5, 0], [0, 0.005, 0]], s),
                   rotation=np.array([[0, 0, 0, 1], [0, 0, 0, 1]], s), linear_velocity=np.zeros((2, 3), s), angular_velocity=np.zeros((2, 3), s),
                   inverse_mass=np.array([0, 1 / M], s), inverse_inertia_local=np.array([np.zeros(6), [Ii[0, 0], Ii[0, 1], Ii[0, 2], Ii[1, 1], Ii[1, 2], Ii[2, 2]]], s),
                   center_of_mass=np.array([np.zeros(3), com], s))
    return scenes.Scene("lblock", b, np.zeros(2, np.int32), np.array([[10, 0.5, 10], [0.5, 0.1, 0.3]]), np.full(2, 0.5), np.zeros(2),
                        collider_body=np.array([0, 1, 1], np.int32), local_position=np.array([[0, 0, 0], parts[0][2], parts[1][2]], float),
                        local_rotation=np.tile([0, 0, 0, 1.0], (3, 1)), collider_shape=np.zeros(3, np.int32),
                        collider_dims=np.array([[10, 0.5, 10], parts[0][1], parts[1][1]], float), collider_friction=np.full(3, 0.5),
                        collider_restitution=np.zeros(3))


@pytest.mark.parametrize("com_shift,tips", [(0.0, False), (-0.5, True)])
def test_an_l_block_rests_or_tips_by_its_centre_of_mass(com_shift, tips):
    """the block's parts' centre of mass lies over the foot: it comes to rest.  Moved past the foot's -x edge it tips over that edge."""
    w = plugins.World(_lblock(com_shift), oracle_lib.oracle_plugins())
    for _ in range(180):
        w.step()
    q = w.bodies.rotation[1].astype(float)
    tilt = np.degrees(2 * np.arcsin(min(1.0, np.linalg.norm(q[:3]))))
    if tips:
        assert tilt > 30.0, tilt
    else:
        assert tilt < 1.0 and np.abs(w.bodies.linear_velocity[1]).max() < 0.05, (tilt, w.bodies.linear_velocity[1])


def test_a_dumbbell_rolls_without_drifting_sideways():
    """a dumbbell (two equal spheres on a capsule along x) pushed along z rolls along z and keeps its x"""
    parts = [(scenes.SHAPE_CAPSULE, (0.08, 0.4, 0.0), (0, 0, 0), scenes._Z90), (scenes.SHAPE_SPHERE, (0.2, 0, 0), (-0.4, 0, 0), (0, 0, 0, 1.0)),
             (scenes.SHAPE_SPHERE, (0.2, 0, 0), (0.4, 0, 0), (0, 0, 0, 1.0))]
    M, c, I = scenes.compound_mass(parts)
    Ii = np.linalg.inv(I)
    s = np.float32
    origin = np.array([-0.4, 0.0, 0.0])   # the body origin at one weight's centre
    b = api.Bodies(kind=np.array([api.BODY_STATIC, api.BODY_DYNAMIC], np.uint8), position=np.array([[0, -0.5, 0], [-0.4, 0.201, 0]], s),
                   rotation=np.array([[0, 0, 0, 1], [0, 0, 0, 1]], s), linear_velocity=np.array([[0, 0, 0], [0, 0, 1.0]], s),
                   angular_velocity=np.array([[0, 0, 0], [1.0 / 0.2, 0, 0]], s), inverse_mass=np.array([0, 1 / M], s),
                   inverse_inertia_local=np.array([np.zeros(6), [Ii[0, 0], Ii[0, 1], Ii[0, 2], Ii[1, 1], Ii[1, 2], Ii[2, 2]]], s),
                   center_of_mass=np.array([np.zeros(3), c - origin], s))
    lp = np.array([[0, 0, 0]] + [np.asarray(p[2]) - origin for p in parts], float)
    sc = scenes.Scene("dumbbell", b, np.zeros(2, np.int32), np.array([[20, 0.5, 20], [0.2, 0, 0]]), np.full(2, 0.5), np.zeros(2),
                      collider_body=np.array([0, 1, 1, 1], np.int32), local_position=lp,
                      local_rotation=np.array([[0, 0, 0, 1.0]] + [p[3] for p in parts], float), collider_shape=np.array([0, 2, 1, 1], np.int32),
                      collider_dims=np.array([[20, 0.5, 20]] + [p[1] for p in parts], float), collider_friction=np.full(4, 0.5),
                      collider_restitution=np.zeros(4))
    w = plugins.World(sc, oracle_lib.oracle_plugins())
    x0 = float(_com_world(w.bodies)[1, 0])
    for _ in range(120):
        w.step()
    com = _com_world(w.bodies)[1]
    assert com[2] > 1.0 and abs(com[0] - x0) < 1e-3, com
    assert abs(com[1] - 0.2) < 0.01, com


def test_compound_pile_mass_properties_and_layout():
    sc = scenes.compound_pile(60, seed=2, single_share=0.2)
    b = sc.bodies
    assert sc.compound and sc.collider_body[0] == 0 and (np.diff(sc.collider_body) >= 0).all()
    parts = np.bincount(sc.collider_body, minlength=b.count)[1:]
    assert parts.min() >= 1 and parts.max() <= 5 and (parts >= 2).sum() > 30
    multi = np.flatnonzero(parts >= 2) + 1
    assert (np.linalg.norm(b.center_of_mass[multi], axis=1) > 0.05).all()   # the origins are away from the centres of mass
    # a table's parallel-axis inertia against a direct sum over its parts
    M, c, I = scenes.compound_mass([(0, (1.0, 0.1, 0.5), (0, 1, 0), (0, 0, 0, 1.0)), (1, (0.3, 0, 0), (0, 0, 0), (0, 0, 0, 1.0))])
    m1, m2 = 8.0 * 1.0 * 0.1 * 0.5, 4.0 / 3.0 * np.pi * 0.3 ** 3
    assert np.isclose(M, m1 + m2) and np.allclose(c, [0, m1 / (m1 + m2), 0])
    d1, d2 = 1 - c[1], c[1]
    assert np.isclose(I[0, 0], m1 / 12 * (0.2 ** 2 + 1.0) + m1 * d1 ** 2 + 0.4 * m2 * 0.09 + m2 * d2 ** 2)


def test_body_frames_layout_matches_the_header():
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "avian_b200.h"\nint main(){printf("%zu %zu\\n", sizeof(AvnBodyFrames), offsetof(AvnBodyFrames, center_of_mass));return 0;}'
    with tempfile.TemporaryDirectory() as d:
        (Path(d) / "s.c").write_text(src)
        subprocess.run(["gcc", "-I", str(ROOT / "include"), "-o", f"{d}/s", f"{d}/s.c"], check=True)
        size, off = map(int, subprocess.run([f"{d}/s"], capture_output=True, text=True, check=True).stdout.split())
    assert size == C.sizeof(api.AvnBodyFrames) and off == api.AvnBodyFrames.center_of_mass.offset
    assert "avn_contacts_set_body_frames" in api.ABI_SYMBOLS


def test_world_refuses_ccd_with_a_collider_table():
    with pytest.raises(ValueError):
        plugins.World(scenes.compound_pile(4), oracle_lib.oracle_plugins(), ccd={"body": [1]})
