"""Swept CCD with capsule colliders on the device (avn_ccd_configure with AVN_CCD_CAPSULES): the CAPS = true TOI kernel against the host
brute force (avh_ccd_solve) bit for bit on a capsule pile under fire, the device world beside the oracle world, a capsule bullet at a thin
wall, and the flag leaving capsule-free scenes byte for byte as they were."""
from __future__ import annotations

import numpy as np
import pytest

from avian_b200 import api, plugins, scenes
from avian_b200.fixture import SHAPE_CAPSULE, SHAPE_CUBOID, SHAPE_SPHERE
from helpers import assert_bodies_close
from oracle_ccd import oracle_ccd_plugins
from test_gpu_ccd import mixed_config, pile_with_projectiles, step_and_check

pytestmark = pytest.mark.gpu
SCALARS = [np.float32, np.float64]


def capsule_pile_with_projectiles(scalar, n=120, layers=3, projectiles=36, seed=0, kinematic_bat=False):
    """scenes.capsule_pile on its static ground (body 0) with capsule, sphere and cube projectiles fired at random pile bodies from 3-5 m at
    250-400 m/s, and one long capsule bat spinning at 60 rad/s just above a pile body.  Returns the scene and the CCD bodies (the
    projectiles and the bat)."""
    base = scenes.capsule_pile(n, seed=8, layers=layers, scalar=scalar)
    b = base.bodies
    rng = np.random.default_rng(seed)
    n0 = b.count
    aim = b.position[1 + rng.integers(0, n, projectiles)].astype(np.float64)
    d = rng.normal(size=(projectiles, 3))
    d[:, 1] = np.abs(d[:, 1])
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    ppos = aim + d * rng.uniform(3.0, 5.0, (projectiles, 1))
    pvel = -d * rng.uniform(250.0, 400.0, (projectiles, 1))
    pshape = np.array([SHAPE_CAPSULE, SHAPE_SPHERE, SHAPE_CUBOID])[np.arange(projectiles) % 3]
    pdims = np.select([pshape[:, None] == SHAPE_CAPSULE, pshape[:, None] == SHAPE_SPHERE], [np.array([[0.1, 0.25, 0]]), np.array([[0.15, 0, 0]])],
                      np.array([[0.15, 0.15, 0.15]]))
    q = rng.normal(size=(projectiles, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    top = b.position[1:].astype(np.float64)
    bat_pos = top[np.argmax(top[:, 1])] + np.array([0.0, 1.2, 0.0])
    s = np.sqrt(0.5)
    pos = np.concatenate([b.position.astype(np.float64), ppos, bat_pos[None]])
    rot = np.concatenate([b.rotation.astype(np.float64), q, [[0, 0, -s, s]]])          # the bat lies along x
    kind = np.concatenate([b.kind, np.zeros(projectiles, np.uint8), [api.BODY_KINEMATIC if kinematic_bat else api.BODY_DYNAMIC]])
    shape = np.concatenate([base.shape_type, pshape, [SHAPE_CAPSULE]])
    dims = np.concatenate([base.dims, pdims, [[0.05, 2.0, 0.0]]])
    linvel = np.concatenate([b.linear_velocity.astype(np.float64), pvel, [[0, 0, 0]]])
    angvel = np.concatenate([b.angular_velocity.astype(np.float64), np.zeros((projectiles, 3)), [[0, 60.0, 0]]])
    scene = scenes._assemble("capsule_ccd_pile", pos, rot, kind, dims, shape, scalar, linvel=linvel, angvel=angvel)
    return scene, np.arange(n0, n0 + projectiles + 1)


def capsule_config(ccd, seed=1):
    cfg = mixed_config(ccd, seed)
    cfg["mode"] = (np.arange(ccd.shape[0]) % 2).astype(np.uint8)   # half Linear, half NonLinear
    cfg["capsules"] = True
    return cfg


@pytest.mark.parametrize("scalar", SCALARS)
@pytest.mark.parametrize("kinematic_bat", [False, True])
def test_device_pass_equals_host_brute_force(scalar, kinematic_bat):
    scene, ccd = capsule_pile_with_projectiles(scalar, kinematic_bat=kinematic_bat)
    cfg = capsule_config(ccd)
    with api.Context(device=0, scalar=scalar) as ctx:
        w = plugins.DeviceGraphWorld(scene, plugins.PhysicsPlugins(ctx), ctx, substeps=4)
        ctx.ccd_configure(**cfg)
        hits = capsule_hits = 0
        for _ in range(4):
            got = step_and_check(ctx, w, cfg, scalar)
            hit = got["hit_body"] >= 0
            hits += int(hit.sum())
            capsule_hits += int((hit & ((scene.shape_type[ccd] == SHAPE_CAPSULE) | (scene.shape_type[np.maximum(got["hit_body"], 0)] == SHAPE_CAPSULE))).sum())
        assert hits > 0 and capsule_hits > 0


def test_device_world_beside_oracle_world():
    """DeviceGraphWorld(ccd={..., capsules}) beside World(oracle solver stage + solve_swept_ccd): the CCD decisions bit-identical every step,
    the bodies within the parity bar."""
    scalar = np.float32
    make = lambda: capsule_pile_with_projectiles(scalar, n=40, layers=2, projectiles=12, seed=2)
    cfg = capsule_config(make()[1])
    with api.Context(device=0, scalar=scalar) as ctx:
        dev = plugins.DeviceGraphWorld(make()[0], plugins.PhysicsPlugins(ctx), ctx, substeps=4, ccd=cfg)
        ref = plugins.World(make()[0], oracle_ccd_plugins(), substeps=4, ccd=cfg)
        hits = 0
        for step in range(30):
            dev.step()
            ref.step()
            got = ctx.ccd_download()
            want = ref.plugins.get("SolverPlugin").last_ccd
            assert np.array_equal(got["min_toi"], np.array([w[0] for w in want], scalar)), step
            assert np.array_equal(got["hit_body"], np.array([w[1] for w in want])), step
            assert np.array_equal(got["hit_contact"], np.array([w[2] for w in want])), step
            assert_bodies_close(dev.bodies, ref.bodies, what=f"capsule ccd step {step}: ")
            hits += int((got["hit_body"] >= 0).sum())
        assert hits > 0


@pytest.mark.parametrize("scalar", SCALARS)
@pytest.mark.parametrize("mode", [api.SWEEP_LINEAR, api.SWEEP_NON_LINEAR])
def test_capsule_bullet_at_a_thin_wall(scalar, mode):
    # a 300 m/s capsule at a 0.04 m static wall 4 m away ends the step on the near side, the pass's decisions equal to the host's.  (With the
    # default speculative margin the substeps' speculative contact already stops it, so the pass finds no TOI left, as for the sphere of
    # test_ccd_world_cpu.test_fast_sphere_stops_at_thin_wall.)
    scene = scenes._assemble("capsule_bullet", np.array([[0, 0, 0], [4.0, 0, 0]]), np.tile([0, 0, 0, 1.0], (2, 1)),
                             np.array([api.BODY_DYNAMIC, api.BODY_STATIC]), np.array([[0.05, 0.2, 0], [0.02, 3, 3]]),
                             np.array([SHAPE_CAPSULE, SHAPE_CUBOID]), scalar, linvel=np.array([[300.0, 0, 0], [0, 0, 0]]))
    cfg = dict(body=np.array([0]), collider=np.array([0]), mode=np.array([mode], np.uint8), capsules=True)
    with api.Context(device=0, scalar=scalar) as ctx:
        w = plugins.DeviceGraphWorld(scene, plugins.PhysicsPlugins(ctx), ctx, substeps=4, ccd=cfg)
        step_and_check(ctx, w, cfg, scalar)
        assert float(w.bodies.position[0, 0]) + 0.05 <= 4.0 - 0.02 + 1e-3


@pytest.mark.parametrize("scalar", SCALARS)
def test_flag_without_capsules_changes_nothing(scalar):
    """With AVN_CCD_CAPSULES set and no capsule in the scene the pass runs the CAPS = false kernel: results and bodies byte-identical."""
    outs = []
    for capsules in (False, True):
        scene, ccd = pile_with_projectiles(scalar)
        cfg = dict(mixed_config(ccd), capsules=capsules)
        with api.Context(device=0, scalar=scalar) as ctx:
            w = plugins.DeviceGraphWorld(scene, plugins.PhysicsPlugins(ctx), ctx, substeps=4, ccd=cfg)
            res = []
            for _ in range(3):
                w.step()
                r = ctx.ccd_download()
                res.append({k: np.asarray(r[k]).copy() for k in ("min_toi", "hit_body", "hit_contact", "candidates", "hits")})
                res.append({k: getattr(w.bodies, k).copy() for k in ("position", "rotation", "linear_velocity", "angular_velocity")})
            outs.append(res)
    for a, b in zip(*outs):
        for k in a:
            assert np.array_equal(np.ascontiguousarray(a[k]).view(np.uint8), np.ascontiguousarray(b[k]).view(np.uint8)), k


def test_flag_lets_capsules_through_and_unknown_bits_are_refused():
    scene, ccd = capsule_pile_with_projectiles(np.float32, n=60, layers=2, projectiles=6)
    with api.Context(device=0) as ctx:
        w = plugins.DeviceGraphWorld(scene, plugins.PhysicsPlugins(ctx), ctx, substeps=4)
        w.step()
        with pytest.raises(api.AvianError) as e:
            ctx.ccd_configure(body=ccd, collider=ccd)
        assert e.value.status == api.ERR_UNSUPPORTED
        w.step()
        for flags in (0x2, 0x3):
            cfg, keep = api.ccd_config(ccd, ccd, flags=flags)
            with pytest.raises(api.AvianError) as e:
                ctx._check(ctx.lib.avn_ccd_configure(ctx.handle, api.C.byref(cfg)))
            assert e.value.status == api.ERR_INVALID_ARGUMENT
        ctx.ccd_configure(body=ccd, collider=ccd, capsules=True)
        w.step()
        assert ctx.ccd_download()["total_candidates"] > 0
        # clearing the configuration forgets the flag: configuring again without it is refused, and the world steps on
        ctx.ccd_configure(None)
        with pytest.raises(api.AvianError) as e:
            ctx.ccd_configure(body=ccd, collider=ccd)
        assert e.value.status == api.ERR_UNSUPPORTED
        w.step()
