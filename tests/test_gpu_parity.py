"""GPU parity tests proper: every test drives the CUDA path through the C ABI (avian_b200.api.Context) and compares
with the CPU oracle on the same seeded inputs.  Bars: bit-exact for the broad phase pair lists (integer/index work),
1e-5 relative for post-step body state and impulses (BASELINE.json north_star)."""
import os

import numpy as np
import pytest

from avian_b200 import api, plugins, scenes

import oracle_lib
from helpers import RTOL, advance_to_solver_input, assert_bodies_close, assert_manifolds_close, oracle_world, rel_err

pytestmark = pytest.mark.gpu


def _gpu_step(ctx, prm, b, m=None, j=None):
    ctx.solver_step(prm, b, m, j)


def _free_bodies(n=257, seed=7, scalar=np.float32):
    rng = np.random.default_rng(seed)
    s = np.dtype(scalar)
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    inv_i = np.zeros((n, 6))
    diag = rng.uniform(0.5, 4.0, size=(n, 3))
    iso = rng.random(n) < 0.5
    diag[iso] = diag[iso, :1]
    inv_i[:, 0], inv_i[:, 3], inv_i[:, 5] = diag[:, 0], diag[:, 1], diag[:, 2]
    off = ~iso & (rng.random(n) < 0.5)
    inv_i[off, 1] = 0.05; inv_i[off, 4] = -0.03
    kind = rng.choice([0, 0, 0, 1, 2], size=n).astype(np.uint8)
    b = api.Bodies(kind=kind, position=rng.normal(size=(n, 3)).astype(s) * 10, rotation=q.astype(s),
                   linear_velocity=rng.normal(size=(n, 3)).astype(s), angular_velocity=(rng.normal(size=(n, 3)) * 3).astype(s),
                   inverse_mass=rng.uniform(0.1, 2.0, size=n).astype(s), inverse_inertia_local=inv_i.astype(s),
                   center_of_mass=(rng.normal(size=(n, 3)) * 0.1).astype(s))
    b.locked_axes = rng.choice([0, 0, 0, 0x20, 0x12, 0x07, 0x3f], size=n).astype(np.uint8)
    b.linear_damping = rng.uniform(0, 1, size=n).astype(s)
    b.angular_damping = rng.uniform(0, 1, size=n).astype(s)
    b.gravity_scale = rng.uniform(-1, 2, size=n).astype(s)
    b.linear_acceleration = rng.normal(size=(n, 3)).astype(s)
    b.angular_acceleration = rng.normal(size=(n, 3)).astype(s)
    b.max_linear_speed = np.where(rng.random(n) < 0.3, 1.0, np.inf).astype(s)
    b.max_angular_speed = np.where(rng.random(n) < 0.3, 2.0, np.inf).astype(s)
    b.integration_flags = rng.choice([0, 0, 0, 1, 2, 3], size=n).astype(np.uint8)
    return b


def test_integrator_all_options(gpu_ctx):
    """I0-I3 + S1 + S6: damping, gravity scale, locked axes, accelerations, gyroscopic torque, speed clamps, kinematic and
    static bodies, custom-integration markers — no contacts."""
    b = _free_bodies()
    prm = api.default_step_params(dt=1.0 / 60.0, substeps=5)
    bo, bg = b.copy(), b.copy()
    for _ in range(3):
        oracle_lib.solver_step(prm, bo)
        _gpu_step(gpu_ctx, prm, bg)
    assert_bodies_close(bg, bo, rtol=2e-6, what="integrator: ")
    # static bodies must come back untouched
    st = b.kind == api.BODY_STATIC
    assert np.array_equal(bg.position[st], b.position[st]) and np.array_equal(bg.linear_velocity[st], b.linear_velocity[st])


def test_reference_integrator_test_on_gpu(gpu_ctx):
    """integrator/mod.rs:561-629 through the CUDA path."""
    s = np.float32
    b = api.Bodies(kind=np.array([0], dtype=np.uint8), position=np.zeros((1, 3), dtype=s), rotation=np.array([[0, 0, 0, 1]], dtype=s),
                   linear_velocity=np.zeros((1, 3), dtype=s), angular_velocity=np.array([[0, 0, 2.0]], dtype=s), inverse_mass=np.ones(1, dtype=s),
                   inverse_inertia_local=np.array([[6.0, 0, 0, 6.0, 0, 6.0]], dtype=s))
    prm = api.default_step_params(dt=0.1, substeps=1)
    for _ in range(100):
        _gpu_step(gpu_ctx, prm, b)
    assert abs(b.position[0, 1] + 490.5) < 10.0
    assert np.allclose(b.linear_velocity[0], [0, -98.1, 0], atol=1e-4)
    assert np.allclose(b.angular_velocity[0], [0, 0, 2.0], atol=1e-5)


@pytest.mark.parametrize("scene_fn,steps,substeps", [
    (lambda: scenes.cubes_example(3), 45, 1),          # BASELINE config 1: 27 cubes, 1 substep, falling then landing
    (lambda: scenes.cubes_example(4), 50, 6),          # the literal examples/cubes.rs scene
    (lambda: scenes.cube_stack(6, 6, 6, brick=True), 3, 8),
    (lambda: scenes.cube_stack(8, 4, 8, brick=False, restitution=0.4), 2, 4),
])
def test_contact_solver_single_step(gpu_ctx, scene_fn, steps, substeps):
    """S0-S7: one solver stage from the same snapshot (bodies + manifolds + warm-start impulses)."""
    _, (prm, b, m, j) = advance_to_solver_input(scene_fn(), steps=steps, substeps=substeps)
    assert m is not None and m.count > 0
    bo, mo, bg, mg = b.copy(), m.copy(), b.copy(), m.copy()
    oracle_lib.solver_step(prm, bo, mo)
    _gpu_step(gpu_ctx, prm, bg, mg)
    assert_bodies_close(bg, bo, what="contacts: ")
    assert_manifolds_close(mg, mo, what="contacts: ")


def test_contact_solver_trajectory(gpu_ctx):
    """60 full steps (warm-start impulses round-tripping through store_contact_impulses and the narrow-phase fixture):
    GPU world vs oracle world."""
    sc_o, sc_g = scenes.cubes_example(3), scenes.cubes_example(3)
    wo = oracle_world(sc_o, substeps=1)
    wg = plugins.World(sc_g, plugins.PhysicsPlugins(gpu_ctx), substeps=1)
    worst = 0.0
    for i in range(60):
        wo.step(); wg.step()
        worst = max(worst, rel_err(wg.bodies.position, wo.bodies.position), rel_err(wg.bodies.linear_velocity, wo.bodies.linear_velocity))
    assert wg.last_pairs.count == wo.last_pairs.count
    assert worst <= RTOL, f"trajectory diverged: {worst:.3e}"


def test_dominance_kinematic_and_overflow_colour(gpu_ctx):
    """relative dominance (contact/mod.rs:129-154), kinematic bodies, and the serial overflow colour 23."""
    w, (prm, b, m, j) = advance_to_solver_input(scenes.cube_stack(4, 3, 4, brick=True), steps=2, substeps=4)
    b.dominance = np.zeros(b.count, dtype=np.int8)
    b.dominance[5::7] = 3
    b.kind = b.kind.copy(); b.kind[9] = api.BODY_KINEMATIC; b.linear_velocity[9] = (0.2, 0.0, 0.0)
    # move the last third of colour 0 into the overflow colour (legal: overflow is solved serially, first)
    off = m.color_offsets.astype(np.int64)
    n0 = int(off[1] - off[0]); k = n0 // 3
    perm = np.concatenate([np.arange(0, n0 - k), np.arange(n0, m.count), np.arange(n0 - k, n0)])
    pts = [np.arange(m.point_offsets[i], m.point_offsets[i + 1]) for i in perm]
    counts = np.array([len(p) for p in pts]); pidx = np.concatenate(pts)
    m2 = api.Manifolds(color_offsets=m.color_offsets.copy(), body1=m.body1[perm].copy(), body2=m.body2[perm].copy(), normal=m.normal[perm].copy(),
                       friction=m.friction[perm].copy(), restitution=m.restitution[perm].copy(),
                       point_offsets=np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32), anchor1=m.anchor1[pidx].copy(),
                       anchor2=m.anchor2[pidx].copy(), penetration=m.penetration[pidx].copy(), normal_speed=m.normal_speed[pidx].copy(),
                       warm_start_normal_impulse=m.warm_start_normal_impulse[pidx].copy(), warm_start_tangent_impulse=m.warm_start_tangent_impulse[pidx].copy(),
                       normal_impulse=m.normal_impulse[pidx].copy())
    co = off.copy(); co[1:] -= k; co[api.COLOR_OVERFLOW + 1] = m.count
    m2.color_offsets = co.astype(np.uint32)
    bo, mo, bg, mg = b.copy(), m2.copy(), b.copy(), m2.copy()
    oracle_lib.solver_step(prm, bo, mo)
    _gpu_step(gpu_ctx, prm, bg, mg)
    assert_bodies_close(bg, bo, what="dominance: ")
    assert_manifolds_close(mg, mo, what="dominance: ")


def _run_in_mode(mode, prm, b, m, j=None, env=None):
    """a fresh context with AVN_LAUNCH_MODE=mode ('' = default: megakernel + wavefront scheduling) and extra environment switches"""
    env = dict(env or {})
    if mode:
        env["AVN_LAUNCH_MODE"] = mode
    os.environ.update(env)
    try:
        with api.Context(device=0) as ctx:
            bb, mm = b.copy(), m.copy()
            ctx.solver_step(prm, bb, mm, j)
            return bb, mm, ctx.timings()
    finally:
        for k in env:
            os.environ.pop(k, None)


@pytest.mark.parametrize("iters", [1, 2])
def test_launch_modes_agree(gpu_ctx, iters):
    """wavefront megakernel == barrier megakernel == one launch per phase: the same arithmetic in the same per-body
    order, so the results must be BIT-identical"""
    _, (prm, b, m, j) = advance_to_solver_input(scenes.cube_stack(7, 6, 7, brick=True), steps=2, substeps=4)
    prm.solver_iterations = iters
    bw, mw, tw = _run_in_mode("", prm, b, m)
    bb, mb, tb = _run_in_mode("barrier", prm, b, m)
    bp, mp, tp = _run_in_mode("phases", prm, b, m)
    bs, ms, ts = _run_in_mode("", prm, b, m)   # the wavefront schedule again: run-to-run deterministic
    assert tw["kernel_launches"] == 1 and tb["kernel_launches"] == 1, "megakernel paths are ONE launch per step"
    assert tw["launch_mode"] == ts["launch_mode"] == 2   # AVN_LAUNCH_MEGA_WAVE
    assert tp["kernel_launches"] > 10
    assert np.array_equal(mw.normal_impulse, ms.normal_impulse) and np.array_equal(mw.warm_start_tangent_impulse, ms.warm_start_tangent_impulse)
    for other, what in ((bb, "barrier"), (bp, "phases"), (bs, "wavefront rerun")):
        for name in ("position", "rotation", "linear_velocity", "angular_velocity"):
            assert np.array_equal(getattr(bw, name), getattr(other, name)), (what, name)
    assert np.array_equal(mw.warm_start_normal_impulse, mb.warm_start_normal_impulse)
    assert np.array_equal(mw.warm_start_tangent_impulse, mp.warm_start_tangent_impulse)
    assert np.array_equal(mw.normal_impulse, mp.normal_impulse)
    bo, mo = b.copy(), m.copy()
    oracle_lib.solver_step(prm, bo, mo)
    assert_bodies_close(bw, bo, what=f"iters={iters}: ")


def test_wavefront_equals_barrier_with_16_manifolds_on_one_body(gpu_ctx):
    """a wide plate resting on a 4 x 4 field of cubes carries 16 manifolds x 4 points: 16 events of the plate per pass, each one waiting for
    the previous.  The wavefront schedule is bit-identical to the barrier schedule."""
    cubes = np.array([[1.5 * ix, 0.49, 1.5 * iz] for ix in range(4) for iz in range(4)])
    pos = np.concatenate([[[2.25, -0.5, 2.25]], cubes, [[2.25, 1.22, 2.25]]])
    he = np.concatenate([[[20.0, 0.5, 20.0]], np.full((16, 3), 0.5), [[3.5, 0.25, 3.5]]])
    kind = np.concatenate([[api.BODY_STATIC], np.full(17, api.BODY_DYNAMIC)])
    rot = np.tile(np.array([0.0, 0.0, 0.0, 1.0]), (18, 1))
    sc = scenes._assemble("plate_on_cubes", pos, rot, kind, he, np.full(18, scenes.SHAPE_CUBOID), np.float32)
    _, (prm, b, m, j) = advance_to_solver_input(sc, steps=3, substeps=4)
    per_body = np.bincount(np.concatenate([m.body1[m.body1 >= 0], m.body2[m.body2 >= 0]]), minlength=b.count)
    assert per_body.max() >= 16 and m.color_offsets[api.COLOR_OVERFLOW + 1] == m.color_offsets[api.COLOR_OVERFLOW], (per_body.max(), m.color_offsets)
    bw, mw, tw = _run_in_mode("wave", prm, b, m)
    bb, mb, _ = _run_in_mode("barrier", prm, b, m)
    assert tw["launch_mode"] == 2   # AVN_LAUNCH_MEGA_WAVE
    for name in ("position", "rotation", "linear_velocity", "angular_velocity"):
        assert np.array_equal(getattr(bw, name), getattr(bb, name)), name
    assert np.array_equal(mw.warm_start_normal_impulse, mb.warm_start_normal_impulse)
    assert np.array_equal(mw.warm_start_tangent_impulse, mb.warm_start_tangent_impulse)


def test_prefetched_body_columns(gpu_ctx):
    """avn_solver_prefetch_bodies: the columns copied ahead on the copy stream give the same step; AVN_BODIES_STATIC_UNCHANGED keeps the mass
    properties of the previous upload; a prefetch of OTHER columns than the upload's is ignored (the upload copies again)"""
    _, (prm, b, m, j) = advance_to_solver_input(scenes.cube_stack(5, 4, 5, brick=True), steps=2, substeps=4)
    ref_b, ref_m = b.copy(), m.copy()
    gpu_ctx.solver_step(prm, ref_b, ref_m)
    with api.Context(device=0) as ctx:
        b1, m1 = b.copy(), m.copy()
        ctx.solver_prefetch_bodies(b1)
        ctx.solver_step(prm, b1, m1)
        assert np.array_equal(b1.position, ref_b.position) and np.array_equal(b1.angular_velocity, ref_b.angular_velocity)
        b2, m2 = b.copy(), m.copy()
        ctx.solver_prefetch_bodies(b2, static_unchanged=True)       # same scene: the static columns of the previous upload stand
        ctx.solver_step(prm, b2, m2)
        assert np.array_equal(b2.position, ref_b.position) and np.array_equal(b2.linear_velocity, ref_b.linear_velocity)
        other, b3, m3 = b.copy(), b.copy(), m.copy()
        other.linear_velocity[:] = 7.0
        ctx.solver_prefetch_bodies(other)                            # not the columns the upload is given
        ctx.solver_step(prm, b3, m3)
        assert np.array_equal(b3.position, ref_b.position) and np.array_equal(m3.normal_impulse, ref_m.normal_impulse)


def test_wavefront_equals_barrier_at_headline_size(gpu_ctx):
    """BASELINE-size property: on the 100k-cube stack (no oracle at this size in seconds) the wavefront schedule and the
    barrier schedule give bit-identical bodies and impulses, and the step stays finite with non-negative normal impulses
    inside the friction cone."""
    sc = scenes.cube_stack(51, 40, 50, brick=True)
    w = plugins.World(sc, plugins.PhysicsPlugins(gpu_ctx), substeps=8)
    w.step()
    w.broad_phase(); m = w.narrow_phase()
    prm, b = w.params, w.bodies
    assert m.count > 300_000
    bw, mw, _ = _run_in_mode("", prm, b, m)
    bb, mb, _ = _run_in_mode("barrier", prm, b, m)
    for name in ("position", "rotation", "linear_velocity", "angular_velocity"):
        assert np.isfinite(getattr(bw, name)).all()
        assert np.array_equal(getattr(bw, name), getattr(bb, name)), name
    assert np.array_equal(mw.normal_impulse, mb.normal_impulse)
    lam_n = mw.warm_start_normal_impulse
    lam_t = np.linalg.norm(mw.warm_start_tangent_impulse, axis=1)
    mu = np.repeat(mw.friction, np.diff(mw.point_offsets))
    assert (lam_n >= 0).all() and (lam_t <= mu * lam_n * (1 + 1e-5) + 1e-7).all()


def test_upload_run_download_split_is_repeatable(gpu_ctx):
    _, (prm, b, m, j) = advance_to_solver_input(scenes.cube_stack(4, 4, 4, brick=True), steps=1, substeps=4)
    b1, m1 = b.copy(), m.copy()
    gpu_ctx.solver_step(prm, b1, m1)
    b2, m2 = b.copy(), m.copy()
    gpu_ctx.solver_upload(prm, b2, m2)
    gpu_ctx.solver_run(); gpu_ctx.solver_run()      # every run restarts from the uploaded snapshot
    gpu_ctx.solver_download()
    assert np.array_equal(b1.position, b2.position) and np.array_equal(m1.normal_impulse, m2.normal_impulse)


# ---- joints ---------------------------------------------------------------------------------------------------------
def test_spherical_chain(gpu_ctx):
    """X0-X4 on chain_3d: 40 links = 40 dependency levels, kinematic anchor, compliance."""
    sc = scenes.spherical_chain(40)
    prm = api.default_step_params(substeps=12)
    bo, bg, jo, jg = sc.bodies.copy(), sc.bodies.copy(), sc.joints.copy(), sc.joints.copy()
    bo.linear_velocity[5] = bg.linear_velocity[5] = (0.5, 0.0, 0.2)
    for _ in range(5):
        oracle_lib.solver_step(prm, bo, None, jo)
        _gpu_step(gpu_ctx, prm, bg, None, jg)
    assert_bodies_close(bg, bo, what="chain: ")
    assert rel_err(jg.types[api.JOINT_SPHERICAL].force, jo.types[api.JOINT_SPHERICAL].force) <= 1e-4
    assert gpu_ctx.timings()["joint_levels"] == 40


def _all_joint_types_scene(scalar=np.float32, n=30, seed=3):
    rng = np.random.default_rng(seed)
    s = np.dtype(scalar)
    nb = 2 * n * 5 + 1
    q = rng.normal(size=(nb, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    kind = np.zeros(nb, dtype=np.uint8); kind[0] = api.BODY_STATIC; kind[3::17] = api.BODY_KINEMATIC
    b = api.Bodies(kind=kind, position=(rng.normal(size=(nb, 3)) * 2).astype(s), rotation=q.astype(s),
                   linear_velocity=(rng.normal(size=(nb, 3)) * 0.5).astype(s), angular_velocity=rng.normal(size=(nb, 3)).astype(s),
                   inverse_mass=rng.uniform(0.5, 2, size=nb).astype(s), inverse_inertia_local=np.zeros((nb, 6), dtype=s),
                   center_of_mass=(rng.normal(size=(nb, 3)) * 0.05).astype(s))
    b.inverse_inertia_local[:, 0] = rng.uniform(1, 3, nb); b.inverse_inertia_local[:, 3] = rng.uniform(1, 3, nb); b.inverse_inertia_local[:, 5] = rng.uniform(1, 3, nb)
    b.dominance = np.zeros(nb, dtype=np.int8); b.dominance[7::11] = 2
    js = api.JointSet()
    for t in range(api.JOINT_TYPE_COUNT):
        b1 = rng.integers(0, nb, size=n).astype(np.int32)
        b2 = ((b1 + rng.integers(1, nb - 1, size=n)) % nb).astype(np.int32)
        lb = rng.normal(size=(2, n, 4)); lb /= np.linalg.norm(lb, axis=2, keepdims=True)
        ax = rng.normal(size=(n, 3)); ax /= np.linalg.norm(ax, axis=1, keepdims=True)
        j = api.Joints(body1=b1, body2=b2, local_anchor1=(rng.normal(size=(n, 3)) * 0.3).astype(s), local_anchor2=(rng.normal(size=(n, 3)) * 0.3).astype(s),
                       local_basis1=lb[0].astype(s), local_basis2=lb[1].astype(s), axis=ax.astype(s),
                       limit_enabled=rng.integers(0, 4, size=n).astype(np.uint8), limit_min=rng.uniform(-1.0, -0.1, n).astype(s),
                       limit_max=rng.uniform(0.1, 1.0, n).astype(s), limit2_min=rng.uniform(-0.5, -0.1, n).astype(s), limit2_max=rng.uniform(0.1, 0.5, n).astype(s),
                       compliance0=rng.choice([0, 1e-4], n).astype(s), compliance1=rng.choice([0, 1e-3], n).astype(s), compliance2=rng.choice([0, 1e-3], n).astype(s),
                       damping_enabled=(rng.random(n) < 0.3).astype(np.uint8), damping_linear=rng.uniform(0, 2, n).astype(s), damping_angular=rng.uniform(0, 2, n).astype(s),
                       force=np.zeros((n, 3), dtype=s), torque=np.zeros((n, 3), dtype=s))
        if t == api.JOINT_DISTANCE:
            j.limit_min = rng.uniform(0.2, 0.8, n).astype(s); j.limit_max = (j.limit_min + rng.uniform(0, 0.5, n)).astype(s)
        js.types[t] = j
    return b, js


def test_all_joint_types_random_graph(gpu_ctx):
    """every joint type, limits, compliance, damping, dominance, static and kinematic ends, random connectivity:
    exercises the order-preserving level schedule against the serial oracle."""
    b, js = _all_joint_types_scene()
    prm = api.default_step_params(substeps=4)
    bo, bg, jo, jg = b.copy(), b.copy(), js.copy(), js.copy()
    oracle_lib.solver_step(prm, bo, None, jo)
    _gpu_step(gpu_ctx, prm, bg, None, jg)
    assert_bodies_close(bg, bo, rtol=2e-5, what="joints: ")
    for t in range(api.JOINT_TYPE_COUNT):
        assert rel_err(jg.types[t].force, jo.types[t].force) <= 1e-4, t
        assert rel_err(jg.types[t].torque, jo.types[t].torque) <= 1e-4, t


def test_ragdolls_with_contacts(gpu_ctx):
    """BASELINE config 4 in miniature: 9 ragdolls falling on the ground, contacts + revolute + spherical joints."""
    _, (prm, b, m, j) = advance_to_solver_input(scenes.ragdoll_field(9, pitch=3.0, drop_height=0.1), steps=25, substeps=8)
    assert m is not None and m.count > 0 and j.count == 9 * 16
    bo, mo, jo, bg, mg, jg = b.copy(), m.copy(), j.copy(), b.copy(), m.copy(), j.copy()
    oracle_lib.solver_step(prm, bo, mo, jo)
    _gpu_step(gpu_ctx, prm, bg, mg, jg)
    assert_bodies_close(bg, bo, what="ragdolls: ")
    assert_manifolds_close(mg, mo, what="ragdolls: ")


@pytest.mark.parametrize("scalar", [np.float64])
def test_f64_contacts_and_joints(scalar):
    with api.Context(device=0, scalar=scalar) as ctx:
        _, (prm, b, m, j) = advance_to_solver_input(scenes.cube_stack(4, 4, 4, brick=True, scalar=scalar), steps=2, substeps=4)
        bo, mo, bg, mg = b.copy(), m.copy(), b.copy(), m.copy()
        oracle_lib.solver_step(prm, bo, mo)
        ctx.solver_step(prm, bg, mg)
        assert_bodies_close(bg, bo, rtol=1e-9, what="f64 contacts: ")
        bj, js = _all_joint_types_scene(scalar=scalar)
        bo, bg, jo, jg = bj.copy(), bj.copy(), js.copy(), js.copy()
        oracle_lib.solver_step(prm, bo, None, jo)
        ctx.solver_step(prm, bg, None, jg)
        assert_bodies_close(bg, bo, rtol=1e-9, what="f64 joints: ")


@pytest.mark.parametrize("scalar,rtol", [(np.float32, RTOL), (np.float64, 1e-9)])
def test_sphere_only_scene_single_point_kernels(scalar, rtol, monkeypatch):
    """BASELINE config 5 in miniature: every manifold has one point, which selects the MAXP = 1 build of the step kernel and the
    quarter-size staging tile; wavefront, barrier and per-phase launches must agree bit for bit, and with the oracle to rtol."""
    sc = scenes.falling_spheres(3000, seed=7, box=(14.0, 6.0, 14.0), scalar=scalar)
    _, (prm, b, m, j) = advance_to_solver_input(sc, steps=2, substeps=4)
    assert m.count > 1000 and m.penetration.shape[0] == m.count
    bo, mo = b.copy(), m.copy()
    oracle_lib.solver_step(prm, bo, mo)
    results = []
    for mode in (None, "barrier", "phases"):
        if mode:
            monkeypatch.setenv("AVN_LAUNCH_MODE", mode)
        with api.Context(device=0, scalar=scalar) as ctx:
            bg, mg = b.copy(), m.copy()
            ctx.solver_step(prm, bg, mg)
        assert_bodies_close(bg, bo, rtol=rtol, what=f"spheres {mode}: ")
        assert_manifolds_close(mg, mo, rtol=rtol, what=f"spheres {mode}: ")
        results.append((bg, mg))
    for bg, mg in results[1:]:
        assert np.array_equal(bg.position, results[0][0].position) and np.array_equal(bg.linear_velocity, results[0][0].linear_velocity)
        assert np.array_equal(mg.warm_start_normal_impulse, results[0][1].warm_start_normal_impulse)


def test_manifold_csr_is_validated(gpu_ctx):
    """More than 4 points in a manifold, or decreasing offsets, is an INVALID_ARGUMENT error, not undefined behaviour."""
    _, (prm, b, m, j) = advance_to_solver_input(scenes.cubes_example(3), steps=45, substeps=1)
    assert m.penetration.shape[0] > 4 and m.count > 2
    wide = m.copy()
    po = wide.point_offsets.copy()
    po[1:-1] = po[-1]        # manifold 0 owns every point
    wide.point_offsets = po
    with pytest.raises(api.AvianError):
        gpu_ctx.solver_step(prm, b.copy(), wide)
    decreasing = m.copy()
    po = decreasing.point_offsets.copy()
    po[1] = po[2] + 1
    decreasing.point_offsets = po
    with pytest.raises(api.AvianError):
        gpu_ctx.solver_step(prm, b.copy(), decreasing)
    gpu_ctx.solver_step(prm, b.copy(), m.copy())   # the context stays usable after a rejected upload


def test_cubes_simulation_is_locally_deterministic_on_gpu(gpu_ctx):
    """src/tests/mod.rs:149-183 on the device: the 4x4x4 cubes scene stepped twice through the GPU plugins gives identical transforms
    (the wavefront schedule orders every body's events, so the result does not depend on warp timing)."""
    def run():
        w = plugins.World(scenes.cubes_example(4), plugins.PhysicsPlugins(gpu_ctx), substeps=6)
        for _ in range(90):
            w.step()
        return w.bodies.position.copy(), w.bodies.rotation.copy(), w.bodies.linear_velocity.copy()
    a, b = run(), run()
    assert a[0][1:, 1].min() > -1.0                       # nothing fell through the ground
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_invalid_inputs_are_refused_not_gathered_through(gpu_ctx):
    """ADVICE r1: a manifold body index outside [-1, B) must be an error at upload, not an out-of-bounds gather on the device."""
    _, (prm, b, m, j) = advance_to_solver_input(scenes.cube_stack(4, 3, 4, brick=True), steps=2, substeps=4)
    for bad in (b.count, b.count + 7, -2):
        mb = m.copy()
        mb.body2 = mb.body2.copy()
        mb.body2[3] = bad
        with pytest.raises(api.AvianError) as e:
            gpu_ctx.solver_step(prm, b.copy(), mb)
        assert e.value.status == api.ERR_INVALID_ARGUMENT
    # the context stays usable
    bg, mg, bo, mo = b.copy(), m.copy(), b.copy(), m.copy()
    gpu_ctx.solver_step(prm, bg, mg)
    oracle_lib.solver_step(prm, bo, mo)
    assert_bodies_close(bg, bo)


def test_bad_colouring_is_reported_not_spun_on(gpu_ctx, monkeypatch):
    """ADVICE r1: the wavefront schedule trusts the colouring only as far as it checks it.  Two constraints of one body in ONE colour would give
    wrong event numbers and a spin until the watchdog; the rank pass detects it, the step falls back to barriers and the download reports it."""
    monkeypatch.setenv("AVN_LAUNCH_MODE", "wave")
    _, (prm, b, m, j) = advance_to_solver_input(scenes.cube_stack(5, 4, 5, brick=True), steps=2, substeps=4)
    with api.Context(device=0) as ctx:
        ok_b, ok_m = b.copy(), m.copy()
        ctx.solver_step(prm, ok_b, ok_m)
        assert ctx.timings()["launch_mode"] == 2          # AVN_LAUNCH_MEGA_WAVE
        bad = m.copy()
        co = bad.color_offsets.copy()
        c0 = next(c for c in range(23) if co[c + 1] - co[c] > 0)
        c1 = next(c for c in range(c0 + 1, 23) if co[c + 1] - co[c] > 0)
        co[c0 + 1:c1 + 1] = co[c1 + 1]                    # merge colour c1 (and the empty ones between) into c0: bodies now repeat inside a colour
        bad.color_offsets = co
        with pytest.raises(api.AvianError) as e:
            ctx.solver_step(prm, b.copy(), bad)
        assert e.value.status == api.ERR_INVALID_ARGUMENT and "colour" in str(e.value)
        again_b, again_m = b.copy(), m.copy()
        ctx.solver_step(prm, again_b, again_m)             # and the context is fine afterwards
        assert np.array_equal(again_b.position, ok_b.position)
