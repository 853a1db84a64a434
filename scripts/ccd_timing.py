#!/usr/bin/env python
"""Swept CCD at the headline size (GPU box): the 100k-cube stack (46 x 47 x 46 aligned columns on a ground slab) stepped by DeviceGraphWorld,
the device-resident pipeline.  Arms, each warmed up and repeated:
  * no CCD configured: the single-launch solver stage;
  * CCD configured on one body far from everything: the split launch (prepare + substeps -> CCD pass -> restitution + finalize) with no
    candidate — what configuring CCD costs by itself;
  * 1 000, 10 000 and 100 000 fast projectiles fired at the stack (half spheres, half cubes; half Linear, half NonLinear), each also
    stepped without CCD.
Reported per arm: the solver stage's device time (AvnTimings::total_ms), the CCD pass's device time (AvnCcdResult::pass_ms), the whole
resident step's wall time (host clock around DeviceGraphWorld.step, which ends in the download's synchronise), candidates and hits.  Prints
the card and its power limit (nvidia-smi, read-only) and writes OUT_DIR/ccd_timing.json.   usage: python scripts/ccd_timing.py OUT_DIR [--steps K]"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from avian_b200 import api, plugins, scenes  # noqa: E402
from avian_b200.fixture import SHAPE_CUBOID, SHAPE_SPHERE  # noqa: E402


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    name, limit = [x.strip() for x in out.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def stack_with_projectiles(projectiles: int, far_body: bool = False, seed: int = 0):
    """The stack plus `projectiles` bodies flying at it at 200-400 m/s from just outside its bounding sphere (plus, with far_body, one body
    1 km away)."""
    base = scenes.cube_stack(46, 47, 46, brick=False)
    b = base.bodies
    rng = np.random.default_rng(seed)
    centre = np.array([46 * 0.525, 47 * 0.5, 46 * 0.525])
    extra = projectiles + (1 if far_body else 0)
    d = rng.normal(size=(projectiles, 3))
    d[:, 1] = np.abs(d[:, 1])
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    ppos = centre + d * rng.uniform(45.0, 50.0, (projectiles, 1))   # just outside the stack's bounding sphere
    pvel = -d * rng.uniform(200.0, 400.0, (projectiles, 1))
    if far_body:
        ppos, pvel = np.concatenate([ppos, [[1000.0, 1000.0, 1000.0]]]), np.concatenate([pvel, [[0, 0, 0]]])
    shape = np.where(np.arange(extra) % 2 == 0, SHAPE_SPHERE, SHAPE_CUBOID)
    dims = np.where(shape[:, None] == SHAPE_SPHERE, np.array([[0.15, 0, 0]]), np.array([[0.15, 0.15, 0.15]]))
    scene = scenes._assemble("ccd_stack", np.concatenate([b.position.astype(np.float64), ppos]),
                             np.concatenate([b.rotation.astype(np.float64), np.tile([0, 0, 0, 1.0], (extra, 1))]),
                             np.concatenate([b.kind, np.zeros(extra, np.uint8)]), np.concatenate([base.dims, dims]),
                             np.concatenate([base.shape_type, shape]), np.float32,
                             linvel=np.concatenate([b.linear_velocity.astype(np.float64), pvel]))
    return scene, np.arange(b.count, b.count + extra)


def run_arm(scene, ccd: dict | None, steps: int, warmup: int) -> dict:
    with api.Context(device=0) as ctx:
        w = plugins.DeviceGraphWorld(scene, plugins.PhysicsPlugins(ctx), ctx, substeps=8, ccd=ccd)
        solver, wall, passes, cand, hits = [], [], [], 0, 0
        for i in range(warmup + steps):
            t0 = time.perf_counter()
            w.step()
            t1 = time.perf_counter()
            if i < warmup:
                continue
            wall.append((t1 - t0) * 1e3)
            solver.append(ctx.timings()["total_ms"])
            if ccd is not None:
                r = ctx.ccd_download()
                passes.append(r["pass_ms"])
                cand += r["total_candidates"]
                hits += int((r["hit_body"] >= 0).sum())
        med = lambda x: float(np.median(x)) if x else None
        return {"solver_stage_ms": med(solver), "ccd_pass_ms": med(passes), "step_wall_ms": med(wall), "candidates_per_step": cand / steps,
                "hits_per_step": hits / steps, "bodies": int(scene.bodies.count)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    out = {"card": card(), "arms": {}}
    print(out["card"], flush=True)
    scene, ccd = stack_with_projectiles(0, far_body=True)
    out["arms"]["stack, no CCD"] = run_arm(scene, None, a.steps, a.warmup)
    scene, ccd = stack_with_projectiles(0, far_body=True)
    out["arms"]["stack, CCD on one far body"] = run_arm(scene, dict(body=ccd, collider=ccd), a.steps, a.warmup)
    for n in (1000, 10000, 100000):
        mode = np.arange(n) % 4 >= 2          # with the alternating shapes: every shape in both modes
        scene, ccd = stack_with_projectiles(n)
        out["arms"][f"{n} projectiles, no CCD"] = run_arm(scene, None, a.steps, a.warmup)
        scene, ccd = stack_with_projectiles(n)
        out["arms"][f"{n} projectiles, CCD"] = run_arm(scene, dict(body=ccd, collider=ccd, mode=mode.astype(np.uint8)), a.steps, a.warmup)
        print(n, out["arms"][f"{n} projectiles, no CCD"], out["arms"][f"{n} projectiles, CCD"], flush=True)
    Path(a.out_dir).mkdir(parents=True, exist_ok=True)
    (Path(a.out_dir) / "ccd_timing.json").write_text(json.dumps(out, indent=1))
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
