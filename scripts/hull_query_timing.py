#!/usr/bin/env python
"""Convex hulls in the spatial queries and move and slide (GPU box), in one job, the measurements alternated round by round:
  * 1 000 000 closest-hit rays (a downward grid + random directions from inside the scene), 1 000 000 closest sphere casts (radius 0.4) and
    250 000 closest hull casts (hulls of the scene's table) straight down, and 1 000 000 project_point calls, against
    scenes.hull_pile(100_000) and scenes.decomposed_pile(`--decomposed`) (landed by `--pile-steps` device-resident steps) and against the
    100k-cube stack (scenes.cube_stack(51, 40, 50) as built, with the same hull table attached, so its kernels are the cuboid / sphere ones);
  * 100 000 capsule characters walking on each scene (avn_move_and_slide, default config): hull obstacles on the piles.
Every query time is one C-ABI call from host columns to host results (upload, kernels, download): CUDA events on the library's stream and the
host clock, both closed by the call's own stream synchronise; move and slide also reports the kernel's own events (kernel_ms).  Prints the
card and its power limit (nvidia-smi, read-only) and writes OUT_DIR/hull_query_timing.json.
   usage: python scripts/hull_query_timing.py OUT_DIR [--repeats R] [--pile-steps S] [--decomposed N]"""
import argparse
import json
import math
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from avian_b200 import api, plugins, scenes  # noqa: E402

SPH, CAP, HULL = 1, 2, 3
IDENT = [0.0, 0.0, 0.0, 1.0]


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    name, limit = [x.strip() for x in out.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def once(ctx, fn) -> tuple:
    import torch
    stream = torch.cuda.ExternalStream(ctx.stream())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0.record(stream)
    r = fn()
    e1.record(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), (time.perf_counter() - t0) * 1e3, (float(r["kernel_ms"]) if isinstance(r, dict) and "kernel_ms" in r else None)


def landed(scene, steps: int):
    with api.Context(device=0) as ctx:
        w = plugins.DeviceGraphWorld(scene, plugins.PhysicsPlugins(ctx), ctx, substeps=4)
        for _ in range(steps):
            w.step()
        return plugins.SpatialQueryPlugin.colliders(w)


def stack() -> api.QueryColliders:
    sc = scenes.cube_stack(51, 40, 50, brick=True)
    return api.QueryColliders(shape=sc.shape_type.astype(np.uint8), dims=sc.dims, position=np.asarray(sc.bodies.position, np.float64),
                              rotation=np.asarray(sc.bodies.rotation, np.float64))


def footprint(cols):
    body = cols.position[~((cols.shape != HULL) & (cols.dims.max(axis=1) >= 10))]   # leave out the ground
    return body.min(axis=0), body.max(axis=0)


def rays_over(cols, n, rng):
    lo, hi = footprint(cols)
    g = int(math.isqrt(n // 2))
    gx, gz = np.meshgrid(np.linspace(lo[0], hi[0], g), np.linspace(lo[2], hi[2], g), indexing="ij")
    k = gx.size
    d_in = rng.normal(size=(n - k, 3))
    d_in /= np.linalg.norm(d_in, axis=1, keepdims=True)
    o = np.concatenate([np.stack([gx.ravel(), np.full(k, hi[1] + 5.0), gz.ravel()], 1), rng.uniform(lo, hi, (n - k, 3))])
    d = np.concatenate([np.tile([0.0, -1.0, 0.0], (k, 1)), d_in])
    return api.Rays(origin=o, direction=d, max_distance=np.full(n, float(hi[1] - lo[1] + 20.0)))


def casts_over(cols, n, shape, n_hulls, rng):
    lo, hi = footprint(cols)
    o = np.stack([rng.uniform(lo[0], hi[0], n), np.full(n, hi[1] + 3.0), rng.uniform(lo[2], hi[2], n)], 1)
    dims = np.tile([0.4, 0.0, 0.0], (n, 1))
    rot = np.tile(IDENT, (n, 1))
    if shape == HULL:
        dims[:, 0] = rng.integers(0, n_hulls, n)
        q = rng.normal(size=(n, 4))
        rot = q / np.linalg.norm(q, axis=1, keepdims=True)
    return api.ShapeQueries(shape=np.full(n, shape, np.uint8), dims=dims, position=o, rotation=rot, direction=np.tile([0.0, -1.0, 0.0], (n, 1)),
                            max_distance=np.full(n, float(hi[1] - lo[1] + 20.0)))


def points_in(cols, n, rng):
    lo, hi = footprint(cols)
    return api.Points(point=rng.uniform(lo, hi, (n, 3)), solid=rng.random(n) < 0.5)


def walkers(cols, n, rng):
    lo, hi = footprint(cols)
    pos = np.stack([rng.uniform(lo[0], hi[0], n), hi[1] + 1.4 + rng.uniform(-0.05, 0.05, n), rng.uniform(lo[2], hi[2], n)], 1)
    a = rng.uniform(0, 2 * math.pi, n)
    vel = np.stack([np.cos(a) * 6, rng.uniform(-60, -20, n), np.sin(a) * 6], 1)
    return api.MoveBatch(shape=np.full(n, CAP, np.uint8), dims=np.tile([0.4, 0.5, 0.0], (n, 1)), position=pos, rotation=np.tile(IDENT, (n, 1)),
                         velocity=vel)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--pile-steps", type=int, default=100)
    ap.add_argument("--decomposed", type=int, default=30_000)
    args = ap.parse_args()
    out_dir = Path(args.out_dir)
    out_dir.mkdir(parents=True, exist_ok=True)
    res = {"card": card(), "pile_steps": args.pile_steps}
    print(res["card"], flush=True)
    rng = np.random.default_rng(1)
    hp, dp = scenes.hull_pile(100_000), scenes.decomposed_pile(args.decomposed)
    worlds = {"hull_pile100k": (landed(hp, args.pile_steps), hp.hulls), f"decomposed_pile{args.decomposed // 1000}k": (landed(dp, args.pile_steps), dp.hulls),
              "stack100k_cubes": (stack(), hp.hulls)}
    with api.Context(device=0) as ctx:
        jobs = []
        for name, (cols, hulls) in worlds.items():
            res[f"{name}/colliders"] = int(cols.shape.shape[0])
            res[f"{name}/hulls"] = int((cols.shape == HULL).sum())
            n_hulls = int(hulls.count)
            batches = {"cast_ray_1M": ("cast_ray", rays_over(cols, 1_000_000, rng)), "sphere_cast_1M": ("cast_shape", casts_over(cols, 1_000_000, SPH, n_hulls, rng)),
                       "hull_cast_250k": ("cast_shape", casts_over(cols, 250_000, HULL, n_hulls, rng)),
                       "project_point_1M": ("project_point", points_in(cols, 1_000_000, rng)), "move_100k_capsule": ("move", walkers(cols, 100_000, rng))}
            for label, (kind, b) in batches.items():
                jobs.append((name, cols, hulls, label, kind, b))
        cfg = api.MoveConfig()
        run = lambda kind, b: ctx.move_and_slide(cfg, b) if kind == "move" else getattr(ctx, kind)(b)
        times = {}
        for rnd in range(args.repeats + 1):                   # round 0 warms up; the scenes and queries alternate within every round
            for name, cols, hulls, label, kind, b in jobs:
                ctx.set_convex_hulls(hulls)
                ctx.query_update(cols)
                t = once(ctx, lambda: run(kind, b))
                if rnd:
                    times.setdefault(f"{name}/{label}", []).append(t)
        s = lambda v: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
        for key, v in times.items():
            ev, wall, k = zip(*v)
            res[key] = {"event_ms": s(ev), "wall_ms": s(wall), "repeats": len(v)}
            if k[0] is not None:
                res[key]["kernel_ms"] = s(k)
            print(key, res[key]["event_ms"], flush=True)
    (out_dir / "hull_query_timing.json").write_text(json.dumps(res, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
