#!/usr/bin/env python
"""Capsules in the spatial queries and move and slide (GPU box), each set against the cuboid / sphere case in the same run:
  * 1 000 000 closest-hit rays (a downward grid + random directions from inside the scene) against the 100k capsule pile
    (scenes.capsule_pile(100_000), landed by `--pile-steps` device-resident steps) and against the 100k-cube stack
    (scenes.cube_stack(51, 40, 50) as built);
  * 1 000 000 closest capsule casts straight down (radius 0.4, half length 0.5: the reference's character capsule) onto both scenes;
  * 100 000 capsule characters walking on the stack (avn_move_and_slide, default config) against 100 000 sphere characters of radius 0.4.
Every query time is one C-ABI call from host columns to host results (upload, kernels, download): CUDA events on the library's stream and the
host clock, both closed by the call's own stream synchronise; move and slide also reports the kernel's own events (kernel_ms).  Prints the
card and its power limit (nvidia-smi, read-only) and writes OUT_DIR/capsule_query_timing.json.
   usage: python scripts/capsule_query_timing.py OUT_DIR [--repeats R] [--pile-steps S]"""
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

CAP, SPH = 2, 1
IDENT = [0.0, 0.0, 0.0, 1.0]


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    name, limit = [x.strip() for x in out.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def timed(ctx, fn, warmup: int, repeats: int) -> dict:
    import torch
    stream = torch.cuda.ExternalStream(ctx.stream())
    for _ in range(warmup):
        fn()
    ev_ms, wall_ms, extra = [], [], []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e0.record(stream)
        r = fn()
        e1.record(stream)
        torch.cuda.synchronize()
        wall_ms.append((time.perf_counter() - t0) * 1e3)
        ev_ms.append(e0.elapsed_time(e1))
        if isinstance(r, dict) and "kernel_ms" in r:
            extra.append(float(r["kernel_ms"]))
    s = lambda v: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
    out = {"event_ms": s(ev_ms), "wall_ms": s(wall_ms), "repeats": repeats}
    if extra:
        out["kernel_ms"] = s(extra)
    return out


def landed_pile(steps: int) -> api.QueryColliders:
    with api.Context(device=0) as ctx:
        w = plugins.DeviceGraphWorld(scenes.capsule_pile(100_000), plugins.PhysicsPlugins(ctx), ctx, substeps=4)
        for _ in range(steps):
            w.step()
        return plugins.SpatialQueryPlugin.colliders(w)


def stack() -> api.QueryColliders:
    sc = scenes.cube_stack(51, 40, 50, brick=True)
    return api.QueryColliders(shape=sc.shape_type.astype(np.uint8), dims=sc.dims, position=np.asarray(sc.bodies.position, np.float64),
                              rotation=np.asarray(sc.bodies.rotation, np.float64))


def footprint(cols):
    body = cols.position[cols.dims.max(axis=1) < 10]                  # leave out the ground
    return body.min(axis=0), body.max(axis=0)


def rays_over(cols, n, rng):
    lo, hi = footprint(cols)
    half = n // 2
    g = int(math.isqrt(half))
    gx, gz = np.meshgrid(np.linspace(lo[0], hi[0], g), np.linspace(lo[2], hi[2], g), indexing="ij")
    k = gx.size
    o_down = np.stack([gx.ravel(), np.full(k, hi[1] + 5.0), gz.ravel()], 1)
    o_in = rng.uniform(lo, hi, (n - k, 3))
    d_in = rng.normal(size=(n - k, 3))
    d_in /= np.linalg.norm(d_in, axis=1, keepdims=True)
    o = np.concatenate([o_down, o_in])
    d = np.concatenate([np.tile([0.0, -1.0, 0.0], (k, 1)), d_in])
    return api.Rays(origin=o, direction=d, max_distance=np.full(n, float(hi[1] - lo[1] + 20.0)))


def casts_over(cols, n, rng):
    lo, hi = footprint(cols)
    o = np.stack([rng.uniform(lo[0], hi[0], n), np.full(n, hi[1] + 3.0), rng.uniform(lo[2], hi[2], n)], 1)
    return api.ShapeQueries(shape=np.full(n, CAP, np.uint8), dims=np.tile([0.4, 0.5, 0.0], (n, 1)), position=o, rotation=np.tile(IDENT, (n, 1)),
                            direction=np.tile([0.0, -1.0, 0.0], (n, 1)), max_distance=np.full(n, float(hi[1] - lo[1] + 20.0)))


def walkers(cols, n, shape, rng):
    lo, hi = footprint(cols)
    top = float(cols.position[cols.dims.max(axis=1) < 10][:, 1].max()) + 0.5
    half_h = 0.9 if shape == CAP else 0.4
    pos = np.stack([rng.uniform(lo[0], hi[0], n), top + half_h + rng.uniform(-0.05, 0.05, n), rng.uniform(lo[2], hi[2], n)], 1)
    a = rng.uniform(0, 2 * math.pi, n)
    vel = np.stack([np.cos(a) * 6, rng.uniform(-10, 0, n), np.sin(a) * 6], 1)
    return api.MoveBatch(shape=np.full(n, shape, np.uint8), dims=np.tile([0.4, 0.5, 0.0], (n, 1)), position=pos, rotation=np.tile(IDENT, (n, 1)),
                         velocity=vel, planes=[np.array([[0.0, 1.0, 0.0]]) if i % 2 else None for i in range(n)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--pile-steps", type=int, default=200)
    args = ap.parse_args()
    out_dir = Path(args.out_dir)
    out_dir.mkdir(parents=True, exist_ok=True)
    res = {"card": card(), "pile_steps": args.pile_steps}
    print(res["card"], flush=True)
    rng = np.random.default_rng(1)
    worlds = {"capsule_pile100k": landed_pile(args.pile_steps), "stack100k_cubes": stack()}
    with api.Context(device=0) as ctx:
        for name, cols in worlds.items():
            ctx.query_update(cols)
            rays = rays_over(cols, 1_000_000, rng)
            casts = casts_over(cols, 1_000_000, rng)
            res[f"{name}/cast_ray_1M"] = timed(ctx, lambda: ctx.cast_ray(rays), 2, args.repeats)
            res[f"{name}/capsule_cast_1M"] = timed(ctx, lambda: ctx.cast_shape(casts), 2, args.repeats)
            res[f"{name}/colliders"] = int(cols.shape.shape[0])
            res[f"{name}/capsules"] = int((cols.shape == CAP).sum())
            print(name, res[f"{name}/cast_ray_1M"]["event_ms"], res[f"{name}/capsule_cast_1M"]["event_ms"], flush=True)
        cols = worlds["stack100k_cubes"]
        ctx.query_update(cols)
        cfg = api.MoveConfig()
        for label, shape in (("capsule", CAP), ("sphere", SPH)):
            batch = walkers(cols, 100_000, shape, rng)
            res[f"stack100k_cubes/move_100k_{label}"] = timed(ctx, lambda: ctx.move_and_slide(cfg, batch), 1, args.repeats)
            print(label, res[f"stack100k_cubes/move_100k_{label}"], flush=True)
    (out_dir / "capsule_query_timing.json").write_text(json.dumps(res, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
