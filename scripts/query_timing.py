#!/usr/bin/env python
"""Spatial queries at the headline scene (GPU box): the 100k-cube stack after bench.py's settle steps, as its device-resident world leaves it.
Times, each warmed up and repeated (median, min, max):
  * the resident step (DeviceGraphWorld.step_from, bench.py's e2e arm) — what the update is set against;
  * avn_query_update over all 100 001 colliders, with and without AVN_QUERY_SHAPES_UNCHANGED;
  * 1 000 000 closest-hit rays: a downward grid over the stack + random directions from inside it;
  * 100 000 ray_hits rays keeping all hits (downward grid);
  * 100 000 AABB queries (a box of half size 0.6 around random cubes);
  * 1 000 000 closest sphere casts and 1 000 000 closest cuboid casts straight down over the stack;
  * 100 000 shape_hits casts keeping all hits (downward, half spheres, half cubes);
  * 1 000 000 project_point queries around random cubes (half solid, half hollow);
  * 100 000 point intersections and 100 000 shape intersections around random cubes.
Every query time is one C-ABI call from host columns (already in the context's scalar) to host results (upload, kernels, download): CUDA
events on the library's stream and the host clock, both closed by the call's own stream synchronise.  Prints the card and its power limit
(nvidia-smi, read-only) and writes OUT_DIR/query_timing.json.   usage: python scripts/query_timing.py OUT_DIR [--repeats R]"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from avian_b200 import api, plugins  # noqa: E402


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    name, limit = [x.strip() for x in out.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def timed(ctx, fn, warmup: int, repeats: int) -> dict:
    """fn is one (or a few) C-ABI calls that end in a stream synchronise; events bracket them on the library's stream"""
    import torch
    stream = torch.cuda.ExternalStream(ctx.stream())
    for _ in range(warmup):
        fn()
    ev_ms, wall_ms = [], []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e0.record(stream)
        fn()
        e1.record(stream)
        torch.cuda.synchronize()
        wall_ms.append((time.perf_counter() - t0) * 1e3)
        ev_ms.append(e0.elapsed_time(e1))
    s = lambda v: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
    return {"event_ms": s(ev_ms), "wall_ms": s(wall_ms), "repeats": repeats}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--steps", type=int, default=20, help="resident steps per repeat of the step timing")
    a = ap.parse_args()
    out_dir = Path(a.out_dir)
    out_dir.mkdir(parents=True, exist_ok=True)
    gpu = card()
    print(f"card: {gpu['name']}, power limit {gpu['power_limit']}")

    class Args:
        pass
    args = Args()
    args.scene, args.settle, args.solver_iterations, args.warmup = "stack100k", bench.SCENES["stack100k"][2], 1, 3
    rng = np.random.default_rng(0)
    res = {"card": gpu, "scene": "stack100k", "settle_steps": args.settle}
    with api.Context(device=0, scalar=np.float32) as ctx:
        w, aabbs, mn, mx, _ = bench._resident_world(args, ctx)
        n = int(w.bodies.count)
        step = timed(ctx, lambda: [w.step_from(aabbs, mn, mx) for _ in range(a.steps)], 1, a.repeats)
        res["resident_step_ms"] = {k: v / a.steps for k, v in step["wall_ms"].items()}
        c0 = plugins.SpatialQueryPlugin.colliders(w)
        cols = api.QueryColliders(shape=np.ascontiguousarray(c0.shape, dtype=np.uint8), dims=np.ascontiguousarray(c0.dims, dtype=np.float32),
                                  position=c0.position, rotation=c0.rotation)      # f32 columns, as the context takes them
        res["colliders"] = n
        res["update_ms"] = timed(ctx, lambda: ctx.query_update(cols), a.warmup, a.repeats)
        res["update_shapes_unchanged_ms"] = timed(ctx, lambda: ctx.query_update(cols, shapes_unchanged=True), a.warmup, a.repeats)
        # the same with the pose columns in page-locked memory: how much of the update is the copy of the poses over the bus
        pinned = api.QueryColliders(shape=cols.shape, dims=cols.dims, position=ctx.pin_like(np.asarray(cols.position)),
                                    rotation=ctx.pin_like(np.asarray(cols.rotation)))
        res["update_shapes_unchanged_pinned_ms"] = timed(ctx, lambda: ctx.query_update(pinned, shapes_unchanged=True), a.warmup, a.repeats)
        ratio = res["update_shapes_unchanged_ms"]["wall_ms"]["median"] / res["resident_step_ms"]["median"]
        res["update_over_resident_step"] = ratio

        pos = np.asarray(w.bodies.position[1:], dtype=np.float64)
        lo, hi = pos.min(axis=0) - 1.0, pos.max(axis=0) + 1.0
        side = 708                                   # 708^2 ~ 501k downward rays
        gx, gz = np.meshgrid(np.linspace(lo[0], hi[0], side), np.linspace(lo[2], hi[2], side), indexing="ij")
        down_o = np.stack([gx.ravel(), np.full(gx.size, hi[1] + 5.0), gz.ravel()], 1)
        k = 1_000_000 - down_o.shape[0]
        d = rng.normal(size=(k, 3))
        inside_o = pos[rng.integers(0, n - 1, k)] + rng.uniform(-0.3, 0.3, (k, 3))
        f = np.float32          # the columns in the context's scalar, built once: the timed calls convert nothing
        rays = api.Rays(origin=np.concatenate([down_o, inside_o]).astype(f), direction=np.concatenate([np.tile([0.0, -1.0, 0.0], (down_o.shape[0], 1)),
                                                                                                       d / np.linalg.norm(d, axis=1, keepdims=True)]).astype(f),
                        max_distance=np.full(down_o.shape[0] + k, 100.0, dtype=f))
        res["cast_ray_1m_ms"] = timed(ctx, lambda: ctx.cast_ray(rays), a.warmup, a.repeats)
        hit = ctx.cast_ray(rays)["collider"] >= 0
        res["cast_ray_1m_hit_fraction"] = float(hit.mean())

        side = 317                                   # 317^2 ~ 100k
        gx, gz = np.meshgrid(np.linspace(lo[0], hi[0], side), np.linspace(lo[2], hi[2], side), indexing="ij")
        m = 100_000
        o = np.stack([gx.ravel(), np.full(gx.size, hi[1] + 5.0), gz.ravel()], 1)[:m]
        hits_rays = api.Rays(origin=o.astype(f), direction=np.tile([0.0, -1.0, 0.0], (m, 1)).astype(f), max_distance=np.full(m, 100.0, dtype=f))
        h = ctx.ray_hits(hits_rays)
        cap = int(h["collider"].shape[0])
        res["ray_hits_100k_total_hits"] = cap
        res["ray_hits_100k_ms"] = timed(ctx, lambda: ctx.ray_hits(hits_rays, capacity=cap), a.warmup, a.repeats)

        c = pos[rng.integers(0, n - 1, 100_000)]
        qmn, qmx = (c - 0.6).astype(f), (c + 0.6).astype(f)
        q = ctx.aabb_intersections(qmn, qmx)
        res["aabb_100k_total_hits"] = int(q["collider"].shape[0])
        acap = res["aabb_100k_total_hits"]
        res["aabb_100k_ms"] = timed(ctx, lambda: ctx.aabb_intersections(qmn, qmx, capacity=acap), a.warmup, a.repeats)

        # shape casts straight down over the stack (a 1000 x 1000 grid), spheres of radius 0.25 and unrotated cubes of half size 0.25
        side = 1000
        gx, gz = np.meshgrid(np.linspace(lo[0], hi[0], side), np.linspace(lo[2], hi[2], side), indexing="ij")
        k = gx.size
        cast_o = np.stack([gx.ravel(), np.full(k, hi[1] + 5.0), gz.ravel()], 1).astype(f)
        for name, shape in (("sphere", 1), ("cuboid", 0)):
            casts = api.ShapeQueries(shape=np.full(k, shape, np.uint8), dims=np.full((k, 3), 0.25, dtype=f), position=cast_o,
                                     rotation=np.tile(np.array([0, 0, 0, 1], dtype=f), (k, 1)), direction=np.tile(np.array([0, -1, 0], dtype=f), (k, 1)),
                                     max_distance=np.full(k, 100.0, dtype=f))
            res[f"cast_shape_{name}_1m_ms"] = timed(ctx, lambda: ctx.cast_shape(casts), a.warmup, a.repeats)
            res[f"cast_shape_{name}_1m_hit_fraction"] = float((ctx.cast_shape(casts)["collider"] >= 0).mean())
        m = 100_000
        idx = np.linspace(0, k - 1, m).astype(np.int64)
        hits_casts = api.ShapeQueries(shape=(np.arange(m) % 2).astype(np.uint8), dims=np.full((m, 3), 0.25, dtype=f), position=cast_o[idx],
                                      rotation=np.tile(np.array([0, 0, 0, 1], dtype=f), (m, 1)), direction=np.tile(np.array([0, -1, 0], dtype=f), (m, 1)),
                                      max_distance=np.full(m, 100.0, dtype=f), max_hits=np.full(m, api.MAX_HITS_ALL, np.uint32))
        sh = ctx.shape_hits(hits_casts)
        scap = int(sh["collider"].shape[0])
        res["shape_hits_100k_total_hits"] = scap
        res["shape_hits_100k_ms"] = timed(ctx, lambda: ctx.shape_hits(hits_casts, capacity=scap), a.warmup, a.repeats)

        # 1M points around random cubes (half of them hollow), and 100k points / shapes for the intersection tests
        c = pos[rng.integers(0, n - 1, 1_000_000)] + rng.uniform(-0.8, 0.8, (1_000_000, 3))
        pts = api.Points(point=c.astype(f), solid=(np.arange(c.shape[0]) % 2 == 0))
        res["project_point_1m_ms"] = timed(ctx, lambda: ctx.project_point(pts), a.warmup, a.repeats)
        ipts = api.Points(point=c[:m].astype(f))
        res["point_intersections_100k_total_hits"] = int(ctx.point_intersections(ipts)["collider"].shape[0])
        pcap = res["point_intersections_100k_total_hits"]
        res["point_intersections_100k_ms"] = timed(ctx, lambda: ctx.point_intersections(ipts, capacity=pcap), a.warmup, a.repeats)
        q = rng.normal(size=(m, 4))
        isect = api.ShapeQueries(shape=(np.arange(m) % 2).astype(np.uint8), dims=np.full((m, 3), 0.4, dtype=f), position=c[:m].astype(f),
                                 rotation=(q / np.linalg.norm(q, axis=1, keepdims=True)).astype(f))
        res["shape_intersections_100k_total_hits"] = int(ctx.shape_intersections(isect)["collider"].shape[0])
        icap = res["shape_intersections_100k_total_hits"]
        res["shape_intersections_100k_ms"] = timed(ctx, lambda: ctx.shape_intersections(isect, capacity=icap), a.warmup, a.repeats)
    (out_dir / "query_timing.json").write_text(json.dumps(res, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
