#!/usr/bin/env python
"""Convex hull colliders on the device-resident step (plugins.DeviceGraphWorld: broad phase, avn_contacts_step, solver stage), in one process:
scenes.hull_pile(30 000) (70 % hulls from a table of 28, the rest cuboids, spheres and capsules) beside the same pile with every hull replaced
by the cuboid of its local bounding box, and scenes.decomposed_pile(5 000) (bodies of 2-4 hull parts).  Per scene, after `--warmup` steps
(the piles land and settle), `--steps` steps are timed on the host clock (every step ends in a device synchronise): the whole step and its
avn_contacts_step call.  Then the narrow kernels alone: avn_narrow_phase on a seeded soup of 100k hull-hull pairs of the pile's table, and on
10k overlapping pairs of a 64-vertex, 124-face hull (the vertex limit: 186 edges, 34 596 edge pairs before the Gauss-map test), the device
time of every kernel whose name holds "narrow" summed by torch.profiler (CUDA activities) over `--calls` calls.  Prints the card and its power
limit (nvidia-smi, read-only) and writes OUT_DIR/hull_timing.json.
usage: python scripts/hull_timing.py OUT_DIR [--steps K] [--warmup W] [--calls N]"""
import argparse
import dataclasses
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from avian_b200 import api, plugins, scenes  # noqa: E402

DT, TOL = 1.0 / 60.0, 0.005


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    name, limit = [x.strip() for x in out.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def stats(v) -> dict:
    return {"median_ms": float(np.median(v)) * 1e3, "min_ms": float(np.min(v)) * 1e3, "max_ms": float(np.max(v)) * 1e3}


def as_cuboids(sc):
    """the pile with every hull body replaced by the cuboid of its hull's local bounding box (mass properties of that cuboid)"""
    hull = sc.shape_type == api.SHAPE_CONVEX_HULL
    dims = sc.dims.copy()
    inv_m, inv_i = sc.bodies.inverse_mass.copy(), sc.bodies.inverse_inertia_local.copy()
    for b in np.nonzero(hull)[0]:
        v, _ = sc.hulls.polyhedron(int(sc.dims[b, 0]))
        he = 0.5 * (v.max(axis=0) - v.min(axis=0))
        dims[b] = he
        m, i = scenes._cuboid_mass(he[None, :])
        inv_m[b] = 1.0 / m[0]
        inv_i[b] = [1.0 / i[0, 0], 0, 0, 1.0 / i[0, 1], 0, 1.0 / i[0, 2]]
    bodies = dataclasses.replace(sc.bodies, inverse_mass=inv_m, inverse_inertia_local=inv_i)
    shape = np.where(hull, scenes.SHAPE_CUBOID, sc.shape_type).astype(np.int32)
    return dataclasses.replace(sc, name=sc.name + "_cuboids", bodies=bodies, shape_type=shape, dims=dims, hulls=None)


def run(scene, steps: int, warmup: int) -> dict:
    with api.Context(device=0, scalar=scene.bodies.position.dtype) as ctx:
        w = plugins.DeviceGraphWorld(scene, plugins.PhysicsPlugins(ctx), ctx, substeps=4)
        contact_s = []
        inner = ctx.contacts_step

        def timed_contacts_step(*a, **kw):
            t0 = time.perf_counter()
            out = inner(*a, **kw)
            contact_s.append(time.perf_counter() - t0)
            return out

        ctx.contacts_step = timed_contacts_step
        for _ in range(warmup):
            w.step()
        contact_s.clear()
        step_s = []
        for _ in range(steps):
            t0 = time.perf_counter()
            w.step()
            step_s.append(time.perf_counter() - t0)
        nc = int(scene.collider_body.shape[0]) if scene.compound else int(scene.bodies.count)
        return {"bodies": int(scene.bodies.count), "colliders": nc, "rows_live": int(w.stats["rows_live"]), "manifolds": int(w.stats["manifold_count"]),
                "step": stats(step_s), "contacts_step": stats(contact_s)}


def hull_soup(hulls, n, seed, overlap=False):
    """n hull-hull pairs of `hulls`: random orientations, centres from overlapping to just past the margin (overlap: within half the radii)"""
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, hulls.count, 2 * n)
    q = rng.normal(size=(2 * n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    r = np.array([np.linalg.norm(hulls.polyhedron(h)[0], axis=1).max() for h in range(hulls.count)])
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    reach = r[idx[0::2]] + r[idx[1::2]]
    d *= (rng.uniform(0.2, 0.5, n) if overlap else rng.uniform(0.3, 1.1, n))[:, None] * reach[:, None]
    pos = np.zeros((2 * n, 3)); pos[0::2] = rng.uniform(-50, 50, (n, 3)); pos[1::2] = pos[0::2] + d
    dims = np.zeros((2 * n, 3)); dims[:, 0] = idx
    cols = {"shape": np.full(2 * n, api.SHAPE_CONVEX_HULL, np.uint8), "dims": dims.astype(np.float32), "position": pos.astype(np.float32),
            "rotation": q.astype(np.float32)}
    c1, c2 = np.arange(0, 2 * n, 2, dtype=np.uint32), np.arange(1, 2 * n, 2, dtype=np.uint32)
    return (c1, c2, c1, c2), cols, np.zeros((2 * n, 3), np.float32), np.zeros((2 * n, 3), np.float32)


def narrow_kernels(hulls, pairs_n: int, calls: int, overlap: bool) -> dict:
    import torch
    from torch.profiler import ProfilerActivity, profile
    pairs, cols, lv, av = hull_soup(hulls, pairs_n, 5, overlap)
    with api.Context(device=0) as ctx:
        ctx.set_convex_hulls(hulls)
        for _ in range(2):
            out = ctx.narrow_phase(DT, TOL, pairs, cols, lv, av)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(calls):
                ctx.narrow_phase(DT, TOL, pairs, cols, lv, av)
            torch.cuda.synchronize()
    ks = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and "narrow" in e.name:
            k = e.name.replace("(anonymous namespace)::", "").split("(")[0]
            ks[k] = ks.get(k, 0.0) + e.device_time / 1e3
    return {"pairs": pairs_n, "calls": calls, "touching": int((out["point_count"] > 0).sum()), "kernel_ms_per_call": {k: v / calls for k, v in ks.items()},
            "total_ms_per_call": sum(ks.values()) / calls}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=240, help="steps before a pile is timed (the top layer lands after ~80)")
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--bodies", type=int, default=30_000)
    ap.add_argument("--decomposed-bodies", type=int, default=5_000)
    args = ap.parse_args()
    out = Path(args.out_dir)
    out.mkdir(parents=True, exist_ok=True)
    result = {"card": card(), "steps": args.steps, "warmup": args.warmup, "scenes": {}}
    print("card:", result["card"], flush=True)
    pile = scenes.hull_pile(args.bodies)
    for name, fn in (("hull_pile", lambda: pile), ("hull_pile_as_cuboids", lambda: as_cuboids(scenes.hull_pile(args.bodies))),
                     ("decomposed_pile", lambda: scenes.decomposed_pile(args.decomposed_bodies))):
        r = run(fn(), args.steps, args.warmup)
        result["scenes"][name] = r
        print(f"{name:22s} bodies {r['bodies']:7d} colliders {r['colliders']:7d} rows {r['rows_live']:7d}  step {r['step']['median_ms']:8.2f} ms"
              f"  contacts_step {r['contacts_step']['median_ms']:8.2f} ms", flush=True)
    k = np.arange(64) + 0.5   # 64 points of a Fibonacci sphere: every one a hull vertex
    z, phi = 1 - 2 * k / 64, np.pi * (1 + 5 ** 0.5) * k
    ball = scenes.convex_hull_of(0.3 * np.stack([np.sqrt(1 - z * z) * np.cos(phi), np.sqrt(1 - z * z) * np.sin(phi), z], axis=1))
    result["narrow_kernels"] = {"pile_table_100k": narrow_kernels(pile.hulls, 100_000, args.calls, False),
                                "limit_hull_10k_overlapping": narrow_kernels(api.ConvexHulls.from_polyhedra([ball]), 10_000, args.calls, True)}
    result["limit_hull"] = {"vertices": int(len(ball[0])), "faces": len(ball[1])}
    for k_, v in result["narrow_kernels"].items():
        print(f"avn_narrow_phase {k_:28s} {v['total_ms_per_call']:.3f} ms per call of {v['pairs']} pairs ({v['touching']} touching): "
              f"{v['kernel_ms_per_call']}", flush=True)
    (out / "hull_timing.json").write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
