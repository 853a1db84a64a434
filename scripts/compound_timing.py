#!/usr/bin/env python
"""Compound bodies on the device-resident step (plugins.DeviceGraphWorld: broad phase, avn_contacts_step with body frames, solver stage) beside
a single-collider pile of the same collider count, in one process: scenes.compound_pile(30 000) (tables, dumbbells and L-blocks, about 100k
colliders) against scenes.compound_pile(C - 1, single_share=1) (one cuboid, sphere or capsule per body, the same C colliders).  Per scene,
after `--warmup` steps (the piles land and settle), `--steps` steps are timed on the host clock (every step ends in a device synchronise): the
whole step and its avn_contacts_step call.  Then the narrow kernels alone, with and without body frames: avn_narrow_phase on one seeded pair
soup (tests/compound_scenes.py), the device time of every kernel whose name holds "narrow" summed by torch.profiler (CUDA activities) over
`--calls` calls of each.  Prints the card and its power limit (nvidia-smi, read-only) and writes OUT_DIR/compound_timing.json.
usage: python scripts/compound_timing.py OUT_DIR [--steps K] [--warmup W] [--calls N]"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
from avian_b200 import api, plugins, scenes  # noqa: E402
from compound_scenes import DT, TOL, soup  # noqa: E402


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    name, limit = [x.strip() for x in out.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def stats(v) -> dict:
    return {"median_ms": float(np.median(v)) * 1e3, "min_ms": float(np.min(v)) * 1e3, "max_ms": float(np.max(v)) * 1e3}


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
        return {"bodies": int(scene.bodies.count), "colliders": int(scene.collider_body.shape[0]), "rows_live": int(w.stats["rows_live"]),
                "manifolds": int(w.stats["manifold_count"]), "step": stats(step_s), "contacts_step": stats(contact_s)}


def narrow_kernels(calls: int, pairs_n: int) -> dict:
    import torch
    from torch.profiler import ProfilerActivity, profile
    pairs, cols, lv, av, frames = soup(np.float32, 5, n=pairs_n)
    out = {}
    with api.Context(device=0) as ctx:
        for name, fr in (("without_frames", None), ("with_frames", frames)):
            if fr is None:
                ctx.contacts_set_body_frames()
            else:
                ctx.contacts_set_body_frames(fr["position"], fr["rotation"], fr["center_of_mass"])
            for _ in range(3):
                ctx.narrow_phase(DT, TOL, pairs, cols, lv, av)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(calls):
                    ctx.narrow_phase(DT, TOL, pairs, cols, lv, av)
                torch.cuda.synchronize()
            ks = {}
            for e in prof.events():
                if e.device_type.name == "CUDA" and "narrow" in e.name:
                    k = e.name.replace("(anonymous namespace)::", "").split("(")[0]
                    ks[k] = ks.get(k, 0.0) + e.device_time / 1e3
            out[name] = {"pairs": pairs_n, "calls": calls, "kernel_ms_per_call": {k: v / calls for k, v in ks.items()},
                         "total_ms_per_call": sum(ks.values()) / calls}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=240, help="steps before a pile is timed (the top layer lands after ~80)")
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--bodies", type=int, default=30_000)
    args = ap.parse_args()
    out = Path(args.out_dir)
    out.mkdir(parents=True, exist_ok=True)
    result = {"card": card(), "steps": args.steps, "warmup": args.warmup, "scenes": {}}
    print("card:", result["card"])
    compound = scenes.compound_pile(args.bodies)
    C = int(compound.collider_body.shape[0])
    for name, sc in (("compound_pile", compound), ("single_collider_pile", scenes.compound_pile(C - 1, single_share=1.0))):
        r = run(sc, args.steps, args.warmup)
        result["scenes"][name] = r
        print(f"{name:22s} bodies {r['bodies']:7d} colliders {r['colliders']:7d} rows {r['rows_live']:7d}  step {r['step']['median_ms']:8.2f} ms"
              f"  contacts_step {r['contacts_step']['median_ms']:8.2f} ms", flush=True)
    result["narrow_kernels"] = narrow_kernels(args.calls, 100_000)
    for k, v in result["narrow_kernels"].items():
        print(f"avn_narrow_phase kernels {k:15s} {v['total_ms_per_call']:.3f} ms per call of {v['pairs']} pairs: {v['kernel_ms_per_call']}", flush=True)
    (out / "compound_timing.json").write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
