#!/usr/bin/env python
"""The device-resident step (plugins.DeviceGraphWorld: broad phase, avn_contacts_step, solver stage) on capsule scenes beside the cuboid scenes
they replace, in one process: 5 000 ragdolls with capsule legs against the cuboid ragdolls (scenes.ragdoll_field), and a 100k-body capsule
pile (scenes.capsule_pile) against the 100k-cube stack (scenes.cube_stack(51, 40, 50)).  Per scene, after `--warmup` steps, `--steps` steps
are timed on the host clock (every step ends in a device synchronise): the whole step and its avn_contacts_step call (the narrow pass over
every live row, matching, the status loop and the colouring).  The host fixture's AABB update is part of the step, as in bench.py's
end-to-end arm.  The capsule pile falls for about two seconds after spawning: it is timed after `--pile-warmup` steps, once it has landed and
settled.  Prints the card and its power limit (nvidia-smi, read-only) and writes OUT_DIR/capsule_timing.json.
usage: python scripts/capsule_timing.py OUT_DIR [--steps K] [--warmup W] [--pile-warmup P]"""
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
        return {"bodies": int(scene.bodies.count), "capsules": int((scene.shape_type == api.SHAPE_CAPSULE).sum()), "rows_live": int(w.stats["rows_live"]),
                "manifolds": int(w.stats["manifold_count"]), "step": stats(step_s), "contacts_step": stats(contact_s)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--pile-warmup", type=int, default=360, help="steps before the capsule pile is timed (it lands after ~120)")
    args = ap.parse_args()
    out = Path(args.out_dir)
    out.mkdir(parents=True, exist_ok=True)
    result = {"card": card(), "steps": args.steps, "warmup": args.warmup, "scenes": {}}
    print("card:", result["card"])
    cases = [("ragdolls5k_cuboid", lambda: scenes.ragdoll_field(5000), args.warmup),
             ("ragdolls5k_capsule_legs", lambda: scenes.ragdoll_field(5000, limbs="capsule"), args.warmup),
             ("stack100k_cubes", lambda: scenes.cube_stack(51, 40, 50), args.warmup), ("capsule_pile100k", lambda: scenes.capsule_pile(100_000), args.pile_warmup)]
    result["pile_warmup"] = args.pile_warmup
    for name, fn, warmup in cases:
        r = run(fn(), args.steps, warmup)
        result["scenes"][name] = r
        print(f"{name:26s} bodies {r['bodies']:7d} capsules {r['capsules']:6d} rows {r['rows_live']:7d}  step {r['step']['median_ms']:8.2f} ms"
              f"  contacts_step {r['contacts_step']['median_ms']:8.2f} ms", flush=True)
    (out / "capsule_timing.json").write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
