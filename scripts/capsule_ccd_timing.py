#!/usr/bin/env python
"""Swept CCD with capsule projectiles (GPU box; BASELINE.md §4.10).  1 000 and 10 000 projectiles (half Linear, half NonLinear) fired at two
targets stepped by DeviceGraphWorld: the 100k-cube stack of scripts/ccd_timing.py and scenes.capsule_pile(100_000).  Per target and count
three arms run alternately in the same job, each warmed up and repeated: capsule projectiles (CCD configured with capsules=True, so the
CAPS = true TOI kernel runs), and the sphere and cube projectiles of scripts/ccd_timing.py (on the capsule pile the store holds capsules,
so those arms need the flag and run the CAPS = true kernel too).  Reported per arm: the CCD pass's device time (AvnCcdResult::pass_ms),
candidates and hits per step, as the median and the spread (min, max) over the timed steps.  Prints the card and its power limit
(nvidia-smi, read-only, in the same call) and writes OUT_DIR/capsule_ccd_timing.json.
usage: python scripts/capsule_ccd_timing.py OUT_DIR [--steps K] [--warmup W] [--rounds R]"""
import argparse
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))
from avian_b200 import api, plugins, scenes  # noqa: E402
from avian_b200.fixture import SHAPE_CAPSULE, SHAPE_CUBOID, SHAPE_SPHERE  # noqa: E402
from ccd_timing import card  # noqa: E402

DIMS = {SHAPE_CAPSULE: [0.1, 0.25, 0.0], SHAPE_SPHERE: [0.15, 0.0, 0.0], SHAPE_CUBOID: [0.15, 0.15, 0.15]}


def target(name: str):
    if name == "cube_stack_100k":
        base = scenes.cube_stack(46, 47, 46, brick=False)
    else:
        base = scenes.capsule_pile(100_000)
    p = base.bodies.position[1:].astype(np.float64)
    centre = 0.5 * (p.min(axis=0) + p.max(axis=0))
    radius = 0.5 * float(np.linalg.norm(p.max(axis=0) - p.min(axis=0)))
    return base, centre, radius


def with_projectiles(base, centre, radius, n: int, shape: int, seed: int = 0):
    """`n` projectiles of one shape at 200-400 m/s from just outside the target's bounding sphere, aimed at its centre"""
    b = base.bodies
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n, 3))
    d[:, 1] = np.abs(d[:, 1])
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    ppos = centre + d * rng.uniform(radius + 1.0, radius + 5.0, (n, 1))
    pvel = -d * rng.uniform(200.0, 400.0, (n, 1))
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    scene = scenes._assemble("ccd_target", np.concatenate([b.position.astype(np.float64), ppos]), np.concatenate([b.rotation.astype(np.float64), q]),
                             np.concatenate([b.kind, np.zeros(n, np.uint8)]), np.concatenate([base.dims, np.tile(DIMS[shape], (n, 1))]),
                             np.concatenate([base.shape_type, np.full(n, shape)]), np.float32,
                             linvel=np.concatenate([b.linear_velocity.astype(np.float64), pvel]))
    return scene, np.arange(b.count, b.count + n)


def run_arm(scene, ccd: dict, steps: int, warmup: int) -> dict:
    with api.Context(device=0) as ctx:
        w = plugins.DeviceGraphWorld(scene, plugins.PhysicsPlugins(ctx), ctx, substeps=8, ccd=ccd)
        passes, cand, hits = [], [], []
        for i in range(warmup + steps):
            w.step()
            if i < warmup:
                continue
            r = ctx.ccd_download()
            passes.append(r["pass_ms"])
            cand.append(r["total_candidates"])
            hits.append(int((r["hit_body"] >= 0).sum()))
    return {"pass_ms": passes, "candidates": cand, "hits": hits}


def summary(samples: list) -> dict:
    a = np.asarray(samples, dtype=np.float64)
    return {"median": float(np.median(a)), "min": float(a.min()), "max": float(a.max()), "n": int(a.size)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2, help="alternations of the three arms")
    a = ap.parse_args()
    out = {"card": card(), "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds, "arms": {}}
    print(out["card"], flush=True)
    names = {SHAPE_CAPSULE: "capsule", SHAPE_SPHERE: "sphere", SHAPE_CUBOID: "cube"}
    for tname in ("cube_stack_100k", "capsule_pile_100k"):
        base, centre, radius = target(tname)
        for n in (1000, 10000):
            raw = {s: {"pass_ms": [], "candidates": [], "hits": []} for s in names}
            scenes_ = {s: with_projectiles(base, centre, radius, n, s) for s in names}
            for _ in range(a.rounds):
                for s in names:                       # the three arms alternate
                    scene, ccd = scenes_[s]
                    cfg = dict(body=ccd, collider=ccd, mode=(np.arange(n) % 2).astype(np.uint8), capsules=True)
                    r = run_arm(scene, cfg, a.steps, a.warmup)
                    for k in raw[s]:
                        raw[s][k] += r[k]
            for s, label in names.items():
                key = f"{tname}, {n} {label} projectiles"
                out["arms"][key] = {k: summary(v) for k, v in raw[s].items()}
                print(key, out["arms"][key], flush=True)
    out["card_after"] = card()
    Path(a.out_dir).mkdir(parents=True, exist_ok=True)
    (Path(a.out_dir) / "capsule_ccd_timing.json").write_text(json.dumps(out, indent=1))
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
