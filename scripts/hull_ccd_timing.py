#!/usr/bin/env python
"""Swept CCD with convex hull projectiles (GPU box; BASELINE.md §4.13).  1 000 and 10 000 projectiles (half Linear, half NonLinear) fired at
two targets stepped by DeviceGraphWorld: the 100k-cube stack of scripts/ccd_timing.py and scenes.hull_pile(100_000).  Per target and count
four arms run alternately in the same job, each warmed up and repeated: hull projectiles (a regular icosahedron of circumradius 0.2 added to
the target's hull table), and the cube, sphere and capsule projectiles of scripts/capsule_ccd_timing.py.  CCD is configured with hulls=True
and capsules=True in every arm, so the TOI kernel is the lowest shape level that covers the store: G = 2 (hulls) for the hull arm and on the
hull pile, G = 1 for the capsule arm on the stack, G = 0 for the cube and sphere arms on the stack.  Reported per arm: the CCD pass's device
time (AvnCcdResult::pass_ms), candidates and hits per step, as the median and the spread (min, max) over the timed steps.  Prints the card
and its power limit (nvidia-smi, read-only, in the same call) and writes OUT_DIR/hull_ccd_timing.json.
usage: python scripts/hull_ccd_timing.py OUT_DIR [--steps K] [--warmup W] [--rounds R]"""
import argparse
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))
from avian_b200 import api, scenes  # noqa: E402
from avian_b200.fixture import SHAPE_CAPSULE, SHAPE_CUBOID, SHAPE_SPHERE  # noqa: E402
from capsule_ccd_timing import DIMS, run_arm, summary  # noqa: E402
from ccd_timing import card  # noqa: E402

HULL = api.SHAPE_CONVEX_HULL
PROJECTILE_HULL = scenes.regular_solids(0.2)[2]   # icosahedron


def polyhedra(hulls):
    """the (vertices, faces) list of an api.ConvexHulls"""
    if hulls is None:
        return []
    out = []
    for h in range(hulls.count):
        v0, v1 = int(hulls.vertex_offsets[h]), int(hulls.vertex_offsets[h + 1])
        lo, lp = np.asarray(hulls.loop_offsets), np.asarray(hulls.loop)
        faces = [list(lp[lo[f]:lo[f + 1]]) for f in range(int(hulls.face_offsets[h]), int(hulls.face_offsets[h + 1]))]
        out.append((np.asarray(hulls.vertices, float).reshape(-1, 3)[v0:v1], faces))
    return out


def target(name: str):
    base = scenes.cube_stack(46, 47, 46, brick=False) if name == "cube_stack_100k" else scenes.hull_pile(100_000)
    p = base.bodies.position[1:].astype(np.float64)
    centre = 0.5 * (p.min(axis=0) + p.max(axis=0))
    radius = 0.5 * float(np.linalg.norm(p.max(axis=0) - p.min(axis=0)))
    return base, centre, radius


def with_projectiles(base, centre, radius, n: int, shape: int, seed: int = 0):
    """`n` projectiles of one shape at 200-400 m/s from just outside the target's bounding sphere, aimed at its centre; the target's bodies
    keep their mass properties, a hull projectile is an icosahedron appended to the target's hull table (its mass that of a 0.15 m cube)"""
    b = base.bodies
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n, 3))
    d[:, 1] = np.abs(d[:, 1])
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    ppos = centre + d * rng.uniform(radius + 1.0, radius + 5.0, (n, 1))
    pvel = -d * rng.uniform(200.0, 400.0, (n, 1))
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    polys = polyhedra(base.hulls)
    hulls = base.hulls
    if shape == HULL:
        hulls = api.ConvexHulls.from_polyhedra(polys + [PROJECTILE_HULL])
    pdims = np.tile([float(len(polys)), 0.0, 0.0] if shape == HULL else DIMS[shape], (n, 1))
    mass_dims = np.tile(DIMS[SHAPE_CUBOID] if shape == HULL else DIMS[shape], (n, 1))
    mass_shape = SHAPE_CUBOID if shape == HULL else shape
    base_mass_dims = np.where((base.shape_type == HULL)[:, None], 0.5, base.dims)
    scene = scenes._assemble("hull_ccd_target", np.concatenate([b.position.astype(np.float64), ppos]), np.concatenate([b.rotation.astype(np.float64), q]),
                             np.concatenate([b.kind, np.zeros(n, np.uint8)]), np.concatenate([base_mass_dims, mass_dims]),
                             np.concatenate([base.shape_type, np.full(n, mass_shape)]), np.float32,
                             linvel=np.concatenate([b.linear_velocity.astype(np.float64), pvel]), hulls=hulls)
    scene.shape_type = np.ascontiguousarray(np.concatenate([base.shape_type, np.full(n, shape)]), dtype=np.int32)
    scene.dims = np.ascontiguousarray(np.concatenate([base.dims, pdims]))
    scene.bodies.inverse_mass[:b.count] = b.inverse_mass
    scene.bodies.inverse_inertia_local[:b.count] = b.inverse_inertia_local
    return scene, np.arange(b.count, b.count + n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2, help="alternations of the four arms")
    a = ap.parse_args()
    out = {"card": card(), "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds, "arms": {}}
    print(out["card"], flush=True)
    names = {HULL: "hull", SHAPE_CUBOID: "cube", SHAPE_SPHERE: "sphere", SHAPE_CAPSULE: "capsule"}
    for tname in ("cube_stack_100k", "hull_pile_100k"):
        base, centre, radius = target(tname)
        for n in (1000, 10000):
            raw = {s: {"pass_ms": [], "candidates": [], "hits": []} for s in names}
            scenes_ = {s: with_projectiles(base, centre, radius, n, s) for s in names}
            for _ in range(a.rounds):
                for s in names:                       # the four arms alternate
                    scene, ccd = scenes_[s]
                    cfg = dict(body=ccd, collider=ccd, mode=(np.arange(n) % 2).astype(np.uint8), capsules=True, hulls=True)
                    r = run_arm(scene, cfg, a.steps, a.warmup)
                    for k in raw[s]:
                        raw[s][k] += r[k]
            for s, label in names.items():
                key = f"{tname}, {n} {label} projectiles"
                out["arms"][key] = {k: summary(v) for k, v in raw[s].items()}
                print(key, out["arms"][key], flush=True)
    out["card_after"] = card()
    Path(a.out_dir).mkdir(parents=True, exist_ok=True)
    (Path(a.out_dir) / "hull_ccd_timing.json").write_text(json.dumps(out, indent=1))
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
