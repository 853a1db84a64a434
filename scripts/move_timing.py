#!/usr/bin/env python
"""avn_move_and_slide at the headline scene (GPU box): characters walking on the 100k-cube stack (scenes.cube_stack(51, 40, 50), its
spawn poses), the reference's default MoveAndSlideConfig, 10k and 100k sphere and cuboid characters, f32 and f64 columns.  Per case, warmed
up and repeated (median, min, max): the move kernel's own device time (AvnMoveResult.kernel_ms, CUDA events around the launch), the whole
call (upload, kernel, download; events on the library's stream), and for scale one avn_query_cast_shape of the same characters along their
sweep (velocity * dt).  Prints the card and its power limit (nvidia-smi, read-only) and writes OUT_DIR/move_timing.json.
usage: python scripts/move_timing.py OUT_DIR [--repeats R]"""
import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
from avian_b200 import api  # noqa: E402
from test_gpu_move_and_slide import stack_world, walkers  # noqa: E402


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    name, limit = [x.strip() for x in out.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def stats(v) -> dict:
    return {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}


def timed(ctx, fn, warmup: int, repeats: int):
    """fn is one C-ABI call that ends in a stream synchronise; events bracket it on the library's stream.  Returns (call stats, results)"""
    import torch
    stream = torch.cuda.ExternalStream(ctx.stream())
    for _ in range(warmup):
        fn()
    ev_ms, wall_ms, outs = [], [], []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e0.record(stream)
        outs.append(fn())
        e1.record(stream)
        torch.cuda.synchronize()
        wall_ms.append((time.perf_counter() - t0) * 1e3)
        ev_ms.append(e0.elapsed_time(e1))
    return {"event_ms": stats(ev_ms), "wall_ms": stats(wall_ms), "repeats": repeats}, outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    out_dir = Path(a.out_dir)
    out_dir.mkdir(parents=True, exist_ok=True)
    gpu = card()
    print(f"card: {gpu['name']}, power limit {gpu['power_limit']}")
    cols = stack_world()
    cfg = api.MoveConfig()
    res = {"card": gpu, "scene": "cube_stack(51, 40, 50) spawn poses", "colliders": int(cols.shape.shape[0]), "config": "MoveAndSlideConfig::default",
           "delta_time": cfg.delta_time, "cases": []}
    for scalar in (np.float32, np.float64):
        with api.Context(device=0, scalar=scalar) as ctx:
            ctx.query_update(cols)
            for n in (10_000, 100_000):
                for name, shape in (("sphere", 1), ("cuboid", 0)):
                    b = walkers(np.random.default_rng(n + shape), cols, n)
                    b.shape[:] = shape
                    b = api.MoveBatch(shape=b.shape, dims=b.dims.astype(scalar), position=b.position.astype(scalar), rotation=b.rotation.astype(scalar),
                                      velocity=b.velocity.astype(scalar), planes=b.planes)
                    # the structs are built once: the timed call is the C-ABI call alone (upload, kernel, download)
                    cs, keep_c = cfg.as_struct()
                    bs, keep_b = b.as_struct(scalar)
                    o, out = api.move_result(n, cfg.move_and_slide_iterations, scalar)

                    def move():
                        ctx._check(ctx.lib.avn_move_and_slide(ctx.handle, C.byref(cs), C.byref(bs), C.byref(o)))
                        return {"kernel_ms": float(o.kernel_ms), "hit_collider": out["hit_collider"]}
                    call, outs = timed(ctx, move, a.warmup, a.repeats)
                    sweep = b.velocity.astype(np.float64) * cfg.delta_time
                    length = np.linalg.norm(sweep, axis=1)
                    casts = api.ShapeQueries(shape=b.shape, dims=b.dims, position=b.position, rotation=b.rotation,
                                             direction=(sweep / length[:, None]).astype(scalar), max_distance=length.astype(scalar),
                                             flags=np.full(n, api.CAST_IGNORE_ORIGIN_PENETRATION, np.uint32))
                    ss, keep_s = casts.as_struct(scalar)
                    so, sout = api.shape_closest(n, scalar)
                    cast, _ = timed(ctx, lambda: ctx._check(ctx.lib.avn_query_cast_shape(ctx.handle, C.byref(ss), C.byref(so))), a.warmup, a.repeats)
                    case = {"scalar": np.dtype(scalar).name, "characters": n, "shape": name, "move_kernel_ms": stats([o["kernel_ms"] for o in outs]),
                            "move_call": call, "cast_shape_call": cast,
                            "sweep_hits_per_character": float((outs[-1]["hit_collider"] >= 0).sum() / n)}
                    print(json.dumps(case))
                    res["cases"].append(case)
    (out_dir / "move_timing.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
