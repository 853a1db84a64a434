#!/usr/bin/env python
"""Latency breakdown of the wavefront items (GPU box).  Loads the -DAVN_WAVE_TRACE build of the library
(avian_b200/lib/libavian_b200_trace.so; build: see DESIGN.md §3.1) and runs a few solver stages; the library prints the
average SM cycles per contact item-warp of stage 1 (delta wait + separations) / wait / loads / compute / store+publish to stderr."""
import ctypes as C
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from avian_b200 import api  # noqa: E402

from avian_b200 import _build  # noqa: E402
lib = C.CDLL(str(_build.build_variant("trace", ["AVN_WAVE_TRACE"])))
api.bind_abi(lib)
api._lib = lib
import bench  # noqa: E402

scene = sys.argv[1] if len(sys.argv) > 1 else "stack100k"
with api.Context(device=0) as ctx:
    sc, prm, bodies, man, aabbs, joints = bench.build_snapshot(scene, bench.SCENES[scene][2], ctx)
    b, m = bodies.copy(), man.copy()
    ctx.solver_upload(prm, b, m, joints)
    for _ in range(4):
        ctx.solver_run()
        ctx.solver_download()
        print("solver stage ms", ctx.timings()["total_ms"], flush=True)
