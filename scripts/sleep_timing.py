"""Cost and gain of applied sleeping (avn_islands_apply / avn_islands_wake, DESIGN.md §7c) on two 100k-cube scenes — 10 000 independent
columns (cube_stack(100, 10, 100, brick=False)) and one coupled pile (cube_stack(51, 40, 50)) — through plugins.DeviceGraphWorld:
  (a) awake, application off (islands configured, avn_islands_step decides only; thresholds negative: nothing ever sleeps),
  (b) awake, application on (the cost of the asleep bytes, avn_islands_wake and the effective kind column),
  (c) every body asleep (generous thresholds, short TimeToSleep),
  (d) the step in which one touched body wakes its island out of (c).
Per case the median wall time of a whole step and of each library call in it (every call ends in a synchronise of the library's stream).
Prints one JSON line; with --out DIR it also writes DIR/sleep_timing.json.

    python scripts/sleep_timing.py [--steps 20] [--settle 8] [--out DIR]
"""
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

CALLS = ("broadphase_upload", "broadphase_run", "contacts_step", "broadphase_download_order", "islands_wake", "solver_step_resident", "islands_step")


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception as e:  # the numbers stay valid, only the label is missing
        return f"unknown ({e})", "unknown"


class _Clock:
    """wall time per library call of one context, by wrapping the bound methods"""
    def __init__(self, ctx):
        self.t = {}
        for name in CALLS:
            fn = getattr(ctx, name)
            setattr(ctx, name, self._wrap(name, fn))

    def _wrap(self, name, fn):
        def timed(*a, **kw):
            t0 = time.perf_counter()
            r = fn(*a, **kw)
            self.t[name] = self.t.get(name, 0.0) + (time.perf_counter() - t0) * 1e3
            return r
        return timed

    def take(self):
        t, self.t = self.t, {}
        return t


def _summary(samples):
    med = lambda xs: round(float(np.median(xs)), 3)
    out = {"step_ms": med([s["step"] for s in samples]), "steps": len(samples)}
    for name in CALLS:
        xs = [s.get(name, 0.0) for s in samples]
        if any(xs):
            out[name + "_ms"] = med(xs)
    return out


def _timed_step(w, clock, decide_only):
    clock.take()
    t0 = time.perf_counter()
    w.step()
    if decide_only:
        w.ctx.islands_step(float(w.params.dt), w.bodies.linear_velocity, w.bodies.angular_velocity)
    s = clock.take()
    s["step"] = (time.perf_counter() - t0) * 1e3
    return s


def _scene_cases(scene_fn, steps, settle):
    res = {}
    n = int(scene_fn().bodies.count)
    never = np.full(n, -1.0, dtype=np.float32)
    always = np.full(n, 1e3, dtype=np.float32)
    # (a) and (b): awake
    for key, applied in (("a_awake_application_off", False), ("b_awake_application_on", True)):
        with api.Context(device=0) as ctx:
            cfg = dict(thr_lin=never, thr_ang=never)
            w = plugins.DeviceGraphWorld(scene_fn(), plugins.PhysicsPlugins(ctx), ctx, substeps=8, sleeping=cfg if applied else None)
            if not applied:
                ctx.islands_configure(w.bodies.kind, **cfg)
            clock = _Clock(ctx)
            for _ in range(settle):
                _timed_step(w, clock, not applied)
            res[key] = _summary([_timed_step(w, clock, not applied) for _ in range(steps)])
            res[key]["manifolds"] = int(w.stats["manifold_count"])
            res["rows"] = int(w.stats["rows_high_water"])
    # (c) and (d): asleep, and the step of a wake
    with api.Context(device=0) as ctx:
        w = plugins.DeviceGraphWorld(scene_fn(), plugins.PhysicsPlugins(ctx), ctx, substeps=8, sleeping=dict(thr_lin=always, thr_ang=always, time_to_sleep=0.05))
        clock = _Clock(ctx)
        dyn = np.nonzero(w.bodies.kind == api.BODY_DYNAMIC)[0]
        for _ in range(settle + 8):
            _timed_step(w, clock, False)
        asleep = int(w.wake_stats["bodies_asleep"])
        res["c_all_asleep"] = _summary([_timed_step(w, clock, False) for _ in range(steps)])
        res["c_all_asleep"].update(bodies_asleep=asleep, dynamic_bodies=int(dyn.shape[0]), manifolds=int(w.wake_stats["manifold_count"]),
                                   rows_asleep=int(w.wake_stats["rows_asleep"]))
        wakes = []
        for k in range(5):
            w.wake = np.zeros(n, dtype=np.uint8)
            w.wake[dyn[(k * 7919) % dyn.shape[0]]] = 1
            s = _timed_step(w, clock, False)
            s_rows, s_rounds = int(w.wake_stats["rows_woken"]), int(w.wake_stats["colouring_rounds"])
            wakes.append((s, s_rows, s_rounds))
            for _ in range(8):                      # back to sleep
                _timed_step(w, clock, False)
        res["d_wake_step"] = _summary([s for s, _, _ in wakes])
        res["d_wake_step"].update(rows_woken=[r for _, r, _ in wakes], colouring_rounds=[r for _, _, r in wakes])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--settle", type=int, default=8)
    ap.add_argument("--out", default=None, help="directory for sleep_timing.json (default: print only)")
    a = ap.parse_args()
    name, power = _card()
    res = {"card": name, "power_limit": power, "substeps": 8, "dtype": "f32",
           "note": "host clock around calls that end in a stream synchronise; medians over the timed steps; a step includes the host AABB update of the fixture",
           "columns_100x10x100": _scene_cases(lambda: scenes.cube_stack(100, 10, 100, brick=False), a.steps, a.settle),
           "pile_51x40x50": _scene_cases(lambda: scenes.cube_stack(51, 40, 50, brick=True), a.steps, a.settle)}
    print(json.dumps(res))
    if a.out:
        out = Path(a.out)
        out.mkdir(parents=True, exist_ok=True)
        (out / "sleep_timing.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
