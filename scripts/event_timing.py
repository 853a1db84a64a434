"""Cost of the contact pipeline's output to the application on the 100k-cube pile (cube_stack(51, 40, 50), DeviceGraphWorld with a sensor
and an events column set): avn_contacts_step with and without a following avn_contacts_events, avn_contacts_report (all pairs and events
only), and the path they replace (avn_contacts_download_graph of the touching flags + a host diff), with the bytes each brings to the host.
Prints one JSON line; with --out DIR it also writes DIR/event_timing.json.

    python scripts/event_timing.py [--steps 30] [--settle 10] [--out DIR]
"""
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
from avian_b200 import api, plugins, scenes  # noqa: E402


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception as e:  # the numbers stay valid, only the label is missing
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--settle", type=int, default=10)
    ap.add_argument("--out", default=None, help="directory for event_timing.json (default: print only)")
    a = ap.parse_args()
    sc = scenes.cube_stack(51, 40, 50, brick=True)
    n = int(sc.bodies.count)
    rng = np.random.default_rng(0)
    events = rng.random(n) < 0.5
    sensor = rng.random(n) < 0.1
    sensor[0] = False
    with api.Context(device=0) as ctx:
        w = plugins.DeviceGraphWorld(sc, plugins.PhysicsPlugins(ctx), ctx, substeps=6, sensor=sensor, events_enabled=events)
        S = np.dtype(w.scalar).itemsize
        for _ in range(a.settle):
            w.step()
        # the output buffers are allocated once, as a shim would keep them: the timings are those of the C calls
        cap = 1 << 20
        # (the structs hold raw pointers: the dicts own the arrays and must live as long as the structs are used)
        (es, es_cols), (ee, ee_cols) = api.collision_events(cap), api.collision_events(cap)
        rs, rs_cols = api.contact_report(cap, w.scalar)
        t_step, t_step_ev, t_ev, t_rep, t_rep_eo, t_old = [], [], [], [], [], []
        b_ev, b_rep, b_rep_eo, b_old = [], [], [], []
        prev_touch = None
        for i in range(a.steps):
            with_events = i % 2 == 1        # alternate: the step followed by avn_contacts_events, and not
            b = w.bodies
            w.aabb_min, w.aabb_max = w.pipeline.update_aabbs(b, w.params.dt)
            aabbs = w.intervals(w.aabb_min, w.aabb_max)
            ctx.broadphase_upload(aabbs)
            ctx.broadphase_run()
            ctx.solver_prefetch_bodies(b, static_unchanged=True)
            cols = {"shape": w._shape, "dims": w._dims, "position": b.position, "rotation": b.rotation, "aabb_min": w.aabb_min, "aabb_max": w.aabb_max}
            t0 = time.perf_counter()
            w.stats = ctx.contacts_step(w.params.dt, 0.005, cols, b.linear_velocity, b.angular_velocity, True, take_pairs=True, shapes_unchanged=True)
            t1 = time.perf_counter()
            if with_events:
                ctx._check(ctx.lib.avn_contacts_events(ctx.handle, C.byref(es), C.byref(ee)))
                t2 = time.perf_counter()
                t_step_ev.append((t2 - t0) * 1e3); t_ev.append((t2 - t1) * 1e3)
                b_ev.append(17 * (int(es.count) + int(ee.count)))
            else:
                t_step.append((t1 - t0) * 1e3)
            ctx.broadphase_download_order()
            kept = int(aabbs.retained_count)
            oo = aabbs.order_out[:kept]
            w.order = np.ascontiguousarray(aabbs.collider[oo])
            ctx.solver_step_resident(w.params, b, w.joints)
            # the replaced path: the touching flag of every row to the host, diffed against the previous step's
            hw = w.stats["rows_high_water"]
            touch = np.zeros(hw, dtype=np.uint8)
            t0 = time.perf_counter()
            ctx.lib.avn_contacts_download_graph(ctx.handle, hw, None, None, None, touch.ctypes.data, None, None)
            if prev_touch is not None:
                m = min(hw, prev_touch.shape[0])
                np.nonzero(touch[:m] != prev_touch[:m])
            t_old.append((time.perf_counter() - t0) * 1e3)
            b_old.append(hw)
            prev_touch = touch
            t0 = time.perf_counter()
            ctx._check(ctx.lib.avn_contacts_report(ctx.handle, 0, C.byref(rs)))
            t1 = time.perf_counter()
            n_all = int(rs.count)
            ctx._check(ctx.lib.avn_contacts_report(ctx.handle, api.REPORT_EVENTS_ONLY, C.byref(rs)))
            t2 = time.perf_counter()
            t_rep.append((t1 - t0) * 1e3); t_rep_eo.append((t2 - t1) * 1e3)
            per = 5 * 4 + 2 + 6 * S
            b_rep.append(per * n_all); b_rep_eo.append(per * int(rs.count))
        name, power = _card()
        med = lambda x: float(np.median(x)) if x else None
        res = {"scene": "cube_stack(51,40,50) brick, 100k cubes, f32, 6 substeps", "bodies": n, "rows": int(w.stats["rows_high_water"]),
               "card": name, "power_limit": power, "steps_timed": a.steps,
               "contacts_step_ms": med(t_step), "contacts_step_plus_events_ms": med(t_step_ev), "events_ms": med(t_ev),
               "report_all_ms": med(t_rep), "report_events_only_ms": med(t_rep_eo), "download_touching_and_diff_ms": med(t_old),
               "bytes_events": med(b_ev), "bytes_report_all": med(b_rep), "bytes_report_events_only": med(b_rep_eo), "bytes_download_touching": med(b_old),
               "note": "host clock around calls that end in a stream synchronise; medians over the timed steps"}
    print(json.dumps(res))
    if a.out:
        out = Path(a.out)
        out.mkdir(parents=True, exist_ok=True)
        (out / "event_timing.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
