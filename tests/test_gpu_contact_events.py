"""Collision events, sensors, removal of colliders and contact reports of the device-resident contact pipeline (avn_contacts_events /
_set_sensors / _remove_colliders / _report) against the host fixture stepped by the ordinary World, against an independent derivation from graph
snapshots, and against the islands oracle."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests")); sys.path.insert(0, str(ROOT / "oracle"))
from avian_b200 import api, plugins, scenes  # noqa: E402
from islands_oracle import IslandsOracle  # noqa: E402
from test_gpu_graph import _check_graphs, _tumble  # noqa: E402

pytestmark = pytest.mark.gpu
GEN, EVENTS = api.PAIR_GENERATE_CONSTRAINTS, api.PAIR_CONTACT_EVENTS
COLS = [k for k, _ in api.EVENT_COLUMNS]


def _columns(n, seed=11):
    """a random half of the colliders with events, a tenth sensors (never the ground, body 0)"""
    rng = np.random.default_rng(seed)
    events = rng.random(n) < 0.5
    sensor = rng.random(n) < 0.1
    sensor[0] = False
    return sensor, events


def _assert_lists_equal(got, want, what):
    for k in COLS:
        assert np.array_equal(got[k], want[k]), f"{what}: {k}\n{got[k]}\n{want[k]}"


def _assert_step_equal(wa, wb, ctx_b, i):
    for name, g, h in zip(("started", "ended"), wb.events, wa.events):
        _assert_lists_equal(g, h, f"step {i}: {name}")
    _check_graphs(wa, wb, ctx_b, i)            # sensor rows hold no colour: -1 on both sides
    for k in ("position", "rotation", "linear_velocity", "angular_velocity"):
        assert np.array_equal(getattr(wa.bodies, k), getattr(wb.bodies, k)), f"step {i}: {k}"


@pytest.mark.parametrize("scene_fn,steps,substeps,kick", [
    (lambda: scenes.cubes_example(4), 70, 4, True),                   # tumbling cubes: pairs separate, ContactIds are reused
    (lambda: scenes.cube_stack(6, 5, 5, brick=True), 12, 4, False),   # the brick pile
    (lambda: scenes.falling_spheres(400, seed=3, box=(6.0, 4.0, 6.0), scalar=np.float64), 30, 4, False),   # f64 spheres
])
def test_device_events_equal_the_host_fixture(gpu_ctx, scene_fn, steps, substeps, kick):
    sc_a, sc_b = scene_fn(), scene_fn()
    scalar = sc_a.bodies.position.dtype
    sensor, events = _columns(int(sc_a.bodies.count))
    with api.Context(device=0, scalar=scalar) as ctx_a, api.Context(device=0, scalar=scalar) as ctx_b:
        wa = plugins.World(sc_a, plugins.PhysicsPlugins(ctx_a), substeps=substeps, sensor=sensor, events_enabled=events)
        wb = plugins.DeviceGraphWorld(sc_b, plugins.PhysicsPlugins(ctx_b), ctx_b, substeps=substeps, sensor=sensor, events_enabled=events)
        if kick:
            _tumble(wa); _tumble(wb)
        n_start = n_end = n_sensor = 0
        for i in range(steps):
            wa.step(); wb.step()
            _assert_step_equal(wa, wb, ctx_b, i)
            n_start += wb.events[0]["flags"].shape[0]; n_end += wb.events[1]["flags"].shape[0]
            n_sensor += int((wb.events[0]["flags"] & GEN == 0).sum())
        assert n_start > 0 and n_sensor > 0
        if kick:
            assert n_end > 0


def _snapshot_events(prev, now, sensor, events):
    """the started / ended lists from two snapshots of the rows: a row ended when it was touching and is not touching the same pair any more
    (removed rows keep their colliders until the next step reuses the row), and started when it touches a pair it did not touch before"""
    n = now["live"].shape[0]
    col = lambda g, k: np.concatenate([g[k], np.zeros(n - g[k].shape[0], dtype=g[k].dtype)])
    pl, pt, p1, p2 = (col(prev, k) for k in ("live", "touching", "collider1", "collider2"))
    nl, nt, n1, n2 = now["live"].astype(bool), now["touching"].astype(bool), now["collider1"], now["collider2"]
    was = pl.astype(bool) & pt.astype(bool)
    same = nl & (p1 == n1) & (p2 == n2)
    ended, started = np.nonzero(was & ~(same & nt))[0], np.nonzero(nl & nt & ~(was & same))[0]
    def lst(ids, c1, c2):
        c1, c2 = c1[ids], c2[ids]
        flags = np.where(events[c1] | events[c2], EVENTS, 0) | np.where(sensor[c1] | sensor[c2], 0, GEN)
        return c1, c2, flags.astype(np.uint8)
    return lst(started, n1, n2), lst(ended, p1, p2)


def test_events_equal_the_snapshot_diff(gpu_ctx):
    sc = scenes.cubes_example(4)
    sensor, events = _columns(int(sc.bodies.count), seed=3)
    with api.Context(device=0) as ctx:
        w = plugins.DeviceGraphWorld(sc, plugins.PhysicsPlugins(ctx), ctx, substeps=4, sensor=sensor, events_enabled=events)
        _tumble(w)
        prev = {k: np.zeros(0, dtype=d) for k, d in (("collider1", np.uint32), ("collider2", np.uint32), ("live", np.uint8), ("touching", np.uint8))}
        reused = 0
        for i in range(70):
            w.step()
            now = ctx.contacts_download_graph(w.stats["rows_high_water"], 0)
            (s1, s2, sf), (e1, e2, ef) = _snapshot_events(prev, now, sensor, events)
            reused += int((prev["live"].shape[0] > 0) and w.stats["pairs_added"] > 0 and w.stats["rows_live"] < w.stats["rows_high_water"])
            s, e = ctx.contacts_events()
            assert np.array_equal(s["collider1"], s1) and np.array_equal(s["collider2"], s2) and np.array_equal(s["flags"], sf), f"step {i}: started"
            assert np.array_equal(e["collider1"], e1) and np.array_equal(e["collider2"], e2) and np.array_equal(e["flags"], ef), f"step {i}: ended"
            assert all(np.array_equal(a[k], b[k]) for a, b in zip((s, e), ctx.contacts_events()) for k in COLS), "a repeated call differs"
            prev = now
        assert reused > 0


class _RemovalOracle(IslandsOracle):
    """the islands oracle with remove_contact (islands/mod.rs:594-667) callable outside a step, as remove_collider calls it
    (collision/narrow_phase/mod.rs:399-459): a listed contact that is linked to an island leaves it, and the island's constraints_removed
    grows by one -- the same bookkeeping as a 'remove' event of IslandsOracle.step"""

    def remove_contacts(self, contact_ids):
        for cid in contact_ids:
            iid = self.contact_island.pop(int(cid), None)
            if iid is None:
                continue
            isl = self.islands[iid]
            isl.contacts.discard(int(cid))
            isl.removed += 1
            self.contact_bodies.pop(int(cid), None)


def _linked(g):
    """rows linked to an island: touching and in the ConstraintGraph"""
    return {int(e): (int(g["collider1"][e]), int(g["collider2"][e])) for e in np.nonzero(g["live"].astype(bool) & (g["colour"] >= 0))[0]}


def _island_events(prev, now):
    ev = [(e, "remove", *prev[e]) for e in prev if now.get(e) != prev[e]]
    ev += [(e, "add", *now[e]) for e in now if prev.get(e) != now[e]]
    return ev


def test_sensors_and_removals_mid_run_with_islands(gpu_ctx):
    sc_a, sc_b = scenes.cube_stack(5, 4, 4, brick=True), scenes.cube_stack(5, 4, 4, brick=True)
    n = int(sc_a.bodies.count)
    sensor, events = _columns(n, seed=5)
    with api.Context(device=0) as ctx_a, api.Context(device=0) as ctx_b:
        wa = plugins.World(sc_a, plugins.PhysicsPlugins(ctx_a), substeps=4, sensor=sensor, events_enabled=events)
        wb = plugins.DeviceGraphWorld(sc_b, plugins.PhysicsPlugins(ctx_b), ctx_b, substeps=4, sensor=sensor, events_enabled=events)
        kind = wb.bodies.kind
        ctx_b.islands_configure(kind, time_to_sleep=0.3)
        orc = _RemovalOracle(kind, time_to_sleep=0.3, candidate="body")
        prev = {}
        removed_at = {}
        for i in range(60):
            if i in (15, 35):                                  # sensors toggled for a few colliders
                sensor = sensor.copy()
                sensor[[3 + i, 7 + i, 11 + i]] ^= True
                wa.set_sensors(sensor); wb.set_sensors(sensor)
            if i in (20, 40):                                  # colliders despawned / disabled
                gone = [5 + i, 9 + i]
                wa.remove_colliders(gone); wb.remove_colliders(gone)
                removed_at[i] = gone
            if i in (15, 20, 35, 40):
                hw = wb.stats["rows_high_water"]
                g = ctx_b.contacts_download_graph(hw, 0)
                if i in removed_at:                            # the removed colliders' rows are gone at once
                    names = np.isin(g["collider1"], removed_at[i]) | np.isin(g["collider2"], removed_at[i])
                    assert not (g["live"].astype(bool) & names).any(), f"step {i}: a removed collider still has rows"
                now = _linked(g)
                orc.remove_contacts([e for e, pair in prev.items() if now.get(e) != pair])
                prev = now
            wa.step(); wb.step()
            _assert_step_equal(wa, wb, ctx_b, i)
            g = ctx_b.contacts_download_graph(wb.stats["rows_high_water"], 0)
            if i - 1 in removed_at:                            # a removed collider's pairs are found again on the next step
                live = g["live"].astype(bool)
                for c in removed_at[i - 1]:
                    assert (live & ((g["collider1"] == c) | (g["collider2"] == c))).any(), f"step {i}: collider {c} has no pair"
            now = _linked(g)
            ev = _island_events(prev, now)
            prev = now
            dt = float(wb.params.dt)
            got = ctx_b.islands_step(dt, wb.bodies.linear_velocity, wb.bodies.angular_velocity)
            lab, slp = orc.step(ev, wb.bodies.linear_velocity, wb.bodies.angular_velocity, np.float32(dt))
            assert np.array_equal(got["island"], lab), f"step {i}: island labels"
            assert np.array_equal(got["sleep_timer"], orc.timer), f"step {i}: sleep timers"
            assert np.array_equal(got["sleeping"], slp), f"step {i}: Sleeping flags"


def _host_report(ctx, w, rep, capacity):
    """total and max impulse from the downloaded rows (point count from the report), in the column type, slot order"""
    S = w.scalar.type
    g = ctx.contacts_download_graph(w.stats["rows_high_water"], 0)
    _, _, ni = ctx.contacts_download_impulses(capacity)
    tot, mx = [], []
    for e, cnt in zip(rep["contact_id"], rep["point_count"]):
        t, m = S(0), S(0)
        for k in range(int(cnt)):
            v = ni[e, k] if g["colour"][e] >= 0 else S(0)
            t = S(t + v)
            m = v if v > m else m
        tot.append(t); mx.append(m)
    return np.array(tot, dtype=w.scalar), np.array(mx, dtype=w.scalar), g


def test_download_impulses_writes_at_most_capacity_rows(gpu_ctx):
    """avn_contacts_download_impulses copies min(capacity, rows) rows: a buffer sized below the store is filled to its capacity and not beyond"""
    with api.Context(device=0) as ctx:
        w = plugins.DeviceGraphWorld(scenes.cube_stack(4, 3, 4, brick=True), plugins.PhysicsPlugins(ctx), ctx, substeps=4)
        for _ in range(3):
            w.step()
        hw = int(w.stats["rows_high_water"])
        n = hw // 2
        assert n > 0
        full = ctx.contacts_download_impulses(hw)
        bufs = [np.full((hw,) + shape, np.float32(-7.5), dtype=np.float32) for shape in ((4,), (4, 2), (4,))]
        ctx._check(ctx.lib.avn_contacts_download_impulses(ctx.handle, n, *(b.ctypes.data for b in bufs)))
        for b, f in zip(bufs, full):
            assert np.array_equal(b[:n], f[:n]), "the first rows differ from a download at full capacity"
            assert (b[n:] == np.float32(-7.5)).all(), "rows past the capacity were written"
        assert any((f[:n] != 0).any() for f in full), "the scene was meant to leave impulses in the first rows"


@pytest.mark.parametrize("scene_fn", [lambda: scenes.cube_stack(6, 5, 5, brick=True),
                                      lambda: scenes.falling_spheres(400, seed=3, box=(6.0, 4.0, 6.0), scalar=np.float64)])
def test_report_equals_a_host_computation(gpu_ctx, scene_fn):
    sc_a, sc_b = scene_fn(), scene_fn()
    scalar = sc_a.bodies.position.dtype
    sensor, events = _columns(int(sc_a.bodies.count), seed=7)
    with api.Context(device=0, scalar=scalar) as ctx_a, api.Context(device=0, scalar=scalar) as ctx_b:
        wa = plugins.World(sc_a, plugins.PhysicsPlugins(ctx_a), substeps=4, sensor=sensor, events_enabled=events)
        wb = plugins.DeviceGraphWorld(sc_b, plugins.PhysicsPlugins(ctx_b), ctx_b, substeps=4, sensor=sensor, events_enabled=events)
        sensors_seen = 0
        for i in range(20):
            wa.step(); wb.step()
            assert wb.stats["rows_high_water"] < 16384
            rep, eo, host = wb.report(), wb.report(events_only=True), wa.report()
            assert (np.diff(rep["contact_id"].astype(np.int64)) > 0).all()
            for k in ("contact_id", "collider1", "collider2", "body1", "body2", "flags", "point_count"):
                assert np.array_equal(rep[k], host[k]), f"step {i}: {k}"
            for k in ("normal", "max_penetration"):
                assert np.array_equal(rep[k].view(np.uint8), host[k].view(np.uint8)), f"step {i}: {k}"
            tot, mx, g = _host_report(ctx_b, wb, rep, wb.stats["rows_high_water"])
            assert np.array_equal(rep["total_normal_impulse"].view(np.uint8), tot.view(np.uint8)), f"step {i}: total"
            assert np.array_equal(rep["max_normal_impulse"].view(np.uint8), mx.view(np.uint8)), f"step {i}: max"
            touching = np.nonzero(g["live"].astype(bool) & g["touching"].astype(bool))[0]
            assert np.array_equal(rep["contact_id"], touching)
            sel = (rep["flags"] & EVENTS) != 0
            assert np.array_equal(eo["contact_id"], rep["contact_id"][sel])
            for k in eo:
                assert np.array_equal(eo[k].view(np.uint8), rep[k][sel].view(np.uint8)), f"step {i}: events_only {k}"
            sens = (rep["flags"] & GEN) == 0
            assert (rep["total_normal_impulse"][sens] == 0).all() and (rep["max_normal_impulse"][sens] == 0).all()
            sensors_seen += int(sens.sum())
            assert (rep["total_normal_impulse"][~sens] > 0).any()
        assert sensors_seen > 0


def test_refusals(gpu_ctx):
    sc = scenes.cube_stack(4, 3, 4, brick=True)
    n = int(sc.bodies.count)
    with api.Context(device=0) as ctx:
        with pytest.raises(api.AvianError) as e:
            ctx.contacts_set_sensors(np.zeros(n, dtype=bool))
        assert e.value.status == api.ERR_UNSUPPORTED                     # before avn_contacts_configure
        w = plugins.DeviceGraphWorld(sc, plugins.PhysicsPlugins(ctx), ctx, substeps=4)
        for call in (lambda: ctx.contacts_events(), lambda: ctx.contacts_report(), lambda: ctx.contacts_remove_colliders([1])):
            with pytest.raises(api.AvianError) as e:
                call()
            assert e.value.status == api.ERR_UNSUPPORTED                 # before the first avn_contacts_step
        ctx.contacts_set_sensors(np.zeros(n, dtype=bool))                # (only stores the column)
        w.step()
        with pytest.raises(api.AvianError) as e:
            ctx.contacts_events(capacity=1)
        assert e.value.status == api.ERR_CAPACITY and e.value.required[0] == w.stats["started_touching"] > 1
        s, _ = ctx.contacts_events(capacity=e.value.required[0])
        assert s["collider1"].shape[0] == w.stats["started_touching"]
        with pytest.raises(api.AvianError) as e:
            ctx.contacts_report(capacity=1)
        assert e.value.status == api.ERR_CAPACITY and e.value.required > 1
        assert ctx.contacts_report(capacity=e.value.required)["contact_id"].shape[0] == e.value.required
        before = ctx.contacts_download_graph(w.stats["rows_high_water"], 0)
        for call in (lambda: ctx.contacts_remove_colliders([1, n]), lambda: ctx.contacts_set_sensors(np.ones(n + 1, dtype=bool))):
            with pytest.raises(api.AvianError) as e:
                call()
            assert e.value.status == api.ERR_INVALID_ARGUMENT
        after = ctx.contacts_download_graph(w.stats["rows_high_water"], 0)
        assert all(np.array_equal(before[k], after[k]) for k in before), "a refused call removed something"
