"""Applied sleeping on the device (avn_islands_apply / avn_islands_wake / avn_islands_step; plugins.DeviceGraphWorld(sleeping=...)) beside the
reference world of tests/sleeping_world.py, which runs the same solver on the lists of the host fixture.  Every step: the same ContactIds, the
same live / touching / asleep flag and colour per row, the overflow colour in the same order, the same island labels, timers and Sleeping
flags, the same collision events, and the bodies bit for bit."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
from avian_b200 import api, plugins, scenes  # noqa: E402
from sleeping_world import SleepingWorld, column_scene  # noqa: E402
from test_gpu_graph import _plate_on_cubes  # noqa: E402

pytestmark = pytest.mark.gpu
COLS = ("position", "rotation", "linear_velocity", "angular_velocity")


def _kick(w, seed, lin=1.5, ang=2.0):
    rng = np.random.default_rng(seed)
    dyn = w.bodies.kind == api.BODY_DYNAMIC
    w.bodies.linear_velocity[dyn] = rng.normal(0, lin, size=(int(dyn.sum()), 3)).astype(w.scalar)
    w.bodies.angular_velocity[dyn] = rng.normal(0, ang, size=(int(dyn.sum()), 3)).astype(w.scalar)


def _check(wa, wb, ctx_b, step):
    g = wa.graph()
    st, wk = wb.stats, wb.wake_stats
    hw = st["rows_high_water"]
    assert st["rows_live"] == g["ids"].shape[0], f"step {step}: live pairs"
    d = ctx_b.contacts_download_graph(hw, wk["manifold_count"])
    sl = ctx_b.contacts_download_sleeping(hw, wb.n)
    live = np.zeros(hw, dtype=bool); live[g["ids"]] = True
    assert np.array_equal(d["live"].astype(bool), live), f"step {step}: ContactIds in use"
    assert np.array_equal(d["collider1"][g["ids"]], g["c1"]) and np.array_equal(d["collider2"][g["ids"]], g["c2"]), f"step {step}: a pair sits in another row"
    touching = np.zeros(hw, dtype=bool); touching[g["sid"]] = g["touching"]
    asleep = np.zeros(hw, dtype=bool); asleep[g["sid"]] = g["asleep"]
    assert np.array_equal(d["touching"].astype(bool), touching), f"step {step}: touching"
    assert np.array_equal(sl["row_asleep"].astype(bool), asleep), f"step {step}: asleep rows {np.nonzero(sl['row_asleep'].astype(bool) != asleep)[0][:10]}"
    assert np.array_equal(sl["body_asleep"].astype(bool), wa.body_asleep), f"step {step}: asleep bodies"
    for k in ("island", "sleeping_flags", "sleep_timer"):
        assert np.array_equal(getattr(wa, k), getattr(wb, k)), f"step {step}: {k}"
    for k in COLS:
        assert np.array_equal(getattr(wa.bodies, k), getattr(wb.bodies, k)), f"step {step}: {k}"
    return d, sl


def _check_solved_graph(wa_graph, wb, d, step):
    """the colour-major list the solver of this step read (after the wake half, before the sleeps of the island step)"""
    co, edge = wa_graph["color_offsets"], wa_graph["edge"]
    assert np.array_equal(wb.wake_stats["color_offsets"], co), f"step {step}: colour offsets\n{wb.wake_stats['color_offsets']}\n{co}"
    for c in range(api.GRAPH_COLOR_COUNT):
        mine, theirs = d[co[c]:co[c + 1]], edge[co[c]:co[c + 1]]
        assert np.array_equal(mine, theirs if c == api.COLOR_OVERFLOW else np.sort(theirs)), f"step {step}: colour {c}"


class _Pair:
    """the two worlds stepped side by side; the list the solver reads is taken between the narrow phase and the solve"""
    def __init__(self, scene_fn, ctx_a, ctx_b, sleeping, substeps=4, **kw):
        self.wa = SleepingWorld(scene_fn(), plugins.PhysicsPlugins(ctx_a), sleeping, substeps=substeps, **kw)
        self.wb = plugins.DeviceGraphWorld(scene_fn(), plugins.PhysicsPlugins(ctx_b), ctx_b, sleeping=sleeping, substeps=substeps, **kw)
        self.ctx_b = ctx_b
        self.step_index = 0
        self.slept = self.woken = 0

    def step(self, wake=None, late_wake=None):
        wa, wb = self.wa, self.wb
        if wake is not None:
            wa.wake, wb.wake = wake.copy(), wake.copy()
        if late_wake is not None:
            wa.late_wake, wb.late_wake = late_wake.copy(), late_wake.copy()
        wa.broad_phase(); wa.narrow_phase()
        solved = wa.graph()
        wa.solve(); wa.step_index += 1
        wb.step()
        # the device's list as the solver read it is gone once the island step has put rows to sleep: compare it when nothing fell asleep
        d, sl = _check(wa, wb, self.ctx_b, self.step_index)
        if wb.islands["islands_put_to_sleep"] == 0:
            _check_solved_graph(solved, wb, d["edge"], self.step_index)
        end = wa.graph()
        colour = np.full(wb.stats["rows_high_water"], -1, dtype=np.int8)
        for c in range(api.GRAPH_COLOR_COUNT):
            colour[end["edge"][end["color_offsets"][c]:end["color_offsets"][c + 1]]] = c
        assert np.array_equal(d["colour"], colour), f"step {self.step_index}: colours differ for rows {np.nonzero(d['colour'] != colour)[0][:10]}"
        if wa.events is not None and wb.events is not None:
            for x, y in zip(wa.events, wb.events):
                for k in x:
                    assert np.array_equal(x[k], y[k]), f"step {self.step_index}: events {k}"
        self.slept += wb.islands["islands_put_to_sleep"]; self.woken += wb.islands["islands_woken"]
        self.step_index += 1


@pytest.mark.parametrize("scene_fn,steps,kick,sleeping,resting", [
    (lambda: scenes.cubes_example(3), 150, 7, dict(time_to_sleep=0.25, thr_lin=np.full(28, 0.5, np.float32), thr_ang=np.full(28, 0.5, np.float32)), True),                                      # tumbling cubes: sleeps, wakes, deferred splits
    (lambda: _plate_on_cubes(5), 60, 0, dict(time_to_sleep=0.2, thr_lin=np.full(27, 0.8, np.float32), thr_ang=np.full(27, 0.8, np.float32)), True),   # overflow colour
    (lambda: scenes.ragdoll_field(6, pitch=2.5, drop_height=0.3), 120, 0, dict(time_to_sleep=0.2, thr_lin=np.full(6 * 16 + 1, 4.0, np.float32),
                                                                               thr_ang=np.full(6 * 16 + 1, 4.0, np.float32)), False),        # joints
    (lambda: scenes.cube_stack(3, 3, 3, brick=False, scalar=np.float64), 80, 0, dict(time_to_sleep=0.2), True),                                  # f64 columns
])
def test_sleeping_world_on_the_device_equals_the_reference_world(gpu_ctx, scene_fn, steps, kick, sleeping, resting):
    """resting: the scene comes to rest in contact within the run, so rows must have gone to sleep and come back"""
    sc = scene_fn()
    n = int(sc.bodies.count)
    sleeping = {k: (v if np.isscalar(v) or v.shape[0] == n else np.full(n, v[0], v.dtype)) for k, v in sleeping.items()}
    scalar = sc.bodies.position.dtype
    with api.Context(device=0, scalar=scalar) as ctx_a, api.Context(device=0, scalar=scalar) as ctx_b:
        p = _Pair(scene_fn, ctx_a, ctx_b, sleeping)
        if kick:
            _kick(p.wa, kick); _kick(p.wb, kick)
        dyn = np.nonzero(sc.bodies.kind == api.BODY_DYNAMIC)[0]
        pending = [int(dyn[0]), int(dyn[-1])]
        for i in range(steps):
            wake = None
            if pending and i < steps - 5 and p.wb.sleeping_flags[pending[0]]:   # the application touches a sleeping body: its island wakes, its rows are pushed again
                wake = np.zeros(n, dtype=np.uint8); wake[pending.pop(0)] = 1
            p.step(wake)
        assert p.slept > 0, "nothing went to sleep: the scene or the thresholds do not exercise the path"
        if resting:
            assert p.woken > 0, "nothing woke"
            assert p.wa.rows_slept > 0 and p.wa.rows_woken > 0
        print(f"islands put to sleep {p.slept}, woken {p.woken}; rows put to sleep {p.wa.rows_slept}, woken {p.wa.rows_woken}")


def test_sixteen_columns_fall_asleep_completely_and_a_projectile_wakes_one(gpu_ctx):
    def scene():
        sc = scenes.cube_stack(4, 3, 4, brick=False)
        return sc
    with api.Context(device=0) as ctx_a, api.Context(device=0) as ctx_b:
        p = _Pair(scene, ctx_a, ctx_b, dict(time_to_sleep=0.3), events_enabled=np.ones(scene().bodies.count, dtype=bool))
        n = p.wb.n
        dyn = p.wb.bodies.kind == api.BODY_DYNAMIC
        for i in range(120):
            p.step()
            if p.wb.sleeping_flags[dyn].all():
                break
        assert p.wb.sleeping_flags[dyn].all(), "the columns never all slept"
        p.step()
        wk = p.wb.wake_stats
        assert wk["manifold_count"] == 0 and wk["bodies_asleep"] == int(dyn.sum())
        touching = ctx_b.contacts_download_graph(p.wb.stats["rows_high_water"], 0)["touching"].astype(bool)
        assert wk["rows_asleep"] == int(touching.sum()) > 0                  # every touching row sleeps: the narrow phase has nothing to update
        assert p.wb.stats["started_touching"] == 0 and p.wb.stats["stopped_touching"] == 0 and p.wb.stats["colouring_rounds"] == 0
        rep_a, rep_b = p.wa.report(), p.wb.report()                          # asleep rows are reported with the impulses of their last solve
        assert rep_b["contact_id"].shape[0] == wk["rows_asleep"] and (rep_b["total_normal_impulse"] > 0).all()
        for k in rep_a:
            assert np.array_equal(rep_a[k], rep_b[k]), k
        # a projectile: the topmost cube of one column is thrown at its neighbour column
        top = int(np.argmax(np.where(dyn, p.wb.bodies.position[:, 1], -1e9)))
        wake = np.zeros(n, dtype=np.uint8); wake[top] = 1
        for w in (p.wa, p.wb):
            w.bodies.linear_velocity[top] = (6.0, 1.0, 0.0)
        woken0 = p.woken
        for i in range(40):
            p.step(wake if i == 0 else None)
        assert p.woken - woken0 >= 1, "the projectile woke nothing"
        assert p.wb.wake_stats["bodies_asleep"] < int(dyn.sum())


def test_removing_and_sensoring_sleeping_colliders(gpu_ctx):
    scene = lambda: scenes.cube_stack(3, 3, 3, brick=False)
    with api.Context(device=0) as ctx_a, api.Context(device=0) as ctx_b:
        p = _Pair(scene, ctx_a, ctx_b, dict(time_to_sleep=0.2), events_enabled=np.ones(scene().bodies.count, dtype=bool))
        n = p.wb.n
        dyn = np.nonzero(p.wb.bodies.kind == api.BODY_DYNAMIC)[0]
        for _ in range(60):
            p.step()
        assert p.wb.sleeping_flags[dyn].all()
        gone = [int(dyn[0])]
        p.wa.remove_colliders(gone); p.wb.remove_colliders(gone)
        wake = np.zeros(n, dtype=np.uint8); wake[gone] = 1           # waking the island stays with the caller
        p.step(wake)
        sensor = np.zeros(n, dtype=bool); sensor[int(dyn[-1])] = True
        p.wa.set_sensors(sensor); p.wb.set_sensors(sensor)
        wake = np.zeros(n, dtype=np.uint8); wake[int(dyn[-1])] = 1
        p.step(wake)
        for _ in range(40):
            p.step()


def test_application_off_reproduces_the_decisions_only_pipeline(gpu_ctx):
    """the opt-in claim: a context on which avn_islands_apply is never called, and one on which it was turned on and off again before the first
    step, compute what the library computed before: same graph, same bodies, same AvnIslandsStep"""
    scene = lambda: scenes.cube_stack(4, 3, 4, brick=False)
    with api.Context(device=0) as ctx_a, api.Context(device=0) as ctx_b:
        wa = plugins.DeviceGraphWorld(scene(), plugins.PhysicsPlugins(ctx_a), ctx_a, substeps=4)
        wb = plugins.DeviceGraphWorld(scene(), plugins.PhysicsPlugins(ctx_b), ctx_b, substeps=4)
        for ctx, w in ((ctx_a, wa), (ctx_b, wb)):
            ctx.islands_configure(w.bodies.kind, time_to_sleep=0.3)
        ctx_b.islands_apply(True); ctx_b.islands_apply(False)
        with pytest.raises(api.AvianError) as e:
            ctx_b.islands_wake()
        assert e.value.status == api.ERR_UNSUPPORTED
        slept = 0
        for i in range(70):
            wa.step(); wb.step()
            ga = ctx_a.islands_step(float(wa.params.dt), wa.bodies.linear_velocity, wa.bodies.angular_velocity)
            gb = ctx_b.islands_step(float(wb.params.dt), wb.bodies.linear_velocity, wb.bodies.angular_velocity)
            for k in ga:
                assert np.array_equal(ga[k], gb[k]), f"step {i}: {k}"
            slept += ga["islands_put_to_sleep"]
            for k in COLS:
                assert np.array_equal(getattr(wa.bodies, k), getattr(wb.bodies, k)), f"step {i}: {k}"
            assert wa.stats["manifold_count"] == wb.stats["manifold_count"] > 0          # sleeping islands stay in the step: nothing is applied
            assert not ctx_b.contacts_download_sleeping(wb.stats["rows_high_water"], wb.n)["row_asleep"].any()
        assert slept > 0


def test_refused_combinations(gpu_ctx):
    sc = scenes.cube_stack(3, 2, 3, brick=False)
    with api.Context(device=0) as ctx:
        w = plugins.DeviceGraphWorld(sc, plugins.PhysicsPlugins(ctx), ctx, substeps=2)
        with pytest.raises(api.AvianError) as e:                     # before avn_islands_configure
            ctx.islands_apply(True)
        assert e.value.status == api.ERR_UNSUPPORTED
        dyn = np.nonzero(w.bodies.kind == api.BODY_DYNAMIC)[0]
        ctx.islands_configure(w.bodies.kind)
        ctx.ccd_configure(body=dyn[:1].astype(np.int32), collider=dyn[:1].astype(np.uint32))
        with pytest.raises(api.AvianError) as e:                     # swept CCD holds a body list
            ctx.islands_apply(True)
        assert e.value.status == api.ERR_UNSUPPORTED
        ctx.ccd_configure(None)
        ctx.islands_apply(True)
        with pytest.raises(api.AvianError) as e:                     # and the other way round
            ctx.ccd_configure(body=dyn[:1].astype(np.int32), collider=dyn[:1].astype(np.uint32))
        assert e.value.status == api.ERR_UNSUPPORTED
        with pytest.raises(api.AvianError) as e:                     # avn_islands_wake skipped: the solver stage refuses the upload
            w.step()
        assert e.value.status == api.ERR_INVALID_ARGUMENT and "avn_islands_wake" in str(e.value)
        ctx.islands_wake()
        with pytest.raises(api.AvianError) as e:                     # once per contact step
            ctx.islands_wake()
        assert e.value.status == api.ERR_INVALID_ARGUMENT
        ctx.solver_step_resident(w.params, w.bodies, w.joints)
        with pytest.raises(api.AvianError) as e:                     # not in the middle of a step
            ctx.islands_apply(False)
        assert e.value.status == api.ERR_INVALID_ARGUMENT
        ctx.islands_step(float(w.params.dt), w.bodies.linear_velocity, w.bodies.angular_velocity)
        for reconfigure in (lambda: ctx.contacts_configure(w.bodies.kind, w.n, sc.friction, sc.restitution), lambda: ctx.islands_configure(w.bodies.kind)):
            with pytest.raises(api.AvianError) as e:                 # the applied state belongs to the configured bodies and rows
                reconfigure()
            assert e.value.status == api.ERR_UNSUPPORTED and "avn_islands_apply" in str(e.value)
        ctx.islands_apply(False)
        ctx.contacts_configure(w.bodies.kind, w.n, sc.friction, sc.restitution)
        ctx.islands_configure(w.bodies.kind)
        ctx.islands_apply(True)


def _greedy_colours(ids, b1, b2, kind):
    """ConstraintGraph::push_manifold for these rows in this order, from an empty graph (constraint_graph.rs:163-238)"""
    bits = [0] * int(kind.shape[0])
    static = (kind == api.BODY_STATIC).tolist()
    dyn_mask, st_mask = (1 << api.DYNAMIC_COLOR_COUNT) - 1, ((1 << api.COLOR_OVERFLOW) - 1) & ~1
    out = {}
    for e, x, y in zip(ids.tolist(), b1.tolist(), b2.tolist()):
        c = api.COLOR_OVERFLOW
        if not static[x] and not static[y]:
            free = ~(bits[x] | bits[y]) & dyn_mask
            if free:
                c = (free & -free).bit_length() - 1
                bits[x] |= 1 << c; bits[y] |= 1 << c
        elif not static[x] or not static[y]:
            b = y if static[x] else x
            free = ~bits[b] & st_mask
            if free:
                c = free.bit_length() - 1
                bits[b] |= 1 << c
        out[e] = c
    return out


def _assert_all_awake_and_greedy(ctx, w, manifold_count):
    hw = w.stats["rows_high_water"]
    g = ctx.contacts_download_graph(hw, 0)
    sl = ctx.contacts_download_sleeping(hw, w.n)
    assert not sl["row_asleep"].any() and not sl["body_asleep"].any()
    rows = np.nonzero(g["live"].astype(bool) & g["touching"].astype(bool))[0]
    assert rows.shape[0] == manifold_count
    want = _greedy_colours(rows, g["collider1"][rows], g["collider2"][rows], w.bodies.kind)     # (colliders are the bodies in this fixture)
    got = g["colour"][rows]
    bad = [int(e) for e, c in zip(rows, got) if want[int(e)] != int(c)]
    assert not bad, f"{len(bad)} rows hold another colour than the sequential greedy push in ascending ContactId gives, e.g. {bad[:5]}"
    assert (g["colour"][~(g["live"].astype(bool) & g["touching"].astype(bool))] == -1).all()


def test_a_pile_above_262144_rows_sleeps_and_wakes(gpu_ctx):
    """the 100k brick pile with generous thresholds: the sleep list's and the wake list's radix passes run their scan path (more than 262 144
    rows).  Asleep: no manifold, every touching row asleep.  Woken as one island: every touching row is pushed again, and the colours are exactly
    the sequential greedy result for ascending ContactId."""
    sc = scenes.cube_stack(51, 40, 50, brick=True)
    n = int(sc.bodies.count)
    thr = np.full(n, 1e3, dtype=np.float32)
    with api.Context(device=0) as ctx:
        w = plugins.DeviceGraphWorld(sc, plugins.PhysicsPlugins(ctx), ctx, substeps=2, sleeping=dict(time_to_sleep=0.05, thr_lin=thr, thr_ang=thr))
        dyn = np.nonzero(w.bodies.kind == api.BODY_DYNAMIC)[0]
        w.step()
        awake_manifolds = w.stats["manifold_count"]
        assert w.stats["rows_high_water"] > 262144 and awake_manifolds > 262144
        for _ in range(6):
            w.step()
            if w.sleeping_flags[dyn].all():
                break
        assert w.sleeping_flags[dyn].all()
        frozen = w.bodies.position.copy()
        w.step()
        wk = w.wake_stats
        touching = ctx.contacts_download_graph(w.stats["rows_high_water"], 0)["touching"].astype(bool)
        assert wk["manifold_count"] == 0 and wk["bodies_asleep"] == dyn.shape[0] and wk["rows_asleep"] == int(touching.sum()) > 262144
        assert np.array_equal(ctx.contacts_download_sleeping(w.stats["rows_high_water"], n)["row_asleep"].astype(bool), touching)
        assert np.array_equal(w.bodies.position, frozen)
        w.wake = np.zeros(n, dtype=np.uint8); w.wake[dyn[12345]] = 1
        w.step()
        wk = w.wake_stats
        assert wk["islands_woken"] == 1 and wk["rows_woken"] == int(touching.sum()) and wk["bodies_asleep"] == 0
        assert wk["color_offsets"][-1] == wk["manifold_count"] == wk["rows_woken"]
        if w.islands["islands_put_to_sleep"] == 0:          # (the island step of the same call may already have put it back to sleep)
            _assert_all_awake_and_greedy(ctx, w, wk["manifold_count"])
        assert not np.array_equal(w.bodies.position, frozen), "the woken pile was not solved"


def test_turning_application_off_wakes_everything(gpu_ctx):
    sc = scenes.cube_stack(4, 3, 4, brick=False)
    with api.Context(device=0) as ctx:
        w = plugins.DeviceGraphWorld(sc, plugins.PhysicsPlugins(ctx), ctx, substeps=4, sleeping=dict(time_to_sleep=0.3))
        dyn = np.nonzero(w.bodies.kind == api.BODY_DYNAMIC)[0]
        for _ in range(60):
            w.step()
        assert w.sleeping_flags[dyn].all() and w.wake_stats["manifold_count"] == 0
        touching = int(ctx.contacts_download_graph(w.stats["rows_high_water"], 0)["touching"].sum())
        ctx.islands_apply(False)
        _assert_all_awake_and_greedy(ctx, w, touching)
        w.sleeping = None                                   # the plain sequence again: every manifold is solved, islands decide only
        before = w.bodies.position.copy()
        w.step()
        assert w.stats["manifold_count"] == touching
        got = ctx.islands_step(float(w.params.dt), w.bodies.linear_velocity, w.bodies.angular_velocity)
        assert not got["sleeping"].any() and (got["sleep_timer"][dyn] <= np.float32(w.params.dt)).all()      # WakeIslands: timers restarted
        assert np.isfinite(w.bodies.position).all() and np.abs(w.bodies.position - before).max() < 1e-2


def test_a_late_wake_in_the_island_step_while_another_island_falls_asleep(gpu_ctx):
    """the `wake` column of avn_islands_step with application on: the island is awake from the next step on, and the same pass puts the islands
    to sleep that were decided in that step (wakes, then sleeps, each with its own list)"""
    scene = lambda: scenes.cube_stack(3, 3, 3, brick=False)
    with api.Context(device=0) as ctx_a, api.Context(device=0) as ctx_b:
        p = _Pair(scene, ctx_a, ctx_b, dict(time_to_sleep=0.2))
        n = p.wb.n
        dyn = np.nonzero(p.wb.bodies.kind == api.BODY_DYNAMIC)[0]
        mark = lambda b: np.bincount([int(b)], minlength=n).astype(np.uint8)
        for _ in range(60):
            p.step()
        assert p.wb.sleeping_flags[dyn].all()
        first, other = dyn[0], [b for b in dyn if p.wb.island[b] != p.wb.island[dyn[0]]][0]
        p.step(wake=mark(first))                            # how long does a woken column take to sleep again?
        k = 0
        while not p.wb.sleeping_flags[first]:
            p.step(); k += 1
            assert k < 60
        p.step(wake=mark(first))
        for _ in range(k - 1):
            p.step()
        assert not p.wb.sleeping_flags[first] and p.wb.sleeping_flags[other]
        p.step(late_wake=mark(other))                       # `first` falls asleep in the step whose island half wakes `other`
        assert p.wb.islands["islands_put_to_sleep"] >= 1 and p.wb.islands["islands_woken"] >= 1
        assert p.wb.sleeping_flags[first] and not p.wb.sleeping_flags[other]
        sl = ctx_b.contacts_download_sleeping(0, n)["body_asleep"]
        assert sl[first] and not sl[other]
        for _ in range(20):
            p.step()


def test_the_sensor_pair_quirk_on_the_device(gpu_ctx):
    scene = lambda: column_scene(extra=[0.2, 3.2, 0.0], extra_kind=api.BODY_KINEMATIC)
    sensor = np.array([0, 0, 0, 0, 1], dtype=bool)
    cfg = dict(time_to_sleep=0.2, disabled=np.array([0, 0, 0, 0, 1], dtype=np.uint8))
    with api.Context(device=0) as ctx_a, api.Context(device=0) as ctx_b:
        p = _Pair(scene, ctx_a, ctx_b, cfg, sensor=sensor)
        for _ in range(40):
            p.step()
        assert p.wb.sleeping_flags[1:4].all() and not p.wb.sleeping_flags[4]
        for w in (p.wa, p.wb):
            w.bodies.linear_velocity[4] = (5.0, 0.0, 0.0)
        for _ in range(30):
            p.step()
        g = ctx_b.contacts_download_graph(p.wb.stats["rows_high_water"], 0)
        row = np.nonzero(g["live"].astype(bool) & ((g["collider1"] == 4) | (g["collider2"] == 4)))[0]
        sl = ctx_b.contacts_download_sleeping(p.wb.stats["rows_high_water"], 5)
        assert row.shape[0] == 1 and g["touching"][row[0]] and sl["row_asleep"][row[0]] and p.wb.bodies.position[4, 0] > 2.0
        p.step(wake=np.array([0, 1, 0, 0, 0], dtype=np.uint8))
        p.step()
        assert len(p.wb.events[1]["collider1"]) == 1       # the CollisionEnd of the pair, once it is updated again
