"""Applied sleeping in the reference world alone (tests/sleeping_world.py over the CPU oracle's solver and broad phase): small scenes whose
outcome can be checked by hand.  The device path is compared with this world step by step in tests/test_gpu_sleeping.py."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests")); sys.path.insert(0, str(ROOT / "oracle"))
from avian_b200 import api, scenes  # noqa: E402
from islands_oracle import IslandsOracle  # noqa: E402
from oracle_lib import oracle_plugins  # noqa: E402
from sleeping_world import SleepingWorld, TwoHalfIslands, column_scene as _column  # noqa: E402

COLS = ("position", "rotation", "linear_velocity", "angular_velocity")


def _world(scene, **kw):
    return SleepingWorld(scene, oracle_plugins(), dict(time_to_sleep=0.2), substeps=4, **kw)


def _snapshot(w, rows):
    return [getattr(w.bodies, k)[rows].copy() for k in COLS]


def _no_body_twice_in_a_colour(w):
    g = w.graph()
    pair = {int(e): (int(a), int(b)) for e, a, b in zip(g["ids"], g["c1"], g["c2"])}
    for c in range(api.GRAPH_COLOR_COUNT - 1):
        seen = []
        for e in g["edge"][g["color_offsets"][c]:g["color_offsets"][c + 1]]:
            seen += [b for b in pair[int(e)] if w.bodies.kind[b] != api.BODY_STATIC]
        assert len(seen) == len(set(seen)), f"colour {c} holds a body twice"


def test_the_two_halves_equal_one_step():
    rng = np.random.default_rng(3)
    kind = np.zeros(12, dtype=np.uint8); kind[0] = api.BODY_STATIC
    a, b = IslandsOracle(kind, time_to_sleep=0.05, candidate="body"), TwoHalfIslands(kind, time_to_sleep=0.05, candidate="body")
    live = {}
    for step in range(120):
        ev = []
        for cid in list(live):
            if rng.random() < 0.1:
                ev.append((cid, "remove", *live.pop(cid)))
        for _ in range(2):
            cid = int(rng.integers(0, 40))
            if cid not in live and all(e[0] != cid for e in ev) and rng.random() < 0.5:
                live[cid] = tuple(int(x) for x in rng.choice(12, 2, replace=False))
                ev.append((cid, "add", *live[cid]))
        v = (rng.random((12, 3)) * (0.3 if step % 40 < 30 else 0.01)).astype(np.float32)
        wake = (rng.random(12) < 0.02).astype(np.uint8) if step % 7 == 0 else None
        la, sa = a.step(ev, v, v, np.float32(1 / 60), wake=wake)
        b.narrow_phase_events(ev, wake)
        lb, sb = b.sleeping_half(v, v, np.float32(1 / 60))
        assert np.array_equal(la, lb) and np.array_equal(sa, sb) and np.array_equal(a.timer, b.timer), step


def test_a_column_sleeps_and_stays_exactly_where_it_is():
    w = _world(_column())
    slept_at = None
    for i in range(80):
        w.step()
        if slept_at is None and w.sleeping_flags[1:].all():
            slept_at = i
            frozen = _snapshot(w, slice(1, 4))
            g0 = w.graph()
            man0 = w.pipeline.report()
            break
    assert slept_at is not None, "the column never slept"
    assert slept_at >= int(0.2 * 60) - 1, "asleep before TimeToSleep"
    assert w.rows_slept == 3 and g0["asleep"].all() and g0["touching"].all() and g0["edge"].shape[0] == 0     # ConstraintGraph empty, pairs kept
    for _ in range(30):
        w.step()
        for a, b in zip(frozen, _snapshot(w, slice(1, 4))):
            assert np.array_equal(a, b), "a sleeping body changed"
        g = w.graph()
        assert np.array_equal(g["ids"], g0["ids"]) and g["asleep"].all() and g["edge"].shape[0] == 0
        rep = w.pipeline.report()
        for k in ("contact_id", "total_normal_impulse", "max_penetration", "normal"):      # manifolds and impulses as they were, still reported
            assert np.array_equal(rep[k], man0[k]), k
    assert (man0["total_normal_impulse"] > 0).all()


def test_a_dropped_cube_wakes_the_column_before_that_steps_solve():
    w = _world(_column(extra=[0, 9.0, 0]))
    w.orc.disabled[4] = True            # the falling cube itself never sleeps (SleepingDisabled)
    woke_at = None
    held = None
    for i in range(200):
        was = w.body_asleep.copy()
        before = _snapshot(w, slice(1, 4))
        w.broad_phase(); w.narrow_phase()
        m = w.last_manifolds                                  # what this step's solve starts from
        start = {(int(a), int(b)): (m.warm_start_normal_impulse[lo:hi].copy(), m.warm_start_tangent_impulse[lo:hi].copy())
                 for a, b, lo, hi in zip(m.body1, m.body2, m.point_offsets[:-1], m.point_offsets[1:])}
        w.solve(); w.step_index += 1
        if not was[1:4].any() and w.body_asleep[1:4].all():   # the column fell asleep after this solve: these impulses are held
            held = {(int(a), int(b)): (m.warm_start_normal_impulse[lo:hi].copy(), m.warm_start_tangent_impulse[lo:hi].copy())
                    for a, b, lo, hi in zip(m.body1, m.body2, m.point_offsets[:-1], m.point_offsets[1:])}
        if was[1:4].all() and not w.body_asleep[1:4].any():
            woke_at = i
            break
    assert woke_at is not None, "the cube never woke the column"
    assert w.rows_woken == 3
    assert (w.sleep_timer[1:4] <= np.float32(w.params.dt)).all()                      # timers restarted at the wake
    moved = any(not np.array_equal(a, b) for a, b in zip(before, _snapshot(w, slice(1, 4))))
    assert moved, "the woken bodies were not solved in the step that woke them"
    g = w.graph()
    coloured = set(g["edge"].tolist())
    assert all(int(e) in coloured for e, t in zip(g["sid"], g["touching"]) if t), "a touching row was not pushed again"
    _no_body_twice_in_a_colour(w)
    assert held is not None and len(held) == 3
    for pair, (wn, wt) in held.items():                       # the woken rows warm-start from exactly what their last solve left
        assert np.array_equal(start[pair][0], wn) and np.array_equal(start[pair][1], wt), pair
        assert (wn > 0).all()


def test_a_host_wake_and_sleeping_disabled():
    w = _world(_column())
    for _ in range(40):
        w.step()
    assert w.body_asleep[1:].all()
    w.wake = np.array([0, 0, 1, 0], dtype=np.uint8)
    w.step()
    assert not w.body_asleep.any() and w.graph()["edge"].shape[0] == 3 and not w.graph()["asleep"].any()
    w2 = SleepingWorld(_column(), oracle_plugins(), dict(time_to_sleep=0.2, disabled=np.array([0, 0, 1, 0], dtype=np.uint8)), substeps=4)
    for _ in range(60):
        w2.step()
    assert not w2.body_asleep.any(), "an island with a SleepingDisabled body slept"


def test_removing_a_sleeping_collider_and_reusing_its_contact_id():
    w = _world(_column())
    for _ in range(40):
        w.step()
    assert w.body_asleep[1:].all()
    g = w.graph()
    top = int(g["ids"][(g["c1"] == 3) | (g["c2"] == 3)][0])
    w.remove_colliders([3])
    g = w.graph()
    assert top not in g["ids"].tolist() and g["asleep"].all()
    w.wake = np.array([0, 1, 0, 0], dtype=np.uint8)      # waking the island is the caller's business
    w.step()                                             # the broad phase finds the pair again: it takes the freed ContactId, awake
    g = w.graph()
    assert top in g["ids"].tolist() and not g["asleep"].any()


def test_sleeping_ragdolls_leave_the_joint_set_and_return_in_order():
    sc = scenes.ragdoll_field(2, pitch=3.0, drop_height=0.1)
    thr = np.full(sc.bodies.count, 50.0, dtype=np.float32)
    w = SleepingWorld(sc, oracle_plugins(), dict(time_to_sleep=0.1, thr_lin=thr, thr_ang=thr), substeps=4)
    total = w.joints.count
    order = {t: (j.body1.copy(), j.body2.copy()) for t, j in w.joints.types.items()}
    for _ in range(30):
        w.step()
    assert w.body_asleep[w.bodies.kind != api.BODY_STATIC].all() and w.solved_joints == 0 and total > 0
    dyn = np.nonzero(w.bodies.kind != api.BODY_STATIC)[0]
    w.wake = np.zeros(sc.bodies.count, dtype=np.uint8); w.wake[dyn[0]] = 1
    w.step()
    assert 0 < w.solved_joints < total, "only the woken ragdoll's joints run"
    w.wake = np.zeros(sc.bodies.count, dtype=np.uint8); w.wake[dyn[-1]] = 1
    w.step()
    for t, j in w.joints.types.items():
        assert np.array_equal(j.body1, order[t][0]) and np.array_equal(j.body2, order[t][1])


def test_an_edge_follows_either_endpoint_the_sensor_pair_quirk():
    """a kinematic sensor overlaps the top cube and never sleeps; its touching pair goes to sleep with the column, and is not updated when the
    sensor moves away, until the column wakes (ContactGraph::sleep_entity_with moves every touching edge of the sleeping collider)"""
    sc = _column(extra=[0.2, 3.2, 0.0], extra_kind=api.BODY_KINEMATIC)
    sensor = np.array([0, 0, 0, 0, 1], dtype=bool)
    w = SleepingWorld(sc, oracle_plugins(), dict(time_to_sleep=0.2, disabled=np.array([0, 0, 0, 0, 1], dtype=np.uint8)), substeps=4, sensor=sensor)
    for _ in range(40):
        w.step()
    assert w.body_asleep[1:4].all() and not w.body_asleep[4]
    g = w.graph()
    quirk = int(g["ids"][((g["c1"] == 4) | (g["c2"] == 4))][0])
    at = lambda g, e: int(np.nonzero(g["sid"] == e)[0][0])
    assert g["touching"][at(g, quirk)] and g["asleep"][at(g, quirk)]
    w.bodies.linear_velocity[4] = (5.0, 0.0, 0.0)          # the awake endpoint leaves
    for _ in range(30):
        w.step()
    assert w.bodies.position[4, 0] > 2.0
    g = w.graph()
    assert quirk in g["ids"].tolist() and g["touching"][at(g, quirk)] and g["asleep"][at(g, quirk)], "the sleeping pair was updated"
    w.wake = np.array([0, 1, 0, 0, 0], dtype=np.uint8)
    w.step()                                               # the wake follows this step's narrow phase: the pair is active from the next one on
    assert not w.graph()["asleep"].any()
    w.step()
    g = w.graph()
    assert quirk not in g["ids"].tolist() or not g["touching"][at(g, quirk)], "the woken pair was not updated"
    assert len(w.events[1]["collider1"]) == 1              # its CollisionEnd comes now
