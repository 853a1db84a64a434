"""TEST INFRASTRUCTURE — the reference world with sleeping applied, in plain Python: plugins.World (host ContactGraph / ConstraintGraph fixture)
+ oracle/islands_oracle.py in candidate="body" mode + the application rules of SleepIslands::apply / WakeIslands::apply
(dynamics/solver/islands/sleeping.rs:354-533, collision/contact_types/contact_graph.rs:702-826) restated:

  * an island put to sleep takes every TOUCHING, not yet sleeping edge of its bodies out of the active pairs (an edge follows either endpoint);
    the fixture pops its manifolds and stops updating it;
  * a woken island's edges return; touching, constraint-generating ones are pushed again (ascending ContactId: the device's stated order);
  * a sleeping body has no SolverBody: the solver sees it as static, so it is neither integrated nor written back; its velocities stay;
  * a sleeping body's interval is inactive in the broad phase;
  * a joint whose two bodies are asleep or static is not solved.

The narrow phase's wakes are applied before the solve of the same step, sleep_islands' decisions after it (schedule/mod.rs:98-105).
The product path is csrc/contacts.cu (avn_islands_apply / avn_islands_wake / avn_islands_step) driven by plugins.DeviceGraphWorld(sleeping=...)."""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "oracle"))
from avian_b200 import api, plugins  # noqa: E402
from islands_oracle import STATIC, IslandsOracle  # noqa: E402


def column_scene(extra=None, extra_kind=api.BODY_DYNAMIC):
    """a static floor (body 0), three unit cubes resting on each other (1, 2, 3), optionally one more unit cube (4) at `extra`"""
    from avian_b200 import scenes
    pos = [[0, -0.5, 0], [0, 0.5, 0], [0, 1.5, 0], [0, 2.5, 0]] + ([list(extra)] if extra is not None else [])
    n = len(pos)
    he = np.concatenate([[[10.0, 0.5, 10.0]], np.full((n - 1, 3), 0.5)])
    kind = np.concatenate([[api.BODY_STATIC], np.full(3, api.BODY_DYNAMIC), [extra_kind] if extra is not None else []]).astype(np.uint8)
    rot = np.tile(np.array([0.0, 0.0, 0.0, 1.0]), (n, 1))
    return scenes._assemble("column", np.array(pos, dtype=float), rot, kind, he, np.full(n, scenes.SHAPE_CUBOID), np.float32)


class TwoHalfIslands(IslandsOracle):
    """IslandsOracle.step() in the two halves the schedule runs them in: `narrow_phase_events` (before the solver) and `sleeping` (after it).
    tests/test_sleeping_cpu.py checks that the halves together equal step()."""

    def narrow_phase_events(self, events, wake=None):
        to_wake = []
        for cid, what, b1, b2 in sorted(events):
            if what == "remove":
                iid = self.contact_island.pop(cid, None)
                if iid is None:
                    continue
                isl = self.islands[iid]
                isl.contacts.discard(cid)
                isl.removed += 1
                self.contact_bodies.pop(cid, None)
            else:
                if not self._has_island(b1) and not self._has_island(b2):
                    continue
                iid = self._merge(b1, b2)
                self.islands[iid].contacts.add(cid)
                self.contact_island[cid] = iid
                self.contact_bodies[cid] = (b1, b2)
                if self.islands[iid].sleeping:
                    to_wake.append(iid)
        self._wake(to_wake)
        if wake is not None:
            self._wake([int(self.body_island[b]) for b in np.nonzero(wake)[0] if self._has_island(b)])

    def sleeping_half(self, lin_vel, ang_vel, delta_secs, wake=None):
        """split_island + update_sleeping_states + sleep_islands: step() with no events runs exactly that (wake: bodies touched after the solve)"""
        return self.step([], lin_vel, ang_vel, delta_secs, wake=wake)


class SleepingWorld(plugins.World):
    def __init__(self, scene, plugin_group, sleeping: dict, **kw):
        super().__init__(scene, plugin_group, **kw)
        n = int(scene.bodies.count)
        self.n = n
        jb = plugins.island_joint_bodies(self.joints)
        cfg = dict(sleeping)
        self.orc = TwoHalfIslands(self.bodies.kind, joints=[] if jb is None else jb.tolist(), thr_lin=cfg.get("thr_lin"), thr_ang=cfg.get("thr_ang"),
                                  disabled=cfg.get("disabled"), time_to_sleep=cfg.get("time_to_sleep", 0.5), length_unit=cfg.get("length_unit", 1.0),
                                  scalar=self.scalar, candidate="body")
        self.body_asleep = np.zeros(n, dtype=bool)       # the applied state (`Sleeping` component)
        self.sleeping_flags = np.zeros(n, dtype=np.uint8)
        self.island = np.arange(n, dtype=np.uint32)
        self.wake: np.ndarray | None = None
        self.late_wake: np.ndarray | None = None         # bodies touched after the solve (the `wake` column of the island step's second half)
        self._linked: dict[int, tuple[int, int]] = {}    # touching constraint-generating pairs the islands know: ContactId -> colliders
        self.rows_woken = self.rows_slept = 0

    # ---- broad phase: Has<Sleeping> makes the interval inactive
    def interval_flags(self, order, flags):
        f = super().interval_flags(order, flags)
        asleep = self.sleeping_flags.astype(bool)
        if self.wake is not None and asleep.any():
            asleep = asleep & ~np.isin(self.island, self.island[np.nonzero(self.wake)[0]])
        return f | np.where(asleep[order], api.AABB_IS_INACTIVE, 0).astype(np.uint8)

    # ---- the contact events the islands receive, from the fixture's pairs (a removed pair's ContactId may already hold another pair)
    def _island_events(self):
        p = self.pipeline
        ids, c1, c2, b1, b2 = p.active_edges()
        sid, touching, _ = p.edge_states()
        t = dict(zip(sid.tolist(), touching.tolist()))
        gen = np.ones(ids.shape[0], dtype=bool) if self.sensor is None else ~(self.sensor[c1] | self.sensor[c2])
        now = {int(e): (int(a), int(b)) for e, a, b, g in zip(ids, c1, c2, gen) if g and t[int(e)]}
        ev = [(e, "remove", *cc) for e, cc in self._linked.items() if now.get(e) != cc]
        ev += [(e, "add", *cc) for e, cc in now.items() if self._linked.get(e) != cc]      # (colliders are the bodies in this fixture)
        self._linked = now
        return ev

    def _edges_of(self, bodies_mask: np.ndarray, want_asleep: bool):
        """live edges with a non-static endpoint in the mask: asleep ones (to wake) or touching awake ones (to put to sleep)"""
        p = self.pipeline
        ids, _, _, b1, b2 = p.active_edges()
        sid, touching, asleep = p.edge_states()
        pos = np.searchsorted(sid, ids)
        t, a = touching[pos], asleep[pos]
        dyn = self.bodies.kind != STATIC
        hit = (bodies_mask[b1] & dyn[b1]) | (bodies_mask[b2] & dyn[b2])
        return np.sort(ids[hit & (a if want_asleep else (t & ~a))])

    def _apply(self):
        """bring the applied state in line with the islands' decisions: wakes first, then sleeps"""
        want = self.orc.sleeping().astype(bool)
        woke, fell = self.body_asleep & ~want, want & ~self.body_asleep
        self.body_asleep = want
        if woke.any():
            ids = self._edges_of(~self.body_asleep, True)
            self.pipeline.wake_edges(ids)
            self.rows_woken += int(ids.shape[0])
        if fell.any():
            ids = self._edges_of(fell, False)
            self.pipeline.sleep_edges(ids)
            self.rows_slept += int(ids.shape[0])
        return bool(woke.any())

    def narrow_phase(self):
        super().narrow_phase()
        self.orc.narrow_phase_events(self._island_events(), self.wake)
        self.wake = None
        if self._apply():
            self.last_manifolds = self.pipeline.export_manifolds()
        return self.last_manifolds

    def solve(self):
        b = self.bodies
        kind, joints = b.kind, self.joints
        still = self.body_asleep | (kind == STATIC)
        b.kind = np.where(self.body_asleep, STATIC, kind).astype(kind.dtype)
        # the joint filter, restated: a joint runs unless both its bodies are asleep or static; the rest keep their order
        kept = None
        if joints is not None and joints.count:
            kept = {t: np.array([not (still[a] and still[c]) for a, c in zip(j.body1, j.body2)], dtype=bool) for t, j in joints.types.items()}
            self.joints = api.JointSet({t: api.Joints(**{n: (None if v is None else np.ascontiguousarray(v[kept[t]])) for n, v in j.__dict__.items()})
                                        for t, j in joints.types.items()})
        self.solved_joints = 0 if self.joints is None else self.joints.count
        try:
            super().solve()
        finally:
            b.kind = kind
            if kept is not None:
                for t, j in joints.types.items():
                    for n in ("force", "torque"):
                        if getattr(j, n) is not None:
                            getattr(j, n)[kept[t]] = getattr(self.joints.types[t], n)
            self.joints = joints
        lab, slp = self.orc.sleeping_half(b.linear_velocity, b.angular_velocity, np.float32(self.params.dt), wake=self.late_wake)
        self.late_wake = None
        self.island, self.sleeping_flags = lab, slp
        self.sleep_timer = self.orc.timer.copy()
        self._apply()

    def _unlink_removed(self):
        """remove_collider applies remove_contact at once (narrow_phase/mod.rs:399-459): the islands hear of the pairs that just left the graph"""
        ids, c1, c2, _, _ = self.pipeline.active_edges()
        live = {int(e): (int(a), int(b)) for e, a, b in zip(ids, c1, c2)}
        gone = [(e, "remove", *cc) for e, cc in self._linked.items() if live.get(e) != cc]
        for e, *_ in gone:
            del self._linked[e]
        self.orc.narrow_phase_events(gone)

    def remove_colliders(self, colliders) -> None:
        super().remove_colliders(colliders)
        self._unlink_removed()

    def set_sensors(self, sensor) -> None:
        super().set_sensors(sensor)
        self._unlink_removed()

    def graph(self):
        """ContactIds, pairs, touching / asleep, colour per row, and the colour-major list, as the device's downloads show them"""
        p = self.pipeline
        ids, c1, c2, _, _ = p.active_edges()
        sid, touching, asleep = p.edge_states()
        co, edge, *_ = p.export_edges(int(p.lib.avh_graph_size(p.h, None)))
        return {"ids": ids, "c1": c1, "c2": c2, "sid": sid, "touching": touching, "asleep": asleep, "color_offsets": co, "edge": edge}
