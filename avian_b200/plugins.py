"""Host-side mirror of the reference's plugin interface for the hot path.

In avian3d an app swaps plugins like this (src/lib.rs:718-733, crates/avian3d/examples/custom_broad_phase.rs:10-16):

    PhysicsPlugins::default().build().disable::<BroadPhasePlugin>().add(GpuBroadPhasePlugin)

The Rust shim that does exactly that is in INTEGRATION.md (no Rust toolchain exists in this image).  This module is
the same structure in Python so the tests and the bench read like the reference's: a `PhysicsPlugins` group holds
`IntegratorPlugin`, `BroadPhasePlugin` and `SolverPlugin` (which covers `XpbdSolverPlugin`, as in the GPU library one
call runs the whole substep schedule); `.disable(...)` / `.add(...)` swap implementations; `World.step()` runs the
PhysicsSchedule order  BroadPhase -> NarrowPhase -> Solver  (src/schedule/mod.rs:96-108).

The GPU plugins call the C ABI (avian_b200.api) and nothing else.  A plugin backed by the CPU oracle exists only in
tests/ (tests/oracle_lib.py) — the product has no CPU path.
"""
from __future__ import annotations

import numpy as np

from . import api
from .fixture import HostPipeline
from .scenes import Scene


class Gravity:
    """integrator/mod.rs:150-166"""
    def __init__(self, x=0.0, y=-9.81, z=0.0):
        self.value = (x, y, z)

    ZERO = None


Gravity.ZERO = Gravity(0.0, 0.0, 0.0)


class SubstepCount(int):
    """solver/schedule.rs:185-191 (default 6)"""
    def __new__(cls, value: int = 6):
        return super().__new__(cls, value)


class SolverConfig:
    """solver/plugin.rs:216-302"""
    def __init__(self, contact_damping_ratio=10.0, contact_frequency_factor=1.5, max_overlap_solve_speed=4.0, warm_start_coefficient=1.0,
                 restitution_threshold=1.0, restitution_iterations=1):
        self.contact_damping_ratio = contact_damping_ratio
        self.contact_frequency_factor = contact_frequency_factor
        self.max_overlap_solve_speed = max_overlap_solve_speed
        self.warm_start_coefficient = warm_start_coefficient
        self.restitution_threshold = restitution_threshold
        self.restitution_iterations = restitution_iterations


class IntegratorPlugin:
    """integrator/mod.rs:45-88.  Owns the `Gravity` resource; the integration kernels run inside the solver stage
    (integrate_velocities / integrate_positions are systems of the SubstepSchedule, solver/schedule.rs:59-69)."""
    def __init__(self, gravity: Gravity | None = None):
        self.gravity = gravity or Gravity()


class BroadPhasePlugin:
    """collision/broad_phase.rs:44-155 on the GPU: collect_collision_pairs -> avn_broadphase."""
    def __init__(self, ctx: api.Context):
        self.ctx = ctx

    def collect_collision_pairs(self, aabbs: api.Aabbs) -> api.PairList:
        return self.ctx.broadphase(aabbs)


class SolverPlugin:
    """solver/plugin.rs:88-157 + xpbd/plugin.rs:21-110 + solver_body/plugin.rs on the GPU: one avn_solver_step."""
    def __init__(self, ctx: api.Context, config: SolverConfig | None = None):
        self.ctx = ctx
        self.config = config or SolverConfig()

    def step(self, params: api.AvnStepParams, bodies: api.Bodies, manifolds: api.Manifolds | None, joints: api.JointSet | None) -> None:
        self.ctx.solver_step(params, bodies, manifolds, joints)


class SpatialQueryPlugin:
    """spatial_query/mod.rs:400-417 on the GPU: update_spatial_query_pipeline (avn_query_update over every collider of the world) and the
    raycast system (RayCaster -> RayHits through avn_query_ray_hits).  Collider = body, as in the narrow phase of this fixture.
    Runs after the physics step (PhysicsStepSystems::SpatialQuery), so it sees the poses the step produced."""
    def __init__(self, ctx: api.Context):
        self.ctx = ctx

    @staticmethod
    def colliders(world: "World", memberships: np.ndarray | None = None) -> api.QueryColliders:
        return api.QueryColliders(shape=world.scene.shape_type.astype(np.uint8), dims=world.scene.dims, position=world.bodies.position,
                                  rotation=world.bodies.rotation, memberships=memberships)

    def update_pipeline(self, world: "World", memberships: np.ndarray | None = None, shapes_unchanged: bool = False) -> None:
        """SpatialQueryPipeline::update from the world's current poses.  shapes_unchanged: the caller vouches that shapes, dims and
        memberships equal those of its previous update of this context (AVN_QUERY_SHAPES_UNCHANGED); only the poses are copied, and
        `memberships` is then not read."""
        self.ctx.query_update(self.colliders(world, memberships), shapes_unchanged=shapes_unchanged)

    @staticmethod
    def ray_casters(origin, direction, max_distance, max_hits=None, solid=None, mask=None, enabled=None, owner=None, ignore_self=None,
                    exclude=None) -> api.Rays:
        """A batch of RayCaster components as rays: a disabled caster keeps no hits (max_hits 0); ignore_self excludes the caster's own
        collider `owner` (-1 = none) on top of its filter's excluded entities `exclude` (per caster, iterables)."""
        n = int(np.asarray(origin).reshape(-1, 3).shape[0])
        mh = np.full(n, api.MAX_HITS_ALL, dtype=np.uint32) if max_hits is None else np.array(max_hits, dtype=np.uint32)
        if enabled is not None:
            mh = np.where(np.asarray(enabled, dtype=bool), mh, 0).astype(np.uint32)
        ex = [list(e) for e in exclude] if exclude is not None else [[] for _ in range(n)]
        if owner is not None:
            own = np.asarray(owner, dtype=np.int64)
            ign = np.ones(n, dtype=bool) if ignore_self is None else np.asarray(ignore_self, dtype=bool)   # RayCaster::ignore_self defaults to true
            for i in np.nonzero(ign & (own >= 0))[0]:
                ex[i].append(int(own[i]))
        return api.Rays(origin=origin, direction=direction, max_distance=max_distance, solid=solid, max_hits=mh, mask=mask, exclude=ex)

    def raycast(self, rays: api.Rays) -> dict:
        """The raycast system: every caster's RayHits (CSR; per caster its max_hits nearest, sorted by distance)."""
        return self.ctx.ray_hits(rays)

    @staticmethod
    def shape_casters(shape, dims, origin, rotation, direction, max_distance=None, max_hits=None, enabled=None, owner=None, ignore_self=None,
                      compute_contact_on_penetration=None, ignore_origin_penetration=None, target_distance=None, mask=None,
                      exclude=None) -> api.ShapeQueries:
        """A batch of ShapeCaster components (shape_caster.rs:63-175) with their global origin, rotation and direction, and the reference
        defaults: max_hits 1, max_distance Scalar::MAX (f32's, finite in both scalars), target_distance 0, compute_contact_on_penetration
        true, ignore_origin_penetration false, ignore_self true (excludes the caster's own collider `owner`, -1 = none).  A disabled caster
        keeps no hits (max_hits 0)."""
        n = int(np.asarray(origin).reshape(-1, 3).shape[0])
        col = lambda v, default, dt: np.full(n, default, dtype=dt) if v is None else np.broadcast_to(np.asarray(v, dtype=dt), (n,)).copy()
        mh = col(max_hits, 1, np.uint32)
        if enabled is not None:
            mh = np.where(np.asarray(enabled, dtype=bool), mh, 0).astype(np.uint32)
        flags = np.where(col(compute_contact_on_penetration, True, bool), 0, api.CAST_NO_CONTACT_ON_PENETRATION).astype(np.uint32)
        flags |= np.where(col(ignore_origin_penetration, False, bool), api.CAST_IGNORE_ORIGIN_PENETRATION, 0).astype(np.uint32)
        ex = [list(e) for e in exclude] if exclude is not None else [[] for _ in range(n)]
        if owner is not None:
            own = np.asarray(owner, dtype=np.int64)
            for i in np.nonzero(col(ignore_self, True, bool) & (own >= 0))[0]:
                ex[i].append(int(own[i]))
        return api.ShapeQueries(shape=shape, dims=dims, position=origin, rotation=rotation, direction=direction,
                                max_distance=col(max_distance, float(np.finfo(np.float32).max), np.float64),
                                target_distance=None if target_distance is None else col(target_distance, 0.0, np.float64), flags=flags, max_hits=mh,
                                mask=mask, exclude=ex)

    def shapecast(self, shapes: api.ShapeQueries) -> dict:
        """The shapecast system: every caster's ShapeHits (CSR; per caster its max_hits nearest, sorted by distance)."""
        return self.ctx.shape_hits(shapes)


class PhysicsPlugins:
    """The plugin group (src/lib.rs:813-843) restricted to the hot path."""
    def __init__(self, ctx: api.Context | None = None):
        self._plugins = {}
        if ctx is not None:
            self.add(IntegratorPlugin()).add(BroadPhasePlugin(ctx)).add(SolverPlugin(ctx))

    def build(self):
        return self

    def disable(self, cls):
        for k in [k for k, v in self._plugins.items() if isinstance(v, cls) or k == getattr(cls, "__name__", cls)]:
            del self._plugins[k]
        return self

    def add(self, plugin, name: str | None = None):
        self._plugins[name or _slot_of(plugin)] = plugin
        return self

    def get(self, name):
        try:
            return self._plugins[name]
        except KeyError:
            raise RuntimeError(f"{name} missing: add it to PhysicsPlugins (cf. `expect(\"add PhysicsSchedule first\")`, solver/plugin.rs:104-106)")


def _slot_of(plugin) -> str:
    for base in type(plugin).__mro__:
        if base.__name__ in ("IntegratorPlugin", "BroadPhasePlugin", "SolverPlugin"):
            return base.__name__
    name = type(plugin).__name__
    for slot in ("IntegratorPlugin", "BroadPhasePlugin", "SolverPlugin"):
        if slot.replace("Plugin", "") in name:
            return slot
    return name


class World:
    """A headless world: body columns + the CPU fixture around the hot path + the plugin group."""

    def __init__(self, scene: Scene, plugins: PhysicsPlugins, dt: float = 1.0 / 60.0, substeps: int = 6, solver_iterations: int = 1,
                 ccd: dict | None = None, sensor=None, events_enabled=None):
        """ccd: the SweptCcd bodies — the keyword arguments of api.Context.ccd_configure (body, collider, mode, include_dynamic,
        linear_threshold, angular_threshold, prediction_distance).  The solver plugin must run solve_swept_ccd (a `step_ccd` method).
        sensor / events_enabled: optional per-collider columns (Sensor, CollisionEventsEnabled).  After every step `events` holds the
        (started, ended) lists of api.Context.contacts_events (DeviceGraphWorld: when either column is given)."""
        self.scene = scene
        self.sensor = None if sensor is None else np.asarray(sensor, dtype=bool)
        self.events_enabled = None if events_enabled is None else np.asarray(events_enabled, dtype=bool)
        self.events: tuple[dict, dict] | None = None
        self.ccd = ccd
        self.bodies = scene.bodies
        self.joints = scene.joints
        self.scalar = scene.bodies.position.dtype
        self.plugins = plugins
        self.pipeline = HostPipeline(scene.shape_type, scene.dims, scene.friction, scene.restitution, scalar=self.scalar)
        integ = plugins.get("IntegratorPlugin")
        cfg = getattr(plugins.get("SolverPlugin"), "config", None) or SolverConfig()
        self.params = api.default_step_params(dt=dt, substeps=substeps, gravity=integ.gravity.value, solver_iterations=solver_iterations,
                                              contact_damping_ratio=cfg.contact_damping_ratio, contact_frequency_factor=cfg.contact_frequency_factor,
                                              max_overlap_solve_speed=cfg.max_overlap_solve_speed, warm_start_coefficient=cfg.warm_start_coefficient,
                                              restitution_threshold=cfg.restitution_threshold, restitution_iterations=cfg.restitution_iterations)
        if self.sensor is not None:
            self.pipeline.set_sensors(self.sensor)
        self.last_manifolds: api.Manifolds | None = None
        self.last_pairs: api.PairList | None = None
        self.last_aabbs: api.Aabbs | None = None
        self.step_index = 0

    # the stages of one PhysicsSchedule run, separately callable so tests/bench can snapshot in between
    def broad_phase(self) -> api.PairList:
        dt = self.params.dt
        self.aabb_min, self.aabb_max = self.pipeline.update_aabbs(self.bodies, dt)
        aabbs = self.pipeline.intervals(self.bodies, self.aabb_min, self.aabb_max)
        aabbs.flags = self.interval_flags(aabbs.collider, aabbs.flags)
        aabbs.joint_disabled_body_pairs = self.scene.joint_disabled_body_pairs
        pairs = self.plugins.get("BroadPhasePlugin").collect_collision_pairs(aabbs)
        self.pipeline.commit_broadphase(aabbs, pairs)
        self.last_aabbs, self.last_pairs = aabbs, pairs
        return pairs

    def interval_flags(self, order: np.ndarray, flags: np.ndarray) -> np.ndarray:
        """init_aabb_interval_flags (broad_phase.rs:318-335) for the optional columns: events_enabled sets CONTACT_EVENTS, a sensor clears
        GENERATE_CONSTRAINTS.  `order` = the colliders of the interval columns."""
        if self.events_enabled is None and self.sensor is None:
            return flags
        f = flags.copy()
        if self.events_enabled is not None:
            f |= np.where(self.events_enabled[order], api.AABB_CONTACT_EVENTS, 0).astype(np.uint8)
        if self.sensor is not None:
            f &= np.where(self.sensor[order], ~np.uint8(api.AABB_GENERATE_CONSTRAINTS), np.uint8(0xFF)).astype(np.uint8)
        return f

    def set_sensors(self, sensor) -> None:
        """The Sensor column changes (On<Add, Sensor> / On<Remove, Sensor>): the changed colliders' pairs leave the graphs at once."""
        self.sensor = None if sensor is None else np.asarray(sensor, dtype=bool)
        self.pipeline.set_sensors(self.sensor)

    def remove_colliders(self, colliders) -> None:
        """remove_collider for despawned / disabled colliders: their pairs leave the graphs, touching ones queue a CollisionEnd."""
        self.pipeline.remove_colliders(colliders)

    def report(self, events_only: bool = False) -> dict:
        """The touching pairs with their impulses as the last solve left them (api.Context.contacts_report)."""
        return self.pipeline.report(events_only)

    def narrow_phase(self) -> api.Manifolds:
        self.last_manifolds = self.pipeline.narrow_phase(self.bodies, self.aabb_min, self.aabb_max, self.params.dt, bool(self.params.match_contacts))
        self.events = self.pipeline.events()
        return self.last_manifolds

    def solve(self) -> None:
        m = self.last_manifolds
        solver = self.plugins.get("SolverPlugin")
        if self.ccd is not None:
            if not hasattr(solver, "step_ccd"):
                raise ValueError(f"{type(solver).__name__} does not run swept CCD: on the GPU it needs the device-resident pipeline (DeviceGraphWorld)")
            solver.step_ccd(self.params, self.bodies, m, self.joints, self.ccd, self.pipeline.active_edges(), self.scene.shape_type, self.scene.dims)
        else:
            solver.step(self.params, self.bodies, m, self.joints)
        if m is not None and m.count:
            self.pipeline.store_impulses(m)

    def step(self) -> None:
        self.broad_phase()
        self.narrow_phase()
        self.solve()
        self.step_index += 1


class ResidentWorld(World):
    """The same world stepped through the RESIDENT protocol (SURVEY.md 8f #1/#3, DESIGN.md §8): what a device-resident pipeline keeps
    on the GPU lives here in edge-indexed arrays (ContactId-indexed, 4 point slots per edge), the host keeps only the graphs.

        geometry (per edge, no host state)  ->  point counts + disjoint flags to the host  ->  touching state machine, contact graph,
        constraint-graph colouring  ->  colour-major list of edge ids back  ->  the solver gathers its manifolds from the edge arrays
        ->  warm-start impulses scattered back into the edge arrays.

    `geometry(dt, tol, pairs, colliders, lin_vel, ang_vel, f64_anchors=True)` is fixture.raw_manifolds here and avn_narrow_phase on the
    device; everything else is the bookkeeping the device kernels will replace one by one.  Stepping this world gives the same
    manifolds, bit for bit, as World (tests/test_resident_cpu.py): it is the executable specification of the protocol."""

    def __init__(self, scene: Scene, plugins: PhysicsPlugins, geometry=None, **kw):
        super().__init__(scene, plugins, **kw)
        from avian_b200 import fixture
        self.geometry = geometry or fixture.raw_manifolds
        self._fixture = fixture
        self.capacity = 0
        self._grow(1024)
        self.edge_key = np.zeros(0, dtype=np.uint64)
        self.bytes_to_host = 0        # what crosses PCIe per step in a device-resident pipeline (counts + flags; pairs come on top)
        self.bytes_to_device = 0      # (edge list of the graph)

    def _grow(self, capacity: int) -> None:
        s = self.scalar
        def grown(name, shape, dtype):
            new = np.zeros((capacity,) + shape, dtype=dtype)
            old = getattr(self, name, None)
            if old is not None:
                new[:old.shape[0]] = old
            setattr(self, name, new)
        grown("e_count", (), np.uint8)                 # resident per-edge state
        grown("e_normal", (3,), s)
        grown("e_anchor1", (4, 3), s); grown("e_anchor2", (4, 3), s)
        grown("e_penetration", (4,), s); grown("e_normal_speed", (4,), s)
        grown("e_prev_count", (), np.uint8)            # what match_contacts compares against, in double like the fixture
        grown("e_prev_a1", (4, 3), np.float64); grown("e_prev_a2", (4, 3), np.float64)
        grown("e_ws_n", (4,), s); grown("e_ws_t", (4, 2), s)
        grown("e_key", (), np.uint64)
        self.capacity = capacity

    def narrow_phase(self) -> api.Manifolds:
        p, b, s = self.pipeline, self.bodies, self.scalar
        ids, c1, c2, b1, b2 = p.active_edges()
        if ids.size and int(ids.max()) >= self.capacity:
            self._grow(max(2 * self.capacity, int(ids.max()) + 1))
        # a ContactId handed to a new pair starts without history
        key = (c1.astype(np.uint64) << np.uint64(32)) | c2.astype(np.uint64)
        fresh = self.e_key[ids] != key
        self.e_prev_count[ids[fresh]] = 0
        self.e_ws_n[ids[fresh]] = 0
        self.e_ws_t[ids[fresh]] = 0
        self.e_key[ids] = key
        colliders = {"shape": self.scene.shape_type.astype(np.uint8), "dims": np.asarray(self.scene.dims, dtype=s), "position": b.position,
                     "rotation": b.rotation, "aabb_min": self.aabb_min, "aabb_max": self.aabb_max}
        raw = self.geometry(s, self.params.dt, 0.005, (c1, c2, b1, b2), colliders, b.linear_velocity, b.angular_velocity, f64_anchors=True)
        # device side: scatter into the edge arrays, carry the warm-start impulses over (match_contacts)
        self.e_count[ids] = raw["point_count"]
        for k in ("normal", "anchor1", "anchor2", "penetration", "normal_speed"):
            getattr(self, "e_" + k)[ids] = raw[k]
        lib = p.lib
        lib.avh_match_raw(p.bits, int(ids.shape[0]), ids.ctypes.data, raw["point_count"].ctypes.data, raw["anchor1_f64"].ctypes.data,
                          raw["anchor2_f64"].ctypes.data, 1.0, 1 if self.params.match_contacts else 0, self.e_prev_count.ctypes.data,
                          self.e_prev_a1.ctypes.data, self.e_prev_a2.ctypes.data, self.e_ws_n.ctypes.data, self.e_ws_t.ctypes.data)
        # host side: counts + flags in, graph updates, edge list out
        self.bytes_to_host = 2 * int(ids.shape[0])
        m, npts = p.apply_counts(b, ids, raw["point_count"], raw["disjoint"])
        co, edge, eb1, eb2, fr, re = p.export_edges(m)
        self.bytes_to_device = 4 * m
        self._edges = edge
        # solver input: gathered from the edge arrays by the edge list (on the device: an indirection in prepare_constraint_item)
        cnt = self.e_count[edge].astype(np.int64)
        po = np.concatenate([[0], np.cumsum(cnt)]).astype(np.uint32)
        slot = np.arange(4)[None, :] < cnt[:, None]                      # [m, 4] live point slots, row-major = CSR order
        self._slot = slot
        take = lambda a: np.ascontiguousarray(a[edge][slot])
        man = api.Manifolds(color_offsets=co, body1=eb1, body2=eb2, normal=np.ascontiguousarray(self.e_normal[edge]), friction=fr.astype(s),
                            restitution=re.astype(s), point_offsets=po, anchor1=take(self.e_anchor1), anchor2=take(self.e_anchor2),
                            penetration=take(self.e_penetration), normal_speed=take(self.e_normal_speed),
                            warm_start_normal_impulse=take(self.e_ws_n), warm_start_tangent_impulse=take(self.e_ws_t),
                            normal_impulse=np.zeros(int(po[-1]), dtype=s))
        assert int(po[-1]) == npts
        self.last_manifolds = man
        return man

    def solve(self) -> None:
        m = self.last_manifolds
        self.plugins.get("SolverPlugin").step(self.params, self.bodies, m, self.joints)
        if m is not None and m.count:          # store_contact_impulses: back into the edge arrays
            wn, wt = self.e_ws_n[self._edges], self.e_ws_t[self._edges]
            wn[self._slot] = m.warm_start_normal_impulse
            wt[self._slot] = m.warm_start_tangent_impulse
            self.e_ws_n[self._edges] = wn
            self.e_ws_t[self._edges] = wt


class DeviceResidentWorld(World):
    """The resident protocol with the device doing its part (ResidentWorld is the CPU specification): contact rows, manifolds and warm-start
    impulses live in the library's contact store; per step the host sends the contact-graph changes (new / removed edges), receives one
    point count and one disjoint flag per row, updates its graphs and sends the colour-major edge list; avn_solver_upload_graph reads the
    manifolds where avn_contacts_narrow_phase left them."""

    def __init__(self, scene: Scene, plugins: PhysicsPlugins, ctx: "api.Context", **kw):
        super().__init__(scene, plugins, **kw)
        self.ctx = ctx
        self.capacity = 0
        self.known = {}          # ContactId -> pair key of the row on the device
        self.bytes_to_host = self.bytes_to_device = 0
        self._steady = None      # step_steady's memory: which rows were touching, which ids are live
        self._colliders = None

    def narrow_phase(self):
        p, b, s = self.pipeline, self.bodies, self.scalar
        ids, c1, c2, b1, b2 = p.active_edges()
        need = int(ids.max()) + 1 if ids.size else 0
        if need > self.capacity:
            self.capacity = max(1024, 2 * need)
            self.ctx.contacts_reserve(self.capacity)
        # contact-graph changes since the last step
        key = (c1.astype(np.uint64) << np.uint64(32)) | c2.astype(np.uint64)
        now = dict(zip(ids.tolist(), key.tolist()))
        gone = [e for e in self.known if e not in now]
        fresh = np.array([i for i, (e, k) in enumerate(now.items()) if self.known.get(e) != k], dtype=np.int64)
        if gone:
            self.ctx.contacts_remove(np.array(gone, dtype=np.uint32))
        if fresh.size:
            self.ctx.contacts_add(ids[fresh], c1[fresh], c2[fresh], b1[fresh], b2[fresh])
        self.known = now
        colliders = {"shape": self.scene.shape_type.astype(np.uint8), "dims": np.asarray(self.scene.dims, dtype=s), "position": b.position,
                     "rotation": b.rotation, "aabb_min": self.aabb_min, "aabb_max": self.aabb_max}
        count, disjoint = self.ctx.contacts_narrow_phase(self.params.dt, 0.005, colliders, b.linear_velocity, b.angular_velocity, self.capacity,
                                                         bool(self.params.match_contacts))
        self.bytes_to_host = 2 * self.capacity
        self.bytes_to_device = 20 * int(fresh.size) + 4 * len(gone)
        m, npts = p.apply_counts(b, ids, count[ids], disjoint[ids])
        co, edge, eb1, eb2, fr, re = p.export_edges(m)
        self.bytes_to_device += 4 * m
        self.graph = {"color_offsets": co, "edge": edge, "body1": eb1, "body2": eb2, "friction": fr.astype(s), "restitution": re.astype(s)}
        self.last_counts = count
        self.last_manifolds = None
        return self.graph

    def solve(self) -> None:
        self.ctx.solver_step_graph(self.params, self.bodies, self.graph, self.joints)

    # ---- the steady-state step, incremental on the host: what an application pays per frame once the contact set has settled ------------
    def step_steady(self, aabbs: api.Aabbs, pairs_out: api.PairList) -> bool:
        """One whole step from HOST body columns through the resident protocol: avn_broadphase (host AABB columns in, new pairs out) ->
        avn_contacts_narrow_phase (collider poses + velocities in, one point count and one disjoint flag per contact row out) ->
        avn_solver_upload_graph + run + download (body columns in and out).  The host touches its graphs only when the device reports that
        a pair appeared, separated, or started / stopped touching; otherwise the colour-major edge list of the previous step is still valid and
        stays on the device.  Returns True when the fast path was taken."""
        ctx, p, b, s = self.ctx, self.pipeline, self.bodies, self.scalar
        ctx.broadphase_upload(aabbs)
        ctx.broadphase_run()
        ctx.broadphase_download(pairs_out)
        if pairs_out.count or self._steady is None:
            # contact-graph changes: the general path (edge deltas, graph update, new edge list)
            if pairs_out.count:
                p.commit_broadphase(aabbs, pairs_out.trimmed())
            self.aabb_min, self.aabb_max = self._aabb_rows(aabbs)
            self.narrow_phase()
            self._steady = {"touching": self.last_counts > 0, "ids": p.active_edges()[0]}
            self.solve()
            return False
        colliders = self._colliders
        colliders["position"], colliders["rotation"] = b.position, b.rotation
        count, disjoint = ctx.contacts_narrow_phase(self.params.dt, 0.005, colliders, b.linear_velocity, b.angular_velocity, self.capacity,
                                                    bool(self.params.match_contacts))
        touching = count > 0
        reuse = not disjoint.any() and np.array_equal(touching, self._steady["touching"])
        if not reuse:
            ids = self._steady["ids"]
            m, _ = p.apply_counts(b, ids, count[ids], disjoint[ids])
            co, edge, eb1, eb2, fr, re = p.export_edges(m)
            self.graph = {"color_offsets": co, "edge": edge, "body1": eb1, "body2": eb2, "friction": fr.astype(s), "restitution": re.astype(s)}
            self._steady = None if disjoint.any() else {"touching": touching, "ids": ids}   # a separated pair changes the id set: general path next
        self.last_counts = count
        ctx.solver_step_graph(self.params, b, self.graph, self.joints, reuse_graph=reuse)
        return reuse

    def prepare_steady(self, aabbs: api.Aabbs) -> None:
        """After the settle steps: freeze what does not change per step (shapes, the AABB columns of the broad-phase input in body order)."""
        s = self.scalar
        self.aabb_min, self.aabb_max = self._aabb_rows(aabbs)
        self._colliders = {"shape": self.scene.shape_type.astype(np.uint8), "dims": np.asarray(self.scene.dims, dtype=s), "position": self.bodies.position,
                           "rotation": self.bodies.rotation, "aabb_min": self.aabb_min, "aabb_max": self.aabb_max}
        self._steady = None

    @staticmethod
    def _aabb_rows(aabbs: api.Aabbs):
        """the interval columns (persistent order) back in collider order (collider index == row of the body columns in this fixture)"""
        n = int(aabbs.collider.shape[0])
        mn, mx = np.empty_like(aabbs.aabb_min), np.empty_like(aabbs.aabb_max)
        mn[aabbs.collider], mx[aabbs.collider] = aabbs.aabb_min, aabbs.aabb_max
        return mn, mx


def island_joint_bodies(joints: "api.JointSet | None") -> np.ndarray | None:
    """[J, 2] the bodies every joint links, in type order: what PhysicsIslands::add_joint sees (avn_islands_configure)."""
    if joints is None or not joints.count:
        return None
    return np.concatenate([np.stack([t.body1, t.body2], axis=1) for t in joints.types.values() if t.count]).astype(np.uint32)


def awake_joints(joints: "api.JointSet | None", still: np.ndarray):
    """The joints the solver runs while sleeping is applied: a joint whose two bodies are both `still` (asleep or static) is left out, the
    others keep their order (a joint links its bodies' islands, so it is never half asleep).  Returns (joint set, kept) where kept[type] is
    the mask of the joints taken, for `restore_joint_outputs`; (joints, None) when nothing is left out."""
    if joints is None or not joints.count or not still.any():
        return joints, None
    kept = {t: ~(still[j.body1] & still[j.body2]) for t, j in joints.types.items()}
    if all(k.all() for k in kept.values()):
        return joints, None
    sub = api.JointSet({t: api.Joints(**{n: (None if v is None else np.ascontiguousarray(v[kept[t]])) for n, v in j.__dict__.items()})
                        for t, j in joints.types.items()})
    return sub, kept


def restore_joint_outputs(joints: "api.JointSet", sub: "api.JointSet", kept: dict | None) -> None:
    """the solver's joint outputs (force, torque) of the joints that ran, back in the full set"""
    if kept is None:
        return
    for t, j in joints.types.items():
        for n in ("force", "torque"):
            if getattr(j, n) is not None:
                getattr(j, n)[kept[t]] = getattr(sub.types[t], n)


class DeviceGraphWorld(World):
    """The whole contact pipeline on the device (SURVEY.md 8f #1 + #3): broad phase -> new pairs taken in device memory by the contact store ->
    geometry + match_contacts -> touching state machine, ContactGraph, ConstraintGraph colouring, colour-major list -> solver stage reading
    all of it in place (avn_contacts_step + avn_solver_upload_resident).  The host keeps the body columns and the persistent interval order;
    per step it sends the AABB and body columns and reads back the order, ~40 counters and the bodies.  Steps bit for bit like World
    (tests/test_gpu_graph.py): same ContactIds, same colours, same bodies.

    sleeping: None, or the keyword arguments of api.Context.islands_configure besides the bodies and the joints (time_to_sleep, thr_lin,
    thr_ang, disabled, length_unit).  The world then configures the islands, lets the library apply their decisions (avn_islands_apply) and
    steps  broad phase (sleeping bodies' intervals inactive) -> contacts_step -> islands_wake -> solver -> islands_step.  `wake` ([B], optional,
    consumed by the next step) marks bodies the application touched before the step, `late_wake` bodies it touched after the solve.  `sleeping_flags`, `island`, `sleep_timer`, `islands` hold the last
    islands_step's output, `wake_stats` the last islands_wake's."""

    def __init__(self, scene: Scene, plugins: PhysicsPlugins, ctx: "api.Context", sleeping: dict | None = None, **kw):
        super().__init__(scene, plugins, **kw)
        self.ctx = ctx
        n = int(scene.bodies.count)
        self.n = n
        ctx.contacts_configure(scene.bodies.kind if scene.bodies.kind is not None else np.zeros(n, dtype=np.uint8), n, scene.friction, scene.restitution)
        if self.sensor is not None:
            ctx.contacts_set_sensors(self.sensor)
        self.order = np.arange(n, dtype=np.uint32)       # AabbIntervals' persistent order (colliders = bodies in this fixture)
        self.stats: dict | None = None
        self.new_pairs = 0
        self._shape = np.ascontiguousarray(scene.shape_type, dtype=np.uint8)
        self._dims = np.ascontiguousarray(scene.dims, dtype=self.scalar)
        self._order_out = np.empty(n, dtype=np.uint32)
        self._uploaded_once = False     # from the second step on the static columns (shapes, mass properties ...) stay on the device
        if self.ccd is not None:
            ctx.ccd_configure(**self.ccd)   # solve_swept_ccd inside the device-resident solver stage
        self.sleeping = sleeping
        self.wake: np.ndarray | None = None
        self.late_wake: np.ndarray | None = None     # bodies touched after the solve: passed to islands_step, awake from the next step on
        self.sleeping_flags = np.zeros(n, dtype=np.uint8)
        self.island = np.arange(n, dtype=np.uint32)
        self.sleep_timer = np.zeros(n, dtype=np.float32)
        self.islands: dict | None = None
        self.wake_stats: dict | None = None
        if sleeping is not None:
            ctx.islands_configure(self.bodies.kind, joints=island_joint_bodies(self.joints), **sleeping)
            ctx.islands_apply(True)

    def intervals(self, aabb_min: np.ndarray, aabb_max: np.ndarray) -> api.Aabbs:
        o, kind = self.order, self.bodies.kind
        flags = np.where(kind[o] == api.BODY_STATIC, api.AABB_IS_INACTIVE, 0).astype(np.uint8) | np.uint8(api.AABB_GENERATE_CONSTRAINTS)
        flags = self.interval_flags(o, flags)
        if self.sleeping is not None:      # Has<Sleeping> when the intervals are refreshed (broad_phase.rs:223-260), minus the islands about to wake
            flags = flags | np.where(self.inactive_bodies()[o], api.AABB_IS_INACTIVE, 0).astype(np.uint8)
        a = api.Aabbs(collider=o.copy(), body=o.copy(), aabb_min=np.ascontiguousarray(aabb_min[o]), aabb_max=np.ascontiguousarray(aabb_max[o]),
                      flags=np.ascontiguousarray(flags), order_out=self._order_out)
        a.joint_disabled_body_pairs = self.scene.joint_disabled_body_pairs
        return a

    def inactive_bodies(self) -> np.ndarray:
        """the bodies that enter this step's broad phase asleep: the last islands_step's Sleeping flags minus the islands `wake` reaches"""
        asleep = self.sleeping_flags.astype(bool)
        if self.wake is not None and asleep.any():
            asleep &= ~np.isin(self.island, self.island[np.nonzero(self.wake)[0]])
        return asleep

    def step_from(self, aabbs: api.Aabbs, aabb_min: np.ndarray, aabb_max: np.ndarray) -> dict:
        """One step from host columns: `aabbs` = the interval columns in the persistent order, aabb_min / aabb_max = the same AABBs in collider order."""
        ctx, b = self.ctx, self.bodies
        ctx.broadphase_upload(aabbs)
        ctx.broadphase_run()
        # the solver's body columns start moving now, on the library's copy stream, under the broad phase and the contact pipeline
        ctx.solver_prefetch_bodies(b, static_unchanged=self._uploaded_once)
        colliders = {"shape": self._shape, "dims": self._dims, "position": b.position, "rotation": b.rotation, "aabb_min": aabb_min, "aabb_max": aabb_max}
        self.stats = ctx.contacts_step(self.params.dt, 0.005, colliders, b.linear_velocity, b.angular_velocity, bool(self.params.match_contacts), take_pairs=True,
                                       shapes_unchanged=self._uploaded_once)
        self.new_pairs = ctx.broadphase_download_order()
        kept = int(aabbs.retained_count if aabbs.retained_count is not None else aabbs.collider.shape[0])
        oo = aabbs.order_out[:kept]
        if kept != aabbs.collider.shape[0] or oo[0] != 0 or not (oo[1:] == oo[:-1] + 1).all():   # (a sorted scene keeps its order: nothing to permute)
            self.order = np.ascontiguousarray(aabbs.collider[oo])
        if self.sensor is not None or self.events_enabled is not None:
            self.events = ctx.contacts_events()
        if self.sleeping is None:
            ctx.solver_step_resident(self.params, b, self.joints)
        else:
            self.wake_stats = ctx.islands_wake(self.wake)
            self.wake = None
            # the bodies asleep after the wake half are a subset of the last island step's flags: the same count means the same set
            still = self.sleeping_flags.astype(bool)
            if self.wake_stats["bodies_asleep"] == 0:
                still = np.zeros(self.n, dtype=bool)
            elif self.wake_stats["bodies_asleep"] != int(still.sum()):
                still = ctx.contacts_download_sleeping(0, self.n)["body_asleep"].astype(bool)
            joints, kept = awake_joints(self.joints, still | (b.kind == api.BODY_STATIC))
            ctx.solver_step_resident(self.params, b, joints)
            restore_joint_outputs(self.joints, joints, kept)
            self.islands = ctx.islands_step(float(self.params.dt), b.linear_velocity, b.angular_velocity, wake=self.late_wake)
            self.late_wake = None
            self.sleeping_flags, self.island, self.sleep_timer = self.islands["sleeping"], self.islands["island"], self.islands["sleep_timer"]
        self._uploaded_once = True
        self.step_index += 1
        return self.stats

    def set_sensors(self, sensor) -> None:
        self.sensor = None if sensor is None else np.asarray(sensor, dtype=bool)
        self.ctx.contacts_set_sensors(self.sensor, collider_count=self.n)

    def remove_colliders(self, colliders) -> None:
        self.ctx.contacts_remove_colliders(colliders)

    def report(self, events_only: bool = False) -> dict:
        return self.ctx.contacts_report(events_only=events_only)

    def step(self) -> None:
        self.aabb_min, self.aabb_max = self.pipeline.update_aabbs(self.bodies, self.params.dt)
        self.step_from(self.intervals(self.aabb_min, self.aabb_max), self.aabb_min, self.aabb_max)
