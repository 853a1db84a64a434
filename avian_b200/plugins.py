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
        sc = world.scene
        if sc.compound:   # a collider table: every part at its world pose
            pos, rot = sc.collider_poses(world.bodies)
            return api.QueryColliders(shape=sc.collider_shape.astype(np.uint8), dims=sc.collider_dims, position=pos, rotation=rot, memberships=memberships)
        return api.QueryColliders(shape=sc.shape_type.astype(np.uint8), dims=sc.dims, position=world.bodies.position,
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
        linear_threshold, angular_threshold, prediction_distance, capsules, hulls).  The solver plugin must run solve_swept_ccd (a `step_ccd` method).
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
        if scene.compound:
            if ccd is not None:
                raise ValueError("swept CCD assumes a collider at its body's origin: a scene with a collider table cannot use it")
            self.pipeline = HostPipeline(scene.collider_shape, scene.collider_dims, scene.collider_friction, scene.collider_restitution, scalar=self.scalar,
                                         collider_body=scene.collider_body, hulls=scene.hulls)
        else:
            self.pipeline = HostPipeline(scene.shape_type, scene.dims, scene.friction, scene.restitution, scalar=self.scalar, hulls=scene.hulls)
        self.collider_pose: dict | None = None   # a collider table: the colliders' world poses of the current step
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
    def update_colliders(self) -> dict | None:
        """A collider table: the colliders' world poses from the body poses, and the body velocity at every collider (for the AABBs)."""
        if not self.scene.compound:
            return None
        pos, rot = self.scene.collider_poses(self.bodies)
        lv, av = self.scene.collider_velocities(self.bodies, pos)
        self.collider_pose = {"position": pos, "rotation": rot, "linear_velocity": lv, "angular_velocity": av}
        return self.collider_pose

    def broad_phase(self) -> api.PairList:
        dt = self.params.dt
        self.aabb_min, self.aabb_max = self.pipeline.update_aabbs(self.bodies, dt, self.update_colliders())
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
        self.last_manifolds = self.pipeline.narrow_phase(self.bodies, self.aabb_min, self.aabb_max, self.params.dt, bool(self.params.match_contacts),
                                                         colliders=self.collider_pose)
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
        if scene.hulls is not None:
            ctx.set_convex_hulls(scene.hulls)
        n = int(scene.bodies.count)
        self.n = n
        nc = int(scene.collider_body.shape[0]) if scene.compound else n
        self.collider_count = nc
        ctx.contacts_configure(scene.bodies.kind if scene.bodies.kind is not None else np.zeros(n, dtype=np.uint8), nc,
                               scene.collider_friction if scene.compound else scene.friction, scene.collider_restitution if scene.compound else scene.restitution)
        if self.sensor is not None:
            ctx.contacts_set_sensors(self.sensor)
        self.order = np.arange(nc, dtype=np.uint32)      # AabbIntervals' persistent order of the colliders
        self.stats: dict | None = None
        self.new_pairs = 0
        self._shape = np.ascontiguousarray(scene.collider_shape if scene.compound else scene.shape_type, dtype=np.uint8)
        self._dims = np.ascontiguousarray(scene.collider_dims if scene.compound else scene.dims, dtype=self.scalar)
        self._order_out = np.empty(nc, dtype=np.uint32)
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
        body = o.copy() if not self.scene.compound else np.ascontiguousarray(self.scene.collider_body[o], dtype=np.uint32)
        flags = np.where(kind[body] == api.BODY_STATIC, api.AABB_IS_INACTIVE, 0).astype(np.uint8) | np.uint8(api.AABB_GENERATE_CONSTRAINTS)
        flags = self.interval_flags(o, flags)
        if self.sleeping is not None:      # Has<Sleeping> when the intervals are refreshed (broad_phase.rs:223-260), minus the islands about to wake
            flags = flags | np.where(self.inactive_bodies()[body], api.AABB_IS_INACTIVE, 0).astype(np.uint8)
        a = api.Aabbs(collider=o.copy(), body=body, aabb_min=np.ascontiguousarray(aabb_min[o]), aabb_max=np.ascontiguousarray(aabb_max[o]),
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
        pose = self.collider_pose if self.scene.compound else {"position": b.position, "rotation": b.rotation}
        colliders = {"shape": self._shape, "dims": self._dims, "position": pose["position"], "rotation": pose["rotation"], "aabb_min": aabb_min,
                     "aabb_max": aabb_max}
        if self.scene.compound:   # the anchors are measured from the bodies' centres of mass
            ctx.contacts_set_body_frames(b.position, b.rotation, b.center_of_mass)
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
        self.ctx.contacts_set_sensors(self.sensor, collider_count=self.collider_count)

    def remove_colliders(self, colliders) -> None:
        self.ctx.contacts_remove_colliders(colliders)

    def report(self, events_only: bool = False) -> dict:
        return self.ctx.contacts_report(events_only=events_only)

    def step(self) -> None:
        self.aabb_min, self.aabb_max = self.pipeline.update_aabbs(self.bodies, self.params.dt, self.update_colliders())
        self.step_from(self.intervals(self.aabb_min, self.aabb_max), self.aabb_min, self.aabb_max)
