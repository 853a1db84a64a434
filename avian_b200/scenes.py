"""Synthetic scenes of BASELINE.json's configs as body columns (+ collider shapes for the host fixture).

All generators are deterministic (no RNG unless a seed is an argument).  Bodies use the reference's defaults:
density 1 (ColliderDensity), friction 0.5 / restitution 0 (physics_material.rs:152-160,320-327), gravity -9.81 y.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from . import api
from .fixture import SHAPE_CAPSULE, SHAPE_CUBOID, SHAPE_SPHERE


@dataclass
class Scene:
    name: str
    bodies: api.Bodies
    shape_type: np.ndarray   # int32[n]
    dims: np.ndarray         # float64[n,3] half extents / radius
    friction: np.ndarray     # float64[n]
    restitution: np.ndarray  # float64[n]
    joints: api.JointSet | None = None
    joint_disabled_body_pairs: np.ndarray | None = None
    # optional collider table (ColliderOf + the collider's Transform relative to its body): several colliders per body, offset from the body
    # origin.  Absent: one collider per body at its origin, described by shape_type / dims / friction / restitution above.
    collider_body: np.ndarray | None = None          # int32[C] the body of every collider
    local_position: np.ndarray | None = None         # float64[C,3] in the body frame
    local_rotation: np.ndarray | None = None         # float64[C,4] (x, y, z, w)
    collider_shape: np.ndarray | None = None         # int32[C]
    collider_dims: np.ndarray | None = None          # float64[C,3]
    collider_friction: np.ndarray | None = None      # float64[C]
    collider_restitution: np.ndarray | None = None   # float64[C]
    # optional convex hull table (api.ConvexHulls): colliders of shape SHAPE_CONVEX_HULL name a hull by index in dims[0]
    hulls: api.ConvexHulls | None = None

    @property
    def compound(self) -> bool:
        return self.collider_body is not None

    def collider_poses(self, bodies: api.Bodies) -> tuple[np.ndarray, np.ndarray]:
        """The colliders' world poses from the body poses (what the reference's Prepare stage propagates): position = body position +
        R * local position, rotation = R * local rotation.  Evaluated in float64 and rounded to the body columns' scalar."""
        b = self.collider_body
        p = np.asarray(bodies.position, dtype=np.float64)[b]
        q = np.asarray(bodies.rotation, dtype=np.float64)[b]
        pos = p + _qrot_rows(q, self.local_position)
        rot = _qmul_rows(q, self.local_rotation)
        return pos.astype(bodies.position.dtype), rot.astype(bodies.rotation.dtype)

    def collider_velocities(self, bodies: api.Bodies, position: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
        """The body's velocity at every collider, for the swept AABB (collider/backend.rs:570-585): v + w x (pos - body pos - R com)."""
        b = self.collider_body
        f = lambda a: np.asarray(a, dtype=np.float64)[b]
        off = np.asarray(position, dtype=np.float64) - f(bodies.position) - _qrot_rows(f(bodies.rotation), f(bodies.center_of_mass))
        w = f(bodies.angular_velocity)
        lv = f(bodies.linear_velocity) + np.cross(w, off)
        return lv.astype(bodies.position.dtype), w.astype(bodies.position.dtype)


def _cuboid_mass(he: np.ndarray, density: float = 1.0):
    """mass and local inverse inertia (diagonal) of solid cuboids given half extents [n,3]."""
    size = 2.0 * he
    m = density * size[:, 0] * size[:, 1] * size[:, 2]
    ix = m / 12.0 * (size[:, 1] ** 2 + size[:, 2] ** 2)
    iy = m / 12.0 * (size[:, 0] ** 2 + size[:, 2] ** 2)
    iz = m / 12.0 * (size[:, 0] ** 2 + size[:, 1] ** 2)
    return m, np.stack([ix, iy, iz], axis=1)


def _capsule_mass(radius: np.ndarray, half_length: np.ndarray, density: float = 1.0):
    """mass and local inertia (diagonal, axis along local y) of solid capsules: a cylinder of length 2 half_length plus two hemispheres.
    Closed form, PARITY UNPINNED: the reference takes capsule mass properties from bevy_heavy, which is not vendored."""
    r, L = np.asarray(radius, dtype=np.float64), 2.0 * np.asarray(half_length, dtype=np.float64)
    m_cyl = density * np.pi * r * r * L
    m_sph = density * 4.0 / 3.0 * np.pi * r ** 3
    iy = m_cyl * r * r / 2.0 + m_sph * 2.0 * r * r / 5.0
    ix = m_cyl * (L * L / 12.0 + r * r / 4.0) + m_sph * (2.0 * r * r / 5.0 + L * L / 4.0 + 3.0 * L * r / 8.0)
    return m_cyl + m_sph, np.stack([ix, iy, ix], axis=1)


def hull_mass(vertices, faces, density: float = 1.0):
    """mass, centre of mass and inertia tensor (about the centre of mass, 3x3) of a solid convex polyhedron: a sum of tetrahedra from the vertex
    mean over the fan triangles of every face, each with the canonical tetrahedron covariance.  PARITY UNPINNED: the reference takes hull mass
    properties from bevy_heavy / parry, which are not vendored."""
    v = np.asarray(vertices, dtype=np.float64)
    ref = v.mean(axis=0)
    c0 = np.array([[2.0, 1.0, 1.0], [1.0, 2.0, 1.0], [1.0, 1.0, 2.0]]) / 120.0
    vol, first, cov = 0.0, np.zeros(3), np.zeros((3, 3))
    for f in faces:
        f = [int(i) for i in f]
        for k in range(1, len(f) - 1):
            A = np.stack([v[f[0]] - ref, v[f[k]] - ref, v[f[k + 1]] - ref], axis=1)
            det = float(np.linalg.det(A))
            vol += det / 6.0
            first += det / 24.0 * A.sum(axis=1)
            cov += det * (A @ c0 @ A.T)
    m = density * vol
    com_rel = first / vol
    cov_c = density * cov - m * np.outer(com_rel, com_rel)
    inertia = np.trace(cov_c) * np.eye(3) - cov_c
    return m, ref + com_rel, inertia


def _assemble(name, pos, rot, kind, he, shape_type, scalar, friction=0.5, restitution=0.0, linvel=None, angvel=None, density=1.0, **extra) -> Scene:
    n = pos.shape[0]
    s = np.dtype(scalar)
    he = np.asarray(he, dtype=np.float64)
    m, inertia = _cuboid_mass(he, density)
    sph = shape_type == SHAPE_SPHERE
    if sph.any():
        r = he[sph, 0]
        ms = density * 4.0 / 3.0 * np.pi * r ** 3
        m[sph] = ms
        inertia[sph] = (0.4 * ms * r * r)[:, None]
    cap = shape_type == SHAPE_CAPSULE
    if cap.any():
        m[cap], inertia[cap] = _capsule_mass(he[cap, 0], he[cap, 1], density)
    dyn = kind == api.BODY_DYNAMIC
    inv_m = np.where(dyn, 1.0 / m, 0.0)
    inv_i = np.zeros((n, 6))
    inv_i[:, 0] = np.where(dyn, 1.0 / inertia[:, 0], 0.0)
    inv_i[:, 3] = np.where(dyn, 1.0 / inertia[:, 1], 0.0)
    inv_i[:, 5] = np.where(dyn, 1.0 / inertia[:, 2], 0.0)
    z3 = np.zeros((n, 3))
    bodies = api.Bodies(
        kind=np.ascontiguousarray(kind, dtype=np.uint8), position=np.ascontiguousarray(pos, dtype=s), rotation=np.ascontiguousarray(rot, dtype=s),
        linear_velocity=np.ascontiguousarray(z3 if linvel is None else linvel, dtype=s),
        angular_velocity=np.ascontiguousarray(z3 if angvel is None else angvel, dtype=s),
        inverse_mass=np.ascontiguousarray(inv_m, dtype=s), inverse_inertia_local=np.ascontiguousarray(inv_i, dtype=s),
        center_of_mass=np.zeros((n, 3), dtype=s))
    fr = np.full(n, friction, dtype=np.float64) if np.isscalar(friction) else np.asarray(friction, dtype=np.float64)
    rs = np.full(n, restitution, dtype=np.float64) if np.isscalar(restitution) else np.asarray(restitution, dtype=np.float64)
    return Scene(name, bodies, np.ascontiguousarray(shape_type, dtype=np.int32), np.ascontiguousarray(he), fr, rs, **extra)


def cube_stack(nx: int, ny: int, nz: int, size: float = 1.0, gap: float = 0.05, overlap: float = 0.01, brick: bool = True,
               scalar=np.float32, ground_half=(0.0, 0.5, 0.0), restitution: float = 0.0) -> Scene:
    """A box stack of nx*ny*nz dynamic cubes on a static ground slab (body 0).

    brick=True  — odd layers are shifted by half a pitch in x and z and hold (nx-1)*(nz-1) cubes, so every cube of an
                  odd layer rests on four cubes and every inner cube of an even layer on four: one coupled pile (one
                  island), ~4 manifolds per cube (the headline scene; 51x40x50 gives exactly 100 000 cubes).
    brick=False — aligned columns with a lateral gap, like crates/avian3d/examples/cubes.rs:42-52 (spacing 2.05 for
                  size-2 cubes): independent columns.
    Layers start `overlap` into each other like benches/src/dim3/large_pyramid.rs (y spacing 0.99 for unit cubes),
    so every contact exists on the first step.  Spawn order is x-major so the broad phase's persistent order starts
    sorted along x (the reference's insertion sort stays linear)."""
    pitch = size + gap
    xs = np.arange(nx) * pitch
    zs = np.arange(nz) * pitch
    layers = []
    for k in range(ny):
        y = size * 0.5 + k * (size - overlap) - overlap
        if brick and (k % 2):
            lx, lz = xs[:-1] + pitch * 0.5, zs[:-1] + pitch * 0.5   # (nx-1) x (nz-1) cubes, each over four cubes below
        else:
            lx, lz = xs, zs
        X, Z = np.meshgrid(lx, lz, indexing="ij")
        layers.append(np.stack([X.ravel(), np.full(X.size, y), Z.ravel()], axis=1))
    pos = np.concatenate(layers)
    pos = pos[np.lexsort((pos[:, 2], pos[:, 1], pos[:, 0]))]   # x-major spawn order
    n = pos.shape[0]
    # ground slab: top face at y = 0
    gx = ground_half[0] or (nx * pitch + 10.0)
    gz = ground_half[2] or (nz * pitch + 10.0)
    gpos = np.array([[xs.mean() if nx else 0.0, -ground_half[1], zs.mean() if nz else 0.0]])
    pos = np.concatenate([gpos, pos])
    he = np.concatenate([[[gx, ground_half[1], gz]], np.full((n, 3), size * 0.5)])
    kind = np.concatenate([[api.BODY_STATIC], np.full(n, api.BODY_DYNAMIC)])
    rot = np.tile(np.array([0.0, 0.0, 0.0, 1.0]), (n + 1, 1))
    st = np.full(n + 1, SHAPE_CUBOID)
    return _assemble(f"cube_stack_{nx}x{ny}x{nz}{'_brick' if brick else ''}", pos, rot, kind, he, st, scalar, restitution=restitution)


def cubes_example(n_side: int = 4, scalar=np.float32) -> Scene:
    """crates/avian3d/examples/cubes.rs:25-52: ground = unit cuboid scaled (100,1,100) at y=-2; n_side^3 cubes of
    side 2.0 at spacing 2.05, y offset +... (the example uses x,z in -2..2 and y in -2..2 plus 10).  n_side=3 is
    BASELINE config 1's reduced scene, n_side=4 the literal example."""
    lo = -(n_side // 2)
    idx = np.arange(lo, lo + n_side)
    X, Y, Z = np.meshgrid(idx, idx, idx, indexing="ij")
    cube_size, spacing = 2.0, 2.05
    pos = np.stack([X.ravel() * spacing, (Y.ravel() + 2) * spacing + 0.025, Z.ravel() * spacing], axis=1).astype(np.float64)
    n = pos.shape[0]
    pos = np.concatenate([[[0.0, -2.0, 0.0]], pos])
    he = np.concatenate([[[50.0, 0.5, 50.0]], np.full((n, 3), cube_size * 0.5)])
    kind = np.concatenate([[api.BODY_STATIC], np.full(n, api.BODY_DYNAMIC)])
    rot = np.tile(np.array([0.0, 0.0, 0.0, 1.0]), (n + 1, 1))
    return _assemble(f"cubes_{n_side}x{n_side}x{n_side}", pos, rot, kind, he, np.full(n + 1, SHAPE_CUBOID), scalar)


def falling_spheres(n: int, seed: int = 42, box=(200.0, 50.0, 200.0), radius: float = 0.5, scalar=np.float64) -> Scene:
    """BASELINE config 5: n spheres r=0.5 uniformly random in a box above a ground slab, zero velocity."""
    rng = np.random.default_rng(seed)
    pos = rng.uniform([0, radius + 0.01, 0], [box[0], box[1], box[2]], size=(n, 3))
    order = np.argsort(pos[:, 0], kind="stable")
    pos = pos[order]
    pos = np.concatenate([[[box[0] * 0.5, -0.5, box[2] * 0.5]], pos])
    he = np.concatenate([[[box[0] * 0.5 + 10, 0.5, box[2] * 0.5 + 10]], np.full((n, 3), radius)])
    kind = np.concatenate([[api.BODY_STATIC], np.full(n, api.BODY_DYNAMIC)])
    rot = np.tile(np.array([0.0, 0.0, 0.0, 1.0]), (n + 1, 1))
    st = np.concatenate([[SHAPE_CUBOID], np.full(n, SHAPE_SPHERE)])
    return _assemble(f"spheres_{n}", pos, rot, kind, he, st, scalar)


def _quat_axis_angle(axis, angle):
    axis = np.asarray(axis, dtype=np.float64)
    axis = axis / np.linalg.norm(axis)
    s = np.sin(angle * 0.5)
    return np.array([axis[0] * s, axis[1] * s, axis[2] * s, np.cos(angle * 0.5)])


# one ragdoll: (name, half extents, centre offset, parent, joint type, anchor in parent frame (world offset from parent centre))
_RAGDOLL = [
    ("pelvis", (0.15, 0.10, 0.10), (0.0, 1.00, 0.0), -1, None),
    ("spine", (0.15, 0.12, 0.10), (0.0, 1.24, 0.0), 0, "S"),
    ("chest", (0.17, 0.13, 0.11), (0.0, 1.51, 0.0), 1, "S"),
    ("neck", (0.05, 0.05, 0.05), (0.0, 1.70, 0.0), 2, "S"),
    ("head", (0.10, 0.11, 0.10), (0.0, 1.87, 0.0), 3, "S"),
    ("l_upper_arm", (0.14, 0.05, 0.05), (-0.33, 1.58, 0.0), 2, "S"),
    ("l_fore_arm", (0.13, 0.04, 0.04), (-0.61, 1.58, 0.0), 5, "R"),
    ("l_hand", (0.05, 0.03, 0.04), (-0.80, 1.58, 0.0), 6, "S"),
    ("r_upper_arm", (0.14, 0.05, 0.05), (0.33, 1.58, 0.0), 2, "S"),
    ("r_fore_arm", (0.13, 0.04, 0.04), (0.61, 1.58, 0.0), 8, "R"),
    ("r_hand", (0.05, 0.03, 0.04), (0.80, 1.58, 0.0), 9, "S"),
    ("l_thigh", (0.07, 0.20, 0.07), (-0.09, 0.69, 0.0), 0, "S"),
    ("l_shin", (0.06, 0.19, 0.06), (-0.09, 0.29, 0.0), 11, "R"),
    ("l_foot", (0.06, 0.04, 0.11), (-0.09, 0.05, 0.04), 12, "S"),
    ("r_thigh", (0.07, 0.20, 0.07), (0.09, 0.69, 0.0), 0, "S"),
    ("r_shin", (0.06, 0.19, 0.06), (0.09, 0.29, 0.0), 14, "R"),
    ("r_foot", (0.06, 0.04, 0.11), (0.09, 0.05, 0.04), 15, "S"),
]


# the limbs whose long axis is the body's local y: the capsule's axis without a rotated collider frame
_CAPSULE_LIMBS = ("l_thigh", "l_shin", "r_thigh", "r_shin")


def ragdoll_field(count: int, pitch: float = 8.0, drop_height: float = 2.0, seed: int = 1234, scalar=np.float32, limbs: str = "cuboid") -> Scene:
    """BASELINE config 4 (SURVEY §8d): `count` ragdolls on a square grid, 17 cuboid bodies and 16 joints each —
    spherical joints (swing +-60 deg, twist +-30 deg) for neck/spine/shoulders/hips/wrists/ankles, revolute joints
    (0..120 deg) for elbows and knees; every joint disables collision between its bodies (JointCollisionDisabled).
    A small deterministic pose jitter (PCG64, seed) breaks symmetry.
    limbs="capsule": thighs and shins are capsules along their long axis (local y), radius = the smaller half extent of the cross-section,
    half length = half height - radius (the same height as the cuboid).  The arms' long axis is local x, and a capsule's segment runs along
    the collider's local y: they stay cuboids, since turning their bodies would change the joint frames."""
    if limbs not in ("cuboid", "capsule"):
        raise ValueError(f"limbs must be 'cuboid' or 'capsule', not {limbs!r}")
    rng = np.random.default_rng(seed)
    side = int(np.ceil(np.sqrt(count)))
    nb = len(_RAGDOLL)
    pos, he, rot = [], [], []
    sj = {k: [] for k in ("b1", "b2", "a1", "a2")}
    rj = {k: [] for k in ("b1", "b2", "a1", "a2")}
    disabled = []
    for r in range(count):
        gx, gz = (r % side) * pitch, (r // side) * pitch
        base = 1 + r * nb
        yaw = _quat_axis_angle((0, 1, 0), rng.uniform(-np.pi, np.pi))
        tilt = _quat_axis_angle((rng.uniform(-1, 1), 0, rng.uniform(-1, 1) + 1e-3), np.deg2rad(rng.uniform(0, 5)))
        q = _qmul(tilt, yaw)
        for i, (_, h, c, parent, jt) in enumerate(_RAGDOLL):
            cw = _qrot(q, np.array(c) - np.array([0, 1.0, 0])) + np.array([gx, 1.0 + drop_height, gz])
            pos.append(cw)
            he.append(h)
            rot.append(q)
            if parent >= 0:
                pc = np.array(_RAGDOLL[parent][2])
                cc = np.array(c)
                # anchor: the point between parent and child along the segment, at the child's near face
                anchor_local_world = (pc + cc) * 0.5
                a1 = anchor_local_world - pc   # in the (common) body frame since all bodies share rotation q
                a2 = anchor_local_world - cc
                d = sj if jt == "S" else rj
                d["b1"].append(base + parent)
                d["b2"].append(base + i)
                d["a1"].append(a1)
                d["a2"].append(a2)
                disabled.append((base + parent, base + i))
    n = len(pos)
    pos = np.concatenate([[[side * pitch * 0.5, -0.5, side * pitch * 0.5]], np.array(pos)])
    he = np.concatenate([[[side * pitch * 0.5 + 20, 0.5, side * pitch * 0.5 + 20]], np.array(he)])
    rot = np.concatenate([[[0, 0, 0, 1.0]], np.array(rot)])
    kind = np.concatenate([[api.BODY_STATIC], np.full(n, api.BODY_DYNAMIC)])
    s = np.dtype(scalar)

    def joints(d, revolute):
        m = len(d["b1"])
        j = api.Joints(body1=np.array(d["b1"], dtype=np.int32), body2=np.array(d["b2"], dtype=np.int32),
                       local_anchor1=np.ascontiguousarray(d["a1"], dtype=s).reshape(m, 3), local_anchor2=np.ascontiguousarray(d["a2"], dtype=s).reshape(m, 3))
        j.limit_enabled = np.full(m, 1 if revolute else 3, dtype=np.uint8)
        if revolute:
            j.axis = np.tile(np.array([1.0, 0, 0], dtype=s), (m, 1))
            j.limit_min = np.zeros(m, dtype=s)
            j.limit_max = np.full(m, np.deg2rad(120.0), dtype=s)
        else:
            j.limit_min = np.full(m, -np.deg2rad(60.0), dtype=s)
            j.limit_max = np.full(m, np.deg2rad(60.0), dtype=s)
            j.limit2_min = np.full(m, -np.deg2rad(30.0), dtype=s)
            j.limit2_max = np.full(m, np.deg2rad(30.0), dtype=s)
        j.force = np.zeros((m, 3), dtype=s)
        j.torque = np.zeros((m, 3), dtype=s)
        return j

    js = api.JointSet({api.JOINT_REVOLUTE: joints(rj, True), api.JOINT_SPHERICAL: joints(sj, False)})
    dis = np.array([(min(a, b) << 32) | max(a, b) for a, b in disabled], dtype=np.uint64)
    shape = np.full(n + 1, SHAPE_CUBOID)
    name = f"ragdolls_{count}"
    if limbs == "capsule":
        name += "_capsule_limbs"
        limb = np.array([part[0] in _CAPSULE_LIMBS for part in _RAGDOLL] * count)
        rows = 1 + np.flatnonzero(limb)
        r = np.minimum(he[rows, 0], he[rows, 2])
        he[rows] = np.stack([r, np.maximum(he[rows, 1] - r, 0.0), np.zeros_like(r)], axis=1)
        shape[rows] = SHAPE_CAPSULE
    return _assemble(name, pos, rot, kind, he, shape, scalar, joints=js, joint_disabled_body_pairs=dis)


def capsule_pile(n: int, seed: int = 7, layers: int = 10, capsule_share: float = 0.8, sphere_share: float = 0.1, scalar=np.float32) -> Scene:
    """A seeded pile of n dynamic bodies falling onto a static ground cuboid (body 0): mostly capsules (radius 0.15..0.3, half length
    0.2..0.5) at uniformly random orientations, plus spheres (radius 0.2..0.4) and cubes (half extent 0.2..0.4, random orientation), on a
    jittered grid of `layers` layers that starts without overlaps.  Every pair type meets: capsule against capsule, sphere, cube and ground.
    Spawn order is x-major like cube_stack."""
    rng = np.random.default_rng(seed)
    u = rng.uniform(size=n)
    shape = np.where(u < capsule_share, SHAPE_CAPSULE, np.where(u < capsule_share + sphere_share, SHAPE_SPHERE, SHAPE_CUBOID))
    he = np.zeros((n, 3))
    cap, sph, box = shape == SHAPE_CAPSULE, shape == SHAPE_SPHERE, shape == SHAPE_CUBOID
    he[cap, 0] = rng.uniform(0.15, 0.3, size=cap.sum())
    he[cap, 1] = rng.uniform(0.2, 0.5, size=cap.sum())
    he[sph] = rng.uniform(0.2, 0.4, size=sph.sum())[:, None]
    he[box] = rng.uniform(0.2, 0.4, size=box.sum())[:, None]
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[sph] = [0.0, 0.0, 0.0, 1.0]
    pitch = 2.0 * (0.5 + 0.3) + 0.2            # the longest capsule plus a gap, in every direction
    side = int(np.ceil(np.sqrt(n / layers)))
    k = np.arange(n)
    layer, cell = k // (side * side), k % (side * side)
    pos = np.stack([(cell // side) * pitch, 0.9 + layer * pitch, (cell % side) * pitch], axis=1) + rng.uniform(-0.05, 0.05, size=(n, 3))
    order = np.lexsort((pos[:, 2], pos[:, 1], pos[:, 0]))
    pos, q, he, shape = pos[order], q[order], he[order], shape[order]
    extent = side * pitch
    pos = np.concatenate([[[extent * 0.5, -0.5, extent * 0.5]], pos])
    he = np.concatenate([[[extent * 0.5 + 10.0, 0.5, extent * 0.5 + 10.0]], he])
    rot = np.concatenate([[[0.0, 0.0, 0.0, 1.0]], q])
    kind = np.concatenate([[api.BODY_STATIC], np.full(n, api.BODY_DYNAMIC)])
    return _assemble(f"capsule_pile_{n}", pos, rot, kind, he, np.concatenate([[SHAPE_CUBOID], shape]), scalar)


def _qrot_rows(q, v):
    """rotate the rows of v [n,3] by the rows of q [n,4] (glam's Quat * Vec3)"""
    b, w = q[:, :3], q[:, 3:4]
    return v * (w * w - np.sum(b * b, axis=1, keepdims=True)) + b * (2.0 * np.sum(v * b, axis=1, keepdims=True)) + np.cross(b, v) * (2.0 * w)


def _qmul_rows(a, b):
    ax, ay, az, aw = a.T
    bx, by, bz, bw = b.T
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], axis=1)


def with_collider_table(scene: Scene, offset=None, center_of_mass=None) -> Scene:
    """A single-collider scene with an explicit collider table (one collider per body).  offset [B,3] (None = 0): every body's origin moves
    by -R * offset, its collider sits at local position `offset` and its centre of mass at `center_of_mass` (None = offset), so the collider
    and the centre of mass stay where they were in the world: the same physical scene, expressed from other body origins."""
    import dataclasses
    n = int(scene.bodies.count)
    d = np.zeros((n, 3)) if offset is None else np.asarray(offset, dtype=np.float64).reshape(n, 3)
    com = d if center_of_mass is None else np.asarray(center_of_mass, dtype=np.float64).reshape(n, 3)
    b = scene.bodies
    s = b.position.dtype
    q = np.asarray(b.rotation, dtype=np.float64)
    bodies = dataclasses.replace(b, position=np.ascontiguousarray(np.asarray(b.position, dtype=np.float64) - _qrot_rows(q, d), dtype=s),
                                 center_of_mass=np.ascontiguousarray(com, dtype=s))
    return dataclasses.replace(scene, name=scene.name + "_table", bodies=bodies, collider_body=np.arange(n, dtype=np.int32), local_position=d.copy(),
                               local_rotation=np.tile([0.0, 0.0, 0.0, 1.0], (n, 1)), collider_shape=scene.shape_type.copy(),
                               collider_dims=scene.dims.copy(), collider_friction=scene.friction.copy(), collider_restitution=scene.restitution.copy())


def _part_mass(shape: int, dims, density: float = 1.0):
    """mass and local inertia (diagonal) of one part"""
    he = np.asarray(dims, dtype=np.float64).reshape(1, 3)
    if shape == SHAPE_SPHERE:
        r = he[0, 0]
        m = density * 4.0 / 3.0 * np.pi * r ** 3
        return m, np.full(3, 0.4 * m * r * r)
    if shape == SHAPE_CAPSULE:
        m, i = _capsule_mass(he[:, 0], he[:, 1], density)
        return float(m[0]), i[0]
    m, i = _cuboid_mass(he, density)
    return float(m[0]), i[0]


def _quat_matrix(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def compound_mass(parts, density: float = 1.0):
    """(mass, centre of mass, inertia tensor about it) of a body made of parts [(shape, dims, local position, local rotation)]: the parts'
    masses summed, the mass-weighted centre, each part's inertia rotated into the body frame and moved by the parallel-axis theorem.
    Closed form, PARITY UNPINNED: the reference takes mass properties from bevy_heavy, which is not vendored."""
    ms, cs, Is = [], [], []
    for shape, dims, lp, lr in parts:
        m, i = _part_mass(shape, dims, density)
        R = _quat_matrix(lr)
        ms.append(m)
        cs.append(np.asarray(lp, dtype=np.float64))
        Is.append(R @ np.diag(i) @ R.T)
    M = float(sum(ms))
    c = sum(m * p for m, p in zip(ms, cs)) / M
    I = np.zeros((3, 3))
    for m, p, i in zip(ms, cs, Is):
        d = p - c
        I += i + m * (np.dot(d, d) * np.eye(3) - np.outer(d, d))
    return M, c, I


_Z90 = (0.0, 0.0, np.sin(np.pi / 4), np.cos(np.pi / 4))   # local y -> -x: a capsule lying along x


def _compound_parts(kind: str, rng):
    """(parts, origin): parts [(shape, dims, position, rotation)] in a design frame, origin = the body origin in that frame"""
    I4 = (0.0, 0.0, 0.0, 1.0)
    if kind == "table":
        w, d, t, h, leg = rng.uniform(0.5, 0.8), rng.uniform(0.4, 0.6), 0.06, rng.uniform(0.3, 0.5), 0.05
        parts = [(SHAPE_CUBOID, (w, t, d), (0.0, h + t, 0.0), I4)]
        for sx in (-1, 1):
            for sz in (-1, 1):
                parts.append((SHAPE_CUBOID, (leg, h * 0.5, leg), (sx * (w - leg), h * 0.5, sz * (d - leg)), I4))
        return parts, np.array([-w, 0.0, -d])                      # origin at a foot corner
    if kind == "dumbbell":
        r, hl, rb = rng.uniform(0.06, 0.1), rng.uniform(0.3, 0.5), rng.uniform(0.18, 0.25)
        parts = [(SHAPE_CAPSULE, (r, hl, 0.0), (0.0, 0.0, 0.0), _Z90), (SHAPE_SPHERE, (rb, 0, 0), (-hl, 0.0, 0.0), I4),
                 (SHAPE_SPHERE, (rb * rng.uniform(0.7, 1.0), 0, 0), (hl, 0.0, 0.0), I4)]
        return parts, np.array([-hl, 0.0, 0.0])                    # origin at one weight's centre
    a, b, t = rng.uniform(0.3, 0.5), rng.uniform(0.3, 0.5), rng.uniform(0.1, 0.15)   # L-block: a foot and an upright
    parts = [(SHAPE_CUBOID, (a, t, t), (a, t, 0.0), I4), (SHAPE_CUBOID, (t, b, t), (t, 2 * t + b, 0.0), I4)]
    return parts, np.zeros(3)                                       # origin at the corner of the foot


def compound_pile(n: int, seed: int = 11, scalar=np.float32, single_share: float = 0.0, layers: int = 4) -> Scene:
    """A seeded pile of n dynamic bodies of 2-5 parts over a static ground cuboid (body 0, one collider): tables (a top on four legs),
    dumbbells (two spheres on a capsule) and L-blocks, at random yaws on a jittered grid that starts without overlaps.  Every body's origin is
    away from its centre of mass (a foot corner, a weight's centre, the L's corner), and every third body also has an explicit centre-of-mass
    offset (CenterOfMass), which leaves the inertia about the parts' centre.  single_share: that share of the bodies are single cuboids,
    spheres or capsules at their body's origin instead.  Mass properties: compound_mass (PARITY UNPINNED)."""
    rng = np.random.default_rng(seed)
    pitch = 2.2
    side = int(np.ceil(np.sqrt(n / layers)))
    pos, rot, com, inv_m, inv_i = [], [], [], [], []
    cb, lp, lr, cs, cd = [], [], [], [], []
    extent = side * pitch
    ground = (SHAPE_CUBOID, (extent * 0.5 + 10.0, 0.5, extent * 0.5 + 10.0))
    for i in range(n):
        layer, cell = i // (side * side), i % (side * side)
        at = np.array([(cell // side) * pitch, 1.0 + layer * pitch, (cell % side) * pitch]) + rng.uniform(-0.05, 0.05, 3)
        if rng.uniform() < single_share:
            k = int(rng.integers(0, 3))
            dims = (rng.uniform(0.2, 0.4),) * 3 if k != SHAPE_CAPSULE else (rng.uniform(0.15, 0.25), rng.uniform(0.2, 0.4), 0.0)
            parts, origin = [(k, dims, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0))], np.zeros(3)
        else:
            parts, origin = _compound_parts(("table", "dumbbell", "lblock")[int(rng.integers(0, 3))], rng)
        M, c, I = compound_mass(parts)
        q = _quat_axis_angle((0, 1, 0), rng.uniform(-np.pi, np.pi))
        c_local = c - origin
        explicit = len(parts) > 1 and i % 3 == 0
        com.append(c_local + (rng.uniform(-0.05, 0.05, 3) if explicit else 0.0))
        pos.append(at - _qrot(q, c_local))
        rot.append(q)
        Iinv = np.linalg.inv(I)
        inv_m.append(1.0 / M)
        inv_i.append([Iinv[0, 0], Iinv[0, 1], Iinv[0, 2], Iinv[1, 1], Iinv[1, 2], Iinv[2, 2]])
        for shape, dims, p, r in parts:
            cb.append(i + 1)
            lp.append(np.asarray(p) - origin)
            lr.append(r)
            cs.append(shape)
            cd.append(dims)
    B = n + 1
    s = np.dtype(scalar)
    kind = np.concatenate([[api.BODY_STATIC], np.full(n, api.BODY_DYNAMIC)]).astype(np.uint8)
    P = np.concatenate([[[extent * 0.5, -0.5, extent * 0.5]], np.array(pos).reshape(-1, 3)])
    R = np.concatenate([[[0.0, 0.0, 0.0, 1.0]], np.array(rot).reshape(-1, 4)])
    z3 = np.zeros((B, 3))
    bodies = api.Bodies(kind=kind, position=np.ascontiguousarray(P, dtype=s), rotation=np.ascontiguousarray(R, dtype=s),
                        linear_velocity=np.ascontiguousarray(z3, dtype=s), angular_velocity=np.ascontiguousarray(z3, dtype=s),
                        inverse_mass=np.ascontiguousarray(np.concatenate([[0.0], inv_m]), dtype=s),
                        inverse_inertia_local=np.ascontiguousarray(np.concatenate([np.zeros((1, 6)), np.array(inv_i).reshape(-1, 6)]), dtype=s),
                        center_of_mass=np.ascontiguousarray(np.concatenate([np.zeros((1, 3)), np.array(com).reshape(-1, 3)]), dtype=s))
    C_ = len(cb) + 1
    cshape = np.concatenate([[ground[0]], cs]).astype(np.int32)
    cdims = np.concatenate([[ground[1]], np.array(cd, dtype=np.float64).reshape(-1, 3)])
    cbody = np.concatenate([[0], cb]).astype(np.int32)
    first = np.searchsorted(cbody, np.arange(B))   # the per-body columns describe each body's first collider
    return Scene(f"compound_pile_{n}", bodies, np.ascontiguousarray(cshape[first]), np.ascontiguousarray(cdims[first]), np.full(B, 0.5), np.zeros(B),
                 collider_body=cbody, local_position=np.concatenate([np.zeros((1, 3)), np.array(lp).reshape(-1, 3)]),
                 local_rotation=np.concatenate([[[0.0, 0.0, 0.0, 1.0]], np.array(lr).reshape(-1, 4)]), collider_shape=cshape,
                 collider_dims=np.ascontiguousarray(cdims), collider_friction=np.full(C_, 0.5), collider_restitution=np.zeros(C_))


def _qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz])


def _qrot(q, v):
    b = q[:3]
    return v * (q[3] * q[3] - b @ b) + b * (2.0 * (v @ b)) + np.cross(b, v) * (2.0 * q[3])


def spherical_chain(links: int = 100, scalar=np.float32) -> Scene:
    """crates/avian3d/examples/chain_3d.rs:36-72: a kinematic anchor and `links` small dynamic spheres joined by
    spherical joints (local_anchor2 = +y * 1.1 * radius*2), collision between neighbours disabled."""
    radius = 0.03 * 2.0  # particle_radius used by the example scaled to metres here
    pos = [np.array([0.0, 0.0, 0.0])]
    for i in range(links):
        pos.append(np.array([0.0, -(i + 1) * (radius * 2.0 + 0.02), 0.0]))
    n = len(pos)
    pos = np.array(pos)
    he = np.full((n, 3), radius)
    kind = np.concatenate([[api.BODY_KINEMATIC], np.full(links, api.BODY_DYNAMIC)])
    rot = np.tile(np.array([0.0, 0.0, 0.0, 1.0]), (n, 1))
    s = np.dtype(scalar)
    b1 = np.arange(0, links, dtype=np.int32)
    b2 = np.arange(1, links + 1, dtype=np.int32)
    j = api.Joints(body1=b1, body2=b2, local_anchor1=np.zeros((links, 3), dtype=s),
                   local_anchor2=np.tile(np.array([0.0, radius * 2.0 + 0.02, 0.0], dtype=s), (links, 1)))
    j.compliance0 = np.full(links, 1e-5, dtype=s)
    j.force = np.zeros((links, 3), dtype=s)
    j.torque = np.zeros((links, 3), dtype=s)
    dis = np.array([(int(a) << 32) | int(b) for a, b in zip(b1, b2)], dtype=np.uint64)
    sc = _assemble(f"chain_{links}", pos, rot, kind, he, np.full(n, SHAPE_SPHERE), scalar, joints=api.JointSet({api.JOINT_SPHERICAL: j}),
                   joint_disabled_body_pairs=dis)
    # a kinematic body keeps its collider mass (SolverBodyInertia::new keeps inv_mass, dominance 128)
    return sc


# ---- convex hulls (DESIGN.md §7k) ------------------------------------------------------------------------------------------------------

def _polygon_faces(points, simplices, equations, tol: float = 1e-9):
    """Qhull's triangles merged into polygon faces: triangles on the same plane become one loop of their vertices, counter-clockwise seen from
    outside (ordered by angle about the face centre)."""
    faces, used = [], np.zeros(len(simplices), dtype=bool)
    for i in range(len(simplices)):
        if used[i]:
            continue
        same = np.nonzero(np.all(np.abs(equations - equations[i]) < tol, axis=1) & ~used)[0]
        used[same] = True
        idx = np.unique(simplices[same].ravel())
        n = equations[i, :3]
        c = points[idx].mean(axis=0)
        u = points[idx[0]] - c
        u /= np.linalg.norm(u)
        w = np.cross(n, u)
        ang = np.arctan2((points[idx] - c) @ w, (points[idx] - c) @ u)
        faces.append([int(k) for k in idx[np.argsort(ang)]])
    return faces


def convex_hull_of(points):
    """(vertices, faces) of the convex hull of a point cloud: scipy's Qhull with coplanar triangles merged, vertices renumbered to those on the hull"""
    from scipy.spatial import ConvexHull
    pts = np.asarray(points, dtype=np.float64)
    h = ConvexHull(pts)
    keep = np.unique(h.simplices.ravel())
    remap = {int(k): i for i, k in enumerate(keep)}
    faces = _polygon_faces(pts, h.simplices, h.equations)
    return pts[keep], [[remap[k] for k in f] for f in faces]


def regular_solids(scale: float = 0.3):
    """tetrahedron, octahedron and icosahedron of circumradius `scale`, and a 32-sided prism (radius scale, half height scale / 2)"""
    t = np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]], dtype=np.float64) / np.sqrt(3.0)
    o = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], dtype=np.float64)
    g = (1 + np.sqrt(5.0)) / 2
    ico = np.array([[0, s1, s2 * g] for s1 in (-1, 1) for s2 in (-1, 1)] + [[s1, s2 * g, 0] for s1 in (-1, 1) for s2 in (-1, 1)]
                   + [[s2 * g, 0, s1] for s1 in (-1, 1) for s2 in (-1, 1)], dtype=np.float64)
    ico /= np.linalg.norm(ico[0])
    out = [convex_hull_of(x * scale) for x in (t, o, ico)]
    k = 32
    a = 2 * np.pi * np.arange(k) / k
    ring = np.stack([np.cos(a) * scale, np.zeros(k), np.sin(a) * scale], axis=1)
    v = np.concatenate([ring + [0, -scale / 2, 0], ring + [0, scale / 2, 0]])
    faces = [list(range(k)), list(range(2 * k - 1, k - 1, -1))]   # bottom seen from below, top seen from above
    faces += [[i, (i + 1) % k, k + (i + 1) % k, k + i][::-1] for i in range(k)]
    out.append((v, _orient(v, faces)))
    return out


def _orient(v, faces):
    """every loop counter-clockwise seen from outside (reversed where its Newell normal points at the vertex mean)"""
    c = v.mean(axis=0)
    res = []
    for f in faces:
        p = v[f]
        n = np.cross(p - p.mean(axis=0), np.roll(p, -1, axis=0) - p.mean(axis=0)).sum(axis=0)
        res.append(list(f) if n @ (p.mean(axis=0) - c) > 0 else list(f)[::-1])
    return res


def _centred(v, faces):
    """the polyhedron moved so its centre of mass is the origin (the body's origin), with its mass properties"""
    m, com, inertia = hull_mass(v, faces)
    v = np.asarray(v, dtype=np.float64) - com
    return v, faces, m, inertia


def hull_pile(n: int, seed: int = 13, layers: int = 4, scalar=np.float32, kinds: int = 24) -> Scene:
    """A seeded pile of n dynamic bodies on a static ground cuboid (body 0): mostly convex hulls - `kinds` random hulls (Qhull over 10-18
    seeded points in a ball of radius 0.2-0.35, coplanar triangles merged into polygons), the regular tetrahedron, octahedron and icosahedron
    and a 32-sided prism - plus some cuboids, spheres and capsules, on a jittered grid that starts without overlaps.  Every hull is moved so its
    centre of mass is its origin; mass properties by hull_mass."""
    rng = np.random.default_rng(seed)
    polys = [convex_hull_of(rng.normal(size=(int(rng.integers(10, 19)), 3)) * rng.uniform(0.2, 0.35) / 2.0) for _ in range(kinds)]
    polys += regular_solids(0.3)
    table = [_centred(v, f) for v, f in polys]
    hulls = api.ConvexHulls.from_polyhedra([(v, f) for v, f, _, _ in table])
    u = rng.uniform(size=n)
    shape = np.where(u < 0.7, api.SHAPE_CONVEX_HULL, np.where(u < 0.8, SHAPE_CUBOID, np.where(u < 0.9, SHAPE_SPHERE, SHAPE_CAPSULE)))
    he = np.zeros((n, 3))
    hull = shape == api.SHAPE_CONVEX_HULL
    idx = rng.integers(0, len(table), size=n)
    he[hull, 0] = idx[hull]
    box, sph, cap = shape == SHAPE_CUBOID, shape == SHAPE_SPHERE, shape == SHAPE_CAPSULE
    he[box] = rng.uniform(0.15, 0.3, size=(box.sum(), 3))
    he[sph] = rng.uniform(0.15, 0.3, size=sph.sum())[:, None]
    he[cap, 0] = rng.uniform(0.1, 0.2, size=cap.sum())
    he[cap, 1] = rng.uniform(0.1, 0.3, size=cap.sum())
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    pitch = 1.2
    side = int(np.ceil(np.sqrt(n / layers)))
    k = np.arange(n)
    layer, cell = k // (side * side), k % (side * side)
    pos = np.stack([(cell // side) * pitch, 0.8 + layer * pitch, (cell % side) * pitch], axis=1) + rng.uniform(-0.05, 0.05, size=(n, 3))
    order = np.lexsort((pos[:, 2], pos[:, 1], pos[:, 0]))
    pos, q, he, shape = pos[order], q[order], he[order], shape[order]
    extent = side * pitch
    pos = np.concatenate([[[extent * 0.5, -0.5, extent * 0.5]], pos])
    he = np.concatenate([[[extent * 0.5 + 10.0, 0.5, extent * 0.5 + 10.0]], he])
    rot = np.concatenate([[[0.0, 0.0, 0.0, 1.0]], q])
    kind = np.concatenate([[api.BODY_STATIC], np.full(n, api.BODY_DYNAMIC)])
    shape = np.concatenate([[SHAPE_CUBOID], shape])
    sc = _assemble(f"hull_pile_{n}", pos, rot, kind, np.where((shape == api.SHAPE_CONVEX_HULL)[:, None], 0.5, he), shape, scalar, hulls=hulls)
    sc.dims = np.ascontiguousarray(he)
    _set_hull_mass(sc, table)
    return _own_velocities(sc)


def _own_velocities(sc: Scene) -> Scene:
    """_assemble hands a float64 scene one zero array for both velocity columns: give the angular velocity its own"""
    sc.bodies.angular_velocity = sc.bodies.angular_velocity.copy()
    return sc


def _set_hull_mass(sc: Scene, table) -> None:
    """the hull bodies' inverse mass and inverse inertia (upper triangle xx, xy, xz, yy, yz, zz) from the table's mass properties"""
    s = sc.bodies.inverse_mass.dtype
    for b in np.nonzero((sc.shape_type == api.SHAPE_CONVEX_HULL) & (sc.bodies.kind == api.BODY_DYNAMIC))[0]:
        _, _, m, inertia = table[int(sc.dims[b, 0])]
        inv = np.linalg.inv(inertia)
        sc.bodies.inverse_mass[b] = s.type(1.0 / m)
        sc.bodies.inverse_inertia_local[b] = np.array([inv[0, 0], inv[0, 1], inv[0, 2], inv[1, 1], inv[1, 2], inv[2, 2]]).astype(s)


def _box_points(he):
    return np.array([[(1 if m & 1 else -1) * he[0], (1 if m & 2 else -1) * he[1], (1 if m & 4 else -1) * he[2]] for m in range(8)], dtype=np.float64)


def _decomposed_scene(name, bodies_parts, ground_extent, at, yaw, scalar) -> Scene:
    """A compound scene from bodies given as convex decompositions: bodies_parts[i] = [(vertices, faces, position)] in the body's design
    frame, the ground cuboid as body 0.  Each part's vertices are centred on its centre of mass and the part sits at that point (its local
    position), like parry's Compound of a convex decomposition.  Every body's origin is its centre of mass; mass properties: hull_mass per
    part, moved by the parallel-axis theorem (PARITY UNPINNED)."""
    polys, cb, lp, cd = [], [], [], []
    pos, rot, inv_m, inv_i = [], [], [], []
    for i, parts in enumerate(bodies_parts):
        props = []
        for v, f, p in parts:
            m, com, inertia = hull_mass(np.asarray(v, dtype=np.float64) + p, f)
            props.append((m, com, inertia, np.asarray(v, dtype=np.float64) + p - com, f))
        M = sum(x[0] for x in props)
        c = sum(x[0] * x[1] for x in props) / M
        I = np.zeros((3, 3))
        for m, com, inertia, v, f in props:
            d = com - c
            I += inertia + m * (d @ d * np.eye(3) - np.outer(d, d))
            cb.append(i + 1)
            lp.append(com - c)
            cd.append([float(len(polys)), 0.0, 0.0])
            polys.append((v, f))
        q = _quat_axis_angle((0, 1, 0), yaw[i])
        pos.append(at[i])
        rot.append(q)
        Iinv = np.linalg.inv(I)
        inv_m.append(1.0 / M)
        inv_i.append([Iinv[0, 0], Iinv[0, 1], Iinv[0, 2], Iinv[1, 1], Iinv[1, 2], Iinv[2, 2]])
    n = len(bodies_parts)
    B, s = n + 1, np.dtype(scalar)
    g = np.asarray(ground_extent, dtype=np.float64)
    kind = np.concatenate([[api.BODY_STATIC], np.full(n, api.BODY_DYNAMIC)]).astype(np.uint8)
    P = np.concatenate([[[g[0], -0.5, g[2]]], np.array(pos).reshape(-1, 3)])
    R = np.concatenate([[[0.0, 0.0, 0.0, 1.0]], np.array(rot).reshape(-1, 4)])
    z3 = np.zeros((B, 3))
    bodies = api.Bodies(kind=kind, position=np.ascontiguousarray(P, dtype=s), rotation=np.ascontiguousarray(R, dtype=s),
                        linear_velocity=np.ascontiguousarray(z3, dtype=s), angular_velocity=np.ascontiguousarray(z3, dtype=s),
                        inverse_mass=np.ascontiguousarray(np.concatenate([[0.0], inv_m]), dtype=s),
                        inverse_inertia_local=np.ascontiguousarray(np.concatenate([np.zeros((1, 6)), np.array(inv_i).reshape(-1, 6)]), dtype=s),
                        center_of_mass=np.zeros((B, 3), dtype=s))
    C_ = len(cb) + 1
    ground_dims = [g[0] + 10.0, 0.5, g[2] + 10.0]
    cshape = np.concatenate([[SHAPE_CUBOID], np.full(C_ - 1, api.SHAPE_CONVEX_HULL)]).astype(np.int32)
    cdims = np.concatenate([[ground_dims], np.array(cd).reshape(-1, 3)])
    return Scene(name, bodies, np.full(B, SHAPE_CUBOID, np.int32), np.tile(ground_dims, (B, 1)), np.full(B, 0.5), np.zeros(B),
                 collider_body=np.concatenate([[0], cb]).astype(np.int32), local_position=np.concatenate([np.zeros((1, 3)), np.array(lp).reshape(-1, 3)]),
                 local_rotation=np.tile([0.0, 0.0, 0.0, 1.0], (C_, 1)), collider_shape=cshape, collider_dims=np.ascontiguousarray(cdims),
                 collider_friction=np.full(C_, 0.5), collider_restitution=np.zeros(C_), hulls=api.ConvexHulls.from_polyhedra(polys))


def decomposed_l_block(upright_x: float = -0.4, scalar=np.float64) -> Scene:
    """One L-block given as a convex decomposition of two hull parts (a foot of half extents 0.5 x 0.1 x 0.2 and an upright of 0.1 x 0.6 x 0.2
    standing on it at x = upright_x) resting on the ground: it stays up while its centre of mass is over the foot (upright_x = -0.4) and tips
    when the upright hangs past the foot's end (upright_x = -1.05)."""
    foot = (_box_points([0.5, 0.1, 0.2]), _CUBE_LOOPS, np.array([0.0, 0.1, 0.0]))
    upright = (_box_points([0.1, 0.6, 0.2]), _CUBE_LOOPS, np.array([upright_x, 0.8, 0.0]))
    # the body origin is the centre of mass: place it so the foot rests 1 mm above the ground
    m1, m2 = 0.5 * 0.1 * 0.2, 0.1 * 0.6 * 0.2
    c = (m1 * foot[2] + m2 * upright[2]) / (m1 + m2)
    return _decomposed_scene("decomposed_l_block", [[foot, upright]], [5.0, 0.0, 5.0], [c + [0.0, 0.001, 0.0]], [0.0], scalar)


_CUBE_LOOPS = [[1, 3, 7, 5], [0, 4, 6, 2], [2, 6, 7, 3], [0, 1, 5, 4], [4, 5, 7, 6], [0, 2, 3, 1]]


def decomposed_pile(n: int, seed: int = 17, layers: int = 4, scalar=np.float32) -> Scene:
    """A seeded pile of n dynamic bodies, each a convex decomposition of 2-4 hull parts (seeded Qhull rocks of 8-14 points, side by side along
    a bent chain so the bodies are concave), at random yaws on a jittered grid over a static ground cuboid; like the compounds of parry's
    convex_decomposition.  See _decomposed_scene for the frames and mass properties."""
    rng = np.random.default_rng(seed)
    pitch = 1.8
    side = int(np.ceil(np.sqrt(n / layers)))
    bodies, at, yaw = [], [], []
    for i in range(n):
        k = int(rng.integers(2, 5))
        parts, p, d = [], np.zeros(3), np.array([1.0, 0.0, 0.0])
        for j in range(k):
            v, f = convex_hull_of(rng.normal(size=(int(rng.integers(8, 15)), 3)) * rng.uniform(0.12, 0.18))
            parts.append((v - v.mean(axis=0), f, p.copy()))
            ang = rng.uniform(-1.2, 1.2)
            d = np.array([d[0] * np.cos(ang) - d[1] * np.sin(ang), d[0] * np.sin(ang) + d[1] * np.cos(ang), 0.0])
            p = p + d * 0.3
        centre = np.mean([x[2] for x in parts], axis=0)
        bodies.append([(v, f, q - centre) for v, f, q in parts])
        layer, cell = i // (side * side), i % (side * side)
        at.append(np.array([(cell // side) * pitch, 1.0 + layer * pitch, (cell % side) * pitch]) + rng.uniform(-0.05, 0.05, 3))
        yaw.append(rng.uniform(-np.pi, np.pi))
    extent = side * pitch
    return _decomposed_scene(f"decomposed_pile_{n}", bodies, [extent * 0.5, 0.0, extent * 0.5], at, yaw, scalar)
