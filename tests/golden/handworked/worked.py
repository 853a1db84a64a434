"""Hand-worked known-answer evaluation of the avian3d substep path for TINY scenes — written from the Rust source, NOT from oracle/.

Purpose (VERDICT r1 "pin the oracle independently"): the C++ oracle (oracle/) and the CUDA kernels were written by one author from one
reading of the reference; a shared misreading passes every oracle-vs-CUDA test.  This module is a second, independent reading: plain
Python/numpy, scalar by scalar in the working precision (numpy float32 or float64 scalars — every operation rounds once, nothing is fused),
serial, in the reference's system order.  It imports nothing from this repository.  `derive.py` runs it on the scenes below and commits the
inputs and results as `vectors.json`; tests/test_handworked.py demands that BOTH the oracle (CPU) and the CUDA path (GPU) reproduce them.

Every function cites the Rust it restates (paths relative to the reference root, avianphysics/avian @ 5bef382).  glam 0.30.8 is not in
the reference tree; its primitives are restated from its published algorithms (scalar formulas; glam's SSE2 `Quat` may associate a
product differently in the last bit, which is why the vectors are compared at 1e-5 relative, not bit for bit — `step(...,
quat_product="sse2")` evaluates the f32 quaternion product in the SSE2 association instead).
f32 transcendentals are taken correctly rounded (evaluated in double, rounded once).

Beyond the tiny vectors, tests/test_wave_scenes_cpu.py evaluates `step` on generated scenes of up to a few hundred manifolds (speed
limits, custom-integration markers, accelerations, full local inverse inertia, several solver iterations) against the oracle.
"""
import math

import numpy as np


class Num:
    """Working precision: T(x) rounds a Python float into it; all arithmetic on T values stays in T (numpy scalar semantics)."""

    def __init__(self, dtype):
        self.T = np.dtype(dtype).type
        self.eps = self.T(np.finfo(dtype).eps)

    def v(self, x, y, z):
        return np.array([x, y, z], dtype=self.T)

    def sin(self, x):
        return self.T(math.sin(float(x)))

    def cos(self, x):
        return self.T(math.cos(float(x)))

    def asin(self, x):
        return self.T(math.asin(float(x)))

    def sqrt(self, x):
        return np.sqrt(x)   # IEEE, correctly rounded in T


# ---- glam primitives (Vec3 / Quat / Mat3, scalar formulas) -------------------------------------------------------------------------
def dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def cross(a, b):   # glam Vec3::cross
    return np.array([a[1] * b[2] - b[1] * a[2], a[2] * b[0] - b[2] * a[0], a[0] * b[1] - b[0] * a[1]], dtype=a.dtype)


def length(N, a):
    return N.sqrt(dot(a, a))


def quat_mul(q, r):   # Hamilton product q * r, glam Quat::mul_quat; components x, y, z, w
    x0, y0, z0, w0 = q
    x1, y1, z1, w1 = r
    return np.array([
        ((w0 * x1 + x0 * w1) + y0 * z1) - z0 * y1,
        ((w0 * y1 - x0 * z1) + y0 * w1) + z0 * x1,
        ((w0 * z1 + x0 * y1) - y0 * x1) + z0 * w1,
        ((w0 * w1 - x0 * x1) - y0 * y1) - z0 * z1], dtype=q.dtype)


def quat_mul_sse2(q, r):
    """glam's SSE2 Quat::mul_quat (the f32 Quat of an x86-64 build): w0 * r and the sign-flipped x0 * r' are summed as one pair, the
    y0 and z0 terms as another, and the two pair sums added last"""
    x0, y0, z0, w0 = q
    x1, y1, z1, w1 = r
    return np.array([
        (w0 * x1 + x0 * w1) + (y0 * z1 - z0 * y1),
        (w0 * y1 - x0 * z1) + (y0 * w1 + z0 * x1),
        (w0 * z1 + x0 * y1) + (-(y0 * x1) + z0 * w1),
        (w0 * w1 - x0 * x1) + (-(y0 * y1) - z0 * z1)], dtype=q.dtype)


def quat_rotate(q, v):   # glam Quat * Vec3: v (w^2 - b.b) + 2 b (v.b) + 2 w (b x v)
    b = q[:3]
    w = q[3]
    two = q.dtype.type(2)
    return (v * (w * w - dot(b, b)) + b * (dot(v, b) * two)) + cross(b, v) * (w * two)


def quat_conj(q):    # unit quaternion inverse = conjugate (glam Quat::inverse)
    return np.array([-q[0], -q[1], -q[2], q[3]], dtype=q.dtype)


def quat_from_scaled_axis(N, v):   # glam Quat::from_scaled_axis: length 0 -> identity, else from_axis_angle(v / length, length)
    ln = length(N, v)
    if ln == 0:
        return np.array([0, 0, 0, 1], dtype=N.T)
    axis = v / ln      # glam: v / length (a division per component)
    half = ln * N.T(0.5)
    s, c = N.sin(half), N.cos(half)
    return np.array([axis[0] * s, axis[1] * s, axis[2] * s, c], dtype=N.T)


def any_orthonormal_vector(N, v):   # glam Vec3::any_orthonormal_vector (Pixar "Building an Orthonormal Basis, Revisited")
    T = N.T
    sign = T(math.copysign(1.0, float(v[2])))
    a = T(-1) / (sign + v[2])
    b = v[0] * v[1] * a
    return np.array([b, sign + v[1] * v[1] * a, -v[1]], dtype=T)


def any_orthogonal_vector(N, v):   # glam Vec3::any_orthogonal_vector: abs(x) > abs(y) ? (-z, 0, x) : (0, z, -y)  (not normalised)
    if abs(v[0]) > abs(v[1]):
        return N.v(-v[2], 0, v[0])
    return N.v(0, v[2], -v[1])


def mat3_from_quat(q):   # glam Mat3::from_quat; returns columns
    x, y, z, w = q
    T = q.dtype.type
    x2, y2, z2 = x + x, y + y, z + z
    xx, xy, xz = x * x2, x * y2, x * z2
    yy, yz, zz = y * y2, y * z2, z * z2
    wx, wy, wz = w * x2, w * y2, w * z2
    one = T(1)
    return [np.array([one - (yy + zz), xy + wz, xz - wy], dtype=q.dtype),
            np.array([xy - wz, one - (xx + zz), yz + wx], dtype=q.dtype),
            np.array([xz + wy, yz - wx, one - (xx + yy)], dtype=q.dtype)]


def sym_mul(m, v):   # SymmetricMat3 {m00,m01,m02,m11,m12,m22} * Vec3
    return np.array([(m[0] * v[0] + m[1] * v[1]) + m[2] * v[2], (m[1] * v[0] + m[3] * v[1]) + m[4] * v[2], (m[2] * v[0] + m[4] * v[1]) + m[5] * v[2]],
                    dtype=v.dtype)


def rotate_inverse_inertia(il, q):
    """ComputedAngularInertia::rotated (mass_properties/components/computed.rs:663-668): (R * I) * R^T, kept as a symmetric matrix
    (from_mat3_unchecked takes the upper triangle)."""
    R = mat3_from_quat(q)                       # columns
    full = [[il[0], il[1], il[2]], [il[1], il[3], il[4]], [il[2], il[4], il[5]]]   # full[r][c]
    # A = R * I: column j of A = R.x * I[0][j] + R.y * I[1][j] + R.z * I[2][j]
    A = [(R[0] * full[0][j] + R[1] * full[1][j]) + R[2] * full[2][j] for j in range(3)]
    # B = A * R^T: column j of B = A.x * R^T[0][j] + A.y * R^T[1][j] + A.z * R^T[2][j], R^T[i][j] = R[i][j] (column i of R, component j)
    B = [(A[0] * R[0][j] + A[1] * R[1][j]) + A[2] * R[2][j] for j in range(3)]
    return np.array([B[0][0], B[1][0], B[2][0], B[1][1], B[2][1], B[2][2]], dtype=q.dtype)


def sym_inverse_or_zero(m):
    """SymmetricMat3::inverse_or_zero (src/math/mod.rs:515-524): zero when the determinant is zero, else the inverse by cofactors
    (the adjugate over the determinant, expanded along the first row).  Any symmetric tensor, not only a diagonal one."""
    m00, m01, m02, m11, m12, m22 = m
    c00 = m11 * m22 - m12 * m12
    c01 = m02 * m12 - m01 * m22
    c02 = m01 * m12 - m02 * m11
    det = (m00 * c00 + m01 * c01) + m02 * c02
    if det == 0:
        return np.zeros(6, dtype=m.dtype)
    inv = m.dtype.type(1) / det
    c11 = m00 * m22 - m02 * m02
    c12 = m01 * m02 - m00 * m12
    c22 = m00 * m11 - m01 * m01
    return np.array([c00 * inv, c01 * inv, c02 * inv, c11 * inv, c12 * inv, c22 * inv], dtype=m.dtype)


def mat3_mul_vec(M, v):   # glam Mat3 * Vec3: x_axis * v.x + y_axis * v.y + z_axis * v.z
    return (M[0] * v[0] + M[1] * v[1]) + M[2] * v[2]


def clamp_length_max(N, v, m):   # glam Vec3::clamp_length_max
    l2 = dot(v, v)
    return m * (v / N.sqrt(l2)) if l2 > m * m else v


def angle_limit_correction(N, lo, hi, limit_axis, axis1, axis2, max_correction):
    """AngleLimit::compute_correction, 3D (dynamics/joints/mod.rs:427-473); None when the limit holds"""
    T = N.T
    PI, TAU = T(math.pi), T(2 * math.pi)
    phi = N.asin(dot(cross(axis1, axis2), limit_axis))
    if dot(axis1, axis2) < 0:
        phi = PI - phi
    if phi > PI:
        phi = phi - TAU
    if phi < lo or phi > hi:
        phi = min(max(phi, lo), hi)
        half = phi * T(0.5)
        s_, c_ = N.sin(half), N.cos(half)                  # Quat::from_axis_angle(limit_axis, phi)
        rot = np.array([limit_axis[0] * s_, limit_axis[1] * s_, limit_axis[2] * s_, c_], dtype=T)
        return clamp_length_max(N, cross(quat_rotate(rot, axis1), axis2), max_correction)
    return None


def recip_or_zero(x):   # math/mod.rs:248-268
    return (x.dtype.type(1) / x) if (x != 0 and np.isfinite(x)) else x.dtype.type(0)


# ---- the step ------------------------------------------------------------------------------------------------------------------------
DYNAMIC, KINEMATIC, STATIC = 0, 1, 2
FIXED, REVOLUTE, SPHERICAL, PRISMATIC, DISTANCE = range(5)


def softness(N, damping_ratio, hz, h):
    """SoftnessParameters::new + compute_coefficients (solver/softness_parameters/mod.rs:27-79)"""
    T = N.T
    double_damping_ratio = T(2) * damping_ratio
    angular_frequency = T(2 * math.pi) * hz      # TAU in T
    a1 = double_damping_ratio + angular_frequency * h
    a2 = angular_frequency * h * a1
    a3 = T(1) / (T(1) + a2)
    return {"bias": angular_frequency / a1, "impulse_scale": a3, "mass_scale": a2 * a3}


def step(scene, dtype=np.float32, quat_product="scalar"):
    """One PhysicsSchedule solver stage over a small scene (dict, see derive.py); returns the outputs as a dict of lists.

    quat_product: "scalar" (glam's scalar formulas, what vectors.json holds) or "sse2" (glam's SSE2 association of the f32 quaternion
    product, which an x86-64 build of the reference runs).  The two differ by an ulp per product; in f32 contact scenes of several
    substeps the soft contact (separation / h in the bias) amplifies that ulp to ~1e-5, so comparisons with code that follows the SSE2
    association use "sse2".  f64 quaternions have no SIMD path in glam: the option changes nothing there."""
    N = Num(dtype)
    T = N.T
    qmul = quat_mul_sse2 if (quat_product == "sse2" and np.dtype(dtype) == np.float32) else quat_mul
    prm = scene["params"]
    dt, h = T(prm["dt"]), T(prm["h"])
    substeps = int(prm["substeps"])
    solver_iterations = max(int(prm.get("solver_iterations", 1)), 1)
    g = N.v(*[T(x) for x in prm["gravity"]])
    nb = len(scene["bodies"])

    # ---- prepare_solver_bodies (solver/solver_body/plugin.rs:173-251)
    B = []
    for b in scene["bodies"]:
        kind = b["kind"]
        rot = np.array(b["rotation"], dtype=T)
        il = np.array(b["inverse_inertia_local"], dtype=T)
        sb = {"kind": kind, "pos": np.array(b["position"], dtype=T), "rot": rot, "com": np.array(b.get("center_of_mass", [0, 0, 0]), dtype=T),
              "lin0": np.array(b["linear_velocity"], dtype=T), "has_solver_body": kind != STATIC}
        sb["v"] = np.array(b["linear_velocity"], dtype=T) if kind != STATIC else N.v(0, 0, 0)
        sb["w"] = np.array(b["angular_velocity"], dtype=T) if kind != STATIC else N.v(0, 0, 0)
        sb["dp"] = N.v(0, 0, 0)
        sb["dq"] = np.array([0, 0, 0, 1], dtype=T)
        sb["inv_mass"] = T(b["inverse_mass"])
        sb["il"] = il
        sb["iw"] = rotate_inverse_inertia(il, rot)
        # LockedAxes (rigid_body/locked_axes.rs:34-47: bits 0b XYZ_xyz = translation X Y Z, rotation x y z)
        locked = int(b.get("locked_axes", 0))
        sb["locked"] = locked
        # SolverBodyInertia::new (solver_body/mod.rs:378-423): a locked rotation axis clears its row and column of the world inverse inertia
        iw = sb["iw"].copy()
        if locked & 0b000_100: iw[0] = iw[1] = iw[2] = T(0)
        if locked & 0b000_010: iw[1] = iw[3] = iw[4] = T(0)
        if locked & 0b000_001: iw[2] = iw[4] = iw[5] = T(0)
        sb["iw"] = iw
        # SolverBodyInertia::new: dominance = Dominance for dynamic bodies, i8::MAX + 1 otherwise (solver_body/mod.rs:414-420)
        sb["dominance"] = int(b.get("dominance", 0)) if kind == DYNAMIC else 128
        eps = T(1e-6)
        iso = (not (abs(il[0] - il[3]) > eps or abs(il[3] - il[5]) > eps)) and abs(il[1]) < eps and abs(il[2]) < eps and abs(il[4]) < eps
        sb["gyro"] = (locked & 0b111) != 0b111 and not iso   # plugin.rs:241-247: rotation unlocked on at least one axis and not isotropic
        # integration markers CustomVelocityIntegration (bit 0) / CustomPositionIntegration (bit 1) (integrator/mod.rs:169-195)
        flags = int(b.get("integration_flags", 0))
        sb["custom_vel"], sb["custom_pos"] = bool(flags & 1), bool(flags & 2)
        # MaxLinearSpeed / MaxAngularSpeed: absent = no clamp (clamp_velocities queries only the bodies that have them)
        sb["max_lin"] = None if b.get("max_linear_speed") is None else T(b["max_linear_speed"])
        sb["max_ang"] = None if b.get("max_angular_speed") is None else T(b["max_angular_speed"])
        # pre_process_velocity_increments (integrator/mod.rs:260-313), dynamic bodies only.  The increments arrive holding the
        # accelerations ForcePlugin wrote (VelocityIntegrationData::apply_linear/angular_acceleration, integrator/mod.rs:236-244)
        sb["lin_rhs"], sb["ang_rhs"] = T(1), T(1)
        sb["lin_inc"], sb["ang_inc"] = N.v(0, 0, 0), N.v(0, 0, 0)
        if kind == DYNAMIC:
            sb["lin_rhs"] = T(1) / (T(1) + h * T(b.get("linear_damping", 0.0)))
            sb["ang_rhs"] = T(1) / (T(1) + h * T(b.get("angular_damping", 0.0)))
            li = np.array(b.get("linear_acceleration", [0, 0, 0]), dtype=T) + g * T(b.get("gravity_scale", 1.0))
            ai = np.array(b.get("angular_acceleration", [0, 0, 0]), dtype=T)
            # LockedAxes::apply_to_vec / apply_to_angular_velocity on the increments (integrator/mod.rs:296-300)
            for ax, (tb, rb) in enumerate(((0b100_000, 0b000_100), (0b010_000, 0b000_010), (0b001_000, 0b000_001))):
                if locked & tb: li[ax] = T(0)
                if locked & rb: ai[ax] = T(0)
            sb["lin_inc"] = li * h
            sb["ang_inc"] = ai * h
        B.append(sb)

    def inertia_of(i, zeroed):
        """(effective_inv_mass Vec3, effective_inv_angular_inertia) — zero for SolverBodyInertia::DUMMY or the dominated side"""
        if i < 0 or not B[i]["has_solver_body"] or zeroed:
            return N.v(0, 0, 0), np.zeros(6, dtype=T)
        m = B[i]["inv_mass"]
        lk = B[i]["locked"]                                   # effective_inv_mass (solver_body/mod.rs:437-451)
        return N.v(T(0) if lk & 0b100_000 else m, T(0) if lk & 0b010_000 else m, T(0) if lk & 0b001_000 else m), B[i]["iw"]

    dummy = {"v": N.v(0, 0, 0), "w": N.v(0, 0, 0), "dp": N.v(0, 0, 0), "dq": np.array([0, 0, 0, 1], dtype=T), "kind": STATIC, "dominance": 128,
             "has_solver_body": False}

    def body(i):
        # static bodies have no SolverBody: every system works on a fresh DUMMY for them (solver/plugin.rs:488-503); writes are lost
        if i < 0 or not B[i]["has_solver_body"]:
            return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in dummy.items()}
        return B[i]

    # ---- update_contact_softness (solver/plugin.rs:326-350)
    max_hz = T(1) / (dt * T(2))
    hz = T(prm["contact_frequency_factor"]) * min(max_hz, T(0.25) / h)
    soft_dyn = softness(N, T(prm["contact_damping_ratio"]), hz, h)
    soft_nondyn = softness(N, T(prm["contact_damping_ratio"]), T(2) * hz, h)
    max_overlap = T(prm["max_overlap_solve_speed"]) * T(prm["length_unit"])
    rest_threshold = T(prm["restitution_threshold"]) * T(prm["length_unit"])
    warm_coeff = T(prm["warm_start_coefficient"])

    # ---- prepare_contact_constraints -> ContactConstraint::generate (solver/plugin.rs:363-448, contact/mod.rs:110-220)
    C = []
    for m in scene.get("manifolds", []):
        i1, i2 = m["body1"], m["body2"]
        k1 = B[i1]["kind"] if i1 >= 0 else STATIC
        k2 = B[i2]["kind"] if i2 >= 0 else STATIC
        if (k1 != DYNAMIC and k2 != DYNAMIC) or not m["points"]:
            C.append(None)
            continue
        d1 = B[i1]["dominance"] if (i1 >= 0 and B[i1]["has_solver_body"]) else 128
        d2 = B[i2]["dominance"] if (i2 >= 0 and B[i2]["has_solver_body"]) else 128
        rel = d1 - d2
        im1, ii1 = inertia_of(i1, rel > 0)
        im2, ii2 = inertia_of(i2, rel < 0)
        soft = soft_nondyn if rel != 0 else soft_dyn
        mass_sum = im1 + im2
        n = np.array(m["normal"], dtype=T)
        # compute_tangent_directions (contact/mod.rs:427-449): LinearVelocity COMPONENTS of the two rigid bodies
        lv1 = B[i1]["lin0"] if i1 >= 0 else N.v(0, 0, 0)
        lv2 = B[i2]["lin0"] if i2 >= 0 else N.v(0, 0, 0)
        fd = -n
        relv = lv1 - lv2
        tv = relv - fd * dot(fd, relv)
        rcp = T(1) / length(N, tv)                          # glam try_normalize: length_recip finite and > 0
        t1 = tv * rcp if (np.isfinite(rcp) and rcp > 0) else any_orthonormal_vector(N, fd)
        t2 = cross(fd, t1)
        friction, restitution = T(m["friction"]), T(m["restitution"])
        surf = np.array(m.get("tangent_velocity", [0, 0, 0]), dtype=T)
        warm = bool(prm["match_contacts"])
        pts = []
        for p in m["points"]:
            r1, r2 = np.array(p["anchor1"], dtype=T), np.array(p["anchor2"], dtype=T)
            r1xn, r2xn = cross(r1, n), cross(r2, n)
            k = (dot(n, mass_sum * n) + dot(r1xn, sym_mul(ii1, r1xn))) + dot(r2xn, sym_mul(ii2, r2xn))      # normal_part.rs:96-104
            pt = {"r1": r1, "r2": r2, "meff": recip_or_zero(k), "imp": T(p["warm_start_normal_impulse"]) if warm else T(0), "total": T(0),
                  "normal_speed": T(p["normal_speed"]), "sep0": -T(p["penetration"]) - dot(r2 - r1, n), "tangent": None}
            if friction > 0:                                  # contact/mod.rs:185
                rt11, rt12, rt21, rt22 = cross(r1, t1), cross(r2, t1), cross(r1, t2), cross(r2, t2)
                i1_rt11, i2_rt12, i1_rt21, i2_rt22 = sym_mul(ii1, rt11), sym_mul(ii2, rt12), sym_mul(ii1, rt21), sym_mul(ii2, rt22)
                k1_ = (dot(t1, mass_sum * t1) + dot(rt11, i1_rt11)) + dot(rt12, i2_rt12)
                k2_ = (dot(t2, mass_sum * t2) + dot(rt21, i1_rt21)) + dot(rt22, i2_rt22)
                k3_ = T(2) * (dot(rt11, i1_rt21) + dot(rt12, i2_rt22))
                ws_t = np.array(p["warm_start_tangent_impulse"], dtype=T) if warm else np.zeros(2, dtype=T)
                pt["tangent"] = {"imp": ws_t, "K": (k1_, k2_, k3_)}
            pts.append(pt)
        C.append({"b1": i1, "b2": i2, "rel": rel, "n": n, "t1": t1, "friction": friction, "restitution": restitution, "surf": surf, "soft": soft,
                  "points": pts})
    # solve order: overflow colour serially first, then colours 0..22 (solver/plugin.rs:461-479)
    co = scene.get("color_offsets")
    if co is None:
        order = list(range(len(C)))
    else:
        order = list(range(co[23], co[24])) + list(range(0, co[23]))
    order = [k for k in order if C[k] is not None]

    def apply(c, b1, b2, in1, in2, r1, r2, imp):
        (im1, ii1), (im2, ii2) = in1, in2
        b1["v"] = b1["v"] - imp * im1
        b1["w"] = b1["w"] - sym_mul(ii1, cross(r1, imp))
        b2["v"] = b2["v"] + imp * im2
        b2["w"] = b2["w"] + sym_mul(ii2, cross(r2, imp))

    def constraint_bodies(c):
        return body(c["b1"]), body(c["b2"]), inertia_of(c["b1"], c["rel"] > 0), inertia_of(c["b2"], c["rel"] < 0)

    def warm_start(c):                                        # contact/mod.rs:223-264
        b1, b2, in1, in2 = constraint_bodies(c)
        n, t1 = c["n"], c["t1"]
        t2 = cross(t1, n)                                     # tangent_directions(): [tangent1, tangent1 x normal] (contact/mod.rs:411-421)
        for p in c["points"]:
            ti = p["tangent"]["imp"] if p["tangent"] is not None else np.zeros(2, dtype=T)
            P = warm_coeff * ((p["imp"] * n + ti[0] * t1) + ti[1] * t2)
            apply(c, b1, b2, in1, in2, p["r1"], p["r2"], P)

    def solve(c, use_bias):                                   # contact/mod.rs:267-354
        b1, b2, in1, in2 = constraint_bodies(c)
        n, t1 = c["n"], c["t1"]
        delta_translation = b2["dp"] - b1["dp"]
        for p in c["points"]:
            r1 = quat_rotate(b1["dq"], p["r1"])
            r2 = quat_rotate(b2["dq"], p["r2"])
            separation = dot(delta_translation + (r2 - r1), n) + p["sep0"]
            r1, r2 = p["r1"], p["r2"]
            relv = (b2["v"] + cross(b2["w"], r2)) - (b1["v"] + cross(b1["w"], r1))
            vn = dot(relv, n)                                 # normal_part.rs:116-166
            if separation > 0:
                impulse = -p["meff"] * (vn + separation / h)
            elif use_bias:
                bias = max(c["soft"]["bias"] * separation, -max_overlap)
                impulse = -(c["soft"]["mass_scale"] * p["meff"]) * (vn + bias) - c["soft"]["impulse_scale"] * p["imp"]
            else:
                impulse = -p["meff"] * vn
            new_impulse = max(p["imp"] + impulse, T(0))
            impulse = new_impulse - p["imp"]
            p["imp"] = new_impulse
            p["total"] = p["total"] + new_impulse
            apply(c, b1, b2, in1, in2, r1, r2, impulse * n)
        t2 = cross(t1, n)
        for p in c["points"]:
            tp = p["tangent"]
            if tp is None:
                continue
            r1, r2 = p["r1"], p["r2"]
            relv = (b2["v"] + cross(b2["w"], r2)) - (b1["v"] + cross(b1["w"], r1))
            limit = c["friction"] * p["imp"]                  # tangent_part.rs:155-244
            relv = relv + c["surf"]
            ts1, ts2 = dot(relv, t1), dot(relv, t2)
            t11, t22, t12 = ts1 * ts1, ts2 * ts2, ts1 * ts2
            inv = (t11 * tp["K"][0] + t22 * tp["K"][1]) + t12 * tp["K"][2]
            with np.errstate(divide="ignore", invalid="ignore"):
                em = (t11 + t22) * (T(1) / inv)
            if not np.isfinite(em):
                continue
            new = np.array([tp["imp"][0] - em * ts1, tp["imp"][1] - em * ts2], dtype=T)
            l2 = new[0] * new[0] + new[1] * new[1]
            if l2 > limit * limit:                            # glam Vec2::clamp_length_max
                new = limit * (new / N.sqrt(l2))
            d = new - tp["imp"]
            tp["imp"] = new
            apply(c, b1, b2, in1, in2, r1, r2, d[0] * t1 + d[1] * t2)

    def restitution(c):                                       # solver/plugin.rs:676-718, contact/mod.rs:358-407
        if c["restitution"] == 0:
            return
        b1, b2, in1, in2 = constraint_bodies(c)
        iters = int(prm["restitution_iterations"]) if len(c["points"]) > 1 else 1
        for _ in range(iters):
            for p in c["points"]:
                if p["normal_speed"] > -rest_threshold or p["total"] == 0:
                    continue
                relv = (b2["v"] + cross(b2["w"], p["r2"])) - (b1["v"] + cross(b1["w"], p["r1"]))
                vn = dot(relv, c["n"])
                impulse = -p["meff"] * (vn + c["restitution"] * p["normal_speed"])
                new_impulse = max(p["imp"] + impulse, T(0))
                impulse = new_impulse - p["imp"]
                p["imp"] = new_impulse
                p["total"] = p["total"] + impulse
                apply(c, b1, b2, in1, in2, p["r1"], p["r2"], impulse * c["n"])

    # ---- prepare_xpbd_joint (xpbd/plugin.rs:125-142; joints/shared/point_constraint.rs:38-51; revolute.rs:51-90; fixed_angle_constraint.rs:38-57)
    J = []
    for j in scene.get("joints", []):
        b1, b2 = B[j["body1"]], B[j["body2"]]
        la1, la2 = np.array(j["local_anchor1"], dtype=T), np.array(j["local_anchor2"], dtype=T)
        d = dict(j)
        d["r1"] = quat_rotate(b1["rot"], la1 - b1["com"])
        d["r2"] = quat_rotate(b2["rot"], la2 - b2["com"])
        d["cd"] = (b2["pos"] - b1["pos"]) + (quat_rotate(b2["rot"], b2["com"]) - quat_rotate(b1["rot"], b1["com"]))
        d["lam_p"] = N.v(0, 0, 0)
        d["lam_a"] = N.v(0, 0, 0)
        if j["type"] == PRISMATIC:                            # xpbd/joints/prismatic.rs:43-77
            basis1 = np.array(j.get("local_basis1", [0, 0, 0, 1]), dtype=T)
            basis2 = np.array(j.get("local_basis2", [0, 0, 0, 1]), dtype=T)
            d["rd"] = qmul(qmul(b1["rot"], basis1), quat_conj(qmul(b2["rot"], basis2)))   # FixedAngleConstraintShared::prepare
            d["ax1"] = quat_rotate(qmul(b1["rot"], basis1), np.array(j.get("axis", [1, 0, 0]), dtype=T))   # free_axis1
        if j["type"] in (FIXED, REVOLUTE):
            basis1 = np.array(j.get("local_basis1", [0, 0, 0, 1]), dtype=T)
            basis2 = np.array(j.get("local_basis2", [0, 0, 0, 1]), dtype=T)
            if j["type"] == REVOLUTE:
                axis = np.array(j.get("axis", [0, 0, 1]), dtype=T)
                d["a1"] = quat_rotate(qmul(b1["rot"], basis1), axis)
                d["a2"] = quat_rotate(qmul(b2["rot"], basis2), axis)
                ortho = any_orthonormal_vector(N, axis)            # revolute.rs:86-89
                d["b1"] = quat_rotate(qmul(b1["rot"], basis1), ortho)
                d["b2"] = quat_rotate(qmul(b2["rot"], basis2), ortho)
            else:
                d["rd"] = qmul(qmul(b1["rot"], basis1), quat_conj(qmul(b2["rot"], basis2)))
        if j["type"] == SPHERICAL:                            # xpbd/joints/spherical.rs:45-82: through rotation MATRICES here
            basis1 = np.array(j.get("local_basis1", [0, 0, 0, 1]), dtype=T)
            basis2 = np.array(j.get("local_basis2", [0, 0, 0, 1]), dtype=T)
            R1, R2 = mat3_from_quat(b1["rot"]), mat3_from_quat(b2["rot"])
            d["r1"] = mat3_mul_vec(R1, la1 - b1["com"])
            d["r2"] = mat3_mul_vec(R2, la2 - b2["com"])
            twist = np.array(j.get("axis", [0, 1, 0]), dtype=T)
            swing = any_orthonormal_vector(N, twist)
            d["sw1"], d["sw2"] = mat3_mul_vec(R1, quat_rotate(basis1, swing)), mat3_mul_vec(R2, quat_rotate(basis2, swing))
            d["tw1"], d["tw2"] = mat3_mul_vec(R1, quat_rotate(basis1, twist)), mat3_mul_vec(R2, quat_rotate(basis2, twist))
            d["lam_b"] = N.v(0, 0, 0)
        d.setdefault("lam_b", N.v(0, 0, 0))
        J.append(d)

    def joint_sides(j):
        # dominance decides per call which side is treated as immovable (xpbd/plugin.rs:176-180)
        i1, i2 = j["body1"], j["body2"]
        d1 = B[i1]["dominance"] if B[i1]["has_solver_body"] else 128
        d2 = B[i2]["dominance"] if B[i2]["has_solver_body"] else 128
        return body(i1), body(i2), inertia_of(i1, d1 - d2 > 0), inertia_of(i2, d1 - d2 < 0)

    def lagrange_update(c_val, ws, compliance):               # xpbd/mod.rs:393-413 with lagrange = 0
        w_sum = T(0)
        for w_ in ws:
            w_sum = w_sum + w_
        if w_sum <= N.eps:
            return T(0)
        tilde = compliance / (h * h)
        return (-c_val - tilde * T(0)) / (w_sum + tilde)

    def positional_impulse(b1, b2, in1, in2, imp, r1, r2):    # xpbd/positional_constraint.rs:9-50
        (im1, ii1), (im2, ii2) = in1, in2
        b1["dp"] = b1["dp"] + imp * im1
        b1["dq"] = qmul(quat_from_scaled_axis(N, sym_mul(ii1, cross(r1, imp))), b1["dq"])
        b2["dp"] = b2["dp"] - imp * im2
        b2["dq"] = qmul(quat_from_scaled_axis(N, sym_mul(ii2, cross(r2, -imp))), b2["dq"])

    def generalized_inverse_mass(im, ii, r, n):               # positional_constraint.rs:66-79 with inv_mass.max_element()
        rxn = cross(r, n)
        return max(im[0], im[1], im[2]) + dot(rxn, sym_mul(ii, rxn))

    def point_constraint(j, b1, b2, in1, in2, compliance):    # joints/shared/point_constraint.rs:54-108
        wr1, wr2 = quat_rotate(b1["dq"], j["r1"]), quat_rotate(b2["dq"], j["r2"])
        sep = ((b2["dp"] - b1["dp"]) + (wr2 - wr1)) + j["cd"]
        m2 = dot(sep, sep)
        if m2 == 0:
            return
        mag = N.sqrt(m2)
        dirn = -sep / mag
        w1 = generalized_inverse_mass(in1[0], in1[1], wr1, dirn)
        w2 = generalized_inverse_mass(in2[0], in2[1], wr2, dirn)
        dl = lagrange_update(mag, [w1, w2], compliance)
        imp = dl * dirn
        j["lam_p"] = j["lam_p"] + imp
        positional_impulse(b1, b2, in1, in2, imp, wr1, wr2)

    def align_orientation(j, b1, b2, in1, in2, difference, compliance):   # xpbd/angular_constraint.rs:149-194, 58-98
        angle = length(N, difference)
        if angle <= N.eps:
            return N.v(0, 0, 0)
        axis = difference / angle
        w1, w2 = dot(axis, sym_mul(in1[1], axis)), dot(axis, sym_mul(in2[1], axis))
        dl = lagrange_update(angle, [w1, w2], compliance)
        if abs(dl) > N.eps:
            imp = -dl * axis
            b1["dq"] = qmul(quat_from_scaled_axis(N, sym_mul(in1[1], imp)), b1["dq"])
            b2["dq"] = qmul(quat_from_scaled_axis(N, sym_mul(in2[1], -imp)), b2["dq"])
        return dl * axis

    def solve_joint(j):
        b1, b2, in1, in2 = joint_sides(j)
        c0, c1 = T(j.get("compliance0", 0.0)), T(j.get("compliance1", 0.0))
        if j["type"] == DISTANCE:                             # xpbd/joints/distance.rs:56-117; joints/mod.rs:321-345
            wr1, wr2 = quat_rotate(b1["dq"], j["r1"]), quat_rotate(b2["dq"], j["r2"])
            sep = ((b2["dp"] - b1["dp"]) + (wr2 - wr1)) + j["cd"]
            d2 = dot(sep, sep)
            lo, hi = T(j["limit_min"]), T(j["limit_max"])
            dirn, dist = N.v(0, 0, 0), T(0)
            if d2 > N.eps:
                dd = N.sqrt(d2)
                if dd < lo:
                    dirn, dist = sep / dd, lo - dd
                elif dd > hi:
                    dirn, dist = -sep / dd, dd - hi
            if dist <= N.eps:
                return
            w1 = generalized_inverse_mass(in1[0], in1[1], wr1, dirn)
            w2 = generalized_inverse_mass(in2[0], in2[1], wr2, dirn)
            dl = lagrange_update(dist, [w1, w2], c0)
            imp = dl * dirn
            j["lam_p"] = j["lam_p"] + imp
            positional_impulse(b1, b2, in1, in2, imp, wr1, wr2)
        elif j["type"] == SPHERICAL:                          # xpbd/joints/spherical.rs:84-207: point, swing limit, twist limit
            c2 = T(j.get("compliance2", 0.0))
            point_constraint(j, b1, b2, in1, in2, c0)
            PI = T(math.pi)
            if j.get("swing_limit") is not None:
                a1, a2 = quat_rotate(b1["dq"], j["sw1"]), quat_rotate(b2["dq"], j["sw2"])
                n = cross(a1, a2)
                nm = length(N, n)
                if nm > N.eps:
                    n = n / nm
                    corr = angle_limit_correction(N, T(j["swing_limit"][0]), T(j["swing_limit"][1]), n, a1, a2, PI)
                    if corr is not None:
                        j["lam_a"] = j["lam_a"] + align_orientation(j, b1, b2, in1, in2, corr, c1)
            if j.get("twist_limit") is not None:
                a1, a2 = quat_rotate(b1["dq"], j["sw1"]), quat_rotate(b2["dq"], j["sw2"])
                n = a1 + a2
                nm = length(N, n)
                if nm > N.eps:
                    tb1, tb2 = quat_rotate(b1["dq"], j["tw1"]), quat_rotate(b2["dq"], j["tw2"])
                    n = n / nm
                    n1 = tb1 - dot(n, tb1) * n
                    n2 = tb2 - dot(n, tb2) * n
                    m1, m2 = length(N, n1), length(N, n2)
                    if not (m1 <= N.eps or m2 <= N.eps):
                        n1, n2 = n1 / m1, n2 / m2
                        max_corr = T(2) * PI if dot(a1, a2) > T(-0.5) else h
                        corr = angle_limit_correction(N, T(j["twist_limit"][0]), T(j["twist_limit"][1]), n, n1, n2, max_corr)
                        if corr is not None:
                            j["lam_b"] = j["lam_b"] + align_orientation(j, b1, b2, in1, in2, corr, c2)
        elif j["type"] == REVOLUTE:                           # xpbd/joints/revolute.rs:92-187: align, angle limit, then point
            a1, a2 = quat_rotate(b1["dq"], j["a1"]), quat_rotate(b2["dq"], j["a2"])
            j["lam_a"] = j["lam_a"] + align_orientation(j, b1, b2, in1, in2, cross(a1, a2), c1)
            if j.get("angle_limit") is not None:
                a1 = quat_rotate(b1["dq"], j["a1"])
                lb1, lb2 = quat_rotate(b1["dq"], j["b1"]), quat_rotate(b2["dq"], j["b2"])
                corr = angle_limit_correction(N, T(j["angle_limit"][0]), T(j["angle_limit"][1]), a1, lb1, lb2, T(math.pi))
                if corr is not None:
                    j["lam_b"] = j["lam_b"] + align_orientation(j, b1, b2, in1, in2, corr, T(j.get("compliance2", 0.0)))
            point_constraint(j, b1, b2, in1, in2, c0)
        elif j["type"] == PRISMATIC:                          # xpbd/joints/prismatic.rs:79-193: fixed angle, then translation off the free axis
            q = qmul(qmul(j["rd"], b1["dq"]), quat_conj(b2["dq"]))
            j["lam_a"] = j["lam_a"] + align_orientation(j, b1, b2, in1, in2, T(-2) * q[:3], c1)      # angle_compliance
            wr1, wr2 = quat_rotate(b1["dq"], j["r1"]), quat_rotate(b2["dq"], j["r2"])
            axis1 = quat_rotate(b1["dq"], j["ax1"])

            def along(lo, hi, sep, axis):                     # DistanceLimit::compute_correction_along_axis (joints/mod.rs:344-357)
                a = dot(sep, axis)
                if a < lo:
                    return axis * (lo - a)
                if a > hi:
                    return -axis * (a - hi)
                return N.v(0, 0, 0)
            dx = N.v(0, 0, 0)
            sep = ((b2["dp"] - b1["dp"]) + (wr2 - wr1)) + j["cd"]
            if j.get("limits") is not None:
                dx = dx + along(T(j["limits"][0]), T(j["limits"][1]), sep, axis1)
            axis2 = any_orthogonal_vector(N, axis1)
            axis3 = cross(axis1, axis2)
            dx = dx + along(T(0), T(0), sep, axis2)
            dx = dx + along(T(0), T(0), sep, axis3)
            mag = length(N, dx)
            if mag <= N.eps:
                return
            dirn = dx / mag
            w1 = generalized_inverse_mass(in1[0], in1[1], wr1, dirn)
            w2 = generalized_inverse_mass(in2[0], in2[1], wr2, dirn)
            imp = lagrange_update(mag, [w1, w2], c0) * dirn   # align_compliance
            j["lam_p"] = j["lam_p"] + imp
            positional_impulse(b1, b2, in1, in2, imp, wr1, wr2)
        elif j["type"] == FIXED:                              # xpbd/joints/fixed.rs:73-89, shared/fixed_angle_constraint.rs:59-96
            q = qmul(qmul(j["rd"], b1["dq"]), quat_conj(b2["dq"]))
            difference = T(-2) * q[:3]
            j["lam_a"] = j["lam_a"] + align_orientation(j, b1, b2, in1, in2, difference, c1)
            point_constraint(j, b1, b2, in1, in2, c0)

    # ---- run_substep_schedule (solver/schedule.rs:59-69,194-213)
    for _ in range(substeps):
        for b in B:                                           # integrate_velocities (integrator/mod.rs:343-391)
            if not b["has_solver_body"] or b["kind"] == KINEMATIC or b["custom_vel"]:
                continue
            b["v"] = b["v"] * b["lin_rhs"]
            b["w"] = b["w"] * b["ang_rhs"]
            b["v"] = b["v"] + b["lin_inc"]
            b["w"] = b["w"] + b["ang_inc"]
            if b["gyro"]:                                     # solve_gyroscopic_torque (integrator/mod.rs:403-460)
                rot = qmul(b["dq"], b["rot"])
                lw = quat_rotate(quat_conj(rot), b["w"])
                il = b["il"]
                # ComputedAngularInertia::tensor() = inverse_or_zero of the stored inverse tensor (computed.rs:617-619)
                tensor = sym_inverse_or_zero(il)
                L = sym_mul(tensor, lw)
                Ln = L - h * cross(lw, L)
                l2 = dot(Ln, Ln)
                if l2 == 0:
                    b["w"] = N.v(0, 0, 0)
                else:
                    Ln = Ln * N.sqrt(dot(L, L) / l2)
                    b["w"] = quat_rotate(rot, sym_mul(il, Ln))
        for b in B:                                           # clamp_velocities (integrator/mod.rs:467-500), chained after it
            if not b["has_solver_body"]:
                continue
            for key, ms in (("v", b["max_lin"]), ("w", b["max_ang"])):
                if ms is None:
                    continue
                l2 = dot(b[key], b[key])
                if l2 > ms * ms:
                    b[key] = b[key] * (ms / N.sqrt(l2))
        for k in order:
            warm_start(C[k])
        for _ in range(solver_iterations):                    # solve_contacts::<true>, done `iterations` times (solver/plugin.rs:517-531)
            for k in order:
                solve(C[k], True)
        for b in B:                                           # integrate_positions (integrator/mod.rs:503-535)
            if not b["has_solver_body"] or b["custom_pos"]:
                continue
            b["dp"] = b["dp"] + b["v"] * h
            b["dq"] = qmul(quat_from_scaled_axis(N, b["w"] * h), b["dq"])
        for k in order:
            solve(C[k], False)
        if J:
            pre = [(b["dp"].copy(), b["dq"].copy()) for b in B]   # xpbd/plugin.rs:61-76
            for jt in (FIXED, REVOLUTE, SPHERICAL, PRISMATIC, DISTANCE):   # type order, then table order (xpbd/plugin.rs:77-82)
                for j in J:
                    if j["type"] == jt:
                        solve_joint(j)
            for b, (pdp, pdq) in zip(B, pre):                 # project_linear_velocity / project_angular_velocity (xpbd/plugin.rs:192-240)
                if not b["has_solver_body"]:
                    continue
                b["v"] = b["v"] + (b["dp"] - pdp) / h
                dr = qmul(b["dq"], quat_conj(pdq))
                nw = T(2) * dr[:3] / h
                if dr[3] < 0:
                    nw = -nw
                b["w"] = b["w"] + nw
            for jt in (FIXED, REVOLUTE, SPHERICAL, PRISMATIC, DISTANCE):   # joint_damping::<T> (solver/plugin.rs:759-806), same order
                # one dummy_body1 / dummy_body2 per system run (plugin.rs:766-767), i.e. per joint type and substep, shared by every joint
                # of that run whose end has no SolverBody.  SolverBody::DUMMY has empty flags (not kinematic), so the angular part writes
                # into it and the next such joint reads that velocity; the linear part adds p * 0 and leaves it at zero.
                dummies = (body(-1), body(-1))
                for j in J:
                    if j["type"] != jt or j.get("damping") is None:
                        continue
                    i1, i2 = j["body1"], j["body2"]
                    jb1 = B[i1] if B[i1]["has_solver_body"] else dummies[0]
                    jb2 = B[i2] if B[i2]["has_solver_body"] else dummies[1]
                    dl, da = T(j["damping"][0]), T(j["damping"][1])
                    d_omega = (jb2["w"] - jb1["w"]) * min(da * h, T(1))
                    if jb1["kind"] != KINEMATIC:
                        jb1["w"] = jb1["w"] + d_omega
                    if jb2["kind"] != KINEMATIC:
                        jb2["w"] = jb2["w"] - d_omega
                    d_v = (jb2["v"] - jb1["v"]) * min(dl * h, T(1))
                    w1, w2 = inertia_of(i1, False)[0], inertia_of(i2, False)[0]
                    ws = w1 + w2
                    pimp = d_v * np.array([recip_or_zero(ws[0]), recip_or_zero(ws[1]), recip_or_zero(ws[2])], dtype=T)
                    jb1["v"] = jb1["v"] + pimp * w1
                    jb2["v"] = jb2["v"] - pimp * w2

    for k in order:
        restitution(C[k])

    # ---- writeback_solver_bodies (solver_body/plugin.rs:255-284), writeback_joint_forces (xpbd/plugin.rs:242-260), store_contact_impulses
    out = {"position": [], "rotation": [], "linear_velocity": [], "angular_velocity": []}
    for b in B:
        pos, rot, lv, av = b["pos"], b["rot"], np.array(b["lin0"], dtype=T), None
        if b["has_solver_body"]:
            old_com = quat_rotate(rot, b["com"])
            q = qmul(b["dq"], rot)
            q = q * (T(0.5) * (T(3) - ((q[0] * q[0] + q[1] * q[1]) + (q[2] * q[2] + q[3] * q[3]))))   # fast_renormalize (transform.rs:811-817)
            new_com = quat_rotate(q, b["com"])
            pos = pos + ((b["dp"] + old_com) - new_com)
            rot, lv, av = q, b["v"], b["w"]
        out["position"].append([float(x) for x in pos])
        out["rotation"].append([float(x) for x in rot])
        out["linear_velocity"].append([float(x) for x in lv])
        out["angular_velocity"].append(None if av is None else [float(x) for x in av])
    # Res<Time> in SolverSystems::Finalize is Time<Physics> again (solver/schedule.rs:211-212): delta_secs = dt, not h
    rhs = recip_or_zero(dt * dt) * T(substeps)
    out["joint_force"] = [[float(x) for x in j["lam_p"] * rhs] for j in J]
    out["joint_torque"] = [[float(x) for x in (j["lam_a"] + j["lam_b"]) * rhs] for j in J]
    out["normal_impulse"], out["warm_start_normal_impulse"], out["warm_start_tangent_impulse"] = [], [], []
    for k, c in enumerate(C):
        for pi, p in enumerate(scene["manifolds"][k]["points"]):
            if c is None:
                continue
            cp = c["points"][pi]
            out["warm_start_normal_impulse"].append(float(cp["imp"]))
            out["warm_start_tangent_impulse"].append([float(x) for x in (cp["tangent"]["imp"] if cp["tangent"] is not None else [0, 0])])
            out["normal_impulse"].append(float(cp["total"]))
    out["softness"] = {"dynamic": {k: float(v) for k, v in soft_dyn.items()}, "non_dynamic": {k: float(v) for k, v in soft_nondyn.items()}}
    return out


# ---- sweep-and-prune by hand (collision/broad_phase.rs:373-474): literal insertion sort + double loop --------------------------------
def sweep_and_prune(intervals):
    """intervals: list of dicts {collider, body, min[3], max[3], memberships, filters, inactive}; returns the ordered pair list and the new
    persistent order (indices into the input list)."""
    order = list(range(len(intervals)))
    for i in range(1, len(order)):                        # insertion_sort: swap while strictly greater (broad_phase.rs:479-487)
        j = i
        while j > 0 and intervals[order[j - 1]]["min"][0] > intervals[order[j]]["min"][0]:
            order[j - 1], order[j] = order[j], order[j - 1]
            j -= 1
    pairs = []
    for a in range(len(order)):
        A = intervals[order[a]]
        for b in range(a + 1, len(order)):
            Bv = intervals[order[b]]
            if Bv["min"][0] > A["max"][0]:                # x-axis: break
                break
            if A["min"][1] > Bv["max"][1] or A["max"][1] < Bv["min"][1]:
                continue
            if A["min"][2] > Bv["max"][2] or A["max"][2] < Bv["min"][2]:
                continue
            if A["inactive"] and Bv["inactive"]:
                continue
            if not ((A["memberships"] & Bv["filters"]) != 0 and (Bv["memberships"] & A["filters"]) != 0):   # layers.rs:423-426
                continue
            if A["body"] == Bv["body"]:
                continue
            pairs.append((A["collider"], Bv["collider"]))
    return pairs, order
