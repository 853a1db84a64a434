"""An independent reference for the contact-manifold geometry of csrc/narrow_math.hpp, written from the geometry rather than from the header.

Methods (each different from the header's where a different one exists):
- rotation: the matrix of the quaternion divided by its norm (the header rotates by the sandwich product of the raw quaternion);
- point-box: clamp the point's local coordinates; the signed surface distance is max_k(|l_k| - h_k) inside, the clamped distance outside;
- SAT: the 15 axes with explicit overlaps |d.n| <= r_A + r_B; an edge axis whose cross product is shorter than EDGE_AXIS_MIN (1e-6,
  i.e. edges within 1e-6 rad of parallel) is skipped, the face axes cover that direction;
- box-box distance: feature enumeration, the 8 + 8 vertices against the other box and the 12 x 12 edge pairs with dependent clamping
  (Ericson, Real-Time Collision Detection §5.1.9), each candidate labelled with the features it joins;
- face-contact region: vertex enumeration in the reference face's 2-D frame (incident corners inside the rectangle, rectangle corners
  inside the incident quad, edge / edge crossings), lifted back onto the incident face; the header clips with Sutherland-Hodgman;
- spheres: closed forms, the centre-inside-the-box case pushes out through the nearest face.

Precision: the vectorised routines evaluate in float64 from the exact values of the input columns (an f32 column is widened
exactly).  `mp_box_box_distance` and `mp_sat` evaluate the same definitions in mpmath at 50 digits; the tests compare the two on a
sample of every class, which bounds the float64 reference's own error far below the tolerances the contract uses (a few ulps of the
column type times the scale of the pair).

Conventions restated from the Avian sources (no code copied):
- Keep rule (narrow_phase/system_param.rs, the retain closure of NarrowPhase::update): with rel = v2 - v1 the relative linear velocity,
  eff_margin = dt * |rel| (speculative margin unbounded), a point with penetration pen (positive = overlap) and normal speed
  ns = dot(rel + w2 x anchor2 - w1 x anchor1, n) is kept iff -pen < eff_margin or ns * dt - pen < eff_margin (both strict).
  The pair is searched up to max_dist = max(eff_margin, contact_tolerance).
- match_contacts (contact_types/mod.rs), feature ids unknown: a new point takes the impulses of the FIRST previous point such that
  |a1 - a1'|^2 < thr^2 and |a2 - a2'|^2 < thr^2, or |a1 - a2'|^2 < thr^2 and |a2 - a1'|^2 < thr^2 (strict, squared distances,
  thr = 0.1 * length_unit); otherwise it starts from zero.

Stated deviations from the reference that the tests pin:
- anchors are each shape's own witness point (anchor1 on A, anchor2 on B); the reference puts both at the midpoint;
- pruning keeps the deepest point, the point farthest from it and the two points farthest on either side of that segment, in their
  original order, and runs before the keep rule; the reference's prune_points keeps different points and runs after it.
"""
from __future__ import annotations

import itertools

import mpmath
import numpy as np

EDGE_AXIS_MIN = 1e-6
FACE_BIAS = 1e-4          # the header prefers a face axis unless an edge axis separates by more than this

# feature labels of a closest pair
VERTEX_FACE, EDGE_EDGE, VERTEX_OTHER = "face", "edge", "vertex"


# ---- rotations ---------------------------------------------------------------------------------------------------------------------
def rotation(q) -> np.ndarray:
    """(..., 4) quaternions (x, y, z, w) -> (..., 3, 3) rotation matrices of the normalised quaternions; columns = local axes."""
    q = np.asarray(q, dtype=np.float64)
    q = q / np.linalg.norm(q, axis=-1, keepdims=True)
    x, y, z, w = (q[..., i] for i in range(4))
    m = np.empty(q.shape[:-1] + (3, 3))
    m[..., 0, 0] = 1 - 2 * (y * y + z * z); m[..., 0, 1] = 2 * (x * y - z * w); m[..., 0, 2] = 2 * (x * z + y * w)
    m[..., 1, 0] = 2 * (x * y + z * w); m[..., 1, 1] = 1 - 2 * (x * x + z * z); m[..., 1, 2] = 2 * (y * z - x * w)
    m[..., 2, 0] = 2 * (x * z - y * w); m[..., 2, 1] = 2 * (y * z + x * w); m[..., 2, 2] = 1 - 2 * (x * x + y * y)
    return m


def mp_rotation(q):
    q = [mpmath.mpf(float(v)) for v in q]
    nq = mpmath.sqrt(sum(v * v for v in q))
    x, y, z, w = (v / nq for v in q)
    return mpmath.matrix([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                          [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                          [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


# ---- point / box ---------------------------------------------------------------------------------------------------------------------
def point_box(p, c, R, h):
    """Closest point of the box (centre c, rotation R, half extents h) to p, distance (0 inside) and the signed surface distance
    (negative inside).  Vectorised over leading axes."""
    l = np.einsum("...ji,...j->...i", R, p - c)
    cl = np.clip(l, -h, h)
    on = c + np.einsum("...ij,...j->...i", R, cl)
    dist = np.linalg.norm(p - on, axis=-1)
    inside = np.max(np.abs(l) - h, axis=-1)
    return on, dist, np.where(inside > 0, dist, inside)


def surface_distance(p, c, R, h):
    """|signed distance of p to the surface of the box|: 0 for a point on the boundary."""
    return np.abs(point_box(p, c, R, h)[2])


# ---- separating axes -----------------------------------------------------------------------------------------------------------------
def sat(ca, Ra, ha, cb, Rb, hb):
    """Minimum overlap over the 15 axes (negative: the largest separation) and its axis, oriented from A to B, and its kind
    ('face' or 'edge').  One pair, float64."""
    d = cb - ca
    best = (np.inf, None, None)
    axes = [(Ra[:, i], "face") for i in range(3)] + [(Rb[:, i], "face") for i in range(3)]
    for i in range(3):
        for j in range(3):
            c = np.cross(Ra[:, i], Rb[:, j])
            nc = np.linalg.norm(c)
            if nc > EDGE_AXIS_MIN:
                axes.append((c / nc, "edge"))
    for n, kind in axes:
        ov = np.abs(Ra.T @ n) @ ha + np.abs(Rb.T @ n) @ hb - abs(d @ n)
        if ov < best[0]:
            best = (ov, n if d @ n >= 0 else -n, kind)
    return best


def sat_overlaps(ca, Ra, ha, cb, Rb, hb):
    """Every axis' overlap (face axes of A, of B, then the edge axes that are not skipped), for tie detection."""
    d = cb - ca
    out = []
    ns = [Ra[:, i] for i in range(3)] + [Rb[:, i] for i in range(3)]
    for i in range(3):
        for j in range(3):
            c = np.cross(Ra[:, i], Rb[:, j])
            if np.linalg.norm(c) > EDGE_AXIS_MIN:
                ns.append(c / np.linalg.norm(c))
    for n in ns:
        out.append(np.abs(Ra.T @ n) @ ha + np.abs(Rb.T @ n) @ hb - abs(d @ n))
    return np.array(out)


def mp_sat(ca, qa, ha, cb, qb, hb, dps=50):
    """The minimum SAT overlap in mpmath at `dps` digits from the exact input values."""
    with mpmath.workdps(dps):
        Ra, Rb = mp_rotation(qa), mp_rotation(qb)
        d = [mpmath.mpf(float(cb[k])) - mpmath.mpf(float(ca[k])) for k in range(3)]
        ha = [mpmath.mpf(float(v)) for v in ha]; hb = [mpmath.mpf(float(v)) for v in hb]
        col = lambda R, i: [R[k, i] for k in range(3)]
        dot = lambda u, v: sum(x * y for x, y in zip(u, v))
        axes = [col(Ra, i) for i in range(3)] + [col(Rb, i) for i in range(3)]
        for i in range(3):
            for j in range(3):
                u, v = col(Ra, i), col(Rb, j)
                c = [u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]]
                nc = mpmath.sqrt(dot(c, c))
                if nc > EDGE_AXIS_MIN:
                    axes.append([x / nc for x in c])
        return min(sum(abs(dot(col(Ra, k), n)) * ha[k] for k in range(3)) + sum(abs(dot(col(Rb, k), n)) * hb[k] for k in range(3))
                   - abs(dot(d, n)) for n in axes)


# ---- features ------------------------------------------------------------------------------------------------------------------------
_SIGNS = np.array(list(itertools.product((-1.0, 1.0), repeat=3)))


def vertices(c, R, h):
    return c + (_SIGNS * h) @ R.T


def edges(c, R, h):
    """12 edges as (start, end, axis)."""
    out = []
    for ax in range(3):
        o = [k for k in range(3) if k != ax]
        for s1, s2 in itertools.product((-1.0, 1.0), repeat=2):
            l = np.zeros(3); l[o[0]] = s1 * h[o[0]]; l[o[1]] = s2 * h[o[1]]
            a, b = l.copy(), l.copy(); a[ax], b[ax] = -h[ax], h[ax]
            out.append((c + R @ a, c + R @ b, ax))
    return out


def segment_segment(p1, q1, p2, q2):
    """Closest points of two segments with dependent clamping; returns (point on 1, point on 2, s, t) with s, t in [0, 1]."""
    d1, d2, r = q1 - p1, q2 - p2, p1 - p2
    a, e, f = d1 @ d1, d2 @ d2, d2 @ r
    c, b = d1 @ r, d1 @ d2
    den = a * e - b * b
    s = float(np.clip((b * f - c * e) / den, 0.0, 1.0)) if den > 1e-14 * a * e else 0.0
    t = (b * s + f) / e
    if t < 0.0:
        t, s = 0.0, float(np.clip(-c / a, 0.0, 1.0))
    elif t > 1.0:
        t, s = 1.0, float(np.clip((b - c) / a, 0.0, 1.0))
    return p1 + d1 * s, p2 + d2 * t, s, t


def box_box_distance(ca, Ra, ha, cb, Rb, hb, end_tol=1e-9):
    """Exact distance of two boxes (0 when they overlap) by feature enumeration.  Returns (distance, point on A, point on B, label,
    candidates) where label is VERTEX_FACE, EDGE_EDGE or VERTEX_OTHER for the closest candidate and candidates lists every
    (distance, point on A, point on B, label) for tie detection."""
    cands = []
    for side, (c1, R1, h1, c2, R2, h2) in enumerate(((ca, Ra, ha, cb, Rb, hb), (cb, Rb, hb, ca, Ra, ha))):
        for v in vertices(c1, R1, h1):
            on, dist, _ = point_box(v, c2, R2, h2)
            l = R2.T @ (on - c2)
            on_face_only = int(np.sum(np.abs(np.abs(l) - h2) <= end_tol * (1 + np.abs(h2)))) == 1
            lab = VERTEX_FACE if on_face_only else VERTEX_OTHER
            cands.append((dist, v, on, lab) if side == 0 else (dist, on, v, lab))
    ea, eb = edges(ca, Ra, ha), edges(cb, Rb, hb)
    for (p1, q1, _) in ea:
        for (p2, q2, _) in eb:
            x, y, s, t = segment_segment(p1, q1, p2, q2)
            interior = end_tol < s < 1 - end_tol and end_tol < t < 1 - end_tol
            cands.append((float(np.linalg.norm(y - x)), x, y, EDGE_EDGE if interior else VERTEX_OTHER))
    cands.sort(key=lambda c: c[0])
    d, x, y, lab = cands[0]
    return d, x, y, lab, cands


def mp_box_box_distance(ca, qa, ha, cb, qb, hb, dps=50):
    """The box-box distance in mpmath at `dps` digits: the same enumeration, evaluated from the exact input values."""
    with mpmath.workdps(dps):
        M = lambda v: [mpmath.mpf(float(x)) for x in v]
        Ra, Rb = mp_rotation(qa), mp_rotation(qb)
        ca, cb, ha, hb = M(ca), M(cb), M(ha), M(hb)
        dot = lambda u, v: sum(x * y for x, y in zip(u, v))
        sub = lambda u, v: [x - y for x, y in zip(u, v)]
        add = lambda u, v: [x + y for x, y in zip(u, v)]
        mul = lambda u, s: [x * s for x in u]
        col = lambda R, i: [R[k, i] for k in range(3)]
        clamp = lambda x, lo, hi: lo if x < lo else (hi if x > hi else x)

        def world(c, R, l):
            return add(c, [sum(R[k, i] * l[i] for i in range(3)) for k in range(3)])

        def pbox(p, c, R, h):
            d = sub(p, c)
            l = [clamp(dot(d, col(R, i)), -h[i], h[i]) for i in range(3)]
            e = sub(p, world(c, R, l))
            return mpmath.sqrt(dot(e, e))

        def segs(c, R, h):
            out = []
            for ax in range(3):
                o = [k for k in range(3) if k != ax]
                for s1, s2 in itertools.product((-1, 1), repeat=2):
                    l = [0, 0, 0]; l[o[0]] = s1 * h[o[0]]; l[o[1]] = s2 * h[o[1]]
                    a, b = list(l), list(l); a[ax], b[ax] = -h[ax], h[ax]
                    out.append((world(c, R, a), world(c, R, b)))
            return out

        best = mpmath.inf
        for c1, R1, h1, c2, R2, h2 in ((ca, Ra, ha, cb, Rb, hb), (cb, Rb, hb, ca, Ra, ha)):
            for sg in itertools.product((-1, 1), repeat=3):
                best = min(best, pbox(world(c1, R1, [sg[i] * h1[i] for i in range(3)]), c2, R2, h2))
        for p1, q1 in segs(ca, Ra, ha):
            for p2, q2 in segs(cb, Rb, hb):
                d1, d2, r = sub(q1, p1), sub(q2, p2), sub(p1, p2)
                a, e, f, c, b = dot(d1, d1), dot(d2, d2), dot(d2, r), dot(d1, r), dot(d1, d2)
                den = a * e - b * b
                s = clamp((b * f - c * e) / den, 0, 1) if den > mpmath.mpf(10) ** (-30) else mpmath.mpf(0)
                t = (b * s + f) / e
                if t < 0:
                    t, s = mpmath.mpf(0), clamp(-c / a, 0, 1)
                elif t > 1:
                    t, s = mpmath.mpf(1), clamp((b - c) / a, 0, 1)
                w = sub(add(p1, mul(d1, s)), add(p2, mul(d2, t)))
                best = min(best, mpmath.sqrt(dot(w, w)))
        return best


# ---- face-contact region -------------------------------------------------------------------------------------------------------------
def face_region(c_ref, R_ref, h_ref, axis, sign, c_inc, R_inc, h_inc):
    """The part of the incident box's face most anti-parallel to the reference face (axis, sign) that lies over the reference
    face: vertex enumeration in the reference face's (u, v) frame, lifted back onto the incident face.  Returns (k, 3) points
    (world) and their heights above the reference face (negative: below it)."""
    rn = R_ref[:, axis] * sign
    u, v = [k for k in range(3) if k != axis]
    eu, ev = R_ref[:, u], R_ref[:, v]
    # incident face: the face of the incident box whose outward normal is most anti-parallel to rn
    k = int(np.argmax(np.abs(R_inc.T @ rn)))
    s = -np.sign(R_inc[:, k] @ rn) or 1.0
    o = [m for m in range(3) if m != k]
    fc = c_inc + R_inc[:, k] * (s * h_inc[k])
    quad = [fc + R_inc[:, o[0]] * (a * h_inc[o[0]]) + R_inc[:, o[1]] * (b * h_inc[o[1]]) for a, b in ((1, 1), (-1, 1), (-1, -1), (1, -1))]
    to2 = lambda p: np.array([(p - c_ref) @ eu, (p - c_ref) @ ev])
    q2 = [to2(p) for p in quad]
    hu, hv = h_ref[u], h_ref[v]
    rect = [np.array(x) for x in ((hu, hv), (-hu, hv), (-hu, -hv), (hu, -hv))]
    eps = 1e-12 * (1 + hu + hv + np.abs(q2).max())

    def cross2(p, q):
        return p[0] * q[1] - p[1] * q[0]

    def in_rect(p):
        return abs(p[0]) <= hu + eps and abs(p[1]) <= hv + eps

    def in_quad(p):
        signs = [cross2(q2[(i + 1) % 4] - q2[i], p - q2[i]) for i in range(4)]
        return all(x >= -eps for x in signs) or all(x <= eps for x in signs)

    pts2 = [p for p in q2 if in_rect(p)] + [p for p in rect if in_quad(p)]
    for i in range(4):
        a, b = q2[i], q2[(i + 1) % 4]
        for j in range(4):
            c, d = rect[j], rect[(j + 1) % 4]
            den = cross2(b - a, d - c)
            if abs(den) < 1e-15:
                continue
            t = cross2(c - a, d - c) / den
            w = cross2(c - a, b - a) / den
            if -1e-12 <= t <= 1 + 1e-12 and -1e-12 <= w <= 1 + 1e-12:
                pts2.append(a + (b - a) * t)
    # lift back onto the incident face plane along rn
    n_inc = R_inc[:, k] * s
    out = []
    for p in pts2:
        base = c_ref + eu * p[0] + ev * p[1]
        # base + rn * z lies on the incident plane: dot(base + rn z - fc, n_inc) = 0
        z = (fc - base) @ n_inc / (rn @ n_inc)
        out.append(base + rn * z)
    out = np.array(out).reshape(-1, 3)
    height = (out - c_ref) @ rn - h_ref[axis]
    return out, height


# ---- spheres -------------------------------------------------------------------------------------------------------------------------
def sphere_sphere(ca, ra, cb, rb):
    """(normal from A to B, gap = |d| - ra - rb); the normal is undefined (None) for coincident centres."""
    d = np.asarray(cb, float) - np.asarray(ca, float)
    l = float(np.linalg.norm(d))
    return (d / l if l > 0 else None), l - ra - rb


def sphere_box(c, R, h, cs, rs):
    """Sphere against box: (normal from the box to the sphere, gap, point on the box).  A centre inside the box leaves through the
    face of least depth; the gap is then -(depth + rs)."""
    on, dist, signed = point_box(cs, c, R, h)
    if dist > 0:
        return (cs - on) / dist, dist - rs, on
    l = R.T @ (cs - c)
    depth = h - np.abs(l)
    ax = int(np.argmin(depth))
    n = R[:, ax] * (1.0 if l[ax] >= 0 else -1.0)
    return n, -(depth[ax] + rs), cs + n * depth[ax]


# ---- keep rule and matching ----------------------------------------------------------------------------------------------------------
def keep(penetration, normal_speed, dt, eff_margin) -> bool:
    return bool(-penetration < eff_margin or normal_speed * dt - penetration < eff_margin)


def normal_speed(rel, w1, w2, anchor1, anchor2, n):
    return float((rel + np.cross(w2, anchor2) - np.cross(w1, anchor1)) @ n)


def match_contacts(new_a1, new_a2, old_a1, old_a2, threshold) -> int:
    """Index of the previous point whose impulses the new point inherits, or -1."""
    t2 = threshold * threshold
    d2 = lambda x, y: float(np.sum((np.asarray(x, float) - np.asarray(y, float)) ** 2))
    for k in range(len(old_a1)):
        if (d2(new_a1, old_a1[k]) < t2 and d2(new_a2, old_a2[k]) < t2) or (d2(new_a1, old_a2[k]) < t2 and d2(new_a2, old_a1[k]) < t2):
            return k
    return -1
