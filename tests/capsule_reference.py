"""TEST INFRASTRUCTURE: an independent float64 restatement of the capsule geometry, written from the definitions (a capsule is the set of points
within `radius` of its segment) and not from csrc/narrow_math.hpp.  Distances are found by enumerating the candidate feature pairs; the depth of
an overlapping segment and box by the 6-axis separating-axis test.  `mp_segment_distance` repeats the segment distance at 50 digits
(mpmath) to bound this module's own rounding, as tests/narrow_reference.py does for the box geometry."""
from __future__ import annotations

import numpy as np

EDGE_AXIS_MIN = 1e-6   # e_k x s axes shorter than this are skipped (the segment is parallel to that box edge)


def quat_rotate(q, v):
    """v rotated by the unit quaternion q = (x, y, z, w), float64"""
    q = np.asarray(q, dtype=np.float64)
    b, w = q[:3], q[3]
    v = np.asarray(v, dtype=np.float64)
    return v * (w * w - b @ b) + b * (2.0 * (v @ b)) + np.cross(b, v) * (2.0 * w)


def quat_matrix(q):
    return np.stack([quat_rotate(q, e) for e in np.eye(3)], axis=1)   # columns: the local axes in the world


def capsule_segment(pos, rot, half_length):
    """the two end points of a capsule's segment, (0, -+half_length, 0) in the collider frame"""
    u = quat_rotate(rot, [0.0, 1.0, 0.0])
    p = np.asarray(pos, dtype=np.float64)
    return p - u * half_length, p + u * half_length


def point_segment(p, a, b):
    """the point of segment ab closest to p"""
    d = b - a
    dd = d @ d
    t = 0.0 if dd == 0.0 else min(1.0, max(0.0, ((p - a) @ d) / dd))
    return a + d * t


def segment_segment(p0, p1, q0, q1):
    """(distance, point on p, point on q): the minimum over the four end point projections and the interior stationary point of the 2x2
    normal equations (when it lies inside both segments)"""
    cands = []
    for p in (p0, p1):
        q = point_segment(p, q0, q1)
        cands.append((np.linalg.norm(p - q), p, q))
    for q in (q0, q1):
        p = point_segment(q, p0, p1)
        cands.append((np.linalg.norm(p - q), p, q))
    d1, d2, r = p1 - p0, q1 - q0, p0 - q0
    a, e, b = d1 @ d1, d2 @ d2, d1 @ d2
    den = a * e - b * b
    if den > 1e-14 * a * e:
        c, f = d1 @ r, d2 @ r
        s = (b * f - c * e) / den
        t = (a * f - b * c) / den
        if 0.0 < s < 1.0 and 0.0 < t < 1.0:
            p, q = p0 + d1 * s, q0 + d2 * t
            cands.append((np.linalg.norm(p - q), p, q))
    return min(cands, key=lambda x: x[0])


def point_box(p, c, R, he):
    """(distance, closest point) of point p and the box (centre c, rotation columns R, half extents he); 0 inside"""
    local = R.T @ (np.asarray(p) - c)
    cl = np.clip(local, -he, he)
    q = c + R @ cl
    return np.linalg.norm(p - q), q


def segment_hits_box(p0, p1, c, R, he):
    """the segment meets the box: clip it against the three slabs in the box frame"""
    a, b = R.T @ (p0 - c), R.T @ (p1 - c)
    lo, hi = 0.0, 1.0
    for k in range(3):
        d = b[k] - a[k]
        if abs(d) < 1e-300:
            if abs(a[k]) > he[k]:
                return False
            continue
        t0, t1 = (-he[k] - a[k]) / d, (he[k] - a[k]) / d
        lo, hi = max(lo, min(t0, t1)), min(hi, max(t0, t1))
    return lo <= hi


def box_edges(c, R, he):
    for k in range(3):
        u, v = (k + 1) % 3, (k + 2) % 3
        for su in (-1, 1):
            for sv in (-1, 1):
                m = c + R[:, u] * (su * he[u]) + R[:, v] * (sv * he[v])
                yield m - R[:, k] * he[k], m + R[:, k] * he[k]


def segment_box(p0, p1, c, R, he):
    """(distance, point on the segment, point on the box): 0 when they meet, else the minimum over both end points against the box and the
    segment against the 12 edges (a disjoint segment's closest box point lies on a face only when an end point's does)"""
    if segment_hits_box(p0, p1, c, R, he):
        return 0.0, None, None
    cands = []
    for p in (p0, p1):
        d, q = point_box(p, c, R, he)
        cands.append((d, p, q))
    for e0, e1 in box_edges(c, R, he):
        cands.append(segment_segment(p0, p1, e0, e1))
    return min(cands, key=lambda x: x[0])


def sat_overlap(p0, p1, c, R, he):
    """the least overlap of the segment and the box over the box's 3 face normals and e_k x s (exact for a segment against a box); negative
    when an axis separates them"""
    s = p1 - p0
    sl = np.linalg.norm(s)
    u = s / sl if sl > 0 else np.array([0.0, 1.0, 0.0])
    h = 0.5 * sl
    m = 0.5 * (p0 + p1)
    axes = [R[:, k] for k in range(3)] + [np.cross(R[:, k], u) for k in range(3)]
    best = np.inf
    for n in axes:
        ln = np.linalg.norm(n)
        if ln < EDGE_AXIS_MIN:
            continue
        n = n / ln
        rb = np.abs(R.T @ n) @ he
        best = min(best, rb + h * abs(u @ n) - abs((m - c) @ n))
    return best


def capsule_depth(shape_a, dims_a, pos_a, rot_a, shape_b, dims_b, pos_b, rot_b):
    """(distance, depth) of a pair with at least one capsule: distance between the surfaces when apart (else 0), penetration depth when they
    overlap (else 0).  Capsule-box depth: the SAT overlap plus the radius when the segment meets the box, the radius minus the segment's
    distance otherwise."""
    from avian_b200.fixture import SHAPE_CAPSULE, SHAPE_CUBOID, SHAPE_SPHERE
    if shape_a != SHAPE_CAPSULE:
        return capsule_depth(shape_b, dims_b, pos_b, rot_b, shape_a, dims_a, pos_a, rot_a)
    p0, p1 = capsule_segment(pos_a, rot_a, dims_a[1])
    r = dims_a[0]
    if shape_b == SHAPE_CUBOID:
        c, R, he = np.asarray(pos_b, float), quat_matrix(rot_b), np.asarray(dims_b, float)
        d, _, _ = segment_box(p0, p1, c, R, he)
        if d == 0.0:
            return 0.0, sat_overlap(p0, p1, c, R, he) + r
        return max(d - r, 0.0), max(r - d, 0.0)
    if shape_b == SHAPE_SPHERE:
        q0 = q1 = np.asarray(pos_b, float)
        rb = dims_b[0]
    else:
        q0, q1 = capsule_segment(pos_b, rot_b, dims_b[1])
        rb = dims_b[0]
    d = segment_segment(p0, p1, q0, q1)[0]
    return max(d - r - rb, 0.0), max(r + rb - d, 0.0)


def surface_distance(shape, dims, pos, rot, x):
    """|signed distance| of point x to the surface of a shape (0 on it)"""
    from avian_b200.fixture import SHAPE_CAPSULE, SHAPE_CUBOID
    x = np.asarray(x, float)
    if shape == SHAPE_CAPSULE:
        p0, p1 = capsule_segment(pos, rot, dims[1])
        return abs(np.linalg.norm(x - point_segment(x, p0, p1)) - dims[0])
    if shape == SHAPE_CUBOID:
        R, he = quat_matrix(rot), np.asarray(dims, float)
        local = R.T @ (x - np.asarray(pos, float))
        q = np.abs(local) - he
        outside = np.linalg.norm(np.maximum(q, 0.0))
        inside = min(max(q[0], q[1], q[2]), 0.0)
        return abs(outside + inside)
    return abs(np.linalg.norm(x - np.asarray(pos, float)) - dims[0])


def capsule_aabb(dtype, dims, pos, rot):
    """parry3d's Capsule::aabb in the column type, operation by operation as the device evaluates it: the segment's end points rotated by
    nalgebra's UnitQuaternion * Vector3 (t = 2 (q.xyz x v); v + q.xyz x t + t w) plus the position, their min / max, loosened by the radius"""
    f = np.dtype(dtype).type
    d = [f(x) for x in dims]
    p = [f(x) for x in pos]
    q = [f(x) for x in rot]
    b = q[:3]

    def cross(a, c):
        return [a[1] * c[2] - a[2] * c[1], a[2] * c[0] - a[0] * c[2], a[0] * c[1] - a[1] * c[0]]

    ends = []
    for hy in (-d[1], d[1]):
        v = [f(0), hy, f(0)]
        t = [x * f(2) for x in cross(b, v)]
        bt = cross(b, t)
        ends.append([((v[k] + bt[k]) + t[k] * q[3]) + p[k] for k in range(3)])
    mn = [min(ends[0][k], ends[1][k]) - d[0] for k in range(3)]
    mx = [max(ends[0][k], ends[1][k]) + d[0] for k in range(3)]
    return np.array(mn, dtype=dtype), np.array(mx, dtype=dtype)


def swept_capsule_aabb(dtype, dims, pos, rot, lin_vel, dt, margin, tol):
    """update_aabb's swept box of a capsule with no angular velocity, in the column type operation by operation: the end pose is
    fast_renormalize(identity * rot) and pos + clamp_length_max(lin_vel * dt, max(margin, tol)); the two poses' boxes are merged and grown by
    tol (no collision margin).  margin = inf stands for Scalar::MAX."""
    f = np.dtype(dtype).type
    q = [f(x) for x in rot]
    i = [f(0), f(0), f(0), f(1)]
    if np.dtype(dtype) == np.float32:     # Quat * Quat as glam's f32 evaluation groups it
        r = [(i[3] * q[0] + i[0] * q[3]) + (i[1] * q[2] - i[2] * q[1]), (i[3] * q[1] - i[0] * q[2]) + (i[1] * q[3] + i[2] * q[0]),
             (i[3] * q[2] + i[0] * q[1]) + (i[2] * q[3] - i[1] * q[0]), (i[3] * q[3] - i[0] * q[0]) + (-(i[1] * q[1]) - i[2] * q[2])]
    else:
        r = [i[3] * q[0] + i[0] * q[3] + i[1] * q[2] - i[2] * q[1], i[3] * q[1] - i[0] * q[2] + i[1] * q[3] + i[2] * q[0],
             i[3] * q[2] + i[0] * q[1] - i[1] * q[0] + i[2] * q[3], i[3] * q[3] - i[0] * q[0] - i[1] * q[1] - i[2] * q[2]]
    l2 = ((r[0] * r[0] + r[1] * r[1]) + r[2] * r[2]) + r[3] * r[3]
    k = f(0.5) * (f(3) - l2)
    end_rot = [x * k for x in r]
    m = np.finfo(dtype).max if np.isinf(margin) else f(margin)
    m = max(f(m), f(tol))
    a = [f(v) * f(dt) for v in lin_vel]
    la = (a[0] * a[0] + a[1] * a[1]) + a[2] * a[2]
    with np.errstate(over="ignore"):
        if la > m * m:
            sq = f(np.sqrt(la))
            a = [m * (x / sq) for x in a]
    end_pos = [f(x) + y for x, y in zip(pos, a)]
    mn0, mx0 = capsule_aabb(dtype, dims, pos, rot)
    mn1, mx1 = capsule_aabb(dtype, dims, end_pos, end_rot)
    g = f(tol)
    return np.minimum(mn0, mn1) - g, np.maximum(mx0, mx1) + g


def mp_segment_distance(p0, p1, q0, q1, digits: int = 50) -> float:
    """segment_segment's distance at `digits` digits: the same enumeration in mpmath"""
    import mpmath
    mpmath.mp.dps = digits
    P0, P1, Q0, Q1 = (mpmath.matrix([mpmath.mpf(float(x)) for x in v]) for v in (p0, p1, q0, q1))

    def dot(a, b):
        return sum(a[i] * b[i] for i in range(3))

    def pseg(p, a, b):
        d = b - a
        dd = dot(d, d)
        t = mpmath.mpf(0) if dd == 0 else min(mpmath.mpf(1), max(mpmath.mpf(0), dot(p - a, d) / dd))
        return a + d * t

    def norm(a):
        return mpmath.sqrt(dot(a, a))

    best = min([norm(p - pseg(p, Q0, Q1)) for p in (P0, P1)] + [norm(q - pseg(q, P0, P1)) for q in (Q0, Q1)])
    d1, d2, r = P1 - P0, Q1 - Q0, P0 - Q0
    a, e, b = dot(d1, d1), dot(d2, d2), dot(d1, d2)
    den = a * e - b * b
    if den > 0:
        c, f = dot(d1, r), dot(d2, r)
        s, t = (b * f - c * e) / den, (a * f - b * c) / den
        if 0 < s < 1 and 0 < t < 1:
            best = min(best, norm(P0 + d1 * s - Q0 - d2 * t))
    return float(best)
