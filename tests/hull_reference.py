"""An independent float64 restatement of the convex hull contact geometry (DESIGN.md §7k) that the tests check csrc/hull_math.hpp against.
It does not use the header's algorithm: the SAT runs over every face normal and every edge pair (no Gauss-map pruning), true distances come
from brute-force feature enumeration (vertex-face, edge-edge, and the segment clipped by every face plane), and spheres and capsules are
closed forms over those distances.  Shapes are (vertices [v,3] world, faces: loops counter-clockwise from outside)."""
import numpy as np

from capsule_reference import point_segment, quat_matrix, segment_segment

CUBE_FACES = [[1, 3, 7, 5], [0, 4, 6, 2], [2, 6, 7, 3], [0, 1, 5, 4], [4, 5, 7, 6], [0, 2, 3, 1]]


def posed(vertices, pos, rot):
    return np.asarray(vertices, float) @ quat_matrix(np.asarray(rot, float)).T + np.asarray(pos, float)


def box_poly(he, pos, rot):
    v = np.array([[(1 if m & 1 else -1) * he[0], (1 if m & 2 else -1) * he[1], (1 if m & 4 else -1) * he[2]] for m in range(8)], float)
    return posed(v, pos, rot), CUBE_FACES


def planes(V, faces):
    """unit outward normal and offset of every face, from the fan triangles' cross products"""
    out = []
    for f in faces:
        p = V[list(f)]
        n = sum(np.cross(p[k] - p[0], p[k + 1] - p[0]) for k in range(1, len(f) - 1))
        n = n / np.linalg.norm(n)
        out.append((n, float(np.mean(p @ n))))
    return out


def edges(faces):
    es = set()
    for f in faces:
        for i in range(len(f)):
            a, b = int(f[i]), int(f[(i + 1) % len(f)])
            es.add((min(a, b), max(a, b)))
    return sorted(es)


def _in_face(V, f, n, q, tol=1e-12):
    p = V[list(f)]
    return all(np.cross(p[(i + 1) % len(f)] - p[i], n) @ (q - p[i]) <= tol for i in range(len(f)))


def point_distance(x, V, faces):
    """signed distance of x to the polyhedron: negative inside (the largest face-plane distance), the true distance outside"""
    pl = planes(V, faces)
    h = max(n @ x - d for n, d in pl)
    if h <= 0:
        return h
    best = np.inf
    for (n, d), f in zip(pl, faces):
        s = n @ x - d
        if s > 0 and _in_face(V, f, n, x - n * s):
            best = min(best, s)
    for a, b in edges(faces):
        best = min(best, np.linalg.norm(x - point_segment(x, V[a], V[b])))
    return best


def distance(VA, FA, VB, FB):
    """the distance of two disjoint polyhedra by feature enumeration (vertex-face both ways, edge-edge)"""
    best = np.inf
    for V, F, W, G in ((VA, FA, VB, FB), (VB, FB, VA, FA)):
        for (n, d), g in zip(planes(W, G), G):
            for x in V:
                s = n @ x - d
                if s >= 0 and _in_face(W, g, n, x - n * s):
                    best = min(best, s)
    for a, b in edges(FA):
        for c, e in edges(FB):
            best = min(best, segment_segment(VA[a], VA[b], VB[c], VB[e])[0])
    return best


def sat(VA, FA, VB, FB):
    """(largest separation, least overlap) over every face normal of both and every edge-pair cross product"""
    axes = [n for n, _ in planes(VA, FA)] + [n for n, _ in planes(VB, FB)]
    for a, b in edges(FA):
        for c, e in edges(FB):
            x = np.cross(VA[b] - VA[a], VB[e] - VB[c])
            l = np.linalg.norm(x)
            if l > 1e-9 * np.linalg.norm(VA[b] - VA[a]) * np.linalg.norm(VB[e] - VB[c]):
                axes.append(x / l)
    sep, overlap = -np.inf, np.inf
    for n in axes:
        pa, pb = VA @ n, VB @ n
        o = min(pa.max() - pb.min(), pb.max() - pa.min())
        sep = max(sep, -o)
        overlap = min(overlap, o)
    return sep, overlap


def segment_clip(p0, p1, V, faces):
    """the part of segment p0 p1 inside the polyhedron, as parameters (t0, t1) of p0 + t (p1 - p0), or None"""
    t0, t1 = 0.0, 1.0
    for n, d in planes(V, faces):
        a, g = n @ p0 - d, n @ (p1 - p0)
        if abs(g) < 1e-15:
            if a > 0:
                return None
            continue
        t = -a / g
        if g > 0:
            t1 = min(t1, t)
        else:
            t0 = max(t0, t)
    return (t0, t1) if t0 <= t1 else None


def segment_distance(p0, p1, V, faces):
    """the distance of a segment to the polyhedron (0 when it meets it)"""
    if segment_clip(p0, p1, V, faces) is not None:
        return 0.0
    best = min(point_distance(p0, V, faces), point_distance(p1, V, faces))
    for a, b in edges(faces):
        best = min(best, segment_segment(p0, p1, V[a], V[b])[0])
    return best


def segment_depth(p0, p1, r, V, faces):
    """the least overlap of a capsule whose segment meets the polyhedron: a SAT over the face normals and every edge x axis direction"""
    u = p1 - p0
    axes = [n for n, _ in planes(V, faces)]
    for a, b in edges(faces):
        x = np.cross(V[b] - V[a], u)
        l = np.linalg.norm(x)
        if l > 1e-6 * np.linalg.norm(V[b] - V[a]) * np.linalg.norm(u):
            axes.append(x / l)
    best = np.inf
    for n in axes:
        pv, ps = V @ n, np.array([p0 @ n, p1 @ n])
        best = min(best, min(pv.max() - ps.min(), ps.max() - pv.min()) + r)
    return best


def hull_aabb(dtype, vertices, pos, rot):
    """parry3d's ConvexPolyhedron::aabb in the column type, operation by operation as the device evaluates it: every vertex rotated by
    nalgebra's UnitQuaternion * Vector3 (t = 2 (q.xyz x v); v + q.xyz x t + t w) plus the position, their min / max"""
    f = np.dtype(dtype).type
    p = [f(x) for x in pos]
    q = [f(x) for x in rot]
    b = q[:3]

    def cross(a, c):
        return [a[1] * c[2] - a[2] * c[1], a[2] * c[0] - a[0] * c[2], a[0] * c[1] - a[1] * c[0]]

    pts = []
    for v in np.asarray(vertices, dtype=dtype):
        v = [f(x) for x in v]
        t = [x * f(2) for x in cross(b, v)]
        bt = cross(b, t)
        pts.append([((v[k] + bt[k]) + t[k] * q[3]) + p[k] for k in range(3)])
    pts = np.array(pts, dtype=dtype)
    return pts.min(axis=0), pts.max(axis=0)


def swept_hull_aabb(dtype, vertices, pos, rot, lin_vel, dt, margin, tol):
    """update_aabb's swept box of a hull with no angular velocity, in the column type: the end pose as capsule_reference.swept_capsule_aabb
    computes it (fast_renormalize(identity * rot), pos + clamp_length_max(lin_vel * dt, max(margin, tol))), the two poses' boxes merged and
    grown by tol"""
    f = np.dtype(dtype).type
    q = [f(x) for x in rot]
    i = [f(0), f(0), f(0), f(1)]
    if np.dtype(dtype) == np.float32:
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
    mn0, mx0 = hull_aabb(dtype, vertices, pos, rot)
    mn1, mx1 = hull_aabb(dtype, vertices, end_pos, end_rot)
    g = f(tol)
    return np.minimum(mn0, mn1) - g, np.maximum(mx0, mx1) + g
