"""An independent float64 restatement of the convex hull query contract (DESIGN.md §7l) that the tests check csrc/hull_query_math.hpp against,
built on tests/hull_reference.py.  It shares no algorithm with the header: rays and polytope casts are linear programs over the face
half-spaces (scipy.optimize.linprog, minimising t; no Cyrus-Beck, no Gauss-map pruning), sphere and capsule casts bisect hull_reference's
distances, which are convex in t along a straight sweep.  Shapes are (vertices [v,3] world, faces: loops counter-clockwise from outside)."""
import numpy as np
from scipy.optimize import linprog

import hull_reference as hr


def table_poly(hulls, h):
    """hull h of an api.ConvexHulls as (local vertices, face loops of local vertex indices)"""
    v0, v1 = int(hulls.vertex_offsets[h]), int(hulls.vertex_offsets[h + 1])
    V = np.asarray(hulls.vertices, float).reshape(-1, 3)[v0:v1]
    lo, lp = np.asarray(hulls.loop_offsets), np.asarray(hulls.loop)
    faces = [list(lp[lo[f]:lo[f + 1]]) for f in range(int(hulls.face_offsets[h]), int(hulls.face_offsets[h + 1]))]
    return V, faces


def ray_lp(o, d, V, faces, maxd):
    """the smallest t in [0, maxd] with o + t d inside every face half-space, or None"""
    pl = hr.planes(V, faces)
    A = np.array([[n @ d] for n, _ in pl])
    b = np.array([c - n @ o for n, c in pl])
    res = linprog([1.0], A_ub=A, b_ub=b, bounds=[(0.0, maxd)], method="highs")
    return float(res.x[0]) if res.status == 0 else None


def poly_cast_lp(VA, FA, VB, FB, d, maxd):
    """the smallest t in [0, maxd] at which polytope A moved by t d meets B: some x lies in B and x - t d in A"""
    rows, rhs = [], []
    for n, c in hr.planes(VA, FA):
        rows.append([*n, -(n @ d)])
        rhs.append(c)
    for n, c in hr.planes(VB, FB):
        rows.append([*n, 0.0])
        rhs.append(c)
    res = linprog([0.0, 0.0, 0.0, 1.0], A_ub=np.array(rows), b_ub=np.array(rhs), bounds=[(None, None)] * 3 + [(0.0, maxd)], method="highs")
    return float(res.x[3]) if res.status == 0 else None


def first_contact(gap, maxd, iters=80):
    """the smallest t in [0, maxd] with gap(t) <= 0 for a gap convex in t (0 when it already is), or None"""
    if gap(0.0) <= 0:
        return 0.0
    lo, hi = 0.0, maxd
    for _ in range(iters):                      # the minimum of the convex gap
        m1, m2 = lo + (hi - lo) / 3, hi - (hi - lo) / 3
        if gap(m1) < gap(m2):
            hi = m2
        else:
            lo = m1
    tm = 0.5 * (lo + hi)
    if gap(tm) > 0:
        return None
    lo, hi = 0.0, tm
    for _ in range(iters):
        mid = 0.5 * (lo + hi)
        if gap(mid) <= 0:
            hi = mid
        else:
            lo = mid
    return hi


def sphere_cast(c, r, d, V, faces, maxd):
    """a sphere (centre c, radius r) moving along d against the polytope"""
    return first_contact(lambda t: hr.point_distance(c + t * d, V, faces) - r, maxd)


def capsule_cast(p0, p1, r, d, V, faces, maxd):
    """a capsule (segment p0 p1, radius r) moving along d against the polytope"""
    return first_contact(lambda t: hr.segment_distance(p0 + t * d, p1 + t * d, V, faces) - r, maxd)


def project(x, V, faces, solid=True):
    """(projection, inside) onto the closed polytope: the closest point outside; x itself inside when solid; the plane of the face of largest
    signed distance inside when hollow (the first such face on a tie)"""
    pl = hr.planes(V, faces)
    h = [n @ x - c for n, c in pl]
    k = int(np.argmax(h))
    if h[k] <= 0:
        return (x.copy() if solid else x - pl[k][0] * h[k]), True
    best, on = np.inf, None
    for (n, c), f in zip(pl, faces):
        s = n @ x - c
        q = x - n * s
        if s > 0 and hr._in_face(V, f, n, q) and s < best:
            best, on = s, q
    for a, b in hr.edges(faces):
        q = hr.point_segment(x, V[a], V[b])
        if np.linalg.norm(x - q) < best:
            best, on = np.linalg.norm(x - q), q
    return on, False
