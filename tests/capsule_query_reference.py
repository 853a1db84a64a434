"""TEST INFRASTRUCTURE: an independent float64 restatement of the capsule spatial queries (ray casts and point projection), written from the
definition of a capsule (the set of points within `radius` of its segment) and not from csrc/query_math.hpp.  It builds on the segment
helpers of tests/capsule_reference.py.  `mp_point_segment_distance` repeats a point-segment distance at 50 digits (mpmath) to bound the
rounding of a ray hit computed in float64."""
from __future__ import annotations

import numpy as np

from capsule_reference import point_segment


def segment_distance(x, p0, p1):
    x = np.asarray(x, float)
    return float(np.linalg.norm(x - point_segment(x, p0, p1)))


def ray_capsule(o, d, p0, p1, r, solid=True, t_max=1e6):
    """(t, normal) of the ray o + t d against the capsule, or None.  f(t) = dist(o + t d, segment) is convex in t, so the entry is the first
    root of f = r left of f's minimum (golden-section search) and the exit of a ray starting inside the root right of it; both by bisection.
    Independent of csrc/query_math.hpp's closed form."""
    o, d = np.asarray(o, float), np.asarray(d, float)
    f = lambda t: segment_distance(o + d * t, p0, p1)
    if f(0.0) <= r:
        if solid:
            return 0.0, np.zeros(3)
        lo, hi = 0.0, 1.0
        while f(hi) <= r:
            lo, hi = hi, hi * 2
            if hi > t_max:
                return None
        for _ in range(200):
            mid = 0.5 * (lo + hi)
            lo, hi = (mid, hi) if f(mid) <= r else (lo, mid)
        t = 0.5 * (lo + hi)
    else:
        a, b = 0.0, t_max
        g = (np.sqrt(5) - 1) / 2
        for _ in range(300):                     # the minimum of the convex f on [0, t_max]
            c1, c2 = b - g * (b - a), a + g * (b - a)
            if f(c1) <= f(c2):
                b = c2
            else:
                a = c1
        tmin = 0.5 * (a + b)
        if f(tmin) > r:
            return None
        lo, hi = 0.0, tmin
        for _ in range(200):
            mid = 0.5 * (lo + hi)
            lo, hi = (lo, mid) if f(mid) <= r else (mid, hi)
        t = 0.5 * (lo + hi)
    h = o + d * t
    e = h - point_segment(h, p0, p1)
    le = np.linalg.norm(e)
    return t, (e / le if le > 0 else np.zeros(3))


def project_capsule(x, p0, p1, r, x_axis, solid=True):
    """(projection, inside) of point x onto the capsule: the closest segment point plus r along x - closest (x_axis on the axis)"""
    x = np.asarray(x, float)
    c = point_segment(x, p0, p1)
    e = x - c
    le = np.linalg.norm(e)
    inside = le <= r
    if inside and solid:
        return x, True
    return c + (e / le if le > 0 else np.asarray(x_axis, float)) * r, inside


def mp_point_segment_distance(x, p0, p1, digits: int = 50) -> float:
    """the distance of point x to the segment at `digits` digits (mpmath): bounds the rounding of a ray hit computed in float64"""
    import mpmath
    mpmath.mp.dps = digits
    X, A, B = (mpmath.matrix([mpmath.mpf(float(v)) for v in w]) for w in (x, p0, p1))
    dot = lambda a, b: sum(a[i] * b[i] for i in range(3))
    dd = B - A
    t = min(mpmath.mpf(1), max(mpmath.mpf(0), dot(X - A, dd) / dot(dd, dd))) if dot(dd, dd) > 0 else mpmath.mpf(0)
    e = X - (A + dd * t)
    return float(mpmath.sqrt(dot(e, e)))
