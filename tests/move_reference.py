"""MoveAndSlide::move_and_slide (character_controller/move_and_slide.rs:464-609) restated in Python, independently of csrc/move_math.hpp.

The control flow — depenetration, the sweep loop, pull-back, plane collection and pruning, Gauss-Seidel, the cone projection
(velocity_project.rs:122-324) — is written here from the reference; only the two geometric primitives come from the host fixture: a single
closest shape cast (fixture.query_cast_shape) and a single pair contact (fixture.move_contact).  Candidates for the intersections are the
colliders whose tight AABB meets the character's grown one, computed here with numpy.  f64 columns; the f32 parts of the reference (Dir: the
sweep direction, plane normals, the similarity dot product) are numpy float32.
"""
from __future__ import annotations

import math

import numpy as np

from avian_b200 import api, fixture

DOT_EPSILON = 0.005
MIN_DISTANCE = 1e-4


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _cross(a, b):
    return np.array([a[1] * b[2] - b[1] * a[2], a[2] * b[0] - b[2] * a[0], a[0] * b[1] - b[0] * a[1]])


def _f32dot(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.float32(np.float32(a[0] * b[0]) + np.float32(a[1] * b[1])) + np.float32(a[2] * b[2])


def project_velocity(v, normals) -> np.ndarray:
    """velocity_project.rs:122-324 in f64; normals are f32 Dirs."""
    x0 = -np.asarray(v, dtype=np.float64)
    ns = [np.asarray(n, dtype=np.float32).astype(np.float64) for n in normals]
    kind, n1, n2, sv, iters = 0, None, None, x0.copy(), 0
    while True:
        if _dot(sv, sv) < DOT_EPSILON * DOT_EPSILON or not ns:
            break
        dots = [_dot(n, sv) for n in ns]
        bi = max(i for i in range(len(ns)) if dots[i] == max(dots))     # max_by: the last of equal maxima
        if dots[bi] <= DOT_EPSILON:
            break
        nd = ns[bi]
        if kind == 0:
            sv, n1, kind = x0 - _dot(nd, x0) * nd, nd, 1
        elif kind == 1:
            c = _cross(nd, n1)
            d = _dot(x0, c)
            sv = d * c / _dot(c, c)
            n1, n2 = (nd, n1) if d > 0 else (n1, nd)
            kind = 2
        else:
            c1, c2 = _cross(n1, nd), _cross(nd, n2)
            d1, d2 = _dot(x0, c1), _dot(x0, c2)
            if d1 <= 0 and d2 <= 0:
                sv = np.zeros(3)
                break
            if d1 * abs(d1) * _dot(c2, c2) > d2 * abs(d2) * _dot(c1, c1):
                sv, n2 = d1 * c1 / _dot(c1, c1), nd
            else:
                sv, n1 = d2 * c2 / _dot(c2, c2), nd
        iters += 1
        if iters >= 10:
            break
    return -sv


def project_velocity_bruteforce(v, normals) -> np.ndarray:
    """velocity_project.rs:15-110"""
    v = np.asarray(v, dtype=np.float64)
    ns = [np.asarray(n, dtype=np.float32).astype(np.float64) for n in normals]
    if not ns or all(_dot(n, v) >= -DOT_EPSILON for n in ns):
        return v
    valid = lambda p: all(_dot(p, n) >= -DOT_EPSILON for n in ns)
    best, best_d = np.zeros(3), math.inf
    for n in ns:
        nv = _dot(n, v)
        if nv < -DOT_EPSILON:
            p = v - nv * n
            d = _dot(v - p, v - p)
            if d < best_d and valid(p):
                best, best_d = p, d
    for i in range(len(ns)):
        for j in range(i + 1, len(ns)):
            e = _cross(ns[i], ns[j])
            el = _dot(e, e)
            if el < DOT_EPSILON:
                continue
            p = e * (_dot(v, e) / el)
            d = _dot(v - p, v - p)
            if d < best_d and valid(p):
                best, best_d = p, d
    return np.zeros(3) if math.isinf(best_d) else best


def _aabb(shape, he, p, q):
    q = np.asarray(q, dtype=np.float64)
    if shape == fixture.SHAPE_SPHERE:
        e = np.full(3, he[0])
    else:
        x, y, z, w = q
        s = _dot(q[:3], q[:3]) + w * w
        r = np.array([[w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
                      [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
                      [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z]]) / s
        e = np.abs(r) @ np.asarray(he, dtype=np.float64)
    return np.asarray(p) - e, np.asarray(p) + e


class Scene:
    """The colliders (f64) and a character's filter."""

    def __init__(self, colliders: "api.QueryColliders", ignored=None):
        self.cols = colliders
        self.n = len(colliders.shape)
        self.boxes = [_aabb(colliders.shape[c], colliders.dims[c], colliders.position[c], colliders.rotation[c]) for c in range(self.n)]
        self.memb = np.ones(self.n, np.uint32) if colliders.memberships is None else np.asarray(colliders.memberships, np.uint32)
        self.ignored = np.zeros(self.n, bool) if ignored is None else np.asarray(ignored).astype(bool)

    def blocked(self, mask, exclude):
        return {c for c in range(self.n) if (int(self.memb[c]) & int(mask)) == 0 or c in exclude or self.ignored[c]}


def move_one(scene: Scene, cfg: "api.MoveConfig", shape, dims, pos, rot, vel, mask=0xFFFFFFFF, exclude=(), planes=()):
    """One character: (position, velocity, [(iteration, collider, safe distance, toi)])."""
    lu = cfg.length_unit
    skin = lu * cfg.skin_width
    skip = scene.blocked(mask, set(exclude))
    pos, vel = np.asarray(pos, np.float64).copy(), np.asarray(vel, np.float64).copy()
    init = [np.asarray(p, np.float32) / np.sqrt(_f32dot(p, p)) for p in planes]

    def intersections(at, pred):
        lo, hi = _aabb(shape, dims, at, rot)
        lo, hi = lo - pred, hi + pred
        out = []
        for c in range(scene.n):
            blo, bhi = scene.boxes[c]
            if c in skip or np.any(lo > bhi) or np.any(hi < blo):
                continue
            k = fixture.move_contact(np.float64, shape, dims, at, rot, scene.cols.shape[c], scene.cols.dims[c], scene.cols.position[c],
                                     scene.cols.rotation[c], pred)
            if k is not None:
                out.append(k)
        return out

    def depenetrate(at):
        fix = np.zeros(3)
        if cfg.depenetration_iterations == 0:
            return fix
        lst = [(n.astype(np.float64), pen + skin) for n, pen in intersections(at, skin)]
        for _ in range(cfg.depenetration_iterations):
            total = 0.0
            for n, dist in lst:
                if dist > lu * cfg.penetration_rejection_threshold:
                    continue
                err = max(dist - _dot(fix, n), 0.0)
                total += err
                fix = fix + err * n
            if total < lu * cfg.max_depenetration_error:
                break
        return fix

    hits = []
    time_left = cfg.delta_time
    pos = pos + depenetrate(pos)
    for it in range(cfg.move_and_slide_iterations):
        sweep = time_left * vel
        sf = sweep.astype(np.float32)
        lf = np.sqrt(_f32dot(sf, sf))
        if not (np.isfinite(lf) and lf > 0):
            break
        d = sf / lf
        distance = float(lf)
        if distance < MIN_DISTANCE:
            break
        q = api.ShapeQueries(shape=np.array([shape], np.uint8), dims=np.array([dims]), position=np.array([pos]), rotation=np.array([rot]),
                             direction=d.astype(np.float64)[None], max_distance=np.array([distance]),
                             flags=np.array([api.CAST_IGNORE_ORIGIN_PENETRATION], np.uint32), exclude=[sorted(skip)])
        h = fixture.query_cast_shape(np.float64, scene.cols, q)
        if h["collider"][0] < 0:
            pos = pos + sweep
            break
        n1 = h["normal1"][0]
        toi = float(h["distance"][0])
        pd = _dot(d.astype(np.float64), -n1)
        safe = max(toi - skin / max(pd, DOT_EPSILON), 0.0)
        hits.append((it, int(h["collider"][0]), safe, toi))
        time_left -= time_left * (safe / distance)
        pos = pos + d.astype(np.float64) * safe
        pl = list(init) + [n1.astype(np.float32)]
        for n, _ in intersections(pos, skin * 2):
            for k, e in enumerate(pl):
                if float(_f32dot(n, e)) >= cfg.plane_similarity_dot_threshold:
                    if _dot(n.astype(np.float64), vel) < _dot(e.astype(np.float64), vel):
                        pl[k] = n
                    break
            else:
                if len(pl) < cfg.max_planes:
                    pl.append(n)
        vel = project_velocity(vel, pl)
    pos = pos + depenetrate(pos)
    return pos, vel, hits
