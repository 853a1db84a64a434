"""The contact-manifold generator (csrc/narrow_math.hpp, through the host fixture and the resident row function) against an independent
reference (tests/narrow_reference.py), in f32 and f64 columns.

The contract.  n is the reported normal, a and b the world witnesses (anchor + collider position), pen the reported penetration,
max_dist = max(dt * |v2 - v1|, contact_tolerance).  Every tolerance is scale-relative: TOL_ULPS ulps of the column type times
(|pos_A| + |pos_B| + |he_A| + |he_B| + 1), and f32 results are compared with the reference evaluated from the f32 inputs.
1. |n| = 1, and n points from A to B (dot(n, c_B - c_A) >= 0).
2. a lies on the boundary of A and b on the boundary of B.
3. b - a is parallel to n and pen = dot(a - b, n).  With rule 2 a reported gap is never smaller than the true distance.
4. Overlapping pairs: max(pen) lies within FACE_BIAS + tol of the SAT minimum overlap.  FACE_BIAS = 1e-4 is the header's preference for
   face axes over edge axes; it works both ways: a face axis whose overlap exceeds a shallower edge axis' by less than 1e-4 wins.  For face contacts every reported incident witness is a vertex of the contact region computed by vertex
   enumeration, and the deepest vertex of that region (or one within the header's 1e-6 duplicate radius of it) is reported whenever
   the keep rule keeps it.
5. Separated pairs: if the true distance D <= max_dist - DELTA, at least one point is reported and the smallest reported gap is
   <= D + KAPPA; a pair with D > max_dist + DELTA reports nothing.  DELTA = 1e-6 keeps the draws off the max_dist boundary, which rule
   9 tests exactly.  KAPPA = 1e-4 (the header's FACE_GAP_SLACK) when the reported normal is a face axis: a separated face contact keeps
   its clipped polygon while its nearest point lies within that much of the true distance, else the closest feature pair replaces
   it.  KAPPA = 0 when the normal is an edge-edge axis or the closest pair's direction.  Rules 4 and 5 apply only where the sign of
   the SAT overlap is beyond the tolerance: an f32 quaternion is unit only to an ulp, which moves the header's boxes by about that.
6. Swap symmetry: collide(B, A) gives the same count (up to pruning), -n, the same deepest depth with swapped witnesses, and the same depths when
   nothing was pruned, skipping pairs where two separating axes are within TIE of each other (the header breaks such ties by axis
   order).  prune4 measures distances on shape A's witnesses, so which 4 of more raw points survive depends on the order.
7. Rigid-motion invariance: moving both shapes by one rotation and a translation of 1e3..1e4 keeps the point count and the depths (to
   the tolerance of the moved positions) and rotates the anchors.
8. At most 4 points; the survivors of a clipped polygon keep its cyclic order and include its deepest vertex (rule 4).  This pins the
   header's prune rule, which differs from the reference's prune_points (stated deviation).
9. The keep rule and normal_speed equal the restated rule of narrow_reference.keep, exactly at -pen == eff_margin +- 1 ulp.

The random soups are built feature by feature (vertex on a face, edge across edge, vertex on a corner, parallel faces) at a chosen
signed gap and then classified by the reference; each class's size is asserted so a test cannot pass by drawing nothing.
"""
import sys
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
from avian_b200 import fixture  # noqa: E402
import narrow_reference as ref  # noqa: E402

DT = 1.0 / 60.0
TOL = 0.005                 # contact_tolerance
CLOSING = 18.0              # B closes on A at 18 m/s: eff_margin = max_dist = 0.3
MARGIN = CLOSING * DT
TOL_ULPS = 64
DELTA = 1e-6
KAPPA_FACE = ref.FACE_BIAS
TIE = 1e-6
DUPLICATE = 1e-6            # the header drops a clipped point within this distance of one it already has
N_PER_CLASS = 1500
GROUPS = ("overlapping", "touching", "speculative")
CLASSES = ("face", "edge", "vertex")
MIN_PER_CLASS = 600


def eps_of(scalar):
    return float(np.finfo(scalar).eps)


# ---- soups ---------------------------------------------------------------------------------------------------------------------------
def _random_quat(rng, n):
    q = rng.normal(size=(n, 4))
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def _quat_about(axis_world, angle):
    s = np.sin(angle / 2)[:, None]
    return np.concatenate([axis_world * s, np.cos(angle / 2)[:, None]], axis=1)


def _qmul(a, b):
    ax, ay, az, aw = a.T; bx, by, bz, bw = b.T
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], axis=1)


def _support(R, h, d):
    """Offset from the centre of the box's vertex farthest along d."""
    return R @ (np.where(R.T @ d >= 0, 1.0, -1.0) * h)


def build(kind, gaps, seed):
    """Pairs of one construction at the given signed gaps (negative: overlap).  Returns ca, qa, ha, cb, qb, hb and the construction
    normal (A to B)."""
    rng = np.random.default_rng(seed)
    n = len(gaps)
    ha, hb = rng.uniform(0.2, 0.8, (n, 3)), rng.uniform(0.2, 0.8, (n, 3))
    qa = _random_quat(rng, n)
    qb = _random_quat(rng, n)
    Ra = ref.rotation(qa)
    ca = rng.uniform(-2, 2, (n, 3))
    cb = np.zeros((n, 3)); nn = np.zeros((n, 3))
    for k in range(n):
        R, g = Ra[k], gaps[k]
        if kind in ("vertex_face", "parallel_face"):
            i, s = rng.integers(3), rng.choice((-1.0, 1.0))
            nrm = R[:, i] * s
            u, v = [m for m in range(3) if m != i]
            p = ca[k] + nrm * ha[k, i] + R[:, u] * rng.uniform(-0.7, 0.7) * ha[k, u] + R[:, v] * rng.uniform(-0.7, 0.7) * ha[k, v]
            if kind == "parallel_face":   # B turned about the face normal only: face on face
                qb[k] = _qmul(_quat_about(nrm[None], rng.uniform(0, 2 * np.pi, 1)), qa[k][None])[0]
                Rb = ref.rotation(qb[k])
                cb[k] = p + nrm * (g + abs(Rb.T @ nrm) @ hb[k])   # B's bottom face at height g above the face
            else:
                Rb = ref.rotation(qb[k])
                cb[k] = p + nrm * g - _support(Rb, hb[k], -nrm)
        elif kind == "edge_edge":
            Rb = ref.rotation(qb[k])
            i, j = rng.integers(3), rng.integers(3)
            nrm = np.cross(R[:, i], Rb[:, j]); nrm /= np.linalg.norm(nrm)
            if rng.random() < 0.5:
                nrm = -nrm
            ma = sum(R[:, m] * (np.sign(R[:, m] @ nrm) * ha[k, m]) for m in range(3) if m != i)
            mb = sum(Rb[:, m] * (-np.sign(Rb[:, m] @ nrm) * hb[k, m]) for m in range(3) if m != j)
            pa = ca[k] + ma + R[:, i] * rng.uniform(-0.6, 0.6) * ha[k, i]
            cb[k] = pa + nrm * g - mb - Rb[:, j] * rng.uniform(-0.6, 0.6) * hb[k, j]
        elif kind == "corner":
            sg = rng.choice((-1.0, 1.0), 3)
            nrm = R @ (sg * rng.uniform(0.2, 1.0, 3)); nrm /= np.linalg.norm(nrm)
            Rb = ref.rotation(qb[k])
            cb[k] = ca[k] + R @ (sg * ha[k]) + nrm * g - _support(Rb, hb[k], -nrm)
        nn[k] = nrm
    return ca, qa, ha, cb, qb, hb, nn


def classify(ca, qa, ha, cb, qb, hb):
    """The reference's view of one pair: SAT overlap and axis kind, exact distance, closest-feature label."""
    Ra, Rb = ref.rotation(qa), ref.rotation(qb)
    ov, axis, kind = ref.sat(ca, Ra, ha, cb, Rb, hb)
    out = {"ov": ov, "axis": axis, "sat_kind": kind, "D": 0.0, "label": None}
    if ov <= 0:
        d, x, y, lab, _ = ref.box_box_distance(ca, Ra, ha, cb, Rb, hb)
        out.update(D=d, label=lab, on_a=x, on_b=y)
    return out


_CONSTRUCTION = {
    "overlapping": {"face": "parallel_face", "vertex": "vertex_face", "edge": "edge_edge"},
    "touching": {"face": "vertex_face", "vertex": "corner", "edge": "edge_edge"},
    "speculative": {"face": "vertex_face", "vertex": "corner", "edge": "edge_edge"},
}


def _gaps(group, rng, n):
    if group == "overlapping":
        return -rng.uniform(0.002, 0.06, n)
    if group == "touching":
        return rng.uniform(-1e-6, 1e-6, n)
    return rng.uniform(1e-5, MARGIN - 0.01, n)


def _belongs(group, cls, info):
    if group == "overlapping":
        if info["ov"] <= 1e-5:
            return False
        return info["sat_kind"] == ("edge" if cls == "edge" else "face")
    if group == "touching":
        return abs(info["ov"]) <= 2e-6 and (info["ov"] > 0 or info["label"] == cls)
    return info["ov"] < 0 and info["label"] == cls


_SOUPS = {}


def soup(group, cls, scalar):
    """N_PER_CLASS constructed pairs of one class, kept when the reference agrees with the class.  Cached per (group, class, scalar)."""
    key = (group, cls, np.dtype(scalar).name)
    if key in _SOUPS:
        return _SOUPS[key]
    seed = 1000 * GROUPS.index(group) + 10 * CLASSES.index(cls) + (1 if np.dtype(scalar) == np.float32 else 0)
    rng = np.random.default_rng(seed)
    ca, qa, ha, cb, qb, hb, nn = build(_CONSTRUCTION[group][cls], _gaps(group, rng, N_PER_CLASS), seed + 7)
    # the columns are what the kernel sees: round to the scalar type, then the reference starts from those exact values
    cols = [np.asarray(x, dtype=scalar).astype(np.float64) for x in (ca, qa, ha, cb, qb, hb)]
    ca, qa, ha, cb, qb, hb = cols
    keep, infos = [], []
    for k in range(N_PER_CLASS):
        info = classify(ca[k], qa[k], ha[k], cb[k], qb[k], hb[k])
        if _belongs(group, cls, info):
            keep.append(k); infos.append(info)
    keep = np.array(keep, dtype=np.int64)
    s = {"ca": ca[keep], "qa": qa[keep], "ha": ha[keep], "cb": cb[keep], "qb": qb[keep], "hb": hb[keep], "nn": nn[keep], "info": infos,
         "scalar": np.dtype(scalar)}
    _SOUPS[key] = s
    return s


def columns(s, swap=False):
    """Collider / body columns of a soup: pair k is colliders (k, N + k) and bodies (k, N + k); B closes on A along the construction
    normal at CLOSING."""
    n = len(s["info"])
    A = ("ca", "qa", "ha"); B = ("cb", "qb", "hb")
    if swap:
        A, B = B, A
    sc = s["scalar"]
    cols = {"shape": np.zeros(2 * n, np.uint8), "dims": np.concatenate([s[A[2]], s[B[2]]]).astype(sc),
            "position": np.concatenate([s[A[0]], s[B[0]]]).astype(sc), "rotation": np.concatenate([s[A[1]], s[B[1]]]).astype(sc)}
    lv = np.zeros((2 * n, 3), dtype=sc)
    (lv[:n] if swap else lv[n:])[:] = (-s["nn"] * CLOSING).astype(sc)
    av = np.zeros((2 * n, 3), dtype=sc)
    c1 = np.arange(n, dtype=np.uint32)
    return cols, lv, av, (c1, c1 + n, c1.copy(), c1 + n)


def run_fixture(s, swap=False):
    cols, lv, av, pairs = columns(s, swap)
    return fixture.raw_manifolds(s["scalar"], DT, TOL, pairs, cols, lv, av), cols, lv


# ---- the contract --------------------------------------------------------------------------------------------------------------------
def contract_violations(s, out, cols, lv, group, cls):
    """Every broken rule (1-5, 8, 9) of every pair as readable strings."""
    bad = []
    n = len(s["info"])
    sc = s["scalar"]
    e = eps_of(sc)
    pos = cols["position"].astype(np.float64)
    for k in range(n):
        info = s["info"][k]
        ca, cb = pos[k], pos[n + k]
        Ra, Rb = ref.rotation(s["qa"][k]), ref.rotation(s["qb"][k])
        ha, hb = s["ha"][k], s["hb"][k]
        scale = np.abs(ca).sum() + np.abs(cb).sum() + ha.sum() + hb.sum() + 1.0
        tol = TOL_ULPS * e * scale
        cnt = int(out["point_count"][k])
        rel = lv[n + k].astype(np.float64) - lv[k].astype(np.float64)
        eff = DT * float(np.linalg.norm(rel))
        max_dist = max(eff, TOL)
        nrm = out["normal"][k].astype(np.float64)
        a = out["anchor1"][k, :cnt].astype(np.float64) + ca
        b = out["anchor2"][k, :cnt].astype(np.float64) + cb
        pen = out["penetration"][k, :cnt].astype(np.float64)
        ns = out["normal_speed"][k, :cnt].astype(np.float64)
        tag = f"{group}/{cls}/{sc.name} pair {k}"
        if cnt:
            if abs(np.linalg.norm(nrm) - 1) > tol:
                bad.append(f"{tag}: |n| = {np.linalg.norm(nrm)!r}")
            if nrm @ (cb - ca) < -tol:
                bad.append(f"{tag}: n points from B to A")
            for p in range(cnt):
                if ref.surface_distance(a[p], ca, Ra, ha) > tol or ref.surface_distance(b[p], cb, Rb, hb) > tol:
                    bad.append(f"{tag}: witness {p} off the surface ({ref.surface_distance(a[p], ca, Ra, ha):.3g}, "
                               f"{ref.surface_distance(b[p], cb, Rb, hb):.3g})")
                if np.linalg.norm(np.cross(b[p] - a[p], nrm)) > tol:
                    bad.append(f"{tag}: witness {p}: b - a not parallel to n ({np.linalg.norm(np.cross(b[p] - a[p], nrm)):.3g})")
                if abs(pen[p] - (a[p] - b[p]) @ nrm) > tol:
                    bad.append(f"{tag}: witness {p}: pen {pen[p]!r} != dot(a - b, n) {(a[p] - b[p]) @ nrm!r}")
                want_ns = ref.normal_speed(rel, np.zeros(3), np.zeros(3), a[p] - ca, b[p] - cb, nrm)
                if abs(ns[p] - want_ns) > tol * (1 + np.abs(rel).sum()):
                    bad.append(f"{tag}: witness {p}: normal_speed {ns[p]!r} != {want_ns!r}")
                if not ref.keep(pen[p], ns[p], DT, eff):
                    bad.append(f"{tag}: witness {p} reported although the keep rule drops it")
        if info["ov"] > tol:
            if cnt == 0:
                bad.append(f"{tag}: overlap {info['ov']:.4g} reports nothing")
            elif not abs(pen.max() - info["ov"]) <= ref.FACE_BIAS + tol:
                bad.append(f"{tag}: max pen {pen.max():.6g} farther than 1e-4 from the overlap {info['ov']:.6g}")
            elif cnt > 1:
                bad += _face_region_violations(tag, a, b, nrm, ca, Ra, ha, cb, Rb, hb, max_dist, pen, ns, eff, tol, 1e3 * e)
        elif info["ov"] < -tol:
            D = info["D"]
            if D <= max_dist - DELTA:
                face_normal = cnt and max(np.abs(Ra.T @ nrm).max(), np.abs(Rb.T @ nrm).max()) > 1 - 1e3 * e
                kappa = KAPPA_FACE if face_normal else 0.0
                if cnt == 0:
                    bad.append(f"{tag}: distance {D:.6g} <= max_dist reports nothing")
                elif -pen.max() > D + kappa + tol:
                    bad.append(f"{tag}: smallest gap {-pen.max():.6g} > distance {D:.6g} + {kappa}")
            elif D > max_dist + DELTA and cnt:
                bad.append(f"{tag}: distance {D:.6g} > max_dist reports {cnt} point(s)")
    return bad


def _face_region_violations(tag, a, b, nrm, ca, Ra, ha, cb, Rb, hb, max_dist, pen, ns, eff, tol, parallel):
    """Rule 4 (region vertices, deepest vertex) and rule 8 (cyclic order) for a face contact: the normal is a face axis of A (reference A,
    incident witnesses b) or of B (reference B, incident witnesses a).  Accept either reading when both apply (parallel faces)."""
    readings = []
    for i in range(3):
        if abs(Ra[:, i] @ nrm) > 1 - parallel:
            readings.append((ca, Ra, ha, i, np.sign(Ra[:, i] @ nrm), cb, Rb, hb, b))
        if abs(Rb[:, i] @ nrm) > 1 - parallel:
            readings.append((cb, Rb, hb, i, -np.sign(Rb[:, i] @ nrm), ca, Ra, ha, a))
    if not readings:
        return [f"{tag}: {len(a)} points but the normal is no face axis"]
    errs = []
    for c_r, R_r, h_r, i, sg, c_i, R_i, h_i, inc in readings:
        verts, height = ref.face_region(c_r, R_r, h_r, i, sg, c_i, R_i, h_i)
        if len(verts) == 0:
            errs.append("empty region"); continue
        dmat = np.linalg.norm(inc[:, None, :] - verts[None, :, :], axis=2)
        if dmat.min(axis=1).max() > 100 * tol:
            errs.append(f"point not a region vertex ({dmat.min(axis=1).max():.3g})"); continue
        deep = int(np.argmin(height))
        if -height[deep] >= -max_dist and ref.keep(-height[deep], ns.min(), DT, eff) and dmat[:, deep].min() > 100 * tol:
            # (a region vertex tied with the deepest one within 1e-12 may stand for it)
            # (the header merges clipped points closer than DUPLICATE; a region vertex tied with the deepest within 1e-9 may stand for it)
            ties = np.nonzero(height <= height[deep] + 1e-9)[0]
            if dmat[:, ties].min() > DUPLICATE + 100 * tol:
                errs.append("deepest region vertex missing"); continue
        # cyclic order of the survivors around their centroid (a subset of a convex polygon in its own order)
        if len(inc) >= 3:
            cen = inc.mean(axis=0)
            u = inc[0] - cen; u /= np.linalg.norm(u) or 1.0
            w = np.cross(nrm, u)
            ang = np.unwrap(np.arctan2((inc - cen) @ w, (inc - cen) @ u))
            steps = np.diff(np.concatenate([ang, ang[:1] + 2 * np.pi * np.sign(ang[-1] - ang[0] or 1)]))
            if not (np.all(steps > -1e-9) or np.all(steps < 1e-9)):
                errs.append("survivors out of cyclic order"); continue
        return []
    return [f"{tag}: face contact: " + "; ".join(errs)]


# ---- tests: soups --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scalar", [np.float64, np.float32])
@pytest.mark.parametrize("group", GROUPS)
@pytest.mark.parametrize("cls", CLASSES)
def test_soup_meets_the_contract(scalar, group, cls):
    s = soup(group, cls, scalar)
    assert len(s["info"]) >= MIN_PER_CLASS, f"{group}/{cls}: only {len(s['info'])} pairs of the class were drawn"
    out, cols, lv = run_fixture(s)
    bad = contract_violations(s, out, cols, lv, group, cls)
    assert not bad, f"{len(bad)} violations, e.g.\n" + "\n".join(bad[:12])


@pytest.mark.parametrize("scalar", [np.float64, np.float32])
def test_resident_row_function_meets_the_contract(scalar):
    """The row function of the device-resident contact store (csrc/contact_rows.hpp through avh_rows_narrow) on the speculative and
    overlapping soups: the same contract as the ordinary narrow phase."""
    for group in ("overlapping", "speculative"):
        for cls in CLASSES:
            s = soup(group, cls, scalar)
            cols, lv, av, (c1, c2, b1, b2) = columns(s)
            out = rows_narrow(scalar, cols, lv, av, c1, c2)
            bad = contract_violations(s, out, cols, lv, group, cls)
            assert not bad, f"{len(bad)} violations, e.g.\n" + "\n".join(bad[:12])


def rows_narrow(scalar, cols, lv, av, c1, c2):
    sc = np.dtype(scalar)
    E = int(c1.shape[0])
    z = lambda shape, dt=sc: np.zeros((E,) + shape, dtype=dt)
    r = {"c1": c1.astype(np.uint32), "c2": c2.astype(np.uint32), "b1": c1.astype(np.uint32), "b2": c2.astype(np.uint32),
         "live": np.ones(E, np.uint8), "count": z((), np.uint8), "disjoint": z((), np.uint8), "normal": z((3,)), "anchor1": z((4, 3)),
         "anchor2": z((4, 3)), "penetration": z((4,)), "normal_speed": z((4,)), "prev_count": z((), np.uint8), "prev_a1": z((4, 3), np.float64),
         "prev_a2": z((4, 3), np.float64), "ws_n_in": z((4,)), "ws_t_in": z((4, 2)), "ws_n_out": z((4,)), "ws_t_out": z((4, 2))}
    n_col = cols["position"].shape[0]
    big = np.full((n_col, 3), 1e6, dtype=sc)        # AABBs that always overlap: the geometry alone decides
    p = lambda x: x.ctypes.data
    fixture._load().avh_rows_narrow(
        32 if sc == np.float32 else 64, E, *(p(r[k]) for k in ("c1", "c2", "b1", "b2", "live", "count", "disjoint", "normal", "anchor1", "anchor2",
                                                                "penetration", "normal_speed", "prev_count", "prev_a1", "prev_a2", "ws_n_in",
                                                                "ws_t_in", "ws_n_out", "ws_t_out")),
        p(cols["shape"]), p(cols["dims"]), p(cols["position"]), p(cols["rotation"]), p(np.ascontiguousarray(lv)), p(np.ascontiguousarray(av)),
        p(-big), p(big), DT, TOL, 1.0, 1)
    return {"point_count": r["count"], "normal": r["normal"], "anchor1": r["anchor1"], "anchor2": r["anchor2"], "penetration": r["penetration"],
            "normal_speed": r["normal_speed"]}


@pytest.mark.parametrize("group", ("overlapping", "speculative"))
def test_float64_reference_agrees_with_mpmath(group):
    """The vectorised float64 reference against the same definitions at 50 digits on a sample of every class."""
    for cls in CLASSES:
        s = soup(group, cls, np.float64)
        for k in range(0, len(s["info"]), max(1, len(s["info"]) // 8)):
            args = (s["ca"][k], s["qa"][k], s["ha"][k], s["cb"][k], s["qb"][k], s["hb"][k])
            if group == "overlapping":
                assert abs(float(ref.mp_sat(*args)) - s["info"][k]["ov"]) < 1e-13
            else:
                assert abs(float(ref.mp_box_box_distance(*args)) - s["info"][k]["D"]) < 1e-13


def _sat_tie(s, k):
    """Whether two axes (edge axes biased by FACE_BIAS as the header does) come within TIE of the best one."""
    Ra, Rb = ref.rotation(s["qa"][k]), ref.rotation(s["qb"][k])
    ov = ref.sat_overlaps(s["ca"][k], Ra, s["ha"][k], s["cb"][k], Rb, s["hb"][k])
    biased = np.sort(np.concatenate([ov[:6], ov[6:] + ref.FACE_BIAS]))
    return biased[1] - biased[0] < TIE or s["info"][k]["ov"] <= 0


@pytest.mark.parametrize("scalar", [np.float64, np.float32])
def test_swap_symmetry(scalar):
    checked = 0
    for group in ("overlapping", "speculative"):
        for cls in CLASSES:
            s = soup(group, cls, scalar)
            o1, _, _ = run_fixture(s)
            o2, cols, _ = run_fixture(s, swap=True)
            e = eps_of(scalar)
            for k in range(len(s["info"])):
                if group == "overlapping" and _sat_tie(s, k):
                    continue
                n1, n2 = int(o1["point_count"][k]), int(o2["point_count"][k])
                scale = np.abs(s["ca"][k]).sum() + np.abs(s["cb"][k]).sum() + s["ha"][k].sum() + s["hb"][k].sum() + 1
                tol = TOL_ULPS * e * scale
                assert n1 == n2 or min(n1, n2) >= 3, f"{group}/{cls} pair {k}: {n1} vs {n2} points"
                if n1 == 0:
                    continue
                # a closest-pair normal is a difference of witnesses over the distance: its rounding grows as 1 / D
                ntol = tol * max(1.0, 1.0 / max(s["info"][k]["D"], 1e-6))
                assert np.abs(o1["normal"][k] + o2["normal"][k]).max() <= ntol, f"{group}/{cls} pair {k}: normal"
                d1, d2 = o1["penetration"][k, :n1], o2["penetration"][k, :n2]
                assert abs(d1.max() - d2.max()) <= tol, f"{group}/{cls} pair {k}: depths {d1} vs {d2}"
                if n1 == n2 < 3:   # (prune4 measures on the first shape's witnesses: with more raw points the order matters)
                    assert np.abs(np.sort(d1) - np.sort(d2)).max() <= tol, f"{group}/{cls} pair {k}: depths {d1} vs {d2}"
                i1, i2 = int(np.argmax(d1)), int(np.argmax(d2))
                assert np.abs(o1["anchor1"][k, i1].astype(np.float64) - o2["anchor2"][k, i2]).max() <= 1e3 * tol, f"{group}/{cls} pair {k}: witnesses"
                assert np.abs(o1["anchor2"][k, i1].astype(np.float64) - o2["anchor1"][k, i2]).max() <= 1e3 * tol, f"{group}/{cls} pair {k}: witnesses"
                checked += 1
    assert checked > 3000


def _near_decision(s, k, o1, o2, width):
    """Whether the reference puts pair k within `width` of a decision the header makes: two SAT axes (edge axes biased by FACE_BIAS)
    tied, the distance at max_dist, or a reported point at the edge of the speculative margin."""
    Ra, Rb = ref.rotation(s["qa"][k]), ref.rotation(s["qb"][k])
    ov = ref.sat_overlaps(s["ca"][k], Ra, s["ha"][k], s["cb"][k], Rb, s["hb"][k])
    biased = np.sort(-np.concatenate([ov[:6], ov[6:] - ref.FACE_BIAS]))[::-1]
    if biased[0] - biased[1] < width or abs(s["info"][k]["D"] - MARGIN) < width:
        return True
    gaps = np.concatenate([-o["penetration"][k, :int(o["point_count"][k])].astype(np.float64) for o in (o1, o2)])
    return bool(np.any(np.abs(gaps - MARGIN) < width))


def _moved(s, q, T, scalar):
    """The soup with both shapes of every pair rotated by q about the origin and then translated by T, rounded to the column type."""
    n = len(s["info"])
    Q = ref.rotation(q)
    out = dict(s)
    for c in ("ca", "cb"):
        out[c] = np.asarray(s[c] @ Q.T + T, dtype=scalar).astype(np.float64)
    for c in ("qa", "qb"):
        out[c] = np.asarray(_qmul(np.repeat(q[None], n, 0), s[c]), dtype=scalar).astype(np.float64)
    out["nn"] = s["nn"] @ Q.T
    return out


@pytest.mark.parametrize("scalar,shift", [(np.float64, 1e4), (np.float32, 1e3), (np.float32, 1e4)])
def test_rigid_motion_invariance(scalar, shift):
    """Rule 7 in two steps, each keeping the point count of every pair.
    - Rotation about the origin: rounding the rotated poses to the column type moves the geometry by a few ulps, so the count is
      compared except where the reference finds a decision within 1e3 ulps of the pair's scale (_near_decision); the deepest depth
      and, when it is unique, the deepest point's anchors (rotated) agree to the tolerance.  Which of more than 4 clipped points
      survive prune4 can flip on a near-tie of its distance comparisons, so the other depths are not compared.
    - Translation by `shift` (1e3..1e4) of poses that lie on the grid of the column's ulp at 4 * shift, so that the moved columns
      are exact: the header works in a frame centred on shape A, so every output column must be the same bit for bit."""
    rng = np.random.default_rng(11)
    e = eps_of(scalar)
    rotated = translated = skipped = 0
    for group in ("overlapping", "speculative"):
        for cls in CLASSES:
            s = soup(group, cls, scalar)
            n = len(s["info"])
            q = _random_quat(rng, 1)[0]
            Q = ref.rotation(q)
            o0, _, _ = run_fixture(s)
            r = _moved(s, q, np.zeros(3), scalar)
            o1, _, _ = run_fixture(r)
            for k in range(n):
                scale = np.abs(s["ca"][k]).sum() + np.abs(s["cb"][k]).sum() + s["ha"][k].sum() + s["hb"][k].sum() + 1
                tol = TOL_ULPS * e * scale
                n0, n1 = int(o0["point_count"][k]), int(o1["point_count"][k])
                if n0 != n1 and _near_decision(s, k, o0, o1, 1e3 * e * scale):
                    skipped += 1
                    continue
                assert n0 == n1, f"rotated {group}/{cls} pair {k}: {n0} vs {n1} points"
                if n0 == 0:
                    continue
                p0, p1 = o0["penetration"][k, :n0], o1["penetration"][k, :n1]
                assert abs(p0.max() - p1.max()) <= tol, f"rotated {group}/{cls} pair {k}: deepest {p0.max()} vs {p1.max()}"
                i0, i1 = int(np.argmax(p0)), int(np.argmax(p1))
                if p0.max() - np.delete(p0, i0).max(initial=-np.inf) > tol:      # a unique deepest point
                    for a in ("anchor1", "anchor2"):
                        want = o0[a][k, i0].astype(np.float64) @ Q.T
                        assert np.abs(want - o1[a][k, i1]).max() <= 10 * tol, f"rotated {group}/{cls} pair {k}: {a}"
                rotated += 1
            # the translation step, from the rotated poses snapped to the grid on which adding T is exact
            grid = float(np.spacing(scalar(4 * shift)))
            T = np.round(rng.uniform(-1, 1, 3) * shift / grid) * grid
            g = dict(r)
            for c in ("ca", "cb"):
                g[c] = np.round(r[c] / grid) * grid
            t = dict(g)
            for c in ("ca", "cb"):
                t[c] = g[c] + T
                assert np.array_equal(np.asarray(t[c], dtype=scalar).astype(np.float64), t[c])
            og, _, _ = run_fixture(g)
            ot, _, _ = run_fixture(t)
            for key in og:
                assert np.array_equal(og[key], ot[key]), f"translated {group}/{cls}: {key} differs"
            translated += int((og["point_count"] > 0).sum())
    assert rotated > 3000 and translated > 3000 and skipped < rotated // 100


# ---- hand-worked cases ---------------------------------------------------------------------------------------------------------------
def qrat(x, y, z, w):
    """A rational quaternion and its exact rotation matrix (Fractions): columns = local axes."""
    x, y, z, w = (Fraction(v) for v in (x, y, z, w))
    n2 = x * x + y * y + z * z + w * w
    m = [[1 - 2 * (y * y + z * z) / n2, 2 * (x * y - z * w) / n2, 2 * (x * z + y * w) / n2],
         [2 * (x * y + z * w) / n2, 1 - 2 * (x * x + z * z) / n2, 2 * (y * z - x * w) / n2],
         [2 * (x * z - y * w) / n2, 2 * (y * z + x * w) / n2, 1 - 2 * (x * x + y * y) / n2]]
    nq = float(n2) ** 0.5
    return np.array([float(x) / nq, float(y) / nq, float(z) / nq, float(w) / nq]), m


def pair(scalar, shapes, dims, pos, rot, vel_b=(0, 0, 0), tol=TOL, dt=DT):
    cols = {"shape": np.array(shapes, np.uint8), "dims": np.array(dims, dtype=scalar), "position": np.array(pos, dtype=scalar),
            "rotation": np.array(rot, dtype=scalar)}
    lv = np.zeros((2, 3), dtype=scalar); lv[1] = vel_b
    z = np.zeros(1, np.uint32); o = np.ones(1, np.uint32)
    out = fixture.raw_manifolds(scalar, dt, tol, (z, o, z.copy(), o.copy()), cols, lv, np.zeros((2, 3), dtype=scalar))
    cnt = int(out["point_count"][0])
    p = cols["position"].astype(np.float64)
    return {"n": cnt, "normal": out["normal"][0].astype(np.float64), "a": out["anchor1"][0, :cnt].astype(np.float64) + p[0],
            "b": out["anchor2"][0, :cnt].astype(np.float64) + p[1], "pen": out["penetration"][0, :cnt].astype(np.float64),
            "ns": out["normal_speed"][0, :cnt].astype(np.float64)}


I = (0.0, 0.0, 0.0, 1.0)
BOX, SPH = fixture.SHAPE_CUBOID, fixture.SHAPE_SPHERE
SCALARS = [np.float64, np.float32]


def close(x, y, scalar, scale=4.0):
    return np.allclose(x, y, rtol=0, atol=TOL_ULPS * eps_of(scalar) * scale)


@pytest.mark.parametrize("scalar", SCALARS)
def test_box_resting_flat(scalar):
    r = pair(scalar, [BOX, BOX], [(2, 0.5, 2), (0.5, 0.5, 0.5)], [(0, 0, 0), (0.25, 0.99, -0.5)], [I, I])
    assert r["n"] == 4 and close(r["normal"], (0, 1, 0), scalar) and close(r["pen"], 0.01, scalar)
    want = {(0.25 + sx, 0.49, -0.5 + sz) for sx in (-0.5, 0.5) for sz in (-0.5, 0.5)}
    assert close(np.array(sorted(map(tuple, r["b"]))), np.array(sorted(want)), scalar)


@pytest.mark.parametrize("scalar", SCALARS)
def test_turned_box_gives_an_octagon_pruned_to_four(scalar):
    q, m = qrat(0, 1, 0, 2)                    # 2 atan(1/2) = 53.13 degrees about y: cos 3/5, sin 4/5
    R = np.array(m, dtype=float)
    r = pair(scalar, [BOX, BOX], [(0.55, 0.5, 0.55), (0.5, 0.5, 0.5)], [(0, 0, 0), (0, 0.98, 0)], [I, q])
    verts, height = ref.face_region(np.zeros(3), np.eye(3), np.array([0.55, 0.5, 0.55]), 1, 1.0, np.array([0, 0.98, 0]), R, np.full(3, 0.5))
    assert len(verts) == 8 and np.allclose(height, -0.02)
    assert r["n"] == 4 and close(r["pen"], 0.02, scalar)
    assert all(np.linalg.norm(verts - b, axis=1).min() < 1e-5 for b in r["b"])


@pytest.mark.parametrize("scalar", SCALARS)
def test_box_on_an_edge_and_on_a_vertex(scalar):
    q, m = qrat(0, 0, 1, 2)                    # about z: the lowest feature is an edge along z
    R = np.array(m, dtype=float)
    low = abs(R[1]) @ np.full(3, 0.5)          # half height of the turned box
    r = pair(scalar, [BOX, BOX], [(2, 0.5, 2), (0.5, 0.5, 0.5)], [(0, 0, 0), (0, 0.5 + low - 0.01, 0)], [I, q])
    assert r["n"] == 2 and close(r["pen"], 0.01, scalar, 8) and close(r["normal"], (0, 1, 0), scalar)
    assert close(np.sort(r["b"][:, 2]), [-0.5, 0.5], scalar, 8)
    q, m = qrat(1, 0, 1, 2)                    # a unique lowest vertex
    R = np.array(m, dtype=float)
    low = abs(R[1]) @ np.full(3, 0.5)
    r = pair(scalar, [BOX, BOX], [(2, 0.5, 2), (0.5, 0.5, 0.5)], [(0, 0, 0), (0, 0.5 + low - 0.01, 0)], [I, q])
    assert r["n"] == 1 and close(r["pen"], 0.01, scalar, 8)
    assert close(r["b"][0], _support(R, np.full(3, 0.5), np.array([0, -1.0, 0])) + (0, 0.5 + low - 0.01, 0), scalar, 8)


def _crossed_boxes(qb_rat):
    """A turned 2 atan(1/2) about x (its top is an edge along x), B turned back about x (its bottom is an edge along x) and then
    about y by the rational quaternion qb_rat.  Returns the quaternions and the heights of A's top edge and of B's bottom edge
    below its centre."""
    qa, _ = qrat(1, 0, 0, 2)
    qy, _ = qrat(*qb_rat)
    qb = _qmul(qy[None], np.array([[-qa[0], 0, 0, qa[3]]]))[0]
    h = np.full(3, 0.5)
    ta = _support(ref.rotation(qa), h, np.array([0, 1.0, 0]))[1]
    tb = -_support(ref.rotation(qb), h, np.array([0, -1.0, 0]))[1]
    return qa, qb, h, ta, tb


def _reference_gap(scalar, qa, qb, h, cb):
    """-overlap or distance of the pair from the exact column values."""
    qa, qb, cb = (np.asarray(x, dtype=scalar).astype(np.float64) for x in (qa, qb, cb))
    Ra, Rb = ref.rotation(qa), ref.rotation(qb)
    ov = ref.sat(np.zeros(3), Ra, h, cb, Rb, h)[0]
    return -ov if ov > 0 else ref.box_box_distance(np.zeros(3), Ra, h, cb, Rb, h)[0]


@pytest.mark.parametrize("scalar", SCALARS)
@pytest.mark.parametrize("qb_rat", [(0, 1, 0, 1), (0, 1, 0, 20)], ids=["90deg", "shallow"])
@pytest.mark.parametrize("gap", [-0.01, 0.05])
def test_crossed_edges(scalar, qb_rat, gap):
    """The edges cross at 90 deg or at the shallow 2 atan(1/20) = 5.7 deg: one point, normal +y, the reference's gap, b - a along n."""
    qa, qb, h, ta, tb = _crossed_boxes(qb_rat)
    cb = np.array([0.0, ta + tb + gap, 0.0])
    assert abs(_reference_gap(np.float64, qa, qb, h, cb) - gap) < 1e-9          # the construction
    d = _reference_gap(scalar, qa, qb, h, cb)
    r = pair(scalar, [BOX, BOX], [h, h], [(0, 0, 0), cb], [qa, qb], vel_b=(0, -CLOSING, 0))
    assert r["n"] == 1 and close(r["normal"], (0, 1, 0), scalar, 8)
    assert close(-r["pen"][0], d, scalar, 8), f"gap {-r['pen'][0]!r}, reference {d!r}"
    assert np.linalg.norm(np.cross(r["b"][0] - r["a"][0], r["normal"])) <= TOL_ULPS * eps_of(scalar) * 8


@pytest.mark.parametrize("scalar", SCALARS)
@pytest.mark.parametrize("qb_rat,past", [((0, 1, 0, 20), 0.1), ((0, 1, 0, 20), 0.2), ((0, 1, 0, -3), 0.1)],
                         ids=["shallow-0.1", "shallow-0.2", "steep-0.1"])
def test_edge_passing_the_end_of_the_other_edge(scalar, qb_rat, past):
    """B's bottom edge crosses the line of A's top edge `past` beyond its end, 0.05 above it and closing: the edge axis separates
    by 0.05 but the closest points lie at the end of A's edge, so the true distance is larger.  The reported gap must be that
    distance (clamping the two edges' parameters independently reported 0.05 here), with b - a along the normal."""
    qa, qb, h, ta, tb = _crossed_boxes(qb_rat)
    cb = np.array([0.5 + past, ta + tb + 0.05, 0.0])
    D = _reference_gap(scalar, qa, qb, h, cb)
    assert D > 0.05 + 1e-3 and D < MARGIN
    r = pair(scalar, [BOX, BOX], [h, h], [(0, 0, 0), cb], [qa, qb], vel_b=(0, -CLOSING, 0))
    tol = TOL_ULPS * eps_of(scalar) * 8
    assert r["n"] >= 1
    assert abs(-r["pen"].max() - D) <= tol, f"gap {-r['pen'].max()!r}, distance {D!r}"
    for p in range(r["n"]):
        assert np.linalg.norm(np.cross(r["b"][p] - r["a"][p], r["normal"])) <= tol


@pytest.mark.parametrize("scalar", SCALARS)
@pytest.mark.parametrize("past", [0.02, 0.08, 0.15])
def test_corner_hanging_past_the_table_edge(scalar, past):
    """A box tilted so its lowest corner hangs `past` beyond the table's edge, just above the table top and closing: the closest
    features are that corner and the table's edge, within the speculative margin, so they must be reported at the true distance."""
    q, m = qrat(1, 0, 1, 3)
    R = np.array(m, dtype=float)
    hb = np.array([0.4, 0.3, 0.5])
    corner = _support(R, hb, np.array([0, -1.0, 0]))
    cb = np.array([1.0 + past, 0.5 + 0.03, 0.2]) - corner
    r = pair(scalar, [BOX, BOX], [(1.0, 0.5, 1.0), hb], [(0, 0, 0), cb], [I, q], vel_b=(0, -CLOSING, 0))
    D = ref.box_box_distance(np.zeros(3), np.eye(3), np.array([1.0, 0.5, 1.0]), cb, R, hb)[0]
    assert D < MARGIN and r["n"] >= 1, f"true distance {D} within the margin, {r['n']} points"
    assert abs(-r["pen"].max() - D) < 1e-4 + 1e-6
    assert np.linalg.norm(np.cross(r["b"][0] - r["a"][0], r["normal"])) < 1e-5


@pytest.mark.parametrize("scalar", SCALARS)
def test_sphere_sphere(scalar):
    r = pair(scalar, [SPH, SPH], [(0.5, 0, 0), (0.25, 0, 0)], [(1, 2, 3), (1, 2, 3)], [I, I])
    assert r["n"] == 1 and close(r["pen"], 0.75, scalar, 8) and close(np.linalg.norm(r["normal"]), 1, scalar)
    # a gap of exactly the contact tolerance is in range (max_dist is inclusive), one ulp more is not.  B closes at 0.1 with
    # dt = 1/16: eff_margin = 0.00625 < tol, so max_dist = tol, and the keep rule's second clause (ns dt - pen < eff_margin) keeps
    # the point, so the range test alone decides
    tol, dt, v = 0.0078125, 0.0625, -0.1
    for xb, want in ((scalar(1.0 + tol), 1), (np.nextafter(scalar(1.0 + tol), scalar(2)), 0)):
        gap = float(xb) - 1.0
        ns = float(scalar(v))
        eff = dt * abs(ns)
        assert eff < tol and ref.keep(-gap, ns, dt, eff)
        r = pair(scalar, [SPH, SPH], [(0.5, 0, 0), (0.5, 0, 0)], [(0, 0, 0), (xb, 0, 0)], [I, I], vel_b=(v, 0, 0), tol=tol, dt=dt)
        assert r["n"] == want, f"gap {gap!r}: {r['n']} points"
        if want:
            assert r["pen"][0] == -gap and r["ns"][0] == ns


@pytest.mark.parametrize("scalar", SCALARS)
@pytest.mark.parametrize("where", ["face", "edge", "corner", "inside", "surface"])
def test_sphere_box(scalar, where):
    q, m = qrat(0, 1, 0, 2)
    R = np.array(m, dtype=float)
    h = np.array([0.5, 0.4, 0.3])
    c = np.array([1.0, -2.0, 0.5])
    local = {"face": (0.1, 0.55, -0.1), "edge": (0.6, 0.45, 0.0), "corner": (0.55, 0.45, 0.35), "inside": (0.1, 0.3, 0.05),
             "surface": (0.1, 0.4, 0.05)}[where]
    cs = np.asarray(c + R @ np.array(local), dtype=scalar).astype(np.float64)
    rs = 0.2
    nw, gap, on = ref.sphere_box(c, ref.rotation(np.asarray(q, dtype=scalar).astype(np.float64)), h, cs, rs)
    r = pair(scalar, [BOX, SPH], [h, (rs, 0, 0)], [c, cs], [q, I])
    assert r["n"] == 1
    assert close(r["normal"], nw, scalar, 16) and close(-r["pen"][0], gap, scalar, 16) and close(r["a"][0], on, scalar, 16)
    # the other order: the normal flips, the witnesses swap
    r2 = pair(scalar, [SPH, BOX], [(rs, 0, 0), h], [cs, c], [I, q])
    assert close(r2["normal"], -nw, scalar, 16) and close(r2["pen"], r["pen"], scalar, 16) and close(r2["b"][0], on, scalar, 16)


@pytest.mark.parametrize("scalar", SCALARS)
@pytest.mark.parametrize("away", [True, False])
def test_keep_rule_at_the_boundary(scalar, away):
    """-pen == eff_margin +- 1 ulp on exactly representable sphere pairs: the kept set equals the restated rule, and normal_speed is
    the relative speed along the normal.  Moving apart the first clause decides (gap < eff_margin); closing, the second one
    (ns dt - pen < eff_margin) with a contact tolerance that keeps the pair in range."""
    dt = 0.0625
    v = 1.0 if away else -1.0
    eff = dt * abs(v)
    edge = eff if away else eff - dt * v        # the gap at which the deciding clause turns
    tol = 0.001 if away else 1.0
    seen = set()
    x = scalar(1.0 + edge)
    for xb in (np.nextafter(x, scalar(0)), x, np.nextafter(x, scalar(2))):     # one ulp of the position column either side
        gap = float(xb) - 1.0
        r = pair(scalar, [SPH, SPH], [(0.5, 0, 0), (0.5, 0, 0)], [(0, 0, 0), (xb, 0, 0)], [I, I], vel_b=(v, 0, 0), tol=tol, dt=dt)
        in_range = gap <= max(eff, tol)
        want = 1 if in_range and ref.keep(-gap, v, dt, eff) else 0
        assert r["n"] == want, f"gap {gap!r}: {r['n']} points, the rule says {want}"
        if want:
            assert r["pen"][0] == -gap and r["ns"][0] == v
        seen.add(want)
    assert seen == {0, 1}


@pytest.mark.parametrize("swap", [False, True])
def test_match_point_at_the_threshold(swap):
    """match_point (through avh_match_raw) against the restated match_contacts with new anchors at the threshold +- 1 ulp, in both
    body orders."""
    lib = fixture._load()
    thr = 0.1
    for step in (np.nextafter(thr, 0), thr, np.nextafter(thr, 1), np.nextafter(np.nextafter(thr, 0), 0)):
        old1 = np.array([[0.3, 0.1, -0.2], [1.0, 1.0, 1.0]]); old2 = np.array([[-0.4, 0.2, 0.0], [2.0, 2.0, 2.0]])
        n1, n2 = old1[0] + (step, 0, 0), old2[0] + (0, 0, step)
        if swap:
            n1, n2 = old2[0] + (step, 0, 0), old1[0] + (0, 0, step)
        want = ref.match_contacts(n1, n2, old1, old2, thr)
        prev_count = np.array([2], np.uint8)
        prev_a1 = np.zeros((1, 4, 3)); prev_a2 = np.zeros((1, 4, 3))
        prev_a1[0, :2], prev_a2[0, :2] = old1, old2
        ws_n = np.zeros((1, 4)); ws_n[0, :2] = (7.0, 9.0)
        ws_t = np.zeros((1, 4, 2))
        new_a1 = np.zeros((1, 4, 3)); new_a2 = np.zeros((1, 4, 3))
        new_a1[0, 0], new_a2[0, 0] = n1, n2
        p = lambda x: x.ctypes.data
        lib.avh_match_raw(64, 1, p(np.zeros(1, np.uint32)), p(np.ones(1, np.uint8)), p(new_a1), p(new_a2), 1.0, 1, p(prev_count), p(prev_a1),
                          p(prev_a2), p(ws_n), p(ws_t))
        assert ws_n[0, 0] == ({0: 7.0, 1: 9.0}.get(want, 0.0)), f"step {step!r}: rule says {want}"
