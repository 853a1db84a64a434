"""Adversarial scenes for the broad phase's (y, z) cell grid, and their check on the CPU.

The cell sweep (csrc/broadphase_cells.cuh) finds the j that overlap interval i through the cells [cell(min_i - edge), cell(max_i)], where
the edge is the largest "small" extent.  With round-to-nearest arithmetic that range is not conservative: when j = [a, b] sits near the
origin, its extent E = fl(b - a) can be smaller than b - a, and for an i whose min touches b, fl(b - E) lies a fraction of an ulp above
a.  A cell boundary in that gap puts j one cell below i's query, and the touching pair, which the reference's inclusive compares accept,
is never tested.

`planted_pair` searches (seeded) for such a j and a grid origin; `minimal_scene` and `filler_scene` build scenes around it that keep E
the cell edge, the origin the smallest min, the cell size E and i on the cell path.  The test below asserts, for every generated scene,
that the reference lists the planted pairs, that the round-to-nearest model of the grid misses them and that the directed-rounding
model visits every reference pair, so the GPU cases in test_gpu_broadphase_cells.py stay adversarial if the generator changes.
"""
from __future__ import annotations

from dataclasses import dataclass
from fractions import Fraction

import numpy as np
import pytest

import cell_grid_model as cgm
import sap_reference as ref

SEEDS = range(16)
N_FILL = 5000


@dataclass
class Plan:
    """j = [a, b] on one axis with E = fl(b - a) < b - a; i starts at b; the grid origin v0 makes cell(fl(b - E)) > cell(a)"""
    a: np.floating
    b: np.floating
    E: np.floating
    v0: np.floating


def _cell(v, v0, inv):
    S = type(v)
    return int(S(S(v - v0) * inv))


def planted_pair(rng, S) -> Plan:
    while True:
        a = S(rng.uniform(-1.0, 2.0))
        b = S(a + S(rng.uniform(0.5, 3.0)))
        E = S(b - a)
        if not Fraction(float(E)) < Fraction(float(b)) - Fraction(float(a)):
            continue                          # the extent must round down
        lo = S(b - E)
        if not lo > a:
            continue
        inv = S(1) / E
        for k in rng.integers(2, 150, size=8):
            v0 = S(a - S(S(int(k)) * E))      # a cell boundary near a ...
            for toward in (S(np.inf), S(-np.inf)):
                v = v0
                for _ in range(16):           # ... walked by ulps until it falls in (a, fl(b - E)]
                    if v < a and _cell(lo, v, inv) > _cell(a, v, inv):
                        return Plan(a, b, E, v)
                    v = np.nextafter(v, toward)


def plans(S, seed):
    rng = np.random.default_rng([seed, np.dtype(S).itemsize])
    return planted_pair(rng, S), planted_pair(rng, S)


@dataclass
class Scene:
    mn: np.ndarray            # [n, 3] in the column scalar, input order
    mx: np.ndarray
    planted: list             # (axis, row of i, row of j, plan) per planted pair
    i_large: bool


def minimal_scene(S, plan: Plan, axis: int, i_large: bool) -> Scene:
    """i (row 0) touches j (row 1) from above on `axis` (1 = y, 2 = z); six fillers sit at the grid origin, far below, so i's x-window
    holds 7 candidates and the cell path runs.  The other axis has one cell (every min 0).  i_large: i's extent on the other axis is 10
    against 1 for the rest, above 4x the mean (8.5), so i is binned in the large list while its query still goes through the cells."""
    a, b, E, v0 = plan.a, plan.b, plan.E, plan.v0
    other = 3 - axis
    mn = np.zeros((8, 3), S)
    mx = np.ones((8, 3), S)
    mn[0, axis], mx[0, axis] = b, S(b + S(0.5) * E)
    mn[1, axis], mx[1, axis] = a, b
    if i_large:
        mx[0, other] = S(10)
    h = np.linspace(0.5, 0.99, 6)
    mn[2:, 0], mx[2:, 0] = S(0.5), S(1.5)
    mn[2:, axis] = v0
    mx[2:, axis] = (v0 + (h * E).astype(S)).astype(S)
    return Scene(mn, mx, [(axis, 0, 1, plan)], i_large)


def filler_scene(S, py: Plan, pz: Plan, i_large: bool, seed: int) -> Scene:
    """the y pair (rows 0, 1) and the z pair (rows 2, 3) among N_FILL fillers whose extents lie in [E/2, 0.99 E] over [v0, v0 + 200 E]
    on each axis (the first filler sits at the origin of both).  The planted pairs span 10 in x over fillers 4 long on [0, 25], so i's
    window holds ~2 000 candidates and each filler's ~800.  Each planted i sits well inside the other axis' range; i_large makes its
    extent there 6 E, above the threshold of about 3 E."""
    rng = np.random.default_rng([seed, 7, np.dtype(S).itemsize])
    n = 4 + N_FILL
    mn, mx = np.empty((n, 3), S), np.empty((n, 3), S)
    x = rng.uniform(0, 25, N_FILL)
    mn[4:, 0], mx[4:, 0] = x.astype(S), (x + 4).astype(S)
    for ax, p in ((1, py), (2, pz)):
        lo = (p.v0 + (rng.uniform(0, 200, N_FILL) * p.E).astype(S)).astype(S)
        lo[0] = p.v0
        mn[4:, ax] = np.maximum(lo, p.v0)
        mx[4:, ax] = (mn[4:, ax] + (rng.uniform(0.5, 0.99, N_FILL) * p.E).astype(S)).astype(S)
    for (ax, p, x0, ri) in ((1, py, 5, 0), (2, pz, 15, 2)):
        other, q = 3 - ax, (pz if ax == 1 else py)
        mn[ri:ri + 2, 0], mx[ri:ri + 2, 0] = S(x0), S(x0 + 10)
        mn[ri, ax], mx[ri, ax] = p.b, S(p.b + S(0.5) * p.E)
        mn[ri + 1, ax], mx[ri + 1, ax] = p.a, p.b
        c = S(q.v0 + S(50) * q.E)
        mn[ri:ri + 2, other] = c
        mx[ri:ri + 2, other] = S(c + S(0.5) * q.E)
        if i_large:
            mx[ri, other] = S(c + S(6) * q.E)
    return Scene(mn, mx, [(1, 0, 1, py), (2, 2, 3, pz)], i_large)


def scenes(S, kind: str, axis: int | None = None, i_large: bool = False):
    """the seeded scenes of one variant: kind 'minimal' (one pair on `axis`) or 'fillers' (one pair on each axis)"""
    out = []
    for seed in SEEDS:
        py, pz = plans(S, seed)
        if kind == "minimal":
            out.append(minimal_scene(S, py if axis == 1 else pz, axis, i_large))
        else:
            out.append(filler_scene(S, py, pz, i_large, seed))
    return out


def reference(sc: Scene) -> ref.SapResult:
    n = sc.mn.shape[0]
    return ref.sweep_and_prune(np.arange(n, dtype=np.uint32), np.arange(n, dtype=np.uint32), sc.mn, sc.mx)


def check_scene(sc: Scene) -> ref.SapResult:
    """the assertions every generated scene must satisfy (see the module docstring); returns the reference result"""
    r = reference(sc)
    listed = set(zip(r.collider1.tolist(), r.collider2.tolist()))
    near = cgm.CellGridModel(sc.mn, sc.mx, "nearest")
    fixed = cgm.CellGridModel(sc.mn, sc.mx, "directed")
    S = sc.mn.dtype.type
    for ax, ri, rj, p in sc.planted:
        assert (ri, rj) in listed, f"the reference does not list the planted pair ({ri}, {rj})"
        assert near.rank[ri] < near.rank[rj]
        assert not near.visits_rows(ri, rj), f"the round-to-nearest grid finds the planted pair ({ri}, {rj})"
        assert fixed.visits_rows(ri, rj)
        for m, edge in ((near, p.E), (fixed, np.nextafter(p.E, S(np.inf)))):
            g = m.y if ax == 1 else m.z
            assert g.v0 == p.v0 and g.cell == edge and g.edge == edge, (g, p)
            assert g.n == g.n_before and g.n > 2
            i = m.rank[ri]
            assert m.path(i) == "cells", m.path(i)
            assert bool(m.large[i]) == sc.i_large and not m.large[m.rank[rj]]
    # the directed rule visits every pair the reference lists
    ranks = np.sort(np.stack([fixed.rank[r.collider1], fixed.rank[r.collider2]]), axis=0)
    assert fixed.visits(ranks[0], ranks[1]).all()
    return r


VARIANTS = [(S, ax, large) for S in (np.float32, np.float64) for ax in (1, 2) for large in (False, True)]


def variant_id(v):
    S, ax, large = v
    return f"{np.dtype(S).name}-{'yz'[ax - 1]}-{'i_large' if large else 'i_small'}"


@pytest.mark.parametrize("variant", VARIANTS, ids=variant_id)
def test_minimal_scenes_are_adversarial(variant):
    S, ax, large = variant
    n = 0
    for sc in scenes(S, "minimal", ax, large):
        check_scene(sc)
        n += 1
    print(f"{variant_id(variant)}: {n} planted pairs, each missed by the round-to-nearest grid")
    assert n == len(SEEDS)


@pytest.mark.parametrize("variant", [(S, large) for S in (np.float32, np.float64) for large in (False, True)],
                         ids=lambda v: f"{np.dtype(v[0]).name}-{'i_large' if v[1] else 'i_small'}")
def test_filler_scenes_are_adversarial(variant):
    S, large = variant
    n = 0
    for sc in scenes(S, "fillers", i_large=large):
        r = check_scene(sc)
        assert r.count > 100
        n += len(sc.planted)
    print(f"{np.dtype(S).name} {'i_large' if large else 'i_small'} in {N_FILL} fillers: {n} planted pairs, each missed by the round-to-nearest grid")


@pytest.mark.parametrize("S", [np.float32, np.float64])
def test_directed_subtraction_is_exact(S):
    """the model's vectorised directed rounding against the rational one, on the planted values and on random operands"""
    rng = np.random.default_rng(3)
    a = np.concatenate([rng.uniform(-4, 4, 2000), rng.uniform(-1e-3, 1e-3, 200), [0.0, -0.0, 1.0, 2.0 ** -30]]).astype(S)
    b = np.concatenate([rng.uniform(-4, 4, 2000), rng.uniform(-1e3, 1e3, 200), [-0.0, 0.0, 1.0, 3.0]]).astype(S)
    for seed in SEEDS:
        for p in plans(S, seed):
            a, b = np.append(a, [p.b, p.b]), np.append(b, [p.a, p.E])
    for up in (True, False):
        got = cgm.sub_directed(a, b, up)
        want = np.array([cgm.sub_directed_exact(x, y, up) for x, y in zip(a, b)], dtype=S)
        assert np.array_equal(got, want)
        exact = [Fraction(float(x)) - Fraction(float(y)) for x, y in zip(a, b)]
        assert all((Fraction(float(g)) >= e) if up else (Fraction(float(g)) <= e) for g, e in zip(got, exact))


def test_model_on_a_hand_found_scene():
    """a hand-found f32 scene: y0 = -32.26491, cell 2.7494977, ny = 14; j in y cell 11, i's query from cell 12"""
    f = np.float32
    a, b, y0 = f(0.72905916), f(3.4785569), f(-32.26491)
    mn = np.array([[0, b, 0], [0, a, 0]] + [[0.5, y0, 0]] * 6, f)
    mx = np.array([[1, f(b + f(1)), 1], [1, b, 1]] + [[1.5, f(y0 + f(1)), 1]] * 6, f)
    near, fixed = cgm.CellGridModel(mn, mx, "nearest"), cgm.CellGridModel(mn, mx, "directed")
    assert near.y.n == 14 and near.y.cell == f(2.7494977) and near.y.v0 == y0
    assert near.key_y[near.rank[1]] == 11 and near.cy_lo[near.rank[0]] == 12
    assert not near.visits_rows(0, 1) and fixed.visits_rows(0, 1)
    assert fixed.cy_lo[fixed.rank[0]] == 11
    r = ref.sweep_and_prune(np.arange(8), np.arange(8), mn, mx)
    assert r.count == 16 and (0, 1) in set(zip(r.collider1.tolist(), r.collider2.tolist()))


@pytest.mark.parametrize("rule", cgm.RULES)
def test_at_scale_scenes_reach_their_grid_paths(rule):
    """the shapes test_gpu_at_scale.py relies on, from the same model: more wide intervals than the cap, and a grid of more than 0xFFFF
    cells before coarsening"""
    from test_gpu_at_scale import coarsening_columns, over_cap_columns
    m = cgm.CellGridModel(*over_cap_columns(), rule)
    assert m.wide.sum() > cgm.SW_WIDE_CAP, m.wide.sum()
    m = cgm.CellGridModel(*coarsening_columns(), rule)
    ny, nz = m.before
    assert ny * nz > cgm.CG_MAX_CELLS and m.y.n * m.z.n <= cgm.CG_MAX_CELLS, (m.before, m.y.n, m.z.n)
