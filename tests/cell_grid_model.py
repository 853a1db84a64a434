"""A restatement of the broad phase's (y, z) cell grid (csrc/broadphase_cells.cuh) in the column scalar, for tests.

It follows the device code expression by expression, in numpy scalars of the column dtype (f32 or f64), with no fused operations (the
library is built with -fmad=false and IEEE division):
  * yz_stats / yz_fold: per axis the min and max of the min corners, and the "large" threshold S(4) * S(sum / n), the sum of the extents
    taken in double (the device sums in a different order; the scenes that rely on this model keep their thresholds far from any extent);
  * yz_small_max / yz_grid: the cell edge is the largest extent <= the threshold (0 if none), the cell size max(edge, range / 1024), the
    cell count int(range / cell) + 1 clamped to [1, 1024], the finer axis halved until ny * nz <= 0xFFFF, and inv = S(1) / cell;
  * cell_coord: t = (v - v0) * inv, cell = t > 0 ? (t < n ? int(t) : n - 1) : 0;
  * cell_keys: an interval is large when its extent on either axis exceeds that axis' edge, else it is binned by its min corner;
  * sweep_bounds / sweep_cells_kernel: the x-window (i, end_i), the query range [cell(min_i - edge), cell(max_i)] per axis, the direct
    window test when the range has more cells than the window has candidates, and the brute-force "wide" path (more than 4 096
    candidates and more than 32 query cells).

Two rules: "nearest" rounds the extents and the query's lower bound to nearest, which can drop touching pairs near the origin;
"directed" (the kernels' rule) rounds the extents up and the lower bound down (__fsub_ru / __fsub_rd, __dsub_ru / __dsub_rd), which
makes the index exact:
    lo = rd(min_i - edge) <= min_i - edge <= max_j - ext_j = min_j   for every small j that overlaps i.
The directed roundings are computed exactly: the round-to-nearest difference plus its exact error term (Knuth's two-sum), then one ulp
with np.nextafter where the error says the nearest result lies on the wrong side.  `sub_directed_exact` is the same with Fraction.
"""
from __future__ import annotations

from dataclasses import dataclass
from fractions import Fraction

import numpy as np

CG_MAX_AXIS = 1024
CG_MAX_CELLS = 0xFFFF
SW_WIDE = 4096            # csrc/broadphase.cu: more x-candidates than this ...
SW_WIDE_CELLS = 32        # ... and more query cells than this: swept brute force
SW_WIDE_CAP = 1 << 14     # at most this many wide intervals; the rest stay in the cell sweep

RULES = ("nearest", "directed")


def sub_directed(a, b, up: bool):
    """a - b rounded up (up=True) or down, elementwise, in the dtype of a and b"""
    a, b = np.asarray(a), np.asarray(b)
    d = a - b
    # two-sum of (a, -b): d + r == a - b exactly
    bb = d - a
    r = (a - (d - bb)) + (-b - bb)
    if up:
        return np.where(r > 0, np.nextafter(d, d.dtype.type(np.inf)), d)
    return np.where(r < 0, np.nextafter(d, d.dtype.type(-np.inf)), d)


def sub_directed_exact(a, b, up: bool):
    """the same for two scalars, from the exact rational difference"""
    S = type(a)
    d = S(a - b)
    exact = Fraction(float(a)) - Fraction(float(b))
    if up and Fraction(float(d)) < exact:
        d = np.nextafter(d, S(np.inf))
    if not up and Fraction(float(d)) > exact:
        d = np.nextafter(d, S(-np.inf))
    return d


def extents(lo, hi, rule: str):
    """the extents that decide small / large and the edge"""
    return hi - lo if rule == "nearest" else sub_directed(hi, lo, up=True)


def query_lower(v, edge, rule: str):
    """the lower bound of the cell query"""
    return v - edge if rule == "nearest" else sub_directed(v, np.full_like(v, edge), up=False)


@dataclass
class Axis:
    v0: np.floating       # min of the min corners (the grid origin)
    cell: np.floating     # cell size
    inv: np.floating      # S(1) / cell, 0 for an empty grid
    n: int                # cells after coarsening
    n_before: int         # cells before coarsening
    edge: np.floating     # largest small extent
    thr: np.floating      # the "large" threshold, 4 x mean extent
    range: np.floating    # max - min of the min corners

    def coord(self, v):
        """cell_coord"""
        S = type(self.v0)
        t = (np.asarray(v, dtype=S) - self.v0) * self.inv
        return np.where(t > 0, np.where(t < S(self.n), np.trunc(np.minimum(t, S(self.n))), self.n - 1), 0).astype(np.int64)


def _axis(lo, hi, rule: str):
    S = lo.dtype.type
    n = lo.shape[0]
    thr = S(4) * S(np.float64((hi - lo).astype(np.float64).sum()) / n)      # yz_fold: the mean of round-to-nearest extents
    ext = extents(lo, hi, rule)
    small = ext <= thr
    edge = max(S(0), ext[small].max()) if small.any() else S(0)             # yz_small_max
    v0 = lo.min()
    rng = S(lo.max() - v0)
    c = max(edge, S(rng / S(CG_MAX_AXIS)))
    k = int(S(rng / c)) + 1 if c > S(0) else 1
    k = max(1, min(k, CG_MAX_AXIS))
    return Axis(v0=v0, cell=c, inv=S(0), n=k, n_before=k, edge=edge, thr=thr, range=rng)


def grid(yz_min, yz_max, rule: str = "nearest") -> tuple[Axis, Axis]:
    """yz_grid for [n, 2] (y, z) min / max columns"""
    assert rule in RULES
    ay, az = _axis(yz_min[:, 0], yz_max[:, 0], rule), _axis(yz_min[:, 1], yz_max[:, 1], rule)
    S = type(ay.v0)
    while ay.n * az.n > CG_MAX_CELLS:          # coarsen the finer axis
        if ay.n >= az.n:
            ay.n, ay.cell = (ay.n + 1) // 2, ay.cell * S(2)
        else:
            az.n, az.cell = (az.n + 1) // 2, az.cell * S(2)
    for a in (ay, az):
        a.inv = S(1) / a.cell if a.cell > S(0) else S(0)
    return ay, az


class CellGridModel:
    """The cell sweep of one broad-phase run over AABB columns in input order ([n, 3] min / max in the column scalar; no halo flags).
    Per x-sorted rank: the bin of every interval, and for every interval i its window end, query range, cell count and path."""

    def __init__(self, aabb_min, aabb_max, rule: str = "nearest"):
        mn, mx = np.asarray(aabb_min), np.asarray(aabb_max)
        assert mn.dtype == mx.dtype and mn.dtype in (np.float32, np.float64)
        self.rule = rule
        self.order = np.argsort(mn[:, 0] + mn.dtype.type(0), kind="stable")    # -0.0 == +0.0, stable
        self.rank = np.empty_like(self.order)
        self.rank[self.order] = np.arange(self.order.shape[0])
        smn, smx = mn[self.order], mx[self.order]
        n = smn.shape[0]
        self.n = n
        self.y, self.z = grid(smn[:, 1:], smx[:, 1:], rule)
        self.ext_y, self.ext_z = extents(smn[:, 1], smx[:, 1], rule), extents(smn[:, 2], smx[:, 2], rule)
        self.large = (self.ext_y > self.y.edge) | (self.ext_z > self.z.edge)                    # cell_keys
        self.key_y, self.key_z = self.y.coord(smn[:, 1]), self.z.coord(smn[:, 2])
        ranks = np.arange(n)
        self.end = np.maximum(np.searchsorted(smn[:, 0], smx[:, 0], side="right"), ranks + 1)
        self.cy_lo, self.cy_hi = self.y.coord(query_lower(smn[:, 1], self.y.edge, rule)), self.y.coord(smx[:, 1])
        self.cz_lo, self.cz_hi = self.z.coord(query_lower(smn[:, 2], self.z.edge, rule)), self.z.coord(smx[:, 2])
        self.ncell = (self.cy_hi - self.cy_lo + 1) * (self.cz_hi - self.cz_lo + 1)
        self.candidates = self.end - ranks - 1
        self.wide = (self.candidates > SW_WIDE) & (self.ncell > SW_WIDE_CELLS)              # before the cap
        self.direct = ~self.wide & (self.ncell > self.candidates)

    @property
    def before(self) -> tuple[int, int]:
        return self.y.n_before, self.z.n_before

    def path(self, i: int) -> str:
        """how the sweep handles rank i: 'empty' window, 'wide' (brute force), 'direct' window test or the 'cells'"""
        if self.candidates[i] <= 0:
            return "empty"
        return "wide" if self.wide[i] else "direct" if self.direct[i] else "cells"

    def visits(self, i, j):
        """whether the sweep of rank i tests rank j (i < j < end_i), elementwise.  A wide-eligible i counts as brute force only while the
        wide list is within its cap (beyond it the device picks which ones stay in the cell sweep)."""
        i, j = np.asarray(i), np.asarray(j)
        inside = (j > i) & (j < self.end[i])
        brute = (self.wide[i] & (self.wide.sum() <= SW_WIDE_CAP)) | self.direct[i]
        cells = (self.cy_lo[i] <= self.key_y[j]) & (self.key_y[j] <= self.cy_hi[i]) & (self.cz_lo[i] <= self.key_z[j]) & (self.key_z[j] <= self.cz_hi[i])
        return inside & (brute | self.large[j] | cells)

    def visits_rows(self, row_a, row_b):
        """visits() for a pair given as input rows, in x-sorted order"""
        ra, rb = self.rank[np.asarray(row_a)], self.rank[np.asarray(row_b)]
        return self.visits(np.minimum(ra, rb), np.maximum(ra, rb))
