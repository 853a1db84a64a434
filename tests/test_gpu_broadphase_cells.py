"""The broad phase's (y, z) cell grid at its edges, bit for bit against tests/sap_reference.py (and the oracle on small scenes).

  * Touching pairs planted next to a cell boundary near the origin (test_broadphase_cells_cpu.py builds them and checks on the CPU that
    a round-to-nearest query range misses each one): f32 and f64, on y and on z, with i small and with i in the large list, alone in
    8-interval scenes and among 5 000 fillers.
  * A table of grid shapes, each asserting through tests/cell_grid_model.py that it is the shape it names: an axis of zero extents, one
    cell on an axis, cells wider than the edge, a coarsened grid, x-windows that end on / start after a large interval, the direct-test
    switch at ncell == window and window + 1, and signed-zero mins.  Each runs in the default f32 context and in an f64 one.
"""
import numpy as np
import pytest

from avian_b200 import api

import cell_grid_model as cgm
import oracle_lib
import test_broadphase_cells_cpu as gen
from test_gpu_at_scale import assert_matches, reference

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def f64_ctx():
    with api.Context(device=0, scalar=np.float64) as ctx:
        yield ctx


@pytest.fixture
def ctx_of(gpu_ctx, f64_ctx):
    return lambda S: gpu_ctx if np.dtype(S) == np.float32 else f64_ctx


def columns(mn, mx) -> api.Aabbs:
    n = mn.shape[0]
    return api.Aabbs(collider=np.arange(n, dtype=np.uint32), body=np.arange(n, dtype=np.uint32), aabb_min=mn.copy(), aabb_max=mx.copy(),
                     flags=np.full(n, api.AABB_GENERATE_CONSTRAINTS, np.uint8), order_out=np.zeros(n, np.uint32))


def compare(ctx, mn, mx, what, oracle=True):
    """the device against the reference (and the oracle); returns the reference result"""
    a = columns(mn, mx)
    r = reference(a)
    g = ctx.broadphase(a)
    want = set(zip(r.collider1.tolist(), r.collider2.tolist()))
    got = set(zip(g.collider1.tolist(), g.collider2.tolist()))
    try:
        assert_matches(g, r, a, what)
    except AssertionError as e:
        raise AssertionError(f"{e}; missing pairs {sorted(want - got)[:8]}, extra pairs {sorted(got - want)[:8]}") from None
    if oracle:
        ao = columns(mn, mx)
        o = oracle_lib.broadphase(ao)
        assert o.count == r.count and np.array_equal(o.collider1, r.collider1) and np.array_equal(o.collider2, r.collider2), what + "oracle"
        assert np.array_equal(o.flags, r.flags) and np.array_equal(ao.order_out, r.order), what + "oracle"
    return r


# ---- planted touching pairs ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", gen.VARIANTS, ids=gen.variant_id)
def test_planted_touching_pairs(ctx_of, variant):
    S, ax, large = variant
    failures = []
    for seed, sc in zip(gen.SEEDS, gen.scenes(S, "minimal", ax, large)):
        try:
            compare(ctx_of(S), sc.mn, sc.mx, f"seed {seed}: ")
        except AssertionError as e:
            failures.append(str(e))
    assert not failures, f"{len(failures)} of {len(gen.SEEDS)} scenes differ:\n" + "\n".join(failures)


@pytest.mark.parametrize("variant", [(S, large) for S in (np.float32, np.float64) for large in (False, True)],
                         ids=lambda v: f"{np.dtype(v[0]).name}-{'i_large' if v[1] else 'i_small'}")
def test_planted_pairs_among_fillers(ctx_of, variant):
    S, large = variant
    failures = []
    for seed, sc in zip(gen.SEEDS, gen.scenes(S, "fillers", i_large=large)):
        try:
            compare(ctx_of(S), sc.mn, sc.mx, f"seed {seed}: ", oracle=False)
        except AssertionError as e:
            failures.append(str(e))
    assert not failures, f"{len(failures)} of {len(gen.SEEDS)} scenes differ:\n" + "\n".join(failures)


# ---- grid shapes ---------------------------------------------------------------------------------------------------------------------
# Each builder returns (min, max) in float64 (cast to the column scalar by the test) and a check of the model built in that scalar.

def _q(v, step=0.25):
    return np.round(np.asarray(v) / step) * step


def zero_extent_axis(rng):
    """every y extent 0: edge_y = 0, cells of range / 1024 (1 024 cells); equal y values are the only y overlaps"""
    n = 2000
    mn = np.column_stack([rng.uniform(0, 10, n), _q(rng.uniform(0, 50, n), 0.5), rng.uniform(0, 20, n)])
    mx = mn + np.column_stack([np.ones(n), np.zeros(n), rng.uniform(0.2, 0.6, n)])

    def check(m):
        assert m.y.edge == 0 and m.y.cell == type(m.y.v0)(m.y.range / type(m.y.v0)(1024)) and m.y.n == 1024, m.y
    return mn, mx, check


def one_cell_axis(rng):
    """every min.y equal: one cell on y, whatever the extents"""
    n = 2000
    mn = np.column_stack([rng.uniform(0, 10, n), np.full(n, 1.25), rng.uniform(0, 20, n)])
    mx = mn + np.column_stack([np.ones(n), _q(rng.uniform(0.25, 3, n)), _q(rng.uniform(0.25, 1, n))])

    def check(m):
        assert m.y.n == 1 and m.y.range == 0 and m.y.edge > 0 and m.z.n > 10, (m.y, m.z)
    return mn, mx, check


def far_outlier(rng):
    """one interval 5 000 away on y: cells of range / 1024, ten times the edge, so a small j overlaps i from the same or the next cell"""
    n = 2000
    mn = np.column_stack([rng.uniform(0, 10, n), _q(rng.uniform(0, 20, n)), _q(rng.uniform(0, 20, n))])
    mx = mn + np.column_stack([np.ones(n), _q(rng.uniform(0.25, 0.5, n)), _q(rng.uniform(0.25, 0.5, n))])
    mn[7, 1], mx[7, 1] = 5000.0, 5000.5

    def check(m):
        assert m.y.cell > 8 * m.y.edge and m.y.cell == type(m.y.v0)(m.y.range / type(m.y.v0)(1024)) and m.y.n == 1024, m.y
    return mn, mx, check


def coarsened(rng):
    """4 000 intervals in clusters over 1 000 x 1 000 in (y, z) on a 1/4 grid (many touching faces): 1 024 x 1 024 cells before
    coarsening, fewer than 0xFFFF after"""
    n, k = 4000, 400
    centre = _q(rng.uniform(0, 1000, (k, 2)))
    c = centre[rng.integers(0, k, n)] + _q(rng.uniform(-1, 1, (n, 2)))
    mn = np.column_stack([rng.uniform(0, 20, n), c])
    mx = mn + np.column_stack([np.ones(n), _q(rng.uniform(0.25, 0.75, (n, 2)))])
    mn[0, 1:], mx[0, 1:] = [0, 0], [0.5, 0.5]
    mn[1, 1:], mx[1, 1:] = [1000, 1000], [1000.5, 1000.5]

    def check(m):
        assert m.before[0] * m.before[1] > cgm.CG_MAX_CELLS and m.y.n * m.z.n <= cgm.CG_MAX_CELLS, (m.before, m.y.n, m.z.n)
        assert m.y.cell > 2 * m.y.edge
    return mn, mx, check


def large_list_bounds(rng):
    """min.x = rank, every window ends exactly on an interval (max.x = min.x + 3..8); ranks 8 and 9 of every ten are large on y (extent
    100 against 1, 20 % of the intervals: above 4x the mean).  Every min.y is 0 (one y cell) and z mins are 0..3 with extent 1, so small
    and large intervals alike take the cell path; windows end on a large interval followed by a large one, large i see the large
    interval right after them, and z faces touch."""
    n = 400
    r = np.arange(n)
    large = r % 10 >= 8
    mn = np.column_stack([r.astype(float), np.zeros(n), rng.integers(0, 4, n).astype(float)])
    mx = mn + np.column_stack([rng.integers(3, 9, n).astype(float), np.where(large, 100.0, 1.0), np.ones(n)])

    def check(m):
        i = np.arange(m.n)
        cells = np.array([m.path(k) == "cells" for k in i])
        e = m.end
        assert np.array_equal(m.large, large[m.order])
        ends_on_large = cells & (e < m.n) & m.large[np.minimum(e, m.n - 1)] & m.large[e - 1]
        starts_after_large = cells & m.large & (i + 1 < m.n) & m.large[np.minimum(i + 1, m.n - 1)]
        assert ends_on_large.sum() >= 10 and starts_after_large.sum() >= 10 and (cells & ~m.large).sum() > 200
    return mn, mx, check


def direct_switch(rng):
    """max.x set so that the window has exactly ncell candidates (cell path) for even ranks and ncell - 1 (direct window test) for odd"""
    n = 600
    mn = np.column_stack([0.5 * np.arange(n), _q(rng.uniform(0, 10, n)), _q(rng.uniform(0, 10, n))])
    mx = mn + np.column_stack([np.zeros(n), _q(rng.uniform(0.25, 1, n)), _q(rng.uniform(0.25, 1, n))])
    mx[0, 1:] = mn[0, 1:] + 1.0
    # the query cells do not depend on x: take them from the model of the y / z columns (exact on this 1/4 grid under either rule)
    m = cgm.CellGridModel(mn, mx, "nearest")
    assert np.array_equal(m.ncell, cgm.CellGridModel(mn, mx, "directed").ncell)
    w = m.ncell - (np.arange(n) % 2)
    mx[:, 0] = mn[np.minimum(np.arange(n) + w, n - 1), 0]

    def check(m):
        i = np.arange(m.n)
        full = i + m.ncell < m.n
        at = full & (m.candidates == m.ncell)
        above = full & (m.candidates == m.ncell - 1)
        assert all(m.path(k) == "cells" for k in np.nonzero(at)[0]) and all(m.path(k) == "direct" for k in np.nonzero(above & (m.candidates > 0))[0])
        assert at.sum() > 200 and (above & (m.candidates > 0)).sum() > 200 and m.ncell.min() >= 2
    return mn, mx, check


def signed_zeros(rng):
    """mins of -0.0 and +0.0 on y (the y origin is a zero) and z, z maxes of -0.0 and +0.0, and min.x of both zeros"""
    n = 1500
    y = rng.choice([-0.0, 0.0, 0.25, 0.5], n)
    z = rng.choice([-1.0, -0.5, -0.0, 0.0, 0.5], n)
    x = np.where(rng.random(n) < 0.3, rng.choice([-0.0, 0.0], n), _q(rng.uniform(-2, 2, n)))
    mn = np.column_stack([x, y, z])
    mx = mn + np.column_stack([np.ones(n), rng.choice([0.25, 0.5], n), rng.choice([0.5, 1.0], n)])
    zero = mx[:, 2] == 0
    mx[zero, 2] = np.where(rng.random(int(zero.sum())) < 0.5, -0.0, 0.0)

    def check(m):
        assert m.y.v0 == 0 and m.z.v0 == -1
    return mn, mx, check


SHAPES = [zero_extent_axis, one_cell_axis, far_outlier, coarsened, large_list_bounds, direct_switch, signed_zeros]


@pytest.mark.parametrize("S", [np.float32, np.float64], ids=["float32", "float64"])
@pytest.mark.parametrize("shape", SHAPES, ids=[f.__name__ for f in SHAPES])
def test_grid_shapes(ctx_of, shape, S):
    mn, mx, check = shape(np.random.default_rng(SHAPES.index(shape)))
    mn, mx = mn.astype(S), mx.astype(S)
    for rule in cgm.RULES:
        check(cgm.CellGridModel(mn, mx, rule))
    r = compare(ctx_of(S), mn, mx, f"{shape.__name__}: ")
    assert r.count > 50
    if shape is signed_zeros:
        assert np.signbit(mn[:, 1:]).any(axis=0).all() and np.signbit(mx[:, 2]).any()
    fixed = cgm.CellGridModel(mn, mx, "directed")
    ranks = np.sort(np.stack([fixed.rank[r.collider1], fixed.rank[r.collider2]]), axis=0)
    assert fixed.visits(ranks[0], ranks[1]).all()
