"""The size-dependent paths of the shared device machinery, checked against plain references at the sizes where they switch on.

The stable radix pass of csrc/device_prims.cuh derives its (digit, block) offsets inside the scatter blocks up to RS_FUSE_MAX_BLOCKS = 128
tiles of RS_TILE = 2 048 keys (262 144 keys); above that a single-block rs_scan walks the 256 x nblocks counters in 16 384-counter chunks with
a running carry, and the non-fused scatter reads its offsets.  scan_block_offsets carries across chunks of 1 024 block sums, so its loop runs
a second time only above 1 048 576 counts.  The broad phase sends at most SW_WIDE_CAP = 16 384 wide intervals to its brute-force kernel; the
rest stay in the tiled sweep and its per-interval segment sort.  Every test below asserts the path it claims to run (launch count, block
count, the wide count in the reference, or rows > 262 144) and compares the device with an independent answer bit for bit:
  * the broad phase against tests/sap_reference.py (pairs, order, flags and the persistent order);
  * the collider tree against the host brute force (fixture.query_*) and a numpy box-overlap check;
  * the device contact graph against the host graphs of the ordinary World;
  * swept CCD against the host brute force (fixture.ccd_solve)."""
import numpy as np
import pytest

from avian_b200 import api, fixture, plugins, scenes

import cell_grid_model as cgm
import sap_reference as ref
from test_gpu_ccd import pile_with_projectiles, step_and_check
from test_gpu_graph import _check_graphs
from test_gpu_query import assert_same, unit, random_quats

pytestmark = pytest.mark.gpu

RS_TILE = 2048
FUSED_MAX_KEYS = 128 * RS_TILE            # the last size the fused scatter sorts
SCAN_CHUNK_COUNTERS = 1024 * 16           # rs_scan: counters per iteration
SCAN_OFFSET_CHUNK = 1024 * 1024           # scan_block_offsets: counts per iteration


# ---- broad phase ---------------------------------------------------------------------------------------------------------------------

def tied_columns(n, seed, dtype=np.float32, zero_share=0.002):
    """n intervals whose min.x sits on a 1/8 grid with ~16 intervals per grid value, in random input order: every tie run is spread over
    many 2 048-key tiles on both sides of the 128-tile boundary.  x-windows stay ~30 candidates, so the reference stays cheap."""
    rng = np.random.default_rng(seed)
    span = n / 128.0
    c = np.empty((n, 3))
    c[:, 0] = np.floor(rng.uniform(0, span, n) * 8) / 8
    c[:, 1:] = rng.uniform(0, 12.0, (n, 2))
    h = rng.uniform(0.2, 0.6, (n, 3))
    mn, mx = c - h, c + h
    mn[:, 0], mx[:, 0] = c[:, 0], c[:, 0] + 0.125
    z = rng.random(n) < zero_share
    mn[z, 0] = np.where(rng.random(int(z.sum())) < 0.5, 0.0, -0.0)
    mx[z, 0] = 0.125
    mn, mx = mn.astype(dtype), mx.astype(dtype)
    body = np.arange(n, dtype=np.uint32)
    body[1::9] = body[0::9][: len(body[1::9])]
    return api.Aabbs(collider=np.arange(n, dtype=np.uint32) * 3 + 1, body=body, aabb_min=mn, aabb_max=mx,
                     flags=rng.choice([4, 4, 4, 5, 6, 12, 20, 0], size=n).astype(np.uint8),
                     memberships=rng.choice([1, 2, 3, 0xFFFFFFFF], size=n).astype(np.uint32),
                     filters=rng.choice([1, 2, 3, 0xFFFFFFFF], size=n).astype(np.uint32), order_out=np.zeros(n, dtype=np.uint32))


def reference(a: api.Aabbs) -> ref.SapResult:
    return ref.sweep_and_prune(a.collider, a.body, a.aabb_min, a.aabb_max, flags=a.flags, memberships=a.memberships, filters=a.filters,
                               existing_pairs=a.existing_pairs, joint_disabled_body_pairs=a.joint_disabled_body_pairs)


def assert_matches(g: api.PairList, r: ref.SapResult, a: api.Aabbs, what=""):
    assert g.count == r.count, f"{what}pair count {g.count} != {r.count}"
    for k in ("collider1", "collider2", "body1", "body2", "flags"):
        a_, b_ = getattr(g, k), getattr(r, k)
        if not np.array_equal(a_, b_):
            bad = np.nonzero(a_ != b_)[0]
            raise AssertionError(f"{what}{k} differs at {bad.size} pairs, first at {bad[:5]}")
    assert a.retained_count == r.order.shape[0]
    assert np.array_equal(a.order_out[: a.retained_count], r.order), f"{what}order_out differs at {np.nonzero(a.order_out != r.order)[0][:5]}"


def launches_of(ctx, a, capacity=None):
    pairs = ctx.broadphase(a, capacity=capacity)
    return pairs, ctx.timings()["kernel_launches"]


def fused_launches(ctx, dtype):
    """kernel launches of a small broad phase (fused radix passes, no hash sets) in this context"""
    _, k = launches_of(ctx, tied_columns(5000, 0, dtype))
    return k


def expected_launches(base, n, dtype):
    """the scan path adds one rs_scan launch per radix pass: 4 (f32) or 8 (f64) for the x keys and 2 for the cell keys"""
    passes = 4 if np.dtype(dtype) == np.float32 else 8
    return base + (passes + 2 if (n + RS_TILE - 1) // RS_TILE > 128 else 0)


@pytest.mark.parametrize("n", [FUSED_MAX_KEYS, FUSED_MAX_KEYS + 1, 600_000, 1_200_000])
def test_sizes_around_the_path_switch(gpu_ctx, n):
    base = fused_launches(gpu_ctx, np.float32)
    a = tied_columns(n, n)
    r = reference(a)
    g, k = launches_of(gpu_ctx, a)
    assert k == expected_launches(base, n, np.float32), (k, base)
    nblocks = (n + RS_TILE - 1) // RS_TILE
    if n > FUSED_MAX_KEYS:
        assert nblocks > 128
    if n >= 600_000:
        assert 256 * nblocks > 2 * SCAN_CHUNK_COUNTERS          # several rs_scan chunks
    if n > SCAN_OFFSET_CHUNK:
        assert (n + 1023) // 1024 > 1024                          # scan_block_offsets carries
    assert r.count > n // 4
    assert_matches(g, r, a, f"n={n}: ")


def test_all_min_x_equal(gpu_ctx):
    """every key equal (each radix pass puts all keys in one digit): the persistent order must come back unchanged.  All but the last 200
    input rows are halo copies (they never start a sweep), so the windows stay small; the last 200 pair with everything after them."""
    n = 300_000
    base = fused_launches(gpu_ctx, np.float32)
    rng = np.random.default_rng(3)
    mn = np.column_stack([np.full(n, 1.5), rng.uniform(0, 4, (n, 2))]).astype(np.float32)
    mx = (mn + np.array([1.0, 0.5, 0.5])).astype(np.float32)
    flags = np.full(n, api.AABB_GENERATE_CONSTRAINTS | ref.AABB_HALO, np.uint8)
    flags[-200:] = api.AABB_GENERATE_CONSTRAINTS
    a = api.Aabbs(collider=np.arange(n, dtype=np.uint32), body=np.arange(n, dtype=np.uint32), aabb_min=mn, aabb_max=mx, flags=flags,
                  order_out=np.zeros(n, np.uint32))
    r = reference(a)
    g, k = launches_of(gpu_ctx, a)
    assert k == expected_launches(base, n, np.float32)
    assert np.array_equal(r.order, np.arange(n)) and r.count > 100
    assert_matches(g, r, a)


@pytest.mark.parametrize("n", [FUSED_MAX_KEYS + 1, 600_000])
def test_f64_keys(n):
    with api.Context(device=0, scalar=np.float64) as ctx:
        base = fused_launches(ctx, np.float64)
        a = tied_columns(n, 7 + n, np.float64)
        a.aabb_min[:, 0] += np.float64(2.0 ** -40) * (np.arange(n) % 3)    # keys that differ only in the low bytes (the first 4 passes)
        r = reference(a)
        g, k = launches_of(ctx, a)
        assert k == expected_launches(base, n, np.float64)
        assert_matches(g, r, a)


def test_persistent_order_across_steps(gpu_ctx):
    """the previous step's order fed back in, small moves that keep the ties: the stability contract of the scan path across steps"""
    n = 300_000
    assert (n + RS_TILE - 1) // RS_TILE > 128
    a = tied_columns(n, 21)
    rng = np.random.default_rng(5)
    for step in range(3):
        r = reference(a)
        g = gpu_ctx.broadphase(a)
        assert_matches(g, r, a, f"step {step}: ")
        perm = a.order_out.copy()
        d = (rng.integers(-2, 3, size=n) * 0.125).astype(np.float32)
        for name in ("collider", "body", "aabb_min", "aabb_max", "flags", "memberships", "filters"):
            setattr(a, name, np.ascontiguousarray(getattr(a, name)[perm]))
        a.aabb_min[:, 0] += d[perm]
        a.aabb_max[:, 0] += d[perm]
        a.order_out = np.zeros(n, dtype=np.uint32)


def over_cap_columns():
    """200 000 small intervals and 17 000 wide thin z layers (see test_over_cap_wide_intervals), in random input order"""
    rng = np.random.default_rng(8)
    ns, nw, L = 200_000, 17_000, 2000.0
    sc = np.column_stack([rng.uniform(0, L, ns), rng.uniform(0, 40, ns), rng.uniform(0, 50, ns)])
    sh = rng.uniform(0.2, 0.5, (ns, 3))
    sh[:, 0] = 0.25
    wx = np.sort(rng.uniform(0, L - 50, nw))
    wz = 0.05 * (np.arange(nw) % 1000)
    wmn = np.column_stack([wx, np.full(nw, -1.0), wz])
    wmx = np.column_stack([wx + 50.0, np.full(nw, 41.0), wz + 0.02])
    mn = np.concatenate([sc - sh, wmn]).astype(np.float32)
    mx = np.concatenate([sc + sh, wmx]).astype(np.float32)
    perm = rng.permutation(ns + nw)
    return mn[perm], mx[perm]


def test_over_cap_wide_intervals(gpu_ctx):
    """17 000 intervals that each reach over 5 000 x-candidates with a (y, z) footprint of far more than 32 cells: 16 384 go to the brute-force
    kernel, the rest stay in the tiled sweep, whose segment sort then orders segments of tens to hundreds of pairs.  The wide intervals are
    thin z layers, disjoint from every other wide interval in their x-window, so each has only tens to hundreds of pairs."""
    mn, mx = over_cap_columns()
    n = mn.shape[0]
    a = api.Aabbs(collider=np.arange(n, dtype=np.uint32), body=np.arange(n, dtype=np.uint32), aabb_min=mn, aabb_max=mx,
                  flags=np.full(n, api.AABB_GENERATE_CONSTRAINTS, np.uint8), order_out=np.zeros(n, np.uint32))
    r = reference(a)
    m = cgm.CellGridModel(mn, mx, "directed")
    assert np.array_equal(m.order, r.order) and np.array_equal(m.candidates, r.x_candidates())
    wide = m.wide
    assert wide.sum() > cgm.SW_WIDE_CAP, wide.sum()
    rank = np.empty(n, np.int64)
    rank[r.order] = np.arange(n)
    i_rank = rank[r.collider1]
    counts = np.bincount(i_rank, minlength=n)
    # tens to hundreds of pairs each: the segments the tiled sweep leaves to segment_sort are longer than a few entries
    assert counts[wide].min() >= 10 and (counts[wide] > 64).mean() > 0.5 and counts[wide].max() < 1000, (counts[wide].min(), counts[wide].max())
    g = gpu_ctx.broadphase(a)
    assert_matches(g, r, a)


def coarsening_columns():
    """300 000 small intervals in 2 000 clusters spread over 1 000 x 1 000 in (y, z)"""
    rng = np.random.default_rng(12)
    n, k = 300_000, 2000
    assert (n + RS_TILE - 1) // RS_TILE > 128
    centre = np.column_stack([rng.uniform(0, 2000, k), rng.uniform(0, 1000, k), rng.uniform(0, 1000, k)])
    c = centre[rng.integers(0, k, n)] + rng.uniform(-1.5, 1.5, (n, 3))
    h = rng.uniform(0.1, 0.3, (n, 3))
    h[:, 0] = 0.25
    return (c - h).astype(np.float32), (c + h).astype(np.float32)


def test_cell_grid_coarsening(gpu_ctx):
    """small intervals in clusters spread over 1 000 x 1 000 in (y, z): a grid of more than 0xFFFF cells before coarsening"""
    mn, mx = coarsening_columns()
    n = mn.shape[0]
    a = api.Aabbs(collider=np.arange(n, dtype=np.uint32), body=np.arange(n, dtype=np.uint32), aabb_min=mn, aabb_max=mx,
                  flags=np.full(n, api.AABB_GENERATE_CONSTRAINTS, np.uint8), order_out=np.zeros(n, np.uint32))
    ny, nz = cgm.CellGridModel(mn, mx, "directed").before
    assert ny * nz > 0xFFFF, (ny, nz)
    r = reference(a)
    assert r.count > n // 10
    assert_matches(gpu_ctx.broadphase(a), r, a)


def test_existing_pair_set_at_scale(gpu_ctx):
    """the previous step's full pair list as the existing set: no new pair; every other pair: exactly the complement"""
    n = 300_000
    assert (n + RS_TILE - 1) // RS_TILE > 128
    a = tied_columns(n, 31)
    full = reference(a)
    assert full.count > 50_000
    keys = ref.pair_key(full.collider1, full.collider2)
    a.existing_pairs = keys.copy()
    g = gpu_ctx.broadphase(a)
    assert g.count == 0
    a.existing_pairs = keys[0::2].copy()
    g = gpu_ctx.broadphase(a)
    assert g.count == full.count // 2
    for k in ("collider1", "collider2", "body1", "body2", "flags"):
        assert np.array_equal(getattr(g, k), getattr(full, k)[1::2]), k
    assert np.array_equal(a.order_out, full.order)


# ---- collider tree -------------------------------------------------------------------------------------------------------------------

N_TREE = 300_000


def test_query_tree_above_the_fused_size(gpu_ctx):
    """~300 000 rotated boxes and spheres (147 radix tiles): closest hits, every hit, box and point queries equal the brute force"""
    assert (N_TREE + RS_TILE - 1) // RS_TILE > 128
    s = np.float32
    rng = np.random.default_rng(40)
    shape = (rng.random(N_TREE) < 0.4).astype(np.uint8)
    cols = api.QueryColliders(shape=shape, dims=rng.uniform(0.2, 1.5, (N_TREE, 3)), position=rng.uniform(-62, 62, (N_TREE, 3)),
                              rotation=random_quats(rng, N_TREE))
    cols.memberships = np.where(rng.random(N_TREE) < 0.2, 2, 1).astype(np.uint32)
    m = 2000
    rays = api.Rays(origin=rng.uniform(-65, 65, (m, 3)), direction=unit(rng.normal(size=(m, 3))), max_distance=rng.uniform(5, 40, m),
                    solid=rng.random(m) < 0.5, mask=np.where(rng.random(m) < 0.2, 1, 0xFFFFFFFF).astype(np.uint32))
    gpu_ctx.query_update(cols)
    assert_same(gpu_ctx.cast_ray(rays), fixture.query_cast_ray(s, cols, rays), "cast_ray ")
    dev = gpu_ctx.ray_hits(rays)
    assert_same(dev, fixture.query_ray_hits(s, cols, rays), "ray_hits ")
    assert dev["collider"].shape[0] > m
    c, h = rng.uniform(-60, 60, (1000, 3)), rng.uniform(0, 3, (1000, 3))
    assert_same(gpu_ctx.aabb_intersections(c - h, c + h), fixture.query_aabb_intersections(s, cols, c - h, c + h), "aabb ")
    pts = api.Points(point=rng.uniform(-62, 62, (1000, 3)), solid=rng.random(1000) < 0.5)
    assert_same(gpu_ctx.project_point(pts), fixture.query_project_point(s, cols, pts), "project_point ")


def test_query_tree_all_colliders_at_one_position(gpu_ctx):
    """300 000 equal Morton codes: the whole hierarchy is split on the index bits; every ray hits every collider"""
    s = np.float32
    cols = api.QueryColliders(shape=(np.arange(N_TREE) % 2).astype(np.uint8), dims=np.full((N_TREE, 3), 0.5),
                              position=np.tile([1.0, 2.0, 3.0], (N_TREE, 1)), rotation=np.tile([0.0, 0.0, 0.0, 1.0], (N_TREE, 1)))
    rng = np.random.default_rng(5)
    m = 4
    d = unit(rng.normal(size=(m, 3)))
    rays = api.Rays(origin=np.array([1.0, 2.0, 3.0]) - 5 * d, direction=d, max_distance=np.full(m, 10.0))
    gpu_ctx.query_update(cols)
    assert_same(gpu_ctx.cast_ray(rays), fixture.query_cast_ray(s, cols, rays), "cast_ray ")
    dev = gpu_ctx.ray_hits(rays)
    assert_same(dev, fixture.query_ray_hits(s, cols, rays), "ray_hits ")
    assert np.array_equal(np.diff(dev["offsets"]), np.full(m, N_TREE))
    box = (np.array([[0.0, 1.0, 2.0], [1.6, 2.0, 3.0]]), np.array([[0.5, 1.5, 2.5], [3.0, 3.0, 3.0]]))
    got = gpu_ctx.aabb_intersections(*box)
    assert_same(got, fixture.query_aabb_intersections(s, cols, *box), "aabb ")
    assert np.array_equal(np.diff(got["offsets"]), [N_TREE, 0])


@pytest.mark.parametrize("scalar", [np.float32, np.float64])
def test_query_tree_aabb_intersections_against_numpy(scalar):
    """inclusive box overlap restated in numpy: axis-aligned boxes (identity rotation) and spheres, whose tight AABB is centre -+ half extent
    / radius rounded once in the column scalar; query boxes whose faces touch collider faces exactly"""
    rng = np.random.default_rng(50)
    shape = (rng.random(N_TREE) < 0.3).astype(np.uint8)
    dims = np.round(rng.uniform(0.25, 1.5, (N_TREE, 3)) * 4) / 4
    pos = np.round(rng.uniform(-60, 60, (N_TREE, 3)) * 4) / 4
    cols = api.QueryColliders(shape=shape, dims=dims, position=pos, rotation=np.tile([0.0, 0.0, 0.0, 1.0], (N_TREE, 1)))
    he = np.where(shape[:, None] == fixture.SHAPE_SPHERE, dims[:, :1], dims).astype(scalar)
    cmn, cmx = pos.astype(scalar) - he, pos.astype(scalar) + he
    q = 600
    qc = np.round(rng.uniform(-60, 60, (q, 3)) * 4) / 4
    qh = np.round(rng.uniform(0, 3, (q, 3)) * 4) / 4
    qmn, qmx = (qc - qh).astype(scalar), (qc + qh).astype(scalar)
    with api.Context(device=0, scalar=scalar) as ctx:
        ctx.query_update(cols)
        got = ctx.aabb_intersections(qmn, qmx)
    offs = got["offsets"].astype(np.int64)
    touching = 0
    for i in range(q):
        hit = np.all((cmn <= qmx[i]) & (cmx >= qmn[i]), axis=1)
        want = np.nonzero(hit)[0]
        mine = np.sort(got["collider"][offs[i]:offs[i + 1]].astype(np.int64))
        assert np.array_equal(mine, want), f"query {i}: {np.setxor1d(mine, want)[:10]}"
        touching += int((hit & np.any((cmn == qmx[i]) | (cmx == qmn[i]), axis=1)).sum())
    assert touching > 100                  # the inclusive edge is exercised


# ---- device contact graph ------------------------------------------------------------------------------------------------------------

def test_contact_graph_above_the_fused_size():
    """the 100k brick stack (384 750 manifolds): the device contact graph equals the host graphs for the first frame and two more steps"""
    with api.Context(device=0) as ctx_a, api.Context(device=0) as ctx_b:
        wa = plugins.World(scenes.cube_stack(51, 40, 50, brick=True), plugins.PhysicsPlugins(ctx_a), substeps=8)
        wb = plugins.DeviceGraphWorld(scenes.cube_stack(51, 40, 50, brick=True), plugins.PhysicsPlugins(ctx_b), ctx_b, substeps=8)
        for i in range(3):
            wa.step(); wb.step()
            assert wb.stats["manifold_count"] > FUSED_MAX_KEYS and wb.stats["rows_live"] > FUSED_MAX_KEYS
            _check_graphs(wa, wb, ctx_b, i)
            for k in ("position", "rotation", "linear_velocity", "angular_velocity"):
                assert np.array_equal(getattr(wa.bodies, k), getattr(wb.bodies, k)), f"step {i}: {k}"


# ---- swept CCD -----------------------------------------------------------------------------------------------------------------------

def test_ccd_above_the_fused_size():
    """more than 131 072 configured CCD bodies: the records sort has 2K > 262 144 keys.  The pile's cubes are configured with thresholds no
    relative velocity reaches (they count for the sort, not for candidates); 35 000 projectiles hit the pile."""
    scalar = np.float32
    scene, proj = pile_with_projectiles(scalar, n_side=46, layers=47, projectiles=35_000, seed=4, standoff=(44.0, 48.0))
    cubes = np.arange(1, proj[0])
    body = np.concatenate([cubes, proj])
    K = body.shape[0]
    assert 2 * K > FUSED_MAX_KEYS
    big = np.full(cubes.shape[0], 1e30)
    cfg = dict(body=body, collider=body, mode=np.arange(K) % 2, linear_threshold=np.concatenate([big, np.zeros(proj.shape[0])]),
               angular_threshold=np.concatenate([big, np.zeros(proj.shape[0])]))
    with api.Context(device=0, scalar=scalar) as ctx:
        w = plugins.DeviceGraphWorld(scene, plugins.PhysicsPlugins(ctx), ctx, substeps=4)
        ctx.ccd_configure(**cfg)
        hits = 0
        for _ in range(3):
            got = step_and_check(ctx, w, cfg, scalar)
            hits += int((got["hit_body"] >= 0).sum())
        print(f"ccd: {K} configured bodies, {hits} hits over 3 steps")
        assert hits > 1000
