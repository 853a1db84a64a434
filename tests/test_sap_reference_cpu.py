"""Pins tests/sap_reference.py (the vectorised numpy sweep that the at-scale GPU tests compare against) on the CPU: it must equal the
hand-worked serial sweep of tests/golden/handworked/worked.py, and the oracle's literal insertion sort + double loop bit for bit (pairs, order,
flags, persistent order) in f32 and f64."""
import importlib.util
import json
from pathlib import Path

import numpy as np
import pytest

from avian_b200 import api

import oracle_lib
import sap_reference as ref

HERE = Path(__file__).resolve().parent
_spec = importlib.util.spec_from_file_location("handworked_worked", HERE / "golden" / "handworked" / "worked.py")
worked = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(worked)


def _worked_intervals(collider, body, mn, mx, memb, filt, inactive):
    return [dict(collider=int(collider[k]), body=int(body[k]), min=mn[k], max=mx[k], memberships=int(memb[k]), filters=int(filt[k]),
                 inactive=bool(inactive[k])) for k in range(len(collider))]


def _check_against_worked(collider, body, mn, mx, memb, filt, inactive):
    pairs, order = worked.sweep_and_prune(_worked_intervals(collider, body, mn, mx, memb, filt, inactive))
    flags = np.where(inactive, api.AABB_IS_INACTIVE, 0).astype(np.uint8) | np.uint8(api.AABB_GENERATE_CONSTRAINTS)
    r = ref.sweep_and_prune(collider, body, mn, mx, flags=flags, memberships=memb, filters=filt)
    assert [(int(a), int(b)) for a, b in zip(r.collider1, r.collider2)] == [tuple(p) for p in pairs]
    assert r.order.tolist() == order
    assert (r.flags == ref.PAIR_GENERATE_CONSTRAINTS).all()
    return r


def test_six_intervals_worked_by_hand():
    vec = json.loads((HERE / "golden" / "handworked" / "vectors.json").read_text())["sap_six"]
    iv = vec["intervals"]
    for dtype in (np.float32, np.float64):
        cols = [np.array([x[k] for x in iv]) for k in ("collider", "body")]
        mn, mx = np.array([x["min"] for x in iv], dtype=dtype), np.array([x["max"] for x in iv], dtype=dtype)
        memb, filt = (np.array([x[k] for x in iv], dtype=np.uint32) for k in ("memberships", "filters"))
        r = _check_against_worked(*cols, mn, mx, memb, filt, np.array([x["inactive"] for x in iv]))
        assert [[int(a), int(b)] for a, b in zip(r.collider1, r.collider2)] == vec["expected_pairs"]
        assert r.order.tolist() == vec["expected_order"]


@pytest.mark.parametrize("seed", range(6))
def test_small_random_equals_worked(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(0, 60))
    dtype = np.float32 if seed % 2 else np.float64
    c = np.round(rng.uniform(-4, 4, (n, 3)) * 2) / 2
    h = rng.uniform(0.1, 1.0, (n, 3))
    mn, mx = (c - h).astype(dtype), (c + h).astype(dtype)
    mn[rng.random(n) < 0.1, 0] = -0.0
    mn[rng.random(n) < 0.1, 0] = 0.0
    body = rng.integers(0, max(n // 2, 1), n)
    memb = rng.choice([1, 2, 3], n).astype(np.uint32)
    filt = rng.choice([1, 2, 0xFFFFFFFF], n).astype(np.uint32)
    _check_against_worked(np.arange(n) * 7 + 3, body, mn, mx, memb, filt, rng.random(n) < 0.3)


def random_columns(n, seed, dtype, halo=False):
    """ties on min.x, +-0, shared bodies, layers, every flag, a few non-finite bounds"""
    rng = np.random.default_rng(seed)
    c = rng.uniform(-20, 20, (n, 3))
    c[:, 0] = np.round(c[:, 0] * 4) / 4
    h = rng.uniform(0.1, 1.5, (n, 3))
    h[:, 0] = rng.choice([0.25, 0.5, 2.0], n)
    mn, mx = (c - h).astype(dtype), (c + h).astype(dtype)
    z = rng.random(n) < 0.05
    mn[z, 0] = np.where(rng.random(int(z.sum())) < 0.5, 0.0, -0.0)
    touch = rng.random(n) < 0.05               # y bounds that touch a neighbour's exactly (inclusive overlap)
    mn[touch, 1] = np.roll(mx[:, 1], 1)[touch]
    body = np.arange(n, dtype=np.uint32)
    body[1::7] = body[0::7][: len(body[1::7])]
    flags = rng.choice([4, 4, 4, 5, 6, 12, 20, 0, 1, 2, 8, 16], n).astype(np.uint8)
    if halo:
        flags |= rng.choice([0, 0, 0, ref.AABB_HALO, ref.AABB_SPLIT_I, ref.AABB_NOT_J], n).astype(np.uint8)
    bad = rng.choice(n, min(n, 5), replace=False) if n > 50 else []
    for k, i in enumerate(bad):
        (mn if k % 2 else mx)[i, k % 3] = [np.nan, np.inf, -np.inf][k % 3]
    return api.Aabbs(collider=(np.arange(n, dtype=np.uint32) * 3 + 1), body=body, aabb_min=mn, aabb_max=mx, flags=flags,
                     memberships=rng.choice([1, 2, 3, 0xFFFFFFFF], n).astype(np.uint32), filters=rng.choice([1, 2, 3, 0xFFFFFFFF], n).astype(np.uint32),
                     order_out=np.zeros(n, dtype=np.uint32))


def reference_of(a: api.Aabbs, **kw) -> ref.SapResult:
    return ref.sweep_and_prune(a.collider, a.body, a.aabb_min, a.aabb_max, flags=a.flags, memberships=a.memberships, filters=a.filters,
                               existing_pairs=a.existing_pairs, joint_disabled_body_pairs=a.joint_disabled_body_pairs, **kw)


def assert_equals_pairlist(r: ref.SapResult, p: api.PairList, order_out=None, retained=None):
    assert r.count == p.count, (r.count, p.count)
    for k in ("collider1", "collider2", "body1", "body2", "flags"):
        assert np.array_equal(getattr(r, k), getattr(p, k)), k
    if order_out is not None:
        assert retained == r.order.shape[0]
        assert np.array_equal(order_out[:retained], r.order)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n,seed,halo", [(0, 0, False), (1, 1, False), (300, 2, True), (3000, 3, False), (4000, 4, True)])
def test_equals_oracle(n, seed, halo, dtype):
    a = random_columns(n, seed, dtype, halo)
    o = oracle_lib.broadphase(a)
    r = reference_of(a, chunk=977)        # a small chunk: many chunk boundaries, including ones inside one interval's window run
    assert_equals_pairlist(r, o, a.order_out, a.retained_count)
    if n >= 3000:
        assert o.count > 1000 and len(np.unique(o.flags)) > 3


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_existing_and_joint_disabled_equal_oracle(dtype):
    a = random_columns(3000, 9, dtype)
    full = oracle_lib.broadphase(random_columns(3000, 9, dtype))
    rng = np.random.default_rng(0)
    pick = rng.random(full.count) < 0.5
    a.existing_pairs = ref.pair_key(full.collider1[pick], full.collider2[pick])
    a.joint_disabled_body_pairs = ref.pair_key(full.body1[~pick][::3], full.body2[~pick][::3])
    o = oracle_lib.broadphase(a)
    assert 0 < o.count < full.count
    assert_equals_pairlist(reference_of(a), o, a.order_out, a.retained_count)


def test_window_bounds_and_inverted_intervals():
    """end = the sweep's break position; an interval with max.x < min.x has an empty window, exactly as the loop's first test breaks"""
    mn = np.array([[0, 0, 0], [1, 0, 0], [1, 0, 0], [3, 0, 0], [5, 0, 0]], dtype=np.float32)
    mx = np.array([[1, 1, 1], [0.5, 1, 1], [4, 1, 1], [3, 1, 1], [6, 1, 1]], dtype=np.float32)
    a = api.Aabbs(collider=np.arange(5, dtype=np.uint32), body=np.arange(5, dtype=np.uint32), aabb_min=mn, aabb_max=mx,
                  flags=np.full(5, 4, np.uint8), order_out=np.zeros(5, np.uint32))
    r = reference_of(a)
    assert r.end.tolist() == [3, 2, 4, 4, 5]
    assert_equals_pairlist(r, oracle_lib.broadphase(a), a.order_out, a.retained_count)


def test_imports_nothing_of_the_library():
    src = (HERE / "sap_reference.py").read_text()
    assert "import avian_b200" not in src and "from avian_b200" not in src and "oracle" not in src.replace("oracle/", "")
