"""An independent, vectorised numpy restatement of the sweep-and-prune broad phase (collision/broad_phase.rs:394-428, the insertion sort of
:479-487), for checking the device at sizes where the literal double loop is far too slow.

It shares nothing with the library or with oracle/: the flag values below are copied from include/avian_b200.h, and everything else follows
the reference's semantics directly:
  * intervals whose AABB has a non-finite bound are dropped (update_aabb_intervals' retain, broad_phase.rs:243-245);
  * the survivors are stably sorted by min.x in their input (persistent) order, -0.0 comparing equal to +0.0 (the insertion sort swaps
    only on a strict '>');
  * interval i is tested against every later j up to the first one whose min.x exceeds max.x[i] (the sweep's `break`);
  * a candidate becomes a pair when y and z overlap (inclusive), the two are not both inactive, each one's memberships meet the other's
    filters, they sit on different bodies, the collider pair is not in the existing set and the body pair is not joint-disabled.  The
    x-slab partition's halo flags (AVN_AABB_HALO / SPLIT_I / NOT_J) are applied as the header defines them;
  * pairs come out ordered by (rank of i, rank of j) in the sorted order.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

# include/avian_b200.h
AABB_IS_INACTIVE = 0x01
AABB_CONTACT_EVENTS = 0x02
AABB_GENERATE_CONSTRAINTS = 0x04
AABB_CUSTOM_FILTER = 0x08
AABB_MODIFY_CONTACTS = 0x10
AABB_NOT_J = 0x20
AABB_SPLIT_I = 0x40
AABB_HALO = 0x80
PAIR_CONTACT_EVENTS = 0x01
PAIR_MODIFY_CONTACTS = 0x02
PAIR_GENERATE_CONSTRAINTS = 0x04
PAIR_NEEDS_HOOK = 0x08


@dataclass
class SapResult:
    collider1: np.ndarray     # uint32[P]
    collider2: np.ndarray
    body1: np.ndarray
    body2: np.ndarray
    flags: np.ndarray         # uint8[P] PAIR_*
    order: np.ndarray         # uint32[R] the new persistent order: input rows of the retained intervals, sorted by min.x
    end: np.ndarray           # int64[R] per sorted rank: one past the last x-candidate (the sweep's break position)

    @property
    def count(self) -> int:
        return int(self.collider1.shape[0])

    def x_candidates(self) -> np.ndarray:
        """per sorted rank: the number of later intervals in its x-window"""
        return self.end - np.arange(self.end.shape[0]) - 1


def pair_key(a, b) -> np.ndarray:
    """PairKey (data_structures/pair_key.rs:15-21): (min << 32) | max"""
    a, b = np.asarray(a, dtype=np.uint64), np.asarray(b, dtype=np.uint64)
    return (np.minimum(a, b) << np.uint64(32)) | np.maximum(a, b)


def pair_flags(fi: np.ndarray, fj: np.ndarray) -> np.ndarray:
    u = fi.astype(np.uint32) | fj.astype(np.uint32)
    out = np.zeros(u.shape, dtype=np.uint8)
    for aabb, pair in ((AABB_CONTACT_EVENTS, PAIR_CONTACT_EVENTS), (AABB_MODIFY_CONTACTS, PAIR_MODIFY_CONTACTS),
                       (AABB_GENERATE_CONSTRAINTS, PAIR_GENERATE_CONSTRAINTS), (AABB_CUSTOM_FILTER, PAIR_NEEDS_HOOK)):
        out |= np.where(u & aabb, pair, 0).astype(np.uint8)
    return out


def sweep_and_prune(collider, body, aabb_min, aabb_max, flags=None, memberships=None, filters=None, existing_pairs=None,
                    joint_disabled_body_pairs=None, chunk: int = 1 << 22) -> SapResult:
    """The broad phase's pair list and persistent order.  Columns as in AvnAabbColumns (aabb_min / aabb_max: [n, 3] in the scalar type the
    comparisons are made in); absent memberships / filters / flags default to 1 / all / GENERATE_CONSTRAINTS.  `chunk` bounds the number of
    x-candidates expanded at once."""
    mn_all, mx_all = np.asarray(aabb_min), np.asarray(aabb_max)
    n_all = mn_all.shape[0]
    finite = np.isfinite(mn_all).all(axis=1) & np.isfinite(mx_all).all(axis=1)
    keep = np.nonzero(finite)[0]
    # + 0.0 turns -0.0 into +0.0, so the stable sort sees them as equal keys, as the reference's '>' does
    order = keep[np.argsort(mn_all[keep, 0] + mn_all.dtype.type(0), kind="stable")]
    n = order.shape[0]
    col = np.asarray(collider, dtype=np.uint32)[order]
    bod = np.asarray(body, dtype=np.uint32)[order]
    fl = (np.full(n_all, AABB_GENERATE_CONSTRAINTS, np.uint8) if flags is None else np.asarray(flags, dtype=np.uint8))[order]
    memb = (np.ones(n_all, np.uint32) if memberships is None else np.asarray(memberships, dtype=np.uint32))[order]
    filt = (np.full(n_all, 0xFFFFFFFF, np.uint32) if filters is None else np.asarray(filters, dtype=np.uint32))[order]
    mn, mx = mn_all[order], mx_all[order]
    minx = mn[:, 0]
    ranks = np.arange(n, dtype=np.int64)
    end = np.maximum(np.searchsorted(minx, mx[:, 0], side="right"), ranks + 1)   # first j > i with min.x[j] > max.x[i]
    cnt = end - ranks - 1
    cnt[(fl & AABB_HALO) != 0] = 0        # a halo interval never starts a sweep
    existing = None if existing_pairs is None or len(existing_pairs) == 0 else np.unique(np.asarray(existing_pairs, dtype=np.uint64))
    jdis = None if joint_disabled_body_pairs is None or len(joint_disabled_body_pairs) == 0 else \
        np.unique(np.asarray(joint_disabled_body_pairs, dtype=np.uint64))

    out_i, out_j = [], []
    cum = np.concatenate([[0], np.cumsum(cnt)])
    lo = 0
    while lo < n:
        # the next run of intervals whose candidates fit the chunk (at least one interval)
        hi = max(lo + 1, int(np.searchsorted(cum, cum[lo] + chunk, side="right")) - 1)
        hi = min(hi, n)
        c = cnt[lo:hi]
        total = int(c.sum())
        lo_next = hi
        if total:
            ii = np.repeat(ranks[lo:hi], c)
            starts = np.repeat(cum[lo:hi] - cum[lo], c)
            jj = ii + 1 + (np.arange(total, dtype=np.int64) - starts)
            ok = ~((mn[ii, 1] > mx[jj, 1]) | (mx[ii, 1] < mn[jj, 1]) | (mn[ii, 2] > mx[jj, 2]) | (mx[ii, 2] < mn[jj, 2]))
            ii, jj = ii[ok], jj[ok]
            fi, fj = fl[ii], fl[jj]
            ok = ((fi & fj & AABB_IS_INACTIVE) == 0) & ((memb[ii] & filt[jj]) != 0) & ((memb[jj] & filt[ii]) != 0) & (bod[ii] != bod[jj])
            ok &= ((fj & AABB_NOT_J) == 0) & ~(((fi & AABB_SPLIT_I) != 0) & ((fj & AABB_HALO) != 0))
            ii, jj = ii[ok], jj[ok]
            if existing is not None:
                ok = ~np.isin(pair_key(col[ii], col[jj]), existing, assume_unique=False)
                ii, jj = ii[ok], jj[ok]
            if jdis is not None:
                ok = ~np.isin(pair_key(bod[ii], bod[jj]), jdis, assume_unique=False)
                ii, jj = ii[ok], jj[ok]
            out_i.append(ii)
            out_j.append(jj)
        lo = lo_next
    ii = np.concatenate(out_i) if out_i else np.zeros(0, np.int64)
    jj = np.concatenate(out_j) if out_j else np.zeros(0, np.int64)
    return SapResult(collider1=col[ii], collider2=col[jj], body1=bod[ii], body2=bod[jj], flags=pair_flags(fl[ii], fl[jj]),
                     order=order.astype(np.uint32), end=end)
