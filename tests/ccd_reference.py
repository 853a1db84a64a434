"""solve_swept_ccd (avian dynamics/ccd/mod.rs:523-687) restated in plain Python, independent of the library's control flow.

Only the pair time of impact (`pair_toi`, parry's cast in the reference) and the delta write of one record (`apply`, glam's from_scaled_axis
and quaternion product) are passed in: everything else — the visiting order, the filters and their order, the mode rule, the strict `<`, the
fallback's acceptance, the overshoot and the sequential application onto the SolverBodies — is written here from the Rust.
"""
from __future__ import annotations

import numpy as np

LINEAR, NON_LINEAR = 0, 1
STATIC, DYNAMIC = 2, 0


def solve_swept_ccd(scalar, dt, ccd_bodies, rows, kind, lin_vel, ang_vel, delta_position, delta_rotation, pair_toi, apply):
    """ccd_bodies: list of dicts (body, collider, mode, include_dynamic, linear_threshold, angular_threshold) in query order.
    rows: list of (contact_id, collider1, collider2, body1, body2), the ContactGraph's live edges in the order a body's neighbours are visited.
    pair_toi(mode, body1, collider1, body2, collider2) -> the TOI in the column scalar, or -1: compute_ccd_toi against the bound dt, fallback
    included.  apply(m, v, w, dp, dq) -> (dp, dq): the write of one record.  delta_position / delta_rotation are updated in place.
    Returns per CCD body (min_toi, hit body or -1, ContactId or -1) and the list of (body, m) writes in the order they happen."""
    s = np.dtype(scalar).type
    dt = s(dt)
    mode_of_body = {c["body"]: c.get("mode", NON_LINEAR) for c in ccd_bodies}
    has_solver_body = lambda b: kind[b] != STATIC
    vel = lambda col, b: np.asarray(col[b], dtype=s) if has_solver_body(b) else np.zeros(3, dtype=s)   # SolverBody::DUMMY
    results, writes = [], []
    for c in ccd_bodies:
        b1 = c["body"]
        if not has_solver_body(b1):                        # no SolverBody: the query item does not match
            results.append((dt, -1, -1))
            continue
        v1, w1 = vel(lin_vel, b1), vel(ang_vel, b1)
        min_toi, hit, hit_id = dt, -1, -1
        lt, at = s(c.get("linear_threshold", 0.0)), s(c.get("angular_threshold", 0.0))
        for (cid, c1, c2, r1, r2) in rows:
            if c["collider"] not in (c1, c2):
                continue
            other, b2 = (c2, r2) if c1 == c["collider"] else (c1, r1)
            if not c.get("include_dynamic", True) and kind[b2] == DYNAMIC:
                continue
            v2, w2 = vel(lin_vel, b2), vel(ang_vel, b2)
            dw, dv = w1 - w2, v1 - v2
            ang_below = (dw[0] * dw[0] + dw[1] * dw[1]) + dw[2] * dw[2] < at * at
            if ang_below and (dv[0] * dv[0] + dv[1] * dv[1]) + dv[2] * dv[2] < lt * lt:
                continue
            linear = c.get("mode", NON_LINEAR) == LINEAR and mode_of_body.get(b2, LINEAR) == LINEAR
            toi = s(pair_toi(LINEAR if linear else NON_LINEAR, b1, c["collider"], b2, other))
            if s(0) < toi < min_toi:
                min_toi, hit, hit_id = toi, b2, cid
        results.append((min_toi, hit, hit_id))
        if hit < 0:
            continue
        m = s(min_toi * s(1.0001))
        for b in (b1, hit):
            if not has_solver_body(b):                     # the dummy body: the write is discarded
                continue
            delta_position[b], delta_rotation[b] = apply(m, vel(lin_vel, b), vel(ang_vel, b), delta_position[b], delta_rotation[b])
            writes.append((b, m))
    return results, writes
