"""An independent float64 restatement of update_contacts' anchor transform for bodies with child colliders and an off-origin centre of mass
(narrow_phase/system_param.rs:540-570, 731-756), written from the reference and not from csrc/narrow_math.hpp:

    anchor       = (anchor relative to the collider + (collider position - body position)) - body rotation * center_of_mass
    normal_speed = dot(v2 - v1 + w2 x anchor2 - w1 x anchor1, n)
    keep         = -penetration < dt |v2 - v1|  or  normal_speed dt - penetration < dt |v2 - v1|
"""
import numpy as np


def qrot(q, v):
    """rotate the rows of v by the rows of q (x, y, z, w): v (w^2 - b.b) + 2 b (v.b) + 2 w (b x v)"""
    q, v = np.asarray(q, dtype=np.float64), np.asarray(v, dtype=np.float64)
    b, w = q[..., :3], q[..., 3:4]
    return v * (w * w - np.sum(b * b, -1, keepdims=True)) + 2.0 * b * np.sum(v * b, -1, keepdims=True) + 2.0 * w * np.cross(b, v)


def transform(anchor, collider_pos, body_pos, body_rot, com):
    """[..., 3] anchors relative to a collider -> relative to its body's centre of mass"""
    f = lambda a: np.asarray(a, dtype=np.float64)
    return (f(anchor) + (f(collider_pos) - f(body_pos))) - qrot(body_rot, f(com))


def normal_speed(a1, a2, n, v1, w1, v2, w2):
    f = lambda a: np.asarray(a, dtype=np.float64)
    rv = (f(v2) - f(v1)) + np.cross(f(w2), f(a2)) - np.cross(f(w1), f(a1))
    return np.sum(rv * f(n), -1)


def keep(penetration, ns, dt, v1, v2):
    m = dt * np.linalg.norm(np.asarray(v2, dtype=np.float64) - np.asarray(v1, dtype=np.float64), axis=-1)
    return (-penetration < m) | (ns * dt - penetration < m)
