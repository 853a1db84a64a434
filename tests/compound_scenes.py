"""Seeded pair soups with random body frames for the compound tests (CPU and GPU): collider 2k on body 2k against collider 2k+1 on body
2k+1, cuboids, spheres and capsules at random orientations and distances from deep to beyond the margin."""
import numpy as np

DT, TOL = 1.0 / 60.0, 1e-3
BOX, SPH, CAP = 0, 1, 2


def _quats(rng, n):
    q = rng.normal(size=(n, 4))
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def soup(scalar, seed, n=600, zero_frames=False, with_com=True):
    """(pairs, colliders, lin_vel, ang_vel, frames): frames = dict position, rotation, center_of_mass of the 2n bodies.  Every 5th body is
    static (no velocity).  zero_frames: every body at its collider's pose with the centre of mass at the origin."""
    rng = np.random.default_rng(seed)
    C = 2 * n
    shape = rng.integers(0, 3, size=C).astype(np.uint8)
    dims = rng.uniform(0.2, 0.8, size=(C, 3))
    dims[shape == CAP, 2] = 0.0
    pos = np.zeros((C, 3))
    pos[1::2] = rng.uniform(-1.6, 1.6, size=(n, 3))
    pos += rng.uniform(-50, 50, size=(n, 1, 3)).repeat(2, axis=0).reshape(C, 3)   # away from the world origin
    rot = _quats(rng, C)
    lv = rng.uniform(-3, 3, size=(C, 3))
    av = rng.uniform(-4, 4, size=(C, 3))
    static = np.arange(C) % 5 == 4
    lv[static] = 0.0
    av[static] = 0.0
    if zero_frames:
        bpos, brot, com = pos.copy(), rot.copy(), np.zeros((C, 3))
    else:
        brot = _quats(rng, C)
        bpos = pos - rng.uniform(-1.5, 1.5, size=(C, 3))
        com = rng.uniform(-0.6, 0.6, size=(C, 3)) if with_com else None
    s = np.dtype(scalar)
    c = lambda a: None if a is None else np.ascontiguousarray(a, dtype=s)
    c1, c2 = np.arange(0, C, 2, dtype=np.uint32), np.arange(1, C, 2, dtype=np.uint32)
    cols = {"shape": shape, "dims": c(dims), "position": c(pos), "rotation": c(rot)}
    return (c1, c2, c1.copy(), c2.copy()), cols, c(lv), c(av), {"position": c(bpos), "rotation": c(brot), "center_of_mass": c(com)}
