"""Seeded scenes for the move-and-slide tests: random colliders (cuboids and spheres, rotated, on two layers, some ignored) and random
characters (mixed shapes, some starting embedded, masks, exclusions, initial planes)."""
from __future__ import annotations

import numpy as np

from avian_b200 import api


def random_quats(rng, n):
    q = rng.normal(size=(n, 4))
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def random_colliders(rng, n, extent):
    shape = (rng.random(n) < 0.4).astype(np.uint8)                 # 40 % spheres
    dims = rng.uniform(0.2, 1.5, (n, 3))
    pos = rng.uniform(-extent, extent, (n, 3))
    memb = rng.choice(np.array([1, 2, 3], np.uint32), n)
    cols = api.QueryColliders(shape=shape, dims=dims, position=pos, rotation=random_quats(rng, n), memberships=memb)
    ignored = (rng.random(n) < 0.05).astype(np.uint8)
    return cols, ignored


def random_characters(rng, n, extent, n_colliders, speed=30.0, planes=True):
    shape = (rng.random(n) < 0.5).astype(np.uint8)
    dims = rng.uniform(0.25, 0.6, (n, 3))
    pos = rng.uniform(-extent, extent, (n, 3))
    rot = random_quats(rng, n)
    rot[rng.random(n) < 0.5] = (0.0, 0.0, 0.0, 1.0)                  # upright characters, the usual case
    d = rng.normal(size=(n, 3))
    vel = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0.0, speed, (n, 1))
    mask = rng.choice(np.array([0xFFFFFFFF, 1, 2], np.uint32), n)
    exclude = [list(rng.choice(n_colliders, size=int(rng.integers(0, 3)), replace=False)) for _ in range(n)]
    pl = None
    if planes:
        pl = []
        for i in range(n):
            r = rng.random()
            if r < 0.3:
                pl.append(np.array([[0.0, 1.0, 0.0]]))               # a ground plane
            elif r < 0.4:
                pl.append(rng.normal(size=(int(rng.integers(1, 4)), 3)))
            else:
                pl.append(None)
    return api.MoveBatch(shape=shape, dims=dims, position=pos, rotation=rot, velocity=vel, mask=mask, exclude=exclude, planes=pl)
