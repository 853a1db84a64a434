"""TEST INFRASTRUCTURE: swept CCD with convex hull colliders in the oracle's solver stage.  tests/oracle_ccd.py's plugin, whose pair TOI
also reads a convex hull table: the oracle's resumable stage runs tests/ccd_reference.py's solve_swept_ccd between its substeps and
restitution, with the G = 2 pair TOI of the library (fixture.ccd_pair_toi(..., hulls=)), checked on its own in tests/test_hull_ccd_cpu.py."""
from __future__ import annotations

import ctypes as C

import numpy as np

import ccd_reference
import oracle_lib
from avian_b200 import api, fixture, plugins
from oracle_ccd import OracleCcdSolverPlugin, bodies_as_ref_config


class OracleHullCcdSolverPlugin(OracleCcdSolverPlugin):
    """OracleCcdSolverPlugin over a scene with convex hulls: `hulls` is the table (api.ConvexHulls) the hull colliders index."""

    def __init__(self, hulls, config=None, threads: int = 1):
        super().__init__(config, threads)
        self.hulls = hulls

    def step_ccd(self, params, bodies: api.Bodies, manifolds, joints, ccd: dict, rows, shape, dims) -> None:
        l, dt_ = self.l, bodies.position.dtype
        bits = 32 if dt_ == np.float32 else 64
        b = bodies.as_struct()
        m = manifolds.as_struct() if manifolds is not None and manifolds.count else None
        j = joints.as_struct() if joints is not None and joints.count else None
        h = l.orc_step_begin(bits, C.byref(params), C.byref(b), C.byref(m) if m is not None else None, C.byref(j) if j is not None else None, self.threads)
        assert h, "oracle step_begin failed"
        B = int(bodies.count)
        idx = np.arange(B, dtype=np.int32)
        owner = np.zeros(B, dtype=np.int32)
        assert l.orc_step_substeps(h, int(params.substeps)) == 0
        # set after the substeps: the packed records hold the velocities themselves (tests/oracle_ccd.py)
        assert l.orc_step_set_boundary(h, C.byref(api.AvnBoundary(B, B, 0, 1, idx.ctypes.data, idx.ctypes.data, owner.ctypes.data))) == 0
        table = np.zeros(B * api.BOUNDARY_RECORD_SCALARS, dtype=dt_)
        assert l.orc_step_boundary_pack(h, table.ctypes.data) == 0
        rec = table.reshape(B, api.BOUNDARY_RECORD_SCALARS)
        lv, av = rec[:, 0:3].copy(), rec[:, 4:7].copy()
        dp, dq = rec[:, 8:11].copy(), rec[:, 12:16].copy()
        kind = bodies.kind if bodies.kind is not None else np.zeros(B, np.uint8)
        pos, rot = bodies.position, bodies.rotation
        com = bodies.center_of_mass if bodies.center_of_mass is not None else np.zeros((B, 3), dt_)
        dims = np.asarray(dims).astype(dt_)
        hull_table = fixture.HullTable(dt_, self.hulls)   # the vertices in the column scalar, as the library holds them

        def motion(body, collider):
            static = kind[body] == api.BODY_STATIC
            return fixture.ccd_motion(shape[collider], dims[collider], pos[body], rot[body], (0, 0, 0) if static else lv[body],
                                      (0, 0, 0) if static else av[body], com[body])

        pred = float(ccd.get("prediction_distance", np.inf))
        eps = 1e-4 * float(params.length_unit)

        def pair_toi(mode, b1, c1, b2, c2):
            return fixture.ccd_pair_toi(dt_, mode, motion(b1, c1), motion(b2, c2), float(params.dt), eps, pred, hulls=hull_table)

        def apply(mm, v, w, p, q):
            p2, q2 = fixture.ccd_apply_record(dt_, float(mm), v, w, p, q)
            return p2.astype(dt_), q2.astype(dt_)

        ids, c1, c2, b1, b2 = rows
        order = np.argsort(ids, kind="stable")   # ascending ContactId: the library's stated tie rule
        edge_rows = [(int(ids[e]), int(c1[e]), int(c2[e]), int(b1[e]), int(b2[e])) for e in order]
        self.last_ccd, _ = ccd_reference.solve_swept_ccd(dt_, float(params.dt), bodies_as_ref_config(ccd), edge_rows, kind, lv, av, dp, dq, pair_toi, apply)
        rec[:, 8:11], rec[:, 12:16] = dp, dq
        assert l.orc_step_boundary_apply(h, table.ctypes.data) == 0
        assert l.orc_step_restitution(h) == 0
        assert l.orc_step_finish(h) == 0


def oracle_hull_ccd_plugins(hulls, threads: int = 1, gravity=None) -> plugins.PhysicsPlugins:
    return (plugins.PhysicsPlugins().add(plugins.IntegratorPlugin(gravity)).add(oracle_lib.OracleBroadPhasePlugin())
            .add(OracleHullCcdSolverPlugin(hulls, threads=threads)))
