"""TEST INFRASTRUCTURE: swept CCD in the oracle's solver stage.  The oracle's resumable stage (orc_step_begin -> substeps -> restitution ->
finish, oracle/oracle_step.cpp) is driven step by step, and solve_swept_ccd runs between the substeps and restitution as
tests/ccd_reference.py restates it (ccd/mod.rs:523-687), on the oracle's own SolverBodies: their velocities and deltas are read and written
through the stage's boundary record table (every body one record, one rank, set after the substeps so that no reference velocity is
subtracted: the table holds the velocities themselves).  Only the pair TOI and the write of one record come from the library (fixture.ccd_pair_toi / ccd_apply_record): that arithmetic
is parry's and glam's in the reference and is checked on its own in tests/test_ccd_cpu.py."""
from __future__ import annotations

import ctypes as C

import numpy as np

import ccd_reference
import oracle_lib
from avian_b200 import api, fixture, plugins


def bodies_as_ref_config(ccd: dict) -> list[dict]:
    """World(ccd=...) keyword arguments -> the per-body dicts of ccd_reference.solve_swept_ccd."""
    n = len(ccd["body"])
    col = lambda k, default: [default] * n if ccd.get(k) is None else list(ccd[k])
    return [dict(body=int(b), collider=int(c), mode=int(m), include_dynamic=bool(i), linear_threshold=float(l), angular_threshold=float(a))
            for b, c, m, i, l, a in zip(ccd["body"], ccd["collider"], col("mode", api.SWEEP_NON_LINEAR), col("include_dynamic", 1),
                                        col("linear_threshold", 0.0), col("angular_threshold", 0.0))]


class OracleCcdSolverPlugin(oracle_lib.OracleSolverPlugin):
    """The oracle's solver stage with solve_swept_ccd; `last_ccd` holds the last step's (min_toi, hit body, ContactId) per CCD body."""

    def __init__(self, config=None, threads: int = 1):
        super().__init__(config, threads)
        oracle_lib.OracleSlabEngine()   # declares the orc_step_* entry points
        self.l = oracle_lib.lib()
        self.last_ccd = None

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
        # set after the substeps (which would snapshot reference velocities into it): the packed records hold the velocities themselves
        assert l.orc_step_set_boundary(h, C.byref(api.AvnBoundary(B, B, 0, 1, idx.ctypes.data, idx.ctypes.data, owner.ctypes.data))) == 0
        table = np.zeros(B * api.BOUNDARY_RECORD_SCALARS, dtype=dt_)
        assert l.orc_step_boundary_pack(h, table.ctypes.data) == 0
        rec = table.reshape(B, api.BOUNDARY_RECORD_SCALARS)
        lv, av = rec[:, 0:3].copy(), rec[:, 4:7].copy()
        dp, dq = rec[:, 8:11].copy(), rec[:, 12:16].copy()
        kind = bodies.kind if bodies.kind is not None else np.zeros(B, np.uint8)
        pos, rot = bodies.position, bodies.rotation      # Position / Rotation before the step: writeback has not run yet
        com = bodies.center_of_mass if bodies.center_of_mass is not None else np.zeros((B, 3), dt_)
        dims = np.asarray(dims).astype(dt_)   # the column scalar, as the contact pipeline holds them

        def motion(body, collider):
            static = kind[body] == api.BODY_STATIC
            return fixture.ccd_motion(shape[collider], dims[collider], pos[body], rot[body], (0, 0, 0) if static else lv[body],
                                      (0, 0, 0) if static else av[body], com[body])

        pred = float(ccd.get("prediction_distance", np.inf))
        eps = 1e-4 * float(params.length_unit)

        def pair_toi(mode, b1, c1, b2, c2):
            return fixture.ccd_pair_toi(dt_, mode, motion(b1, c1), motion(b2, c2), float(params.dt), eps, pred)

        def apply(mm, v, w, p, q):
            p2, q2 = fixture.ccd_apply_record(dt_, float(mm), v, w, p, q)
            return p2.astype(dt_), q2.astype(dt_)

        ids, c1, c2, b1, b2 = rows
        order = np.argsort(ids, kind="stable")   # ascending ContactId: the library's stated tie rule
        edge_rows = [(int(ids[e]), int(c1[e]), int(c2[e]), int(b1[e]), int(b2[e])) for e in order]
        self.last_ccd, _ = ccd_reference.solve_swept_ccd(dt_, float(params.dt), bodies_as_ref_config(ccd), edge_rows, kind, lv, av, dp, dq, pair_toi, apply)
        rec[:, 8:11], rec[:, 12:16] = dp, dq
        assert l.orc_step_boundary_apply(h, table.ctypes.data) == 0   # velocities: 0 + v; deltas: the ones CCD left
        assert l.orc_step_restitution(h) == 0
        assert l.orc_step_finish(h) == 0


def oracle_ccd_plugins(threads: int = 1, gravity=None) -> plugins.PhysicsPlugins:
    return (plugins.PhysicsPlugins().add(plugins.IntegratorPlugin(gravity)).add(oracle_lib.OracleBroadPhasePlugin())
            .add(OracleCcdSolverPlugin(threads=threads)))
