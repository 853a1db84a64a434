"""avian_b200 — H100-native (sm_90a) replacement for the avian3d substep hot path.

Hot path = semi-implicit integration (IntegratorPlugin), sweep-and-prune broad phase (BroadPhasePlugin) and
the TGS-soft contact + XPBD joint solve (SolverPlugin / XpbdSolverPlugin) of avianphysics/avian, behind the
C ABI of include/avian_b200.h.  This package holds the CUDA sources (csrc/), the ctypes binding of the ABI
(api.py), the host-side mirror of the three plugins (plugins.py) and the host fixture that stands in for the
parts of the reference that stay on the CPU (host/: scenes, AABBs, narrow-phase manifolds, contact graph and
constraint-graph colouring).
"""
from . import api  # noqa: F401
from .api import Context, AvianError, default_step_params  # noqa: F401

__all__ = ["api", "Context", "AvianError", "default_step_params"]
