"""The device narrow phase (Context.narrow_phase, csrc/narrow.cu) against the independent reference of tests/narrow_reference.py, not
against the host fixture: the same soups, hand-worked pairs, swap symmetry, rigid-motion invariance and contract as
tests/test_narrow_geometry_cpu.py, in f32 and f64.  The CPU tests are run with the device in place of the fixture."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
from avian_b200 import api  # noqa: E402
import test_narrow_geometry_cpu as cpu  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("scalar", [np.float64, np.float32])
@pytest.mark.parametrize("group", cpu.GROUPS)
def test_device_soup_meets_the_contract(scalar, group):
    with api.Context(device=0, scalar=scalar) as ctx:
        for cls in cpu.CLASSES:
            s = cpu.soup(group, cls, scalar)
            assert len(s["info"]) >= cpu.MIN_PER_CLASS
            cols, lv, av, pairs = cpu.columns(s)
            out = ctx.narrow_phase(cpu.DT, cpu.TOL, pairs, cols, lv, av)
            bad = cpu.contract_violations(s, out, cols, lv, group, cls)
            assert not bad, f"{len(bad)} violations, e.g.\n" + "\n".join(bad[:12])


def _on_device(ctx, monkeypatch):
    """Route the CPU file's calls of fixture.raw_manifolds to the device narrow phase."""
    def device_raw(sc, dt, tol, pairs, cols, lv, av):
        assert np.dtype(sc) == np.dtype(ctx.scalar)
        return ctx.narrow_phase(dt, tol, pairs, cols, lv, av)
    monkeypatch.setattr(cpu.fixture, "raw_manifolds", device_raw)


@pytest.mark.parametrize("scalar", [np.float64, np.float32])
def test_device_swap_symmetry(scalar, monkeypatch):
    with api.Context(device=0, scalar=scalar) as ctx:
        _on_device(ctx, monkeypatch)
        cpu.test_swap_symmetry(scalar)


@pytest.mark.parametrize("scalar,shift", [(np.float64, 1e4), (np.float32, 1e3), (np.float32, 1e4)])
def test_device_rigid_motion_invariance(scalar, shift, monkeypatch):
    with api.Context(device=0, scalar=scalar) as ctx:
        _on_device(ctx, monkeypatch)
        cpu.test_rigid_motion_invariance(scalar, shift)


@pytest.mark.parametrize("scalar", [np.float64, np.float32])
def test_device_hand_worked_pairs(scalar, monkeypatch):
    """The hand-worked cases of the CPU file with the device in place of the fixture."""
    with api.Context(device=0, scalar=scalar) as ctx:
        _on_device(ctx, monkeypatch)
        cpu.test_box_resting_flat(scalar)
        cpu.test_turned_box_gives_an_octagon_pruned_to_four(scalar)
        cpu.test_box_on_an_edge_and_on_a_vertex(scalar)
        for q in ((0, 1, 0, 1), (0, 1, 0, 20)):
            for gap in (-0.01, 0.05):
                cpu.test_crossed_edges(scalar, q, gap)
        for q, past in (((0, 1, 0, 20), 0.1), ((0, 1, 0, 20), 0.2), ((0, 1, 0, -3), 0.1)):
            cpu.test_edge_passing_the_end_of_the_other_edge(scalar, q, past)
        for past in (0.02, 0.08, 0.15):
            cpu.test_corner_hanging_past_the_table_edge(scalar, past)
        cpu.test_sphere_sphere(scalar)
        for where in ("face", "edge", "corner", "inside", "surface"):
            cpu.test_sphere_box(scalar, where)
        for away in (True, False):
            cpu.test_keep_rule_at_the_boundary(scalar, away)
