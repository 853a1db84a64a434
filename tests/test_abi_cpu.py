"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol include/avian_b200.h
declares, its struct layouts match the ctypes mirror, it refuses to run without a GPU (no CPU fallback), and the
host-only joint level schedule is order-preserving and conflict-free."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

from avian_b200 import _build, api, scenes

ROOT = Path(__file__).resolve().parent.parent


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_library_exports_every_declared_symbol():
    header = (ROOT / "include" / "avian_b200.h").read_text()
    declared = set(re.findall(r"\b(avn_[a-z_0-9]+)\s*\(", header))
    assert {"avn_create", "avn_solver_step", "avn_broadphase", "avn_joint_levels"} <= declared
    lib = C.CDLL(str(_build.build_cuda()))
    for sym in sorted(declared):
        assert hasattr(lib, sym), f"{sym} declared in include/avian_b200.h but not exported"
    assert declared == set(api.ABI_SYMBOLS), declared ^ set(api.ABI_SYMBOLS)
    lib.avn_abi_version.restype = C.c_uint32
    assert lib.avn_abi_version() == 1


def test_struct_layouts_match_the_header():
    """sizeof of every ABI struct, compiled from the header with gcc, equals the ctypes mirror"""
    import subprocess, tempfile
    names = ["AvnConfig", "AvnStepParams", "AvnBodyColumns", "AvnManifoldColumns", "AvnJointColumns", "AvnJointSet", "AvnAabbColumns",
             "AvnPairList", "AvnTimings", "AvnBoundary", "AvnNarrowParams", "AvnNarrowInput", "AvnRawManifolds",
             "AvnContactGraphConfig", "AvnContactStep", "AvnIslandsConfig", "AvnIslandsStep"]
    src = '#include <stdio.h>\n#include "avian_b200.h"\nint main(){' + "".join(f'printf("{n} %zu\\n", sizeof({n}));' for n in names) + "return 0;}"
    with tempfile.TemporaryDirectory() as d:
        (Path(d) / "s.c").write_text(src)
        subprocess.run(["gcc", "-I", str(ROOT / "include"), "-o", f"{d}/s", f"{d}/s.c"], check=True)
        out = subprocess.run([f"{d}/s"], capture_output=True, text=True, check=True).stdout
    sizes = dict(line.split() for line in out.strip().splitlines())
    for n in names:
        assert int(sizes[n]) == C.sizeof(getattr(api, n)), n


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU behaviour")
def test_no_cpu_fallback():
    with pytest.raises(api.AvianError) as e:
        api.Context(device=0)
    assert e.value.status == api.ERR_CUDA and "no CPU fallback" in str(e.value)


def test_joint_levels_chain_and_ragdolls():
    sc = scenes.spherical_chain(25)
    lv, n = api.joint_levels(sc.bodies, sc.joints)
    assert n == 25 and np.array_equal(lv, np.arange(25))          # a chain is inherently serial
    sc = scenes.ragdoll_field(4)
    lv, n = api.joint_levels(sc.bodies, sc.joints)
    assert n <= 8 and lv.shape[0] == 64                            # ragdoll trees are shallow, ragdolls are independent


def test_joint_levels_order_preserving_and_conflict_free():
    rng = np.random.default_rng(0)
    nb, n = 60, 40
    s = np.float32
    kind = np.zeros(nb, dtype=np.uint8); kind[::13] = api.BODY_STATIC; kind[5::17] = api.BODY_KINEMATIC
    b = api.Bodies(kind=kind, position=np.zeros((nb, 3), dtype=s), rotation=np.tile(np.array([0, 0, 0, 1], dtype=s), (nb, 1)),
                   linear_velocity=np.zeros((nb, 3), dtype=s), angular_velocity=np.zeros((nb, 3), dtype=s), inverse_mass=np.ones(nb, dtype=s),
                   inverse_inertia_local=np.zeros((nb, 6), dtype=s))
    js = api.JointSet()
    glob = []
    for t in range(api.JOINT_TYPE_COUNT):
        b1 = rng.integers(0, nb, n).astype(np.int32); b2 = ((b1 + rng.integers(1, nb - 1, n)) % nb).astype(np.int32)
        js.types[t] = api.Joints(body1=b1, body2=b2, local_anchor1=np.zeros((n, 3), dtype=s), local_anchor2=np.zeros((n, 3), dtype=s))
        glob += list(zip(b1, b2))
    lv, nl = api.joint_levels(b, js)
    written = lambda x: kind[x] == api.BODY_DYNAMIC      # kinematic/static are dominated (dominance 128) next to dynamic bodies
    last = {}
    for g, (x, y) in enumerate(glob):
        for body in (x, y):
            if kind[body] == api.BODY_DYNAMIC:
                if body in last:
                    assert lv[g] > lv[last[body]], "a later joint sharing a dynamic body must run in a later level"
                last[body] = g
    for l in range(nl):
        members = [g for g in range(len(glob)) if lv[g] == l]
        dyn = [bd for g in members for bd in glob[g] if written(bd)]
        assert len(dyn) == len(set(dyn)), f"level {l} writes a body twice"


def test_fixture_manifolds_are_sane():
    """the narrow-phase fixture (inputs of the hot path): unit normals, <= 4 points, anchors on the cube surfaces"""
    import sys
    sys.path.insert(0, str(ROOT / "tests"))
    from helpers import advance_to_solver_input
    _, (prm, b, m, j) = advance_to_solver_input(scenes.cube_stack(4, 3, 4, brick=True), steps=1, substeps=2)
    assert np.allclose(np.linalg.norm(m.normal, axis=1), 1.0, atol=1e-6)
    cnt = np.diff(m.point_offsets)
    assert cnt.min() >= 1 and cnt.max() <= api.MAX_MANIFOLD_POINTS
    assert np.abs(m.anchor1).max() <= 60 and (np.abs(m.penetration) < 0.05).all()
    dyn1 = b.kind[m.body1] == api.BODY_DYNAMIC
    a1 = m.anchor1[np.repeat(dyn1, cnt)]
    assert (np.abs(a1).max(axis=1) <= 0.5 + 2e-2).all()      # on the (slightly rotated) unit cube of body1, world-frame offsets


def test_c_example_compiles_and_links():
    """examples/resident_step.c — the device-resident step written against include/avian_b200.h in plain C — compiles with -Wall -Werror
    and links with the library (every entry point it calls exists with that signature).  It is not run here (no GPU)."""
    import subprocess, tempfile
    from avian_b200 import _build
    root = Path(__file__).resolve().parent.parent
    lib = _build.build_cuda()
    with tempfile.TemporaryDirectory() as d:
        exe = Path(d) / "resident_step"
        r = subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", "-I", str(root / "include"), str(root / "examples" / "resident_step.c"),
                            "-o", str(exe), str(lib), f"-Wl,-rpath,{lib.parent}"], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        assert exe.exists()
