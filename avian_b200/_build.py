"""In-tree builds (no JIT cache): the CUDA library, the host-side scene/narrow-phase fixture library.

`nvcc` cross-compiles sm_90a without a GPU, so the libraries can be built on a machine that has none; the
`.so` files are build products (git-ignored) and are rebuilt whenever a source is newer.
"""
from __future__ import annotations

import os
import shutil
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parent
REPO = ROOT.parent
LIB_DIR = ROOT / "lib"
CUDA_LIB = LIB_DIR / "libavian_b200.so"
HOST_LIB = LIB_DIR / "libavian_host.so"

CUDA_SOURCES = ["abi.cu", "comm.cu", "solver_host.cu", "broadphase.cu", "aabb.cu", "narrow.cu", "contacts.cu", "queries.cu", "ccd.cu"]
CUDA_HEADERS = ["avn_math.cuh", "solver_dev.cuh", "joints_dev.cuh", "solver_kernels.cuh", "context.hpp", "joint_schedule.hpp", "broadphase_cells.cuh", "narrow_math.hpp", "hull_table.hpp", "shape_column.hpp", "hull_math.hpp", "contact_rows.hpp", "query_math.hpp", "hull_query_math.hpp", "ccd_math.hpp", "move_math.hpp"]
# -fmad=false: the reference (Rust) never contracts a*b+c; parity at 1e-5 on contact dynamics needs the same
# rounding.  Division and sqrt stay IEEE (nvcc defaults -prec-div=true -prec-sqrt=true).
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]   # H100 (Hopper)
NVCC_FLAGS = [
    *GENCODE, "-lineinfo", "-O3", "-std=c++17", "-fmad=false",
    "-Xcompiler", "-fPIC", "-shared",
]
HOST_SOURCES = ["host_api.cpp"]
HOST_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wall"]


def _newer(target: Path, deps: list[Path]) -> bool:
    if not target.exists():
        return False
    t = target.stat().st_mtime
    return all(d.stat().st_mtime <= t for d in deps if d.exists())


def find_nvcc() -> str | None:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    return None


# headers each translation unit depends on (anything not listed: every header)
_UNIT_HEADERS = {
    "comm.cu": ["context.hpp", "hull_table.hpp", "shape_column.hpp"],
    "aabb.cu": ["avn_math.cuh", "context.hpp", "hull_table.hpp", "shape_column.hpp"],
    "broadphase.cu": ["avn_math.cuh", "context.hpp", "hull_table.hpp", "shape_column.hpp", "broadphase_cells.cuh", "device_prims.cuh"],
    "narrow.cu": ["avn_math.cuh", "context.hpp", "hull_table.hpp", "shape_column.hpp", "narrow_math.hpp", "hull_math.hpp", "contact_rows.hpp"],
    "contacts.cu": ["avn_math.cuh", "context.hpp", "hull_table.hpp", "shape_column.hpp", "narrow_math.hpp", "hull_math.hpp", "contact_rows.hpp", "device_prims.cuh"],
    "queries.cu": ["context.hpp", "hull_table.hpp", "shape_column.hpp", "narrow_math.hpp", "hull_math.hpp", "query_math.hpp", "hull_query_math.hpp", "move_math.hpp", "device_prims.cuh"],
    "ccd.cu": ["avn_math.cuh", "context.hpp", "hull_table.hpp", "shape_column.hpp", "narrow_math.hpp", "hull_math.hpp", "query_math.hpp", "hull_query_math.hpp", "ccd_math.hpp", "device_prims.cuh"],
}


def build_cuda(force: bool = False, verbose: bool = False) -> Path:
    """Every translation unit is compiled on its own (in parallel, only when its sources changed) and linked into one shared library."""
    src = ROOT / "csrc"
    header = REPO / "include" / "avian_b200.h"
    all_headers = sorted(p.name for p in src.glob("*.cuh")) + sorted(p.name for p in src.glob("*.hpp"))
    deps = [src / s for s in CUDA_SOURCES] + [src / h for h in all_headers] + [header]
    if not force and _newer(CUDA_LIB, deps):
        return CUDA_LIB
    nvcc = find_nvcc()
    if nvcc is None:
        if CUDA_LIB.exists():
            return CUDA_LIB  # prebuilt library shipped with the snapshot
        raise RuntimeError("nvcc not found and no prebuilt libavian_b200.so: the CUDA path cannot be built")
    LIB_DIR.mkdir(exist_ok=True)
    obj_dir = LIB_DIR / "obj"
    obj_dir.mkdir(exist_ok=True)
    compile_flags = [f for f in NVCC_FLAGS if f != "-shared"]
    jobs = []
    for unit in CUDA_SOURCES:
        obj = obj_dir / (unit + ".o")
        unit_deps = [src / unit, header, Path(__file__)] + [src / h for h in _UNIT_HEADERS.get(unit, all_headers)]
        if force or not _newer(obj, unit_deps):
            jobs.append((unit, [nvcc, *compile_flags, *(["-Xptxas", "-v"] if verbose else []), "-c", "-o", str(obj), str(src / unit)]))
    if jobs:
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 2)) as pool:
            results = list(pool.map(lambda j: (j[0], subprocess.run(j[1], cwd=src, capture_output=True, text=True)), jobs))
        for unit, r in results:
            if verbose or r.returncode != 0:
                print(f"---- {unit}\n{r.stdout}{r.stderr}")
            if r.returncode != 0:
                raise RuntimeError(f"nvcc failed on {unit}")
    subprocess.run([nvcc, "-shared", *GENCODE, "-o", str(CUDA_LIB), *[str(obj_dir / (u + ".o")) for u in CUDA_SOURCES], "-ldl"],
                   check=True, cwd=src)
    return CUDA_LIB


def build_variant(name: str, defines: list[str]) -> Path:
    """An experimental build of the library (scripts/wave_trace.py, scripts/lib_timing.py): solver_host.cu recompiled with extra -D flags,
    linked with the other units of the regular build -> avian_b200/lib/libavian_b200_<name>.so"""
    build_cuda()
    nvcc = find_nvcc()
    src, obj_dir = ROOT / "csrc", LIB_DIR / "obj"
    obj = obj_dir / f"solver_host.{name}.o"
    flags = [f for f in NVCC_FLAGS if f != "-shared"]
    subprocess.run([nvcc, *flags, *[f"-D{d}" for d in defines], "-c", "-o", str(obj), str(src / "solver_host.cu")], check=True, cwd=src)
    out = LIB_DIR / f"libavian_b200_{name}.so"
    objs = [str(obj if u == "solver_host.cu" else obj_dir / (u + ".o")) for u in CUDA_SOURCES]
    subprocess.run([nvcc, "-shared", *GENCODE, "-o", str(out), *objs, "-ldl"], check=True, cwd=src)
    return out


def build_host(force: bool = False) -> Path:
    src = ROOT / "host"
    deps = [p for p in src.glob("*.[ch]pp")] + [REPO / "include" / "avian_b200.h", ROOT / "csrc" / "narrow_math.hpp", ROOT / "csrc" / "contact_rows.hpp",
            ROOT / "csrc" / "query_math.hpp", ROOT / "csrc" / "ccd_math.hpp", ROOT / "csrc" / "move_math.hpp", ROOT / "csrc" / "hull_math.hpp", ROOT / "csrc" / "hull_query_math.hpp",
            ROOT / "csrc" / "hull_table.hpp", ROOT / "csrc" / "shape_column.hpp"]
    if not force and _newer(HOST_LIB, deps):
        return HOST_LIB
    cxx = os.environ.get("CXX") or shutil.which("g++")
    if cxx is None:
        if HOST_LIB.exists():
            return HOST_LIB
        raise RuntimeError("g++ not found and no prebuilt libavian_host.so")
    LIB_DIR.mkdir(exist_ok=True)
    subprocess.run([cxx, *HOST_FLAGS, "-o", str(HOST_LIB), *[str(src / s) for s in HOST_SOURCES]], check=True, cwd=src)
    return HOST_LIB


def build_oracle(force: bool = False) -> Path:
    """Test infrastructure only (tests/, smoke(), bench.py cpu_baseline)."""
    odir = REPO / "oracle"
    target = odir / "_build" / "liboracle.so"
    if force and target.exists():
        target.unlink()
    if shutil.which("make") and (shutil.which("g++") or os.environ.get("CXX")):
        subprocess.run(["make", "-s"], check=True, cwd=odir)
    if not target.exists():
        raise RuntimeError("oracle/_build/liboracle.so missing and cannot be built")
    return target


def build_all(force: bool = False) -> None:
    build_cuda(force)
    build_host(force)
    build_oracle(force)
