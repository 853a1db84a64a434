"""x-slab partition on the device (SURVEY.md §8e row 2).  One GPU is enough for the partition logic itself (the slabs run one after
the other on one context); the NCCL all-gather needs two and is skipped otherwise."""
import os
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
from avian_b200 import api, parallel, scenes  # noqa: E402
import oracle_lib  # noqa: E402
from test_slab_cpu import assert_same_pairs, random_aabbs  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("scalar", [np.float32, np.float64])
@pytest.mark.parametrize("world", [2, 4])
def test_slabs_on_one_device_concatenate_to_the_single_list(world, scalar):
    a = random_aabbs(6000, seed=world + 10, scalar=scalar)
    want = oracle_lib.broadphase(a)
    want_order = a.order_out.copy()
    with api.Context(device=0, scalar=scalar) as ctx:
        single = ctx.broadphase(a)
        assert_same_pairs(single, want)
        cuts = parallel.slab_cuts(a.aabb_min[:, 0], world)
        parts = [parallel.slab_broadphase_local(ctx.broadphase, a, cuts, r) for r in range(world)]
    got, order = parallel.merge_slab_results(parts, a.collider)
    assert_same_pairs(got, want)
    assert np.array_equal(order, want_order)
    assert max(p[0]["collider1"].shape[0] for p in parts) < want.count


def test_stack_scene_slabs_on_one_device(gpu_ctx):
    """The headline scene's geometry (brick stack on a ground slab that every slab's sweep must see) cut into 4 slabs."""
    from avian_b200 import plugins
    sc = scenes.cube_stack(12, 6, 10, brick=True)
    w = plugins.World(sc, plugins.PhysicsPlugins(gpu_ctx), substeps=2)
    w.step()
    a = w.pipeline.intervals(w.bodies, w.aabb_min, w.aabb_max, with_existing=False)
    a.order_out = np.zeros(a.collider.shape[0], dtype=np.uint32)
    want = oracle_lib.broadphase(a)
    want_order = a.order_out.copy()
    cuts = parallel.slab_cuts(a.aabb_min[:, 0], 4)
    parts = [parallel.slab_broadphase_local(gpu_ctx.broadphase, a, cuts, r) for r in range(4)]
    got, order = parallel.merge_slab_results(parts, a.collider)
    assert_same_pairs(got, want)
    assert np.array_equal(order, want_order)


def _nccl_worker(rank, world, port, q):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    info = parallel.init(backend="nccl")
    a = random_aabbs(20000, seed=5)
    with api.Context(device=rank) as ctx:
        got, order = parallel.slab_broadphase(ctx.broadphase, a, info, device=f"cuda:{rank}")
    q.put((rank, got.count, {c: getattr(got, c).copy() for c in parallel.PAIR_COLUMNS}, order))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_nccl_slab_broadphase():
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + (os.getpid() % 1000)
    procs = [ctx.Process(target=_nccl_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = sorted((q.get(timeout=300) for _ in range(world)), key=lambda r: r[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    a = random_aabbs(20000, seed=5)
    want = oracle_lib.broadphase(a)
    for rank, count, cols, order in results:
        assert count == want.count
        for c in parallel.PAIR_COLUMNS:
            assert np.array_equal(cols[c], getattr(want, c)[:want.count]), (rank, c)
        assert np.array_equal(order, a.order_out)


# ---- the solver stage cut into slabs ---------------------------------------------------------------------------------------
from helpers import RTOL, advance_to_solver_input, assert_bodies_close, assert_manifolds_close  # noqa: E402
from test_slab_solver_cpu import stack_input, two_piles_input  # noqa: E402


def _gpu_lockstep(prm, b, m, world, scalar=np.float32, cuts=None):
    ctxs = [api.Context(device=0, scalar=scalar) for _ in range(world)]
    try:
        return parallel.slab_solver_step_local(lambda r: parallel.GpuSlabEngine(ctxs[r]), prm, b, m, world, cuts)
    finally:
        for c in ctxs:
            c.close()


@pytest.mark.parametrize("mode", [None, "barrier", "phases"])
@pytest.mark.parametrize("world", [2, 3])
def test_slab_solver_on_one_device_matches_the_oracle_partition(world, mode, monkeypatch):
    """The same partition, the same exchange arithmetic: CUDA engines vs oracle engines, 1e-5 like every solver parity test."""
    if mode:
        monkeypatch.setenv("AVN_LAUNCH_MODE", mode)
    prm, b, m = stack_input(nx=10, ny=4, nz=4, steps=3, substeps=6)
    bo, mo = b.copy(), m.copy()
    so = parallel.slab_solver_step_local(lambda r: oracle_lib.OracleSlabEngine(), prm, bo, mo, world)
    bg, mg = b.copy(), m.copy()
    sg = _gpu_lockstep(prm, bg, mg, world)
    assert so[0].slot_count == sg[0].slot_count > 0
    assert_bodies_close(bg, bo, what=f"slabs {world} {mode}: ")
    assert_manifolds_close(mg, mo, what=f"slabs {world} {mode}: ")


def test_slab_solver_uncoupled_piles_bit_for_bit(gpu_ctx):
    prm, b, m = two_piles_input()
    bs, ms = b.copy(), m.copy()
    gpu_ctx.solver_step(prm, bs, ms)
    bg, mg = b.copy(), m.copy()
    shards = _gpu_lockstep(prm, bg, mg, 2, cuts=np.array([15.0], dtype=np.float32))
    assert shards[0].slot_count == 0
    for k in parallel.BODY_OUTPUTS:
        assert np.array_equal(getattr(bg, k), getattr(bs, k)), k
    for k in parallel.POINT_OUTPUTS:
        assert np.array_equal(getattr(mg, k), getattr(ms, k)), k


def test_slab_solver_restitution_and_f64():
    _, (prm, b, m, j) = advance_to_solver_input(scenes.cube_stack(6, 3, 3, brick=True, restitution=0.5, scalar=np.float64), steps=2, substeps=3)
    b.linear_velocity[:, 1] -= 2.0
    bo, mo = b.copy(), m.copy()
    parallel.slab_solver_step_local(lambda r: oracle_lib.OracleSlabEngine(), prm, bo, mo, 2)
    bg, mg = b.copy(), m.copy()
    _gpu_lockstep(prm, bg, mg, 2, scalar=np.float64)
    assert_bodies_close(bg, bo, rtol=1e-9, what="slabs f64 restitution: ")


def test_run_range_equals_one_launch(gpu_ctx):
    """avn_solver_run_range substep by substep (no boundary) is the same arithmetic as avn_solver_run."""
    prm, b, m = stack_input()
    b1, m1 = b.copy(), m.copy()
    gpu_ctx.solver_step(prm, b1, m1)
    b2, m2 = b.copy(), m.copy()
    gpu_ctx.solver_upload(prm, b2, m2, None)
    n = int(prm.substeps)
    for s in range(n):
        gpu_ctx.solver_run_range(s, 1, api.RUN_PREPARE if s == 0 else 0)
    gpu_ctx.solver_run_range(n, 0, api.RUN_RESTITUTION)
    gpu_ctx.solver_run_range(n, 0, api.RUN_FINALIZE)
    gpu_ctx.solver_download()
    assert np.array_equal(b1.position, b2.position) and np.array_equal(b1.linear_velocity, b2.linear_velocity)
    assert np.array_equal(m1.warm_start_normal_impulse, m2.warm_start_normal_impulse)
    with pytest.raises(api.AvianError):
        gpu_ctx.solver_upload(prm, b2, m2, None)
        gpu_ctx.solver_run_range(1, 1, 0)          # the first launch after an upload must prepare


def _nccl_solver_worker(rank, world, port, q):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    info = parallel.init(backend="nccl")
    prm, b, m = stack_input(nx=10, ny=4, nz=4, steps=3, substeps=6)
    with api.Context(device=rank) as ctx:
        parallel.slab_solver_step(parallel.GpuSlabEngine(ctx), prm, b, m, info, device=f"cuda:{rank}")
    q.put((rank, {k: getattr(b, k).copy() for k in parallel.BODY_OUTPUTS}, {k: getattr(m, k).copy() for k in parallel.POINT_OUTPUTS}))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_nccl_slab_solver():
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + (os.getpid() % 1000)
    procs = [ctx.Process(target=_nccl_solver_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = sorted((q.get(timeout=300) for _ in range(world)), key=lambda r: r[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    prm, b, m = stack_input(nx=10, ny=4, nz=4, steps=3, substeps=6)
    parallel.slab_solver_step_local(lambda r: oracle_lib.OracleSlabEngine(), prm, b, m, world)
    from helpers import rel_err
    for rank, bodies, points in results:
        for k in parallel.BODY_OUTPUTS:
            assert rel_err(bodies[k], getattr(b, k)) <= RTOL, (rank, k)
    for k in parallel.BODY_OUTPUTS:      # both ranks hold the same bits
        assert np.array_equal(results[0][1][k], results[1][1][k]), k


# ---- the partitioned stage inside the library: NCCL behind the C ABI (avn_comm_init + avn_solver_step_partitioned) -------------------
def test_step_partitioned_with_a_communicator_of_one_equals_solver_run(gpu_ctx):
    """world = 1 needs no NCCL: avn_solver_step_partitioned == avn_solver_run bit for bit."""
    prm, b, m = stack_input()
    b1, m1 = b.copy(), m.copy()
    gpu_ctx.solver_step(prm, b1, m1)
    b2, m2 = b.copy(), m.copy()
    gpu_ctx.comm_init(0, 1, None)
    gpu_ctx.solver_upload(prm, b2, m2, None)
    gpu_ctx.solver_step_partitioned()
    gpu_ctx.solver_download()
    for k in parallel.BODY_OUTPUTS:
        assert np.array_equal(getattr(b1, k), getattr(b2, k)), k
    for k in parallel.POINT_OUTPUTS:
        assert np.array_equal(getattr(m1, k), getattr(m2, k)), k


def _lib_nccl_worker(rank, world, id_path, q):
    """No torch.distributed anywhere: the unique id travels through a file, the collective lives in libavian_b200.so."""
    import time
    torch.cuda.set_device(rank)
    prm, b, m = stack_input(nx=10, ny=4, nz=4, steps=3, substeps=6)
    with api.Context(device=rank) as ctx:
        if rank == 0:
            tmp = id_path + ".tmp"
            with open(tmp, "wb") as f:
                f.write(ctx.comm_unique_id())
            os.replace(tmp, id_path)
        t0 = time.time()
        while not os.path.exists(id_path):
            assert time.time() - t0 < 120, "unique id never arrived"
            time.sleep(0.05)
        with open(id_path, "rb") as f:
            uid = f.read()
        ctx.comm_init(rank, world, uid)
        cuts = parallel.body_slab_cuts(b, world)
        sh = parallel.shard_solver(b, m, cuts, rank, world)
        ctx.solver_upload(prm, sh.bodies, sh.manifolds, None)
        ctx.solver_set_boundary(sh.bnd_body, sh.bnd_source, sh.bnd_owner, sh.record_count, rank, world)
        ctx.solver_step_partitioned()
        ctx.solver_download()
        rows = sh.body_index[sh.owned_body]
        q.put((rank, rows, {k: getattr(sh.bodies, k)[sh.owned_body].copy() for k in parallel.BODY_OUTPUTS}, sh.point_index,
               {} if sh.manifolds is None else {k: getattr(sh.manifolds, k).copy() for k in parallel.POINT_OUTPUTS}, sh.slot_count))
        ctx.comm_destroy()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="NCCL refuses two ranks on one device: needs 2 GPUs "
                                                          "(scripts/multi_gpu_checks.sh runs it)")
def test_two_gpu_library_nccl_partitioned_step(tmp_path):
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    id_path = str(tmp_path / "nccl_id.bin")
    procs = [ctx.Process(target=_lib_nccl_worker, args=(r, world, id_path, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = sorted((q.get(timeout=300) for _ in range(world)), key=lambda r: r[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    prm, b, m = stack_input(nx=10, ny=4, nz=4, steps=3, substeps=6)
    bg, mg = b.copy(), m.copy()
    for rank, rows, bodies, pidx, points, slots in results:
        assert slots > 0
        for k in parallel.BODY_OUTPUTS:
            getattr(bg, k)[rows] = bodies[k]
        for k, v in points.items():
            getattr(mg, k)[pidx] = v
    bo, mo = b.copy(), m.copy()
    parallel.slab_solver_step_local(lambda r: oracle_lib.OracleSlabEngine(), prm, bo, mo, world)
    assert_bodies_close(bg, bo, what="library NCCL slabs: ")
    assert_manifolds_close(mg, mo, what="library NCCL slabs: ")
    # and the library-driven step is the same arithmetic as the caller-driven one (lockstep engines on one device)
    bl, ml = b.copy(), m.copy()
    _gpu_lockstep(prm, bl, ml, world)
    for k in parallel.BODY_OUTPUTS:
        assert np.array_equal(getattr(bg, k), getattr(bl, k)), k


# ---- island sharding of one scene: exact ------------------------------------------------------------------------------------
def test_island_sharded_step_on_device_is_bit_identical(gpu_ctx):
    """SURVEY §8e row 1: the ragdoll field dealt island by island to 3 ranks' worth of avn_solver_step calls (one after the other on this
    device) is the single call bit for bit — contacts, joints, joint forces."""
    from test_island_cpu import assert_same_step, ragdoll_input
    prm, b, m, j = ragdoll_input()
    bs, ms, js = b.copy(), m.copy(), j.copy()
    gpu_ctx.solver_step(prm, bs, ms, js)
    bg, mg, jg = b.copy(), m.copy(), j.copy()
    shards = parallel.island_solver_step_local(gpu_ctx.solver_step, prm, bg, mg, jg, 3)
    assert min(sh.bodies.count for sh in shards) > 17
    assert_same_step(bg, mg, jg, bs, ms, js)
