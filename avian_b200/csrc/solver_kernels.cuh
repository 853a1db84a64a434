// Kernels of the solver stage.
//
// Two launch strategies over the SAME per-item device routines (solver_dev.cuh / joints_dev.cuh):
//   * step_megakernel: ONE persistent cooperative kernel per physics step.  The grid is sized to exactly fill
//     the 132 SMs (occupancy x SM count); every phase of the step (prepare, each graph colour of each pass of each
//     substep, each joint level, finalize) is a grid-stride loop followed by a grid-wide barrier.  A 100k-cube
//     step has ~300-600 dependent phases of only 10^4..10^5 independent items each, so the step is bound by
//     phase latency; removing ~500 kernel launches and keeping the mutable working set hot in the 50 MB L2 between phases
//     is what the GPU wants.
//   * phase kernels: one launch per phase; the same arithmetic, used for timing single phases, for
//     the roofline measurement of the solver-iteration kernel, and as the fallback when a cooperative launch is
//     refused.
#pragma once
#include <cooperative_groups.h>

#include "joints_dev.cuh"

namespace avn {
namespace cg = cooperative_groups;

constexpr int MEGA_BLOCK = 128;  // blocks per SM is a template parameter of the megakernel (register budget = 65536 / (128 * BPS))

enum PhaseOp {
    OP_PREPARE_BODY = 0, OP_PREPARE_CONSTRAINT, OP_PREPARE_JOINT, OP_INTEGRATE_VEL, OP_INTEGRATE_POS, OP_WARM, OP_SOLVE_BIAS,
    OP_RELAX, OP_RESTITUTION, OP_SOLVE_JOINT, OP_PROJECT_VEL, OP_DAMP_JOINT, OP_WRITEBACK_BODY, OP_STORE_IMPULSE, OP_JOINT_FORCE,
    OP_WAVE_RANK, OP_WAVE_PACK
};

template <class S, int OP, int MAXP = AVN_MAX_MANIFOLD_POINTS>
__device__ __forceinline__ void run_item(const DevSolver<S>& d, int i) {
    if (OP == OP_PREPARE_BODY) prepare_body_item(d, i);
    else if (OP == OP_PREPARE_CONSTRAINT) prepare_constraint_item(d, i);
    else if (OP == OP_PREPARE_JOINT) prepare_joint_item(d, i);
    else if (OP == OP_INTEGRATE_VEL) integrate_velocity_item(d, i);
    else if (OP == OP_INTEGRATE_POS) { integrate_position_item(d, i); if (d.J > 0) store_pre_solve_item(d, i); }
    else if (OP == OP_WARM) contact_item<S, PASS_WARM, MAXP>(d, i);
    else if (OP == OP_SOLVE_BIAS) contact_item<S, PASS_SOLVE_BIAS, MAXP>(d, i);
    else if (OP == OP_RELAX) contact_item<S, PASS_RELAX, MAXP>(d, i);
    else if (OP == OP_RESTITUTION) contact_item<S, PASS_RESTITUTION, MAXP>(d, i);
    else if (OP == OP_SOLVE_JOINT) solve_joint_item(d, i);
    else if (OP == OP_PROJECT_VEL) project_velocity_item(d, i);
    else if (OP == OP_DAMP_JOINT) damp_joint_item(d, i);
    else if (OP == OP_WRITEBACK_BODY) writeback_body_item(d, i);
    else if (OP == OP_STORE_IMPULSE) store_impulse_item(d, i);
    else if (OP == OP_JOINT_FORCE) joint_force_item(d, i);
    else if (OP == OP_WAVE_RANK) wave_rank_item(d, i);
    else if (OP == OP_WAVE_PACK) wave_pack_item(d, i);
}

// one launch per phase: items [begin, begin+count).  `serial` = the overflow colour: one thread, list order.
template <class S, int OP>
__global__ void __launch_bounds__(256) phase_kernel(const __grid_constant__ DevSolver<S> d, int begin, int count, int serial) {
    if (serial) {
        if (blockIdx.x == 0 && threadIdx.x == 0)
            for (int i = 0; i < count; ++i) run_item<S, OP>(d, begin + i);
        return;
    }
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) run_item<S, OP>(d, begin + i);
}

// __noinline__: each phase keeps its own register allocation instead of the union of all phases
template <class S, int OP, int MAXP = AVN_MAX_MANIFOLD_POINTS>
__device__ __noinline__ void grid_phase(const DevSolver<S>& d, int begin, int count) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) run_item<S, OP, MAXP>(d, begin + i);
}

template <class S, int OP, int MAXP = AVN_MAX_MANIFOLD_POINTS>
__device__ __noinline__ void grid_serial(const DevSolver<S>& d, int begin, int count) {
    for (int i = 0; i < count; ++i) run_item<S, OP, MAXP>(d, begin + i);
}

// all graph colours of one contact pass, reference order: overflow colour serially first, then colours 0..22
// (solver/plugin.rs:461-479, 553-572, 643-668)
template <class S, int OP, int MAXP = AVN_MAX_MANIFOLD_POINTS>
__device__ __forceinline__ void grid_contact_pass(const DevSolver<S>& d, cg::grid_group& grid) {
    const int ov = d.color_off[AVN_COLOR_OVERFLOW], ovn = d.color_len[AVN_COLOR_OVERFLOW];
    if (ovn > 0) {
        if (blockIdx.x == 0 && threadIdx.x == 0) grid_serial<S, OP, MAXP>(d, ov, ovn);
        grid.sync();
    }
    for (int c = 0; c < AVN_COLOR_OVERFLOW; ++c) {
        const int b = d.color_off[c], n = d.color_len[c];
        if (n <= 0) continue;
        grid_phase<S, OP, MAXP>(d, b, n);
        grid.sync();
    }
}

// ---- wavefront substep loop ------------------------------------------------------------------------------------------
// The whole substep schedule as ONE sequence of 32-item chunks; warp w takes chunks w, w + W, w + 2W, ... in order and
// every item waits on its bodies' event counters instead of a grid barrier (solver_dev.cuh "wavefront mode").  Chunks
// never straddle two phases or two colours because body ranges and colour slot ranges are padded to multiples of 32.
// WAVE_CHUNK items per warp (lanes >= WAVE_CHUNK idle).  A warp waits for the slowest of its items' predecessors, so a smaller chunk
// shortens the per-level latency (fewer predecessors per warp) at the cost of idle lanes — the machine has lanes to spare
// (DESIGN.md 3.1).  Must divide 32; colour slot ranges are padded to multiples of 32, so chunks never straddle colours either way.
#ifndef AVN_WAVE_CHUNK
#define AVN_WAVE_CHUNK 32
#endif
constexpr int WAVE_CHUNK = AVN_WAVE_CHUNK;
// The wavefront routines are __noinline__ (each keeps its own register allocation) and take BPS and MAXP as template parameters so that
// every megakernel variant owns its copies, compiled under that variant's register budget.  The solve routine serves the biased and the
// relax pass.
template <class S, int PASS, int MAXP, int BPS>
__device__ __noinline__ void wave_contact_chunk(const DevSolver<S>& d, int slot, int s, int it, bool active, bool relax) {
    wave_contact_item<S, PASS, MAXP>(d, slot, s, it, active, relax);
}
template <class S, int BPS, int MAXP>
__device__ __noinline__ void wave_iv_chunk(const DevSolver<S>& d, int i, int s, bool active) { integrate_velocity_item<S, true>(d, i, s, active); }
template <class S, int BPS, int MAXP>
__device__ __noinline__ void wave_ip_chunk(const DevSolver<S>& d, int i, int s, bool active) { integrate_position_item<S, true>(d, i, s, active); }

// EXPERIMENT (off): L2 prefetch of the immutable constraint rows of the chunk this warp processes one iteration from now.  The idea: at
// 100k bodies the planes (>100 MB) stream from HBM every pass and an item can do nothing before its index row has arrived.  The measurement
// says the 16 extra CCTL per item cost more than the latency they hide.
template <class S, int MAXP>
__device__ __forceinline__ void wave_prefetch_slot(const DevSolver<S>& d, int slot) {
#ifdef AVN_WAVE_PREFETCH   // slower when it was introduced: kept as an experiment
    const char* base = reinterpret_cast<const char*>(d.cst + slot);
    const size_t stride = size_t(d.Mpad) * sizeof(Vec4<S>);
#pragma unroll
    for (int r = 0; r < CP_PT0 + 3 * MAXP; ++r) asm volatile("prefetch.global.L2 [%0];" ::"l"(base + size_t(r) * stride));
#endif
}

template <class S, int MAXP, int BPS>
__device__ __forceinline__ void wave_substep_loop(const DevSolver<S>& d) {
    const int lane = threadIdx.x & 31;
    const bool active = lane < WAVE_CHUNK;
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    long long warp_id = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (d.sm_slots) {
        // SM-major numbering of the warps: the BPS blocks of one SM take 4 * BPS CONSECUTIVE chunks of the schedule — the same pass, the same
        // colour, neighbouring plane rows — instead of chunks one SM count of blocks apart, so the warps of an SM run the same routine on adjacent memory.
        // Exactly BPS blocks are resident per SM (cooperative launch of BPS x SM-count blocks under a BPS-blocks register limit), every block
        // draws one ticket of its SM; the counters only ever grow by BPS per launch, so they stay multiples of BPS without a reset.
        // %smid values need not be dense (disabled SMs leave gaps): the first block that arrives on an SM claims the next dense index for it,
        // once for the lifetime of the context (sm_slots[256 + smid] = dense index + 1, sm_slots[512] = SMs seen)
        __shared__ int ticket, dense;
        unsigned smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        if (threadIdx.x == 0) {
            const int t = atomicAdd(&d.sm_slots[smid & 255u], 1);
            ticket = t % BPS;
            int* slot = &d.sm_slots[256 + (smid & 255u)];
            if (ticket == 0 && atomicAdd(slot, 0) == 0) atomicExch(slot, atomicAdd(&d.sm_slots[512], 1) + 1);
            int v;
            while ((v = atomicAdd(slot, 0)) == 0) { }      // the SM's other blocks are resident with this one: the claim is on its way
            dense = v - 1;
        }
        __syncthreads();
        warp_id = ((long long)dense * BPS + ticket) * (blockDim.x >> 5) + (threadIdx.x >> 5);
    }
    const int body_chunks = (d.B + WAVE_CHUNK - 1) / WAVE_CHUNK, slot_chunks = d.Mpad / WAVE_CHUNK;
    const int first_chunks = body_chunks;                           // integrate_velocities
    const int front_passes = 1 + d.iters;                           // warm, iters x solve: the slot passes before integrate_positions
    const long long per_substep = (long long)first_chunks + body_chunks + (long long)(front_passes + 1) * slot_chunks;
    const long long total = per_substep * d.sub_end;
    // position of a chunk inside its substep -> slot of its first item, or -1 for a body chunk (prefetch experiment)
    [[maybe_unused]] auto contact_slot_of = [&](long long r) -> int {
        if (r < first_chunks) return -1;
        r -= first_chunks;
        if (r < (long long)front_passes * slot_chunks) return int(r % slot_chunks) * WAVE_CHUNK;
        r -= (long long)front_passes * slot_chunks;
        if (r < body_chunks) return -1;
        return int(r - body_chunks) * WAVE_CHUNK;
    };
    for (long long g = per_substep * d.sub_begin + warp_id; g < total; g += warps) {
        const int s = int(g / per_substep);
        long long r = g - (long long)s * per_substep;
#ifdef AVN_WAVE_PREFETCH
        {   // the chunk after this one
            const long long gn = g + warps;
            if (gn < total) {
                const int ns = contact_slot_of(gn % per_substep);
                if (ns >= 0 && active) wave_prefetch_slot<S, MAXP>(d, ns + lane);
            }
        }
#endif
        if (r < first_chunks) {
            wave_iv_chunk<S, BPS, MAXP>(d, int(r) * WAVE_CHUNK + lane, s, active);
            continue;
        }
        r -= first_chunks;
        if (r < (long long)front_passes * slot_chunks) {
            const int pass = int(r / slot_chunks), slot = int(r - (long long)pass * slot_chunks) * WAVE_CHUNK + lane;
            if (pass == 0) wave_contact_chunk<S, PASS_WARM, MAXP, BPS>(d, slot, s, 0, active, false);
            else wave_contact_chunk<S, PASS_SOLVE_BIAS, MAXP, BPS>(d, slot, s, pass - 1, active, false);
            continue;
        }
        r -= (long long)front_passes * slot_chunks;
        if (r < body_chunks) { wave_ip_chunk<S, BPS, MAXP>(d, int(r) * WAVE_CHUNK + lane, s, active); continue; }
        r -= body_chunks;
        wave_contact_chunk<S, PASS_SOLVE_BIAS, MAXP, BPS>(d, int(r) * WAVE_CHUNK + lane, s, 0, active, true);
    }
}

// ---- island-group substep loop ----------------------------------------------------------------------------------------------------
// A scene of many small islands (island_lists.hpp): thread block k takes island GROUPS k, k + gridDim, ... through the WHOLE substep loop; the
// phases of the barrier schedule follow each other in the same order with __syncthreads() in place of the grid barriers, and since no other
// block touches the group's bodies or constraints, its state lives in this SM's L1 for the duration.  Same per-item routines, same per-body
// order: bit-identical.  (One WARP per island was measured 10x slower than the barrier schedule on 5 000 ragdolls: the handful of joints an
// island has per level are of different types, so the lanes of the warp run the joint routines one type after the other; a group of islands
// per block keeps the items of a level sorted by type across its warps, like the grid-wide phase does.)
template <class S, int OP, int MAXP>
__device__ __noinline__ void island_phase(const DevSolver<S>& d, const int* __restrict__ list, int lo, int hi) {
    for (int k = lo + int(threadIdx.x); k < hi; k += int(blockDim.x)) run_item<S, OP, MAXP>(d, list[k]);
    __syncthreads();
}
template <class S, int OP, int MAXP>
__device__ __forceinline__ void island_contact_pass(const DevSolver<S>& d, int isl) {
    const int* off = d.isl_m_off + size_t(isl) * (AVN_GRAPH_COLOR_COUNT + 1);
    for (int c = 0; c < AVN_COLOR_OVERFLOW; ++c) {
        const int lo = off[c], hi = off[c + 1];
        if (hi > lo) island_phase<S, OP, MAXP>(d, d.isl_mslots, lo, hi);
    }
}
template <class S, int MAXP>
__device__ __forceinline__ void island_substep_loop(const DevSolver<S>& d) {
    for (int isl = int(blockIdx.x); isl < d.isl_count; isl += int(gridDim.x)) {
        const int b0 = d.isl_body_off[isl], b1 = d.isl_body_off[isl + 1];
        const int* joff = d.isl_j_off + size_t(isl) * (d.isl_levels + 1);
        const bool has_m = d.M > 0 && d.isl_m_off[size_t(isl) * (AVN_GRAPH_COLOR_COUNT + 1)] < d.isl_m_off[size_t(isl) * (AVN_GRAPH_COLOR_COUNT + 1) + AVN_GRAPH_COLOR_COUNT];
        for (int sub = d.sub_begin; sub < d.sub_end; ++sub) {
            island_phase<S, OP_INTEGRATE_VEL, MAXP>(d, d.isl_bodies, b0, b1);
            if (has_m) {
                island_contact_pass<S, OP_WARM, MAXP>(d, isl);
                for (int it = 0; it < d.iters; ++it) island_contact_pass<S, OP_SOLVE_BIAS, MAXP>(d, isl);
            }
            island_phase<S, OP_INTEGRATE_POS, MAXP>(d, d.isl_bodies, b0, b1);
            if (has_m) island_contact_pass<S, OP_RELAX, MAXP>(d, isl);
            if (d.J > 0) {
                for (int l = 0; l < d.isl_levels; ++l)
                    if (joff[l + 1] > joff[l]) island_phase<S, OP_SOLVE_JOINT, MAXP>(d, d.isl_jslots, joff[l], joff[l + 1]);
                island_phase<S, OP_PROJECT_VEL, MAXP>(d, d.isl_bodies, b0, b1);
                if (d.any_joint_damping)
                    for (int l = 0; l < d.isl_levels; ++l)
                        if (joff[l + 1] > joff[l]) island_phase<S, OP_DAMP_JOINT, MAXP>(d, d.isl_jslots, joff[l], joff[l + 1]);
            }
        }
    }
}

template <class S, int BPS, int MAXP>
__global__ void __launch_bounds__(MEGA_BLOCK, BPS) step_megakernel(const __grid_constant__ DevSolver<S> d) {
    cg::grid_group grid = cg::this_grid();
    // ---- prepare
    if (d.do_prepare) {
        grid_phase<S, OP_PREPARE_BODY>(d, 0, d.B + 1);
        grid.sync();
        grid_phase<S, OP_PREPARE_CONSTRAINT>(d, 0, d.M);
        grid_phase<S, OP_PREPARE_JOINT>(d, 0, d.J);
        grid.sync();
        if (d.wave) {
            // ranks of every constraint on its bodies, colour by colour in schedule order (deg[] was zeroed by the host)
            for (int c = 0; c < AVN_COLOR_OVERFLOW; ++c) {
                if (d.color_len[c] <= 0) continue;
                grid_phase<S, OP_WAVE_RANK>(d, d.color_off[c], d.color_len[c]);
                grid.sync();
            }
            grid_phase<S, OP_WAVE_PACK>(d, 0, d.Mpad);
            grid.sync();
        }
    }
    // ---- run_substep_schedule (solver/schedule.rs:194-213), substeps [sub_begin, sub_end)
    // the wavefront schedule is only entered with a colouring the rank pass found valid (and no watchdog event in an earlier launch of this
    // step); otherwise the barrier schedule below runs, which terminates on any input (read after a grid barrier: uniform over the grid)
    const bool wave = d.wave && *reinterpret_cast<volatile int*>(d.any_restitution + 1) == 0;
    if (wave && d.sub_end > d.sub_begin) {
        wave_substep_loop<S, MAXP, BPS>(d);
        grid.sync();
    }
    const bool islands = !wave && d.isl_count > 0;
    if (islands && d.sub_end > d.sub_begin) {
        island_substep_loop<S, MAXP>(d);
        grid.sync();
    }
    for (int sub = d.sub_begin; sub < ((wave || islands) ? 0 : d.sub_end); ++sub) {
        grid_phase<S, OP_INTEGRATE_VEL>(d, 0, d.B);
        grid.sync();
        if (d.M > 0) {
            grid_contact_pass<S, OP_WARM, MAXP>(d, grid);
            for (int it = 0; it < d.iters; ++it) grid_contact_pass<S, OP_SOLVE_BIAS, MAXP>(d, grid);
        }
        grid_phase<S, OP_INTEGRATE_POS>(d, 0, d.B);
        grid.sync();
        if (d.M > 0) grid_contact_pass<S, OP_RELAX, MAXP>(d, grid);
        if (d.J > 0) {
            for (int l = 0; l < d.n_levels; ++l) {
                const int b = d.level_off[l], n = d.level_off[l + 1] - b;
                grid_phase<S, OP_SOLVE_JOINT>(d, b, n);
                grid.sync();
            }
            grid_phase<S, OP_PROJECT_VEL>(d, 0, d.B);
            grid.sync();
            if (d.any_joint_damping) {
                for (int l = 0; l < d.n_levels; ++l) {
                    const int b = d.level_off[l], n = d.level_off[l + 1] - b;
                    grid_phase<S, OP_DAMP_JOINT>(d, b, n);
                    grid.sync();
                }
            }
        }
    }
    // ---- restitution, writeback, store impulses
    if (d.do_restitution && d.M > 0 && *d.any_restitution) grid_contact_pass<S, OP_RESTITUTION, MAXP>(d, grid);
    if (d.do_finalize) {
        grid_phase<S, OP_WRITEBACK_BODY>(d, 0, d.B);
        grid_phase<S, OP_STORE_IMPULSE>(d, 0, d.M);
        grid_phase<S, OP_JOINT_FORCE>(d, 0, d.J);
    }
}

}  // namespace avn
