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
// The whole substep schedule as ONE sequence of 32-item chunks, one item per lane; warp w takes chunks w, w + W, w + 2W, ... in order and
// every item waits on its bodies' event counters instead of a grid barrier (solver_dev.cuh "wavefront mode").  Chunks
// never straddle two phases or two colours because body ranges and colour slot ranges are padded to multiples of 32.
constexpr int WAVE_CHUNK = 32;
// The wavefront routines are __noinline__ (each keeps its own register allocation) and take BPS and MAXP as template parameters so that
// every megakernel variant owns its copies, compiled under that variant's register budget.  The solve routine serves the biased and the
// relax pass.
template <class S, int PASS, int MAXP, int BPS>
__device__ __noinline__ void wave_contact_chunk(const DevSolver<S>& d, int slot, int s, int it, bool relax) {
    wave_contact_item<S, PASS, MAXP>(d, slot, s, it, relax);
}
template <class S, int BPS, int MAXP>
__device__ __noinline__ void wave_iv_chunk(const DevSolver<S>& d, int i, int s) { integrate_velocity_item<S, true>(d, i, s); }
template <class S, int BPS, int MAXP>
__device__ __noinline__ void wave_ip_chunk(const DevSolver<S>& d, int i, int s) { integrate_position_item<S, true>(d, i, s); }

template <class S, int MAXP, int BPS>
__device__ __forceinline__ void wave_substep_loop(const DevSolver<S>& d) {
    const int lane = threadIdx.x & 31;
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    const long long warp_id = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int body_chunks = (d.B + WAVE_CHUNK - 1) / WAVE_CHUNK, slot_chunks = d.Mpad / WAVE_CHUNK;
    const int first_chunks = body_chunks;                           // integrate_velocities
    const int front_passes = 1 + d.iters;                           // warm, iters x solve: the slot passes before integrate_positions
    const long long per_substep = (long long)first_chunks + body_chunks + (long long)(front_passes + 1) * slot_chunks;
    const long long total = per_substep * d.sub_end;
    for (long long g = per_substep * d.sub_begin + warp_id; g < total; g += warps) {
        const int s = int(g / per_substep);
        long long r = g - (long long)s * per_substep;
        if (r < first_chunks) {
            wave_iv_chunk<S, BPS, MAXP>(d, int(r) * WAVE_CHUNK + lane, s);
            continue;
        }
        r -= first_chunks;
        if (r < (long long)front_passes * slot_chunks) {
            const int pass = int(r / slot_chunks), slot = int(r - (long long)pass * slot_chunks) * WAVE_CHUNK + lane;
            if (pass == 0) wave_contact_chunk<S, PASS_WARM, MAXP, BPS>(d, slot, s, 0, false);
            else wave_contact_chunk<S, PASS_SOLVE_BIAS, MAXP, BPS>(d, slot, s, pass - 1, false);
            continue;
        }
        r -= (long long)front_passes * slot_chunks;
        if (r < body_chunks) { wave_ip_chunk<S, BPS, MAXP>(d, int(r) * WAVE_CHUNK + lane, s); continue; }
        r -= body_chunks;
        wave_contact_chunk<S, PASS_SOLVE_BIAS, MAXP, BPS>(d, int(r) * WAVE_CHUNK + lane, s, 0, true);
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
    for (int sub = d.sub_begin; sub < (wave ? 0 : d.sub_end); ++sub) {
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
