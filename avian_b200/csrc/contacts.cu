// The device-resident contact store (SURVEY.md 8f #1/#3, DESIGN.md §7b).
// One row per ContactId (contact_graph.rs:521-631 assigns them; so does the ContactGraph below).  A row holds the pair (colliders, bodies), the
// manifold the last narrow phase found (4 point slots, column scalar type: what the solver reads through avn_solver_upload_resident), the
// unrounded anchors of that manifold (double: what the next step's match_contacts compares) and the warm-start impulses (in = what the
// next solve starts from, written by the matching; out = what the last solve left, written by store_contact_impulses).
#include <cooperative_groups.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "context.hpp"
#include "contact_rows.hpp"
#include "device_prims.cuh"

namespace avn {
namespace {
namespace cg = cooperative_groups;

// =====================================================================================================================================
// The ContactGraph and the ConstraintGraph on the device (SURVEY.md 8f #3).
//   ContactGraph::add_edge_and_key_with (contact_graph.rs:521-565): new pairs take the lowest free ContactIds in list order (IdPool,
//     data_structures/id_pool.rs:43-52) — the k-th new pair gets the k-th smallest free row, rows beyond the free ones are appended.
//   NarrowPhase::update's status loop (narrow_phase/system_param.rs:136-389) visits the changed contacts in ASCENDING ContactId: a pair
//     whose AABBs separated leaves the graph (its manifold is popped), a pair that started touching pushes its manifold into the
//     ConstraintGraph, a pair that stopped touching pops it.
//   ConstraintGraph::push_manifold (solver/constraint_graph.rs:163-238) is GREEDY: dynamic-dynamic takes the lowest of the first
//     AVN_DYNAMIC_COLOR_COUNT colours whose body set holds neither body, dynamic-static the highest colour below the overflow colour that does
//     not hold the dynamic body, anything else lands in the overflow colour; pop_manifold (:240-296) clears the bodies from the set.
// The colour a push gets depends on every earlier push and pop that shares a body, so the result is order dependent — and the order of
// the colours IS the Gauss-Seidel order of the solver.  The device reproduces the sequential result exactly with a dependency wavefront:
// in every round a changed edge runs iff it is the smallest pending ContactId on each of its non-static bodies (64-bit atomicMin tagged
// with the round: no reset pass); edges of one round share no non-static body, so they commute.  Pops only clear bits, so they commute with each
// other anyway: a POP waits only for the earlier pending PUSHES on its bodies (second minimum per body), a PUSH for everything earlier.  The number of rounds is the longest chain
// of changed edges linked through shared bodies in ascending id (a few in the steady state, thousands on the first frame of a big pile).
// Inside a colour the order of the manifolds does not influence the solve (they share no dynamic body), so the colour-major list is built
// in ascending ContactId by one stable radix pass; only the overflow colour, which the solver walks serially, keeps the reference's
// push / swap_remove list order, maintained by one thread.
// =====================================================================================================================================
enum { CH_NONE = 0, CH_PUSH = 1, CH_POP = 2, CH_REMOVE = 3, CH_MASK = 3, CH_DONE = 0x10 };
enum { ISL_NONE = 0, ISL_ADD = 1, ISL_REMOVE = 2 };

struct GraphCounters {          // device block, copied to the host once per step
    // cleared at the start of every step
    uint32_t removed, started, stopped, changed, rounds, ovf_dirty, manifolds, any_restitution, aborted, bad_pairs;
    uint32_t rows_woken, rows_slept, bodies_asleep;   // applied sleeping: what the last wake / sleep pass did, bodies asleep after it
    uint32_t round_left[3];
    uint32_t color_offsets[AVN_GRAPH_COLOR_COUNT + 1];
    // persistent
    uint32_t ovf_count;
    uint32_t rows_asleep;
};

struct GraphRows {
    int hw;                                       // rows in use: ContactIds [0, hw)
    uint32_t* c1; uint32_t* c2; uint32_t* b1; uint32_t* b2;
    uint8_t* live; uint8_t* count; uint8_t* disjoint; uint8_t* prev_count;
    uint8_t* pflags; uint8_t* touching; uint8_t* colour /* 0 = none, c + 1 */; uint8_t* change; uint8_t* old_colour;
    uint8_t* fresh;                               // the row was added in this step (its geometry is still to be computed)
    uint8_t* isl_event;                           // this step's event for the islands: ISL_ADD / ISL_REMOVE (a linked contact came or went)
    uint8_t* event;                               // this step's collision event: EV_STARTED / EV_ENDED | the pair's AVN_PAIR_* flags (0 = none)
    uint8_t* asleep;                              // the row sleeps with an island (avn_islands_apply): live and touching, out of the ConstraintGraph, left alone
    const uint8_t* sensor;                        // [C] Sensor per collider (avn_contacts_set_sensors); NULL = none
    uint32_t* ovf_pos; uint32_t* ovf;
    const uint8_t* body_kind; int n_bodies;
    uint32_t* body_bits;                          // [B] bit c: the body is in colour c's body set
    unsigned long long* body_min;                 // [B][2] round-tagged smallest pending ContactId: [0] over all pending edges, [1] over the pending PUSHES
    GraphCounters* ctr;
};

__global__ void add_rows_kernel(GraphRows g, uint32_t n_new, const uint32_t* __restrict__ pc1, const uint32_t* __restrict__ pc2, const uint32_t* __restrict__ pb1,
                                const uint32_t* __restrict__ pb2, const uint8_t* __restrict__ pfl, const uint32_t* __restrict__ free_list, uint32_t n_free,
                                uint32_t old_hw, uint32_t n_colliders) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_new) return;
    const uint32_t e = k < n_free ? free_list[k] : old_hw + (k - n_free);
    // the rows are gathered through on the device (collider poses, body velocities, body sets): a pair outside the configured counts is
    // counted and stored as a pair of body 0 / collider 0 that can never touch (the step then fails with AVN_ERR_INVALID_ARGUMENT)
    const bool bad = pc1[k] >= n_colliders || pc2[k] >= n_colliders || pb1[k] >= uint32_t(g.n_bodies) || pb2[k] >= uint32_t(g.n_bodies);
    if (bad) {
        atomicAdd(&g.ctr->bad_pairs, 1u);
        g.c1[e] = 0; g.c2[e] = 0; g.b1[e] = 0; g.b2[e] = 0; g.pflags[e] = 0; g.isl_event[e] = 0; g.fresh[e] = 0;
        g.live[e] = 0; g.count[e] = 0; g.prev_count[e] = 0; g.touching[e] = 0; g.colour[e] = 0; g.change[e] = 0; g.asleep[e] = 0;
        return;
    }
    g.c1[e] = pc1[k]; g.c2[e] = pc2[k]; g.b1[e] = pb1[k]; g.b2[e] = pb2[k];
    // a pair that involves a sensor never generates constraints (narrow_phase/system_param.rs:583-599)
    const bool sensor = g.sensor && (g.sensor[pc1[k]] | g.sensor[pc2[k]]);
    g.pflags[e] = sensor ? uint8_t(pfl[k] & ~AVN_PAIR_GENERATE_CONSTRAINTS) : pfl[k];
    g.isl_event[e] = 0;
    g.fresh[e] = 1;
    g.live[e] = 1;            // a ContactId handed to a new pair starts without history
    g.count[e] = 0; g.prev_count[e] = 0; g.touching[e] = 0; g.colour[e] = 0; g.change[e] = 0; g.asleep[e] = 0;
}

// key 0 for rows that satisfy the predicate, 1 otherwise: one stable radix pass then lists them in ascending ContactId
__global__ void free_keys_kernel(const uint8_t* __restrict__ live, int n, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    keys[e] = live[e] ? 1u : 0u;
    vals[e] = uint32_t(e);
}

// the collision event of a row (GraphRows::event): the transition bit plus the pair's AVN_PAIR_* flags (bits 0-3), captured when the row changes
// (finalize_rows_kernel clears the flags of a removed row and the next step may hand its ContactId to a new pair)
enum { EV_STARTED = 0x40, EV_ENDED = 0x80, EV_FLAGS = 0x0f };

// the touching state machine of one row -> its change for the graphs
__global__ void classify_kernel(GraphRows g, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= g.hw) return;
    uint8_t ch = CH_NONE, ev = ISL_NONE, cev = 0;
    if (g.live[e] && !g.asleep[e]) {   // update_contacts runs over active_pairs only: a sleeping pair changes nothing
        const uint8_t pf = g.pflags[e];
        const bool gen = (pf & AVN_PAIR_GENERATE_CONSTRAINTS) != 0;
        if (g.disjoint[e]) {
            ch = CH_REMOVE | (g.colour[e] ? 0 : CH_DONE);
            atomicAdd(&g.ctr->removed, 1u);
            if (g.touching[e]) cev = EV_ENDED | pf;       // CollisionEnd (system_param.rs:155-170)
            if (gen && g.touching[e]) ev = ISL_REMOVE;    // PhysicsIslands::remove_contact (system_param.rs:196-205)
        } else {
            const bool now = g.count[e] > 0, was = g.touching[e] != 0;
            if (now && !was) {
                g.touching[e] = 1;
                atomicAdd(&g.ctr->started, 1u);
                cev = EV_STARTED | pf;                     // CollisionStart (system_param.rs:208-218)
                if (gen) { ch = CH_PUSH; ev = ISL_ADD; }   // add_contact (system_param.rs:244-258)
            } else if (!now && was) {
                g.touching[e] = 0;
                atomicAdd(&g.ctr->stopped, 1u);
                cev = EV_ENDED | pf;                       // CollisionEnd (system_param.rs:263-273)
                if (gen && g.colour[e]) ch = CH_POP;
                if (gen) ev = ISL_REMOVE;                  // remove_contact (system_param.rs:306-313)
            }
        }
    }
    g.isl_event[e] = ev;
    g.event[e] = cev;
    g.change[e] = ch;
    if (ch) atomicAdd(&g.ctr->changed, 1u);
    keys[e] = ch ? 0u : 1u;
    vals[e] = uint32_t(e);
}

__device__ __forceinline__ bool graph_static(const GraphRows& g, uint32_t b) { return b >= uint32_t(g.n_bodies) || g.body_kind[b] == AVN_BODY_STATIC; }

// is it this edge's turn on (non-static) body b?  A push needs to be the smallest pending edge of the body; a pop only needs every earlier
// pending PUSH of the body to be done (pops clear different bits and commute)
__device__ __forceinline__ bool graph_turn_body(const GraphRows& g, uint32_t b, unsigned long long key, bool push) {
    return push ? g.body_min[2 * size_t(b)] == key : g.body_min[2 * size_t(b) + 1] > key;
}
__device__ __forceinline__ bool graph_turn(const GraphRows& g, uint32_t b, unsigned long long key, bool push) {
    return graph_static(g, b) || graph_turn_body(g, b, key, push);
}

// ConstraintGraph::push_manifold / pop_manifold for ONE edge whose turn it is
__device__ __forceinline__ void graph_apply(const GraphRows& g, uint32_t e, uint8_t ch) {
    const uint32_t b1 = g.b1[e], b2 = g.b2[e];
    const bool s1 = graph_static(g, b1), s2 = graph_static(g, b2);
    if ((ch & CH_MASK) == CH_PUSH) {
        int c = AVN_COLOR_OVERFLOW;
        if (!s1 && !s2) {
            const uint32_t freec = ~(g.body_bits[b1] | g.body_bits[b2]) & ((1u << AVN_DYNAMIC_COLOR_COUNT) - 1u);
            if (freec) { c = __ffs(int(freec)) - 1; g.body_bits[b1] |= 1u << c; g.body_bits[b2] |= 1u << c; }
        } else if (!s1 || !s2) {
            const uint32_t b = s1 ? b2 : b1;
            const uint32_t freec = ~g.body_bits[b] & (((1u << AVN_COLOR_OVERFLOW) - 1u) & ~1u);   // colours OVERFLOW-1 .. 1, highest first
            if (freec) { c = 31 - __clz(int(freec)); g.body_bits[b] |= 1u << c; }
        }
        g.colour[e] = uint8_t(c + 1);
        if (c == AVN_COLOR_OVERFLOW) g.ctr->ovf_dirty = 1;
    } else {
        const int c = int(g.colour[e]) - 1;
        g.old_colour[e] = uint8_t(c + 1);
        if (c >= 0 && c != AVN_COLOR_OVERFLOW) {
            if (!s1) atomicAnd(&g.body_bits[b1], ~(1u << c));   // several pops of one body may run in the same round
            if (!s2) atomicAnd(&g.body_bits[b2], ~(1u << c));
        }
        if (c == AVN_COLOR_OVERFLOW) g.ctr->ovf_dirty = 1;
        g.colour[e] = 0;
    }
}

constexpr unsigned GRAPH_MAX_ROUNDS = 1u << 22;
__global__ void __launch_bounds__(256) colour_rounds_kernel(GraphRows g, const uint32_t* __restrict__ list, uint32_t skip_upto) {
    cg::grid_group grid = cg::this_grid();
    const uint32_t n = g.ctr->changed;
    if (n <= skip_upto) return;   // uniform: the cluster kernel took it (or nothing changed)
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
    unsigned round = 0;
    for (;; ++round) {
        const unsigned long long tag = (unsigned long long)(GRAPH_MAX_ROUNDS - round) << 32;   // later rounds compare smaller: no reset pass
        if (tid == 0) g.ctr->round_left[(round + 1) % 3] = 0;   // next round's counter: its last readers left before this round began
        for (uint32_t i = tid; i < n; i += nth) {
            const uint32_t e = list[i];
            const uint8_t ch = g.change[e];
            if (ch & CH_DONE) continue;
            const uint32_t b1 = g.b1[e], b2 = g.b2[e];
            const bool push = (ch & CH_MASK) == CH_PUSH;
            if (!graph_static(g, b1)) { atomicMin(&g.body_min[2 * size_t(b1)], tag | e); if (push) atomicMin(&g.body_min[2 * size_t(b1) + 1], tag | e); }
            if (!graph_static(g, b2)) { atomicMin(&g.body_min[2 * size_t(b2)], tag | e); if (push) atomicMin(&g.body_min[2 * size_t(b2) + 1], tag | e); }
        }
        grid.sync();
        uint32_t left = 0;
        for (uint32_t i = tid; i < n; i += nth) {
            const uint32_t e = list[i];
            const uint8_t ch = g.change[e];
            if (ch & CH_DONE) continue;
            const uint32_t b1 = g.b1[e], b2 = g.b2[e];
            const bool push = (ch & CH_MASK) == CH_PUSH;
            const bool mine = graph_turn(g, b1, tag | e, push) && graph_turn(g, b2, tag | e, push);
            if (mine) { graph_apply(g, e, ch); g.change[e] = ch | CH_DONE; }
            else ++left;
        }
        if (left) atomicAdd(&g.ctr->round_left[round % 3], left);
        grid.sync();
        if (*reinterpret_cast<volatile uint32_t*>(&g.ctr->round_left[round % 3]) == 0) break;
        if (round + 2 >= GRAPH_MAX_ROUNDS) { if (tid == 0) g.ctr->aborted = 1; break; }
    }
    if (tid == 0) g.ctr->rounds = round + 1;
}

// The same rounds for a SMALL number of changed edges (the steady state: a few thousand contacts start or stop touching per step) inside ONE
// thread-block cluster: 8 CTAs x 1024 threads, every thread keeps its (at most 4) edges in registers, the two barriers of a round are hardware
// cluster barriers instead of grid-wide ones, and "is anything left" is an OR through distributed shared memory.  A round costs the L2 round
// trips of its atomics and loads instead of two cooperative grid barriers on top of them.
constexpr int CL_BLOCKS = 8, CL_THREADS = 1024, CL_ITEMS = 4;
constexpr uint32_t CL_MAX = uint32_t(CL_BLOCKS) * CL_THREADS * CL_ITEMS;
__global__ void __launch_bounds__(CL_THREADS) colour_rounds_cluster_kernel(GraphRows g, const uint32_t* __restrict__ list) {
    cg::cluster_group cluster = cg::this_cluster();
    __shared__ uint32_t flags[2 * CL_BLOCKS];
    const uint32_t n = g.ctr->changed;
    if (n == 0 || n > CL_MAX) return;   // uniform: the grid-wide kernel takes the large case
    const uint32_t rank = cluster.block_rank();
    const uint32_t tid = rank * CL_THREADS + threadIdx.x, nth = uint32_t(CL_BLOCKS) * CL_THREADS;
    constexpr uint32_t NONE = 0xffffffffu;
    uint32_t e[CL_ITEMS], b1[CL_ITEMS], b2[CL_ITEMS];
    uint8_t ch[CL_ITEMS];
    bool pend[CL_ITEMS];
#pragma unroll
    for (int k = 0; k < CL_ITEMS; ++k) {
        const uint32_t i = tid + uint32_t(k) * nth;
        pend[k] = false; e[k] = 0; b1[k] = b2[k] = NONE; ch[k] = 0;
        if (i < n) {
            e[k] = list[i];
            ch[k] = g.change[e[k]];
            pend[k] = !(ch[k] & CH_DONE);
            if (pend[k]) {
                const uint32_t x = g.b1[e[k]], y = g.b2[e[k]];
                b1[k] = graph_static(g, x) ? NONE : x;
                b2[k] = graph_static(g, y) ? NONE : y;
            }
        }
    }
    uint32_t* flags0 = cluster.map_shared_rank(flags, 0);
    unsigned round = 0;
    for (;; ++round) {
        const unsigned long long tag = (unsigned long long)(GRAPH_MAX_ROUNDS - round) << 32;
#pragma unroll
        for (int k = 0; k < CL_ITEMS; ++k) {
            if (!pend[k]) continue;
            const bool push = (ch[k] & CH_MASK) == CH_PUSH;
            if (b1[k] != NONE) { atomicMin(&g.body_min[2 * size_t(b1[k])], tag | e[k]); if (push) atomicMin(&g.body_min[2 * size_t(b1[k]) + 1], tag | e[k]); }
            if (b2[k] != NONE) { atomicMin(&g.body_min[2 * size_t(b2[k])], tag | e[k]); if (push) atomicMin(&g.body_min[2 * size_t(b2[k]) + 1], tag | e[k]); }
        }
        cluster.sync();
        int left = 0;
#pragma unroll
        for (int k = 0; k < CL_ITEMS; ++k) {
            if (!pend[k]) continue;
            const bool push = (ch[k] & CH_MASK) == CH_PUSH;
            const bool mine = (b1[k] == NONE || graph_turn_body(g, b1[k], tag | e[k], push)) && (b2[k] == NONE || graph_turn_body(g, b2[k], tag | e[k], push));
            if (mine) { graph_apply(g, e[k], ch[k]); g.change[e[k]] = ch[k] | CH_DONE; pend[k] = false; }
            else left = 1;
        }
        const int any = __syncthreads_or(left);
        if (threadIdx.x == 0) flags0[(round & 1u) * CL_BLOCKS + rank] = uint32_t(any);
        cluster.sync();
        uint32_t rem = 0;
#pragma unroll
        for (int r = 0; r < CL_BLOCKS; ++r) rem |= flags0[(round & 1u) * CL_BLOCKS + r];
        if (!rem) break;
        if (round + 2 >= GRAPH_MAX_ROUNDS) { if (tid == 0) g.ctr->aborted = 1; break; }
    }
    cluster.sync();   // CTA 0's shared memory is read by the others until here
    if (tid == 0) g.ctr->rounds = round + 1;
}

// the overflow colour keeps the reference's list order (push at the end, swap_remove): one thread, changed edges in ascending ContactId
__global__ void overflow_list_kernel(GraphRows g, const uint32_t* __restrict__ list) {
    if (blockIdx.x || threadIdx.x || !g.ctr->ovf_dirty) return;
    uint32_t n_ovf = g.ctr->ovf_count;
    const uint32_t n = g.ctr->changed;
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t e = list[i];
        const uint8_t ch = g.change[e] & CH_MASK;
        if (ch == CH_PUSH) {
            if (g.colour[e] == AVN_COLOR_OVERFLOW + 1) { g.ovf[n_ovf] = e; g.ovf_pos[e] = n_ovf++; }
        } else if (g.old_colour[e] == AVN_COLOR_OVERFLOW + 1) {
            const uint32_t pos = g.ovf_pos[e], last = g.ovf[n_ovf - 1];
            g.ovf[pos] = last; g.ovf_pos[last] = pos; --n_ovf;
        }
    }
    g.ctr->ovf_count = n_ovf;
}

// rows that left the ContactGraph; and the radix key of every row for the colour-major list (255 = not in a coloured list)
__global__ void finalize_rows_kernel(GraphRows g, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= g.hw) return;
    const uint8_t ch = g.change[e];
    if ((ch & CH_MASK) == CH_REMOVE) {
        g.live[e] = 0; g.count[e] = 0; g.prev_count[e] = 0; g.touching[e] = 0; g.colour[e] = 0; g.pflags[e] = 0;
        if (g.asleep[e]) { g.asleep[e] = 0; atomicSub(&g.ctr->rows_asleep, 1u); }   // a freed ContactId never hands its sleep on
    }
    g.old_colour[e] = 0;
    const int c = int(g.colour[e]) - 1;
    keys[e] = (c >= 0 && c < AVN_COLOR_OVERFLOW) ? uint32_t(c) : 255u;
    vals[e] = uint32_t(e);
}

// colour offsets from the sorted keys; the overflow colour's list is appended behind the coloured part
__global__ void color_offsets_kernel(GraphRows g, const uint32_t* __restrict__ sorted_keys, uint32_t* __restrict__ edge_list) {
    __shared__ uint32_t off[AVN_GRAPH_COLOR_COUNT + 1];
    const int c = threadIdx.x;
    if (c < AVN_GRAPH_COLOR_COUNT) {   // lower bound of key c
        int lo = 0, hi = g.hw;
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (sorted_keys[mid] < uint32_t(c)) lo = mid + 1; else hi = mid; }
        off[c] = uint32_t(lo);
    }
    __syncthreads();
    const uint32_t n_ovf = g.ctr->ovf_count;
    if (c == 0) off[AVN_GRAPH_COLOR_COUNT] = off[AVN_COLOR_OVERFLOW] + n_ovf;
    __syncthreads();
    if (c <= AVN_GRAPH_COLOR_COUNT) g.ctr->color_offsets[c] = off[c];
    if (c == 0) g.ctr->manifolds = off[AVN_GRAPH_COLOR_COUNT];
    for (uint32_t k = threadIdx.x; k < n_ovf; k += blockDim.x) edge_list[off[AVN_COLOR_OVERFLOW] + k] = g.ovf[k];
}

// what prepare_contact_constraints needs per manifold besides the row: the bodies and the pair's material
template <class S>
__global__ void gather_graph_kernel(GraphRows g, const uint32_t* __restrict__ edge_list, const double* __restrict__ friction, const double* __restrict__ restitution,
                                    int32_t* __restrict__ m_b1, int32_t* __restrict__ m_b2, S* __restrict__ m_fr, S* __restrict__ m_re) {
    const uint32_t M = g.ctr->manifolds;
    for (uint32_t m = blockIdx.x * blockDim.x + threadIdx.x; m < M; m += gridDim.x * blockDim.x) {
        const uint32_t e = edge_list[m];
        m_b1[m] = int32_t(g.b1[e]);
        m_b2[m] = int32_t(g.b2[e]);
        const uint32_t ca = g.c1[e], cb = g.c2[e];
        const double fr = friction ? (friction[ca] + friction[cb]) * 0.5 : 0.5, re = restitution ? (restitution[ca] + restitution[cb]) * 0.5 : 0.0;
        m_fr[m] = S(fr);
        m_re[m] = S(re);
        if (S(re) != S(0)) g.ctr->any_restitution = 1;
    }
}

// ContactGraph::pair_set as the broad phase's "existing pairs" hash set, rebuilt from the live rows
__global__ void pair_set_kernel(GraphRows g, uint64_t* __restrict__ table, uint64_t mask) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= g.hw || !g.live[e]) return;
    const uint32_t a = g.c1[e], b = g.c2[e];
    const uint64_t k = (a < b ? (uint64_t(a) << 32) | b : (uint64_t(b) << 32) | a) + 1;
    uint64_t h = hash64(k) & mask;
    for (;;) {
        unsigned long long prev = atomicCAS((unsigned long long*)&table[h], 0ull, (unsigned long long)k);
        if (prev == 0ull || prev == k) return;
        h = (h + 1) & mask;
    }
}

// =====================================================================================================================================
// The contact pipeline's output to the application (DESIGN.md §7f): collision events, contact reports and the removal of colliders.
//   Events: classify_kernel leaves one byte per row (GraphRows::event); avn_contacts_events turns the bytes into the started and ended lists in
//     ascending ContactId with one stable radix pass (key 0 = started, 1 = ended, 2 = none) and a gather.
//   Removal (remove_collider, narrow_phase/mod.rs:399-459): every live row that names a removed collider is popped from its colour, unlinked from
//     its island, queued as a CollisionEnd when it was touching and freed; then the colour-major list and the pair set are rebuilt by the
//     step's own kernels.
//   Reports: the touching rows in ascending ContactId with their manifold reduced in slot order.
// =====================================================================================================================================
__global__ void event_keys_kernel(const uint8_t* __restrict__ event, int n, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const uint8_t v = event[e];
    keys[e] = (v & EV_STARTED) ? 0u : (v & EV_ENDED) ? 1u : 2u;
    vals[e] = uint32_t(e);
}
// key 0 = a touching row the report lists
__global__ void report_keys_kernel(GraphRows g, uint32_t flags, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= g.hw) return;
    const bool sel = g.live[e] && g.touching[e] && (!(flags & AVN_REPORT_EVENTS_ONLY) || (g.pflags[e] & AVN_PAIR_CONTACT_EVENTS));
    keys[e] = sel ? 0u : 1u;
    vals[e] = uint32_t(e);
}
// out[k - 1] = lower bound of key k in the sorted keys, k = 1 .. nb
__global__ void key_bounds_kernel(const uint32_t* __restrict__ sorted_keys, int n, int nb, uint32_t* __restrict__ out) {
    const int k = threadIdx.x + 1;
    if (k > nb) return;
    int lo = 0, hi = n;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (sorted_keys[mid] < uint32_t(k)) lo = mid + 1; else hi = mid; }
    out[k - 1] = uint32_t(lo);
}
// An event list in device memory, N entries as columns: u32 collider1[N], collider2[N], body1[N], body2[N], then u8 flags[N].
// Entry i < n_started of the sorted rows goes to slot i, the rest (the step's ended rows) behind the `skip` queued CollisionEnds.
__global__ void event_gather_kernel(GraphRows g, const uint32_t* __restrict__ list, uint32_t n_started, uint32_t n, uint32_t skip, uint32_t N,
                                    uint32_t* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t e = list[i], j = i < n_started ? i : i + skip;
    out[j] = g.c1[e]; out[N + j] = g.c2[e]; out[2 * size_t(N) + j] = g.b1[e]; out[3 * size_t(N) + j] = g.b2[e];
    reinterpret_cast<uint8_t*>(out + 4 * size_t(N))[j] = g.event[e] & EV_FLAGS;
}
__global__ void mark_colliders_kernel(const uint32_t* __restrict__ ids, uint32_t n, uint8_t* __restrict__ removed) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) removed[ids[k]] = 1;
}
// the CollisionEnds of the touching removed rows (the first n of the sorted list) appended to the pending list (layout of event_gather_kernel,
// capacity cap) behind its `base` entries
__global__ void queue_ends_kernel(GraphRows g, const uint32_t* __restrict__ list, uint32_t n, uint32_t base, uint32_t cap, uint32_t* __restrict__ pend) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t e = list[i], j = base + i;
    pend[j] = g.c1[e]; pend[cap + j] = g.c2[e]; pend[2 * size_t(cap) + j] = g.b1[e]; pend[3 * size_t(cap) + j] = g.b2[e];
    reinterpret_cast<uint8_t*>(pend + 4 * size_t(cap))[j] = g.pflags[e] & EV_FLAGS;
}
// One report entry per listed row, columns of n entries: S normal[n][3], total[n], max[n], penetration[n]; u32 contact_id[n], collider1[n],
// collider2[n], body1[n], body2[n]; u8 flags[n], point_count[n].  The points are reduced in slot order in S, so a sequential host loop in the
// same type gives the same bits.  Only a row in the ConstraintGraph, or asleep out of it, was solved: any other row (a sensor pair) reports 0 impulses.
template <class S>
__global__ void report_gather_kernel(GraphRows g, const uint32_t* __restrict__ list, uint32_t n, const S* __restrict__ normal, const S* __restrict__ pen,
                                     const S* __restrict__ nimp, void* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t e = list[i];
    S* os = static_cast<S*>(out);
    uint32_t* ou = reinterpret_cast<uint32_t*>(os + 6 * size_t(n));
    uint8_t* ob = reinterpret_cast<uint8_t*>(ou + 5 * size_t(n));
    const int cnt = g.count[e];
    const bool solved = g.colour[e] != 0 || g.asleep[e] != 0;   // an asleep row keeps the impulses of its last solve
    S total = S(0), mx = S(0), deep = S(0);
    for (int k = 0; k < cnt; ++k) {
        const S v = solved ? nimp[4 * size_t(e) + k] : S(0);
        total = total + v;
        if (v > mx) mx = v;
        const S p = pen[4 * size_t(e) + k];
        if (k == 0 || p >= deep) deep = p;
    }
    for (int c = 0; c < 3; ++c) os[3 * size_t(i) + c] = normal[3 * size_t(e) + c];
    os[3 * size_t(n) + i] = total; os[4 * size_t(n) + i] = mx; os[5 * size_t(n) + i] = deep;
    ou[i] = e; ou[n + i] = g.c1[e]; ou[2 * size_t(n) + i] = g.c2[e]; ou[3 * size_t(n) + i] = g.b1[e]; ou[4 * size_t(n) + i] = g.b2[e];
    ob[i] = g.pflags[e] & EV_FLAGS; ob[n + i] = uint8_t(cnt);
}

// capsules != 0: the shape column holds a capsule, and the rows that name one are left to narrow_capsule_edges_kernel; hulls != 0: the column
// holds a convex hull, and the rows that name one are left to narrow_hull_edges_kernel
template <class S>
__global__ void __launch_bounds__(128) narrow_edges_kernel(const __grid_constant__ NarrowEdgeArgs<S> a, uint8_t* fresh, int only_fresh, int capsules, int hulls) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.r.E) return;
    if (hulls && hull_row(a, e)) return;
    if (capsules && capsule_row(a, e)) return;
    if (only_fresh) {            // the rows added after the early pass over the existing rows (Contacts::prefetch_inputs)
        if (!fresh[e]) return;
        fresh[e] = 0;
    }
    narrow_edge_row<S, false>(a, e);   // csrc/contact_rows.hpp: the same function the CPU tests run
}

// the rows that name a capsule (launched after narrow_edges_kernel, on the same stream, only when the shape column holds a capsule)
template <class S>
__global__ void __launch_bounds__(128) narrow_capsule_edges_kernel(const __grid_constant__ NarrowEdgeArgs<S> a, uint8_t* fresh, int only_fresh, int hulls) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.r.E || !capsule_row(a, e)) return;
    if (hulls && hull_row(a, e)) return;
    if (only_fresh) {
        if (!fresh[e]) return;
        fresh[e] = 0;
    }
    narrow_edge_row<S, true>(a, e);
}

// with body frames (avn_contacts_set_body_frames) these two replace the pair above: the same rows, anchors relative to the centres of mass
template <class S, bool CAPSULES>
__global__ void __launch_bounds__(128) narrow_framed_edges_kernel(const __grid_constant__ NarrowEdgeArgs<S> a, const BodyFrameCols<S> f, uint8_t* fresh,
                                                                  int only_fresh, int capsules, int hulls) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.r.E) return;
    if (hulls && hull_row(a, e)) return;
    if (capsules && capsule_row(a, e) != CAPSULES) return;
    if (only_fresh) {
        if (!fresh[e]) return;
        fresh[e] = 0;
    }
    narrow_edge_row<S, CAPSULES, true>(a, e, f);
}

// the rows that name a convex hull (launched after the kernels above, on the same stream, only when the shape column holds a hull), with or
// without body frames
template <class S, bool FRAMES>
__global__ void __launch_bounds__(128) narrow_hull_edges_kernel(const __grid_constant__ NarrowEdgeArgs<S> a, const BodyFrameCols<S> f, uint8_t* fresh,
                                                                int only_fresh, const __grid_constant__ hm::Table t) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.r.E || !hull_row(a, e)) return;
    if (only_fresh) {
        if (!fresh[e]) return;
        fresh[e] = 0;
    }
    narrow_edge_row<S, true, FRAMES, true>(a, e, f, &t);
}


// =====================================================================================================================================
// Persistent simulation islands + sleeping (SURVEY.md 8f #4; dynamics/solver/islands/mod.rs, islands/sleeping.rs).
// An island is a tree of a lock-free union-find forest over the non-static bodies (root = smallest body index).  Merging is the classic
// CAS hook (every edge is processed once, in any order); the per-island state (constraints_removed, is_sleeping) lives at the root and moves
// to the new root when a root is hooked under another.  Nothing is rebuilt per step: islands only change when a linked contact comes (merge),
// goes (constraints_removed += 1) or when the split candidate is split (its bodies are reset to singletons and re-linked through the contacts
// and joints that are still there).
// =====================================================================================================================================
struct IslandCounters {
    uint32_t islands, sleeping, put_to_sleep, woken, split_bodies, merges, split_root;
    uint32_t absorbed;   // sleeping islands that were merged into another island (their bodies are awake with it, without a WakeIslands)
    unsigned long long cand;
};
constexpr uint32_t ISL_NONE_BODY = 0xffffffffu;

struct IslandState {
    int B;
    const uint8_t* kind;
    uint32_t* parent; uint32_t* root; uint32_t* root_prev; uint32_t* removed;
    uint8_t* isl_sleeping; uint8_t* awake; uint8_t* need_wake; uint8_t* touched; uint8_t* in_split;
    float* timer;
    const float* thr_lin; const float* thr_ang; const uint8_t* disabled; const uint8_t* host_wake;
    uint32_t* cand_body;
    IslandCounters* ctr;
    float time_to_sleep, delta_secs;
};
__device__ __forceinline__ bool isl_static(const IslandState& s, uint32_t b) { return b >= uint32_t(s.B) || s.kind[b] == AVN_BODY_STATIC; }
__device__ __forceinline__ uint32_t isl_find(uint32_t* parent, uint32_t x) {
    uint32_t p = *reinterpret_cast<volatile uint32_t*>(&parent[x]);
    while (p != x) {
        const uint32_t gp = *reinterpret_cast<volatile uint32_t*>(&parent[p]);
        if (gp != p) parent[x] = gp;   // path halving: any ancestor is a valid parent (roots only ever move under smaller roots)
        x = p; p = gp;
    }
    return x;
}
__device__ __forceinline__ bool isl_union(uint32_t* parent, uint32_t u, uint32_t v) {
    for (;;) {
        uint32_t ru = isl_find(parent, u), rv = isl_find(parent, v);
        if (ru == rv) return false;
        if (ru < rv) { const uint32_t t = ru; ru = rv; rv = t; }
        if (atomicCAS(&parent[ru], ru, rv) == ru) return true;   // the larger root goes under the smaller one
    }
}
__global__ void isl_init_kernel(IslandState s) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= s.B) return;
    s.parent[b] = uint32_t(b); s.root[b] = uint32_t(b); s.root_prev[b] = uint32_t(b); s.removed[b] = 0;
    s.isl_sleeping[b] = 0; s.awake[b] = 0; s.need_wake[b] = 0; s.touched[b] = 0; s.in_split[b] = 0; s.timer[b] = 0.f;
    if (b == 0) { *s.cand_body = ISL_NONE_BODY; }
}
// PhysicsIslands::add_joint at configuration time, and the joints of a split island
__global__ void isl_joint_kernel(IslandState s, const uint32_t* __restrict__ j1, const uint32_t* __restrict__ j2, int J, int only_split) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= J) return;
    const uint32_t a = j1[j], b = j2[j];
    if (isl_static(s, a) || isl_static(s, b)) return;
    if (only_split && !(s.in_split[a] && s.in_split[b])) return;
    isl_union(s.parent, a, b);
}
// configuration in the middle of a run: the contacts that are touching already link their bodies' islands (as if add_contact had seen them)
__global__ void isl_link_existing_kernel(IslandState s, GraphRows g) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= g.hw || !g.live[e] || !g.touching[e] || !(g.pflags[e] & AVN_PAIR_GENERATE_CONSTRAINTS)) return;
    const uint32_t a = g.b1[e], b = g.b2[e];
    if (!isl_static(s, a) && !isl_static(s, b)) isl_union(s.parent, a, b);
}
// add_contact: merge the islands of the two bodies (mod.rs:513-592); a contact that reaches a sleeping island wakes it (system_param.rs:253-258)
__global__ void isl_add_kernel(IslandState s, GraphRows g) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= g.hw || g.isl_event[e] != ISL_ADD) return;
    const uint32_t a = g.b1[e], b = g.b2[e];
    const bool sa = isl_static(s, a), sb = isl_static(s, b);
    if (!sa) s.touched[a] = 1;
    if (!sb) s.touched[b] = 1;
    if (!sa && !sb && isl_union(s.parent, a, b)) atomicAdd(&s.ctr->merges, 1u);
}
// after the merges: every body learns its root; a root that was hooked under another hands its island state over (merge_islands, mod.rs:965)
__global__ void isl_flatten_kernel(IslandState s, int split_only) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= s.B || isl_static(s, uint32_t(b))) return;
    if (split_only) {
        if (!s.in_split[b]) return;
        s.root[b] = isl_find(s.parent, uint32_t(b));
        s.removed[b] = 0;               // the islands that come out of a split start clean (split_island, mod.rs:995-1270)
        return;
    }
    const uint32_t r = isl_find(s.parent, uint32_t(b));
    s.root[b] = r;
    if (s.root_prev[b] == uint32_t(b) && r != uint32_t(b)) {
        if (s.removed[b]) { atomicAdd(&s.removed[r], s.removed[b]); s.removed[b] = 0; }
        if (s.isl_sleeping[b]) { s.isl_sleeping[b] = 0; s.need_wake[r] = 1; s.touched[b] = 1; atomicAdd(&s.ctr->absorbed, 1u); }
    }
}
__global__ void isl_wake_marks_kernel(IslandState s) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= s.B || isl_static(s, uint32_t(b))) return;
    if (s.touched[b] || (s.host_wake && s.host_wake[b])) s.need_wake[s.root[b]] = 1;
}
// remove_contact: constraints_removed += 1 on the island the contact was linked to (mod.rs:594-667)
__global__ void isl_remove_kernel(IslandState s, GraphRows g) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= g.hw || g.isl_event[e] != ISL_REMOVE) return;
    const uint32_t a = g.b1[e], b = g.b2[e];
    const uint32_t x = !isl_static(s, a) ? a : b;
    if (isl_static(s, x)) return;
    atomicAdd(&s.removed[s.root[x]], 1u);
}
// split_island (SolverSystems::Finalize): the island that holds last step's candidate, if it is awake and lost a constraint
__global__ void isl_split_pick_kernel(IslandState s) {
    if (blockIdx.x || threadIdx.x) return;
    uint32_t pick = ISL_NONE_BODY;
    const uint32_t c = *s.cand_body;
    if (c != ISL_NONE_BODY && !isl_static(s, c)) {
        const uint32_t r = s.root[c];
        if (!s.isl_sleeping[r] && s.removed[r] > 0) pick = r;
    }
    s.ctr->split_root = pick;
}
__global__ void isl_split_reset_kernel(IslandState s) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= s.B) return;
    const uint32_t R = s.ctr->split_root;
    const bool in = R != ISL_NONE_BODY && !isl_static(s, uint32_t(b)) && s.root[b] == R;
    s.in_split[b] = in ? 1 : 0;
    if (in) { s.parent[b] = uint32_t(b); atomicAdd(&s.ctr->split_bodies, 1u); }
}
__global__ void isl_split_link_kernel(IslandState s, GraphRows g) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= g.hw || s.ctr->split_root == ISL_NONE_BODY) return;
    if (!g.live[e] || !g.touching[e] || !(g.pflags[e] & AVN_PAIR_GENERATE_CONSTRAINTS)) return;
    const uint32_t a = g.b1[e], b = g.b2[e];
    if (isl_static(s, a) || isl_static(s, b) || !s.in_split[a] || !s.in_split[b]) return;
    isl_union(s.parent, a, b);
}
// every island is to wake (sleeping stops being applied)
__global__ void isl_mark_all_kernel(IslandState s, uint8_t mark) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < s.B && !isl_static(s, uint32_t(b))) s.need_wake[b] = mark;
}
// WakeIslands for the marked islands: timers back to zero (sleeping.rs WakeIslands::apply)
__global__ void isl_wake_bodies_kernel(IslandState s) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= s.B || isl_static(s, uint32_t(b))) return;
    const uint32_t r = s.root[b];
    if (s.need_wake[r] && s.isl_sleeping[r]) s.timer[b] = 0.f;
}
__global__ void isl_wake_roots_kernel(IslandState s) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= s.B || isl_static(s, uint32_t(b)) || s.root[b] != uint32_t(b)) return;
    if (s.need_wake[b] && s.isl_sleeping[b]) { s.isl_sleeping[b] = 0; atomicAdd(&s.ctr->woken, 1u); }
}
// update_sleeping_states + wake_islands_with_sleeping_disabled (sleeping.rs:164-246)
template <class S>
__global__ void isl_timers_kernel(IslandState s, const S* __restrict__ lv, const S* __restrict__ av, S length_unit_squared) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= s.B || isl_static(s, uint32_t(b))) return;
    const uint32_t r = s.root[b];
    if (s.isl_sleeping[r]) return;                       // Without<Sleeping>
    if (s.disabled && s.disabled[b]) { s.awake[r] = 1; s.timer[b] = 0.f; return; }
    const S lx = lv[3 * b], ly = lv[3 * b + 1], lz = lv[3 * b + 2], ax = av[3 * b], ay = av[3 * b + 1], az = av[3 * b + 2];
    const S lin2 = (lx * lx + ly * ly) + lz * lz, ang2 = (ax * ax + ay * ay) + az * az;
    const float tl = s.thr_lin ? s.thr_lin[b] : 0.15f, ta = s.thr_ang ? s.thr_ang[b] : 0.15f;
    const float tl2 = tl * fabsf(tl), ta2 = ta * fabsf(ta);   // keep signs
    float t = s.timer[b];
    if (lin2 < length_unit_squared * S(tl2) && ang2 < S(ta2)) t += s.delta_secs; else t = 0.f;
    s.timer[b] = t;
    if (t < s.time_to_sleep) {
        s.awake[r] = 1;
    } else if (s.removed[r] > 0) {
        // the sleepiest body that wants to sleep in an island that needs splitting; the first such body in index order on ties
        atomicMax(&s.ctr->cand, ((unsigned long long)__float_as_uint(t) << 32) | (unsigned long long)(0xffffffffu - uint32_t(b)));
    }
}
// sleep_islands (sleeping.rs:248-292)
__global__ void isl_decide_kernel(IslandState s) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= s.B || isl_static(s, uint32_t(b)) || s.root[b] != uint32_t(b)) return;
    atomicAdd(&s.ctr->islands, 1u);
    if (!s.awake[b] && !s.isl_sleeping[b] && s.removed[b] == 0) { s.isl_sleeping[b] = 1; atomicAdd(&s.ctr->put_to_sleep, 1u); }
    if (s.isl_sleeping[b]) atomicAdd(&s.ctr->sleeping, 1u);
}
__global__ void isl_finish_kernel(IslandState s, uint32_t* __restrict__ out_island, uint8_t* __restrict__ out_sleeping) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= s.B) return;
    const bool st = isl_static(s, uint32_t(b));
    const uint32_t r = st ? ISL_NONE_BODY : s.root[b];
    out_island[b] = r;
    out_sleeping[b] = (!st && s.isl_sleeping[r]) ? 1 : 0;
    s.root_prev[b] = st ? uint32_t(b) : r;
    s.awake[b] = 0; s.need_wake[b] = 0; s.touched[b] = 0; s.in_split[b] = 0;
    if (b == 0) {
        const unsigned long long c = s.ctr->cand;
        if (c != 0ull) *s.cand_body = 0xffffffffu - uint32_t(c & 0xffffffffull);   // otherwise the previous candidate stands (sleeping.rs:199)
    }
}

// pop_manifold for a row outside the colouring rounds (pops only clear bits, so one pass may do any number of them; the overflow colour's list
// is fixed afterwards by overflow_list_kernel, which reads old_colour)
__device__ __forceinline__ void graph_pop_now(const GraphRows& g, uint32_t e) {
    const uint32_t b1 = g.b1[e], b2 = g.b2[e];
    const int c = int(g.colour[e]) - 1;
    g.old_colour[e] = g.colour[e];
    if (c == AVN_COLOR_OVERFLOW) {
        g.ctr->ovf_dirty = 1;
    } else if (c >= 0) {
        if (!graph_static(g, b1)) atomicAnd(&g.body_bits[b1], ~(1u << c));
        if (!graph_static(g, b2)) atomicAnd(&g.body_bits[b2], ~(1u << c));
    }
    g.colour[e] = 0;
}

// remove_collider for every live row that names a removed collider: pop its manifold from its colour (pops only clear bits: one pass does them
// all; the overflow colour's list is fixed by overflow_list_kernel), remove_contact on its island when it was a touching, constraint-generating
// contact (islands: 0 = not configured, 1 = the last step's island events were applied, 2 = they are still pending: a contact that avn_islands_step
// has not linked yet is not unlinked either) and mark it CH_REMOVE for finalize_rows_kernel.
// keys: 0 = removed while touching (a CollisionEnd to queue), 1 = removed, 2 = kept.
__global__ void remove_rows_kernel(GraphRows g, const uint8_t* __restrict__ removed, IslandState s, int islands, uint32_t* __restrict__ keys,
                                   uint32_t* __restrict__ vals) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= g.hw) return;
    uint8_t ch = CH_NONE;
    uint32_t key = 2;
    if (g.live[e] && (removed[g.c1[e]] | removed[g.c2[e]])) {
        ch = CH_REMOVE;
        const bool touching = g.touching[e] != 0;
        key = touching ? 0u : 1u;
        atomicAdd(&g.ctr->removed, 1u);
        atomicAdd(&g.ctr->changed, 1u);
        if (touching) atomicAdd(&g.ctr->stopped, 1u);
        const uint32_t b1 = g.b1[e], b2 = g.b2[e];
        graph_pop_now(g, uint32_t(e));
        if (islands == 2 && g.isl_event[e] == ISL_ADD) {
            g.isl_event[e] = ISL_NONE;
        } else if (islands && touching && (g.pflags[e] & AVN_PAIR_GENERATE_CONSTRAINTS)) {
            const uint32_t x = !isl_static(s, b1) ? b1 : b2;
            if (!isl_static(s, x)) atomicAdd(&s.removed[s.root[x]], 1u);
        }
    }
    g.change[e] = ch;
    keys[e] = key;
    vals[e] = uint32_t(e);
}

// =====================================================================================================================================
// Applying sleeping and waking (SleepIslands::apply / WakeIslands::apply, sleeping.rs:354-533; ContactGraph::sleep_entity_with / wake_entity_with,
// contact_graph.rs:702-826).  isl_sleeping[root] is the DECISION, body_asleep[b] the APPLIED state; a pass brings the second in line with the first
// and moves the rows: a touching row sleeps with either endpoint, an asleep row wakes with either endpoint.
// =====================================================================================================================================
// body_asleep := the decision; fell[b] = the body fell asleep in this pass
__global__ void sleep_bodies_kernel(IslandState s, uint8_t* __restrict__ body_asleep, uint8_t* __restrict__ fell, GraphCounters* ctr) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= s.B) return;
    const uint8_t want = (!isl_static(s, uint32_t(b)) && s.isl_sleeping[s.root[b]]) ? 1 : 0;
    fell[b] = (want && !body_asleep[b]) ? 1 : 0;
    body_asleep[b] = want;
    if (want) atomicAdd(&ctr->bodies_asleep, 1u);
}
__device__ __forceinline__ bool row_body_flag(const GraphRows& g, uint32_t b, const uint8_t* __restrict__ flag) { return !graph_static(g, b) && flag[b]; }
// wake_entity_with: an asleep row with an awake (non-static) endpoint returns to the active pairs; a constraint-generating one is keyed as a push
// (key 0) for the colouring rounds, and its warm start is what its last solve left.
template <class S>
__global__ void wake_rows_kernel(GraphRows g, const uint8_t* __restrict__ body_asleep, S* __restrict__ ws_n_in, S* __restrict__ ws_t_in,
                                 const S* __restrict__ ws_n_out, const S* __restrict__ ws_t_out, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= g.hw) return;
    uint8_t ch = CH_NONE;
    if (g.live[e] && g.asleep[e]) {
        const uint32_t b1 = g.b1[e], b2 = g.b2[e];
        const bool awake = (!graph_static(g, b1) && !body_asleep[b1]) || (!graph_static(g, b2) && !body_asleep[b2]);
        if (awake) {
            g.asleep[e] = 0;
            atomicAdd(&g.ctr->rows_woken, 1u);
            atomicSub(&g.ctr->rows_asleep, 1u);
            if (g.pflags[e] & AVN_PAIR_GENERATE_CONSTRAINTS) {
                ch = CH_PUSH;
                atomicAdd(&g.ctr->changed, 1u);
                for (int k = 0; k < 4; ++k) ws_n_in[4 * size_t(e) + k] = ws_n_out[4 * size_t(e) + k];
                for (int k = 0; k < 8; ++k) ws_t_in[8 * size_t(e) + k] = ws_t_out[8 * size_t(e) + k];
            }
        }
    }
    g.change[e] = ch;
    keys[e] = ch ? 0u : 1u;
    vals[e] = uint32_t(e);
}
// sleep_entity_with: a touching, not yet sleeping row with an endpoint that just fell asleep leaves the active pairs; its manifold is popped here
// (key 0: the overflow colour's swap_removes follow in ascending ContactId).  No CH_REMOVE, no remove_contact, no event.
__global__ void sleep_rows_kernel(GraphRows g, const uint8_t* __restrict__ fell, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= g.hw) return;
    uint8_t ch = CH_NONE;
    if (g.live[e] && g.touching[e] && !g.asleep[e] && (row_body_flag(g, g.b1[e], fell) || row_body_flag(g, g.b2[e], fell))) {
        g.asleep[e] = 1;
        atomicAdd(&g.ctr->rows_slept, 1u);
        atomicAdd(&g.ctr->rows_asleep, 1u);
        if (g.colour[e]) {
            graph_pop_now(g, uint32_t(e));
            ch = CH_POP | CH_DONE;
            atomicAdd(&g.ctr->changed, 1u);
        }
    }
    g.change[e] = ch;
    keys[e] = ch ? 0u : 1u;
    vals[e] = uint32_t(e);
}

template <class S>
class Contacts final : public ContactsBase {
   public:
    Contacts(cudaStream_t stream, ErrorSink* err) : stream_(stream), err_(err) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, dev) == cudaSuccess) sm_count_ = prop.multiProcessorCount;
        cudaHostAlloc(&h_ctr_, sizeof(GraphCounters), cudaHostAllocDefault);
        up_stream_ = stream_;
        if (cudaStreamCreateWithFlags(&copy_stream_, cudaStreamNonBlocking) != cudaSuccess) { (void)cudaGetLastError(); copy_stream_ = nullptr; }
        cudaEventCreateWithFlags(&ev_in_, cudaEventDisableTiming);
        if (const char* c = getenv("AVN_GRAPH_CLUSTER")) use_cluster_ = atoi(c) != 0;
    }
    ~Contacts() override {
        if (h_ctr_) cudaFreeHost(h_ctr_);
        if (h_isl_) cudaFreeHost(h_isl_);
        if (ev_in_) cudaEventDestroy(ev_in_);
        if (copy_stream_) { cudaStreamSynchronize(copy_stream_); cudaStreamDestroy(copy_stream_); }
    }

    // ---- the graphs on the device ---------------------------------------------------------------------------------------------------
    AvnStatus configure(const AvnContactGraphConfig* cfg) override {
        if (!cfg || !cfg->body_kind) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "contacts_configure: config and body_kind are required");
        // the applied state is sized and kept for the configured bodies and rows: a reconfiguration starts from avn_islands_apply(ctx, 0)
        if (apply_) return err_->fail(AVN_ERR_UNSUPPORTED, "contacts_configure while sleeping is applied: call avn_islands_apply(ctx, 0) first");
        n_bodies_ = cfg->body_count;
        n_colliders_ = cfg->collider_count;
        AVN_CUDA(kind_.ensure(std::max<size_t>(n_bodies_, 1)));
        AVN_CUDA(cudaMemcpyAsync(kind_.p, cfg->body_kind, n_bodies_, cudaMemcpyHostToDevice, stream_));
        have_fr_ = cfg->friction != nullptr;
        have_re_ = cfg->restitution != nullptr;
        if (have_fr_) { AVN_CUDA(fr_.ensure(size_t(n_colliders_) * 8)); AVN_CUDA(cudaMemcpyAsync(fr_.p, cfg->friction, size_t(n_colliders_) * 8, cudaMemcpyHostToDevice, stream_)); }
        if (have_re_) { AVN_CUDA(re_.ensure(size_t(n_colliders_) * 8)); AVN_CUDA(cudaMemcpyAsync(re_.p, cfg->restitution, size_t(n_colliders_) * 8, cudaMemcpyHostToDevice, stream_)); }
        // the body sets of the colours and the round-tagged minima; a (re)configuration starts from an empty ConstraintGraph
        AVN_CUDA(body_bits_.ensure(std::max<size_t>(n_bodies_, 1) * 4));
        AVN_CUDA(body_min_.ensure(std::max<size_t>(n_bodies_, 1) * 16));
        AVN_CUDA(cudaMemsetAsync(body_bits_.p, 0, std::max<size_t>(n_bodies_, 1) * 4, stream_));
        AVN_CUDA(ctr_.ensure(sizeof(GraphCounters)));
        AVN_CUDA(cudaMemsetAsync(ctr_.p, 0, sizeof(GraphCounters), stream_));
        if (E_) {
            AVN_CUDA(cudaMemsetAsync(colour_.p, 0, E_, stream_));
            AVN_CUDA(cudaMemsetAsync(touching_.p, 0, E_, stream_));
            AVN_CUDA(cudaMemsetAsync(asleep_.p, 0, E_, stream_));
        }
        bodies_asleep_ = rows_asleep_ = 0;
        AVN_CUDA(cudaStreamSynchronize(stream_));   // the host arrays may be reused by the caller
        configured_ = true;
        graph_ = ResidentGraph{};
        sensor_h_.clear();                          // a (re)configuration starts without sensors
        return AVN_OK;
    }

    AvnStatus prefetch_inputs(const AvnNarrowParams* prm, const AvnNarrowInput* in, uint32_t match_contacts, double length_unit, uint32_t flags) override {
        prefetched_ = nullptr;
        early_rows_ = 0;
        if (!copy_stream_ || !in || !prm) return AVN_OK;
        // (the device copies were read by the previous step's narrow phase, which the previous step waited for)
        AvnStatus st = upload_inputs(in, (flags & AVN_CONTACTS_SHAPES_UNCHANGED) != 0, copy_stream_);
        if (st != AVN_OK) return st;
        // the rows that exist already do not depend on this step's broad phase: their geometry + matching starts now, on the copy stream, under
        // the broad-phase kernels; the rows the new pairs add are computed after them (narrow_edges_kernel, only_fresh)
        if (configured_ && hw_ > 0 && in->body_count <= n_bodies_ && in->collider_count <= n_colliders_) {
            if ((st = enqueue_narrow(prm, match_contacts, length_unit, hw_, copy_stream_, false)) != AVN_OK) return st;
            early_rows_ = hw_;
        }
        AVN_CUDA(cudaEventRecord(ev_in_, copy_stream_));
        prefetched_ = in;
        return AVN_OK;
    }

    AvnStatus step(const AvnNarrowParams* prm, const AvnNarrowInput* in, uint32_t match_contacts, double length_unit, const DevicePairs* np,
                   AvnContactStep* out) override {
        if (!prm || !in || !out) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "contacts_step: params, input and out are required");
        if (!configured_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_contacts_step before avn_contacts_configure");
        if (in->body_count > n_bodies_ || in->collider_count > n_colliders_)
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "contacts_step: %u bodies / %u colliders exceed the configured %u / %u", in->body_count, in->collider_count,
                              n_bodies_, n_colliders_);
        hull_generation_ = hulls_->generation;   // the table this step's hull kernels read (swept CCD checks it)
        const uint64_t n_new64 = np ? np->count : 0;
        if (n_new64 > 0x7fffffffull - hw_) return err_->fail(AVN_ERR_CAPACITY, "contacts_step: too many contact pairs");
        const uint32_t n_new = uint32_t(n_new64);
        added_this_step_ = n_new > 0;
        // the CollisionEnds queued by removals since the previous step are reported with this step's events; a new queue starts
        pend_cur_ ^= 1;
        pend_n_[pend_cur_] = 0;
        if (hw_ + n_new > E_ || E_ == 0) {
            if (prefetched_) AVN_CUDA(cudaStreamWaitEvent(stream_, ev_in_, 0));   // the early narrow pass writes the rows that are about to move
            AvnStatus st = reserve(std::max<uint32_t>(1024u, std::max(2 * E_, hw_ + n_new + 1024u)));
            if (st != AVN_OK) return st;
        }
        AVN_CUDA(cudaMemsetAsync(ctr_.p, 0, offsetof(GraphCounters, ovf_count), stream_));   // the per-step counters; ovf_count persists
        GraphRows g = graph_rows();
        const uint32_t added = n_new;
        if (n_new) {
            // ContactGraph::add_edge_and_key_with: lowest free ContactIds first, in list order
            const uint32_t n_free = hw_ - live_n_;
            const uint32_t* free_list = nullptr;
            if (n_free) {
                free_keys_kernel<<<(hw_ + 255) / 256, 256, 0, stream_>>>(live_.as<uint8_t>(), int(hw_), k0_.as<uint32_t>(), v0_.as<uint32_t>());
                radix_pass(int(hw_));
                free_list = v1_.as<uint32_t>();
            }
            if (prefetched_) AVN_CUDA(cudaStreamWaitEvent(stream_, ev_in_, 0));   // the early narrow pass visits the free rows too: it must be through with them
            add_rows_kernel<<<(n_new + 255) / 256, 256, 0, stream_>>>(g, n_new, np->c1, np->c2, np->b1, np->b2, np->flags, free_list, n_free, hw_, n_colliders_);
            AVN_CUDA(cudaGetLastError());
            if (n_new > n_free) hw_ += n_new - n_free;
            live_n_ += n_new;
            g.hw = int(hw_);
        }
        if (hw_) {
            AvnStatus st = launch_narrow(prm, in, match_contacts, length_unit, hw_);
            if (st != AVN_OK) return st;
            const unsigned rb = (hw_ + 255) / 256;
            classify_kernel<<<rb, 256, 0, stream_>>>(g, k0_.as<uint32_t>(), v0_.as<uint32_t>());
            radix_pass(int(hw_));
            AVN_CUDA(cudaMemcpyAsync(list_.p, v1_.p, size_t(hw_) * 4, cudaMemcpyDeviceToDevice, stream_));   // changed rows first, ascending ContactId
            if ((st = colour_changed(g)) != AVN_OK) return st;
            overflow_list_kernel<<<1, 32, 0, stream_>>>(g, list_.as<uint32_t>());
            rebuild_list(g);
            AVN_CUDA(cudaGetLastError());
        }
        AVN_CUDA(cudaMemcpyAsync(h_ctr_, ctr_.p, sizeof(GraphCounters), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        if (h_ctr_->aborted) return err_->fail(AVN_ERR_CUDA, "contacts_step: the colouring did not converge");
        live_n_ -= h_ctr_->removed;
        if (h_ctr_->bad_pairs) {
            live_n_ -= h_ctr_->bad_pairs;
            table_dirty_ = true;
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "contacts_step: %u new pair(s) name a collider >= %u or a body >= %u (avn_contacts_configure): not added",
                              h_ctr_->bad_pairs, n_colliders_, n_bodies_);
        }
        if (hw_ && (added || h_ctr_->removed || table_dirty_)) {   // ContactGraph::pair_set for the next broad phase
            AVN_CUDA(cudaMemsetAsync(table_.p, 0, (table_mask_ + 1) * sizeof(uint64_t), stream_));
            pair_set_kernel<<<(hw_ + 255) / 256, 256, 0, stream_>>>(g, table_.as<uint64_t>(), table_mask_);
            AVN_CUDA(cudaGetLastError());
            table_dirty_ = false;
        }
        *out = AvnContactStep{};
        out->rows_high_water = hw_; out->rows_live = live_n_; out->pairs_added = added; out->pairs_removed = h_ctr_->removed;
        out->started_touching = h_ctr_->started; out->stopped_touching = h_ctr_->stopped; out->manifold_count = h_ctr_->manifolds;
        out->colouring_rounds = h_ctr_->rounds; out->any_restitution = h_ctr_->any_restitution;
        memcpy(out->color_offsets, h_ctr_->color_offsets, sizeof out->color_offsets);
        graph_ = ResidentGraph{};
        graph_.count = h_ctr_->manifolds; graph_.any_restitution = h_ctr_->any_restitution;
        memcpy(graph_.color_offsets, h_ctr_->color_offsets, sizeof graph_.color_offsets);
        graph_.edge = v1_.as<uint32_t>(); graph_.body1 = m_b1_.as<int32_t>(); graph_.body2 = m_b2_.as<int32_t>(); graph_.friction = m_fr_.p; graph_.restitution = m_re_.p;
        stepped_ = true;
        isl_pending_ = true;
        wake_done_ = false;
        return AVN_OK;
    }

    // ---- collision events, sensors, removal of colliders, contact reports -----------------------------------------------------------
    AvnStatus set_sensors(uint32_t collider_count, const uint8_t* sensor) override {
        if (!configured_) return err_->fail(AVN_ERR_UNSUPPORTED, "contacts_set_sensors before avn_contacts_configure");
        if (collider_count != n_colliders_)
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "contacts_set_sensors: %u colliders, configured %u", collider_count, n_colliders_);
        std::vector<uint8_t> now(n_colliders_, 0);
        if (sensor) for (uint32_t c = 0; c < n_colliders_; ++c) now[c] = sensor[c] ? 1 : 0;
        std::vector<uint32_t> changed;   // On<Add, Sensor> / On<Remove, Sensor>: remove_collider for every collider whose flag changed
        for (uint32_t c = 0; c < n_colliders_; ++c)
            if (now[c] != (c < sensor_h_.size() ? sensor_h_[c] : 0)) changed.push_back(c);
        const bool any = std::find(now.begin(), now.end(), uint8_t(1)) != now.end();
        if (any) {
            AVN_CUDA(sensor_.ensure(n_colliders_));
            AVN_CUDA(cudaMemcpyAsync(sensor_.p, now.data(), n_colliders_, cudaMemcpyHostToDevice, stream_));
            AVN_CUDA(cudaStreamSynchronize(stream_));
        }
        sensor_h_ = any ? std::move(now) : std::vector<uint8_t>();   // no sensor: add_rows_kernel sees NULL, as before any call
        if (!stepped_ || changed.empty()) return AVN_OK;
        return remove_rows(uint32_t(changed.size()), changed.data());
    }

    AvnStatus remove_colliders(uint32_t n, const uint32_t* colliders) override {
        if (!stepped_) return err_->fail(AVN_ERR_UNSUPPORTED, "contacts_remove_colliders: no avn_contacts_step has run on this context");
        if (n && !colliders) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "contacts_remove_colliders: colliders are required");
        for (uint32_t k = 0; k < n; ++k)
            if (colliders[k] >= n_colliders_)
                return err_->fail(AVN_ERR_INVALID_ARGUMENT, "contacts_remove_colliders: collider %u >= the configured %u: nothing removed", colliders[k], n_colliders_);
        return remove_rows(n, colliders);
    }

    AvnStatus events(AvnCollisionEvents* started, AvnCollisionEvents* ended) override {
        if (!stepped_) return err_->fail(AVN_ERR_UNSUPPORTED, "contacts_events: no avn_contacts_step has run on this context");
        const int rep = pend_cur_ ^ 1;
        const uint32_t n_pend = pend_n_[rep];
        uint32_t bounds[2] = {0, 0};
        if (hw_) {
            event_keys_kernel<<<(hw_ + 255) / 256, 256, 0, stream_>>>(event_.as<uint8_t>(), int(hw_), k0_.as<uint32_t>(), v0_.as<uint32_t>());
            radix_pass(int(hw_), evl_.as<uint32_t>());   // started rows, then ended rows, each in ascending ContactId
            const AvnStatus st = small_bounds(2, bounds);
            if (st != AVN_OK) return st;
        }
        const uint32_t n_s = bounds[0], n_e = bounds[1] - bounds[0];
        const bool short_s = started && started->capacity < n_s, short_e = ended && ended->capacity < uint64_t(n_pend) + n_e;
        if (started) started->count = n_s;
        if (ended) ended->count = uint64_t(n_pend) + n_e;
        if (short_s || short_e)
            return err_->fail(AVN_ERR_CAPACITY, "contacts_events: %u started / %u ended events exceed the capacities", n_s, n_pend + n_e);
        const uint32_t N = n_s + n_pend + n_e;
        if (N == 0) return AVN_OK;
        AVN_CUDA(evout_.ensure(size_t(N) * 17));
        uint32_t* o = evout_.as<uint32_t>();
        if (n_s + n_e)
            event_gather_kernel<<<(n_s + n_e + 255) / 256, 256, 0, stream_>>>(graph_rows(), evl_.as<uint32_t>(), n_s, n_s + n_e, n_pend, N, o);
        AVN_CUDA(cudaGetLastError());
        if (n_pend) {   // the queued CollisionEnds of the removals, in call order, head the ended list
            const uint32_t* p = pend_[rep].as<uint32_t>();
            const size_t cap = pend_cap_[rep];
            for (int c = 0; c < 4; ++c)
                AVN_CUDA(cudaMemcpyAsync(o + size_t(c) * N + n_s, p + c * cap, size_t(n_pend) * 4, cudaMemcpyDeviceToDevice, stream_));
            AVN_CUDA(cudaMemcpyAsync(reinterpret_cast<uint8_t*>(o + 4 * size_t(N)) + n_s, reinterpret_cast<const uint8_t*>(p + 4 * cap), n_pend,
                                     cudaMemcpyDeviceToDevice, stream_));
        }
        struct { AvnCollisionEvents* list; uint32_t first, count; } parts[2] = {{started, 0, n_s}, {ended, n_s, n_pend + n_e}};
        for (auto& part : parts) {
            if (!part.list || !part.count) continue;
            uint32_t* cols[4] = {part.list->collider1, part.list->collider2, part.list->body1, part.list->body2};
            for (int c = 0; c < 4; ++c)
                if (cols[c]) AVN_CUDA(cudaMemcpyAsync(cols[c], o + size_t(c) * N + part.first, size_t(part.count) * 4, cudaMemcpyDeviceToHost, stream_));
            if (part.list->flags)
                AVN_CUDA(cudaMemcpyAsync(part.list->flags, reinterpret_cast<uint8_t*>(o + 4 * size_t(N)) + part.first, part.count, cudaMemcpyDeviceToHost, stream_));
        }
        AVN_CUDA(cudaStreamSynchronize(stream_));
        return AVN_OK;
    }

    AvnStatus report(uint32_t flags, AvnContactReport* out) override {
        if (!out) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "contacts_report: out is required");
        if (!stepped_) return err_->fail(AVN_ERR_UNSUPPORTED, "contacts_report: no avn_contacts_step has run on this context");
        uint32_t n = 0;
        GraphRows g = graph_rows();
        if (hw_) {
            report_keys_kernel<<<(hw_ + 255) / 256, 256, 0, stream_>>>(g, flags, k0_.as<uint32_t>(), v0_.as<uint32_t>());
            radix_pass(int(hw_), evl_.as<uint32_t>());   // the listed rows first, in ascending ContactId
            const AvnStatus st = small_bounds(1, &n);
            if (st != AVN_OK) return st;
        }
        const bool fits = out->capacity >= n;
        out->count = n;
        if (!fits) return err_->fail(AVN_ERR_CAPACITY, "contacts_report: %u touching pairs exceed the capacity %llu", n, (unsigned long long)out->capacity);
        if (n == 0) return AVN_OK;
        const size_t S_ = sizeof(S);
        AVN_CUDA(repout_.ensure(size_t(n) * (6 * S_ + 22)));
        report_gather_kernel<S><<<(n + 255) / 256, 256, 0, stream_>>>(g, evl_.as<uint32_t>(), n, normal_.as<S>(), pen_.as<S>(), nimp_out_.as<S>(), repout_.p);
        AVN_CUDA(cudaGetLastError());
        const char* r = repout_.as<char>();
        const char* u = r + 6 * S_ * n;
        const char* b = u + 20 * size_t(n);
        struct { void* dst; const char* src; size_t bytes; } cols[] = {
            {out->normal, r, 3 * S_ * n}, {out->total_normal_impulse, r + 3 * S_ * n, S_ * n}, {out->max_normal_impulse, r + 4 * S_ * n, S_ * n},
            {out->max_penetration, r + 5 * S_ * n, S_ * n}, {out->contact_id, u, 4 * size_t(n)}, {out->collider1, u + 4 * size_t(n), 4 * size_t(n)},
            {out->collider2, u + 8 * size_t(n), 4 * size_t(n)}, {out->body1, u + 12 * size_t(n), 4 * size_t(n)}, {out->body2, u + 16 * size_t(n), 4 * size_t(n)},
            {out->flags, b, n}, {out->point_count, b + n, n}};
        for (auto& c : cols)
            if (c.dst) AVN_CUDA(cudaMemcpyAsync(c.dst, c.src, c.bytes, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        return AVN_OK;
    }

    AvnStatus graph_view(ResidentGraph* out) override { *out = graph_; return AVN_OK; }
    void ccd_rows(CcdRows* out) override {
        out->rows = std::min(hw_, E_);
        out->bodies = configured_ ? n_bodies_ : 0;
        out->colliders = configured_ ? n_colliders_ : 0;
        out->c1 = c1_.as<uint32_t>(); out->c2 = c2_.as<uint32_t>(); out->b1 = b1_.as<uint32_t>(); out->b2 = b2_.as<uint32_t>(); out->live = live_.as<uint8_t>();
        out->shape = in_.shape;
        out->dims = in_.dims;
        out->has_capsule = has_capsule_;
        out->has_hull = has_hull_;
        out->hull_generation = hull_generation_;
    }
    void attach_hulls(const HullTable* hulls) override { hulls_ = hulls; }
    bool has_hull() const override { return has_hull_; }
    AvnStatus check_shapes(const AvnNarrowInput* in, uint32_t flags) override {
        if (!in || !in->dims) return AVN_OK;   // step() reports the missing columns
        checked_ = nullptr;
        const uint32_t hull_count = hulls_->count();
        if ((flags & AVN_CONTACTS_SHAPES_UNCHANGED) && in_.colliders == in->collider_count && in_.dims) {   // the column is not copied
            if (has_hull_ && max_hull_ >= hull_count)   // the table changed under the kept column
                return err_->fail(AVN_ERR_INVALID_ARGUMENT, "contacts_step: the kept shape column names convex hull %u, the hull table holds %u", max_hull_,
                                  hull_count);
            return AVN_OK;
        }
        size_t at = 0;
        bool capsule = false, hull = false;
        uint32_t max_hull = 0;
        if (const char* why = check_shape_column(in->shape, in->dims, in->collider_count, sizeof(S) == 8 ? 64 : 32, &at, &capsule, &hull_count, &hull, &max_hull))
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "contacts_step: collider %zu: %s", at, why);
        checked_ = in;                  // upload_inputs commits has_capsule_ / has_hull_ once this column is on the device
        checked_capsule_ = capsule;
        checked_hull_ = hull;
        checked_max_hull_ = max_hull;
        return AVN_OK;
    }
    bool has_capsule() const override { return has_capsule_; }
    AvnStatus set_body_frames(const AvnBodyFrames* f) override {
        if (!f) { frames_set_ = false; return AVN_OK; }
        if (!f->position || !f->rotation)
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "contacts_set_body_frames: position and rotation are required");
        const size_t B = f->body_count;
        frames_.body_count = f->body_count;
        auto copy = [&](std::vector<unsigned char>& dst, const void* src, size_t n) {
            dst.resize(src ? n * sizeof(S) : 0);
            if (src && n) memcpy(dst.data(), src, n * sizeof(S));
        };
        copy(frames_.position, f->position, 3 * B);
        copy(frames_.rotation, f->rotation, 4 * B);
        copy(frames_.com, f->center_of_mass, 3 * B);
        frames_set_ = true;
        return AVN_OK;
    }
    const BodyFrames* body_frames() const override { return frames_set_ ? &frames_ : nullptr; }
    void pair_set(const uint64_t** table, uint64_t* mask) override {
        *table = (configured_ && table_.p && !table_dirty_) ? table_.as<uint64_t>() : nullptr;
        *mask = table_mask_;
    }
    AvnStatus download_graph(uint32_t capacity, uint32_t* c1, uint32_t* c2, uint8_t* live, uint8_t* touching, int8_t* colour, uint32_t* edge_list) override {
        const size_t n = std::min(capacity, E_);
        if (n) {
            if (c1) AVN_CUDA(cudaMemcpyAsync(c1, c1_.p, n * 4, cudaMemcpyDeviceToHost, stream_));
            if (c2) AVN_CUDA(cudaMemcpyAsync(c2, c2_.p, n * 4, cudaMemcpyDeviceToHost, stream_));
            if (live) AVN_CUDA(cudaMemcpyAsync(live, live_.p, n, cudaMemcpyDeviceToHost, stream_));
            if (touching) AVN_CUDA(cudaMemcpyAsync(touching, touching_.p, n, cudaMemcpyDeviceToHost, stream_));
            if (colour) AVN_CUDA(cudaMemcpyAsync(colour, colour_.p, n, cudaMemcpyDeviceToHost, stream_));
        }
        if (edge_list && graph_.count) AVN_CUDA(cudaMemcpyAsync(edge_list, graph_.edge, size_t(graph_.count) * 4, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        if (colour) for (size_t e = 0; e < n; ++e) colour[e] = int8_t(int(uint8_t(colour[e])) - 1);   // stored + 1 (0 = none)
        return AVN_OK;
    }

    void view(RowColumns* out) override {
        out->rows = E_;
        out->point_count = count_.as<uint8_t>();
        out->normal = normal_.p; out->anchor1 = a1_.p; out->anchor2 = a2_.p; out->penetration = pen_.p; out->normal_speed = ns_.p;
        out->warm_start_normal_impulse = ws_n_in_.p;
        out->warm_start_tangent_impulse = ws_t_in_.p;
        out->normal_impulse = nimp_in_.p;
    }
    void outputs(void** ws_n, void** ws_t, void** nimp) override { *ws_n = ws_n_out_.p; *ws_t = ws_t_out_.p; *nimp = nimp_out_.p; }

    AvnStatus download_impulses(uint32_t capacity, void* ws_n, void* ws_t, void* nimp) override {   // tests / tools: the solver's outputs per row
        const size_t n = std::min(capacity, E_);
        if (n) {
            if (ws_n) AVN_CUDA(cudaMemcpyAsync(ws_n, ws_n_out_.p, n * 4 * sizeof(S), cudaMemcpyDeviceToHost, stream_));
            if (ws_t) AVN_CUDA(cudaMemcpyAsync(ws_t, ws_t_out_.p, n * 8 * sizeof(S), cudaMemcpyDeviceToHost, stream_));
            if (nimp) AVN_CUDA(cudaMemcpyAsync(nimp, nimp_out_.p, n * 4 * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        }
        AVN_CUDA(cudaStreamSynchronize(stream_));
        return AVN_OK;
    }

    // ---- islands + sleeping -------------------------------------------------------------------------------------------------------
    AvnStatus islands_configure(const AvnIslandsConfig* cfg) override {
        if (!cfg || !cfg->body_kind) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "islands_configure: config and body_kind are required");
        if (cfg->joint_count && (!cfg->joint_body1 || !cfg->joint_body2)) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "islands_configure: joint bodies are required");
        if (apply_) return err_->fail(AVN_ERR_UNSUPPORTED, "islands_configure while sleeping is applied: call avn_islands_apply(ctx, 0) first");
        const size_t B = cfg->body_count, Bp = std::max<size_t>(B, 1);
        // one allocation, every array 16-byte aligned
        auto up16 = [](size_t x) { return (x + 15) & ~size_t(15); };
        AVN_CUDA(isl_buf_.ensure(7 * up16(Bp * 4) + 7 * up16(Bp) + 64 + up16(sizeof(IslandCounters)) + 256));
        char* p = isl_buf_.as<char>();
        auto take = [&](size_t bytes) { char* q = p; p += up16(bytes); return q; };
        IslandState s{};
        s.B = int(B);
        s.ctr = reinterpret_cast<IslandCounters*>(take(sizeof(IslandCounters)));
        s.cand_body = reinterpret_cast<uint32_t*>(take(16));
        s.parent = reinterpret_cast<uint32_t*>(take(Bp * 4));
        s.root = reinterpret_cast<uint32_t*>(take(Bp * 4));
        s.root_prev = reinterpret_cast<uint32_t*>(take(Bp * 4));
        s.removed = reinterpret_cast<uint32_t*>(take(Bp * 4));
        s.timer = reinterpret_cast<float*>(take(Bp * 4));
        float* thr_lin = reinterpret_cast<float*>(take(Bp * 4));
        float* thr_ang = reinterpret_cast<float*>(take(Bp * 4));
        uint8_t* kind = reinterpret_cast<uint8_t*>(take(Bp));
        s.isl_sleeping = reinterpret_cast<uint8_t*>(take(Bp));
        s.awake = reinterpret_cast<uint8_t*>(take(Bp));
        s.need_wake = reinterpret_cast<uint8_t*>(take(Bp));
        s.touched = reinterpret_cast<uint8_t*>(take(Bp));
        s.in_split = reinterpret_cast<uint8_t*>(take(Bp));
        uint8_t* disabled = reinterpret_cast<uint8_t*>(take(Bp));
        s.kind = kind;
        AVN_CUDA(cudaMemcpyAsync(kind, cfg->body_kind, B, cudaMemcpyHostToDevice, stream_));
        isl_has_thr_lin_ = cfg->sleep_threshold_linear != nullptr; isl_has_thr_ang_ = cfg->sleep_threshold_angular != nullptr;
        isl_has_disabled_ = cfg->sleeping_disabled != nullptr;
        if (isl_has_thr_lin_) AVN_CUDA(cudaMemcpyAsync(thr_lin, cfg->sleep_threshold_linear, B * 4, cudaMemcpyHostToDevice, stream_));
        if (isl_has_thr_ang_) AVN_CUDA(cudaMemcpyAsync(thr_ang, cfg->sleep_threshold_angular, B * 4, cudaMemcpyHostToDevice, stream_));
        if (isl_has_disabled_) AVN_CUDA(cudaMemcpyAsync(disabled, cfg->sleeping_disabled, B, cudaMemcpyHostToDevice, stream_));
        s.thr_lin = isl_has_thr_lin_ ? thr_lin : nullptr; s.thr_ang = isl_has_thr_ang_ ? thr_ang : nullptr; s.disabled = isl_has_disabled_ ? disabled : nullptr;
        s.time_to_sleep = cfg->time_to_sleep > 0.f ? cfg->time_to_sleep : 0.5f;
        isl_length_unit_ = cfg->length_unit > 0.f ? cfg->length_unit : 1.f;
        AVN_CUDA(cudaMemsetAsync(s.ctr, 0, sizeof(IslandCounters), stream_));
        isl_ = s;
        isl_B_ = uint32_t(B);
        isl_J_ = cfg->joint_count;
        if (B) isl_init_kernel<<<unsigned((B + 255) / 256), 256, 0, stream_>>>(isl_);
        bool linked = false;
        if (isl_J_) {   // joints link their bodies' islands from the start (PhysicsIslands::add_joint, mod.rs:669-747)
            AVN_CUDA(isl_j_.ensure(size_t(isl_J_) * 8));
            AVN_CUDA(cudaMemcpyAsync(isl_j_.p, cfg->joint_body1, size_t(isl_J_) * 4, cudaMemcpyHostToDevice, stream_));
            AVN_CUDA(cudaMemcpyAsync(isl_j_.as<uint32_t>() + isl_J_, cfg->joint_body2, size_t(isl_J_) * 4, cudaMemcpyHostToDevice, stream_));
            isl_joint_kernel<<<(isl_J_ + 255) / 256, 256, 0, stream_>>>(isl_, isl_j_.as<uint32_t>(), isl_j_.as<uint32_t>() + isl_J_, int(isl_J_), 0);
            linked = true;
        }
        if (B && configured_ && hw_ > 0 && n_bodies_ <= isl_B_) {   // contacts that are touching already (configuration in the middle of a run)
            GraphRows g = graph_rows();
            isl_link_existing_kernel<<<(hw_ + 255) / 256, 256, 0, stream_>>>(isl_, g);
            linked = true;
        }
        if (linked && B) {
            isl_flatten_kernel<<<unsigned((B + 255) / 256), 256, 0, stream_>>>(isl_, 0);   // (root_prev == the body itself: nothing is handed over)
            AVN_CUDA(cudaMemcpyAsync(isl_.root_prev, isl_.root, B * 4, cudaMemcpyDeviceToDevice, stream_));
        }
        AVN_CUDA(cudaGetLastError());
        if (!h_isl_) AVN_CUDA(cudaHostAlloc(&h_isl_, sizeof(IslandCounters), cudaHostAllocDefault));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        isl_configured_ = true;
        return AVN_OK;
    }

    AvnStatus islands_step(AvnIslandsStep* st) override {
        if (!st || !st->linear_velocity || !st->angular_velocity) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "islands_step: step and the velocity columns are required");
        if (!isl_configured_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_islands_step before avn_islands_configure");
        const size_t B = isl_B_;
        if (B == 0) return AVN_OK;
        AVN_CUDA(isl_in_.ensure(2 * 3 * B * sizeof(S) + B));
        S* lv = isl_in_.as<S>(); S* av = lv + 3 * B;
        uint8_t* wake = reinterpret_cast<uint8_t*>(av + 3 * B);
        AVN_CUDA(cudaMemcpyAsync(lv, st->linear_velocity, 3 * B * sizeof(S), cudaMemcpyHostToDevice, stream_));
        AVN_CUDA(cudaMemcpyAsync(av, st->angular_velocity, 3 * B * sizeof(S), cudaMemcpyHostToDevice, stream_));
        if (st->wake) AVN_CUDA(cudaMemcpyAsync(wake, st->wake, B, cudaMemcpyHostToDevice, stream_));
        AVN_CUDA(isl_out_.ensure(B * 4 + B));
        uint32_t* out_island = isl_out_.as<uint32_t>();
        uint8_t* out_sleeping = reinterpret_cast<uint8_t*>(out_island + B);
        IslandState s = isl_;
        s.host_wake = st->wake ? wake : nullptr;
        s.delta_secs = st->delta_secs;
        AVN_CUDA(cudaMemsetAsync(s.ctr, 0, sizeof(IslandCounters), stream_));
        const unsigned bb = unsigned((B + 255) / 256);
        GraphRows g = graph_rows();
        const unsigned rb = g.hw > 0 ? unsigned((g.hw + 255) / 256) : 0;
        // narrow-phase part: contacts that came (merge) and went (constraints_removed), islands reached by a new contact wake up
        // (avn_islands_wake has linked this step's contacts already when sleeping is applied; the marks of the `wake` column are still to do)
        const bool linked = apply_ && wake_done_ && isl_pending_;
        if (!linked) {
            if (rb) isl_add_kernel<<<rb, 256, 0, stream_>>>(s, g);
            isl_flatten_kernel<<<bb, 256, 0, stream_>>>(s, 0);
        }
        isl_wake_marks_kernel<<<bb, 256, 0, stream_>>>(s);
        if (rb) isl_remove_kernel<<<rb, 256, 0, stream_>>>(s, g);
        // WakeIslands queued by the narrow phase are applied before the solver runs
        isl_wake_bodies_kernel<<<bb, 256, 0, stream_>>>(s);
        isl_wake_roots_kernel<<<bb, 256, 0, stream_>>>(s);
        // SolverSystems::Finalize: split last step's candidate
        isl_split_pick_kernel<<<1, 32, 0, stream_>>>(s);
        isl_split_reset_kernel<<<bb, 256, 0, stream_>>>(s);
        if (rb) isl_split_link_kernel<<<rb, 256, 0, stream_>>>(s, g);
        if (isl_J_) isl_joint_kernel<<<(isl_J_ + 255) / 256, 256, 0, stream_>>>(s, isl_j_.as<uint32_t>(), isl_j_.as<uint32_t>() + isl_J_, int(isl_J_), 1);
        isl_flatten_kernel<<<bb, 256, 0, stream_>>>(s, 1);
        // PhysicsStepSystems::Sleeping
        isl_timers_kernel<S><<<bb, 256, 0, stream_>>>(s, lv, av, S(isl_length_unit_) * S(isl_length_unit_));
        isl_decide_kernel<<<bb, 256, 0, stream_>>>(s);
        isl_finish_kernel<<<bb, 256, 0, stream_>>>(s, out_island, out_sleeping);
        AVN_CUDA(cudaGetLastError());
        AVN_CUDA(cudaMemcpyAsync(h_isl_, s.ctr, sizeof(IslandCounters), cudaMemcpyDeviceToHost, stream_));
        if (st->island) AVN_CUDA(cudaMemcpyAsync(st->island, out_island, B * 4, cudaMemcpyDeviceToHost, stream_));
        if (st->sleeping) AVN_CUDA(cudaMemcpyAsync(st->sleeping, out_sleeping, B, cudaMemcpyDeviceToHost, stream_));
        if (st->sleep_timer) AVN_CUDA(cudaMemcpyAsync(st->sleep_timer, s.timer, B * 4, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        st->island_count = h_isl_->islands; st->sleeping_islands = h_isl_->sleeping; st->islands_put_to_sleep = h_isl_->put_to_sleep;
        st->islands_woken = h_isl_->woken; st->split_bodies = h_isl_->split_bodies; st->merges = h_isl_->merges;
        isl_pending_ = false;
        if (apply_) {
            // SleepIslands for the islands put to sleep, WakeIslands for the ones the `wake` column woke after the solve: awake from the next step on
            const bool wakes = h_isl_->woken > 0 || h_isl_->absorbed > 0, sleeps = h_isl_->put_to_sleep > 0;
            if (linked) { st->islands_woken += wake_woken_; st->merges += wake_merges_; }
            wake_woken_ = wake_merges_ = 0;
            if (wakes || sleeps) return apply_pass(wakes, sleeps);
        }
        return AVN_OK;
    }

    // ---- applied sleeping ---------------------------------------------------------------------------------------------------------------
    AvnStatus islands_apply(uint32_t enable) override {
        if (!enable) {
            if (!apply_) return AVN_OK;
            if (isl_pending_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "islands_apply(0) between avn_contacts_step and avn_islands_step: finish the step first");
            if (bodies_asleep_) {   // wake everything first: WakeIslands for every island, then the rows return
                const unsigned bb = unsigned((size_t(isl_B_) + 255) / 256);
                AVN_CUDA(cudaMemsetAsync(isl_.ctr, 0, sizeof(IslandCounters), stream_));
                isl_mark_all_kernel<<<bb, 256, 0, stream_>>>(isl_, 1);
                isl_wake_bodies_kernel<<<bb, 256, 0, stream_>>>(isl_);
                isl_wake_roots_kernel<<<bb, 256, 0, stream_>>>(isl_);
                isl_mark_all_kernel<<<bb, 256, 0, stream_>>>(isl_, 0);
                const AvnStatus st = apply_pass(true, false);
                if (st != AVN_OK) return st;
            }
            apply_ = false;
            wake_done_ = false;
            return AVN_OK;
        }
        if (!isl_configured_ || !configured_) return err_->fail(AVN_ERR_UNSUPPORTED, "islands_apply before avn_contacts_configure and avn_islands_configure");
        if (isl_B_ != n_bodies_)
            return err_->fail(AVN_ERR_UNSUPPORTED, "islands_apply: avn_islands_configure has %u bodies, avn_contacts_configure %u", isl_B_, n_bodies_);
        if (apply_) return AVN_OK;
        const size_t Bp = std::max<size_t>(n_bodies_, 1);
        AVN_CUDA(body_asleep_.ensure(2 * Bp));
        AVN_CUDA(cudaMemsetAsync(body_asleep_.p, 0, 2 * Bp, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        bodies_asleep_ = 0;
        wake_woken_ = wake_merges_ = 0;
        apply_ = true;
        return AVN_OK;
    }

    AvnStatus islands_wake(const uint8_t* wake, AvnIslandsWake* out) override {
        if (!out) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "islands_wake: out is required");
        if (!apply_) return err_->fail(AVN_ERR_UNSUPPORTED, "avn_islands_wake while sleeping is not applied (avn_islands_apply)");
        if (!stepped_ || !isl_pending_ || wake_done_)
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_islands_wake runs once after every avn_contacts_step, before the solver stage");
        const size_t B = isl_B_;
        IslandState s = isl_;
        if (wake && B) {
            AVN_CUDA(isl_wake_.ensure(B));
            AVN_CUDA(cudaMemcpyAsync(isl_wake_.p, wake, B, cudaMemcpyHostToDevice, stream_));
            s.host_wake = isl_wake_.as<uint8_t>();
        }
        AVN_CUDA(cudaMemsetAsync(s.ctr, 0, sizeof(IslandCounters), stream_));
        GraphRows g = graph_rows();
        if (B) {
            const unsigned bb = unsigned((B + 255) / 256);
            if (g.hw > 0) isl_add_kernel<<<unsigned((g.hw + 255) / 256), 256, 0, stream_>>>(s, g);
            isl_flatten_kernel<<<bb, 256, 0, stream_>>>(s, 0);
            isl_wake_marks_kernel<<<bb, 256, 0, stream_>>>(s);
            isl_wake_bodies_kernel<<<bb, 256, 0, stream_>>>(s);
            isl_wake_roots_kernel<<<bb, 256, 0, stream_>>>(s);
            AVN_CUDA(cudaGetLastError());
        }
        AVN_CUDA(cudaMemcpyAsync(h_isl_, s.ctr, sizeof(IslandCounters), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));   // (the caller's wake column may be reused)
        wake_woken_ = h_isl_->woken;
        wake_merges_ = h_isl_->merges;
        wake_done_ = true;
        *out = AvnIslandsWake{};
        out->islands_woken = wake_woken_;
        if (wake_woken_ || h_isl_->absorbed) {   // no woken island: the graph is the one avn_contacts_step left
            const AvnStatus st = apply_pass(true, false);
            if (st != AVN_OK) return st;
            out->rows_woken = h_ctr_->rows_woken;
            out->colouring_rounds = h_ctr_->rounds;
        }
        out->rows_asleep = rows_asleep_; out->bodies_asleep = bodies_asleep_; out->manifold_count = graph_.count;
        memcpy(out->color_offsets, graph_.color_offsets, sizeof out->color_offsets);
        return AVN_OK;
    }

    AvnStatus download_sleeping(uint32_t capacity, uint8_t* row_asleep, uint32_t body_count, uint8_t* body_asleep) override {
        const size_t n = std::min(capacity, E_), nb = std::min(body_count, n_bodies_);
        if (row_asleep && n) AVN_CUDA(cudaMemcpyAsync(row_asleep, asleep_.p, n, cudaMemcpyDeviceToHost, stream_));
        if (body_asleep && nb) {
            if (apply_) AVN_CUDA(cudaMemcpyAsync(body_asleep, body_asleep_.p, nb, cudaMemcpyDeviceToHost, stream_));
            else memset(body_asleep, 0, nb);
        }
        AVN_CUDA(cudaStreamSynchronize(stream_));
        return AVN_OK;
    }

    void asleep_bodies(AsleepBodies* out) override {
        *out = AsleepBodies{};
        if (!apply_) return;
        out->body_asleep = body_asleep_.as<uint8_t>();
        out->count = n_bodies_;
        out->wake_skipped = isl_pending_ && !wake_done_;
    }

   private:
    AvnStatus reserve(uint32_t capacity) {
        if (capacity <= E_) return AVN_OK;
        const size_t n = capacity;
        struct Col { DevBuf* buf; size_t bytes_per_row; };
        Col cols[] = {{&c1_, 4}, {&c2_, 4}, {&b1_, 4}, {&b2_, 4}, {&live_, 1}, {&count_, 1}, {&disjoint_, 1}, {&normal_, 3 * sizeof(S)}, {&a1_, 12 * sizeof(S)},
                      {&a2_, 12 * sizeof(S)}, {&pen_, 4 * sizeof(S)}, {&ns_, 4 * sizeof(S)}, {&prev_count_, 1}, {&prev_a1_, 12 * sizeof(double)},
                      {&prev_a2_, 12 * sizeof(double)}, {&ws_n_in_, 4 * sizeof(S)}, {&ws_t_in_, 8 * sizeof(S)}, {&ws_n_out_, 4 * sizeof(S)},
                      {&ws_t_out_, 8 * sizeof(S)}, {&nimp_in_, 4 * sizeof(S)}, {&nimp_out_, 4 * sizeof(S)},
                      // graph state per row (zero = no flags, not touching, no colour)
                      {&pflags_, 1}, {&touching_, 1}, {&colour_, 1}, {&change_, 1}, {&old_colour_, 1}, {&ovf_pos_, 4}, {&ovf_, 4}, {&isl_event_, 1}, {&fresh_, 1},
                      {&event_, 1}, {&asleep_, 1}};
        for (Col& c : cols) {   // grow, keep the old rows, zero the new ones
            void* fresh = nullptr;
            AVN_CUDA(cudaMalloc(&fresh, n * c.bytes_per_row));
            AVN_CUDA(cudaMemsetAsync(fresh, 0, n * c.bytes_per_row, stream_));
            if (c.buf->p && E_) AVN_CUDA(cudaMemcpyAsync(fresh, c.buf->p, size_t(E_) * c.bytes_per_row, cudaMemcpyDeviceToDevice, stream_));
            AVN_CUDA(cudaStreamSynchronize(stream_));
            if (c.buf->p) cudaFree(c.buf->p);
            c.buf->p = fresh;
            c.buf->cap = n * c.bytes_per_row;
        }
        E_ = capacity;
        // work buffers of the graph step (contents do not outlive a step) and the pair set (rebuilt by the next step)
        const size_t nblocks = (n + RS_TILE - 1) / RS_TILE;
        AVN_CUDA(k0_.ensure(n * 4)); AVN_CUDA(k1_.ensure(n * 4)); AVN_CUDA(v0_.ensure(n * 4)); AVN_CUDA(v1_.ensure(n * 4)); AVN_CUDA(list_.ensure(n * 4));
        AVN_CUDA(evl_.ensure(n * 4));
        AVN_CUDA(hist_.ensure(256 * nblocks * 4));
        AVN_CUDA(m_b1_.ensure(n * 4)); AVN_CUDA(m_b2_.ensure(n * 4)); AVN_CUDA(m_fr_.ensure(n * sizeof(S))); AVN_CUDA(m_re_.ensure(n * sizeof(S)));
        uint64_t cap = 1024;
        while (cap < uint64_t(n) * 2) cap <<= 1;
        AVN_CUDA(table_.ensure(cap * sizeof(uint64_t)));
        table_mask_ = cap - 1;
        table_dirty_ = true;
        return AVN_OK;
    }
    // the collider / body columns of a step -> device (on `s`); keep_shapes: shape and dims are those of the previous call
    AvnStatus upload_inputs(const AvnNarrowInput* in, bool keep_shapes, cudaStream_t s) {
        const size_t C = in->collider_count, B = in->body_count;
        if (!in->dims || !in->position || !in->rotation || !in->linear_velocity || !in->angular_velocity || !in->aabb_min || !in->aabb_max)
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "contacts_step: dims, position, rotation, velocities and AABBs are required");
        keep_shapes = keep_shapes && in_.colliders == C && in_.dims != nullptr;
        AvnStatus st;
        up_stream_ = s;
#define UPC(buf, host, cnt, T, dst) if ((st = up<T>(buf, host, cnt, &dst)) != AVN_OK) { up_stream_ = stream_; return st; }
        if (!keep_shapes) {
            UPC(i_shape_, in->shape, C, uint8_t, in_.shape);
            UPC(i_dims_, in->dims, 3 * C, S, in_.dims);
            if (checked_ == in) {   // the flags describe the column now on the device
                has_capsule_ = checked_capsule_;
                has_hull_ = checked_hull_;
                max_hull_ = checked_max_hull_;
            }
        }
        UPC(i_pos_, in->position, 3 * C, S, in_.pos);
        UPC(i_rot_, in->rotation, 4 * C, S, in_.rot);
        UPC(i_lv_, in->linear_velocity, 3 * B, S, in_.lv);
        UPC(i_av_, in->angular_velocity, 3 * B, S, in_.av);
        UPC(i_amin_, in->aabb_min, 3 * C, S, in_.amin);
        UPC(i_amax_, in->aabb_max, 3 * C, S, in_.amax);
        in_.framed = frames_set_;
        if (frames_set_) {
            UPC(i_fpos_, frames_.position.data(), 3 * B, S, in_.frames.pos);
            UPC(i_frot_, frames_.rotation.data(), 4 * B, S, in_.frames.rot);
            UPC(i_fcom_, frames_.com.empty() ? nullptr : frames_.com.data(), 3 * B, S, in_.frames.com);
        }
#undef UPC
        up_stream_ = stream_;
        in_.colliders = C;
        return AVN_OK;
    }
    // geometry + match_contacts over rows [0, n)
    AvnStatus launch_narrow(const AvnNarrowParams* prm, const AvnNarrowInput* in, uint32_t match_contacts, double length_unit, uint32_t n) {
        bool only_fresh = false;
        if (prefetched_ == in) {   // prefetch_inputs copied this call's columns on the copy stream (and ran the rows that existed then)
            AVN_CUDA(cudaStreamWaitEvent(stream_, ev_in_, 0));
            only_fresh = early_rows_ > 0;
            if (only_fresh && n == early_rows_ && !added_this_step_) { prefetched_ = nullptr; early_rows_ = 0; return AVN_OK; }   // nothing new
        } else {
            if (prefetched_) AVN_CUDA(cudaStreamWaitEvent(stream_, ev_in_, 0));
            AvnStatus st = upload_inputs(in, false, stream_);
            if (st != AVN_OK) return st;
        }
        prefetched_ = nullptr;
        early_rows_ = 0;
        AvnStatus st = enqueue_narrow(prm, match_contacts, length_unit, n, stream_, only_fresh);
        // a full pass has computed the rows added this step too: they are no longer fresh.  Left set, the next step's fresh pass would run
        // them a second time after its early pass, matching their new points against themselves (visible once two points of one manifold
        // lie within the matching distance of each other, e.g. the corners of a thin table leg)
        if (st == AVN_OK && !only_fresh && n) AVN_CUDA(cudaMemsetAsync(fresh_.p, 0, n, stream_));
        return st;
    }
    AvnStatus enqueue_narrow(const AvnNarrowParams* prm, uint32_t match_contacts, double length_unit, uint32_t n, cudaStream_t s, bool only_fresh) {
        NarrowEdgeArgs<S> a{};
        a.r = rows();
        a.r.E = int(n);
        a.shape = in_.shape; a.dims = in_.dims; a.pos = in_.pos; a.rot = in_.rot; a.lv = in_.lv; a.av = in_.av; a.amin = in_.amin; a.amax = in_.amax;
        a.dt = prm->dt;
        a.tol = prm->contact_tolerance;
        a.thr2 = (0.1 * length_unit) * (0.1 * length_unit);
        a.match = match_contacts ? 1 : 0;
        if (in_.framed) {
            narrow_framed_edges_kernel<S, false><<<(n + 127) / 128, 128, 0, s>>>(a, in_.frames, fresh_.as<uint8_t>(), only_fresh ? 1 : 0, has_capsule_ ? 1 : 0,
                                                                                 has_hull_ ? 1 : 0);
            if (has_capsule_)
                narrow_framed_edges_kernel<S, true><<<(n + 127) / 128, 128, 0, s>>>(a, in_.frames, fresh_.as<uint8_t>(), only_fresh ? 1 : 0, 1, has_hull_ ? 1 : 0);
            if (has_hull_) narrow_hull_edges_kernel<S, true><<<(n + 127) / 128, 128, 0, s>>>(a, in_.frames, fresh_.as<uint8_t>(), only_fresh ? 1 : 0, hulls_->dev);
        } else {
            narrow_edges_kernel<S><<<(n + 127) / 128, 128, 0, s>>>(a, fresh_.as<uint8_t>(), only_fresh ? 1 : 0, has_capsule_ ? 1 : 0, has_hull_ ? 1 : 0);
            if (has_capsule_) narrow_capsule_edges_kernel<S><<<(n + 127) / 128, 128, 0, s>>>(a, fresh_.as<uint8_t>(), only_fresh ? 1 : 0, has_hull_ ? 1 : 0);
            if (has_hull_)
                narrow_hull_edges_kernel<S, false><<<(n + 127) / 128, 128, 0, s>>>(a, BodyFrameCols<S>{}, fresh_.as<uint8_t>(), only_fresh ? 1 : 0, hulls_->dev);
        }
        AVN_CUDA(cudaGetLastError());
        return AVN_OK;
    }
    // one stable 8-bit radix pass (digit = the low byte of the key): (k0_, v0_) -> (k1_, vals_out or v1_).  The event lists, the reports and the
    // removal sort into evl_: v1_ holds the colour-major list the solver reads until the next step
    void radix_pass(int n, uint32_t* vals_out = nullptr) {
        uint32_t* vo = vals_out ? vals_out : v1_.as<uint32_t>();
        const int nblocks = (n + RS_TILE - 1) / RS_TILE;
        rs_histogram<uint32_t><<<nblocks, RS_THREADS, 0, stream_>>>(k0_.as<uint32_t>(), n, 0, hist_.as<uint32_t>(), nblocks);
        if (nblocks <= RS_FUSE_MAX_BLOCKS) {
            rs_scatter<uint32_t, true><<<nblocks, RS_THREADS, 0, stream_>>>(k0_.as<uint32_t>(), v0_.as<uint32_t>(), n, 0, hist_.as<uint32_t>(), nblocks, k1_.as<uint32_t>(), vo);
        } else {
            rs_scan<<<1, 1024, 0, stream_>>>(hist_.as<uint32_t>(), 256 * nblocks);
            rs_scatter<uint32_t, false><<<nblocks, RS_THREADS, 0, stream_>>>(k0_.as<uint32_t>(), v0_.as<uint32_t>(), n, 0, hist_.as<uint32_t>(), nblocks, k1_.as<uint32_t>(), vo);
        }
    }
    // after a radix pass over hw_ rows: out[k - 1] = the number of rows whose key is below k, k = 1 .. nb (on the host)
    AvnStatus small_bounds(int nb, uint32_t* out) {
        AVN_CUDA(bounds_.ensure(16));
        key_bounds_kernel<<<1, 32, 0, stream_>>>(k1_.as<uint32_t>(), int(hw_), nb, bounds_.as<uint32_t>());
        AVN_CUDA(cudaGetLastError());
        AVN_CUDA(cudaMemcpyAsync(out, bounds_.p, size_t(nb) * 4, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        return AVN_OK;
    }
    // room for `need` queued CollisionEnds in pending list i (keeps its entries)
    AvnStatus pend_reserve(int i, uint32_t need) {
        if (need <= pend_cap_[i]) return AVN_OK;
        const uint32_t cap = std::max(need, std::max(2 * pend_cap_[i], 256u)), old = pend_cap_[i];
        void* p = nullptr;
        AVN_CUDA(cudaMalloc(&p, size_t(cap) * 17));
        if (pend_n_[i]) {
            const uint32_t* src = pend_[i].as<uint32_t>();
            uint32_t* dst = static_cast<uint32_t*>(p);
            for (int c = 0; c < 4; ++c)
                AVN_CUDA(cudaMemcpyAsync(dst + size_t(c) * cap, src + size_t(c) * old, size_t(pend_n_[i]) * 4, cudaMemcpyDeviceToDevice, stream_));
            AVN_CUDA(cudaMemcpyAsync(dst + 4 * size_t(cap), src + 4 * size_t(old), pend_n_[i], cudaMemcpyDeviceToDevice, stream_));
            AVN_CUDA(cudaStreamSynchronize(stream_));
        }
        if (pend_[i].p) cudaFree(pend_[i].p);
        pend_[i].p = p;
        pend_[i].cap = size_t(cap) * 17;
        pend_cap_[i] = cap;
        return AVN_OK;
    }
    // remove_collider for each listed collider (indices checked by the caller), then the colour-major list, the colour offsets and the pair set
    // rebuilt as a step leaves them
    AvnStatus remove_rows(uint32_t n, const uint32_t* colliders) {
        if (n == 0 || hw_ == 0) return AVN_OK;
        AVN_CUDA(rm_.ensure(std::max<size_t>(n_colliders_, 1)));
        AVN_CUDA(cudaMemsetAsync(rm_.p, 0, std::max<size_t>(n_colliders_, 1), stream_));
        AVN_CUDA(stage_.ensure(size_t(n) * 4));
        AVN_CUDA(cudaMemcpyAsync(stage_.p, colliders, size_t(n) * 4, cudaMemcpyHostToDevice, stream_));
        mark_colliders_kernel<<<(n + 255) / 256, 256, 0, stream_>>>(stage_.as<uint32_t>(), n, rm_.as<uint8_t>());
        AVN_CUDA(cudaMemsetAsync(ctr_.p, 0, offsetof(GraphCounters, ovf_count), stream_));   // (the step's counters went to the host already)
        GraphRows g = graph_rows();
        const unsigned rb = (hw_ + 255) / 256;
        // (avn_islands_wake has applied the step's add events already: a contact it linked is unlinked like any other)
        const int islands = !isl_configured_ ? 0 : (isl_pending_ && !(apply_ && wake_done_)) ? 2 : 1;
        remove_rows_kernel<<<rb, 256, 0, stream_>>>(g, rm_.as<uint8_t>(), isl_, islands, k0_.as<uint32_t>(), v0_.as<uint32_t>());
        radix_pass(int(hw_), evl_.as<uint32_t>());   // removed touching rows, then the other removed rows, each in ascending ContactId
        AVN_CUDA(cudaMemcpyAsync(h_ctr_, ctr_.p, sizeof(GraphCounters), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        const uint32_t n_rm = h_ctr_->removed, n_end = h_ctr_->stopped;
        if (n_rm == 0) return AVN_OK;   // nothing named these colliders: the graphs are as the last step left them
        AvnStatus st = pend_reserve(pend_cur_, pend_n_[pend_cur_] + n_end);
        if (st != AVN_OK) return st;
        if (n_end) {
            queue_ends_kernel<<<(n_end + 255) / 256, 256, 0, stream_>>>(g, evl_.as<uint32_t>(), n_end, pend_n_[pend_cur_], pend_cap_[pend_cur_],
                                                                         pend_[pend_cur_].as<uint32_t>());
            pend_n_[pend_cur_] += n_end;
        }
        // only touching rows hold a colour, and they lead the list in ascending ContactId: the overflow colour's swap_removes in that order
        overflow_list_kernel<<<1, 32, 0, stream_>>>(g, evl_.as<uint32_t>());
        rebuild_list(g);
        AVN_CUDA(cudaMemsetAsync(table_.p, 0, (table_mask_ + 1) * sizeof(uint64_t), stream_));
        pair_set_kernel<<<rb, 256, 0, stream_>>>(g, table_.as<uint64_t>(), table_mask_);
        AVN_CUDA(cudaGetLastError());
        table_dirty_ = false;
        AVN_CUDA(cudaMemcpyAsync(h_ctr_, ctr_.p, sizeof(GraphCounters), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        live_n_ -= n_rm;
        rows_asleep_ = h_ctr_->rows_asleep;
        take_list_counters();
        return AVN_OK;
    }
    // Brings the applied state in line with the islands' decisions: body_asleep, then the rows of the woken islands (pushed by the colouring
    // rounds in ascending ContactId), then the rows of the islands that fell asleep (popped; the overflow colour's swap_removes in ascending
    // ContactId), then the colour-major list as a step leaves it.  The pair set does not change: an asleep row stays in the ContactGraph.
    AvnStatus apply_pass(bool wakes, bool sleeps) {
        // the step's counters went to the host and into AvnContactStep already; from here on the device block and h_ctr_ describe this pass, not
        // the contact step (nothing reads the step's removed / started / stopped from them afterwards: the events come from the rows' event bytes)
        AVN_CUDA(cudaMemsetAsync(ctr_.p, 0, offsetof(GraphCounters, ovf_count), stream_));
        GraphRows g = graph_rows();
        uint8_t* body_asleep = body_asleep_.as<uint8_t>();
        uint8_t* fell = body_asleep + std::max<size_t>(n_bodies_, 1);
        if (isl_B_) sleep_bodies_kernel<<<unsigned((size_t(isl_B_) + 255) / 256), 256, 0, stream_>>>(isl_, body_asleep, fell, g.ctr);
        if (hw_) {
            const unsigned rb = (hw_ + 255) / 256;
            if (wakes) {
                wake_rows_kernel<S><<<rb, 256, 0, stream_>>>(g, body_asleep, ws_n_in_.as<S>(), ws_t_in_.as<S>(), ws_n_out_.as<S>(), ws_t_out_.as<S>(),
                                                             k0_.as<uint32_t>(), v0_.as<uint32_t>());
                radix_pass(int(hw_), list_.as<uint32_t>());   // the pushes first, in ascending ContactId
                const AvnStatus st = colour_changed(g);
                if (st != AVN_OK) return st;
                overflow_list_kernel<<<1, 32, 0, stream_>>>(g, list_.as<uint32_t>());
            }
            if (sleeps) {
                if (wakes) AVN_CUDA(cudaMemsetAsync(&g.ctr->changed, 0, sizeof(uint32_t), stream_));   // the list below is the sleeping rows' alone
                sleep_rows_kernel<<<rb, 256, 0, stream_>>>(g, fell, k0_.as<uint32_t>(), v0_.as<uint32_t>());
                radix_pass(int(hw_), list_.as<uint32_t>());
                overflow_list_kernel<<<1, 32, 0, stream_>>>(g, list_.as<uint32_t>());
            }
            rebuild_list(g);
            AVN_CUDA(cudaGetLastError());
        }
        AVN_CUDA(cudaMemcpyAsync(h_ctr_, ctr_.p, sizeof(GraphCounters), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        if (h_ctr_->aborted) return err_->fail(AVN_ERR_CUDA, "islands: the colouring of the woken rows did not converge");
        bodies_asleep_ = h_ctr_->bodies_asleep;
        rows_asleep_ = h_ctr_->rows_asleep;
        if (hw_) take_list_counters();
        return AVN_OK;
    }
    // ConstraintGraph pushes / pops of the rows list_[0, ctr->changed) in ascending ContactId: the dependency wavefront (see the top of the file)
    AvnStatus colour_changed(GraphRows& g) {
        AVN_CUDA(cudaMemsetAsync(body_min_.p, 0xff, std::max<size_t>(n_bodies_, 1) * 16, stream_));
        if (use_cluster_) {   // small change sets: one thread-block cluster (returns at once when there are more than CL_MAX changed edges)
            cudaLaunchConfig_t cfg{};
            cfg.gridDim = dim3(CL_BLOCKS); cfg.blockDim = dim3(CL_THREADS); cfg.dynamicSmemBytes = 0; cfg.stream = stream_;
            cudaLaunchAttribute attr[1];
            attr[0].id = cudaLaunchAttributeClusterDimension;
            attr[0].val.clusterDim.x = CL_BLOCKS; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
            cfg.attrs = attr; cfg.numAttrs = 1;
            const uint32_t* list = list_.as<uint32_t>();
            cudaError_t ce = cudaLaunchKernelEx(&cfg, colour_rounds_cluster_kernel, g, list);
            if (ce != cudaSuccess) { (void)cudaGetLastError(); use_cluster_ = false; }
        }
        const uint32_t* list = list_.as<uint32_t>();
        uint32_t skip_upto = use_cluster_ ? CL_MAX : 0u;
        void* args[] = {(void*)&g, (void*)&list, (void*)&skip_upto};
        int per_sm = 0;
        AVN_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, colour_rounds_kernel, 256, 0));
        if (per_sm < 1) return err_->fail(AVN_ERR_CUDA, "contacts_step: the colouring kernel does not fit the device");
        AVN_CUDA(cudaLaunchCooperativeKernel((const void*)colour_rounds_kernel, dim3(sm_count_), dim3(256), args, 0, stream_));
        return AVN_OK;
    }
    // the colour-major list from the rows' colours: frees the removed rows, one stable radix pass over the colour byte -> k1_ sorted colour keys,
    // v1_ = the list (ascending ContactId inside a colour), then the offsets and the per-manifold columns
    void rebuild_list(const GraphRows& g) {
        const unsigned rb = (hw_ + 255) / 256;
        finalize_rows_kernel<<<rb, 256, 0, stream_>>>(g, k0_.as<uint32_t>(), v0_.as<uint32_t>());
        radix_pass(int(hw_));
        color_offsets_kernel<<<1, 64, 0, stream_>>>(g, k1_.as<uint32_t>(), v1_.as<uint32_t>());
        gather_graph_kernel<S><<<std::min<unsigned>(rb, unsigned(sm_count_) * 8u), 256, 0, stream_>>>(g, v1_.as<uint32_t>(), have_fr_ ? fr_.as<double>() : nullptr,
                                                                                                    have_re_ ? re_.as<double>() : nullptr, m_b1_.as<int32_t>(),
                                                                                                    m_b2_.as<int32_t>(), m_fr_.as<S>(), m_re_.as<S>());
    }
    void take_list_counters() {   // h_ctr_ holds the counters rebuild_list left
        graph_.count = h_ctr_->manifolds;
        graph_.any_restitution = h_ctr_->any_restitution;
        memcpy(graph_.color_offsets, h_ctr_->color_offsets, sizeof graph_.color_offsets);
    }
    GraphRows graph_rows() {
        GraphRows g{};
        g.hw = int(hw_);
        g.c1 = c1_.as<uint32_t>(); g.c2 = c2_.as<uint32_t>(); g.b1 = b1_.as<uint32_t>(); g.b2 = b2_.as<uint32_t>();
        g.live = live_.as<uint8_t>(); g.count = count_.as<uint8_t>(); g.disjoint = disjoint_.as<uint8_t>(); g.prev_count = prev_count_.as<uint8_t>();
        g.pflags = pflags_.as<uint8_t>(); g.touching = touching_.as<uint8_t>(); g.colour = colour_.as<uint8_t>(); g.change = change_.as<uint8_t>();
        g.old_colour = old_colour_.as<uint8_t>(); g.ovf_pos = ovf_pos_.as<uint32_t>(); g.ovf = ovf_.as<uint32_t>(); g.isl_event = isl_event_.as<uint8_t>(); g.fresh = fresh_.as<uint8_t>();
        g.event = event_.as<uint8_t>(); g.asleep = asleep_.as<uint8_t>(); g.sensor = sensor_h_.empty() ? nullptr : sensor_.as<uint8_t>();
        g.body_kind = kind_.as<uint8_t>(); g.n_bodies = int(n_bodies_);
        g.body_bits = body_bits_.as<uint32_t>(); g.body_min = body_min_.as<unsigned long long>();
        g.ctr = ctr_.as<GraphCounters>();
        return g;
    }
    EdgeRows<S> rows() {
        EdgeRows<S> r{};
        r.E = int(E_);
        r.c1 = c1_.as<uint32_t>(); r.c2 = c2_.as<uint32_t>(); r.b1 = b1_.as<uint32_t>(); r.b2 = b2_.as<uint32_t>(); r.live = live_.as<uint8_t>();
        r.count = count_.as<uint8_t>(); r.disjoint = disjoint_.as<uint8_t>(); r.normal = normal_.as<S>(); r.a1 = a1_.as<S>(); r.a2 = a2_.as<S>();
        r.pen = pen_.as<S>(); r.ns = ns_.as<S>(); r.prev_count = prev_count_.as<uint8_t>(); r.prev_a1 = prev_a1_.as<double>(); r.prev_a2 = prev_a2_.as<double>();
        r.ws_n_in = ws_n_in_.as<S>(); r.ws_t_in = ws_t_in_.as<S>(); r.ws_n_out = ws_n_out_.as<S>(); r.ws_t_out = ws_t_out_.as<S>();
        r.nimp_in = nimp_in_.as<S>(); r.nimp_out = nimp_out_.as<S>();
        r.asleep = asleep_.as<uint8_t>();
        return r;
    }
    template <class T> AvnStatus up(DevBuf& buf, const void* host, size_t count, const T** dev) {
        *dev = nullptr;
        if (!host || count == 0) return AVN_OK;
        AVN_CUDA(buf.ensure(count * sizeof(T)));
        AVN_CUDA(cudaMemcpyAsync(buf.p, host, count * sizeof(T), cudaMemcpyHostToDevice, up_stream_));
        *dev = buf.as<T>();
        return AVN_OK;
    }
    cudaStream_t stream_;
    cudaStream_t copy_stream_ = nullptr, up_stream_ = nullptr;
    cudaEvent_t ev_in_ = nullptr;
    const AvnNarrowInput* prefetched_ = nullptr;
    struct { const uint8_t* shape = nullptr; const S* dims = nullptr; const S* pos = nullptr; const S* rot = nullptr; const S* lv = nullptr; const S* av = nullptr;
             const S* amin = nullptr; const S* amax = nullptr; size_t colliders = 0;
             bool framed = false; BodyFrameCols<S> frames{}; } in_;   // framed: the body frames below were copied with these columns
    ErrorSink* err_;
    uint32_t E_ = 0;
    DevBuf c1_, c2_, b1_, b2_, live_, count_, disjoint_, normal_, a1_, a2_, pen_, ns_, prev_count_, prev_a1_, prev_a2_, ws_n_in_, ws_t_in_, ws_n_out_, ws_t_out_,
        nimp_in_, nimp_out_, stage_;
    DevBuf i_shape_, i_dims_, i_pos_, i_rot_, i_lv_, i_av_, i_amin_, i_amax_, i_fpos_, i_frot_, i_fcom_;
    BodyFrames frames_;           // avn_contacts_set_body_frames (host copy), in effect while frames_set_
    bool frames_set_ = false;
    // graphs
    using ResidentGraph = ContactsBase::ResidentGraph;
    DevBuf isl_event_, fresh_, isl_buf_, isl_in_, isl_out_, isl_j_;
    uint32_t early_rows_ = 0;     // rows whose geometry prefetch_inputs already launched on the copy stream
    bool has_capsule_ = false;    // the shape column on the device holds a capsule
    const AvnNarrowInput* checked_ = nullptr;   // the input check_shapes last accepted, and whether its column holds a capsule
    bool checked_capsule_ = false;
    const HullTable* hulls_ = nullptr;
    uint64_t hull_generation_ = 0;
    bool has_hull_ = false;       // the shape column on the device holds a convex hull; max_hull_: the largest index it names
    uint32_t max_hull_ = 0;
    bool checked_hull_ = false;
    uint32_t checked_max_hull_ = 0;
    bool added_this_step_ = false;
    IslandState isl_{};
    IslandCounters* h_isl_ = nullptr;
    uint32_t isl_B_ = 0, isl_J_ = 0;
    float isl_length_unit_ = 1.f;
    bool isl_configured_ = false, isl_has_thr_lin_ = false, isl_has_thr_ang_ = false, isl_has_disabled_ = false;
    DevBuf pflags_, touching_, colour_, change_, old_colour_, ovf_pos_, ovf_, kind_, fr_, re_, body_bits_, body_min_, ctr_, k0_, k1_, v0_, v1_, hist_, list_, m_b1_, m_b2_,
        m_fr_, m_re_, table_;
    GraphCounters* h_ctr_ = nullptr;
    ResidentGraph graph_{};
    // collision events, sensors, removals, reports
    DevBuf event_, evl_, evout_, repout_, bounds_, sensor_, rm_, pend_[2];
    // applied sleeping: asleep_ per row; body_asleep_ = [B] applied state, then [B] "fell asleep in this pass"
    DevBuf asleep_, body_asleep_, isl_wake_;
    bool apply_ = false, wake_done_ = false;
    uint32_t bodies_asleep_ = 0, rows_asleep_ = 0, wake_woken_ = 0, wake_merges_ = 0;
    std::vector<uint8_t> sensor_h_;           // the sensor column as last set (empty = no sensor)
    uint32_t pend_n_[2] = {0, 0}, pend_cap_[2] = {0, 0};
    int pend_cur_ = 0;                        // pend_[pend_cur_] queues the removals' CollisionEnds; the other list is reported with the last step
    bool stepped_ = false, isl_pending_ = false;
    uint64_t table_mask_ = 0;
    uint32_t hw_ = 0, live_n_ = 0, n_bodies_ = 0, n_colliders_ = 0;
    int sm_count_ = 132;
    bool configured_ = false, have_fr_ = false, have_re_ = false, table_dirty_ = true, use_cluster_ = true;
};

}  // namespace

ContactsBase* make_contacts(uint32_t scalar_bits, cudaStream_t stream, ErrorSink* err) {
    if (scalar_bits == 32) return new Contacts<float>(stream, err);
    if (scalar_bits == 64) return new Contacts<double>(stream, err);
    return nullptr;
}

}  // namespace avn
