// Order-preserving level schedule for XPBD joints (host code, no CUDA).
// The reference solves joints serially: type order Fixed, Revolute, Spherical, Prismatic, Distance, each in ECS table
// order (xpbd/plugin.rs:58-86,145-189).  level(j) = max over the bodies j shares with EARLIER joints of (their last
// level + 1), counting only bodies some joint actually writes; joints of one level are then conflict-free and running
// the levels in order reproduces the serial sweep exactly.
// joint_damping<T> (solver/plugin.rs:759-806) has a level schedule of its own over the damped joints: it also orders the joints of one type
// whose end on one side has no SolverBody, because that system run hands dummy_body1 / dummy_body2 from one such joint to the next.
#pragma once
#include <algorithm>
#include <string>
#include <vector>

#include "../../include/avian_b200.h"

namespace avn {

struct JointSchedule {
    std::vector<int> type, index;     // per schedule slot: (joint type, index in that type's columns)
    std::vector<int> level_off;       // [n_levels + 1]
    std::vector<int> level_of_global; // per joint in global (reference) order
    int n_levels = 0;
    bool any_damping = false;
    std::vector<int> damp_slot;       // per damping item: the joint's slot in the solve schedule, level by level
    std::vector<int> damp_level_off;  // [n_damp_levels + 1]
    int n_damp_levels = 0;
};

// order-preserving levels of a sequence of items over `n_res` resources: level = 1 + the last level of any earlier item sharing a resource
inline int level_items(const std::vector<int>& r1, const std::vector<int>& r2, size_t n_res, std::vector<int>& level, std::vector<int>& level_off) {
    const size_t n = r1.size();
    std::vector<int> last(n_res, 0);
    level.assign(n, 0);
    int n_levels = 0;
    for (size_t g = 0; g < n; ++g) {
        int l = 0;
        if (r1[g] >= 0) l = std::max(l, last[r1[g]]);
        if (r2[g] >= 0) l = std::max(l, last[r2[g]]);
        level[g] = l;
        if (r1[g] >= 0) last[r1[g]] = l + 1;
        if (r2[g] >= 0) last[r2[g]] = l + 1;
        n_levels = std::max(n_levels, l + 1);
    }
    level_off.assign(n_levels + 1, 0);
    for (size_t g = 0; g < n; ++g) ++level_off[level[g] + 1];
    for (int l = 0; l < n_levels; ++l) level_off[l + 1] += level_off[l];
    return n_levels;
}

inline AvnStatus build_joint_schedule(const AvnBodyColumns& bc, const AvnJointSet& js, JointSchedule& out, std::string& error) {
    size_t J = 0;
    for (int t = 0; t < AVN_JOINT_TYPE_COUNT; ++t) J += js.types[t].count;
    const uint32_t B = bc.count;
    std::vector<int> type(J), index(J), b1(J), b2(J);
    std::vector<uint8_t> conflict(B, 0);
    bool any_damping = false;
    auto kind_of = [&](int b) { return bc.kind ? bc.kind[b] : uint8_t(AVN_BODY_DYNAMIC); };
    auto dom_of = [&](int b) -> int { return kind_of(b) == AVN_BODY_DYNAMIC ? (bc.dominance ? int(bc.dominance[b]) : 0) : 128; };
    auto has_sb = [&](int b) { return kind_of(b) != AVN_BODY_STATIC; };
    size_t g = 0;
    for (int t = 0; t < AVN_JOINT_TYPE_COUNT; ++t) {
        const AvnJointColumns& jc = js.types[t];
        if (jc.count && (!jc.body1 || !jc.body2 || !jc.local_anchor1 || !jc.local_anchor2)) {
            error = "joint type " + std::to_string(t) + ": body1/body2/local_anchor1/local_anchor2 are required";
            return AVN_ERR_INVALID_ARGUMENT;
        }
        for (uint32_t k = 0; k < jc.count; ++k, ++g) {
            int x = jc.body1[k], y = jc.body2[k];
            if (x < 0 || y < 0 || uint32_t(x) >= B || uint32_t(y) >= B) {
                error = "joint type " + std::to_string(t) + " #" + std::to_string(k) + " references a body outside the body columns";
                return AVN_ERR_INVALID_ARGUMENT;
            }
            type[g] = t; index[g] = int(k); b1[g] = x; b2[g] = y;
            if (jc.damping_enabled && jc.damping_enabled[k]) any_damping = true;
        }
    }
    // a body orders the joints that touch it iff some joint WRITES it: it has a SolverBody and is not the dominated side
    // there (xpbd/plugin.rs:176-180).  joint_damping writes every SolverBody it touches (solver/plugin.rs:789-803).
    for (g = 0; g < J; ++g) {
        int rel = dom_of(b1[g]) - dom_of(b2[g]);
        if (has_sb(b1[g]) && (any_damping || !(rel > 0))) conflict[b1[g]] = 1;
        if (has_sb(b2[g]) && (any_damping || !(rel < 0))) conflict[b2[g]] = 1;
    }
    std::vector<int> r1(J), r2(J);
    for (g = 0; g < J; ++g) {
        r1[g] = conflict[b1[g]] ? b1[g] : -1;
        r2[g] = conflict[b2[g]] ? b2[g] : -1;
    }
    const int n_levels = level_items(r1, r2, B, out.level_of_global, out.level_off);
    out.type.resize(J);
    out.index.resize(J);
    std::vector<int> slot_of_global(J);
    std::vector<int> cursor(out.level_off.begin(), out.level_off.end() - 1);
    for (g = 0; g < J; ++g) {  // stable within a level
        int s = cursor[out.level_of_global[g]]++;
        slot_of_global[g] = s;
        out.type[s] = type[g];
        out.index[s] = index[g];
    }
    // damping: every SolverBody is written; an end without one is the run's dummy of that side, resource B + 2 * type + side
    std::vector<int> dg, d1, d2;
    for (g = 0; g < J; ++g) {
        const AvnJointColumns& jc = js.types[type[g]];
        if (!(jc.damping_enabled && jc.damping_enabled[index[g]])) continue;
        dg.push_back(int(g));
        d1.push_back(has_sb(b1[g]) ? b1[g] : int(B) + 2 * type[g]);
        d2.push_back(has_sb(b2[g]) ? b2[g] : int(B) + 2 * type[g] + 1);
    }
    std::vector<int> dlevel;
    out.n_damp_levels = level_items(d1, d2, size_t(B) + 2 * AVN_JOINT_TYPE_COUNT, dlevel, out.damp_level_off);
    out.damp_slot.assign(dg.size(), 0);
    std::vector<int> dcursor(out.damp_level_off.begin(), out.damp_level_off.end() - 1);
    for (size_t k = 0; k < dg.size(); ++k) out.damp_slot[dcursor[dlevel[k]]++] = slot_of_global[dg[k]];
    out.n_levels = n_levels;
    out.any_damping = any_damping;
    return AVN_OK;
}

}  // namespace avn
