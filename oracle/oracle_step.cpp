// TEST INFRASTRUCTURE — NOT PRODUCT CODE.  (see oracle_solver.hpp for the parity statement: PARITY UNPINNED)
// The solver stage driver: restates the system order of SolverSystems / SubstepSchedule
// (solver/schedule.rs:32-69, xpbd/plugin.rs:30-94, SURVEY.md §3.1-3.2).
//
// `threads` > 1 runs the reference's execution structure with a std::thread pool standing in for Bevy's
// ComputeTaskPool (src/utils.rs:62-87): body loops parallel, colours parallel in chunks when len >= 64,
// overflow colour / joints / velocity projection / damping serial.  Results are identical to threads == 1
// because colours are conflict-free (constraint_graph.rs:4-6).
#include <atomic>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>

#include "oracle_solver.hpp"

namespace orc {

// ---- a tiny persistent pool (par_for_each, src/utils.rs:62-87) -----------------------------------------
class Pool {
   public:
    explicit Pool(int n) : n_(n) {
        for (int i = 1; i < n_; ++i) workers_.emplace_back([this, i] { worker(i); });
    }
    ~Pool() {
        {
            std::unique_lock<std::mutex> lk(m_);
            stop_ = true;
            ++gen_;
        }
        cv_.notify_all();
        for (auto& t : workers_) t.join();
    }
    int size() const { return n_; }
    // chunk = len / threads like the reference; serial when len < min_len or a single thread
    void par_for(size_t len, size_t min_len, const std::function<void(size_t, size_t)>& f) {
        if (n_ <= 1 || len < min_len) { f(0, len); return; }
        size_t chunk = std::max<size_t>(1, len / size_t(n_));
        {
            std::unique_lock<std::mutex> lk(m_);
            fn_ = &f; len_ = len; chunk_ = chunk; next_.store(0); pending_ = n_ - 1; ++gen_;
        }
        cv_.notify_all();
        run_chunks();
        std::unique_lock<std::mutex> lk(m_);
        done_.wait(lk, [this] { return pending_ == 0; });
    }

   private:
    void run_chunks() {
        for (;;) {
            size_t s = next_.fetch_add(chunk_);
            if (s >= len_) break;
            (*fn_)(s, std::min(len_, s + chunk_));
        }
    }
    void worker(int) {
        uint64_t seen = 0;
        for (;;) {
            {
                std::unique_lock<std::mutex> lk(m_);
                cv_.wait(lk, [&] { return gen_ != seen; });
                seen = gen_;
                if (stop_) return;
            }
            run_chunks();
            std::unique_lock<std::mutex> lk(m_);
            if (--pending_ == 0) done_.notify_one();
        }
    }
    int n_;
    std::vector<std::thread> workers_;
    std::mutex m_;
    std::condition_variable cv_, done_;
    const std::function<void(size_t, size_t)>* fn_ = nullptr;
    size_t len_ = 0, chunk_ = 1;
    std::atomic<size_t> next_{0};
    int pending_ = 0;
    uint64_t gen_ = 0;
    bool stop_ = false;
};

template <class S>
static void for_each_color(SolverWorld<S>& w, Pool& pool, const std::vector<uint8_t>& has_sb,
                           const std::function<void(ContactConstraint<S>&, SolverBody<S>&, SolverBody<S>&, const SolverBodyInertia<S>&,
                                                    const SolverBodyInertia<S>&)>& f) {
    const SolverBodyInertia<S> dummy_inertia;
    auto run = [&](ContactConstraint<S>& c) {
        SolverBody<S> d1, d2;
        BodyRef<S> r1, r2;
        resolve_bodies(w, c.body1, c.body2, c.relative_dominance, d1, d2, dummy_inertia, r1, r2, has_sb);
        f(c, *r1.body, *r2.body, *r1.inertia, *r2.inertia);
    };
    // overflow colour first, serially (solver/plugin.rs:461-467)
    for (auto& c : w.constraints[AVN_COLOR_OVERFLOW]) run(c);
    for (int col = 0; col < AVN_COLOR_OVERFLOW; ++col) {
        auto& v = w.constraints[col];
        if (v.empty()) continue;
        pool.par_for(v.size(), 64, [&](size_t a, size_t b) {
            for (size_t i = a; i < b; ++i) run(v[i]);
        });
    }
}

// The stage as a resumable object: prepare -> substep x N -> restitution -> finalize.  orc_solver_step runs them back to back; the
// orc_step_* entry points expose them one by one for the x-slab partition tests (include/avian_b200.h, "one coupled scene over
// several GPUs"), where a boundary exchange happens between substeps.
template <class S>
struct StepState {
    using C = Columns<S>;
    AvnStepParams prm;
    AvnBodyColumns bc;
    AvnManifoldColumns mc_store;
    AvnManifoldColumns* mc = nullptr;
    AvnJointSet js_store;
    AvnJointSet* js = nullptr;
    Pool pool;
    size_t B = 0;
    SolverWorld<S> w;
    std::vector<uint8_t> has_sb;  // has SolverBody (dynamic or kinematic)
    std::vector<Quat<S>> rot0;
    std::vector<V3<S>> pos0, linvel0;
    S dt = 0, h = 0, max_overlap_solve_speed = 0, warm_coeff = 0;
    std::vector<V3<S>> pre_dp;
    std::vector<Quat<S>> pre_dq;
    bool have_joints = false;
    const SolverBodyInertia<S> dummy_inertia{};
    uint32_t iters = 1;
    // boundary bodies of the x-slab partition (AvnBoundary)
    std::vector<int> bnd_body, bnd_source, bnd_owner;
    std::vector<V3<S>> ref_lin, ref_ang;
    int bnd_rank = 0, bnd_world = 1;
    size_t bnd_slots = 0;

    StepState(const AvnStepParams& p, const AvnBodyColumns& b, const AvnManifoldColumns* m, const AvnJointSet* j, int threads)
        : prm(p), bc(b), pool(std::max(1, threads)) {
        if (m) { mc_store = *m; mc = &mc_store; }
        if (j) { js_store = *j; js = &js_store; }
    }

    int prepare() {
        B = bc.count;
        w.bodies.assign(B, SolverBody<S>());
        w.inertias.assign(B, SolverBodyInertia<S>());
        w.integ.assign(B, VelocityIntegrationData<S>());
        has_sb.assign(B, 0);
        rot0.resize(B);
        pos0.resize(B);
        linvel0.resize(B);
        dt = S(prm.dt);
        h = S(prm.h);
    // ---- prepare_solver_bodies (solver_body/plugin.rs:173-251)
    pool.par_for(B, 1, [&](size_t a, size_t e) {
        for (size_t i = a; i < e; ++i) {
            uint8_t kind = bc.kind ? bc.kind[i] : uint8_t(AVN_BODY_DYNAMIC);
            rot0[i] = C::quat(bc.rotation, i);
            pos0[i] = C::vec3(bc.position, i);
            linvel0[i] = C::vec3(bc.linear_velocity, i);
            if (kind == AVN_BODY_STATIC) continue;
            has_sb[i] = 1;
            SolverBody<S>& sb = w.bodies[i];
            sb.linear_velocity = linvel0[i];
            sb.angular_velocity = C::vec3(bc.angular_velocity, i);
            uint8_t locked = bc.locked_axes ? bc.locked_axes[i] : 0;
            Sym3<S> inv_local = C::sym3(bc.inverse_inertia_local, i);
            w.inertias[i] = make_inertia<S>(C::scalar(bc.inverse_mass, i), rotate_inverse_inertia(inv_local, rot0[i]), locked,
                                            bc.dominance ? bc.dominance[i] : int8_t(0), kind == AVN_BODY_DYNAMIC);
            sb.flags = locked;
            if (kind == AVN_BODY_KINEMATIC) sb.flags |= (1u << 6);
            bool rotation_locked = (locked & 0x7) == 0x7;
            if (!rotation_locked && !is_isotropic(inv_local, S(1e-6))) sb.flags |= (1u << 7);
        }
    });

    // ---- prepare_xpbd_joint<T> (xpbd/plugin.rs:125-142 + each joint's prepare)
    if (js) {
        for (int t = 0; t < AVN_JOINT_TYPE_COUNT; ++t) {
            const AvnJointColumns& jc = js->types[t];
            for (uint32_t k = 0; k < jc.count; ++k) {
                JointData<S> j;
                j.type = t;
                j.index_in_type = k;
                j.body1 = jc.body1[k];
                j.body2 = jc.body2[k];
                if (j.body1 < 0 || j.body2 < 0 || size_t(j.body1) >= B || size_t(j.body2) >= B) return AVN_ERR_INVALID_ARGUMENT;
                V3<S> la1 = C::vec3(jc.local_anchor1, k), la2 = C::vec3(jc.local_anchor2, k);
                Quat<S> lb1 = C::quat_or_identity(jc.local_basis1, k), lb2 = C::quat_or_identity(jc.local_basis2, k);
                V3<S> com1 = C::vec3_or(bc.center_of_mass, j.body1, V3<S>{0, 0, 0});
                V3<S> com2 = C::vec3_or(bc.center_of_mass, j.body2, V3<S>{0, 0, 0});
                Quat<S> q1 = rot0[j.body1], q2 = rot0[j.body2];
                V3<S> default_axis = t == AVN_JOINT_REVOLUTE ? V3<S>{0, 0, 1} : (t == AVN_JOINT_SPHERICAL ? V3<S>{0, 1, 0} : V3<S>{1, 0, 0});
                V3<S> axis = C::vec3_or(jc.axis, k, default_axis);
                j.limit_enabled = jc.limit_enabled ? jc.limit_enabled[k] : 0;
                j.limit_min = C::scalar_or(jc.limit_min, k, 0);
                j.limit_max = C::scalar_or(jc.limit_max, k, 0);
                j.limit2_min = C::scalar_or(jc.limit2_min, k, 0);
                j.limit2_max = C::scalar_or(jc.limit2_max, k, 0);
                j.c0 = C::scalar_or(jc.compliance0, k, 0);
                j.c1 = C::scalar_or(jc.compliance1, k, 0);
                j.c2 = C::scalar_or(jc.compliance2, k, 0);
                j.damping = jc.damping_enabled && jc.damping_enabled[k];
                j.damping_linear = C::scalar_or(jc.damping_linear, k, 0);
                j.damping_angular = C::scalar_or(jc.damping_angular, k, 0);
                V3<S> cd = (pos0[j.body2] - pos0[j.body1]) + (rotate(q2, com2) - rotate(q1, com1));
                j.center_difference = cd;
                if (t == AVN_JOINT_SPHERICAL) {
                    // spherical.rs:45-82 uses rotation MATRICES for the anchors and axes
                    Mat3<S> r1 = mat3_from_quat(q1), r2 = mat3_from_quat(q2);
                    j.world_r1 = mul(r1, la1 - com1);
                    j.world_r2 = mul(r2, la2 - com2);
                    V3<S> swing_axis = any_orthonormal_vector(axis);
                    j.a1 = mul(r1, rotate(lb1, swing_axis));
                    j.a2 = mul(r2, rotate(lb2, swing_axis));
                    j.b1 = mul(r1, rotate(lb1, axis));
                    j.b2 = mul(r2, rotate(lb2, axis));
                } else {
                    // point_constraint.rs:38-51 / distance.rs:35-54 / prismatic.rs:43-77
                    j.world_r1 = rotate(q1, la1 - com1);
                    j.world_r2 = rotate(q2, la2 - com2);
                }
                if (t == AVN_JOINT_FIXED || t == AVN_JOINT_PRISMATIC) {
                    // fixed_angle_constraint.rs:38-57: (q1*b1) * (q2*b2)^-1
                    j.rotation_difference = mul(mul(q1, lb1), inverse(mul(q2, lb2)));
                }
                if (t == AVN_JOINT_REVOLUTE) {
                    // revolute.rs:83-88: `*rotation * local_basis * axis` = (Rotation * Quat) * Vec3
                    Quat<S> f1 = mul(q1, lb1), f2 = mul(q2, lb2);
                    V3<S> ortho = any_orthonormal_vector(axis);
                    j.a1 = rotate(f1, axis);
                    j.a2 = rotate(f2, axis);
                    j.b1 = rotate(f1, ortho);
                    j.b2 = rotate(f2, ortho);
                }
                if (t == AVN_JOINT_PRISMATIC) j.a1 = rotate(mul(q1, lb1), axis);  // prismatic.rs:76
                w.joints.push_back(j);
            }
        }
    }

    // ---- update_contact_softness (solver/plugin.rs:326-350)
    {
        S max_hz = S(1) / (dt * S(2));
        S hz = S(prm.contact_frequency_factor) * std::fmin(max_hz, S(0.25) / h);
        w.soft_dynamic = softness_coefficients<S>(S(prm.contact_damping_ratio), hz, h);
        w.soft_non_dynamic = softness_coefficients<S>(S(prm.contact_damping_ratio), S(2) * hz, h);
    }

    // ---- prepare_contact_constraints (solver/plugin.rs:363-448)
    if (mc && mc->count) {
        const SolverBodyInertia<S> dummy_inertia;
        for (int col = 0; col < AVN_GRAPH_COLOR_COUNT; ++col) {
            for (uint32_t mi = mc->color_offsets[col]; mi < mc->color_offsets[col + 1]; ++mi) {
                int32_t b1 = mc->body1[mi], b2 = mc->body2[mi];
                bool dyn1 = b1 >= 0 && (bc.kind ? bc.kind[b1] == AVN_BODY_DYNAMIC : true);
                bool dyn2 = b2 >= 0 && (bc.kind ? bc.kind[b2] == AVN_BODY_DYNAMIC : true);
                if (!dyn1 && !dyn2) continue;
                const SolverBodyInertia<S>& in1 = (b1 >= 0 && has_sb[b1]) ? w.inertias[b1] : dummy_inertia;
                const SolverBodyInertia<S>& in2 = (b2 >= 0 && has_sb[b2]) ? w.inertias[b2] : dummy_inertia;
                V3<S> v1 = b1 >= 0 ? linvel0[b1] : V3<S>{0, 0, 0};
                V3<S> v2 = b2 >= 0 ? linvel0[b2] : V3<S>{0, 0, 0};
                if (mc->point_offsets[mi + 1] - mc->point_offsets[mi] > AVN_MAX_MANIFOLD_POINTS) return AVN_ERR_INVALID_ARGUMENT;
                ContactConstraint<S> c =
                    generate_constraint<S>(b1, b2, in1, in2, v1, v2, *mc, mi, prm.match_contacts != 0, w.soft_dynamic, w.soft_non_dynamic);
                if (c.npoints > 0) w.constraints[col].push_back(c);
            }
        }
    }

    // ---- pre_process_velocity_increments (integrator/mod.rs:260-313); delta_secs = Time<Substeps>
    pool.par_for(B, 1, [&](size_t a, size_t e) {
        const V3<S> gravity{S(prm.gravity[0]), S(prm.gravity[1]), S(prm.gravity[2])};
        for (size_t i = a; i < e; ++i) {
            VelocityIntegrationData<S>& vi = w.integ[i];
            vi.linear_increment = C::vec3_or(bc.linear_acceleration, i, V3<S>{0, 0, 0});
            vi.angular_increment = C::vec3_or(bc.angular_acceleration, i, V3<S>{0, 0, 0});
            uint8_t kind = bc.kind ? bc.kind[i] : uint8_t(AVN_BODY_DYNAMIC);
            if (kind != AVN_BODY_DYNAMIC) continue;
            uint8_t locked = bc.locked_axes ? bc.locked_axes[i] : 0;
            vi.linear_damping_rhs = S(1) / (S(1) + h * C::scalar_or(bc.linear_damping, i, 0));
            vi.angular_damping_rhs = S(1) / (S(1) + h * C::scalar_or(bc.angular_damping, i, 0));
            vi.linear_increment += gravity * C::scalar_or(bc.gravity_scale, i, 1);
            if (locked & AVN_LOCK_TRANSLATION_X) vi.linear_increment.x = 0;
            if (locked & AVN_LOCK_TRANSLATION_Y) vi.linear_increment.y = 0;
            if (locked & AVN_LOCK_TRANSLATION_Z) vi.linear_increment.z = 0;
            if (locked & AVN_LOCK_ROTATION_X) vi.angular_increment.x = 0;
            if (locked & AVN_LOCK_ROTATION_Y) vi.angular_increment.y = 0;
            if (locked & AVN_LOCK_ROTATION_Z) vi.angular_increment.z = 0;
            vi.linear_increment *= h;
            vi.angular_increment *= h;
        }
    });

        max_overlap_solve_speed = S(prm.max_overlap_solve_speed) * S(prm.length_unit);
        warm_coeff = S(prm.warm_start_coefficient);
        pre_dp.resize(B);
        pre_dq.resize(B);
        have_joints = !w.joints.empty();
        iters = prm.solver_iterations ? prm.solver_iterations : 1;
        return AVN_OK;
    }

    // one iteration of run_substep_schedule (solver/schedule.rs:194-213)
    void substep() {
    // integrate_velocities (integrator/mod.rs:343-391)
    pool.par_for(B, 1, [&](size_t a, size_t e) {
        for (size_t i = a; i < e; ++i) {
            if (!has_sb[i]) continue;
            if (bc.integration_flags && (bc.integration_flags[i] & AVN_CUSTOM_VELOCITY_INTEGRATION)) continue;
            SolverBody<S>& sb = w.bodies[i];
            if (sb.is_kinematic()) continue;
            const VelocityIntegrationData<S>& vi = w.integ[i];
            sb.linear_velocity *= vi.linear_damping_rhs;
            sb.angular_velocity *= vi.angular_damping_rhs;
            sb.linear_velocity += vi.linear_increment;
            sb.angular_velocity += vi.angular_increment;
            if (sb.is_gyroscopic()) {
                Quat<S> rotation = mul(sb.delta_rotation, rot0[i]);
                solve_gyroscopic_torque(sb.angular_velocity, rotation, C::sym3(bc.inverse_inertia_local, i), h);
            }
        }
    });
    // clamp_velocities (integrator/mod.rs:467-500)
    if (bc.max_linear_speed)
        for (size_t i = 0; i < B; ++i) {
            S ms = C::scalar(bc.max_linear_speed, i);
            if (!has_sb[i] || !std::isfinite(ms)) continue;
            S l2 = length_squared(w.bodies[i].linear_velocity);
            if (l2 > ms * ms) w.bodies[i].linear_velocity *= ms / std::sqrt(l2);
        }
    if (bc.max_angular_speed)
        for (size_t i = 0; i < B; ++i) {
            S ms = C::scalar(bc.max_angular_speed, i);
            if (!has_sb[i] || !std::isfinite(ms)) continue;
            S l2 = length_squared(w.bodies[i].angular_velocity);
            if (l2 > ms * ms) w.bodies[i].angular_velocity *= ms / std::sqrt(l2);
        }
    // x-slab partition: the reference point of this substep's constraint impulses on the boundary bodies
    for (size_t k = 0; k < bnd_body.size(); ++k) {
        ref_lin[k] = w.bodies[bnd_body[k]].linear_velocity;
        ref_ang[k] = w.bodies[bnd_body[k]].angular_velocity;
    }
    // warm_start (solver/plugin.rs:453-482)
    for_each_color<S>(w, pool, has_sb, [&](ContactConstraint<S>& c, SolverBody<S>& b1, SolverBody<S>& b2, const SolverBodyInertia<S>& i1,
                                           const SolverBodyInertia<S>& i2) { warm_start_constraint(c, b1, b2, i1, i2, warm_coeff); });
    // solve_contacts::<true> (solver/plugin.rs:531-581)
    for (uint32_t it = 0; it < iters; ++it)
        for_each_color<S>(w, pool, has_sb, [&](ContactConstraint<S>& c, SolverBody<S>& b1, SolverBody<S>& b2, const SolverBodyInertia<S>& i1,
                                               const SolverBodyInertia<S>& i2) { solve_constraint(c, b1, b2, i1, i2, h, true, max_overlap_solve_speed); });
    // integrate_positions (integrator/mod.rs:503-535)
    pool.par_for(B, 1, [&](size_t a, size_t e) {
        for (size_t i = a; i < e; ++i) {
            if (!has_sb[i]) continue;
            if (bc.integration_flags && (bc.integration_flags[i] & AVN_CUSTOM_POSITION_INTEGRATION)) continue;
            SolverBody<S>& sb = w.bodies[i];
            sb.delta_position += sb.linear_velocity * h;
            sb.delta_rotation = mul(quat_from_scaled_axis(sb.angular_velocity * h), sb.delta_rotation);
        }
    });
    // update_solver_body_angular_inertia recomputes the same value (SURVEY D8) — nothing to do.
    // solve_contacts::<false> (relax)
    for_each_color<S>(w, pool, has_sb, [&](ContactConstraint<S>& c, SolverBody<S>& b1, SolverBody<S>& b2, const SolverBodyInertia<S>& i1,
                                           const SolverBodyInertia<S>& i2) { solve_constraint(c, b1, b2, i1, i2, h, false, max_overlap_solve_speed); });
    // XPBD (xpbd/plugin.rs:58-94). With no joints the projection is an exact no-op (SURVEY A7).
    if (have_joints) {
        for (size_t i = 0; i < B; ++i) { pre_dp[i] = w.bodies[i].delta_position; pre_dq[i] = w.bodies[i].delta_rotation; }
        for (JointData<S>& j : w.joints) {
            SolverBody<S> d1, d2;  // SolverBody::default()
            SolverBody<S>* b1 = &d1; SolverBody<S>* b2 = &d2;
            const SolverBodyInertia<S>* i1 = &dummy_inertia; const SolverBodyInertia<S>* i2 = &dummy_inertia;
            if (has_sb[j.body1]) { b1 = &w.bodies[j.body1]; i1 = &w.inertias[j.body1]; }
            if (has_sb[j.body2]) { b2 = &w.bodies[j.body2]; i2 = &w.inertias[j.body2]; }
            int rel = int(i1->dominance) - int(i2->dominance);
            if (rel > 0) i1 = &dummy_inertia; else if (rel < 0) i2 = &dummy_inertia;
            solve_joint(j, *b1, *b2, *i1, *i2, h);
        }
        // project_linear_velocity / project_angular_velocity (xpbd/plugin.rs:192-240)
        for (size_t i = 0; i < B; ++i) {
            if (!has_sb[i]) continue;
            SolverBody<S>& sb = w.bodies[i];
            sb.linear_velocity += (sb.delta_position - pre_dp[i]) / h;
        }
        for (size_t i = 0; i < B; ++i) {
            if (!has_sb[i]) continue;
            SolverBody<S>& sb = w.bodies[i];
            Quat<S> dr = mul(sb.delta_rotation, inverse(pre_dq[i]));
            V3<S> nav = S(2) * xyz(dr) / h;
            if (dr.w < S(0)) nav = -nav;
            sb.angular_velocity += nav;
        }
        // joint_damping<T> (solver/plugin.rs:759-806).  Each system run (one joint type, one substep) owns one dummy_body1 and one
        // dummy_body2 for the joint ends without a SolverBody.  The dummy is not kinematic, so delta_omega is written into it and the
        // next such joint of the run reads it; its linear velocity stays zero (effective inverse mass 0).
        SolverBody<S> d1, d2;
        int run_type = -1;
        for (JointData<S>& j : w.joints) {
            if (!j.damping) continue;
            if (j.type != run_type) { d1 = SolverBody<S>(); d2 = SolverBody<S>(); run_type = j.type; }
            SolverBody<S>* b1 = &d1; SolverBody<S>* b2 = &d2;
            const SolverBodyInertia<S>* i1 = &dummy_inertia; const SolverBodyInertia<S>* i2 = &dummy_inertia;
            if (has_sb[j.body1]) { b1 = &w.bodies[j.body1]; i1 = &w.inertias[j.body1]; }
            if (has_sb[j.body2]) { b2 = &w.bodies[j.body2]; i2 = &w.inertias[j.body2]; }
            V3<S> delta_omega = (b2->angular_velocity - b1->angular_velocity) * std::fmin(j.damping_angular * h, S(1));
            if (!b1->is_kinematic()) b1->angular_velocity += delta_omega;
            if (!b2->is_kinematic()) b2->angular_velocity -= delta_omega;
            V3<S> delta_v = (b2->linear_velocity - b1->linear_velocity) * std::fmin(j.damping_linear * h, S(1));
            V3<S> w1 = i1->effective_inv_mass(), w2 = i2->effective_inv_mass();
            V3<S> p = delta_v * recip_or_zero(w1 + w2);
            b1->linear_velocity += p * w1;
            b2->linear_velocity -= p * w2;
        }
    }
    }

    void restitution() {
    // ---- solve_restitution (solver/plugin.rs:630-718)
    {
        S threshold = S(prm.restitution_threshold) * S(prm.length_unit);
        for_each_color<S>(w, pool, has_sb, [&](ContactConstraint<S>& c, SolverBody<S>& b1, SolverBody<S>& b2, const SolverBodyInertia<S>& i1,
                                               const SolverBodyInertia<S>& i2) {
            if (c.restitution == S(0)) return;
            uint32_t n = c.npoints > 1 ? prm.restitution_iterations : 1;
            for (uint32_t k = 0; k < n; ++k) apply_restitution(c, b1, b2, i1, i2, threshold);
        });
    }
    }

    int finalize() {
    // ---- writeback_solver_bodies (solver_body/plugin.rs:255-284)
    pool.par_for(B, 1, [&](size_t a, size_t e) {
        for (size_t i = a; i < e; ++i) {
            if (!has_sb[i]) continue;
            const SolverBody<S>& sb = w.bodies[i];
            V3<S> com = C::vec3_or(bc.center_of_mass, i, V3<S>{0, 0, 0});
            V3<S> old_world_com = rotate(rot0[i], com);
            Quat<S> rot = fast_renormalize(mul(sb.delta_rotation, rot0[i]));
            V3<S> new_world_com = rotate(rot, com);
            C::set_vec3(bc.position, i, pos0[i] + (sb.delta_position + old_world_com - new_world_com));
            C::set_quat(bc.rotation, i, rot);
            C::set_vec3(bc.linear_velocity, i, sb.linear_velocity);
            C::set_vec3(bc.angular_velocity, i, sb.angular_velocity);
        }
    });

    // ---- writeback_joint_forces (xpbd/plugin.rs:242-260)
    if (js) {
        // `time: Res<Time>` in SolverSystems::Finalize is Time<Physics> again (run_substep_schedule restores it, solver/schedule.rs:211-212),
        // so delta_seconds_adjusted() is the FULL step dt here, not the substep h: f = sum(lambda) * substeps / dt^2.
        S rhs = recip_or_zero(dt * dt) * S(prm.substeps);
        for (const JointData<S>& j : w.joints) {
            AvnJointColumns& jc = js->types[j.type];
            if (jc.force) C::set_vec3(jc.force, j.index_in_type, j.total_position_lagrange * rhs);
            if (jc.torque) C::set_vec3(jc.torque, j.index_in_type, (j.total_rot_lagrange_a + j.total_rot_lagrange_b) * rhs);
        }
    }

    // ---- store_contact_impulses (solver/plugin.rs:722-755)
    if (mc) {
        for (int col = 0; col < AVN_GRAPH_COLOR_COUNT; ++col)
            for (const ContactConstraint<S>& c : w.constraints[col])
                for (int k = 0; k < c.npoints; ++k) {
                    uint32_t p = c.first_point + k;
                    const ContactPointC<S>& pt = c.points[k];
                    static_cast<S*>(mc->warm_start_normal_impulse)[p] = pt.impulse;
                    S* wt = static_cast<S*>(mc->warm_start_tangent_impulse) + 2 * p;
                    wt[0] = pt.has_tangent ? pt.t_impulse.x : S(0);
                    wt[1] = pt.has_tangent ? pt.t_impulse.y : S(0);
                    static_cast<S*>(mc->normal_impulse)[p] = pt.total_impulse;
                }
    }
    return AVN_OK;
    }

    // ---- boundary exchange of the x-slab partition: the same record layout and arithmetic as boundary_*_kernel (solver_host.cu)
    int set_boundary(const AvnBoundary& b) {
        bnd_body.assign(b.body, b.body + b.count);
        bnd_source.assign(b.source, b.source + size_t(b.count) * b.world);
        bnd_owner.assign(b.owner_rank, b.owner_rank + b.count);
        for (int x : bnd_body)
            if (x < 0 || size_t(x) >= B) return AVN_ERR_INVALID_ARGUMENT;
        ref_lin.assign(b.count, V3<S>{0, 0, 0});
        ref_ang.assign(b.count, V3<S>{0, 0, 0});
        bnd_rank = int(b.rank);
        bnd_world = int(b.world);
        bnd_slots = b.record_count;
        return AVN_OK;
    }
    void boundary_snapshot() {
        for (size_t k = 0; k < bnd_body.size(); ++k) {
            ref_lin[k] = w.bodies[bnd_body[k]].linear_velocity;
            ref_ang[k] = w.bodies[bnd_body[k]].angular_velocity;
        }
    }
    void boundary_pack(S* table) const {
        std::fill(table, table + bnd_slots * AVN_BOUNDARY_RECORD_SCALARS, S(0));
        for (size_t k = 0; k < bnd_body.size(); ++k) {
            const SolverBody<S>& sb = w.bodies[bnd_body[k]];
            S* r = table + k * AVN_BOUNDARY_RECORD_SCALARS;
            const bool owner = bnd_owner[k] == bnd_rank;
            r[0] = sb.linear_velocity.x - ref_lin[k].x; r[1] = sb.linear_velocity.y - ref_lin[k].y; r[2] = sb.linear_velocity.z - ref_lin[k].z; r[3] = S(1);
            r[4] = sb.angular_velocity.x - ref_ang[k].x; r[5] = sb.angular_velocity.y - ref_ang[k].y; r[6] = sb.angular_velocity.z - ref_ang[k].z;
            r[7] = owner ? S(1) : S(0);
            if (owner) {
                r[8] = sb.delta_position.x; r[9] = sb.delta_position.y; r[10] = sb.delta_position.z; r[11] = S(0);
                r[12] = sb.delta_rotation.x; r[13] = sb.delta_rotation.y; r[14] = sb.delta_rotation.z; r[15] = sb.delta_rotation.w;
            }
        }
    }
    void boundary_apply(const S* gathered) {
        for (size_t k = 0; k < bnd_body.size(); ++k) {
            SolverBody<S>& sb = w.bodies[bnd_body[k]];
            V3<S> l = ref_lin[k], a = ref_ang[k];
            for (int r = 0; r < bnd_world; ++r) {
                const int idx = bnd_source[k * size_t(bnd_world) + r];
                if (idx < 0) continue;
                const S* rec = gathered + (size_t(r) * bnd_slots + size_t(idx)) * AVN_BOUNDARY_RECORD_SCALARS;
                l.x = l.x + rec[0]; l.y = l.y + rec[1]; l.z = l.z + rec[2];
                a.x = a.x + rec[4]; a.y = a.y + rec[5]; a.z = a.z + rec[6];
            }
            sb.linear_velocity = l;
            sb.angular_velocity = a;
            const S* own = gathered + (size_t(bnd_owner[k]) * bnd_slots + size_t(bnd_source[k * size_t(bnd_world) + bnd_owner[k]])) * AVN_BOUNDARY_RECORD_SCALARS;
            sb.delta_position = V3<S>{own[8], own[9], own[10]};
            sb.delta_rotation = Quat<S>{own[12], own[13], own[14], own[15]};
        }
    }
    bool needs_restitution() const {
        for (int col = 0; col < AVN_GRAPH_COLOR_COUNT; ++col)
            for (const ContactConstraint<S>& c : w.constraints[col])
                if (c.restitution != S(0)) return true;
        return false;
    }
};

template <class S>
int solver_step(const AvnStepParams& prm, AvnBodyColumns& bc, AvnManifoldColumns* mc, AvnJointSet* js, int threads) {
    StepState<S> st(prm, bc, mc, js, threads);
    int rc = st.prepare();
    if (rc != AVN_OK) return rc;
    for (uint32_t sub = 0; sub < prm.substeps; ++sub) st.substep();
    st.restitution();
    return st.finalize();
}

template int solver_step<float>(const AvnStepParams&, AvnBodyColumns&, AvnManifoldColumns*, AvnJointSet*, int);
template int solver_step<double>(const AvnStepParams&, AvnBodyColumns&, AvnManifoldColumns*, AvnJointSet*, int);

// type-erased handle for the resumable entry points
struct StepHandle {
    uint32_t bits;
    void* state;
};
template <class F32, class F64> static auto dispatch(StepHandle* h, F32 f32, F64 f64) {
    return h->bits == 32 ? f32(static_cast<StepState<float>*>(h->state)) : f64(static_cast<StepState<double>*>(h->state));
}

}  // namespace orc

extern "C" {
int orc_solver_step(uint32_t scalar_bits, const AvnStepParams* prm, AvnBodyColumns* bodies, AvnManifoldColumns* manifolds,
                    AvnJointSet* joints, int threads) {
    if (!prm || !bodies) return AVN_ERR_INVALID_ARGUMENT;
    if (scalar_bits == 32) return orc::solver_step<float>(*prm, *bodies, manifolds, joints, threads);
    if (scalar_bits == 64) return orc::solver_step<double>(*prm, *bodies, manifolds, joints, threads);
    return AVN_ERR_INVALID_ARGUMENT;
}

// ---- the stage in pieces (tests of the x-slab partition): the column buffers must stay alive until orc_step_finish
#define ORC_EACH(h, expr) orc::dispatch((h), [&](auto* st) { return (expr); }, [&](auto* st) { return (expr); })
void* orc_step_begin(uint32_t scalar_bits, const AvnStepParams* prm, AvnBodyColumns* bodies, AvnManifoldColumns* manifolds, AvnJointSet* joints,
                     int threads) {
    if (!prm || !bodies || (scalar_bits != 32 && scalar_bits != 64)) return nullptr;
    auto* h = new orc::StepHandle{scalar_bits, nullptr};
    int rc;
    if (scalar_bits == 32) {
        auto* st = new orc::StepState<float>(*prm, *bodies, manifolds, joints, threads);
        h->state = st;
        rc = st->prepare();
    } else {
        auto* st = new orc::StepState<double>(*prm, *bodies, manifolds, joints, threads);
        h->state = st;
        rc = st->prepare();
    }
    if (rc != AVN_OK) {
        ORC_EACH(h, (delete st, 0));
        delete h;
        return nullptr;
    }
    return h;
}
int orc_step_substeps(void* handle, uint32_t count) {
    auto* h = static_cast<orc::StepHandle*>(handle);
    for (uint32_t i = 0; i < count; ++i) ORC_EACH(h, (st->substep(), 0));
    return AVN_OK;
}
int orc_step_restitution(void* handle) { return ORC_EACH(static_cast<orc::StepHandle*>(handle), (st->restitution(), int(AVN_OK))); }
int orc_step_needs_restitution(void* handle) { return ORC_EACH(static_cast<orc::StepHandle*>(handle), int(st->needs_restitution())); }
int orc_step_set_boundary(void* handle, const AvnBoundary* b) { return ORC_EACH(static_cast<orc::StepHandle*>(handle), st->set_boundary(*b)); }
int orc_step_boundary_snapshot(void* handle) { return ORC_EACH(static_cast<orc::StepHandle*>(handle), (st->boundary_snapshot(), int(AVN_OK))); }
int orc_step_boundary_pack(void* handle, void* table) {
    auto* h = static_cast<orc::StepHandle*>(handle);
    if (h->bits == 32) static_cast<orc::StepState<float>*>(h->state)->boundary_pack(static_cast<float*>(table));
    else static_cast<orc::StepState<double>*>(h->state)->boundary_pack(static_cast<double*>(table));
    return AVN_OK;
}
int orc_step_boundary_apply(void* handle, const void* gathered) {
    auto* h = static_cast<orc::StepHandle*>(handle);
    if (h->bits == 32) static_cast<orc::StepState<float>*>(h->state)->boundary_apply(static_cast<const float*>(gathered));
    else static_cast<orc::StepState<double>*>(h->state)->boundary_apply(static_cast<const double*>(gathered));
    return AVN_OK;
}
// writeback + store impulses into the column buffers given to orc_step_begin, then frees the handle
int orc_step_finish(void* handle) {
    auto* h = static_cast<orc::StepHandle*>(handle);
    int rc = ORC_EACH(h, st->finalize());
    ORC_EACH(h, (delete st, 0));
    delete h;
    return rc;
}
}
