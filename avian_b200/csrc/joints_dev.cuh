// XPBD joints on the device: prepare (xpbd/plugin.rs:125-142 + each joint's `prepare`), one solve per joint per
// substep (xpbd/plugin.rs:145-189 + each joint's `solve`), velocity projection (xpbd/plugin.rs:192-240),
// joint damping (solver/plugin.rs:759-806) and force writeback (xpbd/plugin.rs:242-260).
//
// The reference solves joints serially (type order Fixed, Revolute, Spherical, Prismatic, Distance, then ECS
// table order).  The device reproduces that result exactly with an order-preserving LEVEL SCHEDULE built on the
// host: level(j) = 1 + max level of the earlier joints that share a non-dummy body with j.  Joints in one level
// touch disjoint bodies, so a level is one conflict-free parallel phase, and running levels in order is
// equivalent to the serial sweep.
#pragma once
#include "solver_dev.cuh"

namespace avn {

enum { JI_TYPE_MASK = 0xff, JI_LIMIT_SHIFT = 8, JI_DAMPING = 1 << 16, JI_ZERO1 = 1 << 24, JI_ZERO2 = 1 << 25 };

template <class S> __device__ __forceinline__ Q4<S> to_q(Vec4<S> v) { Q4<S> q; q.x = v.x; q.y = v.y; q.z = v.z; q.w = v.w; return q; }
template <class S> __device__ __forceinline__ Vec4<S> from_q(Q4<S> q) { return mk4<S>(q.x, q.y, q.z, q.w); }

// `slot` = position in the level schedule; (type, k) = the joint's place in the ABI columns
template <class S>
__device__ void prepare_joint_item(const DevSolver<S>& d, int slot) {
    const int t = d.j_src_type[slot], k = d.j_src_index[slot];
    const int b1 = d.jbody1[t][k], b2 = d.jbody2[t][k];
    const S* const* col = d.jc[t];
    V3<S> la1 = ldv3(col[0], k), la2 = ldv3(col[1], k);
    Q4<S> lb1 = col[2] ? ldq(col[2], k) : qidentity<S>(), lb2 = col[3] ? ldq(col[3], k) : qidentity<S>();
    V3<S> def_axis = t == AVN_JOINT_REVOLUTE ? mk3<S>(0, 0, 1) : (t == AVN_JOINT_SPHERICAL ? mk3<S>(0, 1, 0) : mk3<S>(1, 0, 0));
    V3<S> axis = col[4] ? ldv3(col[4], k) : def_axis;
    S lmin = col[5] ? col[5][k] : S(0), lmax = col[6] ? col[6][k] : S(0);
    S l2min = col[7] ? col[7][k] : S(0), l2max = col[8] ? col[8][k] : S(0);
    S c0 = col[9] ? col[9][k] : S(0), c1 = col[10] ? col[10][k] : S(0), c2 = col[11] ? col[11][k] : S(0);
    int limit_en = d.jlimit_en[t] ? d.jlimit_en[t][k] : 0;
    int damping = (d.jdamp_en[t] && d.jdamp_en[t][k]) ? 1 : 0;
    V3<S> com1 = ldv3_or0(d.com, b1), com2 = ldv3_or0(d.com, b2);
    Q4<S> q1 = ldq(d.rotation, b1), q2 = ldq(d.rotation, b2);
    V3<S> cd = (ldv3(d.position, b2) - ldv3(d.position, b1)) + (qrot(q2, com2) - qrot(q1, com1));
    V3<S> wr1, wr2, A1 = zero3<S>(), A2 = zero3<S>(), B1 = zero3<S>(), B2 = zero3<S>();
    Q4<S> rd = qidentity<S>();
    if (t == AVN_JOINT_SPHERICAL) {  // spherical.rs:45-82 (rotation matrices)
        M33<S> r1 = m33_from_quat(q1), r2 = m33_from_quat(q2);
        wr1 = mmul(r1, la1 - com1);
        wr2 = mmul(r2, la2 - com2);
        V3<S> swing = any_orthonormal(axis);
        A1 = mmul(r1, qrot(lb1, swing));
        A2 = mmul(r2, qrot(lb2, swing));
        B1 = mmul(r1, qrot(lb1, axis));
        B2 = mmul(r2, qrot(lb2, axis));
    } else {  // point_constraint.rs:38-51, distance.rs:35-54, prismatic.rs:43-77
        wr1 = qrot(q1, la1 - com1);
        wr2 = qrot(q2, la2 - com2);
    }
    if (t == AVN_JOINT_FIXED || t == AVN_JOINT_PRISMATIC) rd = qmul(qmul(q1, lb1), qconj(qmul(q2, lb2)));  // fixed_angle_constraint.rs:38-57
    if (t == AVN_JOINT_REVOLUTE) {  // revolute.rs:83-88
        Q4<S> f1 = qmul(q1, lb1), f2 = qmul(q2, lb2);
        V3<S> ortho = any_orthonormal(axis);
        A1 = qrot(f1, axis); A2 = qrot(f2, axis); B1 = qrot(f1, ortho); B2 = qrot(f2, ortho);
    }
    if (t == AVN_JOINT_PRISMATIC) A1 = qrot(qmul(q1, lb1), axis);  // prismatic.rs:76
    // dominance of the two inertias (xpbd/plugin.rs:176-180)
    int f1 = as_int(ld4(&d.inr[2 * b1]).y), f2 = as_int(ld4(&d.inr[2 * b2]).y);
    int rel = (f1 >> BF_DOMINANCE_SHIFT) - (f2 >> BF_DOMINANCE_SHIFT);
    int info = t | (limit_en << JI_LIMIT_SHIFT) | (damping ? JI_DAMPING : 0);
    if (rel > 0 || !(f1 & BF_HAS_SOLVER_BODY)) info |= JI_ZERO1;
    if (rel < 0 || !(f2 & BF_HAS_SOLVER_BODY)) info |= JI_ZERO2;
    const size_t JP = size_t(d.Jpad);
    Vec4<S>* j = d.jnt + slot;
    st4(&j[JP_IDX * JP], mk4<S>(int_as(S(0), b1), int_as(S(0), b2), int_as(S(0), info), int_as(S(0), k)));
    st4(&j[JP_R1 * JP], mk4<S>(wr1.x, wr1.y, wr1.z, c0));
    st4(&j[JP_R2 * JP], mk4<S>(wr2.x, wr2.y, wr2.z, c1));
    st4(&j[JP_CD * JP], mk4<S>(cd.x, cd.y, cd.z, c2));
    st4(&j[JP_RD * JP], from_q(rd));
    st4(&j[JP_A1 * JP], mk4<S>(A1.x, A1.y, A1.z, lmin));
    st4(&j[JP_A2 * JP], mk4<S>(A2.x, A2.y, A2.z, lmax));
    st4(&j[JP_B1 * JP], mk4<S>(B1.x, B1.y, B1.z, l2min));
    st4(&j[JP_B2 * JP], mk4<S>(B2.x, B2.y, B2.z, l2max));
    st4(&j[JP_LP * JP], mk4<S>(S(0), S(0), S(0), d.jdamp_lin[t] ? d.jdamp_lin[t][k] : S(0)));
    st4(&j[JP_LA * JP], mk4<S>(S(0), S(0), S(0), d.jdamp_ang[t] ? d.jdamp_ang[t][k] : S(0)));
    st4(&j[JP_LB * JP], mk4<S>(S(0), S(0), S(0), S(0)));
}

// the mutable part of a SolverBody a joint touches + its (possibly dominated) inertia
template <class S> struct JBody {
    V3<S> dp; Q4<S> dq; BodyInertia<S> in;
};

// xpbd/mod.rs:393-413 (every call site passes lagrange = 0, SURVEY A6)
template <class S> __device__ __forceinline__ S lagrange_update(S c, S w1, S w2, S compliance, S dt) {
    S w_sum = w1 + w2;
    if (w_sum <= Eps<S>::v) return S(0);
    S tilde = compliance / (dt * dt);
    return (-c - tilde * S(0)) / (w_sum + tilde);
}
// positional_constraint.rs:63-76
template <class S> __device__ __forceinline__ S pos_w(S inv_mass, const Sym3<S>& ii, V3<S> r, V3<S> n) {
    V3<S> rxn = cross(r, n);
    return inv_mass + dot(rxn, smul(ii, rxn));
}
// positional_constraint.rs:9-50
template <class S> __device__ __forceinline__ void positional_impulse(JBody<S>& a, JBody<S>& b, V3<S> impulse, V3<S> r1, V3<S> r2, bool fast) {
    a.dp = a.dp + cmul(impulse, a.in.inv_mass);
    a.dq = qmul(q_from_scaled_axis(smul(a.in.ii, cross(r1, impulse)), fast), a.dq);
    b.dp = b.dp - cmul(impulse, b.in.inv_mass);
    b.dq = qmul(q_from_scaled_axis(smul(b.in.ii, cross(r2, -impulse)), fast), b.dq);
}
// angular_constraint.rs:149-194 + :52-97
template <class S> __device__ __forceinline__ V3<S> align_orientation(JBody<S>& a, JBody<S>& b, V3<S> rotation_difference, S compliance, S dt, bool fast) {
    S angle = len(rotation_difference);
    if (angle <= Eps<S>::v) return zero3<S>();
    V3<S> axis = rotation_difference / angle;
    S w1 = dot(axis, smul(a.in.ii, axis)), w2 = dot(axis, smul(b.in.ii, axis));
    S dl = lagrange_update(angle, w1, w2, compliance, dt);
    if (!(avn_abs(dl) <= Eps<S>::v)) {
        V3<S> impulse = -dl * axis;
        a.dq = qmul(q_from_scaled_axis(smul(a.in.ii, impulse), fast), a.dq);
        b.dq = qmul(q_from_scaled_axis(smul(b.in.ii, -impulse), fast), b.dq);
    }
    return dl * axis;
}
// joints/mod.rs:427-473
template <class S> __device__ __forceinline__ bool angle_limit(S lo, S hi, V3<S> limit_axis, V3<S> ax1, V3<S> ax2, S max_corr, V3<S>& out, bool fast) {
    const S PI = S(3.14159265358979323846264338327950288), TAU = S(6.28318530717958647692528676655900577);
    S phi = avn_asin(dot(cross(ax1, ax2), limit_axis));
    if (dot(ax1, ax2) < S(0)) phi = PI - phi;
    if (phi > PI) phi -= TAU;
    if (phi < lo || phi > hi) {
        phi = phi < lo ? lo : (phi > hi ? hi : phi);
        Q4<S> rot = q_from_axis_angle(limit_axis, phi, fast);
        out = clamp_len_max(cross(qrot(rot, ax1), ax2), max_corr);
        return true;
    }
    return false;
}
// joints/mod.rs:342-357
template <class S> __device__ __forceinline__ V3<S> limit_along_axis(S lo, S hi, V3<S> sep, V3<S> axis) {
    S a = dot(sep, axis);
    if (a < lo) return axis * (lo - a);
    if (a > hi) return (-axis) * (a - hi);
    return zero3<S>();
}
// shared/point_constraint.rs:53-108
template <class S> __device__ __forceinline__ void point_solve(JBody<S>& a, JBody<S>& b, V3<S> wr1, V3<S> wr2, V3<S> cd, S compliance, S dt, V3<S>& total, bool fast) {
    V3<S> r1 = qrot(a.dq, wr1), r2 = qrot(b.dq, wr2);
    V3<S> sep = ((b.dp - a.dp) + (r2 - r1)) + cd;
    S m2 = len2(sep);
    if (m2 == S(0)) return;
    S mag = avn_sqrt(m2);
    V3<S> dir = (-sep) / mag;
    S w1 = pos_w(max_elem(a.in.inv_mass), a.in.ii, r1, dir), w2 = pos_w(max_elem(b.in.inv_mass), b.in.ii, r2, dir);
    S dl = lagrange_update(mag, w1, w2, compliance, dt);
    V3<S> impulse = dl * dir;
    total = total + impulse;
    positional_impulse(a, b, impulse, r1, r2, fast);
}
// shared/fixed_angle_constraint.rs:59-97
template <class S> __device__ __forceinline__ void fixed_angle_solve(JBody<S>& a, JBody<S>& b, Q4<S> rd, S compliance, S dt, V3<S>& total, bool fast) {
    Q4<S> q = qmul(qmul(rd, a.dq), qconj(b.dq));
    V3<S> diff = S(-2) * qxyz(q);
    total = total + align_orientation(a, b, diff, compliance, dt, fast);
}

template <class S>
__device__ void solve_joint_item(const DevSolver<S>& d, int slot) {
    const size_t JP = size_t(d.Jpad);
    Vec4<S>* j = d.jnt + slot;
    Vec4<S> jidx = ld4(&j[JP_IDX * JP]);
    const int b1 = as_int(jidx.x), b2 = as_int(jidx.y), info = as_int(jidx.z);
    const int type = info & JI_TYPE_MASK, limit_en = (info >> JI_LIMIT_SHIFT) & 0xff;
    Vec4<S> R1 = ld4(&j[JP_R1 * JP]), R2 = ld4(&j[JP_R2 * JP]), CD = ld4(&j[JP_CD * JP]);
    Vec4<S> A1 = ld4(&j[JP_A1 * JP]), A2 = ld4(&j[JP_A2 * JP]), B1 = ld4(&j[JP_B1 * JP]), B2 = ld4(&j[JP_B2 * JP]);
    Vec4<S> LP = ld4(&j[JP_LP * JP]), LA = ld4(&j[JP_LA * JP]), LB = ld4(&j[JP_LB * JP]);
    JBody<S> a, b;
    // a joint whose body has no SolverBody works on a scratch SolverBody::default() (xpbd/plugin.rs:156-170)
    const bool real1 = !(info & JI_ZERO1) || (as_int(ld4(&d.inr[2 * b1]).y) & BF_HAS_SOLVER_BODY);
    const bool real2 = !(info & JI_ZERO2) || (as_int(ld4(&d.inr[2 * b2]).y) & BF_HAS_SOLVER_BODY);
    a.dp = real1 ? xyz(ld4(&d.dlt[2 * b1])) : zero3<S>();
    a.dq = real1 ? to_q(ld4(&d.dlt[2 * b1 + 1])) : qidentity<S>();
    b.dp = real2 ? xyz(ld4(&d.dlt[2 * b2])) : zero3<S>();
    b.dq = real2 ? to_q(ld4(&d.dlt[2 * b2 + 1])) : qidentity<S>();
    a.in = (info & JI_ZERO1) ? zero_inertia<S>() : unpack_inertia(ld4(&d.inr[2 * b1]), ld4(&d.inr[2 * b1 + 1]));
    b.in = (info & JI_ZERO2) ? zero_inertia<S>() : unpack_inertia(ld4(&d.inr[2 * b2]), ld4(&d.inr[2 * b2 + 1]));
    const bool fast = d.fast_trig != 0;
    const S dt = d.h;
    const S PI = S(3.14159265358979323846264338327950288);
    V3<S> tp = xyz(LP), ta = xyz(LA), tb = xyz(LB);
    const S c0 = R1.w, c1 = R2.w, c2 = CD.w;
    switch (type) {
        case AVN_JOINT_FIXED:  // fixed.rs:73-89
            fixed_angle_solve(a, b, to_q(ld4(&j[JP_RD * JP])), c1, dt, ta, fast);
            point_solve(a, b, xyz(R1), xyz(R2), xyz(CD), c0, dt, tp, fast);
            break;
        case AVN_JOINT_REVOLUTE: {  // revolute.rs:92-187
            V3<S> a1 = qrot(a.dq, xyz(A1)), a2 = qrot(b.dq, xyz(A2));
            ta = ta + align_orientation(a, b, cross(a1, a2), c1, dt, fast);
            if (limit_en & 1) {
                V3<S> la1 = qrot(a.dq, xyz(A1)), lb1 = qrot(a.dq, xyz(B1)), lb2 = qrot(b.dq, xyz(B2));
                V3<S> corr;
                if (angle_limit(A1.w, A2.w, la1, lb1, lb2, PI, corr, fast)) tb = tb + align_orientation(a, b, corr, c2, dt, fast);
            }
            point_solve(a, b, xyz(R1), xyz(R2), xyz(CD), c0, dt, tp, fast);
            break;
        }
        case AVN_JOINT_SPHERICAL: {  // spherical.rs:84-207
            point_solve(a, b, xyz(R1), xyz(R2), xyz(CD), c0, dt, tp, fast);
            if (limit_en & 1) {
                V3<S> a1 = qrot(a.dq, xyz(A1)), a2 = qrot(b.dq, xyz(A2));
                V3<S> n = cross(a1, a2);
                S nm = len(n);
                if (!(nm <= Eps<S>::v)) {
                    n = n / nm;
                    V3<S> corr;
                    if (angle_limit(A1.w, A2.w, n, a1, a2, PI, corr, fast)) ta = ta + align_orientation(a, b, corr, c1, dt, fast);
                }
            }
            if (limit_en & 2) {
                V3<S> a1 = qrot(a.dq, xyz(A1)), a2 = qrot(b.dq, xyz(A2));
                V3<S> n = a1 + a2;
                S nm = len(n);
                if (!(nm <= Eps<S>::v)) {
                    V3<S> tb1 = qrot(a.dq, xyz(B1)), tb2 = qrot(b.dq, xyz(B2));
                    n = n / nm;
                    V3<S> n1 = tb1 - dot(n, tb1) * n, n2 = tb2 - dot(n, tb2) * n;
                    S n1m = len(n1), n2m = len(n2);
                    if (!(n1m <= Eps<S>::v || n2m <= Eps<S>::v)) {
                        n1 = n1 / n1m;
                        n2 = n2 / n2m;
                        S max_corr = dot(a1, a2) > S(-0.5) ? S(2) * PI : dt;
                        V3<S> corr;
                        if (angle_limit(B1.w, B2.w, n, n1, n2, max_corr, corr, fast)) tb = tb + align_orientation(a, b, corr, c2, dt, fast);
                    }
                }
            }
            break;
        }
        case AVN_JOINT_PRISMATIC: {  // prismatic.rs:79-193
            fixed_angle_solve(a, b, to_q(ld4(&j[JP_RD * JP])), c1, dt, ta, fast);
            V3<S> r1 = qrot(a.dq, xyz(R1)), r2 = qrot(b.dq, xyz(R2));
            V3<S> axis1 = qrot(a.dq, xyz(A1));
            V3<S> sep = ((b.dp - a.dp) + (r2 - r1)) + xyz(CD);
            V3<S> dx = zero3<S>();
            if (limit_en & 1) dx = dx + limit_along_axis(A1.w, A2.w, sep, axis1);
            V3<S> axis2 = any_orthogonal(axis1);
            V3<S> axis3 = cross(axis1, axis2);
            dx = dx + limit_along_axis(S(0), S(0), sep, axis2);
            dx = dx + limit_along_axis(S(0), S(0), sep, axis3);
            S mag = len(dx);
            if (!(mag <= Eps<S>::v)) {
                V3<S> dir = dx / mag;
                S w1 = pos_w(max_elem(a.in.inv_mass), a.in.ii, r1, dir), w2 = pos_w(max_elem(b.in.inv_mass), b.in.ii, r2, dir);
                S dl = lagrange_update(mag, w1, w2, c0, dt);
                V3<S> impulse = dl * dir;
                tp = tp + impulse;
                positional_impulse(a, b, impulse, r1, r2, fast);
            }
            break;
        }
        default: {  // AVN_JOINT_DISTANCE, distance.rs:56-117 + DistanceLimit::compute_correction (joints/mod.rs:321-340)
            V3<S> r1 = qrot(a.dq, xyz(R1)), r2 = qrot(b.dq, xyz(R2));
            V3<S> sep = ((b.dp - a.dp) + (r2 - r1)) + xyz(CD);
            S d2 = len2(sep);
            V3<S> dir = zero3<S>();
            S dist = S(0);
            if (!(d2 <= Eps<S>::v)) {
                S dd = avn_sqrt(d2);
                if (dd < A1.w) { dir = sep / dd; dist = A1.w - dd; }
                else if (dd > A2.w) { dir = (-sep) / dd; dist = dd - A2.w; }
            }
            if (!(dist <= Eps<S>::v)) {
                S w1 = pos_w(max_elem(a.in.inv_mass), a.in.ii, r1, dir), w2 = pos_w(max_elem(b.in.inv_mass), b.in.ii, r2, dir);
                S dl = lagrange_update(dist, w1, w2, c0, dt);
                V3<S> impulse = dl * dir;
                tp = tp + impulse;
                positional_impulse(a, b, impulse, r1, r2, fast);
            }
            break;
        }
    }
    st4(&j[JP_LP * JP], mk4<S>(tp.x, tp.y, tp.z, LP.w));
    st4(&j[JP_LA * JP], mk4<S>(ta.x, ta.y, ta.z, LA.w));
    st4(&j[JP_LB * JP], mk4<S>(tb.x, tb.y, tb.z, LB.w));
    // bodies with a SolverBody are written even when their inertia is dominated: the update is then the identity
    // (x + 0, identity * q), so skipping the store is exact and keeps levels conflict-free for shared kinematic bodies.
    if (!(info & JI_ZERO1)) {
        st4(&d.dlt[2 * b1], mk4<S>(a.dp.x, a.dp.y, a.dp.z, S(0)));
        st4(&d.dlt[2 * b1 + 1], from_q(a.dq));
    }
    if (!(info & JI_ZERO2)) {
        st4(&d.dlt[2 * b2], mk4<S>(b.dp.x, b.dp.y, b.dp.z, S(0)));
        st4(&d.dlt[2 * b2 + 1], from_q(b.dq));
    }
}

// PreSolveDelta{Position,Rotation} store (xpbd/plugin.rs:61-76)
template <class S> __device__ __forceinline__ void store_pre_solve_item(const DevSolver<S>& d, int i) {
    st4(&d.pre[2 * i], ld4(&d.dlt[2 * i]));
    st4(&d.pre[2 * i + 1], ld4(&d.dlt[2 * i + 1]));
}
// project_linear_velocity + project_angular_velocity (xpbd/plugin.rs:192-240)
template <class S> __device__ __forceinline__ void project_velocity_item(const DevSolver<S>& d, int i) {
    int f = as_int(ld4(&d.inr[2 * i]).y);
    if (!(f & BF_HAS_SOLVER_BODY)) return;
    Vec4<S> dp = ld4(&d.dlt[2 * i]), dq = ld4(&d.dlt[2 * i + 1]), pp = ld4(&d.pre[2 * i]), pq = ld4(&d.pre[2 * i + 1]);
    Vec4<S> l = ld4(&d.vel[2 * i]), a = ld4(&d.vel[2 * i + 1]);
    V3<S> v = xyz(l) + (xyz(dp) - xyz(pp)) / d.h;
    Q4<S> dr = qmul(to_q(dq), qconj(to_q(pq)));
    V3<S> nav = (S(2) * qxyz(dr)) / d.h;
    if (dr.w < S(0)) nav = -nav;
    V3<S> w = xyz(a) + nav;
    st4(&d.vel[2 * i], mk4<S>(v.x, v.y, v.z, S(0)));
    st4(&d.vel[2 * i + 1], mk4<S>(w.x, w.y, w.z, S(0)));
}
// joint_damping<T> (solver/plugin.rs:759-806), on the damping schedule (joint_schedule.hpp).  An end without a SolverBody is the system
// run's dummy_body1 / dummy_body2 (d.jdummy[2 * type + side]): SolverBody::DUMMY is not kinematic, so delta_omega is written into it and
// the next such joint of the same type reads it.  Its linear velocity stays zero (0 + p * 0), so only the angular velocity is kept.
template <class S> __device__ void damp_joint_item(const DevSolver<S>& d, int slot) {
    const size_t JP = size_t(d.Jpad);
    const Vec4<S>* j = d.jnt + slot;
    Vec4<S> jidx = ld4(&j[JP_IDX * JP]);
    const int b1 = as_int(jidx.x), b2 = as_int(jidx.y), info = as_int(jidx.z);
    if (!(info & JI_DAMPING)) return;
    S dlin = ld4(&j[JP_LP * JP]).w, dang = ld4(&j[JP_LA * JP]).w;
    Vec4<S> i1a = ld4(&d.inr[2 * b1]), i2a = ld4(&d.inr[2 * b2]);
    int f1 = as_int(i1a.y), f2 = as_int(i2a.y);
    bool real1 = f1 & BF_HAS_SOLVER_BODY, real2 = f2 & BF_HAS_SOLVER_BODY;
    Vec4<S>* dummy = d.jdummy + 2 * (info & JI_TYPE_MASK);
    // NOTE: joint_damping does not apply the dominance override, only the missing-SolverBody dummy (plugin.rs:773-787)
    V3<S> v1 = real1 ? xyz(ld4(&d.vel[2 * b1])) : zero3<S>(), w1 = xyz(real1 ? ld4(&d.vel[2 * b1 + 1]) : ld4(&dummy[0]));
    V3<S> v2 = real2 ? xyz(ld4(&d.vel[2 * b2])) : zero3<S>(), w2 = xyz(real2 ? ld4(&d.vel[2 * b2 + 1]) : ld4(&dummy[1]));
    BodyInertia<S> in1 = real1 ? unpack_inertia(i1a, ld4(&d.inr[2 * b1 + 1])) : zero_inertia<S>();
    BodyInertia<S> in2 = real2 ? unpack_inertia(i2a, ld4(&d.inr[2 * b2 + 1])) : zero_inertia<S>();
    V3<S> domega = (w2 - w1) * avn_min(dang * d.h, S(1));
    if (!(f1 & BF_KINEMATIC)) w1 = w1 + domega;
    if (!(f2 & BF_KINEMATIC)) w2 = w2 - domega;
    V3<S> dv = (v2 - v1) * avn_min(dlin * d.h, S(1));
    V3<S> ws = in1.inv_mass + in2.inv_mass;
    V3<S> p = cmul(dv, mk3<S>(recip_or_zero(ws.x), recip_or_zero(ws.y), recip_or_zero(ws.z)));
    v1 = v1 + cmul(p, in1.inv_mass);
    v2 = v2 - cmul(p, in2.inv_mass);
    if (real1) { st4(&d.vel[2 * b1], mk4<S>(v1.x, v1.y, v1.z, S(0))); st4(&d.vel[2 * b1 + 1], mk4<S>(w1.x, w1.y, w1.z, S(0))); }
    else st4(&dummy[0], mk4<S>(w1.x, w1.y, w1.z, S(0)));
    if (real2) { st4(&d.vel[2 * b2], mk4<S>(v2.x, v2.y, v2.z, S(0))); st4(&d.vel[2 * b2 + 1], mk4<S>(w2.x, w2.y, w2.z, S(0))); }
    else st4(&dummy[1], mk4<S>(w2.x, w2.y, w2.z, S(0)));
}
// writeback_joint_forces (xpbd/plugin.rs:242-260)
template <class S> __device__ __forceinline__ void joint_force_item(const DevSolver<S>& d, int slot) {
    const size_t JP = size_t(d.Jpad);
    const Vec4<S>* j = d.jnt + slot;
    const int t = d.j_src_type[slot], k = d.j_src_index[slot];
    Vec4<S> LP = ld4(&j[JP_LP * JP]), LA = ld4(&j[JP_LA * JP]), LB = ld4(&j[JP_LB * JP]);
    if (d.jforce[t]) stv3(d.jforce[t], k, xyz(LP) * d.joint_force_rhs);
    if (d.jtorque[t]) stv3(d.jtorque[t], k, (xyz(LA) + xyz(LB)) * d.joint_force_rhs);
}

}  // namespace avn
