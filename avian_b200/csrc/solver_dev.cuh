// Device-side data layout and per-item routines of the solver stage.
//
// HBM layout (S = float or double; Vec4<S> = one 128-bit (f32) or 2x128-bit (f64) access):
//   bodies   vel[2*(B+1)]  = {lin.xyz,-}{ang.xyz,-}            SolverBody velocities      (solver_body/mod.rs:59-91)
//            dlt[2*(B+1)]  = {delta_position.xyz,-}{delta_rotation.xyzw}
//            inr[2*(B+1)]  = {inv_mass, flags, m00, m01}{m02, m11, m12, m22}   SolverBodyInertia (mod.rs:218-261)
//            itg[2*B]      = {linear_increment.xyz, linear_damping_rhs}{angular_increment.xyz, angular_damping_rhs}
//            slot B is SolverBody::DUMMY / SolverBodyInertia::DUMMY (static bodies, AVN_NO_BODY).
//   contacts cst[16][Mpad] planes, slot-major inside a plane so that a warp reads 32 consecutive Vec4.  Manifold m of
//            graph colour c lives in slot color_off[c] + (m - m_color_off[c]); every colour starts at a multiple of 32 so
//            a warp never straddles two colours (padding slots have info = 0 = no points):
//            0 {n.xyz, friction} 1 {t1.xyz, restitution} 2 {tangent_velocity.xyz,-} 3 {body1, body2, info, ranks}
//            4+3k {anchor1.xyz, initial_separation} 5+3k {anchor2.xyz, normal effective_mass}
//            6+3k {K1, K2, K3 (tangent effective inverse mass), normal_speed}
//            pcr[4][Mpad] records {normal impulse, total normal impulse, tangent impulse.x, .y} of point k  <- the only constraint data written in the loop
//   joints   jnt[14][Jpad] planes in level-schedule order (see JP_* below).
#pragma once
#include <cuda_pipeline.h>

#include "../../include/avian_b200.h"
#include "avn_math.cuh"

namespace avn {

// plane numbering of the IMMUTABLE constraint rows (written by prepare, read-only in the substep loop)
enum { CP_N = 0, CP_T1 = 1, CP_TV = 2, CP_IDX = 3, CP_PT0 = 4, CP_PLANES = CP_PT0 + 3 * AVN_MAX_MANIFOLD_POINTS };
// immutable rows of point k in CP_PT0 + 3k + {0: A, 1: B, 2: D}
#define CP_ROW(k, r) (CP_PT0 + 3 * (k) + (r))
// The MUTABLE impulses {lambda_n, sum lambda_n, lambda_t.x, lambda_t.y} of point k live in their own array of RECORDS, pcr, point-major
// like a plane: record (k, slot) at pcr[k * Mpad + slot], one Vec4<S> (16 bytes in f32, 32 in f64).  Together with the body state that
// precedes it in the same allocation (vel | dlt | counters | pcr) it is the "hot" range pinned in L2 by the access-policy window.
// info lane of plane CP_IDX
enum { CI_NP_MASK = 0x7, CI_ZERO1 = 1 << 4, CI_ZERO2 = 1 << 5, CI_NONDYN = 1 << 6, CI_TANGENT = 1 << 7,
       CI_VER1 = 1 << 8, CI_VER2 = 1 << 9 };   // VERx: side x is a versioned body (has a SolverBody) in wavefront mode
// flags lane of inr[2*i]
enum { BF_LOCK_MASK = 0x3f, BF_HAS_SOLVER_BODY = 1 << 8, BF_KINEMATIC = 1 << 9, BF_GYRO = 1 << 10, BF_DYNAMIC = 1 << 11,
       BF_CUSTOM_VEL = 1 << 12, BF_CUSTOM_POS = 1 << 13, BF_DOMINANCE_SHIFT = 16 };

enum { JP_IDX = 0,   // {body1, body2, type | limit_enabled<<8 | damping<<16 | zero1<<24 | zero2<<25, original index}
       JP_R1 = 1,    // {world_r1.xyz, compliance0}
       JP_R2 = 2,    // {world_r2.xyz, compliance1}
       JP_CD = 3,    // {center_difference.xyz, compliance2}
       JP_RD = 4,    // rotation_difference quaternion (fixed / prismatic)
       JP_A1 = 5,    // {a1.xyz, limit_min}
       JP_A2 = 6,    // {a2.xyz, limit_max}
       JP_B1 = 7,    // {b1.xyz, limit2_min}
       JP_B2 = 8,    // {b2.xyz, limit2_max}
       JP_LP = 9,    // {total_position_lagrange.xyz, damping_linear}
       JP_LA = 10,   // {total rotation lagrange (first angular constraint).xyz, damping_angular}
       JP_LB = 11,   // {total rotation lagrange (second angular constraint).xyz, -}
       JP_PLANES = 12 };

template <class S>
struct Soft { S bias, mass_scale, impulse_scale; };

template <class S>
struct DevSolver {
    int B, M, P, Mpad, J, Jpad, n_levels;
    int m_color_off[AVN_GRAPH_COLOR_COUNT + 1];  // manifold index ranges per colour (ABI order)
    int color_off[AVN_GRAPH_COLOR_COUNT + 1];    // SLOT ranges per colour, each start a multiple of 32; [24] = Mpad
    int color_len[AVN_GRAPH_COLOR_COUNT];        // manifolds in the colour
    int wave;                                    // 1: wavefront (dependency-counter) substep loop, 0: grid barriers
    unsigned int* ver;                           // [B+1] per-body event counter (wavefront mode)
    int* deg;                                    // [B+1] contact constraints touching the body (wavefront mode)
    int* stamp;                                  // [B+1] 1 + last colour that ranked the body: detects a body listed twice in one colour
    int substeps, iters, rest_iters, fast_trig, match_contacts;
    S h, dt, max_overlap_speed, warm_coeff, rest_threshold, joint_force_rhs;
    S gx, gy, gz;
    Soft<S> soft_dyn, soft_nondyn;
    // raw body columns (device copies of the ABI columns; NULL when the host column was NULL)
    const uint8_t* kind; const uint8_t* locked; const int8_t* dominance; const uint8_t* integ_flags;
    const S* position; const S* rotation; const S* linvel; const S* angvel; const S* inv_mass; const S* inv_inertia_local;
    const S* com; const S* lin_damp; const S* ang_damp; const S* grav_scale; const S* lin_acc; const S* ang_acc;
    const S* max_lin; const S* max_ang;
    S* out_position; S* out_rotation; S* out_linvel; S* out_angvel;
    Vec4<S>* vel; Vec4<S>* dlt; Vec4<S>* inr; Vec4<S>* itg; Vec4<S>* pre;
    // raw manifold columns
    const int* m_body1; const int* m_body2; const S* m_normal; const S* m_friction; const S* m_restitution; const S* m_tanvel;
    // points of manifold m: rows [m_point_begin[m], m_point_end[m]) of the point columns.  CSR input: begin = offsets, end = offsets + 1
    // (the same buffer).  Edge-indexed input: begin = 4 * edge[m], end = begin + point_count[edge[m]], and the per-manifold normal lives
    // in row m_src[m] (= edge[m]) of the normal column; m_src == NULL means row m.
    const uint32_t* m_point_begin; const uint32_t* m_point_end; const uint32_t* m_src;
    const S* p_anchor1; const S* p_anchor2; const S* p_penetration; const S* p_normal_speed;
    const S* p_ws_normal; const S* p_ws_tangent;               // warm-start inputs (never written: every run restarts from them)
    const S* p_in_normal_impulse;
    S* p_out_ws_normal; S* p_out_ws_tangent; S* p_normal_impulse;  // store_contact_impulses outputs
    Vec4<S>* cst;
    Vec4<S>* pcr;                                // impulse records, see PcRec
    int* any_restitution;
    // joints
    const int* j_src_type; const int* j_src_index;  // schedule slot -> (type, index in type)
    const int* level_off;                           // [n_levels+1]
    Vec4<S>* jnt;
    const S* jc[AVN_JOINT_TYPE_COUNT][12];  // per type raw columns: la1 la2 lb1 lb2 axis lmin lmax l2min l2max c0 c1 c2
    const S* jdamp_lin[AVN_JOINT_TYPE_COUNT]; const S* jdamp_ang[AVN_JOINT_TYPE_COUNT];
    const uint8_t* jlimit_en[AVN_JOINT_TYPE_COUNT]; const uint8_t* jdamp_en[AVN_JOINT_TYPE_COUNT];
    const int* jbody1[AVN_JOINT_TYPE_COUNT]; const int* jbody2[AVN_JOINT_TYPE_COUNT];
    S* jforce[AVN_JOINT_TYPE_COUNT]; S* jtorque[AVN_JOINT_TYPE_COUNT];
    int any_joint_damping;
    // launch range (avn_solver_run_range): which parts of the step this launch runs.  A plain avn_solver_run does everything.
    int do_prepare, sub_begin, sub_end, do_restitution, do_finalize;
    // x-slab partition (multi-GPU, include/avian_b200.h "boundary bodies"): bnd_of[b] = index into the boundary list or -1 (NULL when
    // the step is not partitioned); vel_ref = the boundary bodies' velocities right after integrate_velocities (2 rows per body)
    const int* bnd_of;
    Vec4<S>* vel_ref;
};

template <class S> __device__ __forceinline__ V3<S> ldv3(const S* p, int i) { return mk3<S>(p[3 * i], p[3 * i + 1], p[3 * i + 2]); }
template <class S> __device__ __forceinline__ V3<S> ldv3_or0(const S* p, int i) { return p ? ldv3(p, i) : zero3<S>(); }
template <class S> __device__ __forceinline__ Q4<S> ldq(const S* p, int i) {
    Q4<S> q; q.x = p[4 * i]; q.y = p[4 * i + 1]; q.z = p[4 * i + 2]; q.w = p[4 * i + 3]; return q;
}
template <class S> __device__ __forceinline__ void stv3(S* p, int i, V3<S> v) { p[3 * i] = v.x; p[3 * i + 1] = v.y; p[3 * i + 2] = v.z; }

// impulse record of point k of the manifold in `slot`
template <class S> __device__ __forceinline__ Vec4<S>* pc_ptr(const DevSolver<S>& d, int k, int slot) {
    return d.pcr + size_t(k) * size_t(d.Mpad) + size_t(slot);
}
// store the value {lambda_n, sum, lt.x, lt.y} of an impulse record
template <class S> __device__ __forceinline__ void pc_store(Vec4<S>* p, Vec4<S> v) { st4(p, v); }

template <class S> struct BodyInertia {
    V3<S> inv_mass;  // effective (locked axes applied)
    Sym3<S> ii;
};
template <class S> __device__ __forceinline__ BodyInertia<S> zero_inertia() {
    BodyInertia<S> r;
    r.inv_mass = zero3<S>();
    r.ii.m00 = r.ii.m01 = r.ii.m02 = r.ii.m11 = r.ii.m12 = r.ii.m22 = S(0);
    return r;
}
// SolverBodyInertia::effective_inv_mass (solver_body/mod.rs:437-451)
template <class S> __device__ __forceinline__ BodyInertia<S> unpack_inertia(Vec4<S> a, Vec4<S> b) {
    BodyInertia<S> r;
    int f = as_int(a.y);
    r.inv_mass = mk3<S>((f & AVN_LOCK_TRANSLATION_X) ? S(0) : a.x, (f & AVN_LOCK_TRANSLATION_Y) ? S(0) : a.x,
                        (f & AVN_LOCK_TRANSLATION_Z) ? S(0) : a.x);
    r.ii.m00 = a.z; r.ii.m01 = a.w; r.ii.m02 = b.x; r.ii.m11 = b.y; r.ii.m12 = b.z; r.ii.m22 = b.w;
    return r;
}

// ---------------------------------------------------------------------------------------------------------
// prepare_solver_bodies (solver_body/plugin.rs:173-251) + pre_process_velocity_increments (integrator/mod.rs:260-313)
// ---------------------------------------------------------------------------------------------------------
template <class S>
__device__ void prepare_body_item(const DevSolver<S>& d, int i) {
    Vec4<S> lin = mk4<S>(0, 0, 0, 0), ang = lin, dp = lin, dq = mk4<S>(0, 0, 0, 1);
    Vec4<S> ia = mk4<S>(S(0), int_as(S(0), 128 << BF_DOMINANCE_SHIFT), S(0), S(0)), ib = mk4<S>(0, 0, 0, 0);
    int kind = i < d.B ? (d.kind ? d.kind[i] : AVN_BODY_DYNAMIC) : AVN_BODY_STATIC;
    if (kind != AVN_BODY_STATIC) {
        V3<S> v = ldv3(d.linvel, i), w = ldv3(d.angvel, i);
        lin = mk4<S>(v.x, v.y, v.z, 0);
        ang = mk4<S>(w.x, w.y, w.z, 0);
        int locked = d.locked ? d.locked[i] : 0;
        S inv_mass = d.inv_mass[i];
        Sym3<S> il;
        il.m00 = d.inv_inertia_local[6 * i]; il.m01 = d.inv_inertia_local[6 * i + 1]; il.m02 = d.inv_inertia_local[6 * i + 2];
        il.m11 = d.inv_inertia_local[6 * i + 3]; il.m12 = d.inv_inertia_local[6 * i + 4]; il.m22 = d.inv_inertia_local[6 * i + 5];
        Sym3<S> iw = rotate_inv_inertia(il, ldq(d.rotation, i));
        // SolverBodyInertia::new (solver_body/mod.rs:378-423)
        if (locked & AVN_LOCK_ROTATION_X) { iw.m00 = 0; iw.m01 = 0; iw.m02 = 0; }
        if (locked & AVN_LOCK_ROTATION_Y) { iw.m01 = 0; iw.m11 = 0; iw.m12 = 0; }
        if (locked & AVN_LOCK_ROTATION_Z) { iw.m02 = 0; iw.m12 = 0; iw.m22 = 0; }
        int dom = (kind == AVN_BODY_DYNAMIC) ? (d.dominance ? int(d.dominance[i]) : 0) : 128;
        int flags = (locked & BF_LOCK_MASK) | BF_HAS_SOLVER_BODY | ((dom & 0xffff) << BF_DOMINANCE_SHIFT);
        if (kind == AVN_BODY_KINEMATIC) flags |= BF_KINEMATIC;
        if (kind == AVN_BODY_DYNAMIC) flags |= BF_DYNAMIC;
        int ifl = d.integ_flags ? d.integ_flags[i] : 0;
        if (ifl & AVN_CUSTOM_VELOCITY_INTEGRATION) flags |= BF_CUSTOM_VEL;
        if (ifl & AVN_CUSTOM_POSITION_INTEGRATION) flags |= BF_CUSTOM_POS;
        // gyroscopic iff rotation not fully locked and local inverse inertia not isotropic (eps 1e-6), plugin.rs:241-247
        bool rot_locked = (locked & 0x7) == 0x7;
        S eps = S(1e-6);
        bool iso = !(avn_abs(il.m00 - il.m11) > eps || avn_abs(il.m11 - il.m22) > eps) && avn_abs(il.m01) < eps &&
                   avn_abs(il.m02) < eps && avn_abs(il.m12) < eps;
        if (!rot_locked && !iso) flags |= BF_GYRO;
        ia = mk4<S>(inv_mass, int_as(S(0), flags), iw.m00, iw.m01);
        ib = mk4<S>(iw.m02, iw.m11, iw.m12, iw.m22);
    }
    st4(&d.vel[2 * i], lin); st4(&d.vel[2 * i + 1], ang);
    st4(&d.dlt[2 * i], dp); st4(&d.dlt[2 * i + 1], dq);
    st4(&d.inr[2 * i], ia); st4(&d.inr[2 * i + 1], ib);
    if (i < d.B) {
        V3<S> li = ldv3_or0(d.lin_acc, i), ai = ldv3_or0(d.ang_acc, i);
        S lr = S(1), ar = S(1);
        if (kind == AVN_BODY_DYNAMIC) {
            int locked = d.locked ? d.locked[i] : 0;
            lr = S(1) / (S(1) + d.h * (d.lin_damp ? d.lin_damp[i] : S(0)));
            ar = S(1) / (S(1) + d.h * (d.ang_damp ? d.ang_damp[i] : S(0)));
            li = li + mk3<S>(d.gx, d.gy, d.gz) * (d.grav_scale ? d.grav_scale[i] : S(1));
            if (locked & AVN_LOCK_TRANSLATION_X) li.x = 0;
            if (locked & AVN_LOCK_TRANSLATION_Y) li.y = 0;
            if (locked & AVN_LOCK_TRANSLATION_Z) li.z = 0;
            if (locked & AVN_LOCK_ROTATION_X) ai.x = 0;
            if (locked & AVN_LOCK_ROTATION_Y) ai.y = 0;
            if (locked & AVN_LOCK_ROTATION_Z) ai.z = 0;
            li = li * d.h;
            ai = ai * d.h;
        }
        st4(&d.itg[2 * i], mk4<S>(li.x, li.y, li.z, lr));
        st4(&d.itg[2 * i + 1], mk4<S>(ai.x, ai.y, ai.z, ar));
    }
}

// ---------------------------------------------------------------------------------------------------------
// prepare_contact_constraints -> ContactConstraint::generate (solver/plugin.rs:363-448, contact/mod.rs:110-220,
// normal_part.rs:39-112, tangent_part.rs:35-151)
// ---------------------------------------------------------------------------------------------------------
// manifold index (ABI order, grouped by colour) -> slot in the padded colour-major plane layout
template <class S> __device__ __forceinline__ int slot_of_manifold(const DevSolver<S>& d, int m) {
    int c = 0;
    while (c < AVN_GRAPH_COLOR_COUNT - 1 && m >= d.m_color_off[c + 1]) ++c;
    return d.color_off[c] + (m - d.m_color_off[c]);
}

template <class S>
__device__ void prepare_constraint_item(const DevSolver<S>& d, int m) {
    int rb1 = d.m_body1[m], rb2 = d.m_body2[m];
    int b1 = rb1 < 0 ? d.B : rb1, b2 = rb2 < 0 ? d.B : rb2;
    Vec4<S> i1a = ld4(&d.inr[2 * b1]), i1b = ld4(&d.inr[2 * b1 + 1]);
    Vec4<S> i2a = ld4(&d.inr[2 * b2]), i2b = ld4(&d.inr[2 * b2 + 1]);
    int f1 = as_int(i1a.y), f2 = as_int(i2a.y);
    uint32_t p0 = d.m_point_begin[m], p1 = d.m_point_end[m];
    int np = int(p1 - p0);
    const int slot = slot_of_manifold(d, m);
    Vec4<S>* c = d.cst + slot;
    const size_t MP = size_t(d.Mpad);
    // skip contacts between two non-dynamic bodies (plugin.rs:415-418) and empty manifolds (:434)
    if ((!(f1 & BF_DYNAMIC) && !(f2 & BF_DYNAMIC)) || np <= 0) {
        st4(&c[CP_IDX * MP], mk4<S>(int_as(S(0), b1), int_as(S(0), b2), int_as(S(0), 0), int_as(S(0), 0)));
        return;
    }
    int dom1 = (f1 >> BF_DOMINANCE_SHIFT) << 16 >> 16, dom2 = (f2 >> BF_DOMINANCE_SHIFT) << 16 >> 16;  // sign-extend i16
    int rel = dom1 - dom2;
    BodyInertia<S> in1 = rel > 0 ? zero_inertia<S>() : unpack_inertia(i1a, i1b);
    BodyInertia<S> in2 = rel < 0 ? zero_inertia<S>() : unpack_inertia(i2a, i2b);
    int info = np;
    if (rel > 0 || !(f1 & BF_HAS_SOLVER_BODY)) info |= CI_ZERO1;
    if (rel < 0 || !(f2 & BF_HAS_SOLVER_BODY)) info |= CI_ZERO2;
    if (rel != 0) info |= CI_NONDYN;
    if (f1 & BF_HAS_SOLVER_BODY) info |= CI_VER1;
    if (f2 & BF_HAS_SOLVER_BODY) info |= CI_VER2;
    V3<S> mass_sum = in1.inv_mass + in2.inv_mass;
    V3<S> n = ldv3(d.m_normal, d.m_src ? int(d.m_src[m]) : m);
    // compute_tangent_directions (contact/mod.rs:427-449): LinearVelocity components of the rigid bodies
    V3<S> v1 = rb1 >= 0 ? ldv3(d.linvel, rb1) : zero3<S>();
    V3<S> v2 = rb2 >= 0 ? ldv3(d.linvel, rb2) : zero3<S>();
    V3<S> fd = -n;
    V3<S> rv = v1 - v2;
    V3<S> tvv = rv - fd * dot(fd, rv);
    V3<S> t1;
    {
        S rcp = S(1) / len(tvv);
        if (avn_finite(rcp) && rcp > S(0)) t1 = tvv * rcp; else t1 = any_orthonormal(fd);
    }
    V3<S> t2 = cross(fd, t1);
    S friction = d.m_friction[m], restitution = d.m_restitution[m];
    if (friction > S(0)) info |= CI_TANGENT;
    if (restitution != S(0)) *d.any_restitution = 1;
    V3<S> tv = ldv3_or0(d.m_tanvel, m);
    st4(&c[CP_N * MP], mk4<S>(n.x, n.y, n.z, friction));
    st4(&c[CP_T1 * MP], mk4<S>(t1.x, t1.y, t1.z, restitution));
    st4(&c[CP_TV * MP], mk4<S>(tv.x, tv.y, tv.z, S(0)));
    st4(&c[CP_IDX * MP], mk4<S>(int_as(S(0), b1), int_as(S(0), b2), int_as(S(0), info), int_as(S(0), 0)));
    bool warm = d.match_contacts != 0;
    for (int k = 0; k < np; ++k) {
        uint32_t p = p0 + k;
        V3<S> r1 = ldv3(d.p_anchor1, p), r2 = ldv3(d.p_anchor2, p);
        V3<S> r1xn = cross(r1, n), r2xn = cross(r2, n);
        S k_linear = dot(n, cmul(mass_sum, n));
        S kk = k_linear + dot(r1xn, smul(in1.ii, r1xn)) + dot(r2xn, smul(in2.ii, r2xn));
        S meff = recip_or_zero(kk);
        S sep0 = -d.p_penetration[p] - dot(r2 - r1, n);
        S imp_n = warm ? d.p_ws_normal[p] : S(0);
        S itx = S(0), ity = S(0), K1 = S(0), K2 = S(0), K3 = S(0);
        if (info & CI_TANGENT) {
            if (warm) { itx = d.p_ws_tangent[2 * p]; ity = d.p_ws_tangent[2 * p + 1]; }
            V3<S> rt11 = cross(r1, t1), rt12 = cross(r2, t1), rt21 = cross(r1, t2), rt22 = cross(r2, t2);
            V3<S> i1_rt11 = smul(in1.ii, rt11), i2_rt12 = smul(in2.ii, rt12), i1_rt21 = smul(in1.ii, rt21), i2_rt22 = smul(in2.ii, rt22);
            S kl1 = dot(t1, cmul(mass_sum, t1)), kl2 = dot(t2, cmul(mass_sum, t2));
            K1 = kl1 + dot(rt11, i1_rt11) + dot(rt12, i2_rt12);
            K2 = kl2 + dot(rt21, i1_rt21) + dot(rt22, i2_rt22);
            K3 = S(2) * (dot(rt11, i1_rt21) + dot(rt12, i2_rt22));
        }
        st4(&c[size_t(CP_ROW(k, 0)) * MP], mk4<S>(r1.x, r1.y, r1.z, sep0));
        st4(&c[size_t(CP_ROW(k, 1)) * MP], mk4<S>(r2.x, r2.y, r2.z, meff));
        pc_store(pc_ptr(d, k, slot), mk4<S>(imp_n, S(0), itx, ity));
        st4(&c[size_t(CP_ROW(k, 2)) * MP], mk4<S>(K1, K2, K3, d.p_normal_speed[p]));
    }
}

// ---------------------------------------------------------------------------------------------------------
// warm_start / solve_contacts<BIAS> / relax / restitution for ONE manifold (one thread)
// ---------------------------------------------------------------------------------------------------------
enum { PASS_WARM = 0, PASS_SOLVE_BIAS = 1, PASS_RELAX = 2, PASS_RESTITUTION = 3 };

template <class S>
__device__ __forceinline__ void apply_impulse(V3<S>& v1, V3<S>& w1, V3<S>& v2, V3<S>& w2, const BodyInertia<S>& in1, const BodyInertia<S>& in2,
                                              V3<S> r1, V3<S> r2, V3<S> imp) {
    v1 = v1 - cmul(imp, in1.inv_mass);
    w1 = w1 - smul(in1.ii, cross(r1, imp));
    v2 = v2 + cmul(imp, in2.inv_mass);
    w2 = w2 + smul(in2.ii, cross(r2, imp));
}

// ---- wavefront mode: per-body event counters replace the grid barriers between colours ---------------------------
// Every body with a SolverBody owns a counter ver[b] that counts the work items that have touched it, in the exact order
// the reference's schedule touches it.  Within one substep that order is (k = number of contact constraints on the body,
// r = rank of a constraint among them in colour-major order):
//     integrate_velocities | warm_start r=0..k-1 | (biased solve r=0..k-1) x iters | integrate_positions | relax r=0..k-1
// An item may run when the counters of its bodies equal its position in their sequences, and bumps them when done.
// Items are handed to warps in the global schedule order, all warps are co-resident (cooperative launch), and an item
// only ever waits for items that precede it in that order, so the earliest unfinished item can always run: no deadlock.
// flag words behind any_restitution: [0] some restitution coefficient != 0, [1] WAVE_* event, [2..3] spare, then (8-byte aligned) the
// optional trace counters
enum { FLAG_RESTITUTION = 0, FLAG_WAVE = 1, FLAG_WORDS = 4 };
// Optional latency trace of the wavefront items (build with -DAVN_WAVE_TRACE; scripts/wave_trace.py): per-warp SM-cycle sums of
// [0] wait for the exact event  [1] mutable loads (velocities, impulses) + staged rows  [2] arithmetic (with the impulse record stores)
// [3] velocity stores + release fence + publish, [4] item count, [5] stage 1 of a solve item (wait for the deltas, the separations and the
// normal-impulse coefficients).  The buffer is 8 unsigned long long counters behind
// the FLAG_WORDS int flags of any_restitution.
#ifdef AVN_WAVE_TRACE
#define AVN_TRACE_T(var) const long long var = clock64()
#define AVN_TRACE_ADD(d, i, v) do { if ((threadIdx.x & 31) == 0) atomicAdd(reinterpret_cast<unsigned long long*>((d).any_restitution + FLAG_WORDS) + (i), (unsigned long long)(v)); } while (0)
#else
#define AVN_TRACE_T(var)
#define AVN_TRACE_ADD(d, i, v)
#endif
__device__ __forceinline__ unsigned events_per_substep(int k, int iters) { return 2u + unsigned(2 + iters) * unsigned(k); }
enum { WV_IV = 0, WV_WARM = 1, WV_SOLVE = 2, WV_IP = 3, WV_RELAX = 4 };
// position of an item in its body's event sequence
__device__ __forceinline__ unsigned wave_event(int kind, int it, int s, int iters, int k, int r) {
    unsigned base = unsigned(s) * events_per_substep(k, iters);
    switch (kind) {
        case WV_IV: return base;
        case WV_WARM: return base + 1u + r;
        case WV_SOLVE: return base + 1u + unsigned(1 + it) * k + r;
        case WV_IP: return base + 1u + unsigned(1 + iters) * k;
        default: return base + 2u + unsigned(1 + iters) * k + r;
    }
}
// counters: message passing with acquire / release.  The consumer polls with ld.acquire.gpu (no membar: on sm_90 a strong load plus an
// L1 invalidation) — each lane only reads data that its own counters guard, so the acquire of the poll that succeeds is all it needs.
// The producer issues ONE fence.acq_rel.gpu after its data stores and then stores its counters relaxed (fence + strong store = release).
__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed(unsigned* p, unsigned v) { asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void fence_acq_rel() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
// mutable body / impulse data is read through L2 only in wavefront mode (other SMs write it while this kernel runs)
__device__ __forceinline__ Vec4<float> ld4_cg(const Vec4<float>* p) {
    float4 v = __ldcg(reinterpret_cast<const float4*>(p));
    return mk4<float>(v.x, v.y, v.z, v.w);
}
__device__ __forceinline__ Vec4<double> ld4_cg(const Vec4<double>* p) {
    double2 a = __ldcg(reinterpret_cast<const double2*>(p)), b = __ldcg(reinterpret_cast<const double2*>(p) + 1);
    return mk4<double>(a.x, a.y, b.x, b.y);
}
template <bool WAVE, class S> __device__ __forceinline__ Vec4<S> ldm(const Vec4<S>* p) { return WAVE ? ld4_cg(p) : ld4(p); }
// the value {lambda_n, sum, lt.x, lt.y} of an impulse record
template <bool WAVE, class S> __device__ __forceinline__ Vec4<S> pc_load(const Vec4<S>* p) { return ldm<WAVE>(p); }

// warp-synchronous wait: all 32 lanes of the warp wait until every lane's two counters have reached their targets — exactly (EXACT) or
// at least (counters only grow).  A lane stops polling a counter once it has seen its target: with EXACT the counter cannot move on
// before this item publishes, and either way the acquire of that poll orders the loads that follow it.
// A watchdog bounds the spin (a schedule bug must not hang the device): after ~4M polls the warp gives up and raises
// *watchdog, which the host turns into an error.  seen1 / seen2 (optional) receive the last value each lane's poll of that counter read.
template <bool EXACT = true>
__device__ __forceinline__ void wave_wait(const unsigned* ver, bool need1, int b1, unsigned e1, bool need2, int b2, unsigned e2, int* watchdog,
                                          unsigned* seen1 = nullptr, unsigned* seen2 = nullptr) {
    for (unsigned spins = 0;; ++spins) {
        if (need1) { const unsigned v = ld_acquire(ver + b1); need1 = EXACT ? v != e1 : v < e1; if (seen1) *seen1 = v; }
        if (need2) { const unsigned v = ld_acquire(ver + b2); need2 = EXACT ? v != e2 : v < e2; if (seen2) *seen2 = v; }
        if (__all_sync(0xffffffffu, !(need1 || need2))) break;
        if (spins > (1u << 22)) { *watchdog = 1; break; }
    }
}
__device__ __forceinline__ void wave_publish(unsigned* ver, bool need1, int b1, unsigned e1, bool need2, int b2, unsigned e2) {
    fence_acq_rel();  // release: this item's stores are visible before the counters move
    if (need1) st_relaxed(ver + b1, e1 + 1u);
    if (need2) st_relaxed(ver + b2, e2 + 1u);
}

// ---- shared-memory staging of the immutable per-point constraint rows -------------------------------------------------
// Each thread copies its manifold's {anchor1|sep0}, {anchor2|m_eff}, {K|normal_speed} rows (up to 12 x 16 B) from the planes
// into its own column of a dynamic shared-memory tile with cp.async (LDGSTS: no registers, no local-memory spills), waits
// for its own copies only, and reads a row right where a point needs it.  Layout: row r of thread t at stage[r * T + t]
// (consecutive threads -> consecutive 16-byte words: conflict-free).  The copies fly while the thread waits on its
// dependency counters (wavefront mode) or on the body gathers (barrier mode).
constexpr int STAGE_ROWS = 3 * AVN_MAX_MANIFOLD_POINTS;
template <class S> __device__ __forceinline__ Vec4<S>* stage_base() {
    extern __shared__ __align__(32) unsigned char avn_stage_raw[];
    return reinterpret_cast<Vec4<S>*>(avn_stage_raw);
}
__device__ __forceinline__ void stage_copy(Vec4<float>* dst, const Vec4<float>* src) { __pipeline_memcpy_async(dst, src, 16); }
__device__ __forceinline__ void stage_copy(Vec4<double>* dst, const Vec4<double>* src) {
    __pipeline_memcpy_async(dst, src, 16);
    __pipeline_memcpy_async(reinterpret_cast<char*>(dst) + 16, reinterpret_cast<const char*>(src) + 16, 16);
}
// the tile only needs the rows of the widest manifold of the upload (single-point sphere contacts: a quarter of the tile, the rest
// of the SM's shared-memory / L1 array stays L1)
// (3 staged rows per point + 1 scratch row per point for its impulses: wave_contact_item)
template <class S> __host__ __device__ constexpr size_t stage_bytes(int threads, int max_points = AVN_MAX_MANIFOLD_POINTS) {
    return size_t(4 * max_points) * threads * sizeof(Vec4<S>);
}

// Barrier schedules (grid-wide phases, phase kernels); the wavefront schedule runs wave_contact_item below.
// `slot` indexes the padded colour-major planes (a padding slot returns at once).
// MAXP: compile-time bound on the points of a manifold (1 for sphere-only scenes: a quarter of the registers and no dead unrolled code)
template <class S, int PASS, int MAXP = AVN_MAX_MANIFOLD_POINTS>
__device__ __forceinline__ void contact_item(const DevSolver<S>& d, int slot) {
    const size_t MP = size_t(d.Mpad);
    Vec4<S>* c = d.cst + slot;
    Vec4<S> hidx = ld4(&c[CP_IDX * MP]);
    const int info = as_int(hidx.z);
    const int np = info & CI_NP_MASK;
    if (np == 0) return;
    const int b1 = as_int(hidx.x), b2 = as_int(hidx.y);
    // ---- issue every load up front (independent 128-bit loads -> memory-level parallelism)
    Vec4<S> hn = mk4<S>(0, 0, 0, 0), ht1 = hn, htv = hn;
    BodyInertia<S> in1 = zero_inertia<S>(), in2 = zero_inertia<S>();
    Vec4<S> PC[MAXP];
    constexpr bool SOLVE = (PASS == PASS_SOLVE_BIAS || PASS == PASS_RELAX);
    Vec4<S>* const stage = stage_base<S>() + threadIdx.x;   // this thread's column; row r at stage[r * T]
    const int T = blockDim.x;
#define ROW_A(k) stage[(3 * (k) + 0) * T]
#define ROW_B(k) stage[(3 * (k) + 1) * T]
#define ROW_D(k) stage[(3 * (k) + 2) * T]
    {
        hn = ld4(&c[CP_N * MP]);
        ht1 = ld4(&c[CP_T1 * MP]);
        if (SOLVE) htv = ld4(&c[CP_TV * MP]);
        if (!(info & CI_ZERO1)) in1 = unpack_inertia(ld4(&d.inr[2 * b1]), ld4(&d.inr[2 * b1 + 1]));
        if (!(info & CI_ZERO2)) in2 = unpack_inertia(ld4(&d.inr[2 * b2]), ld4(&d.inr[2 * b2 + 1]));
#pragma unroll
        for (int k = 0; k < MAXP; ++k) {
            if (k < np) {
                stage_copy(&ROW_A(k), &c[size_t(CP_ROW(k, 0)) * MP]);
                stage_copy(&ROW_B(k), &c[size_t(CP_ROW(k, 1)) * MP]);
                if (PASS == PASS_RESTITUTION || (SOLVE && (info & CI_TANGENT))) stage_copy(&ROW_D(k), &c[size_t(CP_ROW(k, 2)) * MP]);
            }
        }
    }
    __pipeline_commit();
    // ---- mutable state: body velocities / deltas and the accumulated impulses
    Vec4<S> l1 = ld4(&d.vel[2 * b1]), a1 = ld4(&d.vel[2 * b1 + 1]);
    Vec4<S> l2 = ld4(&d.vel[2 * b2]), a2 = ld4(&d.vel[2 * b2 + 1]);
    Vec4<S> dp1, dq1, dp2, dq2;
    if (SOLVE) {
        dp1 = ld4(&d.dlt[2 * b1]); dq1 = ld4(&d.dlt[2 * b1 + 1]);
        dp2 = ld4(&d.dlt[2 * b2]); dq2 = ld4(&d.dlt[2 * b2 + 1]);
    }
#pragma unroll
    for (int k = 0; k < MAXP; ++k)
        if (k < np) PC[k] = pc_load<false>(pc_ptr(d, k, slot));
    __pipeline_wait_prior(0);  // this thread's staged rows have landed (only the issuing thread reads them)
    V3<S> v1 = xyz(l1), w1 = xyz(a1), v2 = xyz(l2), w2 = xyz(a2);
    const V3<S> n = xyz(hn), t1 = xyz(ht1);
    const V3<S> t2 = cross(t1, n);  // tangent_directions(): [tangent1, tangent1 x normal] (contact/mod.rs:411-421)

    if (PASS == PASS_WARM) {
        // ContactConstraint::warm_start (contact/mod.rs:223-264)
#pragma unroll
        for (int k = 0; k < MAXP; ++k) {
            if (k < np) {
                const Vec4<S> PAk = ROW_A(k), PBk = ROW_B(k);
                V3<S> r1 = xyz(PAk), r2 = xyz(PBk);
                S tx = (info & CI_TANGENT) ? PC[k].z : S(0), ty = (info & CI_TANGENT) ? PC[k].w : S(0);
                V3<S> p = d.warm_coeff * ((PC[k].x * n + tx * t1) + ty * t2);
                apply_impulse(v1, w1, v2, w2, in1, in2, r1, r2, p);
            }
        }
    } else if (PASS == PASS_SOLVE_BIAS || PASS == PASS_RELAX) {
        // ContactConstraint::solve (contact/mod.rs:267-354)
        const Soft<S> soft = (info & CI_NONDYN) ? d.soft_nondyn : d.soft_dyn;
        Q4<S> q1; q1.x = dq1.x; q1.y = dq1.y; q1.z = dq1.z; q1.w = dq1.w;
        Q4<S> q2; q2.x = dq2.x; q2.y = dq2.y; q2.z = dq2.z; q2.w = dq2.w;
        const V3<S> delta_translation = xyz(dp2) - xyz(dp1);
#pragma unroll
        for (int k = 0; k < MAXP; ++k) {
            if (k < np) {
                const Vec4<S> PAk = ROW_A(k), PBk = ROW_B(k);
                V3<S> r1 = xyz(PAk), r2 = xyz(PBk);
                V3<S> rr1 = qrot(q1, r1), rr2 = qrot(q2, r2);
                V3<S> dsep = delta_translation + (rr2 - rr1);
                S separation = dot(dsep, n) + PAk.w;
                V3<S> relv = (v2 + cross(w2, r2)) - (v1 + cross(w1, r1));
                // ContactNormalPart::solve_impulse (normal_part.rs:116-166)
                S vn = dot(relv, n);
                S meff = PBk.w, acc = PC[k].x;
                S impulse;
                if (separation > S(0)) {
                    impulse = -meff * (vn + separation / d.h);
                } else if (PASS == PASS_SOLVE_BIAS) {
                    S bias = avn_max(soft.bias * separation, -d.max_overlap_speed);
                    S scaled_mass = soft.mass_scale * meff;
                    S scaled_impulse = soft.impulse_scale * acc;
                    impulse = -scaled_mass * (vn + bias) - scaled_impulse;
                } else {
                    impulse = -meff * vn;
                }
                S new_impulse = avn_max(acc + impulse, S(0));
                impulse = new_impulse - acc;
                PC[k].x = new_impulse;
                PC[k].y = PC[k].y + new_impulse;
                apply_impulse(v1, w1, v2, w2, in1, in2, r1, r2, impulse * n);
            }
        }
        if (info & CI_TANGENT) {
            const S friction = hn.w;
            const V3<S> surf = xyz(htv);
#pragma unroll
            for (int k = 0; k < MAXP; ++k) {
                if (k < np) {
                    const Vec4<S> PAk = ROW_A(k), PBk = ROW_B(k), PDk = ROW_D(k);
                    V3<S> r1 = xyz(PAk), r2 = xyz(PBk);
                    V3<S> relv = (v2 + cross(w2, r2)) - (v1 + cross(w1, r1));
                    // ContactTangentPart::solve_impulse (tangent_part.rs:155-244)
                    S limit = friction * PC[k].x;
                    relv = relv + surf;
                    S ts1 = dot(relv, t1), ts2 = dot(relv, t2);
                    S t11 = ts1 * ts1, t22 = ts2 * ts2, t12 = ts1 * ts2;
                    S inv = (t11 * PDk.x + t22 * PDk.y) + t12 * PDk.z;
                    S em = (t11 + t22) * (S(1) / inv);
                    V3<S> imp = zero3<S>();
                    if (avn_finite(em)) {
                        S nx = PC[k].z - em * ts1, ny = PC[k].w - em * ts2;
                        S l2 = nx * nx + ny * ny;
                        if (l2 > limit * limit) {  // Vec2::clamp_length_max
                            S l = avn_sqrt(l2);
                            nx = limit * (nx / l);
                            ny = limit * (ny / l);
                        }
                        S dx = nx - PC[k].z, dy = ny - PC[k].w;
                        PC[k].z = nx;
                        PC[k].w = ny;
                        imp = dx * t1 + dy * t2;
                    }
                    apply_impulse(v1, w1, v2, w2, in1, in2, r1, r2, imp);
                }
            }
        }
    } else {
        // solve_restitution_internal + ContactConstraint::apply_restitution (plugin.rs:676-718, contact/mod.rs:358-407)
        const S e = ht1.w;
        if (e == S(0)) return;
        const int iterations = np > 1 ? d.rest_iters : 1;
        for (int it = 0; it < iterations; ++it) {
#pragma unroll
            for (int k = 0; k < MAXP; ++k) {
                if (k < np) {
                    const Vec4<S> PAk = ROW_A(k), PBk = ROW_B(k), PDk = ROW_D(k);
                    if (PDk.w > -d.rest_threshold || PC[k].y == S(0)) continue;
                    V3<S> r1 = xyz(PAk), r2 = xyz(PBk);
                    V3<S> relv = (v2 + cross(w2, r2)) - (v1 + cross(w1, r1));
                    S vn = dot(relv, n);
                    S impulse = -PBk.w * (vn + e * PDk.w);
                    S new_impulse = avn_max(PC[k].x + impulse, S(0));
                    impulse = new_impulse - PC[k].x;
                    PC[k].x = new_impulse;
                    PC[k].y = PC[k].y + impulse;
                    apply_impulse(v1, w1, v2, w2, in1, in2, r1, r2, impulse * n);
                }
            }
        }
    }
    // ---- write back: impulses and the velocities of the non-dominant sides
    if (PASS != PASS_WARM) {
#pragma unroll
        for (int k = 0; k < MAXP; ++k)
            if (k < np) pc_store(pc_ptr(d, k, slot), PC[k]);
    }
    if (!(info & CI_ZERO1)) {
        st4(&d.vel[2 * b1], mk4<S>(v1.x, v1.y, v1.z, S(0)));
        st4(&d.vel[2 * b1 + 1], mk4<S>(w1.x, w1.y, w1.z, S(0)));
    }
    if (!(info & CI_ZERO2)) {
        st4(&d.vel[2 * b2], mk4<S>(v2.x, v2.y, v2.z, S(0)));
        st4(&d.vel[2 * b2 + 1], mk4<S>(w2.x, w2.y, w2.z, S(0)));
    }
#undef ROW_A
#undef ROW_B
#undef ROW_D
}

// ---- wavefront mode: warm_start / solve_contacts<BIAS> / relax of ONE manifold --------------------------------------------------------
// The same arithmetic in the same order as contact_item (bit-identical); what differs is where the operands live and when the item waits.
//   * Rolled point loops.  Each point's impulses live in this thread's scratch rows of the staging tile (rows 3*MAXP + k), so no register
//     array is indexed dynamically and nothing goes to local memory.  One routine serves the biased and the relax pass (`relax`): fewer
//     routines compete for the SM's instruction cache, whose warps are in several routines at once.
//   * Two-stage wait (solve passes).  A body's deltas change only at its integrate_positions, so stage 1 waits until each body's counter has
//     passed the integrate_positions event that wrote the deltas this pass reads — nearly always true at the first look — then loads them and
//     computes every point's separation and the velocity-independent coefficients of its normal impulse.  Stage 2 waits for the exact event
//     (no poll for a lane whose stage-1 poll already read it) and loads the velocities and impulses.  When about as many warps are resident
//     as a colour has chunks, a warp goes from one level's item straight to the next one's and stage 1 is on the chain, so it is kept short.
//   * Branch-free normal part.  Every case of ContactNormalPart::solve_impulse is impulse = -M * (vn + B) - C, with M and B from stage 1 and
//     C a select, so the lanes of a warp no longer run the separated, biased and relax paths one after another.
//   * Early record stores.  A point's record is stored as soon as it is final (in the normal loop without friction, in the friction loop
//     with it), so those stores are in flight during the rest of the arithmetic and the release fence mostly waits for the velocities.
//   * Acquire / release counters (wave_wait / wave_publish): no membar after a successful poll, one fence before the counter stores.
// PASS = PASS_WARM or PASS_SOLVE_BIAS.  Every lane of the warp must call this (warp-collective waits).  Counters count from the prepare
// launch on, so `s` is the absolute substep index in every launch of a step.
template <class S, int PASS, int MAXP>
__device__ __forceinline__ void wave_contact_item(const DevSolver<S>& d, int slot, int s, int it, bool relax) {
    constexpr bool SOLVE = PASS == PASS_SOLVE_BIAS;
    relax = SOLVE && relax;
    const size_t MP = size_t(d.Mpad);
    const Vec4<S>* c = d.cst + slot;
    const Vec4<S> hidx = ld4(&c[CP_IDX * MP]);
    const int info = as_int(hidx.z);
    const int np = info & CI_NP_MASK;
    const int b1 = as_int(hidx.x), b2 = as_int(hidx.y);
    Vec4<S>* const stage = stage_base<S>() + threadIdx.x;   // this thread's column; row r at stage[r * T]
    const int T = blockDim.x;
    // Staged rows of point k.  Stage 1 of a solve pass overwrites the w lanes of A and B (the initial separation and the normal effective
    // mass, which nothing after it reads) with the coefficients B and M of the point's normal impulse.
#define ROW_A(k) stage[(3 * (k) + 0) * T]
#define ROW_B(k) stage[(3 * (k) + 1) * T]
#define ROW_D(k) stage[(3 * (k) + 2) * T]
#define ROW_PC(k) stage[(3 * MAXP + (k)) * T]
    // ---- immutable part (planes written by prepare, inertia): issued before any wait
    Vec4<S> hn = mk4<S>(0, 0, 0, 0), ht1 = hn, htv = hn;
    BodyInertia<S> in1 = zero_inertia<S>(), in2 = zero_inertia<S>();
    if (np != 0) {
        hn = ld4(&c[CP_N * MP]);
        ht1 = ld4(&c[CP_T1 * MP]);
        if (SOLVE) htv = ld4(&c[CP_TV * MP]);
        if (!(info & CI_ZERO1)) in1 = unpack_inertia(ld4(&d.inr[2 * b1]), ld4(&d.inr[2 * b1 + 1]));
        if (!(info & CI_ZERO2)) in2 = unpack_inertia(ld4(&d.inr[2 * b2]), ld4(&d.inr[2 * b2 + 1]));
#pragma unroll 1
        for (int k = 0; k < np; ++k) {
            stage_copy(&ROW_A(k), &c[size_t(CP_ROW(k, 0)) * MP]);
            stage_copy(&ROW_B(k), &c[size_t(CP_ROW(k, 1)) * MP]);
            if (SOLVE && (info & CI_TANGENT)) stage_copy(&ROW_D(k), &c[size_t(CP_ROW(k, 2)) * MP]);
        }
    }
    __pipeline_commit();
    const bool ver1 = np != 0 && (info & CI_VER1), ver2 = np != 0 && (info & CI_VER2);
    const int rk = as_int(hidx.w);
    const int k1 = (rk >> 8) & 0xff, k2 = (rk >> 24) & 0xff;
    const int kind = SOLVE ? (relax ? WV_RELAX : WV_SOLVE) : WV_WARM;
    const unsigned e1 = wave_event(kind, it, s, d.iters, k1, rk & 0xff);
    const unsigned e2 = wave_event(kind, it, s, d.iters, k2, (rk >> 16) & 0xff);
    int* const watchdog = d.any_restitution + FLAG_WAVE;
    const V3<S> n = xyz(hn), t1 = xyz(ht1);
    const Soft<S> soft = (info & CI_NONDYN) ? d.soft_nondyn : d.soft_dyn;
    unsigned biased_points = 0;   // bit k: point k takes the biased case (C = impulse_scale * accumulated impulse)
    // the counter values stage 1's polls last read: a lane that already read its exact event there skips the first poll of stage 2 (the
    // counter cannot pass that event before this item publishes, and the acquire of that poll orders every later load)
    unsigned seen1 = 0u, seen2 = 0u;

    // ---- stage 1 (solve passes): the deltas -> the separation of every point -> the coefficients of its normal impulse
    if (SOLVE) {
        AVN_TRACE_T(t_d0);
        const int sd = relax ? s : s - 1;   // the substep whose integrate_positions wrote the deltas this pass reads (-1: prepare did)
        if (sd >= 0)
            wave_wait<false>(d.ver, ver1, b1, wave_event(WV_IP, 0, sd, d.iters, k1, 0) + 1u, ver2, b2, wave_event(WV_IP, 0, sd, d.iters, k2, 0) + 1u,
                             watchdog, &seen1, &seen2);
        __pipeline_wait_prior(0);   // this thread's staged rows have landed (only the issuing thread reads them)
        if (np != 0) {
            const Vec4<S> dp1 = ld4_cg(&d.dlt[2 * b1]), dq1 = ld4_cg(&d.dlt[2 * b1 + 1]);
            const Vec4<S> dp2 = ld4_cg(&d.dlt[2 * b2]), dq2 = ld4_cg(&d.dlt[2 * b2 + 1]);
            Q4<S> q1; q1.x = dq1.x; q1.y = dq1.y; q1.z = dq1.z; q1.w = dq1.w;
            Q4<S> q2; q2.x = dq2.x; q2.y = dq2.y; q2.z = dq2.z; q2.w = dq2.w;
            const V3<S> delta_translation = xyz(dp2) - xyz(dp1);
            // unrolled: the points are independent here, so their rotations and coefficients interleave instead of running one after another
#pragma unroll
            for (int k = 0; k < MAXP; ++k) {
                if (k >= np) break;
                const Vec4<S> PAk = ROW_A(k), PBk = ROW_B(k);
                V3<S> rr1 = qrot(q1, xyz(PAk)), rr2 = qrot(q2, xyz(PBk));
                V3<S> dsep = delta_translation + (rr2 - rr1);
                const S separation = dot(dsep, n) + PAk.w;
                // ContactNormalPart::solve_impulse (normal_part.rs:116-166) as impulse = -M * (vn + B) - C.  Per case, the operations of
                // the reference in the same order:
                //   separation > 0:  -meff * (vn + separation / h)                  M = meff,               B = separation / h,  C = +0
                //   biased:          -scaled_mass * (vn + bias) - scaled_impulse     M = mass_scale * meff,  B = bias,            C = impulse_scale * acc
                //   relax:           -meff * vn                                      M = meff,               B = -0,              C = +0
                // with bias = max(soft.bias * separation, -max_overlap_speed).  The added operations are exact: x - (+0) == x and
                // x + (-0) == x bit for bit for every x, -0 included.
                const S meff = PBk.w;
                const bool separated = separation > S(0), biased = !separated && !relax;
                ROW_A(k).w = separated ? separation / d.h : biased ? avn_max(soft.bias * separation, -d.max_overlap_speed) : S(-0.0);   // B
                ROW_B(k).w = biased ? soft.mass_scale * meff : meff;                                                                    // M
                biased_points |= unsigned(biased) << k;
            }
        }
#ifdef AVN_WAVE_TRACE
        if (np != 0 && ROW_A(0).w == S(1.2345e33)) d.any_restitution[1] = 2;   // the coefficients are done here
        AVN_TRACE_ADD(d, 5, clock64() - t_d0);
#endif
    }

    // ---- stage 2: the exact event, then the velocities of the two bodies and the impulses of the points
    AVN_TRACE_T(t_w0);
    wave_wait(d.ver, ver1 && seen1 != e1, b1, e1, ver2 && seen2 != e2, b2, e2, watchdog);
    AVN_TRACE_ADD(d, 0, clock64() - t_w0);
    if (np == 0) return;   // padding slot (after the warp-collective waits)
    AVN_TRACE_T(t_l0);
    const Vec4<S> l1 = ld4_cg(&d.vel[2 * b1]), a1 = ld4_cg(&d.vel[2 * b1 + 1]);
    const Vec4<S> l2 = ld4_cg(&d.vel[2 * b2]), a2 = ld4_cg(&d.vel[2 * b2 + 1]);
    {   // all impulse loads in flight at once, then parked in the scratch rows
        Vec4<S> pc[MAXP];
#pragma unroll
        for (int k = 0; k < MAXP; ++k)
            if (k < np) pc[k] = pc_load<true>(pc_ptr(d, k, slot));
#pragma unroll
        for (int k = 0; k < MAXP; ++k)
            if (k < np) ROW_PC(k) = pc[k];
    }
    if (!SOLVE) __pipeline_wait_prior(0);
#ifdef AVN_WAVE_TRACE
    if ((l1.x + a1.x + l2.x + a2.x) == S(1.2345e33)) d.any_restitution[1] = 2;   // force the loads to complete here
    AVN_TRACE_T(t_c0);
    AVN_TRACE_ADD(d, 1, t_c0 - t_l0);
#endif
    V3<S> v1 = xyz(l1), w1 = xyz(a1), v2 = xyz(l2), w2 = xyz(a2);
    const V3<S> t2 = cross(t1, n);  // tangent_directions(): [tangent1, tangent1 x normal] (contact/mod.rs:411-421)

    if (!SOLVE) {
        // ContactConstraint::warm_start (contact/mod.rs:223-264)
#pragma unroll 1
        for (int k = 0; k < np; ++k) {
            const Vec4<S> PAk = ROW_A(k), PBk = ROW_B(k), pck = ROW_PC(k);
            V3<S> r1 = xyz(PAk), r2 = xyz(PBk);
            S tx = (info & CI_TANGENT) ? pck.z : S(0), ty = (info & CI_TANGENT) ? pck.w : S(0);
            V3<S> p = d.warm_coeff * ((pck.x * n + tx * t1) + ty * t2);
            apply_impulse(v1, w1, v2, w2, in1, in2, r1, r2, p);
        }
    } else {
        // ContactConstraint::solve (contact/mod.rs:267-354)
        const bool tangent = (info & CI_TANGENT) != 0;
#pragma unroll 1
        for (int k = 0; k < np; ++k) {
            const Vec4<S> PAk = ROW_A(k), PBk = ROW_B(k);
            Vec4<S> pck = ROW_PC(k);
            V3<S> r1 = xyz(PAk), r2 = xyz(PBk);
            V3<S> relv = (v2 + cross(w2, r2)) - (v1 + cross(w1, r1));
            // ContactNormalPart::solve_impulse (normal_part.rs:116-166), M and B from stage 1
            S vn = dot(relv, n);
            S acc = pck.x;
            const S C = ((biased_points >> k) & 1u) ? soft.impulse_scale * acc : S(0);
            S impulse = -PBk.w * (vn + PAk.w) - C;
            S new_impulse = avn_max(acc + impulse, S(0));
            impulse = new_impulse - acc;
            pck.x = new_impulse;
            pck.y = pck.y + new_impulse;
            if (tangent) ROW_PC(k) = pck;
            else pc_store(pc_ptr(d, k, slot), pck);   // final: no friction part
            apply_impulse(v1, w1, v2, w2, in1, in2, r1, r2, impulse * n);
        }
        if (tangent) {
            const S friction = hn.w;
            const V3<S> surf = xyz(htv);
#pragma unroll 1
            for (int k = 0; k < np; ++k) {
                const Vec4<S> PAk = ROW_A(k), PBk = ROW_B(k), PDk = ROW_D(k);
                Vec4<S> pck = ROW_PC(k);
                V3<S> r1 = xyz(PAk), r2 = xyz(PBk);
                V3<S> relv = (v2 + cross(w2, r2)) - (v1 + cross(w1, r1));
                // ContactTangentPart::solve_impulse (tangent_part.rs:155-244)
                S limit = friction * pck.x;
                relv = relv + surf;
                S ts1 = dot(relv, t1), ts2 = dot(relv, t2);
                S t11 = ts1 * ts1, t22 = ts2 * ts2, t12 = ts1 * ts2;
                S inv = (t11 * PDk.x + t22 * PDk.y) + t12 * PDk.z;
                S em = (t11 + t22) * (S(1) / inv);
                V3<S> imp = zero3<S>();
                if (avn_finite(em)) {
                    S nx = pck.z - em * ts1, ny = pck.w - em * ts2;
                    S l2 = nx * nx + ny * ny;
                    if (l2 > limit * limit) {  // Vec2::clamp_length_max
                        S l = avn_sqrt(l2);
                        nx = limit * (nx / l);
                        ny = limit * (ny / l);
                    }
                    S dx = nx - pck.z, dy = ny - pck.w;
                    pck.z = nx;
                    pck.w = ny;
                    imp = dx * t1 + dy * t2;
                }
                pc_store(pc_ptr(d, k, slot), pck);   // final
                apply_impulse(v1, w1, v2, w2, in1, in2, r1, r2, imp);
            }
        }
    }
    // ---- write back: the velocities of the non-dominant sides, then the counters
#ifdef AVN_WAVE_TRACE
    if ((v1.x + v2.x + w1.x + w2.x) == S(1.2345e33)) d.any_restitution[1] = 2;
    AVN_TRACE_T(t_s0);
    AVN_TRACE_ADD(d, 2, t_s0 - t_c0);
#endif
    if (!(info & CI_ZERO1)) {
        st4(&d.vel[2 * b1], mk4<S>(v1.x, v1.y, v1.z, S(0)));
        st4(&d.vel[2 * b1 + 1], mk4<S>(w1.x, w1.y, w1.z, S(0)));
    }
    if (!(info & CI_ZERO2)) {
        st4(&d.vel[2 * b2], mk4<S>(v2.x, v2.y, v2.z, S(0)));
        st4(&d.vel[2 * b2 + 1], mk4<S>(w2.x, w2.y, w2.z, S(0)));
    }
    wave_publish(d.ver, ver1, b1, e1, ver2, b2, e2);   // the fence also orders the record stores before the counters
#ifdef AVN_WAVE_TRACE
    AVN_TRACE_ADD(d, 3, clock64() - t_s0);
    AVN_TRACE_ADD(d, 4, 1);
#endif
#undef ROW_A
#undef ROW_B
#undef ROW_D
#undef ROW_PC
}

// ---------------------------------------------------------------------------------------------------------
// integrate_velocities + clamp_velocities (integrator/mod.rs:343-391, 467-500)
// ---------------------------------------------------------------------------------------------------------
// WAVE: every lane of the warp calls this (i may be >= B: padding); `s` = substep index
template <class S, bool WAVE = false>
__device__ __forceinline__ void integrate_velocity_item(const DevSolver<S>& d, int i, int s = 0) {
    const bool in_range = i < d.B;
    int f = 0;
    if (in_range) f = as_int(ld4(&d.inr[2 * i]).y);
    const bool live = in_range && (f & BF_HAS_SOLVER_BODY);
    // the immutable inputs are loaded before the wait: the poll's "memory" clobber would keep them behind it, one more round trip on the chain
    const bool integrate = live && !(f & BF_CUSTOM_VEL) && !(f & BF_KINEMATIC), gyro = integrate && (f & BF_GYRO);
    Vec4<S> li = mk4<S>(0, 0, 0, 0), ai = li;
    Q4<S> rot0; rot0.x = rot0.y = rot0.z = rot0.w = S(0);
    Sym3<S> il; il.m00 = il.m01 = il.m02 = il.m11 = il.m12 = il.m22 = S(0);
    if (integrate) { li = ld4(&d.itg[2 * i]); ai = ld4(&d.itg[2 * i + 1]); }
    if (gyro) {
        rot0 = ldq(d.rotation, i);
        il.m00 = d.inv_inertia_local[6 * i]; il.m01 = d.inv_inertia_local[6 * i + 1]; il.m02 = d.inv_inertia_local[6 * i + 2];
        il.m11 = d.inv_inertia_local[6 * i + 3]; il.m12 = d.inv_inertia_local[6 * i + 4]; il.m22 = d.inv_inertia_local[6 * i + 5];
    }
    const S max_lin = live && d.max_lin ? d.max_lin[i] : S(0), max_ang = live && d.max_ang ? d.max_ang[i] : S(0);
    const int bnd = live && d.bnd_of ? d.bnd_of[i] : -1;
    unsigned e = 0;
    if (WAVE) {
        if (live) e = wave_event(WV_IV, 0, s, d.iters, d.deg[i], 0);
        wave_wait(d.ver, live, i, e, false, 0, 0u, d.any_restitution + 1);
    }
    if (!live) return;
    Vec4<S> l = ldm<WAVE>(&d.vel[2 * i]), a = ldm<WAVE>(&d.vel[2 * i + 1]);
    V3<S> v = xyz(l), w = xyz(a);
    bool touched = false;
    if (integrate) {
        v = v * li.w;
        w = w * ai.w;
        v = v + xyz(li);
        w = w + xyz(ai);
        if (gyro) {
            // solve_gyroscopic_torque (integrator/mod.rs:403-460)
            Vec4<S> dq4 = ldm<WAVE>(&d.dlt[2 * i + 1]);
            Q4<S> dq; dq.x = dq4.x; dq.y = dq4.y; dq.z = dq4.z; dq.w = dq4.w;
            Q4<S> rot = qmul(dq, rot0);
            V3<S> lw = qrot(qconj(rot), w);
            Sym3<S> tensor = sym_inverse_or_zero(il);
            V3<S> L = smul(tensor, lw);
            V3<S> Ln = L - d.h * cross(lw, L);
            S l2 = len2(Ln);
            if (l2 == S(0)) {
                w = zero3<S>();
            } else {
                Ln = Ln * avn_sqrt(len2(L) / l2);
                w = qrot(rot, smul(il, Ln));
            }
        }
        touched = true;
    }
    if (d.max_lin) {
        S l2 = len2(v);
        if (avn_finite(max_lin) && l2 > max_lin * max_lin) { v = v * (max_lin / avn_sqrt(l2)); touched = true; }
    }
    if (d.max_ang) {
        S l2 = len2(w);
        if (avn_finite(max_ang) && l2 > max_ang * max_ang) { w = w * (max_ang / avn_sqrt(l2)); touched = true; }
    }
    if (touched) {
        st4(&d.vel[2 * i], mk4<S>(v.x, v.y, v.z, S(0)));
        st4(&d.vel[2 * i + 1], mk4<S>(w.x, w.y, w.z, S(0)));
    }
    if (bnd >= 0) {  // partitioned step: the reference point of this substep's constraint impulses on a boundary body
        st4(&d.vel_ref[2 * bnd], mk4<S>(v.x, v.y, v.z, S(0)));
        st4(&d.vel_ref[2 * bnd + 1], mk4<S>(w.x, w.y, w.z, S(0)));
    }
    if (WAVE) wave_publish(d.ver, true, i, e, false, 0, 0u);
}

// integrate_positions (integrator/mod.rs:503-535)
template <class S, bool WAVE = false>
__device__ __forceinline__ void integrate_position_item(const DevSolver<S>& d, int i, int s = 0) {
    const bool in_range = i < d.B;
    int f = 0;
    if (in_range) f = as_int(ld4(&d.inr[2 * i]).y);
    const bool live = in_range && (f & BF_HAS_SOLVER_BODY);
    unsigned e = 0;
    if (WAVE) {
        if (live) e = wave_event(WV_IP, 0, s, d.iters, d.deg[i], 0);
        wave_wait(d.ver, live, i, e, false, 0, 0u, d.any_restitution + 1);
    }
    if (!live) return;
    if (f & BF_CUSTOM_POS) {
        if (WAVE) wave_publish(d.ver, true, i, e, false, 0, 0u);
        return;
    }
    Vec4<S> l = ldm<WAVE>(&d.vel[2 * i]), a = ldm<WAVE>(&d.vel[2 * i + 1]);
    Vec4<S> dp = ldm<WAVE>(&d.dlt[2 * i]), dq4 = ldm<WAVE>(&d.dlt[2 * i + 1]);
    V3<S> ndp = xyz(dp) + xyz(l) * d.h;
    Q4<S> dq; dq.x = dq4.x; dq.y = dq4.y; dq.z = dq4.z; dq.w = dq4.w;
    Q4<S> nq = qmul(q_from_scaled_axis(xyz(a) * d.h, d.fast_trig != 0), dq);
    st4(&d.dlt[2 * i], mk4<S>(ndp.x, ndp.y, ndp.z, S(0)));
    st4(&d.dlt[2 * i + 1], mk4<S>(nq.x, nq.y, nq.z, nq.w));
    if (WAVE) wave_publish(d.ver, true, i, e, false, 0, 0u);
}

// ---- wavefront prologue: ranks of every constraint on its two bodies (colour by colour), then pack {r1,k1,r2,k2} ------
// Within one colour a versioned body appears at most once (constraint_graph.rs:4-6), so the per-colour pass is race-free.
// The per-colour pass trusts the colouring only as far as it checks it: every versioned body is stamped with the colour that ranks it
// (atomicExch); meeting its own colour's stamp again means the caller listed the body twice in one colour — a colouring the wavefront
// schedule would turn into wrong event numbers and a spin until the watchdog — so the flag WAVE_BAD_COLOURING is raised instead, the kernel
// falls back to the barrier schedule for this step and avn_solver_download reports AVN_ERR_INVALID_ARGUMENT.
enum { WAVE_WATCHDOG = 1, WAVE_BAD_COLOURING = 3 };
template <class S>
__device__ __forceinline__ void wave_rank_item(const DevSolver<S>& d, int slot) {
    const size_t MP = size_t(d.Mpad);
    Vec4<S>* c = d.cst + slot;
    Vec4<S> hidx = ld4(&c[CP_IDX * MP]);
    const int info = as_int(hidx.z);
    if ((info & CI_NP_MASK) == 0) return;
    const int b1 = as_int(hidx.x), b2 = as_int(hidx.y);
    int colour = 0;
    while (colour < AVN_GRAPH_COLOR_COUNT - 1 && slot >= d.color_off[colour + 1]) ++colour;
    int r1 = 0, r2 = 0;
    bool bad = false;
    if (info & CI_VER1) { bad |= atomicExch(&d.stamp[b1], colour + 1) == colour + 1; r1 = atomicAdd(&d.deg[b1], 1); }
    if (info & CI_VER2) { bad |= atomicExch(&d.stamp[b2], colour + 1) == colour + 1; r2 = atomicAdd(&d.deg[b2], 1); }
    if (bad || r1 > 0xfe || r2 > 0xfe) d.any_restitution[1] = WAVE_BAD_COLOURING;
    hidx.w = int_as(S(0), (r1 & 0xff) | ((r2 & 0xff) << 16));
    st4(&c[CP_IDX * MP], hidx);
}
template <class S>
__device__ __forceinline__ void wave_pack_item(const DevSolver<S>& d, int slot) {
    const size_t MP = size_t(d.Mpad);
    Vec4<S>* c = d.cst + slot;
    Vec4<S> hidx = ld4(&c[CP_IDX * MP]);
    const int info = as_int(hidx.z);
    if ((info & CI_NP_MASK) == 0) return;
    const int b1 = as_int(hidx.x), b2 = as_int(hidx.y);
    int rk = as_int(hidx.w);
    if (info & CI_VER1) rk |= (d.deg[b1] & 0xff) << 8;
    if (info & CI_VER2) rk |= (d.deg[b2] & 0xff) << 24;
    hidx.w = int_as(S(0), rk);
    st4(&c[CP_IDX * MP], hidx);
}

// writeback_solver_bodies (solver_body/plugin.rs:255-284)
template <class S>
__device__ __forceinline__ void writeback_body_item(const DevSolver<S>& d, int i) {
    Vec4<S> ia = ld4(&d.inr[2 * i]);
    int f = as_int(ia.y);
    V3<S> pos = ldv3(d.position, i);
    Q4<S> rot = ldq(d.rotation, i);
    V3<S> lv = ldv3(d.linvel, i), av = ldv3(d.angvel, i);
    if (f & BF_HAS_SOLVER_BODY) {
        Vec4<S> l = ld4(&d.vel[2 * i]), a = ld4(&d.vel[2 * i + 1]);
        Vec4<S> dp = ld4(&d.dlt[2 * i]), dq4 = ld4(&d.dlt[2 * i + 1]);
        V3<S> com = ldv3_or0(d.com, i);
        V3<S> old_com = qrot(rot, com);
        Q4<S> dq; dq.x = dq4.x; dq.y = dq4.y; dq.z = dq4.z; dq.w = dq4.w;
        rot = q_fast_renormalize(qmul(dq, rot));
        V3<S> new_com = qrot(rot, com);
        pos = pos + ((xyz(dp) + old_com) - new_com);
        lv = xyz(l);
        av = xyz(a);
    }
    stv3(d.out_position, i, pos);
    d.out_rotation[4 * i] = rot.x; d.out_rotation[4 * i + 1] = rot.y; d.out_rotation[4 * i + 2] = rot.z; d.out_rotation[4 * i + 3] = rot.w;
    stv3(d.out_linvel, i, lv);
    stv3(d.out_angvel, i, av);
}

// store_contact_impulses (solver/plugin.rs:722-755)
template <class S>
__device__ __forceinline__ void store_impulse_item(const DevSolver<S>& d, int m) {
    const size_t MP = size_t(d.Mpad);
    const int slot = slot_of_manifold(d, m);
    const Vec4<S>* c = d.cst + slot;
    Vec4<S> hidx = ld4(&c[CP_IDX * MP]);
    int info = as_int(hidx.z), np = info & CI_NP_MASK, p0 = int(d.m_point_begin[m]);
    if (np == 0) {  // skipped by prepare (both bodies non-dynamic): the reference leaves the ContactPoints untouched
        for (uint32_t p = d.m_point_begin[m]; p < d.m_point_end[m]; ++p) {
            d.p_out_ws_normal[p] = d.p_ws_normal[p];
            d.p_out_ws_tangent[2 * p] = d.p_ws_tangent[2 * p];
            d.p_out_ws_tangent[2 * p + 1] = d.p_ws_tangent[2 * p + 1];
            d.p_normal_impulse[p] = d.p_in_normal_impulse ? d.p_in_normal_impulse[p] : S(0);
        }
        return;
    }
    for (int k = 0; k < np; ++k) {
        Vec4<S> pc = pc_load<false>(pc_ptr(d, k, slot));
        d.p_out_ws_normal[p0 + k] = pc.x;
        d.p_out_ws_tangent[2 * (p0 + k)] = (info & CI_TANGENT) ? pc.z : S(0);
        d.p_out_ws_tangent[2 * (p0 + k) + 1] = (info & CI_TANGENT) ? pc.w : S(0);
        d.p_normal_impulse[p0 + k] = pc.y;
    }
}

}  // namespace avn
