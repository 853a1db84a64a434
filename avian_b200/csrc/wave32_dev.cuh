// Wavefront schedule, f32: SEQUENCE-TAGGED RECORDS (sm_90a).  EXPERIMENT, built only with -DAVN_WAVE_RECORDS_F32: the 16-byte
// no-tearing property below is not promised by the PTX memory model, and on the H100 the records gave stale reads (solver_kernels.cuh).
//
// The wavefront substep loop (solver_dev.cuh "wavefront mode") replaces grid barriers by per-body event numbers: an item may run when the
// event counters of its bodies equal its position in their event sequences.  Round 1 kept the counters in their own array and passed the
// data by message passing: stores -> __threadfence -> counter store | counter poll -> __threadfence -> data loads, and every dependency hop
// paid  store ack + counter hop + poll + fence + a second L2 round trip for the data.
//
// Here every MUTABLE datum an item consumes sits in a 32-byte record that carries its own sequence tag, read and written with 128-bit
// strong accesses (ld/st.relaxed.gpu.global.v4.f32), the widest single access Hopper has:
//     velocity record  vel[2b..2b+1]  = {lin.xyz, EVENTS | ang.xyz, EVENTS}   EVENTS = number of schedule events completed on body b
//     impulse record   pcr[(k,slot)]  = {ln, sum, WRITES, - | lt.x, lt.y, WRITES, -}   WRITES = passes that have written the point's impulses
//     delta record     dlt[2b..2b+1]  = {dp.xyz, IPS | dq.xyzw}          IPS    = integrate_positions steps completed on body b
// A consumer knows the tag every record must carry when all its predecessors are done (the same arithmetic the event numbers came from),
// loads the records and simply repeats the loads until every tag matches.  A successful poll IS the data: no counter array, no fence, no
// second round trip; a producer publishes by storing its records, in any order.  The hardware property relied on is that a naturally
// aligned 16-byte vector access is performed as one transaction (no tearing inside a quad).  The velocity and impulse records carry the
// tag in BOTH quads, and a tag value is written once per record, so two quads with the expected tag come from the same store.
// The delta record has no lane left for a second tag (the rotation fills its quad): its producer stores the rotation quad, then the tagged
// quad with release semantics, and the consumer polls the tagged quad with acquire semantics before it reads the rotation.  It changes
// once per substep, so the fence this costs stays off the per-item chain of the velocity records.
// The separation terms of a solve pass depend only on the delta records: they are computed BEFORE the wait on the velocity records (the
// delta records are usually valid at the first look), so ~20 % of an item's arithmetic leaves the critical path.
//
// f64 keeps the counter protocol: a Vec4<double> fills a whole quad pair, so there is no lane left for a tag.
#pragma once

namespace avn {

struct Rec32 { Vec4<float> a, b; };
__device__ __forceinline__ Vec4<float> ld_q(const Vec4<float>* p) {
    Vec4<float> r;
    asm volatile("ld.relaxed.gpu.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ Vec4<float> ld_q_acquire(const Vec4<float>* p) {
    Vec4<float> r;
    asm volatile("ld.acquire.gpu.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ void st_q(Vec4<float>* p, float a0, float a1, float a2, float a3) {
    asm volatile("st.relaxed.gpu.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(a0), "f"(a1), "f"(a2), "f"(a3) : "memory");
}
__device__ __forceinline__ void st_q_release(Vec4<float>* p, float a0, float a1, float a2, float a3) {
    asm volatile("st.release.gpu.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(a0), "f"(a1), "f"(a2), "f"(a3) : "memory");
}
__device__ __forceinline__ unsigned tag_of(float lane) { return __float_as_uint(lane); }
__device__ __forceinline__ float tag_lane(unsigned t) { return __uint_as_float(t); }

// velocity record {lin.xyz, T | ang.xyz, T}
__device__ __forceinline__ Rec32 ld_vel(const Vec4<float>* p) { Rec32 r; r.a = ld_q(p); r.b = ld_q(p + 1); return r; }
__device__ __forceinline__ bool vel_is(const Rec32& r, unsigned t) { return tag_of(r.a.w) == t && tag_of(r.b.w) == t; }
__device__ __forceinline__ void st_vel(Vec4<float>* p, V3<float> v, V3<float> w, unsigned t) {
    st_q(p, v.x, v.y, v.z, tag_lane(t));
    st_q(p + 1, w.x, w.y, w.z, tag_lane(t));
}
// impulse record {ln, sum, T, - | lt.x, lt.y, T, -}; its value as {ln, sum, lt.x, lt.y}
__device__ __forceinline__ Rec32 ld_pc(const Vec4<float>* p) { Rec32 r; r.a = ld_q(p); r.b = ld_q(p + 1); return r; }
__device__ __forceinline__ bool pc_is(const Rec32& r, unsigned t) { return tag_of(r.a.z) == t && tag_of(r.b.z) == t; }
__device__ __forceinline__ Vec4<float> pc_val(const Rec32& r) { return mk4<float>(r.a.x, r.a.y, r.b.x, r.b.y); }
__device__ __forceinline__ void st_pc(Vec4<float>* p, Vec4<float> v, unsigned t) {
    st_q(p, v.x, v.y, tag_lane(t), 0.f);
    st_q(p + 1, v.z, v.w, tag_lane(t), 0.f);
}
// delta record {dp.xyz, T | dq.xyzw}: rotation first, then the tag with release semantics; read back in the opposite order
__device__ __forceinline__ Rec32 ld_dlt(const Vec4<float>* p) { Rec32 r; r.a = ld_q_acquire(p); r.b = ld_q(p + 1); return r; }
__device__ __forceinline__ void st_dlt(Vec4<float>* p, V3<float> dp, unsigned t, Vec4<float> dq) {
    st_q(p + 1, dq.x, dq.y, dq.z, dq.w);
    st_q_release(p, dp.x, dp.y, dp.z, tag_lane(t));
}

constexpr unsigned W32_SPIN_LIMIT = 1u << 22;

// impulse-record tag: passes that have written the record before the given pass of substep s (writers: `iters` biased passes + the relax pass)
__device__ __forceinline__ unsigned w32_pc_tag(int pass, int s, int it, int iters) {
    const unsigned base = unsigned(s) * unsigned(iters + 1);
    return pass == PASS_RELAX ? base + unsigned(iters) : (pass == PASS_SOLVE_BIAS ? base + unsigned(it) : base);
}

// ---------------------------------------------------------------------------------------------------------
// warm_start / solve_contacts<BIAS> / relax for ONE manifold, wavefront mode (same arithmetic as contact_item, solver_dev.cuh)
// Every lane of the warp must call this (warp-collective polls).
// ---------------------------------------------------------------------------------------------------------
template <int PASS, int MAXP>
__device__ __forceinline__ void w32_contact_item(const DevSolver<float>& d, int slot, int s, int it, bool lane_active, int wf, int pass) {
    // PASS = PASS_WARM or PASS_SOLVE_BIAS; the solve build serves the biased AND the relax pass (`pass` says which): one routine in the
    // instruction cache instead of two
    const bool relax = PASS != PASS_WARM && pass == PASS_RELAX;
    using S = float;
    const size_t MP = size_t(d.Mpad);
    const Vec4<S>* c = d.cst + (lane_active ? slot : 0);
    const Vec4<S> hidx = ld4(&c[CP_IDX * MP]);
    const int info = lane_active ? as_int(hidx.z) : 0;   // an inactive lane of a partial chunk behaves like a padding slot
    const int np = info & CI_NP_MASK;
    const int b1 = as_int(hidx.x), b2 = as_int(hidx.y);
    constexpr bool SOLVE = (PASS == PASS_SOLVE_BIAS || PASS == PASS_RELAX);
    Vec4<S>* const stage = stage_base<S>() + threadIdx.x;
    const int T = blockDim.x;
#define ROW_A(k) stage[(3 * (k) + 0) * T]
#define ROW_B(k) stage[(3 * (k) + 1) * T]
#define ROW_D(k) stage[(3 * (k) + 2) * T]
    // the item's own scratch rows behind the staged ones: the impulses of its points and their separations.  They live in shared memory so
    // that the loops over the points can stay ROLLED (dynamic index, no local memory): the solve and relax routines shrink from 42 KB of
    // SASS to a quarter, which matters because the SM's instruction cache (32 KB L1.5) serves warps that are in five different routines
    // at once in the wavefront schedule
#define ROW_PC(k) stage[(3 * MAXP + (k)) * T]
    float* const sepv = reinterpret_cast<float*>(&stage[(4 * MAXP) * T]);
    // ---- immutable part: issued before any wait
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
    const int kind = PASS == PASS_WARM ? WV_WARM : (relax ? WV_RELAX : WV_SOLVE);
    const unsigned e1 = wave_event(kind, it, s, d.iters, (rk >> 8) & 0xff, rk & 0xff, wf);
    const unsigned e2 = wave_event(kind, it, s, d.iters, (rk >> 24) & 0xff, (rk >> 16) & 0xff, wf);
    const unsigned ptag = w32_pc_tag(PASS == PASS_WARM ? PASS_WARM : (relax ? PASS_RELAX : PASS_SOLVE_BIAS), s, it, d.iters);
    const V3<S> n = xyz(hn), t1 = xyz(ht1);
    AVN_TRACE_T(t_w0);

    // ---- stage 1 (solve passes): the delta records -> separation of every point, before the velocities are even looked at
    if (SOLVE) {
        const unsigned dtag = unsigned(relax ? s + 1 : s);
        Rec32 D1, D2;
        D1.a = mk4<S>(0, 0, 0, 0); D1.b = mk4<S>(0, 0, 0, 1); D2 = D1;
        bool n1 = ver1, n2 = ver2;
        if (np != 0 && !ver1) { D1.a = ld4(&d.dlt[2 * b1]); D1.b = ld4(&d.dlt[2 * b1 + 1]); }   // no SolverBody: constant (0, identity)
        if (np != 0 && !ver2) { D2.a = ld4(&d.dlt[2 * b2]); D2.b = ld4(&d.dlt[2 * b2 + 1]); }
        for (unsigned spins = 0;; ++spins) {
            if (n1) D1 = ld_dlt(&d.dlt[2 * b1]);
            if (n2) D2 = ld_dlt(&d.dlt[2 * b2]);
            if (n1) n1 = tag_of(D1.a.w) != dtag;
            if (n2) n2 = tag_of(D2.a.w) != dtag;
            if (__all_sync(0xffffffffu, !(n1 || n2))) break;
            if (spins > W32_SPIN_LIMIT) { d.any_restitution[1] = WAVE_WATCHDOG; break; }
            if (d.poll_ns) __nanosleep(unsigned(d.poll_ns));   // (experiment: back off between polls, AVN_WAVE_POLL_NS)
        }
        __pipeline_wait_prior(0);   // this thread's staged rows have landed (only the issuing thread reads them)
        AVN_TRACE_T(t_p0);
        AVN_TRACE_ADD(d, 5, t_p0 - t_w0);
        if (np != 0) {
            Q4<S> q1; q1.x = D1.b.x; q1.y = D1.b.y; q1.z = D1.b.z; q1.w = D1.b.w;
            Q4<S> q2; q2.x = D2.b.x; q2.y = D2.b.y; q2.z = D2.b.z; q2.w = D2.b.w;
            const V3<S> delta_translation = xyz(D2.a) - xyz(D1.a);
#pragma unroll 1
            for (int k = 0; k < np; ++k) {
                const Vec4<S> PAk = ROW_A(k), PBk = ROW_B(k);
                V3<S> rr1 = qrot(q1, xyz(PAk)), rr2 = qrot(q2, xyz(PBk));
                V3<S> dsep = delta_translation + (rr2 - rr1);
                sepv[k] = dot(dsep, n) + PAk.w;
            }
        }
#ifdef AVN_WAVE_TRACE
        { S sink = sepv[0]; if (sink == S(1.2345e33)) d.any_restitution[1] = 2; AVN_TRACE_ADD(d, 1, clock64() - t_p0); }
#endif
    }

    // ---- stage 2: velocity records of the two bodies and the impulse records of the points, all self-validating
    Rec32 R1, R2;
    R1.a = mk4<S>(0, 0, 0, 0); R1.b = R1.a; R2 = R1;
    {
        bool n1 = ver1, n2 = ver2;
        unsigned pend = np != 0 ? ((1u << np) - 1u) : 0u;
        if (np != 0 && !ver1) { R1.a = ld4(&d.vel[2 * b1]); R1.b = ld4(&d.vel[2 * b1 + 1]); }
        if (np != 0 && !ver2) { R2.a = ld4(&d.vel[2 * b2]); R2.b = ld4(&d.vel[2 * b2 + 1]); }
        AVN_TRACE_T(t_w1);
        for (unsigned spins = 0;; ++spins) {
            if (n1) R1 = ld_vel(&d.vel[2 * b1]);
            if (n2) R2 = ld_vel(&d.vel[2 * b2]);
#pragma unroll 1
            for (int k = 0; k < np; ++k) {
                if (pend & (1u << k)) {
                    const Rec32 p = ld_pc(pc_ptr(d, k, slot));
                    ROW_PC(k) = pc_val(p);
                    if (pc_is(p, ptag)) pend &= ~(1u << k);
                }
            }
            if (n1) n1 = !vel_is(R1, e1);
            if (n2) n2 = !vel_is(R2, e2);
            if (__all_sync(0xffffffffu, !(n1 || n2 || pend != 0u))) break;
            if (spins > W32_SPIN_LIMIT) { d.any_restitution[1] = WAVE_WATCHDOG; break; }
            if (d.poll_ns) __nanosleep(unsigned(d.poll_ns));   // (experiment: back off between polls, AVN_WAVE_POLL_NS)
        }
#ifdef AVN_WAVE_TRACE
        AVN_TRACE_ADD(d, 0, clock64() - t_w1);
#endif
    }
    if (!SOLVE) __pipeline_wait_prior(0);
    if (np == 0) return;   // padding slot / inactive lane (after the warp-collective polls)
    AVN_TRACE_T(t_c0);
    V3<S> v1 = xyz(R1.a), w1 = xyz(R1.b), v2 = xyz(R2.a), w2 = xyz(R2.b);
    const V3<S> t2 = cross(t1, n);  // tangent_directions(): [tangent1, tangent1 x normal] (contact/mod.rs:411-421)

    if (PASS == PASS_WARM) {
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
        const Soft<S> soft = (info & CI_NONDYN) ? d.soft_nondyn : d.soft_dyn;
#pragma unroll 1
        for (int k = 0; k < np; ++k) {
            {
                const Vec4<S> PAk = ROW_A(k), PBk = ROW_B(k);
                Vec4<S> pck = ROW_PC(k);
                V3<S> r1 = xyz(PAk), r2 = xyz(PBk);
                const S separation = sepv[k];
                V3<S> relv = (v2 + cross(w2, r2)) - (v1 + cross(w1, r1));
                // ContactNormalPart::solve_impulse (normal_part.rs:116-166)
                S vn = dot(relv, n);
                S meff = PBk.w, acc = pck.x;
                S impulse;
                if (separation > S(0)) {
                    impulse = -meff * (vn + separation / d.h);
                } else if (!relax) {
                    S bias = avn_max(soft.bias * separation, -d.max_overlap_speed);
                    S scaled_mass = soft.mass_scale * meff;
                    S scaled_impulse = soft.impulse_scale * acc;
                    impulse = -scaled_mass * (vn + bias) - scaled_impulse;
                } else {
                    impulse = -meff * vn;
                }
                S new_impulse = avn_max(acc + impulse, S(0));
                impulse = new_impulse - acc;
                pck.x = new_impulse;
                pck.y = pck.y + new_impulse;
                ROW_PC(k) = pck;
                apply_impulse(v1, w1, v2, w2, in1, in2, r1, r2, impulse * n);
            }
        }
        if (info & CI_TANGENT) {
            const S friction = hn.w;
            const V3<S> surf = xyz(htv);
#pragma unroll 1
            for (int k = 0; k < np; ++k) {
                {
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
                        ROW_PC(k) = pck;
                        imp = dx * t1 + dy * t2;
                    }
                    apply_impulse(v1, w1, v2, w2, in1, in2, r1, r2, imp);
                }
            }
        }
    }
    // ---- publish: every record this item is the next writer of, with the next tag.  A side without inertia here (dominated, kinematic)
    //      keeps the value it had bit for bit — only its event number moves on.
#ifdef AVN_WAVE_TRACE
    if ((v1.x + v2.x + w1.x + w2.x) == S(1.2345e33)) d.any_restitution[1] = 2;
    AVN_TRACE_T(t_s0);
    AVN_TRACE_ADD(d, 2, t_s0 - t_c0);
#endif
    if (PASS != PASS_WARM) {
#pragma unroll 1
        for (int k = 0; k < np; ++k) st_pc(pc_ptr(d, k, slot), ROW_PC(k), ptag + 1u);
    }
    if (ver1) {
        if (info & CI_ZERO1) st_vel(&d.vel[2 * b1], xyz(R1.a), xyz(R1.b), e1 + 1u);
        else st_vel(&d.vel[2 * b1], v1, w1, e1 + 1u);
    }
    if (ver2) {
        if (info & CI_ZERO2) st_vel(&d.vel[2 * b2], xyz(R2.a), xyz(R2.b), e2 + 1u);
        else st_vel(&d.vel[2 * b2], v2, w2, e2 + 1u);
    }
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
// The same routine with the loops over the points UNROLLED and the impulses / separations in registers (round 2's first version): 42 KB of
// SASS per pass instead of 17 KB, but no shared-memory round trip inside the dependent chain of an item.  The rolled routine wins when the
// step is throughput-bound (100k cubes: the warps of an SM are in five routines at once and the instruction cache
// holds the rolled ones), the unrolled one when it is bound by the per-body chain (10k cubes).  The host picks
// per step (DevSolver::wave_rolled).
// ---------------------------------------------------------------------------------------------------------
template <int PASS, int MAXP>
__device__ __forceinline__ void w32_contact_item_unrolled(const DevSolver<float>& d, int slot, int s, int it, bool lane_active, int wf) {
    using S = float;
    const size_t MP = size_t(d.Mpad);
    const Vec4<S>* c = d.cst + (lane_active ? slot : 0);
    const Vec4<S> hidx = ld4(&c[CP_IDX * MP]);
    const int info = lane_active ? as_int(hidx.z) : 0;   // an inactive lane of a partial chunk behaves like a padding slot
    const int np = info & CI_NP_MASK;
    const int b1 = as_int(hidx.x), b2 = as_int(hidx.y);
    constexpr bool SOLVE = (PASS == PASS_SOLVE_BIAS || PASS == PASS_RELAX);
    Vec4<S>* const stage = stage_base<S>() + threadIdx.x;
    const int T = blockDim.x;
#define ROW_A(k) stage[(3 * (k) + 0) * T]
#define ROW_B(k) stage[(3 * (k) + 1) * T]
#define ROW_D(k) stage[(3 * (k) + 2) * T]
    // ---- immutable part: issued before any wait
    Vec4<S> hn = mk4<S>(0, 0, 0, 0), ht1 = hn, htv = hn;
    BodyInertia<S> in1 = zero_inertia<S>(), in2 = zero_inertia<S>();
    if (np != 0) {
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
                if (SOLVE && (info & CI_TANGENT)) stage_copy(&ROW_D(k), &c[size_t(CP_ROW(k, 2)) * MP]);
            }
        }
    }
    __pipeline_commit();
    const bool ver1 = np != 0 && (info & CI_VER1), ver2 = np != 0 && (info & CI_VER2);
    const int rk = as_int(hidx.w);
    constexpr int kind = PASS == PASS_WARM ? WV_WARM : (PASS == PASS_SOLVE_BIAS ? WV_SOLVE : WV_RELAX);
    const unsigned e1 = wave_event(kind, it, s, d.iters, (rk >> 8) & 0xff, rk & 0xff, wf);
    const unsigned e2 = wave_event(kind, it, s, d.iters, (rk >> 24) & 0xff, (rk >> 16) & 0xff, wf);
    const unsigned ptag = w32_pc_tag(PASS, s, it, d.iters);
    const V3<S> n = xyz(hn), t1 = xyz(ht1);
    AVN_TRACE_T(t_w0);

    // ---- stage 1 (solve passes): the delta records -> separation of every point, before the velocities are even looked at
    S sep[MAXP];
#pragma unroll
    for (int k = 0; k < MAXP; ++k) sep[k] = S(0);
    if (SOLVE) {
        const unsigned dtag = unsigned(PASS == PASS_RELAX ? s + 1 : s);
        Rec32 D1, D2;
        D1.a = mk4<S>(0, 0, 0, 0); D1.b = mk4<S>(0, 0, 0, 1); D2 = D1;
        bool n1 = ver1, n2 = ver2;
        if (np != 0 && !ver1) { D1.a = ld4(&d.dlt[2 * b1]); D1.b = ld4(&d.dlt[2 * b1 + 1]); }   // no SolverBody: constant (0, identity)
        if (np != 0 && !ver2) { D2.a = ld4(&d.dlt[2 * b2]); D2.b = ld4(&d.dlt[2 * b2 + 1]); }
        for (unsigned spins = 0;; ++spins) {
            if (n1) D1 = ld_dlt(&d.dlt[2 * b1]);
            if (n2) D2 = ld_dlt(&d.dlt[2 * b2]);
            if (n1) n1 = tag_of(D1.a.w) != dtag;
            if (n2) n2 = tag_of(D2.a.w) != dtag;
            if (__all_sync(0xffffffffu, !(n1 || n2))) break;
            if (spins > W32_SPIN_LIMIT) { d.any_restitution[1] = WAVE_WATCHDOG; break; }
            if (d.poll_ns) __nanosleep(unsigned(d.poll_ns));   // (experiment: back off between polls, AVN_WAVE_POLL_NS)
        }
        __pipeline_wait_prior(0);   // this thread's staged rows have landed (only the issuing thread reads them)
        AVN_TRACE_T(t_p0);
        AVN_TRACE_ADD(d, 5, t_p0 - t_w0);
        if (np != 0) {
            Q4<S> q1; q1.x = D1.b.x; q1.y = D1.b.y; q1.z = D1.b.z; q1.w = D1.b.w;
            Q4<S> q2; q2.x = D2.b.x; q2.y = D2.b.y; q2.z = D2.b.z; q2.w = D2.b.w;
            const V3<S> delta_translation = xyz(D2.a) - xyz(D1.a);
#pragma unroll
            for (int k = 0; k < MAXP; ++k) {
                if (k < np) {
                    const Vec4<S> PAk = ROW_A(k), PBk = ROW_B(k);
                    V3<S> rr1 = qrot(q1, xyz(PAk)), rr2 = qrot(q2, xyz(PBk));
                    V3<S> dsep = delta_translation + (rr2 - rr1);
                    sep[k] = dot(dsep, n) + PAk.w;
                }
            }
        }
#ifdef AVN_WAVE_TRACE
        { S sink = sep[0]; if (sink == S(1.2345e33)) d.any_restitution[1] = 2; AVN_TRACE_ADD(d, 1, clock64() - t_p0); }
#endif
    }

    // ---- stage 2: velocity records of the two bodies and the impulse records of the points, all self-validating
    Rec32 R1, R2;
    R1.a = mk4<S>(0, 0, 0, 0); R1.b = R1.a; R2 = R1;
    Vec4<S> PC[MAXP];
#pragma unroll
    for (int k = 0; k < MAXP; ++k) PC[k] = mk4<S>(0, 0, 0, 0);
    {
        bool n1 = ver1, n2 = ver2;
        unsigned pend = np != 0 ? ((1u << np) - 1u) : 0u;
        if (np != 0 && !ver1) { R1.a = ld4(&d.vel[2 * b1]); R1.b = ld4(&d.vel[2 * b1 + 1]); }
        if (np != 0 && !ver2) { R2.a = ld4(&d.vel[2 * b2]); R2.b = ld4(&d.vel[2 * b2 + 1]); }
        AVN_TRACE_T(t_w1);
        for (unsigned spins = 0;; ++spins) {
            if (n1) R1 = ld_vel(&d.vel[2 * b1]);
            if (n2) R2 = ld_vel(&d.vel[2 * b2]);
#pragma unroll
            for (int k = 0; k < MAXP; ++k) {
                if (pend & (1u << k)) {
                    const Rec32 p = ld_pc(pc_ptr(d, k, slot));
                    PC[k] = pc_val(p);
                    if (pc_is(p, ptag)) pend &= ~(1u << k);
                }
            }
            if (n1) n1 = !vel_is(R1, e1);
            if (n2) n2 = !vel_is(R2, e2);
            if (__all_sync(0xffffffffu, !(n1 || n2 || pend != 0u))) break;
            if (spins > W32_SPIN_LIMIT) { d.any_restitution[1] = WAVE_WATCHDOG; break; }
            if (d.poll_ns) __nanosleep(unsigned(d.poll_ns));   // (experiment: back off between polls, AVN_WAVE_POLL_NS)
        }
#ifdef AVN_WAVE_TRACE
        AVN_TRACE_ADD(d, 0, clock64() - t_w1);
#endif
    }
    if (!SOLVE) __pipeline_wait_prior(0);
    if (np == 0) return;   // padding slot / inactive lane (after the warp-collective polls)
    AVN_TRACE_T(t_c0);
    V3<S> v1 = xyz(R1.a), w1 = xyz(R1.b), v2 = xyz(R2.a), w2 = xyz(R2.b);
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
    } else {
        // ContactConstraint::solve (contact/mod.rs:267-354)
        const Soft<S> soft = (info & CI_NONDYN) ? d.soft_nondyn : d.soft_dyn;
#pragma unroll
        for (int k = 0; k < MAXP; ++k) {
            if (k < np) {
                const Vec4<S> PAk = ROW_A(k), PBk = ROW_B(k);
                V3<S> r1 = xyz(PAk), r2 = xyz(PBk);
                const S separation = sep[k];
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
    }
    // ---- publish: every record this item is the next writer of, with the next tag.  A side without inertia here (dominated, kinematic)
    //      keeps the value it had bit for bit — only its event number moves on.
#ifdef AVN_WAVE_TRACE
    if ((v1.x + v2.x + w1.x + w2.x) == S(1.2345e33)) d.any_restitution[1] = 2;
    AVN_TRACE_T(t_s0);
    AVN_TRACE_ADD(d, 2, t_s0 - t_c0);
#endif
    if (PASS != PASS_WARM) {
#pragma unroll
        for (int k = 0; k < MAXP; ++k)
            if (k < np) st_pc(pc_ptr(d, k, slot), PC[k], ptag + 1u);
    }
    if (ver1) {
        if (info & CI_ZERO1) st_vel(&d.vel[2 * b1], xyz(R1.a), xyz(R1.b), e1 + 1u);
        else st_vel(&d.vel[2 * b1], v1, w1, e1 + 1u);
    }
    if (ver2) {
        if (info & CI_ZERO2) st_vel(&d.vel[2 * b2], xyz(R2.a), xyz(R2.b), e2 + 1u);
        else st_vel(&d.vel[2 * b2], v2, w2, e2 + 1u);
    }
#ifdef AVN_WAVE_TRACE
    AVN_TRACE_ADD(d, 3, clock64() - t_s0);
    AVN_TRACE_ADD(d, 4, 1);
#endif
#undef ROW_A
#undef ROW_B
#undef ROW_D
}

// the arithmetic of integrate_velocities + clamp_velocities on one body (shared by the two wavefront items that run it)
__device__ __forceinline__ void w32_integrate_velocity_math(const DevSolver<float>& d, int i, int f, const Rec32& D, V3<float>& v, V3<float>& w) {
    using S = float;
    if (!(f & BF_CUSTOM_VEL) && !(f & BF_KINEMATIC)) {
        Vec4<S> li = ld4(&d.itg[2 * i]), ai = ld4(&d.itg[2 * i + 1]);
        v = v * li.w;
        w = w * ai.w;
        v = v + xyz(li);
        w = w + xyz(ai);
        if (f & BF_GYRO) {
            // solve_gyroscopic_torque (integrator/mod.rs:403-460)
            Q4<S> dq; dq.x = D.b.x; dq.y = D.b.y; dq.z = D.b.z; dq.w = D.b.w;
            Q4<S> rot = qmul(dq, ldq(d.rotation, i));
            Sym3<S> il;
            il.m00 = d.inv_inertia_local[6 * i]; il.m01 = d.inv_inertia_local[6 * i + 1]; il.m02 = d.inv_inertia_local[6 * i + 2];
            il.m11 = d.inv_inertia_local[6 * i + 3]; il.m12 = d.inv_inertia_local[6 * i + 4]; il.m22 = d.inv_inertia_local[6 * i + 5];
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
    }
    if (d.max_lin) {
        S ms = d.max_lin[i];
        S l2 = len2(v);
        if (avn_finite(ms) && l2 > ms * ms) v = v * (ms / avn_sqrt(l2));
    }
    if (d.max_ang) {
        S ms = d.max_ang[i];
        S l2 = len2(w);
        if (avn_finite(ms) && l2 > ms * ms) w = w * (ms / avn_sqrt(l2));
    }
    if (d.bnd_of) {  // partitioned step: the reference point of this substep's constraint impulses on a boundary body
        const int k = d.bnd_of[i];
        if (k >= 0) {
            st4(&d.vel_ref[2 * k], mk4<S>(v.x, v.y, v.z, S(0)));
            st4(&d.vel_ref[2 * k + 1], mk4<S>(w.x, w.y, w.z, S(0)));
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// integrate_velocities + clamp_velocities (integrator/mod.rs:343-391, 467-500), wavefront mode
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void w32_integrate_velocity_item(const DevSolver<float>& d, int i, int s, bool lane_active) {
    using S = float;
    const bool in_range = lane_active && i < d.B;
    int f = 0;
    if (in_range) f = as_int(ld4(&d.inr[2 * i]).y);
    const bool live = in_range && (f & BF_HAS_SOLVER_BODY);
    const unsigned e = live ? wave_event(WV_IV, 0, s, d.iters, d.deg[i], 0) : 0u;
    const bool gyro = live && (f & BF_GYRO) && !(f & BF_CUSTOM_VEL) && !(f & BF_KINEMATIC);
    Rec32 R, D;
    R.a = mk4<S>(0, 0, 0, 0); R.b = R.a; D = R;
    {
        bool nr = live, nd = gyro;
        for (unsigned spins = 0;; ++spins) {
            if (nr) R = ld_vel(&d.vel[2 * i]);
            if (nd) D = ld_dlt(&d.dlt[2 * i]);
            if (nr) nr = !vel_is(R, e);
            if (nd) nd = tag_of(D.a.w) != unsigned(s);
            if (__all_sync(0xffffffffu, !(nr || nd))) break;
            if (spins > W32_SPIN_LIMIT) { d.any_restitution[1] = WAVE_WATCHDOG; break; }
            if (d.poll_ns) __nanosleep(unsigned(d.poll_ns));   // (experiment: back off between polls, AVN_WAVE_POLL_NS)
        }
    }
    if (!live) return;
    V3<S> v = xyz(R.a), w = xyz(R.b);
    w32_integrate_velocity_math(d, i, f, D, v, w);
    st_vel(&d.vel[2 * i], v, w, e + 1u);
}

// ---------------------------------------------------------------------------------------------------------
// BODY-CENTRIC warm start, fused with integrate_velocities: ONE event per body and substep instead of 1 + k.
//
// ContactConstraint::warm_start (contact/mod.rs:223-264) changes a body's velocity by a vector that does not depend on any velocity:
//     v -= P * inv_mass,  w -= I (r x P),   P = coeff * ((ln * n + lt.x * t1) + lt.y * t2)        (body 2: +)
// so the k warm-start items of a body are not a true dependency chain — only the ORDER of the k * np subtractions is part of the result
// (floating-point addition does not associate).  Four lanes per body (8 bodies per warp) compute the per-point deltas of the body's
// constraints as soon as the impulse records of the previous substep's relax pass are there (all of it before the body's own velocity
// record is final), park them in the warp's slice of the staging tile, and the body's first lane then runs integrate_velocities and adds
// the deltas in colour order, point order: 6 dependent additions per point are all that is left on the critical path.  x - a == x + (-a)
// bit for bit, so the deltas are stored with their sign.  26 -> 18 dependency levels per substep at k = 8.
// Tile slice of a warp: rows x 128 floats; delta c of point q of body g at float (q * 6 + c) * 8 + g (the 8 leader lanes read 8
// consecutive floats).  Points beyond the slice (8 * MAXP per body) are computed by the leader on the spot.
// ---------------------------------------------------------------------------------------------------------
struct W32WarmDelta { V3<float> a, bw; };
__device__ __forceinline__ W32WarmDelta w32_warm_delta(const DevSolver<float>& d, const BodyInertia<float>& in, V3<float> n, V3<float> t1, V3<float> t2,
                                                       V3<float> r, Vec4<float> pc, bool tangent, bool side2) {
    using S = float;
    const S tx = tangent ? pc.z : S(0), ty = tangent ? pc.w : S(0);
    const V3<S> p = d.warm_coeff * ((pc.x * n + tx * t1) + ty * t2);
    W32WarmDelta o;
    o.a = cmul(p, in.inv_mass);
    o.bw = smul(in.ii, cross(r, p));
    if (!side2) { o.a = -o.a; o.bw = -o.bw; }
    return o;
}
template <int MAXP>
__device__ __forceinline__ float* w32_delta_slot(int q, int c, int g) {
    const int idx = (q * 6 + c) * 8 + g;
    float* base = reinterpret_cast<float*>(stage_base<float>());
    return base + size_t(idx >> 7) * (size_t(blockDim.x) * 4) + (threadIdx.x >> 5) * 128 + (idx & 127);
}

template <int MAXP>
__device__ __forceinline__ void w32_ivw_item(const DevSolver<float>& d, int chunk, int s) {
    using S = float;
    constexpr int CAPQ = 8 * MAXP;     // points per body that fit the warp's slice of the tile: 3 * MAXP rows * 128 floats / (6 * 8)
    const int lane = threadIdx.x & 31, g = lane >> 2, l = lane & 3;
    const int i = chunk * 8 + g;
    const size_t MP = size_t(d.Mpad);
    const bool in_range = i < d.B;
    int f = 0;
    if (in_range) f = as_int(ld4(&d.inr[2 * i]).y);
    const bool live = in_range && (f & BF_HAS_SOLVER_BODY);
    const int nw = live ? d.wdeg[i] : 0;
    const int npts = live ? d.wpts[i] : 0;
    BodyInertia<S> in = zero_inertia<S>();
    if (nw > 0) in = unpack_inertia(ld4(&d.inr[2 * i]), ld4(&d.inr[2 * i + 1]));
    const unsigned ptag = w32_pc_tag(PASS_WARM, s, 0, d.iters);
    __syncwarp();   // the previous item's reads of its staged rows are done in every lane before the slice is overwritten
    // ---- phase A: the deltas of entries l, l + 4, ... of body g (no dependence on the body's velocity)
    for (int j = l;; j += 4) {
        const bool has = j < nw;
        if (!__any_sync(0xffffffffu, has)) break;
        uint2 ent = make_uint2(0u, 0u);
        if (has) ent = d.adj[size_t(j) * d.adj_stride + i];
        const int np = int(ent.y & WA_NP_MASK), q0 = int(ent.y >> WA_Q0_SHIFT), slot = int(ent.x);
        const bool tangent = (ent.y & WA_TANGENT) != 0, side2 = (ent.y & WA_SIDE2) != 0;
        const Vec4<S>* c = d.cst + slot;
        Vec4<S> hn = mk4<S>(0, 0, 0, 0), ht1 = hn, row[MAXP], PC[MAXP];
#pragma unroll
        for (int k = 0; k < MAXP; ++k) { row[k] = hn; PC[k] = hn; }
        if (np != 0) {
            hn = ld4(&c[CP_N * MP]);
            ht1 = ld4(&c[CP_T1 * MP]);
#pragma unroll
            for (int k = 0; k < MAXP; ++k)
                if (k < np) row[k] = ld4(&c[size_t(CP_ROW(k, side2 ? 1 : 0)) * MP]);
        }
        unsigned pend = np != 0 ? ((1u << np) - 1u) : 0u;
        for (unsigned spins = 0;; ++spins) {
#pragma unroll
            for (int k = 0; k < MAXP; ++k) {
                if (pend & (1u << k)) {
                    const Rec32 p = ld_pc(pc_ptr(d, k, slot));
                    PC[k] = pc_val(p);
                    if (pc_is(p, ptag)) pend &= ~(1u << k);
                }
            }
            if (__all_sync(0xffffffffu, pend == 0u)) break;
            if (spins > W32_SPIN_LIMIT) { d.any_restitution[1] = WAVE_WATCHDOG; break; }
            if (d.poll_ns) __nanosleep(unsigned(d.poll_ns));   // (experiment: back off between polls, AVN_WAVE_POLL_NS)
        }
        const V3<S> n = xyz(hn), t1 = xyz(ht1), t2 = cross(t1, n);
#pragma unroll
        for (int k = 0; k < MAXP; ++k) {
            if (k < np && q0 + k < CAPQ) {
                const W32WarmDelta o = w32_warm_delta(d, in, n, t1, t2, xyz(row[k]), PC[k], tangent, side2);
                *w32_delta_slot<MAXP>(q0 + k, 0, g) = o.a.x;  *w32_delta_slot<MAXP>(q0 + k, 1, g) = o.a.y;  *w32_delta_slot<MAXP>(q0 + k, 2, g) = o.a.z;
                *w32_delta_slot<MAXP>(q0 + k, 3, g) = o.bw.x; *w32_delta_slot<MAXP>(q0 + k, 4, g) = o.bw.y; *w32_delta_slot<MAXP>(q0 + k, 5, g) = o.bw.z;
            }
        }
    }
    __syncwarp();
    // ---- phase B: the leader lane of every body: integrate_velocities, then the deltas in order
    const bool lead = live && l == 0;
    const unsigned e = lead ? wave_event(WV_IV, 0, s, d.iters, d.deg[i], 0, 0) : 0u;
    const bool gyro = lead && (f & BF_GYRO) && !(f & BF_CUSTOM_VEL) && !(f & BF_KINEMATIC);
    Rec32 R, D;
    R.a = mk4<S>(0, 0, 0, 0); R.b = R.a; D = R;
    {
        bool nr = lead, nd = gyro;
        for (unsigned spins = 0;; ++spins) {
            if (nr) R = ld_vel(&d.vel[2 * i]);
            if (nd) D = ld_dlt(&d.dlt[2 * i]);
            if (nr) nr = !vel_is(R, e);
            if (nd) nd = tag_of(D.a.w) != unsigned(s);
            if (__all_sync(0xffffffffu, !(nr || nd))) break;
            if (spins > W32_SPIN_LIMIT) { d.any_restitution[1] = WAVE_WATCHDOG; break; }
            if (d.poll_ns) __nanosleep(unsigned(d.poll_ns));   // (experiment: back off between polls, AVN_WAVE_POLL_NS)
        }
    }
    if (lead) {
        V3<S> v = xyz(R.a), w = xyz(R.b);
        w32_integrate_velocity_math(d, i, f, D, v, w);
        const int nq = npts < CAPQ ? npts : CAPQ;
        for (int q = 0; q < nq; ++q) {
            v.x = v.x + *w32_delta_slot<MAXP>(q, 0, g); v.y = v.y + *w32_delta_slot<MAXP>(q, 1, g); v.z = v.z + *w32_delta_slot<MAXP>(q, 2, g);
            w.x = w.x + *w32_delta_slot<MAXP>(q, 3, g); w.y = w.y + *w32_delta_slot<MAXP>(q, 4, g); w.z = w.z + *w32_delta_slot<MAXP>(q, 5, g);
        }
        if (npts > CAPQ) {   // more points than the slice holds: the rest on the spot (the body's velocity record is final, so the
                             // impulse records of its constraints are written; they are still validated, lane by lane)
            for (int j = 0; j < nw; ++j) {
                const uint2 ent = d.adj[size_t(j) * d.adj_stride + i];
                const int np = int(ent.y & WA_NP_MASK), q0 = int(ent.y >> WA_Q0_SHIFT), slot = int(ent.x);
                if (q0 + np <= CAPQ) continue;
                const bool tangent = (ent.y & WA_TANGENT) != 0, side2 = (ent.y & WA_SIDE2) != 0;
                const Vec4<S>* c = d.cst + slot;
                const V3<S> n = xyz(ld4(&c[CP_N * MP])), t1 = xyz(ld4(&c[CP_T1 * MP])), t2 = cross(t1, n);
                for (int k = 0; k < np; ++k) {
                    if (q0 + k < CAPQ) continue;
                    const V3<S> r = xyz(ld4(&c[size_t(CP_ROW(k, side2 ? 1 : 0)) * MP]));
                    Rec32 p = ld_pc(pc_ptr(d, k, slot));
                    for (unsigned spins = 0; !pc_is(p, ptag); ++spins) {
                        if (spins > W32_SPIN_LIMIT) { d.any_restitution[1] = WAVE_WATCHDOG; break; }
            if (d.poll_ns) __nanosleep(unsigned(d.poll_ns));   // (experiment: back off between polls, AVN_WAVE_POLL_NS)
                        p = ld_pc(pc_ptr(d, k, slot));
                    }
                    const W32WarmDelta o = w32_warm_delta(d, in, n, t1, t2, r, pc_val(p), tangent, side2);
                    v = v + o.a;
                    w = w + o.bw;
                }
            }
        }
        st_vel(&d.vel[2 * i], v, w, e + 1u);
    }
    __syncwarp();   // the slice is free again (the next item stages its rows into it)
}

// integrate_positions (integrator/mod.rs:503-535), wavefront mode
__device__ __forceinline__ void w32_integrate_position_item(const DevSolver<float>& d, int i, int s, bool lane_active, int wf) {
    using S = float;
    const bool in_range = lane_active && i < d.B;
    int f = 0;
    if (in_range) f = as_int(ld4(&d.inr[2 * i]).y);
    const bool live = in_range && (f & BF_HAS_SOLVER_BODY);
    const unsigned e = live ? wave_event(WV_IP, 0, s, d.iters, d.deg[i], 0, wf) : 0u;
    Rec32 R, D;
    R.a = mk4<S>(0, 0, 0, 0); R.b = R.a; D = R;
    {
        bool nr = live, nd = live;
        for (unsigned spins = 0;; ++spins) {
            if (nr) R = ld_vel(&d.vel[2 * i]);
            if (nd) D = ld_dlt(&d.dlt[2 * i]);
            if (nr) nr = !vel_is(R, e);
            if (nd) nd = tag_of(D.a.w) != unsigned(s);
            if (__all_sync(0xffffffffu, !(nr || nd))) break;
            if (spins > W32_SPIN_LIMIT) { d.any_restitution[1] = WAVE_WATCHDOG; break; }
            if (d.poll_ns) __nanosleep(unsigned(d.poll_ns));   // (experiment: back off between polls, AVN_WAVE_POLL_NS)
        }
    }
    if (!live) return;
    const unsigned nt = unsigned(s) + 1u;
    if (f & BF_CUSTOM_POS) {
        st_dlt(&d.dlt[2 * i], xyz(D.a), nt, D.b);
    } else {
        V3<S> ndp = xyz(D.a) + xyz(R.a) * d.h;
        Q4<S> dq; dq.x = D.b.x; dq.y = D.b.y; dq.z = D.b.z; dq.w = D.b.w;
        Q4<S> nq = qmul(q_from_scaled_axis(xyz(R.b) * d.h, d.fast_trig != 0), dq);
        st_dlt(&d.dlt[2 * i], ndp, nt, mk4<float>(nq.x, nq.y, nq.z, nq.w));
    }
    st_vel(&d.vel[2 * i], xyz(R.a), xyz(R.b), e + 1u);
}

}  // namespace avn
