// Host driver of the solver stage: column upload, level schedule for joints, kernel launch, result download.
// Reference systems replaced: see avn_solver_step in include/avian_b200.h.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "context.hpp"
#include "joint_schedule.hpp"
#include "solver_kernels.cuh"

namespace avn {

namespace {

// SoftnessParameters::new + compute_coefficients (softness_parameters/mod.rs:22-79), evaluated in S like the reference
template <class S>
Soft<S> softness(S damping_ratio, S hz, S delta_secs) {
    S double_damping_ratio = S(2) * damping_ratio;
    S angular_frequency = S(6.283185307179586476925286766559) * hz;
    S a1 = double_damping_ratio + angular_frequency * delta_secs;
    S a2 = angular_frequency * delta_secs * a1;
    S a3 = S(1) / (S(1) + a2);
    Soft<S> s;
    s.bias = angular_frequency / a1;
    s.mass_scale = a2 * a3;
    s.impulse_scale = a3;
    return s;
}

template <class S>
class Solver final : public SolverBase {
   public:
    Solver(cudaStream_t stream, ErrorSink* err, uint32_t cfg_flags, int device) : stream_(stream), err_(err), cfg_flags_(cfg_flags) {
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) {
            sm_count_ = prop.multiProcessorCount;
            coop_ok_ = prop.cooperativeLaunch != 0;
        }
        {
            // L2 persistence for the hot range (AVN_L2_PERSIST=0 disables it)
            const char* lp = getenv("AVN_L2_PERSIST");
            l2_persist_ = !(lp && !strcmp(lp, "0")) && prop.persistingL2CacheMaxSize > 0;
            if (l2_persist_) {
                l2_persist_bytes_ = std::min<size_t>(size_t(prop.persistingL2CacheMaxSize), size_t(64) << 20);
                l2_window_max_ = size_t(prop.accessPolicyMaxWindowSize);
                if (cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, l2_persist_bytes_) != cudaSuccess) { (void)cudaGetLastError(); l2_persist_ = false; }
            }
        }
        const char* mode = getenv("AVN_LAUNCH_MODE");
        if (mode && !strcmp(mode, "phases")) use_mega_ = false;
        if (mode && !strcmp(mode, "barrier")) use_wave_ = false;   // megakernel with grid barriers between colours
        // register budget of the persistent kernel: 65536 / (128 threads * blocks per SM); more resident warps hide more
        // latency, fewer registers spill more.  Measured best (scripts/solver_timing.py): 3 blocks/SM for f32, 2 for f64 (whose
        // state is twice as wide).  AVN_MEGA_BPS = 2|3|4 overrides the default for experiments.
        const char* bps = getenv("AVN_MEGA_BPS");
        mega_bps_ = bps ? atoi(bps) : (sizeof(S) == 8 ? 2 : 3);
        if (mega_bps_ < 2 || mega_bps_ > 4) mega_bps_ = 3;
        if (mode && !strcmp(mode, "wave")) force_wave_ = true;
        coop_ok_ = coop_ok_ && select_megakernel(AVN_MAX_MANIFOLD_POINTS);
        for (auto& e : ev_) cudaEventCreate(&e);
        up_stream_ = stream_;
        if (cudaStreamCreateWithFlags(&copy_stream_, cudaStreamNonBlocking) != cudaSuccess) { (void)cudaGetLastError(); copy_stream_ = nullptr; }
        cudaEventCreateWithFlags(&ev_prefetch_, cudaEventDisableTiming);
    }
    ~Solver() override {
        for (auto& e : ev_) cudaEventDestroy(e);
        if (ev_prefetch_) cudaEventDestroy(ev_prefetch_);
        if (copy_stream_) { cudaStreamSynchronize(copy_stream_); cudaStreamDestroy(copy_stream_); }
        if (h_agree_) cudaFreeHost(h_agree_);
    }

    AvnStatus upload(const AvnStepParams* prm, AvnBodyColumns* bc, AvnManifoldColumns* mc, AvnJointSet* js) override;
    AvnStatus upload_resident(const AvnStepParams* prm, AvnBodyColumns* bc, ContactsBase* contacts, AvnJointSet* js) override;
    AvnStatus run_range(uint32_t first, uint32_t count, uint32_t flags) override;
    AvnStatus set_boundary(const AvnBoundary* bnd) override;
    AvnStatus boundary_snapshot() override;
    AvnStatus boundary_pack(void* device_table) override;
    AvnStatus boundary_apply(const void* device_gathered) override;
    AvnStatus step_partitioned(CommBase* comm) override;
    int needs_restitution() const override { return host_any_restitution_ ? 1 : 0; }
    AvnStatus prefetch_bodies(AvnBodyColumns* bc, uint32_t flags) override {
        if (!bc) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "bodies are required");
        if (bc->count && (!bc->position || !bc->rotation || !bc->linear_velocity || !bc->angular_velocity || !bc->inverse_mass || !bc->inverse_inertia_local))
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "bodies: position, rotation, velocities, inverse_mass and inverse_inertia_local are required");
        prefetched_ = false;
        if (!copy_stream_) return AVN_OK;    // no second stream: the next upload copies as usual
        // the device copies are inputs of the previous run: the copy waits for it (not for anything enqueued after it)
        if (ran_ || prepared_) AVN_CUDA(cudaStreamWaitEvent(copy_stream_, ev_[EV_RUN1], 0));
        DevSolver<S> tmp{};
        up_stream_ = copy_stream_;
        const AvnStatus st = upload_body_columns(*bc, (flags & AVN_BODIES_STATIC_UNCHANGED) != 0, tmp);
        up_stream_ = stream_;
        if (st != AVN_OK) return st;
        AVN_CUDA(cudaEventRecord(ev_prefetch_, copy_stream_));
        pref_host_ = *bc;
        prefetched_ = true;
        return AVN_OK;
    }
    AvnStatus run() override;
    AvnStatus download() override;
    void timings(AvnTimings* t) const override { *t = tm_; }
    void attach_ccd(CcdBase* ccd, ContactsBase* contacts) override { ccd_ = ccd; ccd_contacts_ = contacts; }

   private:
    static constexpr int kBlock = 256;
    enum { EV_H2D0, EV_H2D1, EV_RUN0, EV_PREP, EV_LOOP, EV_RUN1, EV_D2H0, EV_D2H1, EV_COUNT };

    // copy one host column to the device; returns nullptr for a NULL host column
    template <class T>
    AvnStatus up(DevBuf& buf, const void* host, size_t count, const T** dev) {
        *dev = nullptr;
        if (!host || count == 0) return AVN_OK;
        AVN_CUDA(buf.ensure(count * sizeof(T)));
        AVN_CUDA(cudaMemcpyAsync(buf.p, host, count * sizeof(T), cudaMemcpyHostToDevice, up_stream_));
        *dev = buf.as<T>();
        h2d_bytes_ += count * sizeof(T);
        return AVN_OK;
    }
    // ---- body columns: uploaded by upload_impl, or ahead of it by avn_solver_prefetch_bodies on the copy stream so that the copy overlaps the
    //      kernels of the stages that run before the solver (broad phase, contact pipeline)
    struct BodyCols {
        const uint8_t* kind = nullptr; const uint8_t* locked = nullptr; const int8_t* dominance = nullptr; const uint8_t* integ_flags = nullptr;
        const S* position = nullptr; const S* rotation = nullptr; const S* linvel = nullptr; const S* angvel = nullptr; const S* inv_mass = nullptr;
        const S* inv_inertia_local = nullptr; const S* com = nullptr; const S* lin_damp = nullptr; const S* ang_damp = nullptr; const S* grav_scale = nullptr;
        const S* lin_acc = nullptr; const S* ang_acc = nullptr; const S* max_lin = nullptr; const S* max_ang = nullptr;
        size_t count = 0;
    };
    BodyCols bcols_{};
    AvnBodyColumns pref_host_{};
    bool prefetched_ = false;
    cudaStream_t copy_stream_ = nullptr, up_stream_ = nullptr;
    cudaEvent_t ev_prefetch_ = nullptr;
    bool prefetch_matches(const AvnBodyColumns& bc) const {
        return bc.count == pref_host_.count && bc.position == pref_host_.position && bc.rotation == pref_host_.rotation &&
               bc.linear_velocity == pref_host_.linear_velocity && bc.angular_velocity == pref_host_.angular_velocity && bc.kind == pref_host_.kind &&
               bc.inverse_mass == pref_host_.inverse_mass && bc.inverse_inertia_local == pref_host_.inverse_inertia_local;
    }
    // keep_static: the columns that describe the body (kind, locked axes, dominance, integration markers, mass properties, damping, gravity
    // scale, speed limits) equal those of the previous upload of the same number of bodies and stay where they are
    AvnStatus upload_body_columns(const AvnBodyColumns& bc, bool keep_static, DevSolver<S>& d) {
        const size_t B = bc.count;
        AvnStatus st;
        keep_static = keep_static && bcols_.count == B && B > 0;
#define UPB(buf, host, n, T, field) if ((st = up<T>(buf, host, n, &d.field)) != AVN_OK) return st
#define UPS(buf, host, n, T, field) if (keep_static) d.field = (host) ? bcols_.field : nullptr; else UPB(buf, host, n, T, field)
        UPS(b_kind_, bc.kind, B, uint8_t, kind);
        UPS(b_locked_, bc.locked_axes, B, uint8_t, locked);
        UPS(b_dom_, bc.dominance, B, int8_t, dominance);
        UPS(b_iflags_, bc.integration_flags, B, uint8_t, integ_flags);
        UPB(b_pos_, bc.position, 3 * B, S, position);
        UPB(b_rot_, bc.rotation, 4 * B, S, rotation);
        UPB(b_lv_, bc.linear_velocity, 3 * B, S, linvel);
        UPB(b_av_, bc.angular_velocity, 3 * B, S, angvel);
        UPS(b_im_, bc.inverse_mass, B, S, inv_mass);
        UPS(b_iil_, bc.inverse_inertia_local, 6 * B, S, inv_inertia_local);
        UPS(b_com_, bc.center_of_mass, 3 * B, S, com);
        UPS(b_ld_, bc.linear_damping, B, S, lin_damp);
        UPS(b_ad_, bc.angular_damping, B, S, ang_damp);
        UPS(b_gs_, bc.gravity_scale, B, S, grav_scale);
        UPB(b_la_, bc.linear_acceleration, 3 * B, S, lin_acc);
        UPB(b_aa_, bc.angular_acceleration, 3 * B, S, ang_acc);
        UPS(b_ml_, bc.max_linear_speed, B, S, max_lin);
        UPS(b_ma_, bc.max_angular_speed, B, S, max_ang);
#undef UPS
#undef UPB
        bcols_.kind = d.kind; bcols_.locked = d.locked; bcols_.dominance = d.dominance; bcols_.integ_flags = d.integ_flags;
        bcols_.position = d.position; bcols_.rotation = d.rotation; bcols_.linvel = d.linvel; bcols_.angvel = d.angvel; bcols_.inv_mass = d.inv_mass;
        bcols_.inv_inertia_local = d.inv_inertia_local; bcols_.com = d.com; bcols_.lin_damp = d.lin_damp; bcols_.ang_damp = d.ang_damp;
        bcols_.grav_scale = d.grav_scale; bcols_.lin_acc = d.lin_acc; bcols_.ang_acc = d.ang_acc; bcols_.max_lin = d.max_lin; bcols_.max_ang = d.max_ang;
        bcols_.count = B;
        return AVN_OK;
    }
    AvnStatus build_joint_schedule(const AvnBodyColumns& bc, const AvnJointSet& js);
    AvnStatus launch_range(uint32_t first, uint32_t count, uint32_t flags);
    bool ccd_active() const { return ccd_ && ccd_->active(); }
    CcdBase* ccd_ = nullptr;
    ContactsBase* ccd_contacts_ = nullptr;
    bool from_store_ = false;     // the upload came from the contact store (upload_resident): swept CCD can run
    double length_unit_ = 1;
    template <int OP> void launch_phase(int begin, int count, bool serial = false) {
        if (count <= 0) return;
        int grid = serial ? 1 : std::min((count + kBlock - 1) / kBlock, sm_count_ * 8);
        const bool contact_op = OP == OP_WARM || OP == OP_SOLVE_BIAS || OP == OP_RELAX || OP == OP_RESTITUTION;
        const size_t smem = contact_op ? stage_bytes<S>(kBlock) : 0;   // staging tile of contact_item
        if (smem > 48 * 1024) cudaFuncSetAttribute(phase_kernel<S, OP>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
        phase_kernel<S, OP><<<grid, kBlock, smem, stream_>>>(dev_, begin, count, serial ? 1 : 0);
        ++launches_;
    }
    template <int OP> void launch_contact_pass() {
        const int* off = dev_.color_off;
        launch_phase<OP>(off[AVN_COLOR_OVERFLOW], dev_.color_len[AVN_COLOR_OVERFLOW], true);
        for (int c = 0; c < AVN_COLOR_OVERFLOW; ++c) launch_phase<OP>(off[c], dev_.color_len[c]);
    }

    cudaStream_t stream_;
    ErrorSink* err_;
    uint32_t cfg_flags_;
    int sm_count_ = 132;
    bool coop_ok_ = false, use_mega_ = true, use_wave_ = true, l2_persist_ = false;
    size_t l2_persist_bytes_ = 0, l2_window_max_ = 0;
    int mega_grid_ = 0, mega_bps_ = 3, mega_maxp_ = 0, mega_sel_bps_ = 0;
    bool force_wave_ = false;

    // The persistent kernel is compiled per (blocks/SM, widest manifold): MAXP = 1 (sphere-only scenes) drops the unrolled code and the
    // registers of points 2..4.  Returns false when the cooperative grid cannot be sized.
    template <int MAXP> const void* mega_variant(int bps) const {
        switch (bps) {
            case 2: return (const void*)step_megakernel<S, 2, MAXP>;
            case 4: return (const void*)step_megakernel<S, 4, MAXP>;
            default: return (const void*)step_megakernel<S, 3, MAXP>;
        }
    }
    // dynamic shared memory of the persistent kernel: the per-thread cp.async tile of the contact routines
    static size_t mega_smem_bytes(int maxp) { return stage_bytes<S>(MEGA_BLOCK, maxp); }
    bool select_megakernel(int max_points, int bps = 0) {
        const int maxp = max_points <= 1 ? 1 : AVN_MAX_MANIFOLD_POINTS;
        if (bps == 0) bps = mega_bps_;
        if (maxp == mega_maxp_ && bps == mega_sel_bps_) return mega_grid_ > 0;
        mega_maxp_ = maxp;
        mega_sel_bps_ = bps;
        mega_fn_ = maxp == 1 ? mega_variant<1>(bps) : mega_variant<AVN_MAX_MANIFOLD_POINTS>(bps);
        const size_t smem = mega_smem_bytes(maxp);
        int per_sm = 0;
        mega_grid_ = 0;
        if (cudaFuncSetAttribute(mega_fn_, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)) == cudaSuccess &&
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, mega_fn_, MEGA_BLOCK, smem) == cudaSuccess && per_sm > 0)
            mega_grid_ = per_sm * sm_count_;
        else
            (void)cudaGetLastError();
        if (getenv("AVN_DEBUG_GRID")) fprintf(stderr, "[avn] megakernel bps=%d maxp=%d: %d blocks/SM resident, grid %d, %zu B dynamic smem\n", bps, maxp, per_sm, mega_grid_, smem);
        return mega_grid_ > 0;
    }
    int max_np_ = AVN_MAX_MANIFOLD_POINTS;  // widest manifold of the current upload
    const void* mega_fn_ = nullptr;
    cudaEvent_t ev_[EV_COUNT];
    AvnTimings tm_{};
    uint32_t launches_ = 0, exchanges_ = 0;
    size_t h2d_bytes_ = 0;
    bool uploaded_ = false, ran_ = false, host_any_restitution_ = false, prepared_ = false, mega_step_ = false;
    DevBuf bnd_of_, bnd_body_, bnd_slot_, bnd_owner_, vel_ref_, bnd_table_, bnd_gathered_, bnd_agree_;
    int* h_agree_ = nullptr;
    int agreed_rest_ = 0;
    bool agreed_valid_ = false;   // the restitution agreement of step_partitioned holds until the next upload
    int bnd_n_ = 0, bnd_rank_ = 0, bnd_world_ = 1, step_bps_ = 0;
    size_t bnd_slots_ = 0;

    DevSolver<S> dev_{};
    // host pointers for download
    AvnBodyColumns hb_{};
    // where the manifolds of an upload come from: the CSR columns of AvnManifoldColumns (host), or the contact store (resident)
    struct ManifoldSource {
        size_t M = 0, P = 0;                               // manifolds, rows of the point columns
        const uint32_t* color_offsets = nullptr;
        const int32_t* body1 = nullptr; const int32_t* body2 = nullptr;
        const void* friction = nullptr; const void* restitution = nullptr; const void* tangent_velocity = nullptr; const void* normal = nullptr;
        const uint32_t* point_offsets = nullptr;           // CSR
        const uint32_t* edge = nullptr; const uint8_t* edge_point_count = nullptr;   // resident: ContactId of manifold m, points per row
        const void* anchor1 = nullptr; const void* anchor2 = nullptr; const void* penetration = nullptr; const void* normal_speed = nullptr;
        void* ws_normal = nullptr; void* ws_tangent = nullptr; void* normal_impulse = nullptr;
        // resident == true: every column above is a DEVICE pointer owned by the contact store (its rows, 4 point slots per row, and its
        // colour-major list), store_contact_impulses writes to out_* (device) instead of buffers of this solver; nothing of them is copied
        bool resident = false;
        bool list_restitution = false;
        void* out_ws_normal = nullptr; void* out_ws_tangent = nullptr; void* out_normal_impulse = nullptr;
    };
    AvnStatus upload_impl(const AvnStepParams* prm, AvnBodyColumns* bc, const ManifoldSource* src, AvnJointSet* js);
    ManifoldSource hm_{};
    DevBuf m_pbegin_, m_pend_;
    AvnJointSet hj_{};
    bool have_m_ = false, have_j_ = false;

    // device storage
    const uint8_t* body_asleep_ = nullptr;   // upload_resident: the contact store's applied sleeping state for the upload in progress
    DevBuf b_kind_eff_;
    DevBuf b_kind_, b_locked_, b_dom_, b_iflags_, b_pos_, b_rot_, b_lv_, b_av_, b_im_, b_iil_, b_com_, b_ld_, b_ad_, b_gs_, b_la_, b_aa_, b_ml_, b_ma_;
    DevBuf o_pos_, o_rot_, o_lv_, o_av_;
    DevBuf s_inr_, s_itg_, s_pre_;
    DevBuf m_b1_, m_b2_, m_n_, m_f_, m_r_, m_tv_, m_po_, p_a1_, p_a2_, p_pen_, p_ns_, p_wn_, p_wt_, p_ni_, p_nin_, p_own_, p_owt_;
    DevBuf hot_, c_flag_;
    size_t hot_bytes_ = 0;
    DevBuf j_type_, j_index_, j_level_, j_planes_, j_damp_slot_, j_damp_level_, j_dummy_;
    DevBuf jcol_[AVN_JOINT_TYPE_COUNT][12], jb1_[AVN_JOINT_TYPE_COUNT], jb2_[AVN_JOINT_TYPE_COUNT], jle_[AVN_JOINT_TYPE_COUNT],
        jde_[AVN_JOINT_TYPE_COUNT], jdl_[AVN_JOINT_TYPE_COUNT], jda_[AVN_JOINT_TYPE_COUNT], jfo_[AVN_JOINT_TYPE_COUNT], jto_[AVN_JOINT_TYPE_COUNT];
    std::vector<int> h_type_, h_index_, h_level_off_, h_damp_slot_, h_damp_level_off_;
};

template <class S>
AvnStatus Solver<S>::build_joint_schedule(const AvnBodyColumns& bc, const AvnJointSet& js) {
    JointSchedule sch;
    std::string error;
    AvnStatus st = avn::build_joint_schedule(bc, js, sch, error);
    if (st != AVN_OK) return err_->fail(st, "%s", error.c_str());
    h_type_.swap(sch.type);
    h_index_.swap(sch.index);
    h_level_off_.swap(sch.level_off);
    h_damp_slot_.swap(sch.damp_slot);
    h_damp_level_off_.swap(sch.damp_level_off);
    const size_t J = h_type_.size();
    dev_.J = int(J);
    dev_.Jpad = int((J + 31) & ~size_t(31));
    dev_.n_levels = sch.n_levels;
    dev_.n_damp_levels = sch.n_damp_levels;
    return AVN_OK;
}

template <class S>
AvnStatus Solver<S>::upload(const AvnStepParams* prm, AvnBodyColumns* bc, AvnManifoldColumns* mc, AvnJointSet* js) {
    if (!mc || mc->count == 0) return upload_impl(prm, bc, nullptr, js);
    if (!mc->body1 || !mc->body2 || !mc->normal || !mc->friction || !mc->restitution || !mc->point_offsets || !mc->anchor1 || !mc->anchor2 ||
        !mc->penetration || !mc->normal_speed || !mc->warm_start_normal_impulse || !mc->warm_start_tangent_impulse || !mc->normal_impulse)
        return err_->fail(AVN_ERR_INVALID_ARGUMENT, "manifolds: every column except tangent_velocity is required");
    ManifoldSource src;
    src.M = mc->count; src.P = mc->point_count;
    src.color_offsets = mc->color_offsets; src.body1 = mc->body1; src.body2 = mc->body2; src.friction = mc->friction; src.restitution = mc->restitution;
    src.tangent_velocity = mc->tangent_velocity; src.normal = mc->normal; src.point_offsets = mc->point_offsets;
    src.anchor1 = mc->anchor1; src.anchor2 = mc->anchor2; src.penetration = mc->penetration; src.normal_speed = mc->normal_speed;
    src.ws_normal = mc->warm_start_normal_impulse; src.ws_tangent = mc->warm_start_tangent_impulse; src.normal_impulse = mc->normal_impulse;
    return upload_impl(prm, bc, &src, js);
}

template <class S>
AvnStatus Solver<S>::upload_resident(const AvnStepParams* prm, AvnBodyColumns* bc, ContactsBase* contacts, AvnJointSet* js) {
    if (!contacts) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "upload_resident: no contact store");
    ContactsBase::AsleepBodies asleep;
    contacts->asleep_bodies(&asleep);
    if (asleep.wake_skipped)
        return err_->fail(AVN_ERR_INVALID_ARGUMENT, "upload_resident: sleeping is applied (avn_islands_apply) and avn_islands_wake has not run since the last avn_contacts_step");
    if (asleep.body_asleep && asleep.count != bc->count)
        return err_->fail(AVN_ERR_INVALID_ARGUMENT, "upload_resident: %zu bodies, sleeping is applied to %u", size_t(bc->count), asleep.count);
    struct Reset { const uint8_t*& p; ~Reset() { p = nullptr; } } reset{body_asleep_};   // only this upload reads the column
    body_asleep_ = asleep.body_asleep;
    ContactsBase::ResidentGraph g;
    AvnStatus st = contacts->graph_view(&g);
    if (st != AVN_OK) return st;
    ContactsBase::RowColumns v;
    contacts->view(&v);
    ManifoldSource src;
    src.resident = true;
    src.M = g.count; src.P = size_t(4) * v.rows;
    src.color_offsets = g.color_offsets; src.body1 = g.body1; src.body2 = g.body2; src.friction = g.friction; src.restitution = g.restitution;
    src.edge = g.edge;
    src.list_restitution = g.any_restitution != 0;
    src.normal = v.normal; src.edge_point_count = v.point_count;
    src.anchor1 = v.anchor1; src.anchor2 = v.anchor2; src.penetration = v.penetration; src.normal_speed = v.normal_speed;
    src.ws_normal = v.warm_start_normal_impulse; src.ws_tangent = v.warm_start_tangent_impulse; src.normal_impulse = v.normal_impulse;
    contacts->outputs(&src.out_ws_normal, &src.out_ws_tangent, &src.out_normal_impulse);
    return upload_impl(prm, bc, &src, js);
}

// the kind column the stage runs with while sleeping is applied: asleep -> static (kind == NULL: every body is dynamic)
__global__ void effective_kind_kernel(int B, const uint8_t* __restrict__ kind, const uint8_t* __restrict__ body_asleep, uint8_t* __restrict__ out) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < B) out[b] = body_asleep[b] ? uint8_t(AVN_BODY_STATIC) : kind ? kind[b] : uint8_t(AVN_BODY_DYNAMIC);
}

// fills the point ranges of the manifolds of a resident upload: 4 slots per row, the first point_count[row] of them live
__global__ void edge_ranges_kernel(const uint32_t* __restrict__ edge, const uint8_t* __restrict__ count, int M, uint32_t* __restrict__ begin,
                                   uint32_t* __restrict__ end) {
    int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    const uint32_t e = edge[m];
    begin[m] = 4u * e;
    end[m] = 4u * e + count[e];
}

template <class S>
AvnStatus Solver<S>::upload_impl(const AvnStepParams* prm, AvnBodyColumns* bc, const ManifoldSource* mc, AvnJointSet* js) {
    if (!prm || !bc) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "params and bodies are required");
    if (bc->count && (!bc->position || !bc->rotation || !bc->linear_velocity || !bc->angular_velocity || !bc->inverse_mass || !bc->inverse_inertia_local))
        return err_->fail(AVN_ERR_INVALID_ARGUMENT, "bodies: position, rotation, velocities, inverse_mass and inverse_inertia_local are required");
    if (!(prm->h > 0) || !(prm->dt > 0) || prm->substeps == 0) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "dt, h and substeps must be positive");
    from_store_ = mc && mc->resident;
    uploaded_ = false;
    ran_ = false;
    agreed_valid_ = false;
    h2d_bytes_ = 0;
    DevSolver<S>& d = dev_;
    d = DevSolver<S>{};
    const size_t B = bc->count;
    cudaEventRecord(ev_[EV_H2D0], stream_);
    // ---- parameters
    d.B = int(B);
    d.substeps = int(prm->substeps);
    d.iters = prm->solver_iterations ? int(prm->solver_iterations) : 1;
    d.rest_iters = int(prm->restitution_iterations);
    d.fast_trig = (cfg_flags_ & AVN_CFG_FAST_TRIG) ? 1 : 0;
    d.match_contacts = int(prm->match_contacts);
    d.h = S(prm->h);
    d.dt = S(prm->dt);
    length_unit_ = prm->length_unit;
    d.max_overlap_speed = S(prm->max_overlap_solve_speed) * S(prm->length_unit);
    d.warm_coeff = S(prm->warm_start_coefficient);
    d.rest_threshold = S(prm->restitution_threshold) * S(prm->length_unit);
    d.gx = S(prm->gravity[0]); d.gy = S(prm->gravity[1]); d.gz = S(prm->gravity[2]);
    {
        // update_contact_softness (solver/plugin.rs:326-350)
        S max_hz = S(1) / (d.dt * S(2));
        S hz = S(prm->contact_frequency_factor) * std::min(max_hz, S(0.25) / d.h);
        d.soft_dyn = softness<S>(S(prm->contact_damping_ratio), hz, d.h);
        d.soft_nondyn = softness<S>(S(prm->contact_damping_ratio), S(2) * hz, d.h);
        // writeback_joint_forces rhs (xpbd/plugin.rs:253): (delta_secs * delta_secs).recip_or_zero() * substeps, where delta_secs is the
        // FULL step dt — the system runs in SolverSystems::Finalize, after run_substep_schedule has set the generic Time back to
        // Time<Physics> (solver/schedule.rs:211-212).  (Round 1 used h here, in the oracle too: substeps^2 too large.)
        S dd = d.dt * d.dt;
        d.joint_force_rhs = ((dd != S(0) && std::isfinite(dd)) ? S(1) / dd : S(0)) * S(prm->substeps);
    }
    // ---- body columns
    AvnStatus st;
#define UP(buf, host, n, T, field) if ((st = up<T>(buf, host, n, &d.field)) != AVN_OK) return st
    if (prefetched_ && prefetch_matches(*bc)) {
        // avn_solver_prefetch_bodies already put this step's body columns on the device (copy stream): the kernels wait for that copy
        d.kind = bcols_.kind; d.locked = bcols_.locked; d.dominance = bcols_.dominance; d.integ_flags = bcols_.integ_flags;
        d.position = bcols_.position; d.rotation = bcols_.rotation; d.linvel = bcols_.linvel; d.angvel = bcols_.angvel;
        d.inv_mass = bcols_.inv_mass; d.inv_inertia_local = bcols_.inv_inertia_local; d.com = bcols_.com; d.lin_damp = bcols_.lin_damp;
        d.ang_damp = bcols_.ang_damp; d.grav_scale = bcols_.grav_scale; d.lin_acc = bcols_.lin_acc; d.ang_acc = bcols_.ang_acc;
        d.max_lin = bcols_.max_lin; d.max_ang = bcols_.max_ang;
        AVN_CUDA(cudaStreamWaitEvent(stream_, ev_prefetch_, 0));
    } else {
        if (prefetched_) AVN_CUDA(cudaStreamWaitEvent(stream_, ev_prefetch_, 0));   // a prefetch of other columns is still writing these buffers
        if ((st = upload_body_columns(*bc, false, d)) != AVN_OK) return st;
    }
    prefetched_ = false;
    if (body_asleep_ && B) {
        // a body that is asleep has no SolverBody (solver_body/plugin.rs:46-110): the stage sees it as static.  The uploaded column stays as it is
        // for AVN_BODIES_STATIC_UNCHANGED
        AVN_CUDA(b_kind_eff_.ensure(B));
        effective_kind_kernel<<<unsigned((B + 255) / 256), 256, 0, stream_>>>(int(B), d.kind, body_asleep_, b_kind_eff_.as<uint8_t>());
        AVN_CUDA(cudaGetLastError());
        d.kind = b_kind_eff_.as<uint8_t>();
    }
    AVN_CUDA(o_pos_.ensure(3 * B * sizeof(S) + 16)); d.out_position = o_pos_.as<S>();
    AVN_CUDA(o_rot_.ensure(4 * B * sizeof(S) + 16)); d.out_rotation = o_rot_.as<S>();
    AVN_CUDA(o_lv_.ensure(3 * B * sizeof(S) + 16)); d.out_linvel = o_lv_.as<S>();
    AVN_CUDA(o_av_.ensure(3 * B * sizeof(S) + 16)); d.out_angvel = o_av_.as<S>();
    const size_t state_bytes = 2 * (B + 1) * sizeof(Vec4<S>);
    AVN_CUDA(s_inr_.ensure(state_bytes)); d.inr = s_inr_.as<Vec4<S>>();
    AVN_CUDA(s_itg_.ensure(state_bytes)); d.itg = s_itg_.as<Vec4<S>>();
    AVN_CUDA(s_pre_.ensure(state_bytes)); d.pre = s_pre_.as<Vec4<S>>();
    // vel | dlt | ver | deg | contact planes are carved out of ONE allocation (after the manifold count is known, below): the
    // mutable front of it (vel, dlt, ver, deg, the four impulse planes) is the L2-persisting window.
    hb_ = *bc;
    // ---- manifolds
    have_m_ = mc != nullptr && mc->M > 0;
    AVN_CUDA(c_flag_.ensure(FLAG_WORDS * sizeof(int) + 8 * sizeof(unsigned long long)));  // FLAG_* words (solver_dev.cuh), then the optional trace counters
    d.any_restitution = c_flag_.as<int>();
    if (have_m_) {
        const size_t M = mc->M, P = mc->P;
        if (mc->color_offsets[0] != 0 || mc->color_offsets[AVN_GRAPH_COLOR_COUNT] != M)
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "manifolds: color_offsets must span [0, count]");
        for (int c = 0; c < AVN_GRAPH_COLOR_COUNT; ++c)
            if (mc->color_offsets[c] > mc->color_offsets[c + 1]) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "manifolds: color_offsets must be non-decreasing");
        if (mc->resident) {
            max_np_ = AVN_MAX_MANIFOLD_POINTS;   // the point counts live on the device: take the general kernel build
        } else {
            // widest manifold: sizes the shared-memory staging tile (3 rows per point) and validates the point ranges
            const uint32_t* po = mc->point_offsets;
            if (po[M] != P) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "manifolds: point_offsets[count] != point_count");
            uint32_t widest = 0, bad = 0;
            for (size_t i = 0; i < M; ++i) {
                bad |= uint32_t(po[i + 1] < po[i]);
                const uint32_t n = po[i + 1] - po[i];
                widest = n > widest ? n : widest;
            }
            if (bad || widest > AVN_MAX_MANIFOLD_POINTS)
                return err_->fail(AVN_ERR_INVALID_ARGUMENT, "manifolds: at most %d points per manifold, point ranges must not decrease", AVN_MAX_MANIFOLD_POINTS);
            max_np_ = int(std::max<uint32_t>(widest, 1));
            // body indices are gathered through on the device (inr[2*b], vel[2*b], ver[b] ...): anything outside [AVN_NO_BODY, B) would read and
            // write out of bounds, so it is rejected here (streaming pass over two int columns)
            const int32_t* hb1 = mc->body1; const int32_t* hb2 = mc->body2;
            const int64_t Bi = int64_t(B);
            uint32_t bad_body = 0;
            for (size_t i = 0; i < M; ++i) bad_body |= uint32_t(hb1[i] < AVN_NO_BODY) | uint32_t(hb1[i] >= Bi) | uint32_t(hb2[i] < AVN_NO_BODY) | uint32_t(hb2[i] >= Bi);
            if (bad_body) {
                for (size_t i = 0; i < M; ++i)
                    if (hb1[i] < AVN_NO_BODY || hb1[i] >= Bi || hb2[i] < AVN_NO_BODY || hb2[i] >= Bi)
                        return err_->fail(AVN_ERR_INVALID_ARGUMENT, "manifolds: body indices (%d, %d) of manifold %zu are outside [-1, %zu)", hb1[i], hb2[i], i, B);
            }
        }
        d.M = int(M);
        d.P = int(P);
        {   // padded slot layout: every colour starts at a multiple of 32
            int slot = 0;
            for (int c = 0; c < AVN_GRAPH_COLOR_COUNT; ++c) {
                d.m_color_off[c] = int(mc->color_offsets[c]);
                d.color_off[c] = slot;
                d.color_len[c] = int(mc->color_offsets[c + 1] - mc->color_offsets[c]);
                slot += (d.color_len[c] + 31) & ~31;
            }
            d.m_color_off[AVN_GRAPH_COLOR_COUNT] = int(M);
            d.color_off[AVN_GRAPH_COLOR_COUNT] = slot;
            d.Mpad = std::max(slot, 32);
        }
        if (mc->resident) {   // the contact store's list and rows, read in place (its bodies are the rows' bodies, validated when the pairs were formed)
            d.m_body1 = reinterpret_cast<const int*>(mc->body1); d.m_body2 = reinterpret_cast<const int*>(mc->body2);
            d.m_friction = static_cast<const S*>(mc->friction); d.m_restitution = static_cast<const S*>(mc->restitution);
            d.m_normal = static_cast<const S*>(mc->normal);
            d.m_src = mc->edge;
            AVN_CUDA(m_pbegin_.ensure(M * sizeof(uint32_t)));
            AVN_CUDA(m_pend_.ensure(M * sizeof(uint32_t)));
            edge_ranges_kernel<<<unsigned((M + 255) / 256), 256, 0, stream_>>>(d.m_src, mc->edge_point_count, int(M), m_pbegin_.as<uint32_t>(), m_pend_.as<uint32_t>());
            AVN_CUDA(cudaGetLastError());
            d.m_point_begin = m_pbegin_.as<uint32_t>();
            d.m_point_end = m_pend_.as<uint32_t>();
            d.p_anchor1 = static_cast<const S*>(mc->anchor1); d.p_anchor2 = static_cast<const S*>(mc->anchor2);
            d.p_penetration = static_cast<const S*>(mc->penetration); d.p_normal_speed = static_cast<const S*>(mc->normal_speed);
            d.p_ws_normal = static_cast<const S*>(mc->ws_normal); d.p_ws_tangent = static_cast<const S*>(mc->ws_tangent);
            d.p_in_normal_impulse = static_cast<const S*>(mc->normal_impulse);
            d.p_out_ws_normal = static_cast<S*>(mc->out_ws_normal); d.p_out_ws_tangent = static_cast<S*>(mc->out_ws_tangent);
            d.p_normal_impulse = static_cast<S*>(mc->out_normal_impulse);
            host_any_restitution_ = mc->list_restitution;
        } else {
            UP(m_b1_, mc->body1, M, int, m_body1);
            UP(m_b2_, mc->body2, M, int, m_body2);
            UP(m_f_, mc->friction, M, S, m_friction);
            UP(m_r_, mc->restitution, M, S, m_restitution);
            UP(m_n_, mc->normal, 3 * M, S, m_normal);
            UP(m_tv_, mc->tangent_velocity, 3 * M, S, m_tanvel);
            UP(m_po_, mc->point_offsets, M + 1, uint32_t, m_point_begin);
            d.m_point_end = d.m_point_begin + 1;
            UP(p_a1_, mc->anchor1, 3 * P, S, p_anchor1);
            UP(p_a2_, mc->anchor2, 3 * P, S, p_anchor2);
            UP(p_pen_, mc->penetration, P, S, p_penetration);
            UP(p_ns_, mc->normal_speed, P, S, p_normal_speed);
            // in/out columns: inputs and outputs live in separate device buffers so that avn_solver_run is repeatable
            UP(p_wn_, mc->ws_normal, P, S, p_ws_normal);
            UP(p_wt_, mc->ws_tangent, 2 * P, S, p_ws_tangent);
            UP(p_nin_, mc->normal_impulse, P, S, p_in_normal_impulse);
            AVN_CUDA(p_own_.ensure(P * sizeof(S) + 16)); d.p_out_ws_normal = p_own_.as<S>();
            AVN_CUDA(p_owt_.ensure(2 * P * sizeof(S) + 16)); d.p_out_ws_tangent = p_owt_.as<S>();
            AVN_CUDA(p_ni_.ensure(P * sizeof(S) + 16));
            d.p_normal_impulse = p_ni_.as<S>();
            host_any_restitution_ = false;
            const S* r = static_cast<const S*>(mc->restitution);
            for (size_t i = 0; i < M; ++i) host_any_restitution_ |= (r[i] != S(0));
        }
        hm_ = *mc;
    }
    {
        auto up256 = [](size_t x) { return (x + 255) & ~size_t(255); };
        const size_t vel_b = up256(state_bytes), dlt_b = up256(state_bytes), ver_b = up256((B + 1) * sizeof(unsigned)), deg_b = up256(2 * (B + 1) * sizeof(int));
        const size_t planes_b = have_m_ ? size_t(CP_PLANES) * d.Mpad * sizeof(Vec4<S>) : 0;
        const size_t pcr_b = have_m_ ? up256(size_t(AVN_MAX_MANIFOLD_POINTS) * d.Mpad * sizeof(Vec4<S>)) : 0;
        AVN_CUDA(hot_.ensure(vel_b + dlt_b + ver_b + deg_b + pcr_b + planes_b + 256));
        char* base = hot_.as<char>();
        d.vel = reinterpret_cast<Vec4<S>*>(base); base += vel_b;
        d.dlt = reinterpret_cast<Vec4<S>*>(base); base += dlt_b;
        d.ver = reinterpret_cast<unsigned*>(base); base += ver_b;
        d.deg = reinterpret_cast<int*>(base); d.stamp = d.deg + (B + 1); base += deg_b;
        d.pcr = have_m_ ? reinterpret_cast<Vec4<S>*>(base) : nullptr; base += pcr_b;
        d.cst = have_m_ ? reinterpret_cast<Vec4<S>*>(base) : nullptr;
        hot_bytes_ = vel_b + dlt_b + ver_b + deg_b + pcr_b;
    }
    // ---- joints
    have_j_ = false;
    if (js) {
        size_t J = 0;
        for (int t = 0; t < AVN_JOINT_TYPE_COUNT; ++t) J += js->types[t].count;
        if (J > 0) {
            if ((st = build_joint_schedule(*bc, *js)) != AVN_OK) return st;
            have_j_ = true;
            for (int t = 0; t < AVN_JOINT_TYPE_COUNT; ++t) {
                const AvnJointColumns& jc = js->types[t];
                const size_t n = jc.count;
                const void* cols[12] = {jc.local_anchor1, jc.local_anchor2, jc.local_basis1, jc.local_basis2, jc.axis, jc.limit_min,
                                        jc.limit_max, jc.limit2_min, jc.limit2_max, jc.compliance0, jc.compliance1, jc.compliance2};
                const size_t width[12] = {3, 3, 4, 4, 3, 1, 1, 1, 1, 1, 1, 1};
                for (int c = 0; c < 12; ++c) UP(jcol_[t][c], cols[c], width[c] * n, S, jc[t][c]);
                UP(jb1_[t], jc.body1, n, int, jbody1[t]);
                UP(jb2_[t], jc.body2, n, int, jbody2[t]);
                UP(jle_[t], jc.limit_enabled, n, uint8_t, jlimit_en[t]);
                UP(jde_[t], jc.damping_enabled, n, uint8_t, jdamp_en[t]);
                UP(jdl_[t], jc.damping_linear, n, S, jdamp_lin[t]);
                UP(jda_[t], jc.damping_angular, n, S, jdamp_ang[t]);
                d.jforce[t] = nullptr;
                d.jtorque[t] = nullptr;
                if (n && jc.force) { AVN_CUDA(jfo_[t].ensure(3 * n * sizeof(S))); d.jforce[t] = jfo_[t].as<S>(); }
                if (n && jc.torque) { AVN_CUDA(jto_[t].ensure(3 * n * sizeof(S))); d.jtorque[t] = jto_[t].as<S>(); }
            }
            UP(j_type_, h_type_.data(), h_type_.size(), int, j_src_type);
            UP(j_index_, h_index_.data(), h_index_.size(), int, j_src_index);
            UP(j_level_, h_level_off_.data(), h_level_off_.size(), int, level_off);
            UP(j_damp_slot_, h_damp_slot_.data(), h_damp_slot_.size(), int, jdamp_slot);
            UP(j_damp_level_, h_damp_level_off_.data(), h_damp_level_off_.size(), int, damp_level_off);
            AVN_CUDA(j_dummy_.ensure(2 * AVN_JOINT_TYPE_COUNT * sizeof(Vec4<S>)));
            d.jdummy = j_dummy_.as<Vec4<S>>();
            AVN_CUDA(j_planes_.ensure(size_t(JP_PLANES) * d.Jpad * sizeof(Vec4<S>)));
            d.jnt = j_planes_.as<Vec4<S>>();
            hj_ = *js;
        }
    }
#undef UP
    cudaEventRecord(ev_[EV_H2D1], stream_);
    uploaded_ = true;
    prepared_ = false;
    ran_ = false;
    dev_.bnd_of = nullptr;   // a new upload renumbers the bodies: the boundary list must be set again
    dev_.vel_ref = nullptr;
    bnd_n_ = 0;
    bnd_slots_ = 0;
    tm_ = AvnTimings{};
    return AVN_OK;
}

template <class S>
AvnStatus Solver<S>::run() {
    if (!ccd_active()) return launch_range(0, dev_.substeps, AVN_RUN_PREPARE | AVN_RUN_RESTITUTION | AVN_RUN_FINALIZE);
    // swept CCD (ccd.cu) runs after the substeps and before restitution (ccd/mod.rs:257-261): the step is split around it
    if (!uploaded_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_solver_run before avn_solver_upload");
    if (!from_store_ || !ccd_contacts_)
        return err_->fail(AVN_ERR_UNSUPPORTED, "swept CCD is configured: it needs the contact store's ContactGraph (avn_solver_upload_resident), "
                                               "not host manifolds");
    AvnStatus st = launch_range(0, uint32_t(dev_.substeps), AVN_RUN_PREPARE);
    if (st != AVN_OK) return st;
    CcdRows rows;
    ccd_contacts_->ccd_rows(&rows);
    CcdSolverState s;
    s.B = dev_.B; s.dt = double(dev_.dt); s.length_unit = length_unit_;
    s.kind = dev_.kind; s.position = dev_.position; s.rotation = dev_.rotation; s.com = dev_.com; s.vel = dev_.vel; s.dlt = dev_.dlt;
    if ((st = ccd_->run(s, rows, &launches_)) != AVN_OK) return st;
    return launch_range(uint32_t(dev_.substeps), 0, AVN_RUN_RESTITUTION | AVN_RUN_FINALIZE);
}

template <class S>
AvnStatus Solver<S>::run_range(uint32_t first, uint32_t count, uint32_t flags) {
    if (ccd_active()) return err_->fail(AVN_ERR_UNSUPPORTED, "avn_solver_run_range: swept CCD is configured (avn_solver_run runs the split step itself)");
    return launch_range(first, count, flags);
}

// One launch covering: prepare (flags & AVN_RUN_PREPARE), substeps [first, first + count), the restitution pass, the finalize phases.
// avn_solver_run is the whole step in one launch; the x-slab partition launches substep by substep with a boundary exchange in between.
template <class S>
AvnStatus Solver<S>::launch_range(uint32_t first, uint32_t count, uint32_t flags) {
    if (!uploaded_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_solver_run before avn_solver_upload");
    const bool prepare = (flags & AVN_RUN_PREPARE) != 0;
    if (!prepare && !prepared_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_solver_run_range: the first launch after an upload must include AVN_RUN_PREPARE");
    if (uint64_t(first) + count > uint64_t(dev_.substeps)) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_solver_run_range: substeps [%u, %u) exceed %d", first, first + count, dev_.substeps);
    dev_.do_prepare = prepare ? 1 : 0;
    dev_.sub_begin = int(first);
    dev_.sub_end = int(first + count);
    dev_.do_restitution = (flags & AVN_RUN_RESTITUTION) ? 1 : 0;
    dev_.do_finalize = (flags & AVN_RUN_FINALIZE) ? 1 : 0;
    bool mega = use_mega_ && coop_ok_;
    // blocks per SM, the same for both schedules: at 3 (170 registers) the f32 wavefront routines run without local-memory spills; at 4
    // (128 registers) the warm-start routine and the megakernel spill (DESIGN.md 3.1)
    if (prepare) step_bps_ = mega_bps_;
    mega = mega && select_megakernel(max_np_, step_bps_);
    if (prepare) {
        launches_ = 0;
        cudaEventRecord(ev_[EV_RUN0], stream_);
        AVN_CUDA(cudaMemsetAsync(dev_.any_restitution, 0, FLAG_WORDS * sizeof(int) + 8 * sizeof(unsigned long long), stream_));
        // wavefront substep loop: contacts only (joints keep the level-by-level barriers), empty overflow colour.  It wins when the step
        // is bound by the per-body dependency chain, i.e. when a colour does not fill the machine; with colours several times the
        // resident thread count (1M-sphere scene) the barriers are cheap and the counters are pure overhead (DESIGN.md 3.1).
        int widest_colour = 0;
        for (int c = 0; c < AVN_COLOR_OVERFLOW; ++c) widest_colour = std::max(widest_colour, dev_.color_len[c]);
        const bool chain_bound = force_wave_ || widest_colour <= 2 * mega_grid_ * MEGA_BLOCK;
        dev_.wave = (mega && use_wave_ && chain_bound && dev_.M > 0 && dev_.J == 0 && dev_.color_len[AVN_COLOR_OVERFLOW] == 0) ? 1 : 0;
        if (dev_.M > 0) {
            // padding slots must read as "no points": clear the index plane before prepare fills the live slots
            AVN_CUDA(cudaMemsetAsync(dev_.cst + size_t(CP_IDX) * dev_.Mpad, 0, size_t(dev_.Mpad) * sizeof(Vec4<S>), stream_));
        }
        if (dev_.wave) {
            AVN_CUDA(cudaMemsetAsync(dev_.ver, 0, (size_t(dev_.B) + 1) * sizeof(unsigned), stream_));
            AVN_CUDA(cudaMemsetAsync(dev_.deg, 0, 2 * (size_t(dev_.B) + 1) * sizeof(int), stream_));   // deg + stamp
        }
        mega_step_ = mega;
    } else {
        mega = mega && mega_step_;   // a step keeps the launch mode its prepare launch chose
    }
    if (l2_persist_ && hot_bytes_ > 0) {
        // pin the mutable state (body velocities/deltas, event counters, impulse planes) in L2: it sits on the critical dependency
        // chain, while the immutable constraint rows only stream through
        cudaStreamAttrValue attr{};
        attr.accessPolicyWindow.base_ptr = hot_.p;
        attr.accessPolicyWindow.num_bytes = std::min(hot_bytes_, l2_window_max_);
        attr.accessPolicyWindow.hitRatio = float(std::min(1.0, double(l2_persist_bytes_) / double(attr.accessPolicyWindow.num_bytes)));
        attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
        attr.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
        cudaStreamSetAttribute(stream_, cudaStreamAttributeAccessPolicyWindow, &attr);
    }
    const DevSolver<S>& d = dev_;
    if (mega) {
        void* args[] = {(void*)&dev_};
        cudaError_t e = cudaLaunchCooperativeKernel(mega_fn_, dim3(mega_grid_), dim3(MEGA_BLOCK), args, mega_smem_bytes(mega_maxp_), stream_);
        if (e != cudaSuccess) {
            (void)cudaGetLastError();
            if (!prepare && dev_.wave)
                return err_->fail(AVN_ERR_CUDA, "cooperative launch refused in the middle of a wavefront-scheduled step: %s", cudaGetErrorString(e));
            mega = false;  // fall through to phase launches (still the same CUDA arithmetic)
            mega_step_ = false;
            dev_.wave = 0;
        } else {
            ++launches_;
            if (prepare) cudaEventRecord(ev_[EV_PREP], stream_);
            if (dev_.do_finalize) cudaEventRecord(ev_[EV_LOOP], stream_);
        }
    }
    if (!mega) {
        if (prepare) {
            launch_phase<OP_PREPARE_BODY>(0, d.B + 1);
            launch_phase<OP_PREPARE_CONSTRAINT>(0, d.M);
            launch_phase<OP_PREPARE_JOINT>(0, d.J);
            cudaEventRecord(ev_[EV_PREP], stream_);
        }
        for (int sub = d.sub_begin; sub < d.sub_end; ++sub) {
            launch_phase<OP_INTEGRATE_VEL>(0, d.B);
            if (d.M > 0) {
                launch_contact_pass<OP_WARM>();
                for (int it = 0; it < d.iters; ++it) launch_contact_pass<OP_SOLVE_BIAS>();
            }
            launch_phase<OP_INTEGRATE_POS>(0, d.B);
            if (d.M > 0) launch_contact_pass<OP_RELAX>();
            if (d.J > 0) {
                for (int l = 0; l < d.n_levels; ++l) launch_phase<OP_SOLVE_JOINT>(h_level_off_[l], h_level_off_[l + 1] - h_level_off_[l]);
                launch_phase<OP_PROJECT_VEL>(0, d.B);
                for (int l = 0; l < d.n_damp_levels; ++l)
                    launch_phase<OP_DAMP_JOINT>(h_damp_level_off_[l], h_damp_level_off_[l + 1] - h_damp_level_off_[l]);
            }
        }
        if (d.do_finalize) cudaEventRecord(ev_[EV_LOOP], stream_);
        // restitution kernels early-out per manifold when e == 0; skipping the launches needs the device flag, which
        // would cost a sync, so in phase mode they are launched only when the host saw a non-zero coefficient
        if (d.do_restitution && d.M > 0 && host_any_restitution_) launch_contact_pass<OP_RESTITUTION>();
        if (d.do_finalize) {
            launch_phase<OP_WRITEBACK_BODY>(0, d.B);
            launch_phase<OP_STORE_IMPULSE>(0, d.M);
            launch_phase<OP_JOINT_FORCE>(0, d.J);
        }
    }
    AVN_CUDA(cudaGetLastError());
    prepared_ = true;
    if (dev_.do_finalize) {
        cudaEventRecord(ev_[EV_RUN1], stream_);
        ran_ = true;
    }
    return AVN_OK;
}

// ---- x-slab partition: boundary bodies (include/avian_b200.h) -------------------------------------------------------------
// record of one boundary slot in the exchange table: 4 rows of Vec4<S>:
//   row 0 = (dv.xyz, holder marker 1)   row 1 = (dw.xyz, owner marker 1)   row 2 = (delta_position.xyz, 0)   row 3 = delta_rotation
template <class S>
__global__ void boundary_snapshot_kernel(DevSolver<S> d, const int* __restrict__ body, int n) {
    int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const int b = body[k];
    st4(&d.vel_ref[2 * k], ld4(&d.vel[2 * b]));
    st4(&d.vel_ref[2 * k + 1], ld4(&d.vel[2 * b + 1]));
}
template <class S>
__global__ void boundary_pack_kernel(DevSolver<S> d, const int* __restrict__ body, const int* __restrict__ owner_rank, int n, int rank,
                                     Vec4<S>* __restrict__ table) {
    int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const int b = body[k];
    Vec4<S>* rec = table + size_t(4) * k;
    const Vec4<S> l = ld4(&d.vel[2 * b]), a = ld4(&d.vel[2 * b + 1]), l0 = ld4(&d.vel_ref[2 * k]), a0 = ld4(&d.vel_ref[2 * k + 1]);
    const bool owner = owner_rank[k] == rank;
    st4(&rec[0], mk4<S>(l.x - l0.x, l.y - l0.y, l.z - l0.z, S(1)));
    st4(&rec[1], mk4<S>(a.x - a0.x, a.y - a0.y, a.z - a0.z, owner ? S(1) : S(0)));
    if (owner) {
        st4(&rec[2], ld4(&d.dlt[2 * b]));
        st4(&rec[3], ld4(&d.dlt[2 * b + 1]));
    }
}
template <class S>
__global__ void boundary_apply_kernel(DevSolver<S> d, const int* __restrict__ body, const int* __restrict__ source, const int* __restrict__ owner_rank,
                                      int n, int world, size_t records, const Vec4<S>* __restrict__ gathered) {
    int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const int b = body[k];
    Vec4<S> l = ld4(&d.vel_ref[2 * k]), a = ld4(&d.vel_ref[2 * k + 1]);
    // every holder's constraint impulses of this substep, summed in rank order (the same order on every rank: identical bits)
    for (int r = 0; r < world; ++r) {
        const int idx = source[size_t(k) * world + r];
        if (idx < 0) continue;  // rank r does not hold this body
        const Vec4<S>* rec = gathered + (size_t(r) * records + size_t(idx)) * 4;
        const Vec4<S> dl = ld4(&rec[0]), da = ld4(&rec[1]);
        l.x = l.x + dl.x; l.y = l.y + dl.y; l.z = l.z + dl.z;
        a.x = a.x + da.x; a.y = a.y + da.y; a.z = a.z + da.z;
    }
    // the spare lanes of the velocity / delta rows are kept as they are
    st4(&d.vel[2 * b], mk4<S>(l.x, l.y, l.z, ld4(&d.vel[2 * b]).w));
    st4(&d.vel[2 * b + 1], mk4<S>(a.x, a.y, a.z, ld4(&d.vel[2 * b + 1]).w));
    const Vec4<S>* own = gathered + (size_t(owner_rank[k]) * records + size_t(source[size_t(k) * world + owner_rank[k]])) * 4;
    Vec4<S> odp = ld4(&own[2]);
    odp.w = ld4(&d.dlt[2 * b]).w;
    st4(&d.dlt[2 * b], odp);
    st4(&d.dlt[2 * b + 1], ld4(&own[3]));
}

template <class S>
AvnStatus Solver<S>::set_boundary(const AvnBoundary* bnd) {
    if (!uploaded_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_solver_set_boundary before avn_solver_upload");
    if (!bnd || bnd->count == 0) {
        dev_.bnd_of = nullptr;
        dev_.vel_ref = nullptr;
        bnd_n_ = 0;
        // a rank that holds no boundary body still takes part in the exchange of the others' tables
        bnd_slots_ = bnd ? size_t(bnd->record_count) : 0;
        bnd_rank_ = bnd ? int(bnd->rank) : 0;
        bnd_world_ = bnd ? int(bnd->world) : 1;
        return AVN_OK;
    }
    if (!bnd->body || !bnd->source || !bnd->owner_rank) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "boundary: body, source and owner_rank are required");
    if (bnd->count > bnd->record_count) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "boundary: count %u exceeds record_count %u", bnd->count, bnd->record_count);
    if (bnd->rank >= bnd->world) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "boundary: rank %u >= world %u", bnd->rank, bnd->world);
    if (dev_.J > 0) return err_->fail(AVN_ERR_UNSUPPORTED, "boundary exchange covers contact constraints only (joints shard by island)");
    const size_t n = bnd->count, B = size_t(dev_.B);
    std::vector<int> of(B + 1, -1);
    for (size_t k = 0; k < n; ++k) {
        const int b = bnd->body[k];
        if (b < 0 || size_t(b) >= B) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "boundary: body[%zu] = %d out of range", k, b);
        if (bnd->owner_rank[k] < 0 || uint32_t(bnd->owner_rank[k]) >= bnd->world) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "boundary: owner_rank[%zu] out of range", k);
        for (uint32_t r = 0; r < bnd->world; ++r) {
            const int idx = bnd->source[k * bnd->world + r];
            if (idx >= int(bnd->record_count)) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "boundary: source[%zu][%u] out of range", k, r);
        }
        if (bnd->source[k * bnd->world + bnd->rank] != int(k)) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "boundary: source[%zu][rank] must be %zu", k, k);
        if (bnd->source[k * bnd->world + bnd->owner_rank[k]] < 0) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "boundary: the owner of body[%zu] must hold it", k);
        if (of[b] != -1) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "boundary: body %d listed twice", b);
        of[b] = int(k);
    }
    AVN_CUDA(bnd_of_.ensure((B + 1) * sizeof(int)));
    AVN_CUDA(bnd_body_.ensure(n * sizeof(int)));
    AVN_CUDA(bnd_slot_.ensure(n * bnd->world * sizeof(int)));
    AVN_CUDA(bnd_owner_.ensure(n * sizeof(int)));
    AVN_CUDA(vel_ref_.ensure(2 * n * sizeof(Vec4<S>)));
    AVN_CUDA(cudaMemcpyAsync(bnd_of_.p, of.data(), (B + 1) * sizeof(int), cudaMemcpyHostToDevice, stream_));
    AVN_CUDA(cudaMemcpyAsync(bnd_body_.p, bnd->body, n * sizeof(int), cudaMemcpyHostToDevice, stream_));
    AVN_CUDA(cudaMemcpyAsync(bnd_slot_.p, bnd->source, n * bnd->world * sizeof(int), cudaMemcpyHostToDevice, stream_));
    AVN_CUDA(cudaMemcpyAsync(bnd_owner_.p, bnd->owner_rank, n * sizeof(int), cudaMemcpyHostToDevice, stream_));
    AVN_CUDA(cudaStreamSynchronize(stream_));   // `of` is a temporary
    dev_.bnd_of = bnd_of_.as<int>();
    dev_.vel_ref = vel_ref_.as<Vec4<S>>();
    bnd_n_ = int(n);
    bnd_rank_ = int(bnd->rank);
    bnd_world_ = int(bnd->world);
    bnd_slots_ = size_t(bnd->record_count);
    return AVN_OK;
}

template <class S>
AvnStatus Solver<S>::boundary_snapshot() {
    if (!prepared_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_solver_boundary_snapshot before the prepare launch");
    if (bnd_n_ > 0) {
        boundary_snapshot_kernel<S><<<(bnd_n_ + 255) / 256, 256, 0, stream_>>>(dev_, bnd_body_.as<int>(), bnd_n_);
        ++launches_;
    }
    AVN_CUDA(cudaGetLastError());
    return AVN_OK;
}

template <class S>
AvnStatus Solver<S>::boundary_pack(void* device_table) {
    if (!prepared_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_solver_boundary_pack before the prepare launch");
    if (bnd_slots_ == 0) return AVN_OK;
    if (!device_table) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "boundary table is required");
    AVN_CUDA(cudaMemsetAsync(device_table, 0, bnd_slots_ * 4 * sizeof(Vec4<S>), stream_));
    if (bnd_n_ > 0) {
        boundary_pack_kernel<S><<<(bnd_n_ + 255) / 256, 256, 0, stream_>>>(dev_, bnd_body_.as<int>(), bnd_owner_.as<int>(), bnd_n_, bnd_rank_,
                                                                            static_cast<Vec4<S>*>(device_table));
        ++launches_;
    }
    AVN_CUDA(cudaGetLastError());
    return AVN_OK;
}

template <class S>
AvnStatus Solver<S>::boundary_apply(const void* device_gathered) {
    if (!prepared_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_solver_boundary_apply before the prepare launch");
    if (bnd_n_ == 0) return AVN_OK;
    if (!device_gathered) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "gathered boundary tables are required");
    boundary_apply_kernel<S><<<(bnd_n_ + 255) / 256, 256, 0, stream_>>>(dev_, bnd_body_.as<int>(), bnd_slot_.as<int>(), bnd_owner_.as<int>(), bnd_n_, bnd_world_,
                                                                         bnd_slots_, static_cast<const Vec4<S>*>(device_gathered));
    ++launches_;
    AVN_CUDA(cudaGetLastError());
    return AVN_OK;
}

// One rank's share of a scene cut into x-slabs (include/avian_b200.h "one coupled scene over several GPUs"): the step kernel substep by
// substep (the wavefront counters keep counting across the launches), and after every substep
//     pack (this rank's records) -> all-gather of the packed tables over the context's communicator -> apply (rank-ordered sums)
// all on the context's stream, so nothing synchronises with the host inside the step except one agreement per step on whether a
// restitution pass is needed anywhere.  Protocol and its CPU twin: DESIGN.md 4.2, oracle/oracle_step.cpp orc_step_*.
template <class S>
AvnStatus Solver<S>::step_partitioned(CommBase* comm) {
    if (!uploaded_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_solver_step_partitioned before avn_solver_upload");
    if (ccd_active()) return err_->fail(AVN_ERR_UNSUPPORTED, "avn_solver_step_partitioned: swept CCD is not supported in the x-slab partition");
    if (!comm) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "no communicator");
    const int world = comm->world();
    if (bnd_slots_ > 0 && (bnd_world_ != world || bnd_rank_ != comm->rank()))
        return err_->fail(AVN_ERR_INVALID_ARGUMENT, "boundary was set for rank %d of %d, the communicator is rank %d of %d", bnd_rank_, bnd_world_, comm->rank(), world);
    const size_t table_bytes = bnd_slots_ * 4 * sizeof(Vec4<S>);
    if (table_bytes) {
        AVN_CUDA(bnd_table_.ensure(table_bytes));
        AVN_CUDA(bnd_gathered_.ensure(table_bytes * size_t(world)));
    }
    AvnStatus st;
    auto exchange = [&]() -> AvnStatus {
        if (table_bytes == 0) return AVN_OK;
        AvnStatus e = boundary_pack(bnd_table_.p);
        if (e != AVN_OK) return e;
        if ((e = comm->all_gather(bnd_table_.p, bnd_gathered_.p, table_bytes)) != AVN_OK) return e;
        ++exchanges_;
        return boundary_apply(bnd_gathered_.p);
    };
    exchanges_ = 0;
    // agreement on the restitution pass (every rank must launch it, and exchange after it, or none): max over ranks of the host flag
    int any_rest = host_any_restitution_ ? 1 : 0;
    if (world > 1 && agreed_valid_) {
        any_rest = agreed_rest_;     // agreed right after this upload already (every rank uploads once per step, in lockstep)
    } else if (world > 1) {
        AVN_CUDA(bnd_agree_.ensure(sizeof(int)));
        if (!h_agree_) AVN_CUDA(cudaHostAlloc(&h_agree_, sizeof(int), cudaHostAllocDefault));
        *h_agree_ = any_rest;
        AVN_CUDA(cudaMemcpyAsync(bnd_agree_.p, h_agree_, sizeof(int), cudaMemcpyHostToDevice, stream_));
        if ((st = comm->all_reduce_max_i32(bnd_agree_.as<int>(), 1)) != AVN_OK) return st;
        AVN_CUDA(cudaMemcpyAsync(h_agree_, bnd_agree_.p, sizeof(int), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        any_rest = *h_agree_;
        agreed_rest_ = any_rest;
        agreed_valid_ = true;
    }
    const uint32_t substeps = uint32_t(dev_.substeps);
    for (uint32_t s = 0; s < substeps; ++s) {
        if ((st = run_range(s, 1, s == 0 ? AVN_RUN_PREPARE : 0u)) != AVN_OK) return st;
        if ((st = exchange()) != AVN_OK) return st;
    }
    if (substeps == 0 && (st = run_range(0, 0, AVN_RUN_PREPARE)) != AVN_OK) return st;
    if (any_rest) {
        if ((st = boundary_snapshot()) != AVN_OK) return st;
        if ((st = run_range(substeps, 0, AVN_RUN_RESTITUTION)) != AVN_OK) return st;
        if ((st = exchange()) != AVN_OK) return st;
    }
    return run_range(substeps, 0, AVN_RUN_FINALIZE);
}

template <class S>
AvnStatus Solver<S>::download() {
    if (!ran_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_solver_download before avn_solver_run");
    const size_t B = hb_.count;
    cudaEventRecord(ev_[EV_D2H0], stream_);
    if (B) {
        AVN_CUDA(cudaMemcpyAsync(hb_.position, dev_.out_position, 3 * B * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(hb_.rotation, dev_.out_rotation, 4 * B * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(hb_.linear_velocity, dev_.out_linvel, 3 * B * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(hb_.angular_velocity, dev_.out_angvel, 3 * B * sizeof(S), cudaMemcpyDeviceToHost, stream_));
    }
    if (have_m_ && !hm_.resident) {
        const size_t P = hm_.P;
        AVN_CUDA(cudaMemcpyAsync(hm_.ws_normal, dev_.p_out_ws_normal, P * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(hm_.ws_tangent, dev_.p_out_ws_tangent, 2 * P * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(hm_.normal_impulse, dev_.p_normal_impulse, P * sizeof(S), cudaMemcpyDeviceToHost, stream_));
    }
    if (have_j_) {
        for (int t = 0; t < AVN_JOINT_TYPE_COUNT; ++t) {
            const size_t n = hj_.types[t].count;
            if (n && dev_.jforce[t]) AVN_CUDA(cudaMemcpyAsync(hj_.types[t].force, dev_.jforce[t], 3 * n * sizeof(S), cudaMemcpyDeviceToHost, stream_));
            if (n && dev_.jtorque[t]) AVN_CUDA(cudaMemcpyAsync(hj_.types[t].torque, dev_.jtorque[t], 3 * n * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        }
    }
    int flags_host[2] = {0, 0};
    AVN_CUDA(cudaMemcpyAsync(flags_host, dev_.any_restitution, sizeof flags_host, cudaMemcpyDeviceToHost, stream_));
    cudaEventRecord(ev_[EV_D2H1], stream_);
    AVN_CUDA(cudaStreamSynchronize(stream_));
#ifdef AVN_WAVE_TRACE
    {
        unsigned long long tr[8];
        cudaMemcpy(tr, dev_.any_restitution + FLAG_WORDS, sizeof tr, cudaMemcpyDeviceToHost);
        if (tr[4]) fprintf(stderr, "[avn wave trace] contact item-warps %llu  avg cycles: stage 1 (wait deltas + separations + coefficients) %.0f  wait %.0f  loads %.0f  compute %.0f  "
                           "store+publish %.0f\n", tr[4], double(tr[5]) / tr[4], double(tr[0]) / tr[4], double(tr[1]) / tr[4], double(tr[2]) / tr[4], double(tr[3]) / tr[4]);
    }
#endif
    if (flags_host[1] == WAVE_BAD_COLOURING)
        return err_->fail(AVN_ERR_INVALID_ARGUMENT, "manifolds: invalid colouring — a body with a SolverBody appears twice in one graph colour (or carries more than 254 "
                                                    "constraints): the colours are not conflict-free, the results of this step are not reliable");
    if (flags_host[1] == WAVE_WATCHDOG) return err_->fail(AVN_ERR_CUDA, "wavefront scheduler watchdog fired: results are invalid (set AVN_LAUNCH_MODE=barrier)");
    float ms = 0;
    if (cudaEventElapsedTime(&ms, ev_[EV_H2D0], ev_[EV_H2D1]) == cudaSuccess) tm_.h2d_ms = ms;
    if (cudaEventElapsedTime(&ms, ev_[EV_RUN0], ev_[EV_PREP]) == cudaSuccess) tm_.prepare_ms = ms;
    if (cudaEventElapsedTime(&ms, ev_[EV_PREP], ev_[EV_LOOP]) == cudaSuccess) tm_.substep_loop_ms = ms;
    if (cudaEventElapsedTime(&ms, ev_[EV_LOOP], ev_[EV_RUN1]) == cudaSuccess) tm_.finalize_ms = ms;
    if (cudaEventElapsedTime(&ms, ev_[EV_D2H0], ev_[EV_D2H1]) == cudaSuccess) tm_.d2h_ms = ms;
    if (cudaEventElapsedTime(&ms, ev_[EV_RUN0], ev_[EV_RUN1]) == cudaSuccess) tm_.total_ms = ms;
    tm_.kernel_launches = launches_;
    tm_.contact_constraint_count = uint32_t(dev_.M);
    tm_.joint_levels = uint32_t(dev_.n_levels);
    uint32_t ac = 0;
    for (int c = 0; c < AVN_GRAPH_COLOR_COUNT; ++c) ac += dev_.color_len[c] > 0;
    tm_.active_colors = ac;
    tm_.launch_mode = !mega_step_ ? AVN_LAUNCH_PHASES : (dev_.wave ? AVN_LAUNCH_MEGA_WAVE : AVN_LAUNCH_MEGA_BARRIER);
    return AVN_OK;
}

}  // namespace

SolverBase* make_solver(uint32_t scalar_bits, cudaStream_t stream, ErrorSink* err, uint32_t cfg_flags, int device) {
    if (scalar_bits == 32) return new Solver<float>(stream, err, cfg_flags, device);
    if (scalar_bits == 64) return new Solver<double>(stream, err, cfg_flags, device);
    return nullptr;
}

}  // namespace avn
