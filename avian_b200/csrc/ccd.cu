// Swept continuous collision detection on the device (include/avian_b200.h avn_ccd_*): solve_swept_ccd (dynamics/ccd/mod.rs:523-687) between
// the substeps and restitution of the device-resident solver stage.  The geometry is csrc/ccd_math.hpp, shared with the host brute force
// (host/host_api.cpp avh_ccd_solve), which the device equals bit for bit.
//
//   1. candidates: one thread per contact row.  A row whose collider is a configured CCD collider (collider -> slot table) passes the
//      filters of its slot and is appended to the candidate list (atomic counter: the results below do not depend on the list's order).
//   2. TOI: one thread per candidate (the grid is sized for every row, the threads past the device-side count leave), so a warp does only
//      real TOI work.  Per slot the smallest accepted TOI (ordered bits, atomicMin), then among the candidates that reached it the lowest
//      ContactId — the stated tie deviation.  The instance is the lowest shape level that covers the contact store's shape column: G = 2
//      (convex hulls, with the context's hull table) when it holds a hull, G = 1 (capsules) when it holds a capsule, else G = 0 (cuboids
//      and spheres); AVN_CCD_HULLS / AVN_CCD_CAPSULES let such a store through.  The other kernels read no geometry.
//   3. apply: per slot with a hit, one record for body 1 and one for body 2 when it has a SolverBody, record index = 2 * slot + side.  A
//      stable radix sort by body keeps every body's records in slot order; one thread per body replays them: the last delta_position wins
//      and the delta_rotation compositions happen in order — the reference's sequential loop, bit for bit.
#include <algorithm>
#include <cmath>
#include <vector>

#include "avn_math.cuh"
#include "ccd_math.hpp"
#include "context.hpp"
#include "device_prims.cuh"

namespace avn {
namespace {

constexpr int CCD_BLOCK = 256;
constexpr uint32_t CAND_SIDE = 1u << 30, CAND_LINEAR = 1u << 31, CAND_ROW = CAND_SIDE - 1;

template <class S> __device__ __forceinline__ unsigned long long toi_key(S t);
template <> __device__ __forceinline__ unsigned long long toi_key(float t) { return __float_as_uint(t); }
template <> __device__ __forceinline__ unsigned long long toi_key(double t) { return (unsigned long long)__double_as_longlong(t); }

template <class S>
struct CcdDev {
    int K, B;
    S dt;
    double eps, prediction;
    const int* body; const uint32_t* collider; const uint8_t* mode; const uint8_t* include_dynamic; const S* lthr; const S* athr;
    const int* slot_of_collider; int n_colliders;
    const int* slot_of_body; int n_bodies;
    // step state
    const uint8_t* kind; const S* position; const S* rotation; const S* com; const Vec4<S>* vel; Vec4<S>* dlt;
    const uint32_t* c1; const uint32_t* c2; const uint32_t* b1; const uint32_t* b2; const uint8_t* live; const uint8_t* shape; const S* dims; int rows;
    // work
    uint32_t* cand; uint32_t* cand_count; S* cand_toi;
    unsigned long long* best; uint32_t* best_row; uint32_t* ncand; uint32_t* nhit;
    S* out_min; int* out_body; int* out_contact; S* m;
    uint32_t* rec_key; uint32_t* rec_val;
};

template <class S> __device__ __forceinline__ bool has_solver_body(const CcdDev<S>& d, uint32_t b) {
    return b < uint32_t(d.B) && (d.kind ? d.kind[b] : AVN_BODY_DYNAMIC) != AVN_BODY_STATIC;
}
template <class S> __device__ __forceinline__ ccd::V3T<S> vel_row(const CcdDev<S>& d, uint32_t b, int r) {
    if (!has_solver_body(d, b)) return {S(0), S(0), S(0)};   // SolverBody::DUMMY
    const Vec4<S> v = d.vel[2 * size_t(b) + r];
    return {v.x, v.y, v.z};
}
template <class S> __device__ ccd::Motion motion(const CcdDev<S>& d, uint32_t b, uint32_t c) {
    ccd::Motion m;
    m.shape = d.shape ? d.shape[c] : nm::SHAPE_CUBOID;
    m.he = nm::V3{double(d.dims[3 * size_t(c)]), double(d.dims[3 * size_t(c) + 1]), double(d.dims[3 * size_t(c) + 2])};
    m.p = nm::V3{double(d.position[3 * size_t(b)]), double(d.position[3 * size_t(b) + 1]), double(d.position[3 * size_t(b) + 2])};
    m.q = nm::Q{double(d.rotation[4 * size_t(b)]), double(d.rotation[4 * size_t(b) + 1]), double(d.rotation[4 * size_t(b) + 2]), double(d.rotation[4 * size_t(b) + 3])};
    m.lc = d.com ? nm::V3{double(d.com[3 * size_t(b)]), double(d.com[3 * size_t(b) + 1]), double(d.com[3 * size_t(b) + 2])} : nm::V3{0, 0, 0};
    const ccd::V3T<S> v = vel_row(d, b, 0), w = vel_row(d, b, 1);
    m.v = nm::V3{double(v.x), double(v.y), double(v.z)};
    m.w = nm::V3{double(w.x), double(w.y), double(w.z)};
    return m;
}

// 1. candidates: the filters of solve_swept_ccd (ccd/mod.rs:566-607) per (row, CCD side)
template <class S>
__global__ void __launch_bounds__(CCD_BLOCK) ccd_candidates_kernel(CcdDev<S> d) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= d.rows || !d.live[e]) return;
    for (int side = 0; side < 2; ++side) {
        const uint32_t own = side ? d.c2[e] : d.c1[e];
        if (own >= uint32_t(d.n_colliders)) continue;
        const int k = d.slot_of_collider[own];
        if (k < 0) continue;
        const uint32_t body1 = uint32_t(d.body[k]), body2 = side ? d.b1[e] : d.b2[e];
        if (!has_solver_body(d, body1) || body2 >= uint32_t(d.B) || body2 == body1) continue;
        const bool dyn2 = (d.kind ? d.kind[body2] : AVN_BODY_DYNAMIC) == AVN_BODY_DYNAMIC;
        if (!d.include_dynamic[k] && dyn2) continue;
        if (ccd::below_thresholds<S>(vel_row(d, body1, 0), vel_row(d, body1, 1), vel_row(d, body2, 0), vel_row(d, body2, 1), d.lthr[k], d.athr[k])) continue;
        const int k2 = body2 < uint32_t(d.n_bodies) ? d.slot_of_body[body2] : -1;
        const bool linear = d.mode[k] == ccd::MODE_LINEAR && (k2 < 0 || d.mode[k2] == ccd::MODE_LINEAR);
        const uint32_t i = atomicAdd(d.cand_count, 1u);
        d.cand[i] = uint32_t(e) | (side ? CAND_SIDE : 0u) | (linear ? CAND_LINEAR : 0u);
        atomicAdd(&d.ncand[k], 1u);
    }
}

// 2. the TOI of every candidate (compute_ccd_toi, ccd/mod.rs:692-780) and the per-slot minimum
template <class S, int G>
__global__ void __launch_bounds__(CCD_BLOCK) ccd_toi_kernel(CcdDev<S> d, hm::Table hulls) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *d.cand_count) return;
    const uint32_t c = d.cand[i], e = c & CAND_ROW;
    const bool side = (c & CAND_SIDE) != 0;
    const uint32_t own = side ? d.c2[e] : d.c1[e], other = side ? d.c1[e] : d.c2[e];
    const int k = d.slot_of_collider[own];
    const uint32_t body1 = uint32_t(d.body[k]), body2 = side ? d.b1[e] : d.b2[e];
    const ccd::Motion A = motion(d, body1, own), Bm = motion(d, body2, other);
    const S t = ccd::pair_toi<S, G>((c & CAND_LINEAR) ? ccd::MODE_LINEAR : ccd::MODE_NON_LINEAR, A, Bm, d.dt, d.eps, d.prediction, &hulls);
    d.cand_toi[i] = t;
    if (t > S(0) && t < d.dt) {
        atomicAdd(&d.nhit[k], 1u);
        atomicMin(&d.best[k], toi_key(t));
    }
}

template <class S>
__global__ void __launch_bounds__(CCD_BLOCK) ccd_tie_kernel(CcdDev<S> d) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *d.cand_count) return;
    const S t = d.cand_toi[i];
    if (!(t > S(0) && t < d.dt)) return;
    const uint32_t c = d.cand[i], e = c & CAND_ROW;
    const int k = d.slot_of_collider[(c & CAND_SIDE) ? d.c2[e] : d.c1[e]];
    if (toi_key(t) == d.best[k]) atomicMin(&d.best_row[k], e);
}

// 3a. per slot: the result and its two records
template <class S>
__global__ void __launch_bounds__(CCD_BLOCK) ccd_records_kernel(CcdDev<S> d) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= d.K) return;
    const uint32_t e = d.best_row[k];
    uint32_t key1 = uint32_t(d.B), key2 = uint32_t(d.B);
    S min_toi = d.dt;
    int hit_body = -1;
    if (e != 0xffffffffu) {
        const bool own_first = d.c1[e] == d.collider[k];
        const uint32_t body2 = own_first ? d.b2[e] : d.b1[e];
        const unsigned long long key = d.best[k];
        if (sizeof(S) == 4) { const float f = __uint_as_float(uint32_t(key)); min_toi = S(f); }
        else { const double g = __longlong_as_double((long long)key); min_toi = S(g); }
        hit_body = int(body2);
        key1 = uint32_t(d.body[k]);
        if (has_solver_body(d, body2)) key2 = body2;
    }
    d.out_min[k] = min_toi;
    d.out_body[k] = hit_body;
    d.out_contact[k] = e == 0xffffffffu ? -1 : int(e);
    d.m[k] = ccd::overshoot(min_toi);
    d.rec_key[2 * k] = key1; d.rec_val[2 * k] = 2u * uint32_t(k);
    d.rec_key[2 * k + 1] = key2; d.rec_val[2 * k + 1] = 2u * uint32_t(k) + 1u;
}

// 3b. one thread per body that has records: replay them in slot order (keys sorted stably, so a body's run is in record order)
template <class S>
__global__ void __launch_bounds__(CCD_BLOCK) ccd_apply_kernel(CcdDev<S> d, const uint32_t* __restrict__ key, const uint32_t* __restrict__ val, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t b = key[i];
    if (b >= uint32_t(d.B) || (i > 0 && key[i - 1] == b)) return;
    const ccd::V3T<S> v = vel_row(d, b, 0), w = vel_row(d, b, 1);
    const Vec4<S> dp4 = d.dlt[2 * size_t(b)], dq4 = d.dlt[2 * size_t(b) + 1];
    ccd::V3T<S> dp{dp4.x, dp4.y, dp4.z};
    ccd::QT<S> dq{dq4.x, dq4.y, dq4.z, dq4.w};
    for (int j = i; j < n && key[j] == b; ++j) ccd::apply_record(d.m[val[j] >> 1], v, w, dp, dq);
    d.dlt[2 * size_t(b)] = mk4<S>(dp.x, dp.y, dp.z, dp4.w);
    d.dlt[2 * size_t(b) + 1] = mk4<S>(dq.x, dq.y, dq.z, dq.w);
}

template <class S>
class Ccd final : public CcdBase {
   public:
    Ccd(cudaStream_t stream, ErrorSink* err) : stream_(stream), err_(err) {
        cudaEventCreate(&ev0_);
        cudaEventCreate(&ev1_);
    }
    ~Ccd() override {
        cudaEventDestroy(ev0_);
        cudaEventDestroy(ev1_);
    }

    AvnStatus configure(const AvnCcdConfig* cfg, const CcdRows& rows) override {
        if (!cfg || cfg->count == 0) {
            K_ = 0;
            ran_ = false;
            capsules_ = hulls_flag_ = false;
            return AVN_OK;
        }
        if (!cfg->body || !cfg->collider) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "ccd: body and collider are required");
        if (rows.bodies == 0 && rows.colliders == 0) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "ccd: avn_contacts_configure first (bodies and colliders are checked against it)");
        if (std::isnan(cfg->prediction_distance)) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "ccd: prediction_distance is NaN");
        const size_t n = cfg->count;
        std::vector<int> slot_c(rows.colliders, -1), slot_b(rows.bodies, -1);
        std::vector<uint8_t> mode(n), inc(n);
        std::vector<S> lt(n), at(n);
        for (size_t k = 0; k < n; ++k) {
            const int b = cfg->body[k];
            const uint32_t c = cfg->collider[k];
            if (b < 0 || uint32_t(b) >= rows.bodies) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "ccd: body[%zu] = %d out of range [0, %u)", k, b, rows.bodies);
            if (c >= rows.colliders) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "ccd: collider[%zu] = %u out of range [0, %u)", k, c, rows.colliders);
            if (slot_b[b] >= 0) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "ccd: body %d listed twice", b);
            if (slot_c[c] >= 0) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "ccd: collider %u listed twice", c);
            mode[k] = cfg->mode ? cfg->mode[k] : uint8_t(AVN_SWEEP_NON_LINEAR);
            if (mode[k] != AVN_SWEEP_LINEAR && mode[k] != AVN_SWEEP_NON_LINEAR) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "ccd: mode[%zu] = %u is not an AvnSweepMode", k, mode[k]);
            const double l = cfg->linear_threshold ? cfg->linear_threshold[k] : 0.0, a = cfg->angular_threshold ? cfg->angular_threshold[k] : 0.0;
            if (std::isnan(l) || std::isnan(a)) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "ccd: threshold %zu is NaN", k);
            inc[k] = cfg->include_dynamic ? (cfg->include_dynamic[k] ? 1 : 0) : 1;
            lt[k] = S(l);
            at[k] = S(a);
            slot_b[b] = int(k);
            slot_c[c] = int(k);
        }
        AVN_CUDA(body_.ensure(n * 4)); AVN_CUDA(coll_.ensure(n * 4)); AVN_CUDA(mode_.ensure(n)); AVN_CUDA(inc_.ensure(n));
        AVN_CUDA(lt_.ensure(n * sizeof(S))); AVN_CUDA(at_.ensure(n * sizeof(S)));
        AVN_CUDA(slot_c_.ensure(std::max<size_t>(slot_c.size(), 1) * 4)); AVN_CUDA(slot_b_.ensure(std::max<size_t>(slot_b.size(), 1) * 4));
        AVN_CUDA(cudaMemcpyAsync(body_.p, cfg->body, n * 4, cudaMemcpyHostToDevice, stream_));
        AVN_CUDA(cudaMemcpyAsync(coll_.p, cfg->collider, n * 4, cudaMemcpyHostToDevice, stream_));
        AVN_CUDA(cudaMemcpyAsync(mode_.p, mode.data(), n, cudaMemcpyHostToDevice, stream_));
        AVN_CUDA(cudaMemcpyAsync(inc_.p, inc.data(), n, cudaMemcpyHostToDevice, stream_));
        AVN_CUDA(cudaMemcpyAsync(lt_.p, lt.data(), n * sizeof(S), cudaMemcpyHostToDevice, stream_));
        AVN_CUDA(cudaMemcpyAsync(at_.p, at.data(), n * sizeof(S), cudaMemcpyHostToDevice, stream_));
        if (!slot_c.empty()) AVN_CUDA(cudaMemcpyAsync(slot_c_.p, slot_c.data(), slot_c.size() * 4, cudaMemcpyHostToDevice, stream_));
        if (!slot_b.empty()) AVN_CUDA(cudaMemcpyAsync(slot_b_.p, slot_b.data(), slot_b.size() * 4, cudaMemcpyHostToDevice, stream_));
        // per-slot results and the records: sized once per configuration
        AVN_CUDA(best_.ensure(n * 8)); AVN_CUDA(best_row_.ensure(n * 4)); AVN_CUDA(ncand_.ensure(n * 4)); AVN_CUDA(nhit_.ensure(n * 4));
        AVN_CUDA(out_min_.ensure(n * sizeof(S))); AVN_CUDA(out_body_.ensure(n * 4)); AVN_CUDA(out_contact_.ensure(n * 4)); AVN_CUDA(m_.ensure(n * sizeof(S)));
        const size_t R = 2 * n, nblocks = (R + RS_TILE - 1) / RS_TILE;
        AVN_CUDA(k0_.ensure(R * 4)); AVN_CUDA(k1_.ensure(R * 4)); AVN_CUDA(v0_.ensure(R * 4)); AVN_CUDA(v1_.ensure(R * 4));
        AVN_CUDA(hist_.ensure(256 * nblocks * 4));
        AVN_CUDA(count_.ensure(4));
        AVN_CUDA(cudaStreamSynchronize(stream_));   // the host vectors are temporaries
        K_ = int(n);
        ran_ = false;
        n_colliders_ = int(rows.colliders);
        n_bodies_ = int(rows.bodies);
        prediction_ = cfg->prediction_distance;
        capsules_ = (cfg->flags & AVN_CCD_CAPSULES) != 0;
        hulls_flag_ = (cfg->flags & AVN_CCD_HULLS) != 0;
        return AVN_OK;
    }

    bool active() const override { return K_ > 0; }
    bool capsules() const override { return capsules_; }
    bool hulls() const override { return hulls_flag_; }
    void attach_hulls(const HullTable* hulls) override { table_ = hulls; }
    bool table_changed(const CcdRows& rows) const override {
        return rows.has_hull && rows.dims && rows.rows > 0 && (!table_ || !table_->set || table_->generation != rows.hull_generation);
    }

    AvnStatus run(const CcdSolverState& st, const CcdRows& rows, uint32_t* launches) override {
        CcdDev<S> d{};
        d.K = K_; d.B = st.B; d.dt = S(st.dt);
        d.eps = ccd::CCD_EPS_PER_LENGTH_UNIT * st.length_unit;
        d.prediction = prediction_;
        d.body = body_.as<int>(); d.collider = coll_.as<uint32_t>(); d.mode = mode_.as<uint8_t>(); d.include_dynamic = inc_.as<uint8_t>();
        d.lthr = lt_.as<S>(); d.athr = at_.as<S>();
        d.slot_of_collider = slot_c_.as<int>(); d.n_colliders = n_colliders_;
        d.slot_of_body = slot_b_.as<int>(); d.n_bodies = n_bodies_;
        d.kind = st.kind; d.position = static_cast<const S*>(st.position); d.rotation = static_cast<const S*>(st.rotation); d.com = static_cast<const S*>(st.com);
        d.vel = static_cast<const Vec4<S>*>(st.vel); d.dlt = static_cast<Vec4<S>*>(st.dlt);
        // no geometry on the device yet (no avn_contacts_step): no candidates
        d.rows = rows.dims ? int(rows.rows) : 0;
        d.c1 = rows.c1; d.c2 = rows.c2; d.b1 = rows.b1; d.b2 = rows.b2; d.live = rows.live; d.shape = rows.shape; d.dims = static_cast<const S*>(rows.dims);
        const size_t cand_cap = 2 * size_t(std::max(d.rows, 1));
        AVN_CUDA(cand_.ensure(cand_cap * 4));
        AVN_CUDA(cand_toi_.ensure(cand_cap * sizeof(S)));
        d.cand = cand_.as<uint32_t>(); d.cand_count = count_.as<uint32_t>(); d.cand_toi = cand_toi_.as<S>();
        d.best = best_.as<unsigned long long>(); d.best_row = best_row_.as<uint32_t>(); d.ncand = ncand_.as<uint32_t>(); d.nhit = nhit_.as<uint32_t>();
        d.out_min = out_min_.as<S>(); d.out_body = out_body_.as<int>(); d.out_contact = out_contact_.as<int>(); d.m = m_.as<S>();
        d.rec_key = k0_.as<uint32_t>(); d.rec_val = v0_.as<uint32_t>();
        const size_t K = size_t(K_);
        AVN_CUDA(cudaEventRecord(ev0_, stream_));
        AVN_CUDA(cudaMemsetAsync(count_.p, 0, 4, stream_));
        AVN_CUDA(cudaMemsetAsync(best_.p, 0xff, K * 8, stream_));
        AVN_CUDA(cudaMemsetAsync(best_row_.p, 0xff, K * 4, stream_));
        AVN_CUDA(cudaMemsetAsync(ncand_.p, 0, K * 4, stream_));
        AVN_CUDA(cudaMemsetAsync(nhit_.p, 0, K * 4, stream_));
        uint32_t n_launch = 0;
        if (d.rows > 0) {
            const int g_rows = (d.rows + CCD_BLOCK - 1) / CCD_BLOCK, g_cand = int((cand_cap + CCD_BLOCK - 1) / CCD_BLOCK);
            ccd_candidates_kernel<S><<<g_rows, CCD_BLOCK, 0, stream_>>>(d);
            if (rows.has_hull) ccd_toi_kernel<S, 2><<<g_cand, CCD_BLOCK, 0, stream_>>>(d, table_->dev);
            else if (rows.has_capsule) ccd_toi_kernel<S, 1><<<g_cand, CCD_BLOCK, 0, stream_>>>(d, hm::Table{});
            else ccd_toi_kernel<S, 0><<<g_cand, CCD_BLOCK, 0, stream_>>>(d, hm::Table{});
            ccd_tie_kernel<S><<<g_cand, CCD_BLOCK, 0, stream_>>>(d);
            n_launch += 3;
        }
        ccd_records_kernel<S><<<int((K + CCD_BLOCK - 1) / CCD_BLOCK), CCD_BLOCK, 0, stream_>>>(d);
        ++n_launch;
        // stable LSD radix sort of the 2K records by body: only the digits the body indices use
        const int R = int(2 * K), nblocks = (R + RS_TILE - 1) / RS_TILE;
        int passes = 1;
        while (passes < 4 && (uint64_t(st.B) >> (8 * passes)) != 0) ++passes;
        uint32_t *ka = k0_.as<uint32_t>(), *kb = k1_.as<uint32_t>(), *va = v0_.as<uint32_t>(), *vb = v1_.as<uint32_t>();
        for (int pass = 0; pass < passes; ++pass) {
            rs_histogram<uint32_t><<<nblocks, RS_THREADS, 0, stream_>>>(ka, R, 8 * pass, hist_.as<uint32_t>(), nblocks);
            if (nblocks <= RS_FUSE_MAX_BLOCKS) {
                rs_scatter<uint32_t, true><<<nblocks, RS_THREADS, 0, stream_>>>(ka, va, R, 8 * pass, hist_.as<uint32_t>(), nblocks, kb, vb);
                n_launch += 2;
            } else {
                rs_scan<<<1, 1024, 0, stream_>>>(hist_.as<uint32_t>(), 256 * nblocks);
                rs_scatter<uint32_t, false><<<nblocks, RS_THREADS, 0, stream_>>>(ka, va, R, 8 * pass, hist_.as<uint32_t>(), nblocks, kb, vb);
                n_launch += 3;
            }
            std::swap(ka, kb);
            std::swap(va, vb);
        }
        ccd_apply_kernel<S><<<(R + CCD_BLOCK - 1) / CCD_BLOCK, CCD_BLOCK, 0, stream_>>>(d, ka, va, R);
        ++n_launch;
        AVN_CUDA(cudaGetLastError());
        AVN_CUDA(cudaEventRecord(ev1_, stream_));
        if (launches) *launches += n_launch;
        ran_ = true;
        return AVN_OK;
    }

    AvnStatus download(AvnCcdResult* out) override {
        if (!out) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "ccd: out is required");
        if (!ran_ || K_ == 0) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_ccd_download before a step that ran the CCD pass");
        const size_t K = size_t(K_);
        if (out->min_toi) AVN_CUDA(cudaMemcpyAsync(out->min_toi, out_min_.p, K * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        if (out->hit_body) AVN_CUDA(cudaMemcpyAsync(out->hit_body, out_body_.p, K * 4, cudaMemcpyDeviceToHost, stream_));
        if (out->hit_contact) AVN_CUDA(cudaMemcpyAsync(out->hit_contact, out_contact_.p, K * 4, cudaMemcpyDeviceToHost, stream_));
        if (out->candidates) AVN_CUDA(cudaMemcpyAsync(out->candidates, ncand_.p, K * 4, cudaMemcpyDeviceToHost, stream_));
        if (out->hits) AVN_CUDA(cudaMemcpyAsync(out->hits, nhit_.p, K * 4, cudaMemcpyDeviceToHost, stream_));
        uint32_t total = 0;
        AVN_CUDA(cudaMemcpyAsync(&total, count_.p, 4, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        float ms = 0;
        out->pass_ms = cudaEventElapsedTime(&ms, ev0_, ev1_) == cudaSuccess ? ms : 0.f;
        out->total_candidates = total;
        return AVN_OK;
    }

   private:
    cudaStream_t stream_;
    ErrorSink* err_;
    cudaEvent_t ev0_ = nullptr, ev1_ = nullptr;
    int K_ = 0, n_colliders_ = 0, n_bodies_ = 0;
    double prediction_ = INFINITY;
    bool ran_ = false, capsules_ = false, hulls_flag_ = false;
    const HullTable* table_ = nullptr;
    DevBuf body_, coll_, mode_, inc_, lt_, at_, slot_c_, slot_b_, best_, best_row_, ncand_, nhit_, out_min_, out_body_, out_contact_, m_, k0_, k1_, v0_, v1_,
        hist_, count_, cand_, cand_toi_;
};

}  // namespace

CcdBase* make_ccd(uint32_t scalar_bits, cudaStream_t stream, ErrorSink* err) {
    if (scalar_bits == 32) return new Ccd<float>(stream, err);
    if (scalar_bits == 64) return new Ccd<double>(stream, err);
    return nullptr;
}

}  // namespace avn
