// Contact manifolds for cuboid / sphere / capsule / convex hull pairs on the device (SURVEY.md 8f "next #1", geometry stage).
// Stands where NarrowPhase::update calls contact_manifolds for every contact pair (narrow_phase/system_param.rs:437-830,
// collider/parry/contact_query.rs:156-261).  The arithmetic is csrc/narrow_math.hpp — the same header the host fixture compiles — evaluated
// in double like the fixture and rounded to the column scalar on store, so the device manifolds equal the fixture's bit for bit
// (tests/test_gpu_narrow.py).  One thread per pair: 128 registers and a 1.8 KB local frame for the clipped polygon (ptxas figures in DESIGN.md §7); 2 poses + 2 velocities
// in (≈ 150 B), ≤ 4 points out (≈ 150 B): a streaming kernel, HBM/L2-bound by the gathers of the pose rows.
#include "context.hpp"
#include "contact_rows.hpp"

namespace avn {
namespace {

template <class S>
struct NarrowArgs {
    int n;                                                        // pairs
    const uint32_t* c1; const uint32_t* c2; const uint32_t* b1; const uint32_t* b2;
    const uint8_t* shape; const S* dims; const S* pos; const S* rot;   // collider columns
    const S* lv; const S* av;                                     // body columns
    const S* amin; const S* amax;                                 // collider AABBs (NULL: no disjoint test)
    uint8_t* count; uint8_t* disjoint; S* normal; S* anchor1; S* anchor2; S* penetration; S* normal_speed;
    double dt, tol;
};

template <class S> __device__ __forceinline__ nm::V3 ld3(const S* p, uint32_t i) { return {double(p[3 * i]), double(p[3 * i + 1]), double(p[3 * i + 2])}; }
template <class S> __device__ __forceinline__ void st3(S* p, size_t i, nm::V3 v) { p[3 * i] = S(v.x); p[3 * i + 1] = S(v.y); p[3 * i + 2] = S(v.z); }

// One thread per pair.  CAPSULES = false (narrow_phase_kernel): the cuboid / sphere pairs, and when `capsules` is set the pairs with a
// capsule are skipped; CAPSULES = true (narrow_capsule_kernel, launched only for a shape column that holds a capsule): those pairs alone.
// FRAMES (narrow_framed_kernel, launched instead of the two when body frames are set): anchors relative to the bodies' centres of mass.
// When `hulls` is set those kernels leave every pair with a convex hull to narrow_hull_kernel (HULLS = true, launched only for a shape column
// that holds a hull), which runs hm::collide over the context's hull table `t`.
template <class S, bool CAPSULES, bool FRAMES = false, bool HULLS = false>
__device__ __forceinline__ void narrow_pair(const NarrowArgs<S>& a, int capsules, const BodyFrameCols<S>& f = BodyFrameCols<S>{}, int hulls = 0,
                                            const hm::Table* t = nullptr) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= a.n) return;
    const uint32_t ca = a.c1[k], cb = a.c2[k], ba = a.b1[k], bb = a.b2[k];
    if (HULLS || hulls) {
        if ((a.shape[ca] == hm::SHAPE_CONVEX_HULL || a.shape[cb] == hm::SHAPE_CONVEX_HULL) != HULLS) return;
    }
    if (!HULLS && capsules && (a.shape[ca] == nm::SHAPE_CAPSULE || a.shape[cb] == nm::SHAPE_CAPSULE) != CAPSULES) return;
    a.count[k] = 0;
    if (a.amin) {  // the pair is removed when the AABBs no longer overlap (system_param.rs:437-470)
        const nm::V3 mina = ld3(a.amin, ca), maxa = ld3(a.amax, ca), minb = ld3(a.amin, cb), maxb = ld3(a.amax, cb);
        const bool overlap = !(mina.x > maxb.x || maxa.x < minb.x || mina.y > maxb.y || maxa.y < minb.y || mina.z > maxb.z || maxa.z < minb.z);
        a.disjoint[k] = overlap ? 0 : 1;
        if (!overlap) return;
    } else if (a.disjoint) {
        a.disjoint[k] = 0;
    }
    const nm::V3 pa = ld3(a.pos, ca), pb = ld3(a.pos, cb);
    const nm::Q qa{double(a.rot[4 * ca]), double(a.rot[4 * ca + 1]), double(a.rot[4 * ca + 2]), double(a.rot[4 * ca + 3])};
    const nm::Q qb{double(a.rot[4 * cb]), double(a.rot[4 * cb + 1]), double(a.rot[4 * cb + 2]), double(a.rot[4 * cb + 3])};
    const nm::V3 v1 = ld3(a.lv, ba), v2 = ld3(a.lv, bb), w1 = ld3(a.av, ba), w2 = ld3(a.av, bb);
    const nm::V3 rel = v2 - v1;
    const double eff_margin = a.dt * nm::len(rel);   // effective speculative margin with margin = MAX (system_param.rs:663-681)
    const double max_dist = nm::smax(eff_margin, a.tol);
    nm::V3 normal;
    nm::Contacts pts;
    const int ta = a.shape ? a.shape[ca] : nm::SHAPE_CUBOID, tb = a.shape ? a.shape[cb] : nm::SHAPE_CUBOID;
    if (HULLS ? !hm::collide(*t, ta, ld3(a.dims, ca), pa, qa, tb, ld3(a.dims, cb), pb, qb, max_dist, normal, pts)
              : !nm::collide<CAPSULES>(ta, ld3(a.dims, ca), pa, qa, tb, ld3(a.dims, cb), pb, qb, max_dist, normal, pts))
        return;
    nm::PointOut out[4];
    const int np = FRAMES ? nm::manifold_points(pts, normal, pa, pb, rel, w1, w2, a.dt, eff_margin, pair_frames(f, ba, pa, bb, pb), out)
                          : nm::manifold_points(pts, normal, pa, pb, rel, w1, w2, a.dt, eff_margin, out);
    a.count[k] = uint8_t(np);
    st3(a.normal, k, normal);
    for (int p = 0; p < np; ++p) {
        st3(a.anchor1, size_t(4) * k + p, out[p].anchor1);
        st3(a.anchor2, size_t(4) * k + p, out[p].anchor2);
        a.penetration[size_t(4) * k + p] = S(out[p].penetration);
        a.normal_speed[size_t(4) * k + p] = S(out[p].normal_speed);
    }
}

template <class S>
__global__ void __launch_bounds__(128) narrow_phase_kernel(const __grid_constant__ NarrowArgs<S> a, int capsules, int hulls) {
    narrow_pair<S, false>(a, capsules, BodyFrameCols<S>{}, hulls);
}
template <class S>
__global__ void __launch_bounds__(128) narrow_capsule_kernel(const __grid_constant__ NarrowArgs<S> a, int hulls) {
    narrow_pair<S, true>(a, 1, BodyFrameCols<S>{}, hulls);
}
template <class S, bool CAPSULES>
__global__ void __launch_bounds__(128) narrow_framed_kernel(const __grid_constant__ NarrowArgs<S> a, const BodyFrameCols<S> f, int capsules, int hulls) {
    narrow_pair<S, CAPSULES, true>(a, capsules, f, hulls);
}
template <class S, bool FRAMES>
__global__ void __launch_bounds__(128) narrow_hull_kernel(const __grid_constant__ NarrowArgs<S> a, const BodyFrameCols<S> f, const __grid_constant__ hm::Table t) {
    narrow_pair<S, true, FRAMES, true>(a, 1, f, 1, &t);
}

template <class S>
class Narrow final : public NarrowBase {
   public:
    Narrow(cudaStream_t stream, ErrorSink* err) : stream_(stream), err_(err) {}
    AvnStatus run(const AvnNarrowParams* prm, const AvnNarrowInput* in, AvnRawManifolds* out, const BodyFrames* frames) override {
        if (!prm || !in || !out) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "params, input and output are required");
        const size_t n = in->pair_count, C = in->collider_count, B = in->body_count;
        if (n == 0) return AVN_OK;
        if (!in->collider1 || !in->collider2 || !in->body1 || !in->body2 || !in->dims || !in->position || !in->rotation || !in->linear_velocity ||
            !in->angular_velocity)
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "narrow phase: pair columns, dims, position, rotation and the body velocities are required");
        if (!out->point_count || !out->normal || !out->anchor1 || !out->anchor2 || !out->penetration || !out->normal_speed)
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "narrow phase: every output column except disjoint is required");
        if ((in->aabb_min == nullptr) != (in->aabb_max == nullptr)) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "narrow phase: aabb_min and aabb_max go together");
        if (frames && frames->body_count != B)
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "narrow phase: the body frames have %u bodies, the input %zu", frames->body_count, B);
        for (size_t k = 0; k < n; ++k)
            if (in->collider1[k] >= C || in->collider2[k] >= C || in->body1[k] >= B || in->body2[k] >= B)
                return err_->fail(AVN_ERR_INVALID_ARGUMENT, "narrow phase: pair %zu indexes past the collider / body columns", k);
        size_t at = 0;
        bool capsules = false, hulls = false;
        const uint32_t hull_count = hulls_->count();
        if (const char* why = check_shape_column(in->shape, in->dims, C, sizeof(S) == 8 ? 64 : 32, &at, &capsules, &hull_count, &hulls))
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "narrow phase: collider %zu: %s", at, why);
        NarrowArgs<S> a{};
        a.n = int(n);
        AvnStatus st;
#define UPN(buf, host, cnt, T, dst) if ((st = up<T>(buf, host, cnt, &dst)) != AVN_OK) return st
        UPN(i_c1_, in->collider1, n, uint32_t, a.c1);
        UPN(i_c2_, in->collider2, n, uint32_t, a.c2);
        UPN(i_b1_, in->body1, n, uint32_t, a.b1);
        UPN(i_b2_, in->body2, n, uint32_t, a.b2);
        UPN(i_shape_, in->shape, C, uint8_t, a.shape);
        UPN(i_dims_, in->dims, 3 * C, S, a.dims);
        UPN(i_pos_, in->position, 3 * C, S, a.pos);
        UPN(i_rot_, in->rotation, 4 * C, S, a.rot);
        UPN(i_lv_, in->linear_velocity, 3 * B, S, a.lv);
        UPN(i_av_, in->angular_velocity, 3 * B, S, a.av);
        UPN(i_amin_, in->aabb_min, 3 * C, S, a.amin);
        UPN(i_amax_, in->aabb_max, 3 * C, S, a.amax);
        BodyFrameCols<S> f{};
        if (frames) {
            UPN(i_fpos_, frames->position.data(), 3 * B, S, f.pos);
            UPN(i_frot_, frames->rotation.data(), 4 * B, S, f.rot);
            if (!frames->com.empty()) UPN(i_fcom_, frames->com.data(), 3 * B, S, f.com);
        }
#undef UPN
        AVN_CUDA(o_cnt_.ensure(n));
        AVN_CUDA(o_dis_.ensure(n));
        AVN_CUDA(o_nrm_.ensure(3 * n * sizeof(S)));
        AVN_CUDA(o_a1_.ensure(12 * n * sizeof(S)));
        AVN_CUDA(o_a2_.ensure(12 * n * sizeof(S)));
        AVN_CUDA(o_pen_.ensure(4 * n * sizeof(S)));
        AVN_CUDA(o_ns_.ensure(4 * n * sizeof(S)));
        a.count = o_cnt_.as<uint8_t>(); a.disjoint = o_dis_.as<uint8_t>(); a.normal = o_nrm_.as<S>(); a.anchor1 = o_a1_.as<S>(); a.anchor2 = o_a2_.as<S>();
        a.penetration = o_pen_.as<S>(); a.normal_speed = o_ns_.as<S>();
        a.dt = prm->dt;
        a.tol = prm->contact_tolerance;
        // unwritten point slots read as zero on the host
        AVN_CUDA(cudaMemsetAsync(a.normal, 0, 3 * n * sizeof(S), stream_));
        AVN_CUDA(cudaMemsetAsync(a.anchor1, 0, 12 * n * sizeof(S), stream_));
        AVN_CUDA(cudaMemsetAsync(a.anchor2, 0, 12 * n * sizeof(S), stream_));
        AVN_CUDA(cudaMemsetAsync(a.penetration, 0, 4 * n * sizeof(S), stream_));
        AVN_CUDA(cudaMemsetAsync(a.normal_speed, 0, 4 * n * sizeof(S), stream_));
        const int h = hulls ? 1 : 0;
        if (frames) {
            narrow_framed_kernel<S, false><<<unsigned((n + 127) / 128), 128, 0, stream_>>>(a, f, capsules ? 1 : 0, h);
            if (capsules) narrow_framed_kernel<S, true><<<unsigned((n + 127) / 128), 128, 0, stream_>>>(a, f, 1, h);
            if (hulls) narrow_hull_kernel<S, true><<<unsigned((n + 127) / 128), 128, 0, stream_>>>(a, f, hulls_->dev);
        } else {
            narrow_phase_kernel<S><<<unsigned((n + 127) / 128), 128, 0, stream_>>>(a, capsules ? 1 : 0, h);
            if (capsules) narrow_capsule_kernel<S><<<unsigned((n + 127) / 128), 128, 0, stream_>>>(a, h);
            if (hulls) narrow_hull_kernel<S, false><<<unsigned((n + 127) / 128), 128, 0, stream_>>>(a, f, hulls_->dev);
        }
        AVN_CUDA(cudaGetLastError());
        AVN_CUDA(cudaMemcpyAsync(out->point_count, a.count, n, cudaMemcpyDeviceToHost, stream_));
        if (out->disjoint) AVN_CUDA(cudaMemcpyAsync(out->disjoint, a.disjoint, n, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(out->normal, a.normal, 3 * n * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(out->anchor1, a.anchor1, 12 * n * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(out->anchor2, a.anchor2, 12 * n * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(out->penetration, a.penetration, 4 * n * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(out->normal_speed, a.normal_speed, 4 * n * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaStreamSynchronize(stream_));
        return AVN_OK;
    }
    void attach_hulls(const HullTable* hulls) override { hulls_ = hulls; }

   private:
    template <class T> AvnStatus up(DevBuf& buf, const void* host, size_t count, const T** dev) {
        *dev = nullptr;
        if (!host || count == 0) return AVN_OK;
        AVN_CUDA(buf.ensure(count * sizeof(T)));
        AVN_CUDA(cudaMemcpyAsync(buf.p, host, count * sizeof(T), cudaMemcpyHostToDevice, stream_));
        *dev = buf.as<T>();
        return AVN_OK;
    }
    cudaStream_t stream_;
    ErrorSink* err_;
    const HullTable* hulls_ = nullptr;
    DevBuf i_c1_, i_c2_, i_b1_, i_b2_, i_shape_, i_dims_, i_pos_, i_rot_, i_lv_, i_av_, i_amin_, i_amax_, i_fpos_, i_frot_, i_fcom_;
    DevBuf o_cnt_, o_dis_, o_nrm_, o_a1_, o_a2_, o_pen_, o_ns_;
};

}  // namespace

NarrowBase* make_narrow(uint32_t scalar_bits, cudaStream_t stream, ErrorSink* err) {
    if (scalar_bits == 32) return new Narrow<float>(stream, err);
    if (scalar_bits == 64) return new Narrow<double>(stream, err);
    return nullptr;
}

}  // namespace avn
