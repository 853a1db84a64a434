// update_aabb on the device for cuboid, sphere, capsule and convex hull colliders.  Replaces update_aabb::<Collider>
// (src/collision/collider/backend.rs:498-625); the shape AABBs follow parry3d's Cuboid::aabb / Ball::aabb / Capsule::aabb
// (center +- |R| half_extents with nalgebra's UnitQuaternion::to_rotation_matrix; center +- radius; capsule_aabb below).
// One thread per collider: 52-68 B in, 24 B out — a pure streaming kernel (HBM-bound, ~90 B per collider).
#include <cmath>
#include <limits>

#include "avn_math.cuh"
#include "context.hpp"

namespace avn {
namespace {

template <class S>
struct AabbArgs {
    int n;
    const uint8_t* shape; const S* dims; const S* pos; const S* rot; const S* lv; const S* av; const S* cm; const S* sm;
    S* omn; S* omx;
    S dt, tol, def_spec, scalar_max;   // scalar_max = Scalar::MAX (what SpeculativeMargin::MAX / SweptCcd stand for)
};

// parry3d's Capsule::aabb: the segment's end points (0, -+half_length, 0) moved by the pose, their componentwise min / max, loosened by the
// radius.  The end points are rotated with nalgebra's UnitQuaternion * Vector3 (t = 2 (q.xyz x v), v + q.xyz x t + t w), not the matrix.
template <class S>
__device__ __noinline__ void capsule_aabb(V3<S> d, V3<S> p, Q4<S> q, V3<S>& mn, V3<S>& mx) {
    const V3<S> b = mk3<S>(q.x, q.y, q.z);
    const V3<S> v0 = mk3<S>(S(0), -d.y, S(0)), v1 = mk3<S>(S(0), d.y, S(0));
    const V3<S> t0 = cross(b, v0) * S(2), t1 = cross(b, v1) * S(2);
    const V3<S> e0 = ((v0 + cross(b, t0)) + t0 * q.w) + p, e1 = ((v1 + cross(b, t1)) + t1 * q.w) + p;
    mn = mk3<S>(avn_min(e0.x, e1.x) - d.x, avn_min(e0.y, e1.y) - d.x, avn_min(e0.z, e1.z) - d.x);
    mx = mk3<S>(avn_max(e0.x, e1.x) + d.x, avn_max(e0.y, e1.y) + d.x, avn_max(e0.z, e1.z) + d.x);
}

template <class S, bool CAPSULES>
__device__ __forceinline__ void shape_aabb(int shape, V3<S> d, V3<S> p, Q4<S> q, V3<S>& mn, V3<S>& mx) {
    if (CAPSULES && shape == AVN_SHAPE_CAPSULE) {
        capsule_aabb<S>(d, p, q, mn, mx);
        return;
    }
    V3<S> he;
    if (shape == AVN_SHAPE_SPHERE) {
        he = mk3<S>(d.x, d.x, d.x);
    } else {
        S i = q.x, j = q.y, k = q.z, w = q.w;
        S ww = w * w, ii = i * i, jj = j * j, kk = k * k;
        S ij = i * j * S(2), wk = w * k * S(2), wj = w * j * S(2), ik = i * k * S(2), jk = j * k * S(2), wi = w * i * S(2);
        S m11 = ww + ii - jj - kk, m12 = ij - wk, m13 = wj + ik;
        S m21 = wk + ij, m22 = ww - ii + jj - kk, m23 = jk - wi;
        S m31 = ik - wj, m32 = wi + jk, m33 = ww - ii - jj + kk;
        he = mk3<S>(avn_abs(m11) * d.x + avn_abs(m12) * d.y + avn_abs(m13) * d.z, avn_abs(m21) * d.x + avn_abs(m22) * d.y + avn_abs(m23) * d.z,
                    avn_abs(m31) * d.x + avn_abs(m32) * d.y + avn_abs(m33) * d.z);
    }
    mn = p - he;
    mx = p + he;
}

// parry3d's ConvexPolyhedron::aabb: every vertex moved by the pose (nalgebra's UnitQuaternion * Vector3, as capsule_aabb), componentwise
// min / max.  PARITY UNPINNED: parry is not vendored.  The table's vertices are the column's values widened to double, so S(v) is exact.
template <class S>
__device__ __noinline__ void hull_aabb(const hm::Table t, uint32_t h, V3<S> p, Q4<S> q, V3<S>& mn, V3<S>& mx) {
    const V3<S> b = mk3<S>(q.x, q.y, q.z);
#pragma unroll 1
    for (uint32_t k = t.voff[h]; k < t.voff[h + 1]; ++k) {
        const V3<S> v = mk3<S>(S(t.vert[3 * k]), S(t.vert[3 * k + 1]), S(t.vert[3 * k + 2]));
        const V3<S> tv = cross(b, v) * S(2);
        const V3<S> e = ((v + cross(b, tv)) + tv * q.w) + p;
        if (k == t.voff[h]) { mn = e; mx = e; continue; }
        mn = mk3<S>(avn_min(mn.x, e.x), avn_min(mn.y, e.y), avn_min(mn.z, e.z));
        mx = mk3<S>(avn_max(mx.x, e.x), avn_max(mx.y, e.y), avn_max(mx.z, e.z));
    }
}

// One thread per collider.  CAPSULES = false (update_aabbs_kernel): cuboids and spheres, skipping the capsules when `capsules` is set and the
// hulls when `hulls` is set; CAPSULES = true (update_capsule_aabbs_kernel, launched only for a shape column that holds a capsule): the capsules
// alone.  The hulls run in update_hull_aabbs_kernel.
template <class S, bool CAPSULES>
__device__ __forceinline__ void update_aabb(const AabbArgs<S>& a, int capsules, int hulls = 0) {
    int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= a.n) return;
    if (hulls && a.shape[n] == AVN_SHAPE_CONVEX_HULL) return;
    if (capsules && (a.shape[n] == AVN_SHAPE_CAPSULE) != CAPSULES) return;
    V3<S> d = mk3<S>(a.dims[3 * n], a.dims[3 * n + 1], a.dims[3 * n + 2]), p = mk3<S>(a.pos[3 * n], a.pos[3 * n + 1], a.pos[3 * n + 2]);
    Q4<S> q; q.x = a.rot[4 * n]; q.y = a.rot[4 * n + 1]; q.z = a.rot[4 * n + 2]; q.w = a.rot[4 * n + 3];
    const int shape = a.shape ? a.shape[n] : AVN_SHAPE_CUBOID;
    S margin = a.cm ? a.cm[n] : S(0);
    S spec = a.sm ? (isinf(a.sm[n]) ? a.scalar_max : a.sm[n]) : a.def_spec;
    V3<S> mn, mx;
    if (spec <= S(0)) {
        shape_aabb<S, CAPSULES>(shape, d, p, q, mn, mx);
    } else {
        V3<S> v = a.lv ? mk3<S>(a.lv[3 * n], a.lv[3 * n + 1], a.lv[3 * n + 2]) : zero3<S>();
        V3<S> w = a.av ? mk3<S>(a.av[3 * n], a.av[3 * n + 1], a.av[3 * n + 2]) : zero3<S>();
        Q4<S> end_rot = q_fast_renormalize(qmul(q_from_scaled_axis(w * a.dt, false), q));
        V3<S> end_pos = p + clamp_len_max(v * a.dt, avn_max(spec, a.tol));
        V3<S> mn0, mx0, mn1, mx1;
        shape_aabb<S, CAPSULES>(shape, d, p, q, mn0, mx0);
        shape_aabb<S, CAPSULES>(shape, d, end_pos, end_rot, mn1, mx1);
        mn = mk3<S>(avn_min(mn0.x, mn1.x), avn_min(mn0.y, mn1.y), avn_min(mn0.z, mn1.z));
        mx = mk3<S>(avn_max(mx0.x, mx1.x), avn_max(mx0.y, mx1.y), avn_max(mx0.z, mx1.z));
    }
    S g = a.tol + margin;
    a.omn[3 * n] = mn.x - g; a.omn[3 * n + 1] = mn.y - g; a.omn[3 * n + 2] = mn.z - g;
    a.omx[3 * n] = mx.x + g; a.omx[3 * n + 1] = mx.y + g; a.omx[3 * n + 2] = mx.z + g;
}

template <class S>
__global__ void update_aabbs_kernel(const __grid_constant__ AabbArgs<S> a, int capsules, int hulls) { update_aabb<S, false>(a, capsules, hulls); }
template <class S>
__global__ void update_capsule_aabbs_kernel(const __grid_constant__ AabbArgs<S> a) { update_aabb<S, true>(a, 1); }

// The hull colliders alone (launched only for a shape column that holds a hull): update_aabb's sweep and margins around hull_aabb.
template <class S>
__global__ void update_hull_aabbs_kernel(const __grid_constant__ AabbArgs<S> a, const hm::Table t) {
    int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= a.n || a.shape[n] != AVN_SHAPE_CONVEX_HULL) return;
    const uint32_t h = uint32_t(a.dims[3 * n]);
    V3<S> p = mk3<S>(a.pos[3 * n], a.pos[3 * n + 1], a.pos[3 * n + 2]);
    Q4<S> q; q.x = a.rot[4 * n]; q.y = a.rot[4 * n + 1]; q.z = a.rot[4 * n + 2]; q.w = a.rot[4 * n + 3];
    S margin = a.cm ? a.cm[n] : S(0);
    S spec = a.sm ? (isinf(a.sm[n]) ? a.scalar_max : a.sm[n]) : a.def_spec;
    V3<S> mn, mx;
    if (spec <= S(0)) {
        hull_aabb<S>(t, h, p, q, mn, mx);
    } else {
        V3<S> v = a.lv ? mk3<S>(a.lv[3 * n], a.lv[3 * n + 1], a.lv[3 * n + 2]) : zero3<S>();
        V3<S> w = a.av ? mk3<S>(a.av[3 * n], a.av[3 * n + 1], a.av[3 * n + 2]) : zero3<S>();
        Q4<S> end_rot = q_fast_renormalize(qmul(q_from_scaled_axis(w * a.dt, false), q));
        V3<S> end_pos = p + clamp_len_max(v * a.dt, avn_max(spec, a.tol));
        V3<S> mn0, mx0, mn1, mx1;
        hull_aabb<S>(t, h, p, q, mn0, mx0);
        hull_aabb<S>(t, h, end_pos, end_rot, mn1, mx1);
        mn = mk3<S>(avn_min(mn0.x, mn1.x), avn_min(mn0.y, mn1.y), avn_min(mn0.z, mn1.z));
        mx = mk3<S>(avn_max(mx0.x, mx1.x), avn_max(mx0.y, mx1.y), avn_max(mx0.z, mx1.z));
    }
    S g = a.tol + margin;
    a.omn[3 * n] = mn.x - g; a.omn[3 * n + 1] = mn.y - g; a.omn[3 * n + 2] = mn.z - g;
    a.omx[3 * n] = mx.x + g; a.omx[3 * n + 1] = mx.y + g; a.omx[3 * n + 2] = mx.z + g;
}

template <class S>
class AabbUpdater final : public AabbBase {
   public:
    AabbUpdater(cudaStream_t stream, ErrorSink* err) : stream_(stream), err_(err) {}
    AvnStatus update(const AvnAabbParams* prm, AvnColliderColumns* c) override {
        if (!prm || !c) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "params and colliders are required");
        const size_t n = c->count;
        if (n == 0) return AVN_OK;
        if (!c->dims || !c->position || !c->rotation || !c->aabb_min || !c->aabb_max)
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "colliders: dims, position, rotation, aabb_min and aabb_max are required");
        size_t at = 0;
        bool capsules = false, hulls = false;
        const uint32_t hull_count = hulls_->count();
        if (const char* why = check_shape_column(c->shape, c->dims, n, sizeof(S) == 8 ? 64 : 32, &at, &capsules, &hull_count, &hulls))
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "colliders: collider %zu: %s", at, why);
        AabbArgs<S> a{};
        a.n = int(n);
        AvnStatus st;
#define UPA(buf, host, cnt, T, dst) if ((st = up<T>(buf, host, cnt, &dst)) != AVN_OK) return st
        UPA(b_shape_, c->shape, n, uint8_t, a.shape);
        UPA(b_dims_, c->dims, 3 * n, S, a.dims);
        UPA(b_pos_, c->position, 3 * n, S, a.pos);
        UPA(b_rot_, c->rotation, 4 * n, S, a.rot);
        UPA(b_lv_, c->linear_velocity, 3 * n, S, a.lv);
        UPA(b_av_, c->angular_velocity, 3 * n, S, a.av);
        UPA(b_cm_, c->collision_margin, n, S, a.cm);
        UPA(b_sm_, c->speculative_margin, n, S, a.sm);
#undef UPA
        AVN_CUDA(o_mn_.ensure(3 * n * sizeof(S)));
        AVN_CUDA(o_mx_.ensure(3 * n * sizeof(S)));
        a.omn = o_mn_.as<S>(); a.omx = o_mx_.as<S>();
        a.dt = S(prm->dt); a.tol = S(prm->contact_tolerance);
        a.scalar_max = std::numeric_limits<S>::max();
        a.def_spec = std::isinf(prm->default_speculative_margin) ? std::numeric_limits<S>::max() : S(prm->default_speculative_margin);
        update_aabbs_kernel<S><<<unsigned((n + 255) / 256), 256, 0, stream_>>>(a, capsules ? 1 : 0, hulls ? 1 : 0);
        if (capsules) update_capsule_aabbs_kernel<S><<<unsigned((n + 255) / 256), 256, 0, stream_>>>(a);
        if (hulls) update_hull_aabbs_kernel<S><<<unsigned((n + 255) / 256), 256, 0, stream_>>>(a, hulls_->dev);
        AVN_CUDA(cudaGetLastError());
        AVN_CUDA(cudaMemcpyAsync(c->aabb_min, a.omn, 3 * n * sizeof(S), cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(c->aabb_max, a.omx, 3 * n * sizeof(S), cudaMemcpyDeviceToHost, stream_));
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
    DevBuf b_shape_, b_dims_, b_pos_, b_rot_, b_lv_, b_av_, b_cm_, b_sm_, o_mn_, o_mx_;
};

}  // namespace

AabbBase* make_aabb_updater(uint32_t scalar_bits, cudaStream_t stream, ErrorSink* err) {
    if (scalar_bits == 32) return new AabbUpdater<float>(stream, err);
    if (scalar_bits == 64) return new AabbUpdater<double>(stream, err);
    return nullptr;
}

}  // namespace avn
