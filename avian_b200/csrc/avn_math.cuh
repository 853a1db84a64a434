// Device math for the avian_b200 kernels (sm_90a).
//
// Every routine evaluates the same floating-point expression tree as the glam / glam_matrix_extras routine
// the reference calls at that point (the call sites are cited next to each function), because the parity bar
// is 1e-5 relative on chaotic contact dynamics: the library is compiled with -fmad=false and IEEE div/sqrt so
// that the only source of difference from a CPU evaluation is sin/cos/asin, and sin/cos are by default taken
// in double and rounded (see AVN_CFG_FAST_TRIG).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace avn {

template <class S> struct Vec4;  // 16/32-byte aligned 4-vector: the unit of every HBM load/store
template <> struct __align__(16) Vec4<float> { float x, y, z, w; };
template <> struct __align__(32) Vec4<double> { double x, y, z, w; };

template <class S> struct V3 { S x, y, z; };
template <class S> struct V2 { S x, y; };
template <class S> struct Q4 { S x, y, z, w; };
template <class S> struct Sym3 { S m00, m01, m02, m11, m12, m22; };
template <class S> struct M33 { V3<S> c0, c1, c2; };

#define AVN_HD __host__ __device__ __forceinline__

template <class S> AVN_HD V3<S> mk3(S x, S y, S z) { V3<S> r; r.x = x; r.y = y; r.z = z; return r; }
template <class S> AVN_HD V3<S> zero3() { return mk3<S>(S(0), S(0), S(0)); }
template <class S> AVN_HD V3<S> operator+(V3<S> a, V3<S> b) { return mk3<S>(a.x + b.x, a.y + b.y, a.z + b.z); }
template <class S> AVN_HD V3<S> operator-(V3<S> a, V3<S> b) { return mk3<S>(a.x - b.x, a.y - b.y, a.z - b.z); }
template <class S> AVN_HD V3<S> operator-(V3<S> a) { return mk3<S>(-a.x, -a.y, -a.z); }
template <class S> AVN_HD V3<S> operator*(V3<S> a, S s) { return mk3<S>(a.x * s, a.y * s, a.z * s); }
template <class S> AVN_HD V3<S> operator*(S s, V3<S> a) { return mk3<S>(s * a.x, s * a.y, s * a.z); }
template <class S> AVN_HD V3<S> cmul(V3<S> a, V3<S> b) { return mk3<S>(a.x * b.x, a.y * b.y, a.z * b.z); }
template <class S> AVN_HD V3<S> operator/(V3<S> a, S s) { return mk3<S>(a.x / s, a.y / s, a.z / s); }
// Vec3::dot — (x*x + y*y) + z*z
template <class S> AVN_HD S dot(V3<S> a, V3<S> b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
// Vec3::cross
template <class S> AVN_HD V3<S> cross(V3<S> a, V3<S> b) {
    return mk3<S>(a.y * b.z - b.y * a.z, a.z * b.x - b.z * a.x, a.x * b.y - b.x * a.y);
}
template <class S> AVN_HD S len2(V3<S> a) { return dot(a, a); }

AVN_HD float avn_sqrt(float x) { return sqrtf(x); }
AVN_HD double avn_sqrt(double x) { return sqrt(x); }
AVN_HD float avn_abs(float x) { return fabsf(x); }
AVN_HD double avn_abs(double x) { return fabs(x); }
AVN_HD float avn_max(float a, float b) { return fmaxf(a, b); }
AVN_HD double avn_max(double a, double b) { return fmax(a, b); }
AVN_HD float avn_min(float a, float b) { return fminf(a, b); }
AVN_HD double avn_min(double a, double b) { return fmin(a, b); }
AVN_HD bool avn_finite(float x) { return isfinite(x); }
AVN_HD bool avn_finite(double x) { return isfinite(x); }
template <class S> struct Eps;
template <> struct Eps<float> { static constexpr float v = 1.1920929e-7f; };
template <> struct Eps<double> { static constexpr double v = 2.220446049250313e-16; };

template <class S> AVN_HD S len(V3<S> a) { return avn_sqrt(dot(a, a)); }
template <class S> AVN_HD S max_elem(V3<S> a) { return avn_max(a.x, avn_max(a.y, a.z)); }
// src/math/mod.rs:244-262
template <class S> AVN_HD S recip_or_zero(S s) { return (s != S(0) && avn_finite(s)) ? S(1) / s : S(0); }

// sin/cos of a half angle.  f32 default: evaluate in double and round once, which equals a correctly rounded
// sinf/cosf except in astronomically rare double-rounding ties; AVN_CFG_FAST_TRIG uses sincosf.
__device__ __forceinline__ void avn_sincos(float a, float& s, float& c, bool fast) {
    if (fast) {
        sincosf(a, &s, &c);
    } else {
        double ds, dc;
        sincos((double)a, &ds, &dc);
        s = (float)ds;
        c = (float)dc;
    }
}
__device__ __forceinline__ void avn_sincos(double a, double& s, double& c, bool) { sincos(a, &s, &c); }
__device__ __forceinline__ float avn_asin(float x) { return (float)asin((double)x); }
__device__ __forceinline__ double avn_asin(double x) { return asin(x); }

template <class S> AVN_HD Q4<S> qidentity() { Q4<S> q; q.x = S(0); q.y = S(0); q.z = S(0); q.w = S(1); return q; }
template <class S> AVN_HD Q4<S> qconj(Q4<S> q) { Q4<S> r; r.x = -q.x; r.y = -q.y; r.z = -q.z; r.w = q.w; return r; }
template <class S> AVN_HD V3<S> qxyz(Q4<S> q) { return mk3<S>(q.x, q.y, q.z); }

// Quat::mul_quat.  f32 follows glam's SSE2 lane association, f64 the scalar left-to-right one.
AVN_HD Q4<float> qmul(Q4<float> a, Q4<float> b) {
    Q4<float> r;
    r.x = (a.w * b.x + a.x * b.w) + (a.y * b.z - a.z * b.y);
    r.y = (a.w * b.y - a.x * b.z) + (a.y * b.w + a.z * b.x);
    r.z = (a.w * b.z + a.x * b.y) + (a.z * b.w - a.y * b.x);
    r.w = (a.w * b.w - a.x * b.x) + (-(a.y * b.y) - a.z * b.z);
    return r;
}
AVN_HD Q4<double> qmul(Q4<double> a, Q4<double> b) {
    Q4<double> r;
    r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
    r.y = a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x;
    r.z = a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w;
    r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
    return r;
}
// Quat * Vec3: v*(w*w - b.b) + b*((v.b)*2) + (b x v)*(w*2)
template <class S> AVN_HD V3<S> qrot(Q4<S> q, V3<S> v) {
    V3<S> b = mk3<S>(q.x, q.y, q.z);
    S b2 = dot(b, b);
    return (v * (q.w * q.w - b2) + b * (dot(v, b) * S(2))) + cross(b, v) * (q.w * S(2));
}
template <class S> __device__ __forceinline__ Q4<S> q_from_axis_angle(V3<S> axis, S angle, bool fast) {
    S s, c;
    avn_sincos(angle * S(0.5), s, c, fast);
    Q4<S> q;
    q.x = axis.x * s; q.y = axis.y * s; q.z = axis.z * s; q.w = c;
    return q;
}
// Quat::from_scaled_axis (integrator/mod.rs:529-530, positional_constraint.rs:92, angular_constraint.rs:279)
template <class S> __device__ __forceinline__ Q4<S> q_from_scaled_axis(V3<S> v, bool fast) {
    S l = len(v);
    if (l == S(0)) return qidentity<S>();
    return q_from_axis_angle(v / l, l, fast);
}
// Rotation::fast_renormalize (physics_transform/transform.rs:811-817)
template <class S> AVN_HD Q4<S> q_fast_renormalize(Q4<S> q) {
    S l2 = ((q.x * q.x + q.y * q.y) + q.z * q.z) + q.w * q.w;
    S k = S(0.5) * (S(3) - l2);
    Q4<S> r; r.x = q.x * k; r.y = q.y * k; r.z = q.z * k; r.w = q.w * k;
    return r;
}

// Mat3::from_quat / Mat3 * Vec3 / Mat3 * Mat3 (computed.rs:663-668, spherical.rs:66-81)
template <class S> AVN_HD M33<S> m33_from_quat(Q4<S> r) {
    S x2 = r.x + r.x, y2 = r.y + r.y, z2 = r.z + r.z;
    S xx = r.x * x2, xy = r.x * y2, xz = r.x * z2, yy = r.y * y2, yz = r.y * z2, zz = r.z * z2;
    S wx = r.w * x2, wy = r.w * y2, wz = r.w * z2;
    M33<S> m;
    m.c0 = mk3<S>(S(1) - (yy + zz), xy + wz, xz - wy);
    m.c1 = mk3<S>(xy - wz, S(1) - (xx + zz), yz + wx);
    m.c2 = mk3<S>(xz + wy, yz - wx, S(1) - (xx + yy));
    return m;
}
template <class S> AVN_HD V3<S> mmul(const M33<S>& m, V3<S> v) { return (m.c0 * v.x + m.c1 * v.y) + m.c2 * v.z; }
// SymmetricMat3 * Vec3
template <class S> AVN_HD V3<S> smul(const Sym3<S>& s, V3<S> v) {
    return mk3<S>((s.m00 * v.x + s.m01 * v.y) + s.m02 * v.z, (s.m01 * v.x + s.m11 * v.y) + s.m12 * v.z,
                  (s.m02 * v.x + s.m12 * v.y) + s.m22 * v.z);
}
// ComputedAngularInertia::rotated(q).inverse(): from_mat3_unchecked((R * I) * R^T)
template <class S> AVN_HD Sym3<S> rotate_inv_inertia(const Sym3<S>& il, Q4<S> q) {
    M33<S> r = m33_from_quat(q);
    M33<S> ri;
    ri.c0 = mmul(r, mk3<S>(il.m00, il.m01, il.m02));
    ri.c1 = mmul(r, mk3<S>(il.m01, il.m11, il.m12));
    ri.c2 = mmul(r, mk3<S>(il.m02, il.m12, il.m22));
    // columns of R^T are the rows of R; only the 6 kept entries are evaluated
    V3<S> t0 = mk3<S>(r.c0.x, r.c1.x, r.c2.x), t1 = mk3<S>(r.c0.y, r.c1.y, r.c2.y), t2 = mk3<S>(r.c0.z, r.c1.z, r.c2.z);
    V3<S> o0 = mmul(ri, t0), o1 = mmul(ri, t1), o2 = mmul(ri, t2);
    Sym3<S> s;
    s.m00 = o0.x; s.m01 = o0.y; s.m02 = o0.z; s.m11 = o1.y; s.m12 = o1.z; s.m22 = o2.z;
    return s;
}
// SymmetricMat3::inverse_or_zero (math/mod.rs:515-524), cofactor form
template <class S> AVN_HD Sym3<S> sym_inverse_or_zero(const Sym3<S>& s) {
    S c00 = s.m11 * s.m22 - s.m12 * s.m12, c01 = s.m02 * s.m12 - s.m01 * s.m22, c02 = s.m01 * s.m12 - s.m02 * s.m11;
    S det = (s.m00 * c00 + s.m01 * c01) + s.m02 * c02;
    Sym3<S> r;
    if (det == S(0)) { r.m00 = r.m01 = r.m02 = r.m11 = r.m12 = r.m22 = S(0); return r; }
    S inv = S(1) / det;
    S c11 = s.m00 * s.m22 - s.m02 * s.m02, c12 = s.m01 * s.m02 - s.m00 * s.m12, c22 = s.m00 * s.m11 - s.m01 * s.m01;
    r.m00 = c00 * inv; r.m01 = c01 * inv; r.m02 = c02 * inv; r.m11 = c11 * inv; r.m12 = c12 * inv; r.m22 = c22 * inv;
    return r;
}
// Vec3::any_orthonormal_vector (contact/mod.rs:443-446, revolute.rs:86-88, spherical.rs:77)
template <class S> AVN_HD V3<S> any_orthonormal(V3<S> a) {
    S sign = signbit(a.z) ? S(-1) : S(1);
    S k = S(-1) / (sign + a.z);
    S b = a.x * a.y * k;
    return mk3<S>(b, sign + a.y * a.y * k, -a.y);
}
// Vec3::any_orthogonal_vector (prismatic.rs:131)
template <class S> AVN_HD V3<S> any_orthogonal(V3<S> a) {
    if (avn_abs(a.x) > avn_abs(a.y)) return mk3<S>(-a.z, S(0), a.x);
    return mk3<S>(S(0), a.z, -a.y);
}
template <class S> AVN_HD V3<S> clamp_len_max(V3<S> a, S m) {
    S l2 = len2(a);
    if (l2 > m * m) return m * (a / avn_sqrt(l2));
    return a;
}

// ---- 128-bit (f32) / 2x128-bit (f64) global accessors ----------------------------------------------------
template <class S> __device__ __forceinline__ Vec4<S> ld4(const Vec4<S>* p) { return *p; }
template <class S> __device__ __forceinline__ void st4(Vec4<S>* p, Vec4<S> v) { *p = v; }
template <class S> AVN_HD Vec4<S> mk4(S x, S y, S z, S w) { Vec4<S> r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }
template <class S> AVN_HD V3<S> xyz(Vec4<S> v) { return mk3<S>(v.x, v.y, v.z); }

// integer payloads travel in the scalar lanes of a Vec4 plane, bit-cast
__device__ __forceinline__ int as_int(float f) { return __float_as_int(f); }
__device__ __forceinline__ int as_int(double f) { return (int)__double_as_longlong(f); }
__device__ __forceinline__ float int_as(float, int i) { return __int_as_float(i); }
__device__ __forceinline__ double int_as(double, int i) { return __longlong_as_double((long long)i); }

}  // namespace avn
