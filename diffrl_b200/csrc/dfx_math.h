// dfx_math.h -- small fixed-size algebra for the articulated rigid-body step, with the
// hand-derived adjoint of every operation.
//
// Conventions are the data ABI of the reference (NVlabs/DiffRL, dflex/dflex/*.h), restated:
//   quaternion      (x, y, z, w), imaginary part first            reference quat.h:3-13
//   transform       p(3) then q(4)                                reference spatial.h:166-173
//   spatial vector  angular (w) then linear (v)                   reference spatial.h:6-13
//   rotate(q, x) is the degree-2 polynomial  x(2w^2-1) + 2w(v x x) + 2v(v.x)   (quat.h:113-116);
//   it is differentiated as that polynomial in all four components of q (quat.h:256-288), i.e.
//   q is NOT assumed to be unit length when taking derivatives.
//
// Everything is plain fp32 inline code usable from device code and (for the CPU-side unit tests
// of the adjoints) from host code.  No reference source is reproduced here: adjoints are written
// from the mathematics of each operation.
#pragma once

#include <math.h>

#if defined(__CUDACC__)
#define DFX_HD __host__ __device__ __forceinline__
#else
#define DFX_HD inline
#endif

namespace dfx {

struct V3 {
    float x, y, z;
};
struct Q4 {
    float x, y, z, w;
};
struct Xf {  // rigid transform
    V3 p;
    Q4 q;
};
struct SV {  // spatial vector: angular part w, linear part v
    V3 w, v;
};
struct M3 {  // row-major 3x3
    float m[3][3];
};

// ---------------------------------------------------------------- V3
DFX_HD V3 v3(float x, float y, float z) { return V3{x, y, z}; }
DFX_HD V3 v3zero() { return V3{0.f, 0.f, 0.f}; }
DFX_HD V3 operator+(V3 a, V3 b) { return V3{a.x + b.x, a.y + b.y, a.z + b.z}; }
DFX_HD V3 operator-(V3 a, V3 b) { return V3{a.x - b.x, a.y - b.y, a.z - b.z}; }
DFX_HD V3 operator-(V3 a) { return V3{-a.x, -a.y, -a.z}; }
DFX_HD V3 operator*(V3 a, float s) { return V3{a.x * s, a.y * s, a.z * s}; }
DFX_HD V3& operator+=(V3& a, V3 b) {
    a.x += b.x; a.y += b.y; a.z += b.z;
    return a;
}
DFX_HD V3& operator-=(V3& a, V3 b) {
    a.x -= b.x; a.y -= b.y; a.z -= b.z;
    return a;
}
DFX_HD float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
DFX_HD V3 cross(V3 a, V3 b) {
    return V3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
// c = a x b ; given dL/dc = r:  dL/da = b x r ,  dL/db = r x a
DFX_HD void cross_adj(V3 a, V3 b, V3 r, V3& aa, V3& ab) {
    aa += cross(b, r);
    ab += cross(r, a);
}
DFX_HD float get(const V3& a, int i) { return i == 0 ? a.x : (i == 1 ? a.y : a.z); }

// ---------------------------------------------------------------- Q4
DFX_HD Q4 q4(float x, float y, float z, float w) { return Q4{x, y, z, w}; }
DFX_HD Q4 qident() { return Q4{0.f, 0.f, 0.f, 1.f}; }
DFX_HD Q4 qzero() { return Q4{0.f, 0.f, 0.f, 0.f}; }
DFX_HD V3 qv(Q4 q) { return V3{q.x, q.y, q.z}; }
DFX_HD Q4 operator+(Q4 a, Q4 b) { return Q4{a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w}; }
DFX_HD Q4 operator*(Q4 a, float s) { return Q4{a.x * s, a.y * s, a.z * s, a.w * s}; }
DFX_HD Q4& operator+=(Q4& a, Q4 b) {
    a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    return a;
}
DFX_HD float qdot(Q4 a, Q4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }

// Hamilton product (reference quat.h:100-106)
DFX_HD Q4 qmul(Q4 a, Q4 b) {
    return Q4{a.w * b.x + b.w * a.x + a.y * b.z - b.y * a.z,
              a.w * b.y + b.w * a.y + a.z * b.x - b.z * a.x,
              a.w * b.z + b.w * a.z + a.x * b.y - b.x * a.y,
              a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}
// c = a*b is bilinear:  dL/da = r * conj(b) ,  dL/db = conj(a) * r   (as 4-vectors)
DFX_HD void qmul_adj(Q4 a, Q4 b, Q4 r, Q4& aa, Q4& ab) {
    aa += qmul(r, Q4{-b.x, -b.y, -b.z, b.w});
    ab += qmul(Q4{-a.x, -a.y, -a.z, a.w}, r);
}
// only the adjoint w.r.t. the first / second factor
DFX_HD Q4 qmul_adj_a(Q4 b, Q4 r) { return qmul(r, Q4{-b.x, -b.y, -b.z, b.w}); }
DFX_HD Q4 qmul_adj_b(Q4 a, Q4 r) { return qmul(Q4{-a.x, -a.y, -a.z, a.w}, r); }

// rotate(q, x) = R(q) x  with the polynomial R(q) = (2w^2-1) I + 2w [v]x + 2 v v^T
DFX_HD V3 qrot(Q4 q, V3 x) {
    V3 v = qv(q);
    return x * (2.0f * q.w * q.w - 1.0f) + cross(v, x) * q.w * 2.0f + v * dot(v, x) * 2.0f;
}
// R(q)^T x  (== rotate(inverse(q), x) of the reference)
DFX_HD V3 qrot_inv(Q4 q, V3 x) {
    V3 v = qv(q);
    return x * (2.0f * q.w * q.w - 1.0f) - cross(v, x) * q.w * 2.0f + v * dot(v, x) * 2.0f;
}
// y = R(q) x, dL/dy = r:  dL/dx = R^T r ; dL/dq from the polynomial
DFX_HD Q4 qrot_adj_q(Q4 q, V3 x, V3 r) {
    V3 v = qv(q);
    V3 av = cross(x, r) * (2.0f * q.w) + r * (2.0f * dot(v, x)) + x * (2.0f * dot(v, r));
    float aw = 4.0f * q.w * dot(r, x) + 2.0f * dot(r, cross(v, x));
    return Q4{av.x, av.y, av.z, aw};
}
// y = R(q)^T x
DFX_HD Q4 qrot_inv_adj_q(Q4 q, V3 x, V3 r) {
    V3 v = qv(q);
    V3 av = cross(r, x) * (2.0f * q.w) + r * (2.0f * dot(v, x)) + x * (2.0f * dot(v, r));
    float aw = 4.0f * q.w * dot(r, x) - 2.0f * dot(r, cross(v, x));
    return Q4{av.x, av.y, av.z, aw};
}

DFX_HD Q4 q_from_axis_angle(V3 axis, float angle) {
    float h = angle * 0.5f;
    float s = sinf(h), c = cosf(h);
    return Q4{axis.x * s, axis.y * s, axis.z * s, c};
}
// d/dangle only (the axis is a model constant)
DFX_HD float q_from_axis_angle_adj_angle(V3 axis, float angle, Q4 r) {
    float h = angle * 0.5f;
    float s = sinf(h), c = cosf(h);
    return 0.5f * (c * (axis.x * r.x + axis.y * r.y + axis.z * r.z) - s * r.w);
}

// normalize with the reference's conventions: |q| == 0 -> identity, zero gradient (quat.h:70-83,182-192)
DFX_HD Q4 qnormalize(Q4 q) {
    float l = sqrtf(qdot(q, q));
    if (l > 0.0f) {
        float inv = 1.0f / l;
        return Q4{q.x * inv, q.y * inv, q.z * inv, q.w * inv};
    }
    return qident();
}
DFX_HD Q4 qnormalize_adj(Q4 q, Q4 r) {
    float l = sqrtf(qdot(q, q));
    if (l > 0.0f) {
        float inv = 1.0f / l;
        float k = inv * inv * inv * qdot(q, r);
        return Q4{r.x * inv - q.x * k, r.y * inv - q.y * k, r.z * inv - q.z * k, r.w * inv - q.w * k};
    }
    return qzero();
}

// ---------------------------------------------------------------- Xf
DFX_HD Xf xf_ident() { return Xf{v3zero(), qident()}; }
DFX_HD Xf xf_zero() { return Xf{v3zero(), qzero()}; }
DFX_HD Xf xf_mul(Xf a, Xf b) { return Xf{qrot(a.q, b.p) + a.p, qmul(a.q, b.q)}; }
DFX_HD V3 xf_point(Xf t, V3 x) { return t.p + qrot(t.q, x); }
// xf_mul with every rounding spelled out as fmaf chains, for the joint-local transforms (dfx_phases.h kin_local_fwd).  Those are
// formed in two places -- phase K1 and, with kFusedPhases, inside integrate_fwd -- that are inlined into different kernels (the
// tape forward, the recompute adjoint).  Left to the compiler, the FMA contraction of qmul / qrot differs between those
// contexts, and a recomputed tape row would differ from the stored one in the last bits wherever X_pj is not axis-aligned.
DFX_HD Q4 qmul_rn(Q4 a, Q4 b) {
    return Q4{fmaf(a.w, b.x, fmaf(b.w, a.x, fmaf(a.y, b.z, -(b.y * a.z)))),
              fmaf(a.w, b.y, fmaf(b.w, a.y, fmaf(a.z, b.x, -(b.z * a.x)))),
              fmaf(a.w, b.z, fmaf(b.w, a.z, fmaf(a.x, b.y, -(b.x * a.y)))),
              fmaf(a.w, b.w, -fmaf(a.x, b.x, fmaf(a.y, b.y, a.z * b.z)))};
}
DFX_HD V3 qrot_rn(Q4 q, V3 x) {
    const float k = fmaf(2.0f * q.w, q.w, -1.0f), w2 = 2.0f * q.w;
    const float d2 = 2.0f * fmaf(q.x, x.x, fmaf(q.y, x.y, q.z * x.z));
    const V3 c{fmaf(q.y, x.z, -(q.z * x.y)), fmaf(q.z, x.x, -(q.x * x.z)), fmaf(q.x, x.y, -(q.y * x.x))};
    return V3{fmaf(x.x, k, fmaf(c.x, w2, q.x * d2)), fmaf(x.y, k, fmaf(c.y, w2, q.y * d2)), fmaf(x.z, k, fmaf(c.z, w2, q.z * d2))};
}
DFX_HD Xf xf_mul_rn(Xf a, Xf b) {
    const V3 r = qrot_rn(a.q, b.p);
    return Xf{V3{r.x + a.p.x, r.y + a.p.y, r.z + a.p.z}, qmul_rn(a.q, b.q)};
}
// c = a*b, dL/dc = r -> accumulate into aa, ab
DFX_HD void xf_mul_adj(Xf a, Xf b, Xf r, Xf& aa, Xf& ab) {
    aa.p += r.p;
    aa.q += qrot_adj_q(a.q, b.p, r.p);
    ab.p += qrot_inv(a.q, r.p);
    aa.q += qmul_adj_a(b.q, r.q);
    ab.q += qmul_adj_b(a.q, r.q);
}
DFX_HD void xf_mul_adj_a(Xf a, Xf b, Xf r, Xf& aa) {
    aa.p += r.p;
    aa.q += qrot_adj_q(a.q, b.p, r.p);
    aa.q += qmul_adj_a(b.q, r.q);
}
// adjoint w.r.t. the second factor only
DFX_HD Xf xf_mul_adj_b(Xf a, Xf r) { return Xf{qrot_inv(a.q, r.p), qmul_adj_b(a.q, r.q)}; }
DFX_HD Xf& operator+=(Xf& a, Xf b) {
    a.p += b.p;
    a.q += b.q;
    return a;
}

// ---------------------------------------------------------------- SV
DFX_HD SV sv_zero() { return SV{v3zero(), v3zero()}; }
DFX_HD SV operator+(SV a, SV b) { return SV{a.w + b.w, a.v + b.v}; }
DFX_HD SV operator-(SV a, SV b) { return SV{a.w - b.w, a.v - b.v}; }
DFX_HD SV operator*(SV a, float s) { return SV{a.w * s, a.v * s}; }
DFX_HD SV& operator+=(SV& a, SV b) {
    a.w += b.w;
    a.v += b.v;
    return a;
}
DFX_HD float sv_dot(SV a, SV b) { return dot(a.w, b.w) + dot(a.v, b.v); }
// motion cross product  [a]x b  (reference spatial.h:56-62)
DFX_HD SV sv_cross(SV a, SV b) { return SV{cross(a.w, b.w), cross(a.v, b.w) + cross(a.w, b.v)}; }
DFX_HD void sv_cross_adj(SV a, SV b, SV r, SV& aa, SV& ab) {
    cross_adj(a.w, b.w, r.w, aa.w, ab.w);
    cross_adj(a.v, b.w, r.v, aa.v, ab.w);
    cross_adj(a.w, b.v, r.v, aa.w, ab.v);
}
// "dual" cross product without the sign flip (reference spatial.h:64-70)
DFX_HD SV sv_cross_dual(SV a, SV b) { return SV{cross(a.w, b.w) + cross(a.v, b.v), cross(a.w, b.v)}; }
DFX_HD void sv_cross_dual_adj(SV a, SV b, SV r, SV& aa, SV& ab) {
    cross_adj(a.w, b.w, r.w, aa.w, ab.w);
    cross_adj(a.v, b.v, r.w, aa.v, ab.v);
    cross_adj(a.w, b.v, r.v, aa.w, ab.v);
}
// change of frame of a twist: (R w, R v + p x R w)   (reference sim.py:1076-1088)
DFX_HD SV xf_twist(Xf t, SV x) {
    V3 w = qrot(t.q, x.w);
    V3 v = qrot(t.q, x.v) + cross(t.p, w);
    return SV{w, v};
}
// adjoint w.r.t. the transform only (x is a model constant on this path)
DFX_HD void xf_twist_adj_t(Xf t, SV x, SV r, Xf& at) {
    V3 w = qrot(t.q, x.w);
    // v = R xv + p x w
    V3 aw = r.w;
    at.q += qrot_adj_q(t.q, x.v, r.v);
    at.p += cross(w, r.v);      // d(p x w)/dp
    aw += cross(r.v, t.p);      // d(p x w)/dw
    at.q += qrot_adj_q(t.q, x.w, aw);
}

// ---------------------------------------------------------------- M3
DFX_HD M3 m3_zero() {
    M3 r;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r.m[i][j] = 0.f;
    return r;
}
DFX_HD V3 m3_mul(const M3& a, V3 x) {
    return V3{a.m[0][0] * x.x + a.m[0][1] * x.y + a.m[0][2] * x.z,
              a.m[1][0] * x.x + a.m[1][1] * x.y + a.m[1][2] * x.z,
              a.m[2][0] * x.x + a.m[2][1] * x.y + a.m[2][2] * x.z};
}
DFX_HD V3 m3_tmul(const M3& a, V3 x) {  // a^T x
    return V3{a.m[0][0] * x.x + a.m[1][0] * x.y + a.m[2][0] * x.z,
              a.m[0][1] * x.x + a.m[1][1] * x.y + a.m[2][1] * x.z,
              a.m[0][2] * x.x + a.m[1][2] * x.y + a.m[2][2] * x.z};
}
DFX_HD M3 m3_mm(const M3& a, const M3& b) {
    M3 r;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            r.m[i][j] = a.m[i][0] * b.m[0][j] + a.m[i][1] * b.m[1][j] + a.m[i][2] * b.m[2][j];
    return r;
}
DFX_HD M3 m3_mmt(const M3& a, const M3& b) {  // a b^T
    M3 r;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            r.m[i][j] = a.m[i][0] * b.m[j][0] + a.m[i][1] * b.m[j][1] + a.m[i][2] * b.m[j][2];
    return r;
}
DFX_HD M3 m3_tmm(const M3& a, const M3& b) {  // a^T b
    M3 r;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            r.m[i][j] = a.m[0][i] * b.m[0][j] + a.m[1][i] * b.m[1][j] + a.m[2][i] * b.m[2][j];
    return r;
}
// polynomial rotation matrix R(q) = (2w^2-1) I + 2w [v]x + 2 v v^T  (columns = rotate(q, e_k))
DFX_HD M3 q_to_m3(Q4 q) {
    float d = 2.0f * q.w * q.w - 1.0f;
    float tw = 2.0f * q.w;
    M3 r;
    r.m[0][0] = d + 2.0f * q.x * q.x;
    r.m[1][1] = d + 2.0f * q.y * q.y;
    r.m[2][2] = d + 2.0f * q.z * q.z;
    r.m[0][1] = 2.0f * q.x * q.y - tw * q.z;
    r.m[1][0] = 2.0f * q.x * q.y + tw * q.z;
    r.m[0][2] = 2.0f * q.x * q.z + tw * q.y;
    r.m[2][0] = 2.0f * q.x * q.z - tw * q.y;
    r.m[1][2] = 2.0f * q.y * q.z - tw * q.x;
    r.m[2][1] = 2.0f * q.y * q.z + tw * q.x;
    return r;
}
// dL/dq given dL/dR = a
DFX_HD Q4 q_to_m3_adj(Q4 q, const M3& a) {
    float tr = a.m[0][0] + a.m[1][1] + a.m[2][2];
    V3 k = V3{a.m[2][1] - a.m[1][2], a.m[0][2] - a.m[2][0], a.m[1][0] - a.m[0][1]};  // sum a o d[v]x/dv
    V3 v = qv(q);
    float aw = 4.0f * q.w * tr + 2.0f * dot(v, k);
    // 2 (a + a^T) v
    V3 s = V3{2.0f * a.m[0][0] * v.x + (a.m[0][1] + a.m[1][0]) * v.y + (a.m[0][2] + a.m[2][0]) * v.z,
              (a.m[1][0] + a.m[0][1]) * v.x + 2.0f * a.m[1][1] * v.y + (a.m[1][2] + a.m[2][1]) * v.z,
              (a.m[2][0] + a.m[0][2]) * v.x + (a.m[2][1] + a.m[1][2]) * v.y + 2.0f * a.m[2][2] * v.z};
    V3 av = k * (2.0f * q.w) + s * 2.0f;
    return Q4{av.x, av.y, av.z, aw};
}

// ---------------------------------------------------------------- scratch pointers and load / store helpers
// Per-environment scratch is addressed through SP: element i of an environment lives at p[i * DFX_ES].
//   DFX_ES == 1  : a plain float* (one contiguous block per environment; lane-group kernels, host emulation)
//   DFX_ES == 32 : structure-of-arrays tile of 32 environments, lane = environment (tile kernels): consecutive
//                  lanes touch consecutive banks, every pack read is a warp-wide broadcast
#ifndef DFX_ES
#define DFX_ES 1
#endif
template <class T>
struct StridedPtr {
    T* p;
    DFX_HD StridedPtr operator+(int o) const { return StridedPtr{p + (long long)o * DFX_ES}; }
    DFX_HD StridedPtr operator-(int o) const { return StridedPtr{p - (long long)o * DFX_ES}; }
    DFX_HD T& operator[](int i) const { return p[(long long)i * DFX_ES]; }
    DFX_HD T& operator*() const { return *p; }
    DFX_HD int operator-(StridedPtr o) const { return (int)((p - o.p) / DFX_ES); }
};
#if DFX_ES == 1
using SP = float*;
using SPi = int*;
using SPu = unsigned*;
DFX_HD SPi sp_int(SP s) { return reinterpret_cast<int*>(s); }
DFX_HD SPu sp_uint(SP s) { return reinterpret_cast<unsigned*>(s); }
DFX_HD float* sp_raw(SP s) { return s; }
#else
using SP = StridedPtr<float>;
using SPi = StridedPtr<int>;
using SPu = StridedPtr<unsigned>;
DFX_HD SPi sp_int(SP s) { return SPi{reinterpret_cast<int*>(s.p)}; }
DFX_HD SPu sp_uint(SP s) { return SPu{reinterpret_cast<unsigned*>(s.p)}; }
DFX_HD float* sp_raw(SP s) { return s.p; }
#endif

template <class P> DFX_HD V3 ld3(P p) { return V3{p[0], p[1], p[2]}; }
template <class P> DFX_HD Q4 ld4(P p) { return Q4{p[0], p[1], p[2], p[3]}; }
template <class P> DFX_HD Xf ld7(P p) { return Xf{V3{p[0], p[1], p[2]}, Q4{p[3], p[4], p[5], p[6]}}; }
template <class P> DFX_HD SV ld6(P p) { return SV{V3{p[0], p[1], p[2]}, V3{p[3], p[4], p[5]}}; }
template <class P> DFX_HD void st3(P p, V3 a) { p[0] = a.x; p[1] = a.y; p[2] = a.z; }
template <class P> DFX_HD void st4(P p, Q4 a) { p[0] = a.x; p[1] = a.y; p[2] = a.z; p[3] = a.w; }
template <class P> DFX_HD void st7(P p, Xf a) { st3(p, a.p); st4(p + 3, a.q); }
template <class P> DFX_HD void st6(P p, SV a) { st3(p, a.w); st3(p + 3, a.v); }
template <class P> DFX_HD void add3(P p, V3 a) { p[0] += a.x; p[1] += a.y; p[2] += a.z; }
template <class P> DFX_HD void add4(P p, Q4 a) { p[0] += a.x; p[1] += a.y; p[2] += a.z; p[3] += a.w; }
template <class P> DFX_HD void add7(P p, Xf a) { add3(p, a.p); add4(p + 3, a.q); }
template <class P> DFX_HD void add6(P p, SV a) { add3(p, a.w); add3(p + 3, a.v); }
template <class P> DFX_HD M3 ld9(P p) {
    M3 r;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r.m[i][j] = p[i * 3 + j];
    return r;
}
template <class P> DFX_HD void st9(P p, const M3& a) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) p[i * 3 + j] = a.m[i][j];
}

}  // namespace dfx
