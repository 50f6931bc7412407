// bik_math.h -- SE(3)/SO(3) primitives for the device kernels (host-compilable for unit tests).
//
// All functions are templates on the scalar type and carry BIK_HD so that the identical source is
// exercised on the CPU by tests/host_emu (one lane per instance) and on sm_90a by the kernels.
// What each routine computes is defined by the reference's Lie layer:
//   so3_log ............ mink/lie/so3.py:176-191
//   se3_log ............ mink/lie/se3.py:159-185
//   so3 ljacinv coeff .. mink/lie/so3.py:215-226
//   se3 ljacinv, Q ..... mink/lie/se3.py:211-249
// but the formulas are re-derived for fp32: every coefficient of the form (1 - x)/theta^k is
// evaluated by its Maclaurin series below |theta| = 1 instead of by the cancelling closed form the
// fp64 reference can afford (see DESIGN.md "fp32 Lie coefficients").  The fp64 instantiations sum
// more terms of the same series, so that they too are accurate to the last bits below |theta| = 1.
#pragma once

#include <math.h>

#if defined(__CUDACC__)
#define BIK_HD __host__ __device__ __forceinline__
#else
#define BIK_HD inline
#endif

namespace bik {

template <typename T> struct V3 { T x, y, z; };
template <typename T> struct Q4 { T w, x, y, z; };
template <typename T> struct M3 { T m[9]; };  // row major

template <typename T> BIK_HD V3<T> v3(T x, T y, T z) { V3<T> r; r.x = x; r.y = y; r.z = z; return r; }
template <typename T> BIK_HD V3<T> operator+(V3<T> a, V3<T> b) { return v3<T>(a.x + b.x, a.y + b.y, a.z + b.z); }
template <typename T> BIK_HD V3<T> operator-(V3<T> a, V3<T> b) { return v3<T>(a.x - b.x, a.y - b.y, a.z - b.z); }
template <typename T> BIK_HD V3<T> operator*(T s, V3<T> a) { return v3<T>(s * a.x, s * a.y, s * a.z); }
template <typename T> BIK_HD T dot(V3<T> a, V3<T> b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <typename T> BIK_HD V3<T> cross(V3<T> a, V3<T> b) {
  return v3<T>(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}

template <typename T> BIK_HD Q4<T> q4(T w, T x, T y, T z) { Q4<T> r; r.w = w; r.x = x; r.y = y; r.z = z; return r; }
template <typename T> BIK_HD Q4<T> qmul(Q4<T> a, Q4<T> b) {
  return q4<T>(a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
               a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x, a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w);
}
template <typename T> BIK_HD Q4<T> qconj(Q4<T> a) { return q4<T>(a.w, -a.x, -a.y, -a.z); }
template <typename T> BIK_HD T bik_sqrt(T x);
template <> BIK_HD float bik_sqrt<float>(float x) { return sqrtf(x); }
template <> BIK_HD double bik_sqrt<double>(double x) { return sqrt(x); }
template <typename T> BIK_HD T bik_min(T a, T b) { return a < b ? a : b; }
template <typename T> BIK_HD T bik_max(T a, T b) { return a > b ? a : b; }
template <typename T> BIK_HD T inv_sqrt(T x) { return T(1) / bik_sqrt<T>(x); }
#if defined(__CUDA_ARCH__)
template <> BIK_HD float inv_sqrt<float>(float x) {  // MUFU.RSQ + one Newton step: < 1 ulp, no division
  float r = rsqrtf(x);
  return r * (1.5f - 0.5f * x * r * r);
}
#endif
template <typename T> BIK_HD Q4<T> qnormalize(Q4<T> a) {
  T n2 = a.w * a.w + a.x * a.x + a.y * a.y + a.z * a.z;
  if (!(n2 > T(1e-30))) return q4<T>(T(1), T(0), T(0), T(0));
  T s = inv_sqrt<T>(n2);
  return q4<T>(a.w * s, a.x * s, a.y * s, a.z * s);
}
// rotate v by unit quaternion q:  v + 2 w (u x v) + 2 u x (u x v)
template <typename T> BIK_HD V3<T> qrot(Q4<T> q, V3<T> v) {
  V3<T> u = v3<T>(q.x, q.y, q.z);
  V3<T> t = cross(u, v);
  t = v3<T>(t.x + t.x, t.y + t.y, t.z + t.z);
  V3<T> c = cross(u, t);
  return v3<T>(v.x + q.w * t.x + c.x, v.y + q.w * t.y + c.y, v.z + q.w * t.z + c.z);
}
template <typename T> BIK_HD V3<T> qrot_inv(Q4<T> q, V3<T> v) { return qrot(qconj(q), v); }

template <typename T> BIK_HD M3<T> q2mat(Q4<T> q) {  // unit quaternion -> rotation matrix
  M3<T> R;
  T xx = q.x * q.x, yy = q.y * q.y, zz = q.z * q.z, xy = q.x * q.y, xz = q.x * q.z, yz = q.y * q.z;
  T wx = q.w * q.x, wy = q.w * q.y, wz = q.w * q.z;
  R.m[0] = T(1) - 2 * (yy + zz); R.m[1] = 2 * (xy - wz); R.m[2] = 2 * (xz + wy);
  R.m[3] = 2 * (xy + wz); R.m[4] = T(1) - 2 * (xx + zz); R.m[5] = 2 * (yz - wx);
  R.m[6] = 2 * (xz - wy); R.m[7] = 2 * (yz + wx); R.m[8] = T(1) - 2 * (xx + yy);
  return R;
}
template <typename T> BIK_HD V3<T> mcol(const M3<T>& R, int c) { return v3<T>(R.m[c], R.m[3 + c], R.m[6 + c]); }
template <typename T> BIK_HD V3<T> mmul(const M3<T>& R, V3<T> v) {
  return v3<T>(R.m[0] * v.x + R.m[1] * v.y + R.m[2] * v.z, R.m[3] * v.x + R.m[4] * v.y + R.m[5] * v.z,
               R.m[6] * v.x + R.m[7] * v.y + R.m[8] * v.z);
}
template <typename T> BIK_HD M3<T> mmul(const M3<T>& A, const M3<T>& B) {
  M3<T> C;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C.m[3 * i + j] = A.m[3 * i] * B.m[j] + A.m[3 * i + 1] * B.m[3 + j] + A.m[3 * i + 2] * B.m[6 + j];
  return C;
}
template <typename T> BIK_HD M3<T> mtrans(const M3<T>& A) {
  M3<T> C;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C.m[3 * i + j] = A.m[3 * j + i];
  return C;
}
template <typename T> BIK_HD M3<T> skew(V3<T> w) {
  M3<T> S;
  S.m[0] = 0; S.m[1] = -w.z; S.m[2] = w.y; S.m[3] = w.z; S.m[4] = 0; S.m[5] = -w.x; S.m[6] = -w.y; S.m[7] = w.x; S.m[8] = 0;
  return S;
}
// mju_mat2Quat branch selection (only used where the quaternion SIGN must match the reference's
// SO3.from_matrix, i.e. in pose outputs; logs are sign invariant).
template <typename T> BIK_HD Q4<T> mat2quat(const M3<T>& R) {
  const T* m = R.m;
  T tr = m[0] + m[4] + m[8];
  Q4<T> q;
  if (tr > 0) { q.w = T(0.5) * sqrt(1 + tr); T k = T(0.25) / q.w; q.x = k * (m[7] - m[5]); q.y = k * (m[2] - m[6]); q.z = k * (m[3] - m[1]); }
  else if (m[0] > m[4] && m[0] > m[8]) { q.x = T(0.5) * sqrt(1 + m[0] - m[4] - m[8]); T k = T(0.25) / q.x; q.w = k * (m[7] - m[5]); q.y = k * (m[3] + m[1]); q.z = k * (m[2] + m[6]); }
  else if (m[4] > m[8]) { q.y = T(0.5) * sqrt(1 - m[0] + m[4] - m[8]); T k = T(0.25) / q.y; q.w = k * (m[2] - m[6]); q.x = k * (m[3] + m[1]); q.z = k * (m[7] + m[5]); }
  else { q.z = T(0.5) * sqrt(1 - m[0] - m[4] + m[8]); T k = T(0.25) / q.z; q.w = k * (m[3] - m[1]); q.x = k * (m[2] + m[6]); q.y = k * (m[7] + m[5]); }
  return qnormalize(q);
}

template <typename T> BIK_HD void bik_sincos(T a, T* s, T* c);
template <> BIK_HD void bik_sincos<float>(float a, float* s, float* c) {
#if defined(__CUDA_ARCH__)
  sincosf(a, s, c);
#else
  *s = sinf(a); *c = cosf(a);
#endif
}
template <> BIK_HD void bik_sincos<double>(double a, double* s, double* c) {
#if defined(__CUDA_ARCH__)
  sincos(a, s, c);
#else
  *s = sin(a); *c = cos(a);
#endif
}

// log of a unit quaternion as a rotation vector (angle in (-pi, pi]); sign invariant (q ~ -q).
template <typename T> BIK_HD V3<T> so3_log(Q4<T> q) {
  T nsq = q.x * q.x + q.y * q.y + q.z * q.z, f;
  if (nsq < T(1e-10)) {
    f = T(2) / q.w - T(2.0 / 3.0) * nsq / (q.w * q.w * q.w);
  } else {
    T n = sqrt(nsq);
    f = T(2) * atan2(q.w < 0 ? -n : n, fabs(q.w)) / n;
  }
  return v3<T>(f * q.x, f * q.y, f * q.z);
}

// A(theta) = (1 - (theta/2) cot(theta/2)) / theta^2 : coefficient of [w]x^2 in both V^-1 (se3 log)
// and the SO(3) inverse left Jacobian.  Series below theta^2 = 1.  Its coefficients |B_2n| / (2n)!
// fall only by ~1/(4 pi^2) per term: six terms leave 1.6e-10 relative at theta^2 -> 1, enough for
// fp32; fp64 takes eleven (2e-18).  The fp64 coefficients below (and those of coef_BCD) are the
// Maclaurin coefficients in theta^2 rounded to double, from sympy's series of the closed forms.
template <typename T> BIK_HD T coef_A(T t2) {
  if (t2 < T(1)) {
    if constexpr (sizeof(T) == 8)
      return T(0.08333333333333333) + t2 * (T(0.001388888888888889) + t2 * (T(3.306878306878307e-05) + t2 * (T(8.267195767195768e-07) +
             t2 * (T(2.08767569878681e-08) + t2 * (T(5.284190138687493e-10) + t2 * (T(1.3382536530684679e-11) + t2 * (T(3.3896802963225827e-13) +
             t2 * (T(8.586062056277845e-15) + t2 * (T(2.174868698558062e-16) + t2 * T(5.5090028283602295e-18))))))))));
    return T(1.0 / 12.0) + t2 * (T(1.0 / 720.0) + t2 * (T(1.0 / 30240.0) + t2 * (T(1.0 / 1209600.0) + t2 * (T(1.0 / 47900160.0) + t2 * T(691.0 / 1307674368000.0)))));
  }
  T th = sqrt(t2), s, c;
  bik_sincos<T>(T(0.5) * th, &s, &c);
  return (T(1) - T(0.5) * th * c / s) / t2;
}
// B = (th - sin th)/th^3, C = (1 - th^2/2 - cos th)/th^4, D = (2 th - 3 sin th + th cos th)/(2 th^5).
// Series below theta^2 = 1: six terms for fp32 (5e-12 relative at most), nine for fp64 (5e-17).
template <typename T> BIK_HD void coef_BCD(T t2, T* B, T* C, T* D) {
  if (t2 < T(1)) {
    if constexpr (sizeof(T) == 8) {
      *B = T(0.16666666666666666) + t2 * (T(-0.008333333333333333) + t2 * (T(0.0001984126984126984) + t2 * (T(-2.7557319223985893e-06) +
           t2 * (T(2.505210838544172e-08) + t2 * (T(-1.6059043836821613e-10) + t2 * (T(7.647163731819816e-13) + t2 * (T(-2.8114572543455206e-15) +
           t2 * T(8.22063524662433e-18))))))));
      *C = T(-0.041666666666666664) + t2 * (T(0.001388888888888889) + t2 * (T(-2.48015873015873e-05) + t2 * (T(2.755731922398589e-07) +
           t2 * (T(-2.08767569878681e-09) + t2 * (T(1.1470745597729725e-11) + t2 * (T(-4.779477332387385e-14) + t2 * (T(1.5619206968586225e-16) +
           t2 * T(-4.110317623312165e-19))))))));
      *D = T(0.008333333333333333) + t2 * (T(-0.0003968253968253968) + t2 * (T(8.267195767195768e-06) + t2 * (T(-1.0020843354176688e-07) +
           t2 * (T(8.029521918410807e-10) + t2 * (T(-4.58829823909189e-12) + t2 * (T(1.9680200780418645e-14) + t2 * (T(-6.576508197299464e-17) +
           t2 * T(1.7615646957052136e-19))))))));
      return;
    }
    *B = T(1.0 / 6.0) + t2 * (T(-1.0 / 120.0) + t2 * (T(1.0 / 5040.0) + t2 * (T(-1.0 / 362880.0) + t2 * (T(1.0 / 39916800.0) + t2 * T(-1.0 / 6227020800.0)))));
    *C = T(-1.0 / 24.0) + t2 * (T(1.0 / 720.0) + t2 * (T(-1.0 / 40320.0) + t2 * (T(1.0 / 3628800.0) + t2 * (T(-1.0 / 479001600.0) + t2 * T(1.0 / 87178291200.0)))));
    *D = T(1.0 / 120.0) + t2 * (T(-1.0 / 2520.0) + t2 * (T(1.0 / 120960.0) + t2 * (T(-1.0 / 9979200.0) + t2 * (T(1.0 / 1245404160.0) + t2 * T(-1.0 / 217945728000.0)))));
    return;
  }
  T th = sqrt(t2), s, c;
  bik_sincos<T>(th, &s, &c);
  *B = (th - s) / (t2 * th);
  *C = (T(1) - T(0.5) * t2 - c) / (t2 * t2);
  *D = (T(2) * th - T(3) * s + th * c) / (T(2) * t2 * t2 * th);
}

// xi = log(T) for T = (q, t): xi = (V^-1 t, w).
template <typename T> BIK_HD void se3_log(Q4<T> q, V3<T> t, V3<T>* v, V3<T>* w) {
  *w = so3_log(q);
  T t2 = dot(*w, *w);
  T A = coef_A(t2);
  V3<T> wt = cross(*w, t);
  V3<T> wwt = cross(*w, wt);
  *v = v3<T>(t.x - T(0.5) * wt.x + A * wwt.x, t.y - T(0.5) * wt.y + A * wwt.y, t.z - T(0.5) * wt.z + A * wwt.z);
}

// Blocks of the SE(3) inverse LEFT Jacobian at xi = (v, w):  [[Ji, Mi], [0, Ji]], Mi = -Ji Q Ji.
// Identity (and Mi = 0) when |w|^2 < 1e-10: the reference's discontinuity, mink/lie/se3.py:212-214.
template <typename T> BIK_HD void se3_ljacinv_blocks(V3<T> v, V3<T> w, M3<T>* Ji, M3<T>* Mi) {
  T t2 = dot(w, w);
  if (t2 < T(1e-10)) {
    for (int i = 0; i < 9; ++i) { Ji->m[i] = (i % 4 == 0) ? T(1) : T(0); Mi->m[i] = T(0); }
    return;
  }
  T A = coef_A(t2), B, C, D;
  coef_BCD(t2, &B, &C, &D);
  M3<T> W = skew(w), V = skew(v), W2 = mmul(W, W);
  for (int i = 0; i < 9; ++i) Ji->m[i] = ((i % 4 == 0) ? T(1) : T(0)) - T(0.5) * W.m[i] + A * W2.m[i];
  M3<T> VW = mmul(V, W), WV = mtrans(VW), WVW = mmul(WV, W), VWW = mmul(VW, W), VWWt = mtrans(VWW);
  M3<T> T1 = mmul(WVW, W), T2 = mmul(W, WVW), Q;
  for (int i = 0; i < 9; ++i)
    Q.m[i] = T(0.5) * V.m[i] + B * (WV.m[i] + VW.m[i] + WVW.m[i]) - C * (VWW.m[i] - VWWt.m[i] - T(3) * WVW.m[i]) + D * (T1.m[i] + T2.m[i]);
  M3<T> JQ = mmul(*Ji, Q), JQJ = mmul(JQ, *Ji);
  for (int i = 0; i < 9; ++i) Mi->m[i] = -JQJ.m[i];
}

// body-frame rotation vector taking quaternion qb to qa (mju_subQuat), angle wrapped to (-pi, pi].
template <typename T> BIK_HD V3<T> quat_sub(Q4<T> qa, Q4<T> qb) {
  Q4<T> d = qmul(qconj(qb), qa);
  T s = sqrt(d.x * d.x + d.y * d.y + d.z * d.z);
  if (!(s > T(1e-15))) return v3<T>(T(0), T(0), T(0));
  T ang = T(2) * atan2(s, d.w);
  if (ang > T(3.14159265358979323846)) ang -= T(6.28318530717958647692);
  T k = ang / s;
  return v3<T>(k * d.x, k * d.y, k * d.z);
}

// q <- normalize(q) * exp(w)  (mju_quatIntegrate with dt folded into w)
template <typename T> BIK_HD Q4<T> quat_integrate(Q4<T> q, V3<T> w) {
  q = qnormalize(q);
  T n = sqrt(dot(w, w));
  if (!(n > T(1e-15))) return q;
  T s, c;
  bik_sincos<T>(T(0.5) * n, &s, &c);
  T k = s / n;
  return qnormalize(qmul(q, q4<T>(c, k * w.x, k * w.y, k * w.z)));
}

}  // namespace bik
