// 3x3 weighted-Procrustes rotation in registers (one-sided Jacobi SVD).
//
// Replaces the reference's host round trip `torch.svd(H.cpu())` + det fix-up
// (reference models/common.py:36-41):  H = U S V^T,  R = V diag(1,1,det(V U^T)) U^T.
//
// One-sided (Hestenes) Jacobi rotates column pairs of G = H until they are orthogonal:
// G = H V = U S.  With columns ordered by decreasing norm,
//     R = v1 u1^T + v2 u2^T + (v1 x v2)(u1 x u2)^T
// because u1 x u2 = det(U) u3 and v1 x v2 = det(V) v3, so the third term equals
// det(V) det(U) v3 u3^T = det(V U^T) v3 u3^T — the reference's reflection fix on the SMALLEST
// singular direction — without ever forming u3 (undetermined when H is rank 2).
#pragma once
#include "common.cuh"

namespace pdsc {

// The solver is templated on its scalar: `float` for the forward's per-seed and refinement solves, `double` for the ICP
// updates (icp.cu).  Each scalar has its own thresholds; the float ones are the literals the float solver has always used.
//
// `rank` is the squared ratio sigma_2 / sigma_1 below which u2 is not worth computing and any unit vector orthogonal to u1 will
// do.  The polar factor of H is determined to |R - R_exact| <= C eps sigma_1 / (sigma_2 + d sigma_3) (C ~ 16, eps the unit
// roundoff): once sigma_2 / sigma_1 drops under ~8 eps that bound exceeds 2, the distance between any two rotations, and every
// choice of u2 is as accurate as any other.  Above it Gram-Schmidt's u2 carries the information, so the threshold is (8 eps)^2:
// 1e-12 ~ (8 * 2^-23)^2 in float, 3.2e-30 ~ (8 * 2^-52)^2 in double.  (The float literal is 10% above (8 eps)^2 = 9.1e-13: at
// its threshold, sigma_2 / sigma_1 = 1e-6, the bound is 1.9 rather than 2.  It stays as it is, and so does every float solve.)
template <typename T> struct KabschTol;
template <> struct KabschTol<float> {
  static constexpr float skip = 1e-9f;     // columns this close to orthogonal (cosine) are left alone
  static constexpr float big = 1e8f;       // |zeta| above which t = 1 / (2 zeta)
  static constexpr float tiny = 1e-30f;    // floor of the squared norms that are inverted
  static constexpr float rank = 1e-12f;    // second squared singular value, relative to the first, below which H is rank 1
  static constexpr float perp = 0.6f;
};
template <> struct KabschTol<double> {
  static constexpr double skip = 1e-18;
  static constexpr double big = 1e8;
  static constexpr double tiny = 1e-30;
  static constexpr double rank = 3.2e-30;
  static constexpr double perp = 0.6;
};

__device__ __forceinline__ float k_abs(float x) { return fabsf(x); }
__device__ __forceinline__ double k_abs(double x) { return fabs(x); }
__device__ __forceinline__ float k_sqrt(float x) { return sqrtf(x); }
__device__ __forceinline__ double k_sqrt(double x) { return sqrt(x); }
__device__ __forceinline__ float k_rsqrt(float x) { return rsqrtf(x); }
__device__ __forceinline__ double k_rsqrt(double x) { return 1.0 / sqrt(x); }
__device__ __forceinline__ float k_copysign(float a, float b) { return copysignf(a, b); }
__device__ __forceinline__ double k_copysign(double a, double b) { return copysign(a, b); }
__device__ __forceinline__ float k_max(float a, float b) { return fmaxf(a, b); }
__device__ __forceinline__ double k_max(double a, double b) { return fmax(a, b); }
__device__ __forceinline__ int k_ilogb(float x) { return ilogbf(x); }
__device__ __forceinline__ int k_ilogb(double x) { return ilogb(x); }
__device__ __forceinline__ float k_scalbn(float x, int e) { return scalbnf(x, e); }
__device__ __forceinline__ double k_scalbn(double x, int e) { return scalbn(x, e); }

template <typename T>
struct Vec3T {
  T x, y, z;
};
using Vec3 = Vec3T<float>;
template <typename T> __device__ __forceinline__ T dot3(Vec3T<T> a, Vec3T<T> b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <typename T> __device__ __forceinline__ Vec3T<T> cross3(Vec3T<T> a, Vec3T<T> b) {
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
template <typename T> __device__ __forceinline__ Vec3T<T> scale3(Vec3T<T> a, T s) { return {a.x * s, a.y * s, a.z * s}; }
template <typename T> __device__ __forceinline__ Vec3T<T> sub3(Vec3T<T> a, Vec3T<T> b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }

template <typename T>
__device__ __forceinline__ void jacobi_pair(Vec3T<T>& gp, Vec3T<T>& gq, Vec3T<T>& vp, Vec3T<T>& vq) {
  const T alpha = dot3(gp, gp), beta = dot3(gq, gq), gamma = dot3(gp, gq);
  if (k_abs(gamma) <= KabschTol<T>::skip * k_sqrt(alpha * beta) || gamma == T(0)) return;
  const T zeta = (beta - alpha) / (T(2) * gamma);
  T t;
  if (k_abs(zeta) > KabschTol<T>::big) {
    t = T(0.5) / zeta;
  } else {
    t = k_copysign(T(1), zeta) / (k_abs(zeta) + k_sqrt(T(1) + zeta * zeta));
  }
  const T c = k_rsqrt(T(1) + t * t), s = c * t;
  const Vec3T<T> gp2 = {c * gp.x - s * gq.x, c * gp.y - s * gq.y, c * gp.z - s * gq.z};
  const Vec3T<T> gq2 = {s * gp.x + c * gq.x, s * gp.y + c * gq.y, s * gp.z + c * gq.z};
  const Vec3T<T> vp2 = {c * vp.x - s * vq.x, c * vp.y - s * vq.y, c * vp.z - s * vq.z};
  const Vec3T<T> vq2 = {s * vp.x + c * vq.x, s * vp.y + c * vq.y, s * vp.z + c * vq.z};
  gp = gp2; gq = gq2; vp = vp2; vq = vq2;
}

template <typename T>
__device__ __forceinline__ Vec3T<T> any_perpendicular(Vec3T<T> a) {
  // unit vector orthogonal to unit vector a
  Vec3T<T> e = (k_abs(a.x) < KabschTol<T>::perp) ? Vec3T<T>{T(1), T(0), T(0)} : Vec3T<T>{T(0), T(1), T(0)};
  Vec3T<T> p = sub3(e, scale3(a, dot3(e, a)));
  return scale3(p, k_rsqrt(k_max(dot3(p, p), KabschTol<T>::tiny)));
}

// H row-major (H[i*3+j] = sum_n w_n Am[n][i] Bm[n][j]); writes R row-major with  b ~= R a.
template <typename T>
__device__ __forceinline__ void kabsch_rotation(const T* H, T* R) {
  // scale to O(1) so the squared norms stay well inside the scalar's range; R is scale invariant.  First by 2^-ilogb(hmax), which
  // is exact (subnormal H included) and leaves the largest entry in [1, 2), then by the reciprocal of that entry.  Dividing by
  // hmax itself overflows to +Inf for hmax below 2^-128 (0 * Inf = NaN) in float.  In this order every scaled entry equals
  // H[i] * (1 / hmax) bit for bit wherever both are normal numbers, and R is bit-identical for H and 2^e H.
  T hmax = T(0);
  bool nan = false;   // fmax returns the other operand of a NaN: hmax alone would not see one
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    hmax = k_max(hmax, k_abs(H[i]));
    nan = nan || isnan(H[i]);
  }
  if (nan || !(hmax > T(0)) || !isfinite(hmax)) {
    // H == 0 (or non-finite): LAPACK returns U = V = I for a zero matrix -> R = I
    R[0] = T(1); R[1] = T(0); R[2] = T(0); R[3] = T(0); R[4] = T(1); R[5] = T(0); R[6] = T(0); R[7] = T(0); R[8] = T(1);
    return;
  }
  const int e = -k_ilogb(hmax);
  const T inv = T(1) / k_scalbn(hmax, e);
  Vec3T<T> g0 = {k_scalbn(H[0], e) * inv, k_scalbn(H[3], e) * inv, k_scalbn(H[6], e) * inv};   // columns of H
  Vec3T<T> g1 = {k_scalbn(H[1], e) * inv, k_scalbn(H[4], e) * inv, k_scalbn(H[7], e) * inv};
  Vec3T<T> g2 = {k_scalbn(H[2], e) * inv, k_scalbn(H[5], e) * inv, k_scalbn(H[8], e) * inv};
  Vec3T<T> v0 = {T(1), T(0), T(0)}, v1 = {T(0), T(1), T(0)}, v2 = {T(0), T(0), T(1)};
#pragma unroll 1
  for (int sweep = 0; sweep < 8; ++sweep) {
    jacobi_pair(g0, g1, v0, v1);
    jacobi_pair(g0, g2, v0, v2);
    jacobi_pair(g1, g2, v1, v2);
  }
  // order by decreasing singular value (column swaps; the cross-product form is blind to det(V))
  T n0 = dot3(g0, g0), n1 = dot3(g1, g1), n2 = dot3(g2, g2);
  if (n0 < n1) { Vec3T<T> t = g0; g0 = g1; g1 = t; t = v0; v0 = v1; v1 = t; T s = n0; n0 = n1; n1 = s; }
  if (n0 < n2) { Vec3T<T> t = g0; g0 = g2; g2 = t; t = v0; v0 = v2; v2 = t; T s = n0; n0 = n2; n2 = s; }
  if (n1 < n2) { Vec3T<T> t = g1; g1 = g2; g2 = t; t = v1; v1 = v2; v2 = t; T s = n1; n1 = n2; n2 = s; }
  // u1, u2 (Gram-Schmidt clean-up); v1, v2 likewise
  const T tiny = KabschTol<T>::tiny;
  Vec3T<T> u1 = scale3(g0, k_rsqrt(k_max(n0, tiny)));
  Vec3T<T> u2 = sub3(g1, scale3(u1, dot3(g1, u1)));
  const T n1c = dot3(u2, u2);
  if (n1c > KabschTol<T>::rank * k_max(n0, tiny)) u2 = scale3(u2, k_rsqrt(n1c)); else u2 = any_perpendicular(u1);
  Vec3T<T> w1 = scale3(v0, k_rsqrt(k_max(dot3(v0, v0), tiny)));
  Vec3T<T> w2 = sub3(v1, scale3(w1, dot3(v1, w1)));
  w2 = scale3(w2, k_rsqrt(k_max(dot3(w2, w2), tiny)));
  const Vec3T<T> u3 = cross3(u1, u2), w3 = cross3(w1, w2);
  R[0] = w1.x * u1.x + w2.x * u2.x + w3.x * u3.x;
  R[1] = w1.x * u1.y + w2.x * u2.y + w3.x * u3.y;
  R[2] = w1.x * u1.z + w2.x * u2.z + w3.x * u3.z;
  R[3] = w1.y * u1.x + w2.y * u2.x + w3.y * u3.x;
  R[4] = w1.y * u1.y + w2.y * u2.y + w3.y * u3.y;
  R[5] = w1.y * u1.z + w2.y * u2.z + w3.y * u3.z;
  R[6] = w1.z * u1.x + w2.z * u2.x + w3.z * u3.x;
  R[7] = w1.z * u1.y + w2.z * u2.y + w3.z * u3.y;
  R[8] = w1.z * u1.z + w2.z * u2.z + w3.z * u3.z;
}

}  // namespace pdsc
