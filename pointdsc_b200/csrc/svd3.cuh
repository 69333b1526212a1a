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

struct Vec3 {
  float x, y, z;
};
__device__ __forceinline__ float dot3(Vec3 a, Vec3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ Vec3 cross3(Vec3 a, Vec3 b) {
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
__device__ __forceinline__ Vec3 scale3(Vec3 a, float s) { return {a.x * s, a.y * s, a.z * s}; }
__device__ __forceinline__ Vec3 sub3(Vec3 a, Vec3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }

__device__ __forceinline__ void jacobi_pair(Vec3& gp, Vec3& gq, Vec3& vp, Vec3& vq) {
  const float alpha = dot3(gp, gp), beta = dot3(gq, gq), gamma = dot3(gp, gq);
  if (fabsf(gamma) <= 1e-9f * sqrtf(alpha * beta) || gamma == 0.0f) return;
  const float zeta = (beta - alpha) / (2.0f * gamma);
  float t;
  if (fabsf(zeta) > 1e8f) {
    t = 0.5f / zeta;
  } else {
    t = copysignf(1.0f, zeta) / (fabsf(zeta) + sqrtf(1.0f + zeta * zeta));
  }
  const float c = rsqrtf(1.0f + t * t), s = c * t;
  const Vec3 gp2 = {c * gp.x - s * gq.x, c * gp.y - s * gq.y, c * gp.z - s * gq.z};
  const Vec3 gq2 = {s * gp.x + c * gq.x, s * gp.y + c * gq.y, s * gp.z + c * gq.z};
  const Vec3 vp2 = {c * vp.x - s * vq.x, c * vp.y - s * vq.y, c * vp.z - s * vq.z};
  const Vec3 vq2 = {s * vp.x + c * vq.x, s * vp.y + c * vq.y, s * vp.z + c * vq.z};
  gp = gp2; gq = gq2; vp = vp2; vq = vq2;
}

__device__ __forceinline__ Vec3 any_perpendicular(Vec3 a) {
  // unit vector orthogonal to unit vector a
  Vec3 e = (fabsf(a.x) < 0.6f) ? Vec3{1.f, 0.f, 0.f} : Vec3{0.f, 1.f, 0.f};
  Vec3 p = sub3(e, scale3(a, dot3(e, a)));
  return scale3(p, rsqrtf(fmaxf(dot3(p, p), 1e-30f)));
}

// H row-major (H[i*3+j] = sum_n w_n Am[n][i] Bm[n][j]); writes R row-major with  b ~= R a.
__device__ __forceinline__ void kabsch_rotation(const float* H, float* R) {
  // scale to O(1) so the squared norms stay well inside fp32 range; R is scale invariant.  First by 2^-ilogb(hmax), which is
  // exact (subnormal H included) and leaves the largest entry in [1, 2), then by the reciprocal of that entry.  Dividing by
  // hmax itself overflows to +Inf for hmax below 2^-128 (0 * Inf = NaN).  In this order every scaled entry equals
  // H[i] * (1 / hmax) bit for bit wherever both are normal floats, and R is bit-identical for H and 2^e H.
  float hmax = 0.f;
  bool nan = false;   // fmaxf returns the other operand of a NaN: hmax alone would not see one
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    hmax = fmaxf(hmax, fabsf(H[i]));
    nan = nan || isnan(H[i]);
  }
  if (nan || !(hmax > 0.f) || !isfinite(hmax)) {
    // H == 0 (or non-finite): LAPACK returns U = V = I for a zero matrix -> R = I
    R[0] = 1.f; R[1] = 0.f; R[2] = 0.f; R[3] = 0.f; R[4] = 1.f; R[5] = 0.f; R[6] = 0.f; R[7] = 0.f; R[8] = 1.f;
    return;
  }
  const int e = -ilogbf(hmax);
  const float inv = 1.0f / scalbnf(hmax, e);
  Vec3 g0 = {scalbnf(H[0], e) * inv, scalbnf(H[3], e) * inv, scalbnf(H[6], e) * inv};   // columns of H
  Vec3 g1 = {scalbnf(H[1], e) * inv, scalbnf(H[4], e) * inv, scalbnf(H[7], e) * inv};
  Vec3 g2 = {scalbnf(H[2], e) * inv, scalbnf(H[5], e) * inv, scalbnf(H[8], e) * inv};
  Vec3 v0 = {1.f, 0.f, 0.f}, v1 = {0.f, 1.f, 0.f}, v2 = {0.f, 0.f, 1.f};
#pragma unroll 1
  for (int sweep = 0; sweep < 8; ++sweep) {
    jacobi_pair(g0, g1, v0, v1);
    jacobi_pair(g0, g2, v0, v2);
    jacobi_pair(g1, g2, v1, v2);
  }
  // order by decreasing singular value (column swaps; the cross-product form is blind to det(V))
  float n0 = dot3(g0, g0), n1 = dot3(g1, g1), n2 = dot3(g2, g2);
  if (n0 < n1) { Vec3 t = g0; g0 = g1; g1 = t; t = v0; v0 = v1; v1 = t; float s = n0; n0 = n1; n1 = s; }
  if (n0 < n2) { Vec3 t = g0; g0 = g2; g2 = t; t = v0; v0 = v2; v2 = t; float s = n0; n0 = n2; n2 = s; }
  if (n1 < n2) { Vec3 t = g1; g1 = g2; g2 = t; t = v1; v1 = v2; v2 = t; float s = n1; n1 = n2; n2 = s; }
  // u1, u2 (Gram-Schmidt clean-up); v1, v2 likewise
  Vec3 u1 = scale3(g0, rsqrtf(fmaxf(n0, 1e-30f)));
  Vec3 u2 = sub3(g1, scale3(u1, dot3(g1, u1)));
  const float n1c = dot3(u2, u2);
  if (n1c > 1e-12f * fmaxf(n0, 1e-30f)) u2 = scale3(u2, rsqrtf(n1c)); else u2 = any_perpendicular(u1);
  Vec3 w1 = scale3(v0, rsqrtf(fmaxf(dot3(v0, v0), 1e-30f)));
  Vec3 w2 = sub3(v1, scale3(w1, dot3(v1, w1)));
  w2 = scale3(w2, rsqrtf(fmaxf(dot3(w2, w2), 1e-30f)));
  const Vec3 u3 = cross3(u1, u2), w3 = cross3(w1, w2);
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
