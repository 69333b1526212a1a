// a10, a11, a12 — weighted Kabsch per seed, hypothesis scoring / selection, post-refinement.
//
// Reference call sites:
//   weights + rigid_transform_3d   models/PointDSC.py:282-316, models/common.py:7-45
//   scoring / argmax / labels      models/PointDSC.py:325-336
//   post_refinement                models/PointDSC.py:403-438
//
// The reference leaves the device for every 3x3 SVD (`torch.svd(H.cpu())`, common.py:36) and syncs
// the host once per refinement iteration (`int(inlier_num ...)`, PointDSC.py:426).  Here the SVD is a
// register-resident Jacobi (svd3.cuh), one warp per seed problem, and the refinement is one CTA per
// set that iterates on the device — no host round trips anywhere on the path.
#include <cmath>

#include "common.cuh"
#include "kernels.h"
#include "sets.cuh"
#include "svd3.cuh"
#include "weighted_kabsch.cuh"

namespace pdsc {

__device__ __forceinline__ float residual(const float* T, float x, float y, float z, float tx, float ty, float tz) {
  const float px = fmaf(T[0], x, fmaf(T[1], y, T[2] * z)) + T[3];
  const float py = fmaf(T[4], x, fmaf(T[5], y, T[6] * z)) + T[7];
  const float pz = fmaf(T[8], x, fmaf(T[9], y, T[10] * z)) + T[11];
  const float dx = px - tx, dy = py - ty, dz = pz - tz;
  return sqrtf(dx * dx + dy * dy + dz * dz);
}

// -------------------------------------------------------------------------------------------------
// one warp per (set, seed): eigenvector -> weights -> weighted Kabsch -> inlier count over all N
// -------------------------------------------------------------------------------------------------
constexpr int kHypChunk = 1024;      // points staged per pass (24 KB)
__global__ void __launch_bounds__(256) seed_hypotheses_kernel(
    const float* __restrict__ src, const float* __restrict__ tgt, const int32_t* __restrict__ knn_idx,
    const float* __restrict__ iterates, const uint32_t* __restrict__ conv_mask, const float* __restrict__ seed_trans_in,
    float* __restrict__ seed_trans, int32_t* __restrict__ inlier_counts, unsigned long long* __restrict__ best_key,
    float* __restrict__ eig_out, int32_t* __restrict__ power_iters, const SetDesc* __restrict__ sets, int iters, float d2_lim,
    int mask_stride) {
  // the set's points, staged once per CTA for its eight seeds: six arrays so that an 8-byte load is the same coordinate of two points
  __shared__ __align__(8) float pts_s[6][kHypChunk];
  const int b = blockIdx.y;
  const SetDesc d = sets[b];
  const int N = d.N, S = d.S, k = d.k;
  if ((int)blockIdx.x * 8 >= S) return;     // the grid is sized by the largest set: the whole CTA leaves
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int s_raw = blockIdx.x * 8 + warp;
  const bool active = s_raw < S;            // inactive warps still take part in the staging barriers
  const int s = active ? s_raw : S - 1;
  const size_t row = (size_t)d.seed0 + s;
  const size_t nb0 = (size_t)d.knn0 + (size_t)s * k;   // the seed's first neighbour slot
  const float* ps = src + (size_t)d.row0 * 3;
  const float* pt = tgt + (size_t)d.row0 * 3;

  // exit iteration of this set: first iteration at which every seed passed allclose, else the cap
  const uint32_t m = conv_mask[(size_t)b * mask_stride] & ((iters >= 32) ? 0xFFFFFFFFu : ((1u << iters) - 1u));
  const int t_exit = m ? (__ffs(m) - 1) : (iters - 1);
  if (active && s == 0 && lane == 0 && power_iters) power_iters[b] = t_exit + 1;

  float T[12];
  if (seed_trans_in) {
#pragma unroll
    for (int i = 0; i < 12; ++i) T[i] = seed_trans_in[row * 16 + i];
  } else {
    constexpr int kPer = kMaxK / 32;
    float w[kPer], ax[kPer], ay[kPer], az[kPer], bx[kPer], by[kPer], bz[kPer];
    float wsum = 0.f;
#pragma unroll
    for (int q = 0; q < kPer; ++q) {
      const int a = lane + q * 32;
      w[q] = 0.f; ax[q] = ay[q] = az[q] = bx[q] = by[q] = bz[q] = 0.f;
      if (a < k) {
        float e = iterates[nb0 * iters + (size_t)t_exit * k + a];
        if (eig_out && active) eig_out[nb0 + a] = e;
        w[q] = e;
        int j = knn_idx[nb0 + a];
        j = min(max(j, 0), N - 1);
        ax[q] = ps[(size_t)j * 3]; ay[q] = ps[(size_t)j * 3 + 1]; az[q] = ps[(size_t)j * 3 + 2];
        bx[q] = pt[(size_t)j * 3]; by[q] = pt[(size_t)j * 3 + 1]; bz[q] = pt[(size_t)j * 3 + 2];
      }
      wsum += w[q];
    }
    // total_weight / (sum + 1e-6)   (PointDSC.py:282)
    wsum = warp_sum(wsum);
    const float wden = wsum + 1e-6f;
    float sw = 0.f, sax = 0.f, say = 0.f, saz = 0.f, sbx = 0.f, sby = 0.f, sbz = 0.f;
#pragma unroll
    for (int q = 0; q < kPer; ++q) {
      w[q] = w[q] / wden;
      if (w[q] < 0.f) w[q] = 0.f;  // weights[weights < 0] = 0   (common.py:20)
      sw += w[q];
      sax = fmaf(w[q], ax[q], sax); say = fmaf(w[q], ay[q], say); saz = fmaf(w[q], az[q], saz);
      sbx = fmaf(w[q], bx[q], sbx); sby = fmaf(w[q], by[q], sby); sbz = fmaf(w[q], bz[q], sbz);
    }
    sw = warp_sum(sw);
    sax = warp_sum(sax); say = warp_sum(say); saz = warp_sum(saz);
    sbx = warp_sum(sbx); sby = warp_sum(sby); sbz = warp_sum(sbz);
    const float den = sw + 1e-6f;  // centroid denominators (common.py:24-25)
    const float cax = sax / den, cay = say / den, caz = saz / den;
    const float cbx = sbx / den, cby = sby / den, cbz = sbz / den;
    float H[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) H[i] = 0.f;
#pragma unroll
    for (int q = 0; q < kPer; ++q) {
      const float mx = ax[q] - cax, my = ay[q] - cay, mz = az[q] - caz;
      const float nx = (bx[q] - cbx) * w[q], ny = (by[q] - cby) * w[q], nz = (bz[q] - cbz) * w[q];
      H[0] = fmaf(mx, nx, H[0]); H[1] = fmaf(mx, ny, H[1]); H[2] = fmaf(mx, nz, H[2]);
      H[3] = fmaf(my, nx, H[3]); H[4] = fmaf(my, ny, H[4]); H[5] = fmaf(my, nz, H[5]);
      H[6] = fmaf(mz, nx, H[6]); H[7] = fmaf(mz, ny, H[7]); H[8] = fmaf(mz, nz, H[8]);
    }
#pragma unroll
    for (int i = 0; i < 9; ++i) H[i] = warp_sum(H[i]);
    float R[9];
    kabsch_rotation(H, R);  // every lane solves the same 3x3 problem in registers
    T[0] = R[0]; T[1] = R[1]; T[2] = R[2];  T[3] = cbx - (R[0] * cax + R[1] * cay + R[2] * caz);
    T[4] = R[3]; T[5] = R[4]; T[6] = R[5];  T[7] = cby - (R[3] * cax + R[4] * cay + R[5] * caz);
    T[8] = R[6]; T[9] = R[7]; T[10] = R[8]; T[11] = cbz - (R[6] * cax + R[7] * cay + R[8] * caz);
  }
  if (lane < 16 && active) {
    float val = (lane == 15) ? 1.0f : 0.0f;
#pragma unroll
    for (int i = 0; i < 12; ++i)
      if (lane == i) val = T[i];
    seed_trans[row * 16 + lane] = val;
  }

  // inlier count of this hypothesis over all N correspondences: ||R p + t - q|| < thr  <=>  the squared length < d2_lim (the smallest
  // float whose correctly rounded root is >= thr: sqrt is monotonic), two points at a time (every lane
  // rounded exactly like residual(): fma(T0, x, fma(T1, y, T2 z)) + T3, then dx^2, fma(dy, dy, .), fma(dz, dz, .))
  int cnt = 0;
  for (int j0 = 0; j0 < N; j0 += kHypChunk) {
    __syncthreads();
    for (int f = threadIdx.x; f < 3 * kHypChunk; f += 256) {
      const int j = f / 3, c = f - 3 * j;
      const bool have = j0 + j < N;
      pts_s[c][j] = have ? ps[(size_t)(j0 + j) * 3 + c] : 0.f;
      pts_s[3 + c][j] = have ? pt[(size_t)(j0 + j) * 3 + c] : INFINITY;   // a pad target is infinitely far away
    }
    __syncthreads();
    const int lim = min(kHypChunk, (N - j0 + 1) & ~1);
    for (int j = 2 * lane; j < lim; j += 64) {
      const float2 x = *reinterpret_cast<const float2*>(&pts_s[0][j]), y = *reinterpret_cast<const float2*>(&pts_s[1][j]),
                   z = *reinterpret_cast<const float2*>(&pts_s[2][j]);
      const float2 tx = *reinterpret_cast<const float2*>(&pts_s[3][j]), ty = *reinterpret_cast<const float2*>(&pts_s[4][j]),
                   tz = *reinterpret_cast<const float2*>(&pts_s[5][j]);
      float2 px = make_float2(__fmul_rn(T[2], z.x), __fmul_rn(T[2], z.y));
      float2 py = make_float2(__fmul_rn(T[6], z.x), __fmul_rn(T[6], z.y));
      float2 pz = make_float2(__fmul_rn(T[10], z.x), __fmul_rn(T[10], z.y));
      ffma2(px.x, px.y, T[1], y.x, y.y); ffma2(px.x, px.y, T[0], x.x, x.y);
      ffma2(py.x, py.y, T[5], y.x, y.y); ffma2(py.x, py.y, T[4], x.x, x.y);
      ffma2(pz.x, pz.y, T[9], y.x, y.y); ffma2(pz.x, pz.y, T[8], x.x, x.y);
      const float2 dx = make_float2(__fsub_rn(__fadd_rn(px.x, T[3]), tx.x), __fsub_rn(__fadd_rn(px.y, T[3]), tx.y));
      const float2 dy = make_float2(__fsub_rn(__fadd_rn(py.x, T[7]), ty.x), __fsub_rn(__fadd_rn(py.y, T[7]), ty.y));
      const float2 dz = make_float2(__fsub_rn(__fadd_rn(pz.x, T[11]), tz.x), __fsub_rn(__fadd_rn(pz.y, T[11]), tz.y));
      const float2 d2 = ffma2_pair(dz, dz, ffma2_pair(dy, dy, fmul2(dx, dx)));
      cnt += (d2.x < d2_lim ? 1 : 0) + (d2.y < d2_lim ? 1 : 0);
    }
  }
  if (!active) return;
  cnt = warp_sum(cnt);
  if (lane == 0) {
    if (inlier_counts) inlier_counts[row] = cnt;
    // argmax(fitness) with first-index tie-break: larger count wins, then smaller seed position
    atomicMax(best_key + b, ((unsigned long long)(unsigned)cnt << 32) | (unsigned)(0xFFFFFFFFu - (unsigned)s));
  }
}

void launch_seed_hypotheses(const float* src, const float* tgt, const int32_t* knn_idx, const float* iterates,
                            const uint32_t* conv_mask, const float* seed_trans_in, float* seed_trans,
                            int32_t* inlier_counts, unsigned long long* best_key, float* eig_out, int32_t* power_iters,
                            int B, int N, int S, int k, int iters, float inlier_threshold, int mask_stride,
                            cudaStream_t st, const SetDesc* sets) {
  if (S <= 0) return;
  // smallest float x with sqrtf(x) >= threshold (IEEE sqrt on the host == the device's sqrt.rn): residual < threshold <=> its square < x
  float d2_lim = inlier_threshold * inlier_threshold;
  while (std::sqrt(d2_lim) >= inlier_threshold && d2_lim > 0.f) d2_lim = std::nextafter(d2_lim, 0.0f);
  while (std::sqrt(d2_lim) < inlier_threshold) d2_lim = std::nextafter(d2_lim, INFINITY);
  seed_hypotheses_kernel<<<dim3((S + 7) / 8, B), 256, 0, st>>>(src, tgt, knn_idx, iterates, conv_mask, seed_trans_in,
                                                              seed_trans, inlier_counts, best_key, eig_out, power_iters, sets,
                                                              iters, d2_lim, mask_stride);
}

// -------------------------------------------------------------------------------------------------
// one CTA per set: pick the best hypothesis, write the labels, run the reweighted-Kabsch refinement
// -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kRefThreads) select_refine_kernel(
    const float* __restrict__ src, const float* __restrict__ tgt, const float* __restrict__ seed_trans,
    const unsigned long long* __restrict__ best_key, float* __restrict__ final_trans, float* __restrict__ final_labels,
    float* __restrict__ init_trans_out, int32_t* __restrict__ best_out, int32_t* __restrict__ refine_solves, const SetDesc* __restrict__ sets,
    float thr, float rthr, int max_refine) {
  __shared__ float T[12];
  __shared__ double red[(kRefThreads / 32) * 10];
  __shared__ double tot[10];
  const int b = blockIdx.x, tid = threadIdx.x;
  const SetDesc d = sets[b];
  const int N = d.N, S = d.S;
  const float* ps = src + (size_t)d.row0 * 3;
  const float* pt = tgt + (size_t)d.row0 * 3;

  int best = 0;
  if (S > 0) {
    best = (int)(0xFFFFFFFFu - (unsigned)(best_key[b] & 0xFFFFFFFFull));
    best = min(max(best, 0), S - 1);
  }
  if (tid < 12) T[tid] = (S > 0) ? seed_trans[((size_t)d.seed0 + best) * 16 + tid] : ((tid % 5 == 0) ? 1.f : 0.f);
  __syncthreads();
  if (tid < 16 && init_trans_out) init_trans_out[(size_t)b * 16 + tid] = (tid < 12) ? T[tid] : (tid == 15 ? 1.f : 0.f);
  if (tid == 0 && best_out) best_out[b] = best;

  // final_labels: inlier mask of the selected hypothesis BEFORE refinement (PointDSC.py:333-335)
  // (non-testing mode returns the confidence logits instead, PointDSC.py:190-191: final_labels is null there)
  for (int j = tid; final_labels && j < N; j += kRefThreads) {
    const float r = residual(T, ps[(size_t)j * 3], ps[(size_t)j * 3 + 1], ps[(size_t)j * 3 + 2], pt[(size_t)j * 3],
                             pt[(size_t)j * 3 + 1], pt[(size_t)j * 3 + 2]);
    final_labels[(size_t)d.row0 + j] = (r < thr) ? 1.0f : 0.0f;
  }

  long long prev = 0;
  int solves = 0;
  for (int it = 0; it < max_refine; ++it) {
    // the inliers of the current transform, weighted 1/(1+(d/tau)^2)
    auto weight = [&](int, float ax, float ay, float az, float bx, float by, float bz, float& w) {
      const float d = residual(T, ax, ay, az, bx, by, bz);
      if (!(d < rthr)) return false;
      const float q = d / rthr;
      w = 1.0f / (1.0f + q * q);
      return true;
    };
    kabsch_centroid_sums(ps, pt, N, weight, red, tot);
    const long long cnt = (long long)(tot[0] + 0.5);
    if (cnt == prev) break;  // inlier count unchanged (PointDSC.py:426); uniform across the CTA
    prev = cnt;
    const float den = (float)tot[1] + 1e-6f;
    const float cax = (float)tot[2] / den, cay = (float)tot[3] / den, caz = (float)tot[4] / den;
    const float cbx = (float)tot[5] / den, cby = (float)tot[6] / den, cbz = (float)tot[7] / den;
    __syncthreads();  // everyone has read tot[] before pass 2 overwrites it
    kabsch_solve(ps, pt, N, weight, cax, cay, caz, cbx, cby, cbz, red, tot, T);
    ++solves;
    __syncthreads();
  }
  if (tid < 16) final_trans[(size_t)b * 16 + tid] = (tid < 12) ? T[tid] : (tid == 15 ? 1.f : 0.f);
  if (tid == 0 && refine_solves) refine_solves[b] = solves;
}

void launch_select_refine(const float* src, const float* tgt, const float* seed_trans,
                          const unsigned long long* best_key, float* final_trans, float* final_labels,
                          float* init_trans_out, int32_t* best_out, int32_t* refine_solves, int B, int N, int S,
                          float inlier_threshold, float refine_threshold, int max_refine, cudaStream_t st,
                          const SetDesc* sets) {
  select_refine_kernel<<<B, kRefThreads, 0, st>>>(src, tgt, seed_trans, best_key, final_trans, final_labels,
                                                  init_trans_out, best_out, refine_solves, sets, inlier_threshold,
                                                  refine_threshold, max_refine);
}

}  // namespace pdsc
