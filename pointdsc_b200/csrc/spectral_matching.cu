// The classical spectral-matching baseline SM (baseline_scripts/baseline_3DMatch.py:19-53), for a group of sets of different
// sizes in one call.
//
// Semantics.  A set of N rows c_i = corr_pos row i [6] (the centred source xyz, then the centred target xyz), src / tgt its key
// points [N,3], tau the inlier threshold:
//   1. M_ij = ||c_j[0:3] - c_i[0:3]|| - ||c_j[3:6] - c_i[3:6]||, then M_ij = max(0, 4.5 - M_ij^2 / 2 / sigma^2) with
//      sigma = tau / 3, and M_ii = 0 (:20-37).  Here: the three squared differences summed left to right, a correctly rounded
//      square root, and M_ij^2 times the fp32 rounding of 1 / (2 sigma^2) = 4.5 / tau^2, every operation rounded on its own
//      (no contraction), so that a host restatement in fp32 reproduces each entry bit for bit.
//   2. v = 1; exactly ten times v <- M v / (||M v|| + 1e-6), no early exit (:40-44).
//   3. S = int(N * 0.1) (num_seeds(N, 0.1), the slice length Python takes); labels = 1 on the first S rows of v sorted
//      descending, 0 elsewhere (:47-49).  Ties: the lowest row first (seeds.cu's a6' sort: the reference's argsort is unstable,
//      so any order of tied entries is a valid reference output).
//   4. T = rigid_transform_3d(src, tgt, v * labels) (models/common.py:7-45): unscaled and weighted, centroids over
//      sum w + 1e-6, H = Am^T diag(w) Bm, R from svd3.cuh with the det(V U^T) fix, t = cb - R ca.  A set with S = 0 (N < 10)
//      or with all-zero weights has H = 0: the solver returns R = I and the centroids are 0, so T is the identity.
// Everything in fp32, as in the reference; the Kabsch sums accumulate in double (weighted_kabsch.cuh).
//
// M is never stored (a stored M would take 4 sum N_b^2 bytes: 1 GB for one set of 16,384 rows).  Each iteration recomputes it:
//   power kernel  grid (row block, set), 256 threads; warp w owns RW consecutive rows of the block (RW = 4, 2 or 1, chosen on the
//                 host so that the call covers the SMs twice over; a set's result does not depend on it).  The set's rows and v
//                 are staged through shared memory kSmTile columns at a time; lane l accumulates columns j = l mod 32 in
//                 ascending order with one fma each, and a row's 32 lane sums are combined by the xor-shuffle tree of warp_sum.
//                 Writes u = M v.  The first iteration reads no v (v = 1).
//   norm kernel   one CTA per set: sum u^2 in a fixed order (thread-strided, warp tree, warps in ascending order), then
//                 v = u / (sqrt(sum) + 1e-6) in place.  The first launch also writes the set table the sort reads.
//   top-S sort    launch_top_seeds (seeds.cu), one CTA per set.
//   Kabsch        one CTA per set: marks the S selected rows, writes labels and the eigenvector, runs weighted_kabsch.cuh.
// 22 launches whatever B; no host synchronisation, no allocation, capturable in a CUDA graph.  Every sum's order depends on the
// set's N only, so a set's outputs are bit for bit the same in any group, in any order, on any SM count.
//
// Cost.  Per entry and iteration: 6 differences, 6 products, 4 additions, 2 square roots, 5 more operations and the fma: about
// 24 FP32 instructions plus the two square-root sequences, 10 N^2 entries per set.
#include <math.h>

#include "common.cuh"
#include "kernels.h"
#include "sets.cuh"
#include "weighted_kabsch.cuh"

namespace pdsc {

namespace {
constexpr int kSmThreads = 256;
constexpr int kSmWarps = kSmThreads / 32;
constexpr int kSmTile = 512;               // columns staged per pass (14 KB)
constexpr int kSmIterations = 10;          // baseline_3DMatch.py:41
constexpr double kSmTopRatio = 0.1;        // top_ratio, baseline_3DMatch.py:19
constexpr int kSmMaxN = 16384;             // the a6' sort's limit (seeds.cu)

__host__ __device__ inline size_t align16(size_t x) { return (x + 15) / 16 * 16; }

struct SmScratch {
  SetDesc* sets;   // [B]
  float* a;        // [R]  u / v of the odd iterations
  float* b;        // [R]  u / v of the even iterations
  int32_t* seeds;  // [R]  set b's sorted rows from row0 (seed0 = row0, S <= N)
};

SmScratch sm_carve(void* scratch, long long R, int B) {
  unsigned char* p = static_cast<unsigned char*>(scratch);
  SmScratch s;
  s.sets = reinterpret_cast<SetDesc*>(p);  p += align16((size_t)B * sizeof(SetDesc));
  s.a = reinterpret_cast<float*>(p);       p += align16((size_t)R * 4);
  s.b = reinterpret_cast<float*>(p);       p += align16((size_t)R * 4);
  s.seeds = reinterpret_cast<int32_t*>(p);
  return s;
}

// M_ij of step 1 from row i (xi) and row j (xj); the caller zeroes the diagonal
__device__ __forceinline__ float sm_entry(const float (&xi)[6], float x0, float x1, float x2, float x3, float x4, float x5,
                                          float coef) {
  const float ax = __fsub_rn(x0, xi[0]), ay = __fsub_rn(x1, xi[1]), az = __fsub_rn(x2, xi[2]);
  const float bx = __fsub_rn(x3, xi[3]), by = __fsub_rn(x4, xi[4]), bz = __fsub_rn(x5, xi[5]);
  const float ds = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(ax, ax), __fmul_rn(ay, ay)), __fmul_rn(az, az)));
  const float dt = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(bx, bx), __fmul_rn(by, by)), __fmul_rn(bz, bz)));
  const float m = __fsub_rn(ds, dt);
  return fmaxf(__fsub_rn(4.5f, __fmul_rn(__fmul_rn(m, m), coef)), 0.0f);
}
}  // namespace

template <int RW>
__global__ void __launch_bounds__(kSmThreads) sm_power_kernel(const float* __restrict__ corr, Offsets off, const float* __restrict__ v,
                                                              float* __restrict__ u, float coef) {
  __shared__ __align__(16) float cs[7][kSmTile];
  const int b = blockIdx.y;
  const int row0 = off.at(b), N = off.at(b + 1) - row0;
  const int r0 = blockIdx.x * (kSmWarps * RW);
  if (r0 >= N) return;                       // the grid is sized by the largest set: the whole CTA leaves
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* c = corr + (size_t)row0 * 6;
  float xi[RW][6], acc[RW];
  int ri[RW];
#pragma unroll
  for (int q = 0; q < RW; ++q) {
    ri[q] = r0 + warp * RW + q;
    const int rc = min(ri[q], N - 1);
#pragma unroll
    for (int k = 0; k < 6; ++k) xi[q][k] = c[(size_t)rc * 6 + k];
    acc[q] = 0.0f;
  }
  for (int j0 = 0; j0 < N; j0 += kSmTile) {
    const int n = min(kSmTile, N - j0);
    __syncthreads();                         // the previous tile has been read by every warp
    for (int f = tid; f < 6 * n; f += kSmThreads) {
      const int k = f / 6;
      cs[f - 6 * k][k] = c[(size_t)j0 * 6 + f];
    }
    for (int k = tid; k < n; k += kSmThreads) cs[6][k] = v ? v[(size_t)row0 + j0 + k] : 1.0f;
    __syncthreads();
    for (int k = lane; k < n; k += 32) {
      const float x0 = cs[0][k], x1 = cs[1][k], x2 = cs[2][k], x3 = cs[3][k], x4 = cs[4][k], x5 = cs[5][k], vj = cs[6][k];
#pragma unroll
      for (int q = 0; q < RW; ++q) {
        const float m = (j0 + k == ri[q]) ? 0.0f : sm_entry(xi[q], x0, x1, x2, x3, x4, x5, coef);
        acc[q] = __fmaf_rn(m, vj, acc[q]);
      }
    }
  }
#pragma unroll
  for (int q = 0; q < RW; ++q) {
    const float s = warp_sum(acc[q]);
    if (lane == 0 && ri[q] < N) u[(size_t)row0 + ri[q]] = s;
  }
}

__global__ void __launch_bounds__(kSmThreads) sm_norm_kernel(float* __restrict__ u, Offsets off, SetDesc* __restrict__ sets) {
  __shared__ float part[kSmWarps];
  __shared__ float den_s;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int row0 = off.at(b), N = off.at(b + 1) - row0;
  float* ub = u + row0;
  float ss = 0.0f;
  for (int j = tid; j < N; j += kSmThreads) ss = __fmaf_rn(ub[j], ub[j], ss);
  ss = warp_sum(ss);
  if (lane == 0) part[warp] = ss;
  __syncthreads();
  if (tid == 0) {
    float t = 0.0f;
    for (int w = 0; w < kSmWarps; ++w) t = __fadd_rn(t, part[w]);
    den_s = __fadd_rn(__fsqrt_rn(t), 1e-6f);
    if (sets) {                              // the table launch_top_seeds reads: S = int(N * 0.1), seeds from row0
      SetDesc d = {};
      d.row0 = row0;
      d.N = N;
      d.S = num_seeds(N, kSmTopRatio);
      d.seed0 = row0;
      sets[b] = d;
    }
  }
  __syncthreads();
  const float den = den_s;
  for (int j = tid; j < N; j += kSmThreads) ub[j] = __fdiv_rn(ub[j], den);
}

__global__ void __launch_bounds__(kRefThreads) sm_kabsch_kernel(const float* __restrict__ src, const float* __restrict__ tgt,
                                                                const float* __restrict__ v, const int32_t* __restrict__ seeds,
                                                                Offsets off, float* __restrict__ trans, float* __restrict__ labels,
                                                                float* __restrict__ eig_out) {
  __shared__ unsigned char sel[kSmMaxN];
  __shared__ float T[12];
  __shared__ double red[(kRefThreads / 32) * 10];
  __shared__ double tot[10];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int row0 = off.at(b), N = off.at(b + 1) - row0;
  const int S = num_seeds(N, kSmTopRatio);
  const float* vb = v + row0;
  for (int j = tid; j < N; j += kRefThreads) sel[j] = 0;
  __syncthreads();
  for (int i = tid; i < S; i += kRefThreads) sel[seeds[(size_t)row0 + i]] = 1;
  __syncthreads();
  for (int j = tid; j < N; j += kRefThreads) {
    labels[(size_t)row0 + j] = sel[j] ? 1.0f : 0.0f;
    if (eig_out) eig_out[(size_t)row0 + j] = vb[j];
  }
  // weights = leading_eig * pred_labels (baseline_3DMatch.py:52); every row takes part, as in the reference's sums
  auto weight = [&](int j, float, float, float, float, float, float, float& w) {
    w = vb[j] * (sel[j] ? 1.0f : 0.0f);
    return true;
  };
  const float* ps = src + (size_t)row0 * 3;
  const float* pt = tgt + (size_t)row0 * 3;
  kabsch_centroid_sums(ps, pt, N, weight, red, tot);
  const float den = (float)tot[1] + 1e-6f;
  const float cax = (float)tot[2] / den, cay = (float)tot[3] / den, caz = (float)tot[4] / den;
  const float cbx = (float)tot[5] / den, cby = (float)tot[6] / den, cbz = (float)tot[7] / den;
  __syncthreads();                           // everyone has read tot[] before pass 2 overwrites it
  kabsch_solve(ps, pt, N, weight, cax, cay, caz, cbx, cby, cbz, red, tot, T);
  __syncthreads();
  if (tid < 16) trans[(size_t)b * 16 + tid] = (tid < 12) ? T[tid] : (tid == 15 ? 1.0f : 0.0f);
}

int spectral_matching_max_n() { return kSmMaxN; }

size_t sm_scratch_bytes(long long R, int B) {
  return align16((size_t)B * sizeof(SetDesc)) + 2 * align16((size_t)R * 4) + (size_t)R * 4;
}

void launch_spectral_matching(int B, const int32_t* h_off, const int32_t* d_off, const float* corr, const float* src, const float* tgt,
                              double inlier_threshold, float* trans, float* labels, float* eig_out, void* scratch, cudaStream_t st) {
  const long long R = h_off[B];
  int Nmax = 0;
  for (int b = 0; b < B; ++b) Nmax = max(Nmax, h_off[b + 1] - h_off[b]);
  const Offsets off{d_off, 0};
  const SmScratch s = sm_carve(scratch, R, B);
  const float coef = (float)(4.5 / (inlier_threshold * inlier_threshold));     // 1 / (2 sigma^2), sigma = tau / 3
  // rows per warp: the most that still gives two CTAs per SM over the call's sets
  const long long want = 2LL * device_sm_count();
  auto ctas = [&](int rows) {
    long long n = 0;
    for (int b = 0; b < B; ++b) n += (h_off[b + 1] - h_off[b] + rows - 1) / rows;
    return n;
  };
  const int RW = ctas(kSmWarps * 4) >= want ? 4 : (ctas(kSmWarps * 2) >= want ? 2 : 1);
  const dim3 grid((unsigned)((Nmax + kSmWarps * RW - 1) / (kSmWarps * RW)), (unsigned)B);
  const float* vin = nullptr;
  float* bufs[2] = {s.a, s.b};
  for (int t = 0; t < kSmIterations; ++t) {
    float* uo = bufs[t & 1];
    if (RW == 4) sm_power_kernel<4><<<grid, kSmThreads, 0, st>>>(corr, off, vin, uo, coef);
    else if (RW == 2) sm_power_kernel<2><<<grid, kSmThreads, 0, st>>>(corr, off, vin, uo, coef);
    else sm_power_kernel<1><<<grid, kSmThreads, 0, st>>>(corr, off, vin, uo, coef);
    sm_norm_kernel<<<B, kSmThreads, 0, st>>>(uo, off, t == 0 ? s.sets : nullptr);
    vin = uo;
  }
  launch_top_seeds(vin, s.seeds, B, Nmax, num_seeds(Nmax, kSmTopRatio), st, s.sets);
  sm_kabsch_kernel<<<B, kRefThreads, 0, st>>>(src, tgt, vin, s.seeds, off, trans, labels, eig_out);
}

}  // namespace pdsc
