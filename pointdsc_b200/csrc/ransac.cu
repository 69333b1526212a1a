// Correspondence RANSAC over the pairs the network kept, for the drivers' --solver RANSAC (evaluation/test_3DMatch.py:59-77,
// test_KITTI.py:59-77, which hand the rows with pred_labels > 0 to open3d 0.9's registration_ransac_based_on_correspondence with
// ransac_n = 3, max_iteration = max_validation = 5000 and no checkers; its inliers replace pred_labels, its transform pred_trans).
//
// Semantics (restated on the CPU by the restatement under oracle/, which names what is recalled from open3d rather than checked).
// The candidates of a set are its rows with label > 0, in ascending row order; M their number.  M < 3: the identity, all-zero
// labels, status 1.  Iteration i < max_iteration draws three candidates with repeats, draw j at index (z >> 33) % M where z is
// SplitMix64 of seed + (3 i + j + 1) * 0x9E3779B97F4A7C15 (open3d seeds rand() from the clock; these draws depend on (seed, i, j)
// only), and solves the unscaled Umeyama over them in double (means, demeaned covariance, svd3.cuh's Jacobi Kabsch,
// t = b - R a).  A sample with a non-finite coordinate scores good = 0.  Scoring walks the M candidates in order:
// d^2 = |R p + t - q|^2 in double, an inlier iff d^2 < r * r (a double product), good = inliers, rmse = sqrt(sum d^2 / good) (0 when
// good = 0).  Hypothesis i replaces the best iff it has more inliers, or as many and a smaller rmse (open3d's fitness / rmse rule):
// the winner is the least key (-good, rmse, i) among good > 0, a total order.  No hypothesis with good > 0: the identity, all-zero
// labels, status 2.  Else trans = the winner's own 3-point solve (no refit), labels = 1 on exactly its inliers, 0 elsewhere.
//
// Sets.  B sets packed back to back, set b owning rows [off[b], off[b+1]).  Draws and every sum depend on the set's own rows
// only, reductions are over a total order, so a set's result is bit for bit the same whatever else its call holds, in any order, on
// any SM count.  Three launches, no host synchronisation, no allocation, capturable in a CUDA graph.
//
// Grid.  (1) candidates: one CTA per set compacts its label > 0 rows by a block scan and writes M_b and their coordinates,
// widened to double, contiguously into the set's scratch region.  (2) scoring: grid (hypothesis chunk, set), one thread per
// hypothesis: it draws and solves, then walks the candidates through shared-memory tiles that every thread reads in the same
// order (broadcast), and writes its key.  A chunk is kRansacChunk = 128 hypotheses (four warps, 40 CTAs for the drivers' 5,000
// hypotheses of one set).  Chosen from calls at batch size 1 (N = 1,000 / 5,000 / 12,000) and in groups of 8 and 64 sets on an
// H100 SXM at 700 W (DESIGN.md §4): 32 and 256 were slower than 64 and 128 at most sizes, and 128 was as fast as 64 or faster
// at every size, within the spread between runs.  CTAs of a set with M < 3 exit at once.  (3) finish: one CTA per set selects the winner, re-solves it with the same (non-inlined) device function,
// so its T is bit-identical to the one scored, and writes the outputs.  When asked for every hypothesis's transform (hyp_trans,
// a test output) it re-solves each iteration with that same function, so each [R | t] is the one its key was scored with.
//
// Cost.  max_iteration * M distance tests per set, about 27 fp64 operations each, plus one 3x3 Jacobi solve per hypothesis.
#include <math.h>

#include <cmath>

#include "abi.h"
#include "common.cuh"
#include "kernels.h"
#include "sets.cuh"
#include "svd3.cuh"

namespace pdsc {

namespace {
#ifndef PDSC_RANSAC_CHUNK
#define PDSC_RANSAC_CHUNK 128
#endif
constexpr int kRansacChunk = PDSC_RANSAC_CHUNK;   // hypotheses (threads) per scoring CTA
constexpr int kRansacTile = 256;                  // candidates per shared-memory tile of the scoring kernel
constexpr int kRansacThreads = 256;               // candidates and finish kernels
constexpr int kRansacWarps = kRansacThreads / 32;
constexpr int kRansacMaxSets = 65535;             // the scoring kernel's sets are its grid's y dimension

// set b's region: candidates [row0, row0 + M_b) as 6 doubles (source x y z, target x y z); keys [b * max_iteration, ...)
struct RansacScratch {
  double* cand;    // [R][6]
  double* rmse;    // [B * max_iteration]
  int* good;       // [B * max_iteration]
  int* row;        // [R]  set-local row of every candidate
  int* M;          // [B]
};

__host__ __device__ inline size_t align16(size_t x) { return (x + 15) / 16 * 16; }

RansacScratch ransac_carve(void* scratch, long long R, int B, int max_iteration) {
  unsigned char* p = static_cast<unsigned char*>(scratch);
  const size_t keys = (size_t)B * (size_t)max_iteration;
  RansacScratch s;
  s.cand = reinterpret_cast<double*>(p);  p += align16((size_t)R * 48);
  s.rmse = reinterpret_cast<double*>(p);  p += align16(keys * 8);
  s.good = reinterpret_cast<int*>(p);     p += align16(keys * 4);
  s.row = reinterpret_cast<int*>(p);      p += align16((size_t)R * 4);
  s.M = reinterpret_cast<int*>(p);
  return s;
}

// draw j of iteration i: SplitMix64 of seed + (3 i + j + 1) * golden, its top 31 bits modulo M
__device__ __forceinline__ int ransac_draw(unsigned long long seed, int i, int j, int M) {
  unsigned long long z = seed + (3ull * (unsigned long long)i + (unsigned long long)j + 1ull) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (int)((z >> 33) % (unsigned long long)M);
}

struct Rigid {
  double R[9], t[3];
  int ok;          // 0: a drawn candidate has a non-finite coordinate
};

// The hypothesis of iteration i: the unscaled Umeyama solve over its three drawn candidates.  Not inlined, so that the scoring
// and the finish kernel run the same instructions and the winner's T is the one that was scored, bit for bit.
__device__ __noinline__ Rigid ransac_solve(const double* __restrict__ cand, unsigned long long seed, int i, int M) {
  double a[3][3], b[3][3];
  bool finite = true;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const double* c = cand + 6 * (size_t)ransac_draw(seed, i, j, M);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      a[j][k] = c[k];
      b[j][k] = c[3 + k];
      finite = finite && isfinite(a[j][k]) && isfinite(b[j][k]);
    }
  }
  Rigid h;
  h.ok = finite;
  if (!finite) {
#pragma unroll
    for (int k = 0; k < 9; ++k) h.R[k] = (k % 4 == 0) ? 1.0 : 0.0;
    h.t[0] = h.t[1] = h.t[2] = 0.0;
    return h;
  }
  double am[3], bm[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    am[k] = __ddiv_rn(__dadd_rn(__dadd_rn(a[0][k], a[1][k]), a[2][k]), 3.0);
    bm[k] = __ddiv_rn(__dadd_rn(__dadd_rn(b[0][k], b[1][k]), b[2][k]), 3.0);
  }
  double H[9];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      double acc = 0.0;
#pragma unroll
      for (int j = 0; j < 3; ++j) acc = __fma_rn(__dsub_rn(a[j][r], am[r]), __dsub_rn(b[j][c], bm[c]), acc);
      H[3 * r + c] = acc;
    }
  kabsch_rotation(H, h.R);
#pragma unroll
  for (int r = 0; r < 3; ++r)
    h.t[r] = __dsub_rn(bm[r], __fma_rn(h.R[3 * r], am[0], __fma_rn(h.R[3 * r + 1], am[1], __dmul_rn(h.R[3 * r + 2], am[2]))));
  return h;
}

// d^2 = |R p + t - q|^2, every rounding pinned so that the scoring and the finish kernel decide each candidate alike
__device__ __forceinline__ double ransac_d2(const double* R, const double* t, const double* c) {
  const double x = __fma_rn(R[0], c[0], __fma_rn(R[1], c[1], __fma_rn(R[2], c[2], t[0])));
  const double y = __fma_rn(R[3], c[0], __fma_rn(R[4], c[1], __fma_rn(R[5], c[2], t[1])));
  const double z = __fma_rn(R[6], c[0], __fma_rn(R[7], c[1], __fma_rn(R[8], c[2], t[2])));
  const double ex = __dsub_rn(x, c[3]), ey = __dsub_rn(y, c[4]), ez = __dsub_rn(z, c[5]);
  return __fma_rn(ex, ex, __fma_rn(ey, ey, __dmul_rn(ez, ez)));
}

// [R | t] row-major, the layout of the winner's T below
__device__ __forceinline__ void store_rigid(double* out, const Rigid& h) {
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    out[4 * r] = h.R[3 * r]; out[4 * r + 1] = h.R[3 * r + 1]; out[4 * r + 2] = h.R[3 * r + 2]; out[4 * r + 3] = h.t[r];
  }
}

// key a ranks before key b: more inliers, then smaller rmse, then earlier iteration
__device__ __forceinline__ bool key_before(int ga, double ra, int ia, int gb, double rb, int ib) {
  return ga > gb || (ga == gb && (ra < rb || (ra == rb && ia < ib)));
}
}  // namespace

size_t ransac_scratch_bytes(long long R, int B, int max_iteration) {
  const size_t keys = (size_t)B * (size_t)max_iteration;
  return align16((size_t)R * 48) + align16(keys * 8) + align16(keys * 4) + align16((size_t)R * 4) + (size_t)B * 4;
}

__global__ void __launch_bounds__(kRansacThreads) ransac_candidates_kernel(const float* __restrict__ src, const float* __restrict__ tgt,
                                                                           const float* __restrict__ labels, Offsets off,
                                                                           RansacScratch s) {
  __shared__ int warp_count[kRansacWarps];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int row0 = off.at(b), N = off.at(b + 1) - row0;
  double* cand = s.cand + 6 * (size_t)row0;
  int* rows = s.row + row0;
  int base = 0;
  for (int c0 = 0; c0 < N; c0 += kRansacThreads) {
    const int j = c0 + tid;
    const bool keep = j < N && labels[row0 + j] > 0.0f;
    const unsigned ballot = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_count[warp] = __popc(ballot);
    __syncthreads();
    int before = base, total = base;
#pragma unroll
    for (int w = 0; w < kRansacWarps; ++w) {
      before += w < warp ? warp_count[w] : 0;
      total += warp_count[w];
    }
    if (keep) {
      const int k = before + __popc(ballot & ((1u << lane) - 1u));
      const size_t r = (size_t)(row0 + j) * 3;
      double* d = cand + 6 * (size_t)k;
      d[0] = (double)src[r]; d[1] = (double)src[r + 1]; d[2] = (double)src[r + 2];
      d[3] = (double)tgt[r]; d[4] = (double)tgt[r + 1]; d[5] = (double)tgt[r + 2];
      rows[k] = j;
    }
    base = total;
    __syncthreads();     // warp_count is rewritten by the next chunk
  }
  if (tid == 0) s.M[b] = base;
}

__global__ void __launch_bounds__(kRansacChunk) ransac_score_kernel(Offsets off, double r2, int max_iteration,
                                                                    unsigned long long seed, RansacScratch s) {
  __shared__ __align__(16) double tile[kRansacTile * 6];
  const int b = blockIdx.y, tid = threadIdx.x;
  const int M = s.M[b];
  if (M < 3) return;
  const int i = blockIdx.x * kRansacChunk + tid;
  const double* cand = s.cand + 6 * (size_t)off.at(b);
  Rigid h;
  h.ok = 0;
  if (i < max_iteration) h = ransac_solve(cand, seed, i, M);
  int good = 0;
  double sum = 0.0;
  for (int k0 = 0; k0 < M; k0 += kRansacTile) {
    const int n = min(kRansacTile, M - k0);
    const double2* g = reinterpret_cast<const double2*>(cand + 6 * (size_t)k0);
    double2* t2 = reinterpret_cast<double2*>(tile);
    for (int q = tid; q < 3 * n; q += kRansacChunk) t2[q] = g[q];
    __syncthreads();
    if (h.ok) {
      for (int k = 0; k < n; ++k) {
        const double d2 = ransac_d2(h.R, h.t, tile + 6 * k);
        if (d2 < r2) {
          ++good;
          sum = __dadd_rn(sum, d2);
        }
      }
    }
    __syncthreads();
  }
  if (i < max_iteration) {
    const size_t key = (size_t)b * (size_t)max_iteration + (size_t)i;
    s.good[key] = good;
    s.rmse[key] = good > 0 ? __dsqrt_rn(__ddiv_rn(sum, (double)good)) : 0.0;
  }
}

__global__ void __launch_bounds__(kRansacThreads) ransac_finish_kernel(const float* __restrict__ labels, Offsets off, double r2,
                                                                       int max_iteration, unsigned long long seed, RansacScratch s,
                                                                       float* __restrict__ trans, float* __restrict__ out_labels,
                                                                       double* __restrict__ fitness_out, double* __restrict__ rmse_out,
                                                                       int32_t* __restrict__ best_out, int32_t* __restrict__ status_out,
                                                                       int32_t* __restrict__ hyp_good, double* __restrict__ hyp_rmse,
                                                                       double* __restrict__ hyp_trans) {
  __shared__ int wg[kRansacWarps], wi[kRansacWarps];
  __shared__ double wr[kRansacWarps];
  __shared__ double T[12];
  __shared__ int win;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int row0 = off.at(b), N = off.at(b + 1) - row0;
  const int M = s.M[b];
  const size_t k0 = (size_t)b * (size_t)max_iteration;
  const double* cand = s.cand + 6 * (size_t)row0;

  // ---- the winner: the least key (-good, rmse, i) among good > 0; -1 when there is none ----
  int bg = 0, bi = -1;
  double br = 0.0;
  if (M >= 3) {
    for (int i = tid; i < max_iteration; i += kRansacThreads) {
      const int g = s.good[k0 + i];
      const double r = s.rmse[k0 + i];
      if (hyp_good) hyp_good[k0 + i] = g;
      if (hyp_rmse) hyp_rmse[k0 + i] = r;
      if (hyp_trans) store_rigid(hyp_trans + 12 * (k0 + i), ransac_solve(cand, seed, i, M));
      if (g > 0 && (bi < 0 || key_before(g, r, i, bg, br, bi))) { bg = g; br = r; bi = i; }
    }
  } else {
    for (int i = tid; i < max_iteration; i += kRansacThreads) {
      if (hyp_good) hyp_good[k0 + i] = 0;
      if (hyp_rmse) hyp_rmse[k0 + i] = 0.0;
      if (hyp_trans)
        for (int k = 0; k < 12; ++k) hyp_trans[12 * (k0 + i) + k] = (k % 5 == 0) ? 1.0 : 0.0;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const int g = __shfl_xor_sync(0xffffffffu, bg, o), i = __shfl_xor_sync(0xffffffffu, bi, o);
    const double r = __shfl_xor_sync(0xffffffffu, br, o);
    if (i >= 0 && (bi < 0 || key_before(g, r, i, bg, br, bi))) { bg = g; br = r; bi = i; }
  }
  if (lane == 0) { wg[warp] = bg; wr[warp] = br; wi[warp] = bi; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < kRansacWarps; ++w)
      if (wi[w] >= 0 && (bi < 0 || key_before(wg[w], wr[w], wi[w], bg, br, bi))) { bg = wg[w]; br = wr[w]; bi = wi[w]; }
    win = bi;
    if (bi >= 0) {
      store_rigid(T, ransac_solve(cand, seed, bi, M));
    } else {
      for (int k = 0; k < 12; ++k) T[k] = (k % 5 == 0) ? 1.0 : 0.0;
    }
    if (fitness_out) fitness_out[b] = bi >= 0 ? (double)bg / (double)M : 0.0;
    if (rmse_out) rmse_out[b] = bi >= 0 ? br : 0.0;
    if (best_out) best_out[b] = bi;
    if (status_out) status_out[b] = M < 3 ? 1 : (bi < 0 ? 2 : 0);
  }
  __syncthreads();
  if (tid < 16) trans[(size_t)b * 16 + tid] = tid < 12 ? (float)T[tid] : (tid == 15 ? 1.0f : 0.0f);

  // ---- labels: 1 on exactly the winner's inliers.  Rows that are not candidates are 0; candidates are decided again ----
  for (int j = tid; j < N; j += kRansacThreads)
    if (!(labels[row0 + j] > 0.0f)) out_labels[row0 + j] = 0.0f;
  const int* rows = s.row + row0;
  if (win < 0) {
    for (int k = tid; k < M; k += kRansacThreads) out_labels[row0 + rows[k]] = 0.0f;
    return;
  }
  const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]}, t[3] = {T[3], T[7], T[11]};
  for (int k = tid; k < M; k += kRansacThreads)
    out_labels[row0 + rows[k]] = ransac_d2(R, t, cand + 6 * (size_t)k) < r2 ? 1.0f : 0.0f;
}

// pdsc_ransac_packed and pdsc_ransac_packed_hypotheses: one set of checks and one launch, under the caller's name
static int ransac_packed(const char* fn, pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets,
                         const float* d_src, const float* d_tgt, const float* d_labels, double max_corr_dist, int32_t max_iteration,
                         uint64_t seed, float* d_trans, float* d_out_labels, double* d_fitness, double* d_rmse, int32_t* d_best,
                         int32_t* d_status, int32_t* d_hyp_good, double* d_hyp_rmse, double* d_hyp_trans, void* d_scratch,
                         size_t scratch_bytes, void* cuda_stream) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (int rc = check_offsets(fn, "", B, h_offsets, 1)) return rc;
  if (B > kRansacMaxSets) return fail(PDSC_ERR_UNSUPPORTED, "%s: at most %d sets per call (got %d)", fn, kRansacMaxSets, B);
  if (!d_offsets || !d_src || !d_tgt || !d_labels || !d_trans || !d_out_labels)
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: null tensor pointer", fn);
  if (!(max_corr_dist > 0.0) || !std::isfinite(max_corr_dist))
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: max_corr_dist must be positive and finite (got %g)", fn, max_corr_dist);
  if (max_iteration < 1)
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: max_iteration must be >= 1 (got %d)", fn, max_iteration);
  const long long R = h_offsets[B];
  if (int rc = check_scratch(fn, "scratch", d_scratch, scratch_bytes, ransac_scratch_bytes(R, B, max_iteration), 16)) return rc;
  DeviceGuard g(engine_config(e).device);
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  const double r2 = max_corr_dist * max_corr_dist;
  const Offsets off{d_offsets, 0};
  const RansacScratch s = ransac_carve(d_scratch, R, B, max_iteration);
  ransac_candidates_kernel<<<B, kRansacThreads, 0, st>>>(d_src, d_tgt, d_labels, off, s);
  const dim3 grid((unsigned)((max_iteration + kRansacChunk - 1) / kRansacChunk), (unsigned)B);
  ransac_score_kernel<<<grid, kRansacChunk, 0, st>>>(off, r2, max_iteration, (unsigned long long)seed, s);
  ransac_finish_kernel<<<B, kRansacThreads, 0, st>>>(d_labels, off, r2, max_iteration, (unsigned long long)seed, s, d_trans,
                                                     d_out_labels, d_fitness, d_rmse, d_best, d_status, d_hyp_good, d_hyp_rmse,
                                                     d_hyp_trans);
  PDSC_CUDA(cudaGetLastError());
  return PDSC_OK;
}

}  // namespace pdsc

// ---- C ABI ------------------------------------------------------------------------------------------------------
using namespace pdsc;

extern "C" {

size_t pdsc_ransac_packed_scratch_bytes(int32_t B, const int32_t* h_offsets, int32_t max_iteration) {
  if (check_offsets("pdsc_ransac_packed_scratch_bytes", "", B, h_offsets, 1)) return 0;
  if (max_iteration < 1) {
    fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_ransac_packed_scratch_bytes: max_iteration must be >= 1 (got %d)", max_iteration);
    return 0;
  }
  return ransac_scratch_bytes(h_offsets[B], B, max_iteration);
}

int pdsc_ransac_packed(pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets, const float* d_src,
                       const float* d_tgt, const float* d_labels, double max_corr_dist, int32_t max_iteration, uint64_t seed,
                       float* d_trans, float* d_out_labels, double* d_fitness, double* d_rmse, int32_t* d_best, int32_t* d_status,
                       int32_t* d_hyp_good, double* d_hyp_rmse, void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  return ransac_packed("pdsc_ransac_packed", e, B, h_offsets, d_offsets, d_src, d_tgt, d_labels, max_corr_dist, max_iteration, seed,
                       d_trans, d_out_labels, d_fitness, d_rmse, d_best, d_status, d_hyp_good, d_hyp_rmse, nullptr, d_scratch,
                       scratch_bytes, cuda_stream);
}

int pdsc_ransac_packed_hypotheses(pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets, const float* d_src,
                                  const float* d_tgt, const float* d_labels, double max_corr_dist, int32_t max_iteration,
                                  uint64_t seed, float* d_trans, float* d_out_labels, double* d_fitness, double* d_rmse,
                                  int32_t* d_best, int32_t* d_status, int32_t* d_hyp_good, double* d_hyp_rmse, double* d_hyp_trans,
                                  void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  return ransac_packed("pdsc_ransac_packed_hypotheses", e, B, h_offsets, d_offsets, d_src, d_tgt, d_labels, max_corr_dist,
                       max_iteration, seed, d_trans, d_out_labels, d_fitness, d_rmse, d_best, d_status, d_hyp_good, d_hyp_rmse,
                       d_hyp_trans, d_scratch, scratch_bytes, cuda_stream);
}

}  // extern "C"
