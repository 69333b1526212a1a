// The N-row weighted Kabsch of one set, run by one CTA of kRefThreads threads: rigid_transform_3d (models/common.py:7-45),
// unscaled, with the weights a caller's functor gives each row.  The refinement (select_refine.cu, models/PointDSC.py:403-438)
// weighs the rows within its threshold of the current transform; the spectral-matching baseline (spectral_matching.cu) weighs
// every row by its eigenvector entry times its label.
//
// weight(j, ax, ay, az, bx, by, bz, w) returns whether row j takes part and sets its weight w.  Every sum is a per-thread
// double accumulation over rows j = tid, tid + kRefThreads, ..., a warp tree and the warps in ascending order: a fixed order
// that depends on N only.  Pass 1 gives tot = {rows taking part, sum w, sum w a (3), sum w b (3)}; the centroids divide by
// (float) sum w + 1e-6 (common.py:24-25); pass 2 gives H = Am^T diag(w) Bm (common.py:33), solved in fp32 by svd3.cuh.
#pragma once
#include "common.cuh"
#include "svd3.cuh"

namespace pdsc {

constexpr int kRefThreads = 512;

template <int NV>
__device__ __forceinline__ void block_sum(double (&vals)[NV], double* red /* [16][NV] */, double* out /* [NV] */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < NV; ++i) vals[i] = warp_sum(vals[i]);
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) red[warp * NV + i] = vals[i];
  }
  __syncthreads();
  if (threadIdx.x < NV) {
    double acc = 0.0;
    for (int w = 0; w < kRefThreads / 32; ++w) acc += red[w * NV + threadIdx.x];
    out[threadIdx.x] = acc;
  }
  __syncthreads();
}

// pass 1: tot[0..7] = {rows taking part, sum w, sum w ax, w ay, w az, w bx, w by, w bz}
template <typename Weight>
__device__ __forceinline__ void kabsch_centroid_sums(const float* ps, const float* pt, int N, Weight weight, double* red,
                                                     double* tot) {
  double acc1[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc1[i] = 0.0;
  for (int j = threadIdx.x; j < N; j += kRefThreads) {
    const float ax = ps[(size_t)j * 3], ay = ps[(size_t)j * 3 + 1], az = ps[(size_t)j * 3 + 2];
    const float bx = pt[(size_t)j * 3], by = pt[(size_t)j * 3 + 1], bz = pt[(size_t)j * 3 + 2];
    float w;
    if (weight(j, ax, ay, az, bx, by, bz, w)) {
      acc1[0] += 1.0; acc1[1] += (double)w;
      acc1[2] += (double)(ax * w); acc1[3] += (double)(ay * w); acc1[4] += (double)(az * w);
      acc1[5] += (double)(bx * w); acc1[6] += (double)(by * w); acc1[7] += (double)(bz * w);
    }
  }
  block_sum<8>(acc1, red, tot);
}

// pass 2 over the same rows and weights, with the centroids of pass 1's tot; thread 0 writes [R | t] (row-major 3 x 4) to T.
// Every thread must have read tot before the call: it is overwritten.
template <typename Weight>
__device__ __forceinline__ void kabsch_solve(const float* ps, const float* pt, int N, Weight weight, float cax, float cay,
                                             float caz, float cbx, float cby, float cbz, double* red, double* tot, float* T) {
  double acc2[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) acc2[i] = 0.0;
  for (int j = threadIdx.x; j < N; j += kRefThreads) {
    const float ax = ps[(size_t)j * 3], ay = ps[(size_t)j * 3 + 1], az = ps[(size_t)j * 3 + 2];
    const float bx = pt[(size_t)j * 3], by = pt[(size_t)j * 3 + 1], bz = pt[(size_t)j * 3 + 2];
    float w;
    if (weight(j, ax, ay, az, bx, by, bz, w)) {
      const float mx = ax - cax, my = ay - cay, mz = az - caz;
      const float nx = (bx - cbx) * w, ny = (by - cby) * w, nz = (bz - cbz) * w;
      acc2[0] += (double)(mx * nx); acc2[1] += (double)(mx * ny); acc2[2] += (double)(mx * nz);
      acc2[3] += (double)(my * nx); acc2[4] += (double)(my * ny); acc2[5] += (double)(my * nz);
      acc2[6] += (double)(mz * nx); acc2[7] += (double)(mz * ny); acc2[8] += (double)(mz * nz);
    }
  }
  block_sum<9>(acc2, red, tot);
  if (threadIdx.x == 0) {
    float H[9], R[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) H[i] = (float)tot[i];
    kabsch_rotation(H, R);
    T[0] = R[0]; T[1] = R[1]; T[2] = R[2];  T[3] = cbx - (R[0] * cax + R[1] * cay + R[2] * caz);
    T[4] = R[3]; T[5] = R[4]; T[6] = R[5];  T[7] = cby - (R[3] * cax + R[4] * cay + R[5] * caz);
    T[8] = R[6]; T[9] = R[7]; T[10] = R[8]; T[11] = cbz - (R[6] * cax + R[7] * cay + R[8] * caz);
  }
}

}  // namespace pdsc
