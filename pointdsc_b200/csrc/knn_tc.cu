// a7 on the tensor cores: feature-space distances of the SEED rows to all N correspondences of their set.
//
// Reference: models/common.py:58-61 (`2 - 2 * x @ x^T` over L2-normalised features) restricted to the rows gathered at
// models/PointDSC.py:252.  D[s][j] = 2 - 2 <f_seed(s), f_j>  is a [S x N x 128] GEMM per set; it runs as fp16 hi/lo split
// products (22 significant bits per operand, fp32 accumulation — the same fp32-grade arithmetic as the encoder's
// default mode) and replaces the gather + SIMT SGEMM of the exact-arithmetic path (26 MFLOP per set).
//
// One CTA = up to 128 seed rows of one set x a range of 64-key tiles, two warpgroups of 64 seed rows.  The seed rows are split
// once into register A operands (hi | lo, K = 128: 8 k-steps); per key tile all 256 threads convert the 64 fp32 key rows into
// the swizzled K-major B image (double-buffered: the next tile is converted while the MMAs of the current one run), and each
// warpgroup writes its 64 x 64 block of 2 - 2 acc straight from the accumulator registers.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "common.cuh"
#include "kernels.h"
#include "sets.cuh"
#include "tc_common.cuh"

namespace pdsc {

constexpr int kKnnThreads = 256;
constexpr int kKnnB = 0;                       // 2 stages x 32 KB: [hi p0 8K][hi p1 8K][lo p0 8K][lo p1 8K]
constexpr int kKnnSmem = 65536;

// 64 key rows of tile `kt` (fp32, rows >= N read as 0) -> swizzled hi | lo image; thread = (key row tid / 4 + 64 i / 4 ..)
__device__ __forceinline__ void knn_stage_keys(uint8_t* Bs, const float* rows, int kt, int N, int tid) {
  constexpr int FMT = kFmtF16;
  float4 v[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int kr = (tid >> 5) + 8 * i, key = kt * 64 + kr;
    v[i] = key < N ? __ldg(reinterpret_cast<const float4*>(rows + (size_t)key * kC) + (tid & 31)) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int kr = (tid >> 5) + 8 * i, lane = tid & 31;
    uint32_t h0, l0, h1, l1;
    split_pair<FMT>(v[i].x, v[i].y, h0, l0);
    split_pair<FMT>(v[i].z, v[i].w, h1, l1);
    const uint32_t off = (uint32_t)(lane >> 4) * 8192u + sw128_offset((uint32_t)kr, (uint32_t)(lane & 15) * 4u);
    *reinterpret_cast<uint2*>(Bs + off) = make_uint2(h0, h1);
    *reinterpret_cast<uint2*>(Bs + 16384 + off) = make_uint2(l0, l1);
  }
  fence_proxy_async_smem();
}

__global__ void __launch_bounds__(kKnnThreads, 1) knn_dist_tc_kernel(const float* __restrict__ normed,
                                                                     const int32_t* __restrict__ seeds,
                                                                     float* __restrict__ dist, const SetDesc* __restrict__ sets, int tiles_per_cta) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t s0 = smem_u32(smem);
  const int tid = threadIdx.x, wg = tid >> 7, wt = tid & 127;
  const int b = blockIdx.y, s_base = blockIdx.x * 128;
  const SetDesc sd = sets[b];
  const int N = sd.N, S = sd.S;
  if (s_base >= S) return;                 // the grid is sized by the largest set
  // key tiles [t0, t0 + T) of this CTA: blockIdx.z splits the keys when seed-row tiles x sets alone would leave SMs idle
  const int t0 = blockIdx.z * tiles_per_cta;
  const int T = min(tiles_per_cta, (N + 63) / 64 - t0);
  constexpr int FMT = kFmtF16;
  const float* rows = normed + (size_t)sd.row0 * kC;
  const int fr = frag_row(wt), fc = frag_col(wt);

  // A operand: this thread's fragment of its warpgroup's 64 seed rows (rows fr, fr + 8), all 128 channels
  uint32_t ahi[8][4], alo[8][4];
  int srow[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int s = s_base + 64 * wg + fr + 8 * h;
    srow[h] = s;
    const float* frow = nullptr;
    if (s < S) {
      int idx = seeds[(size_t)sd.seed0 + s];
      idx = min(max(idx, 0), N - 1);
      frow = rows + (size_t)idx * kC;
    }
#pragma unroll
    for (int ks = 0; ks < 8; ++ks)
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const float2 f = frow ? __ldg(reinterpret_cast<const float2*>(frow + 16 * ks + 8 * hf + fc)) : make_float2(0.f, 0.f);
        split_pair<FMT>(f.x, f.y, ahi[ks][2 * hf + h], alo[ks][2 * hf + h]);
      }
  }
  if (T > 0) knn_stage_keys(smem + kKnnB, rows, t0, N, tid);
  const bool vec_ok = (N & 1) == 0;
  for (int t = 0; t < T; ++t) {
    const int st = t & 1;
    __syncthreads();   // stage st is complete; both warpgroups have retired the MMAs that read stage st ^ 1
    const uint32_t bb = s0 + kKnnB + st * 32768;
    float d[32];
    wgmma_fence();
    // hi*hi, hi*lo, lo*hi over K = 128 (B panels of 64 channels, 8 KB)
    gemm_rs<FMT, 8, 64, 0>(d, ahi, alo, bb, bb + 16384, 8192, 1, 0);
    wgmma_commit();
    if (t + 1 < T) knn_stage_keys(smem + kKnnB + (st ^ 1) * 32768, rows, t0 + t + 1, N, tid);
    wgmma_wait<0>();
    fence_regs(d);
    const int j0 = (t0 + t) * 64;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (srow[h] >= S) continue;
      float* drow = dist + sd.dist0 + (size_t)srow[h] * N;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int j = j0 + 8 * jj + fc;
        const float x0 = fmaf(-2.f, d[4 * jj + 2 * h], 2.f), x1 = fmaf(-2.f, d[4 * jj + 2 * h + 1], 2.f);
        if (vec_ok && j + 1 < N) {
          *reinterpret_cast<float2*>(drow + j) = make_float2(x0, x1);
        } else {
          if (j < N) drow[j] = x0;
          if (j + 1 < N) drow[j + 1] = x1;
        }
      }
    }
  }
}

void launch_knn_dist_tc(const float* normed, const int32_t* seeds, float* dist, int B, int N, int S, cudaStream_t st,
                        const SetDesc* sets) {
  if (S <= 0) return;
  ensure_dynamic_smem(reinterpret_cast<const void*>(knn_dist_tc_kernel), kKnnSmem);
  const int T = (N + 63) / 64, ctas = ((S + 127) / 128) * B, sms = device_sm_count();
  int chunks = ctas >= sms ? 1 : (sms + ctas - 1) / ctas;
  if (chunks > T) chunks = T;
  const int per = (T + chunks - 1) / chunks;
  chunks = (T + per - 1) / per;
  knn_dist_tc_kernel<<<dim3((S + 127) / 128, B, chunks), kKnnThreads, kKnnSmem, st>>>(normed, seeds, dist, sets, per);
}

}  // namespace pdsc
