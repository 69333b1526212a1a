// a6 — seed selection by parallel non-maximum suppression (testing mode).
//
// Reference: models/PointDSC.py:199-217 (pick_seeds)
//   is_local_max_i = all_j ( s_i >= s_j  or  ||x_i - x_j|| >= R )
//   seeds          = argsort(s * is_local_max, descending)[:S]
// The reference reads the materialised N x N `src_dist`; here the distance is recomputed from the
// points with the same rounded operations (common.cuh::length3), so the N x N matrix never exists.
// Ranking contract (SURVEY.md §7 trap 3): keys are compared as fp32 values with +0 == -0, and exact
// ties are broken by the LOWEST index (a stable descending sort; the reference's argsort is unstable,
// so any order of tied keys is a valid reference output).
#include <cmath>

#include "common.cuh"
#include "kernels.h"
#include "sets.cuh"

namespace pdsc {

constexpr int kSeedMaxN = 16384;

// Thread <-> row i; candidate points j staged through shared memory as (x, y, z, s) and read as broadcasts.
// `d2_min` is the smallest fp32 squared length whose correctly rounded square root is >= R (found on the host by
// stepping floats around R^2): sqrt is monotonic, so  length3(d) >= R  <=>  fma-chain(d) >= d2_min  exactly,
// and the kernel needs no square root at all.
// Big batches: 256 rows per CTA.  Small calls (bs = 1 at N = 1000 is four such CTAs, 60 us of one latency-bound loop per thread) use
// nms_key_warp_kernel below instead.
template <int kNmsTile>
__global__ void __launch_bounds__(kNmsTile) nms_key_kernel(const float* __restrict__ src, const float* __restrict__ conf,
                                                           float* __restrict__ key, const SetDesc* __restrict__ sets, float d2_min) {
  // candidates staged as four arrays so that an 8-byte load yields the same coordinate of TWO neighbours: the distance chain
  // then runs on pairs (two candidates at a time, each lane rounded like the scalar operation)
  __shared__ __align__(8) float sx[kNmsTile], sy[kNmsTile], sz[kNmsTile], sw[kNmsTile];
  const int b = blockIdx.y;
  const SetDesc d = sets[b];
  const int N = d.N;
  if ((int)blockIdx.x * kNmsTile >= N) return;   // the grid is sized by the largest set
  const int i = blockIdx.x * kNmsTile + threadIdx.x;
  const float* p = src + (size_t)d.row0 * 3;
  const float* s = conf + d.row0;
  const bool live = i < N;
  const int ic = live ? i : N - 1;
  const float si = s[ic];
  const float xi = p[(size_t)ic * 3], yi = p[(size_t)ic * 3 + 1], zi = p[(size_t)ic * 3 + 2];
  bool ok = true;
  for (int j0 = 0; j0 < N; j0 += kNmsTile) {
    __syncthreads();
    const int j = j0 + threadIdx.x;
    const bool have = j < N;      // a pad candidate has score -inf: it suppresses nobody
    sx[threadIdx.x] = have ? p[(size_t)j * 3] : 0.f;
    sy[threadIdx.x] = have ? p[(size_t)j * 3 + 1] : 0.f;
    sz[threadIdx.x] = have ? p[(size_t)j * 3 + 2] : 0.f;
    sw[threadIdx.x] = have ? s[j] : -INFINITY;
    __syncthreads();
    if (ok) {
#pragma unroll 4
      for (int t = 0; t < kNmsTile; t += 2) {
        const float2 qx = *reinterpret_cast<const float2*>(sx + t), qy = *reinterpret_cast<const float2*>(sy + t),
                     qz = *reinterpret_cast<const float2*>(sz + t), qs = *reinterpret_cast<const float2*>(sw + t);
        const float2 dx = fsub2_scalar(xi, qx), dy = fsub2_scalar(yi, qy), dz = fsub2_scalar(zi, qz);
        const float2 d2 = ffma2_pair(dz, dz, ffma2_pair(dy, dy, fmul2(dx, dx)));  // the argument of length3()'s sqrt, twice
        ok = ok && ((si >= qs.x) || (d2.x >= d2_min)) && ((si >= qs.y) || (d2.y >= d2_min));
      }
    }
  }
  if (live) key[(size_t)d.row0 + i] = si * (ok ? 1.0f : 0.0f);
}

// Small calls: one WARP per row i, the lanes stride over the candidates j, the verdict is a warp vote; a row is decided in
// N / 32 iterations with 32 loads in flight, and N rows spread over N / 8 CTAs.  Same arithmetic, same result.
__global__ void __launch_bounds__(256) nms_key_warp_kernel(const float* __restrict__ src, const float* __restrict__ conf,
                                                           float* __restrict__ key, const SetDesc* __restrict__ sets, float d2_min) {
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  const SetDesc d = sets[b];
  const int N = d.N;
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= N) return;
  const float* p = src + (size_t)d.row0 * 3;
  const float* s = conf + d.row0;
  const float si = s[i];
  const float xi = p[(size_t)i * 3], yi = p[(size_t)i * 3 + 1], zi = p[(size_t)i * 3 + 2];
  bool ok = true;
  for (int j0 = 0; j0 < N; j0 += 128) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = j0 + 32 * u + lane;
      if (j < N) {
        const float dx = xi - p[(size_t)j * 3], dy = yi - p[(size_t)j * 3 + 1], dz = zi - p[(size_t)j * 3 + 2];
        const float d2 = __fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
        ok = ok && ((si >= s[j]) || (d2 >= d2_min));
      }
    }
    if (!__all_sync(0xffffffffu, ok)) break;
  }
  ok = __all_sync(0xffffffffu, ok);
  if (lane == 0) key[(size_t)d.row0 + i] = si * (ok ? 1.0f : 0.0f);
}

__device__ __forceinline__ uint32_t orderable(float f) {
  uint32_t u = __float_as_uint(f);
  if ((u & 0x7FFFFFFFu) == 0u) u = 0u;  // -0 ranks equal to +0, as in a floating-point comparison
  return u ^ ((u & 0x80000000u) ? 0xFFFFFFFFu : 0x80000000u);
}

// one CTA per set: bitonic sort of (descending key, ascending index), emit the first S indices.  P is a power of two >= N
// (every set is sorted at the P of the call's largest set: the pads sort last, the sorted prefix is the same)
__global__ void __launch_bounds__(1024) seed_sort_kernel(const float* __restrict__ key, int32_t* __restrict__ seeds,
                                                         const SetDesc* __restrict__ sets, int P) {
  extern __shared__ unsigned long long skeys[];
  const int b = blockIdx.x;
  const SetDesc d = sets[b];
  const int N = d.N, S = d.S;
  if (S <= 0) return;
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    unsigned long long v = ~0ull;
    if (i < N) v = ((unsigned long long)(~orderable(key[(size_t)d.row0 + i])) << 32) | (unsigned)i;
    skeys[i] = v;
  }
  __syncthreads();
  for (int k = 2; k <= P; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < P; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = skeys[i], c = skeys[ixj];
          const bool asc = (i & k) == 0;
          if ((a > c) == asc) { skeys[i] = c; skeys[ixj] = a; }
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < S; i += blockDim.x) seeds[(size_t)d.seed0 + i] = (int32_t)(skeys[i] & 0xFFFFFFFFull);
}

int pick_seeds_max_n() { return kSeedMaxN; }

static void launch_seed_sort(const float* key, int32_t* seeds, int B, int N, int S, cudaStream_t st, const SetDesc* sets) {
  int P = 2;
  while (P < N) P <<= 1;
  const int smem = P * (int)sizeof(unsigned long long);
  ensure_dynamic_smem(reinterpret_cast<const void*>(seed_sort_kernel), smem);
  const int threads = P / 2 < 1024 ? (P / 2 < 32 ? 32 : P / 2) : 1024;
  seed_sort_kernel<<<B, threads, smem, st>>>(key, seeds, sets, P);
}

// a6' — the non-testing seed rule (models/PointDSC.py:176): argsort(confidence, descending)[:S], no suppression.
// Ties: lowest index first (the reference's argsort is unstable).
void launch_top_seeds(const float* conf, int32_t* seeds, int B, int N, int S, cudaStream_t st, const SetDesc* sets) {
  if (S > 0) launch_seed_sort(conf, seeds, B, N, S, st, sets);
}

void launch_pick_seeds(const float* src, const float* conf, int32_t* seeds, float* key_scratch, int B, int N, int S,
                       float radius, cudaStream_t st, const SetDesc* sets) {
  // smallest float x with sqrtf(x) >= radius (IEEE sqrt on the host == the device's sqrt.rn)
  float d2_min = radius * radius;
  while (std::sqrt(d2_min) >= radius && d2_min > 0.f) d2_min = std::nextafter(d2_min, 0.0f);
  while (std::sqrt(d2_min) < radius) d2_min = std::nextafter(d2_min, INFINITY);
  if ((long long)B * ((N + 255) / 256) >= 2LL * device_sm_count())
    nms_key_kernel<256><<<dim3((N + 255) / 256, B), 256, 0, st>>>(src, conf, key_scratch, sets, d2_min);
  else
    nms_key_warp_kernel<<<dim3((N + 7) / 8, B), 256, 0, st>>>(src, conf, key_scratch, sets, d2_min);
  launch_seed_sort(key_scratch, seeds, B, N, S, st, sets);
}

}  // namespace pdsc
