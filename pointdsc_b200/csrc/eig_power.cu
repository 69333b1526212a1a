// f4 — leading eigenvector of an N x N compatibility matrix by power iteration (SURVEY.md §8 row f4).
//
// Reference: models/PointDSC.py:338-358 (cal_leading_eigenvector, method = 'power'), the N x N use of it at :170 (on the
// learned feature-similarity matrix M of the non-testing forward, disabled in the released code) and the classical spectral
// matching baseline, baseline_scripts/baseline_3DMatch.py:40-44 (ten fixed iterations):
//     v <- 1;  repeat:  v <- M v;  v <- v / (||v|| + 1e-6);  stop when allclose(v, v_prev)  (rtol 1e-5, atol 1e-8)
// The k x k instances of the testing-mode forward run inside nsm.cu (the matrices live in shared memory); this file is the
// N x N form the north star describes: a memory-bound GEMV whose matrix tiles stream from HBM (or L2: M is re-read by every
// iteration and 4 N^2 bytes fit the 50 MB L2 up to N ~ 3500) into shared memory through the TMA engine.
//
// gemv kernel   CTA = R <= 32 rows of one set (R chosen on the host so that a small problem is ONE wave of two CTAs per SM: with
//               32 rows, N = 5000 is 157 CTAs on 132 SMs, i.e. two waves).  Column tiles of R rows x 512 columns arrive as R bulk
//               async copies (cp.async.bulk, one contiguous 2 KB row segment each, mbarrier complete_tx) into a two-stage ring;
//               warp w takes rows w, w + 8, ..., lane l reading columns 4 l + 128 i of the staged tile and of the vector as
//               128-bit shared-memory loads; a row's 32 lane partials are combined by an xor-shuffle tree.  Every CTA also
//               leaves the sum of squares of its outputs (fixed order) for the normalisation.
// norm kernel   one CTA per set: adds the per-CTA partial sums in ascending order, scales, tests allclose against the
//               previous iterate and latches a per-set `done` flag — later iterations of a finished set are no-ops, which is
//               how the data-dependent early exit runs without a host synchronisation.
// Rows whose address is not 16-byte aligned (N % 4 != 0) cannot be bulk-copied: that case takes plain coalesced loads.
#include "abi.h"
#include "common.cuh"
#include "kernels.h"
#include "tc_ptx.cuh"

namespace pdsc {
using namespace ptx;

constexpr int kEigRows = 32, kEigCols = 512, kEigThreads = 256;       // kEigRows: the maximum; R = rows_per_cta at run time
// the largest N accepted: the gemv's two tile stages and its copy of v (N rounded up to kEigCols) fit in 227 KB of shared memory
constexpr int kEigMaxN = 24576;
static_assert(kEigMaxN % kEigCols == 0 && 2 * kEigRows * kEigCols * 4 + 64 + kEigMaxN * 4 <= 227 * 1024,
              "eig_gemv_kernel's shared memory at N = kEigMaxN");

__global__ void __launch_bounds__(kEigThreads) eig_gemv_kernel(const float* __restrict__ M, const float* __restrict__ v,
                                                               float* __restrict__ u, float* __restrict__ partial_ss,
                                                               const int* __restrict__ done, int N, int use_tma, int R) {
  extern __shared__ __align__(128) uint8_t esm[];
  const int b = blockIdx.y, r0 = blockIdx.x * R;
  if (done[b]) return;                                // the set converged in an earlier iteration
  const int tile_bytes = R * kEigCols * 4;            // one stage: R rows x 2 KB
  float* tiles = reinterpret_cast<float*>(esm);
  uint64_t* bars = reinterpret_cast<uint64_t*>(esm + 2 * tile_bytes);
  float* vs = reinterpret_cast<float*>(esm + 2 * tile_bytes + 64);      // [round_up(N, kEigCols)]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* Mb = M + (size_t)b * N * N;
  const float* vb = v + (size_t)b * N;
  const int ntiles = (N + kEigCols - 1) / kEigCols;
  const int NP = ntiles * kEigCols;
  for (int j = tid; j < NP; j += kEigThreads) vs[j] = j < N ? vb[j] : 0.f;
  const uint32_t bar0 = smem_u32(bars), t_base = smem_u32(tiles);
  if (tid == 0) {
    mbar_init(bar0, 1);
    mbar_init(bar0 + 8, 1);
    fence_barrier_init();
  }
  __syncthreads();
  const int rows_here = min(R, N - r0);

  auto issue = [&](int t) {      // one elected thread: 2 KB per row, complete_tx on the stage's barrier
    const int st = t & 1, c0 = t * kEigCols;
    const int cols = min(kEigCols, N - c0);
    mbar_expect_tx(bar0 + 8 * st, (uint32_t)(rows_here * cols * 4));
    for (int r = 0; r < rows_here; ++r)
      bulk_g2s(t_base + (uint32_t)(st * tile_bytes + r * kEigCols * 4), Mb + (size_t)(r0 + r) * N + c0, (uint32_t)(cols * 4),
               bar0 + 8 * st);
  };
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  if (use_tma) {
    if (tid == 0) {
      issue(0);
      if (ntiles > 1) issue(1);
    }
    for (int t = 0; t < ntiles; ++t) {
      const int st = t & 1;
      mbar_wait(bar0 + 8 * st, (uint32_t)((t >> 1) & 1));
      const int cols = min(kEigCols, N - t * kEigCols);
      const float* T = tiles + (size_t)st * (tile_bytes / 4);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int r = warp + 8 * q;
        if (r < rows_here) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int c = 4 * lane + 128 * i;
            if (c < cols) {            // cols is a multiple of 4 on this path (N % 4 == 0)
              const float4 m4 = *reinterpret_cast<const float4*>(T + r * kEigCols + c);
              const float4 v4 = *reinterpret_cast<const float4*>(vs + t * kEigCols + c);
              acc[q] = fmaf(m4.x, v4.x, acc[q]); acc[q] = fmaf(m4.y, v4.y, acc[q]);
              acc[q] = fmaf(m4.z, v4.z, acc[q]); acc[q] = fmaf(m4.w, v4.w, acc[q]);
            }
          }
        }
      }
      __syncthreads();                                   // the stage has been consumed by every warp
      if (tid == 0 && t + 2 < ntiles) issue(t + 2);
    }
  } else {
    for (int q = 0; q < 4; ++q) {
      const int r = warp + 8 * q;
      if (r < rows_here) {
        const float* row = Mb + (size_t)(r0 + r) * N;
        for (int c = lane; c < N; c += 32) acc[q] = fmaf(row[c], vs[c], acc[q]);
      }
    }
  }
  __shared__ float usq[kEigRows];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float s = warp_sum(acc[q]);
    const int r = warp + 8 * q;
    if (lane == 0) {
      usq[r] = (r < rows_here) ? s * s : 0.f;
      if (r < rows_here) u[(size_t)b * N + r0 + r] = s;
    }
  }
  __syncthreads();
  if (tid == 0) {
    float ss = 0.f;
    for (int r = 0; r < kEigRows; ++r) ss += usq[r];
    partial_ss[(size_t)b * gridDim.x + blockIdx.x] = ss;
  }
}

__global__ void __launch_bounds__(256) eig_norm_kernel(const float* __restrict__ u, float* __restrict__ v,
                                                       const float* __restrict__ partial_ss, int* __restrict__ done,
                                                       int* __restrict__ iters_run, int N, int nparts, int early_exit) {
  __shared__ float nrm_s;
  __shared__ int ok_s;
  const int b = blockIdx.x, tid = threadIdx.x;
  if (done[b]) return;
  if (tid == 0) {
    float ss = 0.f;
    for (int p = 0; p < nparts; ++p) ss += partial_ss[(size_t)b * nparts + p];
    nrm_s = sqrtf(ss) + 1e-6f;
    ok_s = 1;
  }
  __syncthreads();
  const float nrm = nrm_s;
  int ok = 1;
  for (int j = tid; j < N; j += blockDim.x) {
    const float vn = u[(size_t)b * N + j] / nrm;
    const float vo = v[(size_t)b * N + j];
    ok &= (fabsf(vn - vo) <= 1e-8f + 1e-5f * fabsf(vo));
    v[(size_t)b * N + j] = vn;
  }
  if (!ok) ok_s = 0;           // benign race: every writer stores 0
  __syncthreads();
  if (tid == 0) {
    iters_run[b] += 1;
    if (early_exit && ok_s) done[b] = 1;
  }
}

__global__ void eig_init_kernel(float* v, int* done, int* iters_run, int B, int N) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < (long long)B * N) v[i] = 1.0f;
  if (i < B) { done[i] = 0; iters_run[i] = 0; }
}

size_t eig_scratch_bytes(int B, int N) {
  const int nparts = (N + 7) / 8;                     // upper bound: the smallest rows-per-CTA is 8
  return (size_t)B * N * 4 + (size_t)B * nparts * 4 + (size_t)B * 4 + 256;
}

}  // namespace pdsc

// ---- C ABI ------------------------------------------------------------------------------------------------------
using namespace pdsc;

extern "C" {

size_t pdsc_leading_eigenvector_scratch_bytes(int32_t B, int32_t N) { return (B > 0 && N > 0) ? eig_scratch_bytes(B, N) : 0; }

// v [B,N] receives the eigenvector, iters_run [B] the iterations executed per set.  scratch: u [B,N] | partial [B,nparts] | done [B]
int pdsc_leading_eigenvector(pdsc_engine* e, int32_t B, int32_t N, const float* d_M, int32_t num_iterations, int32_t early_exit,
                             float* d_eigenvector, int32_t* d_iterations_run, void* d_scratch, size_t scratch_bytes,
                             void* cuda_stream) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (B <= 0 || N <= 0) return fail(PDSC_ERR_SHAPE, "need B >= 1 and N >= 1 (got B=%d N=%d)", B, N);
  if (num_iterations < 1 || num_iterations > 1000) return fail(PDSC_ERR_INVALID_ARGUMENT, "num_iterations %d out of range", num_iterations);
  if (N > kEigMaxN) return fail(PDSC_ERR_UNSUPPORTED, "N=%d exceeds the supported maximum %d", N, kEigMaxN);
  if (!d_M || !d_eigenvector || !d_iterations_run) return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_leading_eigenvector: null tensor pointer");
  if (int rc = check_scratch("pdsc_leading_eigenvector", "scratch", d_scratch, scratch_bytes, eig_scratch_bytes(B, N), 16)) return rc;
  DeviceGuard g(engine_config(e).device);
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  // rows per CTA: 32 when the grid is many waves anyway, else what makes it one wave of two CTAs per SM
  const int sms = device_sm_count();
  int R = kEigRows;
  if ((long long)B * ((N + R - 1) / R) < 4LL * sms) {
    R = (int)(((long long)B * N + 2LL * sms - 1) / (2LL * sms));
    R = R < 8 ? 8 : (R > kEigRows ? kEigRows : R);
  }
  const int nparts = (N + R - 1) / R;
  float* u = static_cast<float*>(d_scratch);
  float* partial = u + (size_t)B * N;
  int* done = reinterpret_cast<int*>(partial + (size_t)B * ((N + 7) / 8));
  const int NP = (N + kEigCols - 1) / kEigCols * kEigCols;
  const int smem = 2 * R * kEigCols * 4 + 64 + NP * 4;
  const int use_tma = (N % 4 == 0) && (reinterpret_cast<uintptr_t>(d_M) % 16 == 0);
  cudaError_t err = ensure_dynamic_smem(reinterpret_cast<const void*>(eig_gemv_kernel), smem);
  if (err == cudaSuccess) {
    eig_init_kernel<<<(unsigned)(((long long)B * N + 255) / 256), 256, 0, st>>>(d_eigenvector, done, d_iterations_run, B, N);
    for (int t = 0; t < num_iterations; ++t) {
      eig_gemv_kernel<<<dim3(nparts, B), kEigThreads, smem, st>>>(d_M, d_eigenvector, u, partial, done, N, use_tma, R);
      eig_norm_kernel<<<B, 256, 0, st>>>(u, d_eigenvector, partial, done, d_iterations_run, N, nparts, early_exit);
    }
    err = cudaGetLastError();
  }
  if (err != cudaSuccess) return fail(PDSC_ERR_CUDA, "power iteration launch failed: %s", cudaGetErrorString(err));
  return PDSC_OK;
}

}  // extern "C"
