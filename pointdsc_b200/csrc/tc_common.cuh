// Shared definitions of the tensor-core kernels (encoder_tc.cu, knn_tc.cu).
#pragma once
#include "common.cuh"
#include "sets.cuh"
#include "tc_ptx.cuh"

namespace pdsc {
using namespace ptx;

// ---- weight arena layout (bytes, per layer) ------------------------------------------------------------
constexpr size_t kW1 = 0, kWq = 65536, kWk = 131072, kWv = 196608, kWm0 = 262144, kWm1 = 294912, kWm2 = 311296,
                 kBias = 344064, kLayerBytes = 348160;
// bias block (floats): b1[128] bq[128] bk[128] bv[128] bm0[64] bm1[64] bm2[128]
constexpr int kB1 = 0, kBq = 128, kBk = 256, kBv = 384, kBm0 = 512, kBm1 = 576, kBm2 = 640, kBiasFloats = 768;

constexpr float kQScale = 1.4426950408889634f / 11.313708498984761f;  // log2(e) / sqrt(128)

enum ChainMode { kPCQ = 0, kKV = 1, kMSG = 2, kMSGPC = 3, kQ = 4 };

struct ChainArgs {
  long long rows;        // rows of the call (all sets)
  int split;
  const SetDesc* sets;   // the call's descriptor table (row0, qt0, kt0)
  const int* tile_set;   // [rows / 128]: the set of the first row of every 128-row chain tile
  int nsets;
  const float* in;       // [rows][128] fp32 A operand
  const float* res;      // MSG, MSGPC: feat1 (residual)
  float* out_f32;        // PCQ: feat1, MSG: feat, MSGPC: the next layer's feat1 (in place over res)
  float* feat_out;       // MSGPC: where feat goes too (the layer_features tap), or nullptr
  uint8_t* qimg;
  uint8_t* kvimg;
  const uint8_t* wimg;   // this kernel's weight images (contiguous)
  const float* bias;     // the layer's bias block
  int wbytes;            // bytes of weight images to stage
  const uint8_t* wimg1;  // MSGPC: the next layer's W1 images (64 KB)
  const float* bias1;    // MSGPC: the next layer's bias block (b1)
};

// Synchronisation rules of the tensor-core kernels.
//  1. An operand image written into shared memory by ordinary stores is read by wgmma through the async proxy: the writers
//     execute fence.proxy.async before the barrier that publishes the image.
//  2. wgmma reads its register A operand and accumulates into its registers asynchronously: nothing touches them between
//     the issue and the wgmma.wait_group that retires the group (fence_regs keeps the compiler from moving such accesses).
//  3. Counted mbarriers (the attention's K / V ring, its Q buffer): every consumer thread arrives once per phase, after the
//     wait_group that retired the last MMA reading the buffer.

// D[64 x NOUT] (+)= A[64 x 64 KP] * W[NOUT x 64 KP]^T, A and W K-major SWIZZLE_128B panels (64 K elements each) in shared
// memory, optionally as the three hi/lo products hi*hi + hi*lo + lo*hi.  One warpgroup; the caller fences, commits, waits.
template <int FMT, int KP, int NOUT>
__device__ __forceinline__ void gemm_ss(float (&d)[NOUT / 2], uint32_t a_hi, uint32_t a_lo, uint32_t a_panel_bytes, uint32_t b_hi,
                                        uint32_t b_lo, uint32_t b_panel_bytes, int split) {
  uint32_t acc = 0;
#pragma unroll
  for (int t = 0; t < 3; ++t) {
    if (t > 0 && !split) break;
    const uint32_t a = (t == 2) ? a_lo : a_hi;
    const uint32_t b = (t == 1) ? b_lo : b_hi;
#pragma unroll
    for (int p = 0; p < KP; ++p) {
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint64_t ad = smem_desc_sw128(a + p * a_panel_bytes + ks * 32);
        const uint64_t bd = smem_desc_sw128(b + p * b_panel_bytes + ks * 32);
        if constexpr (NOUT == 64) wgmma_ss_n64<FMT, 0>(d, ad, bd, acc);
        else wgmma_ss_n128<FMT, 0>(d, ad, bd, acc);
        acc = 1;
      }
    }
  }
}

// D[64 x NOUT] (+)= A[64 x 16 KS] * W[NOUT x 16 KS]^T with A in REGISTERS (k-step fragments, hi and lo images) and W K-major
// SWIZZLE_128B panels in shared memory.  TB = 1: W is instead an MN-major [16 KS rows][NOUT] image (LBO = b_panel_bytes between
// its 64-column blocks).  accumulate = 0 overwrites D.
template <int FMT, int KS, int NOUT, int TB>
__device__ __forceinline__ void gemm_rs(float (&d)[NOUT / 2], const uint32_t (&a_hi)[KS][4], const uint32_t (&a_lo)[KS][4], uint32_t b_hi,
                                        uint32_t b_lo, uint32_t b_panel_bytes, int split, uint32_t accumulate) {
  uint32_t acc = accumulate;
#pragma unroll
  for (int t = 0; t < 3; ++t) {
    if (t > 0 && !split) break;
    const uint32_t b = (t == 1) ? b_lo : b_hi;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      const uint64_t bd = TB ? smem_desc_sw128(b + ks * 2048, b_panel_bytes)
                             : smem_desc_sw128(b + (ks >> 2) * b_panel_bytes + (ks & 3) * 32);
      if constexpr (NOUT == 64) wgmma_rs_n64<FMT, TB>(d, t == 2 ? a_lo[ks] : a_hi[ks], bd, acc);
      else wgmma_rs_n128<FMT, TB>(d, t == 2 ? a_lo[ks] : a_hi[ks], bd, acc);
      acc = 1;
    }
  }
}

// accumulator fragment (16 KS columns) -> register A operand of the next GEMM, as 16-bit hi / lo images
template <int FMT, int KS>
__device__ __forceinline__ void frag_split(const float (&x)[8 * KS], uint32_t (&hi)[KS][4], uint32_t (&lo)[KS][4]) {
#pragma unroll
  for (int ks = 0; ks < KS; ++ks)
#pragma unroll
    for (int i = 0; i < 4; ++i) split_pair<FMT>(x[8 * ks + 2 * i], x[8 * ks + 2 * i + 1], hi[ks][i], lo[ks][i]);
}

// this thread's two accumulator rows within the warpgroup's 64 and its first column within each 8-column group
__device__ __forceinline__ int frag_row(int tid_in_wg) { return ((tid_in_wg >> 5) << 4) + ((tid_in_wg & 31) >> 2); }
__device__ __forceinline__ int frag_col(int tid_in_wg) { return (tid_in_wg & 3) << 1; }

}  // namespace pdsc
