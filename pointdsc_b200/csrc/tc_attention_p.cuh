// tc_attention (persistent): SC-weighted flash attention on wgmma, one CTA per SM looping over (set, 128-query tile)
// work items (included by encoder_tc.cu only).
//
// Reference: models/PointDSC.py:39-42
//     P = softmax_j( SC_ij * (q_i . k_j) / sqrt(C) ),   msg_i = sum_j P_ij v_j          (heads = 1, C = 128)
// SC multiplies the logit (it is not a mask): SC_ij = 0 leaves logit 0, which still takes softmax mass.
//
// Roles (384 threads):
//   warps 0-7   two consumer warpgroups, 64 query rows each, 232 registers per thread (setmaxnreg.inc).  Per 64-key tile:
//               S = Q K^T (wgmma, Q and K from shared memory, S in registers), logits S * SC with the SC tile streamed from
//               HBM one tile-step ahead, online softmax in registers (log2 units: Q carries log2(e) / sqrt(C)), P split into
//               16-bit hi / lo register A operands, O += P V (wgmma, V read as an MN-major B operand, O in registers).
//   warps 8-11  producer warpgroup, 40 registers per thread (setmaxnreg.dec) so that the consumers can have more; warps 9-11
//               leave at once, one lane of warp 8 streams each item's Q image and its K / V tiles (bulk async copies,
//               mbarrier complete_tx) through a two-stage ring, running ahead into the next item while the current one is
//               computed.
#pragma once
#include "tc_attention.cuh"

namespace pdsc {

constexpr int kAttnPQ = 0;                                   // Q image: [hi p0 16K][hi p1 16K][lo p0 16K][lo p1 16K]
constexpr int kAttnPKV = 65536;                              // stage s at + 64 KB s: K [hi p0][hi p1][lo p0][lo p1] 8 KB each, V the same
constexpr int kAttnStages = 2;
constexpr int kAttnPBars = kAttnPKV + kAttnStages * 65536;
constexpr int kAttnPSmem = kAttnPBars + 128;                 // 196,736 B

template <int FMT>
__global__ void __launch_bounds__(kAttnThreads, 1) tc_attention_persistent_kernel(AttnArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kAttnPBars);
  const uint32_t s0 = smem_u32(smem);
  const uint32_t q_full = smem_u32(bars + 0), q_empty = smem_u32(bars + 1);
  const uint32_t kv_full = smem_u32(bars + 2), kv_empty = smem_u32(bars + 4);   // [kAttnStages]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int my_items = (a.items > (int)blockIdx.x) ? (a.items - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;

  if (tid == 0) {
    if (s0 & 1023u) __trap();   // the swizzled operand images need 1024-byte aligned shared memory
    mbar_init(q_full, 1);
    mbar_init(q_empty, 256);
    for (int i = 0; i < kAttnStages; ++i) {
      mbar_init(kv_full + 8 * i, 1);
      mbar_init(kv_empty + 8 * i, 256);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ===================================== producer =====================================
    setmaxnreg_dec<kAttnProducerRegs>();   // the whole warpgroup gives its registers to the consumers
    if (warp == 8 && lane == 0) {
      const uint32_t q_bytes = a.split ? 65536u : 32768u;
      const uint32_t tile_bytes = a.split ? 32768u : 16384u;   // hi (+ lo) image of one 64-key tile of K or V
      int gt = 0;                                              // running tile count of the CTA
      for (int it = 0; it < my_items; ++it) {
        const int witem = blockIdx.x + it * gridDim.x;
        const AttnItem w = attn_item(a, witem);
        if (it > 0) mbar_wait(q_empty, (uint32_t)((it - 1) & 1));   // the previous item's last QK has retired
        mbar_expect_tx(q_full, q_bytes);
        for (uint32_t off = 0; off < q_bytes; off += 32768u)
          bulk_g2s(s0 + kAttnPQ + off, a.qimg + (size_t)w.qtile * 65536 + off, 32768u, q_full);
        for (int j = 0; j < w.T; ++j, ++gt) {
          const int st = gt % kAttnStages, use = gt / kAttnStages;
          if (use > 0) mbar_wait(kv_empty + 8 * st, (uint32_t)((use - 1) & 1));
          const int kt = min(w.t0 + j, w.KT - 1);              // a virtual tile re-reads the last real one (it is masked)
          const uint8_t* kv = a.kvimg + ((size_t)w.kt0 + kt) * 65536;
          const uint32_t dst = s0 + kAttnPKV + st * 65536;
          mbar_expect_tx(kv_full + 8 * st, 2 * tile_bytes);
          bulk_g2s(dst, kv, tile_bytes, kv_full + 8 * st);
          bulk_g2s(dst + 32768, kv + 32768, tile_bytes, kv_full + 8 * st);
        }
      }
    }
    __syncwarp();
    return;
  }

  // ===================================== consumers =====================================
  setmaxnreg_inc<kAttnConsumerRegs>();
  const int wg = warp >> 2, wt = tid & 127;
  const int r0 = 64 * wg + frag_row(wt), fc = frag_col(wt);   // query rows r0, r0 + 8 of the tile; key columns 8 j + fc, + 1
  const uint32_t qa = s0 + kAttnPQ + (uint32_t)wg * 8192u;     // this warpgroup's 64 rows of the Q image
  int gt = 0;
  for (int it = 0; it < my_items; ++it) {
    const int witem = blockIdx.x + it * gridDim.x;
    const AttnItem w = attn_item(a, witem);   // (set, query tile) and the split's key tiles
    const int N = w.N, qt = w.qt, t0 = w.t0, T = w.T, KT = w.KT;
    const size_t tile_stride = (size_t)w.QT << 13;
    const float* sc_cta = a.sc + w.sc0 + ((size_t)qt << 13);
    float o[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l_sum[2] = {0.f, 0.f};
    // this thread's 32 SC values of the next key tile, loaded a full tile-step before the softmax needs them
    float sc[32];
    attn_load_sc(sc, sc_cta + (size_t)min(t0, KT - 1) * tile_stride, r0, fc);
    mbar_wait(q_full, (uint32_t)(it & 1));
    for (int j = 0; j < T; ++j, ++gt) {
      const int st = gt % kAttnStages, use = gt / kAttnStages;
      const uint32_t kb = s0 + kAttnPKV + st * 65536, vb = kb + 32768;
      mbar_wait(kv_full + 8 * st, (uint32_t)(use & 1));
      float s[32];
      wgmma_fence();
      gemm_ss<FMT, 2, 64>(s, qa, qa + 32768, 16384, kb, kb + 16384, 8192, a.split);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s);
      if (j == T - 1) mbar_arrive(q_empty);   // the item's last QK has retired: the Q buffer may be refilled
#pragma unroll
      for (int i = 0; i < 32; ++i) s[i] *= sc[i];
      // never past the item's last tile: the next item may belong to another set
      if (j + 1 < T) attn_load_sc(sc, sc_cta + (size_t)min(t0 + j + 1, KT - 1) * tile_stride, r0, fc);
      if ((t0 + j) * 64 + 63 >= N) {       // the set's last, ragged key tile - or a virtual tile behind it (all masked)
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if ((t0 + j) * 64 + 8 * (i >> 2) + fc + (i & 1) >= N) s[i] = -INFINITY;
      }
      // online softmax: row maximum over the quad that shares the row, rescale O and the row sum when it moves
      float scale[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float tmax = -INFINITY;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) tmax = fmaxf(tmax, fmaxf(s[4 * jj + 2 * h], s[4 * jj + 2 * h + 1]));
        tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 1));
        tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 2));
        const float mn = fmaxf(m[h], tmax);
        scale[h] = (mn > m[h]) ? ex2_approx(m[h] - mn) : 1.0f;
        m[h] = mn;
        l_sum[h] *= scale[h];
      }
      float rsum[2] = {0.f, 0.f};
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int h = (i >> 1) & 1;
        s[i] = ex2_approx(s[i] - m[h]);
        rsum[h] += s[i];
      }
      l_sum[0] += rsum[0];
      l_sum[1] += rsum[1];
#pragma unroll
      for (int i = 0; i < 64; ++i) o[i] *= scale[(i >> 1) & 1];
      uint32_t phi[4][4], plo[4][4];
      frag_split<FMT, 4>(s, phi, plo);
      wgmma_fence();
      gemm_rs<FMT, 4, 128, 1>(o, phi, plo, vb, vb + 16384, 8192, a.split, 1);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(o);
      mbar_arrive(kv_empty + 8 * st);        // K_j and V_j are no longer read
    }
    // ---- epilogue: O / l -> msg.  Key split: the item's UNNORMALISED O, its maximum and its row sum go to the partial
    //      buffers; tc_attention_merge_kernel combines the splits of a query tile in ascending split order ----
    const bool partial = w.sp > 1;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float lt = l_sum[h];
      lt += __shfl_xor_sync(0xffffffffu, lt, 1);
      lt += __shfl_xor_sync(0xffffffffu, lt, 2);
      const int r = r0 + 8 * h;
      const float inv_l = partial ? 1.0f : 1.0f / lt;
      if (partial && (lane & 3) == 0) *reinterpret_cast<float2*>(a.part_ml + ((size_t)witem * 128 + r) * 2) = make_float2(m[h], lt);
      if (!partial && qt * 128 + r >= N) continue;
      float* dst = partial ? a.part_o + ((size_t)witem * 128 + r) * kC : a.msg + ((size_t)w.row0 + qt * 128 + r) * kC;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj)
        *reinterpret_cast<float2*>(dst + 8 * jj + fc) = make_float2(o[4 * jj + 2 * h] * inv_l, o[4 * jj + 2 * h + 1] * inv_l);
    }
  }
}

// ---- key split: combine the partial results of one query tile -------------------------------------------------------------
// msg_i = sum_s O_s[i] 2^(m_s - m*) / sum_s l_s 2^(m_s - m*),  m* = max_s m_s, splits added in ascending order (deterministic).
// One CTA per (query tile, 32-row quarter), thread = (row, 16-byte column piece stride).  Query tiles are numbered set by set
// (qt0); the tiles of sets without a split wrote msg themselves.
__global__ void __launch_bounds__(256) tc_attention_merge_kernel(const float* __restrict__ part_o, const float* __restrict__ part_ml,
                                                                 float* __restrict__ msg, const SetDesc* __restrict__ sets, int nsets) {
  const int qtile = blockIdx.x >> 2, quarter = blockIdx.x & 3;
  const SetDesc d = sets[find_set(nsets, qtile, [&](int i) { return sets[i].qt0; })];
  if (d.sp < 2) return;
  const int N = d.N, qt = qtile - d.qt0, splits = d.sp, row0 = d.row0;
  const int item = d.item0 + qt * splits;   // the tile's first work item
  const int row = quarter * 32 + (threadIdx.x >> 3);
  if (qt * 128 + row >= N) return;
  // the reference maxima first (independent loads), then the partial rows four splits at a time so that their loads overlap:
  // at bs = 1 this kernel is pure L2 latency (8 splits x 5 dependent round trips took 9.5 us per layer)
  float mstar = -INFINITY;
#pragma unroll 4
  for (int s = 0; s < splits; ++s) mstar = fmaxf(mstar, part_ml[(((size_t)item + s) * 128 + row) * 2]);
  float L = 0.f;
  float4 acc[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int s0 = 0; s0 < splits; s0 += 4) {
    float2 ml[4];
    float4 v[4][4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int s = s0 + u < splits ? s0 + u : splits - 1;      // a clamped re-read of the last split is given weight 0 below
      const size_t w = (size_t)item + s;
      ml[u] = *reinterpret_cast<const float2*>(part_ml + (w * 128 + row) * 2);
      const float* o = part_o + (w * 128 + row) * kC;
#pragma unroll
      for (int i = 0; i < 4; ++i) v[u][i] = *reinterpret_cast<const float4*>(o + ((threadIdx.x & 7) + 8 * i) * 4);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {       // ascending split order: the sum is the same as one split at a time
      if (s0 + u < splits) {
        const float wgt = ex2_approx(ml[u].x - mstar);
        L = fmaf(ml[u].y, wgt, L);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          acc[i].x = fmaf(v[u][i].x, wgt, acc[i].x); acc[i].y = fmaf(v[u][i].y, wgt, acc[i].y);
          acc[i].z = fmaf(v[u][i].z, wgt, acc[i].z); acc[i].w = fmaf(v[u][i].w, wgt, acc[i].w);
        }
      }
    }
  }
  const float inv = 1.0f / L;
  float* dst = msg + ((size_t)row0 + qt * 128 + row) * kC;
#pragma unroll
  for (int i = 0; i < 4; ++i)
    *reinterpret_cast<float4*>(dst + ((threadIdx.x & 7) + 8 * i) * 4) = make_float4(acc[i].x * inv, acc[i].y * inv, acc[i].z * inv, acc[i].w * inv);
}

}  // namespace pdsc
