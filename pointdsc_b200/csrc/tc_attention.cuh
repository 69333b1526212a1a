// tc_attention: SC-weighted flash attention on wgmma (included by encoder_tc.cu only).
//
// Reference: models/PointDSC.py:39-42
//     P = softmax_j( SC_ij * (q_i . k_j) / sqrt(C) ),   msg_i = sum_j P_ij v_j          (heads = 1, C = 128)
// SC multiplies the logit (it is not a mask): SC_ij = 0 leaves logit 0, which still takes softmax mass.
//
// This header holds what the attention kernel (tc_attention_p.cuh, persistent CTAs) is built from: the argument block,
// the exponential and the streaming load of the SC tiles.
#pragma once
#include "tc_common.cuh"

namespace pdsc {

struct AttnArgs {
  int split;
  const uint8_t* qimg;
  const uint8_t* kvimg;
  const float* sc;    // tiled, per set from its sc0: [KT][QT][16 key groups][128 queries][4 keys]
  float* msg;
  int items;          // work items of the launch
  float* part_o;      // [items][128][128] unnormalised O of every work item of a split set
  float* part_ml;     // [items][128][2]   its final reference maximum (log2 units) and row sum
  // the descriptor table.  Work items are numbered set by set from each set's item0: set b has QT_b * sp_b of them, a work
  // item is (set, query tile, split) and covers key tiles [split * TS_b, split * TS_b + TS_b); tiles beyond KT_b are "virtual"
  // (fully masked).  sp_b == 1 (key split: small calls only, see encoder_tc.cu): TS_b == KT_b, one item per query tile.
  const SetDesc* sets;
  int nsets;
};

// one work item: (set, query tile, split)
struct AttnItem {
  int N, QT, KT;      // the set's size and tiles
  int qt, t0, T;      // query tile within the set, first key tile and key tiles of the item
  int sp;             // the set's key splits (1: the item writes msg itself)
  int qtile, kt0;     // the item's tile in the Q image, the set's first tile in the K / V image
  int row0;           // the set's first row
  long long sc0;      // the set's SC block
};

__device__ __forceinline__ AttnItem attn_item(const AttnArgs& a, int witem) {
  const SetDesc d = a.sets[find_set(a.nsets, witem, [&](int i) { return a.sets[i].item0; })];
  const int local = witem - d.item0;
  AttnItem w;
  w.N = d.N; w.QT = (d.N + 127) / 128; w.KT = (d.N + 63) / 64;
  w.qt = local / d.sp; w.t0 = (local % d.sp) * d.TS; w.T = d.TS; w.sp = d.sp;
  w.qtile = d.qt0 + w.qt; w.kt0 = d.kt0; w.row0 = d.row0; w.sc0 = d.sc0;
  return w;
}

constexpr int kAttnThreads = 384;                       // two consumer warpgroups + one producer warpgroup
// registers per thread after setmaxnreg.  An SM sub-partition (16,384 registers) holds one warp of each warpgroup, so
// 2 x consumer + producer <= 512; the launch gives every thread 168 (65,536 / 384 rounded down to 8), 3 x 168 = 2 x 232 + 40.
constexpr uint32_t kAttnConsumerRegs = 232, kAttnProducerRegs = 40;

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// streaming read-only load: every SC element is used once per CTA, keep it out of L1
__device__ __forceinline__ float2 ldg_stream2(const float* p) {
  float2 v;
  asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p));
  return v;
}
// this thread's 32 SC values of one tile (layout [16 key groups][128 queries][4 keys]) in the S fragment's order: query
// rows r0 and r0 + 8, key columns 8 jj + fc and + 1
__device__ __forceinline__ void attn_load_sc(float (&sc)[32], const float* tile, int r0, int fc) {
#pragma unroll
  for (int jj = 0; jj < 8; ++jj)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int key = 8 * jj + fc;
      const float2 v = ldg_stream2(tile + ((key >> 2) * 128 + r0 + 8 * h) * 4 + (key & 3));
      sc[4 * jj + 2 * h] = v.x;
      sc[4 * jj + 2 * h + 1] = v.y;
    }
}

}  // namespace pdsc
