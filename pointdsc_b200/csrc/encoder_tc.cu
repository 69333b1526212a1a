// Stage ii on the Hopper tensor cores (wgmma), precisions PDSC_FP16X3 (default) / PDSC_BF16X3 / PDSC_BF16.
//
// Reference: models/PointDSC.py:9-77 — per layer  PointCN (conv+BN+ReLU) -> Q,K,V 1x1 convs ->
//   P = softmax_j(SC_ij * q_i.k_j / sqrt(C)), msg = P V -> fc_message (128->64->64->128) -> residual.
//
// Numerics.  The stack is chaotic (|logit| reaches ~2.6e3, softmax is near-argmax): tools/numerics_probe.py shows single
// bf16 / fp16 / tf32 operands move the final R/t by up to 7e-4, above the 1e-4 bar, while a 16-bit hi/lo split of BOTH
// operands of every contraction (x ~= hi + lo, products hi*hi + hi*lo + lo*hi, fp32 accumulation) stays at the fp32
// noise floor (fp16 split: 22 significant bits, 2.4e-6; bf16 split: 16 bits).  The x3 modes issue those three wgmma products
// per k-step; PDSC_BF16 issues only hi*hi (3x less tensor work, throughput mode).
//
// Operand images.  Every MMA operand read from shared memory is a K-major 16-bit "panel": rows x 64 elements = rows x 128 B in
// the canonical SWIZZLE_128B layout (8-row atoms of 1024 B; 16-byte chunk c of row r stored at chunk c ^ (r & 7)).  A
// 128-channel operand is two panels; "hi" panels come first, "lo" panels second.  Producers write Q / K / V straight into this
// image layout in HBM, so a consumer stages a whole operand tile with ONE bulk async copy (cp.async.bulk -> TMA engine, mbarrier
// complete_tx) and no tensor map.  Per set b:
//     Qimg[b][qt]   qt = 128-query tile : [Qhi 32K][Qlo 32K]                       (Q pre-scaled by log2e/sqrt(C))
//     KVimg[b][kt]  kt = 64-key tile    : [Khi 16K][Klo 16K][Vhi 16K][Vlo 16K]   (V in the K format, read as an MN-major B operand)
//
// Kernels per layer (persistent: one CTA per SM):
//   tc_chain<PCQ>   (layer 0) feat -> PointCN -> feat1 (fp32, HBM; and as a register hi|lo A operand) -> Q image  tc_chain.cuh
//   tc_chain<Q>     (layers 1..) feat1 -> Q image
//   tc_chain<KV>    feat1 -> K image, V image (K format)
//   tc_attention_persistent   flash-style over (set, 128-query tile) items, S and O in registers, SC-weighted online softmax,
//                   P as a register A operand of O += P V; msg (fp32, HBM)                                 tc_attention_p.cuh
//   tc_chain<MSGPC> msg -> fc_message chain (hidden activations stay in registers) -> + feat1 -> feat (registers) -> the
//                   next layer's PointCN -> its feat1 (fp32, HBM, in place)
//   tc_chain<MSG>   (last layer) msg -> fc_message chain -> + feat1 -> feat (fp32, HBM: the head's input)
// Synchronisation rules of these kernels: tc_common.cuh.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "encoder_tc.h"
#include "kernels.h"
#include "tc_attention.cuh"
#include "tc_attention_p.cuh"
#include "tc_chain.cuh"
#include "tc_common.cuh"
#include "tc_ptx.cuh"

namespace pdsc {

// W [rows][K] fp32 (row-major) * scale  ->  [hi panels][lo panels] in the 16-bit format FMT
template <int FMT>
static void build_image(const float* W, int rows, int K, double scale, uint8_t* dst) {
  const int panels = K / 64;
  const size_t panel_bytes = (size_t)rows * 128;
  uint8_t* hi = dst;
  uint8_t* lo = dst + panels * panel_bytes;
  for (int r = 0; r < rows; ++r)
    for (int k = 0; k < K; ++k) {
      const float x = (float)((double)W[(size_t)r * K + k] * scale);
      const uint16_t h = to_16<FMT>(x);
      const uint16_t l = to_16<FMT>(x - from_16<FMT>(h));
      const size_t off = (size_t)(k / 64) * panel_bytes + sw128_offset((uint32_t)r, (uint32_t)(k % 64));
      std::memcpy(hi + off, &h, 2);
      std::memcpy(lo + off, &l, 2);
    }
}

template <int FMT>
static void build_layer(const TcLayerHost& L, uint8_t* base) {
  build_image<FMT>(L.w1, 128, 128, 1.0, base + kW1);
  build_image<FMT>(L.wq, 128, 128, (double)kQScale, base + kWq);
  build_image<FMT>(L.wk, 128, 128, 1.0, base + kWk);
  build_image<FMT>(L.wv, 128, 128, 1.0, base + kWv);
  build_image<FMT>(L.wm0, 64, 128, 1.0, base + kWm0);
  build_image<FMT>(L.wm1, 64, 64, 1.0, base + kWm1);
  build_image<FMT>(L.wm2, 128, 64, 1.0, base + kWm2);
}

int tc_build_weights(const TcLayerHost* layers, int num_layers, TcWeights* out) {
  tc_free_weights(out);
  const size_t per_fmt = (size_t)num_layers * kLayerBytes;
  std::vector<uint8_t> host(2 * per_fmt, 0);  // [fp16 images][bf16 images]
  for (int fmt = 0; fmt < 2; ++fmt)
    for (int l = 0; l < num_layers; ++l) {
      uint8_t* base = host.data() + fmt * per_fmt + (size_t)l * kLayerBytes;
      const TcLayerHost& L = layers[l];
      if (fmt == kFmtF16) build_layer<kFmtF16>(L, base); else build_layer<kFmtBF16>(L, base);
      float* b = reinterpret_cast<float*>(base + kBias);
      for (int i = 0; i < 128; ++i) {
        b[kB1 + i] = L.b1[i];
        b[kBq + i] = (float)((double)L.bq[i] * (double)kQScale);
        b[kBk + i] = L.bk[i];
        b[kBv + i] = L.bv[i];
        b[kBm2 + i] = L.bm2[i];
      }
      for (int i = 0; i < 64; ++i) {
        b[kBm0 + i] = L.bm0[i];
        b[kBm1 + i] = L.bm1[i];
      }
    }
  cudaError_t err = cudaMalloc(&out->arena, host.size());
  if (err != cudaSuccess) return (int)err;
  err = cudaMemcpy(out->arena, host.data(), host.size(), cudaMemcpyHostToDevice);
  if (err != cudaSuccess) return (int)err;
  out->arena_bytes = host.size();
  out->num_layers = num_layers;
  return 0;
}

void tc_free_weights(TcWeights* w) {
  if (w->arena) cudaFree(w->arena);
  w->arena = nullptr;
  w->arena_bytes = 0;
}

TcScratch tc_scratch(void* base, const CallShape& plan) {
  const size_t items = attn_partial_items(plan);
  const size_t kv = (size_t)plan.qtiles * 65536;   // a 128-row Q tile and a 64-row K + V tile: 64 KB of hi | lo panels each
  const size_t o = kv + (size_t)plan.ktiles * 65536;
  const size_t ml = o + items * 128 * kC * sizeof(float);
  TcScratch s{};
  s.bytes = 1024 + ml + items * 128 * 2 * sizeof(float);   // 1024: room to align the start
  if (base) {
    uint8_t* p = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(base) + 1023) & ~uintptr_t(1023));
    s.qimg = p;
    s.kvimg = p + kv;
    s.part_o = reinterpret_cast<float*>(p + o);
    s.part_ml = reinterpret_cast<float*>(p + ml);
  }
  return s;
}

int tc_launches(int num_layers, int attn_split) {   // layer0 + pad clear + 4 per layer (+ the merge of a key-split attention)
  return 2 + (attn_split ? 5 : 4) * num_layers;
}

// ---- zero the never-written pad rows/columns of the last key tile of every set ---------------------------
__global__ void tc_clear_pads_kernel(uint8_t* kvimg, const SetDesc* __restrict__ sets) {
  const int b = blockIdx.x;
  const SetDesc d = sets[b];
  const int first_pad = d.N & 63;
  if (first_pad == 0) return;
  uint8_t* base = kvimg + ((size_t)d.kt0 + (d.N + 63) / 64 - 1) * 65536;
  const int pads = 64 - first_pad;
  // K rows n in [first_pad, 64): both panels, hi and lo;  V rows likewise
  for (int t = threadIdx.x; t < pads * 128; t += blockDim.x) {
    const uint32_t n = (uint32_t)(first_pad + t / 128), c = (uint32_t)(t % 128);
    const uint32_t koff = (c >> 6) * 8192u + sw128_offset(n, c & 63u);
    *reinterpret_cast<uint16_t*>(base + koff) = 0;
    *reinterpret_cast<uint16_t*>(base + 16384 + koff) = 0;
    *reinterpret_cast<uint16_t*>(base + 32768 + koff) = 0;   // V has the K format (rows = keys)
    *reinterpret_cast<uint16_t*>(base + 49152 + koff) = 0;
  }
}

// ---- debug: decode operand images back to fp32 [rows][128] -------------------------------------------------
template <int FMT>
__global__ void tc_decode_kernel(const uint8_t* qimg, const uint8_t* kvimg, float* q, float* k, float* v, long long rows,
                                 const SetDesc* __restrict__ sets, int nsets, int split) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long row = idx / kC;
  const uint32_t c = (uint32_t)(idx % kC);
  if (row >= rows) return;
  const SetDesc d = sets[find_set(nsets, row, [&](int i) { return sets[i].row0; })];
  const int n = (int)(row - d.row0);
  auto rd = [](const uint8_t* p) { return from_16<FMT>(*reinterpret_cast<const uint16_t*>(p)); };
  const uint8_t* qb = qimg + ((size_t)d.qt0 + (n >> 7)) * 65536;
  const uint32_t qo = (c >> 6) * 16384u + sw128_offset((uint32_t)(n & 127), c & 63u);
  q[idx] = rd(qb + qo) + (split ? rd(qb + 32768 + qo) : 0.f);
  const uint8_t* kb = kvimg + ((size_t)d.kt0 + (n >> 6)) * 65536;
  const uint32_t ko = (c >> 6) * 8192u + sw128_offset((uint32_t)(n & 63), c & 63u);
  k[idx] = rd(kb + ko) + (split ? rd(kb + 16384 + ko) : 0.f);
  v[idx] = rd(kb + 32768 + ko) + (split ? rd(kb + 49152 + ko) : 0.f);
}

// debug tap: feat1 from its blocked layout (tc_chain.cuh) to plain [rows][128].  The tap is a caller's fp32 tensor, only 4-byte
// aligned by the ABI: scalar stores (the blocked source lives in the 256-byte aligned workspace)
__global__ void tc_unblock_f32_kernel(const float* __restrict__ blocked, float* __restrict__ plain, long long rows) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // 16-byte piece index
  if (i >= rows * 32) return;
  const long long g = i >> 5;
  const uint32_t piece = (uint32_t)(i & 31);
  const float4 v = *reinterpret_cast<const float4*>(reinterpret_cast<const uint8_t*>(blocked) + blocked_f32_offset(g, piece));
  float* o = plain + 4 * i;
  o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
}

// =========================================================================================================
// host orchestration
// =========================================================================================================
// a chain kernel, launched with programmatic stream serialisation: its CTAs may be scheduled while the previous kernel in the
// stream still runs, stage their weights and wait (griddep_wait, tc_chain.cuh) for that kernel's results, so neither the launch
// nor the weight copy sits between two kernels of the encoder
template <int MODE, int FMT>
static void launch_chain(int grid, const ChainArgs& c, cudaStream_t st) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(kChainThreads);
  cfg.dynamicSmemBytes = kChainSmem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, tc_chain_kernel<MODE, FMT>, c);   // a failed launch is reported by the cudaGetLastError at the end
}

template <int FMT>
static cudaError_t tc_configure_fmt() {
  cudaError_t e;
  if ((e = ensure_dynamic_smem(reinterpret_cast<const void*>(tc_chain_kernel<kPCQ, FMT>), kChainSmem))) return e;
  if ((e = ensure_dynamic_smem(reinterpret_cast<const void*>(tc_chain_kernel<kKV, FMT>), kChainSmem))) return e;
  if ((e = ensure_dynamic_smem(reinterpret_cast<const void*>(tc_chain_kernel<kMSG, FMT>), kChainSmem))) return e;
  if ((e = ensure_dynamic_smem(reinterpret_cast<const void*>(tc_chain_kernel<kMSGPC, FMT>), kChainSmem))) return e;
  if ((e = ensure_dynamic_smem(reinterpret_cast<const void*>(tc_chain_kernel<kQ, FMT>), kChainSmem))) return e;
  return ensure_dynamic_smem(reinterpret_cast<const void*>(tc_attention_persistent_kernel<FMT>), kAttnPSmem);
}

template <int FMT>
static int tc_encoder_forward_fmt(const TcWeights& w, const TcForwardArgs& a, cudaStream_t st) {
  const CallShape& plan = a.plan;
  const long long rows = (long long)plan.R;
  if (rows >= (1LL << 31)) return (int)cudaErrorInvalidValue;  // kernels index rows with 32-bit arithmetic
  const TcScratch s = tc_scratch(a.scratch, plan);
  uint8_t *qimg = s.qimg, *kvimg = s.kvimg;
  const long long tiles = (rows + 127) / 128;
  const int num_sms = plan.num_sms;
  if (num_sms <= 0) return (int)cudaErrorInvalidDevice;
  const int grid = (int)(tiles < num_sms ? tiles : num_sms);
  const uint8_t* arena = static_cast<const uint8_t*>(w.arena) + (size_t)FMT * w.num_layers * kLayerBytes;

  launch_layer0(a.corr_pos, a.l0w, a.l0b, a.feat, rows, a.in_dim, st);
  tc_clear_pads_kernel<<<plan.B, 256, 0, st>>>(kvimg, a.sets);
  for (int l = 0; l < a.num_layers; ++l) {
    const uint8_t* base = arena + (size_t)l * kLayerBytes;
    const bool last = l + 1 == a.num_layers;
    ChainArgs c{};
    c.rows = rows; c.split = a.split;
    c.sets = a.sets; c.tile_set = a.tile_set; c.nsets = plan.B;
    c.qimg = qimg; c.kvimg = kvimg; c.bias = reinterpret_cast<const float*>(base + kBias);
    if (l == 0) {   // PointCN + Q
      c.in = a.feat; c.out_f32 = a.feat1; c.wimg = base + kW1; c.wbytes = 131072;
      launch_chain<kPCQ, FMT>(grid, c, st);
    } else {        // Q (the previous layer's MSGPC ran this layer's PointCN)
      c.in = a.feat1; c.out_f32 = nullptr; c.wimg = base + kWq; c.wbytes = 65536;
      launch_chain<kQ, FMT>(grid, c, st);
    }
    // K + V
    c.in = a.feat1; c.out_f32 = nullptr; c.wimg = base + kWk; c.wbytes = 131072;
    launch_chain<kKV, FMT>(grid, c, st);
    // attention
    const AttnArgs at{a.split, qimg, kvimg, a.sc, a.msg, plan.attn_items, s.part_o, s.part_ml, a.sets, plan.B};
    if (a.attn_events) cudaEventRecord(a.attn_events[2 * l], st);
    tc_attention_persistent_kernel<FMT><<<at.items < num_sms ? at.items : num_sms, kAttnThreads, kAttnPSmem, st>>>(at);
    if (plan.attn_split)   // some sets are split: their merge runs per query tile
      tc_attention_merge_kernel<<<(unsigned)(plan.qtiles * 4), 256, 0, st>>>(s.part_o, s.part_ml, a.msg, a.sets, plan.B);
    if (a.attn_events) cudaEventRecord(a.attn_events[2 * l + 1], st);
    if (a.debug_out && a.debug_layer == l) {
      const size_t plane = (size_t)rows * kC;
      tc_unblock_f32_kernel<<<(unsigned)((plane / 4 + 255) / 256), 256, 0, st>>>(a.feat1, a.debug_out, rows);
      tc_decode_kernel<FMT><<<(unsigned)((plane + 255) / 256), 256, 0, st>>>(qimg, kvimg, a.debug_out + plane, a.debug_out + 2 * plane,
                                                                             a.debug_out + 3 * plane, rows, a.sets, plan.B, a.split);
      cudaMemcpyAsync(a.debug_out + 4 * plane, a.msg, plane * sizeof(float), cudaMemcpyDeviceToDevice, st);
    }
    // fc_message + residual; then, but for the last layer (the head reads its feat), the next layer's PointCN, which
    // overwrites feat1 in place and leaves feat in HBM only for the layer_features tap
    const bool tap = a.layer_tap_out && a.layer_tap == l;
    c.in = a.msg; c.res = a.feat1; c.wimg = base + kWm0; c.wbytes = 81920;
    if (last) {
      c.out_f32 = a.feat;
      launch_chain<kMSG, FMT>(grid, c, st);
    } else {
      const uint8_t* next = base + kLayerBytes;
      c.out_f32 = a.feat1; c.feat_out = tap ? a.feat : nullptr;
      c.wimg1 = next + kW1; c.bias1 = reinterpret_cast<const float*>(next + kBias);
      launch_chain<kMSGPC, FMT>(grid, c, st);
    }
    if (tap)
      cudaMemcpyAsync(a.layer_tap_out, a.feat, (size_t)rows * kC * sizeof(float), cudaMemcpyDeviceToDevice, st);
  }
  return (int)cudaGetLastError();
}

int tc_encoder_forward(const TcWeights& w, const TcForwardArgs& a, cudaStream_t st) {
  const cudaError_t e = a.fmt == kFmtBF16 ? tc_configure_fmt<kFmtBF16>() : tc_configure_fmt<kFmtF16>();
  if (e != cudaSuccess) return (int)e;
  return a.fmt == kFmtBF16 ? tc_encoder_forward_fmt<kFmtBF16>(w, a, st) : tc_encoder_forward_fmt<kFmtF16>(w, a, st);
}

}  // namespace pdsc
