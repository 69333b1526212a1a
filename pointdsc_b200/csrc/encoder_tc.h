// Tensor-core (wgmma) encoder path — host-visible interface.  See encoder_tc.cu.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "sets.cuh"

namespace pdsc {

// Host pointers to one layer's folded fp32 weights (row-major [Cout][Cin]) and biases.
struct TcLayerHost {
  const float *w1, *b1, *wq, *bq, *wk, *bk, *wv, *bv, *wm0, *bm0, *wm1, *bm1, *wm2, *bm2;
};

// Device-resident operand images built once per pdsc_commit_params().
struct TcWeights {
  void* arena = nullptr;   // all images + biases
  size_t arena_bytes = 0;
  int num_layers = 0;
};

// The encoder's scratch: Q images [qtiles][64 KB], K / V images [ktiles][64 KB], then the key split's partial O
// [items][128][128] and (m, l) [items][128][2] (fp32), from the first 1024-byte boundary of the buffer (the SWIZZLE_128B atoms
// of the bulk copies).  tc_scratch(nullptr, plan).bytes sizes the buffer; tc_scratch(buffer, plan) carves it.
struct TcScratch {
  uint8_t *qimg, *kvimg;
  float *part_o, *part_ml;
  size_t bytes;
};

struct TcForwardArgs {
  const CallShape& plan;     // the call's plan (sets.cuh): sets, rows, tiles, the attention's items and key split
  int in_dim, num_layers;
  int split;                 // 1: hi/lo operand split (3 products)   0: single 16-bit operands
  int fmt;                   // operand format of the kind::f16 MMAs: 0 = fp16, 1 = bf16
  const float* corr_pos;     // [rows][in_dim]
  const float *l0w, *l0b;    // layer0 weights (fp32, device)
  const float* sc;           // tiled SC blocks of the sets (SetDesc::sc0)
  float* feat;               // [rows][128]  layer output / final features
  float* feat1;              // [rows][128]  PointCN output (residual source)
  float* msg;                // [rows][128]  attention output
  void* scratch;             // tc_scratch(nullptr, plan).bytes bytes
  int layer_tap;             // -1 or layer index to copy out
  float* layer_tap_out;
  int debug_layer;           // layer whose internals are decoded into debug_out
  float* debug_out;          // [5][rows][128]: feat1, q (scaled by log2e/sqrt(C)), k, v, msg — or nullptr
  cudaEvent_t* attn_events;  // nullptr or 2 events per layer, recorded around the attention launch
  const SetDesc* sets;       // the call's descriptor table (sets.cuh), plan.B entries
  const int* tile_set;       // the set of the first row of every 128-row tile of the call's rows
};

int tc_build_weights(const TcLayerHost* layers, int num_layers, TcWeights* out);  // returns cudaError_t
void tc_free_weights(TcWeights* w);
TcScratch tc_scratch(void* base, const CallShape& plan);
int tc_launches(int num_layers, int attn_split);
int tc_encoder_forward(const TcWeights& w, const TcForwardArgs& a, cudaStream_t st);  // returns cudaError_t

}  // namespace pdsc
