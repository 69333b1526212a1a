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

struct TcForwardArgs {
  int nsets, in_dim, num_layers;
  int split;                 // 1: hi/lo operand split (3 products)   0: single 16-bit operands
  int fmt;                   // operand format of the kind::f16 MMAs: 0 = fp16, 1 = bf16
  const float* corr_pos;     // [rows][in_dim]
  const float *l0w, *l0b;    // layer0 weights (fp32, device)
  const float* sc;           // tiled SC blocks of the sets (SetDesc::sc0)
  float* feat;               // [rows][128]  layer output / final features
  float* feat1;              // [rows][128]  PointCN output (residual source)
  float* msg;                // [rows][128]  attention output
  void* scratch;             // tc_scratch_bytes_tiles(qtiles, ktiles, attn_invariant, attn_split, attn_items)
  int layer_tap;             // -1 or layer index to copy out
  float* layer_tap_out;
  int debug_layer;           // layer whose internals are decoded into debug_out
  float* debug_out;          // [5][rows][128]: feat1, q (scaled by log2e/sqrt(C)), k, v, msg — or nullptr
  cudaEvent_t* attn_events;  // nullptr or 2 events per layer, recorded around the attention launch
  const SetDesc* sets;       // the call's descriptor table (sets.cuh), nsets entries
  const int* tile_set;       // the set of the first row of every 128-row tile of the call's rows
  long long rows;            // rows of the call
  long long qtiles, ktiles;  // query / key tiles of all sets
  int attn_items;            // attention work items (tc_packed_split)
  int attn_split;            // 1: the call is in the key-split regime
  int attn_invariant;        // 1: batch-invariant key split (attn_set_split_invariant)
};

int tc_build_weights(const TcLayerHost* layers, int num_layers, TcWeights* out);  // returns cudaError_t
void tc_free_weights(TcWeights* w);
size_t tc_scratch_bytes_tiles(long long qtiles, long long ktiles, int invariant, int attn_split, int attn_items);
// key-split decision of a call of sets of Ns[0..B) rows (invariant: the batch-invariant rule): returns 1 if the call runs
// the merge; *items = attention work items
int tc_packed_split(const int* Ns, int B, int invariant, int* items);
int tc_launches(int num_layers, int attn_split);
int tc_encoder_forward(const TcWeights& w, const TcForwardArgs& a, cudaStream_t st);  // returns cudaError_t

}  // namespace pdsc
