// Per-set descriptors of a forward call.
//
// A forward call holds B sets of N_b rows each, packed back to back: a packed call (pdsc_forward_packed) takes their offsets,
// a uniform call (pdsc_forward) is the packed call whose offsets are b * N.  set_table_kernel (engine.cu) writes one SetDesc
// per set into the workspace at the start of every call, and every kernel whose work depends on a set's size reads it from
// that table.  A set's indexing is therefore the same whichever entry point ran it.
#pragma once
#include <stdint.h>

namespace pdsc {

struct SetDesc {
  int row0;        // first row of the set in the call's [R] arrays
  int N, S, k;     // correspondences, seeds S = num_seeds(N, ratio), neighbours k = min(cfg.k, N - 1)
  int qt0, kt0;    // first 128-query tile / 64-key tile of the set in the Q / KV operand images
  int seed0;       // first seed slot of the set ([sum S] arrays)
  int item0;       // first attention work item of the set
  int sp, TS;      // key splits of the attention and key tiles per split (sp == 1: TS == KT)
  int pad0, pad1;
  long long sc0;   // first float of the set's SC block (tiled or row-major)
  long long dist0; // first float of the set's seed-row distance block [S][N] (a multiple of 4)
  long long knn0;  // first neighbour slot of the set ([sum S k] arrays; iterates are `iters` times that)
};

// Seeds of a set of N rows: the length of the slice argsort(...)[:, 0:int(N * ratio)] the reference takes (PointDSC.py:174,
// :176, :217), the product and the truncation in double as Python evaluates them.  With m = int(N * ratio) that is min(m, N)
// for m >= 0 and max(N + m, 0) for m < 0: a ratio above 1 takes every row, a negative one drops the last -m.  The product is
// clamped to [-N, N] before the conversion, so no ratio makes it undefined; a NaN ratio gives 0 (pdsc_create refuses one).
__host__ __device__ __forceinline__ int num_seeds(int N, double ratio) {
  const double x = (double)N * ratio;
  if (!(x > -(double)N)) return 0;                   // m <= -N (or NaN)
  if (x >= (double)N) return N;                      // m >= N
  const int m = (int)x;                              // truncation toward zero, as int()
  return m >= 0 ? m : N + m;
}

// Key split of the tensor-core attention for ONE set of N rows in a call of the small regime (encoder_tc.cu): sp chunks of TS key
// tiles, a function of N and the SM count only.  sp == 1 (TS == KT): not split.
__host__ __device__ __forceinline__ void attn_set_split(int N, int num_sms, int* sp, int* TS) {
  const int QT = (N + 127) / 128, KT = (N + 63) / 64;
  *sp = 1;
  *TS = KT;
  if (KT < 4) return;
  const int want = (num_sms + QT - 1) / QT;          // splits that would fill the SMs with ONE set
  int ts = (KT + want - 1) / want;
  if (ts < 2) ts = 2;
  const int s = (KT + ts - 1) / ts;
  if (s < 2) return;
  *sp = s;
  *TS = ts;
}

// Key tiles per split of the batch-invariant mode (pdsc_set_batch_invariant).  Part of that mode's results: a different value
// associates the softmax sums of every set with more than this many key tiles differently.  Chosen from the measurement in
// DESIGN.md §4.
#ifndef PDSC_ATTN_INVARIANT_TILES
#define PDSC_ATTN_INVARIANT_TILES 8
#endif
constexpr int kAttnInvariantTiles = PDSC_ATTN_INVARIANT_TILES;

// Key split of the tensor-core attention for one set of N rows in the batch-invariant mode: a function of N alone (no SM
// count, no batch, no item cap), so a set gives the same bytes in every call and on every device.  sp == 1: not split.
__host__ __device__ __forceinline__ void attn_set_split_invariant(int N, int* sp, int* TS) {
  const int KT = (N + 63) / 64;
  *sp = (KT + kAttnInvariantTiles - 1) / kAttnInvariantTiles;
  *TS = (KT + *sp - 1) / *sp;
}

// Row offsets of a packed call of the stateless entry points (matching, statistics): set b owns rows [at(b), at(b + 1)), read
// from a device table of B + 1 entries, or b * stride when the table is null (one set, or sets of equal size).
struct Offsets {
  const int32_t* table;
  int stride;
  __host__ __device__ __forceinline__ int at(int b) const { return table ? table[b] : b * stride; }
};

// the set b of a call with first(b) <= x < first(b + 1), `first` ascending in b
template <typename F>
__device__ __forceinline__ int find_set(int nsets, long long x, F first) {
  int lo = 0, hi = nsets - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (first(mid) <= x) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

}  // namespace pdsc
