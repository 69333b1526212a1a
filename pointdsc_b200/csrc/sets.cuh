// Per-set descriptors of a forward call, and the plan that sizes it.
//
// A forward call holds B sets of N_b rows each, packed back to back: a packed call (pdsc_forward_packed) takes their offsets,
// a uniform call (pdsc_forward) is the packed call whose offsets are b * N.  set_table_kernel (engine.cu) writes one SetDesc
// per set into the workspace at the start of every call, and every kernel whose work depends on a set's size reads it from
// that table.  A set's indexing is therefore the same whichever entry point ran it.
//
// The host sizes a call's workspace from plan_call, and set_table_kernel writes each set's offsets into it from the same
// set_sizes and attn_key_split, so a set's blocks land inside the regions the workspace holds.
#pragma once
#include <stddef.h>
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

// What one set of N rows occupies in a forward call.
struct SetSizes {
  int S, k;                          // seeds num_seeds(N, ratio), neighbours min(k_cfg, N - 1) (at least 0)
  int QT, KT;                        // 128-query tiles and 64-key tiles of the Q / KV operand images
  int NS;                            // row length of the row-major SC block: N rounded up to 64
  long long sc_rowmajor, sc_tiled;   // floats of the SC block: row-major [N][NS] (fp32), tiled [KT][QT][128 x 64] (tensor cores)
  long long dist;                    // floats of the seed-row distance block [S][N], rounded up to 4 (16-byte aligned blocks)
  long long knn;                     // neighbour slots S * k
};

__host__ __device__ __forceinline__ SetSizes set_sizes(int N, double ratio, int k_cfg) {
  SetSizes z;
  z.S = num_seeds(N, ratio);
  z.k = k_cfg < N - 1 ? k_cfg : N - 1;   // k = min(self.k, num_corr - 1)  (PointDSC.py:250)
  if (z.k < 0) z.k = 0;
  z.QT = (N + 127) / 128;
  z.KT = (N + 63) / 64;
  z.NS = z.KT * 64;
  z.sc_rowmajor = (long long)N * z.NS;
  z.sc_tiled = (long long)z.KT * z.QT * 8192;
  z.dist = ((long long)z.S * N + 3) & ~3ll;
  z.knn = (long long)z.S * z.k;
  return z;
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

// Key split of a set of N rows in a call that runs split (attn_call_splits).
__host__ __device__ __forceinline__ void attn_key_split(int N, int invariant, int num_sms, int* sp, int* TS) {
  if (invariant) attn_set_split_invariant(N, sp, TS);
  else attn_set_split(N, num_sms, sp, TS);
}

// Key split of a call of the default mode: at most this many work items, each with a 64 KB partial O and 1 KB of (m, l)
constexpr int kAttnSplitMaxItems = 320;

// Key split policy of a call whose sets hold `qtiles` (set, query tile) items, and `items` when each set is split by
// attn_key_split.  Default mode: when the items cover at most half of the SMs (the evaluation loops' bs = 1: 8 items at
// N = 1000, 40 at N = 5000), the call is in the split regime, in which a set's split is a function of its N and the SM count
// only.  Calls of the small regime therefore agree bit for bit whatever their batch size, and so do calls of the large regime
// (no split); across the two regimes the softmax sums are associated differently (fp32 rounding, far inside the parity bar).  A
// call whose split would exceed kAttnSplitMaxItems work items, or in which no set would split, is not split.
// Batch-invariant mode: the call splits whenever one of its sets has sp > 1.  No regime, no item cap: the partial buffers are
// sized by the call's items.
__host__ __device__ __forceinline__ bool attn_call_splits(long long qtiles, long long items, int num_sms, int invariant) {
  return invariant ? items > qtiles : 2 * qtiles <= num_sms && qtiles < items && items <= kAttnSplitMaxItems;
}

// The plan of a forward call of B sets: what sizes its workspace, its grids and its attention's key split.  N, S and k are the
// largest of its sets (launch sizes), k_min the smallest k of its sets with seeds, and the totals sum set_sizes over the sets.
struct CallShape {
  int B = 0, N = 0, S = 0, k = 0, k_min = 0;
  size_t R = 0;
  size_t sc_rowmajor = 0, sc_tiled = 0;   // floats of the row-major (fp32) and tiled (tensor-core) SC layouts
  size_t seeds = 0, dist = 0, knn = 0;    // seed slots, seed-row distance floats, neighbour slots
  long long qtiles = 0, ktiles = 0;
  int attn_items = 0;                     // tensor-core attention work items: qtiles, or the split items when attn_split
  int attn_split = 0;                     // 1: the tensor-core attention splits its sets' keys and runs the merge
  int attn_invariant = 0;                 // the engine's key-split policy (pdsc_set_batch_invariant)
  int num_sms = 0;                        // the SM count the split was decided with, which the table and the grids use too
};

// h_offsets: the offsets [B + 1] of a packed call, or nullptr for B sets of N_uniform rows.  tc: a tensor-core call (the
// SIMT attention has no key split).
inline CallShape plan_call(int B, int N_uniform, const int32_t* h_offsets, double ratio, int k_cfg, bool tc, int invariant,
                           int num_sms) {
  CallShape s;
  s.B = B;
  s.k_min = k_cfg;
  s.attn_invariant = invariant;
  s.num_sms = num_sms;
  long long split_items = 0;
  for (int b = 0; b < B; ++b) {
    const int N = h_offsets ? h_offsets[b + 1] - h_offsets[b] : N_uniform;
    const SetSizes z = set_sizes(N, ratio, k_cfg);
    int sp, TS;
    attn_key_split(N, invariant, num_sms, &sp, &TS);
    s.R += (size_t)N;
    if (N > s.N) s.N = N;
    if (z.S > s.S) s.S = z.S;
    if (z.k > s.k) s.k = z.k;
    if (z.S > 0 && z.k < s.k_min) s.k_min = z.k;
    s.sc_rowmajor += (size_t)z.sc_rowmajor;
    s.sc_tiled += (size_t)z.sc_tiled;
    s.seeds += (size_t)z.S;
    s.dist += (size_t)z.dist;
    s.knn += (size_t)z.knn;
    s.qtiles += z.QT;
    s.ktiles += z.KT;
    split_items += (long long)z.QT * sp;
  }
  if (tc) {
    s.attn_split = attn_call_splits(s.qtiles, split_items, num_sms, invariant) ? 1 : 0;
    s.attn_items = (int)(s.attn_split ? split_items : s.qtiles);
  }
  return s;
}

// work items whose partial results the tensor-core scratch holds: a fixed kAttnSplitMaxItems in the default mode (its split is
// capped there), every work item of a split call in the batch-invariant mode
inline size_t attn_partial_items(const CallShape& sh) {
  return sh.attn_invariant ? (sh.attn_split ? (size_t)sh.attn_items : 0) : (size_t)kAttnSplitMaxItems;
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
