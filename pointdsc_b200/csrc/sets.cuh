// Per-set descriptors of a forward call.
//
// A uniform call (pdsc_forward) holds B sets of N rows each; a packed call (pdsc_forward_packed) holds B sets of N_b rows
// each, packed back to back.  Every kernel whose work depends on a set's size asks `set_desc` for it: a packed call reads
// the table that set_table_kernel (engine.cu) wrote into its workspace; a uniform call passes no table and the same
// descriptor is computed from (b, N, S, k), so that its indexing and results are exactly those of the uniform-only kernels.
#pragma once
#include <stdint.h>

namespace pdsc {

struct SetDesc {
  int row0;        // first row of the set in the call's [R] arrays
  int N, S, k;     // correspondences, seeds S = int(N ratio), neighbours k = min(cfg.k, N - 1)
  int qt0, kt0;    // first 128-query tile / 64-key tile of the set in the Q / KV operand images
  int seed0;       // first seed slot of the set ([sum S] arrays)
  int item0;       // first attention work item of the set
  int sp, TS;      // key splits of the attention and key tiles per split (sp == 1: TS == KT)
  int pad0, pad1;
  long long sc0;   // first float of the set's SC block (tiled or row-major)
  long long dist0; // first float of the set's seed-row distance block [S][N] (a multiple of 4)
  long long knn0;  // first neighbour slot of the set ([sum S k] arrays; iterates are `iters` times that)
};

// The uniform call's geometry, with the table pointer of a packed call (nullptr for a uniform call).
struct SetTable {
  const SetDesc* d;
  int N, S, k;     // uniform call: the shape.  Packed call: the largest N, S and k of the call (launch sizes only)
  int tiled;       // SC layout: 1 tiled (tensor-core precisions), 0 row-major with stride round_up(N, 64)
  int sp, TS;      // uniform call: the attention's key split
};

__host__ __device__ __forceinline__ SetDesc set_desc(const SetTable& t, int b) {
  if (t.d) return t.d[b];
  SetDesc d;
  const int N = t.N, QT = (N + 127) / 128, KT = (N + 63) / 64;
  d.row0 = b * N;
  d.N = N; d.S = t.S; d.k = t.k;
  d.qt0 = b * QT; d.kt0 = b * KT;
  d.seed0 = b * t.S;
  d.item0 = b * QT * t.sp;
  d.sp = t.sp; d.TS = t.TS;
  d.pad0 = d.pad1 = 0;
  d.sc0 = t.tiled ? (long long)b * KT * QT * 8192 : (long long)b * N * ((N + 63) / 64 * 64);
  d.dist0 = (long long)b * t.S * N;
  d.knn0 = (long long)b * t.S * t.k;
  return d;
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

// the set b of a packed call with first(b) <= x < first(b + 1), `first` ascending in b
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
