// f8 — FCGF descriptors on the device: the ResUNetBN2C sparse-convolution network of misc/fcgf.py:621-867 with the
// quantisation of misc/cal_fcgf.py:11-85 (rgb = normal = None), for P clouds in one call.  MinkowskiEngine, which the reference
// runs it on, is not a dependency of this project: its conventions are stated in DESIGN.md row f8 (PARITY UNPINNED).
//
// Everything is fp32 and deterministic: no value depends on the order atomics arrive in, a row's sums run in one fixed order,
// and nothing a cloud computes reads another cloud's rows, so a cloud's rows are bit for bit the same in any group, in any order
// and on any SM count.
//
// Rows.  Every level l (tensor stride 2^l, l = 0..3) packs the clouds' rows back to back; lvl_off[l] [P+1] lives on the device
// only, and every buffer is sized by the input's n = offsets[P] rows (a level never has more rows than its cloud has points).
// Launches are sized by that bound; rows at or beyond lvl_off[l][P] return at once.  No host read, capturable in a graph.
//
// quantise     level 0: c = floor((double)x / voxel) as int32 (status bit 1 for a non-finite c or one outside [-2^20, 2^20));
//              level l: floor(c / 2^l) 2^l of level l-1's rows.  Each item is inserted in its cloud's hash region
//              (voxel_hash.cuh, coordinates biased by 2^20 into 21-bit fields), the representative of a voxel is its smallest
//              item index (atomicMin), and the representatives are numbered by a scan in item order: rows come out in order of
//              first occurrence.  Level 0's key point is xyz[representative].
// maps         one int32 [rows, K^3] table per level and kind, -1 where the neighbour is absent, offset index
//              (ox+r) + K(oy+r) + K^2(oz+r): same-stride c + o 2^l (tables 0..3), conv1 c + o (K = 5 or 7), strided (coarse row
//              of level l gathers level l-1 at c + o 2^(l-1)), transposed (fine row of level l gathers level l+1 at c - o 2^l).
// conv         output-stationary gather GEMM: a CTA owns 64 rows x 32 or 64 output channels; for each offset in ascending order
//              it gathers the 64 neighbour rows 32 input channels at a time (zeros for -1) and multiplies them by W[o] from
//              shared memory, 4 x 2 or 4 x 4 FFMA accumulators per thread.  Epilogue: folded BN (acc * scale + shift), an optional
//              residual, an optional ReLU, stored into a column range of the concatenation buffer (ME.cat costs nothing).
// conv1        Cin = 1 and the input is the constant 1, so out = sum of W[o] over the occupied offsets: one warp per row.
// head         conv1_tr (96 -> 64), ReLU, final (64 -> 32, bias), x / (||x|| + 1e-8): one warp per row.
#include <math.h>

#include <algorithm>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/pointdsc_b200.h"
#include "common.cuh"
#include "kernels.h"
#include "voxel_hash.cuh"

namespace pdsc {

namespace {

constexpr int kLevels = 4;
constexpr int kCoordLimit = 1 << 20;     // |voxel coordinate| bound: 21-bit fields with a 2^20 bias
constexpr int kScanBlock = 1024;         // items per block of the representative scan
constexpr double kBnEps = 1e-5;

enum MapKind { MAP_C1 = 0, MAP_SAME = 1, MAP_DOWN = 2, MAP_UP = 3 };

// Feature buffers (widths) of the forward, one per level and role: x = a level's first conv, t = a block's inner conv,
// cat = [decoder | skip] concatenation, d / dt = the decoder's transposed conv and its block's inner conv, s8 = the bottom.
enum Feat {
  F_X0, F_T0, F_CAT0, F_D0, F_DT0,
  F_X1, F_T1, F_CAT1, F_D1, F_DT1,
  F_X2, F_T2, F_CAT2, F_D2, F_DT2,
  F_X3, F_T3, F_S8, F_COUNT
};
constexpr int kFeatWidth[F_COUNT] = {32, 32, 96, 64, 64, 64, 64, 128, 64, 64, 128, 128, 256, 128, 128, 256, 256, 256};

// One convolution of ResUNet2.forward (misc/fcgf.py:800-852) in order: name, map kind, output level, input (buffer, first
// column), residual (buffer or -1, first column), output (buffer, first column), Cout, BN prefix, ReLU.
struct Step {
  const char* name; int kind, level, in, in_col, res, res_col, out, out_col, cout; const char* norm; int relu;
};
constexpr Step kSteps[] = {
    {"conv1", MAP_C1, 0, -1, 0, -1, 0, F_X0, 0, 32, "norm1", 0},
    {"block1.conv1", MAP_SAME, 0, F_X0, 0, -1, 0, F_T0, 0, 32, "block1.norm1", 1},
    {"block1.conv2", MAP_SAME, 0, F_T0, 0, F_X0, 0, F_CAT0, 64, 32, "block1.norm2", 1},
    {"conv2", MAP_DOWN, 1, F_CAT0, 64, -1, 0, F_X1, 0, 64, "norm2", 0},
    {"block2.conv1", MAP_SAME, 1, F_X1, 0, -1, 0, F_T1, 0, 64, "block2.norm1", 1},
    {"block2.conv2", MAP_SAME, 1, F_T1, 0, F_X1, 0, F_CAT1, 64, 64, "block2.norm2", 1},
    {"conv3", MAP_DOWN, 2, F_CAT1, 64, -1, 0, F_X2, 0, 128, "norm3", 0},
    {"block3.conv1", MAP_SAME, 2, F_X2, 0, -1, 0, F_T2, 0, 128, "block3.norm1", 1},
    {"block3.conv2", MAP_SAME, 2, F_T2, 0, F_X2, 0, F_CAT2, 128, 128, "block3.norm2", 1},
    {"conv4", MAP_DOWN, 3, F_CAT2, 128, -1, 0, F_X3, 0, 256, "norm4", 0},
    {"block4.conv1", MAP_SAME, 3, F_X3, 0, -1, 0, F_T3, 0, 256, "block4.norm1", 1},
    {"block4.conv2", MAP_SAME, 3, F_T3, 0, F_X3, 0, F_S8, 0, 256, "block4.norm2", 1},
    {"conv4_tr", MAP_UP, 2, F_S8, 0, -1, 0, F_D2, 0, 128, "norm4_tr", 0},
    {"block4_tr.conv1", MAP_SAME, 2, F_D2, 0, -1, 0, F_DT2, 0, 128, "block4_tr.norm1", 1},
    {"block4_tr.conv2", MAP_SAME, 2, F_DT2, 0, F_D2, 0, F_CAT2, 0, 128, "block4_tr.norm2", 1},
    {"conv3_tr", MAP_UP, 1, F_CAT2, 0, -1, 0, F_D1, 0, 64, "norm3_tr", 0},
    {"block3_tr.conv1", MAP_SAME, 1, F_D1, 0, -1, 0, F_DT1, 0, 64, "block3_tr.norm1", 1},
    {"block3_tr.conv2", MAP_SAME, 1, F_DT1, 0, F_D1, 0, F_CAT1, 0, 64, "block3_tr.norm2", 1},
    {"conv2_tr", MAP_UP, 0, F_CAT1, 0, -1, 0, F_D0, 0, 64, "norm2_tr", 0},
    {"block2_tr.conv1", MAP_SAME, 0, F_D0, 0, -1, 0, F_DT0, 0, 64, "block2_tr.norm1", 1},
    {"block2_tr.conv2", MAP_SAME, 0, F_DT0, 0, F_D0, 0, F_CAT0, 0, 64, "block2_tr.norm2", 1},
};
constexpr int kNumSteps = sizeof(kSteps) / sizeof(kSteps[0]);

int step_cin(const Step& s) {
  if (s.kind == MAP_C1) return 1;
  return kFeatWidth[s.in] - s.in_col;
}
int step_k(const Step& s, int k1) { return s.kind == MAP_C1 ? k1 * k1 * k1 : 27; }

// The scratch: one carve for sizing (null base) and for use, so the two cannot disagree.  Regions are 256-byte aligned and
// listed in the order pdsc_fcgf_scratch_layout() reports them.
struct Scratch {
  int32_t* lvl_off[kLevels];          // [P+1] rows of every cloud at level l
  int32_t* coords[kLevels];           // [n,3] voxel coordinates (multiples of 2^l)
  int32_t* map_c1;                    // [n,K1^3]
  int32_t* map_same[kLevels];         // [n,27]
  int32_t* map_down[kLevels];         // [n,27] l = 1..3 (index 0 unused, null)
  int32_t* map_up[kLevels];           // [n,27] l = 0..2 (index 3 unused, null)
  float* feat[F_COUNT];               // [n,width]
  // quantisation working state (not reported)
  int32_t* rep0;                      // [n] level 0 representative (input point index)
  unsigned long long* slot0;          // [P+1]
  unsigned long long* keys[kLevels];  // [S]
  int32_t* first[kLevels];            // [S] smallest item index of the voxel
  int32_t* row_of[kLevels];           // [S] the voxel's row
  unsigned long long* islot;          // [n] slot of every item (~0: not inserted)
  uint32_t* flags;                    // [n/32 + 1] representative bits
  int32_t* bbase;                     // [blocks + 1] rows before every scan block
  std::vector<size_t> reported;       // byte offsets of the reported regions
  size_t bytes;
};

Scratch carve(void* base, int P, const int32_t* h_off, int k1) {
  Scratch s{};
  unsigned char* b = static_cast<unsigned char*>(base);
  size_t at = 0;
  auto take = [&](size_t bytes, bool report) -> void* {
    at = (at + 255) & ~size_t(255);
    if (report) s.reported.push_back(at);
    void* p = b ? b + at : nullptr;
    at += bytes;
    return p;
  };
  const size_t n = (size_t)h_off[P];
  const unsigned long long S = total_slots(P, h_off);
  const size_t blocks = (n + kScanBlock - 1) / kScanBlock;
  for (int l = 0; l < kLevels; ++l) s.lvl_off[l] = (int32_t*)take((size_t)(P + 1) * 4, true);
  for (int l = 0; l < kLevels; ++l) s.coords[l] = (int32_t*)take(n * 12, true);
  s.map_c1 = (int32_t*)take(n * k1 * k1 * k1 * 4, true);
  for (int l = 0; l < kLevels; ++l) s.map_same[l] = (int32_t*)take(n * 27 * 4, true);
  for (int l = 1; l < kLevels; ++l) s.map_down[l] = (int32_t*)take(n * 27 * 4, true);
  for (int l = 0; l + 1 < kLevels; ++l) s.map_up[l] = (int32_t*)take(n * 27 * 4, true);
  for (int f = 0; f < F_COUNT; ++f) s.feat[f] = (float*)take(n * kFeatWidth[f] * 4, true);
  s.rep0 = (int32_t*)take(n * 4, false);
  s.slot0 = (unsigned long long*)take((size_t)(P + 1) * 8, false);
  for (int l = 0; l < kLevels; ++l) {
    s.keys[l] = (unsigned long long*)take(S * 8, false);
    s.first[l] = (int32_t*)take(S * 4, false);
    s.row_of[l] = (int32_t*)take(S * 4, false);
  }
  s.islot = (unsigned long long*)take(n * 8, false);
  s.flags = (uint32_t*)take((n / 32 + 1) * 4, false);
  s.bbase = (int32_t*)take((blocks + 1) * 4, false);
  s.bytes = (at + 255) & ~size_t(255);
  return s;
}

// ---- quantisation and pyramid ----------------------------------------------------------------------------------------
__global__ void fq_init_kernel(unsigned long long* k0, unsigned long long* k1, unsigned long long* k2, unsigned long long* k3,
                               int32_t* f0, int32_t* f1, int32_t* f2, int32_t* f3, unsigned long long S, int P, int32_t* status) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < S) {
    k0[i] = kEmptyKey; k1[i] = kEmptyKey; k2[i] = kEmptyKey; k3[i] = kEmptyKey;
    f0[i] = INT_MAX; f1[i] = INT_MAX; f2[i] = INT_MAX; f3[i] = INT_MAX;
  }
  if (i < (unsigned long long)P) status[i] = 0;
}

__device__ __forceinline__ unsigned long long coord_key(int x, int y, int z) {
  return pack_key21((unsigned long long)(x + kCoordLimit), (unsigned long long)(y + kCoordLimit), (unsigned long long)(z + kCoordLimit));
}
__device__ __forceinline__ bool coord_ok(long long x) { return x >= -kCoordLimit && x < kCoordLimit; }

// item i of level l: a point (l = 0) or a row of level l - 1; inserted into its cloud's region of table l
__global__ void fq_insert_kernel(int level, long long n, int P, const int32_t* __restrict__ in_off, const float* __restrict__ pts,
                                 double voxel, const int32_t* __restrict__ in_coords, const unsigned long long* __restrict__ slot0,
                                 unsigned long long* keys, int32_t* first, unsigned long long* islot, int32_t* out_coords_tmp,
                                 int32_t* status) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  islot[i] = ~0ull;
  if (i >= in_off[P]) return;
  const int p = find_set(P, i, [&](int q) { return (long long)in_off[q]; });
  int c[3];
  if (level == 0) {
    bool bad = false;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double f = floor((double)pts[3 * i + a] / voxel);
      bad |= !(f >= -(double)kCoordLimit && f < (double)kCoordLimit);     // also catches NaN / inf
      c[a] = bad ? 0 : (int)f;
    }
    if (bad) {
      atomicOr(&status[p], 1);
      return;
    }
  } else {
    const int mask = ~((1 << level) - 1);         // floor(c / 2^l) 2^l in two's complement
#pragma unroll
    for (int a = 0; a < 3; ++a) c[a] = in_coords[3 * i + a] & mask;
  }
  out_coords_tmp[3 * i] = c[0]; out_coords_tmp[3 * i + 1] = c[1]; out_coords_tmp[3 * i + 2] = c[2];
  const unsigned long long base = slot0[p];
  const unsigned long long s = hash_insert(keys, base, slot0[p + 1] - base - 1, coord_key(c[0], c[1], c[2]));
  atomicMin(&first[s], (int)i);
  islot[i] = s;
}

// representative bits (item i is the smallest of its voxel) and the count of every scan block
__global__ void __launch_bounds__(kScanBlock) fq_flag_kernel(long long n, const unsigned long long* __restrict__ islot,
                                                             const int32_t* __restrict__ first, uint32_t* flags, int32_t* bcount) {
  __shared__ int warp_cnt[kScanBlock / 32];
  const long long i = (long long)blockIdx.x * kScanBlock + threadIdx.x;
  bool rep = false;
  if (i < n) {
    const unsigned long long s = islot[i];
    rep = s != ~0ull && first[s] == (int)i;
  }
  const uint32_t b = __ballot_sync(0xffffffffu, rep);
  if ((threadIdx.x & 31) == 0) {
    if (i < n) flags[i >> 5] = b;
    warp_cnt[threadIdx.x >> 5] = __popc(b);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < kScanBlock / 32; ++w) t += warp_cnt[w];
    bcount[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(1024) fq_scan_kernel(int blocks, int32_t* bbase) {
  // bbase holds the block counts in [1, blocks]; it becomes the exclusive scan in [0, blocks] (bbase[blocks] = all rows)
  cta_offsets<int32_t>(blocks, [&](int q) { return bbase[q + 1]; }, (int32_t*)nullptr, bbase + 1);
  if (threadIdx.x == 0) bbase[0] = 0;
}

// rows before item j of the level: representatives at items < j
__device__ __forceinline__ int rows_before(long long j, const uint32_t* __restrict__ flags, const int32_t* __restrict__ bbase) {
  const long long blk = j / kScanBlock;
  int r = bbase[blk];
  for (long long w = blk * (kScanBlock / 32); w < (j >> 5); ++w) r += __popc(flags[w]);
  if (j & 31) r += __popc(flags[j >> 5] & ((1u << (j & 31)) - 1u));
  return r;
}

__global__ void fq_write_kernel(int level, long long n, const uint32_t* __restrict__ flags, const int32_t* __restrict__ bbase,
                                const unsigned long long* __restrict__ islot, const int32_t* __restrict__ tmp_coords,
                                int32_t* row_of, int32_t* coords, int32_t* rep0) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !((flags[i >> 5] >> (i & 31)) & 1u)) return;
  const int row = rows_before(i, flags, bbase);
  row_of[islot[i]] = row;
  coords[3 * (size_t)row] = tmp_coords[3 * i]; coords[3 * (size_t)row + 1] = tmp_coords[3 * i + 1];
  coords[3 * (size_t)row + 2] = tmp_coords[3 * i + 2];
  if (level == 0) rep0[row] = (int)i;
}

__global__ void fq_offsets_kernel(int P, long long n, const int32_t* __restrict__ in_off, const uint32_t* __restrict__ flags,
                                  const int32_t* __restrict__ bbase, int32_t* lvl_off) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > P) return;
  const long long j = in_off[p];
  lvl_off[p] = j >= n ? bbase[(n + kScanBlock - 1) / kScanBlock] : rows_before(j, flags, bbase);
}

// ---- neighbour tables ------------------------------------------------------------------------------------------------
// map[row][o] = the row of table `t` at coords[row] + o * mult, or -1
__global__ void fmap_kernel(long long n, int P, const int32_t* __restrict__ lvl_off, const int32_t* __restrict__ coords, int K,
                            int mult, const unsigned long long* __restrict__ slot0, const unsigned long long* __restrict__ keys,
                            const int32_t* __restrict__ row_of, int32_t* __restrict__ map) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int K3 = K * K * K;
  if (e >= n * K3) return;
  const long long row = e / K3;
  if (row >= lvl_off[P]) return;
  const int o = (int)(e - row * K3), r = (K - 1) / 2;
  const int ox = o % K - r, oy = (o / K) % K - r, oz = o / (K * K) - r;
  const int p = find_set(P, row, [&](int q) { return (long long)lvl_off[q]; });
  const long long x = (long long)coords[3 * row] + (long long)ox * mult, y = (long long)coords[3 * row + 1] + (long long)oy * mult,
                  z = (long long)coords[3 * row + 2] + (long long)oz * mult;
  int out = -1;
  if (coord_ok(x) && coord_ok(y) && coord_ok(z)) {
    const unsigned long long base = slot0[p];
    const unsigned long long s = hash_find(keys, base, slot0[p + 1] - base - 1, coord_key((int)x, (int)y, (int)z));
    if (s != ~0ull) out = row_of[s];
  }
  map[e] = out;
}

// ---- convolutions ----------------------------------------------------------------------------------------------------
constexpr int kBM = 64, kCK = 32;

struct ConvArgs {
  const int32_t* map; int K;
  const float* in; int ldin, cin;
  const float* W;                      // [K][cin][cout]
  const float* scale; const float* shift;
  const float* res; int ldres;
  float* out; int ldo, cout, relu;
  const int32_t* rows;                 // device: the level's row count
};

template <int BN>
__global__ void __launch_bounds__(256) fconv_kernel(ConvArgs a) {
  constexpr int TN = BN / 16;
  __shared__ float As[kCK][kBM + 4];
  __shared__ float Bs[kCK][BN];
  __shared__ int nb[kBM];
  const int M = *a.rows;
  const int row0 = blockIdx.x * kBM;
  if (row0 >= M) return;
  const int col0 = blockIdx.y * BN;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][TN];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
  for (int o = 0; o < a.K; ++o) {
    __syncthreads();
    if (threadIdx.x < kBM) {
      const int r = row0 + threadIdx.x;
      nb[threadIdx.x] = r < M ? a.map[(size_t)r * a.K + o] : -1;
    }
    // an offset no row of the tile has adds nothing (acc starts at +0 and a sum with +-0 terms is unchanged)
    if (!__syncthreads_or(threadIdx.x < kBM && nb[threadIdx.x] >= 0)) continue;
    for (int k0 = 0; k0 < a.cin; k0 += kCK) {
      // A: 64 rows x 32 channels, 8 per thread; row = e / 32 keeps a warp on one row's 32 contiguous channels
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const int e = threadIdx.x + t * 256, r = e >> 5, k = e & 31;
        const int src = nb[r];
        As[k][r] = src >= 0 ? a.in[(size_t)src * a.ldin + k0 + k] : 0.f;
      }
      for (int e = threadIdx.x; e < kCK * BN; e += 256) {
        const int k = e / BN, c = e % BN;
        Bs[k][c] = a.W[((size_t)o * a.cin + k0 + k) * a.cout + col0 + c];
      }
      __syncthreads();
#pragma unroll 8
      for (int k = 0; k < kCK; ++k) {
        const float4 av = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
        float bv[TN];
#pragma unroll
        for (int j = 0; j < TN; ++j) bv[j] = Bs[k][tx * TN + j];
        const float ar[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) acc[i][j] = __fmaf_rn(ar[i], bv[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = row0 + ty * 4 + i;
    if (r >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int c = col0 + tx * TN + j;
      float v = __fmaf_rn(acc[i][j], a.scale[c], a.shift[c]);
      if (a.res) v = __fadd_rn(v, a.res[(size_t)r * a.ldres + c]);
      if (a.relu) v = fmaxf(v, 0.f);
      a.out[(size_t)r * a.ldo + c] = v;
    }
  }
}

// conv1: Cin = 1 with input 1.0, out[q][c] = BN(sum over the occupied offsets, ascending, of W[o][c]); one warp per row
__global__ void __launch_bounds__(256) fconv1_kernel(const int32_t* __restrict__ map, int K3, const float* __restrict__ W,
                                                     const float* __restrict__ scale, const float* __restrict__ shift,
                                                     const int32_t* __restrict__ rows, long long n, float* __restrict__ out) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int c = threadIdx.x & 31;
  if (row >= n || row >= *rows) return;
  float acc = 0.f;
  for (int o = 0; o < K3; ++o)
    if (map[(size_t)row * K3 + o] >= 0) acc = __fadd_rn(acc, W[(size_t)o * 32 + c]);
  out[(size_t)row * 32 + c] = __fmaf_rn(acc, scale[c], shift[c]);
}

// conv1_tr (96 -> 64, no bias), ReLU, final (64 -> 32, bias), x / (||x|| + 1e-8); one warp per level-0 row, written to the
// packed output row out_off + row
__global__ void __launch_bounds__(256) fhead_kernel(const float* __restrict__ cat0, const float* __restrict__ w_tr,
                                                    const float* __restrict__ w_f, const float* __restrict__ b_f,
                                                    const int32_t* __restrict__ rows, long long n, float* __restrict__ desc,
                                                    const int32_t* __restrict__ rep0, const float* __restrict__ pts,
                                                    float* __restrict__ keypts) {
  __shared__ float wt[96 * 64];
  __shared__ float wf[64 * 32];
  for (int e = threadIdx.x; e < 96 * 64; e += 256) wt[e] = w_tr[e];
  for (int e = threadIdx.x; e < 64 * 32; e += 256) wf[e] = w_f[e];
  __syncthreads();
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= n || row >= *rows) return;
  const float* x = cat0 + (size_t)row * 96;
  const float x0 = x[lane], x1 = x[lane + 32], x2 = x[lane + 64];
  float h0 = 0.f, h1 = 0.f;               // hidden channels lane and lane + 32
  for (int k = 0; k < 96; ++k) {
    const float xk = __shfl_sync(0xffffffffu, k < 32 ? x0 : (k < 64 ? x1 : x2), k & 31);
    h0 = __fmaf_rn(xk, wt[k * 64 + lane], h0);
    h1 = __fmaf_rn(xk, wt[k * 64 + lane + 32], h1);
  }
  h0 = fmaxf(h0, 0.f); h1 = fmaxf(h1, 0.f);
  float f = 0.f;
  for (int k = 0; k < 64; ++k) {
    const float hk = __shfl_sync(0xffffffffu, k < 32 ? h0 : h1, k & 31);
    f = __fmaf_rn(hk, wf[k * 32 + lane], f);
  }
  f = __fadd_rn(f, b_f[lane]);
  const float den = __fadd_rn(__fsqrt_rn(warp_sum(__fmul_rn(f, f))), 1e-8f);
  desc[(size_t)row * 32 + lane] = __fdiv_rn(f, den);
  if (lane < 3) keypts[(size_t)row * 3 + lane] = pts[(size_t)rep0[row] * 3 + lane];
}

}  // namespace
}  // namespace pdsc

// ---- weights (the C ABI's pdsc_fcgf handle) --------------------------------------------------------------------------
struct pdsc_fcgf {
  int k1 = 7;
  std::map<std::string, std::vector<float>> params;
  bool committed = false;
  float* d_arena = nullptr;
  // per step: W, scale, shift offsets (floats) into the arena; then the head
  size_t w[pdsc::kNumSteps], scale[pdsc::kNumSteps], shift[pdsc::kNumSteps];
  size_t w_tr = 0, w_f = 0, b_f = 0;
};

namespace pdsc {

struct ParamSpec {
  std::string name;
  size_t numel;
};

static std::vector<ParamSpec> fcgf_param_specs(int k1) {
  std::vector<ParamSpec> v;
  for (const Step& s : kSteps) {
    const int K = step_k(s, k1);
    v.push_back({std::string(s.name) + ".kernel", (size_t)K * step_cin(s) * s.cout});
    for (const char* f : {".bn.weight", ".bn.bias", ".bn.running_mean", ".bn.running_var"})
      v.push_back({std::string(s.norm) + f, (size_t)s.cout});
  }
  v.push_back({"conv1_tr.kernel", 96 * 64});
  v.push_back({"final.kernel", 64 * 32});
  v.push_back({"final.bias", 32});
  return v;
}

pdsc_fcgf* fcgf_new(int k1) {
  pdsc_fcgf* h = new pdsc_fcgf();
  h->k1 = k1;
  return h;
}

void fcgf_free(pdsc_fcgf* h) {
  if (!h) return;
  if (h->d_arena) cudaFree(h->d_arena);
  delete h;
}

// 0, or 1 (unknown name) / 2 (wrong size) with *expected set
int fcgf_set_param(pdsc_fcgf* h, const char* name, const float* data, int64_t numel, size_t* expected) {
  for (const ParamSpec& p : fcgf_param_specs(h->k1)) {
    if (p.name != name) continue;
    *expected = p.numel;
    if ((size_t)numel != p.numel) return 2;
    h->params[p.name].assign(data, data + numel);
    h->committed = false;
    return 0;
  }
  return 1;
}

// folds BN in float64 and uploads; returns the first missing parameter's name in *missing, or a CUDA error
int fcgf_commit(pdsc_fcgf* h, std::string* missing) {
  for (const ParamSpec& p : fcgf_param_specs(h->k1))
    if (!h->params.count(p.name)) { *missing = p.name; return -1; }
  std::vector<float> arena;
  auto put = [&](const float* src, size_t n) {
    while (arena.size() % 4) arena.push_back(0.f);
    const size_t at = arena.size();
    arena.insert(arena.end(), src, src + n);
    return at;
  };
  for (int i = 0; i < kNumSteps; ++i) {
    const Step& s = kSteps[i];
    const std::vector<float>& W = h->params[std::string(s.name) + ".kernel"];
    h->w[i] = put(W.data(), W.size());
    const std::string nm = s.norm;
    const std::vector<float>& g = h->params[nm + ".bn.weight"];
    const std::vector<float>& b = h->params[nm + ".bn.bias"];
    const std::vector<float>& mu = h->params[nm + ".bn.running_mean"];
    const std::vector<float>& var = h->params[nm + ".bn.running_var"];
    std::vector<float> sc(s.cout), sh(s.cout);
    for (int c = 0; c < s.cout; ++c) {
      const double k = (double)g[c] / std::sqrt((double)var[c] + kBnEps);
      sc[c] = (float)k;
      sh[c] = (float)((double)b[c] - (double)mu[c] * k);
    }
    h->scale[i] = put(sc.data(), sc.size());
    h->shift[i] = put(sh.data(), sh.size());
  }
  h->w_tr = put(h->params["conv1_tr.kernel"].data(), 96 * 64);
  h->w_f = put(h->params["final.kernel"].data(), 64 * 32);
  h->b_f = put(h->params["final.bias"].data(), 32);
  if (h->d_arena) { cudaFree(h->d_arena); h->d_arena = nullptr; }
  cudaError_t e = cudaMalloc(&h->d_arena, arena.size() * 4);
  if (e == cudaSuccess) e = cudaMemcpy(h->d_arena, arena.data(), arena.size() * 4, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) return (int)e;
  h->committed = true;
  return 0;
}

bool fcgf_committed(const pdsc_fcgf* h) { return h->committed; }
int fcgf_kernel_size(const pdsc_fcgf* h) { return h->k1; }

size_t fcgf_scratch_bytes(int P, const int32_t* h_off, int k1) { return carve(nullptr, P, h_off, k1).bytes; }

int fcgf_scratch_layout(int P, const int32_t* h_off, int k1, int64_t* offsets, int capacity) {
  const Scratch s = carve(nullptr, P, h_off, k1);
  const int n = (int)s.reported.size();
  for (int i = 0; i < n && i < capacity; ++i) offsets[i] = (int64_t)s.reported[i];
  return n;
}

int launch_fcgf(const pdsc_fcgf* h, int P, const int32_t* h_off, const int32_t* d_off, const float* pts, double voxel,
                float* keypts, float* desc, int32_t* out_off, int32_t* status, void* scratch, cudaStream_t st) {
  const Scratch s = carve(scratch, P, h_off, h->k1);
  const long long n = h_off[P];
  const unsigned long long S = total_slots(P, h_off);
  const int blocks = (int)((n + kScanBlock - 1) / kScanBlock);
  const unsigned g256 = (unsigned)((n + 255) / 256);
  hash_plan_kernel<<<1, 1024, 0, st>>>(P, Offsets{d_off, 0}, s.slot0);
  fq_init_kernel<<<(unsigned)((std::max<unsigned long long>(S, P) + 255) / 256), 256, 0, st>>>(
      s.keys[0], s.keys[1], s.keys[2], s.keys[3], s.first[0], s.first[1], s.first[2], s.first[3], S, P, status);
  // the level's items' coordinates go to the (not yet used) conv1 table before their rows are numbered
  int32_t* tmp = s.map_c1;
  for (int l = 0; l < kLevels; ++l) {
    const int32_t* in_off = l == 0 ? d_off : s.lvl_off[l - 1];
    fq_insert_kernel<<<g256, 256, 0, st>>>(l, n, P, in_off, pts, voxel, l ? s.coords[l - 1] : nullptr, s.slot0, s.keys[l], s.first[l],
                                           s.islot, tmp, status);
    fq_flag_kernel<<<blocks, kScanBlock, 0, st>>>(n, s.islot, s.first[l], s.flags, s.bbase + 1);
    fq_scan_kernel<<<1, 1024, 0, st>>>(blocks, s.bbase);
    fq_write_kernel<<<g256, 256, 0, st>>>(l, n, s.flags, s.bbase, s.islot, tmp, s.row_of[l], s.coords[l], s.rep0);
    fq_offsets_kernel<<<(P + 1 + 255) / 256, 256, 0, st>>>(P, n, in_off, s.flags, s.bbase, s.lvl_off[l]);
  }
  auto map = [&](int level, int table, int K, int mult, int32_t* out) {
    const long long e = n * K * K * K;
    fmap_kernel<<<(unsigned)((e + 255) / 256), 256, 0, st>>>(n, P, s.lvl_off[level], s.coords[level], K, mult, s.slot0, s.keys[table],
                                                              s.row_of[table], out);
  };
  map(0, 0, h->k1, 1, s.map_c1);
  for (int l = 0; l < kLevels; ++l) map(l, l, 3, 1 << l, s.map_same[l]);
  for (int l = 1; l < kLevels; ++l) map(l, l - 1, 3, 1 << (l - 1), s.map_down[l]);
  for (int l = 0; l + 1 < kLevels; ++l) map(l, l + 1, 3, -(1 << l), s.map_up[l]);
  const float* A = h->d_arena;
  for (int i = 0; i < kNumSteps; ++i) {
    const Step& t = kSteps[i];
    const int32_t* rows = s.lvl_off[t.level] + P;
    if (t.kind == MAP_C1) {
      fconv1_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(s.map_c1, h->k1 * h->k1 * h->k1, A + h->w[i], A + h->scale[i],
                                                             A + h->shift[i], rows, n, s.feat[t.out]);
      continue;
    }
    ConvArgs a{};
    a.map = t.kind == MAP_SAME ? s.map_same[t.level] : (t.kind == MAP_DOWN ? s.map_down[t.level] : s.map_up[t.level]);
    a.K = 27;
    a.in = s.feat[t.in] + t.in_col; a.ldin = kFeatWidth[t.in]; a.cin = step_cin(t);
    a.W = A + h->w[i]; a.scale = A + h->scale[i]; a.shift = A + h->shift[i];
    a.res = t.res >= 0 ? s.feat[t.res] + t.res_col : nullptr; a.ldres = t.res >= 0 ? kFeatWidth[t.res] : 0;
    a.out = s.feat[t.out] + t.out_col; a.ldo = kFeatWidth[t.out]; a.cout = t.cout; a.relu = t.relu;
    a.rows = rows;
    const unsigned gx = (unsigned)((n + kBM - 1) / kBM);
    if (t.cout == 32) fconv_kernel<32><<<dim3(gx, 1), 256, 0, st>>>(a);
    else fconv_kernel<64><<<dim3(gx, t.cout / 64), 256, 0, st>>>(a);
  }
  fhead_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(s.feat[F_CAT0], A + h->w_tr, A + h->w_f, A + h->b_f, s.lvl_off[0] + P, n, desc,
                                                        s.rep0, pts, keypts);
  cudaMemcpyAsync(out_off, s.lvl_off[0], (size_t)(P + 1) * 4, cudaMemcpyDeviceToDevice, st);
  return (int)cudaGetLastError();
}

}  // namespace pdsc
