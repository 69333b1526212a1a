// tc_chain: fused row-tile GEMM chains of the encoder's 1x1 convolutions on wgmma (included by encoder_tc.cu).
//
//   PCQ   : feat  --W1,relu--> feat1 (fp32 -> HBM) --Wq--> Q image (HBM)
//   Q     : feat1 --Wq--> Q image (HBM)
//   KV    : feat1 --Wk--> K image (HBM) ;  feat1 --Wv--> V image (HBM, same row-major format as K)
//   MSG   : msg --Wm0,relu--> --Wm1,relu--> --Wm2--> + feat1 --> feat (fp32 -> HBM)
//   MSGPC : MSG, then feat --W1 of the next layer,relu--> the next layer's feat1 (fp32 -> HBM, in place over feat1)
// (reference models/PointDSC.py:56-61 PointCN, :21-23/:36-38 projections, :12-20/:43-44 fc_message + residual)
// A layer is PCQ (layer 0) or Q, then KV, attention, and MSGPC (MSG for the last layer, whose feat the head reads): feat
// between two layers never goes through HBM.  MSGPC and Q compute exactly what MSG and PCQ did, instruction for instruction.
//
// Persistent CTAs (one per SM), weights resident in shared memory, 128-row tiles, two warpgroups of 64 rows each.  A tile's
// fp32 input (64 KB of contiguous memory in every mode) arrives in shared memory by one bulk async copy; each thread reads its
// own accumulator-layout fragment of it and splits it into the hi | lo register A operand of the first GEMM.  As soon as every
// thread holds its fragments, the copy of the CTA's next tile is issued, so that tile's input streams in while this one
// computes and stores.  Chained steps never go back through shared memory: the epilogue of one GEMM (bias, ReLU, hi/lo split)
// turns its accumulator fragment into the register A operand of the next.  The Q / K / V images are written after a transpose
// within each quad of lanes, one whole 16-byte swizzle chunk per lane and store (store_row).  The rows of a ragged last tile
// beyond `rows` hold stale data; they feed only output rows that are never stored (a 1x1 convolution maps each row on its own).
// feat1 (fp32, PCQ / MSGPC -> Q, KV and MSG / MSGPC) lives in HBM in a BLOCKED layout keyed by the 128-row chain tile:
//     [tile][32-column chunk cc][128 rows][128 B], 16-byte piece q of row r at piece q ^ (r & 7)
// so that the fragment reads of a staged feat1 tile are at most 2-way bank conflicted (blocked_f32_offset).
#pragma once
#include <climits>

#include "tc_common.cuh"

namespace pdsc {

constexpr int kChainThreads = 256;
constexpr int kChIn = 0;                         // staged input tile (64 KB): row-major feat / msg, or blocked feat1;
                                                 // MSGPC: also its blocked feat1 residual tile, once the msg fragments are read
constexpr int kChW = 65536;                      // weight images (128 KB for PCQ / KV, 80 KB for MSG / MSGPC, 64 KB for Q)
constexpr int kChRes = kChW + 81920;             // 64 KB behind the fc_message weights.  MSG: staged blocked feat1 residual
                                                 // tile;  MSGPC: the next layer's W1 images
constexpr int kChBias = kChRes + 65536;          // 384 floats: this mode's biases
constexpr int kChBars = kChBias + 1536;          // mbarriers: weights, input, residual
constexpr int kChainSmem = kChBars + 64;         // 214,592 B

// modes that write the Q image (the others that write an operand image write K / V)
template <int MODE>
constexpr bool kWritesQ = MODE == kPCQ || MODE == kQ;

// A chain tile may span several sets (rows are not padded per set).  Its rows find their sets in a window of the table: lane
// l holds the first row and the first operand image tile (PCQ, Q: 128-query tile of the Q image, KV: 64-key tile of the K / V
// image) of set lo + l, lo the set of the tile's first row (ChainArgs::tile_set).
struct SetWindow {
  int lo, row0, t0;
};
template <int MODE>
__device__ __forceinline__ SetWindow load_window(const ChainArgs& a, int lo) {
  const int lane = threadIdx.x & 31, w = min(lo + lane, a.nsets - 1);
  return {lo, lo + lane < a.nsets ? __ldg(&a.sets[w].row0) : INT_MAX, kWritesQ<MODE> ? __ldg(&a.sets[w].qt0) : __ldg(&a.sets[w].kt0)};
}

// operand image tile of row g of the window's chain tile and the row's place within that tile.  All lanes of the warp take part.
template <int MODE>
__device__ __forceinline__ void locate_row(const ChainArgs& a, const SetWindow& win, long long g, int& tile, int& r) {
  int k = 0;                                      // the last window set that starts at or below g
#pragma unroll
  for (int s = 16; s > 0; s >>= 1)
    if (__shfl_sync(0xffffffffu, win.row0, k + s) <= g) k += s;
  int row0 = __shfl_sync(0xffffffffu, win.row0, k), t0 = __shfl_sync(0xffffffffu, win.t0, k);
  if (k == 31) {                                  // more than 31 sets start in the tile (N < 5): step on past the window
    int b = win.lo + 31;
    while (b + 1 < a.nsets && __ldg(&a.sets[b + 1].row0) <= g) ++b;
    row0 = __ldg(&a.sets[b].row0);
    t0 = kWritesQ<MODE> ? __ldg(&a.sets[b].qt0) : __ldg(&a.sets[b].kt0);
  }
  const int nn = (int)(g - row0);
  tile = t0 + (kWritesQ<MODE> ? (nn >> 7) : (nn >> 6));
  r = kWritesQ<MODE> ? (nn & 127) : (nn & 63);
}

// byte offset of the 16-byte piece `piece` (0..31) of global row `g` in the blocked fp32 layout described in the header
__host__ __device__ __forceinline__ size_t blocked_f32_offset(long long g, uint32_t piece) {
  return (size_t)(g >> 7) * 65536 + (size_t)(piece >> 3) * 16384 + (size_t)(g & 127) * 128 + (size_t)(((piece & 7u) ^ ((uint32_t)g & 7u)) << 4);
}

// 4 x 4 transpose of 32-bit words across the 4 lanes q of a quad (the lanes that share an accumulator row): on entry v[k] is
// word q of chunk k, on return word k of chunk q.  Every lane of the warp takes part.
__device__ __forceinline__ void quad_transpose(uint32_t (&v)[4], int q) {
#pragma unroll
  for (int s = 1; s <= 2; s <<= 1)
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (k & s) continue;
      const bool up = (q & s) != 0;
      const uint32_t r = __shfl_xor_sync(0xffffffffu, up ? v[k] : v[k + s], s);
      if (up) v[k] = r;
      else v[k + s] = r;
    }
}

// one row of a [rows][128] 16-bit operand image whose 64-column panels are panel_bytes apart, from the quad's fragments:
// w[j] = columns 8 j + 2 q, + 1 (j = 0..15).  Each lane stores whole 16-byte chunks (8 columns), so every sector is written
// in full by one instruction.  Only lanes with `store` write, but all must call.
__device__ __forceinline__ void store_row(uint8_t* img, uint32_t panel_bytes, uint32_t row, const uint32_t (&w)[16], int q, bool store) {
#pragma unroll
  for (int m = 0; m < 4; ++m) {
    uint32_t v[4] = {w[4 * m], w[4 * m + 1], w[4 * m + 2], w[4 * m + 3]};
    quad_transpose(v, q);
    const uint32_t j = 4u * m + q;
    if (store) *reinterpret_cast<uint4*>(img + (j >> 3) * panel_bytes + sw128_offset(row, 8u * (j & 7u))) = make_uint4(v[0], v[1], v[2], v[3]);
  }
}

template <int MODE, int FMT>
__global__ void __launch_bounds__(kChainThreads, 1) tc_chain_kernel(ChainArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint8_t* stage = smem + kChIn;
  const uint8_t* resbuf = smem + kChRes;
  float* bias = reinterpret_cast<float*>(smem + kChBias);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kChBars);
  const uint32_t s0 = smem_u32(smem);
  const uint32_t bar_w = smem_u32(bars), bar_in = smem_u32(bars + 1), bar_res = smem_u32(bars + 2);
  const int tid = threadIdx.x;
  const int wg = tid >> 7, wt = tid & 127;
  const uint32_t w_base = s0 + kChW;
  constexpr bool kFcMsg = MODE == kMSG || MODE == kMSGPC;   // the fc_message modes: row-major msg in, no operand image out
  constexpr bool kBlockedIn = MODE == kKV || MODE == kQ;    // the modes whose input is blocked feat1
  // this mode's biases, packed: PCQ b1|bq, Q bq, KV bk|bv, MSG bm0|bm1|bm2, MSGPC bm0|bm1|bm2|b1 (b1 of the next layer)
  constexpr int kBiasSrc = (MODE == kPCQ) ? kB1 : (MODE == kQ) ? kBq : (MODE == kKV) ? kBk : kBm0;
  const long long rows = a.rows;
  const long long num_tiles = (rows + 127) / 128;

  // a tile's input is the 64 KB at tile * 65536; feat and msg hold exactly `rows` rows, blocked feat1 is padded to whole tiles
  auto issue_input = [&](long long t) {
    const long long left = rows - t * 128;
    const uint32_t bytes = (kBlockedIn || left >= 128) ? 65536u : (uint32_t)left * 512u;
    mbar_expect_tx(bar_in, bytes);
    bulk_g2s(s0 + kChIn, reinterpret_cast<const uint8_t*>(a.in) + (size_t)t * 65536, bytes, bar_in);
  };
  // byte offset of (row r, column c) in a staged input tile
  auto in_offset = [](int r, int c) -> uint32_t {
    return kBlockedIn ? (uint32_t)blocked_f32_offset(r, (uint32_t)c >> 2) + (c & 3) * 4 : (uint32_t)(r * kC + c) * 4u;
  };

  // The chain kernels are launched with programmatic stream serialisation: the next grid may be scheduled at once and its
  // CTAs take the SMs this grid's CTAs leave, and this grid's CTAs may start while the previous kernel is still running.  Up
  // to griddep_wait a CTA touches only what no kernel of the call writes (the weight arena); everything else comes after.
  griddep_launch_dependents();
  if (tid == 0) {
    if (s0 & 1023u) __trap();   // the swizzled weight images need 1024-byte aligned shared memory
    mbar_init(bar_w, 1);
    mbar_init(bar_in, 1);
    mbar_init(bar_res, 1);
    fence_barrier_init();
  }
  bias[tid] = a.bias[kBiasSrc + tid];
  if (MODE == kMSGPC && tid < 128) bias[256 + tid] = a.bias1[kB1 + tid];
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(bar_w, (uint32_t)a.wbytes + (MODE == kMSGPC ? 65536u : 0u));
    for (int off = 0; off < a.wbytes; off += 32768)
      bulk_g2s(w_base + off, a.wimg + off, (uint32_t)min(32768, a.wbytes - off), bar_w);
    if (MODE == kMSGPC)   // the arena keeps W1 apart from the fc_message weights: a second copy, behind them
      for (int off = 0; off < 65536; off += 32768) bulk_g2s(s0 + kChRes + off, a.wimg1 + off, 32768u, bar_w);
  }
  griddep_wait();   // every thread: the previous kernels' results are complete and visible from here on
  if (tid == 0 && blockIdx.x < num_tiles) issue_input(blockIdx.x);
  mbar_wait(bar_w, 0);   // also keeps a CTA without tiles alive until its weight copy has landed
  const int fr = 64 * wg + frag_row(wt), fc = frag_col(wt);   // fragment rows fr, fr + 8 of the tile; columns 8 j + fc, + 1
  const int quad = fc >> 1;                                   // this lane's place among the 4 lanes that share its rows

  // PCQ, Q, KV: the set window of the CTA's next tile is loaded one tile ahead, from its first set loaded two tiles ahead, so
  // that no lookup waits for memory
  SetWindow win_next{};
  int lo_after = 0;
  if (!kFcMsg && blockIdx.x < num_tiles) {
    win_next = load_window<MODE>(a, __ldg(a.tile_set + blockIdx.x));
    if (blockIdx.x + gridDim.x < num_tiles) lo_after = __ldg(a.tile_set + blockIdx.x + gridDim.x);
  }
  uint32_t phase = 0;
  for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, phase ^= 1u) {
    const long long row0 = tile * 128;
    // the two rows of this thread: global index, operand image tile and row within it
    const long long g[2] = {row0 + fr, row0 + fr + 8};
    int tl[2], tr[2];
    if (!kFcMsg) {
      const SetWindow win = win_next;
      if (tile + gridDim.x < num_tiles) {
        win_next = load_window<MODE>(a, lo_after);
        if (tile + 2 * gridDim.x < num_tiles) lo_after = __ldg(a.tile_set + tile + 2 * gridDim.x);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) locate_row<MODE>(a, win, g[h] < rows ? g[h] : row0, tl[h], tr[h]);
    }
    // ---- this thread's fragment of the staged input tile -> hi / lo register A operand (K = 128) ----
    uint32_t ahi[8][4], alo[8][4];
    mbar_wait(bar_in, phase);
    {
      float x[64];
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float2 v = *reinterpret_cast<const float2*>(stage + in_offset(fr + 8 * h, 8 * j + fc));
          x[4 * j + 2 * h] = v.x;
          x[4 * j + 2 * h + 1] = v.y;
        }
      frag_split<FMT, 8>(x, ahi, alo);
    }
    __syncthreads();   // every thread holds its fragments and is past the previous tile's residual reads: refill both buffers
    if (tid == 0) {
      // MSGPC has no room for a residual buffer behind the next layer's W1: its residual tile goes into the input stage, and
      // the next tile's input follows once the residual has been read
      if (MODE != kMSGPC && tile + gridDim.x < num_tiles) issue_input(tile + gridDim.x);
      if (kFcMsg) {
        mbar_expect_tx(bar_res, 65536u);
        bulk_g2s(s0 + (MODE == kMSG ? kChRes : kChIn), reinterpret_cast<const uint8_t*>(a.res) + (size_t)tile * 65536, 65536u, bar_res);
      }
    }

    if (kWritesQ<MODE>) {
      if (MODE == kPCQ) {
        // ---- PointCN: feat1 = relu(A W1^T + b1) -> HBM (fp32, blocked) and registers (A operand of the Q GEMM) ----
        float x[64];
        wgmma_fence();
        gemm_rs<FMT, 8, 128, 0>(x, ahi, alo, w_base, w_base + 32768, 16384, a.split, 0);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(x);
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int c = 8 * j + fc, e = 4 * j + 2 * h;
            x[e] = fmaxf(x[e] + bias[c], 0.f);
            x[e + 1] = fmaxf(x[e + 1] + bias[c + 1], 0.f);
            if (g[h] < rows)
              *reinterpret_cast<float2*>(reinterpret_cast<uint8_t*>(a.out_f32) + blocked_f32_offset(g[h], (uint32_t)c >> 2) + (c & 3) * 4) =
                  make_float2(x[e], x[e + 1]);
          }
        frag_split<FMT, 8>(x, ahi, alo);
      }
      // PCQ: Wq behind W1, bq behind b1;  Q: Wq and bq alone
      const uint32_t wq = w_base + (MODE == kPCQ ? 65536u : 0u);
      const float* bq = bias + (MODE == kPCQ ? 128 : 0);
      float q[64];
      wgmma_fence();
      gemm_rs<FMT, 8, 128, 0>(q, ahi, alo, wq, wq + 32768, 16384, a.split, 0);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(q);
      // ---- Q image (pre-scaled weights and bias) ----
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        uint8_t* img = a.qimg + (size_t)tl[h] * 65536;
        const uint32_t r = (uint32_t)tr[h];
        uint32_t hi[16], lo[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int c = 8 * j + fc, e = 4 * j + 2 * h;
          split_pair<FMT>(q[e] + bq[c], q[e + 1] + bq[c + 1], hi[j], lo[j]);
        }
        store_row(img, 16384u, r, hi, quad, g[h] < rows);
        if (a.split) store_row(img + 32768, 16384u, r, lo, quad, g[h] < rows);
      }
    } else if (MODE == kKV) {
      // ---- K image, then V image (V behind K in the key tile's 64 KB) ----
#pragma unroll 1
      for (int step = 0; step < 2; ++step) {
        float x[64];
        const uint32_t wb = w_base + (uint32_t)step * 65536u;
        wgmma_fence();
        gemm_rs<FMT, 8, 128, 0>(x, ahi, alo, wb, wb + 32768, 16384, a.split, 0);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(x);
        const float* bvec = bias + 128 * step;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          uint8_t* img = a.kvimg + (size_t)tl[h] * 65536 + 32768 * step;
          const uint32_t r = (uint32_t)tr[h];
          uint32_t hi[16], lo[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int c = 8 * j + fc, e = 4 * j + 2 * h;
            split_pair<FMT>(x[e] + bvec[c], x[e + 1] + bvec[c + 1], hi[j], lo[j]);
          }
          store_row(img, 8192u, r, hi, quad, g[h] < rows);
          if (a.split) store_row(img + 16384, 8192u, r, lo, quad, g[h] < rows);
        }
      }
    } else {
      // ---- fc_message: Wm0 64 x 128 (hi 16K | lo 16K, panel 8K), Wm1 64 x 64 (hi 8K | lo 8K), Wm2 128 x 64 (hi 16K | lo 16K) ----
      float h0[32];
      wgmma_fence();
      gemm_rs<FMT, 8, 64, 0>(h0, ahi, alo, w_base, w_base + 16384, 8192, a.split, 0);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(h0);
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) h0[4 * j + e] = fmaxf(h0[4 * j + e] + bias[8 * j + fc + (e & 1)], 0.f);
      uint32_t bhi[4][4], blo[4][4];
      frag_split<FMT, 4>(h0, bhi, blo);
      float h1[32];
      wgmma_fence();
      gemm_rs<FMT, 4, 64, 0>(h1, bhi, blo, w_base + 32768, w_base + 32768 + 8192, 8192, a.split, 0);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(h1);
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) h1[4 * j + e] = fmaxf(h1[4 * j + e] + bias[64 + 8 * j + fc + (e & 1)], 0.f);
      frag_split<FMT, 4>(h1, bhi, blo);
      float o[64];
      wgmma_fence();
      gemm_rs<FMT, 4, 128, 0>(o, bhi, blo, w_base + 49152, w_base + 49152 + 16384, 16384, a.split, 0);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(o);
      if (MODE == kMSG) {
        // feat = feat1 + (D2 + bm2), feat1 from the staged residual tile
        mbar_wait(bar_res, phase);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (g[h] >= rows) continue;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int c = 8 * j + fc, e = 4 * j + 2 * h;
            const float2 rv = *reinterpret_cast<const float2*>(resbuf + blocked_f32_offset(fr + 8 * h, (uint32_t)c >> 2) + (c & 3) * 4);
            *reinterpret_cast<float2*>(a.out_f32 + g[h] * kC + c) =
                make_float2(rv.x + (o[e] + bias[128 + c]), rv.y + (o[e + 1] + bias[128 + c + 1]));
          }
        }
      } else {
        // feat = feat1 + (D2 + bm2), as MSG computes it, feat1 from the residual tile staged in the input buffer.  feat is then
        // in the fragment layout the PCQ mode reads its staged input in (row fr + 8 h, column 8 j + fc at x[4 j + 2 h]), so
        // its hi / lo split is the A operand PCQ would build.
        mbar_wait(bar_res, phase);
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int c = 8 * j + fc, e = 4 * j + 2 * h;
            const float2 rv = *reinterpret_cast<const float2*>(stage + blocked_f32_offset(fr + 8 * h, (uint32_t)c >> 2) + (c & 3) * 4);
            o[e] = rv.x + (o[e] + bias[128 + c]);
            o[e + 1] = rv.y + (o[e + 1] + bias[128 + c + 1]);
            if (a.feat_out && g[h] < rows) *reinterpret_cast<float2*>(a.feat_out + g[h] * kC + c) = make_float2(o[e], o[e + 1]);
          }
        __syncthreads();   // every thread is past its residual reads: the stage takes the next tile's input
        if (tid == 0 && tile + gridDim.x < num_tiles) issue_input(tile + gridDim.x);
        frag_split<FMT, 8>(o, ahi, alo);
        // ---- the next layer's PointCN: feat1 = relu(feat W1^T + b1) -> HBM (fp32, blocked), in place over this layer's feat1.
        // The tile's residual copy has landed before any of these stores (mbar_wait above), no other CTA reads or writes the
        // tile's rows, and no later kernel reads this layer's feat1.
        float x[64];
        wgmma_fence();
        gemm_rs<FMT, 8, 128, 0>(x, ahi, alo, s0 + kChRes, s0 + kChRes + 32768, 16384, a.split, 0);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(x);
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int c = 8 * j + fc, e = 4 * j + 2 * h;
            if (g[h] < rows)
              *reinterpret_cast<float2*>(reinterpret_cast<uint8_t*>(a.out_f32) + blocked_f32_offset(g[h], (uint32_t)c >> 2) + (c & 3) * 4) =
                  make_float2(fmaxf(x[e] + bias[256 + c], 0.f), fmaxf(x[e + 1] + bias[256 + c + 1], 0.f));
          }
      }
    }
  }
}

}  // namespace pdsc
