// f1 — the correspondence front end on the device (SURVEY.md §8 row f1).
//
// Reference: datasets/ThreeDMatch.py:283-291 (matching, optional mutual check) and :299-308 (network input); the same lines
// in datasets/KITTI.py:80-114 and demo_registration.py:101-108 (no mutual check there):
//     distance   = sqrt(2 - 2 * (src_desc @ tgt_desc.T) + 1e-6)            in the descriptors' dtype (fp32 FCGF, fp64 FPFH)
//     source_idx = argmin(distance, axis=1)                                 numpy: the FIRST minimum
//     mutual     : keep i iff argmin(distance, axis=0)[source_idx[i]] == i
//     corr_pos   = concat(src_keypts[corr[:,0]], tgt_keypts[corr[:,1]]) - mean over the kept correspondences
//
// A call matches P pairs (pdsc_match_packed; pdsc_match is the call with P = 1): pair p owns source rows
// [src_off[p], src_off[p+1]) and target rows [tgt_off[p], tgt_off[p+1]) of the packed descriptor and key-point arrays, and its
// rows are only ever compared with its own columns.  Descriptor dimension D <= 64.
//
// Kernels:
//   match_rows_kernel<T>   nearest column of every row over ONE chunk of its pair's columns (grid.y chunks, so that a
//                          5000 x 5000 problem fills the GPU).  Pair p owns the 128-row tiles [tile0(p), tile0(p+1)),
//                          tile0(p) = (off[p] + 127 p) / 128 — a function of the offset table alone, in which a tile finds its
//                          pair with find_set; a pair has ceil(N_p / 128) tiles or one more, which is idle.  Thread = row, its
//                          descriptor cached 16 channels at a time in registers; the chunk's descriptors are staged
//                          channel-major in shared memory, 64 columns (fp32) or 32 (fp64) per tile, and read as BROADCAST
//                          128-bit loads of four (two) adjacent columns — 64 FMAs per 16 loads, every dot product one
//                          ascending-channel FMA chain in T.  The square root is applied BEFORE the strict '<' comparison, as
//                          the reference does (it merges distances that differ by less than an ulp of the root), which is
//                          numpy's first-minimum rule inside the chunk.  Result: (distance, pair-local index) per (row, chunk).
//   match_reduce_kernel<T> thread = row: scans its chunks in ascending column order with the same strict '<' — the first
//                          minimum of the whole row.  No atomics anywhere.  Chunks are whole column tiles, and a column's
//                          distance does not depend on where it sits in a tile, so the index does not depend on the plan.
//   The mutual check needs argmin along the other axis: the SAME two kernels with the roles of the two descriptor sets
//   swapped.  a*b == b*a exactly and the channel order is the same, so both launches see bit-identical distances — the
//   consistency numpy gets from taking both argmins of one matrix.
//   compact_center_kernel  one CTA per pair: ordered compaction of the kept pairs (ascending source index), gather of the key
//                          points, column means in fp64 summed in a fixed order, centred corr_pos — written in the layout
//                          pdsc_forward_packed consumes.  With the mutual check a pair's first output row is the number of rows
//                          the pairs before it keep, which its CTA counts itself (no inter-CTA communication).
// The reference's BLAS fixes no accumulation order, so indices are only comparable where the best and the second-best distance
// are separated (tests); exact duplicates resolve to the first one, as in numpy.
#include <cfloat>

#include "abi.h"
#include "common.cuh"
#include "kernels.h"
#include "sets.cuh"

namespace pdsc {

constexpr int kMatchRows = 128;   // rows per CTA (one per thread)
constexpr int kMatchMaxD = 64;
constexpr int kMatchMaxChunks = 32;

template <typename T>
__device__ __forceinline__ T feature_distance(T dot) {
  // np.sqrt(2 - 2 * dot + 1e-6): python scalars adopt the array dtype, every operation rounded separately
  if (sizeof(T) == 4) return (T)__fsqrt_rn(__fadd_rn(__fsub_rn(2.0f, __fmul_rn(2.0f, (float)dot)), 1e-6f));
  return (T)__dsqrt_rn(__dadd_rn(__dsub_rn(2.0, __dmul_rn(2.0, (double)dot)), 1e-6));
}
template <typename T>
__device__ __forceinline__ T fma_t(T a, T b, T c) {
  if (sizeof(T) == 4) return (T)__fmaf_rn((float)a, (float)b, (float)c);
  return (T)__fma_rn((double)a, (double)b, (double)c);
}

// first row tile of pair p (see the header): every pair gets at least ceil(N_p / kMatchRows) tiles
__host__ __device__ __forceinline__ long long match_tile0(const Offsets& off, int p) {
  return ((long long)off.at(p) + (long long)(kMatchRows - 1) * p) / kMatchRows;
}
// columns per chunk of a pair with `cols` columns in a plan of `chunks` chunks: whole tiles of TT columns
__host__ __device__ __forceinline__ int match_per_chunk(int cols, int chunks, int TT) {
  const int per = (cols + chunks - 1) / chunks;
  return (per + TT - 1) / TT * TT;
}

template <typename T> struct MatchPartial { T dist; int idx; int pad; };

template <typename T>
__global__ void __launch_bounds__(kMatchRows) match_rows_kernel(const T* __restrict__ row_desc, const T* __restrict__ col_desc,
                                                                Offsets row_off, Offsets col_off, int P, int D, int chunks,
                                                                MatchPartial<T>* __restrict__ partial) {
  constexpr int TT = sizeof(T) == 4 ? 64 : 32;        // columns per shared-memory tile
  constexpr int VW = 16 / (int)sizeof(T);             // columns per 128-bit load
  extern __shared__ __align__(16) unsigned char match_smem[];
  T* s_row = reinterpret_cast<T*>(match_smem);        // [D][kMatchRows]  channel-major: conflict-free per-thread reads
  T* s_col = s_row + (size_t)D * kMatchRows;          // [D][TT]          channel-major: broadcast vector reads
  const int tid = threadIdx.x;
  const int p = find_set(P, (long long)blockIdx.x, [&](int q) { return match_tile0(row_off, q); });
  const int r0 = row_off.at(p), rows = row_off.at(p + 1) - r0;
  const int c0 = col_off.at(p), cols = col_off.at(p + 1) - c0;
  const int lr0 = (int)((long long)blockIdx.x - match_tile0(row_off, p)) * kMatchRows;
  if (lr0 >= rows) return;                            // the pair's idle tile
  row_desc += (size_t)r0 * D;
  col_desc += (size_t)c0 * D;
  const int i = lr0 + tid;
  const int per = match_per_chunk(cols, chunks, TT);
  const int c_begin = blockIdx.y * per, c_end = min(cols, c_begin + per);
  T best = (T)0;
  int best_j = -1;
  if (c_begin < c_end) {                              // else: a chunk past the pair's columns, reported empty
    for (int e = tid; e < D * kMatchRows; e += kMatchRows) {
      const int r = e / D, d = e % D;                 // coalesced over the row-major descriptor block
      const int gi = lr0 + r;
      s_row[(size_t)d * kMatchRows + r] = gi < rows ? row_desc[(size_t)gi * D + d] : (T)0;
    }
    for (int j0 = c_begin; j0 < c_end; j0 += TT) {
      __syncthreads();
      const int cnt = min(TT, c_end - j0);
      for (int e = tid; e < TT * D; e += kMatchRows) {
        const int t = e / D, d = e % D;
        s_col[(size_t)d * TT + t] = t < cnt ? col_desc[(size_t)(j0 + t) * D + d] : (T)0;
      }
      __syncthreads();
      T acc[TT];
#pragma unroll
      for (int t = 0; t < TT; ++t) acc[t] = (T)0;
      for (int d0 = 0; d0 < D; d0 += 16) {
        T sv[16];
#pragma unroll
        for (int q = 0; q < 16; ++q) sv[q] = (d0 + q < D) ? s_row[(size_t)(d0 + q) * kMatchRows + tid] : (T)0;
#pragma unroll
        for (int q = 0; q < 16; ++q) {
          if (d0 + q < D) {                          // warp-uniform
            const T* cv = s_col + (size_t)(d0 + q) * TT;
#pragma unroll
            for (int t = 0; t < TT; t += VW) {
              if (sizeof(T) == 4) {
                const float4 v = *reinterpret_cast<const float4*>(cv + t);
                acc[t] = fma_t<T>(sv[q], (T)v.x, acc[t]); acc[t + 1] = fma_t<T>(sv[q], (T)v.y, acc[t + 1]);
                acc[t + 2] = fma_t<T>(sv[q], (T)v.z, acc[t + 2]); acc[t + 3] = fma_t<T>(sv[q], (T)v.w, acc[t + 3]);
              } else {
                const double2 v = *reinterpret_cast<const double2*>(cv + t);
                acc[t] = fma_t<T>(sv[q], (T)v.x, acc[t]); acc[t + 1] = fma_t<T>(sv[q], (T)v.y, acc[t + 1]);
              }
            }
          }
        }
      }
#pragma unroll
      for (int t = 0; t < TT; ++t) {
        if (t < cnt) {
          const T dist = feature_distance<T>(acc[t]);
          if (best_j < 0 || dist < best) { best = dist; best_j = j0 + t; }    // strict '<': the first minimum wins
        }
      }
    }
  }
  if (i < rows) {
    MatchPartial<T>& o = partial[(size_t)(r0 + i) * gridDim.y + blockIdx.y];
    o.dist = best;
    o.idx = best_j;
  }
}

template <typename T>
__global__ void match_reduce_kernel(const MatchPartial<T>* __restrict__ partial, int rows, int chunks, int32_t* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows) return;
  T best = (T)0;
  int best_j = -1;
  for (int c = 0; c < chunks; ++c) {                  // ascending column ranges: strict '<' keeps the first minimum
    const MatchPartial<T> p = partial[(size_t)i * chunks + c];
    if (p.idx >= 0 && (best_j < 0 || p.dist < best)) { best = p.dist; best_j = p.idx; }
  }
  idx[i] = best_j;
}

// One CTA per pair.  keep[i] = !mutual || col_idx[row_idx[i]] == i ; ordered compaction ; gather ; centre.
constexpr int kCompactThreads = 1024;
constexpr int kCompactWarps = kCompactThreads / 32;

__device__ __forceinline__ bool match_kept(const int32_t* row_idx, const int32_t* col_idx, int s0, int t0, int i, int mutual) {
  const int j = row_idx[s0 + i];
  return j >= 0 && (!mutual || col_idx[t0 + j] == i);
}

__global__ void __launch_bounds__(kCompactThreads) compact_center_kernel(const int32_t* __restrict__ row_idx,
                                                                         const int32_t* __restrict__ col_idx,
                                                                         const float* __restrict__ src_keypts,
                                                                         const float* __restrict__ tgt_keypts, Offsets src_off,
                                                                         Offsets tgt_off, int mutual, int32_t* __restrict__ corr,
                                                                         int32_t* __restrict__ out_first,
                                                                         int32_t* __restrict__ out_ends,
                                                                         float* __restrict__ corr_pos, float* __restrict__ out_src,
                                                                         float* __restrict__ out_tgt) {
  __shared__ int warp_tot[kCompactWarps];
  __shared__ int base_s;
  __shared__ double warp_sums[6][kCompactWarps];
  __shared__ double sums[6];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int p = blockIdx.x;
  const int s0 = src_off.at(p), Ns = src_off.at(p + 1) - s0, t0 = tgt_off.at(p);
  // first output row of the pair: every source row is kept without the mutual check; with it, the kept rows of pairs < p
  int first = s0;
  if (mutual) {
    int cnt = 0;
    for (int q = 0; q < p; ++q) {
      const int q0 = src_off.at(q), nq = src_off.at(q + 1) - q0, u0 = tgt_off.at(q);
      for (int i = tid; i < nq; i += kCompactThreads) cnt += match_kept(row_idx, col_idx, q0, u0, i, 1);
    }
    cnt = warp_sum(cnt);
    if (lane == 0) warp_tot[warp] = cnt;
    __syncthreads();
    first = 0;
    for (int w = 0; w < kCompactWarps; ++w) first += warp_tot[w];
    __syncthreads();
  }
  if (tid == 0) base_s = first;
  __syncthreads();
  double acc[6] = {0, 0, 0, 0, 0, 0};
  for (int i0 = 0; i0 < Ns; i0 += kCompactThreads) {
    const int i = i0 + tid;
    const bool keep = i < Ns && match_kept(row_idx, col_idx, s0, t0, i, mutual);
    const int j = keep ? row_idx[s0 + i] : -1;
    const unsigned ballot = __ballot_sync(0xffffffffu, keep);
    const int in_warp = __popc(ballot & ((1u << lane) - 1u));
    if (lane == 0) warp_tot[warp] = __popc(ballot);
    __syncthreads();
    int before = base_s;
    for (int w = 0; w < warp; ++w) before += warp_tot[w];
    if (keep) {
      const int m = before + in_warp;
      corr[2 * (size_t)m] = i;
      corr[2 * (size_t)m + 1] = j;
      float v[6];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        v[c] = src_keypts[(size_t)(s0 + i) * 3 + c];
        v[3 + c] = tgt_keypts[(size_t)(t0 + j) * 3 + c];
        out_src[(size_t)m * 3 + c] = v[c];
        out_tgt[(size_t)m * 3 + c] = v[3 + c];
      }
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        corr_pos[(size_t)m * 6 + c] = v[c];
        acc[c] += (double)v[c];
      }
    }
    __syncthreads();
    if (tid == 0) {
      int tot = 0;
      for (int w = 0; w < kCompactWarps; ++w) tot += warp_tot[w];
      base_s += tot;
    }
    __syncthreads();
  }
  // column sums in a fixed order: each thread's rows in order, a butterfly over the warp, then the warps in order
#pragma unroll
  for (int c = 0; c < 6; ++c) {
    const double s = warp_sum(acc[c]);
    if (lane == 0) warp_sums[c][warp] = s;
  }
  __syncthreads();
  if (tid < 6) {
    double s = 0.0;
    for (int w = 0; w < kCompactWarps; ++w) s += warp_sums[tid][w];
    sums[tid] = s;
  }
  __syncthreads();
  const int M = base_s - first;
  if (tid == 0) {
    out_ends[p] = base_s;
    if (out_first && p == 0) out_first[0] = 0;
  }
  // corr_pos - corr_pos.mean(0)   (ThreeDMatch.py:305-308): mean rounded to fp32, one rounded subtraction per element
  float* cp = corr_pos + (size_t)first * 6;
  for (int e = tid; e < M * 6; e += kCompactThreads) {
    const float mean = (float)(sums[e % 6] / (double)M);
    cp[e] = __fsub_rn(cp[e], mean);
  }
}

// about four CTAs per SM over the call's row tiles
static int match_chunks(long long row_ctas) {
  long long chunks = (4 * device_sm_count() + row_ctas - 1) / row_ctas;
  return chunks < 1 ? 1 : (chunks > kMatchMaxChunks ? kMatchMaxChunks : (int)chunks);
}

template <typename T>
static void nearest_columns(const T* row_desc, const T* col_desc, int P, const int32_t* h_row_off, const int32_t* h_col_off,
                            Offsets row_off, Offsets col_off, int D, MatchPartial<T>* partial, int32_t* idx, cudaStream_t st) {
  constexpr int TT = sizeof(T) == 4 ? 64 : 32;
  const Offsets hr{h_row_off, 0}, hc{h_col_off, 0};
  const long long tiles = match_tile0(hr, P);
  const int chunks = match_chunks(tiles);
  int grid_y = 1;                                      // the most chunks any pair's columns fill
  for (int p = 0; p < P; ++p) {
    const int cols = hc.at(p + 1) - hc.at(p), per = match_per_chunk(cols, chunks, TT);
    grid_y = max(grid_y, (cols + per - 1) / per);
  }
  const int rows = hr.at(P);
  const int smem = (int)sizeof(T) * D * (kMatchRows + TT);
  ensure_dynamic_smem(reinterpret_cast<const void*>(match_rows_kernel<T>), smem);
  match_rows_kernel<T><<<dim3((unsigned)tiles, grid_y), kMatchRows, smem, st>>>(row_desc, col_desc, row_off, col_off, P, D, chunks,
                                                                               partial);
  match_reduce_kernel<T><<<(rows + 255) / 256, 256, 0, st>>>(partial, rows, grid_y, idx);
}

template <typename T>
static void launch_match_t(int P, const int32_t* h_src_off, const int32_t* h_tgt_off, Offsets src_off, Offsets tgt_off,
                           const T* src_desc, const T* tgt_desc, const float* src_keypts, const float* tgt_keypts, int D,
                           int mutual, void* scratch, int32_t* corr, int32_t* out_first, int32_t* out_ends, float* corr_pos,
                           float* out_src, float* out_tgt, cudaStream_t st) {
  // scratch: row_idx [sum Ns] int32 | col_idx [sum Nt] int32 | partial [max(sum Ns, sum Nt)][kMatchMaxChunks] (16-byte aligned)
  const int Ns = h_src_off[P], Nt = h_tgt_off[P];
  int32_t* row_idx = static_cast<int32_t*>(scratch);
  int32_t* col_idx = row_idx + Ns;
  auto* partial = reinterpret_cast<MatchPartial<T>*>((reinterpret_cast<uintptr_t>(col_idx + Nt) + 15) & ~uintptr_t(15));
  nearest_columns<T>(src_desc, tgt_desc, P, h_src_off, h_tgt_off, src_off, tgt_off, D, partial, row_idx, st);
  if (mutual)                                          // argmin along the other axis
    nearest_columns<T>(tgt_desc, src_desc, P, h_tgt_off, h_src_off, tgt_off, src_off, D, partial, col_idx, st);
  compact_center_kernel<<<P, kCompactThreads, 0, st>>>(row_idx, col_idx, src_keypts, tgt_keypts, src_off, tgt_off, mutual, corr,
                                                       out_first, out_ends, corr_pos, out_src, out_tgt);
}

static size_t match_scratch_bytes(int Ns, int Nt) {
  const size_t rows = (size_t)(Ns > Nt ? Ns : Nt);
  return (size_t)(Ns + Nt) * sizeof(int32_t) + rows * kMatchMaxChunks * sizeof(MatchPartial<double>) + 32;
}

// pdsc_match and pdsc_match_packed: P pairs packed back to back (null device tables: one pair).  Pair p's kept rows end at
// out_ends[p], written by the call, as is out_first[0] = 0 unless out_first is null.
static int match_impl(pdsc_engine* e, int32_t P, int32_t D, const int32_t* h_src_offsets, const int32_t* h_tgt_offsets,
                      const int32_t* d_src_offsets, const int32_t* d_tgt_offsets, const void* d_src_desc, const void* d_tgt_desc,
                      int32_t desc_is_fp64, const float* d_src_keypts, const float* d_tgt_keypts, int32_t use_mutual,
                      int32_t* d_corr, int32_t* d_out_first, int32_t* d_out_ends, float* d_corr_pos, float* d_out_src,
                      float* d_out_tgt, void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  if (D < 1 || D > kMatchMaxD) return fail(PDSC_ERR_UNSUPPORTED, "descriptor dimension %d outside [1, %d]", D, kMatchMaxD);
  const int in_dim = engine_config(e).in_dim;
  if (in_dim != 6) return fail(PDSC_ERR_UNSUPPORTED, "pdsc_match builds the in_dim = 6 input (engine has in_dim = %d)", in_dim);
  if (!d_src_desc || !d_tgt_desc || !d_src_keypts || !d_tgt_keypts || !d_corr || !d_out_ends || !d_corr_pos || !d_out_src || !d_out_tgt)
    return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_match: null tensor pointer");
  if (int rc = check_scratch("pdsc_match", "scratch", d_scratch, scratch_bytes, match_scratch_bytes(h_src_offsets[P], h_tgt_offsets[P]),
                             8))
    return rc;
  DeviceGuard g(engine_config(e).device);
  // without a device table (one pair) the kernels read the offsets {0, N} as 0 * N, 1 * N
  const Offsets so{d_src_offsets, d_src_offsets ? 0 : h_src_offsets[1]}, to{d_tgt_offsets, d_tgt_offsets ? 0 : h_tgt_offsets[1]};
  auto run = [&](auto* src_desc, auto* tgt_desc) {
    launch_match_t(P, h_src_offsets, h_tgt_offsets, so, to, src_desc, tgt_desc, d_src_keypts, d_tgt_keypts, D, use_mutual, d_scratch,
                   d_corr, d_out_first, d_out_ends, d_corr_pos, d_out_src, d_out_tgt, static_cast<cudaStream_t>(cuda_stream));
  };
  if (desc_is_fp64) run(static_cast<const double*>(d_src_desc), static_cast<const double*>(d_tgt_desc));
  else run(static_cast<const float*>(d_src_desc), static_cast<const float*>(d_tgt_desc));
  PDSC_CUDA(cudaGetLastError());
  return PDSC_OK;
}

}  // namespace pdsc

// ---- C ABI ------------------------------------------------------------------------------------------------------
using namespace pdsc;

extern "C" {

size_t pdsc_match_scratch_bytes(int32_t Ns, int32_t Nt) { return (Ns > 0 && Nt > 0) ? match_scratch_bytes(Ns, Nt) : 0; }

size_t pdsc_match_packed_scratch_bytes(int32_t P, const int32_t* h_src_offsets, const int32_t* h_tgt_offsets) {
  const char* who = "pdsc_match_packed_scratch_bytes";
  if (check_offsets(who, "source ", P, h_src_offsets, 1) || check_offsets(who, "target ", P, h_tgt_offsets, 1)) return 0;
  return match_scratch_bytes(h_src_offsets[P], h_tgt_offsets[P]);
}

int pdsc_match(pdsc_engine* e, int32_t Ns, int32_t Nt, int32_t D, const void* d_src_desc, const void* d_tgt_desc,
               int32_t desc_is_fp64, const float* d_src_keypts, const float* d_tgt_keypts, int32_t use_mutual,
               int32_t* d_corr, int32_t* d_count, float* d_corr_pos, float* d_out_src, float* d_out_tgt, void* d_scratch,
               size_t scratch_bytes, void* cuda_stream) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (Ns <= 0 || Nt <= 0) return fail(PDSC_ERR_SHAPE, "need Ns >= 1 and Nt >= 1 (got %d, %d)", Ns, Nt);
  // the packed call with one pair: its offsets need no device table, and its end row is the count
  const int32_t src_off[2] = {0, Ns}, tgt_off[2] = {0, Nt};
  return match_impl(e, 1, D, src_off, tgt_off, nullptr, nullptr, d_src_desc, d_tgt_desc, desc_is_fp64, d_src_keypts, d_tgt_keypts,
                    use_mutual, d_corr, nullptr, d_count, d_corr_pos, d_out_src, d_out_tgt, d_scratch, scratch_bytes, cuda_stream);
}

int pdsc_match_packed(pdsc_engine* e, int32_t P, int32_t D, const int32_t* h_src_offsets, const int32_t* h_tgt_offsets,
                      const int32_t* d_src_offsets, const int32_t* d_tgt_offsets, const void* d_src_desc, const void* d_tgt_desc,
                      int32_t desc_is_fp64, const float* d_src_keypts, const float* d_tgt_keypts, int32_t use_mutual,
                      int32_t* d_corr, int32_t* d_out_offsets, float* d_corr_pos, float* d_out_src, float* d_out_tgt,
                      void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (int rc = check_offsets("pdsc_match_packed", "source ", P, h_src_offsets, 1)) return rc;
  if (int rc = check_offsets("pdsc_match_packed", "target ", P, h_tgt_offsets, 1)) return rc;
  if (!d_src_offsets || !d_tgt_offsets || !d_out_offsets) return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_match_packed: null offsets");
  return match_impl(e, P, D, h_src_offsets, h_tgt_offsets, d_src_offsets, d_tgt_offsets, d_src_desc, d_tgt_desc, desc_is_fp64,
                    d_src_keypts, d_tgt_keypts, use_mutual, d_corr, d_out_offsets, d_out_offsets + 1, d_corr_pos, d_out_src,
                    d_out_tgt, d_scratch, scratch_bytes, cuda_stream);
}

}  // extern "C"
