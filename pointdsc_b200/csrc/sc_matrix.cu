// Stage i — the N x N second-order spatial-consistency matrix (SURVEY.md §8 a1).
//
// Reference: models/PointDSC.py:150-153
//   src_dist = ||x_i - x_j||,  SC_ij = max(0, 1 - (src_dist_ij - ||y_i - y_j||)^2 / sigma_d^2)
// The reference materialises two [N,N,3] broadcast temporaries (>= 40 N^2 bytes of traffic); this
// kernel reads 24 B per point and writes each SC element exactly once (4 N NS bytes), which is the
// stage's algorithmic HBM traffic: it is write-bandwidth bound.
//
// Layout: sc[b][i][j], row stride NS = N rounded up to 64 floats so that every 64-key tile of a row
// is a 256-byte aligned segment for the attention kernels; the pad columns j >= N are written as 0.
// `src_dist` is NOT materialised: its only consumer, the seed NMS (a6), recomputes it from the points.
#include "common.cuh"
#include "kernels.h"
#include "sets.cuh"

namespace pdsc {

constexpr int kScRows = 32;

__global__ void __launch_bounds__(256) sc_matrix_kernel(const float* __restrict__ src, const float* __restrict__ tgt,
                                                        float* __restrict__ sc, const SetDesc* __restrict__ sets, float s2) {
  __shared__ float rs[kScRows][3], rt[kScRows][3];
  const int b = blockIdx.y;
  const SetDesc d = sets[b];
  const int N = d.N, NS = round_up(N, 64);
  const int i0 = blockIdx.x * kScRows;
  if (i0 >= N) return;                     // the grid is sized by the largest set
  const float* ps = src + (size_t)d.row0 * 3;
  const float* pt = tgt + (size_t)d.row0 * 3;
  for (int t = threadIdx.x; t < kScRows * 3; t += blockDim.x) {
    const int r = t / 3, c = t % 3;
    const int i = min(i0 + r, N - 1);
    rs[r][c] = ps[(size_t)i * 3 + c];
    rt[r][c] = pt[(size_t)i * 3 + c];
  }
  __syncthreads();
  const int rows = min(kScRows, N - i0);
  float* out = sc + d.sc0 + (size_t)i0 * NS;
  for (int j = threadIdx.x; j < NS; j += blockDim.x) {
    if (j < N) {
      const float sx = ps[(size_t)j * 3], sy = ps[(size_t)j * 3 + 1], sz = ps[(size_t)j * 3 + 2];
      const float tx = pt[(size_t)j * 3], ty = pt[(size_t)j * 3 + 1], tz = pt[(size_t)j * 3 + 2];
#pragma unroll 4
      for (int r = 0; r < rows; ++r) {
        const float ds = length3(rs[r][0] - sx, rs[r][1] - sy, rs[r][2] - sz);
        const float dt = length3(rt[r][0] - tx, rt[r][1] - ty, rt[r][2] - tz);
        out[(size_t)r * NS + j] = consistency(__fsub_rn(ds, dt), s2);
      }
    } else {
      for (int r = 0; r < rows; ++r) out[(size_t)r * NS + j] = 0.0f;
    }
  }
}

void launch_sc_matrix(const float* src, const float* tgt, float* sc, int B, int N, float sigma_d, cudaStream_t st,
                      const SetDesc* sets) {
  const float s2 = sigma_d * sigma_d;  // fp32 product, as `self.sigma_spat ** 2`
  dim3 grid((N + kScRows - 1) / kScRows, B);
  sc_matrix_kernel<<<grid, 256, 0, st>>>(src, tgt, sc, sets, s2);
}

// ---- tiled layout for the tensor-core attention (tc_attention.cuh) ---------------------------------------
// sc_t[b][kt][qt][16 key groups][128 queries][4 keys]: every (64-key x 128-query) tile the attention CTA (b, qt) consumes
// at key step kt is one contiguous 32 KB block, and inside it the 4 keys of a group are adjacent, so a softmax thread
// (query row r) reads its 64 SC values as 16 fully coalesced 16-byte loads at compile-time offsets (g * 2048 B) from one
// per-tile base pointer — no per-element address arithmetic, a quarter of the load instructions of a [key][query] tile.
// SC is exactly symmetric in fp32 ((x_i - x_j)^2 == (x_j - x_i)^2), so element (key, q) is computed as SC[q][key].
// Pad rows / columns (key >= N or q >= N) are written as 0.
// One CTA = one 128 x 128 super-block (A <= Bq) of one set: it evaluates V[i][j] = SC[128 A + i][128 Bq + j] ONCE and
// writes it in both orientations — keys in A / queries in Bq directly (coalesced over j), and keys in Bq / queries
// in A through a shared-memory transpose (coalesced over i) — so the 2 IEEE square roots + 1 IEEE division per element
// that make this kernel issue-bound are paid for only ~(QT+1)/(2 QT) of the matrix.
constexpr int kScTStride = 129;   // smem transpose tile [32 i][128 j], odd stride: conflict-free both ways

__global__ void __launch_bounds__(256) sc_matrix_tiled_kernel(const float* __restrict__ src, const float* __restrict__ tgt,
                                                              float* __restrict__ sc, const SetDesc* __restrict__ sets, float s2, float rc_s2) {
  // the A range's points as six arrays: an 8-byte broadcast load is the same coordinate of TWO consecutive rows, so the distance
  // chains of two matrix elements run as pairs (each lane rounded exactly like the scalar sequence)
  __shared__ __align__(8) float isx[128], isy[128], isz[128], itx[128], ity[128], itz[128];
  __shared__ float tr[32 * kScTStride];
  const int b = blockIdx.y;
  const SetDesc d = sets[b];
  const int N = d.N, KT = (N + 63) / 64, QT = (N + 127) / 128;
  if ((int)blockIdx.x >= QT * (QT + 1) / 2) return;   // the grid is sized by the largest set
  // blockIdx.x enumerates the pairs A <= Bq
  int A = 0, rem = blockIdx.x;
  while (rem >= QT - A) { rem -= QT - A; ++A; }
  const int Bq = A + rem;
  const float* ps = src + (size_t)d.row0 * 3;
  const float* pt = tgt + (size_t)d.row0 * 3;
  if (threadIdx.x < 128) {
    const int i = min(A * 128 + (int)threadIdx.x, N - 1);
    isx[threadIdx.x] = ps[(size_t)i * 3]; isy[threadIdx.x] = ps[(size_t)i * 3 + 1]; isz[threadIdx.x] = ps[(size_t)i * 3 + 2];
    itx[threadIdx.x] = pt[(size_t)i * 3]; ity[threadIdx.x] = pt[(size_t)i * 3 + 1]; itz[threadIdx.x] = pt[(size_t)i * 3 + 2];
  }
  __syncthreads();
  const int jl = threadIdx.x & 127, half = threadIdx.x >> 7;
  const int j = Bq * 128 + jl;
  const int jc = min(j, N - 1);
  const float sx = ps[(size_t)jc * 3], sy = ps[(size_t)jc * 3 + 1], sz = ps[(size_t)jc * 3 + 2];
  const float tx = pt[(size_t)jc * 3], ty = pt[(size_t)jc * 3 + 1], tz = pt[(size_t)jc * 3 + 2];
  float* const set_sc = sc + d.sc0;
  const int ti = threadIdx.x & 31, tg = threadIdx.x >> 5;   // transposed write-out: lane = i within the chunk, 16 j per warp
  for (int ic = 0; ic < 4; ++ic) {             // 32-row chunks of the A range
    // orientation 1: key = 128 A + i, query = j   ->  tile (kt = 2 A + (ic >> 1), qt = Bq), element [(i & 63)][jl]
    const int kt1 = 2 * A + (ic >> 1);
    const int il0 = ic * 32 + half * 16;
    float* out1 = set_sc + (((size_t)min(kt1, KT - 1) * QT + Bq) << 13) + (((il0 & 63) >> 2) * 128 + jl) * 4;
    float* trw = tr + (half * 16) * kScTStride + jl;
    const bool col_ok = j < N;
    const int i_lim = N - A * 128 - il0;       // rows ii < i_lim are real correspondences
    float vals[16];
#pragma unroll
    for (int ii = 0; ii < 16; ii += 2) {
      const int r = il0 + ii;
      const float2 px = *reinterpret_cast<const float2*>(isx + r), py = *reinterpret_cast<const float2*>(isy + r),
                   pz = *reinterpret_cast<const float2*>(isz + r);
      const float2 qx = *reinterpret_cast<const float2*>(itx + r), qy = *reinterpret_cast<const float2*>(ity + r),
                   qz = *reinterpret_cast<const float2*>(itz + r);
      // length3(): sqrt(fma(dz, dz, fma(dy, dy, dx dx))), the two rows side by side
      const float2 ax = fsub2_pair_scalar(px, sx), ay = fsub2_pair_scalar(py, sy), az = fsub2_pair_scalar(pz, sz);
      const float2 bx = fsub2_pair_scalar(qx, tx), by = fsub2_pair_scalar(qy, ty), bz = fsub2_pair_scalar(qz, tz);
      const float2 a2 = ffma2_pair(az, az, ffma2_pair(ay, ay, fmul2(ax, ax)));
      const float2 b2 = ffma2_pair(bz, bz, ffma2_pair(by, by, fmul2(bx, bx)));
      const float2 ds = make_float2(__fsqrt_rn(a2.x), __fsqrt_rn(a2.y));
      const float2 dt = make_float2(__fsqrt_rn(b2.x), __fsqrt_rn(b2.y));
      const float2 v = consistency_rc2(fsub2(ds, dt), s2, rc_s2);
      vals[ii] = (col_ok && ii < i_lim) ? v.x : 0.0f;
      vals[ii + 1] = (col_ok && ii + 1 < i_lim) ? v.y : 0.0f;
    }
    if (kt1 < KT) {
      // keys (il0 & 63) + ii, ii < 16: four key groups, each one float4 per query
#pragma unroll
      for (int gq = 0; gq < 4; ++gq)
        *reinterpret_cast<float4*>(out1 + gq * 512) = make_float4(vals[4 * gq], vals[4 * gq + 1], vals[4 * gq + 2], vals[4 * gq + 3]);
    }
    if (A != Bq) {
#pragma unroll
      for (int ii = 0; ii < 16; ++ii) trw[ii * kScTStride] = vals[ii];
      __syncthreads();
      // orientation 2: key = 128 Bq + j, query = 128 A + i  ->  tile (kt = 2 Bq + (j >> 6), qt = A), element (j & 63, i)
      const int kt2 = 2 * Bq + (tg >> 2);      // the warp's 16 j share one key tile
      if (kt2 < KT) {
        float* out2 = set_sc + (((size_t)kt2 * QT + A) << 13) + (((tg & 3) * 4) * 128 + ic * 32 + ti) * 4;
        const float* trr = tr + ti * kScTStride + tg * 16;
#pragma unroll
        for (int gq = 0; gq < 4; ++gq)
          *reinterpret_cast<float4*>(out2 + gq * 512) = make_float4(trr[4 * gq], trr[4 * gq + 1], trr[4 * gq + 2], trr[4 * gq + 3]);
      }
      __syncthreads();
    }
  }
}

void launch_sc_matrix_tiled(const float* src, const float* tgt, float* sc, int B, int N, float sigma_d, cudaStream_t st,
                            const SetDesc* sets) {
  const float s2 = sigma_d * sigma_d;
  const int QT = (N + 127) / 128;
  sc_matrix_tiled_kernel<<<dim3(QT * (QT + 1) / 2, B), 256, 0, st>>>(src, tgt, sc, sets, s2, 1.0f / s2);
}

// tiled -> dense [B][N][N] (stage tap only)
__global__ void sc_untile_kernel(const float* __restrict__ sc_t, float* __restrict__ out, int N, int KT, int QT) {
  const int b = blockIdx.z, i = blockIdx.y;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  const float* tile = sc_t + ((((size_t)b * KT + (i >> 6)) * QT + (j >> 7)) << 13);
  out[((size_t)b * N + i) * N + j] = tile[((((i & 63) >> 2) * 128 + (j & 127)) << 2) + (i & 3)];
}
void launch_sc_untile(const float* sc_t, float* out, int B, int N, cudaStream_t st) {
  const int KT = (N + 63) / 64, QT = (N + 127) / 128;
  sc_untile_kernel<<<dim3((N + 255) / 256, N, B), 256, 0, st>>>(sc_t, out, N, KT, QT);
}

__global__ void fill_u32_kernel(uint32_t* p, uint32_t v, long long n) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
__global__ void fill_u64_kernel(unsigned long long* p, unsigned long long v, long long n) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
void launch_fill_u32(uint32_t* p, uint32_t v, long long n, cudaStream_t st) {
  if (n > 0) fill_u32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(p, v, n);
}
void launch_fill_u64(unsigned long long* p, unsigned long long v, long long n, cudaStream_t st) {
  if (n > 0) fill_u64_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(p, v, n);
}

}  // namespace pdsc
