// Stage ii on the fp32 FFMA pipe: the exact-arithmetic encoder path (precision PDSC_FP32_SIMT).
//
// Reference: models/PointDSC.py:9-77 (NonLocalBlock / NonLocalNet).  Every 1x1 Conv1d is a row-major
// linear map on point-major features feat[B*N][C]; eval-mode BatchNorm is folded into the preceding
// conv on the host.  The attention kernel is a flash-style tiling of
//     P = softmax_j( SC_ij * (q_i . k_j) / sqrt(C) ),  msg = P V           (PointDSC.py:39-42)
// so no N x N logits or probabilities reach HBM (the reference materialises both, per layer).
// SC is a multiplicative weight, not a mask: SC_ij = 0 gives logit 0, which still receives softmax
// mass (SURVEY.md §7 trap 2) — nothing is skipped.
//
// This path exists as the arithmetic ground truth on the device (it is what the tensor-core kernels are
// compared with) and as the engine's fallback-free "exact" mode; the throughput path is encoder_tc.cu.
#include "common.cuh"
#include "kernels.h"

namespace pdsc {

// -------------------------------------------------------------------------------------------------
// generic K-contiguous SGEMM:  out[r][o] = epi(sum_c A[r][c] W[o][c])
// -------------------------------------------------------------------------------------------------
constexpr int LBM = 64, LBN = 64, LBK = 16;

__global__ void __launch_bounds__(256) linear_simt_kernel(LinearArgs a) {
  __shared__ __align__(16) float As[LBK][LBM + 4];
  __shared__ __align__(16) float Ws[LBK][LBN + 4];
  const int bz = blockIdx.z;
  const float* A = a.A + (size_t)bz * a.strideA;
  const float* W = a.W + (size_t)bz * a.strideW;
  float* out = a.out + (size_t)bz * a.strideO;
  const int m0 = blockIdx.y * LBM, n0 = blockIdx.x * LBN;
  if (a.epi == 1) {      // seed-row distances of set bz; the grid is sized by the largest set
    const SetDesc d = a.sets[bz];
    A = a.A + (size_t)d.seed0 * a.lda;
    W = a.W + (size_t)d.row0 * a.ldw;
    out = a.out + d.dist0;
    a.M = d.S; a.Nout = d.N; a.ldo = d.N;
    if (m0 >= a.M || n0 >= a.Nout) return;
  }
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int lr = tid / 4, lc = (tid % 4) * 4;  // loader: row within tile, k offset
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < a.K; k0 += LBK) {
    float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vw = va;
    if (m0 + lr < a.M) va = *reinterpret_cast<const float4*>(A + (size_t)(m0 + lr) * a.lda + k0 + lc);
    if (n0 + lr < a.Nout) vw = *reinterpret_cast<const float4*>(W + (size_t)(n0 + lr) * a.ldw + k0 + lc);
    As[lc + 0][lr] = va.x; As[lc + 1][lr] = va.y; As[lc + 2][lr] = va.z; As[lc + 3][lr] = va.w;
    Ws[lc + 0][lr] = vw.x; Ws[lc + 1][lr] = vw.y; Ws[lc + 2][lr] = vw.z; Ws[lc + 3][lr] = vw.w;
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < LBK; ++kk) {
      const float4 av = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      const float4 wv = *reinterpret_cast<const float4*>(&Ws[kk][tx * 4]);
      const float ar[4] = {av.x, av.y, av.z, av.w};
      const float wr[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], wr[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = m0 + ty * 4 + i;
    if (r >= a.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int o = n0 + tx * 4 + j;
      if (o >= a.Nout) continue;
      float v = acc[i][j];
      if (a.epi == 1) {
        v = 2.0f - 2.0f * v;
      } else if (a.epi == 2) {
        v = (r == o) ? 0.0f : fminf(fmaxf(__fsub_rn(1.0f, __fdiv_rn(__fsub_rn(1.0f, v), a.epi_param)), 0.0f), 1.0f);
      } else {
        if (a.bias) v += a.bias[o];
        if (a.relu) v = fmaxf(v, 0.f);
        if (a.res) v += a.res[(size_t)r * a.ldres + o];
      }
      out[(size_t)r * a.ldo + o] = v;
    }
  }
}

void launch_linear_simt(const LinearArgs& a, cudaStream_t st) {
  dim3 grid((a.Nout + LBN - 1) / LBN, (a.M + LBM - 1) / LBM, a.batch);
  linear_simt_kernel<<<grid, 256, 0, st>>>(a);
}

// layer0: Conv1d(in_dim -> 128), in_dim = 6 (PointDSC.py:54, :73).  HBM-write bound (512 B per row out, 24 B in): one
// warp per row per pass, lane = four output channels (weights and bias live in registers across the grid-stride loop),
// one 16-byte store per lane so every warp store is a full 512-byte row.  FMA order: ascending input channel, bias last.
constexpr int kL0MaxIn = 8;
__global__ void __launch_bounds__(256) layer0_kernel(const float* __restrict__ x, const float* __restrict__ W,
                                                     const float* __restrict__ bias, float* __restrict__ out,
                                                     long long rows, int in_dim) {
  const int lane = threadIdx.x & 31;
  const long long warp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * 8;
  if (in_dim <= kL0MaxIn) {
    float w[4][kL0MaxIn];
#pragma unroll
    for (int o = 0; o < 4; ++o)
#pragma unroll
      for (int c = 0; c < kL0MaxIn; ++c) w[o][c] = (c < in_dim) ? W[(lane * 4 + o) * in_dim + c] : 0.f;
    const float4 bv = *reinterpret_cast<const float4*>(bias + lane * 4);
    for (long long r = warp; r < rows; r += nwarps) {
      float xin[kL0MaxIn];
#pragma unroll
      for (int c = 0; c < kL0MaxIn; ++c) xin[c] = (c < in_dim) ? __ldg(x + r * in_dim + c) : 0.f;
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int c = 0; c < kL0MaxIn; ++c) {
        if (c < in_dim) {
#pragma unroll
          for (int o = 0; o < 4; ++o) acc[o] = fmaf(xin[c], w[o][c], acc[o]);
        }
      }
      *reinterpret_cast<float4*>(out + r * kC + lane * 4) = make_float4(acc[0] + bv.x, acc[1] + bv.y, acc[2] + bv.z, acc[3] + bv.w);
    }
  } else {
    for (long long r = warp; r < rows; r += nwarps) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int c = 0; c < in_dim; ++c) {
        const float xv = __ldg(x + r * in_dim + c);
#pragma unroll
        for (int o = 0; o < 4; ++o) acc[o] = fmaf(xv, W[(lane * 4 + o) * in_dim + c], acc[o]);
      }
#pragma unroll
      for (int o = 0; o < 4; ++o) out[r * kC + lane * 4 + o] = acc[o] + bias[lane * 4 + o];
    }
  }
}
void launch_layer0(const float* corr_pos, const float* W, const float* bias, float* out, long long rows, int in_dim,
                   cudaStream_t st) {
  long long blocks = (rows + 7) / 8;
  const long long max_blocks = 8LL * device_sm_count();
  if (blocks > max_blocks) blocks = max_blocks;
  if (blocks < 1) blocks = 1;
  layer0_kernel<<<(unsigned)blocks, 256, 0, st>>>(corr_pos, W, bias, out, rows, in_dim);
}

// -------------------------------------------------------------------------------------------------
// SC-weighted attention, fp32, online softmax.  CTA = 64 queries of one set; 64-key tiles.
// -------------------------------------------------------------------------------------------------
constexpr int AQ = 64, AK = 64;
constexpr int kAttnSmem = (kC * AQ + kC * AK + AK * kC + AQ * AK) * (int)sizeof(float);  // 112 KB

__global__ void __launch_bounds__(256) attention_simt_kernel(const float* __restrict__ Q, const float* __restrict__ K,
                                                             const float* __restrict__ V, const float* __restrict__ SC,
                                                             float* __restrict__ MSG, const SetDesc* __restrict__ sets) {
  extern __shared__ __align__(16) float smem[];
  float* Qs = smem;                 // [C][AQ]   Qs[c][q]
  float* Ks = Qs + kC * AQ;         // [C][AK]   Ks[c][key]
  float* Vs = Ks + kC * AK;         // [AK][C]   Vs[key][c]
  float* Ps = Vs + AK * kC;         // [AQ][AK]  Ps[q][key]
  const int b = blockIdx.y, q0 = blockIdx.x * AQ;
  const SetDesc d = sets[b];
  const int N = d.N, NS = round_up(N, 64);
  if (q0 >= N) return;                 // the grid is sized by the largest set
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const size_t base = (size_t)d.row0;
  SC += d.sc0;
  const float inv_sqrt_c = 1.0f / sqrtf((float)kC);

  // Q tile, transposed into smem: lane <-> query (conflict-free smem stores; L1 absorbs the strided reads)
  for (int t = tid; t < AQ * (kC / 4); t += 256) {
    const int q = t % AQ, c4 = t / AQ;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + q < N) v = *reinterpret_cast<const float4*>(Q + (base + q0 + q) * kC + c4 * 4);
    Qs[(c4 * 4 + 0) * AQ + q] = v.x; Qs[(c4 * 4 + 1) * AQ + q] = v.y;
    Qs[(c4 * 4 + 2) * AQ + q] = v.z; Qs[(c4 * 4 + 3) * AQ + q] = v.w;
  }

  float o_acc[4][8];
  float m_run[4], l_run[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m_run[i] = -INFINITY; l_run[i] = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) o_acc[i][j] = 0.f;
  }

  for (int j0 = 0; j0 < N; j0 += AK) {
    __syncthreads();  // previous tile's Ks/Vs/Ps fully consumed (also orders the Q tile stores)
    for (int t = tid; t < AK * (kC / 4); t += 256) {
      const int key = t % AK, c4 = t / AK;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (j0 + key < N) v = *reinterpret_cast<const float4*>(K + (base + j0 + key) * kC + c4 * 4);
      Ks[(c4 * 4 + 0) * AK + key] = v.x; Ks[(c4 * 4 + 1) * AK + key] = v.y;
      Ks[(c4 * 4 + 2) * AK + key] = v.z; Ks[(c4 * 4 + 3) * AK + key] = v.w;
    }
    for (int t = tid; t < AK * (kC / 4); t += 256) {
      const int key = t / (kC / 4), c4 = t % (kC / 4);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (j0 + key < N) v = *reinterpret_cast<const float4*>(V + (base + j0 + key) * kC + c4 * 4);
      *reinterpret_cast<float4*>(Vs + key * kC + c4 * 4) = v;
    }
    __syncthreads();

    // S = Q K^T  (4 queries x 4 keys per thread)
    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 8
    for (int c = 0; c < kC; ++c) {
      const float4 qv = *reinterpret_cast<const float4*>(Qs + c * AQ + ty * 4);
      const float4 kv = *reinterpret_cast<const float4*>(Ks + c * AK + tx * 4);
      const float qr[4] = {qv.x, qv.y, qv.z, qv.w};
      const float kr[4] = {kv.x, kv.y, kv.z, kv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) s[i][j] = fmaf(qr[i], kr[j], s[i][j]);
    }

    // logits = SC * (S / sqrt(C)); online softmax over the keys of this tile
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int qi = q0 + ty * 4 + i;
      float4 scv = make_float4(0.f, 0.f, 0.f, 0.f);
      if (qi < N) scv = *reinterpret_cast<const float4*>(SC + (size_t)qi * NS + j0 + tx * 4);
      const float scr[4] = {scv.x, scv.y, scv.z, scv.w};
      float tmax = -INFINITY;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const bool valid = (j0 + tx * 4 + j) < N;
        s[i][j] = valid ? scr[j] * (s[i][j] * inv_sqrt_c) : -INFINITY;
        tmax = fmaxf(tmax, s[i][j]);
      }
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, o));
      const float m_new = fmaxf(m_run[i], tmax);
      const float corr = expf(m_run[i] - m_new);  // exp(-inf) = 0 on the first tile
      float psum = 0.f;
      float p[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        p[j] = expf(s[i][j] - m_new);  // exp(-inf) = 0 for masked keys
        psum += p[j];
      }
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) psum += __shfl_xor_sync(0xffffffffu, psum, o);
      l_run[i] = l_run[i] * corr + psum;
      m_run[i] = m_new;
#pragma unroll
      for (int j = 0; j < 8; ++j) o_acc[i][j] *= corr;
      *reinterpret_cast<float4*>(Ps + (ty * 4 + i) * AK + tx * 4) = make_float4(p[0], p[1], p[2], p[3]);
    }
    __syncthreads();

    // O += P V   (4 queries x 8 channels per thread: channels tx*4..+3 and 64+tx*4..+3)
#pragma unroll 4
    for (int key = 0; key < AK; ++key) {
      const float4 v0 = *reinterpret_cast<const float4*>(Vs + key * kC + tx * 4);
      const float4 v1 = *reinterpret_cast<const float4*>(Vs + key * kC + 64 + tx * 4);
      const float vr[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float pv = Ps[(ty * 4 + i) * AK + key];
#pragma unroll
        for (int j = 0; j < 8; ++j) o_acc[i][j] = fmaf(pv, vr[j], o_acc[i][j]);
      }
    }
  }

#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int qi = q0 + ty * 4 + i;
    if (qi >= N) continue;
    const float inv_l = 1.0f / l_run[i];
    float* dst = MSG + (base + qi) * kC;
    *reinterpret_cast<float4*>(dst + tx * 4) =
        make_float4(o_acc[i][0] * inv_l, o_acc[i][1] * inv_l, o_acc[i][2] * inv_l, o_acc[i][3] * inv_l);
    *reinterpret_cast<float4*>(dst + 64 + tx * 4) =
        make_float4(o_acc[i][4] * inv_l, o_acc[i][5] * inv_l, o_acc[i][6] * inv_l, o_acc[i][7] * inv_l);
  }
}

void launch_attention_simt(const float* q, const float* k, const float* v, const float* sc, float* msg, int B, int N,
                           cudaStream_t st, const SetDesc* sets) {
  ensure_dynamic_smem(reinterpret_cast<const void*>(attention_simt_kernel), kAttnSmem);
  dim3 grid((N + AQ - 1) / AQ, B);
  attention_simt_kernel<<<grid, 256, kAttnSmem, st>>>(q, k, v, sc, msg, sets);
}

}  // namespace pdsc
