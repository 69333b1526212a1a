// Internal launch API of the pointdsc_b200 kernels.  Host-callable; every function only enqueues
// work on `st`.  Shapes: B sets, N correspondences per set, NS = SC row stride (N rounded up to 64),
// C = 128 channels, S seeds per set, k neighbours per seed.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "sets.cuh"

namespace pdsc {

// The launchers below take the call's descriptor table `sets` (sets.cuh, never null); their kernels find every set's size and
// offsets there.  B, N, S and k (the largest N, S and k of the call's sets) size the grids and shared memory only.

// ---- stage i ------------------------------------------------------------------------------------
void launch_sc_matrix(const float* src, const float* tgt, float* sc, int B, int N, float sigma_d, cudaStream_t st,
                      const SetDesc* sets);   // row stride NS = N rounded up to 64

// tensor-core path: sc_t[b][kt][qt][16][128][4] tiles (see sc_matrix.cu); size B * ceil(N/64) * ceil(N/128) * 8192 floats
void launch_sc_matrix_tiled(const float* src, const float* tgt, float* sc, int B, int N, float sigma_d, cudaStream_t st,
                            const SetDesc* sets);
void launch_sc_untile(const float* sc_t, float* out, int B, int N, cudaStream_t st);

// ---- stage ii, fp32 SIMT path -------------------------------------------------------------------
// out[b][r][o] = epi( sum_c A[b][r][c] * W[b][o][c] )   A,W K-contiguous; K % 16 == 0.
//   epi 0: (+bias[o]) (relu) (+res[r][o])     epi 1: 2 - 2*acc  (feature-space distance, common.py:58-61)
//   epi 2: clamp(1 - (1 - acc) / epi_param, 0, 1) with a zero diagonal  (feature similarity M, PointDSC.py:160-165)
struct LinearArgs {
  const float* A; long long strideA; int lda;
  const float* W; long long strideW; int ldw;
  const float* bias; const float* res; int ldres;
  float* out; long long strideO; int ldo;
  int M, K, Nout, relu, epi, batch;
  float epi_param;
  // epi 1: batch z is set z of `sets`, A = its seed rows, W = its normalised rows, out = its distance block [S][N]
  const SetDesc* sets;
};
void launch_linear_simt(const LinearArgs& a, cudaStream_t st);
void launch_layer0(const float* corr_pos, const float* W, const float* bias, float* out, long long rows, int in_dim,
                   cudaStream_t st);
void launch_attention_simt(const float* q, const float* k, const float* v, const float* sc, float* msg, int B, int N,
                           cudaStream_t st, const SetDesc* sets);

// ---- a4 + a5: normalise + classification head ---------------------------------------------------
struct HeadWeights {
  const float* w0t;  // [128][32]  classification.0.weight transposed
  const float* b0;   // [32]
  const float* w2t;  // [32][32]   classification.2.weight transposed
  const float* b2;   // [32]
  const float* w4;   // [32]
  const float* b4;   // [1]
};
void launch_head(const float* feat, const HeadWeights& w, float* normed, float* conf, long long rows, int want_conf,
                 cudaStream_t st);

// ---- a6: seeds -----------------------------------------------------------------------------------
void launch_pick_seeds(const float* src, const float* conf, int32_t* seeds, float* key_scratch, int B, int N, int S,
                       float radius, cudaStream_t st, const SetDesc* sets);
void launch_top_seeds(const float* conf, int32_t* seeds, int B, int N, int S, cudaStream_t st,   // a6' (non-testing rule)
                      const SetDesc* sets);
int pick_seeds_max_n();

// ---- a7: seed-row kNN ----------------------------------------------------------------------------
void launch_gather_rows(const float* normed, const int32_t* seeds, float* out, int B, int N, int S, cudaStream_t st,
                        const SetDesc* sets);
// tensor-core seed-row distances (knn_tc.cu): dist[b][s][j] = 2 - 2 <normed[b][seeds[b][s]], normed[b][j]>, fp16 hi/lo split
void launch_knn_dist_tc(const float* normed, const int32_t* seeds, float* dist, int B, int N, int S, cudaStream_t st,
                        const SetDesc* sets);
// total_seeds: sum of the sets' S
void launch_knn_select(const float* dist, int32_t* knn_idx, int B, int N, int S, int k, cudaStream_t st,
                       const SetDesc* sets, int total_seeds);

// ---- a8 + a9: compatibility + power iteration -----------------------------------------------------
void launch_nsm_power(const float* normed, const float* src, const float* tgt, const int32_t* knn_idx, float* iterates,
                      uint32_t* conv_mask, float* compat_out, int B, int N, int S, int k, int iters, float sigma,
                      float sigma_d, int mask_stride, int tensor_gram, cudaStream_t st,    // tensor_gram: fp16 hi/lo mma.sync Gram (k <= 80)
                      const SetDesc* sets, int k_min);   // k_min: the smallest k of the call's sets with seeds

// ---- a10 + a11: weighted Kabsch per seed, hypothesis scoring, selection -----------------------------
void launch_seed_hypotheses(const float* src, const float* tgt, const int32_t* knn_idx, const float* iterates,
                            const uint32_t* conv_mask, const float* seed_trans_in, float* seed_trans,
                            int32_t* inlier_counts, unsigned long long* best_key, float* eig_out, int32_t* power_iters,
                            int B, int N, int S, int k, int iters, float inlier_threshold, int mask_stride,
                            cudaStream_t st, const SetDesc* sets);

// ---- a11 (labels) + a12: refinement ----------------------------------------------------------------
void launch_select_refine(const float* src, const float* tgt, const float* seed_trans,
                          const unsigned long long* best_key, float* final_trans, float* final_labels,
                          float* init_trans_out, int32_t* best_out, int32_t* refine_solves, int B, int N, int S,
                          float inlier_threshold, float refine_threshold, int max_refine, cudaStream_t st,
                          const SetDesc* sets);

// ---- per-device launch configuration (device_state.cu) ----------------------------------------------------
// opt `kernel` in to `bytes` of dynamic shared memory on the CURRENT device (no-op if already granted there)
cudaError_t ensure_dynamic_smem(const void* kernel, int bytes);
int device_sm_count();   // SM count of the current device

// ---- misc ---------------------------------------------------------------------------------------
void launch_fill_u32(uint32_t* p, uint32_t v, long long n, cudaStream_t st);
void launch_fill_u64(unsigned long long* p, unsigned long long v, long long n, cudaStream_t st);

}  // namespace pdsc
