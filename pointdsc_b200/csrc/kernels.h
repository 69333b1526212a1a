// Internal launch API of the pointdsc_b200 kernels.  Host-callable; every function only enqueues
// work on `st`.  Shapes: B sets, N correspondences per set, NS = SC row stride (N rounded up to 64),
// C = 128 channels, S seeds per set, k neighbours per seed.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "sets.cuh"

struct pdsc_fcgf;

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

// ---- f3: per-pair evaluation statistics (eval_stats.cu), 10 floats per set -----------------------------------
void launch_eval_stats(const float* pred_trans, const float* gt_trans, const float* src, const float* tgt,
                       const float* pred_labels, const float* gt_labels, float* stats, int B, const int32_t* d_offsets, int N,
                       float re_thre, float te_thre, cudaStream_t st);   // set b: rows [offsets[b], offsets[b+1]), or b * N without a table

// ---- f1: correspondence front end (frontend.cu): nearest neighbour in descriptor space, mutual check, centred input ----
// P pairs packed back to back (offsets [P + 1], host and device; null device tables: one pair).  Pair p's kept rows end at
// out_ends[p], written by the call, as is out_first[0] = 0 unless out_first is null.
size_t match_scratch_bytes(int Ns, int Nt);      // Ns, Nt: the call's total source / target rows
int match_max_dim();
void launch_match(int P, const int32_t* h_src_off, const int32_t* h_tgt_off, const int32_t* d_src_off, const int32_t* d_tgt_off,
                  const void* src_desc, const void* tgt_desc, int desc_is_fp64, const float* src_keypts, const float* tgt_keypts,
                  int D, int mutual, void* scratch, int32_t* corr, int32_t* out_first, int32_t* out_ends, float* corr_pos,
                  float* out_src, float* out_tgt, cudaStream_t st);

// ---- f4: N x N power iteration (eig_power.cu) -----------------------------------------------------------------
size_t eig_scratch_bytes(int B, int N);
int launch_leading_eigenvector(const float* M, float* v, int* iters_run, int B, int N, int iters, int early_exit, void* scratch,
                               cudaStream_t st);   // returns cudaError_t

// ---- f2: descriptor front end (fpfh.cu): voxel down-sampling, normals, FPFH -------------------------------------
// P clouds packed back to back (offsets [P + 1], host and device; null device tables: one cloud), status [P].  Cloud p's voxel
// means end at row out_ends[p], written by the call, as is out_first[0] = 0 unless out_first is null.
size_t voxel_scratch_bytes(int P, const int32_t* h_off);
void launch_voxel_down_sample(int P, const int32_t* h_off, const int32_t* d_off, const float* pts, double voxel, float* out_pts,
                              int32_t* out_first, int32_t* out_ends, int32_t* status, void* scratch, cudaStream_t st);
size_t fpfh_scratch_bytes(int m, int max_nn);      // m: the call's total key points
int launch_estimate_normals(int P, const int32_t* h_off, const int32_t* d_off, const float* pts, double radius, int max_nn,
                            double* normals, int32_t* status, void* scratch, cudaStream_t st);      // returns cudaError_t
int launch_compute_fpfh(int P, const int32_t* h_off, const int32_t* d_off, const float* pts, const double* normals, double radius,
                        int max_nn, int normalise, double* out, int32_t* status, void* scratch,
                        cudaStream_t st);      // returns cudaError_t

// ---- point-to-point ICP and information matrices between two clouds (icp.cu) ------------------------------------
// B pairs: pair b's source is rows [src_off[b], src_off[b+1]) of src, its target rows [tgt_off[b], tgt_off[b+1]) of tgt (device
// offsets [B + 1]; Rs, Rt = the last entries), init / trans [B,4,4]; fitness, rmse, iterations and status may be null.  The
// correspondence key points are the case src_off = tgt_off.  Scratch: icp_scratch_bytes(Rs, Rt) bytes, 8-byte aligned.
size_t icp_scratch_bytes(long long Rs, long long Rt);
void launch_icp(int B, const int32_t* d_src_off, const int32_t* d_tgt_off, long long Rs, long long Rt, const float* src,
                const float* tgt, const float* init, double r, int max_iteration, float* trans, double* fitness, double* rmse,
                int32_t* iterations, int32_t* status, void* scratch, cudaStream_t st);
// The same pairs, trans [B,4,4] -> info [B,6,6] double; status may be null.  Scratch: information_scratch_bytes(Rt) bytes,
// 8-byte aligned.
size_t information_scratch_bytes(long long Rt);
void launch_information(int B, const int32_t* d_src_off, const int32_t* d_tgt_off, long long Rt, const float* src, const float* tgt,
                        const float* trans, double r, double* info, int32_t* status, void* scratch, cudaStream_t st);

// ---- correspondence RANSAC over the pairs the network kept (ransac.cu) ----------------------------------------
// B sets packed back to back (device offsets [B + 1], R = offsets[B] rows), labels [R] (> 0: a candidate), trans [B,4,4],
// out_labels [R]; fitness, rmse, best, status [B], hyp_good, hyp_rmse [B, max_iteration] and hyp_trans [B, max_iteration, 12]
// may be null.  B <= 65535.
// Scratch: ransac_scratch_bytes(R, B, max_iteration) bytes, 16-byte aligned.
size_t ransac_scratch_bytes(long long R, int B, int max_iteration);
void launch_ransac(int B, const int32_t* d_off, long long R, const float* src, const float* tgt, const float* labels, double r,
                   int max_iteration, unsigned long long seed, float* trans, float* out_labels, double* fitness, double* rmse,
                   int32_t* best, int32_t* status, int32_t* hyp_good, double* hyp_rmse, double* hyp_trans, void* scratch,
                   cudaStream_t st);

// ---- f8: FCGF descriptors (fcgf.cu) -----------------------------------------------------------------------------
// The weight handle of the C ABI (folded, packed and uploaded by fcgf_commit) and the one launch chain of a packed call.
pdsc_fcgf* fcgf_new(int k1);
void fcgf_free(pdsc_fcgf* h);
int fcgf_set_param(pdsc_fcgf* h, const char* name, const float* data, int64_t numel, size_t* expected);   // 1 unknown, 2 size
int fcgf_commit(pdsc_fcgf* h, std::string* missing);      // -1: *missing names an absent parameter; > 0: a cudaError_t
bool fcgf_committed(const pdsc_fcgf* h);
int fcgf_kernel_size(const pdsc_fcgf* h);
size_t fcgf_scratch_bytes(int P, const int32_t* h_off, int k1);
int fcgf_scratch_layout(int P, const int32_t* h_off, int k1, int64_t* offsets, int capacity);
int launch_fcgf(const pdsc_fcgf* h, int P, const int32_t* h_off, const int32_t* d_off, const float* pts, double voxel,
                float* keypts, float* desc, int32_t* out_off, int32_t* status, void* scratch, cudaStream_t st);   // cudaError_t

// ---- the spectral-matching baseline (spectral_matching.cu) ---------------------------------------------------
// B sets packed back to back (host and device offsets [B + 1], R = offsets[B] rows, every set 1 .. spectral_matching_max_n() rows),
// corr [R,6], src / tgt [R,3]; trans [B,4,4], labels [R]; eig_out [R] and iterates [10,R] (row t - 1: iterate v_t, a test
// output) may be null.  B <= 65535.
// Scratch: sm_scratch_bytes(R, B) bytes, 16-byte aligned.
int spectral_matching_max_n();
size_t sm_scratch_bytes(long long R, int B);
void launch_spectral_matching(int B, const int32_t* h_off, const int32_t* d_off, const float* corr, const float* src, const float* tgt,
                              double inlier_threshold, float* trans, float* labels, float* eig_out, float* iterates, void* scratch,
                              cudaStream_t st);

// ---- f9: TSDF integration and surface vertices of RGB-D fragments (fragments.cu) ---------------------------------------
// F fragments of 1 .. kMaxFragmentFrames frames each (device frame offsets [F + 1], NF frames): depth [NF,H,W] uint16, colour
// [NF,H,W,3] uint8, poses [NF,2,16] float64 (extrinsic, camera pose), intrinsic the host fx, fy, cx, cy.  The table
// (tsdf_table_bytes(F, max_units), 8-byte aligned) is written by the touch and read by every later stage of the same volume.
constexpr int kMaxFragmentFrames = 256;
size_t tsdf_table_bytes(int F, int max_units);
size_t tsdf_integrate_scratch_bytes(int F, long long U);
void launch_tsdf_touch(int F, int NF, const int32_t* d_frame_off, int H, int W, const double* intrinsic, const uint16_t* depth,
                       const double* poses, double depth_scale, double depth_trunc, double voxel, double trunc, int max_units,
                       int32_t* counts, int32_t* status, void* table, cudaStream_t st);
void launch_tsdf_integrate(int F, const int32_t* d_frame_off, const int32_t* d_unit_off, long long U, int H, int W,
                           const double* intrinsic, const uint16_t* depth, const uint8_t* color, const double* poses,
                           double depth_scale, double depth_trunc, double voxel, double trunc, int max_units, void* table,
                           int32_t* unit_keys, float* tsdf, float* weight, float* color_out, void* scratch, cudaStream_t st);
void launch_vertex_count(int F, const int32_t* d_unit_off, int U, int max_units, void* table, const int32_t* unit_keys,
                         const float* tsdf, const float* weight, long long* ends, long long* frag_off, cudaStream_t st);
void launch_vertex_write(int F, const int32_t* d_unit_off, int U, int max_units, void* table, const int32_t* unit_keys,
                         const float* tsdf, const float* weight, const float* color, double voxel, const long long* ends,
                         double* vertices, double* colors, cudaStream_t st);

// ---- per-device launch configuration (device_state.cu) ----------------------------------------------------
// opt `kernel` in to `bytes` of dynamic shared memory on the CURRENT device (no-op if already granted there)
cudaError_t ensure_dynamic_smem(const void* kernel, int bytes);
int device_sm_count();   // SM count of the current device

// ---- misc ---------------------------------------------------------------------------------------
void launch_fill_u32(uint32_t* p, uint32_t v, long long n, cudaStream_t st);
void launch_fill_u64(unsigned long long* p, unsigned long long v, long long n, cudaStream_t st);

}  // namespace pdsc
