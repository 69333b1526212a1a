/*
 * pointdsc_b200 — C ABI of the H100-native PointDSC testing-mode forward engine.
 *
 * This is the drop-in boundary for ONE path of the reference: `PointDSC.forward` with the
 * 'testing' key set (reference models/PointDSC.py:128-197).  The reference has no FFI of its
 * own (it is pure Python/PyTorch); the binding a maintainer adds is the ctypes stub in
 * pointdsc_b200/_capi.py (shown in INTEGRATION.md), driven by a torch.nn.Module with the
 * reference's constructor, forward(dict)->dict and state_dict keys (pointdsc_b200/model.py).
 *
 * Conventions
 *   - plain C types only; every entry point returns 0 on success or a pdsc_status code and
 *     records a message retrievable with pdsc_last_error() (thread-local).
 *   - "d_" pointers are device pointers on the engine's device, "h_" pointers host pointers.
 *   - all device work is enqueued on the caller's stream; pdsc_forward() performs NO host
 *     synchronisation and no allocation, so it can be captured in a CUDA graph.
 *   - tensors are dense, row-major, fp32 unless stated; B = number of correspondence sets
 *     in the call, N = correspondences per set (the same N for the whole call, except in
 *     pdsc_forward_packed(), where set b has its own N_b and the sets' rows are packed back to back).
 *   - a batched call is, by definition, the loop of per-set testing forwards (the reference
 *     asserts bs == 1 in testing mode, PointDSC.py:210, :414); in particular the power
 *     iteration's early exit is decided per set (PointDSC.py:354).
 */
#ifndef POINTDSC_B200_H_
#define POINTDSC_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pdsc_engine pdsc_engine;

typedef enum pdsc_status {
  PDSC_OK = 0,
  PDSC_ERR_INVALID_ARGUMENT = 1,
  PDSC_ERR_UNKNOWN_PARAM = 2,
  PDSC_ERR_SHAPE = 3,
  PDSC_ERR_NOT_COMMITTED = 4,
  PDSC_ERR_WORKSPACE = 5,
  PDSC_ERR_CUDA = 6,
  PDSC_ERR_UNSUPPORTED = 7
} pdsc_status;

/* Arithmetic of the encoder's contractions (stage ii).  All other stages are fp32. */
typedef enum pdsc_precision {
  PDSC_FP32_SIMT = 0, /* fp32 FFMA kernels: the exact-arithmetic path                              */
  PDSC_BF16X3 = 1,    /* wgmma f16 / bf16, bf16 hi/lo operand split, 3 products, fp32 accumulate:
                         16 significant bits per operand                                             */
  PDSC_BF16 = 2,      /* wgmma f16 / bf16, single bf16 operands, fp32 accumulate: throughput mode;
                         the 12-layer near-argmax attention amplifies bf16 rounding, so R/t may
                         deviate from the reference by > 1e-4 on some sets (see DESIGN.md)           */
  PDSC_FP16X3 = 3     /* wgmma f16 / bf16, fp16 hi/lo operand split, 3 products, fp32 accumulate:
                         22 significant bits per operand — fp32-grade results on the tensor cores   */
} pdsc_precision;

/* Mirrors PointDSC.__init__ (reference models/PointDSC.py:81-91) plus the engine's precision. */
typedef struct pdsc_config {
  int32_t in_dim;            /* 6                                                        */
  int32_t num_layers;        /* 12 in the released snapshots (ctor default 6)            */
  int32_t num_channels;      /* 128 (only value supported by the kernels)                */
  int32_t num_iterations;    /* power-iteration cap, 10                                  */
  double ratio;              /* seeds: the length of range(N)[:int(N * ratio)], 0.1; any
                                finite value (a ratio above 1 takes every row, a negative
                                one drops the last -int(N * ratio)); pdsc_create refuses
                                a NaN or infinite ratio                                   */
  double inlier_threshold;   /* hypothesis scoring threshold, compared in float32 as the
                                reference's tensors are; also selects the refinement
                                threshold: 0.10 iff == 0.10 exactly, else 1.2
                                (PointDSC.py:415)                                         */
  float sigma_d;             /* initial value of the `sigma_spat` buffer; a loaded
                                state dict overrides it, as in the reference              */
  int32_t k;                 /* neighbourhood size of the NSM module, 40                 */
  float nms_radius;          /* seed NMS radius                                          */
  int32_t precision;         /* pdsc_precision                                           */
  int32_t device;            /* CUDA device ordinal                                      */
} pdsc_config;

/* Optional taps and injection points at the stage boundaries of SURVEY.md §8(a).  Every pointer may
 * be NULL.  `in_*` tensors REPLACE the engine's own result of that stage (used by the parity tests
 * to feed a stage the reference's upstream tensors); `out_*` tensors receive a copy. */
typedef struct pdsc_stage_io {
  /* injection */
  const float* in_features;     /* [B,N,C]  un-normalised encoder output (skips stages i-ii)         */
  const float* in_confidence;   /* [B,N]    confidence logits (requires in_features)                 */
  const int32_t* in_seeds;      /* [B,S]    seed indices                                            */
  const int32_t* in_knn_idx;    /* [B,S,k]  neighbourhoods                                          */
  const float* in_seed_trans;   /* [B,S,4,4] hypotheses                                             */
  /* taps */
  float* out_sc;                /* [B,N,N]  spatial-consistency matrix (a1)                          */
  float* out_features;          /* [B,N,C]  encoder output (a2-a3)                                   */
  float* out_normed;            /* [B,N,C]  L2-normalised features (a4)                              */
  float* out_confidence;        /* [B,N]    (a5)                                                     */
  int32_t* out_seeds;           /* [B,S]    (a6)                                                     */
  int32_t* out_knn_idx;         /* [B,S,k]  (a7)                                                     */
  float* out_compat;            /* [B,S,k,k] (a8)                                                    */
  float* out_eig;               /* [B,S,k]  leading eigenvector at the set's exit iteration (a9)     */
  int32_t* out_power_iters;     /* [B]      iterations run per set (a9); 0 when S = 0                */
  float* out_seed_trans;        /* [B,S,4,4] (a10)                                                   */
  int32_t* out_inlier_counts;   /* [B,S]    inlier count of every hypothesis (a11)                   */
  int32_t* out_best;            /* [B]      selected hypothesis (a11)                                */
  float* out_init_trans;        /* [B,4,4]  selected hypothesis before refinement (a11)              */
  int32_t* out_refine_solves;   /* [B]      Kabsch solves done by the refinement (a12)               */
  int32_t layer_tap;            /* if out_layer_features != NULL: which encoder layer to copy        */
  float* out_layer_features;    /* [B,N,C]  output of encoder layer `layer_tap`                      */
  float* out_layer_debug;       /* [5,B,N,C] internals of layer `layer_tap`: PointCN output, q, k, v, msg.
                                   In the tensor-core modes q carries the folded log2(e)/sqrt(C) scale. */
  int64_t* out_timeline;        /* not written (kept for ABI compatibility); formerly [2,16,4,8] clock64() stamps of CTA 0 of the layer-`layer_tap` PointCN+Q chain
                                   kernel and attention kernel (tensor-core modes; developer tool)            */
} pdsc_stage_io;

/* ---- lifetime --------------------------------------------------------------------------------- */
int pdsc_create(const pdsc_config* cfg, pdsc_engine** out);
int pdsc_destroy(pdsc_engine* e);
const char* pdsc_last_error(void);
const char* pdsc_version(void);

/* ---- parameters: the reference's state dict, key for key (PointDSC.py:93-113) ------------------
 * `name` is a state-dict key ("encoder.layer0.weight", "sigma_spat", ...); `h_data` holds `count`
 * fp32 values in the tensor's own row-major order.  Keys the path does not use
 * (num_batches_tracked, the stray `gamma`) are accepted and ignored, so a released snapshot can be
 * pushed unfiltered.  pdsc_commit_params() folds eval-mode BatchNorm into the preceding 1x1 conv,
 * builds the device-side operand images and must be called before pdsc_forward(). */
int pdsc_set_param(pdsc_engine* e, const char* name, const float* h_data, int64_t count);
int pdsc_commit_params(pdsc_engine* e);
int pdsc_set_precision(pdsc_engine* e, int32_t precision);

/* Batch-invariant mode (off by default).  On: the tensor-core attention splits every set along its keys by a rule of the
 * set's N alone (chunks of PDSC_ATTN_INVARIANT_TILES = 8 key tiles, sets.cuh), in every call, so a set's outputs are bit for
 * bit the same whatever else its call holds (batch size, other sets, their order), whichever entry point runs it and
 * whatever the device's SM count.  Applies to pdsc_forward, _packed, _graph, _host, _host_submit / _wait and
 * pdsc_forward_eval (the validation forward's transform still depends on its batch: the early exit spans the batch);
 * pdsc_workspace_bytes* and pdsc_launches_per_forward report the mode's sizes and merge launches.  Graphs captured in one
 * mode are never replayed in the other.  In PDSC_FP32_SIMT the flag is accepted and changes nothing: that attention never
 * splits.  Off: the default key split, whose choice depends on the whole call and the SM count (DESIGN.md §3). */
int pdsc_set_batch_invariant(pdsc_engine* e, int32_t enable);

/* ---- sizes ------------------------------------------------------------------------------------- */
int32_t pdsc_num_seeds(const pdsc_engine* e, int32_t N);       /* S = len(range(N)[:int(N * ratio)]) */
int32_t pdsc_num_neighbours(const pdsc_engine* e, int32_t N);  /* k = min(cfg.k, N - 1)       */
size_t pdsc_workspace_bytes(const pdsc_engine* e, int32_t B, int32_t N);

/* ---- the path: PointDSC.forward, testing mode (PointDSC.py:128-197) ---------------------------
 * d_corr_pos [B,N,6], d_src_keypts [B,N,3], d_tgt_keypts [B,N,3]  ->
 * d_final_trans [B,4,4] (maps src onto tgt), d_final_labels [B,N] in {0,1}.
 * `io` may be NULL.  `d_workspace` must hold pdsc_workspace_bytes(e,B,N) bytes, 256-byte aligned,
 * and is only used for the duration of the enqueued work. */
int pdsc_forward(pdsc_engine* e, int32_t B, int32_t N, const float* d_corr_pos, const float* d_src_keypts,
                 const float* d_tgt_keypts, float* d_final_trans, float* d_final_labels,
                 const pdsc_stage_io* io, void* d_workspace, size_t workspace_bytes, void* cuda_stream);

/* ---- the path over sets of different sizes (testing mode) -------------------------------------------
 * pdsc_forward(e, B, N, ...) is this call with offsets b * N (the engine builds the same per-set table for both).
 * B sets, set b owning rows [offsets[b], offsets[b+1]) of the packed inputs; offsets has B + 1 entries, offsets[0] = 0,
 * R = offsets[B].  d_corr_pos [R,6], d_src_keypts [R,3], d_tgt_keypts [R,3]  ->  d_final_trans [B,4,4],
 * d_final_labels [R].  h_offsets (host) sizes the launches and the workspace; d_offsets (device, caller-owned, the same
 * values) is what the kernels read.  A set's outputs depend only on its own rows, its N_b and the call's attention regime:
 * within one regime they are bit for bit those of a pdsc_forward() call holding that set (DESIGN.md §3); in the
 * batch-invariant mode (pdsc_set_batch_invariant) there is one regime, so they are in every call.  No host
 * synchronisation, no allocation, capturable in a CUDA graph.  PDSC_ERR_SHAPE for B < 1, offsets[0] != 0, a set with
 * N_b < 2 (non-increasing offsets) or N_b above the supported maximum; pdsc_workspace_bytes_packed() returns 0 for such
 * offsets. */
size_t pdsc_workspace_bytes_packed(const pdsc_engine* e, int32_t B, const int32_t* h_offsets);
int pdsc_forward_packed(pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets,
                        const float* d_corr_pos, const float* d_src_keypts, const float* d_tgt_keypts,
                        float* d_final_trans, float* d_final_labels, void* d_workspace, size_t workspace_bytes,
                        void* cuda_stream);

/* pdsc_forward as ONE graph launch: the first call with a given (B, N, buffer addresses) runs eagerly and captures the
 * forward's kernels into a CUDA graph; later calls with the same arguments replay it (one cudaGraphLaunch instead of ~60
 * kernel launches: the small-batch / bs = 1 case of the evaluation loops, evaluation/test_3DMatch.py:133).  The caller keeps
 * the buffers alive and at the same addresses; up to 8 graphs are cached per engine.  Inside a foreign stream capture, or
 * with profiling enabled, it degrades to pdsc_forward. */
int pdsc_forward_graph(pdsc_engine* e, int32_t B, int32_t N, const float* d_corr_pos, const float* d_src_keypts,
                       const float* d_tgt_keypts, float* d_final_trans, float* d_final_labels, void* d_workspace,
                       size_t workspace_bytes, void* cuda_stream);

/* Same call with HOST buffers (the end-to-end form): pdsc_forward_host_submit below followed by pdsc_forward_host_wait on
 * the slot it took, i.e. the pipelined pair with one call in flight, synchronous on return.  It takes a free slot: with one
 * _submit call in flight it leaves the pipeline as it found it, with two it fails as a third _submit would.  Device staging
 * and workspace are owned by the engine and grown on demand.  The inputs are copied on an engine-owned side stream (not
 * ordered behind `cuda_stream`), key points first: above the size that replays a captured graph the forward starts once
 * they have arrived, so corr_pos (half of the input bytes) is still crossing while the spatial-consistency kernel (which
 * reads only the key points) runs, and is waited for before the first kernel that reads it.  A failed call returns once
 * nothing reads the host inputs any more. */
int pdsc_forward_host(pdsc_engine* e, int32_t B, int32_t N, const float* h_corr_pos, const float* h_src_keypts,
                      const float* h_tgt_keypts, float* h_final_trans, float* h_final_labels, void* cuda_stream);

/* The host form as a two-deep pipeline, for loops over many batches (the evaluation drivers' `for data in loader`,
 * evaluation/test_3DMatch.py:64-101, whose DataLoader workers prefetch the next batch while the model runs the current one):
 * _submit enqueues the host->device copies of this call's inputs on an engine-owned copy stream and the forward on
 * `cuda_stream` behind them, then returns WITHOUT synchronising; `*slot_out` (0 or 1) names the call.  _wait(slot) blocks until
 * that call's forward has finished, copies the two results into the host buffers given to _submit (on a second engine-owned
 * stream, i.e. beside the next call's forward) and returns when they have arrived.  Two calls may be in flight: the input copies
 * of call t + 1 and the result copies of call t - 1 then run beside the forward of call t (the forwards themselves stay
 * serialised on `cuda_stream`: they share one workspace).  All five host buffers must stay valid until _wait returns; the INPUT
 * buffers should be page-locked (from a pageable buffer the copy is synchronous: correct, but without the overlap), the result
 * buffers may be pageable.  A third _submit before a _wait fails with PDSC_ERR_INVALID_ARGUMENT.  Results are bit-identical to
 * pdsc_forward_host's. */
int pdsc_forward_host_submit(pdsc_engine* e, int32_t B, int32_t N, const float* h_corr_pos, const float* h_src_keypts,
                             const float* h_tgt_keypts, float* h_final_trans, float* h_final_labels, void* cuda_stream,
                             int32_t* slot_out);
int pdsc_forward_host_wait(pdsc_engine* e, int32_t slot);

/* ---- the same module call WITHOUT the 'testing' key (validation during training, PointDSC.py:158-165, :176, :190-191):
 * seeds are the top-S correspondences by confidence (no suppression), the power iteration's early exit is decided over the
 * whole batch (the reference's allclose spans [bs*S, k]), there is no post-refinement, `d_confidence` [B,N] receives the
 * classification logits (the reference returns them as final_labels) and, if `d_M` is not NULL, it receives the feature
 * similarity matrix M = clamp(1 - (1 - F F^T) / sigma^2, 0, 1) with a zero diagonal, [B,N,N].  Eval-mode BatchNorm only
 * (running statistics): the training-mode forward and the backward pass are outside this engine. */
int pdsc_forward_eval(pdsc_engine* e, int32_t B, int32_t N, const float* d_corr_pos, const float* d_src_keypts,
                      const float* d_tgt_keypts, float* d_final_trans, float* d_confidence, float* d_M,
                      const pdsc_stage_io* io, void* d_workspace, size_t workspace_bytes, void* cuda_stream);

/* ---- next rows of the path (SURVEY.md section 8f) ---------------------------------------------------------------
 * f3: per-pair evaluation statistics, replacing libs/loss.py:34-63 (TransformationLoss) + :94-100 (ClassificationLoss,
 * scikit-learn on the host) and the per-pair host synchronisation of evaluation/test_3DMatch.py:83-101.
 * d_stats [B,10] = [success, RE deg, TE cm, #gt inliers, gt inlier ratio, #gt inliers among the kept, precision, recall,
 * f1, rmse]; thresholds as the drivers pass them (3DMatch: 15 deg / 30 cm, KITTI: 5 deg / 60 cm).
 * pdsc_eval_stats: B sets of N rows, d_src_keypts / d_tgt_keypts [B,N,3], labels [B,N]; it is the packed call with offsets b * N. */
int pdsc_eval_stats(pdsc_engine* e, int32_t B, int32_t N, const float* d_pred_trans, const float* d_gt_trans,
                    const float* d_src_keypts, const float* d_tgt_keypts, const float* d_pred_labels,
                    const float* d_gt_labels, float re_thre, float te_thre, float* d_stats, void* cuda_stream);
/* The same statistics over sets of different sizes: set b owns rows [offsets[b], offsets[b+1]) of d_src_keypts / d_tgt_keypts
 * [R,3] and the labels [R]; offsets has B + 1 entries, offsets[0] = 0, every set at least one row (else PDSC_ERR_SHAPE).
 * h_offsets (host) is validated, d_offsets (device, the same values) is what the kernel reads; d_pred_trans / d_gt_trans
 * [B,4,4].  A set's row is bit for bit the one pdsc_eval_stats gives for that set alone.  No host synchronisation. */
int pdsc_eval_stats_packed(pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets,
                           const float* d_pred_trans, const float* d_gt_trans, const float* d_src_keypts,
                           const float* d_tgt_keypts, const float* d_pred_labels, const float* d_gt_labels, float re_thre,
                           float te_thre, float* d_stats, void* cuda_stream);

/* f1: the correspondence front end, replacing datasets/ThreeDMatch.py:283-291 + :299-308 (the same lines in
 * datasets/KITTI.py:80-114, demo_registration.py:101-108): nearest neighbour of every source descriptor among the target
 * descriptors under sqrt(2 - 2 <a,b> + 1e-6) evaluated in the descriptors' own dtype (desc_is_fp64: 0 = fp32 FCGF,
 * 1 = fp64 FPFH), first minimum wins, optional mutual check, then the in_dim = 6 network input.
 * pdsc_match: one pair, the packed call below with P = 1.  Outputs in the layout pdsc_forward consumes, sized for the worst
 * case M = Ns: d_corr [Ns,2] int32 (source, target), d_count [1] = M, d_corr_pos [Ns,6] (centred), d_out_src / d_out_tgt
 * [Ns,3]; only the first M rows are written.  D <= 64; d_scratch holds pdsc_match_scratch_bytes(Ns, Nt) bytes, 8-byte
 * aligned. */
size_t pdsc_match_scratch_bytes(int32_t Ns, int32_t Nt);
int pdsc_match(pdsc_engine* e, int32_t Ns, int32_t Nt, int32_t D, const void* d_src_desc, const void* d_tgt_desc,
               int32_t desc_is_fp64, const float* d_src_keypts, const float* d_tgt_keypts, int32_t use_mutual,
               int32_t* d_corr, int32_t* d_count, float* d_corr_pos, float* d_out_src, float* d_out_tgt, void* d_scratch,
               size_t scratch_bytes, void* cuda_stream);
/* P pairs in one call.  Pair p owns source rows [src_offsets[p], src_offsets[p+1]) and target rows [tgt_offsets[p],
 * tgt_offsets[p+1]) of d_src_desc [sum Ns, D] / d_src_keypts [sum Ns, 3] and d_tgt_desc [sum Nt, D] / d_tgt_keypts [sum Nt, 3];
 * each offsets array has P + 1 entries, starts at 0, and every pair needs Ns_p >= 1 and Nt_p >= 1 (else PDSC_ERR_SHAPE, and
 * pdsc_match_packed_scratch_bytes() returns 0).  h_* (host) size the launches, d_* (device, the same values) are what the
 * kernels read.  A pair is matched exactly as pdsc_match matches it alone, against its own targets only (the mutual check
 * too).  Pair p's kept correspondences fill rows [out_offsets[p], out_offsets[p+1]) of d_corr [sum Ns, 2] (pair-local
 * (source, target) indices), d_corr_pos [sum Ns, 6] (centred by the pair's own mean), d_out_src / d_out_tgt [sum Ns, 3], in
 * pair order and ascending source order: the layout pdsc_forward_packed consumes with d_out_offsets [P+1] as its offsets.
 * Without the mutual check out_offsets equals src_offsets.  Rows at or beyond out_offsets[P] are not written.  d_scratch holds
 * pdsc_match_packed_scratch_bytes() bytes, 8-byte aligned.  No host synchronisation, no allocation, capturable in a CUDA
 * graph; results are bit-identical from run to run. */
size_t pdsc_match_packed_scratch_bytes(int32_t P, const int32_t* h_src_offsets, const int32_t* h_tgt_offsets);
int pdsc_match_packed(pdsc_engine* e, int32_t P, int32_t D, const int32_t* h_src_offsets, const int32_t* h_tgt_offsets,
                      const int32_t* d_src_offsets, const int32_t* d_tgt_offsets, const void* d_src_desc, const void* d_tgt_desc,
                      int32_t desc_is_fp64, const float* d_src_keypts, const float* d_tgt_keypts, int32_t use_mutual,
                      int32_t* d_corr, int32_t* d_out_offsets, float* d_corr_pos, float* d_out_src, float* d_out_tgt,
                      void* d_scratch, size_t scratch_bytes, void* cuda_stream);

/* f2: the descriptor front end, replacing the open3d 0.9 calls of misc/cal_fpfh.py:21-26 (and demo_registration.py:37-44):
 *   pcd.voxel_down_sample(voxel)                                                -> pdsc_voxel_down_sample
 *   pcd.estimate_normals(KDTreeSearchParamHybrid(radius = 2 voxel, max_nn = 30)) -> pdsc_estimate_normals
 *   compute_fpfh_feature(pcd, KDTreeSearchParamHybrid(5 voxel, 100))             -> pdsc_compute_fpfh
 *   o3d.io.read_point_cloud(path).points                                         -> pdsc_read_ply (host)
 * open3d is not part of the reference tree: these follow its published algorithms (oracle/fpfh_oracle.py; PARITY UNPINNED).
 * d_points [n,3] float32.  pdsc_voxel_down_sample writes the voxel means to d_out_points (room for [n,3]; rows in ascending
 * (ix, iy, iz) voxel order) and their number to d_count[0]; read d_count after synchronising the stream.  Normals are float64
 * [m,3] (largest-magnitude component positive; (0,0,1) below three neighbours), FPFH float64 [m,33] — the dtype pdsc_match
 * takes with desc_is_fp64 = 1 — with normalise != 0 applying x / (||x|| + 1e-6) per row (demo_registration.py:43).
 * d_status[0] is a bit mask written on the stream: 1 = more than 2^21 voxels along an axis or a non-finite coordinate,
 * 2 = a neighbourhood holds more than 4096 points inside the radius (the search is brute force over the m key points and
 * sized for down-sampled clouds).  Scratch: 8-byte aligned, *_scratch_bytes() bytes. */
size_t pdsc_voxel_down_sample_scratch_bytes(int64_t n);
int pdsc_voxel_down_sample(pdsc_engine* e, int64_t n, const float* d_points, double voxel_size, float* d_out_points,
                           int32_t* d_count, int32_t* d_status, void* d_scratch, size_t scratch_bytes, void* cuda_stream);
size_t pdsc_fpfh_scratch_bytes(int32_t m, int32_t max_nn);
int pdsc_estimate_normals(pdsc_engine* e, int32_t m, const float* d_points, double radius, int32_t max_nn, double* d_normals,
                          int32_t* d_status, void* d_scratch, size_t scratch_bytes, void* cuda_stream);
int pdsc_compute_fpfh(pdsc_engine* e, int32_t m, const float* d_points, const double* d_normals, double radius, int32_t max_nn,
                      int32_t normalise, double* d_fpfh, int32_t* d_status, void* d_scratch, size_t scratch_bytes, void* cuda_stream);
/* The same three steps for P clouds in one call each (misc/cal_fpfh.py:21-26 run over a list of clouds); the calls above are
 * these with P = 1.  Cloud p owns rows [offsets[p], offsets[p+1]) of the packed inputs; offsets has P + 1 entries, starts at 0,
 * and every cloud needs at least one row (else PDSC_ERR_SHAPE, and the *_packed_scratch_bytes() functions return 0).  h_offsets
 * (host) size the launches and the scratch, d_offsets (device, the same values) are what the kernels read.  d_status [P]: cloud
 * p's bits (meanings as above) land in d_status[p] only.  Each cloud is computed exactly as the single-cloud call computes it
 * alone, against its own rows only: its rows are bit for bit that call's.  No host synchronisation, no allocation.
 * pdsc_voxel_down_sample_packed: d_points [n,3], n = offsets[P] <= 2^30; cloud p's voxel means fill rows [out_offsets[p],
 * out_offsets[p+1]) of d_out_points (room for [n,3]), each cloud in ascending (ix, iy, iz) order of its own voxel grid (origin
 * min - voxel / 2 of that cloud); d_out_offsets [P+1] is written on the stream (the key-point offsets of the next two calls).
 * Rows at or beyond out_offsets[P] are not written.
 * pdsc_estimate_normals_packed / pdsc_compute_fpfh_packed: d_points [m,3] key points, m = offsets[P], normals / FPFH as above
 * for all m rows; a row's neighbours are searched among its own cloud's rows.  Scratch: 8-byte aligned,
 * pdsc_voxel_down_sample_packed_scratch_bytes() / pdsc_fpfh_packed_scratch_bytes() bytes (the latter serves both calls). */
size_t pdsc_voxel_down_sample_packed_scratch_bytes(int32_t P, const int32_t* h_offsets);
int pdsc_voxel_down_sample_packed(pdsc_engine* e, int32_t P, const int32_t* h_offsets, const int32_t* d_offsets, const float* d_points,
                                  double voxel_size, float* d_out_points, int32_t* d_out_offsets, int32_t* d_status, void* d_scratch,
                                  size_t scratch_bytes, void* cuda_stream);
size_t pdsc_fpfh_packed_scratch_bytes(int32_t P, const int32_t* h_offsets, int32_t max_nn);
int pdsc_estimate_normals_packed(pdsc_engine* e, int32_t P, const int32_t* h_offsets, const int32_t* d_offsets, const float* d_points,
                                 double radius, int32_t max_nn, double* d_normals, int32_t* d_status, void* d_scratch,
                                 size_t scratch_bytes, void* cuda_stream);
int pdsc_compute_fpfh_packed(pdsc_engine* e, int32_t P, const int32_t* h_offsets, const int32_t* d_offsets, const float* d_points,
                             const double* d_normals, double radius, int32_t max_nn, int32_t normalise, double* d_fpfh,
                             int32_t* d_status, void* d_scratch, size_t scratch_bytes, void* cuda_stream);
/* f8: FCGF descriptors, replacing misc/cal_fcgf.py:11-85 extract_features (rgb = normal = None) with the ResUNetBN2C network of
 * misc/fcgf.py:621-867 (CHANNELS 32/64/128/256, TR_CHANNELS 64/64/64/128, BN, normalize_feature) in MinkowskiEngine 0.5.
 * MinkowskiEngine is not part of the reference tree: the conventions are restated in oracle/fcgf_oracle.py (PARITY UNPINNED).
 * Weights live in a handle of their own, like the engine's: pdsc_fcgf_create(conv1_kernel_size (7: the 3DMatch weights at voxel
 * 0.05; 5: the KITTI weights at voxel 0.30), &h); pdsc_fcgf_set_param(h, name, data, numel) with the checkpoint's state_dict keys
 * and element counts (convolution kernels `<name>.kernel` in MinkowskiEngine's [K^3, Cin, Cout] / [Cin, Cout] layout, norms
 * `<name>.bn.{weight,bias,running_mean,running_var}`, `final.bias`; num_batches_tracked is not passed): PDSC_ERR_UNKNOWN_PARAM for
 * another name, PDSC_ERR_SHAPE for another count; pdsc_fcgf_commit(h) folds every BN (eps 1e-5) in float64 and uploads to the
 * current device (PDSC_ERR_UNKNOWN_PARAM names a missing entry); pdsc_fcgf_destroy(h) frees it.
 * pdsc_fcgf_packed: P clouds, cloud p owning rows [offsets[p], offsets[p+1]) of d_points [n,3] float32 (offsets as for
 * pdsc_voxel_down_sample_packed, n = offsets[P] <= 2^26; h_offsets sizes the launches and the scratch, d_offsets is what the kernels
 * read).  Per cloud: voxel coordinates floor((double)x / voxel_size), one row per occupied voxel in order of its first point, the
 * key point = that first point; the 32-channel unit descriptor of every row.  Outputs: d_out_offsets [P+1] (written on the
 * stream), d_keypts [n,3] and d_desc [n,32] float32 (rows [out_offsets[p], out_offsets[p+1]) are cloud p's; rows at or beyond
 * out_offsets[P] are not written), d_status [P]: bit 1 = a non-finite coordinate or one outside [-2^20, 2^20) voxels (the point
 * is left out).  A cloud's rows are bit for bit the same in any call, in any order, on any SM count.  Scratch:
 * pdsc_fcgf_packed_scratch_bytes() bytes (about 11 KB per input point with conv1_kernel_size 7), 256-byte aligned.  No host
 * synchronisation, no allocation, capturable in a CUDA graph.
 * pdsc_fcgf_scratch_layout (a test aid): the byte offsets inside that scratch, after a call, of 37 regions, in this order: every
 * level's row offsets [P+1] int32 (levels 0..3, tensor strides 1, 2, 4, 8); every level's voxel coordinates [n,3] int32; the conv1
 * neighbour table [n,K^3]; the same-stride 3^3 tables of levels 0..3, the strided tables of levels 1..3 (a row of level l gathers
 * level l-1) and the transposed tables of levels 0..2 (a row of level l gathers level l+1), each [n,27] int32 (-1: no neighbour);
 * then the 18 feature buffers [n,w] float32 (x, t, cat, d, dt of levels 0, 1, 2, then x, t, s8 of level 3) that DESIGN.md's f8
 * table assigns to each convolution.  Returns the count (0 for bad arguments); writes at most `capacity` offsets. */
typedef struct pdsc_fcgf pdsc_fcgf;
int pdsc_fcgf_create(int32_t conv1_kernel_size, pdsc_fcgf** h);
int pdsc_fcgf_set_param(pdsc_fcgf* h, const char* name, const float* h_data, int64_t numel);
int pdsc_fcgf_commit(pdsc_fcgf* h);
int pdsc_fcgf_destroy(pdsc_fcgf* h);
size_t pdsc_fcgf_packed_scratch_bytes(const pdsc_fcgf* h, int32_t P, const int32_t* h_offsets);
int pdsc_fcgf_packed(pdsc_engine* e, const pdsc_fcgf* h, int32_t P, const int32_t* h_offsets, const int32_t* d_offsets,
                     const float* d_points, double voxel_size, float* d_keypts, float* d_desc, int32_t* d_out_offsets,
                     int32_t* d_status, void* d_scratch, size_t scratch_bytes, void* cuda_stream);
int32_t pdsc_fcgf_scratch_layout(const pdsc_fcgf* h, int32_t P, const int32_t* h_offsets, int64_t* offsets, int32_t capacity);
/* f5: point-to-point ICP over the correspondence key points, replacing icp_refine (evaluation/benchmark_utils.py:40-55): open3d 0.9's
 * registration_icp(src, tgt, max_corr_dist, init, TransformationEstimationPointToPoint(False), ICPConvergenceCriteria()) with the
 * criteria fixed at their defaults (relative fitness 1e-6, relative rmse 1e-6).  open3d is not part of the reference tree: this
 * follows its published algorithm (oracle/icp_oracle.py; PARITY UNPINNED).  B sets; set b owns rows [offsets[b], offsets[b+1]) of
 * d_src / d_tgt [R,3] (the pair's src_keypts / tgt_keypts); offsets has B + 1 entries, starts at 0, every set at least one row
 * (else PDSC_ERR_SHAPE, and pdsc_icp_packed_scratch_bytes() returns 0); h_offsets (host) is validated and sizes the scratch,
 * d_offsets (device, the same values) is what the kernel reads.  T starts at d_init [B,4,4] and is kept in fp64; every source row is
 * matched to its nearest target row of the same set, kept iff d^2 < float32(max_corr_dist^2), ties to the lowest row; each
 * iteration applies the unscaled Umeyama update over the kept pairs, for at most max_iteration (>= 1) updates.  Outputs:
 * d_trans [B,4,4] float32; optional (may be NULL) d_fitness [B] (kept / N_b), d_rmse [B] (inlier RMSE), d_iterations [B] (updates
 * applied), d_status [B] (1: a non-finite coordinate, or the target spans 2^21 or more cells of side max_corr_dist along an axis;
 * such a set returns d_init after 0 iterations with fitness = rmse = 0).  PDSC_ERR_INVALID_ARGUMENT for max_corr_dist <= 0 or not
 * finite and for max_iteration < 1.  A set's outputs depend on its own rows only: bit for bit the same in any call, in any order, on
 * any SM count.  Scratch: pdsc_icp_packed_scratch_bytes() bytes, 8-byte aligned.  No host synchronisation, no allocation,
 * capturable in a CUDA graph. */
size_t pdsc_icp_packed_scratch_bytes(int32_t B, const int32_t* h_offsets);
int pdsc_icp_packed(pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets, const float* d_src,
                    const float* d_tgt, const float* d_init, double max_corr_dist, int32_t max_iteration, float* d_trans,
                    double* d_fitness, double* d_rmse, int32_t* d_iterations, int32_t* d_status, void* d_scratch, size_t scratch_bytes,
                    void* cuda_stream);
/* f7: the same ICP between two different clouds, for the multiway registration's local_refinement (multiway/test_multi_ate.py):
 * pair b's source is rows [src_offsets[b], src_offsets[b+1]) of d_src [Rs,3] and its target rows [tgt_offsets[b],
 * tgt_offsets[b+1]) of d_tgt [Rt,3] (two fragments, Ns and Nt rows); both offset arrays have B + 1 entries, start at 0 and give
 * every pair at least one row on each side (else PDSC_ERR_SHAPE, and the scratch-size function returns 0).  Semantics, outputs,
 * errors and guarantees as pdsc_icp_packed, with fitness = kept / Ns; pdsc_icp_packed is this call with tgt_offsets =
 * src_offsets, bit for bit.  The host offsets are validated and size the scratch; the device ones are what the kernel reads and
 * may describe fewer rows: any offsets with at least one row per pair on each side and a last entry no larger than the host
 * one's (they need not start at 0), such as the d_out_offsets of a pdsc_voxel_down_sample_packed call over clouds the host
 * offsets describe, so that a down-sampling and an ICP chain on the stream with nothing read back.  Scratch:
 * pdsc_icp_clouds_packed_scratch_bytes() bytes, 8-byte aligned. */
size_t pdsc_icp_clouds_packed_scratch_bytes(int32_t B, const int32_t* h_src_offsets, const int32_t* h_tgt_offsets);
int pdsc_icp_clouds_packed(pdsc_engine* e, int32_t B, const int32_t* h_src_offsets, const int32_t* h_tgt_offsets,
                           const int32_t* d_src_offsets, const int32_t* d_tgt_offsets, const float* d_src, const float* d_tgt,
                           const float* d_init, double max_corr_dist, int32_t max_iteration, float* d_trans, double* d_fitness,
                           double* d_rmse, int32_t* d_iterations, int32_t* d_status, void* d_scratch, size_t scratch_bytes,
                           void* cuda_stream);
/* f7: open3d 0.9's get_information_matrix_from_point_clouds(src, tgt, max_corr_dist, T) for B pairs in one call (recalled, not
 * checkable here; tests/multiway_oracle.py restates it; PARITY UNPINNED).  Pairs and offsets (device ones included) as
 * pdsc_icp_clouds_packed.  The source is
 * moved by d_trans [B,4,4] float32 in fp64; each source row's nearest target row is kept iff d^2 < float32(max_corr_dist^2), ties to
 * the lowest row; every kept correspondence with target point (x, y, z) adds G G^T for the rows (0, z, -y, 1, 0, 0),
 * (-z, 0, x, 0, 1, 0) and (y, -x, 0, 0, 0, 1) of G, so d_info[b][5][5] is the number kept.  Outputs: d_info [B,6,6] float64;
 * optional (may be NULL) d_status [B] (1: a non-finite coordinate, or the target spans 2^21 or more cells of side max_corr_dist
 * along an axis; such a pair gets the zero matrix).  PDSC_ERR_INVALID_ARGUMENT for null required pointers and max_corr_dist <= 0
 * or not finite.  Sums run in a fixed order: a pair's matrix is bit for bit the same in any call, in any order, on any SM count.
 * Scratch: pdsc_information_matrix_packed_scratch_bytes() bytes, 8-byte aligned.  No host synchronisation, no allocation,
 * capturable in a CUDA graph. */
size_t pdsc_information_matrix_packed_scratch_bytes(int32_t B, const int32_t* h_src_offsets, const int32_t* h_tgt_offsets);
int pdsc_information_matrix_packed(pdsc_engine* e, int32_t B, const int32_t* h_src_offsets, const int32_t* h_tgt_offsets,
                                   const int32_t* d_src_offsets, const int32_t* d_tgt_offsets, const float* d_src, const float* d_tgt,
                                   const float* d_trans, double max_corr_dist, double* d_info, int32_t* d_status, void* d_scratch,
                                   size_t scratch_bytes, void* cuda_stream);

/* f6: correspondence RANSAC over the pairs the network kept, replacing the drivers' --solver RANSAC block
 * (evaluation/test_3DMatch.py:59-77): open3d 0.9's registration_ransac_based_on_correspondence with ransac_n = 3 and
 * max_iteration = max_validation, over the rows with pred_labels > 0.  open3d is not part of the reference tree: this follows its
 * published algorithm (oracle/ransac_oracle.py; PARITY UNPINNED), with draws of its own.  B sets as for pdsc_icp_packed (every set
 * at least one row, else PDSC_ERR_SHAPE and pdsc_ransac_packed_scratch_bytes() returns 0; B <= 65535, else PDSC_ERR_UNSUPPORTED);
 * d_src / d_tgt [R,3] the key points, d_labels [R] the forward's final_labels.  The candidates of set b are its rows with label > 0
 * in ascending order, M_b of them.  Iteration i < max_iteration draws candidates (z >> 33) % M_b, z = SplitMix64(seed + (3 i + j + 1)
 * * 0x9E3779B97F4A7C15) for j = 0, 1, 2, solves the unscaled Umeyama over them in double and counts the candidates with
 * |R p + t - q|^2 < max_corr_dist * max_corr_dist (in double): good, rmse = sqrt(sum d^2 / good).  The winner is the hypothesis
 * with the most inliers, then the smallest rmse, then the earliest iteration, among those with good > 0.  Outputs: d_trans
 * [B,4,4] float32, the winner's 3-point solve; d_out_labels [R] (must not overlap the inputs) 1 on exactly its inliers, 0
 * elsewhere; optional (may be NULL) d_fitness [B] (good / M_b), d_rmse [B], d_best [B] (the winning iteration, -1 when none),
 * d_status [B] (0; 1: M_b < 3; 2: no hypothesis with an inlier; both return the identity and all-zero labels), d_hyp_good /
 * d_hyp_rmse [B, max_iteration] (every hypothesis's key; 0 for a set with status 1).  PDSC_ERR_INVALID_ARGUMENT for null
 * required pointers, max_corr_dist <= 0 or not finite and max_iteration < 1.  A set's outputs depend on its own rows, labels,
 * max_corr_dist, max_iteration and seed only: bit for bit the same in any call, in any order, on any SM count.  Scratch:
 * pdsc_ransac_packed_scratch_bytes() bytes, 16-byte aligned (0 for bad offsets or max_iteration < 1).  No host synchronisation,
 * no allocation, capturable in a CUDA graph. */
size_t pdsc_ransac_packed_scratch_bytes(int32_t B, const int32_t* h_offsets, int32_t max_iteration);
int pdsc_ransac_packed(pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets, const float* d_src,
                       const float* d_tgt, const float* d_labels, double max_corr_dist, int32_t max_iteration, uint64_t seed,
                       float* d_trans, float* d_out_labels, double* d_fitness, double* d_rmse, int32_t* d_best, int32_t* d_status,
                       int32_t* d_hyp_good, double* d_hyp_rmse, void* d_scratch, size_t scratch_bytes, void* cuda_stream);
/* pdsc_ransac_packed with one more optional output, d_hyp_trans [B, max_iteration, 12] double (may be NULL): every hypothesis's
 * [R | t], row-major, the transform its key was scored with; [I | 0] for a set with status 1 and for a sample with a non-finite
 * coordinate.  A test output: the finish kernel solves every hypothesis once more to write it.  Same arguments, checks, scratch
 * and results otherwise. */
int pdsc_ransac_packed_hypotheses(pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets, const float* d_src,
                                  const float* d_tgt, const float* d_labels, double max_corr_dist, int32_t max_iteration,
                                  uint64_t seed, float* d_trans, float* d_out_labels, double* d_fitness, double* d_rmse,
                                  int32_t* d_best, int32_t* d_status, int32_t* d_hyp_good, double* d_hyp_rmse, double* d_hyp_trans,
                                  void* d_scratch, size_t scratch_bytes, void* cuda_stream);

/* The classical spectral-matching baseline SM (baseline_scripts/baseline_3DMatch.py:19-53) for B sets in one call.  Set b owns
 * rows [offsets[b], offsets[b+1]) of d_corr_pos [R,6] (the centred corr_pos of the evaluation loop) and of d_src_keypts /
 * d_tgt_keypts [R,3]; offsets as for pdsc_icp_packed, every set between 1 and 16,384 rows (else PDSC_ERR_SHAPE, and
 * pdsc_spectral_matching_packed_scratch_bytes() returns 0); B <= 65535, else PDSC_ERR_UNSUPPORTED.  Per set of N rows:
 * M_ij = max(0, 4.5 - (||c_j[0:3] - c_i[0:3]|| - ||c_j[3:6] - c_i[3:6]||)^2 / (2 sigma^2)), sigma = inlier_threshold / 3,
 * M_ii = 0 (never stored); v = 1, then exactly ten v <- M v / (||M v|| + 1e-6); labels = 1 on the S = int(N * 0.1) largest
 * entries of v (ties: the lowest row first), 0 elsewhere; T = rigid_transform_3d(src, tgt, v * labels) (models/common.py:7-45),
 * the identity when every weight is 0 (S = 0 included).  Outputs: d_trans [B,4,4] float32, d_labels [R] float32, optional
 * d_eigenvector [R] float32 (v).  PDSC_ERR_INVALID_ARGUMENT for null required pointers and an inlier_threshold <= 0 or not
 * finite.  A set's outputs depend on its own rows and inlier_threshold only: bit for bit the same in any call, in any order, on any
 * SM count.  Scratch: pdsc_spectral_matching_packed_scratch_bytes() bytes, 16-byte aligned.  No host synchronisation, no
 * allocation, capturable in a CUDA graph. */
size_t pdsc_spectral_matching_packed_scratch_bytes(int32_t B, const int32_t* h_offsets);
int pdsc_spectral_matching_packed(pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets,
                                  const float* d_corr_pos, const float* d_src_keypts, const float* d_tgt_keypts, double inlier_threshold,
                                  float* d_trans, float* d_labels, float* d_eigenvector, void* d_scratch, size_t scratch_bytes,
                                  void* cuda_stream);
/* pdsc_spectral_matching_packed with one more optional output, d_iterates [10,R] float32 (may be NULL): row t - 1 holds every
 * set's iterate v_t of the ten power iterations, so that each step can be checked on its own (row 9 is d_eigenvector).  A test
 * output: the normalisation of iteration t writes it as it writes v_t.  Same arguments, checks, scratch and results otherwise. */
int pdsc_spectral_matching_packed_iterates(pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets,
                                           const float* d_corr_pos, const float* d_src_keypts, const float* d_tgt_keypts,
                                           double inlier_threshold, float* d_trans, float* d_labels, float* d_eigenvector,
                                           float* d_iterates, void* d_scratch, size_t scratch_bytes, void* cuda_stream);

/* Vertex positions of a PLY file (ascii or binary_little_endian; x, y, z float or double) into host memory as [n,3] float32.
 * Call with points = NULL to learn *n_vertices, then with a buffer of `capacity` >= n vertices. */
int pdsc_read_ply(const char* path, float* points, int64_t capacity, int64_t* n_vertices);

/* f4: leading eigenvector of N x N compatibility matrices by power iteration, replacing cal_leading_eigenvector(M, 'power')
 * (models/PointDSC.py:338-358) in its N x N uses: the learned feature-similarity matrix of the non-testing forward (:170) and
 * the classical spectral-matching baseline (baseline_scripts/baseline_3DMatch.py:40-44, ten fixed iterations = early_exit 0).
 * d_M [B,N,N] row-major; start vector all ones; v <- M v / (||M v|| + 1e-6); with early_exit the iteration of a set stops
 * when allclose(v, v_prev, rtol 1e-5, atol 1e-8) holds (per set, decided on the device).  d_eigenvector [B,N],
 * d_iterations_run [B]; d_scratch holds pdsc_leading_eigenvector_scratch_bytes(B, N) bytes, 16-byte aligned. */
size_t pdsc_leading_eigenvector_scratch_bytes(int32_t B, int32_t N);
int pdsc_leading_eigenvector(pdsc_engine* e, int32_t B, int32_t N, const float* d_M, int32_t num_iterations, int32_t early_exit,
                             float* d_eigenvector, int32_t* d_iterations_run, void* d_scratch, size_t scratch_bytes,
                             void* cuda_stream);

/* f9: the fragments of the multiway experiment (multiway/make_fragments.py): open3d 0.9's ScalableTSDFVolume(RGB8) integration and
 * the vertices (with colours) of extract_triangle_mesh, for F fragments in one call per stage.  Conventions restated in
 * numpy under oracle/ (PARITY UNPINNED).  Fragment f owns frames h/d_frame_offsets[f] .. [f+1] (1 .. 256 frames) of
 * d_depth [NF,H,W] uint16 (metres = raw / depth_scale, 0 at or beyond depth_trunc), d_color [NF,H,W,3] uint8 and d_poses [NF,2,16]
 * float64 (row-major extrinsic, world to camera, then its inverse, the camera pose); intrinsic is the host {fx, fy, cx, cy}.
 * A volume unit is 16^3 voxels of side voxel_length.  The three stages share one table (pdsc_tsdf_table_bytes(F, max_units), 8-byte
 * aligned, max_units units per fragment at most), which the touch initialises and every later stage of the same volume reads:
 * 1. pdsc_tsdf_touch_packed: d_unit_counts [F] int32 (the units each fragment's frames touch) and d_status [F] int32 (bit 1: more
 *    than max_units units, the volume is incomplete; bit 2: a point beyond 2^20 units from the origin, skipped).
 * 2. pdsc_tsdf_integrate_packed with h/d_unit_offsets [F+1] from those counts: d_unit_keys [U,3] int32 (unit coordinates, each
 *    fragment's sorted ascending), d_tsdf and d_weight [U,16,16,16] float32 and d_voxel_color [U,16,16,16,3] float32 (0 .. 255), bit
 *    for bit the float32 restatement.  Unit offsets above the touch's counts leave the extra rows at the end of their fragment
 *    with coordinates INT32_MIN and weight 0; nothing is written outside the table, the scratch and the outputs.  At most 65535
 *    frames per call.  Scratch: pdsc_tsdf_integrate_scratch_bytes() bytes, 8-byte aligned.
 * 3. pdsc_extract_vertices_count_packed: d_vertex_ends [U] int64 (inclusive ends of every unit's vertices) and d_vertex_offsets
 *    [F+1] int64; then pdsc_extract_vertices_packed: d_vertices and d_vertex_colors [V,3] float64 (colours in 0 .. 1), ordered by
 *    (fragment, unit, x, y, z, edge axis).
 * Everything runs on the caller's stream with no host synchronisation and no allocation; a fragment's outputs are bit for bit the
 * same in any group, in any order, at any SM count. */
size_t pdsc_tsdf_table_bytes(int32_t F, int32_t max_units);
int pdsc_tsdf_touch_packed(pdsc_engine* e, int32_t F, const int32_t* h_frame_offsets, const int32_t* d_frame_offsets, int32_t height,
                           int32_t width, const double* intrinsic, const uint16_t* d_depth, const double* d_poses, double depth_scale,
                           double depth_trunc, double voxel_length, double sdf_trunc, int32_t max_units, int32_t* d_unit_counts,
                           int32_t* d_status, void* d_table, size_t table_bytes, void* cuda_stream);
size_t pdsc_tsdf_integrate_scratch_bytes(int32_t F, const int32_t* h_unit_offsets);
int pdsc_tsdf_integrate_packed(pdsc_engine* e, int32_t F, const int32_t* h_frame_offsets, const int32_t* d_frame_offsets,
                               const int32_t* h_unit_offsets, const int32_t* d_unit_offsets, int32_t height, int32_t width,
                               const double* intrinsic, const uint16_t* d_depth, const uint8_t* d_color, const double* d_poses,
                               double depth_scale, double depth_trunc, double voxel_length, double sdf_trunc, int32_t max_units,
                               void* d_table, size_t table_bytes, int32_t* d_unit_keys, float* d_tsdf, float* d_weight,
                               float* d_voxel_color, void* d_scratch, size_t scratch_bytes, void* cuda_stream);
int pdsc_extract_vertices_count_packed(pdsc_engine* e, int32_t F, const int32_t* h_unit_offsets, const int32_t* d_unit_offsets,
                                       int32_t max_units, void* d_table, size_t table_bytes, const int32_t* d_unit_keys,
                                       const float* d_tsdf, const float* d_weight, int64_t* d_vertex_ends, int64_t* d_vertex_offsets,
                                       void* cuda_stream);
int pdsc_extract_vertices_packed(pdsc_engine* e, int32_t F, const int32_t* h_unit_offsets, const int32_t* d_unit_offsets,
                                 int32_t max_units, void* d_table, size_t table_bytes, const int32_t* d_unit_keys, const float* d_tsdf,
                                 const float* d_weight, const float* d_voxel_color, double voxel_length, const int64_t* d_vertex_ends,
                                 double* d_vertices, double* d_vertex_colors, void* cuda_stream);

/* ---- live profiling with CUDA events on the caller's stream ------------------------------------------
 * When enabled, pdsc_forward() records an event pair around each stage below (and around EVERY launch of
 * the dominant kernel, the per-layer attention).  pdsc_profile_read() waits for the last forward's events
 * and returns, per span, the accumulated milliseconds and the number of launches since the last read.
 * Not capturable in a CUDA graph; costs two event records per span. */
typedef enum pdsc_span {
  PDSC_SPAN_SC = 0,          /* a1  sc_matrix                                   */
  PDSC_SPAN_LINEAR = 1,      /* a2  layer0 + PointCN/QKV/fc_message kernels     */
  PDSC_SPAN_ATTENTION = 2,   /* a3  attention kernel (one span per layer)       */
  PDSC_SPAN_HEAD = 3,        /* a4+a5                                           */
  PDSC_SPAN_SEEDS = 4,       /* a6                                              */
  PDSC_SPAN_KNN = 5,         /* a7                                              */
  PDSC_SPAN_NSM = 6,         /* a8+a9                                           */
  PDSC_SPAN_HYPOTHESES = 7,  /* a10+a11                                         */
  PDSC_SPAN_REFINE = 8,      /* a11 labels + a12                                */
  PDSC_SPAN_TOTAL = 9,       /* whole pdsc_forward                              */
  PDSC_SPAN_COUNT = 10
} pdsc_span;
int pdsc_profile_enable(pdsc_engine* e, int32_t enable);
int pdsc_profile_read(pdsc_engine* e, float* ms_out /* [PDSC_SPAN_COUNT] */, int32_t* launches_out /* [PDSC_SPAN_COUNT] */);

/* Number of kernels one pdsc_forward(B,N) call launches at the current precision (bench.py's
 * `gpu_launches`). */
int32_t pdsc_launches_per_forward(const pdsc_engine* e, int32_t B, int32_t N);

#ifdef __cplusplus
}
#endif
#endif /* POINTDSC_B200_H_ */
