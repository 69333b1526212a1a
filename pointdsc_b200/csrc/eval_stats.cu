// f3 — per-pair evaluation statistics on the device (SURVEY.md §8 row f3).
//
// Reference: libs/loss.py:34-63 (TransformationLoss.forward: RE in degrees through the trace of R^T R_gt clamped into acos'
// domain, TE in cm, success flag, RMSE of the correspondences under the predicted transform — torch.norm(...).mean()),
// libs/loss.py:94-100 (ClassificationLoss: precision / recall / F1 of `pred > 0` against the ground-truth labels, computed
// there with scikit-learn on the host after a device->host copy) and the columns evaluation/test_3DMatch.py:85-96 records
// per pair.  The evaluation loop synchronises with the host once per pair for these numbers; here one CTA per set reduces
// them on the device and a batch costs one launch.  Set b owns rows [offsets[b], offsets[b+1]) of the packed key points and
// labels (pdsc_eval_stats_packed), or rows [b N, (b + 1) N) (pdsc_eval_stats: the same kernel without a table).
//
// Output row (10 floats per set): [success, RE deg, TE cm, #gt inliers, gt inlier ratio, #gt inliers among the kept,
//                                  precision, recall, f1, rmse]
// Counts are exact integers (fp32 holds them below 2^24); sums of distances are accumulated in fp64.
#include <cmath>

#include "abi.h"
#include "common.cuh"
#include "sets.cuh"

namespace pdsc {

constexpr int kStatsThreads = 256;

__global__ void __launch_bounds__(kStatsThreads) eval_stats_kernel(const float* __restrict__ pred_trans,
                                                                   const float* __restrict__ gt_trans,
                                                                   const float* __restrict__ src, const float* __restrict__ tgt,
                                                                   const float* __restrict__ pred_labels,
                                                                   const float* __restrict__ gt_labels, float* __restrict__ stats,
                                                                   Offsets off, float re_thre, float te_thre) {
  __shared__ double red_d[kStatsThreads / 32];
  __shared__ int red_i[4][kStatsThreads / 32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const size_t row0 = (size_t)off.at(b);
  const int N = off.at(b + 1) - off.at(b);
  const float* T = pred_trans + (size_t)b * 16;
  const float* G = gt_trans + (size_t)b * 16;
  const float r00 = T[0], r01 = T[1], r02 = T[2], t0 = T[3], r10 = T[4], r11 = T[5], r12 = T[6], t1 = T[7], r20 = T[8],
              r21 = T[9], r22 = T[10], t2 = T[11];
  const float* ps = src + row0 * 3;
  const float* pt = tgt + row0 * 3;
  const float* pl = pred_labels + row0;
  const float* gl = gt_labels + row0;
  double dist_sum = 0.0;
  int tp = 0, fp = 0, fn = 0, gt_sum = 0;
  for (int i = tid; i < N; i += kStatsThreads) {
    const float x = ps[3 * i], y = ps[3 * i + 1], z = ps[3 * i + 2];
    // warped = R x + t (utils/SE3.py:43-57), distance as torch.norm does it (common.cuh::length3)
    const float wx = __fadd_rn(__fmaf_rn(r02, z, __fmaf_rn(r01, y, __fmul_rn(r00, x))), t0);
    const float wy = __fadd_rn(__fmaf_rn(r12, z, __fmaf_rn(r11, y, __fmul_rn(r10, x))), t1);
    const float wz = __fadd_rn(__fmaf_rn(r22, z, __fmaf_rn(r21, y, __fmul_rn(r20, x))), t2);
    dist_sum += (double)length3(wx - pt[3 * i], wy - pt[3 * i + 1], wz - pt[3 * i + 2]);
    const bool p = pl[i] > 0.f, g = gl[i] > 0.f;
    tp += (p && g); fp += (p && !g); fn += (!p && g); gt_sum += g;
  }
  dist_sum = warp_sum(dist_sum);
  tp = warp_sum(tp); fp = warp_sum(fp); fn = warp_sum(fn); gt_sum = warp_sum(gt_sum);
  if (lane == 0) { red_d[warp] = dist_sum; red_i[0][warp] = tp; red_i[1][warp] = fp; red_i[2][warp] = fn; red_i[3][warp] = gt_sum; }
  __syncthreads();
  if (tid == 0) {
    double ds = 0.0;
    int c[4] = {0, 0, 0, 0};
    for (int w = 0; w < kStatsThreads / 32; ++w) {
      ds += red_d[w];
      for (int q = 0; q < 4; ++q) c[q] += red_i[q][w];
    }
    // trace(R^T R_gt): the three diagonal entries of the product (column dots), then their sum, as the matmul + trace of
    // the reference evaluates them
    float tr = 0.f;
    for (int j = 0; j < 3; ++j) {
      float d = __fmul_rn(T[j], G[j]);
      d = __fmaf_rn(T[4 + j], G[4 + j], d);
      d = __fmaf_rn(T[8 + j], G[8 + j], d);
      tr = __fadd_rn(tr, d);
    }
    const float cosv = fminf(fmaxf((tr - 1.0f) / 2.0f, -1.0f), 1.0f);
    const float re = acosf(cosv) * 180.0f / 3.14159265358979323846f;
    const float dx = T[3] - G[3], dy = T[7] - G[7], dz = T[11] - G[11];
    const float te = sqrtf(dx * dx + dy * dy + dz * dz) * 100.0f;
    const float tpf = (float)c[0], fpf = (float)c[1], fnf = (float)c[2];
    float* row = stats + (size_t)b * 10;
    row[0] = (te < te_thre && re < re_thre) ? 1.0f : 0.0f;
    row[1] = re;
    row[2] = te;
    row[3] = (float)c[3];
    row[4] = N > 0 ? (float)c[3] / (float)N : 0.f;
    row[5] = tpf;                                                  // gt inliers among the kept = true positives
    row[6] = (c[0] + c[1]) > 0 ? tpf / (tpf + fpf) : 0.f;          // scikit-learn's zero-denominator rule: score 0
    row[7] = (c[0] + c[2]) > 0 ? tpf / (tpf + fnf) : 0.f;
    row[8] = (2 * c[0] + c[1] + c[2]) > 0 ? 2.f * tpf / (2.f * tpf + fpf + fnf) : 0.f;
    row[9] = N > 0 ? (float)(ds / (double)N) : 0.f;
  }
}

// set b: rows [offsets[b], offsets[b+1]), or b * N without a table
static int eval_stats_impl(pdsc_engine* e, int32_t B, const int32_t* d_offsets, int32_t N, const float* d_pred_trans,
                           const float* d_gt_trans, const float* d_src, const float* d_tgt, const float* d_pred_labels,
                           const float* d_gt_labels, float re_thre, float te_thre, float* d_stats, void* cuda_stream) {
  if (!d_pred_trans || !d_gt_trans || !d_src || !d_tgt || !d_pred_labels || !d_gt_labels || !d_stats)
    return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_eval_stats: null tensor pointer");
  DeviceGuard g(engine_config(e).device);
  eval_stats_kernel<<<B, kStatsThreads, 0, static_cast<cudaStream_t>(cuda_stream)>>>(
      d_pred_trans, d_gt_trans, d_src, d_tgt, d_pred_labels, d_gt_labels, d_stats, Offsets{d_offsets, d_offsets ? 0 : N}, re_thre,
      te_thre);
  PDSC_CUDA(cudaGetLastError());
  return PDSC_OK;
}

}  // namespace pdsc

// ---- C ABI ------------------------------------------------------------------------------------------------------
using namespace pdsc;

extern "C" {

int pdsc_eval_stats(pdsc_engine* e, int32_t B, int32_t N, const float* d_pred_trans, const float* d_gt_trans,
                    const float* d_src, const float* d_tgt, const float* d_pred_labels, const float* d_gt_labels,
                    float re_thre, float te_thre, float* d_stats, void* cuda_stream) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (B <= 0 || N <= 0) return fail(PDSC_ERR_SHAPE, "need B >= 1 and N >= 1 (got B=%d N=%d)", B, N);
  return eval_stats_impl(e, B, nullptr, N, d_pred_trans, d_gt_trans, d_src, d_tgt, d_pred_labels, d_gt_labels, re_thre, te_thre,
                         d_stats, cuda_stream);
}

int pdsc_eval_stats_packed(pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets,
                           const float* d_pred_trans, const float* d_gt_trans, const float* d_src, const float* d_tgt,
                           const float* d_pred_labels, const float* d_gt_labels, float re_thre, float te_thre, float* d_stats,
                           void* cuda_stream) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (int rc = check_offsets("pdsc_eval_stats_packed", "", B, h_offsets, 1)) return rc;
  if (!d_offsets) return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_eval_stats_packed: null device offsets");
  return eval_stats_impl(e, B, d_offsets, 0, d_pred_trans, d_gt_trans, d_src, d_tgt, d_pred_labels, d_gt_labels, re_thre, te_thre,
                         d_stats, cuda_stream);
}

}  // extern "C"
