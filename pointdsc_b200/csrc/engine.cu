// Host side of the engine: parameter store (state-dict keys), BatchNorm folding, workspace carving,
// stage orchestration for PointDSC.forward in testing mode (reference models/PointDSC.py:128-197),
// and the C ABI declared in include/pointdsc_b200.h.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "../../include/pointdsc_b200.h"
#include "common.cuh"
#include "encoder_tc.h"
#include "kernels.h"

namespace {

thread_local std::string g_last_error;

pdsc_status fail(pdsc_status code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return code;
}

#define PDSC_CUDA(expr)                                                                      \
  do {                                                                                       \
    cudaError_t err__ = (expr);                                                              \
    if (err__ != cudaSuccess)                                                                \
      return fail(PDSC_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(err__), __FILE__, __LINE__); \
  } while (0)

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
    else prev = -1;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

constexpr size_t kGraphRows = 32768;   // B * N up to which the host path replays a captured graph (launch-bound regime)
constexpr double kBnEps = 1e-5;  // torch.nn.BatchNorm1d default (reference PointDSC.py:14, :59)

struct LayerOffsets {  // offsets (in floats) into the device weight arena
  size_t w1, b1, wq, bq, wk, bk, wv, bv, wm0, bm0, wm1, bm1, wm2, bm2;
};

}  // namespace

struct pdsc_engine {
  pdsc_config cfg{};
  bool batch_invariant = false;   // pdsc_set_batch_invariant: the attention's key split is a function of each set's N alone
  std::map<std::string, std::vector<float>> params;
  bool committed = false;
  float sigma = 1.0f;       // learned `sigma`      (PointDSC.py:97)
  float sigma_spat = 0.1f;  // buffer `sigma_spat`  (PointDSC.py:98)
  // device weight arena (fp32, BatchNorm folded)
  float* d_weights = nullptr;
  size_t weights_floats = 0;
  size_t off_l0w = 0, off_l0b = 0;
  std::vector<LayerOffsets> layers;
  size_t off_c0t = 0, off_c0b = 0, off_c2t = 0, off_c2b = 0, off_c4 = 0, off_c4b = 0;
  pdsc::TcWeights tc;  // tensor-core operand images (encoder_tc.cu)
  // engine-owned workspace of the host-input forwards (pdsc_forward_host, pdsc_forward_host_submit)
  void* host_ws = nullptr;
  size_t host_ws_bytes = 0;
  // pdsc_forward_host_submit / _wait: two calls in flight (pdsc_forward_host is one call of the pair).  Each slot owns its
  // device copies of the inputs and outputs and three events; the forwards themselves stay serialised on the caller's stream
  // (one workspace), while the host->device copies of call t + 1 (h2d_stream) and the device->host copies of call t - 1
  // (d2h_stream) run beside the forward of call t.
  struct HostSlot {
    float* io = nullptr;
    size_t io_floats = 0;
    cudaEvent_t keys_ready = nullptr, in_ready = nullptr, fwd_done = nullptr;
    bool busy = false;                   // submitted and not yet waited for
    float *h_trans = nullptr, *h_labels = nullptr;   // where _wait delivers the results ...
    const float *d_trans = nullptr, *d_labels = nullptr;   // ... from
    size_t trans_bytes = 0, labels_bytes = 0;
  } slots[2];
  cudaStream_t h2d_stream = nullptr, d2h_stream = nullptr;
  // live profiling (pdsc_profile_*)
  bool profiling = false;
  bool profile_pending = false;
  std::vector<cudaEvent_t> ev;          // [0..2L) attention pairs, then stage boundary events
  float span_ms[PDSC_SPAN_COUNT] = {};
  int span_launches[PDSC_SPAN_COUNT] = {};
  // pdsc_forward_graph: instantiated CUDA graphs of whole forwards, keyed by shape AND buffer addresses (they are baked
  // into the kernel nodes); a small most-recently-used list
  struct GraphEntry {
    int B, N;
    const void *corr_pos, *src, *tgt, *trans, *labels, *workspace;
    int precision;
    bool batch_invariant;
    cudaGraphExec_t exec;
  };
  std::vector<GraphEntry> graphs;
  cudaStream_t capture_stream = nullptr;   // graphs are captured here (the caller's stream may be the legacy default stream,
                                           // which cannot be captured) and launched into the caller's stream
};

namespace {

using pdsc::CallShape;
using pdsc::kC;

struct Carver {
  char* base;
  size_t off = 0;
  explicit Carver(void* p) : base(static_cast<char*>(p)) {}
  template <typename T>
  T* take(size_t count) {
    off = (off + 255) & ~size_t(255);
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += count * sizeof(T);
    return p;
  }
};

struct Workspace {
  float *sc, *feat_a, *feat_b, *q, *k, *v, *msg, *h1, *h2, *normed, *conf, *key, *seedfeat, *dist, *iterates,
      *seed_trans;
  int32_t *seeds, *knn, *counts;
  uint32_t* conv_mask;
  unsigned long long* best_key;
  pdsc::SetDesc* sets;   // the call's descriptor table
  int32_t* tile_set;     // the set of the first row of every 128-row tile of the call's rows
  void* tc_scratch;
  size_t bytes;
};

// h_offsets: the validated offsets of a packed call, or nullptr for a uniform call of B sets of N rows
CallShape call_shape(const pdsc_engine* e, int B, int N_uniform, const int32_t* h_offsets) {
  return pdsc::plan_call(B, N_uniform, h_offsets, e->cfg.ratio, e->cfg.k, e->cfg.precision != PDSC_FP32_SIMT,
                         e->batch_invariant ? 1 : 0, pdsc::device_sm_count());
}

Workspace carve(const pdsc_engine* e, void* ptr, const CallShape& sh) {
  Workspace w{};
  Carver c(ptr);
  const int B = sh.B;
  const size_t R = sh.R;
  const int T = e->cfg.num_iterations;
  w.sc = c.take<float>(sh.sc_rowmajor > sh.sc_tiled ? sh.sc_rowmajor : sh.sc_tiled);
  w.feat_a = c.take<float>(R * kC);
  w.feat_b = c.take<float>((R + 127) / 128 * 128 * kC);   // tensor-core modes keep feat1 blocked by 128-row tile (tc_chain.cuh)
  w.msg = c.take<float>(R * kC);
  if (e->cfg.precision == PDSC_FP32_SIMT) {
    w.q = c.take<float>(R * kC);
    w.k = c.take<float>(R * kC);
    w.v = c.take<float>(R * kC);
    w.h1 = c.take<float>(R * 64);
    w.h2 = c.take<float>(R * 64);
    w.tc_scratch = nullptr;
  } else {
    w.tc_scratch = c.take<char>(pdsc::tc_scratch(nullptr, sh).bytes);
  }
  w.normed = c.take<float>(R * kC);
  w.conf = c.take<float>(R);
  w.key = c.take<float>(R);
  w.seeds = c.take<int32_t>(sh.seeds + 1);
  w.seedfeat = c.take<float>(sh.seeds * kC + 1);
  w.dist = c.take<float>(sh.dist + 1);
  w.knn = c.take<int32_t>(sh.knn + 1);
  w.iterates = c.take<float>(sh.knn * T + 1);
  w.seed_trans = c.take<float>(sh.seeds * 16 + 16);
  w.counts = c.take<int32_t>(sh.seeds + 1);
  w.conv_mask = c.take<uint32_t>(B);
  w.best_key = c.take<unsigned long long>(B);
  w.sets = c.take<pdsc::SetDesc>(B);
  w.tile_set = c.take<int32_t>((R + 127) / 128);
  w.bytes = (c.off + 255) & ~size_t(255);
  return w;
}

const std::vector<float>* find(const pdsc_engine* e, const std::string& name, size_t count, std::string* missing) {
  auto it = e->params.find(name);
  if (it == e->params.end() || it->second.size() != count) {
    if (missing->empty()) {
      *missing = name + (it == e->params.end() ? " (not set)" : " (wrong element count)");
    }
    return nullptr;
  }
  return &it->second;
}

// conv [Cout,Cin] (+ optional eval BatchNorm `bn`) -> folded weight/bias appended to the arena
bool fold_conv(const pdsc_engine* e, const std::string& conv, const std::string& bn, int cout, int cin,
               std::vector<float>* arena, size_t* off_w, size_t* off_b, std::string* missing) {
  const auto* w = find(e, conv + ".weight", (size_t)cout * cin, missing);
  const auto* b = find(e, conv + ".bias", cout, missing);
  const std::vector<float>*g = nullptr, *beta = nullptr, *mean = nullptr, *var = nullptr;
  if (!bn.empty()) {
    g = find(e, bn + ".weight", cout, missing);
    beta = find(e, bn + ".bias", cout, missing);
    mean = find(e, bn + ".running_mean", cout, missing);
    var = find(e, bn + ".running_var", cout, missing);
  }
  if (!w || !b || (!bn.empty() && (!g || !beta || !mean || !var))) return false;
  *off_w = arena->size();
  arena->resize(arena->size() + (size_t)cout * cin);
  for (int o = 0; o < cout; ++o) {
    const double s = bn.empty() ? 1.0 : (double)(*g)[o] / std::sqrt((double)(*var)[o] + kBnEps);
    for (int c = 0; c < cin; ++c) (*arena)[*off_w + (size_t)o * cin + c] = (float)((double)(*w)[(size_t)o * cin + c] * s);
  }
  while (arena->size() % 4) arena->push_back(0.f);
  *off_b = arena->size();
  arena->resize(arena->size() + cout);
  for (int o = 0; o < cout; ++o) {
    const double s = bn.empty() ? 1.0 : (double)(*g)[o] / std::sqrt((double)(*var)[o] + kBnEps);
    const double sh = bn.empty() ? 0.0 : (double)(*beta)[o] - (double)(*mean)[o] * s;
    (*arena)[*off_b + o] = (float)((double)(*b)[o] * s + sh);
  }
  while (arena->size() % 4) arena->push_back(0.f);
  return true;
}

// Host offsets [n + 1] of a call of n sets packed back to back: n >= 1, offsets[0] = 0, and every set between min_rows and
// max_rows rows.  `what` prefixes "offsets" and "rows" in the message ("source " / "target " for a group of pairs, else "").
pdsc_status check_offsets(const char* who, const char* what, int32_t n, const int32_t* h_offsets, int min_rows,
                          int max_rows = INT_MAX) {
  if (n < 1) return fail(PDSC_ERR_SHAPE, "%s: need at least one set (got %d)", who, n);
  if (!h_offsets) return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: null host offsets", who);
  if (h_offsets[0] != 0) return fail(PDSC_ERR_SHAPE, "%s: %soffsets[0] must be 0 (got %d)", who, what, h_offsets[0]);
  for (int b = 0; b < n; ++b) {
    const long long rows = (long long)h_offsets[b + 1] - h_offsets[b];
    if (rows < min_rows)
      return fail(PDSC_ERR_SHAPE, "%s: set %d has %lld %srows: offsets must increase by at least %d per set", who, b, rows, what,
                  min_rows);
    if (rows > max_rows)
      return fail(PDSC_ERR_SHAPE, "%s: set %d has %lld %srows, above the supported maximum %d", who, b, rows, what, max_rows);
  }
  return PDSC_OK;
}

// A caller's workspace or scratch buffer: at least `need` bytes at an `align`-byte boundary.
pdsc_status check_scratch(const char* who, const char* noun, const void* ptr, size_t bytes, size_t need, size_t align) {
  if (!ptr || bytes < need || reinterpret_cast<uintptr_t>(ptr) % align)
    return fail(PDSC_ERR_WORKSPACE, "%s: %s too small or not %zu-byte aligned (%zu bytes given, %zu needed)", who, noun, align,
                bytes, need);
  return PDSC_OK;
}

void copy_tap(void* dst, const void* src, size_t bytes, cudaStream_t st) {
  if (dst && bytes) cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st);
}

float refinement_threshold(double ctor_threshold) {
  // `if self.inlier_threshold == 0.10` (PointDSC.py:415): Python compares the ctor double with 0.10, exactly
  return ctor_threshold == 0.10 ? 0.10f : 1.2f;
}

int encoder_simt(const pdsc_engine* e, const Workspace& w, const CallShape& sh, const float* corr_pos, const pdsc_stage_io* io,
                 cudaEvent_t* attn_events, cudaStream_t st) {
  using namespace pdsc;
  const long long R = (long long)sh.R;
  const float* W = e->d_weights;
  launch_layer0(corr_pos, W + e->off_l0w, W + e->off_l0b, w.feat_a, R, e->cfg.in_dim, st);
  auto lin = [&](const float* A, int K, size_t ow, size_t ob, const float* res, float* out, int Nout, int relu) {
    LinearArgs a{};
    a.A = A; a.strideA = 0; a.lda = K;
    a.W = W + ow; a.strideW = 0; a.ldw = K;
    a.bias = W + ob; a.res = res; a.ldres = Nout;
    a.out = out; a.strideO = 0; a.ldo = Nout;
    a.M = (int)R; a.K = K; a.Nout = Nout; a.relu = relu; a.epi = 0; a.batch = 1;
    launch_linear_simt(a, st);
  };
  for (int l = 0; l < e->cfg.num_layers; ++l) {
    const LayerOffsets& L = e->layers[l];
    lin(w.feat_a, kC, L.w1, L.b1, nullptr, w.feat_b, kC, 1);            // PointCN: conv + BN + ReLU
    lin(w.feat_b, kC, L.wq, L.bq, nullptr, w.q, kC, 0);
    lin(w.feat_b, kC, L.wk, L.bk, nullptr, w.k, kC, 0);
    lin(w.feat_b, kC, L.wv, L.bv, nullptr, w.v, kC, 0);
    if (attn_events) cudaEventRecord(attn_events[2 * l], st);
    launch_attention_simt(w.q, w.k, w.v, w.sc, w.msg, sh.B, sh.N, st, w.sets);
    if (attn_events) cudaEventRecord(attn_events[2 * l + 1], st);
    if (io && io->out_layer_debug && io->layer_tap == l) {
      const size_t plane = (size_t)R * kC;
      const float* srcs[5] = {w.feat_b, w.q, w.k, w.v, w.msg};
      for (int i = 0; i < 5; ++i) copy_tap(io->out_layer_debug + i * plane, srcs[i], plane * sizeof(float), st);
    }
    lin(w.msg, kC, L.wm0, L.bm0, nullptr, w.h1, 64, 1);                  // fc_message.0-2
    lin(w.h1, 64, L.wm1, L.bm1, nullptr, w.h2, 64, 1);                   // fc_message.3-5
    lin(w.h2, 64, L.wm2, L.bm2, w.feat_b, w.feat_a, kC, 0);              // fc_message.6 + residual
    if (io && io->out_layer_features && io->layer_tap == l)
      copy_tap(io->out_layer_features, w.feat_a, (size_t)R * kC * sizeof(float), st);
  }
  return PDSC_OK;
}

// Descriptor table of a call, from the device copy of a packed call's offsets, or (offsets == nullptr) for B sets of N_uniform
// rows: one warp walks the sets 32 at a time and forms every running offset (tiles, seeds, attention items, SC / distance /
// neighbour blocks) by warp-wide inclusive scans, and records the set of the first row of every 128-row tile (tc_chain.cuh).  A
// uniform call therefore needs no host-to-device copy.
__device__ __forceinline__ long long warp_scan_incl(long long v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  return v;
}

__global__ void set_table_kernel(const int32_t* __restrict__ offsets, int N_uniform, int B, double ratio, int k_cfg, int tiled,
                                 int split, int invariant, int num_sms, pdsc::SetDesc* __restrict__ table,
                                 int32_t* __restrict__ tile_set) {
  const int lane = threadIdx.x;
  long long base[7] = {0, 0, 0, 0, 0, 0, 0};   // qt0, kt0, seed0, item0, sc0, dist0, knn0
  for (int b0 = 0; b0 < B; b0 += 32) {
    const int b = b0 + lane;
    const bool live = b < B;
    int row0 = 0, N = 0;
    if (live) {
      row0 = offsets ? offsets[b] : b * N_uniform;
      N = offsets ? offsets[b + 1] - row0 : N_uniform;
    }
    const pdsc::SetSizes z = pdsc::set_sizes(N, ratio, k_cfg);   // the plan's rule (plan_call); N = 0 past the last set
    int sp = 1, TS = z.KT;
    if (split) pdsc::attn_key_split(N, invariant, num_sms, &sp, &TS);
    const long long size[7] = {z.QT, z.KT, z.S, (long long)z.QT * sp, tiled ? z.sc_tiled : z.sc_rowmajor, z.dist, z.knn};
    long long first[7];
#pragma unroll
    for (int i = 0; i < 7; ++i) {
      const long long incl = warp_scan_incl(size[i], lane);
      first[i] = base[i] + incl - size[i];
      base[i] += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (live) {
      pdsc::SetDesc d;
      d.row0 = row0; d.N = N; d.S = z.S; d.k = z.k;
      d.qt0 = (int)first[0]; d.kt0 = (int)first[1]; d.seed0 = (int)first[2]; d.item0 = (int)first[3];
      d.sp = sp; d.TS = TS; d.pad0 = d.pad1 = 0;
      d.sc0 = first[4]; d.dist0 = first[5]; d.knn0 = first[6];
      table[b] = d;
      for (long long t = (row0 + 127) / 128; t * 128 < (long long)row0 + N; ++t) tile_set[t] = b;
    }
  }
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

const char* pdsc_last_error(void) { return g_last_error.c_str(); }
const char* pdsc_version(void) { return "pointdsc_b200 0.1 (sm_90a)"; }

int pdsc_create(const pdsc_config* cfg, pdsc_engine** out) {
  if (!cfg || !out) return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_create: null argument");
  if (cfg->num_channels != kC) return fail(PDSC_ERR_UNSUPPORTED, "num_channels must be %d, got %d", kC, cfg->num_channels);
  if (cfg->in_dim < 1 || cfg->in_dim > 64) return fail(PDSC_ERR_UNSUPPORTED, "in_dim %d out of range", cfg->in_dim);
  if (cfg->num_layers < 1 || cfg->num_layers > 64) return fail(PDSC_ERR_UNSUPPORTED, "num_layers %d out of range", cfg->num_layers);
  if (cfg->num_iterations < 1 || cfg->num_iterations > pdsc::kMaxIters)
    return fail(PDSC_ERR_UNSUPPORTED, "num_iterations must be in [1,%d]", pdsc::kMaxIters);
  if (cfg->k < 1 || cfg->k > pdsc::kMaxK) return fail(PDSC_ERR_UNSUPPORTED, "k must be in [1,%d]", pdsc::kMaxK);
  if (!std::isfinite(cfg->ratio)) return fail(PDSC_ERR_INVALID_ARGUMENT, "ratio must be finite, got %g", cfg->ratio);
  if (cfg->precision < PDSC_FP32_SIMT || cfg->precision > PDSC_FP16X3)
    return fail(PDSC_ERR_INVALID_ARGUMENT, "unknown precision %d", cfg->precision);
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(PDSC_ERR_CUDA, "no CUDA device: this engine has no CPU path");
  if (cfg->device < 0 || cfg->device >= ndev) return fail(PDSC_ERR_INVALID_ARGUMENT, "device %d out of range", cfg->device);
  cudaDeviceProp prop{};
  PDSC_CUDA(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(PDSC_ERR_UNSUPPORTED, "device %d is sm_%d%d; this library holds only sm_90a code", cfg->device,
                prop.major, prop.minor);
  pdsc_engine* e = new pdsc_engine();
  e->cfg = *cfg;
  e->sigma_spat = cfg->sigma_d;
  *out = e;
  return PDSC_OK;
}

int pdsc_destroy(pdsc_engine* e) {
  if (!e) return PDSC_OK;
  DeviceGuard g(e->cfg.device);
  cudaFree(e->d_weights);
  pdsc::tc_free_weights(&e->tc);
  cudaFree(e->host_ws);
  for (auto& sl : e->slots) {
    if (sl.busy && sl.fwd_done) cudaEventSynchronize(sl.fwd_done);
    cudaFree(sl.io);
    if (sl.keys_ready) cudaEventDestroy(sl.keys_ready);
    if (sl.in_ready) cudaEventDestroy(sl.in_ready);
    if (sl.fwd_done) cudaEventDestroy(sl.fwd_done);
  }
  if (e->h2d_stream) cudaStreamDestroy(e->h2d_stream);
  if (e->d2h_stream) cudaStreamDestroy(e->d2h_stream);
  for (auto& ev : e->ev) cudaEventDestroy(ev);
  for (auto& g : e->graphs) cudaGraphExecDestroy(g.exec);
  if (e->capture_stream) cudaStreamDestroy(e->capture_stream);
  delete e;
  return PDSC_OK;
}

int pdsc_set_param(pdsc_engine* e, const char* name, const float* h_data, int64_t count) {
  if (!e || !name || (!h_data && count > 0) || count < 0) return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_set_param: bad argument");
  e->params[name].assign(h_data, h_data + count);
  e->committed = false;
  return PDSC_OK;
}

int pdsc_set_precision(pdsc_engine* e, int32_t precision) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (precision < PDSC_FP32_SIMT || precision > PDSC_FP16X3) return fail(PDSC_ERR_INVALID_ARGUMENT, "unknown precision %d", precision);
  e->cfg.precision = precision;
  return PDSC_OK;
}

int pdsc_set_batch_invariant(pdsc_engine* e, int32_t enable) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  e->batch_invariant = enable != 0;
  return PDSC_OK;
}

int pdsc_commit_params(pdsc_engine* e) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  DeviceGuard g(e->cfg.device);
  std::string missing;
  std::vector<float> arena;
  arena.reserve(1 << 21);
  const int L = e->cfg.num_layers;
  e->layers.assign(L, LayerOffsets{});
  bool ok = fold_conv(e, "encoder.layer0", "", kC, e->cfg.in_dim, &arena, &e->off_l0w, &e->off_l0b, &missing);
  for (int l = 0; l < L; ++l) {
    const std::string pc = "encoder.blocks.PointCN_layer_" + std::to_string(l);
    const std::string nl = "encoder.blocks.NonLocal_layer_" + std::to_string(l);
    LayerOffsets& o = e->layers[l];
    ok &= fold_conv(e, pc + ".0", pc + ".1", kC, kC, &arena, &o.w1, &o.b1, &missing);
    ok &= fold_conv(e, nl + ".projection_q", "", kC, kC, &arena, &o.wq, &o.bq, &missing);
    ok &= fold_conv(e, nl + ".projection_k", "", kC, kC, &arena, &o.wk, &o.bk, &missing);
    ok &= fold_conv(e, nl + ".projection_v", "", kC, kC, &arena, &o.wv, &o.bv, &missing);
    ok &= fold_conv(e, nl + ".fc_message.0", nl + ".fc_message.1", 64, kC, &arena, &o.wm0, &o.bm0, &missing);
    ok &= fold_conv(e, nl + ".fc_message.3", nl + ".fc_message.4", 64, 64, &arena, &o.wm1, &o.bm1, &missing);
    ok &= fold_conv(e, nl + ".fc_message.6", "", kC, 64, &arena, &o.wm2, &o.bm2, &missing);
  }
  // classification head, first two layers stored transposed ([in][out]) for the warp-per-point kernel
  size_t c0w, c0b, c2w, c2b, c4w, c4b;
  ok &= fold_conv(e, "classification.0", "", 32, kC, &arena, &c0w, &c0b, &missing);
  ok &= fold_conv(e, "classification.2", "", 32, 32, &arena, &c2w, &c2b, &missing);
  ok &= fold_conv(e, "classification.4", "", 1, 32, &arena, &c4w, &c4b, &missing);
  if (!ok) return fail(PDSC_ERR_UNKNOWN_PARAM, "pdsc_commit_params: state-dict entry missing or mis-sized: %s", missing.c_str());
  e->off_c0t = arena.size();
  arena.resize(arena.size() + (size_t)kC * 32);
  for (int c = 0; c < kC; ++c)
    for (int o = 0; o < 32; ++o) arena[e->off_c0t + (size_t)c * 32 + o] = arena[c0w + (size_t)o * kC + c];
  e->off_c2t = arena.size();
  arena.resize(arena.size() + 32 * 32);
  for (int c = 0; c < 32; ++c)
    for (int o = 0; o < 32; ++o) arena[e->off_c2t + (size_t)c * 32 + o] = arena[c2w + (size_t)o * 32 + c];
  e->off_c0b = c0b; e->off_c2b = c2b; e->off_c4 = c4w; e->off_c4b = c4b;

  auto s1 = e->params.find("sigma");
  if (s1 != e->params.end() && s1->second.size() == 1) e->sigma = s1->second[0];
  auto s2 = e->params.find("sigma_spat");
  if (s2 != e->params.end() && s2->second.size() == 1) e->sigma_spat = s2->second[0];

  for (auto& gq : e->graphs) cudaGraphExecDestroy(gq.exec);   // captured graphs hold the old weight pointers
  e->graphs.clear();
  cudaFree(e->d_weights);
  e->d_weights = nullptr;
  PDSC_CUDA(cudaMalloc(&e->d_weights, arena.size() * sizeof(float)));
  PDSC_CUDA(cudaMemcpy(e->d_weights, arena.data(), arena.size() * sizeof(float), cudaMemcpyHostToDevice));
  e->weights_floats = arena.size();

  // tensor-core operand images of the same folded weights
  std::vector<pdsc::TcLayerHost> tl(L);
  for (int l = 0; l < L; ++l) {
    const LayerOffsets& o = e->layers[l];
    tl[l] = pdsc::TcLayerHost{arena.data() + o.w1, arena.data() + o.b1, arena.data() + o.wq, arena.data() + o.bq,
                              arena.data() + o.wk, arena.data() + o.bk, arena.data() + o.wv, arena.data() + o.bv,
                              arena.data() + o.wm0, arena.data() + o.bm0, arena.data() + o.wm1, arena.data() + o.bm1,
                              arena.data() + o.wm2, arena.data() + o.bm2};
  }
  const int rc = pdsc::tc_build_weights(tl.data(), L, &e->tc);
  if (rc != 0) return fail(PDSC_ERR_CUDA, "building tensor-core weight images failed: %s", cudaGetErrorString((cudaError_t)rc));
  e->committed = true;
  return PDSC_OK;
}

int32_t pdsc_num_seeds(const pdsc_engine* e, int32_t N) {
  if (!e || N < 0) return 0;
  // the length of argsort(...)[:, 0:int(num_corr * self.ratio)] (PointDSC.py:174, :217)
  return pdsc::num_seeds(N, e->cfg.ratio);
}
int32_t pdsc_num_neighbours(const pdsc_engine* e, int32_t N) {
  if (!e) return 0;
  return pdsc::set_sizes(N, e->cfg.ratio, e->cfg.k).k;
}

size_t pdsc_workspace_bytes(const pdsc_engine* e, int32_t B, int32_t N) {
  if (!e || B <= 0 || N <= 0) return 0;
  DeviceGuard g(e->cfg.device);
  return carve(e, nullptr, call_shape(e, B, N, nullptr)).bytes;
}

int32_t pdsc_launches_per_forward(const pdsc_engine* e, int32_t B, int32_t N) {
  if (!e || B <= 0 || N <= 0) return 0;
  DeviceGuard g(e->cfg.device);
  const int L = e->cfg.num_layers;
  const int enc = (e->cfg.precision == PDSC_FP32_SIMT) ? (1 + 8 * L) : pdsc::tc_launches(L, call_shape(e, B, N, nullptr).attn_split);
  // set table, sc, encoder, head, nms, sort, (gather +) dist gemm, knn select, 2 fills, nsm, hypotheses, refine
  return 2 + enc + 1 + 2 + ((e->cfg.precision == PDSC_FP32_SIMT) ? 3 : 2) + 2 + 3;
}

// what forward_impl refuses of the engine and the call's shape (a packed call's offsets are checked by its entry point)
static int check_forward(const pdsc_engine* e, int32_t B, int32_t N, const int32_t* h_offsets) {
  if (!e->committed) return fail(PDSC_ERR_NOT_COMMITTED, "pdsc_commit_params() has not been called since the last pdsc_set_param()");
  if (!h_offsets) {
    if (B <= 0 || N <= 1) return fail(PDSC_ERR_SHAPE, "need B >= 1 and N >= 2 (got B=%d N=%d)", B, N);
    const int max_n = pdsc::pick_seeds_max_n();
    if (N > max_n) return fail(PDSC_ERR_UNSUPPORTED, "N=%d exceeds the supported maximum %d", N, max_n);
  }
  return PDSC_OK;
}

// mode 0: testing (PointDSC.py: NMS seeds, per-set early exit, labels = inlier mask, post-refinement)
// mode 1: non-testing / validation (PointDSC.py:158-165, :176, :190-191): seeds = top-S by confidence, batch-global early
//         exit, no refinement, final_labels = confidence logits, optional feature-similarity matrix M [B,N,N]
// h_offsets / d_offsets: a packed call (mode 0, no io), offsets validated by pdsc_forward_packed; N is then ignored
// corr_ready: if not null, the stream waits for it right behind the SC kernel, which reads only the key points, and before
//             the first reader of corr_pos (the host-input path copies corr_pos meanwhile)
static int forward_impl(pdsc_engine* e, int mode, int32_t B, int32_t N, const int32_t* h_offsets, const int32_t* d_offsets,
                        const float* d_corr_pos, const float* d_src,
                        const float* d_tgt, float* d_final_trans, float* d_final_labels, float* d_M, const pdsc_stage_io* io,
                        void* d_workspace, size_t workspace_bytes, void* cuda_stream, cudaEvent_t corr_ready = nullptr) {
  using namespace pdsc;
  const int mask_stride = mode == 0 ? 1 : 0;
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (int rc = check_forward(e, B, N, h_offsets)) return rc;
  if (!d_src || !d_tgt || !d_final_trans || !d_final_labels) return fail(PDSC_ERR_INVALID_ARGUMENT, "null tensor pointer");
  const bool inject_feat = io && io->in_features;
  if (!inject_feat && !d_corr_pos) return fail(PDSC_ERR_INVALID_ARGUMENT, "corr_pos is null");
  if (io && io->in_confidence && !inject_feat) return fail(PDSC_ERR_INVALID_ARGUMENT, "in_confidence requires in_features");
  DeviceGuard g(e->cfg.device);   // the plan reads the SM count of the engine's device
  const CallShape sh = call_shape(e, B, N, h_offsets);
  if (int rc = check_scratch("pdsc_forward", "workspace", d_workspace, workspace_bytes, carve(e, nullptr, sh).bytes, 256))
    return rc;
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  const Workspace w = carve(e, d_workspace, sh);
  N = sh.N;                        // a packed call: the largest set, which sizes the launches
  const size_t R = sh.R;
  const int S = sh.S, k = sh.k, T = e->cfg.num_iterations;
  const SetDesc* sets = w.sets;
  set_table_kernel<<<1, 32, 0, st>>>(d_offsets, N, B, e->cfg.ratio, e->cfg.k, e->cfg.precision == PDSC_FP32_SIMT ? 0 : 1,
                                     sh.attn_split, sh.attn_invariant, sh.num_sms, w.sets, w.tile_set);
  const float* W = e->d_weights;
  const int L = e->cfg.num_layers;
  cudaEvent_t* attn_ev = nullptr;
  cudaEvent_t* bev = nullptr;  // boundary events: 0 start, 1 sc, 2 encoder, 3 head, 4 seeds, 5 knn, 6 nsm, 7 hyp, 8 end
  if (e->profiling) {
    if (e->profile_pending) pdsc_profile_read(e, nullptr, nullptr);  // fold the previous forward before reusing events
    attn_ev = inject_feat ? nullptr : e->ev.data();
    bev = e->ev.data() + 2 * L;
    cudaEventRecord(bev[0], st);
  }
  auto mark = [&](int i) { if (bev) cudaEventRecord(bev[i], st); };

  // ---- stages i + ii ------------------------------------------------------------------------------
  if (!inject_feat) {
    const bool simt = e->cfg.precision == PDSC_FP32_SIMT;
    if (simt) launch_sc_matrix(d_src, d_tgt, w.sc, B, N, e->sigma_spat, st, sets);
    else launch_sc_matrix_tiled(d_src, d_tgt, w.sc, B, N, e->sigma_spat, st, sets);
    mark(1);
    if (corr_ready) PDSC_CUDA(cudaStreamWaitEvent(st, corr_ready, 0));
    if (io && io->out_sc) {
      if (simt)
        cudaMemcpy2DAsync(io->out_sc, (size_t)N * sizeof(float), w.sc, (size_t)set_sizes(N, e->cfg.ratio, e->cfg.k).NS * sizeof(float),
                          (size_t)N * sizeof(float), R, cudaMemcpyDeviceToDevice, st);
      else
        launch_sc_untile(w.sc, io->out_sc, B, N, st);
    }
    if (simt) {
      const int rc = encoder_simt(e, w, sh, d_corr_pos, io, attn_ev, st);
      if (rc) return rc;
    } else {
      TcForwardArgs a{sh};
      a.in_dim = e->cfg.in_dim; a.num_layers = e->cfg.num_layers;
      a.split = (e->cfg.precision == PDSC_BF16X3 || e->cfg.precision == PDSC_FP16X3) ? 1 : 0;
      a.fmt = (e->cfg.precision == PDSC_FP16X3) ? 0 : 1;
      a.corr_pos = d_corr_pos; a.l0w = W + e->off_l0w; a.l0b = W + e->off_l0b;
      a.sc = w.sc; a.feat = w.feat_a; a.feat1 = w.feat_b; a.msg = w.msg; a.scratch = w.tc_scratch;
      a.layer_tap = (io && io->out_layer_features) ? io->layer_tap : -1;
      a.layer_tap_out = io ? io->out_layer_features : nullptr;
      a.debug_layer = io ? io->layer_tap : -1;
      a.debug_out = io ? io->out_layer_debug : nullptr;
      a.attn_events = attn_ev;
      a.sets = sets; a.tile_set = w.tile_set;
      const int rc = tc_encoder_forward(e->tc, a, st);
      if (rc) return fail(PDSC_ERR_CUDA, "tensor-core encoder launch failed: %s", cudaGetErrorString((cudaError_t)rc));
    }
  } else {
    PDSC_CUDA(cudaMemcpyAsync(w.feat_a, io->in_features, R * kC * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  if (inject_feat) mark(1);
  mark(2);
  if (io) copy_tap(io->out_features, w.feat_a, R * kC * sizeof(float), st);

  // ---- a4 + a5 ------------------------------------------------------------------------------------
  HeadWeights hw{W + e->off_c0t, W + e->off_c0b, W + e->off_c2t, W + e->off_c2b, W + e->off_c4, W + e->off_c4b};
  const bool inject_conf = io && io->in_confidence;
  launch_head(w.feat_a, hw, w.normed, w.conf, (long long)R, inject_conf ? 0 : 1, st);
  if (inject_conf) PDSC_CUDA(cudaMemcpyAsync(w.conf, io->in_confidence, R * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (io) {
    copy_tap(io->out_normed, w.normed, R * kC * sizeof(float), st);
    copy_tap(io->out_confidence, w.conf, R * sizeof(float), st);
  }

  mark(3);
  // ---- a6 -----------------------------------------------------------------------------------------
  if (S > 0) {
    if (io && io->in_seeds)
      PDSC_CUDA(cudaMemcpyAsync(w.seeds, io->in_seeds, (size_t)B * S * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    else if (mode == 0)
      launch_pick_seeds(d_src, w.conf, w.seeds, w.key, B, N, S, e->cfg.nms_radius, st, sets);
    else
      launch_top_seeds(w.conf, w.seeds, B, N, S, st, sets);
    if (io) copy_tap(io->out_seeds, w.seeds, (size_t)B * S * sizeof(int32_t), st);
    mark(4);

    // ---- a7 ---------------------------------------------------------------------------------------
    if (io && io->in_knn_idx) {
      PDSC_CUDA(cudaMemcpyAsync(w.knn, io->in_knn_idx, (size_t)B * S * k * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    } else {
      if (e->cfg.precision == PDSC_FP32_SIMT) {
        launch_gather_rows(w.normed, w.seeds, w.seedfeat, B, N, S, st, sets);
        LinearArgs a{};   // epi 1: every set's operands and distance block come from the table
        a.A = w.seedfeat; a.lda = kC;
        a.W = w.normed; a.ldw = kC;
        a.out = w.dist; a.ldo = N;
        a.M = S; a.K = kC; a.Nout = N; a.relu = 0; a.epi = 1; a.batch = B;
        a.sets = sets;
        launch_linear_simt(a, st);
      } else {
        launch_knn_dist_tc(w.normed, w.seeds, w.dist, B, N, S, st, sets);
      }
      launch_knn_select(w.dist, w.knn, B, N, S, k, st, sets, (int)sh.seeds);
    }
    if (io) copy_tap(io->out_knn_idx, w.knn, (size_t)B * S * k * sizeof(int32_t), st);
    mark(5);

    // ---- a8 + a9 ----------------------------------------------------------------------------------
    launch_fill_u32(w.conv_mask, 0xFFFFFFFFu, B, st);
    launch_fill_u64(w.best_key, 0ull, B, st);
    launch_nsm_power(w.normed, d_src, d_tgt, w.knn, w.iterates, w.conv_mask, io ? io->out_compat : nullptr, B, N, S, k, T,
                     e->sigma, e->sigma_spat, mask_stride, e->cfg.precision != PDSC_FP32_SIMT, st, sets, sh.k_min);
    mark(6);
    // ---- a10 + a11 --------------------------------------------------------------------------------
    launch_seed_hypotheses(d_src, d_tgt, w.knn, w.iterates, w.conv_mask, io ? io->in_seed_trans : nullptr, w.seed_trans,
                           w.counts, w.best_key, io ? io->out_eig : nullptr, io ? io->out_power_iters : nullptr, B, N, S,
                           k, T, (float)e->cfg.inlier_threshold, mask_stride, st, sets);
    if (io) {
      copy_tap(io->out_seed_trans, w.seed_trans, (size_t)B * S * 16 * sizeof(float), st);
      copy_tap(io->out_inlier_counts, w.counts, (size_t)B * S * sizeof(int32_t), st);
    }
    mark(7);
  } else {
    launch_fill_u64(w.best_key, 0ull, B, st);
    // no seeds: no power iteration runs, and the tap says so (it would otherwise keep whatever the caller's buffer held)
    if (io && io->out_power_iters) PDSC_CUDA(cudaMemsetAsync(io->out_power_iters, 0, (size_t)B * sizeof(int32_t), st));
    mark(4); mark(5); mark(6); mark(7);
  }
  // ---- a11 (labels) + a12 ---------------------------------------------------------------------------
  launch_select_refine(d_src, d_tgt, w.seed_trans, w.best_key, d_final_trans, mode == 0 ? d_final_labels : nullptr,
                       io ? io->out_init_trans : nullptr, io ? io->out_best : nullptr,
                       io ? io->out_refine_solves : nullptr, B, N, S, (float)e->cfg.inlier_threshold,
                       refinement_threshold(e->cfg.inlier_threshold), mode == 0 ? 20 : 0, st, sets);
  if (mode == 1) {
    PDSC_CUDA(cudaMemcpyAsync(d_final_labels, w.conf, R * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (d_M) {   // M = clamp(1 - (1 - F F^T) / sigma^2, 0, 1), zero diagonal  (PointDSC.py:160-165)
      LinearArgs a{};
      a.A = w.normed; a.strideA = (long long)N * kC; a.lda = kC;
      a.W = w.normed; a.strideW = (long long)N * kC; a.ldw = kC;
      a.bias = nullptr; a.res = nullptr; a.ldres = 0;
      a.out = d_M; a.strideO = (long long)N * N; a.ldo = N;
      a.M = N; a.K = kC; a.Nout = N; a.relu = 0; a.epi = 2; a.batch = B;
      a.epi_param = e->sigma * e->sigma;
      launch_linear_simt(a, st);
    }
  }
  mark(8);
  if (bev) {
    e->profile_pending = true;
    e->span_launches[PDSC_SPAN_ATTENTION] += inject_feat ? 0 : L;
    e->span_launches[PDSC_SPAN_TOTAL] += 1;
  }
  PDSC_CUDA(cudaGetLastError());
  return PDSC_OK;
}

int pdsc_forward(pdsc_engine* e, int32_t B, int32_t N, const float* d_corr_pos, const float* d_src, const float* d_tgt,
                 float* d_final_trans, float* d_final_labels, const pdsc_stage_io* io, void* d_workspace,
                 size_t workspace_bytes, void* cuda_stream) {
  return forward_impl(e, 0, B, N, nullptr, nullptr, d_corr_pos, d_src, d_tgt, d_final_trans, d_final_labels, nullptr, io, d_workspace,
                      workspace_bytes, cuda_stream);
}

size_t pdsc_workspace_bytes_packed(const pdsc_engine* e, int32_t B, const int32_t* h_offsets) {
  if (!e || check_offsets("pdsc_workspace_bytes_packed", "", B, h_offsets, 2, pdsc::pick_seeds_max_n())) return 0;
  DeviceGuard g(e->cfg.device);
  return carve(e, nullptr, call_shape(e, B, 0, h_offsets)).bytes;
}

int pdsc_forward_packed(pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets, const float* d_corr_pos,
                        const float* d_src, const float* d_tgt, float* d_final_trans, float* d_final_labels, void* d_workspace,
                        size_t workspace_bytes, void* cuda_stream) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (int rc = check_offsets("pdsc_forward_packed", "", B, h_offsets, 2, pdsc::pick_seeds_max_n())) return rc;
  if (!d_offsets || !d_corr_pos) return fail(PDSC_ERR_INVALID_ARGUMENT, "null tensor pointer");
  return forward_impl(e, 0, B, 0, h_offsets, d_offsets, d_corr_pos, d_src, d_tgt, d_final_trans, d_final_labels, nullptr, nullptr,
                      d_workspace, workspace_bytes, cuda_stream);
}

int pdsc_forward_graph(pdsc_engine* e, int32_t B, int32_t N, const float* d_corr_pos, const float* d_src, const float* d_tgt,
                       float* d_final_trans, float* d_final_labels, void* d_workspace, size_t workspace_bytes,
                       void* cuda_stream) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  DeviceGuard g(e->cfg.device);
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  PDSC_CUDA(cudaStreamIsCapturing(st, &cap));
  if (cap != cudaStreamCaptureStatusNone || e->profiling || !e->committed)   // already inside someone's capture (or nothing to cache): plain enqueue
    return forward_impl(e, 0, B, N, nullptr, nullptr, d_corr_pos, d_src, d_tgt, d_final_trans, d_final_labels, nullptr, nullptr, d_workspace,
                        workspace_bytes, cuda_stream);
  for (size_t i = 0; i < e->graphs.size(); ++i) {
    const auto& q = e->graphs[i];
    if (q.B == B && q.N == N && q.corr_pos == d_corr_pos && q.src == d_src && q.tgt == d_tgt && q.trans == d_final_trans &&
        q.labels == d_final_labels && q.workspace == d_workspace && q.precision == e->cfg.precision &&
        q.batch_invariant == e->batch_invariant) {
      if (i) std::swap(e->graphs[0], e->graphs[i]);
      PDSC_CUDA(cudaGraphLaunch(e->graphs[0].exec, st));
      return PDSC_OK;
    }
  }
  // first call with these buffers: run once eagerly (per-device opt-ins, lazy module loading), then capture
  int rc = forward_impl(e, 0, B, N, nullptr, nullptr, d_corr_pos, d_src, d_tgt, d_final_trans, d_final_labels, nullptr, nullptr, d_workspace,
                        workspace_bytes, cuda_stream);
  if (rc) return rc;
  if (!e->capture_stream) PDSC_CUDA(cudaStreamCreateWithFlags(&e->capture_stream, cudaStreamNonBlocking));
  PDSC_CUDA(cudaStreamBeginCapture(e->capture_stream, cudaStreamCaptureModeThreadLocal));
  rc = forward_impl(e, 0, B, N, nullptr, nullptr, d_corr_pos, d_src, d_tgt, d_final_trans, d_final_labels, nullptr, nullptr, d_workspace,
                    workspace_bytes, e->capture_stream);
  cudaGraph_t graph = nullptr;
  const cudaError_t end = cudaStreamEndCapture(e->capture_stream, &graph);
  if (rc) {
    if (graph) cudaGraphDestroy(graph);
    return rc;
  }
  if (end != cudaSuccess) return fail(PDSC_ERR_CUDA, "cudaStreamEndCapture failed: %s", cudaGetErrorString(end));
  cudaGraphExec_t exec = nullptr;
  const cudaError_t inst = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  if (inst != cudaSuccess) return fail(PDSC_ERR_CUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(inst));
  if (e->graphs.size() >= 8) {
    cudaGraphExecDestroy(e->graphs.back().exec);
    e->graphs.pop_back();
  }
  e->graphs.insert(e->graphs.begin(), pdsc_engine::GraphEntry{B, N, d_corr_pos, d_src, d_tgt, d_final_trans, d_final_labels,
                                                              d_workspace, e->cfg.precision, e->batch_invariant, exec});
  return PDSC_OK;   // the eager run above already produced this call's result
}

int pdsc_forward_eval(pdsc_engine* e, int32_t B, int32_t N, const float* d_corr_pos, const float* d_src, const float* d_tgt,
                      float* d_final_trans, float* d_confidence, float* d_M, const pdsc_stage_io* io, void* d_workspace,
                      size_t workspace_bytes, void* cuda_stream) {
  return forward_impl(e, 1, B, N, nullptr, nullptr, d_corr_pos, d_src, d_tgt, d_final_trans, d_confidence, d_M, io, d_workspace,
                      workspace_bytes, cuda_stream);
}

static int eval_stats_impl(pdsc_engine* e, int32_t B, const int32_t* d_offsets, int32_t N, const float* d_pred_trans,
                           const float* d_gt_trans, const float* d_src, const float* d_tgt, const float* d_pred_labels,
                           const float* d_gt_labels, float re_thre, float te_thre, float* d_stats, void* cuda_stream) {
  if (!d_pred_trans || !d_gt_trans || !d_src || !d_tgt || !d_pred_labels || !d_gt_labels || !d_stats)
    return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_eval_stats: null tensor pointer");
  DeviceGuard g(e->cfg.device);
  pdsc::launch_eval_stats(d_pred_trans, d_gt_trans, d_src, d_tgt, d_pred_labels, d_gt_labels, d_stats, B, d_offsets, N, re_thre,
                          te_thre, static_cast<cudaStream_t>(cuda_stream));
  PDSC_CUDA(cudaGetLastError());
  return PDSC_OK;
}

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

size_t pdsc_leading_eigenvector_scratch_bytes(int32_t B, int32_t N) {
  return (B > 0 && N > 0) ? pdsc::eig_scratch_bytes(B, N) : 0;
}

int pdsc_leading_eigenvector(pdsc_engine* e, int32_t B, int32_t N, const float* d_M, int32_t num_iterations, int32_t early_exit,
                             float* d_eigenvector, int32_t* d_iterations_run, void* d_scratch, size_t scratch_bytes,
                             void* cuda_stream) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (B <= 0 || N <= 0) return fail(PDSC_ERR_SHAPE, "need B >= 1 and N >= 1 (got B=%d N=%d)", B, N);
  if (num_iterations < 1 || num_iterations > 1000) return fail(PDSC_ERR_INVALID_ARGUMENT, "num_iterations %d out of range", num_iterations);
  if (N > 24576) return fail(PDSC_ERR_UNSUPPORTED, "N=%d exceeds the supported maximum 24576", N);
  if (!d_M || !d_eigenvector || !d_iterations_run) return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_leading_eigenvector: null tensor pointer");
  if (int rc = check_scratch("pdsc_leading_eigenvector", "scratch", d_scratch, scratch_bytes, pdsc::eig_scratch_bytes(B, N), 16))
    return rc;
  DeviceGuard g(e->cfg.device);
  const int rc = pdsc::launch_leading_eigenvector(d_M, d_eigenvector, d_iterations_run, B, N, num_iterations, early_exit, d_scratch,
                                                  static_cast<cudaStream_t>(cuda_stream));
  if (rc) return fail(PDSC_ERR_CUDA, "power iteration launch failed: %s", cudaGetErrorString((cudaError_t)rc));
  return PDSC_OK;
}

size_t pdsc_voxel_down_sample_scratch_bytes(int64_t n) {
  if (n <= 0 || n > (1ll << 30)) return 0;
  const int32_t off[2] = {0, (int32_t)n};
  return pdsc::voxel_scratch_bytes(1, off);
}

size_t pdsc_voxel_down_sample_packed_scratch_bytes(int32_t P, const int32_t* h_offsets) {
  if (check_offsets("pdsc_voxel_down_sample_packed_scratch_bytes", "", P, h_offsets, 1) || h_offsets[P] > (1 << 30)) return 0;
  return pdsc::voxel_scratch_bytes(P, h_offsets);
}

static int voxel_impl(const char* who, pdsc_engine* e, int32_t P, const int32_t* h_offsets, const int32_t* d_offsets,
                      const float* d_points, double voxel_size, float* d_out_points, int32_t* d_out_first, int32_t* d_out_ends,
                      int32_t* d_status, void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  if (h_offsets[P] > (1 << 30)) return fail(PDSC_ERR_SHAPE, "%s: need at most 2^30 points (got %d)", who, h_offsets[P]);
  if (!(voxel_size > 0.0)) return fail(PDSC_ERR_INVALID_ARGUMENT, "voxel_size must be positive (got %g)", voxel_size);
  if (!d_points || !d_out_points || !d_out_ends || !d_status) return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: null tensor pointer", who);
  if (int rc = check_scratch(who, "scratch", d_scratch, scratch_bytes, pdsc::voxel_scratch_bytes(P, h_offsets), 8)) return rc;
  DeviceGuard g(e->cfg.device);
  pdsc::launch_voxel_down_sample(P, h_offsets, d_offsets, d_points, voxel_size, d_out_points, d_out_first, d_out_ends, d_status,
                                 d_scratch, static_cast<cudaStream_t>(cuda_stream));
  PDSC_CUDA(cudaGetLastError());
  return PDSC_OK;
}

int pdsc_voxel_down_sample(pdsc_engine* e, int64_t n, const float* d_points, double voxel_size, float* d_out_points,
                           int32_t* d_count, int32_t* d_status, void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (n <= 0 || n > (1ll << 30)) return fail(PDSC_ERR_SHAPE, "need 1 <= n <= 2^30 points (got %lld)", (long long)n);
  // the packed call with one cloud: its offsets need no device table, and its end row is the count
  const int32_t off[2] = {0, (int32_t)n};
  return voxel_impl("pdsc_voxel_down_sample", e, 1, off, nullptr, d_points, voxel_size, d_out_points, nullptr, d_count, d_status,
                    d_scratch, scratch_bytes, cuda_stream);
}

int pdsc_voxel_down_sample_packed(pdsc_engine* e, int32_t P, const int32_t* h_offsets, const int32_t* d_offsets, const float* d_points,
                                  double voxel_size, float* d_out_points, int32_t* d_out_offsets, int32_t* d_status, void* d_scratch,
                                  size_t scratch_bytes, void* cuda_stream) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (int rc = check_offsets("pdsc_voxel_down_sample_packed", "", P, h_offsets, 1)) return rc;
  if (!d_offsets || !d_out_offsets) return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_voxel_down_sample_packed: null offsets");
  return voxel_impl("pdsc_voxel_down_sample_packed", e, P, h_offsets, d_offsets, d_points, voxel_size, d_out_points, d_out_offsets,
                    d_out_offsets + 1, d_status, d_scratch, scratch_bytes, cuda_stream);
}

size_t pdsc_fpfh_scratch_bytes(int32_t m, int32_t max_nn) { return (m > 0 && max_nn > 0) ? pdsc::fpfh_scratch_bytes(m, max_nn) : 0; }

size_t pdsc_fpfh_packed_scratch_bytes(int32_t P, const int32_t* h_offsets, int32_t max_nn) {
  if (check_offsets("pdsc_fpfh_packed_scratch_bytes", "", P, h_offsets, 1) || max_nn <= 0) return 0;
  return pdsc::fpfh_scratch_bytes(h_offsets[P], max_nn);
}

static int check_search_args(const char* who, pdsc_engine* e, int32_t m, double radius, int32_t max_nn, const void* a, const void* b,
                             const void* c, void* d_scratch, size_t scratch_bytes) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (m <= 0) return fail(PDSC_ERR_SHAPE, "%s: need m >= 1 points (got %d)", who, m);
  if (!(radius > 0.0)) return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: radius must be positive (got %g)", who, radius);
  if (max_nn < 1 || max_nn > 256) return fail(PDSC_ERR_UNSUPPORTED, "%s: max_nn %d outside [1, 256]", who, max_nn);
  if (!a || !b || !c) return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: null tensor pointer", who);
  return check_scratch(who, "scratch", d_scratch, scratch_bytes, pdsc::fpfh_scratch_bytes(m, max_nn), 8);
}

static int search_impl(const char* who, pdsc_engine* e, int32_t P, const int32_t* h_offsets, const int32_t* d_offsets,
                       const float* d_points, const double* d_normals, double radius, int32_t max_nn, int32_t normalise, double* d_out,
                       int32_t* d_status, void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  const int bad = check_search_args(who, e, h_offsets[P], radius, max_nn, d_points, d_out, d_status, d_scratch, scratch_bytes);
  if (bad) return bad;
  DeviceGuard g(e->cfg.device);
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  PDSC_CUDA(cudaMemsetAsync(d_status, 0, 4 * (size_t)P, st));
  const int rc = d_normals ? pdsc::launch_compute_fpfh(P, h_offsets, d_offsets, d_points, d_normals, radius, max_nn, normalise, d_out,
                                                       d_status, d_scratch, st)
                           : pdsc::launch_estimate_normals(P, h_offsets, d_offsets, d_points, radius, max_nn, d_out, d_status, d_scratch,
                                                           st);
  if (rc) return fail(PDSC_ERR_CUDA, "%s: launch failed: %s", who, cudaGetErrorString((cudaError_t)rc));
  return PDSC_OK;
}

int pdsc_estimate_normals(pdsc_engine* e, int32_t m, const float* d_points, double radius, int32_t max_nn, double* d_normals,
                          int32_t* d_status, void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (m <= 0) return fail(PDSC_ERR_SHAPE, "pdsc_estimate_normals: need m >= 1 points (got %d)", m);
  const int32_t off[2] = {0, m};                      // the packed call with one cloud and no device table
  return search_impl("pdsc_estimate_normals", e, 1, off, nullptr, d_points, nullptr, radius, max_nn, 0, d_normals, d_status, d_scratch,
                     scratch_bytes, cuda_stream);
}

int pdsc_estimate_normals_packed(pdsc_engine* e, int32_t P, const int32_t* h_offsets, const int32_t* d_offsets, const float* d_points,
                                 double radius, int32_t max_nn, double* d_normals, int32_t* d_status, void* d_scratch,
                                 size_t scratch_bytes, void* cuda_stream) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (int rc = check_offsets("pdsc_estimate_normals_packed", "", P, h_offsets, 1)) return rc;
  if (!d_offsets) return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_estimate_normals_packed: null device offsets");
  return search_impl("pdsc_estimate_normals_packed", e, P, h_offsets, d_offsets, d_points, nullptr, radius, max_nn, 0, d_normals,
                     d_status, d_scratch, scratch_bytes, cuda_stream);
}

int pdsc_compute_fpfh(pdsc_engine* e, int32_t m, const float* d_points, const double* d_normals, double radius, int32_t max_nn,
                      int32_t normalise, double* d_fpfh, int32_t* d_status, void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (m <= 0) return fail(PDSC_ERR_SHAPE, "pdsc_compute_fpfh: need m >= 1 points (got %d)", m);
  if (!d_normals) return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_compute_fpfh: null normals");
  const int32_t off[2] = {0, m};
  return search_impl("pdsc_compute_fpfh", e, 1, off, nullptr, d_points, d_normals, radius, max_nn, normalise, d_fpfh, d_status,
                     d_scratch, scratch_bytes, cuda_stream);
}

int pdsc_compute_fpfh_packed(pdsc_engine* e, int32_t P, const int32_t* h_offsets, const int32_t* d_offsets, const float* d_points,
                             const double* d_normals, double radius, int32_t max_nn, int32_t normalise, double* d_fpfh,
                             int32_t* d_status, void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (int rc = check_offsets("pdsc_compute_fpfh_packed", "", P, h_offsets, 1)) return rc;
  if (!d_offsets) return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_compute_fpfh_packed: null device offsets");
  if (!d_normals) return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_compute_fpfh_packed: null normals");
  return search_impl("pdsc_compute_fpfh_packed", e, P, h_offsets, d_offsets, d_points, d_normals, radius, max_nn, normalise, d_fpfh,
                     d_status, d_scratch, scratch_bytes, cuda_stream);
}

int pdsc_fcgf_create(int32_t conv1_kernel_size, pdsc_fcgf** out) {
  if (!out) return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_fcgf_create: null handle pointer");
  *out = nullptr;
  if (conv1_kernel_size != 5 && conv1_kernel_size != 7)
    return fail(PDSC_ERR_UNSUPPORTED, "pdsc_fcgf_create: conv1_kernel_size must be 5 or 7 (got %d)", conv1_kernel_size);
  *out = pdsc::fcgf_new(conv1_kernel_size);
  return PDSC_OK;
}

int pdsc_fcgf_destroy(pdsc_fcgf* h) {
  pdsc::fcgf_free(h);
  return PDSC_OK;
}

int pdsc_fcgf_set_param(pdsc_fcgf* h, const char* name, const float* h_data, int64_t numel) {
  if (!h || !name || (!h_data && numel > 0) || numel < 0) return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_fcgf_set_param: bad argument");
  size_t expected = 0;
  const int rc = pdsc::fcgf_set_param(h, name, h_data, numel, &expected);
  if (rc == 1) return fail(PDSC_ERR_UNKNOWN_PARAM, "pdsc_fcgf_set_param: unknown parameter '%s'", name);
  if (rc == 2)
    return fail(PDSC_ERR_SHAPE, "pdsc_fcgf_set_param: '%s' has %lld elements, expected %zu", name, (long long)numel, expected);
  return PDSC_OK;
}

int pdsc_fcgf_commit(pdsc_fcgf* h) {
  if (!h) return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_fcgf_commit: null handle");
  std::string missing;
  const int rc = pdsc::fcgf_commit(h, &missing);
  if (rc < 0) return fail(PDSC_ERR_UNKNOWN_PARAM, "pdsc_fcgf_commit: state-dict entry missing: %s", missing.c_str());
  if (rc > 0) return fail(PDSC_ERR_CUDA, "pdsc_fcgf_commit: upload failed: %s", cudaGetErrorString((cudaError_t)rc));
  return PDSC_OK;
}

// the points of a call bound every level's rows and every int32 table index: at most 2^26 in all
static constexpr int32_t kFcgfMaxPoints = 1 << 26;

size_t pdsc_fcgf_packed_scratch_bytes(const pdsc_fcgf* h, int32_t P, const int32_t* h_offsets) {
  if (!h || check_offsets("pdsc_fcgf_packed_scratch_bytes", "", P, h_offsets, 1) || h_offsets[P] > kFcgfMaxPoints) return 0;
  return pdsc::fcgf_scratch_bytes(P, h_offsets, pdsc::fcgf_kernel_size(h));
}

int32_t pdsc_fcgf_scratch_layout(const pdsc_fcgf* h, int32_t P, const int32_t* h_offsets, int64_t* offsets, int32_t capacity) {
  if (!h || check_offsets("pdsc_fcgf_scratch_layout", "", P, h_offsets, 1) || h_offsets[P] > kFcgfMaxPoints) return 0;
  return pdsc::fcgf_scratch_layout(P, h_offsets, pdsc::fcgf_kernel_size(h), offsets, offsets ? capacity : 0);
}

int pdsc_fcgf_packed(pdsc_engine* e, const pdsc_fcgf* h, int32_t P, const int32_t* h_offsets, const int32_t* d_offsets,
                     const float* d_points, double voxel_size, float* d_keypts, float* d_desc, int32_t* d_out_offsets,
                     int32_t* d_status, void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  const char* fn = "pdsc_fcgf_packed";
  if (!e || !h) return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: null engine or weight handle", fn);
  if (!pdsc::fcgf_committed(h)) return fail(PDSC_ERR_NOT_COMMITTED, "%s: pdsc_fcgf_commit() has not been called since the last "
                                            "pdsc_fcgf_set_param()", fn);
  if (int rc = check_offsets(fn, "", P, h_offsets, 1)) return rc;
  if (h_offsets[P] > kFcgfMaxPoints) return fail(PDSC_ERR_SHAPE, "%s: need at most 2^26 points (got %d)", fn, h_offsets[P]);
  if (!(voxel_size > 0.0) || !std::isfinite(voxel_size))
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: voxel_size must be positive and finite (got %g)", fn, voxel_size);
  if (!d_offsets || !d_points || !d_keypts || !d_desc || !d_out_offsets || !d_status)
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: null tensor pointer", fn);
  const int k1 = pdsc::fcgf_kernel_size(h);
  if (int rc = check_scratch(fn, "scratch", d_scratch, scratch_bytes, pdsc::fcgf_scratch_bytes(P, h_offsets, k1), 256)) return rc;
  DeviceGuard g(e->cfg.device);
  const int rc = pdsc::launch_fcgf(h, P, h_offsets, d_offsets, d_points, voxel_size, d_keypts, d_desc, d_out_offsets, d_status,
                                   d_scratch, static_cast<cudaStream_t>(cuda_stream));
  if (rc) return fail(PDSC_ERR_CUDA, "%s: launch failed: %s", fn, cudaGetErrorString((cudaError_t)rc));
  return PDSC_OK;
}

size_t pdsc_icp_packed_scratch_bytes(int32_t B, const int32_t* h_offsets) {
  return pdsc_icp_clouds_packed_scratch_bytes(B, h_offsets, h_offsets);
}

size_t pdsc_icp_clouds_packed_scratch_bytes(int32_t B, const int32_t* h_src_offsets, const int32_t* h_tgt_offsets) {
  const char* who = "pdsc_icp_clouds_packed_scratch_bytes";
  if (check_offsets(who, "source ", B, h_src_offsets, 1) || check_offsets(who, "target ", B, h_tgt_offsets, 1)) return 0;
  return pdsc::icp_scratch_bytes(h_src_offsets[B], h_tgt_offsets[B]);
}

// pdsc_icp_packed and pdsc_icp_clouds_packed: one set of checks and one launch, under the caller's name
static int icp_clouds(const char* fn, pdsc_engine* e, int32_t B, const int32_t* h_src_offsets, const int32_t* h_tgt_offsets,
                      const int32_t* d_src_offsets, const int32_t* d_tgt_offsets, const float* d_src, const float* d_tgt,
                      const float* d_init, double max_corr_dist, int32_t max_iteration, float* d_trans, double* d_fitness,
                      double* d_rmse, int32_t* d_iterations, int32_t* d_status, void* d_scratch, size_t scratch_bytes,
                      void* cuda_stream) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  const bool one = h_src_offsets == h_tgt_offsets;     // pdsc_icp_packed: one offsets array for both sides
  if (int rc = check_offsets(fn, one ? "" : "source ", B, h_src_offsets, 1)) return rc;
  if (!one)
    if (int rc = check_offsets(fn, "target ", B, h_tgt_offsets, 1)) return rc;
  if (!d_src_offsets || !d_tgt_offsets || !d_src || !d_tgt || !d_init || !d_trans)
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: null tensor pointer", fn);
  if (!(max_corr_dist > 0.0) || !std::isfinite(max_corr_dist))
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: max_corr_dist must be positive and finite (got %g)", fn, max_corr_dist);
  if (max_iteration < 1) return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: max_iteration must be >= 1 (got %d)", fn, max_iteration);
  const long long Rs = h_src_offsets[B], Rt = h_tgt_offsets[B];
  if (int rc = check_scratch(fn, "scratch", d_scratch, scratch_bytes, pdsc::icp_scratch_bytes(Rs, Rt), 8)) return rc;
  DeviceGuard g(e->cfg.device);
  pdsc::launch_icp(B, d_src_offsets, d_tgt_offsets, Rs, Rt, d_src, d_tgt, d_init, max_corr_dist, max_iteration, d_trans, d_fitness,
                   d_rmse, d_iterations, d_status, d_scratch, static_cast<cudaStream_t>(cuda_stream));
  PDSC_CUDA(cudaGetLastError());
  return PDSC_OK;
}

int pdsc_icp_packed(pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets, const float* d_src,
                    const float* d_tgt, const float* d_init, double max_corr_dist, int32_t max_iteration, float* d_trans,
                    double* d_fitness, double* d_rmse, int32_t* d_iterations, int32_t* d_status, void* d_scratch, size_t scratch_bytes,
                    void* cuda_stream) {
  return icp_clouds("pdsc_icp_packed", e, B, h_offsets, h_offsets, d_offsets, d_offsets, d_src, d_tgt, d_init, max_corr_dist,
                    max_iteration, d_trans, d_fitness, d_rmse, d_iterations, d_status, d_scratch, scratch_bytes, cuda_stream);
}

int pdsc_icp_clouds_packed(pdsc_engine* e, int32_t B, const int32_t* h_src_offsets, const int32_t* h_tgt_offsets,
                           const int32_t* d_src_offsets, const int32_t* d_tgt_offsets, const float* d_src, const float* d_tgt,
                           const float* d_init, double max_corr_dist, int32_t max_iteration, float* d_trans, double* d_fitness,
                           double* d_rmse, int32_t* d_iterations, int32_t* d_status, void* d_scratch, size_t scratch_bytes,
                           void* cuda_stream) {
  return icp_clouds("pdsc_icp_clouds_packed", e, B, h_src_offsets, h_tgt_offsets, d_src_offsets, d_tgt_offsets, d_src, d_tgt,
                    d_init, max_corr_dist, max_iteration, d_trans, d_fitness, d_rmse, d_iterations, d_status, d_scratch,
                    scratch_bytes, cuda_stream);
}

size_t pdsc_information_matrix_packed_scratch_bytes(int32_t B, const int32_t* h_src_offsets, const int32_t* h_tgt_offsets) {
  const char* who = "pdsc_information_matrix_packed_scratch_bytes";
  if (check_offsets(who, "source ", B, h_src_offsets, 1) || check_offsets(who, "target ", B, h_tgt_offsets, 1)) return 0;
  return pdsc::information_scratch_bytes(h_tgt_offsets[B]);
}

int pdsc_information_matrix_packed(pdsc_engine* e, int32_t B, const int32_t* h_src_offsets, const int32_t* h_tgt_offsets,
                                   const int32_t* d_src_offsets, const int32_t* d_tgt_offsets, const float* d_src, const float* d_tgt,
                                   const float* d_trans, double max_corr_dist, double* d_info, int32_t* d_status, void* d_scratch,
                                   size_t scratch_bytes, void* cuda_stream) {
  const char* fn = "pdsc_information_matrix_packed";
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (int rc = check_offsets(fn, "source ", B, h_src_offsets, 1)) return rc;
  if (int rc = check_offsets(fn, "target ", B, h_tgt_offsets, 1)) return rc;
  if (!d_src_offsets || !d_tgt_offsets || !d_src || !d_tgt || !d_trans || !d_info)
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: null tensor pointer", fn);
  if (!(max_corr_dist > 0.0) || !std::isfinite(max_corr_dist))
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: max_corr_dist must be positive and finite (got %g)", fn, max_corr_dist);
  if (int rc = check_scratch(fn, "scratch", d_scratch, scratch_bytes, pdsc::information_scratch_bytes(h_tgt_offsets[B]), 8)) return rc;
  DeviceGuard g(e->cfg.device);
  pdsc::launch_information(B, d_src_offsets, d_tgt_offsets, h_tgt_offsets[B], d_src, d_tgt, d_trans, max_corr_dist, d_info, d_status,
                           d_scratch, static_cast<cudaStream_t>(cuda_stream));
  PDSC_CUDA(cudaGetLastError());
  return PDSC_OK;
}

size_t pdsc_ransac_packed_scratch_bytes(int32_t B, const int32_t* h_offsets, int32_t max_iteration) {
  if (check_offsets("pdsc_ransac_packed_scratch_bytes", "", B, h_offsets, 1)) return 0;
  if (max_iteration < 1) {
    fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_ransac_packed_scratch_bytes: max_iteration must be >= 1 (got %d)", max_iteration);
    return 0;
  }
  return pdsc::ransac_scratch_bytes(h_offsets[B], B, max_iteration);
}

// pdsc_ransac_packed and pdsc_ransac_packed_hypotheses: one set of checks and one launch, under the caller's name
static int ransac_packed(const char* fn, pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets,
                         const float* d_src, const float* d_tgt, const float* d_labels, double max_corr_dist, int32_t max_iteration,
                         uint64_t seed, float* d_trans, float* d_out_labels, double* d_fitness, double* d_rmse, int32_t* d_best,
                         int32_t* d_status, int32_t* d_hyp_good, double* d_hyp_rmse, double* d_hyp_trans, void* d_scratch,
                         size_t scratch_bytes, void* cuda_stream) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (int rc = check_offsets(fn, "", B, h_offsets, 1)) return rc;
  if (B > 65535) return fail(PDSC_ERR_UNSUPPORTED, "%s: at most 65535 sets per call (got %d)", fn, B);
  if (!d_offsets || !d_src || !d_tgt || !d_labels || !d_trans || !d_out_labels)
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: null tensor pointer", fn);
  if (!(max_corr_dist > 0.0) || !std::isfinite(max_corr_dist))
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: max_corr_dist must be positive and finite (got %g)", fn, max_corr_dist);
  if (max_iteration < 1)
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: max_iteration must be >= 1 (got %d)", fn, max_iteration);
  if (int rc = check_scratch(fn, "scratch", d_scratch, scratch_bytes, pdsc::ransac_scratch_bytes(h_offsets[B], B, max_iteration), 16))
    return rc;
  DeviceGuard g(e->cfg.device);
  pdsc::launch_ransac(B, d_offsets, h_offsets[B], d_src, d_tgt, d_labels, max_corr_dist, max_iteration, (unsigned long long)seed,
                      d_trans, d_out_labels, d_fitness, d_rmse, d_best, d_status, d_hyp_good, d_hyp_rmse, d_hyp_trans, d_scratch,
                      static_cast<cudaStream_t>(cuda_stream));
  PDSC_CUDA(cudaGetLastError());
  return PDSC_OK;
}

int pdsc_ransac_packed(pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets, const float* d_src,
                       const float* d_tgt, const float* d_labels, double max_corr_dist, int32_t max_iteration, uint64_t seed,
                       float* d_trans, float* d_out_labels, double* d_fitness, double* d_rmse, int32_t* d_best, int32_t* d_status,
                       int32_t* d_hyp_good, double* d_hyp_rmse, void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  return ransac_packed("pdsc_ransac_packed", e, B, h_offsets, d_offsets, d_src, d_tgt, d_labels, max_corr_dist, max_iteration, seed,
                       d_trans, d_out_labels, d_fitness, d_rmse, d_best, d_status, d_hyp_good, d_hyp_rmse, nullptr, d_scratch,
                       scratch_bytes, cuda_stream);
}

int pdsc_ransac_packed_hypotheses(pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets, const float* d_src,
                                  const float* d_tgt, const float* d_labels, double max_corr_dist, int32_t max_iteration,
                                  uint64_t seed, float* d_trans, float* d_out_labels, double* d_fitness, double* d_rmse,
                                  int32_t* d_best, int32_t* d_status, int32_t* d_hyp_good, double* d_hyp_rmse, double* d_hyp_trans,
                                  void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  return ransac_packed("pdsc_ransac_packed_hypotheses", e, B, h_offsets, d_offsets, d_src, d_tgt, d_labels, max_corr_dist,
                       max_iteration, seed, d_trans, d_out_labels, d_fitness, d_rmse, d_best, d_status, d_hyp_good, d_hyp_rmse,
                       d_hyp_trans, d_scratch, scratch_bytes, cuda_stream);
}

size_t pdsc_spectral_matching_packed_scratch_bytes(int32_t B, const int32_t* h_offsets) {
  if (check_offsets("pdsc_spectral_matching_packed_scratch_bytes", "", B, h_offsets, 1, pdsc::spectral_matching_max_n())) return 0;
  return pdsc::sm_scratch_bytes(h_offsets[B], B);
}

// pdsc_spectral_matching_packed and pdsc_spectral_matching_packed_iterates: one set of checks and one launch, under the caller's name
static int spectral_matching_packed(const char* fn, pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets,
                                    const float* d_corr_pos, const float* d_src_keypts, const float* d_tgt_keypts,
                                    double inlier_threshold, float* d_trans, float* d_labels, float* d_eigenvector, float* d_iterates,
                                    void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (int rc = check_offsets(fn, "", B, h_offsets, 1, pdsc::spectral_matching_max_n())) return rc;
  if (B > 65535) return fail(PDSC_ERR_UNSUPPORTED, "%s: at most 65535 sets per call (got %d)", fn, B);
  if (!d_offsets || !d_corr_pos || !d_src_keypts || !d_tgt_keypts || !d_trans || !d_labels)
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: null tensor pointer", fn);
  if (!(inlier_threshold > 0.0) || !std::isfinite(inlier_threshold))
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: inlier_threshold must be positive and finite (got %g)", fn, inlier_threshold);
  if (int rc = check_scratch(fn, "scratch", d_scratch, scratch_bytes, pdsc::sm_scratch_bytes(h_offsets[B], B), 16)) return rc;
  DeviceGuard g(e->cfg.device);
  pdsc::launch_spectral_matching(B, h_offsets, d_offsets, d_corr_pos, d_src_keypts, d_tgt_keypts, inlier_threshold, d_trans, d_labels,
                                 d_eigenvector, d_iterates, d_scratch, static_cast<cudaStream_t>(cuda_stream));
  PDSC_CUDA(cudaGetLastError());
  return PDSC_OK;
}

int pdsc_spectral_matching_packed(pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets,
                                  const float* d_corr_pos, const float* d_src_keypts, const float* d_tgt_keypts, double inlier_threshold,
                                  float* d_trans, float* d_labels, float* d_eigenvector, void* d_scratch, size_t scratch_bytes,
                                  void* cuda_stream) {
  return spectral_matching_packed("pdsc_spectral_matching_packed", e, B, h_offsets, d_offsets, d_corr_pos, d_src_keypts, d_tgt_keypts,
                                  inlier_threshold, d_trans, d_labels, d_eigenvector, nullptr, d_scratch, scratch_bytes, cuda_stream);
}

int pdsc_spectral_matching_packed_iterates(pdsc_engine* e, int32_t B, const int32_t* h_offsets, const int32_t* d_offsets,
                                           const float* d_corr_pos, const float* d_src_keypts, const float* d_tgt_keypts,
                                           double inlier_threshold, float* d_trans, float* d_labels, float* d_eigenvector,
                                           float* d_iterates, void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  return spectral_matching_packed("pdsc_spectral_matching_packed_iterates", e, B, h_offsets, d_offsets, d_corr_pos, d_src_keypts,
                                  d_tgt_keypts, inlier_threshold, d_trans, d_labels, d_eigenvector, d_iterates, d_scratch, scratch_bytes,
                                  cuda_stream);
}

// Host-side PLY vertex reader (ascii / binary_little_endian; x, y, z as float or double; other vertex properties skipped).
int pdsc_read_ply(const char* path, float* points, int64_t capacity, int64_t* n_vertices) {
  if (!path || !n_vertices) return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_read_ply: null argument");
  FILE* f = fopen(path, "rb");
  if (!f) return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_read_ply: cannot open %s", path);
  struct Closer { FILE* f; ~Closer() { fclose(f); } } closer{f};
  char line[512];
  if (!fgets(line, sizeof line, f) || strncmp(line, "ply", 3) != 0) return fail(PDSC_ERR_INVALID_ARGUMENT, "%s is not a PLY file", path);
  int format = -1;                    // 0 ascii, 1 binary little endian
  long long n = -1;
  bool in_vertex = false, vertex_first = true, seen_element = false;
  struct Prop { int size; bool is_float; int axis; };
  std::vector<Prop> props;
  while (true) {
    if (!fgets(line, sizeof line, f)) return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: header ends before end_header", path);
    char a[64] = {0}, b[64] = {0}, c[64] = {0};
    const int got = sscanf(line, "%63s %63s %63s", a, b, c);
    if (got < 1) continue;
    if (!strcmp(a, "end_header")) break;
    if (!strcmp(a, "format")) {
      if (!strcmp(b, "ascii")) format = 0;
      else if (!strcmp(b, "binary_little_endian")) format = 1;
      else return fail(PDSC_ERR_UNSUPPORTED, "%s: PLY format %s is not supported", path, b);
    } else if (!strcmp(a, "element")) {
      in_vertex = !strcmp(b, "vertex");
      if (in_vertex) { n = atoll(c); vertex_first = !seen_element; }
      seen_element = true;
    } else if (!strcmp(a, "property") && in_vertex) {
      if (!strcmp(b, "list")) return fail(PDSC_ERR_UNSUPPORTED, "%s: list properties on vertices are not supported", path);
      Prop p{0, false, -1};
      if (!strcmp(b, "char") || !strcmp(b, "uchar") || !strcmp(b, "int8") || !strcmp(b, "uint8")) p.size = 1;
      else if (!strcmp(b, "short") || !strcmp(b, "ushort") || !strcmp(b, "int16") || !strcmp(b, "uint16")) p.size = 2;
      else if (!strcmp(b, "int") || !strcmp(b, "uint") || !strcmp(b, "int32") || !strcmp(b, "uint32")) p.size = 4;
      else if (!strcmp(b, "float") || !strcmp(b, "float32")) { p.size = 4; p.is_float = true; }
      else if (!strcmp(b, "double") || !strcmp(b, "float64")) { p.size = 8; p.is_float = true; }
      else return fail(PDSC_ERR_UNSUPPORTED, "%s: unknown property type %s", path, b);
      if (!strcmp(c, "x")) p.axis = 0; else if (!strcmp(c, "y")) p.axis = 1; else if (!strcmp(c, "z")) p.axis = 2;
      if (p.axis >= 0 && !p.is_float) return fail(PDSC_ERR_UNSUPPORTED, "%s: integer coordinates are not supported", path);
      props.push_back(p);
    }
  }
  if (format < 0 || n < 0) return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: no format / vertex element in the header", path);
  if (!vertex_first) return fail(PDSC_ERR_UNSUPPORTED, "%s: the vertex element must come first", path);
  int have = 0;
  for (const Prop& p : props) if (p.axis >= 0) have |= 1 << p.axis;
  if (have != 7) return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: vertex properties x, y, z not all present", path);
  *n_vertices = n;
  if (!points) return PDSC_OK;                        // size query
  if (capacity < n) return fail(PDSC_ERR_SHAPE, "pdsc_read_ply: buffer holds %lld vertices, the file has %lld", (long long)capacity, n);
  if (format == 0) {
    for (long long i = 0; i < n; ++i) {
      for (const Prop& p : props) {
        double v;
        if (fscanf(f, "%lf", &v) != 1) return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: truncated at vertex %lld", path, i);
        if (p.axis >= 0) points[3 * i + p.axis] = (float)v;
      }
    }
  } else {
    size_t stride = 0;
    for (const Prop& p : props) stride += (size_t)p.size;
    std::vector<unsigned char> row(stride * 4096);
    for (long long i0 = 0; i0 < n; i0 += 4096) {
      const size_t rows = (size_t)std::min<long long>(4096, n - i0);
      if (fread(row.data(), stride, rows, f) != rows) return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: truncated at vertex %lld", path, i0);
      for (size_t r = 0; r < rows; ++r) {
        size_t off = r * stride;
        for (const Prop& p : props) {
          if (p.axis >= 0) {
            if (p.size == 4) { float v; memcpy(&v, &row[off], 4); points[3 * (i0 + (long long)r) + p.axis] = v; }
            else { double v; memcpy(&v, &row[off], 8); points[3 * (i0 + (long long)r) + p.axis] = (float)v; }
          }
          off += (size_t)p.size;
        }
      }
    }
  }
  return PDSC_OK;
}

size_t pdsc_match_scratch_bytes(int32_t Ns, int32_t Nt) {
  return (Ns > 0 && Nt > 0) ? pdsc::match_scratch_bytes(Ns, Nt) : 0;
}

size_t pdsc_match_packed_scratch_bytes(int32_t P, const int32_t* h_src_offsets, const int32_t* h_tgt_offsets) {
  const char* who = "pdsc_match_packed_scratch_bytes";
  if (check_offsets(who, "source ", P, h_src_offsets, 1) || check_offsets(who, "target ", P, h_tgt_offsets, 1)) return 0;
  return pdsc::match_scratch_bytes(h_src_offsets[P], h_tgt_offsets[P]);
}

static int match_impl(pdsc_engine* e, int32_t P, int32_t D, const int32_t* h_src_offsets, const int32_t* h_tgt_offsets,
                      const int32_t* d_src_offsets, const int32_t* d_tgt_offsets, const void* d_src_desc, const void* d_tgt_desc,
                      int32_t desc_is_fp64, const float* d_src_keypts, const float* d_tgt_keypts, int32_t use_mutual,
                      int32_t* d_corr, int32_t* d_out_first, int32_t* d_out_ends, float* d_corr_pos, float* d_out_src,
                      float* d_out_tgt, void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  if (D < 1 || D > pdsc::match_max_dim()) return fail(PDSC_ERR_UNSUPPORTED, "descriptor dimension %d outside [1, %d]", D, pdsc::match_max_dim());
  if (e->cfg.in_dim != 6) return fail(PDSC_ERR_UNSUPPORTED, "pdsc_match builds the in_dim = 6 input (engine has in_dim = %d)", e->cfg.in_dim);
  if (!d_src_desc || !d_tgt_desc || !d_src_keypts || !d_tgt_keypts || !d_corr || !d_out_ends || !d_corr_pos || !d_out_src || !d_out_tgt)
    return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_match: null tensor pointer");
  if (int rc = check_scratch("pdsc_match", "scratch", d_scratch, scratch_bytes,
                             pdsc::match_scratch_bytes(h_src_offsets[P], h_tgt_offsets[P]), 8))
    return rc;
  DeviceGuard g(e->cfg.device);
  pdsc::launch_match(P, h_src_offsets, h_tgt_offsets, d_src_offsets, d_tgt_offsets, d_src_desc, d_tgt_desc, desc_is_fp64,
                     d_src_keypts, d_tgt_keypts, D, use_mutual, d_scratch, d_corr, d_out_first, d_out_ends, d_corr_pos, d_out_src,
                     d_out_tgt, static_cast<cudaStream_t>(cuda_stream));
  PDSC_CUDA(cudaGetLastError());
  return PDSC_OK;
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

int pdsc_profile_enable(pdsc_engine* e, int32_t enable) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  DeviceGuard g(e->cfg.device);
  if (enable && e->ev.empty()) {
    e->ev.resize(2 * e->cfg.num_layers + 9);
    for (auto& ev : e->ev) PDSC_CUDA(cudaEventCreate(&ev));
  }
  e->profiling = enable != 0;
  e->profile_pending = false;
  for (int i = 0; i < PDSC_SPAN_COUNT; ++i) { e->span_ms[i] = 0.f; e->span_launches[i] = 0; }
  return PDSC_OK;
}

int pdsc_profile_read(pdsc_engine* e, float* ms_out, int32_t* launches_out) {
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  DeviceGuard g(e->cfg.device);
  if (e->profile_pending) {
    const int L = e->cfg.num_layers;
    cudaEvent_t* bev = e->ev.data() + 2 * L;
    PDSC_CUDA(cudaEventSynchronize(bev[8]));
    float attn = 0.f, t = 0.f;
    for (int l = 0; l < L; ++l) {
      if (cudaEventElapsedTime(&t, e->ev[2 * l], e->ev[2 * l + 1]) == cudaSuccess) attn += t;
    }
    cudaGetLastError();  // attention events are not recorded when features are injected
    auto span = [&](int a, int b) { float v = 0.f; cudaEventElapsedTime(&v, bev[a], bev[b]); return v; };
    const float enc = span(1, 2);
    e->span_ms[PDSC_SPAN_SC] += span(0, 1);
    e->span_ms[PDSC_SPAN_ATTENTION] += attn;
    e->span_ms[PDSC_SPAN_LINEAR] += enc > attn ? enc - attn : 0.f;
    e->span_ms[PDSC_SPAN_HEAD] += span(2, 3);
    e->span_ms[PDSC_SPAN_SEEDS] += span(3, 4);
    e->span_ms[PDSC_SPAN_KNN] += span(4, 5);
    e->span_ms[PDSC_SPAN_NSM] += span(5, 6);
    e->span_ms[PDSC_SPAN_HYPOTHESES] += span(6, 7);
    e->span_ms[PDSC_SPAN_REFINE] += span(7, 8);
    e->span_ms[PDSC_SPAN_TOTAL] += span(0, 8);
    e->profile_pending = false;
  }
  if (ms_out && launches_out) {
    for (int i = 0; i < PDSC_SPAN_COUNT; ++i) {
      ms_out[i] = e->span_ms[i];
      launches_out[i] = e->span_launches[i];
      e->span_ms[i] = 0.f;
      e->span_launches[i] = 0;
    }
  }
  return PDSC_OK;
}

int pdsc_forward_host(pdsc_engine* e, int32_t B, int32_t N, const float* h_corr_pos, const float* h_src,
                      const float* h_tgt, float* h_final_trans, float* h_final_labels, void* cuda_stream) {
  int32_t slot = -1;
  if (int rc = pdsc_forward_host_submit(e, B, N, h_corr_pos, h_src, h_tgt, h_final_trans, h_final_labels, cuda_stream, &slot))
    return rc;
  return pdsc_forward_host_wait(e, slot);
}

int pdsc_forward_host_submit(pdsc_engine* e, int32_t B, int32_t N, const float* h_corr_pos, const float* h_src,
                             const float* h_tgt, float* h_final_trans, float* h_final_labels, void* cuda_stream,
                             int32_t* slot_out) {
  if (!e || !slot_out) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine / slot pointer");
  if (!h_corr_pos || !h_src || !h_tgt || !h_final_trans || !h_final_labels) return fail(PDSC_ERR_INVALID_ARGUMENT, "null host pointer");
  // what the forward would refuse is refused here, before any copy out of the caller's buffers is enqueued
  if (int rc = check_forward(e, B, N, nullptr)) return rc;
  // the first free slot: a synchronous pdsc_forward_host between two _submit calls leaves the pipeline's slot free for the
  // next _submit, and repeated synchronous calls stay on slot 0, whose address-stable buffers replay one cached graph
  const int slot = !e->slots[0].busy ? 0 : !e->slots[1].busy ? 1 : -1;
  if (slot < 0) return fail(PDSC_ERR_INVALID_ARGUMENT, "both pipeline slots are in flight: pdsc_forward_host_wait one first");
  pdsc_engine::HostSlot& sl = e->slots[slot];
  DeviceGuard g(e->cfg.device);
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  const size_t R = (size_t)B * N;
  const size_t need_ws = pdsc_workspace_bytes(e, B, N);
  if (need_ws > e->host_ws_bytes) {
    PDSC_CUDA(cudaDeviceSynchronize());          // the other slot's forward may still be using the old workspace
    cudaFree(e->host_ws);
    e->host_ws = nullptr; e->host_ws_bytes = 0;
    PDSC_CUDA(cudaMalloc(&e->host_ws, need_ws));
    e->host_ws_bytes = need_ws;
  }
  const size_t in_dim = (size_t)e->cfg.in_dim;
  const size_t io_floats = R * (in_dim + 3 + 3 + 1) + (size_t)B * 16 + 64;
  if (io_floats > sl.io_floats) {                // the slot is idle (its last call was waited for): safe to replace
    cudaFree(sl.io);
    sl.io = nullptr; sl.io_floats = 0;
    PDSC_CUDA(cudaMalloc(&sl.io, io_floats * sizeof(float)));
    sl.io_floats = io_floats;
  }
  if (!e->h2d_stream) {
    PDSC_CUDA(cudaStreamCreateWithFlags(&e->h2d_stream, cudaStreamNonBlocking));
    PDSC_CUDA(cudaStreamCreateWithFlags(&e->d2h_stream, cudaStreamNonBlocking));
  }
  if (!sl.in_ready) {
    PDSC_CUDA(cudaEventCreateWithFlags(&sl.keys_ready, cudaEventDisableTiming));
    PDSC_CUDA(cudaEventCreateWithFlags(&sl.in_ready, cudaEventDisableTiming));
    PDSC_CUDA(cudaEventCreateWithFlags(&sl.fwd_done, cudaEventDisableTiming));
  }
  float* d_corr = sl.io;
  float* d_src = d_corr + R * in_dim;
  float* d_tgt = d_src + R * 3;
  float* d_lab = d_tgt + R * 3;
  float* d_tr = d_lab + R;
  // small calls (the evaluation loops' bs = 1) are launch-bound: the forward is one graph launch over the slot's
  // address-stable buffers, behind all of its inputs.  A larger, eager forward starts once the key points are in (the SC
  // kernel reads only those) and waits for corr_pos (half of the input bytes) right behind the SC kernel.
  const bool graph = R <= kGraphRows && !e->profiling;
  auto enqueue = [&]() -> int {
    // the slot's previous call has been waited for, so its buffers are free; nothing orders these copies behind the
    // forward that is running now — that is the overlap
    PDSC_CUDA(cudaMemcpyAsync(d_src, h_src, R * 3 * sizeof(float), cudaMemcpyHostToDevice, e->h2d_stream));
    PDSC_CUDA(cudaMemcpyAsync(d_tgt, h_tgt, R * 3 * sizeof(float), cudaMemcpyHostToDevice, e->h2d_stream));
    PDSC_CUDA(cudaEventRecord(sl.keys_ready, e->h2d_stream));
    PDSC_CUDA(cudaMemcpyAsync(d_corr, h_corr_pos, R * in_dim * sizeof(float), cudaMemcpyHostToDevice, e->h2d_stream));
    PDSC_CUDA(cudaEventRecord(sl.in_ready, e->h2d_stream));
    PDSC_CUDA(cudaStreamWaitEvent(st, graph ? sl.in_ready : sl.keys_ready, 0));
    const int rc = graph ? pdsc_forward_graph(e, B, N, d_corr, d_src, d_tgt, d_tr, d_lab, e->host_ws, e->host_ws_bytes, cuda_stream)
                         : forward_impl(e, 0, B, N, nullptr, nullptr, d_corr, d_src, d_tgt, d_tr, d_lab, nullptr, nullptr,
                                        e->host_ws, e->host_ws_bytes, cuda_stream, sl.in_ready);
    if (rc) return rc;
    PDSC_CUDA(cudaEventRecord(sl.fwd_done, st));
    return PDSC_OK;
  };
  if (int rc = enqueue()) {
    // the slot stays free; every copy already enqueued has finished, so nothing reads the caller's inputs once this returns
    cudaStreamSynchronize(e->h2d_stream);
    return rc;
  }
  // the results leave in _wait (on d2h_stream, beside the NEXT call's forward): a device->host copy into pageable memory blocks
  // its caller until the data has arrived, so issuing it here would hold the host inside _submit for the whole forward
  sl.h_trans = h_final_trans; sl.h_labels = h_final_labels;
  sl.d_trans = d_tr; sl.d_labels = d_lab;
  sl.trans_bytes = (size_t)B * 16 * sizeof(float); sl.labels_bytes = R * sizeof(float);
  sl.busy = true;
  *slot_out = slot;
  return PDSC_OK;
}

int pdsc_forward_host_wait(pdsc_engine* e, int32_t slot) {
  if (!e || slot < 0 || slot > 1) return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_forward_host_wait: bad engine / slot %d", slot);
  pdsc_engine::HostSlot& sl = e->slots[slot];
  if (!sl.busy) return fail(PDSC_ERR_INVALID_ARGUMENT, "pdsc_forward_host_wait: slot %d has no call in flight", slot);
  DeviceGuard g(e->cfg.device);
  sl.busy = false;
  PDSC_CUDA(cudaStreamWaitEvent(e->d2h_stream, sl.fwd_done, 0));
  PDSC_CUDA(cudaMemcpyAsync(sl.h_trans, sl.d_trans, sl.trans_bytes, cudaMemcpyDeviceToHost, e->d2h_stream));
  PDSC_CUDA(cudaMemcpyAsync(sl.h_labels, sl.d_labels, sl.labels_bytes, cudaMemcpyDeviceToHost, e->d2h_stream));
  PDSC_CUDA(cudaStreamSynchronize(e->d2h_stream));
  return PDSC_OK;
}

}  // extern "C"
