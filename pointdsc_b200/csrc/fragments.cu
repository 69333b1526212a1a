// TSDF integration and surface vertices of a group of RGB-D fragments (row f9): the ScalableTSDFVolume(RGB8) integrate and the
// vertex half of extract_triangle_mesh that the reference's multiway/make_fragments.py runs through open3d 0.9.  The conventions
// are restated operation by operation under oracle/ in numpy (PARITY UNPINNED: recalled, not checked against open3d).
//
// Sets.  F fragments, fragment f owning frames [frame_off[f], frame_off[f+1]) (1 .. kMaxFrames) of one call's [NF,H,W] uint16
// depth, [NF,H,W,3] uint8 colour and [NF,2,16] float64 poses (row 0 the extrinsic, world to camera; row 1 its inverse, the
// camera pose, both row-major).  A fragment's volume units (16^3 voxels of side v, unit side L = 16 v) live in its own region of
// `slots` hash slots of the caller's table, keyed by the unit's integer coordinates (biased by 2^20, 21 bits each).
//
// Touch (open3d's per-frame touched set).  Every stride-4 pixel of every frame with depth d > 0 (d = float(raw) / float(scale),
// 0 when d >= depth_trunc) is lifted to the world in float64 through the camera pose; every unit from floor((p - trunc) / L) to
// floor((p + trunc) / L) per axis is inserted and gets bit (frame - frame_off[f]) of its frame mask.
//
// Integrate (UniformTSDFVolume::IntegrateWithDepthToCameraDistanceMultiplier, float32, every operation rounded on its own: no
// contraction).  One CTA per unit; thread t owns the voxel column (x, y) = (t / 16, t % 16) and keeps its 16 voxels in registers
// while it walks the frames of the unit's mask in ascending order, so a unit that frame j did not touch is not updated by j.
//
// Extract.  A vertex sits on the voxel edge (g, a) when the tsdf signs (f < 0) of g and g + e_a differ and one of the <= 4 cubes
// sharing the edge has all 8 corner weights non-zero.  Each unit owns the edges of its voxels; it stages the 18^3 neighbourhood
// of tsdf and weight (its 26 neighbours through the hash) in shared memory.  Vertices are numbered in the order (fragment, unit
// coordinates, x, y, z, axis): units are sorted by key when they are numbered, so no hash slot decides anything.
//
// Every fragment's result depends on its own frames only: ranks, masks and the frame order are per fragment, and every sum is in
// a fixed order, so a fragment is bit for bit the same in any group, in any order, at any SM count.
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>

#include "abi.h"
#include "common.cuh"
#include "kernels.h"
#include "sets.cuh"
#include "voxel_hash.cuh"

namespace pdsc {

namespace {
constexpr int kRes = 16;
constexpr int kUnitVoxels = kRes * kRes * kRes;
constexpr int kMaxFrames = 256;          // frames of one fragment: the bits of a unit's frame mask
constexpr int kMaxCallFrames = 65535;    // frames of one call: the touch kernel's grid's y dimension
constexpr int kMaxUnits = 1 << 22;       // units of one fragment (max_units)
constexpr int kMaskWords = kMaxFrames / 32;
constexpr int kKeyBias = 1 << 20;
constexpr int kStage = kRes + 2;
constexpr int kStageCells = kStage * kStage * kStage;

struct Table {
  unsigned long long* keys;   // [F][slots] unit keys
  uint32_t* mask;             // [F][slots][kMaskWords] frames that touched the unit
  int32_t* unit;              // [F][slots] the unit's row in the call's volume (written by the integration)
  long long slots;
};

Table table_carve(void* p, int F, int max_units) {
  Table t;
  t.slots = (long long)table_slots(max_units);
  unsigned char* q = static_cast<unsigned char*>(p);
  t.keys = reinterpret_cast<unsigned long long*>(q); q += (size_t)F * t.slots * 8;
  t.mask = reinterpret_cast<uint32_t*>(q);           q += (size_t)F * t.slots * 4 * kMaskWords;
  t.unit = reinterpret_cast<int32_t*>(q);
  return t;
}

struct Camera {
  int H, W;
  double fx, fy, cx, cy, depth_scale, depth_trunc, voxel, trunc;
};

__device__ __forceinline__ float frame_depth(const uint16_t* __restrict__ depth, long long i, const Camera& c) {
  const float d = __fdiv_rn((float)depth[i], (float)c.depth_scale);
  return (double)d >= c.depth_trunc ? 0.0f : d;
}

__device__ __forceinline__ unsigned long long unit_key(long long x, long long y, long long z) {
  return pack_key21((unsigned long long)(x + kKeyBias), (unsigned long long)(y + kKeyBias), (unsigned long long)(z + kKeyBias));
}

__device__ __forceinline__ int key_field(unsigned long long key, int shift) { return (int)((key >> shift) & 0x1FFFFF) - kKeyBias; }

__device__ __forceinline__ double dot4_rn(const double* r, double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(r[0], x), __dmul_rn(r[1], y)), __dmul_rn(r[2], z)), r[3]);
}

// every slot empty, every mask clear, counts and status 0
__global__ void table_init_kernel(Table t, long long n, int F, int32_t* counts, int32_t* status) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    t.keys[i] = kEmptyKey;
#pragma unroll
    for (int w = 0; w < kMaskWords; ++w) t.mask[i * kMaskWords + w] = 0u;
    t.unit[i] = -1;
    if (i < F) { counts[i] = 0; status[i] = 0; }
  }
}

// one thread per (frame, stride-4 pixel)
__global__ void touch_kernel(int F, Offsets foff, const uint16_t* __restrict__ depth, const double* __restrict__ poses, Camera c,
                             int max_units, Table t, int32_t* __restrict__ counts, int32_t* __restrict__ status) {
  const int j = blockIdx.y;
  const int sw = (c.W + 3) / 4, sh = (c.H + 3) / 4;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= sw * sh) return;
  const int col = 4 * (p % sw), row = 4 * (p / sw);
  const float d = frame_depth(depth, (long long)j * c.H * c.W + (long long)row * c.W + col, c);
  if (!(d > 0.0f)) return;
  const int f = find_set(F, j, [&](int q) { return foff.at(q); });
  const int lf = j - foff.at(f);
  const double z = (double)d;
  const double x = __ddiv_rn(__dmul_rn(__dadd_rn((double)col, -c.cx), z), c.fx);
  const double y = __ddiv_rn(__dmul_rn(__dadd_rn((double)row, -c.cy), z), c.fy);
  const double* cp = poses + (size_t)j * 32 + 16;
  const double L = c.voxel * kRes;
  double pw[3];
  long long lo[3], hi[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    pw[a] = dot4_rn(cp + 4 * a, x, y, z);
    lo[a] = (long long)floor(__ddiv_rn(__dadd_rn(pw[a], -c.trunc), L));
    hi[a] = (long long)floor(__ddiv_rn(__dadd_rn(pw[a], c.trunc), L));
    if (!(lo[a] >= -kKeyBias && hi[a] < kKeyBias)) { atomicOr(&status[f], 2); return; }
  }
  const unsigned long long base = (unsigned long long)f * t.slots, mask = (unsigned long long)t.slots - 1;
  for (long long ux = lo[0]; ux <= hi[0]; ++ux)
    for (long long uy = lo[1]; uy <= hi[1]; ++uy)
      for (long long uz = lo[2]; uz <= hi[2]; ++uz) {
        const unsigned long long key = unit_key(ux, uy, uz);
        unsigned long long s = mix64(key) & mask;
        long long slot = -1;
        for (long long probe = 0; probe < t.slots; ++probe) {
          const unsigned long long prev = atomicCAS(&t.keys[base + s], kEmptyKey, key);
          if (prev == kEmptyKey) {
            if (atomicAdd(&counts[f], 1) >= max_units) atomicOr(&status[f], 1);
            slot = (long long)(base + s);
            break;
          }
          if (prev == key) { slot = (long long)(base + s); break; }
          s = (s + 1) & mask;
        }
        if (slot < 0) { atomicOr(&status[f], 1); continue; }
        atomicOr(&t.mask[slot * kMaskWords + lf / 32], 1u << (lf % 32));
      }
}

// the occupied slots of every fragment, listed in slot order per fragment (order from atomics: the ranking below fixes it)
__global__ void unit_list_kernel(int F, Offsets uoff, Table t, int32_t* __restrict__ cursor, unsigned long long* __restrict__ list_key,
                                 long long* __restrict__ list_slot) {
  const long long n = (long long)F * t.slots;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long key = t.keys[i];
    if (key == kEmptyKey) continue;
    const int f = (int)(i / t.slots);
    const int u0 = uoff.at(f), nu = uoff.at(f + 1) - u0;
    const int r = atomicAdd(&cursor[f], 1);
    if (r >= nu) continue;                   // only after the unit capacity overflowed (status bit 1)
    list_key[u0 + r] = key;
    list_slot[u0 + r] = i;
  }
}

// unit row = fragment start + the number of the fragment's list entries below (key, entry).  Keys are unique, so a unit's row is
// its key's rank; entries the touch did not fill (unit offsets above its counts) keep the empty key and slot -1 and take the
// fragment's last rows, with coordinates INT32_MIN and no frames.
__global__ void unit_rank_kernel(int F, Offsets uoff, long long U, Table t, const unsigned long long* __restrict__ list_key,
                                 const long long* __restrict__ list_slot, int32_t* __restrict__ unit_keys, long long* __restrict__ unit_slot) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= U) return;
  const int f = find_set(F, i, [&](int q) { return uoff.at(q); });
  const int u0 = uoff.at(f), u1 = uoff.at(f + 1);
  const unsigned long long key = list_key[i];
  int rank = 0;
  for (int q = u0; q < u1; ++q) {
    const unsigned long long k = list_key[q];
    rank += k < key || (k == key && q < i);
  }
  const int u = u0 + rank;
  const long long slot = list_slot[i];
  const bool filled = slot >= 0;
  unit_keys[3 * (size_t)u] = filled ? key_field(key, 42) : INT32_MIN;
  unit_keys[3 * (size_t)u + 1] = filled ? key_field(key, 21) : INT32_MIN;
  unit_keys[3 * (size_t)u + 2] = filled ? key_field(key, 0) : INT32_MIN;
  unit_slot[u] = slot;
  if (filled) t.unit[slot] = u;
}

// one CTA of 256 threads per unit; thread t owns the column (x, y) = (t / 16, t % 16)
__global__ void __launch_bounds__(256) integrate_kernel(int F, Offsets foff, Offsets uoff, const uint16_t* __restrict__ depth,
                                                        const uint8_t* __restrict__ color, const double* __restrict__ poses, Camera c,
                                                        Table t, const int32_t* __restrict__ unit_keys,
                                                        const long long* __restrict__ unit_slot, float* __restrict__ tsdf_out,
                                                        float* __restrict__ weight_out, float* __restrict__ color_out) {
  const int u = blockIdx.x;
  const int f = find_set(F, u, [&](int q) { return uoff.at(q); });
  const int j0 = foff.at(f), nf = foff.at(f + 1) - j0;
  const long long slot = unit_slot[u];
  const uint32_t* mask = slot >= 0 ? t.mask + slot * kMaskWords : nullptr;
  const int x = threadIdx.x / kRes, y = threadIdx.x % kRes;
  const float v = (float)c.voxel, half = __fmul_rn(v, 0.5f);
  const float trunc = (float)c.trunc, trunc_inv = __fdiv_rn(1.0f, trunc);
  const float fx = (float)c.fx, fy = (float)c.fy, cx = (float)c.cx, cy = (float)c.cy;
  const float safe_w = __fadd_rn((float)c.W, -0.0001f), safe_h = __fadd_rn((float)c.H, -0.0001f);
  const float ffl0 = __fdiv_rn(1.0f, fx), ffl1 = __fdiv_rn(1.0f, fy);
  const double L = c.voxel * kRes;
  const float ox = (float)((double)unit_keys[3 * (size_t)u] * L), oy = (float)((double)unit_keys[3 * (size_t)u + 1] * L),
              oz = (float)((double)unit_keys[3 * (size_t)u + 2] * L);
  const float bx = __fadd_rn(__fadd_rn(half, __fmul_rn(v, (float)x)), ox);
  const float by = __fadd_rn(__fadd_rn(half, __fmul_rn(v, (float)y)), oy);
  const float bz = __fadd_rn(half, oz);
  float ts[kRes], w[kRes], cr[kRes], cg[kRes], cb[kRes];
#pragma unroll
  for (int z = 0; z < kRes; ++z) ts[z] = w[z] = cr[z] = cg[z] = cb[z] = 0.0f;
  for (int lf = 0; mask && lf < nf; ++lf) {
    if (!((mask[lf / 32] >> (lf % 32)) & 1u)) continue;
    const int j = j0 + lf;
    const double* ex = poses + (size_t)j * 32;
    float e[12], s2[3];
#pragma unroll
    for (int i = 0; i < 12; ++i) e[i] = (float)ex[i];
#pragma unroll
    for (int r = 0; r < 3; ++r) s2[r] = __fmul_rn(e[4 * r + 2], v);
    float p[3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
      p[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(e[4 * r], bx), __fmul_rn(e[4 * r + 1], by)), __fmul_rn(e[4 * r + 2], bz)), e[4 * r + 3]);
    const uint16_t* dj = depth + (size_t)j * c.H * c.W;
    const uint8_t* cj = color + (size_t)j * c.H * c.W * 3;
#pragma unroll
    for (int z = 0; z < kRes; ++z) {
      if (p[2] > 0.0f) {
        const float uf = __fadd_rn(__fadd_rn(__fdiv_rn(__fmul_rn(p[0], fx), p[2]), cx), 0.5f);
        const float vf = __fadd_rn(__fadd_rn(__fdiv_rn(__fmul_rn(p[1], fy), p[2]), cy), 0.5f);
        if (uf >= 0.0001f && uf < safe_w && vf >= 0.0001f && vf < safe_h) {
          const int pu = (int)uf, pv = (int)vf;
          const long long pix = (long long)pv * c.W + pu;
          const float d = frame_depth(dj, pix, c);
          if (d > 0.0f) {
            const float xx = __fmul_rn(__fadd_rn((float)pu, -cx), ffl0), yy = __fmul_rn(__fadd_rn((float)pv, -cy), ffl1);
            const float mult = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(xx, xx), __fmul_rn(yy, yy)), 1.0f));
            const float sdf = __fmul_rn(__fadd_rn(d, -p[2]), mult);
            if (sdf > -trunc) {
              const float tsdf = fminf(1.0f, __fmul_rn(sdf, trunc_inv));
              const float w1 = __fadd_rn(w[z], 1.0f);
              ts[z] = __fdiv_rn(__fadd_rn(__fmul_rn(ts[z], w[z]), tsdf), w1);
              cr[z] = __fdiv_rn(__fadd_rn(__fmul_rn(cr[z], w[z]), (float)cj[3 * pix]), w1);
              cg[z] = __fdiv_rn(__fadd_rn(__fmul_rn(cg[z], w[z]), (float)cj[3 * pix + 1]), w1);
              cb[z] = __fdiv_rn(__fadd_rn(__fmul_rn(cb[z], w[z]), (float)cj[3 * pix + 2]), w1);
              w[z] = w1;
            }
          }
        }
      }
#pragma unroll
      for (int r = 0; r < 3; ++r) p[r] = __fadd_rn(p[r], s2[r]);
    }
  }
  const size_t v0 = (size_t)u * kUnitVoxels + (size_t)threadIdx.x * kRes;
#pragma unroll
  for (int z = 0; z < kRes; ++z) {
    tsdf_out[v0 + z] = ts[z];
    weight_out[v0 + z] = w[z];
    color_out[3 * (v0 + z)] = cr[z];
    color_out[3 * (v0 + z) + 1] = cg[z];
    color_out[3 * (v0 + z) + 2] = cb[z];
  }
}

struct Volume {
  Table t;
  int U;                      // rows of the volume: a table entry naming a row at or above U is treated as absent
  const int32_t* unit_keys;
  const float* tsdf;
  const float* weight;
  const float* color;
};

// the 27 units around u (-1: absent) and the 18^3 tsdf / weight neighbourhood of u, local coordinate -1 .. 16 at index + 1
__device__ void stage_unit(int F, Offsets uoff, const Volume& vol, int u, int* nb, float* st, float* sw) {
  const int f = find_set(F, u, [&](int q) { return uoff.at(q); });
  if (threadIdx.x < 27) {
    const int d = threadIdx.x;
    const long long ux = vol.unit_keys[3 * (size_t)u] + d / 9 - 1, uy = vol.unit_keys[3 * (size_t)u + 1] + (d / 3) % 3 - 1,
                    uz = vol.unit_keys[3 * (size_t)u + 2] + d % 3 - 1;
    int r = -1;
    if (ux >= -kKeyBias && ux < kKeyBias && uy >= -kKeyBias && uy < kKeyBias && uz >= -kKeyBias && uz < kKeyBias) {
      const unsigned long long s = hash_find(vol.t.keys, (unsigned long long)f * vol.t.slots, (unsigned long long)vol.t.slots - 1,
                                             unit_key(ux, uy, uz));
      if (s != ~0ull) r = vol.t.unit[s];
      if (r >= vol.U) r = -1;
    }
    nb[d] = r;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kStageCells; i += blockDim.x) {
    const int lx = i / (kStage * kStage) - 1, ly = (i / kStage) % kStage - 1, lz = i % kStage - 1;
    const int dx = lx < 0 ? 0 : lx < kRes ? 1 : 2, dy = ly < 0 ? 0 : ly < kRes ? 1 : 2, dz = lz < 0 ? 0 : lz < kRes ? 1 : 2;
    const int r = nb[dx * 9 + dy * 3 + dz];
    float tv = 0.0f, wv = 0.0f;
    if (r >= 0) {
      const size_t k = (size_t)r * kUnitVoxels + (size_t)(lx - kRes * (dx - 1)) * kRes * kRes + (size_t)(ly - kRes * (dy - 1)) * kRes +
                       (lz - kRes * (dz - 1));
      tv = vol.tsdf[k];
      wv = vol.weight[k];
    }
    st[i] = tv;
    sw[i] = wv;
  }
  __syncthreads();
}

__device__ __forceinline__ int stage_index(int x, int y, int z) { return ((x + 1) * kStage + (y + 1)) * kStage + (z + 1); }

// does the edge (g, a), g local in [0, 16)^3, carry a vertex
__device__ __forceinline__ bool edge_vertex(const float* st, const float* sw, int x, int y, int z, int a) {
  const int g[3] = {x, y, z};
  int h[3] = {x, y, z};
  h[a] += 1;
  if ((st[stage_index(g[0], g[1], g[2])] < 0.0f) == (st[stage_index(h[0], h[1], h[2])] < 0.0f)) return false;
  const int b = (a + 1) % 3, c2 = (a + 2) % 3;
  for (int db = 0; db < 2; ++db)
    for (int dc = 0; dc < 2; ++dc) {
      int o[3] = {x, y, z};
      o[b] -= db;
      o[c2] -= dc;
      bool ok = true;
      for (int k = 0; k < 8 && ok; ++k) ok = sw[stage_index(o[0] + (k >> 2), o[1] + ((k >> 1) & 1), o[2] + (k & 1))] != 0.0f;
      if (ok) return true;
    }
  return false;
}

// per-thread vertex count of the column (x, y) = (t / 16, t % 16), bits (z, a) in `bits`
__device__ __forceinline__ int column_edges(const float* st, const float* sw, unsigned long long& bits) {
  const int x = threadIdx.x / kRes, y = threadIdx.x % kRes;
  bits = 0ull;
  int n = 0;
  for (int z = 0; z < kRes; ++z)
    for (int a = 0; a < 3; ++a)
      if (edge_vertex(st, sw, x, y, z, a)) { bits |= 1ull << (3 * z + a); ++n; }
  return n;
}

__global__ void __launch_bounds__(256) vertex_count_kernel(int F, Offsets uoff, Volume vol, long long* __restrict__ counts) {
  __shared__ float st[kStageCells], sw[kStageCells];
  __shared__ int nb[27];
  __shared__ int part[8];
  stage_unit(F, uoff, vol, blockIdx.x, nb, st, sw);
  unsigned long long bits;
  const int n = warp_sum(column_edges(st, sw, bits));
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long s = 0;
    for (int w = 0; w < 8; ++w) s += part[w];
    counts[blockIdx.x] = s;
  }
}

// inclusive vertex ends of every unit (in place over the counts) and every fragment's vertex offsets [F + 1]
__global__ void __launch_bounds__(1024) vertex_scan_kernel(int F, Offsets uoff, int U, long long* __restrict__ ends,
                                                           long long* __restrict__ frag_off) {
  cta_offsets<long long>(U, [&](int q) { return ends[q]; }, (long long*)nullptr, ends);
  __syncthreads();
  for (int f = threadIdx.x; f <= F; f += blockDim.x) {
    const int u1 = f == 0 ? 0 : uoff.at(f);
    frag_off[f] = u1 == 0 ? 0 : ends[u1 - 1];
  }
}

__global__ void __launch_bounds__(256) vertex_write_kernel(int F, Offsets uoff, Volume vol, double voxel,
                                                           const long long* __restrict__ ends, double* __restrict__ vertices,
                                                           double* __restrict__ colors) {
  __shared__ float st[kStageCells], sw[kStageCells];
  __shared__ int nb[27];
  __shared__ int part[256];
  const int u = blockIdx.x;
  stage_unit(F, uoff, vol, u, nb, st, sw);
  unsigned long long bits;
  const int n = column_edges(st, sw, bits);
  part[threadIdx.x] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int t = 0; t < 256; ++t) { const int x = part[t]; part[t] = run; run += x; }
  }
  __syncthreads();
  long long out = (u == 0 ? 0 : ends[u - 1]) + part[threadIdx.x];
  const int x = threadIdx.x / kRes, y = threadIdx.x % kRes;
  const long long key[3] = {vol.unit_keys[3 * (size_t)u], vol.unit_keys[3 * (size_t)u + 1], vol.unit_keys[3 * (size_t)u + 2]};
  for (int z = 0; z < kRes; ++z)
    for (int a = 0; a < 3; ++a) {
      if (!((bits >> (3 * z + a)) & 1ull)) continue;
      const int g[3] = {x, y, z};
      int h[3] = {x, y, z};
      h[a] += 1;
      const double f0 = fabs((double)st[stage_index(g[0], g[1], g[2])]), f1 = fabs((double)st[stage_index(h[0], h[1], h[2])]);
      const double den = __dadd_rn(f0, f1);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double centre = __dmul_rn(__dadd_rn((double)(key[k] * kRes + g[k]), 0.5), voxel);
        vertices[3 * out + k] = k == a ? __dadd_rn(centre, __ddiv_rn(__dmul_rn(f0, voxel), den)) : centre;
      }
      const size_t c0 = ((size_t)u * kUnitVoxels + (size_t)(x * kRes + y) * kRes + z) * 3;
      const int dh = h[a] == kRes ? 1 : 0;     // the far end may lie in the next unit along a
      int d3[3] = {1, 1, 1};
      d3[a] += dh;
      const int r1 = nb[d3[0] * 9 + d3[1] * 3 + d3[2]];
      h[a] -= kRes * dh;
      const size_t c1 = ((size_t)r1 * kUnitVoxels + (size_t)(h[0] * kRes + h[1]) * kRes + h[2]) * 3;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double a0 = __ddiv_rn((double)vol.color[c0 + k], 255.0), a1 = __ddiv_rn((double)vol.color[c1 + k], 255.0);
        colors[3 * out + k] = __ddiv_rn(__dadd_rn(__dmul_rn(f1, a0), __dmul_rn(f0, a1)), den);
      }
      ++out;
    }
}

size_t tsdf_table_bytes(int F, int max_units) {
  return (size_t)F * table_slots(max_units) * (8 + 4 * kMaskWords + 4);
}

size_t tsdf_integrate_scratch_bytes(int F, long long U) { return (size_t)U * 24 + (size_t)F * 4; }

// the frame offsets, image and volume parameters every TSDF stage of a call checks alike
pdsc_status check_tsdf(const char* fn, int32_t F, const int32_t* h_frame_offsets, int32_t height, int32_t width,
                       const double* intrinsic, double voxel_length, double sdf_trunc, int32_t max_units) {
  if (pdsc_status rc = check_offsets(fn, "frame ", F, h_frame_offsets, 1, kMaxFrames)) return rc;
  if (h_frame_offsets[F] > kMaxCallFrames)
    return fail(PDSC_ERR_SHAPE, "%s: at most %d frames per call (got %d)", fn, kMaxCallFrames, h_frame_offsets[F]);
  if (height < 1 || width < 1 || (long long)height * width > (1 << 26))
    return fail(PDSC_ERR_SHAPE, "%s: image %d x %d outside 1 .. 2^26 pixels", fn, width, height);
  if (!intrinsic) return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: null intrinsic", fn);
  for (int i = 0; i < 4; ++i)
    if (!std::isfinite(intrinsic[i]) || (i < 2 && !(intrinsic[i] > 0.0)))
      return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: intrinsic %d (%g) must be finite, and the focal lengths positive", fn, i, intrinsic[i]);
  if (!(voxel_length > 0.0) || !std::isfinite(voxel_length) || !(sdf_trunc > 0.0) || !std::isfinite(sdf_trunc))
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: voxel_length (%g) and sdf_trunc (%g) must be positive and finite", fn, voxel_length,
                sdf_trunc);
  if (max_units < 1 || max_units > kMaxUnits)
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: max_units %d outside [1, %d]", fn, max_units, kMaxUnits);
  return PDSC_OK;
}

pdsc_status check_units(const char* fn, int32_t F, const int32_t* h_unit_offsets, int32_t max_units, const void* d_table,
                        size_t table_bytes) {
  if (max_units < 1 || max_units > kMaxUnits)
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: max_units %d outside [1, %d]", fn, max_units, kMaxUnits);
  if (pdsc_status rc = check_offsets(fn, "unit ", F, h_unit_offsets, 0, max_units)) return rc;
  return check_scratch(fn, "table", d_table, table_bytes, tsdf_table_bytes(F, max_units), 8);
}

Camera camera(int H, int W, const double* intrinsic, double depth_scale, double depth_trunc, double voxel, double trunc) {
  return Camera{H, W, intrinsic[0], intrinsic[1], intrinsic[2], intrinsic[3], depth_scale, depth_trunc, voxel, trunc};
}

}  // namespace
}  // namespace pdsc

// ---- C ABI ------------------------------------------------------------------------------------------------------
using namespace pdsc;

extern "C" {

size_t pdsc_tsdf_table_bytes(int32_t F, int32_t max_units) {
  if (F < 1 || max_units < 1 || max_units > kMaxUnits) return 0;
  return tsdf_table_bytes(F, max_units);
}

int pdsc_tsdf_touch_packed(pdsc_engine* e, int32_t F, const int32_t* h_frame_offsets, const int32_t* d_frame_offsets, int32_t height,
                           int32_t width, const double* intrinsic, const uint16_t* d_depth, const double* d_poses, double depth_scale,
                           double depth_trunc, double voxel_length, double sdf_trunc, int32_t max_units, int32_t* d_unit_counts,
                           int32_t* d_status, void* d_table, size_t table_bytes, void* cuda_stream) {
  const char* fn = "pdsc_tsdf_touch_packed";
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (int rc = check_tsdf(fn, F, h_frame_offsets, height, width, intrinsic, voxel_length, sdf_trunc, max_units)) return rc;
  if (!(depth_scale > 0.0) || !std::isfinite(depth_scale))
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: depth_scale must be positive and finite (got %g)", fn, depth_scale);
  if (!d_frame_offsets || !d_depth || !d_poses || !d_unit_counts || !d_status)
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: null tensor pointer", fn);
  if (int rc = check_scratch(fn, "table", d_table, table_bytes, tsdf_table_bytes(F, max_units), 8)) return rc;
  DeviceGuard g(engine_config(e).device);
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  const Table t = table_carve(d_table, F, max_units);
  const Camera c = camera(height, width, intrinsic, depth_scale, depth_trunc, voxel_length, sdf_trunc);
  const long long n = (long long)F * t.slots;
  table_init_kernel<<<(unsigned)std::min<long long>((n + 255) / 256, 65536), 256, 0, st>>>(t, n, F, d_unit_counts, d_status);
  const int pts = ((width + 3) / 4) * ((height + 3) / 4);
  touch_kernel<<<dim3((pts + 127) / 128, h_frame_offsets[F]), 128, 0, st>>>(F, Offsets{d_frame_offsets, 0}, d_depth, d_poses, c,
                                                                             max_units, t, d_unit_counts, d_status);
  PDSC_CUDA(cudaGetLastError());
  return PDSC_OK;
}

size_t pdsc_tsdf_integrate_scratch_bytes(int32_t F, const int32_t* h_unit_offsets) {
  if (check_offsets("pdsc_tsdf_integrate_scratch_bytes", "unit ", F, h_unit_offsets, 0, kMaxUnits)) return 0;
  return tsdf_integrate_scratch_bytes(F, h_unit_offsets[F]);
}

int pdsc_tsdf_integrate_packed(pdsc_engine* e, int32_t F, const int32_t* h_frame_offsets, const int32_t* d_frame_offsets,
                               const int32_t* h_unit_offsets, const int32_t* d_unit_offsets, int32_t height, int32_t width,
                               const double* intrinsic, const uint16_t* d_depth, const uint8_t* d_color, const double* d_poses,
                               double depth_scale, double depth_trunc, double voxel_length, double sdf_trunc, int32_t max_units,
                               void* d_table, size_t table_bytes, int32_t* d_unit_keys, float* d_tsdf, float* d_weight,
                               float* d_voxel_color, void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  const char* fn = "pdsc_tsdf_integrate_packed";
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (int rc = check_tsdf(fn, F, h_frame_offsets, height, width, intrinsic, voxel_length, sdf_trunc, max_units)) return rc;
  if (int rc = check_units(fn, F, h_unit_offsets, max_units, d_table, table_bytes)) return rc;
  if (!(depth_scale > 0.0) || !std::isfinite(depth_scale))
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: depth_scale must be positive and finite (got %g)", fn, depth_scale);
  const long long U = h_unit_offsets[F];
  if (!d_frame_offsets || !d_unit_offsets || !d_depth || !d_color || !d_poses || (U > 0 && (!d_unit_keys || !d_tsdf || !d_weight ||
                                                                                             !d_voxel_color)))
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: null tensor pointer", fn);
  if (int rc = check_scratch(fn, "scratch", d_scratch, scratch_bytes, tsdf_integrate_scratch_bytes(F, U), 8)) return rc;
  DeviceGuard g(engine_config(e).device);
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  const Table t = table_carve(d_table, F, max_units);
  const Camera c = camera(height, width, intrinsic, depth_scale, depth_trunc, voxel_length, sdf_trunc);
  unsigned char* p = static_cast<unsigned char*>(d_scratch);
  unsigned long long* list_key = reinterpret_cast<unsigned long long*>(p); p += (size_t)U * 8;
  long long* list_slot = reinterpret_cast<long long*>(p);                 p += (size_t)U * 8;
  long long* unit_slot = reinterpret_cast<long long*>(p);                 p += (size_t)U * 8;
  int32_t* cursor = reinterpret_cast<int32_t*>(p);
  launch_fill_u32(reinterpret_cast<uint32_t*>(cursor), 0u, F, st);
  launch_fill_u64(list_key, kEmptyKey, 2 * U, st);          // list_key and list_slot: empty key, slot -1
  const long long n = (long long)F * t.slots;
  const Offsets uoff{d_unit_offsets, 0};
  unit_list_kernel<<<(unsigned)std::min<long long>((n + 255) / 256, 65536), 256, 0, st>>>(F, uoff, t, cursor, list_key, list_slot);
  if (U > 0) {
    unit_rank_kernel<<<(unsigned)((U + 255) / 256), 256, 0, st>>>(F, uoff, U, t, list_key, list_slot, d_unit_keys, unit_slot);
    integrate_kernel<<<(unsigned)U, 256, 0, st>>>(F, Offsets{d_frame_offsets, 0}, uoff, d_depth, d_color, d_poses, c, t, d_unit_keys,
                                                  unit_slot, d_tsdf, d_weight, d_voxel_color);
  }
  PDSC_CUDA(cudaGetLastError());
  return PDSC_OK;
}

int pdsc_extract_vertices_count_packed(pdsc_engine* e, int32_t F, const int32_t* h_unit_offsets, const int32_t* d_unit_offsets,
                                       int32_t max_units, void* d_table, size_t table_bytes, const int32_t* d_unit_keys,
                                       const float* d_tsdf, const float* d_weight, int64_t* d_vertex_ends, int64_t* d_vertex_offsets,
                                       void* cuda_stream) {
  const char* fn = "pdsc_extract_vertices_count_packed";
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (int rc = check_units(fn, F, h_unit_offsets, max_units, d_table, table_bytes)) return rc;
  const int U = h_unit_offsets[F];
  if (!d_unit_offsets || !d_vertex_offsets || (U > 0 && (!d_unit_keys || !d_tsdf || !d_weight || !d_vertex_ends)))
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: null tensor pointer", fn);
  DeviceGuard g(engine_config(e).device);
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  const Volume vol{table_carve(d_table, F, max_units), U, d_unit_keys, d_tsdf, d_weight, nullptr};
  const Offsets uoff{d_unit_offsets, 0};
  long long* ends = reinterpret_cast<long long*>(d_vertex_ends);
  if (U > 0) vertex_count_kernel<<<U, 256, 0, st>>>(F, uoff, vol, ends);
  vertex_scan_kernel<<<1, 1024, 0, st>>>(F, uoff, U, ends, reinterpret_cast<long long*>(d_vertex_offsets));
  PDSC_CUDA(cudaGetLastError());
  return PDSC_OK;
}

int pdsc_extract_vertices_packed(pdsc_engine* e, int32_t F, const int32_t* h_unit_offsets, const int32_t* d_unit_offsets,
                                 int32_t max_units, void* d_table, size_t table_bytes, const int32_t* d_unit_keys, const float* d_tsdf,
                                 const float* d_weight, const float* d_voxel_color, double voxel_length, const int64_t* d_vertex_ends,
                                 double* d_vertices, double* d_vertex_colors, void* cuda_stream) {
  const char* fn = "pdsc_extract_vertices_packed";
  if (!e) return fail(PDSC_ERR_INVALID_ARGUMENT, "null engine");
  if (int rc = check_units(fn, F, h_unit_offsets, max_units, d_table, table_bytes)) return rc;
  if (!(voxel_length > 0.0) || !std::isfinite(voxel_length))
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: voxel_length must be positive and finite (got %g)", fn, voxel_length);
  const int U = h_unit_offsets[F];
  if (!d_unit_offsets || (U > 0 && (!d_unit_keys || !d_tsdf || !d_weight || !d_voxel_color || !d_vertex_ends)))
    return fail(PDSC_ERR_INVALID_ARGUMENT, "%s: null tensor pointer", fn);
  DeviceGuard g(engine_config(e).device);
  if (U > 0) {
    const Volume vol{table_carve(d_table, F, max_units), U, d_unit_keys, d_tsdf, d_weight, d_voxel_color};
    vertex_write_kernel<<<U, 256, 0, static_cast<cudaStream_t>(cuda_stream)>>>(
        F, Offsets{d_unit_offsets, 0}, vol, voxel_length, reinterpret_cast<const long long*>(d_vertex_ends), d_vertices, d_vertex_colors);
  }
  PDSC_CUDA(cudaGetLastError());
  return PDSC_OK;
}

}  // extern "C"
