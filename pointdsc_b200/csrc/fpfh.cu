// f2 — the descriptor front end on the device (SURVEY.md §8 row f2): voxel down-sampling, normal estimation, FPFH.
//
// Reference: misc/cal_fpfh.py:21-26 (voxel_down_sample(voxel), estimate_normals(Hybrid(radius = 2 voxel, max_nn = 30)),
// compute_fpfh_feature(Hybrid(radius = 5 voxel, max_nn = 100))) and demo_registration.py:37-44.  In the reference these are calls
// into open3d 0.9, which is not in /root/reference; the algorithms restated here are open3d's published ones (the CPU restatement under oracle/
// states them on the CPU and names the conventions open3d leaves implementation-defined).  PARITY UNPINNED: no open3d output exists
// in this image to pin either side against.
//
// Layout.  points [n,3] float32 in; key points [m,3] float32 out, in ascending voxel order (ix, iy, iz); normals [m,3] float64;
// SPFH / FPFH [m,33] float64 (the dtype the reference's matcher consumes, pdsc_match desc_is_fp64 = 1).
//
// Clouds.  Every launcher takes P clouds packed back to back, cloud p owning rows [off[p], off[p+1]) of its inputs, from host
// offsets (launch sizes) and a device table (what the kernels read); the single-cloud entry points are the calls with P = 1 and
// no table.  Nothing a cloud computes reads another cloud's rows, so a cloud's results are bit for bit those of a call holding
// it alone, and the work is the sum over the clouds of what each would cost alone.  Status words are per cloud.
//
// voxel        (0) every cloud's own region of the hash table, table_slots(n_p) slots from slot0[p].  The 63-bit (ix, iy, iz)
//              key has no spare bits for the cloud index; a region per cloud keeps the key, keeps a cloud's probe chains out of
//              every other cloud's keys, and hands the compaction each cloud's slots as one contiguous range.
//              (1) min bound of every cloud by atomicMin on order-preserving keys (open3d's origin is min - voxel / 2 of THAT
//              cloud); (2) one thread per point: voxel index in fp64 exactly as floor((p - (min - voxel / 2)) / voxel), a 63-bit
//              key, insertion into its cloud's open-addressing region (atomicCAS), and the point's offset inside its voxel added
//              as 2^-40-voxel fixed point with INTEGER atomics — the sum does not depend on the order the threads arrive in, so
//              the means are reproducible bit for bit; (3) compaction of the occupied slots into each cloud's rows; (4) the
//              clouds' voxel counts scanned into the output offsets; (5) rank of every key among its cloud's keys by counting
//              the smaller ones (tiles of keys through shared memory), O(m_p^2) per cloud, which is the row after the cloud's
//              first output row.
// search       one warp per point over its own cloud's rows: squared distances in fp32 ((dx^2 + dy^2) + dz^2, each operation
//              rounded), the in-radius candidates compacted in ascending index order into the warp's shared memory, then
//              warp_select.cuh's radix select + bitonic sort for the max_nn nearest, ties by ascending index.  Neighbour indices
//              are rows of the packed array.  Brute force: m_p^2 distance evaluations per cloud, which for the m ~ 5 k key points
//              of a 3DMatch fragment is 25 M — the k-d tree open3d builds buys nothing at this size.
// normals      one thread per point: fp64 covariance of the neighbourhood, cyclic Jacobi on the 3 x 3 matrix, the eigenvector of
//              the smallest eigenvalue, sign = largest-magnitude component positive; (0, 0, 1) below three neighbours.
// spfh         one warp per point, lanes over neighbours: Darboux-frame pair features in fp64, three 11-bin histograms counted
//              with integer shared-memory atomics (every increment is the same 100 / (#neighbours - 1)).
// fpfh         one warp per point, lanes over bins: the 1 / d^2 weighted sum of the neighbours' SPFHs in rank order, each 11-bin
//              part scaled to 100, plus the point's own SPFH; optional row normalisation x / (||x|| + 1e-6) (demo_registration.py:43).
#include <math.h>

#include <algorithm>

#include "common.cuh"
#include "kernels.h"
#include "sets.cuh"
#include "voxel_hash.cuh"
#include "warp_select.cuh"

namespace pdsc {

namespace {
constexpr unsigned long long kEmpty = kEmptyKey;
constexpr int kCandCap = 4096;          // in-radius candidates one warp can hold
constexpr double kFix = 1099511627776.0;   // 2^40: fixed-point scale of the offset inside a voxel, in voxel units

// first 256-row rank tile of cloud p: a function of the offsets alone (as frontend.cu's tile0); a cloud of n rows owns
// ceil(n / 256) tiles or one more, which is idle
__host__ __device__ inline long long rank_tile0(const Offsets& off, int p) { return ((long long)off.at(p) + 255ll * p) / 256; }

struct VoxScratch {
  unsigned long long* slot0;   // [P+1] first hash slot of every cloud's region
  unsigned long long* keys;    // [S]
  unsigned long long* sums;    // [S][3]
  unsigned long long* ckeys;   // [n]   cloud p's occupied keys at rows [off[p], off[p] + count[p])
  uint32_t* minkey;            // [P][3]
  int* counter;                // [P]   occupied voxels of every cloud
  int* counts;                 // [S]
  uint32_t* cslot;             // [n]   slot of ckeys[i] inside its cloud's region
};

VoxScratch vox_carve(void* scratch, int P, long long n, unsigned long long slots) {
  unsigned char* p = static_cast<unsigned char*>(scratch);
  VoxScratch s;
  s.slot0 = reinterpret_cast<unsigned long long*>(p);  p += (size_t)(P + 1) * 8;
  s.keys = reinterpret_cast<unsigned long long*>(p);   p += slots * 8;
  s.sums = reinterpret_cast<unsigned long long*>(p);   p += slots * 24;
  s.ckeys = reinterpret_cast<unsigned long long*>(p);  p += (size_t)n * 8;
  s.minkey = reinterpret_cast<uint32_t*>(p);           p += (size_t)P * 12;
  s.counter = reinterpret_cast<int*>(p);               p += (size_t)P * 4;
  s.counts = reinterpret_cast<int*>(p);                p += slots * 4;
  s.cslot = reinterpret_cast<uint32_t*>(p);
  return s;
}
}  // namespace

size_t voxel_scratch_bytes(int P, const int32_t* h_off) {
  return (size_t)(P + 1) * 8 + total_slots(P, h_off) * 36 + (size_t)h_off[P] * 12 + (size_t)P * 16;
}

// ---- voxel down-sampling ---------------------------------------------------------------------------------------
__global__ void vox_init_kernel(int P, uint32_t* minkey, int* counter, unsigned long long* keys, unsigned long long* sums, int* counts,
                                unsigned long long slots, int32_t* status) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < slots) {
    keys[i] = kEmpty;
    sums[3 * i] = 0ull; sums[3 * i + 1] = 0ull; sums[3 * i + 2] = 0ull;
    counts[i] = 0;
  }
  if (i < 3ull * P) minkey[i] = 0xFFFFFFFFu;
  if (i < (unsigned long long)P) { counter[i] = 0; status[i] = 0; }
}

// min bound of every cloud: blockIdx.y strides over the clouds, the CTAs of one cloud over its points
__global__ void vox_bounds_kernel(const float* __restrict__ pts, int P, Offsets off, uint32_t* minkey) {
  for (int p = blockIdx.y; p < P; p += gridDim.y) {
    uint32_t m[3] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
    const long long end = off.at(p + 1);
    for (long long i = off.at(p) + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < end; i += (long long)gridDim.x * blockDim.x) {
#pragma unroll
      for (int c = 0; c < 3; ++c) m[c] = min(m[c], dist_key32(pts[3 * i + c]));
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const uint32_t w = __reduce_min_sync(0xffffffffu, m[c]);
      if ((threadIdx.x & 31) == 0) atomicMin(&minkey[3 * p + c], w);
    }
  }
}

__device__ __forceinline__ float key32_to_float(uint32_t k) {      // inverse of dist_key32 (zero comes back as +0)
  const uint32_t u = (k & 0x80000000u) ? (k ^ 0x80000000u) : ~k;
  return __uint_as_float(u);
}

__global__ void vox_insert_kernel(const float* __restrict__ pts, long long n, int P, Offsets off, double voxel,
                                  const uint32_t* __restrict__ minkey, const unsigned long long* __restrict__ slot0,
                                  unsigned long long* keys, unsigned long long* sums, int* counts, int32_t* status) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int p = find_set(P, i, [&](int q) { return (long long)off.at(q); });
  long long ix[3];
  unsigned long long q[3];
  bool bad = false;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const double origin = (double)key32_to_float(minkey[3 * p + c]) - voxel * 0.5;
    const double rel = (double)pts[3 * i + c] - origin;
    const double fi = floor(rel / voxel);
    bad |= !(fi >= 0.0 && fi < 2097152.0);             // also catches NaN / inf
    ix[c] = bad ? 0 : (long long)fi;
    double frac = (rel - fi * voxel) / voxel;          // offset inside the voxel, in [0, 1) up to rounding
    frac = fmin(fmax(frac, 0.0), 1.0);
    q[c] = bad ? 0ull : (unsigned long long)__double2ll_rn(frac * kFix);
  }
  if (bad) {
    atomicOr(&status[p], 1);                           // more than 2^21 voxels along an axis, or a non-finite coordinate
    return;
  }
  const unsigned long long key = pack_key21(ix[0], ix[1], ix[2]);
  const unsigned long long base = slot0[p];
  const unsigned long long s = hash_insert(keys, base, slot0[p + 1] - base - 1, key);
  atomicAdd(&sums[3 * s], q[0]); atomicAdd(&sums[3 * s + 1], q[1]); atomicAdd(&sums[3 * s + 2], q[2]);
  atomicAdd(&counts[s], 1);
}

// occupied slots of cloud p -> ckeys / cslot rows [off[p], off[p] + counter[p]).  Regions are multiples of 1024 slots, so a warp
// never straddles two clouds.
__global__ void vox_compact_kernel(const unsigned long long* __restrict__ keys, unsigned long long slots, int P, Offsets off,
                                   const unsigned long long* __restrict__ slot0, unsigned long long* ckeys, uint32_t* cslot,
                                   int* counter) {
  const unsigned long long s = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool occ = s < slots && keys[s] != kEmpty;
  const uint32_t b = __ballot_sync(0xffffffffu, occ);
  if (!b) return;                                      // warp-uniform
  const int p = find_set(P, (long long)s, [&](int q) { return (long long)slot0[q]; });
  const int lane = threadIdx.x & 31;
  int base = 0;
  if (lane == 0) base = atomicAdd(&counter[p], __popc(b));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (occ) {
    const size_t j = (size_t)off.at(p) + base + __popc(b & ((1u << lane) - 1u));
    ckeys[j] = keys[s];
    cslot[j] = (uint32_t)(s - slot0[p]);
  }
}

__global__ void __launch_bounds__(1024) vox_offsets_kernel(int P, const int* __restrict__ counter, int32_t* out_first,
                                                           int32_t* out_ends) {
  cta_offsets<int32_t>(P, [&](int q) { return counter[q]; }, out_first, out_ends);
}

// rank of every occupied voxel among its cloud's (keys are distinct within a cloud) = its row after the cloud's first output row
__global__ void __launch_bounds__(256) vox_rank_kernel(int P, Offsets off, const unsigned long long* __restrict__ ckeys,
                                                       const uint32_t* __restrict__ cslot, const int* __restrict__ counter,
                                                       const unsigned long long* __restrict__ slot0,
                                                       const unsigned long long* __restrict__ sums, const int* __restrict__ counts,
                                                       const uint32_t* __restrict__ minkey, double voxel,
                                                       const int32_t* __restrict__ out_ends, float* __restrict__ out_pts) {
  __shared__ unsigned long long tile[1024];
  const int p = find_set(P, (long long)blockIdx.x, [&](int q) { return rank_tile0(off, q); });
  const int m = counter[p];
  const long long local0 = ((long long)blockIdx.x - rank_tile0(off, p)) * 256;
  if (local0 >= m) return;
  const unsigned long long* ck = ckeys + off.at(p);
  const int i = (int)local0 + threadIdx.x;
  const unsigned long long mine = i < m ? ck[i] : 0ull;
  int rank = 0;
  for (int t0 = 0; t0 < m; t0 += 1024) {
    __syncthreads();
    for (int j = threadIdx.x; j < 1024; j += 256) tile[j] = (t0 + j < m) ? ck[t0 + j] : kEmpty;
    __syncthreads();
#pragma unroll 8
    for (int j = 0; j < 1024; ++j) rank += tile[j] < mine;
  }
  if (i >= m) return;
  const unsigned long long s = slot0[p] + cslot[(size_t)off.at(p) + i];
  const double cnt = (double)counts[s];
  const long long idx[3] = {(long long)(mine >> 42), (long long)((mine >> 21) & 0x1FFFFF), (long long)(mine & 0x1FFFFF)};
  const size_t row = (size_t)(p ? out_ends[p - 1] : 0) + rank;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const double origin = (double)key32_to_float(minkey[3 * p + c]) - voxel * 0.5;
    const double mean_frac = ((double)sums[3 * s + c] / kFix) / cnt;
    out_pts[3 * row + c] = (float)(origin + ((double)idx[c] + mean_frac) * voxel);
  }
}

void launch_voxel_down_sample(int P, const int32_t* h_off, const int32_t* d_off, const float* pts, double voxel, float* out_pts,
                              int32_t* out_first, int32_t* out_ends, int32_t* status, void* scratch, cudaStream_t st) {
  // without a device table (one cloud) the kernels read the offsets {0, n} as 0 * n, 1 * n
  const Offsets off{d_off, d_off ? 0 : h_off[1]};
  const long long n = h_off[P];
  const unsigned long long slots = total_slots(P, h_off);
  const VoxScratch s = vox_carve(scratch, P, n, slots);
  long long most = 0;
  for (int p = 0; p < P; ++p) most = std::max<long long>(most, (long long)h_off[p + 1] - h_off[p]);
  hash_plan_kernel<<<1, 1024, 0, st>>>(P, off, s.slot0);
  const unsigned long long init = std::max<unsigned long long>(slots, 3ull * P);
  vox_init_kernel<<<(unsigned)((init + 255) / 256), 256, 0, st>>>(P, s.minkey, s.counter, s.keys, s.sums, s.counts, slots, status);
  const int sms = device_sm_count();
  long long bx = (most + 255) / 256, by = std::min(P, 65535);
  bx = std::min<long long>(bx, std::max<long long>(1, 8LL * sms / by));
  vox_bounds_kernel<<<dim3((unsigned)bx, (unsigned)by), 256, 0, st>>>(pts, P, off, s.minkey);
  vox_insert_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(pts, n, P, off, voxel, s.minkey, s.slot0, s.keys, s.sums, s.counts,
                                                                  status);
  vox_compact_kernel<<<(unsigned)((slots + 255) / 256), 256, 0, st>>>(s.keys, slots, P, off, s.slot0, s.ckeys, s.cslot, s.counter);
  vox_offsets_kernel<<<1, 1024, 0, st>>>(P, s.counter, out_first, out_ends);
  vox_rank_kernel<<<(unsigned)rank_tile0(Offsets{h_off, 0}, P), 256, 0, st>>>(P, off, s.ckeys, s.cslot, s.counter, s.slot0, s.sums,
                                                                              s.counts, s.minkey, voxel, out_ends, out_pts);
}

// ---- hybrid (radius + max_nn) neighbour search --------------------------------------------------------------------
__global__ void __launch_bounds__(256) hybrid_search_kernel(const float* __restrict__ pts, int m, int nclouds, Offsets off, float r2,
                                                            int max_nn, int P, int warps_per_cta, int32_t* __restrict__ nb_idx,
                                                            int32_t* __restrict__ nb_cnt, int32_t* status) {
  extern __shared__ __align__(16) unsigned char hs_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int i = blockIdx.x * warps_per_cta + warp;
  if (i >= m) return;
  const size_t per_warp = (size_t)P * 8 + 1024 + (size_t)kCandCap * 8;
  unsigned char* base = hs_smem + (size_t)warp * per_warp;
  unsigned long long* sel = reinterpret_cast<unsigned long long*>(base);      // [P]
  uint32_t* hist = reinterpret_cast<uint32_t*>(base + (size_t)P * 8);         // [256]
  uint32_t* keys = hist + 256;                                                // [kCandCap]
  int32_t* cidx = reinterpret_cast<int32_t*>(keys + kCandCap);                // [kCandCap]
  const int cloud = find_set(nclouds, i, [&](int q) { return (long long)off.at(q); });
  const int r0 = off.at(cloud), r1 = off.at(cloud + 1);
  const float px = pts[3 * (size_t)i], py = pts[3 * (size_t)i + 1], pz = pts[3 * (size_t)i + 2];
  const uint32_t lt_mask = (1u << lane) - 1u;
  int cnt = 0;
  bool overflow = false;
  for (int j0 = r0; j0 < r1; j0 += 32) {
    const int j = j0 + lane;
    float d2 = 0.f;
    bool in = false;
    if (j < r1) {
      const float dx = __fsub_rn(pts[3 * (size_t)j], px), dy = __fsub_rn(pts[3 * (size_t)j + 1], py),
                  dz = __fsub_rn(pts[3 * (size_t)j + 2], pz);
      d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
      in = d2 <= r2;
    }
    const uint32_t b = __ballot_sync(0xffffffffu, in);
    if (cnt + __popc(b) > kCandCap) { overflow = true; break; }     // warp-uniform
    if (in) {
      const int o = cnt + __popc(b & lt_mask);
      keys[o] = dist_key32(d2);
      cidx[o] = j;
    }
    cnt += __popc(b);
  }
  if (overflow) {
    if (lane == 0) { atomicOr(&status[cloud], 2); nb_cnt[i] = 0; }
    for (int r = lane; r < max_nn; r += 32) nb_idx[(size_t)i * max_nn + r] = -1;
    return;
  }
  const int NP = (cnt + 31) & ~31;
  for (int j = cnt + lane; j < NP; j += 32) keys[j] = 0xFFFFFFFFu;
  __syncwarp();
  const int want = cnt < max_nn ? cnt : max_nn;
  if (want > 0) warp_select_sorted(keys, hist, sel, cnt, NP, want, P, lane);
  __syncwarp();
  for (int r = lane; r < max_nn; r += 32)
    nb_idx[(size_t)i * max_nn + r] = r < want ? cidx[(uint32_t)(sel[r] & 0xFFFFFFFFull)] : -1;
  if (lane == 0) nb_cnt[i] = want;
}

static int launch_hybrid_search(int nclouds, const int32_t* h_off, const int32_t* d_off, const float* pts, double radius, int max_nn,
                                int32_t* nb_idx, int32_t* nb_cnt, int32_t* status, cudaStream_t st) {
  const int m = h_off[nclouds];
  const Offsets off{d_off, d_off ? 0 : h_off[1]};     // no device table: one cloud, offsets {0, m}
  int P = 2;
  while (P < max_nn) P <<= 1;
  const size_t per_warp = (size_t)P * 8 + 1024 + (size_t)kCandCap * 8;
  int warps = (int)((200 * 1024) / per_warp);
  warps = warps > 8 ? 8 : warps;
  const int smem = (int)(per_warp * warps);
  const cudaError_t e = ensure_dynamic_smem(reinterpret_cast<const void*>(hybrid_search_kernel), smem);
  if (e != cudaSuccess) return (int)e;
  hybrid_search_kernel<<<(m + warps - 1) / warps, warps * 32, smem, st>>>(pts, m, nclouds, off, (float)(radius * radius), max_nn, P,
                                                                         warps, nb_idx, nb_cnt, status);
  return 0;
}

// ---- normals --------------------------------------------------------------------------------------------------
// cyclic Jacobi on a symmetric 3 x 3 matrix: a (row-major, overwritten with the eigenvalues on its diagonal), v = eigenvectors in columns
__device__ void jacobi3(double a[3][3], double v[3][3]) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) v[r][c] = r == c ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 30; ++sweep) {
    const double off = fabs(a[0][1]) + fabs(a[0][2]) + fabs(a[1][2]);
    const double diag = fabs(a[0][0]) + fabs(a[1][1]) + fabs(a[2][2]);
    if (off <= 1e-300 || off <= 1e-18 * diag) break;
#pragma unroll
    for (int pq = 0; pq < 3; ++pq) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
      const double apq = a[p][q];
      if (apq == 0.0) continue;
      const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
      const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
      const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
      a[p][p] -= t * apq;
      a[q][q] += t * apq;
      a[p][q] = a[q][p] = 0.0;
      const int r = 3 - p - q;
      const double arp = a[r][p], arq = a[r][q];
      a[r][p] = a[p][r] = c * arp - s * arq;
      a[r][q] = a[q][r] = s * arp + c * arq;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double vkp = v[k][p], vkq = v[k][q];
        v[k][p] = c * vkp - s * vkq;
        v[k][q] = s * vkp + c * vkq;
      }
    }
  }
}

__global__ void normals_kernel(const float* __restrict__ pts, int m, int max_nn, const int32_t* __restrict__ nb_idx,
                               const int32_t* __restrict__ nb_cnt, double* __restrict__ normals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const int cnt = nb_cnt[i];
  double n[3] = {0.0, 0.0, 1.0};
  if (cnt >= 3) {
    const int32_t* nb = nb_idx + (size_t)i * max_nn;
    double mean[3] = {0.0, 0.0, 0.0};
    for (int r = 0; r < cnt; ++r) {
      const size_t j = (size_t)nb[r];
      mean[0] += (double)pts[3 * j]; mean[1] += (double)pts[3 * j + 1]; mean[2] += (double)pts[3 * j + 2];
    }
    mean[0] /= cnt; mean[1] /= cnt; mean[2] /= cnt;
    double cxx = 0, cxy = 0, cxz = 0, cyy = 0, cyz = 0, czz = 0;
    for (int r = 0; r < cnt; ++r) {
      const size_t j = (size_t)nb[r];
      const double x = (double)pts[3 * j] - mean[0], y = (double)pts[3 * j + 1] - mean[1], z = (double)pts[3 * j + 2] - mean[2];
      cxx += x * x; cxy += x * y; cxz += x * z; cyy += y * y; cyz += y * z; czz += z * z;
    }
    double a[3][3] = {{cxx / cnt, cxy / cnt, cxz / cnt}, {cxy / cnt, cyy / cnt, cyz / cnt}, {cxz / cnt, cyz / cnt, czz / cnt}};
    double v[3][3];
    jacobi3(a, v);
    int best = 0;
    if (a[1][1] < a[best][best]) best = 1;
    if (a[2][2] < a[best][best]) best = 2;
    const double len = sqrt(v[0][best] * v[0][best] + v[1][best] * v[1][best] + v[2][best] * v[2][best]);
    n[0] = v[0][best] / len; n[1] = v[1][best] / len; n[2] = v[2][best] / len;
    int big = 0;
    if (fabs(n[1]) > fabs(n[big])) big = 1;
    if (fabs(n[2]) > fabs(n[big])) big = 2;
    if (n[big] < 0.0) { n[0] = -n[0]; n[1] = -n[1]; n[2] = -n[2]; }
  }
  normals[3 * (size_t)i] = n[0]; normals[3 * (size_t)i + 1] = n[1]; normals[3 * (size_t)i + 2] = n[2];
}

// ---- SPFH ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int bin11(double x) {
  const int h = (int)floor(x);
  return h < 0 ? 0 : (h > 10 ? 10 : h);
}

__global__ void __launch_bounds__(256) spfh_kernel(const float* __restrict__ pts, const double* __restrict__ normals, int m,
                                                   int max_nn, const int32_t* __restrict__ nb_idx,
                                                   const int32_t* __restrict__ nb_cnt, double* __restrict__ spfh) {
  __shared__ int hist_s[8][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int i = blockIdx.x * 8 + warp;
  if (i >= m) return;
  int* hist = hist_s[warp];
  hist[lane] = 0;
  if (lane == 0) hist[32] = 0;
  __syncwarp();
  const int cnt = nb_cnt[i];
  const double kPi = 3.141592653589793;
  const double p1[3] = {(double)pts[3 * (size_t)i], (double)pts[3 * (size_t)i + 1], (double)pts[3 * (size_t)i + 2]};
  const double n1[3] = {normals[3 * (size_t)i], normals[3 * (size_t)i + 1], normals[3 * (size_t)i + 2]};
  for (int r = 1 + lane; r < cnt; r += 32) {
    const size_t k = (size_t)nb_idx[(size_t)i * max_nn + r];
    const double n2[3] = {normals[3 * k], normals[3 * k + 1], normals[3 * k + 2]};
    double d[3] = {(double)pts[3 * k] - p1[0], (double)pts[3 * k + 1] - p1[1], (double)pts[3 * k + 2] - p1[2]};
    double f0 = 0.0, f1 = 0.0, f2 = 0.0;
    const double dist = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    if (dist != 0.0) {
      const double a1 = (n1[0] * d[0] + n1[1] * d[1] + n1[2] * d[2]) / dist;
      const double a2 = (n2[0] * d[0] + n2[1] * d[1] + n2[2] * d[2]) / dist;
      double u[3], w2[3];      // u: the frame's normal; w2: the other normal
      if (acos(fmin(1.0, fabs(a1))) > acos(fmin(1.0, fabs(a2)))) {
        u[0] = n2[0]; u[1] = n2[1]; u[2] = n2[2];
        w2[0] = n1[0]; w2[1] = n1[1]; w2[2] = n1[2];
        d[0] = -d[0]; d[1] = -d[1]; d[2] = -d[2];
        f2 = -a2;
      } else {
        u[0] = n1[0]; u[1] = n1[1]; u[2] = n1[2];
        w2[0] = n2[0]; w2[1] = n2[1]; w2[2] = n2[2];
        f2 = a1;
      }
      double v[3] = {d[1] * u[2] - d[2] * u[1], d[2] * u[0] - d[0] * u[2], d[0] * u[1] - d[1] * u[0]};
      const double vn = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
      if (vn != 0.0) {
        v[0] /= vn; v[1] /= vn; v[2] /= vn;
        const double w[3] = {u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]};
        f0 = atan2(w[0] * w2[0] + w[1] * w2[1] + w[2] * w2[2], u[0] * w2[0] + u[1] * w2[1] + u[2] * w2[2]);
        f1 = v[0] * w2[0] + v[1] * w2[1] + v[2] * w2[2];
      } else {
        f2 = 0.0;
      }
    }
    atomicAdd(&hist[bin11(11.0 * (f0 + kPi) / (2.0 * kPi))], 1);
    atomicAdd(&hist[11 + bin11(11.0 * (f1 + 1.0) * 0.5)], 1);
    atomicAdd(&hist[22 + bin11(11.0 * (f2 + 1.0) * 0.5)], 1);
  }
  __syncwarp();
  const double inc = cnt > 1 ? 100.0 / (double)(cnt - 1) : 0.0;
  for (int b = lane; b < 33; b += 32) spfh[33 * (size_t)i + b] = (double)hist[b] * inc;
}

// ---- FPFH ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) fpfh_kernel(const float* __restrict__ pts, int m, int max_nn, const int32_t* __restrict__ nb_idx,
                                                   const int32_t* __restrict__ nb_cnt, const double* __restrict__ spfh, int normalise,
                                                   double* __restrict__ out) {
  __shared__ double acc_s[8][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int i = blockIdx.x * 8 + warp;
  if (i >= m) return;
  double* acc = acc_s[warp];
  const int cnt = nb_cnt[i];
  const double p1[3] = {(double)pts[3 * (size_t)i], (double)pts[3 * (size_t)i + 1], (double)pts[3 * (size_t)i + 2]};
  double a0 = 0.0, a1 = 0.0;                  // bins lane and (lane 0 only) 32
  for (int r = 1; r < cnt; ++r) {
    const size_t k = (size_t)nb_idx[(size_t)i * max_nn + r];
    const double dx = (double)pts[3 * k] - p1[0], dy = (double)pts[3 * k + 1] - p1[1], dz = (double)pts[3 * k + 2] - p1[2];
    const double dd = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
    if (dd == 0.0) continue;
    a0 += spfh[33 * k + lane] / dd;
    if (lane == 0) a1 += spfh[33 * k + 32] / dd;
  }
  acc[lane] = a0;
  if (lane == 0) acc[32] = a1;
  __syncwarp();
  double res[2] = {0.0, 0.0};
  for (int q = 0, b = lane; b < 33; b += 32, ++q) {
    double v = 0.0;
    if (cnt > 1) {
      const int part = b / 11;
      double s = 0.0;
#pragma unroll
      for (int t = 0; t < 11; ++t) s += acc[11 * part + t];
      v = acc[b];
      if (s != 0.0) v *= 100.0 / s;
      v += spfh[33 * (size_t)i + b];
    }
    res[q] = v;
  }
  if (normalise) {
    double ss = res[0] * res[0] + res[1] * res[1];    // res[1] is zero except on lane 0
    ss = warp_sum(ss);
    const double den = sqrt(ss) + 1e-6;
    res[0] /= den; res[1] /= den;
  }
  out[33 * (size_t)i + lane] = res[0];
  if (lane == 0) out[33 * (size_t)i + 32] = res[1];
}

// ---- host side -------------------------------------------------------------------------------------------------
size_t fpfh_scratch_bytes(int m, int max_nn) {
  return (size_t)m * max_nn * 4 + (size_t)m * 4 + 16 + (size_t)m * 33 * 8;
}

int launch_estimate_normals(int P, const int32_t* h_off, const int32_t* d_off, const float* pts, double radius, int max_nn,
                            double* normals, int32_t* status, void* scratch, cudaStream_t st) {
  const int m = h_off[P];
  unsigned char* p = static_cast<unsigned char*>(scratch);
  int32_t* nb_idx = reinterpret_cast<int32_t*>(p + (size_t)m * 33 * 8);
  int32_t* nb_cnt = nb_idx + (size_t)m * max_nn;
  const int rc = launch_hybrid_search(P, h_off, d_off, pts, radius, max_nn, nb_idx, nb_cnt, status, st);
  if (rc) return rc;
  normals_kernel<<<(m + 127) / 128, 128, 0, st>>>(pts, m, max_nn, nb_idx, nb_cnt, normals);
  return (int)cudaGetLastError();
}

int launch_compute_fpfh(int P, const int32_t* h_off, const int32_t* d_off, const float* pts, const double* normals, double radius,
                        int max_nn, int normalise, double* out, int32_t* status, void* scratch, cudaStream_t st) {
  const int m = h_off[P];
  unsigned char* p = static_cast<unsigned char*>(scratch);
  double* spfh = reinterpret_cast<double*>(p);
  int32_t* nb_idx = reinterpret_cast<int32_t*>(p + (size_t)m * 33 * 8);
  int32_t* nb_cnt = nb_idx + (size_t)m * max_nn;
  const int rc = launch_hybrid_search(P, h_off, d_off, pts, radius, max_nn, nb_idx, nb_cnt, status, st);
  if (rc) return rc;
  spfh_kernel<<<(m + 7) / 8, 256, 0, st>>>(pts, normals, m, max_nn, nb_idx, nb_cnt, spfh);
  fpfh_kernel<<<(m + 7) / 8, 256, 0, st>>>(pts, m, max_nn, nb_idx, nb_cnt, spfh, normalise, out);
  return (int)cudaGetLastError();
}

}  // namespace pdsc
