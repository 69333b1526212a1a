// Point-to-point ICP over the correspondence key points, for the drivers' --use_icp (evaluation/benchmark_utils.py:40-55, which
// hands the pair to open3d 0.9's registration_icp with max correspondence distance 0.10 and the default convergence criteria).
//
// Semantics (restated on the CPU by the restatement under oracle/, which names the conventions open3d leaves to FLANN): T in fp64 from
// init; P = init src; the correspondences C are every source row's nearest target row of the same set, kept iff
// d^2 < float32(r^2), ties to the lowest target row; fitness = |C| / N, rmse = sqrt(sum d^2 / |C|).  Each iteration solves the
// Umeyama update U over C without scaling (svd3.cuh's Jacobi Kabsch in double), sets T <- U T and P <- U P, recomputes C and
// stops once |d fitness| < 1e-6 and |d rmse| < 1e-6, or after max_iteration updates.
//
// Sets.  B sets packed back to back, set b owning rows [off[b], off[b+1]) of src / tgt; one CTA per set runs everything below
// from its own rows and its own scratch only, with reductions in a fixed order, so a set's result is bit for bit the same
// whatever else its call holds, in whatever order, on any SM count.  No host synchronisation, capturable in a CUDA graph.
//
// Grid.  The target never moves, so each set indexes it once: cells of side h = max(r, sqrt(float32(r^2))) (no kept neighbour is
// further than one cell away on any axis), keyed as in fpfh.cu (21 bits per axis relative to the set's own minimum, 63 bits),
// in the set's own open-addressing region of 2^ceil(log2(2 N)) <= 4 N slots starting at slot 4 off[b].  The rows of each cell
// are counted, scanned and listed; their order inside a cell comes from atomics and does not matter, because the search takes
// the minimum of (d^2, row).  A set with a non-finite coordinate, or whose target spans 2^21 cells or more along an axis, gets
// status 1 and returns init after 0 iterations (fitness = rmse = 0).
//
// Search.  The 27 cells around each moved source point.  The cost is the number of target rows in those cells: for key points a
// few voxels apart that is a handful, but a set whose rows all fall into one cell makes every iteration N^2 (correct, slow).
#include <math.h>

#include "common.cuh"
#include "kernels.h"
#include "sets.cuh"
#include "svd3.cuh"

namespace pdsc {

namespace {
constexpr int kIcpThreads = 256;
constexpr int kIcpWarps = kIcpThreads / 32;
constexpr unsigned long long kEmptyCell = ~0ull;
constexpr double kMaxCells = 2097152.0;   // 2^21 cells per axis

__host__ __device__ inline long long icp_table_slots(long long n) {
  long long c = 2;
  while (c < 2 * n) c <<= 1;
  return c;
}

__device__ __forceinline__ unsigned long long cell_mix(unsigned long long x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
  return x;
}

struct IcpScratch {
  double* P;                 // [R][3] the moved source points
  unsigned long long* keys;  // [4R]   cell keys, set b's region from slot 4 off[b]
  int* start;                // [4R]   first list entry of the cell
  int* count;                // [4R]   rows of the cell
  int* list;                 // [R]    set-local target rows grouped by cell
  int* slot;                 // [R]    region slot of every target row
  int* nn;                   // [R]    kept nearest target row (set-local) of every source row, or -1
};

IcpScratch icp_carve(void* scratch, long long R) {
  unsigned char* p = static_cast<unsigned char*>(scratch);
  IcpScratch s;
  s.P = reinterpret_cast<double*>(p);               p += (size_t)R * 24;
  s.keys = reinterpret_cast<unsigned long long*>(p); p += (size_t)R * 32;
  s.start = reinterpret_cast<int*>(p);              p += (size_t)R * 16;
  s.count = reinterpret_cast<int*>(p);              p += (size_t)R * 16;
  s.list = reinterpret_cast<int*>(p);               p += (size_t)R * 4;
  s.slot = reinterpret_cast<int*>(p);               p += (size_t)R * 4;
  s.nn = reinterpret_cast<int*>(p);
  return s;
}

// fixed-order CTA sum of NV doubles: lanes by xor shuffle, then warps in ascending order; every thread gets the totals
template <int NV>
__device__ __forceinline__ void icp_block_sum(double (&v)[NV], double* red /* [kIcpWarps][NV] */, double* tot /* [NV] */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = warp_sum(v[i]);
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) red[warp * NV + i] = v[i];
  }
  __syncthreads();
  if (threadIdx.x < NV) {
    double acc = 0.0;
    for (int w = 0; w < kIcpWarps; ++w) acc += red[w * NV + threadIdx.x];
    tot[threadIdx.x] = acc;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = tot[i];
  __syncthreads();   // tot / red are free for the next sum
}

__device__ __forceinline__ float icp_block_min(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float m = red[0];
  for (int w = 1; w < kIcpWarps; ++w) m = fminf(m, red[w]);
  __syncthreads();
  return m;
}

struct Grid {
  const unsigned long long* keys;   // the set's region
  const int* start;
  const int* count;
  const int* list;
  unsigned long long mask;
  double lo[3], h;
};

__device__ __forceinline__ int find_cell(const Grid& g, unsigned long long key) {
  unsigned long long s = cell_mix(key) & g.mask;
  while (true) {
    const unsigned long long k = g.keys[s];
    if (k == key) return (int)s;
    if (k == kEmptyCell) return -1;
    s = (s + 1) & g.mask;
  }
}

// nearest target row (set-local) of p by (d^2, row), searched in the 27 cells around p; row -1 when none
__device__ __forceinline__ int nearest_target(const Grid& g, const float* __restrict__ pt, double px, double py, double pz, double& best) {
  best = INFINITY;
  int row = -1;
  const double fc[3] = {floor((px - g.lo[0]) / g.h), floor((py - g.lo[1]) / g.h), floor((pz - g.lo[2]) / g.h)};
  for (int dx = -1; dx <= 1; ++dx) {
    const double cx = fc[0] + dx;
    if (!(cx >= 0.0 && cx < kMaxCells)) continue;     // also NaN
    for (int dy = -1; dy <= 1; ++dy) {
      const double cy = fc[1] + dy;
      if (!(cy >= 0.0 && cy < kMaxCells)) continue;
      for (int dz = -1; dz <= 1; ++dz) {
        const double cz = fc[2] + dz;
        if (!(cz >= 0.0 && cz < kMaxCells)) continue;
        const unsigned long long key =
            ((unsigned long long)cx << 42) | ((unsigned long long)cy << 21) | (unsigned long long)cz;
        const int s = find_cell(g, key);
        if (s < 0) continue;
        const int q1 = g.start[s] + g.count[s];
        for (int q = g.start[s]; q < q1; ++q) {
          const int r = g.list[q];
          const double ex = px - (double)pt[3 * (size_t)r], ey = py - (double)pt[3 * (size_t)r + 1],
                       ez = pz - (double)pt[3 * (size_t)r + 2];
          const double d2 = ex * ex + ey * ey + ez * ez;
          if (d2 < best || (d2 == best && r < row)) { best = d2; row = r; }
        }
      }
    }
  }
  return row;
}
}  // namespace

size_t icp_scratch_bytes(long long R) { return (size_t)R * 100; }

__global__ void __launch_bounds__(kIcpThreads) icp_kernel(const float* __restrict__ src, const float* __restrict__ tgt,
                                                          const float* __restrict__ init, Offsets off, double r, double r2f,
                                                          int max_iteration, IcpScratch s, float* __restrict__ trans,
                                                          double* __restrict__ fitness_out, double* __restrict__ rmse_out,
                                                          int32_t* __restrict__ iterations_out, int32_t* __restrict__ status_out) {
  __shared__ double red[kIcpWarps * 9];
  __shared__ double tot[9];
  __shared__ double T[16], U[12];
  __shared__ float fred[kIcpWarps];
  __shared__ int bad;
  __shared__ int part[kIcpThreads];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int row0 = off.at(b), N = off.at(b + 1) - row0;
  const float* ps = src + (size_t)row0 * 3;
  const float* pt = tgt + (size_t)row0 * 3;
  double* P = s.P + (size_t)row0 * 3;
  int* nn = s.nn + row0;
  if (tid < 16) T[tid] = (double)init[(size_t)b * 16 + tid];
  if (tid == 0) bad = 0;
  __syncthreads();

  // ---- the set's minimum and finiteness ----
  float lo[3] = {INFINITY, INFINITY, INFINITY};
  bool finite = true;
  for (int j = tid; j < N; j += kIcpThreads) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float t = pt[3 * (size_t)j + c];
      finite = finite && isfinite(t) && isfinite(ps[3 * (size_t)j + c]);
      lo[c] = fminf(lo[c], t);
    }
  }
  if (!finite) bad = 1;                    // benign race: every writer stores 1
  Grid g;
  g.h = fmax(r, sqrt(r2f));
#pragma unroll
  for (int c = 0; c < 3; ++c) g.lo[c] = (double)icp_block_min(lo[c], fred);

  // ---- the set's cell index: region init, insertion (with the extent check), scan, lists ----
  const long long slots = icp_table_slots(N), base = 4ll * row0;
  unsigned long long* keys = s.keys + base;
  int* start = s.start + base;
  int* count = s.count + base;
  int* list = s.list + row0;
  int* slot = s.slot + row0;
  for (long long q = tid; q < slots; q += kIcpThreads) { keys[q] = kEmptyCell; count[q] = 0; }
  __syncthreads();
  g.keys = keys; g.start = start; g.count = count; g.list = list;
  g.mask = (unsigned long long)slots - 1;
  if (!bad) {
    for (int j = tid; j < N; j += kIcpThreads) {
      double cc[3];
      bool out = false;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        cc[c] = floor(((double)pt[3 * (size_t)j + c] - g.lo[c]) / g.h);
        out = out || !(cc[c] >= 0.0 && cc[c] < kMaxCells);
      }
      if (out) { bad = 1; continue; }
      const unsigned long long key =
          ((unsigned long long)cc[0] << 42) | ((unsigned long long)cc[1] << 21) | (unsigned long long)cc[2];
      unsigned long long q = cell_mix(key) & g.mask;
      while (true) {
        const unsigned long long prev = atomicCAS(&keys[q], kEmptyCell, key);
        if (prev == kEmptyCell || prev == key) break;
        q = (q + 1) & g.mask;
      }
      atomicAdd(&count[q], 1);
      slot[j] = (int)q;
    }
  }
  __syncthreads();
  if (bad) {
    if (tid < 16) trans[(size_t)b * 16 + tid] = init[(size_t)b * 16 + tid];
    if (tid == 0) {
      if (fitness_out) fitness_out[b] = 0.0;
      if (rmse_out) rmse_out[b] = 0.0;
      if (iterations_out) iterations_out[b] = 0;
      if (status_out) status_out[b] = 1;
    }
    return;
  }
  {  // exclusive scan of the counts into the starts; the counts become fill cursors
    const long long per = (slots + kIcpThreads - 1) / kIcpThreads;
    const long long q0 = min(slots, (long long)tid * per), q1 = min(slots, q0 + per);
    int sum = 0;
    for (long long q = q0; q < q1; ++q) sum += count[q];
    part[tid] = sum;
    __syncthreads();
    if (tid == 0) {
      int run = 0;
      for (int t = 0; t < kIcpThreads; ++t) { const int x = part[t]; part[t] = run; run += x; }
    }
    __syncthreads();
    int run = part[tid];
    for (long long q = q0; q < q1; ++q) { start[q] = run; run += count[q]; count[q] = 0; }
  }
  __syncthreads();
  for (int j = tid; j < N; j += kIcpThreads) {
    const int q = slot[j];
    list[start[q] + atomicAdd(&count[q], 1)] = j;
  }
  __syncthreads();

  // ---- correspondences of the moved cloud (after applying U when `move`): count, sum d^2, sums of P and of its targets ----
  auto correspond = [&](bool move, double (&acc)[8]) {
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.0;
    for (int j = tid; j < N; j += kIcpThreads) {
      double x, y, z;
      if (move) {
        const double ax = P[3 * (size_t)j], ay = P[3 * (size_t)j + 1], az = P[3 * (size_t)j + 2];
        x = U[0] * ax + U[1] * ay + U[2] * az + U[3];
        y = U[4] * ax + U[5] * ay + U[6] * az + U[7];
        z = U[8] * ax + U[9] * ay + U[10] * az + U[11];
      } else {
        const double ax = ps[3 * (size_t)j], ay = ps[3 * (size_t)j + 1], az = ps[3 * (size_t)j + 2];
        x = T[0] * ax + T[1] * ay + T[2] * az + T[3];
        y = T[4] * ax + T[5] * ay + T[6] * az + T[7];
        z = T[8] * ax + T[9] * ay + T[10] * az + T[11];
      }
      P[3 * (size_t)j] = x; P[3 * (size_t)j + 1] = y; P[3 * (size_t)j + 2] = z;
      double d2;
      int k = nearest_target(g, pt, x, y, z, d2);
      if (k >= 0 && !(d2 < r2f)) k = -1;
      nn[j] = k;
      if (k >= 0) {
        acc[0] += 1.0; acc[1] += d2;
        acc[2] += x; acc[3] += y; acc[4] += z;
        acc[5] += (double)pt[3 * (size_t)k]; acc[6] += (double)pt[3 * (size_t)k + 1]; acc[7] += (double)pt[3 * (size_t)k + 2];
      }
    }
    icp_block_sum<8>(acc, red, tot);
  };

  double acc[8];
  correspond(false, acc);
  double fit = acc[0] / (double)N, rmse = acc[0] > 0.0 ? sqrt(acc[1] / acc[0]) : 0.0;
  int its = 0;
  for (int it = 0; it < max_iteration; ++it) {
    if (acc[0] > 0.0) {
      const double ax = acc[2] / acc[0], ay = acc[3] / acc[0], az = acc[4] / acc[0];
      const double bx = acc[5] / acc[0], by = acc[6] / acc[0], bz = acc[7] / acc[0];
      double h[9];
#pragma unroll
      for (int i = 0; i < 9; ++i) h[i] = 0.0;
      for (int j = tid; j < N; j += kIcpThreads) {
        const int k = nn[j];
        if (k < 0) continue;
        const double mx = P[3 * (size_t)j] - ax, my = P[3 * (size_t)j + 1] - ay, mz = P[3 * (size_t)j + 2] - az;
        const double nx = (double)pt[3 * (size_t)k] - bx, ny = (double)pt[3 * (size_t)k + 1] - by,
                     nz = (double)pt[3 * (size_t)k + 2] - bz;
        h[0] += mx * nx; h[1] += mx * ny; h[2] += mx * nz;
        h[3] += my * nx; h[4] += my * ny; h[5] += my * nz;
        h[6] += mz * nx; h[7] += mz * ny; h[8] += mz * nz;
      }
      icp_block_sum<9>(h, red, tot);
      if (tid == 0) {
        double R[9];
        kabsch_rotation(h, R);
        U[0] = R[0]; U[1] = R[1]; U[2] = R[2];  U[3] = bx - (R[0] * ax + R[1] * ay + R[2] * az);
        U[4] = R[3]; U[5] = R[4]; U[6] = R[5];  U[7] = by - (R[3] * ax + R[4] * ay + R[5] * az);
        U[8] = R[6]; U[9] = R[7]; U[10] = R[8]; U[11] = bz - (R[6] * ax + R[7] * ay + R[8] * az);
        double T2[12];
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
          for (int c = 0; c < 4; ++c)
            T2[4 * i + c] = U[4 * i] * T[c] + U[4 * i + 1] * T[4 + c] + U[4 * i + 2] * T[8 + c] + U[4 * i + 3] * T[12 + c];
#pragma unroll
        for (int i = 0; i < 12; ++i) T[i] = T2[i];
      }
      __syncthreads();
    }
    // without correspondences the update is the identity: T, P and C stay as they are
    if (acc[0] > 0.0) correspond(true, acc);
    ++its;
    const double f2 = acc[0] / (double)N, r2 = acc[0] > 0.0 ? sqrt(acc[1] / acc[0]) : 0.0;
    const bool done = fabs(fit - f2) < 1e-6 && fabs(rmse - r2) < 1e-6;
    fit = f2;
    rmse = r2;
    if (done) break;
  }
  if (tid < 16) trans[(size_t)b * 16 + tid] = (float)T[tid];
  if (tid == 0) {
    if (fitness_out) fitness_out[b] = fit;
    if (rmse_out) rmse_out[b] = rmse;
    if (iterations_out) iterations_out[b] = its;
    if (status_out) status_out[b] = 0;
  }
}

void launch_icp(int B, const int32_t* d_off, long long R, const float* src, const float* tgt, const float* init, double r,
                int max_iteration, float* trans, double* fitness, double* rmse, int32_t* iterations, int32_t* status, void* scratch,
                cudaStream_t st) {
  const double r2f = (double)(float)(r * r);
  icp_kernel<<<B, kIcpThreads, 0, st>>>(src, tgt, init, Offsets{d_off, 0}, r, r2f, max_iteration, icp_carve(scratch, R), trans,
                                        fitness, rmse, iterations, status);
}

}  // namespace pdsc
