// Per-cloud open-addressing hash of 63-bit voxel keys, shared by the voxel down-sampling (fpfh.cu) and the FCGF coordinate
// maps (fcgf.cu).  Cloud p owns table_slots(n_p) slots from slot0[p]; a key is three 21-bit fields (x << 42 | y << 21 | z),
// hashed with mix64 and probed linearly inside the cloud's region.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "sets.cuh"

namespace pdsc {

constexpr unsigned long long kEmptyKey = ~0ull;

__host__ __device__ inline unsigned long long table_slots(long long n) {
  unsigned long long c = 1024;
  while (c < 2ull * (unsigned long long)n) c <<= 1;
  return c;
}

inline unsigned long long total_slots(int P, const int32_t* h_off) {
  unsigned long long s = 0;
  for (int p = 0; p < P; ++p) s += table_slots((long long)h_off[p + 1] - h_off[p]);
  return s;
}

__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
  return x;
}

// three fields in [0, 2^21)
__host__ __device__ __forceinline__ unsigned long long pack_key21(unsigned long long x, unsigned long long y, unsigned long long z) {
  return (x << 42) | (y << 21) | z;
}

// the slot holding `key` in the region [base, base + mask + 1), inserted if absent
__device__ __forceinline__ unsigned long long hash_insert(unsigned long long* keys, unsigned long long base, unsigned long long mask,
                                                          unsigned long long key) {
  unsigned long long s = mix64(key) & mask;
  while (true) {
    const unsigned long long prev = atomicCAS(&keys[base + s], kEmptyKey, key);
    if (prev == kEmptyKey || prev == key) return base + s;
    s = (s + 1) & mask;
  }
}

// the slot holding `key`, or ~0 when the region does not hold it (the table is read-only here)
__device__ __forceinline__ unsigned long long hash_find(const unsigned long long* __restrict__ keys, unsigned long long base,
                                                        unsigned long long mask, unsigned long long key) {
  unsigned long long s = mix64(key) & mask;
  while (true) {
    const unsigned long long k = keys[base + s];
    if (k == key) return base + s;
    if (k == kEmptyKey) return ~0ull;
    s = (s + 1) & mask;
  }
}

// exclusive prefix sums of v(0 .. n-1) by ONE CTA of 1024 threads: out_first[0] = 0 (unless null), out_ends[q] = v(0) + .. + v(q)
template <typename T, typename F>
__device__ void cta_offsets(int n, F v, T* out_first, T* out_ends) {
  __shared__ T part[1024];
  const int per = (n + 1023) / 1024;
  const int q0 = min(n, (int)threadIdx.x * per), q1 = min(n, q0 + per);
  T s = 0;
  for (int q = q0; q < q1; ++q) s += v(q);
  part[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    T run = 0;
    for (int t = 0; t < 1024; ++t) { const T x = part[t]; part[t] = run; run += x; }
    if (out_first) out_first[0] = 0;
  }
  __syncthreads();
  T run = part[threadIdx.x];
  for (int q = q0; q < q1; ++q) { run += v(q); out_ends[q] = run; }
}

// every cloud's hash-table region: table_slots(n_p) slots (a power of two, at least 1024) from slot0[p]
static __global__ void __launch_bounds__(1024) hash_plan_kernel(int P, Offsets off, unsigned long long* slot0) {
  cta_offsets<unsigned long long>(P, [&](int q) { return table_slots((long long)off.at(q + 1) - off.at(q)); }, slot0, slot0 + 1);
}

}  // namespace pdsc
