// Test-only harness: runs pdsc::kabsch_rotation (pointdsc_b200/csrc/svd3.cuh, the header the engine compiles) on an array of
// 3x3 matrices, in float (the forward's solves) and in double (the ICP updates).  tests/test_gpu_kabsch.py compiles it with the
// engine's nvcc flags and calls the launchers through ctypes.
#include "svd3.cuh"

template <typename T>
__global__ void kabsch_harness_kernel(const T* __restrict__ H, T* __restrict__ R, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  T h[9], r[9];
#pragma unroll
  for (int j = 0; j < 9; ++j) h[j] = H[(size_t)i * 9 + j];
  pdsc::kabsch_rotation(h, r);
#pragma unroll
  for (int j = 0; j < 9; ++j) R[(size_t)i * 9 + j] = r[j];
}

template <typename T>
static int kabsch_harness_launch(const T* H, T* R, int n) {
  if (n > 0) kabsch_harness_kernel<T><<<(n + 127) / 128, 128>>>(H, R, n);
  cudaError_t err = cudaGetLastError();
  if (err == cudaSuccess) err = cudaDeviceSynchronize();
  return (int)err;
}

// H, R: device arrays of n row-major 3x3 matrices.  Return the CUDA error code after the kernel has finished.
extern "C" int kabsch_harness_run(const float* H, float* R, int n) { return kabsch_harness_launch(H, R, n); }
extern "C" int kabsch_harness_run_f64(const double* H, double* R, int n) { return kabsch_harness_launch(H, R, n); }
