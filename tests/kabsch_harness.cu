// Test-only harness: runs pdsc::kabsch_rotation (pointdsc_b200/csrc/svd3.cuh, the header the engine compiles) on an array of
// 3x3 matrices.  tests/test_gpu_kabsch.py compiles it with the engine's nvcc flags and calls the launcher through ctypes.
#include "svd3.cuh"

__global__ void kabsch_harness_kernel(const float* __restrict__ H, float* __restrict__ R, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float h[9], r[9];
#pragma unroll
  for (int j = 0; j < 9; ++j) h[j] = H[(size_t)i * 9 + j];
  pdsc::kabsch_rotation(h, r);
#pragma unroll
  for (int j = 0; j < 9; ++j) R[(size_t)i * 9 + j] = r[j];
}

// H, R: device arrays of n row-major 3x3 matrices.  Returns the CUDA error code after the kernel has finished.
extern "C" int kabsch_harness_run(const float* H, float* R, int n) {
  if (n > 0) kabsch_harness_kernel<<<(n + 127) / 128, 128>>>(H, R, n);
  cudaError_t err = cudaGetLastError();
  if (err == cudaSuccess) err = cudaDeviceSynchronize();
  return (int)err;
}
