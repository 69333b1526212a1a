// Per-device launch configuration.  cudaFuncSetAttribute(MaxDynamicSharedMemorySize) and the SM count are properties of
// (kernel, DEVICE), not of the process: an engine created on cuda:1 after one on cuda:0 must opt its kernels in again on
// that device.  State is keyed by the current device ordinal and guarded by a mutex (engines on different devices may be
// driven from different host threads).
#include <cuda_runtime.h>

#include <cstdlib>
#include <map>
#include <mutex>

#include "kernels.h"

namespace pdsc {
namespace {
constexpr int kMaxDevices = 64;
struct DeviceState {
  int num_sms = 0;
  std::map<const void*, int> smem_opt_in;   // kernel -> bytes already granted on this device
};
std::mutex g_mu;
DeviceState g_dev[kMaxDevices];
}  // namespace

cudaError_t ensure_dynamic_smem(const void* kernel, int bytes) {
  if (bytes <= 48 * 1024) return cudaSuccess;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= kMaxDevices) return cudaErrorInvalidDevice;
  std::lock_guard<std::mutex> lock(g_mu);
  int& granted = g_dev[dev].smem_opt_in[kernel];
  if (bytes <= granted) return cudaSuccess;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) granted = bytes;
  return e;
}

// PDSC_SM_COUNT=<n> (developer override, read once): size every SM-count-dependent launch and split as if the device had
// min(n, its real count) SMs, so that a test can check which results do not depend on the SM count.  Unset or not a
// positive integer: the real count.
static int sm_count_override() {
  const char* s = std::getenv("PDSC_SM_COUNT");
  if (!s || !*s) return 0;
  char* end = nullptr;
  const long v = std::strtol(s, &end, 10);
  return (*end == '\0' && v > 0 && v < (1L << 20)) ? (int)v : 0;
}

int device_sm_count() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return 0;
  static const int forced = sm_count_override();
  std::lock_guard<std::mutex> lock(g_mu);
  if (g_dev[dev].num_sms == 0) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    g_dev[dev].num_sms = (forced > 0 && forced < n) ? forced : n;
  }
  return g_dev[dev].num_sms;
}

}  // namespace pdsc
