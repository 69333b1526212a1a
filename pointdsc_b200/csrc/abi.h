// What every C entry point of include/pointdsc_b200.h shares, wherever it is defined: the last-error report, the device
// guard and the checks of a grouped call's offsets and scratch.  Each algorithm's entry points live in the file that holds its
// kernels; the definitions below live in engine.cu, which owns pdsc_engine.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <climits>

#include "../../include/pointdsc_b200.h"

namespace pdsc {

// records the message pdsc_last_error() returns on this thread, and returns `code`
pdsc_status fail(pdsc_status code, const char* fmt, ...);

#define PDSC_CUDA(expr)                                                                      \
  do {                                                                                       \
    cudaError_t err__ = (expr);                                                              \
    if (err__ != cudaSuccess)                                                                \
      return pdsc::fail(PDSC_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(err__), __FILE__, __LINE__); \
  } while (0)

// makes `dev` the current device for the guard's lifetime
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

// Host offsets [n + 1] of a call of n sets packed back to back: n >= 1, offsets[0] = 0, and every set between min_rows and
// max_rows rows.  `what` prefixes "offsets" and "rows" in the message ("source " / "target " for a group of pairs, else "").
pdsc_status check_offsets(const char* who, const char* what, int32_t n, const int32_t* h_offsets, int min_rows,
                          int max_rows = INT_MAX);

// A caller's workspace or scratch buffer: at least `need` bytes at an `align`-byte boundary.
pdsc_status check_scratch(const char* who, const char* noun, const void* ptr, size_t bytes, size_t need, size_t align);

// the configuration an engine was created with (pdsc_engine stays opaque outside engine.cu)
const pdsc_config& engine_config(const pdsc_engine* e);

}  // namespace pdsc
