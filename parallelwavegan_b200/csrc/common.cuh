// Shared helpers for libpwgb (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "pwgb.h"

namespace pwgb {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);

#define PWGB_CHECK_ARG(cond, ...)          \
  do {                                     \
    if (!(cond)) {                         \
      ::pwgb::set_error(__VA_ARGS__);      \
      return PWGB_INVALID;                 \
    }                                      \
  } while (0)

#define PWGB_UNSUPPORTED_IF(cond, ...)     \
  do {                                     \
    if (cond) {                            \
      ::pwgb::set_error(__VA_ARGS__);      \
      return PWGB_UNSUPPORTED;             \
    }                                      \
  } while (0)

inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return PWGB_CUDA_ERROR;
  }
  count_launch();
  return PWGB_OK;
}

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

__device__ __forceinline__ float lrelu(float v, float slope) { return v > 0.f ? v : v * slope; }

// Accurate-enough transcendental helpers: tanhf/expf from libdevice (<= 2 ulp);
// the parity bar is 1e-3 relative so these are never the limiting error.
__device__ __forceinline__ float sigmoidf_(float v) { return 1.f / (1.f + __expf(-v)); }

}  // namespace pwgb
