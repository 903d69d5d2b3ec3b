// Shared helpers for libpwgb (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "pwgb.h"

namespace pwgb {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);
// argument check shared by the two history conv entry points (api.cu)
int conv1d_stream_check(const pwgb_conv1d_desc* d, const float* x, const float* hist, int hist_len, const float* y);
// argument check of a pwgb_stream_ext (NULL passes); residual: whether the launch has one; pad_mode: the conv's (an edge
// policy needs PWGB_PAD_HISTORY), -1 for an entry point without an edge policy
int stream_ext_check(const pwgb_stream_ext* e, const float* residual, int pad_mode = -1);
// argument check of the two ragged conv entry points (stream.cu); h: the history descriptor their launch runs
int conv1d_ragged_check(const pwgb_conv1d_desc* d, const float* x, const pwgb_stream_ext* e, const float* y,
                        pwgb_conv1d_desc* h);

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

// A kernel may use 48 KB of shared memory, static and dynamic together, unless it opts in to more: opt in to `dyn`
// dynamic bytes whenever they and the kernel's static arrays together pass 48 KB.
template <typename Kernel>
static int allow_dynamic_smem(Kernel kernel, size_t dyn, const char* what) {
  if (dyn <= 32 * 1024) return PWGB_OK;  // far below the limit: skip the attribute query
  cudaFuncAttributes a;
  cudaError_t e = cudaFuncGetAttributes(&a, kernel);
  if (e == cudaSuccess && dyn + a.sharedSizeBytes > 48 * 1024)
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn);
  if (e != cudaSuccess) {
    set_error("%s: shared memory opt-in: %s", what, cudaGetErrorString(e));
    return PWGB_CUDA_ERROR;
  }
  return PWGB_OK;
}

// the two history padding policies of the stream entry points (flagged slots replicate or reflect)
__host__ __device__ inline bool is_history_pad(int pad_mode) {
  return pad_mode == PWGB_PAD_HISTORY || pad_mode == PWGB_PAD_HISTORY_REFLECT;
}

__device__ __forceinline__ float lrelu(float v, float slope) { return v > 0.f ? v : v * slope; }

// The mask of a pwgb_stream_ext launch: output row `row` of item b lies outside its signal
__device__ __forceinline__ bool stream_outside(const int* frame, const int* end, int rate, int lookahead, int b, long long row) {
  const long long pos = (long long)__ldg(frame + b) * rate - lookahead + row;
  return pos < 0 || pos >= (long long)__ldg(end + b) * rate;
}
// The rows [lo, hi) of a launch of t rows that lie inside item b's signal in the sense of stream_outside
__device__ __forceinline__ void stream_signal_rows(const int* frame, const int* end, int rate, int lookahead, int b, int t, int& lo,
                                                   int& hi) {
  const long long first = (long long)lookahead - (long long)__ldg(frame + b) * rate;
  const long long last = first + (long long)__ldg(end + b) * rate;
  lo = (int)(first < 0 ? 0 : first < t ? first : t);
  hi = (int)(last < lo ? lo : last < t ? last : t);
}

// Accurate-enough transcendental helpers: tanhf/expf from libdevice (<= 2 ulp);
// the parity bar is 1e-3 relative so these are never the limiting error.
__device__ __forceinline__ float sigmoidf_(float v) { return 1.f / (1.f + __expf(-v)); }

}  // namespace pwgb
