// PWG conditioning upsampler stage: nearest repeat x s + (2s+1)-tap FIR (layers/upsample.py:112-128),
// evaluated poly-phase: output o only touches input frames (o-s)/s .. (o+s)/s, no stretched tensor.
// The causal stage (use_causal_conv: the FIR pads 2s on the left and the tail is cropped, upsample.py:98-125) is the
// same FIR with its tap origin at 2s instead of s: every output meets the input frames one frame earlier.  `lag` is
// that shift in frames (0 centred, 1 causal); the per-phase coefficients do not depend on it.
// The streaming form of the causal stage (HIST) takes frames -2 and -1 from a carried state instead of the zero
// padding, so that a chunked run equals the whole-signal stage; the caller carries the state from chunk to chunk.
#include "common.cuh"

namespace pwgb {

// Output o = j*s + ph only touches the input frames j-1, j, j+1 (minus lag): y[o] = A[ph] x[j-1] + B[ph] x[j] + C[ph] x[j+1] with the
// taps pre-summed per phase (A: taps that land in frame j-1, ...).  One thread per input frame writes its s outputs
// (one 16-byte store per 4): 3 FMAs per output instead of 2s+1 taps with an integer division each (the tap loop ran
// at 1/12 of the HBM rate: 13 % of the Parallel WaveGAN forward).
// HIST (causal, lag 1): frames j-2 and j-1 below 0 are hist_in[r][j] and hist_in[r][1] (rows x 2, oldest first).  Same
// three-FMA expression.
// EXT (with HIST): the stage of a lookahead stream (pwgb_upsample_fir_stream_ext_forward); the same expression, with the
// outputs outside the signal (the pwgb_stream_ext mask) stored as +0.0.
template <bool HIST, bool EXT>
__device__ __forceinline__ void upsample_fir_body(int rows, int rows_per_batch, int t_in, int s, int lag, const float* __restrict__ x,
                                                  const float* __restrict__ fir, float* __restrict__ y, long long ybs,
                                                  const float* __restrict__ hist_in, const int* frame, const int* end, int rate,
                                                  int look) {
  extern __shared__ float coef[];  // [3][s]
  for (int ph = threadIdx.x; ph < s; ph += blockDim.x) {
    float a = 0.f, bsum = 0.f, c = 0.f;
    for (int k = 0; k <= 2 * s; ++k) {
      const int d = ph + k - s;
      const float f = fir[k];
      if (d < 0)
        a += f;
      else if (d < s)
        bsum += f;
      else
        c += f;
    }
    coef[ph] = a;
    coef[s + ph] = bsum;
    coef[2 * s + ph] = c;
  }
  __syncthreads();
  const int r = blockIdx.y;
  const int t_out = t_in * s;
  const float* xr = x + (long long)r * t_in;
  float* yr = y + (long long)(r / rows_per_batch) * ybs + (long long)(r % rows_per_batch) * t_out;
  const bool vec = (s % 4 == 0) && ((reinterpret_cast<uintptr_t>(yr) & 15) == 0);
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < t_in; j += gridDim.x * blockDim.x) {
    float xm, x0, xp;
    if constexpr (HIST) {
      const float* hr = hist_in + 2 * (long long)r;
      xm = j >= 2 ? __ldg(xr + j - 2) : __ldg(hr + j);
      x0 = j >= 1 ? __ldg(xr + j - 1) : __ldg(hr + 1);
      xp = __ldg(xr + j);
    } else {
      const int jc = j - lag;
      xm = jc > 0 ? __ldg(xr + jc - 1) : 0.f;
      x0 = jc >= 0 ? __ldg(xr + jc) : 0.f;
      xp = jc + 1 < t_in ? __ldg(xr + jc + 1) : 0.f;
    }
    float* dst = yr + (long long)j * s;
    if constexpr (EXT) {
      // signal sample of output o = j * s + ph; the chunk's outputs are contiguous, so the mask is one interval per frame
      const long long pos0 = (long long)__ldg(frame + r / rows_per_batch) * rate - look + (long long)j * s;
      const long long lim = (long long)__ldg(end + r / rows_per_batch) * rate;
      for (int ph = 0; ph < s; ++ph) {
        const float v = fmaf(coef[2 * s + ph], xp, fmaf(coef[s + ph], x0, coef[ph] * xm));
        dst[ph] = (pos0 + ph < 0 || pos0 + ph >= lim) ? 0.f : v;
      }
      continue;
    }
    if (vec) {
      for (int ph = 0; ph < s; ph += 4) {
        float4 v;
        v.x = fmaf(coef[2 * s + ph], xp, fmaf(coef[s + ph], x0, coef[ph] * xm));
        v.y = fmaf(coef[2 * s + ph + 1], xp, fmaf(coef[s + ph + 1], x0, coef[ph + 1] * xm));
        v.z = fmaf(coef[2 * s + ph + 2], xp, fmaf(coef[s + ph + 2], x0, coef[ph + 2] * xm));
        v.w = fmaf(coef[2 * s + ph + 3], xp, fmaf(coef[s + ph + 3], x0, coef[ph + 3] * xm));
        *reinterpret_cast<float4*>(dst + ph) = v;
      }
    } else {
      for (int ph = 0; ph < s; ++ph) dst[ph] = fmaf(coef[2 * s + ph], xp, fmaf(coef[s + ph], x0, coef[ph] * xm));
    }
  }
}

template <bool HIST>
__global__ void upsample_fir_kernel(int rows, int rows_per_batch, int t_in, int s, int lag, const float* __restrict__ x,
                                    const float* __restrict__ fir, float* __restrict__ y, long long ybs,
                                    const float* __restrict__ hist_in) {
  upsample_fir_body<HIST, false>(rows, rows_per_batch, t_in, s, lag, x, fir, y, ybs, hist_in, nullptr, nullptr, 1, 0);
}

__global__ void upsample_fir_stream_ext_kernel(int rows, int rows_per_batch, int t_in, int s, const float* __restrict__ x,
                                               const float* __restrict__ fir, float* __restrict__ y, long long ybs,
                                               const float* __restrict__ hist_in, const int* __restrict__ frame,
                                               const int* __restrict__ end, int rate, int look) {
  upsample_fir_body<true, true>(rows, rows_per_batch, t_in, s, 1, x, fir, y, ybs, hist_in, frame, end, rate, look);
}

}  // namespace pwgb

using namespace pwgb;

static int upsample_fir_forward(int rows, int rows_per_batch, int t_in, int scale, int lag, const float* x, const float* fir,
                                float* y, long long y_batch_stride, void* stream, const float* hist_in = nullptr) {
  PWGB_CHECK_ARG(x && fir && y, "upsample_fir: null argument");
  PWGB_CHECK_ARG(rows >= 0 && rows_per_batch > 0 && t_in > 0 && scale > 0 && rows % rows_per_batch == 0,
                 "upsample_fir: bad sizes");
  PWGB_UNSUPPORTED_IF(rows > 65535, "upsample_fir: too many rows");
  if (rows == 0) return PWGB_OK;
  const int t_out = t_in * scale;
  const long long ybs = y_batch_stride ? y_batch_stride : (long long)rows_per_batch * t_out;
  dim3 grid(ceil_div(t_in, 256) < 64 ? ceil_div(t_in, 256) : 64, rows);
  const size_t smem = 3 * scale * sizeof(float);
  if (hist_in)
    upsample_fir_kernel<true><<<grid, 256, smem, (cudaStream_t)stream>>>(rows, rows_per_batch, t_in, scale, lag, x, fir, y, ybs,
                                                                         hist_in);
  else
    upsample_fir_kernel<false><<<grid, 256, smem, (cudaStream_t)stream>>>(rows, rows_per_batch, t_in, scale, lag, x, fir, y, ybs,
                                                                          nullptr);
  return check_launch("upsample_fir_kernel");
}

extern "C" int pwgb_upsample_fir_forward(int rows, int rows_per_batch, int t_in, int scale, const float* x,
                                         const float* fir, float* y, long long y_batch_stride, void* stream) {
  return upsample_fir_forward(rows, rows_per_batch, t_in, scale, 0, x, fir, y, y_batch_stride, stream);
}

extern "C" int pwgb_upsample_fir_causal_forward(int rows, int rows_per_batch, int t_in, int scale, const float* x,
                                                const float* fir, float* y, long long y_batch_stride, void* stream) {
  return upsample_fir_forward(rows, rows_per_batch, t_in, scale, 1, x, fir, y, y_batch_stride, stream);
}

extern "C" int pwgb_upsample_fir_causal_stream_forward(int rows, int rows_per_batch, int t_in, int scale, const float* x,
                                                       const float* fir, float* y, long long y_batch_stride, const float* hist_in,
                                                       void* stream) {
  PWGB_CHECK_ARG(hist_in, "upsample_fir_causal_stream: null history");
  return upsample_fir_forward(rows, rows_per_batch, t_in, scale, 1, x, fir, y, y_batch_stride, stream, hist_in);
}

extern "C" int pwgb_upsample_fir_stream_ext_forward(int rows, int rows_per_batch, int t_in, int scale, const float* x, const float* fir,
                                                    float* y, long long y_batch_stride, const float* hist_in,
                                                    const pwgb_stream_ext* ext, void* stream) {
  PWGB_CHECK_ARG(x && fir && y && hist_in, "upsample_fir_stream_ext: null argument");
  PWGB_CHECK_ARG(ext && ext->frame && ext->end && ext->rate >= 1 && ext->lookahead >= 0 && !ext->res_hist_len && !ext->res_delay,
                 "upsample_fir_stream_ext: ext must be a mask (frame, end, rate >= 1, lookahead >= 0) without residual fields");
  PWGB_CHECK_ARG(rows >= 0 && rows_per_batch > 0 && t_in > 0 && scale > 0 && rows % rows_per_batch == 0,
                 "upsample_fir_stream_ext: bad sizes");
  PWGB_UNSUPPORTED_IF(rows > 65535, "upsample_fir_stream_ext: too many rows");
  if (rows == 0) return PWGB_OK;
  const long long ybs = y_batch_stride ? y_batch_stride : (long long)rows_per_batch * t_in * scale;
  dim3 grid(ceil_div(t_in, 256) < 64 ? ceil_div(t_in, 256) : 64, rows);
  upsample_fir_stream_ext_kernel<<<grid, 256, 3 * scale * sizeof(float), (cudaStream_t)stream>>>(
      rows, rows_per_batch, t_in, scale, x, fir, y, ybs, hist_in, ext->frame, ext->end, ext->rate, ext->lookahead);
  return check_launch("upsample_fir_stream_ext_kernel");
}
