// Decode-driver glue on the GPU (bin/decode.py:214-243; SURVEY.md 8f-2): feature normalisation + (T, C) -> (C, T)
// transpose + edge padding of one utterance into its slot of a batch tensor, and float -> PCM16 quantisation of the
// waveform, so that an utterance crosses PCIe once as mels and once as int16 samples.
#include "common.cuh"

namespace pwgb {

// out[ch, t] = norm(c[clamp_or_zero(t - pad_left), ch]),  norm(v) = (v - mean[ch]) / scale[ch]  (hifigan.py:264-265)
// pad_mode 0: frames outside [0, T) are zero (after normalisation: exactly what a zero-padded conv input sees);
// pad_mode 2: replicate the edge frames (ReplicationPad1d(aux_context_window), parallel_wavegan.py:250-251).
__global__ void prep_features_kernel(const float* __restrict__ c, const float* __restrict__ mean, const float* __restrict__ scale,
                                     float* __restrict__ out, int T, int C, int pad_left, int t_out, int pad_mode) {
  __shared__ float tile[32][33];
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  // read 32 frames x 32 channels (coalesced along channels), write transposed (coalesced along time)
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i, ch = c0 + threadIdx.x;
    int src = t - pad_left;
    bool ok = t < t_out && ch < C;
    if (src < 0 || src >= T) {
      if (pad_mode == 2) src = src < 0 ? 0 : T - 1;
      else ok = false;
    }
    float v = 0.f;
    if (ok) {
      v = __ldg(c + (long long)src * C + ch);
      if (mean) v = (v - __ldg(mean + ch)) / __ldg(scale + ch);
    }
    tile[i][threadIdx.x] = v;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int ch = c0 + i, t = t0 + threadIdx.x;
    if (ch < C && t < t_out) out[(long long)ch * t_out + t] = tile[threadIdx.x][i];
  }
}

// libsndfile's float -> PCM_16 conversion as used by sf.write(..., "PCM_16") (decode.py:236-241): lrintf(y * 32767),
// saturated to the int16 range (libsndfile wraps out-of-range values unless clipping is enabled; generators end in tanh).
// The product is one fp32 multiply and rintf rounds half to even.  A NaN sample becomes 0: silence rather than a
// full-scale click (fmaxf would turn it into -32768), and what libsndfile's lrintf gives once cut to 16 bits on x86-64.
__global__ void pcm16_kernel(const float* __restrict__ y, short* __restrict__ out, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = rintf(y[i] * 32767.f);
    out[i] = v != v ? (short)0 : (short)fminf(fmaxf(v, -32768.f), 32767.f);
  }
}

}  // namespace pwgb

using namespace pwgb;

extern "C" int pwgb_prep_features(const float* c, const float* mean, const float* scale, float* out, int t, int channels, int pad_left,
                                  int t_out, int pad_mode, void* stream) {
  PWGB_CHECK_ARG(c && out && t > 0 && channels > 0 && pad_left >= 0 && t_out > 0 && (pad_mode == PWGB_PAD_ZERO || pad_mode == PWGB_PAD_REPLICATE),
                 "prep_features: bad argument");
  PWGB_CHECK_ARG((mean == nullptr) == (scale == nullptr), "prep_features: mean and scale go together");
  dim3 grid((unsigned)ceil_div(t_out, 32), (unsigned)ceil_div(channels, 32));
  prep_features_kernel<<<grid, dim3(32, 8), 0, (cudaStream_t)stream>>>(c, mean, scale, out, t, channels, pad_left, t_out, pad_mode);
  return check_launch("prep_features_kernel");
}

extern "C" int pwgb_pcm16_forward(const float* y, short* out, long long n, void* stream) {
  PWGB_CHECK_ARG(y && out && n >= 0, "pcm16: bad argument");
  if (n == 0) return PWGB_OK;
  int blocks = (int)((n + 255) / 256 > 1184 ? 1184 : (n + 255) / 256);
  pcm16_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(y, out, n);
  return check_launch("pcm16_kernel");
}
