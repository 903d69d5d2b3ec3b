// Small deterministic reductions used by the adversarial / feature-matching losses
// (losses/adversarial_loss.py:29-123, losses/feat_match_loss.py:27-54): mean over n elements of
//   mode 0: (x - c)^2        (LS-GAN terms, c = 1 or 0)
//   mode 1: |x - y|          (feature matching L1)
//   mode 2: max(0, c - s*x)  (hinge terms: real: c=1,s=+1 ; fake: c=1,s=-1)
//   mode 3: s * x            (hinge generator loss: -mean(x))
//   mode 4: (x - y)^2        (MSELoss between two tensors: the VQ-VAE quantisation / commitment losses)
// out[0] (+)= weight * mean.  Two-stage, fixed order: bit-reproducible.
#include "common.cuh"

namespace pwgb {

__global__ void __launch_bounds__(256) reduce_partial_kernel(int mode, const float* __restrict__ x,
                                                              const float* __restrict__ y, long long n, float c,
                                                              float s, float* __restrict__ part) {
  __shared__ float red[8];
  float acc = 0.f;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const float v = x[i];
    float t;
    if (mode == 0) {
      t = (v - c) * (v - c);
    } else if (mode == 1) {
      t = fabsf(v - y[i]);
    } else if (mode == 4) {
      const float e = v - y[i];
      t = e * e;
    } else if (mode == 2) {
      t = fmaxf(0.f, c - s * v);
    } else {
      t = s * v;
    }
    acc += t;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = 0.f;
    for (int i = 0; i < 8; ++i) v += red[i];
    part[blockIdx.x] = v;
  }
}

__global__ void reduce_final_kernel(const float* __restrict__ part, int nparts, double scale, int accumulate,
                                    float* __restrict__ out) {
  __shared__ double red[256];
  double a = 0;
  for (int i = threadIdx.x; i < nparts; i += 256) a += part[i];
  red[threadIdx.x] = a;
  __syncthreads();
  for (int st = 128; st > 0; st >>= 1) {
    if (threadIdx.x < st) red[threadIdx.x] += red[threadIdx.x + st];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = (accumulate ? out[0] : 0.f) + (float)(red[0] * scale);
}

// AvgPool1d(kernel, stride, padding) over (rows, t_in) -> (rows, t_out); count_include_pad selects
// the divisor policy (hifigan.py:788-792 uses True, melgan.py:409-414 False).
__global__ void avg_pool1d_kernel(const float* __restrict__ x, float* __restrict__ y, int rows, int t_in, int t_out,
                                  int k, int s, int pad, int include_pad) {
  const int r = blockIdx.y;
  const float* xr = x + (long long)r * t_in;
  for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < t_out; o += gridDim.x * blockDim.x) {
    const int start = o * s - pad;
    float acc = 0.f;
    int cnt = 0;
    for (int j = 0; j < k; ++j) {
      const int i = start + j;
      if (i >= 0 && i < t_in) {
        acc += xr[i];
        ++cnt;
      }
    }
    int div = cnt;
    if (include_pad) {  // window clipped to the padded extent [-pad, t_in + pad)
      const int hi = min(start + k, t_in + pad);
      div = hi - start;
    }
    y[(long long)r * t_out + o] = acc / (float)div;
  }
}

}  // namespace pwgb

using namespace pwgb;

extern "C" int pwgb_reduce_mean_forward(int mode, const float* x, const float* y, long long n, float c, float s,
                                        float weight, int accumulate, float* out, float* ws, int ws_floats,
                                        void* stream) {
  PWGB_CHECK_ARG(x && out && ws && ((mode != 1 && mode != 4) || y), "reduce_mean: null argument");
  PWGB_CHECK_ARG(mode >= 0 && mode <= 4 && n > 0 && ws_floats >= 1, "reduce_mean: bad arguments");
  long long blocks = (n + 2047) / 2048;
  if (blocks > ws_floats) blocks = ws_floats;
  if (blocks > 1024) blocks = 1024;
  cudaStream_t st = (cudaStream_t)stream;
  reduce_partial_kernel<<<(unsigned)blocks, 256, 0, st>>>(mode, x, y, n, c, s, ws);
  int rc = check_launch("reduce_partial_kernel");
  if (rc) return rc;
  reduce_final_kernel<<<1, 256, 0, st>>>(ws, (int)blocks, (double)weight / (double)n, accumulate, out);
  return check_launch("reduce_final_kernel");
}

extern "C" int pwgb_avg_pool1d_forward(const float* x, float* y, int rows, int t_in, int kernel, int stride,
                                       int padding, int count_include_pad, void* stream) {
  PWGB_CHECK_ARG(x && y && rows >= 0 && t_in > 0 && kernel > 0 && stride > 0 && padding >= 0 && padding <= kernel / 2,
                 "avg_pool1d: bad arguments");
  PWGB_UNSUPPORTED_IF(rows > 65535, "avg_pool1d: too many rows");
  if (rows == 0) return PWGB_OK;
  const int t_out = (t_in + 2 * padding - kernel) / stride + 1;
  PWGB_CHECK_ARG(t_out > 0, "avg_pool1d: input too short");
  dim3 grid(ceil_div(t_out, 256) < 64 ? ceil_div(t_out, 256) : 64, rows);
  avg_pool1d_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, y, rows, t_in, t_out, kernel, stride, padding,
                                                          count_include_pad);
  return check_launch("avg_pool1d_kernel");
}
