// StyleMelGAN generator glue around the conv kernels (layers/tade_res_block.py, models/style_melgan.py):
// InstanceNorm1d, nearest-neighbour upsampling, the TADE modulation  y = cg1 * up(x) + cg2  and the
// softmax / sigmoid gated activation with the block's residual.  All are HBM-bound element / row kernels
// (the heavy work of a TADEResBlock is its six k=9 convs, which run on conv1d_tc / conv1d_simt).
#include "common.cuh"

namespace pwgb {

static int grid_for(long long n) {
  long long b = (n + 255) / 256;
  if (b > 132LL * 16) b = 132LL * 16;
  return b < 1 ? 1 : (int)b;
}

// block-wide sum, result valid in every thread (fixed tree: deterministic)
__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();  // red[] may still be read from the previous call
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float s = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += red[i];
  return s;
}

// torch.nn.InstanceNorm1d(C) (tade_res_block.py:26): per (batch, channel) row, biased variance, eps inside
// the square root, no affine.  `pre_slope` applies a LeakyReLU to the input first (the activation that ends
// StyleMelGANGenerator.noise_upsample feeds the first block's norm).  Two-pass variance (mean first).
__global__ void __launch_bounds__(256) instance_norm_kernel(const float* __restrict__ x, float* __restrict__ y, long long t,
                                                            float eps, float pre_slope) {
  __shared__ float red[8];
  const float* xr = x + (long long)blockIdx.x * t;
  float* yr = y + (long long)blockIdx.x * t;
  float s = 0.f;
  for (long long i = threadIdx.x; i < t; i += 256) s += lrelu(xr[i], pre_slope);
  const float mean = block_sum(s, red) / (float)t;
  float q = 0.f;
  for (long long i = threadIdx.x; i < t; i += 256) {
    const float d = lrelu(xr[i], pre_slope) - mean;
    q = fmaf(d, d, q);
  }
  const float rstd = rsqrtf(block_sum(q, red) / (float)t + eps);
  for (long long i = threadIdx.x; i < t; i += 256) yr[i] = (lrelu(xr[i], pre_slope) - mean) * rstd;
}

// torch.nn.Upsample(scale_factor=s, mode="nearest") on (rows, t_in): y[r, o] = x[r, o / s]
__global__ void upsample_nearest_kernel(const float* __restrict__ x, float* __restrict__ y, long long rows, long long t_in,
                                        int scale) {
  const long long t_out = t_in * scale, n = rows * t_out;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / t_out, o = i - r * t_out;
    y[i] = x[r * t_in + o / scale];
  }
}

__global__ void leaky_relu_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, float slope) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = lrelu(x[i], slope);
}

// TADELayer.forward tail (tade_res_block.py:72-74): cg (B, 2C, T), xn (B, C, T / scale):
//   y[b, c, o] = cg[b, c, o] * xn[b, c, o / scale] + cg[b, C + c, o]
__global__ void tade_combine_kernel(const float* __restrict__ cg, const float* __restrict__ xn, float* __restrict__ y, int B,
                                    int C, long long t_out, int scale) {
  const long long n = (long long)B * C * t_out, t_in = t_out / scale;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long o = i % t_out;
    const long long bc = i / t_out;
    const long long b = bc / C, c = bc - b * C;
    const float* g = cg + ((b * 2 * C + c) * t_out + o);
    y[i] = g[0] * xn[bc * t_in + o / scale] + g[(long long)C * t_out];
  }
}

// TADEResBlock gated activation (tade_res_block.py:150-159): x (B, 2C, T) = [xa | xb];
//   y[b, c, t] = gate(xa)[b, c, t] * tanh(xb[b, c, t]) + (residual ? residual[b, c, t / scale] : 0)
// gate = softmax over the C channels of one (b, t) column, or sigmoid.  One thread per column: loads are
// coalesced across the warp (consecutive t), the three channel sweeps hit L1/L2.
__global__ void tade_gate_kernel(const float* __restrict__ x, const float* __restrict__ residual, float* __restrict__ y,
                                 int B, int C, long long t, int scale, int softmax) {
  const long long n = (long long)B * t, t_res = t / scale;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / t, tt = i - b * t;
    const float* xa = x + (b * 2 * C) * t + tt;
    const float* xb = xa + (long long)C * t;
    float* yo = y + (b * C) * t + tt;
    const float* rr = residual ? residual + (b * C) * t_res + tt / scale : nullptr;
    float mx = 0.f, inv = 1.f;
    if (softmax) {
      mx = xa[0];
      for (int c = 1; c < C; ++c) mx = fmaxf(mx, xa[(long long)c * t]);
      float s = 0.f;
      for (int c = 0; c < C; ++c) s += expf(xa[(long long)c * t] - mx);
      inv = 1.f / s;
    }
    for (int c = 0; c < C; ++c) {
      const float a = xa[(long long)c * t];
      const float g = softmax ? expf(a - mx) * inv : 1.f / (1.f + expf(-a));
      float v = g * tanhf(xb[(long long)c * t]);
      if (rr) v += rr[(long long)c * t_res];
      yo[(long long)c * t] = v;
    }
  }
}

// ------------------------------------------------------------------ adjoints (StyleMelGAN generator training)
// InstanceNorm1d backward: a = lrelu(x), yh = (a - mean) * rstd;  ga = rstd * (gy - mean(gy) - yh * mean(gy * yh));
// gx = ga * lrelu'(x).  Statistics are recomputed from x (two-pass variance, like the forward).
__global__ void __launch_bounds__(256) instance_norm_backward_kernel(const float* __restrict__ x, const float* __restrict__ gy,
                                                                     float* __restrict__ gx, long long t, float eps,
                                                                     float pre_slope) {
  __shared__ float red[8];
  const float* xr = x + (long long)blockIdx.x * t;
  const float* gr = gy + (long long)blockIdx.x * t;
  float* or_ = gx + (long long)blockIdx.x * t;
  float s = 0.f;
  for (long long i = threadIdx.x; i < t; i += 256) s += lrelu(xr[i], pre_slope);
  const float mean = block_sum(s, red) / (float)t;
  float q = 0.f;
  for (long long i = threadIdx.x; i < t; i += 256) {
    const float d = lrelu(xr[i], pre_slope) - mean;
    q = fmaf(d, d, q);
  }
  const float rstd = rsqrtf(block_sum(q, red) / (float)t + eps);
  float s1 = 0.f, s2 = 0.f;
  for (long long i = threadIdx.x; i < t; i += 256) {
    const float g = gr[i];
    s1 += g;
    s2 = fmaf(g, (lrelu(xr[i], pre_slope) - mean) * rstd, s2);
  }
  const float m1 = block_sum(s1, red) / (float)t;
  const float m2 = block_sum(s2, red) / (float)t;
  for (long long i = threadIdx.x; i < t; i += 256) {
    const float xv = xr[i];
    const float yh = (lrelu(xv, pre_slope) - mean) * rstd;
    const float ga = rstd * (gr[i] - m1 - yh * m2);
    or_[i] = ga * (xv > 0.f ? 1.f : pre_slope);
  }
}

// nearest-upsampling backward: gx[r, i] = sum_{j < s} gy[r, i * s + j]
__global__ void upsample_nearest_backward_kernel(const float* __restrict__ gy, float* __restrict__ gx, long long rows,
                                                 long long t_in, int scale) {
  const long long n = rows * t_in;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float* g = gy + i * scale;
    float a = 0.f;
    for (int j = 0; j < scale; ++j) a += g[j];
    gx[i] = a;
  }
}

// TADE modulation backward: gcg[:, :C] = gy * up(xn), gcg[:, C:] = gy, gxn[i] = sum_j gy[i s + j] * cg[:, :C][i s + j]
__global__ void tade_combine_backward_kernel(const float* __restrict__ cg, const float* __restrict__ xn,
                                             const float* __restrict__ gy, float* __restrict__ gcg, float* __restrict__ gxn,
                                             int B, int C, long long t_out, int scale) {
  const long long t_in = t_out / scale, n = (long long)B * C * t_in;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long ti = i % t_in;
    const long long bc = i / t_in;
    const long long b = bc / C, c = bc - b * C;
    const long long base = (b * 2 * C + c) * t_out + ti * scale;
    const float xv = xn[i];
    const float* g = gy + bc * t_out + ti * scale;
    float a = 0.f;
    for (int j = 0; j < scale; ++j) {
      const float gv = g[j];
      a = fmaf(gv, cg[base + j], a);
      gcg[base + j] = gv * xv;
      gcg[base + (long long)C * t_out + j] = gv;
    }
    gxn[i] = a;
  }
}

// gated activation backward, one thread per (b, t) column: u_c = gy_c tanh(xb_c);
//   softmax: gxa_c = g_c (u_c - sum_c' g_c' u_c'),  sigmoid: gxa_c = u_c g_c (1 - g_c);  gxb_c = gy_c g_c (1 - tanh^2)
__global__ void tade_gate_backward_kernel(const float* __restrict__ x, const float* __restrict__ gy, float* __restrict__ gx,
                                          int B, int C, long long t, int softmax) {
  const long long n = (long long)B * t;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / t, tt = i - b * t;
    const float* xa = x + (b * 2 * C) * t + tt;
    const float* xb = xa + (long long)C * t;
    const float* g = gy + (b * C) * t + tt;
    float* ga = gx + (b * 2 * C) * t + tt;
    float* gb = ga + (long long)C * t;
    float mx = 0.f, inv = 1.f, dot = 0.f;
    if (softmax) {
      mx = xa[0];
      for (int c = 1; c < C; ++c) mx = fmaxf(mx, xa[(long long)c * t]);
      float s = 0.f;
      for (int c = 0; c < C; ++c) s += expf(xa[(long long)c * t] - mx);
      inv = 1.f / s;
      for (int c = 0; c < C; ++c)
        dot = fmaf(expf(xa[(long long)c * t] - mx) * inv, g[(long long)c * t] * tanhf(xb[(long long)c * t]), dot);
    }
    for (int c = 0; c < C; ++c) {
      const float a = xa[(long long)c * t];
      const float gt = softmax ? expf(a - mx) * inv : 1.f / (1.f + expf(-a));
      const float th = tanhf(xb[(long long)c * t]);
      const float gv = g[(long long)c * t];
      const float u = gv * th;
      ga[(long long)c * t] = softmax ? gt * (u - dot) : u * gt * (1.f - gt);
      gb[(long long)c * t] = gv * gt * (1.f - th * th);
    }
  }
}

}  // namespace pwgb

using namespace pwgb;

extern "C" int pwgb_instance_norm_forward(const float* x, float* y, long long rows, long long t, float eps, float pre_slope,
                                          void* stream) {
  PWGB_CHECK_ARG(x && y && rows >= 0 && t > 0 && eps >= 0.f, "instance_norm: bad arguments");
  PWGB_CHECK_ARG(rows <= 0x7fffffffLL, "instance_norm: too many rows");
  if (rows == 0) return PWGB_OK;
  instance_norm_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(x, y, t, eps, pre_slope);
  return check_launch("instance_norm_kernel");
}

extern "C" int pwgb_upsample_nearest_forward(const float* x, float* y, long long rows, long long t_in, int scale,
                                             void* stream) {
  PWGB_CHECK_ARG(x && y && rows >= 0 && t_in >= 0 && scale >= 1, "upsample_nearest: bad arguments");
  const long long n = rows * t_in * scale;
  if (n == 0) return PWGB_OK;
  upsample_nearest_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(x, y, rows, t_in, scale);
  return check_launch("upsample_nearest_kernel");
}

extern "C" int pwgb_leaky_relu_forward(const float* x, float* y, long long n, float slope, void* stream) {
  PWGB_CHECK_ARG(x && y && n >= 0, "leaky_relu: bad arguments");
  if (n == 0) return PWGB_OK;
  leaky_relu_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(x, y, n, slope);
  return check_launch("leaky_relu_kernel");
}

extern "C" int pwgb_tade_combine_forward(const float* cg, const float* xn, float* y, int batch, int channels, long long t_out,
                                         int scale, void* stream) {
  PWGB_CHECK_ARG(cg && xn && y && batch >= 0 && channels > 0 && t_out >= 0 && scale >= 1 && t_out % scale == 0,
                 "tade_combine: bad arguments (t_out must be a multiple of scale)");
  const long long n = (long long)batch * channels * t_out;
  if (n == 0) return PWGB_OK;
  tade_combine_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(cg, xn, y, batch, channels, t_out, scale);
  return check_launch("tade_combine_kernel");
}

extern "C" int pwgb_tade_gate_forward(const float* x, const float* residual, float* y, int batch, int channels, long long t,
                                      int scale, int softmax, void* stream) {
  PWGB_CHECK_ARG(x && y && batch >= 0 && channels > 0 && t >= 0 && scale >= 1 && t % scale == 0,
                 "tade_gate: bad arguments (t must be a multiple of scale)");
  const long long n = (long long)batch * t;
  if (n == 0) return PWGB_OK;
  tade_gate_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(x, residual, y, batch, channels, t, scale, softmax ? 1 : 0);
  return check_launch("tade_gate_kernel");
}

extern "C" int pwgb_instance_norm_backward(const float* x, const float* gy, float* gx, long long rows, long long t, float eps,
                                           float pre_slope, void* stream) {
  PWGB_CHECK_ARG(x && gy && gx && rows >= 0 && t > 0 && eps >= 0.f, "instance_norm_backward: bad arguments");
  PWGB_CHECK_ARG(rows <= 0x7fffffffLL, "instance_norm_backward: too many rows");
  if (rows == 0) return PWGB_OK;
  instance_norm_backward_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(x, gy, gx, t, eps, pre_slope);
  return check_launch("instance_norm_backward_kernel");
}

extern "C" int pwgb_upsample_nearest_backward(const float* gy, float* gx, long long rows, long long t_in, int scale, void* stream) {
  PWGB_CHECK_ARG(gy && gx && rows >= 0 && t_in >= 0 && scale >= 1, "upsample_nearest_backward: bad arguments");
  const long long n = rows * t_in;
  if (n == 0) return PWGB_OK;
  upsample_nearest_backward_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(gy, gx, rows, t_in, scale);
  return check_launch("upsample_nearest_backward_kernel");
}

extern "C" int pwgb_tade_combine_backward(const float* cg, const float* xn, const float* gy, float* gcg, float* gxn, int batch,
                                          int channels, long long t_out, int scale, void* stream) {
  PWGB_CHECK_ARG(cg && xn && gy && gcg && gxn && batch >= 0 && channels > 0 && t_out >= 0 && scale >= 1 && t_out % scale == 0,
                 "tade_combine_backward: bad arguments (t_out must be a multiple of scale)");
  const long long n = (long long)batch * channels * (t_out / scale);
  if (n == 0) return PWGB_OK;
  tade_combine_backward_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(cg, xn, gy, gcg, gxn, batch, channels, t_out, scale);
  return check_launch("tade_combine_backward_kernel");
}

extern "C" int pwgb_tade_gate_backward(const float* x, const float* gy, float* gx, int batch, int channels, long long t,
                                       int softmax, void* stream) {
  PWGB_CHECK_ARG(x && gy && gx && batch >= 0 && channels > 0 && t >= 0, "tade_gate_backward: bad arguments");
  const long long n = (long long)batch * t;
  if (n == 0) return PWGB_OK;
  tade_gate_backward_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(x, gy, gx, batch, channels, t, softmax ? 1 : 0);
  return check_launch("tade_gate_backward_kernel");
}
