// Space-to-depth along time: turns a stride-s Conv1d (or the (k,1)-strided Conv2d of the period
// discriminators, hifigan.py:354-381) into a stride-1 conv with s x the input channels and ceil(K/s) taps
// -- the shape the tensor-core kernels take.  With k = s*j + r:
//   y[t] = sum_k w[k] x[s*t + k - pad] = sum_r sum_j w[s*j + r] xs_r[t + j],   xs_r[u] = x[s*u + r - pad].
// One HBM-bound gather pass (and its adjoint, also a gather: (row + pad) <-> (u, r) is a bijection).
#include "common.cuh"

namespace pwgb {

// x: (B, C, rows_in, P)   y: (B, C*s, rows_out, P); channel (g, r, cl) = g*s*Cg + r*Cg + cl
__global__ void s2d_forward_kernel(const float* __restrict__ x, float* __restrict__ y, int C, int Cg, int Cgo, long long rows_in, int P,
                                   int s, int pad, long long rows_out, long long total) {
  const int G = C / Cg;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long inner = rows_out * P;
    const long long f = i % inner;
    long long t = i / inner;
    const int ch = (int)(t % ((long long)G * Cgo));
    const long long b = t / ((long long)G * Cgo);
    const long long u = f / P;
    const int pp = (int)(f - u * P);
    const int g = ch / Cgo;
    const int rem = ch - g * Cgo;  // channels >= s * Cg of a group are zero padding (tensor-core channel granularity)
    const int r = rem / Cg, cl = rem - r * Cg;
    const long long row = (long long)s * u + r - pad;
    float v = 0.f;
    if (rem < s * Cg && row >= 0 && row < rows_in) v = __ldg(x + ((b * C + g * Cg + cl) * rows_in + row) * P + pp);
    y[i] = v;
  }
}

// gx: (B, C, rows_in, P) <- gy: (B, C*s, rows_out, P)
__global__ void s2d_backward_kernel(const float* __restrict__ gy, float* __restrict__ gx, int C, int Cg, int Cgo, long long rows_in, int P,
                                    int s, int pad, long long rows_out, long long total) {
  const int G = C / Cg;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long inner = rows_in * P;
    const long long f = i % inner;
    long long t = i / inner;
    const int c = (int)(t % C);
    const long long b = t / C;
    const long long row = f / P;
    const int pp = (int)(f - row * P);
    const long long q = row + pad;
    const long long u = q / s;
    const int r = (int)(q - u * s);
    const int g = c / Cg, cl = c - g * Cg;
    float v = 0.f;
    if (u < rows_out) v = __ldg(gy + ((b * G * Cgo + (long long)g * Cgo + (long long)r * Cg + cl) * rows_out + u) * P + pp);
    gx[i] = v;
  }
}

}  // namespace pwgb

using namespace pwgb;

static int s2d_args_ok(int batch, int channels, int groups, long long rows_in, int period, int stride, int pad_left, long long rows_out) {
  return batch >= 0 && channels > 0 && groups > 0 && channels % groups == 0 && rows_in > 0 && period > 0 && stride > 0 && pad_left >= 0 &&
         rows_out > 0;
}

extern "C" int pwgb_s2d_forward(const float* x, float* y, int batch, int channels, int groups, long long rows_in, int period, int stride,
                                int pad_left, long long rows_out, int group_channels_out, void* stream) {
  PWGB_CHECK_ARG(x && y && s2d_args_ok(batch, channels, groups, rows_in, period, stride, pad_left, rows_out), "s2d_forward: bad argument");
  const int cgo = group_channels_out > 0 ? group_channels_out : channels / groups * stride;
  PWGB_CHECK_ARG(cgo >= channels / groups * stride, "s2d_forward: group_channels_out smaller than stride * channels per group");
  const long long total = (long long)batch * groups * cgo * rows_out * period;
  if (total == 0) return PWGB_OK;
  int blocks = (int)((total + 255) / 256 > 132 * 16 ? 132 * 16 : (total + 255) / 256);
  s2d_forward_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, y, channels, channels / groups, cgo, rows_in, period, stride, pad_left,
                                                             rows_out, total);
  return check_launch("s2d_forward_kernel");
}

extern "C" int pwgb_s2d_backward(const float* gy, float* gx, int batch, int channels, int groups, long long rows_in, int period, int stride,
                                 int pad_left, long long rows_out, int group_channels_out, void* stream) {
  PWGB_CHECK_ARG(gy && gx && s2d_args_ok(batch, channels, groups, rows_in, period, stride, pad_left, rows_out), "s2d_backward: bad argument");
  const int cgo = group_channels_out > 0 ? group_channels_out : channels / groups * stride;
  PWGB_CHECK_ARG(cgo >= channels / groups * stride, "s2d_backward: group_channels_out smaller than stride * channels per group");
  const long long total = (long long)batch * channels * rows_in * period;
  if (total == 0) return PWGB_OK;
  int blocks = (int)((total + 255) / 256 > 132 * 16 ? 132 * 16 : (total + 255) / 256);
  s2d_backward_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(gy, gx, channels, channels / groups, cgo, rows_in, period, stride, pad_left,
                                                              rows_out, total);
  return check_launch("s2d_backward_kernel");
}
