// ConvTranspose1d as a poly-phase convolution: a stride-s transposed conv with K taps is
// s interleaved ordinary convs with ceil(K/s) taps each (no zero stuffing).  The weight is
// re-laid out on device to the virtual conv  (cout*s, cin, M)  and the generic conv kernel
// writes through a pixel-shuffle epilogue  o = i*s + phase - padding.
#include "common.cuh"
#include "tc_common.cuh"

namespace pwgb {

int conv1d_forward_simt(const pwgb_conv1d_desc* d, const float* x, const float* w, const float* bias,
                        const float* residual, float* y, cudaStream_t st);
int conv1d_tc_chunk(const pwgb_conv1d_desc* d, int co_off, int cout_total, const float* x, const void* packed_w,
                    const float* bias, float* y, cudaStream_t st, int nco);
int conv1d_tc_plan_ok(const pwgb_conv1d_desc* d);
void tc_pack_weight(const float* w, int cin, int cout, int kernel, void* packed, cudaStream_t st);

// w: (cin, cout/groups, K) -> wv: (cout*s, cin/groups, M),
// wv[co*s+ph][ci_l][m'] = w[g*cin_g + ci_l][co_l][ph + (M-1-m')*s]   (co = g*cout_g + co_l)
__global__ void convtr_weight_kernel(const float* __restrict__ w, float* __restrict__ wv, int cin, int cout, int K,
                                     int s, int M, int groups) {
  const int cin_g = cin / groups, cout_g = cout / groups;
  const long long n = (long long)cout * s * cin_g * M;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int m = (int)(i % M);
    long long t = i / M;
    int ci_l = (int)(t % cin_g);
    int cv = (int)(t / cin_g);
    int co = cv / s, ph = cv - co * s;
    int g = co / cout_g, co_l = co - g * cout_g;
    int k = ph + (M - 1 - m) * s;
    wv[i] = k < K ? w[((long long)(g * cin_g + ci_l) * cout_g + co_l) * K + k] : 0.f;
  }
}

}  // namespace pwgb

using namespace pwgb;

extern "C" size_t pwgb_conv_transpose1d_workspace(const pwgb_convtr1d_desc* d) {
  if (!d || d->stride <= 0) return 0;
  const int M = ceil_div(d->kernel, d->stride);
  // [virtual-conv fp32 weights][bf16 hi/lo operand image of the same weights for the tensor-core path]
  const int G = d->groups > 1 ? d->groups : 1;
  return 2 * (size_t)d->cout * d->stride * (d->cin / G) * M * sizeof(float);
}

extern "C" int pwgb_conv_transpose1d_forward(const pwgb_convtr1d_desc* d, const float* x, const float* w,
                                             const float* bias, float* y, void* ws, size_t ws_bytes, void* stream) {
  PWGB_CHECK_ARG(d && x && w && y, "conv_transpose1d: null argument");
  PWGB_CHECK_ARG(d->batch >= 0 && d->cin > 0 && d->cout > 0 && d->t_in > 0 && d->kernel > 0 && d->stride > 0 &&
                     d->padding >= 0,
                 "conv_transpose1d: bad descriptor");
  const int s = d->stride, K = d->kernel, M = ceil_div(K, s);
  const int G = d->groups > 1 ? d->groups : 1, P = d->period > 1 ? d->period : 1;
  PWGB_CHECK_ARG(d->cin % G == 0 && d->cout % G == 0, "conv_transpose1d: channels not divisible by groups");
  const int op = d->t_out - ((d->t_in - 1) * s - 2 * d->padding + K);
  PWGB_CHECK_ARG(op >= 0 && op < s, "conv_transpose1d: t_out=%d inconsistent with t_in=%d k=%d s=%d p=%d", d->t_out,
                 d->t_in, K, s, d->padding);
  const size_t need = pwgb_conv_transpose1d_workspace(d);
  PWGB_CHECK_ARG(ws && ws_bytes >= need, "conv_transpose1d: workspace too small (%zu < %zu)", ws_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  float* wv = (float*)ws;
  const long long n = (long long)d->cout * s * (d->cin / G) * M;
  int blocks = (int)((n + 255) / 256);
  if (blocks > 4096) blocks = 4096;
  convtr_weight_kernel<<<blocks, 256, 0, st>>>(w, wv, d->cin, d->cout, K, s, M, G);
  int rc = check_launch("convtr_weight_kernel");
  if (rc) return rc;
  pwgb_conv1d_desc c = {};
  c.batch = d->batch;
  c.cin = d->cin;
  c.cout = d->cout * s;
  c.t_in = d->t_in;
  c.t_out = (d->t_out - 1 + d->padding) / s + 1;
  c.kernel = M;
  c.stride = 1;
  c.dilation = 1;
  c.groups = G;
  c.pad_left = M - 1;
  c.pad_mode = PWGB_PAD_ZERO;
  c.period = P;
  c.t_valid = d->t_in * P;
  c.pre_slope = d->pre_slope;
  c.post_act = PWGB_ACT_NONE;
  c.out_scale = 1.f;
  c.shuffle = s;
  c.shuffle_pad = d->padding;
  c.shuffle_tout = d->t_out;
  // tensor-core path: N (= cout*s virtual channels) in chunks of <= TC_NMAX accumulator columns
  if (G == 1 && P == 1 && d->cin % 32 == 0 && c.cout % 16 == 0) {
    int chunk = c.cout;
    if (chunk > TC_NMAX) {
      chunk = TC_NMAX;
      while (c.cout % chunk) chunk -= 16;
    }
    pwgb_conv1d_desc cc = c;
    cc.cout = chunk;
    if (conv1d_tc_plan_ok(&cc)) {
      unsigned char* pk = (unsigned char*)ws + need / 2;
      // the operand image is laid out per (32-channel chunk, tap) over the rows of ONE launch, so
      // each column chunk gets its own image
      for (int co = 0; co < c.cout; co += chunk) {
        unsigned char* pkc = pk + (size_t)co * d->cin * M * sizeof(float);
        tc_pack_weight(wv + (size_t)co * d->cin * M, d->cin, chunk, M, pkc, st);
        rc = check_launch("tc_pack_weight_kernel");
        if (rc) return rc;
      }
      return conv1d_tc_chunk(&cc, 0, c.cout, x, pk, bias, y, st, c.cout / chunk);
    }
  }
  return conv1d_forward_simt(&c, x, wv, bias, nullptr, y, st);
}
