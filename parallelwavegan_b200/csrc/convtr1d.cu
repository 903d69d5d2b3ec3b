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
                    const float* bias, float* y, cudaStream_t st, int nco, const float* x2 = nullptr, int cin1 = 0,
                    const float* hist = nullptr, const int* rep = nullptr, int hist_len = 0,
                    const pwgb_stream_ext* ext = nullptr);
int conv1d_stream_simt(const pwgb_conv1d_desc* d, const float* x, const float* hist, int hist_len, const int* rep,
                       const float* w, const float* bias, const float* residual, float* y, cudaStream_t st,
                       const int* zero_flag = nullptr, int zero_rows = 0, const pwgb_stream_ext* ext = nullptr);
int conv1d_tc_plan_ok(const pwgb_conv1d_desc* d, int* raw_staged = nullptr);
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

// The [history | chunk] window of cat(x1, x2) for a two-source stream conv-transpose: xw (B, cin1 + cin2, n), hw (B,
// cin1 + cin2, 1).  Source 1 row j is x1 row j (row -1: hist1); source 2 row j is row j - delay2 of [hist2 | x2].
__global__ void convtr_cat_window_kernel(const float* __restrict__ x1, const float* __restrict__ hist1, const float* __restrict__ x2,
                                         const float* __restrict__ hist2, int hist2_len, int delay2, float* __restrict__ xw,
                                         float* __restrict__ hw, int cin1, int cin, int n, long long total) {
  const int cin2 = cin - cin1;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(i % (n + 1)) - 1;  // row of the chunk, -1 the history frame
    const long long t = i / (n + 1);
    const int c = (int)(t % cin);
    const long long b = t / cin;
    float v;
    if (c < cin1) {
      v = j < 0 ? __ldg(hist1 + b * cin1 + c) : __ldg(x1 + (b * cin1 + c) * n + j);
    } else {
      const int c2 = c - cin1, r = j - delay2;
      v = r >= 0 ? __ldg(x2 + (b * cin2 + c2) * n + r) : __ldg(hist2 + (b * cin2 + c2) * hist2_len + (hist2_len + r));
    }
    if (j < 0)
      hw[b * cin + c] = v;
    else
      xw[(b * cin + c) * n + j] = v;
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

static int convtr_desc_ok(const pwgb_convtr1d_desc* d) {
  PWGB_CHECK_ARG(d->batch >= 0 && d->cin > 0 && d->cout > 0 && d->t_in > 0 && d->kernel > 0 && d->stride > 0 &&
                     d->padding >= 0,
                 "conv_transpose1d: bad descriptor");
  const int G = d->groups > 1 ? d->groups : 1;
  PWGB_CHECK_ARG(d->cin % G == 0 && d->cout % G == 0, "conv_transpose1d: channels not divisible by groups");
  const int op = d->t_out - ((d->t_in - 1) * d->stride - 2 * d->padding + d->kernel);
  PWGB_CHECK_ARG(op >= 0 && op < d->stride, "conv_transpose1d: t_out=%d inconsistent with t_in=%d k=%d s=%d p=%d", d->t_out,
                 d->t_in, d->kernel, d->stride, d->padding);
  return PWGB_OK;
}

// The virtual stride-1 conv (cout*s channels, ceil(K/s) taps) that the conv-transpose lowers to
static pwgb_conv1d_desc convtr_virtual_desc(const pwgb_convtr1d_desc* d) {
  const int s = d->stride, M = ceil_div(d->kernel, s);
  const int P = d->period > 1 ? d->period : 1;
  pwgb_conv1d_desc c = {};
  c.batch = d->batch;
  c.cin = d->cin;
  c.cout = d->cout * s;
  c.t_in = d->t_in;
  c.t_out = (d->t_out - 1 + d->padding) / s + 1;
  c.kernel = M;
  c.stride = 1;
  c.dilation = 1;
  c.groups = d->groups > 1 ? d->groups : 1;
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
  return c;
}

// Tensor-core path: N (= cout*s virtual channels) in chunks of <= TC_NMAX accumulator columns.  Returns the chunk
// width, or 0 when the conv-transpose runs on the FFMA kernel (or, for a two-source input, cannot take it).
static int convtr_tc_chunk(const pwgb_conv1d_desc& c, bool two_source) {
  if (c.groups != 1 || c.period != 1 || c.cin % 32 != 0 || c.cout % 16 != 0) return 0;
  int chunk = c.cout;
  if (chunk > TC_NMAX) {
    chunk = TC_NMAX;
    while (c.cout % chunk) chunk -= 16;
  }
  pwgb_conv1d_desc cc = c;
  cc.cout = chunk;
  int raw_staged = 0;
  if (!conv1d_tc_plan_ok(&cc, &raw_staged) || (two_source && !raw_staged)) return 0;
  return chunk;
}

// x2 / cin1: the second source of a two-source input (cin1 > 0 only on the tensor-core path).  hist_mode: d describes the
// conv-transpose on cat(h, x) along time, x holds its last t_in - 1 frames and frame 0 is hist[b] (or x[b, :, 0] where
// rep[b] is set): the virtual conv runs on x with that frame as a one-row history.
static int convtr_forward(const pwgb_convtr1d_desc* d, const float* x, const float* x2, int cin1, const float* w,
                          const float* bias, float* y, void* ws, size_t ws_bytes, void* stream, bool hist_mode = false,
                          const float* hist = nullptr, const int* rep = nullptr, const pwgb_stream_ext* ext = nullptr) {
  const int s = d->stride, K = d->kernel, M = ceil_div(K, s);
  const int G = d->groups > 1 ? d->groups : 1;
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
  pwgb_conv1d_desc c = convtr_virtual_desc(d);
  if (hist_mode) {
    c.t_in -= 1;
    c.t_valid = c.t_in;
    c.pad_left += 1;
    c.pad_mode = PWGB_PAD_HISTORY;
  }
  const int chunk = convtr_tc_chunk(c, cin1 > 0);
  if (chunk) {
    pwgb_conv1d_desc cc = c;
    cc.cout = chunk;
    unsigned char* pk = (unsigned char*)ws + need / 2;
    // the operand image is laid out per (32-channel chunk, tap) over the rows of ONE launch, so
    // each column chunk gets its own image
    for (int co = 0; co < c.cout; co += chunk) {
      unsigned char* pkc = pk + (size_t)co * d->cin * M * sizeof(float);
      tc_pack_weight(wv + (size_t)co * d->cin * M, d->cin, chunk, M, pkc, st);
      rc = check_launch("tc_pack_weight_kernel");
      if (rc) return rc;
    }
    if (hist_mode) return conv1d_tc_chunk(&cc, 0, c.cout, x, pk, bias, y, st, c.cout / chunk, nullptr, 0, hist, rep, 1, ext);
    return conv1d_tc_chunk(&cc, 0, c.cout, x, pk, bias, y, st, c.cout / chunk, x2, cin1);
  }
  if (hist_mode) return conv1d_stream_simt(&c, x, hist, 1, rep, wv, bias, nullptr, y, st, nullptr, 0, ext);
  if (cin1 > 0) {
    set_error("conv_transpose1d_cat: configuration not supported by the tensor-core path");
    return PWGB_UNSUPPORTED;
  }
  return conv1d_forward_simt(&c, x, wv, bias, nullptr, y, st);
}

extern "C" int pwgb_conv_transpose1d_forward(const pwgb_convtr1d_desc* d, const float* x, const float* w,
                                             const float* bias, float* y, void* ws, size_t ws_bytes, void* stream) {
  PWGB_CHECK_ARG(d && x && w && y, "conv_transpose1d: null argument");
  const int rc = convtr_desc_ok(d);
  if (rc) return rc;
  return convtr_forward(d, x, nullptr, 0, w, bias, y, ws, ws_bytes, stream);
}

extern "C" int pwgb_conv_transpose1d_cat_supported(const pwgb_convtr1d_desc* d, int cin1) {
  if (!d || d->batch < 0 || d->cin <= 0 || d->cout <= 0 || d->t_in <= 0 || d->kernel <= 0 || d->stride <= 0 || d->padding < 0)
    return 0;
  if (cin1 <= 0 || cin1 >= d->cin || cin1 % 32 != 0) return 0;
  const int op = d->t_out - ((d->t_in - 1) * d->stride - 2 * d->padding + d->kernel);
  if (op < 0 || op >= d->stride) return 0;
  return convtr_tc_chunk(convtr_virtual_desc(d), true) > 0;
}

extern "C" int pwgb_conv_transpose1d_cat_forward(const pwgb_convtr1d_desc* d, int cin1, const float* x1, const float* x2,
                                                 const float* w, const float* bias, float* y, void* ws, size_t ws_bytes,
                                                 void* stream) {
  PWGB_CHECK_ARG(d && x1 && x2 && w && y, "conv_transpose1d_cat: null argument");
  PWGB_UNSUPPORTED_IF(!pwgb_conv_transpose1d_cat_supported(d, cin1),
                      "conv_transpose1d_cat: configuration not supported by the two-source tensor-core path");
  return convtr_forward(d, x1, x2, cin1, w, bias, y, ws, ws_bytes, stream);
}

extern "C" int pwgb_conv_transpose1d_stream_forward(const pwgb_convtr1d_desc* d, const float* x, const float* hist,
                                                    const int* replicate, const float* w, const float* bias, float* y, void* ws,
                                                    size_t ws_bytes, void* stream) {
  PWGB_CHECK_ARG(d && x && hist && w && y, "conv_transpose1d_stream: null argument");
  const int rc = convtr_desc_ok(d);
  if (rc) return rc;
  PWGB_CHECK_ARG(d->t_in >= 2, "conv_transpose1d_stream: t_in counts the history frame and at least one input frame");
  PWGB_UNSUPPORTED_IF(d->groups > 1 || d->period > 1 || d->padding != d->stride,
                      "conv_transpose1d_stream: the causal conv-transpose is dense, plain and has padding == stride");
  return convtr_forward(d, x, nullptr, 0, w, bias, y, ws, ws_bytes, stream, true, hist, replicate);
}

extern "C" int pwgb_conv_transpose1d_stream_ext_forward(const pwgb_convtr1d_desc* d, const float* x, const float* hist,
                                                        const int* replicate, const float* w, const float* bias,
                                                        const pwgb_stream_ext* ext, float* y, void* ws, size_t ws_bytes,
                                                        void* stream) {
  PWGB_CHECK_ARG(d && x && hist && w && y, "conv_transpose1d_stream: null argument");
  const int rc = convtr_desc_ok(d);
  if (rc) return rc;
  PWGB_CHECK_ARG(d->t_in >= 2, "conv_transpose1d_stream: t_in counts the history frame and at least one input frame");
  PWGB_UNSUPPORTED_IF(d->groups > 1 || d->period > 1 || d->padding != d->stride,
                      "conv_transpose1d_stream: the stream conv-transpose is dense, plain and has padding == stride");
  if (const int rc2 = stream_ext_check(ext, nullptr)) return rc2;
  return convtr_forward(d, x, nullptr, 0, w, bias, y, ws, ws_bytes, stream, true, hist, replicate, ext);
}

// The window of virtual positions [T0, T0 + n) of the whole signal's virtual conv, all phases: the virtual conv runs on x
// (no rows with flush) with hist as its left history, and the pixel shuffle writes phase ph of position i to i * s + ph,
// which is whole-signal sample T0 * s - padding + that.  The generic FFMA kernel sums in the same order at any position.
extern "C" int pwgb_conv_transpose1d_window_stream_forward(const pwgb_convtr1d_desc* d, const float* x, const float* hist,
                                                           int hist_len, const int* fresh, int flush, const float* w,
                                                           const float* bias, float* y, void* ws, size_t ws_bytes,
                                                           void* stream) {
  PWGB_CHECK_ARG(d && (x || flush) && w && y && (hist || hist_len == 0), "conv_transpose1d_window_stream: null argument");
  PWGB_CHECK_ARG(d->batch >= 0 && d->cin > 0 && d->cout > 0 && d->t_in > 0 && d->kernel > 0 && d->stride > 0 && d->padding >= 0 &&
                     hist_len >= 0,
                 "conv_transpose1d_window_stream: bad descriptor");
  PWGB_CHECK_ARG((long long)d->t_out == (long long)d->t_in * d->stride,
                 "conv_transpose1d_window_stream: t_out (%d) must be t_in (%d) * stride (%d)", d->t_out, d->t_in, d->stride);
  PWGB_UNSUPPORTED_IF(d->groups > 1 || d->period > 1 || d->stride < 2,
                      "conv_transpose1d_window_stream: dense, plain conv-transposes of stride >= 2 only");
  const int s = d->stride, K = d->kernel, M = ceil_div(K, s);
  const size_t need = pwgb_conv_transpose1d_workspace(d);
  PWGB_CHECK_ARG(ws && ws_bytes >= need, "conv_transpose1d_window_stream: workspace too small (%zu < %zu)", ws_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  float* wv = (float*)ws;
  const long long n = (long long)d->cout * s * d->cin * M;
  int blocks = (int)((n + 255) / 256);
  if (blocks > 4096) blocks = 4096;
  convtr_weight_kernel<<<blocks, 256, 0, st>>>(w, wv, d->cin, d->cout, K, s, M, 1);
  if (const int rc = check_launch("convtr_weight_kernel")) return rc;
  pwgb_conv1d_desc c = {};
  c.batch = d->batch;
  c.cin = d->cin;
  c.cout = d->cout * s;
  c.t_in = flush ? 0 : d->t_in;  // a flush reads no input row: every row of the chunk is zero
  c.t_out = d->t_in;
  c.kernel = M;
  c.stride = 1;
  c.dilation = 1;
  c.groups = 1;
  c.pad_left = M - 1;
  c.pad_mode = PWGB_PAD_HISTORY;
  c.period = 1;
  c.t_valid = c.t_in;
  c.pre_slope = d->pre_slope;
  c.post_act = PWGB_ACT_NONE;
  c.out_scale = 1.f;
  c.shuffle = s;
  c.shuffle_pad = 0;
  c.shuffle_tout = d->t_out;
  return conv1d_stream_simt(&c, x, hist, hist_len, nullptr, wv, bias, nullptr, y, st, fresh, d->padding);
}

// the window buffers follow the conv-transpose's own workspace, 256-byte aligned
static size_t convtr_cat_window_offset(const pwgb_convtr1d_desc* d) { return (pwgb_conv_transpose1d_workspace(d) + 255) / 256 * 256; }

extern "C" size_t pwgb_conv_transpose1d_cat_stream_workspace(const pwgb_convtr1d_desc* d) {
  if (!d || d->stride <= 0 || d->batch < 0 || d->cin <= 0 || d->t_in <= 0) return 0;
  return convtr_cat_window_offset(d) + (size_t)d->batch * d->cin * d->t_in * sizeof(float);
}

extern "C" int pwgb_conv_transpose1d_cat_stream_ext_forward(const pwgb_convtr1d_desc* d, int cin1, const float* x1, const float* hist1,
                                                            const float* x2, const float* hist2, int hist2_len, int delay2,
                                                            const float* w, const float* bias, const pwgb_stream_ext* ext, float* y,
                                                            void* ws, size_t ws_bytes, void* stream) {
  PWGB_CHECK_ARG(d && x1 && hist1 && x2 && hist2 && w && y, "conv_transpose1d_cat_stream: null argument");
  const int rc = convtr_desc_ok(d);
  if (rc) return rc;
  PWGB_CHECK_ARG(d->t_in >= 2, "conv_transpose1d_cat_stream: t_in counts the history frame and at least one input frame");
  PWGB_UNSUPPORTED_IF(d->groups > 1 || d->period > 1 || d->padding != d->stride,
                      "conv_transpose1d_cat_stream: the stream conv-transpose is dense, plain and has padding == stride");
  PWGB_CHECK_ARG(cin1 > 0 && cin1 < d->cin, "conv_transpose1d_cat_stream: cin1 %d outside (0, %d)", cin1, d->cin);
  PWGB_CHECK_ARG(delay2 >= 0 && hist2_len >= delay2 + 1, "conv_transpose1d_cat_stream: source 2 needs delay2 + 1 history rows (delay2 %d, "
                 "hist2_len %d)", delay2, hist2_len);
  const size_t need = pwgb_conv_transpose1d_cat_stream_workspace(d);
  PWGB_CHECK_ARG(ws && ws_bytes >= need, "conv_transpose1d_cat_stream: workspace too small (%zu < %zu)", ws_bytes, need);
  if (const int rc2 = stream_ext_check(ext, nullptr)) return rc2;
  if (d->batch == 0) return PWGB_OK;
  const int n = d->t_in - 1;
  float* xw = (float*)((unsigned char*)ws + convtr_cat_window_offset(d));
  float* hw = xw + (size_t)d->batch * d->cin * n;
  const long long total = (long long)d->batch * d->cin * (n + 1);
  const int blocks = (int)((total + 255) / 256 < 4096 ? (total + 255) / 256 : 4096);
  convtr_cat_window_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x1, hist1, x2, hist2, hist2_len, delay2, xw, hw, cin1, d->cin, n,
                                                                      total);
  if (const int rc3 = check_launch("convtr_cat_window_kernel")) return rc3;
  // the single-source stream conv-transpose on the gathered window: pwgb_conv_transpose1d_cat_forward is bit-identical to
  // the single-source entry on the concatenation, so this is too
  return convtr_forward(d, xw, nullptr, 0, w, bias, y, ws, pwgb_conv_transpose1d_workspace(d), stream, true, hw, nullptr, ext);
}
