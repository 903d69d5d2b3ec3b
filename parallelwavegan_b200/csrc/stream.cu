// Streaming a causal conv stack chunk by chunk: the history conv entry point of the FFMA engine, the argument check both
// engines share, and the multi-tensor history carry.
#include "common.cuh"

namespace pwgb {

int conv1d_stream_simt(const pwgb_conv1d_desc* d, const float* x, const float* hist, int hist_len, const int* rep,
                       const float* w, const float* bias, const float* residual, float* y, cudaStream_t st,
                       const int* zero_flag = nullptr, int zero_rows = 0, const pwgb_stream_ext* ext = nullptr);

int stream_ext_check(const pwgb_stream_ext* e, const float* residual, int pad_mode) {
  if (!e) return PWGB_OK;
  PWGB_CHECK_ARG(e->edge == PWGB_PAD_ZERO || e->edge == PWGB_PAD_REFLECT || e->edge == PWGB_PAD_REPLICATE,
                 "stream_ext: edge must be PWGB_PAD_ZERO, PWGB_PAD_REFLECT or PWGB_PAD_REPLICATE (got %d)", e->edge);
  PWGB_CHECK_ARG(e->edge == PWGB_PAD_ZERO || pad_mode >= 0, "stream_ext: this entry point has no edge policy (edge must be 0)");
  PWGB_CHECK_ARG(e->edge == PWGB_PAD_ZERO || e->frame, "stream_ext: an edge policy needs the mask (frame and end)");
  PWGB_CHECK_ARG(e->edge == PWGB_PAD_ZERO || pad_mode == PWGB_PAD_HISTORY, "stream_ext: an edge policy needs pad_mode PWGB_PAD_HISTORY");
  PWGB_CHECK_ARG(e->in_lookahead >= 0, "stream_ext: in_lookahead must be >= 0 (got %d)", e->in_lookahead);
  PWGB_CHECK_ARG(!e->frame || (e->end && e->rate >= 1 && e->lookahead >= 0),
                 "stream_ext: a mask needs end flags, rate >= 1 and lookahead >= 0 (rate %d, lookahead %d)", e->rate, e->lookahead);
  PWGB_CHECK_ARG(e->res_hist_len >= 0 && e->res_delay >= 0 && e->res_delay <= e->res_hist_len &&
                     (e->res_hist_len == 0 || e->res_hist),
                 "stream_ext: bad residual history (res_hist_len %d, res_delay %d)", e->res_hist_len, e->res_delay);
  PWGB_CHECK_ARG(residual || e->res_hist_len == 0, "stream_ext: a residual history needs a residual");
  return PWGB_OK;
}

int conv1d_stream_check(const pwgb_conv1d_desc* d, const float* x, const float* hist, int hist_len, const float* y) {
  PWGB_CHECK_ARG(d && x && y, "conv1d_stream: null argument");
  PWGB_CHECK_ARG(d->batch >= 0 && d->cin > 0 && d->cout > 0 && d->t_in > 0 && d->t_out >= 0, "conv1d_stream: bad sizes");
  PWGB_CHECK_ARG(d->kernel > 0 && d->stride > 0 && d->dilation > 0 && d->groups > 0 && d->pad_left >= 0,
                 "conv1d_stream: bad kernel geometry");
  PWGB_CHECK_ARG(is_history_pad(d->pad_mode), "conv1d_stream: pad_mode must be PWGB_PAD_HISTORY or PWGB_PAD_HISTORY_REFLECT");
  PWGB_CHECK_ARG(hist_len >= 0 && (hist_len == 0 || hist), "conv1d_stream: bad history (hist_len %d)", hist_len);
  // a reflected row -t reads sample t <= pad_left of the chunk itself
  PWGB_CHECK_ARG(d->pad_mode != PWGB_PAD_HISTORY_REFLECT || (d->pad_left < d->t_in && hist_len <= d->pad_left),
                 "conv1d_stream: reflect needs pad_left (%d) < t_in (%d) and hist_len (%d) <= pad_left", d->pad_left, d->t_in,
                 hist_len);
  PWGB_CHECK_ARG(d->cin % d->groups == 0 && d->cout % d->groups == 0, "conv1d_stream: groups must divide cin and cout");
  PWGB_UNSUPPORTED_IF(d->stride != 1 || d->period > 1 || d->pre_gate || d->shuffle > 1,
                      "conv1d_stream: history padding serves plain stride-1 convs (period 1, no pre_gate, one source)");
  PWGB_UNSUPPORTED_IF(d->x_batch_stride || d->y_batch_stride || d->r_batch_stride || (d->t_valid > 0 && d->t_valid != d->t_in),
                      "conv1d_stream: strided or reflect-extended inputs are not supported");
  const long long need = (long long)(d->t_out - 1) + (long long)(d->kernel - 1) * d->dilation + 1 - d->pad_left;
  PWGB_CHECK_ARG(d->t_out == 0 || need <= (long long)d->t_in, "conv1d_stream: t_out too large for t_in");
  return PWGB_OK;
}

// The argument check of the two ragged entry points: h becomes the history descriptor (no history rows) whose EXT or EDGE
// launch computes the whole-signal conv d with each item's pad at its own end
int conv1d_ragged_check(const pwgb_conv1d_desc* d, const float* x, const pwgb_stream_ext* e, const float* y,
                        pwgb_conv1d_desc* h) {
  PWGB_CHECK_ARG(d && x && y && e, "conv1d_ragged: null argument");
  PWGB_CHECK_ARG(d->batch >= 0 && d->cin > 0 && d->cout > 0 && d->t_in > 0 && d->t_out >= 0, "conv1d_ragged: bad sizes");
  PWGB_CHECK_ARG(d->kernel > 0 && d->stride > 0 && d->dilation > 0 && d->groups > 0 && d->pad_left >= 0 &&
                     d->cin % d->groups == 0 && d->cout % d->groups == 0,
                 "conv1d_ragged: bad kernel geometry");
  PWGB_CHECK_ARG(d->pad_mode == PWGB_PAD_ZERO || d->pad_mode == PWGB_PAD_REFLECT || d->pad_mode == PWGB_PAD_REPLICATE,
                 "conv1d_ragged: pad_mode must be PWGB_PAD_ZERO, PWGB_PAD_REFLECT or PWGB_PAD_REPLICATE");
  PWGB_CHECK_ARG(e->frame && e->end && e->rate >= 1 && e->lookahead == 0,
                 "conv1d_ragged: ext must be a mask with frame and end counters, rate >= 1 and lookahead 0");
  PWGB_CHECK_ARG(!e->res_hist && e->res_hist_len == 0 && e->res_delay == 0 && e->in_lookahead == 0,
                 "conv1d_ragged: no delayed residual and no input lookahead");
  PWGB_CHECK_ARG(e->edge == d->pad_mode, "conv1d_ragged: ext->edge (%d) must be the conv's pad_mode (%d)", e->edge, d->pad_mode);
  PWGB_CHECK_ARG(d->pad_mode == PWGB_PAD_ZERO || (d->stride == 1 && d->pad_left < d->t_in),
                 "conv1d_ragged: a reflect or replicate edge needs stride 1 and pad_left (%d) < t_in (%d)", d->pad_left, d->t_in);
  PWGB_UNSUPPORTED_IF(d->period > 1 || d->pre_gate || d->shuffle > 1 || d->x_batch_stride || d->y_batch_stride ||
                          d->r_batch_stride || (d->t_valid > 0 && d->t_valid != d->t_in),
                      "conv1d_ragged: plain convs only (period 1, no pre_gate, no shuffle, contiguous)");
  const long long need = (long long)(d->t_out - 1) * d->stride + (long long)(d->kernel - 1) * d->dilation + 1 - d->pad_left;
  PWGB_CHECK_ARG(d->t_out == 0 || need <= (long long)d->t_in + (d->pad_mode == PWGB_PAD_ZERO ? (1LL << 30) : d->t_in - 1),
                 "conv1d_ragged: t_out too large for t_in");
  *h = *d;
  h->pad_mode = PWGB_PAD_HISTORY;
  h->t_valid = d->t_in;
  return PWGB_OK;
}

// One block per (entry, group of whole rows): the rows of a block are disjoint from every other block's, and within a
// block every pass reads all its sources before any thread writes.  A pass covers ascending flat indices r * H + j of
// its rows and element j reads index j + n of [hist | x], which is never below an index an earlier pass wrote, so the
// in-place shift of a history longer than the chunk reads no overwritten sample.
__global__ void __launch_bounds__(256) stream_carry_kernel(const long long* __restrict__ table, int n_entries) {
  const long long* e = table + 5LL * blockIdx.y;
  const float* x = reinterpret_cast<const float*>(e[0]);
  float* hist = reinterpret_cast<float*>(e[1]);
  const long long rows = e[2], n = e[3];
  const int H = (int)e[4];
  if (H <= 0) return;
  const int rpb = H >= 256 ? 1 : 256 / H;  // rows per block group
  const long long ngroups = (rows + rpb - 1) / rpb;
  for (long long g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const long long r0 = g * rpb;
    const long long nel = ((rows - r0 < rpb) ? rows - r0 : rpb) * (long long)H;
    for (long long base = 0; base < nel; base += 256) {
      const long long i = base + threadIdx.x;
      float v = 0.f;
      long long r = 0, j = 0;
      if (i < nel) {
        r = r0 + i / H;
        j = i % H;
        const long long s = j + n;  // index into [hist | x] of row r
        v = s < H ? hist[r * H + s] : __ldg(x + r * n + (s - H));
      }
      __syncthreads();
      if (i < nel) hist[r * H + j] = v;
      __syncthreads();
    }
  }
}

// y (batch, rows, t) in place: samples outside the signal of the pwgb_stream_ext mask become +0.0
__global__ void stream_mask_kernel(float* __restrict__ y, int rows, int t, const int* __restrict__ frame, const int* __restrict__ end,
                                   int rate, int look) {
  const int b = blockIdx.z;
  float* yr = y + ((long long)b * rows + blockIdx.y) * t;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < t; i += gridDim.x * blockDim.x)
    if (stream_outside(frame, end, rate, look, b, i)) yr[i] = 0.f;
}

}  // namespace pwgb

using namespace pwgb;

extern "C" int pwgb_stream_mask(float* y, int batch, int rows, int t, const pwgb_stream_ext* ext, void* stream) {
  PWGB_CHECK_ARG(ext && ext->frame && ext->end && ext->rate >= 1 && ext->lookahead >= 0, "stream_mask: ext must hold a mask");
  PWGB_CHECK_ARG(batch >= 0 && batch <= 65535 && rows >= 0 && rows <= 65535 && t >= 0, "stream_mask: bad sizes");
  if (batch == 0 || rows == 0 || t == 0) return PWGB_OK;
  PWGB_CHECK_ARG(y, "stream_mask: null argument");
  stream_mask_kernel<<<dim3((unsigned)(ceil_div(t, 256) < 64 ? ceil_div(t, 256) : 64), (unsigned)rows, (unsigned)batch), 256, 0,
                       (cudaStream_t)stream>>>(y, rows, t, ext->frame, ext->end, ext->rate, ext->lookahead);
  return check_launch("stream_mask_kernel");
}

extern "C" int pwgb_conv1d_stream_forward(const pwgb_conv1d_desc* d, const float* x, const float* hist, int hist_len,
                                          const int* replicate, const float* w, const float* bias, const float* residual,
                                          float* y, void* stream) {
  PWGB_CHECK_ARG(w, "conv1d_stream: null argument");
  if (const int rc = conv1d_stream_check(d, x, hist, hist_len, y)) return rc;
  return conv1d_stream_simt(d, x, hist, hist_len, replicate, w, bias, residual, y, (cudaStream_t)stream);
}

extern "C" int pwgb_conv1d_stream_ext_forward(const pwgb_conv1d_desc* d, const float* x, const float* hist, int hist_len,
                                              const int* replicate, const float* w, const float* bias, const float* residual,
                                              const pwgb_stream_ext* ext, float* y, void* stream) {
  PWGB_CHECK_ARG(w, "conv1d_stream: null argument");
  if (const int rc = conv1d_stream_check(d, x, hist, hist_len, y)) return rc;
  if (const int rc = stream_ext_check(ext, residual, d->pad_mode)) return rc;
  return conv1d_stream_simt(d, x, hist, hist_len, replicate, w, bias, residual, y, (cudaStream_t)stream, nullptr, 0, ext);
}

extern "C" int pwgb_conv1d_strided_stream_ext_forward(const pwgb_conv1d_desc* d, const float* x, const float* hist, int hist_len,
                                                      const float* w, const float* bias, const pwgb_stream_ext* ext, float* y,
                                                      void* stream) {
  PWGB_CHECK_ARG(d && x && y && w, "conv1d_strided_stream: null argument");
  PWGB_CHECK_ARG(d->batch >= 0 && d->cin > 0 && d->cout > 0 && d->t_in > 0 && d->t_out >= 0 && d->kernel > 0 && d->stride > 0 &&
                     d->dilation > 0 && d->pad_left >= 0 && d->groups > 0 && d->cin % d->groups == 0 && d->cout % d->groups == 0,
                 "conv1d_strided_stream: bad descriptor");
  PWGB_CHECK_ARG(d->pad_mode == PWGB_PAD_HISTORY, "conv1d_strided_stream: pad_mode must be PWGB_PAD_HISTORY");
  PWGB_CHECK_ARG(hist_len >= 0 && hist_len <= d->pad_left && (hist_len == 0 || hist), "conv1d_strided_stream: bad history (hist_len %d)",
                 hist_len);
  PWGB_UNSUPPORTED_IF(d->period > 1 || d->pre_gate || d->shuffle > 1 || d->accumulate || d->x_batch_stride ||
                          d->y_batch_stride || d->r_batch_stride || (d->t_valid > 0 && d->t_valid != d->t_in),
                      "conv1d_strided_stream: plain convs only (period 1, no pre_gate, no accumulate, one source)");
  const long long need = (long long)(d->t_out - 1) * d->stride + (long long)(d->kernel - 1) * d->dilation + 1 - d->pad_left;
  PWGB_CHECK_ARG(d->t_out == 0 || need <= (long long)d->t_in, "conv1d_strided_stream: t_out too large for t_in");
  if (const int rc = stream_ext_check(ext, nullptr, d->pad_mode)) return rc;
  PWGB_CHECK_ARG(!ext || ext->edge == PWGB_PAD_ZERO, "conv1d_strided_stream: no edge policy");
  // the generic FFMA body is written for any stride: the EXT instantiations of pwgb_conv1d_stream_ext_forward serve it
  return conv1d_stream_simt(d, x, hist, hist_len, nullptr, w, bias, nullptr, y, (cudaStream_t)stream, nullptr, 0, ext);
}

extern "C" int pwgb_conv1d_ragged_forward(const pwgb_conv1d_desc* d, const float* x, const float* w, const float* bias,
                                          const float* residual, const pwgb_stream_ext* ext, float* y, void* stream) {
  if (!ext) return pwgb_conv1d_forward(d, x, w, bias, residual, y, stream);
  PWGB_CHECK_ARG(w, "conv1d_ragged: null argument");
  pwgb_conv1d_desc h;
  if (const int rc = conv1d_ragged_check(d, x, ext, y, &h)) return rc;
  // the generic FFMA body of the history launches, for any stride: rows outside [0, t_in) read zero unless the edge
  // policy moves them onto the item's own reflected or replicated sample
  return conv1d_stream_simt(&h, x, nullptr, 0, nullptr, w, bias, residual, y, (cudaStream_t)stream, nullptr, 0, ext);
}

extern "C" int pwgb_stream_carry(const void* table, int n_entries, void* stream) {
  PWGB_CHECK_ARG(n_entries >= 0 && n_entries <= 65535, "stream_carry: bad entry count %d", n_entries);
  if (n_entries == 0) return PWGB_OK;
  PWGB_CHECK_ARG(table, "stream_carry: null table");
  // a fixed number of blocks per entry, each looping over its row groups: the table stays on the device
  stream_carry_kernel<<<dim3(64, (unsigned)n_entries), 256, 0, (cudaStream_t)stream>>>((const long long*)table, n_entries);
  return check_launch("stream_carry_kernel");
}
