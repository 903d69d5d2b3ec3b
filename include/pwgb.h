/*
 * pwgb.h -- C ABI of the H100-native vocoder hot path (libpwgb.so).
 *
 * The reference (kan-bayashi/ParallelWaveGAN) has no FFI of its own: its seam is
 * the torch.nn.Module surface (SURVEY.md 8b).  Each entry point below replaces
 * the ATen call sequence of one reference forward (cited per function,
 * file:line relative to /root/reference).  INTEGRATION.md shows the ctypes
 * stubs a maintainer adds on the reference side.
 *
 * Conventions
 *  - plain pointers and sizes only; every pointer is a DEVICE pointer to fp32
 *    data owned by the caller (inputs, outputs, workspaces).  The library never
 *    allocates, frees or retains device memory and keeps no global state.
 *  - tensors are (B, C, T) channel-major, time contiguous, like the reference.
 *  - `stream` is a cudaStream_t passed as void*; work is enqueued, never synced.
 *  - return value: 0 = PWGB_OK, negative = error (see pwgb_status); the message
 *    is available from pwgb_last_error() (thread local).
 *  - PWGB_UNSUPPORTED means "this configuration has no kernel"; callers must
 *    raise, there is no CPU fallback anywhere in the product.
 */
#ifndef PWGB_H_
#define PWGB_H_

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define PWGB_API __attribute__((visibility("default")))
#else
#define PWGB_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef enum pwgb_status {
  PWGB_OK = 0,
  PWGB_INVALID = -1,     /* bad descriptor / null pointer / size mismatch */
  PWGB_UNSUPPORTED = -2, /* valid but no kernel for this configuration    */
  PWGB_CUDA_ERROR = -3   /* launch failed; message holds cudaGetErrorString */
} pwgb_status;

/* PWGB_PAD_HISTORY: rows before sample 0 come from a caller-owned history (the stream entry points only);
 * PWGB_PAD_HISTORY_REFLECT: the same, except that a flagged slot reflects instead of replicating */
enum { PWGB_PAD_ZERO = 0, PWGB_PAD_REFLECT = 1, PWGB_PAD_REPLICATE = 2, PWGB_PAD_HISTORY = 3, PWGB_PAD_HISTORY_REFLECT = 4 };
enum { PWGB_ACT_NONE = 0, PWGB_ACT_TANH = 1, PWGB_ACT_LRELU = 2 };

PWGB_API const char* pwgb_last_error(void);
/* library version and the SM architecture the kernels were compiled for (100) */
PWGB_API int pwgb_version(void);
PWGB_API int pwgb_compiled_arch(void);
/* number of kernels launched by this thread since the last reset (bench.py's gpu_launches) */
PWGB_API long long pwgb_launch_count(void);
PWGB_API void pwgb_reset_launch_count(void);

/* ------------------------------------------------------------------------
 * Fused 1-D convolution:  y = [y +] out_scale * ( act( conv(pre(x)) + bias ) + residual )
 *
 * Replaces the ATen chains  LeakyReLU -> [Reflection|Zero pad] -> Conv1d -> [act] -> [+x]
 * of layers/residual_block.py:243-258 (HiFi-GAN ResBlock), layers/residual_stack.py:75-85
 * (MelGAN), models/hifigan.py:586-601, 354-381 (MSD/MPD towers; the MPD Conv2d (k,1)
 * over the (B,C,T/P,P) view is `period` = P), models/melgan.py:364-379,
 * models/parallel_wavegan.py:337-349.
 * ---------------------------------------------------------------------- */
typedef struct pwgb_conv1d_desc {
  int32_t batch;
  int32_t cin, cout;    /* total channels (all groups)                               */
  int32_t t_in;         /* logical input rows (per period column)                    */
  int32_t t_out;        /* output rows                                               */
  int32_t kernel, stride, dilation, groups;
  int32_t pad_left;     /* rows of padding on the left (right is implied by t_out)   */
  int32_t pad_mode;     /* PWGB_PAD_*; reflect/replicate need period == 1            */
  int32_t period;       /* 1 = plain Conv1d; P>1 = Conv2d (k,1) on the (T/P, P) view */
  int32_t t_valid;      /* flat source length (<= t_in*period); flat indices beyond
                           it are reflected (hifigan.py:365-369 F.pad(..,"reflect")) */
  float pre_slope;      /* LeakyReLU slope applied to x on load (1 = identity)       */
  int32_t pre_gate;     /* 1: x has 2*cin channels; in = tanh(x[c]) * sigmoid(x[c+cin]) */
  int32_t post_act;     /* PWGB_ACT_* applied to conv+bias                           */
  float post_slope;
  float out_scale;
  int32_t accumulate;   /* 1: y += result                                            */
  int32_t shuffle;      /* >1: pixel-shuffle epilogue used by conv_transpose (internal) */
  int32_t shuffle_pad;
  int32_t shuffle_tout; /* final output length when shuffle > 1                       */
  int64_t x_batch_stride; /* elements; 0 = contiguous                                 */
  int64_t y_batch_stride;
  int64_t r_batch_stride;
} pwgb_conv1d_desc;

/* w: (cout, cin/groups, kernel); bias: (cout) or NULL; residual: like y or NULL. */
PWGB_API int pwgb_conv1d_forward(const pwgb_conv1d_desc* d, const float* x, const float* w, const float* bias,
                        const float* residual, float* y, void* stream);

/* ------------------------------------------------------------------------
 * ConvTranspose1d(k, stride s, padding p, output_padding op) with fused pre-LeakyReLU,
 * poly-phase (no zero stuffing).  models/hifigan.py:94-107, models/melgan.py:86-101.
 * w: (cin, cout, kernel) -- the reference layout.  ws: workspace of
 * pwgb_conv_transpose1d_workspace() bytes.  t_out = (t_in-1)*s - 2p + k + op.
 * ---------------------------------------------------------------------- */
typedef struct pwgb_convtr1d_desc {
  int32_t batch, cin, cout, t_in, t_out; /* t_in / t_out in rows (per period column) */
  int32_t kernel, stride, padding;
  float pre_slope;
  int32_t groups; /* 0 or 1 = dense; w is (cin, cout/groups, kernel)                         */
  int32_t period; /* 0 or 1 = plain; P > 1 = transposed Conv2d (k,1) on (B, C, rows, P) views  */
} pwgb_convtr1d_desc;
PWGB_API size_t pwgb_conv_transpose1d_workspace(const pwgb_convtr1d_desc* d);
PWGB_API int pwgb_conv_transpose1d_forward(const pwgb_convtr1d_desc* d, const float* x, const float* w, const float* bias,
                                  float* y, void* ws, size_t ws_bytes, void* stream);
/* Two-source input (the skip concatenation of UHiFiGAN's decoder, models/uhifigan.py:289-291): the same conv-transpose
 * on cat(x1, x2) along channels without materialising the concatenation.  d->cin = cin1 + cin2; x1 is
 * (batch, cin1, t_in), x2 is (batch, cin2, t_in); w, bias, y, ws and the fused pre-LeakyReLU are those of
 * pwgb_conv_transpose1d_forward on the concatenated input, and the result is bit-identical to it.
 * pwgb_conv_transpose1d_cat_supported() returns 1 when the conv-transpose takes the tensor-core path and
 * cin1 % 32 == 0 (dense, plain); otherwise concatenate and call pwgb_conv_transpose1d_forward. */
PWGB_API int pwgb_conv_transpose1d_cat_supported(const pwgb_convtr1d_desc* d, int cin1);
PWGB_API int pwgb_conv_transpose1d_cat_forward(const pwgb_convtr1d_desc* d, int cin1, const float* x1, const float* x2,
                                      const float* w, const float* bias, float* y, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Dropout in training mode (torch.nn.Dropout(p); models/uhifigan.py input / downsample convs) over n elements.
 * Element e is kept when word e % 4 of Philox4x32-10(counter = (e / 4, offset), key = seed), as a 24-bit uniform in
 * [0, 1), is >= p; kept elements are multiplied by 1 / (1 - p) computed in fp32, the others are +0.0 (also when the
 * input is -0.0, +-inf or NaN).  p == 0 is the identity; p == 1 gives all +0.0; p outside [0, 1] or NaN is refused.
 * The backward recomputes the same mask from (seed, offset): gx = mask * gy / (1 - p).
 * ---------------------------------------------------------------------- */
PWGB_API int pwgb_dropout_forward(const float* x, float* y, long long n, float p, unsigned long long seed,
                                  unsigned long long offset, void* stream);
PWGB_API int pwgb_dropout_backward(const float* gy, float* gx, long long n, float p, unsigned long long seed,
                                   unsigned long long offset, void* stream);

/* ------------------------------------------------------------------------
 * Tensor-core (Hopper wgmma) path for the wide stride-1 convolutions: same descriptor
 * and semantics as pwgb_conv1d_forward, fp32-accurate through a bf16x3 operand split with
 * fp32 register accumulation.  Weights are re-laid out once per weight update by
 * pwgb_conv1d_tc_pack_weight into a caller-owned buffer of
 * pwgb_conv1d_tc_packed_weight_bytes().  pwgb_conv1d_tc_supported() returns 1 when the
 * configuration can run here (stride 1, cin/groups % 32 == 0, cout/groups % 16 == 0, halo fits shared
 * memory; cout/groups > 128 and groups > 1 run as several column chunks of one launch); everything else stays on
 * pwgb_conv1d_forward.
 * ---------------------------------------------------------------------- */
/* measurement aids (not part of the product contract): set key 1 = conv variant (value 2: stage activations with
 * cp.async instead of TMA; value 4: register epilogue instead of the staged one); get key 1 copies the plan of the last
 * tensor-core conv launch, 8 ints {MT, na, nb, ns, staged, tma_act, win_mode, nco} (a buffer of at least 5 ints gets
 * the leading min(bytes, 32) bytes); get key 2 copies the plan of the last tensor-core weight-gradient launch, 4 ints
 * {nc, tg, ntg, nsplit}; get key 3 copies the last dispatch of the FFMA conv (pwgb_conv1d_forward, and the FFMA
 * conv-transpose), 6 ints {kernel: 0 generic conv1d_fwd_kernel, 1 small_cout, 2 fewcout_long; RCO, WARPS_CO, RT, CI_T
 * of the generic kernel (0 otherwise); CO: its CO_T, the small_cout kernel's cout, the fewcout_long template width};
 * get key 4 copies the last pwgb_conv1d_wgrad launch, 4 ints {path: 0 tiled, 1 narrow; narrow_fast: 1 when the narrow
 * kernel takes its stride-1 no-period loop; nsplit of the tiled kernel or the narrow kernel's blocks; ci_tiles of the
 * tiled kernel (0 narrow)}.  Keys 3 and 4 are recorded on the host at launch (a call that launches nothing, B = 0,
 * leaves them unchanged).  Returns 0, or -1 for any other key or a short buffer. */
PWGB_API void pwgb_debug_set(int key, int value);
PWGB_API int pwgb_debug_get(int key, void* dst, size_t bytes);
PWGB_API size_t pwgb_conv1d_tc_packed_weight_bytes(int cin, int cout, int kernel);
PWGB_API int pwgb_conv1d_tc_pack_weight(const float* w, int cin, int cout, int kernel, void* packed, void* stream);
/* grouped weights (cout, cin/groups, kernel): one image per (group, <=256-column chunk) */
PWGB_API int pwgb_conv1d_tc_pack_weight_grouped(const float* w, int cin_per_group, int cout, int kernel, int groups, void* packed,
                                       void* stream);
PWGB_API int pwgb_conv1d_tc_supported(const pwgb_conv1d_desc* d);
PWGB_API int pwgb_conv1d_tc_forward(const pwgb_conv1d_desc* d, const float* x, const void* packed_w, const float* bias,
                           const float* residual, float* y, void* stream);

/* ------------------------------------------------------------------------
 * Streaming a causal conv stack chunk by chunk (layers/causal_conv.py under a chunked driver): history padding.
 * pwgb_conv1d_stream_forward (FFMA) and pwgb_conv1d_tc_stream_forward (tensor cores, packed weights as for
 * pwgb_conv1d_tc_forward) compute pwgb_conv1d_forward / pwgb_conv1d_tc_forward in every respect (pre-activation,
 * epilogue, residual, out_scale, accumulate) except for the input rows t < 0 in front of sample 0:
 *   t in [-hist_len, 0): hist[b, c, hist_len + t], hist (batch, cin, hist_len) fp32; or x[b, c, 0] where replicate[b] != 0
 *                        (replicate: DEVICE array of batch int32, or NULL) -- ReplicationPad1d for a fresh signal;
 *   t < -hist_len:       zero.
 * History rows are input rows: the pre-activation applies to them.  d->pad_mode must be PWGB_PAD_HISTORY (accepted by
 * these entry points only) with d->pad_left the conv's left padding; the scope is stride 1, period 1, no pre_gate, one
 * source (anything else: PWGB_INVALID or PWGB_UNSUPPORTED); groups as described below pwgb_s2d_stream_grouped_forward.
 * pwgb_conv1d_tc_supported() answers for such a descriptor as for any other.  The FFMA entry always runs the generic kernel, whose sum order does not depend on
 * where a sample sits, so a chunked run is bit-identical to the whole-signal conv on cat(hist, x) when that takes the same
 * kernel.  On the tensor cores the history launch stages activations with per-element copies (never TMA rows); the sum
 * order is the same as for the other plans.
 * d->pad_mode == PWGB_PAD_HISTORY_REFLECT (these entry points only) is the same policy, except that for a slot whose
 * flag is set (the same array, now a fresh-signal flag) row t in [-hist_len, 0) reads x[b, c, -t] -- ReflectionPad1d for a
 * fresh signal; it needs d->pad_left < d->t_in and hist_len <= d->pad_left (else PWGB_INVALID).  With hist_len ==
 * pad_left a flagged slot is bit-identical to the whole-signal conv with PWGB_PAD_REFLECT on x when that takes the same
 * kernel.
 * ---------------------------------------------------------------------- */
PWGB_API int pwgb_conv1d_stream_forward(const pwgb_conv1d_desc* d, const float* x, const float* hist, int hist_len,
                                        const int* replicate, const float* w, const float* bias, const float* residual,
                                        float* y, void* stream);
PWGB_API int pwgb_conv1d_tc_stream_forward(const pwgb_conv1d_desc* d, const float* x, const float* hist, int hist_len,
                                           const int* replicate, const void* packed_w, const float* bias,
                                           const float* residual, float* y, void* stream);
/* The causal conv-transpose of a stream (CausalConvTranspose1d, layers/causal_conv.py:46-79, with its one-frame
 * ReplicationPad1d): d describes the conv-transpose on cat(h, x) along time, so d->t_in = frames of x + 1 and
 * d->padding == d->stride (dense, plain); h[b] = replicate[b] ? x[b, :, 0] : hist[b, :, 0], hist (batch, cin, 1).  The
 * result is bit-identical to pwgb_conv_transpose1d_forward(d) on that concatenation, which is never materialised.  ws:
 * pwgb_conv_transpose1d_workspace(d) bytes. */
PWGB_API int pwgb_conv_transpose1d_stream_forward(const pwgb_convtr1d_desc* d, const float* x, const float* hist,
                                                  const int* replicate, const float* w, const float* bias, float* y, void* ws,
                                                  size_t ws_bytes, void* stream);
/* A window of a conv-transpose over a streamed signal (PQMF synthesis, layers/pqmf.py:133-149, under a chunked driver).
 * d describes the conv-transpose of one chunk (stride s, kernel K, padding p; groups 1, period 1): d->t_in = n rows of
 * x and d->t_out = n * s.  hist (batch, cin, hist_len) holds the signal's rows in front of the chunk (earlier rows read as
 * zero; hist_len >= ceil(K / s) - 1 covers the whole receptive field).  With the chunk starting at row T0 of the signal,
 * y[b, :, j] is output sample T0 * s - p + j of pwgb_conv_transpose1d_forward on the whole signal (any output_padding):
 * the window lags the input by p samples, so it never reads a row after the chunk.  fresh (DEVICE array of batch int32,
 * or NULL): a flagged slot is at the start of its signal (T0 = 0), and its y[b, :, j] for j < p (samples before 0) is
 * written as zero (a flagged slot's window must hold them all: d->t_out >= p).  flush != 0: x is not read (may be NULL) and the chunk's rows are zero -- the signal has ended, and
 * the window computes its last samples against the zero right padding.  It always runs the generic FFMA kernel, so it is
 * bit-identical to the whole-signal call when that runs the same kernel (cin not a multiple of 32, e.g. 4 subbands ->
 * 1).  ws: pwgb_conv_transpose1d_workspace(d) bytes. */
PWGB_API int pwgb_conv_transpose1d_window_stream_forward(const pwgb_convtr1d_desc* d, const float* x, const float* hist,
                                                         int hist_len, const int* fresh, int flush, const float* w,
                                                         const float* bias, float* y, void* ws, size_t ws_bytes, void* stream);
/* History carry of a stream, many signals in one launch.  table: DEVICE array of n_entries rows {x*, hist*, rows, n, H}
 * (5 x int64): x (rows, n) fp32 is this chunk of a signal, hist (rows, H) fp32 its history; afterwards hist holds the
 * last H samples of [hist | x] per row (also for n < H).  Every read of an entry happens before that entry's writes;
 * entries must not overlap each other.  A plain copy: deterministic. */
PWGB_API int pwgb_stream_carry(const void* table, int n_entries, void* stream);
/* Streaming a centred conv stack with a fixed lookahead.  A centred conv over [history | chunk] is the history conv
 * above with its output labelled pad samples earlier, so each signal of such a stream runs in "delayed time": output row
 * t of a chunk is signal sample frame[b] * rate - lookahead + t.  Two extensions of the history launches serve it:
 *   mask (frame != NULL): frame and end are DEVICE arrays of batch int32, the frames a slot has pushed before this chunk
 *     and its end frame (INT32_MAX while the signal is open); an output sample outside [0, end[b] * rate) is stored as
 *     +0.0 (also with accumulate), which is the zero padding the whole-signal conv reads there.  rate >= 1; lookahead >= 0.
 *   delayed residual (res_delay > 0 or res_hist_len > 0): output row t adds row t - res_delay of [res_hist | residual],
 *     res_hist (batch, cout, res_hist_len) fp32; needs a residual and 0 <= res_delay <= res_hist_len.
 *   edge policy (edge != PWGB_PAD_ZERO; the conv entry points only, with a mask and d->pad_mode == PWGB_PAD_HISTORY):
 *     input row r in [-hist_len, t_in) is signal sample u = frame[b] * rate - in_lookahead + r (the same rate and end as
 *     the mask: a stride-1 conv).  A row with u outside [0, end[b] * rate) reads instead the row of [hist | x] that holds
 *     the reflected sample (edge PWGB_PAD_REFLECT: -u before the start, 2 (L - 1) - u after the end L = end[b] * rate)
 *     or the replicated one (PWGB_PAD_REPLICATE: 0 or L - 1), and zero when that row lies outside [-hist_len, t_in).  The
 *     pre-activation applies to it as to any input row.  For a centred conv with padding p over [history (K-1) d |
 *     chunk], in_lookahead = the input signal's lookahead and output lookahead = in_lookahead - p + (K-1) d, every
 *     sample such a pad reads for an output inside the signal lies in the launch's window, so every output inside the
 *     signal is bit-identical to the whole-signal conv with PWGB_PAD_REFLECT / PWGB_PAD_REPLICATE (when that takes the
 *     same kernel); outputs outside it are masked.  The reflect case needs p < L, as ReflectionPad1d does.
 * Every other value is computed exactly as by the entry point without the extension; with ext == NULL (or all fields
 * zero) the call is that entry point.  A tensor-core launch with an extension keeps the register epilogue (same values
 * as the staged one).  edge and in_lookahead were appended to the struct; a zero-initialised struct keeps the meaning it
 * had before them. */
typedef struct pwgb_stream_ext {
  const int* frame;
  const int* end;
  int rate;
  int lookahead;
  const float* res_hist;
  int res_hist_len;
  int res_delay;
  int edge;
  int in_lookahead;
} pwgb_stream_ext;
PWGB_API int pwgb_conv1d_stream_ext_forward(const pwgb_conv1d_desc* d, const float* x, const float* hist, int hist_len,
                                            const int* replicate, const float* w, const float* bias, const float* residual,
                                            const pwgb_stream_ext* ext, float* y, void* stream);
PWGB_API int pwgb_conv1d_tc_stream_ext_forward(const pwgb_conv1d_desc* d, const float* x, const float* hist, int hist_len,
                                               const int* replicate, const void* packed_w, const float* bias,
                                               const float* residual, const pwgb_stream_ext* ext, float* y, void* stream);
/* pwgb_conv_transpose1d_stream_forward with the mask of ext (no residual fields, edge 0).  For a centred layer (kernel 2s,
 * padding p) the window of cat(h, x) is whole-signal samples [a * s - p, (a + n) * s - p) when x starts at input sample
 * a and h is sample a - 1 (zero for a fresh slot: pass no replicate flags), so lookahead = s * (input lookahead) + p. */
PWGB_API int pwgb_conv_transpose1d_stream_ext_forward(const pwgb_convtr1d_desc* d, const float* x, const float* hist,
                                                      const int* replicate, const float* w, const float* bias,
                                                      const pwgb_stream_ext* ext, float* y, void* ws, size_t ws_bytes,
                                                      void* stream);
/* y (batch, rows, t) fp32 in place: every sample outside the signal of ext's mask (rows of item b: frame[b], end[b],
 * rate, lookahead as above) is set to +0.0.  ext must hold a mask; its residual fields are ignored. */
PWGB_API int pwgb_stream_mask(float* y, int batch, int rows, int t, const pwgb_stream_ext* ext, void* stream);

/* Whole-signal convs over a batch of signals of different lengths ("ragged" batches; the VQ-VAE's encoder and decoder).
 * d is the descriptor of pwgb_conv1d_forward / pwgb_conv1d_tc_forward over the padded batch (pad_mode PWGB_PAD_ZERO,
 * PWGB_PAD_REFLECT or PWGB_PAD_REPLICATE; period 1, no pre_gate, contiguous), and ext a mask of pwgb_stream_ext at the
 * output: frame (DEVICE, all 0 for signals that start at sample 0), end (DEVICE, the item's length at this layer's rate
 * in units of rate), rate >= 1, lookahead 0, no residual history, in_lookahead 0, and edge == d->pad_mode.  Item b holds
 * L_b = end[b] * rate valid rows; then for every output row inside [0, L_b):
 *   zero pad: input rows at or past the item's input length read as zero -- the caller keeps them zero (the previous
 *     masked layer leaves them so); any stride;
 *   reflect / replicate pad (stride 1): an input row u >= L_b reads row 2 (L_b - 1) - u (reflect) or L_b - 1
 *     (replicate) of the same item, rows before 0 likewise -- the edge policy of pwgb_stream_ext, applied to the whole
 *     signal; ReflectionPad1d needs pad_left < L_b, which the entry cannot read on the host: the caller checks it (an item
 *     that breaks it reads zeros, never memory outside x);
 * and its value is bit-identical to the entry point without ext on that item alone with t = L_b, whenever that lone call
 * takes the same kernel (the FFMA entry always runs the generic kernel, never conv1d_small_cout_kernel or
 * conv1d_fewcout_long_kernel) and, on the tensor cores, the same tile shape.  Output rows at or past L_b are stored as
 * +0.0 (also with accumulate).  The launches are the EXT / EDGE instantiations of the stream history entry points with no
 * history rows.  ext == NULL: the call is pwgb_conv1d_forward / pwgb_conv1d_tc_forward.  A mask without frame and end
 * counters, an edge other than d->pad_mode, or a reflect / replicate edge with stride > 1 or pad_left >= t_in is
 * PWGB_INVALID. */
PWGB_API int pwgb_conv1d_ragged_forward(const pwgb_conv1d_desc* d, const float* x, const float* w, const float* bias,
                                        const float* residual, const pwgb_stream_ext* ext, float* y, void* stream);
PWGB_API int pwgb_conv1d_tc_ragged_forward(const pwgb_conv1d_desc* d, const float* x, const void* packed_w, const float* bias,
                                           const float* residual, const pwgb_stream_ext* ext, float* y, void* stream);

/* The strided convs of a stream (the encoder of a centred U-Net HiFi-GAN).
 *
 * pwgb_s2d_stream_forward: pwgb_s2d_forward (groups 1, period 1, pad_left 0) on the window [hist | x] without building it:
 * x (batch, channels, rows_in), hist (batch, channels, hist_len) -> y (batch, cgo, rows_out), channel r * channels + c
 * of row u = window row stride * u + r of channel c (zero past the window, and in channels >= stride * channels; cgo 0
 * means stride * channels).  A stream keeps the window starting on a stride boundary of the whole signal's padded
 * input, so its rows are the whole-signal gather's and the stride-1 conv that follows (pwgb_conv1d_tc_stream_ext_forward
 * with the mask) is bit-identical to the whole-signal strided conv's tensor-core route.
 *
 * pwgb_conv1d_strided_stream_ext_forward: pwgb_conv1d_stream_ext_forward (FFMA) for a stride >= 1 conv: input rows
 * [-hist_len, 0) come from hist (pad_left >= hist_len, earlier rows zero), any groups, period 1, no residual, no edge
 * policy, d->pad_mode PWGB_PAD_HISTORY; output row o reads input rows o * stride - pad_left + k * dilation.  The mask of
 * ext applies to the output rows (rate: the output's samples per frame).  Bit-identical to pwgb_conv1d_forward with the
 * same stride on the explicit window when that takes the generic kernel (not conv1d_small_cout_kernel or
 * conv1d_fewcout_long_kernel). */
PWGB_API int pwgb_s2d_stream_forward(const float* x, const float* hist, int hist_len, float* y, int batch, int channels, long long rows_in,
                                     int stride, long long rows_out, int cgo, void* stream);
/* The grouped strided convs of a stream (the MelGANDiscriminator encoder of a VQ-VAE).
 *
 * pwgb_s2d_stream_grouped_forward: pwgb_s2d_forward (groups, period 1, pad_left 0) on the window [hist | x]: y (batch,
 * groups * group_channels_out, rows_out), channel g * group_channels_out + r * (channels / groups) + c of row u = window
 * row stride * u + r of input channel g * (channels / groups) + c (zero past the window, and in a group's channels >=
 * stride * channels / groups; group_channels_out 0 means stride * channels / groups).  pwgb_s2d_stream_forward is this
 * call with groups 1 (its cgo is group_channels_out).  The stride-1 conv that follows runs with the same groups on
 * pwgb_conv1d_tc_stream_ext_forward with pad_left 0 and no history: the window carries it.
 *
 * Groups in the other stream entry points: pwgb_conv1d_stream_forward / pwgb_conv1d_stream_ext_forward /
 * pwgb_conv1d_strided_stream_ext_forward (FFMA) take any groups dividing cin and cout, history rows included (hist holds
 * every input channel).  pwgb_conv1d_tc_stream_forward / pwgb_conv1d_tc_stream_ext_forward take groups > 1 only with
 * d->pad_left 0 and hist_len 0 (pwgb_conv1d_tc_supported answers 0 for a grouped history descriptor with pad_left > 0,
 * the entry PWGB_UNSUPPORTED for hist_len > 0); such a launch is the grouped multi-chunk launch of
 * pwgb_conv1d_tc_forward with the mask, so it is bit-identical to that call on the window when it takes the same tile
 * shape. */
PWGB_API int pwgb_s2d_stream_grouped_forward(const float* x, const float* hist, int hist_len, float* y, int batch, int channels,
                                             int groups, long long rows_in, int stride, long long rows_out, int group_channels_out,
                                             void* stream);
PWGB_API int pwgb_conv1d_strided_stream_ext_forward(const pwgb_conv1d_desc* d, const float* x, const float* hist, int hist_len,
                                                    const float* w, const float* bias, const pwgb_stream_ext* ext, float* y,
                                                    void* stream);
/* The two-source stream conv-transpose of a U-Net decoder level: pwgb_conv_transpose1d_stream_ext_forward on
 * cat(x1, x2) along channels (d->cin = cin1 + cin2, d->t_in = n + 1 counting the history frame), where each source has
 * its own history: source 1 is [hist1 (batch, cin1, 1) | x1 (batch, cin1, n)], source 2 is read delay2 rows back from
 * [hist2 (batch, cin2, hist2_len) | x2 (batch, cin2, n)] (hist2_len >= delay2 + 1), so that its row j is row j - delay2.
 * One gather launch builds the window in ws, then the single-source stream conv-transpose runs on it (tensor cores or
 * FFMA as that entry picks); the result is bit-identical to pwgb_conv_transpose1d_cat_forward / the single-source entry
 * on the explicit windows.  ws: pwgb_conv_transpose1d_cat_stream_workspace(d) bytes. */
PWGB_API size_t pwgb_conv_transpose1d_cat_stream_workspace(const pwgb_convtr1d_desc* d);
PWGB_API int pwgb_conv_transpose1d_cat_stream_ext_forward(const pwgb_convtr1d_desc* d, int cin1, const float* x1, const float* hist1,
                                                          const float* x2, const float* hist2, int hist2_len, int delay2,
                                                          const float* w, const float* bias, const pwgb_stream_ext* ext, float* y,
                                                          void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------
 * One HiFi-GAN ResBlock conv pair (layers/residual_block.py:243-258, non-causal, additional convs) in one
 * tensor-core launch; the intermediate stays in shared memory:
 *     h = conv_{kernel,dilation}(lrelu(x)) + b1 ;  x' = conv_{kernel,1}(lrelu(h)) + b2 + x
 *     y = out_scale * x'   (accumulate: y += out_scale * x')
 * x, y: (batch, channels, t), 16-byte aligned, y must not alias x.  Both convs pad with zeros ("same" length).
 * w1_packed / w2_packed: pwgb_conv1d_tc_pack_weight images of the two (channels, channels, kernel) weights; b1 / b2
 * may be NULL.  The result is bit-identical to the two pwgb_conv1d_tc_forward calls it replaces.
 * pwgb_resblock_pair_supported() == 0 (channels other than 32 / 64, t % 4 != 0, or no shared-memory plan, as for a
 * wide conv1 halo): use those two calls instead.  pwgb_resblock_pair_plan() fills 5 ints {output rows per tile, conv
 * rows per tile, conv1 operand buffers, weight stages of both rings, raw activation stages} and returns 1, or returns 0
 * when unsupported.
 * ---------------------------------------------------------------------- */
typedef struct pwgb_resblock_desc {
  int32_t batch, channels, t;
  int32_t kernel, dilation; /* conv1: (kernel, dilation); conv2: (kernel, 1) */
  float slope;              /* LeakyReLU negative slope before each conv */
  float out_scale;
  int32_t accumulate;
} pwgb_resblock_desc;
PWGB_API int pwgb_resblock_pair_supported(const pwgb_resblock_desc* d);
PWGB_API int pwgb_resblock_pair_plan(const pwgb_resblock_desc* d, int* info);
PWGB_API int pwgb_resblock_pair_forward(const pwgb_resblock_desc* d, const float* x, const void* w1_packed, const float* b1,
                               const void* w2_packed, const float* b2, float* y, void* stream);
/* The same pair at 128 or 256 channels, where the intermediate does not fit on chip: two tensor-core launches that hand
 * it over in h_packed, a caller-owned workspace of 4 * batch * channels * t bytes (16-byte aligned), written by the
 * first launch as the second one's bf16 hi/lo operand image and read by it with tensor copies.  Same arguments and
 * result as pwgb_resblock_pair_forward, bit-identical to the two pwgb_conv1d_tc_forward calls it replaces.
 * pwgb_resblock_pair_packed_supported() == 0 (other channel counts, t % 4 != 0, no tile plan in which the second conv
 * stages its residual in shared memory): use those two calls instead. */
PWGB_API int pwgb_resblock_pair_packed_supported(const pwgb_resblock_desc* d);
PWGB_API int pwgb_resblock_pair_packed_forward(const pwgb_resblock_desc* d, const float* x, const void* w1_packed, const float* b1,
                                               const void* w2_packed, const float* b2, void* h_packed, float* y, void* stream);
/* The two pairs for a batch of signals of different lengths ("ragged" batches): the arguments of the entry point
 * above plus ext, of which only the mask fields are read (frame, end, rate, lookahead as in pwgb_stream_ext; residual
 * and edge fields are ignored).  Row t of item b is signal sample frame[b] * rate - lookahead + t; for a batch that
 * starts every item at sample 0, frame = 0, lookahead = 0 and end[b] * rate = the item's length L_b.  Outside its signal
 * the intermediate that the second conv reads (the shared-memory h image; the packed h image, whose tensor-copy box is
 * only clipped at t) is +0.0, which is the zero padding of that conv on the item alone, and so is y.
 *   precondition: x is zero outside each item's signal (the previous masked layer leaves it so);
 *   accumulate: y must be zero on entry outside each item's signal; it is +0.0 there afterwards (y + 0.0);
 *   then every row of item b inside its signal is bit-identical to the entry point above on that item alone with
 *   t = L_b (or the two pwgb_conv1d_tc_forward calls it replaces, where L_b % 4 != 0).
 * ext == NULL: the call is the entry point without the mask.  The unmasked kernels are separate instantiations and
 * keep their code. */
PWGB_API int pwgb_resblock_pair_ext_forward(const pwgb_resblock_desc* d, const float* x, const void* w1_packed, const float* b1,
                                            const void* w2_packed, const float* b2, const pwgb_stream_ext* ext, float* y,
                                            void* stream);
PWGB_API int pwgb_resblock_pair_packed_ext_forward(const pwgb_resblock_desc* d, const float* x, const void* w1_packed,
                                                   const float* b1, const void* w2_packed, const float* b2,
                                                   const pwgb_stream_ext* ext, void* h_packed, float* y, void* stream);

/* ------------------------------------------------------------------------
 * Fused WaveNet residual layer of ParallelWaveGANGenerator (layers/residual_block.py:102-140,
 * called 30x from models/parallel_wavegan.py:161-166):
 *     g  = conv_{k,dilation}(x) + W_aux c (+ b_conv)
 *     z  = tanh(g[:G/2]) * sigmoid(g[G/2:])
 *     skips += W_skip z + b_skip ;   x_out = (W_out z + b_out + x) * sqrt(0.5)
 * on the tensor-core path (bf16x3, fp32 accumulate).  `c` must be stored with `aux_channels`
 * channels, a multiple of 32 (zero-padded beyond the model's real aux_channels; the pack
 * routine zero-fills the matching weight columns).  g_ws: workspace of batch*G*t floats.
 * b_skip_out = concat(b_skip, b_out) or NULL.  pwgb_wavenet_supported() == 0 means the caller
 * must compose the layer from pwgb_conv1d_forward (pre_gate / accumulate options) instead.
 * ---------------------------------------------------------------------- */
typedef struct pwgb_wavenet_desc {
  int32_t batch, t;
  int32_t residual_channels, gate_channels, skip_channels;
  int32_t aux_channels; /* as stored, padded to a multiple of 32 (0 = no conditioning) */
  int32_t kernel, dilation;
  int32_t causal; /* 0: centred taps (odd kernel); 1: causal taps t - (kernel-1-j)*dilation (any kernel) */
} pwgb_wavenet_desc;
PWGB_API int pwgb_wavenet_supported(const pwgb_wavenet_desc* d);
PWGB_API size_t pwgb_wavenet_packed_bytes(const pwgb_wavenet_desc* d);
PWGB_API int pwgb_wavenet_pack(const pwgb_wavenet_desc* d, const float* w_conv, const float* w_aux, int aux_channels_real,
                      const float* w_skip, const float* w_out, void* packed, void* stream);
PWGB_API int pwgb_wavenet_layer_forward(const pwgb_wavenet_desc* d, const float* x, const float* c, const void* packed,
                               const float* b_conv, const float* b_skip_out, float* x_out, float* skips, float* g_ws,
                               void* stream);

/* ------------------------------------------------------------------------
 * Training collater on the GPU (Collater.__call__, bin/train.py:711-798; SURVEY.md 8f-3): one launch gathers the
 * random crops of a batch from a device-resident corpus.  audio: all waveforms concatenated; feats: all feature
 * matrices (frames, channels) concatenated along frames (NULL: audio-only case).  x_offsets / c_offsets: DEVICE
 * arrays of `batch` int64 -- element offset of each crop's first sample / row offset of its first frame.
 *   y (batch, t)                 = audio[x_offsets[b] + 0..t)
 *   c (batch, channels, frames)  = transpose of feats rows [c_offsets[b], c_offsets[b] + frames)
 * ---------------------------------------------------------------------- */
PWGB_API int pwgb_collate_crop(const float* audio, const long long* x_offsets, const float* feats, const long long* c_offsets, float* y,
                      float* c, int batch, int t, int channels, int frames, void* stream);

/* ------------------------------------------------------------------------
 * Decode-driver glue (bin/decode.py:214-243, SURVEY.md 8f-2).
 * pwgb_prep_features: one utterance's features c (t, channels) row-major -> out (channels, t_out):
 *   out[ch, u] = (c[u - pad_left, ch] - mean[ch]) / scale[ch]  (mean/scale NULL: no normalisation; hifigan.py:264-265),
 *   frames outside [0, t) zero (pad_mode PWGB_PAD_ZERO) or edge-replicated (PWGB_PAD_REPLICATE,
 *   parallel_wavegan.py:250-251).  `out` is usually one batch slot of the generator input.
 * pwgb_pcm16_forward: lrintf(y * 32767) saturated to int16 -- libsndfile's float -> PCM_16 (decode.py:236-241);
 *   the product in fp32, ties to even, +-inf saturate, NaN -> 0.
 * ---------------------------------------------------------------------- */
PWGB_API int pwgb_prep_features(const float* c, const float* mean, const float* scale, float* out, int t, int channels, int pad_left,
                       int t_out, int pad_mode, void* stream);
PWGB_API int pwgb_pcm16_forward(const float* y, short* out, long long n, void* stream);

/* ------------------------------------------------------------------------
 * Multi-tensor optimizer step with fused global-norm clipping (SURVEY.md 8f-1): replaces
 * torch.nn.utils.clip_grad_norm_ + optimizer.step() of Trainer._train_step (bin/train.py:289-293, 329-333)
 * -- Adam (torch.optim.Adam semantics) or the reference's RAdam (optimizers/radam.py:27-99) -- for all
 * parameters of a model in three launches.  `table`: DEVICE array of n_tensors rows
 * {param*, grad*, exp_avg*, exp_avg_sq*, numel} (5 x int64); `chunks`: DEVICE array of n_chunks int32 pairs
 * {tensor index, chunk index}; chunk c of a tensor covers elements [c*chunk_elems, (c+1)*chunk_elems).
 * pwgb_mt_clip_coef: out2[0] = total gradient norm, out2[1] = min(1, max_norm/(norm+1e-6)) (1 if max_norm<=0);
 * partial: n_chunks floats of workspace.  pwgb_mt_adam_step: mode 0 Adam (c1 = lr/(1-beta1^t),
 * c2 = 1/sqrt(1-beta2^t)), 1 RAdam rectified (c1 = step_size*lr), 2 RAdam unrectified (c1 = step_size*lr);
 * coef2 = the out2 of pwgb_mt_clip_coef or NULL (no clipping); gradients are scaled on the fly and written
 * back only if write_clipped_grad.  Deterministic (fixed chunk order, no atomics).
 * ---------------------------------------------------------------------- */
PWGB_API int pwgb_mt_clip_coef(const void* table, const void* chunks, int n_chunks, int chunk_elems, float max_norm, float* partial,
                      float* out2, void* stream);
PWGB_API int pwgb_mt_adam_step(const void* table, const void* chunks, int n_chunks, int chunk_elems, int mode, float lr, float beta1,
                      float beta2, float eps, float weight_decay, float c1, float c2, const float* coef2, int write_clipped_grad,
                      void* stream);

/* ------------------------------------------------------------------------
 * Space-to-depth along time for strided convs (MSD grouped k41 stride 2/4, hifigan.py:586-601; MPD (5,1)
 * stride (3,1), hifigan.py:354-381):  y[b, g*s*Cg + r*Cg + cl, u, p] = x[b, g*Cg + cl, s*u + r - pad_left, p]
 * (zero outside [0, rows_in)), so that  conv_stride_s(x, w) = conv_stride_1(y, w') with
 * w'[co, r*Cg + cl, j] = w[co, cl, s*j + r]  (ceil(K/s) taps, no padding, rows_out = t_out + ceil(K/s) - 1).
 * x: (batch, channels, rows_in, period) -> y: (batch, groups*Cgo, rows_out, period); backward is the adjoint.
 * Cgo = group_channels_out (0: stride * Cg): output channels per group; channels beyond stride * Cg are zero
 * (padding up to the tensor cores' 32-channel granularity, matched by zero weight columns).
 * ---------------------------------------------------------------------- */
PWGB_API int pwgb_s2d_forward(const float* x, float* y, int batch, int channels, int groups, long long rows_in, int period, int stride,
                     int pad_left, long long rows_out, int group_channels_out, void* stream);
PWGB_API int pwgb_s2d_backward(const float* gy, float* gx, int batch, int channels, int groups, long long rows_in, int period, int stride,
                      int pad_left, long long rows_out, int group_channels_out, void* stream);

/* ------------------------------------------------------------------------
 * Packed WaveNet residual stack: the fused ONE-kernel form of WaveNetResidualBlock.forward
 * (layers/residual_block.py:102-140) used by ParallelWaveGANGenerator.forward's layer loop
 * (models/parallel_wavegan.py:161-166).  Between layers the residual stream x and the conditioning c
 * stay in the tensor core's operand layout, split bf16 hi/lo (same bytes per sample as fp32):
 *   xpk [batch][hi|lo][residual_channels/8][t_pad][8] bf16, t_pad = 2*halo + round_up(t,256); rows
 *       [halo, halo+t) hold the samples; every other row MUST be zero (allocate zero-filled once; the
 *       kernels only ever write rows [halo, halo+t));
 *   cpk [batch][hi|lo][ceil(aux_channels/8)][round_up(t,256)][8] bf16 (written completely by pack_c).
 * halo >= (kernel-1)/2 * (largest dilation of the stack), or (kernel-1) * (largest dilation) when causal
 * (the layout stays symmetric; a causal layer only reads the left halo).  Weights: the image written by
 * pwgb_wavenet_pack() for the same channel counts with the aux weight padded to a multiple of 32
 * channels (desc.aux_channels there = round_up(aux_channels, 32)).  b_skip_out = concat(b_skip, b_out).
 * layer_forward:  skips (fp32, (batch, skip_channels, t)) = [skips_init ? 0 : skips] + s;
 * xpk_out = packed x' or NULL when the residual output is not needed (last layer of a stack).
 * pwgb_wnstack_supported() == 0: use pwgb_wavenet_layer_forward / the generic composition instead.
 * ---------------------------------------------------------------------- */
typedef struct pwgb_wnstack_desc {
  int32_t batch, t;
  int32_t residual_channels, gate_channels, skip_channels;
  int32_t aux_channels; /* real conditioning channels (multiple of 16) */
  int32_t kernel, halo;
  int32_t causal; /* 0: centred taps (odd kernel); 1: causal taps t - (kernel-1-j)*dilation (any kernel) */
} pwgb_wnstack_desc;
PWGB_API int pwgb_wnstack_supported(const pwgb_wnstack_desc* d);
PWGB_API size_t pwgb_wnstack_x_bytes(const pwgb_wnstack_desc* d);
PWGB_API size_t pwgb_wnstack_c_bytes(const pwgb_wnstack_desc* d);
PWGB_API int pwgb_wnstack_pack_x(const pwgb_wnstack_desc* d, const float* x, void* xpk, void* stream);
PWGB_API int pwgb_wnstack_unpack_x(const pwgb_wnstack_desc* d, const void* xpk, float* x, void* stream);
/* c: (batch, >= aux_channels stored channels, t) fp32 with batch stride c_batch_stride floats */
PWGB_API int pwgb_wnstack_pack_c(const pwgb_wnstack_desc* d, const float* c, long long c_batch_stride, void* cpk, void* stream);
/* first_conv (Conv1d1x1 in_channels -> residual_channels, parallel_wavegan.py:155): z (batch, in_channels, t),
 * w (residual_channels, in_channels) -> packed residual stream */
PWGB_API int pwgb_wnstack_first_conv(const pwgb_wnstack_desc* d, const float* z, int in_channels, const float* w, const float* bias,
                            void* xpk, void* stream);
PWGB_API int pwgb_wnstack_layer_forward(const pwgb_wnstack_desc* d, int dilation, const void* xpk_in, const void* cpk,
                               const void* packed_w, const float* b_conv, const float* b_skip_out, void* xpk_out,
                               float* skips, int skips_init, void* stream);
/* Streaming a causal stack chunk by chunk.  A causal layer reads only the (kernel-1)*dilation rows in front of sample 0,
 * so those rows of its input buffer may hold the previous chunk's last samples instead of zeros: the unchanged layer
 * then computes the chunk exactly as the whole-signal forward would.  Relaxed contract for such streaming buffers
 * (causal, or a centred stack streamed with lookahead, below): the left halo rows may hold history; the right halo and every row past t stay zero.  Buffers that
 * are not streamed keep the contract above.
 * A layer's history h = (kernel-1)*dilation is a state tensor laid out like the stream, [batch][hi|lo][R/8][h][8] bf16
 * (batch * 2 * residual_channels * h * 2 bytes), all zero for a fresh signal (the whole-signal zero padding).
 * pwgb_wnstack_carry() runs between layer l and layer l+1, before layer l+1 writes into the buffer layer l read:
 *   save: rows [t - h_save, t) of xpk_save (layer l's input) -> hist_save; rows before 0 come from the left halo, so
 *         for t < h_save the previous history shifts through;
 *   load: hist_load -> rows [-h_load, 0) of xpk_load (layer l+1's input).
 * The halves touch disjoint memory; either may be absent (h = 0: load only before layer 0, save only after the last
 * layer).  h_save, h_load <= halo.  A plain copy: deterministic. */
PWGB_API int pwgb_wnstack_carry(const pwgb_wnstack_desc* d, const void* xpk_save, void* hist_save, int h_save, void* xpk_load,
                       const void* hist_load, int h_load, void* stream);
/* Streaming a centred stack with a fixed lookahead (desc.causal = 0, halo >= (kernel-1) * largest dilation).  In delayed
 * time (see pwgb_stream_ext) a centred layer over [history | chunk] is the causal tap pattern with its output labelled
 * (kernel-1)/2 * dilation rows earlier; its input buffer's left halo holds the (kernel-1) * dilation history rows, carried
 * with pwgb_wnstack_carry exactly as for a causal stack.  pwgb_wnstack_layer_stream_ext_forward is
 * pwgb_wnstack_layer_forward with:
 *   - taps t - (kernel-1-j) * dilation, and the residual of output row t read at input row t - (kernel-1)/2 * dilation
 *     (from the halo or the chunk);
 *   - the conditioning of output row t read at row c_row0 + t of cpk, laid out as pwgb_wnstack_pack_c writes it with
 *     c_rows rows per plane ([batch][hi|lo][ceil(aux/8)][c_rows][8] bf16, c_rows >= c_row0 + t);
 *   - the skip of output row t at skips[(b * skip_channels + ch) * skip_row_stride + skip_col0 + t];
 *   - x' rows outside the signal of ext's mask (rate = samples per frame, lookahead = the output's) stored as zero, the
 *     next layer's zero padding.  ext must be a mask without residual fields.
 * Every value is the same fp32 expression as in pwgb_wnstack_layer_forward of the centred stack, so a chunked run equals
 * the whole signal bit for bit.  pwgb_wnstack_first_conv_stream_ext is pwgb_wnstack_first_conv on z rows z_row_stride
 * floats apart (z_row_stride >= t), with the rows outside ext's mask stored as zero. */
PWGB_API int pwgb_wnstack_first_conv_stream_ext(const pwgb_wnstack_desc* d, const float* z, long long z_row_stride, int in_channels,
                                                const float* w, const float* bias, const pwgb_stream_ext* ext, void* xpk, void* stream);
PWGB_API int pwgb_wnstack_layer_stream_ext_forward(const pwgb_wnstack_desc* d, int dilation, const void* xpk_in, const void* cpk,
                                                   int c_rows, int c_row0, const void* packed_w, const float* b_conv,
                                                   const float* b_skip_out, void* xpk_out, float* skips, int skip_col0,
                                                   long long skip_row_stride, int skips_init, const pwgb_stream_ext* ext,
                                                   void* stream);

/* ------------------------------------------------------------------------
 * One stage of the PWG conditioning upsampler (layers/upsample.py:112-128): nearest repeat
 * x`scale` along time followed by the (2*scale+1)-tap FIR shared by all rows, zero padded:
 *   y[r, o] = sum_k f[k] * x[r, (o + k - scale) / scale]   for 0 <= o + k - scale < t_in*scale.
 * x: rows x t_in (row stride t_in); y: row r of batch item r / rows_per_batch starts at
 * (r / rows_per_batch) * y_batch_stride + (r % rows_per_batch) * t_in * scale.
 * ---------------------------------------------------------------------- */
PWGB_API int pwgb_upsample_fir_forward(int rows, int rows_per_batch, int t_in, int scale, const float* x, const float* fir,
                              float* y, long long y_batch_stride, void* stream);
/* Causal stage (layers/upsample.py:98-125 with use_causal_conv: the FIR pads 2*scale on the left and the tail is
 * cropped): the tap origin moves from scale to 2*scale,
 *   y[r, o] = sum_k f[k] * x[r, (o + k - 2*scale) / scale]   for 0 <= o + k - 2*scale < t_in*scale,
 * so output frame j only meets input frames j-2, j-1, j.  Same arguments and layout as the centred pair. */
PWGB_API int pwgb_upsample_fir_causal_forward(int rows, int rows_per_batch, int t_in, int scale, const float* x, const float* fir,
                                     float* y, long long y_batch_stride, void* stream);
/* The causal stage of a stream: input frames -2 and -1 come from hist_in (rows x 2 fp32, oldest first) instead of zero;
 * hist_in is only read (the caller carries it, e.g. with pwgb_stream_carry).  Every output is the same fp32 expression
 * as in pwgb_upsample_fir_causal_forward, so chunked runs equal the whole-signal stage bit for bit. */
PWGB_API int pwgb_upsample_fir_causal_stream_forward(int rows, int rows_per_batch, int t_in, int scale, const float* x,
                                            const float* fir, float* y, long long y_batch_stride, const float* hist_in,
                                            void* stream);
/* The centred stage of a lookahead stream: on [2 history frames | chunk] output frame j reads input frames j-2, j-1, j,
 * i.e. it is the centred stage's output frame j-1 (lookahead <- scale * lookahead + scale).  hist_in as in
 * pwgb_upsample_fir_causal_stream_forward; every output is the same fp32 expression as in pwgb_upsample_fir_forward, and
 * the outputs outside the signal of ext's mask (rate: output samples per input frame of the whole upsampler so far)
 * are stored as +0.0.  ext must be a mask without residual fields. */
PWGB_API int pwgb_upsample_fir_stream_ext_forward(int rows, int rows_per_batch, int t_in, int scale, const float* x, const float* fir,
                                                  float* y, long long y_batch_stride, const float* hist_in, const pwgb_stream_ext* ext,
                                                  void* stream);
PWGB_API int pwgb_upsample_fir_causal_backward(int rows, int rows_per_batch, int t_in, int scale, const float* x, const float* fir,
                                      const float* gy, long long gy_batch_stride, float* gx, float* dfir, void* stream);

/* ------------------------------------------------------------------------
 * Spectral losses.  stft(): losses/stft_loss.py:16-40 (center=True, reflect pad n_fft/2, window of
 * win_length centred in n_fft, rFFT, sqrt(clamp(re^2+im^2, eps))).
 * pwgb_mr_stft_loss_forward = MultiResolutionSTFTLoss.forward (stft_loss.py:146-170) for signals
 * x (predicted) and y (ground truth), both (batch, t): out2[0] = sc, out2[1] = mag, averaged over
 * the n_res resolutions; windows[r] is a DEVICE pointer to win_length floats (the module buffer).
 * pwgb_stft_amplitude_forward writes sqrt(clamp(|STFT|^2, eps)) as (batch, frames, n_fft/2+1) for
 * one or two signals; pwgb_mel_project_forward is the rest of MelSpectrogram(.Loss)
 * (mel_loss.py:105-110, 150-165): mel = clamp(amp @ melmat, eps), log * log_scale, optional
 * (batch, n_mels, frames) output and/or the mean L1 between the two signals' log-mels.
 * ---------------------------------------------------------------------- */
typedef struct pwgb_stft_desc {
  int32_t batch, t, n_fft, hop, win_length;
  float clamp_eps;
} pwgb_stft_desc;
PWGB_API size_t pwgb_mr_stft_loss_workspace(const pwgb_stft_desc* descs, int n_res);
PWGB_API int pwgb_mr_stft_loss_forward(const pwgb_stft_desc* descs, int n_res, const float* x, const float* y,
                              const float* const* windows, float* out2, void* ws, size_t ws_bytes, void* stream);
PWGB_API int pwgb_stft_amplitude_forward(const pwgb_stft_desc* d, const float* x, const float* y, const float* window,
                                float* amp_x, float* amp_y, void* stream);
PWGB_API int pwgb_mel_project_forward(int batch, int frames, int bins, int n_mels, const float* amp_x, const float* amp_y,
                             const float* melmat, float eps, float log_scale, float* mel_x, float* loss, float* ws,
                             void* stream);

/* ------------------------------------------------------------------------
 * Deterministic mean reductions for the GAN losses (losses/adversarial_loss.py:29-123,
 * losses/feat_match_loss.py:27-54): out[0] (+)= weight * mean_i f(x_i [, y_i]) with
 * mode 0: (x-c)^2, 1: |x-y|, 2: max(0, c - s*x), 3: s*x, 4: (x-y)^2.  ws: >= 1 float of scratch
 * (more = more parallel partials, up to 1024).
 * AvgPool1d between discriminator scales (hifigan.py:758-775, melgan.py:478-493).
 * ---------------------------------------------------------------------- */
PWGB_API int pwgb_reduce_mean_forward(int mode, const float* x, const float* y, long long n, float c, float s, float weight,
                             int accumulate, float* out, float* ws, int ws_floats, void* stream);
PWGB_API int pwgb_avg_pool1d_forward(const float* x, float* y, int rows, int t_in, int kernel, int stride, int padding,
                            int count_include_pad, void* stream);

/* ------------------------------------------------------------------------
 * Backward building blocks of the train step (bin/train.py:287-288, 327-328 `loss.backward()`).
 * Data gradients reuse the forward entry points: the dgrad of a stride-1 conv is the conv1d forward entry point (FFMA or tensor cores)
 * with the transposed, tap-flipped weight; the dgrad of a strided / grouped / period conv is
 * pwgb_conv_transpose1d_forward (groups / period fields); the dgrad of a conv-transpose is a strided
 * pwgb_conv1d_forward.  New here:
 *   pwgb_conv1d_wgrad: dw[co, ci, k] (+)= sum_{b,t} lrelu_g(gy[b,co,t]) * pre(x)[b, ci, t*stride + k*dil - pad]
 *     for the conv described by `d` (same descriptor as the forward; d->pre_slope is applied to x,
 *     g_slope to gy -- 1 except for the conv-transpose weight gradient); deterministic split reduce.
 *   pwgb_act_backward:  out (+)= g * scale * f'(ref)   mode 0 LeakyReLU mask (ref > 0), 1 tanh (ref = output), 2 copy
 *   pwgb_bias_grad:     db[c] (+)= sum_{b,t} g[b,c,t]
 *   pwgb_reduce_mean_backward / pwgb_avg_pool1d_backward: adjoints of the forward entry points
 *   pwgb_axpby:         y = a*x + b*y
 * ---------------------------------------------------------------------- */
PWGB_API size_t pwgb_conv1d_wgrad_workspace(const pwgb_conv1d_desc* d);
PWGB_API int pwgb_conv1d_wgrad(const pwgb_conv1d_desc* d, const float* x, const float* gy, float g_slope, float* dw,
                      int accumulate, void* ws, size_t ws_bytes, void* stream);
/* tensor-core variant (stride 1, groups 1, period 1, zero padding, cout % 8 == 0 (>= 32), cin % 32 == 0): the
 * reduction over time is the MMA K dimension, both operands MN-major; same result contract. */
PWGB_API int pwgb_conv1d_wgrad_tc_supported(const pwgb_conv1d_desc* d);
PWGB_API size_t pwgb_conv1d_wgrad_tc_workspace(const pwgb_conv1d_desc* d);
PWGB_API int pwgb_conv1d_wgrad_tc(const pwgb_conv1d_desc* d, const float* x, const float* gy, float g_slope, float* dw, void* ws,
                         size_t ws_bytes, void* stream);
PWGB_API int pwgb_act_backward(int mode, const float* g, const float* ref, float* out, long long n, float slope, float scale,
                      int accumulate, void* stream);
PWGB_API int pwgb_bias_grad(const float* g, float* db, int batch, int channels, long long len, int accumulate, void* stream);
PWGB_API int pwgb_reduce_mean_backward(int mode, const float* x, const float* y, long long n, float c, float s, float weight,
                              const float* gout, float* gx, int accumulate, void* stream);
PWGB_API int pwgb_avg_pool1d_backward(const float* gy, float* gx, int rows, int t_in, int kernel, int stride, int padding,
                             int count_include_pad, void* stream);
PWGB_API int pwgb_axpby(long long n, float a, const float* x, float b, float* y, void* stream);
/* out = a * sum_k xs[k] (index order); xs: DEVICE array of n pointers to len floats; rows_16b_aligned: every xs[k] is 16-byte aligned */
PWGB_API int pwgb_scaled_sum(const float* const* xs, int n, float a, float* out, long long len, int rows_16b_aligned, void* stream);
/* Explicit ReflectionPad1d / ReplicationPad1d (melgan.py:70-72, residual_stack.py:49) of rows x t -> rows x
 * (pad_left + t + pad_right) and its adjoint (gather form, deterministic).  The forward convs fuse the
 * padding into their loaders; the train step materialises it once per layer so the weight / data
 * gradients run on the zero-padding kernels.  pad_mode: PWGB_PAD_REFLECT or PWGB_PAD_REPLICATE. */
PWGB_API int pwgb_pad1d_forward(const float* x, float* xp, long long rows, long long t, int pad_left, int pad_right,
                       int pad_mode, void* stream);
PWGB_API int pwgb_pad1d_backward(const float* gxp, float* gx, long long rows, long long t, int pad_left, int pad_right,
                        int pad_mode, void* stream);
/* adjoints of pwgb_stft_amplitude_forward (dx must be zero-initialised by the caller; frames overlap
 * so it is accumulated with atomics) and of the loss branch of pwgb_mel_project_forward. */
PWGB_API int pwgb_stft_amplitude_backward(const pwgb_stft_desc* d, const float* x, const float* window, const float* amp,
                                 const float* damp, float* dx, void* stream);
PWGB_API int pwgb_mel_project_backward(int batch, int frames, int bins, int n_mels, const float* amp_x, const float* amp_y,
                              const float* melmat, float eps, float log_scale, const float* gout, float* damp_x,
                              void* stream);

/* Training pieces of the Parallel WaveGAN step (config C3): WaveNet gate and its adjoint, adjoint of
 * pwgb_upsample_fir_forward (gx and/or the filter gradient), and the STFT loss on materialised
 * magnitudes (terms: out2 (+)= weight * {sc, mag}, sums3 = {S1, S2, S3} kept for the adjoint;
 * dmag: d loss / d xm given the upstream gradients gout2 = {g_sc, g_mag}). */
PWGB_API int pwgb_gate_forward(const float* g, float* z, int batch, int half_channels, long long t, void* stream);
PWGB_API int pwgb_gate_backward(const float* g, const float* gz, float* gg, int batch, int half_channels, long long t, void* stream);
PWGB_API int pwgb_upsample_fir_backward(int rows, int rows_per_batch, int t_in, int scale, const float* x, const float* fir,
                               const float* gy, long long gy_batch_stride, float* gx, float* dfir, void* stream);
PWGB_API int pwgb_stft_loss_terms(const float* xm, const float* ym, long long n, float weight, int accumulate, float* out2,
                         double* sums3, double* ws, int ws_doubles, void* stream);
PWGB_API int pwgb_stft_loss_dmag(const float* xm, const float* ym, long long n, const double* sums3, const float* gout2,
                        float weight, float* dxm, void* stream);

/* ------------------------------------------------------------------------
 * StyleMelGAN generator glue (layers/tade_res_block.py:56-75, 135-160; models/style_melgan.py:140-160).
 * The six k=9 convs of a TADEResBlock go through the conv entry points above; these are the element /
 * row kernels between them (inference; no adjoints yet):
 *   instance_norm:     torch.nn.InstanceNorm1d (biased variance, no affine) of rows x t, with an optional
 *                      LeakyReLU(pre_slope) applied to the input first (pre_slope = 1: none)
 *   upsample_nearest:  torch.nn.Upsample(scale_factor, "nearest"): y[r, o] = x[r, o / scale]
 *   leaky_relu:        y = LeakyReLU(x) (may run in place)
 *   tade_combine:      cg (B, 2C, t_out), xn (B, C, t_out / scale): y = cg[:, :C] * up(xn) + cg[:, C:]
 *   tade_gate:         x (B, 2C, t): y = gate(x[:, :C]) * tanh(x[:, C:]) [+ up(residual (B, C, t / scale))],
 *                      gate = softmax over channels (softmax != 0) or sigmoid
 * ---------------------------------------------------------------------- */
PWGB_API int pwgb_instance_norm_forward(const float* x, float* y, long long rows, long long t, float eps, float pre_slope,
                               void* stream);
PWGB_API int pwgb_upsample_nearest_forward(const float* x, float* y, long long rows, long long t_in, int scale, void* stream);
PWGB_API int pwgb_leaky_relu_forward(const float* x, float* y, long long n, float slope, void* stream);
PWGB_API int pwgb_tade_combine_forward(const float* cg, const float* xn, float* y, int batch, int channels, long long t_out,
                              int scale, void* stream);
PWGB_API int pwgb_tade_gate_forward(const float* x, const float* residual, float* y, int batch, int channels, long long t,
                           int scale, int softmax, void* stream);
/* adjoints of the four entry points above (StyleMelGAN generator training, layers/tade_res_block.py:52-160 under autograd):
 * instance_norm_backward recomputes the row statistics from x; the residual branch of tade_gate is the adjoint of
 * upsample_nearest (pwgb_upsample_nearest_backward on gy). */
PWGB_API int pwgb_instance_norm_backward(const float* x, const float* gy, float* gx, long long rows, long long t, float eps,
                                float pre_slope, void* stream);
PWGB_API int pwgb_upsample_nearest_backward(const float* gy, float* gx, long long rows, long long t_in, int scale, void* stream);
PWGB_API int pwgb_tade_combine_backward(const float* cg, const float* xn, const float* gy, float* gcg, float* gxn, int batch,
                               int channels, long long t_out, int scale, void* stream);
PWGB_API int pwgb_tade_gate_backward(const float* x, const float* gy, float* gx, int batch, int channels, long long t, int softmax,
                            void* stream);

/* ------------------------------------------------------------------------
 * Discrete-symbol HiFi-GAN front end (models/hifigan.py:867-1289, layers/duration_predictor.py,
 * layers/length_regulator.py, layers/layer_norm.py, losses/duration_prediction_loss.py, bin/train.py:768-783).
 * Deterministic throughout: no float atomics, every reduction in a fixed order.
 *
 *   symbol_embed_forward: y (B, C, t_out) = table[idx[b, 0, j]] (+ spk_table[idx[b, 1, 0]]) -- the channel-major input
 *     of input_conv in one launch.  idx is read in place as int64 (idx_int64 = 1) or float32 truncated toward zero
 *     (torch's c.long()), with element strides for batch / channel / time (the speaker id is channel 1, frame 0).
 *     durations (B, len) int64 or null: length regulation -- frame t of row b takes the symbol j with
 *     prefix[j] <= t < prefix[j] + ds[b, j] (exclusive prefix sums per row); frames past a row's total are 0.  Without
 *     durations t_out == len.  An index outside its table is never read: the column (or, for the speaker, the item)
 *     is written as NaN.
 *   symbol_embed_backward: d_emb (num_embs, C) [and d_spk (num_spk, C)] from the frame-level gradient gy (B, C, t_out)
 *     (after regulation) and / or the symbol-level gradient gsym (B, C, len); either may be null.  Each symbol's frames
 *     are summed in time order, gsym added, and the (b, j) positions are counting-sorted by index (stable) and summed
 *     per (index, channel) in position order.  Rows no position uses get 0; there is no padding_idx.
 *     num_embs <= 8192.  Workspace: pwgb_symbol_embed_backward_workspace bytes.
 *   channel_layernorm_forward / _backward: LayerNorm over C at every (b, t) of (B, C, T) with biased variance, affine
 *     gamma / beta and eps; the forward optionally stores mean / rstd (B, T) for the backward, which writes dx and the
 *     two-level fixed-order dgamma / dbeta (workspace: pwgb_channel_layernorm_backward_workspace bytes).
 *   duration_loss_forward / _backward: out[0] = mean_i (x_i - log(d_i + offset))^2 with int64 d (MSELoss(mean) against
 *     log-domain targets); backward gx = gout[0] * 2 (x - log(d + offset)) / n.
 *   duration_round: with x: ds = max(0, rint(exp(x) - offset)) as int64 (rint: half to even, like torch.round); with
 *     x == null ds is the input.  totals[b] = sum_j ds[b, j].  zero_rule != 0 applies the length regulator's rule in
 *     place: when the whole batch sums to 0, rows that sum to 0 become all ones.  One launch.
 *   collate_runlength: run-length encoding of the cropped feature rows feats[(c_offsets[b] + f) * C + ch], f < frames,
 *     read as int64 by truncation (torch.unique_consecutive(dim=0, return_counts=True) per item).  codes == null: pass 1
 *     writes runs[b], the number of runs.  Else pass 2 writes codes (B, C, max_runs) and counts (B, max_runs), padded
 *     with pad_value / 0 past each item's runs.
 * ---------------------------------------------------------------------- */
PWGB_API int pwgb_symbol_embed_forward(const void* idx, int idx_int64, long long idx_batch_stride, long long idx_chan_stride,
                                       long long idx_time_stride, const float* table, int num_embs, const float* spk_table,
                                       int num_spk, const long long* durations, int batch, int len, int channels, int t_out,
                                       float* y, void* stream);
/* The embedding of a stream chunk of n frames (a centred discrete-symbol HiFi-GAN streamed with a fixed lookahead),
 * written into columns [y_col0, y_col0 + n) of y (batch, channels, y_len): column y_col0 + j of item b is
 * pwgb_symbol_embed_forward's column for symbol idx[b, 0, j] (same fp32 expression, same NaN rules), with the item's
 * latched speaker.  spk_latch (batch) int32 holds each item's speaker row (-2: outside the speaker table); an item whose
 * fresh flag is set takes the speaker of its chunk's first frame, idx[b, 1, 0], and latches it.  frame / end (batch)
 * int32: frame j of item b is signal frame frame[b] + j, and a frame at or past end[b] is stored as +0.0 (the whole
 * utterance's zero padding) without reading its index.  Without a speaker table spk_latch and fresh may be null. */
PWGB_API int pwgb_symbol_embed_stream_forward(const void* idx, int idx_int64, long long idx_batch_stride, long long idx_chan_stride,
                                              long long idx_time_stride, const float* table, int num_embs, const float* spk_table,
                                              int num_spk, int* spk_latch, const int* fresh, const int* frame, const int* end, int batch,
                                              int n, int channels, float* y, long long y_len, int y_col0, void* stream);
/* The duration stream's per-item queue of (symbol id, duration) entries: ring_id / ring_d (batch, queue_len) int64,
 * ring_state (batch, 4) int64 {tail, head, hoff, total} (entries [head, tail) queued at ring index i % queue_len, hoff
 * frames of entry head consumed, total: the sum of every appended duration) and counts (batch, 2) int64 {queued frames,
 * overflow flag}.
 *   duration_queue_append: column j of x (batch, m) log-durations is symbol frame[b] - lookahead + j; a symbol inside
 *     [0, end[b]) is final: its duration max(0, rint(exp(x) - offset)) (pwgb_duration_round's expression) and
 *     ids[b * ids_ld + j] are appended in column order, and dur_out (batch, m) (may be null) gets the duration or -1.
 *     A full queue sets the overflow flag and drops the entry.  zero_rule (batch) int32 flags, with m = 0: an item whose
 *     total is 0 gets duration 1 for every queued entry (the length regulator's all-zero rule for the item alone).
 *   symbol_regulate_stream_forward: columns [y_col0, y_col0 + n) of y (batch, channels, y_len) are the next n frames
 *     of each item's queue, each pwgb_symbol_embed_forward's column of its entry's symbol (same fp32 expression, NaN for
 *     an id outside the table); a frame past the queue, or at or past end[b] of the frame mask (frame j of item b is
 *     frame[b] + j), is +0.0.  head / hoff and the queued count then advance by the frames consumed, so a symbol's run
 *     may continue in a later call. */
PWGB_API int pwgb_duration_queue_append(const float* x, int m, const long long* ids, long long ids_ld, const int* frame, const int* end,
                                        int lookahead, float offset, const int* zero_rule, long long* ring_id, long long* ring_d,
                                        int queue_len, long long* ring_state, long long* counts, long long* dur_out, int batch,
                                        void* stream);
PWGB_API int pwgb_symbol_regulate_stream_forward(const float* table, int num_embs, const long long* ring_id, const long long* ring_d,
                                                 int queue_len, long long* ring_state, long long* counts, const int* frame, const int* end,
                                                 int batch, int n, int channels, float* y, long long y_len, int y_col0, void* stream);
PWGB_API size_t pwgb_symbol_embed_backward_workspace(int batch, int len, int channels, int num_embs);
PWGB_API int pwgb_symbol_embed_backward(const float* gy, const float* gsym, const void* idx, int idx_int64, long long idx_batch_stride,
                                        long long idx_chan_stride, long long idx_time_stride, const long long* durations, int batch,
                                        int len, int channels, int t_out, int num_embs, float* d_emb, int num_spk, float* d_spk,
                                        void* ws, size_t ws_bytes, void* stream);
PWGB_API int pwgb_channel_layernorm_forward(const float* x, const float* gamma, const float* beta, int batch, int channels, long long t,
                                            float eps, float* y, float* mean, float* rstd, void* stream);
PWGB_API size_t pwgb_channel_layernorm_backward_workspace(int batch, int channels, long long t);
PWGB_API int pwgb_channel_layernorm_backward(const float* x, const float* gy, const float* gamma, const float* mean, const float* rstd,
                                             int batch, int channels, long long t, float* dx, float* dgamma, float* dbeta, void* ws,
                                             size_t ws_bytes, void* stream);
PWGB_API int pwgb_duration_loss_forward(const float* x, const long long* d, long long n, float offset, float* out, void* stream);
PWGB_API int pwgb_duration_loss_backward(const float* x, const long long* d, long long n, float offset, const float* gout, float* gx,
                                         void* stream);
PWGB_API int pwgb_duration_round(const float* x, long long* ds, long long* totals, int batch, int len, float offset, int zero_rule,
                                 void* stream);
PWGB_API int pwgb_collate_runlength(const float* feats, const long long* c_offsets, int batch, int channels, int frames, long long* runs,
                                    long long* codes, long long* counts, int max_runs, long long pad_value, void* stream);

/* ------------------------------------------------------------------------
 * VQ-VAE bottleneck (models/vqvae.py, layers/vector_quantize_codebook.py, functions/vector_quantizer.py).
 *
 *   vq_forward: with z_e (B, D, T) fp32 channel-major (read in place), the nearest code of every frame,
 *     d_k = fl(fl(c_sqr[k] + x_sqr) - 2 dot(x, c_k)) with dot, x_sqr and c_sqr accumulated by FFMA over d = 0 .. D-1,
 *     argmin as torch.min(dim): ties to the lower index, a NaN distance wins and the first NaN is taken; written to
 *     indices (B, T) int64.  With z_e == null the search is skipped and indices is read (VQVAE.decode).  Then, for
 *     every frame, z_q (B, D, T) = codebook[index] if z_q is given, and the decoder input dec (B, D + Cl + Cg, T) if
 *     given: channels [0, D) the gathered codes, [D, D + Cl) copied from l (B, Cl, T), [D + Cl, D + Cl + Cg)
 *     global_table[g[b]] broadcast over time.  An index outside [0, K) or a g[b] outside the table is never read: the
 *     frame's (or the item's) z_q / dec columns are NaN.  One launch.  D <= 768.
 *   vq_backward: from the gradient of dec, gz_e (+)= gdec[:, :D] (the straight-through gradient of z_e) and
 *     d_global_table (num_global, Cg) = per table row, in item order, the per-item sums over time of gdec[:, D + Cl:]
 *     (rows no item uses get 0).  Either output may be null.  The codebook gradient is pwgb_symbol_embed_backward on
 *     the indices; the local slice belongs to the local embedding's conv backward.
 * ---------------------------------------------------------------------- */
PWGB_API int pwgb_vq_forward(const float* z_e, const float* codebook, int num_codes, long long* indices, float* z_q, float* dec,
                             const float* l, int local_channels, const float* global_table, const long long* g, int num_global,
                             int global_channels, int batch, int dim, int t, void* stream);
PWGB_API int pwgb_vq_backward(const float* gdec, int batch, int dim, int local_channels, int global_channels, int t, float* gz_e,
                              int accumulate, const long long* g, int num_global, float* d_global_table, void* stream);
/* The bottleneck of a streamed VQ-VAE: pwgb_vq_forward (search and assembly, the same code) on one chunk of t frames
 * of z_e (search required, no z_q), with two stream extensions:
 *   l: row j of the local conditioning is row j of the window [l_hist (B, Cl, l_delay) | l (B, Cl, t)], so l arrives
 *     l_delay frames before the z_e frames it goes with (the encoder's lookahead in frames);
 *   ext: a mask at the frame rate (rate 1, no residual, no edge policy): frame j of item b is signal frame
 *     frame[b] - lookahead + j; outside [0, end[b]) every dec channel is stored as +0.0 and the index as -1.
 * Inside the signal each frame's index and dec column equal pwgb_vq_forward's on the same z_e column, l column and g
 * (NaN rules included): the search of a frame does not depend on its place in the launch. */
PWGB_API int pwgb_vq_stream_forward(const float* z_e, const float* codebook, int num_codes, long long* indices, float* dec,
                                    const float* l, const float* l_hist, int l_delay, int local_channels, const float* global_table,
                                    const long long* g, int num_global, int global_channels, const pwgb_stream_ext* ext, int batch,
                                    int dim, int t, void* stream);

/* ------------------------------------------------------------------------
 * SineGen excitation (layers/sine.py SineGen.forward, flag_for_pulse=False) for `batch` rows of f0 (batch, t) fp32 at
 * the sample rate, dim = harmonic_num + 1.  The random draws come from the caller: rand_ini (batch, dim) uniform, of
 * which column 0 is ignored (the reference zeroes it), and noise_in (batch, t, dim) standard normal.  Writes
 * sine_waves (batch, t, dim), uv (batch, t) and noise (batch, t, dim); phase (batch, t, dim), the fp32 argument of
 * sin, is written when non-null.  Every elementwise step is the reference's fp32 operation in its order; the two
 * prefix sums accumulate in fp64 and round each output to fp32, as CPU torch.cumsum on fp32 does, and equal the
 * sequential sums while every partial sum is exact in fp64 (DESIGN.md §3.15).  Deterministic: five launches, no
 * atomics.  ws: pwgb_sine_gen_workspace(batch, t, harmonic_num) bytes of device memory.  batch <= 65535.
 * ---------------------------------------------------------------------- */
PWGB_API size_t pwgb_sine_gen_workspace(int batch, long long t, int harmonic_num);
PWGB_API int pwgb_sine_gen_forward(const float* f0, int batch, long long t, int harmonic_num, float samp_rate, float sine_amp,
                                   float noise_std, float voiced_threshold, const float* rand_ini, const float* noise_in,
                                   float* sine_waves, float* uv, float* noise, float* phase, void* ws, size_t ws_bytes,
                                   void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PWGB_H_ */
