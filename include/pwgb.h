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

enum { PWGB_PAD_ZERO = 0, PWGB_PAD_REFLECT = 1, PWGB_PAD_REPLICATE = 2 };
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
/* measurement aids (not part of the product contract): set key 1 = conv variant (bit 1: stage activations with
 * cp.async instead of TMA); get returns -1 (no read-back available). */
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
 * pwgb_pcm16_forward: lrintf(y * 32767) saturated to int16 -- libsndfile's float -> PCM_16 (decode.py:236-241).
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
 * halo >= (kernel-1)/2 * (largest dilation of the stack).  Weights: the image written by
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

/* ------------------------------------------------------------------------
 * One stage of the PWG conditioning upsampler (layers/upsample.py:112-128): nearest repeat
 * x`scale` along time followed by the (2*scale+1)-tap FIR shared by all rows, zero padded:
 *   y[r, o] = sum_k f[k] * x[r, (o + k - scale) / scale]   for 0 <= o + k - scale < t_in*scale.
 * x: rows x t_in (row stride t_in); y: row r of batch item r / rows_per_batch starts at
 * (r / rows_per_batch) * y_batch_stride + (r % rows_per_batch) * t_in * scale.
 * ---------------------------------------------------------------------- */
PWGB_API int pwgb_upsample_fir_forward(int rows, int rows_per_batch, int t_in, int scale, const float* x, const float* fir,
                              float* y, long long y_batch_stride, void* stream);

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
 * mode 0: (x-c)^2, 1: |x-y|, 2: max(0, c - s*x), 3: s*x.  ws: >= 1 float of scratch
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

#ifdef __cplusplus
}
#endif
#endif /* PWGB_H_ */
