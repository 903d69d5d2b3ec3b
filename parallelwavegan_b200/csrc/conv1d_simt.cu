// Generic fused 1-D convolution, fp32 FFMA path (any channel count / stride / dilation /
// groups / period).  This is the exact-arithmetic path: narrow layers (Cin or Cout < 16,
// grouped and strided discriminator convs) always use it, and it is the in-library
// cross-check for the tensor-core path (conv1d_tc.cu) that takes the wide stride-1 layers.
//
// Tiling: one CTA = CO_T output channels x TT output positions of one batch item.
// 8 warps = WARPS_CO (channel sub-tiles of RCO channels) x WARPS_T (time sub-tiles of
// 128 positions); lanes run along time so that x reads from shared memory are
// conflict-free and weight reads are warp-wide broadcasts (float4).  The input tile
// (with halo, padding policy and pre-activation already applied) and the weight slice
// are staged in shared memory per CI_T input channels; im2col is never materialised.
#include <stdarg.h>

#include "common.cuh"

namespace pwgb {

struct ConvK {
  int B, Cin, Cout, Cin_g, Cout_g, groups;
  int t_in, t_out, K, S, D, padL, pad_mode, P, t_valid;
  int Lin, Lout;
  float pre_slope;
  int pre_gate;
  int post_act;
  float post_slope;
  float out_scale;
  int accumulate;
  int shuffle, shuffle_pad, shuffle_tout;
  long long xbs, ybs, rbs, xcs;
  int CI_T, XW, tiles_per_group;
};

template <int RCO, int WARPS_CO, int RT>
__global__ void __launch_bounds__(256) conv1d_fwd_kernel(const ConvK p, const float* __restrict__ x,
                                                          const float* __restrict__ w,
                                                          const float* __restrict__ bias,
                                                          const float* __restrict__ res, float* __restrict__ y) {
  constexpr int WARPS_T = 8 / WARPS_CO;
  constexpr int CO_T = RCO * WARPS_CO;
  constexpr int TT = WARPS_T * 32 * RT;
  constexpr int WS = (CO_T % 4 == 0) ? CO_T + 4 : CO_T;

  extern __shared__ __align__(16) float smem[];
  float* xs = smem;
  float* wsm = smem + ((p.CI_T * p.XW + 3) & ~3);

  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int warp = tid >> 5;
  const int warp_co = warp % WARPS_CO;
  const int warp_t = warp / WARPS_CO;
  const int b = blockIdx.z;
  const int g = blockIdx.y / p.tiles_per_group;
  const int co0 = g * p.Cout_g + (blockIdx.y % p.tiles_per_group) * CO_T;
  const int co_end = (g + 1) * p.Cout_g;
  const int tile_start = blockIdx.x * TT;
  const int tile_to0 = tile_start / p.P;
  const long long row0 = (long long)tile_to0 * p.S - p.padL;

  int o_r[RT], xoff[RT];
#pragma unroll
  for (int r = 0; r < RT; ++r) {
    int o = tile_start + warp_t * (32 * RT) + lane + 32 * r;
    o_r[r] = o;
    int oc = o < p.Lout ? o : tile_start;
    int to = oc / p.P;
    int j = oc - to * p.P;
    xoff[r] = (to - tile_to0) * p.S * p.P + j;
  }

  float acc[RCO][RT];
#pragma unroll
  for (int c = 0; c < RCO; ++c)
#pragma unroll
    for (int r = 0; r < RT; ++r) acc[c][r] = 0.f;

  const float* xb = x + (long long)b * p.xbs;
  const int kdp = p.D * p.P;

  for (int ci0 = 0; ci0 < p.Cin_g; ci0 += p.CI_T) {
    const int cit = min(p.CI_T, p.Cin_g - ci0);
    __syncthreads();
    // ---- stage the input tile: padding policy + source reflect extension + pre-activation
    for (int idx = tid; idx < cit * p.XW; idx += 256) {
      int ci = idx / p.XW;
      int r = idx - ci * p.XW;
      long long li = row0 * p.P + r;
      float v = 0.f;
      bool ok = true;
      if (li < 0 || li >= p.Lin) {
        if (p.pad_mode == PWGB_PAD_ZERO) {
          ok = false;
        } else if (p.pad_mode == PWGB_PAD_REFLECT) {
          li = li < 0 ? -li : 2LL * (p.Lin - 1) - li;
          li = li < 0 ? 0 : (li >= p.Lin ? p.Lin - 1 : li);
        } else {
          li = li < 0 ? 0 : p.Lin - 1;
        }
      }
      if (ok) {
        if (li >= p.t_valid) li = 2LL * (p.t_valid - 1) - li;
        if (li < 0) li = 0;
        const int ch = g * p.Cin_g + ci0 + ci;
        if (p.pre_gate) {
          float a = __ldg(xb + (long long)ch * p.xcs + li);
          float s = __ldg(xb + (long long)(ch + p.Cin) * p.xcs + li);
          v = tanhf(a) * sigmoidf_(s);
        } else {
          v = lrelu(__ldg(xb + (long long)ch * p.xcs + li), p.pre_slope);
        }
      }
      xs[idx] = v;
    }
    // ---- stage the weight slice transposed to [ci][k][co] (co fastest, broadcast reads)
    {
      const int per_co = cit * p.K;
      for (int idx = tid; idx < CO_T * per_co; idx += 256) {
        int co_l = idx / per_co;
        int rem = idx - co_l * per_co;
        int co = co0 + co_l;
        float v = 0.f;
        if (co < co_end) v = __ldg(w + ((long long)co * p.Cin_g + ci0) * p.K + rem);
        wsm[rem * WS + co_l] = v;
      }
    }
    __syncthreads();
    // ---- FFMA main loop
    for (int ci = 0; ci < cit; ++ci) {
      const float* xrow = xs + ci * p.XW;
      const float* wrow = wsm + (ci * p.K) * WS + warp_co * RCO;
#pragma unroll 2
      for (int k = 0; k < p.K; ++k) {
        float xv[RT];
#pragma unroll
        for (int r = 0; r < RT; ++r) xv[r] = xrow[xoff[r] + k * kdp];
        float wv[RCO];
        if constexpr (RCO % 4 == 0) {
#pragma unroll
          for (int c = 0; c < RCO; c += 4) {
            float4 t = *reinterpret_cast<const float4*>(wrow + k * WS + c);
            wv[c] = t.x;
            wv[c + 1] = t.y;
            wv[c + 2] = t.z;
            wv[c + 3] = t.w;
          }
        } else {
#pragma unroll
          for (int c = 0; c < RCO; ++c) wv[c] = wrow[k * WS + c];
        }
#pragma unroll
        for (int c = 0; c < RCO; ++c)
#pragma unroll
          for (int r = 0; r < RT; ++r) acc[c][r] = fmaf(wv[c], xv[r], acc[c][r]);
      }
    }
  }

  // ---- epilogue: bias, activation, residual, scale, (accumulate), (pixel shuffle)
#pragma unroll
  for (int c = 0; c < RCO; ++c) {
    const int co = co0 + warp_co * RCO + c;
    if (co >= co_end) continue;
    const float bv = bias ? __ldg(bias + (p.shuffle > 1 ? co / p.shuffle : co)) : 0.f;
#pragma unroll
    for (int r = 0; r < RT; ++r) {
      const int o = o_r[r];
      if (o >= p.Lout) continue;
      float v = acc[c][r] + bv;
      if (p.post_act == PWGB_ACT_TANH)
        v = tanhf(v);
      else if (p.post_act == PWGB_ACT_LRELU)
        v = lrelu(v, p.post_slope);
      long long yi;
      if (p.shuffle > 1) {
        const int cof = co / p.shuffle;
        const int ph = co - cof * p.shuffle;
        const int to = o / p.P;
        const int jj = o - to * p.P;
        const int of = to * p.shuffle + ph - p.shuffle_pad;  // output row
        if (of < 0 || of >= p.shuffle_tout) continue;
        yi = (long long)b * p.ybs + ((long long)cof * p.shuffle_tout + of) * p.P + jj;
      } else {
        yi = (long long)b * p.ybs + (long long)co * p.Lout + o;
      }
      if (res) v += __ldg(res + (long long)b * p.rbs + (long long)co * p.Lout + o);
      v *= p.out_scale;
      if (p.accumulate) v += y[yi];
      y[yi] = v;
    }
  }
}

template <int RCO, int WARPS_CO, int RT>
static int launch_conv_rt(ConvK p, const float* x, const float* w, const float* bias, const float* res, float* y,
                       cudaStream_t st) {
  constexpr int WARPS_T = 8 / WARPS_CO;
  constexpr int CO_T = RCO * WARPS_CO;
  constexpr int TT = WARPS_T * 32 * RT;
  constexpr int WS = (CO_T % 4 == 0) ? CO_T + 4 : CO_T;
  const int nrows_out = (TT + p.P - 2) / p.P + 1;
  const long long NR = (long long)(nrows_out - 1) * p.S + (long long)(p.K - 1) * p.D + 1;
  const long long XW = NR * p.P;
  const size_t limit = 96 * 1024;
  int ci_t = p.Cin_g < 16 ? p.Cin_g : 16;
  size_t bytes = 0;
  for (;; ci_t = ci_t / 2) {
    bytes = ((size_t)((ci_t * XW + 3) & ~3LL) + (size_t)ci_t * p.K * WS) * sizeof(float);
    if (bytes <= limit || ci_t <= 1) break;
  }
  if (bytes > 200 * 1024) {
    set_error("conv1d: tile does not fit shared memory (K=%d dilation=%d stride=%d period=%d)", p.K, p.D, p.S, p.P);
    return PWGB_UNSUPPORTED;
  }
  p.CI_T = ci_t;
  p.XW = (int)XW;
  p.tiles_per_group = ceil_div(p.Cout_g, CO_T);
  auto kern = conv1d_fwd_kernel<RCO, WARPS_CO, RT>;
  if (bytes > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) {
      set_error("conv1d: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      return PWGB_CUDA_ERROR;
    }
  }
  dim3 grid(ceil_div(p.Lout, TT), p.tiles_per_group * p.groups, p.B);
  if (grid.y > 65535 || grid.z > 65535) {
    set_error("conv1d: grid too large");
    return PWGB_UNSUPPORTED;
  }
  kern<<<grid, 256, bytes, st>>>(p, x, w, bias, res, y);
  return check_launch("conv1d_fwd_kernel");
}

// Few output channels (logit convs of the discriminators, cin up to 1024 -> cout 1) with short
// sequences: the generic tiling would launch a handful of CTAs.  Here one CTA = 32 output positions
// x all (<= 4) output channels; its 8 warps split the input channels and reduce through shared memory.
__global__ void __launch_bounds__(256) conv1d_small_cout_kernel(const ConvK p, const float* __restrict__ x,
                                                                 const float* __restrict__ w,
                                                                 const float* __restrict__ bias,
                                                                 float* __restrict__ y) {
  __shared__ float red[8][4][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.y;
  const int o = blockIdx.x * 32 + lane;
  const bool ov = o < p.Lout;
  const int oc = ov ? o : 0;
  const int to = oc / p.P, j = oc - to * p.P;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  const float* xb = x + (long long)b * p.xbs;
  for (int ci = warp; ci < p.Cin; ci += 8) {
    const float* xc = xb + (long long)ci * p.xcs;
    for (int k = 0; k < p.K; ++k) {
      const long long row = (long long)to * p.S + (long long)k * p.D - p.padL;
      float v = 0.f;
      if (row >= 0 && row < p.t_in) {
        long long li = row * p.P + j;
        if (li >= p.t_valid) li = 2LL * (p.t_valid - 1) - li;
        v = lrelu(__ldg(xc + (li < 0 ? 0 : li)), p.pre_slope);
      }
      for (int co = 0; co < p.Cout; ++co) acc[co] = fmaf(v, __ldg(w + ((long long)co * p.Cin + ci) * p.K + k), acc[co]);
    }
  }
  for (int co = 0; co < 4; ++co) red[warp][co][lane] = acc[co];
  __syncthreads();
  if (warp < p.Cout && ov) {
    float v = bias ? __ldg(bias + warp) : 0.f;
    for (int i = 0; i < 8; ++i) v += red[i][warp][lane];
    if (p.post_act == PWGB_ACT_TANH)
      v = tanhf(v);
    else if (p.post_act == PWGB_ACT_LRELU)
      v = lrelu(v, p.post_slope);
    y[(long long)b * p.ybs + (long long)warp * p.Lout + o] = v * p.out_scale;
  }
}

// Few output channels over LONG sequences (the generators' output convs: 32 -> 1 k7 at 16 x 102400
// samples, MelGAN 32 -> 4): HBM-bound by the input read.  One CTA = 1024 consecutive positions, a
// thread owns positions tid + 256 q (coalesced, L1-resident taps), the whole weight tensor sits in
// shared memory (broadcast reads) and all CO accumulators stay in registers.
template <int CO>
__global__ void __launch_bounds__(256) conv1d_fewcout_long_kernel(const ConvK p, const float* __restrict__ x,
                                                                  const float* __restrict__ w,
                                                                  const float* __restrict__ bias,
                                                                  float* __restrict__ y) {
  extern __shared__ __align__(16) float wsm[];  // [ci][k][CO]
  for (int i = threadIdx.x; i < p.Cin * p.K * CO; i += 256) {
    const int co = i % CO, ck = i / CO;
    wsm[i] = co < p.Cout ? __ldg(w + (long long)co * p.Cin * p.K + ck) : 0.f;
  }
  __syncthreads();
  const int b = blockIdx.y;
  const int o0 = blockIdx.x * 1024 + threadIdx.x;
  const float* xb = x + (long long)b * p.xbs;
  float acc[4][CO];
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int co = 0; co < CO; ++co) acc[q][co] = 0.f;
  const long long first = (long long)blockIdx.x * 1024;
  const bool interior = first * p.S - p.padL >= 0 && (first + 1023) * p.S + (long long)(p.K - 1) * p.D - p.padL < p.t_in &&
                        first + 1023 < p.t_out;
  if (interior) {
    // no padding inside this CTA: channel-outer / tap-inner so the K re-reads of a row hit L1 at once
    const float* xq = xb + (long long)o0 * p.S - p.padL;
    const long long qs = 256LL * p.S;
    const float* wk = wsm;
    for (int ci = 0; ci < p.Cin; ++ci, xq += p.xcs) {
      for (int k = 0; k < p.K; ++k, wk += CO) {
        const float* xk = xq + (long long)k * p.D;
        float v[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) v[q] = lrelu(__ldg(xk + q * qs), p.pre_slope);
#pragma unroll
        for (int co = 0; co < CO; ++co) {
          const float wv = wk[co];
#pragma unroll
          for (int q = 0; q < 4; ++q) acc[q][co] = fmaf(v[q], wv, acc[q][co]);
        }
      }
    }
  } else
  for (int k = 0; k < p.K; ++k) {
    // source row of every owned position for this tap (padding policy resolved once per tap)
    long long row[4];
    bool ok[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      long long r = (long long)(o0 + 256 * q) * p.S + (long long)k * p.D - p.padL;
      ok[q] = o0 + 256 * q < p.t_out;
      if (r < 0 || r >= p.t_in) {
        if (p.pad_mode == PWGB_PAD_ZERO) {
          ok[q] = false;
        } else if (p.pad_mode == PWGB_PAD_REFLECT) {
          r = r < 0 ? -r : 2LL * (p.t_in - 1) - r;
          ok[q] = ok[q] && r >= 0 && r < p.t_in;
        } else {
          r = r < 0 ? 0 : p.t_in - 1;
        }
      }
      row[q] = ok[q] ? r : 0;
    }
    const float* wk = wsm + k * CO;
    const float* xc = xb;
#pragma unroll 4
    for (int ci = 0; ci < p.Cin; ++ci, xc += p.xcs, wk += p.K * CO) {
      float v[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) v[q] = ok[q] ? lrelu(__ldg(xc + row[q]), p.pre_slope) : 0.f;
#pragma unroll
      for (int co = 0; co < CO; ++co) {
        const float wv = wk[co];
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[q][co] = fmaf(v[q], wv, acc[q][co]);
      }
    }
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int o = o0 + 256 * q;
    if (o >= p.t_out) continue;
#pragma unroll
    for (int co = 0; co < CO; ++co) {
      if (co >= p.Cout) break;
      float v = acc[q][co] + (bias ? __ldg(bias + co) : 0.f);
      if (p.post_act == PWGB_ACT_TANH)
        v = tanhf(v);
      else if (p.post_act == PWGB_ACT_LRELU)
        v = lrelu(v, p.post_slope);
      y[(long long)b * p.ybs + (long long)co * p.t_out + o] = v * p.out_scale;
    }
  }
}

// short sequences (discriminator tails, 10-50 positions per item): 1 position per lane instead of 4
template <int RCO, int WARPS_CO>
static int launch_conv(ConvK p, const float* x, const float* w, const float* bias, const float* res, float* y,
                       cudaStream_t st) {
  constexpr int WARPS_T = 8 / WARPS_CO;
  if (p.Lout <= 40 * WARPS_T) return launch_conv_rt<RCO, WARPS_CO, 1>(p, x, w, bias, res, y, st);
  return launch_conv_rt<RCO, WARPS_CO, 4>(p, x, w, bias, res, y, st);
}

int conv1d_forward_simt(const pwgb_conv1d_desc* d, const float* x, const float* w, const float* bias,
                        const float* residual, float* y, cudaStream_t st) {
  ConvK p;
  p.B = d->batch;
  p.Cin = d->cin;
  p.Cout = d->cout;
  p.groups = d->groups;
  p.Cin_g = d->cin / d->groups;
  p.Cout_g = d->cout / d->groups;
  p.t_in = d->t_in;
  p.t_out = d->t_out;
  p.K = d->kernel;
  p.S = d->stride;
  p.D = d->dilation;
  p.padL = d->pad_left;
  p.pad_mode = d->pad_mode;
  p.P = d->period < 1 ? 1 : d->period;
  p.Lin = d->t_in * p.P;
  p.Lout = d->t_out * p.P;
  p.t_valid = d->t_valid > 0 ? d->t_valid : p.Lin;
  p.pre_slope = d->pre_slope;
  p.pre_gate = d->pre_gate;
  p.post_act = d->post_act;
  p.post_slope = d->post_slope;
  p.out_scale = d->out_scale;
  p.accumulate = d->accumulate;
  p.shuffle = d->shuffle;
  p.shuffle_pad = d->shuffle_pad;
  p.shuffle_tout = d->shuffle_tout;
  p.xcs = p.t_valid;
  const long long cin_total = (long long)d->cin * (d->pre_gate ? 2 : 1);
  p.xbs = d->x_batch_stride ? d->x_batch_stride : cin_total * p.xcs;
  const long long ylen = d->shuffle > 1 ? (long long)(d->cout / d->shuffle) * d->shuffle_tout * p.P : (long long)d->cout * p.Lout;
  p.ybs = d->y_batch_stride ? d->y_batch_stride : ylen;
  p.rbs = d->r_batch_stride ? d->r_batch_stride : (long long)d->cout * p.Lout;
  if (p.B == 0 || p.Lout == 0) return PWGB_OK;
  if (p.Cout <= 4 && p.groups == 1 && p.Cin >= 64 && p.pad_mode == PWGB_PAD_ZERO && !p.pre_gate && !residual &&
      !p.accumulate && p.shuffle <= 1 && (long long)p.Lout * p.B <= 65536 && p.B <= 65535) {
    conv1d_small_cout_kernel<<<dim3(ceil_div(p.Lout, 32), p.B), 256, 0, st>>>(p, x, w, bias, y);
    return check_launch("conv1d_small_cout_kernel");
  }
  if (p.Cout <= 4 && p.groups == 1 && p.P == 1 && p.t_valid == p.Lin && !p.pre_gate && !residual && !p.accumulate &&
      p.shuffle <= 1 && p.t_out >= 4096 && p.B <= 65535 && (size_t)p.Cin * p.K * 4 * sizeof(float) <= 40 * 1024) {
    const dim3 grid(ceil_div(p.t_out, 1024), p.B);
    if (p.Cout == 1) {
      conv1d_fewcout_long_kernel<1><<<grid, 256, (size_t)p.Cin * p.K * sizeof(float), st>>>(p, x, w, bias, y);
    } else if (p.Cout == 2) {
      conv1d_fewcout_long_kernel<2><<<grid, 256, (size_t)p.Cin * p.K * 2 * sizeof(float), st>>>(p, x, w, bias, y);
    } else {
      conv1d_fewcout_long_kernel<4><<<grid, 256, (size_t)p.Cin * p.K * 4 * sizeof(float), st>>>(p, x, w, bias, y);
    }
    return check_launch("conv1d_fewcout_long_kernel");
  }
  const int cg = p.Cout_g;
  if (cg >= 64) return launch_conv<8, 8>(p, x, w, bias, residual, y, st);
  if (cg >= 32) return launch_conv<8, 4>(p, x, w, bias, residual, y, st);
  if (cg >= 16) return launch_conv<8, 2>(p, x, w, bias, residual, y, st);
  if (cg >= 8) return launch_conv<8, 1>(p, x, w, bias, residual, y, st);
  if (cg >= 4) return launch_conv<4, 1>(p, x, w, bias, residual, y, st);
  return launch_conv<1, 1>(p, x, w, bias, residual, y, st);
}

}  // namespace pwgb
