// Backward building blocks for the train step (bin/train.py:189-340 calls loss.backward()):
//   * wgrad of the generic fused Conv1d (any stride / dilation / groups / period view),
//     deterministic two-stage split reduction;
//   * data gradients reuse the FORWARD kernels (a stride-1 dgrad is a conv with the transposed,
//     tap-flipped weight -> tensor-core path; a strided dgrad is the poly-phase conv-transpose), so only
//     the elementwise chain-rule pieces live here: activation masks, bias sums, loss / pooling grads.
#include <cooperative_groups.h>

#include "common.cuh"

namespace pwgb {

// ------------------------------------------------------------------ wgrad
struct WgK {
  int B, Cin, Cout, Cin_g, Cout_g, groups;
  int t_in, t_out, K, S, D, padL, pad_mode, P, t_valid;
  int Lin, Lout;
  float x_slope;   // LeakyReLU applied to x on load (the conv's fused pre-activation)
  float g_slope;   // LeakyReLU applied to the gradient operand on load (conv-transpose wgrad)
  long long xcs;
  int nsplit, chunks_per_seq, XW, ci_tiles;
};

constexpr int WG_CO = 32, WG_CI = 8, WG_K = 8, WG_T = 128;

// partial[split][co][ci_g][k] += sum over this split's (batch, chunk) items of g[co,o] * x~[ci, src(o,k)]
__global__ void __launch_bounds__(256) conv1d_wgrad_kernel(const WgK p, const float* __restrict__ x,
                                                            const float* __restrict__ gy, float* __restrict__ part) {
  extern __shared__ float sm[];
  float* gs = sm;                         // WG_CO x (WG_T + 1)
  float* xs = gs + WG_CO * (WG_T + 1);    // WG_CI x XW
  int* xoff = reinterpret_cast<int*>(xs + WG_CI * p.XW);  // WG_T
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tiles_co = ceil_div(p.Cout_g, WG_CO);
  const int g = blockIdx.x / (tiles_co * p.ci_tiles);
  const int rem = blockIdx.x - g * tiles_co * p.ci_tiles;
  const int co0 = g * p.Cout_g + (rem / p.ci_tiles) * WG_CO;
  const int ci0 = (rem % p.ci_tiles) * WG_CI;  // within group
  const int k0 = blockIdx.y * WG_K;
  const int split = blockIdx.z;
  const int co = co0 + lane;
  const bool co_ok = co < (g + 1) * p.Cout_g;
  const int ci = ci0 + warp;
  const bool ci_ok = ci < p.Cin_g;
  float acc[WG_K];
#pragma unroll
  for (int k = 0; k < WG_K; ++k) acc[k] = 0.f;
  const int kdp = p.D * p.P;
  const int total_items = p.B * p.chunks_per_seq;
  for (int item = split; item < total_items; item += p.nsplit) {
    const int b = item / p.chunks_per_seq;
    const int o0 = (item - b * p.chunks_per_seq) * WG_T;
    const int to0 = o0 / p.P;
    const long long row0 = (long long)to0 * p.S + (long long)k0 * p.D - p.padL;
    __syncthreads();
    for (int idx = tid; idx < WG_CO * WG_T; idx += 256) {
      const int c = idx / WG_T, o = idx - c * WG_T;
      const int cc = co0 + c;
      float v = 0.f;
      if (cc < (g + 1) * p.Cout_g && o0 + o < p.Lout) v = lrelu(gy[((long long)b * p.Cout + cc) * p.Lout + o0 + o], p.g_slope);
      gs[c * (WG_T + 1) + o] = v;
    }
    for (int o = tid; o < WG_T; o += 256) {
      const int oo = min(o0 + o, p.Lout - 1);
      const int to = oo / p.P;
      xoff[o] = (to - to0) * p.S * p.P + (oo - to * p.P);
    }
    for (int idx = tid; idx < WG_CI * p.XW; idx += 256) {
      const int c = idx / p.XW, r = idx - c * p.XW;
      long long li = row0 * p.P + r;
      float v = 0.f;
      bool ok = ci0 + c < p.Cin_g;
      if (ok && (li < 0 || li >= p.Lin)) {
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
        v = lrelu(x[((long long)b * p.Cin + g * p.Cin_g + ci0 + c) * p.xcs + li], p.x_slope);
      }
      xs[idx] = v;
    }
    __syncthreads();
    if (co_ok && ci_ok) {
      const float* gr = gs + lane * (WG_T + 1);
      const float* xr = xs + warp * p.XW;
      const int nv = min(WG_T, p.Lout - o0);
      for (int o = 0; o < nv; ++o) {
        const float gv = gr[o];
        const float* xq = xr + xoff[o];
#pragma unroll
        for (int k = 0; k < WG_K; ++k) acc[k] = fmaf(gv, xq[k * kdp], acc[k]);
      }
    }
  }
  if (co_ok && ci_ok) {
    float* dst = part + (((long long)split * p.Cout + co) * p.Cin_g + ci) * p.K + k0;
#pragma unroll
    for (int k = 0; k < WG_K; ++k)
      if (k0 + k < p.K) dst[k] = acc[k];
  }
}

// Narrow weight gradients (cin/groups <= 4 or cout <= 4: waveform-side and logit convs): few outputs, very long
// reduction.  One warp owns one (co, ci) pair over a 1024-position chunk of one batch item: the gradient chunk stays
// in registers (32 values per lane, coalesced), every tap is a register x L1-resident-input dot product reduced with
// shuffles.  grid = (pairs / 8, batch * chunks): thousands of CTAs even for a 1 -> 128 conv (the first version gave a
// CTA all 1920 outputs of such a layer and ran for 5.6 ms at the C5 batch).
constexpr int WGN_CHUNK = 1024;
__global__ void __launch_bounds__(256) conv1d_wgrad_narrow_kernel(const WgK p, const float* __restrict__ x,
                                                                   const float* __restrict__ gy, float* __restrict__ part) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int npairs = p.Cout * p.Cin_g;
  const int q = blockIdx.x * 8 + warp;
  if (q >= npairs) return;
  const int b = blockIdx.y / p.chunks_per_seq;
  const int o0 = (blockIdx.y - b * p.chunks_per_seq) * WGN_CHUNK;
  const int co = q / p.Cin_g, ci = q - co * p.Cin_g;
  const int g = co / p.Cout_g;
  const float* gr = gy + ((long long)b * p.Cout + co) * p.Lout;
  const float* xr = x + ((long long)b * p.Cin + g * p.Cin_g + ci) * p.xcs;
  float gv[WGN_CHUNK / 32];
  int base[WGN_CHUNK / 32];  // input row of tap 0 for each position; far negative: position beyond the end
  int colj[WGN_CHUNK / 32];
#pragma unroll
  for (int j = 0; j < WGN_CHUNK / 32; ++j) {
    const int o = o0 + lane + 32 * j;
    const bool ok = o < p.Lout;
    gv[j] = ok ? lrelu(__ldg(gr + o), p.g_slope) : 0.f;
    const int to = ok ? o / p.P : 0;
    colj[j] = ok ? o - to * p.P : 0;
    base[j] = ok ? to * p.S - p.padL : -(1 << 30);
  }
  float* dst = part + ((long long)blockIdx.y * npairs + q) * p.K;
  if (p.P == 1 && p.S == 1 && p.t_valid >= p.t_in) {
    // plain stride-1 conv (the 1 -> C and C -> 1 layers of the generators / discriminators): row = o - pad + k * D,
    // no period view, no reflect extension -- 32-bit index arithmetic only
    for (int k = 0; k < p.K; ++k) {
      float acc = 0.f;
      const int r0 = o0 + lane - p.padL + k * p.D;
#pragma unroll
      for (int j = 0; j < WGN_CHUNK / 32; ++j) {
        const int row = r0 + 32 * j;
        if (row >= 0 && row < p.t_in) acc = fmaf(gv[j], lrelu(__ldg(xr + row), p.x_slope), acc);
      }
#pragma unroll
      for (int sft = 16; sft > 0; sft >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, sft);
      if (lane == 0) dst[k] = acc;
    }
    return;
  }
  for (int k = 0; k < p.K; ++k) {
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < WGN_CHUNK / 32; ++j) {
      const int row = base[j] + k * p.D;
      if (row >= 0 && row < p.t_in) {
        long long li = (long long)row * p.P + colj[j];
        if (li >= p.t_valid) li = 2LL * (p.t_valid - 1) - li;
        acc = fmaf(gv[j], lrelu(__ldg(xr + (li < 0 ? 0 : li)), p.x_slope), acc);
      }
    }
#pragma unroll
    for (int sft = 16; sft > 0; sft >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, sft);
    if (lane == 0) dst[k] = acc;
  }
}

__global__ void split_reduce_kernel(const float* __restrict__ part, float* __restrict__ out, long long n, int nsplit,
                                    int accumulate) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float a = 0.f;
    for (int s = 0; s < nsplit; ++s) a += part[(long long)s * n + i];
    out[i] = accumulate ? out[i] + a : a;
  }
}

// ------------------------------------------------------------------ elementwise chain rule
// mode 0: out = g * scale * (ref > 0 ? 1 : slope)      (LeakyReLU, mask from the input OR the output)
// mode 1: out = g * scale * (1 - ref^2)                (tanh, ref = output)
// mode 2: out = g * scale                              (plain scale / copy)
__global__ void act_backward_kernel(int mode, const float* __restrict__ g, const float* __restrict__ ref,
                                    float* __restrict__ out, long long n, float slope, float scale, int accumulate) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float v = g[i] * scale;
    if (mode == 0)
      v *= ref[i] > 0.f ? 1.f : slope;
    else if (mode == 1)
      v *= 1.f - ref[i] * ref[i];
    out[i] = accumulate ? out[i] + v : v;
  }
}

// db[c] = sum_{b, t} g[b, c, t]: a thread-block CLUSTER of 8 CTAs per channel (one CTA per channel streamed a
// (64, 128, 25600) gradient at 950 GB/s: 10 % of the Parallel WaveGAN training step).  CTA r sums slice r of the time
// axis of every batch row in double precision; rank 0 adds the 8 partials through distributed shared memory in rank
// order: deterministic, no workspace, no atomics.
constexpr int BG_CLUSTER = 8;
__device__ __forceinline__ double block_sum_256(double a, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_down_sync(0xffffffffu, a, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = a;
  __syncthreads();
  double t = 0;
  if (threadIdx.x == 0)
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
  return t;  // valid in thread 0
}
__global__ void __cluster_dims__(BG_CLUSTER, 1, 1) __launch_bounds__(256)
    bias_grad_kernel(const float* __restrict__ g, float* __restrict__ db, int B, int C, long long L, int accumulate) {
  namespace cg = cooperative_groups;
  cg::cluster_group cl = cg::this_cluster();
  __shared__ double red[8];
  __shared__ double part;
  const int c = blockIdx.x / BG_CLUSTER, r = (int)cl.block_rank();
  double a = 0;
  if (L % 4 == 0 && (reinterpret_cast<uintptr_t>(g) & 15) == 0) {
    const long long q4 = L / 4, lo = q4 * r / BG_CLUSTER, hi = q4 * (r + 1) / BG_CLUSTER;
    for (int b = 0; b < B; ++b) {
      const float4* q = reinterpret_cast<const float4*>(g + ((long long)b * C + c) * L);
      for (long long i = lo + threadIdx.x; i < hi; i += 256) {
        const float4 v = __ldg(q + i);
        a += ((double)v.x + (double)v.y) + ((double)v.z + (double)v.w);
      }
    }
  } else {
    const long long lo = L * r / BG_CLUSTER, hi = L * (r + 1) / BG_CLUSTER;
    for (int b = 0; b < B; ++b) {
      const float* q = g + ((long long)b * C + c) * L;
      for (long long i = lo + threadIdx.x; i < hi; i += 256) a += q[i];
    }
  }
  const double t = block_sum_256(a, red);
  if (threadIdx.x == 0) part = t;
  cl.sync();
  if (r == 0 && threadIdx.x == 0) {
    double tot = 0;
    for (int k = 0; k < BG_CLUSTER; ++k) tot += *cl.map_shared_rank(&part, k);
    db[c] = (accumulate ? db[c] : 0.f) + (float)tot;
  }
  cl.sync();  // the partials stay alive until rank 0 has read them
}

// short rows: one CTA per channel, fixed order
__global__ void __launch_bounds__(256) bias_grad_small_kernel(const float* __restrict__ g, float* __restrict__ db, int B, int C,
                                                               long long L, int accumulate) {
  __shared__ double red[8];
  const int c = blockIdx.x;
  double a = 0;
  for (int b = 0; b < B; ++b) {
    const float* q = g + ((long long)b * C + c) * L;
    for (long long i = threadIdx.x; i < L; i += 256) a += q[i];
  }
  const double t = block_sum_256(a, red);
  if (threadIdx.x == 0) db[c] = (accumulate ? db[c] : 0.f) + (float)t;
}

// gradient of pwgb_reduce_mean_forward: gx = gout[0] * weight / n * f'(x [, y])  (+ optional gy = -gx for L1)
__global__ void reduce_mean_backward_kernel(int mode, const float* __restrict__ x, const float* __restrict__ y, long long n,
                                            float c, float s, float weight, const float* __restrict__ gout,
                                            float* __restrict__ gx, int accumulate) {
  const float go = gout[0] * weight / (float)n;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = x[i];
    float d;
    if (mode == 0)
      d = 2.f * (v - c);
    else if (mode == 1)
      d = v > y[i] ? 1.f : (v < y[i] ? -1.f : 0.f);
    else if (mode == 2)
      d = (c - s * v) > 0.f ? -s : 0.f;
    else if (mode == 4)
      d = 2.f * (v - y[i]);
    else
      d = s;
    gx[i] = (accumulate ? gx[i] : 0.f) + go * d;
  }
}

// AvgPool1d backward: gx[r, i] = sum over windows o containing i of gy[r, o] / div(o)
__global__ void avg_pool1d_backward_kernel(const float* __restrict__ gy, float* __restrict__ gx, int rows, int t_in,
                                           int t_out, int k, int s, int pad, int include_pad) {
  const int r = blockIdx.y;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < t_in; i += gridDim.x * blockDim.x) {
    float acc = 0.f;
    // windows o with o*s - pad <= i < o*s - pad + k
    int o_hi = (i + pad) / s;
    int o_lo = (i + pad - k + s) / s;
    if (i + pad - k + 1 <= 0) o_lo = 0;
    if (o_lo < 0) o_lo = 0;
    if (o_hi > t_out - 1) o_hi = t_out - 1;
    for (int o = o_lo; o <= o_hi; ++o) {
      const int start = o * s - pad;
      if (i < start || i >= start + k) continue;
      int div;
      if (include_pad) {
        div = min(start + k, t_in + pad) - start;
      } else {
        div = min(start + k, t_in) - max(start, 0);
      }
      acc += gy[(long long)r * t_out + o] / (float)div;
    }
    gx[(long long)r * t_in + i] = acc;
  }
}

// y = a * x + b * y
__global__ void axpby_kernel(long long n, float a, const float* __restrict__ x, float b, float* __restrict__ y) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = a * x[i] + (b == 0.f ? 0.f : b * y[i]);
}

// out = a * (x_0 + x_1 + ... + x_{n-1}) accumulated in index order (the skip sum of the WaveNet stack, the MRF average of
// HiFi-GAN): every input is read once; `xs` is a device array of n pointers.
__global__ void scaled_sum_kernel(const float* const* __restrict__ xs, int n, float a, float* __restrict__ out, long long len,
                                  int vec) {
  if (vec) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < len / 4; i += (long long)gridDim.x * blockDim.x) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int k = 0; k < n; ++k) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(xs[k]) + i);
        acc.x = fmaf(a, v.x, acc.x);
        acc.y = fmaf(a, v.y, acc.y);
        acc.z = fmaf(a, v.z, acc.z);
        acc.w = fmaf(a, v.w, acc.w);
      }
      reinterpret_cast<float4*>(out)[i] = acc;
    }
  } else {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < len; i += (long long)gridDim.x * blockDim.x) {
      float acc = 0.f;
      for (int k = 0; k < n; ++k) acc = fmaf(a, xs[k][i], acc);
      out[i] = acc;
    }
  }
}

// Explicit reflect / replicate padding (torch.nn.ReflectionPad1d / ReplicationPad1d in front of the MelGAN
// convs, melgan.py:70-72, residual_stack.py:49) and its adjoint.  mode: PWGB_PAD_*.
__device__ __forceinline__ long long pad_src(long long e, long long T, int pl, int mode) {
  long long t = e - pl;
  if (mode == PWGB_PAD_REFLECT) {
    if (t < 0) t = -t;
    if (t >= T) t = 2 * (T - 1) - t;
  } else {
    t = t < 0 ? 0 : (t >= T ? T - 1 : t);
  }
  return t;
}
__global__ void pad1d_forward_kernel(const float* __restrict__ x, float* __restrict__ xp, long long rows, long long T, int pl,
                                     int pr, int mode) {
  const long long Te = T + pl + pr, n = rows * Te;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / Te, e = i % Te;
    xp[i] = x[r * T + pad_src(e, T, pl, mode)];
  }
}
// gx[r, t] = sum over extended positions e with pad_src(e) == t of gxp[r, e]   (gather form, deterministic)
__global__ void pad1d_backward_kernel(const float* __restrict__ gxp, float* __restrict__ gx, long long rows, long long T, int pl,
                                      int pr, int mode) {
  const long long Te = T + pl + pr, n = rows * T;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / T, t = i % T;
    const float* g = gxp + r * Te;
    float acc = g[pl + t];
    if (mode == PWGB_PAD_REFLECT) {
      if (t >= 1 && t <= pl) acc += g[pl - t];                  // left extension e = pl - t
      const long long m = T - 2 - t;                            // right extension e = pl + T + m
      if (m >= 0 && m < pr) acc += g[pl + T + m];
    } else {
      if (t == 0) for (int e = 0; e < pl; ++e) acc += g[e];
      if (t == T - 1) for (int m = 0; m < pr; ++m) acc += g[pl + T + m];
    }
    gx[i] = acc;
  }
}

// WaveNet gate (layers/residual_block.py:128): z[b,h,t] = tanh(g[b,h,t]) * sigmoid(g[b,H+h,t])
// (B, 2H, T) -> (B, H, T); grid.y = B * H rows, 16-byte accesses along T when the rows are 16-byte aligned
__device__ __forceinline__ float gate_exact(float a, float s) { return tanhf(a) * sigmoidf_(s); }
__global__ void gate_forward_kernel(const float* __restrict__ g, float* __restrict__ z, int B, int H, long long T) {
  const long long row = blockIdx.y;
  const long long b = row / H, h = row - b * H;
  const float* ga = g + (b * 2 * H + h) * T;
  const float* gs = ga + (long long)H * T;
  float* zr = z + row * T;
  if (T % 4 == 0 && ((reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(z)) & 15) == 0) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < T / 4; i += (long long)gridDim.x * blockDim.x) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(ga) + i), s = __ldg(reinterpret_cast<const float4*>(gs) + i);
      reinterpret_cast<float4*>(zr)[i] = make_float4(gate_exact(a.x, s.x), gate_exact(a.y, s.y), gate_exact(a.z, s.z), gate_exact(a.w, s.w));
    }
  } else {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < T; i += (long long)gridDim.x * blockDim.x)
      zr[i] = gate_exact(ga[i], gs[i]);
  }
}
__device__ __forceinline__ void gate_grad(float a, float s, float go, float& da, float& ds) {
  const float ta = tanhf(a), sg = sigmoidf_(s);
  da = go * sg * (1.f - ta * ta);
  ds = go * ta * sg * (1.f - sg);
}
__global__ void gate_backward_kernel(const float* __restrict__ g, const float* __restrict__ gz, float* __restrict__ gg, int B,
                                     int H, long long T) {
  const long long row = blockIdx.y;
  const long long b = row / H, h = row - b * H;
  const long long oa = (b * 2 * H + h) * T, os = oa + (long long)H * T;
  const float* gr = gz + row * T;
  if (T % 4 == 0 && ((reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(gz) | reinterpret_cast<uintptr_t>(gg)) & 15) == 0) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < T / 4; i += (long long)gridDim.x * blockDim.x) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(g + oa) + i), s = __ldg(reinterpret_cast<const float4*>(g + os) + i);
      const float4 go = __ldg(reinterpret_cast<const float4*>(gr) + i);
      float4 da, ds;
      gate_grad(a.x, s.x, go.x, da.x, ds.x);
      gate_grad(a.y, s.y, go.y, da.y, ds.y);
      gate_grad(a.z, s.z, go.z, da.z, ds.z);
      gate_grad(a.w, s.w, go.w, da.w, ds.w);
      reinterpret_cast<float4*>(gg + oa)[i] = da;
      reinterpret_cast<float4*>(gg + os)[i] = ds;
    }
  } else {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < T; i += (long long)gridDim.x * blockDim.x) {
      float da, ds;
      gate_grad(g[oa + i], g[os + i], gr[i], da, ds);
      gg[oa + i] = da;
      gg[os + i] = ds;
    }
  }
}

// adjoints of upsample_fir_kernel: y[r,o] = sum_k f[k] x[r, (o+k-s)/s]
__global__ void upsample_fir_backward_x_kernel(int t_in, int s, const float* __restrict__ gy, const float* __restrict__ fir,
                                               float* __restrict__ gx, int rows_per_batch, long long gybs) {
  extern __shared__ float f[];
  for (int i = threadIdx.x; i < 2 * s + 1; i += blockDim.x) f[i] = fir[i];
  __syncthreads();
  const int r = blockIdx.y;
  const int t_out = t_in * s;
  const float* gr = gy + (long long)(r / rows_per_batch) * gybs + (long long)(r % rows_per_batch) * t_out;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < t_in; i += gridDim.x * blockDim.x) {
    float acc = 0.f;
    // positions q = o + k - s with q / s == i  <=>  q in [i*s, i*s + s)
    for (int q = i * s; q < i * s + s; ++q)
      for (int k = 0; k <= 2 * s; ++k) {
        const int o = q - k + s;
        if (o >= 0 && o < t_out) acc = fmaf(f[k], gr[o], acc);
      }
    gx[(long long)r * t_in + i] = acc;
  }
}
// df[k] = sum_{r,o} gy[r,o] * x[r,(o+k-s)/s]: ONE pass over gy for all 2s+1 taps (the one-CTA-per-tap version read gy
// 2s+1 times on 2s+1 SMs: 100 ms per call, 40 % of the Parallel WaveGAN training step).  Output o = j*s + ph only meets
// the input frames j-1, j, j+1, so the kernel accumulates the 3 s sums S[w][ph] = sum gy[j*s+ph] * x[j + w - 1] (three FMAs
// per element, float within a row, double across rows) and folds them into the taps at the end:
// df[k] = sum_ph S[w(ph, k)][ph], w = 0 / 1 / 2 for ph + k - s < 0 / < s / >= s.  A cluster of 8 CTAs splits the rows;
// partials are combined through distributed shared memory in rank order (deterministic, no workspace).
constexpr int UF_CLUSTER = 8, UF_MAXS = 8, UF_MAXT = 2 * UF_MAXS + 1, UF_THREADS = 512;
template <int MAXS>
__global__ void __cluster_dims__(UF_CLUSTER, 1, 1) __launch_bounds__(UF_THREADS)
    upsample_fir_backward_f_kernel(int rows, int t_in, int s, const float* __restrict__ x, const float* __restrict__ gy,
                                   float* __restrict__ df, int rows_per_batch, long long gybs) {
  namespace cg = cooperative_groups;
  cg::cluster_group cl = cg::this_cluster();
  __shared__ double red[UF_THREADS / 32][3 * MAXS];
  __shared__ double part[3 * MAXS];
  const int r = (int)cl.block_rank();
  const int t_out = t_in * s;
  const int row_lo = (int)((long long)rows * r / UF_CLUSTER), row_hi = (int)((long long)rows * (r + 1) / UF_CLUSTER);
  double acc[3][MAXS];
#pragma unroll
  for (int w = 0; w < 3; ++w)
#pragma unroll
    for (int ph = 0; ph < MAXS; ++ph) acc[w][ph] = 0;
  for (int row = row_lo; row < row_hi; ++row) {
    const float* gr = gy + (long long)(row / rows_per_batch) * gybs + (long long)(row % rows_per_batch) * t_out;
    const float* xr = x + (long long)row * t_in;
    float f[3][MAXS];
#pragma unroll
    for (int w = 0; w < 3; ++w)
#pragma unroll
      for (int ph = 0; ph < MAXS; ++ph) f[w][ph] = 0.f;
    for (int j = threadIdx.x; j < t_in; j += UF_THREADS) {
      const float xm = j > 0 ? xr[j - 1] : 0.f, x0 = xr[j], xp = j + 1 < t_in ? xr[j + 1] : 0.f;
      const float* g = gr + (long long)j * s;
#pragma unroll
      for (int ph = 0; ph < MAXS; ++ph) {
        if (ph < s) {
          const float gv = g[ph];
          f[0][ph] = fmaf(gv, xm, f[0][ph]);
          f[1][ph] = fmaf(gv, x0, f[1][ph]);
          f[2][ph] = fmaf(gv, xp, f[2][ph]);
        }
      }
    }
#pragma unroll
    for (int w = 0; w < 3; ++w)
#pragma unroll
      for (int ph = 0; ph < MAXS; ++ph) acc[w][ph] += (double)f[w][ph];
  }
#pragma unroll
  for (int w = 0; w < 3; ++w)
#pragma unroll
    for (int ph = 0; ph < MAXS; ++ph) {
      double a = acc[w][ph];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) a += __shfl_down_sync(0xffffffffu, a, o);
      if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][w * MAXS + ph] = a;
    }
  __syncthreads();
  if (threadIdx.x < 3 * MAXS) {
    double t = 0;
    for (int w = 0; w < UF_THREADS / 32; ++w) t += red[w][threadIdx.x];
    part[threadIdx.x] = t;
  }
  cl.sync();
  if (r == 0 && threadIdx.x <= 2 * s) {
    const int k = threadIdx.x;
    double tot = 0;
    for (int ph = 0; ph < s; ++ph) {
      const int d = ph + k - s;
      const int w = d < 0 ? 0 : (d < s ? 1 : 2);
      for (int c = 0; c < UF_CLUSTER; ++c) tot += cl.map_shared_rank(part, c)[w * MAXS + ph];
    }
    df[k] = (float)tot;
  }
  cl.sync();
}
// scales beyond UF_MAXT taps: one CTA per tap, fixed order
__global__ void __launch_bounds__(256) upsample_fir_backward_f_tap_kernel(int rows, int t_in, int s, const float* __restrict__ x,
                                                                           const float* __restrict__ gy, float* __restrict__ df,
                                                                           int rows_per_batch, long long gybs) {
  __shared__ double red[256];
  const int k = blockIdx.x;
  const int t_out = t_in * s;
  double a = 0;
  for (int r = 0; r < rows; ++r) {
    const float* gr = gy + (long long)(r / rows_per_batch) * gybs + (long long)(r % rows_per_batch) * t_out;
    const float* xr = x + (long long)r * t_in;
    for (int o = threadIdx.x; o < t_out; o += 256) {
      const int q = o + k - s;
      if (q >= 0 && q < t_out) a += (double)gr[o] * xr[q / s];
    }
  }
  red[threadIdx.x] = a;
  __syncthreads();
  for (int st = 128; st > 0; st >>= 1) {
    if (threadIdx.x < st) red[threadIdx.x] += red[threadIdx.x + st];
    __syncthreads();
  }
  if (threadIdx.x == 0) df[k] = (float)red[0];
}

static int grid_for(long long n) {
  long long b = (n + 255) / 256;
  return (int)(b > 132 * 16 ? 132 * 16 : (b < 1 ? 1 : b));
}

}  // namespace pwgb

using namespace pwgb;

static int wg_fill(const pwgb_conv1d_desc* d, WgK& p) {
  if (!d || d->batch < 0 || d->cin <= 0 || d->cout <= 0 || d->groups <= 0 || d->cin % d->groups || d->cout % d->groups ||
      d->kernel <= 0 || d->stride <= 0 || d->dilation <= 0 || d->t_in <= 0 || d->t_out < 0)
    return 0;
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
  p.xcs = p.t_valid;
  p.x_slope = d->pre_slope;
  p.g_slope = 1.f;
  p.chunks_per_seq = ceil_div(p.Lout, WG_T);
  const long long items = (long long)p.B * p.chunks_per_seq;
  p.nsplit = (int)(items < 32 ? (items < 1 ? 1 : items) : 32);
  const int nrows_out = (WG_T + p.P - 2) / p.P + 1;
  const long long NR = (long long)(nrows_out - 1) * p.S + (long long)(WG_K - 1) * p.D + 1;
  p.XW = (int)(NR * p.P);
  p.ci_tiles = ceil_div(p.Cin_g, WG_CI);
  return 1;
}

static size_t ws_bytes_narrow(const pwgb_conv1d_desc* d) {
  const int P = d->period < 1 ? 1 : d->period;
  const long long blocks = (long long)d->batch * ceil_div(d->t_out * P, WGN_CHUNK);
  return (size_t)blocks * d->cout * (d->cin / d->groups) * d->kernel * sizeof(float);
}

extern "C" size_t pwgb_conv1d_wgrad_workspace(const pwgb_conv1d_desc* d) {
  WgK p;
  if (!wg_fill(d, p)) return 0;
  size_t a = (size_t)p.nsplit * d->cout * p.Cin_g * d->kernel * sizeof(float);
  const long long n = (long long)d->cout * p.Cin_g * d->kernel;
  if ((p.Cin_g <= 4 || p.Cout <= 4) && n <= 4096) {
    const size_t b = ws_bytes_narrow(d);
    if (b > a && b <= (1ull << 31)) a = b;
  }
  return a;
}

extern "C" int pwgb_conv1d_wgrad(const pwgb_conv1d_desc* d, const float* x, const float* gy, float g_slope, float* dw,
                                 int accumulate, void* ws, size_t ws_bytes, void* stream) {
  PWGB_CHECK_ARG(d && x && gy && dw && ws, "conv1d_wgrad: null argument");
  WgK p;
  PWGB_CHECK_ARG(wg_fill(d, p), "conv1d_wgrad: bad descriptor");
  PWGB_UNSUPPORTED_IF(d->pre_gate || d->shuffle > 1, "conv1d_wgrad: gate / shuffle variants are not supported");
  p.g_slope = g_slope;
  const size_t need = pwgb_conv1d_wgrad_workspace(d);
  PWGB_CHECK_ARG(ws_bytes >= need, "conv1d_wgrad: workspace too small (%zu < %zu)", ws_bytes, need);
  const long long n = (long long)d->cout * p.Cin_g * d->kernel;
  cudaStream_t st = (cudaStream_t)stream;
  if (p.B == 0 || p.Lout == 0) {
    if (!accumulate) cudaMemsetAsync(dw, 0, n * sizeof(float), st);
    return PWGB_OK;
  }
  if ((p.Cin_g <= 4 || p.Cout <= 4) && n <= 4096 && p.pad_mode == PWGB_PAD_ZERO) {
    const int chunks = ceil_div(p.Lout, WGN_CHUNK);
    const long long blocks = (long long)p.B * chunks;
    if (ws_bytes_narrow(d) <= ws_bytes && blocks <= 65535) {
      p.chunks_per_seq = chunks;
      dim3 ngrid((unsigned)ceil_div(p.Cout * p.Cin_g, 8), (unsigned)blocks);
      conv1d_wgrad_narrow_kernel<<<ngrid, 256, 0, st>>>(p, x, gy, (float*)ws);
      int rc = check_launch("conv1d_wgrad_narrow_kernel");
      if (rc) return rc;
      split_reduce_kernel<<<grid_for(n), 256, 0, st>>>((const float*)ws, dw, n, (int)blocks, accumulate);
      return check_launch("split_reduce_kernel");
    }
  }
  const size_t smem = ((size_t)WG_CO * (WG_T + 1) + (size_t)WG_CI * p.XW + WG_T) * sizeof(float);
  PWGB_UNSUPPORTED_IF(smem > 200 * 1024, "conv1d_wgrad: tile does not fit shared memory");
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(conv1d_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
      set_error("conv1d_wgrad: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      return PWGB_CUDA_ERROR;
    }
  }
  dim3 grid(p.groups * ceil_div(p.Cout_g, WG_CO) * p.ci_tiles, ceil_div(p.K, WG_K), p.nsplit);
  conv1d_wgrad_kernel<<<grid, 256, smem, st>>>(p, x, gy, (float*)ws);
  int rc = check_launch("conv1d_wgrad_kernel");
  if (rc) return rc;
  split_reduce_kernel<<<grid_for(n), 256, 0, st>>>((const float*)ws, dw, n, p.nsplit, accumulate);
  return check_launch("split_reduce_kernel");
}

extern "C" int pwgb_act_backward(int mode, const float* g, const float* ref, float* out, long long n, float slope,
                                 float scale, int accumulate, void* stream) {
  PWGB_CHECK_ARG(g && out && (ref || mode == 2) && n >= 0 && mode >= 0 && mode <= 2, "act_backward: bad arguments");
  if (n == 0) return PWGB_OK;
  act_backward_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(mode, g, ref, out, n, slope, scale, accumulate);
  return check_launch("act_backward_kernel");
}

extern "C" int pwgb_bias_grad(const float* g, float* db, int batch, int channels, long long len, int accumulate,
                              void* stream) {
  PWGB_CHECK_ARG(g && db && batch >= 0 && channels > 0 && len >= 0, "bias_grad: bad arguments");
  if ((long long)batch * len < 65536 || channels >= 592) {  // short rows / many channels: one CTA per channel fills the machine
    bias_grad_small_kernel<<<channels, 256, 0, (cudaStream_t)stream>>>(g, db, batch, channels, len, accumulate);
    return check_launch("bias_grad_small_kernel");
  }
  bias_grad_kernel<<<channels * BG_CLUSTER, 256, 0, (cudaStream_t)stream>>>(g, db, batch, channels, len, accumulate);
  return check_launch("bias_grad_kernel");
}

extern "C" int pwgb_reduce_mean_backward(int mode, const float* x, const float* y, long long n, float c, float s,
                                         float weight, const float* gout, float* gx, int accumulate, void* stream) {
  PWGB_CHECK_ARG(x && gout && gx && n > 0 && mode >= 0 && mode <= 4 && ((mode != 1 && mode != 4) || y), "reduce_mean_backward: bad arguments");
  reduce_mean_backward_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(mode, x, y, n, c, s, weight, gout, gx, accumulate);
  return check_launch("reduce_mean_backward_kernel");
}

extern "C" int pwgb_avg_pool1d_backward(const float* gy, float* gx, int rows, int t_in, int kernel, int stride,
                                        int padding, int count_include_pad, void* stream) {
  PWGB_CHECK_ARG(gy && gx && rows >= 0 && t_in > 0 && kernel > 0 && stride > 0 && padding >= 0, "avg_pool1d_backward: bad arguments");
  PWGB_UNSUPPORTED_IF(rows > 65535, "avg_pool1d_backward: too many rows");
  if (rows == 0) return PWGB_OK;
  const int t_out = (t_in + 2 * padding - kernel) / stride + 1;
  dim3 grid(ceil_div(t_in, 256) < 64 ? ceil_div(t_in, 256) : 64, rows);
  avg_pool1d_backward_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(gy, gx, rows, t_in, t_out, kernel, stride, padding, count_include_pad);
  return check_launch("avg_pool1d_backward_kernel");
}

extern "C" int pwgb_axpby(long long n, float a, const float* x, float b, float* y, void* stream) {
  PWGB_CHECK_ARG(x && y && n >= 0, "axpby: bad arguments");
  if (n == 0) return PWGB_OK;
  axpby_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(n, a, x, b, y);
  return check_launch("axpby_kernel");
}

extern "C" int pwgb_scaled_sum(const float* const* xs, int n, float a, float* out, long long len, int rows_16b_aligned,
                               void* stream) {
  PWGB_CHECK_ARG(xs && out && n > 0 && len >= 0, "scaled_sum: bad arguments");
  if (len == 0) return PWGB_OK;
  const int vec = rows_16b_aligned && len % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
  scaled_sum_kernel<<<grid_for(vec ? len / 4 : len), 256, 0, (cudaStream_t)stream>>>(xs, n, a, out, len, vec);
  return check_launch("scaled_sum_kernel");
}

extern "C" int pwgb_pad1d_forward(const float* x, float* xp, long long rows, long long t, int pad_left, int pad_right,
                                  int pad_mode, void* stream) {
  PWGB_CHECK_ARG(x && xp && rows >= 0 && t > 0 && pad_left >= 0 && pad_right >= 0, "pad1d_forward: bad arguments");
  PWGB_CHECK_ARG(pad_mode == PWGB_PAD_REFLECT || pad_mode == PWGB_PAD_REPLICATE, "pad1d_forward: pad_mode must be reflect or replicate");
  PWGB_CHECK_ARG(pad_mode != PWGB_PAD_REFLECT || (pad_left < t && pad_right < t), "pad1d_forward: reflect padding must be < t");
  const long long n = rows * (t + pad_left + pad_right);
  if (n == 0) return PWGB_OK;
  pad1d_forward_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(x, xp, rows, t, pad_left, pad_right, pad_mode);
  return check_launch("pad1d_forward_kernel");
}

extern "C" int pwgb_pad1d_backward(const float* gxp, float* gx, long long rows, long long t, int pad_left, int pad_right,
                                   int pad_mode, void* stream) {
  PWGB_CHECK_ARG(gxp && gx && rows >= 0 && t > 0 && pad_left >= 0 && pad_right >= 0, "pad1d_backward: bad arguments");
  PWGB_CHECK_ARG(pad_mode == PWGB_PAD_REFLECT || pad_mode == PWGB_PAD_REPLICATE, "pad1d_backward: pad_mode must be reflect or replicate");
  PWGB_CHECK_ARG(pad_mode != PWGB_PAD_REFLECT || (pad_left < t && pad_right < t), "pad1d_backward: reflect padding must be < t");
  const long long n = rows * t;
  if (n == 0) return PWGB_OK;
  pad1d_backward_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(gxp, gx, rows, t, pad_left, pad_right, pad_mode);
  return check_launch("pad1d_backward_kernel");
}

extern "C" int pwgb_gate_forward(const float* g, float* z, int batch, int half_channels, long long t, void* stream) {
  PWGB_CHECK_ARG(g && z && batch >= 0 && half_channels > 0 && t >= 0, "gate_forward: bad arguments");
  const long long n = (long long)batch * half_channels * t;
  if (n == 0) return PWGB_OK;
  PWGB_UNSUPPORTED_IF((long long)batch * half_channels > 65535, "gate_forward: too many rows");
  {
    const long long per_row = (t + 1023) / 1024;
    dim3 grid((unsigned)(per_row < 64 ? (per_row < 1 ? 1 : per_row) : 64), (unsigned)(batch * half_channels));
    gate_forward_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(g, z, batch, half_channels, t);
  }
  return check_launch("gate_forward_kernel");
}

extern "C" int pwgb_gate_backward(const float* g, const float* gz, float* gg, int batch, int half_channels, long long t,
                                  void* stream) {
  PWGB_CHECK_ARG(g && gz && gg && batch >= 0 && half_channels > 0 && t >= 0, "gate_backward: bad arguments");
  const long long n = (long long)batch * half_channels * t;
  if (n == 0) return PWGB_OK;
  PWGB_UNSUPPORTED_IF((long long)batch * half_channels > 65535, "gate_backward: too many rows");
  {
    const long long per_row = (t + 1023) / 1024;
    dim3 grid((unsigned)(per_row < 64 ? (per_row < 1 ? 1 : per_row) : 64), (unsigned)(batch * half_channels));
    gate_backward_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(g, gz, gg, batch, half_channels, t);
  }
  return check_launch("gate_backward_kernel");
}

extern "C" int pwgb_upsample_fir_backward(int rows, int rows_per_batch, int t_in, int scale, const float* x, const float* fir,
                                          const float* gy, long long gy_batch_stride, float* gx, float* dfir, void* stream) {
  PWGB_CHECK_ARG(fir && gy && (gx || (dfir && x)), "upsample_fir_backward: null argument");
  PWGB_CHECK_ARG(rows >= 0 && rows_per_batch > 0 && t_in > 0 && scale > 0 && rows % rows_per_batch == 0, "upsample_fir_backward: bad sizes");
  PWGB_UNSUPPORTED_IF(rows > 65535, "upsample_fir_backward: too many rows");
  if (rows == 0) return PWGB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const long long gybs = gy_batch_stride ? gy_batch_stride : (long long)rows_per_batch * t_in * scale;
  if (gx) {
    dim3 grid(ceil_div(t_in, 256) < 64 ? ceil_div(t_in, 256) : 64, rows);
    upsample_fir_backward_x_kernel<<<grid, 256, (2 * scale + 1) * sizeof(float), st>>>(t_in, scale, gy, fir, gx, rows_per_batch, gybs);
    int rc = check_launch("upsample_fir_backward_x_kernel");
    if (rc) return rc;
  }
  if (dfir) {
    if (2 * scale + 1 <= UF_MAXT) {
      if (scale <= 4)
        upsample_fir_backward_f_kernel<4><<<UF_CLUSTER, UF_THREADS, 0, st>>>(rows, t_in, scale, x, gy, dfir, rows_per_batch, gybs);
      else
        upsample_fir_backward_f_kernel<UF_MAXS><<<UF_CLUSTER, UF_THREADS, 0, st>>>(rows, t_in, scale, x, gy, dfir, rows_per_batch, gybs);
      return check_launch("upsample_fir_backward_f_kernel");
    }
    upsample_fir_backward_f_tap_kernel<<<2 * scale + 1, 256, 0, st>>>(rows, t_in, scale, x, gy, dfir, rows_per_batch, gybs);
    return check_launch("upsample_fir_backward_f_tap_kernel");
  }
  return PWGB_OK;
}
