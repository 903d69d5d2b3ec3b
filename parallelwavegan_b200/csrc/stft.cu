// Fused STFT-magnitude kernels for MultiResolutionSTFTLoss (losses/stft_loss.py:16-170) and
// MelSpectrogramLoss (losses/mel_loss.py:81-165).
//
// One CTA = one frame of BOTH signals: z = w*(x + i*y) goes through ONE complex radix-2 FFT in
// shared memory and X, Y are separated by Hermitian symmetry, so the framed / windowed / complex
// STFT tensors of the reference (torch.stft -> real/imag -> mag -> log, ~720 MB of traffic for 13 MB
// of input at C3) are never materialised: the loss variant reduces straight to three partial
// sums per frame.  Reductions are deterministic (fixed-order two-stage, no atomics).
#include "common.cuh"

namespace pwgb {

struct StftK {
  int B, T, n, log2n, hop, win, frames, bins;
  float eps;
};

__device__ __forceinline__ unsigned bitrev(unsigned v, int bits) { return __brev(v) >> (32 - bits); }

// mode 0: loss partials (sum (ym-xm)^2, sum ym^2, sum |log ym - log xm|) -> part[(b*frames+f)*3]
// mode 1: write amplitudes sqrt(max(|.|^2, eps)) to ax / ay (B, frames, bins) (ay may be null)
template <int MODE>
__global__ void __launch_bounds__(256) stft_pair_kernel(const StftK p, const float* __restrict__ x,
                                                         const float* __restrict__ y,
                                                         const float* __restrict__ window,
                                                         float* __restrict__ out0, float* __restrict__ out1) {
  extern __shared__ float2 sm[];
  float2* z = sm;            // n
  float2* tw = sm + p.n;     // n/2
  __shared__ float red[3][8];
  const int f = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int n = p.n, half_n = n >> 1;
  const int left = (n - p.win) >> 1;
  const float* xb = x + (long long)b * p.T;
  const float* yb = y ? y + (long long)b * p.T : nullptr;
  for (int j = tid; j < half_n; j += 256) {
    float s, c;
    sincospif(-2.0f * (float)j / (float)n, &s, &c);
    tw[j] = make_float2(c, s);
  }
  for (int j = tid; j < n; j += 256) {
    float w = 0.f;
    if (j >= left && j < left + p.win) w = __ldg(window + j - left);
    long long src = (long long)f * p.hop + j - half_n;  // center=True, reflect padding of n/2
    if (src < 0) src = -src;
    if (src >= p.T) src = 2LL * (p.T - 1) - src;
    src = src < 0 ? 0 : (src >= p.T ? p.T - 1 : src);
    const float xv = __ldg(xb + src) * w;
    const float yv = yb ? __ldg(yb + src) * w : 0.f;
    z[bitrev((unsigned)j, p.log2n)] = make_float2(xv, yv);
  }
  __syncthreads();
  for (int s = 1; s <= p.log2n; ++s) {
    const int half = 1 << (s - 1);
    const int tstep = n >> s;
    for (int t = tid; t < half_n; t += 256) {
      const int pos = t & (half - 1);
      const int i0 = ((t >> (s - 1)) << s) + pos;
      const int i1 = i0 + half;
      const float2 w = tw[pos * tstep];
      const float2 a = z[i0], bb = z[i1];
      const float2 m = make_float2(bb.x * w.x - bb.y * w.y, bb.x * w.y + bb.y * w.x);
      z[i0] = make_float2(a.x + m.x, a.y + m.y);
      z[i1] = make_float2(a.x - m.x, a.y - m.y);
    }
    __syncthreads();
  }
  float sd = 0.f, sy = 0.f, sl = 0.f;
  for (int k = tid; k < p.bins; k += 256) {
    const float2 a = z[k];
    const float2 c = z[(n - k) & (n - 1)];
    const float xr = a.x + c.x, xi = a.y - c.y;  // 2 X[k]
    const float yr = a.y + c.y, yi = c.x - a.x;  // 2 Y[k]
    const float px = 0.25f * (xr * xr + xi * xi);
    const float py = 0.25f * (yr * yr + yi * yi);
    const float xm = sqrtf(fmaxf(px, p.eps));
    const float ym = sqrtf(fmaxf(py, p.eps));
    if (MODE == 0) {
      const float d = ym - xm;
      sd = fmaf(d, d, sd);
      sy = fmaf(ym, ym, sy);
      sl += fabsf(logf(ym) - logf(xm));
    } else {
      const long long o = ((long long)b * p.frames + f) * p.bins + k;
      out0[o] = xm;
      if (out1) out1[o] = ym;
    }
  }
  if (MODE == 0) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sd += __shfl_xor_sync(0xffffffffu, sd, o);
      sy += __shfl_xor_sync(0xffffffffu, sy, o);
      sl += __shfl_xor_sync(0xffffffffu, sl, o);
    }
    if ((tid & 31) == 0) {
      red[0][tid >> 5] = sd;
      red[1][tid >> 5] = sy;
      red[2][tid >> 5] = sl;
    }
    __syncthreads();
    if (tid < 3) {
      float v = 0.f;
      for (int i = 0; i < 8; ++i) v += red[tid][i];
      out0[((long long)b * p.frames + f) * 3 + tid] = v;
    }
  }
}

// Final deterministic reduction: one CTA per resolution sums its partials in double, the last
// step averages over resolutions.  out[0] = sc, out[1] = mag (stft_loss.py:157-170).
struct FinalArgs {
  int counts[8];
  long long offsets[8];
  long long nelem[8];
};
__global__ void stft_loss_final_kernel(const float* __restrict__ part, const FinalArgs fa, int n_res,
                                       float* __restrict__ out) {
  const int* counts = fa.counts;
  const long long* offsets = fa.offsets;
  const long long* nelem = fa.nelem;
  __shared__ double red[3][256];
  __shared__ double res_sc[8], res_mag[8];
  const int tid = threadIdx.x;
  for (int r = 0; r < n_res; ++r) {
    double a = 0, b = 0, c = 0;
    const float* pr = part + offsets[r];
    for (int i = tid; i < counts[r]; i += 256) {
      a += pr[3 * (long long)i];
      b += pr[3 * (long long)i + 1];
      c += pr[3 * (long long)i + 2];
    }
    red[0][tid] = a;
    red[1][tid] = b;
    red[2][tid] = c;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
      if (tid < s) {
        red[0][tid] += red[0][tid + s];
        red[1][tid] += red[1][tid + s];
        red[2][tid] += red[2][tid + s];
      }
      __syncthreads();
    }
    if (tid == 0) {
      res_sc[r] = sqrt(red[0][0]) / sqrt(red[1][0]);
      res_mag[r] = red[2][0] / (double)nelem[r];
    }
    __syncthreads();
  }
  if (tid == 0) {
    double sc = 0, mag = 0;
    for (int r = 0; r < n_res; ++r) {
      sc += res_sc[r];
      mag += res_mag[r];
    }
    out[0] = (float)(sc / n_res);
    out[1] = (float)(mag / n_res);
  }
}

// mel_l1: sum over (b, frame, mel) of | log_b(max(ax . M, eps)) - log_b(max(ay . M, eps)) |
// also (optionally) writes the log-mel of x: (B, n_mels, frames)  (mel_loss.py:107-110)
__global__ void __launch_bounds__(128) mel_project_kernel(int B, int frames, int bins, int n_mels,
                                                           const float* __restrict__ ax, const float* __restrict__ ay,
                                                           const float* __restrict__ melmat, float eps, float log_scale,
                                                           float* __restrict__ mel_x, float* __restrict__ part) {
  extern __shared__ float sa[];  // 2 * bins
  __shared__ float red[4];
  const int f = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const long long row = ((long long)b * frames + f) * bins;
  for (int k = tid; k < bins; k += 128) {
    sa[k] = ax[row + k];
    sa[bins + k] = ay ? ay[row + k] : 0.f;
  }
  __syncthreads();
  float acc = 0.f;
  for (int m = tid; m < n_mels; m += 128) {
    float sx = 0.f, sy = 0.f;
    for (int k = 0; k < bins; ++k) {
      const float w = __ldg(melmat + (long long)k * n_mels + m);
      sx = fmaf(sa[k], w, sx);
      sy = fmaf(sa[bins + k], w, sy);
    }
    const float lx = logf(fmaxf(sx, eps)) * log_scale;
    if (mel_x) mel_x[((long long)b * n_mels + m) * frames + f] = lx;
    if (ay) acc += fabsf(lx - logf(fmaxf(sy, eps)) * log_scale);
  }
  if (part) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((tid & 31) == 0) red[tid >> 5] = acc;
    __syncthreads();
    if (tid == 0) part[(long long)b * frames + f] = red[0] + red[1] + red[2] + red[3];
  }
}

__global__ void sum_scale_kernel(const float* __restrict__ part, long long n, double scale, float* __restrict__ out) {
  __shared__ double red[256];
  double a = 0;
  for (long long i = threadIdx.x; i < n; i += 256) a += part[i];
  red[threadIdx.x] = a;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = (float)(red[0] * scale);
}

// ---------------------------------------------------------------- backward
// dx += adjoint of (x -> amp): per frame, recompute X = FFT(w * frame), form
// G[k] = damp[k] * X[k] / amp[k]  (0 where the clamp was active), zero-extend to n bins, inverse
// transform (same butterflies, conjugate twiddles), dframe[j] = Re(z[j]), scatter w[j]*dframe[j]
// back through the reflect-padded framing with atomics (frames overlap).
__global__ void __launch_bounds__(256) stft_amp_backward_kernel(const StftK p, const float* __restrict__ x,
                                                                 const float* __restrict__ window,
                                                                 const float* __restrict__ amp,
                                                                 const float* __restrict__ damp,
                                                                 float* __restrict__ dx) {
  extern __shared__ float2 sm[];
  float2* z = sm;               // n
  float2* g2 = sm + p.n;        // n
  float2* tw = sm + 2 * p.n;    // n/2
  const int f = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int n = p.n, half_n = n >> 1;
  const int left = (n - p.win) >> 1;
  const float* xb = x + (long long)b * p.T;
  auto src_of = [&](int j) -> long long {
    long long src = (long long)f * p.hop + j - half_n;
    if (src < 0) src = -src;
    if (src >= p.T) src = 2LL * (p.T - 1) - src;
    return src < 0 ? 0 : (src >= p.T ? p.T - 1 : src);
  };
  for (int j = tid; j < half_n; j += 256) {
    float s, c;
    sincospif(-2.0f * (float)j / (float)n, &s, &c);
    tw[j] = make_float2(c, s);
  }
  for (int j = tid; j < n; j += 256) {
    float w = 0.f;
    if (j >= left && j < left + p.win) w = __ldg(window + j - left);
    z[bitrev((unsigned)j, p.log2n)] = make_float2(__ldg(xb + src_of(j)) * w, 0.f);
  }
  __syncthreads();
  for (int s = 1; s <= p.log2n; ++s) {
    const int half = 1 << (s - 1);
    const int tstep = n >> s;
    for (int t = tid; t < half_n; t += 256) {
      const int pos = t & (half - 1);
      const int i0 = ((t >> (s - 1)) << s) + pos;
      const int i1 = i0 + half;
      const float2 w = tw[pos * tstep];
      const float2 a = z[i0], bb = z[i1];
      const float2 m = make_float2(bb.x * w.x - bb.y * w.y, bb.x * w.y + bb.y * w.x);
      z[i0] = make_float2(a.x + m.x, a.y + m.y);
      z[i1] = make_float2(a.x - m.x, a.y - m.y);
    }
    __syncthreads();
  }
  const long long row = ((long long)b * p.frames + f) * p.bins;
  for (int k = tid; k < n; k += 256) {
    float2 gk = make_float2(0.f, 0.f);
    if (k < p.bins) {
      const float2 X = z[k];
      const float pw = X.x * X.x + X.y * X.y;
      if (pw > p.eps) {
        const float sc = __ldg(damp + row + k) / __ldg(amp + row + k);
        gk = make_float2(sc * X.x, sc * X.y);
      }
    }
    g2[bitrev((unsigned)k, p.log2n)] = gk;
  }
  __syncthreads();
  for (int s = 1; s <= p.log2n; ++s) {
    const int half = 1 << (s - 1);
    const int tstep = n >> s;
    for (int t = tid; t < half_n; t += 256) {
      const int pos = t & (half - 1);
      const int i0 = ((t >> (s - 1)) << s) + pos;
      const int i1 = i0 + half;
      const float2 w = make_float2(tw[pos * tstep].x, -tw[pos * tstep].y);  // conjugate: e^{+i theta}
      const float2 a = g2[i0], bb = g2[i1];
      const float2 m = make_float2(bb.x * w.x - bb.y * w.y, bb.x * w.y + bb.y * w.x);
      g2[i0] = make_float2(a.x + m.x, a.y + m.y);
      g2[i1] = make_float2(a.x - m.x, a.y - m.y);
    }
    __syncthreads();
  }
  float* dxb = dx + (long long)b * p.T;
  for (int j = tid; j < n; j += 256) {
    if (j < left || j >= left + p.win) continue;
    const float v = g2[j].x * __ldg(window + j - left);
    if (v != 0.f) atomicAdd(dxb + src_of(j), v);
  }
}

// dax[b,f,k] = sum_m melmat[k,m] * dmel[m],  dmel[m] = gout * scale * sign(lx-ly) * log_scale / mx * [mx > eps]
__global__ void __launch_bounds__(128) mel_project_backward_kernel(int B, int frames, int bins, int n_mels,
                                                                    const float* __restrict__ ax,
                                                                    const float* __restrict__ ay,
                                                                    const float* __restrict__ melmat, float eps,
                                                                    float log_scale, const float* __restrict__ gout,
                                                                    float scale, float* __restrict__ dax) {
  extern __shared__ float sa[];  // 2*bins amps + n_mels dmel
  float* dm = sa + 2 * bins;
  const int f = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const long long row = ((long long)b * frames + f) * bins;
  for (int k = tid; k < bins; k += 128) {
    sa[k] = ax[row + k];
    sa[bins + k] = ay[row + k];
  }
  __syncthreads();
  const float go = gout[0] * scale;
  for (int m = tid; m < n_mels; m += 128) {
    float sx = 0.f, sy = 0.f;
    for (int k = 0; k < bins; ++k) {
      const float w = __ldg(melmat + (long long)k * n_mels + m);
      sx = fmaf(sa[k], w, sx);
      sy = fmaf(sa[bins + k], w, sy);
    }
    const float lx = logf(fmaxf(sx, eps)), ly = logf(fmaxf(sy, eps));
    float d = lx > ly ? 1.f : (lx < ly ? -1.f : 0.f);
    dm[m] = sx > eps ? go * d * log_scale / sx : 0.f;
  }
  __syncthreads();
  for (int k = tid; k < bins; k += 128) {
    float a = 0.f;
    for (int m = 0; m < n_mels; ++m) a = fmaf(__ldg(melmat + (long long)k * n_mels + m), dm[m], a);
    dax[row + k] = a;
  }
}

// training form of the STFT loss on materialised magnitudes: three double sums, then d loss / d xm
__global__ void __launch_bounds__(256) stft_loss_terms_kernel(const float* __restrict__ xm, const float* __restrict__ ym,
                                                               long long n, double* __restrict__ sums) {
  __shared__ double red[3][256];
  double a = 0, b = 0, c = 0;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const float x = xm[i], y = ym[i];
    const float d = y - x;
    a += (double)d * d;
    b += (double)y * y;
    c += fabsf(logf(y) - logf(x));
  }
  red[0][threadIdx.x] = a;
  red[1][threadIdx.x] = b;
  red[2][threadIdx.x] = c;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s)
      for (int q = 0; q < 3; ++q) red[q][threadIdx.x] += red[q][threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x < 3) sums[blockIdx.x * 3 + threadIdx.x] = red[threadIdx.x][0];
}
__global__ void stft_loss_finish_kernel(const double* __restrict__ part, int nblocks, long long n, double* __restrict__ sums3,
                                        float* __restrict__ out2, float weight, int accumulate) {
  if (threadIdx.x == 0) {
    double a = 0, b = 0, c = 0;
    for (int i = 0; i < nblocks; ++i) {
      a += part[3 * i];
      b += part[3 * i + 1];
      c += part[3 * i + 2];
    }
    sums3[0] = a;
    sums3[1] = b;
    sums3[2] = c;
    const float sc = (float)(sqrt(a) / sqrt(b)) * weight, mg = (float)(c / (double)n) * weight;
    out2[0] = (accumulate ? out2[0] : 0.f) + sc;
    out2[1] = (accumulate ? out2[1] : 0.f) + mg;
  }
}
// dxm = g_sc * w * d sc/d xm + g_mag * w * d mag/d xm,  sc = sqrt(S1)/sqrt(S2), mag = S3 / n
__global__ void stft_loss_dmag_kernel(const float* __restrict__ xm, const float* __restrict__ ym, long long n,
                                      const double* __restrict__ sums3, const float* __restrict__ gout2, float weight,
                                      float* __restrict__ dxm) {
  const double s1 = sums3[0], s2 = sums3[1];
  const float ksc = s1 > 0 ? (float)(gout2[0] * weight / (sqrt(s1) * sqrt(s2))) : 0.f;
  const float kmg = gout2[1] * weight / (float)n;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const float x = xm[i], y = ym[i];
    const float dl = logf(y) - logf(x);
    const float sg = dl > 0.f ? 1.f : (dl < 0.f ? -1.f : 0.f);
    dxm[i] = -ksc * (y - x) - kmg * sg / x;
  }
}

// The FFT kernels reach the 48 KB shared-memory limit at n_fft = 4096 (stft_pair_kernel<0>: 48 KB dynamic + 96 B
// static), so they opt in through allow_dynamic_smem (common.cuh) whenever their total would pass it.

static int fill(const pwgb_stft_desc* d, StftK& p) {
  if (!d || d->batch < 0 || d->t <= 0 || d->n_fft < 16 || d->n_fft > 4096 || (d->n_fft & (d->n_fft - 1)) ||
      d->hop <= 0 || d->win_length <= 0 || d->win_length > d->n_fft || d->t <= d->n_fft / 2)
    return 0;
  p.B = d->batch;
  p.T = d->t;
  p.n = d->n_fft;
  p.log2n = 0;
  while ((1 << p.log2n) < p.n) ++p.log2n;
  p.hop = d->hop;
  p.win = d->win_length;
  p.frames = 1 + d->t / d->hop;
  p.bins = d->n_fft / 2 + 1;
  p.eps = d->clamp_eps;
  return 1;
}

}  // namespace pwgb

using namespace pwgb;

extern "C" size_t pwgb_mr_stft_loss_workspace(const pwgb_stft_desc* descs, int n_res) {
  if (!descs || n_res <= 0 || n_res > 8) return 0;
  size_t fl = 0;
  for (int r = 0; r < n_res; ++r) {
    StftK p;
    if (!fill(&descs[r], p)) return 0;
    fl += (size_t)p.B * p.frames * 3;
  }
  return fl * sizeof(float);
}

extern "C" int pwgb_mr_stft_loss_forward(const pwgb_stft_desc* descs, int n_res, const float* x, const float* y,
                                         const float* const* windows, float* out2, void* ws, size_t ws_bytes,
                                         void* stream) {
  PWGB_CHECK_ARG(descs && x && y && windows && out2 && ws, "mr_stft_loss: null argument");
  PWGB_CHECK_ARG(n_res > 0 && n_res <= 8, "mr_stft_loss: 1..8 resolutions");
  const size_t need = pwgb_mr_stft_loss_workspace(descs, n_res);
  PWGB_CHECK_ARG(need && ws_bytes >= need, "mr_stft_loss: bad descriptor or workspace too small (%zu < %zu)", ws_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  FinalArgs fa;
  int* counts = fa.counts;
  long long* offsets = fa.offsets;
  long long* nelem = fa.nelem;
  size_t off = 0;
  float* part = (float*)ws;
  for (int r = 0; r < n_res; ++r) {
    StftK p;
    fill(&descs[r], p);
    counts[r] = p.B * p.frames;
    offsets[r] = (long long)off;
    nelem[r] = (long long)p.B * p.frames * p.bins;
    const size_t smem = (size_t)(p.n + p.n / 2) * sizeof(float2);
    if (p.B > 0) {
      int rc = allow_dynamic_smem(stft_pair_kernel<0>, smem, "stft_pair_kernel");
      if (rc) return rc;
      stft_pair_kernel<0><<<dim3(p.frames, p.B), 256, smem, st>>>(p, x, y, windows[r], part + off, nullptr);
      rc = check_launch("stft_pair_kernel");
      if (rc) return rc;
    }
    off += (size_t)counts[r] * 3;
  }
  stft_loss_final_kernel<<<1, 256, 0, st>>>(part, fa, n_res, out2);
  return check_launch("stft_loss_final_kernel");
}

extern "C" int pwgb_stft_amplitude_forward(const pwgb_stft_desc* d, const float* x, const float* y, const float* window,
                                           float* amp_x, float* amp_y, void* stream) {
  PWGB_CHECK_ARG(d && x && window && amp_x && (!y == !amp_y), "stft_amplitude: null / inconsistent arguments");
  StftK p;
  PWGB_CHECK_ARG(fill(d, p), "stft_amplitude: bad descriptor (n_fft must be a power of two <= 4096, t > n_fft/2)");
  if (p.B == 0) return PWGB_OK;
  const size_t smem = (size_t)(p.n + p.n / 2) * sizeof(float2);
  const int rc = allow_dynamic_smem(stft_pair_kernel<1>, smem, "stft_pair_kernel");
  if (rc) return rc;
  stft_pair_kernel<1><<<dim3(p.frames, p.B), 256, smem, (cudaStream_t)stream>>>(p, x, y, window, amp_x, amp_y);
  return check_launch("stft_pair_kernel");
}

extern "C" int pwgb_mel_project_forward(int batch, int frames, int bins, int n_mels, const float* amp_x,
                                        const float* amp_y, const float* melmat, float eps, float log_scale,
                                        float* mel_x, float* loss, float* ws, void* stream) {
  PWGB_CHECK_ARG(amp_x && melmat && (mel_x || (amp_y && loss && ws)), "mel_project: null argument");
  PWGB_CHECK_ARG(batch >= 0 && frames > 0 && bins > 0 && n_mels > 0 && batch <= 65535, "mel_project: bad sizes");
  if (batch == 0) return PWGB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const bool want_loss = amp_y && loss && ws;
  mel_project_kernel<<<dim3(frames, batch), 128, 2 * (size_t)bins * sizeof(float), st>>>(
      batch, frames, bins, n_mels, amp_x, amp_y, melmat, eps, log_scale, mel_x, want_loss ? ws : nullptr);
  int rc = check_launch("mel_project_kernel");
  if (rc || !want_loss) return rc;
  const long long n = (long long)batch * frames;
  sum_scale_kernel<<<1, 256, 0, st>>>(ws, n, 1.0 / ((double)n * n_mels), loss);
  return check_launch("sum_scale_kernel");
}

extern "C" int pwgb_stft_amplitude_backward(const pwgb_stft_desc* d, const float* x, const float* window, const float* amp,
                                            const float* damp, float* dx, void* stream) {
  PWGB_CHECK_ARG(d && x && window && amp && damp && dx, "stft_amplitude_backward: null argument");
  StftK p;
  PWGB_CHECK_ARG(fill(d, p), "stft_amplitude_backward: bad descriptor");
  if (p.B == 0) return PWGB_OK;
  const size_t smem = (size_t)(2 * p.n + p.n / 2) * sizeof(float2);
  const int rc = allow_dynamic_smem(stft_amp_backward_kernel, smem, "stft_amplitude_backward");
  if (rc) return rc;
  stft_amp_backward_kernel<<<dim3(p.frames, p.B), 256, smem, (cudaStream_t)stream>>>(p, x, window, amp, damp, dx);
  return check_launch("stft_amp_backward_kernel");
}

extern "C" int pwgb_mel_project_backward(int batch, int frames, int bins, int n_mels, const float* amp_x,
                                         const float* amp_y, const float* melmat, float eps, float log_scale,
                                         const float* gout, float* damp_x, void* stream) {
  PWGB_CHECK_ARG(amp_x && amp_y && melmat && gout && damp_x, "mel_project_backward: null argument");
  PWGB_CHECK_ARG(batch >= 0 && frames > 0 && bins > 0 && n_mels > 0 && batch <= 65535, "mel_project_backward: bad sizes");
  if (batch == 0) return PWGB_OK;
  const float scale = 1.0f / ((float)batch * (float)frames * (float)n_mels);
  mel_project_backward_kernel<<<dim3(frames, batch), 128, (2 * (size_t)bins + n_mels) * sizeof(float), (cudaStream_t)stream>>>(
      batch, frames, bins, n_mels, amp_x, amp_y, melmat, eps, log_scale, gout, scale, damp_x);
  return check_launch("mel_project_backward_kernel");
}

extern "C" int pwgb_stft_loss_terms(const float* xm, const float* ym, long long n, float weight, int accumulate, float* out2,
                                    double* sums3, double* ws, int ws_doubles, void* stream) {
  PWGB_CHECK_ARG(xm && ym && out2 && sums3 && ws && n > 0 && ws_doubles >= 3, "stft_loss_terms: bad arguments");
  int blocks = (int)((n + 4095) / 4096);
  if (blocks > ws_doubles / 3) blocks = ws_doubles / 3;
  if (blocks > 1024) blocks = 1024;
  cudaStream_t st = (cudaStream_t)stream;
  stft_loss_terms_kernel<<<blocks, 256, 0, st>>>(xm, ym, n, ws);
  int rc = check_launch("stft_loss_terms_kernel");
  if (rc) return rc;
  stft_loss_finish_kernel<<<1, 32, 0, st>>>(ws, blocks, n, sums3, out2, weight, accumulate);
  return check_launch("stft_loss_finish_kernel");
}

extern "C" int pwgb_stft_loss_dmag(const float* xm, const float* ym, long long n, const double* sums3, const float* gout2,
                                   float weight, float* dxm, void* stream) {
  PWGB_CHECK_ARG(xm && ym && sums3 && gout2 && dxm && n > 0, "stft_loss_dmag: bad arguments");
  int blocks = (int)((n + 2047) / 2048);
  if (blocks > 2368) blocks = 2368;
  stft_loss_dmag_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(xm, ym, n, sums3, gout2, weight, dxm);
  return check_launch("stft_loss_dmag_kernel");
}
