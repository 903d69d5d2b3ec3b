// VQ-VAE bottleneck (models/vqvae.py, layers/vector_quantize_codebook.py, functions/vector_quantizer.py): the
// nearest-code search with its gather and the decoder-input assembly in one launch, and the adjoint of the assembly.
// fp32 throughout, every sum in a fixed order, no float atomics: results are identical from run to run.
#include "common.cuh"

namespace pwgb {

constexpr int VQ_TT = 32;   // frames (rows of the search) per CTA: one per lane
constexpr int VQ_KC = 32;   // codes per staged codebook chunk
constexpr int VQ_RT = 4;    // codes per thread per chunk: 8 warps x 4 = VQ_KC
constexpr int VQ_MAX_D = 768;  // two (D x 32) fp32 tiles in shared memory: 192 KiB

struct VqArgs {
  const float* z_e;       // (B, D, T) or null (decode: indices given)
  const float* cb;        // (K, D)
  long long* idx;         // (B, T) int64: written by the search, read when z_e is null
  float* z_q;             // (B, D, T) or null
  float* dec;             // (B, D + Cl + Cg, T) or null
  const float* l;         // (B, Cl, T) or null
  const float* gtab;      // (num_g, Cg) or null
  const long long* g;     // (B,) or null
  int B, D, T, K, Cl, Cg, num_g;
  // the stream launch (pwgb_vq_stream_forward): l row t is row t of [l_hist (B, Cl, l_delay) | l], and frame t of item
  // b is signal frame mframe[b] - mlook + t, stored as +0.0 (index -1) outside [0, mend[b])
  const float* l_hist;
  int l_delay;
  const int* mframe;
  const int* mend;
  int mlook;
};

// torch.min(dim) order: a NaN distance beats every number and the first NaN wins; otherwise the smaller distance,
// ties to the lower index.  A total order, so the merge order of the candidates does not change the result.
__device__ __forceinline__ bool vq_better(float d, int k, float bd, int bk) {
  const bool n = d != d, bn = bd != bd;
  if (n || bn) return n && (!bn || k < bk);
  return d < bd || (d == bd && k < bk);
}

// the swizzled (d, code) slot of the staged chunk: groups of 4 codes stay contiguous (one 16-byte load per group), the
// group is XORed with d % 8 so that a warp storing 32 consecutive d of one code hits 8 banks instead of 1
__device__ __forceinline__ int vq_slot(int d, int kk) { return d * VQ_KC + ((((kk >> 2) ^ (d & 7))) << 2) + (kk & 3); }

constexpr int VQ_MASKED = -3;  // row[] of a stream frame outside its signal

// grid (ceil(T / 32), B), 256 threads.  Dynamic shared memory: xs (D x 32) when searching + cs (D x 32).  STREAM: the
// delayed l and the mask of VqArgs (search and assembly otherwise the same code).
template <bool STREAM>
__device__ __forceinline__ void vq_forward_body(const VqArgs& a) {
  extern __shared__ __align__(16) float vq_smem[];
  __shared__ float bd_sh[8][VQ_TT];
  __shared__ int bk_sh[8][VQ_TT];
  __shared__ int row[VQ_TT];  // code of each frame; -1: index outside the codebook (NaN column)
  const int b = blockIdx.y, t0 = blockIdx.x * VQ_TT, tid = threadIdx.x, lane = tid & 31, q = tid >> 5;
  const int D = a.D, T = a.T;
  if (a.z_e) {
    float* xs = vq_smem;
    float* cs = vq_smem + (size_t)D * VQ_TT;
    const float* zb = a.z_e + (long long)b * D * T;
    for (int i = tid; i < D * VQ_TT; i += 256) {  // coalesced along time
      const int d = i / VQ_TT, tt = i % VQ_TT;
      xs[i] = t0 + tt < T ? zb[(long long)d * T + t0 + tt] : 0.f;
    }
    __syncthreads();
    float xsq = 0.f;
    for (int d = 0; d < D; ++d) xsq = fmaf(xs[d * VQ_TT + lane], xs[d * VQ_TT + lane], xsq);
    float best_d = __int_as_float(0x7f800000);  // +inf: any number ties or wins, so the first code always enters
    int best_k = 0x7fffffff;
    for (int k0 = 0; k0 < a.K; k0 += VQ_KC) {
      __syncthreads();  // the previous chunk is consumed
      for (int i = tid; i < VQ_KC * D; i += 256) {  // coalesced along d
        const int kk = i / D, d = i % D, k = k0 + kk;
        cs[vq_slot(d, kk)] = k < a.K ? __ldg(a.cb + (long long)k * D + d) : 0.f;
      }
      __syncthreads();
      float dot[VQ_RT], csq[VQ_RT];
#pragma unroll
      for (int j = 0; j < VQ_RT; ++j) dot[j] = csq[j] = 0.f;
#pragma unroll 4
      for (int d = 0; d < D; ++d) {
        const float x = xs[d * VQ_TT + lane];
        const float4 c = *reinterpret_cast<const float4*>(cs + d * VQ_KC + ((q ^ (d & 7)) << 2));
        dot[0] = fmaf(x, c.x, dot[0]);
        dot[1] = fmaf(x, c.y, dot[1]);
        dot[2] = fmaf(x, c.z, dot[2]);
        dot[3] = fmaf(x, c.w, dot[3]);
        csq[0] = fmaf(c.x, c.x, csq[0]);
        csq[1] = fmaf(c.y, c.y, csq[1]);
        csq[2] = fmaf(c.z, c.z, csq[2]);
        csq[3] = fmaf(c.w, c.w, csq[3]);
      }
#pragma unroll
      for (int j = 0; j < VQ_RT; ++j) {
        const int k = k0 + q * VQ_RT + j;
        // addmm(c_sqr + x_sqr, x, c^T, beta=1, alpha=-2): 2 * dot is exact, so this is one rounding of the difference
        const float dist = fmaf(-2.f, dot[j], csq[j] + xsq);
        if (k < a.K && vq_better(dist, k, best_d, best_k)) {
          best_d = dist;
          best_k = k;
        }
      }
    }
    bd_sh[q][lane] = best_d;
    bk_sh[q][lane] = best_k;
    __syncthreads();
    if (q == 0) {
      for (int w = 1; w < 8; ++w)
        if (vq_better(bd_sh[w][lane], bk_sh[w][lane], best_d, best_k)) {
          best_d = bd_sh[w][lane];
          best_k = bk_sh[w][lane];
        }
      const bool masked = STREAM && stream_outside(a.mframe, a.mend, 1, a.mlook, b, t0 + lane);
      row[lane] = masked ? VQ_MASKED : best_k;
      if (t0 + lane < T) a.idx[(long long)b * T + t0 + lane] = masked ? -1 : best_k;
    }
  } else if (tid < VQ_TT) {
    int r = 0;
    if (t0 + tid < T) {
      const long long k = a.idx[(long long)b * T + t0 + tid];
      r = (k >= 0 && k < a.K) ? (int)k : -1;
    }
    row[tid] = r;
  }
  __syncthreads();
  const float qnan = __int_as_float(0x7fc00000);
  int gr = -1;  // global table row; -2: outside the table (the item's columns are NaN)
  if (a.g) {
    const long long gv = a.g[b];
    gr = (gv >= 0 && gv < a.num_g) ? (int)gv : -2;
  }
  const int Ct = D + a.Cl + a.Cg;
  // gathered codes: (d, frame) with the frame fastest, so the stores are coalesced; the codebook rows stay in L1 / L2
  for (int i = tid; i < D * VQ_TT; i += 256) {
    const int d = i / VQ_TT, tt = i % VQ_TT, t = t0 + tt;
    if (t >= T) continue;
    const int r = row[tt];
    const float v = r >= 0 ? __ldg(a.cb + (long long)r * D + d) : qnan;
    if (a.z_q) a.z_q[((long long)b * D + d) * T + t] = v;
    if (a.dec) a.dec[((long long)b * Ct + d) * T + t] = (STREAM && r == VQ_MASKED) ? 0.f : gr == -2 ? qnan : v;
  }
  if (!a.dec) return;
  for (int i = tid; i < (a.Cl + a.Cg) * VQ_TT; i += 256) {
    const int c = i / VQ_TT, tt = i % VQ_TT, t = t0 + tt;
    if (t >= T) continue;
    float v;
    if (STREAM && row[tt] == VQ_MASKED)
      v = 0.f;
    else if (gr == -2 || row[tt] < 0)
      v = qnan;
    else if (c < a.Cl)
      v = !STREAM ? a.l[((long long)b * a.Cl + c) * T + t]
          : t < a.l_delay ? a.l_hist[((long long)b * a.Cl + c) * a.l_delay + t]
                          : a.l[((long long)b * a.Cl + c) * T + (t - a.l_delay)];
    else
      v = __ldg(a.gtab + (long long)gr * a.Cg + (c - a.Cl));
    a.dec[((long long)b * Ct + D + c) * T + t] = v;
  }
}

__global__ void __launch_bounds__(256) vq_forward_kernel(const VqArgs a) { vq_forward_body<false>(a); }
__global__ void __launch_bounds__(256) vq_stream_kernel(const VqArgs a) { vq_forward_body<true>(a); }

// straight-through adjoint: gz_e (+)= gdec[:, :D]
__global__ void vq_st_backward_kernel(const float* __restrict__ gdec, float* __restrict__ gz, int D, int Ct, int T, long long n,
                                      int accumulate) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long t = i % T, bd = i / T, b = bd / D, d = bd % D;
    const float v = gdec[(b * Ct + d) * T + t];
    gz[i] = accumulate ? gz[i] + v : v;
  }
}

// global-embedding adjoint: one block per table column c; per item a fixed-order block sum over time, added to the
// item's table row in item order
__global__ void __launch_bounds__(256) vq_global_backward_kernel(const float* __restrict__ gdec, const long long* __restrict__ g,
                                                                  int B, int Ct, int c_off, int T, int Cg, int num_g,
                                                                  float* __restrict__ dtab) {
  __shared__ float red[8];
  const int c = blockIdx.x, tid = threadIdx.x;
  for (int r = tid; r < num_g; r += 256) dtab[(long long)r * Cg + c] = 0.f;
  __syncthreads();
  for (int b = 0; b < B; ++b) {
    const long long gv = g[b];
    if (gv < 0 || gv >= num_g) continue;
    const float* src = gdec + ((long long)b * Ct + c_off + c) * T;
    float s = 0.f;
    for (int t = tid; t < T; t += 256) s += src[t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((tid & 31) == 0) red[tid >> 5] = s;
    __syncthreads();
    if (tid == 0) {
      float v = 0.f;
      for (int w = 0; w < 8; ++w) v += red[w];
      dtab[gv * Cg + c] += v;
    }
    __syncthreads();
  }
}

}  // namespace pwgb

using namespace pwgb;

extern "C" int pwgb_vq_forward(const float* z_e, const float* codebook, int num_codes, long long* indices, float* z_q, float* dec,
                               const float* l, int local_channels, const float* global_table, const long long* g, int num_global,
                               int global_channels, int batch, int dim, int t, void* stream) {
  PWGB_CHECK_ARG(batch >= 0 && dim > 0 && t >= 0 && num_codes > 0 && local_channels >= 0 && global_channels >= 0,
                 "vq_forward: bad sizes");
  PWGB_CHECK_ARG(!local_channels == !l && !global_channels == !global_table && !global_table == !g,
                 "vq_forward: a conditioning tensor and its channel count must come together");
  PWGB_CHECK_ARG(!g || num_global > 0, "vq_forward: global table without rows");
  PWGB_CHECK_ARG(dec || (!l && !g), "vq_forward: conditioning without a decoder input to write");
  PWGB_UNSUPPORTED_IF(dim > VQ_MAX_D, "vq_forward: embed_dim %d > %d", dim, VQ_MAX_D);
  PWGB_UNSUPPORTED_IF(batch > 65535, "vq_forward: batch %d > 65535", batch);
  if (batch == 0 || t == 0) return PWGB_OK;
  PWGB_CHECK_ARG(codebook && indices, "vq_forward: null pointer");
  PWGB_CHECK_ARG(z_e || z_q || dec, "vq_forward: nothing to do");
  VqArgs a{z_e, codebook, indices, z_q, dec, l, global_table, g, batch, dim, t, num_codes, local_channels, global_channels, num_global,
           nullptr, 0, nullptr, nullptr, 0};
  const size_t smem = z_e ? (size_t)2 * dim * VQ_TT * sizeof(float) : 0;
  // the static bd_sh / bk_sh / row arrays count too: D = 184 .. 192 fit 48 KiB dynamically but not in total
  const int rc = allow_dynamic_smem(vq_forward_kernel, smem, "vq_forward");
  if (rc) return rc;
  vq_forward_kernel<<<dim3((unsigned)ceil_div(t, VQ_TT), (unsigned)batch), 256, smem, (cudaStream_t)stream>>>(a);
  return check_launch("vq_forward_kernel");
}

extern "C" int pwgb_vq_stream_forward(const float* z_e, const float* codebook, int num_codes, long long* indices, float* dec,
                                      const float* l, const float* l_hist, int l_delay, int local_channels, const float* global_table,
                                      const long long* g, int num_global, int global_channels, const pwgb_stream_ext* ext, int batch,
                                      int dim, int t, void* stream) {
  PWGB_CHECK_ARG(batch >= 0 && dim > 0 && t >= 0 && num_codes > 0 && local_channels >= 0 && global_channels >= 0 && l_delay >= 0,
                 "vq_stream: bad sizes");
  PWGB_CHECK_ARG(!local_channels == !l && (!local_channels || !l_delay || l_hist) && !global_channels == !global_table &&
                     !global_table == !g,
                 "vq_stream: a conditioning tensor and its channel count must come together");
  PWGB_CHECK_ARG(!g || num_global > 0, "vq_stream: global table without rows");
  PWGB_CHECK_ARG(ext && ext->frame && ext->end && ext->rate == 1 && ext->lookahead >= 0 && !ext->res_hist_len && !ext->res_delay &&
                     ext->edge == PWGB_PAD_ZERO,
                 "vq_stream: ext must hold a frame-rate mask (rate 1) and nothing else");
  PWGB_UNSUPPORTED_IF(dim > VQ_MAX_D, "vq_stream: embed_dim %d > %d", dim, VQ_MAX_D);
  PWGB_UNSUPPORTED_IF(batch > 65535, "vq_stream: batch %d > 65535", batch);
  if (batch == 0 || t == 0) return PWGB_OK;
  PWGB_CHECK_ARG(z_e && codebook && indices && dec, "vq_stream: null pointer");
  VqArgs a{z_e, codebook, indices, nullptr, dec, l, global_table, g, batch, dim, t, num_codes, local_channels, global_channels, num_global,
           l_hist, l_delay, ext->frame, ext->end, ext->lookahead};
  const size_t smem = (size_t)2 * dim * VQ_TT * sizeof(float);
  const int rc = allow_dynamic_smem(vq_stream_kernel, smem, "vq_stream");
  if (rc) return rc;
  vq_stream_kernel<<<dim3((unsigned)ceil_div(t, VQ_TT), (unsigned)batch), 256, smem, (cudaStream_t)stream>>>(a);
  return check_launch("vq_stream_kernel");
}

extern "C" int pwgb_vq_backward(const float* gdec, int batch, int dim, int local_channels, int global_channels, int t, float* gz_e,
                                int accumulate, const long long* g, int num_global, float* d_global_table, void* stream) {
  PWGB_CHECK_ARG(batch >= 0 && dim > 0 && t >= 0 && local_channels >= 0 && global_channels >= 0, "vq_backward: bad sizes");
  PWGB_CHECK_ARG(!d_global_table || (g && global_channels > 0 && num_global > 0), "vq_backward: global gradient needs g and its table size");
  cudaStream_t st = (cudaStream_t)stream;
  const int Ct = dim + local_channels + global_channels;
  const long long n = (long long)batch * dim * t;
  if (n == 0) {
    if (d_global_table && cudaMemsetAsync(d_global_table, 0, (size_t)num_global * global_channels * 4, st) != cudaSuccess) {
      set_error("vq_backward: memset failed");
      return PWGB_CUDA_ERROR;
    }
    return PWGB_OK;
  }
  PWGB_CHECK_ARG(gdec && (gz_e || d_global_table), "vq_backward: null pointer");
  int rc;
  if (gz_e) {
    long long blocks = (n + 255) / 256;
    if (blocks > 4096) blocks = 4096;
    vq_st_backward_kernel<<<(unsigned)blocks, 256, 0, st>>>(gdec, gz_e, dim, Ct, t, n, accumulate);
    if ((rc = check_launch("vq_st_backward_kernel"))) return rc;
  }
  if (d_global_table) {
    vq_global_backward_kernel<<<(unsigned)global_channels, 256, 0, st>>>(gdec, g, batch, Ct, dim + local_channels, t, global_channels,
                                                                        num_global, d_global_table);
    if ((rc = check_launch("vq_global_backward_kernel"))) return rc;
  }
  return PWGB_OK;
}
