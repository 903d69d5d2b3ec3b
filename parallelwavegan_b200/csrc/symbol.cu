// Front end of the discrete-symbol HiFi-GAN generators (models/hifigan.py:867-1289): symbol / speaker embedding with
// optional length regulation, its deterministic backward, LayerNorm over channels (layers/layer_norm.py), the
// duration loss (losses/duration_prediction_loss.py), duration rounding with the length regulator's all-zero rule
// (layers/duration_predictor.py:79-83, layers/length_regulator.py:87-95) and the duration collater's run-length
// encoding (bin/train.py:768-783).  No float atomics: every reduction runs in a fixed order.
#include "common.cuh"

namespace pwgb {

constexpr int SE_TT = 32;  // output frames per embed block
constexpr int SE_CC = 64;  // channels per staged chunk

// an index read as torch's c.long(): int64 as is, float32 truncated toward zero; NaN maps to -1 (outside every table)
__device__ __forceinline__ long long load_index(const void* idx, int is64, long long off) {
  if (is64) return reinterpret_cast<const long long*>(idx)[off];
  const float v = reinterpret_cast<const float*>(idx)[off];
  return v != v ? -1LL : (long long)v;
}

// exclusive prefix sum over a 256-thread block; *total receives the block sum (all threads)
__device__ long long block_exclusive_scan_256(long long v, long long* sh /* 9 entries */, long long* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  long long inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  if (lane == 31) sh[wid] = inc;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long run = 0;
    for (int w = 0; w < 8; ++w) {
      const long long t = sh[w];
      sh[w] = run;
      run += t;
    }
    sh[8] = run;
  }
  __syncthreads();
  const long long ex = sh[wid] + inc - v;
  *total = sh[8];
  __syncthreads();  // sh is reused by the next call
  return ex;
}

struct EmbedArgs {
  const void* idx;
  int idx64;
  long long ib, ic, it;  // element strides of the index tensor: batch, channel (speaker row = channel 1), time
  const float* table;
  int num_embs;
  const float* spk;
  int num_spk;
  const long long* ds;  // (B, S) durations or null
  int B, S, C, T_out;
  float* y;  // (B, C, T_out)
};

// The (C, nf) tile of one block's frames, written to y[c * ld + f]: row[f] >= 0 is table row row[f] (+ speaker row g when
// g >= 0), -1 zero, -2 NaN.  Table rows are read along C and the tile is written along time, both coalesced, through
// the transposing tile in shared memory.  The one fp32 expression of every embed launch.
__device__ __forceinline__ void embed_store_tile(const float* __restrict__ table, const float* __restrict__ spk, int C, const int* row,
                                                 int g, float* __restrict__ y, long long ld, int nf, float (*tile)[SE_TT + 1]) {
  const int tid = threadIdx.x;
  for (int c0 = 0; c0 < C; c0 += SE_CC) {
    for (int i = tid; i < SE_TT * SE_CC; i += 256) {
      const int f = i / SE_CC, ch = i % SE_CC, c = c0 + ch;
      const int r = row[f];
      float v = 0.f;
      if (c < C) {
        if (r >= 0) {
          v = __ldg(table + (long long)r * C + c);
          if (g >= 0) v += __ldg(spk + (long long)g * C + c);
        } else if (r == -2) {
          v = __int_as_float(0x7fc00000);
        }
      }
      tile[ch][f] = v;
    }
    __syncthreads();
    for (int i = tid; i < SE_TT * SE_CC; i += 256) {
      const int ch = i / SE_TT, f = i % SE_TT, c = c0 + ch;
      if (c < C && f < nf) y[(long long)c * ld + f] = tile[ch][f];
    }
    __syncthreads();
  }
}

// grid (ceil(T_out / 32), B), 256 threads.  Frame t of row b takes symbol j with prefix[j] <= t < prefix[j] + ds[j]
// (durations) or j = t (none).
__global__ void __launch_bounds__(256) symbol_embed_kernel(const EmbedArgs a) {
  __shared__ int row[SE_TT];  // table row, -1: zero (past the row total), -2: NaN (index outside the table)
  __shared__ int sym[SE_TT];
  __shared__ long long scan_sh[9];
  __shared__ float tile[SE_CC][SE_TT + 1];
  const int b = blockIdx.y, t0 = blockIdx.x * SE_TT, tid = threadIdx.x;
  if (tid < SE_TT) sym[tid] = -1;
  __syncthreads();
  if (a.ds) {
    long long carry = 0;
    for (int j0 = 0; j0 < a.S && carry < t0 + SE_TT; j0 += 256) {
      const int j = j0 + tid;
      long long d = j < a.S ? a.ds[(long long)b * a.S + j] : 0;
      d = d > 0 ? d : 0;
      long long tot;
      const long long st = carry + block_exclusive_scan_256(d, scan_sh, &tot);
      const long long lo = st > t0 ? st : t0, hi = st + d < t0 + SE_TT ? st + d : t0 + SE_TT;
      for (long long t = lo; t < hi; ++t) sym[t - t0] = j;
      carry += tot;
    }
    __syncthreads();
  } else if (tid < SE_TT && t0 + tid < a.S) {
    sym[tid] = t0 + tid;
  }
  __syncthreads();
  int g = -1;  // speaker row, -2: outside the speaker table
  if (a.spk && a.S > 0) {
    const long long k = load_index(a.idx, a.idx64, (long long)b * a.ib + a.ic);
    g = (k >= 0 && k < a.num_spk) ? (int)k : -2;
  }
  if (tid < SE_TT) {
    const int j = sym[tid];
    int r = -1;
    if (j >= 0) {
      const long long k = load_index(a.idx, a.idx64, (long long)b * a.ib + (long long)j * a.it);
      r = (k >= 0 && k < a.num_embs && g != -2) ? (int)k : -2;
    }
    row[tid] = r;
  }
  __syncthreads();
  embed_store_tile(a.table, a.spk, a.C, row, g, a.y + (long long)b * a.C * a.T_out + t0, a.T_out, min(SE_TT, a.T_out - t0), tile);
}

// grid (ceil(n / 32), B), 256 threads: the chunk's frames t0 .. of item b through the same row table and tile store as
// symbol_embed_kernel, into y's columns col0 + t (row stride ld)
__global__ void __launch_bounds__(256, 4) symbol_embed_stream_kernel(const EmbedArgs a, int* __restrict__ latch, const int* __restrict__ fresh,
                                                                  const int* __restrict__ frame, const int* __restrict__ end, long long ld,
                                                                  int col0) {
  __shared__ int row[SE_TT];
  __shared__ float tile[SE_CC][SE_TT + 1];
  const int b = blockIdx.y, t0 = blockIdx.x * SE_TT, tid = threadIdx.x;
  // the speaker of a fresh item is its chunk's first frame's, latched by block 0; the other blocks of a fresh item read
  // it from the chunk too, so no block reads the latch while it is written
  int g = -1;
  if (a.spk) {
    if (__ldg(fresh + b)) {
      const long long k = load_index(a.idx, a.idx64, (long long)b * a.ib + a.ic);
      g = (k >= 0 && k < a.num_spk) ? (int)k : -2;
      if (blockIdx.x == 0 && tid == 0) latch[b] = g;
    } else {
      g = latch[b];
    }
  }
  if (tid < SE_TT) {
    const int j = t0 + tid;
    int r = -1;
    if (j < a.S && !stream_outside(frame, end, 1, 0, b, j)) {
      const long long k = load_index(a.idx, a.idx64, (long long)b * a.ib + (long long)j * a.it);
      r = (k >= 0 && k < a.num_embs && g != -2) ? (int)k : -2;
    }
    row[tid] = r;
  }
  __syncthreads();
  embed_store_tile(a.table, a.spk, a.C, row, g, a.y + (long long)b * a.C * ld + col0 + t0, ld, min(SE_TT, a.S - t0), tile);
}

// ---- embed backward ------------------------------------------------------------------------------------------------
// 1. per-row exclusive prefix of the durations (one block per row)
__global__ void __launch_bounds__(256) duration_prefix_kernel(const long long* __restrict__ ds, long long* __restrict__ start, int S) {
  __shared__ long long scan_sh[9];
  const int b = blockIdx.x;
  long long carry = 0;
  for (int j0 = 0; j0 < S; j0 += 256) {
    const int j = j0 + threadIdx.x;
    long long d = j < S ? ds[(long long)b * S + j] : 0;
    d = d > 0 ? d : 0;
    long long tot;
    const long long st = carry + block_exclusive_scan_256(d, scan_sh, &tot);
    if (j < S) start[(long long)b * S + j] = st;
    carry += tot;
  }
}

// 2. symbol-level gradient, position-major: gs[(b * S + j) * C + c] = sum_{frames t of symbol j, ascending} gy[b, c, t]
//    (+ gsym[b, c, j]).  grid (ceil(S / 32), ceil(C / 32), B), 32 x 8 threads.
__global__ void __launch_bounds__(256) embed_symbol_grad_kernel(const float* __restrict__ gy, const float* __restrict__ gsym,
                                                                 const long long* __restrict__ ds, const long long* __restrict__ start,
                                                                 int S, int C, int T_out, float* __restrict__ gs) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, j0 = blockIdx.x * 32, c0 = blockIdx.y * 32, tx = threadIdx.x, ty = threadIdx.y;
  const int j = j0 + tx;
  long long lo = j, hi = j + 1;
  if (ds && j < S) {
    const long long d = ds[(long long)b * S + j];
    lo = start[(long long)b * S + j];
    hi = lo + (d > 0 ? d : 0);
    if (hi > T_out) hi = T_out;
  }
  for (int k = ty; k < 32; k += 8) {
    const int c = c0 + k;
    float acc = 0.f;
    if (j < S && c < C) {
      const float* g = gy + ((long long)b * C + c) * T_out;
      if (gy)
        for (long long t = lo; t < hi; ++t) acc += g[t];
      if (gsym) acc += gsym[((long long)b * C + c) * S + j];
    }
    tile[k][tx] = acc;
  }
  __syncthreads();
  for (int k = ty; k < 32; k += 8) {
    const int jj = j0 + k, c = c0 + tx;
    if (jj < S && c < C) gs[((long long)b * S + jj) * C + c] = tile[tx][k];
  }
}

// 3. stable counting sort of the positions p = b * S + j by table index (one block; warp 0 ranks equal keys in position
//    order with __match_any_sync).  Positions whose index is outside the table are left out.  off: E + 1 row offsets.
constexpr int SORT_MAX_EMBS = 8192;
__global__ void __launch_bounds__(256) embed_sort_kernel(const void* idx, int idx64, long long ib, long long it, int B, int S,
                                                          int E, int* __restrict__ off, int* __restrict__ perm) {
  __shared__ int cnt[SORT_MAX_EMBS];
  __shared__ int key[256];
  const long long N = (long long)B * S;
  for (int e = threadIdx.x; e < E; e += 256) cnt[e] = 0;
  __syncthreads();
  for (long long p = threadIdx.x; p < N; p += 256) {
    const long long k = load_index(idx, idx64, (p / S) * ib + (p % S) * it);
    if (k >= 0 && k < E) atomicAdd(&cnt[k], 1);  // integer counts: order-independent
  }
  __syncthreads();
  if (threadIdx.x < 32) {  // exclusive scan of the counts: 32 contiguous segments
    const int lane = threadIdx.x, seg = (E + 31) / 32, lo = lane * seg, hi = min(E, lo + seg);
    int s = 0;
    for (int e = lo; e < hi; ++e) s += cnt[e];
    int inc = s;
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += u;
    }
    int run = inc - s;
    for (int e = lo; e < hi; ++e) {
      const int c = cnt[e];
      cnt[e] = run;  // now the cursor of row e
      off[e] = run;
      run += c;
    }
    if (lane == 31) off[E] = inc;
  }
  __syncthreads();
  for (long long p0 = 0; p0 < N; p0 += 256) {
    const long long p = p0 + threadIdx.x;
    int k = -1;
    if (p < N) {
      const long long kk = load_index(idx, idx64, (p / S) * ib + (p % S) * it);
      k = (kk >= 0 && kk < E) ? (int)kk : -1;
    }
    key[threadIdx.x] = k;
    __syncthreads();
    if (threadIdx.x < 32) {
      const int lane = threadIdx.x;
      for (int q = 0; q < 256; q += 32) {
        const int kq = key[q + lane];
        const unsigned m = __match_any_sync(0xffffffffu, kq);
        const int rank = __popc(m & ((1u << lane) - 1u));
        const int base = kq >= 0 ? cnt[kq] : 0;
        __syncwarp();
        if (kq >= 0) {
          perm[base + rank] = (int)(p0 + q + lane);
          if (rank == 0) cnt[kq] = base + __popc(m);
        }
        __syncwarp();
      }
    }
    __syncthreads();
  }
}

// 4. d_emb[e, c] = sum over the sorted positions of row e (position order) of gs[p, c].  grid (E, ceil(C / 128))
__global__ void __launch_bounds__(128) embed_table_grad_kernel(const float* __restrict__ gs, const int* __restrict__ off,
                                                                const int* __restrict__ perm, int C, float* __restrict__ d_emb) {
  const int e = blockIdx.x, c = blockIdx.y * 128 + threadIdx.x;
  if (c >= C) return;
  float acc = 0.f;
  for (int k = off[e]; k < off[e + 1]; ++k) acc += gs[(long long)perm[k] * C + c];
  d_emb[(long long)e * C + c] = acc;
}

// 5. d_spk[g, c] = sum over items b (in order) with speaker g of sum_j gs[b, j, c].  One thread per channel.
__global__ void __launch_bounds__(128) embed_speaker_grad_kernel(const float* __restrict__ gs, const void* idx, int idx64, long long ib,
                                                                  long long ic, int B, int S, int C, int num_spk,
                                                                  float* __restrict__ d_spk) {
  const int c = blockIdx.x * 128 + threadIdx.x;
  if (c >= C) return;
  for (int g = 0; g < num_spk; ++g) d_spk[(long long)g * C + c] = 0.f;
  for (int b = 0; b < B; ++b) {
    const long long k = load_index(idx, idx64, (long long)b * ib + ic);
    if (k < 0 || k >= num_spk) continue;
    float acc = 0.f;
    for (int j = 0; j < S; ++j) acc += gs[((long long)b * S + j) * C + c];
    d_spk[k * C + c] += acc;
  }
}

// ---- LayerNorm over channels ---------------------------------------------------------------------------------------
// grid (ceil(T / 32), B), 32 x 8 threads: lane = frame, the 8 warps split the channels; fixed-order sums.
__global__ void __launch_bounds__(256) channel_layernorm_forward_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                                         const float* __restrict__ beta, int C, int T, float eps,
                                                                         float* __restrict__ y, float* __restrict__ mean_out,
                                                                         float* __restrict__ rstd_out) {
  __shared__ float red[8][33];
  __shared__ float stat[2][32];
  const int b = blockIdx.y, tx = threadIdx.x, ty = threadIdx.y, t = blockIdx.x * 32 + tx;
  const bool ok = t < T;
  const float* xb = x + (long long)b * C * T + t;
  float s = 0.f;
  if (ok)
    for (int c = ty; c < C; c += 8) s += xb[(long long)c * T];
  red[ty][tx] = s;
  __syncthreads();
  if (ty == 0) {
    float m = 0.f;
    for (int k = 0; k < 8; ++k) m += red[k][tx];
    stat[0][tx] = m / (float)C;
  }
  __syncthreads();
  const float mu = stat[0][tx];
  float v = 0.f;
  if (ok)
    for (int c = ty; c < C; c += 8) {
      const float d = xb[(long long)c * T] - mu;
      v += d * d;
    }
  red[ty][tx] = v;
  __syncthreads();
  if (ty == 0) {
    float q = 0.f;
    for (int k = 0; k < 8; ++k) q += red[k][tx];
    stat[1][tx] = 1.f / sqrtf(q / (float)C + eps);
  }
  __syncthreads();
  const float rs = stat[1][tx];
  if (!ok) return;
  if (ty == 0 && mean_out) {
    mean_out[(long long)b * T + t] = mu;
    rstd_out[(long long)b * T + t] = rs;
  }
  float* yb = y + (long long)b * C * T + t;
  for (int c = ty; c < C; c += 8) yb[(long long)c * T] = (xb[(long long)c * T] - mu) * rs * gamma[c] + beta[c];
}

// dx = rstd * (gy*gamma - mean_c(gy*gamma) - xhat * mean_c(gy*gamma*xhat)); per-block partial sums over the block's 32
// frames of gy*xhat and gy for every channel (warp tree, fixed order) into part[blk][2][C]
__global__ void __launch_bounds__(256) channel_layernorm_backward_kernel(const float* __restrict__ x, const float* __restrict__ gy,
                                                                          const float* __restrict__ gamma,
                                                                          const float* __restrict__ mean, const float* __restrict__ rstd,
                                                                          int C, int T, float* __restrict__ dx, float* __restrict__ part) {
  __shared__ float red[2][8][33];
  __shared__ float stat[2][32];
  const int b = blockIdx.y, tx = threadIdx.x, ty = threadIdx.y, t = blockIdx.x * 32 + tx;
  const bool ok = t < T;
  const long long base = (long long)b * C * T + t;
  const float mu = ok ? mean[(long long)b * T + t] : 0.f, rs = ok ? rstd[(long long)b * T + t] : 0.f;
  float* pb = part + ((long long)b * gridDim.x + blockIdx.x) * 2 * C;
  float s1 = 0.f, s2 = 0.f;
  for (int c = ty; c < C; c += 8) {
    float g = 0.f, xh = 0.f;
    if (ok) {
      g = gy[base + (long long)c * T];
      xh = (x[base + (long long)c * T] - mu) * rs;
    }
    const float gg = g * gamma[c];
    s1 += gg;
    s2 += gg * xh;
    float pg = g * xh, pbeta = g;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      pg += __shfl_xor_sync(0xffffffffu, pg, o);
      pbeta += __shfl_xor_sync(0xffffffffu, pbeta, o);
    }
    if (tx == 0) {
      pb[c] = pg;
      pb[C + c] = pbeta;
    }
  }
  red[0][ty][tx] = s1;
  red[1][ty][tx] = s2;
  __syncthreads();
  if (ty == 0) {
    float a1 = 0.f, a2 = 0.f;
    for (int k = 0; k < 8; ++k) {
      a1 += red[0][k][tx];
      a2 += red[1][k][tx];
    }
    stat[0][tx] = a1 / (float)C;
    stat[1][tx] = a2 / (float)C;
  }
  __syncthreads();
  if (!ok) return;
  const float m1 = stat[0][tx], m2 = stat[1][tx];
  for (int c = ty; c < C; c += 8) {
    const long long o = base + (long long)c * T;
    const float xh = (x[o] - mu) * rs;
    dx[o] = rs * (gy[o] * gamma[c] - m1 - xh * m2);
  }
}

// dgamma / dbeta: sum of the per-block partials in block order
__global__ void layernorm_param_grad_kernel(const float* __restrict__ part, int nblk, int C, float* __restrict__ dgamma,
                                            float* __restrict__ dbeta) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * C) return;
  float acc = 0.f;
  for (int k = 0; k < nblk; ++k) acc += part[(long long)k * 2 * C + i];
  if (i < C)
    dgamma[i] = acc;
  else
    dbeta[i - C] = acc;
}

// ---- duration loss / rounding ---------------------------------------------------------------------------------------
// one block, fixed-order double sums
__global__ void __launch_bounds__(256) duration_loss_kernel(const float* __restrict__ x, const long long* __restrict__ d, long long n,
                                                             float offset, float* __restrict__ out) {
  __shared__ double red[256];
  double a = 0;
  for (long long i = threadIdx.x; i < n; i += 256) {
    const float r = x[i] - logf((float)d[i] + offset);
    a += (double)(r * r);
  }
  red[threadIdx.x] = a;
  __syncthreads();
  for (int st = 128; st > 0; st >>= 1) {
    if (threadIdx.x < st) red[threadIdx.x] += red[threadIdx.x + st];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = (float)(red[0] / (double)n);
}

__global__ void duration_loss_backward_kernel(const float* __restrict__ x, const long long* __restrict__ d, long long n, float offset,
                                              const float* __restrict__ gout, float* __restrict__ gx) {
  const float s = 2.f * gout[0] / (float)n;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    gx[i] = s * (x[i] - logf((float)d[i] + offset));
}

// DurationPredictor.inference's rounding of one log-domain duration: max(0, rint(exp(x) - offset))
__device__ __forceinline__ long long round_duration(float x, float offset) {
  const float r = rintf(expf(x) - offset);
  return r > 0.f ? (long long)r : 0LL;
}

// one block: ds = max(0, rint(exp(x) - offset)) (x given), per-row totals, and with zero_rule the length regulator's
// rule: when the whole batch sums to zero, rows summing to zero become all ones
__global__ void __launch_bounds__(256) duration_round_kernel(const float* __restrict__ x, long long* __restrict__ ds,
                                                              long long* __restrict__ totals, int B, int S, float offset,
                                                              int zero_rule) {
  __shared__ unsigned long long batch_sum;
  if (threadIdx.x == 0) batch_sum = 0ULL;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int b = wid; b < B; b += 8) {
    long long s = 0;
    for (int j = lane; j < S; j += 32) {
      const long long o = (long long)b * S + j;
      long long v;
      if (x) {
        v = round_duration(x[o], offset);
        ds[o] = v;
      } else {
        v = ds[o];
      }
      s += v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) {
      totals[b] = s;
      atomicAdd(&batch_sum, (unsigned long long)s);  // integer (two's complement) sum: order-independent
    }
  }
  __syncthreads();
  if (!zero_rule || batch_sum != 0ULL) return;
  for (int b = wid; b < B; b += 8) {
    if (totals[b] != 0) continue;  // ds[ds.sum(dim=1).eq(0)] = 1: only rows summing to zero change
    for (int j = lane; j < S; j += 32) ds[(long long)b * S + j] = 1;
    if (lane == 0) totals[b] = S;
  }
}

// ---- the duration stream's queue ----------------------------------------------------------------------------------
// Per item b a ring of Q (symbol id, duration) entries and rs[b] = {tail, head, hoff, total}: entries [head, tail) are
// queued (ring index i % Q), hoff frames of entry head are consumed, total is the sum of every appended duration;
// counts[b] = {queued frames, overflow flag}.
struct DurQueue {
  long long* ring_id;
  long long* ring_d;
  int Q;
  long long* rs;
  long long* counts;
};

// one warp per item.  Column j of x (B, m) is symbol frame[b] - lookahead + j, final when inside [0, end[b]): its
// rounded duration and ids[b, j] (row stride ids_ld) are appended in order; dur_out[b, j] gets the duration or -1.
// zero_rule (B) flags (x == null, m == 0): an item whose total is 0 gets duration 1 for every queued entry (the length
// regulator's rule for an item alone).
__global__ void duration_queue_append_kernel(const float* __restrict__ x, int m, const long long* __restrict__ ids, long long ids_ld,
                                             const int* __restrict__ frame, const int* __restrict__ end, int lookahead, float offset,
                                             const int* __restrict__ zero_rule, DurQueue q, long long* __restrict__ dur_out) {
  const int b = blockIdx.x;
  if (threadIdx.x != 0) return;
  long long* rs = q.rs + 4LL * b;
  long long* ct = q.counts + 2LL * b;
  long long tail = rs[0], total = rs[3], queued = ct[0];
  const long long head = rs[1];
  if (zero_rule && zero_rule[b] && total == 0) {
    for (long long i = head; i < tail; ++i) q.ring_d[(long long)b * q.Q + i % q.Q] = 1;
    queued = total = tail - head;  // no frame was consumed, so hoff is 0
  }
  for (int j = 0; j < m; ++j) {
    const long long s = (long long)frame[b] - lookahead + j;
    long long d = -1;
    if (s >= 0 && s < (long long)end[b]) {
      d = round_duration(x[(long long)b * m + j], offset);
      if (tail - head >= q.Q) {
        ct[1] = 1;  // overflow: the entry is dropped and the stream must be reset
      } else {
        const long long o = (long long)b * q.Q + tail % q.Q;
        q.ring_id[o] = ids[(long long)b * ids_ld + j];
        q.ring_d[o] = d;
        ++tail;
        queued += d;
        total += d;
      }
    }
    if (dur_out) dur_out[(long long)b * m + j] = d;
  }
  rs[0] = tail;
  rs[3] = total;
  ct[0] = queued;
}

// one block per item: frames [0, n) of the chunk are the next n frames of the item's queue, written into columns
// col0 + t of y (B, C, ld) through symbol_embed_kernel's row table and tile store (a frame past the queue, or at or past
// end[b] of the frame mask, is +0.0); then head / hoff advance by the frames consumed.
__global__ void __launch_bounds__(256, 4) symbol_regulate_stream_kernel(const float* __restrict__ table, int num_embs, int C, DurQueue q,
                                                                        const int* __restrict__ frame, const int* __restrict__ end, int n,
                                                                        float* __restrict__ y, long long ld, int col0) {
  __shared__ int row[SE_TT];
  __shared__ float tile[SE_CC][SE_TT + 1];
  const int b = blockIdx.x, tid = threadIdx.x;
  long long* rs = q.rs + 4LL * b;
  const long long tail = rs[0], head = rs[1], hoff = rs[2];
  const long long* rid = q.ring_id + (long long)b * q.Q;
  const long long* rd = q.ring_d + (long long)b * q.Q;
  for (int t0 = 0; t0 < n; t0 += SE_TT) {
    if (tid < SE_TT) {
      const int f = t0 + tid;
      int r = -1;
      if (f < n && !stream_outside(frame, end, 1, 0, b, f)) {
        long long rem = hoff + f, i = head;
        for (; i < tail; ++i) {
          const long long d = rd[i % q.Q] > 0 ? rd[i % q.Q] : 0;
          if (rem < d) break;
          rem -= d;
        }
        if (i < tail) {
          const long long k = rid[i % q.Q];
          r = (k >= 0 && k < num_embs) ? (int)k : -2;
        }
      }
      row[tid] = r;
    }
    __syncthreads();
    embed_store_tile(table, nullptr, C, row, -1, y + (long long)b * C * ld + col0 + t0, ld, min(SE_TT, n - t0), tile);
  }
  if (tid == 0) {
    long long inside = (long long)end[b] - frame[b];
    inside = inside < 0 ? 0 : (inside > n ? n : inside);
    long long* ct = q.counts + 2LL * b;
    const long long used = inside < ct[0] ? inside : ct[0];
    long long rem = hoff + used, i = head;
    while (i < tail) {
      const long long d = rd[i % q.Q] > 0 ? rd[i % q.Q] : 0;
      if (rem < d) break;
      rem -= d;
      ++i;
    }
    rs[1] = i;
    rs[2] = i < tail ? rem : 0;
    ct[0] -= used;
  }
}

// ---- duration collater ---------------------------------------------------------------------------------------------
// rows f of item b: feats[(c_off[b] + f) * C + ch], read as int64 (truncation); a run starts where a row differs from
// the previous one in any channel.  One block per item.  codes == null: runs[b] = number of runs.  Else write codes
// (B, C, S) and counts (B, S), padded with pad_value / 0 beyond the item's runs.
__device__ __forceinline__ bool run_starts(const float* src, int f, int C) {
  if (f == 0) return true;
  for (int ch = 0; ch < C; ++ch)
    if ((long long)src[(long long)f * C + ch] != (long long)src[(long long)(f - 1) * C + ch]) return true;
  return false;
}

__global__ void __launch_bounds__(256) collate_runlength_kernel(const float* __restrict__ feats, const long long* __restrict__ c_off,
                                                                 int C, int F, long long* __restrict__ runs, long long* __restrict__ codes,
                                                                 long long* __restrict__ counts, int S, long long pad_value) {
  __shared__ long long scan_sh[9];
  const int b = blockIdx.x;
  const float* src = feats + c_off[b] * C;
  long long carry = 0;
  for (int f0 = 0; f0 < F; f0 += 256) {
    const int f = f0 + threadIdx.x;
    const bool st = f < F && run_starts(src, f, C);
    long long tot;
    const long long r = carry + block_exclusive_scan_256(st ? 1 : 0, scan_sh, &tot);
    if (codes && st && r < S) {
      int e = f + 1;
      while (e < F && !run_starts(src, e, C)) ++e;
      for (int ch = 0; ch < C; ++ch) codes[((long long)b * C + ch) * S + r] = (long long)src[(long long)f * C + ch];
      counts[(long long)b * S + r] = e - f;
    }
    carry += tot;
  }
  if (!codes) {
    if (threadIdx.x == 0) runs[b] = carry;
    return;
  }
  for (long long r = carry + threadIdx.x; r < S; r += 256) {
    for (int ch = 0; ch < C; ++ch) codes[((long long)b * C + ch) * S + r] = pad_value;
    counts[(long long)b * S + r] = 0;
  }
}

}  // namespace pwgb

using namespace pwgb;

extern "C" int pwgb_symbol_embed_forward(const void* idx, int idx_int64, long long idx_batch_stride, long long idx_chan_stride,
                                         long long idx_time_stride, const float* table, int num_embs, const float* spk_table,
                                         int num_spk, const long long* durations, int batch, int len, int channels, int t_out,
                                         float* y, void* stream) {
  PWGB_CHECK_ARG(batch >= 0 && len >= 0 && channels > 0 && t_out >= 0 && num_embs > 0, "symbol_embed_forward: bad sizes");
  PWGB_CHECK_ARG(durations || t_out == len, "symbol_embed_forward: without durations t_out must equal the symbol count");
  PWGB_CHECK_ARG(!spk_table || num_spk > 0, "symbol_embed_forward: speaker table without rows");
  PWGB_UNSUPPORTED_IF(batch > 65535, "symbol_embed_forward: batch %d > 65535", batch);
  if (batch == 0 || t_out == 0) return PWGB_OK;
  PWGB_CHECK_ARG(idx && table && y, "symbol_embed_forward: null pointer");
  EmbedArgs a{idx, idx_int64, idx_batch_stride, idx_chan_stride, idx_time_stride, table, num_embs, spk_table, num_spk, durations,
              batch, len, channels, t_out, y};
  dim3 grid((unsigned)ceil_div(t_out, SE_TT), (unsigned)batch);
  symbol_embed_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a);
  return check_launch("symbol_embed_kernel");
}

extern "C" int pwgb_symbol_embed_stream_forward(const void* idx, int idx_int64, long long idx_batch_stride, long long idx_chan_stride,
                                                long long idx_time_stride, const float* table, int num_embs, const float* spk_table,
                                                int num_spk, int* spk_latch, const int* fresh, const int* frame, const int* end, int batch,
                                                int n, int channels, float* y, long long y_len, int y_col0, void* stream) {
  PWGB_CHECK_ARG(batch >= 0 && n >= 0 && channels > 0 && num_embs > 0, "symbol_embed_stream_forward: bad sizes");
  PWGB_CHECK_ARG(y_col0 >= 0 && (long long)y_col0 + n <= y_len, "symbol_embed_stream_forward: columns [%d, %d) outside a %lld-column y",
                 y_col0, y_col0 + n, y_len);
  PWGB_CHECK_ARG(!spk_table || (num_spk > 0 && spk_latch && fresh), "symbol_embed_stream_forward: a speaker table needs rows, the latch and the fresh flags");
  PWGB_UNSUPPORTED_IF(batch > 65535, "symbol_embed_stream_forward: batch %d > 65535", batch);
  if (batch == 0 || n == 0) return PWGB_OK;
  PWGB_CHECK_ARG(idx && table && y && frame && end, "symbol_embed_stream_forward: null pointer");
  EmbedArgs a{idx, idx_int64, idx_batch_stride, idx_chan_stride, idx_time_stride, table, num_embs, spk_table, num_spk, nullptr,
              batch, n, channels, n, y};
  dim3 grid((unsigned)ceil_div(n, SE_TT), (unsigned)batch);
  symbol_embed_stream_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a, spk_latch, fresh, frame, end, y_len, y_col0);
  return check_launch("symbol_embed_stream_kernel");
}

extern "C" int pwgb_duration_queue_append(const float* x, int m, const long long* ids, long long ids_ld, const int* frame, const int* end,
                                          int lookahead, float offset, const int* zero_rule, long long* ring_id, long long* ring_d,
                                          int queue_len, long long* ring_state, long long* counts, long long* dur_out, int batch,
                                          void* stream) {
  PWGB_CHECK_ARG(batch >= 0 && m >= 0 && lookahead >= 0 && queue_len > 0, "duration_queue_append: bad sizes");
  PWGB_UNSUPPORTED_IF(batch > 65535, "duration_queue_append: batch %d > 65535", batch);
  if (batch == 0) return PWGB_OK;
  PWGB_CHECK_ARG(ring_id && ring_d && ring_state && counts && frame && end, "duration_queue_append: null pointer");
  PWGB_CHECK_ARG(m == 0 || (x && ids && ids_ld >= m), "duration_queue_append: null or short input");
  DurQueue q{ring_id, ring_d, queue_len, ring_state, counts};
  duration_queue_append_kernel<<<batch, 32, 0, (cudaStream_t)stream>>>(x, m, ids, ids_ld, frame, end, lookahead, offset, zero_rule, q,
                                                                       dur_out);
  return check_launch("duration_queue_append_kernel");
}

extern "C" int pwgb_symbol_regulate_stream_forward(const float* table, int num_embs, const long long* ring_id, const long long* ring_d,
                                                   int queue_len, long long* ring_state, long long* counts, const int* frame, const int* end,
                                                   int batch, int n, int channels, float* y, long long y_len, int y_col0, void* stream) {
  PWGB_CHECK_ARG(batch >= 0 && n >= 0 && channels > 0 && num_embs > 0 && queue_len > 0, "symbol_regulate_stream_forward: bad sizes");
  PWGB_CHECK_ARG(y_col0 >= 0 && (long long)y_col0 + n <= y_len, "symbol_regulate_stream_forward: columns [%d, %d) outside a %lld-column y",
                 y_col0, y_col0 + n, y_len);
  PWGB_UNSUPPORTED_IF(batch > 65535, "symbol_regulate_stream_forward: batch %d > 65535", batch);
  if (batch == 0 || n == 0) return PWGB_OK;
  PWGB_CHECK_ARG(table && ring_id && ring_d && ring_state && counts && frame && end && y, "symbol_regulate_stream_forward: null pointer");
  DurQueue q{const_cast<long long*>(ring_id), const_cast<long long*>(ring_d), queue_len, ring_state, counts};
  symbol_regulate_stream_kernel<<<batch, 256, 0, (cudaStream_t)stream>>>(table, num_embs, channels, q, frame, end, n, y, y_len, y_col0);
  return check_launch("symbol_regulate_stream_kernel");
}

extern "C" size_t pwgb_symbol_embed_backward_workspace(int batch, int len, int channels, int num_embs) {
  const size_t n = (size_t)batch * len;
  return n * 8 /* starts */ + n * channels * 4 /* gs */ + n * 4 /* perm */ + ((size_t)num_embs + 1) * 4 + 64;
}

extern "C" int pwgb_symbol_embed_backward(const float* gy, const float* gsym, const void* idx, int idx_int64, long long idx_batch_stride,
                                          long long idx_chan_stride, long long idx_time_stride, const long long* durations, int batch,
                                          int len, int channels, int t_out, int num_embs, float* d_emb, int num_spk, float* d_spk,
                                          void* ws, size_t ws_bytes, void* stream) {
  PWGB_CHECK_ARG(batch >= 0 && len >= 0 && channels > 0 && t_out >= 0 && num_embs > 0 && d_emb, "symbol_embed_backward: bad arguments");
  PWGB_CHECK_ARG(durations || t_out == len, "symbol_embed_backward: without durations t_out must equal the symbol count");
  PWGB_CHECK_ARG(!d_spk || num_spk > 0, "symbol_embed_backward: speaker gradient without rows");
  PWGB_UNSUPPORTED_IF(num_embs > SORT_MAX_EMBS, "symbol_embed_backward: %d table rows > %d", num_embs, SORT_MAX_EMBS);
  PWGB_UNSUPPORTED_IF((long long)batch * len > 0x7fffffffLL, "symbol_embed_backward: too many positions");
  PWGB_CHECK_ARG(ws_bytes >= pwgb_symbol_embed_backward_workspace(batch, len, channels, num_embs), "symbol_embed_backward: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)batch * len;
  if (n == 0) {  // no positions: zero gradients
    if (cudaMemsetAsync(d_emb, 0, (size_t)num_embs * channels * 4, st) != cudaSuccess ||
        (d_spk && cudaMemsetAsync(d_spk, 0, (size_t)num_spk * channels * 4, st) != cudaSuccess)) {
      set_error("symbol_embed_backward: memset failed");
      return PWGB_CUDA_ERROR;
    }
    return PWGB_OK;
  }
  PWGB_CHECK_ARG(idx && ws && (gy || gsym), "symbol_embed_backward: null pointer");
  PWGB_UNSUPPORTED_IF(batch > 65535, "symbol_embed_backward: batch %d > 65535", batch);
  char* w = reinterpret_cast<char*>(ws);
  long long* start = reinterpret_cast<long long*>(w);
  float* gs = reinterpret_cast<float*>(w + n * 8);
  int* perm = reinterpret_cast<int*>(w + n * 8 + n * channels * 4);
  int* off = perm + n;
  int rc;
  if (durations) {
    duration_prefix_kernel<<<batch, 256, 0, st>>>(durations, start, len);
    if ((rc = check_launch("duration_prefix_kernel"))) return rc;
  }
  embed_symbol_grad_kernel<<<dim3((unsigned)ceil_div(len, 32), (unsigned)ceil_div(channels, 32), (unsigned)batch), dim3(32, 8), 0, st>>>(
      gy, gsym, durations, start, len, channels, t_out, gs);
  if ((rc = check_launch("embed_symbol_grad_kernel"))) return rc;
  embed_sort_kernel<<<1, 256, 0, st>>>(idx, idx_int64, idx_batch_stride, idx_time_stride, batch, len, num_embs, off, perm);
  if ((rc = check_launch("embed_sort_kernel"))) return rc;
  embed_table_grad_kernel<<<dim3((unsigned)num_embs, (unsigned)ceil_div(channels, 128)), 128, 0, st>>>(gs, off, perm, channels, d_emb);
  if ((rc = check_launch("embed_table_grad_kernel"))) return rc;
  if (d_spk) {
    embed_speaker_grad_kernel<<<ceil_div(channels, 128), 128, 0, st>>>(gs, idx, idx_int64, idx_batch_stride, idx_chan_stride, batch, len,
                                                                     channels, num_spk, d_spk);
    if ((rc = check_launch("embed_speaker_grad_kernel"))) return rc;
  }
  return PWGB_OK;
}

extern "C" int pwgb_channel_layernorm_forward(const float* x, const float* gamma, const float* beta, int batch, int channels, long long t,
                                              float eps, float* y, float* mean, float* rstd, void* stream) {
  PWGB_CHECK_ARG(batch >= 0 && channels > 0 && t >= 0 && (!mean == !rstd), "channel_layernorm_forward: bad arguments");
  PWGB_UNSUPPORTED_IF(batch > 65535 || t > 0x7fffffffLL, "channel_layernorm_forward: tensor too large");
  if (batch == 0 || t == 0) return PWGB_OK;
  PWGB_CHECK_ARG(x && gamma && beta && y, "channel_layernorm_forward: null pointer");
  channel_layernorm_forward_kernel<<<dim3((unsigned)ceil_div((int)t, 32), (unsigned)batch), dim3(32, 8), 0, (cudaStream_t)stream>>>(
      x, gamma, beta, channels, (int)t, eps, y, mean, rstd);
  return check_launch("channel_layernorm_forward_kernel");
}

extern "C" size_t pwgb_channel_layernorm_backward_workspace(int batch, int channels, long long t) {
  return (size_t)batch * ceil_div((int)t, 32) * 2 * channels * 4 + 16;
}

extern "C" int pwgb_channel_layernorm_backward(const float* x, const float* gy, const float* gamma, const float* mean, const float* rstd,
                                               int batch, int channels, long long t, float* dx, float* dgamma, float* dbeta, void* ws,
                                               size_t ws_bytes, void* stream) {
  PWGB_CHECK_ARG(batch >= 0 && channels > 0 && t >= 0 && dgamma && dbeta, "channel_layernorm_backward: bad arguments");
  PWGB_UNSUPPORTED_IF(batch > 65535 || t > 0x7fffffffLL, "channel_layernorm_backward: tensor too large");
  cudaStream_t st = (cudaStream_t)stream;
  if (batch == 0 || t == 0) {
    if (cudaMemsetAsync(dgamma, 0, (size_t)channels * 4, st) != cudaSuccess || cudaMemsetAsync(dbeta, 0, (size_t)channels * 4, st) != cudaSuccess) {
      set_error("channel_layernorm_backward: memset failed");
      return PWGB_CUDA_ERROR;
    }
    return PWGB_OK;
  }
  PWGB_CHECK_ARG(x && gy && gamma && mean && rstd && dx && ws, "channel_layernorm_backward: null pointer");
  PWGB_CHECK_ARG(ws_bytes >= pwgb_channel_layernorm_backward_workspace(batch, channels, t), "channel_layernorm_backward: workspace too small");
  const int tb = ceil_div((int)t, 32);
  float* part = reinterpret_cast<float*>(ws);
  channel_layernorm_backward_kernel<<<dim3((unsigned)tb, (unsigned)batch), dim3(32, 8), 0, st>>>(x, gy, gamma, mean, rstd, channels, (int)t,
                                                                                                 dx, part);
  int rc = check_launch("channel_layernorm_backward_kernel");
  if (rc) return rc;
  layernorm_param_grad_kernel<<<ceil_div(2 * channels, 256), 256, 0, st>>>(part, batch * tb, channels, dgamma, dbeta);
  return check_launch("layernorm_param_grad_kernel");
}

extern "C" int pwgb_duration_loss_forward(const float* x, const long long* d, long long n, float offset, float* out, void* stream) {
  PWGB_CHECK_ARG(x && d && out && n > 0, "duration_loss_forward: bad arguments");
  duration_loss_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(x, d, n, offset, out);
  return check_launch("duration_loss_kernel");
}

extern "C" int pwgb_duration_loss_backward(const float* x, const long long* d, long long n, float offset, const float* gout, float* gx,
                                           void* stream) {
  PWGB_CHECK_ARG(x && d && gout && gx && n > 0, "duration_loss_backward: bad arguments");
  long long blocks = (n + 255) / 256;
  if (blocks > 1024) blocks = 1024;
  duration_loss_backward_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, d, n, offset, gout, gx);
  return check_launch("duration_loss_backward_kernel");
}

extern "C" int pwgb_duration_round(const float* x, long long* ds, long long* totals, int batch, int len, float offset, int zero_rule,
                                   void* stream) {
  PWGB_CHECK_ARG(batch >= 0 && len >= 0, "duration_round: bad sizes");
  if (batch == 0) return PWGB_OK;
  PWGB_CHECK_ARG(totals && (ds || len == 0), "duration_round: null pointer");
  duration_round_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(x, ds, totals, batch, len, offset, zero_rule);
  return check_launch("duration_round_kernel");
}

extern "C" int pwgb_collate_runlength(const float* feats, const long long* c_offsets, int batch, int channels, int frames, long long* runs,
                                      long long* codes, long long* counts, int max_runs, long long pad_value, void* stream) {
  PWGB_CHECK_ARG(batch >= 0 && channels > 0 && frames > 0, "collate_runlength: bad sizes");
  PWGB_CHECK_ARG(codes ? (counts && max_runs >= 0) : runs != nullptr, "collate_runlength: null output");
  if (batch == 0) return PWGB_OK;
  PWGB_CHECK_ARG(feats && c_offsets, "collate_runlength: null input");
  collate_runlength_kernel<<<batch, 256, 0, (cudaStream_t)stream>>>(feats, c_offsets, channels, frames, runs, codes, counts, max_runs,
                                                                    pad_value);
  return check_launch("collate_runlength_kernel");
}
