// Stride-1 Conv1d on the Hopper tensor cores (wgmma, fp32 accumulators in registers), fp32-accurate via a bf16x3
// operand split:  x = xh + xl, w = wh + wl (bf16 each),  x*w ~= xh*wh + xl*wh + xh*wl  with fp32 accumulation
// (dropped term xl*wl ~ 2^-16 relative).  One pass of plain TF32/BF16 does not meet the 1e-3 parity bar end to end
// (SURVEY.md 7 "hard parts").
//
// Formulation (im2col is never materialised): TIME is the MMA M dimension.
//   D[t, co] += sum_{ci in 16-chunk} A_k[t, ci] * B_k[co, ci]      for every tap k
//   A_k = rows (t0 + t + k*dilation - pad) of the staged activation tile  -> a *row offset*
//         into ONE shared-memory tile, expressed through the wgmma descriptor start address;
//   B_k = W[:, :, k] pre-packed (hi/lo bf16) in global memory in the exact smem image.
// Both operands are K-major, no-swizzle ("interleaved") core-matrix layouts:
//   [ci/8][row][8 ci] bf16  -> 16 B per (row, 8 channels); 8-row core matrices are contiguous
//   (SBO = 128 B) so any row offset is a legal 16 B-aligned descriptor start, and the K-adjacent
//   core matrix sits LBO = rows*16 B away.
// Warp roles (576 threads, one persistent CTA per SM; every role loops over the same tile sequence and
// talks through mbarriers only):
//   warps 0-7   A producers: convert landed raw fp32 stages (pre-activation, padding mask, bf16 hi/lo split)
//               into the K-major operand image, 16 B st.shared.
//   warps 8-15  consumers, two warpgroups: warpgroup g issues the wgmma of its 64 (MT = 2: 128) rows of the tile into
//               registers (<= 128 columns: 64 fp32 per thread), then runs bias / act / residual / scale / accumulate
//               and stores.
//   warp 16     B producer: cp.async.bulk (TMA, 1-D) of one packed weight stage per (chunk, tap).
//   warp 17     raw activation loader: cp.async.bulk row copies into the raw fp32 ring.
#include "tc_common.cuh"

namespace pwgb {

constexpr int NPROD = 256;  // producer threads (warps 0-7); 4 warps measured slower (conversion-bound)
constexpr int NCONS = 256;  // consumer threads (warps 8-15: two warpgroups)
// warp roles after the producers / consumers: weight TMA, activation TMA
constexpr int W_CONS0 = NPROD / 32, W_TMA = (NPROD + NCONS) / 32, W_LDA = W_TMA + 1;
constexpr int TC_THREADS = NPROD + NCONS + 64;
constexpr int NS_MAX = 4;  // raw activation stages

struct TcK {
  int B, Cin, Cout, T_in, T_out, K, D, padL, pad_mode;
  float pre_slope;
  int post_act;
  float post_slope;
  float out_scale;
  int accumulate;
  int shuffle, shuffle_pad, shuffle_tout;
  int MT, R, nchunks, tiles_per_seq, nb, na, total_tiles;
  int ns;                // raw fp32 staging buffers for the activation chunks (0 = direct register path)
  int R4, raw_bytes;     // raw stage: KC rows of R4 floats (R4 = R + alignment slack, multiple of 4)
  int tma_act;           // 1: raw stages are filled by cp.async.bulk row copies (warp W_LDA), 0: by cp.async (producers)
  int nco;               // column chunks of Cout channels sharing this launch (conv-transpose: cout * stride > 256; wide / grouped convs)
  int cpg;               // column chunks per group (grouped convs: chunk cc reads the input channels of group cc / cpg)
  long long xgs;         // input offset between groups (elements): cin_per_group * T_in, 0 for dense convs
  long long xbs, ybs, rbs;
  int a_bytes, b_bytes;  // per buffer / per stage
  int win_mode;          // 1: one TT-row window per tap (halo too large for a contiguous tile)
  int nchunks2, C2;      // auxiliary 1x1 source (WaveNet conditioning): extra K=1 chunks
  int pre_gate;          // producer computes tanh(x[c]) * sigmoid(x[c + Cin])
  int wavenet;           // epilogue: cols < split -> y2 += v ; cols >= split -> y = (v + res) * scale
  int split;
  int co_off;            // first output channel of this launch (N-chunked callers)
  int variant;           // debug (pwgb_debug_set(1, v)): bit 1 stages activations with cp.async instead of TMA
};

// ------------------------------------------------------------------ weight packing
// w (rows, cin_real, K) fp32 -> rows [co_begin, co_begin + rows) of the operand image
// [chunk][tap][hi|lo][ci8][co (cout_total)][8] bf16 (the smem image of a stage); input channels
// >= cin_real (zero padding up to cin_pad, a multiple of KC) pack as zeros.
__global__ void tc_pack_weight_kernel(const float* __restrict__ w, uint4* __restrict__ packed, int cin_real, int cin_pad, int rows,
                                      int K, int co_begin, int cout_total, int chunk) {
  // chunk > 0: `rows` output channels are split into consecutive images of `chunk` columns each (wide / grouped convs:
  // one image per (group, column chunk)); chunk == 0: rows [co_begin, co_begin + rows) of ONE image of cout_total columns
  const int nchunks = cin_pad / KC;
  const long long n = (long long)nchunks * K * (KC / 8) * rows;
  const long long img16 = (long long)nchunks * K * 2 * (KC / 8) * (chunk > 0 ? chunk : cout_total);  // uint4 per image
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int co = (int)(i % rows);
    long long t = i / rows;
    int g = (int)(t % (KC / 8));
    t /= (KC / 8);
    int k = (int)(t % K);
    int c = (int)(t / K);
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int ci = c * KC + g * 8 + j;
      v[j] = ci < cin_real ? w[((long long)co * cin_real + ci) * K + k] : 0.f;
    }
    uint4 hi, lo;
    split8(v, hi, lo);
    const int ct = chunk > 0 ? chunk : cout_total;
    const int col = chunk > 0 ? co % chunk : co_begin + co;
    uint4* img = packed + (chunk > 0 ? (long long)(co / chunk) * img16 : 0);
    const long long base = ((long long)(c * K + k) * 2) * (KC / 8) * ct;
    img[base + (long long)g * ct + col] = hi;
    img[base + (long long)(KC / 8) * ct + (long long)g * ct + col] = lo;
  }
}

void tc_pack_rows(const float* w, void* packed, int cin_real, int cin_pad, int rows, int K, int co_begin,
                         int cout_total, cudaStream_t st) {
  const long long n = (long long)(cin_pad / KC) * K * (KC / 8) * rows;
  int blocks = (int)((n + 127) / 128);
  if (blocks > 8192) blocks = 8192;
  if (blocks < 1) blocks = 1;
  tc_pack_weight_kernel<<<blocks, 128, 0, st>>>(w, (uint4*)packed, cin_real, cin_pad, rows, K, co_begin, cout_total, 0);
}

// Epilogue of one accumulator element (row t, column col of the launch's column chunk starting at co_base).
__device__ __forceinline__ void epi_store(const TcK& p, float a, int b, int t, int col, int co_base, const float* __restrict__ bias,
                                          const float* bias_s, const float* __restrict__ res, float* __restrict__ y,
                                          float* __restrict__ y2) {
  const long long st = p.T_out;
  if (p.shuffle > 1) {
    const int co = co_base + col, cof = co / p.shuffle;
    float v = a + (bias ? __ldg(bias + cof) : 0.f);
    if (p.post_act == PWGB_ACT_TANH)
      v = tanhf(v);
    else if (p.post_act == PWGB_ACT_LRELU)
      v = lrelu(v, p.post_slope);
    const int of = t * p.shuffle + (co - cof * p.shuffle) - p.shuffle_pad;
    if (of >= 0 && of < p.shuffle_tout) y[(long long)b * p.ybs + (long long)cof * p.shuffle_tout + of] = v * p.out_scale;
  } else if (p.wavenet) {
    // WaveNet split epilogue (residual_block.py:131-138): columns [0, split) are the skip 1x1
    // (accumulated into y2), columns [split, Cout) the residual 1x1: y = (v + x) * sqrt(0.5)
    const bool is_skip = col < p.split;
    const int ch = is_skip ? col : col - p.split, nch = is_skip ? p.split : p.Cout - p.split;
    const long long off = ((long long)b * nch + ch) * st + t;
    const float v = a + bias_s[col];
    if (is_skip)
      y2[off] = v + y2[off];
    else
      y[off] = (v + __ldg(res + off)) * p.out_scale;
  } else {
    // several column chunks per launch: bias_s holds the bias of every chunk
    const long long off = (long long)(co_base + col) * st + t;
    float v = a + bias_s[co_base - p.co_off + col];
    if (p.post_act != PWGB_ACT_NONE) v = p.post_act == PWGB_ACT_TANH ? tanhf(v) : lrelu(v, p.post_slope);
    if (res) v += __ldg(res + (long long)b * p.rbs + off);
    v *= p.out_scale;
    float* q = y + (long long)b * p.ybs + off;
    if (p.accumulate) v += *q;
    *q = v;
  }
}

// ------------------------------------------------------------------ main kernel
// Persistent: one CTA per SM loops over (batch, time-tile) work items; every role runs the same
// tile sequence and talks through mbarriers only, so the loads of tile i+1 overlap the MMAs and the
// epilogue of tile i.

// stage one activation chunk (KC channels x R rows) into the operand layout
__device__ __forceinline__ void fill_main_chunk(const TcK& p, const float* __restrict__ xc, int t0, int TT,
                                                unsigned char* dst, int tid) {
  auto src_of = [&](int r, bool& ok) -> long long {
    long long ts;
    if (p.win_mode) {
      const int k = r / TT;
      ts = (long long)t0 - p.padL + (long long)k * p.D + (r - k * TT);
    } else {
      ts = (long long)t0 - p.padL + r;
    }
    ok = true;
    if (ts < 0 || ts >= p.T_in) {
      if (p.pad_mode == PWGB_PAD_ZERO) {
        ok = false;
      } else if (p.pad_mode == PWGB_PAD_REFLECT) {
        ts = ts < 0 ? -ts : 2LL * (p.T_in - 1) - ts;
        ok = ts >= 0 && ts < p.T_in;
      } else {
        ts = ts < 0 ? 0 : p.T_in - 1;
      }
    }
    return ts;
  };
  auto store_row = [&](const float (&v)[KC], int r) {
#pragma unroll
    for (int g = 0; g < KC / 8; ++g) {
      float u[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) u[j] = v[g * 8 + j];
      uint4 hi, lo;
      split8(u, hi, lo);
      *reinterpret_cast<uint4*>(dst + ((size_t)g * p.R + r) * 16) = hi;
      *reinterpret_cast<uint4*>(dst + ((size_t)(KC / 8 + g) * p.R + r) * 16) = lo;
    }
  };
  if (p.pre_gate) {
    const float* xg = xc + (long long)p.Cin * p.T_in;
    for (int r = tid; r < p.R; r += NPROD) {
      bool ok;
      const long long ts = src_of(r, ok);
      float v[KC], sg[KC];
#pragma unroll
      for (int j = 0; j < KC; ++j) {
        v[j] = ok ? __ldg(xc + (long long)j * p.T_in + ts) : 0.f;
        sg[j] = ok ? __ldg(xg + (long long)j * p.T_in + ts) : 0.f;
      }
#pragma unroll
      for (int j = 0; j < KC; ++j) v[j] = tanhf(v[j]) * sigmoidf_(sg[j]);
      store_row(v, r);
    }
    return;
  }
  for (int r = tid; r < p.R; r += NPROD) {
    bool ok;
    const long long ts = src_of(r, ok);
    float v[KC];
#pragma unroll
    for (int j = 0; j < KC; ++j) v[j] = ok ? __ldg(xc + (long long)j * p.T_in + ts) : 0.f;
#pragma unroll
    for (int j = 0; j < KC; ++j) v[j] = lrelu(v[j], p.pre_slope);
    store_row(v, r);
  }
}

__global__ void __launch_bounds__(TC_THREADS, 1)
    conv1d_tc_kernel(const TcK p, const float* __restrict__ x, const float* __restrict__ x2,
                     const uint4* __restrict__ wpk, const float* __restrict__ bias, const float* __restrict__ res,
                     float* __restrict__ y, float* __restrict__ y2) {
  extern __shared__ __align__(128) unsigned char smem[];
  // layout: A[na] | B[nb] | raw staging[ns] | barriers | bias
  unsigned char* a_buf = smem;
  unsigned char* b_buf = smem + (size_t)p.na * p.a_bytes;
  unsigned char* raw_buf = b_buf + (size_t)p.nb * p.b_bytes;
  unsigned long long* bars = reinterpret_cast<unsigned long long*>(raw_buf + (size_t)p.ns * p.raw_bytes);
  const int nbar = 2 * p.na + 2 * p.nb + 4 + 2 * NS_MAX;
  float* bias_s = reinterpret_cast<float*>(bars + nbar + 2);  // Cout floats (0 when bias == nullptr)
  // several column chunks / groups of a plain (non pixel-shuffle) conv share the launch
  const bool MC = p.nco > 1 && p.shuffle <= 1;

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int TT = p.MT * 128;
  const int nc_total = p.nchunks + p.nchunks2;
  const int pct = p.B * p.tiles_per_seq;  // work items per column chunk (nco chunks share one launch)

  const unsigned bar0 = smem_u32(bars);
  auto A_FULL = [&](int i) { return bar0 + 8u * i; };
  auto A_EMPTY = [&](int i) { return bar0 + 8u * (p.na + i); };
  auto B_FULL = [&](int i) { return bar0 + 8u * (2 * p.na + i); };
  auto B_EMPTY = [&](int i) { return bar0 + 8u * (2 * p.na + p.nb + i); };
  auto RAW_FULL = [&](int i) { return bar0 + 8u * (2 * p.na + 2 * p.nb + 4 + i); };
  auto RAW_EMPTY = [&](int i) { return bar0 + 8u * (2 * p.na + 2 * p.nb + 4 + NS_MAX + i); };

  if (tid == 0) {
    for (int i = 0; i < p.na; ++i) {
      mbar_init(A_FULL(i), NPROD);
      mbar_init(A_EMPTY(i), NCONS / 32);
    }
    for (int i = 0; i < p.nb; ++i) {
      mbar_init(B_FULL(i), 1);
      mbar_init(B_EMPTY(i), NCONS / 32);
    }
    for (int i = 0; i < NS_MAX; ++i) {
      mbar_init(RAW_FULL(i), 1);
      mbar_init(RAW_EMPTY(i), NPROD);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = tid; i < p.Cout * (MC ? p.nco : 1); i += TC_THREADS)
    bias_s[i] = bias ? __ldg(bias + (p.shuffle > 1 ? (p.co_off + i) / p.shuffle : p.co_off + i)) : 0.f;
  __syncthreads();

  if (warp < W_CONS0 && p.tma_act) {
    // ===================== A producers, TMA-staged =====================
    // Warp W_LDA streams the raw fp32 rows of chunk q + ns - 1 into shared memory with bulk copies
    // (no LSU instructions, no registers); these 8 warps only convert landed stages to the bf16 hi/lo
    // operand image.  Stages start at a 16-byte aligned sample, `shift` re-aligns the rows; samples
    // outside [0, T) are never copied and are masked here (zero padding).
    int s = 0, sph = 0, buf = 0, aph = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const int tr = p.nco > 1 ? tile % pct : tile;  // tile within its column chunk
      const int b = tr / p.tiles_per_seq;
      const int t0 = (tr - b * p.tiles_per_seq) * TT;
      const int ts_first = t0 - p.padL;
      const int shift = ts_first - (ts_first & ~3);
      for (int c = 0; c < nc_total; ++c) {
        mbar_wait(RAW_FULL(s), sph);
        mbar_wait(A_EMPTY(buf), aph ^ 1);
        unsigned char* dst = a_buf + (size_t)buf * p.a_bytes;
        const float* raw = reinterpret_cast<const float*>(raw_buf + (size_t)s * p.raw_bytes);
        const bool main_chunk = c < p.nchunks;
        const int rows = main_chunk ? p.R : TT;
        const int sh = main_chunk ? shift : 0;
        const int tbase = main_chunk ? ts_first : t0;
        const unsigned tlim = (unsigned)(main_chunk ? p.T_in : p.T_out);
        const float slope = main_chunk ? p.pre_slope : 1.f;
        for (int r = tid; r < rows; r += NPROD) {
          const bool ok = (unsigned)(tbase + r) < tlim;
          const float* rr = raw + r + sh;
#pragma unroll
          for (int g = 0; g < KC / 8; ++g) {
            float u[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) u[j] = ok ? lrelu(rr[(g * 8 + j) * p.R4], slope) : 0.f;
            uint4 hi, lo;
            split8(u, hi, lo);
            *reinterpret_cast<uint4*>(dst + ((size_t)g * p.R + r) * 16) = hi;
            *reinterpret_cast<uint4*>(dst + ((size_t)(KC / 8 + g) * p.R + r) * 16) = lo;
          }
        }
        fence_proxy_async();
        mbar_arrive(A_FULL(buf));
        mbar_arrive(RAW_EMPTY(s));
        if (++s == p.ns) { s = 0; sph ^= 1; }
        if (++buf == p.na) { buf = 0; aph ^= 1; }
      }
    }
  } else if (warp < W_CONS0 && p.ns > 0) {
    // ===================== A producers, cp.async-staged =====================
    // The raw fp32 chunk q+1 streams into shared memory (no registers held, any padding policy by
    // per-element addressing, zero-fill through src-size 0) while chunk q is converted to the bf16
    // hi/lo operand image: global-memory latency is decoupled from the conversion.
    const int ntile_local = (p.total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const int nq = ntile_local * nc_total;
    auto issue = [&](int q) {
      const int tile = blockIdx.x + (q / nc_total) * gridDim.x;
      const int c = q % nc_total;
      const int tr = p.nco > 1 ? tile % pct : tile;  // tile within its column chunk
      const int b = tr / p.tiles_per_seq;
      const int t0 = (tr - b * p.tiles_per_seq) * TT;
      const unsigned raw = smem_u32(raw_buf + (size_t)(q % p.ns) * p.raw_bytes);
      if (c < p.nchunks) {
        const float* xc = x + (long long)b * p.xbs + (long long)(c * KC) * p.T_in + (MC ? (long long)((tile / pct) / p.cpg) * p.xgs : 0);
        for (int r = tid; r < p.R; r += NPROD) {
          long long ts;
          if (p.win_mode) {
            const int k = r / TT;
            ts = (long long)t0 - p.padL + (long long)k * p.D + (r - k * TT);
          } else {
            ts = (long long)t0 - p.padL + r;
          }
          bool ok = true;
          if (ts < 0 || ts >= p.T_in) {
            if (p.pad_mode == PWGB_PAD_ZERO) {
              ok = false;
            } else if (p.pad_mode == PWGB_PAD_REFLECT) {
              ts = ts < 0 ? -ts : 2LL * (p.T_in - 1) - ts;
              ok = ts >= 0 && ts < p.T_in;
            } else {
              ts = ts < 0 ? 0 : p.T_in - 1;
            }
          }
          const float* src = ok ? xc + ts : xc;
          const unsigned nbytes = ok ? 4u : 0u;
          unsigned dq = raw + (unsigned)r * 4u;
          const unsigned dstep = (unsigned)p.R * 4u;
#pragma unroll 8
          for (int j = 0; j < KC; ++j, src += p.T_in, dq += dstep) cp_async4(dq, src, nbytes);
        }
      } else {
        const float* xc = x2 + ((long long)b * p.C2 + (long long)(c - p.nchunks) * KC) * p.T_out;
        for (int r = tid; r < TT; r += NPROD) {
          const long long ts = (long long)t0 + r;
          const bool ok = ts < p.T_out;
          const float* src = ok ? xc + ts : xc;
          const unsigned nbytes = ok ? 4u : 0u;
          unsigned dq = raw + (unsigned)r * 4u;
          const unsigned dstep = (unsigned)p.R * 4u;
#pragma unroll 8
          for (int j = 0; j < KC; ++j, src += p.T_out, dq += dstep) cp_async4(dq, src, nbytes);
        }
      }
      cp_async_commit();
    };
    if (nq > 0) issue(0);
    for (int q = 0; q < nq; ++q) {
      if (q + 1 < nq) {
        issue(q + 1);
        cp_async_wait<1>();
      } else {
        cp_async_wait<0>();
      }
      producer_barrier();  // every producer's copies of chunk q have landed
      const int c = q % nc_total;
      const int buf = q % p.na;
      mbar_wait(A_EMPTY(buf), ((q / p.na) & 1) ^ 1);
      unsigned char* dst = a_buf + (size_t)buf * p.a_bytes;
      const float* raw = reinterpret_cast<const float*>(raw_buf + (size_t)(q % p.ns) * p.raw_bytes);
      const int rows = c < p.nchunks ? p.R : TT;
      const float slope = c < p.nchunks ? p.pre_slope : 1.f;
      for (int r = tid; r < rows; r += NPROD) {
#pragma unroll
        for (int g = 0; g < KC / 8; ++g) {
          float u[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) u[j] = lrelu(raw[(g * 8 + j) * p.R + r], slope);
          uint4 hi, lo;
          split8(u, hi, lo);
          *reinterpret_cast<uint4*>(dst + ((size_t)g * p.R + r) * 16) = hi;
          *reinterpret_cast<uint4*>(dst + ((size_t)(KC / 8 + g) * p.R + r) * 16) = lo;
        }
      }
      fence_proxy_async();
      mbar_arrive(A_FULL(buf));
      producer_barrier();  // raw[q % ns] may be overwritten by issue(q + 2)
    }
  } else if (warp < W_CONS0) {
    // ===================== A producers, direct register path =====================
    unsigned ca = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const int tr = p.nco > 1 ? tile % pct : tile;  // tile within its column chunk
      const int b = tr / p.tiles_per_seq;
      const int t0 = (tr - b * p.tiles_per_seq) * TT;
      const float* xb = x + (long long)b * p.xbs + (MC ? (long long)((tile / pct) / p.cpg) * p.xgs : 0);
      for (int c = 0; c < nc_total; ++c, ++ca) {
        const int buf = ca % p.na;
        mbar_wait(A_EMPTY(buf), ((ca / p.na) & 1) ^ 1);
        unsigned char* dst = a_buf + (size_t)buf * p.a_bytes;
        if (c < p.nchunks) {
          fill_main_chunk(p, xb + (long long)(c * KC) * p.T_in, t0, TT, dst, tid);
        } else {
          // auxiliary 1x1 source: TT rows aligned with the output tile, no padding shift, no activation
          const float* xc = x2 + ((long long)b * p.C2 + (long long)(c - p.nchunks) * KC) * p.T_out;
          for (int r = tid; r < TT; r += NPROD) {
            const long long ts = (long long)t0 + r;
            const bool ok = ts < p.T_out;
#pragma unroll
            for (int g = 0; g < KC / 8; ++g) {
              float u[8];
#pragma unroll
              for (int j = 0; j < 8; ++j) u[j] = ok ? __ldg(xc + (long long)(g * 8 + j) * p.T_out + ts) : 0.f;
              uint4 hi, lo;
              split8(u, hi, lo);
              *reinterpret_cast<uint4*>(dst + ((size_t)g * p.R + r) * 16) = hi;
              *reinterpret_cast<uint4*>(dst + ((size_t)(KC / 8 + g) * p.R + r) * 16) = lo;
            }
          }
        }
        fence_proxy_async();  // generic-proxy smem writes -> visible to the tensor core (async proxy)
        mbar_arrive(A_FULL(buf));
      }
    }
  } else if (warp < W_TMA) {
    // ===================== consumers: wgmma into registers, then the epilogue =====================
    // warpgroup wg owns the 64-row blocks wg * MT + mb of the tile; per (chunk, tap) and 16-channel K-step the three
    // bf16x3 products of every block, one wait per weight stage before the stage is handed back
    const int wg = (warp - W_CONS0) >> 2, wq = warp & 3;
    const int nb16 = p.Cout / 16;
    const unsigned lbo_a = (unsigned)p.R * 16u, lbo_b = (unsigned)p.Cout * 16u;
    const unsigned a_sub = (unsigned)(KC / 8) * p.R, b_sub = (unsigned)(KC / 8) * p.Cout;  // hi -> lo image (16-byte units)
    int buf = 0, aph = 0, s = 0, bph = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      float acc[64];
#pragma unroll
      for (int e = 0; e < 64; ++e) acc[e] = 0.f;
      for (int c = 0; c < nc_total; ++c) {
        mbar_wait_spin(A_FULL(buf), aph);
        const unsigned a_addr = smem_u32(a_buf + (size_t)buf * p.a_bytes);
        const int ntaps = c < p.nchunks ? p.K : 1;
        for (int k = 0; k < ntaps; ++k) {
          mbar_wait_spin(B_FULL(s), bph);
          __syncwarp();
          const unsigned b_addr = smem_u32(b_buf + (size_t)s * p.b_bytes);
          const int tap_row = c < p.nchunks ? (p.win_mode ? k * TT : k * p.D) : 0;
          wg_fence();
#pragma unroll
          for (int ks = 0; ks < KC / 16; ++ks) {
            const unsigned long long bh = gmma_desc(b_addr + (unsigned)(2 * ks) * lbo_b, lbo_b, 128);
            const unsigned long long ah0 =
                gmma_desc(a_addr + ((unsigned)(2 * ks) * p.R + (unsigned)(tap_row + wg * p.MT * 64)) * 16u, lbo_a, 128);
            if (p.MT == 1) {
              wgmma_cols<0, 0, 8>(acc, ah0, bh, nb16, 16);
              wgmma_cols<0, 0, 8>(acc, ah0 + a_sub, bh, nb16, 16);
              wgmma_cols<0, 0, 8>(acc, ah0, bh + b_sub, nb16, 16);
            } else {
              const unsigned long long ah1 = ah0 + 64;  // next 64 rows: 64 x 16 B
              wgmma_cols<0, 0, 4>(acc, ah0, bh, nb16, 16);
              wgmma_cols<0, 0, 4>(acc, ah0 + a_sub, bh, nb16, 16);
              wgmma_cols<0, 0, 4>(acc, ah0, bh + b_sub, nb16, 16);
              wgmma_cols<0, 0, 4>(acc + 32, ah1, bh, nb16, 16);
              wgmma_cols<0, 0, 4>(acc + 32, ah1 + a_sub, bh, nb16, 16);
              wgmma_cols<0, 0, 4>(acc + 32, ah1, bh + b_sub, nb16, 16);
            }
          }
          wg_commit();
          wg_wait<0>();
          __syncwarp();
          if (lane == 0) mbar_arrive(B_EMPTY(s));  // weight stage reusable
          if (++s == p.nb) { s = 0; bph ^= 1; }
        }
        if (lane == 0) mbar_arrive(A_EMPTY(buf));
        if (++buf == p.na) { buf = 0; aph ^= 1; }
      }
      const int tr = p.nco > 1 ? tile % pct : tile;  // tile within its column chunk
      const int b = tr / p.tiles_per_seq;
      const int t0 = (tr - b * p.tiles_per_seq) * TT;
      const int co_base = p.co_off + (p.nco > 1 ? (tile / pct) * p.Cout : 0);
#pragma unroll
      for (int e = 0; e < 64; ++e) {
        const int mb = p.MT == 2 ? (e >> 5) : 0;
        const int i = p.MT == 2 ? (e & 31) : e;
        const int col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        const int t = t0 + (wg * p.MT + mb) * 64 + wq * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
        if (col < p.Cout && t < p.T_out) epi_store(p, acc[e], b, t, col, co_base, bias, bias_s, res, y, y2);
      }
    }
  } else if (warp == W_TMA) {
    // ===================== B producer (TMA bulk copies of packed weight stages) =====================
    const int per_tile = p.nchunks * p.K + p.nchunks2;
    const unsigned char* src = reinterpret_cast<const unsigned char*>(wpk);
    int s = 0, ph = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const unsigned char* srcc = src + (p.nco > 1 ? (size_t)(tile / pct) * per_tile * p.b_bytes : 0);
      for (int j = 0; j < per_tile; ++j) {
        mbar_wait_spin(B_EMPTY(s), ph ^ 1);
        if (elect_one()) {
          mbar_expect_tx(B_FULL(s), (unsigned)p.b_bytes);
          bulk_g2s(smem_u32(b_buf + (size_t)s * p.b_bytes), srcc + (size_t)j * p.b_bytes, (unsigned)p.b_bytes, B_FULL(s));
        }
        __syncwarp();
        if (++s == p.nb) { s = 0; ph ^= 1; }
      }
    }
  } else if (warp == W_LDA) {
    // ===================== raw activation loader (TMA bulk row copies) =====================
    if (p.tma_act) {
      int s = 0, ph = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int tr = p.nco > 1 ? tile % pct : tile;  // tile within its column chunk
      const int b = tr / p.tiles_per_seq;
        const int t0 = (tr - b * p.tiles_per_seq) * TT;
        const int ts0 = (t0 - p.padL) & ~3;
        for (int c = 0; c < nc_total; ++c) {
          mbar_wait(RAW_EMPTY(s), ph ^ 1);
          const float* src;
          int start, end, rowstride, dst_off;
          if (c < p.nchunks) {
            start = ts0 < 0 ? 0 : ts0;
            end = ts0 + p.R4 < p.T_in ? ts0 + p.R4 : p.T_in;
            rowstride = p.T_in;
            dst_off = start - ts0;
            src = x + (long long)b * p.xbs + (long long)(c * KC) * p.T_in + (MC ? (long long)((tile / pct) / p.cpg) * p.xgs : 0);
          } else {
            start = t0;
            end = t0 + TT < p.T_out ? t0 + TT : p.T_out;
            rowstride = p.T_out;
            dst_off = 0;
            src = x2 + ((long long)b * p.C2 + (long long)(c - p.nchunks) * KC) * p.T_out;
          }
          const int nbytes = (end - start) * 4;
          if (nbytes > 0) {
            if (lane == 0) mbar_expect_tx(RAW_FULL(s), (unsigned)nbytes * KC);
            __syncwarp();
            bulk_g2s(smem_u32(raw_buf + (size_t)s * p.raw_bytes) + (unsigned)(lane * p.R4 + dst_off) * 4u,
                     src + (long long)lane * rowstride + start, (unsigned)nbytes, RAW_FULL(s));
          } else if (lane == 0) {
            mbar_arrive(RAW_FULL(s));
          }
          __syncwarp();
          if (++s == p.ns) { s = 0; ph ^= 1; }
        }
      }
    }
  }
}

static int g_tc_variant = 0;

// aux_c2: channels of the auxiliary 1x1 source (0 = none, else multiple of KC); split > 0 selects the
// WaveNet epilogue.  pre_gate: d->cin is the number of gated channels, x holds 2*cin channels.
static int tc_plan(const pwgb_conv1d_desc* d, TcK& p, size_t& smem_bytes, int aux_c2 = 0, int split = 0, int nco_bias = 1) {
  p.variant = g_tc_variant;
  p.co_off = 0;
  p.nco = 1;
  p.cpg = 1;
  p.xgs = 0;
  const int P = d->period < 1 ? 1 : d->period;
  if (d->stride != 1 || d->groups != 1 || P != 1) return 0;
  if (d->cin % KC != 0 || d->cout % 16 != 0 || d->cout < 16 || d->cout > TC_NMAX) return 0;
  if (aux_c2 % KC != 0 || split % 16 != 0 || split > d->cout) return 0;
  if (d->t_valid > 0 && d->t_valid != d->t_in) return 0;
  if (d->x_batch_stride || d->y_batch_stride || d->r_batch_stride) return 0;
  const long long halo = (long long)(d->kernel - 1) * d->dilation;
  p.B = d->batch;
  p.Cin = d->cin;
  p.Cout = d->cout;
  p.T_in = d->t_in;
  p.T_out = d->t_out;
  p.K = d->kernel;
  p.D = d->dilation;
  p.padL = d->pad_left;
  p.pad_mode = d->pad_mode;
  p.pre_slope = d->pre_slope;
  p.pre_gate = d->pre_gate;
  p.post_act = d->post_act;
  p.post_slope = d->post_slope;
  p.out_scale = d->out_scale;
  p.accumulate = d->accumulate;
  p.shuffle = d->shuffle;
  p.shuffle_pad = d->shuffle_pad;
  p.shuffle_tout = d->shuffle_tout;
  p.nchunks = d->cin / KC;
  p.nchunks2 = aux_c2 / KC;
  p.C2 = aux_c2;
  p.wavenet = split > 0;
  p.split = split;
  if (aux_c2 && d->t_in != d->t_out) return 0;
  p.xbs = (long long)d->cin * (d->pre_gate ? 2 : 1) * d->t_in;
  p.ybs = d->shuffle > 1 ? (long long)(d->cout / d->shuffle) * d->shuffle_tout : (long long)d->cout * d->t_out;
  p.rbs = (long long)d->cout * d->t_out;
  p.b_bytes = 2 * (KC / 8) * d->cout * 16;
  // tile shape (1 persistent CTA / SM, ~216 KB of shared memory): prefer a contiguous halo tile of
  // 2 x 128 rows (Cout <= 64: the 64 accumulator registers hold both); fall back to 128 rows, then to
  // one window per tap (very large dilation)
  const size_t budget = 216 * 1024;
  for (int attempt = 0; attempt < 4; ++attempt) {
    if (attempt == 0) {
      p.MT = (d->cout <= TC_NMAX / 2 && d->t_out > 128) ? 2 : 1;
      p.win_mode = 0;
      p.R = p.MT * 128 + (int)halo;
    } else if (attempt == 1) {
      p.MT = 1;
      p.win_mode = 0;
      p.R = 128 + (int)halo;
    } else if (attempt == 2) {
      p.MT = (d->cout <= TC_NMAX / 2 && d->t_out > 128) ? 2 : 1;
      p.win_mode = 1;
      p.R = d->kernel * p.MT * 128;
    } else {
      p.MT = 1;
      p.win_mode = 1;
      p.R = d->kernel * 128;
    }
    if (!p.win_mode && halo > 2048) continue;
    if (p.win_mode && halo <= p.MT * 128) continue;  // a contiguous tile is never larger in that case
    p.a_bytes = 2 * (KC / 8) * p.R * 16;
    p.R4 = (p.R + 6) & ~3;
    p.raw_bytes = KC * p.R4 * 4;
    // activation rows by TMA: zero padding only (out-of-range samples are masked, never copied) and
    // 16-byte aligned rows; anything else is staged with 4-byte cp.async by the producers
    p.tma_act = !(p.variant & 2) && !d->pre_gate && !p.win_mode && d->pad_mode == PWGB_PAD_ZERO && d->t_in % 4 == 0 &&
                (aux_c2 == 0 || d->t_out % 4 == 0);
    // shared-memory split: [na operand buffers][nb weight stages][ns raw staging buffers]
    int na = 0, nb = 0, ns = 0;
    const size_t bias_bytes = 4 * (size_t)(nco_bias > 1 ? nco_bias * d->cout : TC_NMAX);  // bias of every column chunk of the launch
    const size_t A = (size_t)p.a_bytes, Bs = (size_t)p.b_bytes, S = (size_t)p.raw_bytes, slack = 1024 + bias_bytes;
    if (p.tma_act && 2 * A + 3 * S + 3 * Bs + slack <= budget) {
      ns = 3;
      na = 2;
    } else if (!d->pre_gate && 3 * A + 2 * S + 3 * Bs + slack <= budget) {
      ns = 2;
      na = 3;
    } else if (!d->pre_gate && 2 * A + 2 * S + 2 * Bs + slack <= budget) {
      ns = 2;
      na = 2;
    } else if (3 * A + 2 * Bs + slack <= budget) {
      na = 3;
    } else if (2 * A + 2 * Bs + slack <= budget) {
      na = 2;
    } else {
      continue;
    }
    if (ns == 0) p.tma_act = 0;
    nb = (int)((budget - slack - (size_t)na * A - (size_t)ns * S) / Bs);
    if (nb > 24) nb = 24;
    p.na = na;
    p.nb = nb;
    p.ns = ns;
    p.tiles_per_seq = ceil_div(d->t_out, p.MT * 128);
    p.total_tiles = p.tiles_per_seq * d->batch;
    smem_bytes = (size_t)na * p.a_bytes + (size_t)ns * p.raw_bytes + (size_t)nb * p.b_bytes + 8 * (2 * na + 2 * nb + 4 + 2 * NS_MAX) + 16 + bias_bytes;
    return 1;
  }
  return 0;
}

static int tc_launch(TcK& p, size_t bytes, const float* x, const void* packed_w, const float* bias,
                     const float* residual, float* y, cudaStream_t st, const float* x2 = nullptr,
                     float* y2 = nullptr) {
  if (p.B == 0 || p.T_out == 0) return PWGB_OK;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(conv1d_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
    if (e != cudaSuccess) {
      set_error("conv1d_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      return PWGB_CUDA_ERROR;
    }
    attr_set = true;
  }
  static int num_sms = 0;
  if (!num_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (num_sms <= 0) num_sms = 132;
  }
  if ((long long)p.B * p.tiles_per_seq > 0x7fffffffLL) {
    set_error("conv1d_tc: too many tiles");
    return PWGB_UNSUPPORTED;
  }
  if (p.tma_act && ((reinterpret_cast<uintptr_t>(x) & 15) || (x2 && (reinterpret_cast<uintptr_t>(x2) & 15))))
    p.tma_act = 0;  // unaligned base pointer: the producers stage with cp.async instead
  const int grid = p.total_tiles < num_sms ? p.total_tiles : num_sms;
  conv1d_tc_kernel<<<(unsigned)grid, TC_THREADS, bytes, st>>>(p, x, x2, (const uint4*)packed_w, bias, residual, y, y2);
  return check_launch("conv1d_tc_kernel");
}

// Internal entry for N-chunked callers (conv_transpose): runs output channels
// [co_off, co_off + d->cout) of a conv whose full output has cout_total channels.
int conv1d_tc_chunk(const pwgb_conv1d_desc* d, int co_off, int cout_total, const float* x, const void* packed_w,
                    const float* bias, float* y, cudaStream_t st, int nco) {
  TcK p;
  size_t bytes = 0;
  if (!tc_plan(d, p, bytes)) return PWGB_UNSUPPORTED;
  p.co_off = co_off;
  p.ybs = d->shuffle > 1 ? (long long)(cout_total / d->shuffle) * d->shuffle_tout : (long long)cout_total * d->t_out;
  if (nco > 1) {
    // the chunks' packed images are consecutive: one launch walks (chunk, batch, time tile)
    if (d->shuffle <= 1 || (long long)p.total_tiles * nco > 0x7fffffffLL) return PWGB_UNSUPPORTED;
    p.nco = nco;
    p.total_tiles *= nco;
  }
  return tc_launch(p, bytes, x, packed_w, bias, nullptr, y, st);
}

int conv1d_tc_plan_ok(const pwgb_conv1d_desc* d) {
  TcK p;
  size_t bytes;
  return tc_plan(d, p, bytes);
}

void tc_pack_weight(const float* w, int cin, int cout, int kernel, void* packed, cudaStream_t st) {
  tc_pack_rows(w, packed, cin, cin, cout, kernel, 0, cout, st);
}

}  // namespace pwgb

using namespace pwgb;

static int tc_cout_chunk(int cout);

extern "C" void pwgb_debug_set(int key, int value) {
  if (key == 1) g_tc_variant = value;
}

// no debug read-back is available in this build
extern "C" int pwgb_debug_get(int key, void* dst, size_t bytes) {
  (void)key, (void)dst, (void)bytes;
  return -1;
}

extern "C" size_t pwgb_conv1d_tc_packed_weight_bytes(int cin, int cout, int kernel) {
  if (cin <= 0 || cout <= 0 || kernel <= 0 || cin % KC != 0) return 0;
  return (size_t)(cin / KC) * kernel * 2 * (KC / 8) * cout * 16;
}

// w: (cout, cin_g, kernel) with cout = groups * cout_g.  One operand image per (group, column chunk),
// chunk = tc_cout_chunk(cout / groups), laid out consecutively in row order.
extern "C" int pwgb_conv1d_tc_pack_weight_grouped(const float* w, int cin_g, int cout, int kernel, int groups, void* packed,
                                                  void* stream) {
  PWGB_CHECK_ARG(w && packed, "conv1d_tc_pack_weight: null argument");
  PWGB_CHECK_ARG(cin_g > 0 && cin_g % KC == 0 && cout > 0 && kernel > 0 && groups > 0 && cout % groups == 0,
                 "conv1d_tc_pack_weight: channels per group must be a multiple of %d", KC);
  const int chunk = tc_cout_chunk(cout / groups);
  PWGB_CHECK_ARG(chunk > 0, "conv1d_tc_pack_weight: cout / groups must be a multiple of 16");
  // ONE launch packs every (group, column chunk) image: row co of w lands in image co / chunk, column co % chunk
  const long long n = (long long)(cin_g / KC) * kernel * (KC / 8) * cout;
  int blocks = (int)((n + 127) / 128);
  if (blocks > 8192) blocks = 8192;
  if (blocks < 1) blocks = 1;
  tc_pack_weight_kernel<<<blocks, 128, 0, (cudaStream_t)stream>>>(w, (uint4*)packed, cin_g, cin_g, cout, kernel, 0, chunk, chunk);
  return check_launch("tc_pack_weight_kernel");
}

extern "C" int pwgb_conv1d_tc_pack_weight(const float* w, int cin, int cout, int kernel, void* packed, void* stream) {
  return pwgb_conv1d_tc_pack_weight_grouped(w, cin, cout, kernel, 1, packed, stream);
}

// Output channels beyond the TC_NMAX accumulator columns of one launch are processed in column chunks
// (work items of one launch, each re-reading x): chunk = largest multiple of 16 that is <= 128 and divides cout.
static int tc_cout_chunk(int cout) {
  if (cout <= TC_NMAX) return cout;
  for (int c = TC_NMAX; c >= 16; c -= 16)
    if (cout % c == 0) return c;
  return 0;
}

// Grouped convs run one launch per (group, column chunk): a group is an independent dense conv on a
// channel slice (pointer offsets, batch strides of the full tensors).
extern "C" int pwgb_conv1d_tc_supported(const pwgb_conv1d_desc* d) {
  if (!d || d->cout <= 0 || d->groups <= 0 || d->cin % d->groups || d->cout % d->groups) return 0;
  const int G = d->groups;
  if (G > 1 && (d->shuffle > 1 || d->pre_gate || G > 64)) return 0;
  const int chunk = tc_cout_chunk(d->cout / G);
  if (!chunk) return 0;
  if (chunk != d->cout && d->shuffle > 1) return 0;
  pwgb_conv1d_desc c = *d;
  c.cout = chunk;
  c.cin = d->cin / G;
  c.groups = 1;
  TcK p;
  size_t bytes;
  return tc_plan(&c, p, bytes, 0, 0, G * ((d->cout / G) / chunk));
}

extern "C" int pwgb_conv1d_tc_forward(const pwgb_conv1d_desc* d, const float* x, const void* packed_w,
                                      const float* bias, const float* residual, float* y, void* stream) {
  PWGB_CHECK_ARG(d && x && packed_w && y, "conv1d_tc: null argument");
  PWGB_UNSUPPORTED_IF(!pwgb_conv1d_tc_supported(d), "conv1d_tc: configuration not supported by the tensor-core path");
  const int G = d->groups, cin_g = d->cin / G, cout_g = d->cout / G;
  const int chunk = tc_cout_chunk(cout_g);
  pwgb_conv1d_desc c = *d;
  c.cout = chunk;
  c.cin = cin_g;
  c.groups = 1;
  // ONE launch walks every (group, column chunk, batch, time tile) item: the operand images of the chunks are
  // consecutive in `packed_w` (group-major), chunk cc writes output channels [cc * chunk, (cc + 1) * chunk) and reads
  // the input channels of group cc / (cout_g / chunk)
  TcK p;
  size_t bytes = 0;
  const int nco = G * (cout_g / chunk);
  if (!tc_plan(&c, p, bytes, 0, 0, nco)) {
    set_error("conv1d_tc: no tile plan for this configuration");
    return PWGB_UNSUPPORTED;
  }
  if ((long long)p.total_tiles * nco > 0x7fffffffLL) {
    set_error("conv1d_tc: too many tiles");
    return PWGB_UNSUPPORTED;
  }
  p.xbs = (long long)d->cin * (d->pre_gate ? 2 : 1) * d->t_in;
  p.ybs = (long long)d->cout * d->t_out;
  p.rbs = p.ybs;
  if (nco > 1) {
    p.nco = nco;
    p.cpg = cout_g / chunk;
    p.xgs = G > 1 ? (long long)cin_g * d->t_in : 0;
    p.total_tiles *= nco;
  }
  return tc_launch(p, bytes, x, packed_w, bias, residual, y, (cudaStream_t)stream);
}

// ======================================================================================
// WaveNet residual layer (layers/residual_block.py:102-140) as two tensor-core launches:
//   1) g = conv_k,dil(x) + W_aux c + b        (aux 1x1 folded into the same accumulation)
//   2) z = tanh(g[:G/2]) * sigmoid(g[G/2:]) in the producer;  [skip | out] 1x1 stacked as one
//      N = S + R contraction;  epilogue: skips += s,  x' = (o + x) * sqrt(0.5)
// ======================================================================================
static size_t wn_image1_bytes(const pwgb_wavenet_desc* d) {
  return (size_t)(d->residual_channels / KC) * d->kernel * 2 * (KC / 8) * d->gate_channels * 16;
}
static size_t wn_aux_bytes(const pwgb_wavenet_desc* d) {
  return (size_t)(d->aux_channels / KC) * 2 * (KC / 8) * d->gate_channels * 16;
}
static size_t wn_image2_bytes(const pwgb_wavenet_desc* d) {
  return (size_t)((d->gate_channels / 2) / KC) * 2 * (KC / 8) * (d->skip_channels + d->residual_channels) * 16;
}

static void wn_descs(const pwgb_wavenet_desc* d, pwgb_conv1d_desc& c1, pwgb_conv1d_desc& c2) {
  c1 = pwgb_conv1d_desc{};
  c1.batch = d->batch;
  c1.cin = d->residual_channels;
  c1.cout = d->gate_channels;
  c1.t_in = c1.t_out = d->t;
  c1.kernel = d->kernel;
  c1.stride = 1;
  c1.dilation = d->dilation;
  c1.groups = 1;
  c1.pad_left = (d->kernel - 1) / 2 * d->dilation;
  c1.pad_mode = PWGB_PAD_ZERO;
  c1.period = 1;
  c1.t_valid = d->t;
  c1.pre_slope = 1.f;
  c1.out_scale = 1.f;
  c2 = pwgb_conv1d_desc{};
  c2.batch = d->batch;
  c2.cin = d->gate_channels / 2;
  c2.cout = d->skip_channels + d->residual_channels;
  c2.t_in = c2.t_out = d->t;
  c2.kernel = 1;
  c2.stride = 1;
  c2.dilation = 1;
  c2.groups = 1;
  c2.pad_mode = PWGB_PAD_ZERO;
  c2.period = 1;
  c2.t_valid = d->t;
  c2.pre_slope = 1.f;
  c2.pre_gate = 1;
  c2.out_scale = 0.70710678118654752440f;
}

static int wn_valid(const pwgb_wavenet_desc* d) {
  return d && d->batch >= 0 && d->t > 0 && d->kernel > 0 && d->kernel % 2 == 1 && d->dilation > 0 &&
         d->residual_channels > 0 && d->gate_channels > 0 && d->gate_channels % 2 == 0 && d->skip_channels > 0 &&
         d->aux_channels >= 0;
}

extern "C" int pwgb_wavenet_supported(const pwgb_wavenet_desc* d) {
  if (!wn_valid(d)) return 0;
  if (d->residual_channels % KC || (d->gate_channels / 2) % KC || d->aux_channels % KC || d->skip_channels % 16) return 0;
  pwgb_conv1d_desc c1, c2;
  wn_descs(d, c1, c2);
  TcK p;
  size_t bytes;
  return tc_plan(&c1, p, bytes, d->aux_channels, 0) && tc_plan(&c2, p, bytes, 0, d->skip_channels);
}

extern "C" size_t pwgb_wavenet_packed_bytes(const pwgb_wavenet_desc* d) {
  if (!pwgb_wavenet_supported(d)) return 0;
  return wn_image1_bytes(d) + wn_aux_bytes(d) + wn_image2_bytes(d);
}

extern "C" int pwgb_wavenet_pack(const pwgb_wavenet_desc* d, const float* w_conv, const float* w_aux,
                                 int aux_channels_real, const float* w_skip, const float* w_out, void* packed,
                                 void* stream) {
  PWGB_UNSUPPORTED_IF(!pwgb_wavenet_supported(d), "wavenet_pack: configuration not supported by the tensor-core path");
  PWGB_CHECK_ARG(w_conv && w_skip && w_out && packed && (w_aux || d->aux_channels == 0), "wavenet_pack: null argument");
  PWGB_CHECK_ARG(aux_channels_real <= d->aux_channels, "wavenet_pack: aux_channels_real > padded aux_channels");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* img = (unsigned char*)packed;
  const int G = d->gate_channels, H = G / 2, S = d->skip_channels, R = d->residual_channels;
  tc_pack_rows(w_conv, img, R, R, G, d->kernel, 0, G, st);
  int rc = check_launch("tc_pack_weight_kernel");
  if (rc) return rc;
  if (d->aux_channels) {
    tc_pack_rows(w_aux, img + wn_image1_bytes(d), aux_channels_real, d->aux_channels, G, 1, 0, G, st);
    rc = check_launch("tc_pack_weight_kernel");
    if (rc) return rc;
  }
  unsigned char* img2 = img + wn_image1_bytes(d) + wn_aux_bytes(d);
  tc_pack_rows(w_skip, img2, H, H, S, 1, 0, S + R, st);
  rc = check_launch("tc_pack_weight_kernel");
  if (rc) return rc;
  tc_pack_rows(w_out, img2, H, H, R, 1, S, S + R, st);
  return check_launch("tc_pack_weight_kernel");
}

extern "C" int pwgb_wavenet_layer_forward(const pwgb_wavenet_desc* d, const float* x, const float* c,
                                          const void* packed, const float* b_conv, const float* b_skip_out,
                                          float* x_out, float* skips, float* g_ws, void* stream) {
  PWGB_UNSUPPORTED_IF(!pwgb_wavenet_supported(d), "wavenet_layer: configuration not supported by the tensor-core path");
  PWGB_CHECK_ARG(x && packed && x_out && skips && g_ws && (c || d->aux_channels == 0), "wavenet_layer: null argument");
  PWGB_CHECK_ARG(x != x_out, "wavenet_layer: x_out must not alias x (halo reads)");
  cudaStream_t st = (cudaStream_t)stream;
  pwgb_conv1d_desc c1, c2;
  wn_descs(d, c1, c2);
  TcK p;
  size_t bytes = 0;
  tc_plan(&c1, p, bytes, d->aux_channels, 0);
  int rc = tc_launch(p, bytes, x, packed, b_conv, nullptr, g_ws, st, c, nullptr);
  if (rc) return rc;
  tc_plan(&c2, p, bytes, 0, d->skip_channels);
  const unsigned char* img2 = (const unsigned char*)packed + wn_image1_bytes(d) + wn_aux_bytes(d);
  return tc_launch(p, bytes, g_ws, img2, b_skip_out, x, x_out, st, nullptr, skips);
}

// ======================================================================================
// Weight gradient on the tensor cores:  dW[co, ci, k] = sum_{b,t} G[b,co,t] * X~[b,ci,t + k*D - pad]
// is a GEMM whose reduction (MMA K) dimension is TIME.  Both operands are used MN-major: the same
// [channel/8][time row][8 channels] shared-memory tile as the forward activation tile, read with the
// roles of the two axes swapped (wgmma transpose flags), so a tap is again a row offset in the descriptor.
// M = 128 output channels (two warpgroups of 64), N = 32 or 64 input channels, one accumulator block per tap
// (taps x N <= 128 columns: 64 fp32 registers per thread), bf16x3 split, fp32 accumulation over the CTA's
// (batch, time-chunk) items; split partials are reduced deterministically.  The operand images are double
// buffered: the 256 threads convert item n + 1 while the wgmma of item n run.
// ======================================================================================
namespace pwgb {

constexpr int WT_NC = 32;    // input channels per CTA (MMA N); 64 for <= 2 taps (taps x NC <= 128 columns)
constexpr int WT_TK = 128;   // time steps per item (8 MMA k-steps)
constexpr int WT_THREADS = 256;

struct WtK {
  int B, Cin, Cout, T_in, T_out, K, D, padL;
  int G, Cin_g, Cout_g;  // groups: an M tile never straddles two groups (rows beyond the group's channels are zero)
  float x_slope, g_slope;
  int chunks_per_seq, nsplit, RX, ntg, tg;  // tg = taps per CTA, ntg = tap groups
  int nc;                                   // input channels per CTA (32 or 64)
};

// gradient tile (row = time, 8 output channels per 16 B) and activation tile (rows t0 + k0*D - pad ... + RX) of one
// item, converted to the bf16 hi/lo operand images
template <int NC>
__device__ __forceinline__ void wt_fill(const WtK& p, const float* __restrict__ x, const float* __restrict__ gy, int b, int t0,
                                        int co0, int co_end, int grp, int ci0, int k0, bool vec_a, bool vec_b,
                                        unsigned char* a_buf, int a_img, unsigned char* b_buf, int b_img, int tid) {
  const float* gb = gy + ((long long)b * p.Cout + co0) * p.T_out;
  if (vec_a) {
    // a task = (8-channel group, 4 consecutive rows); consecutive lanes take consecutive row quads of one group
    for (int task = tid; task < 16 * (WT_TK / 4); task += WT_THREADS) {
      const int g = task / (WT_TK / 4), rq = task - g * (WT_TK / 4);
      const int t = t0 + 4 * rq;
      const bool cok = t < p.T_out && (co0 + g * 8 < co_end);  // Cout_g % 8 == 0: whole 8-channel groups are in or out
      float4 v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j)
        v[j] = cok ? __ldg(reinterpret_cast<const float4*>(gb + (long long)(g * 8 + j) * p.T_out + t)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int rr = 0; rr < 4; ++rr) {
        float u[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float e = rr == 0 ? v[j].x : (rr == 1 ? v[j].y : (rr == 2 ? v[j].z : v[j].w));
          u[j] = lrelu(e, p.g_slope);
        }
        uint4 hi, lo;
        split8(u, hi, lo);
        const int r = 4 * rq + rr;
        *reinterpret_cast<uint4*>(a_buf + ((size_t)g * WT_TK + r) * 16) = hi;
        *reinterpret_cast<uint4*>(a_buf + a_img + ((size_t)g * WT_TK + r) * 16) = lo;
      }
    }
  } else {
    for (int task = tid; task < 16 * WT_TK; task += WT_THREADS) {
      const int g = task / WT_TK, r = task - g * WT_TK;
      const int t = t0 + r;
      const bool cok = t < p.T_out && (co0 + g * 8 < co_end);
      float u[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) u[j] = cok ? lrelu(__ldg(gb + (long long)(g * 8 + j) * p.T_out + t), p.g_slope) : 0.f;
      uint4 hi, lo;
      split8(u, hi, lo);
      *reinterpret_cast<uint4*>(a_buf + ((size_t)g * WT_TK + r) * 16) = hi;
      *reinterpret_cast<uint4*>(a_buf + a_img + ((size_t)g * WT_TK + r) * 16) = lo;
    }
  }
  const float* xb = x + ((long long)b * p.Cin + grp * p.Cin_g + ci0) * p.T_in;
  const long long ts0 = (long long)t0 + (long long)k0 * p.D - p.padL;
  if (vec_b) {
    for (int task = tid; task < (NC / 8) * (p.RX / 4); task += WT_THREADS) {
      const int g = task / (p.RX / 4), rq = task - g * (p.RX / 4);
      const long long ts = ts0 + 4 * rq;
      const bool ok = ts >= 0 && ts + 3 < p.T_in;  // T_in % 4 == 0 and ts % 4 == 0: a quad is entirely in or out
      float4 v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j)
        v[j] = ok ? __ldg(reinterpret_cast<const float4*>(xb + (long long)(g * 8 + j) * p.T_in + ts)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int rr = 0; rr < 4; ++rr) {
        float u[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float e = rr == 0 ? v[j].x : (rr == 1 ? v[j].y : (rr == 2 ? v[j].z : v[j].w));
          u[j] = lrelu(e, p.x_slope);
        }
        uint4 hi, lo;
        split8(u, hi, lo);
        const int r = 4 * rq + rr;
        *reinterpret_cast<uint4*>(b_buf + ((size_t)g * p.RX + r) * 16) = hi;
        *reinterpret_cast<uint4*>(b_buf + b_img + ((size_t)g * p.RX + r) * 16) = lo;
      }
    }
  } else {
    for (int task = tid; task < (NC / 8) * p.RX; task += WT_THREADS) {
      const int g = task / p.RX, r = task - g * p.RX;
      const long long ts = ts0 + r;
      const bool ok = ts >= 0 && ts < p.T_in;
      float u[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) u[j] = ok ? lrelu(__ldg(xb + (long long)(g * 8 + j) * p.T_in + ts), p.x_slope) : 0.f;
      uint4 hi, lo;
      split8(u, hi, lo);
      *reinterpret_cast<uint4*>(b_buf + ((size_t)g * p.RX + r) * 16) = hi;
      *reinterpret_cast<uint4*>(b_buf + b_img + ((size_t)g * p.RX + r) * 16) = lo;
    }
  }
}

// NC = input channels per CTA (MMA N): 64 halves the number of CTAs that re-read and re-convert the gradient tile
template <int NC>
__global__ void __launch_bounds__(WT_THREADS, 1)
    wgrad_tc_kernel(const WtK p, const float* __restrict__ x, const float* __restrict__ gy, float* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem[];
  // per buffer: A (gradient) image [hi|lo][16 co8][WT_TK rows][16 B];  B (activation) image [hi|lo][NC/8 ci8][RX rows][16 B]
  const int a_img = 16 * WT_TK * 16;
  const int b_img = (NC / 8) * p.RX * 16;
  const int buf_bytes = 2 * a_img + 2 * b_img;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2, wq = warp & 3;
  const int tpg = (p.Cout_g + 127) / 128;  // M tiles per group
  const int grp = blockIdx.x / tpg;
  const int co0 = grp * p.Cout_g + (blockIdx.x - grp * tpg) * 128;
  const int co_end = (grp + 1) * p.Cout_g;
  const int ci0 = (blockIdx.y / p.ntg) * NC;  // within the group
  const int k0 = (blockIdx.y % p.ntg) * p.tg;
  const int ntap = min(p.tg, p.K - k0);
  const int split = blockIdx.z;
  const int total_items = p.B * p.chunks_per_seq;
  // 16-byte loads need 16-byte aligned rows: row pitch and window offset multiples of 4 samples
  const bool vec_a = p.T_out % 4 == 0 && (reinterpret_cast<uintptr_t>(gy) & 15) == 0;
  const bool vec_b = p.T_in % 4 == 0 && p.RX % 4 == 0 && ((long long)k0 * p.D - p.padL) % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
  constexpr int TGMAX = 128 / NC;  // accumulator blocks of NC columns
  float acc[64];
#pragma unroll
  for (int e = 0; e < 64; ++e) acc[e] = 0.f;
  // MN-major no-swizzle: LBO = next 8 time rows (128 B), SBO = next 8 channels (rows * 16 B)
  const unsigned a_sbo = WT_TK * 16, b_sbo = (unsigned)p.RX * 16;
  int buf = 0;
  if (split < total_items) {
    const int b = split / p.chunks_per_seq;
    wt_fill<NC>(p, x, gy, b, (split - b * p.chunks_per_seq) * WT_TK, co0, co_end, grp, ci0, k0, vec_a, vec_b, smem, a_img,
                smem + 2 * a_img, b_img, tid);
  }
  fence_proxy_async();
  __syncthreads();
  for (int item = split; item < total_items; item += p.nsplit) {
    unsigned char* a_buf = smem + (size_t)buf * buf_bytes;
    const unsigned a_addr = smem_u32(a_buf) + (unsigned)(wg * 8) * a_sbo;  // this warpgroup's 64 output channels
    const unsigned b_addr = smem_u32(a_buf + 2 * a_img);
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < WT_TK / 16; ++ks) {
      const unsigned long long ah = gmma_desc(a_addr + (unsigned)(ks * 16 * 16), 128, a_sbo);
      const unsigned long long al = ah + (unsigned)(a_img >> 4);
#pragma unroll
      for (int tp = 0; tp < TGMAX; ++tp) {
        if (tp < ntap) {
          const unsigned long long bh = gmma_desc(b_addr + (unsigned)((tp * p.D + ks * 16) * 16), 128, b_sbo);
          const unsigned long long bl = bh + (unsigned)(b_img >> 4);
          float* d = acc + tp * (NC / 2);
          Wgmma<NC, 1, 1>::run(d, ah, bh);
          Wgmma<NC, 1, 1>::run(d, al, bh);
          Wgmma<NC, 1, 1>::run(d, ah, bl);
        }
      }
    }
    wg_commit();
    // convert the next item into the other buffer while the MMAs run
    const int next = item + p.nsplit;
    if (next < total_items) {
      unsigned char* nb = smem + (size_t)(buf ^ 1) * buf_bytes;
      const int b = next / p.chunks_per_seq;
      wt_fill<NC>(p, x, gy, b, (next - b * p.chunks_per_seq) * WT_TK, co0, co_end, grp, ci0, k0, vec_a, vec_b, nb, a_img,
                  nb + 2 * a_img, b_img, tid);
      fence_proxy_async();
    }
    wg_wait<0>();
    __syncthreads();
    buf ^= 1;
  }
  // ---- epilogue: row = output channel, column = tap * NC + ci
#pragma unroll
  for (int e = 0; e < 64; ++e) {
    const int tp = e / (NC / 2), i = e % (NC / 2);
    const int n = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
    const int co = co0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
    if (tp < ntap && co < co_end)
      part[(((long long)split * p.Cout + co) * p.Cin_g + ci0 + n) * p.K + k0 + tp] = acc[e];
  }
}

__global__ void wt_reduce_kernel(const float* __restrict__ part, float* __restrict__ out, long long n, int nsplit) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float a = 0.f;
    for (int s = 0; s < nsplit; ++s) a += part[(long long)s * n + i];
    out[i] = a;
  }
}

static int wt_plan(const pwgb_conv1d_desc* d, WtK& p) {
  if (!d || d->stride != 1 || d->groups < 1 || (d->period > 1) || d->pre_gate || d->pad_mode != PWGB_PAD_ZERO) return 0;
  if (d->cin % d->groups || d->cout % d->groups) return 0;
  const int cin_g = d->cin / d->groups, cout_g = d->cout / d->groups;
  if (cout_g % 8 != 0 || cout_g < 32 || cin_g % WT_NC != 0 || d->kernel <= 0 || d->dilation <= 0) return 0;
  if (d->t_valid > 0 && d->t_valid != d->t_in) return 0;
  p.B = d->batch;
  p.Cin = d->cin;
  p.Cout = d->cout;
  p.T_in = d->t_in;
  p.T_out = d->t_out;
  p.K = d->kernel;
  p.D = d->dilation;
  p.padL = d->pad_left;
  p.G = d->groups;
  p.Cin_g = cin_g;
  p.Cout_g = cout_g;
  p.x_slope = d->pre_slope;
  p.g_slope = 1.f;
  p.chunks_per_seq = ceil_div(d->t_out, WT_TK);
  // 64 input channels per CTA when the taps fit the accumulator (taps x 64 <= 128 columns): the (dominant)
  // gradient tile is then read and converted once per 64 instead of once per 32 input channels
  p.nc = (cin_g % 64 == 0 && d->kernel <= 2) ? 64 : WT_NC;
  // taps per CTA: as many as fit (the activation window grows with (taps - 1) * dilation)
  const int tg_max = 128 / p.nc;
  int tg = d->kernel < tg_max ? d->kernel : tg_max;
  for (;; tg = (tg + 1) / 2) {
    p.RX = WT_TK + (tg - 1) * d->dilation;
    if (2 * ((size_t)2 * 16 * WT_TK * 16 + (size_t)2 * (p.nc / 8) * p.RX * 16) <= 220 * 1024) break;
    if (tg == 1) return 0;
  }
  p.tg = tg;
  p.ntg = ceil_div(d->kernel, tg);
  const long long items = (long long)p.B * p.chunks_per_seq;
  const long long gxy = (long long)d->groups * ceil_div(cout_g, 128) * (cin_g / p.nc) * p.ntg;
  // enough (tile, split) CTAs for two waves over 132 SMs; a split keeps at least 8 items (1024 time steps) of work
  long long ns = (2 * 132 + gxy - 1) / gxy;
  if (ns > items / 8) ns = items / 8;
  if (ns > 512) ns = 512;
  if (ns < 1) ns = 1;
  p.nsplit = (int)ns;
  return 1;
}

}  // namespace pwgb

extern "C" int pwgb_conv1d_wgrad_tc_supported(const pwgb_conv1d_desc* d) {
  pwgb::WtK p;
  return pwgb::wt_plan(d, p);
}

extern "C" size_t pwgb_conv1d_wgrad_tc_workspace(const pwgb_conv1d_desc* d) {
  pwgb::WtK p;
  if (!pwgb::wt_plan(d, p)) return 0;
  return (size_t)p.nsplit * d->cout * (d->cin / d->groups) * d->kernel * sizeof(float);
}

extern "C" int pwgb_conv1d_wgrad_tc(const pwgb_conv1d_desc* d, const float* x, const float* gy, float g_slope, float* dw,
                                    void* ws, size_t ws_bytes, void* stream) {
  using namespace pwgb;
  PWGB_CHECK_ARG(d && x && gy && dw && ws, "conv1d_wgrad_tc: null argument");
  WtK p;
  PWGB_UNSUPPORTED_IF(!wt_plan(d, p), "conv1d_wgrad_tc: configuration not supported by the tensor-core path");
  p.g_slope = g_slope;
  const size_t need = pwgb_conv1d_wgrad_tc_workspace(d);
  PWGB_CHECK_ARG(ws_bytes >= need, "conv1d_wgrad_tc: workspace too small (%zu < %zu)", ws_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)d->cout * (d->cin / d->groups) * d->kernel;
  if (p.B == 0 || p.T_out == 0) {
    cudaMemsetAsync(dw, 0, n * sizeof(float), st);
    return PWGB_OK;
  }
  const size_t smem = 2 * ((size_t)2 * 16 * WT_TK * 16 + (size_t)2 * (p.nc / 8) * p.RX * 16);
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(wgrad_tc_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(wgrad_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
    if (e != cudaSuccess) {
      set_error("conv1d_wgrad_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      return PWGB_CUDA_ERROR;
    }
    attr_set = true;
  }
  dim3 grid(p.G * ceil_div(p.Cout_g, 128), (p.Cin_g / p.nc) * p.ntg, p.nsplit);
  if (p.nc == 64)
    wgrad_tc_kernel<64><<<grid, WT_THREADS, smem, st>>>(p, x, gy, (float*)ws);
  else
    wgrad_tc_kernel<32><<<grid, WT_THREADS, smem, st>>>(p, x, gy, (float*)ws);
  int rc = check_launch("wgrad_tc_kernel");
  if (rc) return rc;
  int blocks = (int)((n + 255) / 256);
  if (blocks > 4096) blocks = 4096;
  wt_reduce_kernel<<<blocks, 256, 0, st>>>((const float*)ws, dw, n, p.nsplit);
  return check_launch("wt_reduce_kernel");
}
