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
//               and stores.  A plain conv with a residual or an accumulate does that in a shared-memory tile: its
//               residual rows arrive by bulk copy while the MMAs run, its rows leave by bulk store (or bulk fp32 add).
//   warp 16     B producer: cp.async.bulk (TMA, 1-D) of one packed weight stage per (chunk, tap).
//   warp 17     raw activation loader: cp.async.bulk row copies into the raw fp32 ring.
#include <cstring>
#include <type_traits>

#include "tc_common.cuh"
#include "tma.cuh"

namespace pwgb {

constexpr int NPROD = 256;  // producer threads (warps 0-7); 4 warps measured slower (conversion-bound)
constexpr int NCONS = 256;  // consumer threads (warps 8-15: two warpgroups)
// warp roles after the producers / consumers: weight TMA, activation TMA
constexpr int W_CONS0 = NPROD / 32, W_TMA = (NPROD + NCONS) / 32, W_LDA = W_TMA + 1;
constexpr int TC_THREADS = NPROD + NCONS + 64;
constexpr int NS_MAX = 4;  // raw activation stages
constexpr size_t TC_SMEM_STAGED = 227 * 1024;  // H100 opt-in limit of dynamic shared memory per block: staged-epilogue plans
// named barrier 1 of the NPROD producer threads (ids 2 and 3 are the consumer warpgroups', wg_barrier)
__device__ __forceinline__ void producer_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(NPROD) : "memory"); }

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
  int nchunks2, C2;      // channels of x2: the auxiliary 1x1 source (WaveNet conditioning) of nchunks2 extra K=1 chunks, or,
                         // with nchunks2 == 0, the last C2 of the Cin main input channels (two-source input; 0: x holds all)
  int pre_gate;          // producer computes tanh(x[c]) * sigmoid(x[c + Cin])
  int wavenet;           // epilogue: cols < split -> y2 += v ; cols >= split -> y = (v + res) * scale
  int split;
  int co_off;            // first output channel of this launch (N-chunked callers)
  int variant;           // debug (pwgb_debug_set(1, v)): bit 1 stages activations with cp.async instead of TMA,
                         // bit 2 keeps the register epilogue, bit 8 runs the 128- and 256-channel ResBlock pairs as
                         // two fp32 launches (rb_packed_plan declines)
  int staged;            // plain epilogue through a shared-memory tile per consumer warpgroup (tc_plan)
  // packed ResBlock intermediate (pk_plane, tc_common.cuh): pk_out, the epilogue writes lrelu(acc + bias, pk_slope) there
  // as bf16 hi/lo (y: the packed image); pk_in, warp W_LDA lands each chunk's operand image from it with one tensor copy
  // (tm_a) and the producers have no work
  int pk_in, pk_out;
  float pk_slope;
  // history launches (conv1d_tc_hist_kernel, pad_mode PWGB_PAD_HISTORY): input rows [-hist_len, 0) come from hist
  // (B, Cin, hist_len), or from sample 0 of x for an item whose rep flag is set
  const float* hist;
  const int* rep;
  int hist_len;
};

// The parameters of an EXT history launch (conv1d_tc_ext_kernel, pwgb_stream_ext; register epilogue only): the mask
// (output row t, or the shuffled row, is signal sample mframe[b] * mrate - mlook + t; outside the signal it stores +0.0)
// and the delayed residual (row t adds row t - rdelay of [rhist | res], rhist (B, total cout, rhist_len)).  A separate
// struct, so that the kernels without EXT keep their parameters and code.
struct TcKExt : TcK {
  const int* mframe;
  const int* mend;
  int mrate, mlook;
  const float* rhist;
  int rhist_len, rdelay;
  long long rhbs;
};

// The edge policy of an EDGE history launch (conv1d_tc_edge_kernel, pwgb_stream_ext.edge != 0): input row r is signal
// sample mframe[b] * mrate - in_look + r, and a row outside [0, mend[b] * mrate) reads the row of [hist | x] holding the
// reflected (edge PWGB_PAD_REFLECT) or replicated (PWGB_PAD_REPLICATE) sample.
struct TcKEdge : TcKExt {
  int edge, in_look;
};

template <bool EXT, bool EDGE>
using TcKOf = std::conditional_t<EDGE, TcKEdge, std::conditional_t<EXT, TcKExt, TcK>>;

// Staged epilogue: one tile (fp32 [col][stage_ld(MT)], tc_common.cuh) per consumer warpgroup.  Tile shapes compiled with
// it: at MT = 2 and more than 32 columns it made ptxas spill, and its tiles would not fit beside the pipeline there anyway.
__host__ __device__ constexpr bool stage_shape(int mt, int cout) { return mt == 1 || cout <= 32; }

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

// Epilogue of one accumulator element (row t, column col of the launch's column chunk starting at co_base).  The mode
// (EPI_SHUFFLE: p.shuffle > 1, EPI_WAVENET: p.wavenet, else EPI_PLAIN) is a template argument so the consumers branch on
// it once per 64-row block, not per element.
enum { EPI_PLAIN, EPI_SHUFFLE, EPI_WAVENET };
template <int MODE, bool EXT, class P>
__device__ __forceinline__ void epi_store(const P& p, float a, int b, int t, int col, int co_base, const float* __restrict__ bias,
                                          const float* bias_s, const float* __restrict__ res, float* __restrict__ y,
                                          float* __restrict__ y2) {
  const long long st = p.T_out;
  if constexpr (MODE == EPI_SHUFFLE) {
    const int co = co_base + col, cof = co / p.shuffle;
    float v = a + (bias ? __ldg(bias + cof) : 0.f);
    if (p.post_act == PWGB_ACT_TANH)
      v = tanhf(v);
    else if (p.post_act == PWGB_ACT_LRELU)
      v = lrelu(v, p.post_slope);
    const int of = t * p.shuffle + (co - cof * p.shuffle) - p.shuffle_pad;
    if constexpr (EXT) {
      if (of >= 0 && of < p.shuffle_tout) {
        v *= p.out_scale;
        if (p.mframe && stream_outside(p.mframe, p.mend, p.mrate, p.mlook, b, of)) v = 0.f;
        y[(long long)b * p.ybs + (long long)cof * p.shuffle_tout + of] = v;
      }
      return;
    }
    if (of >= 0 && of < p.shuffle_tout) y[(long long)b * p.ybs + (long long)cof * p.shuffle_tout + of] = v * p.out_scale;
  } else if constexpr (MODE == EPI_WAVENET) {
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
    if constexpr (EXT) {
      if (res) {
        const int ro = t - p.rdelay;
        v += ro >= 0 ? __ldg(res + (long long)b * p.rbs + off - p.rdelay)
                     : __ldg(p.rhist + (long long)b * p.rhbs + (long long)(co_base + col) * p.rhist_len + (p.rhist_len + ro));
      }
    } else {
      if (res) v += __ldg(res + (long long)b * p.rbs + off);
    }
    // the scale and the accumulate round separately (never one fma), as the staged epilogue's bulk fp32 add does
    v = __fmul_rn(v, p.out_scale);
    float* q = y + (long long)b * p.ybs + off;
    if (p.accumulate) v = __fadd_rn(v, *q);
    if constexpr (EXT) {
      if (p.mframe && stream_outside(p.mframe, p.mend, p.mrate, p.mlook, b, t)) v = 0.f;
    }
    *q = v;
  }
}

// ------------------------------------------------------------------ main kernel
// Persistent: one CTA per SM loops over (batch, time-tile) work items; every role runs the same
// tile sequence and talks through mbarriers only, so the loads of tile i+1 overlap the MMAs and the
// epilogue of tile i.

// First sample of main chunk c (input channels c*KC .. c*KC + KC) of batch item b.  A two-source conv (nchunks2 == 0,
// C2 > 0) reads channels [0, Cin - C2) from x (B, Cin - C2, T_in) and [Cin - C2, Cin) from x2 (B, C2, T_in): the input
// is cat(x, x2) without the copy.  KC divides C2, so a chunk never straddles the two.  goff: group offset.
__device__ __forceinline__ const float* main_src(const TcK& p, const float* x, const float* x2, int b, int c, long long goff) {
  const int ch = c * KC, c1 = p.Cin - p.C2;
  if (p.nchunks2 == 0 && ch >= c1) return x2 + ((long long)b * p.C2 + (ch - c1)) * p.T_in;
  return x + (long long)b * p.xbs + (long long)ch * p.T_in + goff;
}

// Batch item and first time step of work item `tile` (TT time steps per tile; the items of the nco column chunks of a
// launch follow one another).
__device__ __forceinline__ void tile_origin(const TcK& p, int tile, int TT, int& b, int& t0) {
  const int tr = p.nco > 1 ? tile % (p.B * p.tiles_per_seq) : tile;  // tile within its column chunk
  b = tr / p.tiles_per_seq;
  t0 = (tr - b * p.tiles_per_seq) * TT;
}

// Input sample of operand row r of a main chunk in the tile starting at t0: the row's window and tap (win_mode) or its
// place in the contiguous halo tile, then the padding policy.  ok = false: a zero-padding row.
__device__ __forceinline__ long long tile_sample(const TcK& p, int t0, int TT, int r) {
  if (p.win_mode) {
    const int k = r / TT;
    return (long long)t0 - p.padL + (long long)k * p.D + (r - k * TT);
  }
  return (long long)t0 - p.padL + r;
}

__device__ __forceinline__ long long src_sample(const TcK& p, int t0, int TT, int r, bool& ok) {
  long long ts = tile_sample(p, t0, TT, r);
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
}

// The history padding policy (one more policy of src_sample, for history launches): the source of operand row r of main
// chunk c of batch item b.  Rows [-hist_len, 0) read hist[b, c * KC + j, hist_len + ts], or x[b, c * KC + j, 0] when the
// item's rep flag is set (x[b, c * KC + j, -ts] under PWGB_PAD_HISTORY_REFLECT); rows before -hist_len and from T_in on
// are zero padding (ok = false).  Returns channel j = 0's sample; ld: the channel stride.
__device__ __forceinline__ const float* hist_sample(const TcK& p, const float* xc, int b, int c, int t0, int TT, int r, bool& ok,
                                                    long long& ld) {
  const long long ts = tile_sample(p, t0, TT, r);
  ld = p.T_in;
  ok = ts >= -p.hist_len && ts < p.T_in;
  if (!ok) return xc;
  if (ts >= 0) return xc + ts;
  if (p.rep && p.rep[b]) return p.pad_mode == PWGB_PAD_HISTORY_REFLECT ? xc - ts : xc;
  ld = p.hist_len;
  return p.hist + ((long long)b * p.Cin + (long long)c * KC) * p.hist_len + (p.hist_len + ts);
}

// hist_sample under the edge policy of TcKEdge: the row is first moved to the one holding its reflected or replicated
// sample, which is then read like any row of [hist | x] (zero outside [-hist_len, T_in))
__device__ __forceinline__ const float* hist_sample_edge(const TcKEdge& p, const float* xc, int b, int c, int t0, int TT, int r,
                                                         bool& ok, long long& ld) {
  long long ts = tile_sample(p, t0, TT, r);
  if (p.edge) {
    const long long u = (long long)__ldg(p.mframe + b) * p.mrate - p.in_look + ts;
    const long long L = (long long)__ldg(p.mend + b) * p.mrate;
    if (u < 0 || u >= L) ts += (p.edge == PWGB_PAD_REFLECT ? (u < 0 ? -u : 2 * (L - 1) - u) : (u < 0 ? 0 : L - 1)) - u;
  }
  ld = p.T_in;
  ok = ts >= -p.hist_len && ts < p.T_in;
  if (!ok) return xc;
  if (ts >= 0) return xc + ts;
  if (p.rep && p.rep[b]) return p.pad_mode == PWGB_PAD_HISTORY_REFLECT ? xc - ts : xc;
  ld = p.hist_len;
  return p.hist + ((long long)b * p.Cin + (long long)c * KC) * p.hist_len + (p.hist_len + ts);
}

// stage one activation chunk (KC channels x R rows) into the operand layout; HIST: with the history padding policy
// (chunk c of batch item b); EDGE: with the edge policy as well
template <bool HIST, bool EDGE = false>
__device__ __forceinline__ void fill_main_chunk(const std::conditional_t<EDGE, TcKEdge, TcK>& p, const float* __restrict__ xc,
                                                int t0, int TT, unsigned char* dst, int tid, int b, int c) {
  auto store_row = [&](const float (&v)[KC], int r) {
#pragma unroll
    for (int g = 0; g < KC / 8; ++g) {
      float u[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) u[j] = v[g * 8 + j];
      store_split8(dst, p.R, r, g, u);
    }
  };
  if (!HIST && p.pre_gate) {
    const float* xg = xc + (long long)p.Cin * p.T_in;
    for (int r = tid; r < p.R; r += NPROD) {
      bool ok;
      const long long ts = src_sample(p, t0, TT, r, ok);
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
    float v[KC];
    if constexpr (HIST) {
      long long ld;
      const float* s;
      if constexpr (EDGE)
        s = hist_sample_edge(p, xc, b, c, t0, TT, r, ok, ld);
      else
        s = hist_sample(p, xc, b, c, t0, TT, r, ok, ld);
#pragma unroll
      for (int j = 0; j < KC; ++j) v[j] = ok ? __ldg(s + (long long)j * ld) : 0.f;
    } else {
      const long long ts = src_sample(p, t0, TT, r, ok);
#pragma unroll
      for (int j = 0; j < KC; ++j) v[j] = ok ? __ldg(xc + (long long)j * p.T_in + ts) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < KC; ++j) v[j] = lrelu(v[j], p.pre_slope);
    store_row(v, r);
  }
}

// MT (64-row blocks per warpgroup) and NB16 (16-column blocks, Cout = 16 * NB16) are compile-time constants, so the
// consumers issue a fixed wgmma sequence into fixed accumulator registers (tc_launch picks the instantiation).  HIST: the
// history padding policy on the element-addressed producers (cp.async-staged and direct; history launches never take
// the TMA activation path).  EXT (with HIST only): the mask and the delayed residual of a pwgb_stream_ext launch in the
// register epilogue, with the parameters of TcKExt.  EDGE (with EXT): the edge policy of TcKEdge in the history
// producers' row addressing.  They are template arguments so that the kernels without them keep their code.
template <int MT, int NB16, bool HIST, bool EXT = false, bool EDGE = false>
__device__ __forceinline__ void conv1d_tc_body(const TcKOf<EXT, EDGE>& p, const float* __restrict__ x, const float* __restrict__ x2,
                                               const uint4* __restrict__ wpk, const float* __restrict__ bias,
                                               const float* __restrict__ res, float* __restrict__ y, float* __restrict__ y2,
                                               const CUtensorMap* tm_a) {
  extern __shared__ __align__(128) unsigned char smem[];
  // layout: A[na] | B[nb] | raw staging[ns] | epilogue tiles[2 if staged] | barriers | bias
  constexpr int SLD = stage_ld(MT);
  const bool staged = stage_shape(MT, NB16 * 16) && p.staged;
  unsigned char* a_buf = smem;
  unsigned char* b_buf = smem + (size_t)p.na * p.a_bytes;
  unsigned char* raw_buf = b_buf + (size_t)p.nb * p.b_bytes;
  float* stage_buf = reinterpret_cast<float*>(raw_buf + (size_t)p.ns * p.raw_bytes);
  unsigned long long* bars = reinterpret_cast<unsigned long long*>(stage_buf + (staged ? 2 * p.Cout * SLD : 0));
  const int nbar = 2 * p.na + 2 * p.nb + 4 + 2 * NS_MAX + 2;
  float* bias_s = reinterpret_cast<float*>(bars + nbar + 2);  // Cout floats (0 when bias == nullptr)
  // several column chunks / groups of a plain (non pixel-shuffle) conv share the launch
  const bool MC = p.nco > 1 && p.shuffle <= 1;

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  constexpr int TT = MT * 128;
  const int nc_total = p.nchunks + p.nchunks2;
  const int pct = p.B * p.tiles_per_seq;  // work items per column chunk (nco chunks share one launch)

  const unsigned bar0 = smem_u32(bars);
  auto A_FULL = [&](int i) { return bar0 + 8u * i; };
  auto A_EMPTY = [&](int i) { return bar0 + 8u * (p.na + i); };
  auto B_FULL = [&](int i) { return bar0 + 8u * (2 * p.na + i); };
  auto B_EMPTY = [&](int i) { return bar0 + 8u * (2 * p.na + p.nb + i); };
  auto RAW_FULL = [&](int i) { return bar0 + 8u * (2 * p.na + 2 * p.nb + 4 + i); };
  auto RAW_EMPTY = [&](int i) { return bar0 + 8u * (2 * p.na + 2 * p.nb + 4 + NS_MAX + i); };
  auto RES_FULL = [&](int wg) { return bar0 + 8u * (2 * p.na + 2 * p.nb + 4 + 2 * NS_MAX + wg); };  // staged residual

  if (tid == 0) {
    for (int i = 0; i < p.na; ++i) {
      mbar_init(A_FULL(i), !HIST && p.pk_in ? 1 : NPROD);
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
    // one arrival per channel row: each issuing thread of the warpgroup arrives with its row's byte count
    for (int i = 0; i < 2; ++i) mbar_init(RES_FULL(i), p.Cout);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = tid; i < p.Cout * (MC ? p.nco : 1); i += TC_THREADS)
    bias_s[i] = bias ? __ldg(bias + (p.shuffle > 1 ? (p.co_off + i) / p.shuffle : p.co_off + i)) : 0.f;
  __syncthreads();

  if (warp < W_CONS0 && !HIST && p.pk_in) {
    // packed activations: warp W_LDA lands the operand images, nothing to convert
  } else if (warp < W_CONS0 && !HIST && p.tma_act) {
    // ===================== A producers, TMA-staged =====================
    // Warp W_LDA streams the raw fp32 rows of chunk q + ns - 1 into shared memory with bulk copies
    // (no LSU instructions, no registers); these 8 warps only convert landed stages to the bf16 hi/lo
    // operand image.  Stages start at a 16-byte aligned sample, `shift` re-aligns the rows; samples
    // outside [0, T) are never copied and are masked here (zero padding).
    int s = 0, sph = 0, buf = 0, aph = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      // tile_origin written out: through the helper here, ptxas spilled conv1d_tc_kernel<2, 4> at its 96 registers
      const int tr = p.nco > 1 ? tile % pct : tile;
      const int b = tr / p.tiles_per_seq;
      const int t0 = (tr - b * p.tiles_per_seq) * TT;
      const int ts_first = t0 - p.padL;
      const int shift = ts_first - (ts_first & ~3);
      for (int c = 0; c < nc_total; ++c) {
        mbar_wait(RAW_FULL(s), sph);
        mbar_wait(A_EMPTY(buf), aph ^ 1);
        const float* raw = reinterpret_cast<const float*>(raw_buf + (size_t)s * p.raw_bytes);
        const bool main_chunk = c < p.nchunks;
        convert_raw_stage<NPROD, true>(a_buf + (size_t)buf * p.a_bytes, p.R, raw, main_chunk ? shift : 0, p.R4,
                                       main_chunk ? p.R : TT, main_chunk ? ts_first : t0,
                                       (unsigned)(main_chunk ? p.T_in : p.T_out), main_chunk ? p.pre_slope : 1.f, tid);
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
      int b, t0;
      tile_origin(p, tile, TT, b, t0);
      const unsigned raw = smem_u32(raw_buf + (size_t)(q % p.ns) * p.raw_bytes);
      if (c < p.nchunks) {
        const float* xc = main_src(p, x, x2, b, c, MC ? (long long)((tile / pct) / p.cpg) * p.xgs : 0);
        for (int r = tid; r < p.R; r += NPROD) {
          bool ok;
          if constexpr (HIST) {
            long long ld;
            const float* src;
            if constexpr (EDGE)
              src = hist_sample_edge(p, xc, b, c, t0, TT, r, ok, ld);
            else
              src = hist_sample(p, xc, b, c, t0, TT, r, ok, ld);
            const unsigned nbytes = ok ? 4u : 0u;
            unsigned dq = raw + (unsigned)r * 4u;
            const unsigned dstep = (unsigned)p.R * 4u;
#pragma unroll 8
            for (int j = 0; j < KC; ++j, src += ld, dq += dstep) cp_async4(dq, src, nbytes);
          } else {
            const long long ts = src_sample(p, t0, TT, r, ok);
            const float* src = ok ? xc + ts : xc;
            const unsigned nbytes = ok ? 4u : 0u;
            unsigned dq = raw + (unsigned)r * 4u;
            const unsigned dstep = (unsigned)p.R * 4u;
#pragma unroll 8
            for (int j = 0; j < KC; ++j, src += p.T_in, dq += dstep) cp_async4(dq, src, nbytes);
          }
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
      const float* raw = reinterpret_cast<const float*>(raw_buf + (size_t)(q % p.ns) * p.raw_bytes);
      // the padding is in the stage (cp.async zero fill, reflected / replicated samples)
      convert_raw_stage<NPROD, false>(a_buf + (size_t)buf * p.a_bytes, p.R, raw, 0, p.R, c < p.nchunks ? p.R : TT, 0, 0u,
                                      c < p.nchunks ? p.pre_slope : 1.f, tid);
      fence_proxy_async();
      mbar_arrive(A_FULL(buf));
      producer_barrier();  // raw[q % ns] may be overwritten by issue(q + 2)
    }
  } else if (warp < W_CONS0) {
    // ===================== A producers, direct register path =====================
    // (one source only: conv1d_tc_chunk gives two-source inputs raw-staged plans)
    unsigned ca = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      int b, t0;
      tile_origin(p, tile, TT, b, t0);
      const float* xb = x + (long long)b * p.xbs + (MC ? (long long)((tile / pct) / p.cpg) * p.xgs : 0);
      for (int c = 0; c < nc_total; ++c, ++ca) {
        const int buf = ca % p.na;
        mbar_wait(A_EMPTY(buf), ((ca / p.na) & 1) ^ 1);
        unsigned char* dst = a_buf + (size_t)buf * p.a_bytes;
        if (c < p.nchunks) {
          fill_main_chunk<HIST, EDGE>(p, xb + (long long)(c * KC) * p.T_in, t0, TT, dst, tid, b, c);
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
              store_split8(dst, p.R, r, g, u);
            }
          }
        }
        fence_proxy_async();  // generic-proxy smem writes -> visible to the tensor core (async proxy)
        mbar_arrive(A_FULL(buf));
      }
    }
  } else if (warp < W_TMA) {
    // ===================== consumers: wgmma into registers, then the epilogue =====================
    // warpgroup wg owns the 64-row blocks wg * MT + mb of the tile.  One wgmma group per (chunk, tap): the three bf16x3
    // products of every block and 16-channel K-step.  A group stays in flight while the next one is issued; the wait that
    // retires it hands its weight stage (and, after a chunk's last tap, its A buffer) back to the producers.  The order
    // of the MMAs into each accumulator is the issue order, so the overlap does not change the result.
    const int wg = (warp - W_CONS0) >> 2, wq = warp & 3;
    constexpr int NACC = 8 * NB16;  // fp32 accumulators per thread and 64-row block
    const unsigned lbo_a = (unsigned)p.R * 16u, a_sub = (unsigned)(KC / 8) * p.R;  // a_sub: hi -> lo image (16-byte units)
    // Staged epilogue: thread wt of the warpgroup owns channel row wt of the warpgroup's tile.  It issues that row's
    // residual load and its store (or add), so its own bulk-group wait is the only guard the row needs before reuse.
    const int wt = tid - NPROD - wg * 128;
    float* stg = stage_buf + (size_t)wg * p.Cout * SLD;
    const bool row_owner = staged && wt < p.Cout;
    int buf = 0, aph = 0, s = 0, bph = 0;
    // (batch, first time step, first channel) of a tile
    auto tile_pos = [&](int tile, int& b, int& t0, int& co_base) {
      tile_origin(p, tile, TT, b, t0);
      co_base = p.co_off + (p.nco > 1 ? (tile / pct) * p.Cout : 0);
    };
    // channel row wt of this warpgroup's rows [tw0, tw0 + MT * 64) of a tile: its first element within the batch item
    // (y / residual layout) and its bytes below T_out
    auto row_pos = [&](int t0, int co_base, unsigned& row_bytes) -> long long {
      const int tw0 = t0 + wg * MT * 64;
      const int nrow = p.T_out - tw0 < MT * 64 ? p.T_out - tw0 : MT * 64;
      row_bytes = nrow > 0 ? 4u * (unsigned)nrow : 0u;
      return (long long)(co_base + wt) * p.T_out + tw0;
    };
    // Residual row of a tile, issued before the tile's MMAs (at the end of the previous tile's epilogue, once its store
    // has read the row), so that it streams in while they run.  Nothing of it is live across the MMA loop.
    auto load_res = [&](int tile) {
      int b, t0, co_base;
      unsigned row_bytes;
      tile_pos(tile, b, t0, co_base);
      const long long row_off = row_pos(t0, co_base, row_bytes);
      stage_load_row(smem_u32(stg + wt * SLD), res + (long long)b * p.rbs + row_off, row_bytes, RES_FULL(wg));
    };
    if (row_owner && res && (int)blockIdx.x < p.total_tiles) load_res(blockIdx.x);
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      float acc[MT * NACC];
#pragma unroll
      for (int e = 0; e < MT * NACC; ++e) acc[e] = 0.f;
      int held_s = -1, held_a = -1;  // weight stage / A buffer read by the group in flight
      for (int c = 0; c < nc_total; ++c) {
        mbar_wait_trap(A_FULL(buf), aph);
        const unsigned a_addr = smem_u32(a_buf + (size_t)buf * p.a_bytes);
        const int ntaps = c < p.nchunks ? p.K : 1;
        for (int k = 0; k < ntaps; ++k) {
          mbar_wait_trap(B_FULL(s), bph);
          __syncwarp();
          const int tap_row = c < p.nchunks ? (p.win_mode ? k * TT : k * p.D) : 0;
          mma_stage<MT, NB16>(acc, a_addr, lbo_a, a_sub, tap_row + wg * MT * 64, smem_u32(b_buf + (size_t)s * p.b_bytes));
          wg_wait<1>();  // the previous group has retired: its stage and, at a chunk boundary, its A buffer are free
          __syncwarp();
          if (lane == 0) {
            if (held_s >= 0) mbar_arrive(B_EMPTY(held_s));
            if (held_a >= 0) mbar_arrive(A_EMPTY(held_a));
          }
          held_s = s;
          held_a = k == ntaps - 1 ? buf : -1;
          if (++s == p.nb) { s = 0; bph ^= 1; }
        }
        if (++buf == p.na) { buf = 0; aph ^= 1; }
      }
      wg_wait<0>();
      __syncwarp();
      if (lane == 0) {
        if (held_s >= 0) mbar_arrive(B_EMPTY(held_s));
        if (held_a >= 0) mbar_arrive(A_EMPTY(held_a));
      }
      int b, t0, co_base;
      tile_pos(tile, b, t0, co_base);
      // Staged (plain mode): v = (act(a + bias) + res) * out_scale in the register epilogue's order, written over the
      // residual in the warpgroup's tile, then one bulk store (accumulate: bulk fp32 add, y + v) per channel row.
      if (staged) {
        if (res) {
          mbar_wait_trap(RES_FULL(wg), ((tile - blockIdx.x) / gridDim.x) & 1);  // one phase per tile
        } else {
          if (row_owner) bulk_wait_read();  // the last tile's store has read the tile
          wg_barrier(wg);
        }
      }
      auto stage_block = [&](const float* ab, int mb) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) {
          const int col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
          float* sv = stg + col * SLD + mb * 64 + wq * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
          float v = ab[i] + bias_s[co_base - p.co_off + col];
          if (p.post_act != PWGB_ACT_NONE) v = p.post_act == PWGB_ACT_TANH ? tanhf(v) : lrelu(v, p.post_slope);
          if (res) v += *sv;
          *sv = v * p.out_scale;
        }
      };
      // Packed output (128-column tiles, MT = 1): the quad of lanes holding 8 channels of a row (2 each, of rows r and
      // r + 8 of the fragment) transposes its split halves (two xor-shuffle steps) so that lane q stores one 16-byte run:
      // hi of row r, lo of row r, hi of row r + 8, lo of row r + 8
      auto pack_block = [&](const float* ab, int mb) {
        const int q = lane & 3;
        const bool q1 = q & 1, q2 = q & 2;
        const int t = t0 + (wg * MT + mb) * 64 + wq * 16 + (lane >> 2) + (q2 ? 8 : 0);
        bool outside = false;  // masked launches: row t lies outside the item's signal
        if constexpr (EXT && !HIST) outside = stream_outside(p.mframe, p.mend, p.mrate, p.mlook, b, t);
        const long long ld = 16LL * p.T_out;  // bytes between planes
        unsigned char* dst = reinterpret_cast<unsigned char*>(y) + (pk_plane(b, p.Cout * (MC ? p.nco : 1), co_base) +
                                                                    (q1 ? KC / 8 : 0)) * ld + 16LL * t;
#pragma unroll
        for (int n = 0; n < NACC / 4; ++n) {
          const int col = 8 * n + 2 * q;
          const float bs0 = bias_s[co_base - p.co_off + col], bs1 = bias_s[co_base - p.co_off + col + 1];
          unsigned v0, v1, v2, v3;
          split2(lrelu(ab[4 * n] + bs0, p.pk_slope), lrelu(ab[4 * n + 1] + bs1, p.pk_slope), v0, v1);
          split2(lrelu(ab[4 * n + 2] + bs0, p.pk_slope), lrelu(ab[4 * n + 3] + bs1, p.pk_slope), v2, v3);
          unsigned s0 = q2 ? v0 : v2, s1 = q2 ? v1 : v3;
          s0 = __shfl_xor_sync(0xffffffffu, s0, 2);
          s1 = __shfl_xor_sync(0xffffffffu, s1, 2);
          if (q2) { v0 = s0; v1 = s1; } else { v2 = s0; v3 = s1; }
          s0 = q1 ? v0 : v1;
          s1 = q1 ? v2 : v3;
          s0 = __shfl_xor_sync(0xffffffffu, s0, 1);
          s1 = __shfl_xor_sync(0xffffffffu, s1, 1);
          if (q1) { v0 = s0; v2 = s1; } else { v1 = s0; v3 = s1; }
          if constexpr (EXT && !HIST) {
            if (outside) v0 = v1 = v2 = v3 = 0u;  // +0.0, hi and lo
          }
          // 8-channel group n: plane (n / 4) 2 KC / 8 + n % 4 from the tile's first
          if (t < p.T_out) *reinterpret_cast<uint4*>(dst + ((n >> 2) * (2 * (KC / 8)) + (n & 3)) * ld) = make_uint4(v0, v1, v2, v3);
        }
      };
      // one 64-row block at a time, the mode chosen once per block (branching per element, or once for both blocks,
      // made ptxas spill at MT = 2)
      auto store_block = [&](auto mode, const float* ab, int mb) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) {
          const int col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
          const int t = t0 + (wg * MT + mb) * 64 + wq * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
          // (the masked launches without history take the staged or the packed epilogue only)
          if (t < p.T_out) epi_store<decltype(mode)::value, EXT && HIST>(p, ab[i], b, t, col, co_base, bias, bias_s, res, y, y2);
        }
      };
#pragma unroll
      for (int mb = 0; mb < MT; ++mb) {
        if (staged)
          stage_block(acc + mb * NACC, mb);
        else if (!HIST && MT == 1 && p.pk_out)
          pack_block(acc + mb * NACC, mb);
        else if (p.shuffle > 1)
          store_block(std::integral_constant<int, EPI_SHUFFLE>{}, acc + mb * NACC, mb);
        else if (p.wavenet)
          store_block(std::integral_constant<int, EPI_WAVENET>{}, acc + mb * NACC, mb);
        else
          store_block(std::integral_constant<int, EPI_PLAIN>{}, acc + mb * NACC, mb);
      }
      if (staged) {
        fence_proxy_async();  // generic-proxy writes -> visible to the bulk copies
        wg_barrier(wg);
        unsigned row_bytes;
        const long long row_off = row_pos(t0, co_base, row_bytes);
        if constexpr (EXT && !HIST) {
          // masked launches: the row's samples outside the item's signal become +0.0 before the store (y + 0.0 with
          // accumulate), here where the accumulators are dead
          if (row_owner) {
            int lo, hi;
            stream_signal_rows(p.mframe, p.mend, p.mrate, p.mlook, b, p.T_out, lo, hi);
            const int tw0 = t0 + wg * MT * 64;
            if (tw0 < lo || tw0 + MT * 64 > hi) {  // a tile inside the signal has nothing to mask
              float* row = stg + wt * SLD;
#pragma unroll 1
              for (int r = 0; r < MT * 64; ++r)
                if (tw0 + r < lo || tw0 + r >= hi) row[r] = 0.f;
              fence_proxy_async();  // generic-proxy writes -> visible to this thread's bulk store
            }
          }
        }
        if (row_owner) stage_store_row(y + (long long)b * p.ybs + row_off, smem_u32(stg + wt * SLD), row_bytes, p.accumulate);
        if (row_owner && res && tile + (int)gridDim.x < p.total_tiles) load_res(tile + gridDim.x);
      }
    }
    if (row_owner) bulk_wait();  // the shared-memory source must outlive the CTA's last stores
  } else if (warp == W_TMA) {
    // ===================== B producer (TMA bulk copies of packed weight stages) =====================
    const int per_tile = p.nchunks * p.K + p.nchunks2;
    const unsigned char* src = reinterpret_cast<const unsigned char*>(wpk);
    int s = 0, ph = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const unsigned char* srcc = src + (p.nco > 1 ? (size_t)(tile / pct) * per_tile * p.b_bytes : 0);
      for (int j = 0; j < per_tile; ++j) {
        mbar_wait_trap(B_EMPTY(s), ph ^ 1);
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
    if (!HIST && p.pk_in) {
      // packed activations: chunk c of a tile is the box of 8 planes x R rows at its first plane, rows from t0 - padL
      int buf = 0, ph = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        int b, t0;
        tile_origin(p, tile, TT, b, t0);
        for (int c = 0; c < p.nchunks; ++c) {
          mbar_wait(A_EMPTY(buf), ph ^ 1);
          if (elect_one()) {
            mbar_expect_tx(A_FULL(buf), (unsigned)p.a_bytes);
            tma_load_3d(smem_u32(a_buf + (size_t)buf * p.a_bytes), tm_a, 0, t0 - p.padL, (int)pk_plane(b, p.Cin, c * KC),
                        A_FULL(buf));
          }
          __syncwarp();
          if (++buf == p.na) { buf = 0; ph ^= 1; }
        }
      }
    } else if (!HIST && p.tma_act) {
      int s = 0, ph = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        int b, t0;
        tile_origin(p, tile, TT, b, t0);
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
            src = main_src(p, x, x2, b, c, MC ? (long long)((tile / pct) / p.cpg) * p.xgs : 0);
          } else {
            start = t0;
            end = t0 + TT < p.T_out ? t0 + TT : p.T_out;
            rowstride = p.T_out;
            dst_off = 0;
            src = x2 + ((long long)b * p.C2 + (long long)(c - p.nchunks) * KC) * p.T_out;
          }
          load_raw_stage(smem_u32(raw_buf + (size_t)s * p.raw_bytes), p.R4, src, rowstride, start, end, dst_off, RAW_FULL(s),
                         lane);
          __syncwarp();
          if (++s == p.ns) { s = 0; ph ^= 1; }
        }
      }
    }
  }
}

template <int MT, int NB16>
__global__ void __launch_bounds__(TC_THREADS, 1)
    conv1d_tc_kernel(const TcK p, const float* __restrict__ x, const float* __restrict__ x2,
                     const uint4* __restrict__ wpk, const float* __restrict__ bias, const float* __restrict__ res,
                     float* __restrict__ y, float* __restrict__ y2, const __grid_constant__ CUtensorMap tm_a) {
  conv1d_tc_body<MT, NB16, false>(p, x, x2, wpk, bias, res, y, y2, &tm_a);
}

// history launches (pwgb_conv1d_tc_stream_forward, the causal conv-transpose of a stream): x2 and tm_a are unused
template <int MT, int NB16>
__global__ void __launch_bounds__(TC_THREADS, 1)
    conv1d_tc_hist_kernel(const TcK p, const float* __restrict__ x, const float* __restrict__ x2,
                          const uint4* __restrict__ wpk, const float* __restrict__ bias, const float* __restrict__ res,
                          float* __restrict__ y, float* __restrict__ y2, const __grid_constant__ CUtensorMap tm_a) {
  conv1d_tc_body<MT, NB16, true>(p, x, x2, wpk, bias, res, y, y2, nullptr);
}

// history launches with a pwgb_stream_ext (pwgb_conv1d_tc_stream_ext_forward, the masked stream conv-transpose)
template <int MT, int NB16>
__global__ void __launch_bounds__(TC_THREADS, 1)
    conv1d_tc_ext_kernel(const TcKExt p, const float* __restrict__ x, const float* __restrict__ x2,
                         const uint4* __restrict__ wpk, const float* __restrict__ bias, const float* __restrict__ res,
                         float* __restrict__ y, float* __restrict__ y2) {
  conv1d_tc_body<MT, NB16, true, true>(p, x, x2, wpk, bias, res, y, y2, nullptr);
}

// the two launches of a masked ResBlock pair at 128 / 256 channels (pwgb_resblock_pair_packed_ext_forward): no history,
// the mask of TcKExt in the packed-output and the staged epilogues
template <int MT, int NB16>
__global__ void __launch_bounds__(TC_THREADS, 1)
    conv1d_tc_mask_kernel(const TcKExt p, const float* __restrict__ x, const float* __restrict__ x2,
                          const uint4* __restrict__ wpk, const float* __restrict__ bias, const float* __restrict__ res,
                          float* __restrict__ y, float* __restrict__ y2, const __grid_constant__ CUtensorMap tm_a) {
  conv1d_tc_body<MT, NB16, false, true>(p, x, x2, wpk, bias, res, y, y2, &tm_a);
}

// history launches with a pwgb_stream_ext edge policy (pwgb_conv1d_tc_stream_ext_forward with edge != 0)
template <int MT, int NB16>
__global__ void __launch_bounds__(TC_THREADS, 1)
    conv1d_tc_edge_kernel(const TcKEdge p, const float* __restrict__ x, const float* __restrict__ x2,
                          const uint4* __restrict__ wpk, const float* __restrict__ bias, const float* __restrict__ res,
                          float* __restrict__ y, float* __restrict__ y2) {
  conv1d_tc_body<MT, NB16, true, true, true>(p, x, x2, wpk, bias, res, y, y2, nullptr);
}

static int g_tc_variant = 0;
// the plan of the last conv1d_tc_kernel launch, for pwgb_debug_get(1, ...); the first five fields are the original
// readout, so a caller that asks for five ints keeps working
struct TcPlanInfo {
  int MT, na, nb, ns, staged;
  int tma_act, win_mode, nco;
};
static TcPlanInfo g_tc_last = {};
// the plan of the last wgrad_tc_kernel launch, for pwgb_debug_get(2, ...)
struct WtPlanInfo {
  int nc, tg, ntg, nsplit;
};
static WtPlanInfo g_wt_last = {};

// aux_c2: channels of the auxiliary 1x1 source (0 = none, else multiple of KC); split > 0 selects the
// WaveNet epilogue.  pre_gate: d->cin is the number of gated channels, x holds 2*cin channels.
// has_res: the launch adds a residual (selects the staged epilogue like an accumulate does).
// pk_in: the activations are a packed intermediate (pk_plane) landed by tensor copies, with no raw stages.
static int tc_plan(const pwgb_conv1d_desc* d, TcK& p, size_t& smem_bytes, int aux_c2 = 0, int split = 0, int nco_bias = 1,
                   int has_res = 0, int pk_in = 0) {
  p.variant = g_tc_variant;
  p.pk_in = pk_in;
  p.pk_out = 0;
  p.pk_slope = 0.f;
  p.hist = nullptr;
  p.rep = nullptr;
  p.hist_len = 0;
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
  // Staged epilogue (see conv1d_tc_kernel): plain mode with a residual or an accumulate, 16-byte rows (T_out % 4 == 0;
  // tc_launch also checks the y and residual base pointers).  Its two tiles must fit beside the raw-staged pipeline
  // (three raw stages with TMA activations, else two; two operand buffers) and at least four weight stages, within the
  // opt-in limit TC_SMEM_STAGED instead of the 216 KB of the other plans; a tile shape that cannot gets the next
  // attempt (64 channels: MT = 1 instead of 2), and without any such plan the conv keeps the register epilogue.
  const bool want_stage = !(p.variant & 4) && d->shuffle <= 1 && split == 0 && !d->pre_gate && (has_res || d->accumulate) &&
                          d->t_out % 4 == 0;
  for (int staged = want_stage ? 1 : 0; staged >= 0; --staged) {
    // tile shape (1 persistent CTA / SM, ~216 KB of shared memory): prefer a contiguous halo tile of
    // 2 x 128 rows (Cout <= 64: the 64 accumulator registers hold both); fall back to 128 rows, then to
    // one window per tap (very large dilation)
    const size_t budget = staged ? TC_SMEM_STAGED : 216 * 1024;
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
      if (pk_in && p.win_mode) continue;
      if (p.win_mode && halo <= p.MT * 128) continue;  // a contiguous tile is never larger in that case
      p.a_bytes = 2 * (KC / 8) * p.R * 16;
      p.R4 = (p.R + 6) & ~3;
      p.raw_bytes = KC * p.R4 * 4;
      // activation rows by TMA: zero padding only (out-of-range samples are masked, never copied) and
      // 16-byte aligned rows; anything else is staged with 4-byte cp.async by the producers
      p.tma_act = !(p.variant & 2) && !d->pre_gate && !p.win_mode && d->pad_mode == PWGB_PAD_ZERO && d->t_in % 4 == 0 &&
                  (aux_c2 == 0 || d->t_out % 4 == 0);
      // shared-memory split: [na operand buffers][nb weight stages][ns raw staging buffers][epilogue tiles]
      int na = 0, nb = 0, ns = 0;
      const size_t bias_bytes = 4 * (size_t)(nco_bias > 1 ? nco_bias * d->cout : TC_NMAX);  // bias of every column chunk of the launch
      const size_t A = (size_t)p.a_bytes, Bs = (size_t)p.b_bytes, S = (size_t)p.raw_bytes, slack = 1024 + bias_bytes;
      const size_t E = staged ? 2 * (size_t)d->cout * stage_ld(p.MT) * 4 : 0;
      if (staged && !stage_shape(p.MT, d->cout)) continue;
      if (pk_in) {
        // the raw stages' bytes go to weight stages
        na = 2;
        if (na * A + 4 * Bs + E + slack > budget) continue;
      } else if (staged) {
        ns = p.tma_act ? 3 : 2;
        na = 2;
        if (na * A + ns * S + 4 * Bs + E + slack > budget) continue;
      } else if (p.tma_act && 2 * A + 3 * S + 3 * Bs + slack <= budget) {
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
      nb = (int)((budget - slack - (size_t)na * A - (size_t)ns * S - E) / Bs);
      if (nb > 24) nb = 24;
      p.na = na;
      p.nb = nb;
      p.ns = ns;
      p.staged = staged;
      p.tiles_per_seq = ceil_div(d->t_out, p.MT * 128);
      p.total_tiles = p.tiles_per_seq * d->batch;
      smem_bytes = (size_t)na * p.a_bytes + (size_t)ns * p.raw_bytes + (size_t)nb * p.b_bytes + E +
                   8 * (2 * na + 2 * nb + 4 + 2 * NS_MAX + 2) + 16 + bias_bytes;
      return 1;
    }
  }
  return 0;
}

using TcKernel = void (*)(const TcK, const float*, const float*, const uint4*, const float*, const float*, float*, float*,
                         const CUtensorMap);

// Every tile shape tc_plan produces: MT = 1 at any width of 16 .. TC_NMAX columns (the first 8), MT = 2 up to
// TC_NMAX / 2 (the last 4).
static const TcKernel tc_kernels[12] = {conv1d_tc_kernel<1, 1>, conv1d_tc_kernel<1, 2>, conv1d_tc_kernel<1, 3>,
                                        conv1d_tc_kernel<1, 4>, conv1d_tc_kernel<1, 5>, conv1d_tc_kernel<1, 6>,
                                        conv1d_tc_kernel<1, 7>, conv1d_tc_kernel<1, 8>, conv1d_tc_kernel<2, 1>,
                                        conv1d_tc_kernel<2, 2>, conv1d_tc_kernel<2, 3>, conv1d_tc_kernel<2, 4>};
static const TcKernel tc_hist_kernels[12] = {
    conv1d_tc_hist_kernel<1, 1>, conv1d_tc_hist_kernel<1, 2>, conv1d_tc_hist_kernel<1, 3>, conv1d_tc_hist_kernel<1, 4>,
    conv1d_tc_hist_kernel<1, 5>, conv1d_tc_hist_kernel<1, 6>, conv1d_tc_hist_kernel<1, 7>, conv1d_tc_hist_kernel<1, 8>,
    conv1d_tc_hist_kernel<2, 1>, conv1d_tc_hist_kernel<2, 2>, conv1d_tc_hist_kernel<2, 3>, conv1d_tc_hist_kernel<2, 4>};
using TcKernelExt = void (*)(const TcKExt, const float*, const float*, const uint4*, const float*, const float*, float*, float*);
static const TcKernelExt tc_ext_kernels[12] = {
    conv1d_tc_ext_kernel<1, 1>, conv1d_tc_ext_kernel<1, 2>, conv1d_tc_ext_kernel<1, 3>, conv1d_tc_ext_kernel<1, 4>,
    conv1d_tc_ext_kernel<1, 5>, conv1d_tc_ext_kernel<1, 6>, conv1d_tc_ext_kernel<1, 7>, conv1d_tc_ext_kernel<1, 8>,
    conv1d_tc_ext_kernel<2, 1>, conv1d_tc_ext_kernel<2, 2>, conv1d_tc_ext_kernel<2, 3>, conv1d_tc_ext_kernel<2, 4>};
static TcKernelExt tc_ext_kernel_for(int mt, int cout) {
  if (cout % 16 != 0) return nullptr;
  const int nb16 = cout / 16;
  if (mt == 1 && nb16 >= 1 && nb16 <= 8) return tc_ext_kernels[nb16 - 1];
  if (mt == 2 && nb16 >= 1 && nb16 <= 4) return tc_ext_kernels[8 + nb16 - 1];
  return nullptr;
}
using TcKernelEdge = void (*)(const TcKEdge, const float*, const float*, const uint4*, const float*, const float*, float*, float*);
static const TcKernelEdge tc_edge_kernels[12] = {
    conv1d_tc_edge_kernel<1, 1>, conv1d_tc_edge_kernel<1, 2>, conv1d_tc_edge_kernel<1, 3>, conv1d_tc_edge_kernel<1, 4>,
    conv1d_tc_edge_kernel<1, 5>, conv1d_tc_edge_kernel<1, 6>, conv1d_tc_edge_kernel<1, 7>, conv1d_tc_edge_kernel<1, 8>,
    conv1d_tc_edge_kernel<2, 1>, conv1d_tc_edge_kernel<2, 2>, conv1d_tc_edge_kernel<2, 3>, conv1d_tc_edge_kernel<2, 4>};
static TcKernelEdge tc_edge_kernel_for(int mt, int cout) {
  if (cout % 16 != 0) return nullptr;
  const int nb16 = cout / 16;
  if (mt == 1 && nb16 >= 1 && nb16 <= 8) return tc_edge_kernels[nb16 - 1];
  if (mt == 2 && nb16 >= 1 && nb16 <= 4) return tc_edge_kernels[8 + nb16 - 1];
  return nullptr;
}
static TcKernel tc_kernel_for(int mt, int cout, bool hist) {
  if (cout % 16 != 0) return nullptr;
  const TcKernel* table = hist ? tc_hist_kernels : tc_kernels;
  const int nb16 = cout / 16;
  if (mt == 1 && nb16 >= 1 && nb16 <= 8) return table[nb16 - 1];
  if (mt == 2 && nb16 >= 1 && nb16 <= 4) return table[8 + nb16 - 1];
  return nullptr;
}

// P: TcK, or TcKExt / TcKEdge for the EXT / EDGE kernels of a pwgb_stream_ext launch
template <class P>
static int tc_launch(P& p, size_t bytes, const float* x, const void* packed_w, const float* bias,
                     const float* residual, float* y, cudaStream_t st, const float* x2 = nullptr,
                     float* y2 = nullptr, const CUtensorMap* tm_a = nullptr) {
  if (p.B == 0 || p.T_out == 0) return PWGB_OK;
  constexpr bool ext = std::is_same<P, TcKExt>::value;
  constexpr bool edge = std::is_same<P, TcKEdge>::value;
  const bool hist = is_history_pad(p.pad_mode);
  std::conditional_t<edge, TcKernelEdge, std::conditional_t<ext, TcKernelExt, TcKernel>> kernel;
  if constexpr (edge)
    kernel = tc_edge_kernel_for(p.MT, p.Cout);
  else if constexpr (ext)
    kernel = tc_ext_kernel_for(p.MT, p.Cout);
  else
    kernel = tc_kernel_for(p.MT, p.Cout, hist);
  if (!kernel) {
    set_error("conv1d_tc: no kernel instantiation for MT = %d, Cout = %d", p.MT, p.Cout);
    return PWGB_UNSUPPORTED;
  }
  static bool smem_set = false, smem_set_hist = false;
  if constexpr (edge) {
    if (const int rc = smem_opt_in(smem_set, tc_edge_kernels, (int)TC_SMEM_STAGED, "conv1d_tc")) return rc;
  } else if constexpr (ext) {
    if (const int rc = smem_opt_in(smem_set, tc_ext_kernels, (int)TC_SMEM_STAGED, "conv1d_tc")) return rc;
  } else {
    if (const int rc = hist ? smem_opt_in(smem_set_hist, tc_hist_kernels, (int)TC_SMEM_STAGED, "conv1d_tc")
                            : smem_opt_in(smem_set, tc_kernels, (int)TC_SMEM_STAGED, "conv1d_tc"))
      return rc;
  }
  const int num_sms = tc_num_sms();
  if ((long long)p.B * p.tiles_per_seq > 0x7fffffffLL) {
    set_error("conv1d_tc: too many tiles");
    return PWGB_UNSUPPORTED;
  }
  if (p.tma_act && ((reinterpret_cast<uintptr_t>(x) & 15) || (x2 && (reinterpret_cast<uintptr_t>(x2) & 15))))
    p.tma_act = 0;  // unaligned base pointer: the producers stage with cp.async instead
  if (p.staged && ((reinterpret_cast<uintptr_t>(y) & 15) || (reinterpret_cast<uintptr_t>(residual) & 15)))
    p.staged = 0;  // bulk copies need 16-byte aligned rows: the register epilogue (the plan's tiles stay unused)
  g_tc_last = TcPlanInfo{p.MT, p.na, p.nb, p.ns, p.staged, p.tma_act, p.win_mode, p.nco};
  const int grid = p.total_tiles < num_sms ? p.total_tiles : num_sms;
  if constexpr (edge || ext) {
    kernel<<<(unsigned)grid, TC_THREADS, bytes, st>>>(p, x, x2, (const uint4*)packed_w, bias, residual, y, y2);
  } else {
    CUtensorMap tm;
    if (tm_a)
      tm = *tm_a;
    else
      memset(&tm, 0, sizeof(tm));
    kernel<<<(unsigned)grid, TC_THREADS, bytes, st>>>(p, x, x2, (const uint4*)packed_w, bias, residual, y, y2, tm);
  }
  return check_launch("conv1d_tc_kernel");
}

// The pwgb_stream_ext of a history launch, for the EXT kernels.  Their epilogue reads residual rows one by one and masks each
// store, so the launch keeps the register epilogue, which computes the staged epilogue's values.
static void tc_apply_ext(TcKExt& p, const pwgb_stream_ext* e, int cout_total) {
  p.mframe = e->frame;
  p.mend = e->end;
  p.mrate = e->rate;
  p.mlook = e->lookahead;
  p.rhist = e->res_hist;
  p.rhist_len = e->res_hist_len;
  p.rdelay = e->res_delay;
  p.rhbs = (long long)cout_total * e->res_hist_len;
  p.staged = 0;
}

// Internal entry for N-chunked callers (conv_transpose): runs output channels
// [co_off, co_off + d->cout) of a conv whose full output has cout_total channels.  cin1 > 0: the input is
// cat(x (B, cin1, T), x2 (B, d->cin - cin1, T)) along channels (cin1 a multiple of KC).  d->pad_mode ==
// PWGB_PAD_HISTORY: a history launch reading rows before sample 0 from hist / rep (one source only).
int conv1d_tc_chunk(const pwgb_conv1d_desc* d, int co_off, int cout_total, const float* x, const void* packed_w,
                    const float* bias, float* y, cudaStream_t st, int nco, const float* x2, int cin1, const float* hist,
                    const int* rep, int hist_len, const pwgb_stream_ext* ext) {
  TcK p;
  size_t bytes = 0;
  if (!tc_plan(d, p, bytes)) return PWGB_UNSUPPORTED;
  if (is_history_pad(d->pad_mode)) {
    if (cin1 > 0) return PWGB_UNSUPPORTED;
    p.hist = hist;
    p.rep = rep;
    p.hist_len = hist_len;
  }
  if (cin1 > 0) {
    // the direct register path (ns == 0) reads one source
    if (!x2 || cin1 % KC || cin1 >= d->cin || p.ns == 0) return PWGB_UNSUPPORTED;
    p.C2 = d->cin - cin1;
    p.xbs = (long long)cin1 * d->t_in;
  }
  p.co_off = co_off;
  p.ybs = d->shuffle > 1 ? (long long)(cout_total / d->shuffle) * d->shuffle_tout : (long long)cout_total * d->t_out;
  if (nco > 1) {
    // the chunks' packed images are consecutive: one launch walks (chunk, batch, time tile)
    if (d->shuffle <= 1 || (long long)p.total_tiles * nco > 0x7fffffffLL) return PWGB_UNSUPPORTED;
    p.nco = nco;
    p.total_tiles *= nco;
  }
  if (ext && is_history_pad(d->pad_mode)) {
    TcKExt px;
    static_cast<TcK&>(px) = p;
    tc_apply_ext(px, ext, cout_total);
    return tc_launch(px, bytes, x, packed_w, bias, nullptr, y, st);
  }
  return tc_launch(p, bytes, x, packed_w, bias, nullptr, y, st, cin1 > 0 ? x2 : nullptr);
}

// raw_staged: set to 1 when the plan stages activations through shared memory (TMA or cp.async), as a two-source
// input requires
int conv1d_tc_plan_ok(const pwgb_conv1d_desc* d, int* raw_staged) {
  TcK p;
  size_t bytes;
  const int ok = tc_plan(d, p, bytes);
  if (raw_staged) *raw_staged = ok && p.ns > 0;
  return ok;
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

namespace pwgb {
extern int g_simt_last[6];  // conv1d_simt.cu
extern int g_wgs_last[4];   // backward.cu
}  // namespace pwgb

// key 1: the plan of the last conv1d_tc launch, {MT, na, nb, ns, staged, tma_act, win_mode, nco};
// key 2: the plan of the last conv1d_wgrad_tc launch, {nc, tg, ntg, nsplit};
// key 3: the last FFMA conv dispatch, {kernel, RCO, WARPS_CO, RT, CI_T, CO};
// key 4: the last FFMA weight-gradient launch, {path, narrow_fast, nsplit or narrow blocks, ci_tiles}.
// Copies min(bytes, size of the record); a buffer of at least 5 (key 1) or the whole record (keys 2-4) is required.
extern "C" int pwgb_debug_get(int key, void* dst, size_t bytes) {
  if (!dst) return -1;
  const void* src = key == 1   ? (const void*)&g_tc_last
                    : key == 2 ? (const void*)&g_wt_last
                    : key == 3 ? (const void*)g_simt_last
                    : key == 4 ? (const void*)g_wgs_last
                               : nullptr;
  const size_t size = key == 1 ? sizeof(TcPlanInfo) : key == 2 ? sizeof(WtPlanInfo) : key == 3 ? sizeof(g_simt_last) : sizeof(g_wgs_last);
  const size_t need = key == 1 ? 5 * sizeof(int) : size;
  if (!src || bytes < need) return -1;
  memcpy(dst, src, bytes < size ? bytes : size);
  return 0;
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
  // history padding: one-source convs without pre_gate (pwgb_conv1d_tc_stream_forward); a grouped one reads no row
  // before sample 0 (pad_left 0: a window that carries its own history, as after pwgb_s2d_stream_grouped_forward)
  if (is_history_pad(d->pad_mode) && ((d->groups != 1 && d->pad_left != 0) || d->pre_gate || d->shuffle > 1)) return 0;
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

static int tc_forward(const pwgb_conv1d_desc* d, const float* x, const void* packed_w, const float* bias, const float* residual,
                      float* y, void* stream, const float* hist, const int* rep, int hist_len,
                      const pwgb_stream_ext* ext = nullptr) {
  PWGB_UNSUPPORTED_IF(!pwgb_conv1d_tc_supported(d), "conv1d_tc: configuration not supported by the tensor-core path");
  const int G = d->groups, cin_g = d->cin / G, cout_g = d->cout / G;
  // the history loader addresses hist by the chunk within a group: a grouped launch must not read one
  PWGB_UNSUPPORTED_IF(G > 1 && hist_len > 0, "conv1d_tc_stream: a grouped history launch takes no history rows (hist_len %d)", hist_len);
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
  if (!tc_plan(&c, p, bytes, 0, 0, nco, residual != nullptr)) {
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
  p.hist = hist;
  p.rep = rep;
  p.hist_len = hist_len;
  if (ext && ext->edge) {
    TcKEdge px;
    static_cast<TcK&>(px) = p;
    tc_apply_ext(px, ext, d->cout);
    px.edge = ext->edge;
    px.in_look = ext->in_lookahead;
    return tc_launch(px, bytes, x, packed_w, bias, residual, y, (cudaStream_t)stream);
  }
  if (ext) {
    TcKExt px;
    static_cast<TcK&>(px) = p;
    tc_apply_ext(px, ext, d->cout);
    return tc_launch(px, bytes, x, packed_w, bias, residual, y, (cudaStream_t)stream);
  }
  return tc_launch(p, bytes, x, packed_w, bias, residual, y, (cudaStream_t)stream);
}

extern "C" int pwgb_conv1d_tc_forward(const pwgb_conv1d_desc* d, const float* x, const void* packed_w,
                                      const float* bias, const float* residual, float* y, void* stream) {
  PWGB_CHECK_ARG(d && x && packed_w && y, "conv1d_tc: null argument");
  PWGB_CHECK_ARG(!is_history_pad(d->pad_mode), "conv1d_tc: history padding is served by pwgb_conv1d_tc_stream_forward");
  return tc_forward(d, x, packed_w, bias, residual, y, stream, nullptr, nullptr, 0);
}

extern "C" int pwgb_conv1d_tc_stream_forward(const pwgb_conv1d_desc* d, const float* x, const float* hist, int hist_len,
                                             const int* replicate, const void* packed_w, const float* bias, const float* residual,
                                             float* y, void* stream) {
  PWGB_CHECK_ARG(packed_w, "conv1d_tc_stream: null argument");
  if (const int rc = conv1d_stream_check(d, x, hist, hist_len, y)) return rc;
  return tc_forward(d, x, packed_w, bias, residual, y, stream, hist, replicate, hist_len);
}

extern "C" int pwgb_conv1d_tc_stream_ext_forward(const pwgb_conv1d_desc* d, const float* x, const float* hist, int hist_len,
                                                 const int* replicate, const void* packed_w, const float* bias,
                                                 const float* residual, const pwgb_stream_ext* ext, float* y, void* stream) {
  PWGB_CHECK_ARG(packed_w, "conv1d_tc_stream: null argument");
  if (const int rc = conv1d_stream_check(d, x, hist, hist_len, y)) return rc;
  if (const int rc = stream_ext_check(ext, residual, d->pad_mode)) return rc;
  return tc_forward(d, x, packed_w, bias, residual, y, stream, hist, replicate, hist_len, ext);
}

extern "C" int pwgb_conv1d_tc_ragged_forward(const pwgb_conv1d_desc* d, const float* x, const void* packed_w, const float* bias,
                                             const float* residual, const pwgb_stream_ext* ext, float* y, void* stream) {
  if (!ext) return pwgb_conv1d_tc_forward(d, x, packed_w, bias, residual, y, stream);
  PWGB_CHECK_ARG(packed_w, "conv1d_tc_ragged: null argument");
  pwgb_conv1d_desc h;
  if (const int rc = conv1d_ragged_check(d, x, ext, y, &h)) return rc;
  // the EXT / EDGE history kernels with no history rows: rows outside [0, t_in) stage as zero unless the edge policy
  // moves them onto the item's own reflected or replicated sample
  return tc_forward(&h, x, packed_w, bias, residual, y, stream, nullptr, nullptr, 0, ext);
}

// ======================================================================================
// A 128- or 256-channel HiFi-GAN ResBlock conv pair as two conv1d_tc launches that hand the intermediate over packed
// (pk_plane): conv1's epilogue writes lrelu(conv1 + b1) already split, conv2 lands it with one tensor copy per chunk and
// spends the raw stages' shared memory on weight stages.  conv2 must take the staged epilogue (the residual x).
// ======================================================================================
namespace pwgb {

static int rb_packed_plan(const pwgb_resblock_desc* d, TcK& p1, size_t& bytes1, TcK& p2, size_t& bytes2) {
  if (!d || (g_tc_variant & 8) || (d->channels != 128 && d->channels != 256) || d->batch < 0 || d->t <= 0 || d->t % 4 ||
      d->kernel < 1 || d->kernel % 2 == 0 || d->dilation < 1)
    return 0;
  const int nco = d->channels / TC_NMAX;
  pwgb_conv1d_desc c = {};
  c.batch = d->batch;
  c.cin = d->channels;
  c.cout = TC_NMAX;
  c.t_in = c.t_out = c.t_valid = d->t;
  c.kernel = d->kernel;
  c.stride = 1;
  c.dilation = d->dilation;
  c.groups = 1;
  c.pad_left = (d->kernel - 1) / 2 * d->dilation;
  c.pad_mode = PWGB_PAD_ZERO;
  c.period = 1;
  c.pre_slope = d->slope;
  c.out_scale = 1.f;
  if (!tc_plan(&c, p1, bytes1, 0, 0, nco) || p1.MT != 1) return 0;  // the packed epilogue: 128-column tiles
  c.dilation = 1;
  c.pad_left = (d->kernel - 1) / 2;
  c.out_scale = d->out_scale;
  c.accumulate = d->accumulate;
  if (!tc_plan(&c, p2, bytes2, 0, 0, nco, 1, 1) || !p2.staged || p2.R > 256) return 0;  // one box: at most 256 rows
  if ((long long)p1.total_tiles * nco > 0x7fffffffLL) return 0;
  p1.pk_out = 1;
  p1.pk_slope = d->slope;
  for (TcK* p : {&p1, &p2}) {
    p->xbs = p->ybs = p->rbs = (long long)d->channels * d->t;
    if (nco > 1) {
      p->nco = p->cpg = nco;
      p->total_tiles *= nco;
    }
  }
  return 1;
}

}  // namespace pwgb

extern "C" int pwgb_resblock_pair_packed_supported(const pwgb_resblock_desc* d) {
  TcK p1, p2;
  size_t b1, b2;
  return rb_packed_plan(d, p1, b1, p2, b2);
}

// One masked launch of the packed pair: both are 128-column, one-block tiles (rb_packed_plan)
static int rb_packed_launch_ext(TcKExt& p, size_t bytes, const float* x, const void* packed_w, const float* bias,
                                const float* residual, float* y, cudaStream_t st, const CUtensorMap* tm_a) {
  using Kernel = void (*)(const TcKExt, const float*, const float*, const uint4*, const float*, const float*, float*, float*,
                          const CUtensorMap);
  static const Kernel kernels[1] = {conv1d_tc_mask_kernel<1, TC_NMAX / 16>};
  static bool smem_set = false;
  if (p.MT != 1 || p.Cout != TC_NMAX || !(p.staged || p.pk_out)) {
    set_error("resblock_pair_packed_ext: no masked kernel for MT = %d, Cout = %d", p.MT, p.Cout);
    return PWGB_UNSUPPORTED;
  }
  if (const int rc = smem_opt_in(smem_set, kernels, (int)TC_SMEM_STAGED, "resblock_pair_packed_ext")) return rc;
  CUtensorMap tm;
  if (tm_a)
    tm = *tm_a;
  else
    memset(&tm, 0, sizeof(tm));
  const int num_sms = tc_num_sms();
  const int grid = p.total_tiles < num_sms ? p.total_tiles : num_sms;
  kernels[0]<<<(unsigned)grid, TC_THREADS, bytes, st>>>(p, x, nullptr, (const uint4*)packed_w, bias, residual, y, nullptr, tm);
  return check_launch("conv1d_tc_mask_kernel");
}

extern "C" int pwgb_resblock_pair_packed_ext_forward(const pwgb_resblock_desc* d, const float* x, const void* w1_packed,
                                                     const float* b1, const void* w2_packed, const float* b2,
                                                     const pwgb_stream_ext* ext, void* h_packed, float* y, void* stream) {
  if (!ext) return pwgb_resblock_pair_packed_forward(d, x, w1_packed, b1, w2_packed, b2, h_packed, y, stream);
  PWGB_CHECK_ARG(d && x && w1_packed && w2_packed && h_packed && y, "resblock_pair_packed_ext: null argument");
  PWGB_CHECK_ARG(ext->frame && ext->end && ext->rate >= 1 && ext->lookahead >= 0,
                 "resblock_pair_packed_ext: ext must hold a mask (frame, end, rate >= 1, lookahead >= 0)");
  TcKExt p1, p2;
  size_t bytes1 = 0, bytes2 = 0;
  PWGB_UNSUPPORTED_IF(!rb_packed_plan(d, p1, bytes1, p2, bytes2), "resblock_pair_packed_ext: configuration not supported");
  PWGB_CHECK_ARG(x != y, "resblock_pair_packed_ext: y must not alias x (halo reads)");
  PWGB_UNSUPPORTED_IF(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(h_packed)) & 15),
                      "resblock_pair_packed_ext: x, h_packed and y must be 16-byte aligned");
  if (d->batch == 0) return PWGB_OK;
  for (TcKExt* p : {&p1, &p2}) {
    p->mframe = ext->frame;
    p->mend = ext->end;
    p->mrate = ext->rate;
    p->mlook = ext->lookahead;
    p->rhist = nullptr;
    p->rhist_len = p->rdelay = 0;
    p->rhbs = 0;
  }
  CUtensorMap tm;
  const unsigned long long dims[3] = {8ull, (unsigned long long)d->t, (unsigned long long)pk_plane(d->batch, d->channels, 0)};
  const unsigned box[3] = {8u, (unsigned)p2.R, 2u * (KC / 8)};
  if (const int rc = tma_make(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, 3, h_packed, dims, box)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (const int rc = rb_packed_launch_ext(p1, bytes1, x, w1_packed, b1, nullptr, static_cast<float*>(h_packed), st, nullptr))
    return rc;
  return rb_packed_launch_ext(p2, bytes2, static_cast<const float*>(h_packed), w2_packed, b2, x, y, st, &tm);
}

extern "C" int pwgb_resblock_pair_packed_forward(const pwgb_resblock_desc* d, const float* x, const void* w1_packed,
                                                 const float* b1, const void* w2_packed, const float* b2, void* h_packed,
                                                 float* y, void* stream) {
  PWGB_CHECK_ARG(d && x && w1_packed && w2_packed && h_packed && y, "resblock_pair_packed: null argument");
  TcK p1, p2;
  size_t bytes1 = 0, bytes2 = 0;
  PWGB_UNSUPPORTED_IF(!rb_packed_plan(d, p1, bytes1, p2, bytes2), "resblock_pair_packed: configuration not supported");
  PWGB_CHECK_ARG(x != y, "resblock_pair_packed: y must not alias x (halo reads)");
  PWGB_UNSUPPORTED_IF(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(h_packed)) & 15),
                      "resblock_pair_packed: x, h_packed and y must be 16-byte aligned");
  if (d->batch == 0) return PWGB_OK;
  // the packed image as (8 channels, t rows, planes) bf16; a box is one chunk's 8 planes of R rows
  CUtensorMap tm;
  const unsigned long long dims[3] = {8ull, (unsigned long long)d->t, (unsigned long long)pk_plane(d->batch, d->channels, 0)};
  const unsigned box[3] = {8u, (unsigned)p2.R, 2u * (KC / 8)};
  if (const int rc = tma_make(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, 3, h_packed, dims, box)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (const int rc = tc_launch(p1, bytes1, x, w1_packed, b1, nullptr, static_cast<float*>(h_packed), st)) return rc;
  return tc_launch(p2, bytes2, static_cast<const float*>(h_packed), w2_packed, b2, x, y, st, nullptr, nullptr, &tm);
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
  c1.pad_left = (d->causal ? d->kernel - 1 : (d->kernel - 1) / 2) * d->dilation;
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
  return d && d->batch >= 0 && d->t > 0 && d->kernel > 0 && (d->causal || d->kernel % 2 == 1) && d->dilation > 0 &&
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
  if (d->batch == 0) return PWGB_OK;  // an empty batch: no launch (and the empty tensors have no storage)
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
  using WtKernel = void (*)(const WtK, const float*, const float*, float*);
  static bool smem_set = false;
  if (const int rc = smem_opt_in(smem_set, {WtKernel(wgrad_tc_kernel<32>), WtKernel(wgrad_tc_kernel<64>)}, 220 * 1024,
                                 "conv1d_wgrad_tc"))
    return rc;
  g_wt_last = WtPlanInfo{p.nc, p.tg, p.ntg, p.nsplit};
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
