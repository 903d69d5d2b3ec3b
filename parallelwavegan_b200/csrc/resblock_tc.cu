// One HiFi-GAN ResBlock conv pair (layers/residual_block.py:243-258, non-causal, with the additional convs) in one
// tensor-core kernel:
//   h  = conv_{k,d}(lrelu(x)) + b1                       (zero padding (k-1)/2 * d)
//   x' = conv_{k,1}(lrelu(h)) + b2 + x                   (zero padding (k-1)/2)
//   y  = x' * out_scale,  or  y += x' * out_scale       (the last pair of a block writes the MRF sum)
// The intermediate h never leaves the SM: conv1's accumulators are written, as lrelu(h) split into bf16 hi/lo, straight
// into the K-major operand image that conv2's wgmma reads.  Everything else is the stride-1 conv of conv1d_tc.cu: the
// same weight images (pwgb_conv1d_tc_pack_weight), bf16x3 products, and MMA order into every accumulator (32-channel
// chunk, tap, k16 step, hi*hi, lo*hi, hi*lo), so the result is bit-identical to the two conv1d_tc launches.  The pieces
// of that pipeline (raw-row loader, raw stage conversion, MMA of a weight stage, staged-epilogue row load and store) are
// the ones conv1d_tc_kernel calls, from tc_common.cuh.
//
// Tiling: a tile produces M2 output rows [t0, t0 + M2).  Conv2 needs h rows [t0 - p2, t0 + M2 + p2), p2 = (k-1)/2;
// conv1 computes the TT conv rows [t0 - p2, t0 - p2 + TT) from R1 = TT + (k-1) d input rows, so M2 = TT - (k-1)
// rounded down to a multiple of 4 (16-byte output rows).  Halo rows of h are recomputed by the neighbouring tile.  Conv2
// also runs TT rows per tile; rows >= M2 read beyond the computed h rows and are dropped.
//
// One kernel, rb_pair_split_kernel, one persistent CTA per SM, with the warp roles of conv1d_tc_kernel with TMA-staged
// activations: producer warps convert landed raw fp32 rows of x (pre-activation, padding mask, hi/lo split)
// into conv1's operand image, one warp loads weight stages and one raw activation rows, both by cp.async.bulk.  The two
// consumer warpgroups are split by conv: warpgroup 0 runs conv1 of every tile and writes the h image, warpgroup 1 runs
// conv2 on it and the staged epilogue, so that one warpgroup's drain, h write or epilogue overlaps the other's MMAs.
// Each conv owns a weight ring.  A pair whose conv1 halo leaves no room for two rings of RB_MIN_STAGES stages has no
// plan and runs as the two conv1d_tc launches.
#include <cstring>
#include <type_traits>

#include "tc_common.cuh"

namespace pwgb {

namespace {

// 512 threads, so that a thread may hold 128 registers (warps are allocated in fours: at 18 warps the limit is 96, and
// the 64 accumulator registers spill): warps 0-3 conv1, warps 4-7 conv2 and the epilogue, warps 8-13 the producers
// (a chunk has at most TT + 50 conv1 rows), warp 14 the weight rings, warp 15 the raw activation rows.
constexpr int RB_NPROD = 192;
constexpr int RB_W_PROD0 = 8, RB_W_TMA = RB_W_PROD0 + RB_NPROD / 32, RB_W_LDA = RB_W_TMA + 1;
constexpr int RB_THREADS = 32 * (RB_W_LDA + 1);
constexpr size_t RB_SMEM = 227 * 1024;      // H100 opt-in limit of dynamic shared memory per block
constexpr int RB_MIN_STAGES = 4;            // weight stages a plan must keep per ring

struct RbK {
  int B, C, T, K, D;
  float slope, out_scale;
  int accumulate;
  int MT, M2;              // 64-row blocks per tile, output rows per tile
  int p1, p2;              // left padding of conv1 ((k-1)/2 * d) and conv2 ((k-1)/2)
  int R1, R4, Rh;          // conv1 operand rows, raw stage row pitch (floats), h image rows (TT + k - 1)
  int nchunks, tiles_per_seq, total_tiles;
  int na, nb, ns;          // conv1 operand buffers, weight stages (both rings), raw stages
  int a_bytes, b_bytes, raw_bytes, h_bytes;  // per buffer / stage; h_bytes: one 32-channel chunk of the h image
};

// The mask of a pwgb_resblock_pair_ext_forward launch (the mask fields of pwgb_stream_ext): row t of item b is signal
// sample mframe[b] * mrate - mlook + t, and the h rows conv2 reads and the y rows outside [0, mend[b] * mrate) are +0.0.
// A separate struct and kernel (EXT), so that rb_pair_split_kernel keeps its parameters and code.
struct RbKExt : RbK {
  const int* mframe;
  const int* mend;
  int mrate, mlook;
};

__device__ __forceinline__ void rb_signal_rows(const RbKExt& p, int b, int& lo, int& hi) {
  stream_signal_rows(p.mframe, p.mend, p.mrate, p.mlook, b, p.T, lo, hi);
}

// ===================== A producers: raw fp32 rows -> conv1 operand image =====================
// RB_NPROD producer threads, this one `tid` of them.  Barrier arguments are the first of each array of 8-byte mbarriers.
template <int NCH>
__device__ __forceinline__ void rb_convert_x(const RbK& p, unsigned char* a_buf, const unsigned char* raw_buf, unsigned a_full,
                                             unsigned a_empty, unsigned raw_full, unsigned raw_empty, int tid) {
  int s = 0, sph = 0, buf = 0, aph = 0;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const int b = tile / p.tiles_per_seq;
    const int t0 = (tile - b * p.tiles_per_seq) * p.M2;
    const int ts_first = t0 - p.p2 - p.p1;
    const int shift = ts_first - (ts_first & ~3);
    for (int c = 0; c < NCH; ++c) {
      mbar_wait(raw_full + 8u * s, sph);
      mbar_wait(a_empty + 8u * buf, aph ^ 1);
      const float* raw = reinterpret_cast<const float*>(raw_buf + (size_t)s * p.raw_bytes);
      convert_raw_stage<RB_NPROD, true>(a_buf + (size_t)buf * p.a_bytes, p.R1, raw, shift, p.R4, p.R1, ts_first,
                                        (unsigned)p.T, p.slope, tid);
      fence_proxy_async();
      mbar_arrive(a_full + 8u * buf);
      mbar_arrive(raw_empty + 8u * s);
      if (++s == p.ns) { s = 0; sph ^= 1; }
      if (++buf == p.na) { buf = 0; aph ^= 1; }
    }
  }
}

// ===================== raw activation rows of x (one channel per lane) =====================
template <int NCH>
__device__ __forceinline__ void rb_load_raw(const RbK& p, const float* __restrict__ x, unsigned char* raw_buf, unsigned raw_full,
                                            unsigned raw_empty, int lane) {
  constexpr int C = NCH * KC;
  int s = 0, ph = 0;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const int b = tile / p.tiles_per_seq;
    const int t0 = (tile - b * p.tiles_per_seq) * p.M2;
    const int ts0 = (t0 - p.p2 - p.p1) & ~3;
    const int start = ts0 < 0 ? 0 : ts0;
    const int end = ts0 + p.R4 < p.T ? ts0 + p.R4 : p.T;
    for (int c = 0; c < NCH; ++c) {
      mbar_wait(raw_empty + 8u * s, ph ^ 1);
      load_raw_stage(smem_u32(raw_buf + (size_t)s * p.raw_bytes), p.R4, x + ((long long)b * C + c * KC) * p.T, p.T, start, end,
                     start - ts0, raw_full + 8u * s, lane);
      __syncwarp();
      if (++s == p.ns) { s = 0; ph ^= 1; }
    }
  }
}

// h = lrelu(acc + b1) of the warpgroup's conv rows [row_base, row_base + 64 MT) (time th0 + r for fragment row r) as
// conv2's operand image; rows outside [0, T) are conv2's zero padding (EXT: rows outside the signal's [lo, hi))
template <int MT, int NB16, bool EXT = false>
__device__ __forceinline__ void rb_write_h(const float* acc, unsigned char* h_buf, const RbK& p, int row_base, int th0,
                                           const float* bias1, int lane, int wq, int lo = 0, int hi = 0) {
  constexpr int NACC = 8 * NB16;
#pragma unroll
  for (int e = 0; e < MT * NACC; e += 2) {
    const int i = e % NACC;
    const int col = 8 * (i >> 2) + 2 * (lane & 3);
    const int r = (e / NACC) * 64 + wq * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
    bool ok;
    if constexpr (EXT)
      ok = th0 + r >= lo && th0 + r < hi;
    else
      ok = (unsigned)(th0 + r) < (unsigned)p.T;
    const float h0 = acc[e] + bias1[col], h1 = acc[e + 1] + bias1[col + 1];
    unsigned hi, lo;
    split2(ok ? lrelu(h0, p.slope) : 0.f, ok ? lrelu(h1, p.slope) : 0.f, hi, lo);
    unsigned char* hc = h_buf + (size_t)(col >> 5) * p.h_bytes;
    const size_t off = ((size_t)((col & 31) >> 3) * p.Rh + row_base + r) * 16 + (col & 7) * 2;
    *reinterpret_cast<unsigned*>(hc + off) = hi;
    *reinterpret_cast<unsigned*>(hc + (size_t)(KC / 8) * p.Rh * 16 + off) = lo;
  }
}

// staged epilogue in place over the residual rows of the tile `stg` ([channel][stage_ld(MT)]): v = (a + b2 + x) * out_scale
// (EXT: +0.0 in the tile rows outside [lo, hi), relative to the tile's first row)
template <int MT, int NB16, bool EXT = false>
__device__ __forceinline__ void rb_stage_result(const float* acc, float* stg, const float* bias2, float out_scale, int lane,
                                                int wq, int lo = 0, int hi = 0) {
  constexpr int NACC = 8 * NB16, SLD = stage_ld(MT);
#pragma unroll
  for (int e = 0; e < MT * NACC; ++e) {
    const int i = e % NACC;
    const int col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
    const int r = (e / NACC) * 64 + wq * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
    float* sv = stg + col * SLD + r;
    float v = acc[e] + bias2[col];
    v += *sv;
    if constexpr (EXT) {
      if (r < lo || r >= hi) {
        *sv = 0.f;
        continue;
      }
    }
    *sv = v * out_scale;
  }
}

// Conv split by warpgroup.  MT = TT / 64: the 64-row blocks of a whole tile, run by one warpgroup (independent
// accumulator chains: 2 at 64 channels, 4 at 32, 64 accumulator registers either way).  Warpgroup 0 runs conv1 of tile
// i + 1 while warpgroup 1 runs conv2 and the epilogue of tile i; they hand the single h image over through two
// mbarriers (H_FULL: written, H_FREE: conv2's MMAs have retired).  Weights come in two rings of nb / 2 stages, conv1's
// and conv2's, both filled by the weight warp.  The residual rows belong to conv2's warpgroup.
// EXT: the mask of RbKExt in the h write and the staged epilogue.
template <int MT, int NB16, bool EXT>
__device__ __forceinline__ void rb_pair_split_body(const std::conditional_t<EXT, RbKExt, RbK>& p, const float* __restrict__ x,
                                                   const unsigned char* __restrict__ w1, const float* __restrict__ b1,
                                                   const unsigned char* __restrict__ w2, const float* __restrict__ b2,
                                                   float* __restrict__ y) {
  extern __shared__ __align__(128) unsigned char smem[];
  constexpr int C = 16 * NB16, NCH = C / KC, NACC = 8 * NB16, SLD = stage_ld(MT);
  const int nr = p.nb / 2;  // stages per weight ring
  // layout: A[na] | B1[nr] | B2[nr] | raw staging[ns] | h image[NCH chunks] | epilogue tile | barriers | bias1 | bias2
  unsigned char* a_buf = smem;
  unsigned char* b1_buf = a_buf + (size_t)p.na * p.a_bytes;
  unsigned char* b2_buf = b1_buf + (size_t)nr * p.b_bytes;
  unsigned char* raw_buf = b2_buf + (size_t)nr * p.b_bytes;
  unsigned char* h_buf = raw_buf + (size_t)p.ns * p.raw_bytes;
  float* stg = reinterpret_cast<float*>(h_buf + (size_t)NCH * p.h_bytes);
  unsigned long long* bars = reinterpret_cast<unsigned long long*>(stg + C * SLD);
  const int nbar = 2 * p.na + 2 * p.nb + 2 * p.ns + 3;
  float* bias_s = reinterpret_cast<float*>(bars + nbar);  // b1 | b2 (zeros for a missing bias)

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;

  const unsigned bar0 = smem_u32(bars);
  const unsigned A_FULL = bar0, A_EMPTY = A_FULL + 8u * p.na;
  const unsigned B1_FULL = A_EMPTY + 8u * p.na, B1_EMPTY = B1_FULL + 8u * nr;
  const unsigned B2_FULL = B1_EMPTY + 8u * nr, B2_EMPTY = B2_FULL + 8u * nr;
  const unsigned RAW_FULL = B2_EMPTY + 8u * nr, RAW_EMPTY = RAW_FULL + 8u * p.ns;
  const unsigned RES_FULL = RAW_EMPTY + 8u * p.ns, H_FULL = RES_FULL + 8u, H_FREE = H_FULL + 8u;

  if (tid == 0) {
    for (int i = 0; i < p.na; ++i) {
      mbar_init(A_FULL + 8u * i, RB_NPROD);
      mbar_init(A_EMPTY + 8u * i, 4);  // the warps of conv1's warpgroup
    }
    for (int i = 0; i < nr; ++i) {
      mbar_init(B1_FULL + 8u * i, 1);
      mbar_init(B1_EMPTY + 8u * i, 4);
      mbar_init(B2_FULL + 8u * i, 1);
      mbar_init(B2_EMPTY + 8u * i, 4);
    }
    for (int i = 0; i < p.ns; ++i) {
      mbar_init(RAW_FULL + 8u * i, 1);
      mbar_init(RAW_EMPTY + 8u * i, RB_NPROD);
    }
    mbar_init(RES_FULL, C);  // one arrival per channel row of the tile
    mbar_init(H_FULL, 128);
    mbar_init(H_FREE, 128);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = tid; i < 2 * C; i += RB_THREADS) {
    const float* bb = i < C ? b1 : b2;
    bias_s[i] = bb ? __ldg(bb + (i < C ? i : i - C)) : 0.f;
  }
  // conv2 rows >= M2 read the h rows [64 MT, Rh) that no tile writes: keep them zero
  for (int i = tid; i < NCH * p.h_bytes / 16; i += RB_THREADS) reinterpret_cast<uint4*>(h_buf)[i] = make_uint4(0, 0, 0, 0);
  fence_proxy_async();
  __syncthreads();

  if (warp < 4) {
    // ===================== conv1: staged x rows -> h image =====================
    // One wgmma group per (chunk, tap), kept in flight while the next is issued, as in conv1d_tc_kernel.
    const int wq = warp & 3;
    const unsigned lbo_a = (unsigned)p.R1 * 16u, a_sub = (unsigned)(KC / 8) * p.R1;
    int buf = 0, aph = 0, s = 0, bph = 0, n = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++n) {
      float acc[MT * NACC];
#pragma unroll
      for (int e = 0; e < MT * NACC; ++e) acc[e] = 0.f;
      int held_s = -1, held_a = -1;  // weight stage / A buffer read by the group in flight
      auto release = [&]() {
        __syncwarp();
        if (lane == 0) {
          if (held_s >= 0) mbar_arrive(B1_EMPTY + 8u * held_s);
          if (held_a >= 0) mbar_arrive(A_EMPTY + 8u * held_a);
        }
      };
      for (int c = 0; c < NCH; ++c) {
        mbar_wait_trap(A_FULL + 8u * buf, aph);
        const unsigned a_addr = smem_u32(a_buf + (size_t)buf * p.a_bytes);
        for (int k = 0; k < p.K; ++k) {
          mbar_wait_trap(B1_FULL + 8u * s, bph);
          __syncwarp();
          mma_stage<MT, NB16>(acc, a_addr, lbo_a, a_sub, k * p.D, smem_u32(b1_buf + (size_t)s * p.b_bytes));
          wg_wait<1>();  // the previous group has retired: its stage and, at a chunk boundary, its A buffer are free
          release();
          held_s = s;
          held_a = k == p.K - 1 ? buf : -1;
          if (++s == nr) { s = 0; bph ^= 1; }
        }
        if (++buf == p.na) { buf = 0; aph ^= 1; }
      }
      wg_wait<0>();
      release();
      mbar_wait_trap(H_FREE, (n & 1) ^ 1);  // conv2 of the previous tile has read the image
      const int t0 = (tile % p.tiles_per_seq) * p.M2;
      if constexpr (EXT) {
        int lo, hi;
        rb_signal_rows(p, tile / p.tiles_per_seq, lo, hi);
        rb_write_h<MT, NB16, true>(acc, h_buf, p, 0, t0 - p.p2, bias_s, lane, wq, lo, hi);
      } else {
        rb_write_h<MT, NB16>(acc, h_buf, p, 0, t0 - p.p2, bias_s, lane, wq);
      }
      fence_proxy_async();  // generic-proxy smem writes -> visible to the tensor core
      mbar_arrive(H_FULL);
    }
  } else if (warp < 8) {
    // ===================== conv2 on the h image, staged epilogue =====================
    const int wq = warp & 3;
    const unsigned lbo_h = (unsigned)p.Rh * 16u, h_sub = (unsigned)(KC / 8) * p.Rh;
    // thread wt of the warpgroup owns channel row wt of the tile (residual in, result out)
    const int wt = tid - 128;
    const bool row_owner = wt < C;
    // channel row wt of a tile's output rows: first element and bytes (below M2 and T)
    auto row_pos = [&](int tile, unsigned& row_bytes) -> long long {
      const int b = tile / p.tiles_per_seq;
      const int t0 = (tile - b * p.tiles_per_seq) * p.M2;
      const int nrow = p.M2 < p.T - t0 ? p.M2 : p.T - t0;
      row_bytes = nrow > 0 ? 4u * (unsigned)nrow : 0u;
      return ((long long)b * C + wt) * p.T + t0;
    };
    // the residual (x itself) of a tile, issued at the end of the previous tile's epilogue so that it streams in while
    // this tile's MMAs run
    auto load_res = [&](int tile) {
      unsigned row_bytes;
      const long long off = row_pos(tile, row_bytes);
      stage_load_row(smem_u32(stg + wt * SLD), x + off, row_bytes, RES_FULL);
    };
    if (row_owner && (int)blockIdx.x < p.total_tiles) load_res(blockIdx.x);
    int s = 0, bph = 0, n = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++n) {
      float acc[MT * NACC];
#pragma unroll
      for (int e = 0; e < MT * NACC; ++e) acc[e] = 0.f;
      int held_s = -1;
      auto release = [&]() {
        __syncwarp();
        if (lane == 0 && held_s >= 0) mbar_arrive(B2_EMPTY + 8u * held_s);
      };
      mbar_wait_trap(H_FULL, n & 1);
      for (int c = 0; c < NCH; ++c) {
        const unsigned h_addr = smem_u32(h_buf + (size_t)c * p.h_bytes);
        for (int k = 0; k < p.K; ++k) {
          mbar_wait_trap(B2_FULL + 8u * s, bph);
          __syncwarp();
          mma_stage<MT, NB16>(acc, h_addr, lbo_h, h_sub, k, smem_u32(b2_buf + (size_t)s * p.b_bytes));
          wg_wait<1>();
          release();
          held_s = s;
          if (++s == nr) { s = 0; bph ^= 1; }
        }
      }
      wg_wait<0>();
      release();
      mbar_arrive(H_FREE);
      // ---- staged epilogue over the residual row, one bulk store (or fp32 add) per row
      mbar_wait_trap(RES_FULL, n & 1);  // one phase per tile
      if constexpr (EXT) {
        const int b = tile / p.tiles_per_seq, t0 = (tile - b * p.tiles_per_seq) * p.M2;
        int lo, hi;
        rb_signal_rows(p, b, lo, hi);
        rb_stage_result<MT, NB16, true>(acc, stg, bias_s + C, p.out_scale, lane, wq, lo - t0, hi - t0);
      } else {
        rb_stage_result<MT, NB16>(acc, stg, bias_s + C, p.out_scale, lane, wq);
      }
      fence_proxy_async();  // generic-proxy writes -> visible to the bulk copies
      wg_barrier(1);
      if (row_owner) {
        unsigned row_bytes;
        const long long off = row_pos(tile, row_bytes);
        stage_store_row(y + off, smem_u32(stg + wt * SLD), row_bytes, p.accumulate);
        if (tile + (int)gridDim.x < p.total_tiles) load_res(tile + gridDim.x);
      }
    }
    if (row_owner) bulk_wait();  // the shared-memory source must outlive the CTA's last stores
  } else if (warp < RB_W_TMA) {
    rb_convert_x<NCH>(p, a_buf, raw_buf, A_FULL, A_EMPTY, RAW_FULL, RAW_EMPTY, tid - 32 * RB_W_PROD0);
  } else if (warp == RB_W_TMA) {
    // ===================== weight stages: both rings, NCH * K stages per tile each =====================
    // The two convs run different tiles, so one lane polls both rings and fills whichever has a free stage.
    if (lane == 0) {
      const int per = NCH * p.K;
      const int ntiles = (int)blockIdx.x < p.total_tiles ? (p.total_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
      int n1 = 0, j1 = 0, s1 = 0, ph1 = 0, n2 = 0, j2 = 0, s2 = 0, ph2 = 0;
      unsigned idle = 0;
      while (n1 < ntiles || n2 < ntiles) {
        bool moved = false;
        if (n1 < ntiles && mbar_try(B1_EMPTY + 8u * s1, ph1 ^ 1)) {
          mbar_expect_tx(B1_FULL + 8u * s1, (unsigned)p.b_bytes);
          bulk_g2s(smem_u32(b1_buf + (size_t)s1 * p.b_bytes), w1 + (size_t)j1 * p.b_bytes, (unsigned)p.b_bytes, B1_FULL + 8u * s1);
          if (++j1 == per) { j1 = 0; ++n1; }
          if (++s1 == nr) { s1 = 0; ph1 ^= 1; }
          moved = true;
        }
        if (n2 < ntiles && mbar_try(B2_EMPTY + 8u * s2, ph2 ^ 1)) {
          mbar_expect_tx(B2_FULL + 8u * s2, (unsigned)p.b_bytes);
          bulk_g2s(smem_u32(b2_buf + (size_t)s2 * p.b_bytes), w2 + (size_t)j2 * p.b_bytes, (unsigned)p.b_bytes, B2_FULL + 8u * s2);
          if (++j2 == per) { j2 = 0; ++n2; }
          if (++s2 == nr) { s2 = 0; ph2 ^= 1; }
          moved = true;
        }
        if (moved) idle = 0;
        else if (++idle > SPIN_LIMIT) __trap();
      }
    }
  } else if (warp == RB_W_LDA) {
    rb_load_raw<NCH>(p, x, raw_buf, RAW_FULL, RAW_EMPTY, lane);
  }
}

template <int MT, int NB16>
__global__ void __launch_bounds__(RB_THREADS, 1)
    rb_pair_split_kernel(const RbK p, const float* __restrict__ x, const unsigned char* __restrict__ w1,
                         const float* __restrict__ b1, const unsigned char* __restrict__ w2, const float* __restrict__ b2,
                         float* __restrict__ y) {
  rb_pair_split_body<MT, NB16, false>(p, x, w1, b1, w2, b2, y);
}

// the masked pair (pwgb_resblock_pair_ext_forward)
template <int MT, int NB16>
__global__ void __launch_bounds__(RB_THREADS, 1)
    rb_pair_split_ext_kernel(const RbKExt p, const float* __restrict__ x, const unsigned char* __restrict__ w1,
                             const float* __restrict__ b1, const unsigned char* __restrict__ w2, const float* __restrict__ b2,
                             float* __restrict__ y) {
  rb_pair_split_body<MT, NB16, true>(p, x, w1, b1, w2, b2, y);
}

using RbKernel = void (*)(const RbK, const float*, const unsigned char*, const float*, const unsigned char*, const float*,
                          float*);
using RbKernelExt = void (*)(const RbKExt, const float*, const unsigned char*, const float*, const unsigned char*,
                             const float*, float*);

// Instantiations: 256-row tiles at 32 channels, 128-row tiles at 64 channels (mt: 64-row blocks of a tile)
RbKernel rb_split_kernel_for(int channels, int* mt) {
  *mt = channels == 32 ? 4 : 2;
  if (channels == 32) return rb_pair_split_kernel<4, 2>;
  if (channels == 64) return rb_pair_split_kernel<2, 4>;
  return nullptr;
}
RbKernelExt rb_split_ext_kernel_for(int channels) {
  if (channels == 32) return rb_pair_split_ext_kernel<4, 2>;
  if (channels == 64) return rb_pair_split_ext_kernel<2, 4>;
  return nullptr;
}

// Tile geometry at `mt` and the first (na, ns) that leaves RB_MIN_STAGES weight stages in each of the two rings: two
// conv1 operand buffers with three, then two raw stages; then, with one 32-channel chunk, one operand buffer (the
// producers then convert the next tile while conv2 runs).
int rb_fit(const pwgb_resblock_desc* d, RbK& p, size_t& smem_bytes, int mt) {
  const int tt = 64 * mt;
  const long long halo1 = (long long)(d->kernel - 1) * d->dilation;
  p.MT = mt;
  p.M2 = (tt - (d->kernel - 1)) & ~3;
  p.R1 = tt + (int)halo1;
  p.R4 = (p.R1 + 6) & ~3;
  p.Rh = tt + d->kernel - 1;
  p.a_bytes = 2 * (KC / 8) * p.R1 * 16;
  p.raw_bytes = KC * p.R4 * 4;
  p.h_bytes = 2 * (KC / 8) * p.Rh * 16;
  const size_t epi = (size_t)d->channels * stage_ld(mt) * 4;
  const size_t fixed = (size_t)p.nchunks * p.h_bytes + epi + 2 * (size_t)d->channels * 4 + 1024;
  static const int bufs[3][2] = {{2, 3}, {2, 2}, {1, 2}};  // (na, ns)
  for (const auto& nn : bufs) {
    const int na = nn[0], ns = nn[1];
    if (na < p.nchunks) continue;  // one operand buffer only for a single chunk
    const size_t used = fixed + (size_t)na * p.a_bytes + (size_t)ns * p.raw_bytes;
    if (used + (size_t)2 * RB_MIN_STAGES * p.b_bytes > RB_SMEM) continue;
    int nb = (int)((RB_SMEM - used) / p.b_bytes);
    if (nb > 24) nb = 24;
    nb -= nb % 2;  // two rings of nb / 2 stages
    p.na = na;
    p.nb = nb;
    p.ns = ns;
    p.tiles_per_seq = ceil_div(d->t, p.M2);
    if ((long long)p.tiles_per_seq * d->batch > 0x7fffffffLL) return 0;
    p.total_tiles = p.tiles_per_seq * d->batch;
    smem_bytes = (size_t)na * p.a_bytes + (size_t)nb * p.b_bytes + (size_t)ns * p.raw_bytes + (size_t)p.nchunks * p.h_bytes +
                 epi + 8 * (size_t)(2 * na + 2 * nb + 2 * ns + 3) + 2 * (size_t)d->channels * 4;
    return 1;
  }
  return 0;
}

// Plan of one pair, or 0 when the pair has none (other channel counts, ragged T, a conv1 halo too wide for rb_fit): the
// caller then runs the two conv1d_tc launches.
int rb_plan(const pwgb_resblock_desc* d, RbK& p, size_t& smem_bytes) {
  if (!d || d->batch < 0 || d->t <= 0 || d->kernel < 1 || d->kernel % 2 == 0 || d->dilation < 1) return 0;
  int mt = 0;
  if (!rb_split_kernel_for(d->channels, &mt)) return 0;
  if (d->t % 4 != 0) return 0;  // 16-byte rows for the bulk copies of x and y
  const long long halo1 = (long long)(d->kernel - 1) * d->dilation;
  if (d->kernel - 1 > 64 || halo1 > 2048) return 0;
  p.B = d->batch;
  p.C = d->channels;
  p.T = d->t;
  p.K = d->kernel;
  p.D = d->dilation;
  p.slope = d->slope;
  p.out_scale = d->out_scale;
  p.accumulate = d->accumulate;
  p.p1 = (d->kernel - 1) / 2 * d->dilation;
  p.p2 = (d->kernel - 1) / 2;
  p.nchunks = d->channels / KC;
  p.b_bytes = 2 * (KC / 8) * d->channels * 16;
  return rb_fit(d, p, smem_bytes, mt);
}

}  // namespace

}  // namespace pwgb

using namespace pwgb;

extern "C" int pwgb_resblock_pair_supported(const pwgb_resblock_desc* d) {
  RbK p;
  size_t bytes;
  return rb_plan(d, p, bytes);
}

extern "C" int pwgb_resblock_pair_plan(const pwgb_resblock_desc* d, int* info) {
  RbK p;
  size_t bytes;
  if (!info || !rb_plan(d, p, bytes)) return 0;
  const int v[5] = {p.M2, 64 * p.MT, p.na, p.nb, p.ns};
  memcpy(info, v, sizeof(v));
  return 1;
}

extern "C" int pwgb_resblock_pair_ext_forward(const pwgb_resblock_desc* d, const float* x, const void* w1_packed,
                                              const float* b1, const void* w2_packed, const float* b2,
                                              const pwgb_stream_ext* ext, float* y, void* stream) {
  if (!ext) return pwgb_resblock_pair_forward(d, x, w1_packed, b1, w2_packed, b2, y, stream);
  PWGB_CHECK_ARG(d && x && w1_packed && w2_packed && y, "resblock_pair_ext: null argument");
  PWGB_CHECK_ARG(ext->frame && ext->end && ext->rate >= 1 && ext->lookahead >= 0,
                 "resblock_pair_ext: ext must hold a mask (frame, end, rate >= 1, lookahead >= 0)");
  RbKExt p;
  size_t bytes = 0;
  PWGB_UNSUPPORTED_IF(!rb_plan(d, p, bytes), "resblock_pair_ext: configuration not supported by the fused kernel");
  PWGB_CHECK_ARG(x != y, "resblock_pair_ext: y must not alias x (halo reads)");
  PWGB_UNSUPPORTED_IF((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15),
                      "resblock_pair_ext: x and y must be 16-byte aligned");
  if (p.B == 0) return PWGB_OK;
  p.mframe = ext->frame;
  p.mend = ext->end;
  p.mrate = ext->rate;
  p.mlook = ext->lookahead;
  static bool smem_set = false;
  if (const int rc = smem_opt_in(smem_set, {rb_split_ext_kernel_for(32), rb_split_ext_kernel_for(64)}, (int)RB_SMEM,
                                 "resblock_pair_ext"))
    return rc;
  const int num_sms = tc_num_sms();
  const int grid = p.total_tiles < num_sms ? p.total_tiles : num_sms;
  rb_split_ext_kernel_for(p.C)<<<(unsigned)grid, RB_THREADS, bytes, (cudaStream_t)stream>>>(
      p, x, (const unsigned char*)w1_packed, b1, (const unsigned char*)w2_packed, b2, y);
  return check_launch("rb_pair_split_ext_kernel");
}

extern "C" int pwgb_resblock_pair_forward(const pwgb_resblock_desc* d, const float* x, const void* w1_packed,
                                          const float* b1, const void* w2_packed, const float* b2, float* y,
                                          void* stream) {
  PWGB_CHECK_ARG(d && x && w1_packed && w2_packed && y, "resblock_pair: null argument");
  RbK p;
  size_t bytes = 0;
  PWGB_UNSUPPORTED_IF(!rb_plan(d, p, bytes), "resblock_pair: configuration not supported by the fused kernel");
  PWGB_CHECK_ARG(x != y, "resblock_pair: y must not alias x (halo reads)");
  PWGB_UNSUPPORTED_IF((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15),
                      "resblock_pair: x and y must be 16-byte aligned");
  if (p.B == 0) return PWGB_OK;
  int mt;
  static bool smem_set = false;
  if (const int rc = smem_opt_in(smem_set, {rb_split_kernel_for(32, &mt), rb_split_kernel_for(64, &mt)}, (int)RB_SMEM,
                                 "resblock_pair"))
    return rc;
  const int num_sms = tc_num_sms();
  const int grid = p.total_tiles < num_sms ? p.total_tiles : num_sms;
  const RbKernel k = rb_split_kernel_for(p.C, &mt);
  k<<<(unsigned)grid, RB_THREADS, bytes, (cudaStream_t)stream>>>(p, x, (const unsigned char*)w1_packed, b1,
                                                                 (const unsigned char*)w2_packed, b2, y);
  return check_launch("rb_pair_split_kernel");
}
