// Fused WaveNet residual layer (layers/residual_block.py:102-140) for the Parallel WaveGAN residual
// stack (models/parallel_wavegan.py:161-166): ONE wgmma kernel per layer, fed by TMA.
//
//   g  = conv_{k, dil}(x) + W_aux c + b          G accumulator columns in the registers of the consumer warpgroups
//   z  = tanh(g[:H]) * sigmoid(g[H:])            registers -> bf16 hi/lo operand image in smem (per warpgroup)
//   so = [W_skip ; W_out] z                      second contraction into the same registers (G is dead by then)
//   skips (+)= so[:S] + b_skip ;  x' = (so[S:] + b_out + x) * sqrt(1/2)
//
// Algorithmic HBM bytes per sample and layer: x 4R + c 4A + x' 4R + skips 8S = 1344 B for PWG v1
// (SURVEY.md 8d) -- the gate tensor never leaves the SM.
//
// Data layout: between layers the residual stream and the conditioning live in HBM in the tensor core's
// operand layout, split bf16 hi/lo (the same bytes per sample as fp32):
//   xpk [batch][hi|lo][R/8][t_pad][8 ch] bf16,  t_pad = 2*halo + round_up(t, 256); rows [halo, halo + t) hold
//       the samples, every other row is zero (the conv's zero padding and the tail of the last tile);
//   cpk [batch][hi|lo][ceil(A/8)][round_up(t, 256)][8 ch] bf16.
// A (32 channel, 128 row) operand window of any tap / dilation is then a 3-D box of the packed tensor (planes described
// as vectors of 8-byte elements: 2 KB inner extent): the activation side of a pipeline stage is one cp.async.bulk.tensor
// (TMA), the weight side one bulk copy, and no thread ever converts or re-lays-out an input (the conversion happens
// once, in the epilogue that produces the value).  x = hi + lo carries 16 mantissa bits -- exactly what the bf16x3 MMA
// consumes; the residual add sees the same value.
//
// Warp roles (288 threads, one persistent CTA per SM, work item = one 128-sample tile, mbarriers between the roles):
//   warps 0-7   two consumer warpgroups; warpgroup g owns rows [64 g, 64 g + 64) of the tile: conv wgmma per ring
//               stage, gate in registers, z image, skip / out wgmma on the resident weights, epilogue stores
//   warp  8     TMA loader: per stage one tensor-map load (the tile's activation window) + one bulk copy of the
//               weight stage into a ring of 32 KB slots; the skip / out weights stay resident in shared memory
#include "tc_common.cuh"
#include "tma.cuh"

namespace pwgb {

constexpr int WN_TT = 128;                 // rows (samples) per tile
constexpr int WN_NCONS = 256;              // two consumer warpgroups
constexpr int WN_W_TMA = WN_NCONS / 32;
constexpr int WN_THREADS = WN_NCONS + 32;
constexpr int WN_MAX_SLOTS = 8;
constexpr int WN_BLK = WN_TT * 16;         // one (8 channel, 128 row) operand block: 2 KB

struct WnK {
  int B, T, R, G, S, A, K, D, halo;
  int H;                 // gate output channels = G / 2
  int Tp, Tc;            // rows per plane of xpk / cpk
  int ngx, ngc;          // 8-channel groups of x / c
  int nxc, ncc, nsc;     // 32-channel chunks of x, c and z
  int N2;                // S + R
  int tiles_per_seq, total_tiles;
  int nslot, a_bytes, b_bytes, slot_bytes, z_bytes, wso_bytes;
  int write_x, skip_init;
};

__device__ __forceinline__ float ex2_approx(float v) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v));
  return r;
}
// tanh(a) * sigmoid(b) = (Ea - 1) / ((Ea + 1)(1 + Eb)), Ea = e^{2a}, Eb = e^{-b}: two ex2 and one rcp.
// Absolute error ~3e-7 (ex2.approx: 2^-22 relative).  The accumulators arrive without bias; the biases are pre-scaled
// (ba = 2 log2(e) b_a, bb = -log2(e) b_b) so that one FFMA per operand produces the ex2 argument.  Only a needs a clamp
// (Ea = inf would give inf * 0); b -> -inf gives Eb = inf and the quotient 0, the correct limit.
__device__ __forceinline__ float gate_fast(float ga, float gb, float ba, float bb) {
  const float a2 = fminf(fmaf(ga, 2.8853900817779268f, ba), 43.28f);
  const float ea = ex2_approx(a2);
  const float eb = ex2_approx(fmaf(gb, -1.4426950408889634f, bb));
  return __fdividef(ea - 1.f, (ea + 1.f) * (1.f + eb));
}

__device__ __forceinline__ void bf16x8_to_float(const uint4& v, float (&f)[8]) {
  const unsigned u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    f[2 * i] = __uint_as_float(u[i] << 16);
    f[2 * i + 1] = __uint_as_float(u[i] & 0xFFFF0000u);
  }
}
// two floats -> packed bf16 hi pair and lo pair (the residual of the hi rounding)
__device__ __forceinline__ void split2(float a, float b, unsigned& hi, unsigned& lo) {
  __nv_bfloat162 hh = __floats2bfloat162_rn(a, b);
  const float2 hf = __bfloat1622float2(hh);
  __nv_bfloat162 ll = __floats2bfloat162_rn(a - hf.x, b - hf.y);
  hi = *reinterpret_cast<unsigned*>(&hh);
  lo = *reinterpret_cast<unsigned*>(&ll);
}

// z = gate(g) of this thread's accumulator fragment into the warpgroup's z image [hi|lo][H/8][64 rows][8] bf16.
// HH = H / 2 registers separate gate column c from its partner c + H (H is a multiple of 32).
template <int HH>
__device__ __forceinline__ void gate_to_z(const float* acc, const float* bias1, int H, int lane, int wq, unsigned char* zw) {
#pragma unroll
  for (int e = 0; e < HH; e += 2) {
    const int col = 8 * (e >> 2) + 2 * (lane & 3);
    const int row = wq * 16 + (lane >> 2) + 8 * ((e >> 1) & 1);
    const float z0 = gate_fast(acc[e], acc[e + HH], bias1[col], bias1[H + col]);
    const float z1 = gate_fast(acc[e + 1], acc[e + 1 + HH], bias1[col + 1], bias1[H + col + 1]);
    unsigned hi, lo;
    split2(z0, z1, hi, lo);
    const size_t off = ((size_t)(col >> 3) * 64 + row) * 16 + (col & 7) * 2;
    *reinterpret_cast<unsigned*>(zw + off) = hi;
    *reinterpret_cast<unsigned*>(zw + (size_t)(H / 8) * 64 * 16 + off) = lo;
  }
}

__global__ void __launch_bounds__(WN_THREADS, 1)
    wavenet_fused_kernel(const WnK p, const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_c,
                         const unsigned* __restrict__ xin, const unsigned char* __restrict__ wpk, const float* __restrict__ b_conv,
                         const float* __restrict__ b_so, unsigned* __restrict__ xout, float* __restrict__ skips) {
  extern __shared__ __align__(128) unsigned char smem[];
  // layout: ring[nslot] (A 16 KB | B) | resident skip/out weights | z images (one per warpgroup) | barriers | bias
  unsigned char* ring = smem;
  unsigned char* wso_buf = smem + (size_t)p.nslot * p.slot_bytes;
  unsigned char* z_buf = wso_buf + p.wso_bytes;
  unsigned long long* bars = reinterpret_cast<unsigned long long*>(z_buf + 2 * p.z_bytes);
  constexpr int NBAR = 2 * WN_MAX_SLOTS + 2;
  float* bias1 = reinterpret_cast<float*>(bars + NBAR);
  float* bias2 = bias1 + p.G;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const unsigned bar0 = smem_u32(bars);
  auto FULL = [&](int i) { return bar0 + 8u * i; };
  auto EMPTY = [&](int i) { return bar0 + 8u * (WN_MAX_SLOTS + i); };
  const unsigned WSO_FULL = bar0 + 8u * (2 * WN_MAX_SLOTS);

  if (tid == 0) {
    for (int i = 0; i < p.nslot; ++i) {
      mbar_init(FULL(i), 1);
      mbar_init(EMPTY(i), WN_NCONS / 32);  // one arrival per consumer warp
    }
    mbar_init(WSO_FULL, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  const int H = p.H, S = p.S;
  // biases, pre-scaled for their consumers: gate a-half by 2 log2(e), b-half by -log2(e)
  for (int i = tid; i < p.G; i += WN_THREADS) bias1[i] = (b_conv ? __ldg(b_conv + i) : 0.f) * (i < H ? 2.8853900817779268f : -1.4426950408889634f);
  for (int i = tid; i < p.N2; i += WN_THREADS) bias2[i] = b_so ? __ldg(b_so + i) : 0.f;
  __syncthreads();

  const int ntiles = ((int)p.total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const int conv_stages = p.nxc * p.K + p.ncc;
  const unsigned char* w_aux = wpk + (size_t)p.nxc * p.K * p.b_bytes;
  const unsigned char* w_so = w_aux + (size_t)p.ncc * p.b_bytes;

  if (warp == WN_W_TMA) {
    // ===================== TMA loader: activation windows + weight stages
    if (lane == 0) {
      tma_prefetch_desc(&tm_x);
      tma_prefetch_desc(&tm_c);
      // skip / out weights stay resident for the whole kernel
      mbar_expect_tx(WSO_FULL, (unsigned)p.wso_bytes);
      for (int sc = 0; sc < p.nsc; ++sc)
        bulk_g2s(smem_u32(wso_buf) + (unsigned)(sc * p.b_bytes), w_so + (size_t)sc * p.b_bytes, (unsigned)p.b_bytes, WSO_FULL);
    }
    int s = 0, ph = 0;
    for (int n = 0; n < ntiles; ++n) {
      const int tile = blockIdx.x + n * gridDim.x;
      const int b = tile / p.tiles_per_seq;
      const int t0 = (tile - b * p.tiles_per_seq) * WN_TT;
      for (int j = 0; j < conv_stages; ++j) {
        const bool is_x = j < p.nxc * p.K;
        const int chunk = is_x ? j / p.K : j - p.nxc * p.K;
        const int tap = is_x ? j - chunk * p.K : 0;
        mbar_wait_spin(EMPTY(s), ph ^ 1);
        if (lane == 0) {
          // box (128 rows x 16 B as 256 8-byte elements, 4 groups, hi|lo) = a 16 KB operand image; groups beyond the tensor
          // (last conditioning chunk) arrive as zeros and count towards the transaction bytes
          const unsigned dstA = smem_u32(ring + (size_t)s * p.slot_bytes);
          const unsigned full = FULL(s);
          mbar_expect_tx(full, (unsigned)(p.a_bytes + p.b_bytes));
          if (is_x)
            tma_load_3d(dstA, &tm_x, 2 * (p.halo + t0 + (tap - p.K / 2) * p.D), chunk * 4, 2 * b, full);
          else
            tma_load_3d(dstA, &tm_c, 2 * t0, chunk * 4, 2 * b, full);
          const unsigned char* wsrc = is_x ? wpk + (size_t)j * p.b_bytes : w_aux + (size_t)chunk * p.b_bytes;
          bulk_g2s(dstA + (unsigned)p.a_bytes, wsrc, (unsigned)p.b_bytes, full);
        }
        __syncwarp();
        if (++s == p.nslot) { s = 0; ph ^= 1; }
      }
    }
  } else {
    // ===================== consumers =====================
    const int wg = warp >> 2, wq = warp & 3;
    const int nbg = p.G / 16, nbo = p.N2 / 16;
    const int cgl = p.ngc - (p.ncc - 1) * 4;  // 8-channel groups of the last conditioning chunk
    const unsigned a_sub = (unsigned)(4 * WN_BLK) >> 4, a_step = (unsigned)(2 * WN_BLK) >> 4;  // hi -> lo, second K-step
    const unsigned b1_sub = 4u * p.G, b1_step = 2u * p.G;
    const unsigned b2_sub = 4u * p.N2, b2_step = 2u * p.N2;
    unsigned char* zw = z_buf + (size_t)wg * p.z_bytes;
    const unsigned z_addr = smem_u32(zw), wso_addr = smem_u32(wso_buf);
    const unsigned z_sub = (unsigned)((H / 8) * 64 * 16) >> 4, z_step = (unsigned)(2 * 64 * 16) >> 4;
    const float rs = 0.70710678118654752440f;
    mbar_wait_spin(WSO_FULL, 0);
    int s = 0, ph = 0;
    for (int n = 0; n < ntiles; ++n) {
      const int tile = blockIdx.x + n * gridDim.x;
      const int b = tile / p.tiles_per_seq;
      const int t0 = (tile - b * p.tiles_per_seq) * WN_TT;
      float acc[64];
#pragma unroll
      for (int e = 0; e < 64; ++e) acc[e] = 0.f;
      // ---- conv + aux 1x1: one ring stage per (x chunk, tap) and per conditioning chunk
      for (int j = 0; j < conv_stages; ++j) {
        mbar_wait_spin(FULL(s), ph);
        __syncwarp();
        const unsigned s_addr = smem_u32(ring + (size_t)s * p.slot_bytes);
        const unsigned long long ah = gmma_desc(s_addr + (unsigned)(wg * 64 * 16), WN_BLK, 128);
        const unsigned long long bh = gmma_desc(s_addr + (unsigned)p.a_bytes, (unsigned)p.G * 16u, 128);
        const bool half = j >= p.nxc * p.K && (j - p.nxc * p.K) == p.ncc - 1 && cgl <= 2;  // one K-step only
        wg_fence();
        wgmma_cols<0, 0, 8>(acc, ah, bh, nbg, 16);
        wgmma_cols<0, 0, 8>(acc, ah + a_sub, bh, nbg, 16);
        wgmma_cols<0, 0, 8>(acc, ah, bh + b1_sub, nbg, 16);
        if (!half) {
          wgmma_cols<0, 0, 8>(acc, ah + a_step, bh + b1_step, nbg, 16);
          wgmma_cols<0, 0, 8>(acc, ah + a_step + a_sub, bh + b1_step, nbg, 16);
          wgmma_cols<0, 0, 8>(acc, ah + a_step, bh + b1_step + b1_sub, nbg, 16);
        }
        wg_commit();
        wg_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(EMPTY(s));
        if (++s == p.nslot) { s = 0; ph ^= 1; }
      }
      // ---- gate: registers -> z image of this warpgroup, once every warp's skip / out MMAs of the previous tile are done
      wg_barrier(wg);
      if (H == 64)
        gate_to_z<32>(acc, bias1, H, lane, wq, zw);
      else
        gate_to_z<16>(acc, bias1, H, lane, wq, zw);
      fence_proxy_async();
      wg_barrier(wg);
      // ---- skip / out 1x1: so = z x resident weights
#pragma unroll
      for (int e = 0; e < 64; ++e) acc[e] = 0.f;
      wg_fence();
      for (int sc = 0; sc < p.nsc; ++sc) {
        const unsigned long long ah = gmma_desc(z_addr + (unsigned)(sc * 4 * 64 * 16), 64 * 16, 128);
        const unsigned long long bh = gmma_desc(wso_addr + (unsigned)(sc * p.b_bytes), (unsigned)p.N2 * 16u, 128);
        wgmma_cols<0, 0, 8>(acc, ah, bh, nbo, 16);
        wgmma_cols<0, 0, 8>(acc, ah + z_sub, bh, nbo, 16);
        wgmma_cols<0, 0, 8>(acc, ah, bh + b2_sub, nbo, 16);
        wgmma_cols<0, 0, 8>(acc, ah + z_step, bh + b2_step, nbo, 16);
        wgmma_cols<0, 0, 8>(acc, ah + z_step + z_sub, bh + b2_step, nbo, 16);
        wgmma_cols<0, 0, 8>(acc, ah + z_step, bh + b2_step + b2_sub, nbo, 16);
      }
      wg_commit();
      wg_wait<0>();
      // ---- epilogue: skips (+)= so[:S] + b_skip;  x' = (so[S:] + b_out + x) * sqrt(1/2), packed hi/lo
#pragma unroll
      for (int e = 0; e < 64; e += 2) {
        const int col = 8 * (e >> 2) + 2 * (lane & 3);
        if (col >= p.N2) continue;
        const int t = t0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * ((e >> 1) & 1);
        const bool tv = t < p.T;
        if (col < S) {
          if (tv) {
            float* q = skips + ((long long)b * S + col) * p.T + t;
            const float v0 = acc[e] + bias2[col], v1 = acc[e + 1] + bias2[col + 1];
            if (p.skip_init) {
              q[0] = v0;
              q[p.T] = v1;
            } else {
              q[0] = v0 + q[0];
              q[p.T] = v1 + q[p.T];
            }
          }
        } else if (p.write_x) {
          const int ch = col - S;
          // bf16 pair index of (row, channels ch, ch + 1) in the hi plane; the lo plane is ngx planes further
          const long long hi_i = (((long long)(b * 2) * p.ngx + (ch >> 3)) * p.Tp + p.halo + t) * 4 + ((ch & 7) >> 1);
          const long long lo_i = hi_i + (long long)p.ngx * p.Tp * 4;
          unsigned hi = 0, lo = 0;  // rows past the end of the sequence stay zero (the next layer's padding)
          if (tv) {
            float fh[2], fl[2];
            const unsigned xh = __ldg(xin + hi_i), xl = __ldg(xin + lo_i);
            fh[0] = __uint_as_float(xh << 16), fh[1] = __uint_as_float(xh & 0xFFFF0000u);
            fl[0] = __uint_as_float(xl << 16), fl[1] = __uint_as_float(xl & 0xFFFF0000u);
            const float u0 = ((acc[e] + bias2[col]) + fh[0] + fl[0]) * rs;
            const float u1 = ((acc[e + 1] + bias2[col + 1]) + fh[1] + fl[1]) * rs;
            split2(u0, u1, hi, lo);
          }
          xout[hi_i] = hi;
          xout[lo_i] = lo;
        }
      }
    }
  }
}

// ------------------------------------------------------------------ layout helpers (HBM-bound, one pass)
// fp32 (B, C, T) (batch stride bs) -> packed hi/lo planes [b][hl][ng][rows][8]; rows outside [row0, row0 + T) stay
// untouched for `zero_tail == 0`, rows [row0 + T, rows) are zero-filled otherwise (conditioning tail).
__global__ void wn_pack_kernel(const float* __restrict__ x, long long bs, int C, int T, uint4* __restrict__ pk, int ng,
                               int rows, int row0, int zero_tail) {
  const int b = blockIdx.z, g = blockIdx.y;
  const int tlim = zero_tail ? rows - row0 : T;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < tlim; t += gridDim.x * blockDim.x) {
    float u[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int ch = g * 8 + j;
      u[j] = (t < T && ch < C) ? __ldg(x + (long long)b * bs + (long long)ch * T + t) : 0.f;
    }
    uint4 hi, lo;
    split8(u, hi, lo);
    pk[((long long)(b * 2 + 0) * ng + g) * rows + row0 + t] = hi;
    pk[((long long)(b * 2 + 1) * ng + g) * rows + row0 + t] = lo;
  }
}

__global__ void wn_unpack_kernel(const uint4* __restrict__ pk, int ng, int rows, int row0, float* __restrict__ x, int C, int T) {
  const int b = blockIdx.z, g = blockIdx.y;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < T; t += gridDim.x * blockDim.x) {
    float fh[8], fl[8];
    bf16x8_to_float(pk[((long long)(b * 2 + 0) * ng + g) * rows + row0 + t], fh);
    bf16x8_to_float(pk[((long long)(b * 2 + 1) * ng + g) * rows + row0 + t], fl);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (g * 8 + j < C) x[((long long)b * C + g * 8 + j) * T + t] = fh[j] + fl[j];
  }
}

// first_conv (Conv1d1x1 in_channels -> R, parallel_wavegan.py:155) writing the packed residual stream directly
__global__ void wn_first_conv_kernel(const float* __restrict__ z, int cin, const float* __restrict__ w, const float* __restrict__ bias,
                                     int T, uint4* __restrict__ pk, int ng, int rows, int row0) {
  const int b = blockIdx.z, g = blockIdx.y;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < T; t += gridDim.x * blockDim.x) {
    float u[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) u[j] = bias ? __ldg(bias + g * 8 + j) : 0.f;
    for (int ci = 0; ci < cin; ++ci) {
      const float zv = __ldg(z + ((long long)b * cin + ci) * T + t);
#pragma unroll
      for (int j = 0; j < 8; ++j) u[j] = fmaf(__ldg(w + (long long)(g * 8 + j) * cin + ci), zv, u[j]);
    }
    uint4 hi, lo;
    split8(u, hi, lo);
    pk[((long long)(b * 2 + 0) * ng + g) * rows + row0 + t] = hi;
    pk[((long long)(b * 2 + 1) * ng + g) * rows + row0 + t] = lo;
  }
}


static int wn_plan(const pwgb_wnstack_desc* d, WnK& p, size_t& smem_bytes) {
  if (!d || d->batch < 0 || d->t <= 0 || d->kernel <= 0 || d->kernel % 2 == 0 || d->halo < 0) return 0;
  const int R = d->residual_channels, G = d->gate_channels, S = d->skip_channels, A = d->aux_channels;
  if (R <= 0 || R % KC || G <= 0 || G % 2 || (G / 2) % KC || G % 16 || S <= 0 || S % 16 || A <= 0 || A % 16) return 0;
  const int N2 = S + R;
  const int width = G > N2 ? G : N2;
  if (width > TC_NMAX || N2 % 16 || R % 16) return 0;  // accumulators: 64 rows x <= 128 columns per warpgroup
  p.B = d->batch;
  p.T = d->t;
  p.R = R;
  p.G = G;
  p.S = S;
  p.A = A;
  p.K = d->kernel;
  p.halo = d->halo;
  p.H = G / 2;
  p.D = 1;
  const int tr = ceil_div(d->t, 2 * WN_TT) * (2 * WN_TT);  // packed planes are whole 256-sample blocks
  p.Tp = 2 * d->halo + tr;
  p.Tc = tr;
  p.ngx = R / 8;
  p.ngc = (A + 7) / 8;
  p.nxc = R / KC;
  p.ncc = (A + KC - 1) / KC;
  p.nsc = p.H / KC;
  p.N2 = N2;
  p.tiles_per_seq = tr / WN_TT;
  if ((long long)p.tiles_per_seq * d->batch > 0x3fffffffLL) return 0;
  p.total_tiles = p.tiles_per_seq * d->batch;
  p.a_bytes = 8 * WN_BLK;
  p.b_bytes = 2 * (KC / 8) * width * 16;
  if (G != N2) return 0;  // one weight-stage size (true for every reference config: S = R = G/2)
  p.slot_bytes = p.a_bytes + p.b_bytes;
  p.z_bytes = 2 * (p.H / 8) * 64 * 16;  // per warpgroup: [hi|lo][H/8][64 rows][8]
  p.wso_bytes = p.nsc * p.b_bytes;  // skip / out weights stay resident in shared memory
  const size_t fixed = 2 * (size_t)p.z_bytes + (size_t)p.wso_bytes + 8 * (2 * WN_MAX_SLOTS + 2) + 4 * (size_t)(G + N2) + 128;
  const size_t budget = 227 * 1024;
  if (fixed + 2 * (size_t)p.slot_bytes > budget) return 0;
  const int ns = (int)((budget - fixed) / p.slot_bytes);
  p.nslot = ns > WN_MAX_SLOTS ? WN_MAX_SLOTS : ns;
  smem_bytes = (size_t)p.nslot * p.slot_bytes + fixed;
  p.write_x = 1;
  p.skip_init = 0;
  return 1;
}

}  // namespace pwgb

using namespace pwgb;

extern "C" int pwgb_wnstack_supported(const pwgb_wnstack_desc* d) {
  WnK p;
  size_t bytes;
  return wn_plan(d, p, bytes);
}

extern "C" size_t pwgb_wnstack_x_bytes(const pwgb_wnstack_desc* d) {
  WnK p;
  size_t bytes;
  if (!wn_plan(d, p, bytes)) return 0;
  return (size_t)p.B * 2 * p.ngx * p.Tp * 16;
}

extern "C" size_t pwgb_wnstack_c_bytes(const pwgb_wnstack_desc* d) {
  WnK p;
  size_t bytes;
  if (!wn_plan(d, p, bytes)) return 0;
  return (size_t)p.B * 2 * p.ngc * p.Tc * 16;
}

static dim3 wn_grid(int T, int ng, int B) { return dim3((unsigned)((T + 255) / 256 > 64 ? 64 : (T + 255) / 256), (unsigned)ng, (unsigned)B); }

extern "C" int pwgb_wnstack_pack_x(const pwgb_wnstack_desc* d, const float* x, void* xpk, void* stream) {
  WnK p;
  size_t bytes;
  PWGB_UNSUPPORTED_IF(!wn_plan(d, p, bytes), "wnstack: configuration not supported");
  PWGB_CHECK_ARG(x && xpk, "wnstack_pack_x: null argument");
  if (p.B == 0) return PWGB_OK;
  wn_pack_kernel<<<wn_grid(p.T, p.ngx, p.B), 256, 0, (cudaStream_t)stream>>>(x, (long long)p.R * p.T, p.R, p.T, (uint4*)xpk, p.ngx, p.Tp,
                                                                            p.halo, 0);
  return check_launch("wn_pack_kernel");
}

extern "C" int pwgb_wnstack_pack_c(const pwgb_wnstack_desc* d, const float* c, long long c_batch_stride, void* cpk, void* stream) {
  WnK p;
  size_t bytes;
  PWGB_UNSUPPORTED_IF(!wn_plan(d, p, bytes), "wnstack: configuration not supported");
  PWGB_CHECK_ARG(c && cpk && c_batch_stride >= (long long)p.A * p.T, "wnstack_pack_c: bad argument");
  if (p.B == 0) return PWGB_OK;
  wn_pack_kernel<<<wn_grid(p.Tc, p.ngc, p.B), 256, 0, (cudaStream_t)stream>>>(c, c_batch_stride, p.A, p.T, (uint4*)cpk, p.ngc, p.Tc, 0, 1);
  return check_launch("wn_pack_kernel");
}

extern "C" int pwgb_wnstack_unpack_x(const pwgb_wnstack_desc* d, const void* xpk, float* x, void* stream) {
  WnK p;
  size_t bytes;
  PWGB_UNSUPPORTED_IF(!wn_plan(d, p, bytes), "wnstack: configuration not supported");
  PWGB_CHECK_ARG(x && xpk, "wnstack_unpack_x: null argument");
  if (p.B == 0) return PWGB_OK;
  wn_unpack_kernel<<<wn_grid(p.T, p.ngx, p.B), 256, 0, (cudaStream_t)stream>>>((const uint4*)xpk, p.ngx, p.Tp, p.halo, x, p.R, p.T);
  return check_launch("wn_unpack_kernel");
}

extern "C" int pwgb_wnstack_first_conv(const pwgb_wnstack_desc* d, const float* z, int in_channels, const float* w, const float* bias,
                                       void* xpk, void* stream) {
  WnK p;
  size_t bytes;
  PWGB_UNSUPPORTED_IF(!wn_plan(d, p, bytes), "wnstack: configuration not supported");
  PWGB_CHECK_ARG(z && w && xpk && in_channels > 0, "wnstack_first_conv: bad argument");
  if (p.B == 0) return PWGB_OK;
  wn_first_conv_kernel<<<wn_grid(p.T, p.ngx, p.B), 256, 0, (cudaStream_t)stream>>>(z, in_channels, w, bias, p.T, (uint4*)xpk, p.ngx, p.Tp,
                                                                                  p.halo);
  return check_launch("wn_first_conv_kernel");
}

extern "C" int pwgb_wnstack_layer_forward(const pwgb_wnstack_desc* d, int dilation, const void* xpk_in, const void* cpk,
                                          const void* packed_w, const float* b_conv, const float* b_skip_out, void* xpk_out,
                                          float* skips, int skips_init, void* stream) {
  WnK p;
  size_t bytes = 0;
  PWGB_UNSUPPORTED_IF(!wn_plan(d, p, bytes), "wnstack: configuration not supported by the fused tensor-core layer");
  PWGB_CHECK_ARG(xpk_in && cpk && packed_w && skips, "wnstack_layer: null argument");
  PWGB_CHECK_ARG(dilation > 0 && (long long)(d->kernel / 2) * dilation <= d->halo, "wnstack_layer: dilation %d exceeds the halo %d of the packed stream",
                 dilation, d->halo);
  PWGB_CHECK_ARG(xpk_in != xpk_out, "wnstack_layer: xpk_out must not alias xpk_in (other tiles read the halo)");
  PWGB_CHECK_ARG(!((reinterpret_cast<uintptr_t>(xpk_in) | reinterpret_cast<uintptr_t>(cpk) | reinterpret_cast<uintptr_t>(packed_w) |
                    reinterpret_cast<uintptr_t>(xpk_out)) & 15),
                 "wnstack_layer: packed buffers must be 16-byte aligned");
  if (p.B == 0) return PWGB_OK;
  p.D = dilation;
  p.write_x = xpk_out != nullptr;
  p.skip_init = skips_init != 0;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(wavenet_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) {
      set_error("wnstack_layer: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
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
  const int grid = p.total_tiles < num_sms ? p.total_tiles : num_sms;
  // tensor maps of the packed streams.  A plane ([rows][8 ch] bf16) is contiguous, so it is described as a vector of
  // 8-byte elements (2 per row): dims (2 * rows, 8-channel groups, batch x hi|lo), box (256, 4, 2) = one 16 KB operand
  // window with a 2 KB inner extent
  CUtensorMap tm_x, tm_c;
  {
    const unsigned long long dx[3] = {2ull * p.Tp, (unsigned long long)p.ngx, 2ull * p.B};
    const unsigned long long dc[3] = {2ull * p.Tc, (unsigned long long)p.ngc, 2ull * p.B};
    const unsigned box[3] = {2u * WN_TT, 4u, 2u};
    int rc = tma_make(&tm_x, CU_TENSOR_MAP_DATA_TYPE_UINT64, 8, 3, xpk_in, dx, box);
    if (rc) return rc;
    rc = tma_make(&tm_c, CU_TENSOR_MAP_DATA_TYPE_UINT64, 8, 3, cpk, dc, box);
    if (rc) return rc;
  }
  wavenet_fused_kernel<<<(unsigned)grid, WN_THREADS, bytes, (cudaStream_t)stream>>>(
      p, tm_x, tm_c, (const unsigned*)xpk_in, (const unsigned char*)packed_w, b_conv, b_skip_out, (unsigned*)xpk_out, skips);
  return check_launch("wavenet_fused_kernel");
}
