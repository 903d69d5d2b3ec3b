// mbarrier / bulk-copy PTX helpers, the bf16 hi/lo split, the pieces of the stride-1 conv pipeline and the launch helpers
// shared by the tensor-core kernels (sm_90a).
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace pwgb {

constexpr int KC = 32;  // input channels per activation chunk / weight stage (2 MMA K-steps)
constexpr int TC_NMAX = 128;  // accumulator columns of one launch: 64 rows x 128 fp32 = 64 registers per consumer thread
constexpr unsigned SPIN_LIMIT = 1u << 22;

// ------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try(unsigned bar, unsigned parity) {
  unsigned ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (launch error) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait_spin(unsigned bar, unsigned parity) {
  unsigned n = 0;
  while (!mbar_try(bar, parity)) {
    if (++n > SPIN_LIMIT) {
      printf("pwgb conv1d_tc: mbarrier timeout (block %d thread %d bar %u parity %u)\n", blockIdx.x, threadIdx.x, bar,
             parity);
      __trap();
    }
  }
}
// The same bound without the diagnostic, for kernels that pipeline their wgmma groups: a call (printf) anywhere in the
// kernel, in any warp role, makes ptxas serialize every wgmma of it (C7510).
__device__ __forceinline__ void mbar_wait_trap(unsigned bar, unsigned parity) {
  for (unsigned n = 0; !mbar_try(bar, parity);)
    if (++n > SPIN_LIMIT) __trap();
}
// Same with a sleep back-off: waiting warps must not steal issue slots from the working ones
// (spin loops were 17% of all executed instructions in the first persistent version).  Trap only, like mbar_wait_trap.
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity) {
  unsigned n = 0;
  while (!mbar_try(bar, parity)) {
    if (n > 4) __nanosleep(n > 64 ? 200 : 40);
    if (++n > SPIN_LIMIT) __trap();
  }
}
__device__ __forceinline__ void bulk_g2s(unsigned dst, const void* src, unsigned bytes, unsigned bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// shared -> global bulk copy, and the same as an fp32 add into global memory (y = y + smem, round to nearest); both
// belong to the issuing thread's bulk group
__device__ __forceinline__ void bulk_s2g(void* dst, unsigned src, unsigned bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_s2g_add(float* dst, unsigned src, unsigned bytes) {
  asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// this thread's bulk groups have finished reading their shared-memory source
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// this thread's bulk groups are complete (writes performed)
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void cp_async4(unsigned dst, const float* src, unsigned src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// One elected lane of a converged warp (all 32 lanes must call this).
__device__ __forceinline__ unsigned elect_one() {
  unsigned pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred;
}
// named barrier of the 128 threads of warpgroup `wg` (ids 2.. ; id 1 is the conv producers' barrier)
__device__ __forceinline__ void wg_barrier(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory"); }

__device__ __forceinline__ void split8(const float (&v)[8], uint4& hi, uint4& lo) {
  unsigned h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __nv_bfloat162 hh = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
    float2 hf = __bfloat1622float2(hh);
    __nv_bfloat162 ll = __floats2bfloat162_rn(v[2 * i] - hf.x, v[2 * i + 1] - hf.y);
    h[i] = *reinterpret_cast<unsigned*>(&hh);
    l[i] = *reinterpret_cast<unsigned*>(&ll);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}
// two floats -> packed bf16 hi pair and lo pair (the residual of the hi rounding); the same values as split8
__device__ __forceinline__ void split2(float a, float b, unsigned& hi, unsigned& lo) {
  __nv_bfloat162 hh = __floats2bfloat162_rn(a, b);
  const float2 hf = __bfloat1622float2(hh);
  __nv_bfloat162 ll = __floats2bfloat162_rn(a - hf.x, b - hf.y);
  hi = *reinterpret_cast<unsigned*>(&hh);
  lo = *reinterpret_cast<unsigned*>(&ll);
}

// ------------------------------------------------------------------ pieces of the stride-1 conv pipeline
// shared by conv1d_tc_kernel and the fused ResBlock pair (rb_pair_split_kernel).
//
// Channels 8 g .. 8 g + 7 of row r of a K-major activation operand image of R rows ([hi|lo][ci8][row][8] bf16): hi at
// [g][r], lo at [KC / 8 + g][r].
__device__ __forceinline__ void store_split8(unsigned char* img, int R, int r, int g, const float (&v)[8]) {
  uint4 hi, lo;
  split8(v, hi, lo);
  *reinterpret_cast<uint4*>(img + ((size_t)g * R + r) * 16) = hi;
  *reinterpret_cast<uint4*>(img + ((size_t)(KC / 8 + g) * R + r) * 16) = lo;
}

// Packed activation handed from one conv's epilogue to the next conv's operand buffers (the HiFi-GAN ResBlock
// intermediate): [B][C / KC][hi|lo][KC / 8][T][8] bf16, 4 C T bytes per item, no halo rows.  The 8-channel planes
// ([T][8], 16 bytes per row) are numbered (b C / KC + c) 2 KC / 8 + hi|lo KC / 8 + g, so one box of 8 planes x R rows
// from plane pk_plane(b, C, c KC) is exactly the operand image of chunk c (store_split8's layout); rows outside [0, T)
// read as zero (TMA out-of-bounds fill), the convs' zero padding.  Plane of the hi bf16 of channels co .. co + 7
// (co % 8 == 0); the lo plane is KC / 8 further.
__host__ __device__ __forceinline__ long long pk_plane(int b, int C, int co) {
  return ((long long)b * (C / KC) + co / KC) * (2 * (KC / 8)) + (co % KC) / 8;
}

// A landed raw fp32 stage (KC channel rows of `ld` floats; operand row r is raw[r + shift] of each) -> rows [0, rows) of
// the operand image `img` of R rows, as lrelu(v, slope).  MASK: a row whose sample tbase + r is outside [0, tlim) is zero
// padding (a stage filled by bulk copies holds no sample there); without it the stage already holds the padding.  NTHR
// threads, this one `tid` of them.
template <int NTHR, bool MASK>
__device__ __forceinline__ void convert_raw_stage(unsigned char* img, int R, const float* raw, int shift, int ld, int rows,
                                                  int tbase, unsigned tlim, float slope, int tid) {
  for (int r = tid; r < rows; r += NTHR) {
    const bool ok = !MASK || (unsigned)(tbase + r) < tlim;
    const float* rr = raw + r + shift;
#pragma unroll
    for (int g = 0; g < KC / 8; ++g) {
      float u[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) u[j] = ok ? lrelu(rr[(g * 8 + j) * ld], slope) : 0.f;
      store_split8(img, R, r, g, u);
    }
  }
}

// One raw stage by one warp: samples [start, end) of the KC channel rows src + lane * ld (lane = channel) into the
// stage rows of `pitch` floats at `stage`, `dst_off` floats into each row, one bulk copy per lane, completing on `bar`.
// An empty range only arrives on `bar`.
__device__ __forceinline__ void load_raw_stage(unsigned stage, int pitch, const float* src, long long ld, int start, int end,
                                               int dst_off, unsigned bar, int lane) {
  const int nbytes = (end - start) * 4;
  if (nbytes > 0) {
    if (lane == 0) mbar_expect_tx(bar, (unsigned)nbytes * KC);
    __syncwarp();
    bulk_g2s(stage + (unsigned)(lane * pitch + dst_off) * 4u, src + (long long)lane * ld + start, (unsigned)nbytes, bar);
  } else if (lane == 0) {
    mbar_arrive(bar);
  }
}

// One weight stage of wgmma on the operand image at `a_img` (lbo: the image's rows * 16 B; sub: its hi -> lo offset in
// 16-byte units) from row `row0` on, per k16 step and 64-row block the three bf16x3 products hi*hi, lo*hi, hi*lo.  One
// commit group per call.
template <int MT, int NB16>
__device__ __forceinline__ void mma_stage(float* acc, unsigned a_img, unsigned lbo, unsigned sub, int row0, unsigned b_addr) {
  constexpr int NACC = 8 * NB16;
  constexpr unsigned lbo_b = NB16 * 256u, b_sub = (KC / 8) * NB16 * 16u;
  wg_fence();
#pragma unroll
  for (int ks = 0; ks < KC / 16; ++ks) {
    const unsigned long long bh = gmma_desc(b_addr + (unsigned)(2 * ks) * lbo_b, lbo_b, 128);
    const unsigned long long ah0 = gmma_desc(a_img + ((unsigned)(2 * ks) * (lbo / 16u) + (unsigned)row0) * 16u, lbo, 128);
#pragma unroll
    for (int mb = 0; mb < MT; ++mb) {
      const unsigned long long ah = ah0 + 64 * mb;  // next 64 rows: 64 x 16 B
      wgmma_n<0, 0, NB16>(acc + mb * NACC, ah, bh, 16);
      wgmma_n<0, 0, NB16>(acc + mb * NACC, ah + sub, bh, 16);
      wgmma_n<0, 0, NB16>(acc + mb * NACC, ah, bh + b_sub, 16);
    }
  }
  wg_commit();
}

// Staged epilogue tile: fp32 [channel][stage_ld(MT)] over the 64 MT rows of a tile.  Rows of a channel are contiguous, so
// one bulk copy moves a channel's residual in and its outputs out; the 16-byte pad keeps the rows 16-byte aligned and
// puts the 8 rows x 4 columns of an accumulator-fragment write in 32 distinct banks.
__host__ __device__ constexpr int stage_ld(int mt) { return 64 * mt + 4; }
// Residual of one channel row (`bytes` at src) into the tile row at `row`, once this thread's previous store has read it;
// no bytes (a row beyond T): a bare arrival on `bar`.
__device__ __forceinline__ void stage_load_row(unsigned row, const float* src, unsigned bytes, unsigned bar) {
  bulk_wait_read();
  if (bytes) {
    mbar_expect_tx(bar, bytes);
    bulk_g2s(row, src, bytes, bar);
  } else {
    mbar_arrive(bar);
  }
}
// The tile row at `row` to dst as one bulk store, or with `add` one bulk fp32 add (dst + row).
__device__ __forceinline__ void stage_store_row(float* dst, unsigned row, unsigned bytes, bool add) {
  if (!bytes) return;
  if (add)
    bulk_s2g_add(dst, row, bytes);
  else
    bulk_s2g(dst, row, bytes);
  bulk_commit();
}

// ------------------------------------------------------------------ launch helpers (host)
// SMs of the current device, read once per process: the grid of the persistent tensor-core kernels.
inline int tc_num_sms() {
  static int num_sms = 0;
  if (!num_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (num_sms <= 0) num_sms = 132;
  }
  return num_sms;
}
// Lets every kernel of `kernels` use `bytes` of dynamic shared memory, once per process (`done`).  On a CUDA error the
// message is "<what>: cudaFuncSetAttribute: <error>", the result PWGB_CUDA_ERROR, and the next call tries again.
template <class Kernel, size_t N>
int smem_opt_in(bool& done, const Kernel (&kernels)[N], int bytes, const char* what) {
  if (done) return PWGB_OK;
  for (const Kernel k : kernels) {
    const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) {
      set_error("%s: cudaFuncSetAttribute: %s", what, cudaGetErrorString(e));
      return PWGB_CUDA_ERROR;
    }
  }
  done = true;
  return PWGB_OK;
}

// w (rows, cin_real, K) fp32 -> rows [co_begin, co_begin + rows) of the tensor-core weight operand image
// [chunk][tap][hi|lo][ci8][co (cout_total)][8] bf16 (defined in conv1d_tc.cu)
void tc_pack_rows(const float* w, void* packed, int cin_real, int cin_pad, int rows, int K, int co_begin, int cout_total,
                  cudaStream_t st);

}  // namespace pwgb
