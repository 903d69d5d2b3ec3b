// mbarrier / bulk-copy PTX helpers and the bf16 hi/lo split shared by the tensor-core kernels (sm_90a).
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace pwgb {

constexpr int KC = 32;  // input channels per activation chunk / weight stage (2 MMA K-steps)
constexpr int TC_NMAX = 128;  // accumulator columns of one launch: 64 rows x 128 fp32 = 64 registers per consumer thread
constexpr unsigned SPIN_LIMIT = 1u << 22;
#ifndef PWGB_NPROD
#define PWGB_NPROD 256
#endif

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
// Long waits of the wide roles: the thread is suspended in hardware until the phase completes (or `hint_ns` passed), so a
// waiting warp issues almost nothing -- plain try_wait loops were 35-40 % of the executed instructions of the fused
// WaveNet kernel's gate / epilogue warps.
__device__ __forceinline__ void mbar_wait_hint(unsigned bar, unsigned parity, unsigned hint_ns = 20000u) {
  unsigned n = 0;
  for (;;) {
    unsigned ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity), "r"(hint_ns)
        : "memory");
    if (ok) break;
    if (++n > SPIN_LIMIT) {
      printf("pwgb: mbarrier timeout (block %d thread %d bar %u parity %u)\n", blockIdx.x, threadIdx.x, bar, parity);
      __trap();
    }
  }
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
__device__ __forceinline__ void producer_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(PWGB_NPROD) : "memory"); }
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

// w (rows, cin_real, K) fp32 -> rows [co_begin, co_begin + rows) of the tensor-core weight operand image
// [chunk][tap][hi|lo][ci8][co (cout_total)][8] bf16 (defined in conv1d_tc.cu)
void tc_pack_rows(const float* w, void* packed, int cin_real, int cin_pad, int rows, int K, int co_begin, int cout_total,
                  cudaStream_t st);

}  // namespace pwgb
