// Hopper warpgroup MMA (wgmma.mma_async) wrappers: D (fp32, registers) += A (bf16, smem) x B (bf16, smem), M = 64 rows per
// warpgroup, K = 16, for N = 16 / 32 / 64 / 128.  TA / TB select the operand-major mode of the shared-memory image (0 = K-major,
// 1 = MN-major).  Accumulator fragment of thread `lane` of warp `w` of the warpgroup: register i holds row 16 w + lane / 4 +
// 8 ((i / 2) % 2), column 8 (i / 4) + 2 (lane % 4) + i % 2 -- so an N = 128 block is the concatenation of narrower blocks.
#pragma once

namespace pwgb {

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// No-swizzle ("interleaved") shared-memory matrix descriptor: [0,14) start >> 4, [16,30) LBO >> 4, [32,46) SBO >> 4,
// layout type 0.  K-major: LBO = distance of the K-adjacent 8x8 core matrix, SBO = distance of the next 8 rows (M / N).
// MN-major: LBO = distance of the next 8 K rows, SBO = distance of the next 8 M / N elements.
__device__ __forceinline__ unsigned long long gmma_desc(unsigned addr, unsigned lbo, unsigned sbo) {
  return (unsigned long long)((addr >> 4) & 0x3FFF) | ((unsigned long long)((lbo >> 4) & 0x3FFF) << 16) |
         ((unsigned long long)((sbo >> 4) & 0x3FFF) << 32);
}

template <int N, int TA, int TB>
struct Wgmma;

template <int TA, int TB>
struct Wgmma<16, TA, TB> {
  __device__ __forceinline__ static void run(float* d, unsigned long long a, unsigned long long b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, 1, 1, 1, %10, %11;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "n"(TA), "n"(TB)
        : "memory");
  }
};

template <int TA, int TB>
struct Wgmma<32, TA, TB> {
  __device__ __forceinline__ static void run(float* d, unsigned long long a, unsigned long long b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, 1, 1, 1, %18, %19;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "n"(TA), "n"(TB)
        : "memory");
  }
};

template <int TA, int TB>
struct Wgmma<64, TA, TB> {
  __device__ __forceinline__ static void run(float* d, unsigned long long a, unsigned long long b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, 1, 1, 1, %34, %35;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "n"(TA), "n"(TB)
        : "memory");
  }
};

template <int TA, int TB>
struct Wgmma<128, TA, TB> {
  __device__ __forceinline__ static void run(float* d, unsigned long long a, unsigned long long b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, 1, 1, 1, %66, %67;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "n"(TA), "n"(TB)
        : "memory");
  }
};

// N = 16 * NB16 (compile time, 1 <= NB16 <= 8) as one instruction of 128 columns or at most three of 64 / 32 / 16 columns,
// each into a fixed slice of d.  With the width fixed at compile time ptxas can keep consecutive commit groups in flight;
// the run-time selection below makes it serialize every wgmma.  b_col16: as below.
template <int TA, int TB, int NB16>
__device__ __forceinline__ void wgmma_n(float* d, unsigned long long a, unsigned long long b, unsigned b_col16) {
  static_assert(NB16 >= 1 && NB16 <= 8, "NB16");
  if constexpr (NB16 == 8) {
    Wgmma<128, TA, TB>::run(d, a, b);
  } else {
    constexpr int c32 = NB16 & 4, c16 = NB16 & 6;  // first 16-column block of the 32- and of the 16-column instruction
    if constexpr ((NB16 & 4) != 0) Wgmma<64, TA, TB>::run(d, a, b);
    if constexpr ((NB16 & 2) != 0) Wgmma<32, TA, TB>::run(d + 8 * c32, a, b + (unsigned long long)c32 * b_col16);
    if constexpr ((NB16 & 1) != 0) Wgmma<16, TA, TB>::run(d + 8 * c16, a, b + (unsigned long long)c16 * b_col16);
  }
}

// N = 16 * nb16 (1 <= nb16 <= NBMAX, run time; NBMAX = 4 or 8) as at most three instructions of 64 / 32 / 16 columns
// (or one of 128); d holds the fragment of the whole width.  b_col16: descriptor distance (16-byte units) of the B
// operand's next 16 columns.
template <int TA, int TB, int NBMAX>
__device__ __forceinline__ void wgmma_cols(float* d, unsigned long long a, unsigned long long b, int nb16, unsigned b_col16) {
  static_assert(NBMAX == 4 || NBMAX == 8, "NBMAX");
  if (NBMAX == 8 && nb16 == 8) {
    Wgmma<128, TA, TB>::run(d, a, b);
    return;
  }
  if (nb16 >= 4) {
    Wgmma<64, TA, TB>::run(d, a, b);
    if (NBMAX == 8) {
      if (nb16 & 2) Wgmma<32, TA, TB>::run(d + 32, a, b + 4ull * b_col16);
      if (nb16 & 1) {
        if (nb16 & 2) Wgmma<16, TA, TB>::run(d + 48, a, b + 6ull * b_col16);
        else Wgmma<16, TA, TB>::run(d + 32, a, b + 4ull * b_col16);
      }
    }
    return;
  }
  if (nb16 & 2) Wgmma<32, TA, TB>::run(d, a, b);
  if (nb16 & 1) {
    if (nb16 & 2) Wgmma<16, TA, TB>::run(d + 16, a, b + 2ull * b_col16);
    else Wgmma<16, TA, TB>::run(d, a, b);
  }
}

}  // namespace pwgb
