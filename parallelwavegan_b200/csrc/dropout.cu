// Dropout (torch.nn.Dropout in training mode; UHiFiGAN's input and downsample convs, models/uhifigan.py) with a
// counter-based mask: element e is kept when word e % 4 of Philox4x32-10(counter = (e / 4, offset), key = seed),
// read as a 24-bit uniform in [0, 1), is >= p.  The mask is a pure function of (seed, offset, e), so the backward
// recomputes it and no mask tensor is stored.  Kept elements are scaled by 1 / (1 - p), computed in fp32.
// A dropped element is +0.0 whatever its input (-0.0, +-inf and NaN included); a kept one is exactly v * scale, so
// non-finite inputs stay non-finite and -0.0 stays -0.0.  At p == 1 every element is dropped (u < 1): all +0.0, no NaN.
// p outside [0, 1] or NaN is refused.
#include "common.cuh"

namespace pwgb {

// Philox4x32 with 10 rounds (Salmon, Moraes, Dror, Shaw: "Parallel random numbers: as easy as 1, 2, 3", SC 2011)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
  constexpr unsigned M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const unsigned hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x;
    const unsigned hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += W0;
    k.y += W1;
  }
  return c;
}

__device__ __forceinline__ float drop1(float v, unsigned r, float p, float scale) {
  const float u = (float)(r >> 8) * (1.f / 16777216.f);  // exact: 24 bits
  return u >= p ? v * scale : 0.f;
}

// one thread per group of 4 consecutive elements (one Philox call); 16-byte accesses when both tensors are aligned
__global__ void dropout_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, float p, float scale,
                               unsigned long long seed, unsigned long long offset, int vec) {
  const uint2 key = make_uint2((unsigned)seed, (unsigned)(seed >> 32));
  const long long groups = (n + 3) / 4;
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < groups; g += (long long)gridDim.x * blockDim.x) {
    const uint4 r = philox4x32_10(make_uint4((unsigned)g, (unsigned)(g >> 32), (unsigned)offset, (unsigned)(offset >> 32)), key);
    const long long e = 4 * g;
    if (vec && e + 3 < n) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(x + e));
      *reinterpret_cast<float4*>(y + e) =
          make_float4(drop1(v.x, r.x, p, scale), drop1(v.y, r.y, p, scale), drop1(v.z, r.z, p, scale), drop1(v.w, r.w, p, scale));
    } else {
      const unsigned rr[4] = {r.x, r.y, r.z, r.w};
      for (int j = 0; j < 4 && e + j < n; ++j) y[e + j] = drop1(__ldg(x + e + j), rr[j], p, scale);
    }
  }
}

static int dropout_launch(const float* x, float* y, long long n, float p, unsigned long long seed, unsigned long long offset,
                          void* stream, const char* what) {
  PWGB_CHECK_ARG(n >= 0 && (n == 0 || (x && y)), "%s: bad argument", what);
  PWGB_CHECK_ARG(p >= 0.f && p <= 1.f, "%s: p = %g outside [0, 1]", what, (double)p);
  if (n == 0) return PWGB_OK;
  const float scale = 1.f / (1.f - p);  // +inf at p == 1, where no element is kept
  const int vec = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0;
  const long long groups = (n + 3) / 4;
  long long blocks = (groups + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  dropout_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, y, n, p, scale, seed, offset, vec);
  return check_launch(what);
}

}  // namespace pwgb

extern "C" int pwgb_dropout_forward(const float* x, float* y, long long n, float p, unsigned long long seed,
                                    unsigned long long offset, void* stream) {
  return pwgb::dropout_launch(x, y, n, p, seed, offset, stream, "dropout_forward");
}

extern "C" int pwgb_dropout_backward(const float* gy, float* gx, long long n, float p, unsigned long long seed,
                                     unsigned long long offset, void* stream) {
  return pwgb::dropout_launch(gy, gx, n, p, seed, offset, stream, "dropout_backward");
}
