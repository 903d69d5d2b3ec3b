// SineGen excitation (layers/sine.py, flag_for_pulse=False; the U-Net HiFi-GAN's input, bin/preprocess.py:420-440) as
// a deterministic parallel scan.  Per row b and harmonic h (dim = harmonic_num + 1):
//   rad[t]   = (f0[t] * (h + 1) / sr) % 1            (fp32, torch.remainder), rad[0] += rand_ini[b, h] for h >= 1
//   S1       = cumsum(rad)                           (fp64 running sum, each output rounded to fp32: CPU torch.cumsum)
//   shift[t] = -1 where S1[t] % 1 < S1[t-1] % 1      (fp32, t >= 1)
//   S2       = cumsum(fp32(rad + shift))             (fp64, rounded to fp32)
//   phase    = S2 * 2 * float(pi);  sine = sin(phase) * sine_amp;  uv = f0 > voiced_threshold
//   noise    = (uv * noise_std + (1 - uv) * sine_amp / 3) * n;   sine_waves = sine * uv + noise
// Every step is the reference's fp32 operation in its order, with no contraction into FMA.  The fp64 prefix sums are
// exact, hence equal to the sequential ones in any association, while every partial sum stays below 2^53 ulps of the
// smallest addend (DESIGN.md §3.15).  A row is cut into chunks of kChunk samples; five launches:
//   1. sine_chunk_kernel<0>: per (row, h, chunk) the fp64 sum of rad;
//   2. sine_scan_kernel: exclusive scan of those sums along each (row, h), in place;
//   3. sine_chunk_kernel<1>: S1 within the chunk from its prefix, shift, and the fp64 sum of rad + shift;
//   4. sine_scan_kernel on those sums;
//   5. sine_chunk_kernel<2>: both scans within the chunk from their prefixes, then the outputs.
// Sums combine in a fixed tree order (no atomics), so a launch is deterministic whatever the bound.
#include "common.cuh"

namespace pwgb {

constexpr int kThreads = 256;
constexpr int kItems = 8;
constexpr int kChunk = kThreads * kItems;
constexpr int kScanThreads = 1024;
constexpr float kPi = 3.14159265358979323846f;

// shared-memory index of chunk element i, padded so that a thread's kItems consecutive elements spread over the banks
__host__ __device__ constexpr int spad(int i) { return i + (i >> 5); }

// torch.remainder(a, 1) on fp32 (ATen: m = fmod(a, b); m += b where m != 0 and sign(m) != sign(b))
__device__ __forceinline__ float rem1(float a) {
  float m = fmodf(a, 1.f);
  if (m != 0.f && m < 0.f) m = __fadd_rn(m, 1.f);
  return m;
}

// exclusive scan of one double per thread over the block, in a fixed order; *total gets the block's sum
static __device__ double sine_block_exclusive_scan(double v, double* total) {
  __shared__ double warp_sum[kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  const double up = __shfl_up_sync(0xffffffffu, inc, 1);
  const double in_warp = lane > 0 ? up : 0.0;
  if (lane == 31) warp_sum[warp] = inc;
  __syncthreads();
  double before = 0.0, all = 0.0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) {
    const double s = warp_sum[w];
    if (w < warp) before += s;
    all += s;
  }
  __syncthreads();  // warp_sum is reused by the next call
  *total = all;
  return before + in_warp;
}

// PASS 0: chunk sums of rad into sums1.  PASS 1: S1 and shift from the prefix in sums1, chunk sums of rad + shift into
// sums2.  PASS 2: both scans from the prefixes in sums1 and sums2, then the outputs.
template <int PASS>
__global__ void __launch_bounds__(kThreads) sine_chunk_kernel(
    const float* __restrict__ f0, long long T, int dim, float sr, float sine_amp, float noise_std, float voiced_threshold,
    const float* __restrict__ rand_ini, const float* __restrict__ n, float* __restrict__ sine_waves, float* __restrict__ uv_out,
    float* __restrict__ noise_out, float* __restrict__ phase_out, double* __restrict__ sums1, double* __restrict__ sums2) {
  __shared__ float s_f0[spad(kChunk - 1) + 1];
  __shared__ float s_io[spad(kChunk - 1) + 1];
  const long long nchunks = (T + kChunk - 1) / kChunk;
  const long long chunk = blockIdx.x;
  const int b = blockIdx.y;
  const long long t0 = chunk * kChunk;
  const int len = (int)(T - t0 < kChunk ? T - t0 : kChunk);
  const float* f0_row = f0 + (long long)b * T + t0;
  for (int i = threadIdx.x; i < kChunk; i += kThreads) s_f0[spad(i)] = i < len ? __ldg(f0_row + i) : 0.f;
  __syncthreads();
  const int first = threadIdx.x * kItems;  // this thread's elements [first, first + kItems) of the chunk

  for (int h = 0; h < dim; ++h) {
    const long long row = (long long)b * dim + h;
    float rad[kItems];
    double local = 0.0;
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
      const int i = first + k;
      float r = 0.f;
      if (i < len) {
        const float f = s_f0[spad(i)];
        r = rem1(__fdiv_rn(h == 0 ? f : __fmul_rn(f, (float)(h + 1)), sr));
        if (h > 0 && t0 + i == 0) r = __fadd_rn(r, __ldg(rand_ini + (long long)b * dim + h));
      }
      rad[k] = r;
      local += (double)r;
    }
    double total;
    const double excl1 = sine_block_exclusive_scan(local, &total);
    if (PASS == 0) {
      if (threadIdx.x == 0) sums1[row * nchunks + chunk] = total;
      continue;
    }
    // S1 and shift; x = fp32(rad + shift)
    double s1 = sums1[row * nchunks + chunk] + excl1;
    float prev_tmp = rem1((float)s1);  // S1 % 1 of the element before this thread's first
    float x[kItems];
    double local2 = 0.0;
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
      s1 += (double)rad[k];
      const float tmp = rem1((float)s1);
      const bool wrap = t0 + first + k > 0 && __fsub_rn(tmp, prev_tmp) < 0.f;
      prev_tmp = tmp;
      x[k] = first + k < len ? __fadd_rn(rad[k], wrap ? -1.f : -0.f) : 0.f;
      local2 += (double)x[k];
    }
    const double excl2 = sine_block_exclusive_scan(local2, &total);
    if (PASS == 1) {
      if (threadIdx.x == 0) sums2[row * nchunks + chunk] = total;
      continue;
    }
    // the outputs: phase and the sine first, staged in shared memory and stored coalesced along time
    double s2 = sums2[row * nchunks + chunk] + excl2;
    float* const out_row = sine_waves + ((long long)b * T + t0) * dim + h;
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
      s2 += (double)x[k];
      s_io[spad(first + k)] = __fmul_rn(__fmul_rn((float)s2, 2.f), kPi);
    }
    __syncthreads();
    if (phase_out) {
      float* const ph_row = phase_out + ((long long)b * T + t0) * dim + h;
      for (int i = threadIdx.x; i < len; i += kThreads) ph_row[(long long)i * dim] = s_io[spad(i)];
    }
    const float* const n_row = n + ((long long)b * T + t0) * dim + h;
    float* const nz_row = noise_out + ((long long)b * T + t0) * dim + h;
    for (int i = threadIdx.x; i < len; i += kThreads) {
      const float f = s_f0[spad(i)];
      const float uv = f > voiced_threshold ? 1.f : 0.f;
      const float amp = __fadd_rn(__fmul_rn(uv, noise_std), __fdiv_rn(__fmul_rn(__fsub_rn(1.f, uv), sine_amp), 3.f));
      const float nz = __fmul_rn(amp, __ldg(n_row + (long long)i * dim));
      const float sine = __fmul_rn(sinf(s_io[spad(i)]), sine_amp);
      out_row[(long long)i * dim] = __fadd_rn(__fmul_rn(sine, uv), nz);
      nz_row[(long long)i * dim] = nz;
      if (h == 0) uv_out[(long long)b * T + t0 + i] = uv;
    }
    __syncthreads();  // s_io is rewritten by the next harmonic
  }
}

// exclusive scan of each row of sums (rows x nchunks) in place, one block per row, tiles of kScanThreads in order
__global__ void __launch_bounds__(kScanThreads) sine_scan_kernel(double* __restrict__ sums, long long nchunks) {
  __shared__ double warp_sum[kScanThreads / 32];
  double* const row = sums + (long long)blockIdx.x * nchunks;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double carry = 0.0;
  for (long long base = 0; base < nchunks; base += kScanThreads) {
    const long long i = base + threadIdx.x;
    const double v = i < nchunks ? row[i] : 0.0;
    double inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += u;
    }
    const double up = __shfl_up_sync(0xffffffffu, inc, 1);
    const double in_warp = lane > 0 ? up : 0.0;
    if (lane == 31) warp_sum[warp] = inc;
    __syncthreads();
    double before = 0.0, all = 0.0;
    for (int w = 0; w < kScanThreads / 32; ++w) {
      const double s = warp_sum[w];
      if (w < warp) before += s;
      all += s;
    }
    if (i < nchunks) row[i] = carry + (before + in_warp);
    carry += all;
    __syncthreads();
  }
}

}  // namespace pwgb

extern "C" size_t pwgb_sine_gen_workspace(int batch, long long t, int harmonic_num) {
  if (batch <= 0 || t <= 0 || harmonic_num < 0) return 0;
  const long long nchunks = (t + pwgb::kChunk - 1) / pwgb::kChunk;
  return (size_t)(2 * (long long)batch * (harmonic_num + 1) * nchunks) * sizeof(double);
}

extern "C" int pwgb_sine_gen_forward(const float* f0, int batch, long long t, int harmonic_num, float samp_rate, float sine_amp,
                                     float noise_std, float voiced_threshold, const float* rand_ini, const float* noise_in,
                                     float* sine_waves, float* uv, float* noise, float* phase, void* ws, size_t ws_bytes,
                                     void* stream) {
  using namespace pwgb;
  PWGB_CHECK_ARG(batch >= 0 && t >= 0 && harmonic_num >= 0, "sine_gen_forward: batch %d, t %lld, harmonic_num %d", batch, t,
                 harmonic_num);
  PWGB_CHECK_ARG(batch <= 65535, "sine_gen_forward: batch %d above 65535", batch);
  if (batch == 0 || t == 0) return PWGB_OK;
  PWGB_CHECK_ARG(f0 && rand_ini && noise_in && sine_waves && uv && noise && ws, "sine_gen_forward: null pointer");
  const size_t need = pwgb_sine_gen_workspace(batch, t, harmonic_num);
  PWGB_CHECK_ARG(ws_bytes >= need, "sine_gen_forward: workspace of %zu bytes, %zu needed", ws_bytes, need);
  const int dim = harmonic_num + 1;
  const long long nchunks = (t + kChunk - 1) / kChunk;
  PWGB_CHECK_ARG(nchunks <= 0x7fffffffLL, "sine_gen_forward: t = %lld too long", t);
  double* sums1 = static_cast<double*>(ws);
  double* sums2 = sums1 + (long long)batch * dim * nchunks;
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 grid((unsigned)nchunks, (unsigned)batch);
  const unsigned rows = (unsigned)(batch * dim);
  int rc;
  sine_chunk_kernel<0><<<grid, kThreads, 0, s>>>(f0, t, dim, samp_rate, sine_amp, noise_std, voiced_threshold, rand_ini, noise_in,
                                                 sine_waves, uv, noise, phase, sums1, sums2);
  if ((rc = check_launch("sine_gen_forward (chunk sums)")) != PWGB_OK) return rc;
  sine_scan_kernel<<<rows, kScanThreads, 0, s>>>(sums1, nchunks);
  if ((rc = check_launch("sine_gen_forward (scan 1)")) != PWGB_OK) return rc;
  sine_chunk_kernel<1><<<grid, kThreads, 0, s>>>(f0, t, dim, samp_rate, sine_amp, noise_std, voiced_threshold, rand_ini, noise_in,
                                                 sine_waves, uv, noise, phase, sums1, sums2);
  if ((rc = check_launch("sine_gen_forward (shifted sums)")) != PWGB_OK) return rc;
  sine_scan_kernel<<<rows, kScanThreads, 0, s>>>(sums2, nchunks);
  if ((rc = check_launch("sine_gen_forward (scan 2)")) != PWGB_OK) return rc;
  sine_chunk_kernel<2><<<grid, kThreads, 0, s>>>(f0, t, dim, samp_rate, sine_amp, noise_std, voiced_threshold, rand_ini, noise_in,
                                                 sine_waves, uv, noise, phase, sums1, sums2);
  return check_launch("sine_gen_forward (outputs)");
}
