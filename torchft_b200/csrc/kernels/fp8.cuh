// Row-scaled e4m3 quantisation shared by fp8.cu and the fp8-output RMSNorm in model_ops.cu.
//
// A row (or a column of a weight) is quantised with the power-of-two dequantisation scale 2^e, e = max(-126,
// ceil(log2(amax / 448))), and stores RN_e4m3(x * 2^-e). Since amax * 2^-e <= 448 nothing saturates, and since the scale
// is a power of two the scaling is exact: a CPU model reproduces every byte. e comes from the bit pattern of amax with
// integer operations (log2f is approximate under --use_fast_math). A row holding an inf or a NaN gets a NaN scale and
// 0x7F (e4m3 NaN) in every byte, so the GEMM output row is NaN and the step's non-finite check sees it.
//
// amax is taken over bf16 bit patterns with the sign cleared: as unsigned integers they order like the magnitudes, and
// every inf / NaN pattern (>= 0x7F80) lies above every finite one, so one integer max finds both. A bf16 subnormal
// (< 0x0080) gives e = -126 like zero, and the FTZ multiply by 2^-e flushes it to a signed zero, as the CPU model does.
#pragma once

#include "common.cuh"

namespace tft {

constexpr uint32_t kBf16Inf = 0x7F80u;  // |x| bit patterns at or above this are inf or NaN
constexpr uint8_t kE4m3NaN = 0x7F;

// max(m, |x| bit pattern) over the 8 bf16 lanes of v
__device__ __forceinline__ uint32_t absmax_bits(const Vec16& v, uint32_t m) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) m = max(m, max(w[i] & 0x7FFFu, (w[i] >> 16) & 0x7FFFu));
  return m;
}

// e of a finite amax given as a bf16 magnitude pattern: amax = 1.f * 2^E with f the 23-bit fp32 fraction. amax <= 448 *
// 2^(E-8) = 1.75 * 2^E exactly when the fraction is <= 0.75 (0x600000), else e = E - 7.
__device__ __forceinline__ int fp8_exponent(uint32_t amax_bf16) {
  const uint32_t b = amax_bf16 << 16;
  const int E = (int)(b >> 23) - 127;
  const int e = E - 8 + ((b & 0x7FFFFFu) > 0x600000u ? 1 : 0);
  return e < -126 ? -126 : e;
}

// 2^k for k in [-126, 127] as an fp32 bit pattern
__device__ __forceinline__ float exp2i(int k) { return __uint_as_float((uint32_t)(k + 127) << 23); }

// The dequantisation scale (2^e, or NaN for a non-finite row) and the quantisation multiplier 2^-e of a row's amax.
__device__ __forceinline__ float fp8_scale(uint32_t amax_bf16, float& inv) {
  const int e = fp8_exponent(amax_bf16);
  inv = exp2i(-e);
  return amax_bf16 >= kBf16Inf ? __uint_as_float(0x7FFFFFFFu) : exp2i(e);
}

// 8 bf16 lanes -> 8 e4m3 bytes (lane 0 in the lowest byte): RN_e4m3(x * inv) with the FTZ multiply, or 8 NaN bytes
__device__ __forceinline__ uint2 quant8(const Vec16& v, float inv, bool nonfinite) {
  if (nonfinite) return make_uint2(0x7F7F7F7Fu, 0x7F7F7F7Fu);
  float f[8];
  Pack<__nv_bfloat16>::unpack(v, f);
  uint32_t h[4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
    h[i] = __nv_cvt_float2_to_fp8x2(make_float2(f[2 * i] * inv, f[2 * i + 1] * inv), __NV_SATFINITE,
                                    __NV_E4M3);
  return make_uint2(h[0] | (h[1] << 16), h[2] | (h[3] << 16));
}

// The max of v over a CTA of TPB threads with ONE __syncthreads, like row_sum in model_ops.cu: warp maxima go to the line
// `parity` of a double-buffered smem line, every thread reads all of them, and the next call writes the other line.
template <int TPB>
__device__ __forceinline__ uint32_t row_max_bits(uint32_t v, uint32_t (*red)[TPB / 32], int& parity) {
  v = __reduce_max_sync(0xffffffffu, v);
  constexpr int NW = TPB / 32;
  if ((threadIdx.x & 31) == 0) red[parity][threadIdx.x >> 5] = v;
  __syncthreads();
  uint32_t r = 0;
#pragma unroll
  for (int i = 0; i < NW; ++i) r = max(r, red[parity][i]);
  parity ^= 1;
  return r;
}

}  // namespace tft
