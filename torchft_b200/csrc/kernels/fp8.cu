// Row-scaled e4m3 operands for the fp8 block linears (sm_90a). The GEMMs are rowwise torch._scaled_mm (a row-major with
// one scale per row, b column-major with one scale per column); these kernels make their operands:
//
//   fp8_rows    bf16 [R, C] (row stride ld) -> e4m3 [R, C] + fp32 scale per row: activations, grad-outputs, and W [N, K]
//               in the forward orientation (one scale per output channel)
//   fp8_swiglu  packed gate|up [T, 2F] -> e4m3 silu(g) * u [T, F] + scale per row; the bf16 product is never written
//   fp8_cols_t  W [N, K] -> e4m3 W^T [K, N] + scale per column of W (per input channel), for the input-gradient GEMM
//
// The format and its scale rule are in fp8.cuh. Bytes equal the CPU model in tests/_fp8_ref.py, and fp8_swiglu's bytes
// equal fp8_rows(swiglu_fwd(gu)): the product is computed by swiglu_fwd's expression and rounded to bf16 first.
#include <algorithm>
#include <stdexcept>
#include <string>
#include <utility>

#include "api.h"
#include "fp8.cuh"

namespace tft {

using bf16 = __nv_bfloat16;
using P8 = Pack<bf16>;

// ------------------------------------------------------------------------------------------------------------ rows
// A CTA of TPB threads walks rows blockIdx.x, +gridDim.x, ...; a thread owns NV 16-element chunks of the row (two 16 B
// loads, one 16 B store each), held in registers between the row-max and the cast. The launch shape is the RMSNorm
// forward's rule over 16-element chunks: the CTA starts at 128 threads and doubles until 4 chunks per thread cover the
// row, so rows of up to 4 x 512 x 16 = 32768 elements (the w13 grad-output of Llama-3-8B is 28672) fit.
constexpr int kFp8RowThreads = 128, kFp8RowMaxVec = 4, kFp8RowMaxC = 16 * kFp8RowMaxVec * 512;

template <int NV, int TPB, bool SWIGLU>
__global__ void __launch_bounds__(TPB) fp8_rows_kernel(const bf16* __restrict__ x, size_t ld, uint8_t* __restrict__ q,
                                                       float* __restrict__ scale, int rows, int C) {
  __shared__ uint32_t red[2][TPB / 32];
  const int nch = C / 16;
  int parity = 0;
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const bf16* xr = x + (size_t)row * ld;
    Vec16 v[NV][2];
    if constexpr (SWIGLU) {
      Vec16 g[NV][2], u[NV][2];
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = threadIdx.x + i * TPB;
        if (c < nch) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            g[i][h] = ld_stream(xr + c * 16 + h * 8);
            u[i][h] = ld_stream(xr + C + c * 16 + h * 8);
          }
        }
      }
#pragma unroll
      for (int i = 0; i < NV; ++i) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          // swiglu_fwd_kernel's expression, rounded to bf16 as that kernel stores it
          float gf[8], uf[8], o[8];
          P8::unpack(g[i][h], gf);
          P8::unpack(u[i][h], uf);
#pragma unroll
          for (int k = 0; k < 8; ++k) o[k] = gf[k] / (1.f + __expf(-gf[k])) * uf[k];
          v[i][h] = P8::pack(o);
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = threadIdx.x + i * TPB;
        if (c < nch) {
          v[i][0] = ld_stream(xr + c * 16);
          v[i][1] = ld_stream(xr + c * 16 + 8);
        }
      }
    }
    uint32_t m = 0;
#pragma unroll
    for (int i = 0; i < NV; ++i)
      if (threadIdx.x + i * TPB < nch) m = absmax_bits(v[i][1], absmax_bits(v[i][0], m));
    m = row_max_bits<TPB>(m, red, parity);
    float inv;
    const float s = fp8_scale(m, inv);
    const bool bad = m >= kBf16Inf;
    if (threadIdx.x == 0) scale[row] = s;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = threadIdx.x + i * TPB;
      if (c < nch) {
        const uint2 lo = quant8(v[i][0], inv, bad), hi = quant8(v[i][1], inv, bad);
        st_stream(q + (size_t)row * C + c * 16, Vec16{lo.x, lo.y, hi.x, hi.y});
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------- columns
// W [N, K] -> W^T [K, N]. Pass 1: per-column max of |W| bit patterns. A CTA of 256 threads covers 256 columns (32
// lanes x 8 columns of a 16 B load) and kColRows rows (8 row groups); the row groups meet in shared memory and one
// atomicMax per column goes to the u32 workspace. Max is order-independent: any grid gives the same bits.
constexpr int kColRows = 128;
__global__ void __launch_bounds__(256) fp8_colmax_kernel(const bf16* __restrict__ w, int N, int K,
                                                         uint32_t* __restrict__ amax) {
  __shared__ uint32_t part[8][256];
  const int lane = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int kv = blockIdx.x * 32 + lane;  // 8-column vector index
  const int r0 = blockIdx.y * kColRows;
  const int r1 = min(N, r0 + kColRows);
  uint32_t m[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (kv < K / 8) {
    for (int r = r0 + rg; r < r1; r += 8) {
      const Vec16 v = ld_stream(w + (size_t)r * K + kv * 8);
      const uint32_t ww[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        m[2 * j] = max(m[2 * j], ww[j] & 0x7FFFu);
        m[2 * j + 1] = max(m[2 * j + 1], (ww[j] >> 16) & 0x7FFFu);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) part[rg][lane * 8 + j] = m[j];
  __syncthreads();
  const int k = blockIdx.x * 256 + threadIdx.x;
  if (k < K) {
    uint32_t r = 0;
#pragma unroll
    for (int g = 0; g < 8; ++g) r = max(r, part[g][threadIdx.x]);
    atomicMax(amax + k, r);
  }
}

// Pass 2: a CTA transposes a 64 (n) x 64 (k) tile through shared memory. Each thread loads two 16 B vectors of W rows,
// then reads 16 consecutive n of one column k, casts them with that column's scale and stores them as one 16 B vector
// of the W^T row k. The first row of tiles also writes the scales.
constexpr int kTile = 64;
__global__ void __launch_bounds__(256) fp8_cols_t_kernel(const bf16* __restrict__ w, int N, int K,
                                                         const uint32_t* __restrict__ amax, uint8_t* __restrict__ q,
                                                         float* __restrict__ scale) {
  __shared__ uint16_t tile[kTile][kTile + 2];  // [n][k]; the odd word stride spreads a column over the banks
  const int n0 = blockIdx.y * kTile, k0 = blockIdx.x * kTile;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int idx = threadIdx.x + j * 256;  // 64 rows x 8 vectors
    const int r = idx >> 3, kv = idx & 7;
    const int n = n0 + r, k = k0 + kv * 8;
    Vec16 v{0, 0, 0, 0};
    if (n < N && k < K) v = ld_stream(w + (size_t)n * K + k);
    const uint32_t ww[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      tile[r][kv * 8 + 2 * i] = (uint16_t)(ww[i] & 0xFFFFu);
      tile[r][kv * 8 + 2 * i + 1] = (uint16_t)(ww[i] >> 16);
    }
  }
  __syncthreads();
  const int kl = threadIdx.x >> 2, nc = threadIdx.x & 3;  // 64 columns x 4 chunks of 16 n
  const int k = k0 + kl, n = n0 + nc * 16;
  if (k >= K) return;
  const uint32_t m = amax[k];
  float inv;
  const float s = fp8_scale(m, inv);
  if (blockIdx.y == 0 && nc == 0) scale[k] = s;
  if (n >= N) return;
  uint32_t p[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) p[i] = (uint32_t)tile[nc * 16 + 2 * i][kl] | ((uint32_t)tile[nc * 16 + 2 * i + 1][kl] << 16);
  const uint2 lo = quant8(Vec16{p[0], p[1], p[2], p[3]}, inv, m >= kBf16Inf);
  const uint2 hi = quant8(Vec16{p[4], p[5], p[6], p[7]}, inv, m >= kBf16Inf);
  st_stream(q + (size_t)k * N + n, Vec16{lo.x, lo.y, hi.x, hi.y});
}

// ------------------------------------------------------------------------------------------------------ launchers
// V, the 16-element chunks per thread a row of C needs at 128 threads rounded up to a power of two, selects NV = min(V,
// kFp8RowMaxVec) chunks per thread and TPB = 128 * V / NV threads: (1, 128) (2, 128) (4, 128) (4, 256) (4, 512).
static int fp8_rows_v(int C) {
  int v = 1;
  while (v * kFp8RowThreads < C / 16) v *= 2;
  return v;
}

std::pair<int, int> fp8_rows_shape(int C) {
  const int v = fp8_rows_v(C);
  const int nv = v < kFp8RowMaxVec ? v : kFp8RowMaxVec;
  return {nv, kFp8RowThreads * v / nv};
}

template <bool SWIGLU>
static void fp8_rows_any(const void* x, size_t ld, void* q, float* scale, int rows, int C, cudaStream_t s,
                         const char* what) {
  if (C <= 0 || C % 16 || C > kFp8RowMaxC)
    throw std::runtime_error(std::string(what) + ": the row length must be a positive multiple of 16 and <= 32768, got " +
                             std::to_string(C));
  if (ld % 8 || (uintptr_t)x % 16 || (uintptr_t)q % 16)
    throw std::runtime_error(std::string(what) + ": rows must be 16-byte aligned (pointers and row stride)");
  if (rows <= 0) return;
  dispatch<1, 2, 4, 8, 16>(fp8_rows_v(C), [&](auto V) {
    constexpr int NV = V < kFp8RowMaxVec ? V : kFp8RowMaxVec, TPB = kFp8RowThreads * V / NV;
    // a 4-chunk thread holds 32 registers of row: 1024 threads per SM leave each 64
    const int grid = std::min(rows, kNumSMs * (1024 / TPB));
    fp8_rows_kernel<NV, TPB, SWIGLU><<<grid, TPB, 0, s>>>((const bf16*)x, ld, (uint8_t*)q, scale, rows, C);
  });
  TFT_CUDA_CHECK(cudaGetLastError());
}

void fp8_rows_launch(const void* x, size_t ld, void* q, float* scale, int rows, int C, cudaStream_t s) {
  fp8_rows_any<false>(x, ld, q, scale, rows, C, s, "fp8_rows");
}

void fp8_swiglu_launch(const void* gu, void* q, float* scale, int T, int F, cudaStream_t s) {
  fp8_rows_any<true>(gu, 2 * (size_t)F, q, scale, T, F, s, "fp8_swiglu");
}

void fp8_cols_t_launch(const void* w, int N, int K, void* q, float* scale, uint32_t* amax_ws, cudaStream_t s) {
  if (N <= 0 || K <= 0 || N % 16 || K % 16)
    throw std::runtime_error("fp8_cols_t: both dimensions of W must be positive multiples of 16, got " +
                             std::to_string(N) + " x " + std::to_string(K));
  if ((uintptr_t)w % 16 || (uintptr_t)q % 16) throw std::runtime_error("fp8_cols_t: W and W^T must be 16-byte aligned");
  TFT_CUDA_CHECK(cudaMemsetAsync(amax_ws, 0, sizeof(uint32_t) * (size_t)K, s));
  fp8_colmax_kernel<<<dim3((K + 255) / 256, (N + kColRows - 1) / kColRows), 256, 0, s>>>((const bf16*)w, N, K, amax_ws);
  fp8_cols_t_kernel<<<dim3((K + kTile - 1) / kTile, (N + kTile - 1) / kTile), 256, 0, s>>>((const bf16*)w, N, K, amax_ws,
                                                                                          (uint8_t*)q, scale);
  TFT_CUDA_CHECK(cudaGetLastError());
}

}  // namespace tft
