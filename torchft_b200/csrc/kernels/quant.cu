// Group-wise FP8 (e4m3) quantisation kernels and the fused quantised
// all-reduce over NVLink peer memory (sm_90a).
//
// Parity target: torchft/quantization.py (5 Triton kernels) +
// torchft/collectives.py:297-415 (quantize -> alltoall -> reduce -> allgather
// -> dequantize = 3 kernels + 2 NCCL collectives + 2 allocations per call).
// Here the whole pipeline -- including DiLoCo's pseudo-gradient
// `original - local` (torchft/local_sgd.py:324-337) -- is ONE launch: the
// "alltoall" and "allgather" are P2P loads/stores issued by the kernel itself.
//
// Wire format "Q8G" (ours, not the reference's row format): the flat message is
// cut into groups of G=512 elements; the padded group count NG is a multiple
// of `world`. For every group: one fp32 dequant scale s = absmax/448 and 512
// e4m3 bytes q = x/s. Layout inside the symmetric segment at byte offset off:
//     [ float scales[NG] ][ uint8 payload[NG * 512] ]
// One warp owns one group (16 elements / lane, one 16 B payload vector / lane).
#include <stdexcept>
#include <string>

#include "api.h"
#include "common.cuh"

namespace tft {

constexpr int kGroup = 512;
constexpr float kFp8Max = 448.f;

// 16 elements of p starting at e <-> 16 floats; elements at or past nelem load as 0 and are not stored.
template <typename T>
__device__ __forceinline__ void load16(const T* p, size_t e, size_t nelem, float* f) {
  constexpr int N = Pack<T>::N;
  if (e + 16 <= nelem) {
#pragma unroll
    for (int i = 0; i < 16 / N; ++i) Pack<T>::unpack(ld_stream(p + e + N * i), f + N * i);
  } else {
#pragma unroll
    for (int i = 0; i < 16; ++i) f[i] = (e + i < nelem) ? float(p[e + i]) : 0.f;
  }
}

template <typename T>
__device__ __forceinline__ void store16(T* p, size_t e, size_t nelem, const float* f) {
  constexpr int N = Pack<T>::N;
  if (e + 16 <= nelem) {
#pragma unroll
    for (int i = 0; i < 16 / N; ++i) st_stream(p + e + N * i, Pack<T>::pack(f + N * i));
  } else {
#pragma unroll
    for (int i = 0; i < 16; ++i)
      if (e + i < nelem) p[e + i] = T(f[i]);
  }
}

// 16 floats -> 16 e4m3 bytes (one Vec16), with multiplier m = 448/absmax.
__device__ __forceinline__ Vec16 quant16(const float* f, float m) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __nv_fp8x2_storage_t lo = __nv_cvt_float2_to_fp8x2(
        make_float2(f[4 * i] * m, f[4 * i + 1] * m), __NV_SATFINITE, __NV_E4M3);
    const __nv_fp8x2_storage_t hi = __nv_cvt_float2_to_fp8x2(
        make_float2(f[4 * i + 2] * m, f[4 * i + 3] * m), __NV_SATFINITE, __NV_E4M3);
    w[i] = (uint32_t)lo | ((uint32_t)hi << 16);
  }
  return Vec16{w[0], w[1], w[2], w[3]};
}

// 16 e4m3 bytes -> 16 floats (exact: every e4m3 value is a half).
__device__ __forceinline__ void decode16(const Vec16& v, float* f) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __half2_raw a = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w[i] & 0xffff), __NV_E4M3);
    const __half2_raw b = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w[i] >> 16), __NV_E4M3);
    const float2 fa = __half22float2(*reinterpret_cast<const __half2*>(&a));
    const float2 fb = __half22float2(*reinterpret_cast<const __half2*>(&b));
    f[4 * i] = fa.x;
    f[4 * i + 1] = fa.y;
    f[4 * i + 2] = fb.x;
    f[4 * i + 3] = fb.y;
  }
}

// 16 e4m3 bytes -> 16 floats times dequant scale s.
__device__ __forceinline__ void dequant16(const Vec16& v, float s, float* f) {
  decode16(v, f);
#pragma unroll
  for (int i = 0; i < 16; ++i) f[i] = __fmul_rn(f[i], s);
}

// acc += code * s with a separately rounded multiply and add: the sum of a reduction is then fixed bit for bit (no
// contraction into an FMA left to the compiler), so every rank and the tests' CPU emulation agree on it.
__device__ __forceinline__ void dequant16_add(const Vec16& v, float s, float* acc) {
  float f[16];
  decode16(v, f);
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = __fadd_rn(acc[i], __fmul_rn(f[i], s));
}

// Floor of a group's absmax. With amax >= 2^-116 the dequant scale s = amax/448 >= 2^-124.8 is a normal fp32 (so FTZ
// cannot zero it; 2^-117 is the smallest power of two that would do) and m = 448/amax <= 2^124.8 is finite (an
// infinite m turns the group's zeros into 0 * inf = NaN). A power of two keeps s and m exact scalings of fl(1/448) and
// 448. Groups below the floor get codes below 448; their largest element still dequantises to itself +-1/16.
constexpr float kAmaxFloor = 0x1p-116f;

// Quantise one group held as 16 floats/lane across a warp; returns dequant scale.
// A group whose absmax is inf (or an inf next to NaN) gets scale NaN: it dequantises to NaN, like the unquantised sum
// of an inf would be non-finite, instead of saturating to a finite +-448 * scale. NaN elements of an otherwise finite
// group are ignored by fmaxf and become NaN codes.
__device__ __forceinline__ float group_quant(const float* f, Vec16* q) {
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) amax = fmaxf(amax, fabsf(f[i]));
  amax = fmaxf(warp_max(amax), kAmaxFloor);
  const float s = amax < INFINITY ? __fmul_rn(amax, 1.f / kFp8Max) : __int_as_float(0x7fc00000);
  const float m = __fdiv_rn(kFp8Max, amax);  // exact division (fast math would approximate it); 0 for an inf amax
  *q = quant16(f, m);
  return s;
}

__host__ __device__ __forceinline__ size_t q8_payload_off(size_t ngroups) {
  return (ngroups * sizeof(float) + 15) & ~size_t(15);
}

// ------------------------------- standalone ---------------------------------
template <typename T>
__global__ void __launch_bounds__(512) q8_quantize_kernel(const T* a, const T* b, size_t nelem,
                                                          size_t ngroups, char* qbuf) {
  float* scales = reinterpret_cast<float*>(qbuf);
  char* payload = qbuf + q8_payload_off(ngroups);
  const int lane = threadIdx.x & 31;
  const size_t warps = (size_t)gridDim.x * (blockDim.x >> 5);
  for (size_t g = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); g < ngroups;
       g += warps) {
    const size_t e = g * kGroup + lane * 16;
    float f[16];
    load16<T>(a, e, nelem, f);
    if (b != nullptr) {
      float h[16];
      load16<T>(b, e, nelem, h);
#pragma unroll
      for (int i = 0; i < 16; ++i) f[i] -= h[i];
    }
    Vec16 q;
    const float s = group_quant(f, &q);
    if (lane == 0) scales[g] = s;
    st_stream(payload + g * kGroup + lane * 16, q);
  }
}

template <typename T>
__global__ void __launch_bounds__(512) q8_dequantize_kernel(const char* qbuf, size_t ngroups,
                                                            T* out, size_t nelem) {
  const float* scales = reinterpret_cast<const float*>(qbuf);
  const char* payload = qbuf + q8_payload_off(ngroups);
  const int lane = threadIdx.x & 31;
  const size_t warps = (size_t)gridDim.x * (blockDim.x >> 5);
  // a warp takes kU groups per pass and issues all their loads before the first use (one 16 B load in flight per lane
  // leaves the pass latency-bound)
  constexpr int kU = 4;
  for (size_t g0 = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); g0 < ngroups;
       g0 += warps * kU) {
    Vec16 q[kU];
    float sc[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const size_t g = g0 + u * warps;
      if (g < ngroups && g * kGroup + lane * 16 < nelem) {
        q[u] = ld_stream(payload + g * kGroup + lane * 16);
        sc[u] = scales[g];
      }
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const size_t g = g0 + u * warps;
      const size_t e = g * kGroup + lane * 16;
      if (g < ngroups && e < nelem) {
        float f[16];
        dequant16(q[u], sc[u], f);
        store16<T>(out, e, nelem, f);
      }
    }
  }
}

// Reduce `world` quantised buffers (same layout) for groups [g_lo, g_hi) into dst.
__global__ void __launch_bounds__(512) q8_reduce_kernel(const char* const* srcs, int world,
                                                        int first, size_t ngroups, size_t g_lo,
                                                        size_t g_hi, float post_scale, char* dst) {
  const size_t poff = q8_payload_off(ngroups);
  const int lane = threadIdx.x & 31;
  const size_t warps = (size_t)gridDim.x * (blockDim.x >> 5);
  for (size_t g = g_lo + (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); g < g_hi;
       g += warps) {
    float acc[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = 0.f;
    for (int k = 0; k < world; ++k) {
      const int p = (first + k) % world;  // fixed order starting at `first` (ref: quantization.py:405-407)
      const float s = reinterpret_cast<const float*>(srcs[p])[g];
      dequant16_add(ld_stream(srcs[p] + poff + g * kGroup + lane * 16), s, acc);
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = __fmul_rn(acc[i], post_scale);
    Vec16 q;
    const float s = group_quant(acc, &q);
    if (lane == 0) reinterpret_cast<float*>(dst)[g] = s;
    st_stream(dst + poff + g * kGroup + lane * 16, q);
  }
}

// ------------------------------- fused --------------------------------------
struct Q8Args {
  PeerTable pt;
  StatusBlock* st;
  size_t off;          // byte offset of the Q8G buffer in every peer segment
  const void* in_a;    // input (or `original` when in_b != null)
  const void* in_b;    // nullable: subtract (pseudo-gradient = a - b)
  void* out;           // dequantised result (may alias in_a)
  size_t nelem;
  size_t ngroups;      // padded to multiple of world
  float post_scale;    // 1/num_participants for AVG
  uint64_t flag;
  int channel;
  int contribute;
  // mode 0: all-reduce (slices are contiguous runs of groups: slice_elems == groups_per_slice * 512).
  // mode 1: reduce-scatter (torchft/collectives.py:159-294): rank-slice s covers elements
  //         [s * slice_elems, (s+1) * slice_elems), quantised on its own group grid; `out` receives the
  //         fp32-reduced, scaled slice of THIS rank directly (no requantise, no gather phase).
  int mode;
  size_t slice_elems;
};

template <typename T, int W>
__global__ void __launch_bounds__(512, 1) q8_allreduce_kernel(Q8Args a) {
  const int rank = a.pt.rank;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const size_t poff = q8_payload_off(a.ngroups);
  const size_t slice = a.ngroups / W;
  const size_t chunk = (slice + gridDim.x - 1) / gridDim.x;
  char* mine = reinterpret_cast<char*>(a.pt.data[rank]) + a.off;

  // ---- phase A: (delta +) quantise chunk b of every slice into my segment ----
  for (int s = 0; s < W; ++s) {
    const size_t lo = s * slice + blockIdx.x * chunk;
    const size_t hi = min(lo + chunk, (s + 1) * slice);
    for (size_t g = lo + warp; g < hi; g += nwarp) {
      const size_t e = (size_t)s * a.slice_elems + (g - (size_t)s * slice) * kGroup + lane * 16;
      const size_t lim = min(a.nelem, (size_t)(s + 1) * a.slice_elems);
      float f[16];
      if (a.contribute) {
        load16<T>(reinterpret_cast<const T*>(a.in_a), e, lim, f);
        if (a.in_b != nullptr) {
          float h[16];
          load16<T>(reinterpret_cast<const T*>(a.in_b), e, lim, h);
#pragma unroll
          for (int i = 0; i < 16; ++i) f[i] -= h[i];
        }
      } else {
#pragma unroll
        for (int i = 0; i < 16; ++i) f[i] = 0.f;
      }
      Vec16 q;
      const float sc = group_quant(f, &q);
      if (lane == 0) reinterpret_cast<float*>(mine)[g] = sc;
      st_stream(mine + poff + g * kGroup + lane * 16, q);
    }
  }
  if (!block_barrier(a.pt, a.channel, a.flag + 1, a.st, /*release=*/true, /*acquire=*/false)) return;

  // ---- phase B: fp32 reduce of my slice from every peer, requantise, push ----
  {
    const char* src[W];
    char* dst[W];
#pragma unroll
    for (int p = 0; p < W; ++p) {
      // summation starts at own rank and wraps (order determinism, ref quantization.py:405-407)
      src[p] = reinterpret_cast<const char*>(a.pt.data[(rank + p) % W]) + a.off;
      dst[p] = reinterpret_cast<char*>(a.pt.data[(rank + p) % W]) + a.off;
    }
    const size_t lo = rank * slice + blockIdx.x * chunk;
    const size_t hi = min(lo + chunk, (size_t)(rank + 1) * slice);
    for (size_t g = lo + warp; g < hi; g += nwarp) {
      Vec16 qv[W];
      float sv[W];
#pragma unroll
      for (int p = 0; p < W; ++p) {
        qv[p] = ld_stream(src[p] + poff + g * kGroup + lane * 16);
        sv[p] = __ldcv(reinterpret_cast<const float*>(src[p]) + g);  // never trust L1 for peer-written scales
      }
      float acc[16];
      dequant16(qv[0], sv[0], acc);
#pragma unroll
      for (int p = 1; p < W; ++p) dequant16_add(qv[p], sv[p], acc);
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[i] = __fmul_rn(acc[i], a.post_scale);
      if (a.mode == 1) {
        const size_t base = (size_t)rank * a.slice_elems;
        const size_t valid = a.nelem > base ? min(a.slice_elems, a.nelem - base) : 0;
        const size_t le = (g - (size_t)rank * slice) * kGroup + lane * 16;
        if (le < valid) store16<T>(reinterpret_cast<T*>(a.out), le, valid, acc);
        continue;
      }
      Vec16 q;
      const float sc = group_quant(acc, &q);
#pragma unroll
      for (int p = 0; p < W; ++p) {
        if (lane == 0) reinterpret_cast<float*>(dst[p])[g] = sc;
        st_stream(dst[p] + poff + g * kGroup + lane * 16, q);
      }
    }
  }
  if (a.mode == 1) {
    // peers must not requantise their next message over staging we are still reading
    block_barrier(a.pt, a.channel, a.flag + 2, a.st, /*release=*/false, /*acquire=*/false);
    return;
  }
  if (!block_barrier(a.pt, a.channel, a.flag + 2, a.st, /*release=*/true, /*acquire=*/true)) return;

  // ---- phase C: dequantise chunk b of every slice into the output tensor ----
  for (int s = 0; s < W; ++s) {
    const size_t lo = s * slice + blockIdx.x * chunk;
    const size_t hi = min(lo + chunk, (s + 1) * slice);
    for (size_t g = lo + warp; g < hi; g += nwarp) {
      const size_t e = g * kGroup + lane * 16;
      if (e >= a.nelem) continue;
      float f[16];
      dequant16(ld_stream(mine + poff + g * kGroup + lane * 16),
                __ldcv(reinterpret_cast<const float*>(mine) + g), f);
      store16<T>(reinterpret_cast<T*>(a.out), e, a.nelem, f);
    }
  }
}

// ------------------------------- large messages: sync-free phases ---------------------------
// For multi-GB messages (DiLoCo's outer step: the whole model) the fused kernel above is limited by its own structure:
// per-CTA barriers cap the grid at what is co-resident and one warp per group leaves little memory-level parallelism.
// With a scratch segment that holds the whole message in wire format the pipeline is three bandwidth-bound launches
// separated by one-CTA handshakes (zero1.cu):
//     q8_quantize_kernel (any grid)          a - b -> Q8G in MY scratch
//     handshake
//     q8_slice_reduce_kernel (any grid)      my slice of every peer's scratch (P2P loads) -> fp32 sum, scale, requantise -> my R
//     handshake
//     q8_gather_dequant_kernel (any grid)    slice s from peer s's R (P2P loads) -> dequantise -> out   (the all-gather IS the read)
struct Q8Ptrs {
  const char* p[kMaxRanks];
};

__global__ void __launch_bounds__(512) q8_slice_reduce_kernel(Q8Ptrs q, int world, int rank, size_t ngroups, size_t slice,
                                                              float post_scale, char* __restrict__ r_out,
                                                              const int* __restrict__ ok) {
  if (ok != nullptr && *ok == 0) return;
  const size_t poff = q8_payload_off(ngroups), rpoff = q8_payload_off(slice);
  const int lane = threadIdx.x & 31;
  const size_t warps = (size_t)gridDim.x * (blockDim.x >> 5);
  for (size_t l = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); l < slice; l += warps) {
    const size_t g = (size_t)rank * slice + l;
    Vec16 qv[kMaxRanks];
    float sv[kMaxRanks];
#pragma unroll
    for (int k = 0; k < kMaxRanks; ++k) {  // all loads first; summation starts at own rank and wraps (order determinism)
      if (k < world) {
        const char* src = q.p[(rank + k) % world];
        qv[k] = ld_stream(src + poff + g * kGroup + lane * 16);
        sv[k] = __ldcv(reinterpret_cast<const float*>(src) + g);
      }
    }
    float acc[16];
    dequant16(qv[0], sv[0], acc);
#pragma unroll
    for (int k = 1; k < kMaxRanks; ++k) {
      if (k < world) dequant16_add(qv[k], sv[k], acc);
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = __fmul_rn(acc[i], post_scale);
    Vec16 out;
    const float sc = group_quant(acc, &out);
    if (lane == 0) reinterpret_cast<float*>(r_out)[l] = sc;
    st_stream(r_out + rpoff + l * kGroup + lane * 16, out);
  }
}

template <typename T>
__global__ void __launch_bounds__(512) q8_gather_dequant_kernel(Q8Ptrs r, size_t ngroups, size_t slice, T* __restrict__ out,
                                                                size_t nelem, const int* __restrict__ ok) {
  if (ok != nullptr && *ok == 0) return;
  const size_t rpoff = q8_payload_off(slice);
  const int lane = threadIdx.x & 31;
  const size_t warps = (size_t)gridDim.x * (blockDim.x >> 5);
  for (size_t g = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); g < ngroups; g += warps) {
    const size_t e = g * kGroup + lane * 16;
    if (e >= nelem) continue;
    const size_t s = g / slice, l = g - s * slice;
    const char* src = r.p[s];
    float f[16];
    dequant16(ld_stream(src + rpoff + l * kGroup + lane * 16), __ldcv(reinterpret_cast<const float*>(src) + l), f);
    store16<T>(out, e, nelem, f);
  }
}

// ------------------------------- launchers ----------------------------------
size_t q8_ngroups(size_t nelem, int world) {
  size_t g = (nelem + kGroup - 1) / kGroup;
  const size_t w = world < 1 ? 1 : world;
  return (g + w - 1) / w * w;
}
size_t q8_buffer_bytes(size_t nelem, int world) {
  const size_t g = q8_ngroups(nelem, world);
  return q8_payload_off(g) + g * kGroup;
}

static int q8_grid(size_t ngroups, int max_blocks) {
  size_t b = (ngroups + 15) / 16;
  if (b < 1) b = 1;
  if (b > (size_t)max_blocks) b = max_blocks;
  return (int)b;
}

void q8_quantize_launch(const void* a, const void* b, size_t nelem, size_t ngroups, int dtype, void* qbuf,
                        cudaStream_t stream) {
  if (ngroups == 0) return;
  const int grid = q8_grid(ngroups, kNumSMs * 8);
  const bool known_dtype = dispatch<kF32, kBF16, kF16>(dtype, [&](auto D) {
    using T = Elem<D>;
    q8_quantize_kernel<T><<<grid, 512, 0, stream>>>((const T*)a, (const T*)b, nelem, ngroups, (char*)qbuf);
  });
  if (!known_dtype) throw std::runtime_error("q8_quantize: unsupported dtype");
  TFT_CUDA_CHECK(cudaGetLastError());
}

void q8_dequantize_launch(const void* qbuf, size_t ngroups, void* out, size_t nelem, int dtype, cudaStream_t stream) {
  if (ngroups == 0 || nelem == 0) return;
  const int grid = q8_grid(ngroups, kNumSMs * 8);
  const bool known_dtype = dispatch<kF32, kBF16, kF16>(dtype, [&](auto D) {
    using T = Elem<D>;
    q8_dequantize_kernel<T><<<grid, 512, 0, stream>>>((const char*)qbuf, ngroups, (T*)out, nelem);
  });
  if (!known_dtype) throw std::runtime_error("q8_dequantize: unsupported dtype");
  TFT_CUDA_CHECK(cudaGetLastError());
}

void q8_reduce_launch(const void* const* srcs_dev, int nsrc, int first, size_t ngroups, size_t g_lo, size_t g_hi,
                      float post_scale, void* dst, cudaStream_t stream) {
  if (g_hi <= g_lo) return;
  const int grid = q8_grid(g_hi - g_lo, kNumSMs * 8);
  q8_reduce_kernel<<<grid, 512, 0, stream>>>((const char* const*)srcs_dev, nsrc, first, ngroups, g_lo, g_hi,
                                             post_scale, (char*)dst);
  TFT_CUDA_CHECK(cudaGetLastError());
}

void q8_allreduce_launch(const PeerTable& pt, StatusBlock* st, size_t off, const void* in_a,
                         const void* in_b, void* out, size_t nelem, int dtype, float post_scale,
                         uint64_t flag, int channel, int contribute, int blocks, cudaStream_t stream) {
  if (blocks < 1 || blocks > kMaxBlocks) throw std::runtime_error("q8_allreduce: bad grid");
  if (off & 15) throw std::runtime_error("q8_allreduce: offset must be 16 B aligned");
  Q8Args a;
  a.pt = pt;
  a.st = st;
  a.off = off;
  a.in_a = in_a;
  a.in_b = in_b;
  a.out = out;
  a.nelem = nelem;
  a.ngroups = q8_ngroups(nelem, pt.world);
  a.post_scale = post_scale;
  a.flag = flag;
  a.channel = channel;
  a.contribute = contribute;
  a.mode = 0;
  a.slice_elems = a.ngroups / pt.world * kGroup;
  if (pt.world < 2) throw std::runtime_error("q8_allreduce: world must be >= 2");
  const bool known_dtype = dispatch<kF32, kBF16, kF16>(dtype, [&](auto D) {
    const bool known_world = dispatch<2, 3, 4, 5, 6, 7, 8>(pt.world, [&](auto W) {
      q8_allreduce_kernel<Elem<D>, W><<<blocks, 512, 0, stream>>>(a);
    });
    if (!known_world) throw std::runtime_error("q8_allreduce: world size must be in [2, 8]");
  });
  if (!known_dtype) throw std::runtime_error("q8_allreduce: unsupported dtype");
  TFT_CUDA_CHECK(cudaGetLastError());
}

size_t q8_slice_buffer_bytes(size_t nelem, int world) {
  const size_t slice = q8_ngroups(nelem, world) / (world < 1 ? 1 : world);
  return (q8_payload_off(slice) + slice * kGroup + 255) & ~size_t(255);
}

void q8_slice_reduce_launch(const PeerTable& pt, const int* ok, size_t q_off, size_t r_off, size_t nelem, float post_scale,
                            int blocks, cudaStream_t stream) {
  const size_t ng = q8_ngroups(nelem, pt.world), slice = ng / pt.world;
  Q8Ptrs q;
  for (int p = 0; p < kMaxRanks; ++p) q.p[p] = p < pt.world ? reinterpret_cast<const char*>(pt.data[p]) + q_off : nullptr;
  if (blocks < 1) blocks = 1;
  q8_slice_reduce_kernel<<<blocks, 512, 0, stream>>>(q, pt.world, pt.rank, ng, slice, post_scale,
                                                     reinterpret_cast<char*>(pt.data[pt.rank]) + r_off, ok);
  TFT_CUDA_CHECK(cudaGetLastError());
}

void q8_gather_dequant_launch(const PeerTable& pt, const int* ok, size_t r_off, size_t nelem, int dtype, void* out, int blocks,
                              cudaStream_t stream) {
  const size_t ng = q8_ngroups(nelem, pt.world), slice = ng / pt.world;
  Q8Ptrs r;
  for (int p = 0; p < kMaxRanks; ++p) r.p[p] = p < pt.world ? reinterpret_cast<const char*>(pt.data[p]) + r_off : nullptr;
  if (blocks < 1) blocks = 1;
  const bool known_dtype = dispatch<kF32, kBF16, kF16>(dtype, [&](auto D) {
    using T = Elem<D>;
    q8_gather_dequant_kernel<T><<<blocks, 512, 0, stream>>>(r, ng, slice, (T*)out, nelem, ok);
  });
  if (!known_dtype) throw std::runtime_error("q8_gather_dequant: unsupported dtype");
  TFT_CUDA_CHECK(cudaGetLastError());
}

size_t q8_rs_buffer_bytes(size_t slice_elems, int world) {
  const size_t g = (size_t)world * ((slice_elems + kGroup - 1) / kGroup);
  return q8_payload_off(g) + g * kGroup;
}

void q8_reduce_scatter_launch(const PeerTable& pt, StatusBlock* st, size_t off, const void* in, void* out, size_t nelem,
                              size_t slice_elems, int dtype, float post_scale, uint64_t flag, int channel,
                              int contribute, int blocks, cudaStream_t stream) {
  if (blocks < 1 || blocks > kMaxBlocks) throw std::runtime_error("q8_reduce_scatter: bad grid");
  if (off & 15) throw std::runtime_error("q8_reduce_scatter: offset must be 16 B aligned");
  if (pt.world < 2) throw std::runtime_error("q8_reduce_scatter: world must be >= 2");
  const size_t es = dtype == kF32 ? 4 : 2;
  if ((slice_elems * es) & 15) throw std::runtime_error("q8_reduce_scatter: rank slices must be 16 B aligned");
  Q8Args a;
  a.pt = pt;
  a.st = st;
  a.off = off;
  a.in_a = in;
  a.in_b = nullptr;
  a.out = out;
  a.nelem = nelem;
  a.ngroups = (size_t)pt.world * ((slice_elems + kGroup - 1) / kGroup);
  a.post_scale = post_scale;
  a.flag = flag;
  a.channel = channel;
  a.contribute = contribute;
  a.mode = 1;
  a.slice_elems = slice_elems;
  const bool known_dtype = dispatch<kF32, kBF16, kF16>(dtype, [&](auto D) {
    const bool known_world = dispatch<2, 3, 4, 5, 6, 7, 8>(pt.world, [&](auto W) {
      q8_allreduce_kernel<Elem<D>, W><<<blocks, 512, 0, stream>>>(a);
    });
    if (!known_world) throw std::runtime_error("q8_reduce_scatter: world size must be in [2, 8]");
  });
  if (!known_dtype) throw std::runtime_error("q8_reduce_scatter: unsupported dtype");
  TFT_CUDA_CHECK(cudaGetLastError());
}

}  // namespace tft
