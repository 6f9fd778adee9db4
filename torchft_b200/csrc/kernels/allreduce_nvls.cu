// NVLS (NVSwitch multicast) all-reduce: the switch does the reduction and the broadcast.
//
// Rank r owns slice r of the message. For every 16-byte vector of its slice it issues ONE
// multimem.ld_reduce on the multicast address (the NVSwitch fetches that vector from every
// replica's HBM, adds them in fp32, and returns the sum), applies the fused scale, and issues
// ONE multimem.st (the switch writes the result into every replica's buffer). Per GPU and per
// direction that moves ~S bytes instead of the 2(N-1)/N * S of the P2P two-shot kernel
// (1.75x less at N=8), with no peer pointer arithmetic at all; flags still travel over plain
// peer memory with the same bounded, abortable waits as the P2P kernels.
//
// Requires the message to live in a VMM-backed symmetric segment bound to the quorum's
// multicast object (parallel/symm_mem.py, TORCHFT_B200_SYMM=vmm).
#include <stdexcept>
#include <string>

#include "api.h"
#include "common.cuh"

namespace tft {

template <typename T>
struct MM;

template <>
struct MM<float> {
  __device__ static Vec16 ld_reduce(const void* p) {
    Vec16 r;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p)
                 : "memory");
    return r;
  }
  __device__ static void st(void* p, const Vec16& v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w)
                 : "memory");
  }
};
template <>
struct MM<__nv_bfloat16> {
  __device__ static Vec16 ld_reduce(const void* p) {
    Vec16 r;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p)
                 : "memory");
    return r;
  }
  __device__ static void st(void* p, const Vec16& v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.bf16x2 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y),
                 "r"(v.z), "r"(v.w)
                 : "memory");
  }
};
template <>
struct MM<__half> {
  __device__ static Vec16 ld_reduce(const void* p) {
    Vec16 r;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p)
                 : "memory");
    return r;
  }
  __device__ static void st(void* p, const Vec16& v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f16x2 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w)
                 : "memory");
  }
};

struct NvlsArgs {
  PeerTable pt;      // peers' unicast mappings (flags + own data for the zero-contribution path)
  StatusBlock* st;
  char* mc;          // multicast VA of the segment
  size_t off;        // byte offset of the message inside the segment
  size_t nelem;
  float scale;
  uint64_t flag;
  int channel;
  int contribute;
};

template <typename T>
__global__ void __launch_bounds__(512, 1) allreduce_nvls_kernel(NvlsArgs a) {
  constexpr int N = Pack<T>::N;
  const int W = a.pt.world, rank = a.pt.rank;
  const size_t nvec = (a.nelem + N - 1) / N;
  const size_t slice = (nvec + W - 1) / W;
  const size_t chunk = (slice + gridDim.x - 1) / gridDim.x;

  if (!a.contribute) {
    // the switch cannot skip a replica: a non-participant zeroes its own copy first
    T* mine = reinterpret_cast<T*>(reinterpret_cast<char*>(a.pt.data[rank]) + a.off);
    for (int s = 0; s < W; ++s) {
      const size_t lo = s * slice + blockIdx.x * chunk;
      const size_t hi = min(min(lo + chunk, (size_t)(s + 1) * slice), nvec);
      for (size_t v = lo + threadIdx.x; v < hi; v += blockDim.x) st_stream(mine + v * N, Vec16{0, 0, 0, 0});
    }
  }
  if (!block_barrier(a.pt, a.channel, a.flag + 1, a.st, /*release=*/!a.contribute, /*acquire=*/false))
    return;

  {
    char* base = a.mc + a.off;
    const size_t lo = rank * slice + blockIdx.x * chunk;
    const size_t hi = min(min(lo + chunk, (size_t)(rank + 1) * slice), nvec);
    constexpr int U = 8;
    const bool rescale = a.scale != 1.0f;
    for (size_t b0 = lo; b0 < hi; b0 += (size_t)blockDim.x * U) {
      Vec16 r[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t v = b0 + threadIdx.x + (size_t)u * blockDim.x;
        if (v < hi) r[u] = MM<T>::ld_reduce(base + v * 16);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t v = b0 + threadIdx.x + (size_t)u * blockDim.x;
        if (v < hi) {
          if (rescale) {
            float f[N];
            Pack<T>::unpack(r[u], f);
#pragma unroll
            for (int k = 0; k < N; ++k) f[k] *= a.scale;
            r[u] = Pack<T>::pack(f);
          }
          MM<T>::st(base + v * 16, r[u]);
        }
      }
    }
  }
  block_barrier(a.pt, a.channel, a.flag + 2, a.st, /*release=*/true, /*acquire=*/false);
}

void allreduce_nvls_launch(const PeerTable& pt, StatusBlock* st, void* mc_base, size_t off, size_t nelem, int dtype,
                           float scale, uint64_t flag, int channel, int contribute, int blocks, int threads,
                           cudaStream_t stream) {
  if (blocks < 1 || blocks > kMaxBlocks) throw std::runtime_error("allreduce_nvls: bad grid");
  if (off & 15) throw std::runtime_error("allreduce_nvls: offset must be 16 B aligned");
  if (pt.world < 2) throw std::runtime_error("allreduce_nvls: world must be >= 2");
  NvlsArgs a;
  a.pt = pt;
  a.st = st;
  a.mc = reinterpret_cast<char*>(mc_base);
  a.off = off;
  a.nelem = nelem;
  a.scale = scale;
  a.flag = flag;
  a.channel = channel;
  a.contribute = contribute;
  const bool known_dtype = dispatch<kF32, kBF16, kF16>(dtype, [&](auto D) {
    allreduce_nvls_kernel<Elem<D>><<<blocks, threads, 0, stream>>>(a);
  });
  if (!known_dtype) throw std::runtime_error("allreduce_nvls: unsupported dtype");
  TFT_CUDA_CHECK(cudaGetLastError());
}

}  // namespace tft
