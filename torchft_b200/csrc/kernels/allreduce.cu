// Fault-tolerant all-reduce over NVLink peer memory (sm_90a).
//
// Replaces the reference's `pg.allreduce([t], SUM)` + eager `t /= N`
// (torchft/manager.py:466-478) with ONE kernel that
//   * (optionally) stages the user tensor into the symmetric segment, writing
//     zeros instead when this replica is a non-participant (healing / spare,
//     torchft/manager.py:441-442),
//   * rendezvous with the current healthy replica set through epoch-tagged
//     flags in peer memory (bounded, abortable spins -- never hangs),
//   * reduces its slice straight out of every peer's HBM with 16 B P2P loads,
//     accumulating in fp32 in fixed rank order, applies the 1/num_participants
//     scale and the dtype cast in registers,
//   * pushes the reduced slice to every peer with 16 B P2P stores so both
//     NVLink directions are busy at the same time, and
//   * (optionally) copies the result back to the user tensor.
// No NCCL call is made on this path.
//
// Work decomposition (identical on every rank, which is what makes per-block
// barriers sufficient): the message is cut into `world` slices, each slice into
// `gridDim.x` chunks. Block b owns chunk b of every slice for the staging
// phases and chunk b of slice `rank` for the reduce phase, and only ever
// synchronises with block b of its peers.
#include <stdexcept>
#include <string>

#include "api.h"
#include "common.cuh"

namespace tft {

enum RedOp : int { kSum = 0, kMax = 1, kMin = 2 };

template <int OP>
__device__ __forceinline__ float red(float a, float b) {
  if (OP == kSum) return a + b;
  if (OP == kMax) return fmaxf(a, b);
  return fminf(a, b);
}

struct ARArgs {
  PeerTable pt;
  StatusBlock* st;
  size_t off;            // byte offset of the message inside every peer segment
  const void* user_in;   // nullable: stage from here
  void* user_out;        // nullable: copy result to here
  size_t nelem;          // elements in the message
  float scale;           // fused post-scale (1/num_participants for AVG)
  uint64_t flag;         // barrier values flag+1, flag+2 are consumed
  int channel;
  int contribute;        // 0 => stage zeros (non-participant)
  int barrier_mode;      // memory-ordering recipe of block_barrier
};

template <typename T>
__device__ __forceinline__ void copy_region(T* dst, const T* src, size_t lo, size_t hi,
                                            size_t nelem, bool zero) {
  // [lo, hi) are vector indices (16 B granules) over a message of nelem elements.
  constexpr int N = Pack<T>::N;
  for (size_t v = lo + threadIdx.x; v < hi; v += blockDim.x) {
    const size_t e = v * N;
    if (e + N <= nelem) {
      Vec16 x = zero ? Vec16{0, 0, 0, 0} : ld_stream(src + e);
      st_stream(dst + e, x);
    } else {
      for (size_t k = e; k < nelem; ++k) dst[k] = zero ? T(0.f) : src[k];
    }
  }
}

// ---------------------------------------------------------------------------
// Two-shot: reduce-scatter + all-gather in one kernel, in place in staging.
// ---------------------------------------------------------------------------
template <typename T, int W, int OP>
__global__ void __launch_bounds__(512, 1) allreduce_twoshot_kernel(ARArgs a) {
  constexpr int N = Pack<T>::N;
  const int rank = a.pt.rank;
  const size_t nvec = (a.nelem + N - 1) / N;
  const size_t slice = (nvec + W - 1) / W;                       // vectors per slice
  const size_t chunk = (slice + gridDim.x - 1) / gridDim.x;      // vectors per (slice, block)
  T* mine = reinterpret_cast<T*>(reinterpret_cast<char*>(a.pt.data[rank]) + a.off);

  // ---- phase 0: stage (cast-free) user tensor -> symmetric segment ----
  if (a.user_in != nullptr || !a.contribute) {
    for (int s = 0; s < W; ++s) {
      size_t lo = s * slice + blockIdx.x * chunk;
      size_t hi = min(min(lo + chunk, (s + 1) * slice), nvec);
      if (lo < hi)
        copy_region<T>(mine, reinterpret_cast<const T*>(a.user_in), lo, hi, a.nelem,
                       !a.contribute);
    }
  }
  const bool staged = (a.user_in != nullptr || !a.contribute);
  // peer data read below was produced before the peers' kernels started (or released by their
  // fence when staged) and is only touched with L1-bypassing loads: no acquire fence needed
  if (!block_barrier(a.pt, a.channel, a.flag + 1, a.st, /*release=*/staged, /*acquire=*/false, a.barrier_mode)) return;

  // ---- phase 1+2: reduce my slice from all peers, push result to all peers ----
  {
    // src[] is in rank order (fixed summation order => bitwise identical
    // results wherever a slice is reduced); dst[] is rotated so that ranks do
    // not all hammer the same peer first. The rotation indexes kernel params
    // (constant bank), never a register array.
    const T* src[W];
    T* dst[W];
#pragma unroll
    for (int p = 0; p < W; ++p) {
      src[p] = reinterpret_cast<const T*>(reinterpret_cast<const char*>(a.pt.data[p]) + a.off);
      dst[p] = reinterpret_cast<T*>(reinterpret_cast<char*>(a.pt.data[(rank + p) % W]) + a.off);
    }
    const size_t lo = rank * slice + blockIdx.x * chunk;
    const size_t hi = min(min(lo + chunk, (size_t)(rank + 1) * slice), nvec);
    // vectors in flight per thread: peer loads have microseconds of latency, so keep U*W >= 16 outstanding
    constexpr int U = (W >= 8) ? 2 : (W >= 3 ? 4 : 8);
    for (size_t base = lo; base < hi; base += (size_t)blockDim.x * U) {
      Vec16 in[U][W];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t v = base + threadIdx.x + (size_t)u * blockDim.x;
        if (v < hi) {
#pragma unroll
          for (int p = 0; p < W; ++p) in[u][p] = ld_stream(src[p] + v * N);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t v = base + threadIdx.x + (size_t)u * blockDim.x;
        if (v < hi) {
          float acc[N], f[N];
          Pack<T>::unpack(in[u][0], acc);
#pragma unroll
          for (int p = 1; p < W; ++p) {
            Pack<T>::unpack(in[u][p], f);
#pragma unroll
            for (int k = 0; k < N; ++k) acc[k] = red<OP>(acc[k], f[k]);
          }
#pragma unroll
          for (int k = 0; k < N; ++k) acc[k] *= a.scale;
          const Vec16 out = Pack<T>::pack(acc);
#pragma unroll
          for (int p = 0; p < W; ++p) st_stream(dst[p] + v * N, out);
        }
      }
    }
  }
  if (!block_barrier(a.pt, a.channel, a.flag + 2, a.st, /*release=*/true, /*acquire=*/a.user_out != nullptr, a.barrier_mode)) return;

  // ---- phase 3: symmetric segment -> user tensor ----
  if (a.user_out != nullptr) {
    for (int s = 0; s < W; ++s) {
      size_t lo = s * slice + blockIdx.x * chunk;
      size_t hi = min(min(lo + chunk, (s + 1) * slice), nvec);
      if (lo < hi) copy_region<T>(reinterpret_cast<T*>(a.user_out), mine, lo, hi, a.nelem, false);
    }
  }
}

// ---------------------------------------------------------------------------
// One-shot: every rank reads the whole message from every peer. Latency-bound
// regime (<= a few hundred KB): 2 barriers, no intermediate write.
// ---------------------------------------------------------------------------
template <typename T, int W, int OP>
__global__ void __launch_bounds__(512, 1) allreduce_oneshot_kernel(ARArgs a) {
  constexpr int N = Pack<T>::N;
  const int rank = a.pt.rank;
  const size_t nvec = (a.nelem + N - 1) / N;
  const size_t chunk = (nvec + gridDim.x - 1) / gridDim.x;
  const size_t lo = blockIdx.x * chunk;
  const size_t hi = min(lo + chunk, nvec);
  T* mine = reinterpret_cast<T*>(reinterpret_cast<char*>(a.pt.data[rank]) + a.off);

  if (a.user_in != nullptr || !a.contribute) {
    if (lo < hi)
      copy_region<T>(mine, reinterpret_cast<const T*>(a.user_in), lo, hi, a.nelem, !a.contribute);
  }
  if (!block_barrier(a.pt, a.channel, a.flag + 1, a.st, /*release=*/(a.user_in != nullptr || !a.contribute),
                     /*acquire=*/false, a.barrier_mode))
    return;

  const T* src[W];
#pragma unroll
  for (int p = 0; p < W; ++p)
    src[p] = reinterpret_cast<const T*>(reinterpret_cast<const char*>(a.pt.data[p]) + a.off);
  // Result goes to the user tensor when there is one; otherwise it must not
  // overwrite staging until every peer has finished reading it (barrier 2), so
  // keep it in registers across the barrier: one vector per thread per round.
  T* out = a.user_out ? reinterpret_cast<T*>(a.user_out) : nullptr;
  if (out != nullptr) {
    for (size_t v = lo + threadIdx.x; v < hi; v += blockDim.x) {
      float acc[N], f[N];
      Vec16 in[W];
#pragma unroll
      for (int p = 0; p < W; ++p) in[p] = ld_stream(src[p] + v * N);
      Pack<T>::unpack(in[0], acc);
#pragma unroll
      for (int p = 1; p < W; ++p) {
        Pack<T>::unpack(in[p], f);
#pragma unroll
        for (int k = 0; k < N; ++k) acc[k] = red<OP>(acc[k], f[k]);
      }
#pragma unroll
      for (int k = 0; k < N; ++k) acc[k] *= a.scale;
      const size_t e = v * N;
      if (e + N <= a.nelem) {
        st_stream(out + e, Pack<T>::pack(acc));
      } else {
        for (size_t k = e; k < a.nelem; ++k) out[k] = T(acc[k - e]);
      }
    }
    block_barrier(a.pt, a.channel, a.flag + 2, a.st, /*release=*/false, /*acquire=*/false, a.barrier_mode);
  } else {
    // In-place in staging: host guarantees chunk <= blockDim.x * kMaxRounds.
    constexpr int kMaxRounds = 8;
    Vec16 res[kMaxRounds];
#pragma unroll
    for (int r = 0; r < kMaxRounds; ++r) {
      const size_t v = lo + threadIdx.x + (size_t)r * blockDim.x;
      if (v < hi) {
        float acc[N], f[N];
        Vec16 in[W];
#pragma unroll
        for (int p = 0; p < W; ++p) in[p] = ld_stream(src[p] + v * N);
        Pack<T>::unpack(in[0], acc);
#pragma unroll
        for (int p = 1; p < W; ++p) {
          Pack<T>::unpack(in[p], f);
#pragma unroll
          for (int k = 0; k < N; ++k) acc[k] = red<OP>(acc[k], f[k]);
        }
#pragma unroll
        for (int k = 0; k < N; ++k) acc[k] *= a.scale;
        res[r] = Pack<T>::pack(acc);
      }
    }
    if (!block_barrier(a.pt, a.channel, a.flag + 2, a.st, /*release=*/false, /*acquire=*/false, a.barrier_mode)) return;
#pragma unroll
    for (int r = 0; r < kMaxRounds; ++r) {
      const size_t v = lo + threadIdx.x + (size_t)r * blockDim.x;
      if (v < hi) st_stream(mine + v * N, res[r]);
    }
  }
}

// world == 1 fast path: scale (and copy) only -- still one launch so the
// stream semantics match the multi-rank path.
template <typename T>
__global__ void scale_copy_kernel(T* dst, const T* src, size_t nelem, float scale, int zero) {
  constexpr int N = Pack<T>::N;
  const size_t nvec = nelem / N;
  for (size_t v = blockIdx.x * (size_t)blockDim.x + threadIdx.x; v < nvec;
       v += (size_t)gridDim.x * blockDim.x) {
    float f[N];
    Pack<T>::unpack(ld_stream(src + v * N), f);
#pragma unroll
    for (int k = 0; k < N; ++k) f[k] = zero ? 0.f : f[k] * scale;
    st_stream(dst + v * N, Pack<T>::pack(f));
  }
  if (blockIdx.x == 0) {
    for (size_t k = nvec * N + threadIdx.x; k < nelem; k += blockDim.x)
      dst[k] = zero ? T(0.f) : T(float(src[k]) * scale);
  }
}

template <typename T, int W, int OP>
static void launch_w(const ARArgs& a, int algo, int blocks, int threads, cudaStream_t stream) {
  if (algo == 0)
    allreduce_oneshot_kernel<T, W, OP><<<blocks, threads, 0, stream>>>(a);
  else
    allreduce_twoshot_kernel<T, W, OP><<<blocks, threads, 0, stream>>>(a);
}

template <typename T, int OP>
static void launch_t(const ARArgs& a, int algo, int blocks, int threads, cudaStream_t stream) {
  switch (a.pt.world) {
    case 2: launch_w<T, 2, OP>(a, algo, blocks, threads, stream); break;
    case 3: launch_w<T, 3, OP>(a, algo, blocks, threads, stream); break;
    case 4: launch_w<T, 4, OP>(a, algo, blocks, threads, stream); break;
    case 5: launch_w<T, 5, OP>(a, algo, blocks, threads, stream); break;
    case 6: launch_w<T, 6, OP>(a, algo, blocks, threads, stream); break;
    case 7: launch_w<T, 7, OP>(a, algo, blocks, threads, stream); break;
    case 8: launch_w<T, 8, OP>(a, algo, blocks, threads, stream); break;
    default: throw std::runtime_error("allreduce: world size must be in [2, 8]");
  }
}

template <typename T>
static void launch_op(const ARArgs& a, int op, int algo, int blocks, int threads,
                      cudaStream_t stream) {
  switch (op) {
    case kSum: launch_t<T, kSum>(a, algo, blocks, threads, stream); break;
    case kMax: launch_t<T, kMax>(a, algo, blocks, threads, stream); break;
    case kMin: launch_t<T, kMin>(a, algo, blocks, threads, stream); break;
    default: throw std::runtime_error("allreduce: unsupported reduce op");
  }
}

void allreduce_launch(const PeerTable& pt, StatusBlock* st, size_t off, const void* user_in,
                      void* user_out, size_t nelem, int dtype, int op, float scale,
                      uint64_t flag, int channel, int contribute, int algo, int blocks,
                      int threads, int barrier_mode, cudaStream_t stream) {
  if (blocks < 1 || blocks > kMaxBlocks) throw std::runtime_error("allreduce: bad grid");
  if (threads < 32 || threads > 512 || (threads & 31))
    throw std::runtime_error("allreduce: threads must be a multiple of 32 in [32, 512]");
  if (off & 15) throw std::runtime_error("allreduce: staging offset must be 16 B aligned");
  ARArgs a;
  a.pt = pt;
  a.st = st;
  a.off = off;
  a.user_in = user_in;
  a.user_out = user_out;
  a.nelem = nelem;
  a.scale = scale;
  a.flag = flag;
  a.channel = channel;
  a.contribute = contribute;
  a.barrier_mode = barrier_mode;
  if (pt.world == 1) {
    // Degenerate quorum: out = scale * in (or zeros).
    const void* src = user_in ? user_in : (const char*)pt.data[0] + off;
    void* dst = user_out ? user_out : (char*)pt.data[0] + off;
    const int g = (int)std::min<size_t>(kNumSMs * 8, (nelem + 4095) / 4096 + 1);
    switch (dtype) {
      case kF32:
        scale_copy_kernel<float><<<g, 512, 0, stream>>>((float*)dst, (const float*)src, nelem,
                                                        scale, !contribute);
        break;
      case kBF16:
        scale_copy_kernel<__nv_bfloat16><<<g, 512, 0, stream>>>(
            (__nv_bfloat16*)dst, (const __nv_bfloat16*)src, nelem, scale, !contribute);
        break;
      case kF16:
        scale_copy_kernel<__half><<<g, 512, 0, stream>>>((__half*)dst, (const __half*)src, nelem,
                                                         scale, !contribute);
        break;
      default: throw std::runtime_error("allreduce: unsupported dtype");
    }
    TFT_CUDA_CHECK(cudaGetLastError());
    return;
  }
  if (algo == 0 && user_out == nullptr) {
    // in-place one-shot keeps results in registers: bound the per-block chunk
    const size_t vecs = (nelem * (dtype == kF32 ? 4 : 2) + 15) / 16;
    const size_t chunk = (vecs + blocks - 1) / blocks;
    if (chunk > (size_t)threads * 8) algo = 1;
  }
  switch (dtype) {
    case kF32: launch_op<float>(a, op, algo, blocks, threads, stream); break;
    case kBF16: launch_op<__nv_bfloat16>(a, op, algo, blocks, threads, stream); break;
    case kF16: launch_op<__half>(a, op, algo, blocks, threads, stream); break;
    default: throw std::runtime_error("allreduce: unsupported dtype");
  }
  TFT_CUDA_CHECK(cudaGetLastError());
}

}  // namespace tft
