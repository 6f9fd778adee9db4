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
  if (!block_barrier(a.pt, a.channel, a.flag + 1, a.st, /*release=*/staged, /*acquire=*/false)) return;

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
    // a message that is not a whole number of vectors ends in one partial vector: it is reduced element by element,
    // because in a user segment the bytes after the message belong to someone else
    const size_t nfull = a.nelem / N;
    const size_t e = nfull * N + threadIdx.x;
    if (lo <= nfull && nfull < hi && e < a.nelem) {
      float acc = float(__ldcg(src[0] + e));
#pragma unroll
      for (int p = 1; p < W; ++p) acc = red<OP>(acc, float(__ldcg(src[p] + e)));
      const T out = T(acc * a.scale);
#pragma unroll
      for (int p = 0; p < W; ++p) dst[p][e] = out;
    }
    const size_t vhi = min(hi, nfull);
    // vectors in flight per thread: peer loads have microseconds of latency, so keep U*W >= 16 outstanding
    constexpr int U = (W >= 8) ? 2 : (W >= 3 ? 4 : 8);
    for (size_t base = lo; base < vhi; base += (size_t)blockDim.x * U) {
      Vec16 in[U][W];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t v = base + threadIdx.x + (size_t)u * blockDim.x;
        if (v < vhi) {
#pragma unroll
          for (int p = 0; p < W; ++p) in[u][p] = ld_stream(src[p] + v * N);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t v = base + threadIdx.x + (size_t)u * blockDim.x;
        if (v < vhi) {
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
  if (!block_barrier(a.pt, a.channel, a.flag + 2, a.st, /*release=*/true, /*acquire=*/a.user_out != nullptr)) return;

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
                     /*acquire=*/false))
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
    block_barrier(a.pt, a.channel, a.flag + 2, a.st, /*release=*/false, /*acquire=*/false);
  } else {
    // In-place in staging: host guarantees chunk <= blockDim.x * kMaxRounds. A partial last vector is reduced and
    // stored element by element (one element per thread), so nothing after the message is written.
    constexpr int kMaxRounds = 8;
    const size_t nfull = a.nelem / N;
    const size_t vhi = min(hi, nfull);
    Vec16 res[kMaxRounds];
#pragma unroll
    for (int r = 0; r < kMaxRounds; ++r) {
      const size_t v = lo + threadIdx.x + (size_t)r * blockDim.x;
      if (v < vhi) {
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
    const size_t e = nfull * N + threadIdx.x;
    const bool tail = lo <= nfull && nfull < hi && e < a.nelem;
    T tail_res = T(0.f);
    if (tail) {
      float acc = float(__ldcg(src[0] + e));
#pragma unroll
      for (int p = 1; p < W; ++p) acc = red<OP>(acc, float(__ldcg(src[p] + e)));
      tail_res = T(acc * a.scale);
    }
    if (!block_barrier(a.pt, a.channel, a.flag + 2, a.st, /*release=*/false, /*acquire=*/false)) return;
#pragma unroll
    for (int r = 0; r < kMaxRounds; ++r) {
      const size_t v = lo + threadIdx.x + (size_t)r * blockDim.x;
      if (v < vhi) st_stream(mine + v * N, res[r]);
    }
    if (tail) mine[e] = tail_res;
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

void allreduce_launch(const PeerTable& pt, StatusBlock* st, size_t off, const void* user_in,
                      void* user_out, size_t nelem, int dtype, int op, float scale,
                      uint64_t flag, int channel, int contribute, int algo, int blocks,
                      int threads, cudaStream_t stream) {
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
  if (algo == 0 && user_out == nullptr) {
    // in-place one-shot keeps results in registers: bound the per-block chunk
    const size_t vecs = (nelem * (dtype == kF32 ? 4 : 2) + 15) / 16;
    const size_t chunk = (vecs + blocks - 1) / blocks;
    if (chunk > (size_t)threads * 8) algo = 1;
  }
  const bool known_dtype = dispatch<kF32, kBF16, kF16>(dtype, [&](auto D) {
    using T = Elem<D>;
    if (pt.world == 1) {
      // Degenerate quorum: out = scale * in (or zeros). The reduce op plays no part.
      const void* src = user_in ? user_in : (const char*)pt.data[0] + off;
      void* dst = user_out ? user_out : (char*)pt.data[0] + off;
      const int g = (int)std::min<size_t>(kNumSMs * 8, (nelem + 4095) / 4096 + 1);
      scale_copy_kernel<T><<<g, 512, 0, stream>>>((T*)dst, (const T*)src, nelem, scale, !contribute);
      return;
    }
    const bool known_op = dispatch<kSum, kMax, kMin>(op, [&](auto OP) {
      const bool known_world = dispatch<2, 3, 4, 5, 6, 7, 8>(pt.world, [&](auto W) {
        if (algo == 0)
          allreduce_oneshot_kernel<T, W, OP><<<blocks, threads, 0, stream>>>(a);
        else
          allreduce_twoshot_kernel<T, W, OP><<<blocks, threads, 0, stream>>>(a);
      });
      if (!known_world) throw std::runtime_error("allreduce: world size must be in [2, 8]");
    });
    if (!known_op) throw std::runtime_error("allreduce: unsupported reduce op");
  });
  if (!known_dtype) throw std::runtime_error("allreduce: unsupported dtype");
  TFT_CUDA_CHECK(cudaGetLastError());
}

}  // namespace tft
