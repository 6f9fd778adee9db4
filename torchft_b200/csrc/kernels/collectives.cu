// The rest of the c10d collective surface as peer-memory kernels (sm_90a): all-gather, broadcast,
// all-to-all (one "push exchange" kernel), reduce-scatter, and point-to-point send / recv.
//
// The reference forwards every one of these to a stock backend that is re-created per quorum
// (upstream torchft/process_group.py:510-629); its heal-over-process-group transport is built
// on send/recv (upstream torchft/checkpointing/pg_transport.py:214-303) and its quantised
// reduce-scatter on alltoall (upstream torchft/collectives.py:159-294). Here each is ONE launch
// that moves exactly the algorithmic bytes over NVLink with P2P stores/loads issued by the kernel:
//
//   push exchange   rank r stores what it owes peer p straight into p's staging slot r, one barrier,
//                   every rank copies its slots out. all-gather: everybody owes everybody the same
//                   n bytes; broadcast: only the root owes; all-to-all: chunk p of the input.
//   reduce-scatter  stage the W*n input (skipped when it already lives in symmetric memory), one barrier,
//                   reduce slot `rank` out of every peer's HBM in fixed rank order (fp32 accumulate),
//                   fused scale + cast, write n elements locally. Half of a two-shot all-reduce.
//   send / recv     a mailbox per ordered pair inside the receiver's staging segment, pieces of <= 4 MiB,
//                   data-ready / ack flags per CTA with pair-local sequence numbers (only the two ranks
//                   involved take part, so the quorum-wide flag counter is not touched).
//
// Same failure containment as the all-reduce kernels: epoch-tagged flags, bounded abortable spins, errors
// latched in the status block.
#include <stdexcept>
#include <string>

#include "api.h"
#include "common.cuh"

namespace tft {

namespace {

// Copy `n` bytes; 16-byte vectors with 4 loads in flight when both ends are 16 B aligned.
__device__ __forceinline__ void copy_bytes(char* dst, const char* src, size_t n) {
  if ((((uintptr_t)dst | (uintptr_t)src) & 15) == 0) {
    const size_t nv = n / 16;
    constexpr int U = 4;
    size_t v = threadIdx.x;
    for (; v + (size_t)(U - 1) * blockDim.x < nv; v += (size_t)U * blockDim.x) {
      Vec16 r[U];
#pragma unroll
      for (int u = 0; u < U; ++u) r[u] = ld_stream(src + (v + (size_t)u * blockDim.x) * 16);
#pragma unroll
      for (int u = 0; u < U; ++u) st_stream(dst + (v + (size_t)u * blockDim.x) * 16, r[u]);
    }
    for (; v < nv; v += blockDim.x) st_stream(dst + v * 16, ld_stream(src + v * 16));
    for (size_t k = nv * 16 + threadIdx.x; k < n; k += blockDim.x) dst[k] = src[k];
  } else {
    for (size_t k = threadIdx.x; k < n; k += blockDim.x) dst[k] = src[k];
  }
}

// chunk b of a message of n bytes cut into gridDim.x pieces on 16-byte boundaries
__device__ __forceinline__ void my_chunk(size_t n, size_t* lo, size_t* hi) {
  const size_t per = ((n + gridDim.x - 1) / gridDim.x + 15) & ~size_t(15);
  *lo = min((size_t)blockIdx.x * per, n);
  *hi = min(*lo + per, n);
}

struct XArgs {
  PeerTable pt;              // data[] = staging of every rank
  StatusBlock* st;
  const char* in;            // local input
  char* out;                 // local output
  size_t send_off[kMaxRanks];  // bytes: what I owe peer p starts here in `in`
  size_t send_len[kMaxRanks];
  size_t recv_len[kMaxRanks];  // bytes I get from peer p
  size_t out_off[kMaxRanks];   // where they go in `out`
  size_t slot_stride;        // staging bytes per source rank
  uint64_t flag;             // consumes flag+1, flag+2
  int channel;
  int barrier_mode;
};

__global__ void __launch_bounds__(512, 1) push_exchange_kernel(XArgs a) {
  const int rank = a.pt.rank, W = a.pt.world;
  // ---- push: my slot on every peer (rotated start so ranks do not all hammer the same peer first) ----
  for (int i = 0; i < W; ++i) {
    const int p = (rank + i) % W;
    if (a.send_len[p] == 0) continue;
    size_t lo, hi;
    my_chunk(a.send_len[p], &lo, &hi);
    if (lo < hi)
      copy_bytes(reinterpret_cast<char*>(a.pt.data[p]) + (size_t)rank * a.slot_stride + lo, a.in + a.send_off[p] + lo, hi - lo);
  }
  if (!block_barrier(a.pt, a.channel, a.flag + 1, a.st, /*release=*/true, /*acquire=*/true, a.barrier_mode)) return;
  // ---- copy out: every source's slot of my staging ----
  const char* mine = reinterpret_cast<const char*>(a.pt.data[rank]);
  for (int p = 0; p < W; ++p) {
    if (a.recv_len[p] == 0) continue;
    size_t lo, hi;
    my_chunk(a.recv_len[p], &lo, &hi);
    if (lo < hi) copy_bytes(a.out + a.out_off[p] + lo, mine + (size_t)p * a.slot_stride + lo, hi - lo);
  }
  // nobody may start overwriting my staging (next collective) before I have copied it out
  block_barrier(a.pt, a.channel, a.flag + 2, a.st, /*release=*/false, /*acquire=*/false, a.barrier_mode);
}

enum RedOp : int { kSum = 0, kMax = 1, kMin = 2 };
template <int OP>
__device__ __forceinline__ float red(float x, float y) {
  if (OP == kSum) return x + y;
  if (OP == kMax) return fmaxf(x, y);
  return fminf(x, y);
}

struct RSArgs {
  PeerTable pt;          // data[] = the buffer holding every rank's W*n input (staging or a user segment)
  StatusBlock* st;
  size_t off;            // byte offset of that buffer in the segment
  const void* user_in;   // nullable: stage from here first
  void* out;             // n elements, local
  size_t n;              // elements per rank
  float scale;
  uint64_t flag;
  int channel;
  int barrier_mode;
};

template <typename T, int W, int OP>
__global__ void __launch_bounds__(512, 1) reduce_scatter_kernel(RSArgs a) {
  constexpr int N = Pack<T>::N;
  const int rank = a.pt.rank;
  T* mine = reinterpret_cast<T*>(reinterpret_cast<char*>(a.pt.data[rank]) + a.off);
  // CTA b owns elements [lo, hi) of EVERY slot, in the staging phase and in the reduce phase alike: the per-CTA barrier
  // then orders exactly the bytes this CTA reads from its peers (they were staged by the peers' CTA b).
  const size_t per = (((a.n + gridDim.x - 1) / gridDim.x) + N - 1) / N * N;
  const size_t lo = min((size_t)blockIdx.x * per, a.n), hi = min(lo + per, a.n);
  if (a.user_in != nullptr && lo < hi) {
    const T* in = reinterpret_cast<const T*>(a.user_in);
    for (int s = 0; s < W; ++s)
      copy_bytes(reinterpret_cast<char*>(mine + (size_t)s * a.n + lo), reinterpret_cast<const char*>(in + (size_t)s * a.n + lo),
                 (hi - lo) * sizeof(T));
  }
  if (!block_barrier(a.pt, a.channel, a.flag + 1, a.st, /*release=*/a.user_in != nullptr, /*acquire=*/false, a.barrier_mode)) return;
  {
    const T* src[W];
#pragma unroll
    for (int p = 0; p < W; ++p)
      src[p] = reinterpret_cast<const T*>(reinterpret_cast<const char*>(a.pt.data[p]) + a.off) + (size_t)rank * a.n;
    T* out = reinterpret_cast<T*>(a.out);
    const bool vec_ok = ((a.n * sizeof(T)) % 16 == 0) && (((uintptr_t)out & 15) == 0);
    if (vec_ok) {
      for (size_t v = lo / N + threadIdx.x; v * N < hi; v += blockDim.x) {
        if (v * N + N <= hi) {
          Vec16 in[W];
#pragma unroll
          for (int p = 0; p < W; ++p) in[p] = ld_stream(src[p] + v * N);
          float acc[N], f[N];
          Pack<T>::unpack(in[0], acc);
#pragma unroll
          for (int p = 1; p < W; ++p) {
            Pack<T>::unpack(in[p], f);
#pragma unroll
            for (int k = 0; k < N; ++k) acc[k] = red<OP>(acc[k], f[k]);
          }
#pragma unroll
          for (int k = 0; k < N; ++k) acc[k] *= a.scale;
          st_stream(out + v * N, Pack<T>::pack(acc));
        } else {  // n is a multiple of 16 bytes but not of the vector width of this CTA's last group: cannot happen (per % N == 0)
          for (size_t e = v * N; e < hi; ++e) {
            float acc = float(src[0][e]);
#pragma unroll
            for (int p = 1; p < W; ++p) acc = red<OP>(acc, float(src[p][e]));
            out[e] = T(acc * a.scale);
          }
        }
      }
    } else {  // odd sizes: slots start at unaligned addresses, scalar path over the same element range
      for (size_t e = lo + threadIdx.x; e < hi; e += blockDim.x) {
        float acc = float(src[0][e]);
#pragma unroll
        for (int p = 1; p < W; ++p) acc = red<OP>(acc, float(src[p][e]));
        out[e] = T(acc * a.scale);
      }
    }
  }
  block_barrier(a.pt, a.channel, a.flag + 2, a.st, /*release=*/false, /*acquire=*/false, a.barrier_mode);
}

// ---------------------------------------------------------------------------
// point to point
// ---------------------------------------------------------------------------
constexpr int kP2PBlocks = 8;
constexpr int kP2PDataSlot = 16;                 // sig[ch][kP2PDataSlot + b][src]  on the receiver's pad
constexpr int kP2PAckSlot = 16 + kP2PBlocks;     // sig[ch][kP2PAckSlot + b][dst]   on the sender's pad

struct P2PArgs {
  PeerTable pt;         // data[] = staging of every rank (mailboxes live at mailbox_off + src * mailbox_bytes)
  StatusBlock* st;
  char* buf;            // user buffer (source for send, destination for recv)
  size_t nbytes;
  size_t mailbox_off;
  size_t mailbox_bytes;
  uint64_t seq0;        // pair-local sequence number of the first piece (epoch-tagged, > 0)
  int peer;
  int channel;
};

// CTA b always owns the SAME byte range of the mailbox, whatever the piece length: its data-ready / ack flags then
// order exactly the bytes it touches (a length-dependent split let CTA b of a short last piece overwrite bytes that CTA b'
// of the receiver was still copying out of the previous piece).
__device__ __forceinline__ void piece_chunk(size_t mailbox_bytes, size_t piece_len, size_t* lo, size_t* hi) {
  const size_t per = ((mailbox_bytes + kP2PBlocks - 1) / kP2PBlocks + 15) & ~size_t(15);
  *lo = min((size_t)blockIdx.x * per, piece_len);
  *hi = min(*lo + per, piece_len);
}

__global__ void __launch_bounds__(512, 1) p2p_send_kernel(P2PArgs a) {
  const int rank = a.pt.rank;
  char* box = reinterpret_cast<char*>(a.pt.data[a.peer]) + a.mailbox_off + (size_t)rank * a.mailbox_bytes;
  uint64_t* ready = &a.pt.pads[a.peer]->sig[a.channel][kP2PDataSlot + blockIdx.x][rank];
  const uint64_t* acked = &a.pt.pads[rank]->sig[a.channel][kP2PAckSlot + blockIdx.x][a.peer];
  __shared__ int ok_s;
  uint64_t q = a.seq0;
  for (size_t done = 0; done < a.nbytes; done += a.mailbox_bytes, ++q) {
    const size_t len = min(a.mailbox_bytes, a.nbytes - done);
    if ((q & 0xffffffffull) > 1) {
      // the mailbox still holds the previous piece until the receiver acknowledged it
      if (threadIdx.x == 0) ok_s = wait_flag(acked, q - 1, a.st, a.peer, a.pt.timeout_ns) ? 1 : 0;
      __syncthreads();
      if (!ok_s) return;
    }
    size_t lo, hi;
    piece_chunk(a.mailbox_bytes, len, &lo, &hi);
    if (lo < hi) copy_bytes(box + lo, a.buf + done + lo, hi - lo);
    __syncthreads();
    if (threadIdx.x == 0) {
      fence_acq_rel_sys();
      st_release_sys(ready, q);
    }
  }
}

__global__ void __launch_bounds__(512, 1) p2p_recv_kernel(P2PArgs a) {
  const int rank = a.pt.rank;
  const char* box = reinterpret_cast<const char*>(a.pt.data[rank]) + a.mailbox_off + (size_t)a.peer * a.mailbox_bytes;
  const uint64_t* ready = &a.pt.pads[rank]->sig[a.channel][kP2PDataSlot + blockIdx.x][a.peer];
  uint64_t* acked = &a.pt.pads[a.peer]->sig[a.channel][kP2PAckSlot + blockIdx.x][rank];
  __shared__ int ok_s;
  uint64_t q = a.seq0;
  for (size_t done = 0; done < a.nbytes; done += a.mailbox_bytes, ++q) {
    const size_t len = min(a.mailbox_bytes, a.nbytes - done);
    if (threadIdx.x == 0) {
      ok_s = wait_flag(ready, q, a.st, a.peer, a.pt.timeout_ns) ? 1 : 0;
      fence_acq_rel_sys();
    }
    __syncthreads();
    if (!ok_s) return;
    size_t lo, hi;
    piece_chunk(a.mailbox_bytes, len, &lo, &hi);
    if (lo < hi) copy_bytes(a.buf + done + lo, box + lo, hi - lo);
    __syncthreads();
    if (threadIdx.x == 0) {
      fence_acq_rel_sys();
      st_release_sys(acked, q);
    }
  }
}

template <typename T, int OP>
void launch_rs_w(const RSArgs& a, int blocks, cudaStream_t s) {
  switch (a.pt.world) {
    case 2: reduce_scatter_kernel<T, 2, OP><<<blocks, 512, 0, s>>>(a); break;
    case 3: reduce_scatter_kernel<T, 3, OP><<<blocks, 512, 0, s>>>(a); break;
    case 4: reduce_scatter_kernel<T, 4, OP><<<blocks, 512, 0, s>>>(a); break;
    case 5: reduce_scatter_kernel<T, 5, OP><<<blocks, 512, 0, s>>>(a); break;
    case 6: reduce_scatter_kernel<T, 6, OP><<<blocks, 512, 0, s>>>(a); break;
    case 7: reduce_scatter_kernel<T, 7, OP><<<blocks, 512, 0, s>>>(a); break;
    case 8: reduce_scatter_kernel<T, 8, OP><<<blocks, 512, 0, s>>>(a); break;
    default: throw std::runtime_error("reduce_scatter: world size must be in [2, 8]");
  }
}
template <typename T>
void launch_rs_op(const RSArgs& a, int op, int blocks, cudaStream_t s) {
  switch (op) {
    case kSum: launch_rs_w<T, kSum>(a, blocks, s); break;
    case kMax: launch_rs_w<T, kMax>(a, blocks, s); break;
    case kMin: launch_rs_w<T, kMin>(a, blocks, s); break;
    default: throw std::runtime_error("reduce_scatter: unsupported reduce op");
  }
}

}  // namespace

void push_exchange_launch(const PeerTable& pt, StatusBlock* st, const void* in, void* out, const size_t* send_off,
                          const size_t* send_len, const size_t* recv_len, const size_t* out_off, size_t slot_stride,
                          uint64_t flag, int channel, int blocks, int barrier_mode, cudaStream_t stream) {
  if (blocks < 1 || blocks > kMaxBlocks) throw std::runtime_error("push_exchange: bad grid");
  if (slot_stride & 15) throw std::runtime_error("push_exchange: slot stride must be a multiple of 16 bytes");
  XArgs a;
  a.pt = pt;
  a.st = st;
  a.in = reinterpret_cast<const char*>(in);
  a.out = reinterpret_cast<char*>(out);
  for (int p = 0; p < kMaxRanks; ++p) {
    const bool live = p < pt.world;
    a.send_off[p] = live ? send_off[p] : 0;
    a.send_len[p] = live ? send_len[p] : 0;
    a.recv_len[p] = live ? recv_len[p] : 0;
    a.out_off[p] = live ? out_off[p] : 0;
    if (live && (send_len[p] > slot_stride || recv_len[p] > slot_stride))
      throw std::runtime_error("push_exchange: message larger than its staging slot");
  }
  a.slot_stride = slot_stride;
  a.flag = flag;
  a.channel = channel;
  a.barrier_mode = barrier_mode;
  push_exchange_kernel<<<blocks, 512, 0, stream>>>(a);
  TFT_CUDA_CHECK(cudaGetLastError());
}

void reduce_scatter_launch(const PeerTable& pt, StatusBlock* st, size_t off, const void* user_in, void* out, size_t n,
                           int dtype, int op, float scale, uint64_t flag, int channel, int blocks, int barrier_mode,
                           cudaStream_t stream) {
  if (blocks < 1 || blocks > kMaxBlocks) throw std::runtime_error("reduce_scatter: bad grid");
  if (off & 15) throw std::runtime_error("reduce_scatter: offset must be 16 B aligned");
  RSArgs a{pt, st, off, user_in, out, n, scale, flag, channel, barrier_mode};
  switch (dtype) {
    case kF32: launch_rs_op<float>(a, op, blocks, stream); break;
    case kBF16: launch_rs_op<__nv_bfloat16>(a, op, blocks, stream); break;
    case kF16: launch_rs_op<__half>(a, op, blocks, stream); break;
    default: throw std::runtime_error("reduce_scatter: unsupported dtype");
  }
  TFT_CUDA_CHECK(cudaGetLastError());
}

void p2p_launch(const PeerTable& pt, StatusBlock* st, int is_send, void* buf, size_t nbytes, int peer, size_t mailbox_off,
                size_t mailbox_bytes, uint64_t seq0, int channel, cudaStream_t stream) {
  if (peer < 0 || peer >= pt.world || peer == pt.rank) throw std::runtime_error("p2p: bad peer");
  if (nbytes == 0) return;
  if ((mailbox_off & 15) || (mailbox_bytes & 15) || mailbox_bytes == 0) throw std::runtime_error("p2p: bad mailbox geometry");
  P2PArgs a{pt, st, reinterpret_cast<char*>(buf), nbytes, mailbox_off, mailbox_bytes, seq0, peer, channel};
  if (is_send)
    p2p_send_kernel<<<kP2PBlocks, 512, 0, stream>>>(a);
  else
    p2p_recv_kernel<<<kP2PBlocks, 512, 0, stream>>>(a);
  TFT_CUDA_CHECK(cudaGetLastError());
}

}  // namespace tft
