// Shared device helpers for the torchft_b200 data-plane kernels (sm_90a only).
//
// Everything here is header-only and free of torch/ATen dependencies: the
// Python side hands us raw device pointers + CUDA stream handles, so this
// extension builds in seconds with plain nvcc and has no libtorch ABI coupling.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace tft {

constexpr int kMaxRanks = 8;          // one NVSwitch domain (HGX H100)
constexpr int kNumSMs = 132;          // H100 SXM; sizes the grid caps of the bandwidth-bound kernels
constexpr int kMaxBlocks = 2 * kNumSMs;  // 2 CTAs / SM upper bound for comm grids
constexpr int kSignalChannels = 4;    // independent flag arrays (allreduce / q8 / heal / user)

// dtype codes shared with Python (torchft_b200/ops/_dtypes.py)
enum DType : int { kF32 = 0, kBF16 = 1, kF16 = 2 };

// ---------------------------------------------------------------------------
// Status block: lives in host-pinned, device-mapped memory. The host can flip
// `abort` at any time (ProcessGroup.abort()); kernels poll it inside every
// bounded spin and latch `error` instead of hanging when a peer disappears.
// This is the in-kernel analogue of ncclCommAbort (reference:
// torchft/process_group.py:473-501).
// ---------------------------------------------------------------------------
struct StatusBlock {
  volatile uint32_t abort;        // host -> device: bail out of all spins
  volatile uint32_t error;        // device -> host: 0 ok, 1 timeout, 2 aborted
  volatile uint32_t error_rank;   // peer we were waiting for when we gave up
  volatile uint32_t error_seq;    // low 32 bits of the flag we waited for
  volatile uint64_t timeout_ns;   // host -> device: spin budget per wait
  volatile uint64_t launches;     // device -> host: kernels completed (debug)
  // device -> host: commit verdicts of the device-side commit kernel (zero1.cu). Slot seq % ring
  // holds (seq << 1) | verdict, so the host can tell a stale slot from the one it is waiting for.
  volatile uint32_t verdict[64];
};
constexpr uint32_t kVerdictRing = 64;

enum ErrCode : uint32_t { kOk = 0, kErrTimeout = 1, kErrAborted = 2 };

// One per rank, allocated inside the symmetric segment so peers can write it.
// sig[channel][block][src_rank]; 64-bit epoch-tagged sequence numbers:
//   flag = (quorum_epoch << 32) | seq
// Values from older quorums compare smaller and are ignored, so a zombie
// replica that was evicted can never satisfy a wait of the current quorum and
// the pad never needs to be zeroed on reconfiguration.
struct SignalPad {
  uint64_t sig[kSignalChannels][kMaxBlocks][kMaxRanks];
};

// Peer table passed by value to kernels (fits in constant bank / params).
struct PeerTable {
  void* data[kMaxRanks];          // peer staging buffers (same layout on every rank)
  SignalPad* pads[kMaxRanks];     // peer signal pads
  int rank;
  int world;
  // Spin budget per wait, BY VALUE: every waiter reading it (and the error word) from the
  // host-mapped status block would cost a PCIe round trip per CTA, serialised over PCIe.
  uint64_t timeout_ns;
};

// ---------------------------------------------------------------------------
// Memory-model helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ void st_release_sys(uint64_t* p, uint64_t v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t ld_acquire_sys(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint64_t ld_relaxed_sys(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// 16-byte streaming accesses. Peer (NVLink) addresses bypass the local L2 and
// we touch every byte once, so don't pollute L1 either.
struct alignas(16) Vec16 {
  uint32_t x, y, z, w;
};
__device__ __forceinline__ Vec16 ld_stream(const void* p) {
  Vec16 r;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
__device__ __forceinline__ void st_stream(void* p, const Vec16& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

// ---------------------------------------------------------------------------
// Bounded, abortable wait on a peer flag. Returns false on timeout/abort and
// latches the error into the status block; the caller must then skip the rest
// of the collective (results are garbage; Manager discards the step).
// ---------------------------------------------------------------------------
__device__ __forceinline__ void fence_acq_rel_sys() {
  asm volatile("fence.acq_rel.sys;" ::: "memory");
}
__device__ __forceinline__ void st_relaxed_sys(uint64_t* p, uint64_t v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// Poll a peer flag with RELAXED loads (no fence per poll). Returns false on
// timeout/abort, or immediately when an earlier collective already latched an
// error (so a dead peer costs ONE timeout, not one per queued kernel).
__device__ __forceinline__ bool wait_flag(const uint64_t* flag, uint64_t expected,
                                          StatusBlock* st, int peer, uint64_t budget_ns) {
  // Hot path touches ONLY the flag (local HBM/L2). The host-mapped status block (abort /
  // latched error) is consulted every 256 polls, the clock every 1024.
  if (ld_relaxed_sys(flag) >= expected) return true;
  uint64_t t0 = 0;
  uint32_t spins = 0;
  while (true) {
    if (ld_relaxed_sys(flag) >= expected) return true;
    ++spins;
    if ((spins & 0xff) == 0) {
      if (st->abort || st->error != kOk) {
        if (st->error == kOk) {
          st->error_rank = peer;
          st->error_seq = (uint32_t)expected;
          st->error = kErrAborted;
        }
        return false;
      }
      if ((spins & 0x3ff) == 0) {
        const uint64_t now = globaltimer_ns();
        if (t0 == 0) t0 = now;
        if (now - t0 > budget_ns) {
          st->error_rank = peer;
          st->error_seq = (uint32_t)expected;
          st->error = kErrTimeout;
          __threadfence_system();
          return false;
        }
      }
    }
    __nanosleep(20);
  }
}

// Block-granular barrier across ranks on channel `ch`: block b of every rank
// rendezvous with block b of every peer; threads 0..world-1 each own one peer.
//
//   release: this CTA wrote data (to its own or to peer memory) that peers read
//            after the barrier. Not needed when the data was produced by an
//            earlier kernel (kernel boundaries already order it).
//   acquire: this CTA reads peer-written data after the barrier within this
//            kernel (all such loads bypass L1).
//
// `mode` selects the memory-ordering recipe (tuned on hardware, bench/comm_tune.py):
//   0  per-peer thread: [fence.sc.sys if release] st.release.sys ; poll ld.acquire.sys
//   1  per-peer thread: st.release.sys ; poll ld.relaxed.sys ; fence.acq_rel.sys
//   2  per-peer thread (all in warp 0): [fence.acq_rel.sys if release] ; st.relaxed.sys ; poll relaxed ;
//      [fence.acq_rel.sys if acquire]        (<= 2 warp-wide system fences per CTA, each in program order with its flag access)
//   3  like 2 but the flag is published with red.release.sys (atomic max) so the
//      store cannot linger in a write-combining path
__device__ __forceinline__ bool wait_flag_acquire(const uint64_t* flag, uint64_t expected,
                                                  StatusBlock* st, int peer, uint64_t budget) {
  if (ld_acquire_sys(flag) >= expected) return true;
  uint64_t t0 = 0;
  uint32_t spins = 0;
  while (true) {
    if (ld_acquire_sys(flag) >= expected) return true;
    if ((++spins & 0x3ff) == 0) {
      if (st->abort || st->error != kOk) {
        if (st->error == kOk) {
          st->error_rank = peer;
          st->error_seq = (uint32_t)expected;
          st->error = kErrAborted;
        }
        return false;
      }
      if (t0 == 0) t0 = globaltimer_ns();
      if (globaltimer_ns() - t0 > budget) {
        st->error_rank = peer;
        st->error_seq = (uint32_t)expected;
        st->error = kErrTimeout;
        __threadfence_system();
        return false;
      }
    }
    __nanosleep(32);
  }
}

__device__ __forceinline__ void red_max_release_sys(uint64_t* p, uint64_t v) {
  asm volatile("red.release.sys.global.max.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

__device__ __forceinline__ bool block_barrier(const PeerTable& pt, int ch, uint64_t flag,
                                              StatusBlock* st, bool release, bool acquire, int mode) {
  __syncthreads();
  const int t = threadIdx.x;
  int ok = 1;
  if (mode <= 1) {
    if (t < pt.world && t != pt.rank) {
      if (mode == 0 && release) __threadfence_system();
      st_release_sys(&pt.pads[t]->sig[ch][blockIdx.x][pt.rank], flag);
      if (mode == 0) {
        ok = wait_flag_acquire(&pt.pads[pt.rank]->sig[ch][blockIdx.x][t], flag, st, t, pt.timeout_ns) ? 1 : 0;
      } else {
        ok = wait_flag(&pt.pads[pt.rank]->sig[ch][blockIdx.x][t], flag, st, t, pt.timeout_ns) ? 1 : 0;
        fence_acq_rel_sys();
      }
    }
    return __syncthreads_and(ok) != 0;
  }
  // The signalling threads t < world all sit in warp 0, so "every signalling thread fences" costs one warp-wide fence
  // instruction -- the same as thread 0 alone -- but gives each flag store / flag poll its own fence IN PROGRAM ORDER,
  // i.e. a well-formed release (fence; st.relaxed) and acquire (ld.relaxed; fence) pattern under the PTX memory model.
  // The CTA's data accesses are ordered around them by the __syncthreads() that opened this function (and the
  // __syncthreads_and() below): bar.sync is morally strong at CTA scope and the fences are cumulative.
  const bool signaller = t < pt.world && t != pt.rank;
  if (t < 32) {
    if (signaller) {
      if (release) fence_acq_rel_sys();
      uint64_t* remote = &pt.pads[t]->sig[ch][blockIdx.x][pt.rank];
      if (mode == 3)
        red_max_release_sys(remote, flag);
      else
        st_relaxed_sys(remote, flag);
      ok = wait_flag(&pt.pads[pt.rank]->sig[ch][blockIdx.x][t], flag, st, t, pt.timeout_ns) ? 1 : 0;
    }
    __syncwarp();  // reconverge the pollers so the acquire fence is ONE warp-wide instruction again
    if (signaller && acquire) fence_acq_rel_sys();
  }
  ok = __syncthreads_and(ok);
  return ok != 0;
}

// ---------------------------------------------------------------------------
// Element packing helpers: 16 B vector <-> fp32 lanes
// ---------------------------------------------------------------------------
template <typename T>
struct Pack;

template <>
struct Pack<float> {
  static constexpr int N = 4;
  __device__ static void unpack(const Vec16& v, float* f) {
    f[0] = __uint_as_float(v.x);
    f[1] = __uint_as_float(v.y);
    f[2] = __uint_as_float(v.z);
    f[3] = __uint_as_float(v.w);
  }
  __device__ static Vec16 pack(const float* f) {
    return Vec16{__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]),
                 __float_as_uint(f[3])};
  }
};

template <>
struct Pack<__nv_bfloat16> {
  static constexpr int N = 8;
  __device__ static void unpack(const Vec16& v, float* f) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      f[2 * i] = __uint_as_float(w[i] << 16);
      f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
  }
  __device__ static Vec16 pack(const float* f) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    return Vec16{w[0], w[1], w[2], w[3]};
  }
};

template <>
struct Pack<__half> {
  static constexpr int N = 8;
  __device__ static void unpack(const Vec16& v, float* f) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __half2 h = *reinterpret_cast<const __half2*>(&w[i]);
      float2 ff = __half22float2(h);
      f[2 * i] = ff.x;
      f[2 * i + 1] = ff.y;
    }
  }
  __device__ static Vec16 pack(const float* f) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __half2 h = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    return Vec16{w[0], w[1], w[2], w[3]};
  }
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide reductions (blockDim.x multiple of 32, <= 1024).
__device__ __forceinline__ float block_sum(float v, float* smem32) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) smem32[warp] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  float r = (threadIdx.x < nw) ? smem32[threadIdx.x] : 0.f;
  if (warp == 0) r = warp_sum(r);
  if (threadIdx.x == 0) smem32[0] = r;
  __syncthreads();
  r = smem32[0];
  __syncthreads();
  return r;
}
__device__ __forceinline__ float block_max(float v, float* smem32) {
  v = warp_max(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) smem32[warp] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  float r = (threadIdx.x < nw) ? smem32[threadIdx.x] : -INFINITY;
  if (warp == 0) r = warp_max(r);
  if (threadIdx.x == 0) smem32[0] = r;
  __syncthreads();
  r = smem32[0];
  __syncthreads();
  return r;
}

#define TFT_CUDA_CHECK(expr)                                                              \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      throw std::runtime_error(std::string("CUDA error ") + cudaGetErrorString(_e) +      \
                               " at " __FILE__ ":" + std::to_string(__LINE__) + " (" #expr \
                               ")");                                                      \
    }                                                                                     \
  } while (0)

}  // namespace tft
