// FT-ZeRO-1 replica audit (sm_90a): digests of every replica's bf16 weights and every holder's optimizer state, and a
// one-CTA comparison of the quorum's digests that latches kErrDiverged when replicas or holders disagree.
//
// The digest of a range is the sum mod 2^64 of fmix64(w ^ (i * 0x9E3779B97F4A7C15 + seed)) over its 8-byte words w at
// global word index i. parallel/zero1.py (z1_digest) is the specification; the kernel returns the same bits at any grid,
// in any order, flat or paged.
//
// Own file so that the cubin of zero1.cu stays as it is.
#include <stdexcept>
#include <string>

#include "api.h"
#include "audit.cuh"
#include "common.cuh"

namespace tft {

using audit::CompareArgs;
using audit::DigestEntry;
using audit::kDigestChunkWords;
using audit::kReportHeader;

namespace {

constexpr uint64_t kGolden = 0x9E3779B97F4A7C15ull;
constexpr int kDigestUnroll = 4;  // 16-byte loads in flight per thread

__device__ __forceinline__ uint64_t fmix64(uint64_t k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ull;
  k ^= k >> 33;
  return k;
}

__device__ __forceinline__ uint64_t word_digest(uint64_t w, uint64_t i, uint64_t seed) {
  return fmix64(w ^ (i * kGolden + seed));
}

// Address of global byte g of an entry's array (g is 8-byte aligned; a 16-byte aligned g stays 16-byte aligned).
__device__ __forceinline__ const char* entry_addr(const DigestEntry& e, uint64_t g) {
  if (e.table == nullptr) return e.base + g;
  const uint64_t pmask = (uint64_t(1) << e.page_byte_shift) - 1;
  return e.base + (((uint64_t)__ldg(e.table + (g >> e.page_byte_shift)) << e.page_byte_shift) | (g & pmask));
}

__device__ __forceinline__ uint64_t warp_sum_u64(uint64_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// 3 CTAs of 512 threads per SM (<= 42 registers): the launcher's grid of 3 x SMs runs in one wave.
__global__ void __launch_bounds__(512, 3) z1_digest_kernel(const DigestEntry* __restrict__ tab, int nentries,
                                                        size_t total_chunks, unsigned long long* slots) {
  for (size_t c = blockIdx.x; c < total_chunks; c += gridDim.x) {
    int lo = 0, hi = nentries - 1;  // the last row whose chunk0 is not above c
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (tab[mid].chunk0 <= c) lo = mid; else hi = mid - 1;
    }
    const DigestEntry e = tab[lo];
    const uint64_t w0 = (c - e.chunk0) * kDigestChunkWords;  // even: a chunk starts on a vector
    const uint64_t w1 = min(w0 + (uint64_t)kDigestChunkWords, e.nwords);
    const uint64_t first = e.word0 + w0;  // global index of the chunk's first word
    const uint64_t nv = (w1 - w0) / 2;
    uint64_t s = 0;
    for (uint64_t v = threadIdx.x; v < nv; v += (uint64_t)blockDim.x * kDigestUnroll) {
      Vec16 r[kDigestUnroll];
#pragma unroll
      for (int u = 0; u < kDigestUnroll; ++u) {
        const uint64_t x = v + (uint64_t)u * blockDim.x;
        if (x < nv) r[u] = ld_stream(entry_addr(e, (first + 2 * x) * 8));
      }
#pragma unroll
      for (int u = 0; u < kDigestUnroll; ++u) {
        const uint64_t x = v + (uint64_t)u * blockDim.x;
        if (x < nv) {
          const uint64_t i = first + 2 * x;
          s += word_digest(((uint64_t)r[u].y << 32) | r[u].x, i, e.seed);
          s += word_digest(((uint64_t)r[u].w << 32) | r[u].z, i + 1, e.seed);
        }
      }
    }
    if (((w1 - w0) & 1) && threadIdx.x == 0) {  // an odd word at the end of the entry
      const uint64_t i = first + 2 * nv;
      s += word_digest(*reinterpret_cast<const uint64_t*>(entry_addr(e, i * 8)), i, e.seed);
    }
    s = warp_sum_u64(s);
    if ((threadIdx.x & 31) == 0 && s != 0) atomicAdd(slots + e.slot, (unsigned long long)s);
  }
}

// Behind a handshake, so every rank's digests are complete. Warp w copies the slots of ranks w, w + 8, ... into the
// report; then every thread compares a share of the groups that must agree, reading the slots again over NVLink (the
// report is host memory). Every rank reads the same bytes and so reaches the same decision.
__global__ void __launch_bounds__(256, 1) z1_audit_compare_kernel(CompareArgs a) {
  if (*a.ok == 0) return;  // the handshake failed: a peer's digests may be missing; the report keeps the last audit
  const int W = a.pt.world;
  const int n = a.nunits * a.stride + 1;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  __shared__ uint64_t t[kMaxRanks];
  __shared__ unsigned mismatches, low;
  auto slot = [&](int r, int i) { return ld_relaxed_sys(reinterpret_cast<const uint64_t*>(a.pt.data[r]) + i); };
  if (threadIdx.x == 0) {
    mismatches = 0;
    low = kMaxRanks;
  }
  for (int r = warp; r < W; r += nwarps) {
    unsigned long long* out = a.report + kReportHeader + (size_t)r * n;
    for (int i = lane; i < n; i += 32) {
      const uint64_t x = slot(r, i);
      out[i] = x;
      if (i == n - 1) t[r] = x;
    }
  }
  __syncthreads();
  uint64_t tmax = 0;
  for (int r = 0; r < W; ++r) tmax = max(tmax, t[r]);
  // ranks behind the quorum's update count (a split commit left them there) are not compared
  const int k = min(a.k, W);
  const int per_unit = 1 + (k > 1 ? W * a.narrays : 0);  // the weights, then (slice, array) of the state
  for (int g = threadIdx.x; g < a.nunits * per_unit; g += blockDim.x) {
    const int u = g / per_unit, q = g % per_unit;
    bool seen = false, differ = false;
    uint64_t ref = 0;
    int first = kMaxRanks;
    if (q == 0) {
      for (int r = 0; r < W; ++r) {
        if (t[r] != tmax) continue;
        const uint64_t d = slot(r, u * a.stride);
        if (!seen) ref = d, first = r, seen = true;
        else differ |= d != ref;
      }
    } else {
      const int s = (q - 1) / a.narrays, arr = (q - 1) % a.narrays;
      for (int j = 0; j < k; ++j) {
        const int h = (s + j) % W;  // holds slice s as its j-th held slice
        if (t[h] != tmax) continue;
        const uint64_t d = slot(h, u * a.stride + 1 + j * a.narrays + arr);
        if (!seen) ref = d, seen = true;
        else differ |= d != ref;
        first = min(first, h);
      }
    }
    if (differ) {
      atomicAdd(&mismatches, 1u);
      atomicMin(&low, (unsigned)first);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    a.report[1] = mismatches;
    a.report[2] = W;
    a.report[3] = n;
    __threadfence_system();
    a.report[0] = a.seq;  // last: a report with this seq is complete
    if (mismatches != 0 && a.st->error == kOk) {
      a.st->error_rank = low;
      a.st->error_seq = (uint32_t)a.seq;
      a.st->error = kErrDiverged;
    }
    __threadfence_system();
  }
}

}  // namespace

void z1_digest_launch(const void* table_dev, int nentries, size_t total_chunks, unsigned long long* slots, int blocks,
                      cudaStream_t stream) {
  if (nentries < 1 || total_chunks < 1) return;
  if (blocks < 1 || (reinterpret_cast<uintptr_t>(table_dev) & 7) || slots == nullptr)
    throw std::runtime_error("z1_digest: needs a grid, an 8 B aligned table and the slots");
  z1_digest_kernel<<<blocks, 512, 0, stream>>>(reinterpret_cast<const DigestEntry*>(table_dev), nentries, total_chunks,
                                               slots);
  TFT_CUDA_CHECK(cudaGetLastError());
}

void z1_audit_compare_launch(const CompareArgs& a, cudaStream_t stream) {
  if (a.report == nullptr || a.ok == nullptr || a.nunits < 1 || a.narrays < 1 || a.k < 1 ||
      a.stride < 1 + a.k * a.narrays)
    throw std::runtime_error("z1_audit_compare: needs a report, the handshake word and a slot layout that fits");
  z1_audit_compare_kernel<<<1, 256, 0, stream>>>(a);
  TFT_CUDA_CHECK(cudaGetLastError());
}

}  // namespace tft
