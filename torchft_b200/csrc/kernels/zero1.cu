// FT-ZeRO-1: the partitioned optimizer update fused into the cross-replica collectives (sm_90a).
//
// The reference all-reduces every gradient, divides by N on the host side and then runs the FULL
// optimizer on every replica, gated by a host-synchronous should_commit
// (upstream torchft/manager.py:466-478, upstream torchft/optim.py:52-55). Here the
// replicated dimension also partitions the optimizer:
//
//   backward :  per unit (transformer block), on the comm stream, overlapped with backward:
//                 handshake            "my gradients of this unit are complete" <-> every peer's same message
//                 zero1_reduce_kernel  rank r reduces slice r straight out of every peer's HBM (P2P loads, or ONE
//                                      multimem.ld_reduce per 16 B when the segment is bound to an NVLS multicast
//                                      object), fp32 accumulate in fixed rank order, 1/num_participants scale and
//                                      bf16 cast in registers, and writes the reduced slice to itself AND to its
//                                      k-1 buddies (k-way replicated ownership: a replica that dies never holds
//                                      the only copy of a shard of optimizer state)
//                 handshake            "my pushes have landed / I am done reading yours"
//   commit   :  zero1_commit_kernel    ONE tiny kernel replaces the host sync + RPC: every rank publishes "my step is
//                                      clean" into its peers' signal pads, the verdict is the AND over the quorum,
//                                      written to a device gate word, a device step counter and a host-mapped ring
//                                      the Manager reads lazily at the next start_quorum.
//   update   :  per unit in forward order, on the optimizer stream, gated on the device word:
//                 zero1_update_kernel  AdamW (fp32 master/m/v) on the slices this rank holds, new bf16 weights
//                                      written locally; the PRIMARY holder also stores them into the parameter
//                                      buffer of every replica that does not hold the slice (P2P stores, or ONE
//                                      multimem.st per 16 B) -- the all-gather is the epilogue of the update
//                 handshake            "my weight pushes have landed" (skipped when every rank holds everything)
//
// Gradient clipping (opt-in, CLIP template flag / non-null pointers): the reduce kernel also sums the squares of the
// bf16 values it stores (one fp64 partial per unit and rank, combined over CTAs without float atomics), the commit
// kernel adds every rank's partials in rank order into the global norm and the clip coefficient -- vetoing the step on
// every rank when the norm is not finite -- and the update kernel scales the gradient by that coefficient.
//
// Gradient accumulation (opt-in, ACC template mode / non-null accumulator): every micro-batch but the last reduces its
// slice in fp32 into a per-rank accumulator of the primary slices only (no bf16 rounding, no gradient write, no push);
// the last one adds the accumulator and finishes exactly like a single step (scale, bf16, buddy push, CLIP squares).
//
// Global token mean (opt-in, TM template flag of the commit kernel / non-null slots): every rank publishes its count of
// valid targets, its row count and its loss sum beside the verdict; the commit kernel sums them over the quorum and
// folds P * M * c / N into the coefficient the update kernel already multiplies the gradient by, so the step applies the
// gradient of the mean over every valid target of the quorum. Ranks with different row counts veto the step.
//
// Learning-rate schedule and weight-decay exemptions (opt-in, non-null table / non-zero count, no template flag): the
// update kernel reads the rate of the committed update count gate[1] from a device table, and vectors inside up to
// kMaxNoDecay unit-relative ranges take no decay.
//
// bf16 moments (opt-in, MT template type of the update kernel): m and v are stored as bf16, 8 B of state per parameter
// instead of 12. The arithmetic stays fp32; the moments are rounded stochastically on the way out (bf16_sr) with bits
// that are a pure function of (global element index, gate[1], which moment), so every holder of a slice stores the
// same bits at any grid size, world and paging.
//
// EMA of the weights (opt-in, EMA template flag / non-null ema): the holders of a slice also keep a moving average of
// the new fp32 master weights, of the moments' type (bf16: rounded stochastically with bits of their own), advanced by
// every committed update; mode 2 broadcasts bf16(EMA) of the primary slices into every replica's parameter buffer.
//
// The two big kernels contain NO inter-rank synchronisation at all: any grid size, no co-residency requirement, no
// SM held by a spinning CTA while peers are skewed, profilable stand-alone. Ordering comes from the one-CTA handshake
// kernels around them (bounded, abortable spins; epoch-tagged flags; error latched in the status block and mirrored
// in a device word the big kernels test so a failed handshake turns them into no-ops).
//
// Per rank and step this moves the same NVLink bytes as a two-shot all-reduce but divides the 28 B/param optimizer
// HBM traffic (and the state a replica must hold) by N/k.
#include <algorithm>
#include <stdexcept>
#include <string>

#include "api.h"
#include "common.cuh"
#include "zero1.cuh"

namespace tft {

using zero1::CommitArgs;
using zero1::HsArgs;
using zero1::RSArgs;
using zero1::TokSlot;
using zero1::kVetoRows;
using zero1::UpdArgs;

namespace {

using bf16 = __nv_bfloat16;
using P8 = Pack<bf16>;

__device__ __forceinline__ Vec16 mm_ld_reduce_bf16(const void* p) {
  Vec16 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
__device__ __forceinline__ void mm_st_bf16(void* p, const Vec16& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.bf16x2 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w)
               : "memory");
}

// Slice geometry shared by every kernel here and by parallel/zero1.py (must stay in sync):
// a unit of `nelem` bf16 elements (multiple of 8) = nvec 16-byte vectors, cut into W slices of
// ceil(nvec / W) vectors; slice s belongs to quorum rank s (primary) and ranks s+1..s+k-1 (buddies).
struct Geo {
  size_t nvec, slice;
  __device__ Geo(size_t nelem, int W) : nvec(nelem / 8), slice((nelem / 8 + W - 1) / W) {}
  __device__ size_t lo(int s) const { return min((size_t)s * slice, nvec); }
  __device__ size_t hi(int s) const { return min((size_t)(s + 1) * slice, nvec); }
};

// ---------------------------------------------------------------------------
// Handshake: one CTA, one flag exchange with every peer.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(32, 1) zero1_handshake_kernel(HsArgs a) {
  const bool ok = block_barrier(a.pt, a.channel, a.flag + 1, a.st, a.release != 0, /*acquire=*/true);
  if (threadIdx.x == 0) *a.ok_out = ok ? 1 : 0;
}

// ---------------------------------------------------------------------------
// Reduce-scatter body (no synchronisation).
// ---------------------------------------------------------------------------
// Accumulation mode of the reduce kernel, for a step of M micro-batches:
//   kAccOff  -- M = 1: scale, round to bf16, store to this rank and its k-1 buddies
//   kAccAcc  -- micro-batches 0 .. M-2: the fp32 rank sum goes to the accumulator (micro-batch 0 stores, later ones
//               add); nothing is rounded, written to the gradient segment or pushed
//   kAccLast -- micro-batch M-1: (accumulator + rank sum) * scale, then exactly as kAccOff
enum : int { kAccOff = 0, kAccAcc = 1, kAccLast = 2 };

// 16-byte vectors in flight per thread. A P2P vector holds W x 16 B of loads in registers, the accumulator 32 B more;
// the counts keep every instantiation inside the 128 registers of __launch_bounds__(512, 1) without spilling (W = 7
// keeps three plain vectors in flight, not four).
__host__ __device__ constexpr int reduce_unroll(int W, bool NVLS, int ACC) {
  if (ACC == kAccOff) return NVLS ? 8 : (W >= 8 ? 2 : (W == 7 ? 3 : (W >= 3 ? 4 : 8)));
  if (NVLS) return 6;
  return W <= 1 ? 8 : (W <= 4 ? 4 : (W <= 6 ? 3 : 2));
}

__device__ __forceinline__ float sumsq8(const Vec16& v) {
  float f[8];
  P8::unpack(v, f);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s = fmaf(f[i], f[i], s);
  return s;
}

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The unit's slice sum of squares: per-thread fp32 sums -> fp64 per CTA (fixed warp order) -> the CTA that arrives last
// adds all CTA partials in a fixed order and writes the unit's partial. No float atomics: the bits depend only on the
// data and the grid, never on timing. A bf16 value above ~1.8e19 squares to inf in fp32 and so makes the norm inf, like
// torch's fp32 norm of a bf16 tensor.
__device__ __forceinline__ void finish_unit_sumsq(const RSArgs& a, float sq) {
  __shared__ double warp_sq[32];
  __shared__ int last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const double s = warp_sum_f64((double)sq);
  if (lane == 0) warp_sq[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double b = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) b += warp_sq[w];
    a.cta_sq[blockIdx.x] = b;
    __threadfence();
    last = atomicAdd(a.ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last || warp != 0) return;
  __threadfence();
  double t = 0.0;
  for (unsigned b = lane; b < gridDim.x; b += 32) t += __ldcg(a.cta_sq + b);
  t = warp_sum_f64(t);
  if (lane == 0) {
    *a.gn = t;
    *a.ticket = 0;
  }
}

// What happens to vector v once its fp32 rank sum s is in registers (`av`: the accumulator's two 16-byte halves,
// loaded when `load_acc`). kAccAcc stores acc + s (or s) back to the accumulator; the other modes scale (kAccLast: acc + s
// first), round to bf16 and store to this rank and its buddies.
template <int W, bool CLIP, int ACC>
__device__ __forceinline__ void reduce_epilogue(const RSArgs& a, size_t v, size_t lo, float* s, const Vec16* av,
                                                bool load_acc, bf16* const* dst, int k, float& sq) {
  if constexpr (ACC != kAccOff) {
    if (load_acc) {
      float p[8];
      Pack<float>::unpack(av[0], p);
      Pack<float>::unpack(av[1], p + 4);
#pragma unroll
      for (int i = 0; i < 8; ++i) s[i] = p[i] + s[i];  // ((s_1 + s_2) + ...) + s_m, in micro-batch order
    }
  }
  if constexpr (ACC == kAccAcc) {
    float* o = a.acc + (v - lo) * 8;
    st_stream(o, Pack<float>::pack(s));
    st_stream(o + 4, Pack<float>::pack(s + 4));
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i] *= a.scale;
    const Vec16 out = P8::pack(s);
    if constexpr (CLIP) sq += sumsq8(out);
#pragma unroll
    for (int j = 0; j < W; ++j)
      if (j < k) st_stream(dst[j] + v * 8, out);
  }
}

template <int W, bool NVLS, bool CLIP, int ACC>
__global__ void __launch_bounds__(512, 1) zero1_reduce_kernel(RSArgs a) {
  static_assert(!(CLIP && ACC == kAccAcc), "an accumulating micro-batch produces no bf16 gradient to take the norm of");
  if (*a.ok == 0) return;
  const int rank = a.pt.rank;
  const Geo g(a.nelem, W);
  const bf16* src[W];
  bf16* dst[W];
#pragma unroll
  for (int p = 0; p < W; ++p) {
    src[p] = reinterpret_cast<const bf16*>(reinterpret_cast<const char*>(a.pt.data[p]) + a.off);
    dst[p] = reinterpret_cast<bf16*>(reinterpret_cast<char*>(a.pt.data[(rank + p) % W]) + a.off);
  }
  const char* mcbase = a.mc + a.off;
  const int k = min(a.replication, W);
  const size_t lo = g.lo(rank), hi = g.hi(rank);
  constexpr int U = reduce_unroll(W, NVLS, ACC);
  constexpr int UA = ACC != kAccOff ? U : 1;  // accumulator vectors held in registers
  const bool load_acc = ACC == kAccLast || (ACC == kAccAcc && !a.acc_first);
  const size_t stride = (size_t)gridDim.x * blockDim.x * U;
  float sq = 0.f;  // CLIP: squares of the bf16 values this thread stores
  for (size_t base = lo + (size_t)blockIdx.x * blockDim.x * U; base < hi; base += stride) {
    Vec16 av[UA][2];
    if constexpr (ACC != kAccOff) {
      if (load_acc) {
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const size_t v = base + threadIdx.x + (size_t)u * blockDim.x;
          if (v < hi) {
            av[u][0] = ld_stream(a.acc + (v - lo) * 8);
            av[u][1] = ld_stream(a.acc + (v - lo) * 8 + 4);
          }
        }
      }
    }
    if constexpr (NVLS) {
      Vec16 r[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t v = base + threadIdx.x + (size_t)u * blockDim.x;
        if (v < hi) r[u] = mm_ld_reduce_bf16(mcbase + v * 16);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t v = base + threadIdx.x + (size_t)u * blockDim.x;
        if (v < hi) {
          float f[8];
          P8::unpack(r[u], f);
          reduce_epilogue<W, CLIP, ACC>(a, v, lo, f, av[ACC != kAccOff ? u : 0], load_acc, dst, k, sq);
        }
      }
    } else {
      Vec16 in[U][W];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t v = base + threadIdx.x + (size_t)u * blockDim.x;
        if (v < hi) {
#pragma unroll
          for (int p = 0; p < W; ++p) in[u][p] = ld_stream(src[p] + v * 8);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t v = base + threadIdx.x + (size_t)u * blockDim.x;
        if (v < hi) {
          float acc[8], f[8];
          P8::unpack(in[u][0], acc);
#pragma unroll
          for (int p = 1; p < W; ++p) {
            P8::unpack(in[u][p], f);
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i] += f[i];
          }
          reduce_epilogue<W, CLIP, ACC>(a, v, lo, acc, av[ACC != kAccOff ? u : 0], load_acc, dst, k, sq);
        }
      }
    }
  }
  if constexpr (CLIP) finish_unit_sumsq(a, sq);
}

// ---------------------------------------------------------------------------
// Commit verdict on the device (replaces current-stream synchronize + should_commit RPC for
// replica groups of one rank, upstream torchft/manager.py:884-903).
// ---------------------------------------------------------------------------
// One rank's per-unit partials summed in unit order, 16 loads in flight at a time.
__device__ __forceinline__ double rank_sumsq(const double* p, int n) {
  double s = 0.0;
  for (int u0 = 0; u0 < n; u0 += 16) {
    double x[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) x[i] = (u0 + i < n) ? ld_relaxed_sys_f64(p + u0 + i) : 0.0;
#pragma unroll
    for (int i = 0; i < 16; ++i)
      if (u0 + i < n) s += x[i];
  }
  return s;
}

// Why one buffer of partials is enough: a peer overwrites its partials only in the reduce kernel of its next step, and
// that kernel sits behind the reduce-scatter handshake every rank must reach. This rank reaches its next handshake only
// after this commit kernel (Zero1Optimizer orders the comm stream behind its last commit), so the partials read here
// cannot change under the loads. At W = 1 or without the exchange the same ordering protects this rank's own partials.
//
// Why the token counts need two slots, and why these two are enough (TM). A rank publishes (n, rows, loss) here, in the
// kernel, before any lane stores an arrival flag; a peer reads them after acquiring that flag, in its own commit kernel
// for the same step. The reduce-scatter handshake does not protect them as it protects the partials: they are written
// in the commit, not in the reduce, so without clipping nothing orders a fast rank's next commit behind a slow peer's
// current one. The host therefore alternates the two slots by the parity of the commits since the quorum was
// configured, which is the same on every rank of a quorum (each commit kernel pairs with one of every peer's by flag).
// The slot written for commit c was last read by the peers' kernels for commit c - 2. Each peer's kernel c - 2 finished
// before its kernel c - 1 (same stream) stored the arrival flag that this rank's kernel c - 1 acquired, and this
// kernel follows that one on the commit stream: the reads are done before the write. A kernel c - 1 that did not
// acquire some peer latched an error, and then this kernel writes nothing (and vetoes). At a quorum change every rank
// drains its device before it publishes its mappings, so the old quorum's reads precede the new quorum's writes. The
// inputs n_src and loss_src come from the current stream, which Zero1Optimizer.enqueue orders the commit stream behind.
template <bool TM>
__global__ void __launch_bounds__(32, 1) zero1_commit_kernel(CommitArgs a) {
  const int t = threadIdx.x;
  const int W = a.pt.world, rank = a.pt.rank;
  const int local_ok = (a.host_ok && a.st->error == kOk && !a.st->abort) ? 1 : 0;
  const bool clip = a.gn[rank] != nullptr;
  __shared__ double rank_sq[kMaxRanks];  // a peer whose arrival was not acquired contributes 0 (the verdict is 0 anyway)
  if (clip) {
    if (t < kMaxRanks) rank_sq[t] = (t == rank) ? rank_sumsq(a.gn[rank], a.nunits) : 0.0;
    __syncwarp();
  }
  // TM: every rank's (n, rows, loss); a peer whose arrival was not acquired counts as (0, rows, 0)
  __shared__ unsigned long long rank_n[kMaxRanks], rank_rows[kMaxRanks];
  __shared__ double rank_loss[kMaxRanks];
  // own_*: this rank's real count and loss, which a vetoed step reports; pub_*: what it publishes (0s when it does not
  // contribute, as its gradient counts as 0s)
  unsigned long long own_n = 0, pub_n = 0;
  double own_loss = 0.0, pub_loss = 0.0;
  if constexpr (TM) {
    own_n = (unsigned long long)*a.n_src;
    own_loss = *a.loss_src;
    if (a.contribute) {
      pub_n = own_n;
      pub_loss = own_loss;
    }
    if (t < kMaxRanks) {
      rank_n[t] = t == rank ? pub_n : 0ull;
      rank_rows[t] = (unsigned long long)a.rows;
      rank_loss[t] = t == rank ? pub_loss : 0.0;
    }
    if (t == 0 && a.st->error == kOk) {
      TokSlot* s = a.tm[rank];
      st_relaxed_sys(&s->n, pub_n);
      st_relaxed_sys(&s->rows, (uint64_t)a.rows);
      st_relaxed_sys(&s->loss, (uint64_t)__double_as_longlong(pub_loss));
      __threadfence_system();  // the slot is complete before any lane's arrival flag below
    }
    __syncwarp();
  }
  int ok = local_ok;
  if (a.exchange && W > 1) {
    const uint64_t f = a.flag + 1;
    if (t < W && t != rank) {
      // slot 1 carries the verdict, slot 0 the arrival; a NOT-ok verdict is published too, so
      // clean peers learn immediately instead of waiting out their spin budget
      st_relaxed_sys(&a.pt.pads[t]->sig[a.channel][1][rank], f * 2 + (uint64_t)local_ok);
      fence_acq_rel_sys();
      st_release_sys(&a.pt.pads[t]->sig[a.channel][0][rank], f);
      const uint64_t* arrive = &a.pt.pads[rank]->sig[a.channel][0][t];
      bool got;
      if (a.st->error != kOk) {
        // our own step already failed: do not wait for anybody (their answer cannot change ours)
        got = false;
      } else {
        got = wait_flag(arrive, f, a.st, t, a.pt.timeout_ns);
      }
      if (got) {
        fence_acq_rel_sys();
        const uint64_t v = ld_relaxed_sys(&a.pt.pads[rank]->sig[a.channel][1][t]);
        ok = (v >= f * 2 && (v & 1ull)) ? local_ok : 0;  // stale (older) verdicts compare smaller
        // the peer's reduce kernels (and so its partials) precede its arrival flag: read them over NVLink now
        if (clip) rank_sq[t] = rank_sumsq(a.gn[t], a.nunits);
        if constexpr (TM) {
          // the peer's slot precedes its arrival flag (see above)
          const TokSlot* s = a.tm[t];
          rank_n[t] = ld_relaxed_sys(&s->n);
          rank_rows[t] = ld_relaxed_sys(&s->rows);
          rank_loss[t] = __longlong_as_double((long long)ld_relaxed_sys(&s->loss));
        }
      } else {
        ok = 0;
      }
    }
    ok = __all_sync(0xffffffffu, ok);
  }
  if (clip || TM) __syncwarp();  // rank_sq[] (and the TM arrays) written by the other lanes are visible to lane 0
  if (t == 0) {
    // TM: the quorum's token count and loss sum, in rank order (integers exact, fp64 in a fixed order: the same bits on
    // every rank), and the factor that turns the reduced gradient, divided by pmc, into one divided by N. With no
    // ignored target N = pmc and f is exactly 1.
    unsigned long long N = 0;
    double L = 0.0;
    float f = 1.f;
    uint32_t reason = 0;
    if constexpr (TM) {
      for (int r = 0; r < W; ++r) {
        N += rank_n[r];
        L += rank_loss[r];
        if (rank_rows[r] != (unsigned long long)a.rows) reason = kVetoRows;  // one f cannot serve different shapes
      }
      f = (float)((double)a.pmc / (double)(N > 0 ? N : 1ull));
      if (reason) ok = 0;
    }
    if (clip) {
      // ranks in rank order 0..W-1 in fp64: every rank of the quorum adds the same numbers in the same order, so norm
      // and coefficient are bit-identical everywhere. coef = min(1, max_norm / (norm + 1e-6)) with torch's clip_grad_norm_
      // rounding: torch evaluates float / tensor as reciprocal(tensor) * float, each step IEEE fp32 (max_norm = inf
      // gives exactly 1). TM: the norm of the gradient the update applies is norm * f.
      double sq = 0.0;
      for (int r = 0; r < W; ++r) sq += rank_sq[r];
      float norm = (float)sqrt(sq);
      if constexpr (TM) norm = __fmul_rn(norm, f);
      const float coef = fminf(1.f, __fmul_rn(__frcp_rn(__fadd_rn(norm, 1e-6f)), a.max_norm));
      if ((__float_as_uint(norm) & 0x7f800000u) == 0x7f800000u) ok = 0;  // inf / nan: vetoed on every rank alike
      a.norm[0] = norm;
      a.norm[1] = TM ? __fmul_rn(f, coef) : coef;
      a.st->gnorm[a.seq & (kVerdictRing - 1)] = norm;
      __threadfence_system();  // the norm slot is complete before the host can see this seq's verdict
    } else if (TM) {
      a.norm[1] = f;
    }
    if constexpr (TM) {
      // a vetoed step reports this rank's own token mean (a non-contributing rank's too, though it published 0s): the
      // quorum's sums may be missing a peer
      const unsigned long long n = ok ? N : own_n;
      a.tm_out[0] = (float)((ok ? L : own_loss) / (double)(n > 0 ? n : 1ull));
      a.tm_out[1] = f;
      a.tm_count[0] = (long long)N;
      a.st->reason[a.seq & (kVerdictRing - 1)] = reason;
      __threadfence_system();  // the reason slot is complete before the host can see this seq's verdict
    }
    a.gate[0] = ok;
    if (ok) a.gate[1] += 1;
    a.st->verdict[a.seq & (kVerdictRing - 1)] = (a.seq << 1) | (uint32_t)ok;
    __threadfence_system();
  }
}

// ---------------------------------------------------------------------------
// Stochastic rounding of the bf16 moments. parallel/zero1.py (sr_bits, bf16_sr) is the specification; the two must
// return the same bits.
// ---------------------------------------------------------------------------
// The 32 random bits of element e at update t: murmur3's 32-bit finaliser over a linear mix of the index halves, the
// update count and a fixed seed. The low half rounds m, the high half rounds v.
__device__ __forceinline__ uint32_t sr_bits(uint64_t e, uint32_t t) {
  uint32_t x = (uint32_t)e * 0x9E3779B1u + (uint32_t)(e >> 32) * 0x85EBCA77u + t * 0xC2B2AE3Du + 0x27D4EB2Fu;
  x ^= x >> 16;
  x *= 0x85EBCA6Bu;
  x ^= x >> 13;
  x *= 0xC2B2AE35u;
  x ^= x >> 16;
  return x;
}

// The bits of a bf16 EMA (low half): the same mix and finaliser with another seed, so element e's EMA is not rounded
// with the bits that round its moments. parallel/zero1.py (sr_bits_ema) is the specification.
__device__ __forceinline__ uint32_t sr_bits_ema(uint64_t e, uint32_t t) {
  uint32_t x = (uint32_t)e * 0x9E3779B1u + (uint32_t)(e >> 32) * 0x85EBCA77u + t * 0xC2B2AE3Du + 0x165667B1u;
  x ^= x >> 16;
  x *= 0x85EBCA6Bu;
  x ^= x >> 13;
  x *= 0xC2B2AE35u;
  x ^= x >> 16;
  return x;
}

// fp32 -> bf16 bits: add the 16-bit r to the fp32 bits and keep the upper half. The add is on the magnitude, so it
// rounds away from zero with probability (discarded fraction), which is unbiased for both signs; a value bf16
// represents exactly comes back unchanged for every r. Inf and NaN are not added to; a NaN keeps a mantissa bit.
__device__ __forceinline__ uint32_t bf16_sr(float x, uint32_t r) {
  const uint32_t u = __float_as_uint(x);
  if ((u & 0x7f800000u) == 0x7f800000u) return (u >> 16) | ((u & 0x007fffffu) ? 0x0040u : 0u);
  return (u + r) >> 16;
}

// ---------------------------------------------------------------------------
// Gated AdamW on the held slices + all-gather of the new bf16 weights (no synchronisation).
// ---------------------------------------------------------------------------
template <int W, bool NVLS, bool PAGED, bool CLIP, typename MT, bool EMA>
__global__ void __launch_bounds__(512, 2) zero1_update_kernel(UpdArgs a) {
  constexpr bool BF16M = sizeof(MT) == 2;
  MT* const mp = reinterpret_cast<MT*>(a.m);
  MT* const vp = reinterpret_cast<MT*>(a.v);
  MT* const ep = reinterpret_cast<MT*>(a.ema);  // EMA: the moving average, of the moments' type
  if (a.mode == 0 && a.gate[0] == 0) return;  // uniform over the grid AND (unanimous verdict) over the quorum
  const int rank = a.pt.rank;
  const Geo g(a.nelem, W);
  const int k = min(a.replication, W);
  float cf = 1.f;
  if constexpr (CLIP) {
    if (a.mode == 0) cf = __ldg(a.coef);
  }
  const int t = a.gate[1];
  // the rate follows the committed update count on the device, like the bias correction: one uniform load
  // (a refresh may run at t = 0 and does not use it)
  const float lr = a.lr_tab != nullptr ? __ldg(a.lr_tab + (min(max(t, 1), a.lr_steps) - 1)) : a.lr;
  // 1 - b^t in fp64 from the fp32 betas the moving averages use, rounded once. --use_fast_math turns powf into
  // __log2f/exp2f, whose absolute error in log2(b) becomes a relative error of up to ~1e-4 in 1 - b^t at b = 0.999; the
  // fp64 pow is not approximated and leaves the fp32 result correctly rounded but for near-ties.
  const float bc1 = (float)(1.0 - pow((double)a.b1, (double)t)), bc2 = (float)(1.0 - pow((double)a.b2, (double)t));
  const float step_size = lr / bc1;
  const float inv_bc2_sqrt = rsqrtf(bc2);
  const float decay = 1.f - lr * a.wd;
  // dst[0] = this rank; dst[j] = rank + j. Ranks rank+1 .. rank+k-1 hold the primary slice too and compute the same
  // bits themselves, so the primary only pushes to dst[k .. W-1] (mode 0). A refresh pushes to everybody.
  bf16* dst[W];
#pragma unroll
  for (int p = 0; p < W; ++p)
    dst[p] = reinterpret_cast<bf16*>(reinterpret_cast<char*>(a.pt.data[(rank + p) % W]) + a.poff);
  char* mcbase = a.mc + a.poff;
  const int first_push = a.mode == 0 ? k : 1;
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nthreads = (size_t)gridDim.x * blockDim.x;

  for (int j = 0; j < (a.mode == 0 ? k : 1); ++j) {
    const int s = (rank - j + W) % W;  // j = 0: primary slice, j > 0: slices this rank backs up
    const size_t lo = g.lo(s), hi = g.hi(s);
    // paged: the slot of the NEXT iteration's page is loaded one iteration ahead, so the state loads never wait for a
    // dependent table load (a grid-stride step is larger than a page: every iteration is a different page)
    const size_t pmask = (size_t(1) << a.page_shift) - 1;
    int slot = 0;
    if constexpr (PAGED) {
      if (lo + tid < hi) slot = __ldg(a.table + ((a.soff + (lo + tid) * 8) >> a.page_shift));
    }
    for (size_t v = lo + tid; v < hi; v += nthreads) {
      size_t si = v * 8;  // index of the 8-element group in the state arrays
      if constexpr (PAGED) {
        si = ((size_t)slot << a.page_shift) | ((a.soff + v * 8) & pmask);
        if (v + nthreads < hi) slot = __ldg(a.table + ((a.soff + (v + nthreads) * 8) >> a.page_shift));
      }
      float w[8];
      Vec16 w0, w1;
      if (!EMA || a.mode != 2) {  // mode 2 reads the EMA instead
        w0 = ld_stream(a.master + si);
        w1 = ld_stream(a.master + si + 4);
      }
      if (a.mode == 0) {
        // all 7 x 16 B loads (5 with bf16 moments; EMA: 2 more, 1 in bf16) in flight before any use
        const Vec16 gv = ld_stream(a.grad + v * 8);
        Vec16 m0, m1, v0, v1, e0, e1;
        if constexpr (BF16M) {
          m0 = ld_stream(mp + si);
          v0 = ld_stream(vp + si);
        } else {
          m0 = ld_stream(mp + si);
          m1 = ld_stream(mp + si + 4);
          v0 = ld_stream(vp + si);
          v1 = ld_stream(vp + si + 4);
        }
        if constexpr (EMA) {
          e0 = ld_stream(ep + si);
          if constexpr (!BF16M) e1 = ld_stream(ep + si + 4);
        }
        float gr[8], m[8], vv[8];
        P8::unpack(gv, gr);
        if constexpr (CLIP) {
#pragma unroll
          for (int i = 0; i < 8; ++i) gr[i] *= cf;
        }
        Pack<float>::unpack(w0, w);
        Pack<float>::unpack(w1, w + 4);
        if constexpr (BF16M) {
          P8::unpack(m0, m);
          P8::unpack(v0, vv);
        } else {
          Pack<float>::unpack(m0, m);
          Pack<float>::unpack(m1, m + 4);
          Pack<float>::unpack(v0, vv);
          Pack<float>::unpack(v1, vv + 4);
        }
        float dcy = decay;
        if (a.n_nd > 0) {  // uniform: without exemptions no vector pays for the compares
#pragma unroll
          for (int r = 0; r < kMaxNoDecay; ++r)
            if (r < a.n_nd && v >= a.nd_lo[r] && v < a.nd_hi[r]) dcy = 1.f;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          m[i] = a.b1 * m[i] + (1.f - a.b1) * gr[i];
          // spelled out as the flat AdamW kernel (model_ops.cu) compiles it, so both store the same bits: left to
          // itself the compiler fuses b2 * v here and g * ((1 - b2) * g) there
          vv[i] = __fmaf_rn(gr[i], __fmul_rn(1.f - a.b2, gr[i]), __fmul_rn(a.b2, vv[i]));
          const float denom = sqrtf(vv[i]) * inv_bc2_sqrt + a.eps;
          w[i] = w[i] * dcy - step_size * __fdividef(m[i], denom);
        }
        st_stream(a.master + si, Pack<float>::pack(w));
        st_stream(a.master + si + 4, Pack<float>::pack(w + 4));
        if constexpr (BF16M) {
          // the weights above used the fp32 moments; what is stored is their stochastic rounding
          const uint64_t e0 = a.soff + v * 8;
          uint32_t mo[4], vo[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const uint32_t r0 = sr_bits(e0 + 2 * i, (uint32_t)t), r1 = sr_bits(e0 + 2 * i + 1, (uint32_t)t);
            mo[i] = bf16_sr(m[2 * i], r0 & 0xffffu) | (bf16_sr(m[2 * i + 1], r1 & 0xffffu) << 16);
            vo[i] = bf16_sr(vv[2 * i], r0 >> 16) | (bf16_sr(vv[2 * i + 1], r1 >> 16) << 16);
          }
          st_stream(mp + si, Vec16{mo[0], mo[1], mo[2], mo[3]});
          st_stream(vp + si, Vec16{vo[0], vo[1], vo[2], vo[3]});
        } else {
          st_stream(mp + si, Pack<float>::pack(m));
          st_stream(mp + si + 4, Pack<float>::pack(m + 4));
          st_stream(vp + si, Pack<float>::pack(vv));
          st_stream(vp + si + 4, Pack<float>::pack(vv + 4));
        }
        if constexpr (EMA) {
          // ema + c * (w' - ema), each operation rounded on its own (no FMA): what numpy float32 computes
          float e[8];
          if constexpr (BF16M) {
            P8::unpack(e0, e);
          } else {
            Pack<float>::unpack(e0, e);
            Pack<float>::unpack(e1, e + 4);
          }
#pragma unroll
          for (int i = 0; i < 8; ++i) e[i] = __fadd_rn(e[i], __fmul_rn(a.ema_c, __fsub_rn(w[i], e[i])));
          if constexpr (BF16M) {
            const uint64_t x0 = a.soff + v * 8;
            uint32_t eo[4];
#pragma unroll
            for (int i = 0; i < 4; ++i)
              eo[i] = bf16_sr(e[2 * i], sr_bits_ema(x0 + 2 * i, (uint32_t)t) & 0xffffu) |
                      (bf16_sr(e[2 * i + 1], sr_bits_ema(x0 + 2 * i + 1, (uint32_t)t) & 0xffffu) << 16);
            st_stream(ep + si, Vec16{eo[0], eo[1], eo[2], eo[3]});
          } else {
            st_stream(ep + si, Pack<float>::pack(e));
            st_stream(ep + si + 4, Pack<float>::pack(e + 4));
          }
        }
      } else if (EMA && a.mode == 2) {
        // fp32 EMA: rounded to nearest by the pack below; a bf16 EMA comes back with its own bits
        if constexpr (BF16M) {
          P8::unpack(ld_stream(ep + si), w);
        } else {
          Pack<float>::unpack(ld_stream(ep + si), w);
          Pack<float>::unpack(ld_stream(ep + si + 4), w + 4);
        }
      } else {
        Pack<float>::unpack(w0, w);
        Pack<float>::unpack(w1, w + 4);
      }
      const Vec16 out = P8::pack(w);
      st_stream(dst[0] + v * 8, out);  // every holder refreshes its own copy of the weights
      if (j == 0) {
        if constexpr (NVLS) {
          if (first_push < W) mm_st_bf16(mcbase + v * 16, out);  // the switch replicates (holders get identical bits again)
        } else {
#pragma unroll
          for (int p = 1; p < W; ++p)
            if (p >= first_push) st_stream(dst[p] + v * 8, out);
        }
      }
    }
  }
}

void check_grid(int blocks, int threads, const char* who) {
  if (blocks < 1 || blocks > kZero1MaxBlocks) throw std::runtime_error(std::string(who) + ": bad grid");
  if (threads < 32 || threads > 512 || (threads & 31)) throw std::runtime_error(std::string(who) + ": bad block size");
}

}  // namespace

void zero1_handshake_launch(const HsArgs& a, cudaStream_t stream) {
  zero1_handshake_kernel<<<1, 32, 0, stream>>>(a);
  TFT_CUDA_CHECK(cudaGetLastError());
}

void zero1_reduce_launch(RSArgs a, int acc_mode, int blocks, int threads, cudaStream_t stream) {
  check_grid(blocks, threads, "zero1_reduce");
  if ((a.off & 15) || (a.nelem & 7)) throw std::runtime_error("zero1_reduce: unit must be 16 B aligned and a multiple of 8 elements");
  if (a.replication < 1) throw std::runtime_error("zero1_reduce: replication must be >= 1");
  if (a.gn != nullptr && (a.cta_sq == nullptr || a.ticket == nullptr))
    throw std::runtime_error("zero1_reduce: the gradient norm needs the per-CTA scratch and the ticket");
  if (acc_mode < 0 || acc_mode > 3) throw std::runtime_error("zero1_reduce: acc_mode must be 0 (off), 1 (first), 2 (middle) or 3 (last)");
  if (acc_mode != 0 && (a.acc == nullptr || (reinterpret_cast<uintptr_t>(a.acc) & 15)))
    throw std::runtime_error("zero1_reduce: accumulation needs a 16 B aligned fp32 accumulator");
  if ((acc_mode == 1 || acc_mode == 2) && a.gn != nullptr)
    throw std::runtime_error("zero1_reduce: the gradient norm is taken on the last micro-batch only");
  if (acc_mode == 0) a.acc = nullptr;
  a.acc_first = acc_mode == 1 ? 1 : 0;
  const int acc = acc_mode == 0 ? kAccOff : (acc_mode == 3 ? kAccLast : kAccAcc);
  const char* bad_world = "zero1_reduce: world size must be in [2, 8]";
  const bool known_world = dispatch<1, 2, 3, 4, 5, 6, 7, 8>(a.pt.world, [&](auto W) {
    dispatch<false, true>(a.mc != nullptr, [&](auto NVLS) {
      dispatch<false, true>(a.gn != nullptr, [&](auto CLIP) {
        dispatch<kAccOff, kAccAcc, kAccLast>(acc, [&](auto ACC) {
          // one rank: only clipping and accumulation launch it (in place, no peer access); never multicast. CLIP with
          // kAccAcc was rejected above.
          if constexpr ((W > 1 || ((CLIP || ACC != kAccOff) && !NVLS)) && !(CLIP && ACC == kAccAcc))
            zero1_reduce_kernel<W, NVLS, CLIP, ACC><<<blocks, threads, 0, stream>>>(a);
          else
            throw std::runtime_error(bad_world);
        });
      });
    });
  });
  if (!known_world) throw std::runtime_error(bad_world);
  TFT_CUDA_CHECK(cudaGetLastError());
}

void zero1_commit_launch(const CommitArgs& a, cudaStream_t stream) {
  if (std::any_of(a.gn, a.gn + a.pt.world, [](const double* p) { return p != nullptr; })) {
    if (a.norm == nullptr || a.nunits < 1) throw std::runtime_error("zero1_commit: the gradient norm needs units and an output pair");
    if (!(a.max_norm > 0.f)) throw std::runtime_error("zero1_commit: max_norm must be > 0");
    if (std::count(a.gn, a.gn + a.pt.world, nullptr) != 0) throw std::runtime_error("zero1_commit: one z1_gnorm pointer per rank");
  }
  const bool tm = std::any_of(a.tm, a.tm + a.pt.world, [](const TokSlot* p) { return p != nullptr; });
  if (tm) {
    if (std::count(a.tm, a.tm + a.pt.world, nullptr) != 0) throw std::runtime_error("zero1_commit: one z1_tokmean slot per rank");
    if (a.n_src == nullptr || a.loss_src == nullptr || a.tm_out == nullptr || a.tm_count == nullptr || a.norm == nullptr)
      throw std::runtime_error("zero1_commit: the token mean needs its two inputs and three outputs");
    if (a.rows < 1 || a.pmc < 1) throw std::runtime_error("zero1_commit: the token mean needs rows >= 1 and P * M * c >= 1");
  }
  dispatch<false, true>(tm, [&](auto TM) { zero1_commit_kernel<TM><<<1, 32, 0, stream>>>(a); });
  TFT_CUDA_CHECK(cudaGetLastError());
}

void zero1_update_launch(UpdArgs a, int moment_dtype, int blocks, int threads, cudaStream_t stream) {
  check_grid(blocks, threads, "zero1_update");
  if (moment_dtype != kF32 && moment_dtype != kBF16) throw std::runtime_error("zero1_update: moments are fp32 or bf16");
  if (((reinterpret_cast<uintptr_t>(a.m) | reinterpret_cast<uintptr_t>(a.v)) & 15) || (moment_dtype == kBF16 && (a.soff & 7)))
    throw std::runtime_error("zero1_update: m and v must be 16 B aligned (bf16 moments: and the unit's first element a multiple of 8)");
  if ((a.poff & 15) || (a.nelem & 7)) throw std::runtime_error("zero1_update: unit must be 16 B aligned and a multiple of 8 elements");
  if (a.table != nullptr && (a.page_shift < 3 || a.page_shift > 30 || (a.soff & 7)))
    throw std::runtime_error("zero1_update: pages must be 2^3 .. 2^30 elements and the unit 8-element aligned");
  if (a.lr_tab != nullptr && (a.lr_steps < 1 || (reinterpret_cast<uintptr_t>(a.lr_tab) & 3)))
    throw std::runtime_error("zero1_update: a learning-rate table needs lr_steps >= 1 and 4 B alignment");
  if (a.lr_tab == nullptr) a.lr_steps = 0;
  if (a.mode < 0 || a.mode > 2) throw std::runtime_error("zero1_update: mode is 0 (update), 1 (refresh) or 2 (EMA broadcast)");
  if (a.mode == 2 && a.ema == nullptr) throw std::runtime_error("zero1_update: mode 2 broadcasts the EMA and needs one");
  if (a.ema != nullptr && ((reinterpret_cast<uintptr_t>(a.ema) & 15) || !(a.ema_c > 0.f && a.ema_c < 1.f)))
    throw std::runtime_error("zero1_update: the EMA must be 16 B aligned and its coefficient 1 - decay in (0, 1)");
  if (a.n_nd < 0 || a.n_nd > kMaxNoDecay)
    throw std::runtime_error("zero1_update: at most " + std::to_string(kMaxNoDecay) + " weight-decay exemptions per unit");
  for (int r = 0; r < a.n_nd; ++r) {
    const size_t lo = a.nd_lo[r], hi = a.nd_hi[r];
    if ((lo & 7) || (hi & 7) || lo >= hi || hi > a.nelem)
      throw std::runtime_error("zero1_update: weight-decay exemptions must be non-empty 8-element aligned ranges inside the unit");
    a.nd_lo[r] = lo / 8;
    a.nd_hi[r] = hi / 8;
  }
  const bool known_world = dispatch<1, 2, 3, 4, 5, 6, 7, 8>(a.pt.world, [&](auto W) {
    dispatch<false, true>(a.mc != nullptr, [&](auto NVLS) {
      dispatch<false, true>(a.table != nullptr, [&](auto PAGED) {
        dispatch<false, true>(a.coef != nullptr, [&](auto CLIP) {
          dispatch<kF32, kBF16>(moment_dtype, [&](auto MD) {
            dispatch<false, true>(a.ema != nullptr, [&](auto EMA) {
              // one rank pushes to nobody: never multicast
              zero1_update_kernel<W, (W > 1 && NVLS), PAGED, CLIP, Elem<MD>, EMA><<<blocks, threads, 0, stream>>>(a);
            });
          });
        });
      });
    });
  });
  if (!known_world) throw std::runtime_error("zero1_update: world size must be in [1, 8]");
  TFT_CUDA_CHECK(cudaGetLastError());
}

}  // namespace tft
