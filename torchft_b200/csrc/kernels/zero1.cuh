// Arguments of the FT-ZeRO-1 kernels (zero1.cu). Each struct is its kernel's one parameter, passed by value, so the
// field order and types are the kernel's parameter layout. bindings.cu fills them by field name; the zero1_*_launch
// functions (api.h) check them, derive the fields noted below, pick the template instance and launch it.
#pragma once
#include "common.cuh"

namespace tft {

constexpr int kMaxNoDecay = 4;  // weight-decay exemption ranges per unit
// Grid cap of the reduce and update kernels. The reduce kernel's gradient norm takes one fp64 partial per CTA, so the
// host sizes that scratch from this cap (exported as ZERO1_MAX_BLOCKS).
constexpr int kZero1MaxBlocks = kNumSMs * 32;

namespace zero1 {

// Handshake: one CTA, one flag exchange with every peer.
struct HsArgs {
  PeerTable pt;
  StatusBlock* st;
  int* ok_out;       // device word receiving 1/0, so the sync-free kernels behind it on the stream can turn into no-ops
  uint64_t flag;     // consumes flag+1
  int channel;
  int release;       // this rank wrote peer-visible data in an earlier kernel of this stream: fence before the flag store
};

// Reduce-scatter of one unit in place: rank r reduces slice r and stores it to itself and its k-1 buddies.
struct RSArgs {
  PeerTable pt;       // data[] = every rank's gradient segment
  const int* ok;      // result of the handshake in front of this kernel
  char* mc;           // multicast VA of the gradient segment (nullptr = P2P loads; never at world 1)
  size_t off;         // byte offset of the unit inside the segment (16 B aligned)
  size_t nelem;       // elements in the unit (multiple of 8)
  float scale;
  int replication;    // k
  // gradient clipping (gn != nullptr): gn receives the fp64 sum of squares of the bf16 values of this rank's slice (its
  // slot of the unit in its z1_gnorm segment); cta_sq is scratch of one fp64 per CTA and ticket the last-CTA-done
  // counter (zero between launches: the last CTA resets it). At world 1 the kernel only scales the unit in place.
  double* gn;
  double* cta_sq;
  unsigned* ticket;
  // gradient accumulation, by the launcher's acc_mode: 0 off, 1 first micro-batch (store the fp32 rank sum of the slice
  // in acc), 2 middle (add it), 3 last ((acc + rank sum) * scale to bf16 like 0, with the norm when gn is set). Modes 1
  // and 2 leave the gradient segment untouched and push nothing. acc: this rank's 16 B aligned fp32 accumulator of the
  // unit's primary slice; vector v of the slice lives at acc + (v - lo(rank)) * 8. The launcher sets acc to nullptr in
  // mode 0, and acc_first (uniform per launch: store the sum instead of adding it) from the mode.
  float* acc;
  int acc_first;
};

// Global token mean: what one rank publishes for one commit in its z1_tokmean segment, which holds two of these (the
// commit kernel's comment says why two). Words, so that peers read them with one relaxed 64-bit load each.
struct TokSlot {
  uint64_t n;      // valid targets of this rank's step (0 on a rank that does not contribute)
  uint64_t rows;   // M * B * S of this rank's step
  uint64_t loss;   // bits of the fp64 sum of its per-target losses
  uint64_t pad;
};

// Why the commit kernel vetoed a step, posted beside the verdict (StatusBlock::reason).
constexpr uint32_t kVetoRows = 1;  // the ranks published different row counts M * B * S

// Commit verdict on the device: this rank's verdict, ANDed over the quorum through the signal pads.
struct CommitArgs {
  PeerTable pt;        // pads only
  StatusBlock* st;
  int* gate;           // device: gate[0] = verdict of this step, gate[1] = optimizer step count t
  uint64_t flag;       // consumes flag+1
  uint32_t seq;        // commit sequence number (slot in the host ring)
  int channel;
  int host_ok;         // host-side part of the verdict (enough participants, no host-latched error)
  int exchange;        // 1 = AND the verdict over the quorum through the signal pads
  // gradient clipping (a pointer for every rank, or none): gn[r] is rank r's z1_gnorm segment of nunits fp64 partials.
  // The kernel adds them in rank order, writes norm[0] = global L2 norm and norm[1] = min(1, max_norm / (norm + 1e-6)),
  // posts the norm to the host ring and vetoes a non-finite norm.
  const double* gn[kMaxRanks];
  int nunits;
  float max_norm;
  float* norm;
  // global token mean (a slot for every rank, or none; needs norm): tm[r] is rank r's TokSlot for this commit. The
  // kernel publishes (n_src, rows, loss_src) in tm[rank] (n and loss 0 when !contribute), sums every rank's (n, loss)
  // in rank order into N and L, vetoes the step when some rank's rows differ from this rank's, and writes
  // f = fp32(pmc / max(N, 1)), tm_count[0] = N and tm_out = {L / max(N, 1) (vetoed: this rank's own mean), f}. The
  // coefficient norm[1] becomes f (with clipping: f times the clip coefficient of the norm times f).
  TokSlot* tm[kMaxRanks];
  const long long* n_src;  // device int64: this rank's valid targets
  const double* loss_src;  // device fp64: this rank's sum of per-target losses
  long long rows;          // M * B * S of this rank's step
  long long pmc;           // P * M * c: what the reduced gradient is already divided by
  int contribute;
  float* tm_out;
  long long* tm_count;
};

// Gated AdamW on the held slices of one unit + all-gather of the primary slice's new bf16 weights.
struct UpdArgs {
  PeerTable pt;        // data[] = every rank's PARAMETER segment
  char* mc;            // multicast VA of the parameter segment (nullptr = P2P stores; ignored at world 1)
  const int* gate;     // gate[0] verdict, gate[1] step count (already incremented for this step)
  size_t poff;         // byte offset of the unit inside the parameter segment (16 B aligned)
  const __nv_bfloat16* grad;  // local reduced gradients of the unit
  float* master;       // local fp32 state of the unit (full-size arrays; only held slices are valid)
  // moments, 16 B aligned and indexed like master, of the launcher's moment_dtype: kF32 or kBF16. bf16 moments are
  // stored with stochastic rounding whose bits depend only on (soff + local element index, gate[1], which moment).
  void* m;
  void* v;
  size_t nelem;        // elements in the unit (multiple of 8)
  float lr, b1, b2, eps, wd;
  int replication;
  int mode;            // 0 = gated update + push, 1 = refresh (re-broadcast bf16(master) of the primary slice, ungated),
                       // 2 = the same broadcast of bf16(ema) (needs ema)
  // paged state (table != nullptr): master/m/v are pools of 2^page_shift-element pages (2^3 .. 2^30); element e of the
  // flat vector (e = soff + local index) lives at pool[table[e >> page_shift] << page_shift | (e & (page - 1))]. A page
  // is a multiple of 8 elements, so the two 16-byte vectors of one 8-element group never straddle a page. soff is a
  // multiple of 8; bf16 moments hash soff + local index, so flat launches pass the unit's first element there too.
  const int* table;
  size_t soff;
  int page_shift;
  const float* coef;   // gradient clipping: the clip coefficient the commit kernel wrote; the gradient is scaled by it
  // learning-rate schedule (lr_tab != nullptr, 4 B aligned): lr_tab[i] is the fp32 rate of committed update i + 1;
  // update t uses lr_tab[clamp(t, 1, lr_steps) - 1] in place of lr for the step and the decoupled decay (past the table
  // the last rate holds). The launcher sets lr_steps to 0 without a table.
  const float* lr_tab;
  int lr_steps;
  // weight-decay exemptions: n_nd ranges [nd_lo, nd_hi) of the unit get no decay. They are filled as unit-relative
  // element ranges, multiples of 8; the launcher checks them and converts them to the 8-element vectors the kernel reads.
  int n_nd;
  size_t nd_lo[kMaxNoDecay], nd_hi[kMaxNoDecay];
  // exponential moving average of the weights (ema != nullptr; last, so the fields above keep their offsets): 16 B
  // aligned, of the moment type and indexed like master. Every committed update (mode 0) also stores
  // ema' = ema + ema_c * (w' - ema) with the new fp32 master w' and ema_c = fp32(1 - decay); a bf16 EMA is rounded
  // stochastically with bits that depend only on (soff + local element index, gate[1]). Mode 2 is mode 1 with bf16(ema)
  // in place of bf16(master); the launcher rejects it without an EMA.
  void* ema;
  float ema_c;
};

}  // namespace zero1
}  // namespace tft
