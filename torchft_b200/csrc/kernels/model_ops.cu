// Fused bandwidth-bound model ops for the Llama training step (sm_90a):
// RMSNorm fwd/bwd, SwiGLU fwd/bwd, RoPE, softmax-cross-entropy fwd+bwd,
// flat AdamW with fp32 master weights and a device-side commit gate.
//
// The reference (torchft) ships no model; its flagship config (BASELINE.json:
// Llama-3-8B HSDP) gets these from eager PyTorch/torchtitan. Here every
// elementwise/normalisation/activation step is one pass over HBM with 16 B
// accesses; GEMMs stay on cuBLAS and attention on the SDPA library kernel.
// All activations are bf16, all reductions fp32.
#include <algorithm>
#include <stdexcept>
#include <type_traits>
#include <string>

#include "api.h"
#include "common.cuh"

namespace tft {

using bf16 = __nv_bfloat16;
using P8 = Pack<bf16>;

// ------------------------------- RMSNorm ------------------------------------
// A CTA of TPB threads walks rows blockIdx.x, +gridDim.x, ...; a thread owns NV 16-byte vectors of the row (H <= 8*NV*TPB),
// kept PACKED in registers. The row-wide sum costs ONE __syncthreads (warp partials in a double-buffered smem line, every
// thread adds the <= 16 partials itself), and with PF the next row's loads are issued before the current row's reduction so
// a CTA always has a full row of 16 B loads in flight. Small CTAs (128 threads x 4 vectors) with 4 per SM keep ~64 KB per
// SM in flight, more than HBM bandwidth times latency per SM (Little's law) asks for.
constexpr int kRmsMaxVec = 4;
// {forward, backward}: CTA threads, prefetch, CTAs per SM at 128 threads (rmsnorm_tune() overrides; bench/kernel_micro.py
// sweeps them): forward 128 x 4 vectors at 6 CTAs/SM, backward 256 x 2 vectors at 4 CTAs/SM.
static int g_rms_tpb[2] = {128, 256}, g_rms_pf[2] = {1, 1}, g_rms_cps[2] = {6, 4};

template <int TPB>
__device__ __forceinline__ float row_sum(float v, float (*red)[TPB / 32], int& parity) {
  v = warp_sum(v);
  constexpr int NW = TPB / 32;
  if ((threadIdx.x & 31) == 0) red[parity][threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
#pragma unroll
  for (int i = 0; i < NW; ++i) r += red[parity][i];
  parity ^= 1;  // the next row writes the other line: nobody can be two barriers ahead of a reader
  return r;
}

template <int NV, int TPB, bool PF>
__global__ void __launch_bounds__(TPB) rmsnorm_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                          bf16* __restrict__ y, float* __restrict__ rstd, int rows,
                                                          int H, float eps) {
  __shared__ float red[2][TPB / 32];
  const int nvec = H / 8;
  int parity = 0;
  Vec16 wv[NV], xv[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int v = threadIdx.x + i * TPB;
    if (v < nvec) wv[i] = *reinterpret_cast<const Vec16*>(w + v * 8);
  }
  auto load_row = [&](int row, Vec16* dst) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int v = threadIdx.x + i * TPB;
      if (v < nvec) dst[i] = ld_stream(x + (size_t)row * H + v * 8);
    }
  };
  int row = blockIdx.x;
  if (row < rows) load_row(row, xv);
  for (; row < rows; row += gridDim.x) {
    const int next = row + gridDim.x;
    Vec16 nx[NV];
    if (PF && next < rows) load_row(next, nx);
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      if (threadIdx.x + i * TPB < nvec) {
        float f[8];
        P8::unpack(xv[i], f);
#pragma unroll
        for (int k = 0; k < 8; ++k) ss += f[k] * f[k];
      }
    }
    ss = row_sum<TPB>(ss, red, parity);
    const float r = rsqrtf(ss / H + eps);
    if (threadIdx.x == 0) rstd[row] = r;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int v = threadIdx.x + i * TPB;
      if (v < nvec) {
        float f[8], wf[8], o[8];
        P8::unpack(xv[i], f);
        P8::unpack(wv[i], wf);
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = f[k] * r * wf[k];
        st_stream(y + (size_t)row * H + v * 8, P8::pack(o));
      }
    }
    if (PF) {
#pragma unroll
      for (int i = 0; i < NV; ++i) xv[i] = nx[i];
    } else if (next < rows) {
      load_row(next, xv);
    }
  }
}

// dx = rstd * (dy*w - xhat * mean(dy*w*xhat)) (+ dres); dw_partial[block] += dy * xhat
// dres (optional) is the gradient arriving over the residual connection that bypasses the norm:
// adding it here saves the separate elementwise accumulation pass autograd would run.
template <int NV, int TPB, bool PF>
__global__ void __launch_bounds__(TPB) rmsnorm_bwd_kernel(
    const bf16* __restrict__ dy, const bf16* __restrict__ x, const bf16* __restrict__ w,
    const float* __restrict__ rstd, bf16* __restrict__ dx, float* __restrict__ dw_partial,
    const bf16* __restrict__ dres, int rows, int H) {
  __shared__ float red[2][TPB / 32];
  const int nvec = H / 8;
  int parity = 0;
  float dw[NV][8];
  Vec16 wv[NV], xv[NV], gv[NV], rv[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int v = threadIdx.x + i * TPB;
#pragma unroll
    for (int k = 0; k < 8; ++k) dw[i][k] = 0.f;
    if (v < nvec) wv[i] = *reinterpret_cast<const Vec16*>(w + v * 8);
  }
  auto load_row = [&](int row, Vec16* xd, Vec16* gd, Vec16* rd) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int v = threadIdx.x + i * TPB;
      if (v < nvec) {
        const size_t o = (size_t)row * H + v * 8;
        xd[i] = ld_stream(x + o);
        gd[i] = ld_stream(dy + o);
        if (dres != nullptr) rd[i] = ld_stream(dres + o);
      }
    }
  };
  int row = blockIdx.x;
  float r = 0.f;
  if (row < rows) {
    load_row(row, xv, gv, rv);
    r = rstd[row];
  }
  for (; row < rows; row += gridDim.x) {
    const int next = row + gridDim.x;
    Vec16 nx[NV], ng[NV], nr[NV];
    float rn = 0.f;
    if (PF && next < rows) {
      load_row(next, nx, ng, nr);
      rn = rstd[next];
    }
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      if (threadIdx.x + i * TPB < nvec) {
        float xf[8], dyf[8], wf[8];
        P8::unpack(xv[i], xf);
        P8::unpack(gv[i], dyf);
        P8::unpack(wv[i], wf);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float xh = xf[k] * r;
          dot += dyf[k] * wf[k] * xh;
          dw[i][k] += dyf[k] * xh;
        }
      }
    }
    dot = row_sum<TPB>(dot, red, parity) / H;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int v = threadIdx.x + i * TPB;
      if (v < nvec) {
        float xf[8], dyf[8], wf[8], o[8];
        P8::unpack(xv[i], xf);
        P8::unpack(gv[i], dyf);
        P8::unpack(wv[i], wf);
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = r * (dyf[k] * wf[k] - xf[k] * r * dot);
        if (dres != nullptr) {
          float rf[8];
          P8::unpack(rv[i], rf);
#pragma unroll
          for (int k = 0; k < 8; ++k) o[k] += rf[k];
        }
        st_stream(dx + (size_t)row * H + v * 8, P8::pack(o));
      }
    }
    if (PF) {
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        xv[i] = nx[i];
        gv[i] = ng[i];
        rv[i] = nr[i];
      }
      r = rn;
    } else if (next < rows) {
      load_row(next, xv, gv, rv);
      r = rstd[next];
    }
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int v = threadIdx.x + i * TPB;
    if (v < nvec) {
      float* o = dw_partial + (size_t)blockIdx.x * H + v * 8;
      *reinterpret_cast<float4*>(o) = make_float4(dw[i][0], dw[i][1], dw[i][2], dw[i][3]);
      *reinterpret_cast<float4*>(o + 4) = make_float4(dw[i][4], dw[i][5], dw[i][6], dw[i][7]);
    }
  }
}

// dw[h] (+)= sum_b partial[b][h]: a CTA owns 32 columns; its 32 warps stride over the partial rows (a warp load is one
// 128 B line, up to 8 independent loads in flight per lane), then the 32 per-warp sums meet in shared memory. Fewer warps
// with fewer loads in flight leave the column sum latency-bound: dozens of dependent rounds per CTA.
__global__ void __launch_bounds__(1024) colsum_kernel(const float* __restrict__ partial, int nb, int H,
                                                      bf16* __restrict__ dw, int accumulate) {
  __shared__ float acc[32][33];
  const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
  const int h = blockIdx.x * 32 + lane;
  float s = 0.f;
  if (h < H) {
    int b = wrp;
    for (; b + 7 * 32 < nb; b += 8 * 32) {
      float v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = __ldcs(partial + (size_t)(b + u * 32) * H + h);
#pragma unroll
      for (int u = 0; u < 8; ++u) s += v[u];
    }
    for (; b < nb; b += 32) s += __ldcs(partial + (size_t)b * H + h);
  }
  acc[wrp][lane] = s;
  __syncthreads();
  if (wrp == 0 && h < H) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) t += acc[i][lane];
    if (accumulate) t += __bfloat162float(dw[h]);
    dw[h] = __float2bfloat16(t);
  }
}

// ------------------------------- SwiGLU -------------------------------------
// gu: [T, 2F] (gate | up), y: [T, F]
__global__ void __launch_bounds__(512) swiglu_fwd_kernel(const bf16* __restrict__ gu,
                                                         bf16* __restrict__ y, size_t T, int F) {
  const size_t nvec_row = F / 8;
  const size_t total = T * nvec_row;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const size_t t = i / nvec_row, c = (i % nvec_row) * 8;
    float g[8], u[8], o[8];
    P8::unpack(ld_stream(gu + t * 2 * F + c), g);
    P8::unpack(ld_stream(gu + t * 2 * F + F + c), u);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = g[k] / (1.f + __expf(-g[k])) * u[k];
    st_stream(y + t * F + c, P8::pack(o));
  }
}

__global__ void __launch_bounds__(512) swiglu_bwd_kernel(const bf16* __restrict__ dy,
                                                         const bf16* __restrict__ gu,
                                                         bf16* __restrict__ dgu, size_t T, int F) {
  const size_t nvec_row = F / 8;
  const size_t total = T * nvec_row;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const size_t t = i / nvec_row, c = (i % nvec_row) * 8;
    float g[8], u[8], d[8], dg[8], du[8];
    P8::unpack(ld_stream(gu + t * 2 * F + c), g);
    P8::unpack(ld_stream(gu + t * 2 * F + F + c), u);
    P8::unpack(ld_stream(dy + t * F + c), d);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float s = 1.f / (1.f + __expf(-g[k]));
      const float silu = g[k] * s;
      du[k] = d[k] * silu;
      dg[k] = d[k] * u[k] * (s + silu * (1.f - s));
    }
    st_stream(dgu + t * 2 * F + c, P8::pack(dg));
    st_stream(dgu + t * 2 * F + F + c, P8::pack(du));
  }
}

// ------------------------------- RoPE ---------------------------------------
// Interleaved-pair rotation (x[2i], x[2i+1]) by angle pos * theta_i; cs holds
// (cos, sin) pairs: cs[pos][i] = float2. sign = +1 forward, -1 backward.
// in/out row strides in elements so q/k can be read straight out of the packed
// qkv projection and written contiguous.
// A thread keeps its vector-in-head index for the whole kernel and walks (token, head) "slots" two at a time (both 16 B
// loads issued before either is used); all index math is 32-bit (64-bit divisions per vector and a single load in flight
// per thread leave the kernel latency-bound).
__global__ void __launch_bounds__(256) rope_kernel(const bf16* __restrict__ in, bf16* __restrict__ out,
                                                   const float2* __restrict__ cs, unsigned nslots, unsigned S,
                                                   unsigned heads, unsigned D, size_t in_stride, size_t out_stride,
                                                   float sign) {
  const unsigned vph = D / 8;
  const unsigned vh = threadIdx.x % vph, s0 = threadIdx.x / vph, per = blockDim.x / vph;
  for (unsigned base = blockIdx.x * 2 * per; base < nslots; base += gridDim.x * 2 * per) {
    Vec16 v[2];
    unsigned t[2], h[2];
    bool ok[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const unsigned g = base + s0 + j * per;
      ok[j] = g < nslots;
      t[j] = g / heads;
      h[j] = g - t[j] * heads;
      if (ok[j]) v[j] = ld_stream(in + (size_t)t[j] * in_stride + h[j] * D + vh * 8);
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      if (!ok[j]) continue;
      const unsigned pos = t[j] % S;
      const float4* c = reinterpret_cast<const float4*>(cs + (size_t)pos * (D / 2) + vh * 4);
      const float4 c0 = c[0], c1 = c[1];
      const float cx[4] = {c0.x, c0.z, c1.x, c1.z}, sy[4] = {c0.y, c0.w, c1.y, c1.w};
      float f[8], o[8];
      P8::unpack(v[j], f);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float sn = sy[k] * sign;
        o[2 * k] = f[2 * k] * cx[k] - f[2 * k + 1] * sn;
        o[2 * k + 1] = f[2 * k] * sn + f[2 * k + 1] * cx[k];
      }
      st_stream(out + (size_t)t[j] * out_stride + h[j] * D + vh * 8, P8::pack(o));
    }
  }
}

// RoPE + q/k/v split (dir 0: packed qkv projection -> rotated q, rotated k, v) and its backward (dir 1: dq, dk, dv in ANY
// [B, S, H, D] stride order -> inverse-rotated packed d_qkv) as ONE launch: every (token, head) slot of the packed row is
// read once and written once; the v heads are a plain copy. Replaces two rope launches plus the library's strided copy of
// v in forward, and two rope launches plus three .contiguous()/copy_ kernels in backward.
struct RopeQKVArgs {
  bf16* packed;
  size_t row;  // elements per packed row = (Hq + 2 Hkv) * D
  bf16* sep[3];
  size_t sb[3], ss[3], sh[3];  // element strides of q / k / v: batch, position, head
  unsigned nh[3];
  const float2* cs;
  unsigned T, S, D;
  int dir;
};

__global__ void __launch_bounds__(256) rope_qkv_kernel(const RopeQKVArgs a) {
  const unsigned vph = a.D / 8;
  const unsigned vh = threadIdx.x % vph, s0 = threadIdx.x / vph, per = blockDim.x / vph;
  const unsigned heads = a.nh[0] + a.nh[1] + a.nh[2];
  const unsigned nslots = a.T * heads;
  const float sign = a.dir == 0 ? 1.f : -1.f;
  for (unsigned base = blockIdx.x * 2 * per; base < nslots; base += gridDim.x * 2 * per) {
    Vec16 v[2];
    bf16* dst[2];
    unsigned pos[2];
    bool ok[2], rot[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const unsigned g = base + s0 + j * per;
      ok[j] = g < nslots;
      const unsigned t = g / heads, hh = g - t * heads;
      const unsigned b = t / a.S;
      pos[j] = t - b * a.S;
      const int w = hh < a.nh[0] ? 0 : (hh < a.nh[0] + a.nh[1] ? 1 : 2);
      const unsigned h = hh - (w == 0 ? 0 : (w == 1 ? a.nh[0] : a.nh[0] + a.nh[1]));
      rot[j] = w < 2;
      bf16* pk = a.packed + (size_t)t * a.row + (size_t)hh * a.D + vh * 8;
      bf16* sp = a.sep[w] + b * a.sb[w] + pos[j] * a.ss[w] + h * a.sh[w] + vh * 8;
      dst[j] = a.dir == 0 ? sp : pk;
      if (ok[j]) v[j] = ld_stream(a.dir == 0 ? pk : sp);
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      if (!ok[j]) continue;
      if (rot[j]) {
        const float4* c = reinterpret_cast<const float4*>(a.cs + (size_t)pos[j] * (a.D / 2) + vh * 4);
        const float4 c0 = c[0], c1 = c[1];
        const float cx[4] = {c0.x, c0.z, c1.x, c1.z}, sy[4] = {c0.y, c0.w, c1.y, c1.w};
        float f[8], o[8];
        P8::unpack(v[j], f);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float sn = sy[k] * sign;
          o[2 * k] = f[2 * k] * cx[k] - f[2 * k + 1] * sn;
          o[2 * k + 1] = f[2 * k] * sn + f[2 * k + 1] * cx[k];
        }
        v[j] = P8::pack(o);
      }
      st_stream(dst[j], v[j]);
    }
  }
}

// ------------------------------- Cross entropy ------------------------------
// One CTA per row of logits [rows, V] (bf16). Writes loss[row] (fp32) and
// overwrites the logits row with d(loss_sum * grad_scale)/dlogits in bf16.
// Rows whose target == ignore_index get loss 0 and zero gradient.
__global__ void __launch_bounds__(1024) xent_fwd_bwd_kernel(bf16* __restrict__ logits,
                                                            const long long* __restrict__ target,
                                                            float* __restrict__ loss, int V,
                                                            size_t row_stride, float grad_scale,
                                                            long long ignore_index) {
  __shared__ float red[32];
  const size_t row = blockIdx.x;
  bf16* lr = logits + row * row_stride;
  const long long tgt = target[row];
  const int nvec = V / 8;
  if (tgt == ignore_index) {
    for (int v = threadIdx.x; v < nvec; v += blockDim.x) st_stream(lr + v * 8, Vec16{0, 0, 0, 0});
    for (int k = nvec * 8 + threadIdx.x; k < V; k += blockDim.x) lr[k] = __float2bfloat16(0.f);
    if (threadIdx.x == 0) loss[row] = 0.f;
    return;
  }
  // pass 1: online max / sum-exp
  float m = -INFINITY, s = 0.f;
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    float f[8];
    P8::unpack(*reinterpret_cast<const Vec16*>(lr + v * 8), f);
    float lm = f[0];
#pragma unroll
    for (int k = 1; k < 8; ++k) lm = fmaxf(lm, f[k]);
    const float nm = fmaxf(m, lm);
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) acc += __expf(f[k] - nm);
    s = s * __expf(m - nm) + acc;
    m = nm;
  }
  for (int k = nvec * 8 + threadIdx.x; k < V; k += blockDim.x) {
    const float x = __bfloat162float(lr[k]);
    const float nm = fmaxf(m, x);
    s = s * __expf(m - nm) + __expf(x - nm);
    m = nm;
  }
  const float gm = block_max(m, red);
  s = (m == -INFINITY) ? 0.f : s * __expf(m - gm);
  const float gs = block_sum(s, red);
  const float lse = gm + __logf(gs);
  if (threadIdx.x == 0) loss[row] = lse - __bfloat162float(lr[tgt]);
  __syncthreads();  // everyone done reading lr[tgt] region before overwrite
  const float inv = grad_scale / gs;
  // pass 2: grad = (softmax - onehot) * grad_scale   (row is L2-resident)
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    float f[8], o[8];
    P8::unpack(*reinterpret_cast<const Vec16*>(lr + v * 8), f);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      o[k] = __expf(f[k] - gm) * inv;
      if ((long long)v * 8 + k == tgt) o[k] -= grad_scale;
    }
    st_stream(lr + v * 8, P8::pack(o));
  }
  for (int k = nvec * 8 + threadIdx.x; k < V; k += blockDim.x) {
    float o = __expf(__bfloat162float(lr[k]) - gm) * inv;
    if (k == tgt) o -= grad_scale;
    lr[k] = __float2bfloat16(o);
  }
}

// ------------------------------- AdamW --------------------------------------
// Flat multi-tensor AdamW: bf16 params + fp32 master/m/v, bf16 grads.
// `gate` (nullable) points at a device int: the update is skipped entirely
// when *gate == 0, which lets the launch be enqueued before the host has the
// should_commit verdict (torchft/optim.py:52-55 semantics, no extra sync).
struct AdamArgs {
  bf16* p;
  float* master;
  float* m;
  float* v;
  const bf16* g;
  size_t n;
  float lr, b1, b2, eps, wd, bc1, bc2, gscale;
  const int* gate;
};

__global__ void __launch_bounds__(512, 2) adamw_kernel(AdamArgs a) {
  if (a.gate != nullptr && *a.gate == 0) return;
  const size_t nvec = a.n / 8;
  const float step_size = a.lr / a.bc1;
  const float inv_bc2_sqrt = rsqrtf(a.bc2);
  const float decay = 1.f - a.lr * a.wd;
  for (size_t v = blockIdx.x * (size_t)blockDim.x + threadIdx.x; v < nvec;
       v += (size_t)gridDim.x * blockDim.x) {
    // all 7 x 16 B loads in flight before any use (28 B/param streams through once)
    const Vec16 gv = ld_stream(a.g + v * 8);
    const Vec16 w0 = ld_stream(a.master + v * 8), w1 = ld_stream(a.master + v * 8 + 4);
    const Vec16 m0 = ld_stream(a.m + v * 8), m1 = ld_stream(a.m + v * 8 + 4);
    const Vec16 v0 = ld_stream(a.v + v * 8), v1 = ld_stream(a.v + v * 8 + 4);
    float g[8], w[8], m[8], vv[8];
    P8::unpack(gv, g);
    Pack<float>::unpack(w0, w);
    Pack<float>::unpack(w1, w + 4);
    Pack<float>::unpack(m0, m);
    Pack<float>::unpack(m1, m + 4);
    Pack<float>::unpack(v0, vv);
    Pack<float>::unpack(v1, vv + 4);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float gr = g[k] * a.gscale;
      m[k] = a.b1 * m[k] + (1.f - a.b1) * gr;
      vv[k] = a.b2 * vv[k] + (1.f - a.b2) * gr * gr;
      const float denom = sqrtf(vv[k]) * inv_bc2_sqrt + a.eps;
      w[k] = w[k] * decay - step_size * __fdividef(m[k], denom);
    }
    st_stream(a.master + v * 8, Pack<float>::pack(w));
    st_stream(a.master + v * 8 + 4, Pack<float>::pack(w + 4));
    st_stream(a.m + v * 8, Pack<float>::pack(m));
    st_stream(a.m + v * 8 + 4, Pack<float>::pack(m + 4));
    st_stream(a.v + v * 8, Pack<float>::pack(vv));
    st_stream(a.v + v * 8 + 4, Pack<float>::pack(vv + 4));
    st_stream(a.p + v * 8, P8::pack(w));
  }
  if (blockIdx.x == 0) {
    for (size_t k = nvec * 8 + threadIdx.x; k < a.n; k += blockDim.x) {
      const float gr = __bfloat162float(a.g[k]) * a.gscale;
      const float m = a.b1 * a.m[k] + (1.f - a.b1) * gr;
      const float vv = a.b2 * a.v[k] + (1.f - a.b2) * gr * gr;
      const float denom = sqrtf(vv) * inv_bc2_sqrt + a.eps;
      const float w = a.master[k] * decay - step_size * (m / denom);
      a.m[k] = m;
      a.v[k] = vv;
      a.master[k] = w;
      a.p[k] = __float2bfloat16(w);
    }
  }
}

// DiLoCo outer step, fused: averaged pseudo-gradient -> Nesterov/momentum SGD on the last global weights ->
// new global weights saved to the backup -> live weights = lerp(new global, local, alpha). The reference runs these
// as four passes over the fragment (set grads, outer_optimizer.step(), save_parameters, _merge_parameters:
// upstream torchft/local_sgd.py:339-384,445-475); here every element is read and written once.
template <typename T>
__global__ void __launch_bounds__(512, 2) diloco_outer_kernel(T* __restrict__ param, T* __restrict__ original,
                                                               const T* __restrict__ grad, float* __restrict__ mom,
                                                               size_t n, float lr, float mu, int nesterov, float alpha,
                                                               const int* __restrict__ gate) {
  if (gate != nullptr && *gate == 0) return;
  constexpr int N = Pack<T>::N;
  const size_t nvec = n / N;
  for (size_t v = blockIdx.x * (size_t)blockDim.x + threadIdx.x; v < nvec; v += (size_t)gridDim.x * blockDim.x) {
    const Vec16 gv = ld_stream(grad + v * N), ov = ld_stream(original + v * N), lv = ld_stream(param + v * N);
    float g[N], o[N], l[N], b[N];
    Pack<T>::unpack(gv, g);
    Pack<T>::unpack(ov, o);
    Pack<T>::unpack(lv, l);
#pragma unroll
    for (int i = 0; i < N; i += 4) Pack<float>::unpack(ld_stream(mom + v * N + i), b + i);
#pragma unroll
    for (int i = 0; i < N; ++i) {
      float step = g[i];
      if (mu != 0.f) {
        b[i] = mu * b[i] + g[i];
        step = nesterov ? g[i] + mu * b[i] : b[i];
      }
      o[i] -= lr * step;
      l[i] = o[i] + alpha * (l[i] - o[i]);
    }
#pragma unroll
    for (int i = 0; i < N; i += 4) st_stream(mom + v * N + i, Pack<float>::pack(b + i));
    st_stream(original + v * N, Pack<T>::pack(o));
    st_stream(param + v * N, Pack<T>::pack(l));
  }
  if (blockIdx.x == 0) {
    for (size_t k = nvec * N + threadIdx.x; k < n; k += blockDim.x) {
      const float g = float(grad[k]);
      float b = mom[k], step = g;
      if (mu != 0.f) {
        b = mu * b + g;
        step = nesterov ? g + mu * b : b;
        mom[k] = b;
      }
      const float o = float(original[k]) - lr * step;
      original[k] = T(o);
      param[k] = T(o + alpha * (float(param[k]) - o));
    }
  }
}

// sum of squares of a bf16 buffer -> out[0] (+=), for grad-norm clipping
__global__ void __launch_bounds__(512) sumsq_kernel(const bf16* __restrict__ g, size_t n,
                                                    float* __restrict__ out) {
  __shared__ float red[32];
  const size_t nvec = n / 8;
  float s = 0.f;
  for (size_t v = blockIdx.x * (size_t)blockDim.x + threadIdx.x; v < nvec;
       v += (size_t)gridDim.x * blockDim.x) {
    float f[8];
    P8::unpack(ld_stream(g + v * 8), f);
#pragma unroll
    for (int k = 0; k < 8; ++k) s += f[k] * f[k];
  }
  if (blockIdx.x == 0) {
    for (size_t k = nvec * 8 + threadIdx.x; k < n; k += blockDim.x) {
      const float x = __bfloat162float(g[k]);
      s += x * x;
    }
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) atomicAdd(out, s);
}

// ------------------------------- heal copy ----------------------------------
// Live-recovery transport: stream state_dict shards GPU->GPU over NVLink from
// inside a kernel (reference moves them GPU->CPU->TCP->CPU->GPU,
// torchft/checkpointing/http_transport.py:219-284). Each table entry is one
// contiguous byte range; CTAs stride over fixed-size chunks of all entries.
struct CopyEntry {
  const char* src;
  char* dst;
  size_t bytes;
  size_t chunk0;  // index of this entry's first chunk
};

__global__ void __launch_bounds__(512) heal_copy_kernel(const CopyEntry* __restrict__ table,
                                                        int nentries, size_t total_chunks,
                                                        size_t chunk_bytes) {
  for (size_t c = blockIdx.x; c < total_chunks; c += gridDim.x) {
    // binary search for the entry containing chunk c
    int lo = 0, hi = nentries - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (table[mid].chunk0 <= c) lo = mid; else hi = mid - 1;
    }
    const CopyEntry e = table[lo];
    const size_t start = (c - e.chunk0) * chunk_bytes;
    const size_t end = min(start + chunk_bytes, e.bytes);
    const char* s = e.src + start;
    char* d = e.dst + start;
    const size_t len = end - start;
    if ((((uintptr_t)s | (uintptr_t)d) & 15) == 0) {
      const size_t nv = len / 16;
      // 8 x 16 B loads in flight per thread: a peer (NVLink) read has microseconds of latency,
      // so one outstanding load per thread caps a 64-CTA copy far below link bandwidth; 8 per
      // thread puts > 4 MB in flight, more than link bandwidth times peer latency.
      constexpr int U = 8;
      size_t v = threadIdx.x;
      for (; v + (size_t)(U - 1) * blockDim.x < nv; v += (size_t)U * blockDim.x) {
        Vec16 r[U];
#pragma unroll
        for (int u = 0; u < U; ++u) r[u] = ld_stream(s + (v + (size_t)u * blockDim.x) * 16);
#pragma unroll
        for (int u = 0; u < U; ++u) st_stream(d + (v + (size_t)u * blockDim.x) * 16, r[u]);
      }
      for (; v < nv; v += blockDim.x) st_stream(d + v * 16, ld_stream(s + v * 16));
      for (size_t k = nv * 16 + threadIdx.x; k < len; k += blockDim.x) d[k] = s[k];
    } else {
      for (size_t k = threadIdx.x; k < len; k += blockDim.x) d[k] = s[k];
    }
  }
}

// ------------------------------- heal copy, TMA bulk variant -------------------------------
// Same job, driven by the copy engine instead of the LSU: ONE thread per CTA runs a 4-stage ring of 16 KiB shared-memory
// buffers -- `cp.async.bulk` global->shared (completion on an mbarrier, transaction-byte counted) followed by
// `cp.async.bulk` shared->global (bulk groups) -- so 64 KiB are in flight per CTA with 32 threads and ~30 registers, three
// CTAs per SM. No data ever passes through registers. Source may be a mapped peer (NVLink) address. Needs 16-byte
// aligned ranges; the host falls back to heal_copy_kernel otherwise. SASS: UBLKCP (bulk copy), SYNCS (mbarrier).
constexpr int kBulkStages = 4;
constexpr uint32_t kBulkBytes = 16 * 1024;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done = 0;
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  }
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}

// Cursor over the 16 KiB pieces of the chunks c = blockIdx.x, blockIdx.x + gridDim.x, ... owned by this CTA.
struct PieceCursor {
  const CopyEntry* table;
  int nentries;
  size_t total_chunks, chunk_bytes;
  size_t c;        // current chunk
  size_t off;      // byte offset of the next piece inside the chunk
  const char* src;
  char* dst;
  size_t len;      // bytes of the current chunk (multiple of 16 except possibly the entry's last chunk)
  __device__ void load_chunk() {
    if (c >= total_chunks) return;
    int lo = 0, hi = nentries - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (table[mid].chunk0 <= c) lo = mid; else hi = mid - 1;
    }
    const CopyEntry e = table[lo];
    const size_t start = (c - e.chunk0) * chunk_bytes;
    src = e.src + start;
    dst = e.dst + start;
    len = min(chunk_bytes, e.bytes - start);
    off = 0;
  }
  __device__ bool next(const char** s, char** d, uint32_t* n) {
    while (c < total_chunks && off >= (len & ~size_t(15))) {
      c += gridDim.x;
      load_chunk();
    }
    if (c >= total_chunks) return false;
    const size_t body = len & ~size_t(15);
    *n = (uint32_t)min((size_t)kBulkBytes, body - off);
    *s = src + off;
    *d = dst + off;
    off += *n;
    return true;
  }
};

__global__ void __launch_bounds__(32) heal_copy_bulk_kernel(const CopyEntry* __restrict__ table, int nentries,
                                                            size_t total_chunks, size_t chunk_bytes) {
  extern __shared__ __align__(128) unsigned char ring[];
  __shared__ __align__(8) uint64_t full[kBulkStages];
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 0; i < kBulkStages; ++i) mbar_init(&full[i], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  // sub-16-byte tails of entries (at most one per entry) are copied by the lanes the pipeline does not need
  if (threadIdx.x != 0) {
    for (int e = blockIdx.x * 31 + (threadIdx.x - 1); e < nentries; e += gridDim.x * 31) {
      const CopyEntry t = table[e];
      for (size_t k = t.bytes & ~size_t(15); k < t.bytes; ++k) t.dst[k] = t.src[k];
    }
    return;
  }
  PieceCursor ld{table, nentries, total_chunks, chunk_bytes, blockIdx.x, 0, nullptr, nullptr, 0};
  ld.load_chunk();
  // the store side replays the same sequence of pieces: remember them in a small ring instead of a second cursor
  char* sdst[kBulkStages];
  uint32_t slen[kBulkStages];
  size_t issued = 0, stored = 0;
  const char* s;
  char* d;
  uint32_t n;
  // prologue: fill the ring
  while (issued < kBulkStages && ld.next(&s, &d, &n)) {
    const int st = (int)(issued % kBulkStages);
    mbar_expect_tx(&full[st], n);
    bulk_g2s(ring + (size_t)st * kBulkBytes, s, n, &full[st]);
    sdst[st] = d;
    slen[st] = n;
    ++issued;
  }
  while (stored < issued) {
    const int st = (int)(stored % kBulkStages);
    mbar_wait(&full[st], (uint32_t)((stored / kBulkStages) & 1));
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    bulk_s2g(sdst[st], ring + (size_t)st * kBulkBytes, slen[st]);
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    ++stored;
    // refill the stage of the PREVIOUS piece: its store has finished reading shared memory once at most one group is pending
    if (stored >= 2 && issued == stored - 2 + kBulkStages) {
      asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
      if (ld.next(&s, &d, &n)) {
        const int rs = (int)(issued % kBulkStages);
        mbar_expect_tx(&full[rs], n);
        bulk_g2s(ring + (size_t)rs * kBulkBytes, s, n, &full[rs]);
        sdst[rs] = d;
        slen[rs] = n;
        ++issued;
      }
    }
  }
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// ------------------------------- launchers ----------------------------------
static int grid_for(size_t work_items, int threads, int cap = kNumSMs * 8) {
  size_t g = (work_items + threads - 1) / threads;
  if (g < 1) g = 1;
  if (g > (size_t)cap) g = cap;
  return (int)g;
}

// (TPB, NV) for a row of nvec 16 B vectors: the tuned CTA size if NV <= 4 covers the row, else the next larger CTA.
static void rms_shape(int nvec, int bwd, int& tpb, int& nv) {
  for (tpb = g_rms_tpb[bwd]; tpb <= 512; tpb *= 2) {
    const int need = (nvec + tpb - 1) / tpb;
    nv = need <= 1 ? 1 : need <= 2 ? 2 : 4;
    if (need <= kRmsMaxVec) return;
  }
  tpb = 512;
  nv = kRmsMaxVec;
}
static int rms_grid(int rows, int bwd, int tpb) {
  const int cap = kNumSMs * std::max(1, g_rms_cps[bwd] * 128 / tpb);
  return rows < cap ? rows : cap;
}

void rmsnorm_tune(int bwd, int tpb, int prefetch, int ctas_per_sm_at_128) {
  if (tpb != 128 && tpb != 256 && tpb != 512) throw std::runtime_error("rmsnorm_tune: tpb must be 128, 256 or 512");
  bwd = bwd ? 1 : 0;
  g_rms_tpb[bwd] = tpb;
  g_rms_pf[bwd] = prefetch ? 1 : 0;
  g_rms_cps[bwd] = std::max(1, ctas_per_sm_at_128);
}

#define RMS_DISPATCH(KERNEL, BWD, ...)                                                                         \
  do {                                                                                                     \
    auto go = [&](auto nvc, auto tpbc, auto pfc) {                                                         \
      KERNEL<decltype(nvc)::value, decltype(tpbc)::value, decltype(pfc)::value><<<grid, tpb, 0, s>>>(__VA_ARGS__); \
    };                                                                                                     \
    auto by_pf = [&](auto nvc, auto tpbc) {                                                                \
      if (g_rms_pf[BWD] && !(nv == 4 && tpb == 512)) go(nvc, tpbc, std::true_type{}); else go(nvc, tpbc, std::false_type{}); \
    };                                                                                                     \
    auto by_tpb = [&](auto nvc) {                                                                          \
      if (tpb == 128) by_pf(nvc, std::integral_constant<int, 128>{});                                      \
      else if (tpb == 256) by_pf(nvc, std::integral_constant<int, 256>{});                                 \
      else by_pf(nvc, std::integral_constant<int, 512>{});                                                 \
    };                                                                                                     \
    if (nv == 1) by_tpb(std::integral_constant<int, 1>{});                                                 \
    else if (nv == 2) by_tpb(std::integral_constant<int, 2>{});                                            \
    else by_tpb(std::integral_constant<int, 4>{});                                                         \
  } while (0)

void rmsnorm_fwd_launch(const void* x, const void* w, void* y, float* rstd, int rows, int H,
                        float eps, cudaStream_t s) {
  if (H % 8 || H > 8 * kRmsMaxVec * 512) throw std::runtime_error("rmsnorm: H must be %8 and <= 16384");
  int tpb, nv;
  rms_shape(H / 8, 0, tpb, nv);
  const int grid = rms_grid(rows, 0, tpb);
  RMS_DISPATCH(rmsnorm_fwd_kernel, 0, (const bf16*)x, (const bf16*)w, (bf16*)y, rstd, rows, H, eps);
  TFT_CUDA_CHECK(cudaGetLastError());
}

// rows of the fp32 partial-dw buffer the caller must provide (an upper bound on the grid for any H)
int rmsnorm_bwd_grid(int rows) { return rms_grid(rows, 1, 128); }

void rmsnorm_bwd_launch(const void* dy, const void* x, const void* w, const float* rstd, void* dx,
                        float* dw_partial, void* dw, int accumulate, int rows, int H,
                        cudaStream_t s, const void* dres) {
  if (H % 8 || H > 8 * kRmsMaxVec * 512) throw std::runtime_error("rmsnorm: H must be %8 and <= 16384");
  int tpb, nv;
  rms_shape(H / 8, 1, tpb, nv);
  const int grid = rms_grid(rows, 1, tpb);
  RMS_DISPATCH(rmsnorm_bwd_kernel, 1, (const bf16*)dy, (const bf16*)x, (const bf16*)w, rstd, (bf16*)dx, dw_partial,
               (const bf16*)dres, rows, H);
  colsum_kernel<<<(H + 31) / 32, 1024, 0, s>>>(dw_partial, grid, H, (bf16*)dw, accumulate);
  TFT_CUDA_CHECK(cudaGetLastError());
}

void swiglu_fwd_launch(const void* gu, void* y, size_t T, int F, cudaStream_t s) {
  if (F % 8) throw std::runtime_error("swiglu: F must be a multiple of 8");
  swiglu_fwd_kernel<<<grid_for(T * (F / 8), 512), 512, 0, s>>>((const bf16*)gu, (bf16*)y, T, F);
  TFT_CUDA_CHECK(cudaGetLastError());
}
void swiglu_bwd_launch(const void* dy, const void* gu, void* dgu, size_t T, int F, cudaStream_t s) {
  if (F % 8) throw std::runtime_error("swiglu: F must be a multiple of 8");
  swiglu_bwd_kernel<<<grid_for(T * (F / 8), 512), 512, 0, s>>>((const bf16*)dy, (const bf16*)gu,
                                                               (bf16*)dgu, T, F);
  TFT_CUDA_CHECK(cudaGetLastError());
}

void rope_launch(const void* in, void* out, const void* cs, size_t T, int S, int heads, int D,
                 size_t in_stride, size_t out_stride, float sign, cudaStream_t s) {
  if (D % 8 || D > 2048) throw std::runtime_error("rope: head_dim must be a multiple of 8 and <= 2048");
  if (T * (size_t)heads >= (1ull << 31)) throw std::runtime_error("rope: tokens * heads must be < 2^31");
  if (T == 0) return;
  const unsigned vph = D / 8, per = 256 / vph, threads = per * vph;  // whole (token, head) slots per CTA pass
  const unsigned nslots = (unsigned)(T * heads);
  const unsigned grid = std::min<unsigned>((nslots + 2 * per - 1) / (2 * per), kNumSMs * 8);
  rope_kernel<<<grid, threads, 0, s>>>((const bf16*)in, (bf16*)out, (const float2*)cs, nslots, (unsigned)S,
                                       (unsigned)heads, (unsigned)D, in_stride, out_stride, sign);
  TFT_CUDA_CHECK(cudaGetLastError());
}

void rope_qkv_launch(void* packed, size_t row, void* q, void* k, void* v, const int64_t* strides9, const void* cs,
                     size_t T, int S, int D, int Hq, int Hkv, int dir, cudaStream_t s) {
  if (D % 8 || D > 2048) throw std::runtime_error("rope_qkv: head_dim must be a multiple of 8 and <= 2048");
  // v == nullptr: only q and k are produced (forward keeps v as a strided view of the packed projection)
  const size_t heads = (size_t)Hq + (size_t)Hkv * (v != nullptr ? 2 : 1);
  if (T * heads >= (1ull << 31)) throw std::runtime_error("rope_qkv: tokens * heads must be < 2^31");
  if (row != ((size_t)Hq + 2 * (size_t)Hkv) * D) throw std::runtime_error("rope_qkv: packed row must be (Hq + 2 Hkv) * D");
  if (T == 0) return;
  RopeQKVArgs a{};
  a.packed = (bf16*)packed;
  a.row = row;
  a.sep[0] = (bf16*)q;
  a.sep[1] = (bf16*)k;
  a.sep[2] = (bf16*)v;
  for (int w = 0; w < 3; ++w) {
    a.sb[w] = (size_t)strides9[3 * w];
    a.ss[w] = (size_t)strides9[3 * w + 1];
    a.sh[w] = (size_t)strides9[3 * w + 2];
    if ((a.sb[w] | a.ss[w] | a.sh[w]) % 8) throw std::runtime_error("rope_qkv: strides must be multiples of 8 elements");
  }
  a.nh[0] = Hq;
  a.nh[1] = Hkv;
  a.nh[2] = v != nullptr ? Hkv : 0;
  a.cs = (const float2*)cs;
  a.T = (unsigned)T;
  a.S = (unsigned)S;
  a.D = (unsigned)D;
  a.dir = dir;
  const unsigned vph = D / 8, per = 256 / vph, threads = per * vph;
  const unsigned nslots = (unsigned)(T * heads);
  const unsigned grid = std::min<unsigned>((nslots + 2 * per - 1) / (2 * per), kNumSMs * 8);
  rope_qkv_kernel<<<grid, threads, 0, s>>>(a);
  TFT_CUDA_CHECK(cudaGetLastError());
}

void xent_launch(void* logits, const void* target, float* loss, size_t rows, int V,
                 size_t row_stride, float grad_scale, long long ignore_index, cudaStream_t s) {
  if (row_stride % 8) throw std::runtime_error("xent: row stride must be a multiple of 8");
  if (rows == 0) return;
  xent_fwd_bwd_kernel<<<(unsigned)rows, 1024, 0, s>>>((bf16*)logits, (const long long*)target, loss,
                                                      V, row_stride, grad_scale, ignore_index);
  TFT_CUDA_CHECK(cudaGetLastError());
}

void adamw_launch(void* p, float* master, float* m, float* v, const void* g, size_t n, float lr,
                  float b1, float b2, float eps, float wd, float bc1, float bc2, float gscale,
                  const int* gate, int max_blocks, cudaStream_t s) {
  AdamArgs a{(bf16*)p, master, m, v, (const bf16*)g, n, lr, b1, b2, eps, wd, bc1, bc2, gscale, gate};
  // Many short CTAs (16 per SM) keep both resident slots of every SM refilled; a CTA-cap sweep
  // (bench/kernel_micro.py) reached the most HBM bandwidth at the largest cap. max_blocks > 0 overrides.
  adamw_kernel<<<grid_for(n / 8 + 1, 512, max_blocks > 0 ? max_blocks : kNumSMs * 16), 512, 0, s>>>(a);
  TFT_CUDA_CHECK(cudaGetLastError());
}

void diloco_outer_launch(void* param, void* original, const void* grad, float* mom, size_t n, int dtype, float lr,
                         float mu, int nesterov, float alpha, const int* gate, cudaStream_t s) {
  const int grid = grid_for(n / 4 + 1, 512, kNumSMs * 16);
  switch (dtype) {
    case kF32:
      diloco_outer_kernel<float><<<grid, 512, 0, s>>>((float*)param, (float*)original, (const float*)grad, mom, n, lr, mu,
                                                      nesterov, alpha, gate);
      break;
    case kBF16:
      diloco_outer_kernel<bf16><<<grid, 512, 0, s>>>((bf16*)param, (bf16*)original, (const bf16*)grad, mom, n, lr, mu,
                                                     nesterov, alpha, gate);
      break;
    case kF16:
      diloco_outer_kernel<__half><<<grid, 512, 0, s>>>((__half*)param, (__half*)original, (const __half*)grad, mom, n, lr,
                                                       mu, nesterov, alpha, gate);
      break;
    default: throw std::runtime_error("diloco_outer: unsupported dtype");
  }
  TFT_CUDA_CHECK(cudaGetLastError());
}

void sumsq_launch(const void* g, size_t n, float* out, cudaStream_t s) {
  sumsq_kernel<<<grid_for(n / 8 + 1, 512, kNumSMs * 4), 512, 0, s>>>((const bf16*)g, n, out);
  TFT_CUDA_CHECK(cudaGetLastError());
}

void heal_copy_bulk_launch(const void* table_dev, int nentries, size_t total_chunks, size_t chunk_bytes, int blocks,
                           cudaStream_t s) {
  if (total_chunks == 0) return;
  if (chunk_bytes % 16) throw std::runtime_error("heal_copy_bulk: chunk size must be a multiple of 16 bytes");
  static bool configured = false;
  const int smem = kBulkStages * (int)kBulkBytes;
  if (!configured) {
    TFT_CUDA_CHECK(cudaFuncSetAttribute(heal_copy_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  if (blocks < 1) blocks = 1;
  heal_copy_bulk_kernel<<<blocks, 32, smem, s>>>((const CopyEntry*)table_dev, nentries, total_chunks, chunk_bytes);
  TFT_CUDA_CHECK(cudaGetLastError());
}

void heal_copy_launch(const void* table_dev, int nentries, size_t total_chunks, size_t chunk_bytes,
                      int blocks, cudaStream_t s) {
  if (total_chunks == 0) return;
  if (blocks < 1) blocks = 1;
  heal_copy_kernel<<<blocks, 512, 0, s>>>((const CopyEntry*)table_dev, nentries, total_chunks,
                                          chunk_bytes);
  TFT_CUDA_CHECK(cudaGetLastError());
}

}  // namespace tft
