// Host-callable launchers of the torchft_b200 data-plane kernels.
// Raw pointers + cudaStream_t only: no torch headers anywhere in this extension.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <utility>

namespace tft {

struct PeerTable;
struct StatusBlock;

// allreduce.cu ---------------------------------------------------------------
// algo: 0 = one-shot, 1 = two-shot. op: 0 sum, 1 max, 2 min. Consumes barrier
// values flag+1 and flag+2 on `channel`.
void allreduce_launch(const PeerTable& pt, StatusBlock* st, size_t off, const void* user_in,
                      void* user_out, size_t nelem, int dtype, int op, float scale,
                      uint64_t flag, int channel, int contribute, int algo, int blocks,
                      int threads, cudaStream_t stream);

// allreduce_nvls.cu ---------------------------------------------------------
void allreduce_nvls_launch(const PeerTable& pt, StatusBlock* st, void* mc_base, size_t off, size_t nelem, int dtype,
                           float scale, uint64_t flag, int channel, int contribute, int blocks, int threads,
                           cudaStream_t stream);

// zero1.cu -------------------------------------------------------------------
// FT-ZeRO-1: one-CTA handshake, sync-free reduce-scatter body (+ buddy push), device-side commit verdict, sync-free
// gated AdamW fused with the all-gather of the new bf16 weights. The argument structs and their fields: zero1.cuh.
namespace zero1 {
struct HsArgs;
struct RSArgs;
struct CommitArgs;
struct UpdArgs;
}  // namespace zero1
void zero1_handshake_launch(const zero1::HsArgs& a, cudaStream_t stream);
void zero1_reduce_launch(zero1::RSArgs a, int acc_mode, int blocks, int threads, cudaStream_t stream);
void zero1_commit_launch(const zero1::CommitArgs& a, cudaStream_t stream);
void zero1_update_launch(zero1::UpdArgs a, int moment_dtype, int blocks, int threads, cudaStream_t stream);

// audit.cu -------------------------------------------------------------------
// FT-ZeRO-1 replica audit: digests of the weights and the held state into each rank's z1_audit slots (table rows:
// audit::DigestEntry), and the one-CTA comparison of every rank's slots that latches kErrDiverged (audit.cuh).
namespace audit {
struct CompareArgs;
}  // namespace audit
void z1_digest_launch(const void* table_dev, int nentries, size_t total_chunks, unsigned long long* slots, int blocks,
                      cudaStream_t stream);
void z1_audit_compare_launch(const audit::CompareArgs& a, cudaStream_t stream);

// collectives.cu --------------------------------------------------------------
// push exchange = all-gather / broadcast / all-to-all over staging slots (arrays have pt.world entries);
// reduce-scatter; point-to-point pieces through per-pair mailboxes.
void push_exchange_launch(const PeerTable& pt, StatusBlock* st, const void* in, void* out, const size_t* send_off,
                          const size_t* send_len, const size_t* recv_len, const size_t* out_off, size_t slot_stride,
                          uint64_t flag, int channel, int blocks, cudaStream_t stream);
void reduce_scatter_launch(const PeerTable& pt, StatusBlock* st, size_t off, const void* user_in, void* out, size_t n,
                           int dtype, int op, float scale, uint64_t flag, int channel, int blocks,
                           cudaStream_t stream);
void p2p_launch(const PeerTable& pt, StatusBlock* st, int is_send, void* buf, size_t nbytes, int peer, size_t mailbox_off,
                size_t mailbox_bytes, uint64_t seq0, int channel, cudaStream_t stream);

// quant.cu -------------------------------------------------------------------
size_t q8_ngroups(size_t nelem, int world);
size_t q8_buffer_bytes(size_t nelem, int world);
void q8_quantize_launch(const void* a, const void* b, size_t nelem, size_t ngroups, int dtype, void* qbuf,
                        cudaStream_t stream);
void q8_dequantize_launch(const void* qbuf, size_t ngroups, void* out, size_t nelem, int dtype, cudaStream_t stream);
void q8_reduce_launch(const void* const* srcs_dev, int nsrc, int first, size_t ngroups, size_t g_lo, size_t g_hi,
                      float post_scale, void* dst, cudaStream_t stream);
void q8_allreduce_launch(const PeerTable& pt, StatusBlock* st, size_t off, const void* in_a,
                         const void* in_b, void* out, size_t nelem, int dtype, float post_scale,
                         uint64_t flag, int channel, int contribute, int blocks, cudaStream_t stream);

size_t q8_slice_buffer_bytes(size_t nelem, int world);
void q8_slice_reduce_launch(const PeerTable& pt, const int* ok, size_t q_off, size_t r_off, size_t nelem, float post_scale,
                            int blocks, cudaStream_t stream);
void q8_gather_dequant_launch(const PeerTable& pt, const int* ok, size_t r_off, size_t nelem, int dtype, void* out, int blocks,
                              cudaStream_t stream);
size_t q8_rs_buffer_bytes(size_t slice_elems, int world);
void q8_reduce_scatter_launch(const PeerTable& pt, StatusBlock* st, size_t off, const void* in, void* out, size_t nelem,
                              size_t slice_elems, int dtype, float post_scale, uint64_t flag, int channel,
                              int contribute, int blocks, cudaStream_t stream);

// model_ops.cu ---------------------------------------------------------------
void rmsnorm_fwd_launch(const void* x, const void* w, void* y, float* rstd, int rows, int H,
                        float eps, cudaStream_t s);
// the same normalisation written as e4m3 y8 [rows, H] with one scale per row (fp8.cuh): fp8_rows(rmsnorm_fwd(x))
void rmsnorm_fwd_fp8_launch(const void* x, const void* w, void* y8, float* yscale, float* rstd, int rows, int H,
                            float eps, cudaStream_t s);
int rmsnorm_bwd_grid(int rows);
void rmsnorm_bwd_launch(const void* dy, const void* x, const void* w, const float* rstd, void* dx,
                        float* dw_partial, void* dw, int accumulate, int rows, int H,
                        cudaStream_t s, const void* dres = nullptr);
void swiglu_fwd_launch(const void* gu, void* y, size_t T, int F, cudaStream_t s);
void swiglu_bwd_launch(const void* dy, const void* gu, void* dgu, size_t T, int F, cudaStream_t s);
void rope_qkv_launch(void* packed, size_t row, void* q, void* k, void* v, const int64_t* strides9, const void* cs,
                     size_t T, int S, int D, int Hq, int Hkv, int dir, cudaStream_t s,
                     const int* positions = nullptr);
void xent_launch(void* logits, const void* target, float* loss, size_t rows, int V,
                 size_t row_stride, float grad_scale, long long ignore_index, cudaStream_t s,
                 const float* scale = nullptr);
// grad[v] += sum of dx[t] over the tokens t with id v, in place, bf16 [V, d], one rounding per touched row, deterministic.
// sorted_ids / perm: a stable sort of the int64 token ids and the token index of each sorted position, [T]; dx: bf16
// [T, d] with row stride ldx; partial: fp32 scratch [embedding_bwd_pieces(T), 2, d]. Two launches.
int embedding_bwd_pieces(int T);
void embedding_bwd_launch(const int64_t* sorted_ids, const int64_t* perm, const void* dx, size_t ldx, void* grad,
                          float* partial, int T, int d, cudaStream_t s);
void adamw_launch(void* p, float* master, float* m, float* v, const void* g, size_t n, float lr,
                  float b1, float b2, float eps, float wd, float bc1, float bc2, float gscale,
                  const int* gate, int max_blocks, cudaStream_t s);
void diloco_outer_launch(void* param, void* original, const void* grad, float* mom, size_t n, int dtype, float lr,
                         float mu, int nesterov, float alpha, const int* gate, cudaStream_t s);
void heal_copy_launch(const void* table_dev, int nentries, size_t total_chunks, size_t chunk_bytes,
                      int blocks, cudaStream_t s);

// fp8.cu ---------------------------------------------------------------------
// Row-scaled e4m3 operands of the fp8 block linears (format in fp8.cuh). fp8_rows: bf16 [rows, C] with row stride ld
// (elements) -> e4m3 [rows, C] + fp32 scale per row. fp8_swiglu: packed gate|up [T, 2F] -> e4m3 silu(g) * u [T, F] +
// scale per row. fp8_cols_t: W [N, K] -> e4m3 W^T [K, N] + scale per column of W; amax_ws is a u32 [K] workspace.
void fp8_rows_launch(const void* x, size_t ld, void* q, float* scale, int rows, int C, cudaStream_t s);
// (chunks of 16 per thread, threads) of the fp8_rows / fp8_swiglu CTA for a row of C elements
std::pair<int, int> fp8_rows_shape(int C);
void fp8_swiglu_launch(const void* gu, void* q, float* scale, int T, int F, cudaStream_t s);
void fp8_cols_t_launch(const void* w, int N, int K, void* q, float* scale, uint32_t* amax_ws, cudaStream_t s);

}  // namespace tft
