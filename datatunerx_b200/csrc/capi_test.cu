// Test-only C entry points (include/dtxtune_test.h): each casts its pointers, fills the launcher's argument struct and calls the
// internal launcher from kernels.h, so the kernel-level tests exercise exactly what the training step launches.
#include "kernels.h"
#include "../../include/dtxtune_test.h"

using namespace dtx;

namespace {
inline cudaStream_t S(void* s) { return static_cast<cudaStream_t>(s); }
inline int32_t rc(cudaError_t e) { return e == cudaSuccess ? DTX_OK : (e == cudaErrorInvalidValue ? DTX_ERR_INVALID : DTX_ERR_CUDA); }
inline const int32_t* I(const void* p) { return static_cast<const int32_t*>(p); }
inline int32_t* Iw(void* p) { return static_cast<int32_t*>(p); }
inline const bf16* Bf(const void* p) { return static_cast<const bf16*>(p); }
inline bf16* Bw(void* p) { return static_cast<bf16*>(p); }
inline const float* F(const void* p) { return static_cast<const float*>(p); }
inline float* Fw(void* p) { return static_cast<float*>(p); }
}  // namespace

extern "C" {

int32_t dtx_test_attn_fwd(const void* qkv, void* out, void* lse2, int32_t B, int32_t Sq, int32_t H, int32_t Hkv, float scale,
                          const void* seq_lens, int32_t window, const void* row_start, int32_t total_rows, void* stream) {
  AttnArgs a;
  a.qkv = Bf(qkv); a.out = Bw(out); a.lse = Fw(lse2);
  a.B = B; a.S = Sq; a.H = H; a.Hkv = Hkv; a.scale = scale;
  a.seq_lens = I(seq_lens); a.window = window;
  a.row_start = I(row_start); a.total_rows = total_rows;
  return rc(attn_fwd(a, S(stream)));
}

int32_t dtx_test_attn_bwd(const void* qkv, const void* out, const void* dout, const void* lse2, void* delta, void* dqkv, int32_t B,
                          int32_t Sq, int32_t H, int32_t Hkv, float scale, const void* seq_lens, int32_t window, const void* row_start,
                          int32_t total_rows, const void* rope_cs_t, int32_t rope_stride, int32_t rope_glm, void* stream) {
  AttnArgs a;
  a.qkv = Bf(qkv); a.out = const_cast<bf16*>(Bf(out)); a.lse = const_cast<float*>(F(lse2));
  a.dout = Bf(dout); a.delta = Fw(delta); a.dqkv = Bw(dqkv);
  a.B = B; a.S = Sq; a.H = H; a.Hkv = Hkv; a.scale = scale;
  a.seq_lens = I(seq_lens); a.window = window;
  a.row_start = I(row_start); a.total_rows = total_rows;
  a.rope_cs = static_cast<const float2*>(rope_cs_t); a.rope_stride = rope_stride; a.rope_glm = rope_glm;
  return rc(attn_bwd(a, S(stream)));
}

int32_t dtx_test_pack_rows(const void* ids, const void* labels, int32_t S_src, int32_t n, const int32_t* start, void* ids_out,
                           void* labels_out, void* pos_out, void* start_out, void* stream) {
  if (!start || n < 1 || n > 64) return DTX_ERR_INVALID;  // RowStarts holds at most 64 sequences
  RowStarts rs;
  rs.n = n;
  for (int b = 0; b <= n; ++b) rs.start[b] = start[b];
  return rc(pack_rows(I(ids), I(labels), S_src, rs, Iw(ids_out), Iw(labels_out), Iw(pos_out), Iw(start_out), S(stream)));
}

int32_t dtx_test_gather_rows(const void* ids, const void* labels, const void* lens, int32_t S_src, int32_t n, const int32_t* rows,
                             int32_t S_dst, void* ids_out, void* labels_out, void* lens_out, void* stream) {
  if (!rows || n < 1 || n > 64) return DTX_ERR_INVALID;  // RowList holds at most 64 rows
  RowList rl;
  rl.n = n;
  for (int i = 0; i < n; ++i) rl.rows[i] = rows[i];
  return rc(gather_rows(I(ids), I(labels), I(lens), S_src, rl, S_dst, Iw(ids_out), Iw(labels_out), Iw(lens_out), S(stream)));
}

int32_t dtx_test_shift_labels(const void* labels, void* shifted, void* n_valid, int32_t B, int32_t Sq, void* row_map, void* valid_idx,
                              const void* pos, void* stream) {
  return rc(shift_labels(I(labels), Iw(shifted), Iw(n_valid), B, Sq, S(stream), Iw(row_map), Iw(valid_idx), I(pos)));
}

int32_t dtx_test_cross_entropy(const void* logits, int64_t ldl, const void* labels, const void* n_valid, void* row_loss, void* dlogits,
                               int64_t ldd, int32_t M, int32_t V, const void* valid_idx, int32_t n_div, void* stream) {
  return rc(cross_entropy_fwd_bwd(F(logits), ldl, I(labels), I(n_valid), Fw(row_loss), Bw(dlogits), ldd, M, V, S(stream), I(valid_idx),
                                  n_div));
}

int32_t dtx_test_loss_reduce(const void* row_loss, const void* n_valid, void* loss, int32_t M, int32_t n_div, int32_t accumulate,
                             void* stream) {
  return rc(loss_reduce(F(row_loss), I(n_valid), Fw(loss), M, S(stream), n_div, accumulate));
}

int32_t dtx_test_row_loss_stats(const void* row_loss, const void* shifted, int32_t B, int32_t Sq, void* row_sum, void* row_valid,
                                const void* row_start, void* stream) {
  return rc(row_loss_stats(F(row_loss), I(shifted), B, Sq, Fw(row_sum), Iw(row_valid), S(stream), I(row_start)));
}

int32_t dtx_test_rmsnorm_fwd(const void* x, const void* w, void* y, void* rstd, int32_t M, int32_t d, float eps, const void* row_map,
                             void* stream) {
  return rc(rmsnorm_fwd(Bf(x), Bf(w), Bw(y), Fw(rstd), M, d, eps, S(stream), I(row_map)));
}

int32_t dtx_test_rmsnorm_bwd(const void* dy, const void* x, const void* w, const void* rstd, const void* dres, void* dx, int32_t M,
                             int32_t d, const void* row_map, void* stream) {
  return rc(rmsnorm_bwd(Bf(dy), Bf(x), Bf(w), F(rstd), Bf(dres), Bw(dx), M, d, S(stream), I(row_map)));
}

int32_t dtx_test_gemm_m_eff(const void* A, int64_t lda, int32_t a_mn, const void* B, int64_t ldb, int32_t b_mn, void* C, int64_t ldc,
                            int32_t M, int32_t N, int32_t K, int32_t epilogue, int32_t split_k, int32_t block_n, const void* m_eff,
                            void* stream) {
  GemmArgs g;
  g.A = Bf(A); g.lda = lda; g.a_mn_major = a_mn;
  g.B = Bf(B); g.ldb = ldb; g.b_mn_major = b_mn;
  g.C = C; g.ldc = ldc;
  g.M = M; g.N = N; g.K = K; g.epilogue = epilogue; g.split_k = split_k; g.block_n = block_n;
  g.m_eff = I(m_eff);
  return rc(gemm_bf16(g, S(stream)));
}

int32_t dtx_test_swiglu_fwd(const void* gu, void* act, int32_t M, int32_t Fd, int32_t interleaved, void* stream) {
  return rc(swiglu_fwd(Bf(gu), Bw(act), M, Fd, interleaved, S(stream)));
}

int32_t dtx_test_swiglu_bwd(const void* dact, const void* gu, void* dgu, int32_t M, int32_t Fd, int32_t interleaved, void* stream) {
  return rc(swiglu_bwd(Bf(dact), Bf(gu), Bw(dgu), M, Fd, interleaved, S(stream)));
}

int32_t dtx_test_rmsnorm_dw(const void* dy, const void* x, const void* rstd, int32_t M, int32_t d, void* scratch, void* dw,
                            int32_t accumulate, void* stream) {
  return rc(rmsnorm_dw(Bf(dy), Bf(x), F(rstd), M, d, Fw(scratch), Bw(dw), accumulate, S(stream)));
}

int32_t dtx_test_embedding_bwd(const void* ids, const void* dx, void* dE32, int32_t M, int32_t d, int32_t vocab, void* stream) {
  return rc(embedding_bwd(I(ids), Bf(dx), Fw(dE32), M, d, vocab, S(stream)));
}

int32_t dtx_test_sumsq_bf16_acc(const void* g, int64_t n, void* scratch, void* out, int32_t first, void* stream) {
  return rc(sumsq_bf16_acc(Bf(g), n, Fw(scratch), Fw(out), first, S(stream)));
}

int32_t dtx_test_add_f32_into_bf16(const void* src, void* dst, int64_t n, int32_t accumulate, void* stream) {
  return rc(add_f32_into_bf16(F(src), Bw(dst), n, accumulate, S(stream)));
}

int32_t dtx_test_adamw_shard_step(void* master, void* m, void* v, const void* g, void* w, int64_t n, int64_t nodecay_from, float lr,
                                  float beta1, float beta2, float eps, float weight_decay, float bias1, float bias2, float grad_scale,
                                  const void* sumsq, float max_grad_norm, void* grad_norm_out, void* stream) {
  AdamWShardArgs a;
  a.master = Fw(master); a.m = Fw(m); a.v = Fw(v); a.g = Bf(g); a.w = Bw(w); a.n = n; a.nodecay_from = nodecay_from;
  a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.weight_decay = weight_decay; a.bias1 = bias1; a.bias2 = bias2;
  a.grad_scale = grad_scale; a.sumsq = F(sumsq); a.max_grad_norm = max_grad_norm; a.grad_norm_out = Fw(grad_norm_out);
  return rc(adamw_shard_step(a, S(stream)));
}

}  // extern "C"
