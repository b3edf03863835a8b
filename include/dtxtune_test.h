/* libdtxtune — test-only entry points.
 *
 * Thin pass-throughs into internal launchers that the training step runs but the product ABI (dtxtune.h) does not expose:
 * the packed-batch attention arguments, the compact loss path, the lm_head GEMMs' device row count and the full-parameter SFT
 * kernels.  Each one casts its pointers, fills the launcher's argument struct and returns its status; none has logic of its
 * own, so a test of a hook is a test of the kernel.  They are not part of the versioned ABI: names and signatures may change
 * with the kernels.  All pointers are device pointers unless marked host; stream is a cudaStream_t (NULL = default stream).
 */
#ifndef DTXTUNE_TEST_H_
#define DTXTUNE_TEST_H_

#include "dtxtune.h"

#ifdef __cplusplus
extern "C" {
#endif

/* attention with every AttnArgs field the training step sets: row_start (int32 [B+1], NULL = rows of S tokens) with
 * total_rows = row_start[B]; rope_cs_t / rope_stride / rope_glm as in dtx_attn_bwd_rope */
DTX_API int32_t dtx_test_attn_fwd(const void* qkv, void* out, void* lse2, int32_t B, int32_t S, int32_t H, int32_t Hkv, float scale,
                                  const void* seq_lens, int32_t window, const void* row_start, int32_t total_rows, void* stream);
DTX_API int32_t dtx_test_attn_bwd(const void* qkv, const void* out, const void* dout, const void* lse2, void* delta, void* dqkv,
                                  int32_t B, int32_t S, int32_t H, int32_t Hkv, float scale, const void* seq_lens, int32_t window,
                                  const void* row_start, int32_t total_rows, const void* rope_cs_t, int32_t rope_stride,
                                  int32_t rope_glm, void* stream);
/* pack_rows: start (host int32 [n+1], n <= 64) is the RowStarts table; gather_rows: rows (host int32 [n], n <= 64) */
DTX_API int32_t dtx_test_pack_rows(const void* ids, const void* labels, int32_t S_src, int32_t n, const int32_t* start, void* ids_out,
                                   void* labels_out, void* pos_out, void* start_out, void* stream);
DTX_API int32_t dtx_test_gather_rows(const void* ids, const void* labels, const void* lens, int32_t S_src, int32_t n, const int32_t* rows,
                                     int32_t S_dst, void* ids_out, void* labels_out, void* lens_out, void* stream);
/* labels and loss: row_map / valid_idx / pos / dlogits / row_start may be NULL */
DTX_API int32_t dtx_test_shift_labels(const void* labels, void* shifted, void* n_valid, int32_t B, int32_t S, void* row_map,
                                      void* valid_idx, const void* pos, void* stream);
DTX_API int32_t dtx_test_cross_entropy(const void* logits, int64_t ldl, const void* labels, const void* n_valid, void* row_loss,
                                       void* dlogits, int64_t ldd, int32_t M, int32_t V, const void* valid_idx, int32_t n_div,
                                       void* stream);
DTX_API int32_t dtx_test_loss_reduce(const void* row_loss, const void* n_valid, void* loss, int32_t M, int32_t n_div, int32_t accumulate,
                                     void* stream);
DTX_API int32_t dtx_test_row_loss_stats(const void* row_loss, const void* shifted, int32_t B, int32_t S, void* row_sum, void* row_valid,
                                        const void* row_start, void* stream);
/* RMSNorm with a row map (the compacted final norm) */
DTX_API int32_t dtx_test_rmsnorm_fwd(const void* x, const void* w, void* y, void* rstd, int32_t M, int32_t d, float eps,
                                     const void* row_map, void* stream);
DTX_API int32_t dtx_test_rmsnorm_bwd(const void* dy, const void* x, const void* w, const void* rstd, const void* dres, void* dx,
                                     int32_t M, int32_t d, const void* row_map, void* stream);
/* dtx_gemm_bf16 without the K-extension / residual, with a device row count m_eff (int32 [1], may be NULL) */
DTX_API int32_t dtx_test_gemm_m_eff(const void* A, int64_t lda, int32_t a_mn, const void* B, int64_t ldb, int32_t b_mn, void* C,
                                    int64_t ldc, int32_t M, int32_t N, int32_t K, int32_t epilogue, int32_t split_k, int32_t block_n,
                                    const void* m_eff, void* stream);
/* SwiGLU with the layout switch (interleaved = 1: the trainer's GU-interleaved gate|up columns) */
DTX_API int32_t dtx_test_swiglu_fwd(const void* gu, void* act, int32_t M, int32_t F, int32_t interleaved, void* stream);
DTX_API int32_t dtx_test_swiglu_bwd(const void* dact, const void* gu, void* dgu, int32_t M, int32_t F, int32_t interleaved, void* stream);
/* full-parameter SFT; rmsnorm_dw scratch >= 64 * d floats, sumsq_bf16_acc scratch >= 296 floats */
DTX_API int32_t dtx_test_rmsnorm_dw(const void* dy, const void* x, const void* rstd, int32_t M, int32_t d, void* scratch, void* dw,
                                    int32_t accumulate, void* stream);
DTX_API int32_t dtx_test_embedding_bwd(const void* ids, const void* dx, void* dE32, int32_t M, int32_t d, int32_t vocab, void* stream);
DTX_API int32_t dtx_test_sumsq_bf16_acc(const void* g, int64_t n, void* scratch, void* out, int32_t first, void* stream);
DTX_API int32_t dtx_test_add_f32_into_bf16(const void* src, void* dst, int64_t n, int32_t accumulate, void* stream);
DTX_API int32_t dtx_test_adamw_shard_step(void* master, void* m, void* v, const void* g, void* w, int64_t n, int64_t nodecay_from,
                                          float lr, float beta1, float beta2, float eps, float weight_decay, float bias1, float bias2,
                                          float grad_scale, const void* sumsq, float max_grad_norm, void* grad_norm_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DTXTUNE_TEST_H_ */
