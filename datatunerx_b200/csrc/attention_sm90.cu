// Causal flash attention forward / backward for sm_90a, head_dim 128, on wgmma + TMA.
//
// Replaces HF 4.34 eager LlamaAttention (matmul -> mask add -> fp32 softmax -> matmul, SURVEY §2.3 K6,
// reached from cmd/tuning/train.py:299) and its autograd backward (K10).  The [B,H,S,S] score tensor
// never exists: scores are wgmma accumulator fragments, probabilities are converted to bf16 in registers and are the
// REGISTER A operand of the next wgmma.
//
// Data layout: packed qkv [B*S, (H + 2*Hkv)*128] (per token: q heads | k heads | v heads; Hkv <= H for grouped-query
// attention), out [B*S, H*128],
// lse2 [B,H,S] = log2-domain log-sum-exp of the scaled scores (m + log2 l).
//
// Kernels (one CTA per SM, 384 threads): warpgroup 0 is the TMA producer (one thread loads, the warpgroup gives its registers
// away), warpgroups 1 and 2 are consumers that each own 64 rows of the CTA's 128-row tile and stream 64-row blocks:
//   attn_fwd_kernel : CTA = 128 query rows.  S = Q K^T (wgmma 64x64x16, both operands in shared memory), online softmax on the
//                     accumulator fragment, O += P V (P from registers, V as MN-major B), O in registers.
//   attn_dq_kernel  : CTA = 128 query rows.  S, dP = dO V^T, dS = P o (dP - delta) * scale -> register operand, dQ += dS K (K as
//                     MN-major B); delta = rowsum(dO o O) and the inverse rotary of dQ are computed here.
//   attn_dkv_kernel : CTA = 128 KV rows, loops over 64-row Q blocks of every query head of its KV group.  S^T = K Q^T,
//                     dP^T = V dO^T, P^T / dS^T -> register operands, dV += P^T dO, dK += dS^T Q (dO / Q as MN-major B).
// All three take optional true row lengths (tiles that hold only right padding are skipped and written as zeros), an
// optional sliding window (query i sees keys i - window .. i) and an optional table of first rows (PACKED ragged batches:
// sequence b owns rows row_start[b] .. row_start[b+1]) instead of b*S .. (b+1)*S; everything else in the kernels is
// relative to the sequence start, a tile beyond a sequence's rows returns without touching memory).
// Output tiles leave through a swizzled staging tile and TMA stores (the fragment layout gives 4-byte stores otherwise).
// Two backward kernels instead of one with fp32 atomics on dQ: every reduction has a fixed order, so the
// step is bitwise reproducible (needed for the N-rank == 1-rank parity tests).
#include "common.cuh"
#include "kernels.h"

#include <cfloat>
#include <mutex>
#include <type_traits>

namespace dtx {

bool make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner,
                       uint32_t box_outer);

namespace {

constexpr int HD = 128;           // head dim
constexpr int ATT_THREADS = 384;  // producer warpgroup + two consumer warpgroups
constexpr float LOG2E = 1.4426950408889634f;

struct AttnKParams {
  int B, S, H;
  int Hkv, W;        // kv heads (grouped-query attention: q head h reads kv head h / (H / Hkv)); W = row stride of qkv
  int colK0, colV0;  // first column of the k / v sections inside a qkv row
  float scale_log2;  // softmax scale * log2(e)
  float scale;
  float* lse2;
  bf16* out;
  const float* delta;
  float* delta_w;    // attn_dq_kernel writes delta here (same buffer the dK/dV kernel then reads)
  bf16* dqkv;
  const float2* rope_cs;  // backward: transposed rotary table [64][rope_stride] (cos, sin), or null
  int rope_stride;
  const int32_t* seq_lens;  // [B] true row lengths (right padding beyond), or null = S
  int window;               // sliding-window attention: query i sees keys i - window .. i; 0 = plain causal
  const int32_t* row_start; // [B+1] packed ragged batch: sequence b owns rows row_start[b] .. row_start[b+1]) (multiples of 128); null: b*S ..
};

// first row of sequence b and the number of rows it owns (S, or its 128-rounded length in a packed batch)
__device__ __forceinline__ int seq_base(const AttnKParams& p, int b, int* cap) {
  if (p.row_start) {
    const int r0 = p.row_start[b];
    *cap = p.row_start[b + 1] - r0;
    return r0;
  }
  *cap = p.S;
  return b * p.S;
}

// true length of batch row b (tiles that start at or beyond it hold only padding)
__device__ __forceinline__ int row_len(const AttnKParams& p, int b) {
  return p.seq_lens ? min(max(p.seq_lens[b], 0), p.S) : p.S;
}
// zero a [128 x 128] bf16 tile of a row-major matrix (skipped padding tiles: downstream GEMMs contract over tokens, so the
// rows must hold finite values - and the gradient of a padded token is exactly zero)
__device__ __forceinline__ void zero_tile_128(bf16* base, long long ld, long long row0, int col0, int tid, int nthreads) {
  for (int i = tid; i < 128 * 16; i += nthreads)
    *reinterpret_cast<uint4*>(base + (row0 + (i >> 4)) * ld + col0 + (i & 15) * 8) = make_uint4(0u, 0u, 0u, 0u);
}

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// 2^x on the FMA pipe (no MUFU): round-to-nearest split x = n + f via the 1.5 * 2^23 trick, cubic minimax for 2^f on
// [-0.5, 0.5] (max. relative error 7.5e-5, far below bf16 resolution), 2^n added into the exponent field.
// The polynomial's argument is clamped to >= -125 (its value can sit just below 1, i.e. in exponent 126, and the exponent field
// must stay positive after adding n); below the clamp the result is exactly 0, like ex2.approx.ftz's, so that a masked score
// (-inf) gets weight 0 rather than 2^-125.  Callers guarantee x <= ~16.
__device__ __forceinline__ float exp2_fma(float x) {
  const float xc = fmaxf(x, -125.f);
  const float t = xc + 12582912.f;
  const float n = t - 12582912.f;
  const float f = xc - n;
  float q = fmaf(0.055171649903059006f, f, 0.2426111251115799f);
  q = fmaf(q, f, 0.6932609677314758f);
  q = fmaf(q, f, 0.9999280571937561f);
  return x < -125.f ? 0.f : __int_as_float(__float_as_int(q) + (__float_as_int(t) << 23));
}
// exponential of an element of pair number `pair_idx` of a fragment: every FMA_EVERY-th pair on the FMA pipe (0 = none), the
// rest on the MUFU
template <int FMA_EVERY>
__device__ __forceinline__ float exp2_sel(float x, int pair_idx) {
  if constexpr (FMA_EVERY > 0) {
    if ((pair_idx % FMA_EVERY) == FMA_EVERY - 1) return exp2_fma(x);
  }
  return fast_exp2(x);
}

__device__ __forceinline__ void sts32(uint32_t saddr, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(saddr), "r"(v) : "memory"); }
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// 64 x 64 score-shaped fragment (already bf16-rounded values in fp32) -> the four register A operands of the next wgmma
__device__ __forceinline__ void frag_to_a(const float (&s)[32], uint32_t (&a)[4][4]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
#pragma unroll
    for (int i = 0; i < 4; ++i) a[kk][i] = pack_bf16x2(s[8 * kk + 2 * i], s[8 * kk + 2 * i + 1]);
}

// S-shaped product of two K-major operands over the head dim: acc[64 x 64] = A[64 rows of a 128-row tile pair] B[64 x 128]^T.
// a_addr / b_addr: first of the operand's two 64-column subtiles, a_sub / b_sub: bytes between them
__device__ __forceinline__ void mma_qk(float (&acc)[32], uint32_t a_addr, uint32_t a_sub, uint32_t b_addr, uint32_t b_sub) {
#pragma unroll
  for (int k16 = 0; k16 < 8; ++k16)
    wgmma_ss<0, 0>(acc, wgmma_desc_kmajor(a_addr + (k16 >> 2) * a_sub + (k16 & 3) * 32),
                   wgmma_desc_kmajor(b_addr + (k16 >> 2) * b_sub + (k16 & 3) * 32), k16 > 0 ? 1u : 0u);
}
// acc[64 x 128] (+)= A[registers, 64 x 64] B[64 k-rows x 128], B = two [64 x 64] boxes of 8 KB at b_addr (MN-major)
__device__ __forceinline__ void mma_pv(float (&acc)[64], const uint32_t (&a)[4][4], uint32_t b_addr, uint32_t acc0) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) wgmma_rs<1>(acc, a[kk], wgmma_desc_mnmajor(b_addr + kk * 2048, 8192), kk > 0 ? 1u : acc0);
}

// inverse rotary on a 64 x 128 fragment: columns i and i + 64 are o[4 * j + ..] and o[4 * (j + 8) + ..]
__device__ __forceinline__ void rope_inverse_frag(float (&o)[64], const float2* cs, int stride, int pos0, int cq) {
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int hr = 0; hr < 2; ++hr)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float2 t = __ldg(cs + static_cast<size_t>(8 * j + cq + e) * stride + pos0 + 8 * hr);
        const float x0 = o[4 * j + 2 * hr + e], x1 = o[4 * (j + 8) + 2 * hr + e];
        o[4 * j + 2 * hr + e] = x0 * t.x + x1 * t.y;
        o[4 * (j + 8) + 2 * hr + e] = x1 * t.x - x0 * t.y;
      }
}

// GLM's inverse rotary (partial, interleaved) on a 64 x 128 fragment: columns 2i, 2i + 1 (i < 32) are o[4 * j + 2 * hr + 0 / 1]
// with i = 4 * j + cq / 2, from the transposed [32][stride] table; columns 64..127 pass through
__device__ __forceinline__ void rope_glm_inverse_frag(float (&o)[64], const float2* cs, int stride, int pos0, int cq) {
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const float2 t = __ldg(cs + static_cast<size_t>(4 * j + (cq >> 1)) * stride + pos0 + 8 * hr);
      const float x0 = o[4 * j + 2 * hr], x1 = o[4 * j + 2 * hr + 1];
      o[4 * j + 2 * hr] = x0 * t.x + x1 * t.y;
      o[4 * j + 2 * hr + 1] = x1 * t.x - x0 * t.y;
    }
}

// 64 x 128 fragment * mul -> bf16 -> 128B-swizzled staging tile (two 64-column subtiles `sub` bytes apart at `stage`; this
// thread's rows are row0 and row0 + 8 of the tile, the warpgroup's 64 rows start at wg_row0) -> two [64 x 64] TMA stores at
// (grow, gcol) / (grow, gcol + 64) by one thread of the warpgroup (named barrier `bar_id`)
__device__ __forceinline__ void store_frag_tma(const float (&o)[64], float mul0, float mul1, uint8_t* stage, uint32_t sub, int row0, int cq,
                                               int wg_row0, const CUtensorMap* tm, int gcol, int grow, uint32_t bar_id, bool issuer) {
  const uint32_t sa = smem_u32(stage);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    sts32(sa + (j >> 3) * sub + sw128_offset(row0, j & 7) + cq * 2, pack_bf16x2(o[4 * j] * mul0, o[4 * j + 1] * mul0));
    sts32(sa + (j >> 3) * sub + sw128_offset(row0 + 8, j & 7) + cq * 2, pack_bf16x2(o[4 * j + 2] * mul1, o[4 * j + 3] * mul1));
  }
  fence_proxy_async_smem();
  named_bar_sync(bar_id, 128);
  if (issuer) {
    tma_store_2d(tm, stage + wg_row0 * 128, gcol, grow);
    tma_store_2d(tm, stage + sub + wg_row0 * 128, gcol + 64, grow);
    tma_store_commit();
    tma_store_wait_read0();  // the CTA's shared memory must stay valid until the bulk stores have read it
  }
}

// ================================================================================================
// forward
// ================================================================================================
constexpr int FW_NS = 4;                      // K/V ring depth
constexpr int FW_SQ = 0;                      // 2 x [128 x 128B]  (later the output staging tile)
constexpr int FW_SK = 32768;                  // FW_NS x (2 x [64 x 128B])
constexpr int FW_SV = FW_SK + FW_NS * 16384;
constexpr int FW_BAR = FW_SV + FW_NS * 16384;
constexpr int FW_SMEM = FW_BAR + 256 + 1024;

// WIN: sliding-window instantiation (p.window > 0); the plain causal instantiation carries none of the window code.
template <int EXP_FMA_EVERY, bool WIN>  // every N-th pair of exponentials on the FMA pipe instead of the MUFU (0 = none)
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                const __grid_constant__ CUtensorMap tmOut, const AttnKParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + FW_BAR);
  uint64_t *bar_q = bars, *bar_kv = bars + 1 /*[FW_NS]*/, *bar_free = bars + 1 + FW_NS /*[FW_NS]*/;

  const int nqb = p.S / 128;
  const int qb = nqb - 1 - (blockIdx.x % nqb);  // heavy (late) query tiles first
  const int bh = blockIdx.x / nqb;
  const int h = bh % p.H, b = bh / p.H;
  int cap;
  const int row_base = seq_base(p, b, &cap);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  const int hk = h / (p.H / p.Hkv);
  const int colQ = h * HD, colK = p.colK0 + hk * HD, colV = p.colV0 + hk * HD;
  const int q0 = qb * 128;
  if (q0 >= cap) return;  // packed batch: this sequence has no such tile (the rows there belong to the next sequence)
  const int len = min(row_len(p, b), cap);
  // Sliding window: keys before q0 - window are invisible to every row of this CTA: the K/V ring starts at block jlo.  A row may
  // then meet blocks in which it sees nothing (handled by the -inf-safe softmax reference).
  const int window = WIN ? p.window : 0;
  const int jlo = WIN ? max(0, (q0 - window) / 64) : 0;
  const int n = (q0 + 128) / 64 - jlo;
  if (q0 >= len) {  // the tile lies in this row's padding
    zero_tile_128(p.out, static_cast<long long>(p.H) * HD, row_base + q0, h * HD, tid, ATT_THREADS);
    if (p.lse2 && tid < 128) p.lse2[(static_cast<size_t>(b) * p.H + h) * p.S + q0 + tid] = 0.f;
    return;
  }

  if (tid == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmKV);
    tma_prefetch_desc(&tmOut);
    for (int i = 0; i < 1 + FW_NS; ++i) mbar_init(&bars[i], 1);
    for (int i = 0; i < FW_NS; ++i) mbar_init(&bar_free[i], 8);  // lane 0 of every consumer warp
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------ TMA producer ------------------------------------------
    setmaxnreg_dec<40>();
    if (tid == 0) {
      mbar_arrive_expect_tx(bar_q, 32768);
      tma_load_2d(smem + FW_SQ, &tmQ, bar_q, colQ, row_base + q0);
      tma_load_2d(smem + FW_SQ + 16384, &tmQ, bar_q, colQ + 64, row_base + q0);
      for (int j = 0; j < n; ++j) {
        const int slot = j % FW_NS;
        if (j >= FW_NS) mbar_wait_backoff(&bar_free[slot], ((j / FW_NS) - 1) & 1);  // both warpgroups' P V(j - FW_NS) have read the slot
        mbar_arrive_expect_tx(&bar_kv[slot], 32768);
        tma_load_2d(smem + FW_SK + slot * 16384, &tmKV, &bar_kv[slot], colK, row_base + (jlo + j) * 64);
        tma_load_2d(smem + FW_SK + slot * 16384 + 8192, &tmKV, &bar_kv[slot], colK + 64, row_base + (jlo + j) * 64);
        tma_load_2d(smem + FW_SV + slot * 16384, &tmKV, &bar_kv[slot], colV, row_base + (jlo + j) * 64);
        tma_load_2d(smem + FW_SV + slot * 16384 + 8192, &tmKV, &bar_kv[slot], colV + 64, row_base + (jlo + j) * 64);
      }
    }
    return;
  }

  // ------------------------------------------ consumers: 64 query rows each ------------------------------------------
  setmaxnreg_inc<232>();
  const int cw = wg - 1, wq = warp & 3;
  const int rq = lane >> 2, cq = (lane & 3) * 2;
  const int r0 = cw * 64 + wq * 16 + rq;  // this thread's rows of the tile: r0, r0 + 8
  const int qw0 = q0 + cw * 64;           // first query row of the warpgroup
  const uint32_t sq = smem_u32(smem + FW_SQ) + cw * 8192;
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  mbar_wait(bar_q, 0);
  for (int j = 0; j < n; ++j) {
    const int slot = j % FW_NS;
    const int kv0 = (jlo + j) * 64;
    if (kv0 > qw0 + 63) {  // beyond the diagonal for every row of this warpgroup
      if (lane == 0) mbar_arrive(&bar_free[slot]);
      continue;
    }
    mbar_wait(&bar_kv[slot], (j / FW_NS) & 1);
    float s[32];
    wgmma_fence();
    mma_qk(s, sq, 16384, smem_u32(smem + FW_SK + slot * 16384), 8192);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_touch(s);
    const bool diag = kv0 + 63 > qw0;
    const bool wedge = WIN && kv0 < qw0 + 63 - window;  // blocks that straddle the far edge of the window
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int qrow = q0 + r0 + 8 * hr;
      if (diag || wedge) {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int k = kv0 + 8 * jj + cq + e;
            if (k > qrow || (WIN && k < qrow - window)) s[4 * jj + 2 * hr + e] = -INFINITY;
          }
      }
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * hr], s[4 * jj + 2 * hr + 1]));
      mx = quad_max(mx) * p.scale_log2;  // scale > 0: max commutes with the scaling
      const float m_new = fmaxf(m_run[hr], mx);
      // a windowed row that has not met a visible key yet keeps m = -inf: every score is -inf and must give exp2(-inf) = 0, not
      // exp2(-inf + inf) = NaN
      const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
      const float alpha = fast_exp2(m_run[hr] - m_use);
      m_run[hr] = m_new;
      float rs = 0.f;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float pr = exp2_sel<EXP_FMA_EVERY>(fmaf(s[4 * jj + 2 * hr + e], p.scale_log2, -m_use), 2 * jj + hr);
          rs += pr;
          s[4 * jj + 2 * hr + e] = pr;
        }
      l_run[hr] = l_run[hr] * alpha + rs;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        o[4 * jj + 2 * hr] *= alpha;
        o[4 * jj + 2 * hr + 1] *= alpha;
      }
    }
    uint32_t a[4][4];
    frag_to_a(s, a);
    wgmma_fence();
    mma_pv(o, a, smem_u32(smem + FW_SV + slot * 16384), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_touch(o);
    if (lane == 0) mbar_arrive(&bar_free[slot]);
  }
  const float l0 = quad_sum(l_run[0]), l1 = quad_sum(l_run[1]);
  // output tile -> bf16 -> staging tile (this warpgroup's rows of the Q buffer: its S MMAs have completed) -> TMA store
  store_frag_tma(o, 1.f / l0, 1.f / l1, smem + FW_SQ, 16384, r0, cq, cw * 64, &tmOut, h * HD, row_base + qw0, 1 + cw, (tid & 127) == 0);
  if (p.lse2 && (lane & 3) == 0) {
    float* lse = p.lse2 + (static_cast<size_t>(b) * p.H + h) * p.S + q0 + r0;
    lse[0] = m_run[0] + log2f(l0);
    lse[8] = m_run[1] + log2f(l1);
  }
}

// ================================================================================================
// backward: dQ (and delta)
// ================================================================================================
constexpr int DQ_NS = 3;
constexpr int DQ_SQ = 0;                       // 2 x [128 x 128B]  (TMA landing zone, later the dQ staging tile)
constexpr int DQ_SDO = 32768;                  // 2 x [128 x 128B]
constexpr int DQ_SO = 65536;                   // 2 x [128 x 128B]  forward output tile, only for delta = rowsum(dO o O)
constexpr int DQ_SK = 98304;                   // DQ_NS x (2 x [64 x 128B])
constexpr int DQ_SV = DQ_SK + DQ_NS * 16384;
constexpr int DQ_BAR = DQ_SV + DQ_NS * 16384;
constexpr int DQ_XD = DQ_BAR + 256;            // [128] delta of the tile's rows
constexpr int DQ_SMEM = DQ_XD + 512 + 1024;

// WIN: see attn_fwd_kernel.  EXP_FMA: every N-th pair of exponentials on the FMA pipe (A/B switch "attn_dq_exp_fma_every").
// GLM: the inverse rotary of dQ is GLM's (rope_glm_inverse_frag, [32][rope_stride] table).
template <bool WIN, int EXP_FMA, bool GLM = false>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
               const __grid_constant__ CUtensorMap tmDO, const __grid_constant__ CUtensorMap tmO,
               const __grid_constant__ CUtensorMap tmOut, const AttnKParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + DQ_BAR);
  uint64_t *bar_q = bars, *bar_kv = bars + 1 /*[DQ_NS]*/, *bar_free = bars + 1 + DQ_NS /*[DQ_NS]*/;

  const int nqb = p.S / 128;
  const int qb = nqb - 1 - (blockIdx.x % nqb);  // heavy (late) query tiles first
  const int bh = blockIdx.x / nqb;
  const int h = bh % p.H, b = bh / p.H;
  const int q0 = qb * 128;
  int cap;
  const int row_base = seq_base(p, b, &cap);
  if (q0 >= cap) return;  // packed batch: not a tile of this sequence
  const int window = WIN ? p.window : 0;
  const int jlo = WIN ? max(0, (q0 - window) / 64) : 0;  // sliding window: first K/V block any row of the tile can see
  const int n = (q0 + 128) / 64 - jlo;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  const int hk = h / (p.H / p.Hkv);
  const int colQ = h * HD, colK = p.colK0 + hk * HD, colV = p.colV0 + hk * HD;
  if (q0 >= min(row_len(p, b), cap)) {  // the tile holds only padding: dQ = 0, delta = 0
    zero_tile_128(p.dqkv, p.W, row_base + q0, colQ, tid, ATT_THREADS);
    if (tid < 128) p.delta_w[(static_cast<size_t>(b) * p.H + h) * p.S + q0 + tid] = 0.f;
    return;
  }

  if (tid == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmKV);
    tma_prefetch_desc(&tmDO);
    tma_prefetch_desc(&tmO);
    tma_prefetch_desc(&tmOut);
    for (int i = 0; i < 1 + DQ_NS; ++i) mbar_init(&bars[i], 1);
    for (int i = 0; i < DQ_NS; ++i) mbar_init(&bar_free[i], 8);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------ TMA producer ------------------------------------------
    setmaxnreg_dec<40>();
    if (tid == 0) {
      mbar_arrive_expect_tx(bar_q, 98304);
      tma_load_2d(smem + DQ_SQ, &tmQ, bar_q, colQ, row_base + q0);
      tma_load_2d(smem + DQ_SQ + 16384, &tmQ, bar_q, colQ + 64, row_base + q0);
      tma_load_2d(smem + DQ_SDO, &tmDO, bar_q, h * HD, row_base + q0);
      tma_load_2d(smem + DQ_SDO + 16384, &tmDO, bar_q, h * HD + 64, row_base + q0);
      tma_load_2d(smem + DQ_SO, &tmO, bar_q, h * HD, row_base + q0);
      tma_load_2d(smem + DQ_SO + 16384, &tmO, bar_q, h * HD + 64, row_base + q0);
      for (int j = 0; j < n; ++j) {
        const int slot = j % DQ_NS;
        if (j >= DQ_NS) mbar_wait_backoff(&bar_free[slot], ((j / DQ_NS) - 1) & 1);  // dQ MMAs of block j - DQ_NS have read the slot
        mbar_arrive_expect_tx(&bar_kv[slot], 32768);
        tma_load_2d(smem + DQ_SK + slot * 16384, &tmKV, &bar_kv[slot], colK, row_base + (jlo + j) * 64);
        tma_load_2d(smem + DQ_SK + slot * 16384 + 8192, &tmKV, &bar_kv[slot], colK + 64, row_base + (jlo + j) * 64);
        tma_load_2d(smem + DQ_SV + slot * 16384, &tmKV, &bar_kv[slot], colV, row_base + (jlo + j) * 64);
        tma_load_2d(smem + DQ_SV + slot * 16384 + 8192, &tmKV, &bar_kv[slot], colV + 64, row_base + (jlo + j) * 64);
      }
    }
    return;
  }

  // ------------------------------------------ consumers: 64 query rows each ------------------------------------------
  setmaxnreg_inc<232>();
  const int cw = wg - 1, wq = warp & 3;
  const int rq = lane >> 2, cq = (lane & 3) * 2;
  const int r0 = cw * 64 + wq * 16 + rq;
  const int qw0 = q0 + cw * 64;
  const size_t stat0 = (static_cast<size_t>(b) * p.H + h) * p.S + q0;
  float* xd = reinterpret_cast<float*>(smem + DQ_XD);
  mbar_wait(bar_q, 0);
  {  // delta = rowsum(dO o O): thread pair (2r, 2r + 1) of the warpgroup takes the two 64-column halves of row r; published for
     // the dK/dV kernel
    const int t = tid & 127, rl = cw * 64 + (t >> 1), half = t & 1;
    const uint32_t sdo = smem_u32(smem + DQ_SDO) + half * 16384, so = smem_u32(smem + DQ_SO) + half * 16384;
    float part = 0.f;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const uint4 x = lds128u(so + sw128_offset(rl, c)), y = lds128u(sdo + sw128_offset(rl, c));
      const uint32_t ow[4] = {x.x, x.y, x.z, x.w}, dw[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 o2 = unpack_bf16x2(ow[i]), d2 = unpack_bf16x2(dw[i]);
        part = fmaf(o2.x, d2.x, part);
        part = fmaf(o2.y, d2.y, part);
      }
    }
    part += __shfl_xor_sync(0xffffffffu, part, 1);
    if (half == 0) {
      xd[rl] = part;
      p.delta_w[stat0 + rl] = part;
    }
    named_bar_sync(1 + cw, 128);
  }
  const float nds[2] = {-xd[r0] * p.scale, -xd[r0 + 8] * p.scale};
  const float nl[2] = {-p.lse2[stat0 + r0], -p.lse2[stat0 + r0 + 8]};
  const uint32_t sq = smem_u32(smem + DQ_SQ) + cw * 8192, sdo = smem_u32(smem + DQ_SDO) + cw * 8192;
  float dq[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) dq[i] = 0.f;
  for (int j = 0; j < n; ++j) {
    const int slot = j % DQ_NS;
    const int kv0 = (jlo + j) * 64;
    if (kv0 > qw0 + 63) {  // beyond the diagonal for every row of this warpgroup
      if (lane == 0) mbar_arrive(&bar_free[slot]);
      continue;
    }
    mbar_wait(&bar_kv[slot], (j / DQ_NS) & 1);
    float s[32], dp[32];
    wgmma_fence();
    mma_qk(s, sq, 16384, smem_u32(smem + DQ_SK + slot * 16384), 8192);
    mma_qk(dp, sdo, 16384, smem_u32(smem + DQ_SV + slot * 16384), 8192);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_touch(s);
    wgmma_touch(dp);
    const bool need_mask = (kv0 + 63 > qw0) || (WIN && kv0 < qw0 + 63 - window);
    // dS = P o (dP * scale - delta * scale), P = 2^(S * scale_log2 - lse2)
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int qrow = q0 + r0 + 8 * hr;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int i = 4 * jj + 2 * hr + e;
          float pr = exp2_sel<EXP_FMA>(fmaf(s[i], p.scale_log2, nl[hr]), 2 * jj + hr);
          if (need_mask) {
            const int k = kv0 + 8 * jj + cq + e;
            if (k > qrow || (WIN && k < qrow - window)) pr = 0.f;
          }
          s[i] = pr * fmaf(dp[i], p.scale, nds[hr]);
        }
    }
    uint32_t a[4][4];
    frag_to_a(s, a);
    wgmma_fence();
    mma_pv(dq, a, smem_u32(smem + DQ_SK + slot * 16384), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_touch(dq);
    if (lane == 0) mbar_arrive(&bar_free[slot]);
  }
  if (p.rope_cs) {
    if (GLM) rope_glm_inverse_frag(dq, p.rope_cs, p.rope_stride, q0 + r0, cq);
    else rope_inverse_frag(dq, p.rope_cs, p.rope_stride, q0 + r0, cq);
  }
  // dQ tile -> bf16 -> staging tile (this warpgroup's rows of the Q landing zone) -> TMA store
  store_frag_tma(dq, 1.f, 1.f, smem + DQ_SQ, 16384, r0, cq, cw * 64, &tmOut, colQ, row_base + qw0, 1 + cw, (tid & 127) == 0);
}

// ================================================================================================
// backward: dK, dV
// ================================================================================================
constexpr int DKV_NS = 4;                      // Q / dO ring depth
constexpr int DKV_SK = 0;                      // 2 x [128 x 128B]  (later the dK staging tile)
constexpr int DKV_SV = 32768;                  // 2 x [128 x 128B]  (later the dV staging tile)
constexpr int DKV_SQ = 65536;                  // DKV_NS x (2 x [64 x 128B])
constexpr int DKV_SDO = DKV_SQ + DKV_NS * 16384;    // DKV_NS x (2 x [64 x 128B])
constexpr int DKV_STAT = DKV_SDO + DKV_NS * 16384;  // DKV_NS x (lse2[64], delta[64]) fp32, filled by bulk copies with the Q ring
constexpr int DKV_BAR = DKV_STAT + DKV_NS * 512;
constexpr int DKV_SMEM = DKV_BAR + 256 + 1024;

template <bool WIN, bool GLM = false>  // GLM: see attn_dq_kernel
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_dkv_kernel(const __grid_constant__ CUtensorMap tmKV128, const __grid_constant__ CUtensorMap tmQ64,
                const __grid_constant__ CUtensorMap tmDO64, const __grid_constant__ CUtensorMap tmOut, const AttnKParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + DKV_BAR);
  uint64_t *bar_kv = bars, *bar_q = bars + 1 /*[DKV_NS]*/, *bar_free = bars + 1 + DKV_NS /*[DKV_NS]*/;

  const int nkb = p.S / 128;
  const int kb = blockIdx.x % nkb;  // early KV blocks see the most query blocks: they come first
  const int bh = blockIdx.x / nkb;
  const int hk = bh % p.Hkv, b = bh / p.Hkv;  // one CTA per (batch, KV head, 128-row KV block)
  const int grp = p.H / p.Hkv;                // query heads sharing this KV head (1 = multi-head attention)
  const int kv0 = kb * 128;
  int cap;
  const int row_base = seq_base(p, b, &cap);
  if (kv0 >= cap) return;  // packed batch: not a tile of this sequence
  const int i0 = kv0 / 64;
  const int len = min(row_len(p, b), cap);
  // query blocks per query head that see this KV block and hold a real token; with a sliding window the last query row that
  // sees any key of the tile is kv0 + 127 + window
  const int window = WIN ? p.window : 0;
  const int q_end = WIN ? min((len + 63) / 64, (kv0 + 127 + window) / 64 + 1) : (len + 63) / 64;
  const int nq = q_end - i0;
  const int n = nq * grp;                     // streamed (head, query block) pairs; it -> head it / nq, block it % nq
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  const int colK = p.colK0 + hk * HD, colV = p.colV0 + hk * HD;
  const float* g_lse = p.lse2 + (static_cast<size_t>(b) * p.H + hk * grp) * p.S;
  const float* g_delta = p.delta + (static_cast<size_t>(b) * p.H + hk * grp) * p.S;
  if (kv0 >= len) {  // the KV tile holds only padding: dK = dV = 0
    zero_tile_128(p.dqkv, p.W, row_base + kv0, colK, tid, ATT_THREADS);
    zero_tile_128(p.dqkv, p.W, row_base + kv0, colV, tid, ATT_THREADS);
    return;
  }

  if (tid == 0) {
    tma_prefetch_desc(&tmKV128);
    tma_prefetch_desc(&tmQ64);
    tma_prefetch_desc(&tmDO64);
    tma_prefetch_desc(&tmOut);
    for (int i = 0; i < 1 + DKV_NS; ++i) mbar_init(&bars[i], 1);
    for (int i = 0; i < DKV_NS; ++i) mbar_init(&bar_free[i], 8);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------ TMA producer ------------------------------------------
    setmaxnreg_dec<40>();
    if (tid == 0) {
      mbar_arrive_expect_tx(bar_kv, 65536);
      tma_load_2d(smem + DKV_SK, &tmKV128, bar_kv, colK, row_base + kv0);
      tma_load_2d(smem + DKV_SK + 16384, &tmKV128, bar_kv, colK + 64, row_base + kv0);
      tma_load_2d(smem + DKV_SV, &tmKV128, bar_kv, colV, row_base + kv0);
      tma_load_2d(smem + DKV_SV + 16384, &tmKV128, bar_kv, colV + 64, row_base + kv0);
      int hq = 0, qi = 0;  // (query head of the group, query block) of pair ii
      for (int ii = 0; ii < n; ++ii) {
        const int slot = ii % DKV_NS;
        if (ii >= DKV_NS) mbar_wait_backoff(&bar_free[slot], ((ii / DKV_NS) - 1) & 1);  // dV/dK MMAs of pair ii - DKV_NS have read the slot
        const int qs = (i0 + qi) * 64, colQ = (hk * grp + hq) * HD;
        mbar_arrive_expect_tx(&bar_q[slot], 32768 + 512);
        tma_load_2d(smem + DKV_SQ + slot * 16384, &tmQ64, &bar_q[slot], colQ, row_base + qs);
        tma_load_2d(smem + DKV_SQ + slot * 16384 + 8192, &tmQ64, &bar_q[slot], colQ + 64, row_base + qs);
        tma_load_2d(smem + DKV_SDO + slot * 16384, &tmDO64, &bar_q[slot], colQ, row_base + qs);
        tma_load_2d(smem + DKV_SDO + slot * 16384 + 8192, &tmDO64, &bar_q[slot], colQ + 64, row_base + qs);
        tma_load_1d(smem + DKV_STAT + slot * 512, g_lse + static_cast<size_t>(hq) * p.S + qs, 256, &bar_q[slot]);
        tma_load_1d(smem + DKV_STAT + slot * 512 + 256, g_delta + static_cast<size_t>(hq) * p.S + qs, 256, &bar_q[slot]);
        if (++qi == nq) { qi = 0; ++hq; }
      }
    }
    return;
  }

  // ------------------------------------------ consumers: 64 KV rows each ------------------------------------------
  setmaxnreg_inc<232>();
  const int cw = wg - 1, wq = warp & 3;
  const int rq = lane >> 2, cq = (lane & 3) * 2;
  const int r0 = cw * 64 + wq * 16 + rq;
  const int kw0 = kv0 + cw * 64;  // first KV row of the warpgroup
  const uint32_t sk = smem_u32(smem + DKV_SK) + cw * 8192, sv = smem_u32(smem + DKV_SV) + cw * 8192;
  float dk[64], dv[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) dk[i] = dv[i] = 0.f;
  mbar_wait(bar_kv, 0);
  int qi = 0;
  for (int ii = 0; ii < n; ++ii) {
    const int slot = ii % DKV_NS;
    const int qs = (i0 + qi) * 64;
    if (++qi == nq) qi = 0;
    if (qs + 63 < kw0 || (WIN && qs > kw0 + 63 + window)) {  // no query of the block sees a key of this warpgroup
      // Wait for the pair's loads all the same: the producer re-arms the slot once all eight warps have released it, so a
      // warpgroup that released skipped pairs without waiting could also release the slot's next use (warpgroup 1 skips the
      // first query block of every head of the group) and the producer would re-arm bar_q while those loads are in flight.
      // A plain spin: the watchdog's trap path here makes ptxas move the dK / dV accumulators to the stack.  It cannot hang on
      // its own - the producer issues pair ii as soon as every warp has released pair ii - DKV_NS.
      while (!mbar_try_wait(&bar_q[slot], (ii / DKV_NS) & 1)) {}
      if (lane == 0) mbar_arrive(&bar_free[slot]);
      continue;
    }
    mbar_wait(&bar_q[slot], (ii / DKV_NS) & 1);
    float s[32], dp[32];
    wgmma_fence();
    mma_qk(s, sk, 16384, smem_u32(smem + DKV_SQ + slot * 16384), 8192);
    mma_qk(dp, sv, 16384, smem_u32(smem + DKV_SDO + slot * 16384), 8192);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_touch(s);
    wgmma_touch(dp);
    const float* st = reinterpret_cast<const float*>(smem + DKV_STAT + slot * 512);
    const bool need_mask = (qs < kw0 + 63) || (WIN && qs + 63 > kw0 + window);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const float2 l2 = *reinterpret_cast<const float2*>(st + 8 * jj + cq), d2 = *reinterpret_cast<const float2*>(st + 64 + 8 * jj + cq);
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int kvrow = kv0 + r0 + 8 * hr;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int i = 4 * jj + 2 * hr + e;
          float pr = fast_exp2(fmaf(s[i], p.scale_log2, e ? -l2.y : -l2.x));
          if (need_mask) {
            const int q = qs + 8 * jj + cq + e;  // visible iff kvrow <= q <= kvrow + window
            if (kvrow > q || (WIN && q > kvrow + window)) pr = 0.f;
          }
          s[i] = pr;
          dp[i] = pr * (dp[i] - (e ? d2.y : d2.x)) * p.scale;
        }
      }
    }
    uint32_t a[4][4];
    frag_to_a(s, a);
    wgmma_fence();
    mma_pv(dv, a, smem_u32(smem + DKV_SDO + slot * 16384), 1u);
    frag_to_a(dp, a);
    mma_pv(dk, a, smem_u32(smem + DKV_SQ + slot * 16384), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_touch(dv);
    wgmma_touch(dk);
    if (lane == 0) mbar_arrive(&bar_free[slot]);
  }
  // dV, dK (with the inverse rotary) -> bf16 -> staging tiles (this warpgroup's rows of the V / K tiles) -> TMA stores
  store_frag_tma(dv, 1.f, 1.f, smem + DKV_SV, 16384, r0, cq, cw * 64, &tmOut, colV, row_base + kw0, 1 + cw, (tid & 127) == 0);
  if (p.rope_cs) {
    if (GLM) rope_glm_inverse_frag(dk, p.rope_cs, p.rope_stride, kv0 + r0, cq);
    else rope_inverse_frag(dk, p.rope_cs, p.rope_stride, kv0 + r0, cq);
  }
  store_frag_tma(dk, 1.f, 1.f, smem + DKV_SK, 16384, r0, cq, cw * 64, &tmOut, colK, row_base + kw0, 1 + cw, (tid & 127) == 0);
}

cudaError_t set_smem(const void* fn, int bytes) {
  return cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
}

}  // namespace

// every N-th pair of exponentials on the FMA pipe: off by default in both kernels (not measured on H100)
int g_fwd_exp_fma_every = 0;
int g_dq_exp_fma_every = 0;
void attn_set_dq_exp_fma_every(int n) { g_dq_exp_fma_every = (n == 3 || n == 4) ? n : 0; }
void attn_set_fwd_exp_fma_every(int n) { g_fwd_exp_fma_every = (n == 2 || n == 3 || n == 4) ? n : 0; }  // 0 = all on the MUFU
int attn_bwd_launches() { return 2; }
bool attn_bwd_can_rope() { return true; }

namespace {
// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device property of a function: set it once per device
cudaError_t attn_init_device() {
  static std::mutex mu;
  static bool done[64] = {false};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lk(mu);
  if (dev >= 0 && dev < 64 && done[dev]) return cudaSuccess;
  const void* fwd[] = {reinterpret_cast<const void*>(attn_fwd_kernel<0, false>), reinterpret_cast<const void*>(attn_fwd_kernel<2, false>),
                       reinterpret_cast<const void*>(attn_fwd_kernel<3, false>), reinterpret_cast<const void*>(attn_fwd_kernel<4, false>),
                       reinterpret_cast<const void*>(attn_fwd_kernel<0, true>), reinterpret_cast<const void*>(attn_fwd_kernel<2, true>),
                       reinterpret_cast<const void*>(attn_fwd_kernel<3, true>), reinterpret_cast<const void*>(attn_fwd_kernel<4, true>)};
  for (const void* f : fwd)
    if ((e = set_smem(f, FW_SMEM)) != cudaSuccess) return e;
  const void* dq[] = {reinterpret_cast<const void*>(attn_dq_kernel<false, 0>), reinterpret_cast<const void*>(attn_dq_kernel<false, 3>),
                      reinterpret_cast<const void*>(attn_dq_kernel<false, 4>), reinterpret_cast<const void*>(attn_dq_kernel<true, 0>),
                      reinterpret_cast<const void*>(attn_dq_kernel<true, 3>), reinterpret_cast<const void*>(attn_dq_kernel<true, 4>)};
  for (const void* f : dq)
    if ((e = set_smem(f, DQ_SMEM)) != cudaSuccess) return e;
  if ((e = set_smem(reinterpret_cast<const void*>(attn_dkv_kernel<false>), DKV_SMEM)) != cudaSuccess) return e;
  if ((e = set_smem(reinterpret_cast<const void*>(attn_dkv_kernel<true>), DKV_SMEM)) != cudaSuccess) return e;
  const void* glm[] = {reinterpret_cast<const void*>(attn_dq_kernel<false, 0, true>), reinterpret_cast<const void*>(attn_dq_kernel<false, 3, true>),
                       reinterpret_cast<const void*>(attn_dq_kernel<false, 4, true>)};
  for (const void* f : glm)
    if ((e = set_smem(f, DQ_SMEM)) != cudaSuccess) return e;
  if ((e = set_smem(reinterpret_cast<const void*>(attn_dkv_kernel<false, true>), DKV_SMEM)) != cudaSuccess) return e;
  if (dev >= 0 && dev < 64) done[dev] = true;
  return cudaSuccess;
}
bool aligned16(const void* ptr) { return ptr && (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; }

// The argument rules of AttnArgs, checked on the host before any CUDA call.  Returns the window the kernels run with: a window
// of S - 1 or more hides no key (query i <= S - 1 sees keys from i - window <= 0), so it runs as plain causal attention (0),
// which also keeps kv0 + window and friends in the kernels far from int overflow.  -1 = refused.
int attn_validate(const AttnArgs& a, bool bwd) {
  if (a.S <= 0 || a.S % 128 || a.B <= 0 || a.H <= 0 || a.Hkv < 0 || a.window < 0) return -1;
  if (a.H % (a.Hkv > 0 ? a.Hkv : a.H)) return -1;
  if (!(a.scale > 0.f && a.scale <= FLT_MAX)) return -1;  // the forward's row max commutes with the scaling only for scale > 0
  if (a.row_start && (a.total_rows <= 0 || a.total_rows % 128)) return -1;
  if (!aligned16(a.qkv) || !aligned16(a.out)) return -1;  // TMA bases
  const int window = a.window >= a.S - 1 ? 0 : a.window;
  if (!bwd) return window;
  if (!aligned16(a.dout) || !aligned16(a.dqkv) || !aligned16(a.lse) || !aligned16(a.delta)) return -1;
  // GLM's inverse rotary is instantiated for plain causal attention (GLM has no sliding window)
  if (a.rope_glm != 0 && (a.rope_glm != 1 || window > 0)) return -1;
  // the inverse rotary reads the table at freq * rope_stride + pos for pos up to S - 1
  if (a.rope_cs && a.rope_stride > 0 && a.rope_stride < a.S) return -1;
  return window;
}
}  // namespace

cudaError_t attn_fwd(const AttnArgs& a, cudaStream_t s) {
  const int window = attn_validate(a, false);
  if (window < 0) return cudaErrorInvalidValue;
  cudaError_t e = attn_init_device();
  if (e != cudaSuccess) return e;
  const int Hkv = a.Hkv > 0 ? a.Hkv : a.H;
  const uint64_t M = a.row_start ? static_cast<uint64_t>(a.total_rows) : static_cast<uint64_t>(a.B) * a.S, W = static_cast<uint64_t>(a.H + 2 * Hkv) * HD;
  CUtensorMap tmQ, tmKV, tmOut;
  const uint64_t WO = static_cast<uint64_t>(a.H) * HD;
  if (!make_tmap_2d_bf16(&tmQ, a.qkv, W, M, W, 64, 128) || !make_tmap_2d_bf16(&tmKV, a.qkv, W, M, W, 64, 64) ||
      !make_tmap_2d_bf16(&tmOut, a.out, WO, M, WO, 64, 64))
    return cudaErrorInvalidValue;
  AttnKParams p{};
  p.B = a.B; p.S = a.S; p.H = a.H;
  p.Hkv = Hkv; p.W = static_cast<int>(W); p.colK0 = a.H * HD; p.colV0 = (a.H + Hkv) * HD;
  p.scale = a.scale;
  p.scale_log2 = a.scale * LOG2E;
  p.lse2 = a.lse;
  p.out = a.out;
  p.seq_lens = a.seq_lens;
  p.window = window;
  p.row_start = a.row_start;
  const int grid = a.B * a.H * (a.S / 128);
#define DTX_FWD_LAUNCH(E)                                                                          \
  if (window > 0) attn_fwd_kernel<E, true><<<grid, ATT_THREADS, FW_SMEM, s>>>(tmQ, tmKV, tmOut, p); \
  else attn_fwd_kernel<E, false><<<grid, ATT_THREADS, FW_SMEM, s>>>(tmQ, tmKV, tmOut, p)
  switch (g_fwd_exp_fma_every) {
    case 2: DTX_FWD_LAUNCH(2); break;
    case 3: DTX_FWD_LAUNCH(3); break;
    case 4: DTX_FWD_LAUNCH(4); break;
    default: DTX_FWD_LAUNCH(0); break;
  }
#undef DTX_FWD_LAUNCH
  return cudaGetLastError();
}

cudaError_t attn_bwd(const AttnArgs& a, cudaStream_t s) {
  const int window = attn_validate(a, true);
  if (window < 0) return cudaErrorInvalidValue;
  cudaError_t e = attn_init_device();
  if (e != cudaSuccess) return e;
  const int Hkv = a.Hkv > 0 ? a.Hkv : a.H;
  const uint64_t M = a.row_start ? static_cast<uint64_t>(a.total_rows) : static_cast<uint64_t>(a.B) * a.S, W = static_cast<uint64_t>(a.H + 2 * Hkv) * HD,
                 WO = static_cast<uint64_t>(a.H) * HD;
  CUtensorMap tmQ128, tmKV64, tmDO128, tmDO64, tmDqkv64, tmO128;
  if (!make_tmap_2d_bf16(&tmO128, a.out, WO, M, WO, 64, 128)) return cudaErrorInvalidValue;
  bool ok = make_tmap_2d_bf16(&tmQ128, a.qkv, W, M, W, 64, 128) && make_tmap_2d_bf16(&tmKV64, a.qkv, W, M, W, 64, 64) &&
            make_tmap_2d_bf16(&tmDqkv64, a.dqkv, W, M, W, 64, 64) &&
            make_tmap_2d_bf16(&tmDO128, a.dout, WO, M, WO, 64, 128) && make_tmap_2d_bf16(&tmDO64, a.dout, WO, M, WO, 64, 64);
  if (!ok) return cudaErrorInvalidValue;
  AttnKParams p{};
  p.B = a.B; p.S = a.S; p.H = a.H;
  p.Hkv = Hkv; p.W = static_cast<int>(W); p.colK0 = a.H * HD; p.colV0 = (a.H + Hkv) * HD;
  p.scale = a.scale;
  p.scale_log2 = a.scale * LOG2E;
  p.lse2 = a.lse;
  p.out = a.out;
  p.delta = a.delta;
  p.delta_w = a.delta;
  p.dqkv = a.dqkv;
  p.rope_cs = a.rope_cs;
  p.rope_stride = a.rope_stride > 0 ? a.rope_stride : a.S;
  p.seq_lens = a.seq_lens;
  p.window = window;
  p.row_start = a.row_start;
  const int gq = a.B * a.H * (a.S / 128), gkv = a.B * Hkv * (a.S / 128);
  const bool win = window > 0;
  if (a.rope_glm && a.rope_cs) {
#define DTX_DQ_GLM_LAUNCH(I) attn_dq_kernel<false, I, true><<<gq, ATT_THREADS, DQ_SMEM, s>>>(tmQ128, tmKV64, tmDO128, tmO128, tmDqkv64, p)
    if (g_dq_exp_fma_every == 3) DTX_DQ_GLM_LAUNCH(3); else if (g_dq_exp_fma_every == 4) DTX_DQ_GLM_LAUNCH(4); else DTX_DQ_GLM_LAUNCH(0);
#undef DTX_DQ_GLM_LAUNCH
    attn_dkv_kernel<false, true><<<gkv, ATT_THREADS, DKV_SMEM, s>>>(tmQ128, tmKV64, tmDO64, tmDqkv64, p);
    return cudaGetLastError();
  }
#define DTX_DQ_LAUNCH(W, I) attn_dq_kernel<W, I><<<gq, ATT_THREADS, DQ_SMEM, s>>>(tmQ128, tmKV64, tmDO128, tmO128, tmDqkv64, p)
  if (win) { if (g_dq_exp_fma_every == 3) DTX_DQ_LAUNCH(true, 3); else if (g_dq_exp_fma_every == 4) DTX_DQ_LAUNCH(true, 4); else DTX_DQ_LAUNCH(true, 0); }
  else { if (g_dq_exp_fma_every == 3) DTX_DQ_LAUNCH(false, 3); else if (g_dq_exp_fma_every == 4) DTX_DQ_LAUNCH(false, 4); else DTX_DQ_LAUNCH(false, 0); }
#undef DTX_DQ_LAUNCH
  if (win) attn_dkv_kernel<true><<<gkv, ATT_THREADS, DKV_SMEM, s>>>(tmQ128, tmKV64, tmDO64, tmDqkv64, p);
  else attn_dkv_kernel<false><<<gkv, ATT_THREADS, DKV_SMEM, s>>>(tmQ128, tmKV64, tmDO64, tmDqkv64, p);
  return cudaGetLastError();
}

}  // namespace dtx
