// wgmma / TMA bf16 GEMM for sm_90a — the contraction engine of the LoRA-SFT step.
//
// Replaces the cuBLAS hgemm calls hidden behind nn.Linear / peft lora.Linear on the reference's hot
// path (SURVEY §2.3 K3,K4,K7,K8,K10; call sites cmd/tuning/train.py:236-242,268-280,299).
//
// Structure (one CTA per SM, persistent over 128 x BN output tiles, three warpgroups = 384 threads):
//   warpgroup 0     TMA producer : one elected thread issues cp.async.bulk.tensor loads of A/B k-blocks into a STAGES-deep
//                                  shared-memory ring; the warpgroup hands its registers to the consumers (setmaxnreg)
//   warpgroups 1, 2 consumers    : each owns 64 rows of the tile, issues wgmma.mma_async (64 x BN x 16 per instruction) on the
//                                  ring slots and keeps its 64 x BN fp32 accumulator in registers; the epilogue (convert /
//                                  +residual / rotary / SwiGLU) runs on those registers
// Epilogue: each consumer warpgroup owns a 16 KB staging half (two 64-row x 128-byte boxes, 128B swizzle, the TMA layout) and
// emits its slice of the tile in passes of two boxes: registers -> st.shared -> cp.async.bulk.tensor store. It then goes
// straight on to the next tile's main loop while the stores drain; before it writes the staging half again it waits until the
// previous bulk stores have read it. Epilogue inputs (the residual of EPI_BF16_ADD, gu of EPI_SWIGLU_BWD) are TMA-loaded into
// the same staging boxes and updated in place; the first pass's input is requested before the last k-block's wgmma retires.
// Rows >= M and columns beyond the output are clipped by the tensor maps' bounds.
// The contraction may be extended by a second (A2,B2) segment: that is how the rank-r LoRA update is
// accumulated into the same accumulator as the frozen base weight (one extra k-block, no extra pass).
#include "common.cuh"
#include "kernels.h"

#include <mutex>

namespace dtx {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int GEMM_THREADS = 384;
constexpr int GROUP_M = 32;  // rasterisation group height in 128-row tiles (gemm_set_pair_group_m counts 256 rows)

struct GemmKParams {
  int M, N;
  int kb1, kb2;     // 64-wide k-blocks in segment 1 / segment 2
  int split_k;
  int kb_per_split;
  int m_tiles, n_tiles;
  void* C;
  long long ldc;
  const bf16* R;
  long long ldr;
  int group_m;  // 128-row tiles per rasterisation group
  void* aux;
  long long ld_aux;
  const float2* rope_cs;
  int rope_S, rope_cols, rope_inverse;
  const int32_t* rope_pos;  // optional per-row position (packed ragged batches); null: row % rope_S
  const int32_t* m_eff;  // device-side row count; 256-row blocks that start at or beyond it are skipped
  int c_cols, x_cols;    // inner extents of the tmC / tmX tensor maps: output boxes at or beyond them are not issued
  const bf16* bias;      // BIAS kernels: bf16 [N], added to the accumulator before rounding / rotary
  const bf16 *qk_wq, *qk_wk;  // QKNORM kernels: the [128] q_norm / k_norm weights (columns < qk_q_cols / the rotated ones beyond)
  int qk_q_cols;
  float qk_eps;
};

template <int BN>
struct GemmCfg {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (BN == 256) ? 4 : ((BN == 128) ? 6 : 8);  // 192 KB ring
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;
  static constexpr int BOX_BYTES = 64 * 128;             // one staging box: 64 rows x 128 bytes (64 bf16 or 32 fp32 columns)
  static constexpr int STG_BYTES = 2 * 2 * BOX_BYTES;    // two boxes per consumer warpgroup
  // 230 656 of the 232 448 bytes a block may opt into
  static constexpr int SMEM_BYTES = RING_BYTES + STG_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  // BIAS kernels: each consumer warpgroup stages the tile's BN bias values behind the barriers (231 680 bytes at BN = 256);
  // QKNORM kernels keep the 2 x 128 norm weights there
  static constexpr int BIAS_BYTES = 2 * BN * 2;
};

__device__ __forceinline__ float round_bf16(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// tmC: the output C (fp32: 3-D [split][M][N] with box {32, 64, 1}; bf16: 2-D with box {64, 64});
// tmX: the second operand of the epilogue (R of EPI_BF16_ADD, act of EPI_SWIGLU_FWD, gu of EPI_SWIGLU_BWD), bf16 box {64, 64}
// BIAS (EPI_BF16 / EPI_ROPE only): p.bias[n] is added to column n of the fp32 accumulator before the rounding or the rotary.  Each
// consumer warpgroup copies the tile's slice into its own shared-memory row at the start of the tile (one coalesced load per thread,
// hidden under the main loop); the first pass_begin() barrier of the epilogue orders it before the reads, the last pass_store()
// barrier of the previous tile orders the previous tile's reads before it.
// QKNORM (EPI_ROPE only): every rotated 128-column head is RMS-normalised before the rotary (Qwen3 q_norm / k_norm):
// x = bf16(acc), y = (w * x) * rsqrt(mean(x^2) + eps) in fp32, then the rotary.  A row's 128 values sit in the four lanes of a
// quad (32 each): 32 products and two shfl.xor give the sum of squares.  The pre-norm x is stored to tmX (aux [M, rope_cols])
// in an extra pass before the normalised head goes to C.  The two weight vectors sit in the warpgroup's bias row (read with
// ld.shared: with __ldg the compiler hoists the loads and the epilogue spills).
// ROPE_GLM (EPI_ROPE only, without QKNORM): GLM's partial interleaved rotary - only columns 0..63 of every rotated head turn, in
// adjacent pairs (2i, 2i + 1) with frequency i; columns 64..127 pass through.  A pair is two neighbouring accumulator registers of
// one thread, so no shuffles are needed; the table is [S][32].
template <int BN, bool A_MN, bool B_MN, int EPI, bool BIAS = false, bool QKNORM = false, bool ROPE_GLM = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
            const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
            const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmX, const GemmKParams p) {
  using Cfg = GemmCfg<BN>;
  static_assert(EPI < EPI_ROPE || BN == 256, "the fused epilogues pair columns 64 / 128 apart inside one 256-column tile");
  static_assert(!BIAS || EPI == EPI_BF16 || EPI == EPI_ROPE, "the bias is added by the EPI_BF16 and EPI_ROPE epilogues only");
  static_assert(!QKNORM || (EPI == EPI_ROPE && !BIAS), "the q/k norm runs in the EPI_ROPE epilogue, without a bias");
  static_assert(!ROPE_GLM || (EPI == EPI_ROPE && !QKNORM), "the GLM rotary runs in the EPI_ROPE epilogue, without the q/k norm");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::RING_BYTES + Cfg::STG_BYTES);
  uint64_t* empty_bar = full_bar + Cfg::STAGES;
  uint64_t* x_bar = empty_bar + Cfg::STAGES;  // one per consumer warpgroup: its epilogue-input tiles have landed

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmA2);
    tma_prefetch_desc(&tmB2);
    tma_prefetch_desc(&tmC);
    tma_prefetch_desc(&tmX);
    for (int i = 0; i < Cfg::STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);  // lane 0 of each of the eight consumer warps
    }
    mbar_init(&x_bar[0], 1);
    mbar_init(&x_bar[1], 1);
    fence_barrier_init();
  }
  __syncthreads();

  const int kb_total = p.kb1 + p.kb2;
  const int tiles_mn = p.m_tiles * p.n_tiles;
  const int total_tiles = tiles_mn * p.split_k;
  // rows that exist on the device only (e.g. the number of unmasked tokens of this batch): every role skips the same tiles
  const int m_eff = p.m_eff ? min(p.M, __ldg(p.m_eff)) : p.M;

  auto decode = [&](int tile, int& m_blk, int& n_blk, int& split, int& kb_begin, int& kb_end) {
    split = tile / tiles_mn;
    int t = tile - split * tiles_mn;
    const int per_group = p.group_m * p.n_tiles;
    int group = t / per_group;
    int first_m = group * p.group_m;
    int gsz = min(p.group_m, p.m_tiles - first_m);
    int r = t - group * per_group;
    m_blk = first_m + (r % gsz);
    n_blk = r / gsz;
    kb_begin = split * p.kb_per_split;
    kb_end = min(kb_total, kb_begin + p.kb_per_split);
  };
  auto dead = [&](int m_blk) { return (m_blk >> 1) * 256 >= m_eff; };

  if (wg == 0) {
    // ------------------------------ TMA producer ------------------------------
    setmaxnreg_dec<40>();
    if (warp == 0) {
      const bool leader = elect_one();
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int m_blk, n_blk, split, kb_begin, kb_end;
        decode(tile, m_blk, n_blk, split, kb_begin, kb_end);
        if (dead(m_blk)) continue;
        const int m0 = m_blk * BM, n0 = n_blk * BN;
        for (int kb = kb_begin; kb < kb_end; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          if (leader) mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
          uint8_t* a_dst = smem + stage * Cfg::STAGE_BYTES;
          uint8_t* b_dst = a_dst + Cfg::A_BYTES;
          const bool seg2 = kb >= p.kb1;
          const int kk = (seg2 ? kb - p.kb1 : kb) * BK;
          const CUtensorMap* ma = seg2 ? &tmA2 : &tmA;
          const CUtensorMap* mb = seg2 ? &tmB2 : &tmB;
          if (leader) {
            if (!A_MN) {
              tma_load_2d(a_dst, ma, &full_bar[stage], kk, m0);
            } else {
#pragma unroll
              for (int j = 0; j < BM / 64; ++j) tma_load_2d(a_dst + j * 8192, ma, &full_bar[stage], m0 + 64 * j, kk);
            }
            if (!B_MN) {
              tma_load_2d(b_dst, mb, &full_bar[stage], kk, n0);
            } else {
#pragma unroll
              for (int j = 0; j < BN / 64; ++j) tma_load_2d(b_dst + j * 8192, mb, &full_bar[stage], n0 + 64 * j, kk);
            }
          }
          if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ------------------------------ consumers (warpgroups 1, 2) ------------------------------
    setmaxnreg_inc<232>();
    const int cw = wg - 1;                 // rows 64 * cw .. + 63 of the tile
    const int wq = warp & 3;               // warp inside the warpgroup
    const int rq = lane >> 2, cq = (lane & 3) * 2;
    const bool issuer = (threadIdx.x & 127) == 0;  // issues this warpgroup's epilogue bulk copies and waits for them
    uint8_t* stg = smem + Cfg::RING_BYTES + cw * 2 * Cfg::BOX_BYTES;
    const uint32_t stg_u = smem_u32(stg);
    uint32_t x_phase = 0;
    bf16* bias_s = reinterpret_cast<bf16*>(smem + Cfg::RING_BYTES + Cfg::STG_BYTES + 256) + cw * BN;
    // bias of columns 8 j + cq, + 1 of the tile
    auto bias2 = [&](int j) -> float2 { return __bfloat1622float2(reinterpret_cast<const __nv_bfloat162*>(bias_s)[4 * j + (cq >> 1)]); };
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    if (QKNORM) {  // [q_norm | k_norm] weights in this warpgroup's bias row, once for all tiles
      for (int c = threadIdx.x & 127; c < 256; c += 128) bias_s[c] = c < 128 ? __ldg(p.qk_wq + c) : __ldg(p.qk_wk + c - 128);
      named_bar_sync(1 + cw, 128);
    }

    // staging address of this thread's element pair in row wq * 16 + rq + 8 * hr of box `box`: 16-byte chunk `ch`, byte `b`
    auto sa = [&](int hr, int box, int ch, int b) -> uint32_t {
      return stg_u + box * Cfg::BOX_BYTES + sw128_offset(wq * 16 + rq + 8 * hr, ch) + b;
    };
    // the staging half is written only once the bulk stores of the previous pass have read it
    auto pass_begin = [&]() {
      if (issuer) tma_store_wait_read0();
      named_bar_sync(1 + cw, 128);
    };
    // TMA-load the tmX boxes at columns x0 + b * dx (b < nbox), rows y .. y + 63, into the staging half
    auto x_load = [&](int x0, int dx, int nbox, int y) {
      if (issuer) {
        tma_store_wait_read0();
        uint32_t bytes = 0;
        for (int b = 0; b < nbox; ++b)
          if (y < p.M && x0 + b * dx < p.x_cols) bytes += Cfg::BOX_BYTES;
        mbar_arrive_expect_tx(&x_bar[cw], bytes);
        for (int b = 0; b < nbox; ++b)
          if (y < p.M && x0 + b * dx < p.x_cols) tma_load_2d(stg + b * Cfg::BOX_BYTES, &tmX, &x_bar[cw], x0 + b * dx, y);
      }
    };
    auto x_wait = [&]() {
      mbar_wait(&x_bar[cw], x_phase);
      x_phase ^= 1u;
    };
    // hand the pass to the async proxy and store its boxes to columns x0 + b * dx of `m` (split z of an fp32 output)
    auto pass_store = [&](const CUtensorMap* m, int cols, int x0, int dx, int nbox, int y, int z) {
      fence_proxy_async_smem();
      named_bar_sync(1 + cw, 128);
      if (issuer) {
        for (int b = 0; b < nbox; ++b) {
          if (y >= p.M || x0 + b * dx >= cols) continue;
          if (EPI == EPI_F32) {
            tma_store_3d(m, stg + b * Cfg::BOX_BYTES, x0 + b * dx, y, z);
          } else {
            tma_store_2d(m, stg + b * Cfg::BOX_BYTES, x0 + b * dx, y);
          }
        }
        tma_store_commit();
      }
    };

    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      int m_blk, n_blk, split, kb_begin, kb_end;
      decode(tile, m_blk, n_blk, split, kb_begin, kb_end);
      if (dead(m_blk)) continue;
      const int m0 = m_blk * BM, n0 = n_blk * BN;
      const int y0 = m0 + cw * 64;  // first row of this warpgroup's slice
      if (BIAS)
        for (int c = threadIdx.x & 127; c < BN; c += 128) bias_s[c] = n0 + c < p.N ? __ldg(p.bias + n0 + c) : __float2bfloat16_rn(0.f);
      int prev = -1;
      for (int kb = kb_begin; kb < kb_end; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_base = smem_u32(smem + stage * Cfg::STAGE_BYTES) + cw * 8192;  // 64 rows (K-major) or one 64-column box (MN-major)
        const uint32_t b_base = smem_u32(smem + stage * Cfg::STAGE_BYTES) + Cfg::A_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k16 = 0; k16 < BK / 16; ++k16) {
          const uint64_t da = A_MN ? wgmma_desc_mnmajor(a_base + k16 * 2048, 8192) : wgmma_desc_kmajor(a_base + k16 * 32);
          const uint64_t db = B_MN ? wgmma_desc_mnmajor(b_base + k16 * 2048, 8192) : wgmma_desc_kmajor(b_base + k16 * 32);
          wgmma_ss<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, (kb > kb_begin || k16 > 0) ? 1u : 0u);
        }
        wgmma_commit();
        if (prev >= 0) {  // the previous k-block's MMAs have read their slot once only this one is in flight
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = stage;
        if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1u; }
      }
      // the first pass's epilogue input is requested while the last k-block's MMAs run
      if (EPI == EPI_BF16_ADD) x_load(n0, 64, BN >= 128 ? 2 : 1, y0);
      if (EPI == EPI_SWIGLU_BWD) x_load(2 * n0, 128, 2, y0);
      wgmma_wait<0>();
      wgmma_touch(acc);
      if (lane == 0) mbar_arrive(&empty_bar[prev]);

      // ------------------------------ epilogue: accumulator fragment -> staging boxes -> bulk stores ------------------------------
      if (EPI == EPI_BF16 || EPI == EPI_BF16_ADD) {
        constexpr int NB = BN >= 128 ? 2 : 1;  // 64-column boxes per pass
#pragma unroll
        for (int ps = 0; ps < BN / (64 * NB); ++ps) {
          if (EPI == EPI_BF16_ADD) {
            if (ps > 0) x_load(n0 + 128 * ps, 64, NB, y0);
            x_wait();
          } else {
            pass_begin();
          }
#pragma unroll
          for (int jj = 0; jj < 8 * NB; ++jj) {
            const int j = ps * 8 * NB + jj;
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
              const uint32_t a = sa(hr, jj >> 3, jj & 7, cq * 2);
              float v0 = acc[4 * j + 2 * hr], v1 = acc[4 * j + 2 * hr + 1];
              if (BIAS) {
                const float2 b = bias2(j);
                v0 += b.x;
                v1 += b.y;
              }
              if (EPI == EPI_BF16_ADD) {  // the residual tile sits where the output goes
                const float2 rr = unpack_bf16x2(lds32(a));
                v0 += rr.x;
                v1 += rr.y;
              }
              sts32(a, pack_bf16x2(v0, v1));
            }
          }
          pass_store(&tmC, p.c_cols, n0 + 128 * ps, 64, NB, y0, 0);
        }
      } else if (EPI == EPI_F32) {
        // 64 columns per pass: two boxes of 32 fp32 columns
#pragma unroll
        for (int ps = 0; ps < BN / 64; ++ps) {
          pass_begin();
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = ps * 8 + jj;
#pragma unroll
            for (int hr = 0; hr < 2; ++hr)
              sts64f(sa(hr, jj >> 2, (jj & 3) * 2 + (cq >> 2), (cq & 3) * 4), acc[4 * j + 2 * hr], acc[4 * j + 2 * hr + 1]);
          }
          pass_store(&tmC, p.c_cols, n0 + 64 * ps, 32, 2, y0, split);
        }
      } else if (EPI == EPI_ROPE) {
        // two heads per tile (columns 0-127 / 128-255), one per pass; rotary pairs column i with i + 64 of a head (ROPE_GLM:
        // column 2i with 2i + 1 of the first 64)
        const bool rot = n0 < p.rope_cols;
        const float2* cs[2];
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int row = y0 + wq * 16 + rq + 8 * hr;
          const int pos = row >= p.M ? 0 : (p.rope_pos ? __ldg(p.rope_pos + row) : row % p.rope_S);
          if constexpr (ROPE_GLM) cs[hr] = p.rope_cs + static_cast<long long>(pos) * 32;
          else cs[hr] = p.rope_cs + static_cast<long long>(pos) * 64;
        }
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          float rstd[2] = {1.f, 1.f};
          if (QKNORM && rot) {
            // extra pass: the pre-norm bf16 head x to aux, its sum of squares per row, and w * x in place of acc (the rotary
            // pass below scales by rstd: HF order, q = q_norm(x W^T), then the rotary)
            const uint32_t w_u = smem_u32(bias_s + (n0 + 128 * hh < p.qk_q_cols ? 0 : 128)) + cq * 2;
            float ss[2] = {0.f, 0.f};
            pass_begin();
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int jl = hh * 16 + jj, jh = jl + 8;
              const float2 wl = unpack_bf16x2(lds32(w_u + jj * 16)), wh = unpack_bf16x2(lds32(w_u + 128 + jj * 16));
#pragma unroll
              for (int hr = 0; hr < 2; ++hr) {
                float* l = acc + 4 * jl + 2 * hr;
                float* h = acc + 4 * jh + 2 * hr;
                const float l0 = round_bf16(l[0]), l1 = round_bf16(l[1]), h0 = round_bf16(h[0]), h1 = round_bf16(h[1]);
                ss[hr] += l0 * l0 + l1 * l1 + h0 * h0 + h1 * h1;
                sts32(sa(hr, 0, jj, cq * 2), pack_bf16x2(l0, l1));
                sts32(sa(hr, 1, jj, cq * 2), pack_bf16x2(h0, h1));
                l[0] = wl.x * l0;
                l[1] = wl.y * l1;
                h[0] = wh.x * h0;
                h[1] = wh.y * h1;
              }
            }
            pass_store(&tmX, p.x_cols, n0 + 128 * hh, 64, 2, y0, 0);
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
              ss[hr] += __shfl_xor_sync(0xffffffffu, ss[hr], 1);
              ss[hr] += __shfl_xor_sync(0xffffffffu, ss[hr], 2);
              rstd[hr] = rsqrtf(ss[hr] * (1.f / 128.f) + p.qk_eps);
            }
          }
          pass_begin();
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int jl = hh * 16 + jj, jh = jl + 8;
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
              float lo[2] = {acc[4 * jl + 2 * hr], acc[4 * jl + 2 * hr + 1]}, hi[2] = {acc[4 * jh + 2 * hr], acc[4 * jh + 2 * hr + 1]};
              if (QKNORM && rot) {
                lo[0] *= rstd[hr];
                lo[1] *= rstd[hr];
                hi[0] *= rstd[hr];
                hi[1] *= rstd[hr];
              }
              if (BIAS) {  // HF order: q = x W^T + b, then the rotary
                const float2 bl = bias2(jl), bh = bias2(jh);
                lo[0] += bl.x;
                lo[1] += bl.y;
                hi[0] += bh.x;
                hi[1] += bh.y;
              }
              if constexpr (ROPE_GLM) {
                if (rot) {  // columns 8 jj + cq, + 1 of the head are pair 4 jj + cq / 2
                  const float2 t = __ldg(cs[hr] + jj * 4 + (cq >> 1));
                  const float sn = p.rope_inverse ? -t.y : t.y;
                  const float x0 = lo[0], x1 = lo[1];
                  lo[0] = x0 * t.x - x1 * sn;
                  lo[1] = x1 * t.x + x0 * sn;
                }
              } else if (rot) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const float2 t = __ldg(cs[hr] + jj * 8 + cq + e);
                  const float sn = p.rope_inverse ? -t.y : t.y;
                  const float x0 = lo[e], x1 = hi[e];
                  lo[e] = x0 * t.x - x1 * sn;
                  hi[e] = x1 * t.x + x0 * sn;
                }
              }
              sts32(sa(hr, 0, jj, cq * 2), pack_bf16x2(lo[0], lo[1]));
              sts32(sa(hr, 1, jj, cq * 2), pack_bf16x2(hi[0], hi[1]));
            }
          }
          pass_store(&tmC, p.c_cols, n0 + 128 * hh, 64, 2, y0, 0);
        }
      } else if (EPI == EPI_SWIGLU_FWD) {
        // tile = [gate 128 | up 128] of the same 128 features: pass 0 stores gate and pass 1 up to C, pass 2 the activation to aux
#pragma unroll
        for (int ps = 0; ps < 3; ++ps) {
          pass_begin();
#pragma unroll
          for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
              const float g0 = acc[4 * j + 2 * hr], g1 = acc[4 * j + 2 * hr + 1];
              const float u0 = acc[4 * (j + 16) + 2 * hr], u1 = acc[4 * (j + 16) + 2 * hr + 1];
              uint32_t v;
              if (ps == 0) {
                v = pack_bf16x2(g0, g1);
              } else if (ps == 1) {
                v = pack_bf16x2(u0, u1);
              } else {
                // like the unfused path, gate/up are rounded to bf16 before the activation (fast reciprocal: ~1 ulp apart)
                const float gg0 = round_bf16(g0), gg1 = round_bf16(g1), uu0 = round_bf16(u0), uu1 = round_bf16(u1);
                v = pack_bf16x2(gg0 * __fdividef(1.f, 1.f + __expf(-gg0)) * uu0, gg1 * __fdividef(1.f, 1.f + __expf(-gg1)) * uu1);
              }
              sts32(sa(hr, j >> 3, j & 7, cq * 2), v);
            }
          }
          if (ps < 2) {
            pass_store(&tmC, p.c_cols, n0 + 128 * ps, 64, 2, y0, 0);
          } else {
            pass_store(&tmX, p.x_cols, n0 >> 1, 64, 2, y0, 0);
          }
        }
      } else {
        // EPI_SWIGLU_BWD: acc = d(act) for features n0 + 8j + cq + e; gate/up of feature f live at (f/128)*256 + f%128 (+128) of
        // gu / d(gu). Pass q covers features n0 + 64q .. + 63: their gate and up columns are one box each, rewritten in place.
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int xg = 2 * n0 + (q >> 1) * 256 + (q & 1) * 64;
          if (q > 0) x_load(xg, 128, 2, y0);
          x_wait();
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = 8 * q + jj;
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
              const uint32_t ga = sa(hr, 0, jj, cq * 2), ua = sa(hr, 1, jj, cq * 2);
              const float2 g2 = unpack_bf16x2(lds32(ga));
              const float2 u2 = unpack_bf16x2(lds32(ua));
              // d(act) is rounded to bf16 first, exactly like the unfused path that stores it
              const float d0 = round_bf16(acc[4 * j + 2 * hr]), d1 = round_bf16(acc[4 * j + 2 * hr + 1]);
              const float s0 = __fdividef(1.f, 1.f + __expf(-g2.x)), s1 = __fdividef(1.f, 1.f + __expf(-g2.y));
              const float si0 = g2.x * s0, si1 = g2.y * s1;
              sts32(ga, pack_bf16x2(d0 * u2.x * (s0 + si0 * (1.f - s0)), d1 * u2.y * (s1 + si1 * (1.f - s1))));
              sts32(ua, pack_bf16x2(d0 * si0, d1 * si1));
            }
          }
          pass_store(&tmC, p.c_cols, xg, 128, 2, y0, 0);
        }
      }
    }
    if (issuer) tma_store_wait0();  // the kernel's last bulk stores are complete before its shared memory goes away
  }
}

// ----------------------------------------------------------------------------------------------
// host side: tensor maps
// ----------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

}  // namespace

// 2-D bf16 tensor map over a row-major [outer, inner] array with row stride ld (elements), 128B swizzle.
bool make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner,
                       uint32_t box_outer) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return false;
  cuuint64_t gdim[2] = {inner, outer};
  cuuint64_t gstride[1] = {ld * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

namespace {

// 3-D fp32 tensor map over [outer2][outer][inner] with row stride ld and plane stride plane (elements), box {32, 64, 1}, 128B
// swizzle: the split-K partial sums of EPI_F32, so that rows >= M of one split are clipped rather than written into the next
bool make_tmap_3d_f32(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer, uint64_t outer2, uint64_t ld,
                      uint64_t plane) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return false;
  cuuint64_t gdim[3] = {inner, outer, outer2};
  cuuint64_t gstride[2] = {ld * 4, plane * 4};
  cuuint32_t box[3] = {32, 64, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

}  // namespace

int gemm_num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  }
  return n;
}

namespace {

// runs `fn` once per CUDA device (thread-safe): function attributes are per-device state
struct DeviceOnce {
  std::mutex mu;
  bool done[64] = {false};
  template <typename F>
  cudaError_t run(F fn) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    std::lock_guard<std::mutex> lk(mu);
    if (dev >= 0 && dev < 64 && done[dev]) return cudaSuccess;
    e = fn();
    if (e == cudaSuccess && dev >= 0 && dev < 64) done[dev] = true;
    return e;
  }
};

int g_wide_tiles = 1;
int g_group_m = GROUP_M;

template <int BN, bool A_MN, bool B_MN, int EPI, bool BIAS = false, bool QKNORM = false, bool ROPE_GLM = false>
cudaError_t launch(const GemmArgs& a, cudaStream_t s) {
  using Cfg = GemmCfg<BN>;
  constexpr int SMEM = Cfg::SMEM_BYTES + (BIAS || QKNORM ? Cfg::BIAS_BYTES : 0);
  auto kern = gemm_kernel<BN, A_MN, B_MN, EPI, BIAS, QKNORM, ROPE_GLM>;
  static DeviceOnce attr;  // the attribute is per device: a second trainer on another GPU of the same process needs it too
  if (cudaError_t e = attr.run([&] { return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM); });
      e != cudaSuccess)
    return e;
  CUtensorMap tA, tB, tA2, tB2;
  bool ok = true;
  // K-major operand: global [rows, K], box {64 k, rows_per_tile}; MN-major: global [K, cols], box {64 cols, 64 k}
  ok &= A_MN ? make_tmap_2d_bf16(&tA, a.A, a.M, a.K, a.lda, 64, 64) : make_tmap_2d_bf16(&tA, a.A, a.K, a.M, a.lda, 64, BM);
  ok &= B_MN ? make_tmap_2d_bf16(&tB, a.B, a.N, a.K, a.ldb, 64, 64) : make_tmap_2d_bf16(&tB, a.B, a.K, a.N, a.ldb, 64, BN);
  if (a.K2 > 0) {
    ok &= A_MN ? make_tmap_2d_bf16(&tA2, a.A2, a.M, a.K2, a.lda2, 64, 64)
               : make_tmap_2d_bf16(&tA2, a.A2, a.K2, a.M, a.lda2, 64, BM);
    ok &= B_MN ? make_tmap_2d_bf16(&tB2, a.B2, a.N, a.K2, a.ldb2, 64, 64)
               : make_tmap_2d_bf16(&tB2, a.B2, a.K2, a.N, a.ldb2, 64, BN);
  } else {
    tA2 = tA;
    tB2 = tB;
  }
  // epilogue tensor maps: C (and for the fused epilogues its second operand), boxes of 64 rows x 128 bytes
  CUtensorMap tC, tX;
  int c_cols = a.N, x_cols = 0;
  if (EPI == EPI_SWIGLU_BWD) c_cols = 2 * a.N;  // d(gu) holds gate and up columns of every feature
  if (EPI == EPI_F32) {
    const int splits = a.split_k < 1 ? 1 : a.split_k;
    ok &= make_tmap_3d_f32(&tC, a.C, a.N, a.M, splits, a.ldc, static_cast<uint64_t>(a.M) * a.ldc);
  } else {
    ok &= make_tmap_2d_bf16(&tC, a.C, c_cols, a.M, a.ldc, 64, 64);
  }
  if (EPI == EPI_BF16_ADD) {
    x_cols = a.N;
    ok &= make_tmap_2d_bf16(&tX, a.R, x_cols, a.M, a.ldr, 64, 64);
  } else if (EPI == EPI_SWIGLU_FWD || EPI == EPI_SWIGLU_BWD) {
    x_cols = EPI == EPI_SWIGLU_FWD ? a.N / 2 : 2 * a.N;  // act out / gu in
    ok &= make_tmap_2d_bf16(&tX, a.aux, x_cols, a.M, a.ld_aux, 64, 64);
  } else if (QKNORM) {  // pre-norm q|k out
    x_cols = a.rope_cols;
    ok &= make_tmap_2d_bf16(&tX, a.aux, x_cols, a.M, a.ld_aux, 64, 64);
  } else {
    tX = tC;
  }
  if (!ok) return cudaErrorInvalidValue;

  GemmKParams p;
  p.M = a.M;
  p.N = a.N;
  p.kb1 = (a.K + BK - 1) / BK;
  p.kb2 = (a.K2 + BK - 1) / BK;
  p.split_k = a.split_k < 1 ? 1 : a.split_k;
  int kb_total = p.kb1 + p.kb2;
  if (p.split_k > kb_total) p.split_k = kb_total;
  p.kb_per_split = (kb_total + p.split_k - 1) / p.split_k;
  // every split must own at least one k-block (an empty split would publish a stale accumulator)
  while (p.split_k > 1 && (p.split_k - 1) * p.kb_per_split >= kb_total) --p.split_k;
  if (p.split_k != (a.split_k < 1 ? 1 : a.split_k)) return cudaErrorInvalidValue;
  p.m_tiles = (a.M + BM - 1) / BM;
  p.n_tiles = (a.N + BN - 1) / BN;
  p.C = a.C;
  p.ldc = a.ldc;
  p.R = a.R;
  p.ldr = a.ldr;
  p.group_m = g_group_m;
  p.aux = a.aux;
  p.ld_aux = a.ld_aux;
  p.rope_cs = a.rope_cs;
  p.rope_S = a.rope_S;
  p.rope_cols = a.rope_cols;
  p.rope_inverse = a.rope_inverse;
  p.rope_pos = a.rope_pos;
  p.m_eff = p.split_k > 1 ? nullptr : a.m_eff;
  p.c_cols = c_cols;
  p.x_cols = x_cols;
  p.bias = a.bias;
  p.qk_wq = a.qk_wq;
  p.qk_wk = a.qk_wk;
  p.qk_q_cols = a.qk_q_cols;
  p.qk_eps = a.qk_eps;
  int total = p.m_tiles * p.n_tiles * p.split_k;
  int grid = total < gemm_num_sms() ? total : gemm_num_sms();
  if (grid <= 0) return cudaSuccess;
  kern<<<grid, GEMM_THREADS, SMEM, s>>>(tA, tB, tA2, tB2, tC, tX, p);
  return cudaGetLastError();
}

template <int BN, bool A_MN, bool B_MN>
cudaError_t launch_epi(const GemmArgs& a, cudaStream_t s) {
  switch (a.epilogue) {
    case EPI_BF16: return launch<BN, A_MN, B_MN, EPI_BF16>(a, s);
    case EPI_F32: return launch<BN, A_MN, B_MN, EPI_F32>(a, s);
    case EPI_BF16_ADD: return launch<BN, A_MN, B_MN, EPI_BF16_ADD>(a, s);
  }
  return cudaErrorInvalidValue;
}

template <bool B_MN>
cudaError_t launch_fused(const GemmArgs& a, cudaStream_t s) {
  if (a.rope_glm) {  // EPI_ROPE without the q/k norm (checked by gemm_bf16)
    return a.bias ? launch<256, false, B_MN, EPI_ROPE, true, false, true>(a, s) : launch<256, false, B_MN, EPI_ROPE, false, false, true>(a, s);
  }
  if (a.bias) return a.epilogue == EPI_ROPE ? launch<256, false, B_MN, EPI_ROPE, true>(a, s) : cudaErrorInvalidValue;
  if (a.qk_wq) return a.epilogue == EPI_ROPE ? launch<256, false, B_MN, EPI_ROPE, false, true>(a, s) : cudaErrorInvalidValue;
  switch (a.epilogue) {
    case EPI_ROPE: return launch<256, false, B_MN, EPI_ROPE>(a, s);
    case EPI_SWIGLU_FWD: return launch<256, false, B_MN, EPI_SWIGLU_FWD>(a, s);
    case EPI_SWIGLU_BWD: return launch<256, false, B_MN, EPI_SWIGLU_BWD>(a, s);
  }
  return cudaErrorInvalidValue;
}

template <int BN>
cudaError_t launch_major(const GemmArgs& a, cudaStream_t s) {
  if (a.bias) {  // EPI_BF16 with a K-major A (checked by gemm_bf16)
    return a.b_mn_major ? launch<BN, false, true, EPI_BF16, true>(a, s) : launch<BN, false, false, EPI_BF16, true>(a, s);
  }
  if (!a.a_mn_major && !a.b_mn_major) return launch_epi<BN, false, false>(a, s);
  if (!a.a_mn_major && a.b_mn_major) return launch_epi<BN, false, true>(a, s);
  if (a.a_mn_major && a.b_mn_major) return launch_epi<BN, true, true>(a, s);
  return cudaErrorInvalidValue;  // (MN-major A, K-major B) is not used on the training path
}

}  // namespace

void gemm_set_pair_kernel(int on) { g_wide_tiles = on; }
void gemm_set_pair_group_m(int g) { g_group_m = g > 0 ? 2 * g : GROUP_M; }

cudaError_t gemm_bf16(const GemmArgs& a, cudaStream_t s) {
  if (a.M <= 0 || a.N <= 0 || a.K <= 0) return cudaErrorInvalidValue;
  if (a.split_k > 1 && a.epilogue != EPI_F32) return cudaErrorInvalidValue;
  if (a.epilogue == EPI_BF16_ADD && a.R == nullptr) return cudaErrorInvalidValue;
  // bias variants: the plain bf16 and the RoPE epilogue, K-major A, one split
  if (a.bias && ((a.epilogue != EPI_BF16 && a.epilogue != EPI_ROPE) || a.a_mn_major || a.split_k > 1)) return cudaErrorInvalidValue;
  // q/k norm: EPI_ROPE only, without a bias; whole heads on both sides of the q / k boundary, a 16-byte aligned pre-norm output
  if (a.qk_wq && (a.epilogue != EPI_ROPE || a.bias || !a.qk_wk || (a.qk_q_cols & 127) || a.qk_q_cols < 0 ||
                  a.qk_q_cols > a.rope_cols || !(a.qk_eps >= 0.f) || !a.aux || (a.ld_aux & 7) || a.ld_aux < a.rope_cols ||
                  (reinterpret_cast<uintptr_t>(a.aux) & 15) || (reinterpret_cast<uintptr_t>(a.qk_wq) & 3) ||
                  (reinterpret_cast<uintptr_t>(a.qk_wk) & 3)))
    return cudaErrorInvalidValue;
  // GLM rotary: EPI_ROPE only, not combined with the q/k norm
  if (a.rope_glm && (a.rope_glm != 1 || a.epilogue != EPI_ROPE || a.qk_wq)) return cudaErrorInvalidValue;
  // TMA needs 16-byte aligned bases and row strides
  if ((a.lda & 7) || (a.ldb & 7) || (reinterpret_cast<uintptr_t>(a.A) & 15) || (reinterpret_cast<uintptr_t>(a.B) & 15))
    return cudaErrorInvalidValue;
  if (a.K2 > 0 && ((a.lda2 & 7) || (a.ldb2 & 7) || !a.A2 || !a.B2)) return cudaErrorInvalidValue;
  // the epilogue stores C (and loads R / reads or writes aux) through TMA as well
  const int64_t c_align = a.epilogue == EPI_F32 ? 3 : 7;  // row stride in elements: a multiple of 16 bytes
  if (!a.C || (a.ldc & c_align) || (reinterpret_cast<uintptr_t>(a.C) & 15)) return cudaErrorInvalidValue;
  if (a.epilogue == EPI_BF16_ADD && ((a.ldr & 7) || (reinterpret_cast<uintptr_t>(a.R) & 15))) return cudaErrorInvalidValue;
  if (a.epilogue == EPI_SWIGLU_FWD || a.epilogue == EPI_SWIGLU_BWD) {
    if (!a.aux || (a.ld_aux & 7) || (reinterpret_cast<uintptr_t>(a.aux) & 15)) return cudaErrorInvalidValue;
  }
  if (a.epilogue >= EPI_ROPE) {  // fused epilogues exist only for whole 256-column tiles
    if (a.a_mn_major || a.split_k > 1 || a.M <= 128 || !g_wide_tiles) return cudaErrorInvalidValue;
    if (a.epilogue == EPI_ROPE && (!a.rope_cs || a.rope_S <= 0 || (a.rope_cols & 255) || (a.N & 255))) return cudaErrorInvalidValue;
    if (a.epilogue == EPI_SWIGLU_FWD && (a.N & 255)) return cudaErrorInvalidValue;
    if (a.epilogue == EPI_SWIGLU_BWD && (a.N & 127)) return cudaErrorInvalidValue;
    return a.b_mn_major ? launch_fused<true>(a, s) : launch_fused<false>(a, s);
  }
  int bn = a.block_n;
  if (bn == 0) bn = (a.N <= 64) ? 64 : ((a.N <= 128) ? 128 : 256);
  if (bn == 256 && !g_wide_tiles) bn = 128;
  switch (bn) {
    case 64: return launch_major<64>(a, s);
    case 128: return launch_major<128>(a, s);
    case 256: return launch_major<256>(a, s);
  }
  return cudaErrorInvalidValue;
}

}  // namespace dtx
