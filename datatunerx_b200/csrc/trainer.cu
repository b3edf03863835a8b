// The training step of the DataTunerX fine-tuning worker, rebuilt for H100.
//
// Replaces, for the data-parallel LoRA-SFT path, what the reference reaches through
//   cmd/tuning/train.py:299  trainer.train()  ->  HF Trainer.training_step / LlamaForCausalLM.forward /
//   peft lora.Linear / DeepSpeed ZeRO-0 all-reduce / clip_grad_norm_ / torch.optim.AdamW / get_scheduler
// (SURVEY §8a rows a7-a11).  One dtx_trainer = one GPU rank.  No PyTorch, no CPU fallback.
//
// HBM layout (DESIGN.md §3): frozen base weights bf16 with q|k|v and gate|up row-concatenated so that one
// GEMM serves each pair; LoRA masters fp32 in one flat buffer (A^T[d,r] | B[d,r] per target per layer) with
// m, v and the gradient in identically laid-out flat buffers (one NCCL all-reduce, one AdamW launch);
// bf16 "shadows" of the adapters padded to a 64-wide rank block feed the tensor-core GEMMs.
// Activations needed by backward are kept per layer when they fit in device memory (7B LoRA at 8K tokens/step: 43 GB of
// 80); otherwise one shared set of decoder-layer activations is refilled by re-running each layer's forward in the backward
// pass (gradient checkpointing per layer, DESIGN.md §3).  Both layouts launch the same kernels on the same inputs, so they
// give bitwise-identical results.
#include "kernels.h"
#include "../../include/dtxtune.h"

#include <cuda.h>
#include <dlfcn.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

namespace dtx {

namespace {

// ------------------------------------------------------------------------------------------------
// NCCL, loaded lazily so that libdtxtune.so has no link-time dependency (N=1 runs never touch it)
// ------------------------------------------------------------------------------------------------
struct UidByValue {  // ncclUniqueId is passed by value
  char internal[128];
};
struct NcclApi {
  void* handle = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, UidByValue, int) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*ReduceScatter)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;  // (send, recv, recvcount, dtype, op, comm, stream)
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;           // (send, recv, sendcount, dtype, comm, stream)
  int (*CommDestroy)(void*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
NcclApi* nccl_api() {
  static NcclApi api;
  static bool tried = false;
  if (!tried) {
    tried = true;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      // RTLD_LOCAL: a host that imports PyTorch AFTER this call must still resolve ITS bundled NCCL's newer symbols - with
      // RTLD_GLOBAL the system libnccl (2.27) shadowed them and `import torch` died with "undefined symbol: ncclDevCommCreate"
      api.handle = dlopen(n, RTLD_NOW | RTLD_LOCAL);
      if (api.handle) break;
    }
    if (api.handle) {
      api.GetUniqueId = reinterpret_cast<int (*)(void*)>(dlsym(api.handle, "ncclGetUniqueId"));
      api.CommInitRank = reinterpret_cast<int (*)(void**, int, UidByValue, int)>(dlsym(api.handle, "ncclCommInitRank"));
      api.AllReduce = reinterpret_cast<int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t)>(
          dlsym(api.handle, "ncclAllReduce"));
      api.ReduceScatter = reinterpret_cast<int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t)>(
          dlsym(api.handle, "ncclReduceScatter"));
      api.AllGather = reinterpret_cast<int (*)(const void*, void*, size_t, int, void*, cudaStream_t)>(dlsym(api.handle, "ncclAllGather"));
      api.CommDestroy = reinterpret_cast<int (*)(void*)>(dlsym(api.handle, "ncclCommDestroy"));
      api.GetErrorString = reinterpret_cast<const char* (*)(int)>(dlsym(api.handle, "ncclGetErrorString"));
    }
  }
  if (!api.handle || !api.GetUniqueId || !api.CommInitRank || !api.AllReduce || !api.CommDestroy) return nullptr;
  return &api;
}
constexpr int kNcclFloat32 = 7;
constexpr int kNcclFloat64 = 8;
constexpr int kNcclBfloat16 = 9;
constexpr int kNcclSum = 0;

thread_local std::string g_error;
int g_nf4_prefetch = 1;     // expand the next NF4 matrix on a side stream while the current GEMM runs (0: inline, for A/B runs)
int g_varlen_split = 1;     // ragged micro-batches run as length groups (rows sorted by length, partition chosen by a cost model);
                            // 2: always cut where the 128-rounded lengths differ (parity tests at shapes too small for the model to split)
int g_varlen_pack = 1;      // ragged LoRA micro-batches run PACKED: sequences back to back at 128-rounded lengths, one pass (0: length groups)
int g_varlen_fix_permille = 200;   // fixed cost charged per length group, in thousandths of "one wave of every GEMM of a layer"
int g_fused_epilogues = 1;  // RoPE / SwiGLU fused into the GEMM and attention epilogues (needs M > 128)

// ------------------------------------------------------------------------------------------------
// LoRA-specific small kernels
// ------------------------------------------------------------------------------------------------
// dst[n*r + j] (+)= scale * sum_s part[s*split_stride + (row0+n)*ld + col0 + j]   (fixed order)
__global__ void lora_gather_kernel(const float* __restrict__ part, int splits, long long split_stride, int ld, int row0,
                                   int col0, int rows, int r, float* __restrict__ dst, int accumulate, float scale) {
  const long long total = static_cast<long long>(rows) * r;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int n = static_cast<int>(i / r), j = static_cast<int>(i % r);
    const float* src = part + static_cast<long long>(row0 + n) * ld + col0 + j;
    float s = 0.f;
    for (int k = 0; k < splits; ++k) s += src[k * split_stride];
    s *= scale;
    dst[i] = accumulate ? dst[i] + s : s;
  }
}

// Per-target geometry of the LoRA adapters inside one layer's block of the flat parameter buffer.
struct TargetInfo {
  int row0;        // first row of the target's output features inside wqkv / b_ext
  int d_out;       // output features (n_heads*128 for q, n_kv_heads*128 for k, v)
  long long off;   // offset of this target's [A^T (d x r) | B (d_out x r)] inside the layer block
};

// refresh bf16 shadows of all adapters from the fp32 masters.
//   a_cat[l][(ti*r + j)*KA + a_col0(ti) + c]  = A^T[c*r + j]      (KA = d, a_col0 = 0; with LoRA dropout KA = nt*d, a_col0 = ti*d)
//   b_ext[l][(row0[ti] + n)*RP + ti*r + j]    = scale * B[n*r + j]
struct ShadowArgs {
  const float* params;
  bf16* a_cat;
  bf16* b_ext;
  int L, d, r, RP, nt, KA, W, a_split;
  long long per_layer;
  TargetInfo tg[3];
  float scale;
};
__global__ void lora_shadow_kernel(ShadowArgs a) {
  const long long total = a.per_layer * a.L;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int l = static_cast<int>(i / a.per_layer);
    long long rem = i - l * a.per_layer;
    int ti = 0;
    while (ti + 1 < a.nt && rem >= a.tg[ti + 1].off) ++ti;
    rem -= a.tg[ti].off;
    const float v = a.params[i];
    if (rem < static_cast<long long>(a.d) * a.r) {
      const int c = static_cast<int>(rem / a.r), j = static_cast<int>(rem % a.r);
      a.a_cat[(static_cast<long long>(l) * a.RP + ti * a.r + j) * a.KA + (a.a_split ? ti * a.d : 0) + c] = __float2bfloat16_rn(v);
    } else {
      rem -= static_cast<long long>(a.d) * a.r;
      const int n = static_cast<int>(rem / a.r), j = static_cast<int>(rem % a.r);
      a.b_ext[(static_cast<long long>(l) * a.W + a.tg[ti].row0 + n) * a.RP + ti * a.r + j] = __float2bfloat16_rn(v * a.scale);
    }
  }
}

struct Layer {
  // wgu: [2F, d] in the GU-interleaved layout (128 gate rows | 128 up rows per 128 features)
  bf16 *wqkv = nullptr, *wo = nullptr, *wgu = nullptr, *wdown = nullptr, *norm1 = nullptr, *norm2 = nullptr;
  bf16* bias = nullptr;  // dtx_model_ext.qkv_bias: [W] q|k|v biases in the row order of wqkv (bf16 also under NF4), else null
  bf16* qkn = nullptr;   // dtx_model_ext.qk_norm: [2 * 128] q_norm | k_norm weights (bf16 also under NF4), else null
  bf16* qkf = nullptr;   // dtx_model_ext.qk_norm_full: [dq + dkv] q_norm | k_norm weights (bf16 also under NF4), else null
  bf16* qk_pre = nullptr;  // qk_norm / qk_norm_full, saved: [M, dq + dkv] q|k projection output before the norm (bf16)
  bf16* pn = nullptr;  // dtx_model_ext.post_norms: [2 * d] post_self_attn_layernorm | post_mlp_layernorm (bf16 also under NF4)
  // post_norms, saved: the o- and down-projection outputs before their norms [M, d] and the norms' rstd [M]
  bf16 *o_pre = nullptr, *down_pre = nullptr;
  float *rstd_pn1 = nullptr, *rstd_pn2 = nullptr;
  bf16 *a_cat = nullptr, *b_ext = nullptr;                                               // shadows
  bf16 *h1 = nullptr, *t = nullptr, *qkv = nullptr, *attn = nullptr, *x_mid = nullptr, *gu = nullptr;  // saved (no_pre_norms: no h1)
  bf16* hd = nullptr;  // LoRA dropout only: [M, nt*d] dropped copies of h1, one per target (peft: one nn.Dropout per module)
  float *lse = nullptr, *rstd1 = nullptr, *rstd2 = nullptr;
  // --quantization int4: packed NF4 codes (two per byte) + one fp32 absmax per 64 elements; the bf16 pointers above are then
  // null and the GEMMs read a per-trainer scratch that dequantize() fills right before each launch
  uint8_t* q4[4] = {nullptr, nullptr, nullptr, nullptr};   // wqkv, wo, wgu, wdown
  float* absmax[4] = {nullptr, nullptr, nullptr, nullptr};
};
enum { W_QKV = 0, W_O = 1, W_GU = 2, W_DOWN = 3 };

// One storage slot of a weight block.  dtx_trainer::lslots lists a decoder layer's slots and dtx_trainer::gslots the globals'
// (embed | lm_head | final norm); a tensor only some model families have is a row of its own, absent for the others.  Both
// tables are built once by setup_dims(), and every fact about a block comes from them: full-parameter SFT lays the block out
// in row order, LoRA allocates the slots one by one in that order, and the memory plan, loading, export, random init and NF4
// quantisation walk the rows.
enum { INIT_NORMAL, INIT_ZERO, INIT_ONE };  // dtx_init_random_weights: normal(0.02) with the next seed, 0 (biases), 1 (norms)
template <class Owner>
struct Slot {
  using Ptr = bf16* Owner::*;
  Ptr mem;            // the pointer this slot fills (Layer::wqkv, ..., dtx_trainer::embed, ...)
  int64_t n;          // elements
  int64_t off;        // offset inside the full-SFT block
  bool nodecay;       // no weight decay (HF get_decay_parameter_names skips biases and norm weights): such rows come last
  int nf4;            // W_QKV .. W_DOWN: NF4-packed by dtx_quantize_base (index of Layer::q4 / absmax); -1: always bf16
  int init;           // INIT_*
};

// A checkpoint tensor: the slot it lives in.  gate_proj and up_proj are the halves of the GU-interleaved wgu (128 gate rows,
// then the 128 up rows of the same features, ...); GLM's fused gate_up_proj holds all gate rows, then all up rows.
enum { GU_GATE = 1, GU_UP = 2, GU_BOTH = 3 };
struct WeightName {
  const char* key;     // a layer's: matched in the name after "layers.N.", a global's: anywhere; no key contains another
  const char* hf;      // globals: the checkpoint name (a layer's is "model.layers.N." + key)
  int slot;            // row of lslots / gslots
  int64_t off;         // element offset inside the slot (GU rows: 0)
  int64_t rows, cols;  // HF shape; a vector is [rows, 1]
  int gu;              // GU_*: which halves of wgu the tensor holds; 0: a plain copy at off
};

// activation layouts (dtx_train_cfg.recompute): every layer keeps its own saved set, or all layers share one that the
// backward pass refills by re-running each layer's forward
enum { KEEP_ALL = 1, RECOMPUTE_LAYER = 2 };
// which part of the step asks for a base weight (the NF4 prefetch predicts the next one from it)
enum { PH_FWD = 0, PH_RECOMPUTE = 1, PH_BWD = 2 };
// automatic layout choice: what the trainer may not take of the free device memory (NCCL communicator buffers, created
// after the trainer's own, and cudaMalloc granularity)
constexpr int64_t kHeadroomBytes = int64_t(1) << 30;

}  // namespace
void trainer_set_fused_epilogues(int on) { g_fused_epilogues = on; }
void trainer_set_nf4_prefetch(int on) { g_nf4_prefetch = on; }
void trainer_set_varlen_split(int on) { g_varlen_split = on; }
void trainer_set_varlen_pack(int on) { g_varlen_pack = on; }
void trainer_set_varlen_group_cost(int permille) { g_varlen_fix_permille = permille < 0 ? 0 : permille; }
}  // namespace dtx

using namespace dtx;

struct dtx_trainer {
  dtx_model_cfg mc{};
  dtx_model_ext ext{};          // all zero: plain Llama-2 / Mistral
  dtx_train_cfg tc{};
  int device = 0, rank = 0, world = 1;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  void* nccl_comm = nullptr;
  std::string err;
  std::vector<void*> allocs;
  size_t bytes_allocated = 0;
  bool dry = false;             // sizing only (dtx_plan_device_bytes, automatic layout): alloc() counts bytes, nothing is allocated
  int recompute = KEEP_ALL;     // activation layout in use

  int M = 0, RP = 0, nt = 0;    // M = micro_batch * seq_len: the largest batch this trainer was created for
  int cur_S = 0, cur_M = 0;     // padded length / token count of the batch being processed (<= seq_len / M)
  int cur_B = 0;                // its rows: micro_batch, or the rows of one length group (SubPlan)
  bool sub_accum = false;       // a later length group of the same micro-batch: gradients and loss add to the earlier groups'
  int sub_ndiv = 0;             // > 0: labelled tokens of the WHOLE micro-batch (the divisor of the token-mean loss of every group)
  int n_sms = 132;
  int last_groups = 1;          // length groups of the last training micro-batch (diagnostics; 0 = packed)
  bool packed = false;          // the batch in d_ids / d_labels is PACKED: sequence b owns rows d_row_start[b] .. d_row_start[b+1])
  bool use_seq_lens = false;    // d_seq_lens holds this batch's true row lengths
  int dq = 0, dkv = 0, W = 0;  // q / attention width (n_heads*128), k/v width (n_kv_heads*128), packed qkv row width
  int KA = 0;                  // contraction length of the LoRA down-projection: d, or nt*d with dropout
  bool dropout = false;
  TargetInfo tg[3];
  char tg_name[3] = {0, 0, 0};
  int64_t per_layer = 0, n_train = 0;
  uint64_t fwd_count = 0;      // forward passes so far: seeds the dropout masks

  bf16 *embed = nullptr, *lm_head = nullptr, *normf = nullptr;
  std::vector<Layer> layers;
  std::vector<bf16*> xs;  // residual stream, L+1 entries
  bf16 *a_cat_all = nullptr, *b_ext_all = nullptr;
  float *params = nullptr, *grads = nullptr, *adam_m = nullptr, *adam_v = nullptr;

  // transients
  bf16 *h2 = nullptr, *act = nullptr, *dact = nullptr, *dgu = nullptr, *dx_a = nullptr, *dx_b = nullptr, *dh = nullptr,
       *dattn = nullptr, *dqkv = nullptr, *dt = nullptr, *dlogits = nullptr, *glora = nullptr;
  float *logits = nullptr, *rstdf = nullptr, *row_loss = nullptr, *delta = nullptr, *part_b = nullptr, *part_a = nullptr;
  float *d_loss = nullptr, *d_sumsq = nullptr, *d_gnorm = nullptr, *d_scratch = nullptr;
  int32_t *d_ids = nullptr, *d_labels = nullptr, *d_shift = nullptr, *d_nvalid = nullptr, *d_seq_lens = nullptr;
  int32_t *d_row_map = nullptr, *d_valid_idx = nullptr;  // token -> position among the labelled tokens (-1: none) and back
  int32_t *d_ids_full = nullptr, *d_labels_full = nullptr, *d_lens_full = nullptr;  // the whole ragged micro-batch (length groups gather from it)
  int32_t *d_pos = nullptr, *d_row_start = nullptr;  // packed batch: position of every row inside its sequence; first row of every sequence
  std::vector<int32_t> h_labels, h_lens;  // host copies of a device-resident ragged batch (the partition is planned on the host)
  std::vector<float> h_row_sum;           // per-row evaluation statistics, rows in the order of the passes (RowStats)
  std::vector<int32_t> h_row_valid;
  float* d_row_sum = nullptr;     // [micro_batch] per-row summed token loss (evaluation)
  int32_t* d_row_valid = nullptr; // [micro_batch] per-row valid-token count
  double* d_host_red = nullptr;   // staging for dtx_allreduce_host
  int window = 0;                 // sliding-window attention span (0 = plain causal)
  bool rope_glm = false;          // GLM's partial interleaved rotary: rope_cs / rope_cs_t hold head_dim / 4 frequencies
  // base weights: the slot tables of a layer block and of the globals block (see Slot), the elements they add up to, and the
  // checkpoint names that load into them
  std::vector<Slot<Layer>> lslots;
  std::vector<Slot<dtx_trainer>> gslots;
  int64_t layer_used = 0, glob_used = 0;
  std::vector<WeightName> lnames, gnames;
  // ---- full-parameter SFT (train.full_finetune): every weight trains, no adapters (BASELINE.json configs[3]) ----
  // Weights live in ONE flat bf16 buffer - L layer blocks laid out by lslots, then a globals block laid out by gslots, each
  // padded to a multiple of world * 128 elements - with a gradient buffer of the same layout.  Rank r owns elements
  // [r, r + 1) * block / world of every block: the block's bf16 gradients are reduce-scattered in place (NCCL, on a side
  // stream, as soon as the backward pass has finished the layer), the fp32 master weights and Adam moments exist for the
  // owned slices only (ZeRO-1 style), and the updated bf16 slices are all-gathered in place.
  bool full = false;
  int64_t layer_elems = 0, glob_elems = 0;
  bf16 *w_flat = nullptr, *g_flat = nullptr;
  float *master = nullptr, *fm = nullptr, *fv = nullptr, *embed_g32 = nullptr, *ndw_scratch = nullptr;
  bool master_valid = false;
  bool rs_now = false;  // this backward pass ends an accumulation group: finished layers go to the reduce-scatter stream
  cudaStream_t comm_stream = nullptr;
  std::vector<cudaEvent_t> ev_layer;
  cudaEvent_t ev_comm = nullptr;
  // all-gather of the updated weights runs on the side stream, block by block in the order the NEXT forward pass needs them
  // (globals, layer 0, 1, ...); ag_pending[b] = the main stream has not yet been told to wait for block b (L = globals)
  std::vector<cudaEvent_t> ev_ag;
  std::vector<uint8_t> ag_pending;
  bool quant4 = false;
  bf16* scratch_w[4] = {nullptr, nullptr, nullptr, nullptr};  // dequantised wqkv / wo / wgu / wdown of the layer in flight
  cudaEvent_t ev_deq[4] = {nullptr, nullptr, nullptr, nullptr}, ev_scr[4] = {nullptr, nullptr, nullptr, nullptr};
  int deq_layer[4] = {-1, -1, -1, -1};       // layer whose matrix of that type sits (or is being expanded) in the scratch
  uint8_t deq_pending[4] = {0, 0, 0, 0};     // expansion launched on the side stream, main stream not yet told to wait
  int64_t base_bytes = 0;
  float2* rope_cs = nullptr;
  float2* rope_cs_t = nullptr;  // the same table transposed to [D/2][S]: coalesced when thread r needs position q0 + r (attention backward epilogues)
  int split_b = 1, split_a = 1;

  // which base tensors have been uploaded: one flag per row of gnames, then one per row of lnames for every layer; a step with a
  // hole in this map would train on uninitialised memory
  std::vector<uint8_t> loaded;
  bool all_random = false;
  bool have_lora = false;
  cudaEvent_t ev_fb = nullptr, ev_ar = nullptr;
  float seg_ms[4] = {0.f, 0.f, 0.f, 0.f};
  cudaStream_t copy_stream = nullptr;
  int micro_idx = 0;
  int opt_step = 0;
  int64_t launches = 0;
  float last_ms = 0.f;

  int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    err = buf;
    return code;
  }
  template <typename T>
  bool alloc(T** p, size_t n) {
    if (dry) {
      bytes_allocated += n * sizeof(T);
      *p = nullptr;
      return true;
    }
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, n * sizeof(T));
    if (e != cudaSuccess) {
      fail(DTX_ERR_CUDA, "cudaMalloc(%zu bytes) failed after %zu bytes: %s", n * sizeof(T), bytes_allocated,
           cudaGetErrorString(e));
      return false;
    }
    allocs.push_back(q);
    bytes_allocated += n * sizeof(T);
    *p = static_cast<T*>(q);
    return true;
  }
  void release(void* p, size_t bytes) {
    if (!p) return;
    for (size_t i = 0; i < allocs.size(); ++i)
      if (allocs[i] == p) {
        allocs[i] = allocs.back();
        allocs.pop_back();
        break;
      }
    cudaFree(p);
    bytes_allocated -= bytes;
  }
  // cudaMemset of a buffer create_buffers() just allocated (nothing in a sizing run)
  template <typename T>
  cudaError_t zero(T* p, size_t n) {
    return dry ? cudaSuccess : cudaMemset(p, 0, n * sizeof(T));
  }
  // full-parameter SFT: the gradient of weight element `w` (same layout as the weights)
  bf16* grad_of(const bf16* w) const { return g_flat + (w - w_flat); }
  // first base tensor that has not been loaded, or nullptr when the model is complete
  const char* missing_weight(char* buf, size_t n) const {
    if (all_random) return nullptr;
    const size_t G = gnames.size(), K = lnames.size();
    for (size_t i = 0; i < loaded.size(); ++i) {
      if (loaded[i]) continue;
      if (i < G) {
        snprintf(buf, n, "%s", gnames[i].hf);
        return buf;
      }
      const WeightName& w = lnames[(i - G) % K];
      if (w.gu == GU_BOTH) continue;  // a second name for the gate and up rows, which have flags of their own
      snprintf(buf, n, "model.layers.%zu.%s", (i - G) / K, w.key);
      return buf;
    }
    return nullptr;
  }
};

namespace {

#define CK(expr, nlaunch)                                                                        \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) return t->fail(DTX_ERR_CUDA, "%s: %s", #expr, cudaGetErrorString(_e)); \
    t->launches += (nlaunch);                                                                    \
  } while (0)

// checked copies / fills outside the hot loop (no launch counted)
#define CKM(expr)                                                                                \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) return t->fail(DTX_ERR_CUDA, "%s: %s", #expr, cudaGetErrorString(_e)); \
  } while (0)

// Host -> device copies of weights / adapters go through the TRAINER'S stream and are waited for: cudaMemcpy() from pageable
// memory returns once the data is staged - the DMA may still be in flight - and it runs on the legacy default stream, with
// which the trainer's non-blocking stream does not synchronise.  A kernel launched right behind it (the adapter shadow
// refresh) then read stale parameters: the first step after loading adapters from the host differed from run to run.
inline cudaError_t upload_sync(void* dst, const void* src, size_t bytes, cudaStream_t s) {
  cudaError_t e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s);
  if (e != cudaSuccess) return e;
  return cudaStreamSynchronize(s);
}

// key of the dropout masks of one (forward pass, layer): the per-element keep decision is
// splitmix64(key + target * 0x9E3779B97F4A7C15 + m * d + c) >> 40 >= p * 2^24  (restated in oracle/llama_lora.py)
uint64_t dropout_key(const dtx_trainer* t, int layer) {
  uint64_t x = t->tc.seed * 0xD1B54A32D192ED03ull + t->fwd_count * 0x100000001B3ull + static_cast<uint64_t>(layer) * 0x9E3779B1ull +
               static_cast<uint64_t>(t->rank) * 0xC2B2AE3D27D4EB4Full;
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

int pick_split(int n_sms, int m_tiles, int kb_total) {
  int s = (2 * n_sms + m_tiles - 1) / m_tiles;
  if (s < 1) s = 1;
  if (s > 16) s = 16;
  if (s > kb_total) s = kb_total;
  // every split must own at least one k-block
  while (s > 1 && (s - 1) * ((kb_total + s - 1) / s) >= kb_total) --s;
  return s;
}

// fp32 inverse frequencies of the rotary table (half = head_dim / 2 values) in HF's operation order, so that the table is bitwise
// the one transformers builds: the default type is 1 / theta^(2i/D) (powf), linear divides it by the factor
// (_compute_linear_scaling_rope_parameters), llama3 follows _compute_llama3_parameters - wavelen = 2 pi / inv_freq (torch
// evaluates a scalar over a tensor as reciprocal times scalar), wavelengths below original_max_pos / high_freq_factor keep their
// frequency, those above original_max_pos / low_freq_factor are divided by the factor, the band between is interpolated.
// GLM (ext.rope_glm) rotates the first rotary_dim = head_dim / 2 dims only: GlmRotaryEmbedding builds theta^(-2i/rotary_dim).
int rope_rotary_dim(const dtx_model_cfg& mc, const dtx_model_ext& ext) { return ext.rope_glm ? mc.head_dim / 2 : mc.head_dim; }
void rope_inv_freq(const dtx_model_cfg& mc, const dtx_model_ext& ext, float* out) {
  const int rd = rope_rotary_dim(mc, ext), half = rd / 2;
  for (int i = 0; i < half; ++i) {
    const float base = 1.0f / powf(mc.rope_theta, static_cast<float>(2 * i) / static_cast<float>(rd));
    float f = base;
    if (ext.rope_type == DTX_ROPE_LINEAR) {
      f = base / ext.rope_factor;
    } else if (ext.rope_type == DTX_ROPE_LLAMA3) {
      const double old_len = ext.rope_original_max_pos;
      const float low_wavelen = static_cast<float>(old_len / ext.rope_low_freq_factor);
      const float high_wavelen = static_cast<float>(old_len / ext.rope_high_freq_factor);
      const float factor = ext.rope_factor;
      const float wavelen = (1.0f / base) * static_cast<float>(2.0 * M_PI);
      const float scaled = wavelen > low_wavelen ? base / factor : base;
      if (!(wavelen < high_wavelen) && !(wavelen > low_wavelen)) {
        const float smooth = ((1.0f / wavelen) * static_cast<float>(old_len) - ext.rope_low_freq_factor) /
                             static_cast<float>(static_cast<double>(ext.rope_high_freq_factor) - ext.rope_low_freq_factor);
        const float a = (1.0f - smooth) * scaled;
        const float b = smooth * scaled;
        f = a / factor + b;
      } else {
        f = scaled;
      }
    }
    out[i] = f;
  }
}

int create_buffers(dtx_trainer* t) {
  const dtx_model_cfg& mc = t->mc;
  const dtx_train_cfg& tc = t->tc;
  const size_t d = mc.hidden, F = mc.ffn, V = mc.vocab, L = mc.n_layers, M = t->M, RP = t->RP, W = t->W, KA = t->KA;
  const size_t dq = t->dq, QK = t->dq + t->dkv;  // attention width, q|k width
  bool ok = true;
  const bool full = t->full;
  if (full) {
    // one flat weight buffer + one flat gradient buffer; every block padded so that it splits evenly over the ranks
    const size_t unit = static_cast<size_t>(t->world) * 128;
    auto pad = [&](size_t n) { return (n + unit - 1) / unit * unit; };
    t->layer_elems = pad(t->layer_used);
    t->glob_elems = pad(t->glob_used);
    const size_t total = L * t->layer_elems + t->glob_elems, shard = total / t->world;
    ok = ok && t->alloc(&t->w_flat, total) && t->alloc(&t->g_flat, total);
    ok = ok && t->alloc(&t->master, shard) && t->alloc(&t->fm, shard) && t->alloc(&t->fv, shard);
    // the norms' weight-gradient partials: 64 rows of the widest normalised span (qk_norm_full: the q|k columns)
    ok = ok && t->alloc(&t->embed_g32, V * d) && t->alloc(&t->ndw_scratch, 64 * (t->ext.qk_norm_full ? std::max(d, QK) : d));
    if (!ok) return DTX_ERR_CUDA;
    CKM(t->zero(t->w_flat, total));
    CKM(t->zero(t->g_flat, total));
    CKM(t->zero(t->fm, shard));
    CKM(t->zero(t->fv, shard));
    bf16* gl = t->w_flat + L * t->layer_elems;
    for (const auto& s : t->gslots) t->*s.mem = gl + s.off;
    t->n_train = static_cast<int64_t>(L * t->layer_used + t->glob_used);
  } else {
    for (const auto& s : t->gslots) ok = ok && t->alloc(&(t->*s.mem), s.n);
    ok = ok && t->alloc(&t->a_cat_all, L * RP * KA) && t->alloc(&t->b_ext_all, L * W * RP);
    if (!ok) return DTX_ERR_CUDA;
    CKM(t->zero(t->a_cat_all, L * RP * KA));
    CKM(t->zero(t->b_ext_all, L * W * RP));
  }
  t->base_bytes = static_cast<int64_t>((t->glob_used + L * t->layer_used) * sizeof(bf16));
  t->loaded.assign(t->gnames.size() + L * t->lnames.size(), 0);
  t->layers.resize(L);
  t->xs.resize(L + 1);
  for (size_t l = 0; l <= L; ++l) ok = ok && t->alloc(&t->xs[l], M * d);
  for (size_t l = 0; l < L && ok; ++l) {
    Layer& y = t->layers[l];
    if (full) {
      for (const auto& s : t->lslots) y.*s.mem = t->w_flat + l * t->layer_elems + s.off;
    } else {
      for (const auto& s : t->lslots) ok = ok && t->alloc(&(y.*s.mem), s.n);
      y.a_cat = t->a_cat_all + l * RP * KA;
      y.b_ext = t->b_ext_all + l * W * RP;
    }
    if (t->recompute == RECOMPUTE_LAYER && l > 0) {  // one saved set, refilled layer by layer
      const Layer& y0 = t->layers[0];
      y.h1 = y0.h1; y.t = y0.t; y.hd = y0.hd; y.qkv = y0.qkv; y.attn = y0.attn; y.x_mid = y0.x_mid; y.gu = y0.gu;
      y.qk_pre = y0.qk_pre;
      y.o_pre = y0.o_pre; y.down_pre = y0.down_pre; y.rstd_pn1 = y0.rstd_pn1; y.rstd_pn2 = y0.rstd_pn2;
      y.lse = y0.lse; y.rstd1 = y0.rstd1; y.rstd2 = y0.rstd2;
      continue;
    }
    if (!full) ok = ok && t->alloc(&y.t, M * RP);
    const bool pre_norms = !t->ext.no_pre_norms;  // else the sublayers read xs[l] / x_mid: no h1, rstd1, rstd2
    if (pre_norms) ok = ok && t->alloc(&y.h1, M * d);
    ok = ok && t->alloc(&y.qkv, M * W) && t->alloc(&y.attn, M * dq) && t->alloc(&y.x_mid, M * d) && t->alloc(&y.gu, M * 2 * F);
    if (t->ext.qk_norm || t->ext.qk_norm_full) ok = ok && t->alloc(&y.qk_pre, M * QK);
    if (t->ext.post_norms)
      ok = ok && t->alloc(&y.o_pre, M * d) && t->alloc(&y.down_pre, M * d) && t->alloc(&y.rstd_pn1, M) && t->alloc(&y.rstd_pn2, M);
    if (t->dropout) ok = ok && t->alloc(&y.hd, M * KA);
    ok = ok && t->alloc(&y.lse, static_cast<size_t>(tc.micro_batch) * mc.n_heads * tc.seq_len);
    if (pre_norms) ok = ok && t->alloc(&y.rstd1, M) && t->alloc(&y.rstd2, M);
  }
  if (!ok) return DTX_ERR_CUDA;
  if (!full) {
    ok = ok && t->alloc(&t->params, t->n_train) && t->alloc(&t->grads, t->n_train) && t->alloc(&t->adam_m, t->n_train) &&
         t->alloc(&t->adam_v, t->n_train);
    if (!ok) return DTX_ERR_CUDA;
    CKM(t->zero(t->params, t->n_train));
    CKM(t->zero(t->grads, t->n_train));
    CKM(t->zero(t->adam_m, t->n_train));
    CKM(t->zero(t->adam_v, t->n_train));
  }
  ok = ok && t->alloc(&t->h2, M * d) && t->alloc(&t->act, M * F) && t->alloc(&t->dact, M * F) && t->alloc(&t->dgu, M * 2 * F) &&
       t->alloc(&t->dx_a, M * d) && t->alloc(&t->dx_b, M * d) && t->alloc(&t->dh, M * d) && t->alloc(&t->dattn, M * dq) &&
       t->alloc(&t->dqkv, M * W) && (full || t->alloc(&t->dt, M * RP)) && t->alloc(&t->dlogits, M * V) && t->alloc(&t->logits, M * V) &&
       t->alloc(&t->rstdf, M) && t->alloc(&t->row_loss, M) &&
       t->alloc(&t->delta, static_cast<size_t>(tc.micro_batch) * mc.n_heads * tc.seq_len);
  const int kb_tok = (static_cast<int>(M) + 63) / 64;
  t->split_b = pick_split(t->n_sms, (static_cast<int>(W) + 127) / 128, kb_tok);
  t->split_a = pick_split(t->n_sms, (static_cast<int>(KA) + 127) / 128, kb_tok);
  if (!full)
    ok = ok && t->alloc(&t->part_b, static_cast<size_t>(t->split_b) * W * RP) &&
         t->alloc(&t->part_a, static_cast<size_t>(t->split_a) * KA * RP);
  if (t->dropout) ok = ok && t->alloc(&t->glora, M * KA);
  ok = ok && t->alloc(&t->d_loss, 4) && t->alloc(&t->d_sumsq, 4) && t->alloc(&t->d_gnorm, 4) && t->alloc(&t->d_scratch, 1024);
  ok = ok && t->alloc(&t->d_ids, M) && t->alloc(&t->d_labels, M) && t->alloc(&t->d_shift, M) && t->alloc(&t->d_nvalid, 4);
  ok = ok && t->alloc(&t->d_row_map, M) && t->alloc(&t->d_valid_idx, M);
  ok = ok && t->alloc(&t->d_ids_full, M) && t->alloc(&t->d_labels_full, M) && t->alloc(&t->d_lens_full, static_cast<size_t>(tc.micro_batch)) &&
       t->alloc(&t->d_pos, M) && t->alloc(&t->d_row_start, static_cast<size_t>(tc.micro_batch) + 1);
  ok = ok && t->alloc(&t->d_seq_lens, static_cast<size_t>(tc.micro_batch)) && t->alloc(&t->d_row_sum, static_cast<size_t>(tc.micro_batch)) &&
       t->alloc(&t->d_row_valid, static_cast<size_t>(tc.micro_batch)) && t->alloc(&t->d_host_red, 64);
  const int rope_half = rope_rotary_dim(mc, t->ext) / 2;
  ok = ok && t->alloc(&t->rope_cs, static_cast<size_t>(tc.seq_len) * rope_half);
  ok = ok && t->alloc(&t->rope_cs_t, static_cast<size_t>(tc.seq_len) * rope_half);
  if (!ok) return DTX_ERR_CUDA;
  if (t->dry) return DTX_OK;
  // rotary table in double precision (HF LlamaRotaryEmbedding; inverse frequencies of the model's rope type)
  {
    const int half = rope_half;
    std::vector<float> inv_freq(half);
    rope_inv_freq(mc, t->ext, inv_freq.data());
    std::vector<float2> cs(static_cast<size_t>(tc.seq_len) * half);
    for (int pos = 0; pos < tc.seq_len; ++pos)
      for (int i = 0; i < half; ++i) {
        // HF computes inv_freq and the angle in fp32; reproduce that rounding, then take cos/sin accurately
        const float ang = static_cast<float>(pos) * inv_freq[i];
        cs[static_cast<size_t>(pos) * half + i] = make_float2(static_cast<float>(cos(static_cast<double>(ang))),
                                                              static_cast<float>(sin(static_cast<double>(ang))));
      }
    CKM(cudaMemcpy(t->rope_cs, cs.data(), cs.size() * sizeof(float2), cudaMemcpyHostToDevice));
    std::vector<float2> cst(cs.size());
    for (int pos = 0; pos < tc.seq_len; ++pos)
      for (int i = 0; i < half; ++i) cst[static_cast<size_t>(i) * tc.seq_len + pos] = cs[static_cast<size_t>(pos) * half + i];
    CKM(cudaMemcpy(t->rope_cs_t, cst.data(), cst.size() * sizeof(float2), cudaMemcpyHostToDevice));
  }
  return DTX_OK;
}

int refresh_shadows(dtx_trainer* t) {
  ShadowArgs a;
  a.params = t->params;
  a.a_cat = t->a_cat_all;
  a.b_ext = t->b_ext_all;
  a.L = t->mc.n_layers;
  a.d = t->mc.hidden;
  a.r = t->tc.lora_r;
  a.RP = t->RP;
  a.nt = t->nt;
  a.KA = t->KA;
  a.W = t->W;
  a.a_split = t->dropout ? 1 : 0;
  a.per_layer = t->per_layer;
  for (int i = 0; i < 3; ++i) a.tg[i] = t->tg[i];
  a.scale = t->tc.lora_alpha / static_cast<float>(t->tc.lora_r);
  long long total = t->n_train;
  int grid = static_cast<int>((total + 255) / 256);
  if (grid > 132 * 8) grid = 132 * 8;
  lora_shadow_kernel<<<grid, 256, 0, t->stream>>>(a);
  CK(cudaGetLastError(), 1);
  return DTX_OK;
}

// Frozen base weight `which` of layer l for the next GEMM.  bf16-resident: the pointer.  --quantization int4: the packed NF4
// codes are expanded into the per-trainer scratch of that matrix type (HBM-bound: 0.56 B read + 2 B written per weight, ~85 us
// per layer of a 7B model and direction) - the values are exactly bitsandbytes' dequantize_4bit output, so the GEMM sees what
// the reference's 4-bit matmul multiplies with.  The expansion of the NEXT matrix in program order is launched on a side
// stream as soon as the current one is handed out: its small CTAs (no shared memory) co-reside with the persistent GEMM
// CTAs and use HBM bandwidth the tensor-bound GEMM leaves idle, so that the expansion disappears from the critical path.
int nf4_expand(dtx_trainer* t, int l, int which, cudaStream_t s) {
  Layer& y = t->layers[l];
  for (const auto& sl : t->lslots)
    if (sl.nf4 == which) CK(nf4_dequant_bf16(y.q4[which], y.absmax[which], t->scratch_w[which], sl.n, s), 1);
  return DTX_OK;
}
// next (layer, matrix) the step will ask for after (l, which) in `phase` (PH_*), when it can be expanded ahead: always a
// different matrix type than `which`, whose scratch the GEMM about to be launched reads.  A wrong guess is not merely slow:
// the main stream would expand the mismatched matrix inline while the side stream may still be writing the same scratch.
bool next_weight(const dtx_trainer* t, int l, int which, int phase, bool will_backward, int* nl, int* nw) {
  const int L = t->mc.n_layers;
  if (phase == PH_FWD) {  // forward order: qkv, o, gu, down
    if (which < W_DOWN) { *nl = l; *nw = which + 1; return true; }
    if (l + 1 < L) { *nl = l + 1; *nw = W_QKV; return true; }
    if (will_backward) { *nl = L - 1; *nw = W_DOWN; return true; }
    return false;
  }
  if (phase == PH_RECOMPUTE) {  // qkv, o, gu (the down-projection is not re-run), then the same layer's backward
    *nl = l;
    *nw = which < W_GU ? which + 1 : W_DOWN;
    return true;
  }
  // backward order: down, gu, o, qkv (layer 0's qkv is never asked for: no consumer of its input gradient)
  if (which > W_QKV) {
    if (which - 1 == W_QKV && l == 0) return false;
    *nl = l; *nw = which - 1; return true;
  }
  // With per-layer recompute the layer below starts with its own q|k|v GEMM: the scratch the GEMM about to be launched reads
  // (the prefetch is issued before that launch), so it cannot be expanded ahead; base_weight expands it inline behind that GEMM.
  if (t->recompute == RECOMPUTE_LAYER) return false;
  if (l - 1 >= 0) { *nl = l - 1; *nw = W_DOWN; return true; }
  return false;
}
int base_weight(dtx_trainer* t, int l, int which, int phase, bool will_backward, const bf16** out) {
  Layer& y = t->layers[l];
  bf16* res[4] = {y.wqkv, y.wo, y.wgu, y.wdown};
  if (!t->quant4) {
    *out = res[which];
    return DTX_OK;
  }
  if (t->deq_layer[which] == l) {  // already in the scratch (the frozen weights never change), or on its way there
    if (t->deq_pending[which]) CKM(cudaStreamWaitEvent(t->stream, t->ev_deq[which], 0));
  } else {
    int rc = nf4_expand(t, l, which, t->stream);
    if (rc) return rc;
  }
  t->deq_pending[which] = 0;
  t->deq_layer[which] = l;
  *out = t->scratch_w[which];
  int nl, nw;
  if (t->copy_stream && next_weight(t, l, which, phase, will_backward, &nl, &nw) && t->deq_layer[nw] != nl) {
    // the scratch of type nw was last read by a GEMM launched earlier on the main stream: order the overwrite behind it
    CKM(cudaEventRecord(t->ev_scr[nw], t->stream));
    CKM(cudaStreamWaitEvent(t->copy_stream, t->ev_scr[nw], 0));
    int rc = nf4_expand(t, nl, nw, t->copy_stream);
    if (rc) return rc;
    CKM(cudaEventRecord(t->ev_deq[nw], t->copy_stream));
    t->deq_pending[nw] = 1;
    t->deq_layer[nw] = nl;
  }
  return DTX_OK;
}
#define BASEW(which, ptr)                                                        \
  const bf16* ptr = nullptr;                                                     \
  do {                                                                           \
    int _rc = base_weight(t, l, which, phase, backward, &ptr);                   \
    if (_rc) return _rc;                                                         \
  } while (0)

// full-parameter SFT, world > 1: the updated weights of block b (L = globals) are being all-gathered on the side stream;
// make the main stream wait for it right before the block's first use
inline void wait_weights(dtx_trainer* t, int b) {
  if (!t->ag_pending.empty() && t->ag_pending[b]) {
    cudaStreamWaitEvent(t->stream, t->ev_ag[b], 0);
    t->ag_pending[b] = 0;
  }
}
inline void wait_all_weights(dtx_trainer* t) {
  for (size_t b = 0; b < t->ag_pending.size(); ++b) wait_weights(t, static_cast<int>(b));
}

// full-parameter SFT, world > 1: reduce-scatter one gradient block in place on the side stream once the main stream has
// produced it (event), so that the transfer overlaps the rest of the backward pass
int reduce_scatter_block(dtx_trainer* t, bf16* block, int64_t elems, int ev_idx) {
  NcclApi* api = nccl_api();
  if (!api || !api->ReduceScatter || !t->nccl_comm) return t->fail(DTX_ERR_NCCL, "ncclReduceScatter unavailable for world=%d", t->world);
  cudaEvent_t ev = t->ev_layer[ev_idx];
  CKM(cudaEventRecord(ev, t->stream));
  CKM(cudaStreamWaitEvent(t->comm_stream, ev, 0));
  const int64_t shard = elems / t->world;
  int rc = api->ReduceScatter(block, block + static_cast<int64_t>(t->rank) * shard, static_cast<size_t>(shard), kNcclBfloat16, kNcclSum,
                              t->nccl_comm, t->comm_stream);
  if (rc != 0) return t->fail(DTX_ERR_NCCL, "ncclReduceScatter failed: %s", api->GetErrorString ? api->GetErrorString(rc) : "?");
  t->launches += 1;
  return DTX_OK;
}

// RoPE / SwiGLU run in the GEMM and attention epilogues: the switch is on and the batch fills whole 256-column tiles
bool use_fused(const dtx_trainer* t) {
  return g_fused_epilogues && t->cur_M > 128 && ((t->dq + t->dkv) % 256 == 0) && (t->W % 256 == 0);
}

// Forward of decoder layer l from xs[l]: fills the layer's saved activations (h1, hd, t, qkv, attn, lse, rstd1, x_mid, rstd2, gu)
// and, in the forward pass proper (phase PH_FWD), xs[l + 1].  The per-layer recompute of the backward pass (PH_RECOMPUTE) runs
// the very same launches - same epilogues, unfused fallbacks, packed / ragged arguments and dropout key (fwd_count is not
// advanced) - so that the refilled activations are bitwise the ones the forward pass wrote; only the down-projection, whose
// output xs[l + 1] is kept and not needed again, is skipped.
int layer_fwd(dtx_trainer* t, int l, int phase, bool backward) {
  const dtx_model_cfg& mc = t->mc;
  const dtx_train_cfg& tc = t->tc;
  const int d = mc.hidden, F = mc.ffn, M = t->cur_M, RP = t->RP, H = mc.n_heads, D = mc.head_dim;
  const int Hkv = mc.n_kv_heads, W = t->W, dq = t->dq, QK = t->dq + t->dkv;
  const int B = t->cur_B, S = t->cur_S;
  const int32_t* seq_lens = t->use_seq_lens ? t->d_seq_lens : nullptr;
  cudaStream_t s = t->stream;
  const float att_scale = 1.0f / sqrtf(static_cast<float>(D));
  const bool fused = use_fused(t);
  const bool lora = !t->full;
  const bool drop = lora && t->dropout;  // adapters laid out for per-target dropped inputs (KA = nt*d)
  const float p_drop = backward ? tc.lora_dropout : 0.f;  // eval (model.eval()) runs the same path with p = 0
  Layer& y = t->layers[l];
  const bf16* qk_wq = y.qkn;  // q_norm | k_norm (Qwen3), else null
  const bf16* qk_wk = y.qkn ? y.qkn + D : nullptr;
  const bool pre_norms = !t->ext.no_pre_norms;  // else (OLMo-2) the sublayers read the residual stream itself
  const bf16* h1 = pre_norms ? y.h1 : t->xs[l];
  wait_weights(t, l);
  if (pre_norms) CK(rmsnorm_fwd(t->xs[l], y.norm1, y.h1, y.rstd1, M, d, mc.rms_eps, s), 1);
  const bf16* lora_in = h1;
  if (drop) {  // peft: lora_A(lora_dropout(x)) with one nn.Dropout per wrapped module -> one dropped copy per target
    CK(lora_dropout_fwd(h1, y.hd, M, d, t->nt, p_drop, dropout_key(t, l), s), 1);
    lora_in = y.hd;
  }
  if (lora) {  // LoRA down-projection of all targets at once: t = lora_in * A_cat^T   [M, RP]
    GemmArgs g;
    g.A = lora_in; g.lda = t->KA; g.B = y.a_cat; g.ldb = t->KA; g.C = y.t; g.ldc = RP;
    g.M = M; g.N = RP; g.K = t->KA; g.epilogue = EPI_BF16; g.block_n = 64;
    CK(gemm_bf16(g, s), 1);
  }
  {  // qkv = h1 * Wqkv^T + t * B_ext^T : base projection and LoRA up-projection in one accumulator
    BASEW(W_QKV, wqkv);
    GemmArgs g;
    g.A = h1; g.lda = d; g.B = wqkv; g.ldb = d;
    if (lora) { g.A2 = y.t; g.lda2 = RP; g.B2 = y.b_ext; g.ldb2 = RP; g.K2 = RP; }
    g.C = y.qkv; g.ldc = W; g.M = M; g.N = W; g.K = d; g.epilogue = EPI_BF16;
    g.bias = y.bias;  // q|k|v biases (Qwen2): added to the accumulator before the rounding / the rotary
    // rotary embedding of q and k applied to the fp32 accumulator in the epilogue; not with OLMo-2's full-width q/k norm, whose
    // sums span more columns than a tile: its own pass below does norm + rotary
    if (fused && !y.qkf) {
      g.epilogue = EPI_ROPE; g.rope_cs = t->rope_cs; g.rope_S = S; g.rope_cols = t->dq + t->dkv;
      g.rope_pos = t->packed ? t->d_pos : nullptr;  // packed batch: a row's position is its offset inside its own sequence
      if (qk_wq) {  // q/k norm (Qwen3) before the rotary; the pre-norm q|k is saved for the backward pass
        g.qk_wq = qk_wq; g.qk_wk = qk_wk; g.qk_q_cols = dq; g.qk_eps = mc.rms_eps; g.aux = y.qk_pre; g.ld_aux = QK;
      }
      g.rope_glm = t->rope_glm ? 1 : 0;
    }
    CK(gemm_bf16(g, s), 1);
  }
  if (!fused && t->packed) return t->fail(DTX_ERR_STATE, "packed batches need the fused RoPE epilogue");
  if (y.qkf)  // q|k = rotary(norm(q|k)) in place, the GEMM's bf16 q|k saved for the backward pass
    CK(qk_norm_full_rope_fwd(y.qkv, W, M, dq, QK, y.qkf, y.qkf + dq, mc.rms_eps, t->rope_cs, S, t->packed ? t->d_pos : nullptr, y.qk_pre,
                             QK, s), 1);
  else if (!fused && qk_wq) CK(qk_norm_fwd(y.qkv, W, M, dq, QK, qk_wq, qk_wk, mc.rms_eps, y.qk_pre, QK, s), 1);
  if (!fused && t->rope_glm) CK(rope_glm_qk_inplace(y.qkv, t->rope_cs, B, S, H + Hkv, W, 0, s), 1);
  else if (!fused && !y.qkf) CK(rope_qk_inplace_table(y.qkv, t->rope_cs, B, S, H + Hkv, W, D, 0, s), 1);
  {
    AttnArgs a;
    a.qkv = y.qkv; a.out = y.attn; a.lse = y.lse; a.B = B; a.S = S; a.H = H; a.Hkv = Hkv; a.scale = att_scale;
    a.seq_lens = seq_lens; a.window = t->window;
    if (t->packed) { a.row_start = t->d_row_start; a.total_rows = M; }
    CK(attn_fwd(a, s), 1);
  }
  {  // x_mid = x + attn * Wo^T   (post_norms: x_mid = x + post_self_attn_layernorm(o_pre), o_pre = attn * Wo^T)
    BASEW(W_O, wo);
    GemmArgs g;
    g.A = y.attn; g.lda = dq; g.B = wo; g.ldb = dq; g.C = y.x_mid; g.ldc = d; g.R = t->xs[l]; g.ldr = d;
    g.M = M; g.N = d; g.K = dq; g.epilogue = EPI_BF16_ADD;
    if (y.pn) { g.C = y.o_pre; g.R = nullptr; g.ldr = 0; g.epilogue = EPI_BF16; }
    CK(gemm_bf16(g, s), 1);
  }
  if (y.pn) CK(post_norm_add(y.o_pre, y.pn, t->xs[l], y.x_mid, y.rstd_pn1, M, d, mc.rms_eps, s), 1);
  if (pre_norms) CK(rmsnorm_fwd(y.x_mid, y.norm2, t->h2, y.rstd2, M, d, mc.rms_eps, s), 1);
  {  // [gate | up] = h2 * Wgu^T  (no_pre_norms: x_mid * Wgu^T)
    BASEW(W_GU, wgu);
    GemmArgs g;
    g.A = pre_norms ? t->h2 : y.x_mid; g.lda = d; g.B = wgu; g.ldb = d; g.C = y.gu; g.ldc = 2 * F;
    g.M = M; g.N = 2 * F; g.K = d; g.epilogue = EPI_BF16;
    if (fused) {  // silu(gate) * up computed from the accumulator tile ([gate 128 | up 128] interleaved layout)
      g.epilogue = EPI_SWIGLU_FWD; g.aux = t->act; g.ld_aux = F;
    }
    CK(gemm_bf16(g, s), 1);
  }
  if (!fused) CK(swiglu_fwd(y.gu, t->act, M, F, 1, s), 1);
  // x_next = x_mid + act * Wdown^T   (post_norms: x_next = x_mid + post_mlp_layernorm(down_pre), down_pre = act * Wdown^T; the
  // recompute refills down_pre and its rstd, which the backward pass needs, and leaves the kept x_next alone)
  if (phase == PH_FWD || y.pn) {
    BASEW(W_DOWN, wdown);
    GemmArgs g;
    g.A = t->act; g.lda = F; g.B = wdown; g.ldb = F; g.C = t->xs[l + 1]; g.ldc = d; g.R = y.x_mid; g.ldr = d;
    g.M = M; g.N = d; g.K = F; g.epilogue = EPI_BF16_ADD;
    if (y.pn) { g.C = y.down_pre; g.R = nullptr; g.ldr = 0; g.epilogue = EPI_BF16; }
    CK(gemm_bf16(g, s), 1);
  }
  if (y.pn)
    CK(post_norm_add(y.down_pre, y.pn + d, y.x_mid, phase == PH_FWD ? t->xs[l + 1] : nullptr, y.rstd_pn2, M, d, mc.rms_eps, s), 1);
  return DTX_OK;
}

// forward (+ backward) of one micro-batch whose ids / labels (/ row lengths) are already in t->d_ids / t->d_labels (/ t->d_seq_lens).
// The batch is [micro_batch, cur_S]: cur_S <= seq_len is this batch's own padded length (DataCollatorForSeq2Seq pads to the
// longest row of the batch, cmd/tuning/train.py:282-286); every buffer was sized for seq_len.
int fwd_bwd(dtx_trainer* t, bool backward) {
  const dtx_model_cfg& mc = t->mc;
  const dtx_train_cfg& tc = t->tc;
  const int d = mc.hidden, F = mc.ffn, V = mc.vocab, L = mc.n_layers, M = t->cur_M, RP = t->RP, H = mc.n_heads, D = mc.head_dim;
  const int Hkv = mc.n_kv_heads, W = t->W, dq = t->dq, QK = t->dq + t->dkv;
  const int B = t->cur_B, S = t->cur_S;
  const int32_t* seq_lens = t->use_seq_lens ? t->d_seq_lens : nullptr;
  const int kb_tok = (M + 63) / 64;
  const int split_b = std::min(t->split_b, pick_split(gemm_num_sms(), (W + 127) / 128, kb_tok));
  const int split_a = std::min(t->split_a, pick_split(gemm_num_sms(), (t->KA + 127) / 128, kb_tok));
  cudaStream_t s = t->stream;
  const float att_scale = 1.0f / sqrtf(static_cast<float>(D));
  const bool fused = use_fused(t);
  const bool lora = !t->full;    // full-parameter SFT: no adapters, every weight gets a gradient
  int phase = PH_FWD;            // which part of the step asks for a base weight (prefetch order of the NF4 expansion)
  const bool drop = lora && t->dropout;  // adapters laid out for per-target dropped inputs (KA = nt*d)
  const float p_drop = backward ? tc.lora_dropout : 0.f;  // eval (model.eval()) runs the same path with p = 0
  t->fwd_count += 1;

  wait_weights(t, L);  // globals (embedding, lm_head, final norm)
  CK(embedding_fwd(t->d_ids, t->embed, t->xs[0], M, d, V, s), 1);
  for (int l = 0; l < L; ++l) {
    int rc = layer_fwd(t, l, PH_FWD, backward);
    if (rc) return rc;
  }
  // lm_head, CE and their backward only over the tokens that carry a label (shifted label >= 0): prompt tokens and padding
  // (27 % of the synthetic batch, far more on real instruction data) have zero loss and zero gradient.  The labelled rows
  // are compacted by the final norm (row map from an ordered scan inside shift_labels), the two lm_head GEMMs take the row
  // count from device memory and skip the dead 256-row tiles, the norm backward scatters the gradient back.
  // (full-parameter SFT keeps every row: the lm_head weight gradient contracts over tokens, and its operands must then be zero
  // - not stale - on the unlabelled rows)
  int32_t* row_map = lora ? t->d_row_map : nullptr;
  int32_t* valid_idx = lora ? t->d_valid_idx : nullptr;
  const int32_t* m_eff = lora ? t->d_nvalid : nullptr;
  if (t->packed) CK(shift_labels(t->d_labels, t->d_shift, t->d_nvalid, 1, M, s, row_map, valid_idx, t->d_pos), 1);
  else CK(shift_labels(t->d_labels, t->d_shift, t->d_nvalid, B, S, s, row_map, valid_idx), 1);
  CK(rmsnorm_fwd(t->xs[L], t->normf, t->h2, t->rstdf, M, d, mc.rms_eps, s, row_map), 1);
  {  // fp32 logits (the reference patches lm_head to return fp32: cmd/tuning/train.py:256-264)
    GemmArgs g;
    g.A = t->h2; g.lda = d; g.B = t->lm_head; g.ldb = d; g.C = t->logits; g.ldc = V;
    g.M = M; g.N = V; g.K = d; g.epilogue = EPI_F32; g.m_eff = m_eff;
    CK(gemm_bf16(g, s), 1);
  }
  CKM(cudaMemsetAsync(t->row_loss, 0, static_cast<size_t>(M) * sizeof(float), s));
  // one length group of a ragged micro-batch (t->sub_ndiv > 0): the token mean runs over the labelled tokens of all its groups
  CK(cross_entropy_fwd_bwd(t->logits, V, t->d_shift, t->d_nvalid, t->row_loss, backward ? t->dlogits : nullptr, V, M, V, s, valid_idx,
                           t->sub_ndiv), 1);
  CK(loss_reduce(t->row_loss, t->d_nvalid, t->d_loss, M, s, t->sub_ndiv, t->sub_accum ? 1 : 0), 1);
  if (!backward) return DTX_OK;
  phase = PH_BWD;

  const int accumulate = (t->micro_idx > 0 || t->sub_accum) ? 1 : 0;
  // weight gradient of a Linear: dW[out, in] (+)= dY^T X - a token-contraction GEMM with both operands MN-major
  auto dw_gemm = [&](const bf16* dY, int n_out, const bf16* X, int n_in, bf16* dW) -> cudaError_t {
    GemmArgs g;
    g.A = dY; g.lda = n_out; g.a_mn_major = 1; g.B = X; g.ldb = n_in; g.b_mn_major = 1;
    g.C = dW; g.ldc = n_in; g.M = n_out; g.N = n_in; g.K = M;
    g.epilogue = accumulate ? EPI_BF16_ADD : EPI_BF16; g.R = accumulate ? dW : nullptr; g.ldr = n_in;
    return gemm_bf16(g, s);
  };
  if (t->full) {  // lm_head weight gradient (h2 still holds the final-norm output) and the final norm's weight gradient
    CK(dw_gemm(t->dlogits, V, t->h2, d, t->grad_of(t->lm_head)), 1);
  }
  {  // d h_f = dlogits * W_lm  (compact rows in LoRA mode)
    GemmArgs g;
    g.A = t->dlogits; g.lda = V; g.B = t->lm_head; g.ldb = d; g.b_mn_major = 1; g.C = t->dh; g.ldc = d;
    g.M = M; g.N = d; g.K = V; g.epilogue = EPI_BF16; g.m_eff = m_eff;
    CK(gemm_bf16(g, s), 1);
  }
  if (t->full) CK(rmsnorm_dw(t->dh, t->xs[L], t->rstdf, M, d, t->ndw_scratch, t->grad_of(t->normf), accumulate, s), 2);
  CK(rmsnorm_bwd(t->dh, t->xs[L], t->normf, t->rstdf, nullptr, t->dx_a, M, d, s, row_map), 1);
  bf16* cur = t->dx_a;
  bf16* other = t->dx_b;
  for (int l = L - 1; l >= 0; --l) {
    if (t->recompute == RECOMPUTE_LAYER && l < L - 1) {  // refill the shared saved set (the last layer's is still there)
      int rc = layer_fwd(t, l, PH_RECOMPUTE, backward);
      if (rc) return rc;
    }
    Layer& y = t->layers[l];
    const bool pre_norms = !t->ext.no_pre_norms;  // else the sublayers read xs[l] / x_mid: no norm backward, the residual
                                                  // gradients are added in the dh2 / dh1 GEMMs' epilogues
    const bf16* h1 = pre_norms ? y.h1 : t->xs[l];
    const bf16* d_down = cur;  // gradient of the down-projection output
    if (y.pn) {  // through post_mlp_layernorm: d down_pre into dh (free until the dh2 GEMM below); full SFT: its weight gradient
      if (t->full) CK(rmsnorm_dw(cur, y.down_pre, y.rstd_pn2, M, d, t->ndw_scratch, t->grad_of(y.pn + d), accumulate, s), 2);
      CK(rmsnorm_bwd(cur, y.down_pre, y.pn + d, y.rstd_pn2, nullptr, t->dh, M, d, s), 1);
      d_down = t->dh;
    }
    if (t->full) {  // dWdown = d x_out^T * act: act = silu(gate) * up is recomputed from the saved gate|up (one HBM-bound pass)
      CK(swiglu_fwd(y.gu, t->act, M, F, 1, s), 1);
      CK(dw_gemm(d_down, d, t->act, F, t->grad_of(y.wdown)), 1);
    }
    {  // dact = dx * Wdown ; fused: d[gate|up] straight from the accumulator, dact never touches HBM
      BASEW(W_DOWN, wdown);
      GemmArgs g;
      g.A = d_down; g.lda = d; g.B = wdown; g.ldb = F; g.b_mn_major = 1; g.C = t->dact; g.ldc = F;
      g.M = M; g.N = F; g.K = d; g.epilogue = EPI_BF16;
      if (fused) {
        g.epilogue = EPI_SWIGLU_BWD; g.C = t->dgu; g.ldc = 2 * F; g.aux = y.gu; g.ld_aux = 2 * F;
      }
      CK(gemm_bf16(g, s), 1);
    }
    if (!fused) CK(swiglu_bwd(t->dact, y.gu, t->dgu, M, F, 1, s), 1);
    {  // dh2 = [dgate | dup] * [Wg ; Wu]  (no_pre_norms: other = d x_mid = d x_next + [dgate | dup] * [Wg ; Wu])
      BASEW(W_GU, wgu);
      GemmArgs g;
      g.A = t->dgu; g.lda = 2 * F; g.B = wgu; g.ldb = d; g.b_mn_major = 1; g.C = t->dh; g.ldc = d;
      g.M = M; g.N = d; g.K = 2 * F; g.epilogue = EPI_BF16;
      if (!pre_norms) { g.C = other; g.R = cur; g.ldr = d; g.epilogue = EPI_BF16_ADD; }
      CK(gemm_bf16(g, s), 1);
    }
    if (t->full && !pre_norms) CK(dw_gemm(t->dgu, 2 * F, y.x_mid, d, t->grad_of(y.wgu)), 1);  // dWgu = d[gate|up]^T * x_mid
    if (t->full && pre_norms) {  // dWgu = d[gate|up]^T * h2 (h2 = norm2(x_mid) recomputed) and the norm's own weight gradient
      CK(rmsnorm_fwd(y.x_mid, y.norm2, t->h2, nullptr, M, d, mc.rms_eps, s), 1);
      CK(dw_gemm(t->dgu, 2 * F, t->h2, d, t->grad_of(y.wgu)), 1);
      CK(rmsnorm_dw(t->dh, y.x_mid, y.rstd2, M, d, t->ndw_scratch, t->grad_of(y.norm2), accumulate, s), 2);
    }
    if (pre_norms) CK(rmsnorm_bwd(t->dh, y.x_mid, y.norm2, y.rstd2, cur, other, M, d, s), 1);  // other = d x_mid
    const bf16* d_o = other;  // gradient of the o-projection output
    if (y.pn) {  // through post_self_attn_layernorm: d o_pre into dh (free until the dh1 GEMM below)
      if (t->full) CK(rmsnorm_dw(other, y.o_pre, y.rstd_pn1, M, d, t->ndw_scratch, t->grad_of(y.pn), accumulate, s), 2);
      CK(rmsnorm_bwd(other, y.o_pre, y.pn, y.rstd_pn1, nullptr, t->dh, M, d, s), 1);
      d_o = t->dh;
    }
    {  // dattn = dx_mid * Wo
      BASEW(W_O, wo);
      GemmArgs g;
      g.A = d_o; g.lda = d; g.B = wo; g.ldb = dq; g.b_mn_major = 1; g.C = t->dattn; g.ldc = dq;
      g.M = M; g.N = dq; g.K = d; g.epilogue = EPI_BF16;
      CK(gemm_bf16(g, s), 1);
    }
    if (t->full) CK(dw_gemm(d_o, d, y.attn, dq, t->grad_of(y.wo)), 1);  // dWo = d x_mid^T * attn
    {
      AttnArgs a;
      a.qkv = y.qkv; a.out = y.attn; a.lse = y.lse; a.B = B; a.S = S; a.H = H; a.Hkv = Hkv; a.scale = att_scale;
      a.dout = t->dattn; a.dqkv = t->dqkv; a.delta = t->delta;
      a.seq_lens = seq_lens; a.window = t->window; a.rope_stride = tc.seq_len;
      if (t->packed) { a.row_start = t->d_row_start; a.total_rows = M; }
      // The dQ / dK kernels apply the inverse rotary in their store epilogues from the TRANSPOSED table (thread r of a tile
      // reads position q0 + r: one coalesced 256-byte line per frequency and warp).  A first attempt with the [S][64] table
      // (32 uncoalesced 8-byte reads per thread) cost +270 us/layer, the standalone HBM-bound kernel 92 us.
      const bool rope_in_attn = fused && attn_bwd_can_rope();
      a.rope_cs = rope_in_attn ? t->rope_cs_t : nullptr;
      a.rope_glm = t->rope_glm ? 1 : 0;
      CK(attn_bwd(a, s), attn_bwd_launches());
      if (!rope_in_attn && t->rope_glm) CK(rope_glm_qk_inplace(t->dqkv, t->rope_cs, B, S, H + Hkv, W, 1, s), 1);
      else if (!rope_in_attn) CK(rope_qk_inplace_table(t->dqkv, t->rope_cs, B, S, H + Hkv, W, D, 1, s), 1);
    }
    if (y.qkn) {  // through the q/k norm (Qwen3), in place on the q|k columns of dqkv; full-parameter SFT: d q_norm | d k_norm
      // the dw partials: at most as many 256-float blocks as ndw_scratch (64 * d floats) holds
      const int nblk = std::min(QKN_MAX_BLOCKS, 64 * d / 256);
      CK(qk_norm_bwd(t->dqkv, W, y.qk_pre, QK, M, dq, QK, y.qkn, y.qkn + D, mc.rms_eps, t->full ? t->grad_of(y.qkn) : nullptr,
                     t->ndw_scratch, nblk, accumulate, s), t->full ? 2 : 1);
    }
    if (y.qkf)  // through OLMo-2's full-width q/k norm, in place; full-parameter SFT: d q_norm | d k_norm
      CK(qk_norm_full_bwd(t->dqkv, W, y.qk_pre, QK, M, dq, QK, y.qkf, y.qkf + dq, mc.rms_eps, t->full ? t->grad_of(y.qkf) : nullptr,
                          t->ndw_scratch, accumulate, s), t->full ? 2 : 1);
    if (lora) {  // dt = dqkv * B_ext   [M, RP]
      GemmArgs g;
      g.A = t->dqkv; g.lda = W; g.B = y.b_ext; g.ldb = RP; g.b_mn_major = 1; g.C = t->dt; g.ldc = RP;
      g.M = M; g.N = RP; g.K = W; g.epilogue = EPI_BF16; g.block_n = 64;
      CK(gemm_bf16(g, s), 1);
    }
    if (t->full) CK(dw_gemm(t->dqkv, W, h1, d, t->grad_of(y.wqkv)), 1);  // dWqkv = dqkv^T * h1 (dqkv already carries the inverse rotary)
    if (t->full && y.bias) CK(bias_grad(t->dqkv, W, M, W, t->grad_of(y.bias), accumulate, s), 1);  // db = column sums of dqkv
    // LoRA: layer 0's input gradient has no consumer (the embedding is frozen, SURVEY §8a): its dh1 GEMM, the dropout-branch
    // gradient and the norm-1 backward are skipped.  Full-parameter SFT trains the embedding and needs them.
    const bool need_dx = l > 0 || t->full;
    // no_pre_norms: the GEMM writes d x_in = d x_mid + dqkv * Wqkv (+ dt * A_cat) straight into cur, the dropout branch adds to it
    bf16* dh1 = pre_norms ? t->dh : cur;
    if (need_dx) {  // dh1 = dqkv * Wqkv (+ dt * A_cat in the same accumulator when there is no dropout between h1 and A)
      BASEW(W_QKV, wqkv);
      GemmArgs g;
      g.A = t->dqkv; g.lda = W; g.B = wqkv; g.ldb = d; g.b_mn_major = 1;
      if (lora && !drop) { g.A2 = t->dt; g.lda2 = RP; g.B2 = y.a_cat; g.ldb2 = t->KA; g.K2 = RP; }
      g.C = dh1; g.ldc = d; g.M = M; g.N = d; g.K = W; g.epilogue = EPI_BF16;
      if (!pre_norms) { g.R = other; g.ldr = d; g.epilogue = EPI_BF16_ADD; }
      CK(gemm_bf16(g, s), 1);
    }
    if (drop && need_dx) {  // dh1 += sum_t mask_t o (dt_t * A_t) / (1 - p): the masks are regenerated from the counter-based RNG
      GemmArgs g;
      g.A = t->dt; g.lda = RP; g.B = y.a_cat; g.ldb = t->KA; g.b_mn_major = 1; g.C = t->glora; g.ldc = t->KA;
      g.M = M; g.N = t->KA; g.K = RP; g.epilogue = EPI_BF16;
      CK(gemm_bf16(g, s), 1);
      CK(lora_dropout_bwd_add(dh1, t->glora, M, d, t->nt, p_drop, dropout_key(t, l), s), 1);
    }
    if (lora) {
    {  // grad of B_ext (all rows): dqkv^T * t   [W, RP], split over tokens
      GemmArgs g;
      g.A = t->dqkv; g.lda = W; g.a_mn_major = 1; g.B = y.t; g.ldb = RP; g.b_mn_major = 1;
      g.C = t->part_b; g.ldc = RP; g.M = W; g.N = RP; g.K = M; g.epilogue = EPI_F32; g.split_k = split_b;
      g.block_n = 64;
      CK(gemm_bf16(g, s), 1);
    }
    {  // grad of A_cat^T: lora_in^T * dt   [KA, RP]
      GemmArgs g;
      g.A = drop ? y.hd : h1; g.lda = t->KA; g.a_mn_major = 1; g.B = t->dt; g.ldb = RP; g.b_mn_major = 1;
      g.C = t->part_a; g.ldc = RP; g.M = t->KA; g.N = RP; g.K = M; g.epilogue = EPI_F32; g.split_k = split_a;
      g.block_n = 64;
      CK(gemm_bf16(g, s), 1);
    }
    const int r = tc.lora_r;
    for (int ti = 0; ti < t->nt; ++ti) {
      float* gl = t->grads + static_cast<int64_t>(l) * t->per_layer + t->tg[ti].off;
      const int d_out = t->tg[ti].d_out;
      // dA^T = lora_in^T (dy * sB)  (the scale rides in B_ext);  dB = s * dy^T t  (t is unscaled, so the scale is applied here)
      lora_gather_kernel<<<(d * r + 255) / 256, 256, 0, s>>>(t->part_a, split_a, static_cast<long long>(t->KA) * RP, RP,
                                                            drop ? ti * d : 0, ti * r, d, r, gl, accumulate, 1.0f);
      lora_gather_kernel<<<(d_out * r + 255) / 256, 256, 0, s>>>(t->part_b, split_b, static_cast<long long>(W) * RP, RP,
                                                                t->tg[ti].row0, ti * r, d_out, r, gl + static_cast<int64_t>(d) * r,
                                                                accumulate, tc.lora_alpha / static_cast<float>(r));
      CK(cudaGetLastError(), 2);
    }
    }  // lora
    if (t->full && pre_norms) CK(rmsnorm_dw(t->dh, t->xs[l], y.rstd1, M, d, t->ndw_scratch, t->grad_of(y.norm1), accumulate, s), 2);
    if (need_dx && pre_norms) CK(rmsnorm_bwd(t->dh, t->xs[l], y.norm1, y.rstd1, other, cur, M, d, s), 1);  // cur = d x_in
    if (t->full && t->rs_now && t->world > 1) {  // this layer's gradients are final: reduce-scatter them while the backward pass goes on
      int rc = reduce_scatter_block(t, t->g_flat + static_cast<int64_t>(l) * t->layer_elems, t->layer_elems, l);
      if (rc) return rc;
    }
  }
  if (t->full) {  // embedding gradient: rows of d x_0 scattered by token id (fp32 atomics), then folded into the bf16 gradient block
    const size_t vd = static_cast<size_t>(V) * d;
    CKM(cudaMemsetAsync(t->embed_g32, 0, vd * sizeof(float), s));
    CK(embedding_bwd(t->d_ids, cur, t->embed_g32, M, d, V, s), 1);
    CK(add_f32_into_bf16(t->embed_g32, t->grad_of(t->embed), static_cast<int64_t>(vd), accumulate, s), 1);
  }
  return DTX_OK;
}

int optimizer_step(dtx_trainer* t, float* lr_used) {
  const dtx_train_cfg& tc = t->tc;
  cudaStream_t s = t->stream;
  if (t->world > 1) {
    NcclApi* api = nccl_api();
    if (!api || !t->nccl_comm) return t->fail(DTX_ERR_NCCL, "NCCL communicator missing for world=%d", t->world);
    int rc = api->AllReduce(t->grads, t->grads, static_cast<size_t>(t->n_train), kNcclFloat32, kNcclSum, t->nccl_comm, s);
    if (rc != 0) return t->fail(DTX_ERR_NCCL, "ncclAllReduce failed: %s", api->GetErrorString ? api->GetErrorString(rc) : "?");
    t->launches += 1;
  }
  cudaEventRecord(t->ev_ar, s);
  CK(sumsq(t->grads, t->n_train, t->d_scratch, t->d_sumsq, s), 2);
  const double lam = dtx_lr_lambda(tc.sched, t->opt_step, tc.warmup_steps, tc.total_steps);
  const float lr = static_cast<float>(static_cast<double>(tc.lr) * lam);
  const int step1 = t->opt_step + 1;
  AdamWArgs a;
  a.p = t->params; a.g = t->grads; a.m = t->adam_m; a.v = t->adam_v; a.n = t->n_train;
  a.lr = lr; a.beta1 = tc.beta1; a.beta2 = tc.beta2; a.eps = tc.eps; a.weight_decay = tc.weight_decay;
  a.bias1 = static_cast<float>(1.0 - pow(static_cast<double>(tc.beta1), step1));
  a.bias2 = static_cast<float>(1.0 - pow(static_cast<double>(tc.beta2), step1));
  // HF scales every micro-batch loss by 1/grad_accum whatever the number actually accumulated (forced end-of-epoch step)
  a.grad_scale = 1.0f / static_cast<float>(t->world * (tc.grad_accum > 0 ? tc.grad_accum : 1));
  a.sumsq = t->d_sumsq; a.max_grad_norm = tc.max_grad_norm; a.grad_norm_out = t->d_gnorm;
  CK(adamw_step(a, s), 1);
  int rc = refresh_shadows(t);
  if (rc) return rc;
  t->opt_step += 1;
  if (lr_used) *lr_used = lr;
  return DTX_OK;
}

template <class Owner>
int64_t nodecay_from(const std::vector<Slot<Owner>>& slots, int64_t used) {
  for (const auto& s : slots)
    if (s.nodecay) return s.off;
  return used;
}

// Full-parameter SFT: the blocks' bf16 gradients have been (or are now) reduce-scattered in place; every rank then runs
// clip + AdamW on the slices it owns (fp32 master weights + moments, ZeRO-1 style) and the updated bf16 slices are
// all-gathered in place.  HF's no-decay set (norm weights, biases) sits at the end of every block.
int optimizer_step_full(dtx_trainer* t, float* lr_used) {
  const dtx_train_cfg& tc = t->tc;
  cudaStream_t s = t->stream;
  const int L = t->mc.n_layers, N = t->world;
  NcclApi* api = N > 1 ? nccl_api() : nullptr;
  if (N > 1 && (!api || !api->ReduceScatter || !api->AllGather || !t->nccl_comm))
    return t->fail(DTX_ERR_NCCL, "NCCL reduce-scatter / all-gather unavailable for world=%d", N);
  bf16* gglob = t->g_flat + static_cast<int64_t>(L) * t->layer_elems;
  if (N > 1) {
    if (!t->rs_now)  // gradients of earlier micro-batches only: nothing was sent during the backward pass
      for (int l = L - 1; l >= 0; --l) {
        int rc = reduce_scatter_block(t, t->g_flat + static_cast<int64_t>(l) * t->layer_elems, t->layer_elems, l);
        if (rc) return rc;
      }
    int rc = reduce_scatter_block(t, gglob, t->glob_elems, L);
    if (rc) return rc;
    CKM(cudaEventRecord(t->ev_comm, t->comm_stream));
    CKM(cudaStreamWaitEvent(s, t->ev_comm, 0));
  }
  cudaEventRecord(t->ev_ar, s);
  const int64_t lsh = t->layer_elems / N, gsh = t->glob_elems / N;  // slice lengths
  auto slice = [&](int blk, bf16* base, int64_t* n, int64_t* moff) {  // this rank's slice of block blk (L = globals)
    const int64_t sh = blk < L ? lsh : gsh;
    *n = sh;
    *moff = static_cast<int64_t>(blk) * lsh;  // offset inside the master / moment shards
    return base + (blk < L ? static_cast<int64_t>(blk) * t->layer_elems : static_cast<int64_t>(L) * t->layer_elems) + static_cast<int64_t>(t->rank) * sh;
  };
  if (!t->master_valid) {  // first step (or weights re-loaded): fp32 master copies of the owned bf16 slices
    for (int blk = 0; blk <= L; ++blk) {
      int64_t n, moff;
      bf16* w = slice(blk, t->w_flat, &n, &moff);
      CK(cast_bf16_to_f32(w, t->master + moff, n, s), 1);
    }
    t->master_valid = true;
  }
  for (int blk = 0; blk <= L; ++blk) {
    int64_t n, moff;
    bf16* g = slice(blk, t->g_flat, &n, &moff);
    CK(sumsq_bf16_acc(g, n, t->d_scratch, t->d_sumsq, blk == 0 ? 1 : 0, s), 2);
  }
  if (N > 1) {
    int rc = api->AllReduce(t->d_sumsq, t->d_sumsq, 1, kNcclFloat32, kNcclSum, t->nccl_comm, s);
    if (rc != 0) return t->fail(DTX_ERR_NCCL, "ncclAllReduce failed: %s", api->GetErrorString ? api->GetErrorString(rc) : "?");
    t->launches += 1;
  }
  const double lam = dtx_lr_lambda(tc.sched, t->opt_step, tc.warmup_steps, tc.total_steps);
  const float lr = static_cast<float>(static_cast<double>(tc.lr) * lam);
  const int step1 = t->opt_step + 1;
  // no weight decay from the first no-decay slot of a block on (its tail, see Slot)
  const int64_t nd_layer = nodecay_from(t->lslots, t->layer_used), nd_glob = nodecay_from(t->gslots, t->glob_used);
  for (int blk = 0; blk <= L; ++blk) {
    int64_t n, moff;
    bf16* g = slice(blk, t->g_flat, &n, &moff);
    bf16* w = slice(blk, t->w_flat, &n, &moff);
    AdamWShardArgs a;
    a.master = t->master + moff; a.m = t->fm + moff; a.v = t->fv + moff; a.g = g; a.w = w; a.n = n;
    const int64_t nd_begin = blk < L ? nd_layer : nd_glob, first = static_cast<int64_t>(t->rank) * n;
    a.nodecay_from = nd_begin - first < 0 ? 0 : nd_begin - first;
    a.lr = lr; a.beta1 = tc.beta1; a.beta2 = tc.beta2; a.eps = tc.eps; a.weight_decay = tc.weight_decay;
    a.bias1 = static_cast<float>(1.0 - pow(static_cast<double>(tc.beta1), step1));
    a.bias2 = static_cast<float>(1.0 - pow(static_cast<double>(tc.beta2), step1));
    a.grad_scale = 1.0f / static_cast<float>(N * (tc.grad_accum > 0 ? tc.grad_accum : 1));
    a.sumsq = t->d_sumsq; a.max_grad_norm = tc.max_grad_norm; a.grad_norm_out = t->d_gnorm;
    CK(adamw_shard_step(a, s), 1);
  }
  if (N > 1) {
    // Every rank gets every updated slice (in place: the send slice sits at its final position).  The all-gathers run on the
    // side stream in the order the next forward pass consumes the blocks, so that they overlap it: measured on 8 GPUs (13B),
    // the 26 GB all-gather was 58 of the step's 658 ms when it sat on the main stream.
    CKM(cudaEventRecord(t->ev_comm, s));
    CKM(cudaStreamWaitEvent(t->comm_stream, t->ev_comm, 0));
    for (int i = 0; i <= L; ++i) {
      const int blk = i == 0 ? L : i - 1;  // globals first, then layer 0, 1, ...
      int64_t n, moff;
      bf16* w = slice(blk, t->w_flat, &n, &moff);
      bf16* base = w - static_cast<int64_t>(t->rank) * n;
      int rc = api->AllGather(w, base, static_cast<size_t>(n), kNcclBfloat16, t->nccl_comm, t->comm_stream);
      if (rc != 0) return t->fail(DTX_ERR_NCCL, "ncclAllGather failed: %s", api->GetErrorString ? api->GetErrorString(rc) : "?");
      CKM(cudaEventRecord(t->ev_ag[blk], t->comm_stream));
      t->ag_pending[blk] = 1;
      t->launches += 1;
    }
  }
  t->opt_step += 1;
  if (lr_used) *lr_used = lr;
  return DTX_OK;
}

// validate and record the shape of the batch about to be processed
int set_batch_shape(dtx_trainer* t, int32_t seq_len_batch, bool have_lens) {
  const int S = seq_len_batch > 0 ? seq_len_batch : t->tc.seq_len;
  if (S % 128 || S > t->tc.seq_len)
    return t->fail(DTX_ERR_INVALID, "seq_len_batch %d must be a multiple of 128 and <= seq_len %d", S, t->tc.seq_len);
  t->cur_S = S;
  t->cur_B = t->tc.micro_batch;
  t->cur_M = S * t->tc.micro_batch;
  t->use_seq_lens = have_lens;
  return DTX_OK;
}

// ---- ragged micro-batches as length groups -------------------------------------------------------------------------
// The reference pads a batch to its longest row (DataCollatorForSeq2Seq, cmd/tuning/train.py:282-286) and computes over the
// padding.  Here the attention kernels already skip padding tiles; the GEMMs, norms and CE do not - on instruction data with a
// long tail of row lengths more than half of their rows are padding.  A micro-batch with row lengths is therefore run as
// LENGTH GROUPS: rows sorted by length, cut into contiguous groups, each group padded to its own longest row (128-rounded)
// and sent through forward + backward on its own; gradients accumulate, and every group's loss and dlogits are divided by the
// labelled-token count of the WHOLE micro-batch, so the result is the same token mean (up to summation order).  The cut is
// chosen by dynamic programming over a cost model of the step's GEMMs (128-row tiles x 256-column tiles in waves of one CTA
// per SM) plus a fixed cost per group: few long groups waste rows on padding, many short ones waste waves.
struct SubPlan {
  int n = 0;            // groups (1: run the micro-batch as it is)
  int start[65] = {0};  // group g = order[start[g] .. start[g+1])
  int S[64] = {0};      // padded length of group g
  int order[64] = {0};  // rows sorted by length, longest first
  int n_div = 0;        // labelled tokens of the whole micro-batch, counted the way the groups' shift_labels kernels will
};

// PACKED layout of a ragged micro-batch (LoRA or full-parameter): sequence b gets its length rounded up to 128 rows, sequences back to back - one
// pass over sum_b ceil128(len_b) rows instead of B * S_batch (or one pass per length group).  GEMMs, norms and CE simply see
// fewer rows; the attention kernels take the first row of every sequence from a table; RoPE takes a row's position and the
// label shift a sequence's end from a per-row position array.
// the layout alone (host arithmetic): first row of every sequence; true when it is smaller than the padded rectangle
bool packed_rows(const int32_t* lens, int B, int S_batch, RowStarts* rs) {
  rs->n = B;
  rs->start[0] = 0;
  for (int b = 0; b < B; ++b) {
    const int len = std::min(std::max(lens[b], 0), S_batch);
    rs->start[b + 1] = rs->start[b] + std::min(S_batch, std::max(128, (len + 127) / 128 * 128));
  }
  return rs->start[B] < B * S_batch && rs->start[B] > 128;
}

struct PlanDims { int hidden, ffn, W, dq, n_sms, B; };  // what the cost model needs of the model / device / batch

double group_cost(const PlanDims& t, int rows, int S) {
  const int d = t.hidden, F = t.ffn, W = t.W, dq = t.dq;
  const long long mt = (static_cast<long long>(rows) * S + 127) / 128;
  const long long slots = std::max(1, t.n_sms);
  auto waves = [&](int n_cols, int k) { return static_cast<double>((mt * ((n_cols + 255) / 256) + slots - 1) / slots) * k; };
  // forward: qkv, o, gate|up, down; backward dX: through down (N = F), gate|up, o, qkv
  return waves(W, d) + waves(d, dq) + waves(2 * F, d) + waves(d, F) + waves(F, d) + waves(d, 2 * F) + waves(dq, d) + waves(d, W);
}

// labels may be null (planning only: n_div stays 0)
void plan_groups(const PlanDims& t, const int32_t* lens, const int32_t* labels, int S_batch, SubPlan* p) {
  const int B = t.B;
  p->n = 1;
  if (!g_varlen_split || !lens || B < 2 || B > 64) return;
  auto c128 = [&](int len) { return std::min(S_batch, std::max(128, (std::min(std::max(len, 0), S_batch) + 127) / 128 * 128)); };
  for (int i = 0; i < B; ++i) p->order[i] = i;
  std::stable_sort(p->order, p->order + B, [&](int a, int b) { return lens[a] > lens[b]; });
  const bool force = g_varlen_split == 2;  // tests: minimise padded rows, no fixed cost
  const double fix = force ? 0.0 : 0.001 * g_varlen_fix_permille * group_cost(t, 1, 256);
  auto cost = [&](int rows, int S) { return force ? static_cast<double>(rows) * S : group_cost(t, rows, S); };
  double best[65];
  int cut[65];
  best[0] = 0.0;
  for (int j = 1; j <= B; ++j) {
    best[j] = 1e300;
    for (int i = 0; i < j; ++i) {  // group = sorted rows i .. j-1, padded to the longest of them (row i); at least 256 rows of tokens
      int S = c128(lens[p->order[i]]);
      if ((j - i) * S < 256) {  // every group keeps M >= 256 (whole 256-row GEMM tiles, the fused-epilogue kernels)
        if (S_batch < 256) continue;
        S = 256;
      }
      const double c = best[i] + cost(j - i, S) + fix;
      if (c < best[j]) { best[j] = c; cut[j] = i; }
    }
  }
  if (best[B] > 1e299 || best[B] >= cost(B, S_batch) + fix) return;  // one group at the batch's own padded length is as good
  int ends[65], n = 0;
  for (int j = B; j > 0; j = cut[j]) ends[n++] = j;
  p->n = n;
  p->start[0] = 0;
  for (int g = 0; g < n; ++g) {
    p->start[g + 1] = ends[n - 1 - g];
    int S = c128(lens[p->order[p->start[g]]]);
    if ((p->start[g + 1] - p->start[g]) * S < 256) S = 256;
    p->S[g] = S;
  }
  if (n < 2) { p->n = 1; return; }
  if (!labels) return;
  long long cnt = 0;  // positions 1 .. S_g - 1 of every row carry the shifted label of the position before them
  for (int g = 0; g < n; ++g)
    for (int k = p->start[g]; k < p->start[g + 1]; ++k) {
      const int32_t* row = labels + static_cast<size_t>(p->order[k]) * S_batch;
      for (int j = 1; j < p->S[g]; ++j) cnt += row[j] >= 0 ? 1 : 0;
    }
  p->n_div = static_cast<int>(cnt);
  if (p->n_div <= 0) p->n = 1;  // nothing carries a label: the plain path handles the degenerate batch
}

int check_ready(dtx_trainer* t) {
  char buf[160];
  if (const char* m = t->missing_weight(buf, sizeof(buf)))
    return t->fail(DTX_ERR_STATE, "base weight %s was never loaded (dtx_load_tensor / dtx_init_random_weights)", m);
  if (!t->full && !t->have_lora) return t->fail(DTX_ERR_STATE, "LoRA adapters not initialised (dtx_init_lora / dtx_load_tensor)");
  return DTX_OK;
}

// One micro-batch as the caller hands it over: [micro_batch, S] ids and labels, optional true row lengths [micro_batch].
struct BatchInput {
  const int32_t *ids, *labels, *lens;  // lens null: every row is full
  bool on_device;                      // device pointers (dtx_step_device), else host memory
  int S;                               // seq_len_batch as set_batch_shape resolved it
};

// How a micro-batch runs: packed (one pass over rs), length groups (groups.n > 1) or one pass at the padded shape.
struct BatchPlan {
  bool packed = false;
  RowStarts rs;
  SubPlan groups;
};

// The layout decision for dtx_step, dtx_step_device and dtx_eval_loss alike.  A batch with row lengths is packed when that
// is on, the fused RoPE epilogue applies (it takes per-row positions) and it saves rows; otherwise a LoRA batch runs as length
// groups when the cost model cuts it.  Device input is planned on the host: the row lengths are read back once, and the
// labels (B*S*4 bytes, for the groups' token count) only when grouping is planned - with the lengths when packing is off.
int plan_batch(dtx_trainer* t, const BatchInput& in, BatchPlan* p) {
  const int B = t->tc.micro_batch;
  const size_t M = static_cast<size_t>(B) * in.S;
  p->groups.n = 1;
  const bool pack = in.lens && g_varlen_pack && g_varlen_split == 1 && B <= 64 && g_fused_epilogues && (t->dq + t->dkv) % 256 == 0 &&
                    t->W % 256 == 0;
  const bool group = in.lens && g_varlen_split && !t->full && B > 1 && B <= 64;
  if (!pack && !group) return DTX_OK;
  auto read_back = [&](const int32_t* src, std::vector<int32_t>& dst, size_t n) {
    dst.resize(n);
    return cudaMemcpyAsync(dst.data(), src, n * 4, cudaMemcpyDeviceToHost, t->stream);
  };
  const int32_t* lens = in.lens;
  if (in.on_device) {
    CKM(read_back(in.lens, t->h_lens, static_cast<size_t>(B)));
    if (!pack) CKM(read_back(in.labels, t->h_labels, M));
    CKM(cudaStreamSynchronize(t->stream));
    lens = t->h_lens.data();
  }
  if (pack && packed_rows(lens, B, in.S, &p->rs)) {
    p->packed = true;
    return DTX_OK;
  }
  if (!group) return DTX_OK;
  if (in.on_device && pack) {
    CKM(read_back(in.labels, t->h_labels, M));
    CKM(cudaStreamSynchronize(t->stream));
  }
  plan_groups(PlanDims{t->mc.hidden, t->mc.ffn, t->W, t->dq, t->n_sms, B}, lens, in.on_device ? t->h_labels.data() : in.labels, in.S,
              &p->groups);
  return DTX_OK;
}

// Per-row evaluation statistics (loss sum, labelled tokens) of the arrays the caller wants (either may be null).  run_batch
// copies them pass by pass to h_row_sum / h_row_valid; once the stream is synchronised row k there is the caller's row order[k].
struct RowStats {
  float* sum;
  int32_t* valid;
  std::vector<int> order;
};

// Stage `in` as plan_batch lays it out and run its passes through fwd_bwd(t, backward).  The batch's cur_* / packed /
// sub_accum / sub_ndiv are set here for each pass and put back to the whole micro-batch's on every exit.  A training step's
// ev0 falls after the batch copies and pack_rows and before the groups' gathers.
int run_batch(dtx_trainer* t, const BatchInput& in, bool backward, RowStats* stats = nullptr) {
  BatchPlan p;
  int rc = plan_batch(t, in, &p);
  if (rc) return rc;
  const int B = t->tc.micro_batch, S = in.S;
  const size_t M = static_cast<size_t>(B) * S;
  const bool grouped = p.groups.n > 1;
  const cudaMemcpyKind kind = in.on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  const int32_t *ids = in.ids, *labels = in.labels, *lens = in.lens;  // what pack_rows / gather_rows read
  if (!p.packed && !grouped) {
    CKM(cudaMemcpyAsync(t->d_ids, ids, M * 4, kind, t->stream));
    CKM(cudaMemcpyAsync(t->d_labels, labels, M * 4, kind, t->stream));
    if (lens) CKM(cudaMemcpyAsync(t->d_seq_lens, lens, static_cast<size_t>(B) * 4, kind, t->stream));
  } else if (!in.on_device) {  // host input goes through the staging buffers
    CKM(cudaMemcpyAsync(t->d_ids_full, ids, M * 4, kind, t->stream));
    CKM(cudaMemcpyAsync(t->d_labels_full, labels, M * 4, kind, t->stream));
    ids = t->d_ids_full;
    labels = t->d_labels_full;
    if (grouped) {
      CKM(cudaMemcpyAsync(t->d_lens_full, lens, static_cast<size_t>(B) * 4, kind, t->stream));
      lens = t->d_lens_full;
    }
  }
  if (p.packed) {
    CKM(cudaMemcpyAsync(t->d_seq_lens, in.lens, static_cast<size_t>(B) * 4, kind, t->stream));
    CK(pack_rows(ids, labels, S, p.rs, t->d_ids, t->d_labels, t->d_pos, t->d_row_start, t->stream), 1);
  }
  if (backward) {
    cudaEventRecord(t->ev0, t->stream);
    t->last_groups = p.packed ? 0 : p.groups.n;
  }
  if (stats) {
    t->h_row_sum.resize(static_cast<size_t>(B));
    t->h_row_valid.resize(static_cast<size_t>(B));
    stats->order.resize(static_cast<size_t>(B));
    for (int k = 0; k < B; ++k) stats->order[k] = grouped ? p.groups.order[k] : k;
  }
  for (int g = 0; g < p.groups.n && rc == DTX_OK; ++g) {
    int first = 0, rows = B, S_g = S;
    if (grouped) {
      RowList rl;
      first = p.groups.start[g];
      rows = rl.n = p.groups.start[g + 1] - first;
      S_g = p.groups.S[g];
      for (int k = 0; k < rows; ++k) rl.rows[k] = p.groups.order[first + k];
      cudaError_t e = gather_rows(ids, labels, lens, S, rl, S_g, t->d_ids, t->d_labels, t->d_seq_lens, t->stream);
      if (e != cudaSuccess) {
        rc = t->fail(DTX_ERR_CUDA, "gather_rows: %s", cudaGetErrorString(e));
        break;
      }
      t->launches += 1;
    }
    t->cur_B = rows;
    t->cur_S = S_g;
    t->cur_M = p.packed ? p.rs.start[B] : rows * S_g;
    t->packed = p.packed;
    t->sub_accum = g > 0;
    t->sub_ndiv = grouped ? p.groups.n_div : 0;
    rc = fwd_bwd(t, backward);
    if (rc == DTX_OK && stats) {
      cudaError_t e = row_loss_stats(t->row_loss, t->d_shift, rows, S_g, t->d_row_sum, t->d_row_valid, t->stream,
                                     p.packed ? t->d_row_start : nullptr);
      // d_row_sum / d_row_valid are reused by the next group: these copies are stream-ordered in front of its kernels
      if (e == cudaSuccess && stats->sum)
        e = cudaMemcpyAsync(t->h_row_sum.data() + first, t->d_row_sum, static_cast<size_t>(rows) * 4, cudaMemcpyDeviceToHost, t->stream);
      if (e == cudaSuccess && stats->valid)
        e = cudaMemcpyAsync(t->h_row_valid.data() + first, t->d_row_valid, static_cast<size_t>(rows) * 4, cudaMemcpyDeviceToHost, t->stream);
      if (e != cudaSuccess) rc = t->fail(DTX_ERR_CUDA, "eval row statistics: %s", cudaGetErrorString(e));
      t->launches += 1;
    }
  }
  t->cur_B = B;
  t->cur_S = S;
  t->cur_M = static_cast<int>(M);
  t->packed = t->sub_accum = false;
  t->sub_ndiv = 0;
  return rc;
}

// one training micro-batch: forward + backward, then the optimizer once grad_accum micro-batches (or DTX_STEP_FORCE) are in
int do_step(dtx_trainer* t, const BatchInput& in, int32_t flags, float* loss_out, float* gnorm_out, float* lr_out, int32_t* stepped_out) {
  const int accum = t->tc.grad_accum > 0 ? t->tc.grad_accum : 1;
  t->rs_now = t->full && (t->micro_idx + 1 >= accum || (flags & DTX_STEP_FORCE));
  int rc = run_batch(t, in, true);
  if (rc) return rc;
  cudaEventRecord(t->ev_fb, t->stream);
  t->micro_idx += 1;
  int stepped = 0;
  float lr = 0.f;
  if (t->micro_idx >= accum || (flags & DTX_STEP_FORCE)) {
    rc = t->full ? optimizer_step_full(t, &lr) : optimizer_step(t, &lr);
    if (rc) return rc;
    t->micro_idx = 0;
    stepped = 1;
  }
  cudaEventRecord(t->ev1, t->stream);
  float host[2] = {0.f, 0.f};
  cudaMemcpyAsync(&host[0], t->d_loss, sizeof(float), cudaMemcpyDeviceToHost, t->stream);
  if (stepped) cudaMemcpyAsync(&host[1], t->d_gnorm, sizeof(float), cudaMemcpyDeviceToHost, t->stream);
  cudaError_t e = cudaStreamSynchronize(t->stream);
  if (e != cudaSuccess) return t->fail(DTX_ERR_CUDA, "step failed on device: %s", cudaGetErrorString(e));
  cudaEventElapsedTime(&t->last_ms, t->ev0, t->ev1);
  t->seg_ms[0] = t->last_ms;
  cudaEventElapsedTime(&t->seg_ms[1], t->ev0, t->ev_fb);
  t->seg_ms[2] = t->seg_ms[3] = 0.f;
  if (stepped) {
    cudaEventElapsedTime(&t->seg_ms[2], t->ev_fb, t->ev_ar);
    cudaEventElapsedTime(&t->seg_ms[3], t->ev_ar, t->ev1);
  }
  if (loss_out) *loss_out = host[0];
  if (gnorm_out) *gnorm_out = host[1];
  if (lr_out) *lr_out = lr;
  if (stepped_out) *stepped_out = stepped;
  return DTX_OK;
}

// --- HF tensor-name parsing -----------------------------------------------------------------------
bool parse_layer(const char* name, int* layer, const char** rest) {
  const char* p = strstr(name, "layers.");
  if (!p) return false;
  p += 7;
  char* end = nullptr;
  long v = strtol(p, &end, 10);
  if (end == p || *end != '.') return false;
  *layer = static_cast<int>(v);
  *rest = end + 1;
  return true;
}

// The base tensor an HF checkpoint name refers to.  A layer's tensors match by substring of the part after "layers.N.", the
// globals anywhere in the name - except the final norm, whose key every layer norm's name ends in: it only matches outside a layer.
struct NamedWeight {
  const std::vector<WeightName>* names;  // gnames or lnames
  size_t row;                            // of `names`
  uint8_t* loaded;                       // the block's part of the loaded map, indexed like `names`
  bf16* slot;                            // the slot's first element in the weights (nullptr once NF4-packed)
  bool nf4;                              // the slot is one dtx_quantize_base packs
  const WeightName& w() const { return (*names)[row]; }
};
int find_weight(dtx_trainer* t, const char* name, NamedWeight* out) {
  int layer = -1;
  const char* rest = nullptr;
  const bool in_layer = parse_layer(name, &layer, &rest);
  for (size_t i = 0; i < t->gnames.size(); ++i) {
    const auto& s = t->gslots[t->gnames[i].slot];
    if (strstr(name, t->gnames[i].key) && !(in_layer && s.mem == &dtx_trainer::normf)) {
      *out = {&t->gnames, i, t->loaded.data(), t->*s.mem, false};
      return DTX_OK;
    }
  }
  if (!in_layer) return t->fail(DTX_ERR_INVALID, "unknown tensor name %s", name);
  if (layer < 0 || layer >= t->mc.n_layers) return t->fail(DTX_ERR_INVALID, "%s: layer out of range", name);
  for (size_t i = 0; i < t->lnames.size(); ++i) {
    if (!strstr(rest, t->lnames[i].key)) continue;
    const auto& s = t->lslots[t->lnames[i].slot];
    *out = {&t->lnames, i, t->loaded.data() + t->gnames.size() + layer * t->lnames.size(), t->layers[layer].*s.mem, s.nf4 >= 0};
    return DTX_OK;
  }
  return t->fail(DTX_ERR_INVALID, "unknown tensor name %s", name);
}

// copies the halves of wgu named by `gu` (GU_*) between the GU-interleaved device rows and the HF rows on the host
cudaError_t gu_copy(bf16* dev, bf16* host, int gu, int64_t F, int64_t d, cudaMemcpyKind kind, cudaStream_t s) {
  for (int h = 0; h < 2; ++h) {
    if (!(gu & (1 << h))) continue;
    for (int64_t b = 0; b < F / 128; ++b) {
      bf16* dv = dev + (b * 256 + h * 128) * d;
      bf16* hs = host + ((gu == GU_BOTH ? h * F : 0) + b * 128) * d;
      const size_t bytes = 128 * d * sizeof(bf16);
      cudaError_t e = kind == cudaMemcpyHostToDevice ? cudaMemcpyAsync(dv, hs, bytes, kind, s) : cudaMemcpyAsync(hs, dv, bytes, kind, s);
      if (e != cudaSuccess) return e;
    }
  }
  return cudaSuccess;
}

void to_bf16_host(const void* src, int dtype, size_t n, std::vector<bf16>& out) {
  out.resize(n);
  if (dtype == DTX_BF16) {
    memcpy(out.data(), src, n * 2);
  } else if (dtype == DTX_F32) {
    const float* f = static_cast<const float*>(src);
    for (size_t i = 0; i < n; ++i) out[i] = __float2bfloat16_rn(f[i]);
  } else {
    const __half* h = static_cast<const __half*>(src);
    for (size_t i = 0; i < n; ++i) out[i] = __float2bfloat16_rn(__half2float(h[i]));
  }
}
void to_f32_host(const void* src, int dtype, size_t n, std::vector<float>& out) {
  out.resize(n);
  if (dtype == DTX_F32) {
    memcpy(out.data(), src, n * 4);
  } else if (dtype == DTX_BF16) {
    const bf16* b = static_cast<const bf16*>(src);
    for (size_t i = 0; i < n; ++i) out[i] = __bfloat162float(b[i]);
  } else {
    const __half* h = static_cast<const __half*>(src);
    for (size_t i = 0; i < n; ++i) out[i] = __half2float(h[i]);
  }
}

int target_index(const dtx_trainer* t, char which) {  // 'q','k','v' -> index among enabled targets or -1
  for (int i = 0; i < t->nt; ++i)
    if (t->tg_name[i] == which) return i;
  return -1;
}

// configuration checks of dtx_trainer_create and dtx_plan_device_bytes (host only; the message goes to g_error)
int check_cfg(const dtx_model_cfg* mc, const dtx_train_cfg* tc) {
  auto bad = [&](const char* m) {
    g_error = m;
    return DTX_ERR_INVALID;
  };
  if (mc->head_dim != 128) return bad("only head_dim 128 is implemented (Llama-2 / Mistral family)");
  if (mc->n_kv_heads <= 0 || mc->n_heads % mc->n_kv_heads) return bad("n_heads must be a multiple of n_kv_heads");
  if (mc->hidden % 64 || mc->ffn % 128 || mc->vocab % 8)
    return bad("hidden must be a multiple of 64, ffn a multiple of 128 (GU-interleaved layout), vocab a multiple of 8");
  if (tc->seq_len % 128 || tc->seq_len <= 0 || tc->micro_batch <= 0) return bad("seq_len must be a positive multiple of 128");
  if (tc->seq_len > mc->max_seq) return bad("seq_len exceeds max_seq");
  if (!tc->full_finetune && (tc->lora_r <= 0 || tc->lora_r % 8)) return bad("lora_r must be a positive multiple of 8");
  if (tc->lora_dropout < 0.0f || tc->lora_dropout >= 1.0f) return bad("lora_dropout must be in [0, 1)");
  if (tc->recompute < 0 || tc->recompute > RECOMPUTE_LAYER)
    return bad("recompute must be 0 (automatic), 1 (keep all activations) or 2 (recompute per layer)");
  if (!tc->full_finetune && ((tc->target_mask & ~(DTX_TARGET_Q | DTX_TARGET_K | DTX_TARGET_V)) || tc->target_mask == 0))
    { g_error = "lora_target must be a non-empty subset of q_proj,k_proj,v_proj"; return DTX_ERR_UNSUPPORTED; }
  return DTX_OK;
}

// checks of the model-family extensions (host only; the message goes to g_error)
int check_ext(const dtx_model_cfg* mc, const dtx_model_ext* ext) {
  if (!ext) return DTX_OK;
  auto bad = [&](const char* m) {
    g_error = m;
    return DTX_ERR_INVALID;
  };
  if (ext->qkv_bias != 0 && ext->qkv_bias != 1) return bad("qkv_bias must be 0 or 1");
  if (ext->qk_norm != 0 && ext->qk_norm != 1) return bad("qk_norm must be 0 or 1");
  if (ext->rope_glm != 0 && ext->rope_glm != 1) return bad("rope_glm must be 0 or 1");
  if (ext->rope_glm && ext->qk_norm) return bad("rope_glm cannot be combined with qk_norm");
  if (ext->rope_glm && mc->sliding_window > 0) return bad("rope_glm cannot be combined with a sliding window");
  if (ext->post_norms != 0 && ext->post_norms != 1) return bad("post_norms must be 0 or 1");
  if (ext->qk_norm_full != 0 && ext->qk_norm_full != 1) return bad("qk_norm_full must be 0 or 1");
  if (ext->no_pre_norms != 0 && ext->no_pre_norms != 1) return bad("no_pre_norms must be 0 or 1");
  if (ext->qk_norm_full && (ext->qk_norm || ext->rope_glm)) return bad("qk_norm_full cannot be combined with qk_norm or rope_glm");
  if (ext->no_pre_norms && !ext->post_norms) return bad("no_pre_norms needs post_norms (the sublayers' only norms)");
  if (ext->rope_glm && ext->rope_type != DTX_ROPE_DEFAULT) return bad("rope_glm needs rope_type DTX_ROPE_DEFAULT (no scaled GLM rotary is implemented)");
  if (ext->rope_type < DTX_ROPE_DEFAULT || ext->rope_type > DTX_ROPE_LLAMA3)
    return bad("rope_type must be DTX_ROPE_DEFAULT, DTX_ROPE_LINEAR or DTX_ROPE_LLAMA3 (yarn, dynamic, longrope are not implemented)");
  if (ext->rope_type != DTX_ROPE_DEFAULT && !(ext->rope_factor > 0.0f)) return bad("rope_factor must be > 0");
  if (ext->rope_type == DTX_ROPE_LLAMA3) {
    if (!(ext->rope_low_freq_factor > 0.0f) || !(ext->rope_low_freq_factor < ext->rope_high_freq_factor))
      return bad("llama3 rope scaling needs 0 < low_freq_factor < high_freq_factor");
    if (ext->rope_original_max_pos <= 0) return bad("llama3 rope scaling needs original_max_position_embeddings > 0");
  }
  return DTX_OK;
}

// shapes and adapter geometry derived from the configuration (host only)
void setup_dims(dtx_trainer* t, const dtx_model_cfg* mc, const dtx_model_ext* ext, const dtx_train_cfg* tc, int world) {
  t->mc = *mc;
  if (ext) t->ext = *ext;
  t->rope_glm = t->ext.rope_glm != 0;
  t->tc = *tc;
  t->world = world;
  t->M = tc->micro_batch * tc->seq_len;
  t->dq = mc->n_heads * mc->head_dim;
  t->dkv = mc->n_kv_heads * mc->head_dim;
  t->W = t->dq + 2 * t->dkv;
  t->full = tc->full_finetune != 0;
  t->dropout = !t->full && tc->lora_dropout > 0.0f;
  t->nt = 0;
  t->per_layer = 0;
  if (!t->full) {
    const unsigned bits[3] = {DTX_TARGET_Q, DTX_TARGET_K, DTX_TARGET_V};
    const char names[3] = {'q', 'k', 'v'};
    const int row0[3] = {0, t->dq, t->dq + t->dkv};
    const int dout[3] = {t->dq, t->dkv, t->dkv};
    for (int i = 0; i < 3; ++i)
      if (tc->target_mask & bits[i]) {
        t->tg[t->nt].row0 = row0[i];
        t->tg[t->nt].d_out = dout[i];
        t->tg[t->nt].off = t->per_layer;
        t->tg_name[t->nt] = names[i];
        t->per_layer += static_cast<int64_t>(mc->hidden + dout[i]) * tc->lora_r;
        ++t->nt;
      }
  }
  t->RP = ((t->nt * tc->lora_r + 63) / 64) * 64;
  t->KA = t->dropout ? t->nt * mc->hidden : mc->hidden;
  t->n_train = static_cast<int64_t>(mc->n_layers) * t->per_layer;
  t->cur_S = tc->seq_len;
  t->cur_M = t->M;
  // Mistral-style sliding window: only a different mask once the sequence is longer than the window
  // (transformers 4.34.0 _make_sliding_window_causal_mask: triu(diagonal=-sliding_window), i.e. query i sees keys i - sw .. i)
  t->window = (mc->sliding_window > 0 && tc->seq_len > mc->sliding_window + 1) ? mc->sliding_window : 0;

  // the weight blocks (see Slot and WeightName)
  const int64_t d = mc->hidden, F = mc->ffn, V = mc->vocab, D = mc->head_dim, W = t->W, dq = t->dq, dkv = t->dkv;
  auto lslot = [&](bf16* Layer::*mem, int64_t n, bool nodecay, int nf4, int init) {
    t->lslots.push_back({mem, n, t->layer_used, nodecay, nf4, init});
    t->layer_used += n;
    return static_cast<int>(t->lslots.size()) - 1;
  };
  auto lname = [&](const char* key, int slot, int64_t off, int64_t rows, int64_t cols, int gu = 0) {
    t->lnames.push_back({key, nullptr, slot, off, rows, cols, gu});
  };
  const int qkv = lslot(&Layer::wqkv, W * d, false, W_QKV, INIT_NORMAL);
  lname("self_attn.q_proj.weight", qkv, 0, dq, d);
  lname("self_attn.k_proj.weight", qkv, dq * d, dkv, d);
  lname("self_attn.v_proj.weight", qkv, (dq + dkv) * d, dkv, d);
  lname("self_attn.o_proj.weight", lslot(&Layer::wo, d * dq, false, W_O, INIT_NORMAL), 0, d, dq);
  const int gu = lslot(&Layer::wgu, 2 * F * d, false, W_GU, INIT_NORMAL);
  lname("mlp.gate_proj.weight", gu, 0, F, d, GU_GATE);
  lname("mlp.up_proj.weight", gu, 0, F, d, GU_UP);
  lname("mlp.gate_up_proj.weight", gu, 0, 2 * F, d, GU_BOTH);  // GLM (modeling_glm GlmMLP: chunk(2))
  lname("mlp.down_proj.weight", lslot(&Layer::wdown, d * F, false, W_DOWN, INIT_NORMAL), 0, d, F);
  if (!t->ext.no_pre_norms) {
    lname("input_layernorm.weight", lslot(&Layer::norm1, d, true, -1, INIT_ONE), 0, d, 1);
    lname("post_attention_layernorm.weight", lslot(&Layer::norm2, d, true, -1, INIT_ONE), 0, d, 1);
  }
  if (t->ext.qkv_bias) {  // Qwen2, GLM: one [W] vector in the row order of wqkv
    const int b = lslot(&Layer::bias, W, true, -1, INIT_ZERO);
    lname("self_attn.q_proj.bias", b, 0, dq, 1);
    lname("self_attn.k_proj.bias", b, dq, dkv, 1);
    lname("self_attn.v_proj.bias", b, dq + dkv, dkv, 1);
  }
  if (t->ext.qk_norm) {  // Qwen3: q_norm | k_norm
    const int q = lslot(&Layer::qkn, 2 * D, true, -1, INIT_ONE);
    lname("self_attn.q_norm.weight", q, 0, D, 1);
    lname("self_attn.k_norm.weight", q, D, D, 1);
  }
  if (t->ext.qk_norm_full) {  // OLMo-2: q_norm [dq] | k_norm [dkv]
    const int q = lslot(&Layer::qkf, dq + dkv, true, -1, INIT_ONE);
    lname("self_attn.q_norm.weight", q, 0, dq, 1);
    lname("self_attn.k_norm.weight", q, dq, dkv, 1);
  }
  if (t->ext.post_norms) {  // the norms after the attention and the MLP sublayers, under Glm4's or (no_pre_norms) OLMo-2's names
    const int p = lslot(&Layer::pn, 2 * d, true, -1, INIT_ONE);
    const bool olmo = t->ext.no_pre_norms;
    lname(olmo ? "post_attention_layernorm.weight" : "post_self_attn_layernorm.weight", p, 0, d, 1);
    lname(olmo ? "post_feedforward_layernorm.weight" : "post_mlp_layernorm.weight", p, d, d, 1);
  }
  auto global = [&](bf16* dtx_trainer::*mem, const char* hf, const char* key, int64_t rows, int64_t cols, bool nodecay, int init) {
    t->gnames.push_back({key, hf, static_cast<int>(t->gslots.size()), 0, rows, cols, 0});
    t->gslots.push_back({mem, rows * cols, t->glob_used, nodecay, -1, init});
    t->glob_used += rows * cols;
  };
  global(&dtx_trainer::embed, "model.embed_tokens.weight", "embed_tokens.weight", V, d, false, INIT_NORMAL);
  global(&dtx_trainer::lm_head, "lm_head.weight", "lm_head.weight", V, d, false, INIT_NORMAL);
  global(&dtx_trainer::normf, "model.norm.weight", "norm.weight", d, 1, true, INIT_ONE);
}

// device bytes create_buffers() allocates for this configuration and activation layout: the same function in a sizing run,
// so that the plan cannot drift from the allocation (n_sms sizes the split-K partial buffers of the adapter gradients)
int64_t planned_bytes(const dtx_model_cfg* mc, const dtx_model_ext* ext, const dtx_train_cfg* tc, int world, int n_sms, int layout) {
  dtx_trainer p;
  setup_dims(&p, mc, ext, tc, world);
  p.n_sms = n_sms;
  p.dry = true;
  p.recompute = layout;
  create_buffers(&p);
  return static_cast<int64_t>(p.bytes_allocated);
}

}  // namespace

// ==================================================================================================
// C ABI
// ==================================================================================================
extern "C" {

int32_t dtx_abi_version(void) { return DTX_ABI_VERSION; }
const char* dtx_last_global_error(void) { return g_error.c_str(); }
const char* dtx_last_error(const dtx_trainer* t) { return t ? t->err.c_str() : g_error.c_str(); }

double dtx_lr_lambda(int32_t sched, int32_t step, int32_t warmup, int32_t total) {
  // transformers.optimization get_{linear,cosine,constant}_schedule_with_warmup lambdas
  if (sched == DTX_SCHED_CONSTANT) return 1.0;
  if (step < warmup) return static_cast<double>(step) / static_cast<double>(warmup > 1 ? warmup : 1);
  if (sched == DTX_SCHED_CONSTANT_WITH_WARMUP) return 1.0;
  if (sched == DTX_SCHED_LINEAR) {
    const double v = static_cast<double>(total - step) / static_cast<double>((total - warmup) > 1 ? (total - warmup) : 1);
    return v > 0.0 ? v : 0.0;
  }
  const double prog = static_cast<double>(step - warmup) / static_cast<double>((total - warmup) > 1 ? (total - warmup) : 1);
  const double v = 0.5 * (1.0 + cos(M_PI * 2.0 * 0.5 * prog));
  return v > 0.0 ? v : 0.0;
}

int32_t dtx_get_nccl_unique_id(void* out128) {
  NcclApi* api = nccl_api();
  if (!api) {
    g_error = "libnccl.so.2 could not be loaded";
    return DTX_ERR_NCCL;
  }
  int rc = api->GetUniqueId(out128);
  if (rc != 0) {
    g_error = std::string("ncclGetUniqueId failed: ") + (api->GetErrorString ? api->GetErrorString(rc) : "?");
    return DTX_ERR_NCCL;
  }
  return DTX_OK;
}

int32_t dtx_trainer_create(const dtx_model_cfg* mc, const dtx_train_cfg* tc, int32_t device, int32_t rank, int32_t world,
                           const void* nccl_unique_id, dtx_trainer** out) {
  return dtx_trainer_create_ext(mc, nullptr, tc, device, rank, world, nccl_unique_id, out);
}

int32_t dtx_rope_inv_freq(const dtx_model_cfg* mc, const dtx_model_ext* ext, float* out) {
  if (!mc || !out) {
    g_error = "rope_inv_freq: null argument";
    return DTX_ERR_INVALID;
  }
  if (mc->head_dim <= 0 || mc->head_dim % 2) {
    g_error = "rope_inv_freq: head_dim must be a positive even number";
    return DTX_ERR_INVALID;
  }
  int rc = check_ext(mc, ext);
  if (rc) return rc;
  dtx_model_ext e{};
  if (ext) e = *ext;
  rope_inv_freq(*mc, e, out);
  return DTX_OK;
}

int32_t dtx_trainer_create_ext(const dtx_model_cfg* mc, const dtx_model_ext* ext, const dtx_train_cfg* tc, int32_t device,
                               int32_t rank, int32_t world, const void* nccl_unique_id, dtx_trainer** out) {
  if (!mc || !tc || !out) {
    g_error = "null argument";
    return DTX_ERR_INVALID;
  }
  *out = nullptr;
  int rc = check_cfg(mc, tc);
  if (rc == DTX_OK) rc = check_ext(mc, ext);
  if (rc) return rc;
  if (world < 1 || rank < 0 || rank >= world) {
    g_error = "bad rank/world";
    return DTX_ERR_INVALID;
  }
  if (world > 1 && !nccl_unique_id) {
    g_error = "world > 1 needs an NCCL unique id";
    return DTX_ERR_INVALID;
  }

  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) {
    g_error = std::string("cudaSetDevice failed (no CUDA device? there is no CPU fallback): ") + cudaGetErrorString(e);
    return DTX_ERR_CUDA;
  }
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, device);
  if (e != cudaSuccess || prop.major != 9) {
    g_error = "libdtxtune requires an sm_90 (Hopper H100) device";
    return DTX_ERR_CUDA;
  }
  dtx_trainer* t = new dtx_trainer();
  setup_dims(t, mc, ext, tc, world);
  t->device = device;
  t->rank = rank;
  if (prop.multiProcessorCount > 0) t->n_sms = prop.multiProcessorCount;
  // Activation layout.  Automatic: keep every layer's activations when that fits in the free memory with kHeadroomBytes to
  // spare (the bf16 base is resident at this point even for QLoRA, so this is the true peak), else recompute per layer.
  t->recompute = tc->recompute ? tc->recompute : KEEP_ALL;
  if (tc->recompute == 0) {
    size_t free_b = 0, total_b = 0;
    e = cudaMemGetInfo(&free_b, &total_b);
    if (e != cudaSuccess) {
      g_error = std::string("cudaMemGetInfo failed: ") + cudaGetErrorString(e);
      delete t;
      return DTX_ERR_CUDA;
    }
    const int64_t keep = planned_bytes(mc, ext, tc, world, t->n_sms, KEEP_ALL);
    const int64_t layer = planned_bytes(mc, ext, tc, world, t->n_sms, RECOMPUTE_LAYER);
    const int64_t avail = static_cast<int64_t>(free_b) - kHeadroomBytes;
    if (keep <= avail) {
      t->recompute = KEEP_ALL;
    } else if (layer <= avail) {
      t->recompute = RECOMPUTE_LAYER;
    } else {
      char buf[320];
      snprintf(buf, sizeof(buf),
               "device memory too small: keeping all activations needs %lld bytes, recomputing per layer %lld bytes, "
               "%lld bytes are free (%lld kept in reserve)",
               static_cast<long long>(keep), static_cast<long long>(layer), static_cast<long long>(free_b),
               static_cast<long long>(kHeadroomBytes));
      g_error = buf;
      delete t;
      return DTX_ERR_CUDA;
    }
  }
  cudaStreamCreateWithFlags(&t->stream, cudaStreamNonBlocking);
  cudaEventCreate(&t->ev0);
  cudaEventCreate(&t->ev1);
  cudaEventCreate(&t->ev_fb);
  cudaEventCreate(&t->ev_ar);
  if (t->full) {
    cudaStreamCreateWithFlags(&t->comm_stream, cudaStreamNonBlocking);
    cudaEventCreateWithFlags(&t->ev_comm, cudaEventDisableTiming);
    t->ev_layer.resize(mc->n_layers + 1);
    for (auto& e : t->ev_layer) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    t->ev_ag.resize(mc->n_layers + 1);
    for (auto& e : t->ev_ag) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    t->ag_pending.assign(mc->n_layers + 1, 0);
  }
  rc = create_buffers(t);
  if (rc) {
    g_error = t->err;
    dtx_trainer_destroy(t);
    return rc;
  }
  if (world > 1) {
    NcclApi* api = nccl_api();
    if (!api) {
      g_error = "libnccl.so.2 could not be loaded";
      dtx_trainer_destroy(t);
      return DTX_ERR_NCCL;
    }
    UidByValue uid;
    memcpy(uid.internal, nccl_unique_id, 128);
    int nrc = api->CommInitRank(&t->nccl_comm, world, uid, rank);
    if (nrc != 0) {
      g_error = std::string("ncclCommInitRank failed: ") + (api->GetErrorString ? api->GetErrorString(nrc) : "?");
      dtx_trainer_destroy(t);
      return DTX_ERR_NCCL;
    }
  }
  e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    g_error = std::string("device error during create: ") + cudaGetErrorString(e);
    dtx_trainer_destroy(t);
    return DTX_ERR_CUDA;
  }
  *out = t;
  return DTX_OK;
}

void dtx_trainer_destroy(dtx_trainer* t) {
  if (!t) return;
  cudaSetDevice(t->device);
  cudaDeviceSynchronize();  // includes the side stream's collectives
  if (t->nccl_comm) {
    NcclApi* api = nccl_api();
    if (api) api->CommDestroy(t->nccl_comm);
  }
  for (void* p : t->allocs) cudaFree(p);
  if (t->ev0) cudaEventDestroy(t->ev0);
  if (t->ev1) cudaEventDestroy(t->ev1);
  if (t->ev_fb) cudaEventDestroy(t->ev_fb);
  if (t->ev_ar) cudaEventDestroy(t->ev_ar);
  if (t->ev_comm) cudaEventDestroy(t->ev_comm);
  for (auto e : t->ev_layer) cudaEventDestroy(e);
  for (auto e : t->ev_ag) cudaEventDestroy(e);
  if (t->comm_stream) cudaStreamDestroy(t->comm_stream);
  if (t->copy_stream) cudaStreamDestroy(t->copy_stream);
  for (int i = 0; i < 4; ++i) {
    if (t->ev_deq[i]) cudaEventDestroy(t->ev_deq[i]);
    if (t->ev_scr[i]) cudaEventDestroy(t->ev_scr[i]);
  }
  if (t->stream) cudaStreamDestroy(t->stream);
  delete t;
}

int32_t dtx_load_tensor(dtx_trainer* t, const char* name, const void* host, int32_t dtype, const int64_t* shape, int32_t nd) {
  if (!t || !name || !host || !shape || nd < 1 || nd > 2) return t ? t->fail(DTX_ERR_INVALID, "bad argument") : DTX_ERR_INVALID;
  cudaSetDevice(t->device);
  wait_all_weights(t);      // full-parameter SFT: no all-gather may still be writing the weight buffer
  t->master_valid = false;  // ... and the fp32 master copies are rebuilt from the bf16 weights at the next step
  const int64_t d = t->mc.hidden, r = t->tc.lora_r;
  const int64_t rows = shape[0], cols = nd == 2 ? shape[1] : 1;
  auto expect = [&](int64_t er, int64_t ec) { return rows == er && cols == ec; };
  int layer = -1;
  const char* rest = nullptr;
  if (parse_layer(name, &layer, &rest) && (strstr(rest, "lora_A") || strstr(rest, "lora_B"))) {
    if (layer < 0 || layer >= t->mc.n_layers) return t->fail(DTX_ERR_INVALID, "%s: layer out of range", name);
    const bool is_lora_a = strstr(rest, "lora_A") != nullptr;
    char which = 0;
    if (strstr(rest, "q_proj")) which = 'q';
    else if (strstr(rest, "k_proj")) which = 'k';
    else if (strstr(rest, "v_proj")) which = 'v';
    const int ti = which ? target_index(t, which) : -1;
    if (ti < 0) return t->fail(DTX_ERR_INVALID, "%s: module is not a LoRA target", name);
    float* base = t->params + static_cast<int64_t>(layer) * t->per_layer + t->tg[ti].off;
    const int64_t d_out = t->tg[ti].d_out;
    std::vector<float> f;
    if (is_lora_a) {  // [r, d] -> stored transposed [d, r]
      if (!expect(r, d)) return t->fail(DTX_ERR_INVALID, "%s: expected [%lld,%lld]", name, (long long)r, (long long)d);
      to_f32_host(host, dtype, r * d, f);
      std::vector<float> tr(d * r);
      for (int64_t j = 0; j < r; ++j)
        for (int64_t c = 0; c < d; ++c) tr[c * r + j] = f[j * d + c];
      CKM(upload_sync(base, tr.data(), tr.size() * 4, t->stream));
    } else {
      if (!expect(d_out, r)) return t->fail(DTX_ERR_INVALID, "%s: expected [%lld,%lld]", name, (long long)d_out, (long long)r);
      to_f32_host(host, dtype, d_out * r, f);
      CKM(upload_sync(base + d * r, f.data(), f.size() * 4, t->stream));
    }
    t->have_lora = true;
    int rc = refresh_shadows(t);
    if (rc) return rc;
    CKM(cudaStreamSynchronize(t->stream));
    return DTX_OK;
  }
  NamedWeight nw;
  int rc = find_weight(t, name, &nw);
  if (rc) return rc;
  const WeightName& w = nw.w();
  if (t->quant4 && nw.nf4)
    return t->fail(DTX_ERR_STATE, "%s: the base weights are already NF4-packed; load tensors before dtx_quantize_base", name);
  if (!expect(w.rows, w.cols)) return t->fail(DTX_ERR_INVALID, "%s: expected [%lld,%lld]", name, (long long)w.rows, (long long)w.cols);
  std::vector<bf16> tmp;
  to_bf16_host(host, dtype, static_cast<size_t>(w.rows * w.cols), tmp);
  cudaError_t e = w.gu ? gu_copy(nw.slot, tmp.data(), w.gu, t->mc.ffn, d, cudaMemcpyHostToDevice, t->stream)
                       : cudaMemcpyAsync(nw.slot + w.off, tmp.data(), tmp.size() * sizeof(bf16), cudaMemcpyHostToDevice, t->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(t->stream);  // (see upload_sync)
  if (e != cudaSuccess) return t->fail(DTX_ERR_CUDA, "upload %s: %s", name, cudaGetErrorString(e));
  // a step with a hole in this map is refused (check_ready); GLM's gate_up_proj fills the gate_proj and up_proj rows
  for (size_t j = 0; j < nw.names->size(); ++j)
    if (j == nw.row || ((*nw.names)[j].gu & w.gu)) nw.loaded[j] = 1;
  return DTX_OK;
}

int32_t dtx_init_random_weights(dtx_trainer* t, uint64_t seed) {
  if (!t) return DTX_ERR_INVALID;
  if (t->quant4) return t->fail(DTX_ERR_STATE, "init_random_weights: the base weights are already NF4-packed");
  t->master_valid = false;
  cudaSetDevice(t->device);
  cudaStream_t s = t->stream;
  uint64_t k = seed * 1000003ull;
  // HF _init_weights: Linear and Embedding weights normal(0.02), Linear biases 0, RMSNorm weights 1
  auto fill = [&](bf16* p, int64_t n, int init) {
    return init == INIT_NORMAL ? fill_normal_bf16(p, n, 0.02f, ++k, s) : fill_const_bf16(p, n, init == INIT_ONE ? 1.0f : 0.0f, s);
  };
  for (const auto& sl : t->gslots) CK(fill(t->*sl.mem, sl.n, sl.init), 1);
  for (Layer& y : t->layers)
    for (const auto& sl : t->lslots) CK(fill(y.*sl.mem, sl.n, sl.init), 1);
  cudaError_t e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return t->fail(DTX_ERR_CUDA, "init_random_weights: %s", cudaGetErrorString(e));
  std::fill(t->loaded.begin(), t->loaded.end(), 1);
  return DTX_OK;
}

int32_t dtx_quantize_base(dtx_trainer* t, int32_t mode) {
  // mode 4: NF4 (--quantization int4).  Applies to the decoder-layer Linear weights (bitsandbytes skips lm_head; embeddings
  // and norms are never quantised).  The bf16 copies are replaced by packed codes + absmax and freed.
  if (!t) return DTX_ERR_INVALID;
  if (mode == 8)
    return t->fail(DTX_ERR_UNSUPPORTED, "--quantization int8 (bitsandbytes LLM.int8 with runtime outlier decomposition, "
                                         "cmd/tuning/train.py:231-232) is not implemented natively; use int4 or no quantization");
  if (mode != 4) return t->fail(DTX_ERR_INVALID, "quantize_base: mode must be 4 (nf4)");
  if (t->full) return t->fail(DTX_ERR_INVALID, "quantize_base: full-parameter SFT trains the bf16 weights themselves");
  if (t->quant4) return t->fail(DTX_ERR_STATE, "quantize_base: already quantised");
  {
    char buf[160];
    if (const char* m = t->missing_weight(buf, sizeof(buf)))
      return t->fail(DTX_ERR_STATE, "quantize_base: base weight %s is not loaded yet", m);
  }
  cudaSetDevice(t->device);
  for (const auto& sl : t->lslots)
    if (sl.nf4 >= 0 && sl.n % 64) return t->fail(DTX_ERR_INVALID, "quantize_base: matrix sizes must be multiples of the 64-element NF4 block");
  cudaStream_t s = t->stream;
  for (Layer& y : t->layers) {
    for (const auto& sl : t->lslots) {
      const int i = sl.nf4;
      if (i < 0) continue;
      if (!t->alloc(&y.q4[i], static_cast<size_t>(sl.n / 2)) || !t->alloc(&y.absmax[i], static_cast<size_t>(sl.n / 64))) return DTX_ERR_CUDA;
      CK(nf4_quantize_pack(y.*sl.mem, y.q4[i], y.absmax[i], sl.n, s), 1);
    }
    CKM(cudaStreamSynchronize(s));
    for (const auto& sl : t->lslots) {
      if (sl.nf4 < 0) continue;
      t->release(y.*sl.mem, static_cast<size_t>(sl.n) * sizeof(bf16));
      y.*sl.mem = nullptr;
      t->base_bytes += sl.n / 2 + (sl.n / 64) * 4 - sl.n * static_cast<int64_t>(sizeof(bf16));
    }
  }
  for (const auto& sl : t->lslots)
    if (sl.nf4 >= 0 && !t->alloc(&t->scratch_w[sl.nf4], static_cast<size_t>(sl.n))) return DTX_ERR_CUDA;
  if (g_nf4_prefetch) {
    CKM(cudaStreamCreateWithFlags(&t->copy_stream, cudaStreamNonBlocking));
    for (int i = 0; i < 4; ++i) {
      CKM(cudaEventCreateWithFlags(&t->ev_deq[i], cudaEventDisableTiming));
      CKM(cudaEventCreateWithFlags(&t->ev_scr[i], cudaEventDisableTiming));
    }
  }
  t->quant4 = true;
  return DTX_OK;
}

int64_t dtx_base_weight_bytes(const dtx_trainer* t) { return t ? t->base_bytes : 0; }

int32_t dtx_init_lora(dtx_trainer* t, uint64_t seed) {
  if (!t) return DTX_ERR_INVALID;
  if (t->full) return t->fail(DTX_ERR_STATE, "init_lora: this trainer was created for full-parameter SFT (no adapters)");
  cudaSetDevice(t->device);
  const int64_t d = t->mc.hidden, r = t->tc.lora_r;
  std::vector<float> host(t->n_train, 0.f);
  // peft 0.5.0 LoraLayer.reset_lora_parameters: kaiming_uniform_(A, a=sqrt(5)) => U(-1/sqrt(fan_in), +1/sqrt(fan_in)); B = 0
  const float bound = 1.0f / sqrtf(static_cast<float>(d));
  uint64_t x = seed ? seed : 0x9E3779B97F4A7C15ull;
  auto next = [&]() {
    x += 0x9E3779B97F4A7C15ull;
    uint64_t z = x;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    return static_cast<float>(z >> 40) * (1.0f / 16777216.0f);
  };
  for (int64_t l = 0; l < t->mc.n_layers; ++l)
    for (int ti = 0; ti < t->nt; ++ti) {
      float* a = host.data() + l * t->per_layer + t->tg[ti].off;
      for (int64_t i = 0; i < d * r; ++i) a[i] = (2.f * next() - 1.f) * bound;
    }
  CKM(upload_sync(t->params, host.data(), host.size() * 4, t->stream));
  CKM(cudaMemsetAsync(t->adam_m, 0, t->n_train * 4, t->stream));
  CKM(cudaMemsetAsync(t->adam_v, 0, t->n_train * 4, t->stream));
  t->opt_step = 0;
  t->micro_idx = 0;
  int rc = refresh_shadows(t);
  if (rc) return rc;
  CKM(cudaStreamSynchronize(t->stream));
  t->have_lora = true;
  return DTX_OK;
}

int32_t dtx_step(dtx_trainer* t, const int32_t* ids, const int32_t* labels, const int32_t* seq_lens, int32_t seq_len_batch,
                 int32_t flags, float* loss, float* gnorm, float* lr, int32_t* stepped) {
  if (!t || !ids || !labels) return t ? t->fail(DTX_ERR_INVALID, "null batch") : DTX_ERR_INVALID;
  cudaSetDevice(t->device);
  int rc = check_ready(t);
  if (rc == DTX_OK) rc = set_batch_shape(t, seq_len_batch, seq_lens != nullptr);
  if (rc) return rc;
  return do_step(t, BatchInput{ids, labels, seq_lens, false, t->cur_S}, flags, loss, gnorm, lr, stepped);
}

int32_t dtx_step_device(dtx_trainer* t, const void* d_ids, const void* d_labels, const void* d_seq_lens, int32_t seq_len_batch,
                        int32_t flags, float* loss, float* gnorm, float* lr, int32_t* stepped) {
  if (!t || !d_ids || !d_labels) return t ? t->fail(DTX_ERR_INVALID, "null batch") : DTX_ERR_INVALID;
  cudaSetDevice(t->device);
  int rc = check_ready(t);
  if (rc == DTX_OK) rc = set_batch_shape(t, seq_len_batch, d_seq_lens != nullptr);
  if (rc) return rc;
  const BatchInput in{static_cast<const int32_t*>(d_ids), static_cast<const int32_t*>(d_labels), static_cast<const int32_t*>(d_seq_lens),
                      true, t->cur_S};
  return do_step(t, in, flags, loss, gnorm, lr, stepped);
}

int32_t dtx_eval_loss(dtx_trainer* t, const int32_t* ids, const int32_t* labels, const int32_t* seq_lens, int32_t seq_len_batch,
                      float* loss_out, float* row_sum_out, int32_t* row_valid_out) {
  if (!t || !ids || !labels) return t ? t->fail(DTX_ERR_INVALID, "null batch") : DTX_ERR_INVALID;
  cudaSetDevice(t->device);
  int rc = check_ready(t);
  if (rc == DTX_OK) rc = set_batch_shape(t, seq_len_batch, seq_lens != nullptr);
  if (rc) return rc;
  RowStats rows{row_sum_out, row_valid_out};
  const bool want_rows = row_sum_out || row_valid_out;
  rc = run_batch(t, BatchInput{ids, labels, seq_lens, false, t->cur_S}, false, want_rows ? &rows : nullptr);
  if (rc) return rc;
  float h = 0.f;
  CKM(cudaMemcpyAsync(&h, t->d_loss, 4, cudaMemcpyDeviceToHost, t->stream));
  cudaError_t e = cudaStreamSynchronize(t->stream);
  if (e != cudaSuccess) return t->fail(DTX_ERR_CUDA, "eval failed on device: %s", cudaGetErrorString(e));
  for (int k = 0; want_rows && k < t->tc.micro_batch; ++k) {
    if (row_sum_out) row_sum_out[rows.order[k]] = t->h_row_sum[static_cast<size_t>(k)];
    if (row_valid_out) row_valid_out[rows.order[k]] = t->h_row_valid[static_cast<size_t>(k)];
  }
  if (loss_out) *loss_out = h;
  return DTX_OK;
}

int32_t dtx_allreduce_host(dtx_trainer* t, double* inout, int32_t n) {
  if (!t || !inout || n < 0 || n > 64) return t ? t->fail(DTX_ERR_INVALID, "allreduce_host: n must be in [0, 64]") : DTX_ERR_INVALID;
  if (t->world == 1 || n == 0) return DTX_OK;
  cudaSetDevice(t->device);
  NcclApi* api = nccl_api();
  if (!api || !t->nccl_comm) return t->fail(DTX_ERR_NCCL, "NCCL communicator missing for world=%d", t->world);
  CKM(cudaMemcpyAsync(t->d_host_red, inout, static_cast<size_t>(n) * 8, cudaMemcpyHostToDevice, t->stream));
  int rc = api->AllReduce(t->d_host_red, t->d_host_red, static_cast<size_t>(n), kNcclFloat64, kNcclSum, t->nccl_comm, t->stream);
  if (rc != 0) return t->fail(DTX_ERR_NCCL, "ncclAllReduce failed: %s", api->GetErrorString ? api->GetErrorString(rc) : "?");
  CKM(cudaMemcpyAsync(inout, t->d_host_red, static_cast<size_t>(n) * 8, cudaMemcpyDeviceToHost, t->stream));
  CKM(cudaStreamSynchronize(t->stream));
  return DTX_OK;
}

static int32_t export_lora_tensor(dtx_trainer* t, const float* flat, const char* name, void* host_out, int64_t nbytes) {
  if (!t || !name || !host_out) return t ? t->fail(DTX_ERR_INVALID, "null argument") : DTX_ERR_INVALID;
  if (t->full || !flat) return t->fail(DTX_ERR_STATE, "no adapters: this trainer was created for full-parameter SFT");
  cudaSetDevice(t->device);
  const int64_t d = t->mc.hidden, r = t->tc.lora_r;
  int layer = -1;
  const char* rest = nullptr;
  if (!parse_layer(name, &layer, &rest) || layer < 0 || layer >= t->mc.n_layers)
    return t->fail(DTX_ERR_INVALID, "bad adapter tensor name %s", name);
  char which = 0;
  if (strstr(rest, "q_proj")) which = 'q';
  else if (strstr(rest, "k_proj")) which = 'k';
  else if (strstr(rest, "v_proj")) which = 'v';
  const int ti = which ? target_index(t, which) : -1;
  if (ti < 0) return t->fail(DTX_ERR_INVALID, "%s: module is not a LoRA target", name);
  const int64_t d_out = t->tg[ti].d_out;
  const bool is_a = strstr(rest, "lora_A") != nullptr;
  if (nbytes < (is_a ? d : d_out) * r * 4) return t->fail(DTX_ERR_INVALID, "%s: output buffer too small", name);
  const float* base = flat + static_cast<int64_t>(layer) * t->per_layer + t->tg[ti].off;
  CKM(cudaStreamSynchronize(t->stream));
  std::vector<float> tmp(d * r);
  float* out = static_cast<float*>(host_out);
  if (strstr(rest, "lora_A")) {
    CKM(cudaMemcpyAsync(tmp.data(), base, d * r * 4, cudaMemcpyDeviceToHost, t->stream));
    CKM(cudaStreamSynchronize(t->stream));
    for (int64_t c = 0; c < d; ++c)
      for (int64_t j = 0; j < r; ++j) out[j * d + c] = tmp[c * r + j];
  } else if (strstr(rest, "lora_B")) {
    CKM(cudaMemcpyAsync(out, base + d * r, d_out * r * 4, cudaMemcpyDeviceToHost, t->stream));
    CKM(cudaStreamSynchronize(t->stream));
  } else {
    return t->fail(DTX_ERR_INVALID, "%s: expected lora_A or lora_B", name);
  }
  return DTX_OK;
}

int32_t dtx_export_adapter(dtx_trainer* t, const char* name, void* host_out, int64_t nbytes) {
  return export_lora_tensor(t, t ? t->params : nullptr, name, host_out, nbytes);
}
int32_t dtx_export_adapter_grad(dtx_trainer* t, const char* name, void* host_out, int64_t nbytes) {
  return export_lora_tensor(t, t ? t->grads : nullptr, name, host_out, nbytes);
}

// Full-parameter SFT: one weight (grad = 0) or its accumulated gradient (grad = 1) by HF name, as bf16 bit patterns in the HF
// layout (gate / up rows taken back out of the GU-interleaved storage).  Gradients are only complete on a single rank.
int32_t dtx_export_weight(dtx_trainer* t, const char* name, void* host_out, int64_t nbytes, int32_t grad) {
  if (!t || !name || !host_out) return t ? t->fail(DTX_ERR_INVALID, "null argument") : DTX_ERR_INVALID;
  if (!t->full) return t->fail(DTX_ERR_STATE, "export_weight: only for full-parameter SFT trainers (LoRA: dtx_export_adapter)");
  cudaSetDevice(t->device);
  wait_all_weights(t);
  CKM(cudaStreamSynchronize(t->stream));
  NamedWeight nw;
  int rc = find_weight(t, name, &nw);
  if (rc) return rc;
  const WeightName& w = nw.w();
  if (nbytes < w.rows * w.cols * 2) return t->fail(DTX_ERR_INVALID, "%s: output buffer too small", name);
  bf16* slot = grad ? t->grad_of(nw.slot) : nw.slot;
  cudaError_t e = w.gu ? gu_copy(slot, static_cast<bf16*>(host_out), w.gu, t->mc.ffn, t->mc.hidden, cudaMemcpyDeviceToHost, t->stream)
                       : cudaMemcpyAsync(host_out, slot + w.off, w.rows * w.cols * 2, cudaMemcpyDeviceToHost, t->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(t->stream);
  if (e != cudaSuccess) return t->fail(DTX_ERR_CUDA, "export %s: %s", name, cudaGetErrorString(e));
  return DTX_OK;
}

int64_t dtx_num_trainable(const dtx_trainer* t) { return t ? t->n_train : 0; }
int32_t dtx_recompute(const dtx_trainer* t) { return t ? t->recompute : DTX_ERR_INVALID; }
int64_t dtx_device_bytes(const dtx_trainer* t) { return t ? static_cast<int64_t>(t->bytes_allocated) : 0; }

int32_t dtx_plan_device_bytes(const dtx_model_cfg* mc, const dtx_train_cfg* tc, int32_t world, int32_t layout, int64_t* bytes_out) {
  return dtx_plan_device_bytes_ext(mc, nullptr, tc, world, layout, bytes_out);
}
int32_t dtx_plan_device_bytes_ext(const dtx_model_cfg* mc, const dtx_model_ext* ext, const dtx_train_cfg* tc, int32_t world,
                                  int32_t layout, int64_t* bytes_out) {
  if (!mc || !tc || !bytes_out || world < 1) {
    g_error = "plan_device_bytes: null argument or world < 1";
    return DTX_ERR_INVALID;
  }
  if (layout != KEEP_ALL && layout != RECOMPUTE_LAYER) {
    g_error = "plan_device_bytes: layout must be 1 (keep all activations) or 2 (recompute per layer)";
    return DTX_ERR_INVALID;
  }
  int rc = check_cfg(mc, tc);
  if (rc == DTX_OK) rc = check_ext(mc, ext);
  if (rc) return rc;
  *bytes_out = planned_bytes(mc, ext, tc, world, 132, layout);  // split-K buffers sized for the 132 SMs of an H100 SXM
  return DTX_OK;
}
int64_t dtx_launch_count(const dtx_trainer* t) { return t ? t->launches : 0; }
float dtx_last_step_ms(const dtx_trainer* t) { return t ? t->last_ms : 0.f; }
int32_t dtx_last_step_groups(const dtx_trainer* t) { return t ? t->last_groups : 0; }

int32_t dtx_plan_packed_rows(int32_t micro_batch, const int32_t* seq_lens, int32_t seq_len_batch, int32_t* row_start_out) {
  if (!seq_lens || !row_start_out || micro_batch < 1 || micro_batch > 64 || seq_len_batch < 128 || seq_len_batch % 128) return DTX_ERR_INVALID;
  RowStarts rs;
  const bool saves = packed_rows(seq_lens, micro_batch, seq_len_batch, &rs);
  for (int b = 0; b <= micro_batch; ++b) row_start_out[b] = rs.start[b];
  return saves ? 1 : 0;
}

int32_t dtx_plan_length_groups(const dtx_model_cfg* mc, int32_t micro_batch, int32_t n_sms, const int32_t* seq_lens, int32_t seq_len_batch,
                               int32_t* order_out, int32_t* group_start_out, int32_t* group_len_out) {
  if (!mc || !seq_lens || !order_out || !group_start_out || !group_len_out || micro_batch < 1 || seq_len_batch < 128 || seq_len_batch % 128)
    return DTX_ERR_INVALID;
  const int hkv = mc->n_kv_heads > 0 ? mc->n_kv_heads : mc->n_heads;
  SubPlan plan;
  plan_groups(PlanDims{mc->hidden, mc->ffn, (mc->n_heads + 2 * hkv) * mc->head_dim, mc->n_heads * mc->head_dim, n_sms > 0 ? n_sms : 132,
                       micro_batch}, seq_lens, nullptr,
              seq_len_batch, &plan);
  if (plan.n <= 1) {  // one pass at the batch's padded length, rows in their own order
    for (int i = 0; i < micro_batch; ++i) order_out[i] = i;
    group_start_out[0] = 0;
    group_start_out[1] = micro_batch;
    group_len_out[0] = seq_len_batch;
    return 1;
  }
  for (int i = 0; i < micro_batch; ++i) order_out[i] = plan.order[i];
  for (int g = 0; g <= plan.n; ++g) group_start_out[g] = plan.start[g];
  for (int g = 0; g < plan.n; ++g) group_len_out[g] = plan.S[g];
  return plan.n;
}

int32_t dtx_last_step_timings(const dtx_trainer* t, float* out4) {
  if (!t || !out4) return DTX_ERR_INVALID;
  for (int i = 0; i < 4; ++i) out4[i] = t->seg_ms[i];
  return DTX_OK;
}

}  // extern "C"
