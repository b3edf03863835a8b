"""Throughput of the model families beyond Llama-2 on one GPU, and the cost of the q|k|v bias in the GEMM epilogue.

  * Llama-3.1-8B shape (vocab 128 256, GQA 32 / 8, FFN 14 336, llama3 rope scaling) and Qwen2.5-7B shape (q/k/v biases, GQA 28 / 4,
    FFN 18 944, vocab 152 064), random-init weights, LoRA r=16 on q_proj,v_proj, micro-batch 4 x 2048 - the headline bench.py
    workload on the checkpoints people fine-tune today.  Per config: tokens/s of `--runs` timed windows of `--steps` optimizer
    steps (median and range), the activation layout automatic mode chose, the planned and the held device bytes.
  * Qwen3-8B shape (q/k RMSNorm, GQA 32 / 8, FFN 12 288, vocab 151 936) and Qwen3-4B shape (hidden 2560 with 32 x 128-wide
    heads: the attention is wider than the residual stream), the same workload.
  * The Qwen2.5-7B q|k|v GEMM (M 8192 x N 4608 x K 3584, fused RoPE epilogue) with and without the bias, and the Qwen3-8B one
    (M 8192 x N 6144 x K 4096) with and without the QK-norm epilogue, each pair alternated in one process, timed with CUDA
    events; qk_norm_bwd at the Qwen3-8B shape (time and GB/s of the bytes it must move).
  * GLM-4-9B-0414 shape (Glm4ForCausalLM: GLM's partial interleaved rotary, q/k/v biases, post-sublayer norms, GQA 32 / 2,
    FFN 13 696, vocab 151 552; q|k|v width 4608), the same workload.  Its q|k|v GEMM (M 8192 x N 4608 x K 4096) with the GLM
    epilogue against the half-split EPI_ROPE epilogue, both with the bias, alternated; post_norm_add at M 8192 x d 4096 (time and
    GB/s); attn_dkv_kernel (torch.profiler) at B 4 x S 2048 with GLM's 32 / 2 heads against Llama-3.1-8B's 32 / 8.
  * OLMo-2-1124-7B and -13B shapes (full-width q/k norm, post-sublayer norms and no pre-norms, vocab 100 352), the same workload,
    alternated with the Llama-2-7B shape over `--olmo-rounds` rounds (--olmo); OLMo-2-0325-32B (GQA 40 / 8, FFN 27 648, 64 layers)
    as QLoRA (NF4 base) at the largest micro-batch of 4, 2, 1 whose bf16 creation-time plan fits in 78 GB; qk_norm_full_rope_fwd
    and qk_norm_full_bwd (without and with the weight gradient) at M 8192 over the 7B (4096 + 4096) and 32B (5120 + 1024) q|k
    widths (time and GB/s of the bytes they must move).

The card's name and power limit are read in the same run and printed with the numbers.  Prints one JSON document; --out also
writes it to a file.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from datatunerx_b200 import lib as L  # noqa: E402
from datatunerx_b200.tuning.synthetic import synthetic_batch  # noqa: E402

CONFIGS = {
    "llama3.1-8b": L.ModelConfig(vocab=128256, hidden=4096, n_layers=32, n_heads=32, n_kv_heads=8, ffn=14336, rope_theta=500000.0,
                                 max_seq=131072,
                                 rope_scaling={"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                                               "original_max_position_embeddings": 8192}),
    "qwen2.5-7b": L.ModelConfig(vocab=152064, hidden=3584, n_layers=28, n_heads=28, n_kv_heads=4, ffn=18944, rope_theta=1000000.0,
                                rms_eps=1e-6, max_seq=32768, qkv_bias=True),
    "qwen3-8b": L.ModelConfig(vocab=151936, hidden=4096, n_layers=36, n_heads=32, n_kv_heads=8, ffn=12288, rope_theta=1000000.0,
                              rms_eps=1e-6, max_seq=40960, qk_norm=True),
    "qwen3-4b": L.ModelConfig(vocab=151936, hidden=2560, n_layers=36, n_heads=32, n_kv_heads=8, ffn=9728, rope_theta=1000000.0,
                              rms_eps=1e-6, max_seq=40960, qk_norm=True),
    "glm-4-9b-0414": L.ModelConfig(vocab=151552, hidden=4096, n_layers=40, n_heads=32, n_kv_heads=2, ffn=13696, rope_theta=10000.0,
                                   max_seq=32768, qkv_bias=True, rope_glm=True, post_norms=True),
}
OLMO2 = dict(vocab=100352, rope_theta=500000.0, rms_eps=1e-6, max_seq=4096, qk_norm_full=True, no_pre_norms=True, post_norms=True)
OLMO_CONFIGS = {
    "llama2-7b": L.ModelConfig.llama2_7b(),
    "olmo2-7b": L.ModelConfig(hidden=4096, n_layers=32, n_heads=32, n_kv_heads=32, ffn=11008, **OLMO2),
    "olmo2-13b": L.ModelConfig(hidden=5120, n_layers=40, n_heads=40, n_kv_heads=40, ffn=13824, **OLMO2),
}
OLMO2_32B = L.ModelConfig(hidden=5120, n_layers=64, n_heads=40, n_kv_heads=8, ffn=27648, **OLMO2)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, _, power = q.stdout.strip().splitlines()[0].partition(",")
    return {"name": name.strip(), "power_limit": power.strip()}


def train_throughput(name: str, mc: L.ModelConfig, B: int, S: int, steps: int, warmup: int, runs: int, quant: bool = False) -> dict:
    tc = L.TrainConfig(micro_batch=B, seq_len=S, total_steps=10 ** 6, lora_r=16, lora_alpha=32.0, lora_dropout=0.0, lr=1e-4)
    planned = {k: L.plan_device_bytes(mc, tc, 1, k) for k in ("keep", "layer")}
    tr = L.Trainer(mc, tc)
    tr.init_random_weights(1234)
    if quant:
        tr.quantize_base("int4")
    tr.init_lora(4321)
    batches = [synthetic_batch(s, 0, B, S, mc.vocab) for s in range(4)]
    for s in range(warmup):
        tr.step(*batches[s % 4])
    rates, losses = [], []
    for _ in range(runs):
        t0 = time.perf_counter()
        for s in range(steps):  # dtx_step returns after the step has finished on the device
            loss, _, _, _ = tr.step(*batches[s % 4])
        rates.append(B * S * steps / (time.perf_counter() - t0))
        losses.append(loss)
    out = {"config": name + (" qlora-nf4" if quant else ""), "micro_batch": B, "tokens_per_s_median": statistics.median(rates), "tokens_per_s_range": [min(rates), max(rates)],
           "layout": tr.recompute, "planned_bytes": planned, "held_bytes": tr.device_bytes, "last_loss": losses[-1]}
    tr.close()
    return out


def bias_gemm_cost(iters: int, rounds: int) -> dict:
    import torch
    M, N, K, H, Hkv, D = 8192, 4608, 3584, 28, 4, 128
    lib = L.load()
    g = torch.Generator().manual_seed(0)
    A = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16).cuda()
    Bw = (torch.randn(N, K, generator=g) * 0.02).to(torch.bfloat16).cuda()
    bias = (torch.randn(N, generator=g) * 0.1).to(torch.bfloat16).cuda()
    Cm = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    cs = torch.empty(S_ROPE, D // 2, 2, dtype=torch.float32, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    L.check(lib.dtx_rope_table(C.c_void_p(cs.data_ptr()), S_ROPE, D, 1000000.0, stream))
    P = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731

    def launch(with_bias: bool):
        L.check(lib.dtx_gemm_bias(P(A), K, P(Bw), K, 0, None, 0, None, 0, 0, P(Cm), N, None, 0, P(cs), S_ROPE, (H + Hkv) * D, None,
                                  M, N, K, L.EPI_ROPE, P(bias), stream) if with_bias else
                lib.dtx_gemm_fused(P(A), K, P(Bw), K, 0, None, 0, None, 0, 0, P(Cm), N, None, 0, P(cs), S_ROPE, (H + Hkv) * D,
                                   M, N, K, L.EPI_ROPE, stream))

    for wb in (False, True):
        for _ in range(10):
            launch(wb)
    times = {False: [], True: []}
    for _ in range(rounds):
        for wb in (False, True):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                launch(wb)
            e1.record()
            torch.cuda.synchronize()
            times[wb].append(e0.elapsed_time(e1) / iters)
    flop = 2.0 * M * N * K
    res = {}
    for wb, key in ((False, "no_bias"), (True, "bias")):
        ms = statistics.median(times[wb])
        res[key] = {"ms_median": ms, "ms_range": [min(times[wb]), max(times[wb])], "tflops": flop / ms / 1e9}
    res["shape"] = [M, N, K]
    return res


def _alternate(launch, variants, iters: int, rounds: int) -> dict:
    """ms per launch of every variant (CUDA events over `iters` launches), variants alternated `rounds` times"""
    import torch
    for v in variants:
        for _ in range(10):
            launch(v)
    times = {v: [] for v in variants}
    for _ in range(rounds):
        for v in variants:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                launch(v)
            e1.record()
            torch.cuda.synchronize()
            times[v].append(e0.elapsed_time(e1) / iters)
    return times


def qk_norm_cost(iters: int, rounds: int) -> dict:
    """Qwen3-8B: the q|k|v GEMM with the fused RoPE epilogue with and without QKNORM, and qk_norm_bwd on its dqkv"""
    import torch
    M, N, K, H, Hkv, D = 8192, 6144, 4096, 32, 8, 128
    dq, QK = H * D, (H + Hkv) * D
    lib = L.load()
    g = torch.Generator().manual_seed(0)
    A = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16).cuda()
    Bw = (torch.randn(N, K, generator=g) * 0.02).to(torch.bfloat16).cuda()
    wq = (1 + torch.randn(D, generator=g) * 0.1).to(torch.bfloat16).cuda()
    wk = (1 + torch.randn(D, generator=g) * 0.1).to(torch.bfloat16).cuda()
    Cm = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    pre = torch.empty(M, QK, dtype=torch.bfloat16, device="cuda")
    dy = (torch.randn(M, N, generator=g) * 0.1).to(torch.bfloat16).cuda()
    cs = torch.empty(S_ROPE, D // 2, 2, dtype=torch.float32, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    L.check(lib.dtx_rope_table(C.c_void_p(cs.data_ptr()), S_ROPE, D, 1000000.0, stream))
    P = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731

    def gemm(with_norm: bool):
        L.check(lib.dtx_gemm_qk_norm(P(A), K, P(Bw), K, 0, None, 0, None, 0, 0, P(Cm), N, P(pre), QK, P(cs), S_ROPE, QK, None,
                                     M, N, K, dq, P(wq), P(wk), 1e-6, stream) if with_norm else
                lib.dtx_gemm_fused(P(A), K, P(Bw), K, 0, None, 0, None, 0, 0, P(Cm), N, None, 0, P(cs), S_ROPE, QK,
                                   M, N, K, L.EPI_ROPE, stream))

    times = _alternate(gemm, (False, True), iters, rounds)
    flop = 2.0 * M * N * K
    res = {}
    for wn, key in ((False, "rope"), (True, "rope_qknorm")):
        ms = statistics.median(times[wn])
        res[key] = {"ms_median": ms, "ms_range": [min(times[wn]), max(times[wn])], "tflops": flop / ms / 1e9}
    res["gemm_shape"] = [M, N, K]
    # backward (LoRA: no dw): reads dy and the pre-norm x of the q|k columns, writes dx
    bwd = _alternate(lambda _: L.check(lib.dtx_qk_norm_bwd(P(dy), N, P(pre), QK, M, dq, QK, P(wq), P(wk), 1e-6, None, None, 0, 0,
                                                           stream)), (0,), iters, rounds)[0]
    ms = statistics.median(bwd)
    nbytes = 3 * M * QK * 2
    res["qk_norm_bwd"] = {"ms_median": ms, "ms_range": [min(bwd), max(bwd)], "bytes": nbytes, "gb_per_s": nbytes / ms / 1e6}
    return res


def glm_cost(iters: int, rounds: int) -> dict:
    """GLM-4-9B: the q|k|v GEMM with GLM's epilogue against the half-split one (both + bias), post_norm_add, and attn_dkv_kernel
    at 32 / 2 heads against 32 / 8"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    M, N, K, d = 8192, 4608, 4096, 4096
    lib = L.load()
    g = torch.Generator().manual_seed(0)
    A = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16).cuda()
    Bw = (torch.randn(N, K, generator=g) * 0.02).to(torch.bfloat16).cuda()
    bias = (torch.randn(N, generator=g) * 0.1).to(torch.bfloat16).cuda()
    Cm = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    cs = torch.empty(S_ROPE, 64, 2, dtype=torch.float32, device="cuda")  # the half-split table; GLM reads its first S x 32 pairs
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    L.check(lib.dtx_rope_table(C.c_void_p(cs.data_ptr()), S_ROPE, 128, 10000.0, stream))
    P = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
    QK = 34 * 128

    def gemm(glm: bool):
        L.check(lib.dtx_gemm_rope_glm(P(A), K, P(Bw), K, 0, None, 0, None, 0, 0, P(Cm), N, P(cs), S_ROPE, QK, None, M, N, K, P(bias),
                                      stream) if glm else
                lib.dtx_gemm_bias(P(A), K, P(Bw), K, 0, None, 0, None, 0, 0, P(Cm), N, None, 0, P(cs), S_ROPE, QK, None, M, N, K,
                                  L.EPI_ROPE, P(bias), stream))

    times = _alternate(gemm, (False, True), iters, rounds)
    flop = 2.0 * M * N * K
    res = {"gemm_shape": [M, N, K]}
    for glm, key in ((False, "rope_bias"), (True, "rope_glm_bias")):
        ms = statistics.median(times[glm])
        res[key] = {"ms_median": ms, "ms_range": [min(times[glm]), max(times[glm])], "tflops": flop / ms / 1e9}
    y, res_in = A[:, :d].contiguous(), A[:, :d].contiguous()
    w = (1 + torch.randn(d, generator=g) * 0.1).to(torch.bfloat16).cuda()
    out, rstd = torch.empty(M, d, dtype=torch.bfloat16, device="cuda"), torch.empty(M, dtype=torch.float32, device="cuda")
    pn = _alternate(lambda _: L.check(lib.dtx_post_norm_add(P(y), P(w), P(res_in), P(out), P(rstd), M, d, 1e-5, stream)), (0,), iters,
                    rounds)[0]
    ms = statistics.median(pn)
    nbytes = 3 * M * d * 2 + 4 * M
    res["post_norm_add"] = {"shape": [M, d], "ms_median": ms, "ms_range": [min(pn), max(pn)], "bytes": nbytes, "gb_per_s": nbytes / ms / 1e6}
    B, S, H = 4, 2048, 32
    for hkv, key in ((2, "attn_dkv_32_2"), (8, "attn_dkv_32_8")):
        W = (H + 2 * hkv) * 128
        qkv = (torch.randn(B * S, W, generator=g) * 0.5).to(torch.bfloat16).cuda()
        o, do = torch.empty(B * S, H * 128, dtype=torch.bfloat16, device="cuda"), (torch.randn(B * S, H * 128, generator=g) * 0.1).to(torch.bfloat16).cuda()
        lse, delta = torch.empty(B, H, S, dtype=torch.float32, device="cuda"), torch.empty(B, H, S, dtype=torch.float32, device="cuda")
        dqkv = torch.empty(B * S, W, dtype=torch.bfloat16, device="cuda")
        sc = 1.0 / 128 ** 0.5
        L.check(lib.dtx_attn_fwd(P(qkv), P(o), P(lse), B, S, H, hkv, sc, None, 0, stream))
        bwd = lambda: L.check(lib.dtx_attn_bwd(P(qkv), P(o), P(do), P(lse), P(delta), P(dqkv), B, S, H, hkv, sc, None, 0, None, 0,  # noqa: E731
                                               stream))
        for _ in range(5):
            bwd()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(iters):
                bwd()
            torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if "attn_dkv_kernel" in e.key]
        res[key] = {"ms_mean": sum(e.device_time_total for e in ev) / max(1, sum(e.count for e in ev)) / 1e3,
                    "grid_ctas": B * hkv * (S // 128)}
    return res


def olmo2_norm_cost(iters: int, rounds: int) -> dict:
    """qk_norm_full_rope_fwd and qk_norm_full_bwd at M 8192 over OLMo-2-7B's and -32B's q|k widths.  Bytes they must move: the
    forward reads the q|k columns and writes them twice (pre-norm copy, result in place); the backward reads dy and x and writes dx;
    with the weight gradient it also writes and reads 64 rows of fp32 partials."""
    import torch
    M = 8192
    lib = L.load()
    g = torch.Generator().manual_seed(0)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
    cs = torch.empty(S_ROPE, 64, 2, dtype=torch.float32, device="cuda")
    L.check(lib.dtx_rope_table(C.c_void_p(cs.data_ptr()), S_ROPE, 128, 500000.0, stream))
    res = {}
    for name, dq, dkv in (("7b", 4096, 4096), ("32b", 5120, 1024)):
        W, QK = dq + 2 * dkv, dq + dkv
        qkv = (torch.randn(M, W, generator=g) * 0.5).to(torch.bfloat16).cuda()
        dy = (torch.randn(M, W, generator=g) * 0.1).to(torch.bfloat16).cuda()
        pre = torch.empty(M, QK, dtype=torch.bfloat16, device="cuda")
        w = (1 + torch.randn(QK, generator=g) * 0.1).to(torch.bfloat16).cuda()
        dw = torch.empty(QK, dtype=torch.bfloat16, device="cuda")
        scratch = torch.empty(64 * QK, dtype=torch.float32, device="cuda")
        wq, wk = C.c_void_p(w.data_ptr()), C.c_void_p(w.data_ptr() + 2 * dq)

        def launch(v):
            if v == "fwd":
                L.check(lib.dtx_qk_norm_full_rope_fwd(P(qkv), W, M, dq, QK, wq, wk, 1e-6, P(cs), S_ROPE, None, P(pre), QK, stream))
            else:
                L.check(lib.dtx_qk_norm_full_bwd(P(dy), W, P(pre), QK, M, dq, QK, wq, wk, 1e-6, P(dw) if v == "bwd_dw" else None,
                                                 P(scratch), 0, stream))

        times = _alternate(launch, ("fwd", "bwd", "bwd_dw"), iters, rounds)
        out = {"shape": [M, dq, dkv]}
        for v in ("fwd", "bwd", "bwd_dw"):
            ms = statistics.median(times[v])
            nbytes = 3 * M * QK * 2 + (2 * 64 * QK * 4 if v == "bwd_dw" else 0)
            out[v] = {"ms_median": ms, "ms_range": [min(times[v]), max(times[v])], "bytes": nbytes, "gb_per_s": nbytes / ms / 1e6}
        res[name] = out
    return res


def olmo2_runs(a) -> dict:
    """OLMo-2-7B / 13B LoRA alternated with Llama-2-7B; OLMo-2-32B QLoRA"""
    runs = []
    for _ in range(a.olmo_rounds):
        for name, mc in OLMO_CONFIGS.items():
            runs.append(train_throughput(name, mc, a.batch, a.seq, a.steps, a.warmup, a.runs))
            print(json.dumps(runs[-1]), flush=True)
    tc = lambda B: L.TrainConfig(micro_batch=B, seq_len=a.seq, total_steps=1, lora_r=16, lora_dropout=0.0)  # noqa: E731
    B32 = next((B for B in (4, 2, 1) if L.plan_device_bytes(OLMO2_32B, tc(B), 1, "layer") <= 78e9), 1)
    runs.append(train_throughput("olmo2-32b", OLMO2_32B, B32, a.seq, max(2, a.steps // 2), a.warmup, a.runs, quant=True))
    print(json.dumps(runs[-1]), flush=True)
    return {"runs": runs, "norm_kernels": olmo2_norm_cost(iters=50, rounds=6)}


S_ROPE = 2048


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=4)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--seq", type=int, default=2048)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--out", default=None)
    ap.add_argument("--olmo", action="store_true", help="only the OLMo-2 measurements")
    ap.add_argument("--olmo-rounds", type=int, default=2)
    a = ap.parse_args()
    res = {"card": card(), "lora": "r=16 on q_proj,v_proj", "micro_batch": a.batch, "seq_len": a.seq, "runs": []}
    if a.olmo:
        res["olmo2"] = olmo2_runs(a)
    else:
        for name in a.configs.split(","):
            res["runs"].append(train_throughput(name, CONFIGS[name], a.batch, a.seq, a.steps, a.warmup, a.runs))
            print(json.dumps(res["runs"][-1]), flush=True)
        res["qkv_gemm_bias_cost"] = bias_gemm_cost(iters=50, rounds=6)
        res["qkv_gemm_qk_norm_cost"] = qk_norm_cost(iters=50, rounds=6)
        res["glm_cost"] = glm_cost(iters=50, rounds=6)
    res["card_after"] = card()
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
