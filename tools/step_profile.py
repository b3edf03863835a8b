"""Per-kernel profile of the headline training step (Llama-2-7B LoRA r=16, batch 4 x 2048) on one GPU.

The trainer is built as `bench.py --config 7b` builds it (same model, seeds 1234 / 4321, synthetic batches, device-resident
inputs); after the warm-up steps, --steps steps run under torch.profiler with CUDA activities only.  This is a run of its
own: tracing slows the host, so no timing is taken here besides the kernels' own durations.

Writes, under --out:
  step_trace.pt.trace.json  the profiler's Chrome trace
  step_profile.json         per kernel name (template arguments included, so every GEMM epilogue variant has its own row):
                            launches per step, ms per step, share of the step, and algorithmic TFLOP/s where the FLOP of the
                            kernel follow from the shapes (GEMMs and attention; the arithmetic is in gemm_flops / attn_flops)

DTX_LIB_PATH selects another build of the library (datatunerx_b200/lib.py), so one GPU session can profile two builds.

    python tools/step_profile.py --out DIR [--warmup 3] [--steps 3]
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

B, S, LORA_R = 4, 2048, 16
EPI_NAMES = {0: "EPI_BF16", 1: "EPI_F32", 2: "EPI_BF16_ADD", 3: "EPI_ROPE", 4: "EPI_SWIGLU_FWD", 5: "EPI_SWIGLU_BWD"}
GEMM_RE = re.compile(r"gemm_kernel<(\d+), (true|false), (true|false), (\d+)>")


def gpu_info() -> dict:
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                         check=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def gemm_variant(bn: int, a_mn: bool, b_mn: bool, epi: int) -> str:
    return f"gemm_kernel<{bn}, A_MN={int(a_mn)}, B_MN={int(b_mn)}, {EPI_NAMES[epi]}>"


def gemm_flops(mc, n_valid: float) -> dict:
    """FLOP per step of every GEMM launch of the LoRA (q, v) step with fused epilogues and all activations kept, keyed by the
    kernel variant that runs it (trainer.cu layer_fwd / fwd_bwd).  Shapes are as launched: the LoRA rank is padded to RP."""
    d, F, V, L = mc.hidden, mc.ffn, mc.vocab, mc.n_layers
    hkv = mc.n_kv_heads or mc.n_heads
    W = (mc.n_heads + 2 * hkv) * mc.head_dim
    RP = (2 * LORA_R + 63) // 64 * 64
    M = B * S
    f = collections.Counter()
    # forward, every layer
    f[gemm_variant(64, False, False, 0)] += L * 2 * M * RP * d            # LoRA down-projection t = h1 A_cat^T
    f[gemm_variant(256, False, False, 3)] += L * 2 * M * W * (d + RP)     # q|k|v + LoRA up-projection, RoPE epilogue
    f[gemm_variant(256, False, False, 2)] += L * 2 * M * d * d            # o projection + residual
    f[gemm_variant(256, False, False, 4)] += L * 2 * M * 2 * F * d        # gate|up, SwiGLU epilogue
    f[gemm_variant(256, False, False, 2)] += L * 2 * M * d * F            # down projection + residual
    f[gemm_variant(256, False, False, 1)] += 2 * n_valid * V * d          # lm_head, fp32 logits of the labelled rows
    # backward
    f[gemm_variant(256, False, True, 0)] += 2 * n_valid * d * V           # d h_f = dlogits W_lm
    f[gemm_variant(256, False, True, 5)] += L * 2 * M * F * d             # d act = dx Wdown, SwiGLU-backward epilogue
    f[gemm_variant(256, False, True, 0)] += L * 2 * M * d * 2 * F         # dh2 = d[gate|up] Wgu
    f[gemm_variant(256, False, True, 0)] += L * 2 * M * d * d             # d attn = dx_mid Wo
    f[gemm_variant(64, False, True, 0)] += L * 2 * M * RP * W             # dt = dqkv B_ext
    f[gemm_variant(256, False, True, 0)] += (L - 1) * 2 * M * d * (W + RP)  # dh1 = dqkv Wqkv + dt A_cat (not for layer 0)
    f[gemm_variant(64, True, True, 1)] += L * 2 * M * W * RP + L * 2 * M * d * RP  # split-K LoRA gradients of B_ext and A_cat
    return dict(f)


def attn_flops(mc) -> dict:
    """Causal attention: QK^T and PV over the lower triangle forward; the backward recomputes QK^T and adds dP, dV and dK
    (dK/dV kernel) and dP, dQ (dQ kernel)."""
    L, H, D = mc.n_layers, mc.n_heads, mc.head_dim
    mm = 2.0 * B * H * S * S * D / 2  # one S x S x D product over the causal half
    return {"attn_fwd_kernel": L * 2 * mm, "attn_dkv_kernel": L * 4 * mm, "attn_dq_kernel": L * 3 * mm}


def kernel_key(name: str) -> str:
    m = GEMM_RE.search(name)
    if m:
        return gemm_variant(int(m.group(1)), m.group(2) == "true", m.group(3) == "true", int(m.group(4)))
    m = re.search(r"(attn_[a-z]+_kernel)(<[^>]*>)?", name)
    if m:
        return m.group(1) + (m.group(2) or "")
    return name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    args = ap.parse_args()
    if args.warmup < 3:
        ap.error("--warmup must be at least 3")
    os.makedirs(args.out, exist_ok=True)

    import torch
    from torch.profiler import ProfilerActivity, profile
    from datatunerx_b200 import lib as L
    from datatunerx_b200.tuning.synthetic import synthetic_batch

    mc = L.ModelConfig.llama2_7b()
    total = args.warmup + args.steps + 2
    tc = L.TrainConfig(micro_batch=B, seq_len=S, total_steps=max(total, 100), lora_r=LORA_R, lora_alpha=32.0, lora_dropout=0.0,
                       lr=1e-4)
    tr = L.Trainer(mc, tc, device=0)
    tr.init_random_weights(1234)
    tr.init_lora(4321)
    n_batches = 4
    host = [synthetic_batch(i, 0, B, S, mc.vocab) for i in range(n_batches)]
    dev = [(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()) for a, b in host]
    torch.cuda.synchronize()

    def run(i):
        a, b = dev[i % n_batches]
        return tr.step_ptr(a.data_ptr(), b.data_ptr(), on_device=True, seq_lens_ptr=0, seq_len_batch=S)

    for i in range(args.warmup):
        run(i)
    torch.cuda.synchronize()
    steps = list(range(args.warmup, args.warmup + args.steps))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in steps:
            run(i)
        torch.cuda.synchronize()
    trace_path = os.path.join(args.out, "step_trace.pt.trace.json")
    prof.export_chrome_trace(trace_path)
    tr.close()

    with open(trace_path) as fh:
        events = json.load(fh)["traceEvents"]
    kernels = [e for e in events if e.get("cat") == "kernel" and "dur" in e]
    if not kernels:
        raise SystemExit("the trace holds no CUDA kernels: a GPU is needed")
    t_first = min(e["ts"] for e in kernels)
    t_last = max(e["ts"] + e["dur"] for e in kernels)
    step_ms = (t_last - t_first) / 1e3 / args.steps  # first kernel start to last kernel end, per step
    busy_ms = sum(e["dur"] for e in kernels) / 1e3 / args.steps

    # labelled rows of the profiled batches (lm_head and its backward run over those only)
    n_valid = float(np.mean([(host[i % n_batches][1][:, 1:] >= 0).sum() for i in steps]))
    flops = gemm_flops(mc, n_valid)
    flops.update(attn_flops(mc))

    agg = collections.defaultdict(lambda: {"count": 0, "us": 0.0})
    for e in kernels:
        k = kernel_key(e["name"])
        agg[k]["count"] += 1
        agg[k]["us"] += e["dur"]
    rows = []
    for k, v in agg.items():
        ms = v["us"] / 1e3 / args.steps
        fl = flops.get(k) if k in flops else next((f for n, f in flops.items() if k.startswith(n)), None)
        rows.append({"kernel": k, "count_per_step": v["count"] / args.steps, "ms_per_step": ms, "share_of_step": ms / step_ms,
                     "gflop_per_step": fl / 1e9 if fl else None, "tflops": fl / ms / 1e9 if fl else None})
    rows.sort(key=lambda r: -r["ms_per_step"])
    groups = collections.Counter()
    for r in rows:
        g = "gemm" if r["kernel"].startswith("gemm_kernel") else ("attention" if r["kernel"].startswith("attn_") else "other")
        groups[g] += r["ms_per_step"]
    out = {"gpu": gpu_info(), "lib": L.LIB_PATH, "config": f"Llama-2-7B LoRA r={LORA_R} (q,v), batch {B} x {S}",
           "profiled_steps": args.steps, "warmup": args.warmup, "step_ms": step_ms, "kernel_busy_ms": busy_ms,
           "labelled_rows": n_valid,
           "groups": {g: {"ms_per_step": ms, "share_of_step": ms / step_ms} for g, ms in groups.items()},
           "kernels": rows}
    with open(os.path.join(args.out, "step_profile.json"), "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps({"step_ms": step_ms, "groups": out["groups"],
                      "top": [(r["kernel"], round(r["ms_per_step"], 3), r["tflops"] and round(r["tflops"], 1)) for r in rows[:14]]}))


if __name__ == "__main__":
    main()
