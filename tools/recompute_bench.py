"""Cost and reach of per-layer activation recompute (dtx_train_cfg.recompute) on one GPU.

(a) Llama-2-7B LoRA r=16 (q,v), batch 4 x 2048, synthetic batches as in bench.py: the "keep" and "layer" layouts run as
    alternating legs (warm-up + timed steps each, two rounds) on two trainers that start from the same seeded weights and see
    the same batches.  Reports ms/step, tokens/s, algorithmic TFLOP/s (28.36 GFLOP/token, BASELINE.md §2) and the FLOP/token
    each layout executes, and checks that both give bitwise-equal losses, grad norms, learning rates and trained adapters.
(b) Llama-2-7B LoRA at batch 8 x 4096, which only fits 80 GB with recompute: the layout automatic mode picks, the planned
    bytes of both layouts against the trainer's device_bytes, free memory after the first step, tokens/s.

    python tools/recompute_bench.py --out DIR      (writes DIR/recompute_bench.json; nothing else)
"""
from __future__ import annotations

import argparse
import dataclasses
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

ALGORITHMIC_FLOP_PER_TOKEN = 28.36e9  # BASELINE.md §2, headline config (no recompute counted)


def gpu_info() -> dict:
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                         check=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def flop_per_token(mc, tc, S: int, recompute: bool) -> float:
    """FLOP per token the step executes, from the shapes: forward GEMMs and backward dX GEMMs (incl. lm_head), causal attention
    forward and backward (2.5x forward), LoRA forward and backward (2x forward); with per-layer recompute also the q|k|v, o and
    gate|up GEMMs, the LoRA down/up-projections and the attention forward of every layer but the last."""
    d, F, V, L = mc.hidden, mc.ffn, mc.vocab, mc.n_layers
    W = (mc.n_heads + 2 * (mc.n_kv_heads or mc.n_heads)) * mc.head_dim
    dkv = (mc.n_kv_heads or mc.n_heads) * mc.head_dim
    d_out = {"q_proj": d, "k_proj": dkv, "v_proj": dkv}
    lora_fwd = sum(2 * tc.lora_r * (d + d_out[t]) for t in tc.lora_target)
    attn_fwd = 2 * d * S  # QK^T and PV over the causal half
    n_mm = L * (d * W + d * d + 3 * d * F) + V * d
    total = 2 * n_mm * 2 + L * attn_fwd * 3.5 + L * lora_fwd * 3
    if recompute:
        total += (L - 1) * (2 * (d * W + d * d + 2 * d * F) + attn_fwd + lora_fwd)
    return float(total)


def device_batches(mc, B, S, n):
    import torch
    from datatunerx_b200.tuning.synthetic import synthetic_batch
    out = []
    for i in range(n):
        ids, lab = synthetic_batch(i, 0, B, S, mc.vocab)
        out.append((torch.from_numpy(ids).cuda(), torch.from_numpy(lab).cuda()))
    torch.cuda.synchronize()
    return out


def timed_leg(tr, batches, first, warmup, steps):
    """`warmup` + `steps` steps on device-resident batches from batch index `first`: step outputs and host-clock ms/step."""
    import torch
    outs = []

    def run(i):
        a, b = batches[i % len(batches)]
        outs.append(tr.step_ptr(a.data_ptr(), b.data_ptr(), on_device=True))

    for i in range(warmup):
        run(first + i)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    dev_ms = []
    for i in range(steps):
        run(first + warmup + i)
        dev_ms.append(tr.last_step_ms)
    torch.cuda.synchronize()
    return outs, 1e3 * (time.perf_counter() - t0) / steps, float(np.median(dev_ms))


def part_a(args) -> dict:
    from datatunerx_b200 import lib as L
    mc = L.ModelConfig.llama2_7b()
    B, S = 4, 2048
    tc = L.TrainConfig(micro_batch=B, seq_len=S, total_steps=100, lora_r=16, lora_alpha=32.0, lora_dropout=0.0, lr=1e-4)
    algo = flop_per_token(mc, tc, S, False)
    assert abs(algo - ALGORITHMIC_FLOP_PER_TOKEN) < 0.01e9, algo
    trs = {}
    for layout in ("keep", "layer"):
        tr = L.Trainer(mc, dataclasses.replace(tc, recompute=layout))
        tr.init_random_weights(1234)
        tr.init_lora(4321)
        trs[layout] = tr
    batches = device_batches(mc, B, S, 4)
    legs, outs = [], {"keep": [], "layer": []}
    per_leg = args.warmup + args.steps
    for rnd in range(args.rounds):
        for layout in ("keep", "layer"):
            o, ms, dev_ms = timed_leg(trs[layout], batches, rnd * per_leg, args.warmup, args.steps)
            outs[layout] += o
            legs.append({"round": rnd, "layout": layout, "ms_per_step": ms, "device_ms_per_step_median": dev_ms})
    adapters = {k: {n: v.tobytes() for n, v in tr.export_adapter().items()} for k, tr in trs.items()}
    res = {"config": "Llama-2-7B LoRA r=16 (q,v), B=4, S=2048, synthetic batches", "legs": legs,
           "bitwise_equal": {"step_outputs": outs["keep"] == outs["layer"], "adapters": adapters["keep"] == adapters["layer"],
                             "steps_compared": len(outs["keep"])},
           "planned_bytes": {k: L.plan_device_bytes(mc, tc, 1, k) for k in ("keep", "layer")},
           "device_bytes": {k: tr.device_bytes for k, tr in trs.items()}}
    for layout in ("keep", "layer"):
        ms = [g["ms_per_step"] for g in legs if g["layout"] == layout]
        tok_s = B * S / (float(np.median(ms)) / 1e3)
        executed = flop_per_token(mc, tc, S, layout == "layer")
        res[layout] = {"ms_per_step_median": float(np.median(ms)), "ms_per_step_legs": ms, "tokens_per_s": tok_s,
                       "algorithmic_tflops": tok_s * ALGORITHMIC_FLOP_PER_TOKEN / 1e12,
                       "executed_gflop_per_token": executed / 1e9, "executed_tflops": tok_s * executed / 1e12}
    for tr in trs.values():
        tr.close()
    return res


def part_b(args) -> dict:
    import torch
    from datatunerx_b200 import lib as L
    mc = L.ModelConfig.llama2_7b()
    B, S = 8, 4096
    tc = L.TrainConfig(micro_batch=B, seq_len=S, total_steps=100, lora_r=16, lora_alpha=32.0, lora_dropout=0.0, lr=1e-4)
    planned = {k: L.plan_device_bytes(mc, tc, 1, k) for k in ("keep", "layer")}
    free_before, total = torch.cuda.mem_get_info()
    tr = L.Trainer(mc, tc)  # automatic layout
    res = {"config": "Llama-2-7B LoRA r=16 (q,v), B=8, S=4096, synthetic batches, recompute=auto", "layout": tr.recompute,
           "planned_bytes": planned, "device_bytes_after_create": tr.device_bytes, "free_bytes_before_create": free_before,
           "total_bytes": total}
    tr.init_random_weights(1234)
    tr.init_lora(4321)
    batches = device_batches(mc, B, S, 2)
    a, b = batches[0]
    first = tr.step_ptr(a.data_ptr(), b.data_ptr(), on_device=True)
    torch.cuda.synchronize()
    res["free_bytes_after_first_step"] = torch.cuda.mem_get_info()[0]
    outs, ms, dev_ms = timed_leg(tr, batches, 1, max(0, args.warmup - 1), args.steps)
    res.update({"first_step": first, "ms_per_step": ms, "device_ms_per_step_median": dev_ms, "tokens_per_s": B * S / (ms / 1e3),
                "losses_finite": bool(np.all(np.isfinite([first[0]] + [o[0] for o in outs]))),
                "executed_gflop_per_token": flop_per_token(mc, tc, S, tr.recompute == "layer") / 1e9})
    tr.close()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, metavar="DIR")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--skip-large", action="store_true", help="only part (a)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("recompute_bench needs a GPU (there is no CPU fallback)")
    res = {"gpu": gpu_info()}
    res["a_keep_vs_layer"] = part_a(args)
    if not args.skip_large:
        res["b_7b_b8_s4096"] = part_b(args)
    res["gpu_after"] = gpu_info()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "recompute_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
