"""Is the training step deterministic in context?  One 7B-shaped layer, lr = 0 (parameters never change): every step of one
trainer sees identical inputs, so loss / grad-norm / gradients must repeat bitwise - within a trainer and across trainers."""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from datatunerx_b200 import lib as L  # noqa: E402
from datatunerx_b200.tuning.synthetic import synthetic_batch  # noqa: E402


def main(B=2, S=2048, layers=1):
    mc = L.ModelConfig(vocab=32000, hidden=4096, n_layers=layers, n_heads=32, ffn=11008)
    tc = L.TrainConfig(micro_batch=B, seq_len=S, total_steps=100, lora_r=16, lora_alpha=32.0, lora_dropout=0.0, lr=0.0)
    ids, labels = synthetic_batch(0, 0, B, S, mc.vocab)
    rng = np.random.default_rng(5)
    for opts in ({}, {}, {"fused_epilogues": 0}, {"attn_fwd_exp_fma_every": 0}):
        for k, v in opts.items():
            L.set_option(k, v)
        tr = L.Trainer(mc, tc)
        tr.init_random_weights(1234)
        tr.init_lora(4321)
        # a non-zero B so that every gradient is live
        for name in tr.adapter_names():
            if "lora_B" in name:
                d_out = mc.hidden
                tr.load_tensor(name.replace("base_model.model.", ""), (np.random.default_rng(7).standard_normal((d_out, 16)) * 0.01).astype(np.float32))
        rows = []
        for step in range(6):
            loss, gn, _, _ = tr.step(ids, labels)
            g = tr.export_adapter(grads=True)
            h = {k.split("self_attn.")[1]: hashlib.md5(v.tobytes()).hexdigest()[:8] for k, v in g.items()}
            rows.append((loss, gn, h))
        tr.close()
        for k in opts:
            L.set_option(k, {"fused_epilogues": 1, "attn_fwd_exp_fma_every": 0}[k])
        same = all(r == rows[0] for r in rows)
        print("STEP_REPEAT " + json.dumps({"opts": opts, "all_steps_identical": same, "steps": [[r[0], r[1], r[2]] for r in rows]}), flush=True)


if __name__ == "__main__":
    main()
