"""Qwen3 and decoupled attention widths without a GPU: the oracle of tests/qwen3_oracle.py (q/k RMSNorm,
n_heads * head_dim != hidden) against the installed Qwen3ForCausalLM and MistralForCausalLM, the config loader, the
dtx_model_ext value checks and the device-memory plan of the q/k norm."""
import ctypes as C
import dataclasses
import json

import pytest
import torch

from oracle import llama_lora as O
from tests import qwen3_oracle as FO

# hidden 256 with 4 heads x 128: the attention is twice as wide as the residual stream
QWEN3_TINY = dict(vocab=512, hidden=256, n_layers=2, n_heads=4, n_kv_heads=2, ffn=384, rope_theta=1000000.0, rms_eps=1e-6,
                  qk_norm=True)
NEMO_TINY = dict(vocab=512, hidden=256, n_layers=2, n_heads=4, n_kv_heads=2, ffn=384, rope_theta=1000000.0, rms_eps=1e-5)


def _hf_model(cfg: FO.FamilyConfig, weights, qwen3: bool, tied: bool = False):
    common = dict(vocab_size=cfg.vocab, hidden_size=cfg.hidden, intermediate_size=cfg.ffn, num_hidden_layers=cfg.n_layers,
                  num_attention_heads=cfg.n_heads, num_key_value_heads=cfg.n_kv_heads or cfg.n_heads, head_dim=cfg.head_dim,
                  rms_norm_eps=cfg.rms_eps, tie_word_embeddings=tied, attn_implementation="eager",
                  rope_parameters={"rope_theta": cfg.rope_theta, "rope_type": "default"})
    if qwen3:
        from transformers import Qwen3Config, Qwen3ForCausalLM
        m = Qwen3ForCausalLM(Qwen3Config(**common, max_position_embeddings=40960, use_sliding_window=False, attention_bias=False))
    else:
        from transformers import MistralConfig, MistralForCausalLM
        m = MistralForCausalLM(MistralConfig(**common, max_position_embeddings=131072, sliding_window=None))
    m = m.float()
    sd = {k: v for k, v in weights.items() if not (tied and k == "lm_head.weight")}
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not [k for k in missing if "rotary" not in k and not (tied and k == "lm_head.weight")], missing
    assert not unexpected, unexpected
    return m.eval()


CASES = {
    "qwen3_qv": (QWEN3_TINY, True, ("q_proj", "v_proj"), False),
    "qwen3_qkv_tied": (QWEN3_TINY, True, ("q_proj", "k_proj", "v_proj"), True),
    "nemo_qkv": (NEMO_TINY, False, ("q_proj", "k_proj", "v_proj"), False),
}


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_hf_logits_loss_and_lora_grads(case):
    dims, qwen3, targets, tied = CASES[case]
    cfg = FO.FamilyConfig(**dims, lora_r=8, lora_alpha=16.0, lora_target=targets)
    w = FO.init_base_weights(cfg, seed=7, tied=tied)
    assert w["model.layers.0.self_attn.q_proj.weight"].shape == (512, 256)
    assert w["model.layers.0.self_attn.o_proj.weight"].shape == (256, 512)
    lora = FO.init_lora(cfg, seed=8)
    g = torch.Generator().manual_seed(9)
    for k in lora:
        if "lora_B" in k:
            lora[k] = torch.randn(lora[k].shape, generator=g) * 0.02
    ids, labels = O.synthetic_batch(step=0, rank=0, batch=2, seq_len=96, vocab=cfg.vocab)
    t_ids, t_lab = torch.from_numpy(ids).long(), torch.from_numpy(labels).long()

    m = _hf_model(cfg, w, qwen3, tied)
    for p in m.parameters():
        p.requires_grad_(False)
    wrapped = {}
    from tests.test_oracle_pin import _PeftLoRA
    for l, layer in enumerate(m.model.layers):
        for t in cfg.lora_target:
            key = f"model.layers.{l}.self_attn.{t}."
            mod = _PeftLoRA(getattr(layer.self_attn, t), lora[key + "lora_A.weight"], lora[key + "lora_B.weight"], cfg.lora_alpha / cfg.lora_r)
            setattr(layer.self_attn, t, mod)
            wrapped[key] = mod
    out = m(input_ids=t_ids, labels=t_lab)
    out.loss.backward()

    tr = FO.FamilyTrainer(cfg, w, lora)
    with torch.no_grad():
        logits = FO.forward_logits(cfg, w, tr.lora, t_ids)
        if qwen3:  # the norm weights matter: the same model with unit norm weights gives other logits
            unit = {k: (torch.ones_like(v) if k.endswith("_norm.weight") else v) for k, v in w.items()}
            assert float((FO.forward_logits(cfg, unit, tr.lora, t_ids) - logits).abs().max()) > 1e-3
    assert torch.allclose(logits, out.logits.float(), atol=2e-5, rtol=1e-4), float((logits - out.logits).abs().max())
    loss, grads = tr.loss_and_grads(ids, labels)
    assert abs(loss - float(out.loss)) < 1e-5
    for key, mod in wrapped.items():
        assert torch.allclose(grads[key + "lora_A.weight"], mod.lora_A.grad, atol=1e-6, rtol=1e-4)
        assert torch.allclose(grads[key + "lora_B.weight"], mod.lora_B.grad, atol=1e-6, rtol=1e-4)


@pytest.mark.parametrize("case", ["qwen3_qv", "nemo_qkv"])
def test_oracle_full_sft_grads_match_hf(case):
    dims, qwen3, _, _ = CASES[case]
    cfg = FO.FamilyConfig(**dims, full_finetune=True)
    w = FO.init_base_weights(cfg, seed=11)
    ids, labels = O.synthetic_batch(step=1, rank=0, batch=2, seq_len=64, vocab=cfg.vocab)
    m = _hf_model(cfg, w, qwen3)
    out = m(input_ids=torch.from_numpy(ids).long(), labels=torch.from_numpy(labels).long())
    out.loss.backward()
    tr = FO.FamilyTrainer(cfg, w, {})
    loss, grads = tr.loss_and_grads(ids, labels)
    assert abs(loss - float(out.loss)) < 1e-5
    hf = dict(m.named_parameters())
    assert set(grads) == set(hf)
    for k, gr in grads.items():
        assert torch.allclose(gr, hf[k].grad, atol=1e-6, rtol=1e-3), (k, float((gr - hf[k].grad).abs().max()))
    if qwen3:
        for name in ("q_norm", "k_norm"):
            assert float(grads[f"model.layers.1.self_attn.{name}.weight"].abs().max()) > 0
            assert FO.no_decay(cfg, f"model.layers.1.self_attn.{name}.weight")


# ---------------------------------------------------------------------------------------------------------------------------
# config loader
# ---------------------------------------------------------------------------------------------------------------------------
QWEN3_8B = {"architectures": ["Qwen3ForCausalLM"], "attention_bias": False, "attention_dropout": 0.0, "bos_token_id": 151643,
            "eos_token_id": 151645, "head_dim": 128, "hidden_act": "silu", "hidden_size": 4096, "initializer_range": 0.02,
            "intermediate_size": 12288, "max_position_embeddings": 40960, "max_window_layers": 36, "model_type": "qwen3",
            "num_attention_heads": 32, "num_hidden_layers": 36, "num_key_value_heads": 8, "rms_norm_eps": 1e-06,
            "rope_scaling": None, "rope_theta": 1000000, "sliding_window": None, "tie_word_embeddings": False,
            "torch_dtype": "bfloat16", "use_cache": True, "use_sliding_window": False, "vocab_size": 151936}
QWEN3_4B = dict(QWEN3_8B, hidden_size=2560, intermediate_size=9728, tie_word_embeddings=True)
MISTRAL_NEMO = {"architectures": ["MistralForCausalLM"], "head_dim": 128, "hidden_size": 5120, "intermediate_size": 14336,
                "max_position_embeddings": 1024000, "model_type": "mistral", "num_attention_heads": 32, "num_hidden_layers": 40,
                "num_key_value_heads": 8, "rms_norm_eps": 1e-05, "rope_theta": 1000000.0, "sliding_window": None,
                "tie_word_embeddings": False, "vocab_size": 131072}


def _cfg_dir(tmp_path, cfg):
    d = tmp_path / "m"
    d.mkdir(exist_ok=True)
    (d / "config.json").write_text(json.dumps(cfg))
    return str(d)


def _accepted(lib, mc, full=False):
    """what dtx_trainer_create_ext checks before any device work: the memory plan runs the same checks"""
    from datatunerx_b200 import lib as L
    tc = L.TrainConfig(micro_batch=1, seq_len=2048, total_steps=1, lora_r=16, lora_dropout=0.0, full_finetune=full)
    return L.plan_device_bytes(mc, tc, 8 if full else 1, "layer") > 0


@pytest.mark.parametrize("name,cfg,dq,qk_norm,tied", [
    ("qwen3_8b", QWEN3_8B, 4096, True, False),
    ("qwen3_4b_tied", QWEN3_4B, 4096, True, True),
    ("mistral_nemo", MISTRAL_NEMO, 4096, False, False),
])
def test_loader_accepts(lib, tmp_path, name, cfg, dq, qk_norm, tied):
    from datatunerx_b200.tuning import model_io
    d = _cfg_dir(tmp_path, cfg)
    mc = model_io.load_model_config(d)
    assert mc.n_heads * mc.head_dim == dq and mc.qk_norm == qk_norm and not mc.qkv_bias and mc.sliding_window == 0
    assert mc.rope_theta == 1000000 and mc.rope_scaling is None and mc.ext_to_c().qk_norm == int(qk_norm)
    assert _accepted(lib, mc)
    if not tied:
        assert _accepted(lib, model_io.load_model_config(d, full_finetune=True), full=True)


@pytest.mark.parametrize("case", ["attention_bias", "sliding_window", "tied_full", "moe"])
def test_loader_refusals(tmp_path, case):
    from datatunerx_b200.tuning import model_io
    full = False
    if case == "attention_bias":
        cfg = dict(QWEN3_8B, attention_bias=True)
    elif case == "sliding_window":
        cfg = dict(QWEN3_8B, sliding_window=4096, use_sliding_window=True)
    elif case == "tied_full":
        cfg, full = QWEN3_4B, True
    else:
        cfg = dict(QWEN3_8B, architectures=["Qwen3MoeForCausalLM"], num_experts=128)
    with pytest.raises(ValueError):
        model_io.load_model_config(_cfg_dir(tmp_path, cfg), full_finetune=full)


# ---------------------------------------------------------------------------------------------------------------------------
# ABI and memory plan
# ---------------------------------------------------------------------------------------------------------------------------
def test_bad_qk_norm_is_refused_without_a_device(lib):
    from datatunerx_b200 import lib as L
    mc = L.ModelConfig(vocab=2048, hidden=256, n_layers=1, n_heads=4, ffn=768).to_c()
    tc = L.TrainConfig(micro_batch=1, seq_len=128, total_steps=1, lora_dropout=0.0).to_c()
    out = (C.c_float * 64)()
    for v in (2, -1):
        ext = L.ModelExt(qk_norm=v)
        h, n = C.c_void_p(), C.c_int64()
        assert lib.dtx_trainer_create_ext(C.byref(mc), C.byref(ext), C.byref(tc), 0, 0, 1, None, C.byref(h)) == -1
        assert not h.value
        assert lib.dtx_plan_device_bytes_ext(C.byref(mc), C.byref(ext), C.byref(tc), 1, 1, C.byref(n)) == -1
        assert lib.dtx_rope_inv_freq(C.byref(mc), C.byref(ext), out) == -1
        assert "qk_norm" in L.load().dtx_last_global_error().decode()


def _tiny3(full):
    from datatunerx_b200 import lib as L
    mc = L.ModelConfig(vocab=2048, hidden=256, n_layers=3, n_heads=4, n_kv_heads=2, ffn=768, rms_eps=1e-6, rope_theta=1e6)
    tc = L.TrainConfig(micro_batch=2, seq_len=256, total_steps=4, lora_r=16, lora_dropout=0.0, full_finetune=full,
                       lora_target=("q_proj", "k_proj", "v_proj"))
    return mc, tc


@pytest.mark.parametrize("full,world", [(False, 1), (True, 1), (True, 8)])
def test_qk_norm_adds_exactly_the_pre_norm_and_weight_bytes(lib, full, world):
    from datatunerx_b200 import lib as L
    mc, tc = _tiny3(full)
    mq = dataclasses.replace(mc, qk_norm=True)
    d, F, V, L_, D = mc.hidden, mc.ffn, mc.vocab, mc.n_layers, mc.head_dim
    dq, dkv = mc.n_heads * D, mc.n_kv_heads * D
    W, M = dq + 2 * dkv, tc.micro_batch * tc.seq_len
    for layout, saved_sets in (("keep", L_), ("layer", 1)):
        plain, normed = L.plan_device_bytes(mc, tc, world, layout), L.plan_device_bytes(mq, tc, world, layout)
        pre = saved_sets * M * (dq + dkv) * 2  # the pre-norm q|k of every saved set, bf16
        if not full:
            assert normed - plain == pre + L_ * 2 * D * 2
        else:  # bf16 weight + gradient, fp32 master + two moments for this rank's shard of every padded layer block
            unit = world * 128
            pad = lambda n: (n + unit - 1) // unit * unit  # noqa: E731
            used = W * d + d * dq + 2 * F * d + d * F + 2 * d
            total = lambda layer: L_ * pad(layer) + pad(2 * V * d + d)  # noqa: E731
            t0, t1 = total(used), total(used + 2 * D)
            assert normed - plain == pre + (t1 - t0) * 2 * 2 + (t1 - t0) // world * 4 * 3

