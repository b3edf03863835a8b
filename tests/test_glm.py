"""GLM-4 (GlmForCausalLM, Glm4ForCausalLM) without a GPU: the oracle of tests/glm_oracle.py (partial interleaved rotary, q/k/v
biases, fused gate_up_proj, Glm4's post-sublayer norms) against the installed GlmForCausalLM and Glm4ForCausalLM, the config loader, the rotary frequencies, the dtx_model_ext value checks and
the device-memory plan."""
import ctypes as C
import dataclasses
import json

import numpy as np
import pytest
import torch

from oracle import llama_lora as O
from tests import glm_oracle as FO

# hidden 256 with 2 q heads x 128 over one KV head
GLM_TINY = dict(vocab=512, hidden=256, n_layers=2, n_heads=2, n_kv_heads=1, ffn=384, rope_theta=10000.0, rms_eps=1.5625e-07,
                qkv_bias=True, rope_glm=True)
# GLM-4-9B's 16:1 grouped-query ratio, with an attention width (16 x 128) other than the hidden size
GLM_GQA16 = dict(GLM_TINY, n_heads=16, n_kv_heads=1)
GLM4_TINY = dict(GLM_TINY, post_norms=True)


def _hf_model(cfg: FO.FamilyConfig, weights):
    from transformers import Glm4Config, Glm4ForCausalLM, GlmConfig, GlmForCausalLM
    Cfg, Model = (Glm4Config, Glm4ForCausalLM) if cfg.post_norms else (GlmConfig, GlmForCausalLM)
    m = Model(Cfg(vocab_size=cfg.vocab, hidden_size=cfg.hidden, intermediate_size=cfg.ffn,
                                 num_hidden_layers=cfg.n_layers, num_attention_heads=cfg.n_heads, num_key_value_heads=cfg.n_kv_heads,
                                 head_dim=cfg.head_dim, rms_norm_eps=cfg.rms_eps, tie_word_embeddings=False, attention_bias=True,
                                 pad_token_id=0, max_position_embeddings=8192, attn_implementation="eager",
                                 rope_parameters={"rope_theta": cfg.rope_theta, "rope_type": "default", "partial_rotary_factor": 0.5}))
    m = m.float()
    missing, unexpected = m.load_state_dict(FO.to_hf(weights), strict=False)
    assert not [k for k in missing if "rotary" not in k], missing
    assert not unexpected, unexpected
    return m.eval()


CASES = {
    "glm_qv": (GLM_TINY, ("q_proj", "v_proj")),
    "glm_qkv": (GLM_TINY, ("q_proj", "k_proj", "v_proj")),
    "glm_gqa16_qkv": (GLM_GQA16, ("q_proj", "k_proj", "v_proj")),
    "glm4_qv": (GLM4_TINY, ("q_proj", "v_proj")),
    "glm4_qkv": (GLM4_TINY, ("q_proj", "k_proj", "v_proj")),
}


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_hf_logits_loss_and_lora_grads(case):
    dims, targets = CASES[case]
    cfg = FO.FamilyConfig(**dims, lora_r=8, lora_alpha=16.0, lora_target=targets)
    w = FO.init_base_weights(cfg, seed=7)
    lora = FO.init_lora(cfg, seed=8)
    g = torch.Generator().manual_seed(9)
    for k in lora:
        if "lora_B" in k:
            lora[k] = torch.randn(lora[k].shape, generator=g) * 0.02
    ids, labels = O.synthetic_batch(step=0, rank=0, batch=2, seq_len=96, vocab=cfg.vocab)
    t_ids, t_lab = torch.from_numpy(ids).long(), torch.from_numpy(labels).long()

    m = _hf_model(cfg, w)
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
        # the rotary convention matters: Llama's half-split rotary over the whole head gives other logits
        other = FO.forward_logits(dataclasses.replace(cfg, rope_glm=False), w, tr.lora, t_ids)
        assert float((other - logits).abs().max()) > 1e-3
        if cfg.post_norms:  # the norm weights matter: unit weights give other logits
            unit = {k: (torch.ones_like(v) if k.endswith(("post_self_attn_layernorm.weight", "post_mlp_layernorm.weight")) else v)
                    for k, v in w.items()}
            assert float((FO.forward_logits(cfg, unit, tr.lora, t_ids) - logits).abs().max()) > 1e-3
    assert torch.allclose(logits, out.logits.float(), atol=2e-5, rtol=1e-4), float((logits - out.logits).abs().max())
    loss, grads = tr.loss_and_grads(ids, labels)
    assert abs(loss - float(out.loss)) < 1e-5
    for key, mod in wrapped.items():
        assert torch.allclose(grads[key + "lora_A.weight"], mod.lora_A.grad, atol=1e-6, rtol=1e-4)
        assert torch.allclose(grads[key + "lora_B.weight"], mod.lora_B.grad, atol=1e-6, rtol=1e-4)


@pytest.mark.parametrize("case", ["glm_qv", "glm_gqa16_qkv", "glm4_qv"])
def test_oracle_full_sft_grads_match_hf(case):
    dims, _ = CASES[case]
    cfg = FO.FamilyConfig(**dims, full_finetune=True)
    w = FO.init_base_weights(cfg, seed=11)
    ids, labels = O.synthetic_batch(step=1, rank=0, batch=2, seq_len=64, vocab=cfg.vocab)
    m = _hf_model(cfg, w)
    out = m(input_ids=torch.from_numpy(ids).long(), labels=torch.from_numpy(labels).long())
    out.loss.backward()
    tr = FO.FamilyTrainer(cfg, w, {})
    loss, grads = tr.loss_and_grads(ids, labels)
    assert abs(loss - float(out.loss)) < 1e-5
    grads = FO.fuse_gate_up(grads)
    hf = dict(m.named_parameters())
    assert set(grads) == set(hf)
    for k, gr in grads.items():
        assert torch.allclose(gr, hf[k].grad, atol=1e-6, rtol=1e-3), (k, float((gr - hf[k].grad).abs().max()))
    assert grads["model.layers.1.mlp.gate_up_proj.weight"].shape == (2 * cfg.ffn, cfg.hidden)
    for name in ("q_proj", "k_proj", "v_proj"):
        assert float(grads[f"model.layers.1.self_attn.{name}.bias"].abs().max()) > 0
        assert FO.no_decay(cfg, f"model.layers.1.self_attn.{name}.bias")
    if cfg.post_norms:
        for name in ("post_self_attn_layernorm", "post_mlp_layernorm"):
            assert float(grads[f"model.layers.1.{name}.weight"].abs().max()) > 0
            assert FO.no_decay(cfg, f"model.layers.1.{name}.weight")


def test_fuse_gate_up_puts_gate_rows_first():
    cfg = FO.FamilyConfig(**GLM_TINY)
    w = FO.init_base_weights(cfg, seed=3)
    fused = FO.fuse_gate_up(w)["model.layers.0.mlp.gate_up_proj.weight"]
    gate, up = fused.chunk(2, dim=0)  # GlmMLP.forward
    assert torch.equal(gate, w["model.layers.0.mlp.gate_proj.weight"]) and torch.equal(up, w["model.layers.0.mlp.up_proj.weight"])


# ---------------------------------------------------------------------------------------------------------------------------
# config loader
# ---------------------------------------------------------------------------------------------------------------------------
GLM4_9B_CHAT_HF = {"architectures": ["GlmForCausalLM"], "attention_bias": True, "attention_dropout": 0.0,
                   "eos_token_id": [151329, 151336, 151338], "head_dim": 128, "hidden_act": "silu", "hidden_size": 4096,
                   "initializer_range": 0.02, "intermediate_size": 13696, "max_position_embeddings": 131072, "model_type": "glm",
                   "num_attention_heads": 32, "num_hidden_layers": 40, "num_key_value_heads": 2, "pad_token_id": 151329,
                   "partial_rotary_factor": 0.5, "rms_norm_eps": 1.5625e-07, "rope_theta": 10000.0, "tie_word_embeddings": False,
                   "torch_dtype": "bfloat16", "use_cache": True, "vocab_size": 151552}
# transformers 5 writes the rotary settings into rope_parameters
GLM4_9B_HF_V5 = {k: v for k, v in GLM4_9B_CHAT_HF.items() if k not in ("partial_rotary_factor", "rope_theta")}
GLM4_9B_HF_V5["rope_parameters"] = {"rope_theta": 10000.0, "rope_type": "default", "partial_rotary_factor": 0.5}
GLM4_9B_0414 = {"architectures": ["Glm4ForCausalLM"], "attention_bias": True, "attention_dropout": 0.0,
                "eos_token_id": [151329, 151336, 151338], "head_dim": 128, "hidden_act": "silu", "hidden_size": 4096,
                "initializer_range": 0.02, "intermediate_size": 13696, "max_position_embeddings": 32768, "model_type": "glm4",
                "num_attention_heads": 32, "num_hidden_layers": 40, "num_key_value_heads": 2, "pad_token_id": 151329,
                "partial_rotary_factor": 0.5, "rms_norm_eps": 1e-05, "rope_theta": 10000.0, "tie_word_embeddings": False,
                "torch_dtype": "bfloat16", "use_cache": True, "vocab_size": 151552}
GLM4_32B_0414 = dict(GLM4_9B_0414, hidden_size=6144, num_attention_heads=48, num_hidden_layers=61, intermediate_size=23040)


def _cfg_dir(tmp_path, cfg):
    d = tmp_path / "m"
    d.mkdir(exist_ok=True)
    (d / "config.json").write_text(json.dumps(cfg))
    return str(d)


def _accepted(mc, full=False):
    """what dtx_trainer_create_ext checks before any device work: the memory plan runs the same checks"""
    from datatunerx_b200 import lib as L
    tc = L.TrainConfig(micro_batch=1, seq_len=2048, total_steps=1, lora_r=16, lora_dropout=0.0, full_finetune=full)
    return L.plan_device_bytes(mc, tc, 8 if full else 1, "layer") > 0


@pytest.mark.parametrize("cfg", [GLM4_9B_CHAT_HF, GLM4_9B_HF_V5], ids=["chat_hf", "rope_parameters"])
def test_loader_accepts_glm4_9b(lib, tmp_path, cfg):
    from datatunerx_b200.tuning import model_io
    d = _cfg_dir(tmp_path, cfg)
    mc = model_io.load_model_config(d)
    assert (mc.hidden, mc.n_layers, mc.n_heads, mc.n_kv_heads, mc.head_dim, mc.ffn, mc.vocab) == (4096, 40, 32, 2, 128, 13696, 151552)
    assert mc.rope_glm and mc.qkv_bias and not mc.qk_norm and mc.rope_scaling is None and mc.rope_theta == 10000.0
    ext = mc.ext_to_c()
    assert ext.rope_glm == 1 and ext.qkv_bias == 1 and ext.qk_norm == 0 and ext.rope_type == 0
    assert _accepted(mc)
    assert _accepted(model_io.load_model_config(d, full_finetune=True), full=True)


@pytest.mark.parametrize("cfg,dims", [(GLM4_9B_0414, (4096, 40, 32, 2, 13696)), (GLM4_32B_0414, (6144, 61, 48, 2, 23040))],
                         ids=["9b_0414", "32b_0414"])
def test_loader_accepts_glm4_0414(lib, tmp_path, cfg, dims):
    from datatunerx_b200.tuning import model_io
    d = _cfg_dir(tmp_path, cfg)
    mc = model_io.load_model_config(d)
    assert (mc.hidden, mc.n_layers, mc.n_heads, mc.n_kv_heads, mc.ffn) == dims
    assert mc.rope_glm and mc.post_norms and mc.qkv_bias and not mc.qk_norm
    assert mc.ext_to_c().post_norms == 1 and mc.ext_to_c().rope_glm == 1
    assert _accepted(mc)
    assert _accepted(model_io.load_model_config(d, full_finetune=True), full=True)


def test_glm_attention_bias_defaults_to_true(tmp_path):
    """GlmConfig's attention_bias default is True: a config.json that leaves it out still has the biases."""
    from datatunerx_b200.tuning import model_io
    cfg = {k: v for k, v in GLM4_9B_CHAT_HF.items() if k != "attention_bias"}
    assert model_io.load_model_config(_cfg_dir(tmp_path, cfg)).qkv_bias
    assert not model_io.load_model_config(_cfg_dir(tmp_path, dict(GLM4_9B_CHAT_HF, attention_bias=False))).qkv_bias


@pytest.mark.parametrize("case", ["partial_0_25", "partial_1", "gelu", "rope_linear", "glm4_partial_0_25", "moe", "tied_full"])
def test_loader_refusals(tmp_path, case):
    from datatunerx_b200.tuning import model_io
    full = False
    if case == "partial_0_25":
        cfg = dict(GLM4_9B_CHAT_HF, partial_rotary_factor=0.25)
    elif case == "partial_1":
        cfg = dict(GLM4_9B_HF_V5, rope_parameters={"rope_theta": 10000.0, "rope_type": "default", "partial_rotary_factor": 1.0})
    elif case == "gelu":
        cfg = dict(GLM4_9B_CHAT_HF, hidden_act="gelu")
    elif case == "rope_linear":
        cfg = dict(GLM4_9B_CHAT_HF, rope_scaling={"rope_type": "linear", "factor": 2.0})
    elif case == "glm4_partial_0_25":
        cfg = dict(GLM4_9B_0414, partial_rotary_factor=0.25)
    elif case == "moe":
        cfg = dict(GLM4_9B_CHAT_HF, architectures=["Glm4MoeForCausalLM"], model_type="glm4_moe", n_routed_experts=128)
    else:
        cfg, full = dict(GLM4_9B_CHAT_HF, tie_word_embeddings=True), True
    with pytest.raises(ValueError):
        model_io.load_model_config(_cfg_dir(tmp_path, cfg), full_finetune=full)


def test_tied_glm_is_accepted_for_lora(tmp_path):
    from datatunerx_b200.tuning import model_io
    mc = model_io.load_model_config(_cfg_dir(tmp_path, dict(GLM4_9B_CHAT_HF, tie_word_embeddings=True)))
    assert mc.rope_glm


# ---------------------------------------------------------------------------------------------------------------------------
# rotary frequencies, ABI and memory plan
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("theta", [10000.0, 500000.0])
def test_rope_inv_freq_is_bitwise_glm(lib, theta):
    from transformers import GlmConfig
    from transformers.models.glm.modeling_glm import GlmRotaryEmbedding
    from datatunerx_b200 import lib as L
    hf = GlmRotaryEmbedding(GlmConfig(vocab_size=64, hidden_size=4096, num_attention_heads=32, head_dim=128, pad_token_id=0,
                                      rope_parameters={"rope_theta": theta, "rope_type": "default", "partial_rotary_factor": 0.5}))
    ref = hf.inv_freq.numpy()
    got = L.rope_inv_freq(L.ModelConfig(vocab=256, hidden=4096, n_layers=1, n_heads=32, ffn=256, rope_theta=theta, rope_glm=True))
    assert got.shape == (32,) and np.array_equal(got, ref), (got[:4], ref[:4])
    assert np.array_equal(got, FO.inv_freq(FO.FamilyConfig(rope_theta=theta, rope_glm=True)).numpy())


def test_bad_rope_glm_is_refused_without_a_device(lib):
    from datatunerx_b200 import lib as L
    mc = L.ModelConfig(vocab=2048, hidden=256, n_layers=1, n_heads=2, n_kv_heads=1, ffn=768).to_c()
    tc = L.TrainConfig(micro_batch=1, seq_len=128, total_steps=1, lora_dropout=0.0).to_c()
    out = (C.c_float * 64)()
    bad = [(L.ModelExt(rope_glm=2), "rope_glm"), (L.ModelExt(rope_glm=-1), "rope_glm"), (L.ModelExt(rope_glm=1, qk_norm=1), "rope_glm"),
           (L.ModelExt(rope_glm=1, rope_type=1, rope_factor=2.0), "rope_glm"), (L.ModelExt(post_norms=2), "post_norms"),
           (L.ModelExt(post_norms=-1), "post_norms")]
    for ext, word in bad:
        h, n = C.c_void_p(), C.c_int64()
        assert lib.dtx_trainer_create_ext(C.byref(mc), C.byref(ext), C.byref(tc), 0, 0, 1, None, C.byref(h)) == -1
        assert not h.value
        assert lib.dtx_plan_device_bytes_ext(C.byref(mc), C.byref(ext), C.byref(tc), 1, 1, C.byref(n)) == -1
        assert lib.dtx_rope_inv_freq(C.byref(mc), C.byref(ext), out) == -1
        assert word in L.load().dtx_last_global_error().decode()
    windowed = L.ModelConfig(vocab=2048, hidden=256, n_layers=1, n_heads=2, n_kv_heads=1, ffn=768, sliding_window=64).to_c()
    h, n = C.c_void_p(), C.c_int64()
    ext = L.ModelExt(rope_glm=1)
    assert lib.dtx_trainer_create_ext(C.byref(windowed), C.byref(ext), C.byref(tc), 0, 0, 1, None, C.byref(h)) == -1
    assert lib.dtx_plan_device_bytes_ext(C.byref(windowed), C.byref(ext), C.byref(tc), 1, 1, C.byref(n)) == -1
    assert "sliding window" in L.load().dtx_last_global_error().decode()


@pytest.mark.parametrize("full,world", [(False, 1), (True, 1), (True, 8)])
def test_rope_glm_halves_exactly_the_rotary_tables(lib, full, world):
    """GLM's tables hold head_dim / 4 frequencies instead of head_dim / 2: two [seq_len] x 32 float2 fewer, nothing else moves."""
    from datatunerx_b200 import lib as L
    mc = L.ModelConfig(vocab=2048, hidden=256, n_layers=3, n_heads=16, n_kv_heads=1, ffn=768, qkv_bias=True)
    tc = L.TrainConfig(micro_batch=2, seq_len=256, total_steps=4, lora_r=16, lora_dropout=0.0, full_finetune=full,
                       lora_target=("q_proj", "k_proj", "v_proj"))
    for layout in ("keep", "layer"):
        plain = L.plan_device_bytes(mc, tc, world, layout)
        glm = L.plan_device_bytes(dataclasses.replace(mc, rope_glm=True), tc, world, layout)
        assert plain - glm == 2 * tc.seq_len * (mc.head_dim // 4) * 8


@pytest.mark.parametrize("full,world", [(False, 1), (True, 1), (True, 8)])
def test_post_norms_add_exactly_the_saved_outputs_and_weight_bytes(lib, full, world):
    """o_pre and down_pre [M, d] bf16 plus two rstd [M] fp32 per saved set, and 2 x [d] norm weights per layer."""
    from datatunerx_b200 import lib as L
    mc = L.ModelConfig(vocab=2048, hidden=256, n_layers=3, n_heads=2, n_kv_heads=1, ffn=768, qkv_bias=True, rope_glm=True)
    tc = L.TrainConfig(micro_batch=2, seq_len=256, total_steps=4, lora_r=16, lora_dropout=0.0, full_finetune=full,
                       lora_target=("q_proj", "k_proj", "v_proj"))
    mp = dataclasses.replace(mc, post_norms=True)
    d, F, V, L_ = mc.hidden, mc.ffn, mc.vocab, mc.n_layers
    dq, dkv = mc.n_heads * 128, mc.n_kv_heads * 128
    W, M = dq + 2 * dkv, tc.micro_batch * tc.seq_len
    for layout, saved_sets in (("keep", L_), ("layer", 1)):
        plain, normed = L.plan_device_bytes(mc, tc, world, layout), L.plan_device_bytes(mp, tc, world, layout)
        saved = saved_sets * (2 * M * d * 2 + 2 * M * 4)
        if not full:
            assert normed - plain == saved + L_ * 2 * d * 2
        else:  # bf16 weight + gradient, fp32 master + two moments for this rank's shard of every padded layer block
            unit = world * 128
            pad = lambda n: (n + unit - 1) // unit * unit  # noqa: E731
            used = W * d + d * dq + 2 * F * d + d * F + 2 * d + W
            total = lambda layer: L_ * pad(layer) + pad(2 * V * d + d)  # noqa: E731
            t0, t1 = total(used), total(used + 2 * d)
            assert normed - plain == saved + (t1 - t0) * 2 * 2 + (t1 - t0) // world * 4 * 3


def test_weight_names_give_biases_their_output_widths(lib):
    """q_proj.bias is [n_heads * head_dim], also when that differs from the hidden size (16 x 128 heads over hidden 256)."""
    from datatunerx_b200 import lib as L
    mc = L.ModelConfig(vocab=2048, hidden=256, n_layers=1, n_heads=16, n_kv_heads=1, ffn=768, qkv_bias=True, rope_glm=True,
                       post_norms=True)
    tr = L.Trainer.__new__(L.Trainer)  # weight_names is host arithmetic: no device handle needed
    tr.model, tr.train = mc, L.TrainConfig(micro_batch=1, seq_len=128, total_steps=1, full_finetune=True)
    names = dict(tr.weight_names())
    hf = FO.to_hf(FO.init_base_weights(FO.FamilyConfig(vocab=2048, hidden=256, n_layers=1, n_heads=16, n_kv_heads=1, ffn=768,
                                                         qkv_bias=True, rope_glm=True, post_norms=True), seed=1))
    assert names == {k: tuple(v.shape) for k, v in hf.items()}
    assert names["model.layers.0.self_attn.q_proj.bias"] == (2048,)


def test_weight_names_use_the_fused_gate_up_for_glm(lib):
    from datatunerx_b200 import lib as L
    mc = L.ModelConfig(vocab=2048, hidden=256, n_layers=2, n_heads=2, n_kv_heads=1, ffn=768, qkv_bias=True, rope_glm=True)
    tc = L.TrainConfig(micro_batch=1, seq_len=128, total_steps=1, full_finetune=True)
    tr = L.Trainer.__new__(L.Trainer)  # weight_names is host arithmetic: no device handle needed
    tr.model, tr.train = mc, tc
    names = dict(tr.weight_names())
    assert names["model.layers.1.mlp.gate_up_proj.weight"] == (2 * 768, 256)
    assert not any("gate_proj" in k or ".up_proj" in k for k in names)
    hf = set(FO.to_hf(FO.init_base_weights(FO.FamilyConfig(vocab=2048, hidden=256, n_layers=2, n_heads=2, n_kv_heads=1, ffn=768,
                                                              qkv_bias=True, rope_glm=True), seed=1)))
    assert set(names) == hf
