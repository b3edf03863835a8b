"""Llama-3.x and Qwen2 checkpoints without a GPU: the library's rotary inverse frequencies against transformers, the CPU
oracle of the two families against the installed HF models, the config loader, the dtx_model_ext mirror and the device-memory
plan of the bias vectors."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest
import torch

from oracle import llama_lora as O
from tests import family_oracle as FO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

LLAMA31_8B = {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
              "original_max_position_embeddings": 8192}
LLAMA32_3B = {"rope_type": "llama3", "factor": 32.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
              "original_max_position_embeddings": 8192}


def _hf_inv_freq(kind, theta, params, hidden=4096, heads=32):
    from transformers import LlamaConfig
    from transformers.modeling_rope_utils import ROPE_INIT_FUNCTIONS
    cfg = LlamaConfig(hidden_size=hidden, num_attention_heads=heads, max_position_embeddings=131072,
                      rope_parameters={"rope_theta": theta, **params, "rope_type": kind})
    inv, scaling = ROPE_INIT_FUNCTIONS[kind](cfg, "cpu")
    assert scaling == 1.0  # cos / sin are not rescaled for these types
    return inv.numpy()


@pytest.mark.parametrize("kind,theta,params", [
    ("llama3", 500000.0, LLAMA31_8B),
    ("llama3", 500000.0, LLAMA32_3B),
    ("linear", 10000.0, {"factor": 4.0}),
    ("linear", 500000.0, {"factor": 2.0}),
])
def test_rope_inv_freq_is_bitwise_hf(lib, kind, theta, params):
    from datatunerx_b200 import lib as L
    mc = L.ModelConfig(vocab=128256, hidden=4096, n_layers=32, n_heads=32, n_kv_heads=8, ffn=14336, rope_theta=theta,
                       rope_scaling={"rope_type": kind, **params})
    got = L.rope_inv_freq(mc)
    ref = _hf_inv_freq(kind, theta, params)
    assert got.dtype == np.float32 and got.shape == (64,)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), np.nonzero(got != ref)
    assert np.array_equal(got, FO.inv_freq(FO.FamilyConfig(rope_theta=theta, rope_scaling={"rope_type": kind, **params})).numpy())


@pytest.mark.parametrize("theta", [10000.0, 500000.0, 1000000.0])
def test_default_inv_freq_is_the_powf_table(lib, theta):
    """The default type keeps the plain table bit for bit: 1 / powf(theta, 2i / D) in fp32, as before extensions existed."""
    from datatunerx_b200 import lib as L
    libm = C.CDLL("libm.so.6")
    libm.powf.restype, libm.powf.argtypes = C.c_float, [C.c_float, C.c_float]
    f32 = np.float32
    ref = np.array([f32(1.0) / f32(libm.powf(theta, f32(2 * i) / f32(128))) for i in range(64)], np.float32)
    for rs in (None, {"rope_type": "default"}):
        got = L.rope_inv_freq(L.ModelConfig(vocab=256, hidden=256, n_layers=1, n_heads=2, ffn=256, rope_theta=theta, rope_scaling=rs))
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------------
# the family oracle against the installed transformers
# ---------------------------------------------------------------------------------------------------------------------------
def _hf_family_model(cfg: FO.FamilyConfig, weights, qwen2: bool, tied: bool):
    common = dict(vocab_size=cfg.vocab, hidden_size=cfg.hidden, intermediate_size=cfg.ffn, num_hidden_layers=cfg.n_layers,
                  num_attention_heads=cfg.n_heads, num_key_value_heads=cfg.n_kv_heads or cfg.n_heads, rms_norm_eps=cfg.rms_eps,
                  tie_word_embeddings=tied, attn_implementation="eager")
    rope = {"rope_theta": cfg.rope_theta, "rope_type": "default", **(cfg.rope_scaling or {})}
    if qwen2:
        from transformers import Qwen2Config, Qwen2ForCausalLM
        m = Qwen2ForCausalLM(Qwen2Config(**common, max_position_embeddings=32768, rope_parameters=rope, use_sliding_window=False))
    else:
        from transformers import LlamaConfig, LlamaForCausalLM
        m = LlamaForCausalLM(LlamaConfig(**common, max_position_embeddings=131072, rope_parameters=rope))
    m = m.float()
    sd = {k: v for k, v in weights.items() if not (tied and k == "lm_head.weight")}
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not [k for k in missing if "rotary" not in k and not (tied and k == "lm_head.weight")], missing
    assert not unexpected, unexpected
    return m.eval()


FAMILIES = {
    "llama3_gqa": dict(cfg=dict(vocab=512, hidden=768, n_layers=2, n_heads=6, n_kv_heads=2, ffn=384, rope_theta=500000.0,
                                rope_scaling=dict(LLAMA31_8B, original_max_position_embeddings=64)),
                       qwen2=False, tied=False),
    "qwen2_bias_tied": dict(cfg=dict(vocab=512, hidden=768, n_layers=2, n_heads=6, n_kv_heads=2, ffn=384, rope_theta=1000000.0,
                                     rms_eps=1e-6, qkv_bias=True), qwen2=True, tied=True),
}


@pytest.mark.parametrize("family", list(FAMILIES))
def test_family_oracle_matches_hf_logits_loss_and_lora_grads(family):
    spec = FAMILIES[family]
    cfg = FO.FamilyConfig(**spec["cfg"], lora_r=8, lora_alpha=16.0, lora_target=("q_proj", "k_proj", "v_proj"))
    w = FO.init_base_weights(cfg, seed=7, tied=spec["tied"])
    lora = O.init_lora(cfg, seed=8)
    g = torch.Generator().manual_seed(9)
    for k in lora:
        if "lora_B" in k:
            lora[k] = torch.randn(lora[k].shape, generator=g) * 0.02
    ids, labels = O.synthetic_batch(step=0, rank=0, batch=2, seq_len=96, vocab=cfg.vocab)
    t_ids, t_lab = torch.from_numpy(ids).long(), torch.from_numpy(labels).long()

    m = _hf_family_model(cfg, w, spec["qwen2"], spec["tied"])
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
        plain = O.forward_logits(cfg, w, tr.lora, t_ids)
    assert torch.allclose(logits, out.logits.float(), atol=2e-5, rtol=1e-4), float((logits - out.logits).abs().max())
    assert float((plain - logits).abs().max()) > 1e-3, "the family's rotary table / biases must matter"
    loss, grads = tr.loss_and_grads(ids, labels)
    assert abs(loss - float(out.loss)) < 1e-5
    for key, mod in wrapped.items():
        assert torch.allclose(grads[key + "lora_A.weight"], mod.lora_A.grad, atol=1e-6, rtol=1e-4)
        assert torch.allclose(grads[key + "lora_B.weight"], mod.lora_B.grad, atol=1e-6, rtol=1e-4)


@pytest.mark.parametrize("family", list(FAMILIES))
def test_family_oracle_full_sft_grads_match_hf(family):
    spec = FAMILIES[family]
    cfg = FO.FamilyConfig(**spec["cfg"], full_finetune=True)
    w = FO.init_base_weights(cfg, seed=11)  # untied: full-parameter SFT of tied weights is refused
    ids, labels = O.synthetic_batch(step=1, rank=0, batch=2, seq_len=64, vocab=cfg.vocab)
    m = _hf_family_model(cfg, w, spec["qwen2"], tied=False)
    out = m(input_ids=torch.from_numpy(ids).long(), labels=torch.from_numpy(labels).long())
    out.loss.backward()
    tr = FO.FamilyTrainer(cfg, w, {})
    loss, grads = tr.loss_and_grads(ids, labels)
    assert abs(loss - float(out.loss)) < 1e-5
    hf = dict(m.named_parameters())
    assert set(grads) == set(hf)
    for k, gr in grads.items():
        assert torch.allclose(gr, hf[k].grad, atol=1e-6, rtol=1e-3), (k, float((gr - hf[k].grad).abs().max()))
    if cfg.qkv_bias:
        assert float(grads["model.layers.0.self_attn.q_proj.bias"].abs().max()) > 0


def test_family_oracle_bias_has_no_weight_decay():
    cfg = FO.FamilyConfig(**FAMILIES["qwen2_bias_tied"]["cfg"], full_finetune=True, weight_decay=0.1, lr=1e-2, total_steps=3)
    assert FO.no_decay(cfg, "model.layers.0.self_attn.k_proj.bias") and FO.no_decay(cfg, "model.norm.weight")
    assert not FO.no_decay(cfg, "model.layers.0.self_attn.k_proj.weight")
    w = FO.init_base_weights(cfg, seed=3)
    tr = FO.FamilyTrainer(cfg, w, {})
    name = "model.layers.1.self_attn.v_proj.bias"
    before = tr.lora[name].detach().clone()
    tr.lora[name].register_hook(lambda g: torch.zeros_like(g))  # zero gradient: any change would be weight decay
    tr.step([O.synthetic_batch(0, 0, 1, 64, cfg.vocab)])
    assert torch.equal(tr.lora[name].detach(), before)


# ---------------------------------------------------------------------------------------------------------------------------
# config loader
# ---------------------------------------------------------------------------------------------------------------------------
def _cfg_dir(tmp_path, **cfg):
    base = {"architectures": ["LlamaForCausalLM"], "vocab_size": 128256, "hidden_size": 4096, "num_hidden_layers": 32,
            "num_attention_heads": 32, "num_key_value_heads": 8, "intermediate_size": 14336, "rms_norm_eps": 1e-5,
            "rope_theta": 500000.0, "max_position_embeddings": 131072}
    base.update(cfg)
    d = tmp_path / "m"
    d.mkdir(exist_ok=True)
    (d / "config.json").write_text(json.dumps(base))
    return str(d)


@pytest.mark.parametrize("key", ["rope_type", "type"])
def test_loader_reads_llama31_rope_scaling(tmp_path, key):
    from datatunerx_b200.tuning import model_io
    rs = {key: "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0, "original_max_position_embeddings": 8192}
    mc = model_io.load_model_config(_cfg_dir(tmp_path, rope_scaling=rs))
    assert mc.rope_scaling == rs and not mc.qkv_bias and mc.rope_theta == 500000.0 and mc.n_kv_heads == 8
    ext = mc.ext_to_c()
    assert (ext.qkv_bias, ext.rope_type, ext.rope_factor, ext.rope_low_freq_factor, ext.rope_high_freq_factor,
            ext.rope_original_max_pos) == (0, 2, 8.0, 1.0, 4.0, 8192)


def test_loader_qwen25_drops_the_window_and_sets_bias(tmp_path):
    from datatunerx_b200.tuning import model_io
    d = _cfg_dir(tmp_path, architectures=["Qwen2ForCausalLM"], vocab_size=152064, hidden_size=3584, num_hidden_layers=28,
                 num_attention_heads=28, num_key_value_heads=4, intermediate_size=18944, rope_theta=1000000.0, rms_norm_eps=1e-6,
                 sliding_window=131072, use_sliding_window=False, max_window_layers=28, tie_word_embeddings=False, rope_scaling=None)
    mc = model_io.load_model_config(d)
    assert mc.qkv_bias and mc.sliding_window == 0 and mc.rope_scaling is None and mc.n_heads // mc.n_kv_heads == 7
    assert mc.ext_to_c().qkv_bias == 1 and mc.ext_to_c().rope_type == 0
    model_io.load_model_config(d, full_finetune=True)  # untied: full-parameter SFT allowed


@pytest.mark.parametrize("case", ["yarn", "dynamic", "longrope", "qwen2_window", "attention_bias", "mlp_bias", "qwen2_tied_full"])
def test_loader_refusals(tmp_path, case):
    from datatunerx_b200.tuning import model_io
    full = False
    if case in ("yarn", "dynamic", "longrope"):
        d = _cfg_dir(tmp_path, rope_scaling={"rope_type": case, "factor": 4.0, "original_max_position_embeddings": 32768})
    elif case == "qwen2_window":
        d = _cfg_dir(tmp_path, architectures=["Qwen2ForCausalLM"], sliding_window=4096, use_sliding_window=True)
    elif case in ("attention_bias", "mlp_bias"):
        d = _cfg_dir(tmp_path, **{case: True})
    else:
        d = _cfg_dir(tmp_path, architectures=["Qwen2ForCausalLM"], tie_word_embeddings=True)
        model_io.load_model_config(d)  # LoRA on a tied Qwen2 (Qwen2.5-3B): fine
        full = True
    with pytest.raises(ValueError):
        model_io.load_model_config(d, full_finetune=full)


# ---------------------------------------------------------------------------------------------------------------------------
# ABI
# ---------------------------------------------------------------------------------------------------------------------------
def test_model_ext_mirror_matches_the_header(lib):
    from datatunerx_b200 import lib as L
    src = open(os.path.join(ROOT, "include", "dtxtune.h")).read()
    body = re.search(r"typedef struct \{([^}]*)\} dtx_model_ext;", src).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in filter(None, (x.strip() for x in body.split(";"))):
        ctype, names = decl.split(None, 1)
        fields += [(n.strip(), ctype) for n in names.split(",")]
    ctypes_of = {"int32_t": C.c_int32, "float": C.c_float}
    assert [(n, ctypes_of[t]) for n, t in fields] == [(f[0], f[1]) for f in L.ModelExt._fields_]
    for name in ("DTX_ROPE_DEFAULT", "DTX_ROPE_LINEAR", "DTX_ROPE_LLAMA3"):
        value = int(re.search(r"#define " + name + r"\s+(\d+)", src).group(1))
        assert L.ROPE_TYPES[name[len("DTX_ROPE_"):].lower()] == value


def _recompute_plan_configs():
    from tests.test_recompute_plan import _tiny
    from datatunerx_b200 import lib as L
    out = []
    for kw, world in ((dict(lora_dropout=0.0), 1), (dict(lora_dropout=0.1), 1),
                      (dict(heads=4, kv_heads=2, lora_dropout=0.0, lora_target=("q_proj", "k_proj", "v_proj")), 1),
                      (dict(full_finetune=True), 1), (dict(full_finetune=True), 8), (dict(layers=1, lora_dropout=0.0), 1)):
        mc, tc = _tiny(**kw)
        out.append((mc, tc, world))
    out.append((L.ModelConfig.llama2_7b(), L.TrainConfig(micro_batch=4, seq_len=2048, total_steps=10, lora_r=16, lora_dropout=0.0), 1))
    out.append((L.ModelConfig.llama2_7b(), L.TrainConfig(micro_batch=8, seq_len=4096, total_steps=10, lora_r=16, lora_dropout=0.0), 1))
    out.append((L.ModelConfig(vocab=32000, hidden=5120, n_layers=40, n_heads=40, ffn=13824),
                L.TrainConfig(micro_batch=2, seq_len=2048, total_steps=10, full_finetune=True), 8))
    return out


def test_plan_ext_with_zero_ext_equals_plan(lib):
    from datatunerx_b200 import lib as L
    zero = L.ModelExt()
    for mc, tc, world in _recompute_plan_configs():
        for layout in (1, 2):
            a, b = C.c_int64(), C.c_int64()
            cm, ct = mc.to_c(), tc.to_c()
            assert lib.dtx_plan_device_bytes(C.byref(cm), C.byref(ct), world, layout, C.byref(a)) == 0
            assert lib.dtx_plan_device_bytes_ext(C.byref(cm), C.byref(zero), C.byref(ct), world, layout, C.byref(b)) == 0
            assert lib.dtx_plan_device_bytes_ext(C.byref(cm), None, C.byref(ct), world, layout, C.byref(b)) == 0
            assert a.value == b.value == L.plan_device_bytes(mc, tc, world, layout)


@pytest.mark.parametrize("full,world", [(False, 1), (True, 1), (True, 8)])
def test_bias_adds_exactly_the_bias_bytes(lib, full, world):
    import dataclasses
    from datatunerx_b200 import lib as L
    from tests.test_recompute_plan import _tiny
    mc, tc = _tiny(heads=6, kv_heads=2, full_finetune=full, lora_dropout=0.0)
    mb = dataclasses.replace(mc, qkv_bias=True)
    W = (mc.n_heads + 2 * mc.n_kv_heads) * mc.head_dim
    d, F, V, L_ = mc.hidden, mc.ffn, mc.vocab, mc.n_layers
    for layout in ("keep", "layer"):
        plain, biased = L.plan_device_bytes(mc, tc, world, layout), L.plan_device_bytes(mb, tc, world, layout)
        if not full:
            assert biased - plain == L_ * W * 2
        else:  # bf16 weight + gradient, fp32 master + two moments for this rank's shard of every padded layer block
            unit = world * 128
            pad = lambda n: (n + unit - 1) // unit * unit  # noqa: E731
            used = W * d + d * d + 2 * F * d + d * F + 2 * d
            total = lambda layer: L_ * pad(layer) + pad(2 * V * d + d)  # noqa: E731
            t0, t1 = total(used), total(used + W)
            assert biased - plain == (t1 - t0) * 2 * 2 + (t1 - t0) // world * 4 * 3


def test_bad_ext_values_are_refused_without_a_device(lib):
    from datatunerx_b200 import lib as L
    mc = L.ModelConfig(vocab=2048, hidden=256, n_layers=1, n_heads=2, ffn=768).to_c()
    tc = L.TrainConfig(micro_batch=1, seq_len=128, total_steps=1, lora_dropout=0.0).to_c()
    bad = [L.ModelExt(0, 3, 8.0, 1.0, 4.0, 8192), L.ModelExt(0, -1, 0, 0, 0, 0), L.ModelExt(0, 1, 0.0, 0, 0, 0),
           L.ModelExt(0, 1, -2.0, 0, 0, 0), L.ModelExt(0, 2, 0.0, 1.0, 4.0, 8192), L.ModelExt(0, 2, 8.0, 4.0, 4.0, 8192),
           L.ModelExt(0, 2, 8.0, 4.0, 1.0, 8192), L.ModelExt(0, 2, 8.0, 1.0, 4.0, 0), L.ModelExt(0, 2, 8.0, 1.0, 4.0, -5),
           L.ModelExt(2, 0, 0, 0, 0, 0)]
    out = (C.c_float * 64)()
    for ext in bad:
        h, n = C.c_void_p(), C.c_int64()
        assert lib.dtx_trainer_create_ext(C.byref(mc), C.byref(ext), C.byref(tc), 0, 0, 1, None, C.byref(h)) == -1
        assert not h.value
        assert lib.dtx_plan_device_bytes_ext(C.byref(mc), C.byref(ext), C.byref(tc), 1, 1, C.byref(n)) == -1
        assert lib.dtx_rope_inv_freq(C.byref(mc), C.byref(ext), out) == -1
    with pytest.raises(L.DtxError) as e:
        L.ModelConfig(vocab=256, hidden=256, n_layers=1, n_heads=2, ffn=256, rope_scaling={"rope_type": "yarn", "factor": 4.0}).ext_to_c()
    assert e.value.code == -1


def test_unextended_entry_points_still_refuse_what_they_refused(lib):
    """head_dim 64 and LoRA on o_proj stay refused on the extended entry points too."""
    from datatunerx_b200 import lib as L
    with pytest.raises(L.DtxError):
        L.plan_device_bytes(L.ModelConfig(vocab=256, hidden=256, n_layers=1, n_heads=4, head_dim=64, ffn=256, qkv_bias=True),
                            L.TrainConfig(micro_batch=1, seq_len=128, total_steps=1, lora_dropout=0.0))
