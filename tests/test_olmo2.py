"""OLMo-2 without a GPU: the oracle of tests/olmo2_oracle.py (full-width q/k RMSNorm, no pre-norms) against the installed
Olmo2ForCausalLM, the config loader and its refusals, the dtx_model_ext value checks, the weight names and the device-memory
plan of the OLMo-2 layer."""
import ctypes as C
import dataclasses
import json

import pytest
import torch

from oracle import llama_lora as O
from tests import olmo2_oracle as FO

# 2 x 128 heads over hidden 256; GQA with one k/v head
MHA_TINY = dict(vocab=512, hidden=256, n_layers=2, n_heads=2, n_kv_heads=2, ffn=384, rope_theta=500000.0, rms_eps=1e-6,
                qk_norm_full=True, no_pre_norms=True)
GQA_TINY = dict(MHA_TINY, n_kv_heads=1)


def _hf_model(cfg: FO.FamilyConfig, weights, tied: bool = False):
    from transformers import Olmo2Config, Olmo2ForCausalLM
    m = Olmo2ForCausalLM(Olmo2Config(vocab_size=cfg.vocab, hidden_size=cfg.hidden, intermediate_size=cfg.ffn,
                                     num_hidden_layers=cfg.n_layers, num_attention_heads=cfg.n_heads,
                                     num_key_value_heads=cfg.n_kv_heads or cfg.n_heads, rms_norm_eps=cfg.rms_eps,
                                     tie_word_embeddings=tied, attention_bias=False, max_position_embeddings=4096, pad_token_id=None,
                                     rope_parameters={"rope_theta": cfg.rope_theta, "rope_type": "default"},
                                     attn_implementation="eager")).float()
    sd = {k: v for k, v in weights.items() if not (tied and k == "lm_head.weight")}
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not [k for k in missing if "rotary" not in k and not (tied and k == "lm_head.weight")], missing
    assert not unexpected, unexpected
    return m.eval()


CASES = {
    "mha_qv": (MHA_TINY, ("q_proj", "v_proj")),
    "mha_qkv": (MHA_TINY, ("q_proj", "k_proj", "v_proj")),
    "gqa_qv": (GQA_TINY, ("q_proj", "v_proj")),
    "gqa_qkv": (GQA_TINY, ("q_proj", "k_proj", "v_proj")),
}


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_hf_logits_loss_and_lora_grads(case):
    dims, targets = CASES[case]
    cfg = FO.FamilyConfig(**dims, lora_r=8, lora_alpha=16.0, lora_target=targets)
    w = FO.init_base_weights(cfg, seed=7)
    dq, dkv = cfg.n_heads * 128, (cfg.n_kv_heads or cfg.n_heads) * 128
    assert w["model.layers.0.self_attn.q_norm.weight"].shape == (dq,) and w["model.layers.0.self_attn.k_norm.weight"].shape == (dkv,)
    assert "model.layers.0.input_layernorm.weight" not in w
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
        # every kind of norm weight matters: the same model with any one of them at 1 gives other logits
        for suffix in ("q_norm.weight", "k_norm.weight", "post_attention_layernorm.weight", "post_feedforward_layernorm.weight"):
            unit = {k: (torch.ones_like(v) if k.endswith(suffix) else v) for k, v in w.items()}
            assert float((FO.forward_logits(cfg, unit, tr.lora, t_ids) - logits).abs().max()) > 1e-3, suffix
    assert torch.allclose(logits, out.logits.float(), atol=2e-5, rtol=1e-4), float((logits - out.logits).abs().max())
    loss, grads = tr.loss_and_grads(ids, labels)
    assert abs(loss - float(out.loss)) < 1e-5
    for key, mod in wrapped.items():
        assert torch.allclose(grads[key + "lora_A.weight"], mod.lora_A.grad, atol=1e-6, rtol=1e-4)
        assert torch.allclose(grads[key + "lora_B.weight"], mod.lora_B.grad, atol=1e-6, rtol=1e-4)


@pytest.mark.parametrize("case", ["mha_qv", "gqa_qv"])
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
    hf = dict(m.named_parameters())
    assert set(grads) == set(hf)
    for k, gr in grads.items():
        assert torch.allclose(gr, hf[k].grad, atol=1e-6, rtol=1e-3), (k, float((gr - hf[k].grad).abs().max()))
    for name in ("self_attn.q_norm", "self_attn.k_norm", "post_attention_layernorm", "post_feedforward_layernorm"):
        assert float(grads[f"model.layers.1.{name}.weight"].abs().max()) > 0
        assert FO.no_decay(cfg, f"model.layers.1.{name}.weight")


# ---------------------------------------------------------------------------------------------------------------------------
# config loader
# ---------------------------------------------------------------------------------------------------------------------------
OLMO2_7B = {"architectures": ["Olmo2ForCausalLM"], "attention_bias": False, "attention_dropout": 0.0, "eos_token_id": 100257,
            "hidden_act": "silu", "hidden_size": 4096, "initializer_range": 0.02, "intermediate_size": 11008,
            "max_position_embeddings": 4096, "model_type": "olmo2", "num_attention_heads": 32, "num_hidden_layers": 32,
            "num_key_value_heads": 32, "pad_token_id": 100277, "rms_norm_eps": 1e-06, "rope_scaling": None, "rope_theta": 500000,
            "tie_word_embeddings": False, "torch_dtype": "bfloat16", "use_cache": True, "vocab_size": 100352}
OLMO2_13B = dict(OLMO2_7B, hidden_size=5120, intermediate_size=13824, num_attention_heads=40, num_hidden_layers=40,
                 num_key_value_heads=40)
OLMO2_32B = dict(OLMO2_7B, hidden_size=5120, intermediate_size=27648, num_attention_heads=40, num_hidden_layers=64,
                 num_key_value_heads=8)


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


@pytest.mark.parametrize("name,cfg,d,dkv,layers", [
    ("olmo2_7b", OLMO2_7B, 4096, 4096, 32),
    ("olmo2_13b", OLMO2_13B, 5120, 5120, 40),
    ("olmo2_32b", OLMO2_32B, 5120, 1024, 64),
])
def test_loader_accepts(lib, tmp_path, name, cfg, d, dkv, layers):
    from datatunerx_b200.tuning import model_io
    dd = _cfg_dir(tmp_path, cfg)
    mc = model_io.load_model_config(dd)
    assert mc.hidden == d and mc.n_heads * mc.head_dim == d and mc.n_kv_heads * mc.head_dim == dkv and mc.n_layers == layers
    assert mc.head_dim == 128 and mc.rms_eps == 1e-6 and mc.rope_theta == 500000 and mc.rope_scaling is None
    assert mc.qk_norm_full and mc.no_pre_norms and mc.post_norms and not mc.qk_norm and not mc.qkv_bias and not mc.rope_glm
    ext = mc.ext_to_c()
    assert (ext.qk_norm_full, ext.no_pre_norms, ext.post_norms, ext.qk_norm, ext.rope_glm, ext.qkv_bias) == (1, 1, 1, 0, 0, 0)
    assert _accepted(mc)
    assert _accepted(model_io.load_model_config(dd, full_finetune=True), full=True)


@pytest.mark.parametrize("case", ["attention_bias", "gelu", "yarn", "tied_full", "olmo1", "olmo3", "olmoe"])
def test_loader_refusals(tmp_path, case):
    from datatunerx_b200.tuning import model_io
    full = False
    if case == "attention_bias":
        cfg = dict(OLMO2_7B, attention_bias=True)
    elif case == "gelu":
        cfg = dict(OLMO2_7B, hidden_act="gelu")
    elif case == "yarn":
        cfg = dict(OLMO2_7B, rope_scaling={"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 4096})
    elif case == "tied_full":
        cfg, full = dict(OLMO2_7B, tie_word_embeddings=True), True
    elif case == "olmo1":  # OLMo-1: LayerNorm without weights
        cfg = dict(OLMO2_7B, architectures=["OlmoForCausalLM"], model_type="olmo", clip_qkv=None)
    elif case == "olmo3":  # per-layer sliding windows
        cfg = dict(OLMO2_7B, architectures=["Olmo3ForCausalLM"], model_type="olmo3", sliding_window=4096,
                   layer_types=["sliding_attention", "full_attention"] * 16)
    else:
        cfg = dict(OLMO2_7B, architectures=["OlmoeForCausalLM"], model_type="olmoe", num_experts=64, num_experts_per_tok=8)
    with pytest.raises(ValueError):
        model_io.load_model_config(_cfg_dir(tmp_path, cfg), full_finetune=full)


def test_tied_checkpoint_trains_with_lora(tmp_path):
    from datatunerx_b200.tuning import model_io
    mc = model_io.load_model_config(_cfg_dir(tmp_path, dict(OLMO2_7B, tie_word_embeddings=True)))
    assert mc.qk_norm_full and mc.no_pre_norms


# ---------------------------------------------------------------------------------------------------------------------------
# ABI, weight names and memory plan
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ext_kw,word", [
    (dict(qk_norm_full=2), "qk_norm_full"), (dict(qk_norm_full=-1), "qk_norm_full"),
    (dict(no_pre_norms=2, post_norms=1), "no_pre_norms"), (dict(no_pre_norms=-1, post_norms=1), "no_pre_norms"),
    (dict(qk_norm_full=1, qk_norm=1), "qk_norm_full"), (dict(qk_norm_full=1, rope_glm=1), "qk_norm_full"),
    (dict(no_pre_norms=1), "no_pre_norms"), (dict(no_pre_norms=1, qk_norm_full=1), "no_pre_norms"),
])
def test_bad_ext_is_refused_without_a_device(lib, ext_kw, word):
    from datatunerx_b200 import lib as L
    mc = L.ModelConfig(vocab=2048, hidden=256, n_layers=1, n_heads=4, ffn=768).to_c()
    tc = L.TrainConfig(micro_batch=1, seq_len=128, total_steps=1, lora_dropout=0.0).to_c()
    out = (C.c_float * 64)()
    ext = L.ModelExt(**ext_kw)
    h, n = C.c_void_p(), C.c_int64()
    assert lib.dtx_trainer_create_ext(C.byref(mc), C.byref(ext), C.byref(tc), 0, 0, 1, None, C.byref(h)) == -1
    assert not h.value
    assert word in L.load().dtx_last_global_error().decode()
    assert lib.dtx_plan_device_bytes_ext(C.byref(mc), C.byref(ext), C.byref(tc), 1, 1, C.byref(n)) == -1
    assert lib.dtx_rope_inv_freq(C.byref(mc), C.byref(ext), out) == -1


def test_kernel_entry_points_refuse_bad_shapes_without_a_device(lib):
    """argument checks run before any launch: fake (aligned) device addresses never reach a kernel"""
    p, s = C.c_void_p(1 << 20), None
    # q and k spans must be positive multiples of 128 and fit QKF_MAX_COLS; row strides multiples of 8
    for q_cols, n_cols, ld in ((4096, 4096, 8192), (4000, 8192, 8192), (4096, 8200, 8320), (8192, 16512, 16512), (4096, 8192, 8196)):
        assert lib.dtx_qk_norm_full_rope_fwd(p, ld, 16, q_cols, n_cols, p, p, 1e-6, p, 128, None, p, ld, s) == -1
        assert lib.dtx_qk_norm_full_bwd(p, ld, p, ld, 16, q_cols, n_cols, p, p, 1e-6, None, None, 0, s) == -1
    assert lib.dtx_qk_norm_full_rope_fwd(p, 8192, 16, 4096, 8192, p, p, 1e-6, None, 128, None, p, 8192, s) == -1  # no table
    assert lib.dtx_qk_norm_full_bwd(p, 8192, p, 8192, 16, 4096, 8192, p, p, 1e-6, p, None, 0, s) == -1  # dw without scratch
    assert lib.dtx_qk_norm_full_bwd(p, 8192, C.c_void_p((1 << 20) + 8), 8192, 16, 4096, 8192, p, p, 1e-6, None, None, 0, s) == -1


def _tiny(full, n_kv=2):
    from datatunerx_b200 import lib as L
    mc = L.ModelConfig(vocab=2048, hidden=256, n_layers=3, n_heads=2, n_kv_heads=n_kv, ffn=768, rms_eps=1e-6, rope_theta=5e5)
    tc = L.TrainConfig(micro_batch=2, seq_len=256, total_steps=4, lora_r=16, lora_dropout=0.0, full_finetune=full,
                       lora_target=("q_proj", "k_proj", "v_proj"))
    return mc, tc


def test_weight_names_are_olmo2s():
    from datatunerx_b200 import lib as L
    mc, tc = _tiny(True, n_kv=1)
    olmo = dataclasses.replace(mc, qk_norm_full=True, no_pre_norms=True, post_norms=True)
    tr = L.Trainer.__new__(L.Trainer)  # weight_names only reads the configuration: no device
    tr.model, tr.train = olmo, tc
    names = dict(tr.weight_names())
    cfg = FO.FamilyConfig(vocab=2048, hidden=256, n_layers=3, n_heads=2, n_kv_heads=1, ffn=768, qk_norm_full=True, no_pre_norms=True)
    ref = FO.init_base_weights(cfg)
    assert names == {k: tuple(v.shape) for k, v in ref.items()}
    assert names["model.layers.2.self_attn.q_norm.weight"] == (256,) and names["model.layers.2.self_attn.k_norm.weight"] == (128,)
    assert list(names)[0] == "model.embed_tokens.weight" and list(names)[-1] == "lm_head.weight"


@pytest.mark.parametrize("full,world,n_kv", [(False, 1, 2), (False, 1, 1), (True, 1, 2), (True, 8, 1)])
def test_olmo2_plan_bytes_follow_the_formula(lib, full, world, n_kv):
    """OLMo-2 against the same dimensions with a zero dtx_model_ext, both layouts: no h1 / rstd1 / rstd2 per saved set; the
    pre-norm q|k, o_pre, down_pre and the two post-norm rstd per saved set; per layer q_norm | k_norm and the post-norm weights
    instead of the two pre-norm weights; under full SFT the norm-gradient scratch widened to the q|k columns."""
    from datatunerx_b200 import lib as L
    mc, tc = _tiny(full, n_kv)
    olmo = dataclasses.replace(mc, qk_norm_full=True, no_pre_norms=True, post_norms=True)
    d, F, V, L_, D = mc.hidden, mc.ffn, mc.vocab, mc.n_layers, mc.head_dim
    dq, dkv = mc.n_heads * D, mc.n_kv_heads * D
    W, QK, M = dq + 2 * dkv, dq + dkv, tc.micro_batch * tc.seq_len
    for layout, sets in (("keep", L_), ("layer", 1)):
        plain, o2 = L.plan_device_bytes(mc, tc, world, layout), L.plan_device_bytes(olmo, tc, world, layout)
        per_set = -M * d * 2 - 2 * M * 4 + M * QK * 2 + 2 * M * d * 2 + 2 * M * 4
        if not full:
            assert o2 - plain == sets * per_set + L_ * (QK - 2 * d + 2 * d) * 2
        else:  # bf16 weight + gradient, fp32 master + two moments for this rank's shard of every padded layer block
            unit = world * 128
            pad = lambda n: (n + unit - 1) // unit * unit  # noqa: E731
            base = W * d + d * dq + 2 * F * d + d * F
            total = lambda layer: L_ * pad(layer) + pad(2 * V * d + d)  # noqa: E731
            t0, t1 = total(base + 2 * d), total(base + QK + 2 * d)
            scratch = 64 * (max(d, QK) - d) * 4
            assert o2 - plain == sets * per_set + (t1 - t0) * 2 * 2 + (t1 - t0) // world * 4 * 3 + scratch


def test_zero_ext_plan_is_unchanged_by_the_new_fields(lib):
    """a zero dtx_model_ext plans what the plain entry point plans"""
    from datatunerx_b200 import lib as L
    for full in (False, True):
        mc, tc = _tiny(full)
        for layout in (1, 2):
            a, b = C.c_int64(), C.c_int64()
            cm, ct, ext = mc.to_c(), tc.to_c(), L.ModelExt()
            assert lib.dtx_plan_device_bytes(C.byref(cm), C.byref(ct), 1, layout, C.byref(a)) == 0
            assert lib.dtx_plan_device_bytes_ext(C.byref(cm), C.byref(ext), C.byref(ct), 1, layout, C.byref(b)) == 0
            assert a.value == b.value > 0
