"""Activation layouts: the device-memory planner (host arithmetic inside the library, no GPU needed) and the checks of the
recompute setting, which run before any device work."""
import ctypes as C

import pytest

GiB = 1 << 30


def _saved_per_layer(mc, tc):
    """Bytes of one layer's saved activations, from the shapes: h1, qkv, attn, x_mid, gate|up (bf16), the LoRA t and the
    dropped LoRA inputs (bf16), lse and the two rstd vectors (fp32)."""
    from datatunerx_b200 import lib as L
    d, F, H = mc.hidden, mc.ffn, mc.n_heads
    Hkv = mc.n_kv_heads or H
    B, S = tc.micro_batch, tc.seq_len
    M, W = B * S, (H + 2 * Hkv) * mc.head_dim
    nt = len(tc.lora_target)
    RP = (nt * tc.lora_r + 63) // 64 * 64
    dropout = not tc.full_finetune and tc.lora_dropout > 0
    KA = nt * d if dropout else d
    bf16 = M * d + M * W + M * d + M * d + M * 2 * F
    if not tc.full_finetune:
        bf16 += M * RP
    if dropout:
        bf16 += M * KA
    return 2 * bf16 + 4 * (B * H * S + 2 * M)


def _plan(mc, tc, world=1):
    from datatunerx_b200 import lib as L
    return L.plan_device_bytes(mc, tc, world, "keep"), L.plan_device_bytes(mc, tc, world, "layer")


def _tiny(**kw):
    from datatunerx_b200 import lib as L
    heads, kv = kw.pop("heads", 2), kw.pop("kv_heads", None)
    mc = L.ModelConfig(vocab=2048, hidden=128 * heads, n_layers=kw.pop("layers", 3), n_heads=heads, n_kv_heads=kv, ffn=768)
    tc = L.TrainConfig(micro_batch=2, seq_len=256, total_steps=10, lora_r=16, **kw)
    return mc, tc


@pytest.mark.parametrize("case", ["lora_qv", "lora_dropout", "gqa_qkv", "full_world1", "full_world8"])
def test_layout_difference_is_the_per_layer_saved_set(lib, case):
    kw = {"lora_qv": dict(lora_dropout=0.0),
          "lora_dropout": dict(lora_dropout=0.1),
          "gqa_qkv": dict(heads=4, kv_heads=2, lora_dropout=0.0, lora_target=("q_proj", "k_proj", "v_proj")),
          "full_world1": dict(full_finetune=True),
          "full_world8": dict(full_finetune=True)}[case]
    mc, tc = _tiny(**kw)
    world = 8 if case == "full_world8" else 1
    keep, layer = _plan(mc, tc, world)
    assert keep - layer == (mc.n_layers - 1) * _saved_per_layer(mc, tc), (case, keep, layer)


def test_one_layer_model_has_one_layout(lib):
    mc, tc = _tiny(layers=1, lora_dropout=0.0)
    keep, layer = _plan(mc, tc)
    assert keep == layer


def test_headline_config_keeps_all_activations(lib):
    """Llama-2-7B LoRA at batch 4 x 2048: keep-all fits an 80 GiB card with the 1 GiB reserve, so automatic mode keeps today's
    allocation."""
    from datatunerx_b200 import lib as L
    mc = L.ModelConfig.llama2_7b()
    tc = L.TrainConfig(micro_batch=4, seq_len=2048, total_steps=10, lora_r=16, lora_dropout=0.0)
    keep, layer = _plan(mc, tc)
    assert keep + GiB < 80 * GiB and layer < keep, (keep, layer)


@pytest.mark.parametrize("case", ["7b_lora_b8_s4096", "13b_full_world8"])
def test_large_configs_fit_only_with_recompute(lib, case):
    from datatunerx_b200 import lib as L
    if case == "7b_lora_b8_s4096":
        mc = L.ModelConfig.llama2_7b()
        tc = L.TrainConfig(micro_batch=8, seq_len=4096, total_steps=10, lora_r=16, lora_dropout=0.0)
        world = 1
    else:
        mc = L.ModelConfig(vocab=32000, hidden=5120, n_layers=40, n_heads=40, ffn=13824)
        tc = L.TrainConfig(micro_batch=2, seq_len=2048, total_steps=10, full_finetune=True)
        world = 8
    keep, layer = _plan(mc, tc, world)
    assert keep > 80 * GiB and layer + GiB < 80 * GiB, (case, keep / GiB, layer / GiB)


def test_bad_recompute_value_is_rejected_before_device_work(lib):
    from datatunerx_b200 import lib as L
    mc, tc = _tiny(lora_dropout=0.0)
    cm, ct = mc.to_c(), tc.to_c()
    for bad in (-1, 3, 7):
        ct.recompute = bad
        h = C.c_void_p()
        assert lib.dtx_trainer_create(C.byref(cm), C.byref(ct), 0, 0, 1, None, C.byref(h)) == -1
        assert b"recompute" in lib.dtx_last_global_error()
        assert not h.value
    with pytest.raises(L.DtxError) as e:
        L.TrainConfig(micro_batch=1, seq_len=128, total_steps=1, recompute="sometimes").to_c()
    assert e.value.code == -1


def test_planner_rejects_bad_layouts_and_configs(lib):
    from datatunerx_b200 import lib as L
    mc, tc = _tiny(lora_dropout=0.0)
    for layout in (0, 3, -1, "auto"):
        with pytest.raises(L.DtxError) as e:
            L.plan_device_bytes(mc, tc, 1, layout)
        assert e.value.code == -1, layout
    with pytest.raises(L.DtxError) as e:
        L.plan_device_bytes(mc, tc, 0, "keep")
    assert e.value.code == -1
    bad_mc = L.ModelConfig(vocab=256, hidden=256, n_layers=1, n_heads=4, head_dim=64, ffn=256)
    with pytest.raises(L.DtxError) as e:
        L.plan_device_bytes(bad_mc, tc, 1, "keep")
    assert e.value.code == -1


def test_recompute_strings_map_to_the_struct_field(lib):
    from datatunerx_b200 import lib as L
    for name, code in (("auto", 0), ("keep", 1), ("layer", 2)):
        assert L.TrainConfig(micro_batch=1, seq_len=128, total_steps=1, recompute=name).to_c().recompute == code
    assert L.TrainConfig(micro_batch=1, seq_len=128, total_steps=1).to_c().recompute == 0
