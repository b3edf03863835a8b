"""OLMo-2 (Olmo2ForCausalLM) on the GPU (-m gpu): the full-width q/k RMSNorm + rotary kernel and its backward against fp32
torch at OLMo-2-7B and -32B widths, LoRA and full-parameter SFT traces against the OLMo-2 oracle (tests/olmo2_oracle.py), NF4,
both activation layouts, packed ragged batches, the unfused epilogues, and one OLMo-2-7B-shaped layer."""
import math

import numpy as np
import pytest
import torch

from tests.conftest import has_gpu

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _need_gpu():
    if not has_gpu():
        pytest.skip("no GPU")


def _mods():
    from datatunerx_b200 import lib as L
    from oracle import llama_lora as O
    from tests import olmo2_oracle as FO
    from tests import gpu_checks as G
    return L, O, FO, G


# ---------------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------------
def _table(S, theta=500000.0):
    L, _, _, G = _mods()
    cs = torch.empty(S, 64, 2, dtype=torch.float32, device=G.DEV)
    G.ok(L.load().dtx_rope_table(G.P(cs), S, 128, theta, G.STREAM()))
    return cs


def _norm_rope_ref(x, wq, wk, dq, eps, cs, pos):
    """fp32: RMSNorm over q = x[:, :dq] and over k = x[:, dq:], times the weights, then the half-split rotary of every head"""
    q, k = x[:, :dq], x[:, dq:]
    q = q * torch.rsqrt(q.pow(2).mean(-1, keepdim=True) + eps) * wq
    k = k * torch.rsqrt(k.pow(2).mean(-1, keepdim=True) + eps) * wk
    y = torch.cat([q, k], dim=1)
    M = y.shape[0]
    h = y.reshape(M, -1, 128)
    c, s = cs[pos, :, 0][:, None, :], cs[pos, :, 1][:, None, :]
    a, b = h[..., :64], h[..., 64:]
    return torch.cat([a * c - b * s, b * c + a * s], dim=-1).reshape(M, -1)


WIDTHS = {"7b": (4096, 4096), "32b": (5120, 1024)}


@pytest.mark.parametrize("width", list(WIDTHS))
@pytest.mark.parametrize("packed", [False, True])
def test_qk_norm_full_rope_fwd_matches_torch(width, packed):
    """Norm + rotary of the plain GEMM output against fp32 torch; the saved pre-norm copy is bitwise the GEMM output and the v
    columns are untouched."""
    L, _, _, G = _mods()
    lib = L.load()
    dq, dkv = WIDTHS[width]
    W, QK, K, S, eps = dq + 2 * dkv, dq + dkv, 512, 1024, 1e-6
    M = 1024 + 512 if packed else 2048
    A, Bw = G._rand(M, K, seed=1), G._rand(W, K, scale=0.05, seed=2)
    qkv = G.gemm(A, Bw)
    plain = qkv.clone()
    wq = (1.0 + G._rand(dq, scale=0.1, seed=3).float()).to(torch.bfloat16)
    wk = (1.0 + G._rand(dkv, scale=0.1, seed=4).float()).to(torch.bfloat16)
    cs = _table(S)
    pos = torch.arange(M, device=G.DEV) % S
    rope_pos = None
    if packed:  # sequences of 1024 and 512 rows back to back
        pos = torch.cat([torch.arange(1024), torch.arange(512)]).to(G.DEV)
        rope_pos = pos.to(torch.int32).contiguous()
    pre = torch.full((M, QK), float("nan"), dtype=torch.bfloat16, device=G.DEV)
    G.ok(lib.dtx_qk_norm_full_rope_fwd(G.P(qkv), W, M, dq, QK, G.P(wq), G.P(wk), eps, G.P(cs), S, G.P(rope_pos), G.P(pre), QK,
                                       G.STREAM()))
    torch.cuda.synchronize()
    assert torch.equal(pre, plain[:, :QK])
    assert torch.equal(qkv[:, QK:], plain[:, QK:])
    ref = _norm_rope_ref(plain[:, :QK].float(), wq.float(), wk.float(), dq, eps, cs, pos)
    e = G.rel_err(qkv[:, :QK], ref)
    assert e < 4e-3, e


@pytest.mark.parametrize("width", list(WIDTHS))
def test_qk_norm_full_bwd_matches_autograd_and_dw_repeats_bitwise(width):
    """dx (in place) and the weight gradient against fp32 autograd of the norm; dw is bitwise the same on a second run, and
    accumulate = 1 adds to it."""
    L, _, _, G = _mods()
    lib = L.load()
    dq, dkv = WIDTHS[width]
    W, QK, M, eps = dq + 2 * dkv, dq + dkv, 2000, 1e-6
    x = G._rand(M, QK, scale=0.7, seed=11)
    dy0 = G._rand(M, W, scale=0.3, seed=12)
    wq = (1.0 + G._rand(dq, scale=0.1, seed=13).float()).to(torch.bfloat16)
    wk = (1.0 + G._rand(dkv, scale=0.1, seed=14).float()).to(torch.bfloat16)
    scratch = torch.empty(64 * QK, dtype=torch.float32, device=G.DEV)
    outs = []
    for run in range(2):
        dy = dy0.clone()
        dw = torch.full((QK,), float("nan"), dtype=torch.bfloat16, device=G.DEV)
        G.ok(lib.dtx_qk_norm_full_bwd(G.P(dy), W, G.P(x), QK, M, dq, QK, G.P(wq), G.P(wk), eps, G.P(dw), G.P(scratch), 0, G.STREAM()))
        torch.cuda.synchronize()
        outs.append((dy, dw))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    dy, dw = outs[0]
    # without dw: the same dx
    dy2 = dy0.clone()
    G.ok(lib.dtx_qk_norm_full_bwd(G.P(dy2), W, G.P(x), QK, M, dq, QK, G.P(wq), G.P(wk), eps, None, None, 0, G.STREAM()))
    acc = dw.clone()
    G.ok(lib.dtx_qk_norm_full_bwd(G.P(dy0.clone()), W, G.P(x), QK, M, dq, QK, G.P(wq), G.P(wk), eps, G.P(acc), G.P(scratch), 1,
                                  G.STREAM()))
    torch.cuda.synchronize()
    assert torch.equal(dy2, dy)
    assert torch.equal(dy[:, QK:], dy0[:, QK:])
    xr = x.float().requires_grad_(True)
    wqr, wkr = wq.float().requires_grad_(True), wk.float().requires_grad_(True)
    q, k = xr[:, :dq], xr[:, dq:]
    y = torch.cat([q * torch.rsqrt(q.pow(2).mean(-1, keepdim=True) + eps) * wqr,
                   k * torch.rsqrt(k.pow(2).mean(-1, keepdim=True) + eps) * wkr], dim=1)
    (y * dy0[:, :QK].float()).sum().backward()
    assert G.rel_err(dy[:, :QK], xr.grad) < 4e-3
    assert G.rel_err(dw, torch.cat([wqr.grad, wkr.grad])) < 4e-3
    assert G.rel_err(acc, 2 * torch.cat([wqr.grad, wkr.grad])) < 8e-3


# ---------------------------------------------------------------------------------------------------------------------------
# training against the OLMo-2 oracle
# ---------------------------------------------------------------------------------------------------------------------------
OLMO2 = dict(rope_theta=500000.0, rms_eps=1e-6, qk_norm_full=True, no_pre_norms=True)
DIMS = {
    "mha": dict(vocab=2048, hidden=512, n_layers=2, n_heads=4, n_kv_heads=4, ffn=768, **OLMO2),
    # OLMo-2-32B's 5:1 grouped-query ratio
    "gqa": dict(vocab=2048, hidden=1280, n_layers=2, n_heads=10, n_kv_heads=2, ffn=768, **OLMO2),
}


def _pair(family, targets=("q_proj", "v_proj"), steps=20, full=False, S=256, B=2, quant=False, weight_decay=0.0, dropout=0.0):
    L, O, FO, _ = _mods()
    dims = DIMS[family]
    ocfg = FO.FamilyConfig(**dims, lora_r=16, lora_alpha=32.0, lr=1e-3, total_steps=steps, lora_dropout=dropout,
                           lora_target=tuple(targets), full_finetune=full, weight_decay=weight_decay)
    mc = L.ModelConfig(**dims, post_norms=True)
    tc = L.TrainConfig(micro_batch=B, seq_len=S, total_steps=steps, lora_r=16, lora_alpha=32.0, lora_dropout=dropout, lr=1e-3,
                       lora_target=tuple(targets), full_finetune=full, weight_decay=weight_decay)
    w = FO.init_base_weights(ocfg, 1234)
    lora = {} if full else FO.init_lora(ocfg, 4321)
    tr = L.Trainer(mc, tc)
    tr.load_state_dict({k: v.numpy() for k, v in w.items()})
    if quant:
        tr.quantize_base("int4")
        w = O.quantize_base_nf4(w)
    tr.load_state_dict({k: v.numpy() for k, v in lora.items()})
    return ocfg, FO.FamilyTrainer(ocfg, w, lora), tr


@pytest.mark.parametrize("family,targets,dropout", [
    ("mha", ("q_proj", "v_proj"), 0.0),
    ("mha", ("q_proj", "k_proj", "v_proj"), 0.0),
    ("mha", ("q_proj", "v_proj"), 0.1),
    ("gqa", ("q_proj", "v_proj"), 0.0),
    ("gqa", ("q_proj", "k_proj", "v_proj"), 0.1),
])
def test_lora_trace_matches_olmo2_oracle(family, targets, dropout):
    """20 steps (and one dtx_eval_loss) against the oracle; with dropout both sides draw the same masks"""
    from tests.test_model_families_gpu import _lora_trace
    ocfg, orc, tr = _pair(family, targets, steps=20, dropout=dropout)
    _lora_trace(ocfg, orc, tr, 20)


@pytest.mark.parametrize("family", ["mha", "gqa"])
def test_lora_nf4_olmo2_matches_oracle(family):
    """NF4 packs the four projection matrices; q_norm / k_norm and the post-sublayer norms stay bf16"""
    from tests.test_model_families_gpu import _lora_trace
    ocfg, orc, tr = _pair(family, steps=20, quant=True)
    _lora_trace(ocfg, orc, tr, 20)


@pytest.mark.parametrize("family", ["mha", "gqa"])
def test_full_sft_olmo2_matches_oracle(family):
    L, O, FO, G = _mods()
    steps = 6
    ocfg, orc, tr = _pair(family, full=True, steps=steps, weight_decay=0.1)
    worst_l = worst_g = 0.0
    grad_errs = {}
    for s in range(steps):
        ids, labels = O.synthetic_batch(s, 0, 2, 256, ocfg.vocab)
        ref = orc.step([(ids, labels)])
        loss, gn, _, stepped = tr.step(ids, labels)
        assert stepped
        if s == 0:
            got = tr.export_weights(grads=True)
            assert set(got) == set(orc.last_grads)
            for k, v in got.items():
                r = orc.last_grads[k].numpy()
                assert v.shape == r.shape, k
                grad_errs[k] = float(np.linalg.norm(G._bf16_bits_to_f32(v) - r) / max(np.linalg.norm(r), 1e-12))
        worst_l = max(worst_l, abs(loss - ref.loss) / ref.loss)
        worst_g = max(worst_g, abs(gn - ref.grad_norm) / ref.grad_norm)
    wts = tr.export_weights()
    tr.close()
    want = {k: v.detach() for k, v in orc.lora.items()}
    norms = [k for k in grad_errs if k.endswith(("q_norm.weight", "k_norm.weight", "post_attention_layernorm.weight",
                                                 "post_feedforward_layernorm.weight"))]
    assert len(norms) == 4 * ocfg.n_layers
    drift = {k: float(np.linalg.norm(G._bf16_bits_to_f32(v) - want[k].numpy()) / max(np.linalg.norm(want[k].numpy()), 1e-12))
             for k, v in wts.items()}
    assert max(grad_errs.values()) < 5e-2, grad_errs
    assert worst_l < 2e-3 and worst_g < 3e-2, (worst_l, worst_g)
    assert max(drift.values()) < 1e-2, drift


# ---------------------------------------------------------------------------------------------------------------------------
# an OLMo-2 model through the layouts and paths of the trainer
# ---------------------------------------------------------------------------------------------------------------------------
def _olmo_cfg(full=False, dropout=0.0):
    L, _, _, _ = _mods()
    mc = L.ModelConfig(vocab=2048, hidden=1280, n_layers=3, n_heads=10, n_kv_heads=2, ffn=768, post_norms=True, **OLMO2)
    tc = L.TrainConfig(micro_batch=2, seq_len=384, total_steps=8, lora_r=16, lora_dropout=dropout, lr=1e-3, full_finetune=full,
                       lora_target=("q_proj", "k_proj", "v_proj"), weight_decay=0.1)
    return mc, tc


@pytest.mark.parametrize("full,dropout", [(False, 0.0), (False, 0.1), (True, 0.0)])
def test_olmo2_keep_recompute_and_repeat_are_bitwise_equal(full, dropout):
    from tests.test_model_families_gpu import _batches, _run
    mc, tc = _olmo_cfg(full, dropout)
    batches = _batches(mc.vocab, 4)
    a, b, c = _run(mc, tc, batches, "keep"), _run(mc, tc, batches, "layer"), _run(mc, tc, batches, "keep")
    assert a[0] == b[0] == c[0]
    for k in a[1]:
        assert a[1][k].tobytes() == b[1][k].tobytes() == c[1][k].tobytes(), k
        assert a[2][k].tobytes() == b[2][k].tobytes() == c[2][k].tobytes(), k


@pytest.mark.parametrize("full", [False, True])
def test_olmo2_packed_ragged_matches_padded(full):
    from tests.test_model_families_gpu import _batches, _close, _run
    mc, tc = _olmo_cfg(full)
    batches = _batches(mc.vocab, 3, lens=[384, 200])
    packed = _run(mc, tc, batches)
    padded = _run(mc, tc, batches, options={"varlen_pack": 0, "varlen_split": 0})
    assert packed[3] == 0 and padded[3] == 1
    for (l1, g1), (l2, g2) in zip(packed[0], padded[0]):
        assert abs(l1 - l2) / l2 < 2e-3 and abs(g1 - g2) / g2 < 3e-2, (packed[0], padded[0])
    _close(packed[2], padded[2], 5e-2)


@pytest.mark.parametrize("full", [False, True])
def test_olmo2_unfused_epilogues_match_fused(full):
    from tests.test_model_families_gpu import _batches, _close, _run
    mc, tc = _olmo_cfg(full)
    batches = _batches(mc.vocab, 3)
    fused = _run(mc, tc, batches)
    unfused = _run(mc, tc, batches, options={"fused_epilogues": 0})
    for (l1, g1), (l2, g2) in zip(fused[0], unfused[0]):
        assert abs(l1 - l2) / l2 < 2e-3 and abs(g1 - g2) / g2 < 3e-2, (fused[0], unfused[0])
    _close(_run(mc, tc, batches[:1])[2], _run(mc, tc, batches[:1], options={"fused_epilogues": 0})[2], 5e-2)


def test_layer_olmo2_7b_shape():
    """One OLMo-2-7B-shaped layer (d = 4096, 32 / 32 heads, F = 11008: q|k width 8192 in the norm kernels) + lm_head + CE through
    the trainer at B = 2, S = 2048 against the fp32 oracle on the host cores."""
    L, O, FO, _ = _mods()
    dims = dict(vocab=32000, hidden=4096, n_layers=1, n_heads=32, n_kv_heads=32, ffn=11008, **OLMO2)
    ocfg = FO.FamilyConfig(**dims, lora_r=16, lora_alpha=32.0, lr=1e-4, total_steps=10, lora_dropout=0.0)
    mc = L.ModelConfig(**dims, post_norms=True)
    B, S = 2, 2048
    tc = L.TrainConfig(micro_batch=B, seq_len=S, total_steps=10, lora_r=16, lora_alpha=32.0, lora_dropout=0.0, lr=1e-4)
    w, lora = FO.init_base_weights(ocfg, 1234), FO.init_lora(ocfg, 4321)
    g = torch.Generator().manual_seed(99)
    for k in lora:  # B = 0 at init would leave the A gradients identically zero
        if "lora_B" in k:
            lora[k] = torch.randn(lora[k].shape, generator=g) * 0.01
    tr = L.Trainer(mc, tc)
    tr.load_state_dict({k: v.numpy() for k, v in w.items()})
    tr.load_state_dict({k: v.numpy() for k, v in lora.items()})
    orc = FO.FamilyTrainer(ocfg, w, lora)
    ids, labels = O.synthetic_batch(0, 0, B, S, ocfg.vocab)
    ref_loss, g_ref = orc.loss_and_grads(ids, labels)
    e_eval = abs(tr.eval_loss(ids, labels) - ref_loss) / ref_loss
    loss, gn, _, stepped = tr.step(ids, labels)
    ref_norm = math.sqrt(sum(float((v.double() ** 2).sum()) for v in g_ref.values()))
    errs = {}
    for k, v in tr.export_adapter(grads=True).items():
        r = g_ref[k.replace("base_model.model.", "")].numpy()
        errs[k.split("layers.0.")[1]] = float(np.linalg.norm(v - r) / max(np.linalg.norm(r), 1e-12))
    tr.close()
    assert stepped
    assert e_eval < 1e-3 and abs(loss - ref_loss) / ref_loss < 1e-3, (e_eval, loss, ref_loss)
    assert abs(gn - ref_norm) / ref_norm < 3e-2, (gn, ref_norm)
    assert max(errs.values()) < 5e-2, errs


def test_olmo2_norm_weights_are_required_and_input_layernorm_is_refused():
    L, O, FO, _ = _mods()
    mc, tc = _olmo_cfg()
    tr = L.Trainer(mc, tc)
    with pytest.raises(L.DtxError) as e:
        tr.load_tensor("model.layers.0.input_layernorm.weight", np.ones(1280, np.float32))
    assert e.value.code == -1
    ocfg = FO.FamilyConfig(vocab=2048, hidden=1280, n_layers=3, n_heads=10, n_kv_heads=2, ffn=768, **OLMO2)
    w = FO.init_base_weights(ocfg, 1)
    tr.load_state_dict({k: v.numpy() for k, v in w.items() if not k.endswith("k_norm.weight")})
    tr.init_lora(1)
    ids, labels = O.synthetic_batch(0, 0, 2, 384, mc.vocab)
    with pytest.raises(L.DtxError) as e:
        tr.step(ids, labels)
    assert e.value.code == -4 and "k_norm" in str(e.value)
    tr.close()
