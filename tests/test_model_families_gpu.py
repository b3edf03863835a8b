"""Llama-3.x (llama3-scaled rotary table) and Qwen2 (q/k/v biases) on the GPU (-m gpu): the bias epilogues of the GEMM, the
bias-gradient kernel, LoRA and full-parameter SFT traces against the family oracle (tests/family_oracle.py), NF4, both
activation layouts, packed ragged batches and the unfused epilogues of a bias model."""
import dataclasses

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
    from tests import family_oracle as FO
    from tests import gpu_checks as G
    return L, O, FO, G


# ---------------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------------
def _gemm_bias(A, B, bias, epi, A2=None, B2=None, rope_cs=None, rope_S=0, rope_cols=0, rope_pos=None):
    L, _, _, G = _mods()
    M, K = A.shape
    N = B.shape[0]
    Cm = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=A.device)
    rc = L.load().dtx_gemm_bias(G.P(A), A.stride(0), G.P(B), B.stride(0), 0, G.P(A2), A2.stride(0) if A2 is not None else 0, G.P(B2),
                                B2.stride(0) if B2 is not None else 0, A2.shape[1] if A2 is not None else 0, G.P(Cm), N, None, 0,
                                G.P(rope_cs), rope_S, rope_cols, G.P(rope_pos), M, N, K, epi, G.P(bias), G.STREAM())
    torch.cuda.synchronize()
    return rc, Cm


def _rope_ref_pos(x, pos, n_rot, D=128):
    _, O, _, _ = _mods()
    cos, sin = O.rope_cos_sin(int(pos.max()) + 1, D, 10000.0)
    cos, sin = cos.to(x.device)[pos], sin.to(x.device)[pos]
    M = x.shape[0]
    h = x[:, : n_rot * D].reshape(M, n_rot, D)
    rot = h * cos[:, None, :] + O.rotate_half(h) * sin[:, None, :]
    return torch.cat([rot.reshape(M, -1), x[:, n_rot * D:]], dim=1)


@pytest.mark.parametrize("epi", ["bf16_wide", "bf16_narrow", "rope", "rope_pos"])
@pytest.mark.parametrize("kext", [False, True])
def test_gemm_bias_epilogue(epi, kext):
    """bias added to the fp32 accumulator before the rounding / the rotary, at the tolerance of the existing GEMM checks; a zero
    bias gives bitwise the output of the kernel without bias."""
    L, _, _, G = _mods()
    H, Hkv, D, K = 6, 2, 128, 768
    W = (H + 2 * Hkv) * D
    M = 1000 if epi != "rope_pos" else 640
    A, Bw = G._rand(M, K, seed=61), G._rand(W, K, scale=0.05, seed=62)
    A2, B2 = (G._rand(M, 64, seed=63), G._rand(W, 64, scale=0.05, seed=64)) if kext else (None, None)
    bias = G._rand(W, scale=0.5, seed=65)
    acc = A.float() @ Bw.float().t() + (A2.float() @ B2.float().t() if kext else 0) + bias.float()
    if epi.startswith("bf16"):
        L.set_option("gemm_pair_kernel", 1 if epi == "bf16_wide" else 0)
        try:
            rc, got = _gemm_bias(A, Bw, bias, L.EPI_BF16, A2, B2)
            _, zero = _gemm_bias(A, Bw, torch.zeros_like(bias), L.EPI_BF16, A2, B2)
            plain = G.gemm(A, Bw, A2=A2, B2=B2)
        finally:
            L.set_option("gemm_pair_kernel", 1)
        ref = acc
    else:
        S = 384
        cs = G._rope_table(S)
        pos = torch.arange(M, device=G.DEV) % S
        rope_pos = None
        if epi == "rope_pos":  # packed ragged batch: sequences of 384 and 256 rows back to back
            pos = torch.cat([torch.arange(384), torch.arange(256)]).to(G.DEV)
            rope_pos = pos.to(torch.int32).contiguous()
        rc, got = _gemm_bias(A, Bw, bias, L.EPI_ROPE, A2, B2, cs, S, (H + Hkv) * D, rope_pos)
        _, zero = _gemm_bias(A, Bw, torch.zeros_like(bias), L.EPI_ROPE, A2, B2, cs, S, (H + Hkv) * D, rope_pos)
        plain = G.gemm_fused(A, Bw, L.EPI_ROPE, A2=A2, B2=B2, rope_cs=cs, rope_S=S, rope_cols=(H + Hkv) * D) if rope_pos is None else None
        ref = _rope_ref_pos(acc, pos, H + Hkv)
    assert rc == 0
    e = G.rel_err(got, ref)
    assert e < 6e-3, f"{epi} kext={kext} rel_err {e}"
    if plain is not None:
        assert torch.equal(zero, plain), "a zero bias must give the no-bias kernel's bits"
    assert G.rel_err(got, ref) < G.rel_err(zero, ref), "the bias must matter"


def test_gemm_bias_refuses_other_epilogues():
    L, _, _, G = _mods()
    A, Bw, bias = G._rand(256, 256, seed=1), G._rand(256, 256, seed=2), G._rand(256, seed=3)
    for epi in (L.EPI_F32, L.EPI_BF16_ADD, L.EPI_SWIGLU_FWD, L.EPI_SWIGLU_BWD):
        rc, _ = _gemm_bias(A, Bw, bias, epi)
        assert rc == -1, epi


def test_bias_grad_kernel_matches_column_sums_and_repeats_bitwise():
    L, _, _, G = _mods()
    lib = L.load()
    M, W, ld = 1000, 1280, 1408
    dy = G._rand(M, ld, scale=0.3, seed=71)
    ref = dy[:, :W].float().sum(0)
    outs = []
    for _ in range(2):
        db = torch.zeros(W, dtype=torch.bfloat16, device=G.DEV)
        G.ok(lib.dtx_bias_grad(G.P(dy), ld, M, W, G.P(db), 0, G.STREAM()))
        G.ok(lib.dtx_bias_grad(G.P(dy), ld, M, W, G.P(db), 1, G.STREAM()))  # accumulate: twice the sum
        torch.cuda.synchronize()
        outs.append(db.clone())
    assert torch.equal(outs[0], outs[1]), "the bias gradient must be bitwise repeatable"
    e = G.rel_err(outs[0], 2 * ref)
    assert e < 6e-3, e


# ---------------------------------------------------------------------------------------------------------------------------
# training against the family oracle
# ---------------------------------------------------------------------------------------------------------------------------
LLAMA3 = dict(rope_theta=500000.0, rope_scaling={"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0,
                                                 "high_freq_factor": 4.0, "original_max_position_embeddings": 64})
QWEN2 = dict(rope_theta=1000000.0, rms_eps=1e-6, qkv_bias=True)


def _pair(family, targets=("q_proj", "v_proj"), steps=20, tied=False, full=False, S=256, B=2, quant=False, weight_decay=0.0):
    L, O, FO, _ = _mods()
    ext = LLAMA3 if family == "llama3" else QWEN2
    dims = dict(vocab=2048, hidden=768, n_layers=2, n_heads=6, n_kv_heads=2, ffn=768)
    ocfg = FO.FamilyConfig(**dims, **ext, lora_r=16, lora_alpha=32.0, lr=1e-3, total_steps=steps, lora_dropout=0.0,
                           lora_target=tuple(targets), full_finetune=full, weight_decay=weight_decay)
    mc = L.ModelConfig(**dims, **ext)
    tc = L.TrainConfig(micro_batch=B, seq_len=S, total_steps=steps, lora_r=16, lora_alpha=32.0, lora_dropout=0.0, lr=1e-3,
                       lora_target=tuple(targets), full_finetune=full, weight_decay=weight_decay)
    w = FO.init_base_weights(ocfg, 1234, tied=tied)
    lora = {} if full else O.init_lora(ocfg, 4321)
    tr = L.Trainer(mc, tc)
    tr.load_state_dict({k: v.numpy() for k, v in w.items()})
    if quant:
        tr.quantize_base("int4")
        w = O.quantize_base_nf4(w)
    tr.load_state_dict({k: v.numpy() for k, v in lora.items()})
    return ocfg, FO.FamilyTrainer(ocfg, w, lora), tr


def _lora_trace(ocfg, orc, tr, steps, gnorm_bar=3e-2):
    _, O, _, _ = _mods()
    S, B = tr.train.seq_len, tr.train.micro_batch
    ids, labels = O.synthetic_batch(0, 0, B, S, ocfg.vocab)
    ref_eval = orc.eval_loss(ids, labels)  # one forward pass on each side
    e_eval = abs(tr.eval_loss(ids, labels) - ref_eval) / ref_eval
    worst_l = worst_g = 0.0
    for s in range(steps):
        ids, labels = O.synthetic_batch(s, 0, B, S, ocfg.vocab)
        ref = orc.step([(ids, labels)])
        loss, gn, lr, stepped = tr.step(ids, labels)
        assert stepped and abs(lr - ref.lr) <= 1e-9 + 1e-6 * ref.lr
        worst_l = max(worst_l, abs(loss - ref.loss) / ref.loss)
        worst_g = max(worst_g, abs(gn - ref.grad_norm) / ref.grad_norm)
    ad, ref_ad = tr.export_adapter(), orc.state_dict()
    worst_a = max(float(np.linalg.norm(v - ref_ad[k.replace("base_model.model.", "")]) /
                        max(np.linalg.norm(ref_ad[k.replace("base_model.model.", "")]), 1e-12)) for k, v in ad.items())
    tr.close()
    res = {"eval": e_eval, "loss": worst_l, "gnorm": worst_g, "adapter": worst_a}
    assert e_eval < 1e-3 and worst_l < 1e-3 and worst_g < gnorm_bar and worst_a < 0.15, res  # the bars of check_trainer_tiny
    return res


@pytest.mark.parametrize("family,targets,tied", [
    ("llama3", ("q_proj", "v_proj"), False),
    ("llama3", ("q_proj", "k_proj", "v_proj"), False),
    ("qwen2", ("q_proj", "v_proj"), True),
    ("qwen2", ("q_proj", "k_proj", "v_proj"), False),
])
def test_lora_trace_matches_family_oracle(family, targets, tied):
    ocfg, orc, tr = _pair(family, targets, steps=20, tied=tied)
    # Qwen2's q/k biases (N(0, 0.1) here) shift the attention logits, so the bf16 rounding of q and k moves the softmax more than
    # in the bias-free models: the grad norm of the tied Qwen2 run drifted 3.07 % from the fp32 oracle on an H100 (bar 3 %)
    _lora_trace(ocfg, orc, tr, 20, gnorm_bar=4e-2 if family == "qwen2" else 3e-2)


def test_lora_nf4_with_bias_matches_oracle():
    ocfg, orc, tr = _pair("qwen2", steps=20, quant=True)
    _lora_trace(ocfg, orc, tr, 20, gnorm_bar=4e-2)


def test_full_sft_qwen2_matches_oracle_with_bias_weights_and_grads():
    L, O, _, G = _mods()
    steps = 6
    ocfg, orc, tr = _pair("qwen2", full=True, steps=steps, weight_decay=0.1)
    worst_l = worst_g = 0.0
    grad_errs = {}
    for s in range(steps):
        ids, labels = O.synthetic_batch(s, 0, 2, 256, ocfg.vocab)
        ref = orc.step([(ids, labels)])
        loss, gn, _, stepped = tr.step(ids, labels)
        assert stepped
        if s == 0:
            got = tr.export_weights(grads=True)
            for k, v in got.items():
                r = orc.last_grads[k].numpy()
                grad_errs[k] = float(np.linalg.norm(G._bf16_bits_to_f32(v) - r) / max(np.linalg.norm(r), 1e-12))
        worst_l = max(worst_l, abs(loss - ref.loss) / ref.loss)
        worst_g = max(worst_g, abs(gn - ref.grad_norm) / ref.grad_norm)
    wts = tr.export_weights()
    tr.close()
    assert any(k.endswith(".bias") for k in grad_errs)
    drift = {k: float(np.linalg.norm(G._bf16_bits_to_f32(v) - orc.lora[k].detach().numpy()) /
                      max(np.linalg.norm(orc.lora[k].detach().numpy()), 1e-12)) for k, v in wts.items()}
    assert max(grad_errs.values()) < 5e-2, grad_errs
    assert worst_l < 2e-3 and worst_g < 3e-2, (worst_l, worst_g)
    # bf16 weights: 2^-9 relative rounding.  The biases are small vectors whose Adam steps (lr-sized whatever the gradient) flip
    # with bf16-level gradient differences: they drifted 1.4 % after six steps on an H100
    assert max(v for k, v in drift.items() if not k.endswith(".bias")) < 1e-2, drift
    assert max(v for k, v in drift.items() if k.endswith(".bias")) < 3e-2, drift


# ---------------------------------------------------------------------------------------------------------------------------
# a bias model through the layouts and paths of the trainer
# ---------------------------------------------------------------------------------------------------------------------------
def _run(mc, tc, batches, layout="keep", options=None):
    L, _, _, _ = _mods()
    for k, v in (options or {}).items():
        L.set_option(k, v)
    try:
        tr = L.Trainer(mc, dataclasses.replace(tc, recompute=layout))
        assert tr.recompute == layout
        assert tr.device_bytes == L.plan_device_bytes(mc, tc, 1, layout)
        tr.init_random_weights(1234)
        if not tc.full_finetune:
            tr.init_lora(4321)
        trace = [tr.step(ids, labels, lens)[:2] for ids, labels, lens in batches]
        out = tr.export_weights() if tc.full_finetune else tr.export_adapter()
        grads = tr.export_weights(grads=True) if tc.full_finetune else tr.export_adapter(grads=True)
        groups = tr.last_step_groups
        tr.close()
    finally:
        for k in (options or {}):
            L.set_option(k, 1)
    return trace, out, grads, groups


def _qwen_cfg(full=False, targets=("q_proj", "k_proj", "v_proj")):
    L, _, _, _ = _mods()
    mc = L.ModelConfig(vocab=2048, hidden=768, n_layers=3, n_heads=6, n_kv_heads=2, ffn=768, **QWEN2)
    tc = L.TrainConfig(micro_batch=2, seq_len=384, total_steps=8, lora_r=16, lora_dropout=0.0, lr=1e-3, full_finetune=full,
                       lora_target=targets, weight_decay=0.1)
    return mc, tc


def _batches(vocab, n, lens=None):
    _, O, _, _ = _mods()
    out = []
    for s in range(n):
        ids, labels = O.synthetic_batch(s, 0, 2, 384, vocab)
        ln = None
        if lens is not None:
            ln = np.array(lens, np.int32)
            for b in range(2):
                ids[b, ln[b]:] = 0
                labels[b, ln[b]:] = -100
        out.append((ids, labels, ln))
    return out


@pytest.mark.parametrize("full", [False, True])
def test_bias_model_keep_and_recompute_are_bitwise_equal(full):
    mc, tc = _qwen_cfg(full)
    batches = _batches(mc.vocab, 4)
    a, b = _run(mc, tc, batches, "keep"), _run(mc, tc, batches, "layer")
    assert a[0] == b[0]
    for k in a[1]:
        assert a[1][k].tobytes() == b[1][k].tobytes(), k
        assert a[2][k].tobytes() == b[2][k].tobytes(), k


@pytest.mark.parametrize("full", [False, True])
def test_bias_model_packed_ragged_matches_padded(full):
    """Rows of 384 and 200 tokens: packed (384 + 256 rows, per-row rotary positions in the bias epilogue) vs the padded rectangle."""
    mc, tc = _qwen_cfg(full)
    batches = _batches(mc.vocab, 3, lens=[384, 200])
    packed = _run(mc, tc, batches)
    padded = _run(mc, tc, batches, options={"varlen_pack": 0, "varlen_split": 0})
    assert packed[3] == 0 and padded[3] == 1
    for (l1, g1), (l2, g2) in zip(packed[0], padded[0]):
        assert abs(l1 - l2) / l2 < 2e-3 and abs(g1 - g2) / g2 < 3e-2, (packed[0], padded[0])
    _close(packed[2], padded[2], 5e-2)


def _close(a, b, tol):
    _, _, _, G = _mods()
    for k in a:
        x = G._bf16_bits_to_f32(a[k]) if a[k].dtype == np.uint16 else a[k]
        y = G._bf16_bits_to_f32(b[k]) if b[k].dtype == np.uint16 else b[k]
        e = float(np.linalg.norm(x - y) / max(np.linalg.norm(y), 1e-12))
        assert e < tol, (k, e)


@pytest.mark.parametrize("full", [False, True])
def test_bias_model_unfused_epilogues_match_fused(full):
    mc, tc = _qwen_cfg(full)
    batches = _batches(mc.vocab, 3)
    fused = _run(mc, tc, batches)
    unfused = _run(mc, tc, batches, options={"fused_epilogues": 0})
    for (l1, g1), (l2, g2) in zip(fused[0], unfused[0]):
        assert abs(l1 - l2) / l2 < 2e-3 and abs(g1 - g2) / g2 < 3e-2, (fused[0], unfused[0])
    # gradients of the same weights (first step): after three steps the two roundings have also moved the weights apart
    _close(_run(mc, tc, batches[:1])[2], _run(mc, tc, batches[:1], options={"fused_epilogues": 0})[2], 5e-2)


def test_bias_is_required_and_refused_without_qkv_bias():
    L, O, _, _ = _mods()
    mc, tc = _qwen_cfg()
    tr = L.Trainer(mc, tc)
    w = O.init_base_weights(O.OracleConfig(vocab=2048, hidden=768, n_layers=3, n_heads=6, n_kv_heads=2, ffn=768), 1)
    tr.load_state_dict({k: v.numpy() for k, v in w.items()})
    tr.init_lora(1)
    ids, labels = O.synthetic_batch(0, 0, 2, 384, mc.vocab)
    with pytest.raises(L.DtxError) as e:
        tr.step(ids, labels)
    assert e.value.code == -4 and "bias" in str(e.value)
    tr.close()
    plain = L.Trainer(dataclasses.replace(mc, qkv_bias=False), tc)
    with pytest.raises(L.DtxError) as e:
        plain.load_tensor("model.layers.0.self_attn.q_proj.bias", np.zeros(768, np.float32))
    assert e.value.code == -1
    plain.close()
