"""Qwen3 (q/k RMSNorm) and attention widths other than the hidden size on the GPU (-m gpu): the QK-norm epilogue of the GEMM, the
unfused qk_norm_fwd kernel and qk_norm_bwd, LoRA and full-parameter SFT traces against the Qwen3 oracle (tests/qwen3_oracle.py),
NF4, both activation layouts, packed ragged batches, the unfused epilogues, and one Qwen3-8B-shaped layer."""
import dataclasses
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
    from tests import qwen3_oracle as FO
    from tests import gpu_checks as G
    return L, O, FO, G


# ---------------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------------
def _norm_ref(x, q_cols, n_cols, wq, wk, eps=1e-6):
    """fp32 per-head RMSNorm of columns < n_cols of x [M, N] (x already bf16-rounded), weight wq below q_cols, wk beyond"""
    M = x.shape[0]
    h = x[:, :n_cols].float().reshape(M, n_cols // 128, 128)
    w = torch.stack([(wq if c < q_cols else wk).float() for c in range(0, n_cols, 128)])
    y = w[None] * (h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + eps))
    return torch.cat([y.reshape(M, n_cols), x[:, n_cols:].float()], dim=1)


def _gemm_qk_norm(A, B, q_cols, rope_cols, wq, wk, cs, S, A2=None, B2=None, rope_pos=None, eps=1e-6):
    L, _, _, G = _mods()
    M, K = A.shape
    N = B.shape[0]
    Cm = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=A.device)
    pre = torch.full((M, rope_cols), float("nan"), dtype=torch.bfloat16, device=A.device)
    rc = L.load().dtx_gemm_qk_norm(G.P(A), A.stride(0), G.P(B), B.stride(0), 0, G.P(A2), A2.stride(0) if A2 is not None else 0,
                                   G.P(B2), B2.stride(0) if B2 is not None else 0, A2.shape[1] if A2 is not None else 0, G.P(Cm), N,
                                   G.P(pre), rope_cols, G.P(cs), S, rope_cols, G.P(rope_pos), M, N, K, q_cols, G.P(wq), G.P(wk), eps,
                                   G.STREAM())
    torch.cuda.synchronize()
    return rc, Cm, pre


def _norm_w(seed):
    g = torch.Generator().manual_seed(seed)
    return (1.0 + torch.randn(128, generator=g) * 0.1).to(torch.bfloat16).to("cuda:0")


# (H, Hkv, N): "mixed" has 3 q heads and 1 k head, so the tile of columns 256..511 holds q head 2 and k head 0; the two
# columns tiles beyond rope_cols stand for v
SHAPES = {"gqa": (6, 2, 1280), "mixed": (3, 1, 768)}


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("pos", [False, True])
@pytest.mark.parametrize("kext", [False, True])
def test_gemm_qk_norm_epilogue(shape, pos, kext):
    """norm of the bf16-rounded projection, then the rotary, against fp32 torch; the pre-norm output is bitwise the EPI_BF16
    GEMM's; v columns are the plain rounded projection."""
    L, _, _, G = _mods()
    H, Hkv, N = SHAPES[shape]
    D, K = 128, 768
    q_cols, rope_cols = H * D, (H + Hkv) * D
    M = 640 if pos else 1000
    A, Bw = G._rand(M, K, seed=81), G._rand(N, K, scale=0.05, seed=82)
    A2, B2 = (G._rand(M, 64, seed=83), G._rand(N, 64, scale=0.05, seed=84)) if kext else (None, None)
    wq, wk = _norm_w(85), _norm_w(86)
    S = 384
    cs = G._rope_table(S)
    p = torch.arange(M, device=G.DEV) % S
    rope_pos = None
    if pos:  # packed ragged batch: sequences of 384 and 256 rows back to back
        p = torch.cat([torch.arange(384), torch.arange(256)]).to(G.DEV)
        rope_pos = p.to(torch.int32).contiguous()
    rc, got, pre = _gemm_qk_norm(A, Bw, q_cols, rope_cols, wq, wk, cs, S, A2, B2, rope_pos)
    assert rc == 0
    plain = G.gemm(A, Bw, A2=A2, B2=B2)  # EPI_BF16, 128 x 256 tiles: the same accumulator
    assert torch.equal(pre, plain[:, :rope_cols]), "the pre-norm q|k must be the plain GEMM's bits"
    from tests.test_model_families_gpu import _rope_ref_pos
    ref = _rope_ref_pos(_norm_ref(plain.float(), q_cols, rope_cols, wq, wk), p, H + Hkv)
    e = G.rel_err(got, ref)
    assert e < 6e-3, f"{shape} pos={pos} kext={kext} rel_err {e}"
    assert torch.equal(got[:, rope_cols:], plain[:, rope_cols:])
    # the weights matter: swapping q_norm and k_norm moves the result far beyond the tolerance
    _, swapped, _ = _gemm_qk_norm(A, Bw, q_cols, rope_cols, wk, wq, cs, S, A2, B2, rope_pos)
    assert G.rel_err(swapped, ref) > 5 * e


def test_gemm_qk_norm_refusals():
    L, _, _, G = _mods()
    A, Bw, wq = G._rand(512, 256, seed=1), G._rand(768, 256, seed=2), _norm_w(3)
    cs = G._rope_table(256)
    assert _gemm_qk_norm(A, Bw, 384, 512, wq, wq, cs, 256)[0] == 0
    assert _gemm_qk_norm(A, Bw, 320, 512, wq, wq, cs, 256)[0] == -1  # q / k boundary inside a head
    assert _gemm_qk_norm(A, Bw, 640, 512, wq, wq, cs, 256)[0] == -1  # q_cols beyond the rotated columns
    assert _gemm_qk_norm(A, Bw, 384, 384, wq, wq, cs, 256)[0] == -1  # rope_cols not whole 256-column tiles
    assert _gemm_qk_norm(A, Bw, 384, 512, wq, None, cs, 256)[0] == -1


def test_qk_norm_fwd_kernel_matches_reference():
    L, _, _, G = _mods()
    M, H, Hkv = 1000, 6, 2
    W, QK = (H + 2 * Hkv) * 128, (H + Hkv) * 128
    x = G._rand(M, W, scale=0.7, seed=91)
    wq, wk = _norm_w(92), _norm_w(93)
    y = x.clone()
    pre = torch.full((M, QK), float("nan"), dtype=torch.bfloat16, device=G.DEV)
    G.ok(L.load().dtx_qk_norm_fwd(G.P(y), W, M, H * 128, QK, G.P(wq), G.P(wk), 1e-6, G.P(pre), QK, G.STREAM()))
    torch.cuda.synchronize()
    assert torch.equal(pre, x[:, :QK])
    assert torch.equal(y[:, QK:], x[:, QK:])
    e = G.rel_err(y, _norm_ref(x.float(), H * 128, QK, wq, wk))
    assert e < 4e-3, e


@pytest.mark.parametrize("with_dw", [False, True])
def test_qk_norm_bwd_kernel_matches_autograd(with_dw):
    L, _, _, G = _mods()
    lib = L.load()
    M, H, Hkv = 1000, 6, 2
    W, QK, q_cols = (H + 2 * Hkv) * 128, (H + Hkv) * 128, H * 128
    x = G._rand(M, QK, scale=0.7, seed=101)
    dy = G._rand(M, W, scale=0.3, seed=102)
    wq, wk = _norm_w(103), _norm_w(104)
    xr = x.float().requires_grad_(True)
    wqr, wkr = wq.float().requires_grad_(True), wk.float().requires_grad_(True)
    h = xr.reshape(M, QK // 128, 128)
    w = torch.stack([wqr if c < q_cols else wkr for c in range(0, QK, 128)])
    y = w[None] * (h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + 1e-6))
    y.reshape(M, QK).backward(dy[:, :QK].float())
    nblk = 64
    scratch = torch.empty(nblk * 256, dtype=torch.float32, device=G.DEV)
    outs = []
    for _ in range(2):
        g = dy.clone()
        dw = torch.zeros(256, dtype=torch.bfloat16, device=G.DEV)
        G.ok(lib.dtx_qk_norm_bwd(G.P(g), W, G.P(x), QK, M, q_cols, QK, G.P(wq), G.P(wk), 1e-6, G.P(dw) if with_dw else None,
                                 G.P(scratch), nblk, 0, G.STREAM()))
        if with_dw:  # accumulate: twice the sum
            g2 = dy.clone()
            G.ok(lib.dtx_qk_norm_bwd(G.P(g2), W, G.P(x), QK, M, q_cols, QK, G.P(wq), G.P(wk), 1e-6, G.P(dw), G.P(scratch), nblk, 1,
                                     G.STREAM()))
        torch.cuda.synchronize()
        outs.append((g, dw))
    g, dw = outs[0]
    assert torch.equal(g[:, QK:], dy[:, QK:])
    e = G.rel_err(g[:, :QK], xr.grad)
    assert e < 4e-3, e
    if with_dw:
        assert torch.equal(outs[0][1], outs[1][1]), "dw must be bitwise repeatable"
        assert torch.equal(outs[0][0], outs[1][0])
        e = G.rel_err(dw, 2 * torch.cat([wqr.grad, wkr.grad]))
        assert e < 6e-3, e


# ---------------------------------------------------------------------------------------------------------------------------
# training against the Qwen3 oracle
# ---------------------------------------------------------------------------------------------------------------------------
QWEN3 = dict(rope_theta=1000000.0, rms_eps=1e-6, qk_norm=True)
DIMS = {
    "qwen3": dict(vocab=2048, hidden=768, n_layers=2, n_heads=6, n_kv_heads=2, ffn=768, **QWEN3),
    # hidden 512 with 6 heads x 128: the attention is wider than the residual stream (Qwen3-0.6B / 4B / 32B)
    "qwen3_decoupled": dict(vocab=2048, hidden=512, n_layers=2, n_heads=6, n_kv_heads=2, ffn=768, **QWEN3),
    # Mistral-Nemo: n_heads * head_dim = 4096 < hidden = 5120, no q/k norm
    "nemo": dict(vocab=2048, hidden=1024, n_layers=2, n_heads=6, n_kv_heads=2, ffn=768, rope_theta=1000000.0),
}


def _pair(family, targets=("q_proj", "v_proj"), steps=20, tied=False, full=False, S=256, B=2, quant=False, weight_decay=0.0):
    L, O, FO, _ = _mods()
    dims = DIMS[family]
    ocfg = FO.FamilyConfig(**dims, lora_r=16, lora_alpha=32.0, lr=1e-3, total_steps=steps, lora_dropout=0.0,
                           lora_target=tuple(targets), full_finetune=full, weight_decay=weight_decay)
    mc = L.ModelConfig(**dims)
    tc = L.TrainConfig(micro_batch=B, seq_len=S, total_steps=steps, lora_r=16, lora_alpha=32.0, lora_dropout=0.0, lr=1e-3,
                       lora_target=tuple(targets), full_finetune=full, weight_decay=weight_decay)
    w = FO.init_base_weights(ocfg, 1234, tied=tied)
    lora = {} if full else FO.init_lora(ocfg, 4321)
    tr = L.Trainer(mc, tc)
    tr.load_state_dict({k: v.numpy() for k, v in w.items()})
    if quant:
        tr.quantize_base("int4")
        w = O.quantize_base_nf4(w)
    tr.load_state_dict({k: v.numpy() for k, v in lora.items()})
    return ocfg, FO.FamilyTrainer(ocfg, w, lora), tr


@pytest.mark.parametrize("family,targets,tied", [
    ("qwen3", ("q_proj", "v_proj"), False),
    ("qwen3", ("q_proj", "k_proj", "v_proj"), True),
    ("qwen3_decoupled", ("q_proj", "v_proj"), False),
    ("qwen3_decoupled", ("q_proj", "k_proj", "v_proj"), True),
    ("nemo", ("q_proj", "k_proj", "v_proj"), False),
])
def test_lora_trace_matches_family_oracle(family, targets, tied):
    from tests.test_model_families_gpu import _lora_trace
    ocfg, orc, tr = _pair(family, targets, steps=20, tied=tied)
    _lora_trace(ocfg, orc, tr, 20)


def test_lora_nf4_qwen3_matches_oracle():
    from tests.test_model_families_gpu import _lora_trace
    ocfg, orc, tr = _pair("qwen3_decoupled", steps=20, quant=True)
    _lora_trace(ocfg, orc, tr, 20)


@pytest.mark.parametrize("family", ["qwen3", "qwen3_decoupled"])
def test_full_sft_qwen3_matches_oracle_with_norm_weights_and_grads(family):
    L, O, _, G = _mods()
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
            for k, v in got.items():
                r = orc.last_grads[k].numpy()
                grad_errs[k] = float(np.linalg.norm(G._bf16_bits_to_f32(v) - r) / max(np.linalg.norm(r), 1e-12))
        worst_l = max(worst_l, abs(loss - ref.loss) / ref.loss)
        worst_g = max(worst_g, abs(gn - ref.grad_norm) / ref.grad_norm)
    wts = tr.export_weights()
    tr.close()
    assert sum(k.endswith("_norm.weight") and "self_attn" in k for k in grad_errs) == 2 * ocfg.n_layers
    drift = {k: float(np.linalg.norm(G._bf16_bits_to_f32(v) - orc.lora[k].detach().numpy()) /
                      max(np.linalg.norm(orc.lora[k].detach().numpy()), 1e-12)) for k, v in wts.items()}
    assert max(grad_errs.values()) < 5e-2, grad_errs
    assert worst_l < 2e-3 and worst_g < 3e-2, (worst_l, worst_g)
    assert max(drift.values()) < 1e-2, drift


# ---------------------------------------------------------------------------------------------------------------------------
# a Qwen3 model through the layouts and paths of the trainer
# ---------------------------------------------------------------------------------------------------------------------------
def _qwen3_cfg(full=False):
    L, _, _, _ = _mods()
    mc = L.ModelConfig(vocab=2048, hidden=512, n_layers=3, n_heads=6, n_kv_heads=2, ffn=768, **QWEN3)
    tc = L.TrainConfig(micro_batch=2, seq_len=384, total_steps=8, lora_r=16, lora_dropout=0.0, lr=1e-3, full_finetune=full,
                       lora_target=("q_proj", "k_proj", "v_proj"), weight_decay=0.1)
    return mc, tc


@pytest.mark.parametrize("full", [False, True])
def test_qwen3_keep_and_recompute_are_bitwise_equal(full):
    from tests.test_model_families_gpu import _batches, _run
    mc, tc = _qwen3_cfg(full)
    batches = _batches(mc.vocab, 4)
    a, b = _run(mc, tc, batches, "keep"), _run(mc, tc, batches, "layer")
    assert a[0] == b[0]
    for k in a[1]:
        assert a[1][k].tobytes() == b[1][k].tobytes(), k
        assert a[2][k].tobytes() == b[2][k].tobytes(), k


@pytest.mark.parametrize("full", [False, True])
def test_qwen3_packed_ragged_matches_padded(full):
    from tests.test_model_families_gpu import _batches, _close, _run
    mc, tc = _qwen3_cfg(full)
    batches = _batches(mc.vocab, 3, lens=[384, 200])
    packed = _run(mc, tc, batches)
    padded = _run(mc, tc, batches, options={"varlen_pack": 0, "varlen_split": 0})
    assert packed[3] == 0 and padded[3] == 1
    for (l1, g1), (l2, g2) in zip(packed[0], padded[0]):
        assert abs(l1 - l2) / l2 < 2e-3 and abs(g1 - g2) / g2 < 3e-2, (packed[0], padded[0])
    _close(packed[2], padded[2], 5e-2)


@pytest.mark.parametrize("full", [False, True])
def test_qwen3_unfused_epilogues_match_fused(full):
    from tests.test_model_families_gpu import _batches, _close, _run
    mc, tc = _qwen3_cfg(full)
    batches = _batches(mc.vocab, 3)
    fused = _run(mc, tc, batches)
    unfused = _run(mc, tc, batches, options={"fused_epilogues": 0})
    for (l1, g1), (l2, g2) in zip(fused[0], unfused[0]):
        assert abs(l1 - l2) / l2 < 2e-3 and abs(g1 - g2) / g2 < 3e-2, (fused[0], unfused[0])
    _close(_run(mc, tc, batches[:1])[2], _run(mc, tc, batches[:1], options={"fused_epilogues": 0})[2], 5e-2)


def test_qk_norm_weights_are_required_and_refused_without_qk_norm():
    L, O, FO, _ = _mods()
    mc, tc = _qwen3_cfg()
    tr = L.Trainer(mc, tc)
    ocfg = FO.FamilyConfig(vocab=2048, hidden=512, n_layers=3, n_heads=6, n_kv_heads=2, ffn=768)
    w = FO.init_base_weights(ocfg, 1)  # no q_norm / k_norm
    tr.load_state_dict({k: v.numpy() for k, v in w.items()})
    tr.init_lora(1)
    ids, labels = O.synthetic_batch(0, 0, 2, 384, mc.vocab)
    with pytest.raises(L.DtxError) as e:
        tr.step(ids, labels)
    assert e.value.code == -4 and "q_norm" in str(e.value)
    tr.close()
    plain = L.Trainer(dataclasses.replace(mc, qk_norm=False), tc)
    with pytest.raises(L.DtxError) as e:
        plain.load_tensor("model.layers.0.self_attn.k_norm.weight", np.ones(128, np.float32))
    assert e.value.code == -1
    plain.close()


def test_layer_qwen3_8b_shape():
    """One Qwen3-8B-shaped layer (d = 4096, 32 / 8 heads, F = 12288: q|k|v N = 6144, dq + dkv = 5120) + lm_head through the
    trainer against the fp32 oracle: the QK-norm epilogue at real widths."""
    L, O, FO, _ = _mods()
    dims = dict(vocab=4096, hidden=4096, n_layers=1, n_heads=32, n_kv_heads=8, ffn=12288, **QWEN3)
    ocfg = FO.FamilyConfig(**dims, lora_r=16, lora_alpha=32.0, lr=1e-4, total_steps=10, lora_dropout=0.0)
    mc = L.ModelConfig(**dims)
    B, S = 2, 1024
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


def test_worker_trains_a_tiny_qwen3_checkpoint():
    """The worker end to end on a random-init Qwen3 directory (tied embeddings, 4 heads x 128 over hidden 256, q/k norms):
    config.json -> load_model_config -> native LoRA training -> PEFT adapter with lora_B of q_proj at the attention width."""
    import json
    import os
    import shlex
    import shutil
    import tempfile
    import importlib
    _, O, FO, _ = _mods()
    from datatunerx_b200.tuning import model_io, parser as TP
    tmp = tempfile.mkdtemp(prefix="dtx_qwen3_")
    try:
        mdir, store = os.path.join(tmp, "model"), os.path.join(tmp, "storage")
        os.makedirs(mdir)
        gold = os.path.join(os.path.dirname(__file__), "golden")
        shutil.copy(os.path.join(gold, "tiny_tokenizer.json"), os.path.join(mdir, "tokenizer.json"))
        json.dump({"tokenizer_class": "PreTrainedTokenizerFast", "bos_token": "<s>", "eos_token": "</s>", "unk_token": "<unk>"},
                  open(os.path.join(mdir, "tokenizer_config.json"), "w"))
        ocfg = FO.FamilyConfig(vocab=400, hidden=256, n_layers=2, n_heads=4, n_kv_heads=2, ffn=768, rms_eps=1e-6,
                               rope_theta=1000000.0, qk_norm=True)
        json.dump({"architectures": ["Qwen3ForCausalLM"], "model_type": "qwen3", "vocab_size": 400, "hidden_size": 256,
                   "intermediate_size": 768, "num_hidden_layers": 2, "num_attention_heads": 4, "num_key_value_heads": 2, "head_dim": 128,
                   "rms_norm_eps": 1e-6, "rope_theta": 1000000.0, "max_position_embeddings": 40960, "attention_bias": False,
                   "sliding_window": None, "use_sliding_window": False, "tie_word_embeddings": True},
                  open(os.path.join(mdir, "config.json"), "w"))
        w = {k: v.numpy() for k, v in FO.init_base_weights(ocfg, 7, tied=True).items() if k != "lm_head.weight"}
        model_io.write_safetensors(os.path.join(mdir, "model.safetensors"), w)
        csv_path = os.path.join(tmp, "train.csv")
        with open(csv_path, "w") as f:
            f.write("q,a\n")
            for i in range(48):
                f.write(f"What is {i} plus {i}?,The answer is {2 * i}.\n")
        ckpt_file = os.path.join(tmp, "checkpoint_path")
        os.environ["DTX_CHECKPOINT_PATH_FILE"] = ckpt_file
        from datatunerx_b200.tuning import train as TT
        importlib.reload(TT)
        entry = TP.controller_entrypoint(mdir, csv_path, validate_file=csv_path, columns='{"instruction":"q","response":"a"}',
                                         scheduler="linear", optimizer="adamw_hf", lora_r="16", lora_alpha="32", lora_dropout="0.0",
                                         learning_rate="1e-3", epochs=2, block_size=256, batch_size=4, grad_acc_steps=1,
                                         num_workers=1, storage_path=store, uid="qwen3")
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            rc = TT.main(shlex.split(entry)[2:])
        finally:
            os.chdir(cwd)
        assert rc == 0, f"worker exit status {rc}"
        ckpt = open(ckpt_file).read()
        ad = {k: np.array(a) for k, a, _ in model_io.iter_safetensors(os.path.join(ckpt, "adapter_model.safetensors"))}
        assert len(ad) == 8 and all(np.isfinite(v).all() for v in ad.values())
        qb = [v for k, v in ad.items() if "q_proj.lora_B" in k]
        assert qb and all(v.shape == (512, 16) for v in qb), {k: v.shape for k, v in ad.items()}
        assert any(np.abs(v).max() > 0 for k, v in ad.items() if "lora_B" in k), "B adapters must have moved"
        logs = [json.loads(line) for line in open(os.path.join(tmp, "result", "watch", "trainer_log.jsonl"))]
        assert logs[-1]["loss"] < logs[0]["loss"], logs
    finally:
        os.environ.pop("DTX_CHECKPOINT_PATH_FILE", None)
        shutil.rmtree(tmp, ignore_errors=True)
