"""GLM-4 (GlmForCausalLM, Glm4ForCausalLM) on the GPU (-m gpu): GLM's partial interleaved rotary in the q|k|v GEMM epilogue, in the
unfused kernel and in the attention backward, Glm4's post_norm_add kernel, LoRA and full-parameter SFT traces against the GLM oracle (tests/glm_oracle.py) with checkpoints
in GLM's layout (fused gate_up_proj), NF4, both activation layouts, packed ragged batches, the unfused epilogues, and one
GLM-4-9B-shaped layer."""
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
    from tests import glm_oracle as FO
    from tests import gpu_checks as G
    return L, O, FO, G


# ---------------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------------
def _glm_table(S, theta=10000.0):
    """[S][32] float2 (cos, sin) the way the trainer builds it: fp32 inverse frequencies and angles, cos / sin in double"""
    _, _, FO, G = _mods()
    inv = FO.inv_freq(FO.FamilyConfig(rope_theta=theta, rope_glm=True))
    ang = torch.arange(S, dtype=torch.float32)[:, None] * inv[None]
    return torch.stack([ang.double().cos(), ang.double().sin()], dim=-1).float().contiguous().to(G.DEV)


def _glm_ref(x, cs, pos, n_rot, inverse=False):
    """fp32 GLM rotary of the first n_rot 128-column heads of x [M, N] at per-row positions pos"""
    M = x.shape[0]
    c, s = cs[pos, :, 0], cs[pos, :, 1]
    if inverse:
        s = -s
    h = x[:, :n_rot * 128].reshape(M, n_rot, 128)
    x0, x1 = h[..., 0:64:2], h[..., 1:64:2]
    c, s = c[:, None, :], s[:, None, :]
    rot = torch.stack((x0 * c - x1 * s, x1 * c + x0 * s), dim=-1).flatten(-2)
    return torch.cat([torch.cat([rot, h[..., 64:]], dim=-1).reshape(M, -1), x[:, n_rot * 128:]], dim=1)


def _gemm_rope_glm(A, B, cs, S, rope_cols, A2=None, B2=None, rope_pos=None, bias=None):
    L, _, _, G = _mods()
    M, K = A.shape
    N = B.shape[0]
    Cm = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=A.device)
    rc = L.load().dtx_gemm_rope_glm(G.P(A), A.stride(0), G.P(B), B.stride(0), 0, G.P(A2), A2.stride(0) if A2 is not None else 0,
                                    G.P(B2), B2.stride(0) if B2 is not None else 0, A2.shape[1] if A2 is not None else 0, G.P(Cm), N,
                                    G.P(cs), S, rope_cols, G.P(rope_pos), M, N, K, G.P(bias), G.STREAM())
    torch.cuda.synchronize()
    return rc, Cm


def _plain(A, B, A2, B2, bias):
    """EPI_BF16 (+ bias) GEMM with the same 128 x 256 tiles: the accumulator the rotary epilogue starts from"""
    L, _, _, G = _mods()
    if bias is None:
        return G.gemm(A, B, A2=A2, B2=B2)
    M, K = A.shape
    N = B.shape[0]
    Cm = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=A.device)
    G.ok(L.load().dtx_gemm_bias(G.P(A), A.stride(0), G.P(B), B.stride(0), 0, G.P(A2), A2.stride(0) if A2 is not None else 0,
                                G.P(B2), B2.stride(0) if B2 is not None else 0, A2.shape[1] if A2 is not None else 0, G.P(Cm), N, None,
                                0, None, 0, 0, None, M, N, K, L.EPI_BF16, G.P(bias), G.STREAM()))
    torch.cuda.synchronize()
    return Cm


# (H, Hkv, N): "mixed" has 3 q heads and 1 k head, so the tile of columns 256..511 holds q head 2 and k head 0
SHAPES = {"gqa": (6, 2, 1280), "mixed": (3, 1, 768)}


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("kext", [False, True])
@pytest.mark.parametrize("pos", [False, True])
def test_gemm_rope_glm_epilogue(shape, bias, kext, pos):
    """GLM rotary of the (biased) fp32 accumulator against fp32 torch; columns 64..127 of every q / k head and every v column are
    bitwise the plain (bias) GEMM's output."""
    L, _, _, G = _mods()
    H, Hkv, N = SHAPES[shape]
    K, S = 768, 384
    rope_cols = (H + Hkv) * 128
    M = 640 if pos else 1000
    A, Bw = G._rand(M, K, seed=21), G._rand(N, K, scale=0.05, seed=22)
    A2, B2 = (G._rand(M, 64, seed=23), G._rand(N, 64, scale=0.05, seed=24)) if kext else (None, None)
    b = G._rand(N, scale=0.5, seed=25) if bias else None
    cs = _glm_table(S)
    p = torch.arange(M, device=G.DEV) % S
    rope_pos = None
    if pos:  # packed ragged batch: sequences of 384 and 256 rows back to back
        p = torch.cat([torch.arange(384), torch.arange(256)]).to(G.DEV)
        rope_pos = p.to(torch.int32).contiguous()
    rc, got = _gemm_rope_glm(A, Bw, cs, S, rope_cols, A2, B2, rope_pos, b)
    assert rc == 0
    acc = A.float() @ Bw.float().t() + (A2.float() @ B2.float().t() if kext else 0) + (b.float() if bias else 0)
    e = G.rel_err(got, _glm_ref(acc, cs, p, H + Hkv))
    assert e < 6e-3, f"{shape} bias={bias} kext={kext} pos={pos} rel_err {e}"
    plain = _plain(A, Bw, A2, B2, b)
    heads = got[:, :rope_cols].reshape(M, H + Hkv, 128)
    assert torch.equal(heads[..., 64:], plain[:, :rope_cols].reshape(M, H + Hkv, 128)[..., 64:])
    assert torch.equal(got[:, rope_cols:], plain[:, rope_cols:])
    assert not torch.equal(heads[..., :64], plain[:, :rope_cols].reshape(M, H + Hkv, 128)[..., :64])


def test_gemm_rope_glm_refusals():
    _, _, _, G = _mods()
    A, Bw = G._rand(512, 256, seed=1), G._rand(768, 256, seed=2)
    cs = _glm_table(256)
    assert _gemm_rope_glm(A, Bw, cs, 256, 512)[0] == 0
    assert _gemm_rope_glm(A, Bw, cs, 256, 384)[0] == -1  # rope_cols not whole 256-column tiles
    assert _gemm_rope_glm(A, Bw, None, 256, 512)[0] == -1  # no table


def test_rope_glm_kernel_and_round_trip():
    L, _, _, G = _mods()
    lib = L.load()
    B, S, H, Hkv = 2, 384, 6, 2
    W = (H + 2 * Hkv) * 128
    x = G._rand(B * S, W, seed=31)
    cs = _glm_table(S)
    p = torch.arange(B * S, device=G.DEV) % S
    y = x.clone()
    G.ok(lib.dtx_rope_glm_qk(G.P(y), G.P(cs), B, S, H, Hkv, 0, G.STREAM()))
    torch.cuda.synchronize()
    e = G.rel_err(y, _glm_ref(x.float(), cs, p, H + Hkv))
    assert e < 4e-3, e
    n = (H + Hkv) * 128
    assert torch.equal(y[:, n:], x[:, n:])
    assert torch.equal(y[:, :n].reshape(-1, H + Hkv, 128)[..., 64:], x[:, :n].reshape(-1, H + Hkv, 128)[..., 64:])
    z = y.clone()
    G.ok(lib.dtx_rope_glm_qk(G.P(z), G.P(cs), B, S, H, Hkv, 1, G.STREAM()))
    torch.cuda.synchronize()
    assert G.rel_err(z, x) < 8e-3  # two bf16 roundings away from the input


def test_attn_bwd_glm_inverse_rotary():
    """The GLM inverse rotary inside the dQ / dK store epilogues: gradients with respect to the PRE-rotary q, k of
    attention(glm_rope(q), glm_rope(k), v) against fp32 autograd, at GLM's 16:1 grouped-query ratio."""
    L, _, _, G = _mods()
    lib = L.load()
    B, S, H, Hkv, D = 2, 384, 16, 1, 128
    W = (H + 2 * Hkv) * D
    pre = G._rand(B * S, W, seed=41)
    cs = _glm_table(S)
    cs_t = cs.permute(1, 0, 2).contiguous()  # [32][S]
    p = torch.arange(B * S, device=G.DEV) % S
    rot = _glm_ref(pre.float(), cs, p, H + Hkv).to(torch.bfloat16)
    dout = G._rand(B * S, H * D, seed=42)
    out = torch.empty(B * S, H * D, dtype=torch.bfloat16, device=G.DEV)
    lse2 = torch.empty(B, H, S, dtype=torch.float32, device=G.DEV)
    delta = torch.empty(B, H, S, dtype=torch.float32, device=G.DEV)
    dqkv = torch.full((B * S, W), float("nan"), dtype=torch.bfloat16, device=G.DEV)
    sc = 1.0 / math.sqrt(D)
    G.ok(lib.dtx_attn_fwd(G.P(rot), G.P(out), G.P(lse2), B, S, H, Hkv, sc, None, 0, G.STREAM()))
    G.ok(lib.dtx_attn_bwd_rope(G.P(rot), G.P(out), G.P(dout), G.P(lse2), G.P(delta), G.P(dqkv), B, S, H, Hkv, sc, None, 0, G.P(cs_t), S,
                               1, G.STREAM()))
    torch.cuda.synchronize()
    x = pre.float().requires_grad_(True)
    ref, _ = G._attn_ref(_glm_ref(x, cs, p, H + Hkv), B, S, H, D, Hkv)
    ref.backward(dout.float())
    g = x.grad.view(B, S, H + 2 * Hkv, D)
    got = dqkv.float().view(B, S, H + 2 * Hkv, D)
    errs = {"dq": G.rel_err(got[:, :, :H], g[:, :, :H]), "dk": G.rel_err(got[:, :, H:H + Hkv], g[:, :, H:H + Hkv]),
            "dv": G.rel_err(got[:, :, H + Hkv:], g[:, :, H + Hkv:])}
    assert max(errs.values()) < 1e-2, errs
    # a sliding window has no GLM instantiation
    assert lib.dtx_attn_bwd_rope(G.P(rot), G.P(out), G.P(dout), G.P(lse2), G.P(delta), G.P(dqkv), B, S, H, Hkv, sc, None, 64, G.P(cs_t),
                                 S, 1, G.STREAM()) == -1


def test_post_norm_add_and_its_backward():
    """out = res + w * rmsnorm(y) in fp32 against torch; rmsnorm_bwd on y with dres = null is its gradient with respect to y;
    out = null writes rstd only, bitwise the same rstd."""
    L, _, _, G = _mods()
    lib = L.load()
    M, d, eps = 1000, 4096, 1e-5
    y, res, dy = G._rand(M, d, scale=0.7, seed=51), G._rand(M, d, seed=52), G._rand(M, d, scale=0.3, seed=53)
    w = (1.0 + G._rand(d, scale=0.1, seed=54).float()).to(torch.bfloat16)
    out = torch.full((M, d), float("nan"), dtype=torch.bfloat16, device=G.DEV)
    rstd, rstd2 = torch.empty(M, dtype=torch.float32, device=G.DEV), torch.empty(M, dtype=torch.float32, device=G.DEV)
    G.ok(lib.dtx_post_norm_add(G.P(y), G.P(w), G.P(res), G.P(out), G.P(rstd), M, d, eps, G.STREAM()))
    G.ok(lib.dtx_post_norm_add(G.P(y), None, None, None, G.P(rstd2), M, d, eps, G.STREAM()))
    dx = torch.empty_like(y)
    G.ok(lib.dtx_rmsnorm_bwd(G.P(dy), G.P(y), G.P(w), G.P(rstd), None, G.P(dx), M, d, G.STREAM()))
    torch.cuda.synchronize()
    yr = y.float().requires_grad_(True)
    norm = w.float() * (yr * torch.rsqrt(yr.pow(2).mean(-1, keepdim=True) + eps))
    (norm * dy.float()).sum().backward()
    assert G.rel_err(out, res.float() + norm.detach()) < 4e-3
    assert torch.equal(rstd, rstd2)
    assert G.rel_err(rstd, torch.rsqrt(y.float().pow(2).mean(-1) + eps)) < 1e-5
    assert G.rel_err(dx, yr.grad) < 4e-3


# ---------------------------------------------------------------------------------------------------------------------------
# training against the GLM oracle
# ---------------------------------------------------------------------------------------------------------------------------
GLM = dict(rope_theta=10000.0, rms_eps=1.5625e-07, qkv_bias=True, rope_glm=True)
DIMS = {
    "glm": dict(vocab=2048, hidden=768, n_layers=2, n_heads=6, n_kv_heads=2, ffn=768, **GLM),
    # GLM-4-9B's 16:1 ratio (32 q heads over 2 KV heads) with an attention width (4096) other than the hidden size
    "glm_gqa16": dict(vocab=2048, hidden=512, n_layers=2, n_heads=32, n_kv_heads=2, ffn=768, **GLM),
    # Glm4ForCausalLM: the same with post-sublayer norms
    "glm4": dict(vocab=2048, hidden=768, n_layers=2, n_heads=6, n_kv_heads=2, ffn=768, post_norms=True, **GLM),
}


def _pair(family, targets=("q_proj", "v_proj"), steps=20, full=False, S=256, B=2, quant=False, weight_decay=0.0):
    L, O, FO, _ = _mods()
    dims = DIMS[family]
    ocfg = FO.FamilyConfig(**dims, lora_r=16, lora_alpha=32.0, lr=1e-3, total_steps=steps, lora_dropout=0.0,
                           lora_target=tuple(targets), full_finetune=full, weight_decay=weight_decay)
    mc = L.ModelConfig(**dims)
    tc = L.TrainConfig(micro_batch=B, seq_len=S, total_steps=steps, lora_r=16, lora_alpha=32.0, lora_dropout=0.0, lr=1e-3,
                       lora_target=tuple(targets), full_finetune=full, weight_decay=weight_decay)
    w = FO.init_base_weights(ocfg, 1234)
    lora = {} if full else FO.init_lora(ocfg, 4321)
    tr = L.Trainer(mc, tc)
    tr.load_state_dict({k: v.numpy() for k, v in FO.to_hf(w).items()})  # the checkpoint's layout: fused gate_up_proj
    if quant:
        tr.quantize_base("int4")
        w = O.quantize_base_nf4(w)
    tr.load_state_dict({k: v.numpy() for k, v in lora.items()})
    return ocfg, FO.FamilyTrainer(ocfg, w, lora), tr


@pytest.mark.parametrize("family,targets", [
    ("glm", ("q_proj", "v_proj")),
    ("glm", ("q_proj", "k_proj", "v_proj")),
    ("glm_gqa16", ("q_proj", "v_proj")),
    ("glm4", ("q_proj", "v_proj")),
    ("glm4", ("q_proj", "k_proj", "v_proj")),
])
def test_lora_trace_matches_glm_oracle(family, targets):
    from tests.test_model_families_gpu import _lora_trace
    ocfg, orc, tr = _pair(family, targets, steps=20)
    _lora_trace(ocfg, orc, tr, 20)


@pytest.mark.parametrize("family", ["glm", "glm4"])
def test_lora_nf4_glm_matches_oracle(family):
    """NF4 of the GU-interleaved buffer equals NF4 of the HF gate_up_proj tensor: both quantise the same 64-element blocks; the
    post-sublayer norm weights stay bf16."""
    from tests.test_model_families_gpu import _lora_trace
    ocfg, orc, tr = _pair(family, steps=20, quant=True)
    _lora_trace(ocfg, orc, tr, 20)


@pytest.mark.parametrize("family", ["glm", "glm_gqa16", "glm4"])
def test_full_sft_glm_matches_oracle_with_fused_gate_up(family):
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
            want = FO.fuse_gate_up(orc.last_grads)
            assert set(got) == set(want)
            for k, v in got.items():
                r = want[k].numpy()
                assert v.shape == r.shape, k
                grad_errs[k] = float(np.linalg.norm(G._bf16_bits_to_f32(v) - r) / max(np.linalg.norm(r), 1e-12))
        worst_l = max(worst_l, abs(loss - ref.loss) / ref.loss)
        worst_g = max(worst_g, abs(gn - ref.grad_norm) / ref.grad_norm)
    wts = tr.export_weights()
    tr.close()
    want = {k: v.detach() for k, v in FO.fuse_gate_up(orc.lora).items()}
    assert sum("gate_up_proj" in k for k in wts) == ocfg.n_layers
    assert sum(k.endswith(("post_self_attn_layernorm.weight", "post_mlp_layernorm.weight")) for k in grad_errs) == \
        (2 * ocfg.n_layers if ocfg.post_norms else 0)
    drift = {k: float(np.linalg.norm(G._bf16_bits_to_f32(v) - want[k].numpy()) / max(np.linalg.norm(want[k].numpy()), 1e-12))
             for k, v in wts.items()}
    assert max(grad_errs.values()) < 5e-2, grad_errs
    assert worst_l < 2e-3 and worst_g < 3e-2, (worst_l, worst_g)
    # the biases drift further than the matrices, as in the Qwen2 full-SFT test of test_model_families_gpu.py (3 % bar there)
    assert max(v for k, v in drift.items() if not k.endswith(".bias")) < 1e-2, drift
    assert max(v for k, v in drift.items() if k.endswith(".bias")) < 3e-2, drift


# ---------------------------------------------------------------------------------------------------------------------------
# a GLM model through the layouts and paths of the trainer
# ---------------------------------------------------------------------------------------------------------------------------
def _glm_cfg(full=False, post_norms=False):
    L, _, _, _ = _mods()
    mc = L.ModelConfig(vocab=2048, hidden=512, n_layers=3, n_heads=6, n_kv_heads=2, ffn=768, post_norms=post_norms, **GLM)
    tc = L.TrainConfig(micro_batch=2, seq_len=384, total_steps=8, lora_r=16, lora_dropout=0.0, lr=1e-3, full_finetune=full,
                       lora_target=("q_proj", "k_proj", "v_proj"), weight_decay=0.1)
    return mc, tc


@pytest.mark.parametrize("post_norms", [False, True])
@pytest.mark.parametrize("full", [False, True])
def test_glm_keep_and_recompute_are_bitwise_equal(full, post_norms):
    from tests.test_model_families_gpu import _batches, _run
    mc, tc = _glm_cfg(full, post_norms)
    batches = _batches(mc.vocab, 4)
    a, b = _run(mc, tc, batches, "keep"), _run(mc, tc, batches, "layer")
    assert a[0] == b[0]
    for k in a[1]:
        assert a[1][k].tobytes() == b[1][k].tobytes(), k
        assert a[2][k].tobytes() == b[2][k].tobytes(), k


@pytest.mark.parametrize("post_norms", [False, True])
@pytest.mark.parametrize("full", [False, True])
def test_glm_packed_ragged_matches_padded(full, post_norms):
    from tests.test_model_families_gpu import _batches, _close, _run
    mc, tc = _glm_cfg(full, post_norms)
    batches = _batches(mc.vocab, 3, lens=[384, 200])
    packed = _run(mc, tc, batches)
    padded = _run(mc, tc, batches, options={"varlen_pack": 0, "varlen_split": 0})
    assert packed[3] == 0 and padded[3] == 1
    for (l1, g1), (l2, g2) in zip(packed[0], padded[0]):
        assert abs(l1 - l2) / l2 < 2e-3 and abs(g1 - g2) / g2 < 3e-2, (packed[0], padded[0])
    _close(packed[2], padded[2], 5e-2)


@pytest.mark.parametrize("post_norms", [False, True])
@pytest.mark.parametrize("full", [False, True])
def test_glm_unfused_epilogues_match_fused(full, post_norms):
    from tests.test_model_families_gpu import _batches, _close, _run
    mc, tc = _glm_cfg(full, post_norms)
    batches = _batches(mc.vocab, 3)
    fused = _run(mc, tc, batches)
    unfused = _run(mc, tc, batches, options={"fused_epilogues": 0})
    for (l1, g1), (l2, g2) in zip(fused[0], unfused[0]):
        assert abs(l1 - l2) / l2 < 2e-3 and abs(g1 - g2) / g2 < 3e-2, (fused[0], unfused[0])
    _close(_run(mc, tc, batches[:1])[2], _run(mc, tc, batches[:1], options={"fused_epilogues": 0})[2], 5e-2)


def test_layer_glm4_9b_shape():
    """One GLM-4-9B-shaped layer (d = 4096, 32 / 2 heads, F = 13696: q|k|v N = 4608, dq + dkv = 4352) + lm_head through the
    trainer against the fp32 oracle: the GLM epilogue and attention backward at real widths."""
    L, O, FO, _ = _mods()
    dims = dict(vocab=4096, hidden=4096, n_layers=1, n_heads=32, n_kv_heads=2, ffn=13696, **GLM)
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
    tr.load_state_dict({k: v.numpy() for k, v in FO.to_hf(w).items()})
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


def test_post_norm_weights_are_required_and_refused_without_post_norms():
    L, O, FO, _ = _mods()
    mc, tc = _glm_cfg(post_norms=True)
    tr = L.Trainer(mc, tc)
    ocfg = FO.FamilyConfig(vocab=2048, hidden=512, n_layers=3, n_heads=6, n_kv_heads=2, ffn=768, qkv_bias=True, rope_glm=True)
    w = FO.to_hf(FO.init_base_weights(ocfg, 1))  # no post-sublayer norms
    tr.load_state_dict({k: v.numpy() for k, v in w.items()})
    tr.init_lora(1)
    ids, labels = O.synthetic_batch(0, 0, 2, 384, mc.vocab)
    with pytest.raises(L.DtxError) as e:
        tr.step(ids, labels)
    assert e.value.code == -4 and "post_self_attn_layernorm" in str(e.value)
    tr.close()
    plain = L.Trainer(_glm_cfg()[0], tc)
    with pytest.raises(L.DtxError) as e:
        plain.load_tensor("model.layers.0.post_mlp_layernorm.weight", np.ones(512, np.float32))
    assert e.value.code == -1
    plain.close()


def test_gate_up_proj_loads_like_gate_and_up():
    """The fused tensor and the two separate ones fill the same GU-interleaved buffer: bitwise equal full-SFT exports."""
    L, _, FO, _ = _mods()
    mc, tc = _glm_cfg(full=True)
    w = FO.init_base_weights(FO.FamilyConfig(**{k: getattr(mc, k) for k in ("vocab", "hidden", "n_layers", "n_heads", "n_kv_heads",
                                                                               "ffn")}, qkv_bias=True, rope_glm=True), 5)
    outs = []
    for sd in (w, FO.to_hf(w)):
        tr = L.Trainer(mc, tc)
        tr.load_state_dict({k: v.numpy() for k, v in sd.items()})
        outs.append(tr.export_weights())
        tr.close()
    for k in outs[0]:
        assert outs[0][k].tobytes() == outs[1][k].tobytes(), k
