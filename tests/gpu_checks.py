"""Parity checks of the sm_90a kernels against plain torch fp32 references / the CPU oracle.

Each check is a plain function (returns a dict of error metrics, raises AssertionError on mismatch) so that it
can be driven both by pytest (tests/test_kernels_gpu.py, -m gpu) and by tools/gpu_diag.py, which runs every
check in its own subprocess with a timeout (a trapped kernel poisons the CUDA context of its process only).
All compute calls go through the C ABI (datatunerx_b200.lib -> libdtxtune.so).
"""
from __future__ import annotations

import ctypes as C
import math
import time

import numpy as np
import torch

from datatunerx_b200 import lib as L
from oracle import llama_lora as O

DEV = "cuda:0"


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def STREAM():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ok(code):
    L.check(code)


def rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm().clamp(min=1e-12))


def max_err(a, b) -> float:
    return float((a.float() - b.float()).abs().max())


def gemm(A, B, *, a_mn=False, b_mn=False, A2=None, B2=None, R=None, epi=L.EPI_BF16, split_k=1, block_n=0, M=None, N=None,
         K=None):
    lib = L.load()
    if M is None:
        M = A.shape[1] if a_mn else A.shape[0]
    if K is None:
        K = A.shape[0] if a_mn else A.shape[1]
    if N is None:
        N = B.shape[1] if b_mn else B.shape[0]
    K2 = 0
    if A2 is not None:
        K2 = A2.shape[0] if a_mn else A2.shape[1]
    out_dtype = torch.float32 if epi == L.EPI_F32 else torch.bfloat16
    shape = (split_k, M, N) if split_k > 1 else (M, N)
    Cm = torch.full(shape, float("nan"), dtype=out_dtype, device=A.device)
    ok(lib.dtx_gemm_bf16(P(A), A.stride(0), int(a_mn), P(B), B.stride(0), int(b_mn), P(A2), A2.stride(0) if A2 is not None else 0,
                         P(B2), B2.stride(0) if B2 is not None else 0, K2, P(Cm), N, P(R), R.stride(0) if R is not None else 0,
                         M, N, K, epi, split_k, block_n, STREAM()))
    torch.cuda.synchronize()
    return Cm


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).to(DEV)


def check_gemm_nt(M=256, N=512, K=320, block_n=0):
    A, B = _rand(M, K, seed=1), _rand(N, K, seed=2)
    ref = A.float() @ B.float().t()
    out = gemm(A, B, block_n=block_n)
    e = rel_err(out, ref)
    assert e < 6e-3, f"NT bf16 rel_err {e}"
    out32 = gemm(A, B, epi=L.EPI_F32, block_n=block_n)
    e32 = rel_err(out32, ref)
    assert e32 < 1e-5, f"NT f32 rel_err {e32}"
    R = _rand(M, N, seed=3)
    outr = gemm(A, B, R=R, epi=L.EPI_BF16_ADD, block_n=block_n)
    er = rel_err(outr, ref + R.float())
    assert er < 6e-3, f"NT +residual rel_err {er}"
    return {"bf16": e, "f32": e32, "add": er}


def check_gemm_nn(M=256, N=384, K=448, block_n=0):
    A, B = _rand(M, K, seed=4), _rand(K, N, seed=5)
    ref = A.float() @ B.float()
    out32 = gemm(A, B, b_mn=True, epi=L.EPI_F32, block_n=block_n)
    e = rel_err(out32, ref)
    assert e < 1e-5, f"NN f32 rel_err {e}"
    return {"f32": e}


def check_gemm_tn(Mp=384, N=64, K=1024, split_k=4):
    A, B = _rand(K, Mp, seed=6), _rand(K, N, seed=7)  # C[Mp,N] = A^T B
    ref = A.float().t() @ B.float()
    parts = gemm(A, B, a_mn=True, b_mn=True, epi=L.EPI_F32, split_k=split_k, block_n=64)
    out = parts.sum(0) if split_k > 1 else parts
    e = rel_err(out, ref)
    assert e < 1e-5, f"TN split-K rel_err {e}"
    return {"f32": e}


def check_gemm_tn_pair(Mp=1000, N=768, K=2048):
    """Weight-gradient shape through the 128 x 256-tile kernel with BOTH operands MN-major: C[Mp, N] = A^T B (A [K, Mp], B [K, N]),
    plain and accumulating (EPI_BF16_ADD in place), ragged Mp; bitwise equal to the 128 x 128-tile kernel."""
    A, B = _rand(K, Mp, seed=36), _rand(K, N, seed=37)
    ref = A.float().t() @ B.float()
    out = gemm(A, B, a_mn=True, b_mn=True)
    e = rel_err(out, ref)
    assert e < 6e-3, f"TN pair rel_err {e}"
    R = _rand(Mp, N, seed=38)
    acc = R.clone()
    lib = L.load()
    ok(lib.dtx_gemm_bf16(P(A), A.stride(0), 1, P(B), B.stride(0), 1, None, 0, None, 0, 0, P(acc), N, P(acc), N, Mp, N, K, L.EPI_BF16_ADD, 1, 0, STREAM()))
    torch.cuda.synchronize()
    e_acc = rel_err(acc, ref + R.float())
    assert e_acc < 6e-3, f"TN pair accumulate rel_err {e_acc}"
    L.set_option("gemm_pair_kernel", 0)
    try:
        single = gemm(A, B, a_mn=True, b_mn=True)
    finally:
        L.set_option("gemm_pair_kernel", 1)
    assert torch.equal(out, single), "pair and single-CTA kernels must agree bitwise"
    return {"bf16": e, "accumulate": e_acc}


def check_gemm_kext():
    M, N, K, K2 = 256, 768, 256, 64
    A, B, A2, B2 = _rand(M, K, seed=8), _rand(N, K, seed=9), _rand(M, K2, seed=10), _rand(N, K2, seed=11)
    ref = A.float() @ B.float().t() + A2.float() @ B2.float().t()
    e1 = rel_err(gemm(A, B, A2=A2, B2=B2, epi=L.EPI_F32), ref)
    assert e1 < 1e-5, f"NT k-ext rel_err {e1}"
    Bn, B2n = _rand(K, N, seed=12), _rand(K2, N, seed=13)
    ref2 = A.float() @ Bn.float() + A2.float() @ B2n.float()
    e2 = rel_err(gemm(A, Bn, b_mn=True, A2=A2, B2=B2n, epi=L.EPI_F32), ref2)
    assert e2 < 1e-5, f"NN k-ext rel_err {e2}"
    return {"nt": e1, "nn": e2}


def check_gemm_ragged():
    out = {}
    for (M, N, K) in [(200, 200, 200), (130, 72, 136), (128, 2048, 64), (1000, 264, 520)]:
        A, B = _rand(M, K, seed=M), _rand(N, K, seed=N + 1)
        ref = A.float() @ B.float().t()
        e = rel_err(gemm(A, B, epi=L.EPI_F32), ref)
        assert e < 1e-5, f"ragged {M}x{N}x{K} rel_err {e}"
        Bn = _rand(K, N, seed=K + 2)
        e2 = rel_err(gemm(A, Bn, b_mn=True, epi=L.EPI_F32), A.float() @ Bn.float())
        assert e2 < 1e-5, f"ragged NN {M}x{N}x{K} rel_err {e2}"
        out[f"{M}x{N}x{K}"] = max(e, e2)
    return out


def check_gemm_large(M=4096, N=4096, K=4096, iters=10):
    A, B = _rand(M, K, scale=0.05, seed=20), _rand(N, K, scale=0.05, seed=21)
    out = gemm(A, B)
    ref = (A @ B.t()).float()  # cuBLAS bf16 as the large-shape reference
    e = rel_err(out, ref)
    assert e < 1e-2, f"large NT rel_err {e}"
    lib = L.load()
    Cm = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        ok(lib.dtx_gemm_bf16(P(A), K, 0, P(B), K, 0, None, 0, None, 0, 0, P(Cm), N, None, 0, M, N, K, 0, 1, 0, STREAM()))
    s.record()
    for _ in range(iters):
        ok(lib.dtx_gemm_bf16(P(A), K, 0, P(B), K, 0, None, 0, None, 0, 0, P(Cm), N, None, 0, M, N, K, 0, 1, 0, STREAM()))
    t.record()
    torch.cuda.synchronize()
    ms = s.elapsed_time(t) / iters
    s.record()
    for _ in range(iters):
        torch.matmul(A, B.t())
    t.record()
    torch.cuda.synchronize()
    ms_ref = s.elapsed_time(t) / iters
    return {"rel_err": e, "ms": ms, "tflops": 2.0 * M * N * K / ms / 1e9, "cublas_ms": ms_ref,
            "cublas_tflops": 2.0 * M * N * K / ms_ref / 1e9}


def check_rmsnorm(M=300, d=4096):
    lib = L.load()
    x, w, dy, dres = _rand(M, d, seed=1), (_rand(d, seed=2) * 0.1 + 1).to(torch.bfloat16), _rand(M, d, seed=3), _rand(M, d, seed=4)
    y = torch.empty_like(x)
    rstd = torch.empty(M, dtype=torch.float32, device=DEV)
    ok(lib.dtx_rmsnorm_fwd(P(x), P(w), P(y), P(rstd), M, d, 1e-5, STREAM()))
    xf = x.float().requires_grad_(True)
    ref = O.rmsnorm(xf, w.float(), 1e-5)
    ref.backward(dy.float())
    e_f = rel_err(y, ref)
    assert e_f < 4e-3, f"rmsnorm fwd {e_f}"
    dx = torch.empty_like(x)
    ok(lib.dtx_rmsnorm_bwd(P(dy), P(x), P(w), P(rstd), P(dres), P(dx), M, d, STREAM()))
    torch.cuda.synchronize()
    e_b = rel_err(dx, xf.grad + dres.float())
    assert e_b < 4e-3, f"rmsnorm bwd {e_b}"
    return {"fwd": e_f, "bwd": e_b}


def check_rope(B=2, S=256, H=2, D=128):
    lib = L.load()
    qkv = _rand(B * S, 3 * H * D, seed=5)
    orig = qkv.clone()
    cs = torch.empty(S, D // 2, 2, dtype=torch.float32, device=DEV)
    ok(lib.dtx_rope_table(P(cs), S, D, 10000.0, STREAM()))
    ok(lib.dtx_rope_qk(P(qkv), P(cs), B, S, H, H, D, 0, STREAM()))
    torch.cuda.synchronize()
    cos, sin = O.rope_cos_sin(S, D, 10000.0)
    cos, sin = cos.to(DEV), sin.to(DEV)
    x = orig.float().view(B, S, 3, H, D)
    refq = O.apply_rope(x[:, :, 0].transpose(1, 2), cos, sin).transpose(1, 2)
    refk = O.apply_rope(x[:, :, 1].transpose(1, 2), cos, sin).transpose(1, 2)
    got = qkv.float().view(B, S, 3, H, D)
    e = max(rel_err(got[:, :, 0], refq), rel_err(got[:, :, 1], refk))
    assert e < 4e-3, f"rope {e}"
    assert torch.equal(got[:, :, 2], x[:, :, 2]), "rope must not touch v"
    ok(lib.dtx_rope_qk(P(qkv), P(cs), B, S, H, H, D, 1, STREAM()))
    torch.cuda.synchronize()
    e_inv = rel_err(qkv, orig)
    assert e_inv < 8e-3, f"rope inverse round trip {e_inv}"
    return {"fwd": e, "roundtrip": e_inv}


def check_swiglu(M=257, F=768):
    lib = L.load()
    gu, dact = _rand(M, 2 * F, seed=6), _rand(M, F, seed=7)
    act = torch.empty(M, F, dtype=torch.bfloat16, device=DEV)
    dgu = torch.empty_like(gu)
    ok(lib.dtx_swiglu_fwd(P(gu), P(act), M, F, STREAM()))
    ok(lib.dtx_swiglu_bwd(P(dact), P(gu), P(dgu), M, F, STREAM()))
    torch.cuda.synchronize()
    g = gu.float().requires_grad_(True)
    ref = torch.nn.functional.silu(g[:, :F]) * g[:, F:]
    ref.backward(dact.float())
    e_f, e_b = rel_err(act, ref), rel_err(dgu, g.grad)
    assert e_f < 4e-3 and e_b < 4e-3, (e_f, e_b)
    return {"fwd": e_f, "bwd": e_b}


def check_lora_dropout(M=300, d=256, nt=2, p=0.1):
    """Counter-based dropout masks: the device kernels and the oracle's numpy restatement agree element for element."""
    lib = L.load()
    key = O.dropout_key(42, 5, 3, 0)
    h = _rand(M, d, seed=21)
    hd = torch.empty(M, nt * d, dtype=torch.bfloat16, device=DEV)
    ok(lib.dtx_lora_dropout_fwd(P(h), P(hd), M, d, nt, p, C.c_uint64(key), STREAM()))
    g = _rand(M, nt * d, seed=22)
    dh0 = _rand(M, d, seed=23)
    dh = dh0.clone()
    ok(lib.dtx_lora_dropout_bwd_add(P(dh), P(g), M, d, nt, p, C.c_uint64(key), STREAM()))
    torch.cuda.synchronize()
    ref_add = torch.zeros(M, d, device=DEV)
    for ti in range(nt):
        mask = O.dropout_mask(key, ti, M, d, p).to(DEV)
        got = hd[:, ti * d:(ti + 1) * d].float()
        assert torch.equal(got != 0, (mask != 0) & (h.float() != 0)), f"keep pattern of target {ti} differs from the oracle"
        assert rel_err(got, h.float() * mask / (1 - p)) < 4e-3
        ref_add += g[:, ti * d:(ti + 1) * d].float() * mask / (1 - p)
    e = rel_err(dh, dh0.float() + ref_add)
    assert e < 4e-3, f"dropout backward {e}"
    return {"keep_rate": float((hd != 0).float().mean()), "bwd": e}


def check_nf4(n=64 * 5000):
    """NF4 block quantise-dequantise on the device == the oracle's restatement of bitsandbytes' algorithm, bit for bit."""
    lib = L.load()
    w = _rand(n, scale=0.02, seed=31)
    w[64:128] = 0  # an all-zero block
    ref = O.nf4_roundtrip(w.float().cpu().view(-1, 64)).view(-1)
    got = w.clone()
    ok(lib.dtx_nf4_roundtrip(P(got), n, STREAM()))
    torch.cuda.synchronize()
    assert torch.equal(got.float().cpu(), ref), f"nf4 mismatch: {int((got.float().cpu() != ref).sum())} of {n}"
    return {"distinct_levels": int(torch.unique((got.float() / got.float().view(-1, 64).abs().amax(1, keepdim=True).clamp(min=1e-30)).view(-1)).numel()),
            "rel_quant_err": rel_err(got, w)}


def check_trainer_qlora(steps=6):
    """--quantization int4: native trainer on PACKED NF4 base weights == oracle trained on nf4_roundtrip'ed weights; the packed
    base is 0.5625 / 2 of the bf16 one; int8 is refused loudly.  The last two steps are ragged and run as two length groups
    (the NF4 expansion / prefetch state carries across the groups' forward+backward passes)."""
    ocfg, mc, tc = tiny_configs(S=512, steps=steps)
    w, lora = O.init_base_weights(ocfg, 1234), O.init_lora(ocfg, 4321)
    tr = L.Trainer(mc, tc)
    tr.load_state_dict({k: v.numpy() for k, v in w.items()})
    bytes_bf16 = tr.base_weight_bytes
    try:
        tr.quantize_base("int8")
        raise AssertionError("int8 must be refused")
    except L.DtxError as e:
        assert e.code == -5, e
    tr.quantize_base("int4")
    bytes_nf4 = tr.base_weight_bytes
    lin = sum(v.numel() for k, v in w.items() if k.endswith(O.QUANTIZED_SUFFIXES))
    assert bytes_bf16 - bytes_nf4 == lin * 2 - (lin // 2 + lin // 64 * 4), (bytes_bf16, bytes_nf4, lin)
    tr.load_state_dict({k: v.numpy() for k, v in lora.items()})
    orc = O.OracleTrainer(ocfg, O.quantize_base_nf4(w), lora)
    worst_l = worst_g = 0.0
    groups = []
    for s_ in range(steps):
        ids, labels = O.synthetic_batch(s_, 0, tc.micro_batch, tc.seq_len, ocfg.vocab)
        lens = None
        if s_ >= steps - 2:
            lens = np.array([512, 100 + 30 * s_], dtype=np.int32)
            ids[1, lens[1]:] = 0
            labels[1, lens[1]:] = -100
            L.set_option("varlen_split", 2)
        ref = orc.step([(ids, labels)])
        try:
            loss, gn, _, _ = tr.step(ids, labels, lens)
        finally:
            L.set_option("varlen_split", 1)
        groups.append(tr.last_step_groups)
        worst_l, worst_g = max(worst_l, abs(loss - ref.loss) / ref.loss), max(worst_g, abs(gn - ref.grad_norm) / ref.grad_norm)
    tr.close()
    assert groups[-2:] == [2, 2] and groups[0] == 1, groups
    plain = O.OracleTrainer(ocfg, w, lora).step([O.synthetic_batch(0, 0, tc.micro_batch, tc.seq_len, ocfg.vocab)]).loss
    assert worst_l < 1e-3 and worst_g < 3e-2, (worst_l, worst_g)
    return {"loss": worst_l, "gnorm": worst_g, "loss_shift_vs_unquantized": abs(plain - ref.loss), "base_bytes_bf16": bytes_bf16,
            "base_bytes_nf4": bytes_nf4}


def check_embedding(M=500, d=256, V=1000):
    lib = L.load()
    table = _rand(V, d, seed=8)
    ids = torch.randint(0, V, (M,), dtype=torch.int32, device=DEV)
    out = torch.empty(M, d, dtype=torch.bfloat16, device=DEV)
    ok(lib.dtx_embedding_fwd(P(ids), P(table), P(out), M, d, V, STREAM()))
    torch.cuda.synchronize()
    assert torch.equal(out, table[ids.long()]), "embedding gather must be bit-exact"
    return {"exact": True}


def check_cross_entropy(B=3, S=128, V=2051):
    lib = L.load()
    M = B * S
    Vp = (V + 3) // 4 * 4
    logits = torch.randn(M, Vp, device=DEV) * 3
    labels = torch.randint(0, V, (B, S), dtype=torch.int32, device=DEV)
    labels[:, :20] = -100
    shifted = torch.empty(M, dtype=torch.int32, device=DEV)
    nvalid = torch.zeros(4, dtype=torch.int32, device=DEV)
    row_loss = torch.empty(M, dtype=torch.float32, device=DEV)
    dl = torch.empty(M, Vp, dtype=torch.bfloat16, device=DEV)
    loss = torch.zeros(4, dtype=torch.float32, device=DEV)
    ok(lib.dtx_cross_entropy(P(logits), Vp, P(labels), P(shifted), P(nvalid), P(row_loss), P(dl), Vp, P(loss), B, S, V, STREAM()))
    torch.cuda.synchronize()
    lg = logits[:, :V].view(B, S, V).clone().requires_grad_(True)
    ref = O.causal_lm_loss(lg, labels.long())
    ref.backward()
    e_l = abs(float(loss[0]) - float(ref)) / float(ref)
    assert e_l < 1e-5, f"CE loss {e_l}"
    e_g = rel_err(dl[:, :V].view(B, S, V), lg.grad)
    assert e_g < 4e-3, f"CE dlogits {e_g}"
    assert int(nvalid[0]) == int((labels[:, 1:] >= 0).sum())
    return {"loss": e_l, "dlogits": e_g}


def check_adamw(n=100003 * 4):
    lib = L.load()
    g0 = torch.Generator().manual_seed(0)
    p, m, v = torch.randn(n, generator=g0), torch.zeros(n), torch.zeros(n)
    pd, md, vd = p.to(DEV), m.to(DEV), v.to(DEV)
    sumsq = torch.zeros(4, device=DEV)
    scratch = torch.zeros(1024, device=DEV)
    gn = torch.zeros(4, device=DEV)
    out = {}
    for step in range(1, 4):
        g = torch.randn(n, generator=g0) * (0.5 if step == 2 else 1e-3)
        gd = g.to(DEV)
        ok(lib.dtx_sumsq(P(gd), n, P(scratch), P(sumsq), STREAM()))
        ok(lib.dtx_adamw(P(pd), P(gd), P(md), P(vd), n, 3e-4, 0.9, 0.999, 1e-8, 0.01, step, 0.5, P(sumsq), 1.0, P(gn), STREAM()))
        torch.cuda.synchronize()
        gs = g * 0.5
        norm = float(gs.double().norm())
        coef = O.clip_coef(norm, 1.0)
        O.adamw_update(p, gs * coef, m, v, step, 3e-4, 0.9, 0.999, 1e-8, 0.01)
        assert abs(float(gn[0]) - norm) / norm < 1e-5, (float(gn[0]), norm)
        e = max_err(pd.cpu(), p)
        assert e < 1e-6, f"adamw step {step} max err {e}"
        out[f"step{step}"] = e
    return out


def _attn_ref(qkv, B, S, H, D, Hkv=None, window=0):
    Hkv = Hkv or H
    x = qkv.float().view(B, S, H + 2 * Hkv, D)
    q = x[:, :, :H].transpose(1, 2)
    k = x[:, :, H:H + Hkv].transpose(1, 2).repeat_interleave(H // Hkv, dim=1)
    v = x[:, :, H + Hkv:].transpose(1, 2).repeat_interleave(H // Hkv, dim=1)
    scores = q @ k.transpose(-1, -2) / math.sqrt(D)
    mask = torch.full((S, S), float("-inf"), device=qkv.device).triu(1)
    if window > 0:  # query i sees keys i - window .. i
        mask = mask + torch.full((S, S), float("-inf"), device=qkv.device).tril(-(window + 1))
    p = torch.softmax(scores + mask, dim=-1)
    return (p @ v).transpose(1, 2).reshape(B * S, H * D), torch.logsumexp(scores + mask, dim=-1)


def _growing_scores_qkv(B, S, H, Hkv, D):
    """q.k grows by ~16 (log2 units) per 64 keys: every KV block moves the softmax reference (lazy-rescale path)."""
    g = torch.Generator(device="cpu").manual_seed(5)
    u = torch.ones(D) / math.sqrt(D)
    x = torch.randn(B, S, H + 2 * Hkv, D, generator=g) * 0.1
    pos = torch.arange(S, dtype=torch.float32).view(1, S, 1, 1)
    x[:, :, :H] += 4.0 * u
    x[:, :, H:H + Hkv] += 0.5 * pos * u
    return x.reshape(B * S, (H + 2 * Hkv) * D).to(torch.bfloat16).to(DEV)


def check_attn_fwd(B=2, S=256, H=2, Hkv=None, growing=False):
    lib = L.load()
    D = 128
    Hkv = Hkv or H
    qkv = _growing_scores_qkv(B, S, H, Hkv, D) if growing else _rand(B * S, (H + 2 * Hkv) * D, seed=11)
    out = torch.full((B * S, H * D), float("nan"), dtype=torch.bfloat16, device=DEV)
    lse2 = torch.empty(B, H, S, dtype=torch.float32, device=DEV)
    ok(lib.dtx_attn_fwd(P(qkv), P(out), P(lse2), B, S, H, Hkv, 1.0 / math.sqrt(D), None, 0, STREAM()))
    torch.cuda.synchronize()
    ref, lse = _attn_ref(qkv, B, S, H, D, Hkv)
    e = rel_err(out, ref)
    e_l = max_err(lse2 * math.log(2.0), lse)
    assert e < 8e-3, f"attn fwd {e}"
    assert e_l < 2e-3, f"attn lse {e_l}"
    return {"out": e, "lse": e_l}


def check_attn_fwd_exp_fma():
    """Forward softmax with part of the exponentials on the FMA pipe (cubic polynomial, rel. error 7.5e-5): same parity bar."""
    out = {}
    try:
        for every in (2, 3, 4):
            L.set_option("attn_fwd_exp_fma_every", every)
            out[f"every{every}"] = {"s384": check_attn_fwd(B=2, S=384, H=4, Hkv=2), "rescale": check_attn_fwd(B=1, S=1024, H=2, growing=True)}
    finally:
        L.set_option("attn_fwd_exp_fma_every", 0)
    return out


def check_attn_bwd(B=2, S=256, H=2, Hkv=None):
    lib = L.load()
    D = 128
    Hkv = Hkv or H
    qkv = _rand(B * S, (H + 2 * Hkv) * D, seed=12)
    dout = _rand(B * S, H * D, seed=13)
    out = torch.empty(B * S, H * D, dtype=torch.bfloat16, device=DEV)
    lse2 = torch.empty(B, H, S, dtype=torch.float32, device=DEV)
    delta = torch.empty(B, H, S, dtype=torch.float32, device=DEV)
    dqkv = torch.full((B * S, (H + 2 * Hkv) * D), float("nan"), dtype=torch.bfloat16, device=DEV)
    sc = 1.0 / math.sqrt(D)
    ok(lib.dtx_attn_fwd(P(qkv), P(out), P(lse2), B, S, H, Hkv, sc, None, 0, STREAM()))
    ok(lib.dtx_attn_bwd(P(qkv), P(out), P(dout), P(lse2), P(delta), P(dqkv), B, S, H, Hkv, sc, None, 0, None, 0, STREAM()))
    torch.cuda.synchronize()
    x = qkv.float().requires_grad_(True)
    ref, _ = _attn_ref(x, B, S, H, D, Hkv)
    ref.backward(dout.float())
    g = x.grad.view(B, S, H + 2 * Hkv, D)
    got = dqkv.float().view(B, S, H + 2 * Hkv, D)
    sl = {"dq": slice(0, H), "dk": slice(H, H + Hkv), "dv": slice(H + Hkv, H + 2 * Hkv)}
    errs = {n: rel_err(got[:, :, s_], g[:, :, s_]) for n, s_ in sl.items()}
    for n, e in errs.items():
        assert e < 1.5e-2, f"attn bwd {n} {e}"
    return errs


def check_nf4_pack(n=64 * 4096):
    """Packed NF4 storage: codes and absmax equal the oracle's restatement of bitsandbytes quantize_4bit (first element of a
    pair in the high nibble), and pack -> dequant is bit-identical to the one-kernel round trip and to the oracle."""
    lib = L.load()
    w = _rand(n, scale=0.02, seed=33)
    w[128:192] = 0
    packed = torch.empty(n // 2, dtype=torch.uint8, device=DEV)
    absmax = torch.empty(n // 64, dtype=torch.float32, device=DEV)
    out = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    ok(lib.dtx_nf4_pack(P(w), P(packed), P(absmax), n, STREAM()))
    ok(lib.dtx_nf4_dequant(P(packed), P(absmax), P(out), n, STREAM()))
    rt = w.clone()
    ok(lib.dtx_nf4_roundtrip(P(rt), n, STREAM()))
    torch.cuda.synchronize()
    x = w.float().cpu().numpy().reshape(-1, 64)
    amax = np.abs(x).max(axis=1, keepdims=True).astype(np.float32)
    inv = np.where(amax > 0, np.float32(1.0) / np.where(amax > 0, amax, 1), 0).astype(np.float32)
    mids = (np.float32(0.5) * (O.NF4_LEVELS[:-1] + O.NF4_LEVELS[1:])).astype(np.float32)
    code = (((x * inv)[..., None] > mids).sum(-1)).astype(np.uint8).reshape(-1)
    ref_bytes = (code[0::2] << 4) | code[1::2]
    assert np.array_equal(packed.cpu().numpy(), ref_bytes), "packed NF4 codes differ from the oracle"
    assert np.array_equal(absmax.cpu().numpy(), amax.reshape(-1)), "absmax differs"
    ref = O.nf4_roundtrip(w.float().cpu().view(-1, 64)).view(-1)
    assert torch.equal(out.float().cpu(), ref) and torch.equal(rt, out), "dequantised values differ"
    return {"bytes_per_weight": (packed.numel() + absmax.numel() * 4) / n}


def _rope_table(S, D=128):
    lib = L.load()
    cs = torch.empty(S, D // 2, 2, dtype=torch.float32, device=DEV)
    ok(lib.dtx_rope_table(P(cs), S, D, 10000.0, STREAM()))
    return cs


def _rope_ref(x, S, n_rot_heads, D=128):
    """x: [M, W] fp32 packed heads; rotary (HF rotate_half) on the first n_rot_heads heads, position = row % S."""
    M, W = x.shape
    cos, sin = O.rope_cos_sin(S, D, 10000.0)
    cos, sin = cos.to(x.device), sin.to(x.device)
    pos = torch.arange(M, device=x.device) % S
    h = x[:, : n_rot_heads * D].reshape(M, n_rot_heads, D)
    rot = h * cos[pos][:, None, :] + O.rotate_half(h) * sin[pos][:, None, :]
    return torch.cat([rot.reshape(M, -1), x[:, n_rot_heads * D:]], dim=1)


def gemm_fused(A, B, epi, *, b_mn=False, A2=None, B2=None, C_cols=None, aux=None, ld_aux=0, rope_cs=None, rope_S=0, rope_cols=0, N=None):
    lib = L.load()
    M, K = A.shape
    if N is None:
        N = B.shape[1] if b_mn else B.shape[0]
    K2 = A2.shape[1] if A2 is not None else 0
    Cm = torch.full((M, C_cols or N), float("nan"), dtype=torch.bfloat16, device=A.device)
    ok(lib.dtx_gemm_fused(P(A), A.stride(0), P(B), B.stride(0), int(b_mn), P(A2), A2.stride(0) if A2 is not None else 0, P(B2),
                          B2.stride(0) if B2 is not None else 0, K2, P(Cm), Cm.stride(0), P(aux), ld_aux, P(rope_cs), rope_S, rope_cols,
                          M, N, K, epi, STREAM()))
    torch.cuda.synchronize()
    return Cm


def check_gemm_rope_epilogue(S=640, B=3, H=16, Hkv=4, K=1024, ragged=True):
    """EPI_ROPE as the qkv projection runs it: wide N (many 256-column tiles, two heads per tile), LoRA K-extension, ragged M,
    GQA widths (rope on q and k heads only, v untouched)."""
    D = 128
    M = B * S - (37 if ragged else 0)
    W = (H + 2 * Hkv) * D
    A, Bw = _rand(M, K, seed=41), _rand(W, K, scale=0.05, seed=42)
    A2, B2 = _rand(M, 64, seed=43), _rand(W, 64, scale=0.05, seed=44)
    cs = _rope_table(S)
    got = gemm_fused(A, Bw, L.EPI_ROPE, A2=A2, B2=B2, rope_cs=cs, rope_S=S, rope_cols=(H + Hkv) * D)
    acc = A.float() @ Bw.float().t() + A2.float() @ B2.float().t()
    ref = _rope_ref(acc, S, H + Hkv)
    e = rel_err(got, ref)
    e_v = rel_err(got[:, (H + Hkv) * D:], acc[:, (H + Hkv) * D:])
    assert e < 6e-3 and e_v < 6e-3, f"EPI_ROPE rel_err {e} (v part {e_v})"
    worst_tile = max(rel_err(got[:, c:c + 256], ref[:, c:c + 256]) for c in range(0, W, 256))
    assert worst_tile < 8e-3, f"EPI_ROPE worst 256-column tile {worst_tile}"
    return {"rel_err": e, "worst_tile": worst_tile, "shape": [M, W, K]}


def _interleave_gu(wg, wu):
    """[F, d] gate and up weights -> the trainer's GU-interleaved [2F, d] layout (128 gate rows | 128 up rows per 128 features)."""
    F, d = wg.shape
    return torch.stack([wg.view(F // 128, 128, d), wu.view(F // 128, 128, d)], dim=1).reshape(2 * F, d).contiguous()


def _deinterleave_cols(x, F):
    """[M, 2F] interleaved columns -> (gate [M, F], up [M, F])."""
    M = x.shape[0]
    v = x.reshape(M, F // 128, 2, 128)
    return v[:, :, 0].reshape(M, F), v[:, :, 1].reshape(M, F)


def check_gemm_swiglu_epilogues(M=1500, d=1024, F=11008):
    """EPI_SWIGLU_FWD / EPI_SWIGLU_BWD at the 7B feature width (86 column tiles) with ragged M, against fp32 torch."""
    A = _rand(M, d, seed=51)
    wg, wu = _rand(F, d, scale=0.04, seed=52), _rand(F, d, scale=0.04, seed=53)
    wgu = _interleave_gu(wg, wu)
    act = torch.full((M, F), float("nan"), dtype=torch.bfloat16, device=DEV)
    gu = gemm_fused(A, wgu, L.EPI_SWIGLU_FWD, aux=act, ld_aux=F)
    g_ref, u_ref = A.float() @ wg.float().t(), A.float() @ wu.float().t()
    g_got, u_got = _deinterleave_cols(gu, F)
    e_g, e_u = rel_err(g_got, g_ref), rel_err(u_got, u_ref)
    act_ref = torch.nn.functional.silu(g_ref) * u_ref
    e_a = rel_err(act, act_ref)
    assert max(e_g, e_u) < 6e-3 and e_a < 8e-3, f"EPI_SWIGLU_FWD gate {e_g} up {e_u} act {e_a}"
    # backward: acc = dx * Wdown (Wdown [d, F] row-major = MN-major B), saved gu -> d(gate|up)
    dx = _rand(M, d, seed=54)
    wdown = _rand(d, F, scale=0.04, seed=55)
    dgu = gemm_fused(dx, wdown, L.EPI_SWIGLU_BWD, b_mn=True, C_cols=2 * F, aux=gu, ld_aux=2 * F, N=F)
    dact = (dx.float() @ wdown.float()).to(torch.bfloat16).float()  # the kernel rounds d(act) to bf16 like the unfused path
    g = g_got.float().requires_grad_(True)
    u = u_got.float().requires_grad_(True)
    (torch.nn.functional.silu(g) * u).backward(dact)
    dg_got, du_got = _deinterleave_cols(dgu, F)
    e_dg, e_du = rel_err(dg_got, g.grad), rel_err(du_got, u.grad)
    assert max(e_dg, e_du) < 8e-3, f"EPI_SWIGLU_BWD dgate {e_dg} dup {e_du}"
    worst_tile = max(rel_err(dg_got[:, c:c + 128], g.grad[:, c:c + 128]) for c in range(0, F, 128))
    assert worst_tile < 1.2e-2, f"EPI_SWIGLU_BWD worst tile {worst_tile}"
    return {"gate": e_g, "up": e_u, "act": e_a, "dgate": e_dg, "dup": e_du, "worst_tile": worst_tile}


def _attn_ref_heads(qkv, B, S, H, Hkv, q_heads, D=128, seq_lens=None):
    """fp32 reference on a subset of query heads (and the kv heads they read): returns out [B, S, len(q_heads), D]."""
    x = qkv.float().view(B, S, H + 2 * Hkv, D)
    g = H // Hkv
    outs = []
    mask = torch.full((S, S), float("-inf"), device=qkv.device).triu(1)
    for h in q_heads:
        q, k, v = x[:, :, h], x[:, :, H + h // g], x[:, :, H + Hkv + h // g]
        sc = torch.einsum("bqd,bkd->bqk", q, k) / math.sqrt(D) + mask
        outs.append(torch.softmax(sc, dim=-1) @ v)
    return torch.stack(outs, dim=2)


def check_attn_bench_shape(B=1, S=2048, H=32, Hkv=32, kv_heads=(0, 13, 31)):
    """Attention forward AND backward at the benchmarked geometry (S=2048 H=32; S=4096 H=32/Hkv=8 for the Mistral shape): the
    kernels run on all heads, the fp32 torch reference on the query heads of a few kv heads (full score matrices do not fit
    otherwise).  The backward reference differentiates through those heads only, so dO is zero elsewhere."""
    lib = L.load()
    D, g = 128, H // Hkv
    W = (H + 2 * Hkv) * D
    qkv = _rand(B * S, W, seed=61)
    q_heads = [kh * g + i for kh in kv_heads for i in range(g)]
    dout = torch.zeros(B * S, H * D, dtype=torch.bfloat16, device=DEV)
    dsub = _rand(B * S, len(q_heads) * D, seed=62)
    for i, h in enumerate(q_heads):
        dout[:, h * D:(h + 1) * D] = dsub[:, i * D:(i + 1) * D]
    out = torch.full((B * S, H * D), float("nan"), dtype=torch.bfloat16, device=DEV)
    lse2 = torch.empty(B, H, S, dtype=torch.float32, device=DEV)
    delta = torch.empty(B, H, S, dtype=torch.float32, device=DEV)
    dqkv = torch.full((B * S, W), float("nan"), dtype=torch.bfloat16, device=DEV)
    sc = 1.0 / math.sqrt(D)
    ok(lib.dtx_attn_fwd(P(qkv), P(out), P(lse2), B, S, H, Hkv, sc, None, 0, STREAM()))
    ok(lib.dtx_attn_bwd(P(qkv), P(out), P(dout), P(lse2), P(delta), P(dqkv), B, S, H, Hkv, sc, None, 0, None, 0, STREAM()))
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all() and torch.isfinite(dqkv.float()).all()
    x = qkv.float().requires_grad_(True)
    ref = _attn_ref_heads(x, B, S, H, Hkv, q_heads)
    ref.backward(dsub.float().view(B, S, len(q_heads), D))
    got = out.float().view(B, S, H, D)[:, :, q_heads]
    e_o = rel_err(got, ref)
    assert e_o < 8e-3, f"attention forward at S={S} H={H}/{Hkv}: {e_o}"
    gr = x.grad.view(B, S, H + 2 * Hkv, D)
    gg = dqkv.float().view(B, S, H + 2 * Hkv, D)
    k_idx = [H + kh for kh in kv_heads]
    v_idx = [H + Hkv + kh for kh in kv_heads]
    errs = {"out": e_o, "dq": rel_err(gg[:, :, q_heads], gr[:, :, q_heads]), "dk": rel_err(gg[:, :, k_idx], gr[:, :, k_idx]),
            "dv": rel_err(gg[:, :, v_idx], gr[:, :, v_idx])}
    for n_, e in errs.items():
        assert e < 1.5e-2, f"attention at S={S} H={H}/{Hkv}: {n_} {e}"
    # heads that received no dO have exactly zero dq; kv heads none of whose query heads did have exactly zero dk / dv
    others = [h for h in range(H) if h not in q_heads][:4]
    assert float(gg[:, :, others].abs().max()) == 0.0
    return errs


def check_attn_bwd_rope(B=2, S=384, H=4, Hkv=2):
    """The inverse rotary inside the dQ / dK store epilogues (what the fused training step runs): gradients with respect to the
    PRE-rotary q, k of  attention(rope(q), rope(k), v)  against fp32 autograd."""
    lib = L.load()
    D = 128
    W = (H + 2 * Hkv) * D
    pre = _rand(B * S, W, seed=71)
    cs = _rope_table(S)
    cs_t = cs.permute(1, 0, 2).contiguous()  # [64][S] (cos, sin): the transposed table the backward kernels read
    rot = _rope_ref(pre.float(), S, H + Hkv).to(torch.bfloat16)
    dout = _rand(B * S, H * D, seed=72)
    out = torch.empty(B * S, H * D, dtype=torch.bfloat16, device=DEV)
    lse2 = torch.empty(B, H, S, dtype=torch.float32, device=DEV)
    delta = torch.empty(B, H, S, dtype=torch.float32, device=DEV)
    dqkv = torch.full((B * S, W), float("nan"), dtype=torch.bfloat16, device=DEV)
    sc = 1.0 / math.sqrt(D)
    ok(lib.dtx_attn_fwd(P(rot), P(out), P(lse2), B, S, H, Hkv, sc, None, 0, STREAM()))
    ok(lib.dtx_attn_bwd(P(rot), P(out), P(dout), P(lse2), P(delta), P(dqkv), B, S, H, Hkv, sc, None, 0, P(cs_t), S, STREAM()))
    torch.cuda.synchronize()
    x = pre.float().requires_grad_(True)
    ref, _ = _attn_ref(_rope_ref(x, S, H + Hkv), B, S, H, D, Hkv)
    ref.backward(dout.float())
    g = x.grad.view(B, S, H + 2 * Hkv, D)
    got = dqkv.float().view(B, S, H + 2 * Hkv, D)
    errs = {"dq": rel_err(got[:, :, :H], g[:, :, :H]), "dk": rel_err(got[:, :, H:H + Hkv], g[:, :, H:H + Hkv]),
            "dv": rel_err(got[:, :, H + Hkv:], g[:, :, H + Hkv:])}
    for n_, e in errs.items():
        assert e < 1.5e-2, f"attention backward with fused inverse rotary: {n_} {e}"
    return errs


def check_attn_window(B=2, S=768, H=4, Hkv=2, windows=(1, 63, 64, 200, 511, 5000)):
    """Sliding-window attention (Mistral): forward, lse and all three gradients against fp32 torch for windows smaller than a
    block, block-aligned, straddling several blocks, and wider than the sequence (= plain causal)."""
    lib = L.load()
    D = 128
    W = (H + 2 * Hkv) * D
    qkv = _rand(B * S, W, seed=91)
    dout = _rand(B * S, H * D, seed=92)
    sc = 1.0 / math.sqrt(D)
    res = {}
    for win in windows:
        out = torch.full((B * S, H * D), float("nan"), dtype=torch.bfloat16, device=DEV)
        lse2 = torch.empty(B, H, S, dtype=torch.float32, device=DEV)
        delta = torch.empty(B, H, S, dtype=torch.float32, device=DEV)
        dqkv = torch.full((B * S, W), float("nan"), dtype=torch.bfloat16, device=DEV)
        ok(lib.dtx_attn_fwd(P(qkv), P(out), P(lse2), B, S, H, Hkv, sc, None, win, STREAM()))
        ok(lib.dtx_attn_bwd(P(qkv), P(out), P(dout), P(lse2), P(delta), P(dqkv), B, S, H, Hkv, sc, None, win, None, 0, STREAM()))
        torch.cuda.synchronize()
        x = qkv.float().requires_grad_(True)
        ref, lse = _attn_ref(x, B, S, H, D, Hkv, window=win)
        ref.backward(dout.float())
        e_o, e_l, e_g = rel_err(out, ref), max_err(lse2 * math.log(2.0), lse.detach()), rel_err(dqkv, x.grad)
        assert torch.isfinite(out.float()).all() and torch.isfinite(dqkv.float()).all(), f"window {win}: non-finite"
        assert e_o < 8e-3 and e_l < 2e-3 and e_g < 1.5e-2, f"window {win}: out {e_o} lse {e_l} grad {e_g}"
        res[f"w{win}"] = {"out": e_o, "lse": e_l, "grad": e_g}
    return res


def check_trainer_window(steps=4):
    """Mistral-style model whose sliding_window is shorter than the sequence: native step == oracle (4.34.0 mask width)."""
    ocfg, mc, tc = tiny_configs(S=512, B=2, steps=steps, heads=4, kv_heads=2)
    ocfg.sliding_window = 150
    mc.sliding_window = 150
    w, lora = O.init_base_weights(ocfg, 1234), O.init_lora(ocfg, 4321)
    tr = L.Trainer(mc, tc)
    tr.load_state_dict({k: v.numpy() for k, v in w.items()})
    tr.load_state_dict({k: v.numpy() for k, v in lora.items()})
    orc = O.OracleTrainer(ocfg, w, lora)
    plain = O.OracleTrainer(O.OracleConfig(**{**ocfg.__dict__, "sliding_window": 0}), w, lora)
    worst_l = worst_g = 0.0
    modes = []
    for s_ in range(steps):
        ids, labels = O.synthetic_batch(s_, 0, tc.micro_batch, tc.seq_len, ocfg.vocab)
        lens = None
        if s_ >= steps - 2:  # ragged rows (the second one shorter than / around twice the window): packed, windows inside every sequence
            lens = np.array([512, 140 + 200 * (s_ - (steps - 2))], dtype=np.int32)
            ids[1, lens[1]:] = 0
            labels[1, lens[1]:] = -100
        ref = orc.step([(ids, labels)])
        loss, gn, _, _ = tr.step(ids, labels, lens)
        modes.append(tr.last_step_groups)
        worst_l, worst_g = max(worst_l, abs(loss - ref.loss) / ref.loss), max(worst_g, abs(gn - ref.grad_norm) / ref.grad_norm)
    assert modes[-2:] == [0, 0] and modes[0] == 1, modes
    ids, labels = O.synthetic_batch(0, 0, tc.micro_batch, tc.seq_len, ocfg.vocab)
    shift = abs(plain.eval_loss(ids, labels) - O.OracleTrainer(ocfg, w, lora).eval_loss(ids, labels))
    tr.close()
    assert worst_l < 1e-3 and worst_g < 3e-2, (worst_l, worst_g)
    assert shift > 1e-5, "the window must change the loss at this length"
    return {"loss": worst_l, "gnorm": worst_g, "loss_shift_vs_causal": shift}


def check_attn_varlen(B=4, S=640, H=4, Hkv=2, lens=(640, 1, 129, 300)):
    """Row lengths: rows are right-padded beyond seq_lens[b].  Outputs / gradients of the real tokens equal the reference run on
    the truncated rows; tiles that lie entirely in the padding come back as exact zeros; nothing is NaN."""
    lib = L.load()
    D = 128
    W = (H + 2 * Hkv) * D
    qkv = _rand(B * S, W, seed=81)
    dout = _rand(B * S, H * D, seed=82).view(B, S, H * D)
    for b, n_ in enumerate(lens):
        dout[b, n_:] = 0  # the loss never reaches a padded token
    dout = dout.reshape(B * S, H * D).contiguous()
    sl = torch.tensor(lens, dtype=torch.int32, device=DEV)
    out = torch.full((B * S, H * D), float("nan"), dtype=torch.bfloat16, device=DEV)
    lse2 = torch.full((B, H, S), float("nan"), dtype=torch.float32, device=DEV)
    delta = torch.full((B, H, S), float("nan"), dtype=torch.float32, device=DEV)
    dqkv = torch.full((B * S, W), float("nan"), dtype=torch.bfloat16, device=DEV)
    sc = 1.0 / math.sqrt(D)
    ok(lib.dtx_attn_fwd(P(qkv), P(out), P(lse2), B, S, H, Hkv, sc, P(sl), 0, STREAM()))
    ok(lib.dtx_attn_bwd(P(qkv), P(out), P(dout), P(lse2), P(delta), P(dqkv), B, S, H, Hkv, sc, P(sl), 0, None, 0, STREAM()))
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all() and torch.isfinite(dqkv.float()).all(), "padding must stay finite"
    x = qkv.float().requires_grad_(True)
    ref, _ = _attn_ref(x, B, S, H, D, Hkv)
    ref.backward(dout.float())
    o3, r3 = out.float().view(B, S, -1), ref.view(B, S, -1)
    g3, rg3 = dqkv.float().view(B, S, -1), x.grad.view(B, S, -1)
    worst_o = worst_g = 0.0
    for b, n_ in enumerate(lens):
        worst_o = max(worst_o, rel_err(o3[b, :n_], r3[b, :n_]))
        worst_g = max(worst_g, rel_err(g3[b, :n_], rg3[b, :n_]))
        t0 = (n_ + 127) // 128 * 128  # first tile that holds only padding
        assert float(o3[b, t0:].abs().max() if t0 < S else 0.0) == 0.0, f"row {b}: skipped output tiles must be zero"
        assert float(g3[b, t0:].abs().max() if t0 < S else 0.0) == 0.0, f"row {b}: skipped gradient tiles must be zero"
        assert float(g3[b, n_:t0].abs().max() if n_ < t0 else 0.0) == 0.0, f"row {b}: padded rows inside a live tile have zero gradient"
    assert worst_o < 8e-3 and worst_g < 1.5e-2, (worst_o, worst_g)
    return {"out": worst_o, "grad": worst_g}


def check_trainer_varlen(steps=4):
    """dtx_step with per-batch padded length + true row lengths == the oracle on the same (right-padded, -100-labelled) rows:
    loss, grad-norm and every adapter gradient; and == the same batch padded to the static length without row lengths."""
    ocfg, orc, tr = make_tiny_pair(S=512, B=4, steps=steps)
    worst_l = worst_g = worst_grad = 0.0
    rng = np.random.default_rng(7)
    for s_ in range(steps):
        ids, labels = O.synthetic_batch(s_, 0, 4, 512, ocfg.vocab)
        lens = np.array([[384, 130, 7, 257], [512, 1, 128, 129], [100, 100, 100, 100], [256, 384, 64, 0]][s_ % 4], dtype=np.int32)
        cur = max(128, int(-(-int(lens.max()) // 128) * 128))
        for b in range(4):
            ids[b, lens[b]:] = 0
            labels[b, lens[b]:] = -100
            if lens[b] > 0:
                labels[b, :max(1, lens[b] // 3)] = -100
        ref = orc.step([(ids[:, :cur], labels[:, :cur])])
        loss, gn, _, stepped = tr.step(ids[:, :cur], labels[:, :cur], lens)
        assert stepped
        # default execution of a ragged LoRA micro-batch: PACKED (sequences back to back at 128-rounded lengths, one pass) whenever
        # that saves rows; 0 = packed, 1 = one pass at the padded shape
        saves = int(sum(max(128, -(-int(l) // 128) * 128) for l in lens)) < 4 * cur
        assert tr.last_step_groups == (0 if saves else 1), (lens, tr.last_step_groups)
        if s_ == 0:  # forward-only evaluation of the same ragged batch, packed vs one pass at the padded shape: per-row statistics
            s_pk, c_pk = tr.eval_rows(ids[:, :cur], labels[:, :cur], lens)
            L.set_option("varlen_split", 0)
            s_one, c_one = tr.eval_rows(ids[:, :cur], labels[:, :cur], lens)
            L.set_option("varlen_split", 1)
            assert c_pk.tolist() == c_one.tolist() and float(np.max(np.abs(s_pk - s_one) / np.maximum(np.abs(s_one), 1e-6))) < 2e-3, (s_pk, s_one, c_pk, c_one)
        worst_l, worst_g = max(worst_l, abs(loss - ref.loss) / ref.loss), max(worst_g, abs(gn - ref.grad_norm) / ref.grad_norm)
    # gradient tensors of one more step against the oracle's autograd gradients, from adapters with a sizeable B (B = 0 at init
    # makes dA vanish; after a few Adam steps it is ~1e-3 and the comparison would measure bf16 noise on tiny numbers)
    gen = torch.Generator().manual_seed(5)
    fresh = {k: (torch.randn(v.shape, generator=gen) * 0.02 if "lora_B" in k else v.detach().clone()) for k, v in orc.lora.items()}
    tr.load_state_dict({k: v.numpy() for k, v in fresh.items()})
    with torch.no_grad():
        for k, v in fresh.items():
            orc.lora[k].copy_(v)
    ids, labels = O.synthetic_batch(99, 0, 4, 512, ocfg.vocab)
    lens = np.array([300, 5, 200, 129], dtype=np.int32)
    for b in range(4):
        ids[b, lens[b]:] = 0
        labels[b, lens[b]:] = -100
    _, g_ref = orc.loss_and_grads(ids[:, :384], labels[:, :384])
    tr.step(ids[:, :384], labels[:, :384], lens)
    got = tr.export_adapter(grads=True)
    per = {}
    for k, v in got.items():
        r = g_ref[k.replace("base_model.model.", "")].numpy()
        per[k.split("layers.")[1]] = float(np.linalg.norm(v - r) / max(np.linalg.norm(r), 1e-12))
    worst_grad = max(per.values())
    tr.close()
    assert worst_l < 1e-3 and worst_g < 3e-2 and worst_grad < 4e-2, (worst_l, worst_g, per)
    return {"loss": worst_l, "gnorm": worst_g, "adapter_grads": per}


def check_trainer_varlen_groups():
    """A ragged micro-batch run as LENGTH GROUPS (rows sorted by length, each group padded to its own longest row, gradients
    accumulated, every group's loss divided by the labelled tokens of the whole micro-batch) == the oracle on the batch as a
    whole: loss, grad-norm, adapter gradients - with gradient accumulation over two ragged micro-batches, through both the
    host-buffer and the device-pointer entry points.  "varlen_split" = 2 forces the cut wherever 128-rounded lengths differ
    (the cost model would not split a model this small)."""
    ocfg, mc, tc = tiny_configs(S=512, B=4, steps=6)
    ocfg.grad_accum = 2
    tc.grad_accum = 2
    w, lora = O.init_base_weights(ocfg, 1234), O.init_lora(ocfg, 4321)
    gen = torch.Generator().manual_seed(5)
    lora = {k: (torch.randn(v.shape, generator=gen) * 0.02 if "lora_B" in k else v) for k, v in lora.items()}
    orc = O.OracleTrainer(ocfg, w, lora)
    L.set_option("varlen_split", 2)
    try:
        tr = L.Trainer(mc, tc)
        tr.load_state_dict({k: v.numpy() for k, v in w.items()})
        tr.load_state_dict({k: v.numpy() for k, v in lora.items()})
        patterns = [[384, 130, 7, 257], [512, 1, 128, 129], [100, 100, 100, 100], [256, 384, 64, 0], [500, 20, 300, 300], [129, 128, 127, 1]]
        worst_l = worst_g = 0.0
        groups = []

        def ragged(step, lens):
            ids, labels = O.synthetic_batch(step, 0, 4, 512, ocfg.vocab)
            cur = max(128, int(-(-int(max(lens)) // 128) * 128))
            for b in range(4):
                ids[b, lens[b]:] = 0
                labels[b, lens[b]:] = -100
                if lens[b] > 0:
                    labels[b, :max(1, lens[b] // 3)] = -100
            return np.ascontiguousarray(ids[:, :cur]), np.ascontiguousarray(labels[:, :cur]), np.array(lens, dtype=np.int32)

        # forward-only evaluation of a ragged batch: per-row statistics come back in the caller's row order whatever the grouping
        e_ids, e_lab, e_len = ragged(77, patterns[0])
        s_grp, c_grp = tr.eval_rows(e_ids, e_lab, e_len)
        l_grp = tr.eval_loss(e_ids, e_lab, e_len)
        L.set_option("varlen_split", 0)
        s_one, c_one = tr.eval_rows(e_ids, e_lab, e_len)
        l_one = tr.eval_loss(e_ids, e_lab, e_len)
        L.set_option("varlen_split", 2)
        assert c_grp.tolist() == c_one.tolist() == [int((e_lab[b, 1:] >= 0).sum()) for b in range(4)], (c_grp, c_one)
        eval_rel = float(np.max(np.abs(s_grp - s_one) / np.maximum(np.abs(s_one), 1e-6)))
        assert eval_rel < 2e-3 and abs(l_grp - l_one) < 1e-4 * l_one and abs(l_grp - orc.eval_loss(e_ids, e_lab)) < 1e-3 * l_one, (s_grp, s_one, l_grp, l_one)
        for it in range(3):
            mbs = [ragged(2 * it + k, patterns[(2 * it + k) % len(patterns)]) for k in range(2)]
            ref = orc.step([(m[0], m[1]) for m in mbs])
            losses = []
            for k, (ids, labels, lens) in enumerate(mbs):
                if it == 1:  # device-pointer entry point
                    d_ids, d_lab, d_len = (torch.from_numpy(a).cuda() for a in (ids, labels, lens))
                    loss, gn, _, stepped = tr.step_ptr(d_ids.data_ptr(), d_lab.data_ptr(), True, d_len.data_ptr(), ids.shape[1])
                else:
                    loss, gn, _, stepped = tr.step(ids, labels, lens)
                groups.append(tr.last_step_groups)
                losses.append(loss)
                assert stepped == (k == 1)
            got = float(np.sum(losses)) / 2  # HF: every micro-batch loss divided by grad_accum
            worst_l, worst_g = max(worst_l, abs(got - ref.loss) / ref.loss), max(worst_g, abs(gn - ref.grad_norm) / ref.grad_norm)
        assert max(groups) >= 3 and groups[2] == 1, groups  # [100,100,100,100] stays one group
        # one more optimizer step in the DEFAULT mode (packed) with the same gradient accumulation: two ragged micro-batches of
        # different packed sizes accumulate into one step
        L.set_option("varlen_split", 1)
        mbs = [ragged(20 + k, patterns[k]) for k in range(2)]
        ref = orc.step([(m[0], m[1]) for m in mbs])
        losses, modes = [], []
        for ids, labels, lens in mbs:
            loss, gn, _, stepped = tr.step(ids, labels, lens)
            losses.append(loss)
            modes.append(tr.last_step_groups)
        packed_l, packed_g = abs(float(np.sum(losses)) / 2 - ref.loss) / ref.loss, abs(gn - ref.grad_norm) / ref.grad_norm
        assert stepped and modes == [0, 0] and packed_l < 1e-3 and packed_g < 3e-2, (modes, packed_l, packed_g)
        L.set_option("varlen_split", 2)
        # adapter gradients of one ragged micro-batch pair against the oracle's autograd gradients (fresh adapters as above)
        tr.load_state_dict({k: v.numpy() for k, v in lora.items()})
        with torch.no_grad():
            for k, v in lora.items():
                orc.lora[k].copy_(v)
        a, b = ragged(50, [300, 5, 200, 129]), ragged(51, [64, 511, 128, 260])
        _, g_a = orc.loss_and_grads(a[0], a[1])
        _, g_b = orc.loss_and_grads(b[0], b[1])
        tr.step(*a)
        tr.step(*b)  # the exported buffer holds the SUM over the micro-batches (1 / grad_accum is applied inside the optimizer kernel)
        got = tr.export_adapter(grads=True)
        per = {}
        for k, v in got.items():
            kk = k.replace("base_model.model.", "")
            r = g_a[kk].numpy() + g_b[kk].numpy()
            per[k.split("layers.")[1]] = float(np.linalg.norm(v - r) / max(np.linalg.norm(r), 1e-12))
        tr.close()
    finally:
        L.set_option("varlen_split", 1)
    assert worst_l < 1e-3 and worst_g < 3e-2 and max(per.values()) < 4e-2, (worst_l, worst_g, per)
    return {"loss": worst_l, "gnorm": worst_g, "groups": groups, "adapter_grads": per, "eval_row_sums_rel": eval_rel,
            "packed_with_grad_accum": {"loss": packed_l, "gnorm": packed_g}}


def check_eval_rows_and_force_step():
    """dtx_eval_loss row statistics compose to the batch loss; DTX_STEP_FORCE steps before grad_accum micro-batches are in."""
    ocfg, mc, tc = tiny_configs(steps=4)
    ocfg.grad_accum = 4
    tc.grad_accum = 4
    w, lora = O.init_base_weights(ocfg, 1234), O.init_lora(ocfg, 4321)
    tr = L.Trainer(mc, tc)
    tr.load_state_dict({k: v.numpy() for k, v in w.items()})
    tr.load_state_dict({k: v.numpy() for k, v in lora.items()})
    ids, labels = O.synthetic_batch(0, 0, tc.micro_batch, tc.seq_len, ocfg.vocab)
    sums, cnts = tr.eval_rows(ids, labels)
    loss = tr.eval_loss(ids, labels)
    assert abs(float(sums.sum()) / int(cnts.sum()) - loss) < 1e-5 * loss, (sums, cnts, loss)
    assert cnts.tolist() == [int((labels[b, 1:] >= 0).sum()) for b in range(tc.micro_batch)]
    _, _, _, st0 = tr.step(ids, labels)
    _, gn, _, st1 = tr.step(ids, labels, force_step=True)
    assert not st0 and st1, "the forced step must run after 2 of 4 micro-batches"
    # HF divides every micro-batch loss by grad_accum whatever the number accumulated: the norm is 2/4 of one batch's
    orc = O.OracleTrainer(O.OracleConfig(**{**ocfg.__dict__, "grad_accum": 1}), w, lora)
    orc.fwd_count = 2
    ref = orc.step([(ids, labels)])
    assert abs(gn - 0.5 * ref.grad_norm) / ref.grad_norm < 2e-2, (gn, ref.grad_norm)
    tr.close()
    return {"gnorm_forced": gn, "oracle_full": ref.grad_norm}


def check_missing_weight_is_refused():
    """A checkpoint with a hole must fail loudly (DTX_ERR_STATE), never train on uninitialised memory."""
    ocfg, mc, tc = tiny_configs(steps=2)
    w, lora = O.init_base_weights(ocfg, 1234), O.init_lora(ocfg, 4321)
    tr = L.Trainer(mc, tc)
    tr.load_state_dict({k: v.numpy() for k, v in w.items() if k != "model.layers.1.mlp.up_proj.weight"})
    tr.load_state_dict({k: v.numpy() for k, v in lora.items()})
    ids, labels = O.synthetic_batch(0, 0, tc.micro_batch, tc.seq_len, ocfg.vocab)
    try:
        tr.step(ids, labels)
        raise AssertionError("step must be refused")
    except L.DtxError as e:
        assert e.code == -4 and "model.layers.1.mlp.up_proj.weight" in str(e), e
    tr.load_tensor("model.layers.1.mlp.up_proj.weight", w["model.layers.1.mlp.up_proj.weight"].numpy())
    loss = tr.step(ids, labels)[0]
    tr.close()
    assert np.isfinite(loss)
    return {"loss": loss}


def _bf16_bits_to_f32(a: np.ndarray) -> np.ndarray:
    return (a.astype(np.uint32) << 16).view(np.float32)


def check_trainer_full(steps=8, grad_accum=1, weight_decay=0.01):
    """Full-parameter SFT (BASELINE.json configs[3]): every weight trains.  Native (bf16 weights / gradients, fp32 master + Adam
    state) against the fp32 oracle with all weights trainable: per-tensor gradients of the first step, loss and grad-norm
    traces, and the weights after `steps` optimizer steps."""
    ocfg, mc, tc = tiny_configs(steps=steps)
    ocfg.full_finetune, tc.full_finetune = True, True
    ocfg.grad_accum, tc.grad_accum = grad_accum, grad_accum
    ocfg.weight_decay, tc.weight_decay = weight_decay, weight_decay
    w = O.init_base_weights(ocfg, 1234)
    g = torch.Generator().manual_seed(3)
    for k in w:  # norm weights away from 1 so that their gradients and the no-decay rule are exercised
        if k.endswith("norm.weight"):
            w[k] = O.bf16_round(1.0 + 0.1 * torch.randn(w[k].shape, generator=g))
    tr = L.Trainer(mc, tc)
    tr.load_state_dict({k: v.numpy() for k, v in w.items()})
    assert tr.num_trainable == sum(v.numel() for v in w.values()), (tr.num_trainable, sum(v.numel() for v in w.values()))
    orc = O.OracleTrainer(ocfg, w, {})
    S, B = tc.seq_len, tc.micro_batch
    worst_l = worst_g = 0.0
    grad_errs = {}
    for s_ in range(steps):
        batches = [O.synthetic_batch(grad_accum * s_ + i, 0, B, S, ocfg.vocab) for i in range(grad_accum)]
        if s_ == 0:
            _, g_ref = O.OracleTrainer(ocfg, w, {}).loss_and_grads(*batches[0])
        ref = orc.step(batches)
        losses = []
        for i, (ids, labels) in enumerate(batches):
            loss, gn, lr, stepped = tr.step(ids, labels)
            losses.append(loss)
            if s_ == 0 and i == 0:  # gradients of the first micro-batch, before anything else touches the buffer
                got = tr.export_weights(grads=True)
                for k, v in got.items():
                    r = g_ref[k].numpy()
                    grad_errs[k] = float(np.linalg.norm(_bf16_bits_to_f32(v) - r) / max(np.linalg.norm(r), 1e-12))
            assert stepped == (i == grad_accum - 1)
        assert abs(lr - ref.lr) <= 1e-9 + 1e-6 * ref.lr, (lr, ref.lr)
        worst_l = max(worst_l, abs(float(np.mean(losses)) - ref.loss) / ref.loss)
        worst_g = max(worst_g, abs(gn - ref.grad_norm) / ref.grad_norm)
    wts = tr.export_weights()
    drift = {}
    for k, v in wts.items():
        r = orc.lora[k].detach().numpy()
        drift[k] = float(np.linalg.norm(_bf16_bits_to_f32(v) - r) / max(np.linalg.norm(r), 1e-12))
    moved = float(np.linalg.norm(_bf16_bits_to_f32(wts["model.layers.0.mlp.down_proj.weight"]) - w["model.layers.0.mlp.down_proj.weight"].numpy()))
    tr.close()
    worst_grad = max(grad_errs.values())
    worst_tensor = max(grad_errs, key=grad_errs.get)
    assert worst_grad < 5e-2, f"gradient of {worst_tensor}: {worst_grad}; all {grad_errs}"
    assert worst_l < 2e-3 and worst_g < 3e-2, (worst_l, worst_g)
    assert max(drift.values()) < 1e-2 and moved > 0, (max(drift.values()), moved)  # bf16 weights: 2^-9 relative rounding
    return {"loss": worst_l, "gnorm": worst_g, "worst_grad": [worst_tensor, worst_grad], "weight_drift": max(drift.values()), "moved": moved}


def check_trainer_full_gqa(steps=4):
    """Full-parameter SFT on a grouped-query model at a ragged batch (row lengths): the dK / dV width differs from dQ.  The batch
    runs PACKED (384 + 256 rows instead of 2 x 384): the weight-gradient GEMMs contract over the packed token rows."""
    ocfg, mc, tc = tiny_configs(S=384, B=2, steps=steps, heads=4, kv_heads=2)
    ocfg.full_finetune, tc.full_finetune = True, True
    w = O.init_base_weights(ocfg, 77)
    tr = L.Trainer(mc, tc)
    tr.load_state_dict({k: v.numpy() for k, v in w.items()})
    orc = O.OracleTrainer(ocfg, w, {})
    worst_l = worst_g = 0.0
    for s_ in range(steps):
        ids, labels = O.synthetic_batch(s_, 0, 2, 384, ocfg.vocab)
        lens = np.array([384, 200], dtype=np.int32)
        ids[1, 200:] = 0
        labels[1, 200:] = -100
        ref = orc.step([(ids, labels)])
        loss, gn, _, _ = tr.step(ids, labels, lens)
        assert tr.last_step_groups == 0, tr.last_step_groups  # packed
        worst_l, worst_g = max(worst_l, abs(loss - ref.loss) / ref.loss), max(worst_g, abs(gn - ref.grad_norm) / ref.grad_norm)
    wts = tr.export_weights()
    drift = max(float(np.linalg.norm(_bf16_bits_to_f32(v) - orc.lora[k].detach().numpy()) / max(np.linalg.norm(orc.lora[k].detach().numpy()), 1e-12))
                for k, v in wts.items())
    tr.close()
    assert worst_l < 2e-3 and worst_g < 3e-2 and drift < 1e-2, (worst_l, worst_g, drift)
    return {"loss": worst_l, "gnorm": worst_g, "weight_drift": drift}


def check_layer_7b_shape(B=2, S=2048):
    """One Llama-2-7B-shaped decoder layer (d=4096, H=32, F=11008) + lm_head (V=32000) + CE through the native trainer at the
    benchmark's sequence length, against the fp32 oracle on the host cores: forward loss, step loss, grad-norm and every
    adapter gradient tensor.  This is the geometry bench.py times (86-tile N sweeps, split-K choices, 2048 attention CTAs
    per launch, the fused RoPE / SwiGLU epilogues) - only the layer count is reduced."""
    ocfg = O.OracleConfig(vocab=32000, hidden=4096, n_layers=1, n_heads=32, ffn=11008, lora_r=16, lora_alpha=32.0, lr=1e-4, total_steps=100)
    mc = L.ModelConfig(vocab=32000, hidden=4096, n_layers=1, n_heads=32, ffn=11008)
    tc = L.TrainConfig(micro_batch=B, seq_len=S, total_steps=100, lora_r=16, lora_alpha=32.0, lora_dropout=0.0, lr=1e-4)
    t0 = time.time()
    w, lora = O.init_base_weights(ocfg, 1234), O.init_lora(ocfg, 4321)
    # B = 0 at init would leave the A gradients identically zero: give B a small random value so that every gradient is exercised
    g = torch.Generator().manual_seed(99)
    for k in lora:
        if "lora_B" in k:
            lora[k] = torch.randn(lora[k].shape, generator=g) * 0.01
    tr = L.Trainer(mc, tc)
    tr.load_state_dict({k: v.numpy() for k, v in w.items()})
    tr.load_state_dict({k: v.numpy() for k, v in lora.items()})
    orc = O.OracleTrainer(ocfg, w, lora)
    t_init = time.time() - t0
    ids, labels = O.synthetic_batch(0, 0, B, S, ocfg.vocab)
    t0 = time.time()
    ref_loss, g_ref = orc.loss_and_grads(ids, labels)
    t_cpu = time.time() - t0
    e_eval = abs(tr.eval_loss(ids, labels) - ref_loss) / ref_loss
    loss, gn, _, stepped = tr.step(ids, labels)
    ref_norm = math.sqrt(sum(float((v.double() ** 2).sum()) for v in g_ref.values()))
    got = tr.export_adapter(grads=True)
    errs = {}
    for k, v in got.items():
        r = g_ref[k.replace("base_model.model.", "")].numpy()
        errs[k.split("layers.0.")[1]] = float(np.linalg.norm(v - r) / max(np.linalg.norm(r), 1e-12))
    # the same geometry with RAGGED rows run as two length groups (rows of 2048 and 700 tokens -> rectangles [1, 2048] and
    # [1, 768]) against the oracle on the padded batch as a whole; the adapters are reset to the ones the oracle holds
    ragged = {}
    if B == 2 and S >= 1024:
        tr.load_state_dict({k: v.numpy() for k, v in lora.items()})
        lens = np.array([S, 700], dtype=np.int32)
        ids2, labels2 = O.synthetic_batch(1, 0, B, S, ocfg.vocab)
        ids2[1, 700:] = 0
        labels2[1, 700:] = -100
        ref2, g2 = orc.loss_and_grads(ids2, labels2)
        def rel_errs(got):
            return {k.split("layers.0.")[1]: float(np.linalg.norm(v - g2[k.replace("base_model.model.", "")].numpy()) /
                                                   max(np.linalg.norm(g2[k.replace("base_model.model.", "")].numpy()), 1e-12)) for k, v in got.items()}
        L.set_option("varlen_split", 2)
        try:
            loss2, _, _, _ = tr.step(ids2, labels2, lens)
            n_groups = tr.last_step_groups
        finally:
            L.set_option("varlen_split", 1)
        errs2 = rel_errs(tr.export_adapter(grads=True))
        ragged = {"groups": n_groups, "loss_rel": abs(loss2 - ref2) / ref2, "adapter_grad_rel": errs2}
        assert n_groups == 2 and ragged["loss_rel"] < 1e-3 and max(errs2.values()) < 4e-2, ragged
        # and PACKED (the default): one pass over 2048 + 768 rows, the second sequence starting at row 2048
        tr.load_state_dict({k: v.numpy() for k, v in lora.items()})
        loss3, _, _, _ = tr.step(ids2, labels2, lens)
        errs3 = rel_errs(tr.export_adapter(grads=True))
        ragged["packed"] = {"mode": tr.last_step_groups, "loss_rel": abs(loss3 - ref2) / ref2, "adapter_grad_rel": errs3}
        assert tr.last_step_groups == 0 and ragged["packed"]["loss_rel"] < 1e-3 and max(errs3.values()) < 4e-2, ragged
    tr.close()
    res = {"eval_loss_rel": e_eval, "step_loss_rel": abs(loss - ref_loss) / ref_loss, "gnorm_rel": abs(gn - ref_norm) / ref_norm,
           "adapter_grad_rel": errs, "oracle_loss": ref_loss, "native_loss": loss, "sec_init": t_init, "sec_oracle_fwd_bwd": t_cpu,
           "ragged_length_groups": ragged}
    assert e_eval < 1e-3 and res["step_loss_rel"] < 1e-3, res
    assert res["gnorm_rel"] < 3e-2 and max(errs.values()) < 4e-2, res
    return res




def tiny_configs(S=256, B=2, steps=20, L_layers=2, vocab=2048, heads=2, kv_heads=None, dropout=0.0, targets=("q_proj", "v_proj")):
    ocfg = O.OracleConfig(vocab=vocab, hidden=128 * heads, n_layers=L_layers, n_heads=heads, n_kv_heads=kv_heads, ffn=768, lora_r=16,
                          lora_alpha=32.0, lr=1e-3, total_steps=steps, lora_dropout=dropout, lora_target=tuple(targets))
    mc = L.ModelConfig(vocab=vocab, hidden=128 * heads, n_layers=L_layers, n_heads=heads, n_kv_heads=kv_heads, ffn=768)
    tc = L.TrainConfig(micro_batch=B, seq_len=S, total_steps=steps, lora_r=16, lora_alpha=32.0, lora_dropout=dropout, lr=1e-3,
                       lora_target=tuple(targets))
    return ocfg, mc, tc


def make_tiny_pair(S=256, B=2, steps=20, L_layers=2, vocab=2048, **kw):
    ocfg, mc, tc = tiny_configs(S, B, steps, L_layers, vocab, **kw)
    w, lora = O.init_base_weights(ocfg, 1234), O.init_lora(ocfg, 4321)
    tr = L.Trainer(mc, tc)
    tr.load_state_dict({k: v.numpy() for k, v in w.items()})
    tr.load_state_dict({k: v.numpy() for k, v in lora.items()})
    return ocfg, O.OracleTrainer(ocfg, w, lora), tr


def check_trainer_tiny(steps=10, **kw):
    ocfg, orc, tr = make_tiny_pair(steps=steps, **kw)
    S, B = tr.train.seq_len, tr.train.micro_batch
    ids, labels = O.synthetic_batch(0, 0, B, S, ocfg.vocab)
    ref_eval = orc.eval_loss(ids, labels)  # exactly one forward pass on each side (forward passes key the dropout masks)
    e_eval = abs(tr.eval_loss(ids, labels) - ref_eval) / ref_eval
    assert e_eval < 1e-3, f"forward loss mismatch {e_eval}"
    worst_l = worst_g = 0.0
    trace = []
    for s in range(steps):
        ids, labels = O.synthetic_batch(s, 0, B, S, ocfg.vocab)
        ref = orc.step([(ids, labels)])
        loss, gn, lr, stepped = tr.step(ids, labels)
        assert stepped
        assert abs(lr - ref.lr) <= 1e-9 + 1e-6 * ref.lr, (lr, ref.lr)
        worst_l = max(worst_l, abs(loss - ref.loss) / ref.loss)
        worst_g = max(worst_g, abs(gn - ref.grad_norm) / ref.grad_norm)
        trace.append((loss, ref.loss, gn, ref.grad_norm))
    assert worst_l < 1e-3, f"loss trace rel diff {worst_l}: {trace}"
    assert worst_g < 3e-2, f"grad-norm trace rel diff {worst_g}: {trace}"
    ad, ref_ad = tr.export_adapter(), orc.state_dict()
    worst_a = 0.0
    for k, v in ad.items():
        r = ref_ad[k.replace("base_model.model.", "")]
        worst_a = max(worst_a, float(np.linalg.norm(v - r) / max(np.linalg.norm(r), 1e-12)))
    # Adam normalises tiny, bf16-noisy gradients: a few % relative drift of the adapters after 10 steps is expected;
    # a wrong gradient shows up as O(1)
    assert worst_a < 0.15, f"adapter drift {worst_a}"
    tr.close()
    return {"eval": e_eval, "loss": worst_l, "gnorm": worst_g, "adapter": worst_a, "last": trace[-1]}


def check_trainer_unfused():
    """Same parity run with RoPE / SwiGLU as separate kernels (the fused GEMM / attention epilogues are the default)."""
    L.set_option("fused_epilogues", 0)
    try:
        return check_trainer_tiny()
    finally:
        L.set_option("fused_epilogues", 1)


def check_trainer_deterministic(steps=3):
    runs = []
    for _ in range(2):
        ocfg, _, tr = make_tiny_pair(steps=steps)
        out = []
        for s in range(steps):
            ids, labels = O.synthetic_batch(s, 0, tr.train.micro_batch, tr.train.seq_len, ocfg.vocab)
            out.append(tr.step(ids, labels)[:2])
        runs.append((out, {k: v.tobytes() for k, v in tr.export_adapter().items()}))
        tr.close()
    assert runs[0][0] == runs[1][0], "loss / grad-norm must be bitwise reproducible"
    assert runs[0][1] == runs[1][1], "adapters must be bitwise reproducible"
    return {"bitwise": True}


def check_trainer_grad_accum():
    """2 micro-batches with grad_accum=2 == oracle's mean over both (DeepSpeed ZeRO-0 / HF accumulation)."""
    ocfg, mc, tc = tiny_configs(steps=4)
    ocfg.grad_accum = 2
    tc.grad_accum = 2
    w, lora = O.init_base_weights(ocfg, 1234), O.init_lora(ocfg, 4321)
    tr = L.Trainer(mc, tc)
    tr.load_state_dict({k: v.numpy() for k, v in w.items()})
    tr.load_state_dict({k: v.numpy() for k, v in lora.items()})
    orc = O.OracleTrainer(ocfg, w, lora)
    worst = 0.0
    for s in range(3):
        batches = [O.synthetic_batch(2 * s + i, 0, tc.micro_batch, tc.seq_len, ocfg.vocab) for i in range(2)]
        ref = orc.step(batches)
        l0, _, _, st0 = tr.step(*batches[0])
        l1, gn, lr, st1 = tr.step(*batches[1])
        assert not st0 and st1
        worst = max(worst, abs(0.5 * (l0 + l1) - ref.loss) / ref.loss, abs(gn - ref.grad_norm) / ref.grad_norm / 30)
    assert worst < 1e-3, worst
    tr.close()
    return {"worst": worst}


def check_gemm_single_cta():
    """The 128 x 128-tile kernel stays covered when 128 x 256 tiles are the default for wide GEMMs."""
    L.set_option("gemm_pair_kernel", 0)
    try:
        out = {"nt": check_gemm_nt(), "nn": check_gemm_nn(), "kext": check_gemm_kext(), "ragged": check_gemm_ragged()}
    finally:
        L.set_option("gemm_pair_kernel", 1)
    return out


def check_gemm_pair_vs_single(M=8192, N=8192, K=4096):
    """Bitwise agreement of the two kernels (same fp32 accumulation order along K) + timing of both."""
    A, B = _rand(M, K, scale=0.05, seed=30), _rand(N, K, scale=0.05, seed=31)
    lib = L.load()
    res = {}
    outs = []
    for name, flag in (("pair", 1), ("single", 0)):
        L.set_option("gemm_pair_kernel", flag)
        Cm = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
        s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(3):
            ok(lib.dtx_gemm_bf16(P(A), K, 0, P(B), K, 0, None, 0, None, 0, 0, P(Cm), N, None, 0, M, N, K, 0, 1, 0, STREAM()))
        s.record()
        for _ in range(10):
            ok(lib.dtx_gemm_bf16(P(A), K, 0, P(B), K, 0, None, 0, None, 0, 0, P(Cm), N, None, 0, M, N, K, 0, 1, 0, STREAM()))
        t.record()
        torch.cuda.synchronize()
        res[name + "_tflops"] = 2.0 * M * N * K / (s.elapsed_time(t) / 10) / 1e9
        outs.append(Cm)
    L.set_option("gemm_pair_kernel", 1)
    assert torch.equal(outs[0], outs[1]), "pair and single-CTA kernels must agree bitwise"
    ref = (A @ B.t())
    res["rel_err_vs_cublas"] = rel_err(outs[0], ref)
    assert res["rel_err_vs_cublas"] < 1e-2
    return res


def check_trainer_100_steps():
    """north_star: training loss within 1e-3 relative of the reference CPU path after 100 steps (tiny-Llama config).
    Compared with the live fp32 oracle and with the committed oracle trace tests/golden/tiny_trace_100.json."""
    import json
    import os
    gold = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "tiny_trace_100.json")))
    ocfg, orc, tr = make_tiny_pair(steps=100)
    S, B = tr.train.seq_len, tr.train.micro_batch
    worst = worst_gold = 0.0
    native, ref = [], []
    for s in range(100):
        ids, labels = O.synthetic_batch(s, 0, B, S, ocfg.vocab)
        r = orc.step([(ids, labels)])
        loss, gn, lr, _ = tr.step(ids, labels)
        native.append(loss)
        ref.append(r.loss)
        worst = max(worst, abs(loss - r.loss) / r.loss)
        g = gold["trace_loss_gradnorm_lr"][s]
        worst_gold = max(worst_gold, abs(r.loss - g[0]) / g[0])
        assert abs(lr - g[2]) <= 1e-6 * g[2] + 1e-12
    tr.close()
    w_nat, w_ref = float(np.mean(native[90:])), float(np.mean(ref[90:]))  # the value HF logs at step 100 (window mean)
    res = {"worst_step_rel": worst, "step100_rel": abs(native[99] - ref[99]) / ref[99], "window_91_100_rel": abs(w_nat - w_ref) / w_ref,
           "oracle_vs_golden_rel": worst_gold, "loss_step1": native[0], "loss_step100": native[99], "oracle_step100": ref[99]}
    assert worst_gold < 1e-5, f"oracle drifted from its committed trace: {worst_gold}"
    assert res["step100_rel"] < 1e-3 and res["window_91_100_rel"] < 1e-3 and worst < 1e-3, res
    assert native[99] < native[0] - 0.01, "loss must go down"
    return res


def check_worker_end_to_end():
    """The whole worker behind the controller's command line on a tiny HF-format model directory: argv -> CSV -> llama2
    template -> native training -> PEFT adapter + checkpoint-path file + trainer_log.jsonl (cmd/tuning/train.py:308-389)."""
    import json
    import os
    import shlex
    import shutil
    import tempfile
    from datatunerx_b200.tuning import model_io, parser as TP
    tmp = tempfile.mkdtemp(prefix="dtx_e2e_")
    try:
        mdir, out, store = os.path.join(tmp, "model"), os.path.join(tmp, "result"), os.path.join(tmp, "storage")
        os.makedirs(mdir)
        gold = os.path.join(os.path.dirname(__file__), "golden")
        shutil.copy(os.path.join(gold, "tiny_tokenizer.json"), os.path.join(mdir, "tokenizer.json"))
        json.dump({"tokenizer_class": "PreTrainedTokenizerFast", "bos_token": "<s>", "eos_token": "</s>", "unk_token": "<unk>"},
                  open(os.path.join(mdir, "tokenizer_config.json"), "w"))
        ocfg = O.OracleConfig(vocab=400, hidden=256, n_layers=2, n_heads=2, ffn=768)
        json.dump({"architectures": ["LlamaForCausalLM"], "vocab_size": 400, "hidden_size": 256, "intermediate_size": 768,
                   "num_hidden_layers": 2, "num_attention_heads": 2, "num_key_value_heads": 2, "rms_norm_eps": 1e-5, "rope_theta": 10000.0,
                   "max_position_embeddings": 4096, "model_type": "llama"}, open(os.path.join(mdir, "config.json"), "w"))
        model_io.write_safetensors(os.path.join(mdir, "model.safetensors"), {k: v.numpy() for k, v in O.init_base_weights(ocfg, 7).items()})
        csv_path = os.path.join(tmp, "train.csv")
        with open(csv_path, "w") as f:
            f.write("q,a\n")
            for i in range(48):
                f.write(f"What is {i} plus {i}?,The answer is {2 * i}.\n")
        ckpt_file = os.path.join(tmp, "checkpoint_path")
        os.environ["DTX_CHECKPOINT_PATH_FILE"] = ckpt_file
        import importlib
        from datatunerx_b200.tuning import train as TT
        importlib.reload(TT)
        entry = TP.controller_entrypoint(mdir, csv_path, validate_file=csv_path, columns='{"instruction":"q","response":"a"}',
                                         scheduler="linear", optimizer="adamw_hf", lora_r="16", lora_alpha="32", lora_dropout="0.0",
                                         learning_rate="1e-3", epochs=2, block_size=256, batch_size=4, grad_acc_steps=1,
                                         num_workers=1, storage_path=store, uid="e2e")
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            rc = TT.main(shlex.split(entry)[2:])
        finally:
            os.chdir(cwd)
        assert rc == 0, f"worker exit status {rc}"
        ckpt = open(ckpt_file).read()
        assert not ckpt.endswith("\n") and ckpt.startswith(store) and os.path.isdir(ckpt), f"checkpoint path file: {ckpt!r}"
        cfg = json.load(open(os.path.join(ckpt, "adapter_config.json")))
        assert cfg["r"] == 16 and cfg["target_modules"] == ["q_proj", "v_proj"] and cfg["peft_type"] == "LORA", cfg
        ad = {k: np.array(a) for k, a, _ in model_io.iter_safetensors(os.path.join(ckpt, "adapter_model.safetensors"))}
        logs_dbg = open(os.path.join(tmp, "result", "watch", "trainer_log.jsonl")).read()
        bad = {k: int((~np.isfinite(v)).sum()) for k, v in ad.items() if not np.isfinite(v).all()}
        assert len(ad) == 8 and not bad, f"non-finite adapters {bad}; logs: {logs_dbg[:600]}"
        assert any(np.abs(v).max() > 0 for k, v in ad.items() if "lora_B" in k), "B adapters must have moved"
        logs = [json.loads(l) for l in open(os.path.join(tmp, "result", "watch", "trainer_log.jsonl"))]
        assert len(logs) == 2 and logs[0]["current_steps"] == 10 and logs[0]["total_steps"] == 24, logs
        assert logs[1]["loss"] < logs[0]["loss"], f"loss did not go down: {logs}"
        ev = [json.loads(l) for l in open(os.path.join(tmp, "result", "watch", "eval_log.jsonl"))]
        assert abs(ev[0]["eval_perplexity"] - math.exp(ev[0]["eval_loss"])) < 1e-9, ev
        return {"first_log_loss": logs[0]["loss"], "last_log_loss": logs[1]["loss"], "eval_loss": ev[0]["eval_loss"], "ckpt": os.path.basename(ckpt)}
    finally:
        os.environ.pop("DTX_CHECKPOINT_PATH_FILE", None)
        shutil.rmtree(tmp, ignore_errors=True)


ALL = {
    "gemm_nt": check_gemm_nt, "gemm_nt_bn64": lambda: check_gemm_nt(N=64, block_n=64),
    "gemm_nt_bn128": lambda: check_gemm_nt(N=384, block_n=128), "gemm_nn": check_gemm_nn,
    "gemm_nn_bn64": lambda: check_gemm_nn(N=64, block_n=64), "gemm_tn": check_gemm_tn,
    "gemm_tn_nosplit": lambda: check_gemm_tn(split_k=1), "gemm_tn_pair": check_gemm_tn_pair, "gemm_kext": check_gemm_kext, "gemm_ragged": check_gemm_ragged,
    "gemm_large": check_gemm_large, "gemm_single_cta": check_gemm_single_cta, "gemm_pair_vs_single": check_gemm_pair_vs_single, "rmsnorm": check_rmsnorm, "rmsnorm_small": lambda: check_rmsnorm(M=64, d=256),
    "rope": check_rope, "swiglu": check_swiglu, "lora_dropout": check_lora_dropout, "nf4": check_nf4, "nf4_pack": check_nf4_pack,
    "gemm_rope_epilogue": check_gemm_rope_epilogue,
    "gemm_rope_epilogue_7b": lambda: check_gemm_rope_epilogue(S=2048, B=2, H=32, Hkv=32, K=4096, ragged=False),
    "gemm_swiglu_epilogues": check_gemm_swiglu_epilogues,
    "attn_bench_shape_s2048": check_attn_bench_shape,
    "attn_bench_shape_s4096_gqa": lambda: check_attn_bench_shape(B=1, S=4096, H=32, Hkv=8, kv_heads=(0, 5)),
    "attn_bwd_rope": check_attn_bwd_rope, "attn_varlen": check_attn_varlen, "attn_window": check_attn_window,
    "trainer_window": check_trainer_window,
    "trainer_varlen": check_trainer_varlen, "trainer_varlen_groups": check_trainer_varlen_groups, "eval_rows_force_step": check_eval_rows_and_force_step,
    "missing_weight_refused": check_missing_weight_is_refused, "layer_7b_shape": check_layer_7b_shape,
    "trainer_full": check_trainer_full, "trainer_full_accum": lambda: check_trainer_full(steps=4, grad_accum=2, weight_decay=0.0),
    "trainer_full_gqa": lambda: check_trainer_full_gqa(), "trainer_qlora": check_trainer_qlora, "embedding": check_embedding, "cross_entropy": check_cross_entropy,
    "adamw": check_adamw, "attn_fwd": check_attn_fwd, "attn_fwd_long": lambda: check_attn_fwd(B=1, S=1024, H=1),
    "attn_fwd_rescale": lambda: check_attn_fwd(B=1, S=1024, H=2, growing=True),
    "attn_fwd_odd_tiles": lambda: {"s640": check_attn_fwd(B=1, S=640, H=2), "s128": check_attn_fwd(B=3, S=128, H=2)},
    "attn_fwd_exp_fma": check_attn_fwd_exp_fma,
    "attn_bwd_single_tile": lambda: check_attn_bwd(B=3, S=128, H=2),
    "attn_bwd": check_attn_bwd, "attn_bwd_long": lambda: check_attn_bwd(B=1, S=1024, H=1),
    "attn_gqa": lambda: {"fwd": check_attn_fwd(B=2, S=384, H=4, Hkv=2), "bwd": check_attn_bwd(B=2, S=384, H=4, Hkv=1)},
    "trainer_gqa": lambda: check_trainer_tiny(heads=4, kv_heads=2, targets=("q_proj", "k_proj", "v_proj")),
    "trainer_dropout": lambda: check_trainer_tiny(dropout=0.1),
    "trainer_tiny": check_trainer_tiny, "trainer_unfused": check_trainer_unfused, "trainer_deterministic": check_trainer_deterministic,
    "trainer_grad_accum": check_trainer_grad_accum, "trainer_100_steps": check_trainer_100_steps,
    "worker_end_to_end": check_worker_end_to_end,
}

if __name__ == "__main__":
    # usage: python -m tests.gpu_checks name [name ...]   — runs in order, one RESULT line per check; exits with
    # code 3 right after a failure that may have poisoned the CUDA context so the driver can restart with the rest
    import json
    import sys
    import traceback
    for name in sys.argv[1:]:
        t0 = time.time()
        try:
            res = ALL[name]()
            print("RESULT " + json.dumps({"name": name, "ok": True, "sec": round(time.time() - t0, 2), "metrics": res}, default=str),
                  flush=True)
        except AssertionError as e:
            print("RESULT " + json.dumps({"name": name, "ok": False, "sec": round(time.time() - t0, 2), "error": str(e)[:1500]}),
                  flush=True)
            try:
                torch.cuda.synchronize()
            except Exception:
                sys.exit(3)
        except Exception as e:
            print("RESULT " + json.dumps({"name": name, "ok": False, "sec": round(time.time() - t0, 2),
                                          "error": (str(e) + " | " + traceback.format_exc())[-1500:]}), flush=True)
            sys.exit(3)
