"""Op-level determinism at the 7B layer geometry (M = 4096 tokens): every kernel is run several times on identical inputs and
the outputs are compared bitwise (and against an fp32 torch reference on a row sample).  Localises races."""
import ctypes as C
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from datatunerx_b200 import lib as L  # noqa: E402

DEV = "cuda:0"
P = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
ST = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).to(DEV)


def repeat(name, fn, outs, n=4, ref=None):
    """fn() launches; outs() returns the tensors to compare."""
    sigs = []
    for i in range(n):
        for o in outs():
            o.fill_(float("nan")) if o.is_floating_point() else o.zero_()
        fn()
        torch.cuda.synchronize()
        sigs.append([o.clone() for o in outs()])
    same = all(all(torch.equal(a.view(torch.uint8), b.view(torch.uint8)) for a, b in zip(sigs[0], s)) for s in sigs[1:])
    row = {"op": name, "deterministic": same}
    if not same:
        for k, s in enumerate(sigs[1:], 1):
            for j, (a, b) in enumerate(zip(sigs[0], s)):
                if not torch.equal(a.view(torch.uint8), b.view(torch.uint8)):
                    d = (a.float() - b.float())
                    bad = torch.nonzero(d.abs() > 0)
                    row[f"run{k}_out{j}"] = {"n_diff": int(bad.shape[0]), "max_abs": float(d.abs().max()),
                                             "first": bad[0].tolist() if bad.shape[0] else None, "last": bad[-1].tolist() if bad.shape[0] else None}
    if ref is not None:
        row["rel_err_vs_fp32"] = ref(sigs[0])
    print("DETERMINISM " + json.dumps(row), flush=True)
    return same


def main():
    lib = L.load()
    M, d, F, V, H, S, B = 4096, 4096, 11008, 32000, 32, 2048, 2
    W = 3 * d
    rel = lambda a, b: float((a.float() - b.float()).norm() / b.float().norm())

    def gemm(A, Bm, Cm, *, b_mn=0, a_mn=0, A2=None, B2=None, R=None, epi=0, split=1, bn=0, m=None, n=None, k=None):
        K2 = (A2.shape[0] if a_mn else A2.shape[1]) if A2 is not None else 0
        L.check(lib.dtx_gemm_bf16(P(A), A.stride(0), a_mn, P(Bm), Bm.stride(0), b_mn, P(A2), A2.stride(0) if A2 is not None else 0, P(B2),
                                  B2.stride(0) if B2 is not None else 0, K2, P(Cm), Cm.stride(-2), P(R), R.stride(0) if R is not None else 0, m, n, k, epi,
                                  split, bn, ST()))

    h1, wqkv = rnd(M, d, seed=1), rnd(W, d, scale=0.02, seed=2)
    tt, bext = rnd(M, 64, seed=3), rnd(W, 64, scale=0.02, seed=4)
    qkv = torch.empty(M, W, dtype=torch.bfloat16, device=DEV)
    cs = torch.empty(S, 64, 2, dtype=torch.float32, device=DEV)
    L.check(lib.dtx_rope_table(P(cs), S, 128, 10000.0, ST()))
    repeat("qkv gemm EPI_ROPE + LoRA k-ext", lambda: L.check(lib.dtx_gemm_fused(P(h1), d, P(wqkv), d, 0, P(tt), 64, P(bext), 64, 64, P(qkv), W, None, 0, P(cs), S, 2 * d, M, W, d, 3, ST())), lambda: [qkv])
    acat = rnd(64, d, scale=0.02, seed=5)
    t_out = torch.empty(M, 64, dtype=torch.bfloat16, device=DEV)
    repeat("lora down gemm N=64", lambda: gemm(h1, acat, t_out, bn=64, m=M, n=64, k=d), lambda: [t_out])
    out = torch.empty(M, d, dtype=torch.bfloat16, device=DEV)
    lse = torch.empty(B, H, S, dtype=torch.float32, device=DEV)
    sc = 1.0 / math.sqrt(128)
    for every in (3, 0):
        L.set_option("attn_fwd_exp_fma_every", every)
        repeat(f"attn_fwd exp_fma_every={every}", lambda: L.check(lib.dtx_attn_fwd(P(qkv), P(out), P(lse), B, S, H, H, sc, None, 0, ST())), lambda: [out, lse], n=6)
    L.set_option("attn_fwd_exp_fma_every", 0)
    wo, res = rnd(d, d, scale=0.02, seed=6), rnd(M, d, seed=7)
    xmid = torch.empty(M, d, dtype=torch.bfloat16, device=DEV)
    repeat("o_proj gemm EPI_BF16_ADD", lambda: gemm(out, wo, xmid, R=res, epi=2, m=M, n=d, k=d), lambda: [xmid])
    wgu = rnd(2 * F, d, scale=0.02, seed=8)
    gu = torch.empty(M, 2 * F, dtype=torch.bfloat16, device=DEV)
    act = torch.empty(M, F, dtype=torch.bfloat16, device=DEV)
    repeat("gate|up gemm EPI_SWIGLU_FWD", lambda: L.check(lib.dtx_gemm_fused(P(h1), d, P(wgu), d, 0, None, 0, None, 0, 0, P(gu), 2 * F, P(act), F, None, 0, 0, M, 2 * F, d, 4, ST())), lambda: [gu, act])
    wdown = rnd(d, F, scale=0.02, seed=9)
    xn = torch.empty(M, d, dtype=torch.bfloat16, device=DEV)
    repeat("down gemm EPI_BF16_ADD K=11008", lambda: gemm(act, wdown, xn, R=res, epi=2, m=M, n=d, k=F), lambda: [xn])
    lm = rnd(V, d, scale=0.02, seed=10)
    logits = torch.empty(M, V, dtype=torch.float32, device=DEV)
    repeat("lm_head gemm EPI_F32", lambda: gemm(h1, lm, logits, epi=1, m=M, n=V, k=d), lambda: [logits])
    dlog = rnd(M, V, scale=0.01, seed=11)
    dh = torch.empty(M, d, dtype=torch.bfloat16, device=DEV)
    repeat("dh gemm NN K=32000", lambda: gemm(dlog, lm, dh, b_mn=1, m=M, n=d, k=V), lambda: [dh])
    dx = rnd(M, d, seed=12)
    dgu = torch.empty(M, 2 * F, dtype=torch.bfloat16, device=DEV)
    repeat("down bwd gemm EPI_SWIGLU_BWD", lambda: L.check(lib.dtx_gemm_fused(P(dx), d, P(wdown), F, 1, None, 0, None, 0, 0, P(dgu), 2 * F, P(gu), 2 * F, None, 0, 0, M, F, d, 5, ST())), lambda: [dgu])
    repeat("dh2 gemm NN K=22016", lambda: gemm(dgu, wgu, dh, b_mn=1, m=M, n=d, k=2 * F), lambda: [dh])
    repeat("dattn gemm NN", lambda: gemm(dx, wo, dh, b_mn=1, m=M, n=d, k=d), lambda: [dh])
    dout = rnd(M, d, seed=13)
    delta = torch.empty(B, H, S, dtype=torch.float32, device=DEV)
    dqkv = torch.empty(M, W, dtype=torch.bfloat16, device=DEV)
    cs_t = cs.permute(1, 0, 2).contiguous()
    repeat("attn_bwd (+ inverse rope)", lambda: L.check(lib.dtx_attn_bwd(P(qkv), P(out), P(dout), P(lse), P(delta), P(dqkv), B, S, H, H, sc, None, 0, P(cs_t), S, ST())), lambda: [dqkv, delta], n=6)
    dt = torch.empty(M, 64, dtype=torch.bfloat16, device=DEV)
    repeat("dt gemm NN N=64 K=12288", lambda: gemm(dqkv, bext, dt, b_mn=1, bn=64, m=M, n=64, k=W), lambda: [dt])
    repeat("dh1 gemm NN + k-ext", lambda: gemm(dqkv, wqkv, dh, b_mn=1, A2=dt, B2=acat, m=M, n=d, k=W), lambda: [dh])
    for name, A, rows in (("grad B_ext split-K", dqkv, W), ("grad A_cat split-K", h1, d)):
        for split in (1, 5, 16):
            part = torch.empty(split, rows, 64, dtype=torch.float32, device=DEV)
            repeat(f"{name} TN split={split}", lambda: gemm(A, tt if rows == W else dt, part, a_mn=1, b_mn=1, epi=1, split=split, bn=64, m=rows, n=64, k=M), lambda: [part])


if __name__ == "__main__":
    main()
