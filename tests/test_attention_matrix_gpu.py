"""Kernel-level parity of the attention kernels over all 20 instantiations, with per-element fp64 bounds.

- **Instantiations.**  `variant()` maps the inputs that select a kernel (the forward and dQ exp-FMA switches, an effective
  window > 0, GLM's inverse rotary with a table) to the instantiations a forward + backward call runs: attn_fwd_kernel<E in
  {0, 2, 3, 4}, WIN> (8), attn_dq_kernel<WIN, E in {0, 3, 4}> (6) + <false, E, GLM> (3), attn_dkv_kernel<WIN> (2) + <false, GLM>
  (1).  The sweep reaches all 20 under each layout (rectangular, right-padded with seq_lens, packed with plan_packed_rows).
- **Bounds** (u = 2^-8, twice the unit roundoff of round-to-nearest bf16; fp32 accumulations follow the GEMM's rule 2^-16 sum|ab|).
  Forward: the kernel rounds the unnormalised probabilities p = 2^(t - m) to bf16 before P V, accumulates in fp32, scales by
  1 / l (l = the fp32 sum of the unrounded p) and rounds to bf16.  Every p carries a relative error e_row made of the exponential
  (2^-21 for ex2.approx, plus 7.5e-5 on the FMA path), the score error ln2 * (scale log2e 2^-16 sum_d |q_d k_d| + 2^-22 |t|), one
  ex2 per rescale of the 64-key blocks and the fp32 sum of l (n 2^-24); l carries the same error, so
      |o - ref| <= (u + 2 e_row) (P^|V|) + u |ref|,        |lse2 - ref| <= 1.5 e_row + 2^-21 (|m| + |ref| + 1)
  with P^ the normalised probabilities.  Backward, driven by the kernel's own bf16 out and fp32 lse2: P = 2^(t - lse2),
  delta = rowsum(dO o out) (fp32 rounding of a 128-term sum: 2^-17 sum|dO o out|), dS = P o (dP - delta) scale, with
      |ddS| = u |dS| + scale P [e (|dP| + |delta|) + 2^-16 (|dO| |V|^T) + |ddelta| + 2^-22 (|dP| + |delta|)]
      dQ: |ddS| |K| + 2^-16 |dS| |K|,  dK: |ddS|^T |Q| + 2^-16 |dS|^T |Q|,  dV: ((u + e) P)^T |dO| + 2^-16 P^T |dO|
  each pushed through |R| of the inverse rotary (half-split or GLM), then + u |ref| for the bf16 store.  No safety factor beyond
  u = 2^-8 is applied; a case that fails its bound is a finding, not a bar to move.  One end-to-end relative L2 check against
  autograd on the true fp32 output stays as a sanity check of the whole chain.
- **Exact identities.**  Zero V on every visible key gives out = 0 under every forward E; out / lse are unchanged when rows a
  query cannot see are rewritten (future rows, rows before the window, padding, other packed sequences) with V = +-2^120; dK / dV
  of key j do not see query rows before j and dQ of row i does not see key rows after i; every window >= S - 1 (up to 2^31 - 1)
  equals window 0; permuting a batch permutes every output; packed equals padded; dO = 0 gives dqkv = 0 and delta = 0; every
  case repeats bitwise.
- **Guard bands.**  out, dqkv, lse and delta sit inside sentinel-filled buffers; everything outside the logical window keeps
  the sentinel, lse / delta beyond a packed sequence's rows stay untouched, and the backward changes none of qkv, out, dout, lse.
- **Real model geometries** on all heads, with the reference on the first, a middle and the last KV group.

The refusal contract and the checker's sensitivity (a blockwise torch emulation of the forward passes the per-element checker,
four mutations of it - a dropped rescale, the causal mask or the window edge off by one, masked weights of 2^-125 - do not)
are CPU-only tests.
"""
import ctypes as C
import math
import zlib
from dataclasses import dataclass, replace

import numpy as np
import pytest

from tests.conftest import has_gpu

gpu = pytest.mark.gpu
D = 128
DTX_ERR_INVALID, DTX_ERR_CUDA = -1, -2
U = 2.0 ** -8          # bf16 rounding (round-to-nearest: 2^-9), taken at twice its size
ACC = 2.0 ** -16       # fp32 accumulation rule, as for the GEMM
E_EX2 = 2.0 ** -21     # ex2.approx.ftz.f32
E_FMA = 7.5e-5         # cubic exp2 on the FMA pipe
LOG2E = 1.4426950408889634
LN2 = math.log(2.0)
SENT16 = 0x7FA5        # bf16 NaN sentinel
SENT32 = 0x7FC0A5A5    # fp32 NaN sentinel
G16, G32 = 4096, 256   # guard elements before and after every bf16 / fp32 output (16-byte multiples)
BIG_WINDOW = 2 ** 31 - 1

_vp, _i32, _f32 = C.c_void_p, C.c_int32, C.c_float
_HOOKS = {
    "dtx_test_attn_fwd": [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _vp, _i32, _vp, _i32, _vp],
    "dtx_test_attn_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _vp, _i32, _vp, _i32, _vp, _i32, _i32, _vp],
}


def _bind():
    from datatunerx_b200 import lib as L
    lib = L.load()
    for name, argtypes in _HOOKS.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = _i32
    return lib


def _torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def T():
    """the library with the attention test hooks bound (skips without a GPU); both exp-FMA switches are back at 0 after"""
    if not has_gpu():
        pytest.skip("no GPU")
    from datatunerx_b200 import lib as L
    lib = _bind()
    try:
        yield lib
    finally:
        L.set_option("attn_fwd_exp_fma_every", 0)
        L.set_option("attn_dq_exp_fma_every", 0)


# ---------------------------------------------------------------------------------------------------------------------------
# cases and the instantiation model
# ---------------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Case:
    B: int = 2
    S: int = 384
    H: int = 4
    Hkv: int = 2
    fwd_e: int = 0
    dq_e: int = 0
    window: int = 0
    rope: str = "none"      # none | half | glm (backward inverse rotary from a table)
    layout: str = "rect"    # rect | padded | packed
    lens: tuple = ()        # true lengths (padded / packed)
    scale: float = 1.0 / math.sqrt(128)
    inputs: str = "random"  # random | grow | shrink | peaked | zero_q


ALL_VARIANTS = frozenset(
    [("fwd", e, w) for e in (0, 2, 3, 4) for w in (False, True)]
    + [("dq", w, e) for w in (False, True) for e in (0, 3, 4)] + [("dq", False, e, "glm") for e in (0, 3, 4)]
    + [("dkv", False), ("dkv", True), ("dkv", False, "glm")])


def eff_window(c):
    return 0 if c.window >= c.S - 1 else c.window


def variant(c):
    """the instantiations one forward + backward call of c runs (the launchers' dispatch rules)"""
    win = eff_window(c) > 0
    fwd = ("fwd", c.fwd_e, win)
    if c.rope == "glm":
        assert not win
        return {fwd, ("dq", False, c.dq_e, "glm"), ("dkv", False, "glm")}
    return {fwd, ("dq", win, c.dq_e), ("dkv", win)}


GROUPS = [(2, 2), (4, 2), (5, 1), (7, 1), (16, 1)]  # g = H / Hkv in {1, 2, 5, 7, 16}
SCALES = [1.0 / math.sqrt(128), 0.03, 0.3]
INPUTS = ["random", "grow", "shrink", "peaked", "zero_q"]


def len_sets(S):
    """true lengths at every tile edge; every packed set has a 0-length sequence"""
    return [(S - 1, 0, 129), (1, S, 64), (63, 0, 127), (65, 128, 0), (S, 129, 1)]


def sweep_cases():
    out = []
    i = 0
    for layout in ("rect", "padded", "packed"):
        base = [(fe, (0, 3, 4)[j % 3], win, "none") for j, fe in enumerate((0, 2, 3, 4)) for win in (False, True)]
        base += [((0, 2, 3, 4)[j + 1], de, False, "glm") for j, de in enumerate((0, 3, 4))]
        for fe, de, win, rope in base:
            H, Hkv = GROUPS[i % len(GROUPS)]
            S = 640 if i % 4 == 3 else 384
            ls = len_sets(S)[i % 5]
            if layout == "packed" and 0 not in ls:
                ls = ls[:2] + (0,)
            # GLM runs with window 0 (its large-window identities are checked with every case)
            window = (1, 63, 64, 65, 127, 128, 129, 200)[i % 8] if win else (0 if rope == "glm" else (0, S - 1, S, BIG_WINDOW)[i % 4])
            if rope != "glm" and not win:
                rope = ("none", "half")[i % 2]
            elif rope != "glm":
                rope = ("half", "none")[i % 2]
            out.append(Case(B=3 if layout != "rect" else 2, S=S, H=H, Hkv=Hkv, fwd_e=fe, dq_e=de, window=window, rope=rope,
                            layout=layout, lens=ls if layout != "rect" else (), scale=SCALES[i % 3], inputs=INPUTS[i % 5]))
            i += 1
    # every window edge with row lengths and with packing
    for j, w in enumerate((1, 63, 64, 65, 127, 128, 129, 200, "S-1", "S", BIG_WINDOW)):
        for layout in ("padded", "packed"):
            S = 384
            ls = len_sets(S)[(j + (layout == "packed")) % 5]
            if layout == "packed" and 0 not in ls:
                ls = ls[:2] + (0,)
            H, Hkv = GROUPS[(i + j) % len(GROUPS)]
            out.append(Case(B=3, S=S, H=H, Hkv=Hkv, fwd_e=(0, 2, 3, 4)[j % 4], dq_e=(0, 3, 4)[j % 3],
                            window={"S-1": S - 1, "S": S}.get(w, w), rope=("none", "half")[j % 2], layout=layout, lens=ls,
                            scale=SCALES[j % 3], inputs=INPUTS[j % 5]))
            i += 1
    return out


def _cid(c):
    return (f"{c.layout}-g{c.H // c.Hkv}-H{c.H}-S{c.S}-fe{c.fwd_e}-de{c.dq_e}-w{c.window}-{c.rope}-{c.inputs}-s{c.scale:.3g}"
            + (f"-L{'.'.join(map(str, c.lens))}" if c.lens else ""))


SWEEP = sweep_cases()


def test_instantiation_model_covers_every_instantiation():
    """CPU-only: the sweep reaches all 20 instantiations under every layout, and covers every axis the matrix promises"""
    assert len(ALL_VARIANTS) == 20
    for layout in ("rect", "padded", "packed"):
        reached = set().union(*(variant(c) for c in SWEEP if c.layout == layout))
        assert reached == ALL_VARIANTS, (layout, sorted(ALL_VARIANTS - reached, key=str))
    assert {c.H // c.Hkv for c in SWEEP} == {1, 2, 5, 7, 16}
    assert {c.fwd_e for c in SWEEP} == {0, 2, 3, 4} and {c.dq_e for c in SWEEP} == {0, 3, 4}
    assert {c.rope for c in SWEEP} == {"none", "half", "glm"} and all(eff_window(c) == 0 for c in SWEEP if c.rope == "glm")
    assert set(INPUTS) <= {c.inputs for c in SWEEP} and {round(s, 6) for s in SCALES} == {round(c.scale, 6) for c in SWEEP}
    wins = {(c.window if c.window not in (c.S - 1, c.S) else {c.S - 1: "S-1", c.S: "S"}[c.window]) for c in SWEEP if c.lens}
    assert wins >= {1, 63, 64, 65, 127, 128, 129, 200, "S-1", "S", BIG_WINDOW}, wins
    lens = {n if n not in (c.S - 1, c.S) else {c.S - 1: "S-1", c.S: "S"}[n] for c in SWEEP for n in c.lens}
    assert lens >= {0, 1, 63, 64, 65, 127, 128, 129, "S-1", "S"}, lens
    assert all(0 in c.lens for c in SWEEP if c.layout == "packed")
    assert all(c.B <= 3 and c.S <= 640 and c.H <= 16 for c in SWEEP)


# ---------------------------------------------------------------------------------------------------------------------------
# the fp64 reference and its per-element bounds (also run on the CPU by the checker-sensitivity test)
# ---------------------------------------------------------------------------------------------------------------------------
def visible(rows, keys, window):
    """[len(rows), len(keys)] mask: key j visible from query i iff j <= i and (window == 0 or j >= i - window)"""
    vis = keys[None, :] <= rows[:, None]
    if window > 0:
        vis &= keys[None, :] >= rows[:, None] - window
    return vis


def reference(q, k, v, scale, window, e_fwd, do=None, out_k=None, lse_k=None, e_bwd=0.0, chunk=1024):
    """fp64 attention of one sequence for one KV group and its per-element bounds.  q, do, out_k [g, n, D]; k, v [n, D];
    lse_k [g, n] (the kernel's log2-domain lse).  The backward part (do given) is driven by the kernel's out_k and lse_k.
    Query rows are processed in chunks of `chunk` so the fp64 score blocks stay small."""
    torch = _torch()
    g, n, _ = q.shape
    sl = float(np.float32(scale)) * LOG2E
    sc = float(np.float32(scale))
    q, k, v = q.double(), k.double(), v.double()
    dev = q.device
    r = {"out": torch.zeros(g, n, D, dtype=torch.float64, device=dev), "lse": torch.zeros(g, n, dtype=torch.float64, device=dev)}
    r["out_bd"], r["lse_bd"] = torch.zeros_like(r["out"]), torch.zeros_like(r["lse"])
    bwd = do is not None
    if bwd:
        do, out_k, lse_k = do.double(), out_k.double(), lse_k.double()
        for name in ("dq", "dq_bd", "dq_mag"):
            r[name] = torch.zeros(g, n, D, dtype=torch.float64, device=dev)
        for name in ("dk", "dk_bd", "dk_mag", "dv", "dv_bd"):
            r[name] = torch.zeros(n, D, dtype=torch.float64, device=dev)
        r["delta"] = (do * out_k).sum(-1)
        r["delta_bd"] = 2.0 ** -17 * (do * out_k).abs().sum(-1)
    for r0 in range(0, n, chunk):
        r1 = min(n, r0 + chunk)
        k0 = max(0, r0 - window) if window > 0 else 0
        rows, keys = torch.arange(r0, r1, device=dev), torch.arange(k0, r1, device=dev)
        vis = visible(rows, keys, window)[None]                       # [1, c, m]
        qc, kc, vc = q[:, r0:r1], k[k0:r1], v[k0:r1]
        t = (qc @ kc.T) * sl                                          # [g, c, m] scaled scores, log2 units
        dt = sl * ACC * (qc.abs() @ kc.abs().T) + 2.0 ** -22 * t.abs()
        t = t.masked_fill(~vis, -math.inf)
        dt = dt.masked_fill(~vis, 0.0)
        nvis = vis.sum(-1).double()                                   # [1, c]
        e_row = e_fwd + LN2 * dt.amax(-1) + (nvis / 64 + 2) * E_EX2 + nvis * 2.0 ** -24
        m = t.amax(-1, keepdim=True)
        m = torch.where(torch.isinf(m), torch.zeros_like(m), m)
        p = torch.exp2(t - m)
        l = p.sum(-1, keepdim=True)
        ph = p / l
        out = ph @ vc
        pv = ph @ vc.abs()
        r["out"][:, r0:r1] = out
        r["out_bd"][:, r0:r1] = (U + 2 * e_row[..., None]) * pv + U * out.abs()
        lse = (m + torch.log2(l)).squeeze(-1)
        r["lse"][:, r0:r1] = lse
        r["lse_bd"][:, r0:r1] = 1.5 * e_row + 2.0 ** -21 * (m.squeeze(-1).abs() + lse.abs() + 1)
        if not bwd:
            continue
        doc = do[:, r0:r1]
        P = torch.exp2(t - lse_k[:, r0:r1, None]).masked_fill(~vis, 0.0)
        e_p = e_bwd + LN2 * dt                                       # relative error of the kernel's P, per element
        dP = doc @ vc.T
        dP_err = ACC * (doc.abs() @ vc.abs().T)
        dl = r["delta"][:, r0:r1, None]
        ddl = r["delta_bd"][:, r0:r1, None]
        dS = P * (dP - dl) * sc
        ddS = U * dS.abs() + sc * P * (e_p * (dP.abs() + dl.abs()) + dP_err + ddl + 2.0 ** -22 * (dP.abs() + dl.abs()))
        r["dq"][:, r0:r1] = dS @ kc
        r["dq_bd"][:, r0:r1] = ddS @ kc.abs() + ACC * (dS.abs() @ kc.abs())
        r["dq_mag"][:, r0:r1] = dS.abs() @ kc.abs()
        r["dk"][k0:r1] += torch.einsum("gcm,gcd->md", dS, qc)
        r["dk_bd"][k0:r1] += torch.einsum("gcm,gcd->md", ddS + ACC * dS.abs(), qc.abs())
        r["dk_mag"][k0:r1] += torch.einsum("gcm,gcd->md", dS.abs(), qc.abs())
        r["dv"][k0:r1] += torch.einsum("gcm,gcd->md", P, doc)
        r["dv_bd"][k0:r1] += torch.einsum("gcm,gcd->md", (U + e_p + ACC) * P, doc.abs())
    return r


def inverse_rotary(x, bd, mag, cs_t, pos, glm):
    """fp64 inverse rotary of x [..., n, D] at positions pos from the transposed table cs_t [nf, stride, 2], with the bounds
    pushed through |R| and the rounding of the rotation itself (relative 2^-22 of |R| |x|)"""
    torch = _torch()
    t = cs_t.double()[:, pos]                     # [nf, n, 2]
    c, s = t[..., 0].T, t[..., 1].T               # [n, nf]
    y, yb, ym = x.clone(), bd.clone(), mag.clone()
    if glm:
        i0, i1 = slice(0, 64, 2), slice(1, 64, 2)
    else:
        i0, i1 = slice(0, 64), slice(64, 128)
    x0, x1, b0, b1, m0, m1 = x[..., i0], x[..., i1], bd[..., i0], bd[..., i1], mag[..., i0], mag[..., i1]
    y[..., i0], y[..., i1] = x0 * c + x1 * s, x1 * c - x0 * s
    yb[..., i0] = c.abs() * b0 + s.abs() * b1 + 2.0 ** -22 * (c.abs() * m0 + s.abs() * m1)
    yb[..., i1] = c.abs() * b1 + s.abs() * b0 + 2.0 ** -22 * (c.abs() * m1 + s.abs() * m0)
    ym[..., i0], ym[..., i1] = c.abs() * m0 + s.abs() * m1, c.abs() * m1 + s.abs() * m0
    return y, yb, ym


def _where(bad, err, bd, what):
    idx = bad.nonzero()
    first = tuple(int(i) for i in idx[0])
    ratio = float((err[bad] / bd[bad].clamp(min=1e-300)).max())
    return f"{what}: {idx.shape[0]} elements beyond their bound, first at {first} (worst error / bound {ratio:.3g})"


WORST = {}


def assert_within(got, ref, bd, what, key="sweep"):
    err = (got.double() - ref).abs()
    bad = ~(err <= bd)
    if bool(bad.any()):
        raise AssertionError(_where(bad, err, bd, what))
    if bd.numel():
        k = (key, what.rsplit(": ", 1)[-1])
        WORST[k] = max(WORST.get(k, 0.0), float((err / bd.clamp(min=1e-300)).max()))


# ---------------------------------------------------------------------------------------------------------------------------
# checker sensitivity (CPU): a blockwise emulation of the forward passes, its mutations do not
# ---------------------------------------------------------------------------------------------------------------------------
def emulate_fwd(q, k, v, scale, window, drop_rescale_block=None, causal_shift=0, window_shift=0, masked_weight=0.0):
    """the forward kernel's arithmetic in torch for one head: 64-row warpgroups, 64-key blocks up to the diagonal, fp32 scores,
    running max / sum with rescale factors, bf16-rounded P, fp32 P V, bf16 output.  The keyword arguments inject the defects the
    per-element checker exists to catch."""
    torch = _torch()
    n = q.shape[0]
    sl = float(np.float32(np.float32(scale) * np.float32(LOG2E)))
    qf, kf, vf = q.float(), k.float(), v.float()
    out = torch.zeros(n, D, dtype=torch.bfloat16)
    lse = torch.zeros(n, dtype=torch.float32)
    for w0 in range(0, n, 64):
        rows = torch.arange(w0, w0 + 64)
        o = torch.zeros(64, D)
        m_run = torch.full((64,), -math.inf)
        l_run = torch.zeros(64)
        jlo = max(0, (w0 // 128 * 128 - window) // 64) if window else 0
        for jb in range(jlo, w0 // 64 + 1):
            keys = torch.arange(jb * 64, jb * 64 + 64)
            s = qf[w0:w0 + 64] @ kf[jb * 64:jb * 64 + 64].T
            hide = keys[None, :] > rows[:, None] + causal_shift
            if window:
                hide |= keys[None, :] < rows[:, None] - window - window_shift
            s = s.masked_fill(hide, -math.inf)
            mx = s.amax(-1) * sl
            m_new = torch.maximum(m_run, mx)
            m_use = torch.where(torch.isinf(m_new), torch.zeros_like(m_new), m_new)
            alpha = torch.exp2(m_run - m_use)
            m_run = m_new
            p = torch.exp2(s * sl - m_use[:, None])
            if masked_weight:
                p = torch.where(hide, torch.full_like(p, masked_weight), p)
            l_run = l_run * alpha + p.sum(-1)
            if jb != drop_rescale_block:
                o = o * alpha[:, None]
            o = o + p.to(torch.bfloat16).float() @ vf[jb * 64:jb * 64 + 64]
        out[w0:w0 + 64] = (o * (1.0 / l_run)[:, None]).to(torch.bfloat16)
        lse[w0:w0 + 64] = m_run + torch.log2(l_run)
    return out, lse


def report(key):
    worst = {q: f"{v:.3f}" for (k, q), v in sorted(WORST.items()) if k == key}
    print(f"\n[bounds] {key}: worst error / bound per output {worst}")


def _fwd_checker_passes(q, k, v, scale, window, out, lse):
    r = reference(q[None], k, v, scale, window, 0.0)
    try:
        assert_within(out[None], r["out"], r["out_bd"], "out", key="emulation")
        assert_within(lse[None], r["lse"], r["lse_bd"], "lse", key="emulation")
    except AssertionError:
        return False
    return True


def test_checker_sensitivity():
    """CPU-only: the per-element checker accepts the blockwise emulation of the forward (random, growing-score and windowed
    inputs) and rejects each defect it exists to catch: one block's rescale factor dropped, the causal mask or the window edge
    off by one, and masked keys with weight 2^-125 instead of 0."""
    torch = _torch()
    n, scale = 256, 1.0 / math.sqrt(128)
    g = torch.Generator().manual_seed(3)
    q, k, v = (torch.randn(n, D, generator=g).to(torch.bfloat16) for _ in range(3))
    u = torch.ones(D) / math.sqrt(D)
    qg = (4.0 * u + 0.1 * torch.randn(n, D, generator=g)).to(torch.bfloat16)
    kg = ((12.0 / 64) / (4.0 * scale) * torch.arange(n)[:, None] * u + 0.1 * torch.randn(n, D, generator=g)).to(torch.bfloat16)
    vz = v.clone()
    vz[:96] = 0
    vz[96:128] = (2.0 ** 120) * torch.sign(torch.randn(32, D, generator=g))  # rows 64..95 see only V = 0
    for qq, kk, vv, w in ((q, k, v, 0), (qg, kg, v, 0), (q, k, v, 64), (q, k, vz, 0)):
        assert _fwd_checker_passes(qq, kk, vv, scale, w, *emulate_fwd(qq, kk, vv, scale, w)), "the checker rejects the emulation"
    mutants = {
        "rescale factor of block 2 dropped": (qg, kg, v, 0, dict(drop_rescale_block=2)),
        "causal mask off by one": (q, k, v, 0, dict(causal_shift=1)),
        "window edge off by one": (q, k, v, 64, dict(window_shift=1)),
        "masked weights 2^-125": (q, k, vz, 0, dict(masked_weight=2.0 ** -125)),
    }
    for what, (qq, kk, vv, w, kw) in mutants.items():
        assert not _fwd_checker_passes(qq, kk, vv, scale, w, *emulate_fwd(qq, kk, vv, scale, w, **kw)), f"checker accepts: {what}"
    report("emulation")


# ---------------------------------------------------------------------------------------------------------------------------
# the refusal contract without a GPU
# ---------------------------------------------------------------------------------------------------------------------------
def test_refusals_without_gpu():
    """CPU-only: the attention launchers validate every argument before any CUDA call, so each rule's defect returns
    DTX_ERR_INVALID on fake (16-byte aligned) device addresses while the same call without it gets past validation (DTX_ERR_CUDA:
    no device).  Skipped where a GPU is visible: the valid calls would launch on the fake addresses there."""
    if has_gpu():
        pytest.skip("a GPU is visible")
    lib = _bind()
    F = 1 << 40

    def fwd(qkv=F, out=F, B=2, S=256, H=4, Hkv=2, scale=0.088, window=0, rs=None, total=0, entry="public"):
        if entry == "public":
            return lib.dtx_attn_fwd(qkv, out, F, B, S, H, Hkv, scale, None, window, None)
        return lib.dtx_test_attn_fwd(qkv, out, F, B, S, H, Hkv, scale, None, window, rs, total, None)

    def bwd(qkv=F, out=F, dout=F, lse=F, delta=F, dqkv=F, B=2, S=256, H=4, Hkv=2, scale=0.088, window=0, cs=None, stride=0, glm=0,
            rs=None, total=0, entry="public"):
        if entry == "public":
            return lib.dtx_attn_bwd_rope(qkv, out, dout, lse, delta, dqkv, B, S, H, Hkv, scale, None, window, cs, stride, glm, None)
        return lib.dtx_test_attn_bwd(qkv, out, dout, lse, delta, dqkv, B, S, H, Hkv, scale, None, window, rs, total, cs, stride, glm,
                                     None)

    both = []
    for name, f in (("fwd", fwd), ("bwd", bwd)):
        both += [
            (f"{name}: S % 128", lambda f=f: f(), lambda f=f: f(S=200)),
            (f"{name}: S <= 0", lambda f=f: f(), lambda f=f: f(S=-128)),
            (f"{name}: B <= 0", lambda f=f: f(), lambda f=f: f(B=0)),
            (f"{name}: H <= 0", lambda f=f: f(), lambda f=f: f(H=0)),
            (f"{name}: Hkv < 0", lambda f=f: f(Hkv=0), lambda f=f: f(Hkv=-2)),
            (f"{name}: H % Hkv", lambda f=f: f(), lambda f=f: f(Hkv=3)),
            (f"{name}: window < 0", lambda f=f: f(window=5), lambda f=f: f(window=-1)),
            (f"{name}: scale 0", lambda f=f: f(), lambda f=f: f(scale=0.0)),
            (f"{name}: negative scale", lambda f=f: f(), lambda f=f: f(scale=-0.088)),
            (f"{name}: NaN scale", lambda f=f: f(), lambda f=f: f(scale=float("nan"))),
            (f"{name}: infinite scale", lambda f=f: f(), lambda f=f: f(scale=float("inf"))),
            (f"{name}: row_start with total_rows 0", lambda f=f: f(rs=F, total=512, entry="test"),
             lambda f=f: f(rs=F, total=0, entry="test")),
            (f"{name}: row_start with total_rows % 128", lambda f=f: f(rs=F, total=512, entry="test"),
             lambda f=f: f(rs=F, total=500, entry="test")),
            (f"{name}: null qkv", lambda f=f: f(), lambda f=f: f(qkv=None)),
            (f"{name}: misaligned qkv", lambda f=f: f(), lambda f=f: f(qkv=F + 8)),
            (f"{name}: null out", lambda f=f: f(), lambda f=f: f(out=None)),
            (f"{name}: misaligned out", lambda f=f: f(), lambda f=f: f(out=F + 2)),
        ]
    cases = both + [
        ("bwd: rope_glm 2", lambda: bwd(cs=F, glm=1), lambda: bwd(cs=F, glm=2)),
        ("bwd: rope_glm -1", lambda: bwd(), lambda: bwd(glm=-1)),
        ("bwd: GLM with a window", lambda: bwd(cs=F, glm=1, window=255), lambda: bwd(cs=F, glm=1, window=100)),
        ("bwd: rope_stride in (0, S) with a table", lambda: bwd(cs=F, stride=256), lambda: bwd(cs=F, stride=128)),
        ("bwd: GLM rope_stride in (0, S)", lambda: bwd(cs=F, glm=1, stride=384), lambda: bwd(cs=F, glm=1, stride=255)),
        ("bwd: without lse", lambda: bwd(), lambda: bwd(lse=None)),
        ("bwd: without dout", lambda: bwd(), lambda: bwd(dout=None)),
        ("bwd: without delta", lambda: bwd(), lambda: bwd(delta=None)),
        ("bwd: without dqkv", lambda: bwd(), lambda: bwd(dqkv=None)),
        ("bwd: misaligned dqkv", lambda: bwd(), lambda: bwd(dqkv=F + 8)),
        ("bwd: misaligned lse", lambda: bwd(), lambda: bwd(lse=F + 4)),
    ]
    for what, good, bad in cases:
        rc = good()
        assert rc == DTX_ERR_CUDA, f"{what}: the call without the defect returned {rc}, expected DTX_ERR_CUDA (past validation)"
        assert bad() == DTX_ERR_INVALID, f"{what}: not refused before device work"
    # a window of S - 1 or more is plain causal attention, so GLM takes it, and a rope_stride without a table is not checked
    assert bwd(cs=F, glm=1, window=BIG_WINDOW) == DTX_ERR_CUDA
    assert bwd(stride=5) == DTX_ERR_CUDA


# ---------------------------------------------------------------------------------------------------------------------------
# GPU plumbing: layouts, guarded buffers, calls
# ---------------------------------------------------------------------------------------------------------------------------
def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def ST():
    return C.c_void_p(_torch().cuda.current_stream().cuda_stream)


class Guarded:
    """a flat window of n elements with `guard` sentinel elements before and after it"""

    def __init__(self, n, f32, guard=None):
        torch = _torch()
        self.n, self.f32 = n, f32
        self.g = guard if guard is not None else (G32 if f32 else G16)
        self.sent = SENT32 if f32 else SENT16
        self.bits = torch.full((n + 2 * self.g,), self.sent, dtype=torch.int32 if f32 else torch.int16, device="cuda")
        self.win_bits = self.bits[self.g:self.g + n]
        self.win = self.win_bits.view(torch.float32 if f32 else torch.bfloat16)

    def assert_guard(self, what):
        assert bool((self.bits[:self.g] == self.sent).all()) and bool((self.bits[self.g + self.n:] == self.sent).all()), \
            f"{what}: guard elements written"

    def assert_untouched(self, what):
        assert bool((self.bits == self.sent).all()), f"{what}: a refused call wrote its output"


class Batch:
    """sequences (each [S, W] qkv and [S, H*D] dO rows, true length) laid out as c.layout: rect / padded rows of S, or packed at
    the rows plan_packed_rows gives (caps: S, or the length rounded up to 128 with at least 128 rows)"""

    def __init__(self, c, seqs, douts, lens):
        torch = _torch()
        from datatunerx_b200 import lib as L
        self.c, self.lens = c, list(lens)
        B, S = len(seqs), c.S
        if c.layout == "packed":
            starts, _ = L.plan_packed_rows(np.array(lens, np.int32), S)
        else:
            starts = [b * S for b in range(B + 1)]
        self.starts = [int(s) for s in starts]
        self.caps = [self.starts[b + 1] - self.starts[b] for b in range(B)]
        self.M = self.starts[-1]
        self.qkv = torch.cat([s[:cap] for s, cap in zip(seqs, self.caps)]).contiguous()
        self.dout = torch.cat([d[:cap] for d, cap in zip(douts, self.caps)]).contiguous()
        self.seq_lens = torch.tensor(lens, dtype=torch.int32, device="cuda") if c.layout != "rect" else None
        self.row_start = torch.tensor(self.starts, dtype=torch.int32, device="cuda") if c.layout == "packed" else None

    def live(self, b):
        """rows of sequence b in tiles that hold a real token"""
        return min(self.caps[b], (self.lens[b] + 127) // 128 * 128)


def rope_table(c, seed):
    """random transposed rotary table [nf][stride] (cos, sin), stride >= S"""
    torch = _torch()
    if c.rope == "none":
        return None, 0
    nf = 32 if c.rope == "glm" else 64
    stride = c.S + (128 if c.rope == "half" else 0)
    g = torch.Generator(device="cuda").manual_seed(seed)
    ang = torch.rand((nf, stride), generator=g, device="cuda") * (2 * math.pi)
    return torch.stack([torch.cos(ang), torch.sin(ang)], dim=-1).contiguous(), stride


def make_seq(c, seed, n=None):
    """one sequence of S rows: qkv [S, W] bf16 of the case's input class and dO [S, H*D]"""
    torch = _torch()
    n = n or c.S
    H, Hkv = c.H, c.Hkv
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, H + 2 * Hkv, D, generator=g, device="cuda")
    u = torch.ones(D, device="cuda") / math.sqrt(D)
    pos = torch.arange(n, device="cuda", dtype=torch.float32)[:, None, None]
    if c.inputs in ("grow", "shrink"):  # scaled scores move by ~12 natural units per 64 keys
        rate = (12.0 / 64) / (4.0 * c.scale) * (1 if c.inputs == "grow" else -1)
        x[:, :H] = 4.0 * u + 0.1 * x[:, :H]
        x[:, H:H + Hkv] = rate * pos * u + 0.1 * x[:, H:H + Hkv]
    elif c.inputs == "peaked":  # scaled logits with a spread of about +-40
        x[:, :H] *= (40.0 / 3) / (math.sqrt(D) * c.scale)
    elif c.inputs == "zero_q":
        x[:, :H] = 0
    do = torch.randn(n, H * D, generator=g, device="cuda")
    return x.reshape(n, -1).to(torch.bfloat16), do.to(torch.bfloat16)


def make_batch(c, seed=0):
    lens = list(c.lens) if c.lens else [c.S] * c.B
    seqs, douts = [], []
    for b, n in enumerate(lens):
        q, d = make_seq(c, seed + 17 * b)
        d[n:] = 0  # the loss never reaches a padding token
        seqs.append(q)
        douts.append(d)
    return Batch(c, seqs, douts, lens)


class Run:
    """one forward + backward of a batch with every output in a guarded buffer"""

    def __init__(self, T, c, bt, window=None, cs=None, stride=0, dout=None, check=True):
        torch = _torch()
        from datatunerx_b200 import lib as L
        H, Hkv, S, B = c.H, c.Hkv, c.S, len(bt.lens)
        W = (H + 2 * Hkv) * D
        window = c.window if window is None else window
        dout = bt.dout if dout is None else dout
        self.out, self.dqkv = Guarded(bt.M * H * D, False), Guarded(bt.M * W, False)
        self.lse, self.delta = Guarded(B * H * S, True), Guarded(B * H * S, True)
        q0, d0 = bt.qkv.clone(), dout.clone()
        L.set_option("attn_fwd_exp_fma_every", c.fwd_e)
        L.set_option("attn_dq_exp_fma_every", c.dq_e)
        try:
            glm = int(c.rope == "glm")
            if bt.row_start is None:
                rc = T.dtx_attn_fwd(P(bt.qkv), P(self.out.win), P(self.lse.win), B, S, H, Hkv, c.scale, P(bt.seq_lens), window, ST())
            else:
                rc = T.dtx_test_attn_fwd(P(bt.qkv), P(self.out.win), P(self.lse.win), B, S, H, Hkv, c.scale, P(bt.seq_lens), window,
                                         P(bt.row_start), bt.M, ST())
            assert rc == 0, f"{c}: forward returned {rc}"
            torch.cuda.synchronize()
            o0, l0 = self.out.bits.clone(), self.lse.bits.clone()
            if bt.row_start is None:
                rc = T.dtx_attn_bwd_rope(P(bt.qkv), P(self.out.win), P(dout), P(self.lse.win), P(self.delta.win), P(self.dqkv.win), B,
                                         S, H, Hkv, c.scale, P(bt.seq_lens), window, P(cs), stride, glm, ST())
            else:
                rc = T.dtx_test_attn_bwd(P(bt.qkv), P(self.out.win), P(dout), P(self.lse.win), P(self.delta.win), P(self.dqkv.win), B,
                                         S, H, Hkv, c.scale, P(bt.seq_lens), window, P(bt.row_start), bt.M, P(cs), stride, glm, ST())
            assert rc == 0, f"{c}: backward returned {rc}"
            torch.cuda.synchronize()
        finally:
            L.set_option("attn_fwd_exp_fma_every", 0)
            L.set_option("attn_dq_exp_fma_every", 0)
        if check:
            what = _cid(c)
            for name in ("out", "dqkv", "lse", "delta"):
                getattr(self, name).assert_guard(f"{what}: {name}")
            assert torch.equal(bt.qkv.view(torch.int16), q0.view(torch.int16)), f"{what}: the backward changed qkv"
            assert torch.equal(dout.view(torch.int16), d0.view(torch.int16)), f"{what}: the backward changed dout"
            assert torch.equal(self.out.bits, o0), f"{what}: the backward changed out"
            assert torch.equal(self.lse.bits, l0), f"{what}: the backward changed lse"
        self.W, self.H, self.S, self.B = W, H, S, B

    def o(self):
        return self.out.win.view(-1, self.H * D)

    def g(self):
        return self.dqkv.win.view(-1, self.W)

    def stat(self, which):
        return getattr(self, which).win.view(self.B, self.H, self.S)

    def bits(self):
        return [x.bits.clone() for x in (self.out, self.lse, self.delta, self.dqkv)]


def assert_bits(a, b, what):
    torch = _torch()
    x, y = a.contiguous().view(torch.int16 if a.element_size() == 2 else torch.int32), \
        b.contiguous().view(torch.int16 if b.element_size() == 2 else torch.int32)
    bad = x != y
    if bool(bad.any()):
        raise AssertionError(f"{what}: {int(bad.sum())} elements differ, first at {tuple(int(i) for i in bad.nonzero()[0])}")


def seq_view(r, bt, b):
    """(out [cap, H*D], dqkv [cap, W], lse [H, S], delta [H, S]) of sequence b"""
    r0, cap = bt.starts[b], bt.caps[b]
    return r.o()[r0:r0 + cap], r.g()[r0:r0 + cap], r.stat("lse")[b], r.stat("delta")[b]


# ---------------------------------------------------------------------------------------------------------------------------
# checks of one run against the fp64 reference
# ---------------------------------------------------------------------------------------------------------------------------
def check_reference(c, bt, r, cs, groups=None, key="sweep", chunk=1024):
    """out, lse, delta, dq, dk, dv of every sequence (and of the KV groups in `groups`, default all) within their bounds;
    tiles beyond a sequence's length zero (out, lse, delta, dqkv), lse / delta beyond its rows untouched"""
    torch = _torch()
    H, Hkv = c.H, c.Hkv
    g = H // Hkv
    window = eff_window(c)
    e_fwd = (E_FMA if c.fwd_e else 0.0) + E_EX2
    e_bwd = (E_FMA if c.dq_e else 0.0) + E_EX2
    groups = range(Hkv) if groups is None else groups
    for b in range(len(bt.lens)):
        out, dqkv, lse, delta = seq_view(r, bt, b)
        cap, live = bt.caps[b], bt.live(b)
        what = f"{_cid(c)} seq {b} (len {bt.lens[b]})"
        if cap < c.S:
            assert bool(torch.isnan(lse[:, cap:]).all()) and bool(torch.isnan(delta[:, cap:]).all()), \
                f"{what}: lse / delta written beyond the sequence's rows"
        if live < cap:
            assert float(out[live:].float().abs().max()) == 0.0 and float(dqkv[live:].float().abs().max()) == 0.0, \
                f"{what}: padding tiles not zero"
            assert float(lse[:, live:cap].abs().max()) == 0.0 and float(delta[:, live:cap].abs().max()) == 0.0, \
                f"{what}: lse / delta of padding tiles not zero"
        if live == 0:
            continue
        x = bt.qkv[bt.starts[b]:bt.starts[b] + live].view(live, H + 2 * Hkv, D)
        do = bt.dout[bt.starts[b]:bt.starts[b] + live].view(live, H, D)
        ok_ = out[:live].view(live, H, D)
        pos = torch.arange(live, device="cuda")
        for hk in groups:
            hs = slice(hk * g, hk * g + g)
            rf = reference(x[:, hs].transpose(0, 1), x[:, H + hk], x[:, H + Hkv + hk], c.scale, window, e_fwd,
                           do[:, hs].transpose(0, 1), ok_[:, hs].transpose(0, 1), lse[hs, :live], e_bwd, chunk=chunk)
            w = f"{what} kv group {hk}"
            assert_within(ok_[:, hs].transpose(0, 1), rf["out"], rf["out_bd"], w + ": out", key)
            assert_within(lse[hs, :live], rf["lse"], rf["lse_bd"], w + ": lse", key)
            assert_within(delta[hs, :live], rf["delta"], rf["delta_bd"], w + ": delta", key)
            dq, dq_bd, dq_mag = rf["dq"], rf["dq_bd"], rf["dq_mag"]
            dk, dk_bd, dk_mag = rf["dk"], rf["dk_bd"], rf["dk_mag"]
            if cs is not None:
                dq, dq_bd, _ = inverse_rotary(dq, dq_bd, dq_mag, cs, pos, c.rope == "glm")
                dk, dk_bd, _ = inverse_rotary(dk, dk_bd, dk_mag, cs, pos, c.rope == "glm")
            gq = dqkv[:live].view(live, H + 2 * Hkv, D)
            assert_within(gq[:, hs].transpose(0, 1), dq, dq_bd + U * dq.abs(), w + ": dq", key)
            assert_within(gq[:, H + hk], dk, dk_bd + U * dk.abs(), w + ": dk", key)
            assert_within(gq[:, H + Hkv + hk], rf["dv"], rf["dv_bd"] + U * rf["dv"].abs(), w + ": dv", key)


def run_case(T, c, seed=0):
    bt = make_batch(c, seed)
    cs, stride = rope_table(c, seed + 5)
    return bt, cs, stride, Run(T, c, bt, cs=cs, stride=stride)


def permuted(c, bt, perm):
    seqs = [bt_seq(bt, b) for b in perm]
    return Batch(c, [s[0] for s in seqs], [s[1] for s in seqs], [bt.lens[b] for b in perm])


def bt_seq(bt, b):
    """sequence b of a batch padded back to S rows (rows beyond its cap: zeros)"""
    torch = _torch()
    S = bt.c.S
    q = torch.zeros(S, bt.qkv.shape[1], dtype=torch.bfloat16, device="cuda")
    d = torch.zeros(S, bt.dout.shape[1], dtype=torch.bfloat16, device="cuda")
    r0, cap = bt.starts[b], bt.caps[b]
    q[:cap], d[:cap] = bt.qkv[r0:r0 + cap], bt.dout[r0:r0 + cap]
    return q, d


def rewrite_rows(c, bt, rows_of, seed, v_big=True, cols="qkv"):
    """a copy of the batch with the rows rows_of(b) -> (lo, hi) of every sequence b rewritten: q / k random x4, V = +-2^120 (or
    random x4 with v_big False); cols "qkv", "kv" or "qdo" (q and dO)"""
    torch = _torch()
    H, Hkv = c.H, c.Hkv
    qkv, dout = bt.qkv.clone(), bt.dout.clone()
    g = torch.Generator(device="cuda").manual_seed(seed)
    for b in range(len(bt.lens)):
        lo, hi = rows_of(b)
        lo, hi = max(lo, 0), min(hi, bt.caps[b])
        if hi <= lo:
            continue
        x = qkv[bt.starts[b] + lo:bt.starts[b] + hi].view(hi - lo, H + 2 * Hkv, D)
        rnd = lambda *s: (4 * torch.randn(*s, generator=g, device="cuda")).to(torch.bfloat16)
        if cols in ("qkv", "qdo"):
            x[:, :H] = rnd(hi - lo, H, D)
        if cols in ("qkv", "kv"):
            x[:, H:H + Hkv] = rnd(hi - lo, Hkv, D)
            if v_big:
                x[:, H + Hkv:] = ((2.0 ** 120) * torch.sign(torch.randn(hi - lo, Hkv, D, generator=g, device="cuda"))).to(torch.bfloat16)
            else:
                x[:, H + Hkv:] = rnd(hi - lo, Hkv, D)
        if cols == "qdo":
            dout[bt.starts[b] + lo:bt.starts[b] + hi] = rnd(hi - lo, H * D).view(hi - lo, H * D)
    nb = Batch.__new__(Batch)
    nb.__dict__.update(bt.__dict__)
    nb.qkv, nb.dout = qkv, dout
    return nb


def rows_slice(r, bt, b, lo, hi, which):
    r0 = bt.starts[b]
    if which == "out":
        return r.o()[r0 + lo:r0 + hi]
    return r.stat(which)[b][:, lo:hi]


def check_identities(T, c, bt, cs, stride, base):
    """the exact identities of one case (see the module docstring)"""
    torch = _torch()
    H, Hkv = c.H, c.Hkv
    what = _cid(c)
    B = len(bt.lens)
    live = [bt.live(b) for b in range(B)]
    # repeatability
    again = Run(T, c, bt, cs=cs, stride=stride)
    for x, y, n in zip(base.bits(), again.bits(), ("out", "lse", "delta", "dqkv")):
        assert torch.equal(x, y), f"{what}: {n} does not repeat bitwise"
    # dO = 0: no gradient, delta 0
    z = Run(T, c, bt, cs=cs, stride=stride, dout=torch.zeros_like(bt.dout))
    for b in range(B):
        _, dq, _, dl = seq_view(z, bt, b)
        assert float(dq.float().abs().max()) == 0.0, f"{what}: seq {b}: dO = 0 gives a gradient"
        assert float(dl[:, :bt.caps[b]].abs().max()) == 0.0, f"{what}: seq {b}: dO = 0 gives delta != 0"
    # every window >= S - 1 equals window 0
    if eff_window(c) == 0:
        ref = Run(T, c, bt, window=0, cs=cs, stride=stride).bits() if c.window else base.bits()
        for w in (c.S - 1, c.S, BIG_WINDOW):
            got = Run(T, replace(c, window=w), bt, cs=cs, stride=stride).bits()
            for x, y, n in zip(ref, got, ("out", "lse", "delta", "dqkv")):
                assert torch.equal(x, y), f"{what}: window {w}: {n} differs from window 0"
    # forward isolation: future rows, rows before the window, padding
    cut = [min(live[b], 100) for b in range(B)]
    fut = Run(T, c, rewrite_rows(c, bt, lambda b: (cut[b] + 1, bt.caps[b]), 71), cs=cs, stride=stride, check=False)
    for b in range(B):
        for n in ("out", "lse"):
            assert_bits(rows_slice(fut, bt, b, 0, cut[b] + 1, n), rows_slice(base, bt, b, 0, cut[b] + 1, n),
                        f"{what}: seq {b}: {n} of rows <= {cut[b]} with the rows after them rewritten")
    w = eff_window(c)
    if w:
        c2 = [min(live[b], w + 150) for b in range(B)]
        past = Run(T, c, rewrite_rows(c, bt, lambda b: (0, c2[b] - w), 72), cs=cs, stride=stride, check=False)
        for b in range(B):
            if c2[b] - w > 0:
                for n in ("out", "lse"):
                    assert_bits(rows_slice(past, bt, b, c2[b], live[b], n), rows_slice(base, bt, b, c2[b], live[b], n),
                                f"{what}: seq {b}: {n} of rows >= {c2[b]} with the rows before their window rewritten")
    if c.layout != "rect":
        pad = Run(T, c, rewrite_rows(c, bt, lambda b: (bt.lens[b], bt.caps[b]), 73), cs=cs, stride=stride, check=False)
        for b in range(B):
            for n in ("out", "lse"):
                assert_bits(rows_slice(pad, bt, b, 0, bt.lens[b], n), rows_slice(base, bt, b, 0, bt.lens[b], n),
                            f"{what}: seq {b}: {n} of the real rows with the padding rewritten")
    # other sequences: rewrite every sequence but the first
    oth = Run(T, c, rewrite_rows(c, bt, lambda b: (0, bt.caps[b]) if b else (0, 0), 74), cs=cs, stride=stride, check=False)
    o0, g0, l0, d0 = seq_view(oth, bt, 0)
    o1, g1, l1, d1 = seq_view(base, bt, 0)
    assert_bits(o0, o1, f"{what}: seq 0 out with the other sequences rewritten")
    assert_bits(l0, l1, f"{what}: seq 0 lse with the other sequences rewritten")
    # backward isolation: dK / dV of keys >= cut do not see query rows before cut; dQ of rows <= cut does not see keys after it
    W = (H + 2 * Hkv) * D
    qb = Run(T, c, rewrite_rows(c, bt, lambda b: (0, cut[b]), 75, cols="qdo"), cs=cs, stride=stride, check=False)
    kb = Run(T, c, rewrite_rows(c, bt, lambda b: (cut[b] + 1, bt.caps[b]), 76, v_big=False, cols="kv"), cs=cs, stride=stride,
             check=False)
    for b in range(B):
        r0 = bt.starts[b]
        assert_bits(qb.g()[r0 + cut[b]:r0 + live[b], H * D:], base.g()[r0 + cut[b]:r0 + live[b], H * D:],
                    f"{what}: seq {b}: dk / dv of keys >= {cut[b]} with the query rows before them rewritten")
        assert_bits(kb.g()[r0:r0 + cut[b] + 1, :H * D], base.g()[r0:r0 + cut[b] + 1, :H * D],
                    f"{what}: seq {b}: dq of rows <= {cut[b]} with the key rows after them rewritten")
    # batch permutation (sequences with their lengths)
    perm = list(reversed(range(B)))
    pb = permuted(c, bt, perm)
    pr = Run(T, c, pb, cs=cs, stride=stride)
    for i, b in enumerate(perm):
        for x, y, n in zip(seq_view(pr, pb, i), seq_view(base, bt, b), ("out", "dqkv", "lse", "delta")):
            if n in ("lse", "delta"):
                x, y = x[:, :bt.caps[b]], y[:, :bt.caps[b]]
            assert_bits(x, y, f"{what}: permuted batch, seq {b} -> {i}: {n}")
    # packed equals padded
    if c.layout == "packed":
        pc = replace(c, layout="padded")
        pd = Batch(pc, [bt_seq(bt, b)[0] for b in range(B)], [bt_seq(bt, b)[1] for b in range(B)], bt.lens)
        rp = Run(T, pc, pd, cs=cs, stride=stride)
        for b in range(B):
            for x, y, n in zip(seq_view(base, bt, b), seq_view(rp, pd, b), ("out", "dqkv", "lse", "delta")):
                if n in ("lse", "delta"):
                    x, y = x[:, :bt.caps[b]], y[:, :bt.caps[b]]
                else:
                    y = y[:bt.caps[b]]
                assert_bits(x, y, f"{what}: packed vs padded, seq {b}: {n}")


# ---------------------------------------------------------------------------------------------------------------------------
# 1. the sweep
# ---------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("c", SWEEP, ids=_cid)
def test_sweep(T, c):
    """one case of the sweep: guards, unchanged inputs, padding tiles, per-element bounds of out / lse / delta / dq / dk / dv
    against fp64, and every exact identity"""
    bt, cs, stride, r = run_case(T, c, seed=zlib.crc32(_cid(c).encode()) % 10000)
    check_reference(c, bt, r, cs)
    check_identities(T, c, bt, cs, stride, r)


@gpu
@pytest.mark.parametrize("fwd_e", [0, 2, 3, 4])
@pytest.mark.parametrize("layout", ["rect", "padded", "packed"])
def test_zero_v_gives_zero_output(T, fwd_e, layout):
    """V = 0 on every key a query can see gives out = 0 exactly, under every forward E, while the keys it cannot see hold V =
    +-2^120: causal (V = 0 on rows 0..95, rows 0..95 checked) and with a window of 64 (V = 0 on rows 100..199, rows 164..199
    checked)"""
    torch = _torch()
    for window, (zlo, zhi), (clo, chi) in ((0, (0, 96), (0, 96)), (64, (100, 200), (164, 200))):
        c = Case(B=2, S=256, H=4, Hkv=2, fwd_e=fwd_e, window=window, layout=layout, lens=(256, 200) if layout != "rect" else ())
        bt = make_batch(c, seed=90 + fwd_e)
        H, Hkv = c.H, c.Hkv
        g = torch.Generator(device="cuda").manual_seed(91)
        for b in range(2):
            x = bt.qkv[bt.starts[b]:bt.starts[b] + bt.caps[b]].view(bt.caps[b], H + 2 * Hkv, D)
            big = (2.0 ** 120) * torch.sign(torch.randn(bt.caps[b], Hkv, D, generator=g, device="cuda"))
            x[:, H + Hkv:] = big.to(torch.bfloat16)
            x[zlo:zhi, H + Hkv:] = 0
        r = Run(T, c, bt)
        for b in range(2):
            rows = r.o()[bt.starts[b] + clo:bt.starts[b] + chi].float()
            bad = rows != 0
            assert not bool(bad.any()), f"{_cid(c)}: seq {b}: {int(bad.sum())} outputs of rows that see only V = 0 are not 0 " \
                                        f"(max {float(rows.abs().max()):.3g})"


# ---------------------------------------------------------------------------------------------------------------------------
# 2. end to end against autograd, and refusals on the GPU
# ---------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("c", [Case(layout="padded", lens=(384, 129), H=8, Hkv=2, window=0, rope="half"),
                               Case(layout="packed", lens=(300, 0, 129), B=3, H=7, Hkv=1, window=129, fwd_e=3, dq_e=4),
                               Case(H=4, Hkv=4, rope="glm", fwd_e=2, dq_e=3)], ids=_cid)
def test_end_to_end_autograd(T, c):
    """out and dq / dk / dv (inverse rotary included) of the real rows against fp32 autograd of the true attention: relative L2
    errors below 8e-3 (out) and 1.5e-2 (gradients), as the older checks"""
    torch = _torch()
    bt, cs, stride, r = run_case(T, c, seed=11)
    H, Hkv, g = c.H, c.Hkv, c.H // c.Hkv
    for b in range(len(bt.lens)):
        n = bt.lens[b]
        if n < 2:
            continue
        r0 = bt.starts[b]
        x = bt.qkv[r0:r0 + n].float().view(n, H + 2 * Hkv, D).requires_grad_(True)
        q, k, v = x[:, :H].transpose(0, 1), x[:, H:H + Hkv].repeat_interleave(g, 1).transpose(0, 1), \
            x[:, H + Hkv:].repeat_interleave(g, 1).transpose(0, 1)
        i = torch.arange(n, device="cuda")
        s = (q @ k.transpose(-1, -2)) * c.scale
        s = s.masked_fill(~visible(i, i, eff_window(c))[None], -math.inf)
        o = (torch.softmax(s, -1) @ v).transpose(0, 1).reshape(n, H * D)
        o.backward(bt.dout[r0:r0 + n].float())
        gr = x.grad.view(n, H + 2 * Hkv, D).double()
        if cs is not None:
            gr[:, :H + Hkv] = inverse_rotary(gr[:, :H + Hkv].transpose(0, 1), gr[:, :H + Hkv].transpose(0, 1) * 0,
                                             gr[:, :H + Hkv].transpose(0, 1).abs(), cs, i, c.rope == "glm")[0].transpose(0, 1)
        rel = lambda a, b_: float((a.double() - b_).norm() / b_.norm().clamp(min=1e-30))
        assert rel(r.o()[r0:r0 + n], o.detach().double()) < 8e-3
        got = r.g()[r0:r0 + n].view(n, H + 2 * Hkv, D)
        for name, sl_ in (("dq", slice(0, H)), ("dk", slice(H, H + Hkv)), ("dv", slice(H + Hkv, H + 2 * Hkv))):
            assert rel(got[:, sl_], gr[:, sl_]) < 1.5e-2, (name, b)


@gpu
def test_refusals_leave_outputs_untouched(T):
    """refused calls on real buffers leave out, lse, delta and dqkv at their sentinels: scale 0, negative, NaN or infinite,
    rope_stride in (0, S) against a table allocated for S positions, and window < 0"""
    c = Case(B=2, S=256, H=4, Hkv=2, rope="half")
    bt = make_batch(c, seed=5)
    good = Run(T, c, bt)
    cs, _ = rope_table(replace(c, rope="glm"), 6)  # [32][S]: S/2 as a half-split stride stays inside it
    cs64 = _torch().cat([cs, cs])                  # [64][S]
    B, S, H, Hkv = 2, c.S, c.H, c.Hkv
    W = (H + 2 * Hkv) * D
    for what, scale, window, stride in (("scale 0", 0.0, 0, 0), ("scale -0.088", -0.088, 0, 0), ("scale NaN", float("nan"), 0, 0),
                                        ("scale inf", float("inf"), 0, 0), ("window -1", c.scale, -1, 0),
                                        ("rope_stride S / 2", c.scale, 0, S // 2)):
        out, lse = Guarded(bt.M * H * D, False), Guarded(B * H * S, True)
        if not stride:
            rc = T.dtx_attn_fwd(P(bt.qkv), P(out.win), P(lse.win), B, S, H, Hkv, scale, None, window, ST())
            _torch().cuda.synchronize()
            assert rc == DTX_ERR_INVALID, f"forward, {what}: returned {rc}"
            out.assert_untouched(f"forward, {what}: out")
            lse.assert_untouched(f"forward, {what}: lse")
        delta, dqkv = Guarded(B * H * S, True), Guarded(bt.M * W, False)
        rc = T.dtx_attn_bwd_rope(P(bt.qkv), P(good.out.win), P(bt.dout), P(good.lse.win), P(delta.win), P(dqkv.win), B, S, H, Hkv,
                                 scale, None, window, P(cs64) if stride else None, stride, 0, ST())
        _torch().cuda.synchronize()
        assert rc == DTX_ERR_INVALID, f"backward, {what}: returned {rc}"
        delta.assert_untouched(f"backward, {what}: delta")
        dqkv.assert_untouched(f"backward, {what}: dqkv")


# ---------------------------------------------------------------------------------------------------------------------------
# 3. real model geometries
# ---------------------------------------------------------------------------------------------------------------------------
MODELS = {  # name: (H, Hkv, S, window, rope, packed lengths)
    "llama2-7b": (32, 32, 2048, 0, "half", (2048, 700, 0, 1)),
    "llama2-13b": (40, 40, 2048, 0, "half", (1500, 129, 2048)),
    "mistral-s4096": (32, 8, 4096, 0, "half", (4096, 1000, 63)),
    "mistral-s8192-w4096": (32, 8, 8192, 4096, "half", (8192, 5000, 0)),
    "qwen2.5-7b": (28, 4, 4096, 0, "half", (3000, 4096, 1)),
    "qwen2.5-14b": (40, 8, 4096, 0, "half", (4095, 128, 2000)),
    "glm4-9b": (32, 2, 4096, 0, "glm", (4096, 2500, 0)),
    "mistral-s32768-w4096": (32, 8, 32768, 4096, "half", None),
}


@gpu
@pytest.mark.parametrize("model", list(MODELS))
def test_real_model_geometry(T, model):
    """the kernels on all heads of a real model (one full sequence, then a packed ragged batch); the fp64 reference and the
    per-element bounds on the first, a middle and the last KV group, whose query heads alone carry dO: every other head's dq
    and every other KV head's dk / dv are exactly 0"""
    torch = _torch()
    H, Hkv, S, window, rope, plens = MODELS[model]
    g = H // Hkv
    checked = sorted({0, Hkv // 2, Hkv - 1})
    for layout, lens in (("rect", ()), ("packed", plens)):
        if lens is None:
            continue
        c = Case(B=1 if layout == "rect" else len(lens), S=S, H=H, Hkv=Hkv, window=window, rope=rope, layout=layout, lens=lens)
        bt = make_batch(c, seed=300)
        mask = torch.zeros(H, dtype=torch.bool, device="cuda")
        for hk in checked:
            mask[hk * g:hk * g + g] = True
        bt.dout.view(bt.M, H, D)[:, ~mask] = 0
        cs, stride = rope_table(c, 301)
        r = Run(T, c, bt, cs=cs, stride=stride)
        dq = r.g().view(bt.M, H + 2 * Hkv, D)
        kvmask = torch.zeros(Hkv, dtype=torch.bool, device="cuda")
        kvmask[checked] = True
        if not bool(mask.all()):
            assert float(dq[:, :H][:, ~mask].float().abs().max()) == 0.0, f"{model}: dq of heads without dO"
        if not bool(kvmask.all()):
            assert float(dq[:, H:H + Hkv][:, ~kvmask].float().abs().max()) == 0.0, f"{model}: dk of KV heads without dO"
            assert float(dq[:, H + Hkv:][:, ~kvmask].float().abs().max()) == 0.0, f"{model}: dv of KV heads without dO"
        check_reference(c, bt, r, cs, groups=checked, key=f"models {model}", chunk=512 if S > 8192 else 1024)
        del r, bt
        torch.cuda.empty_cache()
    report(f"models {model}")


@gpu
def test_report_sweep_worst():
    report("sweep")
