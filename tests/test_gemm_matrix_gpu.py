"""Kernel-level parity of gemm_bf16 over every instantiation its dispatcher can reach.

- **Dispatch sweep.**  For each product entry point (dtx_gemm_bf16, dtx_gemm_fused, dtx_gemm_bias, dtx_gemm_qk_norm,
  dtx_gemm_rope_glm), the cartesian product of the dispatch inputs it takes (block_n, both majors, the six epilogues, bias, the
  wide-tile switch, an N that selects the tile width) at one shape with tails in M, N and K.  Accepted combinations are checked
  like every other case below; refused ones must return DTX_ERR_INVALID and leave C, aux and R as they were.  The accepted set
  must cover all 47 gemm_kernel instantiations, derived from the dispatch rules in `variant()`.
- **Exactness.**  EPI_F32 against an fp64 reference element by element: |c - ref| <= 2^-16 * sum_k |a_k b_k|.  Every bf16
  epilogue is a bitwise function of that fp32 accumulator (same tile width, majors and K segments); the epilogue maths
  (rotaries, q/k norm, SwiGLU forward and backward) is checked in fp64 on the kernel's own accumulator to one bf16 ulp (two for
  the q/k norm) at the magnitude of its inputs.  Tile width and rasterisation group do not change a single bit.
- **Guard bands.**  Every output sits inside a sentinel-filled buffer (64 rows above and below, 8 columns before, 64 + after);
  after each call everything outside the logical window still holds the sentinel, and the inputs R / gu are unchanged.
- **Split-K** planes bitwise equal to unsplit calls over their k-block ranges, the persistent loop over partial rasterisation
  groups, m_eff at every tile width, and one case per projection of four real models.

The refusal contract also has a CPU-only test that calls the entry points with fake device addresses.
"""
import contextlib
import ctypes as C
import itertools
import math
from dataclasses import dataclass, replace

import pytest

from tests.conftest import has_gpu

gpu = pytest.mark.gpu
EPI_BF16, EPI_F32, EPI_BF16_ADD, EPI_ROPE, EPI_SWIGLU_FWD, EPI_SWIGLU_BWD = range(6)
EPI_NAME = {EPI_BF16: "bf16", EPI_F32: "f32", EPI_BF16_ADD: "bf16_add"}
DTX_ERR_INVALID = -1
GUARD_ROWS = 64  # sentinel rows above and below every output
COL0 = 8         # first column of an output inside its buffer
SENT16 = 0x7FA5      # bf16 NaN sentinel
SENT32 = 0x7FC0A5A5  # fp32 NaN sentinel
FP32_RULE = 2.0 ** -16
ROPE_S = 97
QK_EPS = 1e-6
N_SMS = 132  # H100 SXM: the SM count the split-K shapes below are chosen for

_vp, _i32, _i64, _f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
_HOOKS = {
    "dtx_test_gemm_m_eff": [_vp, _i64, _i32, _vp, _i64, _i32, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp],
}


def _bind():
    from datatunerx_b200 import lib as L
    lib = L.load()
    for name, argtypes in _HOOKS.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = _i32
    return lib


@contextlib.contextmanager
def options(pair=1, group_m=0):
    from datatunerx_b200 import lib as L
    L.set_option("gemm_pair_kernel", pair)
    L.set_option("gemm_group_m", group_m)
    try:
        yield
    finally:
        L.set_option("gemm_pair_kernel", 1)
        L.set_option("gemm_group_m", 0)


@pytest.fixture(scope="module")
def T():
    """the library with the m_eff test hook bound (skips without a GPU); the GEMM switches are back at their defaults after"""
    if not has_gpu():
        pytest.skip("no GPU")
    from datatunerx_b200 import lib as L
    lib = _bind()
    try:
        yield lib
    finally:
        L.set_option("gemm_pair_kernel", 1)
        L.set_option("gemm_group_m", 0)


# ---------------------------------------------------------------------------------------------------------------------------
# the dispatcher's instantiations
# ---------------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Case:
    epi: int = EPI_BF16
    a_mn: int = 0
    b_mn: int = 0
    block_n: int = 0
    bias: bool = False
    qk: bool = False
    glm: bool = False
    pair: int = 1
    M: int = 200
    N: int = 264
    K: int = 136
    K2: int = 72
    split_k: int = 1
    rope_cols: int = 256
    q_cols: int = 128
    pos: bool = False      # EPI_ROPE: per-row positions instead of row % rope_S
    inplace: bool = False  # EPI_BF16_ADD: R aliases C


LAYOUTS = {(0, 0): "NT", (0, 1): "NN", (1, 1): "TN"}
FUSED = ("rope", "rope+bias", "rope+qk", "glm", "glm+bias", "swiglu_fwd", "swiglu_bwd")
ALL_VARIANTS = frozenset(
    [("plain", bn, lay, e) for bn in (64, 128, 256) for lay in ("NT", "NN", "TN") for e in ("bf16", "f32", "bf16_add")]
    + [("bias", bn, b) for bn in (64, 128, 256) for b in ("B_K", "B_MN")]
    + [("fused", b, f) for b in ("B_K", "B_MN") for f in FUSED])


def eff_bn(c):
    bn = c.block_n or (64 if c.N <= 64 else (128 if c.N <= 128 else 256))
    return 128 if bn == 256 and not c.pair else bn


def variant(c, entry=None):
    """the gemm_kernel instantiation gemm_bf16 runs c with (by its documented dispatch rules), or None where they refuse c;
    `entry`: the product entry point c goes through (dtx_gemm_bf16 passes no rotary table or aux, dtx_gemm_fused only epilogues
    3..5)"""
    if (entry == "bf16" and c.epi >= EPI_ROPE) or (entry == "fused" and c.epi < EPI_ROPE):
        return None
    if c.split_k > 1 and c.epi != EPI_F32:
        return None
    if c.bias and (c.epi not in (EPI_BF16, EPI_ROPE) or c.a_mn or c.split_k > 1):
        return None
    if c.qk and (c.epi != EPI_ROPE or c.bias):
        return None
    if c.glm and (c.epi != EPI_ROPE or c.qk):
        return None
    bk = "B_MN" if c.b_mn else "B_K"
    if c.epi >= EPI_ROPE:
        if c.a_mn or c.M <= 128 or not c.pair:
            return None
        if (c.epi in (EPI_ROPE, EPI_SWIGLU_FWD) and c.N % 256) or (c.epi == EPI_SWIGLU_BWD and c.N % 128):
            return None
        if c.epi == EPI_ROPE:
            if c.rope_cols % 256:
                return None
            name = ("glm" if c.glm else "rope") + ("+bias" if c.bias else "") + ("+qk" if c.qk else "")
        else:
            name = "swiglu_fwd" if c.epi == EPI_SWIGLU_FWD else "swiglu_bwd"
        return ("fused", bk, name)
    if (c.a_mn, c.b_mn) not in LAYOUTS or eff_bn(c) not in (64, 128, 256):
        return None
    if c.bias:
        return ("bias", eff_bn(c), bk)
    return ("plain", eff_bn(c), LAYOUTS[(c.a_mn, c.b_mn)], EPI_NAME[c.epi])


def public_entry(c):
    """the product entry point that expresses c"""
    if c.epi <= EPI_BF16_ADD:
        return "bias" if c.bias else "bf16"
    if c.glm:
        return "glm"
    if c.qk:
        return "qk"
    if c.bias:
        return "bias"
    assert not c.pos, "dtx_gemm_fused takes no row positions: its rotary runs at row % rope_S"
    return "fused"


SWEEP_N = {EPI_BF16: 264, EPI_F32: 264, EPI_BF16_ADD: 264, EPI_ROPE: 512, EPI_SWIGLU_FWD: 512, EPI_SWIGLU_BWD: 384}
NARROW_N = 56  # <= 64: block_n = 0 picks 64-wide tiles


def sweep_cases():
    """(entry point, case): the product of the dispatch inputs each product entry point takes"""
    two = (0, 1)
    for block_n, a_mn, b_mn, epi, narrow, pair in itertools.product((0, 64, 128, 256), two, two, range(6), two, two):
        yield "bf16", Case(epi=epi, a_mn=a_mn, b_mn=b_mn, block_n=block_n, pair=pair, N=NARROW_N if narrow else SWEEP_N[epi])
    for b_mn, epi, pair in itertools.product(two, range(6), two):
        yield "fused", Case(epi=epi, b_mn=b_mn, pair=pair, N=SWEEP_N[epi])
    for b_mn, epi, narrow, pair in itertools.product(two, range(6), two, two):  # the tile width follows N and the switch
        yield "bias", Case(epi=epi, b_mn=b_mn, bias=True, pair=pair, N=NARROW_N if narrow else SWEEP_N[epi])
    for b_mn, pair in itertools.product(two, two):
        yield "qk", Case(epi=EPI_ROPE, b_mn=b_mn, qk=True, pair=pair, N=SWEEP_N[EPI_ROPE])
    for b_mn, bias, pair in itertools.product(two, two, two):
        yield "glm", Case(epi=EPI_ROPE, b_mn=b_mn, glm=True, bias=bool(bias), pair=pair, N=SWEEP_N[EPI_ROPE])


def test_dispatch_model_covers_every_instantiation():
    """CPU-only: the sweep's combinations reach all 47 instantiations under the dispatch model (the GPU sweep then checks that
    the library agrees with the model, combination by combination)"""
    reached = {variant(c, entry) for entry, c in sweep_cases()} - {None}
    assert reached == ALL_VARIANTS and len(ALL_VARIANTS) == 47


# ---------------------------------------------------------------------------------------------------------------------------
# buffers
# ---------------------------------------------------------------------------------------------------------------------------
def _torch():
    import torch
    return torch


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def ST():
    return C.c_void_p(_torch().cuda.current_stream().cuda_stream)


def round_up(x, m):
    return (x + m - 1) // m * m


class Out:
    """An output window of planes x [rows, cols] at column COL0 of a sentinel-filled buffer with GUARD_ROWS guard rows above and
    below and row stride N + 8 + 64 rounded up to 16 bytes (the planes of split-K partials follow each other at rows * ld)."""

    def __init__(self, rows, cols, f32=False, planes=1):
        torch = _torch()
        self.rows, self.cols, self.planes, self.f32 = rows, cols, planes, f32
        self.ld = round_up(cols + COL0 + 64, 4 if f32 else 8)
        self.sent = SENT32 if f32 else SENT16
        self.bits = torch.full((2 * GUARD_ROWS + planes * rows, self.ld), self.sent, dtype=torch.int32 if f32 else torch.int16,
                               device="cuda")
        self.win_bits = self.bits[GUARD_ROWS:GUARD_ROWS + planes * rows, COL0:COL0 + cols]
        self.win = self.win_bits.view(torch.float32 if f32 else torch.bfloat16)

    @property
    def ptr(self):
        return P(self.win)

    def planes_view(self):
        return self.win.view(self.planes, self.rows, self.cols)

    def assert_guard(self, what):
        g = self.bits.clone()
        g[GUARD_ROWS:GUARD_ROWS + self.planes * self.rows, COL0:COL0 + self.cols] = self.sent
        bad = (g != self.sent).nonzero()
        if bad.numel():
            r, c = (int(v) for v in bad[0])
            raise AssertionError(f"{what}: {bad.shape[0]} guard elements written, first at buffer row {r - GUARD_ROWS} (window rows "
                                 f"0..{self.planes * self.rows - 1}), column {c - COL0} (window columns 0..{self.cols - 1})")

    def assert_untouched(self, what):
        assert bool((self.bits == self.sent).all()), f"{what}: a refused call wrote its output"


def operand(x):
    """x [r, c] as a column slice of a wider NaN-filled bf16 buffer: row stride > c, base 8 elements (16 bytes) in"""
    torch = _torch()
    r, c = x.shape
    buf = torch.full((r, round_up(c + COL0 + 40, 8)), float("nan"), dtype=torch.bfloat16, device="cuda")
    buf[:, COL0:COL0 + c] = x
    return buf[:, COL0:COL0 + c]


def randn(shape, seed, scale=1.0):
    torch = _torch()
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


class Prob:
    """Logical operands a [M, K], b [K, N] (+ a2, b2 for the K2 segment), laid out for the case's majors, and every epilogue input:
    R, the gate|up aux of SWIGLU_BWD, a rotary table, row positions, bias and q/k norm weights."""

    def __init__(self, c, seed=0):
        torch = _torch()
        M, N, K, K2 = c.M, c.N, c.K, c.K2
        sb = 1.0 / math.sqrt(K + K2)
        self.a, self.b = randn((M, K), seed), randn((K, N), seed + 1, sb)
        self.A = operand(self.a.t() if c.a_mn else self.a)
        self.B = operand(self.b if c.b_mn else self.b.t())
        self.a2 = self.b2 = self.A2 = self.B2 = None
        if K2:
            self.a2, self.b2 = randn((M, K2), seed + 2), randn((K2, N), seed + 3, sb)
            self.A2 = operand(self.a2.t() if c.a_mn else self.a2)
            self.B2 = operand(self.b2 if c.b_mn else self.b2.t())
        self.r = randn((M, N), seed + 4, 2.0) if c.epi == EPI_BF16_ADD else None
        self.R = operand(self.r) if self.r is not None else None
        self.gu = operand(randn((M, 2 * N), seed + 5, 1.5)) if c.epi == EPI_SWIGLU_BWD else None
        g = torch.Generator(device="cuda").manual_seed(seed + 6)
        ang = torch.rand((ROPE_S, 32 if c.glm else 64), generator=g, device="cuda") * (2 * math.pi)
        self.cs = torch.stack([torch.cos(ang), torch.sin(ang)], dim=-1).contiguous()  # float2 (cos, sin) per pair
        self.pos = torch.randint(0, ROPE_S, (M,), generator=g, device="cuda", dtype=torch.int32) if c.pos else None
        self.bias = randn((N,), seed + 7) if c.bias else None
        self.wq, self.wk = (1 + randn((128,), seed + 8, 0.25).float()).to(torch.bfloat16), (1 + randn((128,), seed + 9, 0.25).float()).to(torch.bfloat16)
        self.R0 = self.R.clone() if self.R is not None else None
        self.gu0 = self.gu.clone() if self.gu is not None else None

    def rows_of(self):
        """rotary position of every row"""
        torch = _torch()
        M = self.a.shape[0]
        return self.pos.long() if self.pos is not None else torch.arange(M, device="cuda") % ROPE_S


def make_outs(c):
    outs = {"C": Out(c.M, 2 * c.N if c.epi == EPI_SWIGLU_BWD else c.N, f32=c.epi == EPI_F32, planes=c.split_k)}
    if c.epi == EPI_SWIGLU_FWD:
        outs["aux"] = Out(c.M, c.N // 2)
    elif c.qk:
        outs["aux"] = Out(c.M, c.rope_cols)
    return outs


def execute(T, c, p, entry, m_eff=None):
    """one call of `entry` for case c on problem p; returns (status, outputs)"""
    torch = _torch()
    outs = make_outs(c)
    Cout, aux = outs["C"], outs.get("aux")
    A, B, A2, B2 = p.A, p.B, p.A2, p.B2
    lda2, ldb2 = (A2.stride(0), B2.stride(0)) if A2 is not None else (0, 0)
    R, ldr = p.R, (p.R.stride(0) if p.R is not None else 0)
    if c.epi == EPI_BF16_ADD and c.inplace:
        Cout.win.copy_(p.r)
        R, ldr = Cout.win, Cout.ld
    if aux is not None:
        auxp, ld_aux = aux.ptr, aux.ld
    elif p.gu is not None:
        auxp, ld_aux = P(p.gu), p.gu.stride(0)
    else:
        auxp, ld_aux = None, 0
    cs = P(p.cs) if (c.epi == EPI_ROPE or c.glm) else None
    rope_S, rope_cols = (ROPE_S, c.rope_cols) if cs is not None else (0, 0)
    common = (P(A), A.stride(0))
    if entry == "bf16":
        rc = T.dtx_gemm_bf16(*common, c.a_mn, P(B), B.stride(0), c.b_mn, P(A2), lda2, P(B2), ldb2, c.K2, Cout.ptr, Cout.ld, P(R), ldr,
                             c.M, c.N, c.K, c.epi, c.split_k, c.block_n, ST())
    elif entry == "fused":
        rc = T.dtx_gemm_fused(*common, P(B), B.stride(0), c.b_mn, P(A2), lda2, P(B2), ldb2, c.K2, Cout.ptr, Cout.ld, auxp, ld_aux, cs,
                              rope_S, rope_cols, c.M, c.N, c.K, c.epi, ST())
    elif entry == "bias":
        rc = T.dtx_gemm_bias(*common, P(B), B.stride(0), c.b_mn, P(A2), lda2, P(B2), ldb2, c.K2, Cout.ptr, Cout.ld, auxp, ld_aux, cs,
                             rope_S, rope_cols, P(p.pos), c.M, c.N, c.K, c.epi, P(p.bias), ST())
    elif entry == "qk":
        rc = T.dtx_gemm_qk_norm(*common, P(B), B.stride(0), c.b_mn, P(A2), lda2, P(B2), ldb2, c.K2, Cout.ptr, Cout.ld, auxp, ld_aux, cs,
                                rope_S, rope_cols, P(p.pos), c.M, c.N, c.K, c.q_cols, P(p.wq), P(p.wk), QK_EPS, ST())
    elif entry == "glm":
        rc = T.dtx_gemm_rope_glm(*common, P(B), B.stride(0), c.b_mn, P(A2), lda2, P(B2), ldb2, c.K2, Cout.ptr, Cout.ld, cs, rope_S,
                                 rope_cols, P(p.pos), c.M, c.N, c.K, P(p.bias), ST())
    elif entry == "m_eff":
        assert c.K2 == 0
        me = torch.tensor([m_eff], dtype=torch.int32, device="cuda") if m_eff is not None else None
        rc = T.dtx_test_gemm_m_eff(*common, c.a_mn, P(B), B.stride(0), c.b_mn, Cout.ptr, Cout.ld, c.M, c.N, c.K, c.epi, c.split_k,
                                   c.block_n, P(me), ST())
    else:
        raise ValueError(entry)
    torch.cuda.synchronize()
    return rc, outs


def assert_refused(rc, c, p, outs, what):
    torch = _torch()
    assert rc == DTX_ERR_INVALID, f"{what}: returned {rc}, expected DTX_ERR_INVALID"
    if c.epi == EPI_BF16_ADD and c.inplace:
        g = outs["C"].bits.clone()
        assert torch.equal(outs["C"].win.view(torch.int16), p.r.view(torch.int16)), f"{what}: a refused call changed R (= C)"
        g[GUARD_ROWS:GUARD_ROWS + c.M, COL0:COL0 + c.N] = SENT16
        assert bool((g == SENT16).all()), f"{what}: a refused call wrote the guard band"
    else:
        outs["C"].assert_untouched(what)
    if "aux" in outs:
        outs["aux"].assert_untouched(what + " (aux)")
    assert_inputs_unchanged(c, p, what)


def assert_inputs_unchanged(c, p, what):
    torch = _torch()
    if p.R is not None:
        assert torch.equal(p.R.view(torch.int16), p.R0.view(torch.int16)), f"{what}: R changed"
    if p.gu is not None:
        assert torch.equal(p.gu.view(torch.int16), p.gu0.view(torch.int16)), f"{what}: the gate|up input changed"


# ---------------------------------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------------------------------
WORST = {}  # fp32 rule: worst |c - ref| / (2^-16 sum|ab|) seen per test


def _where(mask, what, got=None, sent=None):
    idx = mask.nonzero()
    r, c = (int(v) for v in idx[0][-2:])
    boxes = sorted({(int(i[-2]) // 64, int(i[-1]) // 64) for i in idx[:4096]})
    left = ""
    if got is not None and sent is not None:
        left = f", {int((got[mask] == sent).sum())} of them still the sentinel"
    return f"{what}: {idx.shape[0]} elements wrong{left}, first at row {r} column {c}; 64x64 boxes (row, col) {boxes[:8]}"


def ref64(p, rows=None, cols=None):
    """fp64 a b (+ a2 b2) and sum_k |a_k b_k| on the selected rows / columns"""
    def sel(x, r, c):
        x = x if r is None else x[r]
        return x if c is None else x[:, c]
    a, b = sel(p.a, rows, None).double(), sel(p.b, None, cols).double()
    ref, mag = a @ b, a.abs() @ b.abs()
    if p.a2 is not None:
        a2, b2 = sel(p.a2, rows, None).double(), sel(p.b2, None, cols).double()
        ref, mag = ref + a2 @ b2, mag + a2.abs() @ b2.abs()
    return ref, mag


def assert_fp32_rule(got, p, what, key, rows=None, cols=None):
    """EPI_F32 element by element: |c - ref| <= 2^-16 sum_k |a_k b_k|; plus the global rel_err < 1e-5 of the older checks at the
    contraction lengths they use (K + K2 <= 8192: at K = V ~ 150 000 random signs cancel so far that the fp32 sum's relative
    error is ~2e-4 while every element stays well inside the elementwise bound).

    Worst observed |c - ref| / (2^-16 sum|ab|) on an H100 80GB HBM3 at its 700 W limit: 0.017 at the small shapes (K + K2 <=
    592), 0.014 on the rasterisation shape, 0.006 for split-K sums, 0.19 over the real model widths (K up to 152 064)."""
    ref, mag = ref64(p, rows, cols)
    g = got if rows is None else got[rows]
    g = (g if cols is None else g[:, cols]).double()
    err = (g - ref).abs()
    bound = FP32_RULE * mag
    bad = ~(err <= bound)
    if bool(bad.any()):
        raise AssertionError(_where(bad, f"{what}: fp32 rule (worst ratio {float((err / bound).max()):.3g})"))
    WORST[key] = max(WORST.get(key, 0.0), float((err / bound.clamp(min=1e-300)).max()))
    if p.a.shape[1] + (p.a2.shape[1] if p.a2 is not None else 0) <= 8192:
        rel = float((g - ref).norm() / ref.norm().clamp(min=1e-30))
        assert rel < 1e-5, f"{what}: rel_err {rel}"


def assert_bits_equal(got, want, what):
    torch = _torch()
    gb, wb = got.contiguous().view(torch.int16), want.contiguous().view(torch.int16)
    bad = gb != wb
    if bool(bad.any()):
        raise AssertionError(_where(bad, what, gb, SENT16))


def assert_equal_f32(got, want, what):
    torch = _torch()
    gb, wb = got.contiguous().view(torch.int32), want.contiguous().view(torch.int32)
    bad = gb != wb
    if bool(bad.any()):
        raise AssertionError(_where(bad, what, gb, SENT32))


def ulp_bf16(mag):
    torch = _torch()
    _, e = torch.frexp(mag.clamp(min=2.0 ** -100))
    return torch.ldexp(torch.ones_like(mag), e - 8)


def assert_ulps(got, ref, mag, n, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= n * ulp_bf16(mag))
    if bool(bad.any()):
        raise AssertionError(_where(bad, f"{what}: beyond {n} bf16 ulp", got.contiguous().view(_torch().int16), SENT16))


def rotate(x, p, rope_cols, glm):
    """fp64 rotary of columns < rope_cols of x [M, N] (fp64) and the magnitude |x0| + |x1| of every rotated pair"""
    torch = _torch()
    M = x.shape[0]
    t = p.cs.double()[p.rows_of()]  # [M, pairs, 2]
    cs, sn = t[..., 0][:, None, :], t[..., 1][:, None, :]
    out, mag = x.clone(), x.abs()
    h = x[:, :rope_cols].reshape(M, rope_cols // 128, 128)
    if glm:
        x0, x1 = h[:, :, 0:64:2], h[:, :, 1:64:2]
        o = out[:, :rope_cols].view(M, rope_cols // 128, 128)
        m = mag[:, :rope_cols].view(M, rope_cols // 128, 128)
        o[:, :, 0:64:2], o[:, :, 1:64:2] = x0 * cs - x1 * sn, x1 * cs + x0 * sn
        m[:, :, 0:64:2] = m[:, :, 1:64:2] = x0.abs() + x1.abs()
    else:
        x0, x1 = h[:, :, :64], h[:, :, 64:]
        o = out[:, :rope_cols].view(M, rope_cols // 128, 128)
        m = mag[:, :rope_cols].view(M, rope_cols // 128, 128)
        o[:, :, :64], o[:, :, 64:] = x0 * cs - x1 * sn, x1 * cs + x0 * sn
        m[:, :, :64] = m[:, :, 64:] = x0.abs() + x1.abs()
    return out, mag


def silu_parts(g):
    torch = _torch()
    s = torch.sigmoid(g)
    return s, g * s


# ---------------------------------------------------------------------------------------------------------------------------
# one case: run it, its fp32 companion, and every check
# ---------------------------------------------------------------------------------------------------------------------------
def accumulator(T, c, p, key, rows=None, cols=None):
    """the kernel's fp32 accumulator for c: EPI_F32 with the same tile width, majors and K segments (guard-checked, fp32 rule)"""
    f = replace(c, epi=EPI_F32, bias=False, qk=False, glm=False, block_n=eff_bn(c) if c.epi <= EPI_BF16_ADD else 256, inplace=False,
                split_k=1, pos=False)
    rc, outs = execute(T, f, p, "bf16")
    assert rc == 0, f"{f}: fp32 companion returned {rc}"
    outs["C"].assert_guard(f"{f} fp32 companion")
    assert_fp32_rule(outs["C"].win, p, f"{f} fp32 companion", key, rows, cols)
    return outs["C"].win.clone(memory_format=_torch().contiguous_format)


def check_case(T, c, p, outs, key, acc=None, rows=None, cols=None):
    """guard bands, unchanged inputs and the epilogue identities / maths of an accepted call"""
    torch = _torch()
    what = str(c)
    Cout = outs["C"]
    Cout.assert_guard(what)
    if "aux" in outs:
        outs["aux"].assert_guard(what + " aux")
    if not (c.epi == EPI_BF16_ADD and c.inplace):
        assert_inputs_unchanged(c, p, what)
    got = Cout.win
    if c.epi == EPI_F32:
        if c.split_k == 1:
            assert_fp32_rule(got, p, what, key, rows, cols)
        return got.clone(memory_format=torch.contiguous_format)
    if acc is None:
        acc = accumulator(T, c, p, key, rows, cols)
    x32 = acc + p.bias.float() if c.bias else acc  # fp32 adds, in the kernel's order
    if c.epi == EPI_BF16:
        assert_bits_equal(got, x32.to(torch.bfloat16), what + ": C == bf16_rn(F32 (+ bias))")
    elif c.epi == EPI_BF16_ADD:
        assert_bits_equal(got, (acc + p.r.float()).to(torch.bfloat16), what + ": C == bf16_rn(F32 + R)")
    elif c.epi == EPI_ROPE:
        rc_ = c.rope_cols
        assert_bits_equal(got[:, rc_:], x32[:, rc_:].to(torch.bfloat16), what + ": columns >= rope_cols == bf16_rn(F32 (+ bias))")
        if c.qk:
            xb = acc[:, :rc_].to(torch.bfloat16)
            assert_bits_equal(outs["aux"].win, xb, what + ": pre-norm aux == bf16_rn(F32)")
            h = xb.double().view(c.M, rc_ // 128, 128)
            rstd = 1.0 / torch.sqrt((h * h).mean(-1, keepdim=True) + QK_EPS)
            w = torch.where(torch.arange(rc_ // 128, device="cuda")[:, None] * 128 < c.q_cols, p.wq.double()[None, :], p.wk.double()[None, :])
            y = (h * w[None] * rstd).reshape(c.M, rc_)
            ref, mag = rotate(y, p, rc_, False)
            assert_ulps(got[:, :rc_], ref, mag, 2, what + ": q/k norm + rotary")
        else:
            ref, mag = rotate(x32[:, :rc_].double(), p, rc_, c.glm)
            if c.glm:  # columns 64..127 of every rotated head pass through
                v = got[:, :rc_].view(c.M, rc_ // 128, 128)[:, :, 64:]
                assert_bits_equal(v, x32[:, :rc_].view(c.M, rc_ // 128, 128)[:, :, 64:].to(torch.bfloat16), what + ": GLM pass-through half")
            assert_ulps(got[:, :rc_], ref, mag, 1, what + (": GLM rotary" if c.glm else ": rotary"))
    elif c.epi == EPI_SWIGLU_FWD:
        assert_bits_equal(got, acc.to(torch.bfloat16), what + ": C == bf16_rn(F32)")
        F = c.N // 2
        v = acc.to(torch.bfloat16).double().view(c.M, F // 128, 2, 128)
        g, u = v[:, :, 0].reshape(c.M, F), v[:, :, 1].reshape(c.M, F)
        ref = silu_parts(g)[1] * u
        assert_ulps(outs["aux"].win, ref, ref.abs(), 1, what + ": silu(g) * u")
    elif c.epi == EPI_SWIGLU_BWD:
        F = c.N
        d = acc.to(torch.bfloat16).double()
        v = p.gu.double().contiguous().view(c.M, F // 128, 2, 128)
        g, u = v[:, :, 0].reshape(c.M, F), v[:, :, 1].reshape(c.M, F)
        s, si = silu_parts(g)
        dg, du = d * u * (s + si * (1 - s)), d * si
        dg_mag, du_mag = (d * u).abs() * (s + (si * (1 - s)).abs()), du.abs()
        o = got.view(c.M, F // 128, 2, 128)
        assert_ulps(o[:, :, 0].reshape(c.M, F), dg, dg_mag, 1, what + ": SwiGLU backward d(gate)")
        assert_ulps(o[:, :, 1].reshape(c.M, F), du, du_mag, 1, what + ": SwiGLU backward d(up)")
    return acc


def run_checked(T, c, p, entry, key):
    with options(pair=c.pair):
        rc, outs = execute(T, c, p, entry)
        assert rc == 0, f"{c} via {entry}: returned {rc}"
        return check_case(T, c, p, outs, key), outs


def report(key):
    print(f"\n[fp32 rule] {key}: worst |c - ref| / (2^-16 sum|ab|) = {WORST.get(key, 0.0):.4f}")


# ---------------------------------------------------------------------------------------------------------------------------
# 1. the dispatch sweep
# ---------------------------------------------------------------------------------------------------------------------------
@gpu
def test_dispatch_sweep(T):
    """Every combination of dispatch inputs the product entry points take, at M = 200, K = 136 + K2 = 72 and N = 264 (512 / 384
    for the fused epilogues) or 56: accepted exactly when the dispatch model accepts it, checked as a case (guards, fp32 rule,
    identities, maths);
    refused ones return DTX_ERR_INVALID with every output at its sentinel and R / gu unchanged.  The accepted set covers all 47
    instantiations, and the fp32 accumulator does not depend on the tile width (64, 128, 256) in any layout."""
    key = "sweep"
    probs, reached, f32_by = {}, {}, {}
    for entry, c in sweep_cases():
        pk = (c.a_mn, c.b_mn, c.N, c.glm, c.epi == EPI_BF16_ADD, c.epi == EPI_SWIGLU_BWD, c.bias)
        if pk not in probs:
            probs[pk] = Prob(c, seed=len(probs) * 16)
        p = probs[pk]
        want = variant(c, entry)
        with options(pair=c.pair):
            rc, outs = execute(T, c, p, entry)
            if want is None:
                assert_refused(rc, c, p, outs, f"{c} via {entry}")
                continue
            assert rc == 0, f"{c} via {entry}: returned {rc}, the dispatch model expects {want}"
            reached.setdefault(want, (entry, c))
            out = check_case(T, c, p, outs, key)
        if c.epi == EPI_F32 and entry == "bf16":
            f32_by.setdefault((c.a_mn, c.b_mn, c.N), {})[eff_bn(c)] = out
    missing = sorted(ALL_VARIANTS - set(reached), key=str)
    assert not missing, f"instantiations no accepted combination reaches: {missing}"
    assert set(reached) == ALL_VARIANTS
    for lay, by_bn in f32_by.items():
        assert sorted(by_bn) == [64, 128, 256], (lay, sorted(by_bn))
        for bn in (64, 128):
            assert_equal_f32(by_bn[bn], by_bn[256], f"{LAYOUTS[lay[:2]]}, N = {lay[2]}: fp32 accumulator, {bn}-wide tiles vs 256-wide")
    for v in sorted(reached, key=str):
        print(f"[reach] {v}: {reached[v][0]} {reached[v][1]}")
    report(key)


# ---------------------------------------------------------------------------------------------------------------------------
# 3. shapes and edges, per instantiation
# ---------------------------------------------------------------------------------------------------------------------------
def case_for(v):
    kind = v[0]
    if kind == "plain":
        _, bn, lay, e = v
        a_mn, b_mn = {l: k for k, l in LAYOUTS.items()}[lay]
        c = Case(epi={n: k for k, n in EPI_NAME.items()}[e], a_mn=a_mn, b_mn=b_mn, block_n=bn)
    elif kind == "bias":
        _, bn, b = v
        c = Case(epi=EPI_BF16, b_mn=int(b == "B_MN"), bias=True, N=NARROW_N if bn == 64 else 264, pair=int(bn != 128))
    else:
        _, b, f = v
        epi = {"swiglu_fwd": EPI_SWIGLU_FWD, "swiglu_bwd": EPI_SWIGLU_BWD}.get(f, EPI_ROPE)
        c = Case(epi=epi, N=SWEEP_N[epi], b_mn=int(b == "B_MN"), bias="bias" in f, qk="qk" in f, glm="glm" in f)
    assert variant(c) == v
    return c


def shapes_for(c):
    """(M, N, K, K2, extra case fields): every M / N / K / K2 edge below at least once, kept small"""
    if c.bias and c.epi == EPI_BF16:  # dtx_gemm_bias takes no block_n: the tile width follows N and the wide-tile switch
        ns = {64: (8, 56, 64, 40), 128: (72, 128, 264, 640), 256: (264, 640, 384, 1000)}[eff_bn(c)]
        return [(M, n, K, K2, dict(pair=c.pair)) for (M, K, K2), n in zip(((1, 8, 0), (64, 72, 8), (129, 520, 72), (1000, 72, 0)), ns)]
    if c.epi <= EPI_BF16_ADD:
        nmin = 4 if c.epi == EPI_F32 else 8
        return [(1, nmin, 8, 0, {}), (64, 72, 72, 8, {}), (129, 264, 520, 72, {}), (1000, 640, 72, 0, {})]
    if c.epi == EPI_SWIGLU_BWD:
        return [(129, 128, 8, 0, {}), (1000, 384, 72, 8, {}), (129, 640, 520, 72, {})]
    rope = c.epi == EPI_ROPE
    pos = c.bias or c.qk or c.glm  # dtx_gemm_fused takes no positions: its rotary runs at row % rope_S
    return [(129, 256, 8, 0, dict(rope_cols=256, q_cols=128, pos=False) if rope else {}),
            (1000, 768, 72, 8, dict(rope_cols=512, q_cols=384, pos=pos) if rope else {}),
            (129, 512, 520, 72, dict(rope_cols=256, q_cols=256, pos=pos) if rope else {})]


def _vid(v):
    return "-".join(str(x) for x in v)


@gpu
@pytest.mark.parametrize("v", sorted(ALL_VARIANTS, key=str), ids=_vid)
def test_variant_shapes(T, v):
    """One instantiation through its product entry point at M in {1, 64, 129, 1000} (fused: 129, 1000), N from the smallest it
    accepts through 72, 264 and half tiles, K in {8, 72, 520}, K2 in {0, 8, 72}; A (and every operand) a column slice of a wider
    NaN-filled buffer; EPI_BF16_ADD with R separate and R aliasing C; rotaries with and without positions (where the entry
    point takes them) and rope_cols < N; the bias variants at Ns that select their tile width."""
    base = case_for(v)
    key = f"shapes {_vid(v)}"
    for i, (M, N, K, K2, extra) in enumerate(shapes_for(base)):
        for inplace in ((False, True) if base.epi == EPI_BF16_ADD else (False,)):
            c = replace(base, M=M, N=N, K=K, K2=K2, inplace=inplace, **extra)
            assert variant(c) == v, c
            run_checked(T, c, Prob(c, seed=100 + 8 * i), public_entry(c), key)
    report(key)


# ---------------------------------------------------------------------------------------------------------------------------
# 5. split-K
# ---------------------------------------------------------------------------------------------------------------------------
def pick_split(n_sms, m_tiles, kb_total):
    """the trainer's choice of split for the token-contracted weight-gradient GEMMs"""
    s = min(16, max(1, (2 * n_sms + m_tiles - 1) // m_tiles), kb_total)
    while s > 1 and (s - 1) * ((kb_total + s - 1) // s) >= kb_total:
        s -= 1
    return s


SPLITS = {  # M, N, K (tokens), K2
    "uneven": (8448, 64, 1050, 0),
    "straddles_K2": (384, 72, 1050, 72),
    "one_block_each": (384, 64, 520, 0),
}


@gpu
@pytest.mark.parametrize("name", list(SPLITS))
def test_split_k_planes(T, name):
    """TN (both operands MN-major), 64-wide tiles, split as pick_split chooses on a 132-SM H100: every partial plane is bitwise an
    unsplit EPI_F32 call over exactly its k-block range (A / B row slices at 64-element offsets, across the K / K2 boundary), the
    planes' sum meets the fp32 rule, and the 3-D output's guard columns and rows stay untouched."""
    M, N, K, K2 = SPLITS[name]
    kb1, kb2 = (K + 63) // 64, (K2 + 63) // 64
    kbt = kb1 + kb2
    s = pick_split(N_SMS, (M + 127) // 128, kbt)
    per = (kbt + s - 1) // s
    ranges = [(i * per, min(kbt, (i + 1) * per)) for i in range(s)]
    if name == "uneven":
        assert kbt % s and s > 1, (kbt, s)
    elif name == "straddles_K2":
        assert any(b < kb1 < e for b, e in ranges), ranges
    else:
        assert s == kbt, (s, kbt)
    c = Case(epi=EPI_F32, a_mn=1, b_mn=1, block_n=64, M=M, N=N, K=K, K2=K2, split_k=s)
    p = Prob(c, seed=300)
    key = f"split {name}"
    rc, outs = execute(T, c, p, "bf16")
    assert rc == 0, rc
    outs["C"].assert_guard(f"{c} partials")
    planes = outs["C"].planes_view()
    for i, (b, e) in enumerate(ranges):
        segs = []  # (A rows, B rows) of each segment the range covers, in k order
        if b < kb1:
            segs.append((p.A[b * 64:min(e * 64, K)], p.B[b * 64:min(e * 64, K)]))
        if e > kb1:
            lo, hi = max(b - kb1, 0) * 64, min((e - kb1) * 64, K2)
            segs.append((p.A2[lo:hi], p.B2[lo:hi]))
        (A1, B1), (A2, B2) = segs[0], (segs[1] if len(segs) > 1 else (None, None))
        one = Out(M, N, f32=True)
        rc = T.dtx_gemm_bf16(P(A1), A1.stride(0), 1, P(B1), B1.stride(0), 1, P(A2), A2.stride(0) if A2 is not None else 0, P(B2),
                             B2.stride(0) if B2 is not None else 0, A2.shape[0] if A2 is not None else 0, one.ptr, one.ld, None, 0, M,
                             N, A1.shape[0], EPI_F32, 1, 64, ST())
        _torch().cuda.synchronize()
        assert rc == 0, rc
        one.assert_guard(f"split {i} reference call")
        assert_equal_f32(planes[i], one.win, f"{name}: plane {i} (k-blocks {b}..{e - 1}) vs the unsplit call over them")
    assert_fp32_rule(planes.double().sum(0), p, f"{name}: sum of {s} planes", key)
    report(key)


# ---------------------------------------------------------------------------------------------------------------------------
# 6. persistent loop and rasterisation
# ---------------------------------------------------------------------------------------------------------------------------
@gpu
def test_rasterisation_groups(T):
    """M = 4480 (35 row tiles: a full group of 32, then 3), N = 1088 (a 64-column tail), K = 320: more tiles than SMs.  For
    gemm_group_m in {1, 3, default} and both tile widths, EPI_F32 and EPI_BF16_ADD are bitwise the same everywhere (and meet the
    fp32 rule / the bf16(F32 + R) identity); the RoPE epilogue (N = 1024) is bitwise the same for every group size."""
    key = "rasterisation"
    base = Case(epi=EPI_F32, M=4480, N=1088, K=320, K2=0)
    p = Prob(base, seed=400)
    pa = Prob(replace(base, epi=EPI_BF16_ADD), seed=400)
    rope = replace(base, epi=EPI_ROPE, N=1024, rope_cols=512)
    pr = Prob(rope, seed=401)
    f32 = add = rot = None
    for pair, gm in itertools.product((1, 0), (1, 3, 0)):
        with options(pair=pair, group_m=gm):
            what = f"pair {pair}, gemm_group_m {gm}"
            rc, o = execute(T, replace(base, pair=pair), p, "bf16")
            assert rc == 0, rc
            got = check_case(T, replace(base, pair=pair), p, o, key) if f32 is None else o["C"].win
            o["C"].assert_guard(what)
            if f32 is None:
                f32 = got.clone(memory_format=_torch().contiguous_format)
            assert_equal_f32(got, f32, f"EPI_F32, {what}")
            c = replace(base, epi=EPI_BF16_ADD, pair=pair)
            rc, o = execute(T, c, pa, "bf16")
            assert rc == 0, rc
            o["C"].assert_guard(what)
            assert_inputs_unchanged(c, pa, what)
            if add is None:
                acc_add = accumulator(T, c, pa, key)
                add = (acc_add + pa.r.float()).to(_torch().bfloat16)
            assert_bits_equal(o["C"].win, add, f"EPI_BF16_ADD, {what}")
            if pair:
                rc, o = execute(T, rope, pr, public_entry(rope))
                assert rc == 0, rc
                if rot is None:
                    check_case(T, rope, pr, o, key)
                    rot = o["C"].win.clone(memory_format=_torch().contiguous_format)
                o["C"].assert_guard(what)
                assert_bits_equal(o["C"].win, rot, f"EPI_ROPE, {what}")
    report(key)


@gpu
@pytest.mark.parametrize("block_n", [64, 128, 256])
def test_m_eff_every_tile_width(T, block_n):
    """dtx_test_gemm_m_eff on the rasterisation shape: rows below min(M, ceil256(m_eff)) bitwise equal the call without m_eff at
    the same tile width, every row beyond keeps its sentinel (the dead-block rule counts 256-row blocks at every width)."""
    torch = _torch()
    c = Case(epi=EPI_F32, M=4480, N=1088, K=320, K2=0, block_n=block_n)
    p = Prob(c, seed=402)
    rc, full = execute(T, c, p, "m_eff")
    assert rc == 0, rc
    full["C"].assert_guard("no m_eff")
    assert not bool(torch.isnan(full["C"].win).any())
    for m_eff in (0, 1, 255, 256, 257, 2000, 4479, 4480, 5000):
        rc, o = execute(T, c, p, "m_eff", m_eff=m_eff)
        assert rc == 0, rc
        live = min(c.M, (m_eff + 255) // 256 * 256)
        o["C"].assert_guard(f"m_eff {m_eff}")
        assert_equal_f32(o["C"].win[:live], full["C"].win[:live], f"m_eff {m_eff}: live rows")
        assert bool((o["C"].win_bits[live:] == SENT32).all()), f"m_eff {m_eff}: rows of skipped blocks were written"


# ---------------------------------------------------------------------------------------------------------------------------
# 7. the refusal contract without a GPU
# ---------------------------------------------------------------------------------------------------------------------------
def test_refusals_without_gpu():
    """CPU-only: gemm_bf16 validates before any CUDA call, so every documented refusal returns DTX_ERR_INVALID on fake (aligned)
    device addresses, while the same call without the defect gets past validation (DTX_ERR_CUDA: no device).  Skipped where a GPU
    is visible: an accepted case would launch on the fake addresses there; the GPU sweep checks the same rules on real buffers.
    Three of gemm_bf16's rules guard internal callers only, since no entry point can pass their combinations: a bias with an
    MN-major A (dtx_gemm_bias takes no A major), the q/k norm with a bias (dtx_gemm_qk_norm takes no bias) and GLM's rotary with
    the q/k norm (dtx_gemm_rope_glm takes no norm weights)."""
    if has_gpu():
        pytest.skip("a GPU is visible")
    lib = _bind()
    F = 1 << 40  # 16-byte aligned fake device address

    def bf16(A=F, lda=256, a_mn=0, B=F, ldb=256, b_mn=0, C_=F, ldc=512, R=None, ldr=0, M=256, N=512, K=256, epi=EPI_BF16, split_k=1,
             block_n=0):
        return lib.dtx_gemm_bf16(A, lda, a_mn, B, ldb, b_mn, None, 0, None, 0, 0, C_, ldc, R, ldr, M, N, K, epi, split_k, block_n, None)

    def fused(M=256, N=512, epi=EPI_ROPE, C_=F, ldc=None, aux=None, ld_aux=0, rope_cols=256, b_mn=0):
        return lib.dtx_gemm_fused(F, 256, F, 256, b_mn, None, 0, None, 0, 0, C_, ldc or 2 * N, aux, ld_aux, F, 64, rope_cols, M, N, 256,
                                  epi, None)

    def bias(epi=EPI_BF16, N=512, rope_cols=256):
        return lib.dtx_gemm_bias(F, 256, F, 256, 0, None, 0, None, 0, 0, F, 2 * N, None, 0, F, 64, rope_cols, None, 256, N, 256, epi, F,
                                 None)

    def qk(q_cols=256, rope_cols=512, wk=F, aux=F, ld_aux=512):
        return lib.dtx_gemm_qk_norm(F, 256, F, 256, 0, None, 0, None, 0, 0, F, 1024, aux, ld_aux, F, 64, rope_cols, None, 256, 1024, 256,
                                    q_cols, F, wk, QK_EPS, None)

    def glm(rope_cols=256):
        return lib.dtx_gemm_rope_glm(F, 256, F, 256, 0, None, 0, None, 0, 0, F, 512, F, 64, rope_cols, None, 256, 512, 256, None, None)

    cases = [  # (what, valid call, the same call with one defect)
        ("misaligned bf16 ldc", lambda: bf16(), lambda: bf16(ldc=516)),
        ("misaligned fp32 ldc", lambda: bf16(epi=EPI_F32, ldc=516), lambda: bf16(epi=EPI_F32, ldc=514)),
        ("misaligned lda", lambda: bf16(), lambda: bf16(lda=260)),
        ("misaligned ldb", lambda: bf16(), lambda: bf16(ldb=252)),
        ("misaligned A base", lambda: bf16(), lambda: bf16(A=F + 8)),
        ("misaligned B base", lambda: bf16(), lambda: bf16(B=F + 2)),
        ("misaligned C base", lambda: bf16(), lambda: bf16(C_=F + 8)),
        ("misaligned R", lambda: bf16(epi=EPI_BF16_ADD, R=F, ldr=512), lambda: bf16(epi=EPI_BF16_ADD, R=F, ldr=500)),
        ("EPI_BF16_ADD without R", lambda: bf16(epi=EPI_BF16_ADD, R=F, ldr=512), lambda: bf16(epi=EPI_BF16_ADD)),
        ("split_k > 1 with EPI_BF16", lambda: bf16(epi=EPI_F32, split_k=2), lambda: bf16(split_k=2)),
        ("split_k > 1 with EPI_BF16_ADD", lambda: bf16(epi=EPI_F32, split_k=2), lambda: bf16(epi=EPI_BF16_ADD, R=F, ldr=512, split_k=2)),
        ("MN-major A with K-major B", lambda: bf16(a_mn=1, b_mn=1), lambda: bf16(a_mn=1)),
        ("fused with M <= 128", lambda: fused(M=129), lambda: fused(M=128)),
        ("RoPE with N % 256", lambda: fused(), lambda: fused(N=384)),
        ("SwiGLU forward with N % 256", lambda: fused(epi=EPI_SWIGLU_FWD, aux=F, ld_aux=256),
         lambda: fused(epi=EPI_SWIGLU_FWD, N=384, aux=F, ld_aux=256)),
        ("SwiGLU backward with N % 128", lambda: fused(epi=EPI_SWIGLU_BWD, N=384, aux=F, ld_aux=768, b_mn=1),
         lambda: fused(epi=EPI_SWIGLU_BWD, N=320, aux=F, ld_aux=768, b_mn=1)),
        ("SwiGLU without aux", lambda: fused(epi=EPI_SWIGLU_FWD, aux=F, ld_aux=256), lambda: fused(epi=EPI_SWIGLU_FWD)),
        ("dtx_gemm_fused with a plain epilogue", lambda: fused(), lambda: fused(epi=EPI_BF16)),
        ("bias with EPI_F32", lambda: bias(), lambda: bias(epi=EPI_F32)),
        ("bias with EPI_BF16_ADD", lambda: bias(), lambda: bias(epi=EPI_BF16_ADD)),
        ("bias with a SwiGLU epilogue", lambda: bias(epi=EPI_ROPE), lambda: bias(epi=EPI_SWIGLU_FWD)),
        ("q/k norm: q / k boundary inside a head", lambda: qk(), lambda: qk(q_cols=320)),
        ("q/k norm: q_cols beyond the rotated columns", lambda: qk(), lambda: qk(q_cols=640)),
        ("q/k norm without k_norm weights", lambda: qk(), lambda: qk(wk=None)),
        ("q/k norm: misaligned pre-norm output", lambda: qk(), lambda: qk(aux=F + 8)),
        ("q/k norm: pre-norm row stride below rope_cols", lambda: qk(), lambda: qk(ld_aux=504)),
        ("rope_cols % 256", lambda: fused(), lambda: fused(rope_cols=384)),
        ("bias RoPE rope_cols % 256", lambda: bias(epi=EPI_ROPE), lambda: bias(epi=EPI_ROPE, rope_cols=384)),
        ("GLM rope_cols % 256", lambda: glm(), lambda: glm(rope_cols=384)),
        ("q/k norm rope_cols % 256", lambda: qk(), lambda: qk(rope_cols=640)),
    ]
    with options(pair=1):
        for what, good, bad in cases:
            assert good() != DTX_ERR_INVALID, f"{what}: the call without the defect was refused"
            assert bad() == DTX_ERR_INVALID, f"{what}: not refused"
    with options(pair=0):
        for what, call in (("RoPE", fused), ("bias RoPE", lambda: bias(epi=EPI_ROPE)), ("q/k norm", qk), ("GLM", glm)):
            assert call() == DTX_ERR_INVALID, f"{what} epilogue with the wide tiles switched off: not refused"


# ---------------------------------------------------------------------------------------------------------------------------
# 8. real model widths
# ---------------------------------------------------------------------------------------------------------------------------
MODELS = {  # hidden, q heads, kv heads, ffn, vocab, q|k|v epilogue
    "llama3.1-8b": (4096, 32, 8, 14336, 128256, "rope"),
    "qwen2.5-7b": (3584, 28, 4, 18944, 152064, "rope+bias"),
    "qwen3-8b": (4096, 32, 8, 12288, 151936, "rope+qk"),
    "glm4-9b": (4096, 32, 2, 13696, 151552, "glm+bias"),
}
TOKENS = 1152


def sample(n, seed, extra=0):
    """the first and last index of every 64-wide box, plus `extra` random ones"""
    torch = _torch()
    idx = set(range(0, n, 64)) | {min(i + 63, n - 1) for i in range(0, n, 64)}
    if extra:
        g = torch.Generator().manual_seed(seed)
        idx |= set(torch.randint(0, n, (extra,), generator=g).tolist())
    return torch.tensor(sorted(idx), device="cuda")


@gpu
@pytest.mark.parametrize("model", list(MODELS))
def test_real_model_widths(T, model):
    """One call per projection of the model at M = 1152 tokens: q|k|v with its fused epilogue (+ a LoRA K2 segment), gate|up with
    SWIGLU_FWD, the down-projection backward with SWIGLU_BWD, the lm_head forward as EPI_F32 with m_eff, the lm_head backward as
    NN with K = V, and a weight gradient TN at K = 1000 tokens accumulated in place.  The fp32 rule runs on sampled rows / columns
    (first and last of every 64-wide box, plus 64 random rows); the bitwise identities and the epilogue maths on every element."""
    d, H, Hkv, Fd, V, qkv_epi = MODELS[model]
    W, rope_cols = (H + 2 * Hkv) * 128, (H + Hkv) * 128
    key = f"models {model}"
    rows = sample(TOKENS, 1, 64)
    f = dict(bias="bias" in qkv_epi, qk="qk" in qkv_epi, glm="glm" in qkv_epi)
    cases = [
        replace(Case(epi=EPI_ROPE, M=TOKENS, N=W, K=d, K2=64, rope_cols=rope_cols, q_cols=H * 128,
                     pos=qkv_epi != "rope"), **f),
        Case(epi=EPI_SWIGLU_FWD, M=TOKENS, N=2 * Fd, K=d, K2=0),
        Case(epi=EPI_SWIGLU_BWD, b_mn=1, M=TOKENS, N=Fd, K=d, K2=0),
        Case(epi=EPI_BF16, b_mn=1, M=TOKENS, N=d, K=V, K2=0),  # lm_head backward: dh = dlogits W
        Case(epi=EPI_BF16_ADD, a_mn=1, b_mn=1, M=W, N=d, K=1000, K2=0, inplace=True),  # weight gradient of q|k|v
    ]
    for i, c in enumerate(cases):
        p = Prob(c, seed=500 + 16 * i)
        r = rows if c.M == TOKENS else sample(c.M, 2, 64)
        with options(pair=1):
            rc, outs = execute(T, c, p, public_entry(c))
            assert rc == 0, (c, rc)
            check_case(T, c, p, outs, key, rows=r, cols=sample(c.N, 3))
        del p, outs
    # lm_head forward: fp32 logits over the live rows only
    c = Case(epi=EPI_F32, M=TOKENS, N=V, K=d, K2=0)
    p = Prob(c, seed=600)
    rc, outs = execute(T, c, p, "m_eff", m_eff=1000)
    assert rc == 0, rc
    outs["C"].assert_guard(f"{model} lm_head")
    assert bool((outs["C"].win_bits[1024:] == SENT32).all()), "lm_head: rows of skipped blocks were written"
    assert_fp32_rule(outs["C"].win, p, f"{model} lm_head", key, rows=rows[rows < 1024], cols=sample(V, 4))
    report(key)
