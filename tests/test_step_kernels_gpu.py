"""Kernel-level parity of the data path a ragged training step runs, through the test-only entry points of
include/dtxtune_test.h (thin pass-throughs into the internal launchers):

- packed-batch attention (row_start / total_rows with seq_lens, windows, the fused inverse rotaries, the dQ exponential
  A/B switch), against fp32 attention run per sequence on its real rows, and bitwise against the right-padded layout;
- pack_rows / gather_rows / shift_labels against numpy, the compact cross-entropy (valid_idx, n_div, no dlogits) against fp64
  torch, loss_reduce, row_loss_stats and the compacted final norm (rmsnorm with a row map);
- the lm_head GEMMs with a device row count (m_eff);
- the full-parameter SFT kernels: rmsnorm_dw, embedding_bwd, sumsq_bf16_acc, add_f32_into_bf16, adamw_shard_step and the
  GU-interleaved SwiGLU.

Outputs start as NaN / 0x7fffffff sentinels, so rows a kernel must skip are checked rather than assumed.  The export test
needs no GPU; every other test is marked gpu.
"""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

from tests.conftest import has_gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu
SENT = 0x7FFFFFFF  # int32 sentinel
D = 128

_vp, _i32, _i64, _f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
_HOOKS = {
    "dtx_test_attn_fwd": [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _vp, _i32, _vp, _i32, _vp],
    "dtx_test_attn_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _vp, _i32, _vp, _i32, _vp, _i32, _i32, _vp],
    "dtx_test_pack_rows": [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp],
    "dtx_test_gather_rows": [_vp, _vp, _vp, _i32, _i32, _vp, _i32, _vp, _vp, _vp, _vp],
    "dtx_test_shift_labels": [_vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp],
    "dtx_test_cross_entropy": [_vp, _i64, _vp, _vp, _vp, _vp, _i64, _i32, _i32, _vp, _i32, _vp],
    "dtx_test_loss_reduce": [_vp, _vp, _vp, _i32, _i32, _i32, _vp],
    "dtx_test_row_loss_stats": [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp],
    "dtx_test_rmsnorm_fwd": [_vp, _vp, _vp, _vp, _i32, _i32, _f32, _vp, _vp],
    "dtx_test_rmsnorm_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _vp, _vp],
    "dtx_test_gemm_m_eff": [_vp, _i64, _i32, _vp, _i64, _i32, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp],
    "dtx_test_swiglu_fwd": [_vp, _vp, _i32, _i32, _i32, _vp],
    "dtx_test_swiglu_bwd": [_vp, _vp, _vp, _i32, _i32, _i32, _vp],
    "dtx_test_rmsnorm_dw": [_vp, _vp, _vp, _i32, _i32, _vp, _vp, _i32, _vp],
    "dtx_test_embedding_bwd": [_vp, _vp, _vp, _i32, _i32, _i32, _vp],
    "dtx_test_sumsq_bf16_acc": [_vp, _i64, _vp, _vp, _i32, _vp],
    "dtx_test_add_f32_into_bf16": [_vp, _vp, _i64, _i32, _vp],
    "dtx_test_adamw_shard_step": [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _f32, _f32, _f32, _f32, _f32, _f32, _f32, _f32, _vp, _f32,
                                  _vp, _vp],
}


def _declared_hooks():
    src = open(os.path.join(ROOT, "include", "dtxtune_test.h")).read()
    return sorted(set(re.findall(r"DTX_API[^;(]*?\b(dtx_test_\w+)\s*\(", src)))


def test_every_declared_test_hook_is_exported_and_bound(lib):
    """CPU-only: the library exports every dtx_test_* of dtxtune_test.h, this file binds exactly those, and none of them is
    part of the product ABI (dtxtune.h / lib.ABI_SYMBOLS)."""
    from datatunerx_b200 import lib as L
    names = _declared_hooks()
    assert names == sorted(_HOOKS), (names, sorted(_HOOKS))
    for name in names:
        assert hasattr(lib, name), name
    assert not [n for n in L.ABI_SYMBOLS if n.startswith("dtx_test_")]
    assert "dtx_test_" not in open(os.path.join(ROOT, "include", "dtxtune.h")).read()


# ---------------------------------------------------------------------------------------------------------------------------
# helpers (GPU)
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def T():
    """the library with the test hooks bound (skips without a GPU)"""
    if not has_gpu():
        pytest.skip("no GPU")
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


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def ST():
    return C.c_void_p(_torch().cuda.current_stream().cuda_stream)


def ok(code):
    from datatunerx_b200 import lib as L
    L.check(code)
    _torch().cuda.synchronize()


def host_i32(a):
    a = np.ascontiguousarray(a, dtype=np.int32)
    return a, a.ctypes.data_as(C.c_void_p)


def dev(a, dtype=None):
    torch = _torch()
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).cuda()


def rand(*shape, scale=1.0, seed=0, dtype=None):
    torch = _torch()
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype or torch.bfloat16).cuda()


def nan(*shape, dtype=None):
    torch = _torch()
    return torch.full(shape, float("nan"), dtype=dtype or torch.bfloat16, device="cuda")


def sentinel_i32(n):
    torch = _torch()
    return torch.full((n,), SENT, dtype=torch.int32, device="cuda")


def rel_err(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp(min=1e-30))


def pack_plan(lens, S):
    """the trainer's own packed layout of a ragged batch"""
    from datatunerx_b200 import lib as L
    starts, _ = L.plan_packed_rows(lens, S)
    return starts


# ---------------------------------------------------------------------------------------------------------------------------
# packed attention
# ---------------------------------------------------------------------------------------------------------------------------
ATT_S = 384           # tile-grid extent of the batch (the longest row, rounded up to 128)
ATT_ROPE_S = 512      # positions in the rotary table (the trainer's seq_len; its row stride in the transposed table)
ATT_LENS = (129, 1, 384, 0, 127, 128)


def _rope_tables(glm):
    """[ATT_ROPE_S][n_freq] (cos, sin) and its transpose [n_freq][ATT_ROPE_S] (what the backward kernels read)"""
    torch = _torch()
    n = 32 if glm else 64
    inv = 1.0 / (10000.0 ** (torch.arange(0, 2 * n, 2, dtype=torch.float64) / (2 * n)))
    ang = torch.arange(ATT_ROPE_S, dtype=torch.float64)[:, None] * inv[None]
    cs = torch.stack([ang.cos(), ang.sin()], dim=-1).float().cuda()
    return cs, cs.permute(1, 0, 2).contiguous()


def _rope(x, cs, pos, n_rot, glm):
    """fp32 rotary of the first n_rot heads of x [M, W] at positions pos (half-split, or GLM's partial interleaved one)"""
    torch = _torch()
    M = x.shape[0]
    c, s = cs[pos, :, 0][:, None, :], cs[pos, :, 1][:, None, :]
    h = x[:, :n_rot * D].reshape(M, n_rot, D)
    if glm:
        x0, x1 = h[..., 0:64:2], h[..., 1:64:2]
        rot = torch.cat([torch.stack((x0 * c - x1 * s, x1 * c + x0 * s), dim=-1).flatten(-2), h[..., 64:]], dim=-1)
    else:
        x0, x1 = h[..., :64], h[..., 64:]
        rot = torch.cat([x0 * c - x1 * s, x1 * c + x0 * s], dim=-1)
    return torch.cat([rot.reshape(M, -1), x[:, n_rot * D:]], dim=1)


def _attn_ref(x, H, Hkv, window):
    """causal (optionally windowed) attention of one sequence x [n, (H + 2 Hkv) * 128] fp32: out [n, H*128], lse [H, n]"""
    torch = _torch()
    n = x.shape[0]
    v3 = x.view(n, H + 2 * Hkv, D)
    g = H // Hkv
    q = v3[:, :H].transpose(0, 1)
    k = v3[:, H:H + Hkv].transpose(0, 1).repeat_interleave(g, dim=0)
    v = v3[:, H + Hkv:].transpose(0, 1).repeat_interleave(g, dim=0)
    sc = q @ k.transpose(-1, -2) / math.sqrt(D)
    i = torch.arange(n, device=x.device)
    visible = i[None, :] <= i[:, None]
    if window > 0:
        visible &= i[None, :] >= i[:, None] - window
    sc = sc.masked_fill(~visible, float("-inf"))
    return (torch.softmax(sc, dim=-1) @ v).transpose(0, 1).reshape(n, H * D), torch.logsumexp(sc, dim=-1)


def _attn_call(T, qkv, dout, B, H, Hkv, window, lens_d, row_start, total_rows, rope_t, glm):
    torch = _torch()
    M, W = qkv.shape
    out = nan(M, H * D)
    lse2 = nan(B, H, ATT_S, dtype=torch.float32)
    delta = nan(B, H, ATT_S, dtype=torch.float32)
    dqkv = nan(M, W)
    sc = 1.0 / math.sqrt(D)
    ok(T.dtx_test_attn_fwd(P(qkv), P(out), P(lse2), B, ATT_S, H, Hkv, sc, P(lens_d), window, P(row_start), total_rows, ST()))
    ok(T.dtx_test_attn_bwd(P(qkv), P(out), P(dout), P(lse2), P(delta), P(dqkv), B, ATT_S, H, Hkv, sc, P(lens_d), window,
                           P(row_start), total_rows, P(rope_t), ATT_ROPE_S if rope_t is not None else 0, int(glm), ST()))
    return out, lse2, dqkv


_ATT_CASES = [(0, "none"), (0, "half"), (0, "glm"), (63, "none"), (63, "half"), (200, "none"), (200, "half")]


@gpu
@pytest.mark.parametrize("dq_fma", [0, 3, 4])
@pytest.mark.parametrize("window,rope", _ATT_CASES)
@pytest.mark.parametrize("H,Hkv", [(4, 4), (4, 2), (8, 1)])
def test_packed_attention(T, H, Hkv, window, rope, dq_fma):
    """Packed ragged batch (positions restart at 0 in every sequence, the rotary table's stride is the trainer's seq_len):
    forward out / lse and dq, dk, dv (with the fused inverse rotary) against fp32 attention per sequence on its real rows;
    everything in the total_rows rows finite, padding rows of a live tile with exactly zero gradient, lse entries beyond a
    sequence's rows untouched; and bitwise equal to the same sequences right-padded with seq_lens."""
    from datatunerx_b200 import lib as L
    torch = _torch()
    lens = np.array(ATT_LENS, np.int32)
    B = len(lens)
    starts = pack_plan(lens, ATT_S)
    caps = np.diff(starts)
    assert list(caps) == [min(ATT_S, max(128, (n + 127) // 128 * 128)) for n in lens]  # a 0-length sequence still owns 128 rows
    total = int(starts[-1])
    W = (H + 2 * Hkv) * D
    glm = rope == "glm"
    cs, cs_t = _rope_tables(glm) if rope != "none" else (None, None)
    pos = np.concatenate([np.arange(c) for c in caps])
    pre = rand(total, W, seed=1000 + H + Hkv)
    rot = _rope(pre.float(), cs, torch.as_tensor(pos).cuda(), H + Hkv, glm).to(torch.bfloat16) if cs is not None else pre
    dout = rand(total, H * D, seed=2000 + H)
    for b in range(B):
        dout[starts[b] + lens[b]:starts[b + 1]] = 0  # the loss never reaches a padding token
    row_start = dev(np.array(starts, np.int32))
    lens_d = dev(lens)
    L.set_option("attn_dq_exp_fma_every", dq_fma)
    try:
        out, lse2, dqkv = _attn_call(T, rot, dout, B, H, Hkv, window, lens_d, row_start, total, cs_t, glm)
        # the same sequences right-padded to ATT_S rows (the rows beyond a sequence's packed block hold unrelated values)
        rot_p, dout_p = rand(B * ATT_S, W, seed=7), torch.zeros(B * ATT_S, H * D, dtype=torch.bfloat16, device="cuda")
        for b in range(B):
            rot_p[b * ATT_S:b * ATT_S + caps[b]] = rot[starts[b]:starts[b + 1]]
            dout_p[b * ATT_S:b * ATT_S + caps[b]] = dout[starts[b]:starts[b + 1]]
        out_p, lse2_p, dqkv_p = _attn_call(T, rot_p, dout_p, B, H, Hkv, window, lens_d, None, 0, cs_t, glm)
    finally:
        L.set_option("attn_dq_exp_fma_every", 0)
    assert torch.isfinite(out.float()).all() and torch.isfinite(dqkv.float()).all(), "non-finite value in the packed rows"
    sl = {"dq": slice(0, H * D), "dk": slice(H * D, (H + Hkv) * D), "dv": slice((H + Hkv) * D, W)}
    worst = {"out": 0.0, "lse": 0.0}
    got_g, ref_g = [], []  # gradients of the real rows of every sequence (a 1-token sequence has dq = dk = 0: no per-row bar)
    for b in range(B):
        r0, n, cap = int(starts[b]), int(lens[b]), int(caps[b])
        pr = slice(b * ATT_S, b * ATT_S + cap)
        assert torch.equal(out[r0:r0 + cap], out_p[pr]), f"seq {b}: packed out differs from the padded layout"
        assert torch.equal(dqkv[r0:r0 + cap], dqkv_p[pr]), f"seq {b}: packed dqkv differs from the padded layout"
        assert torch.equal(lse2[b, :, :cap], lse2_p[b, :, :cap]), f"seq {b}: packed lse differs from the padded layout"
        assert torch.isnan(lse2[b, :, cap:]).all(), f"seq {b}: lse written beyond the sequence's rows"
        if n < cap:
            assert float(dqkv[r0 + n:r0 + cap].abs().max()) == 0.0, f"seq {b}: padding rows with a gradient"
        if n == 0:
            assert float(out[r0:r0 + cap].abs().max()) == 0.0
            continue
        x = pre[r0:r0 + n].float().requires_grad_(True)
        xr = _rope(x, cs, torch.arange(n, device="cuda"), H + Hkv, glm) if cs is not None else x
        ref, _ = _attn_ref(xr, H, Hkv, window)
        ref.backward(dout[r0:r0 + n].float())
        with torch.no_grad():
            ref_o, ref_lse = _attn_ref(rot[r0:r0 + n].float(), H, Hkv, window)
        worst["out"] = max(worst["out"], rel_err(out[r0:r0 + n], ref_o))
        worst["lse"] = max(worst["lse"], float((lse2[b, :, :n] * math.log(2.0) - ref_lse).abs().max()))
        got_g.append(dqkv[r0:r0 + n])
        ref_g.append(x.grad)
    got_g, ref_g = torch.cat(got_g), torch.cat(ref_g)
    for k, s_ in sl.items():
        worst[k] = rel_err(got_g[:, s_], ref_g[:, s_])
    assert worst["out"] < 8e-3 and worst["lse"] < 2e-3, worst
    assert max(worst["dq"], worst["dk"], worst["dv"]) < 1.5e-2, worst


# ---------------------------------------------------------------------------------------------------------------------------
# batch layout, labels and loss
# ---------------------------------------------------------------------------------------------------------------------------
def _ragged_batch(B, S, lens, seed, vocab=32000):
    """ids / labels [B, S]: padding (id 0, label -100) beyond every row's length, a -100 prompt at the start of every row"""
    rng = np.random.default_rng(seed)
    ids = rng.integers(1, vocab, (B, S)).astype(np.int32)
    labels = ids.copy()
    for b, n in enumerate(lens):
        labels[b, :rng.integers(0, max(1, n // 3) + 1)] = -100
        ids[b, n:] = 0
        labels[b, n:] = -100
    return ids, labels


@gpu
def test_pack_rows_and_gather_rows(T):
    S = 640
    lens = np.array([640, 0, 1, 127, 128, 129, 300, 513], np.int32)
    B = len(lens)
    ids, labels = _ragged_batch(B, S, lens, seed=3)
    starts = pack_plan(lens, S)
    total = starts[-1]
    ids_d, labels_d = dev(ids), dev(labels)
    extra = 256  # rows beyond total_rows must stay untouched
    ids_o, labels_o, pos_o, start_o = sentinel_i32(total + extra), sentinel_i32(total + extra), sentinel_i32(total + extra), sentinel_i32(B + 4)
    st, st_p = host_i32(starts)
    ok(T.dtx_test_pack_rows(P(ids_d), P(labels_d), S, B, st_p, P(ids_o), P(labels_o), P(pos_o), P(start_o), ST()))
    e_ids, e_lab, e_pos = (np.full(total + extra, SENT, np.int32) for _ in range(3))
    for b in range(B):
        cap = starts[b + 1] - starts[b]
        e_ids[starts[b]:starts[b + 1]] = ids[b, :cap]
        e_lab[starts[b]:starts[b + 1]] = labels[b, :cap]
        e_pos[starts[b]:starts[b + 1]] = np.arange(cap)
    assert np.array_equal(ids_o.cpu().numpy(), e_ids)
    assert np.array_equal(labels_o.cpu().numpy(), e_lab)
    assert np.array_equal(pos_o.cpu().numpy(), e_pos)
    assert np.array_equal(start_o.cpu().numpy(), np.concatenate([starts, np.full(3, SENT)]).astype(np.int32))
    # gather_rows: a length group (rows in any order, repeats allowed) at a shorter padded length
    rows = np.array([7, 0, 5, 5, 2], np.int32)
    S_dst = 512
    n = len(rows)
    ids_g, labels_g, lens_g = sentinel_i32(n * S_dst + 64), sentinel_i32(n * S_dst + 64), sentinel_i32(n + 2)
    rw, rw_p = host_i32(rows)
    lens_d = dev(lens)
    ok(T.dtx_test_gather_rows(P(ids_d), P(labels_d), P(lens_d), S, n, rw_p, S_dst, P(ids_g), P(labels_g), P(lens_g), ST()))
    tail = np.full(64, SENT, np.int32)
    assert np.array_equal(ids_g.cpu().numpy(), np.concatenate([ids[rows, :S_dst].reshape(-1), tail]))
    assert np.array_equal(labels_g.cpu().numpy(), np.concatenate([labels[rows, :S_dst].reshape(-1), tail]))
    assert np.array_equal(lens_g.cpu().numpy(), np.concatenate([lens[rows], [SENT, SENT]]).astype(np.int32))


def _shift_ref_rect(labels):
    B, S = labels.shape
    sh = np.full((B, S), -100, np.int32)
    sh[:, :-1] = labels[:, 1:]
    return sh.reshape(-1)


def _shift_ref_packed(labels_src, starts):
    """packed: row t of sequence b predicts the label of row t + 1 of the same sequence's block; the block's last row none"""
    out = np.full(starts[-1], -100, np.int32)
    for b in range(len(starts) - 1):
        cap = starts[b + 1] - starts[b]
        out[starts[b]:starts[b + 1] - 1] = labels_src[b, 1:cap]
    return out


def _run_shift(T, labels_flat, B, S, pos=None):
    M = labels_flat.shape[0]
    lab = dev(labels_flat)
    shifted, nv, row_map, vidx = sentinel_i32(M), sentinel_i32(2), sentinel_i32(M), sentinel_i32(M)
    ok(T.dtx_test_shift_labels(P(lab), P(shifted), P(nv), B, S, P(row_map), P(vidx), P(pos), ST()))
    return shifted.cpu().numpy(), int(nv[0]), int(nv[1]), row_map.cpu().numpy(), vidx.cpu().numpy()


def _check_shift(got, want):
    shifted, nv, nv_next, row_map, vidx = got
    valid = np.nonzero(want >= 0)[0]
    assert np.array_equal(shifted, want), "shifted labels"
    assert nv == len(valid) and nv_next == SENT, (nv, len(valid))
    e_map = np.full(want.shape[0], -1, np.int32)
    e_map[valid] = np.arange(len(valid))
    assert np.array_equal(row_map, e_map), "row_map"
    assert np.array_equal(vidx[:len(valid)], valid) and (vidx[len(valid):] == SENT).all(), "valid_idx"


@gpu
def test_shift_labels_rectangular_and_packed(T):
    """40 000+ tokens (each of the kernel's 1024 threads owns dozens), a row without any label, a 1-token row, a 0-length row,
    and an all-ignored batch; packed: the last row of every sequence's block predicts nothing."""
    B, S = 64, 1024
    lens = np.random.default_rng(11).integers(S // 2, S + 1, B).astype(np.int32)
    lens[:6] = [S, 1, 0, 127, 128, 129]
    ids, labels = _ragged_batch(B, S, lens, seed=12)
    for b in range(1, B, 2):  # no prompt: the first tokens carry labels (and a full block ends on a labelled token)
        labels[b, :lens[b]] = ids[b, :lens[b]]
    labels[6] = -100  # a sequence with no label
    _check_shift(_run_shift(T, labels.reshape(-1), B, S), _shift_ref_rect(labels))
    # packed, through pack_rows (the trainer's path) and the positions it writes
    starts = pack_plan(lens, S)
    total = starts[-1]
    assert total > 30000
    ids_o, labels_o, pos_o, start_o = sentinel_i32(total), sentinel_i32(total), sentinel_i32(total), sentinel_i32(B + 1)
    st, st_p = host_i32(starts)
    ids_d, labels_d = dev(ids), dev(labels)
    ok(T.dtx_test_pack_rows(P(ids_d), P(labels_d), S, B, st_p, P(ids_o), P(labels_o), P(pos_o), P(start_o), ST()))
    got = _run_shift(T, labels_o.cpu().numpy(), 1, total, pos=pos_o)
    _check_shift(got, _shift_ref_packed(labels, starts))
    # all ignored
    none = np.full((B, S), -100, np.int32)
    got = _run_shift(T, none.reshape(-1), B, S)
    assert got[1] == 0 and (got[0] == -100).all() and (got[3] == -1).all() and (got[4] == SENT).all()


def _ce_case(V, n_tok=777, seed=0):
    rng = np.random.default_rng(seed)
    shifted = rng.integers(0, V, n_tok).astype(np.int32)
    shifted[rng.random(n_tok) < 0.35] = -100
    shifted[:5] = [V - 1, 0, -100, V - 1, 3]
    return shifted


@gpu
@pytest.mark.parametrize("V", [2051, 32000])
def test_compact_cross_entropy(T, V):
    """Compact mode (logits / dlogits row k = token valid_idx[k]) with and without n_div and without dlogits, against fp64
    torch cross-entropy; rows at or beyond n_valid keep their sentinel; loss_reduce over the same division."""
    torch = _torch()
    Vp = (V + 3) // 4 * 4
    shifted = _ce_case(V, seed=V)
    M = shifted.shape[0]
    valid = np.nonzero(shifted >= 0)[0].astype(np.int32)
    nv = len(valid)
    vidx = np.full(M, SENT, np.int32)
    vidx[:nv] = valid
    logits = torch.full((M, Vp), float("nan"), device="cuda")
    logits[:nv] = rand(nv, Vp, scale=3.0, seed=5, dtype=torch.float32)
    lab_d, vidx_d, nv_d = dev(shifted), dev(vidx), dev(np.array([nv], np.int32))
    tgt = torch.as_tensor(shifted[valid]).long().cuda()
    ref_tok = torch.nn.functional.cross_entropy(logits[:nv, :V].double(), tgt, reduction="none")
    lg = logits[:nv, :V].double().requires_grad_(True)
    torch.nn.functional.cross_entropy(lg, tgt, reduction="sum").backward()  # p - onehot
    row_losses = {}
    for n_div in (0, nv + 1234):
        div = n_div or nv
        row_loss = torch.zeros(M, device="cuda")
        dl = nan(M, Vp)
        ok(T.dtx_test_cross_entropy(P(logits), Vp, P(lab_d), P(nv_d), P(row_loss), P(dl), Vp, M, V, P(vidx_d), n_div, ST()))
        got_tok = row_loss[torch.as_tensor(valid).long().cuda()].double()
        e_tok = float(((got_tok - ref_tok).abs() / ref_tok.abs().clamp(min=1e-6)).max())
        assert e_tok < 1e-5, f"row_loss per token {e_tok}"
        assert float(row_loss[torch.as_tensor(shifted < 0).cuda()].abs().max()) == 0.0
        e_g = rel_err(dl[:nv, :V], lg.grad / div)
        assert e_g < 4e-3, f"dlogits {e_g}"
        assert torch.isnan(dl[nv:].float()).all(), "dlogits rows at or beyond n_valid must not be written"
        loss = torch.full((2,), float("nan"), device="cuda")
        ok(T.dtx_test_loss_reduce(P(row_loss), P(nv_d), P(loss), M, n_div, 0, ST()))
        ref_loss = float(ref_tok.sum()) / div
        assert abs(float(loss[0]) - ref_loss) / ref_loss < 1e-5, (float(loss[0]), ref_loss)
        row_losses[n_div] = row_loss
    assert torch.equal(row_losses[0], row_losses[nv + 1234])
    # the eval path: no dlogits, the same row losses bit for bit
    row_loss = torch.zeros(M, device="cuda")
    ok(T.dtx_test_cross_entropy(P(logits), Vp, P(lab_d), P(nv_d), P(row_loss), None, Vp, M, V, P(vidx_d), 0, ST()))
    assert torch.equal(row_loss, row_losses[0])


@gpu
def test_cross_entropy_all_ignored_and_loss_reduce_groups(T):
    torch = _torch()
    V, M = 2051, 300
    Vp = (V + 3) // 4 * 4
    shifted = np.full(M, -100, np.int32)
    logits = rand(M, Vp, seed=9, dtype=torch.float32)
    lab_d, nv_d, vidx_d = dev(shifted), dev(np.array([0], np.int32)), sentinel_i32(M)
    for compact in (True, False):
        row_loss, dl = torch.zeros(M, device="cuda"), nan(M, Vp)
        ok(T.dtx_test_cross_entropy(P(logits), Vp, P(lab_d), P(nv_d), P(row_loss), P(dl), Vp, M, V, P(vidx_d) if compact else None, 0,
                                    ST()))
        loss = torch.full((1,), float("nan"), device="cuda")
        ok(T.dtx_test_loss_reduce(P(row_loss), P(nv_d), P(loss), M, 0, 0, ST()))
        assert float(loss[0]) == 0.0 and float(row_loss.abs().max()) == 0.0
        if compact:
            assert torch.isnan(dl.float()).all()
        else:
            assert float(dl[:, :V].float().abs().max()) == 0.0
    # two length groups of one micro-batch: n_div = labelled tokens of both, the second accumulates
    rng = np.random.default_rng(4)
    ga, gb = (torch.as_tensor(rng.random(n).astype(np.float32)).cuda() for n in (500, 700))
    na, nb = dev(np.array([321], np.int32)), dev(np.array([456], np.int32))
    loss = torch.full((1,), float("nan"), device="cuda")
    ok(T.dtx_test_loss_reduce(P(ga), P(na), P(loss), 500, 777, 0, ST()))
    ok(T.dtx_test_loss_reduce(P(gb), P(nb), P(loss), 700, 777, 1, ST()))
    ref = (float(ga.double().sum()) + float(gb.double().sum())) / 777
    assert abs(float(loss[0]) - ref) / ref < 1e-6, (float(loss[0]), ref)


@gpu
def test_row_loss_stats_rectangular_and_packed(T):
    """per-sequence loss sums and label counts; row losses are multiples of 1/8, so every summation order is exact"""
    torch = _torch()
    S = 640
    lens = np.array([640, 0, 1, 129, 300, 128], np.int32)
    B = len(lens)
    _, labels = _ragged_batch(B, S, lens, seed=21)
    shifted = _shift_ref_rect(labels).reshape(B, S)
    rng = np.random.default_rng(22)
    rl = (rng.integers(1, 64, (B, S)) / 8.0).astype(np.float32) * (shifted >= 0)
    for packed in (False, True):
        if packed:
            starts = pack_plan(lens, S)
            r_sh = np.concatenate([shifted[b, :starts[b + 1] - starts[b]] for b in range(B)])
            r_rl = np.concatenate([rl[b, :starts[b + 1] - starts[b]] for b in range(B)])
            rs_d = dev(np.array(starts, np.int32))
        else:
            r_sh, r_rl, rs_d = shifted.reshape(-1), rl.reshape(-1), None
        row_sum, row_valid = torch.full((B + 1,), float("nan"), device="cuda"), sentinel_i32(B + 1)
        rl_d, sh_d = dev(r_rl), dev(r_sh)
        ok(T.dtx_test_row_loss_stats(P(rl_d), P(sh_d), B, S, P(row_sum), P(row_valid), P(rs_d), ST()))
        assert np.array_equal(row_sum.cpu().numpy()[:B], rl.astype(np.float64).sum(1).astype(np.float32)), packed
        assert np.array_equal(row_valid.cpu().numpy()[:B], (shifted >= 0).sum(1).astype(np.int32)), packed
        assert math.isnan(float(row_sum[B])) and int(row_valid[B]) == SENT


@gpu
def test_compacted_final_norm(T):
    """rmsnorm_fwd with a row map writes only the mapped rows (bitwise the uncompacted norm's rows), rstd only for them;
    rmsnorm_bwd scatters the compact gradient back and gives dres (or 0) on unmapped rows; both against autograd."""
    torch = _torch()
    M, d, eps = 300, 4096, 1e-5
    rng = np.random.default_rng(31)
    mapped = rng.random(M) < 0.6
    mapped[:2] = [False, True]
    row_map = np.where(mapped, np.cumsum(mapped) - 1, -1).astype(np.int32)
    nv = int(mapped.sum())
    x = rand(M, d, seed=32)
    w = (rand(d, seed=33) * 0.1 + 1).to(torch.bfloat16)
    rm_d = dev(row_map)
    y, rstd = nan(M, d), torch.full((M,), float("nan"), device="cuda")
    ok(T.dtx_test_rmsnorm_fwd(P(x), P(w), P(y), P(rstd), M, d, eps, P(rm_d), ST()))
    y_full, rstd_full = nan(M, d), torch.full((M,), float("nan"), device="cuda")
    ok(T.dtx_test_rmsnorm_fwd(P(x), P(w), P(y_full), P(rstd_full), M, d, eps, None, ST()))
    idx = torch.as_tensor(np.nonzero(mapped)[0]).long().cuda()
    assert torch.equal(y[:nv], y_full[idx]), "mapped rows must equal the uncompacted norm"
    assert torch.isnan(y[nv:].float()).all(), "destination rows beyond n_valid must keep their sentinel"
    assert torch.equal(rstd[idx], rstd_full[idx]) and torch.isnan(rstd[torch.as_tensor(~mapped).cuda()]).all()
    xf = x.float().requires_grad_(True)
    ref = w.float() * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps))
    assert rel_err(y[:nv], ref[idx]) < 4e-3
    dy = nan(M, d)
    dy[:nv] = rand(nv, d, seed=34)
    dy_full = torch.zeros(M, d, dtype=torch.bfloat16, device="cuda")
    dy_full[idx] = dy[:nv]
    ref.backward(dy_full.float())
    dres = rand(M, d, seed=35)
    for res in (dres, None):
        dx = nan(M, d)
        ok(T.dtx_test_rmsnorm_bwd(P(dy), P(x), P(w), P(rstd), P(res), P(dx), M, d, P(rm_d), ST()))
        unm = torch.as_tensor(~mapped).cuda()
        if res is None:
            assert float(dx[unm].float().abs().max()) == 0.0
        else:
            assert torch.equal(dx[unm], res[unm]), "unmapped rows get dres"
        want = xf.grad[idx] + (res[idx].float() if res is not None else 0)
        assert rel_err(dx[idx], want) < 4e-3
        dx_full = nan(M, d)
        ok(T.dtx_test_rmsnorm_bwd(P(dy_full), P(x), P(w), P(rstd_full), P(res), P(dx_full), M, d, None, ST()))
        assert torch.equal(dx[idx], dx_full[idx]), "scattered rows must equal the uncompacted backward"


# ---------------------------------------------------------------------------------------------------------------------------
# lm_head GEMMs with a device row count
# ---------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("pair", [1, 0])
def test_lm_head_gemms_with_m_eff(T, pair):
    """fp32 NT logits [M, V] = h W^T and bf16 NN dh [M, d] = dlogits W: rows below min(M, ceil256(m_eff)) bitwise equal to the
    GEMM without m_eff, every row beyond keeps its NaN sentinel; split-K ignores m_eff."""
    from datatunerx_b200 import lib as L
    torch = _torch()
    M, d, V = 1100, 256, 1000
    h, wl, dlog = rand(M, d, seed=41), rand(V, d, scale=0.05, seed=42), rand(M, V, scale=0.01, seed=43)
    shapes = {  # name: (A, lda, a_mn, B, ldb, b_mn, N, K, epilogue, dtype)
        "logits": (h, d, 0, wl, d, 0, V, d, L.EPI_F32, torch.float32),
        "dh": (dlog, V, 0, wl, d, 1, d, V, L.EPI_BF16, torch.bfloat16),
    }

    def run(name, m_eff, split_k=1):
        A, lda, a_mn, Bm, ldb, b_mn, N, K, epi, dt = shapes[name]
        Cm = torch.full((split_k, M, N) if split_k > 1 else (M, N), float("nan"), dtype=dt, device="cuda")
        me = dev(np.array([m_eff], np.int32)) if m_eff is not None else None
        ok(T.dtx_test_gemm_m_eff(P(A), lda, a_mn, P(Bm), ldb, b_mn, P(Cm), N, M, N, K, epi, split_k, 0, P(me), ST()))
        return Cm

    L.set_option("gemm_pair_kernel", pair)
    try:
        for name in shapes:
            full = run(name, None)
            A, _, _, Bm, _, b_mn, _, _, _, _ = shapes[name]
            ref = A.float() @ (Bm.float() if b_mn else Bm.float().t())
            assert rel_err(full, ref) < (1e-5 if name == "logits" else 6e-3), name
            for m_eff in (0, 1, 255, 256, 257, M - 1, M, M + 100):
                got = run(name, m_eff)
                live = min(M, (m_eff + 255) // 256 * 256)
                assert torch.equal(got[:live], full[:live]), (name, m_eff)
                assert torch.isnan(got[live:].float()).all(), (name, m_eff, "rows of skipped blocks were written")
        split = run("logits", None, split_k=2)
        got = run("logits", 1, split_k=2)
        assert torch.isfinite(got).all() and torch.equal(got, split), "split-K must ignore m_eff"
    finally:
        L.set_option("gemm_pair_kernel", 1)


# ---------------------------------------------------------------------------------------------------------------------------
# full-parameter SFT kernels
# ---------------------------------------------------------------------------------------------------------------------------
def _bf16_rel_close(got, ref, what):
    """got (bf16) is ref (fp64) rounded once: elementwise within one bf16 rounding, plus fp32 summation slack"""
    err = (got.double() - ref).abs()
    tol = ref.abs() * 2.0 ** -8 + 1e-5 * float(ref.abs().max())
    assert bool((err <= tol).all()), f"{what}: worst {float((err - tol).max())} above tolerance"


@gpu
@pytest.mark.parametrize("M", [37, 64 * 5 + 1, 4096])
def test_rmsnorm_dw(T, M):
    """dw[c] = sum_m dy[m, c] x[m, c] rstd[m] over 64 row blocks (fewer rows than blocks, a ragged last block, all blocks full),
    plain and accumulating into the existing bf16 gradient"""
    torch = _torch()
    d = 1024
    dy, x = rand(M, d, seed=51), rand(M, d, seed=52)
    rstd = (rand(M, seed=53, dtype=torch.float32).abs() + 0.5).contiguous()
    scratch = torch.full((64 * d,), float("nan"), device="cuda")
    ref = (dy.double() * x.double() * rstd.double()[:, None]).sum(0)
    dw = nan(d)
    ok(T.dtx_test_rmsnorm_dw(P(dy), P(x), P(rstd), M, d, P(scratch), P(dw), 0, ST()))
    _bf16_rel_close(dw, ref, "rmsnorm_dw")
    prev = rand(d, scale=5.0, seed=54)
    acc = prev.clone()
    ok(T.dtx_test_rmsnorm_dw(P(dy), P(x), P(rstd), M, d, P(scratch), P(acc), 1, ST()))
    _bf16_rel_close(acc, ref + prev.double(), "rmsnorm_dw accumulate")


@gpu
def test_embedding_bwd(T):
    """one id repeated thousands of times, the last vocabulary row, and ids outside [0, vocab) (ignored) against fp64 index_add"""
    torch = _torch()
    M, d, vocab = 6000, 256, 1000
    rng = np.random.default_rng(61)
    ids = rng.integers(0, vocab, M).astype(np.int32)
    ids[:3000] = 17
    ids[3000:3100] = vocab - 1
    ids[3100:3120] = [-1, -100, vocab, vocab + 5, -(2 ** 31), 2 ** 31 - 1] * 3 + [-1, vocab]
    dx = rand(M, d, seed=62)
    dE = rand(vocab + 8, d, seed=63, dtype=torch.float32)  # 8 rows past the vocabulary that nothing may touch
    dE0 = dE.clone()
    ids_d = dev(ids)
    ok(T.dtx_test_embedding_bwd(P(ids_d), P(dx), P(dE), M, d, vocab, ST()))
    keep = (ids >= 0) & (ids < vocab)
    kid = torch.as_tensor(ids[keep]).long().cuda()
    kx = dx[torch.as_tensor(keep).cuda()].double()
    ref = dE0.double().index_add(0, kid, kx)
    mag = dE0.double().abs().index_add(0, kid, kx.abs())
    assert bool(((dE.double() - ref).abs() <= 3e-5 * mag + 1e-6).all()), float((dE.double() - ref).abs().max())
    touched = torch.zeros(vocab + 8, dtype=torch.bool, device="cuda")
    touched[kid] = True
    assert torch.equal(dE[~touched], dE0[~touched]), "rows of ignored ids changed"


@gpu
def test_sumsq_bf16_acc_chain(T):
    torch = _torch()
    sizes = [1, 255, 256 * 296 + 3, 100003, (1 << 20) + 7]
    scratch = torch.full((296,), float("nan"), device="cuda")
    out = torch.full((2,), float("nan"), device="cuda")
    ref = 0.0
    for i, n in enumerate(sizes):
        g = rand(n, scale=0.3, seed=70 + i)
        ok(T.dtx_test_sumsq_bf16_acc(P(g), n, P(scratch), P(out), 1 if i == 0 else 0, ST()))
        ref += float((g.double() ** 2).sum())
        assert abs(float(out[0]) - ref) / ref < 1e-5, (i, n, float(out[0]), ref)
    assert math.isnan(float(out[1]))


@gpu
def test_add_f32_into_bf16_rounds_like_torch(T):
    torch = _torch()
    n = 100003
    src = rand(n, scale=3.0, seed=81, dtype=torch.float32)
    src[:4] = torch.tensor([1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -(1.0 + 2 ** -8), 3.4e38], device="cuda")  # ties to even, overflow to inf
    dst = nan(n)
    ok(T.dtx_test_add_f32_into_bf16(P(src), P(dst), n, 0, ST()))
    assert torch.equal(dst, src.to(torch.bfloat16))
    prev = rand(n, seed=82)
    acc = prev.clone()
    ok(T.dtx_test_add_f32_into_bf16(P(src), P(acc), n, 1, ST()))
    assert torch.equal(acc, (src + prev.float()).to(torch.bfloat16))


@gpu
@pytest.mark.parametrize("clip", [True, False])
def test_adamw_shard_step(T, clip):
    """three steps against torch.optim.AdamW's update (the oracle's restatement) per element: weight decay below nodecay_from
    (inside a 256-element block), none from it on; clipping on / off; the bf16 weights bitwise the rounded master."""
    from oracle import llama_lora as O
    torch = _torch()
    n, nd = 100003, 70077
    lr, b1, b2, eps, wd, gscale, max_norm = 1e-3, 0.9, 0.999, 1e-8, 0.1, 0.5, (1.0 if clip else 0.0)
    gen = torch.Generator().manual_seed(90)
    p = torch.randn(n, generator=gen)
    p[nd - 2:nd + 2] = torch.tensor([1.0, -2.0, 2.0, -1.0])
    m, v = torch.zeros(n), torch.zeros(n)
    master, md, vd = p.cuda(), m.cuda(), v.cuda()
    w = nan(n)
    gn = torch.full((1,), float("nan"), device="cuda")
    coefs = []
    for step in range(1, 4):
        g = (torch.randn(n, generator=gen) * (0.05 if step == 2 else 1e-3)).to(torch.bfloat16)
        gf, gd = g.float(), g.cuda()
        sumsq = torch.tensor([float((gf.double() ** 2).sum())], dtype=torch.float32, device="cuda")
        bias1, bias2 = float(np.float32(1.0 - b1 ** step)), float(np.float32(1.0 - b2 ** step))
        ok(T.dtx_test_adamw_shard_step(P(master), P(md), P(vd), P(gd), P(w), n, nd, lr, b1, b2, eps, wd, bias1, bias2, gscale,
                                       P(sumsq), max_norm, P(gn), ST()))
        norm = math.sqrt(float(sumsq[0])) * gscale
        coef = O.clip_coef(norm, max_norm) if clip else 1.0
        coefs.append(coef)
        gs = gf * gscale * coef
        lo, hi = slice(0, nd), slice(nd, n)
        pl, ml, vl = p[lo].clone(), m[lo].clone(), v[lo].clone()
        O.adamw_update(pl, gs[lo], ml, vl, step, lr, b1, b2, eps, wd)
        ph, mh, vh = p[hi].clone(), m[hi].clone(), v[hi].clone()
        O.adamw_update(ph, gs[hi], mh, vh, step, lr, b1, b2, eps, 0.0)
        p, m, v = torch.cat([pl, ph]), torch.cat([ml, mh]), torch.cat([vl, vh])
        assert abs(float(gn[0]) - norm) / norm < 1e-5, (float(gn[0]), norm)
        mc = master.cpu()
        e = float((mc - p).abs().max())
        assert e < 1e-6, f"step {step}: master max err {e}"
        assert float((mc[nd - 2:nd + 2] - p[nd - 2:nd + 2]).abs().max()) < 1e-6, "weight-decay boundary"
        # (v: the kernel's 1 - beta2 is formed from the fp32 beta2, 1.3e-5 relative away from the oracle's double 1 - 0.999)
        assert float((md.cpu() - m).abs().max()) < 1e-7 and float(((vd.cpu() - v).abs() / v.clamp(min=1e-20)).max()) < 5e-5
        assert torch.equal(w, master.to(torch.bfloat16)), "bf16 weights must be the rounded master"
    assert (min(coefs) < 1.0) == clip  # step 2's gradient is large enough to be clipped


def _interleave_cols(gate, up):
    """[M, F] gate and up -> the trainer's GU-interleaved [M, 2F] (128 gate columns | 128 up columns per 128 features)"""
    M, F = gate.shape
    return _torch().stack([gate.view(M, F // 128, 128), up.view(M, F // 128, 128)], dim=2).reshape(M, 2 * F).contiguous()


def _deinterleave_cols(x, F):
    M = x.shape[0]
    v = x.reshape(M, F // 128, 2, 128)
    return v[:, :, 0].reshape(M, F), v[:, :, 1].reshape(M, F)


@gpu
@pytest.mark.parametrize("M", [1, 257])
def test_swiglu_interleaved(T, M):
    """interleaved = 1 at F = 11008: against fp32 autograd, and bitwise the [gate | up] kernel on the de-interleaved columns"""
    torch = _torch()
    F = 11008
    gate, up = rand(M, F, scale=2.0, seed=101), rand(M, F, seed=102)
    gu_il, gu_cat = _interleave_cols(gate, up), torch.cat([gate, up], dim=1).contiguous()
    act_il, act_cat = nan(M, F), nan(M, F)
    ok(T.dtx_test_swiglu_fwd(P(gu_il), P(act_il), M, F, 1, ST()))
    ok(T.dtx_test_swiglu_fwd(P(gu_cat), P(act_cat), M, F, 0, ST()))
    g, u = gate.float().requires_grad_(True), up.float().requires_grad_(True)
    ref = torch.nn.functional.silu(g) * u
    assert torch.equal(act_il, act_cat)
    assert rel_err(act_il, ref) < 4e-3
    dact = rand(M, F, seed=103)
    ref.backward(dact.float())
    dgu_il, dgu_cat = nan(M, 2 * F), nan(M, 2 * F)
    ok(T.dtx_test_swiglu_bwd(P(dact), P(gu_il), P(dgu_il), M, F, 1, ST()))
    ok(T.dtx_test_swiglu_bwd(P(dact), P(gu_cat), P(dgu_cat), M, F, 0, ST()))
    dg, du = _deinterleave_cols(dgu_il, F)
    assert torch.equal(dg, dgu_cat[:, :F]) and torch.equal(du, dgu_cat[:, F:])
    assert rel_err(dg, g.grad) < 4e-3 and rel_err(du, u.grad) < 4e-3
