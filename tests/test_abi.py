"""The C-ABI library loads (no GPU needed for that) and exports every symbol include/dtxtune.h declares."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "dtxtune.h")).read()
    return sorted(set(re.findall(r"DTX_API[^;(]*?\b(dtx_\w+)\s*\(", src)))


def test_header_and_binding_agree():
    from datatunerx_b200 import lib as L
    assert sorted(L.ABI_SYMBOLS) == _declared()


def test_library_exports_every_declared_symbol(lib):
    for name in _declared():
        assert hasattr(lib, name), name
    assert lib.dtx_abi_version() == 2


def test_no_cpu_fallback_create_fails_without_gpu(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from datatunerx_b200 import lib as L
    with pytest.raises(L.DtxError) as e:
        L.Trainer(L.ModelConfig(vocab=256, hidden=256, n_layers=1, n_heads=2, ffn=256),
                  L.TrainConfig(micro_batch=1, seq_len=128, total_steps=1, lora_dropout=0.0))
    assert e.value.code == -2  # DTX_ERR_CUDA: the product path never computes on the CPU


def test_unsupported_configs_are_rejected_loudly(lib):
    from datatunerx_b200 import lib as L
    with pytest.raises(L.DtxError):  # head_dim != 128 is not implemented: rejected before any device work
        L.Trainer(L.ModelConfig(vocab=256, hidden=256, n_layers=1, n_heads=4, head_dim=64, ffn=256),
                  L.TrainConfig(micro_batch=1, seq_len=128, total_steps=1, lora_dropout=0.0))
    with pytest.raises(L.DtxError):
        L.TrainConfig(micro_batch=1, seq_len=128, total_steps=1, lora_target=("o_proj",)).to_c()


def test_struct_layouts_match_the_header(lib):
    """ctypes mirrors of dtx_model_cfg / dtx_train_cfg: field order and count as declared in include/dtxtune.h."""
    from datatunerx_b200 import lib as L
    src = open(os.path.join(ROOT, "include", "dtxtune.h")).read()
    for cname, cls in (("dtx_model_cfg", L.ModelCfg), ("dtx_train_cfg", L.TrainCfg)):
        body = re.search(r"typedef struct \{([^}]*)\} " + cname + ";", src).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        names = []
        for decl in body.split(";"):
            decl = decl.strip()
            if decl:
                names += [n.strip() for n in decl.split(None, 1)[1].split(",")]
        assert names == [f[0] for f in cls._fields_], (cname, names)


def test_option_switches_are_known_and_unknown_names_rejected(lib):
    """Every A/B switch documented in include/dtxtune.h / kernels.h is accepted (host-side flags, no device needed)."""
    from datatunerx_b200 import lib as L
    defaults = {"gemm_pair_kernel": 1, "gemm_group_m": 16, "fused_epilogues": 1, "attn_fwd_exp_fma_every": 0, "nf4_prefetch": 1,
                "attn_dq_exp_fma_every": 0, "varlen_split": 1, "varlen_group_cost": 200, "varlen_pack": 1}
    for name, value in defaults.items():
        L.set_option(name, value)  # restores the default: raises DtxError on an unknown name
    with pytest.raises(L.DtxError):
        L.set_option("no_such_option", 1)
    for value in (0, 1, 2):
        L.set_option("varlen_split", value)
    for value in (3, -1):
        with pytest.raises(L.DtxError):
            L.set_option("varlen_split", value)
    L.set_option("varlen_split", 1)
