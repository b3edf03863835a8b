"""Per-layer activation recompute on the GPU (-m gpu): the "layer" layout re-runs each layer's forward inside the backward
pass with the very same launches, so every result must be BITWISE the one of the "keep" layout - losses, grad norms, learning
rates, trained adapters / weights, their gradients and the evaluation row statistics - across the features the forward pass
has (GQA, LoRA dropout, accumulation, NF4 with side-stream prefetch, packed and length-grouped ragged batches, sliding window,
full-parameter SFT).  The same harness checks that the host-buffer and the device-pointer step entries lay a batch out the same
way and compute the same bits with the same launches."""
import dataclasses

import numpy as np
import pytest

from tests.conftest import has_gpu

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _need_gpu():
    if not has_gpu():
        pytest.skip("no GPU")


def _lib():
    from datatunerx_b200 import lib as L
    return L


def _batches(vocab, B, S, n, lens_list=None):
    from oracle import llama_lora as O
    out = []
    for s in range(n):
        ids, labels = O.synthetic_batch(s, 0, B, S, vocab)
        lens = None
        if lens_list:
            lens = np.array(lens_list[s % len(lens_list)], dtype=np.int32)
            cur = max(128, -(-int(lens.max()) // 128) * 128)
            for b in range(B):
                ids[b, lens[b]:] = 0
                labels[b, lens[b]:] = -100
                labels[b, :max(1, int(lens[b]) // 3)] = -100
            ids, labels = np.ascontiguousarray(ids[:, :cur]), np.ascontiguousarray(labels[:, :cur])
        out.append((ids, labels, lens))
    return out


def _train(mc, tc, layout, batches, quant=False, eval_batches=(), options=None, entry="host", launches=False):
    """Train on `batches` from seeded weights with activation layout `layout`; everything the run returns, as bytes.
    entry "host": numpy batches through dtx_step; "device": CUDA tensors through dtx_step_device.  launches: also record the
    kernel launches of every step."""
    L = _lib()
    options = options or {}
    defaults = {"varlen_pack": 1, "varlen_split": 1}
    for k, v in options.items():
        L.set_option(k, v)
    tr = L.Trainer(mc, dataclasses.replace(tc, recompute=layout))
    try:
        assert tr.recompute == layout
        tr.init_random_weights(1234)
        if quant:
            tr.quantize_base("int4")
        if not tc.full_finetune:
            tr.init_lora(4321)
        trace, groups, evals, counts = [], [], [], []
        for ids, labels, lens in batches:
            before = tr.launch_count
            if entry == "host":
                trace.append(tr.step(ids, labels, lens))
            else:
                import torch
                d = [torch.from_numpy(a).cuda() for a in (ids, labels) + ((lens,) if lens is not None else ())]
                torch.cuda.synchronize()  # the trainer's stream does not order itself after torch's
                trace.append(tr.step_ptr(d[0].data_ptr(), d[1].data_ptr(), True, d[2].data_ptr() if lens is not None else 0,
                                         ids.shape[1]))
            counts.append(tr.launch_count - before)
            groups.append(tr.last_step_groups)
        for ids, labels, lens in eval_batches:
            sums, cnts = tr.eval_rows(ids, labels, lens)
            evals.append((sums.tobytes(), cnts.tobytes(), tr.eval_loss(ids, labels, lens)))
            assert tr.last_step_groups == groups[-1], "evaluation changed last_step_groups"
        if tc.full_finetune:
            state = {k: v.tobytes() for k, v in tr.export_weights().items()}
            grads = {k: v.tobytes() for k, v in tr.export_weights(grads=True).items()}
        else:
            state = {k: v.tobytes() for k, v in tr.export_adapter().items()}
            grads = {k: v.tobytes() for k, v in tr.export_adapter(grads=True).items()}
    finally:
        tr.close()
        for k in options:
            L.set_option(k, defaults[k])
    out = {"trace": trace, "groups": groups, "eval": evals, "state": state, "grads": grads}
    if launches:
        out["launches"] = counts
    return out


def _tiny(S=256, B=2, layers=3, heads=2, kv_heads=None, dropout=0.0, targets=("q_proj", "v_proj"), **mkw):
    L = _lib()
    mc = L.ModelConfig(vocab=2048, hidden=128 * heads, n_layers=layers, n_heads=heads, n_kv_heads=kv_heads, ffn=768, **mkw)
    tc = L.TrainConfig(micro_batch=B, seq_len=S, total_steps=20, lora_r=16, lora_alpha=32.0, lora_dropout=dropout, lr=1e-3,
                       lora_target=tuple(targets))
    return mc, tc


PACKED_LENS = [[384, 130, 7, 257], [512, 1, 128, 129], [500, 20, 300, 300], [256, 384, 64, 1]]


def _case(name):
    """(model, train config, batches, _train keyword arguments) of one parity case."""
    if name == "tiny_qv":
        mc, tc = _tiny()
        return mc, tc, _batches(2048, 2, 256, 4), {"eval_batches": _batches(2048, 2, 256, 1)}
    if name == "gqa_qkv":
        mc, tc = _tiny(heads=4, kv_heads=2, targets=("q_proj", "k_proj", "v_proj"))
        return mc, tc, _batches(2048, 2, 256, 4), {}
    if name == "dropout":
        mc, tc = _tiny(dropout=0.1)
        return mc, tc, _batches(2048, 2, 256, 4), {"eval_batches": _batches(2048, 2, 256, 1)}
    if name == "grad_accum":
        mc, tc = _tiny()
        tc.grad_accum = 2
        return mc, tc, _batches(2048, 2, 256, 8), {}
    if name == "qlora_prefetch":
        mc, tc = _tiny(S=512)
        return mc, tc, _batches(2048, 2, 512, 4), {"quant": True}
    if name == "packed":
        mc, tc = _tiny(S=512, B=4)
        b = _batches(2048, 4, 512, 4, PACKED_LENS)
        return mc, tc, b, {"eval_batches": b[:2]}
    if name == "length_groups":
        mc, tc = _tiny(S=512, B=4)
        b = _batches(2048, 4, 512, 4, PACKED_LENS)
        return mc, tc, b, {"eval_batches": b[:2], "options": {"varlen_pack": 0, "varlen_split": 2}}
    if name == "qlora_groups":  # the NF4 prefetch order across the length groups' forward + recompute + backward passes
        mc, tc = _tiny(S=512, B=4)
        return mc, tc, _batches(2048, 4, 512, 4, PACKED_LENS), {"quant": True, "options": {"varlen_pack": 0, "varlen_split": 2}}
    if name == "window":
        mc, tc = _tiny(S=512, heads=4, kv_heads=2, sliding_window=200)
        return mc, tc, _batches(2048, 2, 512, 4), {}
    if name in ("full", "full_accum"):
        mc, tc = _tiny()
        tc.full_finetune = True
        tc.lr = 1e-4
        if name == "full_accum":
            tc.grad_accum = 2
        return mc, tc, _batches(2048, 2, 256, 8 if name == "full_accum" else 4), {}
    if name == "full_packed":
        mc, tc = _tiny(S=512, B=4)
        tc.full_finetune = True
        tc.lr = 1e-4
        b = _batches(2048, 4, 512, 4, PACKED_LENS)
        return mc, tc, b, {"eval_batches": b[:2]}
    if name == "padded_lens":  # one pass at the padded shape that still carries the row lengths
        mc, tc = _tiny(S=512, B=4)
        b = _batches(2048, 4, 512, 4, PACKED_LENS)
        return mc, tc, b, {"eval_batches": b[:2], "options": {"varlen_pack": 0, "varlen_split": 0}}
    if name == "layer4_7b_width":
        L = _lib()
        mc = L.ModelConfig(vocab=32000, hidden=4096, n_layers=4, n_heads=32, ffn=11008)
        tc = L.TrainConfig(micro_batch=2, seq_len=2048, total_steps=20, lora_r=16, lora_alpha=32.0, lora_dropout=0.0, lr=1e-4)
        b = _batches(32000, 2, 2048, 4, [[2048, 700], [1500, 2048], [2048, 2048], [900, 130]])
        return mc, tc, b, {"eval_batches": b[:1]}
    raise KeyError(name)


@pytest.mark.parametrize("name", ["tiny_qv", "gqa_qkv", "dropout", "grad_accum", "qlora_prefetch", "packed", "length_groups",
                                  "qlora_groups", "window", "full", "full_accum", "layer4_7b_width"])
def test_layer_recompute_is_bitwise_keep_all(name):
    mc, tc, batches, kw = _case(name)
    keep = _train(mc, tc, "keep", batches, **kw)
    layer = _train(mc, tc, "layer", batches, **kw)
    assert sum(st for *_, st in keep["trace"]) >= 4, keep["trace"]  # at least 4 optimizer steps
    assert all(np.isfinite(l) for l, *_ in keep["trace"]), keep["trace"]
    assert keep["groups"] == layer["groups"], (keep["groups"], layer["groups"])
    if name in ("packed", "layer4_7b_width"):
        assert 0 in keep["groups"], keep["groups"]
    if name in ("length_groups", "qlora_groups"):
        assert max(keep["groups"]) >= 2, keep["groups"]
    assert keep["trace"] == layer["trace"], list(zip(keep["trace"], layer["trace"]))
    assert keep["eval"] == layer["eval"]
    assert keep["state"].keys() == layer["state"].keys()
    diff = [k for k in keep["state"] if keep["state"][k] != layer["state"][k]]
    assert not diff, f"trained tensors differ: {diff[:5]}"
    diff = [k for k in keep["grads"] if keep["grads"][k] != layer["grads"][k]]
    assert not diff, f"gradients differ: {diff[:5]}"


@pytest.mark.parametrize("name", ["tiny_qv", "dropout", "grad_accum", "packed", "length_groups", "qlora_groups", "full_accum",
                                  "full_packed", "padded_lens"])
def test_host_and_device_entries_are_bitwise_equal(name):
    """dtx_step and dtx_step_device lay a batch out the same way: same groups, same launches, bitwise the same results."""
    mc, tc, batches, kw = _case(name)
    host = _train(mc, tc, "keep", batches, entry="host", launches=True, **kw)
    dev = _train(mc, tc, "keep", batches, entry="device", launches=True, **kw)
    assert host["groups"] == dev["groups"], (host["groups"], dev["groups"])
    if name in ("packed", "full_packed"):
        assert 0 in host["groups"], host["groups"]
    if name in ("length_groups", "qlora_groups"):
        assert max(host["groups"]) >= 2, host["groups"]
    if name == "padded_lens":
        assert set(host["groups"]) == {1}, host["groups"]
    assert host["launches"] == dev["launches"], (host["launches"], dev["launches"])
    assert host["trace"] == dev["trace"], list(zip(host["trace"], dev["trace"]))
    assert host["eval"] == dev["eval"]
    assert host["state"].keys() == dev["state"].keys()
    diff = [k for k in host["state"] if host["state"][k] != dev["state"][k]]
    assert not diff, f"trained tensors differ: {diff[:5]}"
    diff = [k for k in host["grads"] if host["grads"][k] != dev["grads"][k]]
    assert not diff, f"gradients differ: {diff[:5]}"


@pytest.mark.parametrize("name", ["tiny_qv", "dropout", "full", "gqa_qkv"])
def test_device_bytes_match_the_plan(name):
    L = _lib()
    mc, tc, _, _ = _case(name)
    for layout in ("keep", "layer"):
        tr = L.Trainer(mc, dataclasses.replace(tc, recompute=layout))
        try:
            assert tr.recompute == layout
            assert tr.device_bytes == L.plan_device_bytes(mc, tc, 1, layout), (layout, tr.device_bytes)
            if name == "tiny_qv" and layout == "layer":  # the packed NF4 base replaces the bf16 one
                tr.init_random_weights(1)
                before = tr.device_bytes
                tr.quantize_base("int4")
                assert tr.device_bytes < before
        finally:
            tr.close()


def test_automatic_mode_keeps_all_on_a_small_config():
    L = _lib()
    mc, tc = _tiny()
    tr = L.Trainer(mc, tc)
    try:
        assert tc.recompute == "auto" and tr.recompute == "keep"
        assert tr.device_bytes == L.plan_device_bytes(mc, tc, 1, "keep")
    finally:
        tr.close()


def test_automatic_mode_recomputes_7b_at_32k_tokens():
    """Llama-2-7B LoRA at batch 8 x 4096: keeping all activations needs ~132 GB, recomputing per layer ~37 GB."""
    import torch
    L = _lib()
    mc = L.ModelConfig.llama2_7b()
    tc = L.TrainConfig(micro_batch=8, seq_len=4096, total_steps=10, lora_r=16, lora_alpha=32.0, lora_dropout=0.0, lr=1e-4)
    keep, layer = L.plan_device_bytes(mc, tc, 1, "keep"), L.plan_device_bytes(mc, tc, 1, "layer")
    free, _ = torch.cuda.mem_get_info()
    if layer + (1 << 30) > free:
        pytest.skip(f"needs {layer / 1e9:.1f} GB + 1 GiB free, {free / 1e9:.1f} GB free")
    assert keep > free
    tr = L.Trainer(mc, tc)
    try:
        assert tr.recompute == "layer"
        assert tr.device_bytes == layer
        tr.init_random_weights(1234)
        tr.init_lora(4321)
        ids, labels = _batches(32000, 8, 4096, 1)[0][:2]
        loss, gn, _, stepped = tr.step(ids, labels)
        assert stepped and np.isfinite(loss) and np.isfinite(gn), (loss, gn)
    finally:
        tr.close()
