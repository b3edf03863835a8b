"""Model / adapter file IO of the worker, numpy only (no torch, no safetensors package needed at run time).

  * load_model_config  : HF config.json -> ModelConfig  (AutoConfig.from_pretrained, cmd/tuning/train.py:221): Llama-2,
                         Llama-3.x (linear / llama3 rope scaling), Mistral, Qwen2 / Qwen2.5 (q/k/v biases), Qwen3 (q/k norm),
                         GLM-4 (GlmForCausalLM / Glm4ForCausalLM: partial interleaved rotary, q/k/v biases,
                         fused gate_up_proj, Glm4's post-sublayer norms), OLMo-2 (full-width q/k norm, post-sublayer norms
                         and no pre-norms)
  * iter_safetensors   : stream tensors of *.safetensors shards (AutoModelForCausalLM.from_pretrained, train.py:236-242);
                         iter_torch_bin does the same for pytorch_model*.bin shards
  * save_peft_adapter  : adapter_config.json + adapter_model.safetensors (+ adapter_model.bin when torch is importable)
                         in the layout peft 0.5.0 `save_pretrained` writes and the inference image loads
                         (train.py:300; pkg/util/generate/generate.go:287-294 CHECKPOINT_DIR)
"""
from __future__ import annotations

import glob
import json
import os
import struct
from typing import Dict, Iterator, Tuple

import numpy as np

from ..lib import ModelConfig

_ST_DTYPES = {"F32": (np.float32, 4, False), "F16": (np.float16, 2, False), "BF16": (np.uint16, 2, True)}


# HF rope types whose inverse frequencies the library builds (dtx_model_ext.rope_type); yarn, dynamic, longrope... are refused
_ROPE_TYPES = ("default", "linear", "llama3")


def load_model_config(model_dir: str, full_finetune: bool = False) -> ModelConfig:
    """HF config.json -> ModelConfig for the decoders the library trains: Llama-2 / Llama-3.x (`rope_scaling` of type linear or
    llama3), Mistral, Qwen2 / Qwen2.5 (q/k/v biases), Qwen3 (q/k RMSNorm, attention width n_heads * head_dim != hidden) and
    GLM-4 (glm-4-9b-hf, GLM-4-0414, GLM-Z1: GLM's partial interleaved rotary, q/k/v biases from `attention_bias`, and for
    Glm4ForCausalLM the post-sublayer norms) and OLMo-2 (Olmo2ForCausalLM: q_norm / k_norm over all q / k columns of a token,
    norms after the two sublayers and none before them).
    Anything that would train a different model than HF's raises ValueError."""
    cfg = json.load(open(os.path.join(model_dir, "config.json")))
    arch = (cfg.get("architectures") or ["LlamaForCausalLM"])[0]
    qwen2, qwen3 = arch == "Qwen2ForCausalLM", arch == "Qwen3ForCausalLM"
    glm4 = arch == "Glm4ForCausalLM"
    glm = arch == "GlmForCausalLM" or glm4
    olmo2 = arch == "Olmo2ForCausalLM"
    if "Llama" not in arch and "Mistral" not in arch and not qwen2 and not qwen3 and not glm and not olmo2:
        raise ValueError(f"{arch}: only Llama-family, Qwen2, Qwen3, GLM and OLMo-2 decoders are implemented natively")
    if glm:
        _check_glm(cfg, full_finetune)
    elif olmo2:
        _check_olmo2(cfg, full_finetune)
    elif cfg.get("attention_bias") or cfg.get("mlp_bias"):
        raise ValueError(f"{arch}: attention_bias / mlp_bias are not implemented natively")
    # transformers 5 names the dict `rope_parameters` (it then also carries rope_theta); older configs `rope_scaling`
    rs = cfg.get("rope_scaling") or cfg.get("rope_parameters") or None
    rope_theta = cfg.get("rope_theta", (rs or {}).get("rope_theta", 10000.0))
    if rs is not None:
        kind = rs.get("rope_type", rs.get("type", "default"))
        if kind not in _ROPE_TYPES:
            raise ValueError(f"rope_scaling type {kind!r} is not implemented natively (supported: {', '.join(_ROPE_TYPES)})")
        rs = None if kind == "default" else dict(rs)
    window = int(cfg.get("sliding_window") or 0)
    if glm and rs is not None:
        raise ValueError(f"{arch}: rope scaling {rs.get('rope_type', rs.get('type'))!r} of GLM's partial rotary is not implemented natively")
    if qwen2 or qwen3:
        # Qwen2.5 / Qwen3 ship sliding_window with use_sliding_window = false: HF then attends over the whole causal window
        name = "Qwen2" if qwen2 else "Qwen3"
        if cfg.get("use_sliding_window"):
            raise ValueError(f"{name} use_sliding_window (per-layer sliding windows) is not implemented natively")
        window = 0
        if full_finetune and cfg.get("tie_word_embeddings"):
            raise ValueError(f"full-parameter SFT of a {name} checkpoint with tie_word_embeddings would train the embedding and "
                             "lm_head as two tensors, unlike HF; use LoRA")
    heads = cfg["num_attention_heads"]
    return ModelConfig(vocab=cfg["vocab_size"], hidden=cfg["hidden_size"], n_layers=cfg["num_hidden_layers"], n_heads=heads,
                       n_kv_heads=cfg.get("num_key_value_heads", heads), head_dim=cfg.get("head_dim") or cfg["hidden_size"] // heads,
                       ffn=cfg["intermediate_size"], rms_eps=cfg.get("rms_norm_eps", 1e-5), rope_theta=rope_theta,
                       max_seq=cfg.get("max_position_embeddings", 4096), sliding_window=window,
                       qkv_bias=qwen2 or (glm and bool(cfg.get("attention_bias", True))), qk_norm=qwen3, rope_glm=glm,
                       post_norms=glm4 or olmo2, qk_norm_full=olmo2, no_pre_norms=olmo2, rope_scaling=rs)


def _check_glm(cfg: dict, full_finetune: bool) -> None:
    """What GlmForCausalLM may carry and still be the model the library trains (transformers modeling_glm)."""
    prf = cfg.get("partial_rotary_factor", (cfg.get("rope_parameters") or {}).get("partial_rotary_factor", 0.5))
    if prf != 0.5:
        raise ValueError(f"GLM partial_rotary_factor {prf}: only 0.5 (half of every head rotated) is implemented natively")
    if cfg.get("hidden_act", "silu") != "silu":
        raise ValueError(f"GLM hidden_act {cfg.get('hidden_act')!r}: only silu is implemented natively")
    if cfg.get("mlp_bias"):
        raise ValueError("GLM mlp_bias is not implemented natively")
    if full_finetune and cfg.get("tie_word_embeddings"):
        raise ValueError("full-parameter SFT of a GLM checkpoint with tie_word_embeddings would train the embedding and lm_head as "
                         "two tensors, unlike HF; use LoRA")


def _check_olmo2(cfg: dict, full_finetune: bool) -> None:
    """What Olmo2ForCausalLM may carry and still be the model the library trains (transformers modeling_olmo2)."""
    if cfg.get("attention_bias"):
        raise ValueError("OLMo-2 attention_bias is not implemented natively")
    if cfg.get("hidden_act", "silu") != "silu":
        raise ValueError(f"OLMo-2 hidden_act {cfg.get('hidden_act')!r}: only silu is implemented natively")
    if full_finetune and cfg.get("tie_word_embeddings"):
        raise ValueError("full-parameter SFT of an OLMo-2 checkpoint with tie_word_embeddings would train the embedding and lm_head "
                         "as two tensors, unlike HF; use LoRA")


def check_attention_window(model_dir: str, seq_len: int) -> None:
    """Kept for callers of the r01 API: sliding-window attention (Mistral `sliding_window`) is implemented natively - the
    window travels in ModelConfig.sliding_window and only changes the mask once seq_len exceeds it."""
    return None


def iter_safetensors(path: str) -> Iterator[Tuple[str, np.ndarray, bool]]:
    """Yields (name, array, is_bf16_bits).  bf16 tensors come back as uint16 bit patterns."""
    with open(path, "rb") as f:
        (hlen,) = struct.unpack("<Q", f.read(8))
        header = json.loads(f.read(hlen))
        base = 8 + hlen
        mm = np.memmap(path, dtype=np.uint8, mode="r")
        for name, meta in header.items():
            if name == "__metadata__":
                continue
            if meta["dtype"] not in _ST_DTYPES:
                raise ValueError(f"{name}: dtype {meta['dtype']} not supported")
            dt, _, bits = _ST_DTYPES[meta["dtype"]]
            b, e = meta["data_offsets"]
            arr = np.frombuffer(mm[base + b: base + e], dtype=dt).reshape(meta["shape"])
            yield name, arr, bits


def iter_torch_bin(path: str) -> Iterator[Tuple[str, np.ndarray, bool]]:
    """pytorch_model*.bin shards (torch pickles, the pre-safetensors HF format AutoModelForCausalLM.from_pretrained also
    accepts, cmd/tuning/train.py:236-242).  Unpickling needs torch on the host - file plumbing only, no torch compute."""
    import torch
    sd = torch.load(path, map_location="cpu", weights_only=True, mmap=True)
    for name, t in sd.items():
        if t.dtype == torch.bfloat16:
            yield name, t.contiguous().view(torch.uint16).numpy(), True
        elif t.dtype in (torch.float16, torch.float32):
            yield name, t.contiguous().numpy(), False
        else:
            yield name, t.float().contiguous().numpy(), False


def load_weights_into(trainer, model_dir: str) -> int:
    """Stream every checkpoint tensor into the trainer.  The library refuses to step while a base tensor is missing, so a
    partial checkpoint fails loudly instead of training on uninitialised memory."""
    files = sorted(glob.glob(os.path.join(model_dir, "*.safetensors")))
    readers = [(f, iter_safetensors) for f in files]
    if not files:
        bins = sorted(glob.glob(os.path.join(model_dir, "pytorch_model*.bin")))
        if not bins:
            raise FileNotFoundError(f"no *.safetensors or pytorch_model*.bin under {model_dir}")
        readers = [(f, iter_torch_bin) for f in bins]
    cfg = json.load(open(os.path.join(model_dir, "config.json")))
    n, embed, have_head = 0, None, False
    for fpath, reader in readers:
        for name, arr, bits in reader(fpath):
            if "rotary_emb.inv_freq" in name:
                continue
            arr = np.ascontiguousarray(arr)
            trainer.load_tensor(name, arr, bf16_bits=bits)
            if name.endswith("embed_tokens.weight"):
                embed = (arr, bits)
            have_head = have_head or name.endswith("lm_head.weight")
            n += 1
    if not have_head and cfg.get("tie_word_embeddings") and embed is not None:
        trainer.load_tensor("lm_head.weight", embed[0], bf16_bits=embed[1])  # tied output embedding: no separate tensor on disk
        n += 1
    return n


def write_safetensors(path: str, tensors: Dict[str, np.ndarray]) -> None:
    header, off, blobs = {}, 0, []
    for k in sorted(tensors):
        a = np.ascontiguousarray(tensors[k], dtype=np.float32)
        header[k] = {"dtype": "F32", "shape": list(a.shape), "data_offsets": [off, off + a.nbytes]}
        blobs.append(a.tobytes())
        off += a.nbytes
    header["__metadata__"] = {"format": "pt"}
    h = json.dumps(header, separators=(",", ":")).encode()
    h += b" " * ((8 - len(h) % 8) % 8)
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(h)))
        f.write(h)
        for b in blobs:
            f.write(b)


def save_full_model(out_dir: str, weights: Dict[str, np.ndarray], model_dir: str, shard_bytes: int = 5 << 30) -> None:
    """trainer.save_model of a full fine-tune: HF checkpoint directory - bf16 `model-0000x-of-0000y.safetensors` shards (uint16 bit
    patterns straight from the device), `model.safetensors.index.json`, and the base model's config / tokenizer files."""
    import shutil
    os.makedirs(out_dir, exist_ok=True)
    shards, cur, size = [], {}, 0
    for k, a in weights.items():
        if cur and size + a.nbytes > shard_bytes:
            shards.append(cur)
            cur, size = {}, 0
        cur[k] = a
        size += a.nbytes
    shards.append(cur)
    index = {"metadata": {"total_size": int(sum(a.nbytes for a in weights.values()))}, "weight_map": {}}
    for i, sh in enumerate(shards):
        name = "model.safetensors" if len(shards) == 1 else f"model-{i + 1:05d}-of-{len(shards):05d}.safetensors"
        header, off, blobs = {}, 0, []
        for k in sh:
            a = np.ascontiguousarray(sh[k], dtype=np.uint16)
            header[k] = {"dtype": "BF16", "shape": list(a.shape), "data_offsets": [off, off + a.nbytes]}
            blobs.append(a)
            off += a.nbytes
            index["weight_map"][k] = name
        header["__metadata__"] = {"format": "pt"}
        h = json.dumps(header, separators=(",", ":")).encode()
        h += b" " * ((8 - len(h) % 8) % 8)
        with open(os.path.join(out_dir, name), "wb") as f:
            f.write(struct.pack("<Q", len(h)))
            f.write(h)
            for b in blobs:
                f.write(b.tobytes())
    if len(shards) > 1:
        json.dump(index, open(os.path.join(out_dir, "model.safetensors.index.json"), "w"), indent=2)
    for fn in os.listdir(model_dir):
        if fn.endswith(".json") and not fn.endswith(".index.json") or fn.endswith(".model") or fn.startswith("tokenizer"):
            src = os.path.join(model_dir, fn)
            if os.path.isfile(src):
                shutil.copy(src, os.path.join(out_dir, fn))


def save_peft_adapter(out_dir: str, adapter: Dict[str, np.ndarray], *, base_model: str, r: int, alpha: float, dropout: float,
                      target_modules) -> None:
    os.makedirs(out_dir, exist_ok=True)
    cfg = {  # peft 0.5.0 LoraConfig.to_dict() as built at cmd/tuning/train.py:268-276
        "auto_mapping": None, "base_model_name_or_path": base_model, "bias": "none", "fan_in_fan_out": False,
        "inference_mode": True, "init_lora_weights": True, "layers_pattern": None, "layers_to_transform": None,
        "lora_alpha": alpha, "lora_dropout": dropout, "modules_to_save": None, "peft_type": "LORA", "r": r, "revision": None,
        "target_modules": list(target_modules), "task_type": "CAUSAL_LM",
    }
    json.dump(cfg, open(os.path.join(out_dir, "adapter_config.json"), "w"), indent=2, sort_keys=True)
    write_safetensors(os.path.join(out_dir, "adapter_model.safetensors"), adapter)
    try:  # peft 0.5.0 wrote adapter_model.bin (torch pickle); emit it too when torch is around (host plumbing only)
        import torch
        torch.save({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in adapter.items()}, os.path.join(out_dir, "adapter_model.bin"))
    except Exception:
        pass
