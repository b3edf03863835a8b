"""fp32 CPU restatement of the model families beyond Llama-2 (test infrastructure, like oracle/llama_lora.py, which it builds on):

  * scaled rotary inverse frequencies - HF rope_type "linear" (inv_freq / factor) and "llama3"
    (transformers modeling_rope_utils._compute_llama3_parameters: Llama-3.1 / 3.2);
  * Qwen2's q_proj / k_proj / v_proj biases (transformers Qwen2Attention: nn.Linear(bias=True) on q, k, v; o_proj without),
    frozen under LoRA (peft bias="none") and trained without weight decay under full-parameter SFT (HF
    Trainer.get_decay_parameter_names excludes every "bias").

With qkv_bias False and rope_scaling None every function here computes exactly what oracle.llama_lora computes.
tests/test_model_families.py pins it against the installed LlamaForCausalLM (llama3 rope) and Qwen2ForCausalLM.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch

from oracle import llama_lora as O


@dataclass
class FamilyConfig(O.OracleConfig):
    qkv_bias: bool = False
    rope_scaling: Optional[dict] = None  # HF keys: {"rope_type": "linear" | "llama3", "factor", "low_freq_factor", ...}


def inv_freq(cfg: FamilyConfig) -> torch.Tensor:
    """fp32 inverse frequencies in HF's operation order."""
    D = cfg.head_dim
    base = 1.0 / (cfg.rope_theta ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))
    rs = cfg.rope_scaling or {}
    kind = rs.get("rope_type", rs.get("type", "default"))
    if kind == "default":
        return base
    if kind == "linear":
        return base / rs["factor"]
    assert kind == "llama3", kind
    factor, low, high = rs["factor"], rs["low_freq_factor"], rs["high_freq_factor"]
    old = rs["original_max_position_embeddings"]
    low_wavelen, high_wavelen = old / low, old / high
    wavelen = 2 * math.pi / base
    scaled = torch.where(wavelen > low_wavelen, base / factor, base)
    smooth = (old / wavelen - low) / (high - low)
    smoothed = (1 - smooth) * scaled / factor + smooth * scaled
    medium = ~(wavelen < high_wavelen) * ~(wavelen > low_wavelen)
    return torch.where(medium, smoothed, scaled)


def rope_cos_sin(S: int, cfg: FamilyConfig) -> Tuple[torch.Tensor, torch.Tensor]:
    freqs = torch.outer(torch.arange(S, dtype=torch.float32), inv_freq(cfg))
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos(), emb.sin()


def init_base_weights(cfg: FamilyConfig, seed: int = 1234, tied: bool = False) -> Dict[str, torch.Tensor]:
    """oracle.llama_lora.init_base_weights plus bf16-representable q/k/v biases (N(0, 0.1): large enough to matter);
    tied = the lm_head is the embedding (tie_word_embeddings)."""
    w = O.init_base_weights(cfg, seed)
    if cfg.qkv_bias:
        g = torch.Generator().manual_seed(seed + 1)
        dkv = (cfg.n_kv_heads or cfg.n_heads) * cfg.head_dim
        for l in range(cfg.n_layers):
            p = f"model.layers.{l}.self_attn."
            for name, n in (("q_proj", cfg.n_heads * cfg.head_dim), ("k_proj", dkv), ("v_proj", dkv)):
                w[p + name + ".bias"] = O.bf16_round(torch.randn(n, generator=g) * 0.1)
    if tied:
        w["lm_head.weight"] = w["model.embed_tokens.weight"].clone()
    return w


def forward_logits(cfg: FamilyConfig, w: Dict[str, torch.Tensor], lora: Dict[str, torch.Tensor], ids: torch.Tensor,
                   drop_ctx: Optional[Tuple[int, int]] = None):
    """oracle.llama_lora.forward_logits with the family's rotary table and q/k/v biases (y = x W^T + b + LoRA, then RoPE)."""
    B, S = ids.shape
    H, D = cfg.n_heads, cfg.head_dim
    Hkv = cfg.n_kv_heads or H
    targets = [t for t in ("q_proj", "k_proj", "v_proj") if t in cfg.lora_target]
    scale = cfg.lora_alpha / cfg.lora_r
    cos, sin = rope_cos_sin(S, cfg)
    x = w["model.embed_tokens.weight"][ids.long()]
    for l in range(cfg.n_layers):
        p = f"model.layers.{l}."
        h = O.rmsnorm(x, w[p + "input_layernorm.weight"], cfg.rms_eps)

        def proj(name):
            a = lora.get(p + f"self_attn.{name}.lora_A.weight")
            b = lora.get(p + f"self_attn.{name}.lora_B.weight")
            mask = None
            if a is not None and drop_ctx is not None and cfg.lora_dropout > 0:
                key = O.dropout_key(cfg.seed, drop_ctx[0], l, drop_ctx[1])
                mask = O.dropout_mask(key, targets.index(name), B * S, cfg.hidden, cfg.lora_dropout)
            y = O.lora_linear(h, w[p + f"self_attn.{name}.weight"], a, b, scale, mask, cfg.lora_dropout)
            bias = w.get(p + f"self_attn.{name}.bias")
            return y if bias is None else y + bias

        q = proj("q_proj").view(B, S, H, D).transpose(1, 2)
        k = proj("k_proj").view(B, S, Hkv, D).transpose(1, 2)
        v = proj("v_proj").view(B, S, Hkv, D).transpose(1, 2)
        q, k = O.apply_rope(q, cos, sin), O.apply_rope(k, cos, sin)
        if Hkv != H:
            k = k.repeat_interleave(H // Hkv, dim=1)
            v = v.repeat_interleave(H // Hkv, dim=1)
        o = O.attention(q, k, v, cfg.sliding_window if S > cfg.sliding_window + 1 else 0).transpose(1, 2).reshape(B, S, H * D)
        x = x + o @ w[p + "self_attn.o_proj.weight"].t()
        h = O.rmsnorm(x, w[p + "post_attention_layernorm.weight"], cfg.rms_eps)
        g = h @ w[p + "mlp.gate_proj.weight"].t()
        u = h @ w[p + "mlp.up_proj.weight"].t()
        x = x + (torch.nn.functional.silu(g) * u) @ w[p + "mlp.down_proj.weight"].t()
    x = O.rmsnorm(x, w["model.norm.weight"], cfg.rms_eps)
    return (x @ w["lm_head.weight"].t()).float()


def no_decay(cfg: FamilyConfig, name: str) -> bool:
    """HF Trainer.get_decay_parameter_names: LayerNorm weights and every bias are excluded from weight decay."""
    return cfg.full_finetune and (name.endswith("norm.weight") or name.endswith(".bias")) or name.endswith("layernorm.weight")


class FamilyTrainer(O.OracleTrainer):
    """oracle.llama_lora.OracleTrainer over forward_logits above, with biases in the no-decay set."""

    def loss_and_grads(self, ids, labels, rank: int = 0, fwd_count: Optional[int] = None):
        for p in self.lora.values():
            p.grad = None
        if fwd_count is None:
            self.fwd_count += 1
            fwd_count = self.fwd_count
        logits = forward_logits(self.cfg, self.w, self.lora, torch.from_numpy(np.asarray(ids)).long(), (fwd_count, rank))
        loss = O.causal_lm_loss(logits, torch.from_numpy(np.asarray(labels)).long())
        loss.backward()
        return float(loss.detach()), {k: p.grad.detach().clone() for k, p in self.lora.items()}

    def eval_loss(self, ids, labels) -> float:
        self.fwd_count += 1
        with torch.no_grad():
            logits = forward_logits(self.cfg, self.w, self.lora, torch.from_numpy(np.asarray(ids)).long())
            return float(O.causal_lm_loss(logits, torch.from_numpy(np.asarray(labels)).long()))

    def step(self, batches: Sequence[Tuple[np.ndarray, np.ndarray]]) -> O.StepLog:
        cfg = self.cfg
        assert len(batches) == self.world * cfg.grad_accum
        acc = {k: torch.zeros_like(v) for k, v in self.lora.items()}
        losses = []
        base = self.fwd_count
        for i, (ids, labels) in enumerate(batches):
            loss, g = self.loss_and_grads(ids, labels, rank=i // cfg.grad_accum, fwd_count=base + (i % cfg.grad_accum) + 1)
            losses.append(loss)
            for k in acc:
                acc[k] += g[k]
        self.fwd_count = base + cfg.grad_accum
        for k in acc:
            acc[k] /= len(batches)
        self.last_grads = acc
        total_norm = math.sqrt(sum(float((g.double() ** 2).sum()) for g in acc.values()))
        coef = O.clip_coef(total_norm, cfg.max_grad_norm) if cfg.max_grad_norm > 0 else 1.0
        lr = cfg.lr * O.lr_lambda(cfg.sched, self.opt_step, cfg.warmup_steps, cfg.total_steps)
        self.opt_step += 1
        with torch.no_grad():
            for k, p in self.lora.items():
                wd = 0.0 if no_decay(cfg, k) else cfg.weight_decay
                O.adamw_update(p, acc[k] * coef, self.m[k], self.v[k], self.opt_step, lr, cfg.beta1, cfg.beta2, cfg.eps, wd)
        return O.StepLog(loss=float(np.mean(losses)), grad_norm=total_norm, lr=lr)
