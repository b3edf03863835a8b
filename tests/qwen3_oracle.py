"""fp32 CPU restatement of Qwen3 and of attention widths other than the hidden size (test infrastructure, built on
tests/family_oracle.py and oracle/llama_lora.py, which it leaves as they are):

  * Qwen3's q_norm / k_norm (transformers Qwen3Attention: an RMSNorm over every head of q and of k after the projection, before
    the rotary), frozen under LoRA and trained without weight decay under full-parameter SFT (family_oracle.no_decay: HF
    Trainer.get_decay_parameter_names excludes the "_norm." names);
  * an attention width n_heads * head_dim other than hidden (Qwen3-0.6B / 4B / 32B, Mistral-Nemo): q_proj [dq, hidden],
    o_proj [hidden, dq], q_proj's lora_B [dq, r].

With qk_norm False and n_heads * head_dim == hidden every function here computes exactly what tests/family_oracle.py computes.
tests/test_qwen3.py pins it against the installed Qwen3ForCausalLM and MistralForCausalLM with an explicit head_dim.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from oracle import llama_lora as O
from tests import family_oracle as FO

no_decay = FO.no_decay


@dataclass
class FamilyConfig(FO.FamilyConfig):
    qk_norm: bool = False


def init_base_weights(cfg: FamilyConfig, seed: int = 1234, tied: bool = False) -> Dict[str, torch.Tensor]:
    """family_oracle.init_base_weights with q_proj / o_proj at the attention width and, with qk_norm, q_norm / k_norm weights
    1 + N(0, 0.1), bf16-representable (HF initialises them to 1, where they would not matter)."""
    w = FO.init_base_weights(cfg, seed, tied=tied)
    d, dq = cfg.hidden, cfg.n_heads * cfg.head_dim
    if dq != d:  # q_proj / o_proj drawn again at their own shapes (same N(0, 0.02), own stream)
        g = torch.Generator().manual_seed(seed + 2)
        for l in range(cfg.n_layers):
            p = f"model.layers.{l}.self_attn."
            w[p + "q_proj.weight"] = O.bf16_round(torch.randn(dq, d, generator=g) * 0.02)
            w[p + "o_proj.weight"] = O.bf16_round(torch.randn(d, dq, generator=g) * 0.02)
    if cfg.qk_norm:
        g = torch.Generator().manual_seed(seed + 3)
        for l in range(cfg.n_layers):
            for name in ("q_norm", "k_norm"):
                w[f"model.layers.{l}.self_attn.{name}.weight"] = O.bf16_round(1.0 + torch.randn(cfg.head_dim, generator=g) * 0.1)
    return w


def init_lora(cfg: FamilyConfig, seed: int = 4321) -> Dict[str, torch.Tensor]:
    """oracle.llama_lora.init_lora with q_proj's lora_B at the attention width [n_heads * head_dim, r]."""
    lora = O.init_lora(cfg, seed)
    for k in lora:
        if ".q_proj.lora_B" in k:
            lora[k] = torch.zeros(cfg.n_heads * cfg.head_dim, cfg.lora_r)
    return lora


def forward_logits(cfg: FamilyConfig, w: Dict[str, torch.Tensor], lora: Dict[str, torch.Tensor], ids: torch.Tensor,
                   drop_ctx: Optional[Tuple[int, int]] = None):
    """family_oracle.forward_logits with the q/k norms (y = x W^T [+ b] + LoRA, per-head RMSNorm, then RoPE) and an attention
    width of its own."""
    B, S = ids.shape
    H, D = cfg.n_heads, cfg.head_dim
    Hkv = cfg.n_kv_heads or H
    targets = [t for t in ("q_proj", "k_proj", "v_proj") if t in cfg.lora_target]
    scale = cfg.lora_alpha / cfg.lora_r
    cos, sin = FO.rope_cos_sin(S, cfg)
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

        q = proj("q_proj").view(B, S, H, D)
        k = proj("k_proj").view(B, S, Hkv, D)
        if cfg.qk_norm:
            q = O.rmsnorm(q, w[p + "self_attn.q_norm.weight"], cfg.rms_eps)
            k = O.rmsnorm(k, w[p + "self_attn.k_norm.weight"], cfg.rms_eps)
        q, k = O.apply_rope(q.transpose(1, 2), cos, sin), O.apply_rope(k.transpose(1, 2), cos, sin)
        v = proj("v_proj").view(B, S, Hkv, D).transpose(1, 2)
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


class FamilyTrainer(FO.FamilyTrainer):
    """family_oracle.FamilyTrainer over forward_logits above (the q/k norm weights fall in its no-decay set)."""

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
