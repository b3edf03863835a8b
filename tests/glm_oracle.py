"""fp32 CPU restatement of GLM-4 (GlmForCausalLM: glm-4-9b-hf, glm-4-9b-chat-hf; Glm4ForCausalLM) (test infrastructure, built on
tests/qwen3_oracle.py, tests/family_oracle.py and oracle/llama_lora.py, which it leaves as they are):

  * GLM's partial interleaved rotary (transformers modeling_glm apply_rotary_pos_emb): only the first rotary_dim = head_dim / 2
    dims of every q / k head turn, in adjacent pairs (2i, 2i + 1) with inv_freq[i] = theta^(-2i / rotary_dim); the rest passes
    through;
  * the fused mlp.gate_up_proj [2F, d] of GLM checkpoints: gate rows first, then up rows (GlmMLP: chunk(2)).  The weight dicts
    here keep gate_proj / up_proj apart (so oracle.llama_lora's trainer applies unchanged); to_hf() / fuse_gate_up() give the
    checkpoint's names;
  * Glm4's post-sublayer norms (Glm4ForCausalLM: GLM-4-0414, GLM-Z1): post_self_attn_layernorm RMS-normalises the o_proj output
    and post_mlp_layernorm the down_proj output before their residual adds; frozen under LoRA, trained without weight decay
    under full-parameter SFT ("layernorm" names).

q/k/v biases come from family_oracle (qkv_bias=True).  With rope_glm False every function here computes what tests/qwen3_oracle.py
computes.  tests/test_glm.py pins it against the installed GlmForCausalLM and Glm4ForCausalLM.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from oracle import llama_lora as O
from tests import family_oracle as FO
from tests import qwen3_oracle as QO

no_decay = FO.no_decay
init_lora = QO.init_lora


@dataclass
class FamilyConfig(QO.FamilyConfig):
    rope_glm: bool = False
    post_norms: bool = False


def inv_freq(cfg: FamilyConfig) -> torch.Tensor:
    """fp32 inverse frequencies in HF's operation order (GlmRotaryEmbedding.compute_default_rope_parameters for rope_glm)."""
    if not cfg.rope_glm:
        return FO.inv_freq(cfg)
    dim = cfg.head_dim // 2
    return 1.0 / (cfg.rope_theta ** (torch.arange(0, dim, 2, dtype=torch.int64).float() / dim))


def apply_rope_glm(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """x [..., S, D]; cos / sin [S, D / 4] (one value per pair): pairs (2i, 2i + 1) of the first D / 2 dims turn by angle i."""
    rd = 2 * cos.shape[-1]
    xr, xp = x[..., :rd], x[..., rd:]
    x0, x1 = xr[..., 0::2], xr[..., 1::2]
    out = torch.stack((x0 * cos - x1 * sin, x1 * cos + x0 * sin), dim=-1).flatten(-2)
    return torch.cat([out, xp], dim=-1)


def init_base_weights(cfg: FamilyConfig, seed: int = 1234, tied: bool = False) -> Dict[str, torch.Tensor]:
    """qwen3_oracle.init_base_weights plus, with post_norms, post-sublayer norm weights 1 + N(0, 0.1), bf16-representable
    (HF initialises them to 1, where they would not matter)."""
    w = QO.init_base_weights(cfg, seed, tied=tied)
    if cfg.post_norms:
        g = torch.Generator().manual_seed(seed + 4)
        for l in range(cfg.n_layers):
            for name in ("post_self_attn_layernorm", "post_mlp_layernorm"):
                w[f"model.layers.{l}.{name}.weight"] = O.bf16_round(1.0 + torch.randn(cfg.hidden, generator=g) * 0.1)
    return w


def fuse_gate_up(w: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """gate_proj / up_proj of every layer -> one mlp.gate_up_proj [2F, d] (gate rows first), the rest unchanged"""
    out = {}
    for k, v in w.items():
        if k.endswith("mlp.gate_proj.weight"):
            out[k.replace("gate_proj", "gate_up_proj")] = torch.cat([v, w[k.replace("gate_proj", "up_proj")]], dim=0)
        elif not k.endswith("mlp.up_proj.weight"):
            out[k] = v
    return out


to_hf = fuse_gate_up


def forward_logits(cfg: FamilyConfig, w: Dict[str, torch.Tensor], lora: Dict[str, torch.Tensor], ids: torch.Tensor,
                   drop_ctx: Optional[Tuple[int, int]] = None):
    """qwen3_oracle.forward_logits with GLM's rotary (y = x W^T + b + LoRA, then the partial interleaved rotary) and, with
    post_norms, x = x + post_norm(sublayer(x)) around both sublayers."""
    if not cfg.rope_glm:
        return QO.forward_logits(cfg, w, lora, ids, drop_ctx)
    B, S = ids.shape
    H, D = cfg.n_heads, cfg.head_dim
    Hkv = cfg.n_kv_heads or H
    targets = [t for t in ("q_proj", "k_proj", "v_proj") if t in cfg.lora_target]
    scale = cfg.lora_alpha / cfg.lora_r
    freqs = torch.outer(torch.arange(S, dtype=torch.float32), inv_freq(cfg))
    cos, sin = freqs.cos(), freqs.sin()
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

        q = apply_rope_glm(proj("q_proj").view(B, S, H, D).transpose(1, 2), cos, sin)
        k = apply_rope_glm(proj("k_proj").view(B, S, Hkv, D).transpose(1, 2), cos, sin)
        v = proj("v_proj").view(B, S, Hkv, D).transpose(1, 2)
        if Hkv != H:
            k = k.repeat_interleave(H // Hkv, dim=1)
            v = v.repeat_interleave(H // Hkv, dim=1)
        o = O.attention(q, k, v, 0).transpose(1, 2).reshape(B, S, H * D)
        o = o @ w[p + "self_attn.o_proj.weight"].t()
        if cfg.post_norms:
            o = O.rmsnorm(o, w[p + "post_self_attn_layernorm.weight"], cfg.rms_eps)
        x = x + o
        h = O.rmsnorm(x, w[p + "post_attention_layernorm.weight"], cfg.rms_eps)
        g = h @ w[p + "mlp.gate_proj.weight"].t()
        u = h @ w[p + "mlp.up_proj.weight"].t()
        m = (torch.nn.functional.silu(g) * u) @ w[p + "mlp.down_proj.weight"].t()
        if cfg.post_norms:
            m = O.rmsnorm(m, w[p + "post_mlp_layernorm.weight"], cfg.rms_eps)
        x = x + m
    x = O.rmsnorm(x, w["model.norm.weight"], cfg.rms_eps)
    return (x @ w["lm_head.weight"].t()).float()


class FamilyTrainer(QO.FamilyTrainer):
    """qwen3_oracle.FamilyTrainer over forward_logits above."""

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
