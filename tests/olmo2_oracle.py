"""fp32 CPU restatement of OLMo-2 (Olmo2ForCausalLM: OLMo-2-1124-7B / 13B, OLMo-2-0325-32B) (test infrastructure, built on
tests/qwen3_oracle.py, tests/family_oracle.py and oracle/llama_lora.py, which it leaves as they are):

  * q_norm / k_norm over the full width of a token (transformers Olmo2Attention: q = q_norm(q_proj(x)) with one RMSNorm over all
    n_heads * head_dim q columns, the same for k over its n_kv_heads * head_dim columns), then the rotary;
  * no pre-norms (Olmo2DecoderLayer): x_mid = x + post_attention_layernorm(attn(x)), x_next = x_mid +
    post_feedforward_layernorm(mlp(x_mid)) - the q/k/v projections and the MLP read the residual stream itself.

The norm weights are frozen under LoRA and trained without weight decay under full-parameter SFT (family_oracle.no_decay).  With
neither feature every function here computes what tests/qwen3_oracle.py computes.  tests/test_olmo2.py pins it against the
installed Olmo2ForCausalLM.
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
    qk_norm_full: bool = False
    no_pre_norms: bool = False


def init_base_weights(cfg: FamilyConfig, seed: int = 1234, tied: bool = False) -> Dict[str, torch.Tensor]:
    """qwen3_oracle.init_base_weights with OLMo-2's norms, each 1 + N(0, 0.1) and bf16-representable (HF initialises them to 1,
    where they would not matter): with qk_norm_full q_norm [dq] and k_norm [dkv]; with no_pre_norms no input_layernorm, and
    post_attention_layernorm / post_feedforward_layernorm after the two sublayers."""
    w = QO.init_base_weights(cfg, seed, tied=tied)
    g = torch.Generator().manual_seed(seed + 5)
    dq, dkv = cfg.n_heads * cfg.head_dim, (cfg.n_kv_heads or cfg.n_heads) * cfg.head_dim
    for l in range(cfg.n_layers):
        p = f"model.layers.{l}."
        if cfg.qk_norm_full:
            w[p + "self_attn.q_norm.weight"] = O.bf16_round(1.0 + torch.randn(dq, generator=g) * 0.1)
            w[p + "self_attn.k_norm.weight"] = O.bf16_round(1.0 + torch.randn(dkv, generator=g) * 0.1)
        if cfg.no_pre_norms:
            del w[p + "input_layernorm.weight"]
            for name in ("post_attention_layernorm", "post_feedforward_layernorm"):
                w[p + name + ".weight"] = O.bf16_round(1.0 + torch.randn(cfg.hidden, generator=g) * 0.1)
    return w


def forward_logits(cfg: FamilyConfig, w: Dict[str, torch.Tensor], lora: Dict[str, torch.Tensor], ids: torch.Tensor,
                   drop_ctx: Optional[Tuple[int, int]] = None):
    """qwen3_oracle.forward_logits with OLMo-2's full-width q/k norms (y = x W^T + LoRA, RMSNorm over the whole q / k row, then
    RoPE) and, with no_pre_norms, x = x + post_norm(sublayer(x)) around both sublayers."""
    if not (cfg.qk_norm_full or cfg.no_pre_norms):
        return QO.forward_logits(cfg, w, lora, ids, drop_ctx)
    B, S = ids.shape
    H, D = cfg.n_heads, cfg.head_dim
    Hkv = cfg.n_kv_heads or H
    targets = [t for t in ("q_proj", "k_proj", "v_proj") if t in cfg.lora_target]
    scale = cfg.lora_alpha / cfg.lora_r
    cos, sin = FO.rope_cos_sin(S, cfg)
    x = w["model.embed_tokens.weight"][ids.long()]
    for l in range(cfg.n_layers):
        p = f"model.layers.{l}."
        h = x if cfg.no_pre_norms else O.rmsnorm(x, w[p + "input_layernorm.weight"], cfg.rms_eps)

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

        q, k = proj("q_proj"), proj("k_proj")
        if cfg.qk_norm_full:
            q = O.rmsnorm(q, w[p + "self_attn.q_norm.weight"], cfg.rms_eps)
            k = O.rmsnorm(k, w[p + "self_attn.k_norm.weight"], cfg.rms_eps)
        q = O.apply_rope(q.view(B, S, H, D).transpose(1, 2), cos, sin)
        k = O.apply_rope(k.view(B, S, Hkv, D).transpose(1, 2), cos, sin)
        v = proj("v_proj").view(B, S, Hkv, D).transpose(1, 2)
        if Hkv != H:
            k = k.repeat_interleave(H // Hkv, dim=1)
            v = v.repeat_interleave(H // Hkv, dim=1)
        o = O.attention(q, k, v, cfg.sliding_window if S > cfg.sliding_window + 1 else 0).transpose(1, 2).reshape(B, S, H * D)
        o = o @ w[p + "self_attn.o_proj.weight"].t()
        if cfg.no_pre_norms:
            x = x + O.rmsnorm(o, w[p + "post_attention_layernorm.weight"], cfg.rms_eps)
            h = x
        else:
            x = x + o
            h = O.rmsnorm(x, w[p + "post_attention_layernorm.weight"], cfg.rms_eps)
        g = h @ w[p + "mlp.gate_proj.weight"].t()
        u = h @ w[p + "mlp.up_proj.weight"].t()
        m = (torch.nn.functional.silu(g) * u) @ w[p + "mlp.down_proj.weight"].t()
        x = x + (O.rmsnorm(m, w[p + "post_feedforward_layernorm.weight"], cfg.rms_eps) if cfg.no_pre_norms else m)
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
