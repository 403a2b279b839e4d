"""Training path of the LM attention core: causal attention (head dim 128) forward + backward as one torch.autograd.Function
over our CUDA kernels, so that gradients of every decoder layer can flow back through attention (the reference's fine-tuning
recipes train q/k/v/o_proj LoRA adapters and experts of the LM, aria/train.py, recipes/config_lora.yaml).

    forward:   aria_attention_fwd_lse  -> out [B, Tq, H*128] and the row logsumexp lse [B, H, Tq] (fp32)
    backward:  aria_attention_bwd      -> dq, dk, dv from q, k, v, out, lse and dout (P is recomputed from lse, never stored)

The forward is deterministic, so the recomputation of gradient checkpointing (use_reentrant=False, as the reference recipes
set) reproduces the saved tensors exactly.  dk and dv are bit-reproducible; dq is summed with fp32 atomics (DESIGN.md §3).
"""
from __future__ import annotations

from typing import Optional

import torch

from . import ops


class AttentionFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float, causal: bool,
                key_mask: Optional[torch.Tensor] = None):
        """q [B, H, Tq, 128], k / v [B, H, Tk, 128] contiguous bf16 -> out [B, Tq, H*128]."""
        Tq, Tk = q.shape[2], k.shape[2]
        out, lse = ops.attention(q, k, v, Tq, Tk, scale, causal, key_mask=key_mask, return_lse=True)
        ctx.save_for_backward(q, k, v, out, lse, key_mask)
        ctx.scale, ctx.causal = scale, causal
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, out, lse, key_mask = ctx.saved_tensors
        dq, dk, dv = ops.attention_bwd(q, k, v, out, dout.contiguous(), lse, q.shape[2], k.shape[2], ctx.scale, ctx.causal,
                                       key_mask=key_mask)
        return dq, dk, dv, None, None, None


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float, causal: bool = True,
              key_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Differentiable attention core: q [B, H, Tq, 128], k / v [B, H, Tk, 128] (Tq <= Tk, queries are the last Tq positions),
    key_mask [B, Tk] uint8 (1 = masked out) -> out [B, Tq, H*128]."""
    return AttentionFunction.apply(q.contiguous(), k.contiguous(), v.contiguous(), float(scale), bool(causal), key_mask)
