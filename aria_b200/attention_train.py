"""Training path of the LM attention core: causal attention (head dim 128) forward + backward as one torch.autograd.Function
over our CUDA kernels, so that gradients of every decoder layer can flow back through attention (the reference's fine-tuning
recipes train q/k/v/o_proj LoRA adapters and experts of the LM, aria/train.py, recipes/config_lora.yaml).

    forward:   aria_attention_fwd_lse  -> out [B, Tq, H*128] and the row logsumexp lse [B, H, Tq] (fp32)
    backward:  aria_attention_bwd      -> dq, dk, dv from q, k, v, out, lse and dout (P is recomputed from lse, never stored)

Packed (padding-free) batches: with cu_seqlens (int32 [n_seg+1] on the device) q / k / v are [1, H, N, 128] holding n_seg
causal sequences back to back, and the same function runs aria_attention_fwd_varlen / aria_attention_bwd_varlen.  The
backward reads the boundaries from the device only, so it adds no host synchronisation.

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
                key_mask: Optional[torch.Tensor] = None, cu_seqlens: Optional[torch.Tensor] = None):
        """q [B, H, Tq, 128], k / v [B, H, Tk, 128] contiguous bf16 -> out [B, Tq, H*128].  With cu_seqlens: B = 1, Tq = Tk = N
        packed rows, causal within each sequence, no key_mask."""
        if cu_seqlens is not None:
            assert causal and key_mask is None
            N = q.shape[2]
            out, lse = ops.attention_varlen(q, k, v, cu_seqlens, scale, return_lse=True)
            out = out.view(1, N, -1)
        else:
            Tq, Tk = q.shape[2], k.shape[2]
            out, lse = ops.attention(q, k, v, Tq, Tk, scale, causal, key_mask=key_mask, return_lse=True)
        ctx.save_for_backward(q, k, v, out, lse, key_mask, cu_seqlens)
        ctx.scale, ctx.causal = scale, causal
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, out, lse, key_mask, cu_seqlens = ctx.saved_tensors
        if cu_seqlens is not None:
            dq, dk, dv = ops.attention_varlen_bwd(q, k, v, out, dout.contiguous(), lse, cu_seqlens, ctx.scale)
        else:
            dq, dk, dv = ops.attention_bwd(q, k, v, out, dout.contiguous(), lse, q.shape[2], k.shape[2], ctx.scale, ctx.causal,
                                           key_mask=key_mask)
        return dq, dk, dv, None, None, None, None


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float, causal: bool = True,
              key_mask: Optional[torch.Tensor] = None, cu_seqlens: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Differentiable attention core: q [B, H, Tq, 128], k / v [B, H, Tk, 128] (Tq <= Tk, queries are the last Tq positions),
    key_mask [B, Tk] uint8 (1 = masked out) -> out [B, Tq, H*128].  cu_seqlens (CUDA int32 [n_seg+1], 0 .. N, no empty
    sequence): q / k / v [1, H, N, 128] are packed causal sequences (`ops.attention_varlen`) -> out [1, N, H*128]."""
    return AttentionFunction.apply(q.contiguous(), k.contiguous(), v.contiguous(), float(scale), bool(causal), key_mask,
                                   cu_seqlens)
