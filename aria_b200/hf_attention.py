"""Seam 2 of the drop-in boundary (SURVEY §8b): the LM attention of the reference is whatever
`LLAMA_ATTENTION_CLASSES[config._attn_implementation]` builds (aria/model/moe_lm.py:594-596, transformers 4.46.3).  From
transformers 4.48 on (5.5 in this image) that table is gone and `LlamaAttention.forward` dispatches through
`ALL_ATTENTION_FUNCTIONS[config._attn_implementation](module, q, k, v, mask, dropout=, scaling=, **kw)`.

`register()` adds the implementation key "aria_b200" there (and the FA2-style mask factory, so the model hands us `None`
for a purely causal batch and the 2-D padding mask otherwise).  The module keeps its own q/k/v/o_proj, RoPE and HF `Cache`
(`past_key_values.update`, so the KV layout stays [B, H, T, hd]); only the attention core runs on our kernels:

    prefill / chunked prefill (Tq > 1)  -> aria_attention_fwd   (causal, queries are the last Tq positions of Tk keys)
    decode (Tq == 1)                    -> aria_attention_decode (split-KV streaming kernel)
    training (Tq > 1, q/k/v need grad)  -> attention_train.AttentionFunction: aria_attention_fwd_lse, and aria_attention_bwd
                                           in the backward (works under gradient checkpointing with use_reentrant=False)

Padded batches: the 2-D padding mask becomes the kernels' key mask (prefill, decode and the backward).
No fallback: MHA with head_dim 128, bf16, CUDA, no dropout, no decode under autograd — anything else raises.
(Our own mirror `aria_b200.moe_lm.AriaAttention` fuses q/k/v + RoPE + the cache write into the projection GEMM and is what
bench.py times; this seam exists so that an unmodified HF/reference model can switch the core by changing one config string.)
"""
from __future__ import annotations

from typing import Optional

import torch

from . import ops
from .attention_train import AttentionFunction

IMPL_KEY = "aria_b200"


def aria_b200_attention_forward(module, query: torch.Tensor, key: torch.Tensor, value: torch.Tensor,
                                attention_mask: Optional[torch.Tensor], dropout: float = 0.0,
                                scaling: Optional[float] = None, is_causal: Optional[bool] = None, **kwargs):
    """query [B, H, Tq, 128], key/value [B, H, Tk, 128] (already rotated, cache-concatenated) ->
    (attn_output [B, Tq, H, 128], None) — the contract of transformers' attention interface."""
    if dropout:
        raise NotImplementedError("aria_b200 attention: dropout is not supported (inference / frozen-attention path)")
    train = torch.is_grad_enabled() and (query.requires_grad or key.requires_grad or value.requires_grad)
    if train and query.shape[2] == 1:
        raise RuntimeError("aria_b200 attention: decode (one query) has no backward; run it under torch.no_grad()")
    if is_causal is False or getattr(module, "is_causal", True) is False:
        raise NotImplementedError("aria_b200 attention: only causal self-attention goes through this seam")
    B, H, Tq, hd = query.shape
    if key.shape[1] != H or value.shape[1] != H:
        raise NotImplementedError("aria_b200 attention: grouped-query attention is not supported (Aria is MHA, 20 x 128)")
    if hd != 128:
        raise NotImplementedError(f"aria_b200 attention: head_dim must be 128, got {hd}")
    Tk = key.shape[2]
    key_mask = None
    if attention_mask is not None:
        # padded batch: the FA2-style mask factory hands over the 2-D padding mask [B, Tk] (1 = real token); a 4-D additive
        # or boolean mask (other factories) is accepted when it is "causal + key padding", which is all a causal LM produces
        m = attention_mask
        if m.dim() == 4:
            last = m[:, 0, -1, :]                      # the last query row sees every non-padded key
            m = last if last.dtype == torch.bool else (last >= 0)
        if m.dim() != 2 or m.shape[0] != B or m.shape[1] < Tk:
            raise NotImplementedError(f"aria_b200 attention: unsupported attention_mask shape {tuple(attention_mask.shape)}")
        key_mask = (m[:, -Tk:] == 0).to(torch.uint8).contiguous()
    scale = float(scaling) if scaling is not None else hd ** -0.5
    k = key.contiguous()
    v = value.contiguous()
    if k.stride() != v.stride():
        v = v.clone(memory_format=torch.contiguous_format)
    if train:
        out = AttentionFunction.apply(query.contiguous(), k, v, scale, True, key_mask)                  # [B, Tq, H*128]
        return out.view(B, Tq, H, hd), None
    if Tq == 1:
        out = ops.attention_decode(query.reshape(B, H, hd).contiguous(), k, v, Tk, scale, key_mask=key_mask)   # [B, H*128]
        return out.view(B, 1, H, hd), None
    out = ops.attention(query.contiguous(), k, v, Tq, Tk, scale, True, key_mask=key_mask)        # [B, Tq, H*128]
    return out.view(B, Tq, H, hd), None


def register() -> str:
    """Register the attention core (and its mask factory) with transformers; returns the implementation key to put in
    `config._attn_implementation`.  Idempotent.  Raises ImportError on transformers < 4.48 (use the reference's own
    `LLAMA_ATTENTION_CLASSES` table there: a subclass of LlamaAttention calling `aria_b200_attention_forward`)."""
    from transformers.modeling_utils import ALL_ATTENTION_FUNCTIONS
    ALL_ATTENTION_FUNCTIONS.register(IMPL_KEY, aria_b200_attention_forward)
    try:  # mask factory: reuse flash-attention's (None when nothing is padded, else the 2-D mask)
        from transformers.masking_utils import ALL_MASK_ATTENTION_FUNCTIONS, flash_attention_mask
        ALL_MASK_ATTENTION_FUNCTIONS.register(IMPL_KEY, flash_attention_mask)
    except ImportError:  # older 4.5x: masks are built inside the model; a causal 4-D mask would reach us and raise loudly
        pass
    return IMPL_KEY
