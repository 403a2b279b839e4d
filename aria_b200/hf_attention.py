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
    packed, no grad                     -> aria_attention_fwd_varlen (causal within each packed sequence)
    packed, training                    -> AttentionFunction with cu_seqlens: aria_attention_fwd_varlen (+ lse) and
                                           aria_attention_bwd_varlen

Padded batches: the 2-D padding mask becomes the kernels' key mask (prefill, decode and the backward).
Packed (padding-free) batches, as transformers' `DataCollatorWithFlattening` or `aria_b200.packing.pack_batch` make them: one
row [1, N] holding several sequences, no attention mask, `position_ids` restarting at 0 for each sequence and optionally
`cu_seq_lens_q` / `cu_seq_lens_k`.  A call is packed when attention_mask is None, B == 1, Tq == Tk (no cache prefix) and
either cu_seq_lens_* are given or position_ids is not one increasing run (transformers' `_is_packed_sequence`); the
boundaries then sit where position_ids == 0.  The boundaries are read to the host once per distinct tensor (identity and
version): every layer of one forward, and the checkpoint recompute, share the first read.  They are validated before any
kernel runs (ValueError); packing the kernels cannot honour (B > 1 with restarting positions, a cache prefix) raises
NotImplementedError.  Calls with an arange position_ids, padded batches and decode keep the paths above.
No fallback: MHA with head_dim 128, bf16, CUDA, no dropout, no decode under autograd — anything else raises.
(Our own mirror `aria_b200.moe_lm.AriaAttention` fuses q/k/v + RoPE + the cache write into the projection GEMM and is what
bench.py times; this seam exists so that an unmodified HF/reference model can switch the core by changing one config string.)
"""
from __future__ import annotations

import weakref
from typing import Optional

import torch

from . import ops
from .attention_train import AttentionFunction

IMPL_KEY = "aria_b200"

# boundary tensor -> what its host read gave; keyed on identity and version, a few entries (position_ids and cu_seq_lens_*)
_READS: list = []
_READS_MAX = 4
reads = 0   # device -> host boundary reads so far (tests count them)


def _host(t: torch.Tensor, make):
    """make(t.cpu()) once per distinct tensor t (same object, same _version)."""
    global reads
    version = _version(t)
    for ref, v, value in _READS:
        if ref() is t and v == version:
            return value
    reads += 1
    value = make(t.detach().cpu())
    _READS.insert(0, (weakref.ref(t), version, value))
    del _READS[_READS_MAX:]
    return value


def _version(t: torch.Tensor) -> int:
    try:
        return t._version
    except RuntimeError:   # an inference tensor has no version counter (and cannot change outside inference mode)
        return -1


def _cu_from_positions(pos: torch.Tensor):
    """position_ids [B, T] on the host -> None when every row is one increasing run (not packed), else the boundaries of
    row 0 (where position_ids == 0, then T) as a tuple."""
    pos = pos.reshape(-1, pos.shape[-1]).long()
    T = pos.shape[-1]
    runs = torch.arange(T)[None, :] + pos.min(dim=-1, keepdim=True).values
    if bool((runs == pos).all()):
        return None
    if pos.shape[0] != 1:
        return "batched"
    return tuple((pos[0] == 0).nonzero().view(-1).tolist()) + (T,)


def _check_cu(cu: tuple, N: int, what: str):
    if len(cu) < 2 or cu[0] != 0 or cu[-1] != N:
        raise ValueError(f"aria_b200 attention: packed boundaries {what} must run from 0 to the {N} packed rows, got "
                         f"{list(cu[:4])}{'...' if len(cu) > 4 else ''}{list(cu[-1:])}")
    if any(b <= a for a, b in zip(cu, cu[1:])):
        raise ValueError(f"aria_b200 attention: packed boundaries {what} must be increasing (no empty sequence)")


def _packed_boundaries(B: int, Tq: int, Tk: int, attention_mask, kwargs) -> Optional[torch.Tensor]:
    """The device boundaries (int32 [n_seg+1]) of a packed call, None for any other call; raises on packing the kernels
    cannot run or on malformed boundaries (before any kernel)."""
    cu_q, cu_k = kwargs.get("cu_seq_lens_q"), kwargs.get("cu_seq_lens_k")
    if cu_q is not None or cu_k is not None:
        if attention_mask is not None:
            raise NotImplementedError("aria_b200 attention: cu_seq_lens_* together with an attention_mask is not supported")
        if B != 1:
            raise NotImplementedError(f"aria_b200 attention: packed sequences (cu_seq_lens_*) need batch size 1, got {B}")
        if Tq != Tk:
            raise NotImplementedError("aria_b200 attention: packed sequences with a KV cache are not supported")
        as_tuple = lambda t: tuple(int(x) for x in t.reshape(-1).tolist())   # noqa: E731
        hq = _host(cu_q, as_tuple) if cu_q is not None else None
        hk = _host(cu_k, as_tuple) if cu_k is not None else None
        if hq is not None and hk is not None and hq != hk:
            raise ValueError("aria_b200 attention: cu_seq_lens_q must equal cu_seq_lens_k (self-attention without a cache)")
        _check_cu(hq if hq is not None else hk, Tq, "cu_seq_lens")
        src = cu_q if cu_q is not None else cu_k
        return _device_cu(src, hq if hq is not None else hk)
    pos = kwargs.get("position_ids")
    if attention_mask is not None or pos is None or Tq == 1:
        return None
    cu = _host(pos, _cu_from_positions)
    if cu is None:
        return None
    if cu == "batched" or B != 1:
        raise NotImplementedError("aria_b200 attention: position_ids restart inside a row, i.e. packed sequences, which are "
                                  f"supported at batch size 1 only (got {B}); flatten the batch into one row")
    if Tq != Tk:
        raise NotImplementedError("aria_b200 attention: packed sequences (restarting position_ids) with a KV cache are not "
                                  "supported")
    _check_cu(cu, Tq, "(from position_ids; the first position must be 0)")
    return _device_cu(None, cu, pos)


_DEVICE_CU: dict = {}


def _device_cu(src: Optional[torch.Tensor], cu: tuple, like: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The boundaries as CUDA int32 on the device of src / like; src itself when it already is that."""
    if src is not None and src.is_cuda and src.dtype == torch.int32 and src.dim() == 1 and src.is_contiguous():
        return src
    dev = (src if src is not None else like).device
    key = (cu, str(dev))
    t = _DEVICE_CU.get(key)
    if t is None:
        if len(_DEVICE_CU) >= _READS_MAX:
            _DEVICE_CU.clear()
        t = _DEVICE_CU[key] = torch.tensor(cu, dtype=torch.int32, device=dev)
    return t


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
    cu_seqlens = _packed_boundaries(B, Tq, Tk, attention_mask, kwargs)
    if cu_seqlens is not None:
        scale = float(scaling) if scaling is not None else hd ** -0.5
        q, k, v = query.contiguous(), key.contiguous(), value.contiguous()
        if train:
            out = AttentionFunction.apply(q, k, v, scale, True, None, cu_seqlens)                   # [1, N, H*128]
        else:
            out = ops.attention_varlen(q, k, v, cu_seqlens, scale)                                  # [N, H*128]
        return out.view(1, Tq, H, hd), None
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
