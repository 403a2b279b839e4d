"""Padding-free fine-tuning batches: `pack_batch` turns one padded batch of the reference recipe (`aria/train.py` collate_fn,
right- or left-padded as its attention_mask says) into one packed row that the `hf_attention` seam runs as separate causal
sequences, so no projection, expert GEMM, router or attention work is spent on pad tokens.

    input_ids      [B, T]  ->  [1, N]  the real tokens of each example, in order (N = number of real tokens)
    position_ids           ->  [1, N]  restarting at 0 for each example
    labels         [B, T]  ->  [1, N]  with each example's first label set to -100: the last token of one example never
                                       learns to predict the next example's first token
    cu_seq_lens_q / _k     ->  int32 [B+1] boundaries, max_length_q / _k the longest example, only with
                                       return_flash_attn_kwargs=True (the names, meaning and default of transformers'
                                       DataCollatorWithFlattening)
    pixel_values, pixel_mask   unchanged: the images follow their image tokens in example order, which concatenation keeps

There is no attention_mask in the result: the model hands the attention core no mask, and `hf_attention` finds the boundaries
where position_ids restart.  The reference recipe's `AriaForConditionalGeneration.forward` has a fixed signature, so feed it
the default output (`model(**pack_batch(batch))`); return_flash_attn_kwargs=True is for models that pass extra keyword
arguments on to the attention (transformers' own classes), where the boundaries then need no read from position_ids.  Only
one batch's padding is removed: there is no bin-packing across batches.  Host-side tensor reshuffling, no kernel.
"""
from __future__ import annotations

import torch

IGNORE_INDEX = -100


def pack_batch(batch: dict, return_flash_attn_kwargs: bool = False) -> dict:
    """Padded batch (input_ids, attention_mask [B, T], optional labels, pixel_values, pixel_mask, ...) -> packed batch."""
    ids = batch["input_ids"]
    mask = batch.get("attention_mask")
    if mask is None:
        mask = torch.ones_like(ids, dtype=torch.bool)
    mask = mask.to(torch.bool)
    if ids.dim() != 2 or mask.shape != ids.shape:
        raise ValueError(f"pack_batch: input_ids {tuple(ids.shape)} and attention_mask {tuple(mask.shape)} must be [B, T]")
    lens = mask.sum(dim=1)
    if bool((lens == 0).any()):
        raise ValueError("pack_batch: an example has no real token")
    # the real tokens of a row must be one contiguous run (right or left padding), so the order inside an example is kept
    first = mask.float().argmax(dim=1)
    run = torch.arange(ids.shape[1], device=ids.device)[None, :]
    if not torch.equal(mask, (run >= first[:, None]) & (run < (first + lens)[:, None])):
        raise ValueError("pack_batch: attention_mask must mark one contiguous run of tokens per example (right or left padding)")
    out = {}
    out["input_ids"] = ids[mask][None]
    out["position_ids"] = torch.cat([torch.arange(int(n), device=ids.device) for n in lens.tolist()])[None]
    cu = torch.zeros(ids.shape[0] + 1, dtype=torch.int32, device=ids.device)
    cu[1:] = torch.cumsum(lens, 0).to(torch.int32)
    if batch.get("labels") is not None:
        labels = batch["labels"][mask].clone()
        labels[cu[:-1].long()] = IGNORE_INDEX
        out["labels"] = labels[None]
    if return_flash_attn_kwargs:
        out["cu_seq_lens_q"] = cu
        out["cu_seq_lens_k"] = cu
        out["max_length_q"] = int(lens.max())
        out["max_length_k"] = int(lens.max())
    for name, value in batch.items():
        if name not in out and name not in ("input_ids", "attention_mask", "labels", "position_ids"):
            out[name] = value
    return out
