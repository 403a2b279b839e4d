"""Fused lm_head cross-entropy for fine-tuning: `F.cross_entropy(F.linear(hidden, weight), labels)` without the [rows, V]
logits tensor.

Only rows whose label counts are multiplied by the head, a chunk of rows at a time into one reused [chunk_rows, V] bf16
buffer.  Each chunk's logits are turned into their gradient in place (`ops.cross_entropy_rows`), which is consumed right
away by the data-gradient GEMM and the fp32-accumulating weight-gradient GEMM.  So the whole backward runs inside forward,
and only when a gradient is needed; backward scales the saved gradients by grad_output and scatters dH back to its rows.
The softmax is taken in fp32 over the bf16 logits of our GEMM, as the reference takes cross-entropy of bf16 lm_head logits.
"""
from __future__ import annotations

import torch

from . import ops

_DW_SCALE_ROWS = 8192   # rows of the fp32 weight gradient scaled and rounded at a time in backward (bounds the temporary)


def _fused_head(hidden, weight, labels, ignore_index, reduction, chunk_rows, need_h, need_w):
    """-> (loss, idx, dH over the valid rows or None, fp32 dW or None).  One host sync: the valid-row count and the label
    range, read together."""
    N, d = hidden.shape
    V = weight.shape[0]
    mask = labels != ignore_index
    kept = torch.where(mask, labels, 0)
    n, lo, hi = torch.stack([mask.sum(), kept.min(), kept.max()]).tolist() if N else (0, 0, 0)
    if lo < 0 or hi >= V:
        raise ValueError(f"linear_cross_entropy: a label outside [0, {V}) (labels span [{lo}, {hi}], ignore_index {ignore_index})")
    if n == 0:   # torch's mean over no rows is NaN, its sum 0; nothing to launch
        return torch.full((), float("nan") if reduction == "mean" else 0.0, dtype=torch.float32, device=hidden.device), None, \
            None, None
    scale = 1.0 / n if reduction == "mean" else 1.0
    idx = torch.nonzero_static(mask, size=n).squeeze(1)
    h = hidden.index_select(0, idx)
    lab = labels.index_select(0, idx)
    grad_scale = torch.full((1,), scale, dtype=torch.float32, device=hidden.device)
    row_loss = torch.empty((n,), dtype=torch.float32, device=hidden.device)
    buf = torch.empty((min(chunk_rows, n), V), dtype=hidden.dtype, device=hidden.device)
    dh = torch.empty((n, d), dtype=hidden.dtype, device=hidden.device) if need_h else None
    dw32 = torch.zeros((V, d), dtype=torch.float32, device=hidden.device) if need_w else None
    for i in range(0, n, chunk_rows):
        j = min(i + chunk_rows, n)
        h_c = h[i:j]
        g_c = ops.linear(h_c, weight, out=buf[:j - i])
        ops.cross_entropy_rows(g_c, lab[i:j], grad_scale, loss=row_loss[i:j])   # g_c now holds d(loss)/d(logits)
        if need_h:
            dh[i:j] = ops.matmul_kn(g_c, weight)
        if need_w:
            ops.wgrad_accumulate_f32(g_c, h_c, dw32)
    return row_loss.sum() * scale, idx, dh, dw32


class _LinearCrossEntropy(torch.autograd.Function):
    @staticmethod
    def forward(ctx, hidden, weight, labels, ignore_index, reduction, chunk_rows, need_h, need_w):
        loss, idx, dh, dw32 = _fused_head(hidden, weight, labels, ignore_index, reduction, chunk_rows, need_h, need_w)
        ctx.shapes = (hidden.shape, hidden.dtype, weight.shape, weight.dtype)
        ctx.saved = (idx, dh, dw32)
        return loss

    @staticmethod
    def backward(ctx, grad_out):
        (h_shape, h_dtype, w_shape, w_dtype), (idx, dh, dw32) = ctx.shapes, ctx.saved
        dhidden = dweight = None
        if ctx.needs_input_grad[0]:
            dhidden = torch.zeros(h_shape, dtype=h_dtype, device=grad_out.device)
            if dh is not None:
                dhidden.index_copy_(0, idx, (dh * grad_out).to(h_dtype))
        if ctx.needs_input_grad[1]:
            if dw32 is None:
                dweight = torch.zeros(w_shape, dtype=w_dtype, device=grad_out.device)
            else:
                dweight = torch.empty(w_shape, dtype=w_dtype, device=grad_out.device)
                for i in range(0, w_shape[0], _DW_SCALE_ROWS):
                    dweight[i:i + _DW_SCALE_ROWS] = dw32[i:i + _DW_SCALE_ROWS] * grad_out
        return dhidden, dweight, None, None, None, None, None, None


def linear_cross_entropy(hidden: torch.Tensor, weight: torch.Tensor, labels: torch.Tensor, ignore_index: int = -100,
                         reduction: str = "mean", chunk_rows: int = 4096) -> torch.Tensor:
    """fp32 scalar `F.cross_entropy(F.linear(hidden, weight), labels, ignore_index=..., reduction=...)` and its gradients.
    hidden [N, d] bf16, weight [V, d] bf16 (nn.Linear layout, V % 8 == 0), labels [N] int64.  Peak memory beyond the inputs
    and the gradients: one [min(chunk_rows, n_valid), V] bf16 logits buffer and, when the weight needs a gradient, a [V, d]
    fp32 accumulator.  A label outside [0, V) that is not ignore_index raises ValueError before any kernel runs.  With no
    valid row, `mean` is NaN and `sum` 0, both with zero gradients."""
    if reduction not in ("mean", "sum"):
        raise ValueError(f"linear_cross_entropy: reduction must be 'mean' or 'sum', got {reduction!r}")
    if hidden.dim() != 2 or weight.dim() != 2 or labels.shape != hidden.shape[:1] or hidden.shape[1] != weight.shape[1]:
        raise ValueError(f"linear_cross_entropy: expected hidden [N, d], weight [V, d], labels [N]; got "
                         f"{tuple(hidden.shape)}, {tuple(weight.shape)}, {tuple(labels.shape)}")
    if chunk_rows < 1:
        raise ValueError("linear_cross_entropy: chunk_rows must be positive")
    labels = labels.long()
    grad = torch.is_grad_enabled()
    need_h, need_w = grad and hidden.requires_grad, grad and weight.requires_grad
    if not (need_h or need_w):
        return _fused_head(hidden, weight, labels, ignore_index, reduction, chunk_rows, False, False)[0]
    return _LinearCrossEntropy.apply(hidden, weight, labels, ignore_index, reduction, chunk_rows, need_h, need_w)
