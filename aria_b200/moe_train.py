"""Training path of the MoE block (BASELINE cfg 5): `MoELayer` forward + backward as one torch.autograd.Function over our
CUDA kernels.  The reference gets its backward from autograd through `gmm` / ATen (aria/model/moe_lm.py:548-577); here every
gradient is an explicit kernel:

    forward (keeps h1, h, y):  router GEMM -> top-k/softmax -> 16-row-aligned stable permutation -> fc1 grouped GEMM ->
                               glu kernel -> fc2 grouped GEMM -> weighted combine (+ shared expert)
    backward:  combine_bwd (dy, dscores) -> fc2 wgrad (ragged contraction) + dgrad (weight read transposed in place)
               -> glu backward -> fc1 wgrad + dgrad -> un-permute sum -> shared-expert dgrad/wgrad -> top-k softmax backward
               -> router wgrad + dgrad

Router losses: with `router_losses=True` (the reference's `self.training` branch, moe_lm.py:257-258,271-272) the z-loss and
load-balancing-loss gradients (moe_lm.py:84-166) are added to dlogits by `aria_router_aux_bwd`, scaled by
`MoEAuxLossAutoScaler.main_loss_backward_scale` of `loss_scale_source` (read at backward time, as the reference's autograd
function does; default: aria_b200.moe_lm's holder — the trainable seam passes the reference module's own class); the default
(False) is eval-mode routing, which is what BASELINE cfg 5 times.
Expert parallelism: with a process `group` (`expert_parallel.ep_moe_layer_train`, what BASELINE cfg 5 times) this rank holds
only its slice of the experts and the same launches run with the all-to-alls inserted: the 16-padded expert blocks go to their
owners between the permute and fc1 and come back into a zeroed buffer between fc2 and the combine; backward sends dy to the
owners before the fc2 wgrad/dgrad and brings dxp back before the un-permute.  Expert weight grads stay on the owning rank;
router and shared-expert grads are per-rank partial sums (the usual data-parallel all-reduce is left to the caller).
Gradients are bf16 tensors accumulated in fp32 inside the tensor-core kernels.
"""
from __future__ import annotations

import torch

from . import _lib as L
from . import ops
from .expert_parallel import exchange_plan, exchange_rows


class MoELayerFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w_router, fc1, fc2, gate_w, up_w, down_w, topk: int, loss_coeffs=None, loss_scale_source=None,
                group=None):
        shape = x.shape
        x2 = x.reshape(-1, shape[-1]).contiguous()
        scores, idx, counts, _logits = ops.router_topk(x2, w_router, topk)
        offsets, dest, src = ops.build_permutation(idx, counts, row_align=16)
        xp = ops.permute_rows(x2, src)                       # [rows_pad, d], pad rows zero
        # the expert GEMMs' rows xe and offsets: every row here, or under a group the rows all ranks sent to my experts,
        # grouped by (source rank, local expert) (16-aligned: each expert block is sent with its pad rows)
        xe, off, plan, group_mod = xp, offsets, None, 0
        if group is not None:
            plan = exchange_plan(counts, group, row_align=16)
            xe = exchange_rows(xp, plan, group)
            off = ops.offsets_from_counts(plan[0])
            group_mod = fc1.shape[0]
        h1 = ops.grouped_gemm(xe, fc1, off, group_mod=group_mod)   # [rows, 2I]
        h = ops.swiglu_fwd(h1)
        y = ops.grouped_gemm(h, fc2, off, group_mod=group_mod)     # [rows, d]
        if group is not None:
            y = exchange_rows(y, plan, group, back=True, out=torch.zeros_like(xp))
        # shared expert: gate|up in one GEMM (two B segments), unfused glu so that the pre-activation is kept
        hs1 = ops.linear_multi(x2, [gate_w, up_w])
        hs = ops.swiglu_fwd(hs1)
        shared = ops.linear(hs, down_w)
        out = ops.unpermute_combine(y, dest, scores, shared)
        ctx.save_for_backward(x2, w_router, fc1, fc2, gate_w, up_w, down_w, scores, idx, off, dest, xe, h1, h, y, hs1, hs)
        ctx.topk = topk
        ctx.loss_coeffs = loss_coeffs
        ctx.loss_scale_source = loss_scale_source
        if loss_coeffs is not None:  # keep what the loss gradients need: the bf16 logits and tokens_per_expert
            ctx.router_logits, ctx.counts = _logits, counts
        ctx.shape, ctx.plan, ctx.group = shape, plan, group
        return out.view(shape)

    @staticmethod
    def backward(ctx, dout):
        (x2, w_router, fc1, fc2, gate_w, up_w, down_w, scores, idx, off, dest, xe, h1, h, y, hs1, hs) = ctx.saved_tensors
        plan, group = ctx.plan, ctx.group
        E, d = w_router.shape
        Is = gate_w.shape[0]
        T = x2.shape[0]
        do = dout.reshape(-1, d).contiguous()
        # a gradient nobody needs (frozen weight, input without requires_grad) is neither computed nor launched; the ones
        # computed run the same kernels in the same order as when every gradient is needed
        need_x, need_r, need_fc1, need_fc2, need_gate, need_up, need_down = ctx.needs_input_grad[:7]
        # every rank must issue the exchanges (collectives), so under a group the routed data-gradient chain always runs
        need_dxp = need_x or group is not None
        group_mod, num_sources = (0, 1) if group is None else (fc1.shape[0], len(plan[1]))
        dense = torch.tensor([0, T], dtype=torch.int32, device=do.device)  # one 16-aligned "group" for dense wgrads
        d_router = d_fc1 = d_fc2 = d_gate = d_up = d_down = dx = None
        # ---- routed experts
        dy, dscores = ops.combine_bwd(do, y, dest, scores)
        if group is not None:
            dy = exchange_rows(dy, plan, group)                                # to the experts' owners
        if need_fc2:
            d_fc2 = ops.grouped_wgrad(h, dy, off, num_sources=num_sources)    # [E, I, d]
        if need_dxp or need_fc1:
            dh = ops.grouped_gemm_nt(dy, fc2, off, group_mod=group_mod)       # dy @ fc2[e].T -> [rows, I]
            dh1 = ops.swiglu_bwd(h1, dh)
            if need_fc1:
                d_fc1 = ops.grouped_wgrad(xe, dh1, off, num_sources=num_sources)  # [E, d, 2I]
            if need_dxp:
                dxp = ops.grouped_gemm_nt(dh1, fc1, off, group_mod=group_mod)  # [rows, d]
                if group is not None:
                    dxp = exchange_rows(dxp, plan, group, back=True, out=torch.zeros_like(y))
        # ---- shared expert (out += shared: its upstream gradient is dout itself)
        if need_down:
            d_down = ops.grouped_wgrad(do, hs, dense)[0]                      # [d, Is]
        if need_x or need_gate or need_up:
            dhs = ops.matmul_kn(do, down_w)                                   # do @ down_w  ([d, Is] read as K x N)
            dhs1 = ops.swiglu_bwd(hs1, dhs)                                   # [T, 2 Is] = [d gate | d up]
            if need_gate:
                d_gate = ops.grouped_wgrad(dhs1[:, :Is], x2, dense)[0]        # [Is, d]
            if need_up:
                d_up = ops.grouped_wgrad(dhs1[:, Is:], x2, dense)[0]
            if need_x:
                dx = ops.matmul_kn(dhs1[:, :Is], gate_w)
                dx = ops.matmul_kn(dhs1[:, Is:], up_w, residual=dx)
        # ---- router
        if need_x or need_r:
            dlogits = ops.router_bwd(dscores, scores, idx, E)                 # [T, E]
            if ctx.loss_coeffs is not None:
                src = ctx.loss_scale_source
                if src is None:
                    from .moe_lm import MoEAuxLossAutoScaler as src
                z_c, aux_c = ctx.loss_coeffs
                ops.router_aux_bwd(ctx.router_logits, ctx.counts, dlogits, ctx.topk, z_c, aux_c,
                                   float(src.main_loss_backward_scale))
            if need_r:
                d_router = ops.grouped_wgrad(dlogits, x2, dense)[0]           # [E, d]
            if need_x:
                dx = ops.matmul_kn(dlogits, w_router, residual=dx)
        # ---- un-permute: dx[t] += sum_j dxp[dest[t, j]]
        if need_x:
            ones = torch.ones_like(scores)
            dx = ops.unpermute_combine(dxp, dest, ones, dx).view(ctx.shape)
        return dx, d_router, d_fc1, d_fc2, d_gate, d_up, d_down, None, None, None, None


def moe_layer_train(layer, hidden_states: torch.Tensor, router_losses: bool = False) -> torch.Tensor:
    """Differentiable `MoELayer.forward` for an `aria_b200.moe_lm.MoELayer` whose parameters require grad.
    router_losses=True adds the training-mode z-loss / load-balancing-loss gradients (coefficients from the config)."""
    cfg = layer.router.config
    coeffs = (float(cfg.moe_z_loss_coeff), float(cfg.moe_aux_loss_coeff)) if router_losses else None
    return MoELayerFunction.apply(hidden_states, layer.router.weight, layer.experts.fc1.weight, layer.experts.fc2.weight,
                                  layer.shared_experts.gate_proj.weight, layer.shared_experts.up_proj.weight,
                                  layer.shared_experts.down_proj.weight, cfg.moe_topk, coeffs)


# ------------------------------------------------------------------------------------------------ trainable seams
class GroupedGemmFunction(torch.autograd.Function):
    """Differentiable `gmm`: out[rows of e] = a[rows of e] @ w[e] over any int32 row offsets [E+1] (densely packed, as the
    reference's dispatcher produces them, or 16-aligned).  Backward: da = dy @ w[e].T (`aria_gemm`, weight read transposed
    in place), dw = a.T @ dy per group (`aria_grouped_wgrad`); each only when its input requires grad."""

    @staticmethod
    def forward(ctx, a, w, offsets):
        ctx.save_for_backward(a, w, offsets)
        return ops.grouped_gemm(a, w, offsets)

    @staticmethod
    def backward(ctx, dy):
        a, w, offsets = ctx.saved_tensors
        dy = dy.contiguous()
        da = ops.grouped_gemm_nt(dy, w, offsets) if ctx.needs_input_grad[0] else None
        dw = ops.grouped_wgrad(a, dy, offsets) if ctx.needs_input_grad[1] else None
        return da, dw, None


def experts_gemm_train(input: torch.Tensor, weight: torch.Tensor, tokens_per_expert: torch.Tensor) -> torch.Tensor:
    """Trainable drop-in for `grouped_gemm.ops.gmm(a, b, batch_sizes)` (seam 1, moe_lm.py:431-443): same contract as
    `aria_b200.moe_lm.experts_gemm` (counts [E] in any integer dtype on CPU or GPU, or int32 device offsets [E+1]), and
    the result carries a grad_fn when `input` or `weight` requires grad."""
    from .moe_lm import _as_offsets
    off = _as_offsets(tokens_per_expert, weight.shape[0], input.device)
    if torch.is_grad_enabled() and (input.requires_grad or weight.requires_grad):
        return GroupedGemmFunction.apply(input, weight, off)
    return ops.grouped_gemm(input, weight, off)


class LinearFunction(torch.autograd.Function):
    """x @ [W0 | W1 | ...].T in one GEMM (nn.Linear weights [N, K], equal N); backward as MoELayerFunction's shared expert:
    dW_i = dy_i.T @ x (`aria_grouped_wgrad`, one dense group), dx = sum_i dy_i @ W_i (`aria_gemm`, weight in place)."""

    @staticmethod
    def forward(ctx, x, *weights):
        ctx.save_for_backward(x, *weights)
        return ops.linear_multi(x, list(weights))

    @staticmethod
    def backward(ctx, dy):
        x, *weights = ctx.saved_tensors
        dy = dy.contiguous()
        N = weights[0].shape[0]
        dense = torch.tensor([0, x.shape[0]], dtype=torch.int32, device=x.device)
        dws, dx = [], None
        for i, w in enumerate(weights):
            seg = dy[:, i * N:(i + 1) * N]
            dws.append(ops.grouped_wgrad(seg, x, dense)[0] if ctx.needs_input_grad[1 + i] else None)
            if ctx.needs_input_grad[0]:
                dx = ops.matmul_kn(seg, w, residual=dx)
        return (dx, *dws)


class TopKFunction(torch.autograd.Function):
    """Router top-k + softmax over given logits [T, E] (`aria_route_from_logits`) -> (scores [T, k] bf16, idx, counts).
    Backward: dlogits = top-k softmax backward (`aria_router_bwd`) + the training-mode router-loss gradients when
    `loss_coeffs` is set (`aria_router_aux_bwd`, scaled by `loss_scale_source.main_loss_backward_scale`)."""

    @staticmethod
    def forward(ctx, logits, topk: int, loss_coeffs=None, loss_scale_source=None):
        logits = logits.contiguous()
        scores, idx, counts = ops.route_from_logits(logits, topk)
        ctx.save_for_backward(logits, scores, idx, counts)
        ctx.topk, ctx.loss_coeffs, ctx.loss_scale_source = topk, loss_coeffs, loss_scale_source
        ctx.mark_non_differentiable(idx, counts)
        return scores, idx, counts

    @staticmethod
    def backward(ctx, dscores, _didx, _dcounts):
        logits, scores, idx, counts = ctx.saved_tensors
        dlogits = ops.router_bwd(dscores.float().contiguous(), scores, idx, logits.shape[1])
        if ctx.loss_coeffs is not None:
            z_c, aux_c = ctx.loss_coeffs
            ops.router_aux_bwd(logits, counts, dlogits, ctx.topk, z_c, aux_c, float(ctx.loss_scale_source.main_loss_backward_scale))
        return dlogits, None, None, None


class PermuteFunction(torch.autograd.Function):
    """Token rows into expert order (`aria_permute_rows`, pad rows zero); backward sums each token's k copies
    (`aria_unpermute_combine` with unit scores)."""

    @staticmethod
    def forward(ctx, x, src, dest, topk: int):
        ctx.save_for_backward(dest)
        ctx.topk = topk
        return ops.permute_rows(x, src)

    @staticmethod
    def backward(ctx, dxp):
        (dest,) = ctx.saved_tensors
        ones = torch.ones((dest.numel() // ctx.topk, ctx.topk), dtype=torch.bfloat16, device=dxp.device)
        return ops.unpermute_combine(dxp.contiguous(), dest, ones), None, None, None


class CombineFunction(torch.autograd.Function):
    """out[t] = sum_j scores[t, j] * y[dest[t, j]] + shared[t] (`aria_unpermute_combine`); backward `aria_combine_bwd`."""

    @staticmethod
    def forward(ctx, y, dest, scores, shared):
        ctx.save_for_backward(y, dest, scores)
        return ops.unpermute_combine(y, dest, scores, shared)

    @staticmethod
    def backward(ctx, dout):
        y, dest, scores = ctx.saved_tensors
        dy, dscores = ops.combine_bwd(dout.contiguous(), y, dest, scores)
        return dy, None, dscores.to(scores.dtype), dout
