"""Host-side mirror of the reference's `aria/model/moe_lm.py` operator interface, running on the
H100-native kernels (libaria_b200.so).  Same class names, parameter names/shapes (HF checkpoint keys) and
argument meaning as the reference; the arithmetic is ours.

    reference                                  here
    ---------------------------------------   -------------------------------------------------------------
    TopKRouter            moe_lm.py:170-293    TopKRouter        -> aria_router_topk (GEMV + warp top-k)
    TokenDispatcher       moe_lm.py:297-365    TokenDispatcher   -> counting sort + 128-bit row gather / combine
    experts_gemm / gmm    moe_lm.py:431-443    experts_gemm      -> aria_grouped_gemm (no .cpu() sync)
    GroupedGEMM           moe_lm.py:446-484    GroupedGEMM       (class + `weight` [E,in,out] preserved for PEFT)
    GroupedMLP            moe_lm.py:487-525    GroupedMLP        -> fc1 with fused SwiGLU epilogue, fc2
    SharedExpertMLP       moe_lm.py:368-395    SharedExpertMLP   -> gate/up fused SwiGLU GEMM + down GEMM
    MoELayer              moe_lm.py:528-577    MoELayer
    MoEDecoderLayer       moe_lm.py:580-602    MoEDecoderLayer   (+ AriaAttention for LLAMA_ATTENTION_CLASSES[...])
    AriaMoELMModel        moe_lm.py:605-636    AriaMoELMModel
    AriaMoELMForCausalLM  moe_lm.py:639-679    AriaMoELMForCausalLM

These modules are the inference path (eval-mode routing, moe_lm.py:261-269); the differentiable MoE block incl. the
training-mode aux/z losses (moe_lm.py:84-166) lives in aria_b200/moe_train.py.  There is no CPU fallback.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import os

import torch
import torch.nn as nn

from . import _lib as L
from . import ops

bf16 = torch.bfloat16


class AriaMoELMConfig:
    """Plain-attribute stand-in for the reference `AriaMoELMConfig(LlamaConfig)` (moe_lm.py:43-80)."""

    def __init__(self, hidden_size=4096, num_attention_heads=32, num_hidden_layers=32, vocab_size=32000,
                 moe_intermediate_size=4096, moe_num_experts=8, moe_topk=2, moe_num_shared_experts=2,
                 moe_z_loss_coeff=1e-5, moe_aux_loss_coeff=1e-3, rms_norm_eps=1e-6, rope_theta=10000.0, **_ignored):
        self.hidden_size = hidden_size
        self.num_attention_heads = num_attention_heads
        self.num_hidden_layers = num_hidden_layers
        self.vocab_size = vocab_size
        self.moe_intermediate_size = moe_intermediate_size
        self.moe_num_experts = moe_num_experts
        self.moe_topk = moe_topk
        self.moe_num_shared_experts = moe_num_shared_experts
        self.moe_z_loss_coeff = moe_z_loss_coeff      # training-mode router losses (moe_lm.py:57-58); used by moe_train
        self.moe_aux_loss_coeff = moe_aux_loss_coeff
        self.rms_norm_eps = rms_norm_eps
        self.rope_theta = rope_theta
        self.head_dim = hidden_size // num_attention_heads


class MoEAuxLossAutoScaler:
    """Holder of the scale applied to the router-loss gradients (reference `MoEAuxLossAutoScaler`, moe_lm.py:84-125: the
    aux losses never enter the returned loss, their gradient is injected with this scale in backward)."""

    main_loss_backward_scale: float = 1.0

    @staticmethod
    def set_loss_scale(scale):
        MoEAuxLossAutoScaler.main_loss_backward_scale = float(scale)


def _param(*shape, device=None):
    return nn.Parameter(torch.empty(*shape, dtype=bf16, device=device), requires_grad=False)


class Linear(nn.Module):
    """Parameter holder with nn.Linear's names/layout (`weight` [out,in], optional `bias`)."""

    def __init__(self, in_features, out_features, bias=False, device=None):
        super().__init__()
        self.weight = _param(out_features, in_features, device=device)
        self.bias = _param(out_features, device=device) if bias else None

    def forward(self, x, act=L.ACT_NONE, residual=None):
        return ops.linear(x, self.weight, self.bias, act=act, residual=residual)


class Fp8Linear(nn.Module):
    """Linear with W8A8 weights (AriaForConditionalGeneration.quantize_dense_fp8): `weight` [out, in] torch.float8_e4m3fn,
    K-major as nn.Linear stores it, and `weight_scale` [out] fp32, one scale per output channel (amax / 448).  Both are frozen
    parameters, so a quantized model saves and reloads through its state dict (`...q_proj.weight`, `...q_proj.weight_scale`).
    The input is quantized per row to e4m3 right before the GEMM (ops.permute_quantize_fp8); both scales multiply the fp32
    accumulator before the epilogue's first bf16 rounding.  Inference only, no bias."""

    def __init__(self, in_features, out_features, device=None, weight=None, weight_scale=None):
        super().__init__()
        self.in_features = in_features
        self.out_features = out_features
        if weight is None:
            weight = torch.empty(out_features, in_features, dtype=torch.float8_e4m3fn, device=device)
        if weight_scale is None:
            weight_scale = torch.empty(out_features, dtype=torch.float32, device=device)
        if weight.shape != (out_features, in_features) or weight.dtype != torch.float8_e4m3fn:
            raise ValueError(f"weight must be [{out_features}, {in_features}] float8_e4m3fn")
        if weight_scale.shape != (out_features,) or weight_scale.dtype != torch.float32:
            raise ValueError(f"weight_scale must be [{out_features}] float32")
        self.weight = nn.Parameter(weight, requires_grad=False)
        self.weight_scale = nn.Parameter(weight_scale, requires_grad=False)

    @classmethod
    def from_linear(cls, m: "Linear") -> "Fp8Linear":
        """e4m3 codes and output-channel scales of a bias-free Linear, bit for bit
        `(w.float() / scale[:, None]).to(torch.float8_e4m3fn)` with scale = row amax / 448 (the row quantizer on [out, in])."""
        w = m.weight.detach()
        q, scale = ops.permute_quantize_fp8(w)
        return cls(w.shape[1], w.shape[0], weight=q, weight_scale=scale)

    def quantize_input(self, x: torch.Tensor):
        """x [..., in] bf16 -> (e4m3 rows [rows, in], row scales [rows])."""
        _reject_fp8_grad(x)
        return ops.permute_quantize_fp8(x.reshape(-1, x.shape[-1]))

    def forward(self, x, residual=None):
        xq, xs = self.quantize_input(x)
        return ops.linear_w8a8(xq, xs, self.weight, self.weight_scale, residual=residual).view(*x.shape[:-1], self.out_features)


def _all_fp8(mods, what: str) -> bool:
    """Whether the Linear modules `mods` are all Fp8Linear; a mix is an error."""
    f = [type(m) is Fp8Linear for m in mods]
    if any(f) and not all(f):
        raise RuntimeError(f"{what}: the projections must all be fp8 (Fp8Linear) or all not")
    return all(f)


class RMSNorm(nn.Module):
    def __init__(self, d, eps, device=None):
        super().__init__()
        self.weight = _param(d, device=device)
        self.variance_epsilon = eps

    def forward(self, x, residual=None):
        return ops.rmsnorm(x, self.weight, self.variance_epsilon, residual)


class TopKRouter(nn.Module):
    """moe_lm.py:170-293.  forward(input[T,d]) -> (scores [T,k] bf16, top_indices [T,k], tokens_per_expert [E]).
    Indices/counts are int32 and stay on the device (the reference's int64 is an ATen artefact)."""

    def __init__(self, config, device=None):
        super().__init__()
        self.config = config
        self.weight = _param(config.moe_num_experts, config.hidden_size, device=device)
        # Parity / replay hook: when set to an int32 CUDA tensor [T, k], the expert choice of the next forward() is TAKEN
        # from it (scores and counts are still computed on the device from this router's own logits).  The forced-routing
        # parity test injects the oracle's top-k here so that a bf16 near-tie in the router cannot mask other differences.
        self.forced_top_indices: Optional[torch.Tensor] = None

    def forward(self, input: torch.Tensor):
        x = input.reshape(-1, input.shape[-1])
        if self.forced_top_indices is not None:
            logits = ops.linear(x, self.weight)                                   # gating, moe_lm.py:200
            top_indices = self.forced_top_indices
            scores, tokens_per_expert = ops.route_given_indices(logits, top_indices)
            return scores, top_indices, tokens_per_expert
        scores, top_indices, tokens_per_expert, _ = ops.router_topk(x, self.weight, self.config.moe_topk)
        return scores, top_indices, tokens_per_expert


class TokenDispatcher:
    """moe_lm.py:297-365: permutes token rows into expert-sorted order and combines them back."""

    def __init__(self, config):
        self.config = config
        self.hidden_states_shape = None
        self.reversed_input_permutation_mapping = None  # dest_row: flattened (token,slot) -> sorted row
        self.expert_offsets = None

    def token_permutation(self, hidden_states: torch.Tensor, indices: torch.Tensor,
                          tokens_per_expert: Optional[torch.Tensor] = None) -> torch.Tensor:
        self.hidden_states_shape = hidden_states.shape
        x = hidden_states.reshape(-1, hidden_states.shape[-1])
        if tokens_per_expert is None:
            raise RuntimeError("tokens_per_expert (device int32 counts from the router) is required")
        offsets, dest_row, src_token = ops.build_permutation(indices, tokens_per_expert)
        self.reversed_input_permutation_mapping = dest_row
        self.expert_offsets = offsets
        return ops.permute_rows(x, src_token)

    def token_unpermutation(self, permuted_tokens: torch.Tensor, scores: torch.Tensor,
                            shared: Optional[torch.Tensor] = None) -> torch.Tensor:
        sh = None if shared is None else shared.reshape(-1, shared.shape[-1])
        out = ops.unpermute_combine(permuted_tokens, self.reversed_input_permutation_mapping, scores, sh)
        return out.view(self.hidden_states_shape)


def _as_offsets(tokens_per_expert: torch.Tensor, num_experts: int, device) -> torch.Tensor:
    """Accept what the reference passes at moe_lm.py:478-484 (per-expert counts [E], any integer dtype, CPU or
    CUDA) or our int32 device row offsets [E+1] (TokenDispatcher.expert_offsets)."""
    t = tokens_per_expert
    if t.numel() == num_experts + 1:
        if t.dtype != torch.int32:      # (CUDA residency is enforced where the pointer is taken, ops._chk)
            raise RuntimeError("row offsets must be an int32 tensor of E+1 entries")
        return t
    if t.numel() != num_experts:
        raise RuntimeError(f"tokens_per_expert must have {num_experts} (counts) or {num_experts + 1} (offsets) entries")
    return ops.offsets_from_counts(t.to(device=device, dtype=torch.int64).contiguous())


def experts_gemm(input: torch.Tensor, weight: torch.Tensor, tokens_per_expert: torch.Tensor) -> torch.Tensor:
    """Drop-in for `grouped_gemm.ops.gmm` / `sequential_gemm` as bound at moe_lm.py:431-443:
    (input [rows,K] bf16, weight [E,K,N] bf16, tokens_per_expert [E]) -> [rows,N].
    `tokens_per_expert` may be counts [E] (reference contract) or int32 device offsets [E+1]."""
    return ops.grouped_gemm(input, weight, _as_offsets(tokens_per_expert, weight.shape[0], input.device))


gmm = experts_gemm  # name used by `from grouped_gemm.ops import gmm`


class GroupedGEMM(nn.Module):
    """moe_lm.py:446-484: `weight` [groups, in_features, out_features] (out contiguous — HF layout, untouched)."""

    def __init__(self, in_features, out_features, groups, device=None):
        super().__init__()
        self.in_features = in_features
        self.out_features = out_features
        self.groups = groups
        self.weight = _param(groups, in_features, out_features, device=device)

    def forward(self, input, tokens_per_expert):
        return experts_gemm(input, self.weight, tokens_per_expert)


def _reject_fp8_grad(x: torch.Tensor):
    """The fp8 expert weights are an inference format: there is no backward through them."""
    if torch.is_grad_enabled() and x.requires_grad:
        raise RuntimeError("aria_b200: fp8 expert weights are inference-only, but the input requires grad; run under "
                           "torch.no_grad(), or train on the bf16 model")


class Fp8GroupedGEMM(nn.Module):
    """GroupedGEMM with fp8 expert weights (AriaForConditionalGeneration.quantize_experts_fp8): `weight`
    [groups, in_features, out_features] torch.float8_e4m3fn and `weight_scale` [groups, out_features] fp32, one scale per
    (expert, output column).  Both are frozen parameters, so a quantized model saves and reloads through its state dict
    (`...fc1.weight`, `...fc1.weight_scale`).
    `activations` is the mode:
      "bf16"  weight-only (W8A16): the kernel widens the weights to bf16 in shared memory.
      "fp8"   W8A8: the input is quantized per row (ops.permute_quantize_fp8) and both operands go to the fp8 tensor cores.
              fp8 wgmma reads K-major operands only, so `weight` is then the transpose(1, 2) view of a contiguous
              [groups, out_features, in_features] buffer: same shape, codes and state dict as in "bf16" mode, other strides.
    Both scales multiply the fp32 accumulator before the epilogue rounds it."""

    def __init__(self, in_features, out_features, groups, device=None, weight=None, weight_scale=None, activations="bf16"):
        super().__init__()
        if activations not in ("bf16", "fp8"):
            raise ValueError(f"activations must be 'bf16' or 'fp8', got {activations!r}")
        self.in_features = in_features
        self.out_features = out_features
        self.groups = groups
        if weight is None:
            weight = torch.empty(groups, in_features, out_features, dtype=torch.float8_e4m3fn, device=device)
        if weight_scale is None:
            weight_scale = torch.empty(groups, out_features, dtype=torch.float32, device=device)
        if weight.shape != (groups, in_features, out_features) or weight.dtype != torch.float8_e4m3fn:
            raise ValueError(f"weight must be [{groups}, {in_features}, {out_features}] float8_e4m3fn")
        if weight_scale.shape != (groups, out_features) or weight_scale.dtype != torch.float32:
            raise ValueError(f"weight_scale must be [{groups}, {out_features}] float32")
        self.activations = "bf16"
        self.weight = nn.Parameter(weight, requires_grad=False)
        self.weight_scale = nn.Parameter(weight_scale, requires_grad=False)
        self.set_activations(activations)

    @classmethod
    def from_grouped_gemm(cls, m: "GroupedGEMM") -> "Fp8GroupedGEMM":
        q, scale = ops.quantize_fp8_cols(m.weight.detach())
        return cls(m.in_features, m.out_features, m.groups, weight=q, weight_scale=scale)

    def set_activations(self, activations: str) -> None:
        """Switch between W8A16 ("bf16") and W8A8 ("fp8") by re-laying out the existing codes; nothing is re-quantized."""
        if activations not in ("bf16", "fp8"):
            raise ValueError(f"activations must be 'bf16' or 'fp8', got {activations!r}")
        w = self.weight.detach()
        if activations == "fp8" and not w.transpose(1, 2).is_contiguous():
            self.weight = nn.Parameter(w.transpose(1, 2).contiguous().transpose(1, 2), requires_grad=False)
        elif activations == "bf16" and not w.is_contiguous():
            self.weight = nn.Parameter(w.contiguous(), requires_grad=False)
        self.activations = activations

    def forward(self, input, tokens_per_expert):
        _reject_fp8_grad(input)
        off = _as_offsets(tokens_per_expert, self.groups, input.device)
        if self.activations == "fp8":
            aq, a_scale = ops.permute_quantize_fp8(input)
            return ops.grouped_gemm_w8a8(aq, a_scale, self.weight, self.weight_scale, off)
        return ops.grouped_gemm_fp8(input, self.weight, self.weight_scale, off)


class GroupedMLP(nn.Module):
    """moe_lm.py:487-525: fc1 -> glu (first half gate, second half up) -> fc2.  The glu is fused into fc1's
    epilogue with the reference's bf16 rounding points."""

    def __init__(self, config, device=None):
        super().__init__()
        self.config = config
        self.fc1 = GroupedGEMM(config.hidden_size, config.moe_intermediate_size * 2, config.moe_num_experts, device)
        self.fc2 = GroupedGEMM(config.moe_intermediate_size, config.hidden_size, config.moe_num_experts, device)

    def is_fp8(self) -> bool:
        """Whether fc1 / fc2 hold fp8 weights (Fp8GroupedGEMM); one quantized without the other is an error."""
        f1, f2 = type(self.fc1) is Fp8GroupedGEMM, type(self.fc2) is Fp8GroupedGEMM
        if f1 != f2:
            raise RuntimeError("GroupedMLP: fc1 and fc2 must both be fp8 (Fp8GroupedGEMM) or both not")
        return f1

    def fp8_activations(self) -> bool:
        """Whether fc1 / fc2 are W8A8 (Fp8GroupedGEMM with activations="fp8"); the two must be in the same mode."""
        if not self.is_fp8():
            return False
        a1, a2 = self.fc1.activations, self.fc2.activations
        if a1 != a2:
            raise RuntimeError(f"GroupedMLP: fc1 ({a1}) and fc2 ({a2}) must quantize their activations alike")
        return a1 == "fp8"

    def forward(self, permuted_tokens, tokens_per_expert):
        off = _as_offsets(tokens_per_expert, self.fc1.groups, permuted_tokens.device)
        if self.is_fp8():
            _reject_fp8_grad(permuted_tokens)
            if self.fp8_activations():
                xq, xs = ops.permute_quantize_fp8(permuted_tokens)
                h = ops.grouped_gemm_w8a8(xq, xs, self.fc1.weight, self.fc1.weight_scale, off, swiglu=True)
                hq, hs = ops.permute_quantize_fp8(h)
                return ops.grouped_gemm_w8a8(hq, hs, self.fc2.weight, self.fc2.weight_scale, off)
            h = ops.grouped_gemm_fp8(permuted_tokens, self.fc1.weight, self.fc1.weight_scale, off, swiglu=True)
            return ops.grouped_gemm_fp8(h, self.fc2.weight, self.fc2.weight_scale, off)
        if type(self.fc1) is GroupedGEMM and type(self.fc2) is GroupedGEMM:
            h = ops.grouped_gemm(permuted_tokens, self.fc1.weight, off, swiglu=True)
            return ops.grouped_gemm(h, self.fc2.weight, off)
        # fc1 / fc2 wrapped by an adapter (aria_b200.lora.GroupedGemmLoraLayer, what peft does to the reference's
        # GroupedGEMM modules, aria/train.py:107): call through the modules as the reference does (moe_lm.py:521-525);
        # the glu runs as its own (differentiable) kernel because the adapter term must be added before it
        from .lora import swiglu
        return self.fc2(swiglu(self.fc1(permuted_tokens, off)), off)


class SharedExpertMLP(nn.Module):
    """moe_lm.py:368-395 (LlamaMLP with intermediate = I * num_shared): down(silu(gate(x)) * up(x))."""

    def __init__(self, config, device=None):
        super().__init__()
        self.hidden_size = config.hidden_size
        self.intermediate_size = config.moe_intermediate_size * config.moe_num_shared_experts
        self.gate_proj = Linear(self.hidden_size, self.intermediate_size, device=device)
        self.up_proj = Linear(self.hidden_size, self.intermediate_size, device=device)
        self.down_proj = Linear(self.intermediate_size, self.hidden_size, device=device)

    def is_fp8(self) -> bool:
        """Whether gate / up / down are W8A8 (Fp8Linear, AriaForConditionalGeneration.quantize_dense_fp8)."""
        return _all_fp8((self.gate_proj, self.up_proj, self.down_proj), "SharedExpertMLP")

    def forward(self, x):
        if self.is_fp8():
            # x -> e4m3 rows -> SwiGLU (gate | up) -> h -> e4m3 rows -> down, the launches of the fused block's shared branch
            xq, xs = self.gate_proj.quantize_input(x)
            g, u = self.gate_proj, self.up_proj
            h = ops.linear_swiglu_w8a8(xq, xs, g.weight, g.weight_scale, u.weight, u.weight_scale)
            return self.down_proj(h).view(*x.shape[:-1], self.hidden_size)
        h = ops.linear_swiglu(x, self.gate_proj.weight, self.up_proj.weight)
        return ops.linear(h, self.down_proj.weight)


_SIDE_STREAMS = {}


def shared_expert_overlapped(fn, like: torch.Tensor):
    """Run `fn()` (the shared-expert branch, moe_lm.py:575: independent of the routed branch until the final add) on a side
    stream of `like`'s device, forked from / joined to the current stream — under CUDA-graph capture this becomes a parallel
    branch of the graph.  At prefill sizes the branch is two latency-bound weight-streaming GEMMs that otherwise sit
    serialised between HBM-saturating expert GEMMs.  ARIA_MOE_SIDE_STREAM=0 runs it in line."""
    import os
    if os.environ.get("ARIA_MOE_SIDE_STREAM", "1") == "0" or not like.is_cuda:
        return fn()
    dev = like.device
    side = _SIDE_STREAMS.get(dev)
    if side is None:
        side = _SIDE_STREAMS[dev] = torch.cuda.Stream(device=dev)
    cur = torch.cuda.current_stream(dev)
    side.wait_stream(cur)
    with torch.cuda.stream(side):
        out = fn()
    out.record_stream(cur)     # allocated on the side stream, consumed on the current one
    return out, side


def _side_stream(dev):
    """The per-device side stream of the shared-expert branch (None when ARIA_MOE_SIDE_STREAM=0: branch runs in line)."""
    import os
    if os.environ.get("ARIA_MOE_SIDE_STREAM", "1") == "0":
        return None
    side = _SIDE_STREAMS.get(dev)
    if side is None:
        side = _SIDE_STREAMS[dev] = torch.cuda.Stream(device=dev)
    return side


def join_side(forked, like: torch.Tensor):
    """Second half of `shared_expert_overlapped`: make the current stream wait for the side branch; returns its result."""
    if isinstance(forked, tuple):
        out, side = forked
        torch.cuda.current_stream(like.device).wait_stream(side)
        return out
    return forked


class MoELayer(nn.Module):
    """moe_lm.py:528-577.  forward(hidden_states [B,T,d]) -> [B,T,d]."""

    def __init__(self, config, device=None):
        super().__init__()
        self.router = TopKRouter(config, device)
        self.token_dispatcher = TokenDispatcher(config)
        self.experts = GroupedMLP(config, device)
        self.shared_experts = SharedExpertMLP(config, device)
        self.expert_parallel = None  # set by AriaForConditionalGeneration.enable_expert_parallel()

    def forward(self, hidden_states: torch.Tensor) -> torch.Tensor:
        if self.expert_parallel is not None:
            return self.expert_parallel(hidden_states)
        fp8 = self.experts.is_fp8()
        if fp8:
            _reject_fp8_grad(hidden_states)
        if (hidden_states.is_cuda and (fp8 or (type(self.experts.fc1) is GroupedGEMM and type(self.experts.fc2) is GroupedGEMM))
                and os.environ.get("ARIA_MOE_BLOCK", "1") != "0"):   # =0: one C-ABI call per kernel (bench.py's per-kernel table)
            # the whole block behind one C-ABI call (csrc/moe_block.cu); shared experts on the side stream of this device
            x = hidden_states.reshape(-1, hidden_states.shape[-1])
            se = self.shared_experts
            fc1, fc2 = self.experts.fc1, self.experts.fc2
            se_fp8 = se.is_fp8()
            if se_fp8:
                _reject_fp8_grad(hidden_states)
            out = ops.moe_block_fwd(x, self.router.weight, fc1.weight, fc2.weight, se.gate_proj.weight,
                                    se.up_proj.weight, se.down_proj.weight, self.router.config.moe_topk,
                                    forced_top_idx=self.router.forced_top_indices, side_stream=_side_stream(x.device),
                                    fc1_scale=fc1.weight_scale if fp8 else None, fc2_scale=fc2.weight_scale if fp8 else None,
                                    w8a8=self.experts.fp8_activations(),
                                    gate_scale=se.gate_proj.weight_scale if se_fp8 else None,
                                    up_scale=se.up_proj.weight_scale if se_fp8 else None,
                                    down_scale=se.down_proj.weight_scale if se_fp8 else None)
            return out.view(hidden_states.shape)
        # module-by-module path (adapter-wrapped experts, CPU stand-in ops of the host-logic tests)
        forked = shared_expert_overlapped(lambda: self.shared_experts(hidden_states), hidden_states)
        scores, indices, tokens_per_expert = self.router(hidden_states)
        permuted_tokens = self.token_dispatcher.token_permutation(hidden_states, indices, tokens_per_expert)
        expert_output = self.experts(permuted_tokens, self.token_dispatcher.expert_offsets)
        shared_expert_output = join_side(forked, hidden_states)
        # unpermute + score-weighted sum + `output += shared_expert_output` (moe_lm.py:573-576) in one kernel
        return self.token_dispatcher.token_unpermutation(expert_output, scores, shared_expert_output)


KV_CACHE_DTYPES = ("bf16", "fp8")


class KVCache:
    """Static per-layer KV cache in the HF layout [B, H, T_max, head_dim] (modeling_aria.py:49-50).

    dtype "bf16": k[l] / v[l] are bf16.
    dtype "fp8":  k[l] / v[l] are float8_e4m3fn codes and k_scale[l] / v_scale[l] fp32 [B, H, T_max], one scale per
                  (row, head, token): scale = amax / 448, code = e4m3(x / scale) (ops.kv_store_fp8).  There is no calibration
                  data to fix a static scale, and a dynamic scale per 128 values keeps an outlier to its own token and head
                  for 4 bytes in 132.  One bf16 staging pair k_stage / v_stage [B, H, T_max, head_dim], shared by all layers and
                  with the strides of `q`, receives the q/k/v projection's k and v rows before they are quantized; a
                  multi-token forward() attends to it in bf16 (AriaAttention.forward)."""

    def __init__(self, n_layers, B, H, T_max, hd, device, dtype="bf16"):
        if dtype not in KV_CACHE_DTYPES:
            raise ValueError(f"KV cache dtype must be 'bf16' or 'fp8', got {dtype!r}")
        self.dtype = dtype
        # rows >= seq_len are never read (the attention TMA maps cover the valid rows only), so no zero-fill
        kv_dt = torch.float8_e4m3fn if dtype == "fp8" else bf16
        self.k = [torch.empty(B, H, T_max, hd, dtype=kv_dt, device=device) for _ in range(n_layers)]
        self.v = [torch.empty(B, H, T_max, hd, dtype=kv_dt, device=device) for _ in range(n_layers)]
        self.q = torch.empty(B, H, T_max, hd, dtype=bf16, device=device)  # rows [seq_len, seq_len+T) used per step
        if dtype == "fp8":
            self.k_scale = [torch.empty(B, H, T_max, dtype=torch.float32, device=device) for _ in range(n_layers)]
            self.v_scale = [torch.empty(B, H, T_max, dtype=torch.float32, device=device) for _ in range(n_layers)]
            self.k_stage = torch.empty_like(self.q)
            self.v_stage = torch.empty_like(self.q)
        self.seq_len = 0
        self.T_max = T_max

    @property
    def n_positions(self) -> int:
        """The RoPE positions the cache spans: the length of the rope_tables its steps read."""
        return self.T_max

    def scales(self, layer):
        """(k_scale, v_scale) of a layer's fp8 cache, (None, None) for a bf16 one: the ops' k_scale= / v_scale= arguments."""
        if self.dtype == "fp8":
            return self.k_scale[layer], self.v_scale[layer]
        return None, None

    def decode_attention(self, layer, q, k, v, state: "DecodeState", scale: float) -> torch.Tensor:
        """One decode step of `layer` on this cache: the step's k, v rows [B, H, 128] are stored at cache row
        state.write_pos[b] (quantized on an fp8 cache), then q [B, H, 128] attends to rows [0, state.kv_len[b]) minus
        state.key_mask -> o [B, H*128]."""
        kc, vc = self.k[layer], self.v[layer]
        ks, vs = self.scales(layer)
        if ks is None:
            ops.kv_append(k, v, kc, vc, state.write_pos)
        else:
            ops.kv_append_fp8(k, v, kc, vc, ks, vs, state.write_pos)
        return ops.attention_decode_devlen(q, kc, vc, state.kv_len, scale, key_mask=state.key_mask, k_scale=ks, v_scale=vs)


class DecodeState:
    """Device-resident positions of a decode step that is captured once and replayed token after token
    (modeling_aria.GraphedDecode): nothing in the step reads `KVCache.seq_len` or any other host integer.
    The step's token has RoPE position rope_pos[b], its k/v land in cache row write_pos[b], and it attends to cache rows
    [0, kv_len[b]) minus the padded prompt keys of key_mask (1 = masked out).  The advance at the end of the step
    (sample_and_advance) moves all three on for every row that has not finished."""

    def __init__(self, B, H, T_max, device):
        i32 = dict(dtype=torch.int32, device=device)
        self.rope_pos = torch.zeros(B, **i32)
        self.write_pos = torch.zeros(B, **i32)
        self.kv_len = torch.ones(B, **i32)
        self.key_mask = torch.zeros(B, T_max, dtype=torch.uint8, device=device)
        self.qkv = torch.empty(3, B, H, 1, 128, dtype=bf16, device=device)  # staging rows of the step's q, k, v


class SharedPrefixCache(KVCache):
    """KV cache of G prompts decoded n times each (generate(num_return_sequences=n)): the KVCache of the G prompt rows
    [G, H, T_max, head_dim], filled once by forward()'s prefill, plus per-layer tail caches tail_k[l] / tail_v[l]
    [G*n, H, N_max, head_dim] that hold each decoded row's own tokens.  Row r = g * n + j attends to prompt g and then to its
    tail (ops.attention_decode_shared_prefix), so the prompt's keys and values are stored and read once instead of n times.
    bf16 only."""

    def __init__(self, n_layers, G, n, H, T_max, N_max, hd, device):
        super().__init__(n_layers, G, H, T_max, hd, device)
        self.group_size = n
        self.N_max = N_max
        self.tail_k = [torch.empty(G * n, H, N_max, hd, dtype=bf16, device=device) for _ in range(n_layers)]
        self.tail_v = [torch.empty(G * n, H, N_max, hd, dtype=bf16, device=device) for _ in range(n_layers)]

    @property
    def n_positions(self) -> int:
        """A row's tail continues its prompt: the prompt bucket, then the tail."""
        return self.T_max + self.N_max

    def decode_attention(self, layer, q, k, v, state: "SharedDecodeState", scale: float) -> torch.Tensor:
        """KVCache.decode_attention on the shared prompts: row r's k, v go to its tail row state.write_pos[r], then it attends
        to its group's prompt (state.prefix_lens, state.prefix_mask) and to tail rows [0, state.kv_len[r])."""
        tk, tv = self.tail_k[layer], self.tail_v[layer]
        ops.kv_append(k, v, tk, tv, state.write_pos)
        return ops.attention_decode_shared_prefix(q, self.k[layer], self.v[layer], state.prefix_lens, tk, tv, state.kv_len,
                                                  self.group_size, scale, prefix_mask=state.prefix_mask)


class SharedDecodeState(DecodeState):
    """DecodeState of the R = G * n rows of a SharedPrefixCache: write_pos[r] is the row's tail row and kv_len[r] its tail
    length; prefix_lens [G] and prefix_mask [G, T_max] (1 = padded prompt key) describe the prompt each group shares."""

    def __init__(self, G, n, H, T_max, device):
        super().__init__(G * n, H, 0, device)
        self.key_mask = None
        self.prefix_lens = torch.zeros(G, dtype=torch.int32, device=device)
        self.prefix_mask = torch.zeros(G, T_max, dtype=torch.uint8, device=device)


class LookupDecodeState(DecodeState):
    """DecodeState of prompt-lookup decoding (generate(prompt_lookup_num_tokens=K)): the 1-wide step reads the DecodeState fields
    as decode_step does; a K-wide verify step runs Q = K + 1 tokens per row, query i of row b at RoPE position pos_k[b*Q + i],
    cache row write_pos[b] + i and key count lens_k[b*Q + i] (aria_lookup_accept_advance writes both).  qkv_k: the staging rows
    of the verify step's q, k, v [3, B, H, Q, 128]."""

    def __init__(self, B, H, T_max, K, device):
        super().__init__(B, H, T_max, device)
        i32 = dict(dtype=torch.int32, device=device)
        self.pos_k = torch.zeros(B * (K + 1), **i32)
        self.lens_k = torch.ones(B * (K + 1), **i32)
        self.qkv_k = torch.empty(3, B, H, K + 1, 128, dtype=bf16, device=device)


class PagedKVCache:
    """Paged KV cache of continuous batching (serving.Engine): per-layer page pools k[l] / v[l] [n_pages, H, 256, head_dim]
    and one block table [max_rows, max_pages] int32 shared by the layers, row r listing the pages of the request in slot r
    (key 256 s + i of the request is row i of page block_table[r, s]; -1 = no page).  A page holds one decode split
    (PAGE_SIZE = the split-KV kernels' 256 keys), so the paged decode reads exactly the keys, in the order, of the contiguous
    one.  `width`: the table columns a decode step covers (its grid), set by the owner before a step is captured.

    dtype "bf16": the pools are bf16.
    dtype "fp8":  the pools are float8_e4m3fn codes, with fp32 scale pools k_scale[l] / v_scale[l] [n_pages, H, 256], one per
                  (page, head, row), quantized as KVCache(dtype="fp8") quantizes its rows (ops.kv_append_paged,
                  ops.kv_pages_store_varlen)."""

    PAGE_SIZE = 256

    def __init__(self, n_layers, n_pages, H, hd, max_rows, max_pages, device, dtype="bf16"):
        if dtype not in KV_CACHE_DTYPES:
            raise ValueError(f"KV cache dtype must be 'bf16' or 'fp8', got {dtype!r}")
        kv_dt = torch.float8_e4m3fn if dtype == "fp8" else bf16
        self.k = [torch.empty(n_pages, H, self.PAGE_SIZE, hd, dtype=kv_dt, device=device) for _ in range(n_layers)]
        self.v = [torch.empty(n_pages, H, self.PAGE_SIZE, hd, dtype=kv_dt, device=device) for _ in range(n_layers)]
        # page 0 is the null page idle rows attend to (one key): zeros, so their attention output is 0 and not whatever the
        # allocator left there; no request ever gets it, and the paged append never writes it for an idle row
        for t in self.k + self.v:
            t[0].view(torch.uint8).zero_()
        if dtype == "fp8":
            # the null page's codes are 0 and its scales 1: its key scores 0 and its value is 0, as in the bf16 pools
            self.k_scale = [torch.empty(n_pages, H, self.PAGE_SIZE, dtype=torch.float32, device=device) for _ in range(n_layers)]
            self.v_scale = [torch.empty(n_pages, H, self.PAGE_SIZE, dtype=torch.float32, device=device) for _ in range(n_layers)]
            for t in self.k_scale + self.v_scale:
                t[0].fill_(1.0)
        self.block_table = torch.full((max_rows, max_pages), -1, dtype=torch.int32, device=device)
        self.n_pages = n_pages
        self.width = max_pages
        self.dtype = dtype

    @property
    def n_positions(self) -> int:
        """The RoPE positions a request of max_pages pages spans."""
        return self.block_table.shape[1] * self.PAGE_SIZE

    scales = KVCache.scales

    def decode_attention(self, layer, q, k, v, state: "SlotDecodeState", scale: float) -> torch.Tensor:
        """KVCache.decode_attention on the pages: slot r's k, v go to its key state.write_pos[r], then it attends to its keys
        [0, state.kv_len[r]), over the first `width` columns of the block table."""
        kp, vp, bt = self.k[layer], self.v[layer], self.block_table[:, :self.width]
        ks, vs = self.scales(layer)
        ops.kv_append_paged(k, v, kp, vp, bt, state.write_pos, k_scale=ks, v_scale=vs)
        return ops.attention_decode_paged(q, kp, vp, bt, state.kv_len, scale, k_scale=ks, v_scale=vs)


def add_token_fields(st, R, max_out, device, lp_ring: int = 1, lp_width: int = ops.MAX_LOGPROBS, vocab: int = 1,
                     stops: bool = True):
    """Put on st (a DecodeState of R rows) what each row's token stream needs on the device, for sample_and_advance: its
    sampling parameters (temperature, 0 = greedy; top_k; top_p; seed; noise row; RNG offset), its token budget max_new, the
    count n_out and the tokens out_tokens [R, max_out] (int32) it has emitted, its finished flag (set: the row is idle until
    start_rows), and the step's input ids_in [R, 1] and sampled next_ids.
    Log-probabilities: lp_n, the row's top-n (-1: none), and rings of lp_ring entries that the step writes at n_out mod
    lp_ring: lp_ring_lp [R, lp_ring] fp32, lp_ring_ids [R, lp_ring, lp_width] int32 and lp_ring_top [R, lp_ring, lp_width] fp32.
    Logits processors: the row's rep_penalty (1: off), min_p (0: off) and min_new, and presence [R, ceil(vocab / 32)] int32,
    the bitmap of the ids the row has seen.
    Stops (only with stops): the row's stop set stop_bytes [R, 16, 512] uint8, stop_lens [R, 16] int32 and stop_lookback (0:
    no strings), its stop ids stop_ids [R, 8] int64 (the first n_stop_ids), and its prompt tail stop_tail [R, 128] int64, the
    last stop_tail_len ids right-aligned (ops.stop_check_slots)."""
    i32, i64 = dict(dtype=torch.int32, device=device), dict(dtype=torch.int64, device=device)
    f32 = dict(dtype=torch.float32, device=device)
    st.temperature = torch.zeros(R, **f32)
    st.top_k = torch.zeros(R, **i32)
    st.top_p = torch.ones(R, **f32)
    st.seed = torch.zeros(R, **i64)
    st.noise_row = torch.zeros(R, **i32)
    st.rng_offset = torch.zeros(R, **i64)
    st.max_new = torch.ones(R, **i32)
    st.n_out = torch.zeros(R, **i32)
    st.finished = torch.ones(R, dtype=torch.uint8, device=device)
    st.ids_in = torch.zeros(R, 1, **i64)
    st.next_ids = torch.zeros(R, **i64)
    st.out_tokens = torch.zeros(R, max_out, **i32)
    st.lp_n = torch.full((R,), -1, **i32)
    st.lp_ring_lp = torch.zeros(R, lp_ring, **f32)
    st.lp_ring_ids = torch.zeros(R, lp_ring, lp_width, **i32)
    st.lp_ring_top = torch.zeros(R, lp_ring, lp_width, **f32)
    st.rep_penalty = torch.ones(R, **f32)
    st.min_p = torch.zeros(R, **f32)
    st.min_new = torch.zeros(R, **i32)
    st.presence = torch.zeros(R, ops.presence_words(vocab), **i32)
    if stops:
        st.stop_bytes = torch.zeros(R, ops.STOP_MAX_STRINGS, ops.STOP_MAX_BYTES, dtype=torch.uint8, device=device)
        st.stop_lens = torch.zeros(R, ops.STOP_MAX_STRINGS, **i32)
        st.stop_lookback = torch.zeros(R, **i32)
        st.stop_ids = torch.zeros(R, ops.STOP_MAX_IDS, **i64)
        st.n_stop_ids = torch.zeros(R, **i32)
        st.stop_tail = torch.zeros(R, ops.STOP_MAX_TOKENS, **i64)
        st.stop_tail_len = torch.zeros(R, **i32)


def start_rows(st, rows, sampling, max_new: int, logprobs: Optional[int] = None, processors: Optional[tuple] = None):
    """Start the token streams of rows (an index or a slice of st's rows): sampling (temperature, top_k, top_p, seed), the
    budget max_new, logprobs (None or the top-n) and processors (None or (repetition_penalty, min_p, min_new_tokens)); no token
    out, RNG offset 0, not finished.  The noise row, the output row and the stops are the caller's."""
    t, k, p, seed = sampling
    st.temperature[rows] = t
    st.top_k[rows] = k
    st.top_p[rows] = p
    st.seed[rows] = seed - 2 ** 64 if seed >= 2 ** 63 else seed    # int64 storage of the uint64 seed
    st.rng_offset[rows] = 0
    st.max_new[rows] = max_new
    st.n_out[rows] = 0
    st.finished[rows] = 0
    st.lp_n[rows] = -1 if logprobs is None else logprobs
    pen, min_p, min_new = (1.0, 0.0, 0) if processors is None else processors
    st.rep_penalty[rows] = pen
    st.min_p[rows] = min_p
    st.min_new[rows] = min_new


def sample_and_advance(st, logits, eos, pad: int, stop_vocab=None, logprobs: bool = False, processors: bool = False,
                       stops: bool = False, sampling: Optional[tuple] = None) -> None:
    """The tail of a decode step on the per-row token state st (add_token_fields), logits [R, V] -> next token of every row:
    sample (with processors, through each row's logits processors; row r draws the Philox noise of row noise_row[r] at offset
    rng_offset[r]; sampling: (temperature, top_k, top_p, seed) when every row has these, which the sampler then takes as
    launch arguments instead of loading the row's own, the same token either way), then with logprobs the logprobs of the rows with lp_n >= 0 into ring entry n_out mod lp_ring (finished rows
    untouched), then advance (ops.decode_advance_slots: an unfinished row records its token, finishes on an EOS id or its
    budget, and moves on; a finished row keeps its positions and is fed pad); with processors, each row's new input id then
    joins its presence bitmap; with stops, each row's stop ids and strings are checked against its new token (stop_vocab: the
    device vocabulary table, stopping.StopVocab.device).  eos: the EOS ids (at most 8); pad: what a finished row is fed."""
    if processors:
        ops.sample_tokens_processed(logits, st.temperature, st.top_k, st.top_p, st.min_p, st.seed, st.rep_penalty, st.min_new,
                                    st.presence, st.rng_offset, st.n_out, eos, noise_rows=st.noise_row, out=st.next_ids)
    elif sampling is not None:
        ops.sample_tokens_rows(logits, *sampling, st.noise_row, st.rng_offset, out=st.next_ids)
    else:
        ops.sample_tokens_slots(logits, st.temperature, st.top_k, st.top_p, st.seed, st.noise_row, st.rng_offset,
                                out=st.next_ids)
    if logprobs:
        ops.token_logprobs(logits, st.next_ids, st.lp_ring_ids.shape[-1], n_row=st.lp_n, col=st.n_out,
                           ring=st.lp_ring_lp.shape[1], finished=st.finished, finished_fill=False,
                           out=(st.lp_ring_lp, st.lp_ring_ids, st.lp_ring_top))
    ops.decode_advance_slots(st.next_ids, st.ids_in, st.out_tokens, st.n_out, st.max_new, st.rope_pos, st.write_pos, st.kv_len,
                             st.rng_offset, st.finished, eos, pad)
    if processors:
        ops.presence_set(st.ids_in, st.presence, logits.shape[-1])
    if stops:
        ops.stop_check_slots(*stop_vocab, st.stop_bytes, st.stop_lens, st.stop_lookback, st.stop_ids, st.n_stop_ids,
                             st.stop_tail, st.stop_tail_len, st.out_tokens, st.n_out, st.finished, st.ids_in, pad)


class SlotDecodeState(DecodeState):
    """DecodeState of continuous batching: one row per engine slot, max_batch rows, each with the token fields of
    add_token_fields (logprob rings of lp_ring entries, 20 wide; presence bitmaps over vocab ids; stops).  A decode step over
    the first n slots reads rows(n); the other slots are idle."""

    def __init__(self, max_batch, H, max_out, device, lp_ring: int = 1, vocab: int = 1):
        super().__init__(max_batch, H, 0, device)
        self.key_mask = None
        add_token_fields(self, max_batch, max_out, device, lp_ring, vocab=vocab)

    # the per-slot arrays, in the order a slot's row is copied when slots are compacted
    SLOT_FIELDS = ("rope_pos", "write_pos", "kv_len", "temperature", "top_k", "top_p", "seed", "noise_row", "rng_offset",
                   "max_new", "n_out", "finished", "ids_in", "next_ids", "out_tokens", "lp_n", "lp_ring_lp", "lp_ring_ids",
                   "lp_ring_top", "rep_penalty", "min_p", "min_new", "presence", "stop_bytes", "stop_lens", "stop_lookback",
                   "stop_ids", "n_stop_ids", "stop_tail", "stop_tail_len")

    def rows(self, n):
        """A DecodeState view of the first n slots (what decode_step and the sampler of a step over n slots read)."""
        v = object.__new__(SlotDecodeState)
        for f in self.SLOT_FIELDS:
            setattr(v, f, getattr(self, f)[:n])
        v.qkv = self.qkv[:, :n]
        v.key_mask = None
        return v


class AriaAttention(nn.Module):
    """What `LLAMA_ATTENTION_CLASSES[config._attn_implementation]` provides at moe_lm.py:594: MHA, no bias,
    rotate-half RoPE, causal, KV cache.  q/k/v projections + RoPE + cache write are ONE GEMM launch."""

    def __init__(self, config, layer_idx, device=None):
        super().__init__()
        self.config = config
        self.layer_idx = layer_idx
        d = config.hidden_size
        self.num_heads = config.num_attention_heads
        self.head_dim = d // self.num_heads
        if self.head_dim != 128:
            raise RuntimeError("AriaAttention kernels are written for head_dim 128")
        self.q_proj = Linear(d, d, device=device)
        self.k_proj = Linear(d, d, device=device)
        self.v_proj = Linear(d, d, device=device)
        self.o_proj = Linear(d, d, device=device)

    def is_fp8(self) -> bool:
        """Whether q / k / v / o are W8A8 (Fp8Linear, AriaForConditionalGeneration.quantize_dense_fp8)."""
        return _all_fp8((self.q_proj, self.k_proj, self.v_proj, self.o_proj), "AriaAttention")

    def _qkv(self, hidden_states, hq, outs, rows_per_batch, pos0, rope, position_ids):
        """The fused q/k/v launch.  fp8: hq = (e4m3 rows, row scales) of hidden_states when the caller has them
        (rmsnorm_quantize_fp8), else they are quantized here."""
        cos, sin = rope
        if self.is_fp8():
            xq, xs = hq if hq is not None else self.q_proj.quantize_input(hidden_states)
            ws = [self.q_proj, self.k_proj, self.v_proj]
            ops.qkv_heads_w8a8(xq, xs, [m.weight for m in ws], [m.weight_scale for m in ws], outs, self.head_dim, rows_per_batch,
                               pos0=pos0, rope_mask=0b011, rope_cos=cos, rope_sin=sin, position_ids=position_ids)
            return
        ops.qkv_heads(hidden_states, [self.q_proj.weight, self.k_proj.weight, self.v_proj.weight], [None] * 3, outs,
                      self.head_dim, rows_per_batch, pos0=pos0, rope_mask=0b011, rope_cos=cos, rope_sin=sin,
                      position_ids=position_ids)

    def _o_proj(self, o, residual):
        if type(self.o_proj) is Fp8Linear:
            return self.o_proj(o, residual=residual)
        return ops.linear(o, self.o_proj.weight, residual=residual)

    def forward(self, hidden_states, cache: KVCache, rope, residual=None, key_mask=None, position_ids=None, hq=None):
        """key_mask [B, pos0+T] uint8, 1 = key masked out (padded batch); position_ids [B*T] int32 RoPE positions
        (default: cache position pos0 + t, what LlamaModel uses when none are given).  With fp8 projections, hidden_states
        may be the e4m3 rows [B, T, d] with hq = (the same rows, their scales [B*T]) (MoEDecoderLayer: rmsnorm_quantize_fp8)."""
        B, T, d = hidden_states.shape
        H, hd = self.num_heads, self.head_dim
        pos0 = cache.seq_len
        if pos0 + T > cache.T_max:
            # the fused epilogue stores k/v rows at pos0 + t and reads the RoPE table there: never past the cache
            raise RuntimeError(f"KV cache overflow: {pos0} cached + {T} new tokens > T_max = {cache.T_max}")
        kc, vc = cache.k[self.layer_idx], cache.v[self.layer_idx]
        q = cache.q  # staging buffer with the cache's strides: the fused epilogue scatters q, k, v with one stride pair
        cos, sin = rope
        fp8 = cache.dtype == "fp8"
        k_out, v_out = (cache.k_stage, cache.v_stage) if fp8 else (kc, vc)
        self._qkv(hidden_states, hq, [q, k_out, v_out], T, pos0, rope, position_ids)
        Tk = pos0 + T
        scale = hd ** -0.5
        if fp8:
            # fp8 cache: a single token is quantized into the cache and attends to it (as decode_step does); a multi-token
            # step attends in bf16 to the staging pair, holding the dequantized cached rows and its own rows, which are
            # quantized into the cache afterwards.  A one-chunk prefill thus gives the bf16 cache's logits bit for bit.
            ks, vs = cache.scales(self.layer_idx)
            k_st, v_st = cache.k_stage, cache.v_stage
            if T == 1:
                ops.kv_store_fp8(k_st[:, :, pos0:Tk], v_st[:, :, pos0:Tk], kc, vc, ks, vs, pos0)
                o = ops.attention_decode(q[:, :, pos0, :], kc, vc, Tk, scale, key_mask=key_mask, k_scale=ks, v_scale=vs).view(B, 1, d)
            else:
                if pos0 > 0:
                    ops.kv_load_fp8(kc, vc, ks, vs, k_st, v_st, pos0)
                o = ops.attention(q[:, :, pos0:], k_st, v_st, T, Tk, scale, causal=True, key_mask=key_mask)
                ops.kv_store_fp8(k_st[:, :, pos0:Tk], v_st[:, :, pos0:Tk], kc, vc, ks, vs, pos0)
            return self._o_proj(o, residual)
        if T == 1:
            o = ops.attention_decode(q[:, :, pos0, :], kc, vc, Tk, scale, key_mask=key_mask).view(B, 1, d)  # strided view, no copy
        else:  # prefill, or a multi-token continuation (chunked prefill): the queries are the last T of Tk positions
            o = ops.attention(q[:, :, pos0:], kc, vc, T, Tk, scale, causal=True, key_mask=key_mask)
        return self._o_proj(o, residual)

    def decode_step(self, hidden_states, cache: KVCache, rope, state: DecodeState, residual=None, hq=None):
        """One token per row with every position on the device (graph-replayable): the fused projection writes q, k, v
        to the state's staging rows (RoPE at state.rope_pos), and the cache's decode_attention stores k, v at state.write_pos
        and attends over state.kv_len keys.  Same kernels and arithmetic as forward() at T = 1."""
        B, T, d = hidden_states.shape
        q, k, v = state.qkv[0], state.qkv[1], state.qkv[2]
        self._qkv(hidden_states, hq, [q, k, v], 1, 0, rope, state.rope_pos)
        o = cache.decode_attention(self.layer_idx, q[:, :, 0], k[:, :, 0], v[:, :, 0], state, self.head_dim ** -0.5)
        return self._o_proj(o.view(B, 1, d), residual)

    def verify_step(self, hidden_states, cache: KVCache, rope, state: LookupDecodeState, residual=None, hq=None):
        """decode_step for Q tokens per row (a prompt-lookup verify step): hidden_states [B, Q, d]; the fused projection writes
        q, k, v to state.qkv_k (RoPE at state.pos_k), kv_append_rows moves k, v to cache rows write_pos[b] + i, and query i
        attends to state.lens_k[b*Q + i] keys.  Each query gets the arithmetic decode_step gives that token.  bf16 cache."""
        B, Q, d = hidden_states.shape
        kc, vc = cache.k[self.layer_idx], cache.v[self.layer_idx]
        q, k, v = state.qkv_k[0], state.qkv_k[1], state.qkv_k[2]
        self._qkv(hidden_states, hq, [q, k, v], Q, 0, rope, state.pos_k)
        ops.kv_append_rows(k, v, kc, vc, state.write_pos)
        o = ops.attention_decode_multi(q, kc, vc, state.lens_k, self.head_dim ** -0.5, key_mask=state.key_mask)
        return self._o_proj(o, residual)

    def prefill_suffixes(self, hidden_states, cache: SharedPrefixCache, rope, cu_seqlens, position_ids, residual=None, hq=None):
        """Suffixes packed as one [1, S_tot] sequence (AriaMoELMModel.prefill_suffixes) against the prefix held in the cache's
        rows [0, cache.seq_len): the fused projection writes q, k, v to a staging buffer (RoPE at position_ids), the suffixes
        attend to the prefix and to themselves (ops.attention_prefill_shared_prefix), and their k, v rows are copied into the
        tails of each suffix's rows (ops.kv_scatter_tails)."""
        _, S, d = hidden_states.shape
        H, hd = self.num_heads, self.head_dim
        stage = torch.empty(3, 1, H, S, hd, dtype=bf16, device=hidden_states.device)
        q, k, v = stage[0], stage[1], stage[2]
        self._qkv(hidden_states, hq, [q, k, v], S, 0, rope, position_ids)
        o = ops.attention_prefill_shared_prefix(q, k, v, S, cache.k[self.layer_idx], cache.v[self.layer_idx], cache.seq_len,
                                                cu_seqlens, hd ** -0.5)
        n = cache.group_size // (cu_seqlens.numel() - 1)    # rows per suffix
        ops.kv_scatter_tails(k, v, S, cache.tail_k[self.layer_idx], cache.tail_v[self.layer_idx], cu_seqlens, n)
        return self._o_proj(o.view(1, S, d), residual)

    def prefill_paged(self, hidden_states, cache: PagedKVCache, rope, page_table, seg, position_ids, residual=None, hq=None,
                      prefix=None):
        """Packed prompt segments, each after a prefix held in its own pages (AriaMoELMModel.prefill_paged): the fused projection
        writes q, k, v to a staging buffer (RoPE at position_ids), segment b attends to the pages page_table[b, : P_b / 256] and
        causally to itself (ops.attention_prefill_paged_varlen), and its k, v rows are stored after its prefix in its pages
        (ops.kv_pages_store_varlen).
        fp8 pages: every query attends to every key as bf16(code * scale), its own segment's included, so a result does not
        depend on where a prompt was split or which pages were cached.  The rows are stored first, which rewrites the staging
        rows with their dequantized values.  prefix = (pages, table, k_scratch, v_scratch) of AriaMoELMModel.prefill_paged:
        the launch's distinct prefix pages (pages: CUDA int32, or None when no segment has a prefix) are dequantized into the
        bf16 scratch pools (ops.kv_pages_load_fp8), and `table`, the page table renumbered to the scratch, is what attention
        reads in page_table's place."""
        _, S, d = hidden_states.shape
        H, hd = self.num_heads, self.head_dim
        stage = torch.empty(3, 1, H, S, hd, dtype=bf16, device=hidden_states.device)
        q, k, v = stage[0], stage[1], stage[2]
        self._qkv(hidden_states, hq, [q, k, v], S, 0, rope, position_ids)
        kp, vp = cache.k[self.layer_idx], cache.v[self.layer_idx]
        if cache.dtype == "fp8":
            ks, vs = cache.scales(self.layer_idx)
            pages, table, k_scr, v_scr = prefix
            ops.kv_pages_store_varlen(k, v, kp, vp, page_table, seg, k_scale=ks, v_scale=vs)
            if pages is not None:
                ops.kv_pages_load_fp8(kp, vp, ks, vs, pages, k_scr, v_scr)
            o = ops.attention_prefill_paged_varlen(q, k, v, k_scr, v_scr, table, seg, hd ** -0.5)
            return self._o_proj(o.view(1, S, d), residual)
        o = ops.attention_prefill_paged_varlen(q, k, v, kp, vp, page_table, seg, hd ** -0.5)
        ops.kv_pages_store_varlen(k, v, kp, vp, page_table, seg)
        return self._o_proj(o.view(1, S, d), residual)


class MoEDecoderLayer(nn.Module):
    """moe_lm.py:580-602: x + attn(rms(x)); h + moe(rms(h)).  The MoE residual add is deferred into the next
    RMSNorm kernel (same bf16 rounding as the reference's separate add)."""

    def __init__(self, config, layer_idx, device=None):
        super().__init__()
        self.hidden_size = config.hidden_size
        self.self_attn = AriaAttention(config, layer_idx, device)
        self.mlp = MoELayer(config, device)
        self.input_layernorm = RMSNorm(config.hidden_size, config.rms_norm_eps, device)
        self.post_attention_layernorm = RMSNorm(config.hidden_size, config.rms_norm_eps, device)

    def _attn_input(self, x, pending):
        """input_layernorm (+ the pending MoE output) -> (h, hq, residual stream).  fp8 attention: h is the e4m3 rows and hq
        (rows, scales), quantized in the norm's kernel, so no bf16 h is written; else hq is None."""
        norm = self.input_layernorm
        if self.self_attn.is_fp8():
            _reject_fp8_grad(x)
            if pending is None:
                hq = ops.rmsnorm_quantize_fp8(x, norm.weight, norm.variance_epsilon)
            else:
                *hq, x = ops.rmsnorm_quantize_fp8(x, norm.weight, norm.variance_epsilon, pending)
            return hq[0], (hq[0].view(-1, hq[0].shape[-1]), hq[1]), x
        if pending is None:
            return norm(x), None, x
        h, x = norm(x, residual=pending)
        return h, None, x

    def forward(self, x, pending, attend):
        """x: residual stream; pending: MoE output of the previous layer not yet added (or None); attend(self_attn, h, hq,
        residual): the step's attention, one of AriaAttention's forward, decode_step, verify_step, prefill_suffixes or
        prefill_paged, returning the residual stream after it."""
        h, hq, x = self._attn_input(x, pending)
        x = attend(self.self_attn, h, hq, x)
        h = self.post_attention_layernorm(x)
        return x, self.mlp(h)


class AriaMoELMModel(nn.Module):
    """moe_lm.py:605-636."""

    def __init__(self, config, device=None):
        super().__init__()
        self.config = config
        self.embed_tokens = nn.Embedding(config.vocab_size, config.hidden_size, device=device, dtype=bf16)
        self.embed_tokens.weight.requires_grad_(False)
        self.layers = nn.ModuleList([MoEDecoderLayer(config, i, device) for i in range(config.num_hidden_layers)])
        self.norm = RMSNorm(config.hidden_size, config.rms_norm_eps, device)
        self._rope = None

    def rope_tables(self, n_pos, device):
        if self._rope is None or self._rope[0].shape[0] < n_pos or self._rope[0].device != device:
            hd = self.config.head_dim
            # LlamaRotaryEmbedding: inv_freq in fp32 exactly as transformers computes it (moe_lm.py:632)
            inv_freq = 1.0 / (self.config.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.int64).float() / hd))
            self._rope = ops.rope_table(inv_freq.to(device), n_pos)
        return self._rope

    def forward(self, inputs_embeds, cache: KVCache, key_mask=None, position_ids=None):
        B, T, _ = inputs_embeds.shape
        if cache.seq_len + T > cache.T_max:
            raise RuntimeError(f"KV cache overflow: {cache.seq_len} cached + {T} new tokens > T_max = {cache.T_max}")
        rope = self.rope_tables(cache.n_positions, inputs_embeds.device)
        x, pending = self._run_layers(inputs_embeds, lambda a, h, hq, x: a(h, cache, rope, residual=x, key_mask=key_mask,
                                                                           position_ids=position_ids, hq=hq))
        cache.seq_len += T
        return x, pending  # final residual add happens inside the final norm

    def _run_layers(self, x, attend):
        """Every layer on the residual stream x, each attending through attend (MoEDecoderLayer.forward) -> (x, pending)."""
        pending = None
        for layer in self.layers:
            x, pending = layer(x, pending, attend)
        return x, pending

    def decode_step(self, inputs_embeds, cache: KVCache, state: DecodeState, rope):
        """One token per row through every layer with the positions of `state`; `cache.seq_len` is neither read nor
        written (the caller owns it).  `rope`: the tables of rope_tables(cache.n_positions), computed outside any graph
        capture.  cache: a KVCache, SharedPrefixCache or PagedKVCache (its decode_attention)."""
        return self._run_layers(inputs_embeds, lambda a, h, hq, x: a.decode_step(h, cache, rope, state, residual=x, hq=hq))

    def verify_step(self, inputs_embeds, cache: KVCache, state: LookupDecodeState, rope):
        """decode_step for Q tokens per row, inputs_embeds [B, Q, d], positions from `state` (AriaAttention.verify_step)."""
        return self._run_layers(inputs_embeds, lambda a, h, hq, x: a.verify_step(h, cache, rope, state, residual=x, hq=hq))

    def prefill_suffixes(self, inputs_embeds, cache: SharedPrefixCache, cu_seqlens, position_ids):
        """Prefill B suffixes that continue the one prefix already in `cache` (a SharedPrefixCache of one prompt row whose
        forward() prefill left cache.seq_len = P).  inputs_embeds [1, S_tot, d]: the suffixes packed, suffix b at rows
        [cu_seqlens[b], cu_seqlens[b+1]) (CUDA int32 [B+1]); position_ids CUDA int32 [S_tot], their RoPE positions.  Each
        suffix attends to the prefix and to its own earlier rows; its k, v rows land in rows [0, S_b) of the tails
        b*n .. b*n + n-1 (the cache's one group of B*n rows: n = cache.group_size / B).  The MoE layers see the packed rows as one
        [1, S_tot] batch.  cache.seq_len is neither read past P nor changed.  Returns (x, pending) as forward() does."""
        if not isinstance(cache, SharedPrefixCache) or cache.k[0].shape[0] != 1:
            raise ValueError("prefill_suffixes needs a SharedPrefixCache holding one prefix row")
        if cache.group_size % (cu_seqlens.numel() - 1):
            raise ValueError(f"prefill_suffixes: {cu_seqlens.numel() - 1} suffixes do not divide the cache's {cache.group_size} rows")
        if inputs_embeds.dim() != 3 or inputs_embeds.shape[0] != 1:
            raise ValueError(f"prefill_suffixes: inputs_embeds must be [1, S_tot, d], got {tuple(inputs_embeds.shape)}")
        if cache.seq_len < 1:
            raise ValueError("prefill_suffixes: the cache holds no prefix (seq_len 0)")
        rope = self.rope_tables(cache.n_positions, inputs_embeds.device)
        return self._run_layers(inputs_embeds, lambda a, h, hq, x: a.prefill_suffixes(h, cache, rope, cu_seqlens, position_ids,
                                                                                      residual=x, hq=hq))

    def prefill_paged(self, inputs_embeds, cache: PagedKVCache, page_table, seg, position_ids, page_table_host=None):
        """Prefill prompt segments packed along one row, each continuing a prefix whose keys and values are already in the
        pages of its request (batched and chunked admission, prefix caching: serving.Engine).  inputs_embeds [1, S_tot, d]; seg:
        an ops.PackedSegments, segment b = packed rows [seg.cu[b], seg.cu[b + 1]) after a prefix of seg.prefix_lens[b] tokens (a
        multiple of 256; 0 = no prefix); page_table: CUDA int32 [n_seg, width], row b the pages of segment b's request (its first
        P_b / 256 hold the prefix); position_ids CUDA int32 [S_tot], the RoPE positions P_b .. P_b + len_b - 1 of each segment.
        Each segment attends to its prefix and causally to itself, and its keys and values go to its pages after the prefix, as
        forward() on its whole prompt would have stored them.  Every row's output is the one forward() gives that position on
        its own prompt, bit for bit: attention keeps the segments apart and the rest of a layer computes each row on its own.
        n_seg = 1 is one request's prefill.  Returns (x, pending) as forward() does.
        fp8 pages (AriaAttention.prefill_paged): one bf16 scratch pair holding the launch's distinct prefix pages is allocated
        here and shared by the layers, each layer dequantizing its own pages into it; page_table_host, a CPU copy of
        page_table, spares reading the prefix pages back from the device."""
        if not isinstance(cache, PagedKVCache):
            raise ValueError("prefill_paged needs a PagedKVCache")
        if not isinstance(seg, ops.PackedSegments):
            raise ValueError("prefill_paged: seg must be an ops.PackedSegments")
        if inputs_embeds.dim() != 3 or inputs_embeds.shape[0] != 1 or inputs_embeds.shape[1] != seg.S_tot:
            raise ValueError(f"prefill_paged: inputs_embeds must be [1, {seg.S_tot}, d], got {tuple(inputs_embeds.shape)}")
        if position_ids.shape != (seg.S_tot,):
            raise ValueError(f"prefill_paged: position_ids must be [{seg.S_tot}], got {tuple(position_ids.shape)}")
        width = page_table.shape[-1]
        for b, P in enumerate(seg.prefix_lens):
            if P + seg.cu[b + 1] - seg.cu[b] > width * cache.PAGE_SIZE:
                raise ValueError(f"prefill_paged: segment {b} (P = {P}, {seg.cu[b + 1] - seg.cu[b]} tokens) does not fit {width} "
                                 "pages")
        rope = self.rope_tables(cache.n_positions, inputs_embeds.device)
        prefix = self._prefix_scratch(cache, page_table, seg, page_table_host) if cache.dtype == "fp8" else None
        return self._run_layers(inputs_embeds, lambda a, h, hq, x: a.prefill_paged(h, cache, rope, page_table, seg, position_ids,
                                                                                   residual=x, hq=hq, prefix=prefix))

    @staticmethod
    def _prefix_scratch(cache: PagedKVCache, page_table, seg, page_table_host=None):
        """(pages, table, k_scratch, v_scratch) for an fp8 prefill_paged: the distinct prefix pages of the launch in order of
        first use (CUDA int32, None without a prefix), the page table renumbered to them ([n_seg, max prefix pages]) and the
        bf16 scratch pools [max(1, n), H, 256, 128] they are dequantized into."""
        host = page_table.cpu() if page_table_host is None else page_table_host
        index, table = {}, []
        for b, P in enumerate(seg.prefix_lens):
            table.append([index.setdefault(int(host[b, i]), len(index)) for i in range(P // cache.PAGE_SIZE)])
        width = max(1, max(len(r) for r in table))
        renum = torch.zeros(len(table), width, dtype=torch.int32)
        for b, r in enumerate(table):
            renum[b, :len(r)] = torch.tensor(r, dtype=torch.int32)
        dev = torch.cat([torch.tensor(list(index), dtype=torch.int32), renum.flatten()]).pin_memory().to(page_table.device,
                                                                                                         non_blocking=True)
        n = len(index)
        _, H, rows, hd = cache.k[0].shape
        scratch = torch.empty(2, max(1, n), H, rows, hd, dtype=bf16, device=page_table.device)
        return (dev[:n] if n else None), dev[n:].view(len(table), width), scratch[0], scratch[1]


class AriaMoELMForCausalLM(nn.Module):
    """moe_lm.py:639-679."""

    def __init__(self, config, device=None):
        super().__init__()
        self.config = config
        self.model = AriaMoELMModel(config, device)
        self.vocab_size = config.vocab_size
        self.lm_head = Linear(config.hidden_size, config.vocab_size, device=device)

    def new_cache(self, B, T_max, device, kv_cache_dtype="bf16"):
        """A KVCache for B rows of T_max tokens; kv_cache_dtype "fp8" stores K/V as e4m3 with per-token scales (CUDA only)."""
        if kv_cache_dtype not in KV_CACHE_DTYPES:
            raise ValueError(f"kv_cache_dtype must be 'bf16' or 'fp8', got {kv_cache_dtype!r}")
        if kv_cache_dtype == "fp8" and torch.device(device).type != "cuda":
            raise NotImplementedError("aria_b200: the fp8 KV cache runs on the GPU only")
        c = self.config
        return KVCache(c.num_hidden_layers, B, c.num_attention_heads, T_max, c.head_dim, device, kv_cache_dtype)

    # moe_lm.py:663-679: the routers read the coefficients from the shared config object (used by moe_train's router losses)
    def set_z_loss_coeff(self, z_loss_coeff: float):
        self.config.moe_z_loss_coeff = z_loss_coeff

    def set_aux_loss_coeff(self, aux_loss_coeff: float):
        self.config.moe_aux_loss_coeff = aux_loss_coeff

    def get_input_embeddings(self):
        return self.model.embed_tokens

    def set_input_embeddings(self, value):
        self.model.embed_tokens = value

    def get_output_embeddings(self):
        return self.lm_head

    def set_output_embeddings(self, value):
        self.lm_head = value

    def forward(self, inputs_embeds, cache: Optional[KVCache] = None, num_logits_to_keep: int = 0, key_mask=None,
                position_ids=None):
        B, T, _ = inputs_embeds.shape
        if cache is None:
            cache = self.new_cache(B, T, inputs_embeds.device)
        x, pending = self.model(inputs_embeds, cache, key_mask, position_ids)
        if num_logits_to_keep:
            x = x[:, -num_logits_to_keep:, :].contiguous()
            pending = pending[:, -num_logits_to_keep:, :].contiguous()
        return self.head(x, pending), cache

    def head(self, x, pending):
        """Logits of the layers' output (x, pending): the final norm, which adds the last layer's pending MoE output, then
        lm_head."""
        h, _ = self.model.norm(x, residual=pending)
        return self.lm_head(h)

    def prefill_paged(self, inputs_embeds, cache: PagedKVCache, page_table, seg, position_ids, ends=None, page_table_host=None,
                      hidden_rows=None):
        """AriaMoELMModel.prefill_paged, then the final norm and lm_head on the last row of each segment listed in `ends`
        (segment indices in increasing order, the segments that end a prompt; None = every segment) -> logits [1, len(ends), V],
        row i those of forward(num_logits_to_keep=1) on the whole prompt of segment ends[i].
        hidden_rows (host ints, packed row indices): also the final-norm hidden states of those rows -> (logits, h [n, d]), row
        i what forward() feeds lm_head at that position (prompt logprobs: serving.Engine)."""
        x, pending = self.model.prefill_paged(inputs_embeds, cache, page_table, seg, position_ids, page_table_host)
        if hidden_rows is None:
            return self._end_logits(x, pending, seg, ends)
        if len(hidden_rows):
            idx = torch.tensor(hidden_rows, dtype=torch.int64).to(x.device, non_blocking=True)
            h, _ = self.model.norm(x.index_select(1, idx)[0], residual=pending.index_select(1, idx)[0])
        else:
            h = x.new_empty((0, x.shape[-1]))
        return self._end_logits(x, pending, seg, ends), h

    def _end_logits(self, x, pending, seg, ends):
        ends = range(seg.n_seg) if ends is None else ends
        rows = [seg.cu[b + 1] - 1 for b in ends]
        if not rows:                                         # only chunks that end no prompt: no logits
            return x.new_empty((1, 0, self.vocab_size))
        if rows == list(range(seg.S_tot - len(rows), seg.S_tot)):
            x, pending = x[:, -len(rows):, :].contiguous(), pending[:, -len(rows):, :].contiguous()
        else:
            idx = torch.tensor(rows, dtype=torch.int64).to(x.device, non_blocking=True)
            x, pending = x.index_select(1, idx), pending.index_select(1, idx)
        return self.head(x, pending)

    def decode_step(self, inputs_embeds, cache: KVCache, state: DecodeState, rope):
        """inputs_embeds [B, 1, d] -> logits [B, 1, V] for one decode step driven by device positions (graph-replayable)."""
        return self.head(*self.model.decode_step(inputs_embeds, cache, state, rope))

    def verify_step(self, inputs_embeds, cache: KVCache, state: LookupDecodeState, rope):
        """inputs_embeds [B, Q, d] -> logits [B, Q, V]: decode_step for the Q tokens of a prompt-lookup verify step, each row's
        query i with the logits decode_step gives its token (graph-replayable)."""
        return self.head(*self.model.verify_step(inputs_embeds, cache, state, rope))
