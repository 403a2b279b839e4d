"""LoRA on the grouped expert GEMMs (SURVEY §8f-3) — mirror of the reference's `GroupedGemmLoraLayer`
(aria/lora/layers.py:30-152, mapped onto every `GroupedGEMM` by peft at aria/train.py:107):

    result = base_layer(x, tokens_per_expert) + lora_B(lora_A(x, tpe), tpe) * (lora_alpha / r)          (layers.py:132-140)

with `lora_A = GroupedGEMM(in, r, groups)` and `lora_B = GroupedGEMM(r, out, groups)` (layers.py:87-92), i.e. parameters
`lora_A.<adapter>.weight [E, in, r]` and `lora_B.<adapter>.weight [E, r, out]` in the reference's layout.

Tensor-core mapping: r (8 in recipes/config_lora.yaml) is far below a tensor-core tile, so both adapters are zero-padded to
R_PAD = 128 columns / rows in a per-step working copy and run through the same wgmma grouped-GEMM kernels as the experts
(padded lanes multiply zeros: exact).  The scaling is folded into the padded A copy (exact for the usual power-of-two
alpha/r; one bf16 rounding otherwise) and the `+ base` is the residual input of the B GEMM's epilogue, so the adapter
costs two extra launches forward.  Backward (adapters and input only; the base weight is frozen as in the recipe):

    dB = (x A s)^T dy      `aria_grouped_wgrad`          dh = dy B^T          `aria_gemm` B_GNK (weight read transposed)
    dA = s * x^T dh        `aria_grouped_wgrad`          dx = dy W^T + dh (A s)^T

Group rows may start at any row (`aria_grouped_wgrad` handles densely packed groups); the training dispatcher's
`row_align=16` blocks take its cheaper aligned path.
Parity: the oracle's restatement is pinned bit-exactly to the unmodified reference layer, loaded under a stand-in for the two
peft symbols it imports (oracle/ref_loader.py `load_reference_lora`, tests/test_oracle_vs_reference.py) and through
tests/golden/lora_grouped_gemm_*.pt on the GPU.
"""
from __future__ import annotations

import torch
from torch import nn

from . import ops
from .moe_lm import Fp8GroupedGEMM, GroupedGEMM, _as_offsets

R_PAD = 128


def _pad_a(a: torch.Tensor, scale: float) -> torch.Tensor:
    """[E, in, r] -> [E, in, R_PAD] * scale (bf16)."""
    E, K, r = a.shape
    out = torch.zeros((E, K, R_PAD), dtype=a.dtype, device=a.device)
    out[:, :, :r] = a * scale if scale != 1.0 else a
    return out


def _pad_b(b: torch.Tensor) -> torch.Tensor:
    """[E, r, out] -> [E, R_PAD, out]."""
    E, r, N = b.shape
    out = torch.zeros((E, R_PAD, N), dtype=b.dtype, device=b.device)
    out[:, :r] = b
    return out


class _LoraGroupedGemm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, a, b, offsets, scale: float):
        a_pad, b_pad = _pad_a(a.detach(), scale), _pad_b(b.detach())
        base = ops.grouped_gemm(x, w, offsets)
        h = ops.grouped_gemm(x, a_pad, offsets)                     # [rows, R_PAD] = x A s
        out = ops.grouped_gemm(h, b_pad, offsets, residual=base)    # base + h B
        ctx.save_for_backward(x, w, a_pad, b_pad, h, offsets)
        ctx.scale, ctx.r = scale, a.shape[2]
        return out

    @staticmethod
    def backward(ctx, dy):
        x, w, a_pad, b_pad, h, offsets = ctx.saved_tensors
        dy = dy.contiguous()
        r = ctx.r
        d_b = ops.grouped_wgrad(h, dy, offsets)[:, :r].contiguous()             # [E, r, out]
        dh = ops.grouped_gemm_nt(dy, b_pad, offsets)                            # dy @ B_pad[e].T -> [rows, R_PAD]
        d_a = ops.grouped_wgrad(x, dh, offsets)[:, :, :r]                       # x^T dh (d/dA of x (A s) is s x^T dh)
        d_a = (d_a * ctx.scale).contiguous() if ctx.scale != 1.0 else d_a.contiguous()
        dx = None
        if ctx.needs_input_grad[0]:
            dx = ops.grouped_gemm_nt(dy, w, offsets)                            # base path: dy @ W[e].T
            dx = ops.grouped_gemm_nt(dh, a_pad, offsets, residual=dx)           # + adapter path: dh @ (A s)[e].T
        return dx, None, d_a, d_b, None, None


class _SwiGLU(torch.autograd.Function):
    """glu of moe_lm.py:505-507 as a differentiable op over `aria_swiglu_fwd` / `aria_swiglu_bwd`."""

    @staticmethod
    def forward(ctx, h1):
        ctx.save_for_backward(h1)
        return ops.swiglu_fwd(h1)

    @staticmethod
    def backward(ctx, dh):
        (h1,) = ctx.saved_tensors
        return ops.swiglu_bwd(h1, dh.contiguous())


def swiglu(h1: torch.Tensor) -> torch.Tensor:
    return _SwiGLU.apply(h1) if (torch.is_grad_enabled() and h1.requires_grad) else ops.swiglu_fwd(h1)


def get_lora_target_modules(model_named_modules, lora_target_modules, freeze_vit=False, freeze_projector=False,
                            freeze_llm=False, freeze_llm_layers=None):
    """Same selection rule as the reference's `get_lora_target_modules` (aria/lora/utils.py:29-64): a module is a target when
    its qualified name contains one of `lora_target_modules`, unless it lives in a frozen tower or a frozen LM layer."""
    out = []
    for key in model_named_modules:
        if freeze_vit and "vision_tower" in key:
            continue
        if freeze_projector and "multi_modal_projector" in key:
            continue
        if freeze_llm and "language_model" in key:
            continue
        if any(f"language_model.model.layers.{i}." in key for i in (freeze_llm_layers or ())):
            continue
        if any(t in key for t in lora_target_modules):
            out.append(key)
    return out


def inject_lora(model: nn.Module, target_modules, r: int = 8, lora_alpha: int = 32, adapter_name: str = "default") -> list:
    """Wrap every `GroupedGEMM` whose qualified name is in `target_modules` (e.g. from `get_lora_target_modules`) with a
    `GroupedGemmLoraLayer`, in place — the `{GroupedGEMM: GroupedGemmLoraLayer}` custom-module mapping of aria/train.py:107.
    Returns the names wrapped.  Other module types in the list are left alone (their LoRA is peft's stock Linear path)."""
    wanted, done = set(target_modules), []
    for name, mod in list(model.named_modules()):
        if name in wanted and type(mod) is Fp8GroupedGEMM:
            raise NotImplementedError(f"LoRA on fp8 expert weights ({name}) is not supported: inject the adapters into the "
                                      "bf16 model")
        if name in wanted and type(mod) is GroupedGEMM:
            parent = model.get_submodule(name.rsplit(".", 1)[0]) if "." in name else model
            setattr(parent, name.rsplit(".", 1)[-1], GroupedGemmLoraLayer(mod, adapter_name, r=r, lora_alpha=lora_alpha))
            done.append(name)
    return done


class GroupedGemmLoraLayer(nn.Module):
    """Same attribute names as the reference layer (`base_layer`, `lora_A`, `lora_B`, `scaling`, `r`, `lora_alpha`), one
    adapter per name; dropout is the identity (lora_dropout 0 in the recipe; a non-zero value is rejected)."""

    def __init__(self, base_layer: GroupedGEMM, adapter_name: str = "default", r: int = 8, lora_alpha: int = 32,
                 lora_dropout: float = 0.0):
        super().__init__()
        if type(base_layer) is Fp8GroupedGEMM:
            raise NotImplementedError("LoRA on fp8 expert weights is not supported: wrap the bf16 GroupedGEMM")
        if r <= 0:
            raise ValueError(f"`r` should be a positive integer value but the value passed is {r}")   # layers.py:74-77
        if r > R_PAD or r % 8:
            raise ValueError(f"r must be a multiple of 8 and <= {R_PAD} on this path, got {r}")
        if lora_dropout:
            raise ValueError("lora_dropout > 0 is not supported on the CUDA path")
        self.base_layer = base_layer
        self.in_features, self.out_features, self.groups = base_layer.in_features, base_layer.out_features, base_layer.groups
        dev = base_layer.weight.device
        self.r = {adapter_name: r}
        self.lora_alpha = {adapter_name: lora_alpha}
        self.scaling = {adapter_name: lora_alpha / r}
        self.lora_A = nn.ModuleDict({adapter_name: GroupedGEMM(self.in_features, r, self.groups, device=dev)})
        self.lora_B = nn.ModuleDict({adapter_name: GroupedGEMM(r, self.out_features, self.groups, device=dev)})
        self.active_adapters = [adapter_name]
        self.disable_adapters = False
        self.merged_adapters = []
        for m in (self.lora_A[adapter_name], self.lora_B[adapter_name]):
            m.weight.requires_grad_(True)
        self.reset_lora_parameters(adapter_name)

    def reset_lora_parameters(self, adapter_name: str):
        """peft's default for linear-like layers: A ~ kaiming-uniform, B = 0 (the adapter starts as a no-op)."""
        a, b = self.lora_A[adapter_name].weight, self.lora_B[adapter_name].weight
        with torch.no_grad():
            bound = (6.0 / ((1 + 5.0) * self.in_features)) ** 0.5
            a.uniform_(-bound, bound)
            b.zero_()

    @property
    def merged(self) -> bool:
        return bool(self.merged_adapters)

    def get_delta_weight(self, adapter: str) -> torch.Tensor:
        """layers.py:193-228: A @ B * scaling, [E, in, out] (a one-off merge-time product, not on the hot path)."""
        return torch.matmul(self.lora_A[adapter].weight, self.lora_B[adapter].weight) * self.scaling[adapter]

    def merge(self, adapter_names=None) -> None:
        """layers.py:154-191: fold the active adapters into the base weight (W += A B s); forward then runs the plain GEMM."""
        for name in (adapter_names or self.active_adapters):
            if name in self.lora_A and name not in self.merged_adapters:
                with torch.no_grad():
                    self.base_layer.weight.data += self.get_delta_weight(name)
                self.merged_adapters.append(name)

    def unmerge(self) -> None:
        while self.merged_adapters:
            name = self.merged_adapters.pop()
            with torch.no_grad():
                self.base_layer.weight.data -= self.get_delta_weight(name)

    def forward(self, x: torch.Tensor, tokens_per_expert: torch.Tensor) -> torch.Tensor:
        off = _as_offsets(tokens_per_expert, self.groups, x.device)
        if self.disable_adapters:
            if self.merged:
                self.unmerge()                                         # layers.py:113-116
            return ops.grouped_gemm(x, self.base_layer.weight, off)
        if self.merged:
            return ops.grouped_gemm(x, self.base_layer.weight, off)    # layers.py:121-122
        result = None
        for name in self.active_adapters:
            if name not in self.lora_A:
                continue
            a, b = self.lora_A[name].weight, self.lora_B[name].weight
            if result is None:
                result = _LoraGroupedGemm.apply(x, self.base_layer.weight, a, b, off, float(self.scaling[name]))
            else:  # the reference loops over active adapters (layers.py:125-140); one adapter per layer is what its recipe uses
                raise NotImplementedError("more than one active adapter per layer")
        if result is None:
            result = ops.grouped_gemm(x, self.base_layer.weight, off)
        return result
