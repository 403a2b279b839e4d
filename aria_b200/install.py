"""Drop-in installer: rebind the hot-path seams of an *instantiated reference model* (`aria.model.*`, importable in a
transformers-4.46.3 environment or through a loader like oracle/ref_loader.py) to the H100-native kernels, sharing its
parameters (no copy, HF layout untouched).

Seams (SURVEY.md §8b):
  1. `aria.model.moe_lm.experts_gemm` (moe_lm.py:431-443)  -> `aria_b200.moe_lm.experts_gemm` (gmm-compatible)
  2. `MoELayer.forward` (moe_lm.py:548-577)                 -> fused router / dispatch / grouped GEMM / combine path
  3. decoder-layer attention (moe_lm.py:594)                -> `AriaAttention`-style forward on the module's own q/k/v/o_proj
  4. `Idefics2EncoderLayer.forward` (vision_encoder.py:120) -> fused ViT layer
  5. `AriaForConditionalGeneration.forward` (modeling_aria.py:287-323, the loss head) -> `loss.linear_cross_entropy` on the
     final-norm hidden states: logits only for labelled rows, in chunks, never the [B, T, V] tensor

(1) and (2) are wired by `install()` — inference-only by default, differentiable with `install(..., trainable=True)`; (3) is `aria_b200.hf_attention.register()` (an implementation key for transformers'
attention interface — the module keeps its projections, RoPE and HF Cache); (4) is `install_vit()` (per-layer forward on the
HF module's own parameters; the embeddings / mask creation around it stay HF's); (5) is `install_loss()` (training forward
with labels only; every other call runs the original forward).
There is no CPU fallback: the patched modules require CUDA bf16 tensors.
"""
from __future__ import annotations

import sys
import types

import torch
from torch import nn

from . import loss as _loss
from . import lora as _lora
from . import moe_lm as _m
from . import moe_train as _t
from . import ops


def _reject_autograd(what: str, module, *tensors):
    """The seams below are the INFERENCE path: their outputs come straight from the C ABI and carry no grad_fn, so under
    autograd they would silently cut the graph (and drop the training-mode router losses, moe_lm.py:257-272).  Refuse
    instead of training with wrong gradients; `install(..., trainable=True)` binds the differentiable MoE seams."""
    if torch.is_grad_enabled() and (module.training or any(t is not None and t.requires_grad for t in tensors)):
        raise RuntimeError(f"aria_b200.install: {what} is inference-only (no autograd through the fused kernels); call it under "
                           "torch.no_grad() with the module in eval() mode (install(..., trainable=True) binds differentiable MoE seams)")


def _moe_forward(self, hidden_states: torch.Tensor) -> torch.Tensor:
    """Replacement for the reference `MoELayer.forward` (moe_lm.py:548-577) — and for transformers' own `AriaTextMoELayer.forward`,
    which has the same sub-modules with `router` an nn.Linear — using the module's own parameters."""
    _reject_autograd("MoELayer.forward", self, hidden_states)
    return _moe_block(self, hidden_states)


def _moe_block(self, hidden_states: torch.Tensor) -> torch.Tensor:
    """The inference MoE block on the module's own (plain) parameters."""
    cfg = getattr(self.router, "config", None) or self.config
    shape = hidden_states.shape
    x = hidden_states.reshape(-1, shape[-1]).contiguous()
    se = self.shared_experts
    if x.is_cuda:
        # one C-ABI call for the whole block (aria_moe_block_fwd, csrc/moe_block.cu); the shared experts run on a side stream
        out = ops.moe_block_fwd(x, self.router.weight, self.experts.fc1.weight, self.experts.fc2.weight, se.gate_proj.weight,
                                se.up_proj.weight, se.down_proj.weight, cfg.moe_topk, side_stream=_m._side_stream(x.device))
        return out.view(shape)
    # kernel-by-kernel sequence (what the block entry launches); reached only by the host-logic tests, which swap `ops` for
    # oracle-backed stand-ins on CPU (tests/standin_ops.py)
    forked = _m.shared_expert_overlapped(
        lambda: ops.linear(ops.linear_swiglu(x, se.gate_proj.weight, se.up_proj.weight), se.down_proj.weight), x)
    scores, idx, counts, _ = ops.router_topk(x, self.router.weight, cfg.moe_topk)
    offsets, dest, src = ops.build_permutation(idx, counts)
    permuted = ops.permute_rows(x, src)
    h = ops.grouped_gemm(permuted, self.experts.fc1.weight, offsets, swiglu=True)
    y = ops.grouped_gemm(h, self.experts.fc2.weight, offsets)
    shared = _m.join_side(forked, x)
    return ops.unpermute_combine(y, dest, scores, shared).view(shape)


# ------------------------------------------------------------------------------------------------ trainable MoE seam
def _plain_weight(mod):
    """Weight of an unwrapped bias-free projection (nn.Linear, or the reference's TopKRouter), else None (e.g. peft-wrapped)."""
    if type(mod) is nn.Linear and mod.bias is None:
        return mod.weight
    if type(mod).__name__ == "TopKRouter" and not hasattr(mod, "base_layer"):
        return mod.weight
    return None


def _lora_parts(fc):
    """For an expert GEMM wrapped like the reference's `GroupedGemmLoraLayer` (aria/lora/layers.py:30-152: `base_layer`,
    `lora_A`, `lora_B`, `scaling`, `active_adapters`): (base weight, A [E, in, r], B [E, r, out], scaling), or
    (base weight, None, None, None) when no adapter is active (disabled or merged).  None for a plain GroupedGEMM."""
    if not all(hasattr(fc, a) for a in ("base_layer", "lora_A", "lora_B", "scaling", "active_adapters")):
        return None
    base = fc.base_layer.weight
    if getattr(fc, "disable_adapters", False) or getattr(fc, "merged", False):
        return base, None, None, None
    active = [a for a in fc.active_adapters if a in fc.lora_A]
    if len(active) > 1:
        raise NotImplementedError(f"aria_b200.install: {len(active)} active LoRA adapters on one expert GEMM; one is supported")
    if not active:
        return base, None, None, None
    name = active[0]
    drop = getattr(fc, "lora_dropout", None)
    if drop is not None and name in drop and float(getattr(drop[name], "p", 0.0)) > 0.0:
        raise NotImplementedError("aria_b200.install: lora_dropout > 0 is not supported on the expert GEMMs")
    if getattr(fc, "use_dora", {}).get(name, False):
        raise NotImplementedError("aria_b200.install: DoRA is not supported on the expert GEMMs")
    a, b = fc.lora_A[name].weight, fc.lora_B[name].weight
    if a.shape[-1] > _lora.R_PAD:
        raise NotImplementedError(f"aria_b200.install: LoRA rank {a.shape[-1]} > {_lora.R_PAD} on the expert GEMMs")
    return base, a, b, float(fc.scaling[name])


def _expert_gemm(fc, a, offsets):
    parts = _lora_parts(fc)
    w = fc.weight if parts is None else parts[0]
    if parts is not None and parts[1] is not None:
        return _lora._LoraGroupedGemm.apply(a, w, parts[1], parts[2], offsets, parts[3])
    return _t.GroupedGemmFunction.apply(a, w, offsets)


def _router_losses(self):
    """(loss_coeffs, scale holder) of the training-mode router losses (moe_lm.py:257-272): the reference `MoELayer` in train()
    mode gets its router config's coefficients and ITS module's `MoEAuxLossAutoScaler` (train.py sets the scale on that class);
    transformers' `AriaTextMoELayer` has no router losses."""
    router = self.router
    cfg = getattr(router, "config", None)
    if not self.training or type(self).__name__ != "MoELayer" or cfg is None or not hasattr(cfg, "moe_z_loss_coeff"):
        return None, None
    holder = getattr(sys.modules.get(type(router).__module__), "MoEAuxLossAutoScaler", None)
    if holder is None:
        raise RuntimeError(f"aria_b200.install: no MoEAuxLossAutoScaler next to {type(router).__module__}.TopKRouter")
    return (float(cfg.moe_z_loss_coeff), float(cfg.moe_aux_loss_coeff)), holder


def _moe_plain(self):
    """True when router, experts and shared experts are all unwrapped: the layer is one MoELayerFunction."""
    se = self.shared_experts
    return (_plain_weight(self.router) is not None and all(_plain_weight(m) is not None for m in (se.gate_proj, se.up_proj, se.down_proj))
            and all(_lora_parts(f) is None and getattr(f, "weight", None) is not None for f in (self.experts.fc1, self.experts.fc2)))


def _moe_composed(self, x2: torch.Tensor, k: int, coeffs, holder) -> torch.Tensor:
    """The MoE block from per-stage autograd functions, for wrapped sub-modules: LoRA-wrapped expert GEMMs run
    `lora._LoraGroupedGemm`; a wrapped router or shared-expert projection runs through its module."""
    se = self.shared_experts
    wr = _plain_weight(self.router)
    logits = _t.LinearFunction.apply(x2, wr) if wr is not None else self.router(x2)
    scores, idx, counts = _t.TopKFunction.apply(logits, k, coeffs, holder)
    offsets, dest, src = ops.build_permutation(idx, counts, row_align=16)
    xp = _t.PermuteFunction.apply(x2, src, dest, k)
    y = _expert_gemm(self.experts.fc2, _lora.swiglu(_expert_gemm(self.experts.fc1, xp, offsets)), offsets)
    ws = [_plain_weight(m) for m in (se.gate_proj, se.up_proj, se.down_proj)]
    if all(w is not None for w in ws):
        shared = _t.LinearFunction.apply(_lora.swiglu(_t.LinearFunction.apply(x2, ws[0], ws[1])), ws[2])
    else:
        shared = se(x2)
    return _t.CombineFunction.apply(y, dest, scores, shared.reshape(x2.shape).contiguous())


def _moe_train_forward(self, hidden_states: torch.Tensor) -> torch.Tensor:
    """Replacement for `MoELayer.forward` / `AriaTextMoELayer.forward` bound by `install(..., trainable=True)`.
      - no gradient needed (no_grad, or nothing requires grad): the inference path — for unwrapped sub-modules the same
        `ops.moe_block_fwd` call as `install()`;
      - otherwise one `moe_train.MoELayerFunction` on the module's own parameters (16-row-aligned permutation, our router,
        explicit backward), with the reference's router losses in train() mode; wrapped sub-modules (LoRA experts, a
        peft-wrapped router or shared-expert projection) run the same stages as separate autograd functions.
    Frozen parameters get no gradient and cost no kernel."""
    if getattr(self, "expert_parallel", None) is not None:
        raise NotImplementedError("aria_b200.install(trainable=True): expert-parallel MoE layers run their own path "
                                  "(aria_b200.expert_parallel); install the trainable seam without expert parallelism")
    plain = _moe_plain(self)                 # raises for unsupported adapters before any kernel runs
    train = torch.is_grad_enabled() and (hidden_states.requires_grad or any(p.requires_grad for p in self.parameters()))
    if not train and plain:
        return _moe_block(self, hidden_states)
    if not hidden_states.is_cuda:
        raise RuntimeError("aria_b200.install(trainable=True): the MoE training path needs CUDA tensors (there is no CPU path)")
    if hidden_states.dtype != torch.bfloat16:
        raise RuntimeError(f"aria_b200.install(trainable=True): expected bf16 hidden states, got {hidden_states.dtype}")
    cfg = getattr(self.router, "config", None) or self.config
    coeffs, holder = _router_losses(self)
    if plain:
        se = self.shared_experts
        return _t.MoELayerFunction.apply(hidden_states, self.router.weight, self.experts.fc1.weight, self.experts.fc2.weight,
                                         se.gate_proj.weight, se.up_proj.weight, se.down_proj.weight, cfg.moe_topk, coeffs, holder)
    shape = hidden_states.shape
    return _moe_composed(self, hidden_states.reshape(-1, shape[-1]).contiguous(), cfg.moe_topk, coeffs, holder).view(shape)


def _vit_layer_forward(self, hidden_states: torch.Tensor, attention_mask=None, *args, **kwargs):
    """Replacement for transformers' `Idefics2EncoderLayer.forward` (what `AriaVisionTransformer` is built from,
    vision_encoder.py:65-67,120), on the module's own parameters: LN -> fused q/k/v GEMM with head scatter -> non-causal attention
    (hd 72 carried in 128-wide rows, key mask) -> out_proj (+residual) -> LN -> fc1 (+bias, gelu_tanh) -> fc2 (+bias, +residual).
    `attention_mask`: None, the 4-D additive mask [B,1,N,N] HF builds from the patch mask, or a 2-D validity mask [B,N]."""
    from . import _lib as L
    _reject_autograd("Idefics2EncoderLayer.forward", self, hidden_states)
    a, m = self.self_attn, self.mlp
    B, N, _ = hidden_states.shape
    H, hd = a.num_heads, a.head_dim
    key_mask = None
    if attention_mask is not None:
        if attention_mask.dim() == 4 and attention_mask.dtype == torch.bool:      # sdpa-style mask: True = may attend
            key_mask = (~attention_mask[:, 0, 0, :]).to(torch.uint8).contiguous()
        elif attention_mask.dim() == 4:
            key_mask = (attention_mask[:, 0, 0, :] < 0).to(torch.uint8).contiguous()
        else:
            key_mask = (~attention_mask.bool()).to(torch.uint8).contiguous()
    buf = getattr(self, "_aria_qkv", None)
    if buf is None or buf[0].shape != (B, H, N, 128) or buf[0].device != hidden_states.device:
        buf = [torch.zeros(B, H, N, 128, dtype=torch.bfloat16, device=hidden_states.device) for _ in range(3)]
        self._aria_qkv = buf            # pad columns hd..127 stay zero across calls
    x = hidden_states.contiguous()
    h = ops.layernorm(x, self.layer_norm1.weight, self.layer_norm1.bias, self.layer_norm1.eps)
    ops.qkv_heads(h, [a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], [a.q_proj.bias, a.k_proj.bias, a.v_proj.bias],
                  buf, hd, N)
    o = ops.attention(buf[0], buf[1], buf[2], N, N, hd ** -0.5, causal=False, out_hd=hd, key_mask=key_mask)
    x = ops.linear(o, a.out_proj.weight, a.out_proj.bias, residual=x)
    h = ops.layernorm(x, self.layer_norm2.weight, self.layer_norm2.bias, self.layer_norm2.eps)
    h = ops.linear(h, m.fc1.weight, m.fc1.bias, act=L.ACT_GELU_TANH)
    out = ops.linear(h, m.fc2.weight, m.fc2.bias, residual=x)
    return (out,) if getattr(self, "_aria_returns_tuple", False) else out


def install_vit(model) -> int:
    """Seam 3: patch every `Idefics2EncoderLayer` inside `model` (the reference's vision tower) with `_vit_layer_forward`.
    transformers 4.46 layers return a 1-tuple, 5.x layers the tensor: detected from the original signature.  Returns the number
    of layers patched.  Requires `hidden_act = gelu_pytorch_tanh` (what Aria uses); anything else is rejected."""
    import inspect
    n = 0
    for mod in model.modules():
        # Idefics2EncoderLayer: the reference's tower (vision_encoder.py:26-28,65-67); Idefics3EncoderLayer: the identical layer
        # transformers' own `models.aria` builds its tower from
        if type(mod).__name__ in ("Idefics2EncoderLayer", "Idefics3EncoderLayer") and hasattr(mod, "self_attn") and hasattr(mod, "layer_norm1"):
            act = type(getattr(mod.mlp, "activation_fn", None)).__name__
            if act not in ("GELUTanh", "PytorchGELUTanh"):
                raise NotImplementedError(f"install_vit: unsupported MLP activation {act} (the fused epilogue is gelu_pytorch_tanh)")
            mod._aria_returns_tuple = "output_attentions" in inspect.signature(type(mod).forward).parameters
            mod.forward = types.MethodType(_vit_layer_forward, mod)
            n += 1
    return n


def install(model, reference_moe_lm_module=None, trainable: bool = False) -> int:
    """Patch every reference `MoELayer` inside `model` (and, if given, the reference module's global `experts_gemm`).
    Returns the number of layers patched.  Idempotent.
    trainable=False: the inference seams (they refuse autograd).  trainable=True: the MoE layers run `_moe_train_forward`
    (differentiable, router losses in train() mode; inference unchanged) and `experts_gemm` becomes the differentiable
    `moe_train.experts_gemm_train`."""
    if trainable and any(type(mod) is _m.Fp8GroupedGEMM for mod in model.modules()):
        raise NotImplementedError("aria_b200.install(trainable=True): fp8 expert weights are inference-only; install the "
                                  "trainable seam on the bf16 model")
    fwd = _moe_train_forward if trainable else _moe_forward
    n = 0
    for mod in model.modules():
        if type(mod).__name__ in ("MoELayer", "AriaTextMoELayer") and hasattr(mod, "router") and hasattr(mod, "experts") \
                and hasattr(mod, "shared_experts"):
            mod.forward = types.MethodType(fwd, mod)
            n += 1
    if reference_moe_lm_module is not None:
        # seam 1: GroupedGEMM.forward calls the module global
        reference_moe_lm_module.experts_gemm = _t.experts_gemm_train if trainable else _m.experts_gemm
    return n


# ------------------------------------------------------------------------------------------------ seam 5: the loss head
def _loss_forward(self, input_ids=None, pixel_values=None, pixel_mask=None, attention_mask=None, position_ids=None,
                  past_key_values=None, inputs_embeds=None, labels=None, use_cache=None, output_attentions=None,
                  output_hidden_states=None, return_dict=None, cache_position=None, num_logits_to_keep=0):
    """Replacement for the reference `AriaForConditionalGeneration.forward` (modeling_aria.py:194-331) bound by
    `install_loss()`.  A training call (labels given, a gradient needed, every logit requested, a dict output, a plain bias-free
    nn.Linear lm_head) runs the reference's steps on the model's own submodules up to the language model's final norm, then
    `loss.linear_cross_entropy` over the reference's rows: position t < T-1 of every sequence predicts labels[:, t+1], kept
    where attention_mask[:, -(T-1):] != 0 (all positions without a mask), labels == -100 ignored.  It returns the reference's
    output class with that fp32 loss and `logits=None`.  Every other call runs the original forward unchanged."""
    kw = dict(input_ids=input_ids, pixel_values=pixel_values, pixel_mask=pixel_mask, attention_mask=attention_mask,
              position_ids=position_ids, past_key_values=past_key_values, inputs_embeds=inputs_embeds, labels=labels,
              use_cache=use_cache, output_attentions=output_attentions, output_hidden_states=output_hidden_states,
              return_dict=return_dict, cache_position=cache_position, num_logits_to_keep=num_logits_to_keep)
    original = type(self).forward
    output_attentions = output_attentions if output_attentions is not None else self.config.output_attentions
    output_hidden_states = output_hidden_states if output_hidden_states is not None else self.config.output_hidden_states
    return_dict = return_dict if return_dict is not None else self.config.use_return_dict
    head = self.language_model.lm_head
    needs_grad = torch.is_grad_enabled() and (any(p.requires_grad for p in self.parameters())
                                              or (inputs_embeds is not None and inputs_embeds.requires_grad))
    if labels is None or not needs_grad or num_logits_to_keep != 0 or not return_dict or _plain_weight(head) is None:
        return original(self, **kw)
    if head.weight.numel() == 0:
        raise RuntimeError("aria_b200.install_loss: lm_head.weight is empty (a ZeRO-3 partition?); the fused loss reads the "
                           "whole weight, so gather it first (or train without install_loss)")

    # the reference's steps before the language model (modeling_aria.py:248-283)
    if inputs_embeds is None:
        inputs_embeds = self.get_input_embeddings()(input_ids)
    if pixel_values is not None:
        image_outputs, image_attn_mask = self.vision_tower(pixel_values, pixel_mask=pixel_mask)
        image_features = self.multi_modal_projector(image_outputs.last_hidden_state, attn_mask=image_attn_mask)
        n_image_tokens = (input_ids == self.config.image_token_index).sum().item()
        n_image_features = image_features.shape[0] * image_features.shape[1]
        if n_image_tokens != n_image_features:
            raise ValueError(
                f"Image features and image tokens do not match: tokens: {n_image_tokens}, features {n_image_features}")
        special_image_mask = (input_ids == self.config.image_token_index).unsqueeze(-1).expand_as(inputs_embeds)
        special_image_mask = special_image_mask.to(inputs_embeds.device)
        image_features = image_features.to(inputs_embeds.device, inputs_embeds.dtype)
        inputs_embeds = inputs_embeds.masked_scatter(special_image_mask, image_features)

    outputs = self.language_model.model(attention_mask=attention_mask, position_ids=position_ids,
                                        past_key_values=past_key_values, inputs_embeds=inputs_embeds, use_cache=use_cache,
                                        output_attentions=output_attentions, output_hidden_states=output_hidden_states,
                                        return_dict=True, cache_position=cache_position)
    hidden = outputs[0]
    B, T, d = hidden.shape
    # rows of the reference's shift (modeling_aria.py:302-318) as labels: the last position of each sequence and the
    # positions the attention mask drops are ignored, so the hidden states go in as one [B*T, d] view without a copy
    shifted = torch.full((B, T), -100, dtype=torch.long, device=hidden.device)
    shifted[:, :-1] = labels[:, 1:].to(hidden.device)
    if attention_mask is not None:
        keep = attention_mask[:, -(T - 1):].to(hidden.device) != 0
        shifted[:, :-1].masked_fill_(~keep, -100)
    loss = _loss.linear_cross_entropy(hidden.reshape(B * T, d), head.weight, shifted.view(-1))
    out_cls = getattr(sys.modules[type(self).__module__], "AriaCausalLMOutputWithPast")
    return out_cls(loss=loss, logits=None, past_key_values=outputs.past_key_values, hidden_states=outputs.hidden_states,
                   attentions=outputs.attentions)


def install_loss(model) -> int:
    """Seam 5: patch `forward` of every reference `AriaForConditionalGeneration` inside `model` (what aria/train.py trains) with
    `_loss_forward`: the training loss from `loss.linear_cross_entropy` instead of full logits and nn.CrossEntropyLoss.
    transformers' own `models.aria` class and this package's inference mirror are left alone.  Returns the number of models
    patched.  Idempotent."""
    n = 0
    for mod in model.modules():
        cls = type(mod)
        if cls.__name__ == "AriaForConditionalGeneration" and not cls.__module__.startswith(("transformers.", "aria_b200.")) \
                and hasattr(sys.modules.get(cls.__module__), "AriaCausalLMOutputWithPast") \
                and hasattr(mod, "language_model") and hasattr(mod.language_model, "lm_head"):
            mod.forward = types.MethodType(_loss_forward, mod)
            n += 1
    return n
