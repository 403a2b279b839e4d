"""TEST INFRASTRUCTURE ONLY — CPU restatement ("port") of the reference Aria forward.

This file is the *oracle* for the parity tests, `__graft_entry__.smoke()` and the `cpu_baseline` /
`--impl reference` legs of `bench.py`.  Nothing under `aria_b200/` may import it: the product path has
no CPU fallback.

It restates, function by function, what the reference (rhymes-ai/Aria @ 9b25fecb, `/root/reference`)
computes on the hot path, as plain torch CPU code over an explicit state-dict with the Hugging Face
weight names.  Each function cites the reference file:line it follows.  Where the reference reaches
into a third-party package that is not under /root/reference, the package + version is named:

  * LM attention / RMSNorm / RoPE / decoder wiring : transformers (reference pins 4.46.3,
    pyproject.toml:13; checked here against the installed 5.5.0 `LlamaAttention` eager path)
  * ViT                                              : transformers Idefics2VisionTransformer
  * projector attention                              : torch.nn.MultiheadAttention (torch 2.5.1 pinned)
  * expert GEMM                                      : grouped_gemm==0.1.6 — the reference's own
    `sequential_gemm` (moe_lm.py:398-428) is a full restatement and is what we follow.

Parity pinning: the reference ships NO golden vectors / model-forward tests (SURVEY.md §4).  This oracle
is pinned instead against outputs of the reference modules themselves, run in the build container by
`oracle/make_golden.py` (fixtures in tests/golden/, checked by tests/test_oracle_golden.py and, when
/root/reference is present, live by tests/test_oracle_vs_reference.py).

Rounding follows the reference exactly: every torch op on a bf16 tensor rounds its result to bf16
(e.g. fc1 -> bf16, silu -> bf16, product -> bf16), softmax statistics are fp32.

Tie rule for top-k: the reference calls `torch.topk` (moe_lm.py:261) whose tie order is unspecified.
The oracle (and the CUDA kernel) define it: among equal logits the LOWEST expert index wins, and
selected experts are returned in descending-logit order (ties: ascending index).
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor


# ----------------------------------------------------------------------------------------------
# MoE block  (aria/model/moe_lm.py)
# ----------------------------------------------------------------------------------------------
def router_gating(x: Tensor, w_router: Tensor) -> Tensor:
    """moe_lm.py:190-201 `TopKRouter.gating`: logits = F.linear(x, W[E,d]) in the input dtype."""
    return F.linear(x, w_router)


def topk_lowest_index(logits: Tensor, k: int) -> Tuple[Tensor, Tensor]:
    """moe_lm.py:261 `torch.topk(logits, k, dim=1)` with the tie rule made explicit (see header)."""
    idx = torch.sort(logits.detach().float(), dim=1, descending=True, stable=True).indices[:, :k]
    return torch.gather(logits, 1, idx), idx


class _LossGradInjector(torch.autograd.Function):
    """moe_lm.py:84-125 `MoEAuxLossAutoScaler`: identity on `passthrough`; in backward the attached loss receives the
    gradient `scale` (so the loss acts only through d(loss)/d(logits) * scale, never through its value)."""

    scale = 1.0

    @staticmethod
    def forward(ctx, passthrough, loss):
        ctx.save_for_backward(loss)
        return passthrough

    @staticmethod
    def backward(ctx, grad):
        (loss,) = ctx.saved_tensors
        return grad, torch.ones_like(loss) * _LossGradInjector.scale


def z_loss(logits: Tensor, coeff: float) -> Tensor:
    """moe_lm.py:128-140: mean over tokens of logsumexp(logits)^2, times the coefficient (in the logits dtype)."""
    return torch.logsumexp(logits, dim=-1).square().mean() * coeff


def load_balancing_loss(probs: Tensor, counts: Tensor, k: int, coeff: float) -> Tensor:
    """moe_lm.py:143-166 (Switch): sum_e mean_t(probs)_e * count_e * E / (T*k) * coeff."""
    T, E = probs.shape
    return (probs.mean(dim=0) * counts).sum() * (E / (T * k) * coeff)


def router_routing(logits: Tensor, k: int, loss_coeffs: Optional[Tuple[float, float]] = None) -> Tuple[Tensor, Tensor, Tensor]:
    """moe_lm.py:243-273: topk -> softmax(fp32)->dtype -> per-expert histogram.  `loss_coeffs=(z, aux)` selects the
    `self.training` branch (:257-258, :271-272): z-loss attached to the logits before top-k, load-balancing loss
    (fp32 softmax over all experts, :235) attached to the scores."""
    if loss_coeffs is not None:
        logits = _LossGradInjector.apply(logits, z_loss(logits, loss_coeffs[0]))
    top_logits, top_idx = topk_lowest_index(logits, k)
    scores = torch.softmax(top_logits, dim=-1, dtype=torch.float32).type_as(logits)
    counts = torch.bincount(top_idx.flatten(), minlength=logits.shape[1])  # == histc, :264-269
    if loss_coeffs is not None:
        probs = torch.softmax(logits, dim=-1, dtype=torch.float32)
        scores = _LossGradInjector.apply(scores, load_balancing_loss(probs, counts, k, loss_coeffs[1]))
    return scores, top_idx, counts


def router_loss_grad(logits: Tensor, counts: Tensor, k: int, z_coeff: float, aux_coeff: float, scale: float = 1.0) -> Tensor:
    """Closed form (fp32) of what the two attached losses add to d/d(logits):
    scale * p * (2 c_z lse / T + g - <p, g>),  g_e = c_aux * E * count_e / (T k T),  p = softmax(logits), lse = logsumexp."""
    lf = logits.float()
    T, E = lf.shape
    p = torch.softmax(lf, dim=-1)
    lse = torch.logsumexp(lf, dim=-1, keepdim=True)
    g = (aux_coeff * E / (T * k * T)) * counts.float()[None, :]
    return scale * p * (2.0 * z_coeff * lse / T + g - (p * g).sum(-1, keepdim=True))


def token_permutation(x: Tensor, top_idx: Tensor, k: int) -> Tuple[Tensor, Tensor]:
    """moe_lm.py:313-334: stable argsort of the flattened expert ids; rows = x[order // k]."""
    flat = top_idx.flatten()
    order = torch.argsort(flat, stable=True)
    return x.index_select(0, order // k), order


def sequential_gemm(inp: Tensor, weight: Tensor, counts: Tensor) -> Tensor:
    """moe_lm.py:398-428: per-expert matmul over contiguous row groups, weight [E, in, out]."""
    out = torch.zeros(inp.shape[0], weight.shape[-1], dtype=inp.dtype, device=inp.device)
    off = 0
    for e in range(weight.shape[0]):
        n = int(counts[e])
        if n:
            out[off : off + n] = inp[off : off + n] @ weight[e]
        off += n
    return out


def grouped_gemm_lora(x: Tensor, w: Tensor, lora_a: Tensor, lora_b: Tensor, counts: Tensor, scaling: float) -> Tensor:
    """aria/lora/layers.py:125-140 `GroupedGemmLoraLayer.forward` (one active adapter, dropout = identity, no DoRA):
    result = base_layer(x, tpe) + lora_B(lora_A(x, tpe), tpe) * scaling, where lora_A / lora_B are `GroupedGEMM`s
    (layers.py:87-92) with weights [E, in, r] / [E, r, out].  NOT pinned to a live reference run: the layer needs
    `peft`, which is absent offline; the arithmetic is the reference's own `sequential_gemm` applied three times."""
    result = sequential_gemm(x, w, counts)
    return result + sequential_gemm(sequential_gemm(x, lora_a, counts), lora_b, counts) * scaling


def glu(x: Tensor) -> Tensor:
    """moe_lm.py:505-507: first half is the gate (silu), second half the up projection."""
    a, b = torch.chunk(x, 2, dim=-1)
    return F.silu(a) * b


def grouped_mlp(permuted: Tensor, fc1: Tensor, fc2: Tensor, counts: Tensor) -> Tensor:
    """moe_lm.py:511-525 `GroupedMLP.forward`."""
    h = sequential_gemm(permuted, fc1, counts)
    h = glu(h)
    return sequential_gemm(h, fc2, counts)


def token_unpermutation(y: Tensor, order: Tensor, scores: Tensor, k: int) -> Tensor:
    """moe_lm.py:336-365: scatter rows back, scale by scores (bf16 multiply), sum over k."""
    buf = torch.zeros((scores.numel(), y.shape[1]), dtype=y.dtype, device=y.device)
    buf.index_copy_(0, order, y)
    buf = buf.reshape(-1, k, y.shape[1])
    buf = buf * scores.unsqueeze(-1)
    return buf.sum(dim=1).type_as(y)


def shared_expert_mlp(x: Tensor, gate_w: Tensor, up_w: Tensor, down_w: Tensor) -> Tensor:
    """moe_lm.py:368-395 -> LlamaMLP.forward: down(silu(gate(x)) * up(x)), no bias."""
    return F.linear(F.silu(F.linear(x, gate_w)) * F.linear(x, up_w), down_w)


def moe_layer(x: Tensor, w: Dict[str, Tensor], k: int, prefix: str = "", return_parts: bool = False,
              loss_coeffs: Optional[Tuple[float, float]] = None):
    """moe_lm.py:548-577 `MoELayer.forward`.  `w` uses the reference parameter names:
    router.weight [E,d], experts.fc1.weight [E,d,2I], experts.fc2.weight [E,I,d],
    shared_experts.{gate,up,down}_proj.weight."""
    shape = x.shape
    x2 = x.reshape(-1, shape[-1])
    logits = router_gating(x2, w[prefix + "router.weight"])
    scores, top_idx, counts = router_routing(logits, k, loss_coeffs)
    permuted, order = token_permutation(x2, top_idx, k)
    y = grouped_mlp(permuted, w[prefix + "experts.fc1.weight"], w[prefix + "experts.fc2.weight"], counts)
    out = token_unpermutation(y, order, scores, k).view(shape)
    shared = shared_expert_mlp(
        x,
        w[prefix + "shared_experts.gate_proj.weight"],
        w[prefix + "shared_experts.up_proj.weight"],
        w[prefix + "shared_experts.down_proj.weight"],
    )
    out = out + shared  # moe_lm.py:576 `output += shared_expert_output`
    if return_parts:
        return out, dict(logits=logits, scores=scores, top_idx=top_idx, counts=counts, order=order,
                         permuted=permuted, expert_out=y, shared=shared)
    return out


# ----------------------------------------------------------------------------------------------
# LM decoder layer  (moe_lm.py:580-636 wiring; arithmetic from transformers modeling_llama)
# ----------------------------------------------------------------------------------------------
def rms_norm(x: Tensor, weight: Tensor, eps: float) -> Tensor:
    """LlamaRMSNorm.forward (used at moe_lm.py:599-602,631): fp32 statistics, cast, then * weight."""
    dt = x.dtype
    h = x.to(torch.float32)
    var = h.pow(2).mean(-1, keepdim=True)
    h = h * torch.rsqrt(var + eps)
    return weight * h.to(dt)


def rope_cos_sin(position_ids: Tensor, head_dim: int, theta: float, dtype) -> Tuple[Tensor, Tensor]:
    """LlamaRotaryEmbedding.forward (moe_lm.py:632): fp32 angles, cos/sin cast to the model dtype."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.int64).float() / head_dim))
    freqs = position_ids[:, :, None].float() * inv_freq[None, None, :]
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos().to(dtype), emb.sin().to(dtype)


def rotate_half(x: Tensor) -> Tensor:
    x1 = x[..., : x.shape[-1] // 2]
    x2 = x[..., x.shape[-1] // 2 :]
    return torch.cat((-x2, x1), dim=-1)


def apply_rope(q: Tensor, k: Tensor, cos: Tensor, sin: Tensor) -> Tuple[Tensor, Tensor]:
    """apply_rotary_pos_emb, rotate-half convention (HF path; gptfast uses interleaved)."""
    cos = cos.unsqueeze(1)
    sin = sin.unsqueeze(1)
    return (q * cos) + (rotate_half(q) * sin), (k * cos) + (rotate_half(k) * sin)


def attention_core(q: Tensor, k: Tensor, v: Tensor, scaling: float, add_mask: Optional[Tensor]) -> Tensor:
    """transformers `eager_attention_forward`: softmax(q k^T * s + mask) in fp32 -> dtype, @ v.
    q [B,H,Tq,D], k/v [B,H,Tk,D]; returns [B,Tq,H,D]."""
    w = torch.matmul(q, k.transpose(2, 3)) * scaling
    if add_mask is not None:
        w = w + add_mask
    w = F.softmax(w, dim=-1, dtype=torch.float32).to(q.dtype)
    return torch.matmul(w, v).transpose(1, 2).contiguous()


def causal_additive_mask(tq: int, tk: int, dtype) -> Tensor:
    """Causal mask for queries occupying the LAST tq positions of tk keys."""
    i = torch.arange(tq)[:, None] + (tk - tq)
    j = torch.arange(tk)[None, :]
    m = torch.zeros(tq, tk, dtype=dtype)
    m.masked_fill_(j > i, torch.finfo(dtype).min)
    return m[None, None]


def lm_attention(x: Tensor, w: Dict[str, Tensor], prefix: str, n_heads: int, theta: float,
                 position_ids: Tensor, past_kv: Optional[Tuple[Tensor, Tensor]] = None):
    """LlamaAttention.forward selected at moe_lm.py:594 (MHA, no bias): q/k/v proj -> RoPE ->
    cache append -> causal softmax attention -> o_proj.  Returns (out, (k_cache, v_cache))."""
    B, T, d = x.shape
    hd = d // n_heads
    q = F.linear(x, w[prefix + "q_proj.weight"]).view(B, T, n_heads, hd).transpose(1, 2)
    k = F.linear(x, w[prefix + "k_proj.weight"]).view(B, T, n_heads, hd).transpose(1, 2)
    v = F.linear(x, w[prefix + "v_proj.weight"]).view(B, T, n_heads, hd).transpose(1, 2)
    cos, sin = rope_cos_sin(position_ids, hd, theta, x.dtype)
    q, k = apply_rope(q, k, cos, sin)
    if past_kv is not None:
        k = torch.cat([past_kv[0], k], dim=2)
        v = torch.cat([past_kv[1], v], dim=2)
    mask = causal_additive_mask(T, k.shape[2], x.dtype) if T > 1 else None
    o = attention_core(q, k, v, hd ** -0.5, mask).reshape(B, T, d)
    return F.linear(o, w[prefix + "o_proj.weight"]), (k, v)


def moe_decoder_layer(x: Tensor, w: Dict[str, Tensor], prefix: str, cfg, position_ids: Tensor,
                      past_kv=None, router_logits: Optional[list] = None):
    """LlamaDecoderLayer.forward with mlp=MoELayer (moe_lm.py:590-602)."""
    r = x
    h = rms_norm(x, w[prefix + "input_layernorm.weight"], cfg["rms_norm_eps"])
    h, kv = lm_attention(h, w, prefix + "self_attn.", cfg["num_attention_heads"], cfg["rope_theta"],
                         position_ids, past_kv)
    x = r + h
    r = x
    h = rms_norm(x, w[prefix + "post_attention_layernorm.weight"], cfg["rms_norm_eps"])
    if router_logits is not None:
        h, parts = moe_layer(h, w, cfg["moe_topk"], prefix + "mlp.", return_parts=True)
        router_logits.append(parts["logits"])
    else:
        h = moe_layer(h, w, cfg["moe_topk"], prefix + "mlp.")
    return r + h, kv


def lm_forward(inputs_embeds: Tensor, w: Dict[str, Tensor], cfg, prefix: str = "language_model.",
               past=None, num_logits_to_keep: int = 0, router_logits: Optional[list] = None):
    """AriaMoELMForCausalLM.forward (moe_lm.py:605-661): layers -> final RMSNorm -> lm_head."""
    B, T, _ = inputs_embeds.shape
    past_len = 0 if past is None else past[0][0].shape[2]
    position_ids = (torch.arange(T) + past_len)[None].expand(B, T)
    x = inputs_embeds
    new_past = []
    for i in range(cfg["num_hidden_layers"]):
        x, kv = moe_decoder_layer(x, w, f"{prefix}model.layers.{i}.", cfg, position_ids,
                                  None if past is None else past[i], router_logits)
        new_past.append(kv)
    x = rms_norm(x, w[prefix + "model.norm.weight"], cfg["rms_norm_eps"])
    if num_logits_to_keep:
        x = x[:, -num_logits_to_keep:, :]
    return F.linear(x, w[prefix + "lm_head.weight"]), new_past


# ----------------------------------------------------------------------------------------------
# ViT  (aria/model/vision_encoder.py + transformers Idefics2VisionTransformer)
# ----------------------------------------------------------------------------------------------
def patch_attention_mask(pixel_mask: Tensor, patch: int) -> Tensor:
    """vision_encoder.py:132-145: a patch is valid iff any of its pixels is."""
    sub = pixel_mask.unfold(1, patch, patch).unfold(2, patch, patch)
    return (sub.sum(dim=(-1, -2)) > 0).bool()


def vit_position_ids(pmask: Tensor, n_side: int) -> Tensor:
    """Idefics2VisionEmbeddings.forward of transformers 4.46.3 (the release the reference pins, pyproject.toml:13): per image,
    fp32 fractional coordinates `arange(0, 1 - 1e-6, 1 / nb)` bucketised against `arange(1/n, 1, 1/n)` (right=True), ids of
    the nb_h x nb_w valid grid written to the True positions of the patch mask.  (transformers 5.x casts the coordinates to
    the pixel dtype before bucketising; in bf16 that shifts about half of the 70 buckets by one, so it is NOT what a
    checkpoint trained under 4.46.3 saw.)"""
    B, Hp, Wp = pmask.shape
    boundaries = torch.arange(1 / n_side, 1.0, 1 / n_side)
    pos = torch.zeros(B, Hp * Wp, dtype=torch.long)
    for b in range(B):
        p = pmask[b]
        nb_h, nb_w = p[:, 0].sum(), p[0].sum()
        fh = torch.arange(0, 1 - 1e-6, 1 / nb_h)
        fw = torch.arange(0, 1 - 1e-6, 1 / nb_w)
        bh = torch.bucketize(fh, boundaries, right=True)
        bw = torch.bucketize(fw, boundaries, right=True)
        pos[b][p.reshape(-1)] = (bh[:, None] * n_side + bw).flatten()
    return pos


def vit_embeddings(pixel_values: Tensor, pmask: Tensor, w: Dict[str, Tensor], vcfg, prefix: str) -> Tensor:
    """Idefics2VisionEmbeddings.forward: Conv2d patch embedding + bucketised position embedding."""
    P = vcfg["patch_size"]
    x = F.conv2d(pixel_values, w[prefix + "embeddings.patch_embedding.weight"],
                 w[prefix + "embeddings.patch_embedding.bias"], stride=P)
    x = x.flatten(2).transpose(1, 2)
    pos = vit_position_ids(pmask, vcfg["image_size"] // P)
    return x + F.embedding(pos, w[prefix + "embeddings.position_embedding.weight"])


def vit_encoder_layer(x: Tensor, w: Dict[str, Tensor], p: str, vcfg, add_mask: Optional[Tensor]) -> Tensor:
    """Idefics2EncoderLayer.forward: pre-LN MHA (bias, non-causal, key mask) + pre-LN MLP (gelu_pytorch_tanh)."""
    B, N, d = x.shape
    H = vcfg["num_attention_heads"]
    hd = d // H
    eps = vcfg["layer_norm_eps"]
    r = x
    h = F.layer_norm(x, (d,), w[p + "layer_norm1.weight"], w[p + "layer_norm1.bias"], eps)
    q = F.linear(h, w[p + "self_attn.q_proj.weight"], w[p + "self_attn.q_proj.bias"])
    k = F.linear(h, w[p + "self_attn.k_proj.weight"], w[p + "self_attn.k_proj.bias"])
    v = F.linear(h, w[p + "self_attn.v_proj.weight"], w[p + "self_attn.v_proj.bias"])
    q = q.view(B, N, H, hd).transpose(1, 2)
    k = k.view(B, N, H, hd).transpose(1, 2)
    v = v.view(B, N, H, hd).transpose(1, 2)
    o = attention_core(q, k, v, hd ** -0.5, add_mask).reshape(B, N, d)
    o = F.linear(o, w[p + "self_attn.out_proj.weight"], w[p + "self_attn.out_proj.bias"])
    x = r + o
    r = x
    h = F.layer_norm(x, (d,), w[p + "layer_norm2.weight"], w[p + "layer_norm2.bias"], eps)
    h = F.linear(h, w[p + "mlp.fc1.weight"], w[p + "mlp.fc1.bias"])
    h = F.gelu(h, approximate="tanh")  # gelu_pytorch_tanh
    h = F.linear(h, w[p + "mlp.fc2.weight"], w[p + "mlp.fc2.bias"])
    return r + h


def vit_forward(pixel_values: Tensor, pixel_mask: Optional[Tensor], w: Dict[str, Tensor], vcfg,
                prefix: str = "vision_tower.vision_model."):
    """AriaVisionModel.forward (vision_encoder.py:94-130) over AriaVisionTransformer (:58-67: no
    post-layernorm).  Returns (last_hidden_state [B,N,d], image_attn_mask [B,N] bool, True = pad)."""
    P = vcfg["patch_size"]
    B = pixel_values.shape[0]
    dt = pixel_values.dtype
    if pixel_mask is None:
        pmask = torch.ones(B, pixel_values.shape[2] // P, pixel_values.shape[3] // P, dtype=torch.bool)
    else:
        pmask = patch_attention_mask(pixel_mask, P)
    x = vit_embeddings(pixel_values, pmask, w, vcfg, prefix)
    flat = pmask.view(B, -1)
    add_mask = None
    if not bool(flat.all()):
        add_mask = torch.zeros(B, 1, 1, flat.shape[1], dtype=dt)
        add_mask.masked_fill_(~flat[:, None, None, :], torch.finfo(dt).min)
    for i in range(vcfg["num_hidden_layers"]):
        x = vit_encoder_layer(x, w, f"{prefix}encoder.layers.{i}.", vcfg, add_mask)
    return x, torch.logical_not(flat)  # vision_encoder.py:147-152


# ----------------------------------------------------------------------------------------------
# Projector  (aria/model/projector.py)
# ----------------------------------------------------------------------------------------------
def gelu_new(x: Tensor) -> Tensor:
    """transformers ACT2FN['gelu_new'] (projector.py:40)."""
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3.0))))


def projector_forward(x: Tensor, image_attn_mask: Optional[Tensor], w: Dict[str, Tensor], pcfg,
                      prefix: str = "multi_modal_projector."):
    """AriaProjector.forward (projector.py:160-189) incl. CrossAttention (:73-102) and FFN (:42-45).
    nn.MultiheadAttention math: second in-projection (with bias) of q/k/v, scaled dot-product with a
    boolean key mask (True = not allowed), out_proj."""
    B, N, _ = x.shape
    E = pcfg["embed_dim"]
    H = pcfg["num_heads"]
    hd = E // H
    Q = pcfg["patch_to_query_dict"][N]
    queries = w[prefix + "query"][:Q].unsqueeze(0).repeat(B, 1, 1)
    ca = prefix + "cross_attn."
    nq = F.layer_norm(queries, (E,), w[ca + "layer_norm.weight"], w[ca + "layer_norm.bias"], 1e-5)
    query = F.linear(nq, w[ca + "q_proj.weight"])
    xk = F.layer_norm(x, (x.shape[-1],), w[ca + "ln_kv.weight"], w[ca + "ln_kv.bias"], 1e-5)
    key = F.linear(xk, w[ca + "k_proj.weight"])
    value = F.linear(xk, w[ca + "v_proj.weight"])
    wi, bi = w[ca + "multihead_attn.in_proj_weight"], w[ca + "multihead_attn.in_proj_bias"]
    q2 = F.linear(query, wi[:E], bi[:E]).view(B, Q, H, hd).transpose(1, 2)
    k2 = F.linear(key, wi[E : 2 * E], bi[E : 2 * E]).view(B, N, H, hd).transpose(1, 2)
    v2 = F.linear(value, wi[2 * E :], bi[2 * E :]).view(B, N, H, hd).transpose(1, 2)
    # torch MHA: q scaled by 1/sqrt(hd) before the matmul (baddbmm path); softmax in the model dtype
    # for the math path.  We keep fp32 softmax statistics -> dtype, which bounds both.
    add_mask = None
    if image_attn_mask is not None:
        add_mask = torch.zeros(B, 1, 1, N, dtype=x.dtype)
        add_mask.masked_fill_(image_attn_mask[:, None, None, :], float("-inf"))
    o = attention_core(q2, k2, v2, hd ** -0.5, add_mask).reshape(B, Q, E)
    o = F.linear(o, w[ca + "multihead_attn.out_proj.weight"], w[ca + "multihead_attn.out_proj.bias"])
    o = F.linear(o, w[ca + "linear.weight"], w[ca + "linear.bias"])
    h = F.layer_norm(o, (E,), w[prefix + "ln_ffn.weight"], w[prefix + "ln_ffn.bias"], 1e-5)
    h = gelu_new(F.linear(h, w[prefix + "ffn.linear_in.weight"]))
    return F.linear(h, w[prefix + "ffn.linear_out.weight"])


# ----------------------------------------------------------------------------------------------
# Full model  (aria/model/modeling_aria.py:194-335)
# ----------------------------------------------------------------------------------------------
def topk_margin(router_logits: list, k: int) -> Tensor:
    """Per token: the smallest gap, over all layers, between the k-th and (k+1)-th router logit relative to the
    largest |logit|.  Tokens whose margin is within bf16 rounding noise may legitimately be routed to another
    expert by an implementation with a different fp32 summation order; parity tests treat them separately."""
    m = None
    for lg in router_logits:
        v = lg.float().sort(dim=1, descending=True).values
        gap = (v[:, k - 1] - v[:, k]) / v.abs().amax(dim=1).clamp_min(1e-12)
        m = gap if m is None else torch.minimum(m, gap)
    return m


def aria_forward(input_ids: Tensor, pixel_values: Optional[Tensor], pixel_mask: Optional[Tensor],
                 w: Dict[str, Tensor], cfg, num_logits_to_keep: int = 0, router_logits: Optional[list] = None):
    """AriaForConditionalGeneration.forward: embed -> ViT -> projector -> masked_scatter merge -> LM."""
    tcfg = cfg["text_config"]
    emb = F.embedding(input_ids, w["language_model.model.embed_tokens.weight"])
    if pixel_values is not None:
        feats, img_mask = vit_forward(pixel_values, pixel_mask, w, cfg["vision_config"])
        feats = projector_forward(feats, img_mask if pixel_mask is not None else None, w, cfg["projector"])
        n_tok = int((input_ids == cfg["image_token_index"]).sum())
        if n_tok != feats.shape[0] * feats.shape[1]:
            raise ValueError(  # modeling_aria.py:268-271
                f"Image features and image tokens do not match: tokens: {n_tok}, "
                f"features {feats.shape[0] * feats.shape[1]}")
        m = (input_ids == cfg["image_token_index"]).unsqueeze(-1).expand_as(emb)
        emb = emb.masked_scatter(m, feats.to(emb.dtype))
    logits, past = lm_forward(emb, w, tcfg, num_logits_to_keep=num_logits_to_keep, router_logits=router_logits)
    return logits, past
