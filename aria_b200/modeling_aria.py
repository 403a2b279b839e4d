"""Host-side mirror of `aria/model/modeling_aria.py`: AriaForConditionalGeneration.forward()/generate() with the
Hugging Face state-dict layout, running entirely on the H100-native kernels.

forward() follows modeling_aria.py:194-335: embed -> vision tower -> projector -> masked_scatter merge -> LM, with the
reference's argument list (attention_mask, position_ids, labels -> loss, ...).  Differences that are deliberate: no
autograd through this class (inference hot path; training = moe_train / lora), the KV cache is our static `KVCache`
(HF layout [B,H,T,hd] per layer), integer index tensors stay int32 on the device.  The drop-in surface for an
*unmodified* HF / reference model is aria_b200.install + aria_b200.hf_attention (tests/test_gpu_dropin.py).
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from . import ops
from .moe_lm import KV_CACHE_DTYPES, AriaMoELMConfig, AriaMoELMForCausalLM, KVCache, bf16
from .projector import AriaProjector
from .vision_encoder import AriaVisionConfig, AriaVisionModel


class AriaConfig:
    """configuration_aria.py:31-114 (attributes used on the hot path)."""

    def __init__(self, vision_config, text_config, projector_patch_to_query_dict=None, image_token_index=32000,
                 ignore_index=-100, **_ignored):
        self.vision_config = vision_config if not isinstance(vision_config, dict) else AriaVisionConfig(**vision_config)
        self.text_config = text_config if not isinstance(text_config, dict) else AriaMoELMConfig(**text_config)
        self.projector_patch_to_query_dict = {int(k): int(v) for k, v in
                                              (projector_patch_to_query_dict or {1225: 128, 4900: 256}).items()}
        self.image_token_index = image_token_index
        self.ignore_index = ignore_index

    @classmethod
    def from_dict(cls, cfg: dict):
        """From the plain-dict configs used by oracle/configs.py and bench.py."""
        return cls(cfg["vision_config"], cfg["text_config"], cfg["projector"]["patch_to_query_dict"],
                   cfg["image_token_index"])


class AriaCausalLMOutputWithPast:
    def __init__(self, logits, past_key_values):
        self.logits = logits
        self.past_key_values = past_key_values
        self.loss = None


class AriaForConditionalGeneration(nn.Module):
    """modeling_aria.py:125-365."""

    def __init__(self, config: AriaConfig, device=None):
        super().__init__()
        self.config = config
        v, t = config.vision_config, config.text_config
        self.vision_tower = AriaVisionModel(v, device)
        self.multi_modal_projector = AriaProjector(  # build_mm_projector, modeling_aria.py:102-122
            config.projector_patch_to_query_dict, v.hidden_size, v.num_attention_heads, v.hidden_size, t.hidden_size,
            t.hidden_size, device)
        self.vocab_size = t.vocab_size
        self.language_model = AriaMoELMForCausalLM(t, device)

    # ---- modeling_aria.py:145-192: the helpers aria/train.py:70-75 and the recipes call on the model
    def freeze_vit(self):
        for p in self.vision_tower.parameters():
            p.requires_grad = False

    def freeze_projector(self):
        for p in self.multi_modal_projector.parameters():
            p.requires_grad = False

    def freeze_llm(self):
        for p in self.language_model.parameters():
            p.requires_grad = False

    def get_input_embeddings(self):
        return self.language_model.get_input_embeddings()

    def set_input_embeddings(self, value):
        self.language_model.set_input_embeddings(value)

    def get_output_embeddings(self):
        return self.language_model.get_output_embeddings()

    def set_output_embeddings(self, value):
        self.language_model.set_output_embeddings(value)

    def set_moe_z_loss_coeff(self, value):
        self.language_model.set_z_loss_coeff(value)

    def set_moe_aux_loss_coeff(self, value):
        self.language_model.set_aux_loss_coeff(value)

    def enable_expert_parallel(self, max_tokens: int, group=None):
        """Shard the routed experts of every MoE layer over the ranks of `group` (rank r serves experts
        [r*E/W, (r+1)*E/W), a dim-0 view of the HF weights) and exchange token rows over NVLink peer memory
        (aria_b200.expert_parallel.FusedPeerTransport: dispatch fused into the permute kernel, return path fused into the fc2
        GEMM epilogue).  Every rank must then call forward() in lock-step with its own tokens."""
        import torch.distributed as dist
        from .expert_parallel import ExpertParallelMoE, FusedPeerTransport
        if any(layer.mlp.experts.is_fp8() for layer in self.language_model.model.layers):
            raise NotImplementedError("enable_expert_parallel: the experts are quantized to fp8; expert parallelism runs on "
                                      "bf16 expert weights")
        if self._dense_fp8_layers():
            raise NotImplementedError("enable_expert_parallel: the attention projections and shared experts are quantized to "
                                      "fp8 (quantize_dense_fp8); expert parallelism runs on bf16 dense weights")
        t = self.config.text_config
        W, r = dist.get_world_size(group), dist.get_rank(group)
        tr = FusedPeerTransport(max_tokens, t.hidden_size, t.moe_intermediate_size, t.moe_num_experts, t.moe_topk, self.device, group)
        lo, hi = r * t.moe_num_experts // W, (r + 1) * t.moe_num_experts // W
        for layer in self.language_model.model.layers:
            m = layer.mlp
            w = {"router.weight": m.router.weight, "experts.fc1.weight": m.experts.fc1.weight[lo:hi],
                 "experts.fc2.weight": m.experts.fc2.weight[lo:hi],
                 "shared_experts.gate_proj.weight": m.shared_experts.gate_proj.weight,
                 "shared_experts.up_proj.weight": m.shared_experts.up_proj.weight,
                 "shared_experts.down_proj.weight": m.shared_experts.down_proj.weight}
            m.expert_parallel = ExpertParallelMoE(w, t.moe_num_experts, t.moe_topk, group=group, transport=tr)
        self._ep_transport = tr
        return tr

    _DENSE_FP8 = (("self_attn", ("q_proj", "k_proj", "v_proj", "o_proj")),
                  ("mlp.shared_experts", ("gate_proj", "up_proj", "down_proj")))

    def _dense_fp8_layers(self):
        """Indices of the LM layers whose attention projections or shared experts are fp8 (Fp8Linear)."""
        from .moe_lm import Fp8Linear
        out = []
        for i, layer in enumerate(self.language_model.model.layers):
            for owner, names in self._DENSE_FP8:
                mod = layer.get_submodule(owner)
                if any(type(getattr(mod, n)) is Fp8Linear for n in names):
                    out.append(i)
                    break
        return out

    @torch.no_grad()
    def quantize_dense_fp8(self):
        """Quantize every LM layer's attention projections (q, k, v, o) and shared experts (gate, up, down) to W8A8 in
        place: e4m3 weights with one fp32 scale per output channel (amax / 448), Fp8Linear.  Their inputs are quantized to
        e4m3 with one scale per row right before each GEMM (q/k/v: in input_layernorm's kernel, rmsnorm_quantize_fp8).
        The dense linears are more than half of what a batch-1 W8A8 decode step streams.  lm_head, router, embedding and
        the ViT stay bf16.  Layer by layer; the bf16 tensors are freed.  Independent of quantize_experts_fp8 (either mode)
        and of the KV cache dtype.  A second call changes nothing.  Returns the model.
        Raises NotImplementedError under expert parallelism or for a projection that is not a plain bias-free Linear
        (e.g. LoRA-wrapped), and ValueError for non-finite weights, all before anything changes.  The captured decode graph
        of generate() is dropped (it holds the old weight pointers); a GraphedPrefill built before the call must be rebuilt."""
        from .moe_lm import Fp8Linear, Linear
        layers = self.language_model.model.layers
        if any(layer.mlp.expert_parallel is not None for layer in layers):
            raise NotImplementedError("quantize_dense_fp8: expert parallelism is enabled; it runs on bf16 dense weights")
        todo = []
        for i, layer in enumerate(layers):
            for owner, names in self._DENSE_FP8:
                mod = layer.get_submodule(owner)
                for name in names:
                    lin = getattr(mod, name)
                    if type(lin) is Fp8Linear:
                        continue
                    if type(lin) is not Linear or lin.bias is not None:
                        raise NotImplementedError(f"quantize_dense_fp8: layer {i} {owner}.{name} is a {type(lin).__name__} "
                                                  "(e.g. LoRA-wrapped) or has a bias, not a plain bias-free Linear")
                    if not bool(torch.isfinite(lin.weight).all()):
                        raise ValueError(f"quantize_dense_fp8: layer {i} {owner}.{name}.weight has non-finite values")
                    todo.append((mod, name))
        if not todo:
            return self
        self._decode_graph = None
        for mod, name in todo:
            setattr(mod, name, Fp8Linear.from_linear(getattr(mod, name)))   # drops the bf16 module
        return self

    @torch.no_grad()
    def quantize_experts_fp8(self, activations: str = "bf16"):
        """Quantize every MoE layer's routed experts (`experts.fc1` / `experts.fc2`) to fp8 in place: e4m3 weights with one
        fp32 scale per (expert, output column), Fp8GroupedGEMM.  It halves the bytes of the routed experts, which are most of
        the model and most of what a decode step reads.  Layer by layer, so the peak is the bf16 model plus one layer's fp8
        copy; the bf16 expert tensors are freed.  Router, lm_head and the ViT stay bf16, and so do attention and the shared
        experts unless quantize_dense_fp8() is called.
        `activations`: "bf16" keeps the activations in bf16 (weight-only, W8A16); "fp8" also quantizes the expert GEMMs'
        inputs to e4m3 with one scale per row (W8A8, the fp8 tensor cores).  W8A8 rounds the activations as well, so it is
        an explicit choice, never made by row count.  Both modes hold the same codes, scales and state dict; a model
        quantized in one mode is switched to the other by re-laying out its codes, without re-quantizing.  A call in the
        mode the model is already in changes nothing.  Returns the model.
        Raises ValueError for an unknown mode or non-finite expert weights and NotImplementedError under expert
        parallelism, all before anything changes.  The captured decode graph of generate() is dropped (it holds the old
        weight pointers); a GraphedPrefill built before the call must be rebuilt."""
        from .moe_lm import Fp8GroupedGEMM, GroupedGEMM
        if activations not in ("bf16", "fp8"):
            raise ValueError(f"quantize_experts_fp8: activations must be 'bf16' or 'fp8', got {activations!r}")
        mlps = [layer.mlp for layer in self.language_model.model.layers]
        if any(m.expert_parallel is not None for m in mlps):
            raise NotImplementedError("quantize_experts_fp8: expert parallelism is enabled; it runs on bf16 expert weights")
        todo, relayout = [], []
        for i, m in enumerate(mlps):
            if m.experts.is_fp8():
                if m.experts.fp8_activations() != (activations == "fp8"):
                    relayout.append(m.experts)
                continue
            for name in ("fc1", "fc2"):
                fc = getattr(m.experts, name)
                if type(fc) is not GroupedGEMM:
                    raise NotImplementedError(f"quantize_experts_fp8: layer {i} experts.{name} is a {type(fc).__name__} "
                                              "(e.g. LoRA-wrapped), not a plain GroupedGEMM")
                if not bool(torch.isfinite(fc.weight).all()):
                    raise ValueError(f"quantize_experts_fp8: layer {i} experts.{name}.weight has non-finite values")
            todo.append(m.experts)
        if not todo and not relayout:
            return self
        self._decode_graph = None
        for experts in todo:
            for name in ("fc1", "fc2"):
                fc = Fp8GroupedGEMM.from_grouped_gemm(getattr(experts, name))
                setattr(experts, name, fc)              # drops the bf16 module
                fc.set_activations(activations)         # re-laid out after the bf16 weights are gone: the same peak
        for experts in relayout:
            for name in ("fc1", "fc2"):
                getattr(experts, name).set_activations(activations)
        return self

    @property
    def device(self):
        return self.language_model.lm_head.weight.device

    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor = None, pixel_values: Optional[torch.Tensor] = None,
                pixel_mask: Optional[torch.Tensor] = None, attention_mask: Optional[torch.Tensor] = None,
                position_ids: Optional[torch.Tensor] = None, past_key_values: Optional[KVCache] = None,
                inputs_embeds: Optional[torch.Tensor] = None, labels: Optional[torch.Tensor] = None,
                use_cache: Optional[bool] = None, output_attentions: Optional[bool] = None,
                output_hidden_states: Optional[bool] = None, return_dict: Optional[bool] = None,
                cache_position: Optional[torch.Tensor] = None, num_logits_to_keep: int = 0,
                max_cache_len: Optional[int] = None, input_ids_host: Optional[torch.Tensor] = None,
                kv_cache_dtype: Optional[str] = None) -> AriaCausalLMOutputWithPast:
        """Same arguments as the reference forward (modeling_aria.py:194-210); `max_cache_len` / `input_ids_host` /
        `kv_cache_dtype` are ours.  `max_cache_len` and `kv_cache_dtype` ("bf16" or "fp8", default bf16) shape the KV cache
        forward() creates when no past_key_values is given; a kv_cache_dtype that disagrees with a given cache is a ValueError.

        input_ids / pixel_values / pixel_mask may be HOST tensors (pinned for async copies): they are copied to
        the device on the current stream; image-token bookkeeping is then done on the host copy (no device sync).
        Device-resident input_ids cost one sync for the image-token count check, like the reference's `.item()`
        (modeling_aria.py:265).

        attention_mask: the HF 2-D padding mask [B, past + T] (1 = real token).  Padded keys are masked inside the attention
        kernels (prefill and decode).  position_ids [B, T]: RoPE positions (default: cache positions, as in LlamaModel).
        labels: shifted cross-entropy exactly as modeling_aria.py:300-323 (the loss itself is torch glue on our logits;
        this class is the inference path, so it carries no grad_fn — training goes through aria_b200.moe_train / lora).
        Not supported, and rejected loudly: output_attentions / output_hidden_states (no such tensors exist in the fused
        path), return_dict=False."""
        if output_attentions or output_hidden_states:
            raise NotImplementedError("aria_b200: attention weights / per-layer hidden states are not materialised by the fused path")
        if kv_cache_dtype is not None:
            if kv_cache_dtype not in KV_CACHE_DTYPES:
                raise ValueError(f"kv_cache_dtype must be 'bf16' or 'fp8', got {kv_cache_dtype!r}")
            if past_key_values is not None and past_key_values.dtype != kv_cache_dtype:
                raise ValueError(f"kv_cache_dtype={kv_cache_dtype!r} disagrees with the given {past_key_values.dtype} past_key_values")
        if return_dict is False:
            raise NotImplementedError("aria_b200: tuple outputs are not supported (return_dict=False)")
        if cache_position is not None and past_key_values is not None and int(cache_position.reshape(-1)[0]) != past_key_values.seq_len:
            raise NotImplementedError("aria_b200: cache_position must continue the KV cache (static cache, append-only)")
        dev = self.device
        ids_host = input_ids_host  # optional host copy of device-resident ids (bookkeeping without a sync)
        if input_ids is not None and not input_ids.is_cuda:
            ids_host = input_ids
            input_ids = input_ids.to(dev, non_blocking=True)
        if pixel_values is not None and not pixel_values.is_cuda:
            pixel_values = pixel_values.to(dev, non_blocking=True)
        if inputs_embeds is None:
            inputs_embeds = ops.embedding(input_ids.contiguous(), self.get_input_embeddings().weight)
        elif pixel_values is not None:
            inputs_embeds = inputs_embeds.clone()   # the merge below writes in place; the reference's masked_scatter does not

        if pixel_values is not None:
            feats, image_attn_mask = self.vision_tower(pixel_values.to(bf16), pixel_mask)
            image_features = self.multi_modal_projector(feats, image_attn_mask)
            n_image_features = image_features.shape[0] * image_features.shape[1]
            src = ids_host if ids_host is not None else input_ids
            n_image_tokens = int((src == self.config.image_token_index).sum())
            if n_image_tokens != n_image_features:
                raise ValueError(  # modeling_aria.py:268-271
                    f"Image features and image tokens do not match: tokens: {n_image_tokens}, features {n_image_features}")
            ops.merge_image_features(input_ids.reshape(-1).contiguous(), self.config.image_token_index,
                                     image_features.reshape(-1, image_features.shape[-1]),
                                     inputs_embeds.view(-1, inputs_embeds.shape[-1]))

        B, T, _ = inputs_embeds.shape
        cache = past_key_values
        if cache is None:
            cache = self.language_model.new_cache(B, max_cache_len or T, dev, kv_cache_dtype or "bf16")
        key_mask = None
        if attention_mask is not None:
            if attention_mask.shape != (B, cache.seq_len + T):
                raise ValueError(f"attention_mask must be [B, past + T] = {(B, cache.seq_len + T)}, got {tuple(attention_mask.shape)}")
            if not bool((attention_mask != 0).all()):      # host tensor: free; device tensor: one sync, only when a mask is given
                key_mask = (attention_mask == 0).to(device=dev, dtype=torch.uint8).contiguous()
        pos = None
        if position_ids is not None:
            if position_ids.shape != (B, T):
                raise ValueError(f"position_ids must be [B, T] = {(B, T)}, got {tuple(position_ids.shape)}")
            pos = position_ids.to(device=dev, dtype=torch.int32).reshape(-1).contiguous()
        logits, cache = self.language_model(inputs_embeds, cache, num_logits_to_keep, key_mask=key_mask, position_ids=pos)
        out = AriaCausalLMOutputWithPast(logits, cache)
        if labels is not None:
            out.loss = self._shifted_cross_entropy(logits, labels, attention_mask)
        return out

    @staticmethod
    def _shifted_cross_entropy(logits, labels, attention_mask):
        """modeling_aria.py:300-323, verbatim semantics: tokens < n predict n; padded positions dropped through the 2-D mask."""
        labels = labels.to(logits.device)
        if attention_mask is not None:
            shift_mask = attention_mask[:, -(logits.shape[1] - 1):].to(logits.device)
            shift_logits = logits[..., :-1, :][shift_mask != 0].contiguous()
            shift_labels = labels[..., 1:][shift_mask != 0].contiguous()
        else:
            shift_logits = logits[..., :-1, :].contiguous()
            shift_labels = labels[..., 1:].contiguous()
        return nn.functional.cross_entropy(shift_logits.view(-1, shift_logits.size(-1)).float(), shift_labels.view(-1))

    def prepare_inputs_for_generation(self, input_ids, past_key_values=None, inputs_embeds=None, pixel_values=None,
                                      pixel_mask=None, attention_mask=None, cache_position=None, num_logits_to_keep=None,
                                      **kwargs):
        """modeling_aria.py:337-365: with a non-empty cache only the new token ids go in; pixel inputs only at step 0;
        position ids from the padding mask (what LlamaForCausalLM.prepare_inputs_for_generation derives)."""
        past = 0 if past_key_values is None else past_key_values.seq_len
        model_inputs = {"input_ids": input_ids[:, past:] if past else input_ids, "past_key_values": past_key_values,
                        "attention_mask": attention_mask}
        if inputs_embeds is not None and not past:
            model_inputs = {"inputs_embeds": inputs_embeds, "input_ids": input_ids, "past_key_values": past_key_values,
                            "attention_mask": attention_mask}
        if attention_mask is not None:
            pos = (attention_mask.long().cumsum(-1) - 1).clamp_min(0)
            model_inputs["position_ids"] = pos[:, past:] if past else pos
        if num_logits_to_keep is not None:
            model_inputs["num_logits_to_keep"] = num_logits_to_keep
        if not past:
            model_inputs["pixel_values"] = pixel_values
            model_inputs["pixel_mask"] = pixel_mask
        return model_inputs

    @torch.no_grad()
    def generate(self, input_ids, pixel_values=None, pixel_mask=None, max_new_tokens: int = 16, attention_mask=None, *,
                 do_sample: bool = False, temperature: float = 1.0, top_k: int = 50, top_p: float = 1.0, eos_token_id=None,
                 pad_token_id=None, seed: int = 0, poll_every: int = 8, kv_cache_dtype: str = "bf16",
                 num_return_sequences: int = 1, shared_prefix_len: Optional[int] = None,
                 prompt_lookup_num_tokens: Optional[int] = None, max_matching_ngram_size: Optional[int] = None):
        """Greedy or sampled generation (the reference goes through HF GenerationMixin, modeling_aria.py:125,337-365).

        Eager prefill with the image, the first token sampled from its logits, then one CUDA-graph replay per token of a
        captured decode step (GraphedDecode: embedding -> layers -> norm -> lm_head -> sample -> advance), all positions on the
        device.  attention_mask [B, T]: LEFT-padded batches of ragged prompts (the HF generation convention); positions are
        derived from it as GenerationMixin does.
        do_sample=False: argmax (ties to the lowest id).  do_sample=True: transformers' TemperatureLogitsWarper ->
        TopKLogitsWarper (top_k <= 1024, 0 = off) -> TopPLogitsWarper -> softmax -> multinomial, drawn with Philox noise keyed
        by `seed` (reproducible; not torch's generator stream).  top_k = 0 with top_p < 1 is not supported.
        eos_token_id: an id or up to 8 ids; a row that emits one is finished and emits pad_token_id (default: the first EOS
        id) from then on, and generation stops once every row is finished, trimmed as GenerationMixin trims it.  The host
        looks at the finished flag every `poll_every` tokens; the result does not depend on it.
        kv_cache_dtype: "bf16", or "fp8" for e4m3 keys and values with one scale per (row, head, token) (KVCache): the prefill
        still attends in bf16, every decode step reads the fp8 cache.  GPU only.
        num_return_sequences n > 1 (sampling only, bf16 cache, B * n <= 1024): n continuations of every prompt.  Each prompt goes
        through the ViT and the prefill once; its n rows then decode against that one prompt cache (SharedPrefixCache), each
        with its own tail of generated tokens and its own sampling noise (the Philox counter is keyed by row).  Rows are grouped
        as GenerationMixin groups them: prompt b's rows are b*n .. b*n + n - 1, and its ids are repeated for each of them.
        shared_prefix_len P (bf16 cache, B * n <= 1024): many questions about one image.  The first P real tokens of every row
        (after its left padding) are one shared prefix that holds every image token, and pixel_values / pixel_mask are that
        prefix's images, once.  The ViT and the prefix prefill run once; each row's own tokens (its suffix) are prefilled
        against the prefix cache, packed, and all B * n rows decode against that one prefix cache, each with its own tail.
        Positions are those GenerationMixin derives from the left-padded mask, and the result is laid out as without it.  One
        captured step serves every call whose prefix and longest question + max_new_tokens fall in the same 256-row buckets.
        prompt_lookup_num_tokens K (1..15) / max_matching_ngram_size M (1..16, default 2): prompt-lookup decoding, Hugging Face's
        names.  Every row drafts up to K tokens by matching its last n <= M tokens against its own prompt and output
        (PromptLookupCandidateGenerator), and one step verifies the row's next token and its drafts (GraphedLookupDecode).  The
        result is the one generate() gives without these arguments, bit for bit, greedy or sampled: each verified position gets
        the logits and the sampling noise of the plain step that would emit that token.  Not combined with
        num_return_sequences > 1, shared_prefix_len or the fp8 KV cache; B * (K + 1) <= 1024; GPU only.  The host waits for every
        step (poll_every does not apply); the call's counters are in self.prompt_lookup_stats.
        Returns [B * n, T + generated] int64 on the model's device (prompt ids first)."""
        B, T, eos, pad = self._check_generate_args(input_ids, max_new_tokens, attention_mask, do_sample, temperature, top_k,
                                                   top_p, eos_token_id, pad_token_id, seed, poll_every, kv_cache_dtype,
                                                   num_return_sequences, shared_prefix_len)
        n_seq = num_return_sequences
        dev = self.device
        if prompt_lookup_num_tokens is not None:
            K, M = self._check_prompt_lookup(B, prompt_lookup_num_tokens, max_matching_ngram_size, n_seq, shared_prefix_len,
                                             kv_cache_dtype, dev)
            sampling = (float(temperature), int(top_k), float(top_p), int(seed)) if do_sample else (0.0, 0, 1.0, 0)
            return self._generate_prompt_lookup(input_ids, pixel_values, pixel_mask, max_new_tokens, attention_mask, sampling, eos,
                                                pad, K, M)
        if shared_prefix_len is not None:
            ids_host, lens = self._check_shared_prefix(input_ids, attention_mask, shared_prefix_len, self.config.image_token_index,
                                                       kv_cache_dtype, n_seq)
            if dev.type != "cuda":
                raise NotImplementedError("aria_b200: shared_prefix_len runs on the GPU only")
            sampling = (float(temperature), int(top_k), float(top_p), int(seed)) if do_sample else (0.0, 0, 1.0, 0)
            return self._generate_shared_prefix(input_ids, ids_host, lens, pixel_values, pixel_mask, max_new_tokens, sampling, eos,
                                                pad, poll_every, n_seq, shared_prefix_len)
        if dev.type != "cuda":
            if do_sample or eos:
                raise NotImplementedError("aria_b200: sampling and EOS run on the GPU only")
            if kv_cache_dtype == "fp8":
                raise NotImplementedError("aria_b200: the fp8 KV cache runs on the GPU only")
            return self._generate_stepwise(input_ids, pixel_values, pixel_mask, max_new_tokens, attention_mask)
        if do_sample:
            sampling = (float(temperature), int(top_k), float(top_p), int(seed))
        else:
            sampling = (0.0, 0, 1.0, 0)
        # rows are device-driven, so one captured step serves every prompt length of the same 256-row bucket; with
        # n_seq > 1 the cache holds the prompts only (their bucket) and the generated tokens go to the tails
        T_max = -(-(T if n_seq > 1 else T + max_new_tokens) // 256) * 256
        key = (B, T_max, max_new_tokens, sampling, eos, pad, dev, n_seq, None, kv_cache_dtype)
        g = getattr(self, "_decode_graph", None)
        if g is None or g.key != key:
            self._decode_graph = g = None   # release the old graph and cache before building the new one
            g = self._decode_graph = GraphedDecode(self, B, T_max, max_new_tokens, sampling, eos, pad, kv_cache_dtype, n_seq)
        mask = None if attention_mask is None else attention_mask.to("cpu", torch.long)
        inputs = self.prepare_inputs_for_generation(input_ids, None, pixel_values=pixel_values, pixel_mask=pixel_mask,
                                                    attention_mask=mask, num_logits_to_keep=1)
        g.cache.seq_len = 0
        inputs["past_key_values"] = g.cache
        out = self.forward(**inputs)
        g.start(T, mask)
        first = out.logits[:, -1]
        g.sample_and_advance(first if n_seq == 1 else first.repeat_interleave(n_seq, 0))
        n, L = g.run(max_new_tokens, poll_every)
        if n_seq == 1:
            g.cache.seq_len = T + n             # a shared cache keeps the prompt's T; the tails hold the rest
        prompt = input_ids if n_seq == 1 else input_ids.repeat_interleave(n_seq, 0)
        return torch.cat([prompt.to(dev), g.out_tokens[:, :L]], dim=1)

    def _generate_shared_prefix(self, input_ids, ids, lens, pixel_values, pixel_mask, max_new_tokens, sampling, eos, pad,
                                poll_every, n_seq, P):
        """generate(shared_prefix_len=P) on checked arguments (ids: the host copy of input_ids, lens: each row's real length,
        from _check_shared_prefix): ViT + prefix prefill (forward()) into a SharedPrefixCache of one prompt row, the packed
        suffix prefill (AriaMoELMModel.prefill_suffixes), the first token from each suffix's last position, then the graphed
        decode of the B * n rows, one group."""
        dev = self.device
        lm = self.language_model
        B, T = input_ids.shape
        S = (lens - P).tolist()                      # suffix lengths, >= 1 each (checked)
        start = (T - lens).tolist()                  # first real token of each row
        prefix = ids[:1, start[0]:start[0] + P]
        suffix = torch.cat([ids[b, start[b] + P:] for b in range(B)])[None]
        cu = torch.tensor([0] + torch.tensor(S).cumsum(0).tolist(), dtype=torch.int32)
        pos = torch.cat([torch.arange(P, P + s, dtype=torch.int32) for s in S])   # GenerationMixin's cumsum(mask) - 1
        # the prefix and the tails are bucketed like generate()'s cache: every length in the step is a device value
        T_max = -(-P // 256) * 256
        N_max = -(-(max(S) + max_new_tokens) // 256) * 256
        key = (1, T_max, max_new_tokens, sampling, eos, pad, dev, B * n_seq, N_max, "bf16")
        g = getattr(self, "_decode_graph", None)
        if g is None or g.key != key:
            self._decode_graph = g = None
            g = self._decode_graph = GraphedDecode(self, 1, T_max, max_new_tokens, sampling, eos, pad, "bf16", B * n_seq,
                                                   N_max=N_max)
        g.cache.seq_len = 0
        self.forward(prefix, pixel_values, pixel_mask, past_key_values=g.cache, num_logits_to_keep=1)
        cu_dev = cu.to(dev, non_blocking=True)
        emb = ops.embedding(suffix.to(dev, non_blocking=True), lm.get_input_embeddings().weight)
        x, pending = lm.model.prefill_suffixes(emb, g.cache, cu_dev, pos.to(dev, non_blocking=True))
        last = (cu[1:] - 1).to(dev, torch.int64, non_blocking=True)
        h, _ = lm.model.norm(x[0, last].contiguous(), residual=pending[0, last].contiguous())
        first = lm.lm_head(h)                       # [B, V]
        g.start_suffixes(P, S, n_seq)
        g.sample_and_advance(first if n_seq == 1 else first.repeat_interleave(n_seq, 0))
        _, L = g.run(max_new_tokens, poll_every)
        prompt = input_ids if n_seq == 1 else input_ids.repeat_interleave(n_seq, 0)
        return torch.cat([prompt.to(dev), g.out_tokens[:, :L]], dim=1)

    def _generate_prompt_lookup(self, input_ids, pixel_values, pixel_mask, max_new_tokens, attention_mask, sampling, eos, pad,
                                K, M):
        """generate(prompt_lookup_num_tokens=K) on checked arguments: the eager prefill of generate(), the first token and the first
        drafts eagerly, then GraphedLookupDecode.run().  The cache bucket also holds the K rows a verify step writes past a row's
        last token, so no row of a step falls past it; the decode kernels never merge a split past a row's key count, so a larger
        bucket changes no arithmetic.  Nothing in the graph depends on T itself (the history is T_max long too), so one captured
        pair of steps serves every prompt length of the same bucket."""
        dev = self.device
        B, T = input_ids.shape
        T_max = -(-(T + max_new_tokens + K) // 256) * 256
        key = ("lookup", B, T_max, max_new_tokens, sampling, eos, pad, dev, K, M)
        g = getattr(self, "_decode_graph", None)
        if g is None or g.key != key:
            self._decode_graph = g = None
            g = self._decode_graph = GraphedLookupDecode(self, B, T_max, max_new_tokens, sampling, eos, pad, K, M)
        mask = None if attention_mask is None else attention_mask.to("cpu", torch.long)
        inputs = self.prepare_inputs_for_generation(input_ids, None, pixel_values=pixel_values, pixel_mask=pixel_mask,
                                                    attention_mask=mask, num_logits_to_keep=1)
        g.cache.seq_len = 0
        inputs["past_key_values"] = g.cache
        out = self.forward(**inputs)
        g.start(input_ids.to("cpu"), mask)
        g.first(out.logits[:, -1])
        L = g.run()
        self.prompt_lookup_stats = g.stats
        return torch.cat([input_ids.to(dev), g.out_tokens[:, :L]], dim=1)

    def _generate_stepwise(self, input_ids, pixel_values, pixel_mask, max_new_tokens, attention_mask):
        """Greedy decoding through the public step API, one forward(past_key_values=...) per token: what generate() does
        on a device without CUDA graphs, i.e. the torch stand-ins of `ops` that the host-logic tests swap in."""
        B, T = input_ids.shape
        mask = None if attention_mask is None else attention_mask.to("cpu", torch.long)
        inputs = self.prepare_inputs_for_generation(input_ids, None, pixel_values=pixel_values, pixel_mask=pixel_mask,
                                                    attention_mask=mask, num_logits_to_keep=1)
        out = self.forward(**inputs, max_cache_len=T + max_new_tokens)
        cache = out.past_key_values
        tokens = [out.logits[:, -1].float().argmax(-1)]
        all_ids = input_ids.to(tokens[0].device)
        for _ in range(max_new_tokens - 1):
            all_ids = torch.cat([all_ids, tokens[-1].view(B, 1)], dim=1)
            if mask is not None:
                mask = torch.cat([mask, torch.ones(B, 1, dtype=torch.long)], dim=1)
            inputs = self.prepare_inputs_for_generation(all_ids, cache, attention_mask=mask, num_logits_to_keep=1)
            tokens.append(self.forward(**inputs).logits[:, -1].float().argmax(-1))
        return torch.cat([input_ids.to(tokens[0].device), torch.stack(tokens, 1)], dim=1)

    @staticmethod
    def _check_generate_args(input_ids, max_new_tokens, attention_mask, do_sample, temperature, top_k, top_p, eos_token_id,
                             pad_token_id, seed, poll_every, kv_cache_dtype="bf16", num_return_sequences=1, shared_prefix_len=None):
        """All of generate()'s argument checks, on the host, before any device work -> (B, T, eos ids tuple, pad id).  With a
        shared_prefix_len the row limit is left to _check_shared_prefix, which generate() runs next: it comes last there."""
        import math
        if input_ids.dim() != 2 or input_ids.shape[0] < 1 or input_ids.shape[1] < 1:
            raise ValueError(f"input_ids must be [B, T] with B, T >= 1, got {tuple(input_ids.shape)}")
        B, T = input_ids.shape
        rows_checked_here = shared_prefix_len is None
        if rows_checked_here and B > 1024:
            raise NotImplementedError("generate(): at most 1024 rows per batch")
        n = num_return_sequences
        if not isinstance(n, int) or isinstance(n, bool) or n < 1:
            raise ValueError(f"num_return_sequences must be a positive int, got {n!r}")
        if rows_checked_here and B * n > 1024:
            raise NotImplementedError(f"generate(): at most 1024 rows per batch, got {B} prompts x {n} sequences")
        if not isinstance(max_new_tokens, int) or max_new_tokens < 1:
            raise ValueError(f"max_new_tokens must be a positive int, got {max_new_tokens!r}")
        if attention_mask is not None and tuple(attention_mask.shape) != (B, T):
            raise ValueError(f"attention_mask must be [B, T] = {(B, T)}, got {tuple(attention_mask.shape)}")
        if not isinstance(poll_every, int) or poll_every < 1:
            raise ValueError(f"poll_every must be a positive int, got {poll_every!r}")
        if not isinstance(seed, int) or not 0 <= seed < 2 ** 64:
            raise ValueError(f"seed must be an int in [0, 2**64), got {seed!r}")
        if kv_cache_dtype not in KV_CACHE_DTYPES:
            raise ValueError(f"kv_cache_dtype must be 'bf16' or 'fp8', got {kv_cache_dtype!r}")
        if n > 1 and not do_sample:
            raise ValueError("num_return_sequences > 1 needs do_sample=True: greedy rows of one prompt would all be equal")
        if n > 1 and kv_cache_dtype == "fp8":
            raise NotImplementedError("num_return_sequences > 1 shares a bf16 prompt cache; the fp8 KV cache is not supported")
        if do_sample:
            if not (isinstance(temperature, (int, float)) and math.isfinite(temperature) and temperature > 0):
                raise ValueError(f"temperature must be a strictly positive float, got {temperature!r}")
            if not isinstance(top_k, int) or top_k < 0:
                raise ValueError(f"top_k must be a non-negative int, got {top_k!r}")
            if top_k > 1024:
                raise NotImplementedError("top_k > 1024 is not supported by the sampling kernel")
            if not (isinstance(top_p, (int, float)) and 0 < top_p <= 1):
                raise ValueError(f"top_p must be a float in (0, 1], got {top_p!r}")
            if top_k == 0 and top_p < 1:
                raise NotImplementedError("top-p without top-k (a full-vocabulary nucleus) is not supported")
        eos = () if eos_token_id is None else (eos_token_id,) if isinstance(eos_token_id, int) else tuple(eos_token_id)
        if len(eos) > 8 or not all(isinstance(e, int) for e in eos):
            raise ValueError(f"eos_token_id must be an int or at most 8 ints, got {eos_token_id!r}")
        if pad_token_id is None:
            pad_token_id = eos[0] if eos else 0
        if not isinstance(pad_token_id, int):
            raise ValueError(f"pad_token_id must be an int, got {pad_token_id!r}")
        return B, T, eos, pad_token_id

    @staticmethod
    def _check_prompt_lookup(B, K, M, n, shared_prefix_len, kv_cache_dtype, device):
        """generate(prompt_lookup_num_tokens=K, max_matching_ngram_size=M)'s checks after _check_generate_args', in this order:
        K, M (ValueError), then num_return_sequences > 1, shared_prefix_len, the fp8 KV cache, a CPU device and B * (K + 1) > 1024
        (NotImplementedError).  -> (K, M), M defaulting to 2 as in Hugging Face."""
        if not isinstance(K, int) or isinstance(K, bool) or not 1 <= K <= 15:
            raise ValueError(f"prompt_lookup_num_tokens must be an int in [1, 15], got {K!r}")
        M = 2 if M is None else M
        if not isinstance(M, int) or isinstance(M, bool) or not 1 <= M <= 16:
            raise ValueError(f"max_matching_ngram_size must be an int in [1, 16], got {M!r}")
        if n > 1:
            raise NotImplementedError("prompt_lookup_num_tokens with num_return_sequences > 1 is not supported")
        if shared_prefix_len is not None:
            raise NotImplementedError("prompt_lookup_num_tokens with shared_prefix_len is not supported")
        if kv_cache_dtype == "fp8":
            raise NotImplementedError("prompt_lookup_num_tokens verifies against a bf16 KV cache; the fp8 KV cache is not supported")
        if torch.device(device).type != "cuda":
            raise NotImplementedError("aria_b200: prompt_lookup_num_tokens runs on the GPU only")
        if B * (K + 1) > 1024:
            raise NotImplementedError(f"generate(): at most 1024 rows per verify step, got {B} rows x {K + 1} tokens")
        return K, M

    @staticmethod
    def _check_shared_prefix(input_ids, attention_mask, P, image_token_index, kv_cache_dtype, n=1):
        """generate(shared_prefix_len=P)'s checks after _check_generate_args', in this order: P, the mask, the row lengths, the
        prefixes, the image tokens (ValueError), the fp8 cache, B * n <= 1024 (NotImplementedError).  One host copy of the ids
        and of the mask -> (host ids [B, T], the real length of every row, host int64 [B])."""
        if not isinstance(P, int) or isinstance(P, bool) or P < 1:
            raise ValueError(f"shared_prefix_len must be a positive int, got {P!r}")
        B, T = input_ids.shape
        if attention_mask is None:
            lens = torch.full((B,), T, dtype=torch.int64)
        else:
            m = attention_mask.to("cpu", torch.int64)
            if not bool(((m == 0) | (m == 1)).all()) or not bool((m[:, 1:] >= m[:, :-1]).all()):
                raise ValueError("shared_prefix_len needs a left-padded attention_mask (zeros, then ones, in every row)")
            lens = m.sum(-1)
        short = (lens <= P).nonzero()
        if short.numel():
            b = int(short[0])
            raise ValueError(f"shared_prefix_len={P}: row {b} has {int(lens[b])} real tokens; every row needs the prefix and at "
                             "least one token of its own")
        ids = input_ids.to("cpu")
        rows = [ids[b, T - int(lens[b]):] for b in range(B)]
        for b in range(1, B):
            if not torch.equal(rows[b][:P], rows[0][:P]):
                raise ValueError(f"shared_prefix_len={P}: the first {P} real tokens of row {b} differ from those of row 0")
        for b in range(B):
            if bool((rows[b][P:] == image_token_index).any()):
                raise ValueError(f"shared_prefix_len={P}: row {b} has an image token after the shared prefix; every image "
                                 "token must be in the prefix")
        if kv_cache_dtype == "fp8":
            raise NotImplementedError("shared_prefix_len shares a bf16 prefix cache; the fp8 KV cache is not supported")
        if B * n > 1024:
            raise NotImplementedError(f"generate(): at most 1024 rows per batch, got {B} questions x {n} sequences")
        return ids, lens


class GraphedDecode:
    """One decode step captured as a CUDA graph and replayed token after token (AriaForConditionalGeneration.generate).

    The step is embedding -> every layer (AriaMoELMForCausalLM.decode_step) -> norm -> lm_head -> sample_tokens ->
    decode_advance.  Nothing in it is a host integer: the step's input ids, RoPE positions, cache rows and key counts
    (`state`), the RNG offset, the finished flags, the step index and the output tokens all live in static device buffers,
    and decode_advance moves them on at the end of every replay.  The KV cache belongs to the graph: generate() prefills
    into it with forward(past_key_values=g.cache), then calls start() and sample_and_advance() for the first token.
    `logits` is the last replayed step's logits [B, 1, V].
    group_size n > 1: B prompts decoded n times each.  The cache is a SharedPrefixCache of B prompt rows of T_max (the prompt
    bucket) and B * n tails of max_new_tokens rounded up to 256; the state, tokens and logits have B * n rows.
    N_max (generate(shared_prefix_len=...)): a SharedPrefixCache whose tails hold N_max rows (a multiple of 256), each row's
    own prompt tokens and then its generated ones, for any group size."""

    def __init__(self, model: "AriaForConditionalGeneration", B: int, T_max: int, max_new_tokens: int, sampling, eos, pad,
                 kv_cache_dtype: str = "bf16", group_size: int = 1, N_max: Optional[int] = None):
        from .moe_lm import DecodeState, SharedDecodeState, SharedPrefixCache
        dev = model.device
        lm = model.language_model
        c = lm.config
        self.key = (B, T_max, max_new_tokens, sampling, eos, pad, dev, group_size, N_max, kv_cache_dtype)
        self.group_size = group_size
        self.T_max = T_max
        self.sampling, self.eos, self.pad = sampling, eos, pad
        if group_size == 1 and N_max is None:
            self.cache = lm.new_cache(B, T_max, dev, kv_cache_dtype)
            self.state = DecodeState(B, c.num_attention_heads, T_max, dev)
            n_pos = T_max
        else:
            if N_max is None:
                N_max = -(-max_new_tokens // 256) * 256
            self.cache = SharedPrefixCache(c.num_hidden_layers, B, group_size, c.num_attention_heads, T_max, N_max, c.head_dim, dev)
            self.state = SharedDecodeState(B, group_size, c.num_attention_heads, T_max, dev)
            n_pos = T_max + N_max
            B = B * group_size
        self.model, self.B = model, B
        self.rope = lm.model.rope_tables(n_pos, dev)   # held here: the graph reads these tables
        self.ids = torch.zeros(B, 1, dtype=torch.int64, device=dev)
        self.next_ids = torch.zeros(B, dtype=torch.int64, device=dev)
        self.rng_offset = torch.zeros(1, dtype=torch.int64, device=dev)   # read as uint64 by the kernels
        self.step = torch.zeros(1, dtype=torch.int32, device=dev)
        self.done_step = torch.full((1,), -1, dtype=torch.int32, device=dev)
        self.finished = torch.zeros(B, dtype=torch.uint8, device=dev)
        self.out_tokens = torch.zeros(B, max_new_tokens, dtype=torch.int64, device=dev)
        self.done_host = torch.full((1,), -1, dtype=torch.int32).pin_memory()
        self.event = torch.cuda.Event()
        self.dev = dev
        cur = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):               # warm-up (its cache rows and state are reset by start())
            self._step()
        cur.wait_stream(side)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.logits = self._step()

    def _step(self):
        lm = self.model.language_model
        emb = ops.embedding(self.ids, lm.get_input_embeddings().weight)
        logits = lm.decode_step(emb, self.cache, self.state, self.rope)
        self.sample_and_advance(logits[:, -1])
        return logits

    def sample_and_advance(self, logits: torch.Tensor):
        """Sample from logits [B, V] into next_ids, then advance the state (also the eager first token after the prefill)."""
        t, k, p, seed = self.sampling
        ops.sample_tokens(logits, t, k, p, seed, self.rng_offset, out=self.next_ids)
        st = self.state
        ops.decode_advance(self.next_ids, self.ids, self.out_tokens, self.step, st.rope_pos, st.write_pos, st.kv_len,
                           self.rng_offset, self.finished, self.done_step, self.eos, self.pad)
        self.done_host.copy_(self.done_step, non_blocking=True)

    def start(self, T: int, mask: Optional[torch.Tensor]):
        """Reset the state for a prompt of T tokens (mask: host [B, T] padding mask or None) already prefilled into
        self.cache.  The values are those of the last prompt token: the advance after the first sample moves them on."""
        B = self.B // self.group_size      # prompts
        if mask is None:
            last = torch.full((B,), T - 1, dtype=torch.int32)
        else:
            last = (mask.sum(-1) - 1).to(torch.int32)
        km = torch.zeros(B, self.T_max, dtype=torch.uint8)
        if mask is not None:
            km[:, :T] = (mask == 0).to(torch.uint8)
        st = self.state
        if self.group_size == 1:
            st.rope_pos.copy_(last)
            st.write_pos.fill_(T - 1)
            st.kv_len.fill_(T)
            st.key_mask.copy_(km)
        else:
            # every row of a prompt continues from its last position; its tail is empty until the first advance
            st.rope_pos.copy_(last.repeat_interleave(self.group_size))
            st.write_pos.fill_(-1)
            st.kv_len.fill_(0)
            st.prefix_lens.fill_(T)
            st.prefix_mask.copy_(km)
        self._reset()

    def start_suffixes(self, P: int, suffix_lens, n: int):
        """Reset the state for one prefix of P tokens and B suffixes of suffix_lens (host ints) already prefilled: the prefix
        into the cache's prompt row, the suffixes into the tails of their n rows each (AriaMoELMModel.prefill_suffixes).
        Row b * n + j continues from its last suffix token at position P + S_b - 1, tail row S_b - 1."""
        S = torch.tensor(suffix_lens, dtype=torch.int32).repeat_interleave(n)
        st = self.state
        st.rope_pos.copy_(S + (P - 1))
        st.write_pos.copy_(S - 1)
        st.kv_len.copy_(S)
        st.prefix_lens.fill_(P)
        st.prefix_mask.zero_()
        self._reset()

    def _reset(self):
        self.rng_offset.zero_()
        self.step.zero_()
        self.done_step.fill_(-1)
        self.finished.zero_()
        self.done_host.fill_(-1)

    def run(self, max_new_tokens: int, poll_every: int):
        """Replay the step until max_new_tokens tokens are out (the first one is sampled before) or, with EOS ids, every row has
        finished; the host polls every poll_every steps.  -> (steps replayed, tokens to keep per row)."""
        n = 0
        while n < max_new_tokens - 1:
            if self.eos and n % poll_every == 0 and self.done():
                break
            self.graph.replay()
            n += 1
        done = int(self.done_step.item())       # synchronises; -1 when no EOS stopped the batch
        return n, (done + 1 if done >= 0 else max_new_tokens)

    def done(self) -> bool:
        """Whether every row has finished, from the pinned copy of done_step (waits for the work queued so far)."""
        self.event.record(torch.cuda.current_stream(self.dev))
        self.event.synchronize()
        return int(self.done_host[0]) >= 0


class GraphedLookupDecode:
    """Prompt-lookup decoding (generate(prompt_lookup_num_tokens=K)) as two captured steps over one KV cache and one
    LookupDecodeState, replayed until every row is done:

    - the K-wide step: embedding of [B, K + 1] ids (each row's last token, then its drafts) -> every layer
      (AriaMoELMForCausalLM.verify_step) -> norm -> lm_head -> sample_tokens_rows -> lookup_accept_advance -> ngram_draft;
    - the 1-wide step: the same with decode_step on [B, 1], for steps where no row has a draft.

    Logits row b * (K + 1) + i draws the Philox noise of generation row b at offset n_out[b] + i, the counter plain generate()
    uses for that row's token n_out[b] + i.  lookup_accept_advance emits each row's accepted drafts plus one token, stops a row
    after its first EOS or at max_new_tokens and moves its positions on by the count emitted; rows past their end emit nothing,
    and out_tokens is pad-filled at start().  After each replay the host reads the pinned status (every row done; any row has a
    draft) and replays the K-wide step only when some row has a draft: one event wait per step.  `stats`: the last call's steps
    replayed, K-wide steps, drafted and accepted tokens and tokens emitted."""

    def __init__(self, model: "AriaForConditionalGeneration", B: int, T_max: int, max_new_tokens: int, sampling, eos, pad, K: int,
                 M: int):
        from .moe_lm import LookupDecodeState
        dev = model.device
        lm = model.language_model
        c = lm.config
        self.key = ("lookup", B, T_max, max_new_tokens, sampling, eos, pad, dev, K, M)
        self.model, self.B, self.T_max, self.K, self.M = model, B, T_max, K, M
        self.max_new = max_new_tokens
        self.sampling, self.eos, self.pad = sampling, eos, pad
        self.cache = lm.new_cache(B, T_max, dev)
        self.state = LookupDecodeState(B, c.num_attention_heads, T_max, K, dev)
        self.rope = lm.model.rope_tables(T_max, dev)
        i64, i32 = dict(dtype=torch.int64, device=dev), dict(dtype=torch.int32, device=dev)
        Q = K + 1
        self.ids1 = torch.zeros(B, 1, **i64)
        self.idsk = torch.zeros(B, Q, **i64)
        self.targets1 = torch.zeros(B, **i64)
        self.targetsk = torch.zeros(B * Q, **i64)
        self.noise1 = torch.arange(B, **i32)
        self.noisek = torch.arange(B, **i32).repeat_interleave(Q)
        self.off1 = torch.zeros(B, **i64)
        self.offk = torch.zeros(B * Q, **i64)
        self.draft_len = torch.zeros(B, **i32)
        self.out_tokens = torch.zeros(B, max_new_tokens, **i64)
        # a row's history (prompt + output) fits in its cache rows: sized by the bucket, so every prompt length of it is served
        self.hist = torch.zeros(B, T_max, **i64)
        self.hist_len = torch.zeros(B, **i32)
        self.n_out = torch.zeros(B, **i32)
        self.finished = torch.zeros(B, dtype=torch.uint8, device=dev)
        self.status = torch.zeros(2, **i32)
        self.counters = torch.zeros(2, **i64)
        self.status_host = torch.zeros(2, dtype=torch.int32).pin_memory()
        self.event = torch.cuda.Event()
        self.dev = dev
        self.stats = None
        cur = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):               # warm-up (start() resets the cache rows and state it touched)
            self._step_k()
            self._step_1()
        cur.wait_stream(side)
        self.graph_k = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph_k):
            self._step_k()
        self.graph_1 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph_1):
            self._step_1()

    def _sample(self, logits, noise, offsets, out):
        t, k, p, seed = self.sampling
        ops.sample_tokens_rows(logits, t, k, p, seed, noise, offsets, out=out)

    def _step_k(self):
        lm = self.model.language_model
        emb = ops.embedding(self.idsk, lm.get_input_embeddings().weight)
        logits = lm.verify_step(emb, self.cache, self.state, self.rope)
        self._sample(logits.view(-1, logits.shape[-1]), self.noisek, self.offk, self.targetsk)
        self._advance(self.targetsk, self.idsk)

    def _step_1(self):
        lm = self.model.language_model
        emb = ops.embedding(self.ids1, lm.get_input_embeddings().weight)
        logits = lm.decode_step(emb, self.cache, self.state, self.rope)
        self._sample(logits[:, -1], self.noise1, self.off1, self.targets1)
        self._advance(self.targets1, self.ids1)

    def _advance(self, targets, step_ids):
        st = self.state
        ops.lookup_accept_advance(targets, step_ids, self.draft_len, self.ids1, self.idsk, st.pos_k, st.lens_k, self.off1,
                                  self.offk, self.out_tokens, self.hist, self.hist_len, self.n_out, self.finished, st.rope_pos,
                                  st.write_pos, st.kv_len, self.status, self.counters, self.eos)
        ops.ngram_draft(self.hist, self.hist_len, self.finished, self.n_out, self.max_new, self.idsk[:, 1:], self.draft_len,
                        self.status[1:], self.K, self.M, self.eos)
        self.status_host.copy_(self.status, non_blocking=True)

    def start(self, ids: torch.Tensor, mask: Optional[torch.Tensor]):
        """Reset the state for host prompt ids [B, T] (mask: host [B, T] left-padding mask or None) already prefilled into
        self.cache: positions of each row's last prompt token, the key mask, and the history = each row's real tokens."""
        B, T = ids.shape
        lens = torch.full((B,), T, dtype=torch.int64) if mask is None else mask.sum(-1)
        hist = torch.zeros(B, self.hist.shape[1], dtype=torch.int64)
        for b in range(B):
            n = int(lens[b])
            hist[b, :n] = ids[b, T - n:]
        km = torch.zeros(B, self.T_max, dtype=torch.uint8)
        if mask is not None:
            km[:, :T] = (mask == 0).to(torch.uint8)
        st = self.state
        st.rope_pos.copy_((lens - 1).to(torch.int32))
        st.write_pos.fill_(T - 1)
        st.kv_len.fill_(T)
        st.key_mask.copy_(km)
        self.hist.copy_(hist)
        self.hist_len.copy_(lens.to(torch.int32))
        self.n_out.zero_()
        self.finished.zero_()
        self.off1.zero_()
        self.draft_len.zero_()
        self.out_tokens.fill_(self.pad)
        self.status.zero_()
        self.counters.zero_()

    def first(self, logits: torch.Tensor):
        """The first token from the prefill's last-position logits [B, V], and the first drafts (eager)."""
        self._sample(logits, self.noise1, self.off1, self.targets1)
        self._advance(self.targets1, self.ids1)

    def run(self) -> int:
        """Replay until every row is finished or has max_new_tokens tokens -> the number of tokens to keep per row: the longest
        row when every row ended with EOS (GenerationMixin stops after that step), else max_new_tokens."""
        steps = k_steps = 0
        while True:
            self.event.record(torch.cuda.current_stream(self.dev))
            self.event.synchronize()
            done, drafted = int(self.status_host[0]), int(self.status_host[1])
            if done:
                break
            if drafted:
                self.graph_k.replay()
                k_steps += 1
            else:
                self.graph_1.replay()
            steps += 1
        n_out = self.n_out.cpu()
        counters = self.counters.cpu()
        L = int(n_out.max()) if self.eos and bool(self.finished.cpu().all()) else self.max_new
        self.stats = {"steps": steps, "k_steps": k_steps, "drafted": int(counters[0]), "accepted": int(counters[1]),
                      "tokens": int(n_out.sum())}
        return L


class GraphedPrefill:
    """CUDA-graph capture of one prefill `forward()` for fixed shapes (streams + graphs instead of a tracing
    compiler): the whole ViT -> projector -> merge -> LM chain has no host sync, so it is captured once and replayed.

        g = GraphedPrefill(model, input_ids_host, pixel_values_host)      # warm-up + capture
        logits = g(input_ids_host, pixel_values_host)                      # H2D copies + replay; logits on device
        logits = g.replay()                                                # inputs already resident in HBM
    """

    def __init__(self, model: "AriaForConditionalGeneration", input_ids: torch.Tensor, pixel_values: torch.Tensor,
                 num_logits_to_keep: int = 1):
        self.model = model
        dev = model.device
        self.ids_dev = torch.empty(input_ids.shape, dtype=torch.int64, device=dev)
        self.pv_dev = torch.empty(pixel_values.shape, dtype=bf16, device=dev)
        self.ids_dev.copy_(input_ids)
        self.pv_dev.copy_(pixel_values)
        self.n_image_tokens = int((input_ids == model.config.image_token_index).sum())
        ids_host = input_ids.cpu()
        kw = dict(num_logits_to_keep=num_logits_to_keep, input_ids_host=ids_host)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(2):
                model(self.ids_dev, self.pv_dev, None, **kw)
        torch.cuda.current_stream(dev).wait_stream(side)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.logits = model(self.ids_dev, self.pv_dev, None, **kw).logits

    def replay(self) -> torch.Tensor:
        self.graph.replay()
        return self.logits

    def __call__(self, input_ids: torch.Tensor, pixel_values: torch.Tensor) -> torch.Tensor:
        if not input_ids.is_cuda:  # same ValueError contract as forward() (modeling_aria.py:268-271), checked on the host
            n = int((input_ids == self.model.config.image_token_index).sum())
            if n != self.n_image_tokens:
                raise ValueError(f"Image features and image tokens do not match: tokens: {n}, features {self.n_image_tokens}")
        self.ids_dev.copy_(input_ids, non_blocking=True)
        self.pv_dev.copy_(pixel_values, non_blocking=True)
        return self.replay()


def init_random_(model: nn.Module, seed: int = 0, std: float = 0.02):
    """Random-init (no checkpoint offline): N(0, std^2) for matrices / embeddings / biases / queries, 1 for the
    norm scales (the only 1-D parameters named `weight`)."""
    g = torch.Generator(device=next(model.parameters()).device).manual_seed(seed)
    for name, p in model.named_parameters():
        if p.dim() == 1 and name.endswith("weight"):
            p.fill_(1.0)
        else:
            p.normal_(0.0, std, generator=g)
    return model
