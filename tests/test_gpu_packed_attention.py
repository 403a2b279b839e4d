"""GPU: padding-free packed sequences.  The varlen causal attention forward (aria_attention_fwd_varlen) and backward
(aria_attention_bwd_varlen) against the batched kernels on each sequence alone, bit for bit where the tiling is the same; the
`hf_attention` seam on packed batches (restarting position_ids, or cu_seq_lens_* from `packing.pack_batch`) against the same
examples as a right-padded batch in fp32 eager; and the refusals, which come before any kernel."""
import pytest
import torch

from hf_common import tiny_hf_aria, tiny_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda"
SCALE = 128 ** -0.5
TOL = 2e-2


@pytest.fixture(autouse=True)
def _grad_enabled():
    with torch.enable_grad():
        yield


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30))


# segment lengths: 1 / 63 / 64 / 127 / 128 / 129 / 300 / 2048 rows, starts off every 64- and 128-row boundary
SEGMENT_SETS = [
    ([1, 63, 64, 127, 128, 129, 300], 2),
    ([5, 2048, 129, 1, 300], 20),
    ([127, 63, 2048, 64, 1], 2),
    ([2048] * 7 + [2048 - 13], 2),                 # 8 sequences, 16,371 rows
]


def _packed(lens, H, seed):
    g = torch.Generator().manual_seed(seed)
    N = sum(lens)
    q, k, v = (torch.randn(1, H, N, 128, generator=g).bfloat16().to(DEV) for _ in range(3))
    dout = torch.randn(N, H * 128, generator=g).bfloat16().to(DEV)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0).tolist()), dtype=torch.int32, device=DEV)
    return q, k, v, dout, cu


def _segments(lens):
    c = 0
    for n in lens:
        yield c, c + n
        c += n


def _eager_grads(q, k, v, dout, dtype):
    """Causal eager attention + autograd in `dtype` (softmax in fp32) on one sequence [1, H, T, 128]."""
    T, H = q.shape[2], q.shape[1]
    qd, kd, vd = (t.detach().to(dtype).requires_grad_(True) for t in (q, k, v))
    w = (torch.matmul(qd, kd.transpose(2, 3)) * SCALE).masked_fill(
        torch.ones(T, T, dtype=torch.bool, device=DEV).triu(1), float("-inf"))
    p = torch.softmax(w, dim=-1, dtype=torch.float32).to(dtype)
    o = torch.matmul(p, vd).transpose(1, 2).reshape(1, T, H * 128)
    o.backward(dout.to(dtype).reshape(o.shape))
    return qd.grad, kd.grad, vd.grad


@pytest.mark.parametrize("lens,H", SEGMENT_SETS)
def test_forward_bit_identical_per_sequence(lens, H):
    from aria_b200 import ops
    q, k, v, _, cu = _packed(lens, H, seed=sum(lens))
    out, lse = ops.attention_varlen(q, k, v, cu, SCALE, return_lse=True)
    plain = ops.attention_varlen(q, k, v, cu, SCALE)
    torch.cuda.synchronize()
    assert torch.equal(out, plain)
    for a, b in _segments(lens):
        T = b - a
        o1, l1 = ops.attention(q[:, :, a:b].contiguous(), k[:, :, a:b].contiguous(), v[:, :, a:b].contiguous(), T, T, SCALE, True,
                               return_lse=True)
        assert torch.equal(out[a:b], o1[0]), (a, b)
        assert torch.equal(lse[:, a:b], l1[0]), (a, b)


@pytest.mark.parametrize("lens,H", SEGMENT_SETS)
def test_backward_per_sequence(lens, H):
    from aria_b200 import ops
    q, k, v, dout, cu = _packed(lens, H, seed=sum(lens) + 1)
    out, lse = ops.attention_varlen(q, k, v, cu, SCALE, return_lse=True)
    dq, dk, dv = ops.attention_varlen_bwd(q, k, v, out, dout, lse, cu, SCALE)
    dq2, dk2, dv2 = ops.attention_varlen_bwd(q, k, v, out, dout, lse, cu, SCALE)
    torch.cuda.synchronize()
    assert torch.equal(dk, dk2) and torch.equal(dv, dv2)                     # bit-reproducible
    assert _rel(dq2, dq) <= 3e-5
    worst, dq_gap = {}, []
    for a, b in _segments(lens):
        T = b - a
        qs, ks, vs = (t[:, :, a:b].contiguous() for t in (q, k, v))
        o1, l1 = ops.attention(qs, ks, vs, T, T, SCALE, True, return_lse=True)
        g1 = ops.attention_bwd(qs, ks, vs, o1, dout[a:b][None].contiguous(), l1, T, T, SCALE, True)
        g1b = ops.attention_bwd(qs, ks, vs, o1, dout[a:b][None].contiguous(), l1, T, T, SCALE, True)
        assert torch.equal(dk[:, :, a:b], g1[1]), (a, b)
        assert torch.equal(dv[:, :, a:b], g1[2]), (a, b)
        # dq: fp32 atomic sums in another order, then rounded to bf16, so a few roundings flip.  The batched kernel against
        # itself (g1b) is printed beside it: the same effect, measured on the same segment
        dq_gap.append((T, _rel(dq[:, :, a:b], g1[0]), _rel(g1b[0], g1[0])))
        assert dq_gap[-1][1] <= 3e-5, (a, b, dq_gap[-1])
        if T >= 64:                                                          # the eager bar (tiny sequences: too few elements)
            ref32 = _eager_grads(qs, ks, vs, dout[a:b], torch.float32)
            ref16 = _eager_grads(qs, ks, vs, dout[a:b], torch.bfloat16)
            for name, g, r32, r16 in zip(("dq", "dk", "dv"), (dq, dk, dv), ref32, ref16):
                e, e16 = _rel(g[:, :, a:b], r32), _rel(r16, r32)
                worst[name] = max(worst.get(name, 0.0), e)
                assert e <= TOL and e <= 2 * e16 + 1e-3, (name, a, b, e, e16)
    print(f"{lens} H={H}: worst rel-L2 vs fp32 eager {worst}")
    print(f"{lens} H={H}: dq rel-L2 (rows, varlen vs batched, batched vs batched): "
          + ", ".join(f"({T}, {x:.2e}, {y:.2e})" for T, x, y in dq_gap))


def test_sequences_are_isolated():
    from aria_b200 import ops
    lens = [129, 300, 64, 1, 700]
    q, k, v, dout, cu = _packed(lens, 2, seed=9)

    def run(q_, k_, v_, dout_):
        out, lse = ops.attention_varlen(q_, k_, v_, cu, SCALE, return_lse=True)
        return (out, lse) + ops.attention_varlen_bwd(q_, k_, v_, out, dout_, lse, cu, SCALE)

    base = run(q, k, v, dout)
    a, b = 129, 429                                                          # perturb the second sequence
    q2, k2, v2, d2 = q.clone(), k.clone(), v.clone(), dout.clone()
    g = torch.Generator().manual_seed(1)
    for t in (q2, k2, v2):
        t[:, :, a:b] = torch.randn(1, 2, b - a, 128, generator=g).bfloat16().to(DEV)
    d2[a:b] = torch.randn(b - a, 256, generator=g).bfloat16().to(DEV)
    pert = run(q2, k2, v2, d2)
    for name, x, y in zip(("out", "lse", "dq", "dk", "dv"), base, pert):
        rows = (lambda t, s, e: t[s:e]) if name == "out" else (lambda t, s, e: t[..., s:e, :] if t.dim() == 4 else t[:, s:e])
        assert not torch.equal(rows(x, a, b), rows(y, a, b)), name
        for s, e in _segments(lens):
            if (s, e) == (a, b):
                continue
            if name == "dq":                                                 # fp32 atomics: order-dependent last bits
                assert _rel(rows(y, s, e), rows(x, s, e)) <= 1e-5, (name, s)
            else:
                assert torch.equal(rows(x, s, e), rows(y, s, e)), (name, s)


# ------------------------------------------------------------------------------------------------ through the seam
def _param_grads(model):
    return {n: p.grad.detach().float().clone() for n, p in model.named_parameters() if p.grad is not None}


def _check_grads(got, want, what):
    assert got.keys() == want.keys() and got, what
    worst = max(((_rel(got[n], want[n]), n) for n in want), key=lambda x: x[0])
    print(f"{what}: worst parameter-gradient rel-L2 {worst[0]:.3e} ({worst[1]})")
    assert worst[0] <= TOL, (what, worst)


def _padded_batch(lens, vocab, seed):
    g = torch.Generator().manual_seed(seed)
    T = max(lens)
    ids = torch.zeros(len(lens), T, dtype=torch.long)
    am = torch.zeros_like(ids)
    for b, n in enumerate(lens):
        ids[b, :n] = torch.randint(10, vocab, (n,), generator=g)
        am[b, :n] = 1
    labels = ids.masked_fill(am == 0, -100)
    return ids, am, labels


def _tiny_llama():
    from transformers import LlamaConfig, LlamaForCausalLM
    cfg = LlamaConfig(vocab_size=512, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2,
                      num_key_value_heads=2, head_dim=128, max_position_embeddings=4096, pad_token_id=0)
    torch.manual_seed(0)
    return LlamaForCausalLM(cfg)


def _recording(monkeypatch):
    """Record every output of ops.attention_varlen (what the seam's packed forward and its checkpoint recompute return)."""
    from aria_b200 import ops
    outs, inner = [], ops.attention_varlen

    def rec(*a, **kw):
        r = inner(*a, **kw)
        outs.append(tuple(t.detach().clone() for t in r) if isinstance(r, tuple) else r.detach().clone())
        return r

    monkeypatch.setattr(ops, "attention_varlen", rec)
    return outs


def _recompute_is_exact(outs, layers):
    """Under checkpointing each layer's packed attention runs twice: the recompute must equal the forward bit for bit."""
    assert len(outs) == 2 * layers
    first, again = outs[:layers], outs[layers:]
    for o in first:
        assert any(all(torch.equal(x, y) for x, y in zip(o, r)) for r in again)


def _packed_kw(padded, with_cu):
    from aria_b200.packing import pack_batch
    p = pack_batch(padded, return_flash_attn_kwargs=with_cu)
    return {n: (t.to(DEV) if torch.is_tensor(t) else t) for n, t in p.items()}


@pytest.mark.parametrize("with_cu", [False, True])
def test_llama_packed_training_matches_padded(with_cu, monkeypatch):
    from aria_b200 import hf_attention
    lens = [70, 200, 1, 131]
    ids, am, labels = _padded_batch(lens, 512, seed=3)
    padded = dict(input_ids=ids, attention_mask=am, labels=labels)
    ref = _tiny_llama().to(DEV).float().train()
    ref.config._attn_implementation = "eager"
    want_loss = ref(**{n: t.to(DEV) for n, t in padded.items()}).loss
    want_loss.backward()
    want = _param_grads(ref)
    kw = _packed_kw(padded, with_cu)
    grads = {}
    for ckpt in (False, True):
        model = _tiny_llama().to(DEV).bfloat16().train()
        model.config._attn_implementation = hf_attention.register()
        if ckpt:
            model.gradient_checkpointing_enable(gradient_checkpointing_kwargs={"use_reentrant": False})
        outs = _recording(monkeypatch)
        loss = model(**kw).loss
        loss.backward()
        if ckpt:
            _recompute_is_exact(outs, 2)
        assert abs(float(loss) - float(want_loss)) <= TOL * abs(float(want_loss))
        grads[ckpt] = _param_grads(model)
        _check_grads(grads[ckpt], want, f"llama packed (cu_seq_lens {with_cu}), gradient checkpointing {ckpt}")
    for n in grads[False]:                                                   # the recompute reproduces the forward exactly
        assert torch.equal(grads[False][n], grads[True][n]), n


def _aria(dtype, impl, ckpt=False):
    model = tiny_hf_aria(device=DEV, dtype=dtype)
    for m in model.modules():
        c = getattr(m, "config", None)
        if c is not None and hasattr(c, "moe_topk"):
            c.moe_topk = c.moe_num_experts
    for n, p in model.named_parameters():
        p.requires_grad_(not ("vision_tower" in n or "multi_modal_projector" in n))
    model.train()
    model.config.text_config._attn_implementation = impl
    model.model.language_model.config._attn_implementation = impl
    if ckpt:
        model.gradient_checkpointing_enable(gradient_checkpointing_kwargs={"use_reentrant": False})
    return model


def _aria_batch():
    ids0, pv, pm = tiny_inputs(batch=1, n_text=40)                          # example 0 carries the image
    ids, am, labels = _padded_batch([48, 23, 37], 512, seed=6)
    ids[0] = ids0[0]
    labels[0] = ids0[0].masked_fill(ids0[0] == 9, -100)
    return dict(input_ids=ids, attention_mask=am, labels=labels, pixel_values=pv, pixel_mask=pm)


@pytest.mark.parametrize("with_cu", [False, True])
def test_hf_aria_packed_training_matches_padded(with_cu, monkeypatch):
    from aria_b200 import hf_attention
    padded = _aria_batch()
    ref = _aria(torch.float32, "eager")
    want_loss = ref(**{n: t.to(DEV) for n, t in padded.items()}).loss
    want_loss.backward()
    want = _param_grads(ref)
    kw = _packed_kw(padded, with_cu)
    kw["pixel_values"] = kw["pixel_values"].bfloat16()
    grads = {}
    for ckpt in (False, True):
        model = _aria(torch.bfloat16, hf_attention.register(), ckpt)
        outs = _recording(monkeypatch)
        loss = model(**kw).loss
        loss.backward()
        if ckpt:
            _recompute_is_exact(outs, 2)
        assert abs(float(loss) - float(want_loss)) <= TOL * abs(float(want_loss))
        grads[ckpt] = _param_grads(model)
        _check_grads(grads[ckpt], want, f"hf aria packed (cu_seq_lens {with_cu}), gradient checkpointing {ckpt}")
    # transformers' eager MoE scatters its gradients with atomics, so whole-model gradients are compared within the bar above;
    # the exactness of the recompute is checked on the attention outputs themselves


def test_packed_logits_match_padded_rows_without_grad():
    """No-grad packed prefill (aria_attention_fwd_varlen without lse): each example's logits against its padded row in fp32
    eager, within test_registered_core_matches_hf_eager's bar (max-abs 3e-2 of the logit scale)."""
    from aria_b200 import hf_attention
    lens = [70, 200, 1, 131]
    ids, am, _ = _padded_batch(lens, 512, seed=8)
    ref = _tiny_llama().to(DEV).float().eval()
    ref.config._attn_implementation = "eager"
    model = _tiny_llama().to(DEV).bfloat16().eval()
    model.config._attn_implementation = hf_attention.register()
    kw = _packed_kw(dict(input_ids=ids, attention_mask=am), with_cu=False)
    with torch.no_grad():
        want = ref(input_ids=ids.to(DEV), attention_mask=am.to(DEV)).logits.float()
        got = model(**kw).logits.float()[0]
    for b, (a, e) in enumerate(_segments(lens)):
        w = want[b, :e - a]
        err = float((got[a:e] - w).abs().max() / w.abs().max())
        assert err <= 3e-2, (b, err)


def test_refusals_come_before_any_kernel(monkeypatch):
    from aria_b200 import hf_attention, ops

    def boom(*a, **kw):
        raise AssertionError("a kernel ran")

    for name in ("attention", "attention_varlen", "attention_bwd", "attention_varlen_bwd", "attention_decode"):
        monkeypatch.setattr(ops, name, boom)

    class _Stub(torch.nn.Module):
        is_causal = True
        num_key_value_groups = 1

    q = torch.randn(1, 2, 12, 128, device=DEV).bfloat16()
    q2 = torch.randn(2, 2, 12, 128, device=DEV).bfloat16()
    pos = torch.cat([torch.arange(7), torch.arange(5)])[None].to(DEV)
    cu = torch.tensor([0, 7, 12], dtype=torch.int32, device=DEV)
    f = hf_attention.aria_b200_attention_forward
    with pytest.raises(NotImplementedError):
        f(_Stub(), q2, q2, q2, None, position_ids=pos.expand(2, 12))
    with pytest.raises(NotImplementedError):
        f(_Stub(), q[:, :, 4:], q, q, None, position_ids=pos[:, 4:])
    with pytest.raises(ValueError):
        f(_Stub(), q, q, q, None, cu_seq_lens_q=cu, cu_seq_lens_k=torch.tensor([0, 6, 12], dtype=torch.int32, device=DEV))
    for bad in ([0, 7, 11], [0, 7, 7, 12], [2, 7, 12]):
        t = torch.tensor(bad, dtype=torch.int32, device=DEV)
        with pytest.raises(ValueError):
            f(_Stub(), q, q, q, None, cu_seq_lens_q=t, cu_seq_lens_k=t)


# ------------------------------------------------------------------------------------------------ the reference recipe
def _ref():
    from oracle import ref_loader
    if not ref_loader.reference_available():
        pytest.skip("reference files neither in the reference tree nor staged in oracle/_ref (run oracle/build_ref.py)")
    return ref_loader.load_reference()


def _ref_model(dtype, ours, z, aux, monkeypatch):
    ref = _ref()
    from aria_b200 import hf_attention, install
    from oracle import configs as C
    from oracle.make_golden import build_reference_model
    monkeypatch.setattr(ref.moe_lm, "experts_gemm", ref.moe_lm.sequential_gemm)   # install(trainable=True) replaces it
    sd = C.aria_state(C.TINY, seed=0, dtype=torch.float32)
    model = build_reference_model(ref, C.TINY, sd, dtype).to(DEV)
    rot = model.language_model.model.rotary_emb
    rot.inv_freq = rot.inv_freq.float().to(DEV)
    for m in model.modules():
        c = getattr(m, "config", None)
        if c is not None and hasattr(c, "moe_topk"):
            c.moe_topk = c.moe_num_experts
        if c is not None and hasattr(c, "moe_aux_loss_coeff"):
            c.moe_z_loss_coeff, c.moe_aux_loss_coeff = z, aux
    for n, p_ in model.named_parameters():
        p_.requires_grad_(not ("vision_tower" in n or "multi_modal_projector" in n))
    model.train()
    if ours:
        assert install.install(model, ref.moe_lm, trainable=True) == 2
        key = hf_attention.register()
        model.config.text_config._attn_implementation = key
        model.language_model.config._attn_implementation = key
        assert install.install_loss(model) == 1
    return model


def _ref_step(model, kw):
    out = model(**kw)
    out.loss.backward()
    return float(out.loss), {n: p_.grad.detach().float().cpu() for n, p_ in model.named_parameters() if p_.grad is not None}


def _real_token_router_losses(monkeypatch, real):
    """The reference TopKRouter with its two router losses taken over the real (non-pad) rows only: every row is routed as
    before, only the z-loss and the load-balancing loss see the rows `real` (bool [B*T]) selects.  This is what a packed run
    computes, written independently of our seam on the reference's own loss functions."""
    moe = _ref().moe_lm

    def forward(self, input):
        E, k = self.config.moe_num_experts, self.config.moe_topk
        logits = self.gating(input).view(-1, E)
        if self.training:
            logits = moe.MoEAuxLossAutoScaler.apply(logits, moe.z_loss_func(logits[real], self.config.moe_z_loss_coeff))
        top_logits, top_indices = torch.topk(logits, k=k, dim=1)
        scores = torch.softmax(top_logits, dim=-1, dtype=torch.float32).type_as(logits)
        tokens_per_expert = torch.histc(top_indices.flatten(), bins=E, min=0, max=E - 1)
        if self.training:
            real_per_expert = torch.histc(top_indices[real].flatten(), bins=E, min=0, max=E - 1)
            aux = moe.switch_load_balancing_loss_func(torch.softmax(logits[real], dim=-1, dtype=torch.float32), real_per_expert,
                                                      k, self.config.moe_aux_loss_coeff)
            scores = moe.MoEAuxLossAutoScaler.apply(scores, aux)
        return scores, top_indices, tokens_per_expert

    monkeypatch.setattr(moe.TopKRouter, "forward", forward)


def test_reference_recipe_packed_matches_padded(monkeypatch):
    """The reference model with install(trainable=True) + hf_attention + install_loss, fed pack_batch's output unmodified (a
    padded multimodal batch, images in both examples), against the unpatched model on the padded batch in fp32 eager, under
    test_seam_trains_the_reference_model's rule: the loss and every parameter gradient within rel-L2 2e-2, or within 1.25x the
    unpatched bf16 run's own distance from fp32.
    - router losses off: against the padded run as it is;
    - router losses on (z-loss 1.0, load balancing 1.0): the packed run routes no pad token, so its router losses are those of
      the real tokens.  It matches the padded run whose router losses are taken over the real rows only
      (`_real_token_router_losses`), and the padded run as it is differs from both beyond the bar: the whole difference is the
      router-loss term over the pad rows."""
    _ref()
    import hf_common as H
    from aria_b200.packing import pack_batch
    ids, pv, pm = H.tiny_inputs(batch=2, seed=4)                             # images in both examples
    am = torch.ones_like(ids)
    am[1, -9:] = 0
    ids[1, -9:] = 0
    labels = ids.masked_fill(am == 0, -100)
    labels[:, :14] = -100                                                    # the user turn, image included
    padded = dict(input_ids=ids, pixel_values=pv, pixel_mask=pm, attention_mask=am, labels=labels)
    padded32 = {n: t.to(DEV) for n, t in padded.items()}
    padded16 = dict(padded32, pixel_values=padded32["pixel_values"].bfloat16())
    packed = {n: t.to(DEV) for n, t in pack_batch(padded16).items()}         # the recipe's call: model(**pack_batch(batch))
    real = am.view(-1).bool().to(DEV)

    def check(got, loss, want, want_loss, eager_bf16, what):
        assert abs(loss - want_loss) <= TOL * abs(want_loss), (what, loss, want_loss)
        assert got.keys() == want.keys() and "language_model.lm_head.weight" in got
        tol = {n: max(TOL, 1.25 * _rel(eager_bf16[n], want[n])) for n in want}
        worst = max(((_rel(got[n], want[n]) / tol[n], n) for n in want), key=lambda t: t[0])
        print(f"{what}: loss {loss:.5f} vs {want_loss:.5f}, worst gradient {worst[0] * tol[worst[1]]:.3e} ({worst[1]}, "
              f"tolerance {tol[worst[1]]:.3e})")
        assert worst[0] <= 1.0, (what, worst)

    def run(z, aux, real_only):
        with monkeypatch.context() as mp:
            if real_only:
                _real_token_router_losses(mp, real)
            want_loss, want = _ref_step(_ref_model(torch.float32, False, z, aux, mp), padded32)
            eager_bf16 = _ref_step(_ref_model(torch.bfloat16, False, z, aux, mp), padded16)[1]
        with monkeypatch.context() as mp:
            loss, got = _ref_step(_ref_model(torch.bfloat16, True, z, aux, mp), packed)
        return got, loss, want, want_loss, eager_bf16

    got, loss, want, want_loss, eager_bf16 = run(0.0, 0.0, False)
    check(got, loss, want, want_loss, eager_bf16, "router losses off")
    got, loss, want, want_loss, eager_bf16 = run(1.0, 1.0, True)
    check(got, loss, want, want_loss, eager_bf16, "router losses on, padded reference over real rows")
    with monkeypatch.context() as mp:
        all_loss, want_all = _ref_step(_ref_model(torch.float32, False, 1.0, 1.0, mp), padded32)
    assert abs(all_loss - want_loss) <= 1e-6 * abs(want_loss)                 # router losses move gradients, not the loss value
    apart = max(_rel(want_all[n], want[n]) for n in want)
    packed_apart = max(_rel(got[n], want_all[n]) for n in want)
    print(f"router losses on: padded run over all rows vs over real rows {apart:.3e}; packed run vs padded over all rows "
          f"{packed_apart:.3e}")
    assert apart > 2 * TOL and packed_apart > 2 * TOL
