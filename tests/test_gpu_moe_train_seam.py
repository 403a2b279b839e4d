"""GPU: the trainable MoE seams — `aria_grouped_wgrad` over densely packed (unaligned) groups, the differentiable `gmm`
drop-in (seam 1), `install(..., trainable=True)` on the reference's own `MoELayer` (seam 2, router losses, LoRA-wrapped experts),
and whole tiny models (the reference's `AriaForConditionalGeneration`, transformers' own Aria) trained through the seams with
and without gradient checkpointing.  Gradients are compared against fp32 eager autograd on the same bf16 values: rel-L2 <= 2e-2."""
import copy
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = 2e-2


@pytest.fixture(autouse=True)
def _grad_on():
    """Other test modules switch autograd off at import (torch.set_grad_enabled(False)); these tests need it."""
    with torch.enable_grad():
        yield


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _ref():
    from oracle import ref_loader
    if not ref_loader.reference_available():
        pytest.skip("reference files neither in the reference tree nor staged in oracle/_ref (run oracle/build_ref.py)")
    return ref_loader.load_reference()


@pytest.fixture(autouse=True)
def _reference_gmm(monkeypatch):
    """The fp32 eager runs use the reference's own `sequential_gemm` (other tests may have left a seam bound to the module
    global); whatever a test binds there is undone afterwards."""
    from oracle import ref_loader
    if ref_loader.reference_available():
        m = ref_loader.load_reference().moe_lm
        monkeypatch.setattr(m, "experts_gemm", m.sequential_gemm)
    yield


def _offsets(counts):
    return torch.tensor([0] + torch.tensor(counts).cumsum(0).tolist(), dtype=torch.int32)


# ------------------------------------------------------------------------------------------------ wgrad kernel
@pytest.mark.parametrize("Md,Nd", [(200, 136), (256, 384)])
def test_wgrad_unaligned_groups(Md, Nd):
    from aria_b200 import ops
    g = torch.Generator().manual_seed(Md)
    counts = [1, 15, 17, 0, 33, 100, 7]
    rows = sum(counts)
    a = torch.randn(rows + 21, Md, generator=g).bfloat16()      # trailing rows past the last group
    b = torch.randn(rows + 21, Nd, generator=g).bfloat16()
    off = _offsets(counts)
    got = ops.grouped_wgrad(a.to(DEV), b.to(DEV), off.to(DEV)).cpu()
    for e in range(len(counts)):
        lo, hi = int(off[e]), int(off[e + 1])
        if hi == lo:
            assert not got[e].any()
        else:
            assert _rel(got[e], a[lo:hi].float().t() @ b[lo:hi].float()) <= 1e-2, e


def test_wgrad_unaligned_groups_two_sources():
    """The expert-parallel layout: offsets over (source, group) pairs, out[g] sums both sources' rows."""
    from aria_b200 import ops
    g = torch.Generator().manual_seed(5)
    G, S = 6, 2
    counts = torch.randint(0, 40, (S * G,), generator=g).tolist()
    counts[3] = 0
    rows = sum(counts)
    a = torch.randn(rows, 128, generator=g).bfloat16()
    b = torch.randn(rows, 192, generator=g).bfloat16()
    off = _offsets(counts)
    got = ops.grouped_wgrad(a.to(DEV), b.to(DEV), off.to(DEV), num_sources=S).cpu()
    for e in range(G):
        want = torch.zeros(128, 192)
        for s in range(S):
            lo, hi = int(off[s * G + e]), int(off[s * G + e + 1])
            want += a[lo:hi].float().t() @ b[lo:hi].float()
        if not want.any():
            assert not got[e].any()
        else:
            assert _rel(got[e], want) <= 1e-2, e


def test_wgrad_aligned_groups_ignore_rows_past_the_group():
    """16-aligned groups issue exactly the MMAs they did before: each group's result is bit-identical to the same group alone
    in a buffer whose rows past the group are garbage."""
    from aria_b200 import ops
    g = torch.Generator().manual_seed(9)
    counts = [16, 48, 0, 80, 32]
    rows = sum(counts)
    a = torch.randn(rows, 256, generator=g).bfloat16().to(DEV)
    b = torch.randn(rows, 256, generator=g).bfloat16().to(DEV)
    off = _offsets(counts)
    got = ops.grouped_wgrad(a, b, off.to(DEV))
    for e in range(len(counts)):
        lo, hi = int(off[e]), int(off[e + 1])
        pad = 64 - (hi - lo) % 64
        ga = torch.cat([a[lo:hi], (torch.randn(pad, 256, generator=g) * 1e4).bfloat16().to(DEV)])
        gb = torch.cat([b[lo:hi], (torch.randn(pad, 256, generator=g) * 1e4).bfloat16().to(DEV)])
        alone = ops.grouped_wgrad(ga, gb, torch.tensor([0, hi - lo], dtype=torch.int32, device=DEV))
        assert torch.equal(alone[0], got[e]), e


# ------------------------------------------------------------------------------------------------ seam 1: differentiable gmm
@pytest.mark.parametrize("device_offsets", [False, True])
def test_experts_gemm_train_gradients(device_offsets):
    from aria_b200 import moe_train
    g = torch.Generator().manual_seed(2)
    counts = [5, 0, 33, 17, 64, 1, 30, 2]
    E, K, N = len(counts), 256, 192
    rows = sum(counts)
    a = torch.randn(rows, K, generator=g).bfloat16()
    w = (torch.randn(E, K, N, generator=g) * 0.05).bfloat16()
    dy = torch.randn(rows, N, generator=g).bfloat16()
    tpe = _offsets(counts).to(DEV) if device_offsets else torch.tensor(counts, dtype=torch.int64)
    a_g, w_g = a.to(DEV).requires_grad_(True), w.to(DEV).requires_grad_(True)
    out = moe_train.experts_gemm_train(a_g, w_g, tpe)
    out.backward(dy.to(DEV))
    a32, w32 = a.float().requires_grad_(True), w.float().requires_grad_(True)
    want = torch.cat([a32[lo:hi] @ w32[e] for e, (lo, hi) in enumerate(zip(_offsets(counts)[:-1].tolist(),
                                                                            _offsets(counts)[1:].tolist()))])
    want.backward(dy.float())
    assert _rel(out.detach(), want.detach()) <= 1e-2
    assert _rel(a_g.grad, a32.grad) <= TOL
    assert _rel(w_g.grad, w32.grad) <= TOL
    assert not w_g.grad[1].any()                                     # empty expert: exact zeros


def test_experts_gemm_train_frozen_weight_launches_no_wgrad(monkeypatch):
    from aria_b200 import moe_train, ops
    calls = {"wgrad": 0, "nt": 0}
    wg, nt = ops.grouped_wgrad, ops.grouped_gemm_nt
    monkeypatch.setattr(ops, "grouped_wgrad", lambda *a, **k: (calls.__setitem__("wgrad", calls["wgrad"] + 1), wg(*a, **k))[1])
    monkeypatch.setattr(ops, "grouped_gemm_nt", lambda *a, **k: (calls.__setitem__("nt", calls["nt"] + 1), nt(*a, **k))[1])
    a = torch.randn(40, 128, device=DEV).bfloat16().requires_grad_(True)
    w = (torch.randn(4, 128, 64, device=DEV) * 0.05).bfloat16()
    moe_train.experts_gemm_train(a, w, torch.tensor([10, 7, 0, 23])).sum().backward()
    assert w.grad is None and a.grad is not None
    assert calls == {"wgrad": 0, "nt": 1}


def test_experts_gemm_train_rejects_what_the_kernel_rejects():
    from aria_b200 import moe_train
    a = torch.randn(40, 128, device=DEV).bfloat16().requires_grad_(True)
    w = (torch.randn(4, 128, 72, device=DEV) * 0.05).bfloat16().requires_grad_(True)   # N = 72: not a multiple of 64
    with pytest.raises(RuntimeError):
        moe_train.experts_gemm_train(a, w, torch.tensor([10, 7, 0, 23]))


# ------------------------------------------------------------------------------------------------ seam 2 on a reference MoELayer
def _ref_layer(ref, d, E, k, I, seed=0):
    cfg = ref.moe_lm.AriaMoELMConfig(hidden_size=d, num_attention_heads=max(2, d // 128), moe_num_experts=E, moe_topk=k,
                                     moe_intermediate_size=I, moe_num_shared_experts=2, intermediate_size=I,
                                     moe_z_loss_coeff=1.0, moe_aux_loss_coeff=5.0)
    layer = ref.moe_lm.MoELayer(cfg)
    g = torch.Generator().manual_seed(seed + d + E)
    for p_ in layer.parameters():
        p_.data = torch.randn(p_.shape, generator=g) * 0.02
    return layer, g


def _safe_tokens(layer32, x, k):
    """Tokens whose fp32 router top-k has a margin above bf16 noise (tests/test_gpu_dropin.py's filter)."""
    with torch.no_grad():
        lg = torch.nn.functional.linear(x.float().view(-1, x.shape[-1]), layer32.router.weight).cpu()
    srt = lg.sort(1, descending=True).values
    return (srt[:, k - 1] - srt[:, k]) > 2 ** -6 * srt.abs().amax(1)


def _grads(mod):
    return {n: p.grad.detach().float().cpu() for n, p in mod.named_parameters() if p.grad is not None}


def _compare(got, want, what, floor=None):
    """Every gradient within TOL of fp32; with `floor` (the unmodified model's own bf16 gradients), a gradient may exceed TOL
    only where bf16 eager autograd is itself further from fp32, and then by at most 25 %."""
    assert got.keys() == want.keys() and got, (what, sorted(got), sorted(want))
    tol = {n: TOL if floor is None else max(TOL, 1.25 * _rel(floor[n], want[n])) for n in want}
    worst = max(((_rel(got[n], want[n]) / tol[n], n) for n in want), key=lambda t: t[0])
    print(f"{what}: worst gradient rel-L2 {worst[0] * tol[worst[1]]:.3e} ({worst[1]}, tolerance {tol[worst[1]]:.3e})")
    assert worst[0] <= 1.0, (what, worst)


@pytest.mark.parametrize("d,E,k,I,T", [(256, 8, 2, 512, 32), (2560, 64, 6, 1664, 768)])
def test_trainable_seam_on_reference_moe_layer(d, E, k, I, T):
    ref = _ref()
    from aria_b200 import install
    layer, g = _ref_layer(ref, d, E, k, I)
    x = torch.randn(2, T // 2, d, generator=g).bfloat16()
    gout = (torch.randn(2, T // 2, d, generator=g) * 0.01).bfloat16()   # small main gradient: the router losses are visible
    layer32 = copy.deepcopy(layer).to(DEV, torch.bfloat16).float().train()       # fp32 on the bf16 values
    layer = layer.to(DEV, torch.bfloat16).train()
    safe = _safe_tokens(layer32, x.to(DEV), k)
    # near-tie tokens get no upstream gradient, so where bf16 and fp32 routing may differ nothing flows through the experts
    gout = gout.view(-1, d).masked_fill(~safe[:, None], 0).view_as(gout).to(DEV)
    S = ref.moe_lm.MoEAuxLossAutoScaler
    S.set_loss_scale(0.5)
    try:
        x32 = x.to(DEV).float().requires_grad_(True)
        layer32(x32).backward(gout.float())
        assert install.install(torch.nn.ModuleList([layer]), trainable=True) == 1
        xb = x.to(DEV).requires_grad_(True)
        out = layer(xb)
        assert out.grad_fn is not None
        out.backward(gout)
        # the same layer in eval(): no router losses
        layer_nl = copy.deepcopy(layer).eval()
        for p_ in layer_nl.parameters():
            p_.grad = None
        install.install(torch.nn.ModuleList([layer_nl]), trainable=True)
        layer_nl(x.to(DEV)).backward(gout)
    finally:
        S.set_loss_scale(torch.tensor(1.0))
    assert _rel(xb.grad.view(-1, d)[safe.to(DEV)], x32.grad.view(-1, d)[safe.to(DEV)]) <= TOL
    _compare(_grads(layer), _grads(layer32), f"reference MoELayer d={d} E={E}")
    # the router losses are resolved above the bf16 noise: dropping them moves the router gradient at least twice as far
    assert _rel(layer_nl.router.weight.grad, layer32.router.weight.grad) > 2 * _rel(layer.router.weight.grad, layer32.router.weight.grad)
    # inference is unchanged: no_grad + eval() runs the same fused block as install()
    layer.eval()
    with torch.no_grad():
        a = layer(x.to(DEV))
        install.install(torch.nn.ModuleList([layer]))
        b = layer(x.to(DEV))
    assert torch.equal(a, b)


def test_trainable_seam_frozen_parameters_and_checkpointing(monkeypatch):
    """Frozen parameters get no gradient and launch no wgrad; the gradients that are computed equal the all-trainable run's
    bit for bit; under torch.utils.checkpoint (use_reentrant=False) the recomputed forward routes identically, so every
    gradient equals the uncheckpointed one bit for bit (all MoE kernels are deterministic)."""
    ref = _ref()
    from aria_b200 import install, ops
    from torch.utils.checkpoint import checkpoint
    layer, g = _ref_layer(ref, 256, 8, 2, 512)
    layer = layer.to(DEV, torch.bfloat16).train()
    install.install(torch.nn.ModuleList([layer]), trainable=True)
    x = torch.randn(2, 48, 256, generator=g).bfloat16().to(DEV)
    gout = torch.randn(2, 48, 256, generator=g).bfloat16().to(DEV)

    def run(ckpt):
        for p_ in layer.parameters():
            p_.grad = None
        xg = x.clone().requires_grad_(True)
        out = checkpoint(layer, xg, use_reentrant=False) if ckpt else layer(xg)
        out.backward(gout)
        return xg.grad.clone(), {n: p_.grad.clone() for n, p_ in layer.named_parameters() if p_.grad is not None}

    dx, full = run(False)
    dx_c, full_c = run(True)
    assert torch.equal(dx, dx_c) and full.keys() == full_c.keys()
    assert all(torch.equal(full[n], full_c[n]) for n in full)
    calls = []
    wg = ops.grouped_wgrad
    monkeypatch.setattr(ops, "grouped_wgrad", lambda *a, **k: (calls.append(1), wg(*a, **k))[1])
    frozen = ("experts.fc1.weight", "shared_experts.up_proj.weight", "router.weight")
    for n, p_ in layer.named_parameters():
        p_.requires_grad_(n not in frozen)
    dx_f, part = run(False)
    assert set(part) == set(full) - set(frozen)
    assert len(calls) == len(full) - len(frozen)
    assert torch.equal(dx_f, dx) and all(torch.equal(part[n], full[n]) for n in part)


def test_trainable_seam_lora_wrapped_experts():
    """The unmodified reference `GroupedGemmLoraLayer` on fc1 and fc2 (base frozen, as peft leaves it): lora_A / lora_B / input
    gradients against fp32 eager autograd; the base weights get none."""
    ref = _ref()
    from oracle import ref_loader
    from aria_b200 import install
    LL = ref_loader.load_reference_lora()
    layer, g = _ref_layer(ref, 256, 8, 2, 512, seed=3)
    for name in ("fc1", "fc2"):
        fc = LL.GroupedGemmLoraLayer(getattr(layer.experts, name), "default", r=8, lora_alpha=16)
        with torch.no_grad():
            fc.lora_B["default"].weight.normal_(0, 0.02, generator=g)        # peft starts B at 0: make the A gradient non-zero
        setattr(layer.experts, name, fc)
    for n, p_ in layer.named_parameters():
        p_.requires_grad_("lora_" in n)
    x = torch.randn(2, 40, 256, generator=g).bfloat16()
    gout = torch.randn(2, 40, 256, generator=g).bfloat16()
    layer32 = copy.deepcopy(layer).to(DEV, torch.bfloat16).float().train()
    layer = layer.to(DEV, torch.bfloat16).train()
    safe = _safe_tokens(layer32, x.to(DEV), 2)
    gout = gout.view(-1, 256).masked_fill(~safe[:, None], 0).view_as(gout).to(DEV)
    x32 = x.to(DEV).float().requires_grad_(True)
    layer32(x32).backward(gout.float())
    install.install(torch.nn.ModuleList([layer]), trainable=True)
    xb = x.to(DEV).requires_grad_(True)
    layer(xb).backward(gout)
    got = _grads(layer)
    assert set(got) == {f"experts.{f}.lora_{ab}.default.weight" for f in ("fc1", "fc2") for ab in "AB"}
    _compare(got, _grads(layer32), "LoRA-wrapped experts")
    assert _rel(xb.grad.view(-1, 256)[safe.to(DEV)], x32.grad.view(-1, 256)[safe.to(DEV)]) <= TOL
    layer.experts.fc1.lora_dropout["default"] = torch.nn.Dropout(0.1)
    with pytest.raises(NotImplementedError, match="lora_dropout"):
        layer(xb)


# ------------------------------------------------------------------------------------------------ whole models
def _batch(vocab, seed=4):
    import hf_common as H
    ids, pv, pm = H.tiny_inputs(batch=2, seed=seed)
    am = torch.ones_like(ids)
    am[1, -5:] = 0                                                   # right-padded second sequence
    ids[1, -5:] = 0
    labels = ids.masked_fill(am == 0, -100).masked_fill(ids == 9, -100)
    return ids.to(DEV), pv, pm.to(DEV), am.to(DEV), labels.to(DEV)


def _all_experts(model):
    for m in model.modules():
        c = getattr(m, "config", None)
        if c is not None and hasattr(c, "moe_topk"):
            c.moe_topk = c.moe_num_experts                           # no routing boundary can flip under bf16 noise


def _reference_model(dtype):
    ref = _ref()
    from oracle import configs as C
    from oracle.make_golden import build_reference_model
    sd = C.aria_state(C.TINY, seed=0, dtype=torch.float32)
    model = build_reference_model(ref, C.TINY, sd, dtype).to(DEV)
    rot = model.language_model.model.rotary_emb
    rot.inv_freq = rot.inv_freq.float().to(DEV)
    return ref, model


def _hf_model(dtype):
    import hf_common as H
    return None, H.tiny_hf_aria(device=DEV, dtype=dtype)


def _train_model(kind, dtype, ours, ckpt, steps=0):
    from aria_b200 import hf_attention, install
    ref, model = (_reference_model if kind == "reference" else _hf_model)(dtype)
    _all_experts(model)
    for n, p_ in model.named_parameters():
        p_.requires_grad_(not ("vision_tower" in n or "multi_modal_projector" in n))
    model.train()
    lm_cfg = model.language_model.config if kind == "reference" else model.model.language_model.config
    if ref is not None:
        ref.moe_lm.experts_gemm = ref.moe_lm.sequential_gemm
    if ours:
        assert install.install(model, ref.moe_lm if ref is not None else None, trainable=True) == 2
        key = hf_attention.register()
        model.config.text_config._attn_implementation = key
        lm_cfg._attn_implementation = key
    if ckpt:
        model.gradient_checkpointing_enable(gradient_checkpointing_kwargs={"use_reentrant": False})
    ids, pv, pm, am, labels = _batch(512)
    kw = dict(input_ids=ids, pixel_values=pv.to(DEV, dtype), pixel_mask=pm, attention_mask=am, labels=labels)
    if ref is not None:
        ref.moe_lm.MoEAuxLossAutoScaler.set_loss_scale(0.5)
    try:
        model(**kw).loss.backward()
        grads = _grads(model)
        losses = []
        if steps:
            opt = torch.optim.SGD([p_ for p_ in model.parameters() if p_.requires_grad], lr=0.2)
            for _ in range(steps):
                opt.zero_grad()
                loss = model(**kw).loss
                loss.backward()
                opt.step()
                losses.append(float(loss))
    finally:
        if ref is not None:
            ref.moe_lm.MoEAuxLossAutoScaler.set_loss_scale(torch.tensor(1.0))
    return grads, losses


@pytest.mark.parametrize("kind", ["reference", "hf"])
def test_whole_model_training_through_the_seams(kind):
    want, _ = _train_model(kind, torch.float32, False, False)
    eager_bf16, _ = _train_model(kind, torch.bfloat16, False, False)
    for ckpt in (False, True):
        got, losses = _train_model(kind, torch.bfloat16, True, ckpt, steps=4 if not ckpt else 0)
        _compare(got, want, f"{kind} Aria, gradient checkpointing {ckpt}", floor=eager_bf16)
        if losses:
            assert all(map(torch.isfinite, map(torch.tensor, losses))) and losses[-1] < losses[0], losses
