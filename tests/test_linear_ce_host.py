"""CPU: host logic of the fused lm_head loss (`aria_b200.loss.linear_cross_entropy`) and of its seam (`install.install_loss`).

The two new kernels and the data-gradient GEMM are replaced by torch stand-ins defined here (the rest by tests/standin_ops.py),
so what runs is the op's row selection, chunking, launch decisions and the seam's routing around the UNMODIFIED reference
`AriaForConditionalGeneration`, compared with that reference's own forward on CPU in fp32.  The GPU suite runs the same
scenarios on the real kernels (tests/test_gpu_linear_ce.py)."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import standin_ops  # noqa: E402

from oracle.ref_loader import load_reference, reference_available  # noqa: E402

needs_reference = pytest.mark.skipif(not reference_available(), reason="reference sources not present")


@pytest.fixture(autouse=True)
def _grad_on():
    with torch.enable_grad():
        yield


@pytest.fixture(autouse=True)
def _reference_gmm(monkeypatch):
    """The reference's own `sequential_gemm` behind its `experts_gemm` global, whatever another test bound there."""
    if reference_available():
        m = load_reference().moe_lm
        monkeypatch.setattr(m, "experts_gemm", m.sequential_gemm)


# ------------------------------------------------------------------------------------------------ stand-ins, call log
def _cross_entropy_rows(logits, labels, grad_scale, loss=None):
    lf = logits.float()
    lse = lf.logsumexp(1)
    row = lse - lf.gather(1, labels[:, None]).squeeze(1)
    g = torch.softmax(lf, 1)
    g[torch.arange(g.shape[0]), labels] -= 1.0
    logits.copy_(g * grad_scale)
    if loss is not None:
        loss.copy_(row)
    return row


def _wgrad_accumulate_f32(a, b, out):
    out += a.float().T @ b.float()
    return out


def _matmul_kn(a, w_kn, residual=None):
    return a @ w_kn


@pytest.fixture
def calls(monkeypatch):
    """Stand-ins for the ops the loss uses; returns the log of (op name, rows) per call."""
    from aria_b200 import ops
    standin_ops.patch(monkeypatch)
    log = []

    def logged(name, fn):
        def f(a, *args, **kw):
            log.append((name, a.shape[0]))
            return fn(a, *args, **kw)
        return f
    for name, fn in (("linear", standin_ops.linear), ("cross_entropy_rows", _cross_entropy_rows),
                     ("matmul_kn", _matmul_kn), ("wgrad_accumulate_f32", _wgrad_accumulate_f32)):
        monkeypatch.setattr(ops, name, logged(name, fn))
    return log


def _names(log):
    return [n for n, _ in log]


# ------------------------------------------------------------------------------------------------ the op
def _case(N=23, d=32, V=64, ignored=(1, 2, 5, 11, 12, 13, 20), seed=0):
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(N, d, generator=g)
    w = torch.randn(V, d, generator=g) * 0.3
    lab = torch.randint(0, V, (N,), generator=g)
    lab[list(ignored)] = -100
    return h, w, lab


@pytest.mark.parametrize("reduction", ["mean", "sum"])
def test_op_matches_cross_entropy_over_chunks(calls, monkeypatch, reduction):
    """Value and gradients equal F.cross_entropy(F.linear(h, w)); 16 valid rows in chunks of 5 give calls of 5, 5, 5, 1 rows,
    and the whole call reads the device once (one .tolist(), no .item(), no nonzero())."""
    from aria_b200.loss import linear_cross_entropy
    h, w, lab = _case()
    h1, w1 = h.clone().requires_grad_(True), w.clone().requires_grad_(True)
    syncs, saved = [], {}
    for name in ("tolist", "item", "nonzero", "__bool__"):                 # the ways a tensor reaches the host
        saved[name] = orig = getattr(torch.Tensor, name)
        setattr(torch.Tensor, name, (lambda o, n: lambda self, *a, **k: (syncs.append(n), o(self, *a, **k))[1])(orig, name))
    try:
        loss = linear_cross_entropy(h1, w1, lab, reduction=reduction, chunk_rows=5)
    finally:
        for name, orig in saved.items():
            setattr(torch.Tensor, name, orig)
    assert syncs == ["tolist"]
    assert loss.dtype == torch.float32
    (loss / 3).backward()
    h2, w2 = h.clone().requires_grad_(True), w.clone().requires_grad_(True)
    want = F.cross_entropy(F.linear(h2, w2), lab, reduction=reduction)
    (want / 3).backward()
    torch.testing.assert_close(loss, want, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(h1.grad, h2.grad, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(w1.grad, w2.grad, rtol=1e-5, atol=1e-6)
    assert float(h1.grad[[1, 2, 5]].abs().max()) == 0.0
    assert [r for n, r in calls if n == "linear"] == [5, 5, 5, 1]
    assert [r for n, r in calls if n == "cross_entropy_rows"] == [5, 5, 5, 1]
    assert [r for n, r in calls if n == "matmul_kn"] == [5, 5, 5, 1]
    assert [r for n, r in calls if n == "wgrad_accumulate_f32"] == [5, 5, 5, 1]


def test_op_launches_only_what_a_gradient_needs(calls):
    from aria_b200.loss import linear_cross_entropy
    h, w, lab = _case()
    want = F.cross_entropy(F.linear(h, w), lab)
    # frozen weight: no weight-gradient GEMM, and the weight gets no .grad
    wf, hh = w.clone(), h.clone().requires_grad_(True)
    linear_cross_entropy(hh, wf, lab, chunk_rows=8).backward()
    assert "wgrad_accumulate_f32" not in _names(calls) and "matmul_kn" in _names(calls)
    assert wf.grad is None and hh.grad is not None
    calls.clear()
    # hidden needs no gradient: no data-gradient GEMM
    ww = w.clone().requires_grad_(True)
    linear_cross_entropy(h, ww, lab, chunk_rows=8).backward()
    assert "matmul_kn" not in _names(calls) and "wgrad_accumulate_f32" in _names(calls)
    calls.clear()
    # no_grad: logits and loss only
    with torch.no_grad():
        got = linear_cross_entropy(h.requires_grad_(True), ww, lab, chunk_rows=8)
    assert set(_names(calls)) == {"linear", "cross_entropy_rows"}
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-6)


def test_op_all_rows_ignored(calls):
    from aria_b200.loss import linear_cross_entropy
    h, w, lab = _case()
    lab[:] = -100
    for reduction, value in (("mean", float("nan")), ("sum", 0.0)):
        hh, ww = h.clone().requires_grad_(True), w.clone().requires_grad_(True)
        loss = linear_cross_entropy(hh, ww, lab, reduction=reduction)
        torch.testing.assert_close(loss, torch.tensor(value), equal_nan=True)
        torch.testing.assert_close(loss, F.cross_entropy(F.linear(h, w), lab, reduction=reduction), equal_nan=True)
        loss.backward()
        assert float(hh.grad.abs().max()) == 0.0 and float(ww.grad.abs().max()) == 0.0
    assert calls == []


@pytest.mark.parametrize("bad", [64, 1000, -1, -101])
def test_op_rejects_a_label_out_of_range_before_any_launch(calls, bad):
    from aria_b200.loss import linear_cross_entropy
    h, w, lab = _case()
    lab[3] = bad
    with pytest.raises(ValueError, match="outside"):
        linear_cross_entropy(h.requires_grad_(True), w, lab)
    assert calls == []
    # another ignore_index makes -100 a label like any other
    with pytest.raises(ValueError, match="outside"):
        linear_cross_entropy(h, w, _case()[2], ignore_index=-1)
    assert calls == []


# ------------------------------------------------------------------------------------------------ the seam
def _ref_model():
    from oracle import configs as C
    from oracle.make_golden import build_reference_model
    ref = load_reference()
    sd = C.aria_state(C.TINY, seed=0, dtype=torch.float32)
    model = build_reference_model(ref, C.TINY, sd, torch.float32).train()
    return ref, model, C.TINY


def _inputs(cfg, mask, labels, image=True, seed=5):
    g = torch.Generator().manual_seed(seed)
    B, V = 2, cfg["text_config"]["vocab_size"]
    text = torch.randint(10, V, (B, 22), generator=g)
    if image:
        ids = torch.cat([text[:, :3], torch.full((B, 8), cfg["image_token_index"]), text[:, 3:]], dim=1)
        S = cfg["vision_config"]["image_size"]
        pv = torch.randn(B, 3, S, S, generator=g)
    else:
        ids, pv = text, None
    T = ids.shape[1]
    am = torch.ones(B, T, dtype=torch.long)
    if mask == "right":
        am[1, -6:] = 0
    elif mask == "left":
        am[1, :2] = 0
    lab = ids.clone()
    if labels == "user_turn":
        lab[:, :14] = -100                     # the prompt (image included) is not trained on
    elif labels == "all_ignored":
        lab[:] = -100
    lab = lab.masked_fill(am == 0, -100)
    return dict(input_ids=ids, pixel_values=pv, attention_mask=None if mask == "none" else am, labels=lab)


def _grads(model):
    out = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
    model.zero_grad(set_to_none=True)
    return out


@needs_reference
@pytest.mark.parametrize("labels", ["all", "user_turn", "all_ignored"])
@pytest.mark.parametrize("mask", ["none", "right", "left"])
def test_seam_rows_match_the_reference_forward(calls, mask, labels):
    from aria_b200 import install
    ref, model, cfg = _ref_model()
    kw = _inputs(cfg, mask, labels, image=mask != "left")
    want = type(model).forward(model, **kw)
    want.loss.backward()
    want_g = _grads(model)
    assert install.install_loss(model) == 1
    got = model(**kw)
    assert type(got) is ref.modeling_aria.AriaCausalLMOutputWithPast and got.logits is None
    assert got.loss.dtype == torch.float32
    assert ("cross_entropy_rows" in _names(calls)) == (labels != "all_ignored")     # no valid row: nothing to launch
    torch.testing.assert_close(got.loss, want.loss, rtol=1e-5, atol=1e-6, equal_nan=True)
    got.loss.backward()
    got_g = _grads(model)
    assert got_g.keys() == want_g.keys()
    for n in want_g:
        torch.testing.assert_close(got_g[n], want_g[n], rtol=1e-4, atol=1e-6, msg=n)


@needs_reference
@pytest.mark.parametrize("case", ["no_labels", "no_grad", "frozen", "num_logits_to_keep", "return_tuple", "wrapped_head"])
def test_seam_falls_back_to_the_original_forward(calls, case):
    from aria_b200 import install
    _, model, cfg = _ref_model()
    kw = _inputs(cfg, "right", "user_turn")
    if case == "no_labels":
        kw["labels"] = None
    elif case == "num_logits_to_keep":
        kw["num_logits_to_keep"] = 1
    elif case == "return_tuple":
        kw["return_dict"] = False
    elif case == "frozen":
        model.requires_grad_(False)
    elif case == "wrapped_head":
        class Wrapped(torch.nn.Module):       # what an adapter wrapper looks like to the seam: not a plain nn.Linear
            def __init__(self, base):
                super().__init__()
                self.base_layer = base
                self.weight = base.weight

            def forward(self, x):
                return self.base_layer(x)
        model.language_model.lm_head = Wrapped(model.language_model.lm_head)
    ctx = torch.no_grad() if case == "no_grad" else torch.enable_grad()
    with ctx:
        want = type(model).forward(model, **kw)
        assert install.install_loss(model) == 1
        got = model(**kw)
    assert calls == []
    want, got = (want, got) if case == "return_tuple" else (want.to_tuple(), got.to_tuple())
    assert len(got) == len(want)
    for a, b in zip(got, want):
        if isinstance(a, torch.Tensor):
            torch.testing.assert_close(a, b, rtol=0, atol=0)


@needs_reference
def test_seam_refuses_an_empty_weight_and_keeps_the_image_check(calls):
    from aria_b200 import install
    _, model, cfg = _ref_model()
    assert install.install_loss(model) == 1 and install.install_loss(model) == 1
    kw = _inputs(cfg, "none", "all")
    kw["input_ids"] = kw["input_ids"].clone()
    kw["input_ids"][0, 3] = 11                  # one image token short
    with pytest.raises(ValueError, match="Image features and image tokens do not match"):
        model(**kw)
    head = model.language_model.lm_head
    head.weight = torch.nn.Parameter(torch.empty(0))
    with pytest.raises(RuntimeError, match="empty"):
        model(**_inputs(cfg, "none", "all"))
    assert calls == []


def test_install_loss_leaves_other_models_alone():
    from aria_b200 import install
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    mirror = AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device="cpu")
    assert install.install_loss(mirror) == 0
