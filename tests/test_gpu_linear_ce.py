"""GPU: the fused lm_head loss — the cross-entropy row kernel against fp64, `loss.linear_cross_entropy` at full width against
fp64 `F.cross_entropy(F.linear(...))`, its memory bound at the SFT recipes' batch, and the `install_loss` seam on the
reference's own `AriaForConditionalGeneration` trained through all seams against the unpatched model in fp32."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
DEV = "cuda"
D, V = 2560, 100352
TOL = 2e-2


@pytest.fixture(autouse=True)
def _grad_on():
    """Other test modules switch autograd off at import (torch.set_grad_enabled(False)); these tests need it."""
    with torch.enable_grad():
        yield


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


# ------------------------------------------------------------------------------------------------ the kernel
def _kernel_rows(V_, R=12, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(R, V_, generator=g) * 3.0
    lab = torch.randint(0, V_, (R,), generator=g)
    lab[0], lab[1] = 0, V_ - 1
    x[2] = -60.0 + 0.5 * torch.randn(V_, generator=g)                   # peaked, label on the peak
    x[2, 7] = 60.0
    lab[2] = 7
    x[3] = x[2]                                                          # peaked, label elsewhere
    lab[3] = V_ // 3
    x[4] = (torch.rand(V_, generator=g) * 2 - 1) * 3e4                   # wide range
    x[5] = 1.5                                                           # constant
    return x.bfloat16(), lab


@pytest.mark.parametrize("V_", [512, V])
def test_cross_entropy_rows_against_fp64(V_):
    from aria_b200 import ops
    x, lab = _kernel_rows(V_)
    R = x.shape[0]
    store = torch.zeros(R, V_ + 64, dtype=torch.bfloat16, device=DEV)   # row stride > V
    logits = store[:, :V_]
    logits.copy_(x.to(DEV))
    labels = lab.to(DEV)
    gs = torch.full((1,), 1.0 / R, dtype=torch.float32, device=DEV)
    loss = ops.cross_entropy_rows(logits, labels, gs)
    grad = logits.float().cpu().double()
    x64 = x.double()
    lse = torch.logsumexp(x64, 1)
    want_loss = lse - x64.gather(1, lab[:, None]).squeeze(1)
    want_grad = torch.softmax(x64, 1)
    want_grad[torch.arange(R), lab] -= 1.0
    want_grad *= float(gs)
    got_loss = loss.double().cpu()
    loss_err = (got_loss - want_loss).abs()
    assert bool((loss_err <= torch.maximum(1e-5 * want_loss.abs(), torch.full_like(want_loss, 1e-6))).all()), \
        (loss_err.tolist(), want_loss.tolist())
    big = want_grad.abs() > 1e-30
    rel = ((grad - want_grad).abs() / want_grad.abs().clamp_min(1e-300))[big]
    assert float(rel.max()) <= 2 ** -8, float(rel.max())
    assert bool(((grad - want_grad).abs()[~big] <= 1e-30).all())
    assert bool((store[:, V_:] == 0).all())                              # nothing written past V
    # two runs: identical bits
    again = torch.zeros_like(store)
    again[:, :V_].copy_(x.to(DEV))
    loss2 = ops.cross_entropy_rows(again[:, :V_], labels, gs)
    assert torch.equal(loss2, loss) and torch.equal(again, store)


# ------------------------------------------------------------------------------------------------ the op at full width
N_FULL = 8000   # 40 % ignored -> 4,800 valid rows: one full 4,096-row chunk and a partial second one


@pytest.fixture(scope="module")
def full_case():
    g = torch.Generator().manual_seed(1)
    h = (torch.randn(N_FULL, D, generator=g) * 2.0).bfloat16()
    w = (torch.randn(V, D, generator=g) * 0.02).bfloat16()
    lab = torch.randint(0, V, (N_FULL,), generator=g)
    lab[torch.randperm(N_FULL, generator=g)[:int(0.4 * N_FULL)]] = -100
    return h.to(DEV), w.to(DEV), lab.to(DEV)


def _fp64(h, w, lab, reduction):
    with torch.enable_grad():
        h64 = h.double().requires_grad_(True)
        w64 = w.double().requires_grad_(True)
        loss = F.cross_entropy(F.linear(h64, w64), lab, reduction=reduction)
        (loss / 3).backward()
    return loss.detach(), h64.grad, w64.grad


def _run(h, w, lab, reduction="mean", chunk_rows=4096, need_h=True, need_w=True):
    from aria_b200.loss import linear_cross_entropy
    hh = h.detach().clone().requires_grad_(need_h)
    ww = w.detach().clone().requires_grad_(need_w)
    loss = linear_cross_entropy(hh, ww, lab, reduction=reduction, chunk_rows=chunk_rows)
    if need_h or need_w:
        (loss / 3).backward()
    return loss.detach(), hh.grad, ww.grad


@pytest.mark.parametrize("reduction", ["mean", "sum"])
def test_linear_cross_entropy_full_width_against_fp64(full_case, reduction):
    h, w, lab = full_case
    want_loss, want_dh, want_dw = _fp64(h, w, lab, reduction)
    loss, dh, dw = _run(h, w, lab, reduction)
    assert loss.dtype == torch.float32 and dh.dtype == torch.bfloat16 and dw.dtype == torch.bfloat16
    rel_loss = abs(float(loss) - float(want_loss)) / abs(float(want_loss))
    print(f"{reduction}: loss rel {rel_loss:.2e}, dH rel-L2 {_rel(dh, want_dh):.2e}, dW rel-L2 {_rel(dw, want_dw):.2e}")
    assert rel_loss <= 1e-3
    assert _rel(dh, want_dh) <= 1e-2 and _rel(dw, want_dw) <= 1e-2
    assert float(dh[lab == -100].abs().max()) == 0.0


def test_chunk_size_changes_nothing_per_row(full_case, monkeypatch):
    """chunk_rows 1,024 and 8,192 against the default 4,096: per-row losses and dH within 1e-6 relative."""
    from aria_b200 import ops
    h, w, lab = full_case
    seen = []
    real = ops.cross_entropy_rows

    def record(*a, **kw):
        out = real(*a, **kw)
        seen.append(out.clone())
        return out
    monkeypatch.setattr(ops, "cross_entropy_rows", record)
    runs = {}
    for c in (4096, 1024, 8192):
        seen.clear()
        _, dh, dw = _run(h, w, lab, chunk_rows=c)
        runs[c] = (torch.cat(seen), dh.float(), dw.float())
        assert len(seen) == -(-4800 // c)
    for c in (1024, 8192):
        assert _rel(runs[c][0], runs[4096][0]) <= 1e-6
        assert float(((runs[c][0] - runs[4096][0]).abs() / runs[4096][0].abs()).max()) <= 1e-6
        assert _rel(runs[c][1], runs[4096][1]) <= 1e-6
        assert _rel(runs[c][2], runs[4096][2]) <= 1e-3          # fp32 sums in another order, then one bf16 rounding


def test_frozen_inputs_launch_no_gradient_kernel(full_case, monkeypatch):
    from aria_b200 import ops
    h, w, lab = full_case
    n = {"matmul_kn": 0, "wgrad_accumulate_f32": 0}
    for name in n:
        real = getattr(ops, name)
        monkeypatch.setattr(ops, name, (lambda nm, r: lambda *a, **k: (n.__setitem__(nm, n[nm] + 1), r(*a, **k))[1])(name, real))
    _, dh, dw = _run(h, w, lab, need_w=False)
    assert dw is None and dh is not None and n == {"matmul_kn": 2, "wgrad_accumulate_f32": 0}
    _, dh, dw = _run(h, w, lab, need_h=False)
    assert dh is None and dw is not None and n == {"matmul_kn": 2, "wgrad_accumulate_f32": 2}
    with torch.no_grad():
        loss, _, _ = _run(h, w, lab, need_h=False, need_w=False)
    assert n == {"matmul_kn": 2, "wgrad_accumulate_f32": 2}
    assert abs(float(loss) - float(_fp64(h, w, lab, "mean")[0])) <= 1e-3 * abs(float(loss))


def test_all_ignored_and_bad_labels(full_case):
    from aria_b200.loss import linear_cross_entropy
    h, w, lab = full_case
    none = torch.full_like(lab, -100)
    loss, dh, dw = _run(h, w, none)
    assert torch.isnan(loss) and float(dh.abs().max()) == 0.0 and float(dw.abs().max()) == 0.0
    loss, dh, dw = _run(h, w, none, reduction="sum")
    assert float(loss) == 0.0 and float(dh.abs().max()) == 0.0
    bad = lab.clone()
    bad[5] = V
    with pytest.raises(ValueError, match="outside"):
        linear_cross_entropy(h, w, bad)


def test_memory_bound_at_the_recipe_batch():
    """16,384 rows, full width, 60 % ignored: what forward + backward allocates above the inputs and the gradients it returns
    stays under 2.5 GB.  The reference head (bf16 logits of every row, nn.CrossEntropyLoss) is measured beside it."""
    from aria_b200.loss import linear_cross_entropy
    rows = 16384
    g = torch.Generator().manual_seed(2)
    w = (torch.randn(V, D, generator=g) * 0.02).bfloat16().to(DEV).requires_grad_(True)
    h = (torch.randn(rows, D, generator=g) * 2.0).bfloat16().to(DEV).requires_grad_(True)
    lab = torch.randint(0, V, (rows,), generator=g)
    lab[torch.randperm(rows, generator=g)[:int(0.6 * rows)]] = -100
    lab = lab.to(DEV)
    outputs = h.numel() * 2 + w.numel() * 2

    def peak(fn):
        h.grad = w.grad = None
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        fn().backward()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base - outputs

    fused = peak(lambda: linear_cross_entropy(h, w, lab))
    reference = peak(lambda: F.cross_entropy(F.linear(h, w), lab))
    print(f"peak above inputs and gradients, 16,384 rows, 60 % ignored: fused {fused / 1e9:.2f} GB, "
          f"reference head {reference / 1e9:.2f} GB")
    assert fused < 2.5e9


# ------------------------------------------------------------------------------------------------ the seam, whole model
def _ref():
    from oracle import ref_loader
    if not ref_loader.reference_available():
        pytest.skip("reference files neither in the reference tree nor staged in oracle/_ref (run oracle/build_ref.py)")
    return ref_loader.load_reference()


@pytest.fixture(autouse=True)
def _reference_gmm(monkeypatch):
    from oracle import ref_loader
    if ref_loader.reference_available():
        m = ref_loader.load_reference().moe_lm
        monkeypatch.setattr(m, "experts_gemm", m.sequential_gemm)
    yield


def _model(dtype, ours, ckpt):
    ref = _ref()
    from aria_b200 import hf_attention, install
    from oracle import configs as C
    from oracle.make_golden import build_reference_model
    sd = C.aria_state(C.TINY, seed=0, dtype=torch.float32)
    model = build_reference_model(ref, C.TINY, sd, dtype).to(DEV)
    rot = model.language_model.model.rotary_emb
    rot.inv_freq = rot.inv_freq.float().to(DEV)
    for m in model.modules():                                            # every expert: no routing boundary to flip
        c = getattr(m, "config", None)
        if c is not None and hasattr(c, "moe_topk"):
            c.moe_topk = c.moe_num_experts
    for n, p_ in model.named_parameters():
        p_.requires_grad_(not ("vision_tower" in n or "multi_modal_projector" in n))
    model.train()
    if ours:
        assert install.install(model, ref.moe_lm, trainable=True) == 2
        key = hf_attention.register()
        model.config.text_config._attn_implementation = key
        model.language_model.config._attn_implementation = key
        assert install.install_loss(model) == 1
    if ckpt:
        model.gradient_checkpointing_enable(gradient_checkpointing_kwargs={"use_reentrant": False})
    return model


def _batch(kind):
    import hf_common as H
    ids, pv, pm = H.tiny_inputs(batch=2, seed=4)
    am = torch.ones_like(ids)
    if kind == "image_right_padded":
        am[1, -5:] = 0
        ids[1, -5:] = 0
        labels = ids.masked_fill(am == 0, -100)
        labels[:, :14] = -100                                            # the user turn, image included
        return dict(input_ids=ids.to(DEV), pixel_values=pv.to(DEV), pixel_mask=pm.to(DEV), attention_mask=am.to(DEV),
                    labels=labels.to(DEV))
    ids = ids[:, 12:]                                                    # text only, no attention mask
    return dict(input_ids=ids.to(DEV), labels=ids.clone().to(DEV))


def _step(model, kw, dtype):
    kw = dict(kw)
    if "pixel_values" in kw:
        kw["pixel_values"] = kw["pixel_values"].to(dtype)
    out = model(**kw)
    out.loss.backward()
    grads = {n: p_.grad.detach().float().cpu() for n, p_ in model.named_parameters() if p_.grad is not None}
    return float(out.loss), grads


@pytest.mark.parametrize("kind", ["image_right_padded", "text_only"])
def test_seam_trains_the_reference_model(kind):
    """Unpatched fp32 eager vs bf16 with install(trainable=True) + hf_attention + install_loss, gradient checkpointing off and
    on: the loss and every parameter gradient within rel-L2 2e-2; where the unpatched model's own bf16 gradient is further
    from fp32 than that, within 1.25 times its distance (tests/test_gpu_moe_train_seam.py's rule)."""
    kw = _batch(kind)
    want_loss, want = _step(_model(torch.float32, False, False), kw, torch.float32)
    _, eager_bf16 = _step(_model(torch.bfloat16, False, False), kw, torch.bfloat16)
    for ckpt in (False, True):
        model = _model(torch.bfloat16, True, ckpt)
        loss, got = _step(model, kw, torch.bfloat16)
        assert abs(loss - want_loss) <= TOL * abs(want_loss), (loss, want_loss)
        assert got.keys() == want.keys() and "language_model.lm_head.weight" in got
        tol = {n: max(TOL, 1.25 * _rel(eager_bf16[n], want[n])) for n in want}
        worst = max(((_rel(got[n], want[n]) / tol[n], n) for n in want), key=lambda t: t[0])
        print(f"{kind}, checkpointing {ckpt}: loss {loss:.5f} vs {want_loss:.5f}, worst gradient rel-L2 "
              f"{worst[0] * tol[worst[1]]:.3e} ({worst[1]}, tolerance {tol[worst[1]]:.3e}), lm_head "
              f"{_rel(got['language_model.lm_head.weight'], want['language_model.lm_head.weight']):.3e}")
        assert worst[0] <= 1.0, worst


def test_seam_under_no_grad_is_the_original_forward():
    model = _model(torch.bfloat16, True, False)
    kw = _batch("image_right_padded")
    kw["pixel_values"] = kw["pixel_values"].bfloat16()
    with torch.no_grad():
        got = model(**kw)
        want = type(model).forward(model, **kw)
    assert got.logits is not None and torch.equal(got.logits, want.logits)
    assert torch.equal(got.loss, want.loss)
