"""CPU: the attention backward's C-ABI argument validation (before any CUDA call), and the host logic of the differentiable
attention seam — `hf_attention.aria_b200_attention_forward` under autograd through `attention_train.AttentionFunction` — run
with torch-CPU stand-ins for `ops.attention(return_lse=True)` / `ops.attention_bwd` (below, on top of tests/standin_ops.py).  The
GPU suite runs the same scenarios on the kernels (tests/test_gpu_attention_bwd.py)."""
import ctypes

import pytest
import torch
from torch.utils.checkpoint import checkpoint

import standin_ops
from aria_b200 import hf_attention


# ---- stand-ins for the attention training path: the checker's arithmetic (fp32 eager attention), never the product's
def _attention_f32(q, k, v, Tq, Tk, scale, causal, key_mask):
    """fp32 softmax(q k^T * scale + mask) v -> (out [B, Tq, H*128], lse [B, H, Tq]); a row that sees no key gives 0 and -inf."""
    B, H = q.shape[:2]
    q, k, v = q[:, :, :Tq].float(), k[:, :, :Tk].float(), v[:, :, :Tk].float()
    dead = torch.zeros(B, 1, Tq, Tk, dtype=torch.bool)
    if causal:   # -inf rather than an additive finfo.min mask: a query row that sees no key must get exactly nothing
        dead = dead | (torch.arange(Tk)[None, :] > torch.arange(Tk - Tq, Tk)[:, None])
    if key_mask is not None:
        dead = dead | key_mask.bool()[:, None, None, :]
    w = (torch.matmul(q, k.transpose(2, 3)) * scale).masked_fill(dead, float("-inf"))
    lse = torch.logsumexp(w, dim=-1)
    p = torch.exp(w - torch.where(torch.isinf(lse), torch.zeros_like(lse), lse).unsqueeze(-1))
    o = torch.matmul(p, v).transpose(1, 2)
    return o.reshape(B, Tq, H * 128), lse


def _standin_attention(q, k, v, Tq, Tk, scale, causal, out_hd=128, key_mask=None, return_lse=False):
    if not return_lse:
        return standin_ops.attention(q, k, v, Tq, Tk, scale, causal, out_hd=out_hd, key_mask=key_mask)
    out, lse = _attention_f32(q, k, v, Tq, Tk, scale, causal, key_mask)
    return out.to(q.dtype), lse


def _standin_attention_bwd(q, k, v, out, dout, lse, Tq, Tk, scale, causal, key_mask=None):
    with torch.enable_grad():
        qf, kf, vf = (t.detach().float().requires_grad_(True) for t in (q[:, :, :Tq], k[:, :, :Tk], v[:, :, :Tk]))
        o, _ = _attention_f32(qf, kf, vf, Tq, Tk, scale, causal, key_mask)
        o.backward(dout.float())
    return qf.grad.to(q.dtype), kf.grad.to(k.dtype), vf.grad.to(v.dtype)


def _patch_attention_train(monkeypatch):
    from aria_b200 import ops
    standin_ops.patch(monkeypatch)
    monkeypatch.setattr(ops, "attention", _standin_attention)
    monkeypatch.setattr(ops, "attention_bwd", _standin_attention_bwd)


class _Stub(torch.nn.Module):
    is_causal = True
    num_key_value_groups = 1
    training = True


@pytest.fixture(autouse=True)
def _grad_enabled():
    with torch.enable_grad():      # other modules of the suite may have switched autograd off globally
        yield


@pytest.fixture(scope="module")
def lib():
    from aria_b200 import _lib, build
    build.build()
    return _lib.load()


def test_bwd_workspace_formula(lib):
    # fp32 dQ accumulator (128 wide) + lse and rowsum(dO*O), query rows padded to the 64-row step
    assert lib.aria_attention_bwd_workspace_bytes(8, 20, 2048, 2048, 1) == 8 * 20 * 2048 * 130 * 4
    assert lib.aria_attention_bwd_workspace_bytes(2, 3, 300, 300, 1) == 2 * 3 * 320 * 130 * 4
    assert lib.aria_attention_bwd_workspace_bytes(1, 2, 100, 420, 1) == 1 * 2 * 128 * 130 * 4
    assert lib.aria_attention_bwd_workspace_bytes(0, 2, 100, 420, 1) == 0


def test_bwd_bad_arguments_are_errors_before_any_cuda_call(lib):
    fake = ctypes.c_void_p(0x10000)   # never dereferenced: validation fails first
    B, H, Tq, Tk = 1, 2, 128, 128
    ws = lib.aria_attention_bwd_workspace_bytes(B, H, Tq, Tk, 1)
    st = (H * Tq * 128, Tq * 128, H * Tk * 128, Tk * 128)

    def call(q=fake, lse=fake, Tq_=Tq, Tk_=Tk, strides=st, causal=1, ws_bytes=ws, workspace=fake):
        return lib.aria_attention_bwd(q, fake, fake, fake, fake, lse, fake, fake, fake, None, B, H, Tq_, Tk_, *strides, 0.088,
                                      causal, workspace, ws_bytes, None)

    assert call(q=None) == -1                                     # null pointers
    assert call(lse=None) == -1
    assert call(workspace=None) == -1
    assert call(ws_bytes=ws - 1) == -1                            # workspace too small
    assert call(Tq_=256, Tk_=128,
                ws_bytes=lib.aria_attention_bwd_workspace_bytes(B, H, 256, 128, 1)) == -1   # causal needs Tk >= Tq
    assert call(strides=(st[0] + 4, st[1], st[2], st[3])) == -1    # strides must keep rows 16-byte aligned
    assert call(strides=(st[0], st[1], st[2], st[3] + 2)) == -1
    assert call(q=ctypes.c_void_p(0x10008)) == -1                  # misaligned base pointer
    # the forward with lse: a null lse is an argument error too
    assert lib.aria_attention_fwd_lse(fake, fake, fake, fake, None, None, B, H, Tq, Tk, *st, 128, 0.088, 1, None, 0, None) == -1


def _qkv(B, H, Tq, Tk, seed=0, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(B, H, T, 128, generator=g).to(dtype) for T in (Tq, Tk, Tk)]


def _reference_grads(q, k, v, dout, Tq, Tk, key_mask=None):
    """fp32 autograd of eager attention on the same bf16 inputs."""
    qf, kf, vf = (t.float().requires_grad_(True) for t in (q, k, v))
    o, _ = _attention_f32(qf, kf, vf, Tq, Tk, 128 ** -0.5, True, key_mask)
    o.backward(dout.float().reshape(o.shape))
    return qf.grad, kf.grad, vf.grad


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30))


@pytest.mark.parametrize("use_checkpoint", [False, True])
def test_seam_backward_through_hf_views(monkeypatch, use_checkpoint):
    _patch_attention_train(monkeypatch)
    B, H, Tq, Tk = 2, 2, 24, 24
    q, k, v = _qkv(B, H, Tq, Tk)
    # HF hands the core transposed (non-contiguous) query / key / value views of [B, T, H, hd] projections
    leaves = [t.transpose(1, 2).contiguous().requires_grad_(True) for t in (q, k, v)]
    dout = torch.randn(B, Tq, H, 128, generator=torch.Generator().manual_seed(1)).bfloat16()

    def core(qh, kh, vh):
        out, w = hf_attention.aria_b200_attention_forward(_Stub(), qh.transpose(1, 2), kh.transpose(1, 2), vh.transpose(1, 2),
                                                          None, scaling=128 ** -0.5)
        assert w is None
        return out

    out = checkpoint(core, *leaves, use_reentrant=False) if use_checkpoint else core(*leaves)
    assert out.shape == (B, Tq, H, 128)
    out.backward(dout)
    want = _reference_grads(q, k, v, dout, Tq, Tk)
    for leaf, w in zip(leaves, want):
        assert leaf.grad is not None and leaf.grad.shape == (B, Tq, H, 128)
        assert _rel(leaf.grad.transpose(1, 2), w) <= 2e-2


def test_padding_mask_reaches_the_backward_as_key_mask(monkeypatch):
    _patch_attention_train(monkeypatch)
    seen = {}
    from aria_b200 import ops
    inner = ops.attention_bwd

    def spy(*a, key_mask=None, **kw):
        seen["key_mask"] = key_mask
        return inner(*a, key_mask=key_mask, **kw)

    monkeypatch.setattr(ops, "attention_bwd", spy)
    B, H, T = 2, 2, 16
    q, k, v = (t.requires_grad_(True) for t in _qkv(B, H, T, T, seed=2))
    mask = torch.ones(B, T, dtype=torch.long)
    mask[1, :5] = 0                                               # left-padded second sequence
    out, _ = hf_attention.aria_b200_attention_forward(_Stub(), q, k, v, mask, scaling=128 ** -0.5)
    out.float().sum().backward()
    assert torch.equal(seen["key_mask"], (mask == 0).to(torch.uint8))
    key_mask = (mask == 0).to(torch.uint8)
    want = _reference_grads(q.detach(), k.detach(), v.detach(), torch.ones(B, T, H, 128), T, T, key_mask)
    for got, w in zip((q.grad, k.grad, v.grad), want):
        assert torch.isfinite(got.float()).all()
        assert _rel(got, w) <= 2e-2
    assert not k.grad[1, :, :5].any() and not v.grad[1, :, :5].any()     # masked keys get no gradient
    assert not q.grad[1, :, :5].any()                                    # query rows that see no key give none either


def test_decode_under_grad_and_cpu_tensors_still_raise(monkeypatch):
    q = torch.zeros(1, 2, 1, 128, dtype=torch.bfloat16, requires_grad=True)
    kv = torch.zeros(1, 2, 8, 128, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="decode"):
        hf_attention.aria_b200_attention_forward(_Stub(), q, kv, kv, None)
    q4 = torch.zeros(1, 2, 4, 128, dtype=torch.bfloat16, requires_grad=True)
    with pytest.raises(RuntimeError):                             # no CPU path: the real ops refuse CPU tensors
        hf_attention.aria_b200_attention_forward(_Stub(), q4, q4.detach(), q4.detach(), None)
    with pytest.raises(NotImplementedError):                      # dropout still refused
        hf_attention.aria_b200_attention_forward(_Stub(), q4, q4.detach(), q4.detach(), None, dropout=0.1)
