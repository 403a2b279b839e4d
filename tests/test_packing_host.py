"""CPU: padding-free packing.  `packing.pack_batch` on padded batches, the C-ABI argument checks of the varlen attention entries,
and the host logic of the `hf_attention` seam for packed calls (routing, boundary reads, refusals) with torch-CPU stand-ins for
the GPU ops.  The GPU suite runs the same scenarios on the kernels (tests/test_gpu_packed_attention.py)."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import standin_ops
from aria_b200 import hf_attention
from aria_b200.packing import pack_batch
from hf_common import tiny_hf_aria, tiny_inputs

SCALE = 128 ** -0.5


@pytest.fixture(autouse=True)
def _grad_enabled():
    with torch.enable_grad():
        yield


# ------------------------------------------------------------------------------------------------ pack_batch
def _padded(lens, T, left=False, seed=0):
    g = torch.Generator().manual_seed(seed)
    B = len(lens)
    ids = torch.zeros(B, T, dtype=torch.long)
    am = torch.zeros(B, T, dtype=torch.long)
    for b, n in enumerate(lens):
        sl = slice(T - n, T) if left else slice(0, n)
        ids[b, sl] = torch.randint(10, 500, (n,), generator=g)
        am[b, sl] = 1
    labels = ids.masked_fill(am == 0, -100)
    return ids, am, labels


@pytest.mark.parametrize("left", [False, True])
def test_pack_batch_fields(left):
    lens = [5, 9, 3]
    ids, am, labels = _padded(lens, 9, left=left)
    labels[1, 2] = -100                                             # an unlabelled token inside an example stays unlabelled
    out = pack_batch({"input_ids": ids, "attention_mask": am, "labels": labels}, return_flash_attn_kwargs=True)
    real = [ids[b][am[b].bool()] for b in range(3)]
    assert torch.equal(out["input_ids"], torch.cat(real)[None])
    assert out["position_ids"].tolist() == [list(range(5)) + list(range(9)) + list(range(3))]
    want_labels = torch.cat([labels[b][am[b].bool()] for b in range(3)])
    want_labels[[0, 5, 14]] = -100                                  # first label of every example
    assert torch.equal(out["labels"], want_labels[None])
    assert out["cu_seq_lens_q"].dtype == torch.int32 and out["cu_seq_lens_q"].tolist() == [0, 5, 14, 17]
    assert out["cu_seq_lens_k"].tolist() == [0, 5, 14, 17]
    assert out["max_length_q"] == out["max_length_k"] == 9
    assert "attention_mask" not in out


def test_pack_batch_single_example_and_no_labels():
    ids, am, _ = _padded([7], 7)
    out = pack_batch({"input_ids": ids, "attention_mask": am})
    assert torch.equal(out["input_ids"], ids) and out["position_ids"].tolist() == [list(range(7))]
    assert "labels" not in out
    # by default only what a fixed-signature forward (the reference recipe's model) accepts: no flash-attention kwargs
    assert set(out) == {"input_ids", "position_ids"}
    out = pack_batch({"input_ids": ids, "attention_mask": am}, return_flash_attn_kwargs=True)
    assert out["cu_seq_lens_q"].tolist() == [0, 7] and out["max_length_q"] == 7


def test_pack_batch_keeps_images_in_example_order():
    ids, am, labels = _padded([12, 6, 10], 12, seed=1)
    ids[0, 2:6] = 9                                                  # image tokens in examples 0 and 2
    ids[2, 1:5] = 9
    pv, pm = torch.randn(2, 3, 56, 56), torch.ones(2, 56, 56, dtype=torch.bool)
    out = pack_batch({"input_ids": ids, "attention_mask": am, "labels": labels, "pixel_values": pv, "pixel_mask": pm})
    assert out["pixel_values"] is pv and out["pixel_mask"] is pm
    pos = (out["input_ids"][0] == 9).nonzero().view(-1).tolist()
    assert pos == [2, 3, 4, 5, 19, 20, 21, 22]                       # example 0's image, then example 2's (starts at 18)


def test_pack_batch_rejects_holes_and_empty_rows():
    ids, am, _ = _padded([4, 4], 6)
    am[0, 1] = 0
    with pytest.raises(ValueError, match="contiguous"):
        pack_batch({"input_ids": ids, "attention_mask": am})
    am[0] = 0
    with pytest.raises(ValueError, match="no real token"):
        pack_batch({"input_ids": ids, "attention_mask": am})


# ------------------------------------------------------------------------------------------------ C ABI (no CUDA call)
@pytest.fixture(scope="module")
def lib():
    from aria_b200 import _lib, build
    build.build()
    return _lib.load()


def test_varlen_abi_bad_arguments(lib):
    fake = ctypes.c_void_p(0x10000)
    H, N, n_seg = 2, 300, 3
    ws = lib.aria_attention_bwd_varlen_workspace_bytes(n_seg, H, N)
    # dQ accumulator, lse2 and rowsum(dO*O) over N padded to the 64-row step plus one step, then the key-tile list
    assert ws == H * (320 + 64) * 130 * 4 + ((300 + 127) // 128 + n_seg) * 8
    assert lib.aria_attention_bwd_varlen_workspace_bytes(4, H, 3) == 0              # more segments than rows
    st = (N * 128, N * 128)

    def bwd(cu=fake, n=n_seg, N_=N, strides=st, ws_bytes=ws):
        return lib.aria_attention_bwd_varlen(fake, fake, fake, fake, fake, fake, fake, fake, fake, cu, n, H, N_, *strides, 0.088,
                                             fake, ws_bytes, None)

    assert bwd(cu=None) == -1
    assert bwd(ws_bytes=ws - 1) == -1
    assert bwd(n=N + 1) == -1
    assert bwd(strides=(N * 128 - 8, N * 128)) == -1                                 # a head must hold N rows
    assert bwd(strides=(N * 128 + 4, N * 128)) == -1                                 # 16-byte rows
    fwd = lib.aria_attention_fwd_varlen
    assert fwd(fake, fake, fake, fake, None, None, n_seg, H, N, *st, 0.088, None) == -1
    assert fwd(fake, fake, fake, fake, None, fake, 0, H, N, *st, 0.088, None) == -1
    assert fwd(fake, fake, fake, fake, ctypes.c_void_p(0x10002), fake, n_seg, H, N, *st, 0.088, None) == -1


# ------------------------------------------------------------------------------------------------ seam with stand-ins
def _attn_f32(q, k, v, scale):
    """fp32 causal attention of one sequence [1, H, T, 128] -> (out [T, H*128], lse [H, T])."""
    T = q.shape[2]
    w = torch.matmul(q.float(), k.float().transpose(2, 3)) * scale
    w = w.masked_fill(torch.ones(T, T, dtype=torch.bool).triu(1), float("-inf"))
    lse = torch.logsumexp(w, dim=-1)
    o = torch.matmul(torch.softmax(w, dim=-1), v.float())          # [1, H, T, 128]
    return o[0].transpose(0, 1).reshape(T, -1), lse[0]


def _standin_varlen(q, k, v, cu_seqlens, scale, return_lse=False, N=None):
    cu = cu_seqlens.tolist()
    parts = [_attn_f32(q[:, :, a:b], k[:, :, a:b], v[:, :, a:b], scale) for a, b in zip(cu, cu[1:])]
    out = torch.cat([p[0] for p in parts]).to(q.dtype)
    return (out, torch.cat([p[1] for p in parts], dim=1)) if return_lse else out


def _standin_varlen_bwd(q, k, v, out, dout, lse, cu_seqlens, scale, N=None):
    with torch.enable_grad():
        qf, kf, vf = (t.detach().float().requires_grad_(True) for t in (q, k, v))
        o = _standin_varlen(qf, kf, vf, cu_seqlens, scale).float()
        o.backward(dout.float().reshape(o.shape))
    return qf.grad.to(q.dtype), kf.grad.to(k.dtype), vf.grad.to(v.dtype)


def _standin_attention(q, k, v, Tq, Tk, scale, causal, out_hd=128, key_mask=None, return_lse=False):
    if not return_lse:
        return standin_ops.attention(q, k, v, Tq, Tk, scale, causal, out_hd=out_hd, key_mask=key_mask)
    B, H = q.shape[:2]
    w = torch.matmul(q[:, :, :Tq].float(), k[:, :, :Tk].float().transpose(2, 3)) * scale
    dead = torch.arange(Tk)[None, :] > torch.arange(Tk - Tq, Tk)[:, None] if causal else torch.zeros(Tq, Tk, dtype=torch.bool)
    dead = dead[None, None] | (key_mask.bool()[:, None, None, :] if key_mask is not None else False)
    w = w.masked_fill(dead, float("-inf"))
    o = torch.matmul(torch.nan_to_num(torch.softmax(w, dim=-1)), v[:, :, :Tk].float()).transpose(1, 2)
    return o.reshape(B, Tq, H * 128).to(q.dtype), torch.logsumexp(w, dim=-1)


def _standin_attention_bwd(q, k, v, out, dout, lse, Tq, Tk, scale, causal, key_mask=None):
    with torch.enable_grad():
        qf, kf, vf = (t.detach().float().requires_grad_(True) for t in (q, k, v))
        o, _ = _standin_attention(qf, kf, vf, Tq, Tk, scale, causal, key_mask=key_mask, return_lse=True)
        o.float().backward(dout.float().reshape(o.shape))
    return qf.grad.to(q.dtype), kf.grad.to(k.dtype), vf.grad.to(v.dtype)


@pytest.fixture
def calls(monkeypatch):
    """Stand-ins for every attention op the seam reaches, recording which ran."""
    from aria_b200 import ops
    standin_ops.patch(monkeypatch)
    seen = []

    def spy(name, fn):
        def wrapped(*a, **kw):
            seen.append(name)
            return fn(*a, **kw)
        monkeypatch.setattr(ops, name, wrapped)

    spy("attention", _standin_attention)
    spy("attention_bwd", _standin_attention_bwd)
    spy("attention_varlen", _standin_varlen)
    spy("attention_varlen_bwd", _standin_varlen_bwd)
    spy("attention_decode", standin_ops.attention_decode)
    monkeypatch.setattr(hf_attention, "_READS", [])
    monkeypatch.setattr(hf_attention, "_DEVICE_CU", {})
    monkeypatch.setattr(hf_attention, "_device_cu", lambda src, cu, like=None: torch.tensor(cu, dtype=torch.int32))
    return seen


class _Stub(torch.nn.Module):
    is_causal = True
    num_key_value_groups = 1
    training = False


def _qkv(B, H, T, seed=0, grad=False):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(B, H, T, 128, generator=g).bfloat16().requires_grad_(grad) for _ in range(3)]


def _core(q, k, v, mask=None, **kw):
    return hf_attention.aria_b200_attention_forward(_Stub(), q, k, v, mask, scaling=SCALE, **kw)[0]


def test_routing(calls):
    q, k, v = _qkv(1, 2, 12)
    _core(q, k, v, position_ids=torch.arange(12)[None])                           # one run: today's path
    _core(q, k, v, position_ids=torch.arange(3, 15)[None])                        # one run from an offset: today's path
    _core(q, k, v)                                                                # no positions: today's path
    assert calls == ["attention"] * 3
    calls.clear()
    pos = torch.cat([torch.arange(7), torch.arange(5)])[None]
    out = _core(q, k, v, position_ids=pos)
    assert calls == ["attention_varlen"]
    for a, b in ((0, 7), (7, 12)):                                                # each sequence on its own
        alone = _core(q[:, :, a:b], k[:, :, a:b], v[:, :, a:b])                 # (stand-ins round differently: 1 bf16 ulp)
        assert torch.allclose(out[:, a:b].float(), alone.float(), rtol=1e-2, atol=1e-2)
    calls.clear()
    cu = torch.tensor([0, 7, 12], dtype=torch.int32)
    assert torch.equal(_core(q, k, v, cu_seq_lens_q=cu, cu_seq_lens_k=cu), out)
    assert calls == ["attention_varlen"]
    calls.clear()
    q2, k2, v2 = _qkv(2, 2, 12)                                                   # padded batch keeps the key-mask path
    am = torch.ones(2, 12, dtype=torch.long)
    am[1, 9:] = 0
    _core(q2, k2, v2, am, position_ids=torch.arange(12)[None].expand(2, 12))
    _core(q2[:, :, :1], k2, v2, None, position_ids=torch.tensor([[12], [3]]))     # decode: positions are never read
    assert calls == ["attention", "attention_decode"]


def test_boundaries_read_once_across_layers_and_recompute(calls):
    q, k, v = _qkv(1, 2, 12, grad=True)
    pos = torch.cat([torch.arange(4), torch.arange(8)])[None]
    before = hf_attention.reads

    def layer(q_, k_, v_):
        return _core(q_, k_, v_, position_ids=pos)

    from torch.utils.checkpoint import checkpoint
    outs = [checkpoint(layer, q, k, v, use_reentrant=False) for _ in range(4)]    # four "layers", each recomputed once
    torch.stack(outs).float().sum().backward()
    assert hf_attention.reads - before == 1
    assert calls.count("attention_varlen") == 8 and calls.count("attention_varlen_bwd") == 4
    cu = torch.tensor([0, 4, 12], dtype=torch.int32)
    for _ in range(3):
        _core(q.detach(), k.detach(), v.detach(), cu_seq_lens_q=cu, cu_seq_lens_k=cu)
    assert hf_attention.reads - before == 2                                       # one tensor, one read
    pos.add_(0)                                                                   # an in-place write: read again
    _core(q.detach(), k.detach(), v.detach(), position_ids=pos)
    assert hf_attention.reads - before == 3


def test_refusals_before_any_kernel(calls):
    q, k, v = _qkv(1, 2, 12)
    pos = torch.cat([torch.arange(7), torch.arange(5)])[None]
    q2, k2, v2 = _qkv(2, 2, 12)
    with pytest.raises(NotImplementedError, match="batch size 1"):
        _core(q2, k2, v2, position_ids=pos.expand(2, 12))
    with pytest.raises(NotImplementedError, match="cache"):
        _core(q[:, :, 4:], k, v, position_ids=pos[:, 4:])                         # queries after a cache prefix
    cu = torch.tensor([0, 7, 12], dtype=torch.int32)
    with pytest.raises(NotImplementedError, match="cache"):
        _core(q[:, :, 8:], k, v, cu_seq_lens_q=cu, cu_seq_lens_k=cu)
    with pytest.raises(ValueError, match="equal"):
        _core(q, k, v, cu_seq_lens_q=cu, cu_seq_lens_k=torch.tensor([0, 6, 12], dtype=torch.int32))
    for bad in ([0, 7, 11], [1, 7, 12], [0, 7, 7, 12], [0, 9, 7, 12], [0]):
        with pytest.raises(ValueError, match="boundaries"):
            t = torch.tensor(bad, dtype=torch.int32)
            _core(q, k, v, cu_seq_lens_q=t, cu_seq_lens_k=t)
    with pytest.raises(ValueError, match="boundaries"):
        _core(q, k, v, position_ids=torch.cat([torch.arange(1, 8), torch.arange(5)])[None])   # first position is not 0
    assert calls == []


def _hf_aria_packed_vs_padded(use_checkpoint):
    """Tiny HF Aria trained on three examples as a right-padded batch in fp32 eager, and packed through the seam."""
    ids, pv, pm = tiny_inputs(batch=1, n_text=20)
    g = torch.Generator().manual_seed(5)
    lens = [28, 17, 23]
    T = max(lens)
    rows = torch.zeros(3, T, dtype=torch.long)
    am = torch.zeros(3, T, dtype=torch.long)
    rows[0, :28] = ids[0]
    for b, n in ((1, 17), (2, 23)):
        rows[b, :n] = torch.randint(10, 512, (n,), generator=g)
        am[b, :n] = 1
    am[0] = 1
    labels = rows.masked_fill(am == 0, -100).masked_fill(rows == 9, -100)
    batch = {"input_ids": rows, "attention_mask": am, "labels": labels, "pixel_values": pv, "pixel_mask": pm}

    def run(packed):
        model = tiny_hf_aria(dtype=torch.float32)
        for m in model.modules():
            c = getattr(m, "config", None)
            if c is not None and hasattr(c, "moe_topk"):
                c.moe_topk = c.moe_num_experts
        for n, p in model.named_parameters():
            p.requires_grad_(not ("vision_tower" in n or "multi_modal_projector" in n))
        model.train()
        if packed:
            key = hf_attention.register()
            model.config.text_config._attn_implementation = key
            model.model.language_model.config._attn_implementation = key
            if use_checkpoint:
                model.gradient_checkpointing_enable(gradient_checkpointing_kwargs={"use_reentrant": False})
        inputs = pack_batch(batch) if packed else batch
        if packed:
            assert inputs["input_ids"].shape == (1, sum(lens))
        loss = model(**inputs).loss
        loss.backward()
        return loss.detach(), {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}

    return run(False), run(True)


@pytest.mark.parametrize("use_checkpoint", [False, True])
def test_tiny_hf_aria_packed_matches_padded(calls, use_checkpoint):
    (want_loss, want), (got_loss, got) = _hf_aria_packed_vs_padded(use_checkpoint)
    assert "attention_varlen" in calls and "attention_varlen_bwd" in calls and "attention" not in calls
    assert abs(float(got_loss) - float(want_loss)) <= 2e-2 * abs(float(want_loss))
    assert got.keys() == want.keys() and got
    for n in want:
        e = float((got[n] - want[n]).norm() / want[n].norm().clamp_min(1e-30))
        assert e <= 2e-2, (n, e)
