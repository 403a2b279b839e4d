"""Edges of the prefill attention pipeline (csrc/attention.cu): the K/V ring's prologue and epilogue at 1-5 key blocks,
key tails, a last query tile whose second warpgroup has no live rows, causal diagonal blocks with pos_off > 0, the uint8 key
mask, rows that see no key, and the projector's cross-attention shape.  Head dim 72 runs the 80-column path (SW128 chunk +
SW32 tile), head dim 128 the full-width one."""
import pytest
import torch

pytestmark = pytest.mark.gpu

REL = 1e-2
DEV = "cuda"


def rel_inf(got, want):
    got, want = got.float().cpu(), want.float().cpu()
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-12))


def _inputs(B, H, Tq, Tk, hd, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, H, Tq, 128, generator=g).bfloat16()
    k = torch.randn(B, H, Tk, 128, generator=g).bfloat16()
    v = torch.randn(B, H, Tk, 128, generator=g).bfloat16()
    for t in (q, k, v):
        t[..., hd:] = 0
    return q, k, v, g


def _check(q, k, v, Tq, Tk, hd, causal, km=None):
    """Against exact fp32 attention on the same bf16 inputs within REL, and against the oracle (transformers' eager attention,
    which rounds S and P to bf16 on the way) within 2.5 x REL, as the full-image ViT test states it; `out` of the LSE entry
    is bit-identical and lse within 1e-3 of torch.logsumexp."""
    from aria_b200 import ops
    from oracle import aria_oracle as O
    B, H = q.shape[:2]
    add = O.causal_additive_mask(Tq, Tk, torch.bfloat16) if causal else None
    if km is not None:
        add = torch.zeros(B, 1, 1, Tk, dtype=torch.bfloat16).masked_fill_(km[:, None, None, :], float("-inf"))
    want = O.attention_core(q, k, v, hd ** -0.5, add)[..., :hd].reshape(B, Tq, H * hd)
    s = (q[..., :hd].float() @ k[..., :hd].float().transpose(2, 3)) * hd ** -0.5
    if causal:
        s = s + O.causal_additive_mask(Tq, Tk, torch.float32)
    if km is not None:
        s = s.masked_fill(km[:, None, None, :], float("-inf"))
    exact = (s.softmax(-1) @ v[..., :hd].float()).transpose(1, 2).reshape(B, Tq, H * hd)
    kmd = None if km is None else km.to(torch.uint8).to(DEV)
    qd, kd, vd = q.to(DEV), k.to(DEV), v.to(DEV)
    got = ops.attention(qd, kd, vd, Tq, Tk, hd ** -0.5, causal, out_hd=hd, key_mask=kmd)
    out_lse, lse = ops.attention(qd, kd, vd, Tq, Tk, hd ** -0.5, causal, out_hd=hd, key_mask=kmd, return_lse=True)
    assert torch.equal(got, out_lse)
    assert rel_inf(got, exact) <= REL, rel_inf(got, exact)
    assert rel_inf(got, want) <= 2.5 * REL, rel_inf(got, want)
    assert torch.allclose(lse.cpu(), torch.logsumexp(s, -1), atol=1e-3, rtol=0)


# n_kv = 1..5 key blocks, each with a key tail except 256 and 512; Tq = 164 leaves a 36-row last query tile
@pytest.mark.parametrize("hd", [72, 128])
@pytest.mark.parametrize("Tk", [91, 256, 300, 512, 600])
def test_full_attention_key_blocks(hd, Tk):
    q, k, v, _ = _inputs(1, 2, 164, Tk, hd, seed=Tk + hd)
    _check(q, k, v, 164, Tk, hd, False)


# causal: Tq = Tk (pos_off = 0) and Tq = Tk - 50 (queries at the end of a longer key range)
@pytest.mark.parametrize("hd", [72, 128])
@pytest.mark.parametrize("Tk", [91, 256, 300, 512, 600])
@pytest.mark.parametrize("suffix", [False, True])
def test_causal_attention_key_blocks(hd, Tk, suffix):
    Tq = Tk - 50 if suffix else Tk
    q, k, v, _ = _inputs(1, 2, Tq, Tk, hd, seed=3 * Tk + hd + suffix)
    _check(q, k, v, Tq, Tk, hd, True)


@pytest.mark.parametrize("hd", [72, 128])
def test_key_mask_and_rows_without_keys(hd):
    """Batch 0 masks 30 % of the keys; batch 1 masks every key, so its rows see none: output 0, lse -inf."""
    from aria_b200 import ops
    B, H, Tq, Tk = 2, 2, 200, 333
    q, k, v, g = _inputs(B, H, Tq, Tk, hd, seed=hd)
    km = torch.rand(B, Tk, generator=g) < 0.3
    km[0, 0] = False
    km[1] = True
    _check(q[:1], k[:1], v[:1], Tq, Tk, hd, False, km[:1])
    out, lse = ops.attention(q.to(DEV), k.to(DEV), v.to(DEV), Tq, Tk, hd ** -0.5, False, out_hd=hd,
                             key_mask=km.to(torch.uint8).to(DEV), return_lse=True)
    assert torch.all(out[1] == 0)
    assert torch.all(torch.isneginf(lse[1]))


@pytest.mark.parametrize("masked", [False, True])
def test_projector_cross_attention_shape(masked):
    """The projector's cross-attention: 256 queries x 4900 keys (39 key blocks, a 36-key tail), 16 heads of 72."""
    B, H, Tq, Tk, hd = 1, 16, 256, 4900, 72
    q, k, v, _ = _inputs(B, H, Tq, Tk, hd, seed=256)
    km = None
    if masked:
        valid = torch.zeros(70, 70, dtype=torch.bool)
        valid[:52, :52] = True
        km = (~valid).reshape(1, Tk)
    _check(q, k, v, Tq, Tk, hd, False, km)
