"""Dense LINEAR GEMMs that run as CTA pairs sharing their A tile (M >= PAIR_MIN_ROWS, gemm.cu) against the same GEMM computed
on 128-row slices, which take the one-CTA kernel: the pair changes only where A is loaded from, so every output must be equal
bit for bit.  Covers an odd n-tile count (the last pair's second tile is a phantom), M tails (4,900 rows: the last m-tile has
36 rows, so its second half lies wholly past the end; and threshold + 2 rows), bias + GELU, bias + residual, a single n-pair
per m-tile and more pairs than fit on the GPU at once.  The cfg-2 shapes are also checked against torch in fp32."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
PAIR_MIN_ROWS = 2048  # gemm.cu
SLICE = 128


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(BF16)


@pytest.mark.parametrize("M,N,K,bias,act,residual", [
    (4900, 1152, 1152, True, False, True),     # ViT o_proj: 9 n-tiles (phantom), M tail, more pairs than clusters
    (4900, 1152, 4304, True, False, True),     # ViT fc2
    (4900, 4304, 1152, True, True, False),     # ViT fc1: 34 n-tiles, column tail
    (PAIR_MIN_ROWS + 2, 4304, 1152, True, True, False),  # threshold + 2 rows: a 2-row last m-tile
    (PAIR_MIN_ROWS, 256, 512, False, False, False),      # one n-pair per m-tile
    (PAIR_MIN_ROWS, 128, 512, True, False, True),        # one n-pair whose second tile is a phantom
])
def test_linear_pairs_equal_slices(M, N, K, bias, act, residual):
    from aria_b200 import _lib as L
    from aria_b200 import ops
    x = _rand(M, K, seed=1)
    w = _rand(N, K, scale=K ** -0.5, seed=2)
    b = _rand(N, seed=3) if bias else None
    r = _rand(M, N, seed=4) if residual else None
    a = L.ACT_GELU_TANH if act else L.ACT_NONE
    got = ops.linear(x, w, b, act=a, residual=r)
    want = torch.empty_like(got)
    for i in range(0, M, SLICE):
        want[i:i + SLICE] = ops.linear(x[i:i + SLICE], w, b, act=a, residual=None if r is None else r[i:i + SLICE])
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def _close(got, want):
    err = float((got.float() - want).abs().max() / want.abs().max())
    assert err < 1e-2, err


def test_cfg2_vit_mlp_against_fp32():
    from aria_b200 import _lib as L
    from aria_b200 import ops
    M, d, I = 4900, 1152, 4304
    x, h = _rand(M, d, seed=20), _rand(M, I, seed=21)
    w1, b1 = _rand(I, d, scale=d ** -0.5, seed=22), _rand(I, seed=23)
    w2, b2 = _rand(d, I, scale=I ** -0.5, seed=24), _rand(d, seed=25)
    _close(ops.linear(x, w1, b1, act=L.ACT_GELU_TANH), F.gelu(F.linear(x.float(), w1.float(), b1.float()), approximate="tanh"))
    _close(ops.linear(h, w2, b2, residual=x), F.linear(h.float(), w2.float(), b2.float()) + x.float())
