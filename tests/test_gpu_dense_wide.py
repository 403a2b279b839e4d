"""Dense GEMMs of at least PAIR_MIN_ROWS rows run on the 128 x 192 tile kernel whose epilogue works on the accumulator
registers (gemm_wide_kernel, gemm.cu).  Its outputs must equal, bit for bit, the same GEMM computed on 128-row slices, which
take the 128-wide gemm_kernel: the per-element arithmetic, rounding points and k order are the same.  Covers the ViT and
projector shapes, bias +- GELU (tanh and op-by-op) +- residual, the 80-column tail tile of N = 4304, M tails (4,900 rows: the
last m-tile has 36 rows, so its second warpgroup has none; threshold + 70 rows), several weights in one launch, and the q/k/v
head scatter at every batch and token offset with the pad columns left untouched."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
PAIR_MIN_ROWS = 2048  # gemm.cu: fewest rows that take the wide kernel
SLICE = 128


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(BF16)


def _sliced(fn, M):
    return torch.cat([fn(i, min(M, i + SLICE)) for i in range(0, M, SLICE)])


@pytest.mark.parametrize("M,N,K,bias,act,residual", [
    (4900, 1152, 1152, True, "none", True),    # ViT o_proj
    (4900, 1152, 4304, True, "none", True),    # ViT fc2
    (4900, 4304, 1152, True, "tanh", False),   # ViT fc1: 22 whole tiles and an 80-column tail
    (4900, 1152, 1152, False, "none", False),  # projector k / v
    (4900, 4304, 1152, False, "new", True),    # GELU-new, residual without bias, column tail
    (PAIR_MIN_ROWS + 70, 1152, 1152, True, "tanh", True),  # a 70-row last m-tile: the second warpgroup has 6 rows
    (PAIR_MIN_ROWS, 256, 512, True, "none", False),        # one whole tile and a 64-column one
])
def test_wide_linear_equals_slices(M, N, K, bias, act, residual):
    from aria_b200 import _lib as L
    from aria_b200 import ops
    a = {"none": L.ACT_NONE, "tanh": L.ACT_GELU_TANH, "new": L.ACT_GELU_NEW}[act]
    x = _rand(M, K, seed=1)
    w = _rand(N, K, scale=K ** -0.5, seed=2)
    b = _rand(N, seed=3) if bias else None
    r = _rand(M, N, seed=4) if residual else None
    got = ops.linear(x, w, b, act=a, residual=r)
    want = _sliced(lambda i, j: ops.linear(x[i:j], w, b, act=a, residual=None if r is None else r[i:j]), M)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_wide_linear_multi_equals_slices():
    from aria_b200 import ops
    M, N, K = 4900, 1152, 1152
    x = _rand(M, K, seed=1)
    ws = [_rand(N, K, scale=K ** -0.5, seed=2 + s) for s in range(3)]
    got = ops.linear_multi(x, ws)
    want = _sliced(lambda i, j: ops.linear_multi(x[i:j], ws), M)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


@pytest.mark.parametrize("B,T,pos0,n_seg,bias", [
    (1, 4900, 0, 3, True),    # ViT q/k/v: 16 heads of 72 in 128-wide rows
    (1, 4900, 0, 1, True),    # projector in-projection of k (or v)
    (2, 1100, 5, 3, False),   # batch boundary inside a tile, token offset, 2,200 rows
])
def test_wide_heads_equal_sliced_linear(B, T, pos0, n_seg, bias):
    from aria_b200 import ops
    N, K, hd, ld, T_max = 1152, 1152, 72, 128, T + pos0 + 3
    H = N // hd
    M = B * T
    x = _rand(M, K, seed=1)
    ws = [_rand(N, K, scale=K ** -0.5, seed=2 + s) for s in range(n_seg)]
    bs = [_rand(N, seed=5 + s) if bias else None for s in range(n_seg)]
    outs = [torch.full((B, H, T_max, ld), 7.0, dtype=BF16, device="cuda") for _ in range(n_seg)]
    ops.qkv_heads(x, ws, bs, outs, hd, T, pos0=pos0)
    torch.cuda.synchronize()
    for o, w, b in zip(outs, ws, bs):
        ref = _sliced(lambda i, j: ops.linear(x[i:j], w, b), M).view(B, T, H, hd).transpose(1, 2)
        assert torch.equal(o[:, :, pos0:pos0 + T, :hd], ref)
        assert bool((o[:, :, pos0:pos0 + T, hd:] == 7.0).all())
        assert bool((o[:, :, :pos0] == 7.0).all()) and bool((o[:, :, pos0 + T:] == 7.0).all())
