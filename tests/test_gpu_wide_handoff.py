"""The hand-off epilogue of gemm_wide_kernel (gemm.cu): without a residual, the consumer warpgroups write bias + rounding into
their output half and go on to the next tile, and the producer warpgroup's warps 1-3 apply the activation and store (LINEAR)
or scatter (HEADS) the half, signalled through the out_full / out_free barriers.  Every output must still equal, bit for
bit, the same GEMM on 128-row slices (the 128-wide gemm_kernel), as in test_gpu_dense_wide.py.  Covered here: launches
with ~27 tiles per CTA, so both barriers go through many phases; the smallest launches the wide kernel takes (2,048 rows,
one n-tile) and launches where no CTA gets a second tile; CTA pairs without a residual, phantom tile included; HEADS over
several images; and a CUDA graph that alternates GELU, plain, HEADS and residual launches on the same buffers."""
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


def _act(name):
    from aria_b200 import _lib as L
    return {"none": L.ACT_NONE, "tanh": L.ACT_GELU_TANH, "new": L.ACT_GELU_NEW}[name]


def _linear_ref(x, w, b=None, act="none", r=None):
    from aria_b200 import ops
    return _sliced(lambda i, j: ops.linear(x[i:j], w, b, act=_act(act), residual=None if r is None else r[i:j]),
                   x.shape[0])


def _heads_ref(x, w, b, B, T, hd):
    return _linear_ref(x, w, b).view(B, T, -1, hd).transpose(1, 2)


@pytest.mark.parametrize("M,N,K,bias,act", [
    (4 * 4900, 4304, 1152, True, "tanh"),  # 154 m-tiles x 23 n-tiles: ~27 tiles per CTA, and the 80-column tail
    (4 * 4900, 1152, 1152, False, "none"),  # the same without activation: the store right after the hand-off
    (PAIR_MIN_ROWS, 64, 1152, True, "tanh"),  # the smallest launch: one 64-column n-tile, 16 tiles
    (PAIR_MIN_ROWS, 192, 1152, True, "new"),  # one whole n-tile, op-by-op GELU
    (PAIR_MIN_ROWS + 36, 1152, 1152, True, "tanh"),  # 102 tiles, at most one per CTA; the last m-tile has one warpgroup
    (4900, 960, 4304, True, "tanh"),  # CTA pairs without a residual: 5 n-tiles, so the last pair has a phantom tile
])
def test_handoff_linear_equals_slices(M, N, K, bias, act):
    from aria_b200 import ops
    x = _rand(M, K, seed=1)
    w = _rand(N, K, scale=K ** -0.5, seed=2)
    b = _rand(N, seed=3) if bias else None
    got = ops.linear(x, w, b, act=_act(act))
    want = _linear_ref(x, w, b, act)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


@pytest.mark.parametrize("B,T,pos0,n_seg", [
    (4, 4900, 0, 3),  # four images of 4,900 patches: 154 m-tiles, batch boundaries inside tiles, many tiles per CTA
    (3, 700, 2, 1),   # 2,100 rows, at most one tile per CTA, token offset
])
def test_handoff_heads_equal_sliced_linear(B, T, pos0, n_seg):
    from aria_b200 import ops
    N, K, hd, ld, T_max = 1152, 1152, 72, 128, T + pos0 + 3
    H = N // hd
    x = _rand(B * T, K, seed=1)
    ws = [_rand(N, K, scale=K ** -0.5, seed=2 + s) for s in range(n_seg)]
    bs = [_rand(N, seed=5 + s) for s in range(n_seg)]
    outs = [torch.full((B, H, T_max, ld), 7.0, dtype=BF16, device="cuda") for _ in range(n_seg)]
    ops.qkv_heads(x, ws, bs, outs, hd, T, pos0=pos0)
    torch.cuda.synchronize()
    for o, w, b in zip(outs, ws, bs):
        assert torch.equal(o[:, :, pos0:pos0 + T, :hd], _heads_ref(x, w, b, B, T, hd))
        assert bool((o[:, :, pos0:pos0 + T, hd:] == 7.0).all())
        assert bool((o[:, :, :pos0] == 7.0).all()) and bool((o[:, :, pos0 + T:] == 7.0).all())


def test_handoff_alternating_launches_in_one_graph():
    """GELU, HEADS, residual, plain and GELU-new launches back to back in one graph, each reading the previous one's output
    and writing into the same two row-major buffers and the same heads buffer; replayed twice."""
    from aria_b200 import ops
    M, d, hd, ld = 4900, 1152, 72, 128
    H = d // hd
    x = _rand(M, d, seed=1)
    w = [_rand(d, d, scale=d ** -0.5, seed=10 + i) for i in range(6)]
    b = [_rand(d, seed=20 + i) for i in range(6)]
    y1 = torch.empty(M, d, dtype=BF16, device="cuda")
    y2 = torch.empty(M, d, dtype=BF16, device="cuda")
    heads = torch.full((1, H, M, ld), 7.0, dtype=BF16, device="cuda")

    def step():
        ops.linear(x, w[0], b[0], act=_act("tanh"), out=y1)
        ops.qkv_heads(y1, [w[1]], [b[1]], [heads], hd, M)
        ops.linear(y1, w[2], b[2], residual=x, out=y2)
        ops.linear(y2, w[3], None, out=y1)
        ops.linear(y1, w[4], b[4], act=_act("new"), out=y2)
        ops.qkv_heads(y2, [w[5]], [b[5]], [heads], hd, M)

    # reference: the same chain on 128-row slices, eagerly
    r1 = _linear_ref(x, w[0], b[0], "tanh")
    r2 = _linear_ref(r1, w[2], b[2], r=x)
    r1 = _linear_ref(r2, w[3])
    r2 = _linear_ref(r1, w[4], b[4], "new")
    rh = _heads_ref(r2, w[5], b[5], 1, M, hd)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    for _ in range(2):
        y1.zero_()
        y2.zero_()
        heads.fill_(7.0)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(y1, r1)
        assert torch.equal(y2, r2)
        assert torch.equal(heads[..., :hd], rh)
        assert bool((heads[..., hd:] == 7.0).all())
