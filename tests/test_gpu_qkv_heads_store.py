"""qkv_heads without RoPE stores each head row from consecutive threads (heads_store_tile, gemm_common.cuh).  Its outputs must
equal, bit for bit, the same projection through `linear` (same 128-wide tiles, same bias add and rounding) scattered into the
head-major layout by torch, at every batch and token offset, and the pad columns past head_dim must stay untouched."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(BF16)


@pytest.mark.parametrize("B,T,pos0,K,bias", [
    (1, 4900, 0, 1152, True),   # the ViT layer: 16 heads of 72, M tail of 36 rows
    (3, 333, 5, 256, True),     # several batches, token offset, batch boundaries inside a tile
    (2, 200, 0, 512, False),
])
def test_heads_store_equals_linear_scattered(B, T, pos0, K, bias):
    from aria_b200 import ops
    N, hd, ld, T_max = 1152, 72, 128, T + pos0 + 3
    H = N // hd
    x = _rand(B * T, K, seed=1)
    ws = [_rand(N, K, scale=K ** -0.5, seed=2 + s) for s in range(3)]
    bs = [_rand(N, seed=5 + s) if bias else None for s in range(3)]
    outs = [torch.full((B, H, T_max, ld), 7.0, dtype=BF16, device="cuda") for _ in range(3)]
    ops.qkv_heads(x, ws, bs, outs, hd, T, pos0=pos0)
    torch.cuda.synchronize()
    for o, w, b in zip(outs, ws, bs):
        ref = ops.linear(x, w, b).view(B, T, H, hd).transpose(1, 2)
        assert torch.equal(o[:, :, pos0:pos0 + T, :hd], ref)
        assert bool((o[:, :, pos0:pos0 + T, hd:] == 7.0).all())
        assert bool((o[:, :, :pos0] == 7.0).all()) and bool((o[:, :, pos0 + T:] == 7.0).all())
