"""The hand-off epilogue of gemm_kernel (gemm.cu, HANDOFF, launched as gemm_handoff_kernel): in grouped launches without a
residual, SwiGLU launches and HEADS launches with RoPE (bf16 weights, 128-wide tiles, one CTA) the consumer warpgroups write what the epilogue rounds first (bf16(x + bias), bf16(gate) | bf16(up), bf16(x) for RoPE) into a
bf16 output half and go on to the next tile, and the producer warpgroup's warps 1-3 finish and store it, signalled through
the out_full / out_free barriers.

Where an unchanged path computes the same sums in the same order the outputs must be equal bit for bit: a grouped LINEAR
launch against the same launch with a zero residual (the residual launches keep the staged epilogue), RoPE against the
LINEAR output rotated with the kernel's fp32 operations.  SwiGLU is held to the fp64 bars of tests/gemm_ref.py.  Covered:
grouped launches with many tiles per CTA (both barriers through many phases), group sizes at every residue mod 16 and
mod 128, empty groups, last m-tiles of 64 rows or fewer (the second warpgroup sits out), sentinel rows after every group's
end, per-group destinations, HEADS + RoPE with position_ids, pos0 > 0 and several sequences whose length is no multiple
of 128, and one CUDA graph that alternates SwiGLU, LINEAR, HEADS + RoPE and residual launches on the same buffers."""
import os
import re
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import gemm_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
SENTINEL = -3.0


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(BF16)


def _counts(E, seed, extra=()):
    """Group sizes: every residue mod 16 and mod 128 (0 included: empty groups), 1-64 (one warpgroup), 65-128, 129-300"""
    g = torch.Generator().manual_seed(seed)
    base = list(range(0, 129)) + [129, 143, 191, 192, 255, 256, 257, 300] + list(extra)
    pick = torch.randint(0, len(base), (E,), generator=g).tolist()
    return [base[i] for i in pick]


def _offsets(counts):
    off = torch.zeros(len(counts) + 1, dtype=torch.int32)
    off[1:] = torch.tensor(counts, dtype=torch.int32).cumsum(0)
    return off.cuda()


@pytest.mark.parametrize("E,K,N,seed", [
    (64, 256, 2560, 0),   # 20 n-tiles over ~4,000 rows: many tiles per CTA
    (48, 1664, 256, 1),   # 26 k-blocks, two n-tiles
    (8, 64, 128, 2),      # one k-block, one n-tile
])
def test_grouped_linear_equals_staged_epilogue(E, K, N, seed):
    from aria_b200 import ops
    counts = _counts(E, seed)
    off = _offsets(counts)
    rows = sum(counts)
    a = _rand(rows, K, seed=seed + 10)
    b = _rand(E, K, N, scale=K ** -0.5, seed=seed + 20)
    got = ops.grouped_gemm(a, b, off)
    want = ops.grouped_gemm(a, b, off, residual=torch.zeros(rows, N, dtype=BF16, device="cuda"))
    torch.cuda.synchronize()
    assert torch.equal(got, want)


@pytest.mark.parametrize("E,K,N,seed", [(64, 512, 1664, 3), (16, 2560, 128, 4)])
def test_grouped_swiglu_fp64(E, K, N, seed):
    from aria_b200 import ops
    counts = _counts(E, seed)
    off = _offsets(counts)
    a = _rand(sum(counts), K, seed=seed + 10)
    b = _rand(E, K, 2 * N, scale=K ** -0.5, seed=seed + 20)
    got = ops.grouped_gemm(a, b, off, swiglu=True)
    torch.cuda.synchronize()
    z, ez = R.grouped_ref(a, b, off)
    y, ey = R.swiglu_ref(z[:, :N], ez[:, :N], z[:, N:], ez[:, N:])
    R.check(got, y, ey, "grouped SwiGLU")


@pytest.mark.parametrize("swiglu", [False, True])
def test_regions_leave_rows_past_each_group(swiglu):
    """Fixed-capacity regions: rows between a group's end and the next region are sentinels and must come back untouched"""
    from aria_b200 import ops
    E, K, N, cap = 32, 384, 640, 160
    counts = _counts(E, 5)
    counts = [min(c, cap) for c in counts]
    starts = torch.arange(E, dtype=torch.int32) * cap
    a = _rand(E * cap, K, seed=6)
    b = _rand(E, K, 2 * N if swiglu else N, scale=K ** -0.5, seed=7)
    out = torch.full((E * cap, N), SENTINEL, dtype=BF16, device="cuda")
    ops.grouped_gemm_regions(a, b, starts.cuda(), torch.tensor(counts, dtype=torch.int32).cuda(), sum(counts),
                             swiglu=swiglu, out=out)
    torch.cuda.synchronize()
    packed_off = _offsets(counts)
    rows = torch.cat([torch.arange(s, s + c) for s, c in zip(starts.tolist(), counts)]).cuda()
    a_packed = a[rows]
    if swiglu:
        z, ez = R.grouped_ref(a_packed, b, packed_off)
        y, ey = R.swiglu_ref(z[:, :N], ez[:, :N], z[:, N:], ez[:, N:])
        R.check(out[rows], y, ey, "regions SwiGLU")
    else:
        want = ops.grouped_gemm(a_packed, b, packed_off, residual=torch.zeros(len(rows), N, dtype=BF16, device="cuda"))
        assert torch.equal(out[rows], want)
    mask = torch.ones(E * cap, dtype=torch.bool, device="cuda")
    mask[rows] = False
    assert bool((out[mask] == SENTINEL).all())


def test_per_group_destinations():
    """out_group_base / out_group_row0: each group's rows land at their own buffer and row offset, nothing else is written"""
    from aria_b200 import ops
    E, K, N, cap = 24, 320, 384, 200
    counts = [min(c, cap) for c in _counts(E, 8)]
    starts = torch.arange(E, dtype=torch.int32) * cap
    a = _rand(E * cap, K, seed=9)
    b = _rand(E, K, N, scale=K ** -0.5, seed=10)
    slot = cap + 4
    dst = [torch.full((E // 3 * slot, N), SENTINEL, dtype=BF16, device="cuda") for _ in range(3)]
    row0 = [(g // 3) * slot + g % 4 for g in range(E)]
    base = torch.tensor([dst[g % 3].data_ptr() for g in range(E)], dtype=torch.int64, device="cuda")
    ops.grouped_gemm_regions(a, b, starts.cuda(), torch.tensor(counts, dtype=torch.int32, device="cuda"), sum(counts),
                             out_group_base=base, out_group_row0=torch.tensor(row0, dtype=torch.int32, device="cuda"), ldo=N)
    torch.cuda.synchronize()
    written = [torch.zeros(E // 3 * slot, dtype=torch.bool, device="cuda") for _ in range(3)]
    for g, c in enumerate(counts):
        if not c:
            continue
        s = g * cap
        want = ops.grouped_gemm(a[s:s + c], b[g:g + 1], _offsets([c]), residual=torch.zeros(c, N, dtype=BF16, device="cuda"))
        assert torch.equal(dst[g % 3][row0[g]:row0[g] + c], want), f"group {g}"
        written[g % 3][row0[g]:row0[g] + c] = True
    for d, w in zip(dst, written):
        assert bool((d[~w] == SENTINEL).all())


def _rope_bits(y, cos, sin):
    """The kernel's RoPE on bf16 y [..., 128] with bf16 table rows: each product of two bf16 values is exact in fp32 and
    rounded to bf16, the sum is taken in fp32 and rounded: out = bf16(bf16(y cos) + bf16(rotate_half(y) sin))"""
    yf, c, s = y.float(), cos.float(), sin.float()
    a = (yf * c).to(BF16).float()
    b = (R.rotate_half(yf) * s).to(BF16).float()
    return (a + b).to(BF16)


def _rope_table(n_pos):
    from aria_b200 import ops
    inv = 1.0 / (5e6 ** (torch.arange(0, 128, 2, device="cuda", dtype=torch.float32) / 128))
    return ops.rope_table(inv, n_pos)


@pytest.mark.parametrize("B,T,pos0,use_ids", [
    (1, 768, 0, False),   # the LM prefill: 6 m-tiles x 60 n-tiles
    (3, 300, 5, False),   # batch boundaries inside m-tiles, token offset, a 4-row last m-tile
    (2, 200, 0, True),    # position_ids; 400 rows, last m-tile of 16 rows
    (32, 1, 2047, True),  # decode: one token of 32 sequences
])
def test_heads_rope_equals_rotated_linear(B, T, pos0, use_ids):
    from aria_b200 import ops
    D, H, hd = 2560, 20, 128
    x = _rand(B * T, D, seed=11)
    ws = [_rand(D, D, scale=D ** -0.5, seed=12 + s) for s in range(3)]
    bv = _rand(D, seed=15)
    cos, sin = _rope_table(4096)
    T_max = pos0 + T + 3
    outs = [torch.full((B, H, T_max, hd), SENTINEL, dtype=BF16, device="cuda") for _ in range(3)]
    pos = None
    if use_ids:
        g = torch.Generator().manual_seed(16)
        pos = torch.randint(0, 4096, (B * T,), generator=g, dtype=torch.int32).cuda()
    ops.qkv_heads(x, ws, [None, None, bv], outs, hd, T, pos0=pos0, rope_mask=0b011, rope_cos=cos, rope_sin=sin,
                  position_ids=pos)
    torch.cuda.synchronize()
    p = pos.long() if use_ids else (pos0 + torch.arange(T, device="cuda")).repeat(B)
    for s in range(3):
        y = ops.linear(x, ws[s], bv if s == 2 else None)
        want = _rope_bits(y.view(B * T, H, hd), cos[p][:, None], sin[p][:, None]) if s < 2 else y.view(B * T, H, hd)
        got = outs[s][:, :, pos0:pos0 + T].permute(0, 2, 1, 3).reshape(B * T, H, hd)
        assert torch.equal(got, want), f"segment {s}"
        assert bool((outs[s][:, :, :pos0] == SENTINEL).all()) and bool((outs[s][:, :, pos0 + T:] == SENTINEL).all())


def test_alternating_launches_in_one_graph():
    """SwiGLU (dense and grouped), LINEAR, HEADS + RoPE and residual launches back to back in one graph on the same
    buffers, each reading the previous one's output; replayed twice against the same chain run eagerly"""
    from aria_b200 import ops
    T, D, I, E, H, hd = 768, 2560, 1664, 16, 20, 128
    x = _rand(T, D, seed=20)
    wg, wu = _rand(I, D, scale=D ** -0.5, seed=21), _rand(I, D, scale=D ** -0.5, seed=22)
    wd = _rand(D, I, scale=I ** -0.5, seed=23)
    wq = [_rand(D, D, scale=D ** -0.5, seed=24 + s) for s in range(3)]
    w1 = _rand(E, D, 2 * I, scale=D ** -0.5, seed=27)
    w2 = _rand(E, I, D, scale=I ** -0.5, seed=28)
    off = _offsets(_counts(E, 29)[:E - 1] + [0])
    rows = int(off[-1])
    xe = _rand(rows, D, seed=30)
    cos, sin = _rope_table(T + 8)
    h = torch.empty(T, I, dtype=BF16, device="cuda")
    y = torch.empty(T, D, dtype=BF16, device="cuda")
    kv = [torch.full((1, H, T + 8, hd), SENTINEL, dtype=BF16, device="cuda") for _ in range(3)]
    he = torch.empty(rows, I, dtype=BF16, device="cuda")
    ye = torch.empty(rows, D, dtype=BF16, device="cuda")

    def step():
        h.copy_(ops.linear_swiglu(x, wg, wu))
        y.copy_(ops.linear(h, wd))
        ops.qkv_heads(y, wq, [None] * 3, kv, hd, T, pos0=8, rope_mask=0b011, rope_cos=cos, rope_sin=sin)
        y.copy_(ops.linear(h, wd, residual=y))
        he.copy_(ops.grouped_gemm(xe, w1, off, swiglu=True))
        ye.copy_(ops.grouped_gemm(he, w2, off))
        h.copy_(ops.linear_swiglu(y, wg, wu))

    step()
    torch.cuda.synchronize()
    want = [t.clone() for t in (h, y, he, ye, *kv)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    for _ in range(2):
        for t in (h, y, he, ye):
            t.zero_()
        for t in kv:
            t.fill_(SENTINEL)
        g.replay()
        torch.cuda.synchronize()
        for got, ref in zip((h, y, he, ye, *kv), want):
            assert torch.equal(got, ref)


# ------------------------------------------------------------------------------------------------ which kernel runs
def _kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "gemm" in e.name]


def _lin(M, N, K, residual=False):
    from aria_b200 import ops
    x, w = _rand(M, K, seed=1), _rand(N, K, scale=K ** -0.5, seed=2)
    r = torch.zeros(M, N, dtype=BF16, device="cuda") if residual else None
    return lambda: ops.linear(x, w, residual=r)


def _swiglu(M, N, K):
    from aria_b200 import ops
    x = _rand(M, K, seed=1)
    wg, wu = _rand(N, K, scale=K ** -0.5, seed=2), _rand(N, K, scale=K ** -0.5, seed=3)
    return lambda: ops.linear_swiglu(x, wg, wu)


def _heads(M, K, Hn, hd, rope):
    from aria_b200 import ops
    x = _rand(M, K, seed=1)
    ws = [_rand(Hn * hd, K, scale=K ** -0.5, seed=2 + s) for s in range(3)]
    outs = [torch.empty(1, Hn, M, 128, dtype=BF16, device="cuda") for _ in range(3)]
    cos, sin = _rope_table(M)
    if rope:
        return lambda: ops.qkv_heads(x, ws, [None] * 3, outs, hd, M, rope_mask=0b011, rope_cos=cos, rope_sin=sin)
    return lambda: ops.qkv_heads(x, ws, [None] * 3, outs, hd, M)


def _grouped(swiglu, residual=False):
    from aria_b200 import ops
    E, K, N = 8, 256, 256
    off = _offsets(_counts(E, 40))
    rows = int(off[-1])
    a, b = _rand(rows, K, seed=1), _rand(E, K, 2 * N if swiglu else N, scale=K ** -0.5, seed=2)
    r = torch.zeros(rows, N, dtype=BF16, device="cuda") if residual else None
    return lambda: ops.grouped_gemm(a, b, off, swiglu=swiglu, residual=r)


# (what, launch, kernel-name pattern): gemm_handoff_kernel<B_MN, EPI>, gemm_kernel<BN, B_MN, EPI, B_FP8, PAIR>;
# the hand-off takes grouped launches without a residual, SwiGLU and HEADS with RoPE
# EPI 0 = LINEAR, 1 = SWIGLU, 2 = HEADS
PATHS = [
    ("dense LINEAR staged, M = 768", lambda: _lin(768, 2560, 3328), r"gemm_kernel<128, false, 0, false, false>"),
    ("dense SwiGLU hand-off", lambda: _swiglu(768, 1664, 2560), r"gemm_handoff_kernel<false, 1>"),
    ("heads without RoPE staged", lambda: _heads(300, 1152, 16, 72, False), r"gemm_kernel<128, false, 2, false, false>"),
    ("LM heads + RoPE hand-off", lambda: _heads(768, 2560, 20, 128, True), r"gemm_handoff_kernel<false, 2>"),
    ("grouped LINEAR hand-off", lambda: _grouped(False), r"gemm_handoff_kernel<true, 0>"),
    ("grouped SwiGLU hand-off", lambda: _grouped(True), r"gemm_handoff_kernel<true, 1>"),
    ("grouped residual", lambda: _grouped(False, residual=True), r"gemm_kernel<128, true, 0, false, false>"),
]


@pytest.mark.parametrize("what,make,pattern", PATHS, ids=[p[0] for p in PATHS])
def test_gemm_paths(what, make, pattern):
    """Grouped launches without a residual, SwiGLU and HEADS with RoPE reach the hand-off kernel, the rest the staged
    epilogue (profiler kernel names)"""
    launch = make()
    launch()                                   # first launch outside the profiler: module load, smem attribute
    names = _kernel_names(launch)
    assert len(names) == 1 and re.search(pattern.replace(" ", r"\s*"), names[0]), f"{what}: launched {names}"
