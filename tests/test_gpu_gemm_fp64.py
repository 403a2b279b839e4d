"""GPU: every GEMM entry of aria_b200.ops against an fp64 restatement, element by element (references and bounds:
tests/gemm_ref.py, which derives each bound from the kernel's rounding points).

Entry -> test -> bound:
  `linear`               test_linear_vs_fp64, test_linear_epilogues_vs_fp64     linear_ref: acc 2^-12 (|a| @ |b|), bias
                                                                                 in fp32, one rounding per stage, GELU
                                                                                 tanh / NewGELU chain, residual
  `linear_multi`         test_gpu_moe_train_kernels.py::test_linear_multi_vs_fp64, test_linear_multi_pairs_vs_fp64
                                                                                 assert_gemm_close / linear_ref
  `linear_swiglu`        test_linear_swiglu_vs_fp64                              linear_swiglu_ref
  `qkv_heads`            test_qkv_heads_rope_vs_fp64, test_qkv_heads_vit_vs_fp64 rope_ref / linear_ref with bias
  `matmul_kn`            test_gpu_moe_train_kernels.py::test_matmul_kn_vs_fp64   assert_gemm_close
  `grouped_gemm`         test_grouped_gemm_vs_fp64                               grouped_ref + rounding / swiglu_ref /
                                                                                 residual
  `grouped_gemm_regions` test_grouped_gemm_regions_vs_fp64                       grouped_ref + rounding
  `grouped_gemm_nt`      test_grouped_gemm_nt_vs_fp64                            grouped_ref (b [E, N, K]) + residual
  `grouped_wgrad`        test_grouped_wgrad_vs_fp64                              acc 2^-12 + one rounding
  `wgrad_accumulate_f32` test_wgrad_accumulate_f32_vs_fp64                       acc 2^-12 + 2^-22 |out| (fp32 adds, no
                                                                                 bf16 rounding)
  `grouped_gemm_fp8`     test_grouped_gemm_fp8_vs_fp64                           as grouped_gemm on the dequantized
                                                                                 weight: e4m3 widens to bf16 exactly and
                                                                                 the product is a bf16 wgmma
  `grouped_gemm_w8a8`    test_grouped_gemm_w8a8_vs_fp64                          W8A8_ACC (|A| @ |B|) on the dequantized
  `linear_w8a8`          test_linear_w8a8_vs_fp64                                operands, then the bf16 epilogue's
  `linear_swiglu_w8a8`   test_linear_swiglu_w8a8_vs_fp64                         bounds.  W8A8_ACC is the one measured
  `qkv_heads_w8a8`       test_qkv_heads_w8a8_vs_fp64                             bar (see its comment).

Shapes sit at the dispatch boundaries and the tails: M in {1, 63, 64, 65, 127, 129, 2047, 2048, 2049, 4900} reaches the
one-CTA `gemm_kernel` (M < 2048), `gemm_wide_kernel` (dense LINEAR / HEADS without RoPE, M >= 2048; as CTA pairs for
K >= 2048) and the 128-wide CTA pairs (several weights whose N is no multiple of 192); N not a multiple of 128 or 192 and
K below one k-block or not a multiple of 64; 4900 x 4304 is 39 x 23 wide tiles, more than two per SM.  The last m-tile of
2049 rows has one row, and of 4900 rows 36, so the wide kernel's second warpgroup has no row there.  Heads of 72 columns
take 144-wide tiles when n is no multiple of 128.  test_gemm_paths asserts which kernel each case launches.

Tails: A is the leading rows of a buffer whose later rows are NaN (the rows behind the last group, for grouped launches),
or a view whose row stride is past K with NaN columns beyond; a read past the end poisons the result.  Outputs the caller
supplies are filled with a sentinel around the region the call may write, which must survive.  Inputs are N(0, 1)
activations and 0.02-std weights, with a zero row, an element where the result cancels to exactly 0 against a large
|a| @ |b|, and one large outlier per 128-row tile.
"""
import re

import pytest
import torch

import gemm_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
bf16 = torch.bfloat16
f32 = torch.float32
F64 = torch.float64
SENT = 1234.0               # sentinel: exact in bf16 and fp32, and no GEMM here comes near it
# The e4m3 x e4m3 wgmma does not accumulate at full fp32 precision (each 128-wide k-block is summed in the tensor core and
# promoted to fp32 by the kernel).  This bar on err / (|A| @ |B|) rests on a measurement: see W8A8_MEASURED.
# Measured on an H100 80GB HBM3 at a 700 W power limit over the W8A8 shapes below: worst 9.3e-5 (2^-13.4), at K = 128
# and K = 256, where one k-block holds the whole sum; 2.2e-5 to 2.9e-5 at K = 1152 to 2560.  The bar is that worst figure
# with a margin of about 5.
W8A8_MEASURED = 9.3e-5
W8A8_ACC = 2.0 ** -11


def _ops():
    from aria_b200 import ops
    return ops


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _act_in(M, K, seed, pad_rows=0):
    """N(0, 1) bf16 [M, K] as the leading rows of a [M + pad_rows, K] buffer whose other rows are NaN; row M // 2 is zero,
    row M - 1 is symmetric in its two halves (cancellation, with _weight), and one element per 128-row tile is 30."""
    g = _gen(seed)
    buf = torch.full((M + pad_rows, K), float("nan"), dtype=bf16, device=DEV)
    a = torch.randn(M, K, generator=g, device=DEV)
    if M > 2:
        a[M // 2] = 0
    if M > 2 and K % 2 == 0:
        a[M - 1, K // 2:] = a[M - 1, :K // 2]
    for t in range((M + 127) // 128):
        a[min(M - 2 if M > 2 else M - 1, t * 128 + (37 * t) % 128), (61 * t + 5) % K] = 30.0
    buf[:M] = a.to(bf16)
    return buf[:M], buf


def _weight(N, K, seed, std=0.02):
    """0.02-std bf16 [N, K]; columns 0 and N - 1 are antisymmetric in their halves, so row M - 1 of _act_in cancels."""
    w = torch.randn(N, K, generator=_gen(seed), device=DEV) * std
    if K % 2 == 0:
        w[0, K // 2:] = -w[0, :K // 2]
        w[N - 1, K // 2:] = -w[N - 1, :K // 2]
    return w.to(bf16)


def _sentinel_out(M, N, dtype=bf16, pad=64):
    buf = torch.full((M + pad, N), SENT, dtype=dtype, device=DEV)
    return buf[:M], buf


# ------------------------------------------------------------------------------------------------ linear
LINEAR_SHAPES = [                # (M, N, K)
    (1, 8, 8), (63, 200, 40), (64, 264, 72), (65, 256, 1160), (127, 4304, 200), (129, 1160, 2048), (2047, 264, 200),
    (2048, 256, 72),             # wide: the second 192-wide tile has 64 columns
    (2049, 1160, 200),           # wide: the last m-tile has one row
    (4900, 4304, 1160),          # wide, 897 tiles
    (2048, 1160, 2056),          # wide CTA pairs, 7 n-tiles (a phantom), K % 64 = 8
    (2049, 200, 4096),           # wide CTA pairs
]
VARIANTS = [(R.ACT_NONE, True, False), (R.ACT_GELU_TANH, False, False), (R.ACT_GELU_NEW, True, True),
            (R.ACT_NONE, False, True)]


def _linear_case(M, N, K, act, with_bias, with_res, seed):
    ops = _ops()
    x, _ = _act_in(M, K, seed, pad_rows=130)
    w = _weight(N, K, seed + 1)
    g = _gen(seed + 2)
    bias = (torch.randn(N, generator=g, device=DEV) * 0.5).to(bf16) if with_bias else None
    res = torch.randn(M, N, generator=g, device=DEV).to(bf16) if with_res else None
    out, obuf = _sentinel_out(M, N)
    got = ops.linear(x, w, bias=bias, act=act, residual=res, out=out)
    assert got.data_ptr() == out.data_ptr()
    ref, bound = R.linear_ref(x, w, bias, act, res)
    worst = R.check(out, ref, bound, f"linear M={M} N={N} K={K} act={act} bias={with_bias} res={with_res}")
    assert bool((obuf[M:] == SENT).all()), "linear wrote past row M of out"
    if M > 2 and K % 2 == 0 and not with_bias and not with_res and act == R.ACT_NONE:
        assert float(ref[M - 1, 0]) == 0.0 and abs(float(out[M - 1, 0])) <= float(bound[M - 1, 0])
    return worst


@pytest.mark.parametrize("M,N,K", LINEAR_SHAPES)
def test_linear_vs_fp64(M, N, K):
    """Each shape with four epilogues: bias; GELU tanh; NewGELU + bias + residual; residual (on the wide path, the last
    two take the residual protocol, the first two the hand-off)."""
    worst = max(_linear_case(M, N, K, *v, seed=M + N + K + i) for i, v in enumerate(VARIANTS))
    print(f"linear M={M} N={N} K={K}: worst err/bound {worst:.3f}")


@pytest.mark.parametrize("M,N,K", [(65, 264, 200), (2049, 1160, 200), (2048, 256, 2056)])
@pytest.mark.parametrize("act", [R.ACT_NONE, R.ACT_GELU_TANH, R.ACT_GELU_NEW])
@pytest.mark.parametrize("with_bias", [False, True])
@pytest.mark.parametrize("with_res", [False, True])
def test_linear_epilogues_vs_fp64(M, N, K, act, with_bias, with_res):
    """Every act x bias x residual combination on the one-CTA kernel, the wide kernel and the wide pairs."""
    _linear_case(M, N, K, act, with_bias, with_res, seed=act * 4 + with_bias * 2 + with_res)


@pytest.mark.parametrize("M,nseg,N,K", [(2048, 3, 128, 200), (2049, 2, 256, 72), (4900, 2, 640, 1160), (129, 3, 128, 40)])
def test_linear_multi_pairs_vs_fp64(M, nseg, N, K):
    """linear_multi with N no multiple of 192 runs on the 128-wide CTA pairs at M >= 2048 (3 x 128: an odd n-tile count,
    whose last pair has a phantom tile)."""
    ops = _ops()
    x, _ = _act_in(M, K, seed=M + K, pad_rows=130)
    ws = [_weight(N, K, seed=s + 10) for s in range(nseg)]
    got = ops.linear_multi(x, ws)
    ref, bound = R.linear_ref(x, torch.cat(ws, 0))
    R.check(got, ref, bound, f"linear_multi M={M} nseg={nseg} N={N} K={K}")


# ------------------------------------------------------------------------------------------------ linear_swiglu
@pytest.mark.parametrize("M,N,K", [(1, 64, 8), (63, 192, 40), (129, 1664, 200), (2049, 320, 1160), (4900, 192, 72)])
def test_linear_swiglu_vs_fp64(M, N, K):
    """out = bf16(bf16(silu(bf16 g)) bf16 u) for g = x @ gate.T, u = x @ up.T (swiglu_ref).  The gate weight has 0.1 std,
    so gates span several units, where silu is far from linear."""
    ops = _ops()
    x, _ = _act_in(M, K, seed=M * 3 + K, pad_rows=130)
    gw, uw = _weight(N, K, seed=M + 1, std=0.1), _weight(N, K, seed=M + 2)
    got = ops.linear_swiglu(x, gw, uw)
    ref, bound = R.linear_swiglu_ref(x, gw, uw)
    R.check(got, ref, bound, f"linear_swiglu M={M} N={N} K={K}", tile=(128, 64))


# ------------------------------------------------------------------------------------------------ qkv_heads
def _rope_tables(n_pos):
    inv = 1.0 / 10000.0 ** (torch.arange(0, 128, 2, dtype=f32, device=DEV) / 128)
    return _ops().rope_table(inv.contiguous(), n_pos)


def _heads_view(t, B, T, H, hd):
    """[B T, H hd] -> [B, H, T, hd]"""
    return t.view(B, T, H, hd).permute(0, 2, 1, 3)


def _check_heads(outs, refs, bounds, B, T, pos0, hd, what):
    for s, (o, ref, bound) in enumerate(zip(outs, refs, bounds)):
        R.check(o[:, :, pos0:pos0 + T, :hd], ref, bound, f"{what} segment {s}")
        keep = torch.ones_like(o, dtype=torch.bool)
        keep[:, :, pos0:pos0 + T, :hd] = False
        assert bool((o[keep] == SENT).all()), f"{what}: segment {s} wrote outside its tokens and head columns"


@pytest.mark.parametrize("B,T,Hn,K,pos0,head_ld,posids", [(1, 1, 2, 256, 0, 128, False), (2, 65, 2, 200, 7, 136, False),
                                                          (1, 300, 4, 1160, 3, 128, True), (3, 700, 2, 72, 0, 128, True)])
def test_qkv_heads_rope_vs_fp64(B, T, Hn, K, pos0, head_ld, posids):
    """LM q/k/v: three 128-dim-head weights, RoPE on q and k (rope_mask 0b011), v plain.  RoPE at pos0 + t, or at
    position_ids (random positions, unrelated to where the row is stored); the store is at token pos0 + t of each batch row.
    Sentinels fill the tokens before pos0 and after pos0 + T, and the pad columns past head_dim."""
    ops = _ops()
    M, N, hd = B * T, Hn * 128, 128
    x, _ = _act_in(M, K, seed=M + K, pad_rows=130)
    ws = [_weight(N, K, seed=s + M) for s in range(3)]
    T_max = pos0 + T + 5
    outs = [torch.full((B, Hn, T_max, head_ld), SENT, dtype=bf16, device=DEV) for _ in range(3)]
    cos, sin = _rope_tables(4096)
    if posids:
        pos = torch.randint(0, 4096, (M,), generator=_gen(M), device=DEV, dtype=torch.int32)
    else:
        pos = (pos0 + torch.arange(T, device=DEV, dtype=torch.int32)).repeat(B)
    ops.qkv_heads(x, ws, [None] * 3, outs, hd, T, pos0=pos0, rope_mask=0b011, rope_cos=cos, rope_sin=sin,
                  position_ids=pos if posids else None)
    refs, bounds = [], []
    for s, w in enumerate(ws):
        z, e = R.acc_ref(x, w.t())
        z, e = _heads_view(z, B, T, Hn, hd), _heads_view(e, B, T, Hn, hd)
        if s < 2:
            c = _heads_view(cos[pos.long()][:, None, :].expand(M, Hn, hd).reshape(M, N), B, T, Hn, hd)
            sn = _heads_view(sin[pos.long()][:, None, :].expand(M, Hn, hd).reshape(M, N), B, T, Hn, hd)
            ref, bound = R.rope_ref(z, e, c, sn)
        else:
            ref, bound = z, R.rnd(z, e)
        refs.append(ref)
        bounds.append(bound)
    _check_heads(outs, refs, bounds, B, T, pos0, hd, f"qkv_heads rope B={B} T={T} K={K}")


@pytest.mark.parametrize("B,T,Hn,K,pos0", [(1, 65, 16, 200, 0), (2, 300, 16, 1152, 4), (1, 2048, 16, 1152, 0),
                                            (2, 2450, 16, 1160, 0), (1, 129, 10, 1152, 3), (3, 700, 10, 200, 0)])
def test_qkv_heads_vit_vs_fp64(B, T, Hn, K, pos0):
    """q/k/v of 72-column heads with biases into buffers padded to 80 columns, no RoPE.  16 heads (the ViT, n = 1152) run
    128-wide tiles that cut heads at M < 2048 and the wide kernel's head scatter (n = 6 x 192) at M >= 2048; 10 heads
    (n = 720, no multiple of 128 or 192) run 144-wide tiles of two whole heads at any M.  The pad columns 72..79 and the
    tokens around the stored range keep their sentinel."""
    ops = _ops()
    M, hd, head_ld = B * T, 72, 80
    N = Hn * hd
    x, _ = _act_in(M, K, seed=M + K + 1, pad_rows=130)
    ws = [_weight(N, K, seed=s + M + 7) for s in range(3)]
    bs = [(torch.randn(N, generator=_gen(s + 99), device=DEV) * 0.5).to(bf16) for s in range(3)]
    T_max = pos0 + T + 3
    outs = [torch.full((B, Hn, T_max, head_ld), SENT, dtype=bf16, device=DEV) for _ in range(3)]
    ops.qkv_heads(x, ws, bs, outs, hd, T, pos0=pos0)
    refs, bounds = [], []
    for w, b in zip(ws, bs):
        ref, bound = R.linear_ref(x, w, b)
        refs.append(_heads_view(ref, B, T, Hn, hd))
        bounds.append(_heads_view(bound, B, T, Hn, hd))
    _check_heads(outs, refs, bounds, B, T, pos0, hd, f"qkv_heads vit B={B} T={T} K={K}")


def test_qkv_heads_rejects_a_bias_on_a_rope_segment():
    """The RoPE epilogue has no bias term: a bias given for a rotated segment would be dropped without a word, so the launch
    is refused instead (the LM's q/k/v have no bias)."""
    ops = _ops()
    x, _ = _act_in(4, 64, seed=1)
    ws = [_weight(128, 64, seed=s) for s in range(3)]
    outs = [torch.full((1, 1, 4, 128), SENT, dtype=bf16, device=DEV) for _ in range(3)]
    cos, sin = _rope_tables(16)
    b = torch.zeros(128, dtype=bf16, device=DEV)
    with pytest.raises(RuntimeError, match="bad argument"):
        ops.qkv_heads(x, ws, [None, b, None], outs, 128, 4, rope_mask=0b011, rope_cos=cos, rope_sin=sin)
    ops.qkv_heads(x, ws, [None, None, b], outs, 128, 4, rope_mask=0b011, rope_cos=cos, rope_sin=sin)   # v is not rotated


# ------------------------------------------------------------------------------------------------ grouped
def _offsets(counts):
    off = torch.zeros(len(counts) + 1, dtype=torch.int32)
    off[1:] = torch.tensor(counts, dtype=torch.int64).cumsum(0).to(torch.int32)
    return off.to(DEV)


def _mix(name, E):
    from test_gpu_fp8 import _row_mix
    if name == "edges":                              # empty, 1-row and 65-row groups and a tile-crossing one
        return ([0, 1, 65, 0, 129, 1, 300, 0] * ((E + 7) // 8))[:E]
    return _row_mix(name, E=E, seed=E)


GROUPED = [("edges", 8, 128, 256), ("decode_b1", 64, 256, 192), ("ragged", 16, 1152, 320), ("b32", 64, 2560, 128),
           ("edges", 8, 64, 1664)]


@pytest.mark.parametrize("mix,E,K,N", GROUPED)
@pytest.mark.parametrize("epi", ["linear", "swiglu", "residual", "group_mod"])
def test_grouped_gemm_vs_fp64(mix, E, K, N, epi):
    """grouped_gemm over group mixes with empty, 1-row and 65-row groups.  A's rows behind the last group are NaN.
    swiglu: b has 2N columns, gate then up; group_mod: 2E groups (source rank, expert) over E weights."""
    ops = _ops()
    counts = _mix(mix, E)
    G = 2 * E if epi == "group_mod" else E
    if epi == "group_mod":
        counts = counts + counts[::-1]
    off = _offsets(counts)
    rows = int(off[-1])
    a, _ = _act_in(rows, K, seed=rows + K, pad_rows=130)
    Nb = 2 * N if epi == "swiglu" else N
    b = (torch.randn(E, K, Nb, generator=_gen(E + K), device=DEV) * (0.05 if epi == "swiglu" else 0.02)).to(bf16)
    res = torch.randn(rows, N, generator=_gen(rows), device=DEV).to(bf16) if epi == "residual" else None
    got = ops.grouped_gemm(a, b, off, swiglu=epi == "swiglu", group_mod=E if epi == "group_mod" else 0, residual=res)
    z, e = R.grouped_ref(a, b, off, group_mod=E if epi == "group_mod" else 0)
    if epi == "swiglu":
        ref, bound = R.swiglu_ref(z[:, :N], e[:, :N], z[:, N:], e[:, N:])
    else:
        ref, bound = z, R.rnd(z, e)
        if res is not None:
            ref = ref + res.to(F64)
            bound = R.rnd(ref, bound)
    R.check(got, ref, bound, f"grouped_gemm {epi} {mix} E={E} K={K} N={N}")


@pytest.mark.parametrize("mix,E,K,N", [("edges", 8, 128, 256), ("ragged", 16, 1152, 192)])
@pytest.mark.parametrize("swiglu", [False, True])
def test_grouped_gemm_regions_vs_fp64(mix, E, K, N, swiglu):
    """Groups in fixed-capacity regions of a_buf (capacity = the largest count + 17): the unused rows of every region are
    NaN, and the rows of out outside every group keep their sentinel."""
    ops = _ops()
    counts = _mix(mix, E)
    cap = max(counts) + 17
    starts = torch.arange(E, dtype=torch.int32, device=DEV) * cap
    cnt = torch.tensor(counts, dtype=torch.int32, device=DEV)
    a_buf = torch.full((E * cap, K), float("nan"), dtype=bf16, device=DEV)
    valid = torch.zeros(E * cap, dtype=torch.bool, device=DEV)
    for g_, c in enumerate(counts):
        valid[g_ * cap:g_ * cap + c] = True
    a_buf[valid] = torch.randn(int(valid.sum()), K, generator=_gen(K), device=DEV).to(bf16)
    Nb = 2 * N if swiglu else N
    b = (torch.randn(E, K, Nb, generator=_gen(E), device=DEV) * 0.05).to(bf16)
    out = torch.full((E * cap, N), SENT, dtype=bf16, device=DEV)
    ops.grouped_gemm_regions(a_buf, b, starts, cnt, rows_hint=sum(counts), swiglu=swiglu, out=out)
    z = torch.zeros(E * cap, Nb, dtype=F64, device=DEV)
    e = torch.zeros_like(z)
    for g_, c in enumerate(counts):
        if c:
            r = slice(g_ * cap, g_ * cap + c)
            z[r], e[r] = R.acc_ref(a_buf[r], b[g_])
    if swiglu:
        ref, bound = R.swiglu_ref(z[:, :N], e[:, :N], z[:, N:], e[:, N:])
    else:
        ref, bound = z, R.rnd(z, e)
    R.check(out[valid], ref[valid], bound[valid], f"grouped_gemm_regions {mix} swiglu={swiglu}")
    assert bool((out[~valid] == SENT).all()), "grouped_gemm_regions wrote a row outside its groups"


@pytest.mark.parametrize("mix,E,K,N", [("edges", 8, 200, 256), ("ragged", 16, 1664, 1152), ("decode_b1", 64, 72, 128)])
@pytest.mark.parametrize("residual", [False, True])
def test_grouped_gemm_nt_vs_fp64(mix, E, K, N, residual):
    """grouped_gemm_nt: out[rows of g] = a[rows of g] @ b[g].T, b [E, N, K] read K-major in place.  a is contiguous (the
    wrapper requires it), the leading rows of a buffer whose rows behind the last group are NaN."""
    ops = _ops()
    counts = _mix(mix, E)
    off = _offsets(counts)
    rows = int(off[-1])
    a, _ = _act_in(rows, K, seed=rows + 3, pad_rows=130)
    b = (torch.randn(E, N, K, generator=_gen(N + K), device=DEV) * 0.02).to(bf16)
    res = torch.randn(rows, N, generator=_gen(rows + 1), device=DEV).to(bf16) if residual else None
    got = ops.grouped_gemm_nt(a, b, off, residual=res)
    z, e = R.grouped_ref(a, b, off, b_nk=True)
    ref, bound = z, R.rnd(z, e)
    if res is not None:
        ref = ref + res.to(F64)
        bound = R.rnd(ref, bound)
    R.check(got, ref, bound, f"grouped_gemm_nt {mix} K={K} N={N} residual={residual}")


@pytest.mark.parametrize("counts,Md,Nd,sources", [
    ([0, 1, 65, 0, 130, 7, 2049, 16], 256, 200, 1),
    ([3, 0, 17, 300], 1664, 2560, 2),
    ([0] * 5 + [1] * 3 + [64] * 8, 128, 8, 1),
    ([5, 0, 9, 129, 0, 2, 33, 1, 70], 72, 136, 3),
])
def test_grouped_wgrad_vs_fp64(counts, Md, Nd, sources):
    """grouped_wgrad: out[g] = sum over sources of a[rows of (s, g)].T @ b[rows of (s, g)] in fp32, rounded once; empty and
    unaligned groups (an empty group gives zeros); a and b are views into NaN-flanked buffers (row stride past the width),
    and the rows behind the last group are NaN."""
    ops = _ops()
    G = len(counts)
    cts = [c + s for s in range(sources) for c in counts]     # (source, group) blocks, source-major
    off = _offsets(cts)
    rows = int(off[-1])
    g = _gen(rows + Md + Nd)
    af = torch.full((rows + 40, Md + 24), float("nan"), dtype=bf16, device=DEV)
    bf = torch.full((rows + 40, Nd + 8), float("nan"), dtype=bf16, device=DEV)
    af[:rows, :Md] = torch.randn(rows, Md, generator=g, device=DEV).to(bf16)
    bf[:rows, :Nd] = (torch.randn(rows, Nd, generator=g, device=DEV) * 0.1).to(bf16)
    a, b = af[:rows, :Md], bf[:rows, :Nd]
    got = ops.grouped_wgrad(a, b, off, num_sources=sources)
    ol = off.tolist()
    for gi in range(G):
        idx = torch.cat([torch.arange(ol[s * G + gi], ol[s * G + gi + 1], device=DEV) for s in range(sources)])
        if idx.numel() == 0:
            assert bool((got[gi] == 0).all())
            continue
        z, e = R.acc_ref(a[idx].t(), b[idx])
        R.check(got[gi], z, R.rnd(z, e), f"grouped_wgrad group {gi} Md={Md} Nd={Nd} sources={sources}")


@pytest.mark.parametrize("rows,Md,Nd", [(1, 8, 8), (300, 4304, 200), (2049, 1160, 2560), (4900, 256, 72)])
def test_wgrad_accumulate_f32_vs_fp64(rows, Md, Nd):
    """wgrad_accumulate_f32 as the fused-CE backward calls it: out += a.T @ b over two chunks of rows, into a non-zero fp32
    accumulator.  Bound: 2^-12 (|a|.T @ |b|) for the fp32 accumulation, plus 2^-22 (|out0| + |ref|) for the fp32 additions
    into out; there is no bf16 rounding.  a, b are NaN-flanked views; out is the leading rows of a buffer whose later rows
    hold a sentinel."""
    ops = _ops()
    g = _gen(rows + Md)
    af = torch.full((rows, Md + 16), float("nan"), dtype=bf16, device=DEV)
    bf = torch.full((rows, Nd + 8), float("nan"), dtype=bf16, device=DEV)
    af[:, :Md] = torch.randn(rows, Md, generator=g, device=DEV).to(bf16)
    bf[:, :Nd] = (torch.randn(rows, Nd, generator=g, device=DEV) * 0.1).to(bf16)
    a, b = af[:, :Md], bf[:, :Nd]
    obuf = torch.full((Md + 8, Nd), SENT, dtype=f32, device=DEV)
    out = obuf[:Md]
    out.copy_(torch.randn(Md, Nd, generator=g, device=DEV))
    out0 = out.to(F64)
    h = rows // 2
    for r0, r1 in ((0, h), (h, rows)):
        if r1 > r0:
            ops.wgrad_accumulate_f32(a[r0:r1], b[r0:r1], out)
    z, e = R.acc_ref(a.t(), b)
    ref = out0 + z
    bound = e + 2.0 ** -22 * (out0.abs() + ref.abs())
    R.check(out, ref, bound, f"wgrad_accumulate_f32 rows={rows} Md={Md} Nd={Nd}")
    assert bool((obuf[Md:] == SENT).all())


# ------------------------------------------------------------------------------------------------ fp8
def _deq_cols(q, scale):
    return q.to(F64) * scale.to(F64)[:, None, :]


@pytest.mark.parametrize("mix,E,K,N", [("edges", 8, 128, 256), ("ragged", 16, 1152, 320), ("decode_b1", 64, 2560, 192)])
@pytest.mark.parametrize("swiglu", [False, True])
def test_grouped_gemm_fp8_vs_fp64(mix, E, K, N, swiglu):
    """grouped_gemm_fp8 against a @ (q scale) with real per-column scales (quantize_fp8_cols).  The e4m3 codes widen to bf16
    exactly and the MMA is bf16 wgmma into fp32, so the accumulation bound is 2^-12 (|a| @ |q scale|); the scale multiplies
    the fp32 accumulator (2^-24) before the epilogue's roundings."""
    ops = _ops()
    counts = _mix(mix, E)
    off = _offsets(counts)
    rows = int(off[-1])
    a, _ = _act_in(rows, K, seed=rows + 5, pad_rows=130)
    Nb = 2 * N if swiglu else N
    w = (torch.randn(E, K, Nb, generator=_gen(K + N), device=DEV) * 0.05).to(bf16)
    q, scale = ops.quantize_fp8_cols(w)
    got = ops.grouped_gemm_fp8(a, q, scale, off, swiglu=swiglu)
    z, e = R.grouped_ref(a, _deq_cols(q, scale), off)
    if swiglu:
        ref, bound = R.swiglu_ref(z[:, :N], e[:, :N], z[:, N:], e[:, N:])
    else:
        ref, bound = z, R.rnd(z, e)
    R.check(got, ref, bound, f"grouped_gemm_fp8 {mix} swiglu={swiglu}")


_w8a8_worst = {}


def _w8a8_ratio(got, ref, absprod, what):
    """The measured accumulation error of a W8A8 result: max (|got - ref| - 2^-8 |ref|)+ / (|A| @ |B|), printed."""
    r = float(((got.to(F64) - ref).abs() - R.RND * ref.abs()).clamp_min(0).div(absprod.clamp_min(1e-300)).max())
    _w8a8_worst[what] = r
    print(f"{what}: worst err / (|A| @ |B|) = {r:.3e} (2^{torch.tensor(max(r, 1e-30)).log2().item():.2f}); "
          f"bar W8A8_ACC = {W8A8_ACC:.3e}")
    return r


@pytest.mark.parametrize("mix,E,K,N", [("edges", 8, 128, 256), ("ragged", 16, 1152, 320), ("decode_b1", 64, 2560, 192)])
@pytest.mark.parametrize("swiglu", [False, True])
def test_grouped_gemm_w8a8_vs_fp64(mix, E, K, N, swiglu):
    """grouped_gemm_w8a8 against (aq a_s) @ (wq w_s) with real scales (permute_quantize_fp8, quantize_fp8_cols)."""
    ops = _ops()
    counts = _mix(mix, E)
    off = _offsets(counts)
    rows = int(off[-1])
    a, _ = _act_in(rows, K, seed=rows + 6)
    aq, a_s = ops.permute_quantize_fp8(a)
    Nb = 2 * N if swiglu else N
    w = (torch.randn(E, K, Nb, generator=_gen(K + N + 1), device=DEV) * 0.05).to(bf16)
    q, scale = ops.quantize_fp8_cols(w)
    weight = q.transpose(1, 2).contiguous().transpose(1, 2)
    got = ops.grouped_gemm_w8a8(aq, a_s, weight, scale, off, swiglu=swiglu)
    A = aq.to(F64) * a_s.to(F64)[:, None]
    z, e = R.grouped_ref(A, _deq_cols(q, scale), off, acc=W8A8_ACC)
    if swiglu:
        ref, bound = R.swiglu_ref(z[:, :N], e[:, :N], z[:, N:], e[:, N:])
    else:
        ref, bound = z, R.rnd(z, e)
        _w8a8_ratio(got, ref, e / W8A8_ACC, f"grouped_gemm_w8a8 {mix} K={K} N={N}")
    R.check(got, ref, bound, f"grouped_gemm_w8a8 {mix} swiglu={swiglu}")


def _dense_w8a8(N, K, seed):
    w = _weight(N, K, seed)
    return _ops().permute_quantize_fp8(w)


def _deq_rows(q, s):
    return q.to(F64) * s.to(F64)[:, None]


@pytest.mark.parametrize("M,N,K", [(1, 64, 128), (65, 320, 1152), (2049, 2560, 2560), (300, 4352, 256)])
@pytest.mark.parametrize("residual", [False, True])
def test_linear_w8a8_vs_fp64(M, N, K, residual):
    ops = _ops()
    x, _ = _act_in(M, K, seed=M + K + 9)
    xq, xs = ops.permute_quantize_fp8(x)
    wq, ws = _dense_w8a8(N, K, seed=N + K)
    res = torch.randn(M, N, generator=_gen(M), device=DEV).to(bf16) if residual else None
    got = ops.linear_w8a8(xq, xs, wq, ws, residual=res)
    A, W = _deq_rows(xq, xs), _deq_rows(wq, ws)
    ref, bound = R.linear_ref(A, W, residual=res, acc=W8A8_ACC)
    if not residual:
        _w8a8_ratio(got, ref, (A.abs() @ W.abs().t()), f"linear_w8a8 M={M} N={N} K={K}")
    R.check(got, ref, bound, f"linear_w8a8 M={M} N={N} K={K} residual={residual}")


@pytest.mark.parametrize("M,N,K", [(1, 64, 128), (129, 1664, 2560), (2049, 192, 1152)])
def test_linear_swiglu_w8a8_vs_fp64(M, N, K):
    ops = _ops()
    x, _ = _act_in(M, K, seed=M + K + 10)
    xq, xs = ops.permute_quantize_fp8(x)
    gq, gs = _dense_w8a8(N, K, seed=N + 1)
    uq, us = _dense_w8a8(N, K, seed=N + 2)
    got = ops.linear_swiglu_w8a8(xq, xs, gq, gs, uq, us)
    A = _deq_rows(xq, xs)
    ref, bound = R.linear_swiglu_ref(A, _deq_rows(gq, gs), _deq_rows(uq, us), acc=W8A8_ACC)
    R.check(got, ref, bound, f"linear_swiglu_w8a8 M={M} N={N} K={K}", tile=(128, 64))


@pytest.mark.parametrize("B,T,K,pos0,posids", [(1, 1, 256, 5, False), (2, 300, 2560, 0, True)])
def test_qkv_heads_w8a8_vs_fp64(B, T, K, pos0, posids):
    ops = _ops()
    M, Hn, hd = B * T, 2, 128
    N = Hn * hd
    x, _ = _act_in(M, K, seed=M + 11)
    xq, xs = ops.permute_quantize_fp8(x)
    qs = [_dense_w8a8(N, K, seed=s + 40) for s in range(3)]
    T_max = pos0 + T + 2
    outs = [torch.full((B, Hn, T_max, hd), SENT, dtype=bf16, device=DEV) for _ in range(3)]
    cos, sin = _rope_tables(4096)
    pos = (torch.randint(0, 4096, (M,), generator=_gen(M), device=DEV, dtype=torch.int32) if posids
           else (pos0 + torch.arange(T, device=DEV, dtype=torch.int32)).repeat(B))
    ops.qkv_heads_w8a8(xq, xs, [q for q, _ in qs], [s for _, s in qs], outs, hd, T, pos0=pos0, rope_mask=0b011,
                       rope_cos=cos, rope_sin=sin, position_ids=pos if posids else None)
    A = _deq_rows(xq, xs)
    refs, bounds = [], []
    for s, (q, sc) in enumerate(qs):
        z, e = R.acc_ref(A, _deq_rows(q, sc).t(), acc=W8A8_ACC)
        z, e = _heads_view(z, B, T, Hn, hd), _heads_view(e, B, T, Hn, hd)
        if s < 2:
            c = _heads_view(cos[pos.long()][:, None, :].expand(M, Hn, hd).reshape(M, N), B, T, Hn, hd)
            sn = _heads_view(sin[pos.long()][:, None, :].expand(M, Hn, hd).reshape(M, N), B, T, Hn, hd)
            ref, bound = R.rope_ref(z, e, c, sn)
        else:
            ref, bound = z, R.rnd(z, e)
        refs.append(ref)
        bounds.append(bound)
    _check_heads(outs, refs, bounds, B, T, pos0, hd, f"qkv_heads_w8a8 B={B} T={T}")


# ------------------------------------------------------------------------------------------------ which kernel runs
def _kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "gemm" in e.name]


def _lin(M, N, K, residual=False):
    x, w = _act_in(M, K, 1)[0], _weight(N, K, 2)
    r = torch.zeros(M, N, dtype=bf16, device=DEV) if residual else None
    return lambda: _ops().linear(x, w, residual=r)


def _multi(M, nseg, N, K):
    x = _act_in(M, K, 1)[0]
    ws = [_weight(N, K, s) for s in range(nseg)]
    return lambda: _ops().linear_multi(x, ws)


def _vit_heads(M, K, Hn=16):
    x = _act_in(M, K, 1)[0]
    ws = [_weight(Hn * 72, K, s) for s in range(3)]
    outs = [torch.empty(1, Hn, M, 80, dtype=bf16, device=DEV) for _ in range(3)]
    return lambda: _ops().qkv_heads(x, ws, [None] * 3, outs, 72, M)


# (what, launch, kernel-name pattern): gemm_kernel<BN, B_MN, EPI, B_FP8, PAIR>, gemm_wide_kernel<EPI, PAIR, HANDOFF>;
# EPI 0 = LINEAR, 2 = HEADS
PATHS = [
    ("one CTA, M = 2047", lambda: _lin(2047, 264, 200), r"gemm_kernel<128, false, 0, false, false>"),
    ("pairs, 3 x 128 columns", lambda: _multi(2048, 3, 128, 200), r"gemm_kernel<128, false, 0, false, true>"),
    ("wide hand-off", lambda: _lin(2048, 256, 72), r"gemm_wide_kernel<0, false, true>"),
    ("wide residual", lambda: _lin(2049, 1160, 200, residual=True), r"gemm_wide_kernel<0, false, false>"),
    ("wide pairs hand-off", lambda: _lin(2048, 1160, 2056), r"gemm_wide_kernel<0, true, true>"),
    ("wide pairs residual", lambda: _lin(2049, 200, 4096, residual=True), r"gemm_wide_kernel<0, true, false>"),
    ("wide 4900 x 4304", lambda: _lin(4900, 4304, 1160), r"gemm_wide_kernel<0, false, true>"),
    ("128-wide heads", lambda: _vit_heads(300, 1152), r"gemm_kernel<128, false, 2, false, false>"),
    ("144-wide heads", lambda: _vit_heads(2100, 1152, Hn=10), r"gemm_kernel<144, false, 2, false, false>"),
    ("wide heads", lambda: _vit_heads(2048, 1152), r"gemm_wide_kernel<2, false, true>"),
]


@pytest.mark.parametrize("what,make,pattern", PATHS, ids=[p[0] for p in PATHS])
def test_gemm_paths(what, make, pattern):
    """The shapes above reach the kernel they were chosen for (read from the profiler's kernel names, one launch each), so
    a moved dispatch threshold cannot silently route them all onto one path."""
    launch = make()
    launch()                                   # first launch outside the profiler: module load, smem attribute
    names = _kernel_names(launch)
    assert len(names) == 1 and re.search(pattern.replace(" ", r"\s*"), names[0]), f"{what}: launched {names}"
