"""GPU: the MoE training path's kernels one at a time, and MoELayerFunction at the cfg-5 width, against fp64.

Every reference is a plain fp64 restatement of the operation, computed on the GPU in torch.  Each bound follows from the
arithmetic of the kernel it checks (stated in each test's docstring), so a kernel that is wrong in one expert, one
16-row block, one k-block or one corner of an activation fails even when a whole-tensor norm would not notice.
"""
import pytest
import torch

from gemm_ref import assert_gemm_close

pytestmark = pytest.mark.gpu
DEV = "cuda"
bf16 = torch.bfloat16
f64 = torch.float64


def _ops():
    from aria_b200 import ops
    return ops


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _rel_l2(got, ref):
    got, ref = got.double(), ref.double()
    return float((got - ref).norm() / ref.norm().clamp_min(1e-300))


# ------------------------------------------------------------------------------------------------ SwiGLU
def _swiglu_inputs(rows, I, seed):
    """h1 = [gate | up] (bf16) and dh: gates mix uniform [-100, 100], N(0, 3), a cluster around g = -1.278 (where
    d silu/dg crosses zero), and fixed specials (+-0, tiny magnitudes, the rcp flush region below -87, +-100).  Rows 0
    and rows // 2 are pad rows (all zero in h1 and dh) when rows > 1."""
    g = _gen(seed)
    n = rows * I
    kind = torch.randint(0, 3, (n,), generator=g, device=DEV)
    gate = torch.where(kind == 0, torch.rand(n, generator=g, device=DEV) * 200 - 100,
                       torch.where(kind == 1, torch.randn(n, generator=g, device=DEV) * 3,
                                   -1.2785 + torch.randn(n, generator=g, device=DEV) * 0.02))
    specials = torch.tensor([0.0, -0.0, 1e-30, -1e-30, 1e-20, -1e-6, -1.278465, -86.0, -87.5, -88.5, -90.0, 87.0,
                             100.0, -100.0], device=DEV)
    m = min(n, specials.numel())
    gate[:m] = specials[:m]
    if n > 4 * specials.numel():   # specials again, in the middle and last vectors of the row-major array
        gate[n // 2:n // 2 + m] = specials[:m]
        gate[n - m:] = specials[:m]
    gate = gate.view(rows, I)
    up = torch.randn(rows, I, generator=g, device=DEV) * 2
    dh = torch.randn(rows, I, generator=g, device=DEV)
    h1 = torch.cat([gate, up], 1).to(bf16)
    dh = dh.to(bf16)
    pads = [0, rows // 2] if rows > 1 else []
    for r in pads:
        h1[r] = 0
        dh[r] = 0
    return h1, dh, pads


SWIGLU_SHAPES = [(r, i) for r in (1, 17, 8192) for i in (8, 128, 1664)]


@pytest.mark.parametrize("rows,I", SWIGLU_SHAPES)
def test_swiglu_fwd_vs_fp64(rows, I):
    """h = bf16(bf16(silu(g)) * u), the reference model's rounding, evaluated from fp64.

    The kernel computes silu(g) = g * rcp.approx(1 + ex2.approx(-log2(e) g)) in fp32.  The fp32 product -log2(e) g is off
    by up to |g| 2^-24 in the exponent (a relative error of ~|g| 2^-24 in the exponential), and ex2/rcp add ~2^-22 each:
    within eps(g) = 2^-20 + |g| 2^-23 of silu.  bf16(silu) can therefore differ from the fp64 rounding only where silu
    lies within eps(g) of a bf16 rounding boundary, and then by one ulp: the kernel must give bf16(s * u) for s one of
    the roundings of silu * (1 -+ eps(g)).  s * u is exact in fp32 (two 8-bit significands), so that last rounding is the
    reference's.  Fewer than 2^-8 of the elements may differ from the nominal rounding (the boundary windows are narrower).
    Accepted: for g < -87, 1 + e^-g >= 2^126 and rcp.approx.ftz flushes its subnormal result, so silu = 0 where the true
    value is a tiny normal (|silu| < 2^-119); those elements may be exactly zero.  Pad rows (all zero) give exact zeros."""
    ops = _ops()
    h1, _, pads = _swiglu_inputs(rows, I, seed=rows * 31 + I)
    h = ops.swiglu_fwd(h1)
    torch.cuda.synchronize()
    g64, u64 = h1[:, :I].to(f64), h1[:, I:].to(f64)
    silu = g64 * torch.sigmoid(g64)
    eps = 2.0 ** -20 + g64.abs() * 2.0 ** -23
    want = (silu.to(bf16).to(f64) * u64).to(bf16)
    want_a = ((silu * (1 - eps)).to(bf16).to(f64) * u64).to(bf16)
    want_b = ((silu * (1 + eps)).to(bf16).to(f64) * u64).to(bf16)
    flushed = (g64 < -87) & (h == 0)
    ok = (h == want_a) | (h == want_b) | flushed
    assert bool(ok.all()), (f"{int((~ok).sum())} elements off; first at {(~ok).nonzero()[0].tolist()}: "
                            f"g={float(g64[~ok][0])} u={float(u64[~ok][0])} got={float(h[~ok][0])} want={float(want[~ok][0])}")
    n_diff = int(((h != want) & ~flushed).sum())
    print(f"swiglu_fwd rows={rows} I={I}: {n_diff}/{h.numel()} elements one ulp from the fp64 rounding, "
          f"{int(((g64 < -87) & (want != 0)).sum())} flushed")
    assert n_diff <= h.numel() * 2 ** -8 + 2
    for r in pads:
        assert bool((h[r] == 0).all())


@pytest.mark.parametrize("rows,I", SWIGLU_SHAPES)
def test_swiglu_bwd_vs_fp64(rows, I):
    """dgate = dh u sig (1 + g (1 - sig)), dup = dh silu(g), against fp64.

    dgate: the factor f = sig (1 + g (1 - sig)) is evaluated in fp32 from an approximate sig (relative error ~2^-22 for
    g > 0, where it matters).  Its absolute error is at most ~|g| 2^-21 while 1 - sig is resolved (g < 17) and
    (g - 1) e^-g < 2^-20 after 1 + e^-g rounds to 1; for g < 0 every error term carries a factor sig.  So
    |f - f64| <= 2^-16, and |dgate - ref| <= 2^-8 |ref| (one bf16 rounding; the fp32 products' ~2^-22 fit in the gap
    between 2^-8 and the largest relative rounding error, 2^-8 / (1 + 2^-8)) + 2^-16 |dh u|.
    At g ~ -1.278, where f crosses zero and the formula cancels, the floor is what holds, and it is 256 times finer than
    one bf16 rounding of |dh u|: dropping any term of f fails by orders of magnitude.
    dup: |dup - ref| <= (2^-8 + eps(g)) |ref|: one bf16 rounding plus silu's relative error eps(g) (forward test), except
    that for g < -87 the flushed silu gives dup = 0 against a tiny normal value.  Both bounds get an absolute 2^-134:
    below 2^-126 bf16 is subnormal, its spacing is a fixed 2^-133, and dh silu(g) lands there for g near -87.
    Pad rows give exact zeros."""
    ops = _ops()
    h1, dh, pads = _swiglu_inputs(rows, I, seed=rows * 37 + I + 1)
    dh1 = ops.swiglu_bwd(h1, dh)
    torch.cuda.synchronize()
    g64, u64, d64 = h1[:, :I].to(f64), h1[:, I:].to(f64), dh.to(f64)
    sig = torch.sigmoid(g64)
    ref_g = d64 * u64 * (sig * (1 + g64 * (1 - sig)))
    ref_u = d64 * g64 * sig
    got_g, got_u = dh1[:, :I].to(f64), dh1[:, I:].to(f64)
    err_g = (got_g - ref_g).abs()
    bound_g = 2.0 ** -8 * ref_g.abs() + 2.0 ** -16 * (d64 * u64).abs() + 2.0 ** -134
    bad = ~(err_g <= bound_g)
    assert not bool(bad.any()), (f"dgate: {int(bad.sum())} off; first g={float(g64[bad][0])} got={float(got_g[bad][0])} "
                                 f"ref={float(ref_g[bad][0])}")
    err_u = (got_u - ref_u).abs()
    eps = 2.0 ** -20 + g64.abs() * 2.0 ** -23
    bound_u = torch.where(g64 < -87, ref_u.abs(), (2.0 ** -8 + eps) * ref_u.abs()) + 2.0 ** -134
    bad = ~(err_u <= bound_u)
    assert not bool(bad.any()), (f"dup: {int(bad.sum())} off; first g={float(g64[bad][0])} got={float(got_u[bad][0])} "
                                 f"ref={float(ref_u[bad][0])}")
    print(f"swiglu_bwd rows={rows} I={I}: max err/bound dgate {float((err_g / bound_g.clamp_min(1e-300)).max()):.3f}, "
          f"dup {float((err_u / bound_u.clamp_min(1e-300))[g64 >= -87].max()):.3f}")
    for r in pads:
        assert bool((dh1[r] == 0).all())


# ------------------------------------------------------------------------------------------------ combine backward
def _aligned_routing(T, E, k, seed, empty=5):
    """Real routing (route_from_logits) into the training layout (build_permutation(row_align=16)); expert `empty` gets
    no token."""
    ops = _ops()
    logits = torch.randn(T, E, generator=_gen(seed), device=DEV).to(bf16)
    logits[:, empty] = -100.0
    s, idx, c = ops.route_from_logits(logits, k)
    off, dest, src = ops.build_permutation(idx, c, row_align=16)
    assert int(c[empty]) == 0
    return s, idx, c, off, dest, src


@pytest.mark.parametrize("T,k,d", [(1, 1, 8), (37, 2, 256), (300, 8, 4096), (2500, 1, 2560), (4096, 2, 8), (8192, 6, 2560),
                                   (8192, 8, 4096)])
def test_combine_bwd_vs_fp64(T, k, d):
    """combine_bwd on real 16-aligned routing (E = 64, one expert empty).
    dy[dest[t, j]] = bf16(dout[t] * s[t, j]) bit for bit: the product of two bf16 values is exact in fp32, so the one
    rounding is the reference's.  Every other row of dy (pad rows, rows past offsets[E]) is exactly zero, and the pad rows
    of y hold NaN, so a kernel that reads them fails.
    dscores[t, j] = <dout[t], y[dest[t, j]]> in fp32: each thread sums its share of the d products, then a warp and a block
    tree; the error is at most d 2^-24 sum |dout y| (n additions, each rounding by at most 2^-24 of a partial sum)."""
    ops = _ops()
    E = 64
    s, idx, c, off, dest, src = _aligned_routing(T, E, k, seed=T * 3 + k * 7 + d)
    g = _gen(T + d)
    rows = src.numel()
    y = torch.randn(rows, d, generator=g, device=DEV).to(bf16)
    y[src < 0] = float("nan")
    dout = torch.randn(T, d, generator=g, device=DEV).to(bf16)
    dy, ds = ops.combine_bwd(dout, y, dest, s)
    torch.cuda.synchronize()
    dl = dest.long()
    assert torch.unique(dl).numel() == T * k
    want = torch.zeros(rows, d, dtype=bf16, device=DEV)
    want[dl] = (dout.float()[:, None, :] * s.float()[:, :, None]).reshape(T * k, d).to(bf16)
    assert torch.equal(dy, want)
    worst = 0.0
    for t0 in range(0, T, 1024):
        t1 = min(T, t0 + 1024)
        do64 = dout[t0:t1].to(f64)
        y64 = y[dl.view(T, k)[t0:t1]].to(f64)                        # [t, k, d]
        ref = torch.einsum("td,tkd->tk", do64, y64)
        absdot = torch.einsum("td,tkd->tk", do64.abs(), y64.abs())
        err = (ds[t0:t1].to(f64) - ref).abs()
        bound = d * 2.0 ** -24 * absdot
        assert bool((err <= bound).all()), (t0, float((err / bound).max()))
        worst = max(worst, float((err / bound).max()))
    print(f"combine_bwd T={T} k={k} d={d}: dscores max err/bound {worst:.3e}")


# ------------------------------------------------------------------------------------------------ router backward
@pytest.mark.parametrize("T,E,k", [(1, 8, 1), (37, 8, 2), (300, 8, 8), (1000, 200, 1), (513, 200, 8), (4096, 64, 2),
                                   (8192, 64, 6), (20000, 64, 6)])
def test_router_bwd_vs_fp64(T, E, k):
    """Top-k softmax backward over given expert ids: dlogits[t, idx[t, j]] = s_j (g_j - sum_i s_i g_i), zero elsewhere.
    The kernel rounds each s g (2^-24), sums k <= 8 of them (2^-21 of sum |s g| in all), subtracts and multiplies
    (2^-23 of the result) and rounds to bf16 (2^-9): |got - ref| <= 2^-8 |ref| + 2^-20 s sum_i |s_i g_i|.
    Entries outside the selection are exactly zero; with k = 1, s = 1.0 is exact and so is the zero gradient."""
    ops = _ops()
    g = _gen(T * 5 + E + k)
    idx = torch.rand(T, E, generator=g, device=DEV).argsort(1)[:, :k].to(torch.int32).contiguous()
    s = torch.softmax(torch.randn(T, k, generator=g, device=DEV) * 2, -1).to(bf16)
    ds = torch.randn(T, k, generator=g, device=DEV) * 3
    dl = ops.router_bwd(ds, s, idx, E)
    torch.cuda.synchronize()
    if k == 1:
        assert bool((s == 1).all()) and bool((dl == 0).all())
        return
    sel = torch.zeros(T, E, dtype=torch.bool, device=DEV).scatter_(1, idx.long(), True)
    assert bool((dl[~sel] == 0).all())
    s64, g64 = s.to(f64), ds.to(f64)
    ref = s64 * (g64 - (s64 * g64).sum(1, keepdim=True))
    got = dl.gather(1, idx.long()).to(f64)
    bound = 2.0 ** -8 * ref.abs() + 2.0 ** -20 * s64 * (s64 * g64).abs().sum(1, keepdim=True)
    assert bool(((got - ref).abs() <= bound).all()), float(((got - ref).abs() / bound).max())


# ------------------------------------------------------------------------------------------------ dense data-gradient GEMMs
GEMM_KN = [(3328, 2560), (2560, 3328), (200, 256)]   # cfg 5: dx from the shared expert's gate/up, dhs from down_w; K % 64 != 0


@pytest.mark.parametrize("M", [1, 300, 8192])
@pytest.mark.parametrize("K,N", GEMM_KN)
def test_matmul_kn_vs_fp64(M, K, N):
    """matmul_kn (weight [K, N] read in place through the MN-major B path), three ways: contiguous A; A the right half of
    a [M, 2K] buffer (the `dhs1[:, Is:]` view) with a residual; A the left K columns of a [M, K + 64] buffer whose other
    columns are NaN, so a load past column K poisons the result."""
    ops = _ops()
    g = _gen(M * 13 + K + N)
    w = (torch.randn(K, N, generator=g, device=DEV) * 0.02).to(bf16)
    a = torch.randn(M, K, generator=g, device=DEV).to(bf16)
    assert_gemm_close(ops.matmul_kn(a, w), a, w, what=f"contiguous M={M} K={K} N={N}")
    wide = torch.randn(M, 2 * K, generator=g, device=DEV).to(bf16)
    res = (torch.randn(M, N, generator=g, device=DEV) * 0.5).to(bf16)
    av = wide[:, K:]
    assert_gemm_close(ops.matmul_kn(av, w, residual=res), av, w, residual=res, what=f"right view + residual M={M} K={K}")
    flank = torch.full((M, K + 64), float("nan"), dtype=bf16, device=DEV)
    flank[:, :K] = a
    got = ops.matmul_kn(flank[:, :K], w)
    assert_gemm_close(got, a, w, what=f"NaN-flanked view M={M} K={K}")
    torch.cuda.synchronize()


@pytest.mark.parametrize("M", [1, 300, 8192])
@pytest.mark.parametrize("nseg,K,N", [(2, 2560, 3328), (3, 2560, 3328), (2, 200, 256), (3, 200, 256)])
def test_linear_multi_vs_fp64(M, nseg, K, N):
    """linear_multi: [x @ W0.T | x @ W1.T (| x @ W2.T)] in one GEMM; cfg 5's shared-expert gate|up is 2560 -> 2 x 3328."""
    ops = _ops()
    g = _gen(M * 17 + nseg + K)
    ws = [(torch.randn(N, K, generator=g, device=DEV) * 0.02).to(bf16) for _ in range(nseg)]
    x = torch.randn(M, K, generator=g, device=DEV).to(bf16)
    got = ops.linear_multi(x, ws)
    assert got.shape == (M, nseg * N)
    assert_gemm_close(got, x, torch.cat(ws, 0).t(), what=f"linear_multi M={M} nseg={nseg} K={K} N={N}")


# ------------------------------------------------------------------------------------------------ the layer at cfg-5 width
def _layer_state(T, d, E, I, Is, k, empty, seed):
    """bf16 weights (std 0.02, as oracle.configs), x with a constant feature x[:, 0] = 1 and router row `empty` pointing
    against it (logit -2.5 sigma of the others: for it to be picked 58 of the 63 others would have to lie lower), so
    that expert receives no token.  It stays near the others' range, so it does not set the max|logit| that the
    near-tie rule scales by."""
    g = _gen(seed)
    w = {"router.weight": torch.randn(E, d, generator=g, device=DEV) * 0.02,
         "experts.fc1.weight": torch.randn(E, d, 2 * I, generator=g, device=DEV) * 0.02,
         "experts.fc2.weight": torch.randn(E, I, d, generator=g, device=DEV) * 0.02,
         "shared_experts.gate_proj.weight": torch.randn(Is, d, generator=g, device=DEV) * 0.02,
         "shared_experts.up_proj.weight": torch.randn(Is, d, generator=g, device=DEV) * 0.02,
         "shared_experts.down_proj.weight": torch.randn(d, Is, generator=g, device=DEV) * 0.02}
    x = torch.randn(T, d, generator=g, device=DEV)
    x[:, 0] = 1.0
    sigma = 0.02 * d ** 0.5
    w["router.weight"][empty] = 0.0
    w["router.weight"][empty, 0] = -2.5 * sigma
    gout = torch.randn(T, d, generator=g, device=DEV)
    return {n: v.to(bf16) for n, v in w.items()}, x.to(bf16), gout.to(bf16)


NAMES = ["router.weight", "experts.fc1.weight", "experts.fc2.weight", "shared_experts.gate_proj.weight",
         "shared_experts.up_proj.weight", "shared_experts.down_proj.weight"]


def _oracle_grads(w, x, gout, k, dtype):
    from oracle import aria_oracle as O
    wd = {n: v.to(dtype, copy=True).requires_grad_(True) for n, v in w.items()}
    xd = x.to(dtype, copy=True).requires_grad_(True)
    with torch.enable_grad():
        out, parts = O.moe_layer(xd, wd, k, return_parts=True)
        out.backward(gout.to(dtype))
    grads = {"dx": xd.grad, **{n: wd[n].grad for n in NAMES}}
    return out.detach(), parts, grads


def test_moe_layer_function_cfg5_vs_fp64_autograd():
    """MoELayerFunction forward + backward at BASELINE cfg 5 (T=8192, d=2560, E=64, k=6, I=1664, two shared experts)
    against fp64 autograd of the oracle's moe_layer on the same bf16 values.

    Tokens whose fp64 top-k margin is <= 2^-6 max|logit| (the suite's near-tie rule) get a zero upstream gradient; on
    every other token the GPU's expert set must equal the oracle's.  So nothing flows where the two may route
    differently, and every gradient is compared without routing slack.  The bar per gradient is rel-L2 <= 2 e16 + 1e-3,
    e16 being the error of bf16 eager autograd of the same oracle layer against fp64.  The same bar holds per expert for
    d_fc1 and d_fc2 (each expert's own e16) and for dx's worst token row, so one bad expert or block cannot hide in the
    whole-tensor norm.  Expert `empty` receives no token: its weight gradients are exactly zero, and so is dx on the
    zeroed tokens."""
    from aria_b200 import moe_train
    ops = _ops()
    T, d, E, k, I, Is, empty = 8192, 2560, 64, 6, 1664, 2 * 1664, 17
    w, x, gout = _layer_state(T, d, E, I, Is, k, empty, seed=5)
    # routing in fp64: the near-tie tokens lose their upstream gradient
    with torch.no_grad():
        from oracle import aria_oracle as O
        lg = O.router_gating(x.to(f64), w["router.weight"].to(f64))
        top = lg.sort(1, descending=True).values
        safe = (top[:, k - 1] - top[:, k]) / lg.abs().amax(1) > 2 ** -6
    assert int(safe.sum()) >= T // 2
    gout = gout.masked_fill(~safe[:, None], 0)
    out64, parts, ref = _oracle_grads(w, x, gout, k, f64)
    out16, _, ref16 = _oracle_grads(w, x, gout, k, bf16)
    assert int(parts["counts"][empty]) == 0
    _, idx, counts, _ = ops.router_topk(x, w["router.weight"], k)
    assert int(counts[empty]) == 0
    assert torch.equal(idx[safe].long().sort(1).values, parts["top_idx"][safe].sort(1).values)
    # ours
    wg = {n: v.clone().requires_grad_(True) for n, v in w.items()}
    xg = x.clone().requires_grad_(True)
    with torch.enable_grad():
        out = moe_train.MoELayerFunction.apply(xg, *[wg[n] for n in NAMES], k)
        out.backward(gout)
    torch.cuda.synchronize()
    got = {"dx": xg.grad, **{n: wg[n].grad for n in NAMES}}
    e_out, e16_out = _rel_l2(out[safe], out64[safe]), _rel_l2(out16[safe], out64[safe])
    print(f"\nout: rel-L2 {e_out:.3e}  bf16 eager {e16_out:.3e}")
    assert e_out <= 2 * e16_out + 1e-3
    for n in ["dx", *NAMES]:
        e, e16 = _rel_l2(got[n], ref[n]), _rel_l2(ref16[n], ref[n])
        print(f"{n}: rel-L2 {e:.3e}  bf16 eager {e16:.3e}")
        assert e <= 2 * e16 + 1e-3, (n, e, e16)
    for n in ("experts.fc1.weight", "experts.fc2.weight"):
        assert bool((got[n][empty] == 0).all()) and float(ref[n][empty].abs().max()) == 0.0
        worst = 0.0
        for e_ in range(E):
            if e_ == empty:
                continue
            e, e16 = _rel_l2(got[n][e_], ref[n][e_]), _rel_l2(ref16[n][e_], ref[n][e_])
            assert e <= 2 * e16 + 1e-3, (n, e_, e, e16)
            worst = max(worst, e / (2 * e16 + 1e-3))
        print(f"{n}: worst expert at {worst:.3f} of its bar")
    dx, dx64, dx16 = got["dx"].to(f64), ref["dx"], ref16["dx"].to(f64)
    assert bool((dx[~safe] == 0).all())
    rn = dx64[safe].norm(dim=1)
    row, row16 = float(((dx - dx64)[safe].norm(dim=1) / rn).max()), float(((dx16 - dx64)[safe].norm(dim=1) / rn).max())
    print(f"dx worst token row: rel-L2 {row:.3e}  bf16 eager {row16:.3e}")
    assert row <= 2 * row16 + 1e-3
