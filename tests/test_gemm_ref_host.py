"""CPU: the fp64 references and bounds of tests/gemm_ref.py accept a correctly rounded GEMM and reject wrong ones.

A "kernel" here is an emulation on the CPU of what the CUDA kernels compute: fp32 accumulation one 64-wide k-block at a
time, then the epilogue's bf16 roundings at the kernel's points (gemm_common.cuh), with the approximate tanh and silu
pushed to the edge of their stated error.  Each test takes small versions of the GPU test's shapes (a 128 x 128 tile and
its neighbours, k-blocks with a 8-element tail) and N(0, 1) activations with 0.02-std weights.  The bounds must accept the
emulation, and must reject each mistake a tiled GEMM can make: one k-block dropped from or added twice to one tile, a row
shifted by one, a neighbouring segment's bias on one tile, gate and up swapped, the activation skipped on one tile, RoPE at
the next position, and one group multiplied by its neighbour's weight.

Not in that list: erf GELU in place of tanh GELU.  The two differ by less than 2^-11 |x| everywhere, which is below the
error tanh.approx.f32 itself may make (relative 2^-11 of tanh, times 0.5 |x|), so no per-element bound that a correct
kernel passes can tell them apart.

The last tests keep the GPU suite complete: every GEMM entry of aria_b200.ops must be called by a per-element fp64 test,
and listed in the docstring of tests/test_gpu_gemm_fp64.py.
"""
import ast
import math
import os
import re

import pytest
import torch

import gemm_ref as R

bf16 = torch.bfloat16
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BK = 64


def _r(x):
    return x.to(bf16).float()


def _operands(M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g).to(bf16)
    w = (torch.randn(N, K, generator=g) * 0.02).to(bf16)
    a[M // 2] = 0                                   # a row of exact zeros
    if M > 2 and K % 2 == 0:                        # cancellation: ref[M-1, 0] = 0 with |a| @ |w| large
        a[M - 1, K // 2:] = a[M - 1, :K // 2]
        w[0, K // 2:] = -w[0, :K // 2]
    a[3, 5] = 60.0                                  # one large outlier in the tile
    return a, w


def _acc(a, w, drop=None, twice=None):
    """fp32 accumulation over 64-wide k-blocks; drop / twice = (k-block, rows, cols) applied to that region only."""
    af, wf = a.float(), w.float().t()
    acc = torch.zeros(a.shape[0], w.shape[0])
    for kb in range(0, a.shape[1], BK):
        part = af[:, kb:kb + BK] @ wf[kb:kb + BK]
        mult = torch.ones_like(part)
        for m, f in ((drop, 0.0), (twice, 2.0)):
            if m is not None and m[0] == kb // BK:
                mult[m[1], m[2]] = f
        acc = acc + part * mult
    return acc


def _tanh_approx(x, sign):
    """tanh at the edge of tanh.approx.f32's relative error (2^-11), rounded to fp32."""
    return (torch.tanh(x.double()) * (1 + sign * 2.0 ** -11)).float()


def _act(x, act, sign=1):
    if act == R.ACT_GELU_TANH:
        inner = 0.7978845608028654 * (x + 0.044715 * x * x * x)
        return 0.5 * x * (1 + _tanh_approx(inner, sign))
    if act == R.ACT_GELU_NEW:
        p3 = _r(x * x * x)
        t = _r(0.044715 * p3)
        t = _r(x + t)
        t = _r(0.7978845608028654 * t)
        t = _r(_tanh_approx(t, sign))
        t = _r(1.0 + t)
        return _r(0.5 * x) * t
    return x


def _linear_kernel(acc, bias, act, residual, sign=1, act_tiles=None):
    x = acc + bias.float() if bias is not None else acc.clone()
    x = _r(x)
    y = _r(_act(x, act, sign))
    if act_tiles is not None:                       # the activation skipped on these (rows, cols)
        y[act_tiles] = x[act_tiles]
    if residual is not None:
        y = _r(y + residual.float())
    return y.to(bf16)


M, N, K = 160, 264, 200     # tiles (0..1) x (0..2), k-blocks 0..3 with an 8-element tail


@pytest.mark.parametrize("act", [R.ACT_NONE, R.ACT_GELU_TANH, R.ACT_GELU_NEW])
@pytest.mark.parametrize("with_bias", [False, True])
@pytest.mark.parametrize("with_res", [False, True])
@pytest.mark.parametrize("sign", [1, -1])
def test_linear_bound_accepts_the_rounded_result(act, with_bias, with_res, sign):
    a, w = _operands(M, N, K, seed=act * 4 + with_bias * 2 + with_res)
    g = torch.Generator().manual_seed(7)
    bias = (torch.randn(N, generator=g) * 0.5).to(bf16) if with_bias else None
    res = torch.randn(M, N, generator=g).to(bf16) if with_res else None
    got = _linear_kernel(_acc(a, w), bias, act, res, sign)
    ref, bound = R.linear_ref(a, w, bias, act, res)
    worst = R.check(got, ref, bound, "emulated kernel")
    assert worst > 0.01          # the bound is not vacuous: some element uses a real part of it


@pytest.mark.parametrize("act", [R.ACT_NONE, R.ACT_GELU_TANH, R.ACT_GELU_NEW])
def test_linear_bound_rejects_a_dropped_or_doubled_k_block(act):
    a, w = _operands(M, N, K, seed=11)
    ref, bound = R.linear_ref(a, w, None, act)
    tile = (slice(0, 128), slice(0, 128))
    for kb in range(4):          # the 8-element tail block too
        for how in ("drop", "twice"):
            acc = _acc(a, w, **{how: (kb, *tile)})
            with pytest.raises(AssertionError, match=r"tile 0, 0"):
                R.check(_linear_kernel(acc, None, act, None), ref, bound, f"{how} k-block {kb}")


def test_linear_bound_rejects_a_row_shifted_by_one():
    a, w = _operands(M, N, K, seed=12)
    ref, bound = R.linear_ref(a, w)
    got = _linear_kernel(_acc(a, w), None, R.ACT_NONE, None)
    got[129] = got[130]
    with pytest.raises(AssertionError, match=r"index \[129, "):
        R.check(got, ref, bound, "row shift")


def test_linear_bound_rejects_the_neighbouring_segments_bias():
    """Two weights side by side (q | k of a fused projection, 2 x 128 columns), each with its own bias: the kernel's first
    tile of segment 1 taking segment 0's bias (the bias chosen per tile from the wrong column) fails."""
    a, w = _operands(M, 256, K, seed=13)
    g = torch.Generator().manual_seed(8)
    b0, b1 = (torch.randn(128, generator=g) * 0.5).to(bf16), (torch.randn(128, generator=g) * 0.5).to(bf16)
    bias = torch.cat([b0, b1])
    ref, bound = R.linear_ref(a, w, bias)
    R.check(_linear_kernel(_acc(a, w), bias, R.ACT_NONE, None), ref, bound, "right biases")
    wrong = torch.cat([b0, b0])
    with pytest.raises(AssertionError, match=r"tile 0, 1"):
        R.check(_linear_kernel(_acc(a, w), wrong, R.ACT_NONE, None), ref, bound, "segment 0's bias on segment 1")


@pytest.mark.parametrize("act", [R.ACT_GELU_TANH, R.ACT_GELU_NEW])
def test_linear_bound_rejects_a_tile_without_its_activation(act):
    a, w = _operands(M, N, K, seed=14)
    ref, bound = R.linear_ref(a, w, None, act)
    got = _linear_kernel(_acc(a, w), None, act, None, act_tiles=(slice(128, 160), slice(256, 264)))
    with pytest.raises(AssertionError, match=r"tile 1, 2"):
        R.check(got, ref, bound, "no activation on tile (1, 2)")


def _swiglu_kernel(g_acc, u_acc, sign=1):
    g, u = _r(g_acc), _r(u_acc)
    eps = 2.0 ** -20 + g.abs() * 2.0 ** -23
    s = _r((g.double() * torch.sigmoid(g.double()) * (1 + sign * eps.double())).float())
    return (s * u).to(bf16)


@pytest.mark.parametrize("sign", [1, -1])
def test_swiglu_bound_accepts_the_rounded_result_and_rejects_swapped_gate_and_up(sign):
    a, gw = _operands(M, 192, K, seed=15)
    uw = (torch.randn(192, K, generator=torch.Generator().manual_seed(9)) * 0.02).to(bf16)
    gw = gw * 8                                     # gates of a few units, where silu is far from linear
    ref, bound = R.linear_swiglu_ref(a, gw, uw)
    R.check(_swiglu_kernel(_acc(a, gw), _acc(a, uw), sign), ref, bound, "emulated swiglu")
    with pytest.raises(AssertionError):
        R.check(_swiglu_kernel(_acc(a, uw), _acc(a, gw), sign), ref, bound, "gate and up swapped")


def _rope_tables(n_pos, dim=128, base=10000.0):
    inv = 1.0 / base ** (torch.arange(0, dim, 2, dtype=torch.float64) / dim)
    f = torch.outer(torch.arange(n_pos, dtype=torch.float64), inv)
    emb = torch.cat([f, f], -1)
    return emb.cos().to(bf16), emb.sin().to(bf16)


def _rope_kernel(acc, cos, sin):
    x = _r(acc)
    c, s = cos.float(), sin.float()
    h = x.shape[-1] // 2
    lo = _r(_r(x[..., :h] * c[..., :h]) + _r(-x[..., h:] * s[..., :h]))
    hi = _r(_r(x[..., h:] * c[..., h:]) + _r(x[..., :h] * s[..., h:]))
    return torch.cat([lo, hi], -1).to(bf16)


def test_rope_bound_accepts_the_rounded_result_and_rejects_the_next_position():
    T, pos0 = 40, 5
    a, w = _operands(T, 256, K, seed=16)           # two heads of 128
    cos, sin = _rope_tables(64)
    pos = pos0 + torch.arange(T)
    acc = _acc(a, w).view(T, 2, 128)
    z, e = R.acc_ref(a, w.t())
    ref, bound = R.rope_ref(z.view(T, 2, 128), e.view(T, 2, 128), cos[pos][:, None], sin[pos][:, None])
    got = _rope_kernel(acc, cos[pos][:, None], sin[pos][:, None])
    R.check(got, ref, bound, "emulated rope")
    with pytest.raises(AssertionError):
        R.check(_rope_kernel(acc, cos[pos + 1][:, None], sin[pos + 1][:, None]), ref, bound, "rope at p + 1")


def test_grouped_bound_accepts_the_rounded_result_and_rejects_the_neighbours_weight():
    counts = [0, 1, 65, 0, 130, 7]
    off = torch.tensor([0] + torch.tensor(counts).cumsum(0).tolist(), dtype=torch.int32)
    rows, E, Kg, Ng = int(off[-1]), len(counts), 128, 192
    g = torch.Generator().manual_seed(17)
    a = torch.randn(rows, Kg, generator=g).to(bf16)
    b = (torch.randn(E, Kg, Ng, generator=g) * 0.02).to(bf16)
    z, e = R.grouped_ref(a, b, off)
    ref, bound = z, R.rnd(z, e)

    def kernel(wmap):
        out = torch.empty(rows, Ng, dtype=bf16)
        for gi in range(E):
            r0, r1 = int(off[gi]), int(off[gi + 1])
            out[r0:r1] = _r(_acc(a[r0:r1], b[wmap(gi)].t())).to(bf16)
        return out

    R.check(kernel(lambda gi: gi), ref, bound, "emulated grouped")
    with pytest.raises(AssertionError, match=r"index \[66, "):   # group 4 (rows 66..195) with group 5's weight
        R.check(kernel(lambda gi: gi + 1 if gi == 4 else gi), ref, bound, "neighbour's weight")


def test_check_reports_count_index_tile_and_worst_ratio():
    ref = torch.zeros(300, 300, dtype=torch.float64)
    bound = torch.full_like(ref, 0.5)
    got = ref.clone()
    got[130, 260] = 2.0
    got[299, 0] = float("nan")
    with pytest.raises(AssertionError) as ex:
        R.check(got, ref, bound, "probe")
    msg = str(ex.value)
    assert "2/90000" in msg and "index [130, 260] (tile 1, 2)" in msg and "worst err/bound inf" in msg
    got[299, 0] = 0
    got[130, 260] = 0.25
    assert math.isclose(R.check(got, ref, bound), 0.5)


# ------------------------------------------------------------------------------------------------ every GEMM entry is covered
def _gemm_entries():
    """Public functions of aria_b200/ops.py that launch a GEMM: they call _run_gemm / _run_gemm_w8a8 or a C entry whose
    name contains `gemm` or `wgrad`."""
    tree = ast.parse(open(os.path.join(ROOT, "aria_b200", "ops.py")).read())
    out = []
    for f in tree.body:
        if not isinstance(f, ast.FunctionDef) or f.name.startswith("_"):
            continue
        for n in ast.walk(f):
            if isinstance(n, ast.Call):
                fn = n.func
                name = fn.id if isinstance(fn, ast.Name) else fn.attr if isinstance(fn, ast.Attribute) else ""
                if name in ("_run_gemm", "_run_gemm_w8a8") or re.fullmatch(r"aria_\w*(gemm|wgrad)\w*", name):
                    out.append(f.name)
                    break
    return out


def test_gemm_entries_are_found():
    got = set(_gemm_entries())
    assert {"linear", "linear_multi", "linear_swiglu", "qkv_heads", "matmul_kn", "grouped_gemm", "grouped_gemm_nt",
            "grouped_gemm_regions", "grouped_wgrad", "wgrad_accumulate_f32", "grouped_gemm_fp8", "grouped_gemm_w8a8",
            "linear_w8a8", "linear_swiglu_w8a8", "qkv_heads_w8a8"} <= got


def test_every_gemm_entry_has_an_fp64_test():
    src = "".join(open(os.path.join(HERE, f)).read() for f in ("test_gpu_gemm_fp64.py", "test_gpu_moe_train_kernels.py"))
    missing = [n for n in _gemm_entries() if not re.search(rf"\bops\.{n}\(", src)]
    assert not missing, f"GEMM entries of ops without a per-element fp64 test: {missing}"


def test_every_gemm_entry_is_in_the_fp64_test_docstring():
    doc = ast.get_docstring(ast.parse(open(os.path.join(HERE, "test_gpu_gemm_fp64.py")).read()))
    missing = [n for n in _gemm_entries() if not re.search(rf"`{n}`", doc)]
    assert not missing, f"not in test_gpu_gemm_fp64.py's docstring: {missing}"
