"""fp64 references and per-element error bounds for the GEMM kernels and their fused epilogues.

Every builder returns (ref, bound): `ref` is the fp64 value of the operation on the kernel's own operands (bf16 values, or
e4m3 codes times their scales), and `bound` is how far the kernel's output may lie from it, element by element.  `check`
compares.  The bounds follow the rounding points of the kernels (aria_b200/csrc/gemm_common.cuh: act_apply, epilogue_tile,
heads_store_tile; gemm.cu: the wide kernel's epilogues, which round at the same points):

  * fp32 accumulation of K exact bf16 x bf16 products: |acc - a @ b| <= ACC (|a| @ |b|), ACC = 2^-12.  Each addition
    rounds by at most 2^-24 of a partial sum, so K 2^-24 (|a| @ |b|) bounds it for K <= 4096; in practice the error is
    a random walk, far below that.  A dropped or doubled 64-wide k-block moves an element by the sum of 64 products, about
    8 / sqrt(K) of |a @ b| for random data, which is many times the bound.
  * each bf16 rounding of a stage whose exact value is v and whose error so far is e adds RND (|v| + e), RND = 2^-8:
    round-to-nearest moves a value by at most 2^-9 of it, and the other 2^-9 absorbs the few fp32 operations of the stage.
  * a stage's error is carried through the next operation by its Lipschitz constant (|gelu'| <= 1.13, |silu'| <= 1.1,
    x -> x^3 by (|x| + e)^3 - |x|^3, products by |x| e_y + |y| e_x + e_x e_y).
  * tanh.approx.f32 (GELU) is within TANH_APPROX of tanh relative to |tanh|, and the kernel's silu (ex2 / rcp approx)
    within 2^-20 + |g| 2^-23 of silu relative to |silu| (tests/test_gpu_moe_train_kernels.py::test_swiglu_fwd_vs_fp64).

So the bound of an element is small where its own value is small: a bar relative to the largest value of the tensor
would let such an element be wrong by far more than its size.  The builders take fp64-able tensors on any device, so
tests/test_gemm_ref_host.py can prove on the CPU that they accept a correctly rounded result and reject wrong ones.
"""
import math

import torch

F64 = torch.float64
ACC = 2.0 ** -12
RND = 2.0 ** -8
# PTX ISA: tanh.approx.f32 has a maximum relative error of about 2^-11; twice that is the bar
TANH_APPROX = 2.0 ** -10
GELU_LIP, SILU_LIP = 1.13, 1.1
ACT_NONE, ACT_GELU_TANH, ACT_GELU_NEW = 0, 1, 2   # aria_b200/_lib.py
_K0, _K1 = math.sqrt(2.0 / math.pi), 0.044715


def rnd(v, e):
    """Bound after one bf16 rounding of a stage of exact value v and error bound e."""
    return e + RND * (v.abs() + e)


def acc_ref(a, b, acc=ACC):
    """a [M, K] @ b [K, N] in fp64, and the fp32 accumulation bound acc (|a| @ |b|)."""
    a64, b64 = a.to(F64), b.to(F64)
    return a64 @ b64, acc * (a64.abs() @ b64.abs())


def gelu_tanh64(x):
    return 0.5 * x * (1 + torch.tanh(_K0 * (x + _K1 * x ** 3)))


def act_ref(z, ez, act):
    """The activation of the epilogue on z (exact value of the rounded stage, which the kernel holds to within ez), with its
    final bf16 rounding.  GELU_TANH is one fp32 evaluation: the input's error through |gelu'| <= 1.13, tanh.approx's error
    times 0.5 |x|, and the fp32 error of the tanh argument (~4 ops of 2^-24 each of |x| + 0.045 |x|^3) times 0.5 |x|.
    GELU_NEW is act_apply's op-by-op bf16 chain, each of its seven intermediate roundings bounded where it happens; its
    reference is NewGELU(z) with exact operations."""
    if act == ACT_NONE:
        return z, ez
    za = z.abs() + ez
    if act == ACT_GELU_TANH:
        y = gelu_tanh64(z)
        e = GELU_LIP * ez + 0.5 * za * (TANH_APPROX + 2.0 ** -21 * (za + za ** 3))
        return y, rnd(y, e)
    assert act == ACT_GELU_NEW
    p3 = z ** 3
    e = rnd(p3, za ** 3 - z.abs() ** 3)                     # bf16(x * x * x)
    t = _K1 * p3
    e = rnd(t, _K1 * e)                                      # bf16(0.044715 * p3)
    t = z + t
    e = rnd(t, ez + e)                                       # bf16(x + t)
    t = _K0 * t
    e = rnd(t, _K0 * e)                                      # bf16(sqrt(2/pi) * t)
    t = torch.tanh(t)
    e = rnd(t, e + TANH_APPROX * (t.abs() + e).clamp_max(1))  # bf16(tanh.approx(t))
    t = 1 + t
    e_t = rnd(t, e)                                          # bf16(1 + t)
    h = 0.5 * z
    e_h = rnd(h, 0.5 * ez)                                   # bf16(0.5 * x)
    y = h * t
    return y, rnd(y, h.abs() * e_t + t.abs() * e_h + e_h * e_t)   # h * t, rounded by the caller


def linear_ref(x, w, bias=None, act=ACT_NONE, residual=None, acc=ACC):
    """nn.Linear epilogue (EPI_LINEAR): out = bf16(bf16(act(bf16(x @ w.T + bias))) + residual).  The bias is added to the
    fp32 accumulator before the first rounding; the activation, if any, reads that bf16 value and is rounded again; the
    residual is added to the rounded result and rounded once more.  x [M, K], w [N, K] bf16 (or dequantized fp8 with a
    measured `acc`), bias [N], residual [M, N]."""
    z, e = acc_ref(x, w.t(), acc)
    if bias is not None:
        z = z + bias.to(F64)
    y, e = act_ref(z, rnd(z, e), act)
    if residual is not None:
        y = y + residual.to(F64)
        e = rnd(y, e)
    return y, e


def silu64(g):
    return g * torch.sigmoid(g)


def swiglu_ref(g, eg, u, eu):
    """EPI_SWIGLU on exact accumulator values g (gate), u (up) held to within eg, eu: out = bf16(bf16(silu(bf16 g)) bf16 u).
    silu moves the gate's error by at most 1.1 times; the kernel's silu adds eps(g) |silu| (for g < -87 rcp.approx flushes
    and silu may be 0, an error of |silu| < 2^-119).  The product of two bf16 values is exact in fp32."""
    eg, eu = rnd(g, eg), rnd(u, eu)
    s = silu64(g)
    ga = g.abs() + eg
    eps = torch.where(g - eg < -87, torch.ones_like(g), 2.0 ** -20 + ga * 2.0 ** -23)
    es = rnd(s, SILU_LIP * eg + eps * (s.abs() + SILU_LIP * eg))
    y = s * u
    return y, rnd(y, s.abs() * eu + u.abs() * es + es * eu)


def linear_swiglu_ref(x, gate_w, up_w, acc=ACC):
    g, eg = acc_ref(x, gate_w.t(), acc)
    u, eu = acc_ref(x, up_w.t(), acc)
    return swiglu_ref(g, eg, u, eu)


def rotate_half(x):
    h = x.shape[-1] // 2
    return torch.cat([-x[..., h:], x[..., :h]], -1)


def rope_ref(z, ez, cos, sin):
    """EPI_HEADS with RoPE on the exact accumulator values z [..., 128] (no bias: the RoPE epilogue has none), held to within
    ez, and the bf16 table rows cos / sin broadcast to z: out = bf16(bf16(bf16(z) cos) + bf16(rotate_half(bf16 z) sin)),
    HF's apply_rotary_pos_emb with op-by-op rounding."""
    ez = rnd(z, ez)
    c, s = cos.to(F64), sin.to(F64)
    zr, ezr = rotate_half(z), torch.cat([ez[..., ez.shape[-1] // 2:], ez[..., :ez.shape[-1] // 2]], -1)
    a, b = z * c, zr * s
    ea, eb = rnd(a, c.abs() * ez), rnd(b, s.abs() * ezr)
    y = a + b
    return y, rnd(y, ea + eb)


def grouped_ref(a, b, offsets, group_mod=0, b_nk=False, acc=ACC):
    """Rows off[g]:off[g+1] of a times weight block g % group_mod (g when group_mod = 0) of b ([E, K, N], or [E, N, K] with
    b_nk), before the epilogue: (acc value, acc bound) over all rows of a; rows outside every group are NaN."""
    off = [int(v) for v in offsets.tolist()]
    N = b.shape[1] if b_nk else b.shape[2]
    z = torch.full((a.shape[0], N), float("nan"), dtype=F64, device=a.device)
    e = torch.full_like(z, float("nan"))
    for g in range(len(off) - 1):
        if off[g + 1] > off[g]:
            w = b[g % group_mod if group_mod else g]
            z[off[g]:off[g + 1]], e[off[g]:off[g + 1]] = acc_ref(a[off[g]:off[g + 1]], w.t() if b_nk else w, acc)
    return z, e


def check(got, ref, bound, what="", tile=(128, 128)):
    """Asserts |got - ref| <= bound element by element (NaN fails) and returns the worst err / bound.  On failure it reports
    how many elements are out, the first one's index and (for 2-D outputs) its (row, col) tile of `tile`, and the worst
    err / bound."""
    err = (got.to(F64) - ref).abs()
    bad = ~(err <= bound)
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound.clamp_min(1e-300))
    worst = float(torch.nan_to_num(ratio, nan=float("inf")).max()) if ratio.numel() else 0.0
    if bool(bad.any()):
        idx = bad.nonzero()[0].tolist()
        where = f"index {idx}"
        if len(idx) == 2:
            where += f" (tile {idx[0] // tile[0]}, {idx[1] // tile[1]})"
        i = tuple(idx)
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.numel()} elements out of bound, first at {where}: got "
                             f"{float(got[i])}, ref {float(ref[i])}, bound {float(bound[i]):.3g}; worst err/bound {worst:.3g}")
    return worst


def assert_gemm_close(got, a, b, residual=None, what=""):
    """got = a @ b (+ residual) per element:  |got - ref64| <= 2^-8 |ref| + 2^-12 (|a| @ |b|)   [+ 2^-8 (|ref| + |res|)].
    2^-8 |ref| is one bf16 rounding of the output (bf16 keeps 8 significant bits, so a rounding moves a value by less
    than 2^-8 of it); 2^-12 (|a| @ |b|) covers fp32 accumulation (under K 2^-24 of it for K <= 4096) and is far below
    what a dropped or doubled 64-wide k-block moves (the |a||b| mass of 64 of the K products is about 64 / K of it, and
    their sum is not small against 2^-12 of the whole).  With a residual the epilogue rounds the product to bf16 before
    adding the residual and rounds again, so the first rounding adds 2^-8 |a @ b| <= 2^-8 (|ref| + |res|)."""
    ref, bound = acc_ref(a, b)
    if residual is not None:
        ref = ref + residual.to(F64)
        bound += 2.0 ** -8 * (ref.abs() + residual.to(F64).abs())
    bound += 2.0 ** -8 * ref.abs()
    return check(got, ref, bound, what)
