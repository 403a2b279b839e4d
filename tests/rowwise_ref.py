"""fp64 references for the row kernels of aria_b200/csrc/elementwise.cu, rounded to bf16 where the kernels round.

The norm and RoPE builders return (ref, allow): `ref` is the operation computed in fp64 on the kernel's own inputs and
rounded to bf16 (ties to even) at the points the kernel rounds; `allow` is, per element, how many bf16 ulps of ref the
kernel's output may lie from it.  allow is not a tolerance.  It is 0 wherever the kernel's fp32 arithmetic, at its worst,
cannot reach the other side of a bf16 rounding boundary, and elsewhere it is the distance to the bf16 value on the far
side.  So a correct kernel matches ref exactly except on the few elements whose exact value sits within the fp32 error
of a rounding boundary.  The fp32 error bounds follow the kernels' arithmetic (U = 2^-24, gamma(n) = n U / (1 - n U)):

  * a sum of n terms along a reduction tree of depth n is within gamma(n) sum|terms| of the exact sum.  The block kernels
    sum 8 MAXV terms per thread, then 5 shuffle levels and 3 adds across the 4 warps; the warp kernel 8 MAXV per lane,
    then 5 shuffle levels.  rstd = 1 / sqrtf(ss / d + eps) adds a few U; the square root halves the error of its argument.
  * rmsnorm rounds twice: inner = bf16(h rstd), then out = bf16(w inner).  w inner is exact in fp32 (two 8-bit
    significands), so the only freedom is which bf16 neighbour `inner` takes; the outer rounding follows from it.
  * layernorm rounds once, at the end: o = (h - mean) rstd w + b.  The fp32 mean is off by up to gamma(n) mean|h|, which
    for rows with a large common offset is large against h - mean.
  * cosf / sinf are within 2 fp32 ulps of the true value at any argument (CUDA C Programming Guide, single-precision
    functions); the angle itself is the one fp32 product float(pos) * inv_freq that transformers computes, so it is exact
    input, not error.

The copy kernels (embedding, add_pos_embedding, im2col_patches, merge_image_features) are bit-exact: their references are
index_select, bf16(x + table[pos]) (the fp32 sum of two bf16 values rounds to the same bf16 as the exact sum), unfold +
zero padding, and masked_scatter.  The builders take tensors on any device, so tests/test_rowwise_ref_host.py can show on
the CPU that they accept a correctly rounded result and reject each planted mistake.
"""
import math

import torch

F64 = torch.float64
bf16 = torch.bfloat16
U = 2.0 ** -24
E4M3_MAX = 448.0


def gamma(n):
    return n * U / (1 - n * U)


def bf16_rn(x):
    """fp64 x rounded to the nearest bf16 value, ties to even, kept in fp64.  Computed here because torch's fp64 -> bf16 cast
    goes through fp32 and can round twice (1 + 2^-8 + 2^-30 becomes the tie 1 + 2^-8 in fp32, then 1)."""
    _, e = torch.frexp(x)                                  # |x| in [2^(e-1), 2^e): bf16 spacing 2^(e-8), subnormal 2^-133
    step = torch.exp2((e.clamp_min(-125) - 8).to(F64))
    return torch.round(x / step) * step


def _exponent(v):
    """e with |v| in [2^(e-1), 2^e); -125 (the bf16 subnormal range) at 0."""
    _, e = torch.frexp(v)
    return torch.where(v == 0, torch.full_like(e, -125), e.clamp_min(-125)).to(F64)


def ulp(r):
    """bf16 spacing at r (the step above |r| at a power of two), 2^-133 at 0."""
    return torch.exp2(_exponent(r.to(F64)) - 8)


def ulps(got, ref):
    """|got - ref| in bf16 ulps of ref."""
    return (got.to(F64) - ref).abs() / ulp(ref)


def allow_within(ref, lo, hi):
    """Ulps of ref to the farthest bf16 value that correctly rounds some real in [lo, hi] (rounding is monotone, so those are
    the values between bf16(lo) and bf16(hi))."""
    return torch.maximum(ulps(bf16_rn(lo), ref), ulps(bf16_rn(hi), ref))


def f32(v):
    """A Python float as the kernel receives it (a C float argument)."""
    return float(torch.tensor(v, dtype=torch.float32))


def block_depth(d):
    """Reduction depth of the 128-thread block kernels (rmsnorm_kernel, rmsnorm_quantize_kernel, layernorm_kernel)."""
    return 8 * -(-(d // 8) // 128) + 5 + 3


def warp_depth(d):
    """Reduction depth of layernorm_warp_kernel (one warp per row)."""
    return 8 * -(-(d // 8) // 32) + 5


# ------------------------------------------------------------------------------------------------ norms
def residual_sum(x, residual=None):
    """h = bf16(x + residual) (sum_out, bit-exact) or x."""
    x64 = x.to(F64)
    return x64 if residual is None else bf16_rn(x64 + residual.to(F64))


def rmsnorm_ref(x, w, eps, residual=None):
    """LlamaRMSNorm as rmsnorm_kernel rounds it: h = bf16(x + res); out = bf16(w bf16(h rsqrt(mean(h^2) + eps))).
    Returns (h, out, allow)."""
    d = x.shape[-1]
    h = residual_sum(x, residual)
    w64 = w.to(F64)
    rstd = torch.rsqrt((h * h).mean(-1, keepdim=True) + f32(eps))
    v = h * rstd
    out = bf16_rn(w64 * bf16_rn(v))
    # ss: gamma(depth) (squares of bf16 are exact); / d, + eps: 3 U; sqrt halves; 1 / x, h * rstd: 2 U; 1 U of margin
    eps_in = (gamma(block_depth(d)) + 3 * U) / 2 + 3 * U
    lo, hi = bf16_rn(v - eps_in * v.abs()), bf16_rn(v + eps_in * v.abs())
    allow = torch.maximum(ulps(bf16_rn(w64 * lo), out), ulps(bf16_rn(w64 * hi), out))
    return h, out, allow


def quantize_ref(y):
    """permute_quantize_rows' per-row e4m3 quantiser on bf16 rows y [..., d]: scale = amax / 448 (fp32, IEEE division; 1 for
    an all-zero row) and codes = e4m3(y / scale), each quotient rounded to fp32 and then to e4m3, to nearest even.  Returns
    (codes as uint8, scale [rows] fp32).  The quotients are formed in fp64 and then rounded to fp32, because torch on CUDA
    divides by a scalar as a multiplication by its reciprocal.  That is the IEEE fp32 quotient: a bf16 value (8 bits) over
    an fp32 one (24 bits) is either an fp32 rounding boundary (25 bits) or at least 2^-49 of itself away from one, so the
    fp64 rounding (2^-53) cannot move it across."""
    yd = y.to(bf16).double().reshape(-1, y.shape[-1])
    amax = yd.abs().amax(-1)
    scale = torch.where(amax > 0, amax / E4M3_MAX, torch.ones_like(amax)).float()
    q = (yd / scale.double()[:, None]).float().to(torch.float8_e4m3fn)
    return q.view(torch.uint8).view(y.shape), scale


def layernorm_ref(x, w, b, eps, depth=None):
    """nn.LayerNorm as layernorm_kernel / layernorm_warp_kernel compute it: fp32 mean and variance of the bf16 row,
    o = (h - mean) rstd w + b, one rounding.  `depth`: the reduction depth of the kernel that runs (default: the deeper of
    the two that can run at this width).  Returns (out, allow)."""
    d = x.shape[-1]
    if depth is None:
        depth = max(block_depth(d), warp_depth(d) if d // 8 <= 160 else 0)
    h, w64, b64 = x.to(F64), w.to(F64), b.to(F64)
    m = h.mean(-1, keepdim=True)
    c = h - m
    var = (c * c).mean(-1, keepdim=True)
    e2 = f32(eps)
    rstd = torch.rsqrt(var + e2)
    t = c * rstd * w64
    o = t + b64
    out = bf16_rn(o)
    # mean: the sum's gamma(depth) sum|h|, then * fp32(1/d): 2 U of |mean|
    e_m = gamma(depth) * h.abs().mean(-1, keepdim=True) + 2 * U * m.abs()
    # variance of fp32 deltas (each off by e_m, rounded, squared, summed), / d, + eps; relative to var + eps
    e_v = gamma(depth + 3) * (var + e_m * e_m) + e_m * e_m + 3 * U * (var + e2)
    eps_r = e_v / (var + e2) / 2 + 3 * U
    err = w64.abs() * rstd * (e_m + c.abs() * (eps_r + 3 * U)) * (1 + 2 * eps_r) + 3 * U * (t.abs() + b64.abs())
    return out, allow_within(out, o - err, o + err)


# ------------------------------------------------------------------------------------------------ rope table
def rope_angles(inv_freq, n_pos):
    """The fp32 angles float32(pos) * inv_freq[j] (one fp32 product, as transformers' LlamaRotaryEmbedding computes them),
    [n_pos, hd / 2]."""
    pos = torch.arange(n_pos, dtype=torch.float32, device=inv_freq.device)
    return pos[:, None] * inv_freq.float()[None, :]


def rope_table_ref(inv_freq, n_pos, ang=None):
    """cos / sin tables [n_pos, hd] (emb = cat(freqs, freqs)): fp64 cos and sin of the fp32 angle, one bf16 rounding.
    cosf / sinf are within 2 fp32 ulps of the true value.  Returns ((cos, allow_cos), (sin, allow_sin))."""
    a = rope_angles(inv_freq, n_pos) if ang is None else ang
    a = torch.cat([a, a], -1).to(F64)
    res = []
    for v in (torch.cos(a), torch.sin(a)):
        err = torch.where(v == 0, 0.0, 2 * torch.exp2(_exponent(v) - 24))      # 2 fp32 ulps of v
        ref = bf16_rn(v)
        res.append((ref, allow_within(ref, v - err, v + err)))
    return tuple(res)


# ------------------------------------------------------------------------------------------------ gathers (bit-exact)
def embedding_ref(ids, table):
    return table.index_select(0, ids.reshape(-1)).view(*ids.shape, table.shape[1])


def add_pos_ref(x, pos_ids, table):
    """bf16(x + table[pos]) per element."""
    return bf16_rn(x.to(F64) + table.index_select(0, pos_ids.reshape(-1)).to(F64).view(x.shape)).to(bf16)


def im2col_ref(pixels, P, k_pad):
    """patches[b * n^2 + py * n + px, c P^2 + i P + j] = pixels[b, c, py P + i, px P + j], columns past 3 P^2 zero."""
    B, C, S, _ = pixels.shape
    n = S // P
    p = pixels.view(B, C, n, P, n, P).permute(0, 2, 4, 1, 3, 5).reshape(B * n * n, C * P * P)
    return torch.nn.functional.pad(p, (0, k_pad - C * P * P))


def merge_ref(ids, image_token, features, embeds):
    """masked_scatter of features' leading rows into embeds' image-token rows.  Returns (embeds', count)."""
    mask = (ids.reshape(-1) == image_token)
    out = embeds.clone()
    n = int(mask.sum())
    out.view(-1, out.shape[-1])[mask] = features.reshape(-1, features.shape[-1])[:n]
    return out, n


# ------------------------------------------------------------------------------------------------ checks
def check_ulps(got, ref, allow, what="", min_exact=0.0):
    """Asserts |got - ref| <= allow ulps of ref element by element (NaN fails), and that at most (1 - min_exact) n + 2 of the
    n elements differ from ref (two spare, so that a small case may flip a boundary element).  Returns (exact fraction,
    worst ulps, fraction of elements with allow > 0).  On failure it reports how many elements are out, the first one's
    index, and its got / ref / allowance."""
    du = ulps(got, ref)
    bad = ~(du <= allow)
    n = max(du.numel(), 1)
    n_exact = int((du == 0).sum())
    exact = n_exact / n
    worst = float(torch.nan_to_num(du, nan=math.inf).max()) if du.numel() else 0.0
    band = float((allow > 0).sum()) / n
    if bool(bad.any()):
        idx = bad.nonzero()[0].tolist()
        i = tuple(idx)
        raise AssertionError(f"{what}: {int(bad.sum())}/{du.numel()} elements out of their allowance, first at index {idx}: "
                             f"got {float(got[i])!r}, ref {float(ref[i])!r}, {float(du[i]):.3g} ulps, allowed "
                             f"{float(allow[i]):.3g}; worst {worst:.3g} ulps, exact {exact:.5%}")
    assert n - n_exact <= (1 - min_exact) * n + 2, \
        f"{what}: {n - n_exact}/{n} elements differ from the reference ({exact:.5%} exact), more than {1 - min_exact:.3%} + 2"
    return exact, worst, band


def check_bits(got, ref, what=""):
    """Bit-exact comparison (so -0 != +0 and NaN payloads count); reports the first differing index."""
    assert got.shape == ref.shape and got.dtype == ref.dtype, (what, got.shape, ref.shape, got.dtype, ref.dtype)
    itype = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[got.element_size()]
    diff = got.view(itype) != ref.view(itype)
    if bool(diff.any()):
        idx = diff.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(diff.sum())}/{diff.numel()} elements differ, first at index {idx}: got "
                             f"{float(got[tuple(idx)].float())!r}, ref {float(ref[tuple(idx)].float())!r}")
