"""CPU: the fp64 references of tests/rowwise_ref.py accept a correctly rounded result and reject each planted mistake.

A "kernel" here is an emulation on the CPU of what the row kernels of aria_b200/csrc/elementwise.cu compute, in fp32 with
bf16 roundings at the kernels' points, or torch's / transformers' own fp32 implementation of the operation rounded to bf16.
The references must accept both, and reject: eps applied outside the square root, the last 8-element vector of a row left
unnormalized, the residual sum not rounded before the norm, weight and bias (or the two halves of a 16-byte vector)
swapped, a scale computed by a reciprocal, RoPE angles in fp64 or at the next position, one image row shifted by one
pixel, a padding column that is not +0, and feature rows taken from the next slot.

The last tests keep the GPU suite complete: every row-wise entry of aria_b200.ops is called by
tests/test_gpu_rowwise_fp64.py, every kernel of elementwise.cu is named in its docstring, and the dispatch rule it restates
to name the kernel of each case is the one elementwise.cu applies.
"""
import ast
import os
import re

import pytest
import torch
import torch.nn.functional as F

import rowwise_ref as R

bf16 = torch.bfloat16
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EPS_RMS, EPS_LN = 1e-5, 1e-6
ROW_EXP = [-20, 0, 20, -10, 10, 0]          # row magnitudes 2^e: a row normalised with another row's statistics is far off


def _r(x):
    return x.to(bf16).float()


def _rows(rows, d, seed, offset_every=0):
    """bf16 [rows, d]: N(0, 1) rows scaled by 2^ROW_EXP[r % 6], row rows // 2 all zero, and (offset_every) rows with
    mean 1e3 and spread 1."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, d, generator=g)
    x *= torch.exp2(torch.tensor([float(ROW_EXP[r % len(ROW_EXP)]) for r in range(rows)]))[:, None]
    if offset_every:
        x[::offset_every] = 1e3 + torch.randn(x[::offset_every].shape, generator=g)
    x[rows // 2] = 0
    return x.to(bf16)


def _wb(d, seed):
    g = torch.Generator().manual_seed(seed)
    w = 1 + 0.1 * torch.randn(d, generator=g)
    w[::97] *= -1                                   # a few negative weights: the sign of a zero output follows w
    return w.to(bf16), (0.1 * torch.randn(d, generator=g)).to(bf16)


def _swap_words(v):
    """The two bf16 halves of every 32-bit word swapped (bf16_lo / bf16_hi mixed up)."""
    return v.reshape(*v.shape[:-1], -1, 2).flip(-1).reshape(v.shape)


def _swap_halves(v):
    """The two 8-byte halves of every 16-byte vector swapped."""
    return v.reshape(*v.shape[:-1], -1, 2, 4).flip(-2).reshape(v.shape)


# ------------------------------------------------------------------------------------------------ rmsnorm
def _rms_kernel(x, w, eps, res=None, eps_outside=False, tail=False, unrounded=False, swap_w=False):
    """rmsnorm_kernel in fp32: returns (sum_out, out)."""
    d = x.shape[-1]
    h = x.float() + res.float() if res is not None else x.float()
    hr = _r(h)
    hn = h if unrounded else hr
    ms = (hn * hn).sum(-1, keepdim=True) * R.f32(1.0 / d)
    rstd = 1 / (ms.sqrt() + eps) if eps_outside else 1 / (ms + eps).sqrt()
    wf = _swap_words(w.float()) if swap_w else w.float()
    y = _r(wf * _r(hn * rstd))
    if tail:
        y[:, -8:] = hr[:, -8:]
    return hr.to(bf16), y.to(bf16)


D_RMS = [8, 1032, 4096]


@pytest.mark.parametrize("d", D_RMS)
@pytest.mark.parametrize("with_res", [False, True])
def test_rmsnorm_ref_accepts_the_rounded_result(d, with_res):
    from transformers.models.llama.modeling_llama import LlamaRMSNorm
    x, res = _rows(24, d, 1), (_rows(24, d, 2) if with_res else None)
    if with_res:
        x[12] = -res[12]                             # h = x + res = 0 in that row
    w, _ = _wb(d, 3)
    h, ref, allow = R.rmsnorm_ref(x, w, EPS_RMS, res)
    s, got = _rms_kernel(x, w, EPS_RMS, res)
    R.check_bits(s, h.to(bf16), "sum_out")
    exact, worst, band = R.check_ulps(got, ref, allow, "emulated rmsnorm_kernel", min_exact=0.99)
    assert band < 0.01                               # the allowance is a narrow band around the rounding boundaries
    hf = LlamaRMSNorm(d, eps=EPS_RMS).to(bf16)
    with torch.no_grad():
        hf.weight.copy_(w)
        R.check_ulps(hf(h.to(bf16)), ref, allow, "transformers LlamaRMSNorm", min_exact=0.99)
    assert bool((ref[12] == 0).all())


@pytest.mark.parametrize("plant", ["eps_outside", "tail", "unrounded", "swap_w"])
def test_rmsnorm_ref_rejects(plant):
    d = 1032
    x, res = _rows(24, d, 4), _rows(24, d, 5)
    w, _ = _wb(d, 6)
    _, ref, allow = R.rmsnorm_ref(x, w, EPS_RMS, res)
    _, got = _rms_kernel(x, w, EPS_RMS, res, **{plant: True})
    with pytest.raises(AssertionError, match="out of their allowance"):
        R.check_ulps(got, ref, allow, plant)


def test_quantize_ref_matches_the_kernels_arithmetic_and_rejects_a_reciprocal_scale():
    """Rows whose amax runs through all 128 bf16 significands: the scale amax / 448 (IEEE) and amax * (1 / 448) differ on
    some; codes rounded toward zero differ from round-to-nearest-even.  An all-zero row has scale 1 and +0 codes."""
    sig = 1 + torch.arange(128) / 128.0
    g = torch.Generator().manual_seed(7)
    y = (torch.rand(129, 64, generator=g) * 2 - 1)
    y[:128, 0] = sig
    y[:128] = y[:128].clamp(-1, 1) * sig[:, None] * 2.0 ** torch.randint(-10, 10, (128, 1), generator=g)
    y[128] = 0
    y = y.to(bf16)
    q, s = R.quantize_ref(y)
    assert float(s[128]) == 1.0 and bool((q[128] == 0).all())
    yf = y.float()
    amax = yf.abs().amax(-1)
    s_k = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    R.check_bits(s_k, s, "scale")
    R.check_bits((yf / s_k[:, None]).to(torch.float8_e4m3fn).view(torch.uint8), q, "codes")
    with pytest.raises(AssertionError, match="differ"):
        R.check_bits(torch.where(amax > 0, amax * (1.0 / 448.0), torch.ones_like(amax)), s, "reciprocal scale")
    exact = yf / s[:, None]
    toward0 = torch.where(q.view(torch.float8_e4m3fn).float().abs() > exact.abs(), q - 1, q)   # magnitude codes are ordered
    with pytest.raises(AssertionError, match="differ"):
        R.check_bits(toward0, q, "codes rounded toward zero")


# ------------------------------------------------------------------------------------------------ layernorm
def _ln_kernel(x, w, b, eps, eps_outside=False, tail=False, swap=None):
    """layernorm_kernel in fp32 (two-pass mean and variance), one rounding."""
    d = x.shape[-1]
    h = x.float()
    mean = h.sum(-1, keepdim=True) * R.f32(1.0 / d)
    var = ((h - mean) ** 2).sum(-1, keepdim=True) * R.f32(1.0 / d)
    rstd = 1 / (var.sqrt() + eps) if eps_outside else 1 / (var + eps).sqrt()
    wf, bf = w.float(), b.float()
    if swap == "w_b_words":                          # weight and bias swapped on the high half of every 32-bit word
        wf, bf = wf.clone(), bf.clone()
        wf[1::2], bf[1::2] = b.float()[1::2], w.float()[1::2]
    elif swap == "b_halves":
        bf = _swap_halves(bf)
    o = (h - mean) * rstd * wf + bf
    if tail:
        o[:, -8:] = h[:, -8:]
    return o.to(bf16)


@pytest.mark.parametrize("d", [8, 1152, 1288, 4096])
def test_layernorm_ref_accepts_the_rounded_result(d):
    x = _rows(30, d, 8, offset_every=5)
    w, b = _wb(d, 9)
    ref, allow = R.layernorm_ref(x, w, b, EPS_LN)
    R.check_ulps(_ln_kernel(x, w, b, EPS_LN), ref, allow, "emulated layernorm_kernel")
    R.check_ulps(F.layer_norm(x.float(), (d,), w.float(), b.float(), EPS_LN).to(bf16), ref, allow, "torch fp32 LayerNorm")
    R.check_ulps(F.layer_norm(x, (d,), w, b, EPS_LN), ref, allow, "torch bf16 LayerNorm")
    plain = torch.ones(30, dtype=torch.bool)
    plain[::5] = False
    _, _, band = R.check_ulps(_ln_kernel(x, w, b, EPS_LN)[plain], ref[plain], allow[plain], "rows without an offset",
                              min_exact=0.99)
    assert band < 0.01


@pytest.mark.parametrize("plant", ["eps_outside", "tail", "w_b_words", "b_halves"])
def test_layernorm_ref_rejects(plant):
    d = 1152
    x = _rows(30, d, 10, offset_every=5)
    w, b = _wb(d, 11)
    ref, allow = R.layernorm_ref(x, w, b, EPS_LN)
    kw = {"swap": plant} if plant in ("w_b_words", "b_halves") else {plant: True}
    with pytest.raises(AssertionError, match="out of their allowance"):
        R.check_ulps(_ln_kernel(x, w, b, EPS_LN, **kw), ref, allow, plant)


# ------------------------------------------------------------------------------------------------ rope table
def _hf_rope(hd, n_pos, theta):
    from transformers import LlamaConfig
    from transformers.models.llama.modeling_llama import LlamaRotaryEmbedding
    cfg = LlamaConfig(hidden_size=hd * 4, num_attention_heads=4, head_dim=hd, max_position_embeddings=n_pos,
                      rope_parameters={"rope_type": "default", "rope_theta": theta})
    rot = LlamaRotaryEmbedding(cfg)
    cos, sin = rot(torch.zeros(1, dtype=bf16), torch.arange(n_pos)[None])
    return rot.inv_freq, cos[0], sin[0]


def test_rope_ref_accepts_transformers_table_and_rejects_fp64_angles_and_the_next_position():
    n_pos, hd = 8192, 128
    inv_freq, hf_cos, hf_sin = _hf_rope(hd, n_pos, 5e6)
    (cos, ac), (sin, asn) = R.rope_table_ref(inv_freq, n_pos)
    for got, ref, allow, what in ((hf_cos, cos, ac, "cos"), (hf_sin, sin, asn, "sin")):
        _, _, band = R.check_ulps(got, ref, allow, f"transformers {what}", min_exact=0.99)
        assert band < 0.01
    a64 = torch.arange(n_pos, dtype=torch.float64)[:, None] * inv_freq.double()[None, :]
    e64 = torch.cat([a64, a64], -1)
    with pytest.raises(AssertionError, match="out of their allowance"):
        R.check_ulps(e64.cos().to(bf16), cos, ac, "cos of fp64 angles")
    with pytest.raises(AssertionError, match="out of their allowance"):
        R.check_ulps(hf_sin[1:], sin[:-1], asn[:-1], "sin at the next position")


# ------------------------------------------------------------------------------------------------ gathers
def test_add_pos_ref_is_the_rounded_bf16_sum():
    """bf16(x + t) through fp32 equals the fp64 sum rounded once, also where the two are 2^30 apart or cancel."""
    g = torch.Generator().manual_seed(12)
    x = torch.randn(64, 1032, generator=g)
    x[::3] *= 2.0 ** 30
    x = x.to(bf16)
    table = (torch.randn(50, 1032, generator=g) * 0.02).to(bf16)
    pos = torch.randint(0, 50, (64,), generator=g)
    table[pos[5]] = -x[5]                           # exact cancellation
    ref = R.add_pos_ref(x, pos, table)
    R.check_bits((x.float() + table[pos].float()).to(bf16), ref, "fp32 sum")
    R.check_bits(x + table[pos], ref, "torch bf16 add")
    with pytest.raises(AssertionError, match="differ"):
        p2 = pos.clone()
        p2[7] = (p2[7] + 1) % 50
        R.check_bits(x + table[p2], ref, "row 7 at the next position")


def _pixels(B, S, seed):
    return torch.randn(B, 3, S, S, generator=torch.Generator().manual_seed(seed)).to(bf16)


@pytest.mark.parametrize("B,S,k_pad", [(1, 56, 592), (3, 56, 640), (2, 490, 592)])
def test_im2col_ref_matches_unfold_and_rejects_a_shifted_row_and_a_nonzero_pad(B, S, k_pad):
    P = 14
    pix = _pixels(B, S, 13)
    ref = R.im2col_ref(pix, P, k_pad)
    unf = F.unfold(pix.float(), kernel_size=P, stride=P).transpose(1, 2).reshape(-1, 3 * P * P)
    R.check_bits(F.pad(unf, (0, k_pad - 3 * P * P)).to(bf16), ref, "unfold")
    shifted = pix.clone()
    shifted[B - 1, 1, S // 2 + 3] = torch.roll(pix[B - 1, 1, S // 2 + 3], 1)   # one image row read one pixel off
    with pytest.raises(AssertionError, match="differ"):
        R.check_bits(R.im2col_ref(shifted, P, k_pad), ref, "image row shifted by one")
    for v in (1.0, -0.0):
        bad = ref.clone()
        bad[-1, 3 * P * P] = v
        with pytest.raises(AssertionError, match="differ"):
            R.check_bits(bad, ref, f"pad column {v}")


def _merge_scan(ids, tok, feats, embeds, first_slot=0):
    """merge_kernel's loop: a running slot over the image tokens, in order."""
    out, slot = embeds.clone(), first_slot
    for t in range(ids.numel()):
        if int(ids[t]) == tok:
            out[t] = feats[slot]
            slot += 1
    return out, slot - first_slot


def test_merge_ref_is_masked_scatter_and_rejects_the_next_slot():
    g = torch.Generator().manual_seed(14)
    n, d, tok = 300, 64, 9
    ids = torch.randint(10, 500, (n,), generator=g)
    ids[[0, 31, 32, 299]] = tok
    ids[100:140] = tok
    feats = torch.randn(60, d, generator=g).to(bf16)
    emb = torch.randn(n, d, generator=g).to(bf16)
    ref, cnt = R.merge_ref(ids, tok, feats, emb)
    got, c = _merge_scan(ids, tok, feats, emb)
    R.check_bits(got, ref, "scan")
    assert c == cnt == 44
    with pytest.raises(AssertionError, match="differ"):
        R.check_bits(_merge_scan(ids, tok, feats, emb, first_slot=1)[0], ref, "running slot starting at 1")


# ------------------------------------------------------------------------------------------------ the GPU suite is complete
ENTRIES = ["rmsnorm", "rmsnorm_quantize_fp8", "layernorm", "rope_table", "embedding", "merge_image_features",
           "im2col_patches", "add_pos_embedding"]


def _rowwise_section():
    src = open(os.path.join(ROOT, "aria_b200", "ops.py")).read()
    return src[src.index("# ---", src.index("def offsets_from_counts")):src.index("def _attn_qkv_check")]


def test_rowwise_entries_are_all_listed():
    tree = ast.parse(_rowwise_section())
    public = [f.name for f in tree.body if isinstance(f, ast.FunctionDef) and not f.name.startswith("_")]
    assert public == ENTRIES


def test_every_rowwise_entry_has_an_fp64_test():
    src = open(os.path.join(HERE, "test_gpu_rowwise_fp64.py")).read()
    missing = [n for n in ENTRIES if not re.search(rf"\bops\.{n}\(", src)]
    assert not missing, f"row-wise entries of ops without a test in test_gpu_rowwise_fp64.py: {missing}"


def test_every_elementwise_kernel_is_in_the_fp64_test_docstring():
    kernels = re.findall(r"__global__ void (?:__launch_bounds__\(\d+\) )?(\w+)\(",
                         open(os.path.join(ROOT, "aria_b200", "csrc", "elementwise.cu")).read())
    assert len(kernels) == 10
    doc = ast.get_docstring(ast.parse(open(os.path.join(HERE, "test_gpu_rowwise_fp64.py")).read()))
    missing = [k for k in kernels if f"`{k}`" not in doc]
    assert not missing, f"not in test_gpu_rowwise_fp64.py's docstring: {missing}"


def _entry(src, name):
    i = src.index(f'extern "C" int {name}(')
    return src[i:src.index('extern "C"', i + 1)]


def test_dispatch_rules_match_elementwise_cu():
    """The thresholds of elementwise.cu's entry points: the MAXV ladder of the block kernels, the warp LayerNorm's
    (vpr, rows) condition, merge's single-block cut-over and the 16-blocks-per-SM grid cap; and the rules
    test_gpu_rowwise_fp64.py restates from them agree on every width, and on both sides of each row threshold."""
    import test_gpu_rowwise_fp64 as G
    src = open(os.path.join(ROOT, "aria_b200", "csrc", "elementwise.cu")).read()
    for entry, macro in (("aria_rmsnorm", "RMS"), ("aria_rmsnorm_quantize_fp8", "RMSQ"), ("aria_layernorm", "LN")):
        body = _entry(src, entry)
        ladder = re.findall(rf"if \(vpr <= (\d+)\) {macro}\((\d)\);", body)
        assert ladder == [("128", "1"), ("256", "2"), ("384", "3")] and f"else {macro}(4);" in body, entry
        assert "static_cast<int64_t>(sm_count()) * 16" in body, entry
    assert [G._maxv(8 * v) for v in (1, 128, 129, 256, 257, 384, 385, 512)] == [1, 1, 2, 2, 3, 3, 4, 4]
    assert G.rms_kernel(3080) == "rmsnorm_kernel<4>" and G.rms_kernel(2056, quant=True) == "rmsnorm_quantize_kernel<3>"
    ln = _entry(src, "aria_layernorm")
    vpr_max, rows_min = map(int, re.search(r"if \(vpr <= (\d+) && rows >= (\d+)\) \{[^}]*layernorm_warp_kernel<5>", ln).groups())
    for rows in (rows_min - 1, rows_min, 4900):
        for d in (8, 8 * vpr_max, 8 * vpr_max + 8, 4096):
            warp = d // 8 <= vpr_max and rows >= rows_min
            assert G.ln_kernel(rows, d) == ("layernorm_warp_kernel<5>" if warp else f"layernorm_kernel<{G._maxv(d)}>")
    merge = _entry(src, "aria_merge_image_features")
    cut = int(re.search(r"if \(n <= (\d+)\) \{\s*merge_rows_kernel<<<", merge).group(1))
    assert [G.merge_kernel(n) for n in (1, cut, cut + 1)] == ["merge_rows_kernel", "merge_rows_kernel", "merge_kernel"]
    assert "const int64_t cap = static_cast<int64_t>(sm_count()) * 16;" in src[src.index("static inline int rows_grid"):]
