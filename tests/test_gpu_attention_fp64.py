"""GPU: the wgmma prefill attention entries of aria_b200.ops and their backward against fp64, element by element (reference
and allowance: tests/attention_ref.py, which derives the kernels' worst-case fp32 error from their arithmetic).

Entry -> kernel -> test -> bar:
  `attention`                         attn_fwd_kernel<HD, CAUSAL, LSE>   test_dense_fwd_vs_fp64, test_dense_masks_vs_fp64,
                                      test_production_shapes_vs_fp64    allowance on out and lse; probes bit-exact
  `attention_varlen`                  attn_prefill_shared_prefix_kernel<LSE> (P = 0)   test_varlen_vs_fp64   (same bars)
  `attention_varlen_bwd`              attn_bwd_varlen_tiles, attn_bwd_pre, attn_bwd_kernel<true, true>, attn_bwd_post
                                      test_varlen_vs_fp64               allowance on dq, dk, dv; probes bit-exact
  `attention_prefill_shared_prefix`   attn_prefill_shared_prefix_kernel<false>   test_shared_prefix_vs_fp64   (fwd bars)
  `attention_prefill_paged_prefix`    attn_prefill_paged_prefix_kernel   test_paged_prefix_vs_fp64          (fwd bars)
  `attention_prefill_paged_varlen`    attn_prefill_paged_varlen_kernel   test_paged_varlen_vs_fp64          (fwd bars)
  `attention_bwd`                     attn_bwd_pre, attn_bwd_kernel<CAUSAL, false>, attn_bwd_post
                                      test_dense_bwd_vs_fp64            (bwd bars)

Bars: "allowance" is rowwise_ref.check_ulps(got, ref, allow): every element equal to the fp64 value rounded to bf16, or
within the ulps its fp32 error can reach (0 away from a rounding boundary); lse (fp32) within its absolute bound, and -inf
exactly on a row without keys.  "Probes bit-exact": q = 0 and small-integer values (attention_ref.probe_values): the forward
must store bf16(fl32(fl32(sum v) fl32(1 / n))) for every row, which shows the size and membership of its key set; the
backward with lse = 0, scale = 1/8, q = 0 or k = 0 and values in {-1, 0, 1} must store the bf16-rounded exact dV, dQ, dK.
The backward runs on the fp64 forward's rounded out and lse (the function of its own inputs) and once on the kernel's own
forward outputs (the training path).

Families (attention_ref.FAMILIES), on every forward entry: random N(0, 1) and q x 4 (peaked); the exact probe; needles (one key
about 12 nats above the rest, values 3 + d mod 5) at keys 0, 1, 63, 64, 127, 128, 129, 255, 256, Tk - 1 and a query's own
diagonal key, on the prefix / suffix boundary and either side of a page boundary; late-max rows rising 7.9 and 8.1 log2 units
per key tile, either side of the lazy raise; a wide row spanning 200 log2 units, so ex2 flushes; and a row whose weight lies
in its last key tile.

Poison.  What must not be read holds NaN: rows past Tq and Tk of over-allocated q / k / v (the tensor maps end at the
logical length, so TMA fills those rows with zeros), rows past P of the shared prefix buffer, pool pages no list names, page
table entries past a segment's prefix (a NaN page), and columns 80-127 of q, k and v at HD = 80.  Keys the forward loads but
weighs by P = 0 (masked keys) hold +-1e4 instead: the prefill kernels multiply V by P = 0 there, so those keys must hold
finite values.  Unlike decode, a prefill key mask is not a licence to leave NaN in the cache.

Measured on an H100 80GB HBM3: see DESIGN.md section 4 (prefill attention).
"""
import math

import pytest
import torch

import attention_ref as A
import rowwise_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
bf16 = torch.bfloat16
SCALE = 128 ** -0.5
NEEDLES = (0, 1, 63, 64, 127, 128, 129, 255, 256)
FAMILIES = A.FAMILIES


def _ops():
    from aria_b200 import ops
    return ops


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _stage(x, extra=40, front=0, hd=128):
    """x [B, H, T, 128] into a NaN bf16 buffer [B, H, front + T + extra, 128] at rows [front, front + T); returns the view
    from row `front` (T + extra rows, the rows past T NaN).  hd = 80: columns 80-127 NaN too."""
    B, H, T, _ = x.shape
    buf = torch.full((B, H, front + T + extra, 128), math.nan, dtype=bf16, device=DEV)
    buf[:, :, front:front + T, :hd] = x[..., :hd].to(bf16)
    return buf[:, :, front:]


def _poison_keys(buf, dead):
    """+-1e4 in the rows of keys dead for every query (dead [B, T]): loaded, weighed by P = 0."""
    B, H, _, D = buf.shape
    T = dead.shape[1]
    sign = torch.where(torch.arange(D, device=DEV) % 2 == 0, A.POISON, -A.POISON).to(bf16)
    view = buf[:, :, :T]
    view[dead[:, None, :, None].expand(B, H, T, D)] = sign.repeat(int(dead.sum()) * H)


def _report(what, got, ref, allow):
    exact, worst, band = R.check_ulps(got, ref, allow, what)
    print(f"{what}: exact {exact:.5%}, worst {worst:.3g} ulps, allowance band {band:.3%}")


def check_fwd(what, family, out, lse, q, k, v, live, hd=128, out_hd=128, n_kv=None):
    """out [B, Tq, H out_hd] (or [Tq, H out_hd]) against fwd_ref on the logical q / k / v [B, H, T, 128] and live."""
    B, H, Tq, _ = q.shape
    o = out.reshape(B, Tq, H, out_hd).transpose(1, 2)
    if family == "probe":
        R.check_bits(o, A.fwd_probe_ref(v[..., :out_hd], live), what)
        print(f"{what}: probe bit-exact")
        return
    ref, allow, lse64, lse_allow = A.fwd_ref(q, k, v, live, SCALE, hd, n_kv)
    _report(what, o, ref[..., :out_hd], allow[..., :out_hd])
    if lse is not None:
        worst = A.check_lse(lse.reshape(B, H, Tq), lse64, lse_allow, what + " lse")
        print(f"{what} lse: worst {worst:.3g} bf16 ulps")


def _needles(Tk, extra=()):
    return tuple(sorted({n for n in NEEDLES + (Tk - 1,) + tuple(extra) if 0 <= n < Tk}))


# ------------------------------------------------------------------------------------------------ dense forward
HD_CASES = {"hd128": (128, 128), "hd80_72": (80, 72), "hd80_80": (80, 80)}


def _dense(what, family, B, H, Tq, Tk, causal, hd, out_hd, seed, key_mask=None, lse_twice=False):
    ops = _ops()
    g = _gen(seed)
    pos_off = Tk - Tq
    q, k, v = A.family_qkv(B, H, Tq, Tk, family, g, DEV, needles=_needles(Tk, (pos_off + Tq // 2,)))
    live = A.live_dense(B, Tq, Tk, causal, key_mask, DEV)
    qs = _stage(q, front=3, hd=hd)
    ks, vs = _stage(k, hd=hd), _stage(v, hd=hd)
    if key_mask is not None:
        _poison_keys(ks, key_mask.bool())
        _poison_keys(vs, key_mask.bool())
    out, lse = ops.attention(qs, ks, vs, Tq, Tk, SCALE, causal, out_hd=out_hd, key_mask=key_mask, return_lse=True)
    if lse_twice:
        R.check_bits(ops.attention(qs, ks, vs, Tq, Tk, SCALE, causal, out_hd=out_hd, key_mask=key_mask), out,
                     what + " without lse")
    check_fwd(what, family, out, lse, q, k, v, live, hd, out_hd)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("hd_case", list(HD_CASES))
def test_dense_fwd_vs_fp64(hd_case, causal, family):
    """B 3, H 5, q a strided slice of a NaN staging buffer.  Tq at every query-tile edge (164: the last tile's second
    warpgroup has no live rows); causal suffixes pos_off in {1, 50, 64, 127, 128}; 1 .. STAGES + 2 key tiles with and
    without a key tail, so the K/V ring's prologue and epilogue run at 2 and 4 stages."""
    hd, out_hd = HD_CASES[hd_case]
    seed = 100 * list(HD_CASES).index(hd_case) + 10 * causal + FAMILIES.index(family)
    for i, Tq in enumerate([1, 63, 64, 65, 127, 128, 129, 164, 257]):
        Tk = Tq if causal else Tq + 37
        _dense(f"{hd_case} {'causal' if causal else 'full'} {family} Tq {Tq} Tk {Tk}", family, 3, 5, Tq, Tk, causal, hd,
               out_hd, seed + 1000 * i, lse_twice=i == 0)
    if causal:
        for i, off in enumerate([1, 50, 64, 127, 128]):
            _dense(f"{hd_case} causal {family} suffix pos_off {off}", family, 1, 2, 100, 100 + off, True, hd, out_hd,
                   seed + 20000 + i)
    for n in range(1, A.STAGES[hd] + 3):
        for tail in (0, 37):
            Tk = n * A.AT_BN - tail
            if Tk <= 0:
                continue
            _dense(f"{hd_case} {family} n_kv {n} Tk {Tk}", family, 1, 2, min(129, Tk), Tk, causal, hd, out_hd,
                   seed + 30000 + 10 * n + tail)


def _masks(B, Tk, seed):
    """[B, Tk] uint8 (1 = masked): 30 % random with the first and last keys masked; one whole 128-key tile masked (the
    running max stays -inf through it); left padding as HF gives it; every key masked (out 0, lse -inf)."""
    g = _gen(seed)
    m = (torch.rand(B, Tk, generator=g, device=DEV) < 0.3).to(torch.uint8)
    m[0, 0] = m[0, -1] = 1
    m[1] = 0
    m[1, :A.AT_BN] = 1
    m[2] = 0
    m[2, :77] = 1
    m[3] = 1
    return m


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("hd_case", list(HD_CASES))
def test_dense_masks_vs_fp64(hd_case, causal, family):
    hd, out_hd = HD_CASES[hd_case]
    Tq, Tk = (300, 300) if causal else (200, 300)
    km = _masks(4, Tk, 7 + causal)
    _dense(f"{hd_case} {'causal' if causal else 'full'} {family} masked", family, 4, 2, Tq, Tk, causal, hd, out_hd,
           500 + FAMILIES.index(family), key_mask=km)


PRODUCTION = {
    "lm_2048": (1, 20, 2048, 2048, True, 128, 128),
    "lm_8192": (1, 2, 8192, 8192, True, 128, 128),
    "vit_4900": (1, 16, 4900, 4900, False, 80, 72),
    "projector_256x4900": (1, 16, 256, 4900, False, 80, 72),
}


@pytest.mark.parametrize("family", ["random", "probe", "needle"])
@pytest.mark.parametrize("case", list(PRODUCTION))
def test_production_shapes_vs_fp64(case, family):
    """The LM's 20 heads at 2048 causal and 8192 on two heads; the ViT's 16 heads of 72 at 4900 keys; the projector's 256
    queries against 4900 keys with the 52 x 52 valid crop of the 70 x 70 patch grid as its key mask."""
    B, H, Tq, Tk, causal, hd, out_hd = PRODUCTION[case]
    km = None
    if case.startswith("projector"):
        rc = torch.arange(Tk, device=DEV)
        km = ~((rc // 70 < 52) & (rc % 70 < 52))[None]
        km = km.to(torch.uint8)
    _dense(f"{case} {family}", family, B, H, Tq, Tk, causal, hd, out_hd, 900 + len(case), key_mask=km)


# ------------------------------------------------------------------------------------------------ varlen forward + backward
SEG_LENS = [1, 63, 64, 65, 127, 128, 129, 300]
SEG_ORDERS = {"ascending": SEG_LENS, "descending": SEG_LENS[::-1], "mixed": [129, 1, 300, 64, 127, 65, 63, 128]}


def _cu(lens):
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    return cu


def _bwd_probe_inputs(B, H, Tq, Tk, which, seed):
    """q, k, v, dout, out with values in {-1, 0, 1}; q = 0 (which = q0: dQ fingerprints the keys, by their index bits in
    columns 0..12 of k) or k = 0 (k0: dK fingerprints the queries); dout's columns 0..12 fingerprint the queries for dV."""
    g = _gen(seed)

    def tern(*shape):
        return torch.randint(-1, 2, shape, generator=g, device=DEV).float()
    q, k, v, dout, out = tern(B, H, Tq, 128), tern(B, H, Tk, 128), tern(B, H, Tk, 128), tern(B, H, Tq, 128), \
        tern(B, H, Tq, 128)
    i = torch.arange(max(Tq, Tk), device=DEV)
    bits = torch.stack([torch.where((i >> b) & 1 == 1, -1.0, 1.0) for b in range(13)], 1)
    if which == "q0":
        q.zero_()
        k[..., :13] = bits[:Tk]
    else:
        k.zero_()
        q[..., :13] = bits[:Tq]
    dout[..., :13] = bits[:Tq]
    return q, k, v, dout, out


def check_bwd(what, got, q, k, v, out, dout, lse, live, scale, probe):
    """got (dq, dk, dv) [B, H, T, 128] against bwd_ref / bwd_exact (out, dout head-major)."""
    if probe:
        for name, gt, r in zip(("dq", "dk", "dv"), got, A.bwd_exact(q, k, v, out, dout, lse, live, scale)):
            R.check_bits(gt, R.bf16_rn(r).to(bf16), f"{what} {name}")
        print(f"{what}: probe bit-exact")
        return
    for name, gt, (r, al) in zip(("dq", "dk", "dv"), got, A.bwd_ref(q, k, v, out, dout, lse, live, scale)):
        _report(f"{what} {name}", gt, r, al)


def _head_major(x, B, T, H):
    return x.reshape(B, T, H, 128).transpose(1, 2)


def _token_major(x):
    B, H, T, _ = x.shape
    return x.transpose(1, 2).reshape(B, T, H * 128).to(bf16).contiguous()


@pytest.mark.parametrize("family", FAMILIES + ["bwd_probe"])
@pytest.mark.parametrize("order", list(SEG_ORDERS))
def test_varlen_vs_fp64(order, family):
    """Segments of every tile-edge length, packed so that segment starts fall inside query and key tiles; the forward with
    lse, then the backward on the fp64 out / lse and on the kernel's own."""
    ops = _ops()
    lens = SEG_ORDERS[order]
    cu = _cu(lens)
    N, H = cu[-1], 2
    cu_dev = torch.tensor(cu, dtype=torch.int32, device=DEV)
    live = A.live_varlen(cu, N, DEV)
    seed = 3000 + 10 * list(SEG_ORDERS).index(order) + (FAMILIES + ["bwd_probe"]).index(family)
    what = f"varlen {order} {family}"
    if family == "bwd_probe":
        for which in ("q0", "k0"):
            q, k, v, dout, out = _bwd_probe_inputs(1, H, N, N, which, seed)
            lse = torch.zeros(H, N, device=DEV)
            got = ops.attention_varlen_bwd(_stage(q), _stage(k), _stage(v), _token_major(out)[0], _token_major(dout)[0],
                                           lse, cu_dev, 0.125, N=N)
            check_bwd(f"{what} {which}", got, q, k, v, out, dout, lse[None], live, 0.125, True)
        return
    g = _gen(seed)
    starts = [c for c in cu[1:-1]]
    q, k, v = A.family_qkv(1, H, N, N, family, g, DEV, needles=_needles(N, starts + [s - 1 for s in starts]))
    out, lse = ops.attention_varlen(_stage(q), _stage(k), _stage(v), cu_dev, SCALE, return_lse=True, N=N)
    check_fwd(what, family, out, lse, q, k, v, live)
    if family not in ("random", "peaked", "needle"):
        return
    dout = torch.randn(1, H, N, 128, generator=g, device=DEV).to(bf16).float()
    ref, _, lse64, _ = A.fwd_ref(q, k, v, live, SCALE)
    for src, o_in, l_in in (("fp64 out", ref.float(), lse64.float()[0]), ("kernel out", _head_major(out, 1, N, H).float(),
                                                                          lse)):
        got = ops.attention_varlen_bwd(_stage(q), _stage(k), _stage(v), _token_major(o_in)[0], _token_major(dout)[0],
                                       l_in.contiguous(), cu_dev, SCALE, N=N)
        check_bwd(f"{what} bwd on {src}", got, q, k, v, o_in.to(bf16).float(), dout, l_in[None], live, SCALE, False)


# ------------------------------------------------------------------------------------------------ shared prefix
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("P", [1, 127, 128, 129, 256, 300])
def test_shared_prefix_vs_fp64(P, family):
    """Each suffix order of SEG_ORDERS after a P-key prefix; the prefix buffer holds NaN past P."""
    ops = _ops()
    H = 2
    for j, (order, lens) in enumerate(SEG_ORDERS.items()):
        cu = _cu(lens)
        S = cu[-1]
        seed = 4000 + 100 * P + 10 * j + FAMILIES.index(family)
        g = _gen(seed)
        q, kx, vx = A.family_qkv(1, H, S, P + S, family, g, DEV,
                                 needles=_needles(P + S, (P - 1, P, P + cu[1], P + cu[2] - 1)))
        out = ops.attention_prefill_shared_prefix(_stage(q), _stage(kx[:, :, P:]), _stage(vx[:, :, P:]), S,
                                                  _stage(kx[:, :, :P]), _stage(vx[:, :, :P]), P,
                                                  torch.tensor(cu, dtype=torch.int32, device=DEV), SCALE)
        live = A.live_prefix(cu, S, P, device=DEV)
        check_fwd(f"shared prefix P {P} {order} {family}", family, out, None, q, kx, vx, live,
                  n_kv=A.cdiv(P, 128) + A.cdiv(S, 128) + len(lens))


# ------------------------------------------------------------------------------------------------ paged prefix / varlen
def _pool(H, keys_k, keys_v, n_pages, seed):
    """Pools [n_pages, H, 256, 128] of NaN; the listed pages get consecutive 256-key chunks of keys_k / keys_v [1, H, n, 128]
    in a permuted order.  Returns (k_pool, v_pool, page list)."""
    n = A.cdiv(keys_k.shape[2], A.PAGE_ROWS)
    perm = torch.randperm(n_pages, generator=torch.Generator().manual_seed(seed)).tolist()[:n]
    kp = torch.full((n_pages, H, A.PAGE_ROWS, 128), math.nan, dtype=bf16, device=DEV)
    vp = torch.full_like(kp, math.nan)
    for i, pg in enumerate(perm):
        kp[pg] = keys_k[0, :, i * 256:(i + 1) * 256].to(bf16)
        vp[pg] = keys_v[0, :, i * 256:(i + 1) * 256].to(bf16)
    return kp, vp, perm


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("P", [0, 256, 512, 768, "outside"])
def test_paged_prefix_vs_fp64(P, family):
    """Prefixes of 0 .. 3 pages in permuted pool pages among NaN pages; "outside": 512 keys whose second page entry is
    past the pool, which reads zeros."""
    ops = _ops()
    H = 2
    lens = SEG_ORDERS["mixed"]
    cu = _cu(lens)
    S = cu[-1]
    Pk = 512 if P == "outside" else P
    seed = 5000 + Pk + (P == "outside") + 10 * FAMILIES.index(family)
    g = _gen(seed)
    q, kx, vx = A.family_qkv(1, H, S, Pk + S, family, g, DEV, needles=_needles(Pk + S, (255, 256, Pk - 1, Pk)))
    kp, vp, pages = _pool(H, kx[:, :, :Pk], vx[:, :, :Pk], 7, seed)
    if P == "outside":
        pages[1] = 7 + 3
        kx[:, :, 256:512] = 0
        vx[:, :, 256:512] = 0
    pages_dev = torch.tensor(pages + [0], dtype=torch.int32, device=DEV)
    out = ops.attention_prefill_paged_prefix(_stage(q), _stage(kx[:, :, Pk:]), _stage(vx[:, :, Pk:]), S, kp, vp,
                                             pages_dev if Pk else None, Pk, torch.tensor(cu, dtype=torch.int32, device=DEV),
                                             SCALE)
    live = A.live_prefix(cu, S, Pk, device=DEV)
    check_fwd(f"paged prefix P {P} {family}", family, out, None, q, kx, vx, live,
              n_kv=A.cdiv(Pk, 128) + A.cdiv(S, 128) + len(lens))


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("layout", ["mixed", "many_short"])
def test_paged_varlen_vs_fp64(layout, family):
    """Segments with prefixes of 0 .. 3 pages of their own, a page table two pages wider than any prefix whose unused
    entries name a NaN page, and segment counts whose tile count is below the grid's upper bound."""
    ops = _ops()
    H = 2
    if layout == "mixed":
        lens, plens = [129, 1, 300, 64, 127, 65], [512, 0, 256, 768, 0, 256]
    else:
        lens, plens = [200, 3, 130, 5, 1, 250], [256, 256, 0, 512, 0, 256]
    cu = _cu(lens)
    S = cu[-1]
    Ptot = sum(plens)
    seed = 6000 + 10 * (layout == "mixed") + FAMILIES.index(family)
    g = _gen(seed)
    edges = [sum(plens[:b]) + x for b in range(len(plens)) for x in (0, 255, 256) if x < plens[b]]
    q, kx, vx = A.family_qkv(1, H, S, Ptot + S, family, g, DEV, needles=_needles(Ptot + S, edges + [Ptot]))
    n_pages = Ptot // 256 + 3
    kp, vp, perm = _pool(H, kx[:, :, :Ptot], vx[:, :, :Ptot], n_pages, seed)
    nan_page = next(p for p in range(n_pages) if p not in perm)
    W = max(plens) // 256 + 2
    table = torch.full((len(lens), W), nan_page, dtype=torch.int32)
    i = 0
    for b, p in enumerate(plens):
        for j in range(p // 256):
            table[b, j] = perm[i]
            i += 1
    seg = ops.PackedSegments(cu, plens, DEV)
    out = ops.attention_prefill_paged_varlen(_stage(q), _stage(kx[:, :, Ptot:]), _stage(vx[:, :, Ptot:]), kp, vp,
                                             table.to(DEV), seg, SCALE)
    live = A.live_paged_varlen(cu, plens, S, DEV)
    check_fwd(f"paged varlen {layout} {family}", family, out, None, q, kx, vx, live,
              n_kv=A.cdiv(max(plens), 128) + A.cdiv(max(lens), 128) + 1)


# ------------------------------------------------------------------------------------------------ dense backward
BWD_SHAPES = [
    (1, 2, 128, 128, True, 0.0), (2, 3, 300, 300, True, 0.0), (1, 2, 100, 420, True, 0.0), (2, 2, 333, 333, False, 0.3),
    (1, 4, 1030, 1030, True, 0.0), (2, 20, 2048, 2048, True, 0.0), (1, 2, 8192, 8192, True, 0.0),
] + [(1, 2, t, t, True, 0.0) for t in (63, 64, 65, 127, 129)] + [(2, 2, 63, 129, False, 0.3), (1, 2, 65, 193, True, 0.0)]


@pytest.mark.parametrize("family", ["random", "peaked", "probe"])
@pytest.mark.parametrize("B,H,Tq,Tk,causal,mask_p", BWD_SHAPES)
def test_dense_bwd_vs_fp64(B, H, Tq, Tk, causal, mask_p, family):
    ops = _ops()
    seed = 7000 + Tq + 3 * Tk + 100 * ["random", "peaked", "probe"].index(family)
    g = _gen(seed)
    km = None
    if mask_p:
        km = (torch.rand(B, Tk, generator=g, device=DEV) < mask_p).to(torch.uint8)
        km[:, -1] = 0
        km[:, 0] = 1
    live = A.live_dense(B, Tq, Tk, causal, km, DEV)
    what = f"bwd B {B} H {H} Tq {Tq} Tk {Tk} {'causal' if causal else 'full'} {family}"
    if family == "probe":
        if Tk > 2048:
            pytest.skip("probe sums stay below 2^20 up to 2048 keys")
        for which in ("q0", "k0"):
            q, k, v, dout, out = _bwd_probe_inputs(B, H, Tq, Tk, which, seed)
            ks, vs = _stage(k, extra=0), _stage(v, extra=0)
            if km is not None:
                _poison_keys(vs, km.bool())
            lse = torch.zeros(B, H, Tq, device=DEV)
            got = ops.attention_bwd(_stage(q, extra=0), ks, vs, _token_major(out), _token_major(dout), lse, Tq, Tk, 0.125,
                                    causal, key_mask=km)
            check_bwd(f"{what} {which}", got, q, k, v, out, dout, lse, live, 0.125, True)
        return
    q, k, v = A.family_qkv(B, H, Tq, Tk, family, g, DEV)
    dout = torch.randn(B, H, Tq, 128, generator=g, device=DEV).to(bf16).float()
    qs, ks, vs = _stage(q, extra=0), _stage(k, extra=0), _stage(v, extra=0)
    if km is not None:
        _poison_keys(ks, km.bool())
        _poison_keys(vs, km.bool())
    ref, _, lse64, _ = A.fwd_ref(q, k, v, live, SCALE)
    out_k, lse_k = ops.attention(qs, ks, vs, Tq, Tk, SCALE, causal, key_mask=km, return_lse=True)
    for src, o_in, l_in in (("fp64 out", ref.float(), lse64.float()), ("kernel out", _head_major(out_k, B, Tq, H).float(),
                                                                       lse_k)):
        got = ops.attention_bwd(qs, ks, vs, _token_major(o_in), _token_major(dout), l_in.contiguous(), Tq, Tk, SCALE,
                                causal, key_mask=km)
        check_bwd(f"{what} on {src}", got, q, k, v, o_in.to(bf16).float(), dout, l_in, live, SCALE, False)
