"""CPU: tests/attention_ref.py accepts an fp32 evaluation of the prefill attention kernels and their backward, and rejects
planted mistakes.

`emulate_fwd` restates attn_fwd_body of aria_b200/csrc/attention.cu in fp32, in its order: per 128-key tile the mask, the
tile max, the lazy raise of the row max (only when it grows by more than LAZY log2 units; `eager` raises on any growth),
then fp32 P = ex2(s c - m) (flushed below 2^-126) into l and bf16(P) V into O, O and l rescaled on a raise, and finally
o inv_l with inv_l = 1 / l, and lse = (m + log2 l) ln 2.  `emulate_bwd` restates attn_bwd_pre / attn_bwd_kernel /
attn_bwd_post of attention_bwd.cu: per 128-key tile (varlen: aligned at each segment's start) the 64-row query steps from
m_begin, P from lse2 = lse log2 e, bf16(P) into dV, dS = P (dP - D), bf16(dS) into dK and into one dQ partial per key tile.
Both run on the expanded key axis of the layout's live set, so the same emulation serves every prefill entry.  They round
exp2 and the matrix products on the CPU, inside the reference's bound.  Each planted mistake is a flag of the emulation
or a wrong live set or key order fed to it; the test names the input family that catches it.
"""
import math

import pytest
import torch

import attention_ref as A
import rowwise_ref as R

F32 = torch.float32
F64 = torch.float64
bf16 = torch.bfloat16
SCALE = 128 ** -0.5
H = 2


def _bf(x):
    return x.to(bf16).float()


# ------------------------------------------------------------------------------------------------ fp32 emulations
def emulate_fwd(q, k, v, live, scale, hd=128, out_hd=128, eager=False, no_rescale=False, drop_last=False, lse_mode="ln",
                nan_dead=False, head_stride=None):
    """q [B, H, Tq, 128], k / v [B, H, Tk, 128], live [B or 1, Tq, Tk] -> (out [B, Tq, H out_hd] bf16, lse [B, H, Tq])."""
    B, Hh, Tq, _ = q.shape
    Tk = k.shape[2]
    live = live.bool().expand(B, Tq, Tk)
    c = torch.tensor(scale, dtype=F32) * torch.tensor(1.4426950408889634, dtype=F32)
    m = torch.full((B, Hh, Tq), -math.inf)
    l = torch.zeros(B, Hh, Tq)
    O = torch.zeros(B, Hh, Tq, v.shape[-1])
    n_t = A.cdiv(Tk, A.AT_BN)
    for j in range(n_t - 1 if drop_last else n_t):
        j0, j1 = j * A.AT_BN, min(Tk, (j + 1) * A.AT_BN)
        s = q[..., :hd].float() @ k[:, :, j0:j1, :hd].float().transpose(2, 3)
        s = s.masked_fill(~live[:, None, :, j0:j1], -math.inf)
        mx = s.amax(-1)
        mc = torch.maximum(m, (mx * c).float())
        up = (mc > m) if eager else ((mc - m > A.LAZY) | ((m == -math.inf) & (mc > -math.inf)))
        f = torch.where(up, torch.where(m == -math.inf, 0.0, torch.exp2(m - mc)), 1.0)
        m = torch.where(up, mc, m)
        l = l * f
        if not no_rescale:
            O = O * f[..., None]
        neg = torch.where(m == -math.inf, 0.0, -m)
        x = (s.double() * float(c) + neg.double()[..., None]).float()
        P = torch.exp2(x)
        P = torch.where(P < 2.0 ** -126, 0.0, P)
        l = l + P.sum(-1)
        O = O + _bf(P) @ torch.nan_to_num(v[:, :, j0:j1].float())
    inv = torch.where(l > 0, 1.0 / l, 0.0)
    o = O * inv[..., None]
    if nan_dead:
        o = torch.where(l[..., None] > 0, o, math.nan)
    lse = (m + torch.log2(l)) * torch.tensor(0.6931471805599453, dtype=F32)
    if lse_mode == "log2":
        lse = m + torch.log2(l)
    elif lse_mode == "no_log":
        lse = m * torch.tensor(0.6931471805599453, dtype=F32)
    lse = torch.where(l > 0, lse, -math.inf)
    out = torch.zeros(B, Tq, Hh * out_hd)
    hs = out_hd if head_stride is None else head_stride
    for h in range(Hh):
        w = min(out_hd, Hh * out_hd - h * hs)
        if w > 0:
            out[:, :, h * hs:h * hs + w] = o[:, h, :, :w]
    return out.to(bf16), lse


def emulate_bwd(q, k, v, out, dout, lse, scale, tiles, key_live, causal, d_shift=False, no_dk_scale=False, late_m=False,
                keep_qdead=False, lost_tile=None):
    """q / out / dout [B, H, Tq, 128] (out / dout head-major), k / v [B, H, Tk, 128], lse [B, H, Tq]; tiles: per key tile
    (k0, seg_end, m_base, n_steps, m_begin) as the kernel walks it; key_live [B, Tk] (key mask); causal positions
    pos_off = Tk - Tq (varlen: 0).  -> (dq, dk, dv) bf16."""
    B, Hh, Tq, Dm = q.shape
    Tk = k.shape[2]
    pos_off = Tk - Tq
    c = torch.tensor(scale, dtype=F32) * torch.tensor(1.4426950408889634, dtype=F32)
    lse2 = torch.where(lse == -math.inf, math.inf, lse * torch.tensor(1.4426950408889634, dtype=F32))
    Dr = (dout.float() * out.float()).sum(-1)
    if d_shift:
        Dr = torch.cat([Dr[..., 1:], Dr[..., -1:]], -1)
    dk = torch.zeros(B, Hh, Tk, Dm)
    dv = torch.zeros(B, Hh, Tk, Dm)
    parts = []
    for ti, (k0, seg_end, m_base, n_steps, m_begin) in enumerate(tiles):
        k1 = min(k0 + A.AB_BN, Tk)
        keys = torch.arange(k0, k1)
        kdead = (keys >= seg_end)[None, :] | ~key_live[:, k0:k1]
        part = torch.zeros(B, Hh, Tq, Dm)
        for i in range(m_begin + (1 if late_m else 0), n_steps):
            m0 = m_base + i * A.AB_BM
            m1 = min(m0 + A.AB_BM, Tq)
            if m0 >= m1:
                continue
            rows = torch.arange(m0, m1)
            S = q[:, :, m0:m1].float() @ k[:, :, k0:k1].float().transpose(2, 3)
            x = (S.double() * float(c) - lse2[:, :, m0:m1, None].double()).float()
            P = torch.exp2(x)
            P = torch.where(P < 2.0 ** -126, 0.0, P)
            dead = kdead[:, None, None, :].expand(B, 1, m1 - m0, k1 - k0)
            if causal:
                dead = dead | (keys[None, :] > rows[:, None] + pos_off)[None, None]
            if not keep_qdead:
                dead = dead | (rows >= seg_end)[None, None, :, None]
            P = torch.where(dead, 0.0, P)
            dv[:, :, k0:k1] += _bf(P).transpose(2, 3) @ dout[:, :, m0:m1].float()
            dP = dout[:, :, m0:m1].float() @ v[:, :, k0:k1].float().transpose(2, 3)
            dS = P * (dP - Dr[:, :, m0:m1, None])
            dk[:, :, k0:k1] += _bf(dS).transpose(2, 3) @ q[:, :, m0:m1].float()
            part[:, :, m0:m1] += _bf(dS) @ k[:, :, k0:k1].float()
        if ti != lost_tile:
            parts.append(part)
    dq = torch.zeros(B, Hh, Tq, Dm)
    for p in parts:
        dq = dq + p
    sc = torch.tensor(scale, dtype=F32)
    return (dq * sc).to(bf16), (dk if no_dk_scale else dk * sc).to(bf16), dv.to(bf16)


def dense_tiles(Tq, Tk, causal):
    pos_off = Tk - Tq
    n_m = A.cdiv(Tq, A.AB_BM)
    return [(k0, Tk, 0, n_m, max(0, k0 - pos_off) // A.AB_BM if causal else 0) for k0 in range(0, Tk, A.AB_BN)]


def varlen_tiles(cu):
    return [(k0, e, k0, A.cdiv(e - k0, A.AB_BM), 0) for c, e in zip(cu, cu[1:]) for k0 in range(c, e, A.AB_BN)]


# ------------------------------------------------------------------------------------------------ layouts (small shapes)
def _gen(seed):
    return torch.Generator().manual_seed(seed)


CU = [0, 1, 64, 193, 258, 300]                  # segments of 1, 63, 129, 65, 42 rows
PREFIX_P = 129


def layout(name, family, seed, mistake=None):
    """(q, k, v, live, live_emulated, hd, out_hd, n_seg) for one layout at a small shape: the emulation runs on
    live_emulated (a planted layout mistake) and on k / v (possibly with swapped pages)."""
    g = _gen(seed)
    hd, out_hd, n_seg = 128, 128, 1
    if name in ("dense", "dense_causal", "dense_hd80"):
        B, Tq, Tk = 2, 164, 300
        causal = name == "dense_causal"
        km = (torch.rand(B, Tk, generator=g) < 0.3).to(torch.uint8)
        km[:, 0] = km[:, -1] = 1
        km[1, 128:256] = 1                        # a whole key tile masked on batch row 1
        if name == "dense_hd80":
            hd, out_hd = 80, 72
        q, k, v = A.family_qkv(B, H, Tq, Tk, family, g, "cpu", needles=(0, 1, 63, 64, 127, 128, 129, 255, 256, Tk - 1))
        live = A.live_dense(B, Tq, Tk, causal, km)
        lm = live
        if mistake in ("diag+1", "diag-1"):       # a query sees its next key, or not its own
            shift = 1 if mistake == "diag+1" else 0
            edge = torch.arange(Tk)[None, None] == (torch.arange(Tq) + Tk - Tq + shift)[None, :, None]
            lm = (live | (edge & ~km.bool()[:, None])) if shift else (live & ~edge)
        if hd == 80:                              # NaN in the columns past 80 that the HD = 80 path never loads
            q[..., 80:], k[..., 80:], v[..., 80:] = math.nan, math.nan, math.nan
        kk, vv = k.clone(), v.clone()
        return q, k, v, kk, vv, live, lm, hd, out_hd, n_seg
    N = CU[-1]
    n_seg = len(CU) - 1
    if name == "varlen":
        q, k, v = A.family_qkv(1, H, N, N, family, g, "cpu", needles=(0, 1, 63, 64, 127, 128, 129, 255, 256, N - 1))
        live = A.live_varlen(CU, N)
        lm = live
        if mistake == "seg_start":
            cu = torch.tensor(CU)
            lm = live.clone()
            for s in range(1, n_seg):
                lm[0, cu[s]:cu[s + 1], cu[s] - 1] = True
        return q, k, v, k.clone(), v.clone(), live, lm, hd, out_hd, n_seg
    if name == "shared_prefix":
        P_keys = 256                              # buffer rows past P hold keys the kernel must not read
        q, k, v = A.family_qkv(1, H, N, P_keys + N, family, g, "cpu", needles=(0, 127, 128, PREFIX_P - 1, PREFIX_P,
                                                                                 P_keys + 64, P_keys + N - 1))
        live = A.live_prefix(CU, N, PREFIX_P, P_keys)
        lm = A.live_prefix(CU, N, A.cdiv(PREFIX_P, 128) * 128, P_keys) if mistake == "prefix_past_P" else live
        return q, k, v, k.clone(), v.clone(), live, lm, hd, out_hd, n_seg
    # paged: pools of 5 pages; the prefix is 3 of them listed in permuted order, pages 1 and 2 hold other keys
    P = 3 * A.PAGE_ROWS
    X = P + 2 * A.PAGE_ROWS
    q, kt, vt = A.family_qkv(1, H, N, X + N, family, g, "cpu", needles=(0, 255, 256, 511, 512, P - 1, P, X - 1, X))
    pages = [3, 0, 4]
    kp = torch.zeros(5, H, A.PAGE_ROWS, 128)
    vp = torch.zeros(5, H, A.PAGE_ROWS, 128)
    for i, pg in enumerate(pages + [1, 2]):
        kp[pg] = kt[0, :, i * 256:(i + 1) * 256]
        vp[pg] = vt[0, :, i * 256:(i + 1) * 256]
    ks, vs = kt[:, :, X:], vt[:, :, X:]

    def expand(tables, plens):
        return (torch.cat([A.keys_pool(kp, t, n) for t, n in zip(tables, plens)] + [ks], 2),
                torch.cat([A.keys_pool(vp, t, n) for t, n in zip(tables, plens)] + [vs], 2))
    if name == "paged_varlen":
        plens = [P, 0, 256, 0, 512]
        table = [pages, [9, 9, 9], [4, 9, 9], [9, 9, 9], [1, 2, 9]]      # entries past each prefix are never read
        k, v = expand(table, plens)
        kk, vv = k, v
        if mistake == "swap_pages":               # segment 0's second page and segment 4's first trade places
            bad = [list(t) for t in table]
            bad[0][1], bad[4][0] = bad[4][0], bad[0][1]
            kk, vv = expand(bad, plens)
        live = A.live_paged_varlen(CU, plens, N)
        return q, k, v, kk, vv, live, live, hd, out_hd, n_seg
    k, v = expand([pages], [P])
    return q, k, v, k, v, A.live_prefix(CU, N, P), A.live_prefix(CU, N, P), hd, out_hd, n_seg


LAYOUTS = ["dense", "dense_causal", "dense_hd80", "varlen", "shared_prefix", "paged_prefix", "paged_varlen"]


def check_fwd(q, k, v, live, hd, out_hd, family, out, lse, what):
    """The reference check the GPU tests make: probes bit for bit, else the allowance on out and lse."""
    B, Hh, Tq, _ = q.shape
    o = out.view(B, Tq, Hh, out_hd).transpose(1, 2)
    if family == "probe":
        R.check_bits(o, A.fwd_probe_ref(v[..., :out_hd], live), what)
        return
    ref, allow, lse64, lse_allow = A.fwd_ref(q, k, v, live, SCALE, hd)
    R.check_ulps(o, ref[..., :out_hd], allow[..., :out_hd], what)
    A.check_lse(lse, lse64, lse_allow, what + " lse")


def _fwd_case(name, family, seed=0, mistake=None, **flags):
    q, k, v, kk, vv, live, lm, hd, out_hd, n_seg = layout(name, family, seed, mistake)
    out, lse = emulate_fwd(q, kk, vv, lm, SCALE, hd, out_hd, **flags)
    check_fwd(q, k, v, live, hd, out_hd, family, out, lse, f"{name} {family} {mistake or flags}")


# ------------------------------------------------------------------------------------------------ acceptance
@pytest.mark.parametrize("family", A.FAMILIES)
@pytest.mark.parametrize("name", LAYOUTS)
def test_reference_accepts_the_emulation(name, family):
    _fwd_case(name, family, seed=LAYOUTS.index(name) * 10 + A.FAMILIES.index(family))


@pytest.mark.parametrize("family", ["random", "late7.9", "late8.1", "wide", "needle"])
@pytest.mark.parametrize("name", ["dense_causal", "dense_hd80", "shared_prefix"])
def test_reference_accepts_an_eager_max(name, family):
    _fwd_case(name, family, seed=7, eager=True)


def test_lazy_max_families_straddle_the_threshold():
    """late7.9 never raises the lazy max after the first tile, late8.1 raises it every tile: the two families do exercise
    both sides of the rescale."""
    for fam, raises in (("late7.9", False), ("late8.1", True)):
        q, k, v = A.family_qkv(1, 1, 1, 4 * A.AT_BN, fam, _gen(1), "cpu")
        s = (q[0, 0, 0] @ k[0, 0].T) * SCALE * A.LOG2E
        tile_max = s.view(4, A.AT_BN).amax(1)
        assert bool(((tile_max[1:] - tile_max[:-1] > A.LAZY) == raises).all()), (fam, tile_max)


# ------------------------------------------------------------------------------------------------ planted mistakes
def _rejects(fn):
    with pytest.raises(AssertionError):
        fn()


# (mistake, layout, family that catches it, emulation flags)
FWD_MISTAKES = [
    ("last tile dropped", "dense", "probe", dict(drop_last=True)),
    ("last tile dropped", "dense", "lasttile", dict(drop_last=True)),
    ("diagonal one late", "dense_causal", "probe", dict(mistake="diag+1")),
    ("diagonal one early", "dense_causal", "probe", dict(mistake="diag-1")),
    ("diagonal one late", "dense_causal", "needle", dict(mistake="diag+1")),
    ("segment start one early", "varlen", "probe", dict(mistake="seg_start")),
    ("prefix keys >= P visible", "shared_prefix", "probe", dict(mistake="prefix_past_P")),
    ("prefix keys >= P visible", "shared_prefix", "needle", dict(mistake="prefix_past_P")),
    ("two prefix pages swapped", "paged_varlen", "probe", dict(mistake="swap_pages")),
    ("two prefix pages swapped", "paged_varlen", "random", dict(mistake="swap_pages")),
    ("O not rescaled on a raise", "dense", "late8.1", dict(no_rescale=True)),
    ("O not rescaled on a raise", "varlen", "lasttile", dict(no_rescale=True)),
    ("lse in log2 units", "dense", "random", dict(lse_mode="log2")),
    ("lse without log l", "dense_causal", "random", dict(lse_mode="no_log")),
    ("lse without log l", "dense", "late7.9", dict(lse_mode="no_log")),
    ("row with no key stores NaN", "dense", "random", dict(nan_dead=True)),
    ("head h at h 128 instead of h out_hd", "dense_hd80", "random", dict(head_stride=128)),
]


@pytest.mark.parametrize("what,name,family,flags", FWD_MISTAKES, ids=[f"{m[0]}-{m[2]}" for m in FWD_MISTAKES])
def test_reference_rejects_forward_mistake(what, name, family, flags):
    flags = dict(flags)
    mistake = flags.pop("mistake", None)
    if what == "row with no key stores NaN":
        # batch row 1 of the dense layout gets every key masked
        q, k, v, kk, vv, live, lm, hd, out_hd, _ = layout(name, family, 3)
        live = live.clone()
        live[1] = False
        out, lse = emulate_fwd(q, k, v, live, SCALE, hd, out_hd, **flags)
        _rejects(lambda: check_fwd(q, k, v, live, hd, out_hd, family, out, lse, what))
        out, lse = emulate_fwd(q, k, v, live, SCALE, hd, out_hd)
        check_fwd(q, k, v, live, hd, out_hd, family, out, lse, what + " (correct)")
        return
    _rejects(lambda: _fwd_case(name, family, seed=11, mistake=mistake, **flags))


# ------------------------------------------------------------------------------------------------ backward
def bwd_inputs(name, family, seed):
    """Dense (B 2, Tq 129, Tk 300 causal suffix, or non-causal with a key mask) or varlen (CU) backward inputs: q, k, v,
    out / dout head-major [B, H, Tq, 128], lse, the live set, the tiles and key liveness.  out and lse are the fp64
    forward's (rounded), as the GPU test's first run takes them.  family: random, probe_q0 (q = 0), probe_k0 (k = 0)."""
    g = _gen(seed)
    if name == "varlen":
        B, Tq, Tk, causal = 1, CU[-1], CU[-1], True
        live = A.live_varlen(CU, Tq)
        tiles, key_live = varlen_tiles(CU), torch.ones(1, Tk, dtype=torch.bool)
    else:
        causal = name == "dense_causal"
        B, Tq, Tk = 2, 129, 300
        km = torch.zeros(B, Tk, dtype=torch.uint8)
        if not causal:
            km = (torch.rand(B, Tk, generator=g) < 0.3).to(torch.uint8)
        live = A.live_dense(B, Tq, Tk, causal, km)
        tiles, key_live = dense_tiles(Tq, Tk, causal), ~km.bool()
    if family == "random":
        q, k, v = A.family_qkv(B, H, Tq, Tk, "random", g, "cpu")
        dout = _bf(torch.randn(B, H, Tq, 128, generator=g))
        ref, _, lse, _ = A.fwd_ref(q, k, v, live, SCALE)
        out, lse, scale = ref.float(), lse.float(), SCALE
    else:
        def tern(*shape):
            return torch.randint(-1, 2, shape, generator=g).float()
        q, k = tern(B, H, Tq, 128), tern(B, H, Tk, 128)
        i = torch.arange(max(Tq, Tk))
        bits = torch.stack([torch.where((i >> b) & 1 == 1, -1.0, 1.0) for b in range(10)], 1)   # [T, 10]
        if family == "probe_q0":
            q.zero_()
            k[..., :10] = bits[:Tk]                                # dQ fingerprints the keys a query sees
        else:
            k.zero_()
            q[..., :10] = bits[:Tq]                                # dK fingerprints the queries that see a key
        v = tern(B, H, Tk, 128)
        dout = tern(B, H, Tq, 128)
        dout[..., :10] = bits[:Tq]                                 # dV fingerprints the queries that see a key
        out = tern(B, H, Tq, 128)
        lse = torch.zeros(B, H, Tq)
        scale = 0.125
    return q, k, v, out, dout, lse, live, tiles, key_live, causal, scale


def check_bwd(q, k, v, out, dout, lse, live, scale, family, got, what):
    if family != "random":
        for name, g, r in zip(("dq", "dk", "dv"), got, A.bwd_exact(q, k, v, out, dout, lse, live, scale)):
            R.check_bits(g, R.bf16_rn(r).to(bf16), f"{what} {name}")
        return
    for name, g, (r, al) in zip(("dq", "dk", "dv"), got, A.bwd_ref(q, k, v, out, dout, lse, live, scale)):
        R.check_ulps(g, r, al, f"{what} {name}")


def _bwd_case(name, family, seed=0, **flags):
    q, k, v, out, dout, lse, live, tiles, key_live, causal, scale = bwd_inputs(name, family, seed)
    got = emulate_bwd(q, k, v, out, dout, lse, scale, tiles, key_live, causal, **flags)
    check_bwd(q, k, v, out, dout, lse, live, scale, family, got, f"bwd {name} {family} {flags}")


@pytest.mark.parametrize("family", ["random", "probe_q0", "probe_k0"])
@pytest.mark.parametrize("name", ["dense_causal", "dense", "varlen"])
def test_reference_accepts_the_backward_emulation(name, family):
    _bwd_case(name, family, seed=3)


def test_backward_probes_stay_exact():
    """Every dS and D of the probes is an integer of magnitude <= 256 (exact in bf16) and every sum is below 2^20."""
    for name in ("dense_causal", "varlen"):
        for family in ("probe_q0", "probe_k0"):
            q, k, v, out, dout, lse, live, *_ , scale = bwd_inputs(name, family, 3)
            Dr = (dout * out).sum(-1, keepdim=True)
            dS = (dout @ v.transpose(2, 3) - Dr) * live[:, None].float()
            assert float(dS.abs().amax()) <= 256
            for g in A.bwd_exact(q, k, v, out, dout, lse, live, scale):
                assert bool((g * 8 == (g * 8).round()).all()) and float(g.abs().amax()) * 8 < 2 ** 20


BWD_MISTAKES = [
    ("D from the neighbouring row", "dense_causal", "random", dict(d_shift=True)),
    ("D from the neighbouring row", "varlen", "probe_q0", dict(d_shift=True)),
    ("dk missing scale", "dense", "random", dict(no_dk_scale=True)),
    ("dk missing scale", "dense_causal", "probe_k0", dict(no_dk_scale=True)),
    ("m_begin one query tile late", "dense_causal", "probe_q0", dict(late_m=True)),
    ("m_begin one query tile late", "dense_causal", "random", dict(late_m=True)),
    ("varlen rows past the segment end not zeroed", "varlen", "probe_q0", dict(keep_qdead=True)),
    ("varlen rows past the segment end not zeroed", "varlen", "random", dict(keep_qdead=True)),
    ("one key tile's dQ partial lost", "dense_causal", "probe_q0", dict(lost_tile=1)),
    ("one key tile's dQ partial lost", "varlen", "random", dict(lost_tile=2)),
]


@pytest.mark.parametrize("what,name,family,flags", BWD_MISTAKES, ids=[f"{m[0]}-{m[2]}" for m in BWD_MISTAKES])
def test_reference_rejects_backward_mistake(what, name, family, flags):
    _rejects(lambda: _bwd_case(name, family, seed=5, **flags))


def test_constants_follow_the_sources():
    assert A.AT_BM == 128 and A.AT_BN == 128 and A.STAGES == {80: 4, 128: 2} and A.LAZY == 8.0
    assert A.AB_BM == 64 and A.AB_BN == 128 and A.AB_STAGES == 3 and A.PAGE_ROWS == 256
