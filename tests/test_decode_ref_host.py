"""CPU: tests/decode_ref.py accepts a correct fp32 evaluation of the split-KV decode kernels and rejects planted mistakes.

`emulate` restates decode_partial + attn_decode_merge of aria_b200/csrc/attention.cu in fp32 on the CPU, in the kernels'
order: q_d scale_log2 rounded, 4 products per lane summed left to right, a 5-level xor butterfly, the fp8 key scale on the
reduced score; warp w of split s takes keys s SPLIT + 4 w + 16 i + u in (i, u) order with the online max, l and
accumulators; then the 4-warp merge and the split merge, each a max and a sequential sum of rescaled partials; A / L
rounded to bf16.  Its mistakes are the ones a split, page, scale or mask bug makes.  The emulation does not contract
multiply-adds and rounds exp2 on the CPU, both inside decode_ref's bound.
"""
import math
import re

import pytest
import torch

import decode_ref as D
import rowwise_ref as R

F32 = torch.float32
F64 = torch.float64
SCALE = 128 ** -0.5


# ------------------------------------------------------------------------------------------------ the fp32 emulation
def emulate(q, k, v, live, scale, ks=None, vs=None, *, scale_log2=None, merge=None, warp_rescale=True, twice=None):
    """q [N, 128]; k, v [N, T, 128] (bf16 values, or e4m3 code values with ks / vs [N, T]); live [N, T] -> bf16 [N, 128].
    merge: how many splits attn_decode_merge reads (default all); twice: (row, key) updated a second time at the end of
    its warp's loop; scale_log2: the fp32 factor on q (default fl(scale) fl(log2 e), as the entries pass it)."""
    N, T, Dm = k.shape
    S = -(-T // D.SPLIT)
    pad = S * D.SPLIT - T
    live = torch.nn.functional.pad(live.bool(), (0, pad))
    k = torch.nn.functional.pad(torch.where(live[:, :T, None], k.float(), 0.0), (0, 0, 0, pad))
    v = torch.nn.functional.pad(torch.where(live[:, :T, None], v.float(), 0.0), (0, 0, 0, pad))
    fp8 = ks is not None
    if fp8:
        ks = torch.nn.functional.pad(torch.where(live[:, :T], ks.float(), 0.0), (0, pad))
        vs = torch.nn.functional.pad(torch.where(live[:, :T], vs.float(), 0.0), (0, pad))
    c = torch.tensor(scale, dtype=F32) * torch.tensor(1.4426950408889634, dtype=F32) if scale_log2 is None \
        else torch.tensor(scale_log2, dtype=F32)
    qs = q.float() * c
    p = (qs[:, None, :] * k).view(N, S * D.SPLIT, 32, 4)
    s = ((p[..., 0] + p[..., 1]) + p[..., 2]) + p[..., 3]                # each lane's 4 products
    lane = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        s = s + s[..., lane ^ o]
    s = s[..., 0]
    if fp8:
        s = s * ks
    # key s SPLIT + 16 i + 4 w + u -> [N, S, i, w, u]
    shp = (N, S, D.KW // 4, D.WARPS, 4)
    s5, l5 = s.view(shp), live.view(shp)
    v5 = v.view(*shp, Dm)
    vs5 = vs.view(shp) if fp8 else None
    m = torch.full((N, S, D.WARPS), -math.inf)
    l = torch.zeros(N, S, D.WARPS)
    a = torch.zeros(N, S, D.WARPS, Dm)

    def step(sk, lv, vv, vsk):
        nonlocal m, l, a
        m_new = torch.maximum(m, sk)
        f = torch.exp2(m - m_new)
        pw = torch.exp2(sk - m_new)
        pv = pw if vsk is None else pw * vsk
        l2 = l * f + pw
        a2 = a * f[..., None] + pv[..., None] * vv
        m = torch.where(lv, m_new, m)
        l = torch.where(lv, l2, l)
        a = torch.where(lv[..., None], a2, a)

    for i in range(D.KW // 4):
        for u in range(4):
            step(s5[:, :, i, :, u], l5[:, :, i, :, u], v5[:, :, i, :, u], vs5[:, :, i, :, u] if fp8 else None)
    if twice is not None:
        n0, t0 = twice
        sp, r = divmod(t0, D.SPLIT)
        i, w, u = r // D.STEP, (r % D.STEP) // 4, r % 4
        only = torch.zeros(N, S, D.WARPS, dtype=torch.bool)
        only[n0, sp, w] = bool(live[n0, t0])
        sk = torch.full((N, S, D.WARPS), float(s[n0, t0]))
        vv = v[n0, t0].expand(N, S, D.WARPS, Dm)
        step(sk, only, vv, torch.full((N, S, D.WARPS), float(vs[n0, t0])) if fp8 else None)

    def merge_parts(mp, lp, ap, rescale=True):
        """max, then the sequential sum of the rescaled partials over dim 1."""
        M = mp.amax(1)
        L = torch.zeros(mp.shape[0], *mp.shape[2:])
        A = torch.zeros(ap.shape[0], *ap.shape[2:])
        for j in range(mp.shape[1]):
            mj = mp[:, j]
            f = torch.where(mj == -math.inf, 0.0, torch.exp2(mj - M) if rescale else torch.ones_like(mj))
            L = L + lp[:, j] * f
            A = A + ap[:, j] * f[..., None]
        return M, L, A

    Ms, Ls, As = merge_parts(m.reshape(N * S, D.WARPS), l.reshape(N * S, D.WARPS), a.reshape(N * S, D.WARPS, Dm),
                             rescale=warp_rescale)
    Ms, Ls, As = Ms.view(N, S), Ls.view(N, S), As.view(N, S, Dm)
    n = S if merge is None else merge
    _, L, A = merge_parts(Ms[:, :n], Ls[:, :n], As[:, :n])
    return torch.where(L[:, None] > 0, A / L[:, None], 0.0).to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------ inputs
LENS = [600, 517, 300]          # 3 splits at SPLIT = 256: full, full, 88 keys; and shorter rows
T = 600


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _bf(x):
    return x.to(torch.bfloat16).float()


def _rows(seed, q_mul=1.0, kind="random", masked=True):
    """q [3, 128], k, v [3, T, 128] (bf16 values), lens, mask [3, T], live."""
    g = _gen(seed)
    N = len(LENS)
    q = _bf(torch.randn(N, 128, generator=g) * q_mul)
    k = torch.randn(N, T, 128, generator=g)
    v = _bf(torch.randn(N, T, 128, generator=g))
    if kind == "late_max":       # scores increase along the keys, so every key raises its warp's maximum
        qh = q / q.norm(dim=1, keepdim=True)
        k = 0.05 * k + qh[:, None, :] * torch.linspace(0, 40, T)[None, :, None]
    k = _bf(k)
    if kind == "needle":         # key 257 of each row about 12 nats above the rest, with a distinctive value
        sc = SCALE * torch.einsum("ntd,nd->nt", k.double(), q.double())
        lam = (sc.amax(1) + 12) / (SCALE * (q.double() ** 2).sum(1))
        k[:, 257] = _bf((q.double() * lam[:, None]).float())
        v[:, 257] = 3.0 + torch.arange(128).float() % 5
    mask = (torch.rand(N, T, generator=g) < 0.3) if masked else torch.zeros(N, T, dtype=torch.bool)
    if kind == "needle":
        mask[:, 257] = False
    lens = torch.tensor(LENS)
    for b, n in enumerate(LENS):     # the last live key and the first one past it are unmasked, so lens +- 1 shows
        mask[b, n - 1] = False
        if n < T:
            mask[b, n] = False
    return q, k, v, lens, mask, D.live_keys(lens, T, mask)


def _fp8_rows(seed):
    """e4m3 code values (with +-448, zeros and subnormals); per-token scales, non-powers of two, over 2^-16 .. 2^0 (keys)
    and 2^-8 .. 2^8 (values)."""
    g = _gen(seed)
    N = len(LENS)
    q = _bf(torch.randn(N, 128, generator=g))

    def codes():
        x = (torch.randn(N, T, 128, generator=g) * 48).clamp(-448, 448)
        x[:, ::7, 0] = 448.0
        x[:, 1::7, 1] = -448.0
        x[:, 2::7, 2] = 0.0
        x[:, 3::7, 3] = 2.0 ** -9 * 3          # subnormal e4m3
        return x.to(torch.float8_e4m3fn).float()

    def scales(lo, hi):
        return torch.exp2(torch.randint(lo, hi + 1, (N, T), generator=g).float()) * (1 + torch.rand(N, T, generator=g)) / 64

    k, v = codes(), codes()
    ks, vs = scales(-16, 0), scales(-8, 8)
    mask = torch.rand(N, T, generator=g) < 0.3
    lens = torch.tensor(LENS)
    return q, k, v, ks, vs, lens, mask, D.live_keys(lens, T, mask)


def _ref(q, k, v, live, ks=None, vs=None):
    return D.decode_ref(q, k, v, live, SCALE, ks, vs)


# ------------------------------------------------------------------------------------------------ acceptance
@pytest.mark.parametrize("kind,q_mul", [("random", 1.0), ("random", 4.0), ("late_max", 1.0), ("needle", 1.0)])
def test_reference_accepts_the_fp32_emulation(kind, q_mul):
    q, k, v, lens, mask, live = _rows(1, q_mul, kind)
    ref, allow = _ref(q, k, v, live)
    got = emulate(q, k, v, live, SCALE)
    exact, worst, band = R.check_ulps(got, ref, allow, f"{kind} x{q_mul}")
    print(f"{kind} x{q_mul}: exact {exact:.4%}, worst {worst:.2g} ulps, allowance band {band:.3%}")


def test_reference_accepts_the_fp8_emulation():
    q, k, v, ks, vs, lens, mask, live = _fp8_rows(2)
    ref, allow = _ref(q, k, v, live, ks, vs)
    exact, worst, _ = R.check_ulps(emulate(q, k, v, live, SCALE, ks, vs), ref, allow, "fp8")
    print(f"fp8: exact {exact:.4%}, worst {worst:.2g} ulps")


def test_reference_of_a_row_without_live_keys_is_zero():
    q, k, v, lens, mask, live = _rows(3)
    live[1] = False
    ref, allow = _ref(q, k, v, live)
    assert bool((ref[1] == 0).all()) and bool((allow[1] == 0).all())
    R.check_ulps(emulate(q, k, v, live, SCALE), ref, allow, "empty row")


def test_paged_layout_reads_page_rows():
    g = _gen(4)
    pool = torch.randn(6, 2, D.SPLIT, 3, generator=g)
    bt = torch.tensor([[4, 0, 5], [2, 2, 1]], dtype=torch.int32)
    x = D.expand_paged(pool, bt, 3)
    for r in range(2):
        for key in (0, D.SPLIT - 1, D.SPLIT, 2 * D.SPLIT + 7):
            assert torch.equal(x[r, :, key], pool[int(bt[r, key // D.SPLIT]), :, key % D.SPLIT])


# ------------------------------------------------------------------------------------------------ planted mistakes
def _rejects(got, ref, allow, what):
    with pytest.raises(AssertionError):
        R.check_ulps(got, ref, allow, what)


def _last_live(live, row, split):
    keys = live[row, split * D.SPLIT:(split + 1) * D.SPLIT].nonzero()
    return split * D.SPLIT + int(keys[-1])


def _mistakes_bf16():
    q, k, v, lens, mask, live = _rows(5)
    base = dict(q=q, k=k, v=v, live=live)
    drop_last = live.clone()
    drop_last[0, _last_live(live, 0, 1)] = False
    drop_warp = live.clone()
    warp = 2
    for i in range(D.KW // 4):
        for u in range(4):
            drop_warp[0, D.SPLIT + 4 * warp + D.STEP * i + u] = False
    twice_key = int(live[0].nonzero()[40])
    return base, {
        "last key of a split dropped": dict(live=drop_last),
        "one warp's keys in a split dropped": dict(live=drop_warp),
        "one key counted twice": dict(twice=(0, twice_key)),
        "mask of the neighbouring row": dict(live=D.live_keys(lens, T, mask.roll(1, 0))),
        "lens one too long": dict(live=D.live_keys(lens + 1, T, mask)),
        "lens one too short": dict(live=D.live_keys(lens - 1, T, mask)),
        "last split not merged": dict(merge=-(-T // D.SPLIT) - 1),
        "scale instead of scale log2 e": dict(scale_log2=D.f32(SCALE)),
        "warp partial merged without its rescale": dict(warp_rescale=False),
    }


@pytest.mark.parametrize("mistake", list(_mistakes_bf16()[1]))
def test_reference_rejects_planted_mistakes(mistake):
    base, mistakes = _mistakes_bf16()
    ref, allow = _ref(base["q"], base["k"], base["v"], base["live"])
    kw = dict(base)
    kw.update(mistakes[mistake])
    live = kw.pop("live")
    got = emulate(kw.pop("q"), kw.pop("k"), kw.pop("v"), live, SCALE, **kw)
    _rejects(got, ref, allow, mistake)


def test_reference_rejects_rows_of_the_next_page():
    g = _gen(6)
    n_pages, max_pages = 8, 3
    kp = _bf(torch.randn(n_pages, 1, D.SPLIT, 128, generator=g))
    vp = _bf(torch.randn(n_pages, 1, D.SPLIT, 128, generator=g))
    bt = torch.tensor([[5, 1, 3], [6, 0, 2]], dtype=torch.int32)
    q = _bf(torch.randn(2, 128, generator=g))
    lens = torch.tensor([700, 600])
    live = D.live_keys(lens, max_pages * D.SPLIT)

    def rows(table):
        return D.expand_paged(kp, table, max_pages)[:, 0], D.expand_paged(vp, table, max_pages)[:, 0]

    k, v = rows(bt)
    ref, allow = _ref(q, k, v, live)
    R.check_ulps(emulate(q, k, v, live, SCALE), ref, allow, "paged")
    wrong = bt.clone()
    wrong[0, 1] += 1
    _rejects(emulate(q, *rows(wrong), live, SCALE), ref, allow, "rows of the next page")


@pytest.mark.parametrize("mistake", ["neighbouring token's k scale", "neighbouring token's v scale", "k and v scales swapped"])
def test_reference_rejects_fp8_scale_mistakes(mistake):
    q, k, v, ks, vs, lens, mask, live = _fp8_rows(7)
    ref, allow = _ref(q, k, v, live, ks, vs)
    nxt = torch.cat([ks[:, 1:], ks[:, -1:]], 1), torch.cat([vs[:, 1:], vs[:, -1:]], 1)   # min(kk + 1, T - 1)
    ks2, vs2 = {"neighbouring token's k scale": (nxt[0], vs), "neighbouring token's v scale": (ks, nxt[1]),
                "k and v scales swapped": (vs, ks)}[mistake]
    _rejects(emulate(q, k, v, live, SCALE, ks2, vs2), ref, allow, mistake)


# ------------------------------------------------------------------------------------------------ constants and probes
def test_constants_follow_the_kernels():
    src = open(f"{D.CSRC}/attention.cu").read()
    # decode_partial and decode_team_split: warp w takes keys k_begin + 4 w + STEP i + u, 4-warp CTAs / teams
    assert src.count(f"for (int k0 = k_begin + warp * 4; k0 < k_end; k0 += {D.STEP})") >= 3
    assert "__launch_bounds__(128) attn_decode_partial(" in src
    assert D.PAGE_ROWS == D.SPLIT, "a page is one split of the paged decode kernels"
    assert D.SPLIT % D.STEP == 0 and D.KW == D.SPLIT // 4
    # Q <= MULTI_Q_MAX queries per row: the lists reach one team per query and teams serving two
    assert D.MULTI_Q_MAX == 16 and re.search(rf"Q > 0 && Q <= {D.MULTI_Q_MAX}", src)
    assert D.SP_TEAMS < D.MULTI_Q_MAX <= 2 * D.SP_TEAMS
    assert D.MULTI_QS == [1, D.SP_TEAMS, D.SP_TEAMS + 1, D.MULTI_Q_MAX] and D.GROUP_NS[-1] > 2 * D.SP_TEAMS
    assert D.SEAM_LENS[:3] == [D.SPLIT - 1, D.SPLIT, D.SPLIT + 1] and D.LONG_LENS[-1] == 65536


def _probe_claim(L, mask_frac, seed):
    g = _gen(seed)
    mask = torch.rand(1, L, generator=g) < mask_frac
    live = D.live_keys(torch.tensor([L]), L, mask)
    v = D.probe_values(live, gen=g)
    ref = D.probe_ref(v, live)[0]
    x = v[0][live[0]]
    S, n = x.sum(0), x.shape[0]

    def rounded(num, den):
        return (num / den).float().to(torch.bfloat16)

    removed = rounded(S[None] - x, n - 1) if n > 1 else torch.zeros_like(x).float().to(torch.bfloat16)
    assert bool((removed != ref[None]).any(1).all()), f"L {L}: removing some key leaves every column unchanged"
    if n > 1:
        added = rounded(S[None] + x, n + 1)
        assert bool((added != ref[None]).any(1).all()), f"L {L}: counting some key twice leaves every column unchanged"
    dead = (~live[0]).nonzero()
    if len(dead):
        extra = rounded(S + v[0, int(dead[0])], n + 1)
        assert bool((extra != ref).any()), f"L {L}: reading a masked key leaves every column unchanged"


@pytest.mark.parametrize("L", D.WARP_LENS + D.SEAM_LENS + D.LONG_LENS)
def test_probe_shows_every_key(L):
    """For the exact probes: at every length they run, removing or duplicating any single key (duplicating from 2 keys on,
    where a mean can move) or reading a masked one changes at least one column of ref."""
    _probe_claim(L, 0.0, L)
    if L <= 4097:
        _probe_claim(L, 0.3, L + 1)


def test_probe_ref_is_the_fp32_quotient():
    g = _gen(8)
    live = torch.rand(4, 300, generator=g) < 0.7
    live[3] = False
    v = D.probe_values(live, gen=g)
    q = torch.zeros(4, 128)
    k = torch.randn(4, 300, 128, generator=g)
    want = D.probe_ref(v, live)
    R.check_bits(emulate(q, k, v, live, SCALE), want, "probe")
    vs = torch.exp2(torch.randint(-2, 3, (4, 300), generator=g).float())
    R.check_bits(emulate(q, k, v, live, SCALE, torch.rand(4, 300, generator=g) + 0.5, vs), D.probe_ref(v, live, vs), "fp8 probe")
