"""GPU: the split-KV decode attention entries of aria_b200.ops against fp64, element by element (reference and allowance:
tests/decode_ref.py, which derives the kernels' worst-case fp32 error from their arithmetic).

Entry -> kernel(s) -> test -> bar:
  `attention_decode`                  attn_decode_partial<false>, attn_decode_merge<false>
                                      test_contiguous_entries_vs_fp64, test_long_rows_vs_fp64      allowance; probes bit-exact
  `attention_decode` (fp8 cache)      attn_decode_partial_fp8<false>, attn_decode_merge<false>     (same tests and bars)
  `attention_decode_devlen`           attn_decode_partial<true>, attn_decode_merge<true>
                                      test_contiguous_entries_vs_fp64, test_long_rows_vs_fp64,
                                      test_lm_shape_vs_fp64                                        (same bars)
  `attention_decode_devlen` (fp8)     attn_decode_partial_fp8<true>, attn_decode_merge<true>       (same tests and bars)
  `attention_decode_paged`            attn_decode_partial_paged, attn_decode_merge<true>
                                      test_paged_vs_fp64, test_long_rows_vs_fp64                   (same bars)
  `attention_decode_paged` (fp8)      attn_decode_partial_paged_fp8, attn_decode_merge<true>       (same tests and bars)
  `attention_decode_multi`            attn_decode_multi_partial, attn_decode_merge<true>
                                      test_multi_vs_fp64                                           (same bars)
  `attention_decode_shared_prefix`    attn_decode_prefix_partial, attn_decode_partial<true>,
                                      attn_decode_merge_shared   test_shared_prefix_vs_fp64         (same bars)

Bars: "allowance" is rowwise_ref.check_ulps(got, ref, allow): every element equal to the fp64 output rounded to bf16, or
within the ulps its fp32 error can reach (0 away from a rounding boundary).  "Probes bit-exact": with q = 0 and small
integer values (decode_ref.probe_values) the kernels must store bf16(fl32(sum v / n)) bit for bit, which shows the count
and the membership of every row's key set.

Families, on every entry: random (q, k, v ~ N(0, 1) in bf16 at the LM's scale 128^-0.5, and q x 4 for peaked rows), the
exact probe, and needles (one key about 12 nats above the rest with a distinctive value, at keys 0, 3, 4, 15, 16, 63, 64,
255, 256, 257, len - 1 and the last live key of the last split; masked on every other row, where it must leave no trace;
and one row with a needle per split, distinct values, so every split's partial must reach the merge).  Lengths come from
decode_ref (WARP_LENS, SEAM_LENS, LONG_LENS), so they follow DEC_SPLIT_KEYS.  Masks: none; 30 % random with the first and
the last live key masked, a whole split masked (its partial has M = -inf) and a row with every key masked (output 0), at a
row stride larger than T_max where the entry takes one.  q is contiguous or a strided q[:, :, pos] view of a [B, H, T, 128]
buffer whose other positions are NaN.  Every key the kernels must not read (masked, past a row's length, past a page's
live rows, pages a block table lists past a row's length) holds NaN (fp8: the NaN code and NaN scales), so a read shows.

Measured on an H100 80GB HBM3 at a 700 W power limit: see DESIGN.md section 4 (decode attention).
"""
import pytest
import torch

import decode_ref as D
import rowwise_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
bf16 = torch.bfloat16
fp8 = torch.float8_e4m3fn
F64 = torch.float64
SCALE = 128 ** -0.5
SPLIT = D.SPLIT
NAN_CODE = 0x7F
NEEDLE_LIFT = 12.0                    # nats above the row's other scores
NEEDLE_POS = [0, 3, 4, 15, 16, 63, 64, SPLIT - 1, SPLIT, SPLIT + 1]
NEEDLE_T = 4 * SPLIT + 17             # 5 splits, the last with 17 keys


def _ops():
    from aria_b200 import ops
    return ops


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _report(what, got, ref, allow):
    exact, worst, band = R.check_ulps(got.reshape(ref.shape), ref, allow, what)
    print(f"{what}: exact {exact:.5%}, worst {worst:.3g} ulps, allowance band {band:.3%}")
    return exact, worst


# ------------------------------------------------------------------------------------------------ inputs
class Rows:
    """Logical inputs of N rows x H heads over T key slots: q [N, H, 128] bf16, k / v [N, H, T, 128] (bf16, or e4m3 codes
    with ks / vs [N, H, T] fp32) and the live set [N, T]; dead keys hold NaN.  `family` in random | peaked | probe | needle;
    needles: [(row, key, masked)], and per-split needle rows."""

    def __init__(self, N, H, T, family, live, seed, fp8_cache=False, needles=(), split_needle_rows=()):
        g = _gen(seed)
        self.N, self.H, self.T, self.fp8 = N, H, T, fp8_cache
        live = live.clone()
        for r, key, masked in needles:
            live[r, key] = not masked
        self.live = live
        q = torch.randn(N, H, 128, generator=g, device=DEV) * (4.0 if family == "peaked" else 1.0)
        if family == "probe":
            q.zero_()
        self.q = q.to(bf16)
        k = torch.randn(N, H, T, 128, generator=g, device=DEV)
        v = torch.randn(N, H, T, 128, generator=g, device=DEV)
        if family == "probe":
            rows = torch.arange(N * H, device=DEV)
            v = D.probe_values(live.repeat_interleave(H, 0), rows, g).view(N, H, T, 128).float()
        if fp8_cache:
            # key scales over 2^-16 .. 2^0 of the largest (keys of at most about unit size, so the scores stay the LM's),
            # value scales over 2^-8 .. 2^8: a neighbour's scale is off by a large factor
            self.ks = torch.exp2(-torch.randint(0, 17, (N, H, T), generator=g, device=DEV).float()) * \
                (1 + torch.rand(N, H, T, generator=g, device=DEV)) / 64
            if family == "probe":
                self.vs = torch.exp2(torch.randint(-2, 3, (N, H, T), generator=g, device=DEV).float())
                self.v = v.to(fp8)
            else:
                self.vs = torch.exp2(torch.randint(-8, 9, (N, H, T), generator=g, device=DEV).float()) * \
                    (1 + torch.rand(N, H, T, generator=g, device=DEV)) / 64
                self.v = self._codes(v * 48)
            self.k = self._codes(k * 48)
        else:
            self.k, self.v = k.to(bf16), v.to(bf16)
        if family == "needle":
            for r, key, _ in needles:
                self._needle(r, [key], [3.0 + torch.arange(128, device=DEV) % 5])
            for r in split_needle_rows:
                keys = [min(s * SPLIT + 37 * (s + 1) % SPLIT, T - 1) for s in range(-(-T // SPLIT))]
                self.live[r, keys] = True
                self._needle(r, keys, [torch.full((128,), 1.0 + s, device=DEV) for s in range(len(keys))])
        self._poison()

    @staticmethod
    def _codes(x):
        """e4m3 codes with +-448, zeros and subnormals planted."""
        x = x.clamp(-448, 448)
        x[..., ::7, 0] = 448.0
        x[..., 1::7, 1] = -448.0
        x[..., 2::7, 2] = 0.0
        x[..., 3::7, 3] = 2.0 ** -9 * 5
        return x.to(fp8)

    def _needle(self, r, keys, vals):
        """Keys `keys` of row r, every head: about NEEDLE_LIFT nats above the row's other live scores, values vals."""
        for h in range(self.H):
            q = self.q[r, h].to(F64)
            kk = self.k[r, h].to(F64) * (self.ks[r, h].to(F64)[:, None] if self.fp8 else 1.0)
            s = torch.where(self.live[r], SCALE * (kk @ q), -torch.inf)
            s[keys] = -torch.inf
            top = float(s.amax()) if bool(torch.isfinite(s).any()) else 0.0
            kv = q * (top + NEEDLE_LIFT) / (SCALE * float(q @ q))
            for key, val in zip(keys, vals):
                self._set(r, h, key, kv, val)

    def _set(self, r, h, key, kv, val):
        if self.fp8:
            self.ks[r, h, key] = float(kv.abs().amax()) / 448
            self.k[r, h, key] = (kv / float(self.ks[r, h, key])).float().to(fp8)
            self.vs[r, h, key] = 1.0
            self.v[r, h, key] = val.to(fp8)
        else:
            self.k[r, h, key] = kv.to(bf16)
            self.v[r, h, key] = val.to(bf16)

    def _poison(self):
        dead = ~self.live[:, None, :].expand(self.N, self.H, self.T)
        if self.fp8:
            self.k.view(torch.uint8)[dead] = NAN_CODE
            self.v.view(torch.uint8)[dead] = NAN_CODE
            self.ks[dead] = torch.nan
            self.vs[dead] = torch.nan
        else:
            self.k[dead] = torch.nan
            self.v[dead] = torch.nan

    def q_view(self, strided):
        """q as the entries take it: contiguous, or q[:, :, 5] of a NaN [N, H, 9, 128] buffer."""
        if not strided:
            return self.q.contiguous()
        buf = torch.full((self.N, self.H, 9, 128), torch.nan, dtype=bf16, device=DEV)
        buf[:, :, 5] = self.q
        return buf[:, :, 5]

    def cache(self, T_phys=None):
        """k, v (and scales) [N, H, T_phys, 128] with NaN rows past T."""
        T_phys = T_phys or self.T + 16
        pad = T_phys - self.T
        if self.fp8:
            def padc(x):
                return torch.cat([x.view(torch.uint8), torch.full((*x.shape[:2], pad, 128), NAN_CODE, dtype=torch.uint8,
                                                                  device=DEV)], 2).view(fp8)

            def pads(x):
                return torch.cat([x, torch.full((*x.shape[:2], pad), torch.nan, device=DEV)], 2)
            return padc(self.k), padc(self.v), pads(self.ks), pads(self.vs)
        nanp = torch.full((self.N, self.H, pad, 128), torch.nan, dtype=bf16, device=DEV)
        return torch.cat([self.k, nanp], 2), torch.cat([self.v, nanp], 2), None, None

    def reference(self):
        """(ref, allow) [N H, 128] from decode_ref, or the probe's bit-exact value."""
        N, H, T = self.N, self.H, self.T
        live = self.live.repeat_interleave(H, 0)
        ks = self.ks.reshape(N * H, T) if self.fp8 else None
        vs = self.vs.reshape(N * H, T) if self.fp8 else None
        k = (self.k.view(torch.uint8) if self.fp8 else self.k).reshape(N * H, T, 128)
        v = (self.v.view(torch.uint8) if self.fp8 else self.v).reshape(N * H, T, 128)
        if self.fp8:
            k, v = k.view(fp8), v.view(fp8)
        return self.q.reshape(N * H, 128), k, v, live, ks, vs


def check(rows, family, got, what, splits=None):
    q, k, v, live, ks, vs = rows.reference()
    if family == "probe":
        R.check_bits(got.reshape(-1, 128), D.probe_ref(v, live, vs), what)
        print(f"{what}: probe bit-exact")
        return
    ref, allow = D.decode_ref(q, k, v, live, SCALE, ks, vs, splits=splits)
    _report(what, got, ref, allow)


def _masks(B, T, kind, lens, seed):
    """[B, T] bool masks (True = masked out): none; random 30 % with each row's first and last live key masked, a whole
    split masked where a row has three, and the last row fully masked."""
    m = torch.zeros(B, T, dtype=torch.bool, device=DEV)
    if kind == "none":
        return m
    g = _gen(seed)
    m = torch.rand(B, T, generator=g, device=DEV) < 0.3
    for b in range(B):
        n = int(lens[b])
        m[b, 0] = True
        m[b, n - 1] = True
        if n > 2 * SPLIT:
            m[b, SPLIT:2 * SPLIT] = True
    if B > 2:
        m[B - 1] = True
    return m


# ------------------------------------------------------------------------------------------------ contiguous entries
def _run_contiguous(entry, rows, lens, mask, strided):
    """attention_decode (Tk = lens[0] for every row) or attention_decode_devlen (lens on the device, key mask at a row
    stride past T_max) -> [N, H 128]."""
    ops = _ops()
    k, v, ks, vs = rows.cache()
    q = rows.q_view(strided)
    if entry.startswith("plain"):
        Tk = int(lens[0])
        km = mask[:, :Tk].to(torch.uint8).contiguous()
        return ops.attention_decode(q, k, v, Tk, SCALE, key_mask=km, k_scale=ks, v_scale=vs)
    T_max = k.shape[2]
    buf = torch.randint(0, 2, (rows.N, T_max + 40), dtype=torch.uint8, device=DEV)   # garbage past each row's length
    buf[:, :rows.T] = mask.to(torch.uint8)
    km = buf[:, :T_max + 3]
    return ops.attention_decode_devlen(q, k, v, torch.tensor(lens, dtype=torch.int32, device=DEV), SCALE, key_mask=km,
                                       k_scale=ks, v_scale=vs)


def _needle_case(B_mask):
    """Rows of NEEDLE_T keys: one needle per row at NEEDLE_POS, len - 1 and the last live key of the last split (the
    last 3 keys masked); masked on every other row when B_mask; then one row with a needle per split."""
    pos = NEEDLE_POS + [NEEDLE_T - 1, NEEDLE_T - 4]
    B = len(pos) + 1
    lens = [NEEDLE_T] * B
    mask = torch.zeros(B, NEEDLE_T, dtype=torch.bool, device=DEV)
    mask[len(pos) - 1, NEEDLE_T - 3:] = True
    needles = [(b, p, B_mask and b % 2 == 1 and b < len(pos) - 2) for b, p in enumerate(pos)]
    return B, lens, mask, needles, [B - 1]


CONTIGUOUS = ["plain", "plain_fp8", "devlen", "devlen_fp8"]
FAMILIES = ["random", "peaked", "probe", "needle"]


@pytest.mark.parametrize("mask_kind", ["none", "masked"])
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("entry", CONTIGUOUS)
def test_contiguous_entries_vs_fp64(entry, family, mask_kind):
    """Every warp-residue and split-seam length and 700, 2 heads, q contiguous and strided."""
    is_fp8 = entry.endswith("fp8")
    seed = CONTIGUOUS.index(entry) * 100 + FAMILIES.index(family) * 10 + (mask_kind == "masked")
    if family == "needle":
        B, lens, mask, needles, split_rows = _needle_case(mask_kind == "masked")
        rows = Rows(B, 2, NEEDLE_T, family, D.live_keys(torch.tensor(lens, device=DEV), NEEDLE_T, mask), seed, is_fp8,
                    needles, split_rows)
        got = _run_contiguous(entry, rows, lens, ~rows.live, strided=True)
        check(rows, family, got, f"{entry} needle {mask_kind}")
        return
    lengths = D.WARP_LENS + D.SEAM_LENS + [700]
    groups = [[n, n] for n in lengths] if entry.startswith("plain") else [lengths]
    for i, lens in enumerate(groups):
        T = max(lens)
        lens_t = torch.tensor(lens, device=DEV)
        mask = _masks(len(lens), T, "none" if mask_kind == "none" else "random", lens_t, seed + i)
        rows = Rows(len(lens), 2, T, family, D.live_keys(lens_t, T, mask), seed + i, is_fp8)
        got = _run_contiguous(entry, rows, lens, mask, strided=i % 2 == 1)
        check(rows, family, got, f"{entry} {family} {mask_kind} lens {lens if len(lens) < 4 else 'all'}")
    if mask_kind == "masked":                     # every key of a row masked: the output is 0
        T = 2 * SPLIT + 1
        lens = [T, T]
        mask = torch.zeros(2, T, dtype=torch.bool, device=DEV)
        mask[1] = True
        rows = Rows(2, 2, T, family, D.live_keys(torch.tensor(lens, device=DEV), T, mask), seed + 7, is_fp8)
        got = _run_contiguous(entry, rows, lens, mask, strided=False)
        assert bool((got[1] == 0).all())
        check(rows, family, got, f"{entry} {family} all keys masked")


@pytest.mark.parametrize("family", ["random", "probe"])
@pytest.mark.parametrize("entry", CONTIGUOUS + ["paged", "paged_fp8"])
def test_long_rows_vs_fp64(entry, family):
    """4097, 32768 and 65536 keys (the LM's RoPE table length) at one row x 2 heads per length."""
    is_fp8 = entry.endswith("fp8")
    seed = 1000 + 10 * (CONTIGUOUS + ["paged", "paged_fp8"]).index(entry) + (family == "probe")
    for n in D.LONG_LENS[1:]:
        lens = [n]
        mask = torch.zeros(1, n, dtype=torch.bool, device=DEV)
        rows = Rows(1, 2, n, family, D.live_keys(torch.tensor(lens, device=DEV), n, mask), seed + n, is_fp8)
        if entry.startswith("paged"):
            got = _run_paged(rows, lens, seed + n, strided=True)
        else:
            got = _run_contiguous(entry, rows, lens, mask, strided=True)
        check(rows, family, got, f"{entry} {family} {n} keys")


@pytest.mark.parametrize("family", ["random", "probe"])
@pytest.mark.parametrize("entry", ["devlen", "devlen_fp8"])
def test_lm_shape_vs_fp64(entry, family):
    """The LM's 20 heads at the engine's 64 rows, lengths 1 .. 3 splits, 30 % masked."""
    g = torch.Generator().manual_seed(5)
    lens = torch.randint(1, 3 * SPLIT + 1, (64,), generator=g).tolist()
    T = max(lens)
    lens_t = torch.tensor(lens, device=DEV)
    mask = _masks(64, T, "random", lens_t, 6)
    rows = Rows(64, 20, T, family, D.live_keys(lens_t, T, mask), 7, entry.endswith("fp8"))
    got = _run_contiguous(entry, rows, lens, mask, strided=True)
    check(rows, family, got, f"{entry} {family} B 64 H 20")


# ------------------------------------------------------------------------------------------------ paged
def _run_paged(rows, lens, seed, strided):
    """Pools of shuffled pages (rows 0 and 1 share their first page when both have one), a block table at a row stride past
    max_pages whose entries past a row's length name a NaN page, pool rows past lens NaN."""
    ops = _ops()
    N, H, T = rows.N, rows.H, rows.T
    max_pages = -(-T // SPLIT)
    live_pages = [-(-n // SPLIT) for n in lens]
    n_pages = sum(live_pages) + 3
    perm = torch.randperm(n_pages, generator=torch.Generator().manual_seed(seed)).tolist()
    nan_page = perm.pop()
    bt = torch.full((N, max_pages + 5), nan_page, dtype=torch.int32)
    share = N > 1 and lens[0] >= SPLIT and lens[1] >= SPLIT
    for r in range(N):
        for s in range(live_pages[r]):
            bt[r, s] = bt[0, 0] if (share and r == 1 and s == 0) else perm.pop()
    if share:                                    # row 1's first page is row 0's: the same keys
        for t in (rows.k, rows.v) + ((rows.ks, rows.vs) if rows.fp8 else ()):
            t[1, :, :SPLIT] = t[0, :, :SPLIT]
    bt = bt.to(DEV)
    kc, vc, ksc, vsc = rows.cache(max_pages * SPLIT)

    def pool(x, nan):
        p = torch.full((n_pages, H, SPLIT, *x.shape[3:]), nan, dtype=x.dtype if x.dtype != fp8 else torch.uint8,
                       device=DEV)
        src = x.view(torch.uint8) if x.dtype == fp8 else x
        for r in range(N):
            for s in range(live_pages[r]):
                p[int(bt[r, s])] = src[r, :, s * SPLIT:(s + 1) * SPLIT]
        return p.view(fp8) if x.dtype == fp8 else p

    nanv = NAN_CODE if rows.fp8 else torch.nan
    kp, vp = pool(kc, nanv), pool(vc, nanv)
    ksp = vsp = None
    if rows.fp8:
        ksp, vsp = pool(ksc, torch.nan), pool(vsc, torch.nan)
    got = ops.attention_decode_paged(rows.q_view(strided), kp, vp, bt[:, :max_pages],
                                     torch.tensor(lens, dtype=torch.int32, device=DEV), SCALE, k_scale=ksp, v_scale=vsp)
    # the reference reads the pages the table names (decode_ref.expand_paged), not the logical rows
    ek = D.expand_paged(kp.view(torch.uint8) if rows.fp8 else kp, bt, max_pages)
    ev = D.expand_paged(vp.view(torch.uint8) if rows.fp8 else vp, bt, max_pages)
    rows.k, rows.v = (ek.view(fp8), ev.view(fp8)) if rows.fp8 else (ek, ev)
    if rows.fp8:
        rows.ks, rows.vs = D.expand_paged(ksp, bt, max_pages), D.expand_paged(vsp, bt, max_pages)
    rows.T = max_pages * SPLIT
    rows.live = torch.nn.functional.pad(rows.live, (0, rows.T - rows.live.shape[1]))
    return got


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("R_rows", [1, 5, 64])
@pytest.mark.parametrize("is_fp8", [False, True], ids=["bf16", "fp8"])
def test_paged_vs_fp64(is_fp8, R_rows, family):
    seed = 2000 + 100 * is_fp8 + R_rows + 1000 * FAMILIES.index(family)
    H = 20 if R_rows == 64 else 2
    if family == "needle":
        if R_rows != 5:
            pytest.skip("needles run at R = 5")
        B, lens, mask, needles, split_rows = _needle_case(False)
        lens = [NEEDLE_T - int(mask[b].sum()) for b in range(B)]     # no key mask here: the masked tail keys end the row
        mask[:] = False
        T = NEEDLE_T
    else:
        lens = {1: [700], 5: [SPLIT + 1, SPLIT, 1, 2 * SPLIT + 1, 700]}.get(R_rows)
        if lens is None:
            lens = torch.randint(1, 4 * SPLIT + 1, (R_rows,), generator=torch.Generator().manual_seed(seed)).tolist()
        B, needles, split_rows = len(lens), (), ()
        T = max(lens)
        mask = torch.zeros(B, T, dtype=torch.bool, device=DEV)
    rows = Rows(B, H, T, family, D.live_keys(torch.tensor(lens, device=DEV), T, mask), seed, is_fp8, needles, split_rows)
    got = _run_paged(rows, lens, seed, strided=R_rows != 1)
    check(rows, family, got, f"paged {'fp8' if is_fp8 else 'bf16'} R {R_rows} {family}")


# ------------------------------------------------------------------------------------------------ multi-query
@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("Q", D.MULTI_QS)
def test_multi_vs_fp64(Q, family, masked):
    """Row 0's Q consecutive key counts end at SPLIT + 2 (Q = 16: 243 .. 258 cross the seam), row 1's start at 1, row 2's
    end at 700; q is a strided [B, H, Q, 128] view."""
    ops = _ops()
    B, H = 3, 2
    ends = [SPLIT + 2, Q, 700]
    lens = [[e - Q + 1 + i for i in range(Q)] for e in ends]
    T = 700
    seed = 3000 + 10 * Q + FAMILIES.index(family) + 500 * masked
    g = _gen(seed)
    mask = (torch.rand(B, T, generator=g, device=DEV) < 0.3) if masked else torch.zeros(B, T, dtype=torch.bool,
                                                                                          device=DEV)
    needles = [(0, SPLIT - 1, False), (2, 699, False)] if family == "needle" else ()
    # logical rows are the B cache rows (every key some query of the row reads is live there), q per query below
    rows = Rows(B, H, T, family, D.live_keys(torch.tensor([e for e in ends], device=DEV), T, mask), seed, False, needles)
    qbuf = torch.full((B, H, Q, 256), torch.nan, dtype=bf16, device=DEV)
    qs = torch.randn(B, H, Q, 128, generator=g, device=DEV) * (4.0 if family == "peaked" else 1.0)
    if family == "probe":
        qs.zero_()
    qs[:, :, 0] = rows.q.float()
    qbuf[..., :128] = qs.to(bf16)
    k, v, _, _ = rows.cache()
    lens_t = torch.tensor(sum(lens, []), dtype=torch.int32, device=DEV)
    km = None
    if masked:
        km = torch.ones(B, k.shape[2] + 24, dtype=torch.uint8, device=DEV)
        km[:, :T] = mask.to(torch.uint8)
    got = ops.attention_decode_multi(qbuf[..., :128], k, v, lens_t, SCALE, key_mask=km)      # [B, Q, H 128]
    # reference rows (b, i, h): the row's cache, the query's own count
    qq = qbuf[..., :128].transpose(1, 2).reshape(B * Q * H, 128)
    kk = rows.k[:, None].expand(B, Q, H, T, 128).reshape(B * Q * H, T, 128)
    vv = rows.v[:, None].expand(B, Q, H, T, 128).reshape(B * Q * H, T, 128)
    live = D.live_keys(lens_t.to(torch.int64), T, mask.repeat_interleave(Q, 0)).repeat_interleave(H, 0)
    what = f"multi Q {Q} {family} {'masked' if masked else 'unmasked'}"
    if family == "probe":
        R.check_bits(got.reshape(-1, 128), D.probe_ref(vv, live), what)
        print(f"{what}: probe bit-exact")
        return
    ref, allow = D.decode_ref(qq, kk, vv, live, SCALE)
    _report(what, got, ref, allow)


# ------------------------------------------------------------------------------------------------ shared prefix
PREFIX_LENS = [1, SPLIT - 1, SPLIT, SPLIT + 1, 700]
TAIL_LENS = [0, 1, SPLIT, SPLIT + 1]


@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("G,n", [(1, 1), (2, D.SP_TEAMS), (1, D.SP_TEAMS + 1), (2, 4 * D.SP_TEAMS)])
def test_shared_prefix_vs_fp64(G, n, family, masked):
    """Each prefix length in PREFIX_LENS (G = 2: with the next one for group 1), tails cycling through TAIL_LENS; masked: 30 %
    of the prefix and its split 1 (keys SPLIT .. 2 SPLIT - 1 of the 700-key prefix) entirely."""
    ops = _ops()
    H = 2
    R_rows = G * n
    P_max, N_max = 700 + 9, SPLIT + 1 + 7
    for i, P in enumerate(PREFIX_LENS):
        plens = [P, PREFIX_LENS[(i + 1) % len(PREFIX_LENS)]][:G]
        tlens = [TAIL_LENS[(r + i) % len(TAIL_LENS)] for r in range(R_rows)]
        seed = 4000 + 100 * i + 10 * FAMILIES.index(family) + G * n + 5000 * masked
        g = _gen(seed)
        pmask = torch.zeros(G, P_max, dtype=torch.bool, device=DEV)
        if masked:
            pmask = torch.rand(G, P_max, generator=g, device=DEV) < 0.3
            pmask[:, SPLIT:2 * SPLIT] = True
        plens_t = torch.tensor(plens, dtype=torch.int32, device=DEV)
        tlens_t = torch.tensor(tlens, dtype=torch.int32, device=DEV)
        needles = [(0, min(P - 1, SPLIT), False)] if family == "needle" else ()
        pre = Rows(G, H, P_max, family, D.live_keys(plens_t, P_max, pmask), seed, False, needles)
        tail = Rows(R_rows, H, N_max, family, D.live_keys(tlens_t, N_max), seed + 1, False)
        # q: the tail rows' q, strided, and the prefix's needle row lifted for the queries of group 0
        q = tail.q.clone()
        if family == "needle":
            q[:n] = pre.q[0:1].expand(n, H, 128)
        qbuf = torch.full((R_rows, H, 3, 128), torch.nan, dtype=bf16, device=DEV)
        qbuf[:, :, 1] = q
        pk, pv, _, _ = pre.cache(P_max)
        tk, tv, _, _ = tail.cache(N_max)
        km = torch.ones(G, P_max + 11, dtype=torch.uint8, device=DEV)
        km[:, :P_max] = pmask.to(torch.uint8)
        got = ops.attention_decode_shared_prefix(qbuf[:, :, 1], pk, pv, plens_t, tk, tv, tlens_t, n, SCALE,
                                                 prefix_mask=km if masked else None)
        k = D.expand_shared_prefix(pk, tk, n).reshape(R_rows * H, P_max + N_max, 128)
        v = D.expand_shared_prefix(pv, tv, n).reshape(R_rows * H, P_max + N_max, 128)
        live = D.live_shared_prefix(plens_t, tlens_t, n, P_max, N_max, pmask if masked else None).repeat_interleave(H, 0)
        what = f"shared prefix G {G} n {n} {family} {'masked' if masked else 'unmasked'} P {plens}"
        if family == "probe":
            R.check_bits(got.reshape(-1, 128), D.probe_ref(v, live), what)
            print(f"{what}: probe bit-exact")
            continue
        splits = -(-P_max // SPLIT) + -(-N_max // SPLIT)
        ref, allow = D.decode_ref(q.reshape(R_rows * H, 128), k, v, live, SCALE, splits=splits)
        _report(what, got, ref, allow)
