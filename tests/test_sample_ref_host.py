"""CPU proof of tests/sample_ref.py: the Philox known-answer vectors; the reference's kept sets and probabilities against
transformers' warpers and processors; and an fp32 numpy emulation of sample_body (csrc/sample.cu) in the kernel's order,
which the reference accepts on every input family, while each of 14 planted mistakes in it is rejected by a named family."""
import math

import numpy as np
import pytest
import torch

import sample_ref as S

f32 = np.float32
LANES = np.arange(32)


# ---------------------------------------------------------------------------------------------------- the emulation
def block_sum(v):
    """sample.cu block_sum on 1024 fp32 lane values: xor butterfly in each warp, then over the 32 warp sums."""
    v = np.asarray(v, dtype=f32).reshape(32, 32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[:, LANES ^ o]
    w = v[:, 0].copy()
    for o in (16, 8, 4, 2, 1):
        w = w + w[LANES ^ o]
    return w[0]


def block_scan(v):
    """sample.cu block_scan: inclusive Hillis-Steele scan in each warp, then over the warp totals, plus the warps before."""
    v = np.asarray(v, dtype=f32).reshape(32, 32).copy()
    for o in (1, 2, 4, 8, 16):
        n = np.zeros_like(v)
        n[:, o:] = v[:, :-o]
        v = np.where(LANES >= o, v + n, v)
    w = v[:, 31].copy()
    for o in (1, 2, 4, 8, 16):
        n = np.zeros_like(w)
        n[o:] = w[:-o]
        w = np.where(LANES >= o, w + n, w)
    before = np.concatenate([[f32(0)], w[:-1]]).astype(f32)
    return np.where(np.arange(32)[:, None] > 0, v + before[:, None], v).reshape(-1)


def thread_sums(vals):
    """Each thread's sequential fp32 sum over ids tid, tid + 1024, ..."""
    n = -(-vals.size // 1024) * 1024
    a = np.zeros(n, dtype=f32)
    a[:vals.size] = vals
    acc = np.zeros(1024, dtype=f32)
    for c in range(n // 1024):
        acc = acc + a[1024 * c:1024 * (c + 1)]
    return acc


def lanes(vals):
    a = np.zeros(1024, dtype=f32)
    a[:vals.size] = vals
    return a


def bf16_key(u, fix):
    u = u.astype(np.uint32)
    if fix:
        u = np.where(u == 0x8000, np.uint32(0), u)
    return np.where(u & 0x8000, ~u & 0xFFFF, u | 0x8000).astype(np.uint32)


def key_to_float(k):
    u = np.where(k & 0x8000, k & 0x7FFF, ~k & 0xFFFF).astype(np.uint32)
    return (u << np.uint32(16)).view(f32)


def f32_key(v, fix):
    u = np.asarray(v, dtype=f32).view(np.uint32).copy()
    if fix:
        u = np.where(u == 0x80000000, np.uint32(0), u)
    return np.where(u & 0x80000000, ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def f32_key_to_float(k):
    return np.where(k & 0x80000000, k & 0x7FFFFFFF, ~k).astype(np.uint32).view(f32)


def emulate_scores(x, p, mistakes):
    """The kernel's score(i) in fp32, with the processors of sample_tokens_processed."""
    v = x.float().numpy().astype(f32)
    pen = f32(p.get("penalty", 1.0))
    if pen != 1 and p.get("presence") is not None:
        pres = np.asarray(p["presence"], dtype=bool)
        pv = (v / pen) if "penalty_divides_negatives" in mistakes else np.where(v < 0, v * pen, v / pen).astype(f32)
        v = np.where(pres, pv, v).astype(f32)
    n_em, mn = p.get("n_emitted", 0), p.get("min_new", 0)
    if (n_em <= mn) if "eos_mask_one_step_long" in mistakes else (n_em < mn):
        for e in p.get("eos", ()):
            v[e] = -np.inf
    return v


def emulate_row(x, p, mistakes=frozenset()):
    """sample_body up to the draw, in fp32 and in the kernel's order -> (kept ids ascending, their fp32 scaled scores,
    probs_out row) or (greedy token,)."""
    proc = p.get("proc", False)
    fix = "signed_zero_by_key" not in mistakes
    v = emulate_scores(x, p, mistakes)
    V = v.size
    if proc:
        keys, kval, bits = f32_key(v, fix), f32_key_to_float, 32
    else:
        keys, kval, bits = bf16_key(x.view(torch.int16).numpy().astype(np.uint16), fix), key_to_float, 16
    ids = np.arange(V)
    T = f32(p["temperature"])
    comp = (keys.astype(np.uint64) << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - ids.astype(np.uint64))
    if T == 0:
        return (int(np.argmax(comp)),)
    top_k, top_p, min_p = int(p.get("top_k", 0)), f32(p.get("top_p", 1.0)), f32(p.get("min_p", 0.0))
    k = min(top_k, V)
    if k > 0:
        pivot, n_gt = 0, 0
        for shift in range(bits - 8, -1, -8):
            sel = np.ones(V, bool) if shift == bits - 8 else (keys >> np.uint32(shift + 8)) == pivot
            hist = np.bincount(((keys[sel] >> np.uint32(shift)) & 0xFF).astype(np.int64), minlength=256)
            need, cum = k - n_gt, 0
            for b in range(255, -1, -1):
                if cum < need <= cum + hist[b]:
                    binv, above = b, cum
                    break
                cum += hist[b]
            pivot = (pivot << 8) | binv
            n_gt += above
        n_tie = int(hist[binv])
        above_ids = ids[keys > pivot]
        lst = above_ids[np.lexsort((above_ids, keys[above_ids]))]          # ascending (key, id)
        assert lst.size == n_gt
        s_piv = f32(kval(np.uint32(pivot)) / T)
        s_t = (kval(keys[lst]) / T).astype(f32)
        m = s_t[-1] if n_gt else s_piv
        with np.errstate(invalid="ignore", over="ignore"):
            e_t = np.exp(s_t - m).astype(f32)
            e_piv = f32(np.exp(f32(s_piv - m)))
        cum_t = block_scan(lanes(e_t))[:n_gt]
        z = f32(f32(n_tie * e_piv) + block_sum(lanes(e_t)))
        r_tie, fk, idx_cut = 0, 0, -1
        tie_ids = ids[keys == pivot]
        if top_p < 1:
            thr = f32(f32(1) - top_p)
            q_piv = f32(e_piv / z)
            strict = "top_p_strict" in mistakes
            if q_piv <= 0:
                r_tie = n_tie
            else:
                qt = f32(thr / q_piv)
                rf = (math.ceil(qt) - 1) if strict else math.floor(qt)
                r_tie = n_tie if rf >= n_tie else int(rf)
            keep_largest = "largest_not_kept" not in mistakes
            if n_gt == 0 and keep_largest:
                r_tie = min(r_tie, n_tie - 1)
            if r_tie == n_tie:
                c = ((f32(n_tie * e_piv) + cum_t) / z).astype(f32)
                cnt = int(np.sum(c < thr if strict else c <= thr))
                fk = min(cnt, n_gt - 1) if keep_largest else cnt
            if 0 < r_tie < n_tie:
                idx_cut = int(tie_ids[r_tie - 1])
            elif r_tie == n_tie:
                idx_cut = 1 << 40
        keep = np.zeros(V, bool)
        keep[lst[fk:]] = True
        if "pivot_ties_dropped" not in mistakes:
            if "top_p_ties_highest_first" in mistakes:
                keep[tie_ids[:n_tie - r_tie]] = True
            else:
                keep[tie_ids[tie_ids > idx_cut]] = True
            z_kept = f32(f32((n_tie - r_tie) * e_piv) + block_sum(lanes(np.where(np.arange(n_gt) >= fk, e_t, 0))))
        else:
            z_kept = block_sum(lanes(np.where(np.arange(n_gt) >= fk, e_t, 0)))
    else:
        m = f32(kval(keys[int(np.argmax(comp))]) / T)
        with np.errstate(invalid="ignore", over="ignore"):
            z_kept = block_sum(thread_sums(np.exp((v / T).astype(f32) - m).astype(f32)))
        keep = np.ones(V, bool)
    s_all = (kval(keys) / T).astype(f32)
    with np.errstate(invalid="ignore", over="ignore"):
        e_all = np.exp(s_all - m).astype(f32)
    with np.errstate(divide="ignore"):                      # a planted mistake may empty the kept set
        inv_z = f32(f32(1) / z_kept)
    if proc and min_p > 0:
        inv_zm = inv_z
        if "min_p_before_top_k" in mistakes:
            with np.errstate(invalid="ignore", over="ignore"):
                inv_zm = f32(f32(1) / block_sum(thread_sums(np.exp((v / T).astype(f32) - m).astype(f32))))
        keep &= ~((e_all * inv_z).astype(f32) < f32(min_p * inv_zm))
    inv_zp = inv_z
    if proc and min_p > 0:
        inv_zp = f32(f32(1) / block_sum(thread_sums(np.where(keep, e_all, 0).astype(f32))))
    probs = np.where(keep, (e_all * inv_zp).astype(f32), f32(0)).astype(f32)
    kept = ids[keep]
    return kept, s_all[kept], probs


def emulate_draws(kept, s32, seeds, noise_rows, offsets, mistakes=frozenset()):
    """The Gumbel-max draw of sample_body for each (seed, noise row, offset), in fp32."""
    s_lo, s_hi = S.split64(seeds)
    o_lo, o_hi = S.split64(offsets)
    nr = np.asarray(noise_rows, dtype=np.uint64)
    if "offset_hi_dropped" in mistakes:
        o_hi = o_hi * np.uint64(0)
    if "seed_hi_dropped" in mistakes:
        s_hi = s_hi * np.uint64(0)
    i = kept.astype(np.uint64)[None, :]
    c0, c1 = (nr[:, None], i) if "counter_words_swapped" in mistakes else (i, nr[:, None])
    x = S.philox_x0(c0, c1, o_lo[:, None], o_hi[:, None], s_lo[:, None], s_hi[:, None])
    if "u_24_bits" in mistakes:
        u = ((x >> np.uint64(8)).astype(f32) + f32(0.5)) * f32(2.0 ** -24)
    elif "u_without_half" in mistakes:
        u = (x >> np.uint64(9)).astype(f32) * f32(2.0 ** -23)
    else:
        u = ((x >> np.uint64(9)).astype(f32) + f32(0.5)) * f32(2.0 ** -23)
    with np.errstate(divide="ignore", invalid="ignore"):
        g = -np.log(-np.log(u.astype(f32)).astype(f32)).astype(f32)
        sc = (s32[None, :] + g).astype(f32)
    sc = np.where(np.isnan(sc), -np.inf, sc)
    return kept[np.argmax(sc, axis=1)]                    # kept ascending: equal scores go to the lower id


def addressing(p, R, mistakes=frozenset()):
    """The (noise row, offset) each of R batch rows draws with: noise_rows[r] (or r), offsets[r] (per row) or offsets[0]."""
    nr = p.get("noise_rows")
    nr = np.arange(R) if nr is None or "noise_rows_ignored" in mistakes else np.asarray(nr)
    off = list(p["offsets"])
    if len(off) == 1 or "offset_from_first_row" in mistakes:
        off = [off[0]] * R
    return nr, off


# ---------------------------------------------------------------------------------------------------- the families
def bf(v):
    return torch.as_tensor(v, dtype=torch.float32).bfloat16()


def draws(R, seed=7, offsets=None, noise_rows=None):
    return dict(R=R, seeds=[seed] * R if np.isscalar(seed) else list(seed),
                offsets=list(range(R)) if offsets is None else offsets, noise_rows=noise_rows)


def fam_random():
    g = torch.Generator().manual_seed(1)
    cases = []
    for V, scale in ((257, 0.5), (1025, 3.0), (3000, 30.0), (1000, -1)):
        x = torch.randn(V, generator=g) * abs(scale)
        if scale < 0:
            x = -x.abs() - 1                                  # negative-only row
        for T, k, tp in ((1.0, 50, 0.9), (0.7, 0, 1.0), (1.3, 1024, 0.5), (1.0, 2, 1.0), (1.0, min(V, 1024), 1 - 1e-6)):
            cases.append((f"random V={V} x{scale} T={T} k={k} p={tp}", bf(x), dict(temperature=T, top_k=k, top_p=tp), draws(48)))
    return cases


def fam_ties():
    g = torch.Generator().manual_seed(2)
    cases = []
    q = torch.randint(0, 4, (2048,), generator=g).float()     # 4 levels: the k-th value repeated >> k times
    for k, tp in ((5, 1.0), (5, 0.9), (5, 0.3), (600, 0.5)):
        cases.append((f"quantized k={k} p={tp}", bf(q), dict(temperature=1.0, top_k=k, top_p=tp), draws(64)))
    for V, tp in ((4, 0.5), (4, 0.75), (256, 0.75), (256, 0.5), (1000, 0.9), (8, 1 - 2 ** -3)):
        cases.append((f"all-equal V={V} p={tp}", bf(torch.full((V,), 0.75)), dict(temperature=1.0, top_k=3, top_p=tp), draws(64)))
    x = torch.randn(500, generator=g)
    x[[3, 77, 400]] = 4.0
    cases.append(("tied maximum", bf(x), dict(temperature=1.0, top_k=10, top_p=0.8), draws(64)))
    y = torch.randn(300, generator=g) - 3                     # a tied pivot group after two larger entries: fk > 0 with all ties out
    y[[5, 6]] = 2.0
    y[[10, 20, 30, 40]] = 0.5
    cases.append(("ties removed whole, fk > 0", bf(y), dict(temperature=1.0, top_k=6, top_p=0.05), draws(64)))
    low = 1.0 + torch.arange(200) * 2.0 ** -7                 # neighbouring bf16 values: keys differ in the low byte
    cases.append(("low-byte keys", bf(low[torch.randperm(200, generator=g)]), dict(temperature=0.05, top_k=37, top_p=0.7),
                  draws(64)))
    return cases


def fam_tiny_p():
    g = torch.Generator().manual_seed(3)
    cases = []
    for V in (3, 5, 7, 11, 13, 100, 1000):
        for tp in (1e-6, 5e-8, 3e-8):
            cases.append((f"all-equal V={V} p={tp}", bf(torch.full((V,), -2.0)), dict(temperature=1.0, top_k=V, top_p=tp), draws(4)))
    for r in range(12):
        x = torch.randn(400, generator=g) * 2
        cases.append((f"random p=3e-8 #{r}", bf(x), dict(temperature=1.0, top_k=300, top_p=3e-8), draws(4)))
    return cases


def fam_signed_zero():
    cases = []
    row = bf([-5.0, -0.0, -1.0, 0.0, -1.0])
    cases.append(("[-5, -0, -1, +0, -1] greedy", row, dict(temperature=0.0), draws(4)))
    cases.append(("[-5, -0, -1, +0, -1] top_k=1", row, dict(temperature=1.0, top_k=1), draws(64)))
    g = torch.Generator().manual_seed(4)
    x = -1 - torch.rand(600, generator=g) * 3
    x[[11, 50, 90]] = 1.0
    zs = [20, 35, 61, 62, 300, 301, 500]
    x[zs] = torch.tensor([-0.0, 0.0, -0.0, -0.0, 0.0, -0.0, 0.0])
    for k, tp in ((5, 1.0), (5, 0.9), (8, 0.5), (10, 1.0)):
        cases.append((f"+-0 at the pivot k={k} p={tp}", bf(x), dict(temperature=1.0, top_k=k, top_p=tp), draws(64)))
    cases.append(("+-0 at the pivot, processed", bf(x), dict(temperature=1.0, top_k=5, top_p=0.9, proc=True), draws(64)))
    z = torch.full((64,), -3.0)
    z[[4, 9, 33]] = torch.tensor([-0.0, 0.0, -0.0])
    cases.append(("+-0 at the maximum, greedy processed", bf(z), dict(temperature=0.0, proc=True), draws(2)))
    return cases


def fam_special():
    g = torch.Generator().manual_seed(5)
    cases = []
    x = torch.full((700,), float("-inf"))
    x[[1, 99, 650]] = torch.tensor([0.5, 2.0, -1.0])
    for k, tp in ((10, 1.0), (10, 0.6), (0, 1.0)):
        cases.append((f"-inf, 3 finite, k={k} p={tp}", bf(x), dict(temperature=1.0, top_k=k, top_p=tp), draws(32)))
    sub = torch.randn(300, generator=g) * 1e-39
    cases.append(("bf16 subnormals", bf(sub), dict(temperature=1e-38, top_k=40, top_p=0.9), draws(32)))
    big = torch.randn(300, generator=g).sign() * 3e38
    big[7] = 1.0
    cases.append(("+-3e38", bf(big), dict(temperature=1.0, top_k=200, top_p=0.9), draws(32)))
    r = torch.randn(2000, generator=g) * 3
    for T in (1e-3, 100.0):
        for k, tp in ((50, 0.9), (0, 1.0), (1024, 0.5)):
            cases.append((f"T={T} k={k} p={tp}", bf(r), dict(temperature=T, top_k=k, top_p=tp), draws(32)))
    return cases


def fam_addressing():
    g = torch.Generator().manual_seed(6)
    x = bf(torch.randn(1000, generator=g))
    cases = []
    seeds = [0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 63 + 5]
    offs = [0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 40 + 3]
    for s in seeds:
        for k in (0, 100):
            cases.append((f"seed {s} k={k}", x, dict(temperature=1.0, top_k=k, top_p=1.0 if k == 0 else 0.95),
                          dict(R=40, seeds=[s] * 40, offsets=[offs[i % 5] + i // 5 for i in range(40)], noise_rows=None)))
    nr = torch.randint(0, 9, (40,), generator=g).tolist()    # permuted with repeats
    cases.append(("noise_rows permuted", x, dict(temperature=1.0, top_k=100, top_p=0.95),
                  dict(R=40, seeds=[2 ** 63 + 5] * 40, offsets=[2 ** 40 + 3 + i for i in range(40)], noise_rows=nr)))
    K = 4                                                     # prompt lookup: row b (K + 1) + i -> (noise row b, n_out[b] + i)
    n_out = [3, 2 ** 32 - 2, 17, 0]
    cases.append(("prompt-lookup mapping", x, dict(temperature=0.8, top_k=50, top_p=0.9),
                  dict(R=4 * (K + 1), seeds=[2 ** 32] * 20, offsets=[n_out[r // (K + 1)] + r % (K + 1) for r in range(20)],
                       noise_rows=[r // (K + 1) for r in range(20)])))
    cases.append(("one offset for every row", x, dict(temperature=1.0, top_k=0, proc=True),
                  dict(R=24, seeds=[5] * 24, offsets=[2 ** 32 + 9], noise_rows=None)))
    return cases


def fam_probe():
    """Two live ids per row whose logit gap is set, through the temperature, 1e-4 beside their fp64 noise gap, at draws where
    one id's 23 noise bits are within 1024 of the top (where the transform is steepest): any change to the transform
    larger than that flips the draw."""
    cases = []
    seed = 12345
    nr = np.arange(1 << 18, dtype=np.uint64)
    x = S.philox_x0(np.arange(2, dtype=np.uint64)[None, :], nr[:, None], 77, 1, seed & 0xFFFFFFFF, seed >> 32)
    hit = np.flatnonzero(((x >> np.uint64(9)) >= (1 << 23) - 1024).any(axis=1))[:48]
    for j, r in enumerate(hit):
        gg = S.gumbel64(x[r])
        gap = gg[0] - gg[1]                                   # s1 - s0 = 1 / t beside gap: id 1 wins iff 1 / t > gap
        target = gap + (1e-4 if j % 2 else -1e-4)
        if target <= 0:
            row, target = bf([1.0, 0.0]), -target             # then id 0 leads: s0 - s1 = 1 / t beside -gap
        else:
            row = bf([0.0, 1.0])
        cases.append((f"probe draw {int(r)}", row, dict(temperature=float(np.float32(1.0 / target)), top_k=0),
                      dict(R=1, seeds=[seed], offsets=[77 + 2 ** 32], noise_rows=[int(r)])))
    return cases


def fam_processed():
    g = torch.Generator().manual_seed(8)
    V = 3000
    x = torch.randn(V, generator=g) * 2
    x[[10, 20, 30]] = torch.tensor([-4.0, 5.0, 6.0])
    pres = torch.rand(V, generator=g) < 0.3
    pres[[10, 20, 30]] = True
    cases = []
    for pen in (0.5, 1.3, 2.0):
        for k, tp, mp in ((50, 0.9, 0.0), (0, 1.0, 0.05), (20, 0.95, 0.3)):
            cases.append((f"penalty {pen} k={k} p={tp} min_p={mp}", bf(x),
                          dict(temperature=1.0, top_k=k, top_p=tp, min_p=mp, penalty=pen, presence=pres.numpy(), proc=True),
                          draws(48)))
    neg = -(torch.rand(V, generator=g) * 3 + 0.5)             # negative scores with presence bits: the penalty multiplies
    cases.append(("penalty on negatives", bf(neg), dict(temperature=1.0, top_k=40, top_p=0.9, penalty=1.7,
                                                          presence=(torch.rand(V, generator=g) < 0.5).numpy(), proc=True),
                  draws(48)))
    eos = [20, 30, 2999]
    for n_em, mn in ((2, 5), (5, 5), (6, 5)):
        cases.append((f"EOS n_emitted={n_em} min_new={mn}", bf(x), dict(temperature=1.0, top_k=30, top_p=0.95, eos=eos,
                                                                       n_emitted=n_em, min_new=mn, proc=True), draws(48)))
    flat = torch.randn(4000, generator=g) * 0.5
    for k, mp in ((20, 0.3), (0, 0.3), (20, 0.05), (16, 1.0), (0, 1.0)):
        cases.append((f"min-p {mp} k={k}", bf(flat), dict(temperature=1.0, top_k=k, min_p=mp, proc=True), draws(48)))
    return cases


FAMILIES = dict(random=fam_random, ties=fam_ties, tiny_p=fam_tiny_p, signed_zero=fam_signed_zero, special=fam_special,
                addressing=fam_addressing, probe=fam_probe, processed=fam_processed)


def run_case(name, x, p, d, mistakes=frozenset(), stats=None):
    """The emulation of one case, with `mistakes` planted, checked by the reference (with the true addressing)."""
    out = emulate_row(x, p, mistakes)
    R = d["R"]
    v32 = S.scores(x, p.get("penalty", 1.0), p.get("presence"), p.get("eos", ()), p.get("n_emitted", 0), p.get("min_new", 0))
    if len(out) == 1:
        S.check_greedy(v32, [out[0]] * R, what=name)
        return
    kept, s32, probs = out
    nr_k, off_k = addressing(d, R, mistakes)
    tok = emulate_draws(kept, s32, d["seeds"], nr_k, off_k, mistakes) if kept.size else np.full(R, 2 ** 31 - 1)
    ref = S.RowRef(v32, p["temperature"], p.get("top_k", 0), p.get("top_p", 1.0), p.get("min_p", 0.0))
    kept_ref = ref.check_probs(probs, stats, name)
    nr, off = addressing(d, R)
    ref.check_draws(tok, d["seeds"], nr, off, kept_ref, stats, name)


def run_family(fam, mistakes=frozenset(), stats=None):
    for case in FAMILIES[fam]():
        run_case(*case, mistakes=mistakes, stats=stats)


# ---------------------------------------------------------------------------------------------------- tests
def test_philox_known_answers():
    F = 0xFFFFFFFF
    kat = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
           ((F, F, F, F), (F, F), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
           ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
            (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in kat:
        assert tuple(int(w) for w in S.philox4(*ctr, *key)) == want
        assert int(S.philox_x0(*ctr, *key)) == want[0]
    # vectorised: the same words element by element
    c = np.array([0, F, 0x243F6A88], dtype=np.uint64)
    got = S.philox_x0(c, [0, F, 0x85A308D3], [0, F, 0x13198A2E], [0, F, 0x03707344], [0, F, 0xA4093822], [0, F, 0x299F31D0])
    assert [int(v) for v in got] == [k[2][0] for k in kat]


def test_gumbel64_range():
    x = np.array([0, 511, 1 << 31, 0xFFFFFFFF], dtype=np.uint64)
    g = S.gumbel64(x)
    assert np.all(np.isfinite(g))
    assert g[0] == -math.log(-math.log(0.5 * 2 ** -23)) and g[-1] == -math.log(-math.log(1 - 0.5 * 2 ** -23))


def _hf_probs(x, p):
    from transformers import (LogitsProcessorList, MinNewTokensLengthLogitsProcessor, MinPLogitsWarper,
                              RepetitionPenaltyLogitsProcessor, TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper)
    V = x.numel()
    lst = LogitsProcessorList()
    ids = torch.zeros((1, 0), dtype=torch.long)
    if p.get("penalty", 1.0) != 1.0:
        ids = torch.from_numpy(np.flatnonzero(p["presence"])).view(1, -1)
        lst.append(RepetitionPenaltyLogitsProcessor(p["penalty"]))
    if p.get("min_new", 0):
        ids = torch.cat([ids, torch.zeros((1, p["n_emitted"]), dtype=torch.long)], 1)
        lst.append(MinNewTokensLengthLogitsProcessor(ids.shape[1] - p["n_emitted"], p["min_new"], p["eos"]))
    lst.append(TemperatureLogitsWarper(p["temperature"]))
    if p.get("top_k", 0):
        lst.append(TopKLogitsWarper(p["top_k"]))
    if p.get("top_p", 1.0) < 1.0:
        lst.append(TopPLogitsWarper(p["top_p"]))
    if p.get("min_p", 0.0) > 0:
        lst.append(MinPLogitsWarper(p["min_p"]))
    out = lst(ids, x.float().view(1, V).clone())
    return torch.softmax(out, -1).view(V).double().numpy()


@pytest.mark.parametrize("case", range(10))
def test_reference_equals_transformers(case):
    """On rows with one cut in the window, the reference's kept set and fp64 softmax equal transformers' warpers and
    processors within 1e-6."""
    for attempt in range(50):             # transformers' top-p sort is not stable: no cut inside a tie group
        g = torch.Generator().manual_seed(100 + case + 1000 * attempt)
        V = [50, 1000, 5000][case % 3]
        x = (torch.randn(V, generator=g) * [0.5, 3.0, 1.0][case % 3]).bfloat16()
        pres = (torch.rand(V, generator=g) < 0.2).numpy()
        p, v32, ref = _hf_case(case, x, pres)
        c = ref.lo
        if ref.lo == ref.hi and (c == 0 or v32[ref.order[c - 1]] != v32[ref.order[c]]):
            break
    else:
        pytest.fail("no row without a tie at the cut")
    kept = ref.kept(ref.lo)
    hf = _hf_probs(x, p)
    assert np.array_equal(np.sort(kept), np.flatnonzero(hf > 0))
    E = np.zeros(V)
    E[kept] = np.exp(ref.s[kept] - ref.m)
    assert np.abs(E / E.sum() - hf).max() <= 1e-6


def _hf_case(case, x, pres):
    p = [dict(temperature=1.0, top_k=10, top_p=1.0), dict(temperature=0.7, top_k=50, top_p=0.9),
         dict(temperature=1.3, top_k=0, top_p=1.0), dict(temperature=1.0, top_k=200, top_p=0.5),
         dict(temperature=1.0, top_k=0, min_p=0.1), dict(temperature=0.9, top_k=40, top_p=0.95, min_p=0.05),
         dict(temperature=1.0, top_k=30, penalty=1.3, presence=pres), dict(temperature=1.0, top_k=0, penalty=0.7, presence=pres),
         dict(temperature=1.0, top_k=25, top_p=0.9, eos=[int(torch.argmax(x.float()))], n_emitted=1, min_new=3),
         dict(temperature=1.2, top_k=100, top_p=0.8, min_p=0.2, penalty=2.0, presence=pres)][case]
    v32 = S.scores(x, p.get("penalty", 1.0), p.get("presence"), p.get("eos", ()), p.get("n_emitted", 0), p.get("min_new", 0))
    return p, v32, S.RowRef(v32, p["temperature"], p.get("top_k", 0), p.get("top_p", 1.0), p.get("min_p", 0.0))


def test_reference_ties_signed_zero_as_torch():
    """The issue's row: torch.argmax picks id 1 (-0) and TopKLogitsWarper(1) keeps {1, 3}; the reference agrees."""
    from transformers import TopKLogitsWarper
    x = bf([-5.0, -0.0, -1.0, 0.0, -1.0])
    v32 = S.scores(x)
    assert int(torch.argmax(x.float())) == 1
    S.check_greedy(v32, [1])
    S.check_sample(x, 1, temperature=0.0)
    with pytest.raises(AssertionError):
        S.check_sample(x, 3, temperature=0.0)                  # the +0 id: what a key that orders -0 below +0 returns
    kept_hf = torch.isfinite(TopKLogitsWarper(1)(None, x.float().view(1, -1))).view(-1).nonzero().view(-1).tolist()
    assert sorted(S.RowRef(v32, 1.0, 1).kept(0).tolist()) == kept_hf == [1, 3]


@pytest.mark.parametrize("fam", sorted(FAMILIES))
def test_emulation_accepted(fam):
    st = S.Stats()
    run_family(fam, stats=st)
    print(f"{fam}: {st}")
    assert st.near <= max(1, st.draws // 1000)


MISTAKES = {                   # planted mistake -> the family that must reject it
    "counter_words_swapped": "addressing",
    "offset_hi_dropped": "addressing",
    "seed_hi_dropped": "addressing",
    "u_24_bits": "probe",
    "u_without_half": "probe",
    "pivot_ties_dropped": "ties",
    "top_p_ties_highest_first": "ties",
    "top_p_strict": "ties",
    "largest_not_kept": "tiny_p",
    "noise_rows_ignored": "addressing",
    "offset_from_first_row": "addressing",
    "penalty_divides_negatives": "processed",
    "eos_mask_one_step_long": "processed",
    "min_p_before_top_k": "processed",
    "signed_zero_by_key": "signed_zero",
}


@pytest.mark.parametrize("mistake", sorted(MISTAKES))
def test_planted_mistake_rejected(mistake):
    with pytest.raises(AssertionError) as e:
        run_family(MISTAKES[mistake], mistakes=frozenset([mistake]))
    print(f"{mistake}: {str(e.value).splitlines()[0][:160]}")
