"""GPU: the sampling entries of aria_b200.ops against fp64, token by token on their own Philox noise (reference, allowances
and their derivation: tests/sample_ref.py; its CPU proof: tests/test_sample_ref_host.py).

Entry -> kernel -> test -> bar:
  `sample_tokens`            sample_kernel           test_plain_vs_fp64, test_shapes_vs_fp64,
                                                     test_full_vocabulary_vs_fp64, test_signed_zero     kept set, probs, draws
  `sample_tokens` (no probs) sample_kernel           test_plain_vs_fp64 (the same draws without probs_out)  draws, same tokens
  `sample_tokens_rows`       sample_rows_kernel      test_rows_vs_fp64, test_signed_zero                draws
  `sample_tokens_slots`      sample_slots_kernel     test_slots_vs_fp64, test_noise_probes              draws
  `sample_tokens_processed`  sample_processed_kernel test_processed_vs_fp64, test_shapes_vs_fp64,
                                                     test_signed_zero                                   kept set, probs, draws

Bars.  "Kept set": the ids with probs_out > 0 are order[c:] for one cut c inside the reference's window, in the stable
(value asc, id asc) order with -0 equal to +0, and no id outside the top-k set has a nonzero probability.  "Probs": each kept
probability is the fp64 softmax over that set within its derived allowance.  "Draws": every token is the argmax over the
kept set (the entries without probs_out: over a cut of the window) of s + gumbel64(philox_x0(i, noise row, offset lo,
offset hi, seed lo, seed hi)), accepting the runner-up only inside the derived perturbation allowance (a near tie, counted;
more than 0.1 % of a test's draws fails it).  Greedy (temperature 0) is the exact argmax, lowest id on ties, -0 tied with +0.

Draws are many batch rows of one logits row (a stride-0 view, or rows of a buffer wider than V whose padding is NaN), so
each configuration checks up to thousands of draws: row b draws noise row b (or noise_rows[b]) at its offset.  The
full-vocabulary rows at V = 100352 check a few dozen draws each.  Families: random (randn x {0.5, 3, 30}, negative-only),
ties (a tied maximum, 4-level rows with n_tie >> k, all-equal rows, cuts inside the pivot ties and past them with fk > 0,
keys that differ in the low byte), special values (+-0 at the maximum and at the pivot, -inf ids and rows with fewer finite
logits than k, bf16 subnormals, +-3e38, temperatures 1e-3 and 100), the shapes V in {1, 2, 255, 256, 257, 1000, 1023, 1024,
1025, 65537, 100352, 2^18}, top_k in {1, 2, V - 1, V, > V, 1024}, top_p in {1e-6, 0.5, 0.9, 1 - 1e-6, 1}, min_p in
{0.05, 0.3, 1}, seeds {0, 1, 2^32 - 1, 2^32, 2^63 + 5}, offsets {0, 1, 2^32 - 1, 2^32, 2^40 + 3}, permuted noise rows with
repeats, the prompt-lookup mapping, penalties {0.5, 1.3, 2} with presence bits on both sides of the pivot and on negative
logits, and EOS ids inside the top k while min_new_tokens holds and once it has passed.  Noise probes: two-id rows whose
logit gap is set, through the temperature, 1e-4 beside their fp64 noise gap at draws where the noise is steepest, so a
Gumbel transform off by more than that flips them.

Measured on an H100 80GB HBM3 at a 700 W power limit: see DESIGN.md section 4 (sampling).
"""
import numpy as np
import pytest
import torch

import sample_ref as S

pytestmark = pytest.mark.gpu
DEV = "cuda"
bf16 = torch.bfloat16
SEEDS = [0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 63 + 5]
OFFSETS = [0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 40 + 3]
MAX_PROBS_ELEMS = 1 << 25


def _ops():
    from aria_b200 import ops
    return ops


def _i64(v):
    """A uint64 as the int64 the entries read back as uint64."""
    v = int(v) & (2 ** 64 - 1)
    return v - 2 ** 64 if v >= 2 ** 63 else v


def _t64(vals):
    return torch.tensor([_i64(v) for v in vals], dtype=torch.int64, device=DEV)


def _batch(x, D, layout):
    """D batch rows holding the logits row x: a stride-0 view, or rows of a [D, V + 37] buffer whose padding is NaN."""
    V = x.numel()
    if layout == "zero":
        return x.to(DEV).view(1, V).expand(D, V)
    buf = torch.full((D, V + 37), float("nan"), dtype=bf16, device=DEV)
    buf[:, :V] = x.to(DEV)
    return buf[:, :V]


def _finish(st, what):
    print(f"{what}: {st}")
    assert st.near <= st.draws // 1000, f"{what}: {st.near} near ties in {st.draws} draws"


def _same_rows(probs):
    assert torch.equal(probs, probs[:1].expand_as(probs)), "one logits row gave different probs_out in different batch rows"
    return probs[0].cpu().numpy()


# ---------------------------------------------------------------------------------------------------- rows
def row(kind, V, seed=0):
    g = torch.Generator().manual_seed(seed * 7919 + V)
    if kind.startswith("randn"):
        return (torch.randn(V, generator=g) * float(kind[5:])).to(bf16)
    if kind == "negative":
        return (-torch.rand(V, generator=g) * 8 - 0.25).to(bf16)
    if kind == "levels":                                          # the k-th value repeated >> k times
        return (torch.randint(0, 4, (V,), generator=g).float() * 0.5).to(bf16)
    if kind == "equal":
        return torch.full((V,), 0.75, dtype=bf16)
    if kind == "tied_max":
        x = torch.randn(V, generator=g)
        x[torch.randperm(V, generator=g)[:3]] = 5.0
        return x.to(bf16)
    if kind == "fk_past_ties":                                    # two above a tie group: top-p removes the whole group
        x = torch.randn(V, generator=g) - 3
        x[torch.randperm(V, generator=g)[:2]] = 2.0
        x[torch.randperm(V, generator=g)[:6]] = 0.5
        return x.to(bf16)
    if kind == "low_byte":                                        # neighbouring bf16 values: keys differ in the low byte
        return (1.0 + (torch.randperm(V, generator=g) % 128) * 2.0 ** -7).to(bf16)
    if kind == "signed_zero":                                     # +-0 at the maximum (mixed signs, -0 first)
        x = -1 - torch.rand(V, generator=g) * 3
        z = torch.randperm(V, generator=g)[:6].sort().values
        x[z] = torch.tensor([-0.0, 0.0, -0.0, 0.0, -0.0, 0.0])
        return x.to(bf16)
    if kind == "signed_zero_pivot":                               # three above, +-0 at the pivot
        x = -1 - torch.rand(V, generator=g) * 3
        p = torch.randperm(V, generator=g)
        x[p[:3]] = 1.0
        z = p[3:10].sort().values
        x[z] = torch.tensor([-0.0, 0.0, -0.0, -0.0, 0.0, -0.0, 0.0])
        return x.to(bf16)
    if kind == "few_finite":                                      # fewer finite logits than k
        x = torch.full((V,), float("-inf"))
        x[torch.randperm(V, generator=g)[:3]] = torch.tensor([0.5, 2.0, -1.0])
        return x.to(bf16)
    if kind == "neg_inf":
        x = torch.randn(V, generator=g) * 2
        x[torch.rand(V, generator=g) < 0.3] = float("-inf")
        return x.to(bf16)
    if kind == "subnormal":
        return (torch.randn(V, generator=g) * 1e-39).to(bf16)
    if kind == "huge":
        x = torch.randn(V, generator=g).sign() * 3e38
        x[0] = 1.0
        return x.to(bf16)
    raise ValueError(kind)


# (row kind, V, temperature, top_k, top_p)
PLAIN = [
    ("randn0.5", 1000, 1.0, 50, 0.9), ("randn3", 1000, 0.7, 1024, 0.5), ("randn30", 1000, 1.0, 2, 1.0),
    ("negative", 1000, 1.3, 0, 1.0), ("randn3", 1000, 1.0, 1, 1.0), ("randn0.5", 1000, 1.0, 999, 1 - 1e-6),
    ("randn3", 1000, 1.0, 1000, 1e-6), ("randn0.5", 1000, 1.0, 1024, 1.0), ("randn0.5", 1000, 0.9, 1000, 0.9),
    ("levels", 4096, 1.0, 5, 1.0), ("levels", 4096, 1.0, 5, 0.9), ("levels", 4096, 1.0, 700, 0.5),
    ("equal", 1000, 1.0, 3, 0.9), ("equal", 256, 1.0, 1, 0.75), ("equal", 4, 1.0, 4, 0.5), ("tied_max", 1000, 1.0, 10, 0.8),
    ("fk_past_ties", 1000, 1.0, 6, 0.05), ("low_byte", 1000, 0.05, 37, 0.7), ("few_finite", 1000, 1.0, 10, 1.0),
    ("few_finite", 1000, 1.0, 10, 0.6), ("neg_inf", 1000, 1.0, 0, 1.0), ("neg_inf", 1000, 1.0, 100, 0.9),
    ("subnormal", 1000, 1e-38, 40, 0.9), ("huge", 1000, 1.0, 200, 0.9), ("randn3", 2000, 1e-3, 50, 0.9),
    ("randn3", 2000, 1e-3, 1024, 0.5), ("randn3", 2000, 100.0, 1024, 0.9), ("randn3", 2000, 100.0, 0, 1.0),
    ("signed_zero_pivot", 1000, 1.0, 5, 1.0), ("signed_zero_pivot", 1000, 1.0, 8, 0.5),
]


@pytest.mark.parametrize("case", PLAIN, ids=lambda c: "-".join(str(v) for v in c))
def test_plain_vs_fp64(case):
    """sample_tokens with probs_out (kept set, probs, draws), and the same call without probs_out draws the same tokens."""
    ops, st = _ops(), S.Stats()
    kind, V, T, k, p = case
    x = row(kind, V)
    D = min(2048, MAX_PROBS_ELEMS // V)
    ref = S.RowRef(S.scores(x), T, k, p)
    for i, (layout, seed, off) in enumerate((("zero", 7, 0), ("wide", 2 ** 63 + 5, 2 ** 40 + 3))):
        xd = _batch(x, D, layout)
        probs = torch.empty(D, V, device=DEV)
        tok = ops.sample_tokens(xd, T, k, p, seed, _t64([off]), probs_out=probs)
        tok2 = ops.sample_tokens(xd, T, k, p, seed, _t64([off]))
        assert torch.equal(tok, tok2), "probs_out changed the draws"
        kept = ref.check_probs(_same_rows(probs), st, f"{case} {layout}")
        ref.check_draws(tok.cpu().numpy(), seed, np.arange(D), off, kept, st, f"{case} {layout}")
    _finish(st, str(case))


@pytest.mark.parametrize("V", [1, 2, 255, 256, 257, 1000, 1023, 1024, 1025, 65537, 100352])
def test_shapes_vs_fp64(V):
    """Every vocabulary size at top_k {1, 2, V - 1, V, > V, 1024} (those <= 1024), top_p {0.9, 1}, with probs_out; and the
    processed entry at the same V with a penalty and min-p."""
    ops, st = _ops(), S.Stats()
    x = row("randn3", V, seed=1)
    D = max(16, min(1024, (MAX_PROBS_ELEMS // 4) // V))
    ks = sorted({k for k in (1, 2, V - 1, V, V + 5, 1024) if 1 <= k <= 1024})
    for j, k in enumerate(ks):
        for p in (1.0, 0.9):
            probs = torch.empty(D, V, device=DEV)
            seed, off = SEEDS[j % 5], OFFSETS[(j + 2) % 5]
            tok = ops.sample_tokens(_batch(x, D, "zero"), 1.0, k, p, seed, _t64([off]), probs_out=probs)
            ref = S.RowRef(S.scores(x), 1.0, k, p)
            kept = ref.check_probs(_same_rows(probs), st, f"V={V} k={k} p={p}")
            ref.check_draws(tok.cpu().numpy(), seed, np.arange(D), off, kept, st, f"V={V} k={k} p={p}")
    pres = torch.rand(V, generator=torch.Generator().manual_seed(V)) < 0.5
    _processed_case(ops, st, x, D, dict(temperature=0.8, top_k=min(V, 64), top_p=0.9, min_p=0.05, penalty=1.3,
                                        presence=pres), f"processed V={V}")
    _finish(st, f"V={V}")


@pytest.mark.parametrize("V", [100352])
def test_full_vocabulary_vs_fp64(V):
    """top_k = 0 over the LM's full vocabulary (and the processed maximum 2^18): a few dozen draws each."""
    ops, st = _ops(), S.Stats()
    for kind in ("randn3", "randn0.5"):
        x = row(kind, V, seed=2)
        D = 32
        probs = torch.empty(D, V, device=DEV)
        tok = ops.sample_tokens(_batch(x, D, "wide"), 1.0, 0, 1.0, 2 ** 32, _t64([2 ** 32 - 1]), probs_out=probs)
        ref = S.RowRef(S.scores(x), 1.0, 0, 1.0)
        kept = ref.check_probs(_same_rows(probs), st, kind)
        ref.check_draws(tok.cpu().numpy(), 2 ** 32, np.arange(D), 2 ** 32 - 1, kept, st, kind)
    big = 1 << 18
    x = row("randn3", big, seed=3)
    _processed_case(ops, st, x, 24, dict(temperature=1.0, top_k=0, min_p=0.3), "processed V=2^18 min-p")
    _processed_case(ops, st, x, 24, dict(temperature=1.0, top_k=0), "processed V=2^18 full")
    _finish(st, "full vocabulary")


def _processed_case(ops, st, x, D, p, what, layout="zero", noise_rows=None, offsets=None, n_emitted=None, eos=(),
                    min_new=0, with_probs=True, seeds=None):
    """sample_tokens_processed on D batch rows of x with one parameter set; offsets / n_emitted: lists of 1 or D entries."""
    V = x.numel()
    f = lambda v, dt=torch.float32: torch.full((D,), v, dtype=dt, device=DEV)
    pres = p.get("presence")
    bits = np.zeros((D, (V + 31) // 32), dtype=np.uint32)
    if pres is not None:
        words = np.packbits(np.asarray(pres, dtype=np.uint8), bitorder="little")
        words = np.concatenate([words, np.zeros(4 * bits.shape[1] - words.size, np.uint8)]).view(np.uint32)
        bits[:] = words
    presence = torch.from_numpy(bits.view(np.int32)).to(DEV)
    seeds = [11] * D if seeds is None else seeds
    offsets = [5] if offsets is None else offsets
    n_emitted = [0] if n_emitted is None else n_emitted
    probs = torch.empty(D, V, device=DEV) if with_probs else None
    tok = ops.sample_tokens_processed(
        _batch(x, D, layout), f(p["temperature"]), f(p.get("top_k", 0), torch.int32), f(p.get("top_p", 1.0)),
        f(p.get("min_p", 0.0)), _t64(seeds), f(p.get("penalty", 1.0)), f(min_new, torch.int32), presence, _t64(offsets),
        torch.tensor(n_emitted, dtype=torch.int32, device=DEV), eos_token_ids=eos,
        noise_rows=None if noise_rows is None else torch.tensor(noise_rows, dtype=torch.int32, device=DEV), probs_out=probs)
    tok = tok.cpu().numpy()
    nr = np.arange(D) if noise_rows is None else np.asarray(noise_rows)
    off = offsets if len(offsets) == D else offsets * D
    n_em = n_emitted if len(n_emitted) == D else n_emitted * D
    pen = p.get("penalty", 1.0)
    for ne in sorted(set(n_em)):                                  # rows that share their scores
        sel = np.flatnonzero(np.asarray(n_em) == ne)
        v32 = S.scores(x, pen, pres, eos, ne, min_new)
        if p["temperature"] == 0:
            S.check_greedy(v32, tok[sel], None if probs is None else probs[sel[0]].cpu().numpy(), what)
            continue
        ref = S.RowRef(v32, p["temperature"], p.get("top_k", 0), p.get("top_p", 1.0), p.get("min_p", 0.0))
        kept = None
        if probs is not None:
            ps = probs[torch.from_numpy(sel).to(DEV)]
            kept = ref.check_probs(_same_rows(ps), st, f"{what} n_emitted={ne}")
        ref.check_draws(tok[sel], np.asarray(seeds, dtype=object)[sel], nr[sel], np.asarray(off, dtype=object)[sel], kept, st,
                        f"{what} n_emitted={ne}")
    return tok


def test_rows_vs_fp64():
    """sample_tokens_rows: noise rows permuted with repeats, every seed and offset word pattern, and the prompt-lookup
    mapping row b (K + 1) + i -> (noise row b, offset n_out[b] + i)."""
    ops, st = _ops(), S.Stats()
    g = torch.Generator().manual_seed(5)
    for kind, V, T, k, p in (("randn0.5", 1000, 1.0, 100, 0.95), ("randn3", 1000, 0.8, 1024, 0.9), ("levels", 4096, 1.0, 5, 0.9),
                             ("signed_zero_pivot", 1000, 1.0, 5, 1.0)):
        x = row(kind, V, seed=4)
        ref = S.RowRef(S.scores(x), T, k, p)
        for seed in SEEDS:
            D = 2048
            nr = torch.randint(0, 300, (D,), generator=g).tolist()
            off = [OFFSETS[i % 5] + i // 5 for i in range(D)]
            tok = ops.sample_tokens_rows(_batch(x, D, "wide"), T, k, p, seed, torch.tensor(nr, dtype=torch.int32, device=DEV),
                                         _t64(off))
            ref.check_draws(tok.cpu().numpy(), seed, nr, off, None, st, f"rows {kind} seed {seed}")
    K, B = 4, 64                                                  # prompt lookup
    n_out = torch.randint(0, 2 ** 33, (B,), generator=g).tolist()
    R = B * (K + 1)
    nr = [r // (K + 1) for r in range(R)]
    off = [n_out[r // (K + 1)] + r % (K + 1) for r in range(R)]
    x = row("randn0.5", 1000, seed=6)
    tok = ops.sample_tokens_rows(_batch(x, R, "zero"), 0.9, 50, 0.9, 2 ** 63 + 5, torch.tensor(nr, dtype=torch.int32, device=DEV),
                                 _t64(off))
    ref = S.RowRef(S.scores(x), 0.9, 50, 0.9)
    ref.check_draws(tok.cpu().numpy(), 2 ** 63 + 5, nr, off, None, st, "prompt-lookup mapping")
    for b in (0, 17, 63):                                         # each equals generation row b's draw at n_out[b] + i
        for i in range(K + 1):
            one = ops.sample_tokens(_batch(x, b + 1, "zero"), 0.9, 50, 0.9, 2 ** 63 + 5, _t64([n_out[b] + i]))
            assert int(one[b]) == int(tok[b * (K + 1) + i])
    _finish(st, "rows")


def test_slots_vs_fp64():
    """sample_tokens_slots: every row with its own temperature, top_k, top_p and seed (greedy rows among them)."""
    ops, st = _ops(), S.Stats()
    x = row("randn3", 1000, seed=7)
    cfgs = [(1.0, 50, 0.9), (0.7, 1024, 0.5), (1.3, 2, 1.0), (0.0, 0, 1.0), (1.0, 0, 1.0), (2.0, 999, 1e-6), (1.0, 1, 1.0),
            (0.5, 300, 1 - 1e-6)]
    D = 4096
    c = np.arange(D) % len(cfgs)
    seeds = [SEEDS[i % 5] for i in range(D)]
    nr = torch.randint(0, 50, (D,), generator=torch.Generator().manual_seed(8)).tolist()
    off = [OFFSETS[(i // 3) % 5] + i for i in range(D)]
    f = lambda a, dt: torch.tensor(a, dtype=dt, device=DEV)
    tok = ops.sample_tokens_slots(_batch(x, D, "wide"), f([cfgs[j][0] for j in c], torch.float32),
                                  f([cfgs[j][1] for j in c], torch.int32), f([cfgs[j][2] for j in c], torch.float32),
                                  _t64(seeds), f(nr, torch.int32), _t64(off)).cpu().numpy()
    v32 = S.scores(x)
    for j, (T, k, p) in enumerate(cfgs):
        sel = np.flatnonzero(c == j)
        if T == 0:
            S.check_greedy(v32, tok[sel], what="slots greedy")
            continue
        ref = S.RowRef(v32, T, k, p)
        ref.check_draws(tok[sel], np.asarray(seeds, dtype=object)[sel], np.asarray(nr)[sel], np.asarray(off, dtype=object)[sel],
                        None, st, f"slots {cfgs[j]}")
    _finish(st, "slots")


def test_noise_probes():
    """Two-id rows whose logit gap 1 / t sits 1e-4 beside their fp64 noise gap, at draws where one id's 23 noise bits are
    within 1024 of the top (the transform's steepest part): the kernel's Gumbel transform and counter must both be right."""
    ops, st = _ops(), S.Stats()
    seed, off = 2 ** 63 + 5, 2 ** 40 + 3
    o_lo, o_hi = S.split64([off])
    s_lo, s_hi = S.split64([seed])
    nr = np.arange(1 << 20, dtype=np.uint64)
    xx = S.philox_x0(np.arange(2, dtype=np.uint64)[None, :], nr[:, None], o_lo, o_hi, s_lo, s_hi)
    hit = np.flatnonzero(((xx >> np.uint64(9)) >= (1 << 23) - 1024).any(axis=1))[:256]
    assert hit.size >= 128
    rows, temps = [], []
    for j, r in enumerate(hit):
        gg = S.gumbel64(xx[r])
        target = gg[0] - gg[1] + (1e-4 if j % 2 else -1e-4)      # id 1 leads by 1 / t - (g0 - g1)
        rows.append([0.0, 1.0] if target > 0 else [1.0, 0.0])
        temps.append(float(np.float32(1.0 / abs(target))))
    R = len(rows)
    x = torch.tensor(rows).to(bf16).to(DEV)
    f = lambda a, dt: torch.tensor(a, dtype=dt, device=DEV)
    tok = ops.sample_tokens_slots(x, f(temps, torch.float32), f([0] * R, torch.int32), f([1.0] * R, torch.float32),
                                  _t64([seed] * R), f(hit.tolist(), torch.int32), _t64([off] * R)).cpu().numpy()
    for i in range(R):
        ref = S.RowRef(S.scores(x[i].cpu()), temps[i], 0, 1.0)
        ref.check_draws(tok[i:i + 1], seed, int(hit[i]), off, None, st, f"probe {i}")
    _finish(st, "noise probes")


def test_processed_vs_fp64():
    """sample_tokens_processed with and without probs_out and noise_rows, rng_offset / n_emitted per row or shared:
    penalties on both sides of the pivot and on negative logits, EOS in the top k while min_new holds and after, min-p."""
    ops, st = _ops(), S.Stats()
    g = torch.Generator().manual_seed(9)
    V = 3000
    x = (torch.randn(V, generator=g) * 2)
    x[[10, 20, 30, 40]] = torch.tensor([-4.0, 5.0, 6.0, 4.5])
    x = x.to(bf16)
    pres = (torch.rand(V, generator=g) < 0.3).numpy()
    pres[[10, 20, 30]] = True
    D = 1024
    for pen in (0.5, 1.3, 2.0):
        for k, tp, mp in ((50, 0.9, 0.0), (0, 1.0, 0.05), (20, 0.95, 0.3), (16, 1.0, 1.0)):
            _processed_case(ops, st, x, D, dict(temperature=1.0, top_k=k, top_p=tp, min_p=mp, penalty=pen, presence=pres),
                            f"penalty {pen} k={k} p={tp} min_p={mp}", seeds=[SEEDS[i % 5] for i in range(D)],
                            offsets=[OFFSETS[i % 5] + i for i in range(D)])
    neg = (-(torch.rand(V, generator=g) * 3 + 0.5)).to(bf16)
    _processed_case(ops, st, neg, D, dict(temperature=1.0, top_k=40, top_p=0.9, penalty=1.7,
                                          presence=(torch.rand(V, generator=g) < 0.5).numpy()), "penalty on negatives")
    eos = [20, 30, 2999]
    n_em = [i % 8 for i in range(D)]                             # per row: rows below, at and past min_new = 5
    nr = torch.randint(0, 40, (D,), generator=g).tolist()
    for with_probs in (True, False):
        _processed_case(ops, st, x, D, dict(temperature=1.0, top_k=30, top_p=0.95), f"EOS per-row n_emitted probs={with_probs}",
                        layout="wide", noise_rows=nr, offsets=[2 ** 32 + i for i in range(D)], n_emitted=n_em, eos=eos,
                        min_new=5, with_probs=with_probs)
    for ne in (4, 5):                                             # one n_emitted and one offset for every row
        _processed_case(ops, st, x, D, dict(temperature=1.0, top_k=30, top_p=0.95), f"EOS shared n_emitted={ne}",
                        offsets=[2 ** 40 + 3], n_emitted=[ne], eos=eos, min_new=5)
    flat = (torch.randn(4000, generator=g) * 0.5).to(bf16)
    for k, mp in ((20, 0.3), (0, 0.3), (20, 0.05), (0, 1.0)):
        _processed_case(ops, st, flat, D, dict(temperature=1.0, top_k=k, min_p=mp), f"min-p {mp} k={k}")
    _processed_case(ops, st, x, 64, dict(temperature=0.0, penalty=2.0, presence=pres), "greedy processed",
                    n_emitted=[3], eos=eos, min_new=5)
    _finish(st, "processed")


def test_signed_zero():
    """-0 and +0 are one value in every entry: greedy takes the first of them, top-k keeps both, the top-p order puts the
    lower id first whatever its sign."""
    ops, st = _ops(), S.Stats()
    r5 = torch.tensor([-5.0, -0.0, -1.0, 0.0, -1.0]).to(bf16)
    D = 2048
    probs = torch.empty(D, 5, device=DEV)
    tok = ops.sample_tokens(_batch(r5, D, "zero"), 0.0, 0, 1.0, 0, None, probs_out=probs)
    S.check_greedy(S.scores(r5), tok.cpu().numpy(), _same_rows(probs), "greedy [-5, -0, -1, +0, -1]")
    tok = ops.sample_tokens(_batch(r5, D, "zero"), 1.0, 1, 1.0, 3, _t64([9]), probs_out=probs)
    ref = S.RowRef(S.scores(r5), 1.0, 1)
    kept = ref.check_probs(_same_rows(probs), st, "top_k=1 [-5, -0, -1, +0, -1]")
    assert kept.tolist() == [1, 3]
    ref.check_draws(tok.cpu().numpy(), 3, np.arange(D), 9, kept, st, "top_k=1 [-5, -0, -1, +0, -1]")
    f = lambda a, dt: torch.tensor(a, dtype=dt, device=DEV)
    one = lambda v, dt: f([v] * D, dt)
    tok = ops.sample_tokens_slots(_batch(r5, D, "zero"), one(0.0, torch.float32), one(0, torch.int32), one(1.0, torch.float32),
                                  _t64([0] * D), one(0, torch.int32), _t64([0] * D))
    S.check_greedy(S.scores(r5), tok.cpu().numpy(), what="slots greedy")
    tok = ops.sample_tokens_rows(_batch(r5, D, "zero"), 0.0, 0, 1.0, 0, one(0, torch.int32), _t64([0] * D))
    S.check_greedy(S.scores(r5), tok.cpu().numpy(), what="rows greedy")
    for kind in ("signed_zero", "signed_zero_pivot"):
        x = row(kind, 1000, seed=11)
        for k, p in ((6, 1.0), (6, 0.5), (10, 0.9)):
            probs = torch.empty(D, 1000, device=DEV)
            tok = ops.sample_tokens(_batch(x, D, "zero"), 1.0, k, p, 1, _t64([2 ** 32]), probs_out=probs)
            ref = S.RowRef(S.scores(x), 1.0, k, p)
            kept = ref.check_probs(_same_rows(probs), st, f"{kind} k={k} p={p}")
            ref.check_draws(tok.cpu().numpy(), 1, np.arange(D), 2 ** 32, kept, st, f"{kind} k={k} p={p}")
            _processed_case(ops, st, x, D, dict(temperature=1.0, top_k=k, top_p=p), f"processed {kind} k={k} p={p}")
        _processed_case(ops, st, x, 64, dict(temperature=0.0), f"processed greedy {kind}")
        tok = ops.sample_tokens(_batch(x, 64, "zero"), 0.0, 0, 1.0, 0, None)
        S.check_greedy(S.scores(x), tok.cpu().numpy(), what=f"greedy {kind}")
    _finish(st, "signed zero")
