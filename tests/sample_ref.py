"""fp64 reference for the sampling kernels of aria_b200/csrc/sample.cu (sample_kernel, sample_rows_kernel,
sample_slots_kernel and sample_processed_kernel, all compiled from sample_body).

A row is its bf16 logits x and its parameters.  The reference states what the kernel must compute:

  * Scores, exactly as the kernel forms them (`scores`): v = fp32(x); with a repetition penalty, ids set in the presence
    bitmap get torch fp32 where(v < 0, v * pen, v / pen), bit-equal to the kernel's __fmul_rn / __fdiv_rn; EOS ids are -inf
    while n_emitted < min_new.  Then s = v / t in fp64.  -0 and +0 are one value (torch compares them equal).
  * The kept set, a cut in the stable (value asc, id asc) order of the top-k set: top-k keeps every score >= the k-th
    largest, ties kept (k = min(top_k, V)); top-p removes the leading entries whose cumulative probability over the top-k
    set is <= 1 - p, never the last (the largest); min-p removes entries with p < min_p p_max, p over the top-k / top-p
    survivors, i.e. exp(s - s_max) < min_p.  Both are prefix removals in that order, so the final set is order[c:] for one
    cut c, and `RowRef` returns the window [lo, hi] of cuts the kernel may choose (below).
  * The draw: the argmax over the kept set of s + gumbel64(philox_x0(i, noise_row, off_lo, off_hi, seed_lo, seed_hi)),
    ties to the lowest id; gumbel64(x) = -log(-log u), u = ((x >> 9) + 0.5) 2^-23, in fp64.
  * Greedy (t = 0): the argmax of v, lowest id on ties, -0 tied with +0.

Allowances, from the kernel's rounding points (U = 2^-24, gamma(n) = n U / (1 - n U)):

  * Exponents.  s' = fl(v / t) and m' = fl(v_max / t) (relative U each), d' = fl(s' - m') (U |d'|), so
    |d' - d| <= Delta_i = U (|s_i| + |m| + |s_i - m|)(1 + 2U); expf is within 2 ulps (CUDA C Programming Guide; build.py does
    not pass --use_fast_math), 4 U relative.  e_i' = e_i (1 + delta_i), delta_i = exp(Delta_i)(1 + 4U) - 1.  An entry tied
    with the maximum has s' == m' bit for bit, e' = expf(0) = 1 exactly: delta_i = 0.
  * Top-p.  The kernel compares C_j' = (n_tie e_piv + scan_j) / z with thr = fl32(1 - p).  The scan and z add at most
    n_sum = 2 + 5 + 5 + 1 terms on a path (the products n_tie e_piv, the warp shuffles, the warp totals, the combine), the
    pivot-tie rule floor(thr / q_piv) one division more; so |C_j' - C_j| <= eps_p = 1.01 (2 (max delta + gamma(n_sum + 2)) +
    U) + |fl32(1 - p) - (1 - p)|, C_j <= 1.  Positions with C_j <= thr - eps_p are surely removed, those with
    C_j > thr + eps_p surely kept: lo = #{C_j <= thr - eps_p}, hi = #{C_j <= thr + eps_p}, both at most K - 1.  A row whose
    top-k set is one tie group at the maximum (every e' = 1) of power-of-two size n, with 1 - p exact in fp32, is computed
    exactly (sums of ones, q_piv = 1/n, thr / q_piv = thr n): eps_p = 0 there, so the <= of the rule itself is pinned.
  * Min-p.  The kernel removes e' fl(1/z) < fl(min_p fl(1/z)): e_i (1 +- delta_i)(1 +- U) against min_p (1 +- U).
  * Probabilities.  probs_out = fl(e' fl(1 / z')), z' the kernel's sum over its kept set: n_sum roundings in the top-k path,
    ceil(V / 1024) sequential terms per thread + 10 without top-k or when min-p renormalises.  So |p' - p| <= p (delta_i +
    max delta + gamma(n_z) + 2U) 1.01 + 2^-148, p the fp64 softmax over the kernel's own kept set.  Entries with e <
    2^-120 may round to 0 (negligible): their membership is not checked.
  * Draws.  u is exact in fp32; logf is within 1 ulp (2U relative), so -logf(u) = L (1 +- 2U) and g' = -logf(L') is within
    2.01 U + 2U |g| of g; s' adds U |s| and the sum U |s + g|.  delta_i = 1.5 (2.01 U + 2U |g_i| + U |s_i| + U |s_i + g_i|);
    the kernel's token t is accepted when s_t + g_t >= s_b + g_b - (delta_t + delta_b), b the fp64 argmax, and such a
    t != b is counted as a near tie.  Two ids with the same fp32 score and the same 23 noise bits perturb to the same fp32
    value in the kernel, so between them only the lower id is accepted.

Out of scope: NaN logits, and rows whose scores are all -inf (the kernel's m = -inf gives NaN).
"""
import numpy as np
import torch

U = 2.0 ** -24
NEGLIGIBLE = 2.0 ** -120
M32 = np.uint64(0xFFFFFFFF)
PHILOX_M0, PHILOX_M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
PHILOX_W0, PHILOX_W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
THREADS = 1024


def gamma(n):
    return n * U / (1 - n * U)


def _u64(a):
    return np.asarray(a, dtype=np.uint64)


def philox4(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 (Salmon et al., SC'11) on numpy uint64 words < 2^32, broadcast -> the four output words."""
    c0, c1, c2, c3, k0, k1 = (_u64(a) & M32 for a in (c0, c1, c2, c3, k0, k1))
    c0, c1, c2, c3, k0, k1 = np.broadcast_arrays(c0, c1, c2, c3, k0, k1)
    for _ in range(10):
        p0, p1 = PHILOX_M0 * c0, PHILOX_M1 * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M32
        k0, k1 = (k0 + PHILOX_W0) & M32, (k1 + PHILOX_W1) & M32
    return c0, c1, c2, c3


def philox_x0(c0, c1, c2, c3, k0, k1):
    return philox4(c0, c1, c2, c3, k0, k1)[0]


def gumbel64(x):
    u = ((_u64(x) >> np.uint64(9)).astype(np.float64) + 0.5) * 2.0 ** -23
    return -np.log(-np.log(u))


def split64(a):
    """uint64 values (python ints or an array) -> (lo, hi) uint64 arrays of their 32-bit words."""
    a = np.asarray([int(v) & (2 ** 64 - 1) for v in np.atleast_1d(a).tolist()], dtype=np.uint64)
    return a & M32, a >> np.uint64(32)


def scores(x, penalty=1.0, presence=None, eos=(), n_emitted=0, min_new=0):
    """The kernel's fp32 scores of one row of bf16 logits x (torch, 1-D) -> numpy float32 [V], -0 as +0."""
    v = x.detach().to("cpu", torch.bfloat16).float().clone()
    if penalty != 1.0 and presence is not None:
        p = torch.tensor(float(penalty), dtype=torch.float32)
        v = torch.where(torch.as_tensor(presence, dtype=torch.bool), torch.where(v < 0, v * p, v / p), v)
    if n_emitted < min_new:
        for e in eos:
            if 0 <= e < v.numel():
                v[e] = float("-inf")
    return v.numpy().astype(np.float32) + np.float32(0.0)


class Stats:
    """What a test reports: draws checked, near ties accepted, kept sets that used a non-central cut, the worst probs
    error in allowance units, and rows whose cut window held more than one cut."""

    def __init__(self):
        self.draws = self.near = self.window_hits = self.wide_windows = self.rows = 0
        self.probs_worst = 0.0

    def __str__(self):
        return (f"{self.draws} draws, {self.near} near ties, {self.rows} rows ({self.wide_windows} with a wide cut window, "
                f"{self.window_hits} non-central cuts), worst probs error {self.probs_worst:.3f} allowance")


class RowRef:
    """One row under (temperature > 0, top_k, top_p, min_p): the fp64 scores, the top-k set in (value asc, id asc) order,
    and the window [lo, hi] (and the exact-threshold cut mid) of cuts c such that order[c:] may be the kernel's kept set."""

    def __init__(self, v32, temperature, top_k=0, top_p=1.0, min_p=0.0):
        v32 = np.asarray(v32, dtype=np.float32) + np.float32(0.0)
        V = v32.size
        self.V, self.v32 = V, v32
        t32 = np.float32(temperature)
        self.t = float(t32)
        assert self.t > 0
        self.s = v32.astype(np.float64) / self.t
        self.s32 = v32 / t32
        order = np.argsort(v32, kind="stable")
        k = min(int(top_k), V)
        if k > 0:
            order = order[V - int(np.sum(v32 >= v32[order[V - k]])):]
        self.order, K = order, order.size
        self.K = K
        self.m = float(self.s[order[-1]])
        m32 = self.s32[order[-1]]
        with np.errstate(over="ignore", invalid="ignore"):
            so = self.s[order]
            d = so - self.m
            self.E = np.exp(d)                                  # e_j, 1 at the maximum
            self.E[~np.isfinite(so)] = 0.0
            Delta = U * (np.abs(so) + abs(self.m) + np.abs(d)) * (1 + 2 * U)
            Delta[~np.isfinite(Delta)] = np.inf
            self.delta_e = np.exp(Delta) * (1 + 4 * U) - 1
        exact_e = self.s32[order] == m32
        self.delta_e[exact_e] = 0.0
        self.E[exact_e] = 1.0
        with np.errstate(over="ignore", invalid="ignore"):
            self.negligible = ~(self.E * np.exp(-np.minimum(Delta, 700)) >= NEGLIGIBLE)
        self.negligible[exact_e] = False
        live = ~self.negligible
        dmax = float(self.delta_e[live].max())
        if k > 0:
            self.n_sum = 13
        else:
            self.n_sum = -(-V // THREADS) + 10
        if min_p > 0:
            self.n_sum = max(self.n_sum, -(-V // THREADS) + 10)
        lo = hi = mid = 0
        p32 = float(np.float32(top_p))
        if k > 0 and p32 < 1.0:
            thr = 1.0 - p32
            n = K
            exact = bool(exact_e.all()) and n & (n - 1) == 0 and float(np.float32(thr)) == thr
            eps_p = 0.0 if exact else 1.01 * (2 * (dmax + gamma(15)) + U) + abs(float(np.float32(thr)) - thr)
            P = self.E / self.E.sum()
            C = np.cumsum(P)
            if exact:
                C = np.arange(1, n + 1, dtype=np.float64) / n
            lo = min(int(np.sum(C <= thr - eps_p)), K - 1)
            hi = min(int(np.sum(C <= thr + eps_p)), K - 1)
            mid = min(int(np.sum(C <= thr)), K - 1)
        mp = float(np.float32(min_p))
        if mp > 0:
            surely_out = self.E * (1 + self.delta_e) * (1 + U) < mp * (1 - U)
            maybe_out = ~(self.E * (1 - self.delta_e) * (1 - U) >= mp * (1 + U))
            lo, hi = max(lo, int(surely_out.sum())), max(hi, int(maybe_out.sum()))
            mid = max(mid, int(np.sum(self.E < mp)))
        self.lo, self.hi, self.mid = lo, min(hi, K - 1), min(max(mid, lo), hi)

    def kept(self, c):
        return self.order[c:]

    def check_probs(self, probs, stats=None, what=""):
        """probs: the kernel's probs_out row (numpy fp32 [V]) -> its kept ids, after asserting that they are one cut in
        the window and that every probability is the fp64 softmax over that set within its allowance."""
        probs = np.asarray(probs, dtype=np.float32)
        assert np.all(np.isfinite(probs)) and np.all(probs >= 0), f"{what}: probs_out holds NaN, inf or < 0"
        inset = np.zeros(self.V, dtype=bool)
        inset[self.order] = True
        assert not np.any(probs[~inset] != 0), f"{what}: nonzero probability outside the top-k set: " \
            f"{np.flatnonzero((probs != 0) & ~inset)[:8]}"
        obs = probs[self.order] > 0
        live = ~self.negligible
        pos = np.flatnonzero(live)
        ol = obs[live]
        # the live entries the kernel kept must be a suffix of the live entries in (value asc, id asc) order
        n_out = int(np.sum(~ol))
        assert not ol[:n_out].any() and ol[n_out:].all(), \
            f"{what}: the kept set is not one cut of the (value asc, id asc) order (kept flags {ol.astype(int)[:64]})"
        c_min = int(pos[n_out - 1]) + 1 if n_out else 0          # cuts consistent with the live flags
        c_max = int(pos[n_out]) if n_out < pos.size else self.K
        assert c_max >= self.lo and c_min <= self.hi, \
            f"{what}: kept-set cut in [{c_min}, {c_max}] outside the allowed window [{self.lo}, {self.hi}] (mid {self.mid})"
        if stats is not None:
            stats.rows += 1
            stats.wide_windows += self.hi > self.lo
            stats.window_hits += not (c_min <= self.mid <= c_max)
        ids = self.order[obs]
        j = np.flatnonzero(obs)
        E = self.E[j]
        p64 = E / E.sum()
        allow = p64 * (self.delta_e[j] + float(self.delta_e[j].max()) + gamma(self.n_sum) + 2 * U) * 1.01 + 2.0 ** -148
        err = np.abs(probs[ids].astype(np.float64) - p64)
        bad = err > allow
        assert not bad.any(), f"{what}: probs_out off at ids {ids[bad][:8]}: got {probs[ids][bad][:4]}, fp64 {p64[bad][:4]}"
        if stats is not None and ids.size:
            stats.probs_worst = max(stats.probs_worst, float((err / allow).max()))
        return np.sort(ids)

    def check_draws(self, tokens, seeds, noise_rows, offsets, kept_ids=None, stats=None, what=""):
        """tokens [D]: the kernel's draws of this row with per-draw seed, noise row and offset (broadcast).  kept_ids: the
        kernel's kept set (from probs_out); None: any cut of the window, each tried from the central one outward."""
        tokens = np.atleast_1d(np.asarray(tokens, dtype=np.int64))
        D = tokens.size
        s_lo, s_hi = split64(np.broadcast_to(np.asarray(seeds, dtype=object), (D,)))
        o_lo, o_hi = split64(np.broadcast_to(np.asarray(offsets, dtype=object), (D,)))
        nr = np.broadcast_to(np.asarray(noise_rows, dtype=np.int64), (D,)).astype(np.uint64) & M32
        if kept_ids is not None:
            cands = [np.asarray(kept_ids, dtype=np.int64)]
        else:
            cs = sorted(range(self.lo, self.hi + 1), key=lambda c: (abs(c - self.mid), c))
            cands = [np.sort(self.kept(c)) for c in cs]
        ok = np.zeros(D, dtype=bool)
        near = np.zeros(D, dtype=bool)
        first = np.zeros(D, dtype=bool)
        for ci, ids in enumerate(cands):
            todo = np.flatnonzero(~ok)
            if todo.size == 0:
                break
            step = max(1, (1 << 22) // max(1, ids.size))
            for a in range(0, todo.size, step):
                dsel = todo[a:a + step]
                x = philox_x0(ids[None, :], nr[dsel, None], o_lo[dsel, None], o_hi[dsel, None], s_lo[dsel, None],
                              s_hi[dsel, None])
                g = gumbel64(x)
                s = self.s[ids][None, :]
                with np.errstate(invalid="ignore"):
                    sc = s + g
                    dl = 1.5 * (2.01 * U + 2 * U * np.abs(g) + U * np.abs(s) + U * np.abs(sc))
                sc = np.where(np.isfinite(s), sc, -np.inf)
                b = np.argmax(sc, axis=1)                         # ids ascending: exact ties go to the lowest id
                rows = np.arange(dsel.size)
                tpos = np.searchsorted(ids, tokens[dsel])
                tpos_c = np.minimum(tpos, ids.size - 1)
                member = ids[tpos_c] == tokens[dsel]
                same = tpos_c == b
                x23 = x >> np.uint64(9)
                s32 = self.s32[ids]
                ident = (s32[tpos_c] == s32[b]) & (x23[rows, tpos_c] == x23[rows, b])
                gap = sc[rows, b] - sc[rows, tpos_c]
                close = member & ~same & ~ident & (gap <= dl[rows, tpos_c] + dl[rows, b])
                good = member & (same | close)
                ok[dsel] = good
                near[dsel] = close
                first[dsel] = good & (ci == 0)
        if stats is not None:
            stats.draws += D
            stats.near += int(near.sum())
        if not ok.all():
            d = int(np.flatnonzero(~ok)[0])
            raise AssertionError(f"{what}: {int((~ok).sum())} of {D} draws are not the Gumbel argmax, first draw {d}: token "
                                 f"{int(tokens[d])} (seed {int(s_lo[d] | (s_hi[d] << np.uint64(32)))}, noise row {int(nr[d])}, "
                                 f"offset {int(o_lo[d] | (o_hi[d] << np.uint64(32)))}), window [{self.lo}, {self.hi}]")
        return int(near.sum())


def check_greedy(v32, tokens, probs=None, what=""):
    """Temperature 0: every token is the first id of the maximum score (-0 tied with +0); probs_out one-hot there."""
    v32 = np.asarray(v32, dtype=np.float32)
    best = int(np.flatnonzero(v32 == v32.max())[0])
    tokens = np.atleast_1d(np.asarray(tokens))
    assert np.all(tokens == best), f"{what}: greedy tokens {np.unique(tokens)[:8]}, expected {best}"
    if probs is not None:
        want = np.zeros(v32.size, dtype=np.float32)
        want[best] = 1.0
        assert np.array_equal(np.asarray(probs), want), f"{what}: greedy probs_out is not one-hot at {best}"


def check_sample(x, token, *, temperature, top_k=0, top_p=1.0, min_p=0.0, seed=0, noise_row=0, offset=0, probs=None,
                 penalty=1.0, presence=None, eos=(), n_emitted=0, min_new=0, stats=None, what=""):
    """One draw of one row: the kernel's token (and probs_out row, when given) against the reference."""
    v32 = scores(x, penalty, presence, eos, n_emitted, min_new)
    if temperature == 0:
        return check_greedy(v32, [token], probs, what)
    ref = RowRef(v32, temperature, top_k, top_p, min_p)
    kept = ref.check_probs(probs, stats, what) if probs is not None else None
    ref.check_draws([token], seed, noise_row, offset, kept, stats, what)
