"""fp64 reference for the wgmma prefill attention of aria_b200/csrc/attention.cu (attn_fwd_body: `attention`,
`attention_varlen`, `attention_prefill_shared_prefix`, `attention_prefill_paged_prefix`, `attention_prefill_paged_varlen`) and
the backward of aria_b200/csrc/attention_bwd.cu (`attention_bwd`, `attention_varlen_bwd`).

Every layout is stated once as a live set: a bool [B, rows, keys] over an expanded key axis (live_dense, live_varlen,
live_prefix, live_paged_varlen; keys_pool reads a prefix's keys through its page list).  fwd_ref and bwd_ref take q [B, H, rows, 128],
k / v [B, H, keys, 128] and that live set, on any device, and return (ref, allow) with tests/rowwise_ref.py's meaning: ref is
the fp64 value rounded once to bf16, allow the bf16 ulps of ref the kernel's worst-case fp32 error eta can reach (0 away from
a rounding boundary).  U = 2^-24, gamma(n) = n U / (1 - n U), G2(n) = gamma(2 n).  Nobody has measured how the tensor core
rounds its fp32 accumulator on this part; G2 assumes it may truncate, which costs 2 U per addition instead of U.

Forward (c = fl(fl(scale) fl(log2 e)) is the fp32 scale_log2 the entries pass; s_i = c_ex q.k_i with c_ex = fl(scale) log2 e,
the exact score in log2 units; o = sum w v / sum w, w_i = 2^(s_i - max) over the row's live keys; 0 and lse = -inf for a row
without one):
  * Score.  wgmma sums the HD contracted products (exact in fp32: bf16 x bf16) in HD / 16 k-steps of 16: at most HD / 16 + 16
    additions on a term, G2 of that.  c differs from c_ex by two roundings.  So |s_i' - s_i| <= D_i = (G2(HD/16 + 16) + 2 U)
    c |q|.|k_i|.  HD = 80 contracts columns 0-79 only, whatever out_hd is; so does the reference.
  * Exponent.  A key's weight is ex2(fmaf(S_i, c, -m_j)) times ex2(m_a - m_b) for each later raise of the row max.  The
    arguments telescope to s_i' - m_final, and the common shift cancels in O / l.  The fmaf rounds once, U (|s_i - max| + 8):
    the lazy max m lies at most 8 log2 units below the true running max, since it is raised only when it grows by more than
    8.  The raises' subtractions add at most U (max - min over live keys).  So each weight carries an exponent error of at most
    Delta = max_i (D_i + U |s_i - max|) + D_max + U (8 + max - min) + 8 U.  ex2.approx.ftz is within 2^-22 relative
    (the figure the project's MoE kernel tests use) and a key meets at most n_kv + 1 of them (its own and one per raise); each
    raise also multiplies O and l once in fp32 (U).
  * ftz.  ex2 flushes results below 2^-126 to zero.  The exponent is taken against m, which is at most the row's true max, so
    a flushed weight is below 2^-126 of the largest; a raise by more than 126 flushes O and l, whose weights were then below
    2^(8 - 126) of the new max.  The key at the row max has weight >= 1, so l >= 1 and all such keys add at most
    tiny = n 2^-117 (1 + max |v|).
  * l sums the fp32 P: per key tile each thread adds 32 weights in pairs (about 32 additions), after the tile's rescale; then
    2 shuffles at the end: gamma(34 n_kv + 3).  O accumulates bf16(P) V: bf16(P) is 2^-8 relative per weight (numerator
    only; bf16 keeps 8 significant bits, so its unit roundoff is 2^-8, and a peaked row at the lazy max's scale does reach
    more than 2^-9), and the chain is one accumulator addition per 16-key k-step across every tile, plus up to 16 inside a k-step and one
    rescale per tile: G2(9 n_kv + 16).
  * With eps_n bounding every numerator term and eps_d every denominator term relatively,
    |A / L - o| <= (eps_n S + eps_d |o|) / (1 - eps_d), S_d = sum w |v_d| / sum w, plus tiny.  Then inv_l = 1 / l and
    o inv_l add U each of |o| + eta.  eta <= k S_d + k' |o| + tiny; allow = allow_within(ref, o - eta, o + eta).
  * lse = ln2 (m + log2f(l)), fp32: 1.5 eps_d (log2 of the relative error of l), log2f within 2 ulps of |log2 l| <= 8 +
    log2 n, the add and the two roundings of the ln 2 product.  lse is fp32, so its allowance is the absolute bound expressed
    in (fractional) bf16 ulps of the fp64 value.

Backward: the function the kernel computes from its inputs (q, k, v, out, dout, lse), with out and lse taken as given, so the
backward is tested on its own, apart from forward error.  P = exp(scale q.k - lse) on live pairs (0 where lse = -inf),
D_i = sum_d dout_id out_id, dS = P (dout v^T - D), dV = P^T dout, dK = scale dS^T q, dQ = scale dS k.  The rounding points
(attention_bwd.cu header), carried stage to stage as gemm_ref.rnd does, in |.| products:
  * S^T: D_s as in the forward (HD = 128).  lse2 = fl(lse fl(log2 e)): 2 U |lse2|.  fmaf(S, c, -lse2): U |s - lse2|.
    ex2: 2^-22.  So P' = P (1 + eps_P), eps_P = 2^(D_s + 2 U |lse2| + U |x|) (1 + 2^-22) - 1, plus 2^-126 where it flushes.
  * dV += bf16(P') dO: one bf16 rounding (gemm_ref.rnd), then one addition per 16-query k-step over every 64-row query step
    and up to 16 inside a step, G2(4 n_m + 16).
  * dP^T = V dO^T: G2(HD/16 + 16) |dO| |V|.  D: 4 fp32 products and 3 adds per lane, then a 5-level butterfly, gamma(10)
    sum |dO out|.  dP - D and P (dP - D) each round once.  bf16(dS): gemm_ref.rnd.
  * dK += bf16(dS)^T Q: G2(4 n_m + 16); then dK scale, one fp32 rounding.  dQ: each key tile's partial over its 128 keys,
    G2(8 + 16), then one fp32 atomic add per key tile in any order: gamma(n_k) of the sum of |partials| bounds every order.
    Then dQ scale, one rounding.

Exact probes (no allowance): with q = 0 every score is exactly 0, every live weight exactly ex2(0) = 1 and every dead one
ex2(-inf) = 0; with small-integer values (probe_values: |v| < 16, so every partial sum stays below 2^20) the forward must
store bf16(fl32(fl32(sum v) fl32(1 / n))) bit for bit (fwd_probe_ref), which shows the size and membership of every row's
key set.  The backward with lse = 0, scale = 1/8 and q = 0 (or k = 0) has P = 1 on every live pair; with values in {-1, 0, 1}
every dS and D is an integer of magnitude <= 256, exact in bf16, and dV, dQ (q = 0) and dK (k = 0) must equal the
bf16-rounded exact sums (bwd_exact).  Exactness assumes wgmma's fp32 accumulation of integer sums below 2^20 is exact.
"""
import math
import os
import re

import torch

from decode_ref import expand_paged
from gemm_ref import rnd
from rowwise_ref import F64, U, allow_within, bf16_rn, gamma, ulp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "aria_b200", "csrc")
LOG2E = 1.0 / math.log(2.0)
LN2 = math.log(2.0)
EX2 = 2.0 ** -22                 # ex2.approx.ftz relative error
BF16_U = 2.0 ** -8               # bf16 unit roundoff: 8 significant bits
bf16 = torch.bfloat16


def _src(path):
    with open(os.path.join(CSRC, path)) as f:
        return f.read()


def _int(src, pattern):
    m = re.search(pattern, src)
    assert m, f"{pattern!r} not found"
    return int(m.group(1))


def kernel_constants():
    """The prefill and backward kernels' tile constants as attention.cu / attention_bwd.cu define them: the forward's query
    and key tiles, its K/V ring depth per head dim, the lazy-max threshold (log2 units), the backward's query step, key
    tile and Q/dO ring depth."""
    fw, bw = _src("attention.cu"), _src("attention_bwd.cu")
    st = re.search(r"STAGES = HD == 80 \? (\d+) : (\d+);", fw)
    thr = re.search(r"mc_lo - m_lo > ([0-9.]+)f\)", fw)
    assert st and thr
    return dict(AT_BM=_int(fw, r"constexpr int AT_BM = (\d+);"), AT_BN=_int(fw, r"constexpr int AT_BN = (\d+);"),
                STAGES={80: int(st.group(1)), 128: int(st.group(2))}, LAZY=float(thr.group(1)),
                AB_BM=_int(bw, r"constexpr int AB_BM = (\d+);"), AB_BN=_int(bw, r"constexpr int AB_BN = (\d+);"),
                AB_STAGES=_int(bw, r"constexpr int AB_STAGES = (\d+);"),
                PAGE_ROWS=_int(_src("common.cuh"), r"constexpr int PAGE_ROWS = (\d+);"))


_C = kernel_constants()
AT_BM, AT_BN, STAGES, LAZY = _C["AT_BM"], _C["AT_BN"], _C["STAGES"], _C["LAZY"]
AB_BM, AB_BN, AB_STAGES, PAGE_ROWS = _C["AB_BM"], _C["AB_BN"], _C["AB_STAGES"], _C["PAGE_ROWS"]


def G2(n):
    return gamma(2 * n)


def f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------ live sets
def live_dense(B, Tq, Tk, causal, key_mask=None, device="cpu"):
    """[B, Tq, Tk]: causal queries sit at positions pos_off + r, pos_off = Tk - Tq; key_mask [B, Tk] (1 = masked out)."""
    r = torch.arange(Tq, device=device)[:, None]
    t = torch.arange(Tk, device=device)[None, :]
    live = (t <= r + (Tk - Tq)) if causal else torch.ones(Tq, Tk, dtype=torch.bool, device=device)
    live = live[None].expand(B, Tq, Tk).clone()
    if key_mask is not None:
        live &= ~key_mask.bool()[:, None, :Tk].to(device)
    return live


def _segments(cu, n, device):
    cu = torch.as_tensor(cu, device=device).long()
    return torch.bucketize(torch.arange(n, device=device), cu[1:], right=True), cu


def live_varlen(cu, N, device="cpu"):
    """[1, N, N]: query r of segment s sees the packed keys [cu[s], r]."""
    seg, _ = _segments(cu, N, device)
    r = torch.arange(N, device=device)
    return ((seg[:, None] == seg[None, :]) & (r[None, :] <= r[:, None]))[None]


def live_prefix(cu, S_tot, P, P_keys=None, device="cpu"):
    """[1, S_tot, P_keys + S_tot] over keys [prefix rows 0 .. P_keys) + [packed suffix]: every query sees the prefix [0, P)
    and its own segment up to itself."""
    P_keys = P if P_keys is None else P_keys
    pre = (torch.arange(P_keys, device=device) < P)[None, :].expand(S_tot, P_keys)
    return torch.cat([pre, live_varlen(cu, S_tot, device)[0]], 1)[None]


def live_paged_varlen(cu, prefix_lens, S_tot, device="cpu"):
    """[1, S_tot, sum(prefix_lens) + S_tot] over keys [prefix of segment 0, .., prefix of segment n-1] + [packed rows]:
    segment b sees its own prefix_lens[b] keys and its own rows up to itself."""
    seg, _ = _segments(cu, S_tot, device)
    owner = torch.cat([torch.full((p,), b, device=device) for b, p in enumerate(prefix_lens)] +
                      [torch.zeros(0, device=device, dtype=torch.long)]).long()
    pre = seg[:, None] == owner[None, :]
    return torch.cat([pre, live_varlen(cu, S_tot, device)[0]], 1)[None]


def keys_pool(pool, pages, n_keys):
    """Prefix keys [1, H, n_keys, 128] of a page list: key PAGE_ROWS i + r is row r of pages[i]; an entry outside the pool
    reads zeros, as ops.attention_prefill_paged_prefix documents."""
    n = cdiv(n_keys, PAGE_ROWS)
    if n == 0:
        return pool.new_zeros(1, pool.shape[1], 0, pool.shape[3])
    ext = torch.cat([pool, pool.new_zeros(1, *pool.shape[1:])])
    idx = torch.as_tensor(pages[:n], device=pool.device).long()
    idx = torch.where((idx >= 0) & (idx < pool.shape[0]), idx, pool.shape[0])
    return expand_paged(ext, idx[None], n)[:, :, :n_keys]


# ------------------------------------------------------------------------------------------------ forward
def _chunks(n, per_row, budget=1 << 23):
    step = max(1, budget // max(per_row, 1))
    return [(i, min(n, i + step)) for i in range(0, n, step)]


def fwd_ref(q, k, v, live, scale, hd=128, n_kv=None):
    """q [B, H, Tq, 128], k / v [B, H, Tk, 128], live [B or 1, Tq, Tk] -> (ref [B, H, Tq, 128], allow, lse64 [B, H, Tq],
    lse_allow), fp64.  Only columns < hd of q and k are contracted (80 at the ViT path).  n_kv: the most key tiles a row's CTA
    walks (default ceil(Tk / AT_BN) + 1).  Entries outside live are never used (dead keys may hold anything finite or not)."""
    B, H, Tq, _ = q.shape
    Tk = k.shape[2]
    n_kv = cdiv(Tk, AT_BN) + 1 if n_kv is None else n_kv
    c = f32(scale) * LOG2E
    kd = G2(hd // 16 + 16) + 2 * U
    eps_l, eps_o = gamma(34 * n_kv + 3), G2(9 * n_kv + 16)
    live = live.to(q.device).bool().expand(B, Tq, Tk)
    key_any = live.any(1)[:, None, :, None]                                   # [B, 1, Tk, 1]
    k64 = torch.where(key_any, k.to(F64)[..., :hd], 0.0)
    v64 = torch.where(key_any, v.to(F64), 0.0)
    vabs = v64.abs()
    vmax = vabs.amax(2)[:, :, None]                                           # [B, H, 1, D]
    ref = torch.zeros(B, H, Tq, v.shape[-1], dtype=F64, device=q.device)
    allow = torch.zeros_like(ref)
    lse = torch.full((B, H, Tq), -math.inf, dtype=F64, device=q.device)
    lse_allow = torch.zeros_like(lse)
    for r0, r1 in _chunks(Tq, B * H * Tk):
        q64 = q[:, :, r0:r1, :hd].to(F64)
        lv = live[:, None, r0:r1]                                             # [B, 1, r, Tk]
        s = c * (q64 @ k64.transpose(2, 3))
        s = s.masked_fill(~lv, -math.inf)
        any_live = lv.any(-1)                                                 # [B, 1, r]
        smax = torch.where(any_live, s.amax(-1), 0.0)
        smin = torch.where(any_live, s.masked_fill(~lv, math.inf).amin(-1), 0.0)
        w = torch.exp2(s - smax[..., None])
        L = w.sum(-1).clamp_min(1.0)
        o = (w @ v64) / L[..., None]
        S = (w @ vabs) / L[..., None]
        D = (kd * c * (q64.abs() @ k64.abs().transpose(2, 3))).masked_fill(~lv, 0.0)
        gap = (smax[..., None] - s).masked_fill(~lv, 0.0)
        delta = (D + U * gap).amax(-1) + D.amax(-1) + U * (LAZY + smax - smin) + 8 * U
        e_w = torch.exp2(delta) * (1 + EX2) ** (n_kv + 1) * (1 + U) ** n_kv - 1
        e_d = (1 + e_w) * (1 + eps_l) - 1
        e_n = (1 + e_w) * (1 + BF16_U) * (1 + eps_o) - 1
        n = lv.sum(-1).to(F64)
        tiny = n[..., None] * 2.0 ** -117 * (1 + vmax)
        eta = (e_n[..., None] * S + e_d[..., None] * o.abs()) / (1 - e_d[..., None]) + tiny
        eta = eta + 2.01 * U * (o.abs() + eta)
        rb = bf16_rn(o)
        al = allow_within(rb, o - eta, o + eta)
        dead = ~any_live[..., None]
        ref[:, :, r0:r1] = torch.where(dead, 0.0, rb)
        allow[:, :, r0:r1] = torch.where(dead, 0.0, al)
        l2 = smax + torch.log2(L)
        ln = LN2 * l2
        err = LN2 * (1.5 * e_d + 4 * U * (LAZY + 1 + torch.log2(n.clamp_min(1))) + U * l2.abs()) + 3 * U * ln.abs()
        lse[:, :, r0:r1] = torch.where(any_live, ln, -math.inf)
        lse_allow[:, :, r0:r1] = torch.where(any_live, err / ulp(ln), 0.0)
    return ref, allow, lse, lse_allow


def fwd_probe_ref(v, live):
    """bf16(fl32(fl32(sum v) fl32(1 / n))) over each row's live keys, v [B, H, Tk, D] small integers, live [B or 1, Tq, Tk]
    -> bf16 [B, H, Tq, D]; 0 on a row with no live key.  The sums are asserted exact in fp32; 1 / n rounded through fp64 is
    the fp32 quotient (1 / n lies at least 2^-41 of itself from an fp32 midpoint unless n is a power of two)."""
    B, H, Tk, Dm = v.shape
    x = v.to(F64)
    assert bool((x == x.round()).all()) and float(x.abs().amax()) < 16
    lv = live.to(v.device).bool().expand(B, live.shape[1], Tk).to(F64)
    ssum = torch.einsum("bqt,bhtd->bhqd", lv, x)
    assert float(torch.einsum("bqt,bhtd->bhqd", lv, x.abs()).amax()) < 2 ** 20
    n = lv.sum(-1)[:, None, :, None]
    inv = torch.where(n > 0, 1.0 / n.clamp_min(1), 0.0).float()
    return (ssum.float() * inv).to(bf16)


def probe_values(H, T, head0=0, gen=None, device="cpu"):
    """Small integers [H, T, 128] in [-15, 15] that fingerprint the key index t: columns 0..16 (-1)^bit b of t, 17..20 the
    nibbles of t, 21 t mod 7, 22 t mod 13, 23 a constant per head (head0 + h), the rest random in [-8, 8]."""
    t = torch.arange(T, device=device)
    v = torch.randint(-8, 9, (H, T, 128), generator=gen, device=device).to(F64)
    for b in range(17):
        v[:, :, b] = torch.where((t >> b) & 1 == 1, -1.0, 1.0)
    for j in range(4):
        v[:, :, 17 + j] = ((t >> (4 * j)) % 16).to(F64) - 7
    v[:, :, 21] = (t % 7).to(F64)
    v[:, :, 22] = (t % 13).to(F64) - 6
    v[:, :, 23] = ((torch.arange(H, device=device) + head0) % 29 - 14).to(F64)[:, None]
    return v


# ------------------------------------------------------------------------------------------------ backward
def bwd_exact(q, k, v, out, dout, lse, live, scale):
    """The backward's exact value in fp64: q [B, H, Tq, 128], k / v [B, H, Tk, 128], out / dout [B, H, Tq, 128] (head-major
    views of the token-major tensors), lse [B, H, Tq], live [B or 1, Tq, Tk] -> (dq, dk, dv) fp64."""
    return _bwd(q, k, v, out, dout, lse, live, scale, bounds=False)


def bwd_ref(q, k, v, out, dout, lse, live, scale, n_m=None, n_k=None):
    """bwd_exact rounded to bf16 with its allowances: ((dq, allow), (dk, allow), (dv, allow)).  n_m: the most 64-row query
    steps a key tile walks (default ceil(Tq / AB_BM) + 1); n_k: the most key tiles adding to one dQ row (default
    ceil(Tk / AB_BN) + 1)."""
    return _bwd(q, k, v, out, dout, lse, live, scale, bounds=True, n_m=n_m, n_k=n_k)


def _bwd(q, k, v, out, dout, lse, live, scale, bounds, n_m=None, n_k=None):
    B, H, Tq, Dm = q.shape
    Tk = k.shape[2]
    n_m = cdiv(Tq, AB_BM) + 1 if n_m is None else n_m
    n_k = cdiv(Tk, AB_BN) + 1 if n_k is None else n_k
    sc = f32(scale)
    c = sc * LOG2E
    kd = G2(Dm // 16 + 16) + 2 * U
    live = live.to(q.device).bool().expand(B, Tq, Tk)
    key_any = live.any(1)[:, None, :, None]
    k64 = torch.where(key_any, k.to(F64), 0.0)
    v64 = torch.where(key_any, v.to(F64), 0.0)
    ka, va = k64.abs(), v64.abs()
    dk = torch.zeros(B, H, Tk, Dm, dtype=F64, device=q.device)
    dv = torch.zeros_like(dk)
    dq = torch.zeros(B, H, Tq, Dm, dtype=F64, device=q.device)
    if bounds:
        dk_e, dk_a, dv_e, dv_a = (torch.zeros_like(dk) for _ in range(4))
        dq_e = torch.zeros_like(dq)
    for r0, r1 in _chunks(Tq, B * H * Tk):
        q64, o64, g64 = (t[:, :, r0:r1].to(F64) for t in (q, out, dout))
        qa, ga = q64.abs(), g64.abs()
        lv = live[:, None, r0:r1]
        l64 = lse[:, :, r0:r1].to(F64)[..., None]
        lse2 = l64 * LOG2E
        s = c * (q64 @ k64.transpose(2, 3))
        x = s - lse2
        P = torch.where(lv & torch.isfinite(l64), torch.exp2(x), 0.0)
        Dr = (g64 * o64).sum(-1, keepdim=True)
        dP = g64 @ v64.transpose(2, 3)
        dS = P * (dP - Dr)
        dv += P.transpose(2, 3) @ g64
        dk += sc * (dS.transpose(2, 3) @ q64)
        dq[:, :, r0:r1] = sc * (dS @ k64)
        if not bounds:
            continue
        fin = lv & torch.isfinite(l64)
        lse2a = torch.where(torch.isfinite(lse2), lse2.abs(), 0.0)
        xa = torch.where(fin, x.abs(), 0.0)
        dsc = kd * c * (qa @ ka.transpose(2, 3))
        eP = torch.where(fin, P * (torch.exp2(dsc + 2 * U * lse2a + U * xa) * (1 + EX2) - 1) + 2.0 ** -126, 0.0)
        eb = torch.where(fin, rnd(P, eP), 0.0)
        dv_e += eb.transpose(2, 3) @ ga
        dv_a += (P + eb).transpose(2, 3) @ ga
        A = (dP - Dr).abs()
        e_t = G2(Dm // 16 + 16) * (ga @ va.transpose(2, 3)) + gamma(10) * (ga * o64.abs()).sum(-1, keepdim=True)
        e_t = e_t + U * (A + e_t)
        e_dS = torch.where(fin, eP * (A + e_t) + P * e_t + U * (P + eP) * (A + e_t), 0.0)
        e_dSb = torch.where(fin, rnd(dS, e_dS), 0.0)
        dSa = dS.abs() + e_dSb
        dk_e += e_dSb.transpose(2, 3) @ qa
        dk_a += dSa.transpose(2, 3) @ qa
        part = dSa @ ka
        dq_e[:, :, r0:r1] = sc * ((e_dSb @ ka) + (G2(AB_BN // 16 + 16) + gamma(n_k) * (1 + G2(AB_BN // 16 + 16))) * part)
    if not bounds:
        return dq, dk, dv
    g_acc = G2(4 * n_m + 16)
    res = []
    for val, err in ((dq, dq_e), (dk, sc * (dk_e + g_acc * dk_a)), (dv, dv_e + g_acc * dv_a)):
        err = err + 1.01 * U * (val.abs() + err)
        r = bf16_rn(val)
        res.append((r, allow_within(r, val - err, val + err)))
    return tuple(res)


def check_lse(got, lse64, allow, what=""):
    """lse is fp32: |got - lse64| within its allowance (fractional bf16 ulps of lse64), and exactly -inf where the row sees
    no key.  Returns the worst ulps."""
    from rowwise_ref import check_ulps
    got = got.to(F64).reshape(lse64.shape)
    dead = lse64 == -math.inf
    assert bool((got[dead] == -math.inf).all()), f"{what}: a row without keys has lse != -inf"
    _, worst, _ = check_ulps(got[~dead], lse64[~dead], allow[~dead], what)
    return worst


# ------------------------------------------------------------------------------------------------ input families
FAMILIES = ["random", "peaked", "probe", "needle", "late7.9", "late8.1", "wide", "lasttile"]
POISON = 1.0e4                   # finite poison for keys the kernels load and weigh by P = 0


def family_qkv(B, H, Tq, Tk, family, gen, device, needles=(), head0=0):
    """q [B, H, Tq, 128], k / v [B, H, Tk, 128] (fp32 holding bf16 values) of one input family:
      random: N(0, 1); peaked: q x 4; probe: q = 0, v = probe_values;
      needle: every q near one direction q0, keys N(0, 1) / 2, the keys in `needles` about 12 nats above the rest with
        values 3 + (d + i) mod 5 (needle i);
      late7.9 / late8.1: scores rising by 7.9 / 8.1 log2 units per 128-key tile, either side of the lazy raise;
      wide: scores falling linearly over 200 log2 units across the keys, so ex2 flushes the far end;
      lasttile: the row's weight all in its last key tile (scores 30 log2 units above the rest there)."""
    q = torch.randn(B, H, Tq, 128, generator=gen, device=device)
    k = torch.randn(B, H, Tk, 128, generator=gen, device=device)
    v = torch.randn(B, H, Tk, 128, generator=gen, device=device)
    if family == "random":
        pass
    elif family == "peaked":
        q = q * 4
    elif family == "probe":
        q.zero_()
        v = probe_values(B * H, Tk, head0, gen, device).view(B, H, Tk, 128).float()
    else:
        q0 = torch.randn(B, H, 1, 128, generator=gen, device=device)
        q = q0 + 0.02 * q
        q0 = q0.to(bf16).float()
        c = 128 ** -0.5 * LOG2E                   # the tests' scale
        unit = q0 / (c * (q0 * q0).sum(-1, keepdim=True))      # k = t unit scores t log2 units against q0
        t = torch.arange(Tk, device=device, dtype=torch.float32)[:, None]
        if family == "needle":
            k = k * 0.5
            for i, n in enumerate(needles):
                k[:, :, n] = (unit * (14.0 * LOG2E))[:, :, 0]
                v[:, :, n] = 3.0 + (torch.arange(128, device=device) + i) % 5
        else:
            if family.startswith("late"):
                target = float(family[4:]) * torch.div(t, AT_BN, rounding_mode="floor")
            elif family == "wide":
                target = -200.0 * t / max(Tk - 1, 1)
            else:
                target = torch.where(t >= (Tk - 1) // AT_BN * AT_BN, 30.0, 0.0)
            k = unit * target + 0.02 * k
    return q.to(bf16).float(), k.to(bf16).float(), v.to(bf16).float()
