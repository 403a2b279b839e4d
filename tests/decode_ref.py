"""fp64 reference for the split-KV decode attention kernels of aria_b200/csrc/attention.cu (decode_partial and its paged and
fp8 forms, attn_decode_multi_partial, attn_decode_prefix_partial, attn_decode_merge, attn_decode_merge_shared).

decode_ref takes, per (row, head), q [128], the keys and values the row may read [T, 128] and the row's live key set (a bool
[T]), and returns (ref, allow) with tests/rowwise_ref.py's meaning: ref = bf16_rn(o64), o64 = sum_i w_i v_i / sum_i w_i
with w_i = exp(scale q.k_i - max) over the live keys (0 for a row without one, which is what the merge stores, L > 0 ? A / L
: 0), and allow, in bf16 ulps of ref, is 0 wherever the kernel's worst-case fp32 error eta cannot carry its result across a
bf16 rounding boundary.  The live key set is what each entry defines: [0, len) minus masked keys; for the shared prefix,
prefix[0, P_g) minus the prefix mask, then tail[0, tail_len); for paged caches key SPLIT s + i is row i of page
block_table[r, s] (expand_paged).  fp8 keys and values are code x per-token scale, exact in fp64.

eta, from the kernels' arithmetic (U = 2^-24, gamma(n) = n U / (1 - n U), c = fl(fl(scale) fl(log2 e)), the fp32
scale_log2 the entries pass; s_i = c_ex q.k_i with c_ex = fl(scale) log2 e exactly, the score in log2 units):

  * Score.  The kernel forms fl(q_d c) (1 rounding) and each lane sums its 4 products q_d' k_d (at most 4 roundings on a
    term, with or without FMA contraction), then a 5-level xor butterfly (5); the fp8 path multiplies the reduced sum by the
    key scale (1).  c differs from c_ex by two roundings (log2 e to fp32, the product).  So |s_i' - s_i| <= D_i =
    gamma(13) c_ex sum_d |q_d k_id|.
  * Exponents.  A key's weight in the final sums is exp2f(s_i' - m_a) times the rescale factors exp2f(m_a - m_b) of the
    later maxima of its warp, exp2f(m_w - M) of the 4-warp merge and exp2f(M_s - M) of the split merge.  The arguments are
    all <= 0 and telescope to s_i' - M', so their fp32 subtractions add at most U |s_i' - M'| <= U (|s_i - s_max| + 2 D_max)
    to the exponent.  The common shift M' - s_max cancels in A / L, so every weight carries an exponent error of at most
    Delta = max_i (D_i + U |s_i - s_max|) + 2 U D_max, a relative error of 2^Delta - 1.  exp2f is within 2 ulps (CUDA C
    Programming Guide; build.py does not pass --use_fast_math), 4 U relative, and a key meets at most KW + 2 of them: its own,
    KW - 1 rescales in its warp (a warp holds keys k_begin + 4 warp + 16 i + u of a split, KW = SPLIT / 4 of them), the warp
    merge and the split merge.
  * Accumulation.  Each term of A picks up the rounding of pw v (fp8: pv = pw vs, then pv c, 2), then per later key of its
    warp the rounding of a f and of the add (2 each, 2 (KW - 1)), in the 4-warp merge 1 product and at most 4 adds, in the
    split merge 1 product and at most `splits` adds: at most 2 KW + 6 + splits (+1 fp8) roundings, gamma of that.  L is
    summed the same way with fewer.  FMA contraction only removes roundings.
  * With every term of A and L off by at most eps relative, eps = (2^Delta)(1 + 4 U)^(KW + 2)(1 + gamma(n_acc)) - 1,
    |A/L - o64| <= (sum w |v| eps + |o64| sum w eps) / (sum w (1 - eps)) <= 2 eps / (1 - eps) S, S = sum w |v_d| / sum w.
    Weights below 2^-126 of the largest lose the relative guarantees of exp2f and of the products (subnormals); the key
    at the maximum has weight exactly exp2f(0) = 1, so L >= 1 and those keys add at most n 2^-140 (1 + max |v|).  The
    division A / L adds U |A / L|.  eta is the sum; allow = allow_within(ref, o64 - eta, o64 + eta).

The exact probe (probe_values, probe_ref) needs no allowance: with q = 0 every score is exactly 0 and every weight exactly 1
(exp2f(0) = 1, exp2f(-inf) = 0), the sums of small integers (fp8: small integer codes times power-of-two scales) are exact
in fp32, so the kernel must store bf16(fl32(sum v / n)) bit for bit.

The builders take tensors on any device, so tests/test_decode_ref_host.py can show on the CPU that decode_ref accepts an
fp32 emulation of the kernels and rejects each planted mistake; tests/test_gpu_decode_fp64.py runs them on the device.
"""
import math
import os
import re

import torch

from rowwise_ref import F64, U, allow_within, bf16_rn, gamma

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "aria_b200", "csrc")
LOG2E = 1.0 / math.log(2.0)
bf16 = torch.bfloat16


def _constant(path, pattern):
    with open(os.path.join(CSRC, path)) as f:
        m = re.search(pattern, f.read())
    assert m, f"{pattern!r} not found in {path}"
    return int(m.group(1))


def kernel_constants():
    """The decode kernels' constants as attention.cu / common.cuh define them: the split size, the 4-warp teams per
    prefix / multi CTA, the page rows, and the largest Q attention_decode_multi accepts."""
    return dict(SPLIT=_constant("attention.cu", r"constexpr int DEC_SPLIT_KEYS = (\d+);"),
                SP_TEAMS=_constant("attention.cu", r"constexpr int SP_TEAMS = (\d+);"),
                PAGE_ROWS=_constant("common.cuh", r"constexpr int PAGE_ROWS = (\d+);"),
                MULTI_Q_MAX=_constant("attention.cu", r"Q > 0 && Q <= (\d+)"))


_C = kernel_constants()
SPLIT, SP_TEAMS, PAGE_ROWS, MULTI_Q_MAX = _C["SPLIT"], _C["SP_TEAMS"], _C["PAGE_ROWS"], _C["MULTI_Q_MAX"]
WARPS = 4                      # 128-thread CTA
STEP = 4 * WARPS               # keys per loop step of the 4 warps (warp w takes k0 + 4 w + u, u < 4)
KW = SPLIT // WARPS            # keys per warp per split

# Key counts where the kernels change shape: which warps hold keys (1..5, one step +-1, four steps +-1), the split seams,
# and long rows (700, 4097, 32768 and 65536 at SPLIT = 256).
WARP_LENS = [1, 2, 3, 4, 5, STEP - 1, STEP, STEP + 1, 4 * STEP - 1, 4 * STEP, 4 * STEP + 1]
SEAM_LENS = [SPLIT - 1, SPLIT, SPLIT + 1, 2 * SPLIT - 1, 2 * SPLIT, 2 * SPLIT + 1]
LONG_LENS = [700, 16 * SPLIT + 1, 128 * SPLIT, 256 * SPLIT]
# Queries per row of attention_decode_multi and rows per group of attention_decode_shared_prefix: one team, all teams,
# teams that serve two queries or rows.
MULTI_QS = [1, SP_TEAMS, SP_TEAMS + 1, MULTI_Q_MAX]
GROUP_NS = [1, SP_TEAMS, SP_TEAMS + 1, 4 * SP_TEAMS]


def f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def decode_ref(q, k, v, live, scale, k_scale=None, v_scale=None, splits=None):
    """q [N, 128]; k, v [N, T, 128] (bf16, or e4m3 codes with k_scale / v_scale [N, T]); live [N, T] bool.  Entries outside
    live are never used (they may be NaN).  splits: the most splits the kernel merges for a row (default ceil(T / SPLIT)).
    Returns (ref, allow), fp64 [N, 128]."""
    fp8 = k_scale is not None
    live = live.bool()
    lv = live[..., None]
    k64 = k.to(F64) if not fp8 else k.to(F64) * k_scale.to(F64)[..., None]
    v64 = v.to(F64) if not fp8 else v.to(F64) * v_scale.to(F64)[..., None]
    k64 = torch.where(lv, k64, 0.0)
    v64 = torch.where(lv, v64, 0.0)
    q64 = q.to(F64)
    c = f32(scale) * LOG2E
    s = c * torch.einsum("ntd,nd->nt", k64, q64)                        # log2 units
    s = s.masked_fill(~live, -math.inf)
    any_live = live.any(1)
    smax = torch.where(any_live, s.amax(1), 0.0)[:, None]
    w = torch.exp2(s - smax)                                            # 0 at dead keys
    L = w.sum(1).clamp_min(1.0)[:, None]                                # >= 1 on a live row (its maximum has weight 1)
    o = torch.einsum("nt,ntd->nd", w, v64) / L
    S = torch.einsum("nt,ntd->nd", w, v64.abs()) / L
    D = (gamma(13) * c * torch.einsum("ntd,nd->nt", k64.abs(), q64.abs())).masked_fill(~live, 0.0)
    d_max = D.amax(1, keepdim=True)
    delta = (D + U * (smax - s).masked_fill(~live, 0.0)).amax(1, keepdim=True) + 2 * U * d_max
    n_acc = 2 * KW + 6 + (splits if splits is not None else -(-k.shape[1] // SPLIT)) + (1 if fp8 else 0)
    eps = torch.exp2(delta) * (1 + 4 * U) ** (KW + 2) * (1 + gamma(n_acc)) - 1
    n = live.sum(1, keepdim=True).to(F64)
    tiny = n * 2.0 ** -140 * (1 + v64.abs().amax(1))
    eta = 2 * eps / (1 - eps) * S + tiny
    eta = eta + U * (o.abs() + eta)
    ref = bf16_rn(o)
    allow = allow_within(ref, o - eta, o + eta)
    dead = ~any_live[:, None]
    return torch.where(dead, 0.0, ref), torch.where(dead, 0.0, allow)


# ------------------------------------------------------------------------------------------------ layouts
def live_keys(lens, T, mask=None):
    """[B, T] bool: key t of row b is live when t < lens[b] and mask[b, t] (1 = masked out) is not set."""
    t = torch.arange(T, device=lens.device)
    live = t[None, :] < lens.to(torch.int64)[:, None]
    if mask is not None:
        live &= ~mask[:, :T].bool()
    return live


def expand_paged(pool, block_table, max_pages):
    """Page pool [n_pages, H, SPLIT, ...] and block_table [R, >= max_pages] -> [R, H, max_pages SPLIT, ...]: key SPLIT s + i
    of row r is row i of page block_table[r, s] (every entry must be a page of the pool)."""
    bt = block_table[:, :max_pages].long()
    x = pool[bt]                                                        # [R, max_pages, H, SPLIT, ...]
    x = x.transpose(1, 2)                                               # [R, H, max_pages, SPLIT, ...]
    return x.reshape(x.shape[0], x.shape[1], max_pages * SPLIT, *x.shape[4:])


def expand_shared_prefix(prefix, tail, n):
    """Prefix cache [G, H, P_max, ...] and tail caches [G n, H, N_max, ...] -> [G n, H, P_max + N_max, ...], row r holding
    the prefix of group r // n, then its own tail."""
    return torch.cat([prefix.repeat_interleave(n, 0), tail], 2)


def live_shared_prefix(prefix_lens, tail_lens, n, P_max, N_max, prefix_mask=None):
    """[G n, P_max + N_max] live keys of expand_shared_prefix's rows."""
    lp = live_keys(prefix_lens, P_max, prefix_mask).repeat_interleave(n, 0)
    return torch.cat([lp, live_keys(tail_lens, N_max)], 1)


# ------------------------------------------------------------------------------------------------ exact probe
def probe_values(live, rows=None, gen=None):
    """Small-integer values [N, T, 128] in [-16, 16] (exact in bf16 and e4m3) whose mean over the live keys shows their count
    and membership: column 0 is (-1)^rank over the live keys (rank in key order), so its sum is 0 or 1 and any key dropped,
    counted twice or added moves it; columns 1..17 are (-1)^bit b of the key index (b < 17); columns 18..22 the index mod 4,
    the index's nibbles 0..3 (residues mod 16, 256 (with nibble 1), 4096, 65536), column 23 the split index mod 16, column
    24 a constant per (row, head) (rows: its id, default 0..N-1); the rest random in [-8, 8]."""
    N, T = live.shape
    dev = live.device
    i = torch.arange(T, device=dev)
    v = torch.randint(-8, 9, (N, T, 128), generator=gen, device=dev).to(F64)
    rank = torch.cumsum(live.to(torch.int64), 1) - 1
    v[:, :, 0] = torch.where(rank % 2 == 0, 1.0, -1.0)
    for b in range(17):
        v[:, :, 1 + b] = torch.where((i >> b) & 1 == 1, -1.0, 1.0)
    v[:, :, 18] = (i % 4).to(F64)
    for j in range(4):
        v[:, :, 19 + j] = ((i >> (4 * j)) % 16).to(F64)
    v[:, :, 23] = ((i // SPLIT) % 16).to(F64)
    r = torch.arange(N, device=dev) if rows is None else rows.to(dev)
    v[:, :, 24] = ((r % 31) - 15).to(F64)[:, None]
    return v


def probe_ref(v, live, v_scale=None):
    """bf16(fl32(sum v / n)) over the live keys (v [N, T, 128] values, e4m3 codes with v_scale [N, T]); 0 on a row with no
    live key.  The sum is exact in fp32 (asserted), and the fp64 quotient of two fp32 integers-times-2^e rounds to the fp32
    quotient (a midpoint of fp32 values cannot lie within 2^-53 of such a quotient without equaling it)."""
    lv = live.bool()[..., None]
    x = v.to(F64) if v_scale is None else v.to(F64) * v_scale.to(F64)[..., None]
    x = torch.where(lv, x, 0.0)
    e = next((e for e in range(40) if bool(((x * 2.0 ** e).round() == x * 2.0 ** e).all())), None)
    assert e is not None, "probe values must be multiples of a power of two no finer than 2^-39"
    assert float(x.abs().sum(1).amax()) * 2.0 ** e < 2 ** 24, "probe sums must stay exact in fp32"
    n = live.bool().sum(1).to(F64)[:, None]
    o = torch.where(n > 0, x.sum(1) / n.clamp_min(1), 0.0)
    return o.float().to(bf16)
