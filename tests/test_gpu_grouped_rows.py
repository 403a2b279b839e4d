"""GPU: a grouped GEMM's stored rows depend on their own group's rows alone, bit for bit.

The grouped launches load of each A tile only the rows the group owns, rounded up to 16: a whole tile as one 128-row box, a
shorter one as 16-row boxes (csrc/gemm_common.cuh, tma_load_a_rows); and the second consumer warpgroup sits out tiles that end
in their first 64 rows.  The group sizes here take every path: 1, 15, 16 -> one 16-row box; 17 -> two; 63, 64 -> four, the
second warpgroup idle; 65, 72 -> five, both warpgroups; 127, 128 -> the whole box; 129, 200 -> a whole tile and a partial one;
0 -> no tile.  Groups start at unaligned rows.

The reference is one launch per group on a buffer that holds that group's rows alone, zero-padded to whole 128-row tiles: whatever
rows a launch loads there, none is foreign, so the reference does not depend on the load rule.  The packed buffers' rows that
belong to no group (the gaps between fixed-capacity regions, the rows behind the last group) hold NaN bit patterns, so a foreign
or stale row that leaked into a stored value fails the comparison.

These tests pass with whole 128-row A boxes too.  That is their point: cutting the loads to the group's rows changes no stored
value.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16 = torch.bfloat16
COUNTS = [0, 1, 15, 16, 17, 63, 64, 65, 72, 127, 128, 129, 200]
TAIL = 37          # NaN rows behind the last group


def _offsets(counts):
    off = torch.zeros(len(counts) + 1, dtype=torch.int32)
    off[1:] = torch.tensor(counts).cumsum(0)
    return off


def _alone(rows_of_group, fill=0):
    """The group's rows at the top of a buffer of whole 128-row tiles, the rest `fill`; and its [0, n] offsets."""
    n = rows_of_group.shape[0]
    buf = torch.full(((n + 127) // 128 * 128, *rows_of_group.shape[1:]), fill, dtype=torch.float32, device=DEV).to(rows_of_group.dtype)
    buf[:n] = rows_of_group
    return buf, torch.tensor([0, n], dtype=torch.int32, device=DEV)


def _packed(rows, K, seed):
    """[rows + TAIL, K] bf16 with NaN behind row `rows`; the launches get the first `rows` rows as a view."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    full = torch.full((rows + TAIL, K), float("nan"), dtype=BF16, device=DEV)
    full[:rows] = torch.randn(rows, K, generator=g, device=DEV).to(BF16)
    return full[:rows]


def _weights(E, K, N, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(E, K, N, generator=g, device=DEV) * K ** -0.5).to(BF16)


def _check_groups(got, counts, starts, per_group):
    """got[rows of group e] == per_group(e, lo, hi) for every non-empty group; no NaN anywhere in the groups' rows."""
    seen = 0
    for e, n in enumerate(counts):
        if n == 0:
            continue
        lo = int(starts[e])
        want = per_group(e, lo, lo + n)
        assert want.shape[0] >= n and not torch.isnan(want[:n].float()).any()
        assert torch.equal(got[lo:lo + n], want[:n]), f"group {e} ({n} rows at row {lo})"
        seen += n
    assert seen == sum(counts)


@pytest.mark.parametrize("swiglu", [False, True])
def test_bf16_grouped_equals_one_launch_per_group(swiglu):
    from aria_b200 import ops
    K, N = 256, 192
    rows, off = sum(COUNTS), _offsets(COUNTS)
    a = _packed(rows, K, 1)
    w = _weights(len(COUNTS), K, 2 * N if swiglu else N, 2)
    got = ops.grouped_gemm(a, w, off.to(DEV), swiglu=swiglu)

    def one(e, lo, hi):
        buf, o = _alone(a[lo:hi])
        return ops.grouped_gemm(buf, w[e:e + 1].contiguous(), o, swiglu=swiglu)
    _check_groups(got, COUNTS, off, one)


def test_bf16_transposed_weights_equal_one_launch_per_group():
    """The data-gradient form (weights [E, N, K] read in place)."""
    from aria_b200 import ops
    K, N = 192, 256
    rows, off = sum(COUNTS), _offsets(COUNTS)
    a = _packed(rows, K, 3)
    w = _weights(len(COUNTS), N, K, 4)
    got = ops.grouped_gemm_nt(a, w, off.to(DEV))

    def one(e, lo, hi):
        buf, o = _alone(a[lo:hi])
        return ops.grouped_gemm_nt(buf, w[e:e + 1].contiguous(), o)
    _check_groups(got, COUNTS, off, one)


@pytest.mark.parametrize("swiglu", [False, True])
def test_w8a16_grouped_equals_one_launch_per_group(swiglu):
    from aria_b200 import ops
    K, N = 256, 192
    rows, off = sum(COUNTS), _offsets(COUNTS)
    a = _packed(rows, K, 5)
    q, s = ops.quantize_fp8_cols(_weights(len(COUNTS), K, 2 * N if swiglu else N, 6))
    got = ops.grouped_gemm_fp8(a, q, s, off.to(DEV), swiglu=swiglu)

    def one(e, lo, hi):
        buf, o = _alone(a[lo:hi])
        return ops.grouped_gemm_fp8(buf, q[e:e + 1].contiguous(), s[e:e + 1].contiguous(), o, swiglu=swiglu)
    _check_groups(got, COUNTS, off, one)


@pytest.mark.parametrize("swiglu", [False, True])
def test_w8a8_grouped_equals_one_launch_per_group(swiglu):
    from aria_b200 import ops
    K, N = 256, 192
    rows, off = sum(COUNTS), _offsets(COUNTS)
    g = torch.Generator(device=DEV).manual_seed(7)
    aq_rows, as_rows = ops.permute_quantize_fp8(torch.randn(rows, K, generator=g, device=DEV).to(BF16))
    # e4m3 rows with 0x7F (NaN) behind the last group, NaN scales behind the last scale
    aq_full = torch.full((rows + TAIL, K), 0x7F, dtype=torch.uint8, device=DEV)
    aq_full[:rows] = aq_rows.view(torch.uint8)
    aq = aq_full.view(torch.float8_e4m3fn)[:rows]
    as_full = torch.full((rows + TAIL,), float("nan"), dtype=torch.float32, device=DEV)
    as_full[:rows] = as_rows
    a_scale = as_full[:rows]
    q, s = ops.quantize_fp8_cols(_weights(len(COUNTS), K, 2 * N if swiglu else N, 8))
    kq = q.transpose(1, 2).contiguous().transpose(1, 2)      # K-major storage of the same codes
    got = ops.grouped_gemm_w8a8(aq, a_scale, kq, s, off.to(DEV), swiglu=swiglu)

    def one(e, lo, hi):
        buf, o = _alone(aq[lo:hi].view(torch.uint8))
        sc = torch.ones(buf.shape[0], dtype=torch.float32, device=DEV)
        sc[:hi - lo] = a_scale[lo:hi]
        return ops.grouped_gemm_w8a8(buf.view(torch.float8_e4m3fn), sc, kq[e:e + 1], s[e:e + 1].contiguous(), o, swiglu=swiglu)
    _check_groups(got, COUNTS, off, one)


@pytest.mark.parametrize("swiglu", [False, True])
def test_regions_with_gaps_equal_one_launch_per_group(swiglu):
    """Fixed-capacity regions (group_counts): groups at unaligned starts with NaN rows between and behind them."""
    from aria_b200 import ops
    K, N = 256, 192
    gaps = [3, 0, 16, 1, 40, 7, 0, 130, 5, 64, 2, 9, 11]
    starts, r = [], 0
    for n, gap in zip(COUNTS, gaps):
        r += gap
        starts.append(r)
        r += n
    cap = r + TAIL
    g = torch.Generator(device=DEV).manual_seed(9)
    a = torch.full((cap, K), float("nan"), dtype=BF16, device=DEV)
    for st, n in zip(starts, COUNTS):
        a[st:st + n] = torch.randn(n, K, generator=g, device=DEV).to(BF16)
    w = _weights(len(COUNTS), K, 2 * N if swiglu else N, 10)
    st_d = torch.tensor(starts, dtype=torch.int32, device=DEV)
    ct_d = torch.tensor(COUNTS, dtype=torch.int32, device=DEV)
    out = torch.zeros(cap, N, dtype=BF16, device=DEV)
    ops.grouped_gemm_regions(a, w, st_d, ct_d, sum(COUNTS), swiglu=swiglu, out=out)

    def one(e, lo, hi):
        buf, o = _alone(a[lo:hi])
        return ops.grouped_gemm(buf, w[e:e + 1].contiguous(), o, swiglu=swiglu)
    _check_groups(out, COUNTS, starts, one)
    # rows of no group are not written
    owned = torch.zeros(cap, dtype=torch.bool, device=DEV)
    for st, n in zip(starts, COUNTS):
        owned[st:st + n] = True
    assert not out[~owned].any()
