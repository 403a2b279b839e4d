"""GPU parity tests proper: the CUDA path, called through the C ABI (aria_b200.ops / the module mirrors),
against the oracle (oracle/aria_oracle.py, CPU) on the same seeded inputs and against the golden fixtures
captured from the unmodified reference (tests/golden/).

Tolerances (stated per BASELINE.json north_star: "logits matching the reference within 1e-2 relative"):
  * integer / index work (top-k ids on given logits, counts, offsets, permutation, row gathers): bit-exact
  * single ops on bf16 tensors: ||got - want||_inf <= REL * ||want||_inf with REL = 1e-2 — about one bf16 ulp
    (2^-8 = 3.9e-3 relative) of the largest element plus fp32 accumulation-order noise.
  * whole-model logits (bf16, many layers deep): relative L2 error ||got - want||_2 / ||want||_2 <= 1e-2 per tensor,
    and element-wise |got - want| <= 2e-2 * max|want| (= 2 bf16 ulps in the top binade; one ulp alone is 0.78 %),
    evaluated on the tokens whose router top-k is not a bf16 near-tie (see assert_logits_close).
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

GOLD = os.path.join(os.path.dirname(__file__), "golden")
REL = 1e-2
DEV = "cuda"


def _ops():
    from aria_b200 import ops
    return ops


def rel_inf(got, want):
    got, want = got.float().cpu(), want.float().cpu()
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-12))


def _oracle():
    from oracle import aria_oracle as O
    from oracle import configs as C
    return O, C


TIE_MARGIN = 2 ** -6   # k-th vs (k+1)-th router logit within 4 bf16 ulps of the row max: routing may legitimately flip


def assert_logits_close(got, want, router_logits, k, rel=REL, max_tie_frac=0.25):
    """Per-token check.  Tokens whose top-k boundary is NOT a near-tie in any layer must match within `rel`;
    near-tie tokens (different-but-valid expert choice, SURVEY.md §7 "top-k parity") must stay finite and within
    the logit scale, and there must be few of them."""
    O, _ = _oracle()
    got, want = got.float().cpu(), want.float().cpu()
    B, T, V = want.shape
    margin = O.topk_margin(router_logits, k).view(B, -1)[:, -T:]
    scale = want.abs().max()
    err = (got - want).abs().amax(-1)
    safe = margin > TIE_MARGIN
    assert float((~safe).float().mean()) <= max_tie_frac, "too many near-tie tokens for a meaningful check"
    assert torch.isfinite(got).all()
    d = (got - want)[safe]
    rel_l2 = float(d.norm() / want[safe].norm().clamp_min(1e-12))
    assert rel_l2 <= rel, rel_l2
    assert float(err[safe].max()) <= 2 * rel * float(scale), (float(err[safe].max()), float(scale))
    assert float(err.max()) <= 0.5 * float(scale)


# ------------------------------------------------------------------------------------------------ MoE pieces
@pytest.mark.parametrize("T,E,k", [(1, 8, 2), (37, 8, 2), (768, 64, 6), (4099, 64, 6), (5, 64, 8)])
def test_routing_bit_exact(T, E, k):
    """torch.topk + softmax + histc (moe_lm.py:261-269) on given bf16 logits: ids, counts, scores bit-exact."""
    O, _ = _oracle()
    g = torch.Generator().manual_seed(T * 7 + E)
    logits = torch.randn(T, E, generator=g).bfloat16()
    logits[0, :] = 0.5  # a row that is ALL ties: lowest expert ids must win
    s_ref, i_ref, c_ref = O.router_routing(logits, k)
    s, i, c = _ops().route_from_logits(logits.to(DEV), k)
    assert torch.equal(i.cpu().long(), i_ref)
    assert torch.equal(c.cpu().long(), c_ref)
    assert torch.equal(s.cpu(), s_ref)
    assert int(c.sum()) == T * k


_PERM_SHAPES = [(1, 8, 2, 256), (37, 8, 2, 256), (768, 64, 6, 2560), (3001, 64, 6, 512), (5461, 64, 6, 256), (5600, 64, 6, 256)]  # last: > 32768 ids -> the multi-block sort


@pytest.mark.parametrize("T,E,k,d,row_align",
                         [pytest.param(*s, a, id="-".join(map(str, s)) + ("" if a == 1 else f"-align{a}"))
                          for a in (1, 16) for s in _PERM_SHAPES])
def test_permutation_and_combine_bit_exact(T, E, k, d, row_align):
    """stable argsort / index_select / index_copy_ / weighted sum (moe_lm.py:313-365).  row_align=16 is the training
    layout: expert e's block starts at the sum of the earlier counts each rounded up to 16, its rows are the oracle's
    stable order shifted by that base, every other slot of `src` is -1 and its permuted row is exactly zero."""
    O, _ = _oracle()
    ops = _ops()
    g = torch.Generator().manual_seed(T + d)
    logits = torch.randn(T, E, generator=g).bfloat16()
    if E >= 16:
        logits[:, 3] = -100.0  # an expert that receives no tokens (empty group)
    x = torch.randn(T, d, generator=g).bfloat16()
    s_ref, i_ref, c_ref = O.router_routing(logits, k)
    perm_ref, order = O.token_permutation(x, i_ref, k)
    s, i, c = ops.route_from_logits(logits.to(DEV), k)
    off, dest, src = ops.build_permutation(i, c, row_align=row_align)
    inv = torch.empty_like(order)
    inv[order] = torch.arange(order.numel())
    # expert e's rows: dense base (sum of earlier counts) -> aligned base (sum of earlier counts rounded up to row_align)
    dense0 = torch.cat([torch.zeros(1, dtype=torch.long), c_ref.cumsum(0)])
    al0 = torch.cat([torch.zeros(1, dtype=torch.long), ((c_ref + row_align - 1) // row_align * row_align).cumsum(0)])
    eid_flat = i_ref.reshape(-1)
    dest_ref = inv - dense0[eid_flat] + al0[eid_flat]
    assert torch.equal(off.cpu().long(), al0)
    assert torch.equal(dest.cpu().long(), dest_ref)
    rows = src.numel()
    assert rows == T * k + E * (row_align - 1)
    src_ref = torch.full((rows,), -1, dtype=torch.long)
    src_ref[dest_ref] = torch.arange(T * k) // k
    assert torch.equal(src.cpu().long(), src_ref)
    p = ops.permute_rows(x.to(DEV), src)
    p_ref = torch.zeros(rows, d, dtype=torch.bfloat16)
    p_ref[dest_ref[order]] = perm_ref
    assert torch.equal(p.cpu(), p_ref)
    # sortedness property: expert id of each permuted row is non-decreasing
    eid = i.reshape(-1)[torch.argsort(dest)].cpu()
    assert bool((eid[1:] >= eid[:-1]).all())
    y = torch.randn(rows, d, generator=g).bfloat16()
    y[src_ref < 0] = float("nan")  # pad rows are never read
    shared = torch.randn(T, d, generator=g).bfloat16()
    want = O.token_unpermutation(y[dest_ref[order]], order, s_ref, k) + shared
    got = ops.unpermute_combine(y.to(DEV), dest, s, shared.to(DEV))
    assert (got.cpu().float() - want.float()).abs().max() <= 2 ** -7 * want.float().abs().max()
    assert float((got.cpu() == want).float().mean()) > 0.999


def test_permute_unpermute_round_trip_full_size():
    """Size-independent property at the real width (T=8192, E=64, k=6, d=2560): with unit scores and k copies of
    the same row, combine(permute(x)) == k * x exactly (bf16 holds k*x for k=6 only approximately -> use k=1 ids
    replicated: every slot of a token returns the token itself)."""
    ops = _ops()
    T, E, k, d = 8192, 64, 6, 2560
    g = torch.Generator(device=DEV).manual_seed(0)
    x = torch.randn(T, d, generator=g, device=DEV).bfloat16()
    logits = torch.randn(T, E, generator=g, device=DEV).bfloat16()
    s, i, c = ops.route_from_logits(logits, k)
    off, dest, src = ops.build_permutation(i, c)
    p = ops.permute_rows(x, src)
    # every sorted row is the row of its source token
    assert torch.equal(p, x[src.long()])
    assert torch.equal(torch.sort(dest).values, torch.arange(T * k, device=DEV, dtype=torch.int32))
    one_hot = torch.zeros(T, k, device=DEV, dtype=torch.bfloat16)
    one_hot[:, 2] = 1.0
    back = ops.unpermute_combine(p, dest, one_hot, None)
    assert torch.equal(back, x)


@pytest.mark.parametrize("counts,K,N", [([128], 64, 64), ([5, 0, 300, 77], 256, 256), ([1] * 8, 128, 192),
                                         ([0, 0, 0, 513], 192, 128)])
def test_grouped_gemm_vs_oracle(counts, K, N):
    """experts_gemm == reference sequential_gemm (moe_lm.py:398-428), ragged + empty groups."""
    O, _ = _oracle()
    from aria_b200 import moe_lm
    g = torch.Generator().manual_seed(sum(counts) + K)
    rows, E = sum(counts), len(counts)
    a = torch.randn(rows, K, generator=g).bfloat16()
    w = (torch.randn(E, K, N, generator=g) * 0.05).bfloat16()
    want = O.sequential_gemm(a, w, torch.tensor(counts))
    # reference contract: tokens_per_expert as an int64 CPU tensor (moe_lm.py:478)
    got = moe_lm.experts_gemm(a.to(DEV), w.to(DEV), torch.tensor(counts, dtype=torch.int64))
    assert rel_inf(got, want) <= REL
    got2 = moe_lm.gmm(a.to(DEV), w.to(DEV), torch.tensor(counts, dtype=torch.int64, device=DEV))
    assert torch.equal(got, got2)


def test_grouped_gemm_linearity_full_width():
    """Full-size property (E=64, K=2560, N=3328, ~72 rows/expert as in BASELINE cfg 2): linear in A, and every
    expert's block matches a dense GEMM with that expert's weight."""
    ops = _ops()
    E, K, N = 64, 2560, 3328
    g = torch.Generator(device=DEV).manual_seed(1)
    counts = torch.randint(40, 110, (E,), generator=torch.Generator().manual_seed(3))
    rows = int(counts.sum())
    off = torch.cat([torch.zeros(1, dtype=torch.long), counts.cumsum(0)]).to(torch.int32).to(DEV)
    a = torch.randn(rows, K, generator=g, device=DEV).bfloat16()
    w = (torch.randn(E, K, N, generator=g, device=DEV) * 0.02).bfloat16()
    y = ops.grouped_gemm(a, w, off)
    y2 = ops.grouped_gemm((a.float() * 2).bfloat16(), w, off)
    assert torch.equal(y2.float(), y.float() * 2)  # scaling by 2 is exact in bf16
    for e in (0, 17, 63):
        lo, hi = int(off[e]), int(off[e + 1])
        dense = ops.linear(a[lo:hi].contiguous(), w[e].t().contiguous())
        assert rel_inf(y[lo:hi], dense) <= REL


@pytest.mark.parametrize("W,E_loc,d,I,counts_hi", [(2, 4, 256, 128, 60), (2, 8, 512, 256, 300), (4, 4, 256, 128, 140)])
def test_expert_parallel_region_gemms_pair_mode(W, E_loc, d, I, counts_hi):
    """Fixed-capacity regions ordered (expert, source rank) (neighbouring regions share an expert's weights) and the same regions
    addressed in (source rank, expert) order.  Same rows, same weights, same accumulation order per row: the outputs must be
    bit-identical - fc1 + SwiGLU and fc2 (LINEAR) - and match the oracle."""
    from aria_b200 import ops
    from oracle import aria_oracle as O
    dev = "cuda"
    g = torch.Generator().manual_seed(11)
    G, cap = W * E_loc, (counts_hi + 15) // 16 * 16 + 16
    counts = torch.randint(0, counts_hi + 1, (G,), generator=g).to(torch.int32)
    counts[1] = 0                       # an empty region next to a populated one
    counts[2] = counts_hi               # more than 128 rows where counts_hi allows: a second m-tile for one CTA of the pair only
    starts = torch.arange(G, dtype=torch.int32) * cap
    a = torch.randn(G * cap, d, generator=g).bfloat16()
    w1 = (torch.randn(E_loc, d, 2 * I, generator=g) * 0.05).bfloat16()
    w2 = (torch.randn(E_loc, I, 256, generator=g) * 0.05).bfloat16()
    # region index (expert-major) el * W + s  <->  (source-major) s * E_loc + el: same memory, other enumeration
    perm = torch.tensor([(j % E_loc) * W + j // E_loc for j in range(G)])
    ad, w1d, w2d = a.to(dev), w1.to(dev), w2.to(dev)
    outs = []
    for order in ("expert_major", "source_major"):
        st = (starts if order == "expert_major" else starts[perm]).to(dev).contiguous()
        ct = (counts if order == "expert_major" else counts[perm]).to(dev).contiguous()
        gm = -W if order == "expert_major" else E_loc
        h = torch.zeros(G * cap, I, dtype=torch.bfloat16, device=dev)
        ops.grouped_gemm_regions(ad, w1d, st, ct, int(counts.sum()), swiglu=True, group_mod=gm, out=h)
        y = torch.zeros(G * cap, 256, dtype=torch.bfloat16, device=dev)
        ops.grouped_gemm_regions(h, w2d, st, ct, int(counts.sum()), group_mod=gm, out=y)
        outs.append((h.cpu(), y.cpu()))
    torch.cuda.synchronize()
    for gi in range(G):
        r0, n = int(starts[gi]), int(counts[gi])
        if n == 0:
            continue
        el = gi // W
        for t in range(2):
            assert torch.equal(outs[0][t][r0:r0 + n], outs[1][t][r0:r0 + n]), (gi, t)
        want_h = O.glu(a[r0:r0 + n] @ w1[el])
        got_h = outs[0][0][r0:r0 + n].float()
        assert (got_h - want_h.float()).abs().max() <= 1e-2 * max(1.0, float(want_h.float().abs().max())), gi
        want_y = (outs[0][0][r0:r0 + n] @ w2[el]).float()
        assert (outs[0][1][r0:r0 + n].float() - want_y).abs().max() <= 1e-2 * max(1.0, float(want_y.abs().max())), gi


@pytest.mark.parametrize("dtype_tag", ["bf16"])
def test_moe_layer_cfg1_golden(dtype_tag):
    """BASELINE.json configs[0] (d=256, 8 experts, top-2, I=512) against the reference's own outputs."""
    O, C = _oracle()
    from aria_b200 import moe_lm
    gold = torch.load(os.path.join(GOLD, f"moe_layer_cfg1_{dtype_tag}.pt"), weights_only=False)
    gen = torch.Generator().manual_seed(gold["seed"])
    sd = {k: v.bfloat16() for k, v in C.moe_layer_state(C.TINY["text_config"], gen).items()}
    cfg = moe_lm.AriaMoELMConfig(**C.TINY["text_config"])
    layer = moe_lm.MoELayer(cfg, device=DEV)
    layer.load_state_dict({k: v.to(DEV) for k, v in sd.items()}, strict=True)
    x = gold["x"].to(DEV)
    # intermediates
    scores, idx, counts = layer.router(x)
    assert torch.equal(idx.cpu().long().sort(1).values, gold["top_idx"].sort(1).values)
    assert torch.equal(counts.cpu().long(), gold["counts"].long())
    perm = layer.token_dispatcher.token_permutation(x, idx, counts)
    assert torch.equal(perm.cpu(), gold["permuted"])
    eo = layer.experts(perm, layer.token_dispatcher.expert_offsets)
    assert rel_inf(eo, gold["expert_out"]) <= REL
    assert rel_inf(layer.shared_experts(x), gold["shared"]) <= REL
    out = layer(x)
    assert rel_inf(out, gold["out"]) <= REL
    # and against the oracle restatement on the same inputs
    assert rel_inf(out, O.moe_layer(gold["x"], sd, 2)) <= REL


def test_moe_layer_edge_cases():
    """T=1 (decode-like, most experts empty) and a ragged batch, vs the oracle."""
    O, C = _oracle()
    from aria_b200 import moe_lm
    tc = dict(hidden_size=256, moe_num_experts=64, moe_topk=6, moe_intermediate_size=128, moe_num_shared_experts=2)
    gen = torch.Generator().manual_seed(11)
    sd = {k: v.bfloat16() for k, v in C.moe_layer_state(tc, gen).items()}
    layer = moe_lm.MoELayer(moe_lm.AriaMoELMConfig(**tc), device=DEV)
    layer.load_state_dict({k: v.to(DEV) for k, v in sd.items()}, strict=True)
    for T in (1, 3, 130):
        x = torch.randn(1, T, 256, generator=gen).bfloat16()
        want, parts = O.moe_layer(x, sd, 6, return_parts=True)
        got = layer(x.to(DEV))
        # rows whose top-k boundary is a near-tie in bf16 logits may legitimately pick another expert
        lg = parts["logits"].float().sort(1, descending=True).values
        safe = (lg[:, 5] - lg[:, 6]) > 2 ** -6 * lg.abs().max()
        err = (got.cpu().float() - want.float()).abs().amax(-1).view(-1)
        assert float(err[safe].max() if safe.any() else 0.0) <= REL * float(want.float().abs().max())


# ------------------------------------------------------------------------------------------------ dense pieces
@pytest.mark.parametrize("M,N,K", [(1, 64, 64), (130, 264, 200), (768, 2560, 2560), (300, 4304, 1152)])
def test_linear_epilogues_vs_torch_fp32(M, N, K):
    """GEMM + bias + gelu_tanh + residual with the reference's op-by-op bf16 rounding (torch CPU restatement)."""
    import torch.nn.functional as F
    from aria_b200 import _lib as L
    ops = _ops()
    g = torch.Generator().manual_seed(M + N)
    x = torch.randn(M, K, generator=g).bfloat16()
    w = (torch.randn(N, K, generator=g) * 0.05).bfloat16()
    b = torch.randn(N, generator=g).bfloat16()
    r = torch.randn(M, N, generator=g).bfloat16()
    want = F.gelu(F.linear(x, w, b), approximate="tanh") + r
    got = ops.linear(x.to(DEV), w.to(DEV), b.to(DEV), act=L.ACT_GELU_TANH, residual=r.to(DEV))
    assert rel_inf(got, want) <= REL
    from oracle import aria_oracle as O
    want = O.gelu_new(F.linear(x, w))
    got = ops.linear(x.to(DEV), w.to(DEV), act=L.ACT_GELU_NEW)
    assert rel_inf(got, want) <= REL


def test_norms_vs_oracle():
    import torch.nn.functional as F
    O, _ = _oracle()
    ops = _ops()
    g = torch.Generator().manual_seed(5)
    for d in (144, 256, 1152, 2560):
        x = torch.randn(33, d, generator=g).bfloat16()
        r = torch.randn(33, d, generator=g).bfloat16()
        w = (1 + 0.1 * torch.randn(d, generator=g)).bfloat16()
        b = (0.1 * torch.randn(d, generator=g)).bfloat16()
        assert rel_inf(ops.rmsnorm(x.to(DEV), w.to(DEV), 1e-5), O.rms_norm(x, w, 1e-5)) <= 2 ** -7
        y, s = ops.rmsnorm(x.to(DEV), w.to(DEV), 1e-5, residual=r.to(DEV))
        assert torch.equal(s.cpu(), x + r)
        assert rel_inf(y, O.rms_norm(x + r, w, 1e-5)) <= 2 ** -7
        assert rel_inf(ops.layernorm(x.to(DEV), w.to(DEV), b.to(DEV), 1e-6), F.layer_norm(x, (d,), w, b, 1e-6)) <= 2 ** -7


@pytest.mark.parametrize("B,H,Tq,Tk,causal,masked,hd", [
    (1, 1, 1, 1, True, False, 128), (1, 2, 128, 128, True, False, 128), (2, 3, 300, 300, True, False, 128),
    (1, 2, 100, 420, True, False, 128), (2, 2, 200, 333, False, True, 72), (1, 2, 16, 16, False, False, 72),
    (1, 4, 1030, 1030, True, False, 128)])
def test_attention_vs_oracle(B, H, Tq, Tk, causal, masked, hd):
    """softmax(q k^T s + mask) v against the oracle's eager attention (transformers eager_attention_forward)."""
    O, _ = _oracle()
    ops = _ops()
    g = torch.Generator().manual_seed(Tq * 3 + Tk)
    q = torch.randn(B, H, Tq, 128, generator=g).bfloat16()
    k = torch.randn(B, H, Tk, 128, generator=g).bfloat16()
    v = torch.randn(B, H, Tk, 128, generator=g).bfloat16()
    for t in (q, k, v):
        t[..., hd:] = 0
    add = None
    km = None
    if causal:
        add = O.causal_additive_mask(Tq, Tk, torch.bfloat16)
    if masked:
        km = (torch.rand(B, Tk, generator=g) < 0.3)
        km[:, 0] = False
        add = torch.zeros(B, 1, 1, Tk, dtype=torch.bfloat16).masked_fill_(km[:, None, None, :], float("-inf"))
    want = O.attention_core(q, k, v, hd ** -0.5, add)[..., :hd].reshape(B, Tq, H * hd)
    got = ops.attention(q.to(DEV), k.to(DEV), v.to(DEV), Tq, Tk, hd ** -0.5, causal, out_hd=hd,
                        key_mask=None if km is None else km.to(torch.uint8).to(DEV))
    assert rel_inf(got, want) <= REL


def test_decode_attention_matches_prefill_kernel():
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(2)
    B, H, Tk = 4, 20, 777
    q = torch.randn(B, H, 1, 128, generator=g, device=DEV).bfloat16()
    k = torch.randn(B, H, Tk, 128, generator=g, device=DEV).bfloat16()
    v = torch.randn(B, H, Tk, 128, generator=g, device=DEV).bfloat16()
    a = ops.attention(q, k, v, 1, Tk, 128 ** -0.5, True)
    b = ops.attention_decode(q[:, :, 0].contiguous(), k, v, Tk, 128 ** -0.5)
    assert rel_inf(b.view(B, 1, -1), a) <= REL


# ------------------------------------------------------------------------------------------------ whole model
def _tiny_model(dtype=torch.bfloat16, seed=0):
    _, C = _oracle()
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    sd = C.aria_state(C.TINY, seed=seed, dtype=dtype)
    m = AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device=DEV)
    m.load_state_dict({k: v.to(DEV) for k, v in sd.items()}, strict=True)
    return m, sd


@pytest.mark.parametrize("masked", ["full", "masked"])
def test_aria_tiny_forward_golden(masked):
    """ViT -> projector -> merge -> MoE LM: logits against the UNMODIFIED reference's (golden fixture)."""
    gold = torch.load(os.path.join(GOLD, f"aria_tiny_bf16_{masked}.pt"), weights_only=False)
    m, _ = _tiny_model()
    pm = gold["pixel_mask"]
    vit, img_mask = m.vision_tower(gold["pixel_values"].to(DEV), None if pm is None else pm.to(DEV))
    assert rel_inf(vit, gold["vit"]) <= REL
    if pm is not None:
        assert torch.equal(img_mask.cpu(), gold["image_attn_mask"])
    proj = m.multi_modal_projector(vit, img_mask)
    assert rel_inf(proj, gold["projector"]) <= REL
    # host inputs (the e2e call path): pinned host ids / pixels / mask
    out = m(gold["input_ids"], gold["pixel_values"], pm)
    assert out.logits.shape == gold["logits"].shape
    O, C = _oracle()
    rl = []
    want, _ = O.aria_forward(gold["input_ids"], gold["pixel_values"], pm, C.aria_state(C.TINY, seed=0, dtype=torch.bfloat16),
                             C.TINY, router_logits=rl)
    # the oracle supplies the router logits for the tie check; its bit-exact agreement with the golden logits is a property of the
    # CPU it runs on and is asserted by tests/test_oracle_golden.py::test_aria_tiny_forward on the CPU test machine
    assert rel_inf(want, gold["logits"]) <= REL
    assert_logits_close(out.logits, gold["logits"], rl, C.TINY["text_config"]["moe_topk"])


def test_image_token_mismatch_raises():
    gold = torch.load(os.path.join(GOLD, "aria_tiny_bf16_full.pt"), weights_only=False)
    m, _ = _tiny_model()
    ids = gold["input_ids"].clone()
    ids[0, 5] = 11
    with pytest.raises(ValueError):
        m(ids, gold["pixel_values"], None)


def test_generate_decode_consistent_with_prefill():
    """KV-cache decode: logits of step t from the cache == logits of a fresh prefill of the longer prompt."""
    O, C = _oracle()
    m, sd = _tiny_model(seed=3)
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(10, 512, (2, 21), generator=g)
    full = m(ids.to(DEV)).logits
    part = m(ids[:, :-1].to(DEV), max_cache_len=32)
    step = m(ids[:, -1:].to(DEV), past_key_values=part.past_key_values).logits
    # and the oracle agrees with both the prefill and the cached decode step
    import torch.nn.functional as F
    emb = F.embedding(ids, sd["language_model.model.embed_tokens.weight"])
    rl = []
    want, _ = O.lm_forward(emb, sd, C.TINY["text_config"], router_logits=rl)
    k = C.TINY["text_config"]["moe_topk"]
    assert_logits_close(full, want, rl, k)
    rl_last = [x.view(2, 21, -1)[:, -1:].reshape(2, -1) for x in rl]
    assert_logits_close(step, want[:, -1:], rl_last, k, max_tie_frac=0.5)
    toks = m.generate(ids[:1].to(DEV), max_new_tokens=4)
    assert toks.shape == (1, 25)


def test_graphed_prefill_equals_eager():
    """CUDA-graph replay of the prefill (bench.py's throughput path) is bit-identical to the eager forward, also
    after new inputs are copied into its static buffers; the image-token check still raises."""
    from aria_b200.modeling_aria import GraphedPrefill
    gold = torch.load(os.path.join(GOLD, "aria_tiny_bf16_full.pt"), weights_only=False)
    m, _ = _tiny_model()
    ids, pv = gold["input_ids"], gold["pixel_values"]
    eager = m(ids, pv, None, num_logits_to_keep=1).logits.clone()
    g = GraphedPrefill(m, ids, pv, num_logits_to_keep=1)
    assert torch.equal(g.replay(), eager)
    ids2 = ids.clone()
    ids2[0, -3:] = torch.tensor([17, 33, 65])
    pv2 = (pv.float() * 0.5).bfloat16()
    want = m(ids2, pv2, None, num_logits_to_keep=1).logits.clone()
    assert torch.equal(g(ids2.pin_memory(), pv2.pin_memory()), want)
    bad = ids.clone()
    bad[0, 5] = 11
    with pytest.raises(ValueError):
        g(bad, pv)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_one_process_two_devices():
    """The reference can span GPUs inside ONE process (`device_map="auto"`, aria/inference.py:55-57; hence the
    `torch.cuda.set_device(input.device)` at moe_lm.py:483).  Every C-ABI call must honour the tensor's device: the
    dynamic-shared-memory opt-ins and the SM count are per-device state inside the library."""
    from aria_b200 import ops
    g = torch.Generator().manual_seed(0)
    x = torch.randn(300, 512, generator=g).bfloat16()
    w = (torch.randn(384, 512, generator=g) * 0.05).bfloat16()
    q = torch.randn(1, 2, 200, 128, generator=g).bfloat16()
    ref = x.float() @ w.float().t()
    outs = []
    for dev in ("cuda:0", "cuda:1", "cuda:0"):
        y = ops.linear(x.to(dev), w.to(dev))
        o = ops.attention(q.to(dev), q.to(dev), q.to(dev), 200, 200, 128 ** -0.5, True)
        torch.cuda.synchronize(dev)
        assert y.device == torch.device(dev)
        assert float((y.float().cpu() - ref).abs().max()) <= 2e-2 * float(ref.abs().max())
        outs.append(o.float().cpu())
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
