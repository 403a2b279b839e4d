"""GPU: many questions about one image — the suffix prefill attention over a shared prefix bit for bit against the prefill
kernel on each row's own [prefix, suffix] layout, the tail scatter, and generate(shared_prefix_len=P) against generate() on the
repeated-image batch and on each row's own prompt."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LENS = [1, 127, 128, 129, 300, 5, 64, 200]
SCALE = 128 ** -0.5


def _ops():
    from aria_b200 import ops
    return ops


def _bucket(x):
    return -(-x // 256) * 256


def _case(B, H, P, seed, lens=None):
    """Packed suffixes of B rows in staging buffers with spare rows, and a prefix cache with rows past P."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    S = lens or [LENS[(b + seed) % len(LENS)] for b in range(B)]
    S_tot = sum(S)
    cu = [0]
    for s in S:
        cu.append(cu[-1] + s)
    qkv = torch.randn(3, 1, H, S_tot + 40, 128, generator=g, device=DEV).bfloat16()
    pre = torch.randn(2, 1, H, P + 70, 128, generator=g, device=DEV).bfloat16()
    return qkv, pre, S, cu


def _row_layout(qkv, pre, P, cu, b):
    q = qkv[0, :, :, cu[b]:cu[b + 1]].contiguous()
    k = torch.cat([pre[0, :, :, :P], qkv[1, :, :, cu[b]:cu[b + 1]]], dim=2).contiguous()
    v = torch.cat([pre[1, :, :, :P], qkv[2, :, :, cu[b]:cu[b + 1]]], dim=2).contiguous()
    return q, k, v


def _shared(qkv, pre, P, cu):
    """The new kernel, with NaN in every prefix row >= P and every staging row >= S_tot (never read)."""
    S_tot = cu[-1]
    qkv, pre = qkv.clone(), pre.clone()
    qkv[:, :, :, S_tot:] = float("nan")
    pre[:, :, :, P:] = float("nan")
    cu_dev = torch.tensor(cu, dtype=torch.int32, device=DEV)
    return _ops().attention_prefill_shared_prefix(qkv[0], qkv[1], qkv[2], S_tot, pre[0], pre[1], P, cu_dev, SCALE)


@pytest.mark.parametrize("H", [20, 2])
@pytest.mark.parametrize("B", [1, 3, 17])
@pytest.mark.parametrize("P", [128, 256, 1024])
def test_kernel_bit_identical_to_prefill_on_each_rows_layout(P, B, H):
    ops = _ops()
    qkv, pre, S, cu = _case(B, H, P, seed=P + 7 * B + H)
    got = _shared(qkv, pre, P, cu)
    assert got.shape == (cu[-1], H * 128) and not got.isnan().any()
    for b in range(B):
        q, k, v = _row_layout(qkv, pre, P, cu, b)
        want = ops.attention(q, k, v, S[b], P + S[b], SCALE, causal=True)[0]
        assert torch.equal(got[cu[b]:cu[b + 1]], want), (b, S[b])


def test_kernel_covers_the_listed_suffix_lengths():
    ops = _ops()
    lens = [1, 127, 128, 129, 300]
    for P in (128, 256):
        qkv, pre, S, cu = _case(len(lens), 20, P, seed=P, lens=lens)
        got = _shared(qkv, pre, P, cu)
        for b in range(len(lens)):
            q, k, v = _row_layout(qkv, pre, P, cu, b)
            assert torch.equal(got[cu[b]:cu[b + 1]], ops.attention(q, k, v, S[b], P + S[b], SCALE, causal=True)[0])


def _fp64_rows(q, k, v):
    s = torch.einsum("hqd,hkd->hqk", q[0].double(), k[0].double()) * SCALE
    Tq, Tk = q.shape[2], k.shape[2]
    s = s.masked_fill(torch.ones(Tq, Tk, dtype=torch.bool, device=DEV).triu(Tk - Tq + 1), float("-inf"))
    return torch.einsum("hqk,hkd->qhd", s.softmax(-1), v[0].double()).reshape(Tq, -1)


@pytest.mark.parametrize("P", [1, 127, 300, 700])
def test_kernel_within_prefill_error_when_the_prefix_is_not_tile_aligned(P):
    ops = _ops()
    B, H = 5, 4
    qkv, pre, S, cu = _case(B, H, P, seed=P)
    got = _shared(qkv, pre, P, cu).double()
    err_new = err_ref = amax = 0.0
    for b in range(B):
        q, k, v = _row_layout(qkv, pre, P, cu, b)
        ref = _fp64_rows(q, k, v)
        base = ops.attention(q, k, v, S[b], P + S[b], SCALE, causal=True)[0].double()
        err_new = max(err_new, float((got[cu[b]:cu[b + 1]] - ref).abs().max()))
        err_ref = max(err_ref, float((base - ref).abs().max()))
        amax = max(amax, float(ref.abs().max()))
    ulp = 2.0 ** (torch.tensor(amax).log2().floor().item() - 7)    # one bf16 ulp at the output's largest magnitude
    print(f"P={P}: max abs error vs fp64 {err_new:.3e} (prefill kernel on the row layouts {err_ref:.3e}, 1 ulp {ulp:.3e})")
    assert err_new <= err_ref + ulp


def test_scatter_fills_every_copy_and_leaves_the_rest():
    ops = _ops()
    B, n, H, N = 3, 4, 2, 512
    qkv, _, S, cu = _case(B, H, 1, seed=3, lens=[1, 300, 129])
    tk = torch.full((B * n, H, N, 128), 7.0, dtype=torch.bfloat16, device=DEV)
    tv = torch.full_like(tk, -7.0)
    ops.kv_scatter_tails(qkv[1], qkv[2], cu[-1], tk, tv, torch.tensor(cu, dtype=torch.int32, device=DEV), n)
    for b in range(B):
        for j in range(n):
            r = b * n + j
            assert torch.equal(tk[r, :, :S[b]], qkv[1, 0, :, cu[b]:cu[b + 1]])
            assert torch.equal(tv[r, :, :S[b]], qkv[2, 0, :, cu[b]:cu[b + 1]])
            assert bool((tk[r, :, S[b]:] == 7.0).all()) and bool((tv[r, :, S[b]:] == -7.0).all())


# ------------------------------------------------------------------------------------------------ tiny model
def _tiny():
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    sd = C.aria_state(C.TINY, seed=0, dtype=torch.bfloat16)
    m = AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device=DEV)
    m.load_state_dict({k: v.to(DEV) for k, v in sd.items()}, strict=True)
    return m, C.TINY


def _questions(cfg, P, S, seed=0):
    """One image (8 image tokens) in a prefix of P tokens, and B = len(S) questions of S[b] tokens about it, left-padded with 0
    -> (ids [B, P + max S], pixel values [1, 3, s, s], mask or None when the lengths are equal)."""
    g = torch.Generator().manual_seed(seed)
    V, img = cfg["text_config"]["vocab_size"], cfg["image_token_index"]
    size = cfg["vision_config"]["image_size"]
    pv = torch.randn(1, 3, size, size, generator=g).bfloat16()
    text = torch.randint(10, V, (P - 8,), generator=g)
    prefix = torch.cat([text[:4], torch.full((8,), img), text[4:]])
    T = P + max(S)
    ids = torch.zeros(len(S), T, dtype=torch.long)
    mask = torch.zeros(len(S), T, dtype=torch.long)
    for b, s in enumerate(S):
        ids[b, T - P - s:] = torch.cat([prefix, torch.randint(10, V, (s,), generator=g)])
        mask[b, T - P - s:] = 1
    return ids, pv, (None if len(set(S)) == 1 else mask)


SAMPLING = dict(do_sample=True, temperature=1.3, top_k=40, top_p=0.95)


@pytest.mark.parametrize("n", [1, 3])
def test_equal_questions_match_the_repeated_image_batch(n):
    m, cfg = _tiny()
    ids, pv, _ = _questions(cfg, 256, [20, 20, 20])
    B, new = ids.shape[0], 10
    got = m.generate(ids, pv, max_new_tokens=new, shared_prefix_len=256, num_return_sequences=n, seed=4, **SAMPLING)
    want = m.generate(ids.repeat_interleave(n, 0), pv.repeat(B * n, 1, 1, 1), max_new_tokens=new, seed=4, **SAMPLING)
    assert got.shape == (B * n, ids.shape[1] + new)
    assert torch.equal(got, want)


def test_eos_pad_and_trim_match_the_repeated_image_batch_at_every_poll():
    m, cfg = _tiny()
    n, new = 3, 12
    ids, pv, _ = _questions(cfg, 256, [17, 17])
    B, T = ids.shape
    free = m.generate(ids, pv, max_new_tokens=new, shared_prefix_len=256, num_return_sequences=n, seed=3, **SAMPLING)[:, T:].cpu()
    eos = [int(free[0, 3]), int(free[4, 6])]
    for poll in (1, 3, 100):
        kw = dict(max_new_tokens=new, eos_token_id=eos, pad_token_id=1, poll_every=poll, seed=3, **SAMPLING)
        got = m.generate(ids, pv, shared_prefix_len=256, num_return_sequences=n, **kw)
        want = m.generate(ids.repeat_interleave(n, 0), pv.repeat(B * n, 1, 1, 1), **kw)
        assert torch.equal(got, want), poll


def test_equal_questions_with_fp8_experts_and_dense_weights():
    m, cfg = _tiny()
    m.quantize_experts_fp8("fp8").quantize_dense_fp8()
    ids, pv, _ = _questions(cfg, 256, [24, 24, 24], seed=1)
    B, n = ids.shape[0], 2
    got = m.generate(ids, pv, max_new_tokens=8, shared_prefix_len=256, num_return_sequences=n, seed=9, **SAMPLING)
    want = m.generate(ids.repeat_interleave(n, 0), pv.repeat(B * n, 1, 1, 1), max_new_tokens=8, seed=9, **SAMPLING)
    assert torch.equal(got, want)


def test_ragged_questions_greedy_match_each_rows_own_prompt():
    m, cfg = _tiny()
    S = [5, 33, 1, 20]
    ids, pv, mask = _questions(cfg, 256, S, seed=2)
    T, new = ids.shape[1], 9
    got = m.generate(ids, pv, max_new_tokens=new, attention_mask=mask, shared_prefix_len=256)
    assert got.shape == (len(S), T + new)
    assert torch.equal(got[:, :T].cpu(), ids)
    for b, s in enumerate(S):
        own = ids[b, T - 256 - s:][None]
        want = m.generate(own, pv, max_new_tokens=new)
        assert torch.equal(got[b, T:], want[0, own.shape[1]:]), b


def _first_logits_shared(m, ids, pv, mask, P):
    """First-token logits of generate(shared_prefix_len=P)'s prefill, through the public model pieces."""
    from aria_b200 import ops
    from aria_b200.moe_lm import SharedPrefixCache
    lm = m.language_model
    c = lm.config
    B, T = ids.shape
    lens = mask.sum(-1)
    S = (lens - P).tolist()
    cache = SharedPrefixCache(c.num_hidden_layers, 1, B, c.num_attention_heads, _bucket(P), _bucket(max(S)), c.head_dim, DEV)
    start = T - int(lens[0])
    m.forward(ids[:1, start:start + P], pv, past_key_values=cache, num_logits_to_keep=1)
    suffix = torch.cat([ids[b, T - s:] for b, s in enumerate(S)])[None].to(DEV)
    cu = torch.tensor([0] + torch.tensor(S).cumsum(0).tolist(), dtype=torch.int32)
    pos = torch.cat([torch.arange(P, P + s, dtype=torch.int32) for s in S]).to(DEV)
    x, pending = lm.model.prefill_suffixes(ops.embedding(suffix, lm.get_input_embeddings().weight), cache, cu.to(DEV), pos)
    last = (cu[1:] - 1).long().to(DEV)
    h, _ = lm.model.norm(x[0, last].contiguous(), residual=pending[0, last].contiguous())
    return lm.lm_head(h).float()


# rel-L2 of the first-token logits against forward() on each row's own prompt at P = 300: measured 0 on an H100 80GB HBM3
# (700 W).  That is a measured coincidence of these inputs, not a property of the kernel: for P % 128 != 0 the prefix tile at
# keys 256-299 and the suffix tiles split the keys differently from the row's own layout, and here the differences in the fp32
# sums happen to round to the same bf16 values.  The bound is twice the measured value (never above 1e-2); every kernel is
# deterministic, so it holds run after run, but a change to the attention's rounding must measure it again.
REL_L2_BOUND = 0.0


def test_ragged_questions_unaligned_prefix_first_logits():
    m, cfg = _tiny()
    S = [5, 33, 1, 20]
    P = 300
    ids, pv, mask = _questions(cfg, P, S, seed=5)
    got = _first_logits_shared(m, ids, pv, mask, P)
    T = ids.shape[1]
    worst = 0.0
    for b, s in enumerate(S):
        want = m(ids[b, T - P - s:][None], pv).logits[0, -1].float()
        worst = max(worst, float((got[b] - want).norm() / want.norm()))
    print(f"P={P}: first-token logits rel-L2 vs forward() on each row's own prompt: {worst:.3e}")
    assert worst <= REL_L2_BOUND


def test_cache_shapes_graph_key_and_plain_generate_after():
    m, cfg = _tiny()
    S, new, n = [5, 40, 12], 30, 2
    ids, pv, mask = _questions(cfg, 300, S, seed=6)
    m.generate(ids, pv, max_new_tokens=new, attention_mask=mask, shared_prefix_len=300, num_return_sequences=n, **SAMPLING)
    g = m._decode_graph
    H = cfg["text_config"]["num_attention_heads"]
    assert type(g.cache).__name__ == "SharedPrefixCache"
    assert all(t.shape == (1, H, _bucket(300), 128) for t in g.cache.k + g.cache.v)
    assert all(t.shape == (3 * n, H, _bucket(40 + new), 128) for t in g.cache.tail_k + g.cache.tail_v)
    assert g.key[0] == 1 and g.key[7] == 3 * n and g.key[8] == _bucket(40 + new)
    m.generate(ids, pv.repeat(3, 1, 1, 1), max_new_tokens=new, attention_mask=mask)
    g1 = m._decode_graph
    assert type(g1.cache).__name__ == "KVCache" and g1.cache.k[0].shape == (3, H, _bucket(ids.shape[1] + new), 128)


def test_graph_serves_every_question_length_of_its_bucket():
    """Shared calls whose longest question + max_new_tokens share a 256-row bucket reuse one captured step, and the reused step
    gives the tokens of a freshly captured one."""
    m, cfg = _tiny()
    new = 20
    ids, pv, mask = _questions(cfg, 256, [5, 40, 12], seed=7)
    m.generate(ids, pv, max_new_tokens=new, attention_mask=mask, shared_prefix_len=256)
    g = m._decode_graph
    ids2, pv2, mask2 = _questions(cfg, 256, [33, 7, 61, 2], seed=8)     # other lengths, other B * n, same buckets
    got = m.generate(ids2, pv2, max_new_tokens=new, attention_mask=mask2, shared_prefix_len=256, num_return_sequences=1)
    assert m._decode_graph is not g            # 4 rows instead of 3: another step
    g4 = m._decode_graph
    ids3, pv3, mask3 = _questions(cfg, 256, [9, 18, 3, 50], seed=9)
    again = m.generate(ids3, pv3, max_new_tokens=new, attention_mask=mask3, shared_prefix_len=256)
    assert m._decode_graph is g4               # longest question 50 instead of 61: the same step
    got_re = m.generate(ids2, pv2, max_new_tokens=new, attention_mask=mask2, shared_prefix_len=256)
    assert m._decode_graph is g4 and torch.equal(got_re, got)
    m._decode_graph = None
    assert torch.equal(m.generate(ids3, pv3, max_new_tokens=new, attention_mask=mask3, shared_prefix_len=256), again)
