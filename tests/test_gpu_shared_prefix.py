"""GPU: n continuations per prompt from one shared prompt cache — the shared-prefix decode attention bit for bit against the
device-length kernel on the expanded layout, the graphed generate(num_return_sequences=n) against a teacher-forced decode on an
expanded cache built by hand, and against generate() on the repeated prompts."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TAILS = [1, 256, 257, 17, 100, 2, 255]


def _ops():
    from aria_b200 import ops
    return ops


def _bucket(x):
    return -(-x // 256) * 256


def _expanded_reference(q, pk, pv, plens, pmask, tk, tv, tlens, n, scale):
    """attention_decode_devlen on the expanded layout: row r holds prefix g = r // n at [0, P), masked rows up to S = bucket(P)
    and its tail from S on."""
    ops = _ops()
    G, H = pk.shape[:2]
    R = G * n
    S = [_bucket(p) for p in plens]
    T_max = max(S) + tk.shape[2]
    k = torch.zeros(R, H, T_max, 128, dtype=torch.bfloat16, device=DEV)
    v = torch.zeros_like(k)
    km = torch.zeros(R, T_max + 8, dtype=torch.uint8, device=DEV)    # row stride > T_max
    lens = []
    for r in range(R):
        g, P, s, t = r // n, plens[r // n], S[r // n], tlens[r]
        k[r, :, :P], v[r, :, :P] = pk[g, :, :P], pv[g, :, :P]
        k[r, :, s:s + t], v[r, :, s:s + t] = tk[r, :, :t], tv[r, :, :t]
        if pmask is not None:
            km[r, :P] = pmask[g, :P]
        km[r, P:s] = 1
        lens.append(s + t)
    return ops.attention_decode_devlen(q, k, v, torch.tensor(lens, dtype=torch.int32, device=DEV), scale, key_mask=km)


def _case(G, n, H, plens, masked, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    R, P_max, N_max = G * n, max(plens), 300
    qs = torch.randn(R, H, 2, 128, generator=g, device=DEV).bfloat16()          # q [R, H, 128] at a row stride of 256
    q = qs[:, :, 0]
    pk = torch.randn(G, H, P_max, 128, generator=g, device=DEV).bfloat16()
    pv = torch.randn(G, H, P_max, 128, generator=g, device=DEV).bfloat16()
    tk = torch.randn(R, H, N_max, 128, generator=g, device=DEV).bfloat16()
    tv = torch.randn(R, H, N_max, 128, generator=g, device=DEV).bfloat16()
    tlens = [TAILS[r % len(TAILS)] for r in range(R)]
    pmask = None
    if masked:
        pmask = (torch.rand(G, P_max + 24, generator=g, device=DEV) < 0.3).to(torch.uint8)   # row stride > P_max
        pmask[:, 0] = 0
    return q, pk, pv, plens, pmask, tk, tv, tlens


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("n", [1, 2, 5, 32])
@pytest.mark.parametrize("plens", [[1], [255], [256], [700], [1, 256, 700], [255, 700, 256]])
def test_kernel_bit_identical_to_expanded_devlen(plens, n, masked):
    _run_kernel_case(len(plens), n, 20, plens, masked)


@pytest.mark.parametrize("n", [2, 5])
def test_kernel_bit_identical_small_h(n):
    _run_kernel_case(3, n, 2, [700, 1, 255], True)


def _run_kernel_case(G, n, H, plens, masked):
    ops = _ops()
    scale = 128 ** -0.5
    q, pk, pv, plens, pmask, tk, tv, tlens = _case(G, n, H, plens, masked, seed=G * 100 + n * 7 + H + int(masked))
    want = _expanded_reference(q, pk, pv, plens, pmask, tk, tv, tlens, n, scale)
    # rows at or past the lengths, and masked prompt rows, are never read
    for gi, P in enumerate(plens):
        pk[gi, :, P:] = float("nan")
        pv[gi, :, P:] = float("nan")
        if pmask is not None:
            dead = pmask[gi, :pk.shape[2]].bool()
            pk[gi, :, dead] = float("nan")
            pv[gi, :, dead] = float("nan")
    for r, t in enumerate(tlens):
        tk[r, :, t:] = float("nan")
        tv[r, :, t:] = float("nan")
    got = ops.attention_decode_shared_prefix(q, pk, pv, torch.tensor(plens, dtype=torch.int32, device=DEV), tk, tv,
                                             torch.tensor(tlens, dtype=torch.int32, device=DEV), n, scale, prefix_mask=pmask)
    assert not got.isnan().any()
    assert torch.equal(got, want)


# ------------------------------------------------------------------------------------------------ tiny model
def _tiny():
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    sd = C.aria_state(C.TINY, seed=0, dtype=torch.bfloat16)
    m = AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device=DEV)
    m.load_state_dict({k: v.to(DEV) for k, v in sd.items()}, strict=True)
    return m, C.TINY


def _prompts(cfg, T, padded, B=2):
    """B prompts of T tokens with one image each (8 image tokens); padded: the second is 5 tokens shorter, left-padded with 0."""
    g = torch.Generator().manual_seed(T)
    S = cfg["vision_config"]["image_size"]
    pv = torch.randn(B, 3, S, S, generator=g).bfloat16()
    rows = []
    for _ in range(B):
        text = torch.randint(10, cfg["text_config"]["vocab_size"], (T - 8,), generator=g)
        rows.append(torch.cat([text[:4], torch.full((8,), cfg["image_token_index"]), text[4:]]))
    ids = torch.stack(rows)
    mask = None
    if padded:
        mask = torch.ones_like(ids)
        ids[1, 5:] = ids[1, :-5].clone()
        ids[1, :5] = 0
        mask[1, :5] = 0
    return ids, pv, mask


SAMPLING = dict(do_sample=True, temperature=1.3, top_k=40, top_p=0.95)


@pytest.mark.parametrize("padded", [False, True])
def test_generate_equals_teacher_forced_expanded_cache(padded):
    """The graphed shared step against decode_step on a plain KVCache holding the expanded layout: every sampled token and the
    last step's logits bit for bit."""
    from aria_b200 import ops
    from aria_b200.moe_lm import DecodeState
    m, cfg = _tiny()
    n, new = 3, 12
    ids, pv, mask = _prompts(cfg, 40, padded)
    B, T = ids.shape
    R = B * n
    got = m.generate(ids, pv, None, max_new_tokens=new, attention_mask=mask, num_return_sequences=n, seed=5, **SAMPLING)
    assert got.shape == (R, T + new)
    assert torch.equal(got[:, :T].cpu(), ids.repeat_interleave(n, 0))
    toks = got[:, T:]
    g = m._decode_graph
    lm = m.language_model
    c = lm.config
    S = _bucket(T)
    exp = lm.new_cache(R, S + _bucket(new), DEV)
    for layer in range(c.num_hidden_layers):
        exp.k[layer][:, :, :T] = g.cache.k[layer][:, :, :T].repeat_interleave(n, 0)
        exp.v[layer][:, :, :T] = g.cache.v[layer][:, :, :T].repeat_interleave(n, 0)
    st = DecodeState(R, c.num_attention_heads, exp.T_max, DEV)
    km = torch.zeros(R, exp.T_max, dtype=torch.uint8)
    if mask is not None:
        km[:, :T] = (mask == 0).to(torch.uint8).repeat_interleave(n, 0)
    km[:, T:S] = 1
    st.key_mask.copy_(km)
    last = (torch.full((B,), T - 1) if mask is None else mask.sum(-1) - 1).to(torch.int32).repeat_interleave(n)
    rope = lm.model.rope_tables(exp.T_max, DEV)
    t, k, p = SAMPLING["temperature"], SAMPLING["top_k"], SAMPLING["top_p"]
    for step in range(1, new):
        st.rope_pos.copy_(last + step)
        st.write_pos.fill_(S + step - 1)
        st.kv_len.fill_(S + step)
        emb = ops.embedding(toks[:, step - 1:step].contiguous(), lm.get_input_embeddings().weight)
        logits = lm.decode_step(emb, exp, st, rope)[:, -1]
        off = torch.tensor([step], dtype=torch.int64, device=DEV)
        assert torch.equal(ops.sample_tokens(logits, t, k, p, 5, off), toks[:, step]), step
    assert torch.equal(g.logits[:, -1], logits)


@pytest.mark.parametrize("n", [2, 5])
def test_generate_equals_generate_on_repeated_prompts(n):
    """Unpadded prompts whose T is a multiple of 256: the expanded layout is the repeated batch's own cache layout."""
    m, cfg = _tiny()
    ids, pv, _ = _prompts(cfg, 256, False)
    new = 10
    got = m.generate(ids, pv, None, max_new_tokens=new, num_return_sequences=n, seed=11, **SAMPLING)
    want = m.generate(ids.repeat_interleave(n, 0), pv.repeat_interleave(n, 0), None, max_new_tokens=new, seed=11, **SAMPLING)
    assert torch.equal(got, want)


def test_eos_pad_and_trim_match_the_repeated_batch_at_every_poll():
    m, cfg = _tiny()
    n, new = 3, 12
    ids, pv, _ = _prompts(cfg, 256, False)
    rep_ids, rep_pv = ids.repeat_interleave(n, 0), pv.repeat_interleave(n, 0)
    free = m.generate(ids, pv, None, max_new_tokens=new, num_return_sequences=n, seed=3, **SAMPLING)[:, -new:].cpu()
    eos = [int(free[0, 3]), int(free[4, 6])]
    for poll in (1, 3, 100):
        kw = dict(max_new_tokens=new, eos_token_id=eos, pad_token_id=1, poll_every=poll, seed=3, **SAMPLING)
        got = m.generate(ids, pv, None, num_return_sequences=n, **kw)
        want = m.generate(rep_ids, rep_pv, None, **kw)
        assert torch.equal(got, want), poll
        for r in range(got.shape[0]):                          # a finished row emits pad from then on
            row = got[r, ids.shape[1]:].tolist()
            hit = [i for i, x in enumerate(row) if x in eos]
            if hit:
                assert all(x == 1 for x in row[hit[0] + 1:])


def test_rows_differ_reproduce_and_the_caches_are_shared():
    m, cfg = _tiny()
    n, new = 4, 20
    ids, pv, mask = _prompts(cfg, 300, True)
    a = m.generate(ids, pv, None, max_new_tokens=new, attention_mask=mask, num_return_sequences=n, seed=21, **SAMPLING)
    for b in range(ids.shape[0]):
        rows = a[b * n:(b + 1) * n, -new:]
        assert not all(torch.equal(rows[0], rows[j]) for j in range(1, n)), b
    again = m.generate(ids, pv, None, max_new_tokens=new, attention_mask=mask, num_return_sequences=n, seed=21, **SAMPLING)
    assert torch.equal(again, a)
    other = m.generate(ids, pv, None, max_new_tokens=new, attention_mask=mask, num_return_sequences=n, seed=22, **SAMPLING)
    assert not torch.equal(other, a)
    g = m._decode_graph
    B, H = ids.shape[0], cfg["text_config"]["num_attention_heads"]
    assert all(t.shape == (B, H, 512, 128) for t in g.cache.k + g.cache.v)                       # B x bucket(T)
    assert all(t.shape == (B * n, H, 256, 128) for t in g.cache.tail_k + g.cache.tail_v)         # B*n x bucket(new)
    # n == 1 still builds today's graph and cache
    m.generate(ids, pv, None, max_new_tokens=new, attention_mask=mask, seed=21, **SAMPLING)
    g1 = m._decode_graph
    assert type(g1.cache).__name__ == "KVCache" and g1.cache.k[0].shape == (B, H, _bucket(300 + new), 128)
