"""GPU: prompt-lookup decoding — the multi-query decode attention bit for bit against the device-length kernel per query, the
per-row sampler against sample_tokens, the draft and accept kernels against the Python rules, and
generate(prompt_lookup_num_tokens=K) token for token against generate()."""
import pytest
import torch

from prompt_lookup_ref import accept, draft

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SAMPLING = dict(do_sample=True, temperature=1.3, top_k=40, top_p=0.95)


def _ops():
    from aria_b200 import ops
    return ops


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("B,Q", [(1, 1), (1, 5), (3, 2), (3, 16), (32, 5)])
@pytest.mark.parametrize("masked", [False, True])
def test_attention_decode_multi_equals_devlen_per_query(B, Q, masked):
    ops = _ops()
    H, T_max = 4, 8192 if B == 1 else 1024
    g = torch.Generator(device=DEV).manual_seed(B * 100 + Q)
    q = torch.randn(B, H, Q, 128, generator=g, device=DEV).bfloat16()
    k = torch.randn(B, H, T_max, 128, generator=g, device=DEV).bfloat16()
    v = torch.randn(B, H, T_max, 128, generator=g, device=DEV).bfloat16()
    starts = [255 - Q // 2, 256 - Q, 257, 1, 511, T_max - Q, 100, 700]                # around split boundaries, and up to T_max
    if B == 1:
        starts = [T_max - Q - 3]
    base = torch.tensor([max(1, starts[b % len(starts)]) for b in range(B)], dtype=torch.int32)
    lens = (base[:, None] + torch.arange(Q, dtype=torch.int32)).reshape(-1).to(DEV)
    km = None
    if masked:
        km = (torch.rand(B, T_max + 8, generator=g, device=DEV) < 0.3).to(torch.uint8)   # row stride > T_max
        km[:, 0] = 0
    for b in range(B):                                                                  # rows no query may read
        last = int(base[b]) + Q - 1
        k[b, :, last:] = float("nan")
        v[b, :, last:] = float("nan")
    got = ops.attention_decode_multi(q, k, v, lens, 128 ** -0.5, key_mask=km)
    assert got.shape == (B, Q, H * 128) and not got.isnan().any()
    for i in range(Q):
        want = ops.attention_decode_devlen(q[:, :, i], k, v, lens.view(B, Q)[:, i].contiguous(), 128 ** -0.5, key_mask=km)
        assert torch.equal(got[:, i], want), i


@pytest.mark.parametrize("greedy", [True, False])
def test_sample_tokens_rows_equals_sample_tokens(greedy):
    ops = _ops()
    R, V = 12, 1000
    g = torch.Generator(device=DEV).manual_seed(1)
    logits = (torch.randn(R, V, generator=g, device=DEV) * 3).bfloat16()
    noise = torch.tensor([r // 3 for r in range(R)], dtype=torch.int32, device=DEV)
    offs = torch.tensor([7 + r % 3 for r in range(R)], dtype=torch.int64, device=DEV)
    t, k, p = (0.0, 0, 1.0) if greedy else (SAMPLING["temperature"], SAMPLING["top_k"], SAMPLING["top_p"])
    got = ops.sample_tokens_rows(logits, t, k, p, 5, noise, offs)
    for r in range(R):
        # row r as row noise[r] of a batch at offset offs[r]: put it there in a batch of its own
        batch = torch.zeros(int(noise[r]) + 1, V, dtype=torch.bfloat16, device=DEV)
        batch[-1] = logits[r]
        want = ops.sample_tokens(batch, t, k, p, 5, offs[r:r + 1].clone())
        assert int(got[r]) == int(want[-1]), r


def _hist_batch(B, H_max, seed):
    g = torch.Generator().manual_seed(seed)
    hist = torch.zeros(B, H_max, dtype=torch.int64)
    lens = []
    for b in range(B):
        n = int(torch.randint(1, H_max, (1,), generator=g))
        vocab = [3, 5, 50][b % 3]
        hist[b, :n] = torch.randint(0, vocab, (n,), generator=g)
        lens.append(n)
    return hist, lens


@pytest.mark.parametrize("K,M", [(1, 1), (4, 2), (10, 3), (15, 16)])
def test_ngram_draft_equals_the_rule(K, M):
    ops = _ops()
    B, H_max, max_new = 40, 300, 20
    hist, lens = _hist_batch(B, H_max, K * 31 + M)
    eos = (2,)
    n_out = torch.tensor([b % 22 for b in range(B)], dtype=torch.int32)         # some rows at or near max_new
    fin = torch.tensor([b % 7 == 3 for b in range(B)], dtype=torch.uint8)
    drafts = torch.full((B, K + 3), -5, dtype=torch.int64, device=DEV)          # row stride K + 3
    dl = torch.zeros(B, dtype=torch.int32, device=DEV)
    flag = torch.zeros(2, dtype=torch.int32, device=DEV)
    ops.ngram_draft(hist.to(DEV), torch.tensor(lens, dtype=torch.int32, device=DEV), fin.to(DEV), n_out.to(DEV), max_new,
                    drafts[:, :K + 1], dl, flag[1:], K, M, eos)
    drafts, dl = drafts.cpu(), dl.cpu()
    anyd = False
    for b in range(B):
        h = hist[b, :lens[b]].tolist()
        want = [] if fin[b] else draft(h, K, M, eos, room=max_new - 1 - int(n_out[b]))
        assert int(dl[b]) == len(want) and drafts[b, :len(want)].tolist() == want, b
        assert all(x == h[-1] for x in drafts[b, len(want):K].tolist())
        assert (drafts[b, K:] == -5).all()
        anyd |= bool(want)
    assert anyd and int(flag[1]) == 1 and int(flag[0]) == 0


def test_lookup_accept_advance_equals_the_rule():
    ops = _ops()
    K, max_new, H_max = 4, 10, 64
    Q = K + 1
    eos = (99,)
    # rows: full / partial / no acceptance, EOS in the accepted run, the max_new clip, already finished, no draft, at max_new
    drafts = [[5, 6, 7, 8], [5, 6, 7, 8], [5, 6, 7, 8], [5, 99, 7, 8], [5, 6, 7, 8], [5, 6, 7, 8], [], [1]]
    targets = [[5, 6, 7, 8, 9], [5, 6, 1, 8, 9], [4, 6, 7, 8, 9], [5, 99, 7, 8, 9], [5, 6, 7, 8, 9], [5, 6, 7, 8, 9],
               [3, 0, 0, 0, 0], [1, 2, 0, 0, 0]]
    n_out0 = [2, 2, 2, 2, 7, 3, 0, 10]
    fin0 = [0, 0, 0, 0, 0, 1, 0, 0]
    B = len(drafts)
    step_ids = torch.zeros(B, Q, dtype=torch.int64)
    for b, d in enumerate(drafts):
        step_ids[b, 0] = 42
        step_ids[b, 1:1 + len(d)] = torch.tensor(d, dtype=torch.int64)
    i64, i32 = dict(dtype=torch.int64, device=DEV), dict(dtype=torch.int32, device=DEV)
    hist = torch.zeros(B, H_max, **i64)
    hist_len = torch.tensor([10 + b for b in range(B)], **i32)
    out_tokens = torch.full((B, max_new), -1, **i64)
    rope = torch.tensor([20 + b for b in range(B)], **i32)
    write = torch.tensor([30 + b for b in range(B)], **i32)
    kvl = torch.tensor([31 + b for b in range(B)], **i32)
    n_out = torch.tensor(n_out0, **i32)
    fin = torch.tensor(fin0, dtype=torch.uint8, device=DEV)
    ids1, idsk = torch.zeros(B, 1, **i64), step_ids.to(DEV)
    pos_k, lens_k, off1, offk = torch.zeros(B * Q, **i32), torch.zeros(B * Q, **i32), torch.zeros(B, **i64), torch.zeros(B * Q, **i64)
    status, counters = torch.full((2,), 7, **i32), torch.zeros(2, **i64)
    ops.lookup_accept_advance(torch.tensor(targets, **i64).view(-1), idsk, torch.tensor([len(d) for d in drafts], **i32), ids1, idsk,
                              pos_k, lens_k, off1, offk, out_tokens, hist, hist_len, n_out, fin, rope, write, kvl, status, counters,
                              eos)
    drafted = accepted = 0
    all_done = True
    for b in range(B):
        live = not fin0[b] and n_out0[b] < max_new
        emitted, f = accept(drafts[b], targets[b], n_out0[b], max_new, eos) if live else ([], bool(fin0[b]))
        e = len(emitted)
        n = n_out0[b] + e
        assert out_tokens[b, n_out0[b]:n].tolist() == emitted and (out_tokens[b, :n_out0[b]] == -1).all()
        assert (out_tokens[b, n:] == -1).all(), b
        assert hist[b, 10 + b:10 + b + e].tolist() == emitted and int(hist_len[b]) == 10 + b + e
        assert int(n_out[b]) == n and bool(fin[b]) == f
        assert (int(rope[b]), int(write[b]), int(kvl[b])) == (20 + b + e, 30 + b + e, 31 + b + e)
        last = emitted[-1] if e else None
        if last is not None:
            assert int(ids1[b, 0]) == last and int(idsk[b, 0]) == last
        assert pos_k.view(B, Q)[b].tolist() == [20 + b + e + i for i in range(Q)]
        assert lens_k.view(B, Q)[b].tolist() == [31 + b + e + i for i in range(Q)]
        assert offk.view(B, Q)[b].tolist() == [n + i for i in range(Q)] and int(off1[b]) == n
        if live and drafts[b]:
            drafted += len(drafts[b])
            accepted += e - 1
        all_done &= f or n >= max_new
    assert idsk[:, 1:].cpu().equal(step_ids[:, 1:])                         # the drafts' slots are left to ngram_draft
    assert counters.tolist() == [drafted, accepted]
    assert status.tolist() == [int(all_done), 0] and not all_done
    assert [len(accept(drafts[b], targets[b], n_out0[b], max_new, eos)[0]) for b in range(5)] == [5, 3, 1, 2, 3]


# ------------------------------------------------------------------------------------------------ generate()
def _tiny():
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    sd = C.aria_state(C.TINY, seed=0, dtype=torch.bfloat16)
    m = AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device=DEV)
    m.load_state_dict({k: v.to(DEV) for k, v in sd.items()}, strict=True)
    return m, C.TINY


def _prompts(cfg, T, B, repeat=False):
    """B prompts of T tokens with one image each (8 image tokens), rows after the first left-padded by 3 b tokens; repeat: the
    text is a short phrase repeated, so greedy continuations copy n-grams of the prompt."""
    g = torch.Generator().manual_seed(T + B)
    S = cfg["vision_config"]["image_size"]
    pv = torch.randn(B, 3, S, S, generator=g).bfloat16()
    V = cfg["text_config"]["vocab_size"]
    ids = torch.zeros(B, T, dtype=torch.int64)
    mask = torch.ones(B, T, dtype=torch.int64)
    for b in range(B):
        n = T - 3 * b
        text = torch.randint(10, V, (n - 8,), generator=g)
        if repeat:
            text = torch.randint(10, V, (6,), generator=g).repeat(n)[:n - 8]
        ids[b, T - n:] = torch.cat([text[:4], torch.full((8,), cfg["image_token_index"]), text[4:]])
        mask[b, :T - n] = 0
    return ids, pv, (mask if B > 1 else None)


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("sampled", [False, True])
@pytest.mark.parametrize("K,M", [(1, 1), (4, 2), (10, 3)])
def test_generate_equals_generate(B, sampled, K, M):
    m, cfg = _tiny()
    ids, pv, mask = _prompts(cfg, 60, B, repeat=True)
    kw = dict(max_new_tokens=24, attention_mask=mask, seed=7, **(SAMPLING if sampled else {}))
    want = m.generate(ids, pv, None, **kw)
    got = m.generate(ids, pv, None, prompt_lookup_num_tokens=K, max_matching_ngram_size=M, **kw)
    assert torch.equal(got, want)
    st = m.prompt_lookup_stats
    assert st["tokens"] == B * 24 and st["steps"] <= 23 and st["accepted"] <= st["drafted"]


def test_one_graph_serves_every_prompt_length_of_a_bucket():
    """Prompts of 20, 100 and 236 tokens with 16 new tokens and K = 4 all fall in the 256-row bucket: one captured pair of steps
    serves them, each call equals generate(), and every row's whole history (prompt + output) is kept for drafting."""
    m, cfg = _tiny()
    new, K = 16, 4
    cases = [_prompts(cfg, T, 3, repeat=True) for T in (20, 100, 236)]
    want = [m.generate(ids, pv, None, max_new_tokens=new, attention_mask=mask) for ids, pv, mask in cases]
    g = None
    for (ids, pv, mask), w in zip(cases, want):
        got = m.generate(ids, pv, None, max_new_tokens=new, attention_mask=mask, prompt_lookup_num_tokens=K)
        assert torch.equal(got, w), ids.shape
        assert g is None or m._decode_graph is g
        g = m._decode_graph
        assert g.T_max == 256
        assert g.hist_len.tolist() == (mask.sum(-1) + new).tolist()                # nothing of the history was dropped
        for b in range(3):
            n = int(mask[b].sum())
            assert torch.equal(g.hist[b, :n + new].cpu(), torch.cat([ids[b, -n:], w[b, -new:].cpu()]))


@pytest.mark.parametrize("sampled", [False, True])
def test_lookup_bucket_past_the_plain_bucket(sampled):
    """T + max_new_tokens = 254 fits generate()'s 256-row cache, and the K = 4 verify rows push the lookup cache to 512 rows: the
    prefill and every step run on a cache of another row count, with the same tokens."""
    m, cfg = _tiny()
    ids, pv, mask = _prompts(cfg, 230, 3, repeat=True)
    kw = dict(max_new_tokens=24, attention_mask=mask, seed=13, **(SAMPLING if sampled else {}))
    want = m.generate(ids, pv, None, **kw)
    assert m._decode_graph.cache.T_max == 256
    got = m.generate(ids, pv, None, prompt_lookup_num_tokens=4, **kw)
    assert m._decode_graph.cache.T_max == 512
    assert torch.equal(got, want)


def test_eos_pad_and_trim_at_every_poll():
    m, cfg = _tiny()
    ids, pv, mask = _prompts(cfg, 60, 3, repeat=True)
    new = 16
    free = m.generate(ids, pv, None, max_new_tokens=new, attention_mask=mask, seed=3, **SAMPLING)[:, -new:].cpu()
    for eos in ([int(free[0, 3]), int(free[2, 6])], [int(free[0, 2]), int(free[1, 1]), int(free[2, 4])]):
        kw = dict(max_new_tokens=new, attention_mask=mask, eos_token_id=eos, pad_token_id=1, seed=3, **SAMPLING)
        got = m.generate(ids, pv, None, prompt_lookup_num_tokens=4, **kw)
        for poll in (1, 3, 100):
            assert torch.equal(got, m.generate(ids, pv, None, poll_every=poll, **kw)), (eos, poll)


def test_w8a8_experts_with_fp8_dense_projections():
    m, cfg = _tiny()
    m.quantize_experts_fp8("fp8").quantize_dense_fp8()
    ids, pv, mask = _prompts(cfg, 60, 3, repeat=True)
    for sampling in ({}, SAMPLING):
        kw = dict(max_new_tokens=20, attention_mask=mask, seed=9, **sampling)
        assert torch.equal(m.generate(ids, pv, None, prompt_lookup_num_tokens=4, **kw), m.generate(ids, pv, None, **kw))


def test_drafting_happens_on_a_repeating_continuation():
    """A greedy continuation that repeats an n-gram of its history: K-wide steps run, drafts are accepted, and fewer steps than
    tokens are replayed."""
    m, cfg = _tiny()
    new = 48
    for T in range(60, 80):                     # the first fixed prompt whose continuation takes a draft's first token
        ids, pv, _ = _prompts(cfg, T, 1, repeat=True)
        want = m.generate(ids, pv, None, max_new_tokens=new)
        hist = ids[0].tolist() + want[0, -new:].cpu().tolist()
        if any(draft(hist[:T + j], 4, 2)[:1] == [hist[T + j]] for j in range(1, new)):
            break
    else:
        pytest.fail("no prompt of the family has a continuation that repeats an n-gram of its history")
    got = m.generate(ids, pv, None, max_new_tokens=new, prompt_lookup_num_tokens=4)
    assert torch.equal(got, want)
    st = m.prompt_lookup_stats
    assert st["k_steps"] > 0 and st["accepted"] > 0 and st["steps"] < st["tokens"] - 1, st


def test_plain_generate_rebuilds_its_graph_after_a_lookup_call():
    m, cfg = _tiny()
    ids, pv, mask = _prompts(cfg, 60, 3)
    kw = dict(max_new_tokens=12, attention_mask=mask, seed=1)
    want = m.generate(ids, pv, None, **kw)
    m.generate(ids, pv, None, prompt_lookup_num_tokens=4, **kw)
    assert m._decode_graph.key[0] == "lookup" and m._decode_graph.cache.T_max == 256
    got = m.generate(ids, pv, None, **kw)
    g = m._decode_graph
    assert torch.equal(got, want) and g.key[0] == 3 and g.cache.T_max == 256 and g.state.qkv.shape[3] == 1


def test_rope_tables_do_not_depend_on_their_length():
    m, _ = _tiny()
    model = m.language_model.model
    model._rope = None
    a = model.rope_tables(256, DEV)
    model._rope = None
    b = model.rope_tables(8192, DEV)
    assert torch.equal(a[0], b[0][:256]) and torch.equal(a[1], b[1][:256])
