"""GPU: batched and chunked admission in serving.Engine — the varlen paged-prefix attention and page store bit for bit against
their one-segment kernels, a packed multi-request prefill_paged against one-request calls, and the engine end to end on the
tiny model under prefill budgets: every result equals batch-1 generate() bit for bit.  All inputs and seeds are fixed."""
import random

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PAGE = 256
SCALE = 128 ** -0.5


def _ops():
    from aria_b200 import ops
    return ops


def _bf16(shape, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(*shape, generator=g, device=DEV).bfloat16()


def _varlen_case(lens, prefixes, H, seed, share=None):
    """Packed segments `lens` (NaN staging rows past S_tot) with prefixes `prefixes` on shuffled pages of a pool whose other
    pages hold NaN; share = (a, b): segment b's prefix is segment a's pages -> (qkv, seg, kp, vp, table)."""
    ops = _ops()
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    S_tot = cu[-1]
    qkv = _bf16((3, 1, H, S_tot + 40, 128), seed)
    qkv[:, :, :, S_tot:] = float("nan")
    need = [P // PAGE for P in prefixes]
    n_pages = sum(need) + 5
    perm = torch.randperm(n_pages - 1, generator=torch.Generator().manual_seed(seed))[:sum(need)] + 1
    kp = torch.full((n_pages, H, PAGE, 128), float("nan"), dtype=torch.bfloat16, device=DEV)
    vp = torch.full_like(kp, float("nan"))
    width = max(need + [1]) + 2
    table = torch.full((len(lens), width), -1, dtype=torch.int32)
    at = 0
    for b, n in enumerate(need):
        table[b, :n] = perm[at:at + n].to(torch.int32)
        at += n
    if share is not None:
        a, b = share
        table[b] = table[a]
    for p in perm.tolist():
        kp[p] = _bf16((H, PAGE, 128), seed + 7 * p)
        vp[p] = _bf16((H, PAGE, 128), seed + 7 * p + 3)
    return qkv, ops.PackedSegments(cu, prefixes, DEV), kp, vp, table.to(DEV)


CASES = [
    # lens, prefixes: 1-token segments, segments straddling 128-query tiles, S_tot not a multiple of 128
    ([1, 1, 1], [0, 256, 1024]),
    ([129, 300, 1, 127, 700], [0, 256, 1024, 256, 0]),
    ([128, 128, 5], [1024, 0, 256]),
    ([2048], [2048]),
    ([64, 1000, 333, 17, 256, 400], [256, 0, 1024, 1024, 256, 0]),
]


@pytest.mark.parametrize("H", [2, 20])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_varlen_attention_equals_the_paged_prefix_kernel_per_segment(case, H):
    ops = _ops()
    lens, prefixes = CASES[case]
    share = (1, 3) if case == 1 else None                    # two segments on the same prefix pages
    qkv, seg, kp, vp, table = _varlen_case(lens, prefixes, H, seed=10 * case + H, share=share)
    got = ops.attention_prefill_paged_varlen(qkv[0], qkv[1], qkv[2], kp, vp, table, seg, SCALE)
    assert got.shape == (seg.S_tot, H * 128) and not got.isnan().any()
    for b in range(seg.n_seg):
        c, e = seg.cu[b], seg.cu[b + 1]
        one = qkv[:, :, :, c:e].contiguous()
        cu1 = torch.tensor([0, e - c], dtype=torch.int32, device=DEV)
        want = ops.attention_prefill_paged_prefix(one[0], one[1], one[2], e - c, kp, vp, table[b], seg.prefix_lens[b], cu1, SCALE)
        assert torch.equal(got[c:e], want), (b, lens[b], seg.prefix_lens[b])


def test_varlen_attention_refusals():
    ops = _ops()
    qkv, seg, kp, vp, table = _varlen_case([5, 9], [256, 0], 2, seed=1)
    for bad in ([100, 0], [-256, 0], [0, 256 * 8]):
        with pytest.raises(ValueError):
            s = ops.PackedSegments(seg.cu, bad, DEV)
            ops.attention_prefill_paged_varlen(qkv[0], qkv[1], qkv[2], kp, vp, table, s, SCALE)
    with pytest.raises(ValueError):                          # a prefix longer than its listed pages
        ops.attention_prefill_paged_varlen(qkv[0], qkv[1], qkv[2], kp, vp, table[:, :1],
                                           ops.PackedSegments(seg.cu, [512, 0], DEV), SCALE)
    with pytest.raises(RuntimeError):                        # one table row per segment
        ops.attention_prefill_paged_varlen(qkv[0], qkv[1], qkv[2], kp, vp, table[:1], seg, SCALE)
    with pytest.raises(ValueError):                          # q shorter than S_tot
        ops.attention_prefill_paged_varlen(qkv[0][:, :, :10], qkv[1], qkv[2], kp, vp, table,
                                           ops.PackedSegments([0, 5, 60], [256, 0], DEV), SCALE)
    for cu in ([0, 5, 5], [1, 5, 9], [0, 9, 5]):
        with pytest.raises(ValueError):
            ops.PackedSegments(cu, [0, 0], DEV)


def test_varlen_page_store_equals_the_one_segment_store():
    ops = _ops()
    H, n_pages = 4, 24
    lens, prefixes = [300, 1, 256, 700, 40], [0, 256, 512, 0, 1024]
    qkv, seg, _, _, _ = _varlen_case(lens, prefixes, H, seed=3)
    k, v = qkv[1].contiguous(), qkv[2].contiguous()
    perm = (torch.randperm(n_pages - 1, generator=torch.Generator().manual_seed(5)) + 1).tolist()
    width = 8
    table = torch.full((len(lens), width), -1, dtype=torch.int32)
    for b, (n, P) in enumerate(zip(lens, prefixes)):
        used = -(-(P + n) // PAGE) - P // PAGE
        table[b, P // PAGE:P // PAGE + used] = torch.tensor([perm.pop() for _ in range(used)], dtype=torch.int32)
    table[1, 1] = 0                                          # a null page entry is never written
    table = table.to(DEV)
    sentinel = -7.0
    got_k = torch.full((n_pages, H, PAGE, 128), sentinel, dtype=torch.bfloat16, device=DEV)
    got_v = got_k.clone()
    got_k[0] = 0
    got_v[0] = 0
    want_k, want_v = got_k.clone(), got_v.clone()
    ops.kv_pages_store_varlen(k, v, got_k, got_v, table, seg)
    for b, P in enumerate(prefixes):
        c, e = seg.cu[b], seg.cu[b + 1]
        row = table[b, P // PAGE:].clone()
        if b == 1:
            row[0] = -1                                      # the one-segment store would write page 0: leave it out
        ops.kv_pages_store(k[:, :, c:e].contiguous(), v[:, :, c:e].contiguous(), e - c, want_k, want_v, row)
    assert torch.equal(got_k, want_k) and torch.equal(got_v, want_v)
    assert not got_k[0].any() and not got_v[0].any()
    listed = set(table[table > 0].tolist())
    for p in range(n_pages):
        if p not in listed and p:
            assert bool((got_k[p] == sentinel).all()) and bool((got_v[p] == sentinel).all()), p


# ------------------------------------------------------------------------------------------------ tiny model
def _tiny(w8a8=False):
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    sd = C.aria_state(C.TINY, seed=0, dtype=torch.bfloat16)
    m = AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device=DEV)
    m.load_state_dict({k: v.to(DEV) for k, v in sd.items()}, strict=True)
    if w8a8:
        m.quantize_experts_fp8(activations="fp8")
        m.quantize_dense_fp8()
    return m, C.TINY


@pytest.fixture(scope="module")
def tiny():
    return _tiny()


def _text(cfg, n, seed):
    return torch.randint(10, cfg["text_config"]["vocab_size"], (n,), generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("w8a8", [False, True])
def test_packed_prefill_paged_equals_one_segment_calls(tiny, w8a8):
    from aria_b200.moe_lm import PagedKVCache
    ops = _ops()
    m, cfg = _tiny(w8a8=True) if w8a8 else tiny
    lm = m.language_model
    c = lm.config
    prompts = [_text(cfg, n, seed=n) for n in (300, 456, 513, 1)]
    prefixes = [0, 256, 512, 0]
    pages = [[1, 2], [3, 4], [5, 6, 7], [8]]
    width = 4

    def emb(ids):
        return ops.embedding(ids.to(DEV)[None], lm.get_input_embeddings().weight)

    def call(cache, parts):
        """parts [(request index, start, end)] as one packed prefill -> logits of every segment."""
        table = torch.full((len(parts), width), -1, dtype=torch.int32)
        for b, (i, _, _) in enumerate(parts):
            table[b, :len(pages[i])] = torch.tensor(pages[i], dtype=torch.int32)
        cu = [0]
        for _, s, e in parts:
            cu.append(cu[-1] + e - s)
        seg = ops.PackedSegments(cu, [s for _, s, _ in parts], DEV)
        ids = torch.cat([prompts[i][s:e] for i, s, e in parts])
        pos = torch.cat([torch.arange(s, e, dtype=torch.int32) for _, s, e in parts]).to(DEV)
        return lm.prefill_paged(emb(ids), cache, table.to(DEV), seg, pos)[0]

    caches = []
    for packed in (False, True):
        cache = PagedKVCache(c.num_hidden_layers, 12, c.num_attention_heads, c.head_dim, 4, width, DEV)
        for i, P in enumerate(prefixes):
            if P:
                call(cache, [(i, 0, P)])
        parts = [(i, P, prompts[i].numel()) for i, P in enumerate(prefixes)]
        logits = call(cache, parts) if packed else torch.cat([call(cache, [p]) for p in parts])
        caches.append((logits, cache))
    (a, ca), (b, cb) = caches
    assert a.shape == (4, c.vocab_size) and torch.equal(a, b)
    for i, ids in enumerate(prompts):                         # the prompt rows of every request's pages (no others are written)
        for x, y in zip(ca.k + ca.v, cb.k + cb.v):
            assert torch.equal(x[pages[i]].transpose(0, 1).flatten(1, 2)[:, :ids.numel()],
                               y[pages[i]].transpose(0, 1).flatten(1, 2)[:, :ids.numel()]), i


def _generate(m, ids, kw, eos=None, pad=None):
    return m.generate(ids[None], kw.get("pixel_values"), kw.get("pixel_mask"), max_new_tokens=kw["max_new_tokens"],
                      do_sample=kw.get("do_sample", False), temperature=kw.get("temperature", 1.0), top_k=kw.get("top_k", 50),
                      top_p=kw.get("top_p", 1.0), seed=kw.get("seed", 0), eos_token_id=eos, pad_token_id=pad)[0]


SAMPLED = dict(do_sample=True, temperature=1.1, top_k=40, top_p=0.95)


def _workload(cfg, n=16, seed=0):
    """n requests: prompts of 5-700 tokens, a third with one or two images, greedy and sampled, varied budgets."""
    rng = random.Random(seed)
    g = torch.Generator().manual_seed(seed)
    V, img, S = cfg["text_config"]["vocab_size"], cfg["image_token_index"], cfg["vision_config"]["image_size"]
    lengths = [5, 40, 300, 257, 100, 31, 256, 700, 90, 12, 60, 17]
    reqs = []
    for i in range(n):
        T = lengths[i % len(lengths)]
        text = torch.randint(10, V, (T,), generator=g)
        kw = dict(max_new_tokens=rng.choice([1, 3, 9, 17, 30]))
        if i % 3 == 1:
            rows = 1 + i % 2
            kw.update(pixel_values=torch.randn(rows, 3, S, S, generator=g).bfloat16())
            at = min(250, T // 2)
            text = torch.cat([text[:at], torch.full((8 * rows,), img), text[at:]])
        if i % 2:
            kw.update(SAMPLED, seed=1000 + i)
        reqs.append((text, kw))
    return reqs


@pytest.fixture(scope="module")
def tiny_case(tiny):
    m, cfg = tiny
    reqs = _workload(cfg)
    for i in (2, 4):                                         # long enough budgets for the EOS picks
        reqs[i][1]["max_new_tokens"] = 30
    free = [_generate(m, *reqs[i]) for i in (2, 4)]
    eos = [int(free[0][reqs[2][0].numel() + 2]), int(free[1][reqs[4][0].numel() + 5])]
    return m, cfg, reqs, eos, [_generate(m, ids, kw, eos, 3) for ids, kw in reqs]


def _engine(m, pages=64, **kw):
    from aria_b200.serving import Engine
    return Engine(m, max_batch=kw.pop("max_batch", 8), max_kv_tokens=pages * PAGE, poll_every=kw.pop("poll_every", 3), **kw)


@pytest.mark.parametrize("budget,poll_every", [(256, 1), (512, 3), (4096, 2), (None, 5)])
def test_engine_results_equal_generate_under_every_budget(tiny_case, budget, poll_every):
    m, cfg, reqs, eos, want = tiny_case
    eng = _engine(m, max_batch=16, eos_token_id=eos, pad_token_id=3, poll_every=poll_every, max_prefill_tokens=budget)
    rids = [eng.add_request(ids, **kw) for ids, kw in reqs]
    got = eng.run()
    for i, (rid, w) in enumerate(zip(rids, want)):
        assert torch.equal(got[rid], w), (budget, i)
    assert eng.stats["prefill_launches"] < len(reqs)
    assert (eng.stats["prefill_chunks"] > 0) == (budget is not None and budget <= 512)
    assert eng.n_active == 0 and eng.sched.pages.n_free == eng.sched.pages.n_pages - 1


def test_a_long_prompt_runs_in_three_chunks_while_another_request_decodes(tiny):
    m, cfg = tiny
    short = (_text(cfg, 20, seed=1), dict(max_new_tokens=40))
    long = (_text(cfg, 1500, seed=2), dict(max_new_tokens=6, seed=5, **SAMPLED))
    eng = _engine(m, max_prefill_tokens=512, poll_every=2)
    a = eng.add_request(short[0], **short[1])
    eng.step()                                               # the short request is admitted and decodes from now on
    b = eng.add_request(long[0], **long[1])
    launches, decoded = [], []
    got = {}
    while eng.n_active or eng.n_waiting:
        n = eng.stats["prefill_launches"]
        got.update(eng.step())
        launches.append(eng.stats["prefill_launches"] - n)
        decoded.append(int(eng.state.n_out[0]) if a not in got else None)
    assert eng.stats["prefill_launches"] == 4 and eng.stats["prefill_chunks"] == 2
    # the long prompt's three launches ran in three steps, and the short request gained tokens between them
    steps = [i for i, x in enumerate(launches) if x]
    assert len(steps) == 3 and steps == list(range(steps[0], steps[0] + 3))
    assert decoded[steps[0]] < decoded[steps[1]] < decoded[steps[2]]
    assert torch.equal(got[a], _generate(m, *short)) and torch.equal(got[b], _generate(m, *long))


def test_a_chunk_boundary_inside_an_image_runs_each_crop_once(tiny):
    m, cfg = tiny
    S, img = cfg["vision_config"]["image_size"], cfg["image_token_index"]
    text = _text(cfg, 600, seed=3)
    ids = torch.cat([text[:252], torch.full((16,), img), text[252:]])      # crop 0: tokens 252-259, crop 1: 260-267
    pv = torch.randn(2, 3, S, S, generator=torch.Generator().manual_seed(4)).bfloat16()
    pm = torch.ones(2, S, S, dtype=torch.bool)
    pm[1, :, 40:] = False
    req = (ids, dict(pixel_values=pv, pixel_mask=pm, max_new_tokens=7))
    for budget in (256, 512):
        eng = _engine(m, max_prefill_tokens=budget)
        rid = eng.add_request(ids, **req[1])
        got = eng.run()[rid]
        assert torch.equal(got, _generate(m, *req)), budget
        assert eng.stats["vit_rows_run"] == 2 and eng.stats["vit_rows_skipped"] == 0
        assert eng.stats["prefill_launches"] == -(-ids.numel() // budget)


@pytest.mark.parametrize("budget", [256, 1024, None])
def test_shared_prompts_in_one_burst_hit_what_one_at_a_time_admission_hits(tiny, budget):
    m, cfg = tiny
    system = _text(cfg, 400, seed=2)
    reqs = [(torch.cat([system, _text(cfg, n, seed=10 + n)]), dict(max_new_tokens=9 + i, **(SAMPLED if i % 2 else {}), seed=i))
            for i, n in enumerate([1, 30, 200, 500, 113])]
    same = _text(cfg, 700, seed=3)
    reqs += [(same, dict(max_new_tokens=12))] + [(same, dict(max_new_tokens=12, seed=s, **SAMPLED)) for s in (1, 2, 3)]
    eng = _engine(m, max_prefill_tokens=budget)
    rids = [eng.add_request(ids, **kw) for ids, kw in reqs]
    got = eng.run()
    for i, (rid, (ids, kw)) in enumerate(zip(rids, reqs)):
        assert torch.equal(got[rid], _generate(m, ids, kw)), (budget, i)
    assert eng.stats["prefix_hit_tokens"] == 4 * PAGE + 3 * 2 * PAGE
    assert eng.stats["prompt_tokens"] == sum(r[0].numel() for r in reqs)


def test_pool_pressure_drains_and_returns_every_page(tiny_case):
    m, cfg, reqs, eos, want = tiny_case
    eng = _engine(m, pages=9, poll_every=2, eos_token_id=eos, pad_token_id=3, max_prefill_tokens=512)
    sel = [i for i, (ids, kw) in enumerate(reqs) if ids.numel() + kw["max_new_tokens"] <= 9 * PAGE]
    rids = [eng.add_request(reqs[i][0], **reqs[i][1]) for i in sel]
    got = eng.run()
    assert [torch.equal(got[r], want[i]) for r, i in zip(rids, sel)] == [True] * len(sel)
    assert eng.sched.pages.n_free == 9 and all(eng.sched.pages.refs(p) == 0 for p in range(10))
    assert all(not bool(t[0].any()) for t in eng.cache.k + eng.cache.v)     # the null page stays zero


def test_a_bad_image_request_in_a_packed_step_is_dropped_alone(tiny_case):
    m, cfg, reqs, eos, want = tiny_case
    img = cfg["image_token_index"]
    bad_ids = torch.cat([torch.arange(10, 20), torch.full((4,), img)])    # 4 image tokens, the image gives 8 features
    eng = _engine(m, eos_token_id=eos, pad_token_id=3, max_prefill_tokens=4096)
    a = eng.add_request(reqs[0][0], **reqs[0][1])
    b = eng.add_request(reqs[2][0], **reqs[2][1])
    eng.add_request(bad_ids, reqs[1][1]["pixel_values"], max_new_tokens=4)
    c = eng.add_request(reqs[3][0], **reqs[3][1])
    with pytest.raises(ValueError, match="image"):
        eng.step()
    assert eng.n_active == 2 and eng.n_waiting == 1 and eng.stats["prefill_launches"] == 1
    got = eng.run()
    assert sorted(got) == [a, b, c]
    assert torch.equal(got[a], want[0]) and torch.equal(got[b], want[2]) and torch.equal(got[c], want[3])
    assert eng.sched.pages.n_free == 64 and eng.n_active == 0
