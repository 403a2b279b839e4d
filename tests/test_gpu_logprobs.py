"""GPU: token log-probabilities.  ops.token_logprobs against the fp64 reference (tokens and top lists, ties, n past V, strided
rows) and its output modes; generate(output_logprobs=k) against the kernel on the logits it sampled from, with its sequences
unchanged; serving.Engine's logprobs equal generate()'s bit for bit, and its prompt_logprobs equal the kernel on forward()'s
full-prompt logits.  Every input is seeded."""
import pytest
import torch

from logprobs_ref import lp_bound, token_logprobs_ref

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PAGE = 256


def _ops():
    from aria_b200 import ops
    return ops


def _rows(R, V, seed):
    """R rows cycling through: randn at scale 1 and 30, a peaked row, a constant row, rows quantized to 4 values, and rows
    whose top entries are -0 and +0 ties in mixed order below three larger logits (the pivot of n = 5 among them)."""
    g = torch.Generator().manual_seed(seed)
    out = torch.empty(R, V)
    for r in range(R):
        kind = r % 6
        if kind == 0:
            x = torch.randn(V, generator=g)
        elif kind == 1:
            x = 30 * torch.randn(V, generator=g)
        elif kind == 2:
            x = torch.randn(V, generator=g)
            x[int(torch.randint(V, (1,), generator=g))] += 60
        elif kind == 3:
            x = torch.full((V,), 0.75)
        elif kind == 4:
            x = torch.randint(0, 4, (V,), generator=g).float() - 1.5
        else:
            x = -1 - torch.rand(V, generator=g)
            p = torch.randperm(V, generator=g)
            x[p[:3]] = 2.0
            z = p[3:15].sort().values
            x[z] = torch.tensor([-0.0, 0.0] * 6)[:z.numel()]
        out[r] = x
    return out.bfloat16()


def _check(logits, tokens, n, got):
    lp, ids, top = got
    lp64, ids64, top64 = token_logprobs_ref(logits, tokens, n)
    assert torch.equal(ids.cpu().long(), ids64)
    err = (lp.cpu().double() - lp64).abs()
    assert bool((err <= lp_bound(lp64)).all()), float((err / lp_bound(lp64)).max())
    fin = torch.isfinite(top64)
    assert torch.equal(torch.isfinite(top.cpu()), fin)
    terr = (top.cpu().double() - top64)[fin].abs()
    assert bool((terr <= lp_bound(top64[fin])).all())


@pytest.mark.parametrize("V", [1, 7, 512, 100351, 100352])
@pytest.mark.parametrize("R", [1, 3, 64, 257])
def test_kernel_against_fp64(V, R):
    ops = _ops()
    g = torch.Generator().manual_seed(V + R)
    x = _rows(R, V, seed=V * 7 + R)
    tokens = torch.randint(V, (R,), generator=g)
    pad = 13                                                    # strided rows, not 16-byte aligned
    buf = torch.zeros(R, V + pad, dtype=torch.bfloat16)
    buf[:, :V] = x
    xd = buf.to(DEV)[:, :V]
    for n in (0, 1, 5, 20):
        got = ops.token_logprobs(xd, tokens.to(DEV), n)
        _check(x, tokens, n, got)
        if n in (0, 20):                                        # the same row gives the same bits anywhere
            alone = [ops.token_logprobs(x[r:r + 1].to(DEV), tokens[r:r + 1].to(DEV), n) for r in range(min(R, 6))]
            for r, a in enumerate(alone):
                for u, w in zip(got, a):
                    assert torch.equal(u[r], w[0]), (n, r)
        if n:                                                    # a chosen token in its top list matches it bit for bit
            lp, ids, top = got
            hit = ids.long() == tokens.to(DEV)[:, None]
            assert torch.equal(top[hit], lp[:, None].expand_as(top)[hit])


@pytest.mark.parametrize("V", [100351, 100352])
def test_a_token_in_its_own_top_list_has_the_same_bits(V):
    """lp of token top_ids[:, j] equals top_logprobs[:, j] bit for bit for every j < 20, on rows whose threads see different
    maxima (randn at scales 1 and 30), and tied entries of a top list carry the same logprob."""
    ops = _ops()
    g = torch.Generator().manual_seed(V)
    x = torch.randn(64, V, generator=g)
    x[32:] *= 30
    xd = x.bfloat16().to(DEV)
    _, ids, top = ops.token_logprobs(xd, torch.zeros(64, dtype=torch.int64, device=DEV), 20)
    for j in range(20):
        lp, _, _ = ops.token_logprobs(xd, ids[:, j].long().contiguous(), 0)
        assert torch.equal(lp, top[:, j]), j
    q = (torch.randint(0, 6, (64, V), generator=g).float() + x * 1e-3).bfloat16().to(DEV)   # many ties near the top
    _, ids, top = ops.token_logprobs(q, torch.zeros(64, dtype=torch.int64, device=DEV), 20)
    vals = q.gather(1, ids.long())
    same = vals[:, 1:] == vals[:, :-1]
    assert bool(same.any()) and torch.equal(top[:, 1:][same], top[:, :-1][same])
    for j in (0, 7, 19):
        lp, _, _ = ops.token_logprobs(q, ids[:, j].long().contiguous(), 0)
        assert torch.equal(lp, top[:, j]), j


def test_output_modes_touch_only_their_entries():
    ops = _ops()
    R, V, n, cols = 6, 1000, 4, 5
    x = _rows(R, V, seed=3).to(DEV)
    tok = torch.arange(R, device=DEV) * 7
    ref = ops.token_logprobs(x, tok, n)

    def fresh():
        return (torch.full((R, cols), 9.0, device=DEV), torch.full((R, cols, n), 9, dtype=torch.int32, device=DEV),
                torch.full((R, cols, n), 9.0, device=DEV))

    fin = torch.tensor([0, 1, 0, 0, 1, 0], dtype=torch.uint8, device=DEV)
    for mode in ("column", "ring", "per_row"):
        out = fresh()
        if mode == "column":
            col, ring, cs = torch.tensor([2], dtype=torch.int32, device=DEV), 0, [2] * R
        elif mode == "ring":
            col, ring, cs = torch.tensor([7, 8, 9, 10, 11, 3], dtype=torch.int32, device=DEV), 4, [3, 0, 1, 2, 3, 3]
        else:
            col, ring, cs = torch.tensor([0, 4, 1, 5, 2, -1], dtype=torch.int32, device=DEV), 0, [0, 4, 1, None, 2, None]
        for fill in (True, False):
            out = fresh()
            ops.token_logprobs(x, tok, n, col=col, ring=ring, finished=fin, finished_fill=fill, out=out)
            for r in range(R):
                for c in range(cols):
                    e = [out[0][r, c], out[1][r, c], out[2][r, c]]
                    if c != cs[r] or (fin[r] and not fill):
                        assert float(e[0]) == 9.0 and bool((e[1] == 9).all()) and bool((e[2] == 9.0).all()), (mode, r, c)
                    elif fin[r]:
                        assert float(e[0]) == 0.0 and bool((e[1] == -1).all()) and bool((e[2] == float("-inf")).all())
                    else:
                        assert torch.equal(e[0], ref[0][r]) and torch.equal(e[1], ref[1][r]) and torch.equal(e[2], ref[2][r])
    out = fresh()                                               # n_row: -1 skips, a smaller n fills the rest
    n_row = torch.tensor([-1, 0, 2, 4, 9, 1], dtype=torch.int32, device=DEV)
    ops.token_logprobs(x, tok, n, n_row=n_row, col=torch.tensor([1], dtype=torch.int32, device=DEV), out=out)
    assert float(out[0][0, 1]) == 9.0
    for r in range(1, R):
        k = min(int(n_row[r]), n)
        assert torch.equal(out[1][r, 1, :k], ref[1][r, :k]) and bool((out[1][r, 1, k:] == -1).all())
        assert torch.equal(out[0][r, 1], ref[0][r])


# ------------------------------------------------------------------------------------------------ generate()
def _tiny():
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    sd = C.aria_state(C.TINY, seed=0, dtype=torch.bfloat16)
    m = AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device=DEV)
    m.load_state_dict({k: v.to(DEV) for k, v in sd.items()}, strict=True)
    return m, C.TINY


@pytest.fixture(scope="module")
def tiny():
    return _tiny()


def _text(cfg, B, T, seed):
    return torch.randint(10, cfg["text_config"]["vocab_size"], (B, T), generator=torch.Generator().manual_seed(seed))


SAMPLED = dict(do_sample=True, temperature=1.1, top_k=5, top_p=0.95, seed=7)


@pytest.mark.parametrize("case", ["greedy", "sampled", "nrs", "shared_prefix", "fp8", "eos"])
def test_generate_output_logprobs(tiny, case):
    ops = _ops()
    m, cfg = tiny
    ids = _text(cfg, 3, 40, seed=1)
    kw = dict(max_new_tokens=12)
    if case in ("sampled", "nrs", "shared_prefix"):
        kw.update(SAMPLED)
    if case == "nrs":
        kw["num_return_sequences"] = 4
    if case == "shared_prefix":
        ids[:, :20] = ids[0, :20]
        kw["shared_prefix_len"] = 20
    if case == "fp8":
        kw["kv_cache_dtype"] = "fp8"
    if case == "eos":
        free = m.generate(ids, **kw)
        kw.update(eos_token_id=int(free[0, 40 + 3]), pad_token_id=1)
    want = m.generate(ids, **kw)
    for k in (0, 5, 20):
        out = m.generate(ids, output_logprobs=k, **kw)
        seq = out.sequences
        assert torch.equal(seq, want), (case, k)
        Bn, L = seq.shape[0], seq.shape[1] - 40
        assert out.logprobs.shape == (Bn, L) and out.top_ids.shape == (Bn, L, k) and out.top_ids.dtype == torch.int64
        gen = seq[:, 40:]
        if case == "shared_prefix":
            # its first token's logits come from the packed question prefill over the prefix cache, not from forward() on
            # each row's prompt; column 0 is checked against its own top list below instead
            first = None
        elif case == "fp8":
            # generate()'s prefill writes an fp8 cache: the same call on a cache of the same kind
            cache = m.language_model.new_cache(ids.shape[0], 256, DEV, "fp8")
            first = m(ids, past_key_values=cache, num_logits_to_keep=1).logits[:, -1]
        else:
            first = m(ids, num_logits_to_keep=1).logits[:, -1]
            if case == "nrs":
                first = first.repeat_interleave(4, 0)
        if first is not None:                                   # column 0: the kernel on the prefill's last logits
            r = ops.token_logprobs(first.contiguous(), gen[:, 0].contiguous(), k)
            assert torch.equal(out.logprobs[:, 0], r[0]) and torch.equal(out.top_ids[:, 0], r[1].long())
            assert torch.equal(out.top_logprobs[:, 0], r[2])
        if k:                                                   # a token in its own top list: the same bits
            hit = out.top_ids == gen[..., None]
            assert torch.equal(out.top_logprobs[hit], out.logprobs[..., None].expand_as(out.top_logprobs)[hit])
        if L == 12:                                             # the last column: the last replayed step's logits
            g = m._decode_graph
            r = ops.token_logprobs(g.logits[:, -1], gen[:, -1].contiguous(), k)
            live = torch.ones(Bn, dtype=torch.bool, device=DEV)
            if case == "eos":                                   # rows finished before the last step hold the filler
                live = ~(gen[:, :-1] == kw["eos_token_id"]).any(-1)
            assert torch.equal(out.logprobs[live, -1], r[0][live]) and torch.equal(out.top_logprobs[live, -1], r[2][live])
        if k and case in ("greedy", "fp8"):
            assert torch.equal(out.top_ids[..., 0], gen) and torch.equal(out.top_logprobs[..., 0], out.logprobs)
        if k >= 5 and case in ("sampled", "nrs", "shared_prefix"):
            # top_k = 5 keeps every tie of the 5th value, so a sampled token is one of the 5 listed or ties the 5th
            listed = (out.top_ids[..., :5] == gen[..., None]).any(-1)
            assert bool((listed | (out.logprobs == out.top_logprobs[..., 4])).all())
        if case == "eos":
            eos = kw["eos_token_id"]
            for b in range(Bn):
                hit = (gen[b] == eos).nonzero()
                if hit.numel() and int(hit[0]) + 1 < L:
                    e = int(hit[0])
                    assert bool((out.logprobs[b, e + 1:] == 0).all()) and bool((out.top_ids[b, e + 1:] == -1).all())
                    assert bool((out.top_logprobs[b, e + 1:] == float("-inf")).all())


# ------------------------------------------------------------------------------------------------ the engine
def _generate(m, ids, kw, eos=None, pad=None, k=None):
    return m.generate(ids[None], kw.get("pixel_values"), kw.get("pixel_mask"), max_new_tokens=kw["max_new_tokens"],
                      do_sample=kw.get("do_sample", False), temperature=kw.get("temperature", 1.0), top_k=kw.get("top_k", 50),
                      top_p=kw.get("top_p", 1.0), seed=kw.get("seed", 0), eos_token_id=eos, pad_token_id=pad, output_logprobs=k)


def _workload(cfg, n=12, seed=0):
    """n requests built like test_gpu_admission's: prompts of 5-700 tokens, a third with images, greedy and sampled, logprobs
    None / 0 / 5 / 20 in turn."""
    import random
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
            kw.update(do_sample=True, temperature=1.1, top_k=40, top_p=0.95, seed=1000 + i)
        reqs.append((text, kw, [None, 0, 5, 20][i % 4]))
    return reqs


@pytest.fixture(scope="module")
def tiny_case(tiny):
    m, cfg = tiny
    reqs = _workload(cfg)
    free = _generate(m, reqs[2][0], dict(reqs[2][1], max_new_tokens=30))
    eos = [int(free[0, reqs[2][0].numel() + 2])]
    # fp8 pages are compared across budgets and poll intervals (their reference is not plain generate())
    want = {"bf16": [_generate(m, ids, kw, eos, 3, k) for ids, kw, k in reqs]}
    return m, cfg, reqs, eos, want


def _engine(m, pages=64, **kw):
    from aria_b200.serving import Engine
    return Engine(m, max_batch=kw.pop("max_batch", 16), max_kv_tokens=pages * PAGE, **kw)


@pytest.mark.parametrize("kv", ["bf16", "fp8"])
@pytest.mark.parametrize("budget", [256, None])
@pytest.mark.parametrize("poll_every", [1, 3, 5])
def test_engine_logprobs_equal_generate(tiny_case, kv, budget, poll_every):
    m, cfg, reqs, eos, want = tiny_case
    eng = _engine(m, eos_token_id=eos, pad_token_id=3, poll_every=poll_every, max_prefill_tokens=budget, kv_cache_dtype=kv)
    rids = [eng.add_request(ids, logprobs=k, **kw) for ids, kw, k in reqs]
    got = eng.run()
    assert set(eng.logprobs) == {rid for rid, (_, _, k) in zip(rids, reqs) if k is not None}
    results = []
    for i, (rid, (ids, kw, k)) in enumerate(zip(rids, reqs)):
        w = want["bf16"][i]
        if kv == "bf16":
            seq = w[0] if k is None else w.sequences[0]
            assert torch.equal(got[rid], seq), i
        if k is None:
            continue
        lp = eng.logprobs[rid]
        n_gen = got[rid].numel() - ids.numel()
        assert lp.token_logprobs.shape == (n_gen,) and lp.top_ids.shape == (n_gen, k) and lp.prompt_logprobs is None
        if kv == "bf16":
            assert torch.equal(lp.token_logprobs, w.logprobs[0].cpu()), i
            assert torch.equal(lp.top_ids, w.top_ids[0].cpu()) and torch.equal(lp.top_logprobs, w.top_logprobs[0].cpu()), i
        results.append((got[rid].cpu(), lp.token_logprobs, lp.top_ids, lp.top_logprobs))
    if kv == "fp8":
        key = ("fp8_results",)
        prev = tiny_case[4].setdefault(key, results)
        for a, b in zip(prev, results):
            for u, v in zip(a, b):
                assert torch.equal(u, v)


def test_engine_without_logprobs_captures_todays_graphs(tiny_case):
    m, cfg, reqs, eos, _ = tiny_case
    eng = _engine(m, eos_token_id=eos, pad_token_id=3, poll_every=3)
    for ids, kw, _ in reqs:
        eng.add_request(ids, **kw)
    eng.run()
    assert eng.logprobs == {} and all(len(key) == 2 for key in eng._graphs)
    assert eng.stats["graphs_captured"] == len(eng._graphs)


@pytest.mark.parametrize("budget", [256, 512, None])
def test_engine_prompt_logprobs_equal_forward(tiny, budget):
    ops = _ops()
    m, cfg = tiny
    reqs = _workload(cfg, n=6, seed=5)
    eng = _engine(m, poll_every=2, max_prefill_tokens=budget)
    ks = [0, 5, 20, 3, 1, 20]
    rids = [eng.add_request(ids, prompt_logprobs=k, **kw) for (ids, kw, _), k in zip(reqs, ks)]
    eng.run()
    for rid, (ids, kw, _), k in zip(rids, reqs, ks):
        T = ids.numel()
        lp = eng.logprobs[rid]
        assert lp.token_logprobs is None and lp.prompt_logprobs.shape == (T - 1,) and lp.prompt_top_ids.shape == (T - 1, k)
        logits = m(ids[None], kw.get("pixel_values")).logits[0, :-1]
        r = ops.token_logprobs(logits.contiguous(), ids[1:].to(DEV), k)
        assert torch.equal(lp.prompt_logprobs, r[0].cpu()), (budget, rid)
        assert torch.equal(lp.prompt_top_ids, r[1].cpu().long()) and torch.equal(lp.prompt_top_logprobs, r[2].cpu())


def test_engine_prompt_logprobs_fp8_across_budgets_and_a_cached_repeat(tiny):
    m, cfg = tiny
    reqs = _workload(cfg, n=4, seed=9)
    runs = []
    for budget in (256, None):
        eng = _engine(m, poll_every=2, max_prefill_tokens=budget, kv_cache_dtype="fp8")
        rids = [eng.add_request(ids, prompt_logprobs=5, **kw) for ids, kw, _ in reqs]
        eng.run()
        runs.append([eng.logprobs[r] for r in rids])
    for a, b in zip(*runs):
        assert torch.equal(a.prompt_logprobs, b.prompt_logprobs) and torch.equal(a.prompt_top_ids, b.prompt_top_ids)
    # a repeat of a cached prompt: full prompt logprobs again, identical, and no hit counted
    eng = _engine(m, poll_every=2)
    ids, kw, _ = reqs[2]                                      # 300 tokens: one full page
    first = eng.add_request(ids, prompt_logprobs=5, **kw)
    eng.run()
    hits = eng.stats["prefix_hit_tokens"]
    again = eng.add_request(ids, prompt_logprobs=5, **kw)
    eng.run()
    assert eng.stats["prefix_hit_tokens"] == hits
    a, b = eng.logprobs[first], eng.logprobs[again]
    assert torch.equal(a.prompt_logprobs, b.prompt_logprobs) and torch.equal(a.prompt_top_logprobs, b.prompt_top_logprobs)
    assert a.prompt_logprobs.shape == (ids.numel() - 1,)
    plain = eng.add_request(ids, **kw)                        # a plain request still hits the pages it keyed
    eng.run()
    assert eng.stats["prefix_hit_tokens"] == hits + PAGE
