"""GPU: stop strings.  ops.stop_check_slots with one stop set in every row against transformers' StopStringCriteria row for
row on adversarial histories (both tokenizer styles, at a small vocabulary and at V = 100,352, at 1, 33 and 1,024 rows), with
finished rows left alone and stopped rows fed pad; generate(stop_strings=...) on the tiny model against its own unconstrained
run cut where StopStringCriteria first fires, across the paths generate() has; and the captured step kept without stop
strings and shared between sets of strings."""
import random

import pytest
import torch

import stop_ref

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _hf(tok, strings, hist):
    from transformers.generation.stopping_criteria import StopStringCriteria
    return StopStringCriteria(tok, list(strings))(hist, None)


_TOKS = {}


def _tok(kind, V):
    if (kind, V) not in _TOKS:
        make = stop_ref.byte_level_tokenizer if kind == "byte" else stop_ref.sentencepiece_tokenizer
        _TOKS[kind, V] = make(V)
    return _TOKS[kind, V]


def _launch(table, strings, hist, n_gen, finished=None):
    """ops.stop_check_slots with the stop set of strings in every row (no stop ids) on histories [R, H] whose last n_gen ids
    are the generated ones -> finished; every row it stops, and no other, is fed pad."""
    from aria_b200 import ops, stopping
    R, H = hist.shape
    data, lens, lookback = stopping.encode_stop_set(strings)
    tail, n = stopping.prompt_tail(hist[:, :H - n_gen]) if H > n_gen else (torch.zeros(R, 128, dtype=torch.int64), 0)
    out = torch.full((R, n_gen + 3), -5, dtype=torch.int32)
    out[:, :n_gen] = hist[:, H - n_gen:]
    fin = torch.zeros(R, dtype=torch.uint8) if finished is None else finished.clone()
    d = dict(device=DEV)
    i32 = dict(dtype=torch.int32, **d)
    dev_fin, ids_in = fin.to(DEV), torch.full((R,), 99, dtype=torch.int64, **d)
    ops.stop_check_slots(*table.device(DEV), data.repeat(R, 1, 1).to(DEV), lens.repeat(R, 1).to(DEV),
                         torch.full((R,), lookback, **i32), torch.zeros(R, 8, dtype=torch.int64, **d), torch.zeros(R, **i32),
                         tail.to(DEV), torch.full((R,), n, **i32), out.to(DEV), torch.full((R,), n_gen, **i32), dev_fin, ids_in, 3)
    got = dev_fin.cpu()
    assert ids_in.cpu().tolist() == [3 if a and not b else 99 for a, b in zip(got.tolist(), fin.tolist())]
    return got


@pytest.mark.parametrize("kind", ["byte", "sp"])
@pytest.mark.parametrize("V", [1000, 100352])
def test_kernel_one_set_in_every_row_equals_hf(kind, V):
    from aria_b200 import stopping
    tok = _tok(kind, V)
    table = stopping.vocab_table(tok)
    rng = random.Random(3)
    stopped = total = 0
    big = dict(sizes=((1, 4), (2, 24)), extra=((1, 1), (1, 128))) if V > 1000 else {}   # HF's tables are slow to build there
    for strings, hist in stop_ref.cases(tok, 12 if V == 1000 else 2, 160, seed=V, **big):
        want = _hf(tok, strings, hist).to(torch.uint8)
        for R in (1, 33, 1024):
            idx = torch.tensor([rng.randrange(hist.shape[0]) for _ in range(R)])
            n_gen = rng.randint(1, hist.shape[1])
            fin = _launch(table, strings, hist[idx], n_gen)
            assert torch.equal(fin, want[idx]), (strings, n_gen)
            stopped += int(want[idx].sum())
            total += R
    assert 0.05 * total < stopped < 0.95 * total


def test_kernel_leaves_finished_rows_and_feeds_stopped_rows_pad():
    from aria_b200 import stopping
    tok = _tok("byte", 1000)
    table = stopping.vocab_table(tok)
    v = tok.get_vocab()
    st, op, x = v["st"], v["op"], v["s"]
    hist = torch.tensor([[x, st, op], [x, x, st], [x, st, op], [x, x, x]])
    # rows 0 and 2 stop; row 1 finished before (an EOS) and is left alone, row 3 does not stop
    fin = _launch(table, ["stop"], hist, 2, finished=torch.tensor([0, 1, 0, 0], dtype=torch.uint8))
    assert fin.tolist() == [1, 1, 1, 0]
    # row 3 finished before too: every row is finished after this step
    fin = _launch(table, ["stop"], hist, 2, finished=torch.tensor([0, 1, 0, 1], dtype=torch.uint8))
    assert fin.tolist() == [1, 1, 1, 1]
    # every row finished already: nothing is checked (no row is fed pad)
    fin = _launch(table, ["stop"], hist, 2, finished=torch.ones(4, dtype=torch.uint8))
    assert fin.tolist() == [1, 1, 1, 1]


# ------------------------------------------------------------------------------------------------ generate()
@pytest.fixture(scope="module")
def tiny():
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    sd = C.aria_state(C.TINY, seed=0, dtype=torch.bfloat16)
    m = AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device=DEV)
    m.load_state_dict({k: v.to(DEV) for k, v in sd.items()}, strict=True)
    return m, C.TINY


def _prompts(cfg, padded, B=4, T=24, seed=2):
    """B prompts with one image each (8 image tokens); padded: row 1 is 5 tokens shorter, left-padded with id 0."""
    g = torch.Generator().manual_seed(seed)
    S = cfg["vision_config"]["image_size"]
    pv = torch.randn(B, 3, S, S, generator=g).bfloat16()
    rows = []
    for _ in range(B):
        text = torch.randint(10, cfg["text_config"]["vocab_size"], (T,), generator=g)
        rows.append(torch.cat([text[:4], torch.full((8,), cfg["image_token_index"]), text[4:]]))
    ids = torch.stack(rows)
    mask = None
    if padded:
        mask = torch.ones_like(ids)
        ids[1, 5:] = ids[1, :-5].clone()
        ids[1, :5] = 0
        mask[1, :5] = 0
    return ids, pv, mask


def _strings_from(tok, seqs, T, rng, n=3):
    """Stop strings from tokens the run produced: pieces of the cleaned text of 1..3 consecutive generated tokens, cut
    inside the outer ones, from different rows and positions; fewer when the run spells too few (after 500 tries)."""
    from aria_b200 import stopping
    table = stopping.vocab_table(tok)
    data, off = bytes(table.data.numpy()), table.offsets.tolist()

    def text(i):
        return data[off[i]:off[i + 1]].decode("utf-8", "replace") if 0 <= i < table.V else ""

    out = []
    for _ in range(500):
        if len(out) == n:
            break
        r = rng.randrange(seqs.shape[0])
        gen = seqs[r, T:].tolist()
        k = rng.randint(1, 3)
        j = rng.randrange(0, max(1, len(gen) - k))
        s = "".join(text(i) for i in gen[j:j + k])
        s = s[rng.randint(0, 1):len(s) - rng.randint(0, 1)] if len(s) > 2 else s
        if s and "�" not in s:
            out.append(s[:128])
    return out


def _oracle(tok, strings, plain, T, pad, eos=()):
    """The plain run cut where StopStringCriteria first fires on a row's prefix (prompt included), padded after, and trimmed
    as GenerationMixin trims when every row has finished -> (sequences, per-row stop position or None)."""
    seqs = plain.clone().cpu()
    R, N = seqs.shape
    fired, ends = [], []
    for r in range(R):
        end = None
        for t in range(T, N):
            if seqs[r, t].item() in eos or (strings is not None and bool(_hf(tok, strings, seqs[r:r + 1, :t + 1])[0])):
                end = t
                break
        if end is not None:
            seqs[r, end + 1:] = pad
            fired.append(end if seqs[r, end].item() not in eos else None)
        else:
            fired.append(None)
        ends.append(end)
    if all(e is not None for e in ends):
        seqs = seqs[:, :max(ends) + 1]
    return seqs, fired


CASES = {
    "greedy": dict(),
    "greedy_padded_eos": dict(padded=True, eos=(7, 11)),
    "sampled": dict(do_sample=True, temperature=1.3, top_k=60, top_p=0.95, seed=4),
    "sampled_padded": dict(padded=True, do_sample=True, temperature=1.3, top_k=60, top_p=0.95, seed=9),
    "fp8": dict(kv_cache_dtype="fp8", do_sample=True, temperature=1.2, top_k=50, seed=3),
    "processors": dict(do_sample=True, temperature=1.2, top_k=50, seed=6, repetition_penalty=1.2, min_new_tokens=3),
    "num_return_sequences": dict(do_sample=True, temperature=1.3, top_k=60, seed=8, num_return_sequences=3),
}


@pytest.mark.parametrize("name", list(CASES))
def test_generate_equals_the_cut_plain_run(tiny, name):
    m, cfg = tiny
    kw = dict(CASES[name])
    padded, eos = kw.pop("padded", False), kw.pop("eos", ())
    tok = _tok("byte", 1000)
    ids, pv, mask = _prompts(cfg, padded)
    T, pad, n = ids.shape[1], 3, 24
    common = dict(max_new_tokens=n, attention_mask=mask, pad_token_id=pad, eos_token_id=list(eos) or None, **kw)
    plain = m.generate(ids, pv, **common)
    rng = random.Random(hash(name) % 1000)
    rows_fired = 0
    for _ in range(3):
        strings = _strings_from(tok, plain[:, :T + n] if plain.shape[1] >= T + 2 else plain, T, rng)
        want, fired = _oracle(tok, strings, plain, T, pad, eos)
        got = m.generate(ids, pv, stop_strings=strings, tokenizer=tok, **common)
        assert torch.equal(got.cpu(), want), (strings, fired)
        rows_fired += sum(f is not None for f in fired)
    assert rows_fired >= plain.shape[0], "the stop strings fired too rarely for the test to mean anything"


def test_generate_logprobs_get_the_filler_after_a_stop(tiny):
    m, cfg = tiny
    tok = _tok("byte", 1000)
    ids, pv, _ = _prompts(cfg, False)
    T = ids.shape[1]
    common = dict(max_new_tokens=16, pad_token_id=3, output_logprobs=2)
    plain = m.generate(ids, pv, **common)
    strings = _strings_from(tok, plain.sequences, T, random.Random(1), n=4)
    want, fired = _oracle(tok, strings, plain.sequences, T, 3)
    got = m.generate(ids, pv, stop_strings=strings, tokenizer=tok, **common)
    assert torch.equal(got.sequences.cpu(), want)
    L = want.shape[1] - T
    for r, f in enumerate(fired):
        end = (f - T + 1) if f is not None else L
        assert torch.equal(got.logprobs[r, :end], plain.logprobs[r, :end])
        assert bool((got.logprobs[r, end:] == 0).all()) and bool((got.top_ids[r, end:] == -1).all())
        assert bool(torch.isneginf(got.top_logprobs[r, end:]).all())
    assert any(f is not None for f in fired)


def test_generate_shared_prefix(tiny):
    m, cfg = tiny
    tok = _tok("byte", 1000)
    ids, pv, _ = _prompts(cfg, False, B=1)
    g = torch.Generator().manual_seed(11)
    q = torch.randint(10, cfg["text_config"]["vocab_size"], (3, 6), generator=g)
    rows = torch.cat([ids.repeat(3, 1), q], dim=1)
    T = rows.shape[1]
    common = dict(max_new_tokens=20, pad_token_id=3, shared_prefix_len=ids.shape[1], do_sample=True, temperature=1.3, top_k=60,
                  seed=2)
    plain = m.generate(rows, pv, **common)
    strings = _strings_from(tok, plain, T, random.Random(2))
    want, fired = _oracle(tok, strings, plain, T, 3)
    assert torch.equal(m.generate(rows, pv, stop_strings=strings, tokenizer=tok, **common).cpu(), want)
    assert any(f is not None for f in fired)


def test_first_token_completes_a_stop_against_the_prompt(tiny):
    m, cfg = tiny
    tok = _tok("byte", 1000)
    from aria_b200 import stopping
    table = stopping.vocab_table(tok)
    data, off = bytes(table.data.numpy()), table.offsets.tolist()
    ids, pv, _ = _prompts(cfg, False)
    T = ids.shape[1]
    plain = m.generate(ids, pv, max_new_tokens=4, pad_token_id=3)
    # the prompt's last token's text and the first generated token's text, across the boundary
    r = 0
    a = data[off[int(ids[r, -1])]:off[int(ids[r, -1]) + 1]].decode()
    b = data[off[int(plain[r, T])]:off[int(plain[r, T]) + 1]].decode()
    s = (a[-1:] + b[:1])
    got = m.generate(ids, pv, max_new_tokens=4, pad_token_id=3, stop_strings=s, tokenizer=tok)
    want, fired = _oracle(tok, [s], plain, T, 3)
    assert fired[r] == T
    assert torch.equal(got.cpu(), want)


def test_plain_generate_keeps_its_captured_step_and_strings_share_one(tiny):
    m, cfg = tiny
    tok = _tok("byte", 1000)
    ids, pv, _ = _prompts(cfg, False)
    plain = m.generate(ids, pv, max_new_tokens=6, pad_token_id=3)
    g0 = m._decode_graph
    assert g0.stop is None
    m.generate(ids, pv, max_new_tokens=6, pad_token_id=3, stop_strings=["ab"], tokenizer=tok)
    g1 = m._decode_graph
    assert g1.stop is not None
    m.generate(ids, pv, max_new_tokens=6, pad_token_id=3, stop_strings=["xy", "<|im_end|>"], tokenizer=tok)
    assert m._decode_graph is g1            # other strings, the same tokenizer: no new capture
    assert torch.equal(m.generate(ids, pv, max_new_tokens=6, pad_token_id=3), plain)
    assert m._decode_graph.stop is None


# ------------------------------------------------------------------------------------------------ serving.Engine
PAGE = 256


def _workload(cfg, n=10, seed=7):
    """Requests of mixed lengths, some with images, half sampled: (ids [T], add_request kwargs without stops)."""
    g = torch.Generator().manual_seed(seed)
    rng = random.Random(seed)
    V, S, img = cfg["text_config"]["vocab_size"], cfg["vision_config"]["image_size"], cfg["image_token_index"]
    reqs = []
    for i, T in enumerate([5, 40, 300, 257, 100, 31, 256, 700, 90, 12][:n]):
        text = torch.randint(10, V, (T,), generator=g)
        kw = dict(max_new_tokens=rng.choice([3, 9, 17, 30]))
        if i % 3 == 1:
            kw.update(pixel_values=torch.randn(1, 3, S, S, generator=g).bfloat16())
            at = min(250, T // 2)
            text = torch.cat([text[:at], torch.full((8,), img), text[at:]])
        if i % 2:
            kw.update(do_sample=True, temperature=1.3, top_k=60, seed=1000 + i)
        if i == 4:
            kw.update(repetition_penalty=1.2)
        reqs.append((text, kw))
    return reqs


def _batch1(m, ids, kw, eos, pad, **extra):
    return m.generate(ids[None], kw.get("pixel_values"), max_new_tokens=kw["max_new_tokens"], do_sample=kw.get("do_sample", False),
                      temperature=kw.get("temperature", 1.0), top_k=kw.get("top_k", 50), seed=kw.get("seed", 0),
                      eos_token_id=eos or None, pad_token_id=pad, repetition_penalty=kw.get("repetition_penalty", 1.0),
                      **extra)[0]


@pytest.fixture(scope="module")
def engine_case(tiny):
    """The workload with stops drawn from each request's own unconstrained run: strings (i % 3 == 0), stop ids (i % 3 == 1,
    and i == 6 both), none (the rest); and each request's batch-1 generate() with the same stops."""
    m, cfg = tiny
    tok = _tok("byte", 1000)
    rng = random.Random(5)
    reqs, eos = _workload(cfg), [7]
    out = []
    for i, (ids, kw) in enumerate(reqs):
        T = ids.numel()
        free = _batch1(m, ids, kw, eos, 3)[None].cpu()
        stops = {}
        if i % 3 == 0 or i == 6:
            strings = _strings_from(tok, free, T, rng, n=2) if free.shape[1] > T + 1 else []
            if strings:
                stops["stop_strings"] = strings
        if (i % 3 == 1 or i == 6) and free.shape[1] > T + 2:
            stops["stop_token_ids"] = [int(free[0, T + free.shape[1] // 2 % (free.shape[1] - T)])]
        out.append((ids, dict(kw, **stops)))
    want = [_batch1(m, ids, kw, eos + kw.get("stop_token_ids", []), 3, stop_strings=kw.get("stop_strings"),
                    tokenizer=tok if "stop_strings" in kw else None) for ids, kw in out]
    free = [_batch1(m, ids, kw, eos, 3) for ids, kw in out]
    assert sum(int(w.numel() < f.numel()) for w, f in zip(want, free)) >= 3, "the stops fired too rarely to mean anything"
    return m, out, eos, want, tok


@pytest.mark.parametrize("budget,poll_every,max_batch", [(None, 3, 16), (256, 1, 4), (512, 5, 3)])
def test_engine_equals_batch1_generate(engine_case, budget, poll_every, max_batch):
    from aria_b200.serving import Engine
    m, reqs, eos, want, tok = engine_case
    eng = Engine(m, max_batch=max_batch, max_kv_tokens=64 * PAGE, eos_token_id=eos, pad_token_id=3, poll_every=poll_every,
                 max_prefill_tokens=budget, tokenizer=tok)
    rids = [eng.add_request(ids, **kw) for ids, kw in reqs]
    got = eng.run()
    for i, rid in enumerate(rids):
        assert torch.equal(got[rid], want[i]), i
    assert any(k[-1] == "stops" for k in eng._graphs)


def test_engine_without_stops_replays_the_plain_graphs(engine_case):
    from aria_b200.serving import Engine
    m, reqs, eos, want, tok = engine_case
    eng = Engine(m, max_batch=8, max_kv_tokens=64 * PAGE, eos_token_id=eos, pad_token_id=3, poll_every=2, tokenizer=tok)
    plain = [(i, ids, kw) for i, (ids, kw) in enumerate(reqs)
             if not any(k in kw for k in ("stop_strings", "stop_token_ids", "repetition_penalty"))]
    rids = [eng.add_request(ids, **kw) for _, ids, kw in plain]
    got = eng.run()
    assert all(len(k) == 2 for k in eng._graphs), list(eng._graphs)
    for (i, _, _), rid in zip(plain, rids):
        assert torch.equal(got[rid], want[i]), i


def test_engine_fp8_pages_equal_their_cut_plain_run(engine_case):
    """fp8 pages: each request equals the same engine's run without stops cut where its stops first fire, at every budget,
    poll interval and slot count."""
    from aria_b200.serving import Engine
    m, reqs, eos, _, tok = engine_case

    def serve(with_stops, budget, poll, mb):
        eng = Engine(m, max_batch=mb, max_kv_tokens=64 * PAGE, eos_token_id=eos, pad_token_id=3, poll_every=poll,
                     max_prefill_tokens=budget, kv_cache_dtype="fp8", tokenizer=tok)
        strip = ("stop_strings", "stop_token_ids")
        rids = [eng.add_request(ids, **(kw if with_stops else {k: v for k, v in kw.items() if k not in strip})) for ids, kw in reqs]
        got = eng.run()
        return [got[r].cpu() for r in rids]

    plain = serve(False, None, 3, 16)
    for budget, poll, mb in ((None, 3, 16), (256, 1, 4)):
        got = serve(True, budget, poll, mb)
        for i, (ids, kw) in enumerate(reqs):
            T = ids.numel()
            strings = kw.get("stop_strings")
            want, _ = _oracle(tok, strings, plain[i][None], T, 3, tuple(eos + kw.get("stop_token_ids", [])))
            assert torch.equal(got[i], want[0]), i


def test_kernel_slots_equal_hf():
    """ops.stop_check_slots: every slot its own strings (or none) and stop ids, against StopStringCriteria per slot."""
    from aria_b200 import ops, stopping
    tok = _tok("sp", 1000)
    table = stopping.vocab_table(tok)
    sets = stop_ref.cases(tok, 6, 64, seed=11)
    R, rng = 160, random.Random(4)
    d = dict(device=DEV)
    data = torch.zeros(R, 16, 512, dtype=torch.uint8)
    lens = torch.zeros(R, 16, dtype=torch.int32)
    look = torch.zeros(R, dtype=torch.int32)
    ids = torch.zeros(R, 8, dtype=torch.int64)
    n_ids = torch.zeros(R, dtype=torch.int32)
    tail = torch.zeros(R, 128, dtype=torch.int64)
    tail_len = torch.zeros(R, dtype=torch.int32)
    out = torch.zeros(R, 260, dtype=torch.int32)
    n_out = torch.zeros(R, dtype=torch.int32)
    fin = torch.zeros(R, dtype=torch.uint8)
    want = []
    for r in range(R):
        strings, hist = sets[rng.randrange(len(sets))]
        h = hist[rng.randrange(hist.shape[0])].tolist()
        with_strings = r % 5 != 0
        if with_strings:
            data[r], lens[r], lb = stopping.encode_stop_set(strings)
            look[r] = lb
        k = r % 3
        stop_ids = [h[-1]] if k == 1 else [5, 6] if k == 2 else []
        ids[r, :len(stop_ids)] = torch.tensor(stop_ids, dtype=torch.int64)
        n_ids[r] = len(stop_ids)
        g = rng.randint(1, len(h))
        t, n = stopping.prompt_tail(torch.tensor(h[:len(h) - g])[None]) if g < len(h) else (torch.zeros(1, 128), 0)
        tail[r], tail_len[r] = t[0], n
        out[r, :g] = torch.tensor(h[len(h) - g:], dtype=torch.int32)
        n_out[r] = g
        fin[r] = int(r % 7 == 0)
        w = bool(fin[r]) or h[-1] in stop_ids or (with_strings and bool(_hf(tok, strings, torch.tensor([h]))[0]))
        want.append(int(w))
    ids_in = torch.full((R,), 99, dtype=torch.int64)
    dev_fin, dev_ids_in = fin.to(DEV), ids_in.to(DEV)
    ops.stop_check_slots(*table.device(DEV), data.to(DEV), lens.to(DEV), look.to(DEV), ids.to(DEV), n_ids.to(DEV), tail.to(DEV),
                         tail_len.to(DEV), out.to(DEV), n_out.to(DEV), dev_fin, dev_ids_in, 3)
    assert dev_fin.cpu().tolist() == want
    stopped_now = [r for r in range(R) if want[r] and not fin[r]]
    assert len(stopped_now) > 20
    assert dev_ids_in.cpu().tolist() == [3 if r in stopped_now else 99 for r in range(R)]


@pytest.mark.parametrize("R", [33, 1024])
def test_kernel_finished_flags_over_many_ctas(R):
    """Only stopping rows, or stopping rows and rows finished before, over many CTAs: every row ends finished; one row that
    does not stop stays unfinished."""
    from aria_b200 import stopping
    tok = _tok("byte", 1000)
    table = stopping.vocab_table(tok)
    v = tok.get_vocab()
    stop_row = [v["s"], v["st"], v["op"]]
    hist = torch.tensor([stop_row] * R)
    fin = _launch(table, ["stop"], hist, 2)
    assert bool(fin.all())
    pre = (torch.arange(R) % 3 == 0).to(torch.uint8)
    fin = _launch(table, ["stop"], hist, 2, finished=pre)
    assert bool(fin.all())
    hist[R // 2, -1] = v["s"]
    fin = _launch(table, ["stop"], hist, 2, finished=pre)
    assert int(fin.sum()) == R - (0 if pre[R // 2] else 1)
