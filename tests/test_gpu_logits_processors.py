"""GPU: repetition penalty, min_new_tokens and min-p.  ops.sample_tokens_processed against transformers' own processor classes
on fp32 copies of the logits (greedy argmax, the sampled kept set and its probabilities, a chi-square fit of the draws), bit
for bit against the plain samplers when every processor is off; ops.presence_set against a torch scatter; generate() with the
processors against a per-token forward() loop that applies transformers' processors, and against the repeated batches that
num_return_sequences and shared_prefix_len already equal; serving.Engine against batch-1 generate().  Every input is seeded."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PAGE = 256


def _ops():
    from aria_b200 import ops
    return ops


def _logits(R, V, seed, scale=3.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(R, V, generator=g, device=DEV) * scale).bfloat16()


def _history(R, V, T, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    h = torch.randint(0, V, (R, T), generator=g, device=DEV)
    h[:, T // 2:] = h[:, :T - T // 2]                       # every id of the second half repeats one of the first
    return h


def hf_process(x, hist, penalty, min_new=0, eos=None, emitted=0):
    """RepetitionPenaltyLogitsProcessor -> MinNewTokensLengthLogitsProcessor on an fp32 copy of bf16 logits x [R, V], with
    input_ids = hist [R, T] whose last `emitted` ids are the generated ones."""
    from transformers.generation.logits_process import MinNewTokensLengthLogitsProcessor, RepetitionPenaltyLogitsProcessor
    s = x.float()
    if penalty != 1.0:
        s = RepetitionPenaltyLogitsProcessor(penalty)(hist, s)
    if min_new and eos is not None:
        s = MinNewTokensLengthLogitsProcessor(hist.shape[1] - emitted, min_new, eos, device=DEV)(hist, s)
    return s


def hf_warp(s, temperature, top_k, top_p, min_p):
    """TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper -> MinPLogitsWarper -> softmax (transformers' classes)."""
    from transformers.generation.logits_process import (MinPLogitsWarper, TemperatureLogitsWarper, TopKLogitsWarper,
                                                        TopPLogitsWarper)
    ids = torch.zeros(s.shape[0], 1, dtype=torch.long, device=s.device)
    s = TemperatureLogitsWarper(temperature)(ids, s)
    if top_k:
        s = TopKLogitsWarper(top_k)(ids, s)
    if top_p < 1.0:
        s = TopPLogitsWarper(top_p)(ids, s)
    pre = s.softmax(-1)                                      # min-p's probabilities, before its cut
    if min_p > 0:
        s = MinPLogitsWarper(min_p)(ids, s)
    return s.softmax(-1), pre


def _rows(R, **kw):
    """Per-row parameter arrays of sample_tokens_processed from scalars (or per-row lists)."""
    def col(v, dt):
        return torch.tensor(v if isinstance(v, list) else [v] * R, dtype=dt, device=DEV)
    return (col(kw.get("temperature", 0.0), torch.float32), col(kw.get("top_k", 0), torch.int32),
            col(kw.get("top_p", 1.0), torch.float32), col(kw.get("min_p", 0.0), torch.float32), col(kw.get("seed", 0), torch.int64),
            col(kw.get("penalty", 1.0), torch.float32), col(kw.get("min_new", 0), torch.int32))


def _presence(hist, V):
    ops = _ops()
    bm = torch.zeros(hist.shape[0], ops.presence_words(V), dtype=torch.int32, device=DEV)
    return ops.presence_set(hist, bm, V, clear=True)


def _scalar(v, dt):
    return torch.tensor([v], dtype=dt, device=DEV)


@pytest.mark.parametrize("V", [1000, 100352])
@pytest.mark.parametrize("penalty", [0.7, 1.3, 2.0])
def test_greedy_processed_argmax_equals_hf(V, penalty):
    ops = _ops()
    R = 6
    x = _logits(R, V, seed=V + int(penalty * 10))
    hist = _history(R, V, 300, seed=V)
    big = torch.tensor(40.0, dtype=torch.bfloat16, device=DEV)
    x[0, [V - 1, 50, 20]] = big                              # ties at the top; id 20 is in the history
    hist[0, 7] = 20
    x[1] = -(x[1].float().abs() + 1).bfloat16()              # every logit negative: the penalty multiplies
    hist[1, :10] = x[1].float().topk(10).indices
    x[2, :] = 0.5                                            # one constant row: ties everywhere, the history penalised
    x[3, hist[3, :40]] = big                                 # the top ids all in the history, repeated
    x[4, [3, 9]] = big                                       # an EOS at the top while min_new_tokens holds
    eos = [3, 9, 11]
    emitted, min_new = 2, [0, 0, 0, 0, 5, 0]
    ids = ops.sample_tokens_processed(x, *_rows(R, penalty=penalty, min_new=min_new), _presence(hist, V),
                                      _scalar(0, torch.int64), _scalar(emitted, torch.int32), eos)
    want = torch.stack([hf_process(x[r:r + 1], hist[r:r + 1], penalty, min_new[r], eos, emitted)[0] for r in range(R)])
    assert torch.equal(ids, want.argmax(-1))
    assert int(ids[4]) not in eos


CASES = [(1.0, 50, 1.0, 0.05, 1.2), (0.7, 300, 0.9, 0.1, 0.8), (1.3, 1024, 0.5, 0.0, 1.5), (1.0, 0, 1.0, 0.05, 1.1),
         (0.8, 0, 1.0, 0.2, 1.0), (1.0, 7, 0.95, 0.3, 1.3)]


@pytest.mark.parametrize("V", [1000, 100352])
@pytest.mark.parametrize("temperature,top_k,top_p,min_p,penalty", CASES)
def test_sampled_kept_set_and_probs_match_hf(V, temperature, top_k, top_p, min_p, penalty):
    ops = _ops()
    R = 6
    x = _logits(R, V, seed=V + top_k, scale=2.0)
    x[0, :4] = x[0].max()                                    # ties at the top
    hist = _history(R, V, 500, seed=top_k + 1)
    probs = torch.empty(R, V, device=DEV)
    ops.sample_tokens_processed(x, *_rows(R, temperature=temperature, top_k=top_k, top_p=top_p, min_p=min_p, penalty=penalty,
                                          seed=1), _presence(hist, V), _scalar(0, torch.int64), _scalar(0, torch.int32),
                                probs_out=probs)
    s = hf_process(x, hist, penalty)
    want, pre = hf_warp(s, temperature, top_k, top_p, min_p)
    for b in range(R):
        got_keep, want_keep = probs[b] > 0, want[b] > 0
        if not torch.equal(got_keep, want_keep):
            # only tokens at the top-p or the min-p boundary (within 1e-6) may differ
            sc = s[b] / temperature
            kth = torch.topk(sc, top_k)[0][-1] if top_k else -float("inf")
            sl, si = torch.sort(torch.where(sc >= kth, sc, -float("inf")), stable=True)
            cum = torch.empty_like(sl)
            cum[si] = sl.softmax(-1).cumsum(-1)
            thr = min_p * float(pre[b].max())
            for i in (got_keep != want_keep).nonzero().flatten().tolist():
                at_top_p = top_p < 1.0 and abs(float(cum[i]) - (1 - top_p)) <= 1e-6
                at_min_p = min_p > 0 and abs(float(pre[b, i]) - thr) <= 1e-6
                assert at_top_p or at_min_p, (b, i)
            continue
        assert torch.allclose(probs[b][want_keep], want[b][want_keep], rtol=1e-5, atol=0.0), b
        assert float(probs[b].sum()) == pytest.approx(1.0, abs=1e-5)


def test_chi_square_goodness_of_fit_with_penalty_and_min_p():
    """65536 draws of one row (row stride 0), each with its own Philox counter, against the kernel's own probs_out."""
    from scipy.stats import chisquare
    ops = _ops()
    V, N = 1000, 65536
    row = _logits(1, V, seed=11, scale=1.0)
    hist = _history(1, V, 200, seed=3)
    kw = dict(temperature=1.0, top_k=0, min_p=0.05, penalty=1.3, seed=1234)
    probs = torch.empty(1, V, device=DEV)
    ops.sample_tokens_processed(row, *_rows(1, **kw), _presence(hist, V), _scalar(0, torch.int64), _scalar(0, torch.int32),
                                probs_out=probs)
    pres = _presence(hist, V).expand(N, -1).contiguous()
    draws = ops.sample_tokens_processed(row.expand(N, V), *_rows(N, **kw), pres, _scalar(0, torch.int64),
                                        _scalar(0, torch.int32))
    counts = torch.bincount(draws, minlength=V).double().cpu()
    p = probs[0].double().cpu()
    assert float(counts[p == 0].sum()) == 0, "a draw fell outside the kept set"
    keep = p > 0
    exp, obs = p[keep] * N, counts[keep]
    small = exp < 5
    if small.any():
        exp = torch.cat([exp[~small], exp[small].sum().view(1)])
        obs = torch.cat([obs[~small], obs[small].sum().view(1)])
    assert chisquare(obs.numpy(), exp.numpy() * (obs.sum() / exp.sum()).item()).pvalue > 1e-3


@pytest.mark.parametrize("V", [1000, 100352])
def test_identity_parameters_are_bit_identical_to_the_plain_samplers(V):
    ops = _ops()
    R = 8
    x = _logits(R, V, seed=5 + V)
    x[1, :6] = x[1].max()
    pres = torch.full((R, ops.presence_words(V)), -1, dtype=torch.int32, device=DEV)   # every id seen: penalty 1 reads nothing
    eos = [0, 5]
    # per-row parameters and offsets against sample_tokens_slots
    t = [0.0, 0.8, 1.0, 1.3, 0.7, 1.0, 0.0, 2.0]
    k = [0, 50, 0, 1024, 7, 300, 20, 1]
    p = [1.0, 0.9, 1.0, 0.5, 0.95, 1.0, 1.0, 1.0]
    seed = [3, 4, 5, 6, 7, 8, 9, 2 ** 62]
    noise = torch.tensor([2, 0, 1, 7, 3, 3, 5, 6], dtype=torch.int32, device=DEV)
    offs = torch.tensor([0, 1, 5, 2 ** 33, 7, 7, 3, 11], dtype=torch.int64, device=DEV)
    rows = _rows(R, temperature=t, top_k=k, top_p=p, seed=seed)
    got = ops.sample_tokens_processed(x, *rows, pres, offs, torch.zeros(R, dtype=torch.int32, device=DEV), eos, noise_rows=noise)
    want = ops.sample_tokens_slots(x, rows[0], rows[1], rows[2], rows[4], noise, offs)
    assert torch.equal(got, want)
    # one offset for every row, noise row = row: sample_tokens, tokens and probs_out
    for tt, kk, pp in ((0.0, 0, 1.0), (0.9, 40, 0.9), (1.0, 0, 1.0), (1.2, 1024, 1.0)):
        off = _scalar(9, torch.int64)
        pg, pw = torch.empty(R, V, device=DEV), torch.empty(R, V, device=DEV)
        got = ops.sample_tokens_processed(x, *_rows(R, temperature=tt, top_k=kk, top_p=pp, seed=77), pres, off,
                                          _scalar(0, torch.int32), probs_out=pg)
        want = ops.sample_tokens(x, tt, kk, pp, 77, off, probs_out=pw)
        assert torch.equal(got, want) and torch.equal(pg, pw), (tt, kk, pp)


@pytest.mark.parametrize("top_k", [0, 16, 1024])
def test_suppressed_eos_is_never_drawn(top_k):
    ops = _ops()
    V, N = 16, 4096
    x = _logits(1, V, seed=2)
    x[0, [3, 7]] = 30.0                                      # the EOS ids would win almost every draw
    eos = [3, 7]
    pres = torch.zeros(N, 1, dtype=torch.int32, device=DEV)
    for t in (0.0, 1.0, 5.0):
        kw = dict(temperature=t, top_k=top_k, min_new=4, seed=1)
        draws = ops.sample_tokens_processed(x.expand(N, V), *_rows(N, **kw), pres, _scalar(0, torch.int64),
                                            torch.randint(0, 4, (N,), dtype=torch.int32, device=DEV), eos)
        assert not bool(((draws == 3) | (draws == 7)).any()), t
        # once min_new tokens are out, the EOS ids are back (greedy: the EOS with the lower id)
        draws = ops.sample_tokens_processed(x.expand(N, V), *_rows(N, **kw), pres, _scalar(0, torch.int64),
                                            _scalar(4, torch.int32), eos)
        assert bool(((draws == 3) | (draws == 7)).any()), t
        if t == 0.0:
            assert bool((draws == 3).all())


@pytest.mark.parametrize("V", [1, 31, 32, 1000, 100352])
def test_presence_set_equals_scatter(V):
    ops = _ops()
    R, T = 5, 300
    g = torch.Generator(device=DEV).manual_seed(V)
    big = torch.randint(-3, V + 3, (R, T + 17), generator=g, device=DEV)   # ids outside [0, V) included
    ids = big[:, 5:5 + T]                                                  # strided rows
    lengths = torch.tensor([0, 1, 17, T, T + 9], dtype=torch.int32, device=DEV)
    W = ops.presence_words(V)

    def ref(ids_, n=None, init=None):
        seen = torch.zeros(R, W * 32, dtype=torch.bool, device=DEV) if init is None else init.clone()
        for r in range(R):
            row = ids_[r, :None if n is None else int(n[r])]
            row = row[(row >= 0) & (row < V)]
            seen[r].scatter_(0, row, torch.ones_like(row, dtype=torch.bool))
        return seen

    def bits(bm):
        w = bm.to(torch.int64) & 0xFFFFFFFF
        return ((w[:, :, None] >> torch.arange(32, device=DEV)) & 1).bool().flatten(1)

    bm = torch.full((R, W), -1, dtype=torch.int32, device=DEV)
    ops.presence_set(ids, bm, V, clear=True)
    assert torch.equal(bits(bm), ref(ids))
    ops.presence_set(ids, bm, V, lengths=lengths, clear=True)
    first = ref(ids, lengths)
    assert torch.equal(bits(bm), first)
    more = torch.randint(0, V, (R, 1), generator=g, device=DEV)            # accumulate, the decode step's update
    ops.presence_set(more, bm, V)
    assert torch.equal(bits(bm), ref(more, init=first))


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


def _prompts(cfg, padded, T=24):
    """Two prompts with one image each (8 image tokens); padded: the second is 5 tokens shorter, left-padded with id 0."""
    g = torch.Generator().manual_seed(2)
    S = cfg["vision_config"]["image_size"]
    pv = torch.randn(2, 3, S, S, generator=g).bfloat16()
    rows = []
    for _ in range(2):
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


def _forward_loop(m, ids, pv, mask, n, penalty, min_new, eos):
    """Greedy per-token forward() loop with transformers' repetition-penalty and min-new-tokens processors on the fp32 logits
    (a row past its EOS keeps appending EOS: its tokens are not compared)."""
    B, T = ids.shape
    inputs = m.prepare_inputs_for_generation(ids, None, pixel_values=pv, attention_mask=mask, num_logits_to_keep=1)
    out = m.forward(**inputs, max_cache_len=T + n)
    cache, logits = out.past_key_values, out.logits[:, -1]
    all_ids = ids.to(DEV)
    for t in range(n):
        tok = hf_process(logits, all_ids, penalty, min_new, eos, emitted=t).argmax(-1)
        all_ids = torch.cat([all_ids, tok.view(B, 1)], dim=1)
        if t == n - 1:
            break
        if mask is not None:
            mask = torch.cat([mask, torch.ones(B, 1, dtype=mask.dtype)], dim=1)
        inputs = m.prepare_inputs_for_generation(all_ids, cache, attention_mask=mask, num_logits_to_keep=1)
        logits = m.forward(**inputs).logits[:, -1]
    return all_ids[:, T:]


@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("penalty", [1.5, 0.8])
def test_greedy_generate_equals_forward_loop_with_processors(tiny, padded, penalty):
    m, cfg = tiny
    ids, pv, mask = _prompts(cfg, padded)
    n, T = 10, ids.shape[1]
    free = m.generate(ids, pv, None, max_new_tokens=n, attention_mask=mask)[:, T:]
    eos = [int(free[0, 1]), int(free[1, 2])]                 # EOS ids the plain decode emits early
    want = _forward_loop(m, ids, pv, mask, n, penalty, 0, None)
    for min_new in (0, 6):              # without eos_token_id, min_new_tokens changes nothing, as in transformers
        got = m.generate(ids, pv, None, max_new_tokens=n, attention_mask=mask, repetition_penalty=penalty,
                         min_new_tokens=min_new)
        assert torch.equal(got[:, T:], want), min_new
        assert torch.equal(got[:, :T].cpu(), ids)
    # with EOS: min_new_tokens keeps it out of the first 6 tokens, and the rows then stop as GenerationMixin stops them
    got = m.generate(ids, pv, None, max_new_tokens=n, attention_mask=mask, eos_token_id=eos, pad_token_id=1,
                     repetition_penalty=penalty, min_new_tokens=6)
    want = _forward_loop(m, ids, pv, mask, n, penalty, 6, eos)
    for b in range(2):
        row = got[b, T:]
        assert not any(int(v) in eos for v in row[:6])
        hit = [i for i, v in enumerate(want[b].tolist()) if v in eos]
        end = hit[0] + 1 if hit else n
        assert torch.equal(row[:end], want[b, :end]), b
        assert bool((row[end:] == 1).all()), b


def test_plain_generate_keeps_its_captured_step(tiny):
    m, cfg = tiny
    ids, pv, _ = _prompts(cfg, False)
    plain = m.generate(ids, pv, max_new_tokens=6)
    assert m._decode_graph.processors is None
    m.generate(ids, pv, max_new_tokens=6, repetition_penalty=1.2)
    assert m._decode_graph.processors == (1.2, 0.0, 0)
    assert torch.equal(m.generate(ids, pv, max_new_tokens=6), plain)
    assert torch.equal(m.generate(ids, pv, max_new_tokens=6, repetition_penalty=1.0, min_p=0.0, min_new_tokens=0), plain)


SAMPLED = dict(do_sample=True, temperature=1.1, top_k=40, top_p=0.95, repetition_penalty=1.3, min_p=0.05)


def test_sampled_generate_reproduces_and_uses_the_processors(tiny):
    m, cfg = tiny
    ids, pv, _ = _prompts(cfg, True)
    a = m.generate(ids, pv, max_new_tokens=12, seed=5, **SAMPLED)
    assert torch.equal(m.generate(ids, pv, max_new_tokens=12, seed=5, **SAMPLED), a)
    plain = dict(SAMPLED, repetition_penalty=1.0, min_p=0.0)
    assert not torch.equal(m.generate(ids, pv, max_new_tokens=12, seed=5, **plain), a)
    top0 = dict(SAMPLED, top_k=0, top_p=1.0, min_p=0.2)       # full-vocabulary min-p
    b = m.generate(ids, pv, max_new_tokens=12, seed=5, **top0)
    assert torch.equal(m.generate(ids, pv, max_new_tokens=12, seed=5, **top0), b)


@pytest.mark.parametrize("n", [2, 3])
def test_num_return_sequences_equal_the_repeated_prompts(tiny, n):
    """Unpadded prompts whose T is a multiple of 256: each row's bitmap starts from its prompt's ids."""
    m, cfg = tiny
    ids, pv, _ = _prompts(cfg, False, T=248)
    got = m.generate(ids, pv, max_new_tokens=10, num_return_sequences=n, seed=11, **SAMPLED)
    want = m.generate(ids.repeat_interleave(n, 0), pv.repeat_interleave(n, 0), max_new_tokens=10, seed=11, **SAMPLED)
    assert torch.equal(got, want)


def test_shared_prefix_equals_the_repeated_image_batch(tiny):
    m, cfg = tiny
    g = torch.Generator().manual_seed(0)
    V, img, size = cfg["text_config"]["vocab_size"], cfg["image_token_index"], cfg["vision_config"]["image_size"]
    pv = torch.randn(1, 3, size, size, generator=g).bfloat16()
    text = torch.randint(10, V, (248,), generator=g)
    prefix = torch.cat([text[:4], torch.full((8,), img), text[4:]])
    S = [20, 13, 20]
    T = 256 + max(S)
    ids = torch.zeros(len(S), T, dtype=torch.long)
    mask = torch.zeros(len(S), T, dtype=torch.long)
    for b, s in enumerate(S):
        ids[b, T - 256 - s:] = torch.cat([prefix, torch.randint(10, V, (s,), generator=g)])
        mask[b, T - 256 - s:] = 1
    n = 2
    kw = dict(max_new_tokens=10, seed=4, eos_token_id=[5, 6], min_new_tokens=3, **SAMPLED)
    got = m.generate(ids, pv, attention_mask=mask, shared_prefix_len=256, num_return_sequences=n, **kw)
    want = m.generate(ids.repeat_interleave(n, 0), pv.repeat(len(S) * n, 1, 1, 1), attention_mask=mask.repeat_interleave(n, 0),
                      **kw)
    assert torch.equal(got, want)


def test_output_logprobs_stay_those_of_the_raw_distribution(tiny):
    ops = _ops()
    m, cfg = tiny
    ids, pv, _ = _prompts(cfg, False)
    out = m.generate(ids, pv, max_new_tokens=8, seed=2, output_logprobs=5, **SAMPLED)
    assert torch.equal(out.sequences, m.generate(ids, pv, max_new_tokens=8, seed=2, **SAMPLED))
    first = m(ids, pv, num_logits_to_keep=1).logits[:, -1]
    r = ops.token_logprobs(first.contiguous(), out.sequences[:, ids.shape[1]].contiguous(), 5)
    assert torch.equal(out.logprobs[:, 0], r[0]) and torch.equal(out.top_logprobs[:, 0], r[2])


# ------------------------------------------------------------------------------------------------ the engine
def _workload(cfg, n=10, seed=0):
    """n requests: prompts of 5-700 tokens, a third with images, greedy and sampled, every other one with processors."""
    import random
    rng = random.Random(seed)
    g = torch.Generator().manual_seed(seed)
    V, img, S = cfg["text_config"]["vocab_size"], cfg["image_token_index"], cfg["vision_config"]["image_size"]
    lengths = [5, 40, 300, 257, 100, 31, 256, 700, 90, 12]
    procs = [dict(repetition_penalty=1.4), dict(min_p=0.1, repetition_penalty=0.9), dict(min_new_tokens=8),
             dict(repetition_penalty=1.2, min_p=0.3, min_new_tokens=3)]
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
        if i % 4 in (0, 1) or i == 7:
            kw.update(procs[i % len(procs)])
        reqs.append((text, kw))
    return reqs


def _generate(m, ids, kw, eos, pad, **extra):
    return m.generate(ids[None], kw.get("pixel_values"), max_new_tokens=kw["max_new_tokens"], do_sample=kw.get("do_sample", False),
                      temperature=kw.get("temperature", 1.0), top_k=kw.get("top_k", 50), top_p=kw.get("top_p", 1.0),
                      seed=kw.get("seed", 0), eos_token_id=eos, pad_token_id=pad,
                      repetition_penalty=kw.get("repetition_penalty", 1.0), min_p=kw.get("min_p", 0.0),
                      min_new_tokens=kw.get("min_new_tokens", 0), **extra)[0]


@pytest.fixture(scope="module")
def engine_case(tiny):
    m, cfg = tiny
    reqs = _workload(cfg)
    free = _generate(m, reqs[2][0], dict(reqs[2][1], max_new_tokens=30), None, None)
    eos = [int(free[reqs[2][0].numel() + 2])]
    return m, cfg, reqs, eos, [_generate(m, ids, kw, eos, 3) for ids, kw in reqs]


@pytest.mark.parametrize("budget,poll_every,max_batch", [(None, 3, 16), (256, 1, 4), (512, 5, 3)])
def test_engine_equals_generate(engine_case, budget, poll_every, max_batch):
    from aria_b200.serving import Engine
    m, cfg, reqs, eos, want = engine_case
    eng = Engine(m, max_batch=max_batch, max_kv_tokens=64 * PAGE, eos_token_id=eos, pad_token_id=3, poll_every=poll_every,
                 max_prefill_tokens=budget)
    rids = [eng.add_request(ids, **kw) for ids, kw in reqs]
    got = eng.run()
    for i, rid in enumerate(rids):
        assert torch.equal(got[rid], want[i]), i
    keys = list(eng._graphs)
    assert any(len(k) == 4 and k[3] == "processors" for k in keys)


def test_engine_without_processors_replays_the_plain_graphs(engine_case):
    from aria_b200.serving import Engine
    m, cfg, reqs, eos, want = engine_case
    eng = Engine(m, max_batch=8, max_kv_tokens=64 * PAGE, eos_token_id=eos, pad_token_id=3, poll_every=2)
    plain = [(i, ids, kw) for i, (ids, kw) in enumerate(reqs)
             if not any(k in kw for k in ("repetition_penalty", "min_p", "min_new_tokens"))]
    rids = [eng.add_request(ids, **kw) for _, ids, kw in plain]
    got = eng.run()
    assert all(k in ((k[0], k[1]),) for k in eng._graphs), list(eng._graphs)
    for (i, _, _), rid in zip(plain, rids):
        assert torch.equal(got[rid], want[i]), i


def test_engine_fp8_pages_with_processors(engine_case):
    """fp8 pages: the engine's results do not depend on the poll interval, the budget or the slot count, and a request equals
    itself served alone."""
    from aria_b200.serving import Engine
    m, cfg, reqs, eos, _ = engine_case
    runs = []
    for budget, poll, mb in ((None, 3, 16), (256, 1, 4)):
        eng = Engine(m, max_batch=mb, max_kv_tokens=64 * PAGE, eos_token_id=eos, pad_token_id=3, poll_every=poll,
                     max_prefill_tokens=budget, kv_cache_dtype="fp8")
        rids = [eng.add_request(ids, **kw) for ids, kw in reqs]
        got = eng.run()
        runs.append([got[r] for r in rids])
    for i in range(len(reqs)):
        assert torch.equal(runs[0][i], runs[1][i]), i
    eng = Engine(m, max_batch=2, max_kv_tokens=64 * PAGE, eos_token_id=eos, pad_token_id=3, kv_cache_dtype="fp8")
    ids, kw = reqs[1]
    rid = eng.add_request(ids, **kw)
    assert torch.equal(eng.run()[rid], runs[0][1])
