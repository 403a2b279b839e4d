"""GPU: generation — the sampling kernel against transformers' warper chain, the device-length decode attention against the
host-length one, and the CUDA-graph decode loop of generate() against a per-token forward() loop on the tiny model.
All inputs and seeds are fixed, so every test is deterministic."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _ops():
    from aria_b200 import ops
    return ops


def hf_probs(logits, temperature, top_k, top_p):
    """TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper -> softmax, as transformers writes them (the sort made
    stable, so boundary ties are removed lowest index first)."""
    s = logits.float() / temperature
    if top_k:
        thr = torch.topk(s, min(top_k, s.shape[-1]))[0][..., -1, None]
        s = s.masked_fill(s < thr, -float("inf"))
    if top_p < 1.0:
        sl, si = torch.sort(s, descending=False, stable=True)
        cum = sl.softmax(-1).cumsum(-1)
        rm = cum <= (1 - top_p)
        rm[..., -1:] = False
        s = s.masked_fill(rm.scatter(1, si, rm), -float("inf"))
    return s.softmax(-1)


def _logits(B, V, seed, scale=3.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(B, V, generator=g, device=DEV) * scale).bfloat16()


@pytest.mark.parametrize("V", [1000, 100352])
@pytest.mark.parametrize("B", [1, 3, 32])
def test_greedy_equals_argmax_with_ties(B, V):
    ops = _ops()
    x = _logits(B, V, seed=B * 7 + V)
    # crafted ties: the maximum repeated at several ids (the lowest must win), and a row of equal logits
    big = torch.tensor(40.0, dtype=torch.bfloat16, device=DEV)
    x[0, [V - 1, V // 2, 17]] = big
    if B > 1:
        x[1] = 0.5
    if B > 2:
        x[2, [5, 3]] = big
    ids = ops.sample_tokens(x, temperature=0.0)
    assert torch.equal(ids, x.float().argmax(-1))
    assert int(ids[0]) == 17
    probs = torch.empty(B, V, device=DEV)
    ops.sample_tokens(x, temperature=0.0, probs_out=probs)
    assert torch.equal(probs, torch.nn.functional.one_hot(ids, V).float())


@pytest.mark.parametrize("V", [1000, 100352])
@pytest.mark.parametrize("temperature,top_k,top_p", [(0.8, 200, 1.0), (1.0, 50, 1.0), (0.7, 300, 0.9), (1.3, 1024, 0.5),
                                                     (1.0, 0, 1.0), (0.6, 7, 0.95)])
def test_probs_match_hf_warpers(V, temperature, top_k, top_p):
    ops = _ops()
    B = 8
    x = _logits(B, V, seed=V + top_k, scale=2.0)
    x[0, :4] = x[0].max()                      # ties at the top
    probs = torch.empty(B, V, device=DEV)
    ops.sample_tokens(x, temperature, top_k, top_p, seed=1, probs_out=probs)
    want = hf_probs(x, temperature, top_k, top_p)
    for b in range(B):
        got_keep, want_keep = probs[b] > 0, want[b] > 0
        if not torch.equal(got_keep, want_keep):
            # only tokens tied with the top-p boundary, or within 1e-6 of it, may differ
            assert top_p < 1.0 and top_k > 0, b
            s = x[b].float() / temperature
            sl, si = torch.sort(torch.where(s >= torch.topk(s, top_k)[0][-1], s, -float("inf")), stable=True)
            cum = torch.empty_like(sl)
            cum[si] = sl.softmax(-1).cumsum(-1)
            diff = (got_keep != want_keep).nonzero().flatten()
            boundary = s[want_keep].min()
            for i in diff.tolist():
                assert s[i] == boundary or abs(float(cum[i]) - (1 - top_p)) <= 1e-6, (b, i)
            continue
        assert torch.allclose(probs[b][want_keep], want[b][want_keep], rtol=1e-5, atol=0.0), b
        assert float(probs[b].sum()) == pytest.approx(1.0, abs=1e-5)


@pytest.mark.parametrize("temperature,top_k,top_p", [(0.8, 20, 1.0), (1.0, 40, 0.8), (1.0, 0, 1.0)])
def test_chi_square_goodness_of_fit(temperature, top_k, top_p):
    """65536 draws from one row (row stride 0: every row reads the same logits, each with its own Philox counter)."""
    from scipy.stats import chisquare
    ops = _ops()
    V, N = 1000 if top_k else 64, 65536
    row = _logits(1, V, seed=11, scale=1.0)
    probs = torch.empty(1, V, device=DEV)
    ops.sample_tokens(row, temperature, top_k, top_p, seed=1234, probs_out=probs)
    draws = ops.sample_tokens(row.expand(N, V), temperature, top_k, top_p, seed=1234)
    counts = torch.bincount(draws, minlength=V).double().cpu()
    p = probs[0].double().cpu()
    assert float(counts[p == 0].sum()) == 0, "a draw fell outside the kept set"
    keep = p > 0
    exp = p[keep] * N
    obs = counts[keep]
    # merge the cells whose expectation is below 5 (the usual validity condition of the test)
    small = exp < 5
    if small.any():
        exp = torch.cat([exp[~small], exp[small].sum().view(1)])
        obs = torch.cat([obs[~small], obs[small].sum().view(1)])
    exp = exp * (obs.sum() / exp.sum())
    stat, pval = chisquare(obs.numpy(), exp.numpy())
    assert pval > 1e-3, (stat, pval)


def test_seed_and_offset_reproduce():
    ops = _ops()
    x = _logits(64, 1000, seed=5, scale=0.5)
    off = torch.tensor([5], dtype=torch.int64, device=DEV)
    a = ops.sample_tokens(x, 1.0, 0, 1.0, seed=42, rng_offset=off).clone()
    b = ops.sample_tokens(x, 1.0, 0, 1.0, seed=42, rng_offset=off).clone()
    assert torch.equal(a, b)
    off += 1
    c = ops.sample_tokens(x, 1.0, 0, 1.0, seed=42, rng_offset=off)
    assert not torch.equal(a, c)
    d = ops.sample_tokens(x, 1.0, 0, 1.0, seed=43, rng_offset=off - 1)
    assert not torch.equal(a, d)


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("lens", [[1, 255, 256], [257, 511, 700], [700, 700, 700]])
def test_decode_devlen_bit_identical(lens, masked):
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(3)
    B, H, T_max = 3, 4, 700
    q = torch.randn(B, H, 128, generator=g, device=DEV).bfloat16()
    k = torch.randn(B, H, T_max, 128, generator=g, device=DEV).bfloat16()
    v = torch.randn(B, H, T_max, 128, generator=g, device=DEV).bfloat16()
    km = None
    if masked:
        km = (torch.rand(B, T_max + 16, generator=g, device=DEV) < 0.3).to(torch.uint8)   # row stride > T_max
        km[:, 0] = 0
    want = []
    for b, n in enumerate(lens):
        m = None if km is None else km[b:b + 1, :n].clone()
        want.append(ops.attention_decode(q[b:b + 1], k[b:b + 1].contiguous(), v[b:b + 1].contiguous(), n, 128 ** -0.5, key_mask=m))
    want = torch.cat(want)
    for b, n in enumerate(lens):                    # rows at or past lens[b] are never read
        k[b, :, n:] = float("nan")
        v[b, :, n:] = float("nan")
    got = ops.attention_decode_devlen(q, k, v, torch.tensor(lens, dtype=torch.int32, device=DEV), 128 ** -0.5, key_mask=km)
    assert torch.equal(got, want)


def test_kv_append_writes_the_device_row():
    ops = _ops()
    B, H, T_max = 3, 2, 40
    kc = torch.zeros(B, H, T_max, 128, dtype=torch.bfloat16, device=DEV)
    vc = torch.zeros_like(kc)
    new = torch.randn(2, B, H, 1, 128, device=DEV).bfloat16()
    pos = torch.tensor([0, 17, 39], dtype=torch.int32, device=DEV)
    ops.kv_append(new[0, :, :, 0], new[1, :, :, 0], kc, vc, pos)
    for b, p in enumerate(pos.tolist()):
        assert torch.equal(kc[b, :, p], new[0, b, :, 0]) and torch.equal(vc[b, :, p], new[1, b, :, 0])
    assert int((kc != 0).any(-1).sum()) == B * H


# ------------------------------------------------------------------------------------------------ tiny model
def _tiny():
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    sd = C.aria_state(C.TINY, seed=0, dtype=torch.bfloat16)
    m = AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device=DEV)
    m.load_state_dict({k: v.to(DEV) for k, v in sd.items()}, strict=True)
    return m, C.TINY


def _prompts(cfg, padded):
    """Two prompts with one image each (8 image tokens); padded: the second is 5 tokens shorter, left-padded with id 0."""
    g = torch.Generator().manual_seed(2)
    S = cfg["vision_config"]["image_size"]
    pv = torch.randn(2, 3, S, S, generator=g).bfloat16()
    rows = []
    for _ in range(2):
        text = torch.randint(10, cfg["text_config"]["vocab_size"], (24,), generator=g)
        rows.append(torch.cat([text[:4], torch.full((8,), cfg["image_token_index"]), text[4:]]))
    ids = torch.stack(rows)
    mask = None
    if padded:
        mask = torch.ones_like(ids)
        ids[1, 5:] = ids[1, :-5].clone()
        ids[1, :5] = 0
        mask[1, :5] = 0
    return ids, pv, mask


def _forward_loop(m, ids, pv, mask, n, tokens=None):
    """The per-token forward() loop generate() replaced: greedy, or teacher-forced with `tokens` -> (tokens, step logits)."""
    B, T = ids.shape
    inputs = m.prepare_inputs_for_generation(ids, None, pixel_values=pv, attention_mask=mask, num_logits_to_keep=1)
    out = m.forward(**inputs, max_cache_len=T + n)
    cache, logits, toks = out.past_key_values, [out.logits[:, -1].clone()], []
    all_ids = ids.to(DEV)
    for t in range(n):
        toks.append(logits[-1].float().argmax(-1) if tokens is None else tokens[:, t])
        if t == n - 1:
            break
        all_ids = torch.cat([all_ids, toks[-1].view(B, 1)], dim=1)
        if mask is not None:
            mask = torch.cat([mask, torch.ones(B, 1, dtype=mask.dtype)], dim=1)
        inputs = m.prepare_inputs_for_generation(all_ids, cache, attention_mask=mask, num_logits_to_keep=1)
        logits.append(m.forward(**inputs).logits[:, -1].clone())
    return torch.stack(toks, 1), logits


@pytest.mark.parametrize("padded", [False, True])
def test_greedy_generate_equals_forward_loop(padded):
    m, cfg = _tiny()
    ids, pv, mask = _prompts(cfg, padded)
    n = 7
    want, logits = _forward_loop(m, ids, pv, mask, n)
    got = m.generate(ids, pv, None, max_new_tokens=n, attention_mask=mask)
    assert got.shape == (2, ids.shape[1] + n)
    assert torch.equal(got[:, :ids.shape[1]].cpu(), ids)
    assert torch.equal(got[:, -n:], want)
    assert torch.equal(m._decode_graph.logits[:, -1], logits[-1])     # the last replayed step's logits, bit for bit
    # a second call reuses the captured step and gives the same tokens
    assert torch.equal(m.generate(ids, pv, None, max_new_tokens=n, attention_mask=mask), got)


def test_sampled_tokens_lie_in_the_top_k_set_and_reproduce():
    m, cfg = _tiny()
    ids, pv, mask = _prompts(cfg, True)
    n, k, t = 10, 5, 0.8
    got = m.generate(ids, pv, None, max_new_tokens=n, attention_mask=mask, do_sample=True, temperature=t, top_k=k, seed=7)
    toks = got[:, -n:]
    _, logits = _forward_loop(m, ids, pv, mask, n, tokens=toks)
    for step, lg in enumerate(logits):
        s = lg.float() / t
        kth = torch.topk(s, k, dim=-1)[0][:, -1:]
        assert bool((s.gather(1, toks[:, step:step + 1]) >= kth).all()), step
    again = m.generate(ids, pv, None, max_new_tokens=n, attention_mask=mask, do_sample=True, temperature=t, top_k=k, seed=7)
    assert torch.equal(again, got)


def test_eos_pad_and_trim_do_not_depend_on_polling():
    m, cfg = _tiny()
    ids, pv, _ = _prompts(cfg, False)
    n = 9
    free = m.generate(ids, pv, None, max_new_tokens=n)[:, -n:].cpu()
    # EOS ids: the token row 0 emits at step 2 and the one row 1 emits at step 5 (unless row 1 meets either earlier)
    eos = [int(free[0, 2]), int(free[1, 5])]
    pad = 3
    first = []
    for b in range(2):
        hits = [t for t in range(n) if int(free[b, t]) in eos]
        first.append(hits[0])
    L = max(first) + 1
    want = free[:, :L].clone()
    for b in range(2):
        want[b, first[b] + 1:] = pad
    outs = [m.generate(ids, pv, None, max_new_tokens=n, eos_token_id=eos, pad_token_id=pad, poll_every=p) for p in (1, 3, 100)]
    for o in outs:
        assert o.shape == (2, ids.shape[1] + L)
        assert torch.equal(o[:, -L:].cpu(), want)
    # no EOS among the tokens: the full length comes back
    never = m.generate(ids, pv, None, max_new_tokens=n, eos_token_id=cfg["text_config"]["vocab_size"] + 5)
    assert torch.equal(never[:, -n:].cpu(), free)
