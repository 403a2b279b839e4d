"""GPU: continuous batching — the paged decode kernel against the contiguous devlen one, the paged append and page store, the
per-slot sampler against the scalar one, the per-slot advance, and serving.Engine end to end on the tiny model: every request's
result equals batch-1 generate() on its own prompt, bit for bit, whatever the arrivals, slots, buckets and polling.
All inputs and seeds are fixed, so every test is deterministic."""
import random

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PAGE = 256


def _ops():
    from aria_b200 import ops
    return ops


def _bf16(shape, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(*shape, generator=g, device=DEV).bfloat16()


def _paged_copy(k, v, n_pages, seed):
    """The rows of contiguous k / v [R, H, T_max, 128] in a shared pool of n_pages, each row on shuffled, non-monotonic pages ->
    (k_pool, v_pool, block_table [R, T_max / 256])."""
    R, H, T_max, _ = k.shape
    P = T_max // PAGE
    perm = torch.randperm(n_pages, generator=torch.Generator().manual_seed(seed))[:R * P]
    bt = perm.view(R, P).to(torch.int32)
    kp = _bf16((n_pages, H, PAGE, 128), seed + 1)
    vp = _bf16((n_pages, H, PAGE, 128), seed + 2)
    for r in range(R):
        for s in range(P):
            kp[bt[r, s]] = k[r, :, s * PAGE:(s + 1) * PAGE]
            vp[bt[r, s]] = v[r, :, s * PAGE:(s + 1) * PAGE]
    return kp, vp, bt.to(DEV)


@pytest.mark.parametrize("R", [1, 6, 64])
def test_paged_decode_is_bit_identical_to_devlen(R):
    ops = _ops()
    H, T_max = 2, 17 * PAGE
    lens_set = [1, 255, 256, 257, 1000, 4097]
    lens = torch.tensor([lens_set[(r * 5 + R) % len(lens_set)] for r in range(R)], dtype=torch.int32, device=DEV)
    q = _bf16((R, H, 128), 10 + R)
    k, v = _bf16((R, H, T_max, 128), 20 + R), _bf16((R, H, T_max, 128), 30 + R)
    kp, vp, bt = _paged_copy(k, v, R * 17 + 5, seed=R)
    want = ops.attention_decode_devlen(q, k, v, lens, 128 ** -0.5)
    got = ops.attention_decode_paged(q, kp, vp, bt, lens, 128 ** -0.5)
    assert torch.equal(got, want)
    # a table wider than the live pages (unmapped columns = -1) and a table with a larger row stride change nothing
    wide = torch.full((R, 24), -1, dtype=torch.int32, device=DEV)
    wide[:, :17] = bt
    assert torch.equal(ops.attention_decode_paged(q, kp, vp, wide, lens, 128 ** -0.5), want)
    strided = torch.full((R + 3, 40), -1, dtype=torch.int32, device=DEV)
    strided[:R, :17] = bt
    assert torch.equal(ops.attention_decode_paged(q, kp, vp, strided[:, :20], lens, 128 ** -0.5), want)


def test_paged_append_writes_exactly_one_row_or_nothing():
    ops = _ops()
    R, H, n_pages, P = 6, 2, 20, 3
    kp, vp = _bf16((n_pages, H, PAGE, 128), 1), _bf16((n_pages, H, PAGE, 128), 2)
    bt = torch.tensor([[4, 9, 1], [7, -1, -1], [0, 2, 3], [5, 6, 8], [10, -1, 12], [13, 14, 15]], dtype=torch.int32, device=DEV)
    # slots: a valid row in page 1 of its table, a valid row 0, negative, past the table, on an unmapped (-1) column, the last row
    pos = torch.tensor([256 + 17, 0, -1, P * PAGE, 300, 3 * PAGE - 1], dtype=torch.int32, device=DEV)
    kn, vn = _bf16((R, H, 128), 3), _bf16((R, H, 128), 4)
    k0, v0 = kp.clone(), vp.clone()
    ops.kv_append_paged(kn, vn, kp, vp, bt, pos)
    want_k, want_v = k0.clone(), v0.clone()
    for r, (page, row) in {0: (9, 17), 1: (7, 0), 5: (15, 255)}.items():
        want_k[page, :, row] = kn[r]
        want_v[page, :, row] = vn[r]
    assert torch.equal(kp, want_k) and torch.equal(vp, want_v)
    # nothing but refused rows: the whole pool is bit-unchanged
    ops.kv_append_paged(kn, vn, kp, vp, bt, torch.tensor([-5, 256, -1, 10 ** 6, 256, -2], dtype=torch.int32, device=DEV))
    assert torch.equal(kp, want_k) and torch.equal(vp, want_v)


def test_pages_store_then_gather_gives_the_contiguous_rows():
    ops = _ops()
    H, T, T_max, n_pages = 2, 700, 768, 12
    k, v = _bf16((1, H, T_max, 128), 5), _bf16((1, H, T_max, 128), 6)
    kp, vp = _bf16((n_pages, H, PAGE, 128), 7), _bf16((n_pages, H, PAGE, 128), 8)
    row = torch.tensor([7, 2, 10, -1, -1], dtype=torch.int32, device=DEV)
    before_k = kp.clone()
    ops.kv_pages_store(k, v, T, kp, vp, row)
    gk = torch.cat([kp[p] for p in (7, 2, 10)], dim=1)[:, :T]
    gv = torch.cat([vp[p] for p in (7, 2, 10)], dim=1)[:, :T]
    assert torch.equal(gk, k[0, :, :T]) and torch.equal(gv, v[0, :, :T])
    # rows past T and pages outside the row are untouched
    assert torch.equal(kp[10, :, T - 512:], before_k[10, :, T - 512:])
    others = [p for p in range(n_pages) if p not in (7, 2, 10)]
    assert torch.equal(kp[others], before_k[others])


@pytest.mark.parametrize("V", [1000, 100352])
def test_slot_sampler_equals_the_scalar_sampler_row_by_row(V):
    ops = _ops()
    params = [(0.0, 0, 1.0, 0, 0), (0.8, 200, 1.0, 1, 3), (1.3, 1024, 0.5, 2 ** 63 + 5, 17), (0.0, 0, 1.0, 9, 4),
              (1.0, 50, 0.9, 7, 0), (0.6, 7, 0.95, 123, 2 ** 33 + 1), (1.0, 0, 1.0, 5, 1), (2.0, 1, 1.0, 11, 8)]
    R = len(params)
    g = torch.Generator(device=DEV).manual_seed(V)
    x = (torch.randn(R, V, generator=g, device=DEV) * 2.5).bfloat16()
    x[3, [9, 2]] = x[3].max()                               # a greedy tie
    i64 = lambda vals: torch.tensor([(s - 2 ** 64 if s >= 2 ** 63 else s) for s in vals], dtype=torch.int64, device=DEV)
    temp = torch.tensor([p[0] for p in params], dtype=torch.float32, device=DEV)
    top_k = torch.tensor([p[1] for p in params], dtype=torch.int32, device=DEV)
    top_p = torch.tensor([p[2] for p in params], dtype=torch.float32, device=DEV)
    seed, off = i64([p[3] for p in params]), i64([p[4] for p in params])
    noise = torch.zeros(R, dtype=torch.int32, device=DEV)
    for rep in range(2):                                    # the offsets move on: fresh noise, same rule
        got = ops.sample_tokens_slots(x, temp, top_k, top_p, seed, noise, off + rep)
        for r, (t, k, p, s, o) in enumerate(params):
            want = ops.sample_tokens(x[r:r + 1], t, k, p, s, rng_offset=i64([o + rep]))
            assert int(got[r]) == int(want[0]), (r, rep)


def test_advance_slots_budgets_eos_and_frozen_finished_slots():
    ops = _ops()
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=DEV)
    i64 = lambda v: torch.tensor(v, dtype=torch.int64, device=DEV)
    R, L = 5, 8
    ids_in = i64([[0]] * R)
    out = torch.full((R, L), -7, dtype=torch.int32, device=DEV)
    n_out, max_new = i32([0, 2, 0, 3, 0]), i32([4, 3, 1, 8, 4])
    rope, wpos, kvl = i32([10, 20, 30, 40, 0]), i32([10, 20, 30, 40, -1]), i32([11, 21, 31, 41, 1])
    off = i64([0, 2, 0, 3, 0])
    fin = torch.tensor([0, 0, 0, 0, 1], dtype=torch.uint8, device=DEV)   # slot 4 is idle
    eos, pad = [99, 77], 5
    # step 1: slot 0 emits a plain token, slot 1 its last budgeted one, slot 2 (budget 1) its only one, slot 3 an EOS id
    ops.decode_advance_slots(i64([11, 12, 13, 77, 14]), ids_in, out, n_out, max_new, rope, wpos, kvl, off, fin, eos, pad)
    assert fin.tolist() == [0, 1, 1, 1, 1]
    assert n_out.tolist() == [1, 3, 1, 4, 0]
    assert out[:, :4].tolist() == [[11, -7, -7, -7], [-7, -7, 12, -7], [13, -7, -7, -7], [-7, -7, -7, 77], [-7] * 4]
    assert ids_in.flatten().tolist() == [11, pad, pad, pad, 0]
    assert rope.tolist() == [11, 21, 31, 41, 0] and wpos.tolist() == [11, 21, 31, 41, -1] and kvl.tolist() == [12, 22, 32, 42, 1]
    assert off.tolist() == [1, 3, 1, 4, 0]
    # step 2: the finished and idle slots are frozen, whatever they sampled
    snap = [t.clone() for t in (out, n_out, rope, wpos, kvl, off, fin, ids_in)]
    ops.decode_advance_slots(i64([99, 1, 2, 3, 4]), ids_in, out, n_out, max_new, rope, wpos, kvl, off, fin, eos, pad)
    assert fin.tolist() == [1, 1, 1, 1, 1] and out[0, 1] == 99 and n_out[0] == 2 and rope[0] == 12 and off[0] == 2
    for a, b in zip((out, n_out, rope, wpos, kvl, off, fin, ids_in), snap):
        assert torch.equal(a[1:], b[1:])


# ------------------------------------------------------------------------------------------------ the engine
def _tiny(w8a8=False):
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    sd = C.aria_state(C.TINY, seed=0, dtype=torch.bfloat16)
    m = AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device=DEV)
    m.load_state_dict({k: v.to(DEV) for k, v in sd.items()}, strict=True)
    if w8a8:
        m.quantize_experts_fp8(activations="fp8")
    return m, C.TINY


SAMPLED = dict(do_sample=True, temperature=1.1, top_k=40, top_p=0.95)


def _workload(cfg, n=12, seed=0):
    """n requests: prompts under and over 256 tokens, some with one image (8 image tokens), greedy and sampled, varied budgets."""
    rng = random.Random(seed)
    g = torch.Generator().manual_seed(seed)
    V, img, S = cfg["text_config"]["vocab_size"], cfg["image_token_index"], cfg["vision_config"]["image_size"]
    lengths = [5, 40, 300, 257, 600, 31, 256, 12, 90, 255, 420, 17]
    reqs = []
    for i in range(n):
        T = lengths[i % len(lengths)]
        text = torch.randint(10, V, (T,), generator=g)
        kw = dict(max_new_tokens=rng.choice([1, 3, 9, 17, 30, 41]))
        if i % 3 == 1:
            kw.update(pixel_values=torch.randn(1, 3, S, S, generator=g).bfloat16())
            text = torch.cat([text[:3], torch.full((8,), img), text[3:]])
        if i % 2:
            kw.update(SAMPLED, seed=1000 + i)
        reqs.append((text, kw))
    return reqs


def _reference(m, reqs, eos=None, pad=None):
    return [m.generate(ids[None], kw.get("pixel_values"), None, max_new_tokens=kw["max_new_tokens"],
                       do_sample=kw.get("do_sample", False), temperature=kw.get("temperature", 1.0), top_k=kw.get("top_k", 50),
                       top_p=kw.get("top_p", 1.0), seed=kw.get("seed", 0), eos_token_id=eos, pad_token_id=pad)[0]
            for ids, kw in reqs]


def _eos_from_free_run(m, reqs):
    """EOS ids taken from a free run, as test_eos_pad_and_trim_do_not_depend_on_polling does: the token request 2 emits at
    step 4 and the one request 4 emits at step 10."""
    free = _reference(m, [reqs[2], reqs[4]])
    return [int(free[0][reqs[2][0].numel() + 4]), int(free[1][reqs[4][0].numel() + 10])]


@pytest.fixture(scope="module")
def tiny_case():
    m, cfg = _tiny()
    reqs = _workload(cfg)
    for i in (2, 4):                                    # long enough budgets for the EOS picks
        reqs[i][1]["max_new_tokens"] = 30
    eos = _eos_from_free_run(m, reqs)
    return m, cfg, reqs, eos, _reference(m, reqs, eos, 3)


def _serve(eng, reqs, first=5):
    """Add `first` requests, then one more between every two step() calls -> {request index: result}."""
    ids = {}
    got = {}
    for i, (t, kw) in enumerate(reqs[:first]):
        ids[eng.add_request(t, **kw)] = i
    rest = list(enumerate(reqs))[first:]
    while rest or eng.n_active or eng.n_waiting:
        got.update(eng.step())
        if rest:
            i, (t, kw) = rest.pop(0)
            ids[eng.add_request(t, **kw)] = i
    return {ids[rid]: out for rid, out in got.items()}


@pytest.mark.parametrize("poll_every", [1, 3, 100])
def test_engine_results_equal_batch1_generate(tiny_case, poll_every):
    from aria_b200.serving import Engine
    m, cfg, reqs, eos, want = tiny_case
    assert any(w.numel() < r[0].numel() + r[1]["max_new_tokens"] for w, r in zip(want, reqs))   # some stop at an EOS id
    eng = Engine(m, max_batch=4, max_kv_tokens=64 * PAGE, eos_token_id=eos, pad_token_id=3, poll_every=poll_every)
    got = _serve(eng, reqs)
    assert sorted(got) == list(range(len(reqs)))
    for i, w in enumerate(want):
        assert torch.equal(got[i], w), i
    assert eng.sched.pages.n_free == 64 and eng.n_active == 0
    assert eng.stats["graphs_captured"] >= 2                        # several slot buckets were used


def test_engine_under_pool_pressure_and_graph_reuse(tiny_case):
    from aria_b200.serving import Engine
    m, cfg, reqs, eos, want = tiny_case
    # every request here needs 2 or 3 pages; a pool of 5 holds two of them at a time
    sel = [i for i, (t, kw) in enumerate(reqs) if 257 <= t.numel() + kw["max_new_tokens"] <= 3 * PAGE]
    assert len(sel) >= 4
    eng = Engine(m, max_batch=8, max_kv_tokens=5 * PAGE, eos_token_id=eos, pad_token_id=3, poll_every=3)
    peak = 0
    for i in sel:
        eng.add_request(reqs[i][0], **reqs[i][1])
    got = {}
    while eng.n_active or eng.n_waiting:
        got.update(eng.step())
        peak = max(peak, eng.n_active)
    assert 1 <= peak <= 2
    assert [torch.equal(got[j], want[i]) for j, i in enumerate(sel)] == [True] * len(sel)
    assert eng.sched.pages.n_free == 5
    # the same workload again: every bucket is captured already
    captured = eng.stats["graphs_captured"]
    for i in sel:
        eng.add_request(reqs[i][0], **reqs[i][1])
    again = eng.run()
    assert eng.stats["graphs_captured"] == captured
    assert [torch.equal(again[len(sel) + j], want[i]) for j, i in enumerate(sel)] == [True] * len(sel)


def test_engine_with_w8a8_experts():
    from aria_b200.serving import Engine
    m, cfg = _tiny(w8a8=True)
    reqs = _workload(cfg, n=6, seed=3)
    want = _reference(m, reqs)
    eng = Engine(m, max_batch=4, max_kv_tokens=32 * PAGE, poll_every=4)
    got = _serve(eng, reqs, first=3)
    for i, w in enumerate(want):
        assert torch.equal(got[i], w), i


def _null_page_is_zero(eng):
    return all(not bool(t[0].any()) for t in eng.cache.k + eng.cache.v)


def test_null_page_is_zero_and_idle_rows_stay_finite(tiny_case):
    """Idle rows of a graph bucket attend to one key on the null page 0: it must hold zeros (not allocator leftovers) from the
    engine's construction on, and no step may write it."""
    from aria_b200 import ops
    from aria_b200.serving import Engine
    m, cfg, reqs, eos, want = tiny_case
    lm = m.language_model
    eng = Engine(m, max_batch=4, max_kv_tokens=16 * PAGE, eos_token_id=eos, pad_token_id=3, poll_every=2)
    assert _null_page_is_zero(eng)
    st = eng.state.rows(4)                                  # four idle slots, stepped eagerly
    eng.cache.width = 1
    logits = lm.decode_step(ops.embedding(st.ids_in, lm.get_input_embeddings().weight), eng.cache, st, eng.rope)
    assert bool(torch.isfinite(logits.float()).all())
    assert _null_page_is_zero(eng)
    for t, kw in reqs[:5]:
        eng.add_request(t, **kw)
    got = eng.run()
    assert [torch.equal(got[i], want[i]) for i in range(5)] == [True] * 5
    assert _null_page_is_zero(eng)


def test_failed_admission_is_dropped_and_the_engine_goes_on(tiny_case):
    from aria_b200.serving import Engine
    m, cfg, reqs, eos, want = tiny_case
    img = cfg["image_token_index"]
    bad_ids = torch.cat([torch.arange(10, 20), torch.full((4,), img)])    # 4 image tokens, the image gives 8 features
    bad_pv = reqs[1][1]["pixel_values"]
    eng = Engine(m, max_batch=4, max_kv_tokens=16 * PAGE, eos_token_id=eos, pad_token_id=3, poll_every=3)
    a = eng.add_request(reqs[0][0], **reqs[0][1])
    eng.add_request(bad_ids, bad_pv, max_new_tokens=4)
    c = eng.add_request(reqs[2][0], **reqs[2][1])
    with pytest.raises(ValueError, match="image"):
        eng.step()
    assert eng.n_active == 1 and eng.n_waiting == 1
    got = eng.run()
    assert sorted(got) == [a, c] and torch.equal(got[a], want[0]) and torch.equal(got[c], want[2])
    assert eng.sched.pages.n_free == 16 and eng.n_active == 0
