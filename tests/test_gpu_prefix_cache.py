"""GPU: prefix caching in serving.Engine — the paged-prefix prefill kernel bit for bit against the contiguous shared-prefix one
(and the varlen forward at P = 0), the per-row invariance of the ViT that partial image hits rely on, and the engine end to end
on the tiny model: every request's result equals batch-1 generate() bit for bit, whatever it shared with the requests before
it.  All inputs and seeds are fixed, so every test is deterministic."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PAGE = 256
SCALE = 128 ** -0.5
LENS = [1, 17, 128, 129, 700]


def _ops():
    from aria_b200 import ops
    return ops


def _bf16(shape, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(*shape, generator=g, device=DEV).bfloat16()


def _paged_case(P, S, H, seed):
    """Packed suffixes S with NaN staging rows past S_tot, a contiguous prefix of P keys, and the same prefix on shuffled,
    non-monotonic pages of a pool whose other pages hold NaN -> (qkv, cu, pre_k, pre_v, k_pool, v_pool, pages)."""
    S_tot = sum(S)
    cu = [0]
    for s in S:
        cu.append(cu[-1] + s)
    qkv = _bf16((3, 1, H, S_tot + 50, 128), seed)
    qkv[:, :, :, S_tot:] = float("nan")
    pre_k, pre_v = _bf16((1, H, max(P, PAGE), 128), seed + 1), _bf16((1, H, max(P, PAGE), 128), seed + 2)
    n = P // PAGE
    n_pages = n + 7
    perm = torch.randperm(n_pages, generator=torch.Generator().manual_seed(seed))[:n]
    kp = torch.full((n_pages, H, PAGE, 128), float("nan"), dtype=torch.bfloat16, device=DEV)
    vp = torch.full_like(kp, float("nan"))
    for i in range(n):
        kp[perm[i]] = pre_k[0, :, i * PAGE:(i + 1) * PAGE]
        vp[perm[i]] = pre_v[0, :, i * PAGE:(i + 1) * PAGE]
    pages = torch.full((n + 3,), -1, dtype=torch.int32)
    pages[:n] = perm.to(torch.int32)
    return qkv, torch.tensor(cu, dtype=torch.int32, device=DEV), pre_k, pre_v, kp, vp, pages.to(DEV)


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("P", [0, 256, 512, 1280, 4096])
def test_paged_prefix_kernel_bit_identical_to_the_contiguous_prefix(P, B):
    ops = _ops()
    H = 4
    groups = [[s] for s in LENS] if B == 1 else [LENS[i:i + 3] for i in range(0, len(LENS), 2)]
    for g, S in enumerate(groups):
        qkv, cu, pre_k, pre_v, kp, vp, pages = _paged_case(P, S, H, seed=P + 10 * B + g)
        S_tot = sum(S)
        got = ops.attention_prefill_paged_prefix(qkv[0], qkv[1], qkv[2], S_tot, kp, vp, pages, P, cu, SCALE)
        if P:
            want = ops.attention_prefill_shared_prefix(qkv[0], qkv[1], qkv[2], S_tot, pre_k, pre_v, P, cu, SCALE)
        else:
            want = ops.attention_varlen(qkv[0], qkv[1], qkv[2], cu, SCALE, N=S_tot)
        assert got.shape == (S_tot, H * 128) and not got.isnan().any(), S
        assert torch.equal(got, want), S


def test_paged_prefix_kernel_refusals():
    ops = _ops()
    qkv, cu, _, _, kp, vp, pages = _paged_case(512, [5], 2, seed=1)
    for bad in (100, 256 * 6, -256):
        with pytest.raises(ValueError):
            ops.attention_prefill_paged_prefix(qkv[0], qkv[1], qkv[2], 5, kp, vp, pages, bad, cu, SCALE)
    with pytest.raises(ValueError):
        ops.attention_prefill_paged_prefix(qkv[0], qkv[1], qkv[2], 5, kp, vp, None, 256, cu, SCALE)


# ------------------------------------------------------------------------------------------------ tiny model
def _tiny(w8a8=False):
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    sd = C.aria_state(C.TINY, seed=0, dtype=torch.bfloat16)
    m = AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device=DEV)
    m.load_state_dict({k: v.to(DEV) for k, v in sd.items()}, strict=True)
    if w8a8:
        m.quantize_experts_fp8(activations="fp8")
    return m, C.TINY


@pytest.fixture(scope="module")
def tiny():
    return _tiny()


def _text(cfg, n, seed):
    return torch.randint(10, cfg["text_config"]["vocab_size"], (n,), generator=torch.Generator().manual_seed(seed))


def _pixels(cfg, rows, seed):
    s = cfg["vision_config"]["image_size"]
    return torch.randn(rows, 3, s, s, generator=torch.Generator().manual_seed(seed)).bfloat16()


def _with_image(cfg, text, at, rows):
    """text with rows x 8 image tokens inserted at position `at`."""
    return torch.cat([text[:at], torch.full((8 * rows,), cfg["image_token_index"]), text[at:]])


SAMPLED = dict(do_sample=True, temperature=1.1, top_k=40, top_p=0.95)


def _generate(m, ids, kw, eos=None, pad=None):
    return m.generate(ids[None], kw.get("pixel_values"), kw.get("pixel_mask"), max_new_tokens=kw["max_new_tokens"],
                      do_sample=kw.get("do_sample", False), temperature=kw.get("temperature", 1.0), top_k=kw.get("top_k", 50),
                      top_p=kw.get("top_p", 1.0), seed=kw.get("seed", 0), eos_token_id=eos, pad_token_id=pad)[0]


def _engine(m, pages=64, **kw):
    from aria_b200.serving import Engine
    return Engine(m, max_batch=kw.pop("max_batch", 4), max_kv_tokens=pages * PAGE, poll_every=kw.pop("poll_every", 3), **kw)


def _serve(eng, reqs, one_by_one=True):
    """Submit reqs [(ids, kw)], each after the previous one has finished (one_by_one) or all at once -> results in order."""
    got = []
    if one_by_one:
        for ids, kw in reqs:
            rid = eng.add_request(ids, **kw)
            got.append(eng.run()[rid])
        return got
    rids = [eng.add_request(ids, **kw) for ids, kw in reqs]
    out = eng.run()
    return [out[r] for r in rids]


def _check(m, eng, reqs, got, eos=None, pad=None):
    for i, ((ids, kw), g) in enumerate(zip(reqs, got)):
        assert torch.equal(g, _generate(m, ids, kw, eos, pad)), i
    assert eng.n_active == 0 and eng.sched.pages.n_free == eng.sched.pages.n_pages - 1


def test_vit_rows_do_not_depend_on_the_rows_beside_them(tiny):
    m, cfg = tiny
    pv = _pixels(cfg, 4, seed=1).to(DEV)
    s = cfg["vision_config"]["image_size"]
    mask = torch.ones(4, s, s, dtype=torch.bool)
    mask[2, :, 28:] = False                                         # one padded crop among full ones
    for pm in (None, mask):
        feats, am = m.vision_tower(pv, pm)
        full = m.multi_modal_projector(feats, am)
        for r0 in (1, 2, 3):
            f, a = m.vision_tower(pv[r0:], None if pm is None else pm[r0:])
            assert torch.equal(m.multi_modal_projector(f, a), full[r0:]), (pm is None, r0)


@pytest.mark.parametrize("one_by_one", [True, False])
def test_shared_system_prompt(tiny, one_by_one):
    m, cfg = tiny
    system = _text(cfg, 400, seed=2)
    reqs = [(torch.cat([system, _text(cfg, n, seed=10 + n)]), dict(max_new_tokens=9 + i, **(SAMPLED if i % 2 else {}), seed=i))
            for i, n in enumerate([1, 30, 200, 500, 113])]
    eng = _engine(m)
    got = _serve(eng, reqs, one_by_one)
    _check(m, eng, reqs, got)
    assert eng.stats["prefix_hit_tokens"] == 4 * PAGE          # page 0 (tokens 0-255) for every request after the first
    assert eng.stats["prompt_tokens"] == sum(r[0].numel() for r in reqs)


def test_identical_prompts_greedy_and_sampled(tiny):
    m, cfg = tiny
    ids = _text(cfg, 700, seed=3)
    reqs = [(ids, dict(max_new_tokens=12))] + [(ids, dict(max_new_tokens=12, seed=s, **SAMPLED)) for s in (1, 2, 3)]
    eng = _engine(m)
    got = _serve(eng, reqs, one_by_one=False)
    _check(m, eng, reqs, got)
    assert eng.stats["prefix_hit_tokens"] == 3 * 2 * PAGE     # 2 full pages each, the third page holds the last token


def test_multi_turn_conversation(tiny):
    m, cfg = tiny
    eng = _engine(m)
    prompt = _text(cfg, 300, seed=4)
    hits = []
    for turn in range(4):
        kw = dict(max_new_tokens=40)
        before = eng.stats["prefix_hit_tokens"]
        out = _serve(eng, [(prompt, kw)])[0]
        assert torch.equal(out, _generate(m, prompt, kw)), turn
        hits.append(eng.stats["prefix_hit_tokens"] - before)
        prompt = torch.cat([out.cpu(), _text(cfg, 60 + 50 * turn, seed=20 + turn)])
    # each turn hits the full pages the previous turn's prompt prefilled (decode-written pages are never keyed)
    assert hits[0] == 0 and all(h >= PAGE for h in hits[1:])


def test_image_straddling_the_hit_boundary_runs_the_vit_on_its_last_crop(tiny):
    m, cfg = tiny
    text = _text(cfg, 700, seed=5)
    ids = _with_image(cfg, text, 500, rows=2)                       # crop 0: tokens 500-507, crop 1: 508-515
    pv = _pixels(cfg, 2, seed=6)
    first = (ids, dict(pixel_values=pv, max_new_tokens=5))
    second = (torch.cat([ids[:600], _text(cfg, 30, seed=7)]), dict(pixel_values=pv, max_new_tokens=7, seed=4, **SAMPLED))
    eng = _engine(m)
    got = _serve(eng, [first])
    run, skipped = eng.stats["vit_rows_run"], eng.stats["vit_rows_skipped"]
    got += _serve(eng, [second])
    _check(m, eng, [first, second], got)
    assert eng.stats["prefix_hit_tokens"] == 2 * PAGE
    assert (run, skipped) == (2, 0) and (eng.stats["vit_rows_run"], eng.stats["vit_rows_skipped"]) == (3, 1)


def test_images_wholly_inside_the_hit_skip_the_vit(tiny):
    m, cfg = tiny
    ids = _with_image(cfg, _text(cfg, 600, seed=8), 20, rows=2)
    pv = _pixels(cfg, 2, seed=9)
    s = cfg["vision_config"]["image_size"]
    pm = torch.ones(2, s, s, dtype=torch.bool)
    pm[1, 42:] = False
    reqs = [(torch.cat([ids, _text(cfg, n, seed=30 + n)]), dict(pixel_values=pv, pixel_mask=pm, max_new_tokens=6)) for n in (3, 90)]
    eng = _engine(m)
    got = _serve(eng, reqs)
    _check(m, eng, reqs, got)
    assert eng.stats["vit_rows_run"] == 2 and eng.stats["vit_rows_skipped"] == 2
    assert eng.stats["prefix_hit_tokens"] == 2 * PAGE


def test_same_ids_with_another_image_share_nothing(tiny):
    m, cfg = tiny
    ids = _with_image(cfg, _text(cfg, 600, seed=10), 5, rows=1)
    s = cfg["vision_config"]["image_size"]
    pm = torch.ones(1, s, s, dtype=torch.bool)
    pm[0, :, 50:] = False
    reqs = [(ids, dict(pixel_values=_pixels(cfg, 1, seed=11), max_new_tokens=5)),
            (ids, dict(pixel_values=_pixels(cfg, 1, seed=12), max_new_tokens=5)),
            (ids, dict(pixel_values=_pixels(cfg, 1, seed=11), pixel_mask=pm, max_new_tokens=5))]
    eng = _engine(m)
    got = _serve(eng, reqs)
    _check(m, eng, reqs, got)
    assert eng.stats["prefix_hit_tokens"] == 0 and eng.stats["vit_rows_skipped"] == 0


def test_pool_pressure_evicts_cached_pages(tiny):
    m, cfg = tiny
    bases = [_text(cfg, 520, seed=40 + i) for i in range(3)]
    reqs = [(torch.cat([bases[i % 3], _text(cfg, 20, seed=50 + i)]), dict(max_new_tokens=30)) for i in range(9)]
    eng = _engine(m, pages=7, poll_every=2)                         # 3 pages per request: two at a time
    got = _serve(eng, reqs, one_by_one=False)
    _check(m, eng, reqs, got)
    assert eng.stats["pages_evicted"] > 0 and eng.stats["prefix_hit_tokens"] > 0


def test_w8a8_experts():
    m, cfg = _tiny(w8a8=True)
    system = _text(cfg, 300, seed=13)
    reqs = [(torch.cat([system, _text(cfg, n, seed=60 + n)]), dict(max_new_tokens=8, seed=n, **SAMPLED)) for n in (5, 70, 300)]
    eng = _engine(m)
    got = _serve(eng, reqs, one_by_one=False)
    _check(m, eng, reqs, got)
    assert eng.stats["prefix_hit_tokens"] == 2 * PAGE


def test_eos_and_pad(tiny):
    m, cfg = tiny
    system = _text(cfg, 520, seed=14)
    reqs = [(torch.cat([system, _text(cfg, n, seed=70 + n)]), dict(max_new_tokens=25, seed=n, **SAMPLED)) for n in (4, 40, 9)]
    free = _generate(m, reqs[1][0], reqs[1][1])
    eos = [int(free[reqs[1][0].numel() + 6])]
    eng = _engine(m, eos_token_id=eos, pad_token_id=3)
    got = _serve(eng, reqs, one_by_one=False)
    _check(m, eng, reqs, got, eos, 3)
    assert got[1].numel() < reqs[1][0].numel() + 25


def _prompt_kv(eng, rid):
    req = next(r for r in eng.sched.slots if r.rid == rid)
    T = req.input_ids.numel()
    return [torch.cat([pool[p] for p in req.pages], dim=1)[:, :T] for pool in eng.cache.k + eng.cache.v]


def test_pages_a_hit_computed_equal_those_of_a_fresh_engine(tiny):
    m, cfg = tiny
    ids = _with_image(cfg, _text(cfg, 900, seed=15), 250, rows=2)   # an image across the page boundary at 256
    pv = _pixels(cfg, 2, seed=16)
    other = torch.cat([ids[:700], _text(cfg, 111, seed=17)])
    eng = _engine(m)
    eng.add_request(ids, pv, max_new_tokens=4)
    eng.step()
    rid = eng.add_request(other, pv, max_new_tokens=4)
    eng.step()
    assert eng.stats["prefix_hit_tokens"] == 2 * PAGE
    hit = _prompt_kv(eng, rid)
    fresh = _engine(m)
    rid2 = fresh.add_request(other, pv, max_new_tokens=4)
    fresh.step()
    assert fresh.stats["prefix_hit_tokens"] == 0
    assert all(torch.equal(a, b) for a, b in zip(hit, _prompt_kv(fresh, rid2)))
    eng.run()
    fresh.run()
