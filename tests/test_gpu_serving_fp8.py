"""GPU: fp8 KV pages in serving.Engine — the paged fp8 decode, append, varlen store and page load kernels bit for bit against the
contiguous fp8 cache's kernels, and the engine end to end on the tiny model: every result equals generate(kv_cache_dtype="fp8")
with its prefill attending to the dequantized keys of its own rows (the engine's rule, patched into AriaAttention.forward
here), for every budget, poll interval, arrival order and cache hit.  All inputs and seeds are fixed."""
import contextlib
import random

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PAGE = 256
SCALE = 128 ** -0.5
E4M3 = torch.float8_e4m3fn
NAN_CODE = 0x7F                                              # e4m3fn NaN


def _ops():
    from aria_b200 import ops
    return ops


def _bf16(shape, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * scale).bfloat16()


def _fp8_pools(n_pages, H):
    """fp8 page pools full of NaN codes and NaN scales, with the null page 0 as PagedKVCache makes it (codes 0, scale 1)."""
    kp = torch.full((n_pages, H, PAGE, 128), NAN_CODE, dtype=torch.uint8, device=DEV).view(E4M3)
    vp = kp.clone()
    ks = torch.full((n_pages, H, PAGE), float("nan"), device=DEV)
    vs = ks.clone()
    for t in (kp, vp):
        t[0].view(torch.uint8).zero_()
    ks[0], vs[0] = 1.0, 1.0
    return kp, vp, ks, vs


def _u8(t):
    return t.view(torch.uint8)


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("R", [1, 5, 64])
def test_paged_fp8_decode_equals_devlen_fp8(R):
    ops = _ops()
    H, max_pages = 4, 6
    T_max = max_pages * PAGE
    base = [1, 255, 256, 257, 1000, 1536, 700, 513]
    lens = [base[i % len(base)] for i in range(R)]
    # a contiguous fp8 cache, quantized by the store kernel (keys and values of varied magnitude per row)
    kc = torch.empty(R, H, T_max, 128, dtype=E4M3, device=DEV)
    vc = torch.empty_like(kc)
    ksc = torch.empty(R, H, T_max, device=DEV)
    vsc = torch.empty_like(ksc)
    k_src = _bf16((R, H, T_max, 128), 1) * torch.logspace(-2, 2, T_max, device=DEV).bfloat16()[None, None, :, None]
    v_src = _bf16((R, H, T_max, 128), 2)
    ops.kv_store_fp8(k_src, v_src, kc, vc, ksc, vsc, 0)
    # the same codes and scales on shuffled, non-monotonic pages; every other page is NaN
    used = [-(-n // PAGE) for n in lens]
    n_pages = sum(used) + 7
    perm = (torch.randperm(n_pages - 1, generator=torch.Generator().manual_seed(R)) + 1).tolist()
    kp, vp, ks, vs = _fp8_pools(n_pages, H)
    table = torch.full((R, max_pages), -1, dtype=torch.int32)
    for r, n in enumerate(used):
        for s in range(n):
            p = perm.pop()
            table[r, s] = p
            rows = slice(s * PAGE, (s + 1) * PAGE)
            _u8(kp)[p], _u8(vp)[p] = _u8(kc)[r, :, rows], _u8(vc)[r, :, rows]
            ks[p], vs[p] = ksc[r, :, rows], vsc[r, :, rows]
    lens_dev = torch.tensor(lens, dtype=torch.int32, device=DEV)
    q = _bf16((R, H, 128), 3)
    got = ops.attention_decode_paged(q, kp, vp, table.to(DEV), lens_dev, SCALE, k_scale=ks, v_scale=vs)
    # the contiguous cache's rows past each length hold NaN too: the devlen kernel must not read them either
    for r, n in enumerate(lens):
        _u8(kc)[r, :, n:] = NAN_CODE
        ksc[r, :, n:] = float("nan")
    want = ops.attention_decode_devlen(q, kc, vc, lens_dev, SCALE, k_scale=ksc, v_scale=vsc)
    assert not want.isnan().any()
    assert torch.equal(got, want)
    # idle rows: one key on the null page -> exact zeros
    idle = torch.full((R, max_pages), -1, dtype=torch.int32, device=DEV)
    idle[:, 0] = 0
    z = ops.attention_decode_paged(q, kp, vp, idle, torch.ones(R, dtype=torch.int32, device=DEV), SCALE, k_scale=ks, v_scale=vs)
    assert not bool(z.any()) and not z.isnan().any()


def test_paged_fp8_append_equals_kv_append_fp8_and_writes_nothing_else():
    ops = _ops()
    R, H, max_pages, n_pages = 6, 3, 3, 10
    new = _bf16((2, R, H, 128), 5) * torch.tensor([1e-3, 1, 30, 0, 2, 400], device=DEV).bfloat16()[None, :, None, None]
    kp, vp, ks, vs = _fp8_pools(n_pages, H)
    table = torch.tensor([[3, 7, 2], [5, -1, -1], [9, 4, 1], [6, 8, -1], [0, -1, -1], [12, -1, -1]], dtype=torch.int32,
                         device=DEV)
    pos = torch.tensor([300, 17, 600, 255, 0, 3], dtype=torch.int32, device=DEV)
    ops.kv_append_paged(new[0], new[1], kp, vp, table, pos, k_scale=ks, v_scale=vs)
    # the contiguous append of the same rows at the same positions
    kc = torch.zeros(R, H, max_pages * PAGE, 128, dtype=E4M3, device=DEV)
    vc = torch.zeros_like(kc)
    ksc = torch.zeros(R, H, max_pages * PAGE, device=DEV)
    vsc = torch.zeros_like(ksc)
    ops.kv_append_fp8(new[0], new[1], kc, vc, ksc, vsc, pos)
    for r in range(4):                                       # rows 4 (null page) and 5 (outside the pool) write nothing
        p = int(pos[r])
        page, row = int(table[r, p // PAGE]), p % PAGE
        for pool, sc, cc, csc, x in ((kp, ks, kc, ksc, new[0]), (vp, vs, vc, vsc, new[1])):
            assert torch.equal(_u8(pool)[page, :, row], _u8(cc)[r, :, p])
            assert torch.equal(sc[page, :, row], csc[r, :, p])
            oracle = (x[r].float() / csc[r, :, p, None]).to(E4M3)
            assert torch.equal(_u8(pool)[page, :, row], _u8(oracle))
    assert bool((ks[6, :, 255] == 1).all())                  # an all-zero row gets scale 1
    # nothing else changes: negative positions, positions past the table's columns, and entries that are the null page, past
    # the pool or unmapped
    before = [_u8(kp).clone(), _u8(vp).clone(), ks.clone(), vs.clone()]
    bad = torch.tensor([[0, n_pages, -1]] * R, dtype=torch.int32, device=DEV)
    cases = [(table, [-1] * R), (table, [3 * PAGE] * R), (bad, [(r % 3) * PAGE + 5 for r in range(R)])]
    for bt, p in cases:
        ops.kv_append_paged(new[0], new[1], kp, vp, bt, torch.tensor(p, dtype=torch.int32, device=DEV), k_scale=ks, v_scale=vs)
    assert torch.equal(_u8(kp), before[0]) and torch.equal(_u8(vp), before[1])
    assert torch.equal(ks.nan_to_num(7.0), before[2].nan_to_num(7.0)) and torch.equal(vs.nan_to_num(7.0), before[3].nan_to_num(7.0))


def test_varlen_fp8_store_round_trips_the_rows_and_writes_only_listed_pages():
    ops = _ops()
    H, n_pages, width = 4, 24, 8
    lens, prefixes = [300, 1, 256, 700, 40], [0, 256, 512, 0, 1024]
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    seg = ops.PackedSegments(cu, prefixes, DEV)
    S = cu[-1]
    k = _bf16((1, H, S, 128), 7) * 3
    v = _bf16((1, H, S, 128), 8)
    k_in, v_in = k.clone(), v.clone()
    perm = (torch.randperm(n_pages - 1, generator=torch.Generator().manual_seed(5)) + 1).tolist()
    table = torch.full((len(lens), width), -1, dtype=torch.int32)
    for b, (n, P) in enumerate(zip(lens, prefixes)):
        used = -(-(P + n) // PAGE) - P // PAGE
        table[b, P // PAGE:P // PAGE + used] = torch.tensor([perm.pop() for _ in range(used)], dtype=torch.int32)
    table[1, 1] = 0                                          # a null page entry is never written
    kp, vp, ks, vs = _fp8_pools(n_pages, H)
    before = [_u8(kp).clone(), _u8(vp).clone()]
    ops.kv_pages_store_varlen(k, v, kp, vp, table.to(DEV), seg, k_scale=ks, v_scale=vs)
    for b, (n, P) in enumerate(zip(lens, prefixes)):
        c = cu[b]
        kc = torch.empty(1, H, n, 128, dtype=E4M3, device=DEV)
        vc = torch.empty_like(kc)
        ksc = torch.empty(1, H, n, device=DEV)
        vsc = torch.empty_like(ksc)
        ops.kv_store_fp8(k_in[:, :, c:c + n].contiguous(), v_in[:, :, c:c + n].contiguous(), kc, vc, ksc, vsc, 0)
        kl, vl = torch.empty(1, H, n, 128, dtype=torch.bfloat16, device=DEV), torch.empty(1, H, n, 128, dtype=torch.bfloat16,
                                                                                             device=DEV)
        ops.kv_load_fp8(kc, vc, ksc, vsc, kl, vl, n)
        assert torch.equal(k[:, :, c:c + n], kl) and torch.equal(v[:, :, c:c + n], vl), b   # the rewritten source rows
        for t in range(n):
            p = P + t
            page, row = int(table[b, p // PAGE]), p % PAGE
            if page == 0:
                continue
            assert torch.equal(_u8(kp)[page, :, row], _u8(kc)[0, :, t]) and torch.equal(_u8(vp)[page, :, row], _u8(vc)[0, :, t])
            assert torch.equal(ks[page, :, row], ksc[0, :, t]) and torch.equal(vs[page, :, row], vsc[0, :, t])
    assert not _u8(kp)[0].any() and not _u8(vp)[0].any() and bool((ks[0] == 1).all())
    listed = set(table[table > 0].tolist())
    for p in range(1, n_pages):
        if p not in listed:
            assert torch.equal(_u8(kp)[p], before[0][p]) and torch.equal(_u8(vp)[p], before[1][p]), p
            assert bool(ks[p].isnan().all()) and bool(vs[p].isnan().all()), p


def test_pages_load_fp8_equals_kv_load_fp8():
    ops = _ops()
    H, n_pages = 5, 9
    src = _bf16((2, n_pages, H, PAGE, 128), 11) * 40
    kp, vp = (torch.empty(n_pages, H, PAGE, 128, dtype=E4M3, device=DEV) for _ in range(2))
    ks, vs = (torch.empty(n_pages, H, PAGE, device=DEV) for _ in range(2))
    ops.kv_store_fp8(src[0], src[1], kp, vp, ks, vs, 0)      # pages as the rows of a [n_pages, H, 256] cache
    pages = torch.tensor([4, 1, 8, 4, 2], dtype=torch.int32, device=DEV)
    k_out = torch.full((6, H, PAGE, 128), float("nan"), dtype=torch.bfloat16, device=DEV)
    v_out = k_out.clone()
    ops.kv_pages_load_fp8(kp, vp, ks, vs, pages, k_out, v_out)
    kl, vl = torch.empty_like(src[0]), torch.empty_like(src[1])
    ops.kv_load_fp8(kp, vp, ks, vs, kl, vl, PAGE)
    idx = pages.long()
    assert torch.equal(k_out[:5], kl[idx]) and torch.equal(v_out[:5], vl[idx])
    assert bool(k_out[5].isnan().all())                      # past the listed pages: untouched


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


@contextlib.contextmanager
def _own_rows_dequantized():
    """AriaAttention.forward's multi-token fp8 branch with the engine's rule: the new rows are quantized into the cache first,
    and the step attends in bf16 to the dequantized values of every row, its own included."""
    from aria_b200 import moe_lm, ops
    orig = moe_lm.AriaAttention.forward

    def forward(self, hidden_states, cache, rope, residual=None, key_mask=None, position_ids=None, hq=None):
        B, T, d = hidden_states.shape
        if cache.dtype != "fp8" or T == 1:
            return orig(self, hidden_states, cache, rope, residual, key_mask, position_ids, hq)
        pos0 = cache.seq_len
        Tk = pos0 + T
        assert Tk <= cache.T_max
        kc, vc = cache.k[self.layer_idx], cache.v[self.layer_idx]
        ks, vs = cache.k_scale[self.layer_idx], cache.v_scale[self.layer_idx]
        q, k_st, v_st = cache.q, cache.k_stage, cache.v_stage
        self._qkv(hidden_states, hq, [q, k_st, v_st], T, pos0, rope, position_ids)
        ops.kv_store_fp8(k_st[:, :, pos0:Tk], v_st[:, :, pos0:Tk], kc, vc, ks, vs, pos0)
        ops.kv_load_fp8(kc, vc, ks, vs, k_st, v_st, Tk)
        o = ops.attention(q[:, :, pos0:], k_st, v_st, T, Tk, self.head_dim ** -0.5, causal=True, key_mask=key_mask)
        return self._o_proj(o, residual)

    moe_lm.AriaAttention.forward = forward
    try:
        yield
    finally:
        moe_lm.AriaAttention.forward = orig


def _reference(m, ids, kw, eos=None, pad=None):
    with _own_rows_dequantized():
        return m.generate(ids[None], kw.get("pixel_values"), kw.get("pixel_mask"), max_new_tokens=kw["max_new_tokens"],
                          do_sample=kw.get("do_sample", False), temperature=kw.get("temperature", 1.0), top_k=kw.get("top_k", 50),
                          top_p=kw.get("top_p", 1.0), seed=kw.get("seed", 0), eos_token_id=eos, pad_token_id=pad,
                          kv_cache_dtype="fp8")[0]


SAMPLED = dict(do_sample=True, temperature=1.1, top_k=40, top_p=0.95)


def _text(cfg, n, seed):
    return torch.randint(10, cfg["text_config"]["vocab_size"], (n,), generator=torch.Generator().manual_seed(seed))


def _workload(cfg, n=12, seed=0):
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
    free = [_reference(m, *reqs[i]) for i in (2, 4)]
    eos = [int(free[0][reqs[2][0].numel() + 2]), int(free[1][reqs[4][0].numel() + 5])]
    return m, cfg, reqs, eos, [_reference(m, ids, kw, eos, 3) for ids, kw in reqs]


def _engine(m, pages=64, **kw):
    from aria_b200.serving import Engine
    return Engine(m, max_batch=kw.pop("max_batch", 8), max_kv_tokens=pages * PAGE, poll_every=kw.pop("poll_every", 3),
                  kv_cache_dtype="fp8", **kw)


@pytest.mark.parametrize("budget,poll_every,burst", [(None, 5, True), (256, 1, True), (512, 3, False), (256, 2, False)])
def test_engine_results_equal_the_reference(tiny_case, budget, poll_every, burst):
    m, cfg, reqs, eos, want = tiny_case
    eng = _engine(m, max_batch=16 if burst else 4, eos_token_id=eos, pad_token_id=3, poll_every=poll_every,
                  max_prefill_tokens=budget)
    assert eng.cache.dtype == "fp8" and eng.cache.k[0].dtype == E4M3
    got = {}
    if burst:
        rids = [eng.add_request(ids, **kw) for ids, kw in reqs]
        got = eng.run()
    else:                                                    # one by one, a step between arrivals
        rids = []
        for ids, kw in reqs:
            rids.append(eng.add_request(ids, **kw))
            got.update(eng.step())
        got.update(eng.run())
    for i, (rid, w) in enumerate(zip(rids, want)):
        assert torch.equal(got[rid], w), (budget, burst, i)
    assert eng.n_active == 0 and eng.sched.pages.n_free == eng.sched.pages.n_pages - 1


@pytest.mark.parametrize("budget", [256, None])
def test_shared_system_prompt_and_image_hit_cached_pages(tiny, budget):
    m, cfg = tiny
    S, img = cfg["vision_config"]["image_size"], cfg["image_token_index"]
    system = _text(cfg, 400, seed=2)
    reqs = [(torch.cat([system, _text(cfg, n, seed=10 + n)]), dict(max_new_tokens=9 + i, **(SAMPLED if i % 2 else {}), seed=i))
            for i, n in enumerate([30, 200, 500])]
    pv = torch.randn(1, 3, S, S, generator=torch.Generator().manual_seed(9)).bfloat16()
    image_prompt = torch.cat([_text(cfg, 300, seed=4), torch.full((8,), img), _text(cfg, 260, seed=5)])
    reqs += [(torch.cat([image_prompt, _text(cfg, n, seed=20 + n)]), dict(pixel_values=pv, max_new_tokens=6, seed=n, **SAMPLED))
             for n in (3, 90)]
    eng = _engine(m, max_prefill_tokens=budget)
    rids = [eng.add_request(ids, **kw) for ids, kw in reqs]
    got = eng.run()
    for i, (rid, (ids, kw)) in enumerate(zip(rids, reqs)):
        assert torch.equal(got[rid], _reference(m, ids, kw)), (budget, i)
    assert eng.stats["prefix_hit_tokens"] == 2 * PAGE + 2 * PAGE
    assert eng.stats["vit_rows_skipped"] == 1


def test_a_chunk_boundary_inside_an_image(tiny):
    m, cfg = tiny
    S, img = cfg["vision_config"]["image_size"], cfg["image_token_index"]
    text = _text(cfg, 600, seed=3)
    ids = torch.cat([text[:252], torch.full((16,), img), text[252:]])      # crop 0: tokens 252-259, crop 1: 260-267
    pv = torch.randn(2, 3, S, S, generator=torch.Generator().manual_seed(4)).bfloat16()
    kw = dict(pixel_values=pv, max_new_tokens=7)
    want = _reference(m, ids, kw)
    for budget in (256, 512):
        eng = _engine(m, max_prefill_tokens=budget)
        rid = eng.add_request(ids, **kw)
        assert torch.equal(eng.run()[rid], want), budget
        assert eng.stats["prefill_launches"] == -(-ids.numel() // budget)


def test_w8a8_experts_and_fp8_dense_projections():
    m, cfg = _tiny(w8a8=True)
    reqs = _workload(cfg, n=6, seed=1)
    eng = _engine(m, max_prefill_tokens=256)
    rids = [eng.add_request(ids, **kw) for ids, kw in reqs]
    got = eng.run()
    for i, (rid, (ids, kw)) in enumerate(zip(rids, reqs)):
        assert torch.equal(got[rid], _reference(m, ids, kw)), i


def test_pool_pressure_returns_every_page_and_the_null_page_stays_zero(tiny_case):
    m, cfg, reqs, eos, want = tiny_case
    eng = _engine(m, pages=9, poll_every=2, eos_token_id=eos, pad_token_id=3, max_prefill_tokens=512)
    sel = [i for i, (ids, kw) in enumerate(reqs) if ids.numel() + kw["max_new_tokens"] <= 9 * PAGE]
    rids = [eng.add_request(reqs[i][0], **reqs[i][1]) for i in sel]
    got = eng.run()
    assert [torch.equal(got[r], want[i]) for r, i in zip(rids, sel)] == [True] * len(sel)
    assert eng.sched.pages.n_free == 9 and all(eng.sched.pages.refs(p) == 0 for p in range(10))
    c = eng.cache
    assert all(not bool(t[0].view(torch.uint8).any()) for t in c.k + c.v)
    assert all(bool((t[0] == 1).all()) for t in c.k_scale + c.v_scale)


# ------------------------------------------------------------------------------------------------ quality
def _forward_loop(m, ids, n, kv_cache_dtype, tokens=None, routes=None):
    """The per-token forward() loop, teacher-forced with `tokens` when given -> (tokens, step logits); routes[t]: the per-layer
    expert choice forced on step t (t = 0 is the prefill)."""
    layers = m.language_model.model.layers

    def force(t):
        if routes is not None:
            for layer, idx in zip(layers, routes[t]):
                layer.mlp.router.forced_top_indices = idx

    B, T = ids.shape
    force(0)
    inputs = m.prepare_inputs_for_generation(ids, None, num_logits_to_keep=1)
    out = m.forward(**inputs, max_cache_len=T + n, kv_cache_dtype=kv_cache_dtype)
    cache, logits, toks = out.past_key_values, [out.logits[:, -1].clone()], []
    all_ids = ids.to(DEV)
    for t in range(n):
        toks.append(logits[-1].float().argmax(-1) if tokens is None else tokens[:, t])
        if t == n - 1:
            break
        all_ids = torch.cat([all_ids, toks[-1].view(B, 1)], dim=1)
        force(t + 1)
        inputs = m.prepare_inputs_for_generation(all_ids, cache, num_logits_to_keep=1)
        logits.append(m.forward(**inputs).logits[:, -1].clone())
    for layer in layers:
        layer.mlp.router.forced_top_indices = None
    return torch.stack(toks, 1), logits


def test_decode_logits_close_to_bf16_cache_with_forced_routing(tiny):
    from aria_b200 import ops
    m, cfg = tiny
    ids = torch.stack([_text(cfg, 300, seed=40), _text(cfg, 300, seed=41)])
    n, k = 12, cfg["text_config"]["moe_topk"]
    tokens, _ = _forward_loop(m, ids, n, "bf16")
    step, hooks = [], []
    for layer in m.language_model.model.layers:
        hooks.append(layer.mlp.register_forward_pre_hook(
            lambda mod, args: step.append(ops.router_topk(args[0].reshape(-1, args[0].shape[-1]), mod.router.weight, k)[1])))
    _, want = _forward_loop(m, ids, n, "bf16", tokens=tokens)
    for h in hooks:
        h.remove()
    L = len(m.language_model.model.layers)
    routes = [step[i:i + L] for i in range(0, len(step), L)]
    with _own_rows_dequantized():
        _, got = _forward_loop(m, ids, n, "fp8", tokens=tokens, routes=routes)
    first = float((got[0].float() - want[0].float()).norm() / want[0].float().norm())
    want, got = torch.stack(want[1:]).float(), torch.stack(got[1:]).float()      # the decode steps
    rel = float((got - want).norm() / want.norm())
    print(f"fp8 KV pages rule, routing forced: first-token logits rel-L2 {first:.2e}, decode logits rel-L2 {rel:.2e} to the "
          "bf16 cache's")
    assert rel < 5e-2, rel


# ------------------------------------------------------------------------------------------------ memory
def test_fp8_paged_cache_allocates_codes_and_scales():
    from aria_b200 import configs as C
    from aria_b200.moe_lm import AriaMoELMConfig, PagedKVCache
    _ops()
    cfg = AriaMoELMConfig(**C.with_layers(C.ARIA_25B, lm_layers=2, vit_layers=1)["text_config"])
    L, H, hd, n_pages, rows, width = 2, cfg.num_attention_heads, cfg.head_dim, 65, 8, 64
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    before = torch.cuda.memory_allocated()
    cache = PagedKVCache(L, n_pages, H, hd, rows, width, DEV, dtype="fp8")
    torch.cuda.synchronize()
    used = torch.cuda.memory_allocated() - before
    codes, scales, table = L * 2 * n_pages * H * PAGE * hd, L * 2 * n_pages * H * PAGE * 4, rows * width * 4
    held = cache.k + cache.v + cache.k_scale + cache.v_scale
    assert [t.dtype for t in cache.k + cache.v] == [E4M3] * 2 * L
    assert sum(t.numel() * t.element_size() for t in held) == codes + scales
    assert codes + scales <= used <= codes + scales + table + (len(held) + 1) * 2 ** 20, (used, codes, scales)
    bf16 = L * 2 * n_pages * H * PAGE * hd * 2
    print(f"fp8 pages {used / 2**20:.1f} MiB, bf16 pages {bf16 / 2**20:.1f} MiB ({bf16 / (codes + scales):.2f}x the tokens)")
    del cache, held
