"""H100: the fp8 KV cache.  The quantizer (store / append) is bit-identical to torch's cast and the dequantizer to torch's
product; the fp8 decode kernels are bit-identical to the bf16 ones on code * scale when the scales are powers of two and stay
close to fp32 attention on random data; on the tiny model an fp8 cache gives the bf16 prefill logits bit for bit, generate()
matches the eager forward() loop, continuation chunks attend to the dequantized rows, and the decode logits stay close to the
bf16 cache's; the cache allocates codes, scales and one staging pair."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
bf16, e4m3 = torch.bfloat16, torch.float8_e4m3fn


def _ops():
    from aria_b200 import build, ops
    build.build()
    return ops


def _bits(q):
    return q.view(torch.uint8)


def _quantize_oracle(x):
    """(x.float() / scale[..., None]).to(float8_e4m3fn) with scale = amax / 448 per row (1 for an all-zero row), on the CPU."""
    x = x.cpu().float()
    amax = x.abs().amax(-1)
    scale = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    return (x / scale[..., None]).to(e4m3), scale


def _empty_cache(B, H, T_max):
    """An fp8 cache of one layer, filled with recognisable values: codes 0x55, scales -1."""
    kc = torch.full((B, H, T_max, 128), 0x55, dtype=torch.uint8, device=DEV).view(e4m3)
    vc = kc.clone()
    ks = torch.full((B, H, T_max), -1.0, device=DEV)
    return kc, vc, ks, ks.clone()


def _crafted_rows(B, H, n, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(2, B, H, n, 128, generator=g, device=DEV)
    x[0, 0, 0, min(3, n - 1)] = 0.0                      # an all-zero row (scale 1)
    x[1, -1, -1, n // 2] = 0.0
    x[0, -1, 0, n - 1, 7] = 448.0 * 64                   # outliers far above the rest of their row
    x[1, 0, -1, 0, 100] = -448.0 * 3
    x[0, 0, -1, n // 3, :] *= 1e-3                       # a small-valued row
    return x.to(bf16)


# ------------------------------------------------------------------------------------------------ 1. quantizer
@pytest.mark.parametrize("B,H,n,row0,T_max", [(1, 2, 10, 3, 16), (2, 20, 3000, 0, 3000), (2, 20, 3000, 17, 3100)],
                         ids=["tiny", "3000-rows", "3000-rows-offset"])
def test_kv_store_bit_identical(B, H, n, row0, T_max):
    ops = _ops()
    x = _crafted_rows(B, H, n, seed=n)
    src = torch.zeros(2, B, H, T_max, 128, dtype=bf16, device=DEV)     # source rows with a row stride of 128 inside a bigger buffer
    src[:, :, :, row0:row0 + n] = x
    kc, vc, ks, vs = _empty_cache(B, H, T_max)
    ops.kv_store_fp8(src[0, :, :, row0:row0 + n], src[1, :, :, row0:row0 + n], kc, vc, ks, vs, row0)
    for i, (c, s) in enumerate(((kc, ks), (vc, vs))):
        wq, ws = _quantize_oracle(x[i])
        assert torch.equal(_bits(c[:, :, row0:row0 + n]).cpu(), _bits(wq)), i
        assert torch.equal(s[:, :, row0:row0 + n].cpu(), ws), i
        assert bool((_bits(c[:, :, :row0]) == 0x55).all()) and bool((_bits(c[:, :, row0 + n:]) == 0x55).all())
        assert bool((s[:, :, :row0] == -1).all()) and bool((s[:, :, row0 + n:] == -1).all())


def test_kv_append_writes_only_the_device_row():
    ops = _ops()
    B, H, T_max = 4, 3, 40
    pos = torch.tensor([0, 17, T_max - 1, T_max + 5], dtype=torch.int32, device=DEV)   # the last row is out of range
    new = _crafted_rows(B, H, 1, seed=5)                                                # [2, B, H, 1, 128]
    kc, vc, ks, vs = _empty_cache(B, H, T_max)
    ops.kv_append_fp8(new[0, :, :, 0], new[1, :, :, 0], kc, vc, ks, vs, pos)
    rc, rv, rks, rvs = _empty_cache(B, H, T_max)
    for b, p in enumerate(pos.tolist()):
        if p < T_max:
            ops.kv_store_fp8(new[0, b:b + 1], new[1, b:b + 1], rc[b:b + 1], rv[b:b + 1], rks[b:b + 1], rvs[b:b + 1], p)
    assert torch.equal(_bits(kc), _bits(rc)) and torch.equal(_bits(vc), _bits(rv))
    assert torch.equal(ks, rks) and torch.equal(vs, rvs)
    assert int((_bits(kc) != 0x55).any(-1).sum()) <= (B - 1) * H      # one row per (b, h) at most, none for b = 3
    assert bool((ks[3] == -1).all()) and bool((_bits(kc[3]) == 0x55).all())


def test_kv_load_bit_identical():
    ops = _ops()
    B, H, T_max, n = 2, 20, 1000, 777
    g = torch.Generator(device=DEV).manual_seed(9)
    codes = torch.randint(0, 256, (2, B, H, T_max, 128), generator=g, device=DEV, dtype=torch.uint8)
    codes[(codes & 0x7F) == 0x7F] = 0                                  # no NaN codes
    scales = torch.rand(2, B, H, T_max, generator=g, device=DEV) * 3 + 1e-3
    out = torch.zeros(2, B, H, T_max + 8, 128, dtype=bf16, device=DEV)
    ops.kv_load_fp8(codes[0].view(e4m3), codes[1].view(e4m3), scales[0], scales[1], out[0], out[1], n)
    want = (codes[..., :n, :].view(e4m3).cpu().float() * scales[..., :n, None].cpu()).bfloat16()
    assert torch.equal(out[..., :n, :].cpu(), want)
    assert bool((out[..., n:, :] == 0).all())


# ------------------------------------------------------------------------------------------------ 2. decode kernels
def _random_fp8_cache(B, H, T_max, g, pow2=True):
    codes = torch.randint(0, 256, (2, B, H, T_max, 128), generator=g, device=DEV, dtype=torch.uint8)
    codes[(codes & 0x7F) == 0x7F] = 0
    if pow2:
        scales = torch.exp2(torch.randint(-9, -3, (2, B, H, T_max), generator=g, device=DEV).float())
    else:
        scales = torch.rand(2, B, H, T_max, generator=g, device=DEV) * 0.01 + 1e-3
    return codes.view(e4m3), scales


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("lens", [[1, 255, 256], [257, 511, 700], [700, 700, 700]])
def test_decode_fp8_bit_identical_to_bf16_with_pow2_scales(lens, masked):
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(3)
    B, H, T_max = 3, 4, 700
    q = torch.randn(B, H, 128, generator=g, device=DEV).bfloat16()
    codes, scales = _random_fp8_cache(B, H, T_max, g)
    kv = (codes.float() * scales[..., None]).bfloat16()              # exact: an e4m3 value times a power of two
    km = None
    if masked:
        km = (torch.rand(B, T_max + 16, generator=g, device=DEV) < 0.3).to(torch.uint8)
        km[:, 0] = 0
    sc = 128 ** -0.5
    want, host = [], []
    for b, n in enumerate(lens):
        m = None if km is None else km[b:b + 1, :n].clone()
        want.append(ops.attention_decode(q[b:b + 1], kv[0, b:b + 1].contiguous(), kv[1, b:b + 1].contiguous(), n, sc, key_mask=m))
        got = ops.attention_decode(q[b:b + 1], codes[0, b:b + 1], codes[1, b:b + 1], n, sc, key_mask=m,
                                   k_scale=scales[0, b:b + 1], v_scale=scales[1, b:b + 1])
        host.append(got)
        assert torch.equal(got, want[-1]), (b, n)
    for b, n in enumerate(lens):                    # rows at or past lens[b] are never read
        codes.view(torch.uint8)[:, b, :, n:] = 0x7F
        scales[:, b, :, n:] = float("nan")
    got = ops.attention_decode_devlen(q, codes[0], codes[1], torch.tensor(lens, dtype=torch.int32, device=DEV), sc, key_mask=km,
                                      k_scale=scales[0], v_scale=scales[1])
    assert torch.equal(got, torch.cat(want))
    assert torch.equal(got, torch.cat(host))


def test_decode_fp8_needs_scales():
    ops = _ops()
    codes = torch.zeros(1, 2, 64, 128, dtype=e4m3, device=DEV)
    q = torch.zeros(1, 2, 128, dtype=bf16, device=DEV)
    with pytest.raises(ValueError):
        ops.attention_decode(q, codes, codes, 10, 0.1)
    with pytest.raises(ValueError):
        ops.attention_decode_devlen(q, codes, codes, torch.ones(1, dtype=torch.int32, device=DEV), 0.1)


def _fp32_attention(q, k, v, n, scale):
    s = torch.einsum("bhd,bhtd->bht", q.float(), k[:, :, :n].float()) * scale
    return torch.einsum("bht,bhtd->bhd", s.softmax(-1), v[:, :, :n].float()).reshape(q.shape[0], -1)


@pytest.mark.parametrize("B,H,n", [(4, 20, 2048), (1, 20, 5000)])
def test_decode_fp8_close_to_fp32(B, H, n):
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(n)
    q = torch.randn(B, H, 128, generator=g, device=DEV).bfloat16()
    kv = torch.randn(2, B, H, n, 128, generator=g, device=DEV).bfloat16()
    kc, vc, ks, vs = _empty_cache(B, H, n)
    ops.kv_store_fp8(kv[0], kv[1], kc, vc, ks, vs, 0)
    sc = 128 ** -0.5
    got = ops.attention_decode(q, kc, vc, n, sc, k_scale=ks, v_scale=vs).float()
    deq = (kc.float() * ks[..., None]), (vc.float() * vs[..., None])
    want = _fp32_attention(q, *deq, n, sc)
    rel = float((got - want).norm() / want.norm())
    orig = _fp32_attention(q, kv[0], kv[1], n, sc)
    rel_orig = float((got - orig).norm() / orig.norm())
    print(f"fp8 decode B={B} n={n}: rel-L2 {rel:.2e} to fp32 over the dequantized K/V, {rel_orig:.2e} over the original K/V")
    assert rel < 1e-2, rel


# ------------------------------------------------------------------------------------------------ 3. tiny model
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


def _forward_loop(m, ids, pv, mask, n, kv_cache_dtype, tokens=None, routes=None):
    """The per-token forward() loop: greedy, or teacher-forced with `tokens` -> (tokens, step logits).  routes[t]: the per-layer
    expert choice forced on step t (t = 0 is the prefill)."""
    B, T = ids.shape
    layers = m.language_model.model.layers

    def force(t):
        if routes is not None:
            for layer, idx in zip(layers, routes[t]):
                layer.mlp.router.forced_top_indices = idx

    force(0)
    inputs = m.prepare_inputs_for_generation(ids, None, pixel_values=pv, attention_mask=mask, num_logits_to_keep=1)
    out = m.forward(**inputs, max_cache_len=T + n, kv_cache_dtype=kv_cache_dtype)
    cache, logits, toks = out.past_key_values, [out.logits[:, -1].clone()], []
    assert cache.dtype == kv_cache_dtype
    all_ids = ids.to(DEV)
    for t in range(n):
        toks.append(logits[-1].float().argmax(-1) if tokens is None else tokens[:, t])
        if t == n - 1:
            break
        all_ids = torch.cat([all_ids, toks[-1].view(B, 1)], dim=1)
        if mask is not None:
            mask = torch.cat([mask, torch.ones(B, 1, dtype=mask.dtype)], dim=1)
        force(t + 1)
        inputs = m.prepare_inputs_for_generation(all_ids, cache, attention_mask=mask, num_logits_to_keep=1)
        logits.append(m.forward(**inputs).logits[:, -1].clone())
    for layer in layers:
        layer.mlp.router.forced_top_indices = None
    return torch.stack(toks, 1), logits


@pytest.mark.parametrize("padded", [False, True])
def test_prefill_logits_bit_identical_to_bf16_cache(padded):
    m, cfg = _tiny()
    ids, pv, mask = _prompts(cfg, padded)
    want = m(input_ids=ids, pixel_values=pv, attention_mask=mask).logits
    out = m(input_ids=ids, pixel_values=pv, attention_mask=mask, kv_cache_dtype="fp8")
    assert out.past_key_values.dtype == "fp8"
    assert torch.equal(out.logits, want)


@pytest.mark.parametrize("experts", [None, "bf16", "fp8"], ids=["bf16-experts", "w8a16", "w8a8"])
@pytest.mark.parametrize("padded", [False, True])
def test_greedy_generate_fp8_equals_forward_loop(padded, experts):
    m, cfg = _tiny()
    if experts is not None:
        m.quantize_experts_fp8(activations=experts)
    ids, pv, mask = _prompts(cfg, padded)
    n = 7
    want, logits = _forward_loop(m, ids, pv, mask, n, "fp8")
    got = m.generate(ids, pv, None, max_new_tokens=n, attention_mask=mask, kv_cache_dtype="fp8")
    assert m._decode_graph.cache.dtype == "fp8"
    assert torch.equal(got[:, :ids.shape[1]].cpu(), ids)
    assert torch.equal(got[:, -n:], want)
    assert torch.equal(m._decode_graph.logits[:, -1], logits[-1])     # the last replayed step's logits, bit for bit


def test_sampled_generate_fp8_reproduces():
    m, cfg = _tiny()
    ids, pv, mask = _prompts(cfg, True)
    kw = dict(max_new_tokens=10, attention_mask=mask, do_sample=True, temperature=0.8, top_k=5, seed=7, kv_cache_dtype="fp8")
    got = m.generate(ids, pv, None, **kw)
    m._decode_graph = None                                            # a fresh capture gives the same tokens
    assert torch.equal(m.generate(ids, pv, None, **kw), got)


def test_bf16_generate_after_fp8_generate():
    m, cfg = _tiny()
    ids, pv, mask = _prompts(cfg, True)
    want = m.generate(ids, pv, None, max_new_tokens=6, attention_mask=mask)
    m.generate(ids, pv, None, max_new_tokens=6, attention_mask=mask, kv_cache_dtype="fp8")
    assert m._decode_graph.key[-1] == "fp8"
    assert torch.equal(m.generate(ids, pv, None, max_new_tokens=6, attention_mask=mask), want)
    assert m._decode_graph.cache.dtype == "bf16"


def test_forward_rejects_mismatched_cache():
    m, cfg = _tiny()
    ids, pv, _ = _prompts(cfg, False)
    out = m(input_ids=ids, pixel_values=pv, kv_cache_dtype="fp8", max_cache_len=ids.shape[1] + 4)
    with pytest.raises(ValueError):
        m(input_ids=ids[:, :1], past_key_values=out.past_key_values, kv_cache_dtype="bf16")


def test_continuation_attends_to_dequantized_rows():
    from aria_b200 import ops
    m, cfg = _tiny()
    g = torch.Generator().manual_seed(4)
    T1, T2 = 37, 21
    ids = torch.randint(10, cfg["text_config"]["vocab_size"], (2, T1 + T2), generator=g)
    c8 = m(input_ids=ids[:, :T1], max_cache_len=T1 + T2, kv_cache_dtype="fp8").past_key_values
    got = m(input_ids=ids[:, T1:], past_key_values=c8).logits
    cb = m(input_ids=ids[:, :T1], max_cache_len=T1 + T2).past_key_values
    for l in range(len(cb.k)):
        ops.kv_load_fp8(c8.k[l], c8.v[l], c8.k_scale[l], c8.v_scale[l], cb.k[l], cb.v[l], T1)
    want = m(input_ids=ids[:, T1:], past_key_values=cb).logits
    assert torch.equal(got, want)


def test_decode_logits_close_to_bf16_cache_with_forced_routing():
    from aria_b200 import ops
    m, cfg = _tiny()
    ids, pv, mask = _prompts(cfg, True)
    n, k = 12, cfg["text_config"]["moe_topk"]
    tokens, _ = _forward_loop(m, ids, pv, mask, n, "bf16")
    routes, step, hooks = [], [], []
    for layer in m.language_model.model.layers:
        hooks.append(layer.mlp.register_forward_pre_hook(
            lambda mod, args: step.append(ops.router_topk(args[0].reshape(-1, args[0].shape[-1]), mod.router.weight, k)[1])))
    _, want = _forward_loop(m, ids, pv, mask, n, "bf16", tokens=tokens)
    for h in hooks:
        h.remove()
    L = len(m.language_model.model.layers)
    routes = [step[i:i + L] for i in range(0, len(step), L)]
    _, got = _forward_loop(m, ids, pv, mask, n, "fp8", tokens=tokens, routes=routes)
    want, got = torch.stack(want[1:]).float(), torch.stack(got[1:]).float()      # the decode steps
    rel = float((got - want).norm() / want.norm())
    print(f"fp8-KV decode logits, routing forced: rel-L2 {rel:.2e} to the bf16 cache's")
    assert rel < 5e-2, rel


# ------------------------------------------------------------------------------------------------ 4. memory
def test_fp8_cache_allocates_codes_scales_and_one_staging_pair():
    from aria_b200 import configs as C
    from aria_b200.moe_lm import AriaMoELMConfig, AriaMoELMForCausalLM
    _ops()
    cfg = C.with_layers(C.ARIA_25B, lm_layers=2, vit_layers=1)["text_config"]
    lm = AriaMoELMForCausalLM(AriaMoELMConfig(**cfg), device="meta")        # the cache needs the config only
    B, T_max, L, H = 4, 4096, 2, cfg["num_attention_heads"]
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    before = torch.cuda.memory_allocated()
    cache = lm.new_cache(B, T_max, DEV, kv_cache_dtype="fp8")
    torch.cuda.synchronize()
    used = torch.cuda.memory_allocated() - before
    rows = B * H * T_max
    codes, scales, bf16_rows = L * 2 * rows * 128, L * 2 * rows * 4, 3 * rows * 128 * 2   # q plus the k / v staging pair
    held = cache.k + cache.v + cache.k_scale + cache.v_scale + [cache.q, cache.k_stage, cache.v_stage]
    assert [t.dtype for t in cache.k + cache.v] == [e4m3] * 2 * L
    assert sum(t.numel() * t.element_size() for t in held) == codes + scales + bf16_rows
    # nothing else is allocated: the caching allocator may hand a tensor a block up to 1 MiB larger than asked for when it
    # reuses a cached segment, far less than any other cache-sized buffer
    assert codes + scales + bf16_rows <= used <= codes + scales + bf16_rows + len(held) * 2 ** 20, (used, codes, scales, bf16_rows)
    bf16_cache = L * 2 * rows * 128 * 2 + rows * 128 * 2
    print(f"fp8 cache {used / 2**20:.1f} MiB, bf16 cache {bf16_cache / 2**20:.1f} MiB")
    del cache, held
