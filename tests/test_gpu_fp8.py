"""H100: fp8 expert weights.  The quantizer is bit-identical to torch's cast; the fp8 grouped GEMM matches the dequantized
oracle within one bf16 ulp (LINEAR) and is bit-identical to the bf16 kernels when the scales are powers of two, alone, in the
MoE block and through a whole model (forward, greedy and sampled generate); quantization error on the tiny model stays in
the expected range; quantize_experts_fp8() frees the bf16 experts and the cached decode graph."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
bf16, e4m3 = torch.bfloat16, torch.float8_e4m3fn


def _ops():
    from aria_b200 import build, ops
    build.build()
    return ops


def _quantize_oracle(w):
    """(w.float() / scale).to(float8_e4m3fn) with scale = amax / 448 (1 for an all-zero column)."""
    amax = w.float().abs().amax(dim=1)
    scale = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    return (w.float() / scale[:, None, :]).to(e4m3), scale


def _bits(q):
    return q.view(torch.uint8)


# ------------------------------------------------------------------------------------------------ 1. quantizer
@pytest.mark.parametrize("shape", [(64, 2560, 3328), (64, 1664, 2560)], ids=["fc1", "fc2"])
def test_quantizer_bit_identical_full_width(shape):
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(0)
    w = (torch.randn(shape, device=DEV, generator=g) * 0.02).to(bf16)
    q, s = ops.quantize_fp8_cols(w)
    # oracle on the CPU, where torch divides (IEEE) and casts (round to nearest even) elementwise; on CUDA torch divides by a
    # scalar through its reciprocal.  Eight experts at a time.
    for e in range(0, shape[0], 8):
        cq, cs = _quantize_oracle(w[e:e + 8].cpu())
        assert torch.equal(s[e:e + 8].cpu(), cs), e
        assert torch.equal(_bits(q[e:e + 8]).cpu(), _bits(cq)), e


def test_quantizer_crafted_columns():
    ops = _ops()
    G, K, N = 2, 128, 192
    g = torch.Generator().manual_seed(1)
    w = (torch.randn(G, K, N, generator=g) * 0.02)
    w[0, :, 3] = 0.0                                  # all-zero column: scale 1, q 0
    w[1, :, 10] = 1e-6                                # ...
    w[1, 77, 10] = 3.0                                # single outlier: every other entry becomes an e4m3 subnormal or 0
    w[0, :, 100] = torch.linspace(-1, 1, K) * 2.0 ** -12   # values in the subnormal range after scaling
    w[0, 5, 100] = 1.0
    w[1, :, 150] = -w[1, :, 150].abs()               # negative column
    w = w.to(bf16)
    q, s = ops.quantize_fp8_cols(w.to(DEV))
    wq, ws = _quantize_oracle(w)
    assert torch.equal(s.cpu(), ws) and float(ws[0, 3]) == 1.0
    assert torch.equal(_bits(q).cpu(), _bits(wq))
    assert int((_bits(wq)[0, :, 3]).count_nonzero()) == 0
    sub = _bits(wq)[0, :, 100] & 0x78                # exponent field 0: subnormals (and zeros)
    assert int(((sub == 0) & ((_bits(wq)[0, :, 100] & 0x07) != 0)).sum()) > 0


# ------------------------------------------------------------------------------------------------ 2. GEMM vs dequantized oracle
def _offsets(counts):
    off = torch.zeros(len(counts) + 1, dtype=torch.int32)
    off[1:] = torch.tensor(counts, dtype=torch.int64).cumsum(0).to(torch.int32)
    return off


def _row_mix(name, E=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    if name == "decode_b1":                          # 6 groups x 1 row, the rest empty
        counts = [0] * E
        for e in torch.randperm(E, generator=g)[:6].tolist():
            counts[e] = 1
        return counts
    rows = {"b32": 192, "cfg2": 4608, "cfg4": 196608, "ragged": 700}[name]
    counts = torch.bincount(torch.randint(0, E, (rows,), generator=g), minlength=E)
    if name == "ragged":                             # empty groups, 1-row groups, one large group
        z = max(1, E // 16)
        counts[:z] = 0
        counts[z:2 * z] = 1
        counts[2 * z] += 300
    return counts.tolist()


def _ulp_ok(got, want, sum_abs, K):
    """|got - want| <= one bf16 ulp + the fp32 summation-order bound of a K-term dot product (2 K 2^-24 sum |a_k w_k|).  The
    second term only matters where the terms cancel to a value far below their size; elsewhere the check is one ulp."""
    got, want = got.float(), want.float()
    mag = torch.maximum(got.abs(), want.abs()).clamp_min(2.0 ** -120)
    ulp = torch.exp2(torch.floor(torch.log2(mag)) - 7)
    return bool(((got - want).abs() <= ulp + 2 * K * 2.0 ** -24 * sum_abs).all())


def _gemm_case(mix, K, N, swiglu, seed):
    counts = _row_mix(mix, seed=seed)
    E = len(counts)
    g = torch.Generator(device=DEV).manual_seed(seed)
    rows = sum(counts)
    a = torch.randn(rows, K, device=DEV, generator=g).to(bf16)
    w = (torch.randn(E, K, N, device=DEV, generator=g) * 0.02).to(bf16)
    return counts, a, w


@pytest.mark.parametrize("mix", ["decode_b1", "b32", "cfg2", "ragged", "cfg4"])
@pytest.mark.parametrize("swiglu", [False, True], ids=["linear", "swiglu"])
def test_grouped_gemm_fp8_matches_dequantized_oracle(mix, swiglu):
    from oracle import aria_oracle as O
    ops = _ops()
    # full width (fc1: 2560 -> 3328, fc2: 1664 -> 2560); the 196,608-row mix at a narrower width to keep the fp32 oracle short
    K, N = (2560, 3328) if swiglu else (1664, 2560)
    if mix == "cfg4":
        K, N = 256, 384
    counts, a, w = _gemm_case(mix, K, N, swiglu, seed=3)
    q, s = ops.quantize_fp8_cols(w)
    off = _offsets(counts).to(DEV)
    got = ops.grouped_gemm_fp8(a, q, s, off, swiglu=swiglu)
    assert got.shape == (a.shape[0], N // 2 if swiglu else N)
    r0 = 0
    for e, n in enumerate(counts):
        if n == 0:
            continue
        want = ((a[r0:r0 + n].float() @ q[e].float()) * s[e]).to(bf16)
        sum_abs = (a[r0:r0 + n].float().abs() @ q[e].float().abs()) * s[e]
        if swiglu:
            want = O.glu(want)
            diff = (got[r0:r0 + n].float() - want.float()).abs().max()
            assert diff <= 1e-2 * max(1.0, float(want.float().abs().max())), (e, float(diff))
        else:
            assert _ulp_ok(got[r0:r0 + n], want, sum_abs, K), e
        r0 += n


# ------------------------------------------------------------------------------------------------ 3. power-of-two bit identity
def _pow2_weights(E, K, N, seed):
    """q covering every finite e4m3 code (subnormals and -0 included), power-of-two column scales, w = q * scale (exact)."""
    g = torch.Generator().manual_seed(seed)
    codes = torch.tensor([c for c in range(256) if c not in (0x7F, 0xFF)], dtype=torch.uint8)
    idx = torch.randint(0, codes.numel(), (E, K, N), generator=g)
    idx.view(-1)[:codes.numel()] = torch.arange(codes.numel())
    q = codes[idx].view(e4m3)
    scale = torch.exp2(torch.randint(-14, -6, (E, N), generator=g).float())
    w = (q.to(bf16) * scale[:, None, :].to(bf16))
    assert torch.equal(w.float(), q.float() * scale[:, None, :])
    return q.to(DEV), scale.to(DEV), w.to(DEV)


@pytest.mark.parametrize("mix", ["ragged", "cfg2"])        # cfg2: many tiles per persistent CTA
@pytest.mark.parametrize("swiglu", [False, True], ids=["linear", "swiglu"])
def test_pow2_scales_bit_identical_to_bf16_gemm(swiglu, mix):
    ops = _ops()
    K, N = (512, 1024) if swiglu else (512, 512)
    counts = _row_mix(mix, E=64, seed=5)
    q, s, w = _pow2_weights(64, K, N, seed=6)
    a = torch.randn(sum(counts), K, generator=torch.Generator().manual_seed(7)).to(bf16).to(DEV)
    off = _offsets(counts).to(DEV)
    got = ops.grouped_gemm_fp8(a, q, s, off, swiglu=swiglu)
    want = ops.grouped_gemm(a, w, off, swiglu=swiglu)
    assert torch.equal(got, want)


def test_pow2_scales_bit_identical_moe_block():
    ops = _ops()
    T, d, E, k, I, Is = 96, 256, 8, 2, 512, 1024
    g = torch.Generator().manual_seed(8)
    x = torch.randn(T, d, generator=g).to(bf16).to(DEV)
    wr = (torch.randn(E, d, generator=g) * 0.05).to(bf16).to(DEV)
    q1, s1, w1 = _pow2_weights(E, d, 2 * I, seed=9)
    q2, s2, w2 = _pow2_weights(E, I, d, seed=10)
    gw, uw, dw = [(torch.randn(*sh, generator=g) * 0.02).to(bf16).to(DEV) for sh in ((Is, d), (Is, d), (d, Is))]
    want = ops.moe_block_fwd(x, wr, w1, w2, gw, uw, dw, k)
    got = ops.moe_block_fwd(x, wr, q1, q2, gw, uw, dw, k, fc1_scale=s1, fc2_scale=s2)
    assert torch.equal(got, want)


def _tiny(sd=None):
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    _ops()
    sd = sd if sd is not None else C.aria_state(C.TINY, seed=0, dtype=torch.bfloat16)
    m = AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device=DEV)
    m.load_state_dict({k: v.to(DEV) for k, v in sd.items()}, strict=True)
    return m, C.TINY


def _prompts(cfg, padded):
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


def _experts(m):
    return [layer.mlp.experts for layer in m.language_model.model.layers]


def test_pow2_scales_bit_identical_whole_model():
    from oracle import configs as C
    sd = C.aria_state(C.TINY, seed=0, dtype=torch.bfloat16)
    fp8_sd = {}
    for i, key in enumerate(sorted(k for k in sd if ".experts.fc" in k)):
        E, K, N = sd[key].shape
        q, s, w = _pow2_weights(E, K, N, seed=20 + i)
        sd[key] = w.cpu()
        fp8_sd[key], fp8_sd[key.replace(".weight", ".weight_scale")] = q, s
    ref, cfg = _tiny(sd)
    m, _ = _tiny(sd)
    m.quantize_experts_fp8()                         # real quantizer, then overwritten by the power-of-two tensors
    full = m.state_dict()
    full.update(fp8_sd)
    m.load_state_dict(full, strict=True)
    ids, pv, mask = _prompts(cfg, True)
    assert torch.equal(m(input_ids=ids, pixel_values=pv, attention_mask=mask).logits,
                       ref(input_ids=ids, pixel_values=pv, attention_mask=mask).logits)
    for kw in (dict(), dict(do_sample=True, temperature=0.8, top_k=5, seed=3)):
        assert torch.equal(m.generate(ids, pv, None, max_new_tokens=6, attention_mask=mask, **kw),
                           ref.generate(ids, pv, None, max_new_tokens=6, attention_mask=mask, **kw))


# ------------------------------------------------------------------------------------------------ 4. quantization error
def test_fp8_logits_close_to_bf16_with_forced_routing():
    from aria_b200 import ops
    ref, cfg = _tiny()
    ids, pv, _ = _prompts(cfg, False)
    k = cfg["text_config"]["moe_topk"]
    routes, hooks = [], []
    for layer in ref.language_model.model.layers:
        mlp = layer.mlp
        hooks.append(mlp.register_forward_pre_hook(
            lambda mod, args: routes.append(ops.router_topk(args[0].reshape(-1, args[0].shape[-1]), mod.router.weight, k)[1])))
    want = ref(input_ids=ids, pixel_values=pv).logits.float()
    for h in hooks:
        h.remove()
    m, _ = _tiny()
    m.quantize_experts_fp8()
    for layer, idx in zip(m.language_model.model.layers, routes):
        layer.mlp.router.forced_top_indices = idx
    got = m(input_ids=ids, pixel_values=pv).logits.float()
    rel = float((got - want).norm() / want.norm())
    assert rel < 5e-2, rel


@pytest.mark.parametrize("padded", [False, True])
def test_fp8_generate_equals_forward_loop(padded):
    m, cfg = _tiny()
    m.quantize_experts_fp8()
    ids, pv, mask = _prompts(cfg, padded)
    n = 7
    B, T = ids.shape
    inputs = m.prepare_inputs_for_generation(ids, None, pixel_values=pv, attention_mask=mask, num_logits_to_keep=1)
    out = m.forward(**inputs, max_cache_len=T + n)
    cache, toks, all_ids, msk = out.past_key_values, [out.logits[:, -1].float().argmax(-1)], ids.to(DEV), mask
    for _ in range(n - 1):
        all_ids = torch.cat([all_ids, toks[-1].view(B, 1)], dim=1)
        if msk is not None:
            msk = torch.cat([msk, torch.ones(B, 1, dtype=msk.dtype)], dim=1)
        inputs = m.prepare_inputs_for_generation(all_ids, cache, attention_mask=msk, num_logits_to_keep=1)
        toks.append(m.forward(**inputs).logits[:, -1].float().argmax(-1))
    got = m.generate(ids, pv, None, max_new_tokens=n, attention_mask=mask)
    assert torch.equal(got[:, -n:], torch.stack(toks, 1))


# ------------------------------------------------------------------------------------------------ 5. memory and lifecycle
def test_quantize_frees_the_bf16_experts_full_width():
    from aria_b200 import configs as C
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration, init_random_
    _ops()
    cfg = C.with_layers(C.ARIA_25B, lm_layers=2, vit_layers=1)
    m = AriaForConditionalGeneration(AriaConfig.from_dict(cfg), device=DEV)
    init_random_(m, seed=0)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    m.quantize_experts_fp8()
    torch.cuda.synchronize()
    after = torch.cuda.memory_allocated()
    # per layer and expert: fc1 + fc2 drop from 2 to 1 byte per weight (12.78 MB saved) and gain (3328 + 2560) fp32 scales
    saved = 2 * 64 * ((2560 * 3328 + 1664 * 2560) - (3328 + 2560) * 4)
    assert before - after >= saved, (before, after, saved)
    del m
    torch.cuda.empty_cache()


def test_generate_before_and_after_quantizing():
    m, cfg = _tiny()
    ids, pv, mask = _prompts(cfg, True)
    m.generate(ids, pv, None, max_new_tokens=5, attention_mask=mask)      # captures a bf16 decode graph
    m.quantize_experts_fp8()
    fresh, _ = _tiny()
    fresh.quantize_experts_fp8()
    want = fresh.generate(ids, pv, None, max_new_tokens=5, attention_mask=mask)
    assert torch.equal(m.generate(ids, pv, None, max_new_tokens=5, attention_mask=mask), want)
