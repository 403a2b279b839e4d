"""H100: fp8 activations and weights (W8A8) for the routed experts.  The row quantizer is bit-identical to torch's cast; with
small integer codes and power-of-two scales the W8A8 GEMM is bit-identical to the bf16 GEMM on the dequantized operands
(layout, both scales, group boundaries and the k-block promotion); on random data it matches the fp32 oracle of the dequantized
operands; the re-layout keeps codes, scales, state dict and memory; the one-call block equals the per-kernel path; a whole tiny
model stays close to bf16, replays its graphs exactly and generates what its forward loop generates."""
import pytest
import torch

from test_gpu_fp8 import _offsets, _prompts, _row_mix, _tiny, _ulp_ok
from test_gpu_generate import _forward_loop

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
bf16, e4m3 = torch.bfloat16, torch.float8_e4m3fn


def _ops():
    from aria_b200 import build, ops
    build.build()
    return ops


def _rows_oracle(x):
    """(x.float() / scale[:, None]).to(float8_e4m3fn) with scale = row amax / 448 (1 for an all-zero row), on the CPU."""
    amax = x.float().abs().amax(dim=1)
    scale = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    return (x.float() / scale[:, None]).to(e4m3), scale


def _bits(q):
    return q.view(torch.uint8)


def _kmajor(q):
    """[E, K, N] codes as the transpose(1, 2) view of a contiguous [E, N, K] buffer (the W8A8 parameter layout)."""
    return q.transpose(1, 2).contiguous().transpose(1, 2)


# ------------------------------------------------------------------------------------------------ 1. row quantizer
@pytest.mark.parametrize("d,gather", [(2560, True), (1664, False)])
def test_row_quantizer_bit_identical_full_width(d, gather):
    ops = _ops()
    g = torch.Generator().manual_seed(0)
    x = torch.randn(4608, d, generator=g).mul(torch.rand(4608, 1, generator=g) * 4).to(bf16)
    src = torch.randint(0, 4608, (6 * 768,), generator=g, dtype=torch.int32) if gather else None
    q, s = ops.permute_quantize_fp8(x.to(DEV), None if src is None else src.to(DEV))
    wq, ws = _rows_oracle(x if src is None else x[src.long()])
    assert torch.equal(s.cpu(), ws)
    assert torch.equal(_bits(q).cpu(), _bits(wq))


def test_row_quantizer_crafted_rows():
    ops = _ops()
    x = torch.randn(6, 256, generator=torch.Generator().manual_seed(1)) * 0.02
    x[0] = 0.0                                                   # all zero: scale 1, codes 0
    x[1] = 1e-6
    x[1, 77] = 3.0                                               # single outlier: the rest becomes subnormal or 0
    x[2] = torch.linspace(-1, 1, 256) * 2.0 ** -12               # subnormal range after scaling
    x[2, 5] = 1.0
    x[3] = -x[3].abs()                                           # negative row
    x[4] = -0.0
    x = x.to(bf16)
    q, s = ops.permute_quantize_fp8(x.to(DEV))
    wq, ws = _rows_oracle(x)
    assert torch.equal(s.cpu(), ws) and float(ws[0]) == 1.0 and float(ws[4]) == 1.0
    assert torch.equal(_bits(q).cpu(), _bits(wq))
    sub = _bits(wq)[2] & 0x78
    assert int(((sub == 0) & ((_bits(wq)[2] & 0x07) != 0)).sum()) > 0


# ------------------------------------------------------------------------------------------------ 2. GEMM bit identity
def _int_codes(shape, g):
    return torch.randint(-3, 4, shape, generator=g).float().to(e4m3)


@pytest.mark.parametrize("mix", ["decode_b1", "b32", "cfg2", "ragged", "cfg4"])
@pytest.mark.parametrize("swiglu", [False, True], ids=["linear", "swiglu"])
def test_int_codes_bit_identical_to_bf16_gemm(mix, swiglu):
    """Codes in [-3, 3] and power-of-two scales make every partial sum exact, in the tensor core and in fp32."""
    ops = _ops()
    K, N = (2560, 3328) if swiglu else (1664, 2560)
    if mix == "cfg4":
        K, N = 256, 384 if not swiglu else 512
    counts = _row_mix(mix, seed=11)
    rows, E = sum(counts), len(counts)
    g = torch.Generator().manual_seed(12)
    aq = _int_codes((rows, K), g)
    a_s = torch.exp2(torch.randint(-8, 0, (rows,), generator=g).float())
    wq = _int_codes((E, K, N), g)
    w_s = torch.exp2(torch.randint(-10, -4, (E, N), generator=g).float())
    a_deq = (aq.float() * a_s[:, None]).to(bf16)
    w_deq = (wq.float() * w_s[:, None, :]).to(bf16)
    off = _offsets(counts).to(DEV)
    got = ops.grouped_gemm_w8a8(aq.to(DEV), a_s.to(DEV), _kmajor(wq.to(DEV)), w_s.to(DEV), off, swiglu=swiglu)
    want = ops.grouped_gemm(a_deq.to(DEV), w_deq.to(DEV), off, swiglu=swiglu)
    assert torch.equal(got, want)


# ------------------------------------------------------------------------------------------------ 3. GEMM vs fp32 oracle
@pytest.mark.parametrize("mix", ["decode_b1", "b32", "cfg2", "ragged"])
@pytest.mark.parametrize("swiglu", [False, True], ids=["linear", "swiglu"])
def test_gemm_matches_dequantized_oracle(mix, swiglu):
    from oracle import aria_oracle as O
    ops = _ops()
    K, N = (2560, 3328) if swiglu else (1664, 2560)
    counts = _row_mix(mix, seed=3)
    E = len(counts)
    g = torch.Generator(device=DEV).manual_seed(3)
    a = torch.randn(sum(counts), K, device=DEV, generator=g).to(bf16)
    w = (torch.randn(E, K, N, device=DEV, generator=g) * 0.02).to(bf16)
    q, s = ops.quantize_fp8_cols(w)
    aq, a_s = ops.permute_quantize_fp8(a)
    off = _offsets(counts).to(DEV)
    got = ops.grouped_gemm_w8a8(aq, a_s, _kmajor(q), s, off, swiglu=swiglu)
    r0 = 0
    for e, n in enumerate(counts):
        if n == 0:
            continue
        ad = aq[r0:r0 + n].float() * a_s[r0:r0 + n, None]
        want = ((ad @ q[e].float()) * s[e]).to(bf16)
        sum_abs = (ad.abs() @ q[e].float().abs()) * s[e]
        if swiglu:
            want = O.glu(want)
            rel = float((got[r0:r0 + n].float() - want.float()).norm() / want.float().norm().clamp_min(1e-30))
            assert rel < 1e-2, (e, rel)
        else:
            assert _ulp_ok(got[r0:r0 + n], want, sum_abs, K), e
        r0 += n


# ------------------------------------------------------------------------------------------------ 4. re-layout
def test_relayout_keeps_codes_scales_and_state_dict():
    from oracle import configs as C
    m16, _ = _tiny()
    m16.quantize_experts_fp8()
    m8, _ = _tiny()
    m8.quantize_experts_fp8(activations="fp8")
    for a, b in zip(m8.language_model.model.layers, m16.language_model.model.layers):
        for name in ("fc1", "fc2"):
            f8, f16 = getattr(a.mlp.experts, name), getattr(b.mlp.experts, name)
            assert f8.weight.transpose(1, 2).is_contiguous() and f16.weight.is_contiguous()
            assert torch.equal(_bits(f8.weight.transpose(1, 2)), _bits(f16.weight).transpose(1, 2))
            assert torch.equal(f8.weight_scale, f16.weight_scale)
    sd8, sd16 = m8.state_dict(), m16.state_dict()
    assert list(sd8) == list(sd16)
    for k in sd8:
        a, b = sd8[k], sd16[k]
        assert a.dtype == b.dtype and torch.equal(a.view(torch.uint8) if a.dtype == e4m3 else a,
                                                  b.view(torch.uint8) if b.dtype == e4m3 else b), k
    # a checkpoint of either mode, loaded strictly into the other, gives the in-process W8A8 logits
    ids, pv, _ = _prompts(C.TINY, False)
    want = m8(input_ids=ids, pixel_values=pv).logits
    cross, _ = _tiny()
    cross.quantize_experts_fp8(activations="fp8")
    cross.load_state_dict(sd16, strict=True)
    assert torch.equal(cross(input_ids=ids, pixel_values=pv).logits, want)
    back, _ = _tiny()
    back.quantize_experts_fp8()
    back.load_state_dict(sd8, strict=True)
    back.quantize_experts_fp8(activations="fp8")
    assert torch.equal(back(input_ids=ids, pixel_values=pv).logits, want)


def _freed_by_quantizing(mode):
    m, _ = _tiny()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    m.quantize_experts_fp8(activations=mode)
    torch.cuda.synchronize()
    return before - torch.cuda.memory_allocated()


def test_w8a8_model_takes_the_memory_of_the_w8a16_model():
    assert _freed_by_quantizing("fp8") == _freed_by_quantizing("bf16") > 0


# ------------------------------------------------------------------------------------------------ 5. block == per-kernel path
def _block_vs_kernels(model, ids, pv, monkeypatch):
    got = model(input_ids=ids, pixel_values=pv).logits
    monkeypatch.setenv("ARIA_MOE_BLOCK", "0")
    want = model(input_ids=ids, pixel_values=pv).logits
    monkeypatch.delenv("ARIA_MOE_BLOCK")
    return got, want


@pytest.mark.parametrize("forced", [False, True], ids=["free", "forced"])
def test_block_equals_per_kernel_path_tiny(forced, monkeypatch):
    from oracle import configs as C
    m, cfg = _tiny()
    m.quantize_experts_fp8(activations="fp8")
    ids, pv, _ = _prompts(cfg, False)
    if forced:
        k, E = cfg["text_config"]["moe_topk"], cfg["text_config"]["moe_num_experts"]
        T = ids.numel()
        g = torch.Generator().manual_seed(5)
        for layer in m.language_model.model.layers:
            layer.mlp.router.forced_top_indices = torch.stack(
                [torch.randperm(E, generator=g)[:k] for _ in range(T)]).to(torch.int32).to(DEV)
    got, want = _block_vs_kernels(m, ids, pv, monkeypatch)
    assert torch.equal(got, want)


@pytest.mark.parametrize("forced", [False, True], ids=["free", "forced"])
def test_block_equals_per_kernel_path_full_width_layer(forced, monkeypatch):
    from aria_b200 import configs as C
    from aria_b200.modeling_aria import AriaConfig, init_random_
    from aria_b200.moe_lm import MoELayer
    from aria_b200.modeling_aria import AriaForConditionalGeneration
    _ops()
    cfg = C.with_layers(C.ARIA_25B, lm_layers=1, vit_layers=1)
    model = AriaForConditionalGeneration(AriaConfig.from_dict(cfg), device=DEV)
    init_random_(model, seed=0)
    model.quantize_experts_fp8(activations="fp8")
    layer = model.language_model.model.layers[0].mlp
    assert isinstance(layer, MoELayer)
    T = 700
    x = torch.randn(1, T, 2560, generator=torch.Generator().manual_seed(4)).to(bf16).to(DEV)
    if forced:
        g = torch.Generator().manual_seed(6)
        layer.router.forced_top_indices = torch.stack([torch.randperm(64, generator=g)[:6] for _ in range(T)]).to(torch.int32).to(DEV)
    got = layer(x)
    monkeypatch.setenv("ARIA_MOE_BLOCK", "0")
    want = layer(x)
    assert torch.equal(got, want)
    del model
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ 6. whole tiny model
def _forced_logits(cfg, mode):
    from aria_b200 import ops
    ref, _ = _tiny()
    ids, pv, _ = _prompts(cfg, False)
    k = cfg["text_config"]["moe_topk"]
    routes, hooks = [], []
    for layer in ref.language_model.model.layers:
        hooks.append(layer.mlp.register_forward_pre_hook(
            lambda mod, args: routes.append(ops.router_topk(args[0].reshape(-1, args[0].shape[-1]), mod.router.weight, k)[1])))
    want = ref(input_ids=ids, pixel_values=pv).logits.float()
    for h in hooks:
        h.remove()
    m, _ = _tiny()
    m.quantize_experts_fp8(activations=mode)
    for layer, idx in zip(m.language_model.model.layers, routes):
        layer.mlp.router.forced_top_indices = idx
    got = m(input_ids=ids, pixel_values=pv).logits.float()
    return float((got - want).norm() / want.norm())


def test_w8a8_logits_close_to_bf16_with_forced_routing():
    from oracle import configs as C
    e8 = _forced_logits(C.TINY, "fp8")
    e16 = _forced_logits(C.TINY, "bf16")
    print(f"forced-routing logits rel-L2 vs bf16: W8A8 {e8:.4e}, W8A16 {e16:.4e}")
    # measured on an H100: W8A8 1.74e-2, W8A16 1.35e-2; the bounds keep about 3x and 1.5x of margin
    assert e8 < 5e-2 and e8 < 2 * e16, (e8, e16)


def test_graphed_prefill_replay_equals_eager():
    from aria_b200.modeling_aria import GraphedPrefill
    m, cfg = _tiny()
    m.quantize_experts_fp8(activations="fp8")
    ids, pv, _ = _prompts(cfg, False)
    want = m(input_ids=ids, pixel_values=pv, num_logits_to_keep=1).logits
    gp = GraphedPrefill(m, ids, pv, num_logits_to_keep=1)
    for _ in range(2):
        assert torch.equal(gp.replay(), want)


@pytest.mark.parametrize("padded", [False, True])
def test_w8a8_greedy_generate_equals_forward_loop(padded):
    m, cfg = _tiny()
    m.quantize_experts_fp8(activations="fp8")
    ids, pv, mask = _prompts(cfg, padded)
    n = 7
    want, logits = _forward_loop(m, ids, pv, mask, n)
    got = m.generate(ids, pv, None, max_new_tokens=n, attention_mask=mask)
    assert torch.equal(got[:, -n:], want)
    assert torch.equal(m._decode_graph.logits[:, -1], logits[-1])     # the last replayed step's logits, bit for bit


def test_w8a8_sampled_generate_equals_forward_loop():
    m, cfg = _tiny()
    m.quantize_experts_fp8(activations="fp8")
    ids, pv, mask = _prompts(cfg, True)
    n, k, t = 8, 5, 0.8
    got = m.generate(ids, pv, None, max_new_tokens=n, attention_mask=mask, do_sample=True, temperature=t, top_k=k, seed=3)
    toks = got[:, -n:]
    _, logits = _forward_loop(m, ids, pv, mask, n, tokens=toks)      # teacher-forced with the sampled tokens
    assert torch.equal(m._decode_graph.logits[:, -1], logits[-1])
    for step, lg in enumerate(logits):
        s = lg.float() / t
        assert bool((s.gather(1, toks[:, step:step + 1]) >= torch.topk(s, k, dim=-1)[0][:, -1:]).all()), step
