"""H100: W8A8 attention projections and shared experts (quantize_dense_fp8).  With small integer codes and power-of-two scales
the dense W8A8 GEMM is bit-identical to aria_gemm on the dequantized operands in every epilogue; on random data it matches the
fp32 oracle; the fused RMSNorm quantizer equals rmsnorm + the row quantizer bit for bit; the one-call MoE block equals the
per-kernel path in every expert mode; a whole tiny model stays close to bf16, replays its graphs exactly, generates what its
forward loop generates, and round-trips its state dict."""
import pytest
import torch

from test_gpu_fp8 import _prompts, _tiny, _ulp_ok
from test_gpu_kv_fp8 import _forward_loop

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
bf16, e4m3 = torch.bfloat16, torch.float8_e4m3fn
ROWS = [1, 32, 768, 1000]


def _ops():
    from aria_b200 import build, ops
    build.build()
    return ops


def _rows_oracle(x):
    amax = x.float().abs().amax(dim=1)
    scale = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    return (x.float() / scale[:, None]).to(e4m3), scale


def _bits(q):
    return q.view(torch.uint8)


def _int_codes(shape, g):
    return torch.randint(-3, 4, shape, generator=g).float().to(e4m3)


def _operand(rows, K, g):
    """Integer e4m3 codes with power-of-two row scales, and their exact bf16 dequantization."""
    q = _int_codes((rows, K), g)
    s = torch.exp2(torch.randint(-9, -3, (rows,), generator=g).float())
    return q.to(DEV), s.to(DEV), (q.float() * s[:, None]).to(bf16).to(DEV)


# ------------------------------------------------------------------------------------------------ 1. GEMM bit identity
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("kind", ["linear", "linear_residual", "swiglu", "down"])
def test_int_codes_bit_identical_linear(kind, rows):
    ops = _ops()
    K, N = {"linear": (2560, 2560), "linear_residual": (2560, 2560), "swiglu": (2560, 3328), "down": (3328, 2560)}[kind]
    g = torch.Generator().manual_seed(rows + K)
    aq, a_s, a = _operand(rows, K, g)
    ws = [_operand(N, K, g) for _ in range(2 if kind == "swiglu" else 1)]
    if kind == "swiglu":
        (gq, gs, gw), (uq, us, uw) = ws
        got = ops.linear_swiglu_w8a8(aq, a_s, gq, gs, uq, us)
        want = ops.linear_swiglu(a, gw, uw)
    else:
        (wq, w_s, w), = ws
        res = (torch.randn(rows, N, generator=g) * 0.1).to(bf16).to(DEV) if kind == "linear_residual" else None
        got = ops.linear_w8a8(aq, a_s, wq, w_s, residual=res)
        want = ops.linear(a, w, residual=res)
    assert torch.equal(got, want)


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("positions", ["pos0", "position_ids"])
def test_int_codes_bit_identical_qkv_heads_rope(positions, rows):
    ops = _ops()
    K = N = 2560
    H, T_max = 20, 1100
    g = torch.Generator().manual_seed(rows + 7)
    aq, a_s, a = _operand(rows, K, g)
    ws = [_operand(N, K, g) for _ in range(3)]
    inv_freq = 1.0 / (5e6 ** (torch.arange(0, 128, 2, dtype=torch.int64).float() / 128))
    cos, sin = ops.rope_table(inv_freq.to(DEV), 4096)
    pos0, pid = (37, None) if positions == "pos0" else (0, torch.randint(0, 4096, (rows,), generator=g, dtype=torch.int32).to(DEV))
    outs = []
    for fp8 in (True, False):
        o = [torch.zeros(1, H, T_max, 128, dtype=bf16, device=DEV) for _ in range(3)]
        kw = dict(pos0=pos0, rope_mask=0b011, rope_cos=cos, rope_sin=sin, position_ids=pid)
        if fp8:
            ops.qkv_heads_w8a8(aq, a_s, [w[0] for w in ws], [w[1] for w in ws], o, 128, rows, **kw)
        else:
            ops.qkv_heads(a, [w[2] for w in ws], [None] * 3, o, 128, rows, **kw)
        outs.append(o)
    for x, y in zip(*outs):
        assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------------ 2. GEMM vs fp32 oracle
@pytest.mark.parametrize("rows", [32, 1000])
@pytest.mark.parametrize("K,N", [(2560, 2560), (3328, 2560), (2560, 7680)])
def test_gemm_matches_dequantized_oracle(K, N, rows):
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(3)
    a = torch.randn(rows, K, device=DEV, generator=g).to(bf16)
    w = (torch.randn(N, K, device=DEV, generator=g) * 0.02).to(bf16)
    wq, w_s = ops.permute_quantize_fp8(w)
    aq, a_s = ops.permute_quantize_fp8(a)
    got = ops.linear_w8a8(aq, a_s, wq, w_s)
    ad, wd = aq.float() * a_s[:, None], wq.float() * w_s[:, None]
    want = (ad @ wd.T).to(bf16)
    assert _ulp_ok(got, want, ad.abs() @ wd.abs().T, K)


# ------------------------------------------------------------------------------------------------ 3. quantizers
@pytest.mark.parametrize("d", [256, 2560, 4096])
@pytest.mark.parametrize("residual", [False, True])
def test_rmsnorm_quantize_bit_identical(d, residual):
    ops = _ops()
    g = torch.Generator().manual_seed(d)
    x = (torch.randn(777, d, generator=g) * torch.rand(777, 1, generator=g) * 4).to(bf16).to(DEV)
    x[3] = 0.0
    w = (1 + 0.1 * torch.randn(d, generator=g)).to(bf16).to(DEV)
    r = (torch.randn(777, d, generator=g)).to(bf16).to(DEV) if residual else None
    got = ops.rmsnorm_quantize_fp8(x, w, 1e-5, r)
    ref = ops.rmsnorm(x, w, 1e-5, r)
    h = ref[0] if residual else ref
    wq, ws = ops.permute_quantize_fp8(h)
    assert torch.equal(_bits(got[0]), _bits(wq)) and torch.equal(got[1], ws)
    if residual:
        assert torch.equal(got[2], ref[1])


def test_weight_quantizer_matches_torch_formula():
    from aria_b200.moe_lm import Fp8Linear, Linear
    _ops()
    lin = Linear(3328, 2560, device=DEV)
    lin.weight.data = (torch.randn(2560, 3328, generator=torch.Generator().manual_seed(9)) * 0.02).to(bf16).to(DEV)
    lin.weight.data[5] = 0.0
    f = Fp8Linear.from_linear(lin)
    wq, ws = _rows_oracle(lin.weight.cpu())
    assert torch.equal(f.weight_scale.cpu(), ws) and torch.equal(_bits(f.weight).cpu(), _bits(wq))


# ------------------------------------------------------------------------------------------------ 4. block == per-kernel path
EXPERT_MODES = [None, "bf16", "fp8"]


def _quantize(m, experts):
    m.quantize_dense_fp8()
    if experts is not None:
        m.quantize_experts_fp8(activations=experts)
    return m


@pytest.mark.parametrize("experts", EXPERT_MODES, ids=["bf16_experts", "w8a16_experts", "w8a8_experts"])
def test_block_equals_per_kernel_path_tiny(experts, monkeypatch):
    m, cfg = _tiny()
    _quantize(m, experts)
    ids, pv, _ = _prompts(cfg, False)
    got = m(input_ids=ids, pixel_values=pv).logits
    monkeypatch.setenv("ARIA_MOE_BLOCK", "0")
    want = m(input_ids=ids, pixel_values=pv).logits
    assert torch.equal(got, want)


@pytest.mark.parametrize("experts", EXPERT_MODES, ids=["bf16_experts", "w8a16_experts", "w8a8_experts"])
def test_block_equals_per_kernel_path_full_width_layer(experts, monkeypatch):
    from aria_b200 import configs as C
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration, init_random_
    _ops()
    cfg = C.with_layers(C.ARIA_25B, lm_layers=1, vit_layers=1)
    model = AriaForConditionalGeneration(AriaConfig.from_dict(cfg), device=DEV)
    init_random_(model, seed=0)
    _quantize(model, experts)
    layer = model.language_model.model.layers[0].mlp
    x = torch.randn(1, 700, 2560, generator=torch.Generator().manual_seed(4)).to(bf16).to(DEV)
    got = layer(x)
    monkeypatch.setenv("ARIA_MOE_BLOCK", "0")
    want = layer(x)
    assert torch.equal(got, want)
    del model
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ 5. whole tiny model
def _forced_logits(cfg, experts):
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
    _quantize(m, experts)
    for layer, idx in zip(m.language_model.model.layers, routes):
        layer.mlp.router.forced_top_indices = idx
    got = m(input_ids=ids, pixel_values=pv).logits.float()
    return float((got - want).norm() / want.norm())


def test_dense_fp8_logits_close_to_bf16_with_forced_routing():
    from oracle import configs as C
    dense = _forced_logits(C.TINY, None)
    both = _forced_logits(C.TINY, "fp8")
    print(f"forced-routing logits rel-L2 vs bf16: dense W8A8 {dense:.4e}, dense + expert W8A8 {both:.4e}")
    # measured on an H100: 6.62e-2 and 6.87e-2.  The dense linears are seven of the nine GEMMs of a layer (the W8A8 experts
    # alone give 1.74e-2, test_gpu_fp8_w8a8); the bound keeps about 1.5x of margin
    assert dense < 1e-1 and both < 1e-1, (dense, both)


def test_quantize_dense_fp8_is_idempotent_and_combines_in_either_order():
    from oracle import configs as C
    ids, pv, _ = _prompts(C.TINY, False)
    a, _ = _tiny()
    a.quantize_dense_fp8().quantize_experts_fp8(activations="fp8")
    b, _ = _tiny()
    b.quantize_experts_fp8(activations="fp8").quantize_dense_fp8()
    want = a(input_ids=ids, pixel_values=pv).logits
    assert torch.equal(b(input_ids=ids, pixel_values=pv).logits, want)
    w = a.language_model.model.layers[0].self_attn.q_proj.weight
    a.quantize_dense_fp8()
    assert a.language_model.model.layers[0].self_attn.q_proj.weight is w
    assert torch.equal(a(input_ids=ids, pixel_values=pv).logits, want)


def test_graphed_prefill_replay_equals_eager():
    from aria_b200.modeling_aria import GraphedPrefill
    m, cfg = _tiny()
    _quantize(m, "fp8")
    ids, pv, _ = _prompts(cfg, False)
    want = m(input_ids=ids, pixel_values=pv, num_logits_to_keep=1).logits
    gp = GraphedPrefill(m, ids, pv, num_logits_to_keep=1)
    for _ in range(2):
        assert torch.equal(gp.replay(), want)


@pytest.mark.parametrize("kv", ["bf16", "fp8"])
@pytest.mark.parametrize("padded", [False, True])
def test_greedy_generate_equals_forward_loop(padded, kv):
    from test_gpu_generate import _prompts as gen_prompts
    m, cfg = _tiny()
    _quantize(m, None)
    ids, pv, mask = gen_prompts(cfg, padded)
    n = 7
    want, logits = _forward_loop(m, ids, pv, mask, n, kv)
    got = m.generate(ids, pv, None, max_new_tokens=n, attention_mask=mask, kv_cache_dtype=kv)
    assert torch.equal(got[:, -n:], want)
    assert torch.equal(m._decode_graph.logits[:, -1], logits[-1])


@pytest.mark.parametrize("kv", ["bf16", "fp8"])
def test_sampled_generate_equals_forward_loop(kv):
    from test_gpu_generate import _prompts as gen_prompts
    m, cfg = _tiny()
    _quantize(m, "fp8")
    ids, pv, mask = gen_prompts(cfg, True)
    n, k, t = 8, 5, 0.8
    got = m.generate(ids, pv, None, max_new_tokens=n, attention_mask=mask, do_sample=True, temperature=t, top_k=k, seed=3,
                     kv_cache_dtype=kv)
    toks = got[:, -n:]
    _, logits = _forward_loop(m, ids, pv, mask, n, kv, tokens=toks)
    assert torch.equal(m._decode_graph.logits[:, -1], logits[-1])
    for step, lg in enumerate(logits):
        s = lg.float() / t
        assert bool((s.gather(1, toks[:, step:step + 1]) >= torch.topk(s, k, dim=-1)[0][:, -1:]).all()), step


# ------------------------------------------------------------------------------------------------ 7. state dict and memory
def test_state_dict_round_trip_and_memory():
    from oracle import configs as C
    m, _ = _tiny()
    lins = [getattr(layer.get_submodule(o), n) for layer in m.language_model.model.layers
            for o, names in m._DENSE_FP8 for n in names]
    bf16_bytes = sum(lin.weight.numel() * 2 for lin in lins)
    fp8_bytes = sum(lin.weight.numel() + lin.weight.shape[0] * 4 for lin in lins)
    del lins
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    m.quantize_dense_fp8()
    torch.cuda.synchronize()
    assert before - torch.cuda.memory_allocated() == bf16_bytes - fp8_bytes > 0
    sd = m.state_dict()
    key = "language_model.model.layers.0.self_attn.q_proj"
    assert sd[key + ".weight"].dtype == e4m3 and sd[key + ".weight_scale"].dtype == torch.float32
    assert sd["language_model.model.layers.1.mlp.shared_experts.down_proj.weight_scale"].shape == (256,)
    ids, pv, _ = _prompts(C.TINY, False)
    want = m(input_ids=ids, pixel_values=pv).logits
    back, _ = _tiny()
    back.quantize_dense_fp8()
    back.load_state_dict(sd, strict=True)
    assert torch.equal(back(input_ids=ids, pixel_values=pv).logits, want)
