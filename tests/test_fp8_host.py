"""CPU: argument validation of the fp8 expert-weight entries happens before any CUDA call, and the host logic of
`quantize_experts_fp8()` (refusals, no-op second call, state-dict keys and dtypes, dropped decode graph) with torch
stand-ins for the quantizer and the fp8 grouped GEMM."""
import ctypes

import pytest
import torch

BAD = -1
fake = ctypes.c_void_p(0x1000)   # never dereferenced: validation fails first
odd = ctypes.c_void_p(0x1008)    # not 16-byte aligned
EPI_LINEAR, EPI_SWIGLU, EPI_HEADS = 0, 1, 2


@pytest.fixture(scope="module")
def lib():
    from aria_b200 import build, _lib
    build.build()
    return _lib.load()


def test_quantize_validation(lib):
    f = lib.aria_quantize_fp8_cols
    assert f(None, fake, fake, 64, 2560, 3328, None) == BAD         # null pointers
    assert f(fake, None, fake, 64, 2560, 3328, None) == BAD
    assert f(fake, fake, None, 64, 2560, 3328, None) == BAD
    assert f(fake, fake, fake, 0, 2560, 3328, None) == BAD          # no experts
    assert f(fake, fake, fake, 64, 2560 + 8, 3328, None) == BAD     # k % 64
    assert f(fake, fake, fake, 64, 2560, 3328 + 8, None) == BAD     # n % 64
    assert f(fake, fake, fake, 64, 0, 3328, None) == BAD
    assert f(odd, fake, fake, 64, 2560, 3328, None) == BAD          # alignment
    assert f(fake, odd, fake, 64, 2560, 3328, None) == BAD
    assert f(fake, fake, odd, 64, 2560, 3328, None) == BAD


def test_grouped_gemm_fp8_validation(lib):
    f = lib.aria_grouped_gemm_fp8
    ok = [fake, fake, fake, fake, fake, 4608, 2560, 1664, 64, EPI_SWIGLU, None]
    for i in range(5):                                               # a, b, scale, out, offsets
        args = list(ok)
        args[i] = None
        assert f(*args) == BAD
    for i, v in ((5, -1), (6, 2560 + 8), (7, 1664 + 8), (7, 0), (8, 0), (9, EPI_HEADS), (9, 7)):
        args = list(ok)
        args[i] = v
        assert f(*args) == BAD, (i, v)
    for i in range(4):                                               # alignment of a, b, scale, out
        args = list(ok)
        args[i] = odd
        assert f(*args) == BAD


def test_moe_block_fp8_validation(lib):
    f = lib.aria_moe_block_fwd_fp8
    nb = lib.aria_moe_block_fwd_workspace_bytes(768, 2560, 64, 6, 1664, 3328)
    ok = [fake, fake, fake, fake, fake, fake, fake, fake, fake, fake, 768, 2560, 64, 6, 1664, 3328, None, fake, nb, None, None]
    for i in (0, 1, 2, 3, 4, 5, 9, 17):                               # x, router, fc1, fc2, both scales, out, workspace
        args = list(ok)
        args[i] = None
        assert f(*args) == BAD, i
    for i, v in ((11, 2560 + 8), (14, 1664 + 8), (12, 128), (13, 9), (18, nb - 1)):
        args = list(ok)
        args[i] = v
        assert f(*args) == BAD, (i, v)
    for i in (2, 3, 4, 5):                                           # alignment of the fp8 weights and scales
        args = list(ok)
        args[i] = odd
        assert f(*args) == BAD, i
    args = list(ok)
    args[6] = args[7] = args[8] = None                               # shared experts without their weights
    assert f(*args) == BAD


# ----------------------------------------------------------------------------- host logic of quantize_experts_fp8()
def _quantize_ref(w):
    amax = w.float().abs().amax(dim=1)
    scale = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    return (w.float() / scale[:, None, :]).to(torch.float8_e4m3fn), scale


def _grouped_gemm_fp8_ref(a, q, scale, offsets, swiglu=False):
    from oracle import aria_oracle as O
    counts = (offsets[1:] - offsets[:-1]).long()
    outs, r0 = [], 0
    for e, n in enumerate(counts.tolist()):
        outs.append(((a[r0:r0 + n].float() @ q[e].float()) * scale[e]).to(torch.bfloat16))
        r0 += n
    y = torch.cat(outs)
    return O.glu(y) if swiglu else y


@pytest.fixture
def tiny(monkeypatch):
    import standin_ops
    from aria_b200 import ops
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as OC
    standin_ops.patch(monkeypatch)
    monkeypatch.setattr(ops, "quantize_fp8_cols", _quantize_ref)
    monkeypatch.setattr(ops, "grouped_gemm_fp8", _grouped_gemm_fp8_ref)
    m = AriaForConditionalGeneration(AriaConfig.from_dict(OC.TINY), device="cpu")
    m.load_state_dict(OC.aria_state(OC.TINY, seed=0, dtype=torch.bfloat16))
    return m


def _experts(m):
    return [layer.mlp.experts for layer in m.language_model.model.layers]


def test_quantize_state_dict_keys_and_reload(tiny):
    from aria_b200.moe_lm import Fp8GroupedGEMM
    from aria_b200.modeling_aria import AriaForConditionalGeneration
    bf16_w = _experts(tiny)[0].fc1.weight.clone()
    keys_before = set(tiny.state_dict())
    assert tiny.quantize_experts_fp8() is tiny
    sd = tiny.state_dict()
    new = set(sd) - keys_before
    assert new == {k.replace(".weight", ".weight_scale") for k in keys_before if ".experts.fc" in k}
    E, I2 = bf16_w.shape[0], bf16_w.shape[2]
    for e in _experts(tiny):
        assert type(e.fc1) is Fp8GroupedGEMM and type(e.fc2) is Fp8GroupedGEMM and e.is_fp8()
        assert e.fc1.weight.dtype == torch.float8_e4m3fn and e.fc1.weight_scale.dtype == torch.float32
        assert not e.fc1.weight.requires_grad and not e.fc1.weight_scale.requires_grad
    q, s = _quantize_ref(bf16_w)
    assert torch.equal(_experts(tiny)[0].fc1.weight.view(torch.uint8), q.view(torch.uint8))
    assert torch.equal(_experts(tiny)[0].fc1.weight_scale, s) and s.shape == (E, I2)
    # a freshly built model, quantized, reloads the quantized state dict strictly
    other = AriaForConditionalGeneration(tiny.config, device="cpu")
    for e in _experts(other):                                        # torch.empty may hold NaNs, which the quantizer refuses
        e.fc1.weight.zero_()
        e.fc2.weight.zero_()
    other.quantize_experts_fp8()
    other.load_state_dict(sd, strict=True)
    assert torch.equal(_experts(other)[1].fc2.weight.view(torch.uint8), _experts(tiny)[1].fc2.weight.view(torch.uint8))


def test_quantize_second_call_is_a_noop_and_drops_the_decode_graph(tiny):
    sentinel = object()
    tiny._decode_graph = sentinel
    tiny.quantize_experts_fp8()
    assert tiny._decode_graph is None
    mods = [(e.fc1, e.fc2) for e in _experts(tiny)]
    tiny._decode_graph = sentinel
    tiny.quantize_experts_fp8()
    assert tiny._decode_graph is sentinel
    assert [(e.fc1, e.fc2) for e in _experts(tiny)] == mods


def test_quantize_refuses_non_finite_before_changing_anything(tiny):
    _experts(tiny)[1].fc2.weight[3, 5, 7] = float("nan")
    with pytest.raises(ValueError, match="non-finite"):
        tiny.quantize_experts_fp8()
    assert not any(e.is_fp8() for e in _experts(tiny))


def test_expert_parallel_and_quantization_refuse_each_other(tiny):
    tiny.language_model.model.layers[0].mlp.expert_parallel = object()
    with pytest.raises(NotImplementedError, match="expert parallelism"):
        tiny.quantize_experts_fp8()
    assert not any(e.is_fp8() for e in _experts(tiny))
    tiny.language_model.model.layers[0].mlp.expert_parallel = None
    tiny.quantize_experts_fp8()
    with pytest.raises(NotImplementedError, match="fp8"):
        tiny.enable_expert_parallel(64)


def test_fp8_refuses_autograd_lora_and_trainable_install(tiny):
    from aria_b200 import install, lora
    tiny.quantize_experts_fp8()
    e = _experts(tiny)[0]
    x = torch.zeros(4, e.fc1.in_features, dtype=torch.bfloat16, requires_grad=True)
    off = torch.tensor([0, 4] + [4] * (e.fc1.groups - 1), dtype=torch.int32)
    with torch.enable_grad():
        with pytest.raises(RuntimeError, match="requires grad"):
            e.fc1(x, off)
        with pytest.raises(RuntimeError, match="requires grad"):
            e(x, off)
        with pytest.raises(RuntimeError, match="requires grad"):
            tiny.language_model.model.layers[0].mlp(x.view(1, 4, -1))
    with pytest.raises(NotImplementedError, match="fp8"):
        lora.inject_lora(tiny, ["language_model.model.layers.0.mlp.experts.fc1"])
    with pytest.raises(NotImplementedError, match="fp8"):
        lora.GroupedGemmLoraLayer(e.fc1)
    with pytest.raises(NotImplementedError, match="fp8"):
        install.install(tiny, trainable=True)


def test_quantized_forward_takes_the_fp8_path(tiny):
    """Module-by-module path with the stand-ins: logits stay close to bf16 and generate() still runs."""
    hi = min(tiny.vocab_size, tiny.config.image_token_index)       # text tokens only
    ids = torch.randint(0, hi, (2, 12), generator=torch.Generator().manual_seed(0))
    ref = tiny(input_ids=ids).logits.float()
    tiny.quantize_experts_fp8()
    got = tiny(input_ids=ids).logits.float()
    assert ((got - ref).norm() / ref.norm()).item() < 5e-2
    out = tiny.generate(ids, max_new_tokens=3)
    assert out.shape == (2, 15)
