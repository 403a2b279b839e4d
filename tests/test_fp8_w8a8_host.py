"""CPU: argument validation of the W8A8 entries (fp8 activations and weights) happens before any CUDA call, and the host
logic of `quantize_experts_fp8(activations=...)` (invalid mode, re-layout both ways without re-quantizing, no-op in the same
mode, dropped decode graph, state dict identical to W8A16's) with torch stand-ins for the quantizers and fp8 GEMMs."""
import ctypes

import pytest
import torch

BAD = -1
fake = ctypes.c_void_p(0x1000)   # never dereferenced: validation fails first
odd = ctypes.c_void_p(0x1008)    # not 16-byte aligned
odd4 = ctypes.c_void_p(0x1002)   # not 4-byte aligned
EPI_LINEAR, EPI_SWIGLU, EPI_HEADS = 0, 1, 2


@pytest.fixture(scope="module")
def lib():
    from aria_b200 import build, _lib
    build.build()
    return _lib.load()


def test_permute_quantize_validation(lib):
    f = lib.aria_permute_quantize_fp8_rows
    ok = [fake, fake, fake, fake, 4608, 2560, None]
    for i in (0, 2, 3):                                              # x, q, scale (src_token may be NULL)
        args = list(ok)
        args[i] = None
        assert f(*args) == BAD, i
    for i, v in ((4, -1), (5, 0), (5, 2560 + 4), (5, 4096 + 8)):     # rows, d % 8, d beyond one warp's registers
        args = list(ok)
        args[i] = v
        assert f(*args) == BAD, (i, v)
    for i, p in ((0, odd), (2, odd), (3, odd4)):                     # alignment of x, q, scale
        args = list(ok)
        args[i] = p
        assert f(*args) == BAD, i


def test_grouped_gemm_w8a8_validation(lib):
    f = lib.aria_grouped_gemm_w8a8
    ok = [fake, fake, fake, fake, fake, fake, 4608, 2560, 1664, 64, EPI_SWIGLU, None]
    for i in range(6):                                               # a, a_scale, b, b_scale, out, offsets
        args = list(ok)
        args[i] = None
        assert f(*args) == BAD, i
    for i, v in ((6, -1), (7, 2560 - 64), (7, 0), (8, 1664 + 32), (8, 0), (9, 0), (10, EPI_HEADS), (10, 7)):
        args = list(ok)                                              # rows, k % 128, n % 64, groups, epilogue
        args[i] = v
        assert f(*args) == BAD, (i, v)
    for i, p in ((0, odd), (1, odd4), (2, odd), (3, odd), (4, odd)):  # alignment
        args = list(ok)
        args[i] = p
        assert f(*args) == BAD, i


def test_moe_block_w8a8_validation(lib):
    f = lib.aria_moe_block_fwd_w8a8
    nb = lib.aria_moe_block_fwd_workspace_bytes(768, 2560, 64, 6, 1664, 3328)
    ok = [fake, fake, fake, fake, fake, fake, fake, fake, fake, fake, 768, 2560, 64, 6, 1664, 3328, None, fake, nb, None, None]
    for i in (0, 1, 2, 3, 4, 5, 9, 17):                               # x, router, fc1, fc2, both scales, out, workspace
        args = list(ok)
        args[i] = None
        assert f(*args) == BAD, i
    # d % 128, I % 128, I <= 2 d (the rows of h must fit the workspace), E, k, too small a workspace
    for i, v in ((11, 2560 + 64), (14, 1664 + 64), (14, 2 * 2560 + 128), (12, 128), (13, 9), (18, nb - 1)):
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
def _quantize_cols_ref(w):
    amax = w.float().abs().amax(dim=1)
    scale = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    return (w.float() / scale[:, None, :]).to(torch.float8_e4m3fn), scale


def _quantize_rows_ref(x, src_token=None):
    x = x if src_token is None else x[src_token.long()]
    amax = x.float().abs().amax(dim=1)
    scale = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    return (x.float() / scale[:, None]).to(torch.float8_e4m3fn), scale


def _grouped_ref(a, w, offsets, swiglu):
    from oracle import aria_oracle as O
    counts = (offsets[1:] - offsets[:-1]).long()
    outs, r0 = [], 0
    for e, n in enumerate(counts.tolist()):
        outs.append(w(e, a[r0:r0 + n]).to(torch.bfloat16))
        r0 += n
    y = torch.cat(outs)
    return O.glu(y) if swiglu else y


def _gemm_fp8_ref(a, q, scale, offsets, swiglu=False):
    assert q.is_contiguous()                                         # W8A16 layout
    return _grouped_ref(a, lambda e, x: (x.float() @ q[e].float()) * scale[e], offsets, swiglu)


def _gemm_w8a8_ref(aq, a_scale, weight, weight_scale, offsets, swiglu=False):
    assert weight.transpose(1, 2).is_contiguous()                   # W8A8 layout
    from oracle import aria_oracle as O
    counts = (offsets[1:] - offsets[:-1]).long()
    outs, r0 = [], 0
    for e, n in enumerate(counts.tolist()):
        acc = aq[r0:r0 + n].float() @ weight[e].float()
        outs.append((acc * a_scale[r0:r0 + n, None] * weight_scale[e]).to(torch.bfloat16))
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
    monkeypatch.setattr(ops, "quantize_fp8_cols", _quantize_cols_ref)
    monkeypatch.setattr(ops, "grouped_gemm_fp8", _gemm_fp8_ref)
    monkeypatch.setattr(ops, "permute_quantize_fp8", _quantize_rows_ref)
    monkeypatch.setattr(ops, "grouped_gemm_w8a8", _gemm_w8a8_ref)
    m = AriaForConditionalGeneration(AriaConfig.from_dict(OC.TINY), device="cpu")
    m.load_state_dict(OC.aria_state(OC.TINY, seed=0, dtype=torch.bfloat16))
    return m


def _fcs(m):
    return [fc for layer in m.language_model.model.layers for fc in (layer.mlp.experts.fc1, layer.mlp.experts.fc2)]


def _codes(m):
    return [fc.weight.detach().clone().view(torch.uint8) for fc in _fcs(m)]


def test_invalid_mode_changes_nothing(tiny):
    from aria_b200.moe_lm import GroupedGEMM
    sentinel = object()
    tiny._decode_graph = sentinel
    for bad in ("e4m3", "FP8", None, 8):
        with pytest.raises(ValueError, match="activations"):
            tiny.quantize_experts_fp8(activations=bad)
    assert all(type(fc) is GroupedGEMM for fc in _fcs(tiny)) and tiny._decode_graph is sentinel
    tiny.quantize_experts_fp8()
    codes = _codes(tiny)
    with pytest.raises(ValueError, match="activations"):
        tiny.quantize_experts_fp8(activations="int8")
    assert all(fc.activations == "bf16" for fc in _fcs(tiny))
    assert all(torch.equal(a, b) for a, b in zip(codes, _codes(tiny)))


@pytest.mark.parametrize("first", ["bf16", "fp8"])
def test_relayout_both_ways_keeps_the_codes(tiny, first):
    other = "fp8" if first == "bf16" else "bf16"
    tiny.quantize_experts_fp8(activations=first)
    codes = _codes(tiny)
    scales = [fc.weight_scale.detach().clone() for fc in _fcs(tiny)]
    for mode in (other, first):
        tiny._decode_graph = object()
        tiny.quantize_experts_fp8(activations=mode)
        assert tiny._decode_graph is None                            # the graph holds the old weight pointers
        for fc, c, s in zip(_fcs(tiny), codes, scales):
            assert fc.activations == mode
            assert (fc.weight.transpose(1, 2) if mode == "fp8" else fc.weight).is_contiguous()
            assert torch.equal(fc.weight.view(torch.uint8), c) and torch.equal(fc.weight_scale, s)
            assert not fc.weight.requires_grad


def test_fp8_from_bf16_equals_w8a16_codes(tiny):
    import copy
    twin = copy.deepcopy(tiny)
    tiny.quantize_experts_fp8(activations="fp8")
    twin.quantize_experts_fp8()
    for a, b in zip(_fcs(tiny), _fcs(twin)):
        assert a.activations == "fp8" and b.activations == "bf16"
        assert a.weight.transpose(1, 2).is_contiguous() and b.weight.is_contiguous()
        assert torch.equal(a.weight.view(torch.uint8), b.weight.view(torch.uint8))
        assert torch.equal(a.weight_scale, b.weight_scale)


def test_same_mode_again_is_a_noop(tiny):
    tiny.quantize_experts_fp8(activations="fp8")
    mods = [(fc, fc.weight) for fc in _fcs(tiny)]
    sentinel = object()
    tiny._decode_graph = sentinel
    tiny.quantize_experts_fp8(activations="fp8")
    assert tiny._decode_graph is sentinel
    assert all(fc is m and fc.weight is w for (m, w), fc in zip(mods, _fcs(tiny)))


def test_state_dict_identical_to_w8a16_and_cross_loads(tiny):
    import copy
    from aria_b200.modeling_aria import AriaForConditionalGeneration
    twin = copy.deepcopy(tiny)
    tiny.quantize_experts_fp8(activations="fp8")
    twin.quantize_experts_fp8(activations="bf16")
    sd8, sd16 = tiny.state_dict(), twin.state_dict()
    assert list(sd8) == list(sd16)
    for k in sd8:
        assert sd8[k].shape == sd16[k].shape and sd8[k].dtype == sd16[k].dtype, k
        a, b = (t.view(torch.uint8) if t.dtype == torch.float8_e4m3fn else t for t in (sd8[k], sd16[k]))
        assert torch.equal(a, b), k
    for src, mode in ((sd16, "fp8"), (sd8, "bf16")):                # a checkpoint of either mode loads into either mode
        other = AriaForConditionalGeneration(tiny.config, device="cpu")
        for fc in _fcs(other):                                       # torch.empty may hold NaNs, which the quantizer refuses
            fc.weight.zero_()
        other.quantize_experts_fp8(activations=mode)
        other.load_state_dict(src, strict=True)
        for fc, ref in zip(_fcs(other), _fcs(tiny)):
            assert fc.activations == mode
            assert (fc.weight.transpose(1, 2) if mode == "fp8" else fc.weight).is_contiguous()
            assert torch.equal(fc.weight.view(torch.uint8), ref.weight.view(torch.uint8))


def test_w8a8_refuses_autograd_lora_trainable_install_and_expert_parallel(tiny):
    from aria_b200 import install, lora
    tiny.quantize_experts_fp8(activations="fp8")
    e = tiny.language_model.model.layers[0].mlp.experts
    assert e.is_fp8() and e.fp8_activations()
    x = torch.zeros(4, e.fc1.in_features, dtype=torch.bfloat16, requires_grad=True)
    off = torch.tensor([0, 4] + [4] * (e.fc1.groups - 1), dtype=torch.int32)
    with torch.enable_grad():
        with pytest.raises(RuntimeError, match="requires grad"):
            e(x, off)
        with pytest.raises(RuntimeError, match="requires grad"):
            tiny.language_model.model.layers[0].mlp(x.view(1, 4, -1))
    with pytest.raises(NotImplementedError, match="fp8"):
        lora.inject_lora(tiny, ["language_model.model.layers.0.mlp.experts.fc1"])
    with pytest.raises(NotImplementedError, match="fp8"):
        install.install(tiny, trainable=True)
    with pytest.raises(NotImplementedError, match="fp8"):
        tiny.enable_expert_parallel(64)


def test_w8a8_forward_takes_the_w8a8_path(tiny):
    """Module-by-module path with the stand-ins: W8A8 logits stay close to bf16, and differ from W8A16's."""
    hi = min(tiny.vocab_size, tiny.config.image_token_index)       # text tokens only
    ids = torch.randint(0, hi, (2, 12), generator=torch.Generator().manual_seed(0))
    ref = tiny(input_ids=ids).logits.float()
    tiny.quantize_experts_fp8()
    w8a16 = tiny(input_ids=ids).logits.float()
    tiny.quantize_experts_fp8(activations="fp8")
    got = tiny(input_ids=ids).logits.float()
    assert ((got - ref).norm() / ref.norm()).item() < 1e-1
    assert not torch.equal(got, w8a16)
