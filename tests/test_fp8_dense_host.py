"""CPU: the W8A8 dense entries (aria_gemm_w8a8, aria_rmsnorm_quantize_fp8, aria_moe_block_fwd_shared_fp8) reject bad
arguments before any CUDA call, and quantize_dense_fp8 / enable_expert_parallel refuse what they do not support before
anything changes."""
import ctypes

import pytest
import torch

FAKE = 0x10000      # 16-byte aligned, never dereferenced: validation fails first
BAD_ARG = -1


@pytest.fixture(scope="module")
def lib():
    from aria_b200 import build, _lib
    build.build()
    return _lib.load()


def _desc(epilogue=0, m=32, n=2560, k=2560, n_seg=1):
    from aria_b200 import _lib as L
    d = L.GemmDesc()
    d.a, d.lda, d.m, d.n, d.k = FAKE, k, m, n, k
    for s in range(3):
        d.b[s] = FAKE
        d.out[s] = FAKE
    d.n_seg, d.b_layout, d.num_groups, d.epilogue = n_seg, L.B_NK, 1, epilogue
    d.ldo = n * (1 if epilogue == L.EPI_SWIGLU else n_seg)
    if epilogue == L.EPI_HEADS:
        d.head_dim, d.head_ld, d.rows_per_batch = 128, 128, m
        d.rope_mask, d.rope_cos, d.rope_sin = 0b011, FAKE, FAKE
    return d


def _scales(n=3, ptr=FAKE):
    return ctypes.cast((ctypes.c_void_p * 3)(*([ptr] * n + [None] * (3 - n))), ctypes.c_void_p)


def _gemm(lib, d, a_scale=FAKE, scales=None):
    return lib.aria_gemm_w8a8(ctypes.byref(d), ctypes.c_void_p(a_scale), scales if scales is not None else _scales(), None)


def test_gemm_w8a8_rejects_bad_arguments(lib):
    from aria_b200 import _lib as L
    assert lib.aria_gemm_w8a8(None, ctypes.c_void_p(FAKE), _scales(), None) == BAD_ARG
    assert _gemm(lib, _desc(), scales=ctypes.c_void_p(None)) == BAD_ARG         # no scale array
    assert _gemm(lib, _desc(), a_scale=0) == BAD_ARG                            # no row scales
    assert _gemm(lib, _desc(), scales=_scales(0)) == BAD_ARG                    # no column scales
    assert _gemm(lib, _desc(), scales=_scales(1, FAKE + 8)) == BAD_ARG          # column scales not 16-byte aligned
    assert _gemm(lib, _desc(k=2560 + 64)) == BAD_ARG                           # k % 128
    assert _gemm(lib, _desc(n=2560 + 32)) == BAD_ARG                           # n % 64
    d = _desc()
    d.a = FAKE + 8                                                              # a not 16-byte aligned
    assert _gemm(lib, d) == BAD_ARG
    d = _desc()
    d.b[0] = FAKE + 4
    assert _gemm(lib, d) == BAD_ARG
    d = _desc()
    d.b_layout = L.B_GKN                                                        # grouped layouts go to aria_grouped_gemm_w8a8
    assert _gemm(lib, d) == BAD_ARG
    d = _desc()
    d.num_groups = 2
    assert _gemm(lib, d) == BAD_ARG
    d = _desc()
    d.group_offsets = FAKE
    assert _gemm(lib, d) == BAD_ARG
    assert _gemm(lib, _desc(n=2560 - 64, n_seg=3)) == BAD_ARG                  # a tile would straddle two weights
    assert _gemm(lib, _desc(epilogue=L.EPI_SWIGLU, n_seg=1)) == BAD_ARG        # SwiGLU takes gate and up
    assert _gemm(lib, _desc(epilogue=L.EPI_SWIGLU, n_seg=2), scales=_scales(1)) == BAD_ARG  # ... and both scales
    d = _desc(epilogue=L.EPI_HEADS, n_seg=3)
    d.head_dim = 64                                                             # RoPE needs head_dim 128
    assert _gemm(lib, d) == BAD_ARG
    d = _desc(epilogue=L.EPI_HEADS, n_seg=3)
    d.rope_cos = None
    assert _gemm(lib, d) == BAD_ARG
    d = _desc(epilogue=L.EPI_HEADS, n_seg=3)
    d.out[2] = None
    assert _gemm(lib, d) == BAD_ARG
    d = _desc(epilogue=L.EPI_HEADS, n=1224, n_seg=3)                          # 17 heads of 72: 128-wide tiles only
    d.head_dim, d.head_ld, d.rope_mask = 72, 72, 0
    assert _gemm(lib, d) == BAD_ARG
    d = _desc()
    d.residual, d.ldr = FAKE + 2, 2560
    assert _gemm(lib, d) == BAD_ARG
    d = _desc(epilogue=L.EPI_HEADS, n_seg=3)
    d.residual, d.ldr = FAKE, 2560                                             # residual: LINEAR only
    assert _gemm(lib, d) == BAD_ARG
    assert _gemm(lib, _desc(m=0)) == 0                                          # nothing to do: no launch


def test_rmsnorm_quantize_rejects_bad_arguments(lib):
    f = lib.aria_rmsnorm_quantize_fp8
    assert f(None, None, FAKE, FAKE, FAKE, None, 4, 2560, 1e-5, None) == BAD_ARG
    assert f(FAKE, None, FAKE, None, FAKE, None, 4, 2560, 1e-5, None) == BAD_ARG
    assert f(FAKE, None, FAKE, FAKE, None, None, 4, 2560, 1e-5, None) == BAD_ARG
    assert f(FAKE, None, FAKE, FAKE, FAKE, None, 4, 2564, 1e-5, None) == BAD_ARG    # d % 8
    assert f(FAKE, None, FAKE, FAKE, FAKE, None, 4, 4096 + 8, 1e-5, None) == BAD_ARG  # d <= 4096
    assert f(FAKE + 8, None, FAKE, FAKE, FAKE, None, 4, 2560, 1e-5, None) == BAD_ARG
    assert f(FAKE, FAKE + 8, FAKE, FAKE, FAKE, FAKE, 4, 2560, 1e-5, None) == BAD_ARG
    assert f(FAKE, None, FAKE, FAKE, FAKE + 2, None, 4, 2560, 1e-5, None) == BAD_ARG
    assert f(FAKE, None, FAKE, FAKE, FAKE, None, 0, 2560, 1e-5, None) == 0


def test_moe_block_shared_fp8_rejects_bad_arguments(lib):
    from aria_b200 import _lib as L
    T, d, E, k, I, Is = 768, 2560, 64, 6, 1664, 3328
    nb = lib.aria_moe_block_fwd_shared_fp8_workspace_bytes(T, d, E, k, I, Is)
    base = lib.aria_moe_block_fwd_workspace_bytes(T, d, E, k, I, Is)
    assert nb >= base + T * (d + Is + 8) and nb % 256 == 0
    assert lib.aria_moe_block_fwd_shared_fp8_workspace_bytes(T, d, E, k, I, 0) == BAD_ARG
    f = lib.aria_moe_block_fwd_shared_fp8

    def call(mode=L.MOE_EXPERTS_W8A8, fc_scale=FAKE, sh_scale=FAKE, d=d, I=I, Is=Is, ws=nb, down=FAKE):
        return f(FAKE, FAKE, FAKE, FAKE, fc_scale, fc_scale, mode, FAKE, FAKE, down, sh_scale, sh_scale, sh_scale, FAKE, T, d,
                 E, k, I, Is, None, FAKE, ws, None, None)

    assert call(sh_scale=None) == BAD_ARG                       # shared scales are required
    assert call(down=None) == BAD_ARG
    assert call(sh_scale=FAKE + 4) == BAD_ARG                   # 16-byte aligned scales
    assert call(Is=3328 + 64) == BAD_ARG                        # I_shared % 128 (down's K)
    assert call(Is=0) == BAD_ARG
    assert call(mode=3) == BAD_ARG                              # unknown expert mode
    assert call(mode=L.MOE_EXPERTS_BF16) == BAD_ARG             # bf16 experts take no expert scales
    assert call(mode=L.MOE_EXPERTS_FP8, fc_scale=None) == BAD_ARG
    assert call(mode=L.MOE_EXPERTS_W8A8, I=1664 + 64) == BAD_ARG  # W8A8 experts: I % 128
    assert call(ws=base) == BAD_ARG                             # the shared branch's regions are missing
    assert call(mode=L.MOE_EXPERTS_BF16, fc_scale=None, ws=nb - 1) == BAD_ARG


# ------------------------------------------------------------------------------------------------ model-level refusals
def _model():
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    m = AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device="cpu")
    m.load_state_dict(C.aria_state(C.TINY, seed=0, dtype=torch.bfloat16), strict=True)
    return m


def _dense_weights(m):
    return [getattr(layer.get_submodule(o), n).weight for layer in m.language_model.model.layers
            for o, names in m._DENSE_FP8 for n in names]


def test_quantize_dense_fp8_refuses_expert_parallel():
    m = _model()
    m.language_model.model.layers[1].mlp.expert_parallel = object()
    before = _dense_weights(m)
    with pytest.raises(NotImplementedError, match="expert parallelism"):
        m.quantize_dense_fp8()
    assert all(a is b for a, b in zip(before, _dense_weights(m)))


def test_quantize_dense_fp8_validates_every_layer_before_changing_any():
    m = _model()
    m._decode_graph = "graph"
    before = _dense_weights(m)
    m.language_model.model.layers[1].mlp.shared_experts.down_proj.weight.data[3, 5] = float("nan")
    with pytest.raises(ValueError, match="layer 1 mlp.shared_experts.down_proj"):
        m.quantize_dense_fp8()
    assert all(a is b for a, b in zip(before, _dense_weights(m))) and m._decode_graph == "graph"
    m = _model()
    attn = m.language_model.model.layers[1].self_attn
    attn.v_proj = torch.nn.Linear(256, 256, bias=False, dtype=torch.bfloat16)        # e.g. what an adapter wraps
    with pytest.raises(NotImplementedError, match="layer 1 self_attn.v_proj"):
        m.quantize_dense_fp8()
    assert type(m.language_model.model.layers[0].self_attn.q_proj).__name__ == "Linear"


def test_enable_expert_parallel_refuses_dense_fp8_model():
    from aria_b200.moe_lm import Fp8Linear
    m = _model()
    se = m.language_model.model.layers[0].mlp.shared_experts
    se.up_proj = Fp8Linear(se.up_proj.weight.shape[1], se.up_proj.weight.shape[0], device="cpu")
    with pytest.raises(NotImplementedError, match="quantize_dense_fp8"):
        m.enable_expert_parallel(64)


def test_fp8_linear_shapes_and_state_dict_keys():
    from aria_b200.moe_lm import Fp8Linear
    f = Fp8Linear(256, 512, device="cpu")
    assert f.weight.dtype == torch.float8_e4m3fn and f.weight.shape == (512, 256) and not f.weight.requires_grad
    assert f.weight_scale.dtype == torch.float32 and f.weight_scale.shape == (512,) and not f.weight_scale.requires_grad
    assert list(f.state_dict()) == ["weight", "weight_scale"]
    with pytest.raises(ValueError):
        Fp8Linear(256, 512, weight=torch.empty(512, 256, dtype=torch.bfloat16))
    x = torch.zeros(2, 256, dtype=torch.bfloat16, requires_grad=True)
    with torch.enable_grad(), pytest.raises(RuntimeError, match="inference-only"):
        f(x)
