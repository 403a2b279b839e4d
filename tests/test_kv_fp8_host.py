"""CPU: the fp8 KV cache entries validate their arguments before any CUDA call, and forward() / generate() reject a bad
kv_cache_dtype before any device work."""
import ctypes

import pytest
import torch

BAD = -1
fake = ctypes.c_void_p(0x1000)   # never dereferenced: validation fails first
B, H, T = 2, 4, 512
CSB, CSH = H * T * 128, T * 128          # e4m3 cache strides (elements = bytes)
SSB, SSH = H * T, T                      # scale strides


@pytest.fixture(scope="module")
def lib():
    from aria_b200 import build, _lib
    build.build()
    return _lib.load()


def _expect_bad(f, ok, cases):
    for i, v in cases:
        args = list(ok)
        args[i] = v
        assert f(*args) == BAD, (f.__name__, i, v)


def test_decode_fp8_validation(lib):
    ws = lib.aria_attention_decode_workspace_bytes(B, H, T)
    f = lib.aria_attention_decode_fp8
    ok = [fake, fake, fake, fake, fake, fake, None, B, H, T, H * 128, 128, CSB, CSH, SSB, SSH, 0.1, fake, ws, None]
    _expect_bad(f, ok, [(0, None), (1, None), (2, None), (3, None), (4, None), (5, None), (17, None),
                        (7, 0), (8, 0), (9, 0),                 # B, H, Tk
                        (12, CSB + 8), (13, 136),               # cache strides not multiples of 16 codes
                        (10, 6),                                # q stride
                        (18, ws - 1)])                          # workspace too small
    d = lib.aria_attention_decode_devlen_fp8
    ok = [fake, fake, fake, fake, fake, fake, None, 0, fake, B, H, T, H * 128, 128, CSB, CSH, SSB, SSH, 0.1, fake, ws, None]
    _expect_bad(d, ok, [(0, None), (3, None), (4, None), (8, None), (19, None),
                        (11, 0),                                # T_max
                        (14, CSB + 8), (15, 120),
                        (20, ws - 1)])
    short_mask = list(ok)
    short_mask[6], short_mask[7] = fake, T - 1                  # key-mask row stride < T_max
    assert d(*short_mask) == BAD


def test_kv_store_append_load_validation(lib):
    s = lib.aria_kv_store_fp8
    ok = [fake, fake, CSH * H, CSH, fake, fake, fake, fake, CSB, CSH, SSB, SSH, 0, 16, B, H, T, None]
    _expect_bad(s, ok, [(0, None), (1, None), (4, None), (5, None), (6, None), (7, None),
                        (2, 100), (3, 36),                      # bf16 source strides not multiples of 8
                        (8, CSB + 8), (9, 200),                 # cache strides not multiples of 16
                        (12, -1), (13, 0), (12, T - 15),        # rows outside [0, T_max)
                        (16, 0), (14, 0), (15, 0)])
    a = lib.aria_kv_append_fp8
    ok = [fake, fake, H * 128, 128, fake, fake, fake, fake, CSB, CSH, SSB, SSH, fake, B, H, T, None]
    _expect_bad(a, ok, [(0, None), (4, None), (6, None), (7, None), (12, None),   # pos is required
                        (3, 12), (9, 136), (15, 0), (13, 0)])
    ld = lib.aria_kv_load_fp8
    ok = [fake, fake, fake, fake, CSB, CSH, SSB, SSH, fake, fake, CSB, CSH, 16, B, H, T, None]
    _expect_bad(ld, ok, [(0, None), (2, None), (8, None), (9, None),
                         (4, CSB + 4), (10, 4), (11, 4),
                         (12, 0), (12, T + 1), (15, 0)])


def _cpu_model():
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    return AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device="cpu")


@pytest.mark.parametrize("dtype,exc", [("int8", ValueError), ("e4m3", ValueError), (None, ValueError),
                                       ("fp8", NotImplementedError)])
def test_generate_rejects_kv_cache_dtype_before_device_work(dtype, exc):
    m = _cpu_model()
    with pytest.raises(exc):
        m.generate(torch.randint(10, 500, (1, 6)), max_new_tokens=2, kv_cache_dtype=dtype)


def test_check_generate_args_kv_cache_dtype():
    from aria_b200.modeling_aria import AriaForConditionalGeneration as A
    ids = torch.zeros(2, 3, dtype=torch.long)
    assert A._check_generate_args(ids, 4, None, False, 1.0, 50, 1.0, None, None, 0, 8, "fp8") == (2, 3, (), 0)
    with pytest.raises(ValueError):
        A._check_generate_args(ids, 4, None, False, 1.0, 50, 1.0, None, None, 0, 8, "int8")


def test_forward_rejects_bad_or_mismatched_kv_cache_dtype():
    from aria_b200.moe_lm import KVCache
    m = _cpu_model()
    ids = torch.randint(10, 500, (1, 6))
    with pytest.raises(ValueError):
        m.forward(input_ids=ids, kv_cache_dtype="int8")
    cache = KVCache(2, 1, 4, 16, 128, "cpu")                     # a bf16 cache (no device work to build it)
    with pytest.raises(ValueError):
        m.forward(input_ids=ids, past_key_values=cache, kv_cache_dtype="fp8")
    with pytest.raises(NotImplementedError):                     # the fp8 cache runs on the GPU only
        m.language_model.new_cache(1, 16, "cpu", kv_cache_dtype="fp8")
    with pytest.raises(ValueError):
        KVCache(2, 1, 4, 16, 128, "cpu", dtype="fp16")
