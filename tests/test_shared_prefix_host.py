"""CPU: generate(num_return_sequences=n) refuses what it does not serve before any device work, in a fixed order, and the
shared-prefix decode attention entry validates its arguments before any CUDA call."""
import ctypes

import pytest
import torch

BAD = -1
fake = ctypes.c_void_p(0x1000)   # never dereferenced: validation fails first


@pytest.fixture(scope="module")
def lib():
    from aria_b200 import build, _lib
    build.build()
    return _lib.load()


def _cpu_model():
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    m = AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device="cpu")

    def no_device_work(*a, **k):
        raise AssertionError("generate() reached the model before refusing its arguments")
    m.forward = no_device_work
    return m


@pytest.mark.parametrize("n", [0, -1, 2.0, "2", True, None])
def test_num_return_sequences_must_be_a_positive_int(n):
    with pytest.raises(ValueError, match="num_return_sequences"):
        _cpu_model().generate(torch.randint(10, 500, (1, 6)), do_sample=True, num_return_sequences=n)


def test_more_than_one_sequence_needs_sampling():
    with pytest.raises(ValueError, match="do_sample"):
        _cpu_model().generate(torch.randint(10, 500, (2, 6)), num_return_sequences=2)


def test_rows_beyond_the_advance_limit_are_refused():
    ids = torch.randint(10, 500, (33, 6))
    with pytest.raises(NotImplementedError, match="1024"):
        _cpu_model().generate(ids, do_sample=True, num_return_sequences=32)       # 1056 rows
    from aria_b200.modeling_aria import AriaForConditionalGeneration as A
    # 1024 rows exactly pass the checks
    assert A._check_generate_args(torch.zeros(32, 3, dtype=torch.long), 4, None, True, 1.0, 50, 1.0, None, None, 0, 8, "bf16",
                                  32) == (32, 3, (), 0)


def test_fp8_cache_is_refused_with_sharing():
    with pytest.raises(NotImplementedError, match="fp8"):
        _cpu_model().generate(torch.randint(10, 500, (1, 6)), do_sample=True, kv_cache_dtype="fp8", num_return_sequences=4)


def test_sampling_on_a_cpu_device_is_refused():
    with pytest.raises(NotImplementedError, match="GPU"):
        _cpu_model().generate(torch.randint(10, 500, (1, 6)), do_sample=True, num_return_sequences=4)


@pytest.mark.parametrize("shape,kw,exc,match", [
    # input shape first, then the batch limit, then n's type, then B * n
    ((6,), dict(num_return_sequences=0), ValueError, "input_ids"),
    ((1025, 2), dict(num_return_sequences=0), NotImplementedError, "1024"),
    ((2, 6), dict(num_return_sequences=0, max_new_tokens=0), ValueError, "num_return_sequences"),
    ((600, 6), dict(num_return_sequences=2, max_new_tokens=0), NotImplementedError, "1024"),
    # the other arguments' checks come before the combinations with n
    ((1, 6), dict(num_return_sequences=2, max_new_tokens=0), ValueError, "max_new_tokens"),
    ((1, 6), dict(num_return_sequences=2, kv_cache_dtype="fp16"), ValueError, "kv_cache_dtype"),
    # greedy is refused before the fp8 cache, and both before the sampling knobs
    ((1, 6), dict(num_return_sequences=2, kv_cache_dtype="fp8"), ValueError, "do_sample"),
    ((1, 6), dict(num_return_sequences=2, kv_cache_dtype="fp8", do_sample=True, top_k=-1), NotImplementedError, "fp8"),
    ((1, 6), dict(num_return_sequences=2, do_sample=True, top_k=-1), ValueError, "top_k"),
])
def test_order_of_the_checks(shape, kw, exc, match):
    with pytest.raises(exc, match=match):
        _cpu_model().generate(torch.zeros(shape, dtype=torch.long), **kw)


def test_shared_prefix_entry_validation(lib):
    f = lib.aria_attention_decode_shared_prefix
    G, n, H, P, N = 2, 3, 4, 700, 300
    ws = lib.aria_attention_decode_shared_prefix_workspace_bytes(G, n, H, P, N)
    assert ws == G * n * H * (3 + 2) * 130 * 4
    for bad in ((0, n, H, P, N), (G, 0, H, P, N), (G, n, -1, P, N), (G, n, H, 0, N), (G, n, H, P, 0)):
        assert lib.aria_attention_decode_shared_prefix_workspace_bytes(*bad) == -1
    # q, prefix_k, prefix_v, prefix_lens, prefix_mask, mask_stride, tail_k, tail_v, tail_lens, out, G, n, H, P_max, N_max,
    # q strides, prefix strides, tail strides, scale, workspace, workspace_bytes, stream
    ok = [fake, fake, fake, fake, None, 0, fake, fake, fake, fake, G, n, H, P, N, H * 128, 128, H * P * 128, P * 128,
          H * N * 128, N * 128, 0.1, fake, ws, None]

    def call(**changes):
        args = list(ok)
        for i, v in changes.items():
            args[int(i[1:])] = v
        return f(*args)

    for i in (0, 1, 2, 3, 6, 7, 8, 9, 22):                   # every pointer but the mask is required
        assert call(**{f"a{i}": None}) == BAD, i
    for i in (10, 11, 12, 13, 14):                           # G, n, H, P_max, N_max > 0
        assert call(**{f"a{i}": 0}) == BAD, i
    assert call(a11=1 << 20, a12=1 << 11) == BAD             # G * n * H >= 2^31
    assert call(a13=65535 * 256 + 1) == BAD                  # more prefix splits than grid.y holds
    assert call(a15=H * 128 + 2) == BAD                      # q stride % 4
    assert call(a17=H * P * 128 + 4) == BAD                  # prefix stride % 8
    assert call(a20=N * 128 + 4) == BAD                      # tail stride % 8
    assert call(a4=fake, a5=P - 1) == BAD                    # mask row stride < P_max
    assert call(a4=fake, a5=1 << 31) == BAD
    assert call(a23=ws - 1) == BAD                           # workspace too small


def test_shared_prefix_op_refuses_cpu_tensors():
    from aria_b200 import ops
    z = torch.zeros(2, 4, 256, 128, dtype=torch.bfloat16)
    lens = torch.ones(2, dtype=torch.int32)
    with pytest.raises(RuntimeError):
        ops.attention_decode_shared_prefix(torch.zeros(4, 4, 128, dtype=torch.bfloat16), z, z, lens, z, z, lens, 2, 0.1)
