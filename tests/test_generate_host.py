"""CPU: argument validation of the generation entries (sampling, device-length decode attention, KV append, decode-state
advance) happens before any CUDA call, and generate() rejects bad arguments before it touches the device."""
import ctypes

import pytest
import torch

BAD, UNSUPPORTED = -1, -2
fake = ctypes.c_void_p(0x1000)   # never dereferenced: validation fails first


@pytest.fixture(scope="module")
def lib():
    from aria_b200 import build, _lib
    build.build()
    return _lib.load()


def test_sample_tokens_validation(lib):
    f = lib.aria_sample_tokens
    assert f(None, 1000, fake, None, 1, 1000, 1.0, 50, 1.0, 0, None, None) == BAD          # null logits
    assert f(fake, 1000, None, None, 1, 1000, 1.0, 50, 1.0, 0, None, None) == BAD          # null output
    assert f(fake, 1000, fake, None, 0, 1000, 1.0, 50, 1.0, 0, None, None) == BAD          # B = 0
    assert f(fake, 1000, fake, None, (1 << 20) + 1, 1000, 1.0, 50, 1.0, 0, None, None) == BAD
    assert f(fake, 1000, fake, None, 1, 0, 1.0, 50, 1.0, 0, None, None) == BAD             # V = 0
    assert f(fake, 1000, fake, None, 1, (1 << 24) + 1, 1.0, 50, 1.0, 0, None, None) == BAD
    assert f(fake, -1, fake, None, 1, 1000, 1.0, 50, 1.0, 0, None, None) == BAD            # negative row stride
    assert f(fake, 1000, fake, None, 1, 1000, -0.5, 50, 1.0, 0, None, None) == BAD         # temperature < 0
    assert f(fake, 1000, fake, None, 1, 1000, float("nan"), 50, 1.0, 0, None, None) == BAD
    assert f(fake, 1000, fake, None, 1, 1000, float("inf"), 50, 1.0, 0, None, None) == BAD
    assert f(fake, 1000, fake, None, 1, 1000, 1.0, -1, 1.0, 0, None, None) == BAD          # k out of [0, 1024]
    assert f(fake, 1000, fake, None, 1, 1000, 1.0, 1025, 1.0, 0, None, None) == BAD
    assert f(fake, 1000, fake, None, 1, 1000, 1.0, 50, 0.0, 0, None, None) == BAD          # p out of (0, 1]
    assert f(fake, 1000, fake, None, 1, 1000, 1.0, 50, 1.5, 0, None, None) == BAD
    assert f(fake, 1000, fake, None, 1, 1000, 1.0, 50, float("nan"), 0, None, None) == BAD
    assert f(fake, 1000, fake, None, 1, 1000, 1.0, 0, 0.9, 0, None, None) == UNSUPPORTED   # full-vocabulary nucleus


def test_decode_devlen_kv_append_advance_validation(lib):
    a = lib.aria_attention_decode_devlen
    ws = lib.aria_attention_decode_workspace_bytes(2, 4, 512)
    args = [fake, fake, fake, fake, None, 0, fake, 2, 4, 512, 4 * 512 * 128, 512 * 128, 4 * 512 * 128, 512 * 128, 0.1, fake, ws, None]
    bad_lens = list(args)
    bad_lens[6] = None
    assert a(*bad_lens) == BAD                                    # lens is required
    short_mask = list(args)
    short_mask[4], short_mask[5] = fake, 511
    assert a(*short_mask) == BAD                                  # key-mask row stride < T_max
    small_ws = list(args)
    small_ws[16] = ws - 1
    assert a(*small_ws) == BAD
    zero_b = list(args)
    zero_b[7] = 0
    assert a(*zero_b) == BAD

    k = lib.aria_kv_append
    assert k(None, fake, 512, 128, fake, fake, 4 * 512 * 128, 512 * 128, fake, 2, 4, 512, None) == BAD
    assert k(fake, fake, 512, 128, fake, fake, 4 * 512 * 128, 512 * 128, None, 2, 4, 512, None) == BAD   # pos required
    assert k(fake, fake, 512, 100, fake, fake, 4 * 512 * 128, 512 * 128, fake, 2, 4, 512, None) == BAD   # stride % 8
    assert k(fake, fake, 512, 128, fake, fake, 4 * 512 * 128, 512 * 128, fake, 2, 4, 0, None) == BAD     # T_max = 0

    d = lib.aria_decode_advance
    ok = [fake] * 3 + [16] + [fake] * 7 + [None, 0, 0, 4, None]
    for i in (0, 1, 2, 4, 5, 6, 7, 8, 9, 10):
        bad = list(ok)
        bad[i] = None
        assert d(*bad) == BAD, i
    eos = (ctypes.c_int64 * 9)(*range(9))
    for i, v in ((3, 0), (14, 0), (14, 1025), (12, 9), (12, -1)):
        bad = list(ok)
        bad[i] = v
        if i == 12:
            bad[11] = ctypes.cast(eos, ctypes.c_void_p)
        assert d(*bad) == BAD, (i, v)
    bad = list(ok)
    bad[12] = 2                                                   # EOS ids without the array
    assert d(*bad) == BAD


def _cpu_model():
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    return AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device="cpu")


@pytest.mark.parametrize("kw,exc", [
    (dict(max_new_tokens=0), ValueError),
    (dict(max_new_tokens=2.5), ValueError),
    (dict(do_sample=True, temperature=0.0), ValueError),
    (dict(do_sample=True, temperature=float("nan")), ValueError),
    (dict(do_sample=True, top_k=-1), ValueError),
    (dict(do_sample=True, top_k=1025), NotImplementedError),
    (dict(do_sample=True, top_p=0.0), ValueError),
    (dict(do_sample=True, top_p=1.2), ValueError),
    (dict(do_sample=True, top_k=0, top_p=0.9), NotImplementedError),
    (dict(eos_token_id=list(range(9))), ValueError),
    (dict(eos_token_id="2"), ValueError),
    (dict(seed=-1), ValueError),
    (dict(poll_every=0), ValueError),
    (dict(attention_mask=torch.ones(2, 5, dtype=torch.long)), ValueError),
])
def test_generate_rejects_bad_arguments_before_device_work(kw, exc):
    m = _cpu_model()
    ids = torch.randint(10, 500, (1, 6))
    with pytest.raises(exc):
        m.generate(ids, **kw)


def test_generate_checks_input_shape_and_pad_default():
    from aria_b200.modeling_aria import AriaForConditionalGeneration as A
    with pytest.raises(ValueError):
        A._check_generate_args(torch.zeros(6, dtype=torch.long), 4, None, False, 1.0, 50, 1.0, None, None, 0, 8)
    with pytest.raises(NotImplementedError):
        A._check_generate_args(torch.zeros(1025, 2, dtype=torch.long), 4, None, False, 1.0, 50, 1.0, None, None, 0, 8)
    # greedy ignores the sampling knobs, as GenerationMixin does without do_sample
    assert A._check_generate_args(torch.zeros(2, 3, dtype=torch.long), 4, None, False, 0.0, 0, 0.5, [7, 9], None, 0, 8) == (2, 3, (7, 9), 7)
    assert A._check_generate_args(torch.zeros(2, 3, dtype=torch.long), 4, None, True, 0.8, 200, 1.0, 5, 0, 0, 8) == (2, 3, (5,), 0)
