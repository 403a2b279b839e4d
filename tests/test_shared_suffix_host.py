"""CPU: generate(shared_prefix_len=P) refuses what it does not serve before any device work, in a fixed order, and the suffix
prefill attention and tail scatter entries validate their arguments before any CUDA call."""
import ctypes

import pytest
import torch

BAD = -1
fake = ctypes.c_void_p(0x1000)   # never dereferenced: validation fails first
IMG = 9                          # TINY's image token


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


def _batch():
    """Three rows sharing a 6-token prefix with two image tokens; row 1 is left-padded by 2."""
    prefix = [11, IMG, IMG, 12, 13, 14]
    rows = [prefix + [20, 21, 22], [0, 0] + prefix + [30], prefix + [40, 41, 42]]
    mask = torch.tensor([[1] * 9, [0, 0] + [1] * 7, [1] * 9])
    return torch.tensor(rows), mask


def test_valid_batch_passes_the_checks():
    from aria_b200.modeling_aria import AriaForConditionalGeneration as A
    ids, mask = _batch()
    ids_host, lens = A._check_shared_prefix(ids, mask, 6, IMG, "bf16")
    assert torch.equal(ids_host, ids) and lens.tolist() == [9, 7, 9]
    assert A._check_generate_args(ids, 4, mask, False, 1.0, 50, 1.0, None, None, 0, 8, "bf16", 1, 6) == (3, 9, (), 0)
    # 1024 rows exactly pass
    assert A._check_shared_prefix(ids, mask, 6, IMG, "bf16", 341)[1].tolist() == [9, 7, 9]


@pytest.mark.parametrize("P", [0, -1, 2.0, "6", True])
def test_prefix_length_must_be_a_positive_int(P):
    ids, mask = _batch()
    with pytest.raises(ValueError, match="shared_prefix_len must be a positive int"):
        _cpu_model().generate(ids, attention_mask=mask, shared_prefix_len=P)


@pytest.mark.parametrize("bad", [[1, 0, 1, 1, 1, 1, 1, 1, 1], [1] * 8 + [0], [0, 2] + [1] * 7])
def test_mask_must_be_left_padding(bad):
    ids, mask = _batch()
    mask[1] = torch.tensor(bad)
    with pytest.raises(ValueError, match="left-padded"):
        _cpu_model().generate(ids, attention_mask=mask, shared_prefix_len=6)


def test_every_row_needs_a_token_of_its_own():
    ids, mask = _batch()
    with pytest.raises(ValueError, match="row 1 has 7 real tokens"):
        _cpu_model().generate(ids, attention_mask=mask, shared_prefix_len=7)


def test_prefixes_must_agree_and_the_first_differing_row_is_named():
    ids, mask = _batch()
    ids[2, 4] = 99
    ids[1, 5] = 98                 # row 1's fourth real token
    with pytest.raises(ValueError, match="row 1 differ"):
        _cpu_model().generate(ids, attention_mask=mask, shared_prefix_len=6)


def test_image_token_after_the_prefix_is_refused():
    ids, mask = _batch()
    ids[2, 7] = IMG
    with pytest.raises(ValueError, match="row 2 has an image token"):
        _cpu_model().generate(ids, attention_mask=mask, shared_prefix_len=6)
    # the prefix that stops before its images leaves them in the suffixes
    ids, mask = _batch()
    with pytest.raises(ValueError, match="row 0 has an image token"):
        _cpu_model().generate(ids, attention_mask=mask, shared_prefix_len=1)


def test_fp8_cache_is_refused():
    ids, mask = _batch()
    with pytest.raises(NotImplementedError, match="fp8"):
        _cpu_model().generate(ids, attention_mask=mask, shared_prefix_len=6, kv_cache_dtype="fp8")


def test_rows_beyond_the_advance_limit_are_refused():
    ids = torch.tensor([[11, IMG, 12, 13]]).repeat(512, 1)
    with pytest.raises(NotImplementedError, match="1024"):
        _cpu_model().generate(ids, shared_prefix_len=2, do_sample=True, num_return_sequences=3)


def test_cpu_device_is_refused():
    ids, mask = _batch()
    with pytest.raises(NotImplementedError, match="GPU"):
        _cpu_model().generate(ids, attention_mask=mask, shared_prefix_len=6)


@pytest.mark.parametrize("change,kw,exc,match", [
    # generate()'s own checks come first
    ({}, dict(max_new_tokens=0, shared_prefix_len=0), ValueError, "max_new_tokens"),
    ({}, dict(num_return_sequences=2, shared_prefix_len=0), ValueError, "do_sample"),
    # then P, the mask, the lengths, the prefixes, the image tokens, the cache dtype
    ({"mask_row1": [1, 0] + [1] * 7}, dict(shared_prefix_len=0, kv_cache_dtype="fp8"), ValueError, "positive int"),
    ({"mask_row1": [1, 0] + [1] * 7}, dict(shared_prefix_len=8, kv_cache_dtype="fp8"), ValueError, "left-padded"),
    ({"ids": (2, 4, 99)}, dict(shared_prefix_len=8, kv_cache_dtype="fp8"), ValueError, "real tokens"),
    ({"ids": (2, 4, 99), "ids2": (0, 7, IMG)}, dict(shared_prefix_len=6, kv_cache_dtype="fp8"), ValueError, "differ"),
    ({"ids2": (0, 7, IMG)}, dict(shared_prefix_len=6, kv_cache_dtype="fp8"), ValueError, "image token"),
    ({}, dict(shared_prefix_len=6, kv_cache_dtype="fp8"), NotImplementedError, "fp8"),
    # and the row limit B * n <= 1024 last
    ({"ids2": (0, 7, IMG)}, dict(shared_prefix_len=6, num_return_sequences=400, do_sample=True), ValueError, "image token"),
    ({}, dict(shared_prefix_len=6, num_return_sequences=400, do_sample=True), NotImplementedError, "1024"),
])
def test_order_of_the_checks(change, kw, exc, match):
    ids, mask = _batch()
    if "mask_row1" in change:
        mask[1] = torch.tensor(change["mask_row1"])
    for k in ("ids", "ids2"):
        if k in change:
            r, c, v = change[k]
            ids[r, c] = v
    with pytest.raises(exc, match=match):
        _cpu_model().generate(ids, attention_mask=mask, **kw)


def test_prefill_entry_validation(lib):
    f = lib.aria_attention_prefill_shared_prefix
    B, H, S, P, Pm = 3, 4, 300, 290, 512
    # q, k, v, prefix_k, prefix_v, cu_seqlens, out, B, H, S_tot, P, P_max, q stride_h, kv stride_h, prefix stride_h, scale,
    # stream
    ok = [fake, fake, fake, fake, fake, fake, fake, B, H, S, P, Pm, S * 128, S * 128, Pm * 128, 0.1, None]

    def call(**changes):
        args = list(ok)
        for i, v in changes.items():
            args[int(i[1:])] = v
        return f(*args)

    for i in range(7):                                       # every pointer is required
        assert call(**{f"a{i}": None}) == BAD, i
    for i in (7, 8, 9, 10):                                  # B, H, S_tot, P > 0
        assert call(**{f"a{i}": 0}) == BAD, i
    assert call(a9=B - 1) == BAD                             # fewer packed rows than suffixes
    assert call(a10=Pm + 1) == BAD                           # P > P_max
    assert call(a12=S * 128 - 8) == BAD                      # head strides shorter than the rows they hold
    assert call(a13=S * 128 - 8) == BAD
    assert call(a14=Pm * 128 - 8) == BAD
    assert call(a12=S * 128 + 4) == BAD                      # strides % 8
    assert call(a13=S * 128 + 4) == BAD
    assert call(a14=Pm * 128 + 4) == BAD
    assert call(a8=1 << 24, a9=1 << 20, a12=(1 << 27) + 128, a13=(1 << 27) + 128) == BAD   # grid >= 2^31


def test_scatter_entry_validation(lib):
    f = lib.aria_kv_scatter_tails
    B, n, H, S, N = 3, 4, 2, 300, 512
    # k, v, src stride_h, tail_k, tail_v, tail stride_b, tail stride_h, cu_seqlens, B, n, H, S_tot, N_max, stream
    ok = [fake, fake, S * 128, fake, fake, H * N * 128, N * 128, fake, B, n, H, S, N, None]

    def call(**changes):
        args = list(ok)
        for i, v in changes.items():
            args[int(i[1:])] = v
        return f(*args)

    for i in (0, 1, 3, 4, 7):
        assert call(**{f"a{i}": None}) == BAD, i
    for i in (8, 9, 10, 11, 12):                             # B, n, H, S_tot, N_max > 0
        assert call(**{f"a{i}": 0}) == BAD, i
    assert call(a11=B - 1) == BAD
    assert call(a2=S * 128 - 8) == BAD
    assert call(a6=N * 128 - 8) == BAD
    assert call(a2=S * 128 + 4) == BAD
    assert call(a5=H * N * 128 + 4) == BAD
    assert call(a6=N * 128 + 4) == BAD
    assert call(a5=H * N * 128 - 8) == BAD                   # tails of two rows overlap
    assert call(a10=1 << 12, a11=1 << 20, a2=(1 << 27) + 128, a5=(1 << 12) * N * 128) == BAD   # S_tot * H >= 2^31


def test_ops_refuse_cpu_tensors():
    from aria_b200 import ops
    z = torch.zeros(1, 2, 256, 128, dtype=torch.bfloat16)
    cu = torch.tensor([0, 3, 7], dtype=torch.int32)
    with pytest.raises(RuntimeError):
        ops.attention_prefill_shared_prefix(z, z, z, 7, z, z, 128, cu, 0.1)
    with pytest.raises(RuntimeError):
        ops.kv_scatter_tails(z, z, 7, torch.zeros(4, 2, 256, 128, dtype=torch.bfloat16), torch.zeros(4, 2, 256, 128,
                             dtype=torch.bfloat16), cu, 2)
