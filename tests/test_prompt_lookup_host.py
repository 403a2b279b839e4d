"""CPU: generate(prompt_lookup_num_tokens=K)'s argument checks and their order, the C entries' argument validation, and the
Python statement of the draft rule against transformers' PromptLookupCandidateGenerator."""
import ctypes
import random

import pytest
import torch

from prompt_lookup_ref import accept, draft

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


IDS = torch.tensor([[11, 12, 13, 11, 12], [0, 0, 14, 15, 16]])
MASK = torch.tensor([[1] * 5, [0, 0, 1, 1, 1]])


# ------------------------------------------------------------------------------------------------ generate() checks
@pytest.mark.parametrize("K", [0, 16, -1, 2.0, "4", True])
def test_num_tokens_must_be_an_int_in_1_15(K):
    with pytest.raises(ValueError, match="prompt_lookup_num_tokens"):
        _cpu_model().generate(IDS, attention_mask=MASK, prompt_lookup_num_tokens=K)


@pytest.mark.parametrize("M", [0, 17, 1.0, False])
def test_ngram_size_must_be_an_int_in_1_16(M):
    with pytest.raises(ValueError, match="max_matching_ngram_size"):
        _cpu_model().generate(IDS, attention_mask=MASK, prompt_lookup_num_tokens=4, max_matching_ngram_size=M)


def test_valid_arguments_pass_the_checks():
    from aria_b200.modeling_aria import AriaForConditionalGeneration as A
    assert A._check_prompt_lookup(2, 4, None, 1, None, "bf16", "cuda") == (4, 2)       # HF's default M = 2
    assert A._check_prompt_lookup(64, 15, 16, 1, None, "bf16", "cuda") == (15, 16)     # 64 x 16 = 1024 rows exactly


@pytest.mark.parametrize("kw,match", [
    (dict(num_return_sequences=2, do_sample=True), "num_return_sequences"),
    (dict(shared_prefix_len=1), "shared_prefix_len"),
    (dict(kv_cache_dtype="fp8"), "fp8"),
    (dict(), "GPU"),
])
def test_unsupported_combinations_are_refused(kw, match):
    with pytest.raises(NotImplementedError, match=match):
        _cpu_model().generate(IDS, attention_mask=MASK, prompt_lookup_num_tokens=4, **kw)


def test_rows_times_width_beyond_1024_are_refused():
    from aria_b200.modeling_aria import AriaForConditionalGeneration as A
    with pytest.raises(NotImplementedError, match="1024"):
        A._check_prompt_lookup(205, 4, 2, 1, None, "bf16", "cuda")      # 205 x 5 = 1025
    ids = torch.full((205, 3), 11)
    with pytest.raises(NotImplementedError, match="GPU"):               # on the CPU the device check comes first
        _cpu_model().generate(ids, prompt_lookup_num_tokens=4)


@pytest.mark.parametrize("kw,exc,match", [
    # generate()'s own checks come first
    (dict(max_new_tokens=0, prompt_lookup_num_tokens=0), ValueError, "max_new_tokens"),
    (dict(num_return_sequences=2, prompt_lookup_num_tokens=0), ValueError, "do_sample"),
    # then K, M, and the unsupported combinations in this order
    (dict(prompt_lookup_num_tokens=0, max_matching_ngram_size=0, kv_cache_dtype="fp8"), ValueError, "prompt_lookup_num_tokens"),
    (dict(prompt_lookup_num_tokens=3, max_matching_ngram_size=0, kv_cache_dtype="fp8"), ValueError, "max_matching_ngram_size"),
    (dict(prompt_lookup_num_tokens=3, num_return_sequences=2, do_sample=True, shared_prefix_len=1, kv_cache_dtype="fp8"),
     NotImplementedError, "num_return_sequences"),
    (dict(prompt_lookup_num_tokens=3, shared_prefix_len=1, kv_cache_dtype="fp8"), NotImplementedError, "shared_prefix_len"),
    (dict(prompt_lookup_num_tokens=3, kv_cache_dtype="fp8"), NotImplementedError, "fp8"),
])
def test_order_of_the_checks(kw, exc, match):
    with pytest.raises(exc, match=match):
        _cpu_model().generate(IDS, attention_mask=MASK, **kw)


def test_without_the_arguments_generate_is_unchanged():
    """max_matching_ngram_size alone does nothing (as in Hugging Face), and the CPU path still runs generate()'s stepwise decode."""
    with pytest.raises(AssertionError, match="reached the model"):
        _cpu_model().generate(IDS, attention_mask=MASK, max_matching_ngram_size=3)


# ------------------------------------------------------------------------------------------------ the draft rule
def _hf(hist, K, M, eos):
    from transformers.generation.candidate_generator import PromptLookupCandidateGenerator
    gen = PromptLookupCandidateGenerator(eos_token_id=torch.tensor(list(eos) or [-1]), num_output_tokens=K,
                                         max_matching_ngram_size=M, max_length=10 ** 6)
    ids = torch.tensor([hist])
    cand, _ = gen.get_candidates(ids)
    return cand[0, len(hist):].tolist()


CONSTRUCTED = [
    ([1, 2, 3, 1, 2, 3, 4, 1, 2], 4, 2, ()),           # repeated n-gram: the earliest match wins
    ([5, 6, 7, 8, 5, 6], 3, 2, ()),
    ([9, 1, 2, 9, 1], 10, 2, ()),                      # the continuation stops at the end of the history
    ([1, 2, 3, 4, 5], 4, 3, ()),                       # no match
    ([7, 7], 4, 2, ()),                                # M > history: n = min(M, len - 1)
    ([7], 4, 2, ()),                                   # a single token has no n-gram to match
    ([3, 4, 3, 4], 4, 16, ()),
    ([1, 2, 0, 5, 6, 1, 2], 4, 2, (5,)),               # EOS inside the candidate cuts it
    ([1, 2, 5, 6, 1, 2], 4, 2, (5,)),                  # EOS first: no draft, and no smaller n is tried
    ([4, 1, 2, 4, 9, 1, 2], 3, 2, ()),                 # n = 2 matches; n = 1 would match earlier
    ([8, 3, 1, 8, 2, 3, 1], 5, 3, ()),                 # the longest matching n wins
    ([2, 2, 2, 2, 2], 3, 2, ()),
    ([1, 2, 3, 9, 2, 3], 2, 1, ()),                    # M = 1
]


@pytest.mark.parametrize("hist,K,M,eos", CONSTRUCTED)
def test_draft_rule_matches_transformers_on_constructed_histories(hist, K, M, eos):
    assert draft(hist, K, M, eos) == _hf(hist, K, M, eos)


def test_draft_rule_matches_transformers_on_random_histories():
    rnd = random.Random(0)
    hits = 0
    for _ in range(600):
        L = rnd.randint(1, 40)
        vocab = rnd.choice([3, 6, 20])
        hist = [rnd.randrange(vocab) for _ in range(L)]
        K, M = rnd.randint(1, 15), rnd.randint(1, 16)
        eos = tuple(rnd.sample(range(vocab), rnd.randint(0, 2)))
        got = draft(hist, K, M, eos)
        assert got == _hf(hist, K, M, eos), (hist, K, M, eos)
        hits += bool(got)
    assert hits > 100


def test_draft_room_cut():
    assert draft([1, 2, 3, 4, 1, 2], 4, 2, room=1) == [3]
    assert draft([1, 2, 3, 4, 1, 2], 4, 2, room=0) == []


def test_accept_rule():
    assert accept([3, 4, 5], [3, 4, 5, 6], 0, 100) == ([3, 4, 5, 6], False)     # full acceptance: K + 1 tokens
    assert accept([3, 4, 5], [3, 9, 5, 6], 0, 100) == ([3, 9], False)           # partial
    assert accept([3, 4, 5], [7, 4, 5, 6], 0, 100) == ([7], False)              # none
    assert accept([3, 4, 5], [3, 4, 5, 6], 0, 100, eos=(4,)) == ([3, 4], True)  # EOS in the accepted run
    assert accept([3, 4, 5], [3, 4, 5, 6], 98, 100) == ([3, 4], False)          # the max_new_tokens clip
    assert accept([], [8], 0, 100) == ([8], False)


# ------------------------------------------------------------------------------------------------ C entries
def _caller(f, ok):
    def call(**changes):
        args = list(ok)
        for i, v in changes.items():
            args[int(i[1:])] = v
        return f(*args)
    return call


def test_attention_decode_multi_entry_validation(lib):
    B, Q, H, T = 3, 5, 4, 512
    # q, k, v, out, key_mask, mask stride, lens, B, Q, H, T_max, q strides b/h/q, kv strides b/h, scale, ws, ws bytes, stream
    ws = lib.aria_attention_decode_workspace_bytes(B * Q, H, T)
    ok = [fake, fake, fake, fake, None, 0, fake, B, Q, H, T, H * Q * 128, Q * 128, 128, H * T * 128, T * 128, 0.1, fake, ws, None]
    call = _caller(lib.aria_attention_decode_multi, ok)
    for i in (0, 1, 2, 3, 6, 17):
        assert call(**{f"a{i}": None}) == BAD, i
    for i in (7, 8, 9, 10):
        assert call(**{f"a{i}": 0}) == BAD, i
    assert call(a8=17) == BAD                                  # Q <= 16
    assert call(a11=H * Q * 128 + 2) == BAD                    # q strides % 4
    assert call(a13=130) == BAD
    assert call(a14=H * T * 128 + 4) == BAD                    # kv strides % 8
    assert call(a4=fake, a5=T - 1) == BAD                      # mask rows shorter than the cache
    assert call(a18=ws - 1) == BAD                             # workspace too small
    assert call(a10=65536 * 256) == BAD                        # splits are grid.y


def test_kv_append_rows_entry_validation(lib):
    B, Q, H, T = 2, 5, 4, 256
    ok = [fake, fake, H * Q * 128, Q * 128, 128, fake, fake, H * T * 128, T * 128, fake, B, Q, H, T, None]
    call = _caller(lib.aria_kv_append_rows, ok)
    for i in (0, 1, 5, 6, 9):
        assert call(**{f"a{i}": None}) == BAD, i
    for i in (10, 11, 12, 13):
        assert call(**{f"a{i}": 0}) == BAD, i
    for i in (2, 3, 4, 7, 8):
        assert call(**{f"a{i}": ok[i] + 4}) == BAD, i
    assert call(a10=1 << 20, a11=16, a12=1 << 8) == BAD        # grid >= 2^31


def test_sample_tokens_rows_entry_validation(lib):
    # logits, stride, next_ids, R, V, temperature, top_k, top_p, seed, noise_rows, offsets, stream
    ok = [fake, 100, fake, 4, 100, 1.0, 10, 0.9, 0, fake, fake, None]
    call = _caller(lib.aria_sample_tokens_rows, ok)
    for i in (0, 2, 9, 10):
        assert call(**{f"a{i}": None}) == BAD, i
    assert call(a3=0) == BAD and call(a4=0) == BAD
    assert call(a5=-1.0) == BAD and call(a6=1025) == BAD and call(a7=0.0) == BAD
    assert call(a6=0, a7=0.5) == -2                            # a full-vocabulary nucleus is unsupported, as in sample_tokens


def test_ngram_draft_entry_validation(lib):
    B, K, M = 3, 4, 2
    # hist, hist stride, hist_len, finished, n_out, max_new, drafts, draft stride, draft_len, any_draft, B, K, M, eos, n_eos, stream
    ok = [fake, 64, fake, fake, fake, 16, fake, K + 1, fake, fake, B, K, M, None, 0, None]
    call = _caller(lib.aria_ngram_draft, ok)
    for i in (0, 2, 3, 4, 6, 8, 9):
        assert call(**{f"a{i}": None}) == BAD, i
    assert call(a10=0) == BAD and call(a11=0) == BAD and call(a11=16) == BAD and call(a12=0) == BAD and call(a12=17) == BAD
    assert call(a5=0) == BAD and call(a1=0) == BAD and call(a7=K - 1) == BAD
    assert call(a14=1) == BAD and call(a14=9, a13=fake) == BAD  # EOS ids: a pointer when n_eos > 0, at most 8


def test_lookup_accept_advance_entry_validation(lib):
    B, Kp1 = 3, 5
    ok = [fake, fake, fake, Kp1, fake, fake, Kp1, fake, fake, fake, fake, fake, 16, fake, 64, fake, fake, fake, fake, fake, fake,
          fake, fake, None, 0, B, None]
    call = _caller(lib.aria_lookup_accept_advance, ok)
    for i in (0, 1, 2, 4, 5, 7, 8, 9, 10, 11, 13, 15, 16, 17, 18, 19, 20, 21, 22):
        assert call(**{f"a{i}": None}) == BAD, i
    assert call(a25=0) == BAD and call(a25=1025) == BAD       # 1 <= B <= 1024
    assert call(a3=2) == BAD                                   # the step is 1 or K + 1 wide
    assert call(a6=1, a3=1) == BAD and call(a6=17, a3=17) == BAD
    assert call(a12=0) == BAD and call(a14=0) == BAD
    assert call(a24=1) == BAD and call(a24=9, a23=fake) == BAD


def test_ops_refuse_cpu_tensors():
    from aria_b200 import ops
    z = torch.zeros(1, 2, 256, 128, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError):
        ops.attention_decode_multi(torch.zeros(1, 2, 3, 128, dtype=torch.bfloat16), z, z, torch.ones(3, dtype=torch.int32), 0.1)
    with pytest.raises(RuntimeError):
        ops.kv_append_rows(torch.zeros(1, 2, 3, 128, dtype=torch.bfloat16), torch.zeros(1, 2, 3, 128, dtype=torch.bfloat16), z, z,
                           torch.zeros(1, dtype=torch.int32))
    with pytest.raises(RuntimeError):
        ops.sample_tokens_rows(torch.zeros(2, 10, dtype=torch.bfloat16), 0.0, 0, 1.0, 0, torch.zeros(2, dtype=torch.int32),
                               torch.zeros(2, dtype=torch.int64))
