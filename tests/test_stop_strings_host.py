"""CPU: stop strings.  The plain-Python restatement of the stop-check kernel (stop_ref.stops) against transformers'
StopStringCriteria on thousands of adversarial histories, for a byte-level and a SentencePiece-style tokenizer at a small
vocabulary and at V = 100,352; the vocabulary table against HF's cleaned vocabulary; generate()'s argument checks and their
order before any device work; and the C entry's argument checks."""
import ctypes

import pytest
import torch

import stop_ref
from aria_b200 import modeling_aria, stopping

_TOKS = {}


def _tok(kind, V):
    if (kind, V) not in _TOKS:
        make = stop_ref.byte_level_tokenizer if kind == "byte" else stop_ref.sentencepiece_tokenizer
        _TOKS[kind, V] = make(V)
    return _TOKS[kind, V]


@pytest.mark.parametrize("kind", ["byte", "sp"])
@pytest.mark.parametrize("V", [1000, 100352])
def test_restatement_equals_hf(kind, V):
    from transformers.generation.stopping_criteria import StopStringCriteria
    tok = _tok(kind, V)
    table = stopping.vocab_table(tok)
    n = fired = 0
    # HF's own tables for 16 strings of 128 characters take minutes to build at V = 100,352: one such string there
    big = dict(sizes=((1, 4), (2, 24)), extra=((1, 1), (1, 128))) if V > 1000 else {}
    for strings, hist in stop_ref.cases(tok, 30 if V == 1000 else 3, 200 if V == 1000 else 300, seed=V + len(kind), **big):
        want = StopStringCriteria(tok, list(strings))(hist, None).tolist()
        got = [stop_ref.stops(table, strings, h) for h in hist.tolist()]
        assert got == want, strings
        n += len(got)
        fired += sum(want)
    assert 0.1 * n < fired < 0.9 * n


@pytest.mark.parametrize("kind", ["byte", "sp"])
def test_table_is_hf_cleaned_vocabulary(kind):
    from transformers.generation.stopping_criteria import StopStringCriteria
    tok = _tok(kind, 1000)
    table = stopping.vocab_table(tok)
    assert stopping.vocab_table(tok) is table
    clean, idx = StopStringCriteria.clean_tokenizer_vocab(tok)
    data, off = bytes(table.data.numpy()), table.offsets.tolist()
    assert table.V == max(idx) + 1 and len(off) == table.V + 1
    for s, i in zip(clean, idx):
        assert data[off[i]:off[i + 1]] == s.encode("utf-8", "surrogatepass")
    if kind == "byte":
        assert data[off[tok.convert_tokens_to_ids("Ġstop")]:off[tok.convert_tokens_to_ids("Ġstop") + 1]] == b" stop"
    else:
        assert "" in clean                                   # "<e>"
        nl = tok.convert_tokens_to_ids("<0x0A>")
        assert data[off[nl]:off[nl + 1]] == b"\n"


def test_missing_ids_inside_the_table_match_nothing():
    t = stopping.StopVocab({0: "a", 2: "b"})
    assert t.V == 3 and bytes(t.data.numpy()) == b"a\xffb"
    assert stop_ref.stops(t, ["ab"], [0, 2]) and not stop_ref.stops(t, ["ab"], [0, 1, 2])
    assert not stop_ref.stops(t, ["b"], [2, 7])            # an id past the table


def test_stop_set_encoding():
    data, lens, lookback = stopping.encode_stop_set(["<|im_end|>", "日本", "é"])
    assert lens.tolist()[:4] == [10, 6, 2, 0] and lookback == 10
    assert bytes(data[1, :6].numpy()) == "日本".encode() and data.shape == (16, 512)
    tail, n = stopping.prompt_tail(torch.arange(200).view(1, 200))
    assert n == 128 and tail[0, 0] == 72 and tail[0, -1] == 199
    tail, n = stopping.prompt_tail(torch.arange(5).view(1, 5))
    assert n == 5 and tail[0, -5:].tolist() == [0, 1, 2, 3, 4]


class _NoDevice:
    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) before the refusal")


def _cpu_model():
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    return AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device="cpu")


TOK = object()   # never used: every case is refused before the vocabulary is read
REFUSALS = [
    (dict(stop_strings=5, tokenizer=TOK), ValueError, "str"),
    (dict(stop_strings=[], tokenizer=TOK), ValueError, "str"),
    (dict(stop_strings=["a", ""], tokenizer=TOK), ValueError, "empty"),
    (dict(stop_strings="a"), ValueError, "tokenizer"),
    (dict(stop_strings=["a"] * 17, tokenizer=TOK), NotImplementedError, "16"),
    (dict(stop_strings="a" * 129, tokenizer=TOK), NotImplementedError, "128"),
    (dict(stop_strings="a", tokenizer=TOK, prompt_lookup_num_tokens=2), NotImplementedError, "prompt_lookup"),
    (dict(stop_strings="a", tokenizer=TOK), NotImplementedError, "GPU only"),
]


@pytest.mark.parametrize("kw,exc,match", REFUSALS)
def test_generate_refuses_before_device_work(monkeypatch, kw, exc, match):
    m = _cpu_model()
    monkeypatch.setattr(modeling_aria, "ops", _NoDevice())
    with pytest.raises(exc, match=match):
        m.generate(torch.randint(10, 500, (1, 6)), max_new_tokens=4, **kw)


def test_order_of_the_checks():
    check = modeling_aria.AriaForConditionalGeneration._check_stop_strings
    # the strings before the tokenizer, the tokenizer before the limits, the limits before prompt lookup and the device
    with pytest.raises(ValueError, match="empty"):
        check([""], None, (), None, 2, "cpu")
    with pytest.raises(ValueError, match="tokenizer"):
        check(["a"] * 17, None, (), None, 2, "cpu")
    with pytest.raises(NotImplementedError, match="16"):
        check(["a"] * 17, TOK, (), None, 2, "cpu")
    with pytest.raises(NotImplementedError, match="prompt_lookup"):
        check("a", TOK, (), None, 2, "cpu")
    # no EOS and no pad_token_id: refused (a stopped row is always padded); either one is enough
    with pytest.raises(ValueError, match="pad_token_id"):
        check("a", TOK, (), None, None, "cuda")
    assert check("a", TOK, (2,), None, None, "cuda") == ("a",)
    assert check(["a", "b"], TOK, (), 0, None, "cuda") == ("a", "b")
    assert check(None, None, (), None, 2, "cpu") is None


def _engine(tokenizer=None, eos=(2,)):
    """An Engine shell with what add_request's checks read, and a queue that must stay empty."""
    from aria_b200 import serving
    eng = object.__new__(serving.Engine)
    eng.model, eng.tokenizer, eng.eos, eng.pad, eng.poll_every = _cpu_model(), tokenizer, tuple(eos), 0, 8
    eng.sched = type("Sched", (), {"submit": lambda self, req: (_ for _ in ()).throw(AssertionError("queued"))})()
    eng._next_rid = 0
    return eng


ADD_REFUSALS = [
    (dict(stop_strings="a"), ValueError, "tokenizer"),
    (dict(stop_strings=[""], tokenizer=TOK), ValueError, "empty"),
    (dict(stop_strings=["a"] * 17, tokenizer=TOK), NotImplementedError, "16"),
    (dict(stop_token_ids="5"), ValueError, "stop_token_ids"),
    (dict(stop_token_ids=[]), ValueError, "stop_token_ids"),
    (dict(stop_token_ids=list(range(8))), ValueError, "more than 8"),
    (dict(stop_token_ids=[5], min_new_tokens=2), NotImplementedError, "min_new_tokens"),
    # the strings are checked before the ids, the ids before min_new_tokens
    (dict(stop_strings=[""], stop_token_ids="x", tokenizer=TOK), ValueError, "empty"),
    (dict(stop_token_ids=list(range(8)), min_new_tokens=2), ValueError, "more than 8"),
]


@pytest.mark.parametrize("kw,exc,match", ADD_REFUSALS)
def test_add_request_refuses_before_device_work(monkeypatch, kw, exc, match):
    from aria_b200 import serving
    kw = dict(kw)
    eng = _engine(kw.pop("tokenizer", None))
    monkeypatch.setattr(serving, "ops", _NoDevice())
    with pytest.raises(exc, match=match):
        eng.add_request(torch.randint(10, 500, (6,)), max_new_tokens=4, **kw)


def test_move_slot_moves_the_stop_fields():
    from aria_b200 import serving
    from aria_b200.moe_lm import SlotDecodeState
    st = SlotDecodeState(4, 2, 512, "cpu", lp_ring=2, vocab=1000)
    fields = ("stop_bytes", "stop_lens", "stop_lookback", "stop_ids", "n_stop_ids", "stop_tail", "stop_tail_len")
    for f in fields:
        assert f in st.SLOT_FIELDS
    assert st.stop_bytes.shape == (4, 16, 512) and st.stop_ids.shape == (4, 8) and st.stop_tail.shape == (4, 128)
    data, lens, lookback = stopping.encode_stop_set(["<|im_end|>", "日本"])
    st.stop_bytes[3], st.stop_lens[3], st.stop_lookback[3] = data, lens, lookback
    st.stop_ids[3, :2] = torch.tensor([11, 12])
    st.n_stop_ids[3] = 2
    st.stop_tail[3] = torch.arange(128)
    st.stop_tail_len[3] = 40
    eng = object.__new__(serving.Engine)
    eng.state = st
    eng.cache = type("Cache", (), {"block_table": torch.zeros(4, 3, dtype=torch.int32)})()
    eng._move_slot(3, 1)
    for f in fields:
        assert torch.equal(getattr(st, f)[1], getattr(st, f)[3]), f
    assert int(st.stop_lookback[1]) == 10 and int(st.n_stop_ids[1]) == 2
    v = st.rows(2)
    assert v.stop_bytes.shape == (2, 16, 512)


def test_slots_c_entry_rejects_bad_arguments():
    from aria_b200 import _lib, build
    build.build()
    lib = _lib.load()
    f = ctypes.c_void_p(0x1000)   # never dereferenced: validation fails first
    ok = [f, f, 100, f, f, f, f, f, f, f, f, 8, f, f, f, 0, 4, None]
    bad = {0: None, 2: 0, 6: None, 11: 0, 14: None, 16: 0}
    for i, v in bad.items():
        args = list(ok)
        args[i] = v
        assert lib.aria_stop_check_slots(*args) == -1, i
    args = list(ok)
    args[16] = 1025
    assert lib.aria_stop_check_slots(*args) == -1
