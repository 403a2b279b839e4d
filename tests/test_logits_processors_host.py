"""CPU: the argument checks of generate(repetition_penalty=..., min_p=..., min_new_tokens=...) and Engine.add_request(...) and
their order, before any device work; their refusal with prompt lookup and on the CPU; the engine's new slot fields moving with
their slot; and the C entries' argument checks."""
import ctypes

import pytest
import torch

from aria_b200 import modeling_aria, serving
from aria_b200.serving import Scheduler

BAD = -1
fake = ctypes.c_void_p(0x1000)   # never dereferenced: validation fails first
check = modeling_aria.AriaForConditionalGeneration._check_logits_processors


class _NoDevice:
    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) before the refusal")


def _cpu_model():
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    return AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device="cpu")


BAD_VALUES = [dict(repetition_penalty=0.0), dict(repetition_penalty=-1.2), dict(repetition_penalty=float("inf")),
              dict(repetition_penalty=float("nan")), dict(repetition_penalty="1.1"), dict(repetition_penalty=True),
              dict(min_p=-0.1), dict(min_p=1.5), dict(min_p=float("nan")), dict(min_p=None),
              dict(min_new_tokens=-1), dict(min_new_tokens=2.0), dict(min_new_tokens=True)]


@pytest.mark.parametrize("kw", BAD_VALUES)
def test_generate_refuses_bad_values_before_device_work(monkeypatch, kw):
    m = _cpu_model()
    monkeypatch.setattr(modeling_aria, "ops", _NoDevice())
    with pytest.raises(ValueError):
        m.generate(torch.randint(10, 500, (1, 6)), max_new_tokens=4, **kw)


@pytest.mark.parametrize("kw", [dict(repetition_penalty=1.2), dict(min_p=0.1), dict(min_new_tokens=2)])
def test_generate_refuses_the_cpu_and_prompt_lookup(monkeypatch, kw):
    m = _cpu_model()
    monkeypatch.setattr(modeling_aria, "ops", _NoDevice())
    with pytest.raises(NotImplementedError, match="GPU only"):
        m.generate(torch.randint(10, 500, (1, 6)), max_new_tokens=4, **kw)
    with pytest.raises(NotImplementedError, match="prompt_lookup"):
        m.generate(torch.randint(10, 500, (1, 6)), max_new_tokens=4, prompt_lookup_num_tokens=2, **kw)


def test_the_order_of_the_checks(monkeypatch):
    m = _cpu_model()
    monkeypatch.setattr(modeling_aria, "ops", _NoDevice())
    ids = torch.randint(10, 500, (1, 6))
    with pytest.raises(ValueError, match="max_new_tokens"):          # generate()'s own checks come first
        m.generate(ids, max_new_tokens=0, repetition_penalty=0.0)
    with pytest.raises(ValueError, match="repetition_penalty"):      # then the values, before prompt lookup and the device
        m.generate(ids, max_new_tokens=4, repetition_penalty=0.0, prompt_lookup_num_tokens=2)
    with pytest.raises(ValueError, match="min_p"):                   # then the processors, before output_logprobs
        m.generate(ids, max_new_tokens=4, min_p=2.0, output_logprobs=-1)


def test_check_returns_none_when_every_processor_is_off():
    assert check(1.0, 0.0, 0, None, "cpu") is None
    assert check(1, 0, 0, 3, "cpu") is None                          # off: nothing to refuse
    assert check(1.2, 0.05, 3, None, "cuda:0") == (1.2, 0.05, 3)
    assert check(1, 1, 0, None, "cuda:0") == (1.0, 1.0, 0)


class _StandInModel:
    _check_generate_args = staticmethod(modeling_aria.AriaForConditionalGeneration._check_generate_args)
    config = None

    def __init__(self):
        self.device = torch.device("cuda:0")


def _host_engine(monkeypatch, max_batch=4, n_pages=17):
    monkeypatch.setattr(serving, "ops", _NoDevice())
    eng = object.__new__(serving.Engine)
    eng.model = _StandInModel()
    eng.eos, eng.pad, eng.poll_every = (), 0, 8
    eng.sched = Scheduler(max_batch, n_pages)
    eng._next_rid = 0
    eng._undelivered = {}
    return eng


@pytest.mark.parametrize("kw", BAD_VALUES)
def test_add_request_refuses_bad_values_before_device_work(monkeypatch, kw):
    eng = _host_engine(monkeypatch)
    with pytest.raises(ValueError):
        eng.add_request(torch.arange(10, 20), **kw)
    assert not eng.sched.queue


def test_add_request_checks_generate_args_first(monkeypatch):
    eng = _host_engine(monkeypatch)
    with pytest.raises(ValueError, match="max_new_tokens"):
        eng.add_request(torch.arange(10, 20), max_new_tokens=0, min_p=3.0)
    assert not eng.sched.queue


def test_add_request_takes_the_processors(monkeypatch):
    eng = _host_engine(monkeypatch)
    eng.add_request(torch.arange(10, 20), repetition_penalty=1.1, min_p=0.05, min_new_tokens=4)
    eng.add_request(torch.arange(10, 20))
    assert eng.sched.queue[0].processors == (1.1, 0.05, 4) and eng.sched.queue[1].processors is None


def test_move_slot_moves_the_processor_fields():
    from aria_b200.moe_lm import SlotDecodeState
    st = SlotDecodeState(4, 2, 512, "cpu", lp_ring=2, vocab=1000)
    for f in ("rep_penalty", "min_p", "min_new", "presence"):
        assert f in st.SLOT_FIELDS
    assert st.presence.shape == (4, 32) and st.presence.dtype == torch.int32
    st.rep_penalty[3], st.min_p[3], st.min_new[3] = 1.3, 0.2, 7
    st.presence[3] = torch.arange(32, dtype=torch.int32)
    eng = object.__new__(serving.Engine)
    eng.state = st
    eng.cache = type("Cache", (), {"block_table": torch.zeros(4, 3, dtype=torch.int32)})()
    eng._move_slot(3, 1)
    assert float(st.rep_penalty[1]) == pytest.approx(1.3) and float(st.min_p[1]) == pytest.approx(0.2)
    assert int(st.min_new[1]) == 7 and torch.equal(st.presence[1], torch.arange(32, dtype=torch.int32))
    v = st.rows(2)
    assert v.presence.shape == (2, 32) and v.min_new.shape == (2,)


# ------------------------------------------------------------------------------------------------ C entry checks
@pytest.fixture(scope="module")
def lib():
    from aria_b200 import build, _lib
    build.build()
    return _lib.load()


def test_sample_tokens_processed_entry_validation(lib):
    f = lib.aria_sample_tokens_processed
    eos = (ctypes.c_int64 * 8)(*range(8))
    #     logits stride out  probs R  V     temp  k     p     min_p seed  pen   min_new pres noise off  per  emit per eos  n  stream
    ok = [fake, 1000, fake, None, 1, 1000, fake, fake, fake, fake, fake, fake, fake, fake, None, fake, 0, fake, 0, eos, 2, None]
    for i, v in ((0, None), (2, None), (6, None), (7, None), (8, None), (9, None), (10, None), (11, None), (12, None), (13, None),
                 (15, None), (17, None), (4, 0), (4, (1 << 20) + 1), (5, 0), (5, (1 << 18) + 1), (1, -1), (20, -1), (20, 9),
                 (19, None)):
        bad = list(ok)
        bad[i] = v
        assert f(*bad) == BAD, (i, v)


def test_presence_set_entry_validation(lib):
    f = lib.aria_presence_set
    #     ids  stride R  T  lengths clear bitmap V    stream
    ok = [fake, 10, 1, 10, None, 1, fake, 1000, None]
    for i, v in ((0, None), (6, None), (2, 0), (2, (1 << 20) + 1), (3, 0), (1, -1), (7, 0), (7, (1 << 18) + 1)):
        bad = list(ok)
        bad[i] = v
        assert f(*bad) == BAD, (i, v)
