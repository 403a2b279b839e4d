"""CPU: the fp64 logprob reference on hand-made rows, the argument refusals of generate(output_logprobs=...) and
Engine.add_request(logprobs=..., prompt_logprobs=...) before any device work, the engine's ring-drain arithmetic, the C entry's
argument checks, and a prompt_logprobs request taking no prefix-cache hit."""
import ctypes
import math

import pytest
import torch

from aria_b200 import modeling_aria, serving
from aria_b200.serving import Request, Scheduler, page_keys, ring_entries
from logprobs_ref import token_logprobs_ref

BAD = -1
fake = ctypes.c_void_p(0x1000)   # never dereferenced: validation fails first


# ------------------------------------------------------------------------------------------------ the reference
def test_reference_ties_go_to_the_lowest_id():
    x = torch.tensor([[1.0, 3.0, 3.0, 2.0, 3.0, 0.0]])
    lp, ids, top = token_logprobs_ref(x, torch.tensor([4]), 4)
    assert ids.tolist() == [[1, 2, 4, 3]]
    z = math.log(sum(math.exp(v) for v in x[0].tolist()))
    assert lp.item() == pytest.approx(3.0 - z, abs=1e-12)
    assert top[0, :3].tolist() == pytest.approx([3.0 - z] * 3, abs=1e-12) and top[0, 3].item() == pytest.approx(2.0 - z)


def test_reference_n_past_v_and_v_equal_one():
    lp, ids, top = token_logprobs_ref(torch.tensor([[0.5, -1.0]]), torch.tensor([1]), 4)
    assert ids.tolist() == [[0, 1, -1, -1]] and top[0, 2:].tolist() == [float("-inf")] * 2
    lp, ids, top = token_logprobs_ref(torch.tensor([[7.0]]), torch.tensor([0]), 3)
    assert lp.tolist() == [0.0] and ids.tolist() == [[0, -1, -1]] and top[0, 0].item() == 0.0


def test_reference_constant_row_and_n_zero():
    V = 10
    lp, ids, top = token_logprobs_ref(torch.zeros(2, V), torch.tensor([3, 9]), 5)
    assert lp.tolist() == pytest.approx([-math.log(V)] * 2) and ids.tolist() == [list(range(5))] * 2
    lp, ids, top = token_logprobs_ref(torch.zeros(1, V), torch.tensor([0]), 0)
    assert ids.shape == (1, 0) and top.shape == (1, 0)


# ------------------------------------------------------------------------------------------------ C entry checks
@pytest.fixture(scope="module")
def lib():
    from aria_b200 import build, _lib
    build.build()
    return _lib.load()


def test_token_logprobs_entry_validation(lib):
    f = lib.aria_token_logprobs
    #       logits stride tokens R  V    n  n_row col per ring fin fill lp    ids   top   cols
    ok = [fake, 1000, fake, 1, 1000, 5, None, None, 0, 0, None, 1, fake, fake, fake, 1, None]
    for i, v in ((0, None), (2, None), (12, None), (3, 0), (3, (1 << 20) + 1), (4, 0), (4, (1 << 24) + 1), (1, -1), (5, -1),
                 (5, 21), (13, None), (14, None), (15, 0), (9, 1), (8, 1), (11, 2)):
        bad = list(ok)
        bad[i] = v
        assert f(*bad) == BAD, (i, v)
    bad = list(ok)
    bad[7], bad[9], bad[15] = fake, 3, 2                         # a ring longer than the output's columns
    assert f(*bad) == BAD


# ------------------------------------------------------------------------------------------------ refusals
class _NoDevice:
    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) before the refusal")


def _cpu_model():
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    return AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device="cpu")


@pytest.mark.parametrize("kw,exc", [
    (dict(output_logprobs=-1), ValueError),
    (dict(output_logprobs=21), ValueError),
    (dict(output_logprobs=2.0), ValueError),
    (dict(output_logprobs=True), ValueError),
    (dict(output_logprobs=3, prompt_lookup_num_tokens=2), NotImplementedError),
    (dict(output_logprobs=0), NotImplementedError),                  # the CPU step-wise path
])
def test_generate_refuses_bad_logprob_arguments_before_device_work(monkeypatch, kw, exc):
    m = _cpu_model()
    monkeypatch.setattr(modeling_aria, "ops", _NoDevice())
    with pytest.raises(exc):
        m.generate(torch.randint(10, 500, (1, 6)), max_new_tokens=4, **kw)


def test_check_output_logprobs_accepts_the_range():
    chk = modeling_aria.AriaForConditionalGeneration._check_output_logprobs
    for k in (None, 0, 5, 20):
        chk(k, None, "cuda:0")
    chk(None, 3, "cpu")                                                # no logprobs: nothing to refuse


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


@pytest.mark.parametrize("kw", [dict(logprobs=-1), dict(logprobs=21), dict(logprobs=1.5), dict(logprobs=False),
                                dict(prompt_logprobs=-2), dict(prompt_logprobs=21), dict(prompt_logprobs="5")])
def test_add_request_refuses_bad_logprob_arguments_before_device_work(monkeypatch, kw):
    eng = _host_engine(monkeypatch)
    with pytest.raises(ValueError):
        eng.add_request(torch.arange(10, 20), **kw)
    assert not eng.sched.queue


def test_add_request_takes_the_logprob_arguments(monkeypatch):
    eng = _host_engine(monkeypatch)
    eng.add_request(torch.arange(10, 20), logprobs=0, prompt_logprobs=20)
    req = eng.sched.queue[0]
    assert req.logprobs == 0 and req.prompt_logprobs == 20


# ------------------------------------------------------------------------------------------------ the ring
def test_ring_entries_wrap_around():
    assert ring_entries(0, 0, 4) == []
    assert ring_entries(0, 4, 4) == [0, 1, 2, 3]
    assert ring_entries(3, 6, 4) == [3, 0, 1]
    assert ring_entries(7, 11, 4) == [3, 0, 1, 2]


def test_ring_entries_follow_the_engine_schedule():
    """A first token and then poll_every replays per poll, with a finish anywhere: every token lands in its own live entry."""
    for poll_every in (1, 2, 3, 5, 8):
        ring = poll_every + 1
        for max_new in range(1, 30):
            ring_host = [None] * ring
            drained, n_out, got = 0, 0, []
            n_out = 1                                                  # the first token, from the admission prefill
            ring_host[0] = 0
            while True:
                for _ in range(poll_every):
                    if n_out < max_new:
                        ring_host[n_out % ring] = n_out
                        n_out += 1
                got += [ring_host[i] for i in ring_entries(drained, n_out, ring)]
                drained = n_out
                if n_out == max_new:
                    break
            assert got == list(range(max_new)), (poll_every, max_new)


def test_ring_entries_refuse_more_than_the_ring_holds():
    with pytest.raises(RuntimeError):
        ring_entries(0, 5, 4)
    with pytest.raises(RuntimeError):
        ring_entries(5, 4, 4)


# ------------------------------------------------------------------------------------------------ no prefix hit
def test_a_prompt_logprobs_request_gets_no_hit_but_its_pages_stay_keyed():
    s = Scheduler(max_batch=4, n_pages=1 + 16)
    ids = torch.arange(1000, dtype=torch.int64) % 97
    a = Request(0, ids, 4, (0.0, 0, 1.0, 0))
    a.keys = page_keys(ids)
    s.submit(a)
    s.admit_one()
    s.register(a)
    s.unlaunched = set()
    b = Request(1, ids.clone(), 4, (0.0, 0, 1.0, 0), prompt_logprobs=5)
    b.keys = page_keys(ids)
    s.submit(b)
    assert s._head_hits() == [] and s.head_fits(256) and not s.head_waits()
    _, got = s.admit_one()
    assert got is b and b.prefix_len == 0 and b.chunk == (0, 1000) and not set(b.pages) & set(a.pages)
    c = Request(2, ids.clone(), 4, (0.0, 0, 1.0, 0))                  # a plain request still hits a's pages
    c.keys = page_keys(ids)
    s.submit(c)
    assert s._head_hits() == a.pages[:3]
