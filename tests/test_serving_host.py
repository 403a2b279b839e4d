"""CPU: the continuous-batching scheduler (serving.Scheduler, serving.PageAllocator) and the engine's refusals.  The scheduler is
plain host code; the refusals are raised before any device work, which the stand-ins below would turn into an error."""
import random

import pytest
import torch

from aria_b200 import serving
from aria_b200.modeling_aria import AriaForConditionalGeneration
from aria_b200.serving import Engine, PageAllocator, Request, Scheduler


def _req(rid, T, new):
    return Request(rid, torch.zeros(T, dtype=torch.int64), new, (0.0, 0, 1.0, 0))


class _NoDevice:
    """Stand-in for the `ops` module: any kernel call is a test failure."""

    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) before the refusal")


class _StandInModel:
    """What Engine reads of a model before it allocates anything."""

    _check_generate_args = staticmethod(AriaForConditionalGeneration._check_generate_args)

    def __init__(self, device="cuda:0", ep=False):
        self.device = torch.device(device)
        if ep:
            self._ep_transport = object()


def _host_engine(monkeypatch, max_batch=4, n_pages=9, eos=(), pad=0):
    """An Engine with its host half only: the scheduler, the checked defaults, and no device state."""
    monkeypatch.setattr(serving, "ops", _NoDevice())
    eng = object.__new__(Engine)
    eng.model = _StandInModel()
    eng.eos, eng.pad, eng.poll_every = eos, pad, 8
    eng.sched = Scheduler(max_batch, n_pages)
    eng._next_rid = 0
    eng._undelivered = {}
    return eng


def test_pages_needed_is_prompt_plus_budget_in_256_token_pages():
    assert _req(0, 1, 1).n_pages == 1
    assert _req(0, 200, 56).n_pages == 1
    assert _req(0, 200, 57).n_pages == 2
    assert _req(0, 1000, 24).n_pages == 4
    assert _req(0, 4097, 16).n_pages == 17


def test_allocator_never_hands_out_the_null_page_or_a_page_twice():
    a = PageAllocator(6)
    got = a.alloc(3) + a.alloc(2)
    assert sorted(got) == [1, 2, 3, 4, 5] and a.n_free == 0
    with pytest.raises(RuntimeError):
        a.alloc(1)
    a.free(got[1:3])
    assert a.n_free == 2 and set(a.alloc(2)) == set(got[1:3])
    with pytest.raises(ValueError):
        PageAllocator(1)


def test_fifo_admission_without_overcommit():
    s = Scheduler(max_batch=3, n_pages=1 + 6)          # 6 usable pages
    reqs = [_req(0, 300, 100), _req(1, 10, 10), _req(2, 600, 10), _req(3, 1, 1), _req(4, 1, 1)]   # 2, 1, 3, 1, 1 pages
    for r in reqs:
        s.submit(r)
    adm = s.admit()
    assert [(slot, r.rid) for slot, r in adm] == [(0, 0), (1, 1), (2, 2)]   # 6 pages, 3 slots: full
    assert s.pages.n_free == 0 and [r.rid for r in s.queue] == [3, 4]
    assert s.admit() == []
    # retiring slot 1 frees a slot and one page; the last slot moves into it
    assert s.retire(1) == (2, 1)
    assert [r.rid for r in s.slots] == [0, 2]
    assert [r.rid for _, r in s.admit()] == [3]          # FIFO: request 3 before 4, and 4 does not fit a slot
    assert [r.rid for r in s.slots] == [0, 2, 3] and [r.rid for r in s.queue] == [4]


def test_head_of_line_request_blocks_later_smaller_ones():
    s = Scheduler(max_batch=8, n_pages=1 + 4)
    for r in (_req(0, 700, 100), _req(1, 700, 100), _req(2, 1, 1)):  # 4, 4, 1 pages
        s.submit(r)
    assert [r.rid for _, r in s.admit()] == [0]
    assert s.admit() == []                                # request 2 would fit, but FIFO keeps it behind request 1
    s.retire(0)
    assert [r.rid for _, r in s.admit()] == [1]


def test_request_that_can_never_fit_is_refused_at_submit():
    s = Scheduler(max_batch=4, n_pages=1 + 2)
    with pytest.raises(ValueError, match="pages"):
        s.submit(_req(0, 500, 13))                        # 3 pages > 2
    s.submit(_req(1, 500, 12))                            # exactly 2


def test_slots_stay_dense_and_every_page_comes_back_after_out_of_order_retirements():
    rng = random.Random(0)
    s = Scheduler(max_batch=5, n_pages=1 + 20)
    pending = [_req(i, rng.randint(1, 900), rng.randint(1, 300)) for i in range(40)]
    for r in pending:
        s.submit(r)
    owner = {}                                            # page -> rid, to catch a page given to two live requests
    order = []
    while s.queue or s.slots:
        for slot, r in s.admit():
            assert s.slots[slot] is r
            for p in r.pages:
                assert p not in owner and 1 <= p <= 20
                owner[p] = r.rid
            order.append(r.rid)
        assert 0 < len(s.slots) <= 5
        # retire a random subset, in a random order (what the engine does in descending slot order is one such order)
        for slot in sorted(rng.sample(range(len(s.slots)), rng.randint(1, len(s.slots))), reverse=True):
            r = s.slots[slot]
            for p in r.pages:
                del owner[p]
            before = [x.rid for x in s.slots]
            move = s.retire(slot)
            after = [x.rid for x in s.slots]
            assert len(after) == len(before) - 1 and r.rid not in after
            if move is None:
                assert slot == len(before) - 1 and after == before[:-1]
            else:
                assert move == (len(before) - 1, slot) and after[slot] == before[-1]
    assert order == list(range(40))                       # FIFO
    assert s.pages.n_free == 20 and not owner


def test_engine_refusals_before_any_device_work(monkeypatch):
    monkeypatch.setattr(serving, "ops", _NoDevice())
    with pytest.raises(NotImplementedError, match="GPU"):
        Engine(_StandInModel("cpu"))
    with pytest.raises(NotImplementedError, match="expert parallelism"):
        Engine(_StandInModel(ep=True))
    with pytest.raises(NotImplementedError, match="1024"):
        Engine(_StandInModel(), max_batch=1025)
    with pytest.raises(ValueError):
        Engine(_StandInModel(), max_batch=0)
    with pytest.raises(ValueError):
        Engine(_StandInModel(), poll_every=0)
    with pytest.raises(ValueError):
        Engine(_StandInModel(), eos_token_id=list(range(9)))


def test_add_request_refusals_before_any_device_work(monkeypatch):
    eng = _host_engine(monkeypatch, n_pages=1 + 4)
    ids = torch.arange(10, 30)
    bad = [dict(max_new_tokens=0), dict(do_sample=True, temperature=0.0), dict(do_sample=True, top_k=-1),
           dict(do_sample=True, top_p=0.0), dict(seed=-1), dict(seed=2 ** 64)]
    for kw in bad:
        with pytest.raises(ValueError):
            eng.add_request(ids, **kw)
    with pytest.raises(NotImplementedError):
        eng.add_request(ids, do_sample=True, top_k=2048)
    with pytest.raises(NotImplementedError):
        eng.add_request(ids, do_sample=True, top_k=0, top_p=0.5)
    with pytest.raises(ValueError):
        eng.add_request(torch.zeros(2, 5, dtype=torch.long))
    with pytest.raises(ValueError):
        eng.add_request(torch.zeros(0, dtype=torch.long))
    with pytest.raises(ValueError, match="pages"):
        eng.add_request(ids, max_new_tokens=4 * 256 - 19)   # 20 + 1005 tokens: 5 pages, the pool has 4
    assert eng.n_waiting == 0
    # valid requests only queue (no device work until step())
    assert eng.add_request(ids, max_new_tokens=4 * 256 - 20) == 0
    assert eng.add_request(ids[None], do_sample=True, temperature=0.7, top_k=5, top_p=0.9, seed=2 ** 64 - 1) == 1
    assert eng.n_waiting == 2 and [r.sampling for r in eng.sched.queue] == [(0.0, 0, 1.0, 0), (0.7, 5, 0.9, 2 ** 64 - 1)]


def test_pow2_buckets():
    assert [serving._pow2_at_least(n, 64) for n in (1, 2, 3, 4, 5, 33, 64)] == [1, 2, 4, 4, 8, 64, 64]
    assert serving._pow2_at_least(5, 6) == 6              # a max_batch that is not a power of two is its own last bucket


def test_failed_admission_frees_its_slot_and_pages_and_keeps_the_queue(monkeypatch):
    eng = _host_engine(monkeypatch, max_batch=4, n_pages=1 + 8)
    admitted, idled = [], []

    def admit(s, req):
        if req.rid == 1:
            raise ValueError("image features and image tokens do not match")
        admitted.append((s, req.rid))

    eng._admit = admit
    eng._idle = lambda lo, hi: idled.append((lo, hi))
    for T in (300, 10, 20, 30):                              # 2, 1, 1, 1 pages
        eng.add_request(torch.arange(10, 10 + T), max_new_tokens=5)
    with pytest.raises(ValueError, match="image"):
        eng.step()
    assert admitted == [(0, 0)] and idled == [(1, 2)]         # request 1's slot is made idle again
    assert [r.rid for r in eng.sched.slots] == [0] and eng.sched.pages.n_free == 6
    assert [r.rid for r in eng.sched.queue] == [2, 3]         # the requests behind it are still queued, in order
    eng.sched.retire(0)                                      # (request 0 done) so that this host-only step has nothing to replay
    assert eng.step() == {} and admitted[1:] == [(0, 2), (1, 3)] and eng.sched.pages.n_free == 6


def test_graph_capture_pauses_garbage_collection(monkeypatch):
    """Graph captures (the engine's step graphs, generate()'s decode graphs) run with the garbage collector paused, so a
    collection cannot release a dead object's CUDA graph or memory pool mid-capture; it is re-enabled afterwards, also when
    the capture raises, and stays off if it was off."""
    import contextlib
    import gc

    from aria_b200 import ops
    seen = []

    @contextlib.contextmanager
    def fake_graph(graph, pool=None):
        seen.append((graph, pool, gc.isenabled()))
        yield

    monkeypatch.setattr(torch.cuda, "graph", fake_graph)
    was = gc.isenabled()
    try:
        gc.enable()
        with ops.graph_capture("g", pool="p"):
            assert not gc.isenabled()
        assert seen == [("g", "p", False)] and gc.isenabled()
        with pytest.raises(RuntimeError):
            with ops.graph_capture("g"):
                raise RuntimeError("capture failed")
        assert gc.isenabled()
        gc.disable()
        with ops.graph_capture("g"):
            pass
        assert not gc.isenabled()
    finally:
        (gc.enable if was else gc.disable)()
