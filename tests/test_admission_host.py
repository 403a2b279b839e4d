"""CPU: batched and chunked admission in the continuous-batching engine — the chunk planner of serving.Scheduler and the
admission loop of Engine.step() with stand-ins for its device work (no GPU)."""
import random

import pytest

import torch

from aria_b200 import serving
from aria_b200.serving import PAGE, Request, Scheduler, page_keys


class _NoDevice:
    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) in a host-only test")


class _StandInModel:
    from aria_b200.modeling_aria import AriaForConditionalGeneration as _M
    _check_generate_args = staticmethod(_M._check_generate_args)
    device = torch.device("cuda:0")


class _Graph:
    def replay(self):
        pass


def _ids(T, seed=0):
    return torch.randint(10, 1000, (T,), generator=torch.Generator().manual_seed(seed))


def _host_engine(monkeypatch, max_batch=4, n_pages=17, budget=None):
    """An Engine with its host half only; _admit records, _launch records the packed launches (as (rid, start, end) lists),
    and the decode replays and polls are left out (the tests retire requests themselves)."""
    monkeypatch.setattr(serving, "ops", _NoDevice())
    eng = object.__new__(serving.Engine)
    eng.model = _StandInModel()
    eng.eos, eng.pad, eng.poll_every = (), 0, 8
    eng.sched = Scheduler(max_batch, n_pages)
    eng._next_rid = 0
    eng._undelivered = {}
    eng.max_prefill_tokens = budget
    eng.max_batch, eng.max_pages = max_batch, n_pages - 1
    eng.stats = {"steps": 0, "active_slot_steps": 0}
    eng.launches = []
    eng._graph = lambda n, w: _Graph()
    eng._poll_and_retire = lambda: {}
    eng._admit = lambda s, req: eng._staged.append(req)

    def launch():
        staged, eng._staged = eng._staged, []
        eng.sched.unlaunched.clear()
        if staged:
            eng.launches.append([(r.rid, *r.chunk) for r in staged])
    eng._launch = launch
    return eng


# ------------------------------------------------------------------------------------------------ the planner
def test_chunk_end_is_page_aligned_and_the_last_chunk_holds_the_last_token():
    ce = Scheduler.chunk_end
    assert ce(1500, 0, None) == 1500 and ce(1500, 0, 4096) == 1500 and ce(1500, 0, 1500) == 1500
    assert ce(1500, 0, 512) == 512 and ce(1500, 512, 512) == 1024 and ce(1500, 1024, 512) == 1500
    assert ce(1500, 256, 700) == 768                        # the end is a multiple of 256 of the absolute position
    assert ce(1500, 256, 255) == 256                        # not one page fits: nothing
    assert ce(300, 256, 44) == 300                          # a prompt's final piece may be short


def test_a_long_prompt_runs_in_page_aligned_chunks_within_the_budget(monkeypatch):
    eng = _host_engine(monkeypatch, budget=512)
    eng.add_request(_ids(1500), max_new_tokens=4)
    for _ in range(3):
        eng.step()
    assert eng.launches == [[(0, 0, 512)], [(0, 512, 1024)], [(0, 1024, 1500)]]
    assert eng.sched.partial is None and eng.sched.n_active == 1


def test_requests_pack_into_one_launch_and_fifo_holds(monkeypatch):
    eng = _host_engine(monkeypatch, max_batch=8, n_pages=1 + 40, budget=1024)
    for i, T in enumerate((100, 300, 700, 50)):
        eng.add_request(_ids(T, seed=i), max_new_tokens=4)
    eng.step()
    # 100 + 300 = 400 fit; 700 does not fit the 624 left: its first chunk ends at 512, and admission stops there
    assert eng.launches == [[(0, 0, 100), (1, 0, 300), (2, 0, 512)]]
    assert eng.sched.partial.rid == 2 and [r.rid for r in eng.sched.queue] == [3]
    eng.step()
    assert eng.launches[1] == [(2, 512, 700), (3, 0, 50)]
    assert eng.sched.partial is None and not eng.sched.queue


def test_no_budget_packs_every_admission_into_one_launch(monkeypatch):
    eng = _host_engine(monkeypatch, max_batch=8, n_pages=1 + 40, budget=None)
    for i, T in enumerate((100, 3000, 700, 50)):
        eng.add_request(_ids(T, seed=i), max_new_tokens=4)
    eng.step()
    assert eng.launches == [[(0, 0, 100), (1, 0, 3000), (2, 0, 700), (3, 0, 50)]]


def test_a_partly_prefilled_request_holds_its_slot_and_pages(monkeypatch):
    eng = _host_engine(monkeypatch, max_batch=2, n_pages=1 + 12, budget=256)
    eng.add_request(_ids(1000), max_new_tokens=24)          # 4 pages
    eng.add_request(_ids(10, seed=1), max_new_tokens=4)
    eng.add_request(_ids(10, seed=2), max_new_tokens=4)
    eng.step()
    req = eng.sched.partial
    assert req.rid == 0 and len(req.pages) == 4 and all(eng.sched.pages.refs(p) == 1 for p in req.pages)
    assert eng.sched.n_active == 1 and eng.sched.pages.n_free == 12 - 4
    for _ in range(3):
        eng.step()
    # the last chunk leaves 24 tokens of the budget: the next request fits them; max_batch 2: the third one waits
    assert eng.sched.partial is None and eng.launches[3] == [(0, 768, 1000), (1, 0, 10)]
    assert eng.sched.n_active == 2 and [r.rid for r in eng.sched.queue] == [2]


def test_only_prefilled_pages_are_keyed():
    s = Scheduler(max_batch=4, n_pages=1 + 8)
    r = Request(0, _ids(900), 4, (0.0, 0, 1.0, 0))
    r.keys = page_keys(r.input_ids)
    s.submit(r)
    s.admit_one()
    s.plan(r, 0, 512)
    s.register(r)
    assert s.pages.n_cached == 2 and s.unlaunched == set(r.pages[:2])
    s.plan(r, 512, 512)
    s.register(r)
    assert s.pages.n_cached == 3 and s.partial is None


def test_a_hit_on_an_unlaunched_prefill_launches_it_first(monkeypatch):
    """Identical prompts in one burst: each later one hits the first one's pages, so the first launch must run before the
    second request's; the third joins the second's launch (its hits are launched by then) and every prefix_len is what
    one-at-a-time admission gives."""
    eng = _host_engine(monkeypatch, max_batch=8, n_pages=1 + 40, budget=4096)
    ids = _ids(700)
    for i in range(3):
        eng.add_request(ids.clone(), max_new_tokens=4)
    eng.add_request(_ids(300, seed=5), max_new_tokens=4)
    eng.step()
    assert eng.launches == [[(0, 0, 700)], [(1, 512, 700), (2, 512, 700), (3, 0, 300)]]
    assert [r.prefix_len for r in eng.sched.slots] == [0, 512, 512, 0]


def _one_at_a_time_prefix_lens(reqs, max_batch, n_pages):
    s = Scheduler(max_batch, n_pages)
    for r in reqs:
        s.submit(r)
    out = {}
    while (a := s.admit_one()) is not None:
        out[a[1].rid] = a[1].prefix_len
        s.register(a[1])
    return out


def test_packed_admission_hits_what_one_at_a_time_admission_hits(monkeypatch):
    rng = random.Random(3)
    bases = [_ids(rng.randint(300, 1400), seed=40 + i) for i in range(3)]
    prompts = [torch.cat([bases[rng.randrange(3)][:rng.randint(200, 1400)], _ids(rng.randint(1, 300), seed=i)])
               for i in range(24)]
    for budget in (256, 512, 1024, 4096, None):
        reqs = [Request(i, p, 8, (0.0, 0, 1.0, 0)) for i, p in enumerate(prompts)]
        for r in reqs:
            r.keys = page_keys(r.input_ids)
        want = _one_at_a_time_prefix_lens(reqs, 64, 1 + 200)
        eng = _host_engine(monkeypatch, max_batch=64, n_pages=1 + 200, budget=budget)
        for p in prompts:
            eng.add_request(p, max_new_tokens=8)
        while eng.sched.queue or eng.sched.partial is not None:
            eng.step()
        assert {r.rid: r.prefix_len for r in eng.sched.slots} == want, budget
        pages = {r.rid: r.pages for r in eng.sched.slots}
        for launch in eng.launches:
            assert budget is None or sum(e - s for _, s, e in launch) <= budget
            assert len({rid for rid, _, _ in launch}) == len(launch)
            written = {p for rid, s, e in launch for p in pages[rid][s // PAGE:-(-e // PAGE)]}
            read = {p for rid, s, e in launch for p in pages[rid][:s // PAGE]}
            assert not read & written, budget                # a launch never reads pages it writes itself


def test_randomized_chunked_admission_with_retirements(monkeypatch):
    rng = random.Random(0)
    n_pages = 1 + 30
    bases = [_ids(rng.randint(300, 1500), seed=100 + i) for i in range(4)]
    for budget in (256, 768, 2048):
        eng = _host_engine(monkeypatch, max_batch=6, n_pages=n_pages, budget=budget)
        T = {}
        for i in range(60):
            b = bases[rng.randrange(4)]
            ids = torch.cat([b[:rng.randint(1, b.numel())], _ids(rng.randint(1, 300), seed=i)])
            T[eng.add_request(ids, max_new_tokens=rng.randint(1, 300))] = ids.numel()
        done_tokens = {}
        while eng.sched.queue or eng.sched.slots:
            n_launch = len(eng.launches)
            eng.step()
            for launch in eng.launches[n_launch:]:
                assert sum(e - s for _, s, e in launch) <= budget
                for rid, s, e in launch:
                    assert s % PAGE == 0 and (e % PAGE == 0 or e == T[rid]) and e > s
                    assert done_tokens.get(rid, s) == s         # chunks follow one another
                    done_tokens[rid] = e
            held = {}
            for r in eng.sched.slots:
                for p in r.pages:
                    held.setdefault(p, set()).add(r.rid)
            assert all(1 <= p < n_pages and eng.sched.pages.refs(p) == len(h) for p, h in held.items())
            partial = [r for r in eng.sched.slots if done_tokens.get(r.rid, r.prefix_len) < T[r.rid]]
            assert len(partial) <= 1 and (not partial or partial[0] is eng.sched.partial)
            assert eng.sched.n_active <= 6
            # retire some requests that are wholly prefilled (a poll would)
            live = [s for s, r in enumerate(eng.sched.slots) if r is not eng.sched.partial]
            for s in sorted(rng.sample(live, rng.randint(0, len(live))), reverse=True):
                eng.sched.retire(s)
        assert all(done_tokens[rid] == t for rid, t in T.items())
        assert eng.sched.pages.n_free == n_pages - 1 and all(eng.sched.pages.refs(p) == 0 for p in range(n_pages))


def _engine_with_prefill(monkeypatch, budget, prefill):
    """The host engine with the real staging and launch, and `prefill` standing in for the device prefill."""
    eng = _host_engine(monkeypatch, max_batch=4, n_pages=1 + 16, budget=budget)
    del eng._admit, eng._launch                             # back to Engine._admit / Engine._launch
    eng.stats.update(prompt_tokens=0, prefix_hit_tokens=0, pages_evicted=0)
    eng._idle = lambda lo, hi: None
    eng._prefill = prefill
    return eng


def test_a_failed_prefill_leaves_no_keyed_page_behind(monkeypatch):
    """Pages are keyed when their chunk is staged; if the launch then fails, they hold nothing known, so a resubmitted prompt
    must not hit them."""
    def oom(staged):
        raise RuntimeError("CUDA out of memory")
    ids = _ids(900)
    for budget in (None, 512):
        eng = _engine_with_prefill(monkeypatch, budget, oom)
        eng.add_request(ids, max_new_tokens=4)                # budget 512: its first chunk, pages 0 and 1 keyed
        eng.add_request(_ids(300, seed=1), max_new_tokens=4)
        with pytest.raises(RuntimeError, match="out of memory"):
            eng.step()
        assert eng.sched.n_active == 0 and eng.sched.partial is None and not eng.sched.unlaunched
        assert eng.sched.pages.n_cached == 0 and eng.sched.pages.n_free == 16
        launched = []
        eng._prefill = launched.append
        eng.add_request(ids, max_new_tokens=4)
        eng.step()
        assert [r.prefix_len for r in launched[0]] == [0], budget


def test_a_failed_later_chunk_keeps_the_pages_of_the_chunks_before_it(monkeypatch):
    eng = _engine_with_prefill(monkeypatch, 512, lambda staged: None)
    ids = _ids(1500)
    eng.add_request(ids, max_new_tokens=4)
    eng.step()                                              # chunk [0, 512) launched: pages 0 and 1 keyed
    first = list(eng.sched.partial.pages[:2])

    def oom(staged):
        raise RuntimeError("CUDA out of memory")
    eng._prefill = oom
    with pytest.raises(RuntimeError):
        eng.step()                                          # chunk [512, 1024) fails
    assert eng.sched.pages.lookup(page_keys(ids)) == first


def test_a_lone_partly_prefilled_request_runs_no_decode_steps(monkeypatch):
    eng = _host_engine(monkeypatch, max_batch=4, n_pages=1 + 16, budget=256)
    replays = []
    eng._graph = lambda n, w: type("G", (), {"replay": lambda self: replays.append(n)})()
    eng.add_request(_ids(1000), max_new_tokens=8)
    for _ in range(4):                                      # four chunks; the request decodes from the fifth step on
        eng.step()
    assert len(eng.launches) == 4 and not replays and eng.stats["steps"] == eng.stats["active_slot_steps"] == 0
    eng.add_request(_ids(600, seed=1), max_new_tokens=8)
    eng.step()                                              # the first request decodes beside the second one's first chunk
    assert replays == [1] * 8 and eng.stats["active_slot_steps"] == 8
