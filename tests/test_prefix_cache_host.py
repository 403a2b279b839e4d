"""CPU: prefix caching in the continuous-batching scheduler — the page keys (serving.page_keys), the cache lookup, reference
counts, eviction order and the admission check of serving.Scheduler / serving.PageAllocator."""
import random

import pytest
import torch

from aria_b200 import serving
from aria_b200.serving import PAGE, PageAllocator, Request, Scheduler, page_keys

IMG = 7


class _NoDevice:
    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) in a host-only test")


class _StandInModel:
    """What Engine.add_request reads of a model for a text prompt: no config."""

    from aria_b200.modeling_aria import AriaForConditionalGeneration as _M
    _check_generate_args = staticmethod(_M._check_generate_args)
    device = torch.device("cuda:0")


def _host_engine(monkeypatch, max_batch=4, n_pages=9):
    """An Engine with its host half only (the attributes step() and add_request() read)."""
    monkeypatch.setattr(serving, "ops", _NoDevice())
    eng = object.__new__(serving.Engine)
    eng.model = _StandInModel()
    eng.eos, eng.pad, eng.poll_every = (), 0, 8
    eng.sched = Scheduler(max_batch, n_pages)
    eng._next_rid = 0
    eng._undelivered = {}
    return eng


def _ids(T, seed=0):
    return torch.randint(10, 1000, (T,), generator=torch.Generator().manual_seed(seed))


def _req(rid, ids, new, keys=True):
    r = Request(rid, ids, new, (0.0, 0, 1.0, 0))
    if keys:
        r.keys = page_keys(ids)
    return r


def _image_prompt(T, at, n_img, rows, seed=0):
    """A prompt of T tokens with rows x n_img image tokens from position `at` on, and pixel rows [rows, 3, 28, 28]."""
    ids = _ids(T, seed)
    ids[at:at + rows * n_img] = IMG
    pv = torch.randn(rows, 3, 28, 28, generator=torch.Generator().manual_seed(seed + 1))
    return ids, pv


# ------------------------------------------------------------------------------------------------ page keys
def test_only_full_prompt_pages_are_keyed():
    for T, n in ((1, 0), (255, 0), (256, 1), (257, 1), (511, 1), (512, 2), (1000, 3)):
        keys = page_keys(_ids(T))
        assert len(keys) == n and len(set(keys)) == n and all(len(k) == 16 for k in keys)


def test_keys_are_a_chain_one_token_changes_every_later_key():
    a = _ids(1100, seed=1)
    ka = page_keys(a)
    for t in (0, 255, 256, 700, 1023):
        b = a.clone()
        b[t] += 1
        kb = page_keys(b)
        i = t // PAGE
        assert kb[:i] == ka[:i] and all(x != y for x, y in zip(ka[i:], kb[i:])), t
    # a token past the last full page changes no key; a longer prompt with the same start shares every key of the shorter one
    b = a.clone()
    b[1050] += 1
    assert page_keys(b) == ka
    assert page_keys(torch.cat([a, _ids(300, seed=9)]))[:4] == ka


def test_images_change_the_keys_from_the_page_of_their_first_token_on():
    ids, pv = _image_prompt(1100, at=300, n_img=200, rows=2)        # image tokens 300 .. 699: pages 1 and 2
    base = page_keys(ids, pv, None, IMG)
    assert len(base) == 4 and base[0] == page_keys(ids)[0] and base[1] != page_keys(ids)[1]
    other = pv.clone()
    other[1, 0, 0, 0] += 1.0                                        # row 1 owns tokens 500 .. 699: page 1 (500-511) on
    ko = page_keys(ids, other, None, IMG)
    assert ko[0] == base[0] and all(x != y for x, y in zip(ko[1:], base[1:]))
    mask = torch.ones(2, 28, 28, dtype=torch.bool)
    km = page_keys(ids, pv, mask, IMG)
    assert km[0] == base[0] and all(x != y for x, y in zip(km[1:], base[1:]))
    mask2 = mask.clone()
    mask2[1, :, 20:] = False
    km2 = page_keys(ids, pv, mask2, IMG)
    assert km2[0] == base[0] and all(x != y for x, y in zip(km2[1:], km[1:]))
    # an image whose tokens all lie past the full pages changes no key
    ids3, pv3 = _image_prompt(600, at=520, n_img=40, rows=1)
    assert page_keys(ids3, pv3, None, IMG) == page_keys(ids3, -pv3, None, IMG)


def test_fp32_and_bf16_copies_of_one_image_share_keys():
    ids, pv = _image_prompt(800, at=100, n_img=64, rows=2, seed=3)
    assert page_keys(ids, pv.bfloat16(), None, IMG) == page_keys(ids, pv.bfloat16().float(), None, IMG)


def test_a_bad_image_token_count_gives_no_keys():
    ids, pv = _image_prompt(800, at=100, n_img=64, rows=2)
    ids[100] = 11                                                   # 127 image tokens for 2 rows
    assert page_keys(ids, pv, None, IMG) == []
    assert page_keys(_ids(800), pv, None, IMG) == []                # pixel rows but no image token


# ------------------------------------------------------------------------------------------------ scheduler and allocator
def test_hits_are_capped_below_the_last_prompt_token():
    for T, hits in ((256, 0), (257, 1), (511, 1), (512, 1), (513, 2), (1024, 3)):
        s = Scheduler(max_batch=4, n_pages=1 + 20)
        ids = _ids(T, seed=5)
        s.submit(_req(0, ids.clone(), 1))
        (_, a), = s.admit()
        s.register(a)
        s.submit(_req(1, ids.clone(), 1))
        (_, b), = s.admit()
        assert b.prefix_len == hits * PAGE and b.pages[:hits] == a.pages[:hits], T
        assert not set(b.pages[hits:]) & set(a.pages), T


def test_refcounts_lru_and_reverse_order_eviction():
    s = Scheduler(max_batch=4, n_pages=1 + 6)
    a = _req(0, _ids(3 * PAGE + 10, seed=1), 1)                     # 4 pages, 3 keyed
    s.submit(a)
    s.admit()
    s.register(a)
    pa = list(a.pages)
    assert s.pages.n_free == 2 and s.pages.n_cached == 3
    b = _req(1, a.input_ids.clone(), 1)                             # same prompt: 3 hits, 1 own page
    s.submit(b)
    s.admit()
    assert b.pages[:3] == pa[:3] and [s.pages.refs(p) for p in pa[:3]] == [2, 2, 2] and s.pages.n_free == 1
    s.retire(0)                                                     # a's pages: the hits stay held by b, page 4 is free
    assert [s.pages.refs(p) for p in pa] == [1, 1, 1, 0] and s.pages.n_free == 2
    s.retire(0)
    assert s.pages.n_free == 6 and s.pages.n_cached == 3
    # the 3 uncached free pages go first, then the idle cached ones: a's last keyed page before its first
    c = _req(2, _ids(2 * PAGE + 300, seed=9), 300)                  # 5 pages, nothing shared
    s.submit(c)
    s.admit()
    assert s.pages.n_evicted == 2 and set(pa[1:3]) <= set(c.pages) and pa[0] not in c.pages
    assert s.pages.lookup(a.keys) == [pa[0]]                        # the chain now stops after page 0


def test_admission_counts_idle_hit_pages_against_the_free_pages():
    s = Scheduler(max_batch=4, n_pages=1 + 4)
    ids = _ids(2 * PAGE + 5, seed=2)
    a = _req(0, ids.clone(), 10)                                    # 3 pages, 2 keyed
    s.submit(a)
    s.admit()
    s.register(a)
    s.retire(0)                                                     # 4 free: 2 idle cached, 2 uncached
    b = _req(1, ids.clone(), 2 * PAGE + 200)                        # 5 pages: 2 hits + 3 more, but only 2 free that are not hits
    with pytest.raises(ValueError):
        s.submit(b)                                                 # (more than the pool: refused at submit)
    b = _req(1, ids.clone(), PAGE + 200)                            # 4 pages: 2 hits + 2 more = exactly the free pages
    s.submit(b)
    assert len(s.admit()) == 1 and b.prefix_len == 2 * PAGE and s.pages.n_free == 0
    s.retire(0)
    # a held hit does not count against the free pages: c hits a's pages while d holds them
    d = _req(2, ids.clone(), 1)
    s.submit(d)
    s.admit()
    c = _req(3, ids.clone(), 1)                                     # 3 pages: 2 held hits + the 1 free page
    s.submit(c)
    assert len(s.admit()) == 1 and c.pages[:2] == d.pages[:2] and s.pages.n_free == 0


def test_failed_admission_leaves_refcounts_as_they_were(monkeypatch):
    eng = _host_engine(monkeypatch, max_batch=4, n_pages=1 + 8)
    ids = torch.arange(10, 10 + 600)
    seen = {}

    def admit(s, req):
        if req.rid == 1:                                            # the second request hits the first one's 2 keyed pages
            seen["hit"] = req.prefix_len
            seen["refs"] = [eng.sched.pages.refs(p) for p in req.pages[:2]]
            raise ValueError("image features and image tokens do not match")

    eng._admit = admit
    eng._idle = lambda lo, hi: None
    eng.add_request(ids, max_new_tokens=5)                          # 3 pages, 2 keyed
    eng.add_request(ids.clone(), max_new_tokens=5)
    with pytest.raises(ValueError):
        eng.step()
    first = eng.sched.slots[0]
    assert seen == {"hit": 2 * PAGE, "refs": [2, 2]}
    assert [eng.sched.pages.refs(p) for p in range(9)] == [1 if p in first.pages else 0 for p in range(9)]
    assert eng.sched.pages.n_cached == 2 and eng.sched.pages.lookup(first.keys) == first.pages[:2]
    assert eng.sched.pages.n_free == 8 - 3


def test_randomized_sharing_never_hands_out_a_held_page():
    rng = random.Random(0)
    s = Scheduler(max_batch=6, n_pages=1 + 24)
    bases = [_ids(rng.randint(300, 1500), seed=100 + i) for i in range(4)]
    reqs = []
    for i in range(80):
        b = bases[rng.randrange(4)]
        ids = torch.cat([b[:rng.randint(1, b.numel())], _ids(rng.randint(1, 300), seed=i)])
        reqs.append(_req(i, ids, rng.randint(1, 300)))
    for r in reqs:
        s.submit(r)
    holders = {}                                                    # page -> set of live rids
    hit_tokens = 0
    while s.queue or s.slots:
        while (a := s.admit_one()) is not None:                     # one at a time, registered as the engine does
            r = a[1]
            n_hit = r.prefix_len // PAGE
            hit_tokens += r.prefix_len
            assert r.prefix_len <= (r.input_ids.numel() - 1) // PAGE * PAGE
            for i, p in enumerate(r.pages):
                assert 1 <= p <= 24
                if i < n_hit:
                    assert holders.get(p) or s.pages.refs(p) == 1       # a hit: cached, maybe held by others
                else:
                    assert not holders.get(p)                           # a fresh page: no live holder
                holders.setdefault(p, set()).add(r.rid)
            assert all(s.pages.refs(p) == len(holders[p]) for p in r.pages)
            s.register(r)
        for slot in sorted(rng.sample(range(len(s.slots)), rng.randint(1, len(s.slots))), reverse=True):
            r = s.slots[slot]
            for p in r.pages:
                holders[p].discard(r.rid)
            s.retire(slot)
        assert all(s.pages.refs(p) == len(h) for p, h in holders.items())
    assert hit_tokens > 0 and s.pages.n_evicted > 0
    assert s.pages.n_free == 24 and all(s.pages.refs(p) == 0 for p in range(25))


def test_text_keys_do_not_read_the_model_config(monkeypatch):
    eng = _host_engine(monkeypatch)                                 # its stand-in model has no config
    eng.add_request(torch.arange(10, 10 + 700), max_new_tokens=3)
    assert len(eng.sched.queue[0].keys) == 2


def test_allocator_refuses_a_page_freed_twice():
    a = PageAllocator(4)
    p = a.alloc(1)
    a.free(p)
    with pytest.raises(RuntimeError):
        a.free(p)
    assert serving._pages_for(PAGE + 1) == 2
