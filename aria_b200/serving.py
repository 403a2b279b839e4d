"""Continuous batching: an engine that admits and retires generation requests between graph-replayed decode steps.

    eng = Engine(model, max_batch=64, max_kv_tokens=131072, eos_token_id=None, pad_token_id=None, poll_every=8)
    rid = eng.add_request(input_ids, pixel_values=None, pixel_mask=None, max_new_tokens=16,
                          do_sample=False, temperature=1.0, top_k=50, top_p=1.0, seed=0)
    done = eng.step()   # decode replays up to the next poll, retire, admit -> {rid: ids}
    out = eng.run()     # until every request has finished -> {rid: ids}

Every request's result equals model.generate(ids[None], pixel_values, pixel_mask, max_new_tokens=m, <its sampling arguments>,
eos_token_id=E, pad_token_id=P)[0] bit for bit: the prompt ids, then the generated tokens up to and including the first EOS.
It does not depend on max_batch, poll_every, when the request arrived, its slot or the other requests, because

  - admission is generate()'s batch-1 prefill (eager forward(), ViT included) into a one-row staging cache, whose rows are then
    copied into the request's pages (ops.kv_pages_store), and its first token comes from its own sampling parameters at
    RNG offset 0;
  - a decode step reads every row's keys from its own pages with the arithmetic of the contiguous decode kernel
    (ops.attention_decode_paged: a page is one split), samples each row with its own parameters, noise row 0 and offset =
    tokens emitted (ops.sample_tokens_slots), and the other kernels of the step compute each row on its own.

Memory is a pool of 256-token pages (moe_lm.PagedKVCache) and a request reserves ceil((T + max_new_tokens) / 256) of them when
it is admitted, so it never waits for memory once running (no preemption).  Admission is FIFO.  Slots stay dense: when a
request retires, the last active slot moves into its place.  A decode step over n active slots replays the graph captured
for the smallest power of two >= n (and the smallest power of two of table columns that covers their pages); the rows past
n are idle: finished, one key on the reserved null page 0, and no write position, so they never write into a request's pages.
The host looks at the finished flags every poll_every steps.

The scheduler (Scheduler, PageAllocator) is plain host code with no device calls.  GPU only; bf16 KV pages; no expert
parallelism.  Fp8 or bf16 expert and dense weights are fine (they live inside the layers).
"""
from __future__ import annotations

import collections
import time
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch

from . import ops

PAGE = 256
MAX_BATCH = 1024   # the slot advance runs one thread per slot in one CTA


def _pages_for(tokens: int) -> int:
    return -(-tokens // PAGE)


def _pow2_at_least(n: int, cap: int) -> int:
    p = 1
    while p < n:
        p *= 2
    return min(p, cap)


class PageAllocator:
    """Free list of the pool's pages 1 .. n_pages - 1; page 0 is the null page idle slots point at, never handed out."""

    def __init__(self, n_pages: int):
        if n_pages < 2:
            raise ValueError(f"a page pool needs the null page and at least one more, got {n_pages} pages")
        self.n_pages = n_pages
        self._free = list(range(n_pages - 1, 0, -1))   # pop() hands out the lowest page first

    @property
    def n_free(self) -> int:
        return len(self._free)

    def alloc(self, n: int) -> List[int]:
        if n > len(self._free):
            raise RuntimeError(f"page pool: {n} pages asked, {len(self._free)} free")
        return [self._free.pop() for _ in range(n)]

    def free(self, pages: List[int]) -> None:
        self._free.extend(reversed(pages))


@dataclass
class Request:
    rid: int
    input_ids: torch.Tensor            # host int64 [T]
    max_new_tokens: int
    sampling: tuple                    # (temperature, top_k, top_p, seed); temperature 0 = greedy
    pixel_values: Optional[torch.Tensor] = None
    pixel_mask: Optional[torch.Tensor] = None
    pages: List[int] = field(default_factory=list)

    @property
    def n_pages(self) -> int:
        return _pages_for(self.input_ids.numel() + self.max_new_tokens)


class Scheduler:
    """FIFO admission without overcommit, dense slots, no preemption.  slots[s] is the request in slot s (s < n_active).

    admit() admits the queue's head while a slot is free and its pages are free, reserving them; retire(s) frees the pages of
    slot s and moves the last active slot into s, returning that move (src, dst) or None when s was the last slot."""

    def __init__(self, max_batch: int, n_pages: int):
        self.max_batch = max_batch
        self.pages = PageAllocator(n_pages)
        self.queue: collections.deque = collections.deque()
        self.slots: List[Request] = []

    @property
    def n_active(self) -> int:
        return len(self.slots)

    def submit(self, req: Request) -> None:
        if req.n_pages > self.pages.n_pages - 1:
            raise ValueError(f"request {req.rid} needs {req.n_pages} pages; the pool has {self.pages.n_pages - 1}")
        self.queue.append(req)

    def admit_one(self) -> Optional[tuple]:
        """-> (slot, request) for the queue's head, its pages reserved, when a slot and its pages are free; else None."""
        if not (self.queue and len(self.slots) < self.max_batch and self.queue[0].n_pages <= self.pages.n_free):
            return None
        req = self.queue.popleft()
        req.pages = self.pages.alloc(req.n_pages)
        self.slots.append(req)
        return len(self.slots) - 1, req

    def admit(self) -> List[tuple]:
        """-> [(slot, request)] admitted, in FIFO order, their pages reserved."""
        out = []
        while (a := self.admit_one()) is not None:
            out.append(a)
        return out

    def retire(self, s: int) -> Optional[tuple]:
        req = self.slots[s]
        self.pages.free(req.pages)
        req.pages = []
        last = len(self.slots) - 1
        self.slots[s] = self.slots[last]
        self.slots.pop()
        return (last, s) if s != last else None

    def width(self) -> int:
        """Block-table columns the active slots use."""
        return max((r.n_pages for r in self.slots), default=1)


class Engine:
    """Continuous batching over `model` (an AriaForConditionalGeneration on a GPU); see the module docstring.

    max_batch: decode slots (<= 1024).  max_kv_tokens: KV cache capacity in tokens, rounded up to 256-token pages (plus the
    null page); a request needs ceil((prompt + max_new_tokens) / 256) pages.  eos_token_id / pad_token_id: as generate()'s, for
    every request.  poll_every: decode steps between two looks at the finished flags.
    Memory: the page pools (2 x layers x heads x 128 bf16 values per token of max_kv_tokens, plus the null page), and one int32
    output row per slot as long as the pool, since a request may spend the whole pool on its budget: 4 x max_batch x
    256 ceil(max_kv_tokens / 256) bytes (32 MiB at the defaults, 4 GiB at 1024 slots and a 2^20-token pool).
    `stats`: graphs captured, decode steps replayed, slot-steps of active requests (mean occupancy = active_slot_steps /
    (steps * max_batch)), host seconds spent waiting in polls.  `times[rid]`: host clock (time.perf_counter) when its first
    token and its last token were known done (first poll after admission, poll that saw it finish)."""

    def __init__(self, model, max_batch: int = 64, max_kv_tokens: int = 131072, eos_token_id=None, pad_token_id=None,
                 poll_every: int = 8):
        from .moe_lm import PagedKVCache, SlotDecodeState
        if not isinstance(max_batch, int) or max_batch < 1:
            raise ValueError(f"max_batch must be a positive int, got {max_batch!r}")
        if max_batch > MAX_BATCH:
            raise NotImplementedError(f"Engine: at most {MAX_BATCH} slots, got max_batch={max_batch}")
        if not isinstance(max_kv_tokens, int) or max_kv_tokens < 1:
            raise ValueError(f"max_kv_tokens must be a positive int, got {max_kv_tokens!r}")
        _, _, eos, pad = model._check_generate_args(torch.zeros(1, 1, dtype=torch.long), 1, None, False, 1.0, 50, 1.0,
                                                    eos_token_id, pad_token_id, 0, poll_every)
        dev = model.device
        if dev.type != "cuda":
            raise NotImplementedError("Engine: continuous batching runs on the GPU only")
        if getattr(model, "_ep_transport", None) is not None:
            raise NotImplementedError("Engine: expert parallelism is not supported")
        self.model, self.dev = model, dev
        self.max_batch, self.poll_every = max_batch, poll_every
        self.eos, self.pad = eos, pad
        lm = model.language_model
        c = lm.config
        self.max_pages = _pages_for(max_kv_tokens)
        n_pages = self.max_pages + 1
        self.sched = Scheduler(max_batch, n_pages)
        self.cache = PagedKVCache(c.num_hidden_layers, n_pages, c.num_attention_heads, c.head_dim, max_batch, self.max_pages, dev)
        self.state = SlotDecodeState(max_batch, c.num_attention_heads, self.max_pages * PAGE, dev)
        self._idle(0, max_batch)
        self.rope = lm.model.rope_tables(self.max_pages * PAGE, dev)   # held here: the graphs read these tables
        self._staging = None                                            # one-row prefill cache, grown by 256-row buckets
        self._graphs: Dict[tuple, torch.cuda.CUDAGraph] = {}
        self._pool = torch.cuda.graph_pool_handle()
        self._fin_host = torch.ones(max_batch, dtype=torch.uint8).pin_memory()
        self._nout_host = torch.zeros(max_batch, dtype=torch.int32).pin_memory()
        self._event = torch.cuda.Event()
        self._next_rid = 0
        self._undelivered: Dict[int, torch.Tensor] = {}
        self._first_seen = set()
        self.stats = {"graphs_captured": 0, "steps": 0, "active_slot_steps": 0, "poll_host_s": 0.0, "polls": 0}
        self.times: Dict[int, list] = {}

    # ------------------------------------------------------------------------------------------------ public API
    def add_request(self, input_ids, pixel_values=None, pixel_mask=None, max_new_tokens: int = 16, do_sample: bool = False,
                    temperature: float = 1.0, top_k: int = 50, top_p: float = 1.0, seed: int = 0) -> int:
        """Queue one request (input_ids [T] or [1, T]; pixel inputs as generate()'s for that one row) -> its id.  Arguments are
        checked as generate() checks them, and a request that needs more pages than the pool has is refused, here, before
        any device work."""
        if not isinstance(input_ids, torch.Tensor) or input_ids.dim() not in (1, 2):
            raise ValueError("input_ids must be a tensor [T] or [1, T]")
        ids = input_ids.reshape(1, -1) if input_ids.dim() == 1 else input_ids
        if ids.shape[0] != 1:
            raise ValueError(f"add_request takes one prompt, got input_ids {tuple(input_ids.shape)}")
        self.model._check_generate_args(ids, max_new_tokens, None, do_sample, temperature, top_k, top_p, list(self.eos),
                                        self.pad, seed, self.poll_every)
        sampling = (float(temperature), int(top_k), float(top_p), int(seed)) if do_sample else (0.0, 0, 1.0, 0)
        req = Request(self._next_rid, ids[0].to("cpu", torch.int64), max_new_tokens, sampling, pixel_values, pixel_mask)
        self.sched.submit(req)
        self._next_rid += 1
        return req.rid

    @property
    def n_active(self) -> int:
        return self.sched.n_active

    @property
    def n_waiting(self) -> int:
        return len(self.sched.queue)

    def step(self) -> Dict[int, torch.Tensor]:
        """Replay the decode step poll_every times over the active slots, poll, retire the finished requests, admit what fits
        -> {rid: result [T + generated] int64 on the model's device} of the requests that finished.
        A request whose admission raises (e.g. pixel inputs that do not match its image tokens, or running out of memory in its
        prefill) is dropped, its slot and pages freed, and the error reaches the caller; the requests behind it stay queued,
        and the results this call had retired come with the next call."""
        done, self._undelivered = self._undelivered, {}
        if self.sched.n_active:
            g = self._graph(_pow2_at_least(self.sched.n_active, self.max_batch),
                            _pow2_at_least(self.sched.width(), self.max_pages))
            for _ in range(self.poll_every):
                g.replay()
            self.stats["steps"] += self.poll_every
            self.stats["active_slot_steps"] += self.poll_every * self.sched.n_active
        if self.sched.n_active:
            done.update(self._poll_and_retire())
        while (a := self.sched.admit_one()) is not None:
            s, req = a
            try:
                self._admit(s, req)
            except BaseException:
                self.sched.retire(s)                       # the last slot: nothing moves
                self._idle(s, s + 1)
                self._undelivered = done
                raise
        return done

    def run(self) -> Dict[int, torch.Tensor]:
        """step() until no request is queued or running -> {rid: result} of every request that finished meanwhile."""
        out = {}
        while self.sched.n_active or self.sched.queue or self._undelivered:
            out.update(self.step())
        return out

    # ------------------------------------------------------------------------------------------------ device side
    def _idle(self, lo: int, hi: int) -> None:
        """Make slots [lo, hi) idle: finished, one key on the null page, no write position."""
        st = self.state
        st.finished[lo:hi] = 1
        st.kv_len[lo:hi] = 1
        st.write_pos[lo:hi] = -1
        st.rope_pos[lo:hi] = 0
        st.n_out[lo:hi] = 0
        st.temperature[lo:hi] = 0.0
        self.cache.block_table[lo:hi] = -1
        self.cache.block_table[lo:hi, 0] = 0

    def _step(self, n: int) -> None:
        lm = self.model.language_model
        st = self.state.rows(n)
        emb = ops.embedding(st.ids_in, lm.get_input_embeddings().weight)
        logits = lm.decode_step(emb, self.cache, st, self.rope)
        self._sample_and_advance(st, logits[:, -1])
        self._fin_host.copy_(self.state.finished, non_blocking=True)
        self._nout_host.copy_(self.state.n_out, non_blocking=True)

    def _sample_and_advance(self, st, logits) -> None:
        ops.sample_tokens_slots(logits, st.temperature, st.top_k, st.top_p, st.seed, st.noise_row, st.rng_offset, out=st.next_ids)
        ops.decode_advance_slots(st.next_ids, st.ids_in, st.out_tokens, st.n_out, st.max_new, st.rope_pos, st.write_pos,
                                 st.kv_len, st.rng_offset, st.finished, self.eos, self.pad)

    def _graph(self, n: int, width: int) -> torch.cuda.CUDAGraph:
        """The captured step over slots [0, n) and table columns [0, width), captured on first use.  The warm-up run before the
        capture computes the very step the next replay computes; the slot rows it advanced are put back afterwards."""
        key = (n, width)
        g = self._graphs.get(key)
        if g is not None:
            return g
        self.cache.width = width
        keep = {f: getattr(self.state, f).clone() for f in self.state.SLOT_FIELDS if f != "out_tokens"}
        cur = torch.cuda.current_stream(self.dev)
        side = torch.cuda.Stream(device=self.dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            self._step(n)
        cur.wait_stream(side)
        for f, t in keep.items():
            getattr(self.state, f).copy_(t)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, pool=self._pool):
            self._step(n)
        self._graphs[key] = g
        self.stats["graphs_captured"] += 1
        return g

    def _admit(self, s: int, req: Request) -> None:
        """generate()'s batch-1 prefill into the staging cache, its rows into the request's pages, then slot s's state and its
        first token (sampled at offset 0 and recorded by the slot advance, as generate() records its first token)."""
        m, lm = self.model, self.model.language_model
        T = req.input_ids.numel()
        bucket = _pages_for(T) * PAGE
        if self._staging is None or self._staging.T_max < bucket:
            self._staging = None
            self._staging = lm.new_cache(1, bucket, self.dev)
        cache = self._staging
        cache.seq_len = 0
        out = m.forward(req.input_ids[None], req.pixel_values, req.pixel_mask, past_key_values=cache, num_logits_to_keep=1)
        row = torch.full((self.max_pages,), -1, dtype=torch.int32)
        row[:len(req.pages)] = torch.tensor(req.pages, dtype=torch.int32)
        bt = self.cache.block_table[s]
        bt.copy_(row)
        for kc, vc, kp, vp in zip(cache.k, cache.v, self.cache.k, self.cache.v):
            ops.kv_pages_store(kc, vc, T, kp, vp, bt)
        t, k, p, seed = req.sampling
        st = self.state
        st.rope_pos[s] = T - 1
        st.write_pos[s] = T - 1
        st.kv_len[s] = T
        st.temperature[s] = t
        st.top_k[s] = k
        st.top_p[s] = p
        st.seed[s] = seed - 2 ** 64 if seed >= 2 ** 63 else seed    # int64 storage of the uint64 seed
        st.noise_row[s] = 0
        st.rng_offset[s] = 0
        st.max_new[s] = req.max_new_tokens
        st.n_out[s] = 0
        st.finished[s] = 0
        self._sample_and_advance(_slot_rows(st, s), out.logits[:, -1])

    def _poll_and_retire(self) -> Dict[int, torch.Tensor]:
        t0 = time.perf_counter()
        self._event.record(torch.cuda.current_stream(self.dev))
        self._event.synchronize()
        now = time.perf_counter()
        self.stats["poll_host_s"] += now - t0
        self.stats["polls"] += 1
        fin = self._fin_host[:self.sched.n_active].tolist()
        n_out = self._nout_host[:self.sched.n_active].tolist()
        for req in self.sched.slots:
            if req.rid not in self._first_seen:
                self._first_seen.add(req.rid)
                self.times[req.rid] = [now, None]
        done = {}
        for s in range(self.sched.n_active - 1, -1, -1):   # descending: the slot moved into s is always a live one
            if not fin[s]:
                continue
            req = self.sched.slots[s]
            done[req.rid] = torch.cat([req.input_ids.to(self.dev), self.state.out_tokens[s, :n_out[s]].to(torch.int64)])
            self.times[req.rid][1] = now
            self._first_seen.discard(req.rid)
            move = self.sched.retire(s)
            if move is not None:
                src, dst = move
                for f in self.state.SLOT_FIELDS:
                    t = getattr(self.state, f)
                    t[dst].copy_(t[src])
                self.cache.block_table[dst].copy_(self.cache.block_table[src])
                fin[dst] = fin[src]
                n_out[dst] = n_out[src]
            self._idle(self.sched.n_active, self.sched.n_active + 1)
        return done


def _slot_rows(st, s: int):
    """The one-slot view [s, s + 1) of a SlotDecodeState (what the sampler and the slot advance read)."""
    v = object.__new__(type(st))
    for f in st.SLOT_FIELDS:
        setattr(v, f, getattr(st, f)[s:s + 1])
    return v
