"""Continuous batching: an engine that admits and retires generation requests between graph-replayed decode steps.

    eng = Engine(model, max_batch=64, max_kv_tokens=131072, eos_token_id=None, pad_token_id=None, poll_every=8,
                 max_prefill_tokens=8192)
    rid = eng.add_request(input_ids, pixel_values=None, pixel_mask=None, max_new_tokens=16,
                          do_sample=False, temperature=1.0, top_k=50, top_p=1.0, seed=0)
    done = eng.step()   # decode replays up to the next poll, retire, admit and prefill -> {rid: ids}
    out = eng.run()     # until every request has finished -> {rid: ids}

Every request's result equals model.generate(ids[None], pixel_values, pixel_mask, max_new_tokens=m, <its sampling arguments>,
eos_token_id=E, pad_token_id=P)[0] bit for bit: the prompt ids, then the generated tokens up to and including the first EOS.
It does not depend on max_batch, poll_every, when the request arrived, its slot or the other requests, because

  - admission is generate()'s prefill of the prompt (the ViT, then the prompt through every layer) written straight into the
    request's pages (moe_lm.AriaMoELMForCausalLM.prefill_paged), and its first token comes from its own sampling parameters
    at RNG offset 0.  Several requests' prompts are packed into one prefill launch, and a long prompt is split into chunks
    that end at multiples of 256 of its position; attention keeps every packed segment to its own pages
    (ops.attention_prefill_paged_varlen: each segment exactly the one-request kernel), a later chunk reads the earlier ones
    as a page-aligned prefix, and the rest of a layer computes each row on its own;
  - a decode step reads every row's keys from its own pages with the arithmetic of the contiguous decode kernel
    (ops.attention_decode_paged: a page is one split), samples each row with its own parameters, noise row 0 and offset =
    tokens emitted (ops.sample_tokens_slots), and the other kernels of the step compute each row on its own.

Memory is a pool of 256-token pages (moe_lm.PagedKVCache) and a request reserves ceil((T + max_new_tokens) / 256) of them when
it is admitted, so it never waits for memory once running (no preemption).  Admission is FIFO.  Slots stay dense: when a
request retires, the last active slot moves into its place.  A decode step over n active slots replays the graph captured
for the smallest power of two >= n (and the smallest power of two of table columns that covers their pages); the rows past
n are idle: finished, one key on the reserved null page 0, and no write position, so they never write into a request's pages.
The host looks at the finished flags every poll_every steps.

Prefix caching: the full 256-token pages of a prompt that a prefill wrote are kept, keyed by a hash chain over the prompt's
ids and images (page_keys), until their page is needed for something else.  A request whose prompt starts with keyed pages
(the same image, system prompt or earlier turn) holds them instead of computing them: its prefill starts at the first page
that is not cached (AriaMoELMModel.prefill_paged reads the earlier keys from the pages) and the ViT runs only on the images
that have tokens from there on.  The hit stops before the prompt's last token, which is always prefilled for the first
token's logits.  A page's keys and values do not depend on what follows it in the prompt, and the paged-prefix prefill
attends to 256-key-aligned pages with the tile order of a prefill of the whole prompt, so a hit changes no result bit.
Pages written by decode steps are never keyed: their keys and values come from the decode arithmetic, not the prefill's.

Batched and chunked admission: each step() prefills at most max_prefill_tokens prompt tokens past the cached prefixes (None:
no limit), so a long prompt delays the running requests' decode by a bounded prefill, and short prompts share one pass over
the expert weights.  It first continues the partly prefilled request, if any, then admits FIFO as before and packs the
admitted requests' chunks into one launch.  A chunk that does not fit what is left of the budget ends at the last multiple
of 256 of its absolute position the budget reaches (never a piece under 256 tokens but a prompt's last one), and admission
stops there, so at most one request is partly prefilled.  It holds its slot and pages, its slot stays idle on the null page,
no poll retires it, and its first token is sampled after its last chunk.  Pages are keyed as their chunk is staged; a head
whose hit would read a page of a launch not yet run waits for that launch, so the hits are those of one-at-a-time admission.

FP8 KV pages (kv_cache_dtype="fp8"): the pages hold e4m3 keys and values with one fp32 scale per (page, head, row), quantized
as generate()'s fp8 KV cache quantizes them, so the same pool holds about twice the tokens.  Every query attends to every key as
bf16(code * scale), the keys of its own prefill chunk included: a prefill stores its rows into the pages first and attends to
their dequantized values, and reads a cached prefix, or its prompt's earlier chunks, as the same values.  A result therefore
does not depend on chunking or cache hits either.  It equals generate(kv_cache_dtype="fp8") with that one rule applied to its
prefill; decode steps use the contiguous fp8 decode arithmetic (ops.attention_decode_paged: a page is one split).

The scheduler (Scheduler, PageAllocator) and the page keys are plain host code with no device calls.  GPU only; no expert
parallelism.  Fp8 or bf16 expert and dense weights are fine (they live inside the layers).
"""
from __future__ import annotations

import collections
import hashlib
import time
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch

from . import ops, stopping
from .moe_lm import sample_and_advance, start_rows
from .ops import MAX_LOGPROBS

PAGE = 256
MAX_BATCH = 1024   # the slot advance runs one thread per slot in one CTA
DEFAULT_PREFILL_TOKENS = 8192


def _pages_for(tokens: int) -> int:
    return -(-tokens // PAGE)


def _pow2_at_least(n: int, cap: int) -> int:
    p = 1
    while p < n:
        p *= 2
    return min(p, cap)


def _hash(*parts) -> bytes:
    """128 bits of SHA-256 over the parts (bytes or contiguous buffers; SHA-256 has CPU instructions on current hosts and ran
    twice as fast as BLAKE2b on an image)."""
    h = hashlib.sha256()
    for p in parts:
        h.update(p)
    return h.digest()[:16]


def _pixel_row_digest(pixels: torch.Tensor, mask: Optional[torch.Tensor]) -> bytes:
    """128-bit digest of one pixel row: its bf16 bytes (what the ViT reads), its shape and its pixel_mask row."""
    x = pixels.detach().to("cpu", torch.bfloat16).contiguous()
    m = b"-" if mask is None else mask.detach().to("cpu", torch.bool).contiguous().numpy().tobytes()
    return _hash(repr(tuple(x.shape)).encode(), x.view(torch.int16).numpy(), m)


def page_keys(ids: torch.Tensor, pixel_values: Optional[torch.Tensor] = None, pixel_mask: Optional[torch.Tensor] = None,
              image_token: Optional[int] = None) -> List[bytes]:
    """Keys of the full 256-token pages of a prompt (host int64 ids [T]): page i (256 (i + 1) <= T) has key
    H(key of page i - 1 | its ids | the digests of the pixel rows whose image tokens fall in it), so two prompts share page i's key
    only if they agree on every token and image up to its end.  Pixel row r owns the image tokens r n .. r n + n - 1 in order,
    n = image tokens / pixel rows; a prompt whose image-token count is not a positive multiple of its pixel rows gets no keys
    (its admission fails as forward() would)."""
    n_full = ids.numel() // PAGE
    if n_full == 0:
        return []
    ids_np = ids.numpy()
    rows_in_page: List[List[int]] = [[] for _ in range(n_full)]
    digest: Dict[int, bytes] = {}
    if pixel_values is not None:
        pos = (ids == image_token).nonzero().flatten().tolist()
        R = pixel_values.shape[0]
        if not pos or R == 0 or len(pos) % R:
            return []
        n = len(pos) // R
        for k, t in enumerate(pos):
            i = t // PAGE
            if i < n_full and (not rows_in_page[i] or rows_in_page[i][-1] != k // n):
                rows_in_page[i].append(k // n)
        needed = sorted({r for rows in rows_in_page for r in rows})
        digest = {r: _pixel_row_digest(pixel_values[r], None if pixel_mask is None else pixel_mask[r]) for r in needed}
    keys, prev = [], b""
    for i in range(n_full):
        prev = _hash(prev, ids_np[i * PAGE:(i + 1) * PAGE].tobytes(), *(digest[r] for r in rows_in_page[i]))
        keys.append(prev)
    return keys


class PageAllocator:
    """The pool's pages 1 .. n_pages - 1 with reference counts and a cache of keyed pages; page 0 is the null page idle slots
    point at, never handed out.

    A page is held by every live request that lists it (hold / alloc add one holder, free removes one).  A page no request
    holds is free: uncached, or cached (it has a key) and idle, kept in the order it was released.  n_free counts both.  alloc
    hands out uncached free pages first (the lowest first), then idle cached pages, least recently released first, dropping
    their keys (an eviction, counted in n_evicted).  A held page is never handed out."""

    def __init__(self, n_pages: int):
        if n_pages < 2:
            raise ValueError(f"a page pool needs the null page and at least one more, got {n_pages} pages")
        self.n_pages = n_pages
        self._free = list(range(n_pages - 1, 0, -1))   # uncached free pages; pop() hands out the lowest page first
        self._refs = [0] * n_pages
        self._idle: "collections.OrderedDict[int, None]" = collections.OrderedDict()   # cached, unheld; oldest release first
        self._page_of: Dict[bytes, int] = {}
        self._key_of: Dict[int, bytes] = {}
        self.n_evicted = 0

    @property
    def n_free(self) -> int:
        return len(self._free) + len(self._idle)

    @property
    def n_cached(self) -> int:
        return len(self._key_of)

    def refs(self, page: int) -> int:
        return self._refs[page]

    def alloc(self, n: int) -> List[int]:
        if n > self.n_free:
            raise RuntimeError(f"page pool: {n} pages asked, {self.n_free} free")
        out = []
        for _ in range(n):
            if self._free:
                p = self._free.pop()
            else:
                p, _ = self._idle.popitem(last=False)
                del self._page_of[self._key_of.pop(p)]
                self.n_evicted += 1
            self._refs[p] = 1
            out.append(p)
        return out

    def free(self, pages: List[int]) -> None:
        """Remove one holder from each page, the last page first: a prompt's later pages become least recently released, so
        they are evicted before its earlier ones."""
        for p in reversed(pages):
            if self._refs[p] < 1:
                raise RuntimeError(f"page pool: page {p} freed but not held")
            self._refs[p] -= 1
            if self._refs[p] == 0:
                if p in self._key_of:
                    self._idle[p] = None
                else:
                    self._free.append(p)

    def lookup(self, keys: List[bytes]) -> List[int]:
        """The cached pages of the longest run of keys[0], keys[1], ... that are all cached."""
        out = []
        for k in keys:
            p = self._page_of.get(k)
            if p is None:
                break
            out.append(p)
        return out

    def hold(self, pages: List[int]) -> None:
        """Add one holder to each of these cached pages (a hit)."""
        for p in pages:
            if self._refs[p] == 0:
                del self._idle[p]
            self._refs[p] += 1

    def register(self, page: int, key: bytes) -> None:
        """Key a held page, unless the key or the page is keyed already."""
        if key in self._page_of or page in self._key_of:
            return
        assert self._refs[page] > 0, "only a held page's contents are known"
        self._page_of[key] = page
        self._key_of[page] = key

    def unregister(self, pages) -> None:
        """Drop the keys of these pages: their prefill failed, so what they hold is not known."""
        for p in pages:
            key = self._key_of.pop(p, None)
            if key is not None:
                del self._page_of[key]


@dataclass
class Logprobs:
    """A finished request's log-probabilities (Engine.logprobs[rid]), host tensors under the model's raw distribution
    (ops.token_logprobs), None where not asked: token_logprobs [n_gen] fp32, top_ids [n_gen, k] int64 and top_logprobs [n_gen, k]
    fp32 for its generated tokens (k = logprobs); prompt_logprobs [T - 1], prompt_top_ids and prompt_top_logprobs [T - 1, k] for
    prompt positions 1 .. T - 1 (k = prompt_logprobs)."""
    token_logprobs: Optional[torch.Tensor] = None
    top_ids: Optional[torch.Tensor] = None
    top_logprobs: Optional[torch.Tensor] = None
    prompt_logprobs: Optional[torch.Tensor] = None
    prompt_top_ids: Optional[torch.Tensor] = None
    prompt_top_logprobs: Optional[torch.Tensor] = None


def ring_entries(drained: int, n_out: int, ring: int) -> List[int]:
    """Ring indices of a slot's generated tokens [drained, n_out), token i at i mod ring.  Between two polls a slot emits at
    most ring = poll_every + 1 tokens (its first token from the admission prefill, then one per replay of the poll_every
    replays), so the ring never overwrites an entry the host has not copied; a count past that is an engine bug and raises."""
    n = n_out - drained
    if not 0 <= n <= ring:
        raise RuntimeError(f"logprob ring: {n} tokens since the last poll, the ring holds {ring}")
    return [(drained + i) % ring for i in range(n)]


def _check_logprobs_arg(name: str, k) -> None:
    if k is not None and (not isinstance(k, int) or isinstance(k, bool) or not 0 <= k <= MAX_LOGPROBS):
        raise ValueError(f"{name} must be None or an int in [0, {MAX_LOGPROBS}], got {k!r}")


@dataclass
class Request:
    rid: int
    input_ids: torch.Tensor            # host int64 [T]
    max_new_tokens: int
    sampling: tuple                    # (temperature, top_k, top_p, seed); temperature 0 = greedy
    pixel_values: Optional[torch.Tensor] = None
    pixel_mask: Optional[torch.Tensor] = None
    pages: List[int] = field(default_factory=list)
    keys: List[bytes] = field(default_factory=list)    # page_keys of the prompt's full pages
    prefix_len: int = 0                                 # prompt tokens found in cached pages at admission (a multiple of 256)
    chunk: tuple = (0, 0)                               # prompt positions [start, end) of its newest planned prefill chunk
    feats: Optional[torch.Tensor] = None                # image features of pixel rows [feat_row, vit_rows) not merged yet
    feat_row: int = 0
    vit_rows: int = 0                                   # pixel rows the ViT has run on (rows inside the hit count as run)
    logprobs: Optional[int] = None                      # top-n of the generated tokens' logprobs (None: none)
    prompt_logprobs: Optional[int] = None               # top-n of the prompt tokens' logprobs (None: none; no prefix-cache hit)
    lp_drained: int = 0                                 # generated tokens whose logprobs the host has copied out of the ring
    lp_parts: list = field(default_factory=list)        # host (logprob [m], ids [m, k], logprobs [m, k]) pieces, in order
    processors: Optional[tuple] = None                  # (repetition_penalty, min_p, min_new_tokens), None when all are off
    stop_strings: Optional[tuple] = None                # the request's stop strings (None: none)
    stop_token_ids: tuple = ()                          # its own ids that finish it like EOS
    plp_parts: list = field(default_factory=list)       # device pieces of the prompt logprobs, in order

    @property
    def n_pages(self) -> int:
        return _pages_for(self.input_ids.numel() + self.max_new_tokens)


class Scheduler:
    """FIFO admission without overcommit, dense slots, no preemption.  slots[s] is the request in slot s (s < n_active).

    admit() admits the queue's head while a slot is free and its pages are free, reserving them; retire(s) frees the pages of
    slot s and moves the last active slot into s, returning that move (src, dst) or None when s was the last slot.
    Prefix caching: admission first follows the head's page keys through the cache, at most floor((T - 1) / 256) pages (the
    prompt's last token is always prefilled); the hit pages come first in req.pages and req.prefix_len = 256 x hits.  The
    head is admitted when a slot is free and its other pages fit the free pages that are not among its hits.  register(req),
    after a successful admission, keys its full prompt pages that are not cached yet, up to the end of its planned prefill.
    Chunked admission: an admitted request's prompt past its hit is planned as one chunk, req.chunk = (prefix_len, T); plan()
    cuts it to a step's budget of prompt tokens at a multiple of 256 of its absolute position, so the next chunk's prefix is
    page-aligned, and the request stays `partial` until a chunk ends at T.  Admission is FIFO and stops at a partial request,
    so at most one is partly prefilled; it holds its slot and pages meanwhile.  Pages keyed from chunks that are staged but not
    launched yet are in `unlaunched`: a head that would hit one must wait for that launch (head_waits)."""

    def __init__(self, max_batch: int, n_pages: int):
        self.max_batch = max_batch
        self.pages = PageAllocator(n_pages)
        self.queue: collections.deque = collections.deque()
        self.slots: List[Request] = []
        self.partial: Optional[Request] = None
        self.unlaunched: set = set()

    @property
    def n_active(self) -> int:
        return len(self.slots)

    def submit(self, req: Request) -> None:
        if req.n_pages > self.pages.n_pages - 1:
            raise ValueError(f"request {req.rid} needs {req.n_pages} pages; the pool has {self.pages.n_pages - 1}")
        self.queue.append(req)

    def admit_one(self) -> Optional[tuple]:
        """-> (slot, request) for the queue's head, its pages reserved, when a slot and its pages are free; else None."""
        if not (self.queue and len(self.slots) < self.max_batch):
            return None
        req = self.queue[0]
        hits = self._head_hits()
        idle_hits = sum(1 for p in hits if self.pages.refs(p) == 0)
        if req.n_pages - len(hits) > self.pages.n_free - idle_hits:
            return None
        self.queue.popleft()
        self.pages.hold(hits)                     # before alloc, which may evict idle cached pages
        req.pages = hits + self.pages.alloc(req.n_pages - len(hits))
        req.prefix_len = PAGE * len(hits)
        req.chunk = (req.prefix_len, req.input_ids.numel())
        self.slots.append(req)
        return len(self.slots) - 1, req

    def _head_hits(self) -> List[int]:
        """The cached pages the queue's head would hold; none for a request that wants its prompt logprobs, whose every prompt
        row must be computed (its pages are still keyed for others)."""
        req = self.queue[0]
        if req.prompt_logprobs is not None:
            return []
        return self.pages.lookup(req.keys[:(req.input_ids.numel() - 1) // PAGE])

    def register(self, req: Request) -> None:
        """Key req's full prompt pages that are not cached yet and lie before the end of its planned prefill (their prefill is
        staged or in flight on the admission stream, so a later launch on that stream reads them finished).  The pages of its
        newest chunk join `unlaunched`."""
        start, end = req.chunk
        for i, (page, key) in enumerate(zip(req.pages[:end // PAGE], req.keys)):
            self.pages.register(page, key)
            if i >= start // PAGE:
                self.unlaunched.add(page)

    @staticmethod
    def chunk_end(T: int, start: int, budget: Optional[int]) -> int:
        """End of the chunk of a T-token prompt that starts at `start` (a multiple of 256) within `budget` prompt tokens (None:
        no limit): T when the rest fits, else the last multiple of 256 the budget reaches; `start` when not one page fits."""
        if budget is None or T - start <= budget:
            return T
        return max(start, (start + budget) // PAGE * PAGE)

    def head_fits(self, budget: Optional[int]) -> bool:
        """Whether the queue's head, admitted now, would get a chunk within `budget`."""
        req = self.queue[0]
        start = PAGE * len(self._head_hits())
        return self.chunk_end(req.input_ids.numel(), start, budget) > start

    def head_waits(self) -> bool:
        """Whether the queue's head would hit a page whose prefill is staged but not launched yet: launch it first."""
        return bool(self.queue) and any(p in self.unlaunched for p in self._head_hits())

    def plan(self, req: Request, start: int, budget: Optional[int]) -> int:
        """Plan req's next chunk from prompt position `start` within `budget` -> its token count; req becomes (or stays)
        `partial` unless the chunk reaches the end of its prompt."""
        T = req.input_ids.numel()
        end = self.chunk_end(T, start, budget)
        req.chunk = (start, end)
        self.partial = req if end < T else None
        return end - start

    def admit(self) -> List[tuple]:
        """-> [(slot, request)] admitted, in FIFO order, their pages reserved."""
        out = []
        while (a := self.admit_one()) is not None:
            out.append(a)
        return out

    def retire(self, s: int) -> Optional[tuple]:
        req = self.slots[s]
        if req is self.partial:
            self.partial = None
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
    kv_cache_dtype: "bf16" (default) or "fp8" KV pages (see the module docstring); max_kv_tokens counts tokens either way.
    Memory: the page pools (2 x layers x heads x 128 bf16 values per token of max_kv_tokens, plus the null page; with fp8 pages
    2 x layers x heads x (128 one-byte codes + one 4-byte scale) per token, 132 bytes where bf16 takes 256), and one int32
    output row per slot as long as the pool, since a request may spend the whole pool on its budget: 4 x max_batch x
    256 ceil(max_kv_tokens / 256) bytes (32 MiB at the defaults, 4 GiB at 1024 slots and a 2^20-token pool).  An fp8 prefill
    whose segments have a cached prefix also holds, while it runs, a bf16 scratch copy of the launch's distinct prefix pages:
    2 x heads x 256 x 128 x 2 bytes per page (2.6 MB at 20 heads), shared by the layers.  Logits processors: a token-presence
    bitmap of ceil(V / 32) int32 words per slot, 12.5 KB at V = 100,352 (0.8 MB at 64 slots, 12.3 MiB at 1024), and 12 bytes
    of parameters.
    `stats`: graphs captured, decode steps replayed, slot-steps of active requests (mean occupancy = active_slot_steps /
    (steps * max_batch); a partly prefilled request is not counted), host seconds spent waiting in polls; prefix caching: prompt tokens admitted, those found in cached
    pages (prefix_hit_tokens), pixel rows the ViT ran on and skipped, cached pages evicted; admission: packed prefills run
    (prefill_launches) and the segments among them that did not end a prompt (prefill_chunks).
    max_prefill_tokens: the most prompt tokens one step() prefills (a multiple of 256; None = no limit; cached prefix tokens do
    not count), so that a long admission delays the running requests' decode steps by a bounded prefill.
    `times[rid]`: host clock (time.perf_counter) when its first token and its last token were known done (first poll after
    its prompt was prefilled, poll that saw it finish).
    Log-probabilities: `logprobs[rid]`, a Logprobs for each finished request that asked for logprobs or prompt_logprobs.  The
    decode step writes each asking slot's entries into per-slot rings of poll_every + 1 entries (SlotDecodeState.lp_ring_*),
    copied to the host at each poll, so the device memory does not grow with the pool (4 x 41 x max_batch x (poll_every + 1)
    bytes).  A step with no asking slot replays a graph without the logprob kernel.  Prompt logprobs are computed from the
    prefill's final hidden states in chunks of at most 1024 rows (a logits scratch of 2 x 1024 x V bytes).
    tokenizer: the tokenizer whose cleaned vocabulary spells the tokens for add_request(stop_strings=...) (its table is built
    here, stopping.vocab_table; None: no request may ask for stop strings).  Stops: 9.4 KB of per-slot state (a stop set of
    16 x 512 bytes, eight stop ids, a 128-id prompt tail); a step with no stopping slot replays a graph without the check."""

    max_prefill_tokens: Optional[int] = DEFAULT_PREFILL_TOKENS
    tokenizer = None

    def __init__(self, model, max_batch: int = 64, max_kv_tokens: int = 131072, eos_token_id=None, pad_token_id=None,
                 poll_every: int = 8, max_prefill_tokens: Optional[int] = DEFAULT_PREFILL_TOKENS, kv_cache_dtype: str = "bf16",
                 tokenizer=None):
        from .moe_lm import KV_CACHE_DTYPES, PagedKVCache, SlotDecodeState
        if not isinstance(kv_cache_dtype, str) or kv_cache_dtype not in KV_CACHE_DTYPES:
            raise ValueError(f"kv_cache_dtype must be 'bf16' or 'fp8', got {kv_cache_dtype!r}")
        if max_prefill_tokens is not None and (not isinstance(max_prefill_tokens, int) or max_prefill_tokens < PAGE
                                               or max_prefill_tokens % PAGE):
            raise ValueError(f"max_prefill_tokens must be None or a positive multiple of {PAGE}, got {max_prefill_tokens!r}")
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
        self.max_batch, self.poll_every, self.max_prefill_tokens = max_batch, poll_every, max_prefill_tokens
        self.eos, self.pad = eos, pad
        self.tokenizer = tokenizer
        # without a tokenizer only stop ids can stop a request, and the check reads a one-id table no slot's strings use
        self.stop_vocab = (stopping.StopVocab({0: ""}) if tokenizer is None else stopping.vocab_table(tokenizer)).device(dev)
        lm = model.language_model
        c = lm.config
        self.max_pages = _pages_for(max_kv_tokens)
        n_pages = self.max_pages + 1
        self.sched = Scheduler(max_batch, n_pages)
        self.kv_cache_dtype = kv_cache_dtype
        self.cache = PagedKVCache(c.num_hidden_layers, n_pages, c.num_attention_heads, c.head_dim, max_batch, self.max_pages, dev,
                                  kv_cache_dtype)
        self.lp_ring = poll_every + 1
        self.state = SlotDecodeState(max_batch, c.num_attention_heads, self.max_pages * PAGE, dev, self.lp_ring, c.vocab_size)
        self._idle(0, max_batch)
        self.rope = lm.model.rope_tables(self.cache.n_positions, dev)   # held here: the graphs read these tables
        self._graphs: Dict[tuple, torch.cuda.CUDAGraph] = {}
        self._pool = torch.cuda.graph_pool_handle()
        self._fin_host = torch.ones(max_batch, dtype=torch.uint8).pin_memory()
        self._nout_host = torch.zeros(max_batch, dtype=torch.int32).pin_memory()
        st = self.state
        self._lp_host = [torch.empty_like(t, device="cpu").pin_memory() for t in (st.lp_ring_lp, st.lp_ring_ids, st.lp_ring_top)]
        self._event = torch.cuda.Event()
        self._next_rid = 0
        self._undelivered: Dict[int, torch.Tensor] = {}
        self._first_seen = set()
        self.stats = {"graphs_captured": 0, "steps": 0, "active_slot_steps": 0, "poll_host_s": 0.0, "polls": 0,
                      "prompt_tokens": 0, "prefix_hit_tokens": 0, "vit_rows_run": 0, "vit_rows_skipped": 0, "pages_evicted": 0,
                      "prefill_launches": 0, "prefill_chunks": 0}
        self.times: Dict[int, list] = {}
        self.logprobs: Dict[int, Logprobs] = {}

    # ------------------------------------------------------------------------------------------------ public API
    def add_request(self, input_ids, pixel_values=None, pixel_mask=None, max_new_tokens: int = 16, do_sample: bool = False,
                    temperature: float = 1.0, top_k: int = 50, top_p: float = 1.0, seed: int = 0, logprobs: Optional[int] = None,
                    prompt_logprobs: Optional[int] = None, repetition_penalty: float = 1.0, min_p: float = 0.0,
                    min_new_tokens: int = 0, stop_strings=None, stop_token_ids=None) -> int:
        """Queue one request (input_ids [T] or [1, T]; pixel inputs as generate()'s for that one row) -> its id.  Arguments are
        checked as generate() checks them, and a request that needs more pages than the pool has is refused, here, before
        any device work.  The prompt's page keys (page_keys) are computed here, on the host.
        logprobs / prompt_logprobs (None, or an int k in [0, 20]): the logprob of each generated / prompt token under the model's
        raw distribution and its k most likely tokens, in self.logprobs[rid] once it finishes (Logprobs); the generated ones are
        generate(output_logprobs=k)'s bit for bit.  A request with prompt_logprobs takes no prefix-cache hit.
        repetition_penalty / min_p / min_new_tokens: generate()'s logits processors; the request's tokens are batch-1 generate()'s
        with the same arguments bit for bit.  A decode step runs the processed sampler only when some active slot asks for one.
        stop_strings (generate()'s, with the engine's tokenizer) and stop_token_ids (an id or a list of ids that finish this
        request like an EOS; with the engine's EOS ids at most 8): the result is batch-1 generate(ids, ..., stop_strings=...,
        tokenizer=tokenizer, eos_token_id=eos + stop_token_ids, pad_token_id=pad)[0] bit for bit.  stop_token_ids is a stopping
        criterion only, so it is not combined with min_new_tokens > 0 (which masks EOS ids).  A decode step runs the stop check
        only when some active slot has stops."""
        if not isinstance(input_ids, torch.Tensor) or input_ids.dim() not in (1, 2):
            raise ValueError("input_ids must be a tensor [T] or [1, T]")
        ids = input_ids.reshape(1, -1) if input_ids.dim() == 1 else input_ids
        if ids.shape[0] != 1:
            raise ValueError(f"add_request takes one prompt, got input_ids {tuple(input_ids.shape)}")
        self.model._check_generate_args(ids, max_new_tokens, None, do_sample, temperature, top_k, top_p, list(self.eos),
                                        self.pad, seed, self.poll_every)
        from .modeling_aria import AriaForConditionalGeneration
        processors = AriaForConditionalGeneration._check_logits_processors(repetition_penalty, min_p, min_new_tokens, None, "cuda")
        _check_logprobs_arg("logprobs", logprobs)
        _check_logprobs_arg("prompt_logprobs", prompt_logprobs)
        stops, stop_ids = self._check_stops(stop_strings, stop_token_ids, min_new_tokens)
        sampling = (float(temperature), int(top_k), float(top_p), int(seed)) if do_sample else (0.0, 0, 1.0, 0)
        req = Request(self._next_rid, ids[0].to("cpu", torch.int64), max_new_tokens, sampling, pixel_values, pixel_mask,
                      logprobs=logprobs, prompt_logprobs=prompt_logprobs, processors=processors, stop_strings=stops,
                      stop_token_ids=stop_ids)
        image_token = None if pixel_values is None else self.model.config.image_token_index
        req.keys = page_keys(req.input_ids, pixel_values, pixel_mask, image_token)
        self.sched.submit(req)
        self._next_rid += 1
        return req.rid

    def _check_stops(self, stop_strings, stop_token_ids, min_new_tokens):
        """add_request's checks of its stops, after the logprob checks, in this order: the strings and the engine's tokenizer
        (stopping.check_stop_strings), then stop_token_ids: its type, then more than 8 ids with the engine's EOS ids
        (ValueError), then min_new_tokens > 0 (NotImplementedError).  -> (strings or None, ids tuple)."""
        stops = stopping.check_stop_strings(stop_strings, self.tokenizer)
        if stop_token_ids is None:
            return stops, ()
        ids = (stop_token_ids,) if isinstance(stop_token_ids, int) else stop_token_ids
        if (not isinstance(ids, (list, tuple)) or not ids
                or not all(isinstance(e, int) and not isinstance(e, bool) for e in ids)):
            raise ValueError(f"stop_token_ids must be an int or a non-empty list of ints, got {stop_token_ids!r}")
        if len(self.eos) + len(ids) > stopping.MAX_IDS:
            raise ValueError(f"stop_token_ids: the engine's {len(self.eos)} EOS ids and the request's {len(ids)} stop ids are "
                             f"more than {stopping.MAX_IDS}")
        if min_new_tokens > 0:
            raise NotImplementedError("stop_token_ids with min_new_tokens > 0 is not supported")
        return stops, tuple(ids)

    @property
    def n_active(self) -> int:
        return self.sched.n_active

    @property
    def n_waiting(self) -> int:
        return len(self.sched.queue)

    def step(self) -> Dict[int, torch.Tensor]:
        """Replay the decode step poll_every times over the active slots, poll, retire the finished requests (neither when the
        only active request is the partly prefilled one), then prefill up
        to max_prefill_tokens prompt tokens -> {rid: result [T + generated] int64 on the model's device} of the requests that
        finished.  The prefill first continues the partly prefilled request, if any, then admits FIFO what fits (a slot and all
        its pages), and packs their chunks into as few packed prefills as it can (a head that would hit a page of a prefill
        not launched yet waits for that launch).  A request whose admission raises (e.g. pixel inputs that do not match its
        image tokens) is dropped, its slot and pages freed, after the requests packed ahead of it are prefilled, and the error
        reaches the caller; a device error in a packed prefill drops every request of that launch and unkeys the pages it was to
        write.  The requests behind stay queued, and the results this call had retired come with the next call."""
        done, self._undelivered = self._undelivered, {}
        decoding = self.sched.n_active - (self.sched.partial is not None)    # a partly prefilled request's slot is idle
        if decoding:
            n, width = _pow2_at_least(self.sched.n_active, self.max_batch), _pow2_at_least(self.sched.width(), self.max_pages)
            if self._any_stops():
                g = self._graph(n, width, self._any_logprobs(), self._any_processors(), True)
            elif self._any_processors():
                g = self._graph(n, width, self._any_logprobs(), True)
            else:
                g = self._graph(n, width, True) if self._any_logprobs() else self._graph(n, width)
            for _ in range(self.poll_every):
                g.replay()
            self.stats["steps"] += self.poll_every
            self.stats["active_slot_steps"] += self.poll_every * decoding
            done.update(self._poll_and_retire())
        sched, budget = self.sched, self.max_prefill_tokens
        self._staged = []
        try:
            if (req := sched.partial) is not None:
                n = sched.plan(req, req.chunk[1], budget)
                budget = None if budget is None else budget - n
                self._staged.append(req)
                sched.register(req)
            while sched.partial is None and sched.queue and (budget is None or budget > 0):
                if sched.head_waits():
                    self._launch()
                if not sched.head_fits(budget):
                    break
                a = sched.admit_one()
                if a is None:
                    break
                s, req = a
                n = sched.plan(req, req.prefix_len, budget)
                try:
                    self._admit(s, req)
                except BaseException:
                    self._launch()                             # the requests packed ahead of it
                    self._drop(sched.slots.index(req))
                    raise
                budget = None if budget is None else budget - n
                sched.register(req)
            self._launch()
        except BaseException:
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
        st.lp_n[lo:hi] = -1
        st.temperature[lo:hi] = 0.0
        st.rep_penalty[lo:hi] = 1.0
        st.min_p[lo:hi] = 0.0
        st.min_new[lo:hi] = 0
        st.stop_lookback[lo:hi] = 0
        st.n_stop_ids[lo:hi] = 0
        self.cache.block_table[lo:hi] = -1
        self.cache.block_table[lo:hi, 0] = 0

    def _any_logprobs(self) -> bool:
        return any(r.logprobs is not None for r in self.sched.slots)

    def _any_processors(self) -> bool:
        return any(r.processors is not None for r in self.sched.slots)

    def _any_stops(self) -> bool:
        return any(r.stop_strings is not None or r.stop_token_ids for r in self.sched.slots)

    def _step(self, n: int, lp: bool, proc: bool = False, stop: bool = False) -> None:
        lm = self.model.language_model
        st = self.state.rows(n)
        emb = ops.embedding(st.ids_in, lm.get_input_embeddings().weight)
        logits = lm.decode_step(emb, self.cache, st, self.rope)
        sample_and_advance(st, logits[:, -1], self.eos, self.pad, self.stop_vocab, lp, proc, stop)
        self._fin_host.copy_(self.state.finished, non_blocking=True)
        self._nout_host.copy_(self.state.n_out, non_blocking=True)

    def _graph(self, n: int, width: int, lp: bool = False, proc: bool = False, stop: bool = False) -> torch.cuda.CUDAGraph:
        """The captured step over slots [0, n) and table columns [0, width), with the logprob kernel when lp and the processed
        sampler when proc, captured on first use; its key is (n, width), (n, width, True) with the logprob kernel, and
        (n, width, lp, "processors") with the processed sampler, and (n, width, lp, proc, "stops") with the stop check.  The warm-up run before the capture computes the very step the
        next replay computes; the slot rows it advanced are put back afterwards."""
        key = ((n, width, lp, proc, "stops") if stop else (n, width, lp, "processors") if proc else (n, width, True) if lp
               else (n, width))
        g = self._graphs.get(key)
        if g is not None:
            return g
        self.cache.width = width
        keep = {f: getattr(self.state, f).clone() for f in self.state.SLOT_FIELDS if f != "out_tokens"}
        cur = torch.cuda.current_stream(self.dev)
        side = torch.cuda.Stream(device=self.dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            self._step(n, lp, proc, stop)
        cur.wait_stream(side)
        for f, t in keep.items():
            getattr(self.state, f).copy_(t)
        g = torch.cuda.CUDAGraph()
        with ops.graph_capture(g, pool=self._pool):
            self._step(n, lp, proc, stop)
        self._graphs[key] = g
        self.stats["graphs_captured"] += 1
        return g

    def _admit(self, s: int, req: Request) -> None:
        """Admit req into slot s: forward()'s image-token check, on the host and before any device work, then its first chunk
        (req.chunk, from its cached prefix on) joins the packed prefill being staged."""
        m = self.model
        ids, P = req.input_ids, req.prefix_len
        pv = req.pixel_values
        if pv is not None:
            # forward()'s image-token check: pixel rows x queries per row
            n_query = self._queries_per_row(pv)
            n_img = int((ids == m.config.image_token_index).sum())
            if n_img != pv.shape[0] * n_query:
                raise ValueError(f"Image features and image tokens do not match: tokens: {n_img}, features "
                                 f"{pv.shape[0] * n_query}")
            k0 = int((ids[:P] == m.config.image_token_index).sum())     # image tokens inside the cached prefix
            req.vit_rows = req.feat_row = k0 // n_query                 # pixel rows wholly inside it are never run
            self.stats["vit_rows_skipped"] += req.vit_rows
        self.stats["prompt_tokens"] += ids.numel()
        self.stats["prefix_hit_tokens"] += P
        self.stats["pages_evicted"] = self.sched.pages.n_evicted
        self._staged.append(req)

    def _queries_per_row(self, pv) -> int:
        cfg = self.model.config
        n_patch = (pv.shape[-1] // cfg.vision_config.patch_size) ** 2
        n_query = cfg.projector_patch_to_query_dict.get(n_patch)
        assert n_query is not None, f"Query number for {n_patch} patches is not provided"
        return n_query

    def _launch(self) -> None:
        """One packed prefill of the staged chunks (AriaMoELMForCausalLM.prefill_paged), each written into its request's pages;
        then, for each request whose prompt it completes, slot state and its first token (sampled at offset 0 and recorded by
        the slot advance, as generate() records its first token).  Nothing staged: no device work."""
        staged, self._staged = self._staged, []
        keyed, self.sched.unlaunched = self.sched.unlaunched, set()
        if not staged:
            return
        try:
            self._prefill(staged)
        except BaseException:
            # the pages this launch was to write were keyed when their chunks were staged; no other request holds them
            # (head_waits), and their contents are now unknown, so they must not stay in the cache as their requests retire
            self.sched.pages.unregister(keyed)
            for s in sorted((self.sched.slots.index(r) for r in staged), reverse=True):
                self._drop(s)
            raise

    def _prefill(self, staged: List[Request]) -> None:
        lm = self.model.language_model
        cu, starts, ends = [0], [], []
        for req in staged:
            start, end = req.chunk
            cu.append(cu[-1] + end - start)
            starts.append(start)
            if end == req.input_ids.numel():
                ends.append(len(starts) - 1)
        ids = torch.cat([r.input_ids[r.chunk[0]:r.chunk[1]] for r in staged])
        pos = torch.cat([torch.arange(r.chunk[0], r.chunk[1], dtype=torch.int32) for r in staged])
        width = max(len(r.pages) for r in staged)
        table = torch.full((len(staged), width), -1, dtype=torch.int32)
        for b, r in enumerate(staged):
            table[b, :len(r.pages)] = torch.tensor(r.pages, dtype=torch.int32)
        host = torch.cat([ids, pos.to(torch.int64), table.flatten().to(torch.int64)]).pin_memory()
        dev = host.to(self.dev, non_blocking=True)
        S = ids.numel()
        ids_dev, pos_dev, table_dev = dev[:S], dev[S:2 * S].to(torch.int32), dev[2 * S:].to(torch.int32).view(len(staged), width)
        seg = ops.PackedSegments(cu, starts, self.dev)
        emb = ops.embedding(ids_dev[None], lm.get_input_embeddings().weight)
        for b, req in enumerate(staged):
            if req.pixel_values is not None:
                self._merge_images(req, ids_dev[cu[b]:cu[b + 1]], emb[0, cu[b]:cu[b + 1]])
        # prompt logprobs: rows [start, min(end, T - 1)) of each asking chunk give positions start + 1 .. min(end, T - 1); the
        # last prompt row's logits are the first generated token's
        want = [(b, r, min(r.chunk[1], r.input_ids.numel() - 1) - r.chunk[0]) for b, r in enumerate(staged)
                if r.prompt_logprobs is not None]
        if want:
            rows = [i for b, _, n in want for i in range(cu[b], cu[b] + n)]
            logits, h = lm.prefill_paged(emb, self.cache, table_dev, seg, pos_dev, ends, page_table_host=table, hidden_rows=rows)
            self._prompt_logprobs(want, h)
        else:
            logits = lm.prefill_paged(emb, self.cache, table_dev, seg, pos_dev, ends, page_table_host=table)
        self.stats["prefill_launches"] += 1
        self.stats["prefill_chunks"] += len(staged) - len(ends)
        for i, b in enumerate(ends):
            req = staged[b]
            self._start_decode(self.sched.slots.index(req), req, logits[0, i:i + 1])

    PROMPT_LP_ROWS = 1024   # lm_head rows per prompt-logprob chunk: a logits scratch of 2 x 1024 x V bytes (205 MB at V = 100,352)

    def _prompt_logprobs(self, want, h) -> None:
        """Prompt logprobs of the staged chunks in `want` [(packed segment, request, rows)] from their final hidden states h
        [sum rows, d]: lm_head and ops.token_logprobs over at most PROMPT_LP_ROWS rows at a time, targets the next prompt ids.
        The results stay on the device with their request until it retires."""
        N = h.shape[0]
        if N == 0:
            return
        lm = self.model.language_model
        tgt = torch.cat([r.input_ids[r.chunk[0] + 1:r.chunk[0] + 1 + n] for _, r, n in want])
        nrow = torch.cat([torch.full((n,), r.prompt_logprobs, dtype=torch.int64) for _, r, n in want])
        host = torch.cat([tgt, nrow]).pin_memory()
        dev = host.to(self.dev, non_blocking=True)
        tgt_dev, nrow_dev = dev[:N], dev[N:].to(torch.int32)
        k = max(r.prompt_logprobs for _, r, _ in want)
        lp = torch.empty(N, dtype=torch.float32, device=self.dev)
        ids = torch.empty(N, k, dtype=torch.int32, device=self.dev)
        top = torch.empty(N, k, dtype=torch.float32, device=self.dev)
        for i in range(0, N, self.PROMPT_LP_ROWS):
            j = min(N, i + self.PROMPT_LP_ROWS)
            ops.token_logprobs(lm.lm_head(h[i:j]), tgt_dev[i:j], k, n_row=nrow_dev[i:j], out=(lp[i:j], ids[i:j], top[i:j]))
        o = 0
        for _, r, n in want:       # each request's own copy, so the launch's buffers go when this call returns
            k = r.prompt_logprobs
            r.plp_parts.append((lp[o:o + n].clone(), ids[o:o + n, :k].clone(), top[o:o + n, :k].clone()))
            o += n

    def _merge_images(self, req: Request, ids_dev, emb) -> None:
        """Image features of the chunk req.chunk into its embedding rows: the ViT and the projector run on the pixel rows whose
        first token past the cached prefix falls into this chunk, and the features of a row's tokens in later chunks are kept
        with the request (req.feats, rows [req.feat_row, req.vit_rows)).  Each pixel row's features do not depend on the rows
        that share its launch."""
        m, pv, pm = self.model, req.pixel_values, req.pixel_mask
        tok = m.config.image_token_index
        n_query = self._queries_per_row(pv)
        start, end = req.chunk
        img = req.input_ids[:end] == tok
        k0, k1 = int(img[:start].sum()), int(img.sum())       # the chunk's image tokens are k0 .. k1 - 1
        if k1 == k0:
            return
        r_end = -(-k1 // n_query)                            # pixel rows the chunk reads features of: up to r_end
        if r_end > req.vit_rows:
            r0 = req.vit_rows
            pix = pv[r0:r_end].to(self.dev, non_blocking=True).to(torch.bfloat16)
            feats, image_attn_mask = m.vision_tower(pix, None if pm is None else pm[r0:r_end])
            feats = m.multi_modal_projector(feats, image_attn_mask)
            feats = feats.reshape(-1, feats.shape[-1])
            req.feats = feats if req.feats is None else torch.cat([req.feats, feats])
            req.vit_rows = r_end
            self.stats["vit_rows_run"] += r_end - r0
        ops.merge_image_features(ids_dev, tok, req.feats[k0 - req.feat_row * n_query:], emb)
        keep = k1 // n_query                                  # rows wholly merged are dropped
        req.feats = req.feats[(keep - req.feat_row) * n_query:] if keep < req.vit_rows else None
        req.feat_row = keep

    def _start_decode(self, s: int, req: Request, logits) -> None:
        """Slot s's table row and state once req's prompt is prefilled, and its first token."""
        row = torch.full((self.max_pages,), -1, dtype=torch.int32)
        row[:len(req.pages)] = torch.tensor(req.pages, dtype=torch.int32)
        self.cache.block_table[s].copy_(row)
        T = req.input_ids.numel()
        st = self.state
        st.rope_pos[s] = T - 1
        st.write_pos[s] = T - 1
        st.kv_len[s] = T
        start_rows(st, s, req.sampling, req.max_new_tokens, req.logprobs, req.processors)
        st.noise_row[s] = 0
        if req.processors is not None:      # the prompt's ids, before the first token is sampled
            ops.presence_set(req.input_ids.to(self.dev)[None], st.presence[s:s + 1], self.model.language_model.config.vocab_size,
                             clear=True)
        stop = req.stop_strings is not None or bool(req.stop_token_ids)
        if stop:            # the prompt's tail and the request's stops, before the first token is checked
            data, lens, lookback = stopping.encode_stop_set(req.stop_strings or ())
            tail, n = stopping.prompt_tail(req.input_ids[None])
            ids = torch.zeros(stopping.MAX_IDS, dtype=torch.int64)
            ids[:len(req.stop_token_ids)] = torch.tensor(req.stop_token_ids, dtype=torch.int64)
            st.stop_bytes[s].copy_(data)
            st.stop_lens[s].copy_(lens)
            st.stop_lookback[s] = lookback
            st.stop_ids[s].copy_(ids)
            st.n_stop_ids[s] = len(req.stop_token_ids)
            st.stop_tail[s].copy_(tail[0])
            st.stop_tail_len[s] = n
        else:
            st.stop_lookback[s] = 0
            st.n_stop_ids[s] = 0
        sample_and_advance(_slot_rows(st, s), logits, self.eos, self.pad, self.stop_vocab, req.logprobs is not None,
                           req.processors is not None, stop)

    def _drop(self, s: int) -> None:
        """Retire slot s without a result: the last active slot moves into s and the slot it left becomes idle."""
        move = self.sched.retire(s)
        if move is not None:
            self._move_slot(*move)
        self._idle(self.sched.n_active, self.sched.n_active + 1)

    def _move_slot(self, src: int, dst: int) -> None:
        for f in self.state.SLOT_FIELDS:
            t = getattr(self.state, f)
            t[dst].copy_(t[src])
        self.cache.block_table[dst].copy_(self.cache.block_table[src])

    def _poll_and_retire(self) -> Dict[int, torch.Tensor]:
        t0 = time.perf_counter()
        n_act = self.sched.n_active
        lp = self._any_logprobs()
        if lp:      # the rings of the active slots, queued before the event the host waits on
            st = self.state
            for h, t in zip(self._lp_host, (st.lp_ring_lp, st.lp_ring_ids, st.lp_ring_top)):
                h[:n_act].copy_(t[:n_act], non_blocking=True)
        self._event.record(torch.cuda.current_stream(self.dev))
        self._event.synchronize()
        now = time.perf_counter()
        self.stats["poll_host_s"] += now - t0
        self.stats["polls"] += 1
        fin = self._fin_host[:self.sched.n_active].tolist()
        n_out = self._nout_host[:self.sched.n_active].tolist()
        for req in self.sched.slots:
            if req is not self.sched.partial and req.rid not in self._first_seen:
                self._first_seen.add(req.rid)
                self.times[req.rid] = [now, None]
        if lp:
            for s, req in enumerate(self.sched.slots):
                if req.logprobs is not None and req is not self.sched.partial:
                    self._drain(req, s, n_out[s])
        done = {}
        for s in range(self.sched.n_active - 1, -1, -1):   # descending: the slot moved into s is always a live one
            req = self.sched.slots[s]
            if not fin[s] or req is self.sched.partial:    # a partly prefilled request's slot is idle, not finished
                continue
            done[req.rid] = torch.cat([req.input_ids.to(self.dev), self.state.out_tokens[s, :n_out[s]].to(torch.int64)])
            self.times[req.rid][1] = now
            if req.logprobs is not None or req.prompt_logprobs is not None:
                self.logprobs[req.rid] = self._logprobs_result(req)
            self._first_seen.discard(req.rid)
            move = self.sched.retire(s)
            if move is not None:
                src, dst = move
                self._move_slot(src, dst)
                fin[dst] = fin[src]
                n_out[dst] = n_out[src]
            self._idle(self.sched.n_active, self.sched.n_active + 1)
        return done

    def _drain(self, req: Request, s: int, n_out: int) -> None:
        """Copy slot s's ring entries [req.lp_drained, n_out) out of the pinned copy of the rings into req.lp_parts."""
        idx = torch.tensor(ring_entries(req.lp_drained, n_out, self.lp_ring), dtype=torch.int64)
        if idx.numel():
            lp, ids, top = self._lp_host
            k = req.logprobs
            req.lp_parts.append((lp[s, idx].clone(), ids[s, idx, :k].to(torch.int64), top[s, idx, :k].clone()))
        req.lp_drained = n_out

    @staticmethod
    def _logprobs_result(req: Request) -> Logprobs:
        out = Logprobs()
        if req.logprobs is not None:
            k = req.logprobs
            parts = req.lp_parts or [(torch.empty(0), torch.empty(0, k, dtype=torch.int64), torch.empty(0, k))]
            out.token_logprobs, out.top_ids, out.top_logprobs = (torch.cat(t) for t in zip(*parts))
        if req.prompt_logprobs is not None:
            k = req.prompt_logprobs
            if req.plp_parts:
                lp, ids, top = (torch.cat(t).cpu() for t in zip(*req.plp_parts))
                out.prompt_logprobs, out.prompt_top_ids, out.prompt_top_logprobs = lp, ids.to(torch.int64), top
            else:   # a one-token prompt
                out.prompt_logprobs, out.prompt_top_ids, out.prompt_top_logprobs = (
                    torch.empty(0), torch.empty(0, k, dtype=torch.int64), torch.empty(0, k))
        return out


def _slot_rows(st, s: int):
    """The one-slot view [s, s + 1) of a SlotDecodeState (what the sampler and the slot advance read)."""
    v = object.__new__(type(st))
    for f in st.SLOT_FIELDS:
        setattr(v, f, getattr(st, f)[s:s + 1])
    return v
