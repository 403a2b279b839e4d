"""Stop strings: the host side of generate(stop_strings=..., tokenizer=...) and Engine.add_request(stop_strings=...).

Hugging Face's StopStringCriteria, checked on the GPU by ops.stop_check_slots.  The kernel reads two things
built here: the vocabulary table, every token's cleaned string (StopStringCriteria.clean_tokenizer_vocab: the string the
token really yields, with "Ġ" / "▁" / byte-fallback spellings resolved) as UTF-8 bytes with int32 offsets, and a stop set,
up to 16 strings of at most 128 characters in fixed-size buffers with the lookback window HF uses (the characters of the
longest string, in tokens).
"""
from __future__ import annotations

import collections
import weakref
from typing import Optional, Sequence

import numpy as np
import torch

from . import ops

MAX_STRINGS = ops.STOP_MAX_STRINGS
MAX_CHARS = ops.STOP_MAX_TOKENS       # characters per string, so also the lookback and the prompt tail
MAX_BYTES = ops.STOP_MAX_BYTES
TAIL = ops.STOP_MAX_TOKENS
MAX_IDS = ops.STOP_MAX_IDS            # the engine's EOS ids and a request's stop ids together
MISSING = b"\xff"   # an id inside the table that the vocabulary lacks: a byte no UTF-8 string holds, so it matches nothing

_CACHE: "collections.OrderedDict[tuple, StopVocab]" = collections.OrderedDict()
_CACHE_SIZE = 4
_BY_TOKENIZER: "weakref.WeakKeyDictionary" = weakref.WeakKeyDictionary()   # tokenizer -> (len(tokenizer), its StopVocab)


class StopVocab:
    """The cleaned vocabulary as the kernels read it: token i's string is data[offsets[i]:offsets[i + 1]] (UTF-8), for ids
    0 <= i < V = max id + 1.  Host tensors; device() copies them once per device."""

    def __init__(self, strings: dict):
        V = max(strings) + 1
        pieces = [strings[i].encode("utf-8", "surrogatepass") if i in strings else MISSING for i in range(V)]
        lens = np.fromiter((len(p) for p in pieces), dtype=np.int64, count=V)
        offsets = np.zeros(V + 1, dtype=np.int64)
        np.cumsum(lens, out=offsets[1:])
        if offsets[-1] >= 2 ** 31:
            raise NotImplementedError("stop strings: the cleaned vocabulary exceeds 2 GB")
        blob = b"".join(pieces) or b"\0"
        self.V = V
        self.data = torch.frombuffer(bytearray(blob), dtype=torch.uint8)
        self.offsets = torch.from_numpy(offsets.astype(np.int32))
        self._device = {}

    def device(self, dev) -> tuple:
        """(bytes, offsets) on device dev."""
        dev = torch.device(dev)
        if dev not in self._device:
            self._device[dev] = (self.data.to(dev), self.offsets.to(dev))
        return self._device[dev]


def vocab_table(tokenizer) -> StopVocab:
    """The tokenizer's StopVocab, built once per vocabulary: cached, least recently used first out, on the vocabulary's
    contents as StopStringCriteria caches its own tables (a tokenizer's equality is not to be trusted).  In front of that, a
    tokenizer seen before whose length has not changed since (so no token was added) gets its table without reading its
    vocabulary again, which at V = 100,352 takes a third of a second."""
    n = len(tokenizer)
    hit = _BY_TOKENIZER.get(tokenizer)
    if hit is not None and hit[0] == n:
        return hit[1]
    table = _content_table(tokenizer)
    _BY_TOKENIZER[tokenizer] = (n, table)
    return table


def _content_table(tokenizer) -> StopVocab:
    key = tuple(sorted(tokenizer.get_vocab().items(), key=lambda kv: kv[1]))   # get_vocab()'s order is not stable
    if key in _CACHE:
        _CACHE.move_to_end(key)
        return _CACHE[key]
    from transformers.generation.stopping_criteria import StopStringCriteria
    clean, idx = StopStringCriteria.clean_tokenizer_vocab(tokenizer)
    table = StopVocab(dict(zip(idx, clean)))
    _CACHE[key] = table
    if len(_CACHE) > _CACHE_SIZE:
        _CACHE.popitem(last=False)
    return table


def check_stop_strings(stop_strings, tokenizer) -> Optional[tuple]:
    """The argument checks of stop_strings, in this order: its type and an empty string (ValueError), a missing tokenizer
    (ValueError, Hugging Face's check), more than 16 strings or one of more than 128 characters (NotImplementedError).
    -> None for None, else the strings as a tuple."""
    if stop_strings is None:
        return None
    strings = (stop_strings,) if isinstance(stop_strings, str) else stop_strings
    if not isinstance(strings, (list, tuple)) or not strings or not all(isinstance(s, str) for s in strings):
        raise ValueError(f"stop_strings must be a str or a non-empty list of str, got {stop_strings!r}")
    if not all(strings):
        raise ValueError("stop_strings: the empty string is not a stop string")
    if tokenizer is None:
        raise ValueError("There are one or more stop strings, but no tokenizer was given. When generating with stop "
                         "strings, you must pass the model's tokenizer to the `tokenizer` argument.")
    if len(strings) > MAX_STRINGS:
        raise NotImplementedError(f"stop_strings: at most {MAX_STRINGS} strings, got {len(strings)}")
    if max(len(s) for s in strings) > MAX_CHARS:
        raise NotImplementedError(f"stop_strings: at most {MAX_CHARS} characters per string")
    return tuple(strings)


def encode_stop_set(strings: Sequence[str]):
    """A stop set as the kernels read it -> (bytes uint8 [16, 512], byte lengths int32 [16], lookback): each string's UTF-8
    bytes (unused entries have length 0) and HF's window, the characters of the longest string."""
    data = np.zeros((MAX_STRINGS, MAX_BYTES), dtype=np.uint8)
    lens = np.zeros(MAX_STRINGS, dtype=np.int32)
    for i, s in enumerate(strings):
        b = s.encode("utf-8", "surrogatepass")
        data[i, :len(b)] = np.frombuffer(b, dtype=np.uint8)
        lens[i] = len(b)
    return torch.from_numpy(data), torch.from_numpy(lens), max((len(s) for s in strings), default=0)


def prompt_tail(ids: torch.Tensor) -> tuple:
    """The last <= 128 ids of every row of ids [R, T] (pads included), right-aligned -> (host int64 [R, 128], length)."""
    R, T = ids.shape
    n = min(T, TAIL)
    tail = torch.zeros(R, TAIL, dtype=torch.int64)
    tail[:, TAIL - n:] = ids[:, T - n:].to("cpu", torch.int64)
    return tail, n
