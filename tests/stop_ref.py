"""Stop strings on the host: the stop-check kernel's algorithm restated in plain Python (stops), and the offline tokenizers the
tests check it with (byte_level_tokenizer, sentencepiece_tokenizer), built in-process with the `tokenizers` library."""
import random

from aria_b200 import stopping


def stops(table: "stopping.StopVocab", strings, history) -> bool:
    """Whether a row whose ids so far are `history` (prompt and generated, oldest first) stops after its last id: what
    ops.stop_check_slots computes for one row with these strings and no stop ids, byte for byte (see csrc/stop.cu)."""
    data, offsets = bytes(table.data.numpy()), table.offsets.tolist()
    W = min(max(len(s) for s in strings), stopping.TAIL)
    window = list(history)[::-1][:W]

    def tok(i):
        return data[offsets[i]:offsets[i + 1]] if 0 <= i < table.V else None

    toks = [tok(i) for i in window]
    if not toks or not toks[0]:
        return False
    T0 = toks[0]
    for s in strings:
        S = s.encode("utf-8", "surrogatepass")
        L = len(S)
        for m in range(1, len(T0) + 1):
            if m >= L:
                if T0[m - L:m] == S:
                    return True
                continue
            if T0[:m] != S[L - m:]:
                continue
            p = m
            for T in toks[1:]:
                if p >= L or T is None:
                    break
                k = min(len(T), L - p)
                if T[len(T) - k:] != S[L - p - k:L - p]:
                    break
                p += len(T)
            if p >= L:
                return True
    return False


IM_END = "<|im_end|>"


def _fill(base, extra, V, seed, alphabet):
    """base + extra tokens, then random distinct strings over `alphabet` up to V entries."""
    toks = list(dict.fromkeys(base + extra))
    seen = set(toks)
    rng = random.Random(seed)
    while len(toks) < V:
        t = "".join(rng.choice(alphabet) for _ in range(rng.randint(2, 8)))
        if t not in seen:
            seen.add(t)
            toks.append(t)
    return toks


def byte_level_tokenizer(V: int = 1000, seed: int = 0):
    """A GPT-2-style byte-level BPE tokenizer of V ids (plus the added special token <|im_end|>): the 256 byte symbols,
    multi-token spellings of "stop", "<|im_end|>", "é" and "日", "Ġ"-prefixed words, then random byte-symbol strings."""
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers
    from tokenizers.pre_tokenizers import ByteLevel
    from transformers import PreTrainedTokenizerFast
    alpha = sorted(ByteLevel.alphabet())
    e_acute, ri = "Ã©", "æĹ¥"          # "é" and "日" in byte-level spelling
    extra = ["st", "op", "sto", "stop", "Ġstop", "xstopy", "topper", "las", "pped", "to", "s", "<|", "im", "_end", "|>", "<|im",
             "_end|>", "end", "Ġthe", "Ġa", "ĠÃ©", e_acute, "caf" + e_acute, ri, ri + "æľ¬", "Ċ", "ĊĊ", "Ġ" + ri, "æĹ", "¥"]
    toks = _fill(alpha, extra, V, seed, alpha[:200] + ["Ġ"] * 20)
    tk = Tokenizer(models.BPE(vocab={t: i for i, t in enumerate(toks)}, merges=[]))
    tk.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False)
    tk.decoder = decoders.ByteLevel()
    tok = PreTrainedTokenizerFast(tokenizer_object=tk)
    tok.add_special_tokens({"additional_special_tokens": [IM_END]})
    return tok


def sentencepiece_tokenizer(V: int = 1000, seed: int = 0):
    """A Llama-style SentencePiece tokenizer of V ids: "▁" word starts, <0x00>..<0xFF> byte fallback (so "\\n" is <0x0A>),
    multi-token spellings of "stop" and "<|im_end|>", a token "<e>" that cleans to the empty string, then random strings."""
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers
    from transformers import PreTrainedTokenizerFast
    bytes_ = [f"<0x{i:02X}>" for i in range(256)]
    letters = [chr(c) for c in range(ord("a"), ord("z") + 1)] + list("<|>_.,!?") + ["é", "日", "本"]
    extra = ["▁", "▁stop", "st", "op", "stop", "▁st", "sto", "p", "<|", "im", "_end", "|>", "▁<|", "▁the", "▁a", "é", "日本",
             "caf", "café", "▁日", "<e>"]
    toks = _fill(["<unk>", "<s>", "</s>"] + bytes_ + letters, extra, V, seed, letters + ["▁"] * 6)
    tk = Tokenizer(models.BPE(vocab={t: i for i, t in enumerate(toks)}, merges=[], unk_token="<unk>", byte_fallback=True))
    tk.pre_tokenizer = pre_tokenizers.Metaspace(replacement="▁", prepend_scheme="first")
    # "<e>" cleans to the empty string
    tk.decoder = decoders.Sequence([decoders.Replace("<e>", ""), decoders.Replace("▁", " "), decoders.ByteFallback(), decoders.Fuse(),
                                    decoders.Strip(" ", 1, 0)])
    return PreTrainedTokenizerFast(tokenizer_object=tk, unk_token="<unk>", bos_token="<s>", eos_token="</s>")


def cases(tok, n_sets: int, n_rows: int, seed: int = 0, sizes=((1, 4), (1, 24), (16, 24)), extra=((1, 1), (16, 128))):
    """Adversarial stop-string cases for tokenizer tok -> [(strings, histories int64 [n_rows, H])].  The strings are pieces of
    the concatenated strings of a few tokens, cut inside the first and the last token (overhangs at both ends), and sizes
    gives (count, most characters) per set in turn, then the sets of `extra`.  The rows plant those tokens, or
    mutated copies, at the end of the history, before one or more further tokens (a match that does not touch the final
    token), or inside a longer final token; others are random ids from the planted ones, empty-cleaning tokens and ids
    outside the vocabulary.  H varies from 1 (a history shorter than the string) upwards."""
    import torch
    from transformers.generation.stopping_criteria import StopStringCriteria
    rng = random.Random(seed)
    clean, idx = StopStringCriteria.clean_tokenizer_vocab(tok)
    strings_of = dict(zip(idx, clean))
    V = max(idx) + 1
    useful = sorted(i for i, s in strings_of.items() if s)     # get_vocab()'s order is not stable
    empty = sorted(i for i, s in strings_of.items() if not s)
    hot = [i for i in useful if len(strings_of[i]) <= 6][:600]
    by_text = {}
    for i in useful:
        by_text.setdefault(strings_of[i], i)
    out = []
    specs = [sizes[k % len(sizes)] for k in range(n_sets)] + list(extra)
    for count, most in specs:
        strings, plants = [], []
        while len(strings) < count:
            ids = [rng.choice(hot) for _ in range(rng.randint(1, 5))]
            text = "".join(strings_of[i] for i in ids)
            a = rng.randint(0, min(2, len(strings_of[ids[0]]) - 1))
            b = len(text) - rng.randint(0, min(2, len(strings_of[ids[-1]]) - 1))
            s = text[a:b][:most]
            if s:
                strings.append(s)
                plants.append(ids)
        if most == 128:   # full-length strings: long concatenations of single characters the vocabulary spells
            singles = [by_text[c] for c in "abcdefghijklmnopqrstuvwxyz" if c in by_text] or hot
            plants = [[rng.choice(singles) for _ in range(128)] for _ in range(count)]
            strings = ["".join(strings_of[i] for i in p) for p in plants]
        H = rng.choice([1, 2, 3, 7, 20, 64, 140, 200])
        rows = []
        for _ in range(n_rows):
            kind = rng.random()
            p = list(rng.choice(plants))
            if kind < 0.15:
                row = [rng.choice(hot + empty + [V, V + 7]) for _ in range(H)]
            else:
                if kind < 0.3:       # a mutated token
                    p[rng.randrange(len(p))] = rng.choice(hot)
                elif kind < 0.4 and empty:   # an empty-cleaning token inside the match
                    p.insert(rng.randrange(len(p) + 1), rng.choice(empty))
                elif kind < 0.5:     # tokens after the match
                    p += [rng.choice(hot) for _ in range(rng.randint(1, 3))]
                elif kind < 0.55:    # an unknown id inside the match
                    p.insert(rng.randrange(len(p)), V + rng.randint(0, 9))
                if kind > 0.9 and len(p) > 1:   # the final token: a longer one starting with the planted one's text
                    t = strings_of[p[-1]]
                    longer = [i for i in useful if strings_of[i].startswith(t) and strings_of[i] != t]
                    if longer:
                        p[-1] = rng.choice(longer)
                row = [rng.choice(useful) for _ in range(max(0, H - len(p)))] + p
                row = row[-H:] if rng.random() < 0.8 else row
            rows.append(row)
        Hr = max(len(r) for r in rows)
        hist = torch.tensor([[rng.choice(useful)] * (Hr - len(r)) + r for r in rows], dtype=torch.int64)
        out.append((tuple(strings), hist))
    return out
