"""Python statements of prompt-lookup decoding's per-row rules, the references of tests/test_prompt_lookup_host.py and
tests/test_gpu_prompt_lookup.py."""


def draft(hist, K, M, eos=(), room=None):
    """The draft of one row with history `hist` (its real tokens: prompt after the left padding, then its output), as
    transformers' PromptLookupCandidateGenerator.get_candidates finds it: for n = min(M, len - 1) down to 1, the earliest
    occurrence of the last n tokens whose continuation is not empty; the continuation (at most K tokens, not past the history)
    cut before its first EOS.  A match whose continuation starts with EOS gives no draft, without trying a smaller n.
    room: the draft is then cut to that many tokens (what the step can still emit after the row's next token)."""
    hist = list(hist)
    L = len(hist)
    out = []
    for n in range(min(M, L - 1), 0, -1):
        tail = hist[L - n:]
        hit = next((p for p in range(L - n) if hist[p:p + n] == tail), None)   # p = L - n is the tail itself: no continuation
        if hit is None:
            continue
        for t in hist[hit + n:min(hit + n + K, L)]:
            if t in eos:
                break
            out.append(t)
        break
    return out if room is None else out[:max(room, 0)]


def accept(drafts, targets, n_out, max_new, eos=()):
    """One row of a verify step: drafts d_1..d_k, targets t_0..t_k (t_i sampled at the position after d_i).  Drafts are accepted
    while d_{i+1} == t_i; the row emits t_0..t_a, stopping after its first EOS and at max_new tokens in all.
    -> (emitted tokens, finished)."""
    a = 0
    while a < len(drafts) and drafts[a] == targets[a]:
        a += 1
    out = []
    for t in targets[:a + 1]:
        if n_out + len(out) >= max_new:
            break
        out.append(t)
        if t in eos:
            return out, True
    return out, False
