"""n sampled continuations per prompt from one shared prompt cache (generate(num_return_sequences=n)); prints one JSON line.

    python bench_shared_prefix.py [--runs 3] [--warmup 1]

Model: full-width Aria (25.3B), random init with seed 0; no checkpoint is needed to time the kernels.  The GPU's name and power
limit are read in the same run.  Parts:
  attention  the shared-prefix decode attention alone against attention_decode_devlen on the expanded cache (n copies of the
             prompt), H = 20, one prompt, every row 32 tail tokens; P = 2048 with n in {4, 16, 32, 64} and P = 6144 with n = 32.
             CUDA events around 20 launches, median of `--runs` alternated rounds.  bytes = the K/V bytes each kernel must read;
             hbm_floor = bytes / 3.35 TB/s (H100 SXM data sheet).  issue_floor (shared kernel only) = the prompt keys' warp
             instructions over every SM's 4 issue slots at the card's maximum SM clock: each 4-key step of a query's team
             issues about ISSUE_PER_STEP warp instructions (counted in the SASS of attn_decode_prefix_partial's loop with a
             prefix mask and every key live).  The kernel's time sits near the larger of the two floors.
  b32        n = 32 continuations of one 2048-token prompt (one 980 px image = 256 image tokens + 1792 text tokens), 64 new
             tokens, top_k = 200, temperature = 0.8: ms per decode step (CUDA events around the replays of the captured step)
             of the shared graph against generate()'s graph for the prompt repeated 32 times, alternating; the allocator's
             peak memory of each arm; whether both give the same tokens (they should: T is a multiple of 256).  The
             repeated arm prefills the prompt once and copies it into its 32 cache rows (repeated_decode).  With bf16
             experts and again after quantize_experts_fp8("fp8") (W8A8 experts).
  six_k      n = 32 from a 6144-token prompt (one image + 5888 text tokens) in bf16; the repeated batch's 32 x 6400-row cache
             alone (58.7 GB) does not fit beside the bf16 model, so only the shared arm runs.
  gptfast_n8 gpt-fast's protocol with n = 8: one 980 px image + 32 text tokens, 200 new tokens, top_k = 200, temperature = 0.8,
             no EOS; tokens/s = 8 * 200 / wall time of the whole generate() call (ViT and prefill included), against
             generate() on the repeated prompt, alternating.
"""
import argparse
import json
import subprocess
import time

import torch

from bench_generate import HBM_GBS, gpu_info, timed_replays

ISSUE_PER_STEP = 250
KV_BYTES_PER_KEY = 2 * 128 * 2        # K and V of one head, bf16


def max_sm_clock_mhz():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def _events(fn, iters=20):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / iters * 1e3      # us


def run_attention(args, dev, clock_mhz):
    from aria_b200 import ops
    H, tail, scale = 20, 32, 128 ** -0.5
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    res = []
    for P, n in ((2048, 4), (2048, 16), (2048, 32), (2048, 64), (6144, 32)):
        g = torch.Generator(device=dev).manual_seed(P + n)
        N_max = 256
        q = torch.randn(n, H, 128, generator=g, device=dev).bfloat16()
        pk = torch.randn(1, H, P, 128, generator=g, device=dev).bfloat16()
        pv = torch.randn(1, H, P, 128, generator=g, device=dev).bfloat16()
        tk = torch.randn(n, H, N_max, 128, generator=g, device=dev).bfloat16()
        tv = torch.randn(n, H, N_max, 128, generator=g, device=dev).bfloat16()
        plens = torch.tensor([P], dtype=torch.int32, device=dev)
        tlens = torch.full((n,), tail, dtype=torch.int32, device=dev)
        pmask = torch.zeros(1, P, dtype=torch.uint8, device=dev)
        # expanded: the prompt copied into every row, the tail right after it (P is a multiple of 256)
        ek = torch.empty(n, H, P + N_max, 128, dtype=torch.bfloat16, device=dev)
        ev = torch.empty_like(ek)
        ek[:, :, :P], ev[:, :, :P] = pk, pv
        ek[:, :, P:], ev[:, :, P:] = tk, tv
        elens = torch.full((n,), P + tail, dtype=torch.int32, device=dev)
        ekm = torch.zeros(n, P + N_max, dtype=torch.uint8, device=dev)
        shared = lambda: ops.attention_decode_shared_prefix(q, pk, pv, plens, tk, tv, tlens, n, scale, prefix_mask=pmask)
        expanded = lambda: ops.attention_decode_devlen(q, ek, ev, elens, scale, key_mask=ekm)
        same = torch.equal(shared(), expanded())
        for _ in range(3):
            shared(), expanded()
        ts, te = [], []
        for _ in range(args.runs):
            ts.append(_events(shared))
            te.append(_events(expanded))
        us_s, us_e = sorted(ts)[len(ts) // 2], sorted(te)[len(te) // 2]
        b_s = H * P * KV_BYTES_PER_KEY + n * H * tail * KV_BYTES_PER_KEY
        b_e = n * H * (P + tail) * KV_BYTES_PER_KEY
        issue_us = None
        if clock_mhz:
            issue_us = n * H * (P / 4) * ISSUE_PER_STEP / (sms * 4 * clock_mhz * 1e6) * 1e6
        res.append({"P": P, "n": n, "H": H, "tail": tail, "bit_identical": bool(same),
                    "shared_us": round(us_s, 2), "shared_bytes": b_s,
                    "shared_hbm_floor_us": round(b_s / (HBM_GBS * 1e9) * 1e6, 2),
                    "shared_issue_floor_us": None if issue_us is None else round(issue_us, 2),
                    "expanded_devlen_us": round(us_e, 2), "expanded_bytes": b_e,
                    "expanded_hbm_floor_us": round(b_e / (HBM_GBS * 1e9) * 1e6, 2),
                    "speedup": round(us_e / us_s, 3)})
        del ek, ev, pk, pv, tk, tv
        torch.cuda.empty_cache()
    return res


def _prompt(cfg, n_text, seed):
    g = torch.Generator().manual_seed(seed)
    pv = torch.randn(1, 3, 980, 980, generator=g).bfloat16()
    text = torch.randint(10, cfg["text_config"]["vocab_size"], (n_text,), generator=g)
    ids = torch.cat([text[:16], torch.full((256,), cfg["image_token_index"]), text[16:]])[None]
    return ids, pv


def _peak_gb(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return out, round(torch.cuda.max_memory_allocated() / 1e9, 2)


def repeated_decode(model, ids, pv, n, new, kw):
    """generate()'s decode on the prompt repeated n times, with the repeated batch's own graph and cache.  Its 32 identical
    prefills (65,536 tokens at T = 2048) are replaced by one prefill copied into every row, which gives the same cache rows
    (the tests check that prefill rows do not depend on the batch) without the activations of a 65,536-token forward()."""
    from aria_b200.modeling_aria import GraphedDecode
    T = ids.shape[1]
    sampling = (float(kw["temperature"]), int(kw["top_k"]), 1.0, int(kw["seed"]))
    g = GraphedDecode(model, n, -(-(T + new) // 256) * 256, new, sampling, (), 0)
    out = model.forward(ids, pv, None, max_cache_len=T, num_logits_to_keep=1)
    for dst, src in zip(g.cache.k + g.cache.v, out.past_key_values.k + out.past_key_values.v):
        dst[:, :, :T] = src[:, :, :T]
    g.start(T, None)
    g.sample_and_advance(out.logits[:, -1].expand(n, -1))     # row stride 0: every row samples the same logits
    for _ in range(new - 1):
        g.graph.replay()
    return g, g.state.out_tokens.to(torch.int64)


def run_b32(model, cfg, args, kw):
    n, new = 32, 64
    ids, pv = _prompt(cfg, 2048 - 256, seed=7)
    T = ids.shape[1]
    model._decode_graph = None
    torch.cuda.empty_cache()
    a, peak_shared = _peak_gb(lambda: model.generate(ids, pv, None, max_new_tokens=new, num_return_sequences=n, **kw))
    model._decode_graph = None
    torch.cuda.empty_cache()
    (g_rep, b), peak_rep = _peak_gb(lambda: repeated_decode(model, ids, pv, n, new, kw))
    model.generate(ids, pv, None, max_new_tokens=new, num_return_sequences=n, **kw)
    g_sh = model._decode_graph
    timed_replays(g_sh, T, new - 1)
    timed_replays(g_rep, T, new - 1)
    ms_s, ms_r = [], []
    for _ in range(args.runs):
        ms_s.append(timed_replays(g_sh, T, new - 1))
        ms_r.append(timed_replays(g_rep, T, new - 1))
    med = lambda xs: sorted(xs)[len(xs) // 2]
    del g_rep, g_sh
    model._decode_graph = None
    torch.cuda.empty_cache()
    return {"T": T, "n": n, "new_tokens": new, "tokens_identical": bool(torch.equal(a[:, T:], b)),
            "shared_ms_per_step": round(med(ms_s), 4), "repeated_ms_per_step": round(med(ms_r), 4),
            "speedup": round(med(ms_r) / med(ms_s), 3), "shared_ms_runs": [round(x, 4) for x in ms_s],
            "repeated_ms_runs": [round(x, 4) for x in ms_r], "shared_peak_gb": peak_shared, "repeated_peak_gb": peak_rep}


def run_six_k(model, cfg, args, kw):
    n, new = 32, 64
    ids, pv = _prompt(cfg, 6144 - 256, seed=8)
    T = ids.shape[1]
    model._decode_graph = None
    torch.cuda.empty_cache()
    _, peak = _peak_gb(lambda: model.generate(ids, pv, None, max_new_tokens=new, num_return_sequences=n, **kw))
    g = model._decode_graph
    timed_replays(g, T, new - 1)
    ms = sorted(timed_replays(g, T, new - 1) for _ in range(args.runs))[args.runs // 2]
    model._decode_graph = None
    torch.cuda.empty_cache()
    return {"T": T, "n": n, "new_tokens": new, "shared_ms_per_step": round(ms, 4), "shared_peak_gb": peak,
            "repeated": "not run: its bf16 cache of 32 x 6400 rows alone is 58.7 GB"}


def run_gptfast_n8(model, cfg, args, kw):
    n, new = 8, 200
    ids, pv = _prompt(cfg, 32, seed=1234)
    rep_ids, rep_pv = ids.repeat_interleave(n, 0), pv.repeat_interleave(n, 0)

    def wall(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    shared = lambda: model.generate(ids, pv, None, max_new_tokens=new, num_return_sequences=n, **kw)
    repeated = lambda: model.generate(rep_ids, rep_pv, None, max_new_tokens=new, **kw)
    for _ in range(args.warmup):
        shared(), repeated()
    ts, tr = [], []
    for _ in range(args.runs):
        ts.append(wall(shared))
        tr.append(wall(repeated))
    med = lambda xs: sorted(xs)[len(xs) // 2]
    model._decode_graph = None
    return {"n": n, "new_tokens": new, "shared_tokens_per_s": round(n * new / med(ts), 1),
            "repeated_tokens_per_s": round(n * new / med(tr), 1), "speedup": round(med(tr) / med(ts), 3),
            "shared_wall_s": [round(x, 4) for x in ts], "repeated_wall_s": [round(x, 4) for x in tr]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    from aria_b200 import configs as C
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration, init_random_
    dev = "cuda:0"
    name, power = gpu_info(0)
    clock = max_sm_clock_mhz()
    out = {"bench": "shared_prefix", "gpu": name, "power_limit_w": power, "max_sm_clock_mhz": clock,
           "hbm_floor_source": f"{HBM_GBS} GB/s, H100 SXM data sheet", "runs": args.runs}
    kw = dict(do_sample=True, top_k=200, temperature=0.8, seed=0)
    with torch.no_grad():
        out["attention"] = run_attention(args, dev, clock)
        cfg = C.ARIA_25B
        model = AriaForConditionalGeneration(AriaConfig.from_dict(cfg), device=dev)
        init_random_(model, seed=0)
        out["b32_bf16"] = run_b32(model, cfg, args, kw)
        out["six_k_bf16"] = run_six_k(model, cfg, args, kw)
        out["gptfast_n8_bf16"] = run_gptfast_n8(model, cfg, args, kw)
        model.quantize_experts_fp8("fp8")
        torch.cuda.empty_cache()
        out["b32_w8a8_experts"] = run_b32(model, cfg, args, kw)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
