"""Prompt-lookup decoding (generate(prompt_lookup_num_tokens=K)); prints one JSON line.

    python bench_prompt_lookup.py [--runs 3]

Model: full-width Aria (25.3B), random init with seed 0.  The GPU's name and power limit are read in the same run.  Parts:
  attention  attention_decode_multi (Q queries per row, one launch) against Q attention_decode_devlen launches, H = 20:
             B = 1 with 8K and 32K keys, B = 32 with 2K keys, Q in {1, 3, 5, 9}.  CUDA events around 20 launches, median of
             `--runs` alternated rounds.  bytes = the K/V bytes of the live keys, read once; hbm_floor = bytes / 3.35 TB/s (H100
             SXM data sheet).  identical: every query's output against its devlen launch, bit for bit.
  steps      ms per replay of the captured K-wide step (K in {2, 4, 8}), of the 1-wide step and of generate()'s own step (CUDA
             events around 20 replays), at B = 1 from the gpt-fast prompt (288 tokens) and at B = 32 from 2048-token prompts,
             with bf16 experts and with W8A8 experts.  The caches hold random rows: no prefill is timed.
             breakeven_accepted = K-wide ms / plain ms - 1: the mean number of accepted drafts per row and K-wide step at which
             lookup decoding breaks even, computed from these measured times.
  e2e        whole generate() calls against generate() without the arguments, alternating: gpt-fast's protocol (one 980 px image
             + 32 text tokens, 200 new tokens, greedy and top_k = 200 / temperature = 0.8) and B = 32 text prompts of 512 tokens
             (64 new tokens, greedy); tokens/s, K-wide steps, mean accepted drafts per K-wide step and row that drafted, and
             whether the tokens are identical.  The weights are random: acceptance here says nothing about Aria's.
  host_wait  the 1-wide step replayed with the event wait generate() does after every lookup step, against generate()'s own
             step replayed back to back: the per-step cost of a lookup call in which no row ever drafts.
"""
import argparse
import json
import time

import torch

from bench_generate import HBM_GBS, gpu_info

KV_BYTES_PER_KEY = 2 * 128 * 2        # K and V of one head, bf16
med = lambda xs: sorted(xs)[len(xs) // 2]


def _events(fn, iters=20):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / iters          # ms


def run_attention(args, dev):
    from aria_b200 import ops
    H, scale = 20, 128 ** -0.5
    res = []
    for B, T in ((1, 8192), (1, 32768), (32, 2048)):
        g = torch.Generator(device=dev).manual_seed(B + T)
        T_max = T + 256
        k = torch.randn(B, H, T_max, 128, generator=g, device=dev).bfloat16()
        v = torch.randn(B, H, T_max, 128, generator=g, device=dev).bfloat16()
        for Q in (1, 3, 5, 9):
            q = torch.randn(B, H, Q, 128, generator=g, device=dev).bfloat16()
            lens = (torch.full((B, 1), T - Q + 1, dtype=torch.int32) + torch.arange(Q, dtype=torch.int32)).reshape(-1).to(dev)
            lq = [lens.view(B, Q)[:, i].contiguous() for i in range(Q)]
            qs = [q[:, :, i] for i in range(Q)]
            multi = lambda: ops.attention_decode_multi(q, k, v, lens, scale)
            sep = lambda: [ops.attention_decode_devlen(qs[i], k, v, lq[i], scale) for i in range(Q)]
            got, want = multi(), sep()
            same = all(torch.equal(got[:, i], want[i]) for i in range(Q))
            _events(multi), _events(sep)
            tm, ts = [], []
            for _ in range(args.runs):
                tm.append(_events(multi) * 1e3)
                ts.append(_events(sep) * 1e3)
            nbytes = B * H * T * KV_BYTES_PER_KEY
            floor = nbytes / (HBM_GBS * 1e3)   # us
            res.append({"B": B, "keys": T, "Q": Q, "multi_us": round(med(tm), 2), "devlen_x_Q_us": round(med(ts), 2),
                        "speedup": round(med(ts) / med(tm), 3), "bytes_once": nbytes, "hbm_floor_us": round(floor, 2),
                        "multi_floor_fraction": round(floor / med(tm), 3), "identical": same})
        del k, v
        torch.cuda.empty_cache()
    return res


def _fill_cache(cache, gen):
    for t in cache.k + cache.v:
        t.normal_(0.0, 1.0, generator=gen)


def _steps_case(model, B, T, args, dev):
    """ms per replay of generate()'s step and of the lookup steps, over caches holding T random rows per row."""
    from aria_b200.modeling_aria import GraphedDecode, GraphedLookupDecode
    V = model.config.text_config.vocab_size
    gen = torch.Generator(device=dev).manual_seed(T + B)
    ids = torch.randint(10, V, (B, T), generator=torch.Generator().manual_seed(B))
    logits = torch.randn(B, V, generator=gen, device=dev).bfloat16()
    new, sampling = 64, (0.0, 0, 1.0, 0)
    out = {}
    model._decode_graph = None
    torch.cuda.empty_cache()
    g = GraphedDecode(model, B, -(-(T + new) // 256) * 256, new, sampling, (), 0)
    _fill_cache(g.cache, gen)
    g.start(T, None)
    g.sample_and_advance(logits)
    _events(g.graph.replay)
    out["plain_ms"] = round(med([_events(g.graph.replay) for _ in range(args.runs)]), 4)
    del g
    torch.cuda.empty_cache()
    for K in (2, 4, 8):
        lg = GraphedLookupDecode(model, B, -(-(T + new + K) // 256) * 256, new, sampling, (), 0, K, 2)
        _fill_cache(lg.cache, gen)
        lg.start(ids, None)
        lg.first(logits)
        _events(lg.graph_k.replay)
        out[f"k{K}_ms"] = round(med([_events(lg.graph_k.replay) for _ in range(args.runs)]), 4)
        if K == 2:
            _events(lg.graph_1.replay)
            out["one_wide_ms"] = round(med([_events(lg.graph_1.replay) for _ in range(args.runs)]), 4)
        out[f"k{K}_breakeven_accepted"] = round(out[f"k{K}_ms"] / out["plain_ms"] - 1, 3)
        del lg
        torch.cuda.empty_cache()
    return out


def run_steps(model, args, dev):
    return {"b1_T288": _steps_case(model, 1, 288, args, dev), "b32_T2048": _steps_case(model, 32, 2048, args, dev)}


def _wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def _e2e(model, ids, pv, new, kw, K, args):
    plain = lambda: model.generate(ids, pv, None, max_new_tokens=new, **kw)
    look = lambda: model.generate(ids, pv, None, max_new_tokens=new, prompt_lookup_num_tokens=K, **kw)
    for _ in range(args.warmup):
        plain(), look()
    tp, tl, same = [], [], True
    for _ in range(args.runs):
        t, a = _wall(plain)
        tp.append(t)
        t, b = _wall(look)
        tl.append(t)
        same &= bool(torch.equal(a, b))
    st = model.prompt_lookup_stats
    B = ids.shape[0]
    model._decode_graph = None
    return {"B": B, "T": ids.shape[1], "new_tokens": new, "K": K, "plain_tokens_per_s": round(B * new / med(tp), 1),
            "lookup_tokens_per_s": round(B * new / med(tl), 1), "speedup": round(med(tp) / med(tl), 3),
            "steps": st["steps"], "k_steps": st["k_steps"], "drafted": st["drafted"], "accepted": st["accepted"],
            "identical": same}


def run_e2e(model, cfg, args, dev):
    g = torch.Generator().manual_seed(1234)
    V = cfg["text_config"]["vocab_size"]
    pv = torch.randn(1, 3, 980, 980, generator=g).bfloat16()
    text = torch.randint(10, V, (32,), generator=g)
    ids = torch.cat([text[:16], torch.full((256,), cfg["image_token_index"]), text[16:]])[None]
    out = {"gptfast_greedy": _e2e(model, ids, pv, 200, dict(seed=0), 4, args),
           "gptfast_sampled": _e2e(model, ids, pv, 200, dict(do_sample=True, top_k=200, temperature=0.8, seed=0), 4, args)}
    ids32 = torch.randint(10, V, (32, 512), generator=g)
    out["b32_T512_greedy"] = _e2e(model, ids32, None, 64, dict(seed=0), 4, args)
    return out


def run_host_wait(model, args, dev):
    """Per-step wall time of the 1-wide lookup step with generate()'s per-step event wait against generate()'s step replayed
    back to back (batch 1, gpt-fast prompt length)."""
    from aria_b200.modeling_aria import GraphedDecode, GraphedLookupDecode
    B, T, new, n = 1, 288, 64, 200
    V = model.config.text_config.vocab_size
    gen = torch.Generator(device=dev).manual_seed(3)
    logits = torch.randn(B, V, generator=gen, device=dev).bfloat16()
    model._decode_graph = None
    g = GraphedDecode(model, B, 512, new, (0.0, 0, 1.0, 0), (), 0)
    _fill_cache(g.cache, gen)
    g.start(T, None)
    g.sample_and_advance(logits)
    lg = GraphedLookupDecode(model, B, 512, new, (0.0, 0, 1.0, 0), (), 0, 4, 2)
    _fill_cache(lg.cache, gen)
    lg.start(torch.randint(10, V, (B, T)), None)
    lg.first(logits)
    stream = torch.cuda.current_stream(dev)

    def plain():
        for _ in range(n):
            g.graph.replay()

    def waited():
        for _ in range(n):
            lg.graph_1.replay()
            lg.event.record(stream)
            lg.event.synchronize()
    plain(), waited()
    tp, tw = [], []
    for _ in range(args.runs):
        tp.append(_wall(plain)[0] / n * 1e3)
        tw.append(_wall(waited)[0] / n * 1e3)
    return {"plain_ms_per_step": round(med(tp), 4), "lookup_1wide_waited_ms_per_step": round(med(tw), 4),
            "overhead_ms_per_step": round(med(tw) - med(tp), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    from aria_b200 import configs as C
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration, init_random_
    dev = "cuda:0"
    name, power = gpu_info(0)
    out = {"bench": "prompt_lookup", "gpu": name, "power_limit_w": power,
           "hbm_floor_source": f"{HBM_GBS} GB/s, H100 SXM data sheet", "runs": args.runs,
           "note": "random-init weights: acceptance rates say nothing about Aria's; breakeven_accepted is computed from the "
                   "measured step times"}
    with torch.no_grad():
        out["attention"] = run_attention(args, dev)
        cfg = C.ARIA_25B
        model = AriaForConditionalGeneration(AriaConfig.from_dict(cfg), device=dev)
        init_random_(model, seed=0)
        out["steps_bf16"] = run_steps(model, args, dev)
        out["e2e_bf16"] = run_e2e(model, cfg, args, dev)
        out["host_wait_bf16"] = run_host_wait(model, args, dev)
        model._decode_graph = None
        model.quantize_experts_fp8("fp8")
        torch.cuda.empty_cache()
        out["steps_w8a8_experts"] = run_steps(model, args, dev)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
