"""Prefix caching in serving.Engine against the same traces with nothing to share; prints one JSON line.

    python bench_prefix_cache.py [--max-batch 64] [--max-kv-tokens 65536] [--rate 8.0] [--lm-layers 16] [--seed 0]

Model: full-width Aria with random weights (seed 0) and --lm-layers of the 28 LM layers, as bench_serving.py.  Greedy, no EOS.
Workloads (seeded):
  images_<c>crop   32 images x 8 questions each: 16 text tokens, c 980 px crops (256 image tokens each), a 16-128-token
                   question; the 8 questions of an image follow one another in the trace.  c = 1 and 4, every request at t = 0,
                   then Poisson arrivals at --rate requests/s.  max_new_tokens 16-128.
  system_prompt    256 requests: one 2,048-token system prompt, then a 16-512-token user text; t = 0; max_new_tokens 16-128.
  conversations    64 conversations of 4 turns: a 200-600-token first prompt, and each later turn is the previous turn's result
                   plus a 32-256-token user text, submitted when the previous turn finishes; max_new_tokens 32-128.
Every workload also runs "salted": the same trace with the first token of every request replaced by a distinct id, so lengths
and images are equal but no page key matches (the no-sharing baseline).
Reported per run: time to first token (p50, p99; first poll after admission less arrival, as bench_serving.py), generated
tokens/s, prefill tokens computed / prompt tokens, ViT rows run / submitted, cached pages evicted, peak memory.  Also: host time
of the page keys per 980 px crop, token equality of 4 requests that hit cached pages with batch-1 generate(), the paged-prefix
prefill kernel against the contiguous shared-prefix kernel (H = 20) with its bf16 FLOP floor (989 TFLOP/s, H100 SXM data
sheet), and the card name and power limit, read in the same call.
"""
import argparse
import json
import random
import time

import torch

from bench_serving import gpu_info, pct

BF16_TFLOPS = 989.0


def _text(rng, V, n):
    return torch.tensor([rng.randrange(10, V) for _ in range(n)], dtype=torch.long)


def image_trace(cfg, crops, rng, g):
    V, img = cfg["text_config"]["vocab_size"], cfg["image_token_index"]
    trace = []
    for _ in range(32):
        pv = torch.randn(crops, 3, 980, 980, generator=g).bfloat16()
        head = torch.cat([_text(rng, V, 16), torch.full((256 * crops,), img)])
        for _ in range(8):
            trace.append(dict(ids=torch.cat([head, _text(rng, V, rng.randint(16, 128))]), pv=pv, new=rng.randint(16, 128)))
    return trace


def system_trace(cfg, rng):
    V = cfg["text_config"]["vocab_size"]
    system = _text(rng, V, 2048)
    return [dict(ids=torch.cat([system, _text(rng, V, rng.randint(16, 512))]), pv=None, new=rng.randint(16, 128))
            for _ in range(256)]


def salted(trace, V):
    """The same requests with a distinct first token each: nothing shared."""
    out = []
    for i, r in enumerate(trace):
        ids = r["ids"].clone()
        ids[0] = 10 + i % (V - 10)
        out.append(dict(r, ids=ids))
    return out


def _report(eng, t0, ttft, gen, wall, submitted_rows):
    st = eng.stats
    return {"generated_tokens_per_s": round(gen / wall, 1), "wall_s": round(wall, 3),
            "ttft_s": {"p50": pct(ttft, 0.5), "p99": pct(ttft, 0.99)},
            "prefill_computed_over_prompt_tokens": round(1 - st["prefix_hit_tokens"] / max(1, st["prompt_tokens"]), 4),
            "prompt_tokens": st["prompt_tokens"], "prefix_hit_tokens": st["prefix_hit_tokens"],
            "vit_rows_run_over_submitted": f"{st['vit_rows_run']}/{submitted_rows}", "pages_evicted": st["pages_evicted"],
            "peak_memory_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}


def run_open(model, trace, arrivals, args):
    """Requests submitted at their arrival times (open loop)."""
    from aria_b200.serving import Engine
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    eng = Engine(model, max_batch=args.max_batch, max_kv_tokens=args.max_kv_tokens, poll_every=args.poll_every)
    order = sorted(range(len(trace)), key=lambda i: arrivals[i])
    rid_of, results, nxt = {}, {}, 0
    t0 = time.perf_counter()
    while nxt < len(order) or eng.n_active or eng.n_waiting:
        now = time.perf_counter() - t0
        while nxt < len(order) and arrivals[order[nxt]] <= now:
            r = trace[order[nxt]]
            rid_of[eng.add_request(r["ids"], r["pv"], max_new_tokens=r["new"])] = order[nxt]
            nxt += 1
        if not eng.n_active and not eng.n_waiting:
            time.sleep(max(0.0, arrivals[order[nxt]] - (time.perf_counter() - t0)))
            continue
        results.update(eng.step())
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    ttft = [eng.times[rid][0] - t0 - arrivals[i] for rid, i in rid_of.items()]
    assert all(results[rid].numel() == trace[i]["ids"].numel() + trace[i]["new"] for rid, i in rid_of.items())
    rows = sum(r["pv"].shape[0] for r in trace if r["pv"] is not None)
    out = _report(eng, t0, ttft, sum(r["new"] for r in trace), wall, rows)
    del eng
    torch.cuda.empty_cache()
    return out


def run_conversations(model, cfg, args, salt):
    """64 conversations x 4 turns, each turn submitted when the previous one finishes (closed loop)."""
    from aria_b200.serving import Engine
    rng = random.Random(args.seed + 7)
    V = cfg["text_config"]["vocab_size"]
    # every draw is made up front, so the cached and the salted runs see the same lengths whatever order turns finish in
    convs = [dict(prompt=_text(rng, V, rng.randint(200, 600)), turn=0, new=[rng.randint(32, 128) for _ in range(4)],
                  user=[_text(rng, V, rng.randint(32, 256)) for _ in range(3)]) for _ in range(64)]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    eng = Engine(model, max_batch=args.max_batch, max_kv_tokens=args.max_kv_tokens, poll_every=args.poll_every)
    live, ttft, gen, n_req = {}, [], 0, 0
    t0 = time.perf_counter()

    def submit(c):
        nonlocal gen, n_req
        ids = c["prompt"].clone()
        if salt:
            ids[0] = 10 + n_req
        new = c["new"][c["turn"]]
        gen += new
        n_req += 1
        live[eng.add_request(ids, max_new_tokens=new)] = (c, time.perf_counter())

    for c in convs:
        submit(c)
    while live:
        for rid, out in eng.step().items():
            c, arrived = live.pop(rid)
            ttft.append(eng.times[rid][0] - arrived)
            c["turn"] += 1
            if c["turn"] < 4:
                c["prompt"] = torch.cat([out.cpu(), c["user"][c["turn"] - 1]])
                submit(c)
    torch.cuda.synchronize()
    out = _report(eng, t0, ttft, gen, time.perf_counter() - t0, 0)
    del eng
    torch.cuda.empty_cache()
    return out


def key_host_time(cfg, g):
    from aria_b200.serving import page_keys
    img = cfg["image_token_index"]
    out = {}
    for crops in (1, 4):
        pv = torch.randn(crops, 3, 980, 980, generator=g).bfloat16()
        ids = torch.cat([torch.arange(10, 26), torch.full((256 * crops,), img), torch.arange(10, 300)])
        page_keys(ids, pv, None, img)
        t = time.perf_counter()
        for _ in range(5):
            page_keys(ids, pv, None, img)
        out[f"{crops}_crop_us_per_crop"] = round((time.perf_counter() - t) / 5 / crops * 1e6, 1)
    ids = torch.arange(10, 10 + 4096)
    t = time.perf_counter()
    for _ in range(20):
        page_keys(ids)
    out["text_4096_tokens_us"] = round((time.perf_counter() - t) / 20 * 1e6, 1)
    return out


def token_equality(model, trace):
    """4 questions about one image: the last 3 hit the first one's pages; each result against batch-1 generate()."""
    from aria_b200.serving import Engine
    eng = Engine(model, max_batch=4, max_kv_tokens=16 * 1024)
    picks = [dict(r, new=min(r["new"], 32)) for r in trace[:4]]
    rids = []
    for r in picks:
        rids.append(eng.add_request(r["ids"], r["pv"], max_new_tokens=r["new"]))
    got = eng.run()
    hit = eng.stats["prefix_hit_tokens"]
    del eng
    same = [bool(torch.equal(got[rid], model.generate(r["ids"][None], r["pv"], None, max_new_tokens=r["new"])[0]))
            for rid, r in zip(rids, picks)]
    model._decode_graph = None
    torch.cuda.empty_cache()
    return {"equal": same, "prefix_hit_tokens": hit}


def kernel(H=20, runs=50):
    from aria_b200 import ops
    dev = "cuda:0"
    out = {}
    for P in (1280, 4096, 16384):
        n = P // 256
        pre_k = torch.randn(1, H, P, 128, device=dev).bfloat16()
        pre_v = torch.randn_like(pre_k)
        perm = torch.randperm(n + 8, generator=torch.Generator().manual_seed(P))[:n]
        kp = torch.zeros(n + 8, H, 256, 128, device=dev, dtype=torch.bfloat16)
        vp = torch.zeros_like(kp)
        kp[perm.to(dev)] = pre_k[0].view(H, n, 256, 128).transpose(0, 1)
        vp[perm.to(dev)] = pre_v[0].view(H, n, 256, 128).transpose(0, 1)
        pages = perm.to(torch.int32).to(dev)
        for S in (1, 64, 512):
            qkv = torch.randn(3, 1, H, S, 128, device=dev).bfloat16()
            cu = torch.tensor([0, S], dtype=torch.int32, device=dev)
            a = lambda: ops.attention_prefill_shared_prefix(qkv[0], qkv[1], qkv[2], S, pre_k, pre_v, P, cu, 128 ** -0.5)
            b = lambda: ops.attention_prefill_paged_prefix(qkv[0], qkv[1], qkv[2], S, kp, vp, pages, P, cu, 128 ** -0.5)
            same = bool(torch.equal(a(), b()))

            def timed(fn):
                for _ in range(5):
                    fn()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(runs):
                    fn()
                e.record()
                e.synchronize()
                return s.elapsed_time(e) / runs
            ms = {"contiguous": [], "paged": []}
            for _ in range(3):                                   # alternate the two kernels
                ms["contiguous"].append(timed(a))
                ms["paged"].append(timed(b))
            med = {k: sorted(v)[1] for k, v in ms.items()}
            flops = 4.0 * H * 128 * S * (P + (S + 1) / 2)        # QK^T and PV over the keys each query sees
            floor_ms = flops / (BF16_TFLOPS * 1e12) * 1e3
            out[f"P{P}_S{S}"] = {"contiguous_ms": round(med["contiguous"], 4), "paged_ms": round(med["paged"], 4),
                                 "flop_floor_ms": round(floor_ms, 5), "paged_flop_floor_fraction": round(floor_ms / med["paged"], 3),
                                 "bit_identical": same}
        del pre_k, pre_v, kp, vp
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rate", type=float, default=8.0)
    ap.add_argument("--max-batch", type=int, default=64)
    ap.add_argument("--max-kv-tokens", type=int, default=65536)
    ap.add_argument("--poll-every", type=int, default=8)
    ap.add_argument("--lm-layers", type=int, default=16)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    from aria_b200 import configs as C
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration, init_random_
    if not torch.cuda.is_available():
        raise SystemExit("bench_prefix_cache.py needs a GPU")
    cfg = C.with_layers(C.ARIA_25B, lm_layers=args.lm_layers)
    V = cfg["text_config"]["vocab_size"]
    name, power = gpu_info(0)
    out = {"bench": "prefix_cache", "gpu": name, "power_limit_w": power, "dtype": "bf16",
           "model": f"Aria full width, {args.lm_layers} of 28 LM layers, random init (seed 0)",
           "max_batch": args.max_batch, "max_kv_tokens": args.max_kv_tokens, "poll_every": args.poll_every, "seed": args.seed,
           "flop_floor_source": f"{BF16_TFLOPS} TFLOP/s dense bf16, H100 SXM data sheet"}
    g = torch.Generator().manual_seed(args.seed)
    out["page_keys_host"] = key_host_time(cfg, g)
    with torch.no_grad():
        model = AriaForConditionalGeneration(AriaConfig.from_dict(cfg), device="cuda:0")
        init_random_(model, seed=0)
        out["paged_prefix_kernel"] = kernel(cfg["text_config"]["num_attention_heads"])
        rng = random.Random(args.seed)
        traces = {"images_1crop": image_trace(cfg, 1, rng, g), "images_4crop": image_trace(cfg, 4, rng, g),
                  "system_prompt": system_trace(cfg, rng)}
        out["hit_requests_equal_generate"] = token_equality(model, traces["images_4crop"])
        arr = random.Random(args.seed + 1)
        for name_, trace in traces.items():
            zero = [0.0] * len(trace)
            runs = {"t0": zero}
            if name_.startswith("images"):
                poisson, t = [], 0.0
                for _ in trace:
                    t += arr.expovariate(args.rate)
                    poisson.append(t)
                runs[f"poisson_{args.rate}_per_s"] = poisson
            for when, arrivals in runs.items():
                out[f"{name_}_{when}"] = {"cached": run_open(model, trace, arrivals, args),
                                          "salted": run_open(model, salted(trace, V), arrivals, args)}
        out["conversations"] = {"cached": run_conversations(model, cfg, args, False),
                                "salted": run_conversations(model, cfg, args, True)}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
