"""Batched and chunked admission in aria_b200.serving.Engine on one GPU; prints one JSON line.

    python bench_admission.py [--requests 256] [--rate 4.0] [--max-batch 64] [--max-kv-tokens 65536] [--lm-layers 16]
                              [--budgets none,2048,4096,8192,16384]

Model: full-width Aria (hidden 2560, 64 experts, the 27-layer ViT) with random weights (seed 0) and --lm-layers of the 28 LM
layers, as in bench_serving.py.
Parts:
  kernel   aria_attention_prefill_paged_varlen over 16 segments of 64-2048 tokens with prefixes of 0, 256 or 2048 keys on
           shuffled pages, against one aria_attention_prefill_paged_prefix launch per segment on the same segments (H = 20),
           with the FLOP floor (QK^T and PV over the keys each query sees, at the 989 TFLOP/s dense BF16 of the H100 SXM data
           sheet) and bit-identity.
  prefill  one packed prefill_paged of k text prompts (64-2048 tokens, log-uniform) against k batch-1 prefill_paged calls,
           k in {1, 4, 16}: ms and prompt tokens/s.
  engine   Engine(max_prefill_tokens=b) for each budget b on bench_serving.py's trace (all at t = 0, and Poisson arrivals at
           --rate requests/s) and on bench_prefix_cache.py's 32-image (4 crops) and 2,048-token system-prompt traces, all at
           t = 0: generated tokens/s, time to first token and time per output token (p50, p99; defined as bench_serving.py
           defines the engine's), peak memory, prefill launches and chunks.
The card name and power limit are read in the same call.
"""
import argparse
import json
import math
import random
import time

import torch

from bench_serving import gpu_info, make_trace, pct

BF16_TFLOPS = 989.0


def _timed(fn, runs):
    for _ in range(3):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(runs):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / runs


def kernel(H=20, runs=20):
    from aria_b200 import ops
    dev = "cuda:0"
    rng = random.Random(0)
    lens = [int(round(math.exp(rng.uniform(math.log(64), math.log(2048))))) for _ in range(16)]
    prefixes = [rng.choice((0, 256, 2048)) for _ in lens]
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    S = cu[-1]
    n_pages = sum(P // 256 for P in prefixes) + 1
    qkv = torch.randn(3, 1, H, S, 128, device=dev).bfloat16()
    kp = torch.randn(n_pages, H, 256, 128, device=dev).bfloat16()
    vp = torch.randn_like(kp)
    perm = (torch.randperm(n_pages - 1, generator=torch.Generator().manual_seed(1)) + 1).tolist()
    table = torch.full((16, 8), -1, dtype=torch.int32)
    for b, P in enumerate(prefixes):
        for i in range(P // 256):
            table[b, i] = perm.pop()
    table = table.to(dev)
    seg = ops.PackedSegments(cu, prefixes, dev)
    parts = [qkv[:, :, :, cu[b]:cu[b + 1]].contiguous() for b in range(16)]
    cus = [torch.tensor([0, n], dtype=torch.int32, device=dev) for n in lens]
    varlen = lambda: ops.attention_prefill_paged_varlen(qkv[0], qkv[1], qkv[2], kp, vp, table, seg, 128 ** -0.5)

    def per_segment():
        return [ops.attention_prefill_paged_prefix(p[0], p[1], p[2], n, kp, vp, table[b], P, c, 128 ** -0.5)
                for b, (p, n, P, c) in enumerate(zip(parts, lens, prefixes, cus))]
    same = bool(torch.equal(varlen(), torch.cat(per_segment())))
    ms = {"varlen": [], "per_segment": []}
    for _ in range(3):                                       # alternate the two
        ms["varlen"].append(_timed(varlen, runs))
        ms["per_segment"].append(_timed(per_segment, runs))
    med = {k: sorted(v)[1] for k, v in ms.items()}
    flops = sum(4.0 * H * 128 * n * (P + (n + 1) / 2) for n, P in zip(lens, prefixes))
    floor_ms = flops / (BF16_TFLOPS * 1e12) * 1e3
    return {"segments": lens, "prefixes": prefixes, "heads": H, "varlen_ms": round(med["varlen"], 4),
            "per_segment_ms": round(med["per_segment"], 4), "flop_floor_ms": round(floor_ms, 4),
            "varlen_flop_floor_fraction": round(floor_ms / med["varlen"], 3), "bit_identical": same}


def prefill(model, runs=3):
    from aria_b200 import ops
    from aria_b200.moe_lm import PagedKVCache
    lm = model.language_model
    c = lm.config
    dev = "cuda:0"
    rng = random.Random(2)
    g = torch.Generator().manual_seed(2)
    out = {}
    for k in (1, 4, 16):
        lens = [int(round(math.exp(rng.uniform(math.log(64), math.log(2048))))) for _ in range(k)]
        prompts = [torch.randint(10, c.vocab_size, (n,), generator=g) for n in lens]
        width = 8
        cache = PagedKVCache(c.num_hidden_layers, k * width + 1, c.num_attention_heads, c.head_dim, k, width, dev)
        table = (torch.arange(k * width, dtype=torch.int32) + 1).view(k, width).to(dev)
        emb = [ops.embedding(p.to(dev)[None], lm.get_input_embeddings().weight) for p in prompts]
        pos = [torch.arange(n, dtype=torch.int32, device=dev) for n in lens]
        singles = [ops.PackedSegments([0, n], [0], dev) for n in lens]
        cu = [0]
        for n in lens:
            cu.append(cu[-1] + n)
        packed_seg = ops.PackedSegments(cu, [0] * k, dev)
        packed_emb, packed_pos = torch.cat(emb, dim=1), torch.cat(pos)

        def one_by_one():
            return [lm.prefill_paged(emb[b], cache, table[b:b + 1], singles[b], pos[b]) for b in range(k)]

        def packed():
            return lm.prefill_paged(packed_emb, cache, table, packed_seg, packed_pos)
        same = bool(torch.equal(torch.cat([x[0] for x in one_by_one()]), packed()[0]))
        ms = {"batch1_calls": [], "packed": []}
        for _ in range(3):
            ms["batch1_calls"].append(_timed(one_by_one, runs))
            ms["packed"].append(_timed(packed, runs))
        med = {kk: sorted(v)[1] for kk, v in ms.items()}
        out[f"k{k}"] = {"prompt_tokens": sum(lens), "batch1_calls_ms": round(med["batch1_calls"], 2),
                        "packed_ms": round(med["packed"], 2),
                        "batch1_calls_tokens_per_s": round(sum(lens) / med["batch1_calls"] * 1e3),
                        "packed_tokens_per_s": round(sum(lens) / med["packed"] * 1e3), "logits_bit_identical": same}
        del cache
        torch.cuda.empty_cache()
    return out


def run_engine(model, trace, arrivals, args, budget):
    from aria_b200.serving import Engine
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    eng = Engine(model, max_batch=args.max_batch, max_kv_tokens=args.max_kv_tokens, poll_every=args.poll_every,
                 max_prefill_tokens=budget)
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
    ttft, tpot = [], []
    for rid, i in rid_of.items():
        first, last = eng.times[rid]
        ttft.append(first - t0 - arrivals[i])
        if trace[i]["new"] > 1:
            tpot.append((last - first) / (trace[i]["new"] - 1))
    assert all(results[rid].numel() == trace[i]["ids"].numel() + trace[i]["new"] for rid, i in rid_of.items())
    st = eng.stats
    out = {"generated_tokens_per_s": round(sum(r["new"] for r in trace) / wall, 1), "wall_s": round(wall, 3),
           "ttft_s": {"p50": pct(ttft, 0.5), "p99": pct(ttft, 0.99)},
           "tpot_ms": {"p50": pct([x * 1e3 for x in tpot], 0.5), "p99": pct([x * 1e3 for x in tpot], 0.99)},
           "peak_memory_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
           "prefill_launches": st["prefill_launches"], "prefill_chunks": st["prefill_chunks"],
           "prefix_hit_tokens": st["prefix_hit_tokens"]}
    del eng
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--rate", type=float, default=4.0)
    ap.add_argument("--max-batch", type=int, default=64)
    ap.add_argument("--max-kv-tokens", type=int, default=65536)
    ap.add_argument("--poll-every", type=int, default=8)
    ap.add_argument("--lm-layers", type=int, default=16)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--budgets", default="none,2048,4096,8192,16384")
    ap.add_argument("--parts", default="kernel,prefill,engine")
    ap.add_argument("--traces", default="t0,poisson,images,system")
    args = ap.parse_args()
    from aria_b200 import configs as C
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration, init_random_
    from bench_prefix_cache import image_trace, system_trace
    if not torch.cuda.is_available():
        raise SystemExit("bench_admission.py needs a GPU")
    budgets = [None if b == "none" else int(b) for b in args.budgets.split(",")]
    parts = args.parts.split(",")
    cfg = C.with_layers(C.ARIA_25B, lm_layers=args.lm_layers)
    name, power = gpu_info(0)
    out = {"bench": "admission", "gpu": name, "power_limit_w": power, "dtype": "bf16",
           "model": f"Aria full width, {args.lm_layers} of 28 LM layers, random init (seed 0)",
           "max_batch": args.max_batch, "max_kv_tokens": args.max_kv_tokens, "poll_every": args.poll_every,
           "flop_floor_source": f"{BF16_TFLOPS} TFLOP/s dense BF16, H100 SXM data sheet"}
    with torch.no_grad():
        if "kernel" in parts:
            out["kernel"] = kernel(cfg["text_config"]["num_attention_heads"])
        model = AriaForConditionalGeneration(AriaConfig.from_dict(cfg), device="cuda:0")
        init_random_(model, seed=0)
        if "prefill" in parts:
            out["prefill"] = prefill(model)
        if "engine" in parts:
            trace = make_trace(cfg, args.requests, args.seed)
            rng = random.Random(args.seed + 1)
            poisson, t = [], 0.0
            for _ in trace:
                t += rng.expovariate(args.rate)
                poisson.append(t)
            rng2, g2 = random.Random(args.seed), torch.Generator().manual_seed(args.seed)
            img = image_trace(cfg, 4, rng2, g2)
            sys_ = system_trace(cfg, rng2)
            traces = {"t0": ("serving_all_at_t0", trace, [0.0] * len(trace)),
                      "poisson": (f"serving_poisson_{args.rate}_per_s", trace, poisson),
                      "images": ("prefix_cache_32_images_4_crops_at_t0", img, [0.0] * len(img)),
                      "system": ("prefix_cache_system_prompt_at_t0", sys_, [0.0] * len(sys_))}
            out["engine"] = {}
            for key in args.traces.split(","):
                tname, tr, arr = traces[key]
                out["engine"][tname] = {str(b): run_engine(model, tr, arr, args, b) for b in budgets}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
