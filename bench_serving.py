"""Continuous batching (aria_b200.serving.Engine) against static batching on one GPU; prints one JSON line.

    python bench_serving.py [--requests 256] [--rate 4.0] [--max-batch 64] [--max-kv-tokens 65536] [--lm-layers 16]

Model: full-width Aria (hidden 2560, 64 experts, the 27-layer ViT) with random weights (seed 0) and --lm-layers of the 28 LM
layers, so that the weights, the engine's page pool and the static baseline's cache fit on one 80 GB card together.
Trace (seeded): --requests requests, text prompts of 64-2048 tokens (log-uniform), a quarter of them with one 980 px image
(256 image tokens), max_new_tokens uniform in 16-512, greedy, no EOS (random weights emit no meaningful EOS, so the budgets are
what makes the rows ragged).
Arms:
  engine   Engine(max_batch) over the trace, every request at t = 0, then with Poisson arrivals at --rate requests/s.
  static   generate() on left-padded groups of 32 in arrival order, each with its members' largest max_new_tokens, run back to
           back once; for Poisson arrivals a group starts when its last member has arrived and the previous group is done (the
           same measured group durations, on a virtual clock).  Its tokens are delivered when generate() returns.
Reported: generated tokens/s (tokens each request asked for, over the wall time from the first arrival to the last result),
time to first token and time per output token (p50, p99), peak memory, mean slot occupancy, host time in polls.  The two arms
define the per-request times as follows (`definitions` in the output):
  engine   first token: the first poll after the request's admission, less its arrival; per output token: (the poll that saw
           it finish - that first poll) / (max_new_tokens - 1), so decode only, with the admissions of other requests that ran
           meanwhile included; both are upper bounds at poll granularity.  Mean slot occupancy: slot-steps of admitted requests
           not yet retired / (decode steps x max_batch); a request that finished between two polls counts until the poll.
  static   first token: when its group's generate() returns (it delivers every token then), less its arrival; per output
           token: (the group's generate() time - the same call's time with max_new_tokens=1) / (group budget - 1), the
           decode steps only.
Also reported: the paged decode kernel against the devlen one at (R 32, 2K keys) and (R 64, 8K keys) with their HBM floor (K + V bytes / 3.35 TB/s, the H100 SXM data sheet); token equality
of 4 engine requests with batch-1 generate(); the card name and power limit, read in the same call.
"""
import argparse
import json
import math
import random
import subprocess
import time

import torch

HBM_GBS = 3350.0


def gpu_info(idx=0):
    name = torch.cuda.get_device_name(idx)
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(idx), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:
        power = None
    return name, power


def make_trace(cfg, n, seed=0):
    rng = random.Random(seed)
    g = torch.Generator().manual_seed(seed)
    V, img = cfg["text_config"]["vocab_size"], cfg["image_token_index"]
    trace = []
    for i in range(n):
        T = int(round(math.exp(rng.uniform(math.log(64), math.log(2048)))))
        ids = torch.randint(10, V, (T,), generator=g)
        pv = None
        if rng.random() < 0.25:
            ids = torch.cat([ids[:8], torch.full((256,), img), ids[8:]])
            pv = torch.randn(1, 3, 980, 980, generator=g).bfloat16()
        trace.append(dict(ids=ids, pv=pv, new=rng.randint(16, 512)))
    return trace


def pct(xs, q):
    xs = sorted(xs)
    return round(xs[min(len(xs) - 1, int(q * len(xs)))], 4)


def run_engine(model, trace, arrivals, args):
    from aria_b200.serving import Engine
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    eng = Engine(model, max_batch=args.max_batch, max_kv_tokens=args.max_kv_tokens, poll_every=args.poll_every)
    order = sorted(range(len(trace)), key=lambda i: arrivals[i])
    rid_of = {}
    t0 = time.perf_counter()
    nxt, results = 0, {}
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
    st = eng.stats
    gen = sum(r["new"] for r in trace)
    assert all(results[rid].numel() == trace[i]["ids"].numel() + trace[i]["new"] for rid, i in rid_of.items())
    out = {"generated_tokens_per_s": round(gen / wall, 1), "wall_s": round(wall, 3),
           "ttft_s": {"p50": pct(ttft, 0.5), "p99": pct(ttft, 0.99)},
           "tpot_ms": {"p50": pct([x * 1e3 for x in tpot], 0.5), "p99": pct([x * 1e3 for x in tpot], 0.99)},
           "peak_memory_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
           "mean_slot_occupancy": round(st["active_slot_steps"] / max(1, st["steps"] * args.max_batch), 4),
           "decode_steps": st["steps"], "polls": st["polls"], "poll_host_s": round(st["poll_host_s"], 3),
           "graphs_captured": st["graphs_captured"]}
    del eng
    torch.cuda.empty_cache()
    return out


def run_static(model, trace, args):
    """Groups of 32 in arrival (index) order, back to back -> per group (members, duration s, duration s of the same call with
    max_new_tokens=1: graph capture, ViT, prefill and first token)."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    groups = []
    for g0 in range(0, len(trace), 32):
        mem = list(range(g0, min(g0 + 32, len(trace))))
        T = max(trace[i]["ids"].numel() for i in mem)
        ids = torch.zeros(len(mem), T, dtype=torch.long)
        mask = torch.zeros(len(mem), T, dtype=torch.long)
        for b, i in enumerate(mem):
            n = trace[i]["ids"].numel()
            ids[b, T - n:] = trace[i]["ids"]
            mask[b, T - n:] = 1
        pvs = [trace[i]["pv"] for i in mem if trace[i]["pv"] is not None]
        pv = torch.cat(pvs) if pvs else None
        new = max(trace[i]["new"] for i in mem)
        durs = []
        for n in (1, new):
            torch.cuda.synchronize()
            t = time.perf_counter()
            model.generate(ids, pv, None, max_new_tokens=n, attention_mask=mask)
            torch.cuda.synchronize()
            durs.append(time.perf_counter() - t)
            model._decode_graph = None
            torch.cuda.empty_cache()
        groups.append((mem, durs[1], durs[0]))
    return groups, round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)


def static_report(trace, groups, arrivals, peak):
    clock, ttft, tpot = 0.0, [], []
    for mem, dur, first in groups:
        start = max(clock, max(arrivals[i] for i in mem))
        clock = start + dur
        new = max(trace[m]["new"] for m in mem)
        for i in mem:
            ttft.append(clock - arrivals[i])                 # tokens are delivered when generate() returns
            tpot.append((dur - first) / max(1, new - 1))     # the group's decode steps, prefill and first token excluded
    gen = sum(r["new"] for r in trace)
    return {"generated_tokens_per_s": round(gen / clock, 1), "wall_s": round(clock, 3),
            "ttft_s": {"p50": pct(ttft, 0.5), "p99": pct(ttft, 0.99)},
            "tpot_ms": {"p50": pct([x * 1e3 for x in tpot], 0.5), "p99": pct([x * 1e3 for x in tpot], 0.99)},
            "peak_memory_gib": peak}


def paged_kernel(H, runs=200):
    from aria_b200 import ops
    dev = "cuda:0"
    out = {}
    for R, keys in ((32, 2048), (64, 8192)):
        P = keys // 256
        q = torch.randn(R, H, 128, device=dev).bfloat16()
        k = torch.randn(R, H, keys, 128, device=dev).bfloat16()
        v = torch.randn_like(k)
        lens = torch.full((R,), keys, dtype=torch.int32, device=dev)
        perm = torch.randperm(R * P, generator=torch.Generator().manual_seed(R)).to(dev)
        bt = perm.view(R, P).to(torch.int32)
        kp = torch.empty(R * P, H, 256, 128, device=dev, dtype=torch.bfloat16)
        vp = torch.empty_like(kp)
        kp[perm] = k.view(R, H, P, 256, 128).permute(0, 2, 1, 3, 4).reshape(R * P, H, 256, 128)
        vp[perm] = v.view(R, H, P, 256, 128).permute(0, 2, 1, 3, 4).reshape(R * P, H, 256, 128)
        a = ops.attention_decode_devlen(q, k, v, lens, 128 ** -0.5)
        b = ops.attention_decode_paged(q, kp, vp, bt, lens, 128 ** -0.5)
        same = bool(torch.equal(a, b))

        def timed(fn):
            for _ in range(10):
                fn()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(runs):
                fn()
            e.record()
            e.synchronize()
            return s.elapsed_time(e) / runs
        ms = {}
        for rep in range(3):                                   # alternate the two kernels
            ms.setdefault("devlen", []).append(timed(lambda: ops.attention_decode_devlen(q, k, v, lens, 128 ** -0.5)))
            ms.setdefault("paged", []).append(timed(lambda: ops.attention_decode_paged(q, kp, vp, bt, lens, 128 ** -0.5)))
        floor_ms = 2 * R * H * keys * 128 * 2 / (HBM_GBS * 1e9) * 1e3
        med = {kk: sorted(x)[1] for kk, x in ms.items()}
        out[f"R{R}_keys{keys}"] = {"devlen_ms": round(med["devlen"], 4), "paged_ms": round(med["paged"], 4),
                                   "hbm_floor_ms": round(floor_ms, 4),
                                   "paged_hbm_floor_fraction": round(floor_ms / med["paged"], 3),
                                   "devlen_hbm_floor_fraction": round(floor_ms / med["devlen"], 3), "bit_identical": same}
        del k, v, kp, vp
        torch.cuda.empty_cache()
    return out


def token_equality(model, trace, args):
    from aria_b200.serving import Engine
    eng = Engine(model, max_batch=4, max_kv_tokens=16 * 1024, poll_every=args.poll_every)
    picks = [dict(trace[i], new=min(trace[i]["new"], 48)) for i in range(4)]
    rids = [eng.add_request(r["ids"], r["pv"], max_new_tokens=r["new"]) for r in picks]
    got = eng.run()
    del eng
    same = []
    for rid, r in zip(rids, picks):
        want = model.generate(r["ids"][None], r["pv"], None, max_new_tokens=r["new"])[0]
        same.append(bool(torch.equal(got[rid], want)))
    model._decode_graph = None
    torch.cuda.empty_cache()
    return same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--rate", type=float, default=4.0)
    ap.add_argument("--max-batch", type=int, default=64)
    ap.add_argument("--max-kv-tokens", type=int, default=65536)
    ap.add_argument("--poll-every", type=int, default=8)
    ap.add_argument("--lm-layers", type=int, default=16)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    from aria_b200 import configs as C
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration, init_random_
    if not torch.cuda.is_available():
        raise SystemExit("bench_serving.py needs a GPU")
    cfg = C.with_layers(C.ARIA_25B, lm_layers=args.lm_layers)
    name, power = gpu_info(0)
    out = {"bench": "serving", "gpu": name, "power_limit_w": power, "dtype": "bf16",
           "model": f"Aria full width, {args.lm_layers} of 28 LM layers, random init (seed 0)",
           "trace": {"requests": args.requests, "prompt_tokens": "64-2048 log-uniform", "images": "1 in 4, 980 px",
                     "max_new_tokens": "16-512 uniform", "sampling": "greedy, no EOS", "seed": args.seed},
           "max_batch": args.max_batch, "max_kv_tokens": args.max_kv_tokens, "poll_every": args.poll_every,
           "hbm_floor_source": f"{HBM_GBS} GB/s, H100 SXM data sheet",
           "definitions": {
               "engine_ttft": "first poll after admission - arrival (poll granularity)",
               "engine_tpot": "(poll that saw it finish - first poll) / (max_new_tokens - 1): decode, with other requests' "
                              "admissions that ran meanwhile",
               "static_ttft": "its group's generate() return - arrival (tokens delivered at return)",
               "static_tpot": "(group generate() time - same call with max_new_tokens=1) / (group budget - 1): decode steps only",
               "mean_slot_occupancy": "slot-steps of admitted, not yet retired requests / (decode steps x max_batch); finished "
                                      "requests count until the poll that retires them"}}
    with torch.no_grad():
        model = AriaForConditionalGeneration(AriaConfig.from_dict(cfg), device="cuda:0")
        init_random_(model, seed=0)
        out["paged_decode_kernel"] = paged_kernel(cfg["text_config"]["num_attention_heads"])
        trace = make_trace(cfg, args.requests, args.seed)
        out["tokens_equal_generate_4_requests"] = token_equality(model, trace, args)
        zero = [0.0] * len(trace)
        rng = random.Random(args.seed + 1)
        poisson, t = [], 0.0
        for _ in trace:
            t += rng.expovariate(args.rate)
            poisson.append(t)
        groups, static_peak = run_static(model, trace, args)
        out["all_at_t0"] = {"engine": run_engine(model, trace, zero, args),
                            "static": static_report(trace, groups, zero, static_peak)}
        out[f"poisson_{args.rate}_per_s"] = {"engine": run_engine(model, trace, poisson, args),
                                             "static": static_report(trace, groups, poisson, static_peak)}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
