"""Token log-probabilities on the GPU; prints one JSON line with the card's name and power limit, read in the same run.

    python bench_logprobs.py [--iters 50] [--lm-layers 4] [--requests 128] [--kernel-only]

  kernel          ops.token_logprobs at V = 100,352 for R rows x top-n (CUDA events), against the HBM floor of one read of the
                  logits (R x V x 2 bytes at 3.35 TB/s, the H100 SXM data sheet) and ops.sample_tokens_slots on the same rows.
  generate        generate()'s decode ms per step with output_logprobs None / 0 / 5 / 20, greedy, at batch 1 from a 16-token
                  prompt (gpt-fast's protocol) and at batch 32
                  from 2K-token prompts, as bench_generate.py times them (the captured step replayed, CUDA events).
  engine_step     serving.Engine decode step at 64 slots with 2K-token prompts, none / all logprobs = 5 / all logprobs = 20
                  asking: wall time of step() calls after every request is admitted, over the decode steps they replayed; this
                  includes the polls and the host copy of the logprob rings.
  serving_trace   bench_serving.py's trace (seeded, --requests of them) with every request at t = 0, none vs every request
                  logprobs = 5: generated tokens/s, TTFT and TPOT p50.
  prompt_scoring  64 prompts of 2,048 tokens, max_new_tokens = 1, prompt_logprobs None / 0 / 5: prompt tokens/s and peak memory.
Model (all but the kernel): full-width Aria with random weights (seed 0) and --lm-layers of the 28 LM layers.
"""
import argparse
import json
import subprocess
import time

import torch

V = 100352
HBM_BPS = 3.35e12


def _time(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def _wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def bench_generate(model, V, dev, iters=3):
    """The captured decode step of generate() (GraphedDecode, greedy) with logprobs None / 0 / 5 / 20, as bench_generate.py times
    it: the graph replayed n - 1 times from a T-token prompt state (cache rows random), ms per step by CUDA events, min of
    iters runs."""
    from aria_b200.modeling_aria import GraphedDecode
    out = {}
    for B, T, n in ((1, 16, 128), (32, 2048, 64)):
        row = {}
        for k in (None, 0, 5, 20):
            model._decode_graph = None
            torch.cuda.empty_cache()
            g = GraphedDecode(model, B, -(-(T + n) // 256) * 256, n, (0.0, 0, 1.0, 0), (), 0, logprobs=k)
            for t in g.cache.k + g.cache.v:
                t.normal_()
            gen = torch.Generator(device=dev).manual_seed(5)
            g.state.ids_in.copy_(torch.randint(10, V, (B, 1), generator=gen, device=dev))

            def replays():
                g.start(T, None)
                g.sample_and_advance(g.logits[:, -1])
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(n - 1):
                    g.graph.replay()
                b.record()
                b.synchronize()
                return a.elapsed_time(b) / (n - 1)

            replays()
            row[str(k)] = round(min(replays() for _ in range(iters)), 4)
            del g
        out[f"B{B}_T{T}_ms_per_step"] = row
    torch.cuda.empty_cache()
    return out


def bench_engine_step(model, V):
    from aria_b200.serving import Engine
    g = torch.Generator().manual_seed(2)
    prompts = [torch.randint(10, V, (2048,), generator=g) for _ in range(64)]
    out = {}
    for k in (None, 5, 20):
        eng = Engine(model, max_batch=64, max_kv_tokens=64 * (2048 + 256), poll_every=8)
        for p in prompts:
            eng.add_request(p, max_new_tokens=200, logprobs=k)
        while eng.n_waiting or eng.sched.partial is not None:  # admits and prefills all 64
            eng.step()
        eng.step()                                               # captures the step graph
        steps0 = eng.stats["steps"]
        dt, _ = _wall(lambda: [eng.step() for _ in range(16)])
        out[str(k)] = round(dt / (eng.stats["steps"] - steps0) * 1e3, 3)
        eng.run()
        del eng
        torch.cuda.empty_cache()
    return out


def _run_trace(model, trace, k):
    from aria_b200.serving import Engine
    eng = Engine(model, max_batch=64, max_kv_tokens=65536, poll_every=8)
    t0 = time.perf_counter()
    rids = {eng.add_request(r["ids"], r["pv"], max_new_tokens=r["new"], logprobs=k): r for r in trace}
    eng.run()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    ttft = sorted(eng.times[rid][0] - t0 for rid in rids)
    tpot = sorted((eng.times[rid][1] - eng.times[rid][0]) / (r["new"] - 1) for rid, r in rids.items() if r["new"] > 1)
    if k is not None:
        assert all(eng.logprobs[rid].top_ids.shape == (r["new"], k) for rid, r in rids.items())
    res = {"generated_tokens_per_s": round(sum(r["new"] for r in trace) / wall, 1),
           "ttft_p50_s": round(ttft[len(ttft) // 2], 3), "tpot_p50_ms": round(tpot[len(tpot) // 2] * 1e3, 3)}
    del eng
    torch.cuda.empty_cache()
    return res


def bench_serving_trace(model, cfg, n):
    from bench_serving import make_trace
    trace = make_trace(cfg, n, 0)
    _run_trace(model, trace[:8], 5)                              # warm-up: graphs of both kinds, the ViT
    out = {}
    for rnd in range(2):                                         # alternated, two rounds
        for k in (None, 5):
            out.setdefault(str(k), []).append(_run_trace(model, trace, k))
    return out


def bench_prompt_scoring(model, V):
    from aria_b200.serving import Engine
    g = torch.Generator().manual_seed(3)
    prompts = [torch.randint(10, V, (2048,), generator=g) for _ in range(64)]
    out = {}
    for k in (None, 0, 5):
        eng = Engine(model, max_batch=64, max_kv_tokens=64 * 2304, poll_every=8)
        eng.add_request(prompts[0][:300], max_new_tokens=1, prompt_logprobs=k)   # warm-up
        eng.run()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        for i, p in enumerate(prompts):
            p = p.clone()
            p[0] = 10 + i                                        # distinct first pages: no prefix hits in any arm
            eng.add_request(p, max_new_tokens=1, prompt_logprobs=k)
        dt, _ = _wall(eng.run)
        out[str(k)] = {"prompt_tokens_per_s": round(64 * 2048 / dt, 1),
                       "peak_memory_above_start_gib": round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 3)}
        del eng
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--lm-layers", type=int, default=4)
    ap.add_argument("--requests", type=int, default=128)
    ap.add_argument("--kernel-only", action="store_true")
    args = ap.parse_args()
    from aria_b200 import ops
    if not torch.cuda.is_available():
        raise SystemExit("bench_logprobs.py needs a GPU")
    dev = "cuda:0"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    g = torch.Generator(device=dev).manual_seed(0)
    rows = []
    for R in (1, 32, 64, 256, 1024):
        x = (3 * torch.randn(R, V, generator=g, device=dev)).bfloat16()
        tok = torch.randint(V, (R,), generator=g, device=dev)
        i32 = dict(dtype=torch.int32, device=dev)
        samp = (torch.ones(R, device=dev), torch.full((R,), 50, **i32), torch.full((R,), 0.9, device=dev),
                torch.zeros(R, dtype=torch.int64, device=dev), torch.zeros(R, **i32), torch.zeros(R, dtype=torch.int64, device=dev))
        s_ms = _time(lambda: ops.sample_tokens_slots(x, *samp), args.iters)
        floor_ms = R * V * 2 / HBM_BPS * 1e3
        for n in (0, 5, 20):
            out = ops.token_logprobs(x, tok, n)
            ms = _time(lambda: ops.token_logprobs(x, tok, n, out=out), args.iters)
            rows.append({"R": R, "n": n, "ms": round(ms, 4), "hbm_floor_ms": round(floor_ms, 4),
                         "floor_share": round(floor_ms / ms, 3), "sample_tokens_slots_ms": round(s_ms, 4)})
    result = {"bench": "token_logprobs", "V": V, "card": card, "kernel": rows}
    if not args.kernel_only:
        from aria_b200 import configs as C
        from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration, init_random_
        cfg = C.with_layers(C.ARIA_25B, lm_layers=args.lm_layers)
        result["model"] = f"Aria full width, {args.lm_layers} of 28 LM layers, random init (seed 0)"
        with torch.no_grad():
            model = AriaForConditionalGeneration(AriaConfig.from_dict(cfg), device=dev)
            init_random_(model, seed=0)
            Vm = cfg["text_config"]["vocab_size"]
            result["generate"] = bench_generate(model, Vm, dev)
            result["engine_step_ms_64_slots_2k"] = bench_engine_step(model, Vm)
            result["prompt_scoring_64x2048"] = bench_prompt_scoring(model, Vm)
            result[f"serving_trace_{args.requests}_at_t0"] = bench_serving_trace(model, cfg, args.requests)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
