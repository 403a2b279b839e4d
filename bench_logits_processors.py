"""Repetition penalty, min-p and min_new_tokens on the GPU; prints one JSON line with the card's name and power limit, read in the
same run.

    python bench_logits_processors.py [--iters 50] [--lm-layers 4] [--requests 128] [--kernel-only]

  sampler         at V = 100,352 and R rows (CUDA events, the arms alternated over rounds): ops.sample_tokens_slots (today's
                  kernel) against ops.sample_tokens_processed with every processor off, with repetition_penalty 1.1 (a 2K-id
                  history per row), and with min_p 0.05 at top_k 0; sampling at temperature 1, top_k 50, top_p 0.9 otherwise.
                  Each against the HBM floor of one read of the logits (R x V x 2 bytes at 3.35 TB/s, the H100 SXM data sheet).
  presence_set    the per-step bitmap update (one id per row) at 64 and 1024 rows.
  generate        generate()'s decode ms per step, greedy, at batch 1 from a 16-token prompt and at batch 32 from 2K-token
                  prompts, without and with repetition_penalty = 1.1 (the captured step replayed, CUDA events, as
                  bench_logprobs.py times it).
  serving_trace   bench_serving.py's trace (seeded, --requests of them) with every request at t = 0 and sampled (temperature 1,
                  top_k 50), without and with repetition_penalty = 1.05, min_p = 0.05: generated tokens/s, TTFT and TPOT p50.
Model (all but the kernels): full-width Aria with random weights (seed 0) and --lm-layers of the 28 LM layers.
"""
import argparse
import json
import subprocess
import time

import torch

V = 100352
HBM_BPS = 3.35e12


def _time(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def bench_sampler(ops, dev, iters, rounds=3):
    g = torch.Generator(device=dev).manual_seed(0)
    rows = []
    for R in (1, 32, 256, 1024):
        x = (3 * torch.randn(R, V, generator=g, device=dev)).bfloat16()
        i32, f32, i64 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.float32, device=dev), dict(dtype=torch.int64, device=dev)
        temp, k50, p09 = torch.ones(R, **f32), torch.full((R,), 50, **i32), torch.full((R,), 0.9, **f32)
        k0, p1 = torch.zeros(R, **i32), torch.ones(R, **f32)
        seed, noise, offs = torch.zeros(R, **i64), torch.arange(R, **i32), torch.zeros(R, **i64)
        hist = torch.randint(V, (R, 2048), generator=g, device=dev)
        pres = ops.presence_set(hist, torch.zeros(R, ops.presence_words(V), **i32), V, clear=True)
        off, zero_p, one = torch.zeros(R, **f32), torch.zeros(R, **f32), torch.ones(R, **f32)
        mn, emitted = torch.zeros(R, **i32), torch.zeros(R, **i32)
        arms = {
            "sample_tokens_slots": lambda: ops.sample_tokens_slots(x, temp, k50, p09, seed, noise, offs),
            "processed_identity": lambda: ops.sample_tokens_processed(x, temp, k50, p09, zero_p, seed, one, mn, pres, offs, emitted,
                                                                      noise_rows=noise),
            "processed_penalty_1.1": lambda: ops.sample_tokens_processed(x, temp, k50, p09, zero_p, seed, one * 1.1, mn, pres, offs,
                                                                         emitted, noise_rows=noise),
            "processed_min_p_0.05_top_k_0": lambda: ops.sample_tokens_processed(x, temp, k0, p1, off + 0.05, seed, one, mn, pres,
                                                                                offs, emitted, noise_rows=noise),
        }
        for fn in arms.values():                                    # warm-up
            fn()
        torch.cuda.synchronize()
        ms = {name: [] for name in arms}
        for _ in range(rounds):
            for name, fn in arms.items():
                ms[name].append(_time(fn, iters))
        floor_ms = R * V * 2 / HBM_BPS * 1e3
        row = {"R": R, "hbm_floor_ms": round(floor_ms, 4)}
        for name, t in ms.items():
            best = min(t)
            row[name] = {"ms": round(best, 4), "floor_share": round(floor_ms / best, 3)}
        rows.append(row)
    return rows


def bench_presence(ops, dev, iters):
    out = {}
    for R in (64, 1024):
        ids = torch.randint(V, (R, 1), device=dev)
        bm = torch.zeros(R, ops.presence_words(V), dtype=torch.int32, device=dev)
        ops.presence_set(ids, bm, V)
        torch.cuda.synchronize()
        out[str(R)] = round(min(_time(lambda: ops.presence_set(ids, bm, V), iters) for _ in range(3)) * 1e3, 2)
    return {"us_per_call": out}


def bench_generate(model, Vm, dev, iters=3):
    from aria_b200.modeling_aria import GraphedDecode
    out = {}
    for B, T, n in ((1, 16, 128), (32, 2048, 64)):
        row = {}
        for name, proc in (("plain", None), ("repetition_penalty_1.1", (1.1, 0.0, 0))):
            model._decode_graph = None
            torch.cuda.empty_cache()
            g = GraphedDecode(model, B, -(-(T + n) // 256) * 256, n, (0.0, 0, 1.0, 0), (), 0, processors=proc)
            for t in g.cache.k + g.cache.v:
                t.normal_()
            gen = torch.Generator(device=dev).manual_seed(5)
            prompt = torch.randint(10, Vm, (B, T), generator=gen, device=dev)
            g.state.ids_in.copy_(prompt[:, -1:])

            def replays():
                g.start(T, None)
                if proc is not None:
                    g.start_presence(prompt)
                g.sample_and_advance(g.logits[:, -1])
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(n - 1):
                    g.graph.replay()
                b.record()
                b.synchronize()
                return a.elapsed_time(b) / (n - 1)

            replays()
            row[name] = round(min(replays() for _ in range(iters)), 4)
            del g
        out[f"B{B}_T{T}_ms_per_step"] = row
    model._decode_graph = None
    torch.cuda.empty_cache()
    return out


def _run_trace(model, trace, proc):
    from aria_b200.serving import Engine
    eng = Engine(model, max_batch=64, max_kv_tokens=65536, poll_every=8)
    t0 = time.perf_counter()
    rids = {eng.add_request(r["ids"], r["pv"], max_new_tokens=r["new"], do_sample=True, temperature=1.0, top_k=50, seed=i,
                            **proc): r for i, r in enumerate(trace)}
    eng.run()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    ttft = sorted(eng.times[rid][0] - t0 for rid in rids)
    tpot = sorted((eng.times[rid][1] - eng.times[rid][0]) / (r["new"] - 1) for rid, r in rids.items() if r["new"] > 1)
    res = {"generated_tokens_per_s": round(sum(r["new"] for r in trace) / wall, 1),
           "ttft_p50_s": round(ttft[len(ttft) // 2], 3), "tpot_p50_ms": round(tpot[len(tpot) // 2] * 1e3, 3)}
    del eng
    torch.cuda.empty_cache()
    return res


def bench_serving_trace(model, cfg, n):
    from bench_serving import make_trace
    trace = make_trace(cfg, n, 0)
    arms = {"plain": {}, "repetition_penalty_1.05_min_p_0.05": dict(repetition_penalty=1.05, min_p=0.05)}
    for proc in arms.values():                                   # warm-up: graphs of both kinds, the ViT
        _run_trace(model, trace[:8], proc)
    out = {}
    for _ in range(2):                                           # alternated, two rounds
        for name, proc in arms.items():
            out.setdefault(name, []).append(_run_trace(model, trace, proc))
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
        raise SystemExit("bench_logits_processors.py needs a GPU")
    dev = "cuda:0"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    result = {"bench": "logits_processors", "V": V, "card": card, "sampler": bench_sampler(ops, dev, args.iters),
              "presence_set": bench_presence(ops, dev, args.iters)}
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
            result[f"serving_trace_{args.requests}_at_t0"] = bench_serving_trace(model, cfg, args.requests)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
