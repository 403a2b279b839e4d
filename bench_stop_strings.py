"""Stop strings on the GPU; prints one JSON line with the card's name and power limit, read in the same run.

    python bench_stop_strings.py [--iters 200] [--lm-layers 4] [--requests 64] [--kernel-only]

  table_build_s   host seconds of the first vocabulary-table build (stopping.vocab_table) for a byte-level BPE tokenizer of
                  100,352 ids, and of a second, cached call.
  stop_check_slots  the kernel's own time per launch: --iters ops.stop_check_slots launches captured in one CUDA graph, the
                  graph replayed and timed with CUDA events, at 1, 32, 256 and 1,024 rows, each with the same 1 or 16 strings
                  of 10 or 128 characters and no stop ids, on random 64-token histories that never stop (every row is checked).
  generate        generate()'s decode ms per step, greedy, at batch 1 from a 16-token prompt and at batch 32 from 2K-token
                  prompts, without and with stop_strings=["<|im_end|>"] (the captured step replayed, CUDA events, as
                  bench_logits_processors.py times it).
  serving_trace   bench_serving.py's trace (seeded, --requests of them) with every request at t = 0 and sampled (temperature 1,
                  top_k 50), without stops and with stop_strings=["<|im_end|>"] on every request (random weights never spell
                  it, so both arms generate the same tokens): generated tokens/s, TTFT and TPOT p50, two alternated rounds.
Model (generate, serving_trace): full-width Aria with random weights (seed 0) and --lm-layers of the 28 LM layers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tests"))
V = 100352


def bench_table():
    import stop_ref
    from aria_b200 import stopping
    tok = stop_ref.byte_level_tokenizer(V)
    t = time.perf_counter()
    table = stopping.vocab_table(tok)
    first = time.perf_counter() - t
    t = time.perf_counter()
    stopping.vocab_table(tok)
    return tok, table, {"first": round(first, 3), "cached": round(time.perf_counter() - t, 3), "bytes": int(table.data.numel())}


def bench_kernel(ops, table, dev, iters):
    from aria_b200 import stopping
    g = torch.Generator().manual_seed(0)
    vb, vo = table.device(dev)
    out = {}
    for R in (1, 32, 256, 1024):
        hist = torch.randint(300, V, (R, 64), generator=g)
        for n, chars in ((1, 10), (16, 10), (1, 128), (16, 128)):
            strings = ["".join(chr(0x4e00 + int(c)) if i % 3 == 0 else chr(97 + int(c) % 26) for i, c in
                               enumerate(torch.randint(0, 500, (chars,), generator=g))) for _ in range(n)]
            data, lens, lookback = stopping.encode_stop_set(strings)
            tail, k = stopping.prompt_tail(hist[:, :32])
            i32 = dict(dtype=torch.int32, device=dev)
            fin = torch.zeros(R, dtype=torch.uint8, device=dev)
            args = (vb, vo, data.repeat(R, 1, 1).to(dev), lens.repeat(R, 1).to(dev), torch.full((R,), lookback, **i32),
                    torch.zeros(R, 8, dtype=torch.int64, device=dev), torch.zeros(R, **i32), tail.to(dev),
                    torch.full((R,), k, **i32), hist[:, 32:].to(dev, torch.int32), torch.full((R,), 32, **i32), fin,
                    torch.zeros(R, dtype=torch.int64, device=dev), 0)
            ops.stop_check_slots(*args)
            graph = torch.cuda.CUDAGraph()
            with ops.graph_capture(graph):
                for _ in range(iters):
                    ops.stop_check_slots(*args)
            graph.replay()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            graph.replay()
            b.record()
            b.synchronize()
            assert not bool(fin.any())
            out[f"R{R}_{n}x{chars}_us"] = round(a.elapsed_time(b) / iters * 1e3, 2)
    return out


def bench_generate(model, Vm, table, dev, iters=3):
    from aria_b200.modeling_aria import GraphedDecode
    out = {}
    for B, T, n in ((1, 16, 128), (32, 2048, 64)):
        row = {}
        for rnd in range(2):                                # the arms alternated over two rounds
            for name, stop in (("plain", None), ("stop_im_end", table)):
                model._decode_graph = None
                torch.cuda.empty_cache()
                g = GraphedDecode(model, B, -(-(T + n) // 256) * 256, n, (0.0, 0, 1.0, 0), (), 0, stop=stop)
                for t in g.cache.k + g.cache.v:
                    t.normal_()
                gen = torch.Generator(device=dev).manual_seed(5)
                prompt = torch.randint(10, Vm, (B, T), generator=gen, device=dev)
                g.state.ids_in.copy_(prompt[:, -1:])

                def replays():
                    g.start(T, None)
                    if stop is not None:
                        g.start_stops(["<|im_end|>"], prompt.cpu())
                    g.sample_and_advance(g.logits[:, -1])
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    for _ in range(n - 1):
                        g.graph.replay()
                    b.record()
                    b.synchronize()
                    return a.elapsed_time(b) / (n - 1)

                replays()
                ms = min(replays() for _ in range(iters))
                row[name] = round(min(ms, row.get(name, ms)), 4)
                del g
        out[f"B{B}_T{T}_ms_per_step"] = row
    model._decode_graph = None
    torch.cuda.empty_cache()
    return out


def _run_trace(model, trace, tok, stops):
    from aria_b200.serving import Engine
    eng = Engine(model, max_batch=64, max_kv_tokens=65536, poll_every=8, tokenizer=tok)
    t0 = time.perf_counter()
    rids = {eng.add_request(r["ids"], r["pv"], max_new_tokens=r["new"], do_sample=True, temperature=1.0, top_k=50, seed=i,
                            **stops): r for i, r in enumerate(trace)}
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


def bench_serving_trace(model, cfg, tok, n):
    from bench_serving import make_trace
    trace = make_trace(cfg, n, 0)
    arms = {"plain": {}, "stop_im_end": dict(stop_strings=["<|im_end|>"])}
    for stops in arms.values():                                  # warm-up: graphs of both kinds, the ViT
        _run_trace(model, trace[:8], tok, stops)
    out = {}
    for _ in range(2):                                           # alternated, two rounds
        for name, stops in arms.items():
            out.setdefault(name, []).append(_run_trace(model, trace, tok, stops))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--lm-layers", type=int, default=4)
    ap.add_argument("--requests", type=int, default=64)
    ap.add_argument("--kernel-only", action="store_true")
    args = ap.parse_args()
    from aria_b200 import ops
    if not torch.cuda.is_available():
        raise SystemExit("bench_stop_strings.py needs a GPU")
    dev = "cuda:0"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    tok, table, build = bench_table()
    result = {"bench": "stop_strings", "V": V, "card": card, "table_build_s": build,
              "stop_check_slots": bench_kernel(ops, table, dev, args.iters)}
    if not args.kernel_only:
        from aria_b200 import configs as C
        from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration, init_random_
        cfg = C.with_layers(C.ARIA_25B, lm_layers=args.lm_layers)
        result["model"] = f"Aria full width, {args.lm_layers} of 28 LM layers, random init (seed 0)"
        with torch.no_grad():
            model = AriaForConditionalGeneration(AriaConfig.from_dict(cfg), device=dev)
            init_random_(model, seed=0)
            result["generate"] = bench_generate(model, cfg["text_config"]["vocab_size"], table, dev)
            result[f"serving_trace_{args.requests}_at_t0"] = bench_serving_trace(model, cfg, tok, args.requests)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
