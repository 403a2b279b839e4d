"""FP8 KV pages in the serving engine (Engine(kv_cache_dtype="fp8")) against bf16 pages on one GPU; prints one JSON line.

    python bench_serving_fp8.py [--requests 256] [--pool-requests 128] [--lm-layers 16] [--decode-lm-layers 4]

Model: full-width Aria (hidden 2560, 20 heads, 64 experts, the 27-layer ViT) with random weights (seed 0) and --lm-layers of the
28 LM layers, as bench_serving.py builds it.
  1. decode_kernels: the paged fp8 decode against the paged bf16 one and the contiguous devlen fp8 one at (R 32, 2K keys) and
     (R 64, 8K keys), 20 heads: ms per call (CUDA events over 200 calls, the three kernels alternated in 3 rounds), the HBM
     floor (code + scale bytes, or bf16 K + V bytes, / 3.35 TB/s, the H100 SXM data sheet), and bit identity of the paged fp8
     output to devlen fp8 on the same codes and scales, checked in the same run.
  2. engine_decode: ms per captured decode step with 64 active slots at 2K and 8K contexts, bf16 and fp8 pages, on a model with
     --decode-lm-layers LM layers (64 x 8K bf16 tokens of 16 layers would not fit the card).
  3. traces, each with three arms: bf16 pages at 65,536 tokens; fp8 pages at the same pool bytes (126,976 tokens); fp8 pages at
     65,536 tokens.  "serving": bench_serving.py's trace (--requests, 64-2048-token prompts, a quarter with an image), all at
     t = 0.  "pool_bound": --pool-requests text prompts of 4K-16K tokens (log-uniform), 64-256 new tokens, all at t = 0.  Per
     arm: generated tokens/s, TTFT and TPOT p50 / p99, peak GiB, mean slot occupancy (bench_serving.run_engine's definitions).
  4. admission: the step() that prefills one 256-token suffix after a cached 2K or 16K prefix (median of 5), bf16 against fp8
     pages: the price of dequantizing the prefix pages into the bf16 scratch.
The card name and power limit are read in the same call.
"""
import argparse
import contextlib
import json
import math
import random
import statistics
import time

import torch

import bench_serving as BS

PAGE = 256
H = 20


def _events_ms(fn, runs):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(runs):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / runs


def decode_kernels(runs=200):
    from aria_b200 import ops
    out = {}
    for R, T in ((32, 2048), (64, 8192)):
        g = torch.Generator(device="cuda").manual_seed(R)
        n_pg = T // PAGE
        src = torch.randn(2, R, H, T, 128, generator=g, device="cuda").bfloat16()
        kc = torch.empty(R, H, T, 128, dtype=torch.float8_e4m3fn, device="cuda")
        vc = torch.empty_like(kc)
        ksc, vsc = torch.empty(R, H, T, device="cuda"), torch.empty(R, H, T, device="cuda")
        ops.kv_store_fp8(src[0], src[1], kc, vc, ksc, vsc, 0)
        # pools of R * n_pg pages (+ the null page) in a shuffled order
        perm = torch.randperm(R * n_pg, generator=torch.Generator().manual_seed(1)) + 1
        table = perm.view(R, n_pg).to(torch.int32).cuda()
        n_pages = R * n_pg + 1
        kp8 = torch.zeros(n_pages, H, PAGE, 128, dtype=torch.float8_e4m3fn, device="cuda")
        vp8 = torch.zeros_like(kp8)
        ks, vs = torch.ones(n_pages, H, PAGE, device="cuda"), torch.ones(n_pages, H, PAGE, device="cuda")
        idx = table.long().flatten()
        kp8.view(torch.uint8)[idx] = kc.view(torch.uint8).view(R, H, n_pg, PAGE, 128).transpose(1, 2).reshape(-1, H, PAGE, 128)
        vp8.view(torch.uint8)[idx] = vc.view(torch.uint8).view(R, H, n_pg, PAGE, 128).transpose(1, 2).reshape(-1, H, PAGE, 128)
        ks[idx] = ksc.view(R, H, n_pg, PAGE).transpose(1, 2).reshape(-1, H, PAGE)
        vs[idx] = vsc.view(R, H, n_pg, PAGE).transpose(1, 2).reshape(-1, H, PAGE)
        kpb = torch.zeros(n_pages, H, PAGE, 128, dtype=torch.bfloat16, device="cuda")
        vpb = torch.zeros_like(kpb)
        kpb[idx] = src[0].view(R, H, n_pg, PAGE, 128).transpose(1, 2).reshape(-1, H, PAGE, 128)
        vpb[idx] = src[1].view(R, H, n_pg, PAGE, 128).transpose(1, 2).reshape(-1, H, PAGE, 128)
        del src
        q = torch.randn(R, H, 128, generator=g, device="cuda").bfloat16()
        lens = torch.full((R,), T, dtype=torch.int32, device="cuda")
        sc = 128 ** -0.5
        arms = {"paged_fp8": lambda: ops.attention_decode_paged(q, kp8, vp8, table, lens, sc, k_scale=ks, v_scale=vs),
                "paged_bf16": lambda: ops.attention_decode_paged(q, kpb, vpb, table, lens, sc),
                "devlen_fp8": lambda: ops.attention_decode_devlen(q, kc, vc, lens, sc, k_scale=ksc, v_scale=vsc)}
        identical = torch.equal(arms["paged_fp8"](), arms["devlen_fp8"]())
        times = {k: [] for k in arms}
        for _ in range(3):
            for k, fn in arms.items():
                times[k].append(round(_events_ms(fn, runs), 4))
        fp8_bytes = 2 * R * H * T * (128 + 4)
        bf16_bytes = 2 * R * H * T * 128 * 2
        out[f"R{R}_T{T}"] = {
            "ms_rounds": times, "ms_min": {k: min(v) for k, v in times.items()},
            "hbm_floor_ms": {"fp8": round(fp8_bytes / BS.HBM_GBS / 1e6, 4), "bf16": round(bf16_bytes / BS.HBM_GBS / 1e6, 4)},
            "paged_fp8_bit_identical_to_devlen_fp8": identical}
        del kc, vc, kp8, vp8, kpb, vpb
        torch.cuda.empty_cache()
    return out


def _model(layers):
    from aria_b200 import configs as C
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration, init_random_
    cfg = C.with_layers(C.ARIA_25B, lm_layers=layers)
    model = AriaForConditionalGeneration(AriaConfig.from_dict(cfg), device="cuda:0")
    init_random_(model, seed=0)
    return model, cfg


def engine_decode(model, cfg, steps=64):
    from aria_b200.serving import Engine, _pow2_at_least
    V = cfg["text_config"]["vocab_size"]
    out = {}
    for ctx in (2048, 8192):
        for dt in ("bf16", "fp8"):
            eng = Engine(model, max_batch=64, max_kv_tokens=64 * (ctx + 4 * steps + PAGE), poll_every=1,
                         max_prefill_tokens=16384, kv_cache_dtype=dt)
            g = torch.Generator().manual_seed(ctx)
            for _ in range(64):
                eng.add_request(torch.randint(10, V, (ctx,), generator=g), max_new_tokens=4 * steps)
            while eng.n_waiting or eng.sched.partial is not None:
                eng.step()
            graph = eng._graph(_pow2_at_least(eng.sched.n_active, eng.max_batch), _pow2_at_least(eng.sched.width(), eng.max_pages))
            ms = _events_ms(graph.replay, steps)
            out[f"ctx{ctx}_{dt}"] = round(ms, 3)
            del eng, graph
            torch.cuda.empty_cache()
    return out


def pool_trace(cfg, n, seed=1):
    rng = random.Random(seed)
    g = torch.Generator().manual_seed(seed)
    V = cfg["text_config"]["vocab_size"]
    trace = []
    for _ in range(n):
        T = int(round(math.exp(rng.uniform(math.log(4096), math.log(16384)))))
        trace.append(dict(ids=torch.randint(10, V, (T,), generator=g), pv=None, new=rng.randint(64, 256)))
    return trace


@contextlib.contextmanager
def _kv_dtype(dt):
    """bench_serving.run_engine builds its Engine from aria_b200.serving at call time: give it kv_cache_dtype=dt."""
    from aria_b200 import serving
    orig = serving.Engine

    class Engine(orig):
        def __init__(self, *a, **kw):
            super().__init__(*a, kv_cache_dtype=dt, **kw)

    serving.Engine = Engine
    try:
        yield
    finally:
        serving.Engine = orig


def traces(model, cfg, args):
    same_bytes = 65536 * 256 // 132 // PAGE * PAGE            # fp8 pages in the bytes of 65,536 bf16 tokens: 126,976
    arms = [("bf16_65536", "bf16", 65536), (f"fp8_{same_bytes}", "fp8", same_bytes), ("fp8_65536", "fp8", 65536)]
    out = {}
    for name, trace in (("serving", BS.make_trace(cfg, args.requests, 0)), ("pool_bound", pool_trace(cfg, args.pool_requests))):
        zero = [0.0] * len(trace)
        res = {}
        for arm, dt, tokens in arms:
            a = argparse.Namespace(max_batch=64, max_kv_tokens=tokens, poll_every=8)
            with _kv_dtype(dt):
                res[arm] = BS.run_engine(model, trace, zero, a)
        out[name] = res
    return out


def admission(model, cfg, reps=5):
    from aria_b200.serving import Engine
    V = cfg["text_config"]["vocab_size"]
    out = {}
    for P in (2048, 16384):
        for dt in ("bf16", "fp8"):
            eng = Engine(model, max_batch=8, max_kv_tokens=P + 4096, poll_every=1, max_prefill_tokens=None, kv_cache_dtype=dt)
            g = torch.Generator().manual_seed(P)
            prefix = torch.randint(10, V, (P,), generator=g)
            eng.add_request(torch.cat([prefix, torch.randint(10, V, (256,), generator=g)]), max_new_tokens=1)
            eng.run()
            ms = []
            for _ in range(reps + 1):
                eng.add_request(torch.cat([prefix, torch.randint(10, V, (256,), generator=g)]), max_new_tokens=1)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                eng.step()
                torch.cuda.synchronize()
                ms.append((time.perf_counter() - t0) * 1e3)
                eng.run()
            assert eng.stats["prefix_hit_tokens"] == (reps + 1) * P
            out[f"prefix{P}_{dt}_ms"] = round(statistics.median(ms[1:]), 3)
            del eng
            torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--pool-requests", type=int, default=128)
    ap.add_argument("--lm-layers", type=int, default=16)
    ap.add_argument("--decode-lm-layers", type=int, default=4)
    ap.add_argument("--skip", default="", help="comma-separated parts to skip: kernels,engine_decode,traces,admission")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_serving_fp8.py needs a GPU")
    skip = set(filter(None, args.skip.split(",")))
    name, power = BS.gpu_info(0)
    out = {"bench": "serving_fp8", "gpu": name, "power_limit_w": power, "heads": H,
           "hbm_floor_source": f"{BS.HBM_GBS} GB/s, H100 SXM data sheet",
           "model": f"Aria full width, {args.lm_layers} of 28 LM layers, random init (seed 0); engine_decode: "
                    f"{args.decode_lm_layers} LM layers"}
    with torch.no_grad():
        if "kernels" not in skip:
            out["decode_kernels"] = decode_kernels()
        if "engine_decode" not in skip:
            model, cfg = _model(args.decode_lm_layers)
            out["engine_decode_ms_per_step_64_slots"] = engine_decode(model, cfg)
            del model
            torch.cuda.empty_cache()
        model, cfg = _model(args.lm_layers)
        if "admission" not in skip:
            out["admission_256_suffix"] = admission(model, cfg)
        if "traces" not in skip:
            out["traces"] = traces(model, cfg, args)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
