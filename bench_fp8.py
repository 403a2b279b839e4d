"""FP8 expert weights against bf16 on one GPU; prints one JSON line.

    python bench_fp8.py [--arm all|kernel|model|long] [--runs 5] [--warmup 2]

Arms (full-width Aria, random init with seed 0; inputs and seeds are bench.py's and bench_generate.py's):
  kernel  the routed-expert GEMMs alone: fc1 + SwiGLU (2560 -> 2 x 1664) and fc2 (1664 -> 2560), bf16 weights and e4m3
          weights timed alternately in one process with CUDA events, at four row distributions over the 64 experts: decode
          B = 1 (6 groups x 1 row), B = 32 (192 rows), cfg 2 (4608 rows) and cfg 4 (196,608 rows).  Reported: microseconds and
          the weight bytes of the experts hit over time, against the 3.35 TB/s HBM floor (H100 SXM data sheet).
  model   bench.py's cfg 2 prefill (one 980 px image + 512 text tokens, CUDA-graph replay; GraphedPrefill rebuilt after
          quantizing), bench_generate.py's gpt-fast protocol (tokens/s of sampled generate()) and its batch-32 decode from
          2048-token prompts (ms per step): bf16 first, then quantize_experts_fp8(), then again.  Also memory_allocated after
          each phase and the rel-L2 of the fp8 cfg-2 logits against the bf16 ones.
  long    fp8 only (the bf16 model leaves too little room): one 65,536-token prefill (16 frames = 4096 image tokens + 61,440
          text tokens, num_logits_to_keep = 1): ms and max_memory_allocated.
The model and long arms share one model: with --arm all the long arm runs on the model arm's quantized model.
"""
import argparse
import json
import time

import torch

import bench
import bench_generate as BG

HBM_GBS = BG.HBM_GBS
E, D, I = 64, 2560, 1664


def _median(xs):
    return sorted(xs)[len(xs) // 2]


def expert_bytes(hit, fp8):
    """HBM bytes of the fc1 + fc2 weights of `hit` experts (plus their scales in fp8)."""
    n = hit * (D * 2 * I + I * D)
    return n * 1 + hit * (2 * I + D) * 4 if fp8 else n * 2


# ------------------------------------------------------------------------------------------------ kernel arm
def _row_counts(name):
    g = torch.Generator().manual_seed(0)
    if name == "decode_b1":
        counts = torch.zeros(E, dtype=torch.int64)
        counts[torch.randperm(E, generator=g)[:6]] = 1
        return counts
    rows = {"b32": 192, "cfg2": 4608, "cfg4": 196608}[name]
    return torch.bincount(torch.randint(0, E, (rows,), generator=g), minlength=E)


def run_kernel_arm(args, dev):
    from aria_b200 import ops
    g = torch.Generator(device=dev).manual_seed(0)
    w1 = torch.empty(E, D, 2 * I, dtype=torch.bfloat16, device=dev).normal_(0.0, 0.02, generator=g)
    w2 = torch.empty(E, I, D, dtype=torch.bfloat16, device=dev).normal_(0.0, 0.02, generator=g)
    q1, s1 = ops.quantize_fp8_cols(w1)
    q2, s2 = ops.quantize_fp8_cols(w2)
    out = {}
    for name in ("decode_b1", "b32", "cfg2", "cfg4"):
        counts = _row_counts(name)
        rows = int(counts.sum())
        off = torch.zeros(E + 1, dtype=torch.int32)
        off[1:] = counts.cumsum(0).to(torch.int32)
        off = off.to(dev)
        a = torch.empty(rows, D, dtype=torch.bfloat16, device=dev).normal_(generator=g)
        hit = int((counts > 0).sum())
        arms = {"bf16": lambda: ops.grouped_gemm(ops.grouped_gemm(a, w1, off, swiglu=True), w2, off),
                "fp8": lambda: ops.grouped_gemm_fp8(ops.grouped_gemm_fp8(a, q1, s1, off, swiglu=True), q2, s2, off)}
        iters = 3 if name == "cfg4" else 50
        for fn in arms.values():                     # warm-up of both arms
            for _ in range(args.warmup):
                fn()
        times = {k: [] for k in arms}
        for _ in range(args.runs):                   # alternate the arms
            for k, fn in arms.items():
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(iters):
                    fn()
                e.record()
                e.synchronize()
                times[k].append(s.elapsed_time(e) * 1e3 / iters)
        res = {"rows": rows, "experts_hit": hit}
        for k in arms:
            us = _median(times[k])
            nbytes = expert_bytes(hit, k == "fp8")
            floor_us = nbytes / (HBM_GBS * 1e9) * 1e6
            res[k] = {"us_fc1_fc2": round(us, 2), "us_runs": [round(x, 2) for x in times[k]], "weight_bytes": nbytes,
                      "weight_tb_per_s": round(nbytes / us / 1e6, 3), "hbm_floor_us": round(floor_us, 2),
                      "hbm_floor_fraction": round(floor_us / us, 4)}
        res["fp8_speedup"] = round(res["bf16"]["us_fc1_fc2"] / res["fp8"]["us_fc1_fc2"], 3)
        out[name] = res
        del a
    del w1, w2, q1, q2, s1, s2
    torch.cuda.empty_cache()
    return out


# ------------------------------------------------------------------------------------------------ model arm
def _gb():
    return round(torch.cuda.memory_allocated() / 1e9, 3)


def _decode_floor(tc, B, T, n, ms, fp8):
    """bench_generate.decode_report with the routed-expert bytes of the weight format in use."""
    rep = BG.decode_report(tc, B, T, n, ms)
    if fp8:
        hit = E * (1 - (1 - tc.moe_topk / E) ** B)
        nbytes = rep["bytes_per_step"] - tc.num_hidden_layers * (expert_bytes(hit, False) - expert_bytes(hit, True))
        floor_ms = nbytes / (HBM_GBS * 1e9) * 1e3
        rep.update(bytes_per_step=int(nbytes), hbm_floor_ms=round(floor_ms, 4), hbm_floor_fraction=round(floor_ms / ms, 4))
    return rep


def _phase(w, args, dev, fp8):
    model = w.model
    res = {}
    # cfg 2 prefill, graph replay
    for _ in range(args.warmup):
        w.step_resident()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(args.runs):
        s.record()
        for _ in range(5):
            last = w.step_resident()
        e.record()
        e.synchronize()
        times.append(s.elapsed_time(e) / 5)
    res["cfg2_prefill_ms"] = round(_median(times), 3)
    res["cfg2_prefill_ms_runs"] = [round(x, 3) for x in times]
    logits = last.float().cpu()
    w.graphed = None                                 # free the prefill graph's pool before the decode graphs
    torch.cuda.empty_cache()
    # gpt-fast protocol: sampled generate(), wall time incl. ViT + prefill
    from aria_b200 import configs as C
    gcfg = C.ARIA_25B
    g = torch.Generator().manual_seed(1234)
    pv = torch.randn(1, 3, 980, 980, generator=g).bfloat16()
    text = torch.randint(10, gcfg["text_config"]["vocab_size"], (32,), generator=g)
    ids = torch.cat([text[:16], torch.full((256,), gcfg["image_token_index"]), text[16:]])[None]
    n = 200
    kw = dict(max_new_tokens=n, do_sample=True, top_k=200, temperature=0.8, seed=0)
    for _ in range(args.warmup):
        model.generate(ids, pv, None, **kw)
    walls = []
    for _ in range(args.runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        toks = model.generate(ids, pv, None, **kw)
        torch.cuda.synchronize()
        walls.append(time.perf_counter() - t0)
    tc = model.config.text_config
    ms_step = BG.timed_replays(model._decode_graph, ids.shape[1], n - 1)
    res["gptfast"] = {"tokens_per_s": round(n / _median(walls), 2), "wall_s_runs": [round(x, 4) for x in walls],
                      "decode": _decode_floor(tc, 1, ids.shape[1], n - 1, ms_step, fp8), "tokens": toks[0, -n:].tolist()}
    # batch 32 from 2048-token prompts
    b32 = BG.run_b32(model, gcfg, args, dev)
    ms = b32["decode"]["ms_per_decode_step"]
    res["b32"] = {"tokens_per_s": b32["tokens_per_s"], "decode": _decode_floor(tc, 32, 2048, 63, ms, fp8)}
    model._decode_graph = None
    torch.cuda.empty_cache()
    res["memory_allocated_gb"] = _gb()
    return res, logits


def run_model_arm(args, dev):
    from aria_b200.modeling_aria import GraphedPrefill
    w = bench.Cfg2Prefill(torch, dev, 0, 1, "")
    out = {"memory_allocated_gb_bf16_model": _gb()}
    out["bf16"], ref = _phase(w, args, dev, fp8=False)
    t0 = time.perf_counter()
    w.model.quantize_experts_fp8()
    torch.cuda.synchronize()
    out["quantize_s"] = round(time.perf_counter() - t0, 2)
    torch.cuda.empty_cache()
    out["memory_allocated_gb_fp8_model"] = _gb()
    w.graphed = GraphedPrefill(w.model, w.ids_host, w.pv_host, num_logits_to_keep=1)
    out["fp8"], got = _phase(w, args, dev, fp8=True)
    out["cfg2_logits_rel_l2"] = float((got - ref).norm() / ref.norm())
    same = sum(a == b for a, b in zip(out["bf16"]["gptfast"]["tokens"], out["fp8"]["gptfast"]["tokens"]))
    out["gptfast_tokens_equal_prefix"] = same
    for k in ("bf16", "fp8"):
        out[k]["gptfast"].pop("tokens")
    return out, w.model


# ------------------------------------------------------------------------------------------------ long arm
def run_long_arm(args, dev, model=None):
    from aria_b200 import configs as C
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration, init_random_
    cfg = C.ARIA_25B
    if model is None:
        model = AriaForConditionalGeneration(AriaConfig.from_dict(cfg), device=dev)
        init_random_(model, seed=0)
        model.quantize_experts_fp8()
    torch.cuda.empty_cache()
    T, frames = 65536, 16
    g = torch.Generator().manual_seed(99)           # bench.py's cfg 4 seed
    ids = torch.randint(10, cfg["text_config"]["vocab_size"], (1, T), generator=g)
    ids[0, 64:64 + 256 * frames] = cfg["image_token_index"]
    pv = torch.randn(frames, 3, 980, 980, generator=g).bfloat16().to(dev)
    ids_dev = ids.to(dev)
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    times = []
    for i in range(1 + max(1, args.runs // 2)):     # the first call is a warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        logits = model(ids_dev, pv, None, num_logits_to_keep=1, input_ids_host=ids).logits
        torch.cuda.synchronize()
        if i:
            times.append((time.perf_counter() - t0) * 1e3)
        del logits
    return {"tokens": T, "image_tokens": 256 * frames, "text_tokens": T - 256 * frames, "prefill_ms": round(_median(times), 1),
            "prefill_ms_runs": [round(x, 1) for x in times], "max_memory_allocated_gb": round(torch.cuda.max_memory_allocated() / 1e9, 3),
            "model_memory_allocated_gb": round(base / 1e9, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arm", choices=["all", "kernel", "model", "long"], default="all")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    dev = "cuda:0"
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8.py measures on the GPU; none is available")
    name, power = BG.gpu_info(0)
    out = {"bench": "fp8_experts", "gpu": name, "power_limit_w": power, "model": "Aria 25.3B, random init (seed 0)",
           "hbm_floor_source": f"{HBM_GBS} GB/s, H100 SXM data sheet", "runs": args.runs}
    with torch.no_grad():
        if args.arm in ("all", "kernel"):
            out["kernel"] = run_kernel_arm(args, dev)
        model = None
        if args.arm in ("all", "model"):
            out["model"], model = run_model_arm(args, dev)
        if args.arm in ("all", "long"):
            out["long_fp8"] = run_long_arm(args, dev, model)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
