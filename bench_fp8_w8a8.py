"""FP8 activations and weights (W8A8) against bf16 and weight-only fp8 (W8A16) on one GPU; prints one JSON line.

    python bench_fp8_w8a8.py [--arm all|kernel|model] [--runs 5] [--warmup 2]

Arms (full-width Aria, random init with seed 0; inputs and seeds are bench_fp8.py's):
  kernel  the routed-expert GEMMs alone, fc1 + SwiGLU (2560 -> 2 x 1664) then fc2 (1664 -> 2560), at bench_fp8.py's four row
          mixes (decode B = 1, B = 32, cfg 2 = 4608 rows, cfg 4 = 196,608 rows).  bf16, W8A16 and W8A8 alternate in one
          process, timed with CUDA events.  The W8A8 arm includes its two row-quantize passes (the gathered tokens before fc1
          and h before fc2), which are also timed alone.  Reported: microseconds, the fraction of the HBM floor (weight bytes
          of the experts hit, 1 byte per fp8 weight plus the scales, plus the activation bytes read and written) and, at
          cfg 4, the fraction of the 1,979 TFLOP/s dense fp8 data-sheet rate (H100 SXM, 700 W).
  model   bench_fp8.py's model arm with three phases: bf16, then quantize_experts_fp8() (W8A16), then a re-layout to W8A8
          (quantize_experts_fp8(activations="fp8")).  Each phase: cfg 2 prefill (graph replay), gpt-fast protocol tokens/s
          and batch-32 decode ms per step; also the cfg-2 logits' rel-L2 against bf16 and the leading gpt-fast tokens that
          match bf16.
"""
import argparse
import json
import time

import torch

import bench
import bench_fp8 as BF
import bench_generate as BG

E, D, I = BF.E, BF.D, BF.I
HBM_GBS = BG.HBM_GBS
FP8_TFLOPS = 1979.0


def _act_bytes(rows, mode):
    """Activation bytes of fc1 + SwiGLU then fc2 (and of the W8A8 row-quantize passes), read and written."""
    if mode != "w8a8":
        return rows * (D * 2 + I * 2) + rows * (I * 2 + D * 2)
    quant = rows * (D * 2 + D + 4) + rows * (I * 2 + I + 4)         # bf16 row in, e4m3 row + scale out, twice
    return quant + rows * (D + 4 + I * 2) + rows * (I + 4 + D * 2)


def _time(fn, iters, runs, store):
    for _ in range(runs):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(iters):
            fn()
        e.record()
        e.synchronize()
        store.append(s.elapsed_time(e) * 1e3 / iters)


def run_kernel_arm(args, dev):
    from aria_b200 import ops
    g = torch.Generator(device=dev).manual_seed(0)
    w1 = torch.empty(E, D, 2 * I, dtype=torch.bfloat16, device=dev).normal_(0.0, 0.02, generator=g)
    w2 = torch.empty(E, I, D, dtype=torch.bfloat16, device=dev).normal_(0.0, 0.02, generator=g)
    q1, s1 = ops.quantize_fp8_cols(w1)
    q2, s2 = ops.quantize_fp8_cols(w2)
    k1, k2 = (q.transpose(1, 2).contiguous().transpose(1, 2) for q in (q1, q2))   # the W8A8 layout of the same codes
    out = {}
    for name in ("decode_b1", "b32", "cfg2", "cfg4"):
        counts = BF._row_counts(name)
        rows = int(counts.sum())
        off = torch.zeros(E + 1, dtype=torch.int32)
        off[1:] = counts.cumsum(0).to(torch.int32)
        off = off.to(dev)
        a = torch.empty(rows, D, dtype=torch.bfloat16, device=dev).normal_(generator=g)
        h = ops.grouped_gemm(a, w1, off, swiglu=True)
        hit = int((counts > 0).sum())

        def w8a8():
            aq, as_ = ops.permute_quantize_fp8(a)
            hh = ops.grouped_gemm_w8a8(aq, as_, k1, s1, off, swiglu=True)
            hq, hs = ops.permute_quantize_fp8(hh)
            return ops.grouped_gemm_w8a8(hq, hs, k2, s2, off)

        arms = {"bf16": lambda: ops.grouped_gemm(ops.grouped_gemm(a, w1, off, swiglu=True), w2, off),
                "w8a16": lambda: ops.grouped_gemm_fp8(ops.grouped_gemm_fp8(a, q1, s1, off, swiglu=True), q2, s2, off),
                "w8a8": w8a8,
                "quant_x": lambda: ops.permute_quantize_fp8(a),
                "quant_h": lambda: ops.permute_quantize_fp8(h)}
        iters = 3 if name == "cfg4" else 50
        for fn in arms.values():
            for _ in range(args.warmup):
                fn()
        times = {k: [] for k in arms}
        for _ in range(args.runs):                   # alternate the arms
            for k, fn in arms.items():
                _time(fn, iters, 1, times[k])
        res = {"rows": rows, "experts_hit": hit}
        flops = 2 * rows * (D * 2 * I + I * D)
        for k in ("bf16", "w8a16", "w8a8"):
            us = BF._median(times[k])
            nbytes = BF.expert_bytes(hit, k != "bf16") + _act_bytes(rows, k)
            floor_us = nbytes / (HBM_GBS * 1e9) * 1e6
            res[k] = {"us_fc1_fc2": round(us, 2), "us_runs": [round(x, 2) for x in times[k]], "bytes": nbytes,
                      "hbm_floor_us": round(floor_us, 2), "hbm_floor_fraction": round(floor_us / us, 4)}
            if name == "cfg4":
                res[k]["tflops"] = round(flops / us / 1e6, 1)
                res[k]["fp8_datasheet_fraction"] = round(flops / us / 1e6 / FP8_TFLOPS, 4)
        for k in ("quant_x", "quant_h"):
            res[k + "_us"] = round(BF._median(times[k]), 2)
        res["quant_share_of_w8a8"] = round((res["quant_x_us"] + res["quant_h_us"]) / res["w8a8"]["us_fc1_fc2"], 4)
        res["w8a8_speedup_vs_bf16"] = round(res["bf16"]["us_fc1_fc2"] / res["w8a8"]["us_fc1_fc2"], 3)
        res["w8a8_speedup_vs_w8a16"] = round(res["w8a16"]["us_fc1_fc2"] / res["w8a8"]["us_fc1_fc2"], 3)
        out[name] = res
        del a, h
    del w1, w2, q1, q2, s1, s2, k1, k2
    torch.cuda.empty_cache()
    return out


def run_model_arm(args, dev):
    from aria_b200.modeling_aria import GraphedPrefill
    w = bench.Cfg2Prefill(torch, dev, 0, 1, "")
    out = {"memory_allocated_gb_bf16_model": BF._gb()}
    out["bf16"], ref = BF._phase(w, args, dev, fp8=False)
    toks = {"bf16": out["bf16"]["gptfast"].pop("tokens")}
    for mode, key in (("bf16", "w8a16"), ("fp8", "w8a8")):
        t0 = time.perf_counter()
        w.model.quantize_experts_fp8(activations=mode)
        torch.cuda.synchronize()
        out[f"quantize_s_{key}"] = round(time.perf_counter() - t0, 2)
        torch.cuda.empty_cache()
        out[f"memory_allocated_gb_{key}_model"] = BF._gb()
        w.graphed = GraphedPrefill(w.model, w.ids_host, w.pv_host, num_logits_to_keep=1)
        out[key], got = BF._phase(w, args, dev, fp8=True)
        out[key]["cfg2_logits_rel_l2_vs_bf16"] = float((got - ref).norm() / ref.norm())
        toks[key] = out[key]["gptfast"].pop("tokens")
        out[key]["gptfast_tokens_equal_prefix_vs_bf16"] = next(
            (i for i, (a, b) in enumerate(zip(toks["bf16"], toks[key])) if a != b), len(toks[key]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arm", choices=["all", "kernel", "model"], default="all")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    dev = "cuda:0"
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8_w8a8.py measures on the GPU; none is available")
    name, power = BG.gpu_info(0)
    out = {"bench": "fp8_w8a8_experts", "gpu": name, "power_limit_w": power, "model": "Aria 25.3B, random init (seed 0)",
           "hbm_floor_source": f"{HBM_GBS} GB/s, H100 SXM data sheet", "fp8_rate_source": f"{FP8_TFLOPS} TFLOP/s dense, "
           "H100 SXM data sheet", "runs": args.runs}
    with torch.no_grad():
        if args.arm in ("all", "kernel"):
            out["kernel"] = run_kernel_arm(args, dev)
        if args.arm in ("all", "model"):
            out["model"] = run_model_arm(args, dev)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
