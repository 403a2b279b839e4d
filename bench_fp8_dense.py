"""W8A8 attention projections and shared experts (quantize_dense_fp8) against bf16 on one GPU; prints one JSON line.

    python bench_fp8_dense.py [--arm all|kernel|model] [--runs 3] [--warmup 2]

Arms (full-width Aria, random init with seed 0):
  kernel  each dense LM GEMM shape at 1, 32 and 768 rows: q/k/v (2560 -> 3 x 2560, RoPE + head scatter), o_proj (2560 -> 2560
          + residual), shared gate/up (2560 -> 2 x 3328, SwiGLU) and shared down (3328 -> 2560).  The bf16 `ops` call against
          the W8A8 GEMM alone and the W8A8 GEMM plus the row-quantize pass of its input, alternating in one process, each
          captured 20 times in a CUDA graph and timed over graph replays with CUDA events.  In the model the q/k/v input is quantized inside input_layernorm's kernel, so there the separate pass
          is an upper bound.  Reported: microseconds, the HBM floor (weights, scales and activations read and written once) and
          the tensor floor (989 TFLOP/s dense bf16, 1,979 dense fp8, H100 SXM data sheet).
  model   the model with W8A8 routed experts, alternating bf16 dense weights and fp8 dense weights (quantize_dense_fp8; the
          bf16 modules are kept aside and swapped back in): cfg 2 prefill (graph replay), gpt-fast protocol tokens/s and
          batch-32 decode ms per step from 2K prompts (bench_fp8.py's phase), the cfg-2 logits' rel-L2 of fp8 dense against
          bf16 dense, and memory_allocated of each model once the other's modules are freed.
"""
import argparse
import json
import time

import torch

import bench
import bench_fp8 as BF
import bench_generate as BG

HBM_GBS = BG.HBM_GBS
BF16_TFLOPS, FP8_TFLOPS = 989.0, 1979.0
D, IS = 2560, 3328
SHAPES = {"qkv": (D, D, 3), "o_proj": (D, D, 1), "gate_up": (D, IS, 2), "down": (IS, D, 1)}   # K, N per weight, weights


CALLS_PER_GRAPH = 20


def _graphed(fn):
    """CALLS_PER_GRAPH calls of fn captured in one CUDA graph: a replay times the kernels, not the Python wrappers' host
    work, which at 1 and 32 rows takes longer than the GPU does (the model's decode step is a graph replay too)."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(CALLS_PER_GRAPH):
            fn()
    return g


def _time(g, iters, store):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        g.replay()
    e.record()
    e.synchronize()
    store.append(s.elapsed_time(e) * 1e3 / (iters * CALLS_PER_GRAPH))


def _arms(ops, name, rows, dev, g):
    K, N, nw = SHAPES[name]
    x = torch.empty(rows, K, dtype=torch.bfloat16, device=dev).normal_(generator=g)
    ws = [torch.empty(N, K, dtype=torch.bfloat16, device=dev).normal_(0.0, 0.02, generator=g) for _ in range(nw)]
    qs = [ops.permute_quantize_fp8(w) for w in ws]
    xq, xs = ops.permute_quantize_fp8(x)
    if name == "qkv":
        cos, sin = ops.rope_table(torch.ones(64, device=dev), 4096)
        outs = [torch.empty(1, 20, rows, 128, dtype=torch.bfloat16, device=dev) for _ in range(3)]
        kw = dict(pos0=0, rope_mask=0b011, rope_cos=cos, rope_sin=sin)
        bf = lambda: ops.qkv_heads(x, ws, [None] * 3, outs, 128, rows, **kw)
        f8 = lambda: ops.qkv_heads_w8a8(xq, xs, [q for q, _ in qs], [s for _, s in qs], outs, 128, rows, **kw)
    elif name == "gate_up":
        bf = lambda: ops.linear_swiglu(x, ws[0], ws[1])
        f8 = lambda: ops.linear_swiglu_w8a8(xq, xs, qs[0][0], qs[0][1], qs[1][0], qs[1][1])
    else:
        res = torch.empty(rows, N, dtype=torch.bfloat16, device=dev).normal_(generator=g) if name == "o_proj" else None
        bf = lambda: ops.linear(x, ws[0], residual=res)
        f8 = lambda: ops.linear_w8a8(xq, xs, qs[0][0], qs[0][1], residual=res)

    def f8q():
        ops.permute_quantize_fp8(x)
        f8()

    out_cols = N if name == "gate_up" else N * nw
    act_out = rows * out_cols * 2 + (rows * N * 2 if name == "o_proj" else 0)
    nbytes = {"bf16": nw * N * K * 2 + rows * K * 2 + act_out,
              "w8a8": nw * (N * K + N * 4) + rows * (K + 4) + act_out,
              "w8a8_plus_quant": nw * (N * K + N * 4) + rows * (K * 2 + 2 * (K + 4)) + act_out}
    flops = 2 * rows * K * N * nw
    return {"bf16": bf, "w8a8": f8, "w8a8_plus_quant": f8q}, nbytes, flops


def run_kernel_arm(args, dev):
    from aria_b200 import ops
    g = torch.Generator(device=dev).manual_seed(0)
    out = {}
    for name in SHAPES:
        for rows in (1, 32, 768):
            arms, nbytes, flops = _arms(ops, name, rows, dev, g)
            graphs = {k: _graphed(fn) for k, fn in arms.items()}
            for gr in graphs.values():
                for _ in range(args.warmup):
                    gr.replay()
            times = {k: [] for k in arms}
            for _ in range(args.runs):                   # alternate the arms
                for k, gr in graphs.items():
                    _time(gr, 10, times[k])
            res = {}
            for k in arms:
                us = BF._median(times[k])
                hbm = nbytes[k] / (HBM_GBS * 1e9) * 1e6
                tc = flops / ((BF16_TFLOPS if k == "bf16" else FP8_TFLOPS) * 1e12) * 1e6
                res[k] = {"us": round(us, 2), "us_runs": [round(x, 2) for x in times[k]], "hbm_floor_us": round(hbm, 2),
                          "tensor_floor_us": round(tc, 2), "floor_fraction": round(max(hbm, tc) / us, 4)}
            res["w8a8_speedup"] = round(res["bf16"]["us"] / res["w8a8"]["us"], 3)
            res["w8a8_plus_quant_speedup"] = round(res["bf16"]["us"] / res["w8a8_plus_quant"]["us"], 3)
            out[f"{name}_rows{rows}"] = res
            del graphs
            torch.cuda.empty_cache()
    return out


def _dense_modules(model):
    return {(i, o, n): getattr(layer.get_submodule(o), n) for i, layer in enumerate(model.language_model.model.layers)
            for o, names in model._DENSE_FP8 for n in names}


def _install(model, mods):
    layers = model.language_model.model.layers
    for (i, o, n), m in mods.items():
        setattr(layers[i].get_submodule(o), n, m)
    model._decode_graph = None                        # it holds the other modules' weight pointers


def run_model_arm(args, dev):
    from aria_b200.modeling_aria import GraphedPrefill
    w = bench.Cfg2Prefill(torch, dev, 0, 1, "")
    w.graphed = None                                  # captured on the bf16 experts; rebuilt per phase below
    w.model.quantize_experts_fp8(activations="fp8")
    torch.cuda.empty_cache()
    out = {"memory_allocated_gb_bf16_dense": BF._gb()}
    mods = {"bf16": _dense_modules(w.model)}
    # bytes a decode step no longer reads: bf16 weights minus e4m3 codes and fp32 scales
    saved = sum(m.weight.numel() * 2 - m.weight.numel() - m.weight.shape[0] * 4 for m in mods["bf16"].values())
    out["dense_bytes_saved_per_step"] = saved
    t0 = time.perf_counter()
    w.model.quantize_dense_fp8()
    torch.cuda.synchronize()
    out["quantize_dense_s"] = round(time.perf_counter() - t0, 2)
    mods["fp8"] = _dense_modules(w.model)
    ref = None
    for rnd in range(2):
        for key in ("bf16", "fp8"):
            _install(w.model, mods[key])
            torch.cuda.empty_cache()
            w.graphed = GraphedPrefill(w.model, w.ids_host, w.pv_host, num_logits_to_keep=1)
            res, logits = BF._phase(w, args, dev, fp8=True)
            res["gptfast"].pop("tokens")
            out[f"{key}_dense_round{rnd}"] = res
            if key == "bf16":
                ref = logits
            else:
                res["cfg2_logits_rel_l2_vs_bf16_dense"] = float((logits - ref).norm() / ref.norm())
                for rep in (res["gptfast"]["decode"], res["b32"]["decode"]):   # the floors with the fp8 dense bytes
                    rep["bytes_per_step"] = int(rep["bytes_per_step"] - saved)
                    rep["hbm_floor_ms"] = round(rep["bytes_per_step"] / (HBM_GBS * 1e9) * 1e3, 4)
                    rep["hbm_floor_fraction"] = round(rep["hbm_floor_ms"] / rep["ms_per_decode_step"], 4)
    w.graphed = None
    w.model._decode_graph = None                      # its KV cache is not model memory
    mods["bf16"] = None
    torch.cuda.empty_cache()
    out["memory_allocated_gb_fp8_dense"] = BF._gb()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arm", choices=["all", "kernel", "model"], default="all")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    dev = "cuda:0"
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8_dense.py measures on the GPU; none is available")
    name, power = BG.gpu_info(0)
    out = {"bench": "fp8_dense", "gpu": name, "power_limit_w": power, "sm_clock_mhz": _sm_clock(),
           "model": "Aria 25.3B, random init (seed 0), W8A8 routed experts",
           "floor_source": f"{HBM_GBS} GB/s, {BF16_TFLOPS} / {FP8_TFLOPS} TFLOP/s dense bf16 / fp8, H100 SXM data sheet",
           "runs": args.runs}
    with torch.no_grad():
        if args.arm in ("all", "kernel"):
            out["kernel"] = run_kernel_arm(args, dev)
        if args.arm in ("all", "model"):
            out["model"] = run_model_arm(args, dev)
    print(json.dumps(out), flush=True)


def _sm_clock():
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        cur, mx = (float(v) for v in r.splitlines()[0].split(","))
        return {"current": cur, "max": mx}
    except Exception:
        return None


if __name__ == "__main__":
    main()
