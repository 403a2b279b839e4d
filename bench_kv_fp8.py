"""The fp8 KV cache (e4m3 keys and values, one fp32 scale per row, head and token) against the bf16 cache on one GPU; prints one
JSON line.

    python bench_kv_fp8.py [--arm all|kernel|model] [--runs 5] [--warmup 2]

Arms (H = 20 KV heads of 128 dims, Aria's LM; nothing is read from outside the repository):
  kernel  decode attention with device lengths (the kernel a captured decode step runs), bf16 and fp8 alternating in one process,
          CUDA events, at B = 32 x 2K keys, B = 32 x 8K and B = 1 x 64K.  The cache rows are random: randn cast to e4m3 with
          positive random scales.  Also kv_append_fp8 at B = 32 and kv_store_fp8 for a 2,048-token prefill.  The HBM floor of
          each counts the bytes the kernel must move: 256 bytes per key of bf16 K + V, 264 (2 x (128 + 4)) for fp8.
  model   full-width Aria, random init (seed 0):
          - batch-32 decode from 2,048-token prompts (random cache rows, as in bench_generate.py), bf16 and W8A8 experts, each
            with a bf16 and an fp8 cache; ms per step and the fraction of the step's HBM floor.  The two caches do not fit
            beside the bf16 model together, so each arm captures its own graph, one after the other.
          - W8A8 experts with an fp8 cache, batch 32 from 6,144-token prompts: ms per step and max_memory_allocated; the bytes
            the bf16 cache would need are computed, not run (it does not fit beside the model).
          - gpt-fast protocol (bench_generate.py): tokens/s with a bf16 and an fp8 cache, and how many of the 200 sampled tokens
            agree.
          - cfg-2 prefill (one image + 512 text tokens), eager forward() with a bf16 and an fp8 cache, alternating: the cost of
            quantizing the new rows into the fp8 cache.
The step-bytes formula is bench_generate.py's with the routed-expert bytes of the weight format in use and 132 bytes per 128
cached K or V values in fp8.
"""
import argparse
import json
import time

import torch

import bench_generate as BG

HBM_GBS = BG.HBM_GBS
H, HD = 20, 128


def _median(xs):
    return sorted(xs)[len(xs) // 2]


def _time_us(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) * 1e3 / iters


def _alternate(arms, iters, args):
    for fn in arms.values():
        for _ in range(args.warmup):
            fn()
    times = {k: [] for k in arms}
    for _ in range(args.runs):
        for k, fn in arms.items():
            times[k].append(_time_us(fn, iters))
    return times


def _random_fp8(shape, dev, g):
    codes = torch.randn(shape, generator=g, device=dev).to(torch.float8_e4m3fn)
    scales = torch.rand(shape[:-1], generator=g, device=dev) * 0.02 + 0.001
    return codes, scales


def _floor(nbytes, us):
    floor_us = nbytes / (HBM_GBS * 1e9) * 1e6
    return {"us": round(us, 2), "bytes": int(nbytes), "hbm_floor_us": round(floor_us, 2), "hbm_floor_fraction": round(floor_us / us, 4)}


def run_kernel_arm(args, dev):
    from aria_b200 import ops
    g = torch.Generator(device=dev).manual_seed(0)
    out = {}
    for name, B, T in (("b32_2k", 32, 2048), ("b32_8k", 32, 8192), ("b1_64k", 1, 65536)):
        q = torch.randn(B, H, HD, generator=g, device=dev).bfloat16()
        kb = torch.randn(B, H, T, HD, generator=g, device=dev).bfloat16()
        vb = torch.randn(B, H, T, HD, generator=g, device=dev).bfloat16()
        k8, ks = _random_fp8((B, H, T, HD), dev, g)
        v8, vs = _random_fp8((B, H, T, HD), dev, g)
        lens = torch.full((B,), T, dtype=torch.int32, device=dev)
        arms = {"bf16": lambda: ops.attention_decode_devlen(q, kb, vb, lens, HD ** -0.5),
                "fp8": lambda: ops.attention_decode_devlen(q, k8, v8, lens, HD ** -0.5, k_scale=ks, v_scale=vs)}
        times = _alternate(arms, 50, args)
        res = {"B": B, "keys": T, "heads": H}
        for k, per_key in (("bf16", 2 * HD * 2), ("fp8", 2 * (HD + 4))):
            res[k] = _floor(B * H * T * per_key, _median(times[k]))
            res[k]["us_runs"] = [round(x, 2) for x in times[k]]
        res["fp8_speedup"] = round(res["bf16"]["us"] / res["fp8"]["us"], 3)
        out[name] = res
        del q, kb, vb, k8, v8, ks, vs
        torch.cuda.empty_cache()
    # append at B = 32 (one row per (b, h)) and the store of a 2,048-token prefill (B = 1), one layer each
    B, T_max = 32, 2304
    kc, ks = _random_fp8((B, H, T_max, HD), dev, g)
    vc, vs = _random_fp8((B, H, T_max, HD), dev, g)
    new = torch.randn(2, B, H, 1, HD, generator=g, device=dev).bfloat16()
    pos = torch.full((B,), 2048, dtype=torch.int32, device=dev)
    rows = torch.randn(2, 1, H, 2048, HD, generator=g, device=dev).bfloat16()
    arms = {"append_b32": lambda: ops.kv_append_fp8(new[0, :, :, 0], new[1, :, :, 0], kc, vc, ks, vs, pos),
            "store_2048": lambda: ops.kv_store_fp8(rows[0], rows[1], kc[:1], vc[:1], ks[:1], vs[:1], 0)}
    times = _alternate(arms, 200, args)
    out["kv_append_fp8_b32"] = _floor(2 * B * H * (HD * 2 + HD + 4), _median(times["append_b32"]))
    out["kv_store_fp8_2048_rows"] = _floor(2 * 2048 * H * (HD * 2 + HD + 4), _median(times["store_2048"]))
    return out


def step_bytes(tc, B, ctx, w8a8, kv):
    """HBM bytes of one decode step: bench_generate.step_bytes with fp8 expert weights (1 byte + column scales) under W8A8 and
    132 bytes per 128 cached K or V values with an fp8 cache."""
    d, E, k, I = tc.hidden_size, tc.moe_num_experts, tc.moe_topk, tc.moe_intermediate_size
    nbytes = BG.step_bytes(tc, B, ctx)
    hit = E * (1 - (1 - k / E) ** B)
    if w8a8:
        nbytes -= tc.num_hidden_layers * (hit * 3 * d * I * 2 - (hit * 3 * d * I + hit * (2 * I + d) * 4))
    if kv == "fp8":
        nbytes -= tc.num_hidden_layers * (B * 2 * d * ctx * 2 - B * 2 * (d // HD) * ctx * (HD + 4))
    return nbytes


def _decode(model, B, T, n, kv, w8a8, args, dev):
    from aria_b200.modeling_aria import GraphedDecode
    model._decode_graph = None
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    T_max = -(-(T + n) // 256) * 256
    g = GraphedDecode(model, B, T_max, n, (0.0, 0, 1.0, 0), (), 0, kv)
    gen = torch.Generator(device=dev).manual_seed(5)
    c = g.cache
    if kv == "fp8":
        for t in c.k + c.v:
            t.copy_(torch.randn(t.shape, generator=gen, device=dev).to(torch.float8_e4m3fn))
        for t in c.k_scale + c.v_scale:
            t.uniform_(0.001, 0.02, generator=gen)
    else:
        for t in c.k + c.v:
            t.normal_(generator=gen)
    g.state.ids_in.copy_(torch.randint(10, model.config.text_config.vocab_size, (B, 1), generator=gen, device=dev))
    BG.timed_replays(g, T, n - 1)
    ms = _median([BG.timed_replays(g, T, n - 1) for _ in range(args.runs)])
    tc = model.config.text_config
    ctx = T + (n + 1) / 2
    nbytes = step_bytes(tc, B, ctx, w8a8, kv)
    floor_ms = nbytes / (HBM_GBS * 1e9) * 1e3
    res = {"ms_per_decode_step": round(ms, 4), "bytes_per_step": int(nbytes), "hbm_floor_ms": round(floor_ms, 4),
           "hbm_floor_fraction": round(floor_ms / ms, 4), "max_memory_allocated_gb": round(torch.cuda.max_memory_allocated() / 1e9, 2)}
    model._decode_graph = None
    del g, c
    torch.cuda.empty_cache()
    return res


def _gptfast(model, args):
    gen = torch.Generator().manual_seed(1234)
    pv = torch.randn(1, 3, 980, 980, generator=gen).bfloat16()
    text = torch.randint(10, model.config.text_config.vocab_size, (32,), generator=gen)
    ids = torch.cat([text[:16], torch.full((256,), model.config.image_token_index), text[16:]])[None]
    n = 200
    res, toks = {}, {}
    for kv in ("bf16", "fp8"):
        kw = dict(max_new_tokens=n, do_sample=True, top_k=200, temperature=0.8, seed=0, kv_cache_dtype=kv)
        for _ in range(args.warmup):
            model.generate(ids, pv, None, **kw)
        walls = []
        for _ in range(args.runs):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = model.generate(ids, pv, None, **kw)
            torch.cuda.synchronize()
            walls.append(time.perf_counter() - t0)
        toks[kv] = out[0, -n:].tolist()
        res[kv] = {"tokens_per_s": round(n / _median(walls), 2), "wall_s_runs": [round(x, 4) for x in walls]}
    res["tokens_agreeing_of_200"] = sum(a == b for a, b in zip(toks["bf16"], toks["fp8"]))
    res["leading_tokens_agreeing"] = next((i for i, (a, b) in enumerate(zip(toks["bf16"], toks["fp8"])) if a != b), n)
    model._decode_graph = None
    torch.cuda.empty_cache()
    return res


def _cfg2_prefill(model, args, dev):
    import bench
    gen = torch.Generator().manual_seed(1234)
    pv = torch.randn(1, 3, 980, 980, generator=gen).bfloat16().to(dev)
    text = torch.randint(10, model.config.text_config.vocab_size, (bench.T_TEXT,), generator=gen)
    ids_host = torch.cat([text[:16], torch.full((bench.T_IMG,), model.config.image_token_index), text[16:]])[None]
    ids = ids_host.to(dev)
    arms = {kv: (lambda kv=kv: model(ids, pv, None, num_logits_to_keep=1, input_ids_host=ids_host, kv_cache_dtype=kv))
            for kv in ("bf16", "fp8")}
    times = _alternate(arms, 3, args)
    res = {kv: {"ms": round(_median(t) / 1e3, 3), "ms_runs": [round(x / 1e3, 3) for x in t]} for kv, t in times.items()}
    res["fp8_extra_ms"] = round(res["fp8"]["ms"] - res["bf16"]["ms"], 3)
    return res


def run_model_arm(args, dev):
    from aria_b200 import configs as C
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration, init_random_
    model = AriaForConditionalGeneration(AriaConfig.from_dict(C.ARIA_25B), device=dev)
    init_random_(model, seed=0)
    tc = model.config.text_config
    out = {"cfg2_prefill_eager": _cfg2_prefill(model, args, dev), "gptfast": _gptfast(model, args),
           "b32_2k": {"bf16_experts": {kv: _decode(model, 32, 2048, 64, kv, False, args, dev) for kv in ("bf16", "fp8")}}}
    model.quantize_experts_fp8(activations="fp8")
    torch.cuda.empty_cache()
    out["b32_2k"]["w8a8_experts"] = {kv: _decode(model, 32, 2048, 64, kv, True, args, dev) for kv in ("bf16", "fp8")}
    T6 = 6144
    T_max6 = -(-(T6 + 64) // 256) * 256
    out["b32_6k_w8a8"] = {"fp8": _decode(model, 32, T6, 64, "fp8", True, args, dev),
                          "bf16_cache_gb_not_run": round(tc.num_hidden_layers * 2 * 32 * T_max6 * tc.hidden_size * 2 / 1e9, 2),
                          "fp8_cache_gb": round(tc.num_hidden_layers * 2 * 32 * T_max6 * (tc.hidden_size // HD) * (HD + 4) / 1e9, 2)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arm", choices=["all", "kernel", "model"], default="all")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kv_fp8.py measures on the GPU; none is available")
    dev = "cuda:0"
    name, power = BG.gpu_info(0)
    out = {"bench": "kv_fp8", "gpu": name, "power_limit_w": power, "hbm_floor_source": f"{HBM_GBS} GB/s, H100 SXM data sheet",
           "runs": args.runs}
    with torch.no_grad():
        if args.arm in ("all", "kernel"):
            out["kernel"] = run_kernel_arm(args, dev)
        if args.arm in ("all", "model"):
            out["model"] = run_model_arm(args, dev)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
