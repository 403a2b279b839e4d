"""Generation throughput of AriaForConditionalGeneration.generate() on one GPU; prints one JSON line.

    python bench_generate.py [--runs 5] [--warmup 2] [--workload all|gptfast|b32]

Workloads (full-width Aria, random init with seed 0 — no checkpoint is needed to time the kernels):
  gptfast  gpt-fast's protocol (gptfast/benchmark.py): batch 1, one 980 px image (256 image tokens) + 32 text tokens,
           200 new tokens sampled with top_k=200, temperature=0.8, no EOS.  tokens/s = 200 / wall time of the whole
           generate() call (ViT, projector and prefill included, device synchronised at the end); `--warmup` untimed calls,
           then `--runs` timed ones.  Comparison arm: the per-token eager loop generate() used to be (one forward() per
           token, greedy), alternating with greedy generate() on the same model; both arms' tokens must be identical.
  b32      decode at batch 32 from 2048-token text prompts, 64 new tokens (greedy).  The cache rows of the prompts hold
           random values: the 65536-token prefill is not what is measured here.
For each: ms per decode step (CUDA events around the replays of the captured step) and the bytes one step must move,
computed from the shapes: the weights of the experts hit (64 * (1 - (1 - 6/64)^B) per layer), attention, shared-expert and
router weights, the KV rows read, and the lm_head.  `hbm_floor_fraction` = (bytes / 3.35 TB/s, the H100 SXM data-sheet
bandwidth) / measured step time.
"""
import argparse
import json
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


def eager_greedy(model, input_ids, pixel_values, max_new_tokens):
    """The per-token loop generate() used to run: prepare_inputs_for_generation + torch.cat + one eager forward() per token."""
    B, T = input_ids.shape
    inputs = model.prepare_inputs_for_generation(input_ids, None, pixel_values=pixel_values, num_logits_to_keep=1)
    out = model.forward(**inputs, max_cache_len=T + max_new_tokens)
    cache = out.past_key_values
    tokens = [out.logits[:, -1].float().argmax(-1)]
    all_ids = input_ids.to(tokens[0].device)
    for _ in range(max_new_tokens - 1):
        all_ids = torch.cat([all_ids, tokens[-1].view(B, 1)], dim=1)
        inputs = model.prepare_inputs_for_generation(all_ids, cache, num_logits_to_keep=1)
        tokens.append(model.forward(**inputs).logits[:, -1].float().argmax(-1))
    return torch.cat([input_ids.to(tokens[0].device), torch.stack(tokens, 1)], dim=1)


def step_bytes(tc, B, ctx):
    """HBM bytes of one decode step at batch B with `ctx` cached keys per row (bf16 everywhere)."""
    d, E, k, I = tc.hidden_size, tc.moe_num_experts, tc.moe_topk, tc.moe_intermediate_size
    Is = I * tc.moe_num_shared_experts
    hit = E * (1 - (1 - k / E) ** B)
    per_layer = (4 * d * d + 3 * d * Is + E * d + hit * 3 * d * I) * 2 + B * 2 * d * ctx * 2
    return tc.num_hidden_layers * per_layer + tc.vocab_size * d * 2


def timed_replays(g, T, n):
    """ms per replay of the captured decode step over n steps from a prompt of T cached rows."""
    g.start(T, None)
    g.sample_and_advance(g.logits[:, -1])
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        g.graph.replay()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / n


def decode_report(tc, B, T, n, ms):
    ctx = T + (n + 1) / 2                       # mean number of keys a step reads
    nbytes = step_bytes(tc, B, ctx)
    floor_ms = nbytes / (HBM_GBS * 1e9) * 1e3
    return {"ms_per_decode_step": round(ms, 4), "bytes_per_step": int(nbytes), "hbm_floor_ms": round(floor_ms, 4),
            "hbm_floor_fraction": round(floor_ms / ms, 4)}


def run_gptfast(model, cfg, args, dev):
    g = torch.Generator().manual_seed(1234)
    pv = torch.randn(1, 3, 980, 980, generator=g).bfloat16()
    text = torch.randint(10, cfg["text_config"]["vocab_size"], (32,), generator=g)
    ids = torch.cat([text[:16], torch.full((256,), cfg["image_token_index"]), text[16:]])[None]
    n = 200
    kw = dict(max_new_tokens=n, do_sample=True, top_k=200, temperature=0.8, seed=0)

    def wall(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, out

    for _ in range(args.warmup):
        model.generate(ids, pv, None, **kw)
    sampled = [wall(lambda: model.generate(ids, pv, None, **kw))[0] for _ in range(args.runs)]
    ms_step = timed_replays(model._decode_graph, ids.shape[1], n - 1)
    # comparison arm: the eager per-token loop against greedy generate(), alternating
    greedy_t, eager_t, same = [], [], True
    model.generate(ids, pv, None, max_new_tokens=n)
    eager_greedy(model, ids, pv, n)
    for _ in range(args.runs):
        tg, a = wall(lambda: model.generate(ids, pv, None, max_new_tokens=n))
        te, b = wall(lambda: eager_greedy(model, ids, pv, n))
        greedy_t.append(tg)
        eager_t.append(te)
        same = same and torch.equal(a, b)
    ms_greedy_step = timed_replays(model._decode_graph, ids.shape[1], n - 1)
    med = lambda xs: sorted(xs)[len(xs) // 2]
    tc = model.config.text_config
    return {
        "protocol": "batch 1, one 980 px image (256 image tokens) + 32 text tokens, 200 new tokens, top_k=200, "
                    "temperature=0.8, no EOS; wall time of generate() incl. ViT + prefill, median of runs",
        "tokens_per_s": round(n / med(sampled), 2), "wall_s_runs": [round(x, 4) for x in sampled],
        "decode": decode_report(tc, 1, ids.shape[1], n - 1, ms_step),
        "comparison_greedy": {"graph_generate_tokens_per_s": round(n / med(greedy_t), 2),
                              "eager_loop_tokens_per_s": round(n / med(eager_t), 2),
                              "speedup": round(med(eager_t) / med(greedy_t), 3), "tokens_identical": bool(same),
                              "graph_decode": decode_report(tc, 1, ids.shape[1], n - 1, ms_greedy_step)},
    }


def run_b32(model, cfg, args, dev):
    from aria_b200.modeling_aria import GraphedDecode
    B, T, n = 32, 2048, 64
    model._decode_graph = None
    torch.cuda.empty_cache()
    T_max = -(-(T + n) // 256) * 256
    g = GraphedDecode(model, B, T_max, n, (0.0, 0, 1.0, 0), (), 0)
    for t in g.cache.k + g.cache.v:
        t.normal_()
    gen = torch.Generator(device=dev).manual_seed(5)
    g.ids.copy_(torch.randint(10, cfg["text_config"]["vocab_size"], (B, 1), generator=gen, device=dev))
    timed_replays(g, T, n - 1)                  # warm
    ms = sorted(timed_replays(g, T, n - 1) for _ in range(args.runs))[args.runs // 2]
    return {"protocol": "batch 32, 2048-token text prompts (cache rows random), 64 new tokens, greedy; median of runs",
            "tokens_per_s": round(B * 1e3 / ms, 1), "decode": decode_report(model.config.text_config, B, T, n - 1, ms)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--workload", choices=["all", "gptfast", "b32"], default="all")
    args = ap.parse_args()
    from aria_b200 import configs as C
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration, init_random_
    dev = "cuda:0"
    cfg = C.ARIA_25B
    model = AriaForConditionalGeneration(AriaConfig.from_dict(cfg), device=dev)
    init_random_(model, seed=0)
    name, power = gpu_info(0)
    out = {"bench": "generate", "gpu": name, "power_limit_w": power, "dtype": "bf16", "model": "Aria 25.3B, random init (seed 0)",
           "hbm_floor_source": f"{HBM_GBS} GB/s, H100 SXM data sheet", "workloads": {},
           "reference_published": {"tokens_per_s": 130.0, "eager_tokens_per_s": 25.2,
                                   "source": "gpt-fast README (torch.compile); its GPU, power limit and prompt are not ours"}}
    with torch.no_grad():
        if args.workload in ("all", "gptfast"):
            out["workloads"]["gptfast"] = run_gptfast(model, cfg, args, dev)
        if args.workload in ("all", "b32"):
            out["workloads"]["b32"] = run_b32(model, cfg, args, dev)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
