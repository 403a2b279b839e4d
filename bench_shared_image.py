"""Many questions about one image (generate(shared_prefix_len=P)) against generate() on the left-padded repeated-image batch;
prints one JSON line.

    python bench_shared_image.py [--runs 3] [--warmup 1]

Model: full-width Aria (25.3B), random init with seed 0; no checkpoint is needed to time the kernels.  The GPU's name, power
limit and maximum SM clock are read in the same run.  Parts:
  attention  the suffix prefill attention alone (B = 32 questions of 16-64 tokens, H = 20) against `ops.attention` on the
             expanded batch, each row's [prefix, question] layout with the questions right-padded to the longest, at
             P in {290, 1300, 2304}.  CUDA events around 20 launches, median of `--runs` alternated rounds.  flops = 4 * 128 * H
             per visible (query, key) pair of the real rows; bytes = what each kernel must read and write (the shared kernel
             reads the prefix once, the expanded one B times); floor = max(flops / 989 TFLOP/s, bytes / 3.35 TB/s), the H100
             SXM data sheet's dense BF16 rate and HBM3 bandwidth.
  generate   B in {8, 32} questions with lengths drawn from 16-64 tokens about one 980 px image (prefix: 34 template tokens +
             256 image tokens = 290), and with 4 crops besides the image (5 x 256 image tokens + 20 = 1300), 64 new tokens,
             top_k = 200, temperature = 0.8, no EOS.  Every call draws a new image and new questions, as a loop over images
             does.  First each arm alone, from no captured step: the first call's wall time (cache allocation and graph capture
             included) and the allocator's peak memory of that arm.  Then the two arms alternate, each reusing its own captured
             step (the lengths stay inside its 256-row buckets), medians of `--runs`: time to first token (CUDA events from the
             call to the first sample: ViT + prefill), decode ms per step (CUDA events from the first sample to the end, over 63
             steps), the whole call's wall time and tokens/s.
  identical  greedy, 8 questions of 32 tokens about one image with a 512-token prefix (P % 256 == 0): the shared tokens against
             generate() on each question's own prompt, which must be the same.
"""
import argparse
import json
import time

import torch

from bench_generate import HBM_GBS, gpu_info
from bench_shared_prefix import max_sm_clock_mhz

BF16_TFLOPS = 989.0
H, D = 20, 128


def _med(xs):
    return sorted(xs)[len(xs) // 2]


def _floor_us(flops, nbytes):
    return max(flops / (BF16_TFLOPS * 1e12), nbytes / (HBM_GBS * 1e9)) * 1e6


def _events(fn, iters=20):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / iters * 1e3      # us


def run_attention(args, dev):
    from aria_b200 import ops
    scale = D ** -0.5
    g = torch.Generator().manual_seed(0)
    S = torch.randint(16, 65, (32,), generator=g).tolist()
    B, S_tot, Sm = len(S), sum(S), max(S)
    cu = [0]
    for s in S:
        cu.append(cu[-1] + s)
    cu_dev = torch.tensor(cu, dtype=torch.int32, device=dev)
    res = []
    for P in (290, 1300, 2304):
        gd = torch.Generator(device=dev).manual_seed(P)
        q, k, v = (torch.randn(1, H, S_tot, D, generator=gd, device=dev).bfloat16() for _ in range(3))
        pk, pv = (torch.randn(1, H, P, D, generator=gd, device=dev).bfloat16() for _ in range(2))
        eq = torch.zeros(B, H, Sm, D, dtype=torch.bfloat16, device=dev)
        ek = torch.zeros(B, H, P + Sm, D, dtype=torch.bfloat16, device=dev)
        ev = torch.zeros_like(ek)
        ek[:, :, :P], ev[:, :, :P] = pk, pv
        for b in range(B):
            eq[b, :, :S[b]] = q[0, :, cu[b]:cu[b + 1]]
            ek[b, :, P:P + S[b]], ev[b, :, P:P + S[b]] = k[0, :, cu[b]:cu[b + 1]], v[0, :, cu[b]:cu[b + 1]]
        shared = lambda: ops.attention_prefill_shared_prefix(q, k, v, S_tot, pk, pv, P, cu_dev, scale)
        expanded = lambda: ops.attention(eq, ek, ev, Sm, P + Sm, scale, causal=True)
        for _ in range(3):
            shared(), expanded()
        ts, te = [], []
        for _ in range(args.runs):
            ts.append(_events(shared))
            te.append(_events(expanded))
        pairs = sum(s * P + s * (s + 1) // 2 for s in S)
        flops = 4 * D * H * pairs
        row = 2 * D                                            # one bf16 row of one head
        b_s = H * row * (2 * P + 4 * S_tot)                    # prefix K, V once; suffix q, k, v and out
        b_e = H * row * (B * 2 * (P + Sm) + 2 * B * Sm)        # every row's K, V; padded q and out
        res.append({"P": P, "B": B, "H": H, "S_tot": S_tot, "shared_us": round(_med(ts), 2),
                    "expanded_us": round(_med(te), 2), "speedup": round(_med(te) / _med(ts), 3), "flops": flops,
                    "shared_bytes": b_s, "shared_floor_us": round(_floor_us(flops, b_s), 2),
                    "expanded_bytes": b_e, "expanded_floor_us": round(_floor_us(flops, b_e), 2)})
        del q, k, v, pk, pv, eq, ek, ev
        torch.cuda.empty_cache()
    return res


def _workload(cfg, B, n_images, n_template, seed, lens=None):
    """Left-padded ids of B questions about n_images images of 256 tokens each, the prefix = n_template tokens + the images."""
    g = torch.Generator().manual_seed(seed)
    V, img = cfg["text_config"]["vocab_size"], cfg["image_token_index"]
    pv = torch.randn(n_images, 3, 980, 980, generator=g).bfloat16()
    text = torch.randint(10, V, (n_template,), generator=g)
    prefix = torch.cat([text[:4]] + [torch.full((256,), img)] * n_images + [text[4:]])
    S = lens or torch.randint(16, 65, (B,), generator=g).tolist()
    T = prefix.numel() + max(S)
    ids = torch.zeros(B, T, dtype=torch.long)
    mask = torch.zeros(B, T, dtype=torch.long)
    for b, s in enumerate(S):
        ids[b, T - prefix.numel() - s:] = torch.cat([prefix, torch.randint(10, V, (s,), generator=g)])
        mask[b, T - prefix.numel() - s:] = 1
    return ids, pv, mask, prefix.numel()


def _timed_call(model, graphs, arm, fn):
    """One generate() call with the arm's own decode graph (none yet: the call captures it)
    -> (ttft ms, decode ms per step summed, wall s, peak GB).  The peak counts every graph alive during the call."""
    model._decode_graph = graphs.get(arm)
    g = model._decode_graph
    first = torch.cuda.Event(enable_timing=True)
    if g is not None:
        orig = g.sample_and_advance
        g.sample_and_advance = lambda logits: (orig(logits), first.record())
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    start.record()
    fn()
    end.record()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated() / 1e9
    graphs[arm] = model._decode_graph
    if g is None:
        return None, None, wall, peak
    del g.sample_and_advance
    return start.elapsed_time(first), first.elapsed_time(end), wall, peak


def run_generate(model, cfg, args, kw, B, crops):
    """Every call gets a new image and new questions (lengths and tokens drawn again), as a loop over images would: the
    captured steps are reused only where the 256-row buckets of the cache allow it."""
    new = 64
    n_tmpl = 34 if crops == 0 else 20

    def calls(i):
        ids, pv, mask, P = _workload(cfg, B, 1 + crops, n_tmpl, seed=1000 * B + 10 * crops + i)
        rep_pv = pv.repeat(B, 1, 1, 1)
        return {"shared": lambda: model.generate(ids, pv, None, max_new_tokens=new, attention_mask=mask, shared_prefix_len=P,
                                                 **kw),
                "repeated": lambda: model.generate(ids, rep_pv, None, max_new_tokens=new, attention_mask=mask, **kw)}, P

    out = {"B": B, "crops": crops, "new_tokens": new}
    # each arm alone, from no captured step: the first call's wall time (capture included) and the arm's own peak memory
    arms = []
    for arm in ("shared", "repeated"):
        model._decode_graph = None
        torch.cuda.empty_cache()
        fns, out["P"] = calls(0)
        try:
            _, _, wall, peak = _timed_call(model, {}, arm, fns[arm])
        except torch.cuda.OutOfMemoryError:   # the repeated arm runs the ViT on B * (1 + crops) images at once
            out[arm] = "not run: out of memory"
            continue
        out[arm] = {"first_call_s": round(wall, 4), "peak_gb_alone": round(peak, 2)}
        arms.append(arm)
    model._decode_graph = None
    torch.cuda.empty_cache()
    graphs = {}
    for i in range(max(args.warmup, 1)):
        fns, _ = calls(1 + i)
        for arm in arms:
            _timed_call(model, graphs, arm, fns[arm])
    r = {arm: [] for arm in arms}
    for i in range(args.runs):
        fns, _ = calls(100 + i)
        for arm in arms:
            r[arm].append(_timed_call(model, graphs, arm, fns[arm])[:3])
    for arm in arms:
        ttft, step, wall = (list(x) for x in zip(*r[arm]))
        out[arm].update({"ttft_ms": round(_med(ttft), 3), "decode_ms_per_step": round(_med(step) / (new - 1), 4),
                         "wall_s": round(_med(wall), 4), "tokens_per_s": round(B * new / _med(wall), 1),
                         "wall_s_runs": [round(x, 4) for x in wall]})
    if len(arms) == 2:
        sh, rp = out["shared"], out["repeated"]
        out["ttft_speedup"] = round(rp["ttft_ms"] / sh["ttft_ms"], 3)
        out["decode_speedup"] = round(rp["decode_ms_per_step"] / sh["decode_ms_per_step"], 3)
        out["wall_speedup"] = round(rp["wall_s"] / sh["wall_s"], 3)
    model._decode_graph = None
    del graphs
    torch.cuda.empty_cache()
    return out


def run_identical(model, cfg):
    """Greedy, 8 questions of 32 tokens about one image with a 512-token prefix (P % 256 == 0), against generate() on each
    question's own prompt.  The repeated-image batch is no bitwise reference at full width: the projector's output for an
    image depends on how many images share its batch."""
    ids, pv, _, P = _workload(cfg, 8, 1, 256, seed=99, lens=[32] * 8)
    a = model.generate(ids, pv, None, max_new_tokens=32, shared_prefix_len=P)
    same = all(torch.equal(a[b], model.generate(ids[b:b + 1], pv, None, max_new_tokens=32)[0]) for b in range(8))
    model._decode_graph = None
    torch.cuda.empty_cache()
    return {"B": 8, "P": P, "question_tokens": 32, "new_tokens": 32, "greedy": True, "tokens_identical": bool(same)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    from aria_b200 import configs as C
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration, init_random_
    dev = "cuda:0"
    name, power = gpu_info(0)
    out = {"bench": "shared_image", "gpu": name, "power_limit_w": power, "max_sm_clock_mhz": max_sm_clock_mhz(),
           "floor_source": f"{BF16_TFLOPS} TFLOP/s dense BF16, {HBM_GBS} GB/s HBM3, H100 SXM data sheet", "runs": args.runs}
    kw = dict(do_sample=True, top_k=200, temperature=0.8, seed=0)
    with torch.no_grad():
        out["attention"] = run_attention(args, dev)
        cfg = C.ARIA_25B
        model = AriaForConditionalGeneration(AriaConfig.from_dict(cfg), device=dev)
        init_random_(model, seed=0)
        out["identical"] = run_identical(model, cfg)
        out["generate"] = [run_generate(model, cfg, args, kw, B, crops) for B in (8, 32) for crops in (0, 4)]
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
