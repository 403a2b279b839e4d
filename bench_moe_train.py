#!/usr/bin/env python
"""bench_moe_train.py — one full-width MoE layer as fine-tuning runs it, on one H100: forward + backward of the reference's own
`MoELayer` (d 2560, 64 experts, top-6, I 1664, two shared experts) in train() mode (router losses on) at the SFT recipes' tokens
per step (8 x 2048), three ways on the same module parameters and inputs:

    reference  the unmodified layer (its `sequential_gemm` fallback: a Python loop over the 64 experts, ATen autograd)
    seam1      the unmodified layer with only `experts_gemm` rebound to the differentiable gmm (`moe_train.experts_gemm_train`)
    seam2      `install(..., trainable=True)`: the whole layer as one `MoELayerFunction` on our kernels

    python bench_moe_train.py [--steps N] [--warmup W]

The arms are timed alternately in one process with CUDA events (median of 5 rounds of N forward + backward calls each) and the
gradients of each seam arm are compared with the reference arm's (rel-L2 of the input gradient and the worst parameter
gradient; bf16 routing near-ties may send a token to another expert, so these are not exact).  Needs the reference model files
staged by build() (oracle/_ref).  Prints one JSON line with the GPU name and power limit read in the same run; writes nothing.
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def _power_limit_w(gpu_index):
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(gpu_index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def run_moe_train(args):
    import torch

    from aria_b200 import _lib as L
    from aria_b200 import install, moe_train
    from oracle import ref_loader

    L.load()
    ref = ref_loader.load_reference()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, rounds, warm = max(args.steps, 1), 5, max(args.warmup, 1)
    d, E, k, I, B, T = 2560, 64, 6, 1664, 8, 2048
    cfg = ref.moe_lm.AriaMoELMConfig(hidden_size=d, num_attention_heads=d // 128, moe_num_experts=E, moe_topk=k,
                                     moe_intermediate_size=I, moe_num_shared_experts=2, intermediate_size=I)
    layer = ref.moe_lm.MoELayer(cfg)
    g = torch.Generator().manual_seed(0)
    for p_ in layer.parameters():                      # `torch.empty` + FIXME in the reference (moe_lm.py:185-188,465)
        p_.data = torch.randn(p_.shape, generator=g) * 0.02
    layer = layer.to(dev, torch.bfloat16).train()
    seamed = copy.deepcopy(layer)
    install.install(torch.nn.ModuleList([seamed]), trainable=True)
    x = torch.randn(B, T, d, generator=g).bfloat16().to(dev)
    gout = torch.randn(B, T, d, generator=g).bfloat16().to(dev)
    sequential = ref.moe_lm.sequential_gemm

    def step(mod, gmm):
        ref.moe_lm.experts_gemm = gmm
        for p_ in mod.parameters():
            p_.grad = None
        xg = x.detach().requires_grad_(True)
        mod(xg).backward(gout)
        return xg

    arms = {"reference": lambda: step(layer, sequential), "seam1": lambda: step(layer, moe_train.experts_gemm_train),
            "seam2": lambda: step(seamed, sequential)}

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    try:
        for f in arms.values():
            for _ in range(warm):
                f()
        t = {name: [] for name in arms}
        for _ in range(rounds):                        # alternate the arms so that all see the same clocks
            for name, f in arms.items():
                t[name].append(timed(f))
        ms = {name: statistics.median(v) for name, v in t.items()}

        def grads(name):
            mod = seamed if name == "seam2" else layer
            xg = arms[name]()
            return {"x": xg.grad.float()} | {nm: p_.grad.float() for nm, p_ in mod.named_parameters()}

        want = grads("reference")
        rel = {}
        for name in ("seam1", "seam2"):
            got = grads(name)
            r = {nm: float((got[nm] - want[nm]).norm() / want[nm].norm()) for nm in want}
            worst = max((v, nm) for nm, v in r.items() if nm != "x")
            rel[name] = {"x": r["x"], "worst_param": worst[0], "worst_param_name": worst[1]}
    finally:
        ref.moe_lm.experts_gemm = sequential
    tokens = B * T
    line = {"metric": "MoE layer forward + backward, train() mode, d 2560, E 64, top-6, I 1664, 2 shared experts, bf16",
            "unit": "ms", "tokens": tokens, "gpu": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit_w(0),
            "iters_per_round": n, "rounds": rounds, "timing": "CUDA events, median over rounds, arms alternating",
            "ms": ms, "tokens_per_s": {a: tokens / (v * 1e-3) for a, v in ms.items()},
            "speedup_vs_reference": {a: ms["reference"] / v for a, v in ms.items()},
            "grad_rel_l2_vs_reference": rel, "impl": "aria_b200"}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5, help="forward + backward calls per timed round")
    ap.add_argument("--warmup", type=int, default=2)
    run_moe_train(ap.parse_args())


if __name__ == "__main__":
    main()
