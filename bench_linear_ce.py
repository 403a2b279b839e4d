#!/usr/bin/env python
"""bench_linear_ce.py — the fine-tuning loss head alone on one H100: lm_head + cross-entropy, forward + backward, at the SFT
recipes' batch (8 sequences x 2048 = 16,384 rows, d 2560, V 100,352, bf16) with 0 %, 50 % and 75 % of the labels ignored
(-100, as aria/data.py sets on the user turn), two ways on the same inputs:

    reference  bf16 F.linear -> the reference's mask-and-copy of the kept rows -> nn.CrossEntropyLoss, autograd backward
               (modeling_aria.py:302-323; no padding here, so the attention mask keeps every row)
    fused      aria_b200.loss.linear_cross_entropy: logits for the labelled rows only, 4,096 rows at a time

    python bench_linear_ce.py [--steps N] [--warmup W]

Per ignored fraction: ms per forward + backward (CUDA events, median of 5 rounds of N calls, arms alternating), the peak
memory each arm allocates above its inputs (the gradients it returns included), and the fused arm's loss and gradients
against the reference arm's (rel-L2).  Then the cross-entropy kernel alone on one 4,096-row chunk against its HBM floor (it
reads the logits twice and writes them once), and the GEMM FLOP floor of the head (2 rows d V forward, twice that backward).
Prints one JSON line with the GPU name and power limit read in the same run; writes nothing.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12        # H100 SXM data sheet
BF16_DENSE_FLOP_PER_S = 989e12   # H100 SXM data sheet, dense


def _power_limit_w(gpu_index):
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(gpu_index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def run(args):
    import torch
    import torch.nn.functional as F

    from aria_b200 import _lib as L
    from aria_b200 import ops
    from aria_b200.loss import linear_cross_entropy

    L.load()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, rounds, warm = max(args.steps, 1), 5, max(args.warmup, 1)
    B, T, d, V = 8, 2048, 2560, 100352
    rows = B * T
    g = torch.Generator().manual_seed(0)
    weight = (torch.randn(V, d, generator=g) * 0.02).bfloat16().to(dev).requires_grad_(True)
    hidden = (torch.randn(rows, d, generator=g) * 2.0).bfloat16().to(dev).requires_grad_(True)
    ids = torch.randint(0, V, (B, T), generator=g).to(dev)
    attn = torch.ones(B, T, dtype=torch.long, device=dev)

    def reference(labels):
        logits = F.linear(hidden, weight).view(B, T, V)
        kept = logits[attn != 0].contiguous()
        loss = torch.nn.CrossEntropyLoss()(kept.view(-1, V), labels[attn != 0].contiguous().view(-1))
        loss.backward()
        return loss

    def fused(labels):
        loss = linear_cross_entropy(hidden, weight, labels.view(-1))
        loss.backward()
        return loss

    def step(fn, labels):
        hidden.grad = weight.grad = None
        return fn(labels)

    def timed(fn, labels):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            step(fn, labels)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    def peak_bytes(fn, labels):
        hidden.grad = weight.grad = None
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        loss = fn(labels)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated(dev) - base
        return peak, loss.detach().float(), hidden.grad.float(), weight.grad.float()

    def rel(a, b):
        return float((a - b).norm() / b.norm())

    arms = {"reference": reference, "fused": fused}
    cases = {}
    for frac in (0.0, 0.5, 0.75):
        labels = ids.clone()
        labels[:, :int(round(frac * T))] = -100          # the user turn of every sequence
        n_valid = int((labels != -100).sum())
        for fn in arms.values():
            for _ in range(warm):
                step(fn, labels)
        t = {a: [] for a in arms}
        for _ in range(rounds):
            for a, fn in arms.items():
                t[a].append(timed(fn, labels))
        ms = {a: statistics.median(v) for a, v in t.items()}
        pk_ref, loss_ref, dh_ref, dw_ref = peak_bytes(reference, labels)
        pk_fused, loss_fused, dh_fused, dw_fused = peak_bytes(fused, labels)
        flop_fused = 6.0 * n_valid * d * V
        cases[f"{int(frac * 100)}%_ignored"] = {
            "valid_rows": n_valid, "ms": ms, "speedup_vs_reference": ms["reference"] / ms["fused"],
            "peak_gb_above_inputs": {"reference": pk_ref / 1e9, "fused": pk_fused / 1e9},
            "loss": {"reference": float(loss_ref), "fused": float(loss_fused)},
            "rel_l2_fused_vs_reference": {"loss": abs(float(loss_fused - loss_ref)) / abs(float(loss_ref)),
                                          "d_hidden": rel(dh_fused, dh_ref), "d_weight": rel(dw_fused, dw_ref)},
            # the reference computes every row's logits; the fused arm only the labelled rows'
            "gemm_flop": {"reference": 6.0 * rows * d * V, "fused": flop_fused},
            "gemm_flop_floor_ms_fused": flop_fused / BF16_DENSE_FLOP_PER_S * 1e3,
            "fused_tflop_per_s": flop_fused / (ms["fused"] * 1e-3) / 1e12,
        }
        del dh_ref, dw_ref, dh_fused, dw_fused
        hidden.grad = weight.grad = None

    # the cross-entropy kernel alone, one 4,096-row chunk (in place: later launches see gradients, still finite logits)
    chunk = 4096
    buf = torch.randn(chunk, V, generator=g).mul_(3.0).bfloat16().to(dev)
    lab = torch.randint(0, V, (chunk,), generator=g).to(dev)
    gs = torch.full((1,), 1.0 / chunk, dtype=torch.float32, device=dev)
    loss_rows = torch.empty(chunk, dtype=torch.float32, device=dev)
    for _ in range(3):
        ops.cross_entropy_rows(buf, lab, gs, loss=loss_rows)
    reps = 20
    ce_ms = []
    for _ in range(rounds):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            ops.cross_entropy_rows(buf, lab, gs, loss=loss_rows)
        e1.record()
        torch.cuda.synchronize()
        ce_ms.append(e0.elapsed_time(e1) / reps)
    ce = statistics.median(ce_ms)
    ce_bytes = 3 * chunk * V * 2
    line = {"metric": "lm_head + cross-entropy forward + backward, 8 x 2048 rows, d 2560, V 100352, bf16", "unit": "ms",
            "gpu": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit_w(0), "iters_per_round": n,
            "rounds": rounds, "timing": "CUDA events, median over rounds, arms alternating", "cases": cases,
            "ce_kernel_4096_rows": {"ms": ce, "hbm_bytes": ce_bytes, "hbm_floor_ms": ce_bytes / HBM_BYTES_PER_S * 1e3,
                                    "share_of_hbm_floor": ce_bytes / HBM_BYTES_PER_S * 1e3 / ce,
                                    "achieved_tb_per_s": ce_bytes / (ce * 1e-3) / 1e12},
            "impl": "aria_b200"}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5, help="forward + backward calls per timed round")
    ap.add_argument("--warmup", type=int, default=2)
    run(ap.parse_args())


if __name__ == "__main__":
    main()
