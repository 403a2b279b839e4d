#!/usr/bin/env python
"""bench_attention_train.py — the LM attention core as fine-tuning runs it, on one H100: our forward with LSE
(aria_attention_fwd_lse) and backward (aria_attention_bwd) against torch.nn.functional.scaled_dot_product_attention.

    python bench_attention_train.py [--steps N] [--warmup W]

Causal, 20 heads x 128, bf16, at B=8, T=2048 (the reference LoRA recipe's per-device batch and max_seq_length) and B=1, T=8192.
Both implementations run on the same seeded inputs in the same process and are timed alternately with CUDA events (median of 5
rounds of max(N, 50) calls).  Prints one JSON line: ms and TFLOP/s of forward, backward and forward + backward for each (FLOPs:
forward 4*B*H*pairs*128, backward 2.5x), the SDPA backend's kernels, the rel-L2 between our gradients and SDPA's, and the
GPU name and power limit read in the same run.  Writes nothing to disk.
"""
import argparse
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


def run_attention_train(args):
    """The LM attention core as fine-tuning runs it (causal, 20 heads x 128, bf16): our forward with LSE
    (aria_attention_fwd_lse) and backward (aria_attention_bwd) against torch.nn.functional.scaled_dot_product_attention
    (is_causal=True) forward + autograd backward on the same inputs, the two timed alternately in the same process with CUDA
    events.  Shapes: B=8, T=2048 (the reference LoRA recipe's batch and max_seq_length) and B=1, T=8192."""
    import torch
    import torch.nn.functional as F

    from aria_b200 import _lib as L
    from aria_b200 import ops

    L.load()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, rounds, warm = max(args.steps, 50), 5, max(args.warmup, 3)

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    def rel(a, b):
        return float((a.float() - b.float()).norm() / b.float().norm())

    rows, backends = [], set()
    for B, H, T in ((8, 20, 2048), (1, 20, 8192)):
        g = torch.Generator(device=dev).manual_seed(0)
        q, k, v = (torch.randn(B, H, T, 128, generator=g, device=dev, dtype=torch.bfloat16) for _ in range(3))
        dout = torch.randn(B, T, H * 128, generator=g, device=dev, dtype=torch.bfloat16)
        scale = 128 ** -0.5
        out, lse = ops.attention(q, k, v, T, T, scale, True, return_lse=True)
        qs, ks, vs = (t.clone().requires_grad_(True) for t in (q, k, v))
        dout_s = dout.view(B, T, H, 128).transpose(1, 2)

        def ours_fwd():
            return ops.attention(q, k, v, T, T, scale, True, return_lse=True)

        def ours_bwd():
            return ops.attention_bwd(q, k, v, out, dout, lse, T, T, scale, True)

        def ours_both():
            o, l_ = ours_fwd()
            return ops.attention_bwd(q, k, v, o, dout, l_, T, T, scale, True)

        def sdpa_fwd():
            with torch.no_grad():
                return F.scaled_dot_product_attention(qs, ks, vs, is_causal=True)

        def sdpa_both():
            o = F.scaled_dot_product_attention(qs, ks, vs, is_causal=True)
            return torch.autograd.grad(o, (qs, ks, vs), dout_s)

        fns = {"ours_fwd": ours_fwd, "ours_bwd": ours_bwd, "ours_fwdbwd": ours_both, "sdpa_fwd": sdpa_fwd, "sdpa_fwdbwd": sdpa_both}
        for f in fns.values():
            for _ in range(warm):
                f()
        t = {name: [] for name in fns}
        for _ in range(rounds):                        # alternate ours and SDPA so that both see the same clocks
            for name, f in fns.items():
                t[name].append(timed(f))
        ms = {name: statistics.median(v_) for name, v_ in t.items()}
        ms["sdpa_bwd"] = ms["sdpa_fwdbwd"] - ms["sdpa_fwd"]
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            sdpa_both()
            torch.cuda.synchronize()
        for e in prof.key_averages():
            low = e.key.lower()
            for tag in ("flash", "cudnn", "efficient", "fmha", "math"):
                if tag in low:
                    backends.add(f"{tag}: {e.key[:80]}")
        fl_fwd = 4 * B * H * (T * (T + 1) // 2) * 128
        fl = {"fwd": fl_fwd, "bwd": 2.5 * fl_fwd, "fwdbwd": 3.5 * fl_fwd}

        def side(prefix):
            return {f"{ph}_ms": ms[f"{prefix}_{ph}"] for ph in ("fwd", "bwd", "fwdbwd")} | \
                   {f"{ph}_tflops": fl[ph] / (ms[f"{prefix}_{ph}"] * 1e-3) / 1e12 for ph in ("fwd", "bwd", "fwdbwd")}

        dq, dk, dv = ours_bwd()
        sq, sk, sv = sdpa_both()
        rows.append({"B": B, "H": H, "T": T, "causal": True, "ours": side("ours"), "sdpa": side("sdpa"),
                     "rel_l2_vs_sdpa": {"dq": rel(dq, sq), "dk": rel(dk, sk), "dv": rel(dv, sv),
                                        "out": rel(out, F.scaled_dot_product_attention(q, k, v, is_causal=True).transpose(1, 2).reshape(B, T, H * 128))}})
        del qs, ks, vs, q, k, v, out, lse, dout
        torch.cuda.empty_cache()
    line = {"metric": "LM attention core forward (with LSE) + backward, causal, 20 heads x 128, bf16", "unit": "ms",
            "gpu": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit_w(0), "iters_per_round": n, "rounds": rounds,
            "timing": "CUDA events, median over rounds, ours and SDPA alternating", "flops": "fwd 4*B*H*pairs*128, bwd 2.5x fwd",
            "sdpa_backend": sorted(backends), "shapes": rows, "impl": "aria_b200"}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50, help="calls per timed round (at least 50)")
    ap.add_argument("--warmup", type=int, default=3)
    run_attention_train(ap.parse_args())


if __name__ == "__main__":
    main()
