"""Writes the outputs of the GEMM `ops` calls of one cfg-2 prefill step at their cfg-2 shapes, from seeded operands, as
DIR/<name>.npy (bf16 bits as uint16), so that two builds of the library can be compared bit for bit.

    python dump_gemm_ops.py DIR

Calls: routed fc1 + SwiGLU and fc2 (4,608 rows over 64 experts, d 2560, I 1664), LM q/k/v + RoPE into the KV-cache layout
(768 rows, 20 heads of 128) and the shared expert's gate/up + SwiGLU and down (768 rows, 2 x 1664 columns).  Without a
GPU the script fails."""
import os
import sys

import numpy as np
import torch


def main():
    out_dir = sys.argv[1]
    if not torch.cuda.is_available():
        raise SystemExit("dump_gemm_ops.py runs the kernels on the GPU; none is available")
    from aria_b200 import _lib as L
    from aria_b200 import ops
    from bench_expert_gemm import row_counts
    L.load()
    os.makedirs(out_dir, exist_ok=True)
    dev, bf16 = "cuda:0", torch.bfloat16
    torch.set_grad_enabled(False)
    g = torch.Generator(device=dev).manual_seed(0)

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, generator=g, device=dev) * scale).to(bf16)

    D, I, E, T, H = 2560, 1664, 64, 768, 20
    outs = {}
    counts = row_counts(4608)
    off = torch.zeros(E + 1, dtype=torch.int32)
    off[1:] = torch.tensor(counts).cumsum(0).to(torch.int32)
    off = off.to(dev)
    a = rnd(4608, D)
    w1, w2 = rnd(E, D, 2 * I, scale=0.02), rnd(E, I, D, scale=0.02)
    outs["fc1_swiglu"] = ops.grouped_gemm(a, w1, off, swiglu=True)
    outs["fc2"] = ops.grouped_gemm(outs["fc1_swiglu"], w2, off)

    x = rnd(T, D)
    wq = [rnd(D, D, scale=D ** -0.5) for _ in range(3)]
    inv = 1.0 / (5e6 ** (torch.arange(0, 128, 2, device=dev, dtype=torch.float32) / 128))
    cos, sin = ops.rope_table(inv, 4096)
    kv = [torch.zeros(1, H, T, 128, dtype=bf16, device=dev) for _ in range(3)]
    ops.qkv_heads(x, wq, [None] * 3, kv, 128, T, pos0=0, rope_mask=0b011, rope_cos=cos, rope_sin=sin)
    outs["qkv_rope_q"], outs["qkv_rope_k"], outs["qkv_v"] = kv
    wg, wu, wd = rnd(I, D, scale=D ** -0.5), rnd(I, D, scale=D ** -0.5), rnd(D, I, scale=I ** -0.5)
    outs["shared_gate_up"] = ops.linear_swiglu(x, wg, wu)
    outs["shared_down"] = ops.linear(outs["shared_gate_up"], wd)
    torch.cuda.synchronize()
    for name, t in outs.items():
        np.save(os.path.join(out_dir, f"{name}.npy"), t.contiguous().view(torch.int16).cpu().numpy().view(np.uint16))
    print(f"wrote {len(outs)} arrays to {out_dir} with {L.LIB_PATH}")


if __name__ == "__main__":
    main()
