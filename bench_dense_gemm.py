"""The dense GEMMs of one cfg-2 prefill step (one 980 px image + 512 text tokens), each timed on its own through the public
`ops` call the model makes, next to torch.nn.functional.linear (cuBLAS) on the same operands; prints one JSON line.

    python bench_dense_gemm.py [--iters 200] [--runs 3] [--warmup 20]

Shapes (Aria-25.3B, bf16, random operands; nothing is read from outside the repository):
  ViT (4,900 patch rows, d 1152): q/k/v + bias scattered to 72-dim heads (128-wide tiles: 1152 = 9 x 128), o_proj + bias
  + residual, fc1 + bias + GELU-tanh, fc2 + bias + residual.  Projector: its k/v projections and in-projections at 4,900 rows, q / out / FFN at 256 query rows.
  LM at 768 rows (cfg 2) and 32 rows (cfg 3 decode: one token of 32 sequences): q/k/v + RoPE into the KV-cache layout, o_proj
  + residual, shared expert gate|up + SwiGLU and down.
Per shape: microseconds per launch (CUDA events around `--iters` launches, median of `--runs` rounds that alternate ours and
cuBLAS), TFLOP/s, and the L2 -> shared-memory traffic the mainloop implies.  A 128 x BN tile pulls (128 + BN) x 64 bf16 per
64-deep k-block for 2 x 128 x BN x 64 FLOP; a CTA pair that shares its A tile pulls (64 + BN) x 64 per CTA.  Both rates are
printed: `l2_tbs_1cta` at the first intensity, `l2_tbs_pair` at the second.  The card name, power limit and the SM clock
sampled during the timed rounds come with the result.
"""
import argparse
import json
import subprocess

import torch
import torch.nn.functional as F

import bench

BF16 = torch.bfloat16


def _power_limit(idx=0):
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(idx), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


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


def _w(n, k, g, dev):
    return (torch.randn(n, k, generator=g, device=dev) * k ** -0.5).to(BF16)


def _x(m, k, g, dev):
    return torch.randn(m, k, generator=g, device=dev).to(BF16)


def shapes(dev):
    """name -> (ours, cuBLAS, M, N (tile columns), K, BN)"""
    from aria_b200 import _lib as L
    from aria_b200 import ops
    g = torch.Generator(device=dev).manual_seed(0)
    out = {}

    # ---- ViT: 4,900 rows, 16 heads of 72 in [1, 16, 4900, 128] buffers
    M, d, I = 4900, 1152, 4304
    x, o, res = _x(M, d, g, dev), _x(M, d, g, dev), _x(M, d, g, dev)
    h1 = _x(M, I, g, dev)
    wq = [_w(d, d, g, dev) for _ in range(3)]
    bq = [_x(d, 1, g, dev).view(d) for _ in range(3)]
    bufs = [torch.zeros(1, 16, M, 128, dtype=BF16, device=dev) for _ in range(3)]
    wqkv, bqkv = torch.cat(wq), torch.cat(bq)
    out["vit_qkv"] = (lambda: ops.qkv_heads(x, wq, bq, bufs, 72, M), lambda: F.linear(x, wqkv, bqkv), M, 3 * d, d, 128)
    wo, bo = _w(d, d, g, dev), _x(d, 1, g, dev).view(d)
    out["vit_o_proj"] = (lambda: ops.linear(o, wo, bo, residual=res), lambda: torch.add(F.linear(o, wo, bo), res), M, d, d, 128)
    w1, b1 = _w(I, d, g, dev), _x(I, 1, g, dev).view(I)
    out["vit_fc1"] = (lambda: ops.linear(x, w1, b1, act=L.ACT_GELU_TANH),
                      lambda: F.gelu(F.linear(x, w1, b1), approximate="tanh"), M, I, d, 128)
    w2, b2 = _w(d, I, g, dev), _x(d, 1, g, dev).view(d)
    out["vit_fc2"] = (lambda: ops.linear(h1, w2, b2, residual=res), lambda: torch.add(F.linear(h1, w2, b2), res), M, d, I, 128)

    # ---- projector: k / v and their in-projections over the 4,900 ViT rows, the rest over 256 queries
    Q, E, ff, od = 256, 1152, 2560, 2560
    q = _x(Q, E, g, dev)
    wp = _w(E, E, g, dev)
    bp = _x(E, 1, g, dev).view(E)
    k2 = torch.zeros(1, 16, M, 128, dtype=BF16, device=dev)
    q2 = torch.zeros(1, 16, Q, 128, dtype=BF16, device=dev)
    out["proj_kv"] = (lambda: ops.linear(x, wp), lambda: F.linear(x, wp), M, E, E, 128)
    out["proj_in_kv"] = (lambda: ops.qkv_heads(x, [wp], [bp], [k2], 72, M), lambda: F.linear(x, wp, bp), M, E, E, 128)
    out["proj_q"] = (lambda: ops.linear(q, wp), lambda: F.linear(q, wp), Q, E, E, 128)
    out["proj_in_q"] = (lambda: ops.qkv_heads(q, [wp], [bp], [q2], 72, Q), lambda: F.linear(q, wp, bp), Q, E, E, 128)
    out["proj_out"] = (lambda: ops.linear(q, wp, bp), lambda: F.linear(q, wp, bp), Q, E, E, 128)
    wl = _w(od, E, g, dev)
    bl = _x(od, 1, g, dev).view(od)
    out["proj_linear"] = (lambda: ops.linear(q, wl, bl), lambda: F.linear(q, wl, bl), Q, od, E, 128)
    qf = _x(Q, od, g, dev)
    wi, wf = _w(ff, od, g, dev), _w(od, ff, g, dev)
    out["proj_ffn_in"] = (lambda: ops.linear(qf, wi, act=L.ACT_GELU_NEW),
                          lambda: F.gelu(F.linear(qf, wi), approximate="tanh"), Q, ff, od, 128)
    out["proj_ffn_out"] = (lambda: ops.linear(qf, wf), lambda: F.linear(qf, wf), Q, od, ff, 128)

    # ---- LM: 20 heads of 128, RoPE on q and k; shared expert 2 x 1664
    D, H, Is = 2560, 20, 3328
    wlq = [_w(D, D, g, dev) for _ in range(3)]
    wlqkv = torch.cat(wlq)
    wlo = _w(D, D, g, dev)
    wg, wu, wd = _w(Is, D, g, dev), _w(Is, D, g, dev), _w(D, Is, g, dev)
    wgu = torch.cat([wg, wu])
    inv = 1.0 / (5e6 ** (torch.arange(0, 128, 2, device=dev, dtype=torch.float32) / 128))
    cos, sin = ops.rope_table(inv, 4096)
    for rows, tag in ((768, "lm768"), (32, "lm32")):
        B, T = (1, rows) if rows == 768 else (rows, 1)
        xl, ol, rl, hl = _x(rows, D, g, dev), _x(rows, D, g, dev), _x(rows, D, g, dev), _x(rows, Is, g, dev)
        kv = [torch.zeros(B, H, T + 8 if T > 1 else 2048, 128, dtype=BF16, device=dev) for _ in range(3)]
        pos = torch.full((rows,), 2047 if T == 1 else 0, dtype=torch.int32, device=dev)
        pos_ids = None if T > 1 else pos

        def qkv(xl=xl, kv=kv, T=T, pos_ids=pos_ids):
            ops.qkv_heads(xl, wlq, [None] * 3, kv, 128, T, pos0=0, rope_mask=0b011, rope_cos=cos, rope_sin=sin,
                          position_ids=pos_ids)
        out[f"{tag}_qkv_rope"] = (qkv, lambda xl=xl: F.linear(xl, wlqkv), rows, 3 * D, D, 128)
        out[f"{tag}_o_proj"] = (lambda ol=ol, rl=rl: ops.linear(ol, wlo, residual=rl),
                                lambda ol=ol, rl=rl: torch.add(F.linear(ol, wlo), rl), rows, D, D, 128)
        out[f"{tag}_shared_gate_up"] = (lambda xl=xl: ops.linear_swiglu(xl, wg, wu),
                                        lambda xl=xl: F.linear(xl, wgu), rows, 2 * Is, D, 128)
        out[f"{tag}_shared_down"] = (lambda hl=hl: ops.linear(hl, wd), lambda hl=hl: F.linear(hl, wd), rows, D, Is, 128)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200, help="launches per timed window (>= 200)")
    ap.add_argument("--runs", type=int, default=3, help="alternating rounds of ours / cuBLAS; the median is reported")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--only", default=None, help="comma-separated shape names")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dense_gemm.py measures on the GPU; none is available")
    from aria_b200 import _lib as L
    L.load()
    dev = "cuda:0"
    torch.set_grad_enabled(False)
    table = shapes(dev)
    if args.only:
        table = {k: v for k, v in table.items() if k in args.only.split(",")}
    sampler = bench.ClockSampler(0)
    sampler.start()
    rows = {}
    for name, (ours, ref, M, N, K, BN) in table.items():
        for _ in range(args.warmup):
            ours(), ref()
        t = {"ours": [], "cublas": []}
        for _ in range(args.runs):
            t["ours"].append(_time_us(ours, args.iters))
            t["cublas"].append(_time_us(ref, args.iters))
        us, us_ref = _median(t["ours"]), _median(t["cublas"])
        flop = 2.0 * M * N * K
        rows[name] = {"M": M, "N": N, "K": K, "BN": BN, "us": round(us, 2), "us_runs": [round(v, 2) for v in t["ours"]],
                      "tflops": round(flop / us / 1e6, 1), "cublas_us": round(us_ref, 2),
                      "cublas_tflops": round(flop / us_ref / 1e6, 1),
                      "l2_tbs_1cta": round(flop / (128 * BN / (128 + BN)) / us / 1e6, 2),
                      "l2_tbs_pair": round(flop / (128 * BN / (64 + BN)) / us / 1e6, 2)}
    clocks = sampler.stop()
    print(json.dumps({"bench": "dense_gemm", "gpu": torch.cuda.get_device_name(0), "power_limit_w": _power_limit(0),
                      "lib": L.LIB_PATH, "clocks": clocks, "iters": args.iters, "runs": args.runs, "shapes": rows}), flush=True)


if __name__ == "__main__":
    main()
