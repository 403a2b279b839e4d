"""The routed-expert grouped GEMMs alone, each launch timed on its own through the public `ops` call the model makes; prints
one JSON line.

    python bench_expert_gemm.py [--rows 6,192,4608,196608] [--modes bf16,w8a16,w8a8] [--iters 200] [--runs 3] [--warmup 20]

Full-width Aria experts (d 2560, I 1664, E 64, random operands; nothing is read from outside the repository): fc1 + SwiGLU
(2560 -> 2 x 1664 -> 1664) and fc2 (1664 -> 2560) at 6 (batch-1 decode), 192 (batch-32 decode), 4,608 (cfg 2) and 196,608
(32,768 tokens) routed rows, spread over the experts by a seeded multinomial draw; bf16 weights, e4m3 weights with bf16
activations (W8A16) and e4m3 weights and activations (W8A8, the row-quantize passes not included).

Per case: microseconds per launch (CUDA events around `--iters` launches, median of `--runs` rounds, after `--warmup`
launches), and two byte counts with their rates.
  weight_bytes   the weights of the experts that own a row: what the launch must read from HBM at least.
  l2_smem_bytes  what the tiles pull from L2 into shared memory, computed from the row counts with the kernel's rule
                 (tile_a_rows): per 128-byte-deep k-block a 128 x 128 tile loads its B stage and, of A, the rows of its
                 m-tile that the group owns, rounded up to 16.  `l2_smem_bytes_box128` is the same sum with a whole 128-row A
                 box per tile, which is what the kernel loaded before it cut A to the group's rows.
The card name, its power limit and the SM clock sampled during the timed rounds come with the result.  Without a GPU the
script fails: a CPU has nothing to say about these numbers.
"""
import argparse
import json

D, I, E = 2560, 1664, 64
BM, A_BOX_MIN, TILE_N = 128, 16, 128
KBLOCK_BYTES = 128                      # one row of a k-block in shared memory: 64 bf16 or 128 e4m3 (one SW128 row)
MODES = {"bf16": (2, 2), "w8a16": (2, 1), "w8a8": (1, 1)}     # bytes per A element / per B element


def tile_a_rows(count, m_idx, rule="cover"):
    """Rows of A that m-tile m_idx of a group of `count` rows loads per k-block: the kernel's tile_a_rows ("cover"), or the
    whole box ("box128")."""
    left = count - m_idx * BM
    assert left > 0
    if rule == "box128":
        return BM
    return min(BM, -(-left // A_BOX_MIN) * A_BOX_MIN)


def launch_shape(which):
    """(K, B columns, n-tiles) of fc1 + SwiGLU ("fc1": a tile holds 64 gate and 64 up columns) or fc2."""
    return (D, 2 * I, I // (TILE_N // 2)) if which == "fc1" else (I, D, D // TILE_N)


def weight_bytes(counts, which, mode):
    K, n_cols, _ = launch_shape(which)
    return sum(1 for c in counts if c > 0) * K * n_cols * MODES[mode][1]


def l2_smem_bytes(counts, which, mode, rule="cover"):
    """Bytes the launch's tiles load into shared memory: per tile and k-block, tile_a_rows(..) rows of A and one B stage."""
    a_el, b_el = MODES[mode]
    K, _, n_tiles = launch_shape(which)
    k_elems = KBLOCK_BYTES // a_el                       # elements of K per k-block
    k_blocks = -(-K // k_elems)
    b_stage = TILE_N * k_elems * b_el
    total = 0
    for c in counts:
        for m in range(-(-c // BM)):
            total += n_tiles * k_blocks * (tile_a_rows(c, m, rule) * KBLOCK_BYTES + b_stage)
    return total


def row_counts(rows, seed=0):
    """`rows` routed rows over the E experts: one seeded multinomial draw with equal probabilities."""
    import torch
    g = torch.Generator().manual_seed(seed)
    pick = torch.multinomial(torch.ones(E), rows, replacement=True, generator=g)
    return torch.bincount(pick, minlength=E).tolist()


def _time_us(torch, fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rows", default="6,192,4608,196608", help="comma-separated routed-row counts")
    ap.add_argument("--modes", default="bf16,w8a16,w8a8", help="comma-separated subset of bf16,w8a16,w8a8")
    ap.add_argument("--iters", type=int, default=200, help="launches per timed window (>= 200)")
    ap.add_argument("--runs", type=int, default=3, help="timed rounds per case; the median is reported")
    ap.add_argument("--warmup", type=int, default=20, help="launches before the timed rounds (>= 20)")
    args = ap.parse_args()
    modes = args.modes.split(",")
    if any(m not in MODES for m in modes):
        ap.error(f"--modes takes {','.join(MODES)}")

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_expert_gemm.py measures on the GPU; none is available")
    import bench
    from bench_dense_gemm import _median, _power_limit
    from aria_b200 import _lib as L
    from aria_b200 import ops
    L.load()
    dev = "cuda:0"
    torch.set_grad_enabled(False)
    g = torch.Generator(device=dev).manual_seed(0)
    w1 = torch.empty(E, D, 2 * I, dtype=torch.bfloat16, device=dev).normal_(0.0, 0.02, generator=g)
    w2 = torch.empty(E, I, D, dtype=torch.bfloat16, device=dev).normal_(0.0, 0.02, generator=g)
    q1 = s1 = q2 = s2 = k1 = k2 = None
    if "w8a16" in modes or "w8a8" in modes:
        q1, s1 = ops.quantize_fp8_cols(w1)
        q2, s2 = ops.quantize_fp8_cols(w2)
    if "w8a8" in modes:     # the K-major layout of the same codes
        k1, k2 = (q.transpose(1, 2).contiguous().transpose(1, 2) for q in (q1, q2))

    sampler = bench.ClockSampler(0)
    sampler.start()
    cases = {}
    for rows in (int(r) for r in args.rows.split(",")):
        counts = row_counts(rows)
        off = torch.zeros(E + 1, dtype=torch.int32)
        off[1:] = torch.tensor(counts).cumsum(0).to(torch.int32)
        off = off.to(dev)
        a = torch.empty(rows, D, dtype=torch.bfloat16, device=dev).normal_(generator=g)
        h = ops.grouped_gemm(a, w1, off, swiglu=True)
        aq, a_s = ops.permute_quantize_fp8(a)
        hq, h_s = ops.permute_quantize_fp8(h)
        launches = {
            ("bf16", "fc1"): lambda: ops.grouped_gemm(a, w1, off, swiglu=True),
            ("bf16", "fc2"): lambda: ops.grouped_gemm(h, w2, off),
            ("w8a16", "fc1"): lambda: ops.grouped_gemm_fp8(a, q1, s1, off, swiglu=True),
            ("w8a16", "fc2"): lambda: ops.grouped_gemm_fp8(h, q2, s2, off),
            ("w8a8", "fc1"): lambda: ops.grouped_gemm_w8a8(aq, a_s, k1, s1, off, swiglu=True),
            ("w8a8", "fc2"): lambda: ops.grouped_gemm_w8a8(hq, h_s, k2, s2, off),
        }
        res = {"experts_hit": sum(1 for c in counts if c > 0), "max_rows_per_expert": max(counts)}
        for (mode, which), fn in launches.items():
            if mode not in modes:
                continue
            for _ in range(args.warmup):
                fn()
            runs = [_time_us(torch, fn, args.iters) for _ in range(args.runs)]
            us = _median(runs)
            wb = weight_bytes(counts, which, mode)
            lb, lb128 = l2_smem_bytes(counts, which, mode), l2_smem_bytes(counts, which, mode, "box128")
            res[f"{mode}_{which}"] = {"us": round(us, 2), "us_runs": [round(v, 2) for v in runs], "weight_bytes": wb,
                                      "weight_tbs": round(wb / us / 1e6, 3), "l2_smem_bytes": lb,
                                      "l2_smem_tbs": round(lb / us / 1e6, 3), "l2_smem_bytes_box128": lb128,
                                      "l2_smem_tbs_box128": round(lb128 / us / 1e6, 3)}
        cases[str(rows)] = res
        del a, h, aq, hq
    clocks = sampler.stop()
    print(json.dumps({"bench": "expert_gemm", "gpu": torch.cuda.get_device_name(0), "power_limit_w": _power_limit(0),
                      "lib": L.LIB_PATH, "clocks": clocks, "iters": args.iters, "runs": args.runs, "warmup": args.warmup,
                      "experts": E, "d": D, "intermediate": I, "cases": cases}), flush=True)


if __name__ == "__main__":
    main()
