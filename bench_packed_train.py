#!/usr/bin/env python
"""bench_packed_train.py — padding-free fine-tuning on one H100: the same eight examples as a right-padded [8, 2048] batch (the
reference recipe's collate_fn) and packed into one row (`aria_b200.packing.pack_batch`), timed alternately in one process.

    python bench_packed_train.py [--steps N] [--warmup W]

The eight lengths are a fixed, seeded draw from [128, 2048]: a synthetic mix, since there is no fine-tuning dataset here.
Arms:
  attention      the LM attention core (20 heads x 128, bf16), forward with LSE + backward: padded [8, 2048] with the key mask
                 (aria_attention_fwd_lse + aria_attention_bwd) vs packed (aria_attention_fwd_varlen + aria_attention_bwd_varlen).
                 TFLOP/s against the causal floor 4*H*128*sum len(len+1)/2 forward, 2.5x that backward, for both arms.
  control        the same with no padding at all: 8 x 2048 packed vs [8, 2048], i.e. the varlen kernels' overhead on identical work.
  decoder_layer  transformers' AriaTextDecoderLayer at Aria's text config (d 2560, 20 heads, 64 experts top-6, 2 shared), bf16,
                 with install(trainable=True) and the hf_attention seam: forward + backward, ms and real (non-pad) tokens/s.
                 Also an unpadded [8, 2048] batch with no mask, with and without the seam's host read of position_ids (its
                 packing check) in every step: what that read costs a step.
CUDA events, warm-up, median of 5 rounds, arms alternating.  Prints one JSON line with the GPU name and power limit read in the
same run.  Writes nothing to disk.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

H, D, T_MAX, B = 20, 128, 2048, 8


def _power_limit_w(gpu_index):
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(gpu_index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def lengths(seed=0):
    """The synthetic length mix: eight draws from [128, 2048] with a fixed seed, one of them the full 2048 (the padded batch's
    width, as the recipe's longest example sets it)."""
    import torch
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(128, T_MAX + 1, (B,), generator=g).tolist()
    lens[0] = T_MAX
    return lens


def causal_flops(lens):
    """Forward floor 4*H*128*sum len(len+1)/2; the backward counts 2.5x (DESIGN §6b)."""
    fwd = 4 * H * D * sum(n * (n + 1) // 2 for n in lens)
    return {"fwd": fwd, "bwd": 2.5 * fwd, "fwdbwd": 3.5 * fwd}


def run(args):
    import torch

    from aria_b200 import _lib as L
    from aria_b200 import ops

    L.load()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, rounds, warm = max(args.steps, 10), 5, max(args.warmup, 3)
    scale = D ** -0.5

    def timed(fn, iters):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    def alternate(fns, iters):
        for f in fns.values():
            for _ in range(warm):
                f()
        t = {name: [] for name in fns}
        for _ in range(rounds):
            for name, f in fns.items():
                t[name].append(timed(f, iters))
        return {name: statistics.median(v) for name, v in t.items()}

    def attention_arms(lens):
        N = sum(lens)
        g = torch.Generator(device=dev).manual_seed(1)
        q, k, v = (torch.randn(B, H, T_MAX, D, generator=g, device=dev, dtype=torch.bfloat16) for _ in range(3))
        dout = torch.randn(B, T_MAX, H * D, generator=g, device=dev, dtype=torch.bfloat16)
        km = torch.ones(B, T_MAX, dtype=torch.uint8, device=dev)
        for b, m in enumerate(lens):
            km[b, :m] = 0
        # the packed row holds the same real rows
        pq, pk, pv = (torch.cat([t[b, :, :m] for b, m in enumerate(lens)], dim=1)[None].contiguous() for t in (q, k, v))
        pdout = torch.cat([dout[b, :m] for b, m in enumerate(lens)]).contiguous()
        cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=dev)

        def padded():
            o, lse = ops.attention(q, k, v, T_MAX, T_MAX, scale, True, key_mask=km, return_lse=True)
            return ops.attention_bwd(q, k, v, o, dout, lse, T_MAX, T_MAX, scale, True, key_mask=km)

        def packed():
            o, lse = ops.attention_varlen(pq, pk, pv, cu, scale, return_lse=True)
            return ops.attention_varlen_bwd(pq, pk, pv, o, pdout, lse, cu, scale)

        def padded_fwd():
            return ops.attention(q, k, v, T_MAX, T_MAX, scale, True, key_mask=km, return_lse=True)

        def packed_fwd():
            return ops.attention_varlen(pq, pk, pv, cu, scale, return_lse=True)

        ms = alternate({"padded_fwd": padded_fwd, "packed_fwd": packed_fwd, "padded_fwdbwd": padded, "packed_fwdbwd": packed}, n)
        fl = causal_flops(lens)
        res = {}
        for arm in ("padded", "packed"):
            res[arm] = {"fwd_ms": ms[f"{arm}_fwd"], "fwdbwd_ms": ms[f"{arm}_fwdbwd"],
                        "fwd_tflops": fl["fwd"] / (ms[f"{arm}_fwd"] * 1e-3) / 1e12,
                        "fwdbwd_tflops": fl["fwdbwd"] / (ms[f"{arm}_fwdbwd"] * 1e-3) / 1e12}
        res["speedup_fwdbwd"] = ms["padded_fwdbwd"] / ms["packed_fwdbwd"]
        res["real_rows"] = N
        del q, k, v, dout, pq, pk, pv, pdout
        torch.cuda.empty_cache()
        return res

    lens = lengths()
    pad_frac = 1.0 - sum(lens) / (B * T_MAX)
    attn = attention_arms(lens)
    control = attention_arms([T_MAX] * B)
    layer = decoder_layer_arms(lens, alternate, max(args.steps // 5, 3), dev)
    line = {"metric": "padding-free fine-tuning: padded [8, 2048] vs packed, same examples", "unit": "ms",
            "gpu": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit_w(0), "lengths": lens,
            "lengths_note": "synthetic: seeded draw from [128, 2048], no dataset here", "padding_fraction": pad_frac,
            "timing": "CUDA events, median of 5 rounds, arms alternating", "flops": "causal floor fwd 4*H*128*sum len(len+1)/2, bwd 2.5x",
            "attention": attn, "attention_no_padding_control": control, "decoder_layer": layer, "impl": "aria_b200"}
    print(json.dumps(line), flush=True)


def decoder_layer_arms(lens, alternate, iters, dev):
    """transformers' AriaTextDecoderLayer (Aria's text config) with the trainable MoE seam and the attention seam: forward +
    backward of the eight examples, padded [8, 2048] with the 2-D padding mask vs one packed row with restarting positions."""
    import torch
    from transformers.models.aria.configuration_aria import AriaTextConfig
    from transformers.models.aria.modeling_aria import AriaTextDecoderLayer, AriaTextRotaryEmbedding

    from aria_b200 import hf_attention, install

    cfg = AriaTextConfig(hidden_size=2560, intermediate_size=1664, num_hidden_layers=1, num_attention_heads=20,
                         num_key_value_heads=20, head_dim=128, max_position_embeddings=65536, rms_norm_eps=1e-6,
                         rope_parameters={"rope_type": "default", "rope_theta": 5e6}, moe_num_experts=64, moe_topk=6,
                         moe_num_shared_experts=2, vocab_size=100352)
    cfg._attn_implementation = hf_attention.register()
    torch.manual_seed(0)
    layer = AriaTextDecoderLayer(cfg, layer_idx=0)
    g = torch.Generator().manual_seed(0)
    with torch.no_grad():
        for p in layer.parameters():
            p.copy_(torch.randn(p.shape, generator=g) * 0.02 if p.dim() > 1 else torch.ones(p.shape))   # norms: 1
    layer = layer.to(dev, torch.bfloat16).train()
    assert install.install(torch.nn.ModuleList([layer]), trainable=True) == 1
    rope = AriaTextRotaryEmbedding(cfg).to(dev)
    N, d = sum(lens), cfg.hidden_size
    x = torch.randn(B, T_MAX, d, generator=g).bfloat16().to(dev)
    gout = torch.randn(B, T_MAX, d, generator=g).bfloat16().to(dev)
    am = torch.zeros(B, T_MAX, dtype=torch.long, device=dev)
    for b, m in enumerate(lens):
        am[b, :m] = 1
    pos = torch.arange(T_MAX, device=dev)[None].expand(B, T_MAX)
    px = torch.cat([x[b, :m] for b, m in enumerate(lens)])[None].contiguous()
    pgout = torch.cat([gout[b, :m] for b, m in enumerate(lens)])[None].contiguous()
    ppos = torch.cat([torch.arange(m, device=dev) for m in lens])[None]

    def step(h, mask, position_ids, grad, seam_positions=True):
        for p in layer.parameters():
            p.grad = None
        hg = h.detach().requires_grad_(True)
        pe = rope(hg, position_ids)
        out = layer(hg, attention_mask=mask, position_ids=position_ids if seam_positions else None, position_embeddings=pe)
        out = out[0] if isinstance(out, tuple) else out
        out.backward(grad)

    # the cost of the seam's packing check on an unpacked batch: with no mask and position_ids given, the seam reads
    # position_ids to the host once per distinct tensor (once per model forward).  A fresh tensor every step forces that read
    # into every step; the other arm hands the attention no position_ids (nothing to read, same arithmetic).
    ms = alternate({"padded": lambda: step(x, am, pos, gout), "packed": lambda: step(px, None, ppos, pgout),
                    "unpadded_position_read": lambda: step(x, None, pos.clone(), gout),
                    "unpadded_no_read": lambda: step(x, None, pos, gout, seam_positions=False)}, iters)
    return {"padded_ms": ms["padded"], "packed_ms": ms["packed"], "real_tokens": N,
            "padded_real_tokens_per_s": N / (ms["padded"] * 1e-3), "packed_real_tokens_per_s": N / (ms["packed"] * 1e-3),
            "speedup": ms["padded"] / ms["packed"],
            "unpadded_8x2048_ms": {"position_ids_read_every_step": ms["unpadded_position_read"],
                                   "no_read": ms["unpadded_no_read"],
                                   "read_cost_ms": ms["unpadded_position_read"] - ms["unpadded_no_read"]}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="calls per timed round (attention; the layer runs a fifth of them)")
    ap.add_argument("--warmup", type=int, default=3)
    run(ap.parse_args())


if __name__ == "__main__":
    main()
