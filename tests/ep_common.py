"""Shared helpers for the expert-parallel tests (CPU/gloo and GPU/nccl)."""
import os
import socket

import torch


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class OracleBackend:
    """TEST-ONLY compute backend for ExpertParallelMoE: the oracle's CPU functions, so the host-side exchange logic
    (counts all-to-all, split sizes, (source rank, expert) grouping, reverse exchange) runs under gloo without a GPU."""

    def __init__(self, k):
        self.k = k

    def router(self, x, w_router, k):
        from oracle import aria_oracle as O
        s, i, c = O.router_routing(O.router_gating(x, w_router), k)
        return s, i, c

    def permute(self, x, idx, counts):
        from oracle import aria_oracle as O
        perm, order = O.token_permutation(x, idx, self.k)
        return perm, order

    def grouped_mlp(self, rows, fc1, fc2, group_counts, n_local_experts):
        from oracle import aria_oracle as O
        out = torch.zeros(rows.shape[0], fc2.shape[-1], dtype=rows.dtype)
        off = 0
        for g, n in enumerate(group_counts.tolist()):
            if n:
                e = g % n_local_experts
                h = O.glu(rows[off:off + n] @ fc1[e])
                out[off:off + n] = h @ fc2[e]
            off += n
        return out

    def shared(self, x, gate_w, up_w, down_w):
        from oracle import aria_oracle as O
        return O.shared_expert_mlp(x, gate_w, up_w, down_w)

    def combine(self, y, order, scores, shared):
        from oracle import aria_oracle as O
        return O.token_unpermutation(y, order, scores, self.k) + shared


def ep_worker(rank, world, port, backend_name, device_kind, tc, T, dtype_name, result_dir):
    """One rank: EP forward vs the single-device layer on this rank's tokens. Writes max error to result_dir."""
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    import torch.distributed as dist
    from aria_b200.expert_parallel import ExpertParallelMoE
    from oracle import aria_oracle as O
    from oracle import configs as C

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.set_grad_enabled(False)
    dtype = getattr(torch, dtype_name)
    if device_kind == "cuda":
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
        dev = torch.device("cuda", rank)
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
        dev = torch.device("cpu")
    gen = torch.Generator().manual_seed(1234)
    full = {k: v.to(dtype) for k, v in C.moe_layer_state(tc, gen).items()}
    xg = torch.Generator().manual_seed(100 + rank)
    x = torch.randn(T + 3 * rank, tc["hidden_size"], generator=xg).to(dtype)  # ragged: ranks own different token counts
    want, parts = O.moe_layer(x, full, tc["moe_topk"], return_parts=True)
    shard = {k: v.to(dev) for k, v in ExpertParallelMoE.shard_state(full, rank, world).items()}
    backend = OracleBackend(tc["moe_topk"]) if backend_name == "oracle" else None
    transport = None
    if backend_name == "fused":
        from aria_b200.expert_parallel import FusedPeerTransport
        transport = FusedPeerTransport(T + 3 * world, tc["hidden_size"], tc["moe_intermediate_size"], tc["moe_num_experts"],
                                       tc["moe_topk"], dev)
    ep = ExpertParallelMoE(shard, tc["moe_num_experts"], tc["moe_topk"], backend=backend, transport=transport)
    got = ep(x.to(dev)).float().cpu()
    if backend_name == "fused":  # a second layer through the same arena (buffer reuse across layers) must agree too
        got2 = ep(x.to(dev)).float().cpu()
        assert torch.equal(got, got2)
    if device_kind == "cuda":
        torch.cuda.synchronize()
    lg = parts["logits"].float().sort(1, descending=True).values
    k = tc["moe_topk"]
    safe = (lg[:, k - 1] - lg[:, k]) / lg.abs().amax(1) > 2 ** -6
    err = (got - want.float()).abs().amax(-1)
    scale = float(want.float().abs().max())
    torch.save({"err_safe": float(err[safe].max()) / scale, "err_all": float(err.max()) / scale,
                "n_safe": int(safe.sum()), "n": int(safe.numel())}, os.path.join(result_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def ep_train_worker(rank, world, port, tc, T, result_dir):
    """One rank: expert-parallel MoE forward+backward (CUDA/NCCL) vs fp32 autograd through the oracle on the CONCATENATED
    batch of all ranks (expert weight grads sum over every rank's tokens)."""
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    import torch.distributed as dist
    from aria_b200.expert_parallel import ExpertParallelMoE, ep_moe_layer_train
    from oracle import aria_oracle as O
    from oracle import configs as C

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    k, d, E = tc["moe_topk"], tc["hidden_size"], tc["moe_num_experts"]
    gen = torch.Generator().manual_seed(1234)
    full = {n: v.bfloat16() for n, v in C.moe_layer_state(tc, gen).items()}
    xs, gs = [], []
    for r in range(world):
        xg = torch.Generator().manual_seed(100 + r)
        xs.append(torch.randn(T + 3 * r, d, generator=xg).bfloat16())
        gs.append(torch.randn(T + 3 * r, d, generator=xg).bfloat16())
    # reference: fp32 autograd over all ranks' tokens
    sd32 = {n: v.float().requires_grad_(True) for n, v in full.items()}
    xall = torch.cat(xs).float().requires_grad_(True)
    with torch.enable_grad():
        want, parts = O.moe_layer(xall, sd32, k, return_parts=True)
        want.backward(torch.cat(gs).float())
    lo = sum(x.shape[0] for x in xs[:rank])
    hi = lo + xs[rank].shape[0]
    # ours
    shard = {n: v.to(dev).requires_grad_(True) for n, v in ExpertParallelMoE.shard_state(full, rank, world).items()}
    xr = xs[rank].to(dev).requires_grad_(True)
    with torch.enable_grad():
        got = ep_moe_layer_train(xr, shard, k)
        got.backward(gs[rank].to(dev))
    torch.cuda.synchronize()

    def rel(a, b):
        a, b = a.float().cpu(), b.float().cpu()
        return float((a - b).norm() / b.norm().clamp_min(1e-12))

    lg = parts["logits"].detach().float().sort(1, descending=True).values
    safe_all = (lg[:, k - 1] - lg[:, k]) / lg.abs().amax(1) > 2 ** -6
    safe = safe_all[lo:hi]
    E_loc = E // world
    e0, e1 = rank * E_loc, (rank + 1) * E_loc
    res = {"out": rel(got.detach()[safe], want.detach()[lo:hi][safe]), "dx": rel(xr.grad[safe], xall.grad[lo:hi][safe]),
           "d_fc1": rel(shard["experts.fc1.weight"].grad, sd32["experts.fc1.weight"].grad[e0:e1]),
           "d_fc2": rel(shard["experts.fc2.weight"].grad, sd32["experts.fc2.weight"].grad[e0:e1]),
           "all_safe": bool(safe_all.all()), "n_safe": int(safe.sum()), "n": int(safe.numel())}
    torch.save(res, os.path.join(result_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()
