"""Expert parallelism for the MoE block (BASELINE.json configs[4], SURVEY.md §8e).

The reference has no EP: its `TokenDispatcher` is Megatron's all-to-all dispatcher with the communication stripped
(aria/model/moe_lm.py:296-365).  Here experts are block-partitioned over the W ranks of one NVSwitch box (rank r owns
experts [r*E/W, (r+1)*E/W) — a pure dim-0 slice of the HF `experts.fc1/fc2.weight`), tokens stay data-parallel, and
each MoE layer does

    router (local) -> stable sort by expert (= by destination rank) -> all-to-all of per-(rank,expert) counts
    -> all-to-all-v of rows (dispatch) -> grouped expert MLP over rows grouped by (source rank, local expert)
    -> reverse all-to-all-v (combine) -> score-weighted sum + local shared expert

over `torch.distributed` (NCCL on NVLink 5 / NVSwitch: uniform bandwidth, so a flat all-to-all).  The grouped GEMM takes
the (source rank, local expert) groups directly (`group_mod`), so received rows are never re-sorted.  Inference forward
(`ExpertParallelMoE`) and training forward+backward (`ep_moe_layer_train`); one 4*E-byte D2H of the counts per layer is needed because NCCL's all-to-all-v takes host split sizes.

Parity: the W-rank result equals the single-device `MoELayer` on each rank's tokens (tests/test_ep_gloo.py on CPU
through the oracle backend, tests/test_gpu_ep.py on 2 GPUs).
"""
from __future__ import annotations

from typing import List

import torch
import torch.distributed as dist


class CudaBackend:
    """The product compute backend: our CUDA kernels through aria_b200.ops."""

    def router(self, x, w_router, k):
        from . import ops
        scores, idx, counts, _ = ops.router_topk(x, w_router, k)
        return scores, idx, counts

    def permute(self, x, idx, counts):
        from . import ops
        offsets, dest, src = ops.build_permutation(idx, counts)
        return ops.permute_rows(x, src), dest

    def grouped_mlp(self, rows, fc1, fc2, group_counts, n_local_experts):
        """rows grouped by (source rank, local expert); group_counts: int64 [W*E_loc] on the rows' device."""
        from . import ops
        off = ops.offsets_from_counts(group_counts)
        h = ops.grouped_gemm(rows, fc1, off, swiglu=True, group_mod=n_local_experts)
        return ops.grouped_gemm(h, fc2, off, group_mod=n_local_experts)

    def shared(self, x, gate_w, up_w, down_w):
        from . import ops
        return ops.linear(ops.linear_swiglu(x, gate_w, up_w), down_w)

    def combine(self, y, dest, scores, shared):
        from . import ops
        return ops.unpermute_combine(y, dest, scores, shared)


def exchange_plan(counts: torch.Tensor, group, row_align: int = 1):
    """The NCCL exchange plan of one layer from my per-expert row counts [E] (rows sorted by global expert id, so by
    destination rank): all-to-all of the per-(rank, local expert) counts, then the one host sync per layer (NCCL's
    all-to-all-v takes host split sizes).  row_align > 1: every expert block is sent padded to a multiple of it (the
    training layout, so the received groups stay 16-aligned).  Returns (recv_counts int64 [W*E_loc] on the counts'
    device, groups ordered (source rank, local expert); rows sent to each rank; rows received from each rank)."""
    send_counts = counts.to(torch.int64)
    if row_align > 1:
        send_counts = (send_counts + row_align - 1) // row_align * row_align
    send_counts = send_counts.view(dist.get_world_size(group), -1)
    recv_counts = torch.empty_like(send_counts)
    dist.all_to_all_single(recv_counts, send_counts, group=group)
    return recv_counts.reshape(-1), send_counts.sum(1).tolist(), recv_counts.sum(1).tolist()


def exchange_rows(rows: torch.Tensor, plan, group, back: bool = False, out=None) -> torch.Tensor:
    """All-to-all-v of rows along `plan` (from `exchange_plan`).  Forward: the first rows the plan sends (expert order) go
    to the owners of their experts; returns the received rows, grouped (source rank, local expert).  back=True: the
    reverse, rows laid out as received go back to their source ranks, into the first rows of `out` (the rows past them,
    e.g. zeroed pads, are left as they are); returns `out`."""
    _, send, recv = plan
    if back:
        dist.all_to_all_single(out[:sum(send)], rows, output_split_sizes=send, input_split_sizes=recv, group=group)
        return out
    out = torch.empty((sum(recv), rows.shape[1]), dtype=rows.dtype, device=rows.device)
    dist.all_to_all_single(out, rows[:sum(send)], output_split_sizes=recv, input_split_sizes=send, group=group)
    return out


class ExpertParallelMoE:
    """Expert-parallel `MoELayer.forward` (moe_lm.py:548-577) for one layer.

    weights: dict with the reference parameter names; `experts.fc1.weight` / `experts.fc2.weight` hold ONLY this rank's
    slice [E/W, ...]; router and shared-expert weights are replicated."""

    def __init__(self, weights: dict, num_experts: int, topk: int, group=None, backend=None, transport=None):
        """transport: a `FusedPeerTransport` -> the exchange runs over NVLink peer memory with our own kernels (fused
        permute+dispatch, device-side barriers, no host sync); None -> NCCL all-to-all-v (needs one host sync)."""
        self.transport = transport
        self.w = weights
        self.E = num_experts
        self.k = topk
        self.group = group
        self.W = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        assert self.E % self.W == 0
        self.E_loc = self.E // self.W
        assert weights["experts.fc1.weight"].shape[0] == self.E_loc
        self.backend = backend or CudaBackend()

    @staticmethod
    def shard_state(full: dict, rank: int, world: int) -> dict:
        """Slice a full MoELayer state dict for `rank` (experts on dim 0; everything else replicated)."""
        E = full["experts.fc1.weight"].shape[0]
        lo, hi = rank * E // world, (rank + 1) * E // world
        out = dict(full)
        out["experts.fc1.weight"] = full["experts.fc1.weight"][lo:hi].contiguous()
        out["experts.fc2.weight"] = full["experts.fc2.weight"][lo:hi].contiguous()
        return out

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.transport is not None:
            return _ep_forward_fused(self, x)
        shape = x.shape
        x2 = x.reshape(-1, shape[-1])
        be = self.backend
        scores, idx, counts = be.router(x2, self.w["router.weight"], self.k)
        permuted, dest = be.permute(x2, idx, counts)  # rows sorted by global expert id == by destination rank
        plan = exchange_plan(counts, self.group)
        recv_rows = exchange_rows(permuted, plan, self.group)
        # shared expert is local work that overlaps with the exchange on the GPU (separate NCCL stream)
        shared = be.shared(x2, self.w["shared_experts.gate_proj.weight"], self.w["shared_experts.up_proj.weight"],
                           self.w["shared_experts.down_proj.weight"])
        y_recv = be.grouped_mlp(recv_rows, self.w["experts.fc1.weight"], self.w["experts.fc2.weight"], plan[0], self.E_loc)
        y = exchange_rows(y_recv, plan, self.group, back=True, out=torch.empty_like(permuted))
        return be.combine(y, dest, scores, shared).view(shape)

    __call__ = forward


class FusedPeerTransport:
    """NVLink peer-memory exchange (csrc/ep.cu): fixed-capacity receive regions, the dispatch fused into the permute
    kernel, the return path fused into the fc2 GEMM epilogue, two device-side barriers per layer, no host sync, CUDA-graph
    friendly.  Arena of every rank (mapped by all peers):

        meta_counts [W*E_loc] int32 | meta_row0 [W*E_loc] int32 | flags [W] int32
        | recv_x [E_loc*W][cap][d] bf16 (region el * W + s = rows rank s routed to my expert el) | ret_y [T_max*k][d] bf16

    cap = T_max rounded up to 16 (+16 for the training layout's alignment pads): a token picks an expert at most once."""

    def __init__(self, T_max: int, hidden: int, inter: int, num_experts: int, topk: int, device, group=None):
        from .peer import PeerArena
        self.group = group
        self.W = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.E, self.k, self.d = num_experts, topk, hidden
        self.E_loc = num_experts // self.W
        self.G = self.W * self.E_loc
        self.cap = (T_max + 15) // 16 * 16 + 16
        self.ret_rows = T_max * topk + num_experts * 15
        al = lambda n: (n + 1023) // 1024 * 1024
        self.off_counts = 0
        self.off_row0 = al(self.G * 4)
        self.off_flags = self.off_row0 + al(self.G * 4)
        self.off_recv = self.off_flags + al(self.W * 4)
        self.off_ret = self.off_recv + al(self.G * self.cap * hidden * 2)
        total = self.off_ret + al(self.ret_rows * hidden * 2)
        self.arena = PeerArena(total, device, group)
        dev = torch.device(device)
        mk = lambda off: torch.tensor([self.arena.ptr(r, off) for r in range(self.W)], dtype=torch.int64, device=dev)
        self.p_counts, self.p_row0, self.p_flags = mk(self.off_counts), mk(self.off_row0), mk(self.off_flags)
        self.p_recv, self.p_ret = mk(self.off_recv), mk(self.off_ret)
        self.meta_counts = self.arena.local_view(self.off_counts, (self.G,), torch.int32)
        self.meta_row0 = self.arena.local_view(self.off_row0, (self.G,), torch.int32)
        self.recv_x = self.arena.local_view(self.off_recv, (self.G * self.cap, hidden), torch.bfloat16)
        self.ret_y = self.arena.local_view(self.off_ret, (self.ret_rows, hidden), torch.bfloat16)
        self.starts = (torch.arange(self.G, dtype=torch.int32) * self.cap).to(dev)
        # group g = (local expert g // W, source rank g % W): its outputs go back into rank s's ret_y
        self.out_base = self.p_ret.repeat(self.E_loc).contiguous()
        self.h_buf = torch.empty((self.G * self.cap, inter), dtype=torch.bfloat16, device=dev)
        self.epoch = torch.zeros(1, dtype=torch.int32, device=dev)
        self.device = dev

    def barrier(self):
        from . import _lib as L
        import ctypes as C
        with torch.cuda.device(self.device):
            L.check(L.load().aria_peer_barrier(C.c_void_p(self.p_flags.data_ptr()), self.rank, self.W,
                                               C.c_void_p(self.epoch.data_ptr()),
                                               C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)), "peer_barrier")


def _ep_forward_fused(self, x: torch.Tensor) -> torch.Tensor:
    """ExpertParallelMoE.forward on the fused exchange: 2 barriers + 0 copy kernels on top of the single-GPU launch sequence."""
    import ctypes as C
    from . import _lib as L
    from . import ops
    tr = self.transport
    lib = L.load()
    shape = x.shape
    x2 = x.reshape(-1, shape[-1]).contiguous()
    T = x2.shape[0]
    assert T <= tr.cap - 16 and T * self.k <= tr.ret_rows, "FusedPeerTransport was sized for fewer tokens"
    stream = C.c_void_p(torch.cuda.current_stream(x2.device).cuda_stream)
    vp = lambda t: C.c_void_p(t.data_ptr())
    from .moe_lm import join_side, shared_expert_overlapped
    # the local shared expert runs as a parallel branch (side stream) while rows are in flight and experts compute
    forked = shared_expert_overlapped(
        lambda: ops.linear(ops.linear_swiglu(x2, self.w["shared_experts.gate_proj.weight"],
                                             self.w["shared_experts.up_proj.weight"]), self.w["shared_experts.down_proj.weight"]), x2)
    scores, idx, counts, _ = ops.router_topk(x2, self.w["router.weight"], self.k)
    offsets, dest, src = ops.build_permutation(idx, counts)
    with torch.cuda.device(x2.device):
        # fused permute + dispatch over NVLink, and my per-block (count, first sorted row) into the owners' meta arrays
        L.check(lib.aria_ep_dispatch(vp(x2), vp(src), vp(offsets), vp(tr.p_recv), vp(tr.p_counts), vp(tr.p_row0), tr.rank, tr.W,
                                     tr.E, tr.cap, tr.d, T * self.k, stream), "ep_dispatch")
    tr.barrier()
    ops.grouped_gemm_regions(tr.recv_x, self.w["experts.fc1.weight"], tr.starts, tr.meta_counts, T * self.k, swiglu=True,
                             group_mod=-tr.W, out=tr.h_buf)
    # fc2: every output row is stored by the GEMM epilogue straight into its SOURCE rank's combine buffer (the return all-to-all)
    ops.grouped_gemm_regions(tr.h_buf, self.w["experts.fc2.weight"], tr.starts, tr.meta_counts, T * self.k, group_mod=-tr.W,
                             out_group_base=tr.out_base, out_group_row0=tr.meta_row0, ldo=tr.d)
    tr.barrier()
    shared = join_side(forked, x2)
    return ops.unpermute_combine(tr.ret_y, dest, scores, shared).view(shape)


def exchange_bytes_per_layer(tokens_per_rank: int, topk: int, hidden: int, world: int) -> float:
    """Expected bytes a rank sends per direction per layer: (W-1)/W of its k*T rows leave the rank (SURVEY.md §8e)."""
    return tokens_per_rank * topk * hidden * 2 * (world - 1) / world


def ep_moe_layer_train(x, w: dict, topk: int, group=None):
    """Differentiable expert-parallel MoE layer (BASELINE cfg 5): `moe_train.MoELayerFunction` over `group` (default: the
    world), eval-mode routing; `w` as in ExpertParallelMoE (expert weights = this rank's slice)."""
    from .moe_train import MoELayerFunction
    return MoELayerFunction.apply(x, w["router.weight"], w["experts.fc1.weight"], w["experts.fc2.weight"],
                                  w["shared_experts.gate_proj.weight"], w["shared_experts.up_proj.weight"],
                                  w["shared_experts.down_proj.weight"], topk, None, None,
                                  dist.group.WORLD if group is None else group)
