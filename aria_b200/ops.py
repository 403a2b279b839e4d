"""Torch-facing wrappers over the C ABI: tensors in, tensors out, raw pointers underneath.

PyTorch is used for device memory and streams only; every computation below is one of our CUDA kernels.
All wrappers launch on the current stream of the input's device and never synchronise.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import gc
from typing import Optional, Sequence

import torch

from . import _lib as L

bf16 = torch.bfloat16


def _p(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream(t: torch.Tensor):
    return C.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


@contextlib.contextmanager
def graph_capture(graph: torch.cuda.CUDAGraph, pool=None):
    """torch.cuda.graph(graph, pool) with Python's garbage collector paused.  A collection during the capture can run the
    destructor of a dead object that holds CUDA resources (another CUDA graph, its memory pool), whose release is not
    allowed while a stream captures, and the process aborts; torch.cuda.graph no longer collects before it captures.
    The garbage is collected after the capture instead."""
    enabled = gc.isenabled()
    gc.disable()
    try:
        with torch.cuda.graph(graph, pool=pool):
            yield
    finally:
        if enabled:
            gc.enable()


def _chk(t: torch.Tensor, dtype=bf16, align: int = 16):
    if not t.is_cuda:
        raise RuntimeError("aria_b200 ops need CUDA tensors (there is no CPU path)")
    if t.dtype != dtype:
        raise RuntimeError(f"expected {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise RuntimeError("expected a contiguous tensor")
    if t.data_ptr() % align:
        raise RuntimeError(f"expected {align}-byte aligned storage")
    return t


# ------------------------------------------------------------------------------------------- GEMMs
def _run_gemm(d: L.GemmDesc, ref: torch.Tensor, what: str):
    with torch.cuda.device(ref.device):
        L.check(L.load().aria_gemm(C.byref(d), _stream(ref)), what)


def linear(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None, act: int = L.ACT_NONE,
           residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """F.linear(x, weight, bias) -> act -> (+ residual); x [..., K], weight [N, K] (nn.Linear layout)."""
    _chk(x), _chk(weight)
    K = x.shape[-1]
    N = weight.shape[0]
    x2 = x.reshape(-1, K)
    M = x2.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=bf16, device=x.device)
    d = L.GemmDesc()
    d.a, d.lda, d.m, d.n, d.k = x2.data_ptr(), K, M, N, K
    d.b[0] = weight.data_ptr()
    d.n_seg, d.b_layout, d.num_groups = 1, L.B_NK, 1
    d.epilogue, d.act = L.EPI_LINEAR, act
    if bias is not None:
        d.bias[0] = _chk(bias).data_ptr()
    if residual is not None:
        r2 = _chk(residual).reshape(-1, N)
        d.residual, d.ldr = r2.data_ptr(), N
    d.out[0], d.ldo = out.data_ptr(), N
    _run_gemm(d, x, "linear")
    return out.view(*x.shape[:-1], N)


def linear_multi(x: torch.Tensor, weights: Sequence[torch.Tensor]) -> torch.Tensor:
    """[x @ W0.T | x @ W1.T | ...] in one GEMM launch (up to 3 nn.Linear weights with equal out_features)."""
    _chk(x)
    K = x.shape[-1]
    N = weights[0].shape[0]
    x2 = x.reshape(-1, K)
    M = x2.shape[0]
    out = torch.empty((M, N * len(weights)), dtype=bf16, device=x.device)
    d = L.GemmDesc()
    d.a, d.lda, d.m, d.n, d.k = x2.data_ptr(), K, M, N, K
    for s_, w in enumerate(weights):
        _chk(w)
        assert w.shape == weights[0].shape
        d.b[s_] = w.data_ptr()
    d.n_seg, d.b_layout, d.num_groups = len(weights), L.B_NK, 1
    d.epilogue = L.EPI_LINEAR
    d.out[0], d.ldo = out.data_ptr(), N * len(weights)
    _run_gemm(d, x, "linear_multi")
    return out


def linear_swiglu(x: torch.Tensor, gate_w: torch.Tensor, up_w: torch.Tensor) -> torch.Tensor:
    """silu(x @ gate_w.T) * (x @ up_w.T) in one GEMM (LlamaMLP front half, moe_lm.py:368-395)."""
    _chk(x), _chk(gate_w), _chk(up_w)
    K = x.shape[-1]
    N = gate_w.shape[0]
    x2 = x.reshape(-1, K)
    M = x2.shape[0]
    out = torch.empty((M, N), dtype=bf16, device=x.device)
    d = L.GemmDesc()
    d.a, d.lda, d.m, d.n, d.k = x2.data_ptr(), K, M, N, K
    d.b[0], d.b[1] = gate_w.data_ptr(), up_w.data_ptr()
    d.n_seg, d.b_layout, d.num_groups = 2, L.B_NK, 1
    d.epilogue = L.EPI_SWIGLU
    d.out[0], d.ldo = out.data_ptr(), N
    _run_gemm(d, x, "linear_swiglu")
    return out.view(*x.shape[:-1], N)


def grouped_gemm(a: torch.Tensor, b: torch.Tensor, offsets: torch.Tensor, swiglu: bool = False,
                 group_mod: int = 0, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[off[e]:off[e+1]] = a[off[e]:off[e+1]] @ b[e] (+ residual); b [E, K, N] (GroupedGEMM.weight, moe_lm.py:465).
    swiglu=True fuses `glu` (moe_lm.py:505-507): b has 2I columns, out has I."""
    _chk(a), _chk(b), _chk(offsets, torch.int32)
    rows, K = a.shape
    E, Kb, Nb = b.shape
    G = offsets.numel() - 1  # groups; with group_mod, group g multiplies by weight block g % group_mod
    assert Kb == K and (G == E if not group_mod else (group_mod == E and G % E == 0))
    N = Nb // 2 if swiglu else Nb
    out = torch.empty((rows, N), dtype=bf16, device=a.device)
    d = L.GemmDesc()
    d.a, d.lda, d.m, d.n, d.k = a.data_ptr(), K, rows, N, K
    d.b[0] = b.data_ptr()
    d.n_seg, d.b_layout, d.num_groups = 1, L.B_GKN, G
    d.group_mod = group_mod
    d.group_offsets = offsets.data_ptr()
    d.epilogue = L.EPI_SWIGLU if swiglu else L.EPI_LINEAR
    d.out[0], d.ldo = out.data_ptr(), N
    if residual is not None:
        assert not swiglu and residual.shape == out.shape
        _chk(residual)
        d.residual, d.ldr = residual.data_ptr(), N
    _run_gemm(d, a, "grouped_gemm")
    return out


def quantize_fp8_cols(w: torch.Tensor):
    """Per-(expert, output column) e4m3 quantisation of GroupedGEMM weights w [E, K, N] bf16 -> (q [E, K, N]
    torch.float8_e4m3fn, scale [E, N] fp32): scale = amax over K / 448 (an all-zero column gets 1), q = e4m3(w / scale),
    bit for bit `(w.float() / scale).to(torch.float8_e4m3fn)`."""
    _chk(w)
    if w.dim() != 3:
        raise ValueError(f"expected [E, K, N] expert weights, got {tuple(w.shape)}")
    E, K, N = w.shape
    q = torch.empty((E, K, N), dtype=torch.float8_e4m3fn, device=w.device)
    scale = torch.empty((E, N), dtype=torch.float32, device=w.device)
    with torch.cuda.device(w.device):
        L.check(L.load().aria_quantize_fp8_cols(_p(w), _p(q), _p(scale), E, K, N, _stream(w)), "quantize_fp8_cols")
    return q, scale


def grouped_gemm_fp8(a: torch.Tensor, q: torch.Tensor, scale: torch.Tensor, offsets: torch.Tensor,
                     swiglu: bool = False) -> torch.Tensor:
    """grouped_gemm with e4m3 weights q [E, K, N_b] (float8_e4m3fn) and per-column scales scale [E, N_b] fp32: the fp32
    accumulator of column c of expert e is multiplied by scale[e, c] before the epilogue rounds it.  swiglu=True: N_b = 2I
    (gate then up, each column with its own scale), out [rows, I]."""
    _chk(a), _chk(q, torch.float8_e4m3fn), _chk(scale, torch.float32), _chk(offsets, torch.int32)
    rows, K = a.shape
    E, Kb, Nb = q.shape
    if Kb != K or scale.shape != (E, Nb) or offsets.numel() != E + 1:
        raise ValueError(f"grouped_gemm_fp8: a {tuple(a.shape)}, q {tuple(q.shape)}, scale {tuple(scale.shape)}, "
                         f"offsets {offsets.numel()} do not fit together")
    N = Nb // 2 if swiglu else Nb
    out = torch.empty((rows, N), dtype=bf16, device=a.device)
    with torch.cuda.device(a.device):
        L.check(L.load().aria_grouped_gemm_fp8(_p(a), _p(q), _p(scale), _p(out), _p(offsets), rows, K, N, E,
                                               L.EPI_SWIGLU if swiglu else L.EPI_LINEAR, _stream(a)), "grouped_gemm_fp8")
    return out


def permute_quantize_fp8(x: torch.Tensor, src_token: Optional[torch.Tensor] = None):
    """Per-row e4m3 quantisation of activations x [*, d] bf16, gathered through src_token [rows] int32 when given ->
    (q [rows, d] torch.float8_e4m3fn, scale [rows] fp32): scale = amax of the row / 448 (an all-zero row gets 1),
    q = e4m3(row / scale), bit for bit `(x.float() / scale[:, None]).to(torch.float8_e4m3fn)`."""
    _chk(x)
    if x.dim() != 2:
        raise ValueError(f"expected [rows, d] activations, got {tuple(x.shape)}")
    rows, d = x.shape
    if src_token is not None:
        _chk(src_token, torch.int32, align=4)
        rows = src_token.numel()
    q = torch.empty((rows, d), dtype=torch.float8_e4m3fn, device=x.device)
    scale = torch.empty((rows,), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        L.check(L.load().aria_permute_quantize_fp8_rows(_p(x), _p(src_token), _p(q), _p(scale), rows, d, _stream(x)),
                "permute_quantize_fp8")
    return q, scale


def _kmajor(weight: torch.Tensor) -> torch.Tensor:
    """The [E, N, K] e4m3 buffer behind a W8A8 expert weight, the [E, K, N] parameter's transpose(1, 2) view."""
    if weight.dim() != 3 or not weight.transpose(1, 2).is_contiguous():
        raise ValueError("W8A8 expert weights must be the transpose(1, 2) view of a contiguous [E, N, K] buffer "
                         "(quantize_experts_fp8(activations=\"fp8\"))")
    return _chk(weight.transpose(1, 2), torch.float8_e4m3fn)


def grouped_gemm_w8a8(aq: torch.Tensor, a_scale: torch.Tensor, weight: torch.Tensor, weight_scale: torch.Tensor,
                      offsets: torch.Tensor, swiglu: bool = False) -> torch.Tensor:
    """grouped_gemm with e4m3 activations aq [rows, K] (per-row scales a_scale [rows], permute_quantize_fp8) and e4m3 weights
    weight [E, K, N_b] (K-major storage, see _kmajor) with per-column scales weight_scale [E, N_b]: the fp32 accumulator is
    multiplied by a_scale[row] * weight_scale[e, col] before the epilogue rounds it.  swiglu=True: N_b = 2I, out [rows, I]."""
    _chk(aq, torch.float8_e4m3fn), _chk(a_scale, torch.float32, align=4), _chk(weight_scale, torch.float32)
    _chk(offsets, torch.int32)
    b = _kmajor(weight)
    rows, K = aq.shape
    E, Kb, Nb = weight.shape
    if Kb != K or a_scale.shape != (rows,) or weight_scale.shape != (E, Nb) or offsets.numel() != E + 1:
        raise ValueError(f"grouped_gemm_w8a8: aq {tuple(aq.shape)}, a_scale {tuple(a_scale.shape)}, weight {tuple(weight.shape)}, "
                         f"weight_scale {tuple(weight_scale.shape)}, offsets {offsets.numel()} do not fit together")
    N = Nb // 2 if swiglu else Nb
    out = torch.empty((rows, N), dtype=bf16, device=aq.device)
    with torch.cuda.device(aq.device):
        L.check(L.load().aria_grouped_gemm_w8a8(_p(aq), _p(a_scale), _p(b), _p(weight_scale), _p(out), _p(offsets), rows, K, N, E,
                                                L.EPI_SWIGLU if swiglu else L.EPI_LINEAR, _stream(aq)), "grouped_gemm_w8a8")
    return out


def _run_gemm_w8a8(d: L.GemmDesc, a_scale: torch.Tensor, scales: Sequence[torch.Tensor], ref: torch.Tensor, what: str):
    arr = (C.c_void_p * 3)(*[s.data_ptr() for s in scales], *([None] * (3 - len(scales))))
    with torch.cuda.device(ref.device):
        L.check(L.load().aria_gemm_w8a8(C.byref(d), _p(a_scale), C.cast(arr, C.c_void_p), _stream(ref)), what)


def _w8a8_operands(xq: torch.Tensor, x_scale: torch.Tensor, weights: Sequence[torch.Tensor], scales: Sequence[torch.Tensor],
                   what: str):
    """Checks the e4m3 rows xq [..., K] with row scales x_scale [rows] and the e4m3 nn.Linear weights [N, K] with their
    output-channel scales [N]; returns (xq as [rows, K], rows, N, K)."""
    _chk(xq, torch.float8_e4m3fn), _chk(x_scale, torch.float32, align=4)
    K = xq.shape[-1]
    x2 = xq.reshape(-1, K)
    N = weights[0].shape[0]
    for w, sc in zip(weights, scales):
        _chk(w, torch.float8_e4m3fn), _chk(sc, torch.float32)
        if w.shape != (N, K) or sc.shape != (N,):
            raise ValueError(f"{what}: weight {tuple(w.shape)} / scale {tuple(sc.shape)} do not fit rows of {K} and {N} outputs")
    if x_scale.shape != (x2.shape[0],):
        raise ValueError(f"{what}: x_scale {tuple(x_scale.shape)} does not fit {x2.shape[0]} rows")
    return x2, x2.shape[0], N, K


def linear_w8a8(xq: torch.Tensor, x_scale: torch.Tensor, weight: torch.Tensor, weight_scale: torch.Tensor,
                residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """W8A8 nn.Linear (+ residual): e4m3 rows xq [..., K] with row scales x_scale [rows] (permute_quantize_fp8,
    rmsnorm_quantize_fp8), e4m3 weight [N, K] with output-channel scales weight_scale [N] -> bf16 [..., N].  The fp32 accumulator
    is multiplied by x_scale[row] * weight_scale[col] before the first bf16 rounding; the rest is `linear`'s epilogue."""
    x2, M, N, K = _w8a8_operands(xq, x_scale, [weight], [weight_scale], "linear_w8a8")
    out = torch.empty((M, N), dtype=bf16, device=xq.device)
    d = L.GemmDesc()
    d.a, d.lda, d.m, d.n, d.k = x2.data_ptr(), K, M, N, K
    d.b[0] = weight.data_ptr()
    d.n_seg, d.b_layout, d.num_groups = 1, L.B_NK, 1
    d.epilogue = L.EPI_LINEAR
    if residual is not None:
        r2 = _chk(residual).reshape(-1, N)
        d.residual, d.ldr = r2.data_ptr(), N
    d.out[0], d.ldo = out.data_ptr(), N
    _run_gemm_w8a8(d, x_scale, [weight_scale], xq, "linear_w8a8")
    return out.view(*xq.shape[:-1], N)


def linear_swiglu_w8a8(xq: torch.Tensor, x_scale: torch.Tensor, gate_w: torch.Tensor, gate_scale: torch.Tensor,
                       up_w: torch.Tensor, up_scale: torch.Tensor) -> torch.Tensor:
    """linear_swiglu with e4m3 operands (see linear_w8a8): silu(gate) * up, each accumulator scaled before rounding."""
    x2, M, N, K = _w8a8_operands(xq, x_scale, [gate_w, up_w], [gate_scale, up_scale], "linear_swiglu_w8a8")
    out = torch.empty((M, N), dtype=bf16, device=xq.device)
    d = L.GemmDesc()
    d.a, d.lda, d.m, d.n, d.k = x2.data_ptr(), K, M, N, K
    d.b[0], d.b[1] = gate_w.data_ptr(), up_w.data_ptr()
    d.n_seg, d.b_layout, d.num_groups = 2, L.B_NK, 1
    d.epilogue = L.EPI_SWIGLU
    d.out[0], d.ldo = out.data_ptr(), N
    _run_gemm_w8a8(d, x_scale, [gate_scale, up_scale], xq, "linear_swiglu_w8a8")
    return out.view(*xq.shape[:-1], N)


def qkv_heads_w8a8(xq: torch.Tensor, x_scale: torch.Tensor, weights: Sequence[torch.Tensor], scales: Sequence[torch.Tensor],
                   outs: Sequence[torch.Tensor], head_dim: int, rows_per_batch: int, pos0: int = 0, rope_mask: int = 0,
                   rope_cos: Optional[torch.Tensor] = None, rope_sin: Optional[torch.Tensor] = None,
                   position_ids: Optional[torch.Tensor] = None):
    """qkv_heads with e4m3 operands (see linear_w8a8): the q/k/v projections of xq, RoPE, scattered head-major."""
    x2, M, N, K = _w8a8_operands(xq, x_scale, weights, scales, "qkv_heads_w8a8")
    d = L.GemmDesc()
    d.a, d.lda, d.m, d.n, d.k = x2.data_ptr(), K, M, N, K
    d.n_seg, d.b_layout, d.num_groups = len(weights), L.B_NK, 1
    d.epilogue = L.EPI_HEADS
    o0 = outs[0]
    for s, (w, o) in enumerate(zip(weights, outs)):
        _chk(o)
        assert o.shape[1:] == o0.shape[1:] and o.stride() == o0.stride()
        d.b[s] = w.data_ptr()
        d.out[s] = o.data_ptr()
    d.head_dim, d.head_ld = head_dim, o0.shape[-1]
    d.rows_per_batch, d.pos0 = rows_per_batch, pos0
    d.stride_b, d.stride_h = o0.stride(0), o0.stride(1)
    d.rope_mask = rope_mask
    if rope_mask:
        d.rope_cos, d.rope_sin = _chk(rope_cos).data_ptr(), _chk(rope_sin).data_ptr()
    if position_ids is not None:
        d.position_ids = _chk(position_ids, torch.int32).data_ptr()
    _run_gemm_w8a8(d, x_scale, scales, xq, "qkv_heads_w8a8")


def grouped_gemm_regions(a_buf: torch.Tensor, b: torch.Tensor, starts: torch.Tensor, counts: torch.Tensor, rows_hint: int,
                         swiglu: bool = False, group_mod: int = 0, out: Optional[torch.Tensor] = None,
                         out_group_base: Optional[torch.Tensor] = None, out_group_row0: Optional[torch.Tensor] = None,
                         ldo: Optional[int] = None) -> Optional[torch.Tensor]:
    """Grouped GEMM over FIXED-CAPACITY row regions (expert parallelism, csrc/ep.cu): group g = rows
    [starts[g], starts[g] + counts[g]) of `a_buf`, multiplied by weight block g % group_mod (group_mod > 0) or g // -group_mod (< 0).  `counts` may be written by peer
    GPUs (it is read on the device at launch).  rows_hint = expected total rows (tile-shape heuristics only).
    With out_group_base / out_group_row0 the rows of group g are stored at (bf16*)out_group_base[g] + (out_group_row0[g] + r)*ldo
    — e.g. straight into the source rank's combine buffer over NVLink — and nothing is returned."""
    _chk(a_buf), _chk(b), _chk(starts, torch.int32, align=4), _chk(counts, torch.int32, align=4)
    cap_rows, K = a_buf.shape
    E, Kb, Nb = b.shape
    G = starts.numel()
    assert Kb == K and counts.numel() == G and (G == E if not group_mod else ((group_mod == E and G % E == 0) if group_mod > 0 else G == E * -group_mod))
    N = Nb // 2 if swiglu else Nb
    d = L.GemmDesc()
    d.a, d.lda, d.m, d.n, d.k = a_buf.data_ptr(), K, max(1, min(rows_hint, cap_rows)), N, K
    d.a_rows = cap_rows
    d.b[0] = b.data_ptr()
    d.n_seg, d.b_layout, d.num_groups = 1, L.B_GKN, G
    d.group_mod = group_mod
    d.group_offsets, d.group_counts = starts.data_ptr(), counts.data_ptr()
    d.epilogue = L.EPI_SWIGLU if swiglu else L.EPI_LINEAR
    if out_group_base is not None:
        assert not swiglu and out_group_row0 is not None and ldo is not None
        _chk(out_group_base, torch.int64, align=8), _chk(out_group_row0, torch.int32, align=4)
        d.out_group_base, d.out_group_row0 = out_group_base.data_ptr(), out_group_row0.data_ptr()
        d.out[0], d.ldo = a_buf.data_ptr(), ldo      # out[0] is never dereferenced on this path (must be non-NULL)
        ret = None
    else:
        if out is None:
            out = torch.empty((cap_rows, N), dtype=bf16, device=a_buf.device)
        _chk(out)
        assert out.shape == (cap_rows, N)
        d.out[0], d.ldo = out.data_ptr(), N
        ret = out
    _run_gemm(d, a_buf, "grouped_gemm")
    return ret


def grouped_gemm_nt(a: torch.Tensor, b: torch.Tensor, offsets: torch.Tensor, group_mod: int = 0,
                    residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Data-gradient of the grouped GEMM: out[rows of e] = a[rows of e] @ b[e].T (+ residual) with b [E, N_out, K]
    (K contiguous) — i.e. the forward weight [E, in, out] used transposed, read in place (ARIA_B_GNK)."""
    _chk(a), _chk(b), _chk(offsets, torch.int32)
    rows, K = a.shape
    E, N, Kb = b.shape
    G = offsets.numel() - 1
    assert Kb == K and (G == E if not group_mod else (group_mod == E and G % E == 0))
    out = torch.empty((rows, N), dtype=bf16, device=a.device)
    d = L.GemmDesc()
    d.a, d.lda, d.m, d.n, d.k = a.data_ptr(), a.stride(0), rows, N, K
    d.b[0] = b.data_ptr()
    d.n_seg, d.b_layout, d.num_groups = 1, L.B_GNK, G
    d.group_mod = group_mod
    d.group_offsets = offsets.data_ptr()
    d.epilogue = L.EPI_LINEAR
    d.out[0], d.ldo = out.data_ptr(), N
    if residual is not None:
        assert residual.shape == out.shape
        _chk(residual)
        d.residual, d.ldr = residual.data_ptr(), N
    _run_gemm(d, a, "grouped_gemm_nt")
    return out


def matmul_kn(a: torch.Tensor, w_kn: torch.Tensor, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """a [M, K] (row stride may exceed K) @ w_kn [K, N] (N contiguous) (+ residual): dense data-gradients, where the
    nn.Linear weight [out, in] = [K, N] is consumed in place through the MN-major B path."""
    if not (a.is_cuda and a.dtype == bf16 and a.stride(1) == 1 and a.data_ptr() % 16 == 0):
        raise RuntimeError("matmul_kn: a must be CUDA bf16 with contiguous rows")
    _chk(w_kn)
    M, K = a.shape
    Kw, N = w_kn.shape
    assert K == Kw
    out = torch.empty((M, N), dtype=bf16, device=a.device)
    off = torch.tensor([0, M], dtype=torch.int32, device=a.device)
    d = L.GemmDesc()
    d.a, d.lda, d.m, d.n, d.k = a.data_ptr(), a.stride(0), M, N, K
    d.b[0] = w_kn.data_ptr()
    d.n_seg, d.b_layout, d.num_groups = 1, L.B_GKN, 1
    d.group_offsets = off.data_ptr()
    d.epilogue = L.EPI_LINEAR
    if residual is not None:
        d.residual, d.ldr = _chk(residual).data_ptr(), N
    d.out[0], d.ldo = out.data_ptr(), N
    _run_gemm(d, a, "matmul_kn")
    return out


def grouped_wgrad(a: torch.Tensor, b: torch.Tensor, offsets: torch.Tensor, num_sources: int = 1) -> torch.Tensor:
    """out[g] = a[rows of g].T @ b[rows of g]; a [rows, Md], b [rows, Nd] (row strides allowed), offsets [G+1] int32,
    non-decreasing, any alignment (16-aligned groups take no extra work) -> out [G, Md, Nd] bf16 (fp32 accumulation); an
    empty group gives zeros.  num_sources=S: offsets [S*G+1] over (source, g) row groups, out[g] sums over the sources."""
    for t in (a, b):
        if not (t.is_cuda and t.dtype == bf16 and t.stride(1) == 1 and t.data_ptr() % 16 == 0):
            raise RuntimeError("grouped_wgrad: operands must be CUDA bf16 with contiguous rows")
    _chk(offsets, torch.int32)
    rows, Md = a.shape
    Nd = b.shape[1]
    G = (offsets.numel() - 1) // num_sources
    assert G * num_sources + 1 == offsets.numel()
    out = torch.empty((G, Md, Nd), dtype=bf16, device=a.device)
    with torch.cuda.device(a.device):
        L.check(L.load().aria_grouped_wgrad(_p(a), a.stride(0), _p(b), b.stride(0), _p(out), _p(offsets), rows, Md, Nd, G,
                                            num_sources, _stream(a)), "grouped_wgrad")
    return out


def wgrad_accumulate_f32(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out += a.T @ b in fp32, in place; a [rows, Md], b [rows, Nd] bf16 (row strides allowed), out [Md, Nd] fp32 contiguous.
    The weight gradient of nn.Linear built up over chunks of rows without a bf16 rounding per chunk."""
    for t in (a, b):
        if not (t.is_cuda and t.dtype == bf16 and t.stride(1) == 1 and t.data_ptr() % 16 == 0):
            raise RuntimeError("wgrad_accumulate_f32: operands must be CUDA bf16 with contiguous rows")
    _chk(out, torch.float32, align=8)
    rows, Md = a.shape
    Nd = b.shape[1]
    assert b.shape[0] == rows and out.shape == (Md, Nd)
    with torch.cuda.device(a.device):
        L.check(L.load().aria_wgrad_accumulate_f32(_p(a), a.stride(0), _p(b), b.stride(0), _p(out), rows, Md, Nd, _stream(a)),
                "wgrad_accumulate_f32")
    return out


def cross_entropy_rows(logits: torch.Tensor, labels: torch.Tensor, grad_scale: torch.Tensor,
                       loss: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Per-row cross-entropy of bf16 logits [rows, V] (V % 8 == 0, contiguous last dim, row stride a multiple of 8) against
    int64 labels [rows] in [0, V): returns loss [rows] fp32 (logsumexp - logit[label], softmax in fp32) and overwrites each
    logits row IN PLACE with (softmax - onehot(label)) * grad_scale in bf16.  grad_scale: device fp32 [1] (no host sync)."""
    if not (logits.is_cuda and logits.dtype == bf16 and logits.dim() == 2 and logits.stride(1) == 1
            and logits.data_ptr() % 16 == 0):
        raise RuntimeError("cross_entropy_rows: logits must be CUDA bf16 [rows, V] with contiguous, 16-byte aligned rows")
    rows, V = logits.shape
    _chk(labels, torch.int64, align=8), _chk(grad_scale, torch.float32, align=4)
    assert labels.shape == (rows,) and grad_scale.numel() == 1
    if loss is None:
        loss = torch.empty((rows,), dtype=torch.float32, device=logits.device)
    _chk(loss, torch.float32, align=4)
    assert loss.shape == (rows,)
    with torch.cuda.device(logits.device):
        L.check(L.load().aria_cross_entropy_rows(_p(logits), logits.stride(0), _p(labels), _p(grad_scale), _p(loss), rows, V,
                                                 _stream(logits)), "cross_entropy_rows")
    return loss


def swiglu_fwd(h1: torch.Tensor) -> torch.Tensor:
    _chk(h1)
    rows, I2 = h1.shape
    h = torch.empty((rows, I2 // 2), dtype=bf16, device=h1.device)
    with torch.cuda.device(h1.device):
        L.check(L.load().aria_swiglu_fwd(_p(h1), _p(h), rows, I2 // 2, _stream(h1)), "swiglu_fwd")
    return h


def swiglu_bwd(h1: torch.Tensor, dh: torch.Tensor) -> torch.Tensor:
    _chk(h1), _chk(dh)
    rows, I2 = h1.shape
    dh1 = torch.empty_like(h1)
    with torch.cuda.device(h1.device):
        L.check(L.load().aria_swiglu_bwd(_p(h1), _p(dh), _p(dh1), rows, I2 // 2, _stream(h1)), "swiglu_bwd")
    return dh1


def combine_bwd(dout: torch.Tensor, y: torch.Tensor, dest_row: torch.Tensor, scores: torch.Tensor):
    """-> (dy [rows(y), d] bf16 with pad rows zero, dscores [T, k] fp32)."""
    _chk(dout), _chk(y), _chk(dest_row, torch.int32), _chk(scores)
    T, k = scores.shape
    dy = torch.zeros_like(y)
    ds = torch.empty((T, k), dtype=torch.float32, device=y.device)
    with torch.cuda.device(y.device):
        L.check(L.load().aria_combine_bwd(_p(dout), _p(y), _p(dest_row), _p(scores), _p(dy), _p(ds), T, y.shape[1], k,
                                          _stream(y)), "combine_bwd")
    return dy, ds


def router_bwd(dscores: torch.Tensor, scores: torch.Tensor, top_idx: torch.Tensor, E: int) -> torch.Tensor:
    _chk(dscores, torch.float32), _chk(scores), _chk(top_idx, torch.int32)
    T, k = scores.shape
    dl = torch.empty((T, E), dtype=bf16, device=scores.device)
    with torch.cuda.device(scores.device):
        L.check(L.load().aria_router_bwd(_p(dscores), _p(scores), _p(top_idx), _p(dl), T, E, k, _stream(scores)), "router_bwd")
    return dl


def router_aux_loss(logits: torch.Tensor, counts: torch.Tensor, k: int, z_coeff: float, aux_coeff: float) -> torch.Tensor:
    """[z_loss, aux_loss] (fp32) of the training-mode router (moe_lm.py:128-166); values are for logging only."""
    _chk(logits), _chk(counts, torch.int32)
    T, E = logits.shape
    lib = L.load()
    nbytes = lib.aria_router_aux_workspace_bytes(E)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=logits.device)
    out = torch.empty(2, dtype=torch.float32, device=logits.device)
    with torch.cuda.device(logits.device):
        L.check(lib.aria_router_aux_loss(_p(logits), _p(counts), _p(out), T, E, k, z_coeff, aux_coeff, _p(ws), nbytes,
                                         _stream(logits)), "router_aux_loss")
    return out


def router_aux_bwd(logits: torch.Tensor, counts: torch.Tensor, dlogits: torch.Tensor, k: int, z_coeff: float, aux_coeff: float,
                   loss_scale: float = 1.0) -> torch.Tensor:
    """dlogits += loss_scale * d(z_loss + aux_loss)/d(logits)  (MoEAuxLossAutoScaler.backward, moe_lm.py:103-117), in place."""
    _chk(logits), _chk(counts, torch.int32), _chk(dlogits)
    T, E = logits.shape
    with torch.cuda.device(logits.device):
        L.check(L.load().aria_router_aux_bwd(_p(logits), _p(counts), _p(dlogits), T, E, k, z_coeff, aux_coeff, loss_scale,
                                             _stream(logits)), "router_aux_bwd")
    return dlogits


def qkv_heads(x: torch.Tensor, weights: Sequence[torch.Tensor], biases: Sequence[Optional[torch.Tensor]],
              outs: Sequence[torch.Tensor], head_dim: int, rows_per_batch: int, pos0: int = 0, rope_mask: int = 0,
              rope_cos: Optional[torch.Tensor] = None, rope_sin: Optional[torch.Tensor] = None,
              position_ids: Optional[torch.Tensor] = None):
    """Fused q/k/v projections: x [B*T, K] @ W_s.T (+bias) (+RoPE) scattered into head-major buffers
    outs[s] [B, H, T_max, head_ld] at token offset pos0 (HF KV-cache layout)."""
    _chk(x)
    K = x.shape[-1]
    x2 = x.reshape(-1, K)
    d = L.GemmDesc()
    d.a, d.lda, d.m, d.k = x2.data_ptr(), K, x2.shape[0], K
    d.n = weights[0].shape[0]
    d.n_seg, d.b_layout, d.num_groups = len(weights), L.B_NK, 1
    d.epilogue = L.EPI_HEADS
    o0 = outs[0]
    for s, (w, b, o) in enumerate(zip(weights, biases, outs)):
        _chk(w), _chk(o)
        assert w.shape[0] == d.n and o.shape[1:] == o0.shape[1:] and o.stride() == o0.stride()
        d.b[s] = w.data_ptr()
        d.out[s] = o.data_ptr()
        if b is not None:
            d.bias[s] = _chk(b).data_ptr()
    d.head_dim, d.head_ld = head_dim, o0.shape[-1]
    d.rows_per_batch, d.pos0 = rows_per_batch, pos0
    d.stride_b, d.stride_h = o0.stride(0), o0.stride(1)
    d.rope_mask = rope_mask
    if rope_mask:
        d.rope_cos, d.rope_sin = _chk(rope_cos).data_ptr(), _chk(rope_sin).data_ptr()
    if position_ids is not None:
        d.position_ids = _chk(position_ids, torch.int32).data_ptr()
    _run_gemm(d, x, "qkv_heads")


# ------------------------------------------------------------------------------------------- MoE routing
def router_topk(x: torch.Tensor, w_router: torch.Tensor, k: int):
    _chk(x), _chk(w_router)
    T, dm = x.shape
    E = w_router.shape[0]
    dev = x.device
    logits = torch.empty((T, E), dtype=bf16, device=dev)
    idx = torch.empty((T, k), dtype=torch.int32, device=dev)
    scores = torch.empty((T, k), dtype=bf16, device=dev)
    counts = torch.empty((E,), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        L.check(L.load().aria_router_topk(_p(x), _p(w_router), _p(logits), _p(idx), _p(scores), _p(counts), T, dm, E, k,
                                          _stream(x)), "router_topk")
    return scores, idx, counts, logits


def route_from_logits(logits: torch.Tensor, k: int):
    _chk(logits)
    T, E = logits.shape
    dev = logits.device
    idx = torch.empty((T, k), dtype=torch.int32, device=dev)
    scores = torch.empty((T, k), dtype=bf16, device=dev)
    counts = torch.empty((E,), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        L.check(L.load().aria_route_from_logits(_p(logits), _p(idx), _p(scores), _p(counts), T, E, k, _stream(logits)),
                "route_from_logits")
    return scores, idx, counts


def route_given_indices(logits: torch.Tensor, top_idx: torch.Tensor):
    """Scores / counts for a GIVEN expert choice (parity / replay hook; see include/aria_b200.h)."""
    _chk(logits), _chk(top_idx, torch.int32)
    T, E = logits.shape
    k = top_idx.shape[1]
    assert top_idx.shape[0] == T
    scores = torch.empty((T, k), dtype=bf16, device=logits.device)
    counts = torch.empty((E,), dtype=torch.int32, device=logits.device)
    with torch.cuda.device(logits.device):
        L.check(L.load().aria_route_given_indices(_p(logits), _p(top_idx), _p(scores), _p(counts), T, E, k, _stream(logits)),
                "route_given_indices")
    return scores, counts


def build_permutation(top_idx: torch.Tensor, counts: torch.Tensor, row_align: int = 1):
    """row_align=16 (training): expert blocks start on multiples of 16 rows; `src` then has T*k + E*15 slots (upper bound
    of the padded row count, the true total is offsets[E]) and pad rows carry -1."""
    _chk(top_idx, torch.int32), _chk(counts, torch.int32)
    T, k = top_idx.shape
    E = counts.numel()
    dev = top_idx.device
    offsets = torch.empty((E + 1,), dtype=torch.int32, device=dev)
    dest = torch.empty((T * k,), dtype=torch.int32, device=dev)
    src = torch.empty((T * k + E * (row_align - 1),), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        L.check(L.load().aria_build_permutation(_p(top_idx), _p(counts), _p(offsets), _p(dest), _p(src), T, E, k, row_align,
                                                _stream(top_idx)), "build_permutation")
    return offsets, dest, src


def permute_rows(x: torch.Tensor, src_token: torch.Tensor) -> torch.Tensor:
    _chk(x), _chk(src_token, torch.int32)
    rows = src_token.numel()
    out = torch.empty((rows, x.shape[1]), dtype=bf16, device=x.device)
    with torch.cuda.device(x.device):
        L.check(L.load().aria_permute_rows(_p(x), _p(src_token), _p(out), rows, x.shape[1], _stream(x)), "permute_rows")
    return out


def permute_rows_to_ptr(x: torch.Tensor, src_token: torch.Tensor, out_ptr: int) -> None:
    """permute_rows writing to a raw device address — e.g. a PEER GPU's arena (aria_b200.peer.PeerArena): the row copy
    kernel then stores over NVLink."""
    _chk(x), _chk(src_token, torch.int32)
    with torch.cuda.device(x.device):
        L.check(L.load().aria_permute_rows(_p(x), _p(src_token), C.c_void_p(out_ptr), src_token.numel(), x.shape[1], _stream(x)),
                "permute_rows")


def unpermute_combine(y: torch.Tensor, dest_row: torch.Tensor, scores: torch.Tensor,
                      shared: Optional[torch.Tensor] = None) -> torch.Tensor:
    _chk(y), _chk(dest_row, torch.int32), _chk(scores)
    T, k = scores.shape
    out = torch.empty((T, y.shape[1]), dtype=bf16, device=y.device)
    if shared is not None:
        _chk(shared)
    with torch.cuda.device(y.device):
        L.check(L.load().aria_unpermute_combine(_p(y), _p(dest_row), _p(scores), _p(shared), _p(out), T, y.shape[1], k,
                                                _stream(y)), "unpermute_combine")
    return out


def moe_block_fwd(x: torch.Tensor, w_router: torch.Tensor, fc1_w: torch.Tensor, fc2_w: torch.Tensor, gate_w: Optional[torch.Tensor],
                  up_w: Optional[torch.Tensor], down_w: Optional[torch.Tensor], k: int,
                  forced_top_idx: Optional[torch.Tensor] = None, side_stream: Optional[torch.cuda.Stream] = None,
                  fc1_scale: Optional[torch.Tensor] = None, fc2_scale: Optional[torch.Tensor] = None,
                  w8a8: bool = False, gate_scale: Optional[torch.Tensor] = None, up_scale: Optional[torch.Tensor] = None,
                  down_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """MoELayer.forward (moe_lm.py:548-577) as one C-ABI call (`aria_moe_block_fwd`): x [T, d] -> [T, d].
    With fc1_scale [E, 2I] / fc2_scale [E, d] fp32, fc1_w / fc2_w are e4m3 (quantize_fp8_cols) and the call is
    `aria_moe_block_fwd_fp8`; with w8a8=True as well, the weights are K-major (see grouped_gemm_w8a8), the activations are
    quantized per row too and the call is `aria_moe_block_fwd_w8a8`.
    With gate_scale / up_scale [I_shared] and down_scale [d] fp32, the shared experts' weights are e4m3 nn.Linear weights
    (W8A8, see linear_w8a8) and the call is `aria_moe_block_fwd_shared_fp8` in the expert mode given by the other arguments."""
    fp8 = fc1_scale is not None or fc2_scale is not None
    if fp8 and (fc1_scale is None or fc2_scale is None):
        raise ValueError("moe_block_fwd: give both fc1_scale and fc2_scale, or neither")
    if w8a8 and not fp8:
        raise ValueError("moe_block_fwd: w8a8 needs the fp8 weight scales")
    wdt = torch.float8_e4m3fn if fp8 else bf16
    _chk(x), _chk(w_router)
    if w8a8:
        _kmajor(fc1_w), _kmajor(fc2_w)
    else:
        _chk(fc1_w, wdt), _chk(fc2_w, wdt)
    T, d = x.shape
    E, I = fc2_w.shape[0], fc2_w.shape[1]
    assert w_router.shape == (E, d) and fc1_w.shape == (E, d, 2 * I) and fc2_w.shape == (E, I, d)
    if fp8:
        _chk(fc1_scale, torch.float32), _chk(fc2_scale, torch.float32)
        assert fc1_scale.shape == (E, 2 * I) and fc2_scale.shape == (E, d)
    shared_fp8 = gate_scale is not None or up_scale is not None or down_scale is not None
    if shared_fp8 and (gate_scale is None or up_scale is None or down_scale is None or gate_w is None):
        raise ValueError("moe_block_fwd: fp8 shared experts need their weights and all three scales")
    Is = 0
    if gate_w is not None:
        sdt = torch.float8_e4m3fn if shared_fp8 else bf16
        _chk(gate_w, sdt), _chk(up_w, sdt), _chk(down_w, sdt)
        Is = gate_w.shape[0]
        assert gate_w.shape == (Is, d) and up_w.shape == (Is, d) and down_w.shape == (d, Is)
    if shared_fp8:
        _chk(gate_scale, torch.float32), _chk(up_scale, torch.float32), _chk(down_scale, torch.float32)
        assert gate_scale.shape == (Is,) and up_scale.shape == (Is,) and down_scale.shape == (d,)
    if forced_top_idx is not None:
        _chk(forced_top_idx, torch.int32, align=4)
        assert forced_top_idx.shape == (T, k)
    lib = L.load()
    if shared_fp8:
        nbytes = lib.aria_moe_block_fwd_shared_fp8_workspace_bytes(T, d, E, k, I, Is)
    else:
        nbytes = lib.aria_moe_block_fwd_workspace_bytes(T, d, E, k, I, Is)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    out = torch.empty((T, d), dtype=bf16, device=x.device)
    side = C.c_void_p(side_stream.cuda_stream) if side_stream is not None else None
    with torch.cuda.device(x.device):
        if shared_fp8:
            mode, name = (L.MOE_EXPERTS_W8A8, "w8a8") if w8a8 else ((L.MOE_EXPERTS_FP8, "fp8") if fp8 else (L.MOE_EXPERTS_BF16, "bf16"))
            L.check(lib.aria_moe_block_fwd_shared_fp8(_p(x), _p(w_router), _p(fc1_w), _p(fc2_w), _p(fc1_scale), _p(fc2_scale), mode,
                                                      _p(gate_w), _p(up_w), _p(down_w), _p(gate_scale), _p(up_scale),
                                                      _p(down_scale), _p(out), T, d, E, k, I, Is, _p(forced_top_idx), _p(ws), nbytes,
                                                      _stream(x), side), f"moe_block_fwd_{name}_shared_fp8")
        elif w8a8:
            L.check(lib.aria_moe_block_fwd_w8a8(_p(x), _p(w_router), _p(fc1_w), _p(fc2_w), _p(fc1_scale), _p(fc2_scale),
                                                _p(gate_w), _p(up_w), _p(down_w), _p(out), T, d, E, k, I, Is, _p(forced_top_idx),
                                                _p(ws), nbytes, _stream(x), side), "moe_block_fwd_w8a8")
        elif fp8:
            L.check(lib.aria_moe_block_fwd_fp8(_p(x), _p(w_router), _p(fc1_w), _p(fc2_w), _p(fc1_scale), _p(fc2_scale), _p(gate_w),
                                               _p(up_w), _p(down_w), _p(out), T, d, E, k, I, Is, _p(forced_top_idx), _p(ws), nbytes,
                                               _stream(x), side), "moe_block_fwd_fp8")
        else:
            L.check(lib.aria_moe_block_fwd(_p(x), _p(w_router), _p(fc1_w), _p(fc2_w), _p(gate_w), _p(up_w), _p(down_w), _p(out), T, d,
                                           E, k, I, Is, _p(forced_top_idx), _p(ws), nbytes, _stream(x), side), "moe_block_fwd")
    return out


def offsets_from_counts(counts: torch.Tensor) -> torch.Tensor:
    _chk(counts, torch.int64)
    off = torch.empty((counts.numel() + 1,), dtype=torch.int32, device=counts.device)
    with torch.cuda.device(counts.device):
        L.check(L.load().aria_offsets_from_counts(_p(counts), _p(off), counts.numel(), _stream(counts)), "offsets_from_counts")
    return off


# ------------------------------------------------------------------------------------------- row-wise
def rmsnorm(x: torch.Tensor, weight: torch.Tensor, eps: float, residual: Optional[torch.Tensor] = None):
    """Returns norm(x) or, with residual, (norm(x + residual), x + residual)."""
    _chk(x), _chk(weight)
    d = x.shape[-1]
    rows = x.numel() // d
    out = torch.empty_like(x)
    s = torch.empty_like(x) if residual is not None else None
    if residual is not None:
        _chk(residual)
    with torch.cuda.device(x.device):
        L.check(L.load().aria_rmsnorm(_p(x), _p(residual), _p(weight), _p(out), _p(s), rows, d, eps, _stream(x)), "rmsnorm")
    return out if residual is None else (out, s)


def rmsnorm_quantize_fp8(x: torch.Tensor, weight: torch.Tensor, eps: float, residual: Optional[torch.Tensor] = None):
    """rmsnorm whose bf16 output is quantized per row in the same kernel: returns (q, scale) or, with residual,
    (q, scale, x + residual); q [..., d] float8_e4m3fn and scale [rows] fp32 are bit for bit
    permute_quantize_fp8(rmsnorm(x, weight, eps, residual)[0]).  d <= 4096."""
    _chk(x), _chk(weight)
    d = x.shape[-1]
    rows = x.numel() // d
    q = torch.empty(x.shape, dtype=torch.float8_e4m3fn, device=x.device)
    scale = torch.empty((rows,), dtype=torch.float32, device=x.device)
    s = torch.empty_like(x) if residual is not None else None
    if residual is not None:
        _chk(residual)
    with torch.cuda.device(x.device):
        L.check(L.load().aria_rmsnorm_quantize_fp8(_p(x), _p(residual), _p(weight), _p(q), _p(scale), _p(s), rows, d, eps,
                                                   _stream(x)), "rmsnorm_quantize_fp8")
    return (q, scale) if residual is None else (q, scale, s)


def layernorm(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, eps: float) -> torch.Tensor:
    _chk(x), _chk(weight), _chk(bias)
    d = x.shape[-1]
    out = torch.empty_like(x)
    with torch.cuda.device(x.device):
        L.check(L.load().aria_layernorm(_p(x), _p(weight), _p(bias), _p(out), x.numel() // d, d, eps, _stream(x)), "layernorm")
    return out


def rope_table(inv_freq: torch.Tensor, n_pos: int):
    _chk(inv_freq, torch.float32)
    hd = inv_freq.numel() * 2
    cos = torch.empty((n_pos, hd), dtype=bf16, device=inv_freq.device)
    sin = torch.empty_like(cos)
    with torch.cuda.device(inv_freq.device):
        L.check(L.load().aria_rope_table(_p(inv_freq), _p(cos), _p(sin), n_pos, hd, _stream(inv_freq)), "rope_table")
    return cos, sin


def embedding(ids: torch.Tensor, table: torch.Tensor) -> torch.Tensor:
    _chk(ids, torch.int64, align=8), _chk(table)      # ids are read element-wise (a [1, 1] slice of a longer id row is fine)
    out = torch.empty((*ids.shape, table.shape[1]), dtype=bf16, device=table.device)
    with torch.cuda.device(table.device):
        L.check(L.load().aria_embedding(_p(ids), _p(table), _p(out), ids.numel(), table.shape[1], _stream(table)), "embedding")
    return out


def merge_image_features(ids: torch.Tensor, image_token: int, features: torch.Tensor, embeds: torch.Tensor,
                         count_out: Optional[torch.Tensor] = None):
    """In place: embeds rows at <|img|> positions <- consecutive rows of features (masked_scatter)."""
    _chk(ids, torch.int64, align=8), _chk(features), _chk(embeds)
    d = embeds.shape[-1]
    with torch.cuda.device(embeds.device):
        L.check(L.load().aria_merge_image_features(_p(ids), image_token, _p(features), _p(embeds), _p(count_out),
                                                   ids.numel(), d, _stream(embeds)), "merge_image_features")
    return embeds


def im2col_patches(pixels: torch.Tensor, patch: int, k_pad: int) -> torch.Tensor:
    _chk(pixels)
    B, Cc, S, S2 = pixels.shape
    assert Cc == 3 and S == S2
    n = (S // patch) ** 2
    out = torch.empty((B * n, k_pad), dtype=bf16, device=pixels.device)
    with torch.cuda.device(pixels.device):
        L.check(L.load().aria_im2col_patches(_p(pixels), _p(out), B, S, patch, k_pad, _stream(pixels)), "im2col_patches")
    return out


def add_pos_embedding(x: torch.Tensor, pos_ids: torch.Tensor, table: torch.Tensor) -> torch.Tensor:
    _chk(x), _chk(pos_ids, torch.int64), _chk(table)
    out = torch.empty_like(x)
    d = x.shape[-1]
    with torch.cuda.device(x.device):
        L.check(L.load().aria_add_pos_embedding(_p(x), _p(pos_ids), _p(table), _p(out), x.numel() // d, d, _stream(x)),
                "add_pos_embedding")
    return out


# ------------------------------------------------------------------------------------------- attention
def _attn_qkv_check(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, what: str):
    for t in (q, k, v):
        if not (t.is_cuda and t.dtype == bf16 and t.dim() == 4 and t.stride(-1) == 1 and t.stride(-2) == 128 and t.data_ptr() % 16 == 0):
            raise RuntimeError(f"{what}: q/k/v must be CUDA bf16 [B,H,T,128] with 128-element token rows (16-byte aligned)")
    assert q.shape[-1] == 128 and k.shape[-1] == 128 and k.stride() == v.stride()


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, Tq: int, Tk: int, scale: float, causal: bool,
              out_hd: int = 128, key_mask: Optional[torch.Tensor] = None, return_lse: bool = False):
    """q [B,H,>=Tq,128], k/v [B,H,>=Tk,128] head-major (first Tq/Tk rows used) -> out [B, Tq, H*out_hd].
    Token rows must be 128 contiguous bf16 at a row stride of 128 (a slice q[:, :, pos0:] of a staging buffer is fine).
    return_lse=True -> (out, lse): lse [B, H, Tq] fp32 is the natural-log logsumexp of scale * q.k over the visible keys
    (-inf for a row that sees none), what `attention_bwd` needs; `out` is bit-identical to the return_lse=False call."""
    _attn_qkv_check(q, k, v, "attention")
    B, H = q.shape[0], q.shape[1]
    assert q.shape[2] >= Tq and k.shape[2] >= Tk
    out = torch.empty((B, Tq, H * out_hd), dtype=bf16, device=q.device)
    if key_mask is not None:
        _chk(key_mask, torch.uint8)
        assert key_mask.shape == (B, Tk)
    lib = L.load()
    ws_bytes = lib.aria_attention_fwd_workspace_bytes(B, H, Tq, Tk, out_hd, int(causal))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=q.device) if ws_bytes > 0 else None
    with torch.cuda.device(q.device):
        if return_lse:
            lse = torch.empty((B, H, Tq), dtype=torch.float32, device=q.device)
            L.check(lib.aria_attention_fwd_lse(_p(q), _p(k), _p(v), _p(out), _p(lse), _p(key_mask), B, H, Tq, Tk, q.stride(0),
                                               q.stride(1), k.stride(0), k.stride(1), out_hd, scale, int(causal), _p(ws), ws_bytes,
                                               _stream(q)), "attention_fwd")
            return out, lse
        L.check(lib.aria_attention_fwd(_p(q), _p(k), _p(v), _p(out), _p(key_mask), B, H, Tq, Tk, q.stride(0), q.stride(1),
                                       k.stride(0), k.stride(1), out_hd, scale, int(causal), _p(ws), ws_bytes, _stream(q)),
                "attention_fwd")
    return out


def attention_bwd(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, dout: torch.Tensor, lse: torch.Tensor,
                  Tq: int, Tk: int, scale: float, causal: bool, key_mask: Optional[torch.Tensor] = None):
    """Backward of `attention(..., return_lse=True)` (head dim 128): q [B,H,>=Tq,128], k/v [B,H,>=Tk,128] as in the forward,
    out / dout [B, Tq, H*128] token-major, lse [B, H, Tq] -> (dq [B,H,Tq,128], dk [B,H,Tk,128], dv [B,H,Tk,128]) bf16.
    dk and dv are bit-reproducible; dq's last bits depend on the order of fp32 atomic additions."""
    _attn_qkv_check(q, k, v, "attention_bwd")
    B, H = q.shape[0], q.shape[1]
    assert q.shape[2] >= Tq and k.shape[2] >= Tk
    _chk(out), _chk(dout), _chk(lse, torch.float32, align=4)
    assert out.shape == (B, Tq, H * 128) and dout.shape == out.shape and lse.shape == (B, H, Tq)
    if key_mask is not None:
        _chk(key_mask, torch.uint8)
        assert key_mask.shape == (B, Tk)
    dq = torch.empty((B, H, Tq, 128), dtype=bf16, device=q.device)
    dk = torch.empty((B, H, Tk, 128), dtype=bf16, device=q.device)
    dv = torch.empty_like(dk)
    lib = L.load()
    ws_bytes = lib.aria_attention_bwd_workspace_bytes(B, H, Tq, Tk, int(causal))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=q.device)
    # the kernel reads q with q's strides and writes dq with the same strides; k/v/dk/dv likewise share theirs
    if q.stride() != dq.stride():
        q = q[:, :, :Tq].contiguous()
    if k.stride() != dk.stride():
        k, v = k[:, :, :Tk].contiguous(), v[:, :, :Tk].contiguous()
    with torch.cuda.device(q.device):
        L.check(lib.aria_attention_bwd(_p(q), _p(k), _p(v), _p(out), _p(dout), _p(lse), _p(dq), _p(dk), _p(dv), _p(key_mask),
                                       B, H, Tq, Tk, q.stride(0), q.stride(1), k.stride(0), k.stride(1), scale, int(causal),
                                       _p(ws), ws_bytes, _stream(q)), "attention_bwd")
    return dq, dk, dv


fp8 = torch.float8_e4m3fn


def _fp8_cache_check(k: torch.Tensor, v: torch.Tensor, k_scale: Optional[torch.Tensor], v_scale: Optional[torch.Tensor],
                     what: str):
    """An fp8 KV cache: e4m3 k / v [B, H, T_max, 128] with 16-byte rows and fp32 scales k_scale / v_scale [B, H, T_max]."""
    if k_scale is None or v_scale is None:
        raise ValueError(f"{what}: an fp8 (float8_e4m3fn) cache needs k_scale= and v_scale=")
    for t in (k, v):
        if not (t.is_cuda and t.dtype == fp8 and t.dim() == 4 and t.shape[-1] == 128 and t.stride(-1) == 1 and t.stride(-2) == 128
                and t.data_ptr() % 16 == 0):
            raise RuntimeError(f"{what}: fp8 k/v must be CUDA float8_e4m3fn [B,H,T_max,128] with 128-code rows (16-byte aligned)")
    for t in (k_scale, v_scale):
        if not (t.is_cuda and t.dtype == torch.float32 and t.shape == k.shape[:3] and t.stride(-1) == 1):
            raise RuntimeError(f"{what}: k_scale / v_scale must be CUDA float32 [B,H,T_max] with contiguous rows")
    if k.stride() != v.stride() or k_scale.stride() != v_scale.stride() or v.shape != k.shape:
        raise RuntimeError(f"{what}: k and v (and their scales) must share shape and strides")


def attention_decode(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, Tk: int, scale: float,
                     key_mask: Optional[torch.Tensor] = None, k_scale: Optional[torch.Tensor] = None,
                     v_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """q [B,H,128] (any strides with a contiguous last dim, e.g. a row of the q staging buffer), cache k/v
    [B,H,T_max,128] -> out [B, H*128].  key_mask [B, Tk] uint8, 1 = masked out (padded batch).
    With an fp8 cache (k.dtype float8_e4m3fn) k_scale / v_scale [B,H,T_max] fp32 are required and the fp8 kernel runs."""
    if not (q.is_cuda and q.dtype == bf16 and q.stride(-1) == 1 and q.data_ptr() % 8 == 0):
        raise RuntimeError("attention_decode: q must be a CUDA bf16 tensor with a contiguous last dim")
    is_fp8 = k.dtype == fp8
    if is_fp8:
        _fp8_cache_check(k, v, k_scale, v_scale, "attention_decode")
    else:
        _chk(k), _chk(v)
    B, H = q.shape[0], q.shape[1]
    lib = L.load()
    ws_bytes = lib.aria_attention_decode_workspace_bytes(B, H, Tk)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=q.device)
    out = torch.empty((B, H * 128), dtype=bf16, device=q.device)
    if key_mask is not None:
        _chk(key_mask, torch.uint8)
        assert key_mask.shape == (B, Tk)
    with torch.cuda.device(q.device):
        if is_fp8:
            L.check(lib.aria_attention_decode_fp8(_p(q), _p(k), _p(v), _p(k_scale), _p(v_scale), _p(out), _p(key_mask), B, H, Tk,
                                                  q.stride(0), q.stride(1), k.stride(0), k.stride(1), k_scale.stride(0),
                                                  k_scale.stride(1), scale, _p(ws), ws_bytes, _stream(q)), "attention_decode_fp8")
        else:
            L.check(lib.aria_attention_decode(_p(q), _p(k), _p(v), _p(out), _p(key_mask), B, H, Tk, q.stride(0), q.stride(1),
                                              k.stride(0), k.stride(1), scale, _p(ws), ws_bytes, _stream(q)), "attention_decode")
    return out


def attention_decode_devlen(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, lens: torch.Tensor, scale: float,
                            key_mask: Optional[torch.Tensor] = None, k_scale: Optional[torch.Tensor] = None,
                            v_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """attention_decode with the key count of each row on the device: row b sees cache rows [0, lens[b]) (lens int32 [B]).
    Cache k/v [B,H,T_max,128]; key_mask [B, >=T_max] uint8 (1 = masked out; any row stride).  Row b is bit-identical to
    attention_decode(..., Tk=lens[b]); nothing reads the host value of lens, so one captured launch serves every step.
    With an fp8 cache (k.dtype float8_e4m3fn) k_scale / v_scale [B,H,T_max] fp32 are required and the fp8 kernel runs."""
    is_fp8 = k.dtype == fp8
    if is_fp8:
        _fp8_cache_check(k, v, k_scale, v_scale, "attention_decode_devlen")
    else:
        _chk(k), _chk(v)
    _chk(lens, torch.int32, align=4)
    if not (q.is_cuda and q.dtype == bf16 and q.stride(-1) == 1 and q.data_ptr() % 8 == 0):
        raise RuntimeError("attention_decode_devlen: q must be a CUDA bf16 tensor with a contiguous last dim")
    B, H, T_max = q.shape[0], q.shape[1], k.shape[2]
    assert lens.shape == (B,) and k.shape[:2] == (B, H)
    lib = L.load()
    ws_bytes = lib.aria_attention_decode_workspace_bytes(B, H, T_max)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=q.device)
    out = torch.empty((B, H * 128), dtype=bf16, device=q.device)
    mask_stride = 0
    if key_mask is not None:
        if not (key_mask.is_cuda and key_mask.dtype == torch.uint8 and key_mask.stride(-1) == 1 and key_mask.shape[0] == B
                and key_mask.shape[1] >= T_max):
            raise RuntimeError("attention_decode_devlen: key_mask must be CUDA uint8 [B, >= T_max] with contiguous rows")
        mask_stride = key_mask.stride(0)
    with torch.cuda.device(q.device):
        if is_fp8:
            L.check(lib.aria_attention_decode_devlen_fp8(_p(q), _p(k), _p(v), _p(k_scale), _p(v_scale), _p(out), _p(key_mask),
                                                         mask_stride, _p(lens), B, H, T_max, q.stride(0), q.stride(1), k.stride(0),
                                                         k.stride(1), k_scale.stride(0), k_scale.stride(1), scale, _p(ws), ws_bytes,
                                                         _stream(q)), "attention_decode_devlen_fp8")
        else:
            L.check(lib.aria_attention_decode_devlen(_p(q), _p(k), _p(v), _p(out), _p(key_mask), mask_stride, _p(lens), B, H, T_max,
                                                     q.stride(0), q.stride(1), k.stride(0), k.stride(1), scale, _p(ws), ws_bytes,
                                                     _stream(q)), "attention_decode_devlen")
    return out


def attention_decode_shared_prefix(q: torch.Tensor, prefix_k: torch.Tensor, prefix_v: torch.Tensor, prefix_lens: torch.Tensor,
                                   tail_k: torch.Tensor, tail_v: torch.Tensor, tail_lens: torch.Tensor, group_size: int,
                                   scale: float, prefix_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Decode attention of R = G * group_size rows that share their group's prompt cache: row r = g * group_size + j attends
    to prefix rows [0, prefix_lens[g]) of prefix_k / prefix_v [G,H,P_max,128] (minus prefix_mask [G, >= P_max] uint8, 1 = masked
    out, any row stride), then to its own rows [0, tail_lens[r]) of tail_k / tail_v [R,H,N_max,128].  q [R,H,128] (contiguous
    last dim, any strides); prefix_lens int32 [G], tail_lens int32 [R] on the device -> out [R, H*128].  Row r is bit-identical
    to attention_decode_devlen on a cache that holds the prefix at [0, P), masked rows up to S = 256 * ceil(P / 256) and the tail
    from S on; each prefix key and value is read once per (group, head).  See aria_attention_decode_shared_prefix."""
    _chk(prefix_k), _chk(prefix_v), _chk(tail_k), _chk(tail_v)
    _chk(prefix_lens, torch.int32, align=4), _chk(tail_lens, torch.int32, align=4)
    if not (q.is_cuda and q.dtype == bf16 and q.dim() == 3 and q.stride(-1) == 1 and q.data_ptr() % 8 == 0):
        raise RuntimeError("attention_decode_shared_prefix: q must be a CUDA bf16 [R,H,128] tensor with a contiguous last dim")
    if not isinstance(group_size, int) or group_size < 1:
        raise ValueError(f"attention_decode_shared_prefix: group_size must be a positive int, got {group_size!r}")
    R, H = q.shape[0], q.shape[1]
    G, P_max, N_max = prefix_k.shape[0], prefix_k.shape[2], tail_k.shape[2]
    if (q.shape[2] != 128 or R != G * group_size or prefix_k.shape != (G, H, P_max, 128) or prefix_v.shape != prefix_k.shape
            or tail_k.shape != (R, H, N_max, 128) or tail_v.shape != tail_k.shape or prefix_lens.shape != (G,)
            or tail_lens.shape != (R,)):
        raise ValueError(f"attention_decode_shared_prefix: q {tuple(q.shape)}, prefix {tuple(prefix_k.shape)}, tail "
                         f"{tuple(tail_k.shape)}, lens {tuple(prefix_lens.shape)} / {tuple(tail_lens.shape)} do not fit "
                         f"groups of {group_size}")
    mask_stride = 0
    if prefix_mask is not None:
        if not (prefix_mask.is_cuda and prefix_mask.dtype == torch.uint8 and prefix_mask.dim() == 2
                and prefix_mask.stride(-1) == 1 and prefix_mask.shape[0] == G and prefix_mask.shape[1] >= P_max):
            raise RuntimeError("attention_decode_shared_prefix: prefix_mask must be CUDA uint8 [G, >= P_max] with contiguous rows")
        mask_stride = prefix_mask.stride(0)
    lib = L.load()
    ws_bytes = lib.aria_attention_decode_shared_prefix_workspace_bytes(G, group_size, H, P_max, N_max)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=q.device)
    out = torch.empty((R, H * 128), dtype=bf16, device=q.device)
    with torch.cuda.device(q.device):
        L.check(lib.aria_attention_decode_shared_prefix(_p(q), _p(prefix_k), _p(prefix_v), _p(prefix_lens), _p(prefix_mask),
                                                        mask_stride, _p(tail_k), _p(tail_v), _p(tail_lens), _p(out), G, group_size,
                                                        H, P_max, N_max, q.stride(0), q.stride(1), prefix_k.stride(0),
                                                        prefix_k.stride(1), tail_k.stride(0), tail_k.stride(1), scale, _p(ws),
                                                        ws_bytes, _stream(q)), "attention_decode_shared_prefix")
    return out


def attention_decode_multi(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, lens: torch.Tensor, scale: float,
                           key_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Q consecutive queries per row (prompt-lookup verification): q [B,H,Q,128] (contiguous last dim, any strides), bf16 cache
    k/v [B,H,T_max,128]; query i of row b sees cache rows [0, lens[b*Q + i]) (lens CUDA int32 [B*Q]) minus key_mask [B, >= T_max]
    uint8 (1 = masked out, any row stride) -> out [B, Q, H*128].  Query i of row b is bit-identical to
    attention_decode_devlen(..., lens=lens[b*Q + i]); each key and value is read once per (row, head) for all Q queries."""
    _chk(k), _chk(v)
    _chk(lens, torch.int32, align=4)
    if not (q.is_cuda and q.dtype == bf16 and q.dim() == 4 and q.stride(-1) == 1 and q.data_ptr() % 8 == 0):
        raise RuntimeError("attention_decode_multi: q must be a CUDA bf16 [B,H,Q,128] tensor with a contiguous last dim")
    B, H, Q = q.shape[:3]
    T_max = k.shape[2]
    if (q.shape[3] != 128 or k.shape != (B, H, T_max, 128) or v.shape != k.shape or v.stride() != k.stride()
            or lens.shape != (B * Q,)):
        raise ValueError(f"attention_decode_multi: q {tuple(q.shape)}, cache {tuple(k.shape)}, lens {tuple(lens.shape)} do not fit")
    mask_stride = 0
    if key_mask is not None:
        if not (key_mask.is_cuda and key_mask.dtype == torch.uint8 and key_mask.dim() == 2 and key_mask.stride(-1) == 1
                and key_mask.shape[0] == B and key_mask.shape[1] >= T_max):
            raise RuntimeError("attention_decode_multi: key_mask must be CUDA uint8 [B, >= T_max] with contiguous rows")
        mask_stride = key_mask.stride(0)
    lib = L.load()
    ws_bytes = lib.aria_attention_decode_workspace_bytes(B * Q, H, T_max)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=q.device)
    out = torch.empty((B, Q, H * 128), dtype=bf16, device=q.device)
    with torch.cuda.device(q.device):
        L.check(lib.aria_attention_decode_multi(_p(q), _p(k), _p(v), _p(out), _p(key_mask), mask_stride, _p(lens), B, Q, H, T_max,
                                                q.stride(0), q.stride(1), q.stride(2), k.stride(0), k.stride(1), scale, _p(ws),
                                                ws_bytes, _stream(q)), "attention_decode_multi")
    return out


def _packed_check(S_tot: int, cu_seqlens: torch.Tensor, what: str) -> int:
    """Packed segments: cu_seqlens CUDA int32 [B+1] (B >= 1) and S_tot >= B rows -> B."""
    _chk(cu_seqlens, torch.int32, align=4)
    if cu_seqlens.dim() != 1 or cu_seqlens.numel() < 2:
        raise ValueError(f"{what}: cu_seqlens must be int32 [B+1] with B >= 1, got {tuple(cu_seqlens.shape)}")
    B = cu_seqlens.numel() - 1
    if not isinstance(S_tot, int) or S_tot < B:
        raise ValueError(f"{what}: S_tot must be an int >= B = {B} (every segment has a row), got {S_tot!r}")
    return B


def attention_prefill_shared_prefix(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, S_tot: int, prefix_k: torch.Tensor,
                                    prefix_v: torch.Tensor, P: int, cu_seqlens: torch.Tensor, scale: float) -> torch.Tensor:
    """Causal prefill of B suffixes sharing one prefix.  q / k / v [1,H,>=S_tot,128] head-major (first S_tot rows used; 128-element
    rows as in `attention`) hold the suffixes packed: suffix b is rows [cu_seqlens[b], cu_seqlens[b+1]) (cu_seqlens CUDA int32
    [B+1], nondecreasing from 0 to S_tot).  prefix_k / prefix_v [1,H,P_max,128]: the prefix is its rows [0, P).  The query at
    packed row q of suffix b sees the whole prefix and the packed keys [cu_seqlens[b], q] -> out [S_tot, H*128].  With
    P % 128 == 0, row b is bit-identical to `attention(..., causal=True)` on its own [prefix, suffix b] layout.
    See aria_attention_prefill_shared_prefix."""
    _attn_qkv_check(q, k, v, "attention_prefill_shared_prefix")
    _attn_qkv_check(prefix_k, prefix_v, prefix_v, "attention_prefill_shared_prefix")
    B = _packed_check(S_tot, cu_seqlens, "attention_prefill_shared_prefix")
    H, P_max = q.shape[1], prefix_k.shape[2]
    if q.shape[0] != 1 or q.shape[2] < S_tot or k.shape[:2] != (1, H) or k.shape[2] < S_tot or v.shape != k.shape:
        raise ValueError(f"attention_prefill_shared_prefix: q {tuple(q.shape)} / k {tuple(k.shape)} must be [1, H, >= {S_tot}, 128]")
    if prefix_k.shape != (1, H, P_max, 128) or prefix_v.shape != prefix_k.shape or prefix_v.stride() != prefix_k.stride():
        raise ValueError(f"attention_prefill_shared_prefix: prefix {tuple(prefix_k.shape)} / {tuple(prefix_v.shape)} must be "
                         f"[1, {H}, P_max, 128] with equal strides")
    if not isinstance(P, int) or not 1 <= P <= P_max:
        raise ValueError(f"attention_prefill_shared_prefix: P must be an int in [1, {P_max}], got {P!r}")
    out = torch.empty((S_tot, H * 128), dtype=bf16, device=q.device)
    with torch.cuda.device(q.device):
        L.check(L.load().aria_attention_prefill_shared_prefix(_p(q), _p(k), _p(v), _p(prefix_k), _p(prefix_v), _p(cu_seqlens),
                                                              _p(out), B, H, S_tot, P, P_max, q.stride(1), k.stride(1),
                                                              prefix_k.stride(1), scale, _stream(q)),
                "attention_prefill_shared_prefix")
    return out


def _varlen_qkv(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, cu_seqlens: torch.Tensor, N: Optional[int], what: str):
    """Packed q / k / v [1,H,>=N,128] and cu_seqlens int32 [n_seg+1] -> (n_seg, H, N)."""
    _attn_qkv_check(q, k, v, what)
    N = q.shape[2] if N is None else N
    n_seg = _packed_check(N, cu_seqlens, what)
    H = q.shape[1]
    if q.shape[0] != 1 or q.shape[2] < N or k.shape[:2] != (1, H) or k.shape[2] < N or v.shape != k.shape:
        raise ValueError(f"{what}: q {tuple(q.shape)} / k {tuple(k.shape)} must be [1, H, >= {N}, 128]")
    return n_seg, H, N


def attention_varlen(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, cu_seqlens: torch.Tensor, scale: float,
                     return_lse: bool = False, N: Optional[int] = None):
    """Causal attention over packed sequences (padding-free batches).  q / k / v [1,H,>=N,128] head-major (first N rows used,
    N = q.shape[2] by default; 128-element rows as in `attention`) hold n_seg sequences back to back: sequence s is rows
    [cu_seqlens[s], cu_seqlens[s+1]) (cu_seqlens CUDA int32 [n_seg+1], nondecreasing from 0 to N, no empty sequence; not checked
    here, see hf_attention).  The query at packed row r of sequence s sees the packed keys [cu_seqlens[s], r] -> out [N, H*128],
    and with return_lse=True also lse [H, N] fp32.  Each sequence's out and lse are bit-identical to
    `attention(..., causal=True, return_lse=True)` on that sequence alone.  See aria_attention_fwd_varlen."""
    n_seg, H, N = _varlen_qkv(q, k, v, cu_seqlens, N, "attention_varlen")
    out = torch.empty((N, H * 128), dtype=bf16, device=q.device)
    lse = torch.empty((H, N), dtype=torch.float32, device=q.device) if return_lse else None
    with torch.cuda.device(q.device):
        L.check(L.load().aria_attention_fwd_varlen(_p(q), _p(k), _p(v), _p(out), _p(lse), _p(cu_seqlens), n_seg, H, N, q.stride(1),
                                                   k.stride(1), scale, _stream(q)), "attention_fwd_varlen")
    return (out, lse) if return_lse else out


def attention_varlen_bwd(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, dout: torch.Tensor, lse: torch.Tensor,
                         cu_seqlens: torch.Tensor, scale: float, N: Optional[int] = None):
    """Backward of `attention_varlen(..., return_lse=True)`: q / k / v and cu_seqlens as there, out / dout [N, H*128] (or
    [1, N, H*128]), lse [H, N] -> (dq, dk, dv) [1,H,N,128] bf16.  Per sequence, dk and dv are bit-identical to `attention_bwd`
    (causal) on that sequence alone, dq equal to it up to the order of fp32 atomic additions."""
    n_seg, H, N = _varlen_qkv(q, k, v, cu_seqlens, N, "attention_varlen_bwd")
    _chk(out), _chk(dout), _chk(lse, torch.float32, align=4)
    assert out.numel() == N * H * 128 and dout.shape == out.shape and lse.shape == (H, N)
    dq = torch.empty((1, H, N, 128), dtype=bf16, device=q.device)
    dk = torch.empty_like(dq)
    dv = torch.empty_like(dq)
    lib = L.load()
    ws_bytes = lib.aria_attention_bwd_varlen_workspace_bytes(n_seg, H, N)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=q.device)
    # the kernel reads q with q's strides and writes dq with the same strides; k/v/dk/dv likewise share theirs
    if q.stride() != dq.stride():
        q = q[:, :, :N].contiguous()
    if k.stride() != dk.stride():
        k, v = k[:, :, :N].contiguous(), v[:, :, :N].contiguous()
    with torch.cuda.device(q.device):
        L.check(lib.aria_attention_bwd_varlen(_p(q), _p(k), _p(v), _p(out), _p(dout), _p(lse), _p(dq), _p(dk), _p(dv),
                                              _p(cu_seqlens), n_seg, H, N, q.stride(1), k.stride(1), scale, _p(ws), ws_bytes,
                                              _stream(q)), "attention_bwd_varlen")
    return dq, dk, dv


def kv_scatter_tails(k: torch.Tensor, v: torch.Tensor, S_tot: int, tail_k: torch.Tensor, tail_v: torch.Tensor,
                     cu_seqlens: torch.Tensor, group_size: int):
    """Copy packed suffix rows k / v [1,H,>=S_tot,128] (segments as in `attention_prefill_shared_prefix`) into the tails
    tail_k / tail_v [B*group_size, H, N_max, 128]: packed row s of suffix b -> row s - cu_seqlens[b] of tails
    b*group_size .. b*group_size + group_size - 1.  Tail rows at or past each suffix's length are left as they are."""
    _attn_qkv_check(k, v, v, "kv_scatter_tails")
    _chk(tail_k), _chk(tail_v)
    B = _packed_check(S_tot, cu_seqlens, "kv_scatter_tails")
    if not isinstance(group_size, int) or group_size < 1:
        raise ValueError(f"kv_scatter_tails: group_size must be a positive int, got {group_size!r}")
    H, N_max = k.shape[1], tail_k.shape[2]
    if k.shape[0] != 1 or k.shape[2] < S_tot or tail_k.shape != (B * group_size, H, N_max, 128) or tail_v.shape != tail_k.shape:
        raise ValueError(f"kv_scatter_tails: rows {tuple(k.shape)} and tails {tuple(tail_k.shape)} do not fit {B} suffixes x "
                         f"{group_size} rows of {S_tot} packed rows")
    with torch.cuda.device(k.device):
        L.check(L.load().aria_kv_scatter_tails(_p(k), _p(v), k.stride(1), _p(tail_k), _p(tail_v), tail_k.stride(0), tail_k.stride(1),
                                               _p(cu_seqlens), B, group_size, H, S_tot, N_max, _stream(k)), "kv_scatter_tails")


# ------------------------------------------------------------------------------------------- generation
def sample_tokens(logits: torch.Tensor, temperature: float = 0.0, top_k: int = 0, top_p: float = 1.0, seed: int = 0,
                  rng_offset: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
                  probs_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Next token per row of bf16 logits [B, V] (contiguous last dim, any row stride, 0 repeats one row): transformers'
    temperature -> top-k -> top-p -> softmax -> multinomial on an fp32 copy; temperature 0 = greedy argmax (lowest id on ties).
    rng_offset: device int64 [1] read as the uint64 Philox offset (None: 0).  out: int64 [B] (allocated when None).
    probs_out: fp32 [B, V], receives the final distribution (zero outside the kept set).  See aria_sample_tokens."""
    if not (logits.is_cuda and logits.dtype == bf16 and logits.dim() == 2 and logits.stride(-1) == 1):
        raise RuntimeError("sample_tokens: logits must be CUDA bf16 [B, V] with a contiguous last dim")
    B, V = logits.shape
    if out is None:
        out = torch.empty((B,), dtype=torch.int64, device=logits.device)
    _chk(out, torch.int64, align=8)
    assert out.shape == (B,)
    if rng_offset is not None:
        _chk(rng_offset, torch.int64, align=8)
    if probs_out is not None:
        _chk(probs_out, torch.float32, align=4)
        assert probs_out.shape == (B, V)
    with torch.cuda.device(logits.device):
        L.check(L.load().aria_sample_tokens(_p(logits), logits.stride(0), _p(out), _p(probs_out), B, V, float(temperature),
                                            int(top_k), float(top_p), int(seed) & (2 ** 64 - 1), _p(rng_offset), _stream(logits)),
                "sample_tokens")
    return out


def kv_append(k_new: torch.Tensor, v_new: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, pos: torch.Tensor):
    """k_cache[b, :, pos[b]] = k_new[b], v_cache[b, :, pos[b]] = v_new[b]; k_new / v_new [B, H, 128] (any strides with 128
    contiguous elements), caches [B, H, T_max, 128], pos int32 [B] on the device."""
    _chk(k_cache), _chk(v_cache), _chk(pos, torch.int32, align=4)
    for t in (k_new, v_new):
        if not (t.is_cuda and t.dtype == bf16 and t.stride(-1) == 1 and t.data_ptr() % 16 == 0):
            raise RuntimeError("kv_append: new rows must be CUDA bf16 with a contiguous, 16-byte aligned last dim")
    assert k_new.stride() == v_new.stride() and k_cache.stride() == v_cache.stride()
    B, H, T_max = k_cache.shape[0], k_cache.shape[1], k_cache.shape[2]
    assert k_new.shape == (B, H, 128) and v_new.shape == (B, H, 128) and pos.shape == (B,)
    with torch.cuda.device(k_cache.device):
        L.check(L.load().aria_kv_append(_p(k_new), _p(v_new), k_new.stride(0), k_new.stride(1), _p(k_cache), _p(v_cache),
                                        k_cache.stride(0), k_cache.stride(1), _p(pos), B, H, T_max, _stream(k_cache)), "kv_append")


def sample_tokens_rows(logits: torch.Tensor, temperature: float, top_k: int, top_p: float, seed: int, noise_rows: torch.Tensor,
                       offsets: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """sample_tokens where logits row r [R, V] draws the Philox noise of row noise_rows[r] (CUDA int32 [R]) at offset
    offsets[r] (CUDA int64 [R], read as uint64): row r equals sample_tokens on that row with rng_offset = offsets[r] as row
    noise_rows[r].  out: int64 [R] (allocated when None).  See aria_sample_tokens_rows."""
    if not (logits.is_cuda and logits.dtype == bf16 and logits.dim() == 2 and logits.stride(-1) == 1):
        raise RuntimeError("sample_tokens_rows: logits must be CUDA bf16 [R, V] with a contiguous last dim")
    R, V = logits.shape
    if out is None:
        out = torch.empty((R,), dtype=torch.int64, device=logits.device)
    _chk(out, torch.int64, align=8), _chk(noise_rows, torch.int32, align=4), _chk(offsets, torch.int64, align=8)
    if out.shape != (R,) or noise_rows.shape != (R,) or offsets.shape != (R,):
        raise ValueError(f"sample_tokens_rows: out / noise_rows / offsets must be [{R}]")
    with torch.cuda.device(logits.device):
        L.check(L.load().aria_sample_tokens_rows(_p(logits), logits.stride(0), _p(out), R, V, float(temperature), int(top_k),
                                                 float(top_p), int(seed) & (2 ** 64 - 1), _p(noise_rows), _p(offsets),
                                                 _stream(logits)), "sample_tokens_rows")
    return out


def kv_append_rows(k_new: torch.Tensor, v_new: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, pos: torch.Tensor):
    """k_cache[b, :, pos[b] + i] = k_new[b, :, i] (and v) for the Q rows of k_new / v_new [B, H, Q, 128] (128 contiguous, 16-byte
    aligned elements per row); caches [B, H, T_max, 128], pos CUDA int32 [B].  Rows at or past T_max are dropped."""
    _chk(k_cache), _chk(v_cache), _chk(pos, torch.int32, align=4)
    for t in (k_new, v_new):
        if not (t.is_cuda and t.dtype == bf16 and t.dim() == 4 and t.stride(-1) == 1 and t.data_ptr() % 16 == 0):
            raise RuntimeError("kv_append_rows: new rows must be CUDA bf16 [B, H, Q, 128] with a contiguous, 16-byte aligned last dim")
    assert k_new.stride() == v_new.stride() and k_cache.stride() == v_cache.stride()
    B, H, T_max = k_cache.shape[0], k_cache.shape[1], k_cache.shape[2]
    Q = k_new.shape[2]
    assert k_new.shape == (B, H, Q, 128) and v_new.shape == k_new.shape and pos.shape == (B,)
    with torch.cuda.device(k_cache.device):
        L.check(L.load().aria_kv_append_rows(_p(k_new), _p(v_new), k_new.stride(0), k_new.stride(1), k_new.stride(2), _p(k_cache),
                                             _p(v_cache), k_cache.stride(0), k_cache.stride(1), _p(pos), B, Q, H, T_max,
                                             _stream(k_cache)), "kv_append_rows")


def _eos_array(eos_token_ids):
    eos = list(eos_token_ids)
    return (C.c_int64 * max(1, len(eos)))(*eos), len(eos)    # the caller holds the array across the call


def ngram_draft(hist: torch.Tensor, hist_len: torch.Tensor, finished: torch.Tensor, n_out: torch.Tensor, max_new: int,
                drafts: torch.Tensor, draft_len: torch.Tensor, any_draft: torch.Tensor, K: int, M: int,
                eos_token_ids: Sequence[int] = ()):
    """Prompt-lookup drafts of every row (Hugging Face's PromptLookupCandidateGenerator.get_candidates with num_output_tokens=K,
    max_matching_ngram_size=M) from hist [B, H_max] int64, the first hist_len[b] tokens of row b; then cut to
    max_new - 1 - n_out[b] tokens, none for a finished row.  Writes drafts [B, >= K] (int64, row stride any; entries past a draft
    repeat the last token), draft_len int32 [B], and any_draft int32 [>= 1] <- 1 when a row has a draft.  See aria_ngram_draft."""
    for t, dt in ((hist, torch.int64), (hist_len, torch.int32), (finished, torch.uint8), (n_out, torch.int32),
                  (draft_len, torch.int32), (any_draft, torch.int32)):
        _chk(t, dt, align=1)
    if not (drafts.is_cuda and drafts.dtype == torch.int64):
        raise RuntimeError("ngram_draft: drafts must be CUDA int64")
    B = hist.shape[0]
    if hist.dim() != 2 or drafts.dim() != 2 or drafts.stride(1) != 1 or drafts.shape[0] != B or drafts.shape[1] < K:
        raise ValueError(f"ngram_draft: hist must be [B, H_max] and drafts [B, >= {K}] with contiguous rows")
    assert hist_len.shape == (B,) and finished.shape == (B,) and n_out.shape == (B,) and draft_len.shape == (B,)
    eos, n_eos = _eos_array(eos_token_ids)
    with torch.cuda.device(hist.device):
        L.check(L.load().aria_ngram_draft(_p(hist), hist.stride(0), _p(hist_len), _p(finished), _p(n_out), int(max_new), _p(drafts),
                                          drafts.stride(0), _p(draft_len), _p(any_draft), B, int(K), int(M), C.cast(eos, C.c_void_p), n_eos,
                                          _stream(hist)), "ngram_draft")


def lookup_accept_advance(targets: torch.Tensor, step_ids: torch.Tensor, draft_len: torch.Tensor, ids1: torch.Tensor,
                          idsk: torch.Tensor, pos_k: torch.Tensor, lens_k: torch.Tensor, off1: torch.Tensor, offk: torch.Tensor,
                          out_tokens: torch.Tensor, hist: torch.Tensor, hist_len: torch.Tensor, n_out: torch.Tensor,
                          finished: torch.Tensor, rope_pos: torch.Tensor, write_pos: torch.Tensor, kv_len: torch.Tensor,
                          status: torch.Tensor, counters: torch.Tensor, eos_token_ids: Sequence[int] = ()):
    """Accept / emit / advance after a prompt-lookup step of width Q = step_ids.shape[1] (1, or K + 1 = idsk.shape[1]): targets
    [B*Q] sampled, step_ids [B, Q] the step's input (last token, then the drafts of draft_len [B]).  Emits each live row's accepted
    drafts plus one token into out_tokens [B, max_new] and hist, applies the EOS rule, moves the positions on and writes the next
    step's inputs (ids1 [B], idsk[:, 0], pos_k / lens_k int32 and off1 / offk int64 offsets), status int32 [2] (every row done,
    any draft = 0) and counters int64 [2] (drafts verified, accepted).  See aria_lookup_accept_advance."""
    i64, i32 = torch.int64, torch.int32
    for t, dt in ((targets, i64), (step_ids, i64), (draft_len, i32), (ids1, i64), (idsk, i64), (pos_k, i32), (lens_k, i32),
                  (off1, i64), (offk, i64), (out_tokens, i64), (hist, i64), (hist_len, i32), (n_out, i32),
                  (finished, torch.uint8), (rope_pos, i32), (write_pos, i32), (kv_len, i32), (status, i32), (counters, i64)):
        _chk(t, dt, align=1)
    B, Q = step_ids.shape
    Kp1 = idsk.shape[1]
    if (targets.numel() != B * Q or idsk.shape != (B, Kp1) or pos_k.numel() != B * Kp1 or lens_k.numel() != B * Kp1
            or offk.numel() != B * Kp1 or ids1.numel() != B or off1.numel() != B or out_tokens.shape[0] != B
            or hist.shape[0] != B or hist.stride(1) != 1 or status.numel() < 2 or counters.numel() < 2):
        raise ValueError("lookup_accept_advance: the buffers do not fit one another")
    eos, n_eos = _eos_array(eos_token_ids)
    with torch.cuda.device(targets.device):
        L.check(L.load().aria_lookup_accept_advance(_p(targets), _p(step_ids), _p(draft_len), Q, _p(ids1), _p(idsk), Kp1, _p(pos_k),
                                                    _p(lens_k), _p(off1), _p(offk), _p(out_tokens), out_tokens.shape[1], _p(hist),
                                                    hist.stride(0), _p(hist_len), _p(n_out), _p(finished), _p(rope_pos),
                                                    _p(write_pos), _p(kv_len), _p(status), _p(counters), C.cast(eos, C.c_void_p), n_eos, B,
                                                    _stream(targets)), "lookup_accept_advance")


def _bf16_rows_check(ts, what: str):
    for t in ts:
        if not (t.is_cuda and t.dtype == bf16 and t.stride(-1) == 1 and t.data_ptr() % 16 == 0
                and (t.dim() == 3 or t.stride(-2) == 128)):
            raise RuntimeError(f"{what}: bf16 rows must be CUDA bf16 with 128 contiguous, 16-byte aligned elements per row")
    if ts[0].stride() != ts[1].stride() or ts[0].shape != ts[1].shape:
        raise RuntimeError(f"{what}: the k and v rows must share shape and strides")


def kv_store_fp8(k_src: torch.Tensor, v_src: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, k_scale: torch.Tensor,
                 v_scale: torch.Tensor, row0: int):
    """Quantise bf16 rows k_src / v_src [B, H, n, 128] (row stride 128, e.g. rows of the staging pair) into fp8 cache rows
    [row0, row0 + n): one fp32 scale per (row, head, token) = amax / 448 (1 for an all-zero row), codes e4m3(x / scale), bit for
    bit `(x.float() / scale[..., None]).to(torch.float8_e4m3fn)`."""
    _fp8_cache_check(k_cache, v_cache, k_scale, v_scale, "kv_store_fp8")
    _bf16_rows_check((k_src, v_src), "kv_store_fp8")
    B, H, T_max = k_cache.shape[:3]
    n = k_src.shape[2]
    if k_src.shape != (B, H, n, 128) or not 0 <= row0 <= T_max - n:
        raise ValueError(f"kv_store_fp8: rows {tuple(k_src.shape)} at row {row0} do not fit a cache of {tuple(k_cache.shape)}")
    with torch.cuda.device(k_cache.device):
        L.check(L.load().aria_kv_store_fp8(_p(k_src), _p(v_src), k_src.stride(0), k_src.stride(1), _p(k_cache), _p(v_cache),
                                           _p(k_scale), _p(v_scale), k_cache.stride(0), k_cache.stride(1), k_scale.stride(0),
                                           k_scale.stride(1), row0, n, B, H, T_max, _stream(k_cache)), "kv_store_fp8")


def kv_append_fp8(k_new: torch.Tensor, v_new: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, k_scale: torch.Tensor,
                  v_scale: torch.Tensor, pos: torch.Tensor):
    """kv_append for the fp8 cache: quantise k_new / v_new [B, H, 128] into cache row pos[b] (int32 [B] on the device) with the
    quantiser of kv_store_fp8, so the row gets the same codes and scale as kv_store_fp8 would give it."""
    _fp8_cache_check(k_cache, v_cache, k_scale, v_scale, "kv_append_fp8")
    _bf16_rows_check((k_new, v_new), "kv_append_fp8")
    _chk(pos, torch.int32, align=4)
    B, H, T_max = k_cache.shape[:3]
    assert k_new.shape == (B, H, 128) and pos.shape == (B,)
    with torch.cuda.device(k_cache.device):
        L.check(L.load().aria_kv_append_fp8(_p(k_new), _p(v_new), k_new.stride(0), k_new.stride(1), _p(k_cache), _p(v_cache),
                                            _p(k_scale), _p(v_scale), k_cache.stride(0), k_cache.stride(1), k_scale.stride(0),
                                            k_scale.stride(1), _p(pos), B, H, T_max, _stream(k_cache)), "kv_append_fp8")


def kv_load_fp8(k_cache: torch.Tensor, v_cache: torch.Tensor, k_scale: torch.Tensor, v_scale: torch.Tensor, k_out: torch.Tensor,
                v_out: torch.Tensor, n: int):
    """Dequantise fp8 cache rows [0, n) into bf16 k_out / v_out [B, H, >= n, 128] (row stride 128): bf16(code.float() * scale)."""
    _fp8_cache_check(k_cache, v_cache, k_scale, v_scale, "kv_load_fp8")
    _bf16_rows_check((k_out, v_out), "kv_load_fp8")
    B, H, T_max = k_cache.shape[:3]
    if k_out.shape[:2] != (B, H) or k_out.shape[2] < n or not 0 < n <= T_max:
        raise ValueError(f"kv_load_fp8: {n} rows of a cache of {tuple(k_cache.shape)} do not fit {tuple(k_out.shape)}")
    with torch.cuda.device(k_cache.device):
        L.check(L.load().aria_kv_load_fp8(_p(k_cache), _p(v_cache), _p(k_scale), _p(v_scale), k_cache.stride(0), k_cache.stride(1),
                                          k_scale.stride(0), k_scale.stride(1), _p(k_out), _p(v_out), k_out.stride(0),
                                          k_out.stride(1), n, B, H, T_max, _stream(k_cache)), "kv_load_fp8")


# ------------------------------------------------------------------------------------------- continuous batching (paged KV cache)
def _paged_pool_check(k_pool: torch.Tensor, v_pool: torch.Tensor, what: str):
    """Page pools k_pool / v_pool: CUDA bf16 [n_pages, H, 256, 128], contiguous and sharing one shape."""
    for t in (k_pool, v_pool):
        _chk(t)
        if t.dim() != 4 or t.shape[2:] != (256, 128):
            raise RuntimeError(f"{what}: page pools must be bf16 [n_pages, H, 256, 128], got {tuple(t.shape)}")
    if k_pool.shape != v_pool.shape:
        raise RuntimeError(f"{what}: k_pool and v_pool must share one shape")


def _paged_fp8_pool_check(k_pool: torch.Tensor, v_pool: torch.Tensor, k_scale: Optional[torch.Tensor],
                          v_scale: Optional[torch.Tensor], what: str):
    """fp8 KV pages: e4m3 code pools k_pool / v_pool [n_pages, H, 256, 128] and fp32 scale pools k_scale / v_scale
    [n_pages, H, 256], each contiguous, the code pools sharing one shape and the scale pools theirs."""
    if k_scale is None or v_scale is None:
        raise ValueError(f"{what}: fp8 (float8_e4m3fn) page pools need k_scale= and v_scale=")
    for t in (k_pool, v_pool):
        if not (t.is_cuda and t.dtype == fp8 and t.dim() == 4 and t.shape[2:] == (256, 128) and t.is_contiguous()
                and t.data_ptr() % 16 == 0):
            raise RuntimeError(f"{what}: fp8 page pools must be contiguous CUDA float8_e4m3fn [n_pages, H, 256, 128]")
    for t in (k_scale, v_scale):
        if not (t.is_cuda and t.dtype == torch.float32 and t.shape == k_pool.shape[:3] and t.is_contiguous()):
            raise RuntimeError(f"{what}: k_scale / v_scale must be contiguous CUDA float32 [n_pages, H, 256]")
    if k_pool.shape != v_pool.shape:
        raise RuntimeError(f"{what}: k_pool and v_pool must share one shape")


def _block_table_check(block_table: torch.Tensor, rows: int, what: str):
    """Block table: CUDA int32 [>= rows, max_pages] with contiguous rows (any row stride)."""
    if not (block_table.is_cuda and block_table.dtype == torch.int32 and block_table.dim() == 2 and block_table.stride(1) == 1
            and block_table.shape[0] >= rows and block_table.shape[1] >= 1):
        raise RuntimeError(f"{what}: block_table must be CUDA int32 [>= {rows}, max_pages] with contiguous rows")


def attention_decode_paged(q: torch.Tensor, k_pool: torch.Tensor, v_pool: torch.Tensor, block_table: torch.Tensor,
                           lens: torch.Tensor, scale: float, k_scale: Optional[torch.Tensor] = None,
                           v_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """attention_decode_devlen over a paged cache: q [R, H, 128] (contiguous last dim), page pools [n_pages, H, 256, 128] bf16,
    block_table int32 [>= R, max_pages] (row r's key 256 s + i is row i of page block_table[r, s]; its columns are the splits the
    grid covers), lens int32 [R] -> out [R, H*128].  Row r is bit-identical to attention_decode_devlen on a contiguous cache
    holding the same keys.  With fp8 pools (float8_e4m3fn) k_scale / v_scale [n_pages, H, 256] fp32 are required and the fp8
    kernel runs, bit-identical to the fp8 attention_decode_devlen on the same codes and scales.  See
    aria_attention_decode_paged(_fp8)."""
    is_fp8 = k_pool.dtype == fp8
    if is_fp8:
        _paged_fp8_pool_check(k_pool, v_pool, k_scale, v_scale, "attention_decode_paged")
    else:
        _paged_pool_check(k_pool, v_pool, "attention_decode_paged")
    _chk(lens, torch.int32, align=4)
    if not (q.is_cuda and q.dtype == bf16 and q.dim() == 3 and q.stride(-1) == 1 and q.data_ptr() % 8 == 0):
        raise RuntimeError("attention_decode_paged: q must be a CUDA bf16 [R, H, 128] tensor with a contiguous last dim")
    R, H = q.shape[0], q.shape[1]
    _block_table_check(block_table, R, "attention_decode_paged")
    if q.shape[2] != 128 or k_pool.shape[1] != H or lens.shape != (R,):
        raise ValueError(f"attention_decode_paged: q {tuple(q.shape)}, pools {tuple(k_pool.shape)} and lens {tuple(lens.shape)} "
                         "do not fit one another")
    max_pages = block_table.shape[1]
    lib = L.load()
    ws_bytes = lib.aria_attention_decode_workspace_bytes(R, H, max_pages * 256)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=q.device)
    out = torch.empty((R, H * 128), dtype=bf16, device=q.device)
    with torch.cuda.device(q.device):
        if is_fp8:
            L.check(lib.aria_attention_decode_paged_fp8(_p(q), _p(k_pool), _p(v_pool), _p(k_scale), _p(v_scale), _p(block_table),
                                                        block_table.stride(0), max_pages, k_pool.shape[0], _p(lens), _p(out), R, H,
                                                        q.stride(0), q.stride(1), k_pool.stride(0), k_pool.stride(1),
                                                        k_scale.stride(0), k_scale.stride(1), scale, _p(ws), ws_bytes, _stream(q)),
                    "attention_decode_paged_fp8")
            return out
        L.check(lib.aria_attention_decode_paged(_p(q), _p(k_pool), _p(v_pool), _p(block_table), block_table.stride(0), max_pages,
                                                k_pool.shape[0], _p(lens), _p(out), R, H, q.stride(0), q.stride(1),
                                                k_pool.stride(0), k_pool.stride(1), scale, _p(ws), ws_bytes, _stream(q)),
                "attention_decode_paged")
    return out


def kv_append_paged(k_new: torch.Tensor, v_new: torch.Tensor, k_pool: torch.Tensor, v_pool: torch.Tensor,
                    block_table: torch.Tensor, write_pos: torch.Tensor, k_scale: Optional[torch.Tensor] = None,
                    v_scale: Optional[torch.Tensor] = None):
    """kv_append into a paged cache: k_new / v_new [R, H, 128] (128 contiguous, 16-byte aligned elements per row) go to row
    write_pos[r] % 256 of page block_table[r, write_pos[r] // 256] (write_pos CUDA int32 [R]).  A negative write_pos, one past
    the table's columns, or an entry outside the pool writes nothing.  With fp8 pools (k_scale / v_scale [n_pages, H, 256]
    required) the rows are quantized as kv_append_fp8 quantizes them, and the null page 0 is never written either.  See
    aria_kv_append_paged(_fp8)."""
    is_fp8 = k_pool.dtype == fp8
    if is_fp8:
        _paged_fp8_pool_check(k_pool, v_pool, k_scale, v_scale, "kv_append_paged")
    else:
        _paged_pool_check(k_pool, v_pool, "kv_append_paged")
    _chk(write_pos, torch.int32, align=4)
    for t in (k_new, v_new):
        if not (t.is_cuda and t.dtype == bf16 and t.dim() == 3 and t.stride(-1) == 1 and t.data_ptr() % 16 == 0):
            raise RuntimeError("kv_append_paged: new rows must be CUDA bf16 [R, H, 128] with a contiguous, 16-byte aligned last dim")
    if k_new.stride() != v_new.stride() or k_new.shape != v_new.shape:
        raise RuntimeError("kv_append_paged: k_new and v_new must share shape and strides")
    R, H = k_new.shape[0], k_new.shape[1]
    _block_table_check(block_table, R, "kv_append_paged")
    if k_new.shape[2] != 128 or k_pool.shape[1] != H or write_pos.shape != (R,):
        raise ValueError("kv_append_paged: the rows, pools and write_pos do not fit one another")
    with torch.cuda.device(k_pool.device):
        if is_fp8:
            L.check(L.load().aria_kv_append_paged_fp8(_p(k_new), _p(v_new), k_new.stride(0), k_new.stride(1), _p(k_pool),
                                                      _p(v_pool), _p(k_scale), _p(v_scale), k_pool.stride(0), k_pool.stride(1),
                                                      k_scale.stride(0), k_scale.stride(1), _p(block_table), block_table.stride(0),
                                                      block_table.shape[1], k_pool.shape[0], _p(write_pos), R, H, _stream(k_pool)),
                    "kv_append_paged_fp8")
            return
        L.check(L.load().aria_kv_append_paged(_p(k_new), _p(v_new), k_new.stride(0), k_new.stride(1), _p(k_pool), _p(v_pool),
                                              k_pool.stride(0), k_pool.stride(1), _p(block_table), block_table.stride(0),
                                              block_table.shape[1], k_pool.shape[0], _p(write_pos), R, H, _stream(k_pool)),
                "kv_append_paged")


def kv_pages_store(k: torch.Tensor, v: torch.Tensor, T: int, k_pool: torch.Tensor, v_pool: torch.Tensor, pages: torch.Tensor):
    """Rows [0, T) of a one-row contiguous cache k / v [1, H, >= T, 128] (bf16, contiguous) into the pages of one request: row t
    to row t % 256 of page pages[t // 256] (pages CUDA int32 [max_pages], e.g. a block-table row).  See aria_kv_pages_store."""
    _paged_pool_check(k_pool, v_pool, "kv_pages_store")
    _chk(k), _chk(v), _chk(pages, torch.int32, align=4)
    H = k_pool.shape[1]
    if (k.dim() != 4 or k.shape[0] != 1 or k.shape[1] != H or k.shape[3] != 128 or v.shape != k.shape or pages.dim() != 1
            or not 0 < T <= min(k.shape[2], 256 * pages.numel())):
        raise ValueError(f"kv_pages_store: {T} rows of {tuple(k.shape)} do not fit {pages.numel()} pages of {tuple(k_pool.shape)}")
    with torch.cuda.device(k_pool.device):
        L.check(L.load().aria_kv_pages_store(_p(k), _p(v), k.stride(1), int(T), _p(k_pool), _p(v_pool), k_pool.stride(0),
                                             k_pool.stride(1), _p(pages), pages.numel(), k_pool.shape[0], H, _stream(k_pool)),
                "kv_pages_store")


def attention_prefill_paged_prefix(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, S_tot: int, k_pool: torch.Tensor,
                                   v_pool: torch.Tensor, pages: Optional[torch.Tensor], P: int, cu_seqlens: torch.Tensor,
                                   scale: float) -> torch.Tensor:
    """attention_prefill_shared_prefix with the prefix read from pool pages (prefix caching): q / k / v, S_tot and cu_seqlens as
    there; the prefix is P keys (a multiple of 256), key 256 i + r at row r of page pages[i] (pages CUDA int32 [>= P / 256]) of the
    pools [n_pages, H, 256, 128].  P = 0 is no prefix (pages may be None): the varlen causal forward -> out [S_tot, H*128].  Every
    row is bit-identical to attention_prefill_shared_prefix on a contiguous copy of the prefix (P = 0: attention_varlen).  A page
    entry outside the pool reads zeros.  See aria_attention_prefill_paged_prefix."""
    what = "attention_prefill_paged_prefix"
    _attn_qkv_check(q, k, v, what)
    _paged_pool_check(k_pool, v_pool, what)
    B = _packed_check(S_tot, cu_seqlens, what)
    H = q.shape[1]
    if q.shape[0] != 1 or q.shape[2] < S_tot or k.shape[:2] != (1, H) or k.shape[2] < S_tot or v.shape != k.shape:
        raise ValueError(f"{what}: q {tuple(q.shape)} / k {tuple(k.shape)} must be [1, H, >= {S_tot}, 128]")
    if k_pool.shape[1] != H:
        raise ValueError(f"{what}: pools {tuple(k_pool.shape)} do not have the {H} heads of q")
    n_list = 0
    if pages is not None:
        _chk(pages, torch.int32, align=4)
        if pages.dim() != 1:
            raise ValueError(f"{what}: pages must be int32 [n], got {tuple(pages.shape)}")
        n_list = pages.numel()
    if not isinstance(P, int) or P < 0 or P % 256 or P // 256 > n_list:
        raise ValueError(f"{what}: P must be a multiple of 256 in [0, 256 x {n_list} listed pages], got {P!r}")
    out = torch.empty((S_tot, H * 128), dtype=bf16, device=q.device)
    with torch.cuda.device(q.device):
        L.check(L.load().aria_attention_prefill_paged_prefix(_p(q), _p(k), _p(v), _p(k_pool), _p(v_pool), _p(pages), n_list,
                                                             k_pool.shape[0], _p(cu_seqlens), _p(out), B, H, S_tot, P,
                                                             q.stride(1), k.stride(1), k_pool.stride(0), k_pool.stride(1), scale,
                                                             _stream(q)), what)
    return out


class PackedSegments:
    """n_seg prompt segments packed along one row, each after a paged prefix of its own: segment b is packed rows
    [cu[b], cu[b + 1]) and follows prefix_lens[b] cached keys (a multiple of 256).  Holds the host lists, which the ops below
    check before they launch, and one device int32 copy of both (cu_dev [n_seg + 1], prefix_dev [n_seg]), which the kernels
    read.  Every segment has at least one row."""

    def __init__(self, cu, prefix_lens, device):
        cu, P = [int(c) for c in cu], [int(p) for p in prefix_lens]
        if len(cu) < 2 or cu[0] != 0 or any(b <= a for a, b in zip(cu, cu[1:])) or len(P) != len(cu) - 1:
            raise ValueError(f"PackedSegments: cu must increase from 0 with one prefix length per segment, got {cu} and {P}")
        if any(p < 0 or p % 256 for p in P):
            raise ValueError(f"PackedSegments: prefix lengths must be multiples of 256, got {P}")
        self.cu, self.prefix_lens = cu, P
        dev = torch.tensor(cu + P, dtype=torch.int32).pin_memory().to(device, non_blocking=True)
        self.cu_dev, self.prefix_dev = dev[:len(cu)], dev[len(cu):]

    @property
    def n_seg(self) -> int:
        return len(self.prefix_lens)

    @property
    def S_tot(self) -> int:
        return self.cu[-1]


def _page_table_check(page_table: torch.Tensor, seg: PackedSegments, rows_after_prefix: bool, what: str):
    """page_table: CUDA int32 [n_seg, width] with contiguous rows; every prefix (and, rows_after_prefix, the segment's rows after
    it) fits the width's pages."""
    if not (page_table.is_cuda and page_table.dtype == torch.int32 and page_table.dim() == 2 and page_table.stride(1) == 1
            and page_table.shape[0] == seg.n_seg and page_table.shape[1] >= 1 and page_table.data_ptr() % 4 == 0):
        raise RuntimeError(f"{what}: page_table must be CUDA int32 [{seg.n_seg}, width] with contiguous rows")
    W = page_table.shape[1]
    for b, P in enumerate(seg.prefix_lens):
        end = P + (seg.cu[b + 1] - seg.cu[b] if rows_after_prefix else 0)
        if end > 256 * W:
            raise ValueError(f"{what}: segment {b} needs {-(-end // 256)} pages; its page_table row lists {W}")


def attention_prefill_paged_varlen(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, k_pool: torch.Tensor, v_pool: torch.Tensor,
                                   page_table: torch.Tensor, seg: PackedSegments, scale: float) -> torch.Tensor:
    """attention_prefill_paged_prefix with a prefix per segment: q / k / v [1, H, >= seg.S_tot, 128] hold the packed segments
    (seg), segment b attends to its seg.prefix_lens[b] keys, key 256 i + r at row r of page page_table[b, i] (CUDA int32
    [n_seg, width]) of the pools [n_pages, H, 256, 128], and causally to its own rows -> out [S_tot, H*128].  Every row of segment
    b is bit-identical to attention_prefill_paged_prefix on that segment alone, with its own page list and P.  A page entry
    outside the pool reads zeros.  See aria_attention_prefill_paged_varlen."""
    what = "attention_prefill_paged_varlen"
    _attn_qkv_check(q, k, v, what)
    _paged_pool_check(k_pool, v_pool, what)
    S_tot, H = seg.S_tot, q.shape[1]
    if q.shape[0] != 1 or q.shape[2] < S_tot or k.shape[:2] != (1, H) or k.shape[2] < S_tot or v.shape != k.shape:
        raise ValueError(f"{what}: q {tuple(q.shape)} / k {tuple(k.shape)} must be [1, H, >= {S_tot}, 128]")
    if k_pool.shape[1] != H:
        raise ValueError(f"{what}: pools {tuple(k_pool.shape)} do not have the {H} heads of q")
    _page_table_check(page_table, seg, False, what)
    out = torch.empty((S_tot, H * 128), dtype=bf16, device=q.device)
    with torch.cuda.device(q.device):
        L.check(L.load().aria_attention_prefill_paged_varlen(_p(q), _p(k), _p(v), _p(k_pool), _p(v_pool), _p(page_table),
                                                             page_table.stride(0), k_pool.shape[0], _p(seg.prefix_dev),
                                                             _p(seg.cu_dev), _p(out), seg.n_seg, H, S_tot, q.stride(1), k.stride(1),
                                                             k_pool.stride(0), k_pool.stride(1), scale, _stream(q)), what)
    return out


def kv_pages_store_varlen(k: torch.Tensor, v: torch.Tensor, k_pool: torch.Tensor, v_pool: torch.Tensor, page_table: torch.Tensor,
                          seg: PackedSegments, k_scale: Optional[torch.Tensor] = None, v_scale: Optional[torch.Tensor] = None):
    """kv_pages_store for packed segments: row t of segment b of k / v [1, H, >= S_tot, 128] (bf16, contiguous) is position
    p = prefix_lens[b] + t - cu[b] of its request and goes to row p % 256 of page page_table[b, p // 256].  Writes nothing outside
    the listed pages and never the null page 0; each segment's pages are those kv_pages_store gives it alone.
    With fp8 pools (k_scale / v_scale [n_pages, H, 256] required) the rows are quantized as kv_store_fp8 quantizes them, and
    rows [0, S_tot) of k / v are overwritten in place with bf16(code * scale), the values a later read of the pages gives
    (kv_pages_load_fp8).  See aria_kv_pages_store_varlen(_fp8)."""
    what = "kv_pages_store_varlen"
    is_fp8 = k_pool.dtype == fp8
    if is_fp8:
        _paged_fp8_pool_check(k_pool, v_pool, k_scale, v_scale, what)
    else:
        _paged_pool_check(k_pool, v_pool, what)
    _chk(k), _chk(v)
    H, S_tot = k_pool.shape[1], seg.S_tot
    if k.dim() != 4 or k.shape[0] != 1 or k.shape[1] != H or k.shape[3] != 128 or v.shape != k.shape or k.shape[2] < S_tot:
        raise ValueError(f"{what}: k {tuple(k.shape)} must be [1, {H}, >= {S_tot}, 128] like v")
    _page_table_check(page_table, seg, True, what)
    with torch.cuda.device(k_pool.device):
        if is_fp8:
            L.check(L.load().aria_kv_pages_store_varlen_fp8(_p(k), _p(v), k.stride(1), S_tot, _p(k_pool), _p(v_pool), _p(k_scale),
                                                            _p(v_scale), k_pool.stride(0), k_pool.stride(1), k_scale.stride(0),
                                                            k_scale.stride(1), _p(page_table), page_table.stride(0),
                                                            page_table.shape[1], k_pool.shape[0], _p(seg.prefix_dev),
                                                            _p(seg.cu_dev), seg.n_seg, H, _stream(k_pool)), what + "_fp8")
            return
        L.check(L.load().aria_kv_pages_store_varlen(_p(k), _p(v), k.stride(1), S_tot, _p(k_pool), _p(v_pool), k_pool.stride(0),
                                                    k_pool.stride(1), _p(page_table), page_table.stride(0), page_table.shape[1],
                                                    k_pool.shape[0], _p(seg.prefix_dev), _p(seg.cu_dev), seg.n_seg, H,
                                                    _stream(k_pool)), what)


def kv_pages_load_fp8(k_pool: torch.Tensor, v_pool: torch.Tensor, k_scale: torch.Tensor, v_scale: torch.Tensor,
                      pages: torch.Tensor, k_out: torch.Tensor, v_out: torch.Tensor):
    """Dequantize pages pages[i] (CUDA int32 [n]) of fp8 page pools into page i of bf16 pools k_out / v_out [>= n, H, 256, 128]
    (contiguous): bf16(code.float() * scale), the values kv_load_fp8 gives the same rows.  An entry outside the pool gives zeros.
    See aria_kv_pages_load_fp8."""
    what = "kv_pages_load_fp8"
    _paged_fp8_pool_check(k_pool, v_pool, k_scale, v_scale, what)
    _paged_pool_check(k_out, v_out, what)
    _chk(pages, torch.int32, align=4)
    H = k_pool.shape[1]
    if pages.dim() != 1 or pages.numel() < 1 or k_out.shape[0] < pages.numel() or k_out.shape[1] != H:
        raise ValueError(f"{what}: {tuple(pages.shape)} pages of {tuple(k_pool.shape)} do not fit {tuple(k_out.shape)}")
    with torch.cuda.device(k_pool.device):
        L.check(L.load().aria_kv_pages_load_fp8(_p(k_pool), _p(v_pool), _p(k_scale), _p(v_scale), k_pool.stride(0), k_pool.stride(1),
                                                k_scale.stride(0), k_scale.stride(1), _p(pages), pages.numel(), k_pool.shape[0],
                                                _p(k_out), _p(v_out), k_out.stride(0), k_out.stride(1), H, _stream(k_pool)), what)


def sample_tokens_slots(logits: torch.Tensor, temperature: torch.Tensor, top_k: torch.Tensor, top_p: torch.Tensor,
                        seed: torch.Tensor, noise_rows: torch.Tensor, offsets: torch.Tensor,
                        out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """sample_tokens_rows with every parameter per row, CUDA arrays [R]: temperature fp32 (0 = greedy), top_k int32, top_p fp32,
    seed int64 (read as uint64), noise_rows int32, offsets int64 (read as uint64).  Row r equals sample_tokens on that row with
    its own scalars, rng_offset = offsets[r], as row noise_rows[r].  out: int64 [R] (allocated when None).  The caller checks
    the parameters as generate() does.  See aria_sample_tokens_slots."""
    if not (logits.is_cuda and logits.dtype == bf16 and logits.dim() == 2 and logits.stride(-1) == 1):
        raise RuntimeError("sample_tokens_slots: logits must be CUDA bf16 [R, V] with a contiguous last dim")
    R, V = logits.shape
    if out is None:
        out = torch.empty((R,), dtype=torch.int64, device=logits.device)
    args = ((out, torch.int64), (temperature, torch.float32), (top_k, torch.int32), (top_p, torch.float32), (seed, torch.int64),
            (noise_rows, torch.int32), (offsets, torch.int64))
    for t, dt in args:
        _chk(t, dt, align=4)
        if t.shape != (R,):
            raise ValueError(f"sample_tokens_slots: out and every per-row array must be [{R}], got {tuple(t.shape)}")
    with torch.cuda.device(logits.device):
        L.check(L.load().aria_sample_tokens_slots(_p(logits), logits.stride(0), _p(out), R, V, _p(temperature), _p(top_k), _p(top_p),
                                                  _p(seed), _p(noise_rows), _p(offsets), _stream(logits)), "sample_tokens_slots")
    return out


PROCESSED_MAX_VOCAB = 1 << 18   # the presence bitmap of a row is staged in the sampler's shared memory


def presence_words(V: int) -> int:
    """int32 words of one row's token-presence bitmap over a vocabulary of V ids."""
    return (V + 31) // 32


def sample_tokens_processed(logits: torch.Tensor, temperature: torch.Tensor, top_k: torch.Tensor, top_p: torch.Tensor,
                            min_p: torch.Tensor, seed: torch.Tensor, repetition_penalty: torch.Tensor,
                            min_new_tokens: torch.Tensor, presence: torch.Tensor, rng_offset: torch.Tensor,
                            n_emitted: torch.Tensor, eos_token_ids: Sequence[int] = (), noise_rows: Optional[torch.Tensor] = None,
                            out: Optional[torch.Tensor] = None, probs_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """sample_tokens_slots behind Hugging Face's repetition penalty, min_new_tokens and min-p, every parameter per row, CUDA
    arrays [R]: temperature fp32 (0 = greedy), top_k int32, top_p fp32, min_p fp32 (0 = off), seed int64 (read as uint64),
    repetition_penalty fp32 (1 = off), min_new_tokens int32.  presence: int32 [R, presence_words(V)], the ids each row has seen
    (presence_set).  rng_offset int64 and n_emitted int32 (tokens the row has emitted): [R], or [1] for every row.  noise_rows:
    int32 [R], or None for row r.  eos_token_ids: at most 8 ids, masked while a row has emitted fewer than its min_new_tokens.
    out: int64 [R] (allocated when None); probs_out: fp32 [R, V], the final distribution.  The caller checks the parameters as
    generate() does.  See aria_sample_tokens_processed."""
    if not (logits.is_cuda and logits.dtype == bf16 and logits.dim() == 2 and logits.stride(-1) == 1):
        raise RuntimeError("sample_tokens_processed: logits must be CUDA bf16 [R, V] with a contiguous last dim")
    R, V = logits.shape
    if out is None:
        out = torch.empty((R,), dtype=torch.int64, device=logits.device)
    args = ((out, torch.int64), (temperature, torch.float32), (top_k, torch.int32), (top_p, torch.float32), (min_p, torch.float32),
            (seed, torch.int64), (repetition_penalty, torch.float32), (min_new_tokens, torch.int32))
    if noise_rows is not None:
        args += ((noise_rows, torch.int32),)
    for t, dt in args:
        _chk(t, dt, align=4)
        if t.shape != (R,):
            raise ValueError(f"sample_tokens_processed: out and every per-row array must be [{R}], got {tuple(t.shape)}")
    for t, dt, name in ((rng_offset, torch.int64, "rng_offset"), (n_emitted, torch.int32, "n_emitted")):
        _chk(t, dt, align=4)
        if t.shape not in ((1,), (R,)):
            raise ValueError(f"sample_tokens_processed: {name} must be [1] or [{R}], got {tuple(t.shape)}")
    _chk(presence, torch.int32, align=4)
    if presence.shape != (R, presence_words(V)):
        raise ValueError(f"sample_tokens_processed: presence must be [{R}, {presence_words(V)}], got {tuple(presence.shape)}")
    if probs_out is not None:
        _chk(probs_out, torch.float32, align=4)
        if probs_out.shape != (R, V):
            raise ValueError(f"sample_tokens_processed: probs_out must be [{R}, {V}], got {tuple(probs_out.shape)}")
    eos, n_eos = _eos_array(eos_token_ids)
    with torch.cuda.device(logits.device):
        L.check(L.load().aria_sample_tokens_processed(
            _p(logits), logits.stride(0), _p(out), _p(probs_out), R, V, _p(temperature), _p(top_k), _p(top_p), _p(min_p), _p(seed),
            _p(repetition_penalty), _p(min_new_tokens), _p(presence), _p(noise_rows), _p(rng_offset),
            int(rng_offset.numel() == R and R > 1), _p(n_emitted), int(n_emitted.numel() == R and R > 1),
            C.cast(eos, C.c_void_p), n_eos, _stream(logits)), "sample_tokens_processed")
    return out


def presence_set(ids: torch.Tensor, presence: torch.Tensor, V: int, lengths: Optional[torch.Tensor] = None,
                 clear: bool = False) -> torch.Tensor:
    """Set bit id of presence row r (int32 [R, presence_words(V)]) for every id of ids row r (CUDA int64 [R, T], contiguous
    last dim, any row stride), only its first lengths[r] (CUDA int32 [R]) when given; ids outside [0, V) are skipped.  clear:
    zero each row first.  -> presence.  See aria_presence_set."""
    if not (ids.is_cuda and ids.dtype == torch.int64 and ids.dim() == 2 and ids.stride(-1) == 1):
        raise RuntimeError("presence_set: ids must be CUDA int64 [R, T] with a contiguous last dim")
    R, T = ids.shape
    _chk(presence, torch.int32, align=4)
    if presence.shape != (R, presence_words(V)):
        raise ValueError(f"presence_set: presence must be [{R}, {presence_words(V)}], got {tuple(presence.shape)}")
    if lengths is not None:
        _chk(lengths, torch.int32, align=4)
        if lengths.shape != (R,):
            raise ValueError(f"presence_set: lengths must be [{R}], got {tuple(lengths.shape)}")
    with torch.cuda.device(ids.device):
        L.check(L.load().aria_presence_set(_p(ids), ids.stride(0), R, T, _p(lengths), int(bool(clear)), _p(presence), int(V),
                                           _stream(ids)), "presence_set")
    return presence


MAX_LOGPROBS = 20


def token_logprobs(logits: torch.Tensor, tokens: torch.Tensor, n_max: int, *, n_row: Optional[torch.Tensor] = None,
                   col: Optional[torch.Tensor] = None, ring: int = 0, finished: Optional[torch.Tensor] = None,
                   finished_fill: bool = True, out: Optional[tuple] = None) -> tuple:
    """Log-probabilities of `tokens` (CUDA int64 [R]) under the raw distribution of each row of bf16 logits [R, V] (contiguous
    last dim, any row stride): lp = (x_t - max) - log(sum exp(x - max)) in fp32, and the n_max (0..20) largest logits of the row
    by (value desc, id asc) with their logprobs.  -> (logprobs, top_ids int32, top_logprobs), allocated as [R], [R, n_max],
    [R, n_max] when out is None; else out = (logprobs [R] or [R, cols] fp32, top_ids [R(, cols), n_max] int32, top_logprobs
    likewise fp32) and row r writes column c of its output row:
      col: None -> c = 0; a CUDA int32 [1] (every row) or [R] (one per row) -> c = col, or col mod ring when ring > 0; rows
      whose column falls outside [0, cols) write nothing.
      n_row: CUDA int32 [R], the row's n (-1: the row writes nothing); entries past it, or past V, hold id -1 / logprob -inf.
      finished: CUDA uint8 [R]; a finished row writes the filler (0, -1, -inf) if finished_fill, else nothing.
    A row's result depends only on its own logits, token and n (not on R, its index, the stride or where it is written).
    See aria_token_logprobs."""
    if not (logits.is_cuda and logits.dtype == bf16 and logits.dim() == 2 and logits.stride(-1) == 1):
        raise RuntimeError("token_logprobs: logits must be CUDA bf16 [R, V] with a contiguous last dim")
    if not isinstance(n_max, int) or isinstance(n_max, bool) or not 0 <= n_max <= MAX_LOGPROBS:
        raise ValueError(f"token_logprobs: n_max must be an int in [0, {MAX_LOGPROBS}], got {n_max!r}")
    R, V = logits.shape
    _chk(tokens, torch.int64, align=8)
    if tokens.shape != (R,):
        raise ValueError(f"token_logprobs: tokens must be [{R}], got {tuple(tokens.shape)}")
    if out is None:
        out = (torch.empty((R,), dtype=torch.float32, device=logits.device),
               torch.empty((R, n_max), dtype=torch.int32, device=logits.device),
               torch.empty((R, n_max), dtype=torch.float32, device=logits.device))
    lp, ids, tlp = out
    _chk(lp, torch.float32, align=4), _chk(ids, torch.int32, align=4), _chk(tlp, torch.float32, align=4)
    cols = 1 if lp.dim() == 1 else lp.shape[1]
    if lp.shape[0] != R or lp.dim() not in (1, 2) or ids.shape != lp.shape + (n_max,) or tlp.shape != ids.shape:
        raise ValueError(f"token_logprobs: out must be [{R}(, cols)], [{R}(, cols), {n_max}] x 2, got "
                         f"{[tuple(t.shape) for t in out]}")
    if col is not None:
        _chk(col, torch.int32, align=4)
        if col.numel() not in (1, R):
            raise ValueError(f"token_logprobs: col must have 1 or {R} entries, got {col.numel()}")
    elif ring:
        raise ValueError("token_logprobs: ring needs col")
    if not isinstance(ring, int) or not 0 <= ring <= cols:
        raise ValueError(f"token_logprobs: ring must be an int in [0, {cols}], got {ring!r}")
    for t, dt, name in ((n_row, torch.int32, "n_row"), (finished, torch.uint8, "finished")):
        if t is not None:
            _chk(t, dt, align=1)
            if t.shape != (R,):
                raise ValueError(f"token_logprobs: {name} must be [{R}], got {tuple(t.shape)}")
    with torch.cuda.device(logits.device):
        L.check(L.load().aria_token_logprobs(_p(logits), logits.stride(0), _p(tokens), R, V, n_max, _p(n_row), _p(col),
                                             int(col is not None and col.numel() == R and R > 1), int(ring), _p(finished),
                                             int(bool(finished_fill)), _p(lp), _p(ids), _p(tlp), cols, _stream(logits)),
                "token_logprobs")
    return lp, ids, tlp


def decode_advance_slots(next_ids: torch.Tensor, ids_in: torch.Tensor, out_tokens: torch.Tensor, n_out: torch.Tensor,
                         max_new: torch.Tensor, rope_pos: torch.Tensor, write_pos: torch.Tensor, kv_len: torch.Tensor,
                         rng_offset: torch.Tensor, finished: torch.Tensor, eos_token_ids: Sequence[int] = (),
                         pad_token_id: int = 0):
    """One launch after the sampler, R = next_ids.numel() rows: an unfinished row stores its token at out_tokens[r, n_out[r]]
    (int32 [R, L]) and feeds it back as ids_in[r], finishes on an EOS id (at most 8, baked into the launch) or at max_new[r]
    tokens (then ids_in[r] = pad_token_id), and moves n_out, its positions and its rng_offset (int64, read as uint64) on by one;
    a finished row changes nothing.  See aria_decode_advance_slots."""
    R = next_ids.numel()
    for t, dt in ((next_ids, torch.int64), (ids_in, torch.int64), (out_tokens, torch.int32), (n_out, torch.int32),
                  (max_new, torch.int32), (rope_pos, torch.int32), (write_pos, torch.int32), (kv_len, torch.int32),
                  (rng_offset, torch.int64), (finished, torch.uint8)):
        _chk(t, dt, align=1)
    if out_tokens.dim() != 2 or out_tokens.shape[0] != R or any(
            t.numel() != R for t in (ids_in, n_out, max_new, rope_pos, write_pos, kv_len, rng_offset, finished)):
        raise ValueError(f"decode_advance_slots: every slot array must have {R} entries and out_tokens [{R}, L]")
    eos, n_eos = _eos_array(eos_token_ids)
    with torch.cuda.device(next_ids.device):
        L.check(L.load().aria_decode_advance_slots(_p(next_ids), _p(ids_in), _p(out_tokens), out_tokens.shape[1], _p(n_out),
                                                   _p(max_new), _p(rope_pos), _p(write_pos), _p(kv_len), _p(rng_offset),
                                                   _p(finished), C.cast(eos, C.c_void_p), n_eos, int(pad_token_id), R,
                                                   _stream(next_ids)), "decode_advance_slots")


# ------------------------------------------------------------------------------------------- stop strings
STOP_MAX_STRINGS, STOP_MAX_BYTES, STOP_MAX_TOKENS, STOP_MAX_IDS = 16, 512, 128, 8


def stop_check_slots(vocab_bytes: torch.Tensor, vocab_offsets: torch.Tensor, stop_bytes: torch.Tensor, stop_lens: torch.Tensor,
                     lookback: torch.Tensor, stop_ids: torch.Tensor, n_stop_ids: torch.Tensor, prompt_tail: torch.Tensor,
                     tail_len: torch.Tensor, out_tokens: torch.Tensor, n_out: torch.Tensor, finished: torch.Tensor,
                     ids_in: torch.Tensor, pad_token_id: int):
    """Hugging Face's StopStringCriteria on R rows, after decode_advance_slots: row r has its own stop set (stop_bytes uint8
    [R, 16, 512], stop_lens int32 [R, 16], lookback int32 [R], 0 = no strings; stopping.encode_stop_set) and its own stop ids
    (stop_ids int64 [R, 8], the first n_stop_ids[r]); its history is its prompt tail (int64 [R, 128], its last tail_len[r] ids
    right-aligned), then out_tokens[r, :n_out[r]] (int32).  The vocabulary table: uint8 bytes and int32 offsets [V + 1]
    (stopping.StopVocab).  A row that is not finished and stops gets finished[r] = 1 and ids_in[r] = pad_token_id.  See
    aria_stop_check_slots."""
    R = finished.numel()
    for t, dt in ((vocab_bytes, torch.uint8), (vocab_offsets, torch.int32), (stop_bytes, torch.uint8), (stop_lens, torch.int32),
                  (lookback, torch.int32), (stop_ids, torch.int64), (n_stop_ids, torch.int32), (prompt_tail, torch.int64),
                  (tail_len, torch.int32), (out_tokens, torch.int32), (n_out, torch.int32), (finished, torch.uint8),
                  (ids_in, torch.int64)):
        _chk(t, dt, align=1)
    if vocab_offsets.dim() != 1 or vocab_offsets.numel() < 2:
        raise ValueError(f"stop_check_slots: vocab_offsets must be [V + 1] with V >= 1, got {tuple(vocab_offsets.shape)}")
    if (stop_bytes.shape != (R, STOP_MAX_STRINGS, STOP_MAX_BYTES) or stop_lens.shape != (R, STOP_MAX_STRINGS)
            or lookback.shape != (R,) or stop_ids.shape != (R, STOP_MAX_IDS) or n_stop_ids.shape != (R,)
            or prompt_tail.shape != (R, STOP_MAX_TOKENS) or tail_len.shape != (R,) or out_tokens.dim() != 2
            or out_tokens.shape[0] != R or n_out.shape != (R,) or ids_in.numel() != R):
        raise ValueError(f"stop_check_slots: every slot array must have {R} rows")
    with torch.cuda.device(finished.device):
        L.check(L.load().aria_stop_check_slots(_p(vocab_bytes), _p(vocab_offsets), vocab_offsets.numel() - 1, _p(stop_bytes),
                                               _p(stop_lens), _p(lookback), _p(stop_ids), _p(n_stop_ids), _p(prompt_tail),
                                               _p(tail_len), _p(out_tokens), out_tokens.shape[1], _p(n_out), _p(finished),
                                               _p(ids_in), int(pad_token_id), R, _stream(finished)), "stop_check_slots")
