"""CPU: host logic of the trainable MoE seams — which path `install(..., trainable=True)` takes in each mode, its refusals, the
router-loss scale plumbing, the `needs_input_grad` skipping of the backward kernels and the MoE layer's launch sequence with and
without expert parallelism.  The kernels are replaced by shape-only
recorders (zeros of the right shape; every call logged), or by the oracle-backed stand-ins of tests/standin_ops.py for the
inference path; the arithmetic is covered on the GPU by tests/test_gpu_moe_train_seam.py."""
import os
import sys
import types

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import standin_ops  # noqa: E402

bf16 = torch.bfloat16


@pytest.fixture(autouse=True)
def _grad_on():
    """Other test modules switch autograd off at import (torch.set_grad_enabled(False)); these tests need it."""
    with torch.enable_grad():
        yield


class Recorder:
    """Shape-only stand-ins for the `ops` entries the MoE training path calls."""

    def __init__(self):
        self.calls = []
        self.seq = []             # the calls with the expert-grouping arguments, e.g. "grouped_gemm group_mod=4"
        self.loss_scales = []

    def _log(self, name, **kw):
        self.calls.append(name)
        self.seq.append(" ".join([name] + [f"{k}={v}" for k, v in kw.items()]))

    def router_topk(self, x, w, k):
        self._log("router_topk")
        T, E = x.shape[0], w.shape[0]
        idx = (torch.arange(T * k) % E).view(T, k).to(torch.int32)
        counts = torch.bincount(idx.flatten().long(), minlength=E).to(torch.int32)
        return torch.zeros(T, k, dtype=bf16), idx, counts, torch.zeros(T, E, dtype=bf16)

    def build_permutation(self, idx, counts, row_align=1):
        self._log("build_permutation")
        T, k = idx.shape
        E = counts.numel()
        return (torch.zeros(E + 1, dtype=torch.int32), torch.zeros(T * k, dtype=torch.int32),
                torch.zeros(T * k + E * (row_align - 1), dtype=torch.int32))

    def permute_rows(self, x, src):
        self._log("permute_rows")
        return torch.zeros(src.numel(), x.shape[1], dtype=bf16)

    def offsets_from_counts(self, counts):
        self._log("offsets_from_counts")
        return torch.zeros(counts.numel() + 1, dtype=torch.int32)

    def grouped_gemm(self, a, b, off, swiglu=False, group_mod=0, residual=None):
        self._log("grouped_gemm", group_mod=group_mod)
        return torch.zeros(a.shape[0], b.shape[2] // (2 if swiglu else 1), dtype=bf16)

    def grouped_gemm_nt(self, a, b, off, group_mod=0, residual=None):
        self._log("grouped_gemm_nt", group_mod=group_mod)
        return torch.zeros(a.shape[0], b.shape[1], dtype=bf16)

    def grouped_wgrad(self, a, b, off, num_sources=1):
        self._log("grouped_wgrad", num_sources=num_sources)
        return torch.zeros((off.numel() - 1) // num_sources, a.shape[1], b.shape[1], dtype=bf16)

    def swiglu_fwd(self, h1):
        self._log("swiglu_fwd")
        return torch.zeros(h1.shape[0], h1.shape[1] // 2, dtype=bf16)

    def swiglu_bwd(self, h1, dh):
        self._log("swiglu_bwd")
        return torch.zeros_like(h1)

    def linear_multi(self, x, ws):
        self._log("linear_multi")
        return torch.zeros(x.shape[0], ws[0].shape[0] * len(ws), dtype=bf16)

    def linear(self, x, w, bias=None, act=0, residual=None, out=None):
        self._log("linear")
        return torch.zeros(*x.shape[:-1], w.shape[0], dtype=bf16)

    def matmul_kn(self, a, w, residual=None):
        self._log("matmul_kn")
        return torch.zeros(a.shape[0], w.shape[1], dtype=bf16)

    def unpermute_combine(self, y, dest, scores, shared=None):
        self._log("unpermute_combine")
        return torch.zeros(scores.shape[0], y.shape[1], dtype=bf16)

    def combine_bwd(self, do, y, dest, scores):
        self._log("combine_bwd")
        return torch.zeros_like(y), torch.zeros(scores.shape, dtype=torch.float32)

    def router_bwd(self, ds, s, idx, E):
        self._log("router_bwd")
        return torch.zeros(s.shape[0], E, dtype=bf16)

    def router_aux_bwd(self, logits, counts, dlogits, k, z, aux, loss_scale=1.0):
        self._log("router_aux_bwd")
        self.loss_scales.append((z, aux, loss_scale))
        return dlogits


@pytest.fixture()
def rec(monkeypatch):
    from aria_b200 import ops
    r = Recorder()
    for n in [n for n in dir(Recorder) if not n.startswith("_")]:
        monkeypatch.setattr(ops, n, getattr(r, n))
    return r


def _block_args(T=20, d=64, E=4, I=32, Is=48):
    g = torch.Generator().manual_seed(0)
    mk = lambda *s: torch.randn(*s, generator=g).to(bf16)          # noqa: E731
    return [mk(1, T, d), mk(E, d), mk(E, d, 2 * I), mk(E, I, d), mk(Is, d), mk(Is, d), mk(d, Is)]


NAMES = ["x", "router", "fc1", "fc2", "gate", "up", "down"]


@pytest.mark.parametrize("trainable", [("fc1", "router"), ("x",), ("x", "fc2", "down"), ("gate",), tuple(NAMES)])
def test_moe_layer_function_skips_unneeded_gradients(rec, trainable):
    from aria_b200 import moe_train
    args = [t.requires_grad_(n in trainable) for n, t in zip(NAMES, _block_args())]
    out = moe_train.MoELayerFunction.apply(*args, 2, None)
    rec.calls.clear()
    out.sum().backward()
    got = {n for n, t in zip(NAMES, args) if t.grad is not None}
    assert got == set(trainable)
    assert rec.calls.count("grouped_wgrad") == len(set(trainable) - {"x"})
    assert ("grouped_gemm_nt" in rec.calls) == bool({"x", "fc1"} & set(trainable))
    assert ("router_bwd" in rec.calls) == bool({"x", "router"} & set(trainable))


def test_loss_scale_is_read_from_the_given_holder_at_backward_time(rec, monkeypatch):
    from aria_b200 import moe_train
    holder = types.SimpleNamespace(main_loss_backward_scale=torch.tensor(1.0))
    args = [t.requires_grad_(True) for t in _block_args()]
    out = moe_train.MoELayerFunction.apply(*args, 2, (0.25, 0.5), holder)
    holder.main_loss_backward_scale = torch.tensor(0.125)          # what train.py's set_loss_scale does before backward
    out.sum().backward()
    assert rec.loss_scales == [(0.25, 0.5, 0.125)]
    # the composed path's router stage reads it the same way
    rec.loss_scales.clear()
    logits = torch.zeros(20, 4, dtype=bf16, requires_grad=True)
    from aria_b200 import ops
    monkeypatch.setattr(ops, "route_from_logits", standin_ops.route_from_logits)
    scores, _, _ = moe_train.TopKFunction.apply(logits, 2, (0.25, 0.5), holder)
    holder.main_loss_backward_scale = 3.0
    scores.float().sum().backward()
    assert rec.loss_scales == [(0.25, 0.5, 3.0)]


_FWD = ["router_topk", "build_permutation", "permute_rows", "grouped_gemm group_mod=0", "swiglu_fwd", "grouped_gemm group_mod=0",
        "linear_multi", "swiglu_fwd", "linear", "unpermute_combine"]
_BWD = ["combine_bwd", "grouped_wgrad num_sources=1", "grouped_gemm_nt group_mod=0", "swiglu_bwd", "grouped_wgrad num_sources=1",
        "grouped_gemm_nt group_mod=0", "grouped_wgrad num_sources=1", "matmul_kn", "swiglu_bwd", "grouped_wgrad num_sources=1",
        "grouped_wgrad num_sources=1", "matmul_kn", "matmul_kn", "router_bwd", "grouped_wgrad num_sources=1", "matmul_kn",
        "unpermute_combine"]
# one rank over E=4 experts: the same launches with the exchange steps inserted and the expert GEMMs over (source, expert) groups
_EP_FWD = ["router_topk", "build_permutation", "permute_rows", "all_to_all_single", "all_to_all_single", "offsets_from_counts",
           "grouped_gemm group_mod=4", "swiglu_fwd", "grouped_gemm group_mod=4", "all_to_all_single", "linear_multi", "swiglu_fwd",
           "linear", "unpermute_combine"]
_EP_BWD = ["combine_bwd", "all_to_all_single", "grouped_wgrad num_sources=1", "grouped_gemm_nt group_mod=4", "swiglu_bwd",
           "grouped_wgrad num_sources=1", "grouped_gemm_nt group_mod=4", "all_to_all_single", "grouped_wgrad num_sources=1",
           "matmul_kn", "swiglu_bwd", "grouped_wgrad num_sources=1", "grouped_wgrad num_sources=1", "matmul_kn", "matmul_kn",
           "router_bwd", "grouped_wgrad num_sources=1", "matmul_kn", "unpermute_combine"]


def test_moe_layer_launch_sequence_with_and_without_expert_parallelism(rec, monkeypatch, tmp_path):
    """The full sequence of kernel calls of the MoE layer's forward and backward, single-device and through
    `ep_moe_layer_train` on a one-rank gloo group (the all-to-alls logged where they are issued)."""
    import torch.distributed as dist
    from aria_b200 import moe_train
    from aria_b200.expert_parallel import ep_moe_layer_train
    args = [t.requires_grad_(True) for t in _block_args()]
    out = moe_train.MoELayerFunction.apply(*args, 2)
    assert rec.seq == _FWD
    rec.seq.clear()
    out.sum().backward()
    assert rec.seq == _BWD
    real = dist.all_to_all_single

    def all_to_all_single(*a, **kw):
        rec._log("all_to_all_single")
        return real(*a, **kw)

    monkeypatch.setattr(dist, "all_to_all_single", all_to_all_single)
    dist.init_process_group("gloo", init_method=f"file://{tmp_path}/store", rank=0, world_size=1)
    try:
        args = [t.detach().requires_grad_(True) for t in _block_args()]
        w = dict(zip(["router.weight", "experts.fc1.weight", "experts.fc2.weight", "shared_experts.gate_proj.weight",
                      "shared_experts.up_proj.weight", "shared_experts.down_proj.weight"], args[1:]))
        rec.seq.clear()
        out = ep_moe_layer_train(args[0], w, 2)
        assert rec.seq == _EP_FWD
        rec.seq.clear()
        out.sum().backward()
        assert rec.seq == _EP_BWD
        assert all(t.grad is not None for t in args)
        # skipped gradients under a group: only the wgrads and the local kernels go; the exchanges and the routed
        # data-gradient chain between them are collective work every rank issues
        for t in args:
            t.requires_grad_(t is w["experts.fc2.weight"])
        out = ep_moe_layer_train(args[0], w, 2)
        rec.seq.clear()
        out.sum().backward()
        assert rec.seq == ["combine_bwd", "all_to_all_single", "grouped_wgrad num_sources=1", "grouped_gemm_nt group_mod=4",
                           "swiglu_bwd", "grouped_gemm_nt group_mod=4", "all_to_all_single"]
    finally:
        dist.destroy_process_group()


def test_differentiable_gmm_skips_unneeded_gradients(rec):
    from aria_b200 import moe_train
    a = torch.randn(30, 64).to(bf16).requires_grad_(True)
    w = torch.randn(3, 64, 64).to(bf16)
    off = torch.tensor([0, 7, 7, 30], dtype=torch.int32)
    moe_train.GroupedGemmFunction.apply(a, w, off).sum().backward()
    assert rec.calls == ["grouped_gemm", "grouped_gemm_nt"] and w.grad is None
    rec.calls.clear()
    a2, w2 = a.detach(), w.clone().requires_grad_(True)
    moe_train.GroupedGemmFunction.apply(a2, w2, off).sum().backward()
    assert rec.calls == ["grouped_gemm", "grouped_wgrad"] and w2.grad is not None
    rec.calls.clear()
    with torch.no_grad():
        moe_train.experts_gemm_train(a, w2, off)
    assert rec.calls == ["grouped_gemm"]


# ------------------------------------------------------------------------------------------------ the seam on a reference layer
def _ref_layer():
    from oracle import ref_loader
    if not ref_loader.reference_available():
        pytest.skip("reference files not available")
    ref = ref_loader.load_reference()
    cfg = ref.moe_lm.AriaMoELMConfig(hidden_size=64, num_attention_heads=2, moe_num_experts=4, moe_topk=2,
                                     moe_intermediate_size=32, moe_num_shared_experts=2, intermediate_size=32,
                                     moe_z_loss_coeff=0.3, moe_aux_loss_coeff=0.7)
    layer = ref.moe_lm.MoELayer(cfg)
    g = torch.Generator().manual_seed(1)
    for p_ in layer.parameters():
        p_.data = (torch.randn(p_.shape, generator=g) * 0.02).to(bf16)
    return ref, layer


def test_trainable_seam_paths_and_refusals(monkeypatch):
    from aria_b200 import install
    ref, layer = _ref_layer()
    standin_ops.patch(monkeypatch)
    monkeypatch.setattr(ref.moe_lm, "experts_gemm", ref.moe_lm.experts_gemm)    # restored after the test
    blocks = []
    monkeypatch.setattr(install, "_moe_block", lambda self, h: (blocks.append(1), h)[1])
    assert install.install(torch.nn.ModuleList([layer]), ref.moe_lm, trainable=True) == 1
    from aria_b200 import moe_train
    assert ref.moe_lm.experts_gemm is moe_train.experts_gemm_train
    x = torch.randn(1, 6, 64).to(bf16)
    # inference: no_grad (any mode), or nothing requires grad -> the fused block
    layer.eval()
    with torch.no_grad():
        layer(x)
    layer.train()
    with torch.no_grad():
        layer(x)
    for p_ in layer.parameters():
        p_.requires_grad_(False)
    layer(x)
    assert len(blocks) == 3
    # training: CPU tensors are refused with a message
    with pytest.raises(RuntimeError, match="needs CUDA tensors"):
        layer(x.clone().requires_grad_(True))
    for p_ in layer.parameters():
        p_.requires_grad_(True)
    with pytest.raises(RuntimeError, match="needs CUDA tensors"):
        layer(x)
    # expert parallelism keeps its own path
    layer.expert_parallel = object()
    with pytest.raises(NotImplementedError, match="expert-parallel"):
        with torch.no_grad():
            layer(x)
    del layer.expert_parallel
    # the default install keeps refusing autograd
    install.install(torch.nn.ModuleList([layer]), ref.moe_lm)
    assert ref.moe_lm.experts_gemm is not moe_train.experts_gemm_train
    with pytest.raises(RuntimeError, match="inference-only"):
        layer(x)


def test_router_losses_come_from_the_reference_module_in_train_mode():
    from aria_b200 import install
    ref, layer = _ref_layer()
    layer.train()
    coeffs, holder = install._router_losses(layer)
    assert coeffs == (0.3, 0.7) and holder is ref.moe_lm.MoEAuxLossAutoScaler
    layer.eval()
    assert install._router_losses(layer) == (None, None)
    import hf_common as H
    hf = H.tiny_hf_aria(layers=1)
    moe = next(m for m in hf.modules() if type(m).__name__ == "AriaTextMoELayer")
    moe.train()
    assert install._router_losses(moe) == (None, None)
    assert install._moe_plain(moe) and install._moe_plain(layer)


def test_lora_wrapped_experts_are_recognised_and_checked():
    from oracle import ref_loader
    from aria_b200 import install
    ref, layer = _ref_layer()
    LL = ref_loader.load_reference_lora()
    layer.experts.fc1 = LL.GroupedGemmLoraLayer(layer.experts.fc1, "default", r=8, lora_alpha=16)
    assert not install._moe_plain(layer)
    w, a, b, s = install._lora_parts(layer.experts.fc1)
    assert w is layer.experts.fc1.base_layer.weight and a.shape == (4, 64, 8) and b.shape == (4, 8, 64) and s == 2.0
    assert install._lora_parts(layer.experts.fc2) is None
    layer.experts.fc1.lora_dropout["default"] = torch.nn.Dropout(0.1)
    with pytest.raises(NotImplementedError, match="lora_dropout"):
        install._moe_plain(layer)
    layer.experts.fc1.lora_dropout["default"] = torch.nn.Identity()
    layer.experts.fc1.update_layer("second", 8, 16, 0.0, True, False)
    layer.experts.fc1.set_adapter(["default", "second"])
    with pytest.raises(NotImplementedError, match="active LoRA adapters"):
        install._moe_plain(layer)
