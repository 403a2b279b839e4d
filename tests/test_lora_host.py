"""CPU: host-side contract of the LoRA mirror (aria/lora/layers.py:30-152) — parameter names/shapes as peft saves them,
argument validation, and that there is no CPU fallback."""
import pytest
import torch

from aria_b200 import lora, moe_lm


def test_lora_layer_state_dict_layout_and_init():
    base = moe_lm.GroupedGEMM(64, 96, 4)
    layer = lora.GroupedGemmLoraLayer(base, "default", r=8, lora_alpha=32)
    sd = layer.state_dict()
    assert set(sd) == {"base_layer.weight", "lora_A.default.weight", "lora_B.default.weight"}
    assert sd["lora_A.default.weight"].shape == (4, 64, 8)       # GroupedGEMM(in, r, groups).weight  (layers.py:87-89)
    assert sd["lora_B.default.weight"].shape == (4, 8, 96)       # GroupedGEMM(r, out, groups).weight (layers.py:90-92)
    assert layer.scaling["default"] == 4.0                        # lora_alpha / r (layers.py:93)
    assert float(sd["lora_B.default.weight"].float().abs().max()) == 0.0
    assert float(sd["lora_A.default.weight"].float().abs().max()) > 0.0
    trainable = {n for n, p in layer.named_parameters() if p.requires_grad}
    assert trainable == {"lora_A.default.weight", "lora_B.default.weight"}


def test_lora_layer_rejects_bad_arguments():
    base = moe_lm.GroupedGEMM(64, 96, 4)
    with pytest.raises(ValueError):   # same message as the reference (layers.py:74-77)
        lora.GroupedGemmLoraLayer(base, r=0)
    with pytest.raises(ValueError):
        lora.GroupedGemmLoraLayer(base, r=12)
    with pytest.raises(ValueError):
        lora.GroupedGemmLoraLayer(base, r=8, lora_dropout=0.1)


def test_lora_layer_has_no_cpu_path():
    base = moe_lm.GroupedGEMM(64, 96, 4)
    layer = lora.GroupedGemmLoraLayer(base, r=8)
    with pytest.raises(RuntimeError):
        layer(torch.zeros(16, 64, dtype=torch.bfloat16), torch.tensor([16, 0, 0, 0]))


def test_merge_and_unmerge_fold_the_adapter_into_the_base_weight():
    """layers.py:154-228: W += A @ B * scaling; unmerge restores W (fp32 here so the round trip is exact to rounding)."""
    base = moe_lm.GroupedGEMM(64, 96, 4)
    layer = lora.GroupedGemmLoraLayer(base, r=8, lora_alpha=32).float()
    with torch.no_grad():
        base.weight.normal_(0, 0.05)
        layer.lora_B["default"].weight.normal_(0, 0.05)
    w0 = base.weight.detach().clone()
    delta = torch.matmul(layer.lora_A["default"].weight, layer.lora_B["default"].weight) * 4.0
    layer.merge()
    assert layer.merged and torch.allclose(base.weight, w0 + delta, atol=1e-6)
    layer.merge()                                     # idempotent
    assert torch.allclose(base.weight, w0 + delta, atol=1e-6)
    layer.unmerge()
    assert not layer.merged and torch.allclose(base.weight, w0, atol=1e-6)


def test_target_module_selection_follows_the_reference_rule():
    """aria/lora/utils.py:29-64 (the reference pins it in tests/test_get_target_modules.py): substring match on qualified names,
    minus frozen towers and frozen LM layers."""
    names = ["vision_tower.vision_model.encoder.layers.0.mlp.fc1", "multi_modal_projector.ffn.linear_in",
             "language_model.model.layers.0.mlp.experts.fc1", "language_model.model.layers.0.mlp.experts.fc2",
             "language_model.model.layers.1.mlp.experts.fc1", "language_model.model.layers.1.self_attn.q_proj",
             "language_model.lm_head"]
    sel = lora.get_lora_target_modules(names, ["fc1", "fc2", "q_proj"], freeze_vit=True)
    assert sel == names[2:6]
    sel = lora.get_lora_target_modules(names, ["fc1"], freeze_llm_layers=[0])
    assert sel == [names[0], names[4]]
    assert lora.get_lora_target_modules(names, ["fc1"], freeze_vit=True, freeze_llm=True) == []
    assert lora.get_lora_target_modules(names, ["linear_in"], freeze_projector=True) == []


def test_inject_lora_wraps_only_grouped_gemms_and_keeps_checkpoint_names():
    cfg = moe_lm.AriaMoELMConfig(hidden_size=128, num_attention_heads=1, num_hidden_layers=2, vocab_size=32,
                                 moe_intermediate_size=32, moe_num_experts=4, moe_topk=2)
    model = torch.nn.Module()
    model.language_model = moe_lm.AriaMoELMForCausalLM(cfg)      # names as in AriaForConditionalGeneration
    names = [n for n, _ in model.named_modules()]
    targets = lora.get_lora_target_modules(names, ["experts.fc1", "experts.fc2", "q_proj"], freeze_llm_layers=[0])
    wrapped = lora.inject_lora(model, targets, r=8, lora_alpha=16)
    p1 = "language_model.model.layers.1.mlp.experts."
    assert wrapped == [p1 + "fc1", p1 + "fc2"]                                     # q_proj is not a GroupedGEMM
    sd = model.state_dict()
    assert p1 + "fc1.base_layer.weight" in sd                                      # peft's key layout for a wrapped module
    assert sd[p1 + "fc2.lora_B.default.weight"].shape == (4, 8, 128)
    assert "language_model.model.layers.0.mlp.experts.fc1.weight" in sd            # frozen layer untouched
    assert type(model.language_model.model.layers[0].mlp.experts.fc1) is moe_lm.GroupedGEMM


def _stand_in_ops(monkeypatch):
    """Replace the CUDA wrappers used by aria_b200.lora with plain torch (bf16 output rounding like the kernels), so the
    autograd LOGIC of the adapter path - padding, scaling fold, slicing, which gradient goes where - is checked on CPU."""
    from aria_b200 import ops

    def offs(off):
        return [int(v) for v in off]

    def from_counts(c):
        return torch.cat([torch.zeros(1, dtype=torch.int64), c.cumsum(0)]).to(torch.int32)

    def grouped_gemm(a, b, off, swiglu=False, group_mod=0, residual=None):
        o, out = offs(off), torch.zeros(a.shape[0], b.shape[2], dtype=a.dtype)
        for e in range(b.shape[0]):
            out[o[e]:o[e + 1]] = (a[o[e]:o[e + 1]].float() @ b[e].float()).to(a.dtype)
        return out if residual is None else (out.float() + residual.float()).to(a.dtype)

    def grouped_gemm_nt(a, b, off, group_mod=0, residual=None):
        o, out = offs(off), torch.zeros(a.shape[0], b.shape[1], dtype=a.dtype)
        for e in range(b.shape[0]):
            out[o[e]:o[e + 1]] = (a[o[e]:o[e + 1]].float() @ b[e].float().t()).to(a.dtype)
        return out if residual is None else (out.float() + residual.float()).to(a.dtype)

    def grouped_wgrad(a, b, off, num_sources=1):
        o = offs(off)
        return torch.stack([(a[o[e]:o[e + 1]].float().t() @ b[o[e]:o[e + 1]].float()).to(a.dtype) for e in range(len(o) - 1)])

    for name, fn in dict(grouped_gemm=grouped_gemm, grouped_gemm_nt=grouped_gemm_nt, grouped_wgrad=grouped_wgrad,
                         offsets_from_counts=from_counts).items():
        monkeypatch.setattr(ops, name, fn)
    monkeypatch.setattr(lora, "_as_offsets", lambda t, E, dev: t if t.numel() == E + 1 else from_counts(t.to(torch.int64)))


def test_lora_autograd_logic_reproduces_the_reference_golden(monkeypatch):
    """Same comparison as the GPU golden test, with CPU stand-ins for the kernels: separates the Python logic from the CUDA
    path (useful because that GPU test failed on hardware at the end of round 1 while this one passes)."""
    import os
    _stand_in_ops(monkeypatch)
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "lora_grouped_gemm_bf16.pt"), weights_only=False)
    E, K, N = g["w"].shape
    base = moe_lm.GroupedGEMM(K, N, E)
    base.weight.data.copy_(g["w"])
    layer = lora.GroupedGemmLoraLayer(base, "default", r=g["r"], lora_alpha=g["lora_alpha"])
    layer.lora_A["default"].weight.data.copy_(g["a"])
    layer.lora_B["default"].weight.data.copy_(g["b"])
    x = g["x"].clone().requires_grad_(True)
    with torch.enable_grad():
        out = layer(x, g["counts"])
        out.backward(g["dy"])

    def rel(a, b):
        return float((a.float() - b.float()).norm() / b.float().norm())

    assert rel(out.detach(), g["out"]) <= 1e-3
    assert rel(layer.lora_A["default"].weight.grad, g["d_a"]) <= 1e-3
    assert rel(layer.lora_B["default"].weight.grad, g["d_b"]) <= 1e-3
    assert rel(x.grad, g["dx"]) <= 1e-3
    with torch.no_grad():
        layer.merge()
        assert rel(layer(g["x"], g["counts"]), g["out"]) <= 1e-2
