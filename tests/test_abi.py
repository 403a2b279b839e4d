"""CPU: the C-ABI shared library loads and exports every symbol include/aria_b200.h declares; the ctypes
mirror of the descriptor struct matches the header field for field.  No compute calls (no GPU here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "aria_b200.h")


def _declared_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(aria_[a-z0-9_]+)\s*\(", src)))


@pytest.fixture(scope="module")
def lib():
    from aria_b200 import build, _lib
    build.build()  # nvcc cross-compiles sm_90a without a GPU
    return _lib.load()


def test_exports_every_declared_symbol(lib):
    from aria_b200 import _lib
    syms = _declared_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/aria_b200.h but not exported"
        assert s in _lib.SIGNATURES, f"{s} has no ctypes signature in aria_b200/_lib.py"


def test_abi_version_3_and_arch(lib):
    """Version 3: `aria_gemm_desc_t` without the descriptor debug fields, and 41 entries (no round-1 peer transport)."""
    assert lib.aria_abi_version() == 3
    assert lib.aria_build_arch() == b"sm_90a"


def test_gemm_desc_matches_header():
    from aria_b200 import _lib
    src = open(HEADER).read()
    body = src[src.index("typedef struct aria_gemm_desc {"):src.index("} aria_gemm_desc_t;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split("{", 1)[1].split(";"):
        decl = decl.strip()
        if not decl:
            continue
        decl = re.sub(r"^(const\s+)?(void|int64_t|int32_t)\s*\*?", "", decl).strip()
        for part in decl.split(","):
            names.append(re.sub(r"[\*\s]|\[\d+\]", "", part))
    assert names == [f[0] for f in _lib.GemmDesc._fields_]
    # 8-byte pointers / int64, natural alignment
    assert ctypes.sizeof(_lib.GemmDesc) % 8 == 0


def test_bad_arguments_are_errors_not_crashes(lib):
    """Argument validation happens before any CUDA call, so it is testable without a GPU."""
    from aria_b200 import _lib
    d = _lib.GemmDesc()
    assert lib.aria_gemm(ctypes.byref(d), None) == -1  # null pointers
    assert lib.aria_route_from_logits(None, None, None, None, 4, 8, 2, None) == -1
    assert lib.aria_permute_rows(None, None, None, 4, 256, None) == -1
    assert lib.aria_attention_decode_workspace_bytes(32, 20, 2048) == 32 * 20 * 8 * 130 * 4
    # training-mode router losses: null pointers and more experts than one warp pass covers (E <= 256) are rejected
    assert lib.aria_router_aux_bwd(None, None, None, 4, 8, 2, 0.1, 0.1, 1.0, None) == -1
    fake = ctypes.c_void_p(0x1000)   # never dereferenced: validation fails first
    assert lib.aria_router_aux_bwd(fake, fake, fake, 4, 300, 2, 0.1, 0.1, 1.0, None) == -1
    assert lib.aria_router_aux_loss(fake, fake, fake, 4, 8, 2, 0.1, 0.1, fake, 0, None) == -1   # workspace too small
    assert lib.aria_router_aux_workspace_bytes(64) % (65 * 4) == 0
    # whole-block entry: workspace query, null pointers, too many experts, workspace too small — all before any CUDA call
    nb = lib.aria_moe_block_fwd_workspace_bytes(768, 2560, 64, 6, 1664, 3328)
    assert nb >= 2 * (768 * 6 * (2560 * 2 + 1664) + 768 * (3328 + 2560)) and nb % 256 == 0
    assert lib.aria_moe_block_fwd_workspace_bytes(0, 2560, 64, 6, 1664, 3328) == -1
    assert lib.aria_moe_block_fwd(None, None, None, None, None, None, None, None, 768, 2560, 64, 6, 1664, 3328, None, None, 0, None, None) == -1
    assert lib.aria_moe_block_fwd(fake, fake, fake, fake, fake, fake, fake, fake, 768, 2560, 128, 6, 1664, 3328, None, fake, nb, None, None) == -1
    assert lib.aria_moe_block_fwd(fake, fake, fake, fake, fake, fake, fake, fake, 768, 2560, 64, 6, 1664, 3328, None, fake, nb - 1, None, None) == -1
    assert lib.aria_moe_block_fwd(fake, fake, fake, fake, None, None, None, fake, 768, 2560, 64, 6, 1664, 3328, None, fake, nb, None, None) == -1
    # GEMM descriptor validation: n must be a multiple of 8 (16-byte rows)
    d.a = d.b[0] = d.out[0] = 0x1000
    d.m, d.n, d.k, d.lda, d.n_seg, d.num_groups = 16, 12, 64, 64, 1, 1
    assert lib.aria_gemm(ctypes.byref(d), None) == -1


def test_no_cpu_fallback():
    """ops refuse CPU tensors loudly."""
    import torch
    from aria_b200 import ops
    with pytest.raises(RuntimeError):
        ops.linear(torch.zeros(4, 64, dtype=torch.bfloat16), torch.zeros(8, 64, dtype=torch.bfloat16))


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "aria_b200")
    for f in os.listdir(pkg):
        if f.endswith(".py"):
            src = open(os.path.join(pkg, f)).read()
            assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f
            assert "import_module(\"oracle" not in src and "__import__(\"oracle" not in src, f


def test_state_dict_keys_match_hf_layout():
    import torch
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as C
    m = AriaForConditionalGeneration(AriaConfig.from_dict(C.TINY), device="cpu")
    sd = C.aria_state(C.TINY, seed=0, dtype=torch.bfloat16)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    # reference GroupedGEMM layout: [E, in, out] (moe_lm.py:465)
    w = m.language_model.model.layers[0].mlp.experts.fc1.weight
    assert tuple(w.shape) == (8, 256, 1024)


def test_offsets_contract():
    import torch
    from aria_b200 import moe_lm
    with pytest.raises(RuntimeError):
        moe_lm._as_offsets(torch.zeros(5, dtype=torch.int64), 8, "cpu")  # neither E nor E+1 entries
    with pytest.raises(RuntimeError):
        moe_lm._as_offsets(torch.zeros(9, dtype=torch.int64), 8, "cpu")  # offsets must be int32 CUDA


def test_bench_gpu_leg_does_not_touch_oracle():
    """Only bench.py's cpu_baseline / --impl reference leg may execute oracle/ code."""
    import ast
    src = open(os.path.join(ROOT, "bench.py")).read()
    tree = ast.parse(src)
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "run_aria")
    body = ast.get_source_segment(src, fn)
    imports = re.findall(r"^\s*(?:from|import)\s+(\S+)", body, flags=re.M)
    assert not [m for m in imports if m.startswith("oracle")], imports
    assert "make_cpu_reference" in body  # the one allowed use: the cpu_baseline leg at N=1
    # ... and the GPU workload classes (what run_aria times) never import oracle/ either
    for cls in (n for n in tree.body if isinstance(n, ast.ClassDef) and n.name.startswith("Cfg")):
        seg = ast.get_source_segment(src, cls)
        assert not [m for m in re.findall(r"^\s*(?:from|import)\s+(\S+)", seg, flags=re.M) if m.startswith("oracle")], cls.name


def test_top_level_model_helpers_match_the_reference_api():
    """modeling_aria.py:145-192 / moe_lm.py:663-679: freeze_*, embedding accessors, MoE loss-coefficient setters."""
    from aria_b200 import configs as C
    from aria_b200.modeling_aria import AriaConfig, AriaForConditionalGeneration
    from oracle import configs as OC
    model = AriaForConditionalGeneration(AriaConfig.from_dict(OC.TINY))
    for p in model.parameters():
        p.requires_grad = True
    model.freeze_vit()
    model.freeze_projector()
    assert not any(p.requires_grad for p in model.vision_tower.parameters())
    assert not any(p.requires_grad for p in model.multi_modal_projector.parameters())
    assert all(p.requires_grad for p in model.language_model.parameters())
    model.freeze_llm()
    assert not any(p.requires_grad for p in model.parameters())
    assert model.get_input_embeddings() is model.language_model.model.embed_tokens
    assert model.get_output_embeddings() is model.language_model.lm_head
    model.set_moe_z_loss_coeff(0.25)
    model.set_moe_aux_loss_coeff(0.5)
    router_cfg = model.language_model.model.layers[0].mlp.router.config
    assert router_cfg.moe_z_loss_coeff == 0.25 and router_cfg.moe_aux_loss_coeff == 0.5
    assert C.ARIA_25B["text_config"]["moe_num_experts"] == 64
