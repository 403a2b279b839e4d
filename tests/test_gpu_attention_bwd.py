"""GPU: the causal LM attention backward (aria_attention_fwd_lse + aria_attention_bwd) and the differentiable HF attention seam.

Kernel parity is against fp32 autograd of eager attention on the same bf16 inputs; the bar per gradient is the project's
backward bar (rel-L2 <= 2e-2) and no worse than twice (+1e-3) what torch's own bf16 eager attention backward reaches against
the same fp32 reference."""
import pytest
import torch

from hf_common import tiny_hf_aria, tiny_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda"
SCALE = 128 ** -0.5


@pytest.fixture(autouse=True)
def _grad_enabled():
    with torch.enable_grad():      # other modules of the suite may have switched autograd off globally
        yield


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30))


def _inputs(B, H, Tq, Tk, seed, key_mask_p=0.0):
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(B, H, T, 128, generator=g).bfloat16().to(DEV) for T in (Tq, Tk, Tk))
    dout = torch.randn(B, Tq, H * 128, generator=g).bfloat16().to(DEV)
    km = None
    if key_mask_p:
        km = (torch.rand(B, Tk, generator=g) < key_mask_p).to(torch.uint8)
        km[:, -1] = 0                                              # every query sees at least one key
        km = km.to(DEV)
    return q, k, v, dout, km


def _dead(B, Tq, Tk, causal, km):
    dead = torch.zeros(B, 1, Tq, Tk, dtype=torch.bool, device=DEV)
    if causal:
        dead = dead | (torch.arange(Tk, device=DEV)[None, :] > torch.arange(Tk - Tq, Tk, device=DEV)[:, None])
    if km is not None:
        dead = dead | km.bool()[:, None, None, :]
    return dead


def _eager_grads(q, k, v, dout, causal, km, dtype):
    """Eager attention + autograd in `dtype` (softmax in fp32, as transformers' eager attention) -> (dq, dk, dv)."""
    B, H, Tq, _ = q.shape
    Tk = k.shape[2]
    qd, kd, vd = (t.detach().to(dtype).requires_grad_(True) for t in (q, k, v))
    w = torch.matmul(qd, kd.transpose(2, 3)) * SCALE
    w = w.masked_fill(_dead(B, Tq, Tk, causal, km), float("-inf"))
    p = torch.softmax(w, dim=-1, dtype=torch.float32).to(dtype)
    o = torch.matmul(p, vd).transpose(1, 2).reshape(B, Tq, H * 128)
    o.backward(dout.to(dtype))
    return qd.grad, kd.grad, vd.grad


@pytest.mark.parametrize("B,H,Tq,Tk,causal,key_mask_p", [
    (1, 2, 128, 128, True, 0.0),
    (2, 3, 300, 300, True, 0.0),         # ragged query and key tails
    (1, 2, 100, 420, True, 0.0),         # causal suffix: queries are the last 100 of 420 positions
    (2, 2, 333, 333, False, 0.3),        # non-causal with a random key mask
    (1, 4, 1030, 1030, True, 0.0),
    (2, 20, 2048, 2048, True, 0.0),      # the LM's 20 heads at the LoRA recipe's sequence length
    (1, 2, 8192, 8192, True, 0.0),
])
def test_bwd_parity_with_eager(B, H, Tq, Tk, causal, key_mask_p):
    from aria_b200 import ops
    q, k, v, dout, km = _inputs(B, H, Tq, Tk, seed=Tq + Tk, key_mask_p=key_mask_p)
    out, lse = ops.attention(q, k, v, Tq, Tk, SCALE, causal, key_mask=km, return_lse=True)
    got = ops.attention_bwd(q, k, v, out, dout, lse, Tq, Tk, SCALE, causal, key_mask=km)
    torch.cuda.synchronize()
    ref32 = _eager_grads(q, k, v, dout, causal, km, torch.float32)
    ref16 = _eager_grads(q, k, v, dout, causal, km, torch.bfloat16)
    for name, g, r32, r16 in zip(("dq", "dk", "dv"), got, ref32, ref16):
        assert g.shape == r32.shape
        e, e16 = _rel(g, r32), _rel(r16, r32)
        print(f"{name} ({B},{H},{Tq},{Tk}) rel-L2 {e:.3e}  torch bf16 eager {e16:.3e}")
        assert e <= 2e-2, (name, e)
        assert e <= 2 * e16 + 1e-3, (name, e, e16)


@pytest.mark.parametrize("causal", [True, False])
def test_lse_and_forward_identity(causal):
    from aria_b200 import ops
    B, H, Tq, Tk = 2, 3, 300, 300 if causal else 420
    q, k, v, _, km = _inputs(B, H, Tq, Tk, seed=7, key_mask_p=0.2)
    out, lse = ops.attention(q, k, v, Tq, Tk, SCALE, causal, key_mask=km, return_lse=True)
    plain = ops.attention(q, k, v, Tq, Tk, SCALE, causal, key_mask=km)
    assert torch.equal(out, plain)                                  # bit-identical output
    w = (torch.matmul(q.float(), k.float().transpose(2, 3)) * SCALE).masked_fill(_dead(B, Tq, Tk, causal, km), float("-inf"))
    want = torch.logsumexp(w, dim=-1)
    assert float((lse - want).abs().max()) <= 1e-3


def test_left_padded_rows_and_keys():
    from aria_b200 import ops
    B, H, T = 2, 2, 256
    q, k, v, dout, _ = _inputs(B, H, T, T, seed=11)
    km = torch.zeros(B, T, dtype=torch.uint8, device=DEV)
    km[1, :37] = 1                                                   # first 37 keys of the second sequence are padding
    out, lse = ops.attention(q, k, v, T, T, SCALE, True, key_mask=km, return_lse=True)
    dq, dk, dv = ops.attention_bwd(q, k, v, out, dout, lse, T, T, SCALE, True, key_mask=km)
    for t in (out, lse[0], dq, dk, dv):
        assert torch.isfinite(t.float()).all()
    assert torch.isinf(lse[1, :, :37]).all() and (lse[1, :, :37] < 0).all()
    assert not dq[1, :, :37].any()                                   # queries that see no key
    assert not dk[1, :, :37].any() and not dv[1, :, :37].any()       # masked keys
    ref = _eager_grads(q[:1], k[:1], v[:1], dout[:1], True, None, torch.float32)
    for g, r in zip((dq, dk, dv), ref):
        assert _rel(g[:1], r) <= 2e-2


def test_dk_dv_bit_reproducible():
    from aria_b200 import ops
    B, H, T = 2, 4, 1030
    q, k, v, dout, _ = _inputs(B, H, T, T, seed=5)
    out, lse = ops.attention(q, k, v, T, T, SCALE, True, return_lse=True)
    a = ops.attention_bwd(q, k, v, out, dout, lse, T, T, SCALE, True)
    b = ops.attention_bwd(q, k, v, out, dout, lse, T, T, SCALE, True)
    assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    assert _rel(a[0], b[0]) <= 1e-5                                  # dq: fp32 atomics, order-dependent last bits


# ------------------------------------------------------------------------------------------------ end to end through the seam
def _param_grads(model):
    return {n: p.grad.detach().float().clone() for n, p in model.named_parameters() if p.grad is not None}


def _check_grads(got, want, what):
    assert got.keys() == want.keys() and got, what
    worst = max(((_rel(got[n], want[n]), n) for n in want), key=lambda x: x[0])
    print(f"{what}: worst parameter-gradient rel-L2 {worst[0]:.3e} ({worst[1]})")
    assert worst[0] <= 2e-2, (what, worst)


def _tiny_llama():
    from transformers import LlamaConfig, LlamaForCausalLM
    cfg = LlamaConfig(vocab_size=512, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2,
                      num_key_value_heads=2, head_dim=128, max_position_embeddings=512, pad_token_id=0)
    torch.manual_seed(0)
    return LlamaForCausalLM(cfg)


def _llama_batch():
    g = torch.Generator().manual_seed(4)
    ids = torch.randint(3, 512, (2, 96), generator=g)
    am = torch.ones_like(ids)
    am[1, 70:] = 0                                                   # right-padded second sequence
    ids[1, 70:] = 0
    labels = ids.masked_fill(am == 0, -100)
    return ids.to(DEV), am.to(DEV), labels.to(DEV)


def test_llama_training_step_through_the_seam():
    from aria_b200 import hf_attention
    ids, am, labels = _llama_batch()
    ref = _tiny_llama().to(DEV).float().train()
    ref.config._attn_implementation = "eager"
    ref(input_ids=ids, attention_mask=am, labels=labels).loss.backward()
    want = _param_grads(ref)

    for ckpt in (False, True):
        model = _tiny_llama().to(DEV).bfloat16().train()
        model.config._attn_implementation = hf_attention.register()
        if ckpt:
            model.gradient_checkpointing_enable(gradient_checkpointing_kwargs={"use_reentrant": False})
        model(input_ids=ids, attention_mask=am, labels=labels).loss.backward()
        _check_grads(_param_grads(model), want, f"llama, gradient checkpointing {ckpt}")


def test_hf_aria_lm_training_step_through_the_seam():
    """transformers' own Aria (tiny), vision tower and projector frozen as in the reference LoRA recipe, top-k = all experts so
    that no routing boundary can flip under bf16 noise; the LM attention runs on our kernels through the seam."""
    from aria_b200 import hf_attention
    ids, pv, pm = tiny_inputs(batch=2)
    am = torch.ones_like(ids)
    am[1, -4:] = 0
    labels = ids.masked_fill(am == 0, -100).masked_fill(ids == 9, -100)

    def run(dtype, impl):
        model = tiny_hf_aria(device=DEV, dtype=dtype)
        for m in model.modules():
            c = getattr(m, "config", None)
            if c is not None and hasattr(c, "moe_topk"):
                c.moe_topk = c.moe_num_experts
        for n, p in model.named_parameters():
            p.requires_grad_(not ("vision_tower" in n or "multi_modal_projector" in n))
        model.train()
        model.config.text_config._attn_implementation = impl
        model.model.language_model.config._attn_implementation = impl
        out = model(input_ids=ids.to(DEV), pixel_values=pv.to(DEV, dtype), pixel_mask=pm.to(DEV), attention_mask=am.to(DEV),
                    labels=labels.to(DEV))
        out.loss.backward()
        return _param_grads(model)

    want = run(torch.float32, "eager")
    got = run(torch.bfloat16, hf_attention.register())
    _check_grads(got, want, "hf aria")
