"""TEST INFRASTRUCTURE — torch-CPU stand-ins for `aria_b200.ops` (same signatures, same layouts), built on the oracle.

`patch(monkeypatch)` swaps them in so that the HOST logic above the C ABI — the module mirrors, `install` / `install_vit` /
`hf_attention` seams, padding masks, position ids, chunked prefill, KV-cache bookkeeping — runs on a box without a GPU (the
`-m "not gpu"` suite).  The arithmetic here is the checker's, never the product's: nothing under aria_b200/ imports this file,
and the GPU suite runs the same scenarios on the real kernels (tests/test_gpu_parity_full.py, tests/test_gpu_dropin.py).
"""
import torch
import torch.nn.functional as F

from oracle import aria_oracle as O

ACT_NONE, ACT_GELU_TANH, ACT_GELU_NEW = 0, 1, 2


def _act(y, act):
    if act == ACT_GELU_TANH:
        return F.gelu(y, approximate="tanh")
    if act == ACT_GELU_NEW:
        return O.gelu_new(y)
    return y


def linear(x, weight, bias=None, act=ACT_NONE, residual=None, out=None):
    y = _act(F.linear(x, weight, bias), act)
    if residual is not None:
        y = y + residual.reshape(y.shape)
    return y


def linear_multi(x, weights):
    return torch.cat([F.linear(x.reshape(-1, x.shape[-1]), w) for w in weights], dim=1)


def linear_swiglu(x, gate_w, up_w):
    return F.silu(F.linear(x, gate_w)) * F.linear(x, up_w)


def _counts(offsets):
    return (offsets[1:] - offsets[:-1]).long()


def grouped_gemm(a, b, offsets, swiglu=False, group_mod=0, residual=None):
    assert not group_mod
    y = O.sequential_gemm(a, b, _counts(offsets))
    if swiglu:
        y = O.glu(y)
    return y if residual is None else y + residual


def router_topk(x, w_router, k):
    logits = O.router_gating(x, w_router)
    s, i, c = O.router_routing(logits, k)
    return s, i.to(torch.int32), c.to(torch.int32), logits


def route_from_logits(logits, k):
    s, i, c = O.router_routing(logits, k)
    return s, i.to(torch.int32), c.to(torch.int32)


def route_given_indices(logits, top_idx):
    top = torch.gather(logits, 1, top_idx.long())
    scores = torch.softmax(top, dim=-1, dtype=torch.float32).type_as(logits)
    return scores, torch.bincount(top_idx.flatten().long(), minlength=logits.shape[1]).to(torch.int32)


def build_permutation(top_idx, counts, row_align=1):
    assert row_align == 1
    k = top_idx.shape[1]
    order = torch.argsort(top_idx.flatten().long(), stable=True)
    dest = torch.empty_like(order)
    dest[order] = torch.arange(order.numel())
    offsets = torch.zeros(counts.numel() + 1, dtype=torch.int32)
    offsets[1:] = torch.cumsum(counts.long(), 0).to(torch.int32)
    return offsets, dest.to(torch.int32), (order // k).to(torch.int32)


def permute_rows(x, src_token):
    return x.index_select(0, src_token.long())


def unpermute_combine(y, dest_row, scores, shared=None):
    T, k = scores.shape
    rows = y[dest_row.long()].view(T, k, -1)
    out = (rows * scores.unsqueeze(-1)).sum(1).type_as(y)
    return out if shared is None else out + shared


def offsets_from_counts(counts):
    off = torch.zeros(counts.numel() + 1, dtype=torch.int32)
    off[1:] = torch.cumsum(counts.long(), 0).to(torch.int32)
    return off


def rmsnorm(x, weight, eps, residual=None):
    if residual is None:
        return O.rms_norm(x, weight, eps)
    s = x + residual
    return O.rms_norm(s, weight, eps), s


def layernorm(x, weight, bias, eps):
    return F.layer_norm(x, (x.shape[-1],), weight, bias, eps)


def rope_table(inv_freq, n_pos):
    freqs = torch.arange(n_pos).float()[:, None] * inv_freq[None, :]
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos().bfloat16(), emb.sin().bfloat16()


def embedding(ids, table):
    return F.embedding(ids, table)


def merge_image_features(ids, image_token, features, embeds, count_out=None):
    embeds[ids.reshape(-1) == image_token] = features.to(embeds.dtype)
    return embeds


def im2col_patches(pixels, patch, k_pad):
    B, C, S, _ = pixels.shape
    p = pixels.unfold(2, patch, patch).unfold(3, patch, patch)            # [B, C, n, n, P, P]
    p = p.permute(0, 2, 3, 1, 4, 5).reshape(B * (S // patch) ** 2, C * patch * patch)
    out = torch.zeros(p.shape[0], k_pad, dtype=pixels.dtype)
    out[:, : p.shape[1]] = p
    return out


def add_pos_embedding(x, pos_ids, table):
    return x + F.embedding(pos_ids, table)


def qkv_heads(x, weights, biases, outs, head_dim, rows_per_batch, pos0=0, rope_mask=0, rope_cos=None, rope_sin=None,
              position_ids=None):
    x2 = x.reshape(-1, x.shape[-1])
    T = rows_per_batch
    B = x2.shape[0] // T
    for s, (w, b, o) in enumerate(zip(weights, biases, outs)):
        y = F.linear(x2, w, b).view(B, T, -1, head_dim).transpose(1, 2)   # [B, H, T, hd]
        if (rope_mask >> s) & 1:
            pos = (torch.arange(T) + pos0)[None].expand(B, T) if position_ids is None else position_ids.view(B, T).long()
            cos, sin = rope_cos[pos].to(y.dtype).unsqueeze(1), rope_sin[pos].to(y.dtype).unsqueeze(1)
            y = (y * cos) + (O.rotate_half(y) * sin)
        o[:, :, pos0:pos0 + T, :head_dim] = y


def attention(q, k, v, Tq, Tk, scale, causal, out_hd=128, key_mask=None):
    B, H = q.shape[:2]
    q, k, v = q[:, :, :Tq], k[:, :, :Tk], v[:, :, :Tk]
    add = torch.zeros(B, 1, Tq, Tk, dtype=torch.float32)
    if causal:
        add = add + O.causal_additive_mask(Tq, Tk, torch.float32)
    if key_mask is not None:
        add = add.masked_fill(key_mask.bool()[:, None, None, :], float("-inf"))
    w = torch.matmul(q.float(), k.float().transpose(2, 3)) * scale + add
    w = torch.nan_to_num(F.softmax(w, dim=-1), nan=0.0).to(q.dtype)       # fully masked rows -> 0, like the kernel
    o = torch.matmul(w, v).transpose(1, 2)                                # [B, Tq, H, 128]
    return o[..., :out_hd].reshape(B, Tq, H * out_hd).contiguous()


def attention_decode(q, k, v, Tk, scale, key_mask=None):
    B, H = q.shape[:2]
    return attention(q.reshape(B, H, 1, 128), k, v, 1, Tk, scale, False, key_mask=key_mask).view(B, H * 128)


_NAMES = [n for n, f in list(globals().items()) if callable(f) and not n.startswith("_") and n not in ("patch",)
          and getattr(f, "__module__", None) == __name__]


def patch(monkeypatch):
    from aria_b200 import ops
    for n in _NAMES:
        monkeypatch.setattr(ops, n, globals()[n])
