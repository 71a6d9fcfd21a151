"""Differentiable restatement of oracle/phi3_oracle.py's text decoder, for the Cambrian-Phi3 training tests.

The layer and the mask rule are the oracle's (`sliding_mask`: key slot j visible from query slot i iff 0 <= i - j < W,
plus the padding mask), with three differences that matter only for training tests:
  * a query row that sees no key (a right-padded query past the window) attends to nothing: its softmax runs on zeros
    and is then zeroed, so torch autograd gives it zero gradients instead of the NaN an all -inf softmax row gives,
    even under a zero upstream gradient (the oracle's forward zeroes that row with nan_to_num, which autograd cannot
    undo);
  * it runs on the device of its inputs (the fp32 oracle on the GPU for full-size layers);
  * in bf16 it is the reference's eager numerics (RMSNorm statistics in fp32, RoPE tables rounded to the input dtype),
    the eager-bf16 arm of tests/helpers.py's parity criterion.
In fp32 on live rows it equals the oracle's forward (tests/test_phi3_train_cpu.py checks it), and its gradients match
the reference's Phi3DecoderLayer in train mode (tests/golden/phi3_layer_grad.npz).
"""
from __future__ import annotations

import torch

from oracle.phi3_oracle import sliding_mask


def _rms(x, w, eps):
    xf = x.float()
    return w * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)).to(x.dtype)


def _rope(x, pos, theta):
    hd = x.shape[-1]
    inv = 1.0 / (theta ** (torch.arange(0, hd, 2, dtype=torch.int64, device=x.device).float() / hd))
    emb = torch.cat([pos.float()[..., None] * inv] * 2, -1)
    cos, sin = emb.cos()[:, :, None].to(x.dtype), emb.sin()[:, :, None].to(x.dtype)
    x1, x2 = x[..., : hd // 2], x[..., hd // 2:]
    return x * cos + torch.cat([-x2, x1], -1) * sin


def layer(sd, pre, cfg, x, pos, kmask):
    """One Phi3DecoderLayer on x [B, S, H] (dropouts 0), differentiable, fully masked rows included."""
    B, S, H = x.shape
    nh, nkv = cfg["num_attention_heads"], cfg["num_key_value_heads"]
    hd = H // nh
    h = _rms(x, sd[pre + "input_layernorm.weight"], cfg["rms_norm_eps"])
    qkv = h @ sd[pre + "self_attn.qkv_proj.weight"].T
    q = qkv[..., : nh * hd].view(B, S, nh, hd)
    k = qkv[..., nh * hd:(nh + nkv) * hd].view(B, S, nkv, hd)
    v = qkv[..., (nh + nkv) * hd:].view(B, S, nkv, hd)
    q, k = _rope(q, pos, cfg["rope_theta"]), _rope(k, pos, cfg["rope_theta"])
    q, k, v = (t.transpose(1, 2) for t in (q, k, v))
    k = k.repeat_interleave(nh // nkv, 1)
    v = v.repeat_interleave(nh // nkv, 1)
    s = q @ k.transpose(-1, -2) / hd ** 0.5
    km = None if kmask is None else kmask.cpu()
    allow = sliding_mask(S, S, cfg["sliding_window"], km)[:, None].to(x.device)
    live = allow.any(-1, keepdim=True)
    p = torch.softmax(s.masked_fill(~allow, float("-inf")).masked_fill(~live, 0.0), -1).masked_fill(~live, 0.0)
    a = (p @ v).transpose(1, 2).reshape(B, S, nh * hd)
    x = x + a @ sd[pre + "self_attn.o_proj.weight"].T
    h = _rms(x, sd[pre + "post_attention_layernorm.weight"], cfg["rms_norm_eps"])
    gate, up = (h @ sd[pre + "mlp.gate_up_proj.weight"].T).chunk(2, -1)
    return x + (torch.nn.functional.silu(gate) * up) @ sd[pre + "mlp.down_proj.weight"].T


def logits(sd, cfg, ids, pos=None, kmask=None):
    """Logits [B, S, V] of the text decoder, in the dtype of `sd`, on the device of `ids`."""
    B, S = ids.shape
    if pos is None:
        pos = torch.arange(S, device=ids.device)[None].expand(B, S)
    x = sd["model.embed_tokens.weight"][ids]
    for li in range(cfg["num_hidden_layers"]):
        x = layer(sd, f"model.layers.{li}.", cfg, x, pos, kmask)
    x = _rms(x, sd["model.norm.weight"], cfg["rms_norm_eps"])
    return x @ sd["lm_head.weight"].T


def sketch(g, seed=0, rank=8):
    """Two-sided random sketch of a gradient matrix [N, K]: (g @ R [K, rank], L [rank, N] @ g) with seeded Gaussian R, L.
    An error in g survives in a random projection with probability 1, so the sketches stand in for the full matrix
    in the gradient fixture at a fraction of its size.  Vectors are returned as they are."""
    if g.dim() == 1:
        return (g,)
    gen = torch.Generator().manual_seed(seed)
    R = torch.randn(g.shape[1], rank, generator=gen, dtype=torch.float64)
    L = torch.randn(rank, g.shape[0], generator=gen, dtype=torch.float64)
    g = g.detach().double().cpu()
    return g @ R, L @ g
