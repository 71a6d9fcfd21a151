"""Torch reference of the FP8 decode KV cache (cambrian_b200/kv_fp8.py states the definition): the row quantiser (the
rule of tests/fp8_reference.py applied to every hd-element head row), its dequantiser, and decode attention in fp64 over
a dequantised cache.  CPU stand-ins of the two entry points for host-logic tests are built from these."""
import torch

import fp8_reference as R


def quantize_rows(x):
    """x [..., hd] -> (q float8_e4m3fn [..., hd], s fp32 [...]): one scale per head row."""
    q, s = R.quantize_rows(x.reshape(-1, x.shape[-1]))
    return q.view(x.shape), s.view(x.shape[:-1])


def dequantize(q, s, dtype=torch.float64):
    """float(q) * s, in `dtype` (fp64: exact)."""
    return q.to(dtype) * s.to(dtype)[..., None]


def decode_attention(q, kq, ks, vq, vs, length, kmask=None, scale=None, dtype=torch.float64):
    """q [B, nh, hd] -> o [B, nh, hd] in `dtype`: softmax((q . K~) * scale) V~ over the positions below `length` whose
    kmask is set, K~ / V~ the dequantised cache [B, S_max, nkv, hd].  fp64 is the reference; bf16 mimics eager bf16
    (bf16 matmuls, fp32 softmax rounded to bf16), the yardstick of the parity criterion."""
    B, nh, hd = q.shape
    G = nh // kq.shape[2]
    scale = hd ** -0.5 if scale is None else scale
    k = dequantize(kq[:, :length], ks[:, :length], dtype).repeat_interleave(G, 2)      # [B, L, nh, hd]
    v = dequantize(vq[:, :length], vs[:, :length], dtype).repeat_interleave(G, 2)
    s = torch.einsum("bhd,bthd->bht", q.to(dtype), k) * scale
    if kmask is not None:
        s = s.masked_fill(~kmask[:, None, :length].bool(), float("-inf"))
    p = torch.softmax(s.to(torch.float64 if dtype == torch.float64 else torch.float32), -1).to(dtype)
    return torch.einsum("bht,bthd->bhd", p, v)


# ---- CPU stand-ins of ops.kv_fp8_append / ops.attn_decode_fp8 (host-logic tests on machines without a GPU) ----
def kv_fp8_append(k, v, kq, vq, ks, vs, offset=0, offset_dev=None):
    o = int(offset) + (int(offset_dev.reshape(-1)[0]) if offset_dev is not None else 0)
    S = k.shape[1]
    for src, dq, ds in ((k, kq, ks), (v, vq, vs)):
        q, s = quantize_rows(src.float())
        dq[:, o:o + S] = q
        ds[:, o:o + S] = s


def attn_decode_fp8(q, kq, vq, ks, vs, workspace, *, length, length_dev=None, kmask=None, scale=None):
    L = int(length) + (int(length_dev.reshape(-1)[0]) if length_dev is not None else 0)
    o = decode_attention(q[:, 0], kq, ks, vq, vs, L, kmask, scale)
    return o.to(torch.bfloat16)[:, None]


def attn_decode_fp8_workspace(B, nh, nkv, S_max, hd, device):
    return torch.empty(1, dtype=torch.float32, device=device)


def install(monkeypatch):
    from cambrian_b200 import ops
    for n in ("kv_fp8_append", "attn_decode_fp8", "attn_decode_fp8_workspace"):
        monkeypatch.setattr(ops, n, globals()[n])


def oracle_layer_kv_fp8(S0):
    """O.llama_layer with the FP8 cache's attention: query rows at positions >= S0 (the decode steps) attend over K / V
    passed through the reference quantiser; the prompt's rows attend over the plain K / V, as the prefill does."""
    import math

    import torch.nn.functional as F_

    from oracle import cambrian_oracle as O

    def layer(sd, p, x, cos, sin, attn_mask_2d, cfg):
        B, S, H = x.shape
        nh, nkv = cfg["num_attention_heads"], cfg["num_key_value_heads"]
        hd = H // nh
        h = O.rms_norm(x, sd[p + "input_layernorm.weight"], cfg["rms_norm_eps"])
        q = O.F.linear(h, sd[p + "self_attn.q_proj.weight"]).view(B, S, nh, hd).transpose(1, 2)
        k = O.F.linear(h, sd[p + "self_attn.k_proj.weight"]).view(B, S, nkv, hd).transpose(1, 2)
        v = O.F.linear(h, sd[p + "self_attn.v_proj.weight"]).view(B, S, nkv, hd).transpose(1, 2)
        q, k = O.apply_rope(q, cos, sin), O.apply_rope(k, cos, sin)
        kd, vd = (dequantize(*quantize_rows(t), dtype=t.dtype) for t in (k, v))
        allow = torch.ones(S, S, dtype=torch.bool, device=x.device).tril()[None, None]
        if attn_mask_2d is not None:
            allow = allow & attn_mask_2d.bool().to(x.device)[:, None, None, :]
        outs = []
        for kk, vv in ((k, v), (kd, vd)):
            kk, vv = kk.repeat_interleave(nh // nkv, 1), vv.repeat_interleave(nh // nkv, 1)
            s = ((q @ kk.transpose(-1, -2)) / math.sqrt(hd)).masked_fill(~allow, torch.finfo(q.dtype).min)
            outs.append(torch.softmax(s.float(), -1).to(q.dtype) @ vv)
        a = torch.cat([outs[0][:, :, :S0], outs[1][:, :, S0:]], 2).transpose(1, 2).reshape(B, S, H)
        x = x + O.F.linear(a, sd[p + "self_attn.o_proj.weight"])
        h = O.rms_norm(x, sd[p + "post_attention_layernorm.weight"], cfg["rms_norm_eps"])
        g = F_.silu(O.F.linear(h, sd[p + "mlp.gate_proj.weight"])) * O.F.linear(h, sd[p + "mlp.up_proj.weight"])
        return x + O.F.linear(g, sd[p + "mlp.down_proj.weight"])

    return layer
