"""TEST INFRASTRUCTURE ONLY — plain-torch stand-ins for a subset of `cambrian_b200.ops`, installed by monkeypatching inside
a CPU test process (tests/test_autograd_blocks_cpu.py) so that the HOST logic of the autograd blocks — argument order,
saved tensors, gradient routing, main_grad accumulation, layout conventions — runs in the `-m "not gpu"` suite.

This is NOT a fallback: nothing under `cambrian_b200/` imports this file, the product still raises without the CUDA
library / CUDA tensors (tests/test_abi_cpu.py), and the numerical parity claims rest on the `-m gpu` tests alone.  Each
stand-in computes in fp32 and rounds once to bf16, like the kernels it mirrors (include/cambrian_b200.h documents each).
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

_ACT = {"gelu": F.gelu, "quick_gelu": lambda x: x * torch.sigmoid(1.702 * x), "silu": F.silu,
        "gelu_tanh": lambda x: F.gelu(x, approximate="tanh")}


def gemm(a, b, *, a_mn=False, b_mn=False, bias=None, colscale=None, residual=None, out=None, out_dtype=torch.bfloat16,
         accumulate=False, alpha=1.0, act=None, force_bn=0):
    A = a.float().transpose(-1, -2) if a_mn else a.float()
    B = b.float() if b_mn else b.float().transpose(-1, -2)
    y = (A @ B) * alpha
    if bias is not None:
        y = y + bias.float()
    if act not in (None, "none"):
        y = _ACT[act](y)
    if colscale is not None:
        y = y * colscale.float()
    if residual is not None:
        assert residual.shape == y.shape, (residual.shape, y.shape)
        y = y + residual.float()
    if out is not None:
        assert out.shape == y.shape, (out.shape, y.shape)
        if accumulate:
            y = y + out.float()
        out.copy_(y.to(out.dtype))
        return out
    assert not accumulate, "accumulate=True needs an explicit `out`"
    return y.to(out_dtype)


def linear(x, weight, bias=None, **kw):
    lead = x.shape[:-1]
    res = kw.pop("residual", None)
    if res is not None:
        res = res.reshape(-1, weight.shape[0])
    return gemm(x.reshape(-1, x.shape[-1]), weight, bias=bias, residual=res, **kw).view(*lead, weight.shape[0])


def f32_to_bf16(src, dst, scale=1.0, cols=None, out_ld=None):
    dst.copy_((src.float() * scale).reshape(dst.shape).to(dst.dtype))
    return dst


def _norm_input(x, pos, side, r):
    """x [rows, C] in fp32, plus the pos_embed row of each latent's window position rounded to bf16 (the kernels fuse the
    bf16 add `latents + pos_embed` into the load): natural layout (row = (b, y, x) of a side x side grid) -> window
    position (y % r) * r + (x % r); window-rearranged layout (side == 0) -> row % r^2."""
    if pos is None:
        return x.float()
    idx = torch.arange(x.shape[0])
    if side == 0:
        w = idx % (r * r)
    else:
        w = ((idx // side) % side % r) * r + (idx % side) % r
    return (x.float() + pos.float()[w]).to(torch.bfloat16).float()


def layernorm_fwd(x, gamma, beta, eps=1e-5, pos=None, side=0, r=0, save_stats=False, out=None):
    C = x.shape[-1]
    xp = _norm_input(x.reshape(-1, C), pos, side, r)
    mean, var = xp.mean(-1), xp.var(-1, unbiased=False)
    rstd = torch.rsqrt(var + eps)
    y = ((xp - mean[:, None]) * rstd[:, None] * gamma.float() + (beta.float() if beta is not None else 0)).to(torch.bfloat16)
    if out is not None:
        out.copy_(y)
        y = out
    y = y.view(x.shape)
    return (y, mean, rstd) if save_stats else y


def layernorm_bwd(dy, x, gamma, mean, rstd, pos=None, side=0, r=0, has_beta=True, dres=None):
    C = x.shape[-1]
    dy2 = dy.reshape(-1, C).float()
    xp = _norm_input(x.reshape(-1, C), pos, side, r)
    xh = (xp - mean[:, None]) * rstd[:, None]
    g = dy2 * gamma.float()
    dx = rstd[:, None] * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True))
    if dres is not None:
        dx = dx + dres.reshape(-1, C).float()
    return (dx.to(torch.bfloat16).view(x.shape), (dy2 * xh).sum(0).to(torch.bfloat16),
            dy2.sum(0).to(torch.bfloat16) if has_beta else None)


def _win(t, batch, q_side, r, windowed, n):
    if windowed:
        return t.reshape(n, r * r, -1)
    return t.reshape(batch, q_side, r, q_side, r, -1).permute(0, 1, 3, 2, 4, 5).reshape(n, r * r, -1)


def _sva(q, ks, vs, masks, rs, batch, q_side, windowed):
    """(out [N, 1024], log2-domain LSE [N, 16]).  A query whose keys are all masked attends to nothing: out = 0 and
    LSE = +inf, as the kernel writes them (its gradients are then 0 too)."""
    n = q.shape[0]
    K = torch.cat([_win(k, batch, q_side, r, windowed, n) for k, r in zip(ks, rs)], 1).view(n, -1, 16, 64).transpose(1, 2)
    V = torch.cat([_win(v, batch, q_side, r, windowed, n) for v, r in zip(vs, rs)], 1).view(n, -1, 16, 64).transpose(1, 2)
    ms = [torch.ones(n, r * r, dtype=torch.bool, device=q.device) if masks is None or masks[i] is None
          else masks[i].reshape(n, -1).bool() for i, r in enumerate(rs)]
    keep = torch.cat(ms, 1)[:, None, None, :]
    any_key = keep.any(-1, keepdim=True)
    s = (q.view(n, 1, 16, 64).transpose(1, 2) @ K.transpose(-1, -2)) / 8.0
    s = s.masked_fill(~keep, float("-inf")).masked_fill(~any_key, 0.0)
    out = ((torch.softmax(s, -1) * any_key) @ V).transpose(1, 2).reshape(n, 1024)
    lse = (torch.logsumexp(s, -1) / math.log(2.0)).masked_fill(~any_key[..., 0], float("inf")).reshape(n, 16)
    return out, lse


def sva_window_attn_fwd(q, ks, vs, masks, rs, batch, q_side, need_lse=True, windowed=False):
    out, lse = _sva(q.float(), [k.float() for k in ks], [v.float() for v in vs], masks, rs, batch, q_side, windowed)
    return out.to(torch.bfloat16), (lse if need_lse else None)


def sva_window_attn_bwd(q, out, dout, lse, ks, vs, masks, rs, batch, q_side, windowed=False, dks=None, dvs=None):
    qf = q.float().requires_grad_()
    kf = [k.float().requires_grad_() for k in ks]
    vf = [v.float().requires_grad_() for v in vs]
    with torch.enable_grad():
        o = _sva(qf, kf, vf, masks, rs, batch, q_side, windowed)[0]
    gs = [g.to(torch.bfloat16) for g in torch.autograd.grad(o, [qf] + kf + vf, dout.float())]
    T = len(ks)
    gk, gv = gs[1:1 + T], gs[1 + T:]
    if dks is not None:
        for d, g in zip(list(dks) + list(dvs), gk + gv):
            d.copy_(g)
        return gs[0], dks, dvs
    return gs[0], gk, gv


def act_fwd(x, act):
    return _ACT[act](x.float()).to(torch.bfloat16)


def act_bwd(dy, x, act):
    xf = x.float().requires_grad_()
    with torch.enable_grad():
        y = _ACT[act](xf)
    return torch.autograd.grad(y, xf, dy.float())[0].to(torch.bfloat16)


def tower_combine_fwd(logits, aggs, q_in):
    T = len(aggs)
    w = torch.softmax(logits.float()[:, :T], -1)
    return (q_in.float() + sum(w[:, t:t + 1] * aggs[t].float() for t in range(T))).to(torch.bfloat16)


def tower_combine_bwd(logits, aggs, dout):
    T = len(aggs)
    w, d = torch.softmax(logits.float()[:, :T], -1), dout.float()
    g = torch.stack([(d * a.float()).sum(-1) for a in aggs], 1)
    dl = torch.zeros(logits.shape, dtype=torch.float32)
    dl[:, :T] = w * (g - (w * g).sum(-1, keepdim=True))
    return [(w[:, t:t + 1] * d).to(torch.bfloat16) for t in range(T)], dl.to(torch.bfloat16)


def _store(y, out, accumulate):
    """the kernels' epilogue: round y (+ out when accumulating) once into `out`, or return a fresh tensor."""
    if out is None:
        return y
    out.copy_(y + out.float() if accumulate else y)
    return out


def pos_grad(dx, B, side, r, out=None, accumulate=False):
    C = dx.shape[-1]
    y = dx.float().reshape(B, side // r, r, side // r, r, C).sum((0, 1, 3)).reshape(r * r, C)
    return _store(y, out, accumulate) if out is not None else y.to(torch.bfloat16)


def bilinear(x, h, w, th, tw, *, in_bs=None, out=None, out_ld=None, out_col0=0):
    """rows of a batch are read at batch stride in_bs (default x.stride(0)); with `out`, written at row stride out_ld
    (default out.stride(1)) from column out_col0 — a column slice of a wider buffer."""
    B, C = x.shape[0], x.shape[-1]
    src = x.as_strided((B, h * w, C), (x.stride(0) if in_bs is None else in_bs, C, 1))
    y = F.interpolate(src.float().reshape(B, h, w, C).permute(0, 3, 1, 2), size=(th, tw), mode="bilinear",
                      align_corners=False)
    y = y.permute(0, 2, 3, 1).reshape(B, th * tw, C).to(torch.bfloat16)
    if out is None:
        return y
    ld = out.stride(1) if out_ld is None else out_ld
    out.as_strided((B, th * tw, C), (out.stride(0), ld, 1), out.storage_offset() + out_col0).copy_(y)
    return out


def bilinear_bwd(dout, h, w, th, tw):
    B, C = dout.shape[0], dout.shape[-1]
    x = torch.zeros(B, C, h, w, requires_grad=True)
    with torch.enable_grad():
        y = F.interpolate(x, size=(th, tw), mode="bilinear", align_corners=False)
    g = torch.autograd.grad(y, x, dout.float().reshape(B, th, tw, C).permute(0, 3, 1, 2))[0]
    return g.permute(0, 2, 3, 1).reshape(B, h * w, C).to(torch.bfloat16)


def group_colsum(x, groups, scale=1.0, out=None, accumulate=False, fp32=False):
    y = x.float().reshape(groups, -1, x.shape[-1]).sum(1) * scale
    if out is not None:
        return _store(y, out, accumulate)
    return y if fp32 else y.to(torch.bfloat16)


def group_broadcast(dmean, rows_per_group, scale, out=None, accumulate=False):
    G, C = dmean.shape
    y = (dmean.float() * scale)[:, None, :].expand(G, rows_per_group, C).reshape(G * rows_per_group, C)
    return _store(y, out, accumulate) if out is not None else y.to(torch.bfloat16)


def add_(dst, src):
    dst.add_(src)
    return dst


def adamw(p32, m, v, g16, p16, lr, beta1, beta2, eps, wd, step, grad_scale=1.0, clip_coef=None, background=False):
    """adamw_kernel (elementwise.cu): torch.optim.AdamW arithmetic on fp32 master / moments, bf16 gradients in, bf16 copy out."""
    f32 = lambda x: float(torch.tensor(x, dtype=torch.float32))     # the kernel's hyper-parameters are fp32
    lr, beta1, beta2, eps, wd = map(f32, (lr, beta1, beta2, eps, wd))
    gs = float(clip_coef[0]) if clip_coef is not None else f32(grad_scale)
    g = g16.float() * gs
    bc1, bc2 = 1.0 - beta1 ** step, 1.0 - beta2 ** step
    p32.mul_(1.0 - lr * wd)
    m.mul_(beta1).add_(g, alpha=1.0 - beta1)
    v.mul_(beta2).addcmul_(g, g, value=1.0 - beta2)
    p32.sub_((lr / bc1) * m / (v.sqrt() / bc2 ** 0.5 + eps))
    p16.copy_(p32.to(torch.bfloat16))


def sumsq_accumulate(g16, acc, ws, background=True):
    acc[0] += g16.float().pow(2).sum()


def clip_coef(sumsq, max_norm, inv_world, coef):
    norm = sumsq[0].sqrt() * inv_world
    coef[0] = inv_world * min(1.0, max_norm / (float(norm) + 1e-6))
    coef[1] = norm
    sumsq[0] = 0.0


# ---- decoder layer, splice, loss (norm.cu, attention.cu, elementwise.cu) ---------------------------------------------
def rmsnorm_fwd(x, gamma, eps=1e-6, hf_cast=False, save_stats=False):
    """y = gamma * x_hat, x_hat = x * rsqrt(mean(x^2) + eps); hf_cast rounds x_hat to bf16 first (HF LlamaRMSNorm), else
    the product is rounded once (the reference's training-time patch, train_fsdp.py:1429-1435)."""
    C = x.shape[-1]
    xf = x.reshape(-1, C).float()
    rstd = torch.rsqrt(xf.pow(2).mean(-1) + eps)
    xh = xf * rstd[:, None]
    if hf_cast:
        xh = xh.to(torch.bfloat16).float()
    y = (gamma.float() * xh).to(torch.bfloat16).view(x.shape)
    return (y, rstd) if save_stats else y


def rmsnorm_bwd(dy, x, gamma, rstd, dres=None):
    C = x.shape[-1]
    xf, dyf = x.reshape(-1, C).float(), dy.reshape(-1, C).float()
    xh = xf * rstd[:, None]
    g = dyf * gamma.float()
    dx = rstd[:, None] * (g - xh * (g * xh).mean(-1, keepdim=True))
    if dres is not None:
        dx = dx + dres.reshape(-1, C).float()
    return dx.to(torch.bfloat16).view(x.shape), (dyf * xh).sum(0).to(torch.bfloat16)


def rope_(buf, pos, cos_t, sin_t, n_heads, hd, inverse=False):
    """In place on the first n_heads * hd columns of the packed [rows, ld] buffer, rotate_half convention; cos / sin
    [max_pos, hd/2] fp32 rounded to bf16 like HF; inverse = the transposed rotation (backward)."""
    rows, half = buf.shape[0], hd // 2
    p = pos.clamp(0, cos_t.shape[0] - 1)
    c = cos_t[p].to(torch.bfloat16).float()[:, None, :]
    s_ = sin_t[p].to(torch.bfloat16).float()[:, None, :]
    if inverse:
        s_ = -s_
    x = buf[:, : n_heads * hd].float().reshape(rows, n_heads, hd)
    x1, x2 = x[..., :half], x[..., half:]
    rb = lambda t: t.to(torch.bfloat16).float()          # every product is rounded to bf16, as in the kernel / HF
    o = torch.cat([rb(x1 * c) + rb(-x2 * s_), rb(x2 * c) + rb(x1 * s_)], -1)
    buf[:, : n_heads * hd] = o.reshape(rows, n_heads * hd).to(torch.bfloat16)
    return buf


def attn_visible(Sq, Skv, causal, window=0, kmask=None, device=None):
    """[B or 1, Sq, Skv] bool: query row r (slot i = r + Skv - Sq) sees key j iff j <= i when causal, i - j < window when
    window > 0, and kmask[b, j]."""
    i = torch.arange(Sq, device=device)[:, None] + (Skv - Sq)
    j = torch.arange(Skv, device=device)[None, :]
    vis = torch.ones(Sq, Skv, dtype=torch.bool, device=device)
    if causal:
        vis = vis & (j <= i)
    if window:
        vis = vis & (i - j < window)
    vis = vis[None]
    if kmask is not None:
        vis = vis & kmask.bool()[:, None, :]
    return vis


def _attn_scores(q, k, causal, kmask, scale, window):
    """fp32 scores [B, nh, Sq, Skv] (K repeated over the GQA group) with hidden pairs at -inf, and the visibility."""
    B, Sq, nh, hd = q.shape
    Skv, nkv = k.shape[1], k.shape[2]
    K = k.float().transpose(1, 2).repeat_interleave(nh // nkv, 1)
    s = q.float().transpose(1, 2) @ K.transpose(-1, -2) * (scale if scale is not None else hd ** -0.5)
    vis = attn_visible(Sq, Skv, causal, window, kmask, q.device)[:, None]
    return s.masked_fill(~vis, float("-inf")), vis


def _store_into(g, dst):
    g = g.to(torch.bfloat16)
    if dst is None:
        return g.contiguous()
    dst.copy_(g)
    return dst


def attn_fwd(q, k, v, *, causal, kmask=None, scale=None, need_lse=False, out=None, window=0):
    """O and the log2-domain LSE of the scaled scores; a row that sees no key gets O = 0 and LSE = +inf, as the kernel
    writes them."""
    B, Sq, nh, hd = q.shape
    s, vis = _attn_scores(q, k, causal, kmask, scale, window)
    live = vis.any(-1, keepdim=True)
    p = torch.softmax(s.masked_fill(~live, 0.0), -1) * live
    V = v.float().transpose(1, 2).repeat_interleave(nh // k.shape[2], 1)
    o = _store_into((p @ V).transpose(1, 2), out)
    if not need_lse:
        return o
    lse = (torch.logsumexp(s.masked_fill(~live, 0.0), -1) / math.log(2.0)).masked_fill(~live[..., 0], float("inf"))
    return o, lse


def attn_bwd(q, k, v, o, do, lse, *, causal, kmask=None, scale=None, dq=None, dk=None, dv=None, window=0):
    """The kernels' closed form: P = exp2(S log2(e) - LSE) from the forward's LSE, delta = rowsum(dO * O) from the stored
    O, dS = P (dO V^T - delta), dQ = scale dS K, dK = scale dS^T Q and dV = P^T dO summed over the GQA group."""
    B, Sq, nh, hd = q.shape
    Skv, nkv = k.shape[1], k.shape[2]
    G = nh // nkv
    sc = scale if scale is not None else hd ** -0.5
    s, vis = _attn_scores(q, k, causal, kmask, sc, window)
    L = lse.float()[..., None]
    p = torch.exp2(s * (1.0 / math.log(2.0)) - L.masked_fill(torch.isinf(L), 0.0)).masked_fill(~vis | torch.isinf(L), 0.0)
    Q, dO = q.float().transpose(1, 2), do.float().transpose(1, 2)
    K = k.float().transpose(1, 2).repeat_interleave(G, 1)
    V = v.float().transpose(1, 2).repeat_interleave(G, 1)
    delta = (dO * o.float().transpose(1, 2)).sum(-1, keepdim=True)
    ds = p * (dO @ V.transpose(-1, -2) - delta)
    group = lambda t: t.view(B, nkv, G, Skv, hd).sum(2).transpose(1, 2)
    return (_store_into((ds @ K * sc).transpose(1, 2), dq), _store_into(group(ds.transpose(-1, -2) @ Q * sc), dk),
            _store_into(group(p.transpose(-1, -2) @ dO), dv))


def swiglu_fwd(gate, up):
    return (F.silu(gate.float()).to(torch.bfloat16).float() * up.float()).to(torch.bfloat16)


def swiglu_bwd(dout, gate, up, dgate, dup):
    g, u, d = gate.float(), up.float(), dout.float()
    sg = torch.sigmoid(g)
    dup.copy_((d * g * sg).to(torch.bfloat16))
    dgate.copy_((d * u * sg * (1 + g * (1 - sg))).to(torch.bfloat16))


def mlp_gate_up(h2d, w_gu):
    gu = gemm(h2d, w_gu)
    I = w_gu.shape[0] // 2
    return gu, swiglu_fwd(gu[:, :I], gu[:, I:])


def _span_index(B, S, start, q_side, per_sample_start=None):
    """flat positions (b * S + s) of the q x q latent rows of the image span (q rows of q latents + 1 newline)."""
    rows = torch.arange(q_side)[:, None] * (q_side + 1) + torch.arange(q_side)[None, :]
    return (torch.arange(B)[:, None] * S + start + rows.reshape(1, -1)).reshape(-1)


def span_gather(hidden, start, q_side):
    B, S, H = hidden.shape
    return hidden.reshape(B * S, H)[_span_index(B, S, start, q_side)].clone()


def span_scatter_(hidden, lat, start, q_side):
    B, S, H = hidden.shape
    hidden.view(B * S, H)[_span_index(B, S, start, q_side)] = lat.to(hidden.dtype)
    return hidden


def _splice_maps(ids, img_start, q_side, has_img):
    """per flattened position: kind 0 = text, 1 = image latent, 2 = newline; and the image row / newline row it maps to."""
    B, S = ids.shape
    span = q_side * (q_side + 1)
    pos = torch.arange(S)[None].expand(B, S)
    st = img_start.to(torch.long)[:, None] if (has_img and img_start is not None) else torch.full((B, 1), -1)
    inside = (st >= 0) & (pos >= st) & (pos < st + span)
    k = (pos - st).clamp(min=0)
    row, col = k // (q_side + 1), k % (q_side + 1)
    kind = torch.where(inside, torch.where(col == q_side, 2, 1), 0)
    img_row = torch.arange(B)[:, None] * q_side * q_side + row * q_side + col.clamp(max=q_side - 1)
    nl_row = torch.arange(B)[:, None] * q_side + row
    return kind.reshape(-1), img_row.reshape(-1), nl_row.reshape(-1)


def embed_splice(ids, img_start, embed, img, newline, q_side):
    B, S = ids.shape
    H = embed.shape[1]
    idc = ids.reshape(-1).clone()
    idc[(idc < 0) | (idc >= embed.shape[0])] = 0
    out = embed[idc].clone()
    if img is not None:
        kind, img_row, _ = _splice_maps(ids, img_start, q_side, True)
        out[kind == 1] = img.reshape(-1, H)[img_row[kind == 1]]
        out[kind == 2] = newline
    return out.view(B, S, H)


def embed_splice_bwd(dout, ids, img_start, d_embed, q_side, has_img):
    B, S, H = dout.shape
    if not has_img:
        return None, None
    kind, img_row, nl_row = _splice_maps(ids, img_start, q_side, True)
    d = dout.reshape(-1, H)
    d_img = torch.zeros(B * q_side * q_side, H, dtype=torch.bfloat16)
    d_nl = torch.zeros(B * q_side, H, dtype=torch.bfloat16)
    d_img[img_row[kind == 1]] = d[kind == 1]
    d_nl[nl_row[kind == 2]] = d[kind == 2]
    return d_img.view(B, q_side * q_side, H), d_nl


def embed_grad_sorted(dout, ids, img_start, d_embed, q_side):
    B, S, H = dout.shape
    idc = ids.reshape(-1).clone()
    idc[(idc < 0) | (idc >= d_embed.shape[0])] = 0
    kind, _, _ = _splice_maps(ids, img_start, q_side, img_start is not None)
    text = kind == 0
    acc = torch.zeros(d_embed.shape, dtype=torch.float32)
    acc.index_add_(0, idc[text], dout.reshape(-1, H)[text].float())
    touched = torch.zeros(d_embed.shape[0], dtype=torch.bool)
    touched[idc[text]] = True
    d_embed[touched] = (d_embed[touched].float() + acc[touched]).to(d_embed.dtype)


def cross_entropy(logits, labels, loss_rows, loss_acc, grad_scale, write_grad, ignore_index=-100, scale_dev=None):
    """loss_row = logsumexp(fp32 logits) - logit[label] (0 for ignored rows); loss_acc[0] += sum, [1] += count; with
    write_grad the rows are overwritten IN PLACE by (softmax - onehot) * grad_scale (* scale_dev[0])."""
    rows, V = logits.shape
    if scale_dev is not None:
        grad_scale = grad_scale * float(scale_dev[0])
    lf = logits.float()
    valid = (labels != ignore_index) & (labels >= 0) & (labels < V)
    lab = labels.clamp(0, V - 1)
    lse = torch.logsumexp(lf, -1)
    lr = torch.where(valid, lse - lf.gather(1, lab[:, None])[:, 0], torch.zeros_like(lse))
    loss_rows.copy_(lr)
    if loss_acc is not None:
        loss_acc[0] += lr.sum()
        loss_acc[1] += valid.sum()
    if write_grad:
        g = torch.softmax(lf, -1)
        g[torch.arange(rows), lab] -= 1.0
        g = g * grad_scale
        g[~valid] = 0.0
        logits.copy_(g.to(logits.dtype))


# ---- dynamic-shape (inference) branch ------------------------------------------------------------------------------------
def _span_index_hw(B, S, start, q_h, q_w):
    rows = torch.arange(q_h)[:, None] * (q_w + 1) + torch.arange(q_w)[None, :]
    return (torch.arange(B)[:, None] * S + start + rows.reshape(1, -1)).reshape(-1)


def span_gather_hw(hidden, start, q_h, q_w):
    B, S, H = hidden.shape
    return hidden.reshape(B * S, H)[_span_index_hw(B, S, start, q_h, q_w)].clone()


def span_scatter_hw_(hidden, lat, start, q_h, q_w):
    B, S, H = hidden.shape
    hidden.view(B * S, H)[_span_index_hw(B, S, start, q_h, q_w)] = lat.reshape(-1, H).to(hidden.dtype)
    return hidden


def window_gather(feat, q_side, crop=None):
    B, N, C = feat.shape
    side = int(round(N ** 0.5))
    if side * side != N or side % q_side != 0:
        raise AssertionError("window_gather: token grid is not a square multiple of the query grid")
    r = side // q_side
    y0, y1, x0, x1 = crop if crop is not None else (0, q_side, 0, q_side)
    t = feat.reshape(B, q_side, r, q_side, r, C).permute(0, 1, 3, 2, 4, 5)[:, y0:y1, x0:x1]
    return t.reshape(B * (y1 - y0) * (x1 - x0), r * r, C).contiguous()


def embed_splice_ragged(embed_w, img, newline, src, batch, max_len):
    H = embed_w.shape[1]
    src = src.to(torch.long)
    out = torch.zeros(batch * max_len, H, dtype=torch.bfloat16)
    tok = src >= 0
    out[tok] = embed_w[src[tok]]
    nl = src == -(2 ** 31)
    out[nl] = newline
    im = (src <= -2) & ~nl
    if im.any():
        out[im] = img.reshape(-1, H)[-2 - src[im]]
    return out.view(batch, max_len, H)


def require_cuda_bf16_params(params, what):
    if any(p.dtype != torch.bfloat16 for p in params):
        raise RuntimeError(f"cambrian_b200 {what} run in bf16")


_NAMES = ("gemm", "linear", "f32_to_bf16", "layernorm_fwd", "layernorm_bwd", "sva_window_attn_fwd", "sva_window_attn_bwd",
          "act_fwd", "act_bwd", "tower_combine_fwd", "tower_combine_bwd", "pos_grad", "bilinear", "bilinear_bwd",
          "group_colsum", "group_broadcast", "add_", "require_cuda_bf16_params", "adamw", "sumsq_accumulate", "clip_coef", "rmsnorm_fwd", "rmsnorm_bwd",
          "rope_", "attn_fwd", "attn_bwd", "swiglu_fwd", "swiglu_bwd", "mlp_gate_up", "span_gather", "span_scatter_",
          "embed_splice", "embed_splice_bwd", "embed_grad_sorted", "cross_entropy", "span_gather_hw", "span_scatter_hw_",
          "window_gather", "embed_splice_ragged")


class _Setter:
    """monkeypatch look-alike for spawned worker processes (the process ends with the test)."""

    @staticmethod
    def setattr(obj, name, value):
        setattr(obj, name, value)


def install(monkeypatch=None):
    """Replace the emulated entry points of `cambrian_b200.ops` for the duration of one test (pytest's monkeypatch undoes
    it; a spawned worker passes nothing); every other op keeps raising without the CUDA library."""
    if torch.cuda.is_available():
        raise RuntimeError("tests/ops_emulation.py: refusing to install kernel stand-ins in a process that can see a GPU — "
                           "they exist for host-logic tests on GPU-less machines, not as a fallback")
    monkeypatch = monkeypatch or _Setter
    from cambrian_b200 import ops
    for n in _NAMES:
        monkeypatch.setattr(ops, n, globals()[n])
    monkeypatch.setattr(ops, "_require_cuda_bf16", lambda *a: None)
