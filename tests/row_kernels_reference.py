"""fp64 references and error bounds for tests/test_row_kernels_gpu.py: the norm, RoPE, loss, optimizer, SwiGLU, activation
and gradient-routing kernels of a training step.

Each reference is written from the operation's definition in float64.  Where the kernel rounds an intermediate to bf16 (the
LayerNorm's x + pos, HF's x_hat cast, SwiGLU's silu, RoPE's products) the reference rounds the same intermediate; where the
fp32 value being rounded may lie on either side of a rounding boundary, the reference keeps both neighbours.

Bounds.  A bf16 output that the kernel computes in fp32 and rounds once is held to

    |got - ref64| <= 2^-8 |ref64| + tol

2^-8 is half a bf16 ulp (relative).  `tol` is the error of the fp32 arithmetic before that rounding, derived here from the
kernel's operation order: a summation tree of height h has error <= h * u * sum|terms| (u = 2^-24, Higham's bound for any
fixed-order summation), and each further fp32 operation adds <= u relative.  The tree heights are computed from the launch
configuration the kernel picks (threads per row, vectors per thread, partial-sum rows), so they follow the kernel's loops.
fp32 outputs are held to `tol` alone.
"""
from __future__ import annotations

import math

import torch

U = 2.0 ** -24          # fp32 unit roundoff
HALF_ULP = 2.0 ** -8    # half a bf16 ulp, relative


def sm_count() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------------------- checks
def check_bf16(name, got, ref, tol):
    """got bf16 (or any) vs ref float64: |got - ref| <= 2^-8 |ref| + tol elementwise; prints the worst err / bound."""
    return check_abs(name, got, ref, HALF_ULP * ref.abs() + tol)


def check_abs(name, got, ref, bound):
    got = got.to(ref.device)
    err = (got.double() - ref).abs()
    bound = torch.as_tensor(bound, dtype=torch.float64, device=ref.device).expand_as(err)
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    ratio = torch.nan_to_num(ratio, nan=float("inf"))
    worst = float(ratio.max()) if ratio.numel() else 0.0
    print(f"    {name}: worst |err|/bound = {worst:.3g}")
    if not worst <= 1.0:
        i = int(ratio.reshape(-1).argmax())
        raise AssertionError(f"{name}: worst |err|/bound = {worst:.3g} at flat index {i}: got {float(got.reshape(-1)[i])!r}, "
                             f"ref {float(ref.reshape(-1)[i])!r}, bound {float(bound.reshape(-1)[i]):.3g}; "
                             f"{int((ratio > 1).sum())} of {ratio.numel()} elements out of bound")
    return worst


def bits(t):
    return t.contiguous().view({torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.float16: torch.int16}[t.dtype])


def assert_bitwise(name, got, ref):
    g, r = bits(got.to(ref.device)), bits(ref)
    bad = int((g != r).sum())
    print(f"    {name}: {bad} of {g.numel()} elements differ bitwise")
    assert bad == 0, f"{name}: {bad} of {g.numel()} elements differ bitwise"


def sentinel_like(shape, dtype, device):
    """A buffer filled with a quiet-NaN payload: a kernel that reads it produces NaN, one that writes it changes the bits."""
    t = torch.empty(shape, dtype=dtype, device=device)
    if dtype == torch.bfloat16:
        t.view(torch.int16).fill_(0x7FA5)
    else:
        t.view(torch.int32).fill_(0x7FC0A5A5)
    return t


def round_either(v64, rel):
    """bf16 neighbours of a value the kernel computed in fp32 with relative error <= rel: (round(v(1-rel)), round(v(1+rel)))."""
    lo = (v64 * (1 - rel)).to(torch.bfloat16)
    hi = (v64 * (1 + rel)).to(torch.bfloat16)
    return lo, hi


def assert_either(name, got, lo, hi):
    g = bits(got)
    bad = int(((g != bits(lo)) & (g != bits(hi))).sum())
    split = int((bits(lo) != bits(hi)).sum())
    print(f"    {name}: {bad} of {g.numel()} elements off both roundings ({split} on a rounding boundary)")
    assert bad == 0, f"{name}: {bad} of {g.numel()} elements are neither rounding of the reference"


# ------------------------------------------------------------------------------------------------------- norms (norm.cu)
def _pow2_tpr(need):
    for t in (32, 64, 128, 256, 512):
        if need <= t:
            return t
    raise ValueError("row too wide")


def norm_fwd_cfg(C):
    """threads per row of norm_fwd_kernel (pick_tpr with 4 vectors per thread) and rows per 256-thread block."""
    tpr = _pow2_tpr(-(-(C // 8) // 4))
    return tpr, (256 // tpr if tpr < 256 else 1)


def norm_bwd_cfg(C):
    """(threads per row, vectors per thread, rows per block) of norm_bwd_kernel (bwd_cfg)."""
    vpt = 2 if C // 8 <= 1024 else 4
    tpr = _pow2_tpr(-(-(C // 8) // vpt))
    return tpr, vpt, (256 // tpr if tpr < 256 else 1)


def row_tree_height(C, tpr):
    """height of a row reduction: a thread adds its 8 * ceil(nvec / tpr) values in order, then a 5-level warp tree, then
    (tpr > 32) the warp partials in order."""
    return 8 * -(-(C // 8) // tpr) + 5 + (tpr // 32 if tpr > 32 else 0)


def norm_input(x, pos, side, r):
    """x (+ pos_embed of the row's window position, rounded to bf16 like the kernel's fused load) in float64."""
    xp = x.reshape(-1, x.shape[-1]).double()
    if pos is None:
        return xp
    rows = xp.shape[0]
    idx = torch.arange(rows, device=x.device)
    if side == 0:
        w = idx % (r * r)
    else:
        cell = idx % (side * side)
        w = (cell // side % r) * r + cell % side % r
    return (xp + pos.double()[w]).to(torch.bfloat16).double()


def norm_fwd_ref(xp, gamma, beta, eps, rms):
    """float64 statistics and output.  Returns dict(mean, rstd, xh, y)."""
    C = xp.shape[1]
    g = gamma.double()
    if rms:
        mean = torch.zeros(xp.shape[0], dtype=torch.float64, device=xp.device)
        rstd = torch.rsqrt((xp * xp).mean(1) + eps)
        xh = xp * rstd[:, None]
        y = g * xh
    else:
        mean = xp.mean(1)
        rstd = torch.rsqrt(((xp - mean[:, None]) ** 2).mean(1) + eps)
        xh = (xp - mean[:, None]) * rstd[:, None]
        y = xh * g + (beta.double() if beta is not None else 0.0)
    return dict(mean=mean, rstd=rstd, xh=xh, y=y, C=C)


def norm_fwd_tols(ref, xp, gamma, beta, rms):
    """Per-row error allowances of the forward's fp32 arithmetic.  h = the row tree's height (norm_fwd_cfg):
      mean:  a tree of C terms then a division           -> (h + 2) u mean|x|
      rstd:  variance (tree + division: (h + 2) u relative; the mean's error enters it only squared), + eps, rsqrtf
             (2 ulp), the square root halving the variance's error -> (h + 8) u relative, rounded up from h/2 + 5
      y:     gamma * rstd * (x - mean) + beta sees the mean's error times rstd * |gamma|, rstd's relative error times
             |gamma x_hat|, and 4 roundings of its own."""
    C = ref["C"]
    tpr, _ = norm_fwd_cfg(C)
    h = row_tree_height(C, tpr)
    absx = xp.abs().mean(1)
    t_mean = (h + 2) * U * absx
    t_rstd_rel = (h + 8) * U
    g = gamma.double().abs()
    gx = (ref["xh"].abs() * g).amax(1)
    b = beta.double().abs().amax() if (beta is not None and not rms) else 0.0
    t_y = (1 + HALF_ULP) * (g.amax() * ref["rstd"] * t_mean * (0.0 if rms else 1.0) + t_rstd_rel * gx + 4 * U * (gx + b))
    return dict(h=h, mean=t_mean, rstd=t_rstd_rel * ref["rstd"], y=t_y[:, None])


def norm_bwd_ref(xp, dy, gamma, dres, ref, rms):
    """float64 backward from the definition: dx = rstd (g dy - mean(g dy) - x_hat mean(g dy x_hat)) (+ dres),
    dgamma = sum_rows dy x_hat, dbeta = sum_rows dy."""
    xh, rstd = ref["xh"], ref["rstd"][:, None]
    dyf = dy.reshape(xp.shape).double()
    gd = dyf * gamma.double()
    s1 = gd.mean(1, keepdim=True) if not rms else torch.zeros_like(rstd)
    s2 = (gd * xh).mean(1, keepdim=True)
    dx = rstd * (gd - s1 - xh * s2)
    if dres is not None:
        dx = dx + dres.reshape(xp.shape).double()
    return dict(dx=dx, dgamma=(dyf * xh).sum(0), dbeta=dyf.sum(0), gd=gd, s1=s1, s2=s2, dyf=dyf)


def norm_bwd_tols(xp, ref, bref, dres, rms, rows, C, sms):
    """Per-element allowances of the backward.  The kernel rebuilds x_hat from the saved fp32 mean and rstd (their errors
    as in norm_fwd_tols), sums g dy and g dy x_hat over the row (tree height hb of norm_bwd_cfg) and applies
    dx = rstd (g dy - s1 - x_hat s2) (+ dres) in fp32.  dgamma / dbeta: each partial-sum row adds its rows in order
    (`iters` grid passes), then colsum_kernel adds ceil(P / 32) partial rows per lane and the 32 lanes in order."""
    tf = norm_fwd_tols(ref, xp, torch.ones(C, dtype=torch.float64, device=xp.device), None, rms)
    tpr, _, rpb = norm_bwd_cfg(C)
    hb = row_tree_height(C, tpr)
    rstd = ref["rstd"][:, None]
    xh = ref["xh"]
    d_xh = xh.abs() * (tf["rstd"][:, None] / rstd + 2 * U) + (0.0 if rms else rstd * tf["mean"][:, None])
    gd = bref["gd"]
    d_s1 = 0.0 if rms else (hb + 2) * U * gd.abs().mean(1, keepdim=True)
    d_s2 = (hb + 3) * U * (gd * xh).abs().mean(1, keepdim=True) + (gd.abs() * d_xh).mean(1, keepdim=True)
    core = rstd * (gd - bref["s1"] - xh * bref["s2"])
    t_dx = (rstd * (d_s1 + xh.abs() * d_s2 + bref["s2"].abs() * d_xh) + core.abs() * tf["rstd"][:, None] / rstd
            + 4 * U * rstd * (gd.abs() + bref["s1"].abs() + (xh * bref["s2"]).abs()))
    if dres is not None:
        t_dx = t_dx + U * (core.abs() + dres.reshape(xp.shape).double().abs())
    grid = min(-(-rows // rpb), 2 * sms)
    P = grid * rpb
    iters = -(-rows // P)
    hc = iters + 1 + -(-P // 32) + 32
    dyf = bref["dyf"]
    t_dg = (hc * U * (dyf * xh).abs().sum(0) + (dyf.abs() * d_xh).sum(0)) * (1 + HALF_ULP)
    t_db = hc * U * dyf.abs().sum(0) * (1 + HALF_ULP)
    return dict(dx=t_dx * (1 + HALF_ULP), dgamma=t_dg, dbeta=t_db)


# ------------------------------------------------------------------------------------------------------------------ RoPE
def rope_tables(max_pos, hd, theta=10000.0):
    """HF's fp32 cos / sin tables [max_pos, hd / 2]."""
    inv = 1.0 / (theta ** (torch.arange(0, hd, 2, dtype=torch.int64).float() / hd))
    f = torch.outer(torch.arange(max_pos, dtype=torch.float32), inv)
    return f.cos(), f.sin()


def rope_fp32_ref(buf, pos, cos_t, sin_t, n_heads, hd, inverse):
    """The kernel's arithmetic in fp32: cos / sin rounded to bf16, every product rounded to bf16 (exact in fp32: both
    factors are bf16), the two products added in fp32 and rounded.  Returns the whole new buffer."""
    rows, half = buf.shape[0], hd // 2
    p = pos.clamp(0, cos_t.shape[0] - 1)
    c = cos_t[p].to(torch.bfloat16).float()[:, None, :]
    s = sin_t[p].to(torch.bfloat16).float()[:, None, :]
    if inverse:
        s = -s
    x = buf[:, : n_heads * hd].float().reshape(rows, n_heads, hd)
    x1, x2 = x[..., :half], x[..., half:]
    rb = lambda t: t.to(torch.bfloat16).float()
    o = torch.cat([rb(x1 * c) + rb(-x2 * s), rb(x2 * c) + rb(x1 * s)], -1).to(torch.bfloat16)
    out = buf.clone()
    out[:, : n_heads * hd] = o.reshape(rows, n_heads * hd)
    return out


def rope_fp64_ref(buf, pos, cos_t, sin_t, n_heads, hd, inverse):
    """The unrounded rotation in float64 with the fp32 tables, and its allowance: cos and sin rounded to bf16 (<= 2^-8
    relative each), the two products rounded (<= 2^-8 each): 2^-7 (1 + 2^-8) (|x1 c| + |x2 s|) before the final rounding."""
    rows, half = buf.shape[0], hd // 2
    p = pos.clamp(0, cos_t.shape[0] - 1)
    c = cos_t[p].double()[:, None, :]
    s = sin_t[p].double()[:, None, :] * (-1.0 if inverse else 1.0)
    x = buf[:, : n_heads * hd].double().reshape(rows, n_heads, hd)
    x1, x2 = x[..., :half], x[..., half:]
    o = torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1)
    mag = torch.cat([(x1 * c).abs() + (x2 * s).abs(), (x2 * c).abs() + (x1 * s).abs()], -1)
    tol = 2.0 ** -7 * mag * (1 + HALF_ULP) ** 2
    return o.reshape(rows, n_heads * hd), tol.reshape(rows, n_heads * hd)
