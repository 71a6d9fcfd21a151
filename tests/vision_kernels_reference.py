"""fp64 references, error bounds and shared case tables for tests/test_vision_kernels_gpu.py and
tests/test_vision_kernels_cpu.py: the SVA window attention (sva.cu), the vision-tower kernels (dwconv7, bilinear, patchify,
add_pos_tokens), the token gathers and splices (elementwise.cu) and the bf16 decode GEMV (gemv.cu).

Each reference is written from the operation's definition in float64.  Copies and gathers are held bitwise to an indexing
reference; `add_pos_tokens` bitwise to torch's fp32 add rounded once.  An arithmetic bf16 output is held to

    |got - ref64| <= 2^-8 |ref64| + tol

(half a bf16 ulp plus the error of the fp32 arithmetic before the one rounding), an fp32 output to `tol` alone.  `tol`
follows the kernel's operation order, with u = 2^-24 and Higham's bound h u sum|terms| for a fixed-order sum of height h:

SVA forward (per query, head and key).  A score is 8 sequential products per lane, then a 3-level shuffle tree (h = 11),
then one multiply by the fp32 constant 0.125 log2(e) (itself rounded): ds <= 11 u sum|q k| / 8 + 2 u |s| in natural-log
units.  The online softmax turns every score into a weight p = exp2(s - m) and rescales the running sums by
corr = exp2(m_old - m_new) at most once per later key: each exp2f is within 2 ulp (4 u), each subtraction rounds
(ln2 u |s - m|, and the m's telescope to the score range), each rescale multiplies once.  So every final weight has
relative error <= eta = ds_max + 2 u range2 + (6 L + 6) u (L = unmasked keys, range2 = score range in log2 units).  With
the L-term sums (L u) and the final 1/l and product (2 u): |O - ref| <= (2 eta + (2 L + 2) u) sum_k w_k |v_k|.  LSE is
m + log2(l) in the log2 domain: 1.5 (eta + (L + 2) u) + 2 u (|LSE| + |log2 l|).

SVA backward.  p = exp2(s - LSE) uses the forward's fp32 LSE: relative error theta = ds + ln2 tol_LSE + u |s2 - LSE| + 4 u.
dp = dO . v and delta = dO . O are 64-term sums (h = 11); delta is taken from the bf16 O the forward stored, so its bound
also carries sum |dO| (2^-8 |O| + tol_O), the distance of that O from the exact one.  ds = p (dp - delta) / 8 then has
dds = w (theta |dp - delta| + ddp + ddelta + u |dp - delta|) / 8 + 2 u |ds|; dV = p dO: (theta + u) w |dO|;
dK = ds q: dds |q| + u |ds q|; dQ = sum_k ds_k k_k in key order: sum_k dds_k |k_k| + (L + 1) u sum_k |ds_k k_k|.

dwconv7: the accumulator starts at the bias and takes the 49 taps by fused multiply-add, one rounding each:
49 u (|bias| + sum |w x|).

GEMV: a lane accumulates its 8-element slices of every 2048-chunk by fmaf, at most 8 ceil(K / 256) terms, then a 5-level
warp tree, then + bias and + residual: (8 ceil(K / 256) + 7) u (sum |x w| + |bias| + |residual|).  The tensor-core tile
path that `ops.gemm` keeps for M >= 6, N >= 16384 has no fixed narrow tree the test can follow, so its bound takes any
order of K additions at 2 u each (round-toward-zero accumulation included): (2 K + 7) u (sum |x w| + |bias| + |residual|).

bilinear: the source coordinate f = max((o + 0.5) (in / out) - 0.5, 0) is computed in fp32 as the kernel does: in / out
rounded once, (o + 0.5) exact, and the multiply-subtract fused into one fma (nvcc contracts it, as it does in torch's CUDA
F.interpolate).  Taps floor(f), min(floor(f) + 1, in - 1) and the weight f - floor(f) are then exact; the two lerps
(1 - l) a + l b in fp32 (two weights, two products, a sum, each rounded once, then the same again across rows) are
within 7 u max(|a|, |b|, |c|, |d|).  torch's CPU F.interpolate may round the product before subtracting: its taps and
weights are then those of an f one fp32 ulp away, which moves the output by at most ulp32(f) times the largest tap
difference; its allowance adds 2^-22 (max(fy, 1) + max(fx, 1)) max|x|.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from row_kernels_reference import HALF_ULP, U

LOG2E = 1.0 / math.log(2.0)
INT32_MIN = -(2 ** 31)


def gen(seed, device):
    return torch.Generator(device=device).manual_seed(seed)


def randn(shape, seed, device, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(shape, generator=gen(seed, device), device=device) * scale).to(dtype)


# ========================================================================================================= SVA (sva.cu)
# (q_side, B, rs, mask mode, q / k standard deviation).  Every rs list meets every mask mode; q_side, B and the score scale
# rotate so each rs also meets each of them.  Query counts 576 B, 144 B and 25 B: 25 and 75 are not multiples of the 4
# queries per CTA.
SVA_RS = [[1, 1, 1, 1], [1, 1, 1, 4], [2, 1, 3], [4], [1, 2, 1, 3, 1, 1, 2, 1]]
SVA_MASKS = ["none", "mixed", "all_masked", "tower_masked"]
_SVA_QB = [(24, 1), (12, 3), (5, 3), (5, 1), (12, 1), (24, 3)]
SVA_CASES = [(_SVA_QB[(i + j) % len(_SVA_QB)][0], _SVA_QB[(i + j) % len(_SVA_QB)][1], rs, mode, (1.0, 3.0)[(i + j) % 2])
             for i, rs in enumerate(SVA_RS) for j, mode in enumerate(SVA_MASKS)]


def sva_case_id(case):
    q, B, rs, mode, std = case
    return f"q{q}-B{B}-r{''.join(map(str, rs))}-{mode}-std{std:g}"


def sva_inputs(case, device, seed=0):
    """q [N, 1024], natural-layout K / V [B, (r q)^2, 1024] per tower, masks per the mode, dO [N, 1024]."""
    q_side, B, rs, mode, std = case
    n = B * q_side * q_side
    q = randn((n, 1024), seed + 1, device, std)
    ks = [randn((B, (r * q_side) ** 2, 1024), seed + 10 + t, device, std) for t, r in enumerate(rs)]
    vs = [randn((B, (r * q_side) ** 2, 1024), seed + 30 + t, device) for t, r in enumerate(rs)]
    dout = randn((n, 1024), seed + 2, device)
    T = len(rs)
    rnd = lambda t, r: torch.rand((n, r * r), generator=gen(seed + 50 + t, device), device=device) < 0.6
    idx = torch.arange(n, device=device)
    if mode == "none":
        masks = None
    elif mode == "mixed":
        masks = [None if t % 2 == 0 else rnd(t, r) for t, r in enumerate(rs)]
    elif mode == "all_masked":
        masks = [rnd(t, r) & (idx % 7 != 3)[:, None] for t, r in enumerate(rs)]
    else:
        masks = [rnd(t, r) & ~((idx % 5 == 1) & (idx % T == t))[:, None] for t, r in enumerate(rs)]
    return q, ks, vs, masks, dout


def window_rows(batch, q_side, r, device):
    """row of the natural [B * (r q)^2] grid that window slot w = dy * r + dx of query n = (b, qy, qx) reads: [N, r^2]."""
    side = r * q_side
    n = torch.arange(batch * q_side * q_side, device=device)
    b, qi = n // (q_side * q_side), n % (q_side * q_side)
    qy, qx = qi // q_side, qi % q_side
    w = torch.arange(r * r, device=device)
    dy, dx = w // r, w % r
    return b[:, None] * side * side + (qy[:, None] * r + dy[None]) * side + (qx[:, None] * r + dx[None])


def sva_ref(q, ks, vs, masks, rs, batch, q_side, dout):
    """fp64 forward and backward from the definition, natural layout, with the bounds of the module docstring.
    Returns dict(o, lse2, dq, dk, dv (lists shaped like ks / vs), empty [N] (no unmasked key), and tol_* of each)."""
    dev = q.device
    n = q.shape[0]
    rows = [window_rows(batch, q_side, r, dev) for r in rs]
    Kw = torch.cat([k.reshape(-1, 1024)[ix] for k, ix in zip(ks, rows)], 1).double().view(n, -1, 16, 64)
    Vw = torch.cat([v.reshape(-1, 1024)[ix] for v, ix in zip(vs, rows)], 1).double().view(n, -1, 16, 64)
    valid = torch.cat([torch.ones(n, r * r, dtype=torch.bool, device=dev) if masks is None or masks[t] is None
                       else masks[t].reshape(n, r * r).bool() for t, r in enumerate(rs)], 1)
    Q = q.double().view(n, 16, 64)
    dO = dout.double().view(n, 16, 64)
    S = torch.einsum("nhd,nlhd->nhl", Q, Kw) / 8.0
    A = torch.einsum("nhd,nlhd->nhl", Q.abs(), Kw.abs())
    vm = valid[:, None, :].expand_as(S)
    Lv = valid.sum(1).double()[:, None]                                   # [N, 1]
    empty = Lv[:, 0] == 0
    Sm = S.masked_fill(~vm, -math.inf)
    m = Sm.amax(-1, keepdim=True).masked_fill(empty[:, None, None], 0.0)
    P = torch.exp(Sm - m)
    l = P.sum(-1, keepdim=True)
    W = P / l.clamp(min=1e-300)                                          # 0 on every masked key and empty query
    O = torch.einsum("nhl,nlhd->nhd", W, Vw)
    lse2 = ((m + torch.log(l)) * LOG2E)[..., 0].masked_fill(empty[:, None], math.inf)
    log2l = torch.log2(l.clamp(min=1e-300))[..., 0]

    ds = (11 * U * A / 8 + 2 * U * S.abs()).masked_fill(~vm, 0.0)
    smin = S.masked_fill(~vm, math.inf).amin(-1).masked_fill(empty[:, None], 0.0)
    range2 = (m[..., 0] - smin) * LOG2E
    eta = 1.01 * ds.amax(-1) + 2 * U * range2 + (6 * Lv + 6) * U       # [N, 16]
    wv = torch.einsum("nhl,nlhd->nhd", W, Vw.abs())
    tol_o = (2 * eta + (2 * Lv + 2) * U)[..., None] * wv * 1.01
    tol_lse = 1.5 * (eta + (Lv + 2) * U) + 2 * U * (lse2.masked_fill(empty[:, None], 0.0).abs() + log2l.abs())

    dP = torch.einsum("nhd,nlhd->nhl", dO, Vw)
    Ad = torch.einsum("nhd,nlhd->nhl", dO.abs(), Vw.abs())
    Delta = (dO * O).sum(-1, keepdim=True)
    Ob = O.abs() * (1 + HALF_ULP) + tol_o
    d_delta = 11 * U * (dO.abs() * Ob).sum(-1, keepdim=True) + (dO.abs() * (HALF_ULP * O.abs() + tol_o)).sum(-1, keepdim=True)
    G = dP - Delta
    dS = W * G / 8.0
    s2_lse = (S * LOG2E - lse2[..., None].masked_fill(empty[:, None, None], 0.0)).abs()
    theta = 1.01 * (ds + math.log(2) * tol_lse[..., None]) + U * s2_lse + 4 * U
    d_ds = W * (theta * G.abs() + 11 * U * Ad + d_delta + U * G.abs()) / 8.0 + 2 * U * dS.abs()
    dVw = torch.einsum("nhl,nhd->nlhd", W, dO)
    t_dVw = torch.einsum("nhl,nhd->nlhd", (theta + U) * W, dO.abs())
    dKw = torch.einsum("nhl,nhd->nlhd", dS, Q)
    t_dKw = torch.einsum("nhl,nhd->nlhd", d_ds, Q.abs()) + U * torch.einsum("nhl,nhd->nlhd", dS.abs(), Q.abs())
    dQ = torch.einsum("nhl,nlhd->nhd", dS, Kw)
    t_dQ = (torch.einsum("nhl,nlhd->nhd", d_ds, Kw.abs())
            + (Lv + 1)[..., None] * U * torch.einsum("nhl,nlhd->nhd", dS.abs(), Kw.abs()))

    def scatter(win, like_list):
        """[N, L, 16, 64] per key -> natural-layout tensors shaped like ks (every row belongs to exactly one window)."""
        outs, c0 = [], 0
        for t, (like, ix) in enumerate(zip(like_list, rows)):
            rr = ix.shape[1]
            o = torch.zeros(like.numel() // 1024, 1024, dtype=torch.float64, device=dev)
            o[ix.reshape(-1)] = win[:, c0:c0 + rr].reshape(-1, 1024)
            outs.append(o.view(like.shape))
            c0 += rr
        return outs

    return dict(o=O.reshape(n, 1024), tol_o=tol_o.reshape(n, 1024), lse2=lse2, tol_lse=tol_lse, empty=empty,
                dq=dQ.reshape(n, 1024), tol_dq=t_dQ.reshape(n, 1024), dk=scatter(dKw, ks), tol_dk=scatter(t_dKw, ks),
                dv=scatter(dVw, vs), tol_dv=scatter(t_dVw, vs))


def check_lse(name, got, ref, check_abs):
    """LSE: exactly +inf where the query has no unmasked key, within tol elsewhere."""
    got = got.to(ref["lse2"].device)
    inf = ref["empty"][:, None].expand_as(got)
    bad = int((torch.isinf(got) & (got > 0) != inf).sum())
    print(f"    {name}: {int(inf[:, 0].sum())} fully masked queries, {bad} LSE entries with the wrong +inf pattern")
    assert bad == 0, f"{name}: {bad} LSE entries are +inf where keys exist or finite where none do"
    keep = ~inf
    return check_abs(name, got[keep], ref["lse2"][keep], ref["tol_lse"][keep])


# ================================================================================================ dwconv7 (elementwise.cu)
DW_MINB = 3   # CB_DW_MINB
DW_CV = 16    # channel vectors per block


def dwconv7_cfg(B, H, W, C, sms):
    """the launch dwconv7_launch picks: (channel chunks, 8-column strips, 8-row steps, ysplit, steps per y-part)."""
    nchunk = -(-(C // 8) // DW_CV)
    strips, steps = -(-W // 8), -(-H // 8)
    base = nchunk * strips * B
    want = -(-4 * DW_MINB * sms // base)
    ysplit = max(1, min(steps, want))
    return dict(nchunk=nchunk, strips=strips, steps=steps, ysplit=ysplit, per=-(-steps // ysplit))


def dwconv7_uneven_height(B, W, C, sms):
    """an H, not a multiple of 8, for which ysplit > 1 does not divide the row steps and the last y-parts are empty."""
    cfg = dwconv7_cfg(B, 8, W, C, sms)
    want = -(-4 * DW_MINB * sms // (cfg["nchunk"] * cfg["strips"] * B))
    return 8 * (2 * want + 1) - 3


# (B, H, W, C): W < 8; W <= 4 (the second 4-column half of a strip exits early); W = 1; C = 8; a partial 128-channel chunk
# after two full ones; 'uneven' = H from dwconv7_uneven_height (needs the SM count); the ConvNeXt-XXL@1024 stages.
DW_EDGE_CASES = [(2, 13, 7, 64), (1, 9, 4, 32), (1, 10, 3, 16), (1, 5, 1, 8), (1, 16, 16, 8), (2, 11, 12, 8),
                 (1, 20, 12, 264), (1, 17, 9, 136)]
DW_UNEVEN_CASES = [(1, 64, 1536), (2, 24, 264)]      # (B, W, C)
DW_STAGE_CASES = [(1, 256, 256, 384), (1, 128, 128, 768), (1, 64, 64, 1536), (1, 32, 32, 3072)]


def dwconv7_inputs(B, H, W, C, device, seed=0):
    return (randn((B, H, W, C), seed + 1, device), randn((7, 7, C), seed + 2, device, 0.15),
            randn((C,), seed + 3, device, 0.5))


def dwconv7_ref(x, w, bias):
    """y[b, y, x, c] = bias[c] + sum_{dy, dx} w[dy, dx, c] x[b, y + dy - 3, x + dx - 3, c] (zero padding) and its bound."""
    B, H, W, C = x.shape
    xp = F.pad(x.double(), (0, 0, 3, 3, 3, 3))
    wd = w.double()
    y = bias.double().expand(B, H, W, C).clone()
    mag = y.abs()
    for dy in range(7):
        for dx in range(7):
            t = xp[:, dy:dy + H, dx:dx + W] * wd[dy, dx]
            y += t
            mag += t.abs()
    return y, 49 * U * mag * 1.01


# ============================================================================================== bilinear (elementwise.cu)
# (h, w, th, tw): downsample < 2x, > 1.5x, identity, upsample 2.4x, one h != w
BILINEAR_CASES = [(27, 27, 24, 24), (37, 37, 24, 24), (24, 24, 24, 24), (10, 10, 24, 24), (18, 30, 24, 20)]
# ConvNeXt-XXL@1024 stages (side, channels), each resized to 96 x 96 into its column slice of [B, 96^2, 5760]
CONVNEXT_STAGES = [(256, 384), (128, 768), (64, 1536), (32, 3072)]
CONVNEXT_OUT = 96


def _src_coord(n_in, n_out, device):
    """the kernel's fp32 source coordinate (one fused multiply-add) -> (floor, next tap, fp64 weight, f)."""
    s = torch.tensor(float(n_in), dtype=torch.float32) / torch.tensor(float(n_out), dtype=torch.float32)
    od = torch.arange(n_out, device=device, dtype=torch.float32) + 0.5
    f = (od.double() * float(s) - 0.5).float().clamp(min=0.0)      # exact product, one rounding: fp32 fma
    i0 = f.long()
    i1 = (i0 + 1).clamp(max=n_in - 1)
    return i0, i1, (f.double() - i0.double()), f.double()


def bilinear_ref(x, h, w, th, tw):
    """x [B, h * w, C] (any dtype) -> fp64 [B, th * tw, C], the kernel's bound, and the stand-in's extra allowance."""
    B, C = x.shape[0], x.shape[-1]
    dev = x.device
    g = x[:, :h * w].double().reshape(B, h, w, C)
    y0, y1, ly, fy = _src_coord(h, th, dev)
    x0, x1, lx, fx = _src_coord(w, tw, dev)
    a, b_ = g[:, y0][:, :, x0], g[:, y0][:, :, x1]
    c, d = g[:, y1][:, :, x0], g[:, y1][:, :, x1]
    LY, LX = ly[None, :, None, None], lx[None, None, :, None]
    out = (1 - LY) * ((1 - LX) * a + LX * b_) + LY * ((1 - LX) * c + LX * d)
    mx = torch.maximum(torch.maximum(a.abs(), b_.abs()), torch.maximum(c.abs(), d.abs()))
    tol = 7 * U * mx
    coord = 2.0 ** -22 * (fy.clamp(min=1)[None, :, None, None] + fx.clamp(min=1)[None, None, :, None]) * \
        g.abs().amax((1, 2))[:, None, None, :]
    return out.reshape(B, th * tw, C), tol.reshape(B, th * tw, C), coord.reshape(B, th * tw, C)


# ================================================================================================ patchify (elementwise.cu)
PATCHIFY_NCHW_CASES = [(336, 14), (384, 14), (378, 14), (1024, 4)]     # (R, p): 24, 27 (6 px dropped), 27, 256 patches
PATCHIFY_NHWC_CASES = [(2, 16, 16, 64), (2, 15, 13, 32), (1, 7, 9, 8), (1, 12, 12, 8)]   # (B, H, W, C), p = 2


def patchify_nchw_ref(img, p):
    """[B, Cin, R, R] -> [B g g, Kpad]: row (b, gy, gx), column (c, py, px), zero columns up to Kpad = ceil8(Cin p p)."""
    B, Cin, R, _ = img.shape
    g = R // p
    K = Cin * p * p
    t = img[:, :, :g * p, :g * p].reshape(B, Cin, g, p, g, p).permute(0, 2, 4, 1, 3, 5).reshape(B * g * g, K)
    return torch.cat([t, torch.zeros(B * g * g, -(-K // 8) * 8 - K, dtype=img.dtype, device=img.device)], 1)


def patchify_nhwc_ref(x, p):
    """[B, H, W, C] -> [B gh gw, p p C]: row (b, gy, gx), column (py, px, c); trailing rows / columns dropped."""
    B, H, W, C = x.shape
    gh, gw = H // p, W // p
    return x[:, :gh * p, :gw * p].reshape(B, gh, p, gw, p, C).permute(0, 1, 3, 2, 4, 5).reshape(B * gh * gw, p * p * C)


# =========================================================================================== ViT tokens (elementwise.cu)
ADD_POS_CASES = [(576, True), (576, False), (729, True), (729, False)]   # (N, CLS): CLIP / DINOv2 with, SigLIP without


def add_pos_tokens_ref(patch, cls, pos):
    """out[b, 0] = cls + pos[0] (with CLS), out[b, c + i] = patch[b, i] + pos[c + i]: fp32 add, one rounding."""
    tok = patch.float() if cls is None else torch.cat([cls.float().expand(patch.shape[0], 1, -1), patch.float()], 1)
    return (tok + pos.float()[None]).to(torch.bfloat16)


# ======================================================================================= gathers and splices (elementwise.cu)
def window_gather_crops(q):
    """the full grid, and a single row or column at each edge: (y0, y1, x0, x1)."""
    return [None, (0, 1, 0, q), (q - 1, q, 0, q), (0, q, 0, 1), (0, q, q - 1, q)]


def window_gather_ref(feat, q_side, crop):
    """row (b, qy, qx, wy, wx) of the output = feat[b, (qy r + wy) * side + qx r + wx], qy / qx over the crop."""
    B, N, C = feat.shape
    side = int(round(N ** 0.5))
    r = side // q_side
    y0, y1, x0, x1 = crop if crop is not None else (0, q_side, 0, q_side)
    idx = [b * N + (qy * r + wy) * side + qx * r + wx for b in range(B) for qy in range(y0, y1) for qx in range(x0, x1)
           for wy in range(r) for wx in range(r)]
    return feat.reshape(B * N, C)[torch.tensor(idx, device=feat.device)].reshape(-1, r * r, C)


def span_rows(B, S, start, q_h, q_w):
    """flat positions b S + start + row (q_w + 1) + col of the latent rows of each sample's image span."""
    return [b * S + start + row * (q_w + 1) + col for b in range(B) for row in range(q_h) for col in range(q_w)]


# (B, S, start, q_h, q_w): a span ending exactly at S; one inside the sequence; a single latent row
SPAN_CASES = [(3, 40, 40 - 4 * 6, 4, 5), (2, 64, 7, 3, 6), (2, 20, 3, 1, 9)]


def embed_splice_ref(ids, img_start, embed, img, newline, q_side):
    """image span [st, st + q (q + 1)) of sample b: column q of each row is the newline, the rest img[b, row q + col];
    every other position embed[id], ids outside [0, vocab) read row 0."""
    B, S = ids.shape
    V, H = embed.shape
    out = torch.empty(B, S, H, dtype=embed.dtype, device=embed.device)
    for b in range(B):
        st = int(img_start[b]) if img is not None else -1
        for s in range(S):
            k = s - st
            if st >= 0 and 0 <= k < q_side * (q_side + 1):
                row, col = divmod(k, q_side + 1)
                out[b, s] = newline if col == q_side else img[b, row * q_side + col]
            else:
                i = int(ids[b, s])
                out[b, s] = embed[i if 0 <= i < V else 0]
    return out


def embed_splice_inputs(device, q_side=3, B=3, S=20, V=50, H=64, seed=0):
    """sample 0: span ending at S; sample 1: no image (img_start -1); sample 2: span at 2; ids >= vocab and negative
    non-image ids among the text."""
    ids = torch.randint(0, V, (B, S), generator=gen(seed + 1, device), device=device)
    ids[:, 1] = V + 3
    ids[:, -1] = -5
    ids[1, 5] = V
    span = q_side * (q_side + 1)
    starts = [S - span, -1, 2]
    for b, st in enumerate(starts):
        if st >= 0:
            ids[b, st] = -200
    img_start = torch.tensor(starts, dtype=torch.int32, device=device)
    embed = randn((V, H), seed + 2, device)
    img = randn((B, q_side * q_side, H), seed + 3, device)
    newline = randn((H,), seed + 4, device)
    return ids, img_start, embed, img, newline


def ragged_src(rows, V, n_img, device, with_img=True):
    """src row map: token ids (0 and V - 1 included), -1 (zeros), INT32_MIN (newline) and, with_img, -2 - image row."""
    kinds = [0, V - 1, -1, INT32_MIN] + ([-2, -2 - (n_img - 1)] if with_img else [])
    src = [kinds[i] if i < len(kinds) else (i * 7) % V if i % 3 == 0 else -1 if i % 3 == 1 else
           (-2 - (i % n_img) if with_img else INT32_MIN) for i in range(rows)]
    return torch.tensor(src, dtype=torch.int32, device=device)


def embed_splice_ragged_ref(embed_w, img, newline, src, batch, max_len):
    H = embed_w.shape[1]
    out = torch.empty(batch * max_len, H, dtype=torch.bfloat16, device=embed_w.device)
    for i, s in enumerate(src.tolist()):
        if s >= 0:
            out[i] = embed_w[s]
        elif s == INT32_MIN:
            out[i] = newline
        elif s == -1:
            out[i] = 0
        else:
            out[i] = img.reshape(-1, H)[-2 - s]
    return out.view(batch, max_len, H)


# ============================================================================================================ GEMV (gemv.cu)
GEMV_K = [8, 1032, 2048, 2056, 14336]
GEMV_N = [1, 15, 16, 17, 520, 4104]
# bias, residual, fp32 out
GEMV_EPILOGUES = [(b, r, f) for b in (False, True) for r in (False, True) for f in (False, True)]


def gemv_inputs(M, N, K, device, seed=0, bias=False, residual=False):
    x = randn((M, K), seed + 1, device)
    w = randn((N, K), seed + 2, device, K ** -0.5)
    b = randn((N,), seed + 3, device, 0.5) if bias else None
    r = randn((M, N), seed + 4, device) if residual else None
    return x, w, b, r


def gemv_ref(x, w, bias=None, residual=None, tile=False):
    """fp64 x w^T (+ bias) (+ residual) and the bound of the GEMV (tile=False) or of the tensor-core tile path."""
    K = x.shape[1]
    y = x.double() @ w.double().T
    mag = x.double().abs() @ w.double().abs().T
    if bias is not None:
        y = y + bias.double()
        mag = mag + bias.double().abs()
    if residual is not None:
        y = y + residual.double()
        mag = mag + residual.double().abs()
    h = (2 * K + 7) if tile else (8 * -(-K // 256) + 7)
    return y, h * U * mag * 1.01
