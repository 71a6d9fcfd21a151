"""fp64 references, error bounds and shared case tables for tests/test_aggregate_preprocess_gpu.py and
tests/test_aggregate_preprocess_cpu.py: the tower combine of the `sep` SVA layer and the adjoint of the bilinear token-grid
resize (aggregate.cu), and the GPU image preprocessing (preprocess.cu).

Arithmetic bf16 outputs are held, as in tests/vision_kernels_reference.py, to |got - ref64| <= 2^-8 |ref64| + tol, where
`tol` is the error of the fp32 arithmetic before the one rounding (u = 2^-24; a fixed-order sum of height h is within
h u sum|terms|).  Every tol below is multiplied by 1.01 (second-order terms) and by 1 + 2^-8 (the rounding of an fp32
value that is itself tol away from ref64).

Tower combine, forward.  The softmax runs over the T bf16 logits of a row (exact in fp32).  d_t = l_t - max is one fp32
subtraction (u |d_t| relative to exp(d_t)); `__expf` is within 2 + floor(1.173 |d_t|) ulp (CUDA C++ Programming Guide,
intrinsic functions table), an ulp being at most 2^-23 relative, and an underflowed or flushed value is off by at most
2^-126 absolute.  So e_t has relative error eps_t = (2 + floor(1.173 |d_t|)) 2^-23 + u |d_t|.  The sum s adds the T
positive terms in order ((T - 1) u relative, plus max eps), 1 / s and e_t * (1 / s) round once each:
    dw_t = (eps_t + max_s eps_s + (T + 1) u) w_t + T 2^-125.
Then acc = q_in and T sequential fmaf(w_t, agg_t, acc), one rounding each, and one bf16 rounding:
    tol_out = T u (|q| + sum_t w_t |a_t|) + sum_t dw_t |a_t|.

Tower combine, backward.  dagg_t = w_t * dout is one product: tol = (dw_t + u w_t) |dout|.  g_t = <dout, agg_t> is
8 ceil(C / 256) sequential fmaf per lane (a lane owns every 32nd 8-element vector), then a 5-level warp tree:
h = 8 ceil(C / 256) + 5 and dg_t = h u sum|dout agg_t|.  dot = sum_s w_s g_s in tower order (T products and T adds):
d_dot = (T + 1) u sum_s w_s |g_s| + sum_s (dw_s |g_s| + w_s dg_s).  dlogits_t = w_t (g_t - dot) with one rounding for
the difference and one for the product:
    tol_dl = dw_t |g_t - dot| + w_t (dg_t + d_dot) + 2 u w_t |g_t - dot|,
which, because |g_t - dot| <= |g_t| + sum_s w_s |g_s|, is a bound in w_t (|g_t| + sum_s w_s |g_s|) and the error of g, not
in the (possibly cancelled) result.  The padding columns [T, ld_logits) of dlogits are exactly +0.

Bilinear backward (the adjoint of elementwise.cu's bilinear).  The per-axis tap weights come from the same fp32 fused
source coordinate as the forward (vision_kernels_reference._src_coord), so taps and l = f - floor(f) are exact; 1 - l and,
at the clamped last tap, (1 - l) + l round (2 u per axis), and wy * wx rounds once: 5 u per weight.  An input pixel is an
ordered fmaf sum over its n contributing output pixels:
    tol_din = (n + 5) u sum |wy wx dout|.
The adjoint identity <bilinear(x), g> = <x, bilinear_bwd(g)> on the two kernels' bf16 outputs, summed in fp64, is then
within sum |g| (2^-8 |Y| + tol_Y) + sum |x| (2^-8 |DIN| + tol_DIN) of zero, with Y, tol_Y the forward's reference and bound.

Preprocessing.  The uint8 image is Pillow's: expand2square, then the two-pass 22-bit fixed-point bicubic resize; the
integer model below restates the two passes from `ops.resample_coeffs` and both are compared bit for bit.  The bf16 output
is one rounding of (u8 * fp32(1/255) - mean) * fp32(1 / std) in fp32; the first two operations may be contracted into one
fma (nvcc does), so an element must equal the bf16 rounding of either the fused or the unfused fp32 evaluation.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from row_kernels_reference import HALF_ULP, U
from vision_kernels_reference import _src_coord, gen, randn

SAFE = 1.01 * (1 + HALF_ULP)
ULP_REL = 2.0 ** -23            # one fp32 ulp, relative, at most
TINY = 2.0 ** -125              # 2 x the smallest normal fp32: an underflowed or flushed exponential


# ================================================================================================= tower combine (aggregate.cu)
AGG_ROWS_PER_BLOCK = 8
AGG_BLOCKS_PER_SM = 16


def combine_grid_rows(sms):
    """rows one launch covers before the grid-stride loop takes over: agg_grid_for caps the grid at 16 x SMs blocks of 8."""
    return AGG_BLOCKS_PER_SM * AGG_ROWS_PER_BLOCK * sms


def combine_rows(n, sms):
    """'cap+' = just past the grid cap (some warps take a second row), '2cap+' = two and a bit grid passes."""
    cap = combine_grid_rows(sms)
    return {"cap+": cap + 8 * sms + 5, "2cap+": 2 * cap + 13}.get(n, n)


COMBINE_C = [8, 264, 1000, 1024, 1152]         # C / 8 = 1, 33, 125, 128, 144 vectors: partly idle lanes except 1024
COMBINE_REGIMES = ["spread", "flat", "dominant", "large"]
_COMBINE_N = [1, 37, 300, 7, 1000, 129]


def _combine_cases():
    """(T, ld_logits, C, N, regime, cancel): T = 1..8 each with a dense logits row and with the model's stride 8
    (NarrowLinearFn.PAD); C, N, the score regime and near-equal <dout, agg_t> rotate across them; then the grid-stride rows."""
    cases, i = [], 0
    for T in range(1, 9):
        for ldl in sorted({T, 8}):
            cases.append((T, ldl, COMBINE_C[i % 5], _COMBINE_N[i % 6], COMBINE_REGIMES[i % 4], i % 3 == 1))
            i += 1
    cases += [(3, 8, 1024, "cap+", "spread", False), (8, 8, 264, "2cap+", "large", True),
              (5, 5, 8, "2cap+", "dominant", False), (2, 8, 1152, "cap+", "flat", True)]
    return cases


COMBINE_CASES = _combine_cases()


def combine_case_id(case):
    T, ldl, C, N, regime, cancel = case
    return f"T{T}-ld{ldl}-C{C}-N{N}-{regime}" + ("-cancel" if cancel else "")


def combine_inputs(case, N, device, seed=0):
    """logits [N, ld] (padding columns hold large values the kernel must ignore), T aggregates, q_in and dout [N, C].
    Regimes: 'spread' N(0, 2); 'flat' equal to bf16 precision; 'dominant' one tower 12 above N(0, 1); 'large' rows of
    +-100 + N(0, 4), where an unshifted exp overflows (or flushes to zero).  cancel: the aggregates share a common part,
    so the <dout, agg_t> are nearly equal and dlogits = w (g - sum w g) cancels."""
    T, ldl, C, _, regime, cancel = case
    z = torch.randn((N, T), generator=gen(seed + 1, device), device=device)
    if regime == "spread":
        lg = 2 * z
    elif regime == "flat":
        lg = 0.3 + 1e-3 * z
    elif regime == "dominant":
        lg = z.clone()
        lg[torch.arange(N, device=device), torch.arange(N, device=device) % T] += 12
    else:
        sign = torch.where(torch.arange(N, device=device) % 2 == 0, 1.0, -1.0)[:, None]
        lg = sign * 100 + 4 * z
    logits = torch.full((N, ldl), 60.0, device=device)
    logits[:, :T] = lg
    logits = logits.to(torch.bfloat16)
    if cancel:
        base = torch.randn((N, C), generator=gen(seed + 2, device), device=device)
        aggs = [(base + 1e-2 * torch.randn((N, C), generator=gen(seed + 10 + t, device), device=device)).to(torch.bfloat16)
                for t in range(T)]
    else:
        aggs = [randn((N, C), seed + 10 + t, device) for t in range(T)]
    return logits, aggs, randn((N, C), seed + 3, device), randn((N, C), seed + 4, device)


def combine_weights(logits, T):
    """fp64 softmax of the first T logits and the kernel's weight error dw (module docstring)."""
    x = logits[:, :T].double()
    d = x - x.amax(1, keepdim=True)
    e = d.exp()
    w = e / e.sum(1, keepdim=True)
    eps = (2 + torch.floor(1.173 * d.abs())) * ULP_REL + U * d.abs()
    dw = (eps + eps.amax(1, keepdim=True) + (T + 1) * U) * w + T * TINY
    return w, dw


def combine_ref(logits, aggs, q_in, dout):
    """fp64 forward and backward of the tower combine with the bounds of the module docstring.
    Returns dict(out, tol_out, dagg, tol_dagg (lists over towers), dl [N, T], tol_dl)."""
    T, C = len(aggs), q_in.shape[1]
    w, dw = combine_weights(logits, T)
    A = torch.stack([a.double() for a in aggs], 1)                       # [N, T, C]
    q, d = q_in.double(), dout.double()
    out = q + (w[..., None] * A).sum(1)
    tol_out = T * U * (q.abs() + (w[..., None] * A.abs()).sum(1)) + (dw[..., None] * A.abs()).sum(1)

    dagg = [w[:, t:t + 1] * d for t in range(T)]
    tol_dagg = [SAFE * (dw[:, t:t + 1] + U * w[:, t:t + 1]) * d.abs() for t in range(T)]
    g = (A * d[:, None]).sum(-1)                                         # [N, T]
    h = 8 * -(-C // 256) + 5
    dg = h * U * (A.abs() * d.abs()[:, None]).sum(-1)
    dot = (w * g).sum(1, keepdim=True)
    d_dot = (T + 1) * U * (w * g.abs()).sum(1, keepdim=True) + (dw * g.abs() + w * dg).sum(1, keepdim=True)
    r = g - dot
    dl = w * r
    tol_dl = dw * r.abs() + w * (dg + d_dot) + 2 * U * w * r.abs()
    return dict(out=out, tol_out=SAFE * tol_out, dagg=dagg, tol_dagg=tol_dagg, dl=dl, tol_dl=SAFE * tol_dl)


# ====================================================================================== bilinear backward (aggregate.cu)
def bilinear_bwd_cap(sms):
    """work items (input pixel, 8 channels) one launch covers before the grid-stride loop: SMs x 8 blocks of 256."""
    return sms * 8 * 256


def bilinear_bwd_batch(B, h, w, C, sms):
    """'grid' = the smallest batch whose B h w C / 8 work items exceed the cap."""
    return bilinear_bwd_cap(sms) // (h * w * C // 8) + 1 if B == "grid" else B


# (h, w, th, tw, B, C): square down / up, non-square both ways, identity, a 1-row input, up-sampling 2 -> 96 and
# 64 -> 1024, the ConvNeXt-XXL stage sides, the model's query-group resize 12 -> 24 (and 6 -> 24), and that resize at a
# batch past the grid cap
BILINEAR_BWD_CASES = [(37, 37, 24, 24, 2, 64), (24, 24, 12, 12, 2, 1024), (12, 12, 24, 24, 2, 1024),
                      (6, 6, 24, 24, 3, 1024), (18, 30, 24, 20, 2, 72), (5, 64, 40, 3, 1, 16),
                      (24, 24, 24, 24, 2, 64), (1, 16, 4, 24, 2, 8), (16, 1, 3, 1, 1, 8), (2, 2, 96, 96, 2, 16),
                      (3, 7, 96, 50, 1, 8), (64, 64, 1024, 1024, 1, 8), (256, 256, 96, 96, 1, 8),
                      (100, 100, 7, 7, 1, 24), (12, 12, 24, 24, "grid", 1024)]


def bilinear_bwd_case_id(case):
    h, w, th, tw, B, C = case
    return f"{h}x{w}-to-{th}x{tw}-B{B}-C{C}"


def axis_weights(n_in, n_out, device):
    """[n_out, n_in] fp64 tap-weight matrix of one axis of the forward (taps of the fp32 fused source coordinate)."""
    i0, i1, lam, _ = _src_coord(n_in, n_out, device)
    M = torch.zeros(n_out, n_in, dtype=torch.float64, device=device)
    o = torch.arange(n_out, device=device)
    M.index_put_((o, i0), 1 - lam, accumulate=True)
    M.index_put_((o, i1), lam, accumulate=True)
    return M


def bilinear_bwd_ref(dout, h, w, th, tw):
    """dout [B, th tw, C] -> fp64 din [B, h w, C] = My^T dout Mx, and the kernel's bound."""
    B, C = dout.shape[0], dout.shape[-1]
    dev = dout.device
    My, Mx = axis_weights(h, th, dev), axis_weights(w, tw, dev)
    d = dout.double().reshape(B, th, tw, C)
    din = torch.einsum("oi,bojc->bijc", My, torch.einsum("pj,bopc->bojc", Mx, d))
    mag = torch.einsum("oi,bojc->bijc", My.abs(), torch.einsum("pj,bopc->bojc", Mx.abs(), d.abs()))
    n = (My != 0).sum(0).double()[:, None] * (Mx != 0).sum(0).double()[None, :]
    tol = SAFE * (n[None, :, :, None] + 5) * U * mag
    return din.reshape(B, h * w, C), tol.reshape(B, h * w, C)


def bilinear_bwd_coord_allowance(dout, h, w, th, tw):
    """extra allowance of a stand-in built on torch's CPU F.interpolate, whose source coordinate may be one fp32 ulp from the
    kernel's (vision_kernels_reference.bilinear_ref): every output pixel within one input pixel of (iy, ix) may move its
    weight there by 2^-22 (max(fy, 1) + max(fx, 1))."""
    B, C = dout.shape[0], dout.shape[-1]
    dev = dout.device
    near = []
    for n_in, n_out in ((h, th), (w, tw)):
        _, _, _, f = _src_coord(n_in, n_out, dev)
        i = torch.arange(n_in, device=dev, dtype=torch.float64)
        near.append(((f[:, None] - i[None]).abs() <= 1.0).double())      # [n_out, n_in]
        near.append(2.0 ** -22 * f.clamp(min=1))
    Ny, ey, Nx, ex = near
    a = dout.double().abs().reshape(B, th, tw, C)
    t1 = torch.einsum("oi,bojc->bijc", Ny * ey[:, None], torch.einsum("pj,bopc->bojc", Nx, a))
    t2 = torch.einsum("oi,bojc->bijc", Ny, torch.einsum("pj,bopc->bojc", Nx * ex[:, None], a))
    return (t1 + t2).reshape(B, h * w, C)


# =========================================================================================== preprocessing (preprocess.cu)
def tower_processors():
    """(name, resolution, mean, std) of each vision tower's processor (towers.py), pad colour int(mean * 255)."""
    from cambrian_b200.model.multimodal_encoder.towers import CLIP_MEAN, CLIP_STD, IMNET_MEAN, IMNET_STD
    half = (0.5, 0.5, 0.5)
    return {"clip": (336, CLIP_MEAN, CLIP_STD), "siglip": (384, half, half), "dino378": (378, IMNET_MEAN, IMNET_STD),
            "dino518": (518, IMNET_MEAN, IMNET_STD), "convnext": (1024, CLIP_MEAN, CLIP_STD)}


# (H, W, tower): 1-pixel sides, tiny images up-scaled up to 1024, near-square odd sizes, strong down-scaling (ksize 49
# and 73), then one ordinary photo per tower, then a seeded set with odd |H - W| (an odd pad offset) in both orientations
PREPROCESS_EDGE = [(1, 1, "siglip"), (1, 500, "clip"), (500, 1, "dino378"), (3, 2, "dino518"), (7, 5, "siglip"),
                   (2, 1000, "convnext"), (1000, 999, "dino518"), (4000, 3000, "clip"), (337, 335, "clip"),
                   (335, 336, "clip"), (6000, 17, "clip"), (16, 16, "convnext")]
PREPROCESS_TOWER = [(480, 640, "clip"), (700, 300, "siglip"), (333, 500, "dino378"), (517, 519, "dino518"),
                    (900, 1201, "convnext")]


def _odd_offset_cases(n=4, seed=7):
    rng = np.random.default_rng(seed)
    names = ["clip", "siglip", "dino378", "dino518", "convnext"]
    out = []
    for i in range(n):
        a = int(rng.integers(2, 800))
        b = a + 2 * int(rng.integers(1, 300)) - 1
        out.append((a, b, names[int(rng.integers(0, 5))]) if i % 2 == 0 else (b, a, names[int(rng.integers(0, 5))]))
    return out


PREPROCESS_CASES = PREPROCESS_EDGE + PREPROCESS_TOWER + _odd_offset_cases()


def preprocess_case_id(case):
    H, W, tower = case
    return f"{H}x{W}-{tower}"


def preprocess_image_input(H, W, seed=0):
    """uint8 [H, W, 3] noise: every pixel an edge, so the bicubic overshoots below 0 and above 255 at every scale."""
    return np.random.default_rng(seed + H * 7919 + W).integers(0, 256, size=(H, W, 3), dtype=np.uint8)


def pad_offsets(H, W):
    """expand2square (mm_utils.py:153-164) pastes the image at ((S - W) // 2, 0) or (0, (S - H) // 2): (off_y, off_x)."""
    return ((W - H) // 2, 0) if W > H else (0, (H - W) // 2)


def expand2square(arr, pad):
    H, W, _ = arr.shape
    S = max(H, W)
    sq = np.empty((S, S, 3), dtype=np.uint8)
    sq[...] = np.asarray(pad, dtype=np.uint8)
    oy, ox = pad_offsets(H, W)
    sq[oy:oy + H, ox:ox + W] = arr
    return sq


def pillow_resize(arr, R, pad):
    """the reference's host chain: expand2square, then PIL Image.resize((R, R)) (bicubic on uint8)."""
    from PIL import Image
    return np.asarray(Image.fromarray(expand2square(arr, pad)).resize((R, R)))


def resize_model(arr, R, pad):
    """integer model of the two device passes on `ops.resample_coeffs`: per output column a sum of k[x] * pixel from
    1 << 21, an arithmetic shift by 22 and a clamp to [0, 255]; rows first, then columns, of the padded square."""
    from cambrian_b200 import ops
    sq = expand2square(arr, pad)
    S = sq.shape[0]
    bounds, kk = ops.resample_coeffs(S, R)
    bounds, kk = bounds.numpy(), kk.numpy()
    # the coefficients as a dense [S, R] matrix: every product and partial sum is an integer below 2^36, so an fp64
    # matrix product gives the exact integer sums in any order
    K = np.zeros((S, R), dtype=np.float64)
    for xx in range(R):
        x0, n = bounds[xx]
        K[x0:x0 + n, xx] = kk[xx, :n]

    def one_pass(src):                                   # resample axis 1 of [rows, S, 3]
        out = np.empty((src.shape[0], R, 3), dtype=np.uint8)
        for c in range(3):
            for r0 in range(0, src.shape[0], 1024):
                acc = (src[r0:r0 + 1024, :, c].astype(np.float64) @ K).astype(np.int64) + (1 << 21)
                out[r0:r0 + 1024, :, c] = np.clip(acc >> 22, 0, 255)
        return out
    tmp = one_pass(sq)
    return np.ascontiguousarray(one_pass(np.ascontiguousarray(tmp.transpose(1, 0, 2))).transpose(1, 0, 2))


def normalise_candidates(u8, mean, std):
    """the bf16 [3, R, R] output from the uint8 [R, R, 3] image, evaluated in fp32 as the kernel does: (fused, unfused)."""
    v = torch.from_numpy(np.ascontiguousarray(u8.transpose(2, 0, 1))).double()
    inv255 = float(np.float32(1.0) / np.float32(255.0))
    m = torch.tensor([float(np.float32(x)) for x in mean], dtype=torch.float64).view(3, 1, 1)
    inv_std = torch.tensor([float(np.float32(1.0) / np.float32(x)) for x in std], dtype=torch.float32).view(3, 1, 1)
    fused = (v * inv255 - m).float()                                    # exact in fp64, one rounding: an fma
    unfused = ((v * inv255).float().double() - m).float()
    return [(a * inv_std).to(torch.bfloat16) for a in (fused, unfused)]


def resample_ksize(S, R):
    """taps per output of Pillow's bicubic at scale S / R (csrc/preprocess.cu resample_ksize)."""
    return math.ceil(2.0 * max(S / R, 1.0)) * 2 + 1
