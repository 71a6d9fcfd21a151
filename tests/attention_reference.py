"""fp64 references, error bounds and case tables for tests/test_attention_gpu.py and tests/test_attention_cpu.py: the
flash-attention forward and backward of csrc/attention.cu (`ops.attn_fwd` / `ops.attn_bwd`).

Mask rule.  Query row r sits at slot i = r + Skv - Sq.  Key j is visible iff j <= i (causal), i - j < W (window W > 0) and
kmask[b, j].  A row that sees no key has O = 0 and LSE = +inf; the LSE is log2 sum_j 2^(s_j), s_j = scale log2(e) q . k_j.

Every reference is written from that definition in float64, from the bf16 inputs.  As in tests/vision_kernels_reference.py
the backward reference takes delta = rowsum(dO * O) from the bf16 O the kernel stored and P = 2^(s - LSE) from the
kernel's fp32 LSE; the forward tests hold the LSE itself.  A bf16 output is held to

    |got - ref64| <= 2^-8 |ref64| + tol

and the fp32 LSE to tol, with u = 2^-24 and the notation of tests/row_kernels_reference.py.  tol follows the kernel's order
of operations (T = 128-key tiles the row's CTA walks, hd = head dim):

Scores.  S = Q K^T is a tensor-core dot product over hd: any order of additions at 2 u each (round-toward-zero
accumulation included), 2 hd u A with A = |q| . |k|.  One multiply by the fp32 constant scale log2(e), itself rounded from
fl(scale) and fl(log2 e): 4 u |s|.  So ds = c 2 hd u A + 4 u |s| (log2 units, c = scale log2 e).

Forward.  p = ex2.approx.ftz(s - m_t) with m_t the running max (2 ulp = 4 u relative; the subtraction rounds,
u |s - m_t| <= u range, range = max s - min s over the row's visible keys); every later tile rescales o and l by
corr = ex2(m_old - m_new), 4 u for the exp2 and u for the multiply, at most T times, and the corr arguments telescope to
the range.  So every unnormalised weight has relative error rho <= ln2 (ds_max + 2 u range) + (5 T + 4) u, and a
normalised one 2 rho.  Flush-to-zero drops weights below 2^-126 of the row max: Skv 2^-126 max|v| in all.  P is rounded
to bf16 before P V while l sums the unrounded fp32 P: 2^-8 sum_j w_j |v_j|; this term dominates.  P V accumulates over
the T 128-key tiles in any order: 2 (128 T) u sum w |v|; l is 32 T sequential adds per lane and a 2-level quad tree:
(32 T + 2) u; 1 / l and o / l: 2 u.  tol_o = (2 rho + 2^-8 + (256 T + 32 T + 4) u) sum_j w_j |v_j|.
LSE = m + log2f(l): (rho + (32 T + 2) u) / ln2 + 2 u |log2 l| + u |LSE|.

Backward.  P = ex2(fmaf(s_raw, c, -LSE)): theta = ln2 (c 2 hd u A + 3 u |s| + u |s - LSE|) + 4 u relative.
dP = dO V^T on the tensor cores: 2 hd u |dO| . |v|.  delta is summed in attn_delta_kernel's lane order: 8 sequential
products per lane, then log2(lanes per head) shuffle levels (8 lanes at hd 64, 16 at hd 96 and 128): h_delta = 11 or 12,
h_delta u sum |dO O|.  dS = P (dP - delta), each of the subtraction and the product rounded once:
d_ds = P (theta |G| + 2 hd u |dO|.|v| + h_delta u sum|dO O| + u |G|) + u |dS|, G = dP - delta.  P and dS are rounded to
bf16 before the dV, dK and dQ MMAs (2^-8 each).  dV and dK accumulate over the G Sq' queries of the GQA group
(Sq' = Sq rounded up to the 64-row tile), dQ over Skv' keys (64-key tiles), any order at 2 u each; dK and dQ are
multiplied once by the fp32 scale (2 u) and every value is rounded once to bf16:
    tol_dv = sum_q (theta + 2^-8) P |dO| + 2 G Sq' u sum_q P |dO|
    tol_dk = scale [sum_q (d_ds + 2^-8 |dS|) |q| + 2 G Sq' u sum_q |dS| |q|] + 2 u |dK|
    tol_dq = scale [sum_j (d_ds + 2^-8 |dS|) |k| + 2 Skv' u sum_j |dS| |k|] + 2 u |dQ|
Each bound carries a 1 % slack for the second-order terms.  A key that no query sees gets dK = dV = 0 exactly (tol 0), and
a row that sees no key dQ = 0.
"""
from __future__ import annotations

import math

import torch

from row_kernels_reference import HALF_ULP, U

LOG2E = 1.0 / math.log(2.0)
LN2 = math.log(2.0)
BIG = 1000.0        # what hidden K / V rows are overwritten with: a key that leaked in would move every output


def gen(seed, device):
    return torch.Generator(device=device).manual_seed(seed)


def visible(Sq, Skv, causal, window, kmask, device):
    """[B or 1, Sq, Skv] bool under the module's mask rule."""
    i = torch.arange(Sq, device=device)[:, None] + (Skv - Sq)
    j = torch.arange(Skv, device=device)[None, :]
    vis = torch.ones(Sq, Skv, dtype=torch.bool, device=device)
    if causal:
        vis = vis & (j <= i)
    if window:
        vis = vis & (i - j < window)
    vis = vis[None]
    if kmask is not None:
        vis = vis & kmask.to(device).bool()[:, None, :]
    return vis


# ============================================================================================================ case tables
class Case(dict):
    """One attention problem; fields below, `id` for the test name."""
    __getattr__ = dict.__getitem__

    @property
    def id(self):
        c = self
        s = (f"{c.kind}-hd{c.hd}-B{c.B}-h{c.nh}x{c.nkv}-{c.Sq}x{c.Skv}-{'causal' if c.causal else 'full'}"
             f"{f'-w{c.window}' if c.window else ''}-{c.mask}-{c.layout}-{c.regime}")
        return s + (f"-scale{c.scale:g}" if c.scale else "")


def case(kind, hd, B, nh, nkv, Sq, Skv, causal, window=0, mask="none", layout="contig", regime="std1", scale=None):
    return Case(kind=kind, hd=hd, B=B, nh=nh, nkv=nkv, Sq=Sq, Skv=Skv, causal=causal, window=window, mask=mask,
                layout=layout, regime=regime, scale=scale)


# mask: none | all_true | left | right | hole (spans a tile boundary) | rand20 (20 % hidden) | row_false (batch row 1
# entirely hidden) | decode (slot-validity mask of a graph-replayed decode step over the whole cache)
# layout: contig | packed (q / k / v slices of one [B S, (nh + 2 nkv) hd] buffer; dq / dk / dv of a dQKV buffer) |
# padded_batch (batch stride larger than the rows) | out_slice (O written into a column slice of a wider buffer)
# regime: std1 | std3 (peaked softmax, exp2 underflow) | ramp (keys grow so the running max rises in every tile) |
# first (the row max lies in the first key tile)
FWD_CASES = [
    case("fwd", 32, 2, 4, 4, 129, 129, True, mask="right"),
    case("fwd", 64, 1, 4, 2, 577, 577, False, layout="packed"),
    case("fwd", 72, 2, 3, 3, 729, 729, False, layout="packed"),
    case("fwd", 80, 1, 6, 2, 300, 300, True, mask="hole", regime="std3"),
    case("fwd", 88, 2, 7, 1, 65, 65, True, mask="all_true", layout="padded_batch"),
    case("fwd", 96, 2, 8, 1, 128, 128, True, window=64, mask="left"),
    case("fwd", 104, 1, 3, 1, 127, 127, True, mask="rand20"),
    case("fwd", 128, 2, 8, 2, 2048, 2048, True, mask="right", layout="packed"),
    case("fwd", 128, 1, 8, 8, 1, 4096, True),
    case("fwd", 64, 2, 4, 1, 5, 700, True, mask="left"),
    case("fwd", 96, 1, 4, 4, 130, 900, True, window=257, mask="hole"),
    case("fwd", 128, 2, 2, 2, 300, 129, True),
    case("fwd", 96, 1, 2, 1, 63, 63, True, window=1, regime="std3"),
    case("fwd", 64, 2, 4, 2, 300, 300, True, window=127, mask="row_false"),
    case("fwd", 128, 1, 2, 1, 300, 300, True, window=128, mask="rand20"),
    case("fwd", 96, 1, 3, 3, 729, 729, True, window=129, mask="right"),
    case("fwd", 80, 1, 2, 2, 730, 730, True, window=729),
    case("fwd", 128, 2, 4, 1, 1, 730, False, mask="decode"),
    case("fwd", 64, 2, 4, 4, 64, 64, False, layout="out_slice", regime="std3", scale=0.3),
    case("fwd", 128, 1, 2, 1, 64, 2048, False, regime="ramp"),
    case("fwd", 128, 1, 2, 2, 128, 2048, False, regime="first"),
    case("fwd", 32, 3, 2, 2, 127, 127, False, mask="left", layout="padded_batch"),
    case("fwd", 72, 2, 3, 3, 1, 1, True),
    case("fwd", 104, 2, 6, 2, 63, 65, False, mask="rand20", layout="out_slice"),
    case("fwd", 88, 1, 4, 4, 577, 63, True, mask="hole"),
    case("fwd", 32, 1, 8, 1, 64, 127, True, window=64, mask="rand20", layout="packed"),
    case("fwd", 72, 1, 4, 2, 129, 128, False, mask="row_false", regime="std3"),
    case("fwd", 104, 1, 3, 1, 65, 300, True, window=257, mask="left", layout="packed"),
]

BWD_CASES = [
    case("bwd", 64, 2, 4, 4, 65, 65, True, layout="packed"),
    case("bwd", 96, 1, 3, 1, 127, 127, True, mask="right"),
    case("bwd", 128, 2, 8, 2, 129, 129, True, mask="rand20", layout="packed"),
    case("bwd", 64, 1, 8, 1, 191, 191, False, mask="hole"),
    case("bwd", 96, 2, 4, 4, 300, 300, True, window=64, mask="left", layout="packed"),
    case("bwd", 128, 1, 2, 2, 65, 1000, True, window=129),
    case("bwd", 64, 1, 3, 1, 1000, 300, True, layout="packed"),
    case("bwd", 96, 2, 3, 3, 127, 1000, False, mask="row_false"),
    case("bwd", 64, 1, 1, 1, 129, 129, True, mask="rand20", regime="std3"),
    case("bwd", 128, 2, 4, 1, 1000, 1000, True, window=257, mask="right", layout="packed"),
    case("bwd", 96, 2, 2, 2, 191, 191, True, window=1),
    case("bwd", 128, 1, 2, 1, 5, 700, True, mask="left"),
    case("bwd", 96, 1, 3, 1, 65, 129, False, mask="all_true", regime="std3", scale=0.3),
    case("bwd", 64, 1, 8, 8, 300, 191, True, window=127, mask="hole"),
]

# the head dims that reach every padded class (HDP 64, 80, 96, 128) of the forward
HDP_CLASSES = {64: (32, 64), 80: (72, 80), 96: (88, 96), 128: (104, 128)}


def make_kmask(c, device):
    """the case's [B, Skv] bool key mask, or None."""
    B, Skv, mode = c.B, c.Skv, c.mask
    if mode == "none":
        return None
    m = torch.ones(B, Skv, dtype=torch.bool, device=device)
    b = torch.arange(B, device=device)[:, None]
    j = torch.arange(Skv, device=device)[None, :]
    if mode == "left":
        m = j >= (b * 7 + Skv // 5)
    elif mode == "right":
        m = j < Skv - (b * 11 + Skv // 4)
    elif mode == "hole":
        lo = min(Skv - 1, 100)
        m = ~((j >= lo) & (j < lo + 40)) | (b == 1)
    elif mode == "rand20":
        m = torch.rand(B, Skv, generator=gen(77, device), device=device) >= 0.2
    elif mode == "row_false":
        m = (b != 1).expand(B, Skv).clone()
    elif mode == "decode":
        m = j <= (Skv - 1 - 37 * (b + 1))          # slots not written yet are hidden: the cache holds fewer rows
    return m.contiguous()


def make_inputs(c, device, seed=0):
    """q [B, Sq, nh, hd], k / v [B, Skv, nkv, hd] (contiguous, bf16) in the case's score regime, and dO like q."""
    B, Sq, Skv, nh, nkv, hd = c.B, c.Sq, c.Skv, c.nh, c.nkv, c.hd
    std = 3.0 if c.regime == "std3" else 1.0
    r = lambda shape, s, sd=1.0: (torch.randn(shape, generator=gen(seed + s, device), device=device) * sd)
    q = r((B, Sq, nh, hd), 1, std)
    k = r((B, Skv, nkv, hd), 2, std)
    v = r((B, Skv, nkv, hd), 3)
    if c.regime == "ramp":          # q . k grows with the key index: every 128-key tile raises the running max
        q = q.abs() * 0.5 + 0.5
        k = k * 0.5 + (torch.arange(Skv, device=device, dtype=torch.float32) / Skv * 1.5)[None, :, None, None]
    elif c.regime == "first":       # the largest scores sit in the first tile, the rest underflow in later ones
        q = q.abs() * 0.5 + 0.5
        k = k * 0.5 - 0.6
        k[:, :128] = k[:, :128] + 1.2
    do = r((B, Sq, nh, hd), 4)
    return [t.to(torch.bfloat16) for t in (q, k, v, do)]


# ================================================================================================================ forward
def fwd_ref(q, k, v, *, causal, kmask=None, scale=None, window=0):
    """fp64 O [B, Sq, nh, hd], LSE [B, nh, Sq] (log2) with tol_o, tol_lse and empty [B, nh, Sq]; computed per (b, head)."""
    B, Sq, nh, hd = q.shape
    Skv, nkv = k.shape[1], k.shape[2]
    G = nh // nkv
    dev = q.device
    scale = hd ** -0.5 if scale is None else scale
    c2 = scale * LOG2E
    T = -(-Skv // 128)
    vis_all = visible(Sq, Skv, causal, window, kmask, dev)
    O = torch.zeros(B, Sq, nh, hd, dtype=torch.float64, device=dev)
    tol_o = torch.zeros_like(O)
    lse = torch.zeros(B, nh, Sq, dtype=torch.float64, device=dev)
    tol_lse = torch.zeros_like(lse)
    empty = torch.zeros(B, nh, Sq, dtype=torch.bool, device=dev)
    for b in range(B):
        vis = vis_all[min(b, vis_all.shape[0] - 1)]
        L = vis.sum(1)
        emp = L == 0
        for h in range(nh):
            Q = q[b, :, h].double()
            K, V = k[b, :, h // G].double(), v[b, :, h // G].double()
            S2 = Q @ K.T * c2
            ds = c2 * 2 * hd * U * (Q.abs() @ K.abs().T) + 4 * U * S2.abs()
            Sm = S2.masked_fill(~vis, -math.inf)
            m = Sm.amax(1).masked_fill(emp, 0.0)
            P = torch.exp2(Sm - m[:, None])
            l = P.sum(1)
            W = P / l.clamp(min=1e-300)[:, None]
            O[b, :, h] = W @ V
            smin = S2.masked_fill(~vis, math.inf).amin(1).masked_fill(emp, 0.0)
            rng = m - smin
            rho = LN2 * (ds.masked_fill(~vis, 0.0).amax(1) + 2 * U * rng) + (5 * T + 4) * U
            wv = W @ V.abs()
            tol_o[b, :, h] = 1.01 * (2 * rho + HALF_ULP + (288 * T + 4) * U)[:, None] * wv + Skv * 2.0 ** -126 * float(
                V.abs().max()) * (~emp)[:, None]
            log2l = torch.log2(l.clamp(min=1e-300))
            lse[b, h] = (m + log2l).masked_fill(emp, math.inf)
            tol_lse[b, h] = 1.01 * (rho + (32 * T + 2) * U) / LN2 + 2 * U * log2l.abs() + U * (m + log2l).abs() + Skv * 2.0 ** -120
            empty[b, h] = emp
    return dict(o=O, tol_o=tol_o, lse=lse, tol_lse=tol_lse, empty=empty)


# =============================================================================================================== backward
def bwd_ref(q, k, v, o, do, lse, *, causal, kmask=None, scale=None, window=0):
    """fp64 dQ, dK, dV with their tolerances, from the kernel's bf16 O and fp32 LSE; computed per (b, head)."""
    B, Sq, nh, hd = q.shape
    Skv, nkv = k.shape[1], k.shape[2]
    G = nh // nkv
    dev = q.device
    scale = hd ** -0.5 if scale is None else scale
    c2 = scale * LOG2E
    h_delta = 11 if hd == 64 else 12
    nq = G * (-(-Sq // 64) * 64)
    nk = -(-Skv // 64) * 64
    vis_all = visible(Sq, Skv, causal, window, kmask, dev)
    dQ = torch.zeros(B, Sq, nh, hd, dtype=torch.float64, device=dev)
    t_dQ = torch.zeros_like(dQ)
    dK = torch.zeros(B, Skv, nkv, hd, dtype=torch.float64, device=dev)
    t_dK, dV, t_dV = torch.zeros_like(dK), torch.zeros_like(dK), torch.zeros_like(dK)
    for b in range(B):
        vis = vis_all[min(b, vis_all.shape[0] - 1)]
        for h in range(nh):
            hk = h // G
            Q, dO, Ob = q[b, :, h].double(), do[b, :, h].double(), o[b, :, h].double()
            K, V = k[b, :, hk].double(), v[b, :, hk].double()
            Lk = lse[b, h].double().to(dev)
            live = torch.isfinite(Lk)
            keep = vis & live[:, None]
            Lz = Lk.masked_fill(~live, 0.0)[:, None]
            S2 = Q @ K.T * c2
            P = torch.exp2(S2 - Lz).masked_fill(~keep, 0.0)
            theta = LN2 * (c2 * 2 * hd * U * (Q.abs() @ K.abs().T) + 3 * U * S2.abs() + U * (S2 - Lz).abs()) + 4 * U
            dP = dO @ V.T
            Ad = dO.abs() @ V.abs().T
            Dlt = (dO * Ob).sum(1, keepdim=True)
            d_dlt = h_delta * U * (dO * Ob).abs().sum(1, keepdim=True)
            Gm = dP - Dlt
            dS = P * Gm
            d_ds = P * (theta * Gm.abs() + 2 * hd * U * Ad + d_dlt + U * Gm.abs()) + U * dS.abs()
            dv = P.T @ dO
            dV[b, :, hk] += dv
            t_dV[b, :, hk] += 1.01 * (((theta + HALF_ULP) * P).T @ dO.abs() + 2 * nq * U * (P.T @ dO.abs()))
            e = 1.01 * (d_ds + HALF_ULP * dS.abs())
            dk = scale * dS.T @ Q
            dK[b, :, hk] += dk
            t_dK[b, :, hk] += scale * (e.T @ Q.abs() + 1.01 * 2 * nq * U * (dS.abs().T @ Q.abs()))
            dq = scale * dS @ K
            dQ[b, :, h] = dq
            t_dQ[b, :, h] = scale * (e @ K.abs() + 1.01 * 2 * nk * U * (dS.abs() @ K.abs())) + 2 * U * dq.abs()
    t_dK += 2 * U * dK.abs()
    return dict(dq=dQ, tol_dq=t_dQ, dk=dK, tol_dk=t_dK, dv=dV, tol_dv=t_dV)


def check_lse(name, got, ref, check_abs):
    """LSE: exactly +inf on rows that see no key, within tol elsewhere."""
    got = got.to(ref["lse"].device)
    inf = ref["empty"]
    bad = int(((torch.isinf(got) & (got > 0)) != inf).sum())
    print(f"    {name}: {int(inf.sum())} rows see no key, {bad} LSE entries with the wrong +inf pattern")
    assert bad == 0, f"{name}: {bad} LSE entries are +inf where keys are visible or finite where none are"
    keep = ~inf
    return check_abs(name, got[keep], ref["lse"][keep], ref["tol_lse"][keep])
