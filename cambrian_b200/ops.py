"""Raw (non-autograd) Python wrappers over the C ABI: one function per entry point of
include/cambrian_b200.h.  Tensors are torch CUDA tensors used purely as device buffers; every call
launches the hand-written sm_90a kernel on the current torch stream.  No fallbacks."""
from __future__ import annotations

import ctypes
import os

import torch

from . import _lib
from ._lib import check, int_array, ptr, ptr_array, stream

ACT = {None: 0, "none": 0, "gelu": 1, "gelu_erf": 1, "gelu_tanh": 2, "gelu_pytorch_tanh": 2,
       "quick_gelu": 3, "silu": 4}

_ws_cache: dict = {}

# NVTX ranges around every block of the hot path (decoder layer fwd / bwd, SVA layer fwd / bwd, each tower, fused loss,
# optimizer): CB_NVTX=1 turns them on for nsys / ncu --nvtx captures; off, `nvtx()` is a shared no-op context.
_NVTX = os.environ.get("CB_NVTX", "0") != "0"


class _Null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


_NULL = _Null()


class _Range:
    __slots__ = ("name",)

    def __init__(self, name):
        self.name = name

    def __enter__(self):
        torch.cuda.nvtx.range_push(self.name)
        return self

    def __exit__(self, *a):
        torch.cuda.nvtx.range_pop()
        return False


def nvtx(name: str):
    return _Range(name) if _NVTX else _NULL


def _require_cuda_bf16(*ts):
    for t in ts:
        if t is None:
            continue
        if not t.is_cuda:
            raise _lib.CambrianB200Error("cambrian_b200 kernels need CUDA tensors (no CPU fallback)")
        if t.dtype != torch.bfloat16:
            raise ValueError(f"expected bf16 tensor, got {t.dtype}")


def require_cuda_bf16_params(params, what: str):
    """Module-level guard: every parameter must already live on the GPU in bf16 (there is no CPU / fp32 fallback)."""
    if any(p.dtype != torch.bfloat16 or not p.is_cuda for p in params):
        raise RuntimeError(f"cambrian_b200 {what} run in bf16 on CUDA only (no CPU / fp32 fallback): "
                           "call .to(device='cuda', dtype=torch.bfloat16)")


def _chk(t, name):
    _require_cuda_bf16(t)
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")


def workspace(nfloats: int, device) -> torch.Tensor:
    key = (device, torch.cuda.current_stream(device).cuda_stream)
    w = _ws_cache.get(key)
    if w is None or w.numel() < nfloats:
        w = torch.empty(max(nfloats, 1 << 20), dtype=torch.float32, device=device)
        _ws_cache[key] = w
    return w


def gemm(a: torch.Tensor, b: torch.Tensor, *, a_mn: bool = False, b_mn: bool = False, bias=None,
         colscale=None, residual=None, act=None, alpha: float = 1.0, out: torch.Tensor | None = None,
         out_dtype=torch.bfloat16, accumulate: bool = False, force_bn: int = 0) -> torch.Tensor:
    """C = epi(alpha * opA(a) @ opB(b)).  2-D or batched 3-D (leading batch dim on every operand).

    a: [M, K] (a_mn=False) or [K, M] (a_mn=True);  b: [N, K] (b_mn=False, nn.Linear layout) or [K, N].
    Row strides may exceed the logical width (ld), the last dim must be contiguous.
    """
    _require_cuda_bf16(a, b, bias, colscale, residual)
    batched = a.dim() == 3
    if batched != (b.dim() == 3):
        raise ValueError("gemm: a and b must both be 2-D or both 3-D")

    def dims(t):
        if t.stride(-1) != 1:
            raise ValueError("gemm: innermost dimension must be contiguous")
        if batched:
            return t.shape[0], t.shape[1], t.shape[2], t.stride(1), t.stride(0)
        return 1, t.shape[0], t.shape[1], t.stride(0), 0

    ba, ar, ac, lda, bsa = dims(a)
    bb, br, bc, ldb, bsb = dims(b)
    M, K = (ac, ar) if a_mn else (ar, ac)
    N, Kb = (bc, br) if b_mn else (br, bc)
    if K != Kb or ba != bb:
        raise ValueError(f"gemm: shape mismatch a={tuple(a.shape)} b={tuple(b.shape)} a_mn={a_mn} b_mn={b_mn}")
    # decode step: weight streaming.  The CUDA-core GEMV is FMA-bound at 6-8 rows, so wide outputs (N >= 16384) at
    # those row counts keep the tensor-core kernel (a threshold carried over from an earlier GPU; not re-measured on H100).
    if (_GEMV and M <= 8 and not (M >= 6 and N >= 16384) and not batched and not a_mn and not b_mn
            and act in (None, "none") and colscale is None
            and not accumulate and alpha == 1.0 and force_bn == 0 and K % 8 == 0 and lda % 8 == 0 and ldb % 8 == 0
            and a.data_ptr() % 16 == 0 and b.data_ptr() % 16 == 0):
        return gemv(a, b, bias=bias, residual=residual, out=out, out_dtype=out_dtype)
    if out is None:
        if accumulate:
            raise ValueError("gemm: accumulate=True needs an explicit `out`")
        shape = (ba, M, N) if batched else (M, N)
        out = torch.empty(shape, dtype=out_dtype, device=a.device)
    if out.dtype not in (torch.bfloat16, torch.float32) or out.stride(-1) != 1:
        raise ValueError("gemm: out must be bf16/fp32 with contiguous last dim")
    ldc = out.stride(-2)
    bsc = out.stride(0) if batched else 0
    ldr = bsr = 0
    if residual is not None:
        if residual.shape != out.shape or residual.stride(-1) != 1:
            raise ValueError("gemm: residual must match the output shape")
        ldr = residual.stride(-2)
        bsr = residual.stride(0) if batched else 0
    rc = _lib.load().cb_gemm_bf16(ptr(a), ptr(b), ptr(out), M, N, K, ba, lda, ldb, ldc, bsa, bsb, bsc,
                                  int(a_mn), int(b_mn), ptr(bias), ptr(colscale), ptr(residual), ldr, bsr,
                                  float(alpha), ACT[act], int(out.dtype == torch.float32), int(accumulate),
                                  int(force_bn), stream())
    check(rc, "cb_gemm_bf16")
    return out


_GEMV = os.environ.get("CB_GEMV", "1") != "0"


def gemv(x: torch.Tensor, w: torch.Tensor, bias=None, residual=None, out=None, out_dtype=torch.bfloat16) -> torch.Tensor:
    """y[M, N] = x[M, K] @ w[N, K]^T (+ bias) (+ residual) for M <= 8 (the KV-cache decode step)."""
    _require_cuda_bf16(x, w, bias, residual)
    M, K = x.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=out_dtype, device=x.device)
    if out.dtype not in (torch.bfloat16, torch.float32) or out.stride(-1) != 1 or out.shape != (M, N):
        raise ValueError("gemv: out must be a bf16 / fp32 [M, N] tensor with contiguous rows")
    if residual is not None and (residual.shape != out.shape or residual.stride(-1) != 1):
        raise ValueError("gemv: residual must match the output shape")
    check(_lib.load().cb_gemv_bf16(ptr(x), ptr(w), ptr(out), M, N, K, x.stride(0), w.stride(0), out.stride(0), ptr(bias),
                                   ptr(residual), residual.stride(0) if residual is not None else 0,
                                   int(out.dtype == torch.float32), stream()), "cb_gemv_bf16")
    return out


def linear(x: torch.Tensor, weight: torch.Tensor, bias=None, **kw) -> torch.Tensor:
    """y = x @ weight.T + bias for x [..., K], weight [N, K] (nn.Linear)."""
    lead = x.shape[:-1]
    x2 = x.reshape(-1, x.shape[-1])
    res = kw.pop("residual", None)
    if res is not None:
        res = res.reshape(-1, weight.shape[0])
    y = gemm(x2, weight, bias=bias, residual=res, **kw)
    return y.view(*lead, weight.shape[0])


def sva_window_attn_fwd(q, ks, vs, masks, rs, batch: int, q_side: int, need_lse: bool = True, windowed: bool = False):
    _require_cuda_bf16(q, *ks, *vs)
    n, hidden = q.shape
    out = torch.empty_like(q)
    lse = torch.empty((n, 16), dtype=torch.float32, device=q.device) if need_lse else None
    mk = None
    if masks is not None:
        masks = [None if m is None else m.contiguous().view(torch.uint8) if m.dtype == torch.bool else m
                 for m in masks]
        mk = ptr_array(masks)
    rc = _lib.load().cb_sva_window_attn_fwd(ptr(q), ptr(out), ptr(lse), len(ks), ptr_array(ks), ptr_array(vs),
                                            mk, int_array(rs), batch, q_side, hidden, int(windowed), stream())
    check(rc, "cb_sva_window_attn_fwd")
    return out, lse


def sva_window_attn_bwd(q, out, dout, lse, ks, vs, masks, rs, batch: int, q_side: int, windowed: bool = False,
                        dks=None, dvs=None):
    """dks / dvs: optional preallocated contiguous destinations (slabs of a batched-GEMM operand)."""
    _require_cuda_bf16(q, out, dout, *ks, *vs)
    dq = torch.empty_like(q)
    dks = [torch.empty_like(k) for k in ks] if dks is None else dks
    dvs = [torch.empty_like(v) for v in vs] if dvs is None else dvs
    for d, k in zip(list(dks) + list(dvs), list(ks) + list(vs)):
        if d.shape != k.shape or not d.is_contiguous():
            raise ValueError("sva_window_attn_bwd: dk / dv destinations must be contiguous and shaped like k / v")
    mk = None
    if masks is not None:
        masks = [None if m is None else m.contiguous().view(torch.uint8) if m.dtype == torch.bool else m
                 for m in masks]
        mk = ptr_array(masks)
    rc = _lib.load().cb_sva_window_attn_bwd(ptr(q), ptr(out), ptr(dout), ptr(lse), ptr(dq), len(ks),
                                            ptr_array(ks), ptr_array(vs), mk, ptr_array(dks), ptr_array(dvs),
                                            int_array(rs), batch, q_side, q.shape[1], int(windowed), stream())
    check(rc, "cb_sva_window_attn_bwd")
    return dq, dks, dvs


def layernorm_fwd(x, gamma, beta, eps: float = 1e-5, pos=None, side: int = 0, r: int = 0, save_stats=False, out=None):
    """out: optional preallocated contiguous [rows, C] bf16 destination (e.g. one slab of a batched-GEMM operand)."""
    _require_cuda_bf16(x, gamma, beta, pos)
    C_ = x.shape[-1]
    x2 = x.reshape(-1, C_)
    rows = x2.shape[0]
    if out is not None:
        if out.shape != x2.shape or not out.is_contiguous() or out.dtype != torch.bfloat16:
            raise ValueError("layernorm_fwd: `out` must be a contiguous bf16 [rows, C] tensor")
        y = out
    else:
        y = torch.empty_like(x2)
    mean = rstd = None
    if save_stats:
        mean = torch.empty(rows, dtype=torch.float32, device=x.device)
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
    rc = _lib.load().cb_layernorm_fwd(ptr(x2), ptr(gamma), ptr(beta), ptr(y), ptr(mean), ptr(rstd), rows, C_,
                                      float(eps), ptr(pos), side, r, stream())
    check(rc, "cb_layernorm_fwd")
    y = y.view(x.shape)
    return (y, mean, rstd) if save_stats else y


def layernorm_bwd(dy, x, gamma, mean, rstd, pos=None, side: int = 0, r: int = 0, has_beta: bool = True, dres=None):
    _require_cuda_bf16(dy, x, gamma, pos)
    C_ = x.shape[-1]
    x2, dy2 = x.reshape(-1, C_), dy.reshape(-1, C_)
    rows = x2.shape[0]
    dx = torch.empty_like(x2)
    dgamma = torch.empty_like(gamma)
    dbeta = torch.empty_like(gamma) if has_beta else None
    nws = _lib.load().cb_norm_bwd_workspace_floats(rows, C_)
    ws = workspace(nws, x.device)
    rc = _lib.load().cb_layernorm_bwd(ptr(dy2), ptr(x2), ptr(gamma), ptr(mean), ptr(rstd), ptr(dx), ptr(dres),
                                      ptr(dgamma), ptr(dbeta), ptr(ws), ws.numel(), rows, C_, ptr(pos), side, r,
                                      stream())
    check(rc, "cb_layernorm_bwd")
    return dx.view(x.shape), dgamma, dbeta


def rmsnorm_fwd(x, gamma, eps: float = 1e-6, hf_cast: bool = False, save_stats=False):
    _require_cuda_bf16(x, gamma)
    C_ = x.shape[-1]
    x2 = x.reshape(-1, C_)
    rows = x2.shape[0]
    y = torch.empty_like(x2)
    rstd = torch.empty(rows, dtype=torch.float32, device=x.device) if save_stats else None
    rc = _lib.load().cb_rmsnorm_fwd(ptr(x2), ptr(gamma), ptr(y), ptr(rstd), rows, C_, float(eps), int(hf_cast),
                                    stream())
    check(rc, "cb_rmsnorm_fwd")
    y = y.view(x.shape)
    return (y, rstd) if save_stats else y


def rmsnorm_bwd(dy, x, gamma, rstd, dres=None):
    _require_cuda_bf16(dy, x, gamma)
    C_ = x.shape[-1]
    x2, dy2 = x.reshape(-1, C_), dy.reshape(-1, C_)
    rows = x2.shape[0]
    dx = torch.empty_like(x2)
    dgamma = torch.empty_like(gamma)
    nws = _lib.load().cb_norm_bwd_workspace_floats(rows, C_)
    ws = workspace(nws, x.device)
    rc = _lib.load().cb_rmsnorm_bwd(ptr(dy2), ptr(x2), ptr(gamma), ptr(rstd), ptr(dx), ptr(dres), ptr(dgamma), ptr(ws),
                                    ws.numel(), rows, C_, stream())
    check(rc, "cb_rmsnorm_bwd")
    return dx.view(x.shape), dgamma


# ------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------
def _bshd_strides(t, hd):
    """t is a [B, S, heads, hd] view (possibly a slice of a packed QKV buffer) with unit stride on hd and
    heads packed at stride hd."""
    if t.dim() != 4 or t.stride(3) != 1 or (t.shape[2] > 1 and t.stride(2) != hd):
        raise ValueError(f"attention operand must be [B,S,heads,hd] with packed heads, got strides {t.stride()}")
    return t.stride(0), t.stride(1)


def _kmask_u8(kmask, B: int, Skv: int):
    """The key mask as the kernels read it: [B, Skv] contiguous uint8, row b at b * Skv (1 = attend).  A mask over a
    longer buffer (e.g. the whole [B, S_max] cache while K / V are a prefix of it) would shift every row b >= 1, so it is
    refused: slice it to the keys the call attends over."""
    if kmask is None:
        return None
    if tuple(kmask.shape) != (B, Skv):
        raise ValueError(f"attention: kmask must be [B, Skv] = [{B}, {Skv}], got {list(kmask.shape)}")
    kmask = kmask.contiguous()
    return kmask.view(torch.uint8) if kmask.dtype == torch.bool else kmask.to(torch.uint8)


def attn_fwd(q, k, v, *, causal: bool, kmask=None, scale: float | None = None, need_lse: bool = False, out=None,
             window: int = 0):
    """q [B,Sq,nh,hd], k/v [B,Skv,nkv,hd] (views are fine) -> o [B,Sq,nh,hd] contiguous (+ lse [B,nh,Sq]).
    window > 0 (causal only): query slot i = row + Skv - Sq sees key slot j iff 0 <= i - j < window (Phi-3's sliding
    window as transformers' `_prepare_4d_causal_attention_mask` builds it)."""
    _require_cuda_bf16(q, k, v)
    B, Sq, nh, hd = q.shape
    Skv, nkv = k.shape[1], k.shape[2]
    if scale is None:
        scale = hd ** -0.5
    o = out if out is not None else torch.empty((B, Sq, nh, hd), dtype=torch.bfloat16, device=q.device)
    lse = torch.empty((B, nh, Sq), dtype=torch.float32, device=q.device) if need_lse else None
    qb, qs = _bshd_strides(q, hd)
    kb, ks = _bshd_strides(k, hd)
    vb, vs_ = _bshd_strides(v, hd)
    ob, os_ = _bshd_strides(o, hd)
    kmask = _kmask_u8(kmask, B, Skv)
    if window:
        rc = _lib.load().cb_attn_fwd_window(ptr(q), ptr(k), ptr(v), ptr(o), ptr(lse), ptr(kmask), B, nh, nkv, Sq, Skv,
                                            hd, qb, qs, kb, ks, vb, vs_, ob, os_, float(scale), int(causal), int(window),
                                            stream())
        check(rc, "cb_attn_fwd_window")
        return (o, lse) if need_lse else o
    rc = _lib.load().cb_attn_fwd(ptr(q), ptr(k), ptr(v), ptr(o), ptr(lse), ptr(kmask), B, nh, nkv, Sq, Skv, hd,
                                 qb, qs, kb, ks, vb, vs_, ob, os_, float(scale), int(causal), stream())
    check(rc, "cb_attn_fwd")
    return (o, lse) if need_lse else o


def attn_bwd(q, k, v, o, do, lse, *, causal: bool, kmask=None, scale: float | None = None, dq=None, dk=None, dv=None,
             window: int = 0):
    """Returns dq [B,Sq,nh,hd], dk, dv [B,Skv,nkv,hd] (bf16).  dq/dk/dv may be preallocated (strided views ok).
    window: the sliding window the forward ran with (see attn_fwd); a query row that sees no key gets dq = 0."""
    _require_cuda_bf16(q, k, v, o, do)
    B, Sq, nh, hd = q.shape
    Skv, nkv = k.shape[1], k.shape[2]
    if scale is None:
        scale = hd ** -0.5
    dev = q.device
    delta = torch.empty((B, nh, Sq), dtype=torch.float32, device=dev)
    dq = dq if dq is not None else torch.empty((B, Sq, nh, hd), dtype=torch.bfloat16, device=dev)
    dk = dk if dk is not None else torch.empty((B, Skv, nkv, hd), dtype=torch.bfloat16, device=dev)
    dv = dv if dv is not None else torch.empty((B, Skv, nkv, hd), dtype=torch.bfloat16, device=dev)
    qb, qs = _bshd_strides(q, hd)
    kb, ks = _bshd_strides(k, hd)
    vb, vs_ = _bshd_strides(v, hd)
    ob, os_ = _bshd_strides(o, hd)
    dob, dos = _bshd_strides(do, hd)
    dqb, dqs = _bshd_strides(dq, hd)
    dkb, dks = _bshd_strides(dk, hd)
    dvb, dvs = _bshd_strides(dv, hd)
    kmask = _kmask_u8(kmask, B, Skv)
    if window:
        rc = _lib.load().cb_attn_bwd_window(ptr(q), ptr(k), ptr(v), ptr(o), ptr(do), ptr(lse), ptr(delta), ptr(dq),
                                            ptr(dk), ptr(dv), ptr(kmask), B, nh, nkv, Sq, Skv, hd, qb, qs, kb, ks, vb,
                                            vs_, ob, os_, dob, dos, dqb, dqs, dkb, dks, dvb, dvs, float(scale),
                                            int(causal), int(window), stream())
        check(rc, "cb_attn_bwd_window")
        return dq, dk, dv
    rc = _lib.load().cb_attn_bwd(ptr(q), ptr(k), ptr(v), ptr(o), ptr(do), ptr(lse), ptr(delta), ptr(dq), ptr(dk),
                                 ptr(dv), ptr(kmask), B, nh, nkv, Sq, Skv, hd, qb, qs, kb, ks, vb, vs_, ob, os_, dob, dos,
                                 dqb, dqs, dkb, dks, dvb, dvs, float(scale), int(causal), stream())
    check(rc, "cb_attn_bwd")
    return dq, dk, dv


# ------------------------------------------------------------------------------------------------
# elementwise / gather / reductions
# ------------------------------------------------------------------------------------------------
def act_fwd(x, act):
    _require_cuda_bf16(x)
    x = x.contiguous()
    y = torch.empty_like(x)
    check(_lib.load().cb_act_fwd(ptr(x), ptr(y), x.numel(), ACT[act], stream()), "cb_act_fwd")
    return y


def act_bwd(dy, x, act):
    _require_cuda_bf16(dy, x)
    dy, x = dy.contiguous(), x.contiguous()
    dx = torch.empty_like(x)
    check(_lib.load().cb_act_bwd(ptr(dy), ptr(x), ptr(dx), x.numel(), ACT[act], stream()), "cb_act_bwd")
    return dx


def swiglu_fwd(gate, up):
    """gate/up: [rows, I] views with a common row stride (e.g. the two halves of a fused [rows, 2I] buffer)."""
    _require_cuda_bf16(gate, up)
    rows, I = gate.shape
    assert gate.stride(1) == 1 and up.stride(1) == 1 and gate.stride(0) == up.stride(0)
    out = torch.empty((rows, I), dtype=torch.bfloat16, device=gate.device)
    check(_lib.load().cb_swiglu_fwd(ptr(gate), ptr(up), ptr(out), rows, I, gate.stride(0), I, stream()), "cb_swiglu_fwd")
    return out


def swiglu_bwd(dout, gate, up, dgate, dup):
    _require_cuda_bf16(dout, gate, up, dgate, dup)
    rows, I = gate.shape
    assert dgate.stride(0) == dup.stride(0) and dout.stride(1) == 1
    check(_lib.load().cb_swiglu_bwd(ptr(dout), ptr(gate), ptr(up), ptr(dgate), ptr(dup), rows, I, gate.stride(0),
                                    dout.stride(0), dgate.stride(0), stream()), "cb_swiglu_bwd")


def rope_(buf, pos, cos_t, sin_t, n_heads: int, hd: int, inverse: bool = False):
    """In-place RoPE on the first n_heads heads of each row of buf [rows, ld]."""
    _require_cuda_bf16(buf)
    assert buf.dim() == 2 and buf.stride(1) == 1 and pos.dtype == torch.int64 and pos.is_contiguous()
    check(_lib.load().cb_rope(ptr(buf), ptr(pos), ptr(cos_t), ptr(sin_t), buf.shape[0], n_heads, hd, buf.stride(0),
                              cos_t.shape[0], int(inverse), stream()), "cb_rope")
    return buf


def embed_splice(ids, img_start, embed, img, newline, q_side: int):
    B, S = ids.shape
    H = embed.shape[1]
    out = torch.empty((B, S, H), dtype=torch.bfloat16, device=embed.device)
    check(_lib.load().cb_embed_splice(ptr(ids), ptr(img_start), ptr(embed), ptr(img), ptr(newline), ptr(out), B, S, H,
                                      q_side, embed.shape[0], stream()), "cb_embed_splice")
    return out


def embed_splice_bwd(dout, ids, img_start, d_embed, q_side: int, has_img: bool):
    B, S, H = dout.shape
    dev = dout.device
    d_img = torch.empty((B, q_side * q_side, H), dtype=torch.bfloat16, device=dev) if has_img else None
    d_nl = torch.empty((B * q_side, H), dtype=torch.bfloat16, device=dev) if has_img else None
    vocab = d_embed.shape[0] if d_embed is not None else 0
    check(_lib.load().cb_embed_splice_bwd(ptr(dout), ptr(ids), ptr(img_start), ptr(d_embed), ptr(d_img), ptr(d_nl), B, S,
                                          H, q_side, vocab, stream()), "cb_embed_splice_bwd")
    return d_img, d_nl


def embed_grad_sorted(dout, ids, img_start, d_embed, q_side: int):
    """Deterministic embedding-row gradient: d_embed[id] += sum over the text positions holding `id` of dout rows, summed in
    position order (ids outside [0, vocab) add to row 0, the row embed_splice reads for them; rows of ids that do not occur
    are not touched).  The sort of 8 K token ids is device-side index plumbing (torch)."""
    B, S, H = dout.shape
    vocab = d_embed.shape[0]
    keys = ids.reshape(B, S).clamp(min=0)
    keys = torch.where(keys >= vocab, torch.zeros_like(keys), keys)
    if img_start is not None:
        span = q_side * (q_side + 1)
        pos = torch.arange(S, device=ids.device)[None]
        st = img_start.to(torch.long)[:, None]
        keys = torch.where((st >= 0) & (pos >= st) & (pos < st + span), torch.full_like(keys, vocab), keys)
    keys = keys.reshape(-1).contiguous()
    order = torch.argsort(keys, stable=True).to(torch.int32)
    check(_lib.load().cb_embed_grad_sorted(ptr(dout), ptr(keys), ptr(order), ptr(d_embed), B * S, H, vocab, stream()),
          "cb_embed_grad_sorted")


def add_pos_tokens(patch, cls, pos):
    B, N, C_ = patch.shape
    T = N + (1 if cls is not None else 0)
    out = torch.empty((B, T, C_), dtype=torch.bfloat16, device=patch.device)
    check(_lib.load().cb_add_pos_tokens(ptr(patch), ptr(cls), ptr(pos), ptr(out), B, N, C_, stream()), "cb_add_pos_tokens")
    return out


def bilinear(x, h: int, w: int, th: int, tw: int, *, in_bs=None, out=None, out_ld=None, out_col0: int = 0):
    """x: [B, >=h*w, C] token grid (first h*w rows of each batch used, e.g. after skipping CLS via a view)."""
    B, C_ = x.shape[0], x.shape[-1]
    in_bs = x.stride(0) if in_bs is None else in_bs
    if out is None:
        out = torch.empty((B, th * tw, C_), dtype=torch.bfloat16, device=x.device)
    out_ld = out.stride(1) if out_ld is None else out_ld
    check(_lib.load().cb_bilinear(ptr(x), ptr(out), B, h, w, th, tw, C_, in_bs, out.stride(0), out_ld, out_col0, stream()),
          "cb_bilinear")
    return out


def bilinear_bwd(dout, h: int, w: int, th: int, tw: int):
    """Adjoint of `bilinear` on contiguous grids: dout [B, th*tw, C] -> din [B, h*w, C]."""
    _require_cuda_bf16(dout)
    dout = dout.contiguous()
    B, C_ = dout.shape[0], dout.shape[-1]
    if dout.shape[1] != th * tw:
        raise ValueError(f"bilinear_bwd: gradient has {dout.shape[1]} tokens, expected {th} x {tw}")
    din = torch.empty((B, h * w, C_), dtype=torch.bfloat16, device=dout.device)
    check(_lib.load().cb_bilinear_bwd(ptr(dout), ptr(din), B, h, w, th, tw, C_, stream()), "cb_bilinear_bwd")
    return din


def tower_combine_fwd(logits, aggs, q_in):
    """out = q_in + sum_t softmax(logits[:, :T])[:, t] * aggs[t]  (vision_sampler.py:369-371, :396-398).
    logits [N, >= T] bf16 (extra columns are padding), aggs: T tensors [N, C], q_in [N, C]."""
    _require_cuda_bf16(logits, q_in, *aggs)
    N, C_ = q_in.shape
    if not q_in.is_contiguous():
        raise ValueError("tower_combine_fwd: q_in must be contiguous (the kernel reads it at row stride C)")
    if logits.shape[0] != N or logits.stride(1) != 1 or any(a.shape != q_in.shape or not a.is_contiguous() for a in aggs):
        raise ValueError("tower_combine_fwd: logits [N, Tpad] and T contiguous aggregates shaped like q_in are required")
    out = torch.empty_like(q_in)
    check(_lib.load().cb_tower_combine_fwd(ptr(logits), logits.stride(0), ptr_array(aggs), ptr(q_in), ptr(out), N, C_,
                                           len(aggs), stream()), "cb_tower_combine_fwd")
    return out


def tower_combine_bwd(logits, aggs, dout):
    """Returns (daggs: list of T [N, C], dlogits [N, Tpad] with zero padding columns); d q_in is dout itself."""
    _require_cuda_bf16(logits, dout, *aggs)
    N, C_ = dout.shape
    if not logits.is_contiguous() or not dout.is_contiguous():
        raise ValueError("tower_combine_bwd: contiguous logits / dout are required")
    if logits.dim() != 2 or logits.shape[0] != N or logits.shape[1] > 32:
        raise ValueError(f"tower_combine_bwd: logits {tuple(logits.shape)} must be [N={N}, Tpad <= 32]")
    if any(a.shape != dout.shape or not a.is_contiguous() for a in aggs):
        raise ValueError("tower_combine_bwd: T contiguous aggregates shaped like dout are required")
    daggs = [torch.empty_like(a) for a in aggs]
    dlogits = torch.empty_like(logits)
    check(_lib.load().cb_tower_combine_bwd(ptr(logits), logits.stride(0), ptr_array(aggs), ptr(dout), ptr_array(daggs),
                                           ptr(dlogits), N, C_, len(aggs), stream()), "cb_tower_combine_bwd")
    return daggs, dlogits


def patchify_nchw(img, p: int):
    B, Cin, R, _ = img.shape
    img = img.contiguous()
    K = Cin * p * p
    Kpad = (K + 7) // 8 * 8
    g = R // p
    out = torch.empty((B * g * g, Kpad), dtype=torch.bfloat16, device=img.device)
    check(_lib.load().cb_patchify_nchw(ptr(img), ptr(out), B, Cin, R, p, Kpad, stream()), "cb_patchify_nchw")
    return out


def patchify_nhwc(x, p: int):
    B, H, W, C_ = x.shape
    out = torch.empty((B * (H // p) * (W // p), p * p * C_), dtype=torch.bfloat16, device=x.device)
    check(_lib.load().cb_patchify_nhwc(ptr(x), ptr(out), B, H, W, C_, p, stream()), "cb_patchify_nhwc")
    return out


def dwconv7(x, w, bias):
    B, H, W, C_ = x.shape
    out = torch.empty_like(x)
    check(_lib.load().cb_dwconv7(ptr(x), ptr(w), ptr(bias), ptr(out), B, H, W, C_, stream()), "cb_dwconv7")
    return out


def add_(dst, src):
    assert dst.is_contiguous() and src.is_contiguous() and dst.numel() == src.numel()
    check(_lib.load().cb_add_inplace(ptr(dst), ptr(src), dst.numel(), stream()), "cb_add_inplace")
    return dst


def group_colsum(x, groups: int, scale: float = 1.0, out=None, accumulate: bool = False, fp32: bool = False):
    C_ = x.shape[-1]
    x2 = x.reshape(-1, C_)
    rpg = x2.shape[0] // groups
    if out is None:
        out = torch.empty((groups, C_), dtype=torch.float32 if fp32 else torch.bfloat16, device=x.device)
    ob, of = (None, out) if out.dtype == torch.float32 else (out, None)
    check(_lib.load().cb_group_colsum(ptr(x2), ptr(ob), ptr(of), groups, rpg, C_, float(scale), int(accumulate), stream()),
          "cb_group_colsum")
    return out


def group_broadcast(dmean, rows_per_group: int, scale: float, out=None, accumulate: bool = False):
    groups, C_ = dmean.shape
    if out is None:
        out = torch.empty((groups * rows_per_group, C_), dtype=torch.bfloat16, device=dmean.device)
    check(_lib.load().cb_group_broadcast(ptr(dmean), ptr(out), groups, rows_per_group, C_, float(scale), int(accumulate),
                                         stream()), "cb_group_broadcast")
    return out


def pos_grad(dx, B: int, side: int, r: int, out=None, accumulate: bool = False):
    C_ = dx.shape[-1]
    if out is None:
        out = torch.empty((r * r, C_), dtype=torch.bfloat16, device=dx.device)
    check(_lib.load().cb_pos_grad(ptr(dx), ptr(out), B, side, r, C_, int(accumulate), stream()), "cb_pos_grad")
    return out


def f32_to_bf16(src, dst, scale: float = 1.0, cols: int | None = None, out_ld: int | None = None):
    """src fp32 contiguous viewed as [rows, cols]; dst bf16 rows at stride out_ld."""
    cols = src.shape[-1] if cols is None else cols
    rows = src.numel() // cols
    out_ld = cols if out_ld is None else out_ld
    check(_lib.load().cb_f32_to_bf16(ptr(src), ptr(dst), rows, cols, out_ld, float(scale), stream()), "cb_f32_to_bf16")
    return dst


def cross_entropy(logits, labels, loss_rows, loss_acc, grad_scale: float, write_grad: bool, ignore_index: int = -100,
                  scale_dev=None):
    """scale_dev: optional fp32 device tensor; its element 0 multiplies grad_scale on the device (1 / #valid labels)."""
    rows, V = logits.shape
    check(_lib.load().cb_cross_entropy_ex(ptr(logits), ptr(labels), ptr(loss_rows), ptr(loss_acc), rows, V,
                                          logits.stride(0), float(grad_scale), ptr(scale_dev), int(write_grad), ignore_index,
                                          stream()), "cb_cross_entropy_ex")


def adamw(p32, m, v, g16, p16, lr, beta1, beta2, eps, wd, step: int, grad_scale: float = 1.0, clip_coef=None,
          background: bool = False):
    """clip_coef: optional fp32 DEVICE tensor whose element 0 replaces grad_scale (written by `clip_coef`);
    background: one small block per SM so the update co-resides with persistent GEMM CTAs."""
    check(_lib.load().cb_adamw_ex(ptr(p32), ptr(m), ptr(v), ptr(g16), ptr(p16), p32.numel(), float(lr), float(beta1),
                                  float(beta2), float(eps), float(wd), int(step), float(grad_scale), ptr(clip_coef),
                                  int(background), stream()), "cb_adamw_ex")


def adamw_host(p32, m, v, g16, p16, lr, beta1, beta2, eps, wd, step: int, grad_scale: float = 1.0, clip_coef=None,
               ctas: int = 0):
    """`adamw` with p32, m, v in host memory registered by `host_register` (the update streams them over PCIe and is
    bitwise equal to `adamw`); g16, p16 and clip_coef on the device.  ctas: grid size, 0 = the measured default."""
    check(_lib.load().cb_adamw_host(ptr(p32), ptr(m), ptr(v), ptr(g16), ptr(p16), p32.numel(), float(lr), float(beta1),
                                    float(beta2), float(eps), float(wd), int(step), float(grad_scale), ptr(clip_coef),
                                    int(ctas), stream()), "cb_adamw_host")


def adamw8(p32, qm, qv, sm, sv, g16, p16, lr, beta1, beta2, eps, wd, step: int, grad_scale: float = 1.0, clip_coef=None,
           background: bool = False):
    """`adamw` with 8-bit block-wise moments (adam8bit.py states the format): qm / qv uint8 codes (one per element), sm /
    sv fp32 absmax per 256-element block (ceil(n / 256) each); p32 stays the fp32 master."""
    check(_lib.load().cb_adamw8(ptr(p32), ptr(qm), ptr(qv), ptr(sm), ptr(sv), ptr(g16), ptr(p16), p32.numel(), float(lr),
                                float(beta1), float(beta2), float(eps), float(wd), int(step), float(grad_scale),
                                ptr(clip_coef), int(background), stream()), "cb_adamw8")


def adamw8_host(p32, qm, qv, sm, sv, g16, p16, lr, beta1, beta2, eps, wd, step: int, grad_scale: float = 1.0,
                clip_coef=None, ctas: int = 0):
    """`adamw8` with p32, qm, qv, sm, sv in host memory registered by `host_register` (bitwise equal to `adamw8`)."""
    check(_lib.load().cb_adamw8_host(ptr(p32), ptr(qm), ptr(qv), ptr(sm), ptr(sv), ptr(g16), ptr(p16), p32.numel(),
                                     float(lr), float(beta1), float(beta2), float(eps), float(wd), int(step),
                                     float(grad_scale), ptr(clip_coef), int(ctas), stream()), "cb_adamw8_host")


_HOST_REGISTER_PORTABLE, _HOST_REGISTER_MAPPED = 1, 2


def host_register(t):
    """Page-lock a contiguous CPU tensor's own bytes and map them into the device address space (cudaHostRegister, mapped
    | portable), for `adamw_host`.  torch's pinned allocator would round a 33 GB request up to 64 GB; this pins exactly
    the tensor.  Call `host_unregister` before the tensor is freed."""
    if t.is_cuda or not t.is_contiguous():
        raise ValueError("host_register: expects a contiguous CPU tensor")
    torch.cuda.check_error(torch.cuda.cudart().cudaHostRegister(
        t.data_ptr(), t.numel() * t.element_size(), _HOST_REGISTER_PORTABLE | _HOST_REGISTER_MAPPED))
    return t


def host_unregister(t):
    torch.cuda.check_error(torch.cuda.cudart().cudaHostUnregister(t.data_ptr()))


def sumsq_accumulate(g16, acc, ws, background: bool = True):
    """acc[0] += sum(g16^2) (deterministic); g16 bf16 contiguous with numel % 8 == 0; ws fp32 scratch (>= 4096)."""
    _require_cuda_bf16(g16)
    check(_lib.load().cb_sumsq_bf16(ptr(g16), g16.numel(), ptr(acc), ptr(ws), ws.numel(), int(background), stream()),
          "cb_sumsq_bf16")


def clip_coef(sumsq, max_norm: float, inv_world: float, coef):
    """coef[0] = inv_world * min(1, max_norm / (norm + 1e-6)), coef[1] = norm of the averaged gradient; resets sumsq."""
    check(_lib.load().cb_clip_coef(ptr(sumsq), float(max_norm), float(inv_world), ptr(coef), stream()), "cb_clip_coef")


def span_gather(hidden, start: int, q_side: int):
    B, S, H = hidden.shape
    lat = torch.empty((B * q_side * q_side, H), dtype=torch.bfloat16, device=hidden.device)
    check(_lib.load().cb_span_gather(ptr(hidden), ptr(lat), B, S, H, start, q_side, stream()), "cb_span_gather")
    return lat


def span_scatter_(hidden, lat, start: int, q_side: int):
    B, S, H = hidden.shape
    check(_lib.load().cb_span_scatter(ptr(hidden), ptr(lat), B, S, H, start, q_side, stream()), "cb_span_scatter")
    return hidden


def span_gather_hw(hidden, start: int, q_h: int, q_w: int):
    """Dynamic branch (cambrian_llama.py:208-253): q_h rows of (q_w latent queries + 1 newline) -> [B*q_h*q_w, H]."""
    B, S, H = hidden.shape
    _chk(hidden, "hidden")
    lat = torch.empty((B * q_h * q_w, H), dtype=torch.bfloat16, device=hidden.device)
    check(_lib.load().cb_span_gather_hw(ptr(hidden), ptr(lat), B, S, H, start, q_h, q_w, stream()), "cb_span_gather_hw")
    return lat


def span_scatter_hw_(hidden, lat, start: int, q_h: int, q_w: int):
    B, S, H = hidden.shape
    _chk(hidden, "hidden")
    _chk(lat, "lat")
    if lat.numel() != B * q_h * q_w * H:
        raise ValueError("span_scatter_hw_: lat has the wrong number of rows")
    check(_lib.load().cb_span_scatter_hw(ptr(hidden), ptr(lat), B, S, H, start, q_h, q_w, stream()), "cb_span_scatter_hw")
    return hidden


def window_gather(feat, q_side: int, crop=None):
    """feat [B, (q r)^2, C] (natural row-major grid) -> [B*h*w, r*r, C] windows of the query rows/cols in
    crop = (y0, y1, x0, x1) (default: the whole q x q grid) — cambrian_arch.py:271-330."""
    _chk(feat, "feat")
    B, N, Cc = feat.shape
    side = int(round(N ** 0.5))
    if side * side != N or side % q_side != 0:
        raise AssertionError("window_gather: token grid is not a square multiple of the query grid")   # :277
    r = side // q_side
    y0, y1, x0, x1 = crop if crop is not None else (0, q_side, 0, q_side)
    out = torch.empty((B * (y1 - y0) * (x1 - x0), r * r, Cc), dtype=torch.bfloat16, device=feat.device)
    check(_lib.load().cb_window_gather(ptr(feat), ptr(out), B, q_side, r, Cc, y0, y1, x0, x1, stream()), "cb_window_gather")
    return out


def embed_splice_ragged(embed_w, img, newline, src, batch: int, max_len: int):
    """src: int32 [batch*max_len] row map (>=0 token id, -1 zeros, INT32_MIN newline, <=-2 image row -2-src)."""
    _chk(embed_w, "embed_w")
    H = embed_w.shape[1]
    if src.dtype != torch.int32 or src.numel() != batch * max_len or not src.is_contiguous():
        raise ValueError("embed_splice_ragged: src must be contiguous int32 [batch*max_len]")
    if img is not None:
        _chk(img, "img")
    if newline is not None:
        _chk(newline, "newline")
    out = torch.empty((batch, max_len, H), dtype=torch.bfloat16, device=embed_w.device)
    check(_lib.load().cb_embed_splice_ragged(ptr(out), ptr(embed_w), ptr(img) if img is not None else None,
                                             ptr(newline) if newline is not None else None, ptr(src), batch * max_len, H,
                                             stream()), "cb_embed_splice_ragged")
    return out


def resample_coeffs(in_size: int, out_size: int):
    """Host-side Pillow-compatible bicubic coefficient tables: (bounds int32 [out, 2], kk int32 [out, ksize])."""
    lib = _lib.load()
    ks = lib.cb_resample_ksize(in_size, out_size)
    bounds = torch.empty((out_size, 2), dtype=torch.int32)
    kk = torch.empty((out_size, ks), dtype=torch.int32)
    check(lib.cb_resample_coeffs(in_size, out_size, bounds.data_ptr(), kk.data_ptr()), "cb_resample_coeffs")
    return bounds, kk


def preprocess_image(img_u8, size: int, pad_rgb, mean, std, return_u8: bool = False):
    """img_u8: CUDA uint8 [H, W, 3] RGB -> bf16 [3, size, size] = normalise(resize(expand2square(img))) with Pillow's
    exact uint8 bicubic arithmetic (mm_utils.py:186-201).  Optionally also returns the resized uint8 image."""
    if not img_u8.is_cuda or img_u8.dtype != torch.uint8 or img_u8.dim() != 3 or img_u8.shape[2] != 3:
        raise ValueError("preprocess_image: expected a CUDA uint8 [H, W, 3] tensor")
    img_u8 = img_u8.contiguous()
    H, W = int(img_u8.shape[0]), int(img_u8.shape[1])
    lib = _lib.load()
    nbytes = lib.cb_preprocess_workspace_bytes(H, W, size)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=img_u8.device)
    out = torch.empty((3, size, size), dtype=torch.bfloat16, device=img_u8.device)
    u8 = torch.empty((size, size, 3), dtype=torch.uint8, device=img_u8.device) if return_u8 else None
    pad = (ctypes.c_int32 * 3)(*[int(v) for v in pad_rgb])
    m = (ctypes.c_float * 3)(*[float(v) for v in mean])
    sd = (ctypes.c_float * 3)(*[float(v) for v in std])
    check(lib.cb_preprocess_image(ptr(img_u8), H, W, size, ctypes.addressof(pad), ctypes.addressof(m), ctypes.addressof(sd),
                                  ptr(out), ptr(u8), ptr(ws), nbytes, stream()), "cb_preprocess_image")
    return (out, u8) if return_u8 else out


def gemm_swiglu(x2d, w_gu, gu_out=None, act_out=None):
    """(gu, act) = fused gate/up projection + SwiGLU: gu = x @ [gate; up]^T [M, 2F], act = silu(gu[:, :F]) * gu[:, F:]."""
    _require_cuda_bf16(x2d, w_gu)
    M, K = x2d.shape
    F2 = w_gu.shape[0]
    if F2 % 256 or x2d.stride(1) != 1 or w_gu.stride(1) != 1:
        raise ValueError("gemm_swiglu: need contiguous rows and F % 128 == 0")
    F = F2 // 2
    gu = gu_out if gu_out is not None else torch.empty((M, F2), dtype=torch.bfloat16, device=x2d.device)
    act = act_out if act_out is not None else torch.empty((M, F), dtype=torch.bfloat16, device=x2d.device)
    check(_lib.load().cb_gemm_swiglu_bf16(ptr(x2d), ptr(w_gu), ptr(gu), ptr(act), M, F, K, x2d.stride(0), w_gu.stride(0),
                                          gu.stride(0), act.stride(0), stream()), "cb_gemm_swiglu_bf16")
    return gu, act


# CB_FUSED_SWIGLU=0 runs GEMM + the stand-alone SwiGLU kernel instead (an A/B switch; both are CUDA paths)
_FUSED_SWIGLU = os.environ.get("CB_FUSED_SWIGLU", "1") != "0"


def mlp_gate_up(h2d, w_gu):
    """gate/up projection + SwiGLU: the fused kernel (128-row x 128-feature tiles) when the [M, 2F] output holds at least
    3 x SMs blocks of 128 x 128 and F % 128 == 0, otherwise GEMM (whose tile width adapts to small problems) followed by
    the SwiGLU kernel."""
    M = h2d.shape[0]
    F2 = w_gu.shape[0]
    I = F2 // 2
    sms = max(_lib.load().cb_sm_count(), 1)
    if (_FUSED_SWIGLU and F2 % 256 == 0 and ((M + 127) // 128) * (F2 // 128) >= 3 * sms and h2d.is_contiguous()
            and w_gu.is_contiguous()):
        return gemm_swiglu(h2d, w_gu)
    gu = gemm(h2d, w_gu)
    return gu, swiglu_fwd(gu[:, :I], gu[:, I:])


# ------------------------------------------------------------------------------------------------
# NF4 decoder weights (load_4bit; the format lives in quant.py)
# ------------------------------------------------------------------------------------------------
def nf4_quantize(w, workspace, packed, qabsmax, absmax2, offset):
    """Quantise one contiguous bf16 [N, K] weight into caller-allocated NF4 buffers (workspace: fp32, >= N*K/64)."""
    _chk(w, "w")
    N, K = w.shape
    check(_lib.load().cb_nf4_quantize(ptr(w), N, K, ptr(workspace), workspace.numel(), ptr(packed), ptr(qabsmax),
                                      ptr(absmax2), ptr(offset), stream()), "cb_nf4_quantize")


def _nf4_segments(qw):
    row0, packed, qabsmax, absmax2, offset = qw.segment_arrays()
    return len(row0), int_array(row0), ptr_array(packed), ptr_array(qabsmax), ptr_array(absmax2), ptr_array(offset)


def gemv_nf4(x, qw, bias=None, residual=None, out=None, out_dtype=torch.bfloat16) -> torch.Tensor:
    """y[M, N] = x[M, K] @ W~^T (+ bias) (+ residual) for M <= 8 on an NF4 projection (quant.NF4Projection)."""
    _require_cuda_bf16(x, bias, residual)
    M = x.shape[0]
    if out is None:
        out = torch.empty((M, qw.N), dtype=out_dtype, device=x.device)
    if out.dtype not in (torch.bfloat16, torch.float32) or out.stride(-1) != 1 or out.shape != (M, qw.N):
        raise ValueError("gemv_nf4: out must be a bf16 / fp32 [M, N] tensor with contiguous rows")
    if residual is not None and (residual.shape != out.shape or residual.stride(-1) != 1):
        raise ValueError("gemv_nf4: residual must match the output shape")
    if x.shape[1] != qw.K or x.stride(1) != 1:
        raise ValueError(f"gemv_nf4: x {tuple(x.shape)} does not match K = {qw.K}")
    check(_lib.load().cb_gemv_nf4(ptr(x), ptr(out), M, qw.N, qw.K, x.stride(0), out.stride(0), *_nf4_segments(qw),
                                  ptr(bias), ptr(residual), residual.stride(0) if residual is not None else 0,
                                  int(out.dtype == torch.float32), stream()), "cb_gemv_nf4")
    return out


def nf4_dequant(qw) -> torch.Tensor:
    """W~ [N, K] bf16 of an NF4 projection, written into (a view of) its model-owned scratch buffer."""
    out = qw.scratch[: qw.N * qw.K].view(qw.N, qw.K)
    check(_lib.load().cb_nf4_dequant(ptr(out), qw.N, qw.K, *_nf4_segments(qw), stream()), "cb_nf4_dequant")
    return out


def nf4_linear(x, qw, residual=None, out=None, out_dtype=torch.bfloat16) -> torch.Tensor:
    """y = x @ W~^T (+ residual) on an NF4 projection: the NF4 GEMV for M <= 8 rows (decode), otherwise W~ is
    dequantised into the model's scratch buffer and the bf16 GEMM runs on it (prefill, batches above 8)."""
    if x.shape[0] <= 8:
        return gemv_nf4(x, qw, residual=residual, out=out, out_dtype=out_dtype)
    return gemm(x, nf4_dequant(qw), residual=residual, out=out, out_dtype=out_dtype)


def nf4_mlp_gate_up(h2d, qw):
    """`mlp_gate_up` on the fused NF4 gate|up projection: (gu [M, 2F], act = silu(gate) * up)."""
    if h2d.shape[0] <= 8:
        gu = gemv_nf4(h2d, qw)
        I = qw.N // 2
        return gu, swiglu_fwd(gu[:, :I], gu[:, I:])
    return mlp_gate_up(h2d, nf4_dequant(qw))


# ------------------------------------------------------------------------------------------------
# LLM.int8 decoder weights (load_8bit; the format and the epilogue order live in quant_int8.py)
# ------------------------------------------------------------------------------------------------
def int8_quantize_weight(w, cb, scb):
    """Quantise one bf16 [N, K] weight (contiguous rows) into caller-allocated cb int8 [N, K] and scb fp32 [N]."""
    _require_cuda_bf16(w)
    N, K = w.shape
    if w.stride(1) != 1 or cb.shape != (N, K) or not cb.is_contiguous() or scb.shape != (N,) or scb.dtype != torch.float32:
        raise ValueError("int8_quantize_weight: need w [N, K] with contiguous rows, cb int8 [N, K], scb fp32 [N]")
    check(_lib.load().cb_int8_quantize_weight(ptr(w), N, K, w.stride(0), ptr(cb), ptr(scb), stream()),
          "cb_int8_quantize_weight")


def int8_quantize_act(x, threshold: float):
    """x [M, K] bf16 -> (xq int8 [M, K], sca fp32 [M], outlier_idx int32 [K] (first n_outlier used, ascending),
    n_outlier int32 [1]); all on the device, no host sync."""
    _require_cuda_bf16(x)
    M, K = x.shape
    if x.stride(1) != 1:
        raise ValueError("int8_quantize_act: x must have contiguous rows")
    dev = x.device
    xq = torch.empty((M, K), dtype=torch.int8, device=dev)
    sca = torch.empty(M, dtype=torch.float32, device=dev)
    colmax = torch.empty(K, dtype=torch.int32, device=dev)
    idx = torch.empty(K, dtype=torch.int32, device=dev)
    cnt = torch.empty(1, dtype=torch.int32, device=dev)
    check(_lib.load().cb_int8_quantize_act(ptr(x), M, K, x.stride(0), float(threshold), ptr(xq), ptr(sca), ptr(colmax),
                                           ptr(idx), ptr(cnt), stream()), "cb_int8_quantize_act")
    return xq, sca, idx, cnt


def _int8_matmul(entry, x, qa, qw, bias, residual, out, out_dtype):
    _require_cuda_bf16(x, bias, residual)
    xq, sca, idx, cnt = qa
    M, K = xq.shape
    N = qw.N
    if K != qw.K or x.shape != (M, K) or x.stride(1) != 1:
        raise ValueError(f"{entry}: activation {tuple(x.shape)} does not match K = {qw.K}")
    if out is None:
        out = torch.empty((M, N), dtype=out_dtype, device=x.device)
    if out.dtype not in (torch.bfloat16, torch.float32) or out.stride(-1) != 1 or out.shape != (M, N):
        raise ValueError(f"{entry}: out must be a bf16 / fp32 [M, N] tensor with contiguous rows")
    if residual is not None and (residual.shape != out.shape or residual.stride(-1) != 1):
        raise ValueError(f"{entry}: residual must match the output shape")
    check(getattr(_lib.load(), entry)(ptr(xq), ptr(qw.w.cb), ptr(sca), ptr(qw.w.scb), ptr(x), x.stride(0), ptr(idx),
                                      ptr(cnt), ptr(out), M, N, K, out.stride(0), ptr(bias), ptr(residual),
                                      residual.stride(0) if residual is not None else 0, int(out.dtype == torch.float32),
                                      stream()), entry)
    return out


def gemv_int8(x, qa, qw, bias=None, residual=None, out=None, out_dtype=torch.bfloat16) -> torch.Tensor:
    """y[M, N] for M <= 8 rows (decode) from x, its quantisation qa = int8_quantize_act(x) and an Int8Projection."""
    return _int8_matmul("cb_gemv_int8", x, qa, qw, bias, residual, out, out_dtype)


def gemm_int8(x, qa, qw, bias=None, residual=None, out=None, out_dtype=torch.bfloat16) -> torch.Tensor:
    """The same product on the int8 tensor cores, any M (prefill, batches above 8 rows)."""
    return _int8_matmul("cb_gemm_int8", x, qa, qw, bias, residual, out, out_dtype)


def int8_linear(x, qw, residual=None, out=None, out_dtype=torch.bfloat16) -> torch.Tensor:
    """y = x @ W^T (+ residual) on an int8 projection (quant_int8.Int8Projection): the activation is quantised with the
    projection's outlier threshold, then M <= 8 rows run the dp4a GEMV and larger M the int8 tensor-core GEMM."""
    qa = int8_quantize_act(x, qw.threshold)
    if x.shape[0] <= 8:
        return gemv_int8(x, qa, qw, residual=residual, out=out, out_dtype=out_dtype)
    return gemm_int8(x, qa, qw, residual=residual, out=out, out_dtype=out_dtype)


def int8_mlp_gate_up(h2d, qw):
    """`mlp_gate_up` on the stacked int8 gate|up projection: (gu [M, 2F], act = silu(gate) * up)."""
    gu = int8_linear(h2d, qw)
    I = qw.N // 2
    return gu, swiglu_fwd(gu[:, :I], gu[:, I:])


# ------------------------------------------------------------------------------------------------
# FP8 E4M3 decoder weights (load_fp8; the format and the epilogue order live in quant_fp8.py)
# ------------------------------------------------------------------------------------------------
def fp8_quantize_weight(w, wq, sw):
    """Quantise one bf16 [N, K] weight (contiguous rows) into caller-allocated wq float8_e4m3fn [N, K] and sw fp32 [N]."""
    _require_cuda_bf16(w)
    N, K = w.shape
    if (w.stride(1) != 1 or wq.shape != (N, K) or not wq.is_contiguous() or wq.dtype != torch.float8_e4m3fn
            or sw.shape != (N,) or sw.dtype != torch.float32):
        raise ValueError("fp8_quantize_weight: need w [N, K] with contiguous rows, wq float8_e4m3fn [N, K], sw fp32 [N]")
    check(_lib.load().cb_fp8_quantize_weight(ptr(w), N, K, w.stride(0), ptr(wq), ptr(sw), stream()),
          "cb_fp8_quantize_weight")


def fp8_quantize_act(x):
    """x [M, K] bf16 -> (xq float8_e4m3fn [M, K], sa fp32 [M]) on the device, no host sync."""
    _require_cuda_bf16(x)
    M, K = x.shape
    if x.stride(1) != 1:
        raise ValueError("fp8_quantize_act: x must have contiguous rows")
    xq = torch.empty((M, K), dtype=torch.float8_e4m3fn, device=x.device)
    sa = torch.empty(M, dtype=torch.float32, device=x.device)
    check(_lib.load().cb_fp8_quantize_act(ptr(x), M, K, x.stride(0), ptr(xq), ptr(sa), stream()), "cb_fp8_quantize_act")
    return xq, sa


def _fp8_matmul(entry, qa, qw, bias, residual, out, out_dtype):
    _require_cuda_bf16(bias, residual)
    xq, sa = qa
    M, K = xq.shape
    N = qw.N
    if K != qw.K or xq.dtype != torch.float8_e4m3fn or not xq.is_contiguous() or sa.shape != (M,):
        raise ValueError(f"{entry}: quantised activation {tuple(xq.shape)} does not match K = {qw.K}")
    if out is None:
        out = torch.empty((M, N), dtype=out_dtype, device=xq.device)
    if out.dtype not in (torch.bfloat16, torch.float32) or out.stride(-1) != 1 or out.shape != (M, N):
        raise ValueError(f"{entry}: out must be a bf16 / fp32 [M, N] tensor with contiguous rows")
    if residual is not None and (residual.shape != out.shape or residual.stride(-1) != 1):
        raise ValueError(f"{entry}: residual must match the output shape")
    check(getattr(_lib.load(), entry)(ptr(xq), ptr(qw.w.wq), ptr(sa), ptr(qw.w.sw), ptr(out), M, N, K, out.stride(0),
                                      ptr(bias), ptr(residual), residual.stride(0) if residual is not None else 0,
                                      int(out.dtype == torch.float32), stream()), entry)
    return out


def gemv_fp8(qa, qw, bias=None, residual=None, out=None, out_dtype=torch.bfloat16) -> torch.Tensor:
    """y[M, N] for M <= 8 rows (decode) from qa = fp8_quantize_act(x) and an Fp8Projection: wgmma with W as A."""
    return _fp8_matmul("cb_gemv_fp8", qa, qw, bias, residual, out, out_dtype)


def gemm_fp8(qa, qw, bias=None, residual=None, out=None, out_dtype=torch.bfloat16) -> torch.Tensor:
    """The same product on the FP8 tensor-core GEMM, any M (prefill, batches above 8 rows)."""
    return _fp8_matmul("cb_gemm_fp8", qa, qw, bias, residual, out, out_dtype)


def fp8_linear(x, qw, residual=None, out=None, out_dtype=torch.bfloat16) -> torch.Tensor:
    """y = x @ W^T (+ residual) on an FP8 projection (quant_fp8.Fp8Projection): the activation is quantised per row,
    then M <= 8 rows run the GEMV and larger M the GEMM."""
    qa = fp8_quantize_act(x)
    if x.shape[0] <= 8:
        return gemv_fp8(qa, qw, residual=residual, out=out, out_dtype=out_dtype)
    return gemm_fp8(qa, qw, residual=residual, out=out, out_dtype=out_dtype)


def fp8_mlp_gate_up(h2d, qw):
    """`mlp_gate_up` on the stacked FP8 gate|up projection: (gu [M, 2F], act = silu(gate) * up)."""
    gu = fp8_linear(h2d, qw)
    I = qw.N // 2
    return gu, swiglu_fwd(gu[:, :I], gu[:, I:])


# ------------------------------------------------------------------------------------------------
# FP8 E4M3 training of the decoder projections (fp8_training; the format lives in train_fp8.py)
# ------------------------------------------------------------------------------------------------
def fp8_quantize_weight_t(w, wtq, st):
    """Quantise the transpose of one bf16 [N, K] weight (contiguous rows, any row stride) into caller-allocated
    wtq float8_e4m3fn [K, N] and st fp32 [K]: bit for bit fp8_quantize_weight(w.t().contiguous())."""
    _require_cuda_bf16(w)
    N, K = w.shape
    if (w.stride(1) != 1 or wtq.shape != (K, N) or not wtq.is_contiguous() or wtq.dtype != torch.float8_e4m3fn
            or st.shape != (K,) or st.dtype != torch.float32):
        raise ValueError("fp8_quantize_weight_t: need w [N, K] with contiguous rows, wtq float8_e4m3fn [K, N], st fp32 [K]")
    lib = _lib.load()
    ws = workspace(max(int(lib.cb_fp8_quantize_weight_t_workspace_floats(N, K)), 1), w.device)
    check(lib.cb_fp8_quantize_weight_t(ptr(w), N, K, w.stride(0), ptr(wtq), ptr(st), ptr(ws), ws.numel(), stream()),
          "cb_fp8_quantize_weight_t")


def rmsnorm_fwd_fp8(x, gamma, eps: float = 1e-6, hf_cast: bool = False):
    """rmsnorm_fwd with an E4M3 output: x [rows, C] -> ((xq float8_e4m3fn [rows, C], sa fp32 [rows]), rstd fp32 [rows]),
    bit for bit fp8_quantize_act(rmsnorm_fwd(x)) and rmsnorm_fwd's rstd; the bf16 y is not written."""
    _require_cuda_bf16(x, gamma)
    C_ = x.shape[-1]
    if not x.is_contiguous() or gamma.shape != (C_,):
        raise ValueError("rmsnorm_fwd_fp8: x must be contiguous and gamma [C]")
    x2 = x.reshape(-1, C_)
    rows = x2.shape[0]
    xq = torch.empty((rows, C_), dtype=torch.float8_e4m3fn, device=x.device)
    sa = torch.empty(rows, dtype=torch.float32, device=x.device)
    rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
    check(_lib.load().cb_rmsnorm_fwd_fp8(ptr(x2), ptr(gamma), ptr(xq), ptr(sa), ptr(rstd), rows, C_, float(eps),
                                         int(hf_cast), stream()), "cb_rmsnorm_fwd_fp8")
    return (xq, sa), rstd


def swiglu_bwd_fp8(dout, gate, up, dgate, dup):
    """swiglu_bwd (dgate / dup written as swiglu_bwd writes them) plus the E4M3 rows of [dgate | dup]: returns
    (dguq float8_e4m3fn [rows, 2I], sdgu fp32 [rows]), bit for bit fp8_quantize_act of the bf16 [rows, 2I] gradient."""
    _require_cuda_bf16(dout, gate, up, dgate, dup)
    rows, I = gate.shape
    if (up.shape != (rows, I) or dout.shape != (rows, I) or dgate.shape != (rows, I) or dup.shape != (rows, I)
            or gate.stride(0) != up.stride(0) or dgate.stride(0) != dup.stride(0)
            or any(t.stride(1) != 1 for t in (dout, gate, up, dgate, dup))):
        raise ValueError("swiglu_bwd_fp8: need [rows, I] views with contiguous rows, gate / up and dgate / dup each at "
                         "one common row stride")
    dguq = torch.empty((rows, 2 * I), dtype=torch.float8_e4m3fn, device=gate.device)
    sdgu = torch.empty(rows, dtype=torch.float32, device=gate.device)
    check(_lib.load().cb_swiglu_bwd_fp8(ptr(dout), ptr(gate), ptr(up), ptr(dgate), ptr(dup), ptr(dguq), ptr(sdgu), rows,
                                        I, gate.stride(0), dout.stride(0), dgate.stride(0), stream()), "cb_swiglu_bwd_fp8")
    return dguq, sdgu


# ------------------------------------------------------------------------------------------------
# Decode KV caches: the dense FP8 cache (kv_cache_dtype="fp8"; the format and the decode arithmetic live in kv_fp8.py)
# and the paged cache (serving.BatchedGenerator; the format lives in paged_kv.py)
# ------------------------------------------------------------------------------------------------
def _kv_new_rows(what, k, v, rows="B") -> int:
    """The row stride of the new K / V rows k, v [rows, S, nkv, hd] an append reads in place, after checking them;
    `rows` names the first dimension in the error message."""
    _require_cuda_bf16(k, v)
    B, S, nkv, hd = k.shape
    # the row stride: a size-1 dimension's stride says nothing, so one token per sequence takes it from the batch stride
    ld = k.stride(1) if S > 1 else (k.stride(0) if B > 1 else nkv * hd)
    if (v.shape != k.shape or v.stride() != k.stride() or k.stride(3) != 1 or (nkv > 1 and k.stride(2) != hd)
            or (B > 1 and k.stride(0) != S * ld)):
        raise ValueError(f"{what}: k, v must be [{rows}, S, nkv, hd] rows at one common stride, got {k.stride()}")
    return ld


def kv_fp8_append(k, v, kq, vq, ks, vs, offset: int = 0, offset_dev=None):
    """Quantise the new rows k, v [B, S, nkv, hd] (views of the packed post-RoPE qkv rows, read in place) into one
    layer's FP8 cache kq, vq [B, S_max, nkv, hd] float8_e4m3fn, ks, vs [B, S_max, nkv] fp32 at positions offset + s
    (+ offset_dev[0], a device int64, for the graph-replayed step)."""
    ld = _kv_new_rows("kv_fp8_append", k, v)
    B, S, nkv, hd = k.shape
    S_max = kq.shape[1]
    if (kq.shape != (B, S_max, nkv, hd) or vq.shape != kq.shape or kq.dtype != torch.float8_e4m3fn
            or vq.dtype != kq.dtype or ks.shape != (B, S_max, nkv) or vs.shape != ks.shape or ks.dtype != torch.float32
            or vs.dtype != torch.float32 or not all(t.is_contiguous() for t in (kq, vq, ks, vs))):
        raise ValueError("kv_fp8_append: cache buffers must be contiguous kq, vq float8_e4m3fn [B, S_max, nkv, hd] and "
                         "ks, vs fp32 [B, S_max, nkv]")
    if offset_dev is not None and (offset_dev.dtype != torch.int64 or offset_dev.numel() != 1):
        raise ValueError("kv_fp8_append: offset_dev must be one device int64")
    check(_lib.load().cb_kv_fp8_append(ptr(k), ptr(v), ld, ptr(kq), ptr(vq), ptr(ks), ptr(vs), B, S, S_max, nkv,
                                       hd, int(offset), ptr(offset_dev), stream()), "cb_kv_fp8_append")


def attn_decode_fp8_workspace(B: int, nh: int, nkv: int, S_max: int, hd: int, device) -> torch.Tensor:
    """The fp32 workspace `attn_decode_fp8` needs for this shape on `device` (at least one element)."""
    with torch.cuda.device(device):
        n = _lib.load().cb_attn_decode_fp8_workspace_floats(B, nh, nkv, S_max, hd)
    return torch.empty(max(int(n), 1), dtype=torch.float32, device=device)


def attn_decode_fp8(q, kq, vq, ks, vs, workspace, *, length: int, length_dev=None, kmask=None,
                    scale: float | None = None):
    """Decode attention over one layer's FP8 cache: q [B, 1, nh, hd] (a view of the packed qkv row) -> o [B, 1, nh, hd]
    bf16.  Valid keys: positions below length (+ length_dev[0]), with kmask [B, >= those positions] set."""
    _require_cuda_bf16(q)
    B, Sq, nh, hd = q.shape
    S_max, nkv = kq.shape[1], kq.shape[2]
    if scale is None:
        scale = hd ** -0.5
    qb, _ = _bshd_strides(q, hd)
    if (kq.dtype != torch.float8_e4m3fn or vq.dtype != kq.dtype or ks.dtype != torch.float32 or vs.dtype != torch.float32
            or kq.shape != (B, S_max, nkv, hd) or vq.shape != kq.shape or ks.shape != (B, S_max, nkv)
            or vs.shape != ks.shape or not all(t.is_contiguous() for t in (kq, vq, ks, vs))):
        raise ValueError("attn_decode_fp8: cache buffers must be contiguous kq, vq float8_e4m3fn [B, S_max, nkv, hd] and "
                         "ks, vs fp32 [B, S_max, nkv]")
    if workspace.dtype != torch.float32:
        raise ValueError("attn_decode_fp8: the workspace must be fp32")
    if length_dev is not None and (length_dev.dtype != torch.int64 or length_dev.numel() != 1):
        raise ValueError("attn_decode_fp8: length_dev must be one device int64")
    km, km_ld = None, 0
    if kmask is not None:
        if kmask.dim() != 2 or kmask.shape[0] != B or kmask.stride(1) != 1:
            raise ValueError("attn_decode_fp8: kmask must be [B, positions] with contiguous rows")
        km = kmask.view(torch.uint8) if kmask.dtype == torch.bool else kmask.to(torch.uint8)
        km_ld = km.stride(0) if B > 1 else km.shape[1]
    o = torch.empty((B, Sq, nh, hd), dtype=torch.bfloat16, device=q.device)
    check(_lib.load().cb_attn_decode_fp8(ptr(q), qb, ptr(kq), ptr(vq), ptr(ks), ptr(vs), ptr(km), km_ld, ptr(o),
                                         ptr(workspace), workspace.numel(), B, Sq, nh, nkv, S_max, hd, int(length),
                                         ptr(length_dev), float(scale), stream()), "cb_attn_decode_fp8")
    return o


def _paged_pages(what, kp, vp, ksc, vsc, hd=None):
    """(fp8, num_pages, page_size, nkv, hd) of one layer's pages, after checking dtypes and shapes."""
    if kp.dim() != 4 or vp.shape != kp.shape or vp.dtype != kp.dtype or not (kp.is_contiguous() and vp.is_contiguous()):
        raise ValueError(f"{what}: k / v pages must be contiguous [num_pages, page_size, nkv, hd] of one dtype")
    fp8 = kp.dtype == torch.float8_e4m3fn
    if not fp8 and kp.dtype != torch.bfloat16:
        raise ValueError(f"{what}: pages must be bf16 or float8_e4m3fn, not {kp.dtype}")
    if fp8 and (ksc is None or vsc is None or ksc.shape != kp.shape[:3] or vsc.shape != ksc.shape
                or ksc.dtype != torch.float32 or vsc.dtype != torch.float32
                or not (ksc.is_contiguous() and vsc.is_contiguous())):
        raise ValueError(f"{what}: FP8 pages need contiguous fp32 scales [num_pages, page_size, nkv]")
    if not fp8 and (ksc is not None or vsc is not None):
        raise ValueError(f"{what}: bf16 pages take no scales")
    num_pages, page_size, nkv, phd = kp.shape
    if hd is not None and phd != hd:
        raise ValueError(f"{what}: pages hold head_dim {phd}, the rows {hd}")
    return int(fp8), num_pages, page_size, nkv, phd


def _paged_table(what, table, lens, rows, need_lens):
    if table.dim() != 2 or table.dtype != torch.int32 or table.shape[0] != rows or table.stride(1) != 1:
        raise ValueError(f"{what}: block_table must be int32 [rows={rows}, max_pages] with contiguous rows")
    if lens is None:
        if need_lens:
            raise ValueError(f"{what}: lens is required")
    elif lens.dtype != torch.int32 or lens.shape != (rows,) or not lens.is_contiguous():
        raise ValueError(f"{what}: lens must be a contiguous int32 [rows={rows}]")
    return table.shape[1], (table.stride(0) if rows > 1 else table.shape[1])


def paged_kv_append(k, v, k_pages, v_pages, k_scales, v_scales, block_table, lens=None, offset: int = 0,
                    offset_from_lens: bool = False):
    """Write the new rows k, v [rows, S, nkv, hd] (views of the packed post-RoPE qkv rows, read in place) into one
    layer's pages at positions offset (+ lens[b] with offset_from_lens) + s through block_table; a row with lens[b] < 0
    writes nothing."""
    ld = _kv_new_rows("paged_kv_append", k, v, "rows")
    B, S, nkv, hd = k.shape
    fp8, num_pages, page_size, pnkv, _ = _paged_pages("paged_kv_append", k_pages, v_pages, k_scales, v_scales, hd)
    if pnkv != nkv:
        raise ValueError(f"paged_kv_append: pages hold {pnkv} kv heads, the rows {nkv}")
    max_pages, tld = _paged_table("paged_kv_append", block_table, lens, B, offset_from_lens)
    check(_lib.load().cb_paged_kv_append(ptr(k), ptr(v), ld, ptr(k_pages), ptr(v_pages), ptr(k_scales), ptr(v_scales),
                                         fp8, ptr(block_table), tld, ptr(lens), B, S, nkv, hd, page_size, num_pages,
                                         max_pages, int(offset), int(bool(offset_from_lens)), stream()),
          "cb_paged_kv_append")


def attn_decode_paged_workspace(rows: int, nh: int, max_pages: int, page_size: int, hd: int, device) -> torch.Tensor:
    """The fp32 workspace `attn_decode_paged` needs for up to `rows` rows (at least one element)."""
    n = _lib.load().cb_attn_decode_paged_workspace_floats(rows, nh, max_pages, page_size, hd)
    return torch.empty(max(int(n), 1), dtype=torch.float32, device=device)


def attn_decode_paged(q, k_pages, v_pages, k_scales, v_scales, block_table, lens, workspace, *, len_add: int = 1,
                      scale: float | None = None):
    """Decode attention over one layer's pages: q [rows, 1, nh, hd] (a view of the packed qkv row) -> o [rows, 1, nh, hd]
    bf16.  Row b attends over its positions below lens[b] + len_add; a row with lens[b] < 0 gets zeros."""
    _require_cuda_bf16(q)
    B, Sq, nh, hd = q.shape
    if Sq != 1:
        raise ValueError(f"attn_decode_paged: Sq={Sq}; the paged decode kernel takes one query per row")
    if scale is None:
        scale = hd ** -0.5
    qb, _ = _bshd_strides(q, hd)
    fp8, num_pages, page_size, nkv, _ = _paged_pages("attn_decode_paged", k_pages, v_pages, k_scales, v_scales, hd)
    max_pages, tld = _paged_table("attn_decode_paged", block_table, lens, B, True)
    if workspace.dtype != torch.float32:
        raise ValueError("attn_decode_paged: the workspace must be fp32")
    o = torch.empty((B, 1, nh, hd), dtype=torch.bfloat16, device=q.device)
    check(_lib.load().cb_attn_decode_paged(ptr(q), qb, ptr(k_pages), ptr(v_pages), ptr(k_scales), ptr(v_scales), fp8,
                                           ptr(block_table), tld, ptr(lens), int(len_add), ptr(o), ptr(workspace),
                                           workspace.numel(), B, nh, nkv, hd, page_size, num_pages, max_pages,
                                           float(scale), stream()), "cb_attn_decode_paged")
    return o


def paged_kv_gather(k_pages, v_pages, k_scales, v_scales, block_table_row, P: int, out_k, out_v):
    """Positions [0, P) of one block-table row (int32 [max_pages]) out of one layer's pages into out_k, out_v
    [>= P, nkv, hd] bf16 (row stride >= nkv * hd, e.g. the head of a [1, P + n, nkv, hd] buffer): bf16 pages are copied,
    FP8 pages dequantised to bf16(float(e4m3) * scale), one rounding per element."""
    fp8, num_pages, page_size, nkv, hd = _paged_pages("paged_kv_gather", k_pages, v_pages, k_scales, v_scales)
    if block_table_row.dim() != 1 or block_table_row.dtype != torch.int32 or not block_table_row.is_contiguous():
        raise ValueError("paged_kv_gather: block_table_row must be a contiguous int32 [max_pages]")
    _require_cuda_bf16(out_k, out_v)
    if out_k.dim() == 4 and out_k.shape[0] == 1 and out_v.dim() == 4:      # [1, P + n, nkv, hd] buffers
        out_k, out_v = out_k[0], out_v[0]
    if (out_k.dim() != 3 or out_k.shape[1:] != (nkv, hd) or out_v.shape != out_k.shape or out_v.stride() != out_k.stride()
            or out_k.shape[0] < P or out_k.stride(2) != 1 or out_k.stride(1) != hd):
        raise ValueError(f"paged_kv_gather: out_k, out_v must be [>= {P}, {nkv}, {hd}] bf16 at one common row stride")
    ld = out_k.stride(0) if out_k.shape[0] > 1 else nkv * hd
    check(_lib.load().cb_paged_kv_gather(ptr(k_pages), ptr(v_pages), ptr(k_scales), ptr(v_scales), fp8,
                                         ptr(block_table_row), nkv, hd, page_size, num_pages, block_table_row.shape[0],
                                         int(P), ptr(out_k), ptr(out_v), ld, stream()), "cb_paged_kv_gather")


def sample_tokens_workspace(rows: int, V: int, device) -> torch.Tensor:
    """The fp32 workspace `sample_tokens` needs for up to `rows` rows of V logits (at least one element)."""
    n = _lib.load().cb_sample_tokens_workspace_floats(int(rows), int(V))
    return torch.empty(max(int(n), 1), dtype=torch.float32, device=device)


def sample_tokens(logits, temperature, top_k, top_p, seed, step, out=None, workspace=None):
    """One sampled token per row of fp32 logits [rows, V] (unit column stride, any row stride >= V) into out int64
    [rows], each row under its own temperature (fp32 [rows]), top_k (int32 [rows]; 0 or >= V: off), top_p (fp32 [rows];
    1: off), seed (int64 [rows], read as uint64) and step (int64 [rows]).  The rule is in generation.py's docstring; a
    row's token depends only on its logits, parameters, seed and step."""
    if not logits.is_cuda:
        raise _lib.CambrianB200Error("cambrian_b200 kernels need CUDA tensors (no CPU fallback)")
    if logits.dtype != torch.float32 or logits.dim() != 2 or logits.stride(1) != 1 or logits.shape[0] == 0:
        raise ValueError("sample_tokens: logits must be fp32 [rows >= 1, V] with unit column stride")
    rows, V = logits.shape
    ld = logits.stride(0) if rows > 1 else V
    for name, t, dt in (("temperature", temperature, torch.float32), ("top_k", top_k, torch.int32),
                        ("top_p", top_p, torch.float32), ("seed", seed, torch.int64), ("step", step, torch.int64)):
        if t.dtype != dt or t.shape != (rows,) or not t.is_contiguous() or t.device != logits.device:
            raise ValueError(f"sample_tokens: {name} must be a contiguous {dt} [{rows}] on {logits.device}")
    if out is None:
        out = torch.empty(rows, dtype=torch.int64, device=logits.device)
    elif out.dtype != torch.int64 or out.shape != (rows,) or not out.is_contiguous() or out.device != logits.device:
        raise ValueError(f"sample_tokens: out must be a contiguous int64 [{rows}] on {logits.device}")
    if workspace is not None and workspace.dtype != torch.float32:
        raise ValueError("sample_tokens: the workspace must be fp32")
    check(_lib.load().cb_sample_tokens(ptr(logits), ld, rows, V, ptr(temperature), ptr(top_k), ptr(top_p), ptr(seed),
                                       ptr(step), ptr(out), ptr(workspace),
                                       0 if workspace is None else workspace.numel(), stream()), "cb_sample_tokens")
    return out
