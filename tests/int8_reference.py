"""Torch reference of the LLM.int8 format and arithmetic (cambrian_b200/quant_int8.py states the definition), written
from the definition: the weight and activation quantisers, the linear with its outlier decomposition in the stated
order, and CPU stand-ins of the four int8 entry points for host-logic tests.

The integer sums are exact: int64 on the CPU; on the GPU (no integer matmul there) an fp64 matmul, which is exact as
well because every product is an integer of at most 127^2 and every partial sum stays far below 2^53."""
import torch

INV127 = torch.tensor(1.0 / 127.0, dtype=torch.float32)        # 1/127 rounded to fp32 (== fp32(1) / fp32(127))
INV16129 = torch.tensor(1.0 / 16129.0, dtype=torch.float32)    # 1/16129 rounded to fp32


def quantize_weight(w):
    """bf16 [N, K] -> (cb int8 [N, K], scb fp32 [N])."""
    wf = w.detach().float()
    scb = wf.abs().amax(1)
    s = torch.where(scb > 0, torch.tensor(127.0, device=w.device) / scb, torch.zeros_like(scb))
    cb = torch.round(wf * s[:, None]).clamp(-127, 127).to(torch.int8)
    return cb, scb


def quantize_act(x, threshold=6.0):
    """[M, K] -> (xq int8 [M, K], sca fp32 [M], ascending outlier columns int64 [n])."""
    xf = x.detach().float()
    colmax = xf.abs().amax(0)
    out = colmax >= threshold if threshold > 0 else torch.zeros_like(colmax, dtype=torch.bool)
    sca = torch.where(out[None, :], torch.zeros_like(xf), xf.abs()).amax(1)
    s = torch.where(sca > 0, torch.tensor(127.0, device=x.device) / sca, torch.zeros_like(sca))
    xq = torch.where(out[None, :], torch.zeros_like(xf), torch.round(xf * s[:, None])).to(torch.int8)
    return xq, sca, out.nonzero()[:, 0]


def int_matmul(a, b):
    """sum_k a[m, k] * b[n, k], exact, as int64."""
    if a.device.type == "cpu":
        return a.long() @ b.long().t()
    return (a.double() @ b.double().t()).long()


def linear_q(x, xq, sca, idx, cb, scb, bias=None, residual=None, out_dtype=torch.bfloat16):
    """The output of the definition from an already quantised activation; every operation a separate fp32 rounding."""
    acc = int_matmul(xq, cb)
    v = (acc.to(torch.float32) * (sca[:, None] * scb[None, :])) * INV16129.to(x.device)
    o = torch.zeros_like(v)
    wsc = scb * INV127.to(x.device)
    xf = x.detach().float()
    for j in idx.tolist():
        o = o + xf[:, j:j + 1] * (cb[:, j].float() * wsc)[None, :]
    y = v + o
    if bias is not None:
        y = y + bias.float()[None, :]
    if residual is not None:
        y = y + residual.float()
    return y.to(out_dtype)


def linear(x, cb, scb, threshold=6.0, bias=None, residual=None, out_dtype=torch.bfloat16):
    xq, sca, idx = quantize_act(x, threshold)
    return linear_q(x, xq, sca, idx, cb, scb, bias, residual, out_dtype)


# ---- CPU stand-ins of the four entry points (host-logic tests on machines without a GPU) ----
def int8_quantize_weight(w, cb, scb):
    c, s = quantize_weight(w)
    cb.copy_(c)
    scb.copy_(s)


def int8_quantize_act(x, threshold):
    xq, sca, idx = quantize_act(x, threshold)
    K = x.shape[1]
    full = torch.zeros(K, dtype=torch.int32, device=x.device)
    full[: idx.numel()] = idx.to(torch.int32)
    return xq, sca, full, torch.tensor([idx.numel()], dtype=torch.int32, device=x.device)


def _matmul(x, qa, qw, bias=None, residual=None, out=None, out_dtype=torch.bfloat16):
    xq, sca, full, cnt = qa
    idx = full[: int(cnt[0])].long()
    y = linear_q(x, xq, sca, idx, qw.w.cb, qw.w.scb, bias, residual, out_dtype if out is None else out.dtype)
    if out is not None:
        out.copy_(y)
        return out
    return y


def gemv_int8(x, qa, qw, bias=None, residual=None, out=None, out_dtype=torch.bfloat16):
    assert x.shape[0] <= 8
    return _matmul(x, qa, qw, bias, residual, out, out_dtype)


def gemm_int8(x, qa, qw, bias=None, residual=None, out=None, out_dtype=torch.bfloat16):
    return _matmul(x, qa, qw, bias, residual, out, out_dtype)


def install(monkeypatch):
    from cambrian_b200 import ops
    for n in ("int8_quantize_weight", "int8_quantize_act", "gemv_int8", "gemm_int8"):
        monkeypatch.setattr(ops, n, globals()[n])
