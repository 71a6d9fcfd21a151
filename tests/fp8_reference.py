"""Torch reference of the FP8 E4M3 format and arithmetic (cambrian_b200/quant_fp8.py states the definition), written
from the definition: E4M3 rounding from the bit layout (not torch's float8 conversion, which the tests check it
against), the row quantiser, the linear in the stated order, and CPU stand-ins of the four FP8 entry points for
host-logic tests.

The reference sums the products in fp64 (`acc64`): every product of two E4M3 values is exact, and the fp64 sum over
K <= 20480 of them is within 2^-40 of the exact one, so it stands for the exact sum the kernels approximate in fp32."""
import torch

E4M3_MAX = 448.0
FLT_MAX = torch.finfo(torch.float32).max


def e4m3_rn_satfinite(v):
    """fp32 -> the nearest E4M3 value (ties to even), |v| > 448 -> +-448, sign of zero kept; returned as fp32."""
    v = v.to(torch.float32)
    _, e = torch.frexp(v)                                  # |v| = f * 2^e, f in [0.5, 1)
    q_exp = torch.clamp(e - 1, min=-6) - 3                 # quantum: 2^(floor(log2|v|) - 3), subnormals 2^-9
    quantum = torch.ldexp(torch.ones_like(v), q_exp)
    r = torch.round(v / quantum) * quantum                 # exact scaling by a power of two, round half to even
    r = torch.where(r.abs() > E4M3_MAX, torch.sign(v) * E4M3_MAX, r)
    return torch.where(v == 0, v, r)                       # keep the sign of zero (round(-0.) is -0. as well)


def to_e4m3(v):
    """e4m3_rn_satfinite as float8_e4m3fn storage (the values above are exactly representable)."""
    return e4m3_rn_satfinite(v).to(torch.float8_e4m3fn)


def quantize_rows(x):
    """bf16 [R, K] -> (q float8_e4m3fn [R, K], s fp32 [R]), the rule of quant_fp8.py."""
    xf = x.detach().float()
    amax = xf.abs().amax(1)
    c448 = torch.full_like(amax, E4M3_MAX)                 # tensor / tensor: torch turns a division by a CUDA scalar
    s = amax / c448                                        # into a multiplication by its reciprocal
    r = torch.clamp(c448 / amax, max=FLT_MAX)              # 448 / 0 = inf -> FLT_MAX
    return to_e4m3(xf * r[:, None]), s


quantize_weight = quantize_rows
quantize_act = quantize_rows


def acc64(xq, wq):
    """sum_k float(xq[m, k]) * float(wq[n, k]) in fp64 (the exact sum to within 2^-40 relative)."""
    return xq.double() @ wq.double().t()


def epilogue(acc, sa, sw, bias=None, residual=None, out_dtype=torch.bfloat16):
    """Steps 2-5 of the output definition on an fp32 acc; every operation rounded to fp32 on its own."""
    y = acc.to(torch.float32) * (sa[:, None] * sw[None, :])
    if bias is not None:
        y = y + bias.float()[None, :]
    if residual is not None:
        y = y + residual.float()
    return y.to(out_dtype)


def linear_q(xq, sa, wq, sw, bias=None, residual=None, out_dtype=torch.bfloat16):
    """The output from already quantised operands, acc from the fp64 sum rounded once to fp32."""
    return epilogue(acc64(xq, wq).float(), sa, sw, bias, residual, out_dtype)


def linear(x, wq, sw, bias=None, residual=None, out_dtype=torch.bfloat16):
    xq, sa = quantize_act(x)
    return linear_q(xq, sa, wq, sw, bias, residual, out_dtype)


# ---- CPU stand-ins of the four entry points (host-logic tests on machines without a GPU) ----
def fp8_quantize_weight(w, wq, sw):
    q, s = quantize_weight(w)
    wq.copy_(q)
    sw.copy_(s)


def fp8_quantize_act(x):
    return quantize_act(x)


def _matmul(qa, qw, bias=None, residual=None, out=None, out_dtype=torch.bfloat16):
    xq, sa = qa
    y = linear_q(xq, sa, qw.w.wq, qw.w.sw, bias, residual, out_dtype if out is None else out.dtype)
    if out is not None:
        out.copy_(y)
        return out
    return y


def gemv_fp8(qa, qw, bias=None, residual=None, out=None, out_dtype=torch.bfloat16):
    assert qa[0].shape[0] <= 8
    return _matmul(qa, qw, bias, residual, out, out_dtype)


def gemm_fp8(qa, qw, bias=None, residual=None, out=None, out_dtype=torch.bfloat16):
    return _matmul(qa, qw, bias, residual, out, out_dtype)


def install(monkeypatch):
    from cambrian_b200 import ops
    for n in ("fp8_quantize_weight", "fp8_quantize_act", "gemv_fp8", "gemm_fp8"):
        monkeypatch.setattr(ops, n, globals()[n])
