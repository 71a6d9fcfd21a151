"""Plain-torch fp32 restatement of the 8-bit AdamW format and step (cambrian_b200/adam8bit.py states the definition),
written from the definition with its own map builder: the quantiser, the dequantiser, one step bit for bit in the
kernel's rounding order, and CPU stand-ins of `ops.adamw8` / `ops.adamw8_host` for host-logic tests.

Every rounding of the kernel is restated: products, sums, quotients and square roots are fp32 torch ops (IEEE,
round-to-nearest on the CPU), except the square root, taken in float64 and rounded once; a fused multiply-add is computed in float64 with round-to-odd, which then rounds to the
correctly rounded fp32 result; `powf` is the host's libm, as the launcher's.  The kernel's `rsqrtf(bc2)` is within 2
ulp of 1 / sqrt(bc2) but not correctly rounded: a test that compares bit for bit passes the value as `inv_sqrt_bc2`."""
import ctypes
import ctypes.util

import torch

BLOCK = 256


def dynamic_map(signed):
    """0, 1.0 and, per decade i = 0..6, 10^(i-6) times the interval means of linspace(0.1, 1, k + 1) (fp32): k = 2^i
    means and their negatives (signed), or k = 2^(i+1) means (unsigned); sorted."""
    vals = [0.0, 1.0]
    for i in range(7):
        b = torch.linspace(0.1, 1.0, (2 ** i if signed else 2 ** (i + 1)) + 1, dtype=torch.float32)
        m = (b[:-1] + b[1:]) / 2.0
        vals += (m * 10.0 ** (i - 6)).tolist()
        if signed:
            vals += (m * -(10.0 ** (i - 6))).tolist()
    return torch.tensor(sorted(vals), dtype=torch.float32)


_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.powf.restype, _libm.powf.argtypes = ctypes.c_float, [ctypes.c_float, ctypes.c_float]

SMAP, UMAP = dynamic_map(True), dynamic_map(False)
SZERO = int((SMAP == 0).nonzero())


def fma32(a, b, c):
    """fp32 fma(a, b, c), correctly rounded: a * b is exact in float64, the sum is rounded to odd, then to fp32."""
    a, b, c = torch.as_tensor(a, dtype=torch.float64), torch.as_tensor(b, dtype=torch.float64), torch.as_tensor(
        c, dtype=torch.float64)
    p = a * b
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)                      # TwoSum: s + err == p + c exactly
    even = (s.view(torch.int64) & 1) == 0
    toward = torch.where(err > 0, torch.full_like(s, float("inf")), torch.full_like(s, -float("inf")))
    s = torch.where((err != 0) & even, torch.nextafter(s, toward), s)
    return s.float()


def f32(x):
    return torch.tensor(x, dtype=torch.float32)


def quantize(x, qmap, zero_code):
    """fp32 [n] -> (codes uint8 [n], absmax fp32 [ceil(n / 256)]); the last block may be partial."""
    n = x.numel()
    nb = (n + BLOCK - 1) // BLOCK
    blk = torch.arange(n) // BLOCK
    absmax = torch.zeros(nb, dtype=torch.float32).scatter_reduce(0, blk, x.abs(), "amax", include_self=True)
    v = x * (f32(1.0) / absmax)[blk]
    idx = torch.searchsorted(qmap, v.contiguous()).clamp(max=255)
    lo = (idx - 1).clamp(min=0)
    take_hi = (idx == 0) | ((qmap[idx] - v) <= (v - qmap[lo]))
    q = torch.where(take_hi, idx, lo)
    q[absmax[blk] == 0] = zero_code
    return q.to(torch.uint8), absmax


def dequantize(codes, absmax, qmap):
    return qmap[codes.long()] * absmax[torch.arange(codes.numel()) // BLOCK]


def scalars(lr, b1, b2, eps, wd, step, grad_scale, clip_coef, inv_sqrt_bc2=None):
    """The kernel's per-launch scalars, as the host code and adamw_scalars compute them."""
    lr, b1, b2, eps, wd = (f32(x) for x in (lr, b1, b2, eps, wd))
    one = f32(1.0)
    bc1 = one - f32(_libm.powf(float(b1), float(step)))                # 1.f - powf(b1, step), the host's libm
    bc2 = one - f32(_libm.powf(float(b2), float(step)))
    gs = f32(float(clip_coef[0])) if clip_coef is not None else f32(float(grad_scale))
    if inv_sqrt_bc2 is None:
        inv_sqrt_bc2 = torch.rsqrt(bc2)
    return dict(gs=gs, lr=lr, b1=b1, b2=b2, eps=eps, wd=wd, bc1=bc1, isq=f32(float(inv_sqrt_bc2)))


def bc2(b2, step):
    """1 - powf(b2, step) in fp32, as the launcher computes it."""
    return f32(1.0) - f32(_libm.powf(float(b2), float(step)))


def adamw_elementwise(p, m, v, g16, sc):
    """adamw_kernel's arithmetic on fp32 [n] tensors (n % 8 == 0): returns the new p, m, v."""
    gg = g16.float() * sc["gs"]
    one = f32(1.0)
    m = fma32(one - sc["b1"], gg, sc["b1"] * m)
    v = fma32(gg, (one - sc["b2"]) * gg, sc["b2"] * v)
    denom = fma32(v.double().sqrt().float(), sc["isq"], sc["eps"])     # correctly rounded: torch's fp32 sqrt may not be
    step_size = sc["lr"] / sc["bc1"]
    decay = fma32(-sc["lr"], sc["wd"], one)
    q = m / denom
    pd = p * decay
    last = (torch.arange(p.numel()) % 8) == 7
    p = torch.where(last, fma32(-step_size, q, pd), pd - step_size * q)
    return p, m, v


def step(p, qm, qv, sm, sv, g16, lr, b1, b2, eps, wd, step, grad_scale=1.0, clip_coef=None, inv_sqrt_bc2=None):
    """One cb_adamw8 step on CPU tensors: returns (p, p16, qm, qv, sm, sv) and the unquantised updated (m, v)."""
    sc = scalars(lr, b1, b2, eps, wd, step, grad_scale, clip_coef, inv_sqrt_bc2)
    m = dequantize(qm, sm, SMAP)
    v = dequantize(qv, sv, UMAP)
    p, m, v = adamw_elementwise(p.float(), m, v, g16.cpu(), sc)
    qm, sm = quantize(m, SMAP, SZERO)
    qv, sv = quantize(v, UMAP, 0)
    return (p, p.to(torch.bfloat16), qm, qv, sm, sv), (m, v)


# ---- CPU stand-ins of the two entry points (host-logic tests on machines without a GPU) ----
def adamw8(p32, qm, qv, sm, sv, g16, p16, lr, beta1, beta2, eps, wd, step_, grad_scale=1.0, clip_coef=None,
           background=False):
    (p, p16n, qmn, qvn, smn, svn), _ = step(p32, qm, qv, sm, sv, g16, lr, beta1, beta2, eps, wd, step_,
                                            grad_scale=grad_scale, clip_coef=clip_coef)
    for dst, src in ((p32, p), (p16, p16n), (qm, qmn), (qv, qvn), (sm, smn), (sv, svn)):
        dst.copy_(src)


def adamw8_host(p32, qm, qv, sm, sv, g16, p16, lr, beta1, beta2, eps, wd, step_, grad_scale=1.0, clip_coef=None, ctas=0):
    assert not any(t.is_cuda for t in (p32, qm, qv, sm, sv))
    adamw8(p32, qm, qv, sm, sv, g16, p16, lr, beta1, beta2, eps, wd, step_, grad_scale=grad_scale, clip_coef=clip_coef)


def _adamw_host(p32, m, v, g16, p16, lr, beta1, beta2, eps, wd, step_, grad_scale=1.0, clip_coef=None, ctas=0):
    import ops_emulation
    assert not any(t.is_cuda for t in (p32, m, v))
    ops_emulation.adamw(p32, m, v, g16, p16, lr, beta1, beta2, eps, wd, step_, grad_scale=grad_scale, clip_coef=clip_coef)


def install(monkeypatch=None):
    """tests/ops_emulation.py's stand-ins, plus both 8-bit entry points and the fp32 offload one."""
    import ops_emulation
    ops_emulation.install(monkeypatch)
    from cambrian_b200 import ops
    setter = monkeypatch or ops_emulation._Setter
    setter.setattr(ops, "adamw8", adamw8)
    setter.setattr(ops, "adamw8_host", adamw8_host)
    setter.setattr(ops, "adamw_host", _adamw_host)
