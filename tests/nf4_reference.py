"""Torch reference of the NF4 + double-quantisation format (cambrian_b200/quant.py states the definition), written from
the definition with its own copy of both tables: the quantiser, the dequantiser W~, and CPU stand-ins of the three NF4
entry points for host-logic tests."""
import torch

NF4 = torch.tensor([-1.0, -0.6961928009986877, -0.5250730514526367, -0.39491748809814453, -0.28444138169288635,
                    -0.18477343022823334, -0.09105003625154495, 0.0, 0.07958029955625534, 0.16093020141124725,
                    0.24611230194568634, 0.33791524171829224, 0.44070982933044434, 0.5626170039176941,
                    0.7229568362236023, 1.0], dtype=torch.float32)


def signed_dynamic_map():
    """0, 1.0 and, for i = 0..6, +-10^(i-6) * m for the 2^i midpoints m of linspace(0.1, 1, 2^i + 1) (fp32), sorted."""
    vals = [0.0, 1.0]
    for i in range(7):
        b = torch.linspace(0.1, 1.0, 2 ** i + 1, dtype=torch.float32)
        m = (b[:-1] + b[1:]) / 2.0
        vals += (m * 10.0 ** (i - 6)).tolist()
        vals += (m * -(10.0 ** (i - 6))).tolist()
    return torch.tensor(sorted(vals), dtype=torch.float32)


DMAP = signed_dynamic_map()
ZERO_INDEX = int((DMAP == 0).nonzero())


def quantize(w, offset=None):
    """bf16 [N, K] -> (packed uint8 [N, K/2], qabsmax uint8 [nb], absmax2 fp32 [ng], offset fp32 [1]); `offset` may be
    given (the device's fixed-order mean) so the rest can be compared bitwise."""
    N, K = w.shape
    dev = w.device
    c, dmap = NF4.to(dev), DMAP.to(dev)
    blocks = w.detach().float().reshape(-1, 64)
    absmax = blocks.abs().amax(1)
    x = blocks * (1.0 / absmax)[:, None]
    mids = (c[:-1] + c[1:]) / 2
    codes = (mids[None, None, :] < x[..., None]).sum(-1)
    codes[absmax == 0] = 7
    codes = codes.reshape(N, K)
    packed = ((codes[:, 0::2] << 4) | codes[:, 1::2]).to(torch.uint8)
    if offset is None:
        offset = absmax.double().mean().float().reshape(1)
    offset = offset.detach().to(dev).float().reshape(1)
    nb = absmax.numel()
    g = torch.arange(nb, device=dev) // 256
    dv = absmax - offset
    ng = (nb + 255) // 256
    absmax2 = torch.zeros(ng, dtype=torch.float32, device=dev).scatter_reduce(0, g, dv.abs(), "amax", include_self=True)
    v = dv * (1.0 / absmax2[g])
    idx = torch.searchsorted(dmap, v.contiguous()).clamp(max=255)
    lo = (idx - 1).clamp(min=0)
    take_hi = (idx == 0) | ((dmap[idx] - v) <= (v - dmap[lo]))
    q = torch.where(take_hi, idx, lo)
    q[absmax2[g] == 0] = ZERO_INDEX
    return packed, q.to(torch.uint8), absmax2, offset


def dequantize(packed, qabsmax, absmax2, offset):
    """W~ (bf16 [N, K]): bf16(c[code] * (map[q] * absmax2 + offset)), every product and sum rounded on its own."""
    N = packed.shape[0]
    dev = packed.device
    p = packed.long()
    codes = torch.stack([p >> 4, p & 15], -1).reshape(N, -1)
    q = qabsmax.long()
    scale = DMAP.to(dev)[q] * absmax2[torch.arange(q.numel(), device=dev) // 256]
    scale = scale + offset
    return (NF4.to(dev)[codes].reshape(-1, 64) * scale[:, None]).reshape(N, -1).to(torch.bfloat16)


def projection_weight(qw):
    """W~ of a (possibly fused) NF4 projection: its segments' W~ stacked by rows."""
    return torch.cat([dequantize(p.packed, p.qabsmax, p.absmax2, p.offset) for p in qw.parts], 0)


# ---- CPU stand-ins of the three entry points (host-logic tests on machines without a GPU) ----
def nf4_quantize(w, workspace, packed, qabsmax, absmax2, offset):
    pk, q, a2, off = quantize(w)
    packed.copy_(pk)
    qabsmax.copy_(q)
    absmax2.copy_(a2)
    offset.copy_(off)


def gemv_nf4(x, qw, bias=None, residual=None, out=None, out_dtype=torch.bfloat16):
    assert x.shape[0] <= 8
    y = x.float() @ projection_weight(qw).float().t()
    if bias is not None:
        y = y + bias.float()
    if residual is not None:
        y = y + residual.float()
    y = y.to(out_dtype)
    if out is not None:
        out.copy_(y)
        return out
    return y


def nf4_dequant(qw):
    out = qw.scratch[: qw.N * qw.K].view(qw.N, qw.K)
    out.copy_(projection_weight(qw))
    return out


def install(monkeypatch):
    from cambrian_b200 import ops
    for n in ("nf4_quantize", "gemv_nf4", "nf4_dequant"):
        monkeypatch.setattr(ops, n, globals()[n])
