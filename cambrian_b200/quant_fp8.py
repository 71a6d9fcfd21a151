"""FP8 E4M3 decoder weights for inference (`load_fp8`).

This module is the one place on the host that knows the format and its arithmetic (the kernels in csrc/fp8.cu are the
other side).  E4M3 is `torch.float8_e4m3fn`: 1 sign, 4 exponent (bias 7), 3 mantissa bits, no infinities, largest
finite 448, smallest subnormal 2^-9.  e4m3_rn_satfinite(v) rounds an fp32 v to the nearest E4M3 value, ties to even,
and gives +-448 for |v| > 448 (PTX `cvt.rn.satfinite.e4m3x2.f32`); the sign of a zero is kept (-0 -> 0x80).

Weight W [N, K] (bf16, K % 16 == 0), quantised once at load, per row n:
  * amax = max_k |W[n, k]| (exact);
  * sw[n] = amax / 448, one fp32 division;
  * r = 448 / amax, one fp32 division, replaced by the largest finite fp32 (0x1.fffffep127) when it overflows: that is
    the zero row (448 / 0 = +inf) and a row whose amax is below about 448 * 2^-128, e.g. a row of bf16 subnormals.  For
    such a row every |W| * r stays at or below 448, so nothing saturates, and r * sw is no longer 1: the row dequantises to
    W * (amax * r / 448) (the row carries less than 2^-119 per element either way);
  * wq[n, k] = e4m3_rn_satfinite(fp32(float(W[n, k]) * r)): the product rounded to fp32, then to E4M3;
  * a zero row gives wq = +-0 (the sign of each W) and sw = 0.
Storage is `wq` float8_e4m3fn [N, K] (row-major, the nn.Linear layout, which is the K-major operand f8 wgmma requires)
and `sw` fp32 [N], N * K + 4 N bytes (1.0005 B per weight at K = 4096).  The scales are per row, so q|k|v and gate|up are
each one stacked [sum N, K] matrix with concatenated `sw`.

Activation X [M, K] (bf16), per call: the same rule per row gives xq float8_e4m3fn [M, K] and sa fp32 [M].  There is no
threshold and no outlier list; the quantiser runs on the device without a host sync, so the decode CUDA graph captures
it.

Output, in this order:
  1. acc[m, n] = sum_k float(xq[m, k]) * float(wq[n, k]): each product is exact in fp32 (two 4-bit significands); the
     sum is accumulated in fp32.  The FP8 tensor-core MMA keeps fewer than 32 accumulator bits internally, so the kernels
     let it sum each 128-deep k-block on its own (scale-d = 0 on the block's first MMA) and add each block's result to
     an fp32 register total; no MMA accumulator runs over more than 128 products;
  2. s = sa[m] * sw[n], rounded to fp32;
  3. y = acc * s, rounded to fp32;
  4. y = y + bias[n] (if any), then y = y + residual[m, n] (if any), each rounded to fp32;
  5. one rounding to bf16 (or none for fp32 output).
The summation order in step 1 is not part of the format: the tensor-core GEMM (M > 8) and the decode GEMV (M <= 8)
order their sums differently, so a row computed by one and by the other agrees to fp32 accumulation error, not bit for
bit.  Each kernel is deterministic run to run.

Everything outside the seven decoder projections stays bf16, as under int8: embeddings, lm_head, norms, attention, SwiGLU,
the connector, the SVA layers and the towers.
"""
from __future__ import annotations

import torch

from .quant import PROJECTIONS  # noqa: F401  (the seven quantised projections, shared with NF4 and int8)

E4M3_MAX = 448.0


class Fp8Weight:
    """One FP8 operand: wq [N, K] float8_e4m3fn (row-major) and sw [N] fp32; several Linear weights may be stacked."""

    def __init__(self, N: int, K: int, device):
        if K % 16:
            raise ValueError(f"fp8: K = {K} must be a multiple of 16")
        self.shape = (N, K)
        self.wq = torch.empty((N, K), dtype=torch.float8_e4m3fn, device=device)
        self.sw = torch.empty(N, dtype=torch.float32, device=device)

    @property
    def nbytes(self) -> int:
        return self.wq.numel() + 4 * self.sw.numel()


class Fp8Projection:
    """The operand of one launch (q|k|v, o, gate|up or down) behind the projection interface the decoder layer uses."""

    def __init__(self, weight: Fp8Weight):
        self.w = weight
        self.N, self.K = weight.shape

    def linear(self, x, residual=None):
        from . import ops
        return ops.fp8_linear(x, self, residual=residual)

    def gate_up(self, x):
        from . import ops
        return ops.fp8_mlp_gate_up(x, self)


def bytes_per_weight(N: int, K: int) -> int:
    return N * K + 4 * N


def bytes_per_layer(config) -> int:
    """FP8 bytes (wq + sw) of the seven projections of one decoder layer."""
    H, I = config.hidden_size, config.intermediate_size
    nh, nkv = config.num_attention_heads, config.num_key_value_heads
    hd = getattr(config, "head_dim", None) or H // nh
    shapes = [(nh * hd, H), (nkv * hd, H), (nkv * hd, H), (H, nh * hd), (I, H), (I, H), (H, I)]
    return sum(bytes_per_weight(n, k) for n, k in shapes)


def quantize(*ws: torch.Tensor) -> Fp8Weight:
    """Quantise one or more bf16 [n_i, K] weights, stacked by rows, on their device (cb_fp8_quantize_weight);
    deterministic, no host sync."""
    from . import ops
    N, K = sum(w.shape[0] for w in ws), ws[0].shape[1]
    qw = Fp8Weight(N, K, ws[0].device)
    r = 0
    for w in ws:
        n = w.shape[0]
        ops.fp8_quantize_weight(w.contiguous(), qw.wq[r:r + n], qw.sw[r:r + n])
        r += n
    return qw


@torch.no_grad()
def quantize_decoder_fp8_(model, device) -> dict:
    """Quantise the seven projections of every decoder layer to FP8 in place, one layer at a time: the layer (which may
    still be on the CPU) moves to `device` in bf16, its projections are quantised there and their bf16 storage is freed
    (`p.data = empty`).  Peak device memory: the quantised layers + one bf16 layer + whatever else is already there.
    Embeddings, lm_head, norms, connector, SVA layers and towers are untouched (bf16).  Returns byte counts."""
    device = torch.device(device)
    layers = list(model.get_model().layers)
    bf16_bytes = fp8_bytes = 0
    for layer in layers:
        layer.to(device=device, dtype=torch.bfloat16)
        a, m = layer.self_attn, layer.mlp
        groups = dict(qkv=[a.q_proj, a.k_proj, a.v_proj], o=[a.o_proj], gate_up=[m.gate_proj, m.up_proj],
                      down=[m.down_proj])
        projs = {}
        for key, lins in groups.items():
            qw = quantize(*[lin.weight.data for lin in lins])
            fp8_bytes += qw.nbytes
            for lin in lins:
                bf16_bytes += lin.weight.numel() * lin.weight.element_size()
                lin.weight.data = torch.empty(0, dtype=torch.bfloat16, device=device)
                lin.weight.requires_grad_(False)
            projs[key] = Fp8Projection(qw)
        layer._fp8 = projs
    return dict(layers=len(layers), bf16_bytes=bf16_bytes, fp8_bytes=fp8_bytes)
