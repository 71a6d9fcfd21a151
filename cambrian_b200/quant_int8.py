"""8-bit LLM.int8 weights for inference (`load_8bit`, model/builder.py:35-36).

The scheme is bitsandbytes' LLM.int8 (vector-wise absmax quantisation with mixed-precision outlier decomposition); this
module is the one place on the host that knows its format and arithmetic (the kernels in csrc/int8.cu are the other
side).  Byte compatibility with bitsandbytes serialisation (`SCB` keys) is not claimed.

Weight W [N, K] (bf16, K % 16 == 0), quantised once at load:
  * scb[n] = max |W[n, :]| (fp32);
  * cb[n, k] = int8 rint(W[n, k] * (127 / scb[n])), round half to even, clamped to +-127; a zero row gives cb = 0,
    scb = 0.  The scales are per row, so q|k|v and gate|up are one stacked int8 matrix with concatenated scb.

Activation X [M, K] (bf16), per call, threshold tau = 6.0 (bitsandbytes' `llm_int8_threshold`):
  * outlier columns O = { j : max over the M rows of |X[m, j]| >= tau }, kept as an ascending int32 index list and a
    device count; tau <= 0 disables outliers;
  * sca[m] = max |X[m, j]| over j not in O;
  * xq[m, j] = rint(X[m, j] * (127 / sca[m])) for j not in O, 0 for j in O; a zero row gives 0.

Output, in this order, each product and sum rounded to fp32 on its own (no FMA contraction):
  * acc = sum_j xq[m, j] * cb[n, j], exact in int32;
  * v = (float(acc) * (sca[m] * scb[n])) * (1/16129)                         (1/16129 rounded to fp32)
  * o = 0, then for j in O ascending: o = o + x[m, j] * (float(cb[n, j]) * (scb[n] * (1/127)))   (1/127 rounded to fp32)
  * y = v + o, then y = y + bias[n] (if any), then y = y + residual[m, n] (if any), then one rounding to bf16 (or fp32
    output).
The int8 tensor-core GEMM (M > 8) and the dp4a GEMV (M <= 8) both follow it, so prefill and decode rows agree bit for
bit.  Everything outside the seven decoder projections (embeddings, lm_head, norms, attention, SwiGLU, connector, SVA
layers, towers) stays bf16.
"""
from __future__ import annotations

import torch

from .quant import PROJECTIONS  # noqa: F401  (the seven quantised projections, shared with NF4)

THRESHOLD = 6.0


class Int8Weight:
    """One int8 operand: cb [N, K] int8 (row-major) and scb [N] fp32; several Linear weights may be stacked by rows."""

    def __init__(self, N: int, K: int, device):
        if K % 16:
            raise ValueError(f"int8: K = {K} must be a multiple of 16")
        self.shape = (N, K)
        self.cb = torch.empty((N, K), dtype=torch.int8, device=device)
        self.scb = torch.empty(N, dtype=torch.float32, device=device)

    @property
    def nbytes(self) -> int:
        return self.cb.numel() + 4 * self.scb.numel()


class Int8Projection:
    """The operand of one launch (q|k|v, o, gate|up or down) behind the projection interface the decoder layer uses."""

    def __init__(self, weight: Int8Weight, threshold: float = THRESHOLD):
        self.w = weight
        self.N, self.K = weight.shape
        self.threshold = threshold

    def linear(self, x, residual=None):
        from . import ops
        return ops.int8_linear(x, self, residual=residual)

    def gate_up(self, x):
        from . import ops
        return ops.int8_mlp_gate_up(x, self)


def bytes_per_weight(N: int, K: int) -> int:
    return N * K + 4 * N


def bytes_per_layer(config) -> int:
    """int8 bytes (cb + scb) of the seven projections of one decoder layer."""
    H, I = config.hidden_size, config.intermediate_size
    nh, nkv = config.num_attention_heads, config.num_key_value_heads
    hd = getattr(config, "head_dim", None) or H // nh
    shapes = [(nh * hd, H), (nkv * hd, H), (nkv * hd, H), (H, nh * hd), (I, H), (I, H), (H, I)]
    return sum(bytes_per_weight(n, k) for n, k in shapes)


def quantize_into(w: torch.Tensor, qw: Int8Weight, row0: int = 0) -> None:
    """Quantise one bf16 [n, K] weight on its device into rows [row0, row0 + n) of `qw` (cb_int8_quantize_weight)."""
    from . import ops
    n = w.shape[0]
    ops.int8_quantize_weight(w.contiguous(), qw.cb[row0:row0 + n], qw.scb[row0:row0 + n])


def quantize(*ws: torch.Tensor) -> Int8Weight:
    """Quantise one or more bf16 [n_i, K] weights, stacked by rows, on their device; deterministic, no host sync."""
    N, K = sum(w.shape[0] for w in ws), ws[0].shape[1]
    qw = Int8Weight(N, K, ws[0].device)
    r = 0
    for w in ws:
        quantize_into(w, qw, r)
        r += w.shape[0]
    return qw


@torch.no_grad()
def quantize_decoder_int8_(model, device, threshold: float = THRESHOLD) -> dict:
    """Quantise the seven projections of every decoder layer to int8 in place, one layer at a time: the layer (which may
    still be on the CPU) moves to `device` in bf16, its projections are quantised there and their bf16 storage is freed
    (`p.data = empty`).  Peak device memory: the quantised layers + one bf16 layer + whatever else is already there.
    Embeddings, lm_head, norms, connector, SVA layers and towers are untouched (bf16).  Returns byte counts."""
    device = torch.device(device)
    layers = list(model.get_model().layers)
    bf16_bytes = int8_bytes = 0
    for layer in layers:
        layer.to(device=device, dtype=torch.bfloat16)
        a, m = layer.self_attn, layer.mlp
        groups = dict(qkv=[a.q_proj, a.k_proj, a.v_proj], o=[a.o_proj], gate_up=[m.gate_proj, m.up_proj],
                      down=[m.down_proj])
        projs = {}
        for key, lins in groups.items():
            qw = quantize(*[lin.weight.data for lin in lins])
            int8_bytes += qw.nbytes
            for lin in lins:
                bf16_bytes += lin.weight.numel() * lin.weight.element_size()
                lin.weight.data = torch.empty(0, dtype=torch.bfloat16, device=device)
                lin.weight.requires_grad_(False)
            projs[key] = Int8Projection(qw, threshold)
        layer._int8 = projs
    return dict(layers=len(layers), bf16_bytes=bf16_bytes, int8_bytes=int8_bytes)
