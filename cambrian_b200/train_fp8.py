"""FP8 E4M3 training of the decoder projections (`config.fp8_training`).

This module is the one place on the host that states the training format (csrc/train_fp8.cu, the E4M3 output of the
RMSNorm in csrc/norm.cu and the dual-output SwiGLU backward in csrc/elementwise.cu are the other side).  It reuses the
row rule and the output order of quant_fp8.py unchanged:
  * E4M3 values; per row: s = amax / 448, r = min(448 / amax, FLT_MAX), q = e4m3_rn_satfinite(fp32(v * r)), one fp32
    scale per row;
  * output: 128-deep k-blocks summed in fp32, then acc * (sa * sw), then + residual, then one rounding to bf16
    (`cb_gemm_fp8` as it stands).

Scaling is current per-row scaling: no amax history, no delayed scaling, no state, so a step is deterministic and needs no
host sync.  The scale is constant along the reduction dimension of every GEMM:

  GEMM (per layer)      A operand (rows x reduction)        B operand (rows x reduction)
  fwd   y  = x W^T      x  [M, K], per token                W   [N, K], per output row of W
  dgrad dx = dy W       dy [M, N], per token                W^T [K, N], per input column of W

f8 wgmma takes only K-major operands, so dgrad uses a transposed, separately quantised copy of each fused weight (q|k|v
stacked, o, gate|up stacked, down), made by `cb_fp8_quantize_weight_t`.

Which GEMMs run in FP8, per decoder layer: the four forward projections (q|k|v, o, gate|up, down), again in the
per-layer recompute, and their four input-gradient GEMMs.  Their operands:
  * q|k|v and gate|up in forward: `cb_rmsnorm_fwd_fp8` quantises the RMSNorm output (rounded to bf16 first) directly;
  * o and down in forward: `cb_fp8_quantize_act` of the attention output and of silu(gate) * up;
  * down, o and q|k|v dgrad: `cb_fp8_quantize_act` of dout, dx1 and dqkv;
  * gate|up dgrad: the E4M3 output of `cb_swiglu_bwd_fp8`, which also writes the bf16 gradient the wgrad GEMM reads.
Weights are quantised per layer and per call (row-wise copies in forward and in the recompute, the transposed copy in
backward) and dropped after use: a cache would hold 2 B per parameter of device memory and would have to be invalidated
after every optimizer update.

Everything else stays bf16 and unchanged: every weight-gradient GEMM (wgrad; it still accumulates into `main_grad`),
attention forward / backward, norms, SwiGLU arithmetic, RoPE, embeddings, lm_head and the fused loss, the connector, the
SVA layers and the towers.  wgrad reduces over the tokens of a step, so a per-row scale there would be one scale per
channel across all tokens, which flushes the tokens with small gradients; it needs a block-scaled mainloop.
`generate()` and the KV-cache path (`CBLlamaDecoderLayer.infer`) ignore the flag; `load_fp8` is the FP8 inference format.
"""
from __future__ import annotations

import torch

from .quant_fp8 import Fp8Projection, Fp8Weight, quantize


def enabled(config) -> bool:
    """`config.fp8_training`, read like `config.fused_lm_loss` (absent means off)."""
    return bool(getattr(config, "fp8_training", False))


def check_widths(hidden: int, intermediate: int, qkv: int) -> None:
    """Every reduction and every row length of the FP8 operands is one of these widths; f8 wgmma and the quantisers need
    multiples of 16."""
    for name, v in (("hidden_size", hidden), ("intermediate_size", intermediate), ("q|k|v width", qkv)):
        if v % 16:
            raise ValueError(f"fp8_training: {name} = {v} must be a multiple of 16")


def weight_rows(w: torch.Tensor) -> Fp8Projection:
    """The forward operand of one (fused) bf16 weight [N, K]: row-wise E4M3 with one scale per output row."""
    return Fp8Projection(quantize(w))


def weight_t(w: torch.Tensor) -> Fp8Projection:
    """The dgrad operand of one (fused) bf16 weight [N, K]: W^T [K, N] in E4M3 with one scale per input column of W."""
    from . import ops
    N, K = w.shape
    qw = Fp8Weight(K, N, w.device)
    ops.fp8_quantize_weight_t(w, qw.wq, qw.sw)
    return Fp8Projection(qw)
