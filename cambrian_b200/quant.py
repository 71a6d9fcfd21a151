"""4-bit NF4 weights with double-quantised scales for inference (`load_4bit`, model/builder.py:37-44).

The format follows bitsandbytes NF4 with double quantisation; this module is the one place on the host that knows it
(the kernels in csrc/nf4.cu are the other side).  Per HF `nn.Linear` weight W [N, K] (bf16, K % 64 == 0):

  * blocks of 64 consecutive row-major elements; absmax_b = max |w| over the block (fp32);
  * code = number of the 15 fp32 midpoints (c[i] + c[i+1]) / 2 of the NF4 table `NF4_CODE` strictly below
    x = w * (1 / absmax_b); an all-zero block gets code 7 (0.0);
  * two codes per byte, element 2j in the HIGH nibble -> packed uint8 [N, K / 2];
  * double quantisation: offset = mean(absmax) (fp32, fixed-order reduction), groups of 256 blocks (the last may be
    partial), absmax2_g = max |absmax_b - offset| over the group, qabsmax_b = index of the entry of the signed dynamic map
    nearest to (absmax_b - offset) * (1 / absmax2_g): the first entry >= v or the one before it, whichever is closer in
    fp32, the larger one on a tie; absmax2_g == 0 stores the index of 0.0;
  * dequantisation: absmax_b = map[qabsmax_b] * absmax2_g + offset (two roundings, no FMA), w~ = bf16(c[code] * absmax_b).

Compute stays bf16 with fp32 accumulation: decode (M <= 8 rows) runs the NF4 GEMV, larger batches dequantise the fused
projection into one model-owned bf16 scratch buffer and run the bf16 GEMM on it (ops.nf4_linear).
"""
from __future__ import annotations

import torch

BLOCK = 64
GROUP = 256
NF4_CODE = (-1.0, -0.6961928009986877, -0.5250730514526367, -0.39491748809814453, -0.28444138169288635,
            -0.18477343022823334, -0.09105003625154495, 0.0, 0.07958029955625534, 0.16093020141124725,
            0.24611230194568634, 0.33791524171829224, 0.44070982933044434, 0.5626170039176941, 0.7229568362236023, 1.0)
PROJECTIONS = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")


def dynamic_map(signed: bool = True) -> torch.Tensor:
    """bitsandbytes `create_dynamic_map(signed)`: 256 sorted fp32 values.  Both hold 0 and 1.0; decade i = 0..6 adds
    10^(i-6) times the interval means of linspace(0.1, 1, k + 1), with k = 2^i means and their negatives (signed) or
    k = 2^(i+1) means (unsigned)."""
    data = [0.0, 1.0]
    for i in range(7):
        b = torch.linspace(0.1, 1, 2 ** (i if signed else i + 1) + 1, dtype=torch.float32)
        means = (b[:-1] + b[1:]) / 2.0
        data += ((10 ** (i - 6)) * means).tolist()
        if signed:
            data += (-(10 ** (i - 6)) * means).tolist()
    return torch.tensor(sorted(data), dtype=torch.float32)


class NF4Weight:
    """One quantised HF Linear weight [N, K]: packed codes, per-block 8-bit scale indices, per-group fp32 scales and the
    device-resident fp32 offset."""

    def __init__(self, N: int, K: int, device):
        if K % BLOCK:
            raise ValueError(f"NF4: K = {K} must be a multiple of {BLOCK}")
        nb = N * K // BLOCK
        self.shape = (N, K)
        self.packed = torch.empty((N, K // 2), dtype=torch.uint8, device=device)
        self.qabsmax = torch.empty(nb, dtype=torch.uint8, device=device)
        self.absmax2 = torch.empty((nb + GROUP - 1) // GROUP, dtype=torch.float32, device=device)
        self.offset = torch.empty(1, dtype=torch.float32, device=device)

    @property
    def nbytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in (self.packed, self.qabsmax, self.absmax2, self.offset))


class NF4Projection:
    """The operand of one launch: 1-3 NF4Weights stacked by rows (q|k|v, gate|up), each quantised on its own, plus the
    model's shared bf16 dequantisation scratch."""

    def __init__(self, parts, scratch):
        self.parts = list(parts)
        self.K = parts[0].shape[1]
        if any(p.shape[1] != self.K for p in parts):
            raise ValueError("NF4Projection: segments must share K")
        self.N = sum(p.shape[0] for p in parts)
        self.row0 = [sum(p.shape[0] for p in parts[:i]) for i in range(len(parts))]
        self.scratch = scratch

    def linear(self, x, residual=None):
        from . import ops
        return ops.nf4_linear(x, self, residual=residual)

    def gate_up(self, x):
        from . import ops
        return ops.nf4_mlp_gate_up(x, self)

    def segment_arrays(self):
        return self.row0, [p.packed for p in self.parts], [p.qabsmax for p in self.parts], \
            [p.absmax2 for p in self.parts], [p.offset for p in self.parts]


def bytes_per_weight(N: int, K: int) -> int:
    nb = N * K // BLOCK
    return N * K // 2 + nb + 4 * ((nb + GROUP - 1) // GROUP) + 4


def bytes_per_layer(config) -> int:
    """NF4 bytes of the seven projections of one decoder layer."""
    H, I = config.hidden_size, config.intermediate_size
    nh, nkv = config.num_attention_heads, config.num_key_value_heads
    hd = getattr(config, "head_dim", None) or H // nh
    shapes = [(nh * hd, H), (nkv * hd, H), (nkv * hd, H), (H, nh * hd), (I, H), (I, H), (H, I)]
    return sum(bytes_per_weight(n, k) for n, k in shapes)


def quantize(w: torch.Tensor, workspace: torch.Tensor | None = None) -> NF4Weight:
    """Quantise one bf16 [N, K] weight on its device (cb_nf4_quantize); deterministic, no host sync."""
    from . import ops
    N, K = w.shape
    qw = NF4Weight(N, K, w.device)
    nb = N * K // BLOCK
    if workspace is None or workspace.numel() < nb:
        workspace = torch.empty(nb, dtype=torch.float32, device=w.device)
    ops.nf4_quantize(w.contiguous(), workspace, qw.packed, qw.qabsmax, qw.absmax2, qw.offset)
    return qw


def quantized_format(model) -> str | None:
    """"4-bit (NF4)", "8-bit (LLM.int8)" or "8-bit (FP8)" when a decoder layer of `model` carries quantised weights
    (quantize_decoder_nf4_ / quant_int8.quantize_decoder_int8_ / quant_fp8.quantize_decoder_fp8_), else None: the
    wording of every refusal."""
    for m in model.modules():
        if getattr(m, "_nf4", None) is not None:
            return "4-bit (NF4)"
        if getattr(m, "_int8", None) is not None:
            return "8-bit (LLM.int8)"
        if getattr(m, "_fp8", None) is not None:
            return "8-bit (FP8)"
    return None


def is_quantized(model) -> bool:
    """True when any decoder layer of `model` carries NF4, int8 or FP8 weights."""
    return quantized_format(model) is not None


@torch.no_grad()
def quantize_decoder_nf4_(model, device) -> dict:
    """Quantise the seven projections of every decoder layer to NF4 in place, one layer at a time: the layer (which may
    still be on the CPU) moves to `device` in bf16, its projections are quantised there and their bf16 storage is freed
    (`p.data = empty`).  Peak device memory: the quantised layers + one bf16 layer + whatever else is already there.
    Embeddings, lm_head, norms, connector, SVA layers and towers are untouched (bf16).  Returns byte counts."""
    device = torch.device(device)
    inner = model.get_model()
    layers = list(inner.layers)
    cfg = model.config
    H, I = cfg.hidden_size, cfg.intermediate_size
    nh, nkv = cfg.num_attention_heads, cfg.num_key_value_heads
    hd = getattr(cfg, "head_dim", None) or H // nh
    rows_k = [((nh + 2 * nkv) * hd, H), (H, nh * hd), (2 * I, H), (H, I)]
    scratch = torch.empty(max(r * k for r, k in rows_k), dtype=torch.bfloat16, device=device)
    workspace = torch.empty(max(r * k for r, k in rows_k) // BLOCK, dtype=torch.float32, device=device)
    bf16_bytes = nf4_bytes = 0
    for layer in layers:
        layer.to(device=device, dtype=torch.bfloat16)
        a, m = layer.self_attn, layer.mlp
        q = {}
        for name, lin in (("q_proj", a.q_proj), ("k_proj", a.k_proj), ("v_proj", a.v_proj), ("o_proj", a.o_proj),
                          ("gate_proj", m.gate_proj), ("up_proj", m.up_proj), ("down_proj", m.down_proj)):
            w = lin.weight
            q[name] = quantize(w.data, workspace)
            bf16_bytes += w.numel() * w.element_size()
            nf4_bytes += q[name].nbytes
            w.data = torch.empty(0, dtype=torch.bfloat16, device=device)
            w.requires_grad_(False)
        layer._nf4 = dict(qkv=NF4Projection([q["q_proj"], q["k_proj"], q["v_proj"]], scratch),
                          o=NF4Projection([q["o_proj"]], scratch),
                          gate_up=NF4Projection([q["gate_proj"], q["up_proj"]], scratch),
                          down=NF4Projection([q["down_proj"]], scratch))
    del workspace
    inner._nf4_scratch = scratch
    return dict(layers=len(layers), bf16_bytes=bf16_bytes, nf4_bytes=nf4_bytes, scratch_bytes=scratch.numel() * 2)
