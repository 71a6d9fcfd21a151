"""FP8 E4M3 decode KV cache (`generate(..., kv_cache_dtype="fp8")`).

This module is the one place on the host that states the format and its arithmetic (the kernels `kv_append_kernel` and
`kv_decode_kernel` over `DenseCells` in csrc/kv_cache.cu are the other side; the paged cache of paged_kv.py runs the same
kernels over `PagedCells`).  E4M3 and e4m3_rn_satfinite are those of quant_fp8.py.

Rows.  Each cached row is the hd elements of one (sequence, position, kv head) of K or of V, after RoPE, as the decoder
layer's packed qkv GEMM output holds them (bf16).  K and V are separate rows.

Quantisation, per row, the rule quant_fp8.py uses for weights and activations:
  * amax = max_d |x[d]| (exact);  s = amax / 448, one fp32 division;
  * r = 448 / amax, one fp32 division, replaced by the largest finite fp32 when it overflows (a zero row, a row of bf16
    subnormals), so nothing saturates there and nothing is NaN;
  * q[d] = e4m3_rn_satfinite(fp32(float(x[d]) * r));  a zero row keeps the sign of each zero and gets s = 0.

Storage per layer: kq, vq float8_e4m3fn [B, S_max, nkv, hd] and ks, vs fp32 [B, S_max, nkv], 2 * nkv * (hd + 4) bytes per
token (51.6 % of the bf16 cache at hd 128).  The scales start at zero; a slot is written once, by the step that appends
its token.

Decode attention for one query row q (bf16, after RoPE) of query head j, served by kv head j // (nh / nkv), over the valid
keys t (below the valid length, key mask set), in this order:
  1. score_t = (sum_d float(q[d]) * float(kq[t, d])) * ks[t], then * softmax_scale (hd^-0.5), each product fp32-rounded;
  2. softmax over t in fp32 (online: running max and sum);
  3. o = sum_t p_t * vs[t] * float(vq[t, :]), normalised by sum_t p_t;
  4. one rounding to bf16.
The summation order is not part of the format (the kernel splits keys over CTAs and lanes); each kernel is deterministic
from run to run.

Prefill.  The prompt attends over its own fresh bf16 K / V with the flash kernel, exactly as with the bf16 cache, and is
then appended; only later decode steps read the quantised cache.  So the prefill hidden states and the first generated
token are bitwise those of the bf16-cache path.  A decode step appends its own K / V row first and then attends over the
cache including it.
"""
from __future__ import annotations

import torch

CACHE_DTYPES = ("bf16", "fp8")


def resolve_cache_dtype(config, value=None) -> str:
    """`kv_cache_dtype` of generate(): the keyword, else `config.kv_cache_dtype`, else "bf16"."""
    v = getattr(config, "kv_cache_dtype", None) if value is None else value
    v = "bf16" if v is None else v
    if v not in CACHE_DTYPES:
        raise ValueError(f"kv_cache_dtype={v!r} is not supported: use one of {CACHE_DTYPES}")
    return v


def bytes_per_token(config) -> int:
    """FP8 cache bytes per token over all layers: kq + vq + ks + vs."""
    nkv = config.num_key_value_heads
    hd = getattr(config, "head_dim", None) or config.hidden_size // config.num_attention_heads
    return config.num_hidden_layers * 2 * nkv * (hd + 4)


class Fp8KVLayers:
    """The FP8 cache buffers of every layer and the decode workspace (fp32, shared by the layers, which run one after
    another on one stream), allocated once so that a captured decode step allocates nothing."""

    def __init__(self, L: int, batch: int, max_len: int, nh: int, nkv: int, hd: int, device):
        if hd not in (64, 128):
            raise ValueError(f"kv_cache_dtype='fp8' supports head_dim 64 or 128, not {hd}")
        if nh % nkv or not 1 <= nh // nkv <= 8:
            raise ValueError(f"kv_cache_dtype='fp8' supports 1..8 query heads per kv head, not {nh} / {nkv}")
        f8 = torch.float8_e4m3fn
        self.kq = [torch.zeros((batch, max_len, nkv, hd), dtype=f8, device=device) for _ in range(L)]
        self.vq = [torch.zeros((batch, max_len, nkv, hd), dtype=f8, device=device) for _ in range(L)]
        self.ks = [torch.zeros((batch, max_len, nkv), dtype=torch.float32, device=device) for _ in range(L)]
        self.vs = [torch.zeros((batch, max_len, nkv), dtype=torch.float32, device=device) for _ in range(L)]
        from . import ops
        self.ws = ops.attn_decode_fp8_workspace(batch, nh, nkv, max_len, hd, device)

    def layer(self, i: int):
        return self.kq[i], self.vq[i], self.ks[i], self.vs[i]

    def nbytes(self) -> int:
        ts = self.kq + self.vq + self.ks + self.vs + [self.ws]
        return sum(t.numel() * t.element_size() for t in ts)
