"""Paged decode KV cache (`serving.BatchedGenerator`).

This module is the one place on the host that states the format (the kernels `kv_append_kernel` and `kv_decode_kernel`
over `PagedCells` in csrc/kv_cache.cu are the other side; the dense FP8 cache of kv_fp8.py runs the same kernels over
`DenseCells`).

Pages.  Each decoder layer has a pool of `num_pages` fixed-size pages for K and one for V, each
[num_pages, page_size, nkv, hd].  Inside a page the layout is position-major, the row layout of the dense `KVCache`: page
slot i holds the nkv head rows of one position.  So one page holds `page_size` consecutive positions of one sequence.
`page_size` is a power of two >= 16 (default 64).
  * bf16 pages hold the bf16 K / V rows (after RoPE) unchanged.
  * FP8 pages hold E4M3 rows plus fp32 scales [num_pages, page_size, nkv], quantised per head row by exactly the rule of
    kv_fp8.py (the bytes and scales are bit for bit those `cb_kv_fp8_append` writes for the same rows).

Block table.  int32 [rows, max_pages_per_seq]: entry (b, p) is the page that holds positions [p * page_size,
(p + 1) * page_size) of the sequence in row b.  Entries past a sequence's reservation are never read.

Lengths.  A device int32 `lens[rows]` holds each row's cached length; a negative length marks an inactive (padding) row,
which is neither written nor read and whose attention output is zero.

Append.  Row s of sequence b goes to position start + s, where start is a host offset (a prefill, into empty pages) or
lens[b] read on the device (a graph-replayed decode step).

Decode attention, one query per row, over the positions below lens[b] + 1 (the row appended just before):
  * bf16 pages: score_t = (q . k_t) * hd^-0.5 and the softmax and the PV sum in fp32, one rounding to bf16;
  * FP8 pages: the decode arithmetic of kv_fp8.py.
Keys are split into chunks of SPLIT_KEYS positions, a constant: it does not depend on the batch, the bucket or the SM
count, and the per-split partials are merged in split order.  So a sequence's output is bitwise independent of which
other sequences share the launch and of how many padding rows there are.

Prefill attends over its own fresh bf16 K / V with the flash kernel, exactly as `generate()` does, and is then appended;
so a served request's prefill hidden states and first token are bitwise those of `generate()` for the same prompt.
"""
from __future__ import annotations

import torch

from .kv_fp8 import CACHE_DTYPES

SPLIT_KEYS = 256          # key positions per split of the decode kernel (KVD_PAGED_CHUNK in csrc/kv_cache.cu)
DEFAULT_PAGE_SIZE = 64


def _dims(config):
    nkv = config.num_key_value_heads
    hd = getattr(config, "head_dim", None) or config.hidden_size // config.num_attention_heads
    return config.num_hidden_layers, config.num_attention_heads, nkv, hd


def bytes_per_token(config, dtype: str = "bf16") -> int:
    """Page bytes per cached token over all layers: K and V rows (bf16: 2 bytes per element; fp8: 1 byte plus a 4-byte
    scale per head row)."""
    L, _, nkv, hd = _dims(config)
    if dtype not in CACHE_DTYPES:
        raise ValueError(f"kv_cache_dtype={dtype!r} is not supported: use one of {CACHE_DTYPES}")
    return L * 2 * nkv * (hd * 2 if dtype == "bf16" else hd + 4)


def check_page_size(page_size: int) -> int:
    page_size = int(page_size)
    if page_size < 16 or page_size & (page_size - 1):
        raise ValueError(f"page_size={page_size} must be a power of two >= 16")
    return page_size


def pages_for(tokens: int, page_size: int) -> int:
    return (int(tokens) + page_size - 1) // page_size


class PagedKVPool:
    """The pages of every layer, a free list of page indices, and the decode workspace.  Pages are handed out lowest
    index first and returned on release, so allocation is deterministic."""

    def __init__(self, config, num_pages: int, page_size: int, dtype: str, max_rows: int, max_pages_per_seq: int,
                 device):
        from . import ops
        L, nh, nkv, hd = _dims(config)
        if dtype not in CACHE_DTYPES:
            raise ValueError(f"kv_cache_dtype={dtype!r} is not supported: use one of {CACHE_DTYPES}")
        if hd not in (64, 128):
            raise ValueError(f"the paged KV cache supports head_dim 64 or 128, not {hd}")
        if nh % nkv or not 1 <= nh // nkv <= 8:
            raise ValueError(f"the paged KV cache supports 1..8 query heads per kv head, not {nh} / {nkv}")
        self.page_size = check_page_size(page_size)
        self.num_pages = int(num_pages)
        if self.num_pages < 1:
            raise ValueError("the paged KV cache needs at least one page")
        self.dtype = dtype
        self.fp8 = dtype == "fp8"
        self.max_pages_per_seq = int(max_pages_per_seq)
        shape = (self.num_pages, self.page_size, nkv, hd)
        el = torch.float8_e4m3fn if self.fp8 else torch.bfloat16
        self.k = [torch.zeros(shape, dtype=el, device=device) for _ in range(L)]
        self.v = [torch.zeros(shape, dtype=el, device=device) for _ in range(L)]
        self.ks = self.vs = None
        if self.fp8:
            self.ks = [torch.zeros(shape[:3], dtype=torch.float32, device=device) for _ in range(L)]
            self.vs = [torch.zeros(shape[:3], dtype=torch.float32, device=device) for _ in range(L)]
        self.ws = ops.attn_decode_paged_workspace(max_rows, nh, self.max_pages_per_seq, self.page_size, hd, device)
        self._free = list(range(self.num_pages))

    def layer(self, i: int):
        """(k pages, v pages, k scales or None, v scales or None) of layer i."""
        return self.k[i], self.v[i], (self.ks[i] if self.fp8 else None), (self.vs[i] if self.fp8 else None)

    def free_pages(self) -> int:
        return len(self._free)

    def alloc(self, n: int) -> list[int]:
        if n > len(self._free):
            raise RuntimeError(f"paged KV cache: {n} pages requested, {len(self._free)} free")
        out, self._free = self._free[:n], self._free[n:]
        return out

    def release(self, pages) -> None:
        self._free = sorted(self._free + list(pages))

    def nbytes(self) -> int:
        """Device bytes of the pages, the scales and the decode workspace."""
        ts = self.k + self.v + (self.ks + self.vs if self.fp8 else []) + [self.ws]
        return sum(t.numel() * t.element_size() for t in ts)


class PagedCacheView:
    """What `CambrianLlamaModel.forward` takes in `past_key_values` to run on the pages: the rows' block table and lengths
    (device int32).  `prefill=True`: one sequence into empty pages (the flash kernel over its own K / V, then an append at
    position 0); otherwise one decode token per row, appended at lens[b] and attended over positions <= lens[b]."""

    slot = None               # the dense cache's graph-replay slot; the paged view keeps its state in `lens`

    def __init__(self, pool: PagedKVPool, table: torch.Tensor, lens: torch.Tensor, prefill: bool):
        self.pool, self.table, self.lens, self.prefill = pool, table, lens, prefill
        self.length = 0
        self.kmask = None
