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
That holds for every request of a server without the prefix cache, and for every miss of one with it.

Prefix cache (`BatchedGenerator(prefix_cache=True)`; the page format does not change).
  * Contents.  A position's content is its token id (generated tokens included), or for each position of an image span
    after the splice the request's image digest (serving.py).  `image_span` maps a digest to its span length, learned
    from the first prefill of that image.
  * Index.  A trie whose nodes are full pages, keyed by (parent node, the tuple of the page's page_size contents):
    exact keys, so two different prefixes never share a node.  A page enters it once its last position is written (a
    request's full prompt pages right after its prefill; a decode-filled page at the step that writes its last
    position), and a page in the index is never written again.  Contents already indexed under another page are not
    indexed twice: the request that wrote them again references that page and goes on indexing below it.
  * Reference counts.  A page is free, referenced (held by the tables of one or more running requests), or cached-idle
    (in the index, count 0).  A request holds every page above the ones it holds, so an idle page's indexed children
    are idle too.  `alloc` takes free pages lowest index first, then evicts idle pages without indexed children, least
    recently released first, so no indexed page is left without its parent.  `free_pages()` counts free plus idle
    pages; `cached_pages()` counts the index.
  * Gather.  A hit's prefill reads its cached positions [0, P) out of the pages with `kv_gather_kernel`
    (`ops.paged_kv_gather`) into dense bf16 rows: bf16 pages are copied, FP8 rows dequantised once as
    bf16(float(e4m3) * scale).  Its suffix's own K / V follow in bf16, the flash kernel attends over both (Sq < Skv,
    causal aligned bottom-right), and the suffix is appended at P.  So a hit's first-token logits are not bitwise a
    miss's: the suffix's projections see n rows instead of S0 (ops.gemm takes the GEMV at 8 rows or fewer), the flash
    kernel runs with Sq < Skv, and FP8 prefix rows come back dequantised rather than as the fresh bf16 rows.
"""
from __future__ import annotations

from collections import OrderedDict

import torch

from .kv_fp8 import CACHE_DTYPES

SPLIT_KEYS = 256          # key positions per split of the decode kernel (KVD_PAGED_CHUNK in csrc/kv_cache.cu)
DEFAULT_PAGE_SIZE = 64
ROOT = -1                 # the prefix index's root node (pages are nodes 0 .. num_pages - 1)


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
    """The pages of every layer, a free list of page indices, the decode workspace, and the prefix index (module
    docstring).  Pages are handed out lowest free index first, then by evicting cached-idle pages least recently used
    first, so allocation is deterministic."""

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
        self._ref = [0] * self.num_pages
        self._kids: dict[int, dict[tuple, int]] = {}     # trie node (ROOT or a page) -> {page contents: child page}
        self._node: dict[int, tuple] = {}                 # indexed page -> (parent node, page contents)
        self._idle: OrderedDict[int, None] = OrderedDict()   # cached-idle pages, least recently released first
        self.image_span: dict[bytes, int] = {}            # image digest -> positions of its span after the splice

    def layer(self, i: int):
        """(k pages, v pages, k scales or None, v scales or None) of layer i."""
        return self.k[i], self.v[i], (self.ks[i] if self.fp8 else None), (self.vs[i] if self.fp8 else None)

    def free_pages(self) -> int:
        """Pages an allocation can take: free ones plus cached-idle ones (evictable)."""
        return len(self._free) + len(self._idle)

    def cached_pages(self) -> int:
        """Pages in the prefix index, referenced or idle."""
        return len(self._node)

    def idle_among(self, pages) -> int:
        """How many of `pages` are cached-idle, i.e. counted by free_pages() until they are referenced."""
        return sum(1 for p in pages if self._ref[p] == 0)

    def alloc(self, n: int) -> list[int]:
        if n > self.free_pages():
            raise RuntimeError(f"paged KV cache: {n} pages requested, {self.free_pages()} free")
        out, self._free = self._free[:n], self._free[n:]
        while len(out) < n:
            out.append(self._evict())
        for p in out:
            self._ref[p] = 1
        return out

    def ref(self, pages) -> None:
        """Take one more reference on indexed pages (a prefix hit); a cached-idle page stops being evictable."""
        for p in pages:
            self._ref[p] += 1
            self._idle.pop(p, None)

    def release(self, pages) -> None:
        """Drop one reference on each page: at zero an indexed page becomes cached-idle, any other page free."""
        freed = []
        for p in pages:
            self._ref[p] -= 1
            if self._ref[p] == 0:
                if p in self._node:
                    self._idle[p] = None
                else:
                    freed.append(p)
        if freed:
            self._free = sorted(self._free + freed)

    def _evict(self) -> int:
        # the least recently released idle page without indexed children: an idle page's children are idle too (a
        # request holds every page above the ones it holds), so one exists, and no indexed page loses its parent
        p = next(q for q in self._idle if q not in self._kids)
        del self._idle[p]
        parent, key = self._node.pop(p)
        kids = self._kids[parent]
        del kids[key]
        if not kids:
            del self._kids[parent]
        return p

    # ---- the prefix index: a trie of full pages keyed by (parent node, the page's page_size position contents) ----
    def match(self, content):
        """The longest indexed prefix of `content` (a sequence of position contents): (pages of whole matching pages,
        (page, rows) of the indexed page after them that matches the most leading rows of the rest, or None)."""
        ps, node, full = self.page_size, ROOT, []
        for i in range(len(content) // ps):
            page = self._kids.get(node, {}).get(tuple(content[i * ps:(i + 1) * ps]))
            if page is None:
                break
            full.append(page)
            node = page
        rest = content[len(full) * ps:(len(full) + 1) * ps]
        part = None
        for key, page in self._kids.get(node, {}).items():
            n = 0
            while n < len(rest) and key[n] == rest[n]:
                n += 1
            if n and (part is None or n > part[1]):
                part = (page, n)
        return full, part

    def insert(self, parent: int, key: tuple, page: int):
        """Index `page`, whose positions are all written and hold `key`, under trie node `parent`, which the caller
        holds.  Returns the node of these contents: `page`, or the page they are indexed under already (which the caller
        then references, so that it keeps holding every page above the ones it indexes)."""
        kids = self._kids.setdefault(parent, {})
        if key in kids:
            return kids[key]
        kids[key] = page
        self._node[page] = (parent, key)
        return page

    def nbytes(self) -> int:
        """Device bytes of the pages, the scales and the decode workspace."""
        ts = self.k + self.v + (self.ks + self.vs if self.fp8 else []) + [self.ws]
        return sum(t.numel() * t.element_size() for t in ts)


class PagedCacheView:
    """What `CambrianLlamaModel.forward` takes in `past_key_values` to run on the pages: the rows' block table and lengths
    (device int32).  `prefill=True`: one sequence into its pages after `prefix` cached positions (prefix 0: the flash
    kernel over its own K / V, then an append at position 0; prefix P > 0: positions [0, P) gathered out of the pages
    into `kv_buf`, the suffix's own K / V after them, the flash kernel over both, then an append at P); otherwise one
    decode token per row, appended at lens[b] and attended over positions <= lens[b]."""

    slot = None               # the dense cache's graph-replay slot; the paged view keeps its state in `lens`

    def __init__(self, pool: PagedKVPool, table: torch.Tensor, lens: torch.Tensor, prefill: bool, prefix: int = 0):
        self.pool, self.table, self.lens, self.prefill = pool, table, lens, prefill
        self.prefix = self.length = int(prefix)
        self.kmask = None
        self.kv_buf = None    # a hit's bf16 K and V rows [1, P + n, nkv, hd], shared by the layers of one prefill

    def prefix_buffers(self, n: int, nkv: int, hd: int, device):
        """The bf16 K / V buffers [1, prefix + n, nkv, hd] of a prefill after a cached prefix (allocated once)."""
        if self.kv_buf is None:
            shape = (1, self.prefix + n, nkv, hd)
            self.kv_buf = (torch.empty(shape, dtype=torch.bfloat16, device=device),
                           torch.empty(shape, dtype=torch.bfloat16, device=device))
        return self.kv_buf
