"""Continuous batching over a paged KV cache: many independent generation requests served at once.

The reference serves many requests at once through an SGLang worker next to its one-request model worker
(serve/sglang_worker.py batches them); this module is that batching for the decoder here.  `generate()` owns a dense
cache per call and a batch that is fixed from its first token to its last; `BatchedGenerator` keeps one pool of
fixed-size pages (paged_kv.py) and lets requests join and leave between decode steps:

    srv = BatchedGenerator(model, max_batch=32, max_cached_tokens=65536, page_size=64, kv_cache_dtype="bf16")
    rid = srv.submit(input_ids, images=None, image_sizes=None, **generate_kwargs)   # one unpadded sequence
    for rid, token, finished in srv.step(): ...                                      # one decode step for every request
    outs = srv.run()                                                                # drain: {rid: LongTensor of new ids}

Requests.  The keywords are those of `generate()` (GenerationArgs.from_kwargs): greedy or temperature / top-k / top-p
sampling with the request's own `generator`, `eos_token_id`, `max_new_tokens` / `max_length`, `stopping_criteria`,
`streamer`; everything `generate()` refuses is refused at `submit` with the same exception.

Admission is FIFO and deterministic, without preemption: the head of the queue is admitted when a row is free and the
pages for its prompt plus `max_new_tokens` can be reserved; its pages return to the pool when it finishes.  A request
that could never fit the pool raises ValueError at `submit`.  Before the prefill the prompt length is bounded from
above (a bare <image> indicator expands to at most image_token_len + sqrt(image_token_len) positions); the pages beyond
the true length are returned right after it.

A step (1) prefills the newly admitted requests one at a time through the prefill of `generate()` (towers, SVA, the
dynamic branch for non-square images), which gives each its first token; (2) packs the running requests into rows
[0, n), compacting when one retires; (3) runs one decode step for all of them, padded to a bucket of 1, 2, 4, ...
rows (padding rows are inactive), as one CUDA graph per bucket captured on first use; (4) picks each row's token: the
argmax for greedy rows and, when a row samples, ops.sample_tokens for all rows with each row's own parameters, seed and
step in device buffers (written when the row set changes, the steps advanced by the step itself), one torch.where
choosing per row, inside the same graph (a bucket has a second graph for steps with sampled rows); (5) applies EOS and
stopping criteria, retires and streams.  A sampled request's seed is the one row 0 of a solo `generate()` with its
generator draws (generation.py), drawn at its first token, and its token t uses step t, so its tokens are solo
`generate()`'s wherever their logits are equal.  Graph and eager (`use_graph=False`) steps run the same
kernels on the same padded shapes and give bitwise identical tokens.  The paged decode attention's result for a row is
bitwise independent of the other rows.  The rest of the step is not: the projection and lm_head GEMMs pick their kernel
by the bucket's row count (ops.gemm: the CUDA-core GEMV up to 8 rows, except wide outputs at 6-8 rows; the tensor-core
GEMM above), and those kernels sum in different orders.  So a request's logits can change in the last bits with the
number of requests running beside it, and a close greedy race can then go the other way.

Prefix cache (`prefix_cache=True`, off by default; paged_kv.py states the index).  Multi-turn chat resends the whole
conversation with its image, and several questions about one image repeat the system prompt and the image; a hit
reuses those cached pages instead of running the towers, the connector, the SVA sites and the prefill over them.
  * Contents.  A request's prompt contents are its ids with the <image> indicator expanded to the image's span, every
    span position carrying the image digest: SHA-256 of the host bytes, dtypes and shapes of the per-tower image
    tensors plus `image_sizes`, computed at `submit`.  The span length is learned from the first prefill of the
    image (the dynamic branch makes it depend on `image_sizes`, which the digest includes).
  * Matching, when the request reaches the head of the queue: whole matching pages of the index, then the longest
    match of leading rows inside one more indexed page, whose rows are copied into the request's first private page.
    The hit is capped at S0 - 1 positions, so at least one position is prefilled and gives the first token.
  * Image rule.  A request with an image hits only if the hit covers its whole image span, since the in-LLM SVA sites
    address the span at `cfg.image_position` of the forward's own hidden states; otherwise it gets a full prefill.  An
    image request whose span length is not known yet, whose ids already hold an expanded span, or whose <image> is not
    at `image_position` while SVA sites run, is served without the cache.  Text-only requests hit on any prefix.
  * Admission references the matched pages before it allocates, so it never evicts its own hit, and reserves
    pages_for(S0 + max_new_tokens) minus the shared whole pages (S0 is exact on a hit).  Retirement drops the
    references: indexed pages become cached-idle, the others free.
  * Numerics.  A miss is bitwise the server without the cache.  A hit's first-token logits are not bitwise a miss's:
    the suffix's projections see n rows (ops.gemm takes the GEMV at 8 rows or fewer), the flash kernel runs with
    Sq < Skv over the gathered prefix, and FP8 prefix rows are dequantised once to bf16.
  * `hit_rate()` is reused prompt positions over prefilled prompt positions; `cached_pages()` the index's size.
"""
from __future__ import annotations

import hashlib
from collections import deque
from dataclasses import dataclass, field

import torch

from . import ops
from .generation import GenerationArgs, as_int64, draw_seed, next_tokens, should_stop
from .kv_fp8 import resolve_cache_dtype
from .model.cambrian_arch import IMAGE_TOKEN_INDEX
from .paged_kv import DEFAULT_PAGE_SIZE, ROOT, PagedCacheView, PagedKVPool, check_page_size, pages_for


@dataclass
class _Request:
    rid: int
    ids: torch.Tensor               # [1, S] on the model's device
    images: object
    image_sizes: object
    kwargs: dict
    args: GenerationArgs
    reserve: int                    # pages reserved at admission
    pages: list = field(default_factory=list)
    table: torch.Tensor = None      # int32 [max_pages_per_seq] on the host
    tokens: list = field(default_factory=list)
    length: int = 0                 # cached positions
    pos: int = 0                    # position id of the next decode token
    # prefix cache (prefix_cache=True)
    host_ids: list = None           # the prompt ids on the host
    digest: bytes = None            # the image digest (None: no image, or an image the cache cannot key)
    content: list = None            # the prompt's position contents after the splice (None: not known)
    image_end: int = 0              # the first position after the image span (0: no image)
    prefix: int = 0                 # positions reused from the index at admission
    node: int = ROOT                # the index node of the request's leading indexed pages
    indexed: int = 0                # leading pages of the request that are in the index
    held: list = field(default_factory=list)   # index pages referenced in place of its own pages of equal contents


class BatchedGenerator:
    """Serve generation requests of one model at once over a paged KV cache (see the module docstring)."""

    def __init__(self, model, max_batch: int = 32, max_cached_tokens: int = 65536, page_size: int = DEFAULT_PAGE_SIZE,
                 kv_cache_dtype: str | None = None, use_graph: bool = True, prefix_cache: bool = False):
        from .model.language_model.cambrian_phi3 import CambrianPhi3ForCausalLM
        if isinstance(model, CambrianPhi3ForCausalLM):
            raise NotImplementedError("BatchedGenerator does not serve Cambrian-Phi3 yet: the paged decode kernel has no "
                                      "head_dim 96 and no sliding window")
        if getattr(model.get_model(), "_zero3", None) is not None:
            raise NotImplementedError("BatchedGenerator does not serve a model sharded by Zero3Inference")
        if not 1 <= int(max_batch) <= 1024:
            raise ValueError(f"max_batch={max_batch} must be in [1, 1024]")
        cfg = model.config
        self.model = model
        self.kv_dtype = resolve_cache_dtype(cfg, kv_cache_dtype)
        self.page_size = check_page_size(page_size)
        self.max_batch = int(max_batch)
        dev = model.lm_head.weight.device
        self.device = dev
        num_pages = pages_for(max_cached_tokens, self.page_size)
        self.max_pos = int(cfg.max_position_embeddings)
        mpps = max(1, min(num_pages, pages_for(self.max_pos, self.page_size)))
        self.pool = PagedKVPool(cfg, num_pages, self.page_size, self.kv_dtype, self.max_batch, mpps, dev)
        self.use_graph = bool(use_graph) and dev.type == "cuda"
        V, H = model.lm_head.weight.shape
        mb = self.max_batch
        self._tok = torch.zeros(mb, dtype=torch.long, device=dev)
        self._pos = torch.zeros((mb, 1), dtype=torch.long, device=dev)
        self._lens = torch.full((mb,), -1, dtype=torch.int32, device=dev)
        self._table = torch.zeros((mb, mpps), dtype=torch.int32, device=dev)
        self._logits = torch.zeros((mb, V), dtype=torch.float32, device=dev)
        # per-row sampling parameters (greedy and padding rows: T = 1, top_k = 1, top_p = 1), seed, step and pick
        self._temp = torch.ones(mb, dtype=torch.float32, device=dev)
        self._topk = torch.ones(mb, dtype=torch.int32, device=dev)
        self._topp = torch.ones(mb, dtype=torch.float32, device=dev)
        self._seed = torch.zeros(mb, dtype=torch.long, device=dev)
        self._step = torch.zeros(mb, dtype=torch.long, device=dev)
        self._sample = torch.zeros(mb, dtype=torch.bool, device=dev)
        self._drawn = torch.zeros(mb, dtype=torch.long, device=dev)
        self._next = torch.zeros(mb, dtype=torch.long, device=dev)
        self.buckets = sorted({min(1 << i, mb) for i in range(mb.bit_length() + 1)})
        self._graphs = {}
        self._graph_pool = torch.cuda.graph_pool_handle() if self.use_graph else None
        self._queue = deque()
        self._active: list[_Request] = []
        self._results = {}
        self._next_rid = 0
        self._dirty = True           # the row set changed since lens / pos / table / sampling rows were last uploaded
        q_num = int(getattr(cfg, "image_token_len", 576))
        self._image_extra = q_num + int(q_num ** 0.5) - 1
        self.prefix_cache = bool(prefix_cache)
        self.prompt_positions = 0    # prompt positions of the prefilled requests
        self.reused_positions = 0    # of those, positions taken from the prefix index instead of being prefilled

    # ------------------------------------------------------------------------------------------------ public API
    def nbytes(self) -> int:
        """Device bytes of the page pool (pages, scales, decode workspace)."""
        return self.pool.nbytes()

    def free_pages(self) -> int:
        return self.pool.free_pages()

    def cached_pages(self) -> int:
        """Pages in the prefix index (referenced or cached-idle)."""
        return self.pool.cached_pages()

    def hit_rate(self) -> float:
        """Prompt positions reused from the prefix index over all prompt positions prefilled so far."""
        return self.reused_positions / max(self.prompt_positions, 1)

    def pending(self) -> int:
        """Requests submitted and not finished (queued or running)."""
        return len(self._queue) + len(self._active)

    def submit(self, input_ids, images=None, image_sizes=None, **kwargs) -> int:
        """Queue one unpadded sequence (input_ids [S] or [1, S]) with the keywords of generate(); returns its id."""
        if "inputs_embeds" in kwargs:
            raise NotImplementedError("`inputs_embeds` is not supported")
        kv = kwargs.pop("kv_cache_dtype", None)
        if kv is not None and resolve_cache_dtype(self.model.config, kv) != self.kv_dtype:
            raise ValueError(f"kv_cache_dtype={kv!r}: this server keeps a {self.kv_dtype!r} page pool")
        mask = kwargs.pop("attention_mask", None)
        if mask is not None and not bool(mask.bool().all()):
            raise ValueError("submit() takes one unpadded sequence: attention_mask must be all ones")
        if kwargs.pop("position_ids", None) is not None:
            raise ValueError("submit() takes one unpadded sequence: its positions are 0 .. S-1")
        ids = input_ids.reshape(1, -1) if input_ids.dim() == 1 else input_ids
        if ids.dim() != 2 or ids.shape[0] != 1 or ids.shape[1] == 0:
            raise ValueError(f"submit() takes one sequence of token ids, got shape {tuple(input_ids.shape)}")
        bound = ids.shape[1] + (self._image_extra if images is not None else 0)
        args = GenerationArgs.from_kwargs(self.model, bound, kwargs)
        tokens = bound + args.max_new_tokens
        need = pages_for(tokens, self.page_size)
        if need > self.pool.num_pages or need > self.pool.max_pages_per_seq or tokens > self.max_pos:
            raise ValueError(f"a request of up to {bound} prompt positions and {args.max_new_tokens} new tokens needs "
                             f"{need} pages of {self.page_size}; the pool holds {self.pool.num_pages} pages, "
                             f"{self.pool.max_pages_per_seq} per sequence, positions up to {self.max_pos}")
        rid = self._next_rid
        self._next_rid += 1
        r = _Request(rid, ids.to(self.device), images, image_sizes, dict(kwargs), args, need)
        if self.prefix_cache:
            r.host_ids = ids[0].tolist()
            if images is not None:
                r.digest = _image_digest(images, image_sizes)
        self._queue.append(r)
        return rid

    @torch.no_grad()
    def step(self):
        """Admit and prefill what fits, then one decode step for every running request.  Returns a list of
        (rid, token, finished) in row order: first tokens of new requests, then one token per running request."""
        sync = getattr(self.model, "_cb_param_sync", None)
        if sync is not None:
            sync()      # a TrainEngine with deferred parameter sync: the kernels read parameters directly
        was_training = self.model.training
        self.model.eval()
        try:
            events = self._admit()
            if self._active:
                events += self._decode()
        finally:
            self.model.train(was_training)
        return events

    def run(self) -> dict:
        """Step until every submitted request has finished; returns {rid: LongTensor of its new ids} for the requests that
        finished since the last run()."""
        while self.pending():
            self.step()
        out, self._results = self._results, {}
        return out

    # ------------------------------------------------------------------------------------------------ internals
    def _admit(self):
        events = []
        while self._queue and len(self._active) < self.max_batch:
            r = self._queue[0]
            hit = self._match(r) if self.prefix_cache else None
            if hit is None:
                if self.pool.free_pages() < r.reserve:
                    break
                self._queue.popleft()
                r.pages = self.pool.alloc(r.reserve)
            else:
                shared, src, P, reserve = hit
                held = shared + ([src] if src is not None else [])
                # the matched pages are referenced before the allocation, so it cannot evict them
                if self.pool.free_pages() - self.pool.idle_among(held) < reserve:
                    break
                self._queue.popleft()
                self.pool.ref(held)
                r.pages = shared + self.pool.alloc(reserve)
                if src is not None:
                    self._copy_rows(src, r.pages[len(shared)], P % self.page_size)
                    self.pool.release([src])
                r.prefix, r.node, r.indexed = P, (shared[-1] if shared else ROOT), len(shared)
            try:
                events.append(self._prefill(r))
            except BaseException:
                # a request whose prefill fails (e.g. two <image> indicators) is dropped and its pages go back to the
                # pool; _prefill adds a request to the running rows only as its last step, so r is not running here
                self.pool.release(r.pages)
                r.pages = []
                raise
        return events

    # ---- prefix cache ----
    def _content(self, r: _Request):
        """The request's prompt position contents after the splice (token ids; the image digest over its span), or
        None while its image's span length is unknown or when the cache cannot key the request."""
        if r.content is not None or r.host_ids is None:
            return r.content
        ids = r.host_ids
        if r.images is None:
            r.content = list(ids)
            return r.content
        span = self.pool.image_span.get(r.digest) if r.digest is not None else None
        if span is None or ids.count(IMAGE_TOKEN_INDEX) != 1:
            return None
        p0 = ids.index(IMAGE_TOKEN_INDEX)
        cfg = self.model.config
        if not getattr(cfg, "connector_only", True) and p0 != getattr(cfg, "image_position", p0):
            return None         # the in-LLM SVA sites would rewrite positions outside the image span
        if (getattr(cfg, "inputs_pre_expanded", False)
                or (p0 + span <= len(ids) and not any(ids[p0 + 1:p0 + span]))):
            return None         # an already expanded span: the splice keeps the ids' length
        content = ids[:p0] + [r.digest] * span + ids[p0 + 1:]
        max_tok = getattr(cfg, "tokenizer_model_max_length", None)
        if max_tok is not None and len(content) > max_tok:
            return None         # the splice truncates
        r.content, r.image_end = content, p0 + span
        return content

    def _match(self, r: _Request):
        """(shared pages, partial source page or None, P, private pages to reserve) of the request's hit, or None."""
        C = self._content(r)
        if C is None:
            return None
        ps, S0 = self.page_size, len(C)
        full, part = self.pool.match(C)
        P = min(len(full) * ps + (part[1] if part is not None else 0), S0 - 1)
        if P <= 0 or P < r.image_end:
            return None         # no hit, or a hit that ends before the end of the image span
        nfull = P // ps
        src = None
        if P % ps:
            src = full[nfull] if nfull < len(full) else part[0]
        max_new = GenerationArgs.from_kwargs(self.model, S0, r.kwargs).max_new_tokens
        return full[:nfull], src, P, pages_for(S0 + max_new, ps) - nfull

    def _copy_rows(self, src: int, dst: int, rows: int):
        """The first `rows` positions of page src into page dst, in every layer (FP8: bytes and scales)."""
        for i in range(len(self.pool.k)):
            for t in self.pool.layer(i):
                if t is not None:
                    t[dst, :rows].copy_(t[src, :rows])

    def _index(self, r: _Request):
        """Index the request's pages whose positions are all written (prompt contents, then generated tokens)."""
        if r.content is None:
            return
        ps = self.page_size
        S0 = len(r.content)
        while (r.indexed + 1) * ps <= r.length:
            a, b = r.indexed * ps, (r.indexed + 1) * ps
            key = tuple(r.content[a:b] if b <= S0 else r.content[a:] + r.tokens[:b - S0])
            page = r.pages[r.indexed]
            r.node = self.pool.insert(r.node, key, page)
            if r.node != page:          # indexed already (by a request that prefilled the same prompt): hold that page
                self.pool.ref([r.node])
                r.held.append(r.node)
            r.indexed += 1

    def _learn(self, r: _Request, S0: int):
        """After a miss's prefill: learn its image's span length and its contents, if the cache can key it."""
        if r.host_ids is None or r.content is not None:
            return
        if r.digest is not None and r.digest not in self.pool.image_span and r.host_ids.count(IMAGE_TOKEN_INDEX) == 1:
            span = S0 - len(r.host_ids) + 1
            if span > 1:
                self.pool.image_span[r.digest] = span
        if self._content(r) is not None and len(r.content) != S0:
            r.content = None

    def _prefill(self, r: _Request):
        mpps = self.pool.max_pages_per_seq
        r.table = torch.zeros(mpps, dtype=torch.int32)
        r.table[:len(r.pages)] = torch.tensor(r.pages, dtype=torch.int32)
        table = r.table.view(1, mpps).to(self.device)
        view = PagedCacheView(self.pool, table, None, prefill=True, prefix=r.prefix)
        reserved = len(r.pages) * self.page_size

        def make_cache(B, S0, max_new):
            if S0 + max_new > reserved:
                raise RuntimeError(f"prefill of {S0} positions + {max_new} new tokens exceeds the {reserved} reserved")
            return view

        if r.prefix:
            # a hit covers any image span: the suffix is text only and runs without the towers
            suffix = torch.tensor([r.content[r.prefix:]], dtype=torch.long, device=self.device)
            args, _, h_last, next_pos, S0 = self.model._prefill(suffix, None, None, None, None, r.kwargs, make_cache,
                                                                prefix=r.prefix)
        else:
            args, _, h_last, next_pos, S0 = self.model._prefill(r.ids, r.images, r.image_sizes, None, None, r.kwargs,
                                                                make_cache)
        r.args = args
        keep = pages_for(S0 + args.max_new_tokens, self.page_size)
        if keep < len(r.pages):
            self.pool.release(r.pages[keep:])
            r.table[keep:] = 0
            r.pages = r.pages[:keep]
        r.length, r.pos = S0, int(next_pos.reshape(-1)[0])
        if self.prefix_cache:
            self._learn(r, S0)
            self._index(r)
            self.prompt_positions += S0
            self.reused_positions += r.prefix
        r.images = r.image_sizes = None
        if args.streamer is not None:
            args.streamer.put(torch.empty((1, 0), dtype=torch.long))     # HF streams the (here: empty) prompt ids first
        logits = ops.gemm(h_last, self.model.lm_head.weight, out_dtype=torch.float32)
        if args.do_sample:
            draw_seed(args, self.device)
        tok = int(next_tokens(logits, args)[0])
        finished = self._emit(r, tok, logits)
        if finished:
            self._retire(r)
        else:
            self._active.append(r)
            self._dirty = True
        return r.rid, tok, finished

    def _emit(self, r: _Request, tok: int, logits) -> bool:
        """Record and stream one token; True when the request is finished."""
        r.tokens.append(tok)
        a = r.args
        if a.streamer is not None:
            a.streamer.put(torch.tensor([tok], dtype=torch.long))
        done = len(r.tokens) >= a.max_new_tokens or tok in a.eos_token_ids
        if not done and a.stopping_criteria:
            gen = torch.tensor([r.tokens], dtype=torch.long, device=self.device)
            done = bool(should_stop(a, gen, logits, torch.zeros(1, dtype=torch.bool, device=self.device)).all())
        return done

    def _retire(self, r: _Request):
        self.pool.release(r.pages + r.held)
        r.pages, r.held = [], []
        if r.args.streamer is not None:
            r.args.streamer.end()
        self._results[r.rid] = torch.tensor(r.tokens, dtype=torch.long)

    def _bucket(self, n: int) -> int:
        return next(b for b in self.buckets if b >= n)

    def _decode_step(self, nb: int, sample: bool):
        """One decode step over rows [0, nb): embedding -> layers (paged attention) -> norm -> fp32 logits (with `sample`:
        then each row's token into _next, sampled or the argmax), then the active rows' lengths, positions and steps
        advance on the device.  Captured as the bucket's CUDA graph."""
        m = self.model
        view = PagedCacheView(self.pool, self._table[:nb], self._lens[:nb], prefill=False)
        out = m.model(input_ids=self._tok[:nb].view(nb, 1), position_ids=self._pos[:nb], past_key_values=view,
                      use_cache=True)
        logits = self._logits[:nb]
        ops.gemm(out.last_hidden_state.view(nb, -1), m.lm_head.weight, out=logits)
        live = self._lens[:nb] >= 0
        if sample:
            ops.sample_tokens(logits, self._temp[:nb], self._topk[:nb], self._topp[:nb], self._seed[:nb], self._step[:nb],
                              out=self._drawn[:nb])
            self._next[:nb].copy_(torch.where(self._sample[:nb], self._drawn[:nb], logits.argmax(-1)))
            self._step[:nb].add_(live.long())
        self._pos[:nb].add_(live.view(nb, 1).long())
        self._lens[:nb].add_(live.int())

    def _graph(self, nb: int, sample: bool):
        g = self._graphs.get((nb, sample))
        if g is None:
            state = (self._pos, self._lens, self._step)
            snap = tuple(t.clone() for t in state)
            side = torch.cuda.Stream(device=self.device)
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):            # warm-up outside capture (lazy kernel attributes, allocator)
                self._decode_step(nb, sample)
            torch.cuda.current_stream().wait_stream(side)
            # the warm-up advanced lens / pos / steps: rewind (its K / V rows are rewritten with the same values by the
            # replay)
            for t, t0 in zip(state, snap):
                t.copy_(t0)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=self._graph_pool):
                self._decode_step(nb, sample)
            for t, t0 in zip(state, snap):
                t.copy_(t0)
            self._graphs[(nb, sample)] = g
        return g

    def _decode(self):
        act = self._active
        n = len(act)
        nb = self._bucket(n)
        if self._dirty:
            mpps = self.pool.max_pages_per_seq
            lens = torch.full((nb,), -1, dtype=torch.int32)
            pos = torch.zeros((nb, 1), dtype=torch.long)
            table = torch.zeros((nb, mpps), dtype=torch.int32)
            temp, topk, topp = torch.ones(nb), torch.ones(nb, dtype=torch.int32), torch.ones(nb)
            seed, step = torch.zeros(nb, dtype=torch.long), torch.zeros(nb, dtype=torch.long)
            samp = torch.zeros(nb, dtype=torch.bool)
            for i, r in enumerate(act):
                lens[i], pos[i, 0], table[i] = r.length, r.pos, r.table
                a = r.args
                if a.do_sample:
                    temp[i], topk[i], topp[i] = a.temperature, min(a.top_k, (1 << 31) - 1), a.top_p
                    seed[i], step[i], samp[i] = as_int64(a.seed), len(r.tokens), True
            self._lens[:nb].copy_(lens)
            self._pos[:nb].copy_(pos)
            self._table[:nb].copy_(table)
            for buf, v in ((self._temp, temp), (self._topk, topk), (self._topp, topp), (self._seed, seed),
                           (self._step, step), (self._sample, samp)):
                buf[:nb].copy_(v)
            self._dirty = False
        self._tok[:nb].copy_(torch.tensor([r.tokens[-1] for r in act] + [0] * (nb - n), dtype=torch.long))
        sample = any(r.args.do_sample for r in act)
        if self.use_graph:
            self._graph(nb, sample).replay()
        else:
            self._decode_step(nb, sample)
        logits = self._logits[:n]
        toks = (self._next[:n] if sample else logits.argmax(-1)).tolist()
        events, keep = [], []
        for i, (r, tok) in enumerate(zip(act, toks)):
            r.length += 1
            r.pos += 1
            if self.prefix_cache:
                self._index(r)      # a page whose last position this step wrote
            finished = self._emit(r, tok, logits[i:i + 1])
            if finished:
                self._retire(r)
            else:
                keep.append(r)
            events.append((r.rid, tok, finished))
        if len(keep) != n:
            self._active = keep
            self._dirty = True
        return events


def _image_digest(images, image_sizes) -> bytes | None:
    """SHA-256 of the request's per-tower image tensors (host bytes, dtype, shape) and image_sizes; None when an image
    is not a tensor."""
    h = hashlib.sha256()
    for t in ([images] if torch.is_tensor(images) else list(images)):
        if not torch.is_tensor(t):
            return None
        t = t.detach().contiguous().cpu()
        h.update(repr((str(t.dtype), tuple(t.shape))).encode())
        h.update(t.view(torch.uint8).numpy().tobytes() if t.numel() else b"")
    h.update(repr(None if image_sizes is None else [tuple(int(x) for x in s) for s in image_sizes]).encode())
    return h.digest()
