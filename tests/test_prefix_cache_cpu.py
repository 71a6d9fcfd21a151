"""CPU checks of the server's prefix cache (BatchedGenerator(prefix_cache=True); paged_kv.py states the index): argument
validation of cb_paged_kv_gather, the prefix index and reference counts of the page pool, and the server end to end
over the plain-torch stand-ins (tests/ops_emulation.py, tests/paged_reference.py and the gather stand-in below) on the
peaked tiny model: multi-turn chat and several questions on one image, every request's tokens equal to solo generate()
and the fp32 oracle, the towers run once per distinct image.  The gather kernel itself is covered under `-m gpu`
(tests/test_prefix_cache_gpu.py)."""
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ops_emulation  # noqa: E402
import paged_reference as PR  # noqa: E402
from helpers import oracle_cfg, tiny_cambrian_config  # noqa: E402

needs_no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="kernel stand-ins are for GPU-less machines only")
PS = 16


def test_gather_argument_validation_without_gpu(lib):
    one = ctypes.c_void_p(16)                   # non-null, 16-byte aligned dummy pointer (never dereferenced)
    odd = ctypes.c_void_p(24)

    def gat(kp=one, out=one, table=one, fp8=0, ks=None, hd=64, ps=16, max_pages=4, P=10, ld=128):
        return lib.cb_paged_kv_gather(kp, one, ks, ks, fp8, table, 2, hd, ps, 8, max_pages, P, out, one, ld, None)

    for kw, msg in ((dict(kp=None), b"null"), (dict(out=None), b"null"), (dict(table=None), b"null"),
                    (dict(fp8=1), b"null"), (dict(hd=96, ld=192), b"hd"), (dict(ps=24), b"page_size"),
                    (dict(ps=8), b"page_size"), (dict(P=65), b"outside"), (dict(P=-1), b"outside"),
                    (dict(kp=odd), b"aligned"), (dict(out=odd), b"aligned"), (dict(ld=120), b"stride"),
                    (dict(ld=132), b"stride"), (dict(max_pages=0), b"empty")):
        assert gat(**kw) == 1 and msg in lib.cb_last_error(), (kw, lib.cb_last_error())


# ------------------------------------------------------------------------------------------------ the index and pool
def _pool(num_pages=8):
    from cambrian_b200.paged_kv import PagedKVPool
    return PagedKVPool(tiny_cambrian_config(), num_pages, PS, "bf16", 2, 8, "cpu")


def _chain(pool, content, pages):
    """Index `pages` as the full pages of `content` (what the server does once their positions are written)."""
    from cambrian_b200.paged_kv import ROOT
    node = ROOT
    for i, p in enumerate(pages):
        node = pool.insert(node, tuple(content[i * PS:(i + 1) * PS]), p)
    return node


def test_index_matches_exact_keys_at_page_and_position_granularity():
    pool = _pool()
    a = list(range(100, 148))                                       # 48 positions: three full pages
    pages = pool.alloc(3)
    assert _chain(pool, a, pages) == pages[-1] and pool.cached_pages() == 3
    # a prefix that shares 2 whole pages and 5 rows of the third
    b = a[:37] + [7] * 20
    full, part = pool.match(b)
    assert full == pages[:2] and part == (pages[2], 5)
    # whole pages only: the rest shares nothing
    full, part = pool.match(a[:32] + [9] * 3)
    assert full == pages[:2] and part is None
    # a difference in the first page: no whole page, the longest partial row match of the root's children
    full, part = pool.match(a[:3] + [1] + a[4:])
    assert full == [] and part == (pages[0], 3)
    # keys are exact contents: the same tokens under another parent do not match, and ints never equal a digest
    assert pool.match(a[16:32] + a[16:32]) == ([], None)
    d = b"\x01" * 32
    assert pool.match([d] * 16) == ([], None)
    # contents already indexed under another page are not indexed twice: insert returns that page
    other = pool.alloc(1)
    from cambrian_b200.paged_kv import ROOT
    assert pool.insert(ROOT, tuple(a[:16]), other[0]) == pages[0] and pool.cached_pages() == 3
    pool.release(other)
    pool.release(pages)
    assert pool.free_pages() == pool.num_pages and pool.cached_pages() == 3


def test_reference_counts_and_lru_leaf_first_eviction():
    pool = _pool(6)
    a, b = list(range(200, 232)), list(range(300, 348))
    pa = pool.alloc(2)
    _chain(pool, a, pa)
    pb = pool.alloc(3)
    _chain(pool, b, pb)
    # a second request shares a's pages: one more reference each
    pool.ref(pa)
    pool.release(pa)                                                # the first one retires: still referenced
    assert pool.free_pages() == 1 and pool.idle_among(pa) == 0
    pool.release(pa)                                                # the sharer retires: a's pages become idle
    assert pool.free_pages() == 3 and pool.idle_among(pa) == 2
    pool.release(pb)
    assert pool.free_pages() == 6 and pool.cached_pages() == 5
    # free pages first, then idle leaves least recently released first: a's leaf, then a's root (now a leaf), then b's
    assert pool.alloc(1) == [5]
    got = pool.alloc(3)
    assert got == [pa[1], pa[0], pb[2]], got
    assert pool.cached_pages() == 2 and pool.match(b)[0] == pb[:2]
    assert pool.match(a) == ([], None)
    pool.release(got + [5])
    assert pool.free_pages() == 6
    # a referenced page is never evicted
    pool.ref(pb[:2])
    with pytest.raises(RuntimeError, match="pages requested"):
        pool.alloc(5)
    assert sorted(pool.alloc(4)) == sorted(set(range(6)) - set(pb[:2]))


# ------------------------------------------------------------------------------------------------ the server
def _peaked():
    from test_model_host_logic_cpu import _build
    cfg = tiny_cambrian_config()
    cfg.fused_lm_loss = True
    model = _build(cfg)
    with torch.no_grad():
        emb = model.get_model().embed_tokens.weight
        perm = torch.randperm(emb.shape[0], generator=torch.Generator().manual_seed(9))
        model.lm_head.weight.copy_(emb[perm] * 24.0)
        for n_, p in model.named_parameters():
            if ((n_.endswith("o_proj.weight") and "layers." in n_ and "vision_sampler" not in n_)
                    or n_.endswith("down_proj.weight")
                    or ("vision_sampler_layers" in n_ and n_.endswith("proj_out.linear_2.weight"))):
                p.mul_(0.4)
    return cfg, model.eval()


def paged_kv_gather(k_pages, v_pages, k_scales, v_scales, block_table_row, P, out_k, out_v):
    """CPU stand-in of ops.paged_kv_gather: PR.gather, FP8 rows as bf16(float(e4m3) * scale)."""
    ps = k_pages.shape[1]
    for pages, sc, out in ((k_pages, k_scales, out_k), (v_pages, v_scales, out_v)):
        rows = PR.gather(pages, block_table_row, P, ps)
        if sc is not None:
            rows = rows.float() * PR.gather(sc, block_table_row, P, ps)[..., None]
        out.view(-1, *out.shape[-2:])[:P].copy_(rows.to(torch.bfloat16))


class _Towers:
    """encode_images stand-in: fixed tower features per image (keyed by the image's fill value), counting calls."""

    def __init__(self, model, cfg):
        from test_model_host_logic_cpu import _tower_feats
        self.feats = {k: [f[:1] for f in _tower_feats(model, cfg, 2, 31 + k)] for k in range(3)}
        self.calls = []

    def images(self, k):
        return [torch.full((1, 3, 8, 8), float(k), dtype=torch.bfloat16) for _ in self.feats[0]]

    def __call__(self, model, imgs):
        k = int(imgs[0].flatten()[0])
        self.calls.append(k)
        return self.feats[k]


def _setup(monkeypatch):
    ops_emulation.install(monkeypatch)
    PR.install(monkeypatch)
    from cambrian_b200 import ops
    monkeypatch.setattr(ops, "paged_kv_gather", paged_kv_gather)
    cfg, model = _peaked()
    towers = _Towers(model, cfg)
    monkeypatch.setattr(type(model), "encode_images", lambda self, imgs: towers(self, imgs))
    return cfg, model, towers


def _tok(g, cfg, n):
    return torch.randint(3, cfg.vocab_size, (n,), generator=g)


def _image_prompt(cfg, sys_ids, question):
    """System text up to image_position, a bare <image> indicator, then the question."""
    return torch.cat([sys_ids[:cfg.image_position], torch.tensor([-200]), question])


def _expanded(cfg, ids):
    """The collator's form of a bare <image> prompt (the oracle's input): -200 then span - 1 zeros."""
    q = int(cfg.image_token_len ** 0.5)
    p0 = int((ids == -200).nonzero()[0, 0])
    return torch.cat([ids[:p0 + 1], torch.zeros(q * (q + 1) - 1, dtype=ids.dtype), ids[p0 + 1:]])


@needs_no_gpu
def test_image_rule_and_digest(monkeypatch):
    """A hit must cover the whole image span: a match that stops inside it gives a full prefill; a match across it with
    the same digest skips the towers; the same pixels with another image_sizes is another digest."""
    from cambrian_b200.serving import BatchedGenerator
    cfg, model, towers = _setup(monkeypatch)
    g = torch.Generator().manual_seed(3)
    sys_ids = _tok(g, cfg, cfg.image_position)
    srv = BatchedGenerator(model, max_batch=4, max_cached_tokens=40 * PS, page_size=PS, prefix_cache=True)
    span = cfg.image_token_len + int(cfg.image_token_len ** 0.5)
    end = cfg.image_position + span                                  # 25 at the tiny config
    img = dict(images=towers.images(0), image_sizes=[(56, 56)])
    # 27 prompt positions + 2 cached new tokens: only page 0 [0, 16) fills, and it ends inside the image span
    srv.submit(_image_prompt(cfg, sys_ids, _tok(g, cfg, 2)), max_new_tokens=3, eos_token_id=None, **img)
    srv.run()
    assert towers.calls == [0] and srv.pool.image_span and list(srv.pool.image_span.values()) == [span]
    assert srv.cached_pages() == 1
    srv.submit(_image_prompt(cfg, sys_ids, _tok(g, cfg, 12)), max_new_tokens=4, eos_token_id=None, **img)
    srv.run()
    assert towers.calls == [0, 0] and srv.reused_positions == 0, "a hit ending inside the image span"
    # the second request filled pages 0 and 1 [0, 32): a third request on the same image hits across the span
    q3 = _image_prompt(cfg, sys_ids, _tok(g, cfg, 9))
    r3 = srv.submit(q3, max_new_tokens=5, eos_token_id=None, **img)
    out = srv.run()
    assert towers.calls == [0, 0] and srv.reused_positions >= end
    assert out[r3].tolist() == model.generate(q3[None], max_new_tokens=5, eos_token_id=None, **img)[0].tolist()
    # another image_sizes (same pixels): another digest, so no hit and the towers run
    srv.submit(q3, max_new_tokens=2, eos_token_id=None, images=towers.images(0), image_sizes=[(60, 60)])
    before, calls = srv.reused_positions, len(towers.calls)
    srv.run()
    assert len(towers.calls) == calls + 1 and srv.reused_positions == before
    assert srv.free_pages() == srv.pool.num_pages and srv.pending() == 0


@needs_no_gpu
def test_admission_never_evicts_its_own_match(monkeypatch):
    from cambrian_b200.serving import BatchedGenerator
    cfg, model, towers = _setup(monkeypatch)
    g = torch.Generator().manual_seed(5)
    srv = BatchedGenerator(model, max_batch=2, max_cached_tokens=6 * PS, page_size=PS, prefix_cache=True)
    a, b = _tok(g, cfg, 40), _tok(g, cfg, 60)
    srv.submit(a, max_new_tokens=8, eos_token_id=None)              # 47 positions written: pages 0, 1 indexed
    srv.run()
    srv.submit(b, max_new_tokens=4, eos_token_id=None)              # 63 written: pages 0..2 indexed
    srv.run()
    assert srv.cached_pages() == 5 and srv.free_pages() == 6
    a_pages = srv.pool.match(a.tolist())[0]
    b_pages = srv.pool.match(b.tolist())[0]
    assert len(a_pages) == 2 and len(b_pages) == 3
    # a's first turn plus more: the hit is a's two pages (the least recently released idle ones); its 3 private pages
    # take the free page and evict b's two deepest pages, never its own
    c = torch.cat([a, _tok(g, cfg, 10)])
    rc = srv.submit(c, max_new_tokens=30, eos_token_id=None)            # 80 positions: 5 pages, 3 private
    srv.step()
    run = srv._active[0]
    assert run.rid == rc and run.pages[:2] == a_pages and run.prefix == 32
    assert srv.pool.match(b.tolist())[0] == b_pages[:1]
    out = srv.run()
    assert out[rc].tolist() == model.generate(c[None], max_new_tokens=30, eos_token_id=None)[0].tolist()
    assert srv.free_pages() == srv.pool.num_pages


@needs_no_gpu
@pytest.mark.parametrize("prefix_cache", [True, False])
def test_chat_and_shared_image_mix(monkeypatch, prefix_cache):
    """A three-turn conversation about image 1 and four questions on image 2, three of them submitted while the first is
    still decoding.  Every request's tokens equal solo generate() and the fp32 oracle; with the prefix cache the towers
    run once per distinct image, without it once per request, as before."""
    from test_parity_gpu import _oracle_greedy

    from cambrian_b200.serving import BatchedGenerator
    cfg, model, towers = _setup(monkeypatch)
    g = torch.Generator().manual_seed(11)
    sys_ids = _tok(g, cfg, cfg.image_position)
    srv = BatchedGenerator(model, max_batch=4, max_cached_tokens=64 * PS, page_size=PS, prefix_cache=prefix_cache)
    sd = {k: v.detach().float() for k, v in model.state_dict().items()}
    ocfg = oracle_cfg(cfg)
    served = []                                                    # (prompt, image key, max_new, tokens)

    # the conversation: each turn resends the previous turns and the answers
    conv = _image_prompt(cfg, sys_ids, _tok(g, cfg, 11))
    for turn in range(3):
        n = 7 + turn
        rid = srv.submit(conv, max_new_tokens=n, eos_token_id=None, images=towers.images(1), image_sizes=[(56, 56)])
        ans = srv.run()[rid]
        served.append((conv, 1, n, ans.tolist()))
        conv = torch.cat([conv, ans, _tok(g, cfg, 6 + 3 * turn)])
    # four questions on one image, three of them arriving while the first decodes
    qs = [_image_prompt(cfg, sys_ids, _tok(g, cfg, 8 + 5 * i)) for i in range(4)]
    news = [12, 6, 9, 5]
    img2 = dict(images=towers.images(2), image_sizes=[(56, 56)])
    rids = [srv.submit(qs[0], max_new_tokens=news[0], eos_token_id=None, **img2)]
    srv.step()
    srv.step()
    assert srv._active and srv._active[0].rid == rids[0]
    rids += [srv.submit(q, max_new_tokens=n, eos_token_id=None, **img2) for q, n in zip(qs[1:], news[1:])]
    outs = srv.run()
    served += [(q, 2, n, outs[r].tolist()) for q, n, r in zip(qs, news, rids)]

    if prefix_cache:
        assert towers.calls == [1, 2], towers.calls                 # once per distinct image
        assert 0 < srv.hit_rate() < 1 and srv.cached_pages() > 0
    else:
        assert towers.calls == [1] * 3 + [2] * 4
        assert srv.reused_positions == 0 and srv.cached_pages() == 0
    assert srv.free_pages() == srv.pool.num_pages and srv.pending() == 0
    towers.calls.clear()
    for ids, k, n, got in served:
        solo = model.generate(ids[None], max_new_tokens=n, eos_token_id=None, images=towers.images(k),
                              image_sizes=[(56, 56)])[0].tolist()
        assert got == solo, (got, solo)
        o, margins = _oracle_greedy(sd, cfg, ocfg, [f.float() for f in towers.feats[k]], _expanded(cfg, ids)[None], n,
                                    torch.float32, torch.device("cpu"))
        assert o == got, (o, got, margins)
