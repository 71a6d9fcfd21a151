"""CPU checks of continuous batching over the paged KV cache (cambrian_b200/serving.py, paged_kv.py): argument validation
of the two entry points, the page allocator and FIFO admission, the refusals, and the whole server over the plain-torch
stand-ins of tests/paged_reference.py on the peaked tiny model — every request's tokens equal its solo generate() and the
fp32 oracle's.  The kernels' numerics are covered under `-m gpu` (tests/test_paged_gpu.py)."""
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


def test_entry_point_argument_validation_without_gpu(lib):
    one = ctypes.c_void_p(16)                                   # non-null, 16-byte aligned dummy pointer (never dereferenced)
    odd = ctypes.c_void_p(24)
    f = ctypes.c_float(0.125)

    def dec(q=one, q_bs=512, rows=2, nh=4, nkv=2, hd=64, ps=64, num_pages=8, max_pages=4, table_ld=4, lens=one,
            table=one, fp8=0, ks=None, len_add=1, ws_floats=1 << 20):
        return lib.cb_attn_decode_paged(q, q_bs, one, one, ks, ks, fp8, table, table_ld, lens, len_add, one, one,
                                        ws_floats, rows, nh, nkv, hd, ps, num_pages, max_pages, f, None)

    for kw, msg in ((dict(q=None), b"null"), (dict(lens=None), b"null"), (dict(table=None), b"null"),
                    (dict(fp8=1), b"null"), (dict(hd=96), b"hd"), (dict(nh=32, nkv=2), b"nh"), (dict(nh=6, nkv=4), b"nh"),
                    (dict(ps=48), b"page_size"), (dict(ps=8), b"page_size"), (dict(table_ld=3), b"stride"),
                    (dict(num_pages=0), b"empty"), (dict(max_pages=0), b"empty"), (dict(rows=0), b"shape"),
                    (dict(q=odd), b"aligned"), (dict(q_bs=516), b"aligned"), (dict(len_add=-1), b"len_add"),
                    (dict(ws_floats=10), b"workspace")):
        assert dec(**kw) == 1 and msg in lib.cb_last_error(), (kw, lib.cb_last_error())
    # workspace: rows * nh * ceil(max_pages * page_size / 256) * (hd + 2), independent of the device
    assert lib.cb_attn_decode_paged_workspace_floats(32, 32, 128, 64, 128) == 32 * 32 * 32 * 130
    assert lib.cb_attn_decode_paged_workspace_floats(1, 4, 1, 16, 64) == 4 * 66
    assert lib.cb_attn_decode_paged_workspace_floats(0, 4, 1, 16, 64) == 0

    def app(k=one, ld=256, S=1, hd=64, ps=64, max_pages=2, table_ld=2, lens=None, offset=0, from_lens=0, fp8=0, ks=None,
            table=one):
        return lib.cb_paged_kv_append(k, one, ld, one, one, ks, ks, fp8, table, table_ld, lens, 1, S, 2, hd, ps, 4,
                                      max_pages, offset, from_lens, None)

    for kw, msg in ((dict(k=None), b"null"), (dict(table=None), b"null"), (dict(fp8=1), b"null"),
                    (dict(from_lens=1), b"lens"), (dict(hd=128, ld=128), b"stride"), (dict(hd=80), b"hd"),
                    (dict(ps=100), b"page_size"), (dict(k=odd), b"aligned"), (dict(ld=100), b"stride"),
                    (dict(S=4, offset=126), b"outside"), (dict(table_ld=1), b"stride"), (dict(S=0), b"S=")):
        assert app(**kw) == 1 and msg in lib.cb_last_error(), (kw, lib.cb_last_error())


def test_format_arithmetic():
    from cambrian_b200 import paged_kv
    cfg = tiny_cambrian_config()
    L, nkv, hd = cfg.num_hidden_layers, cfg.num_key_value_heads, cfg.hidden_size // cfg.num_attention_heads
    assert paged_kv.bytes_per_token(cfg, "bf16") == L * 2 * nkv * hd * 2
    assert paged_kv.bytes_per_token(cfg, "fp8") == L * 2 * nkv * (hd + 4)
    from cambrian_b200 import kv_fp8
    assert paged_kv.bytes_per_token(cfg, "fp8") == kv_fp8.bytes_per_token(cfg)
    assert [paged_kv.pages_for(n, 16) for n in (0, 1, 16, 17, 32)] == [0, 1, 1, 2, 2]
    for bad in (0, 8, 48, 100):
        with pytest.raises(ValueError, match="page_size"):
            paged_kv.check_page_size(bad)
    with pytest.raises(ValueError, match="kv_cache_dtype"):
        paged_kv.bytes_per_token(cfg, "int8")


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


def _setup(monkeypatch):
    from test_model_host_logic_cpu import _batch, _tower_feats
    ops_emulation.install(monkeypatch)
    PR.install(monkeypatch)
    cfg, model = _peaked()
    ids = _batch(cfg, B=8, S=96)[0]
    feats = [f[:1] for f in _tower_feats(model, cfg, 2, 31)]
    monkeypatch.setattr(type(model), "encode_images", lambda self, imgs: feats)
    images = [torch.zeros(1, 3, 8, 8, dtype=torch.bfloat16) for _ in feats]
    return cfg, model, ids, feats, images


@needs_no_gpu
def test_allocator_and_fifo_admission(monkeypatch):
    from cambrian_b200.serving import BatchedGenerator
    cfg, model, ids, feats, images = _setup(monkeypatch)
    ps = 16
    srv = BatchedGenerator(model, max_batch=2, max_cached_tokens=6 * ps, page_size=ps)
    total = srv.free_pages()
    from cambrian_b200.paged_kv import bytes_per_token
    assert total == 6 and srv.nbytes() >= 6 * ps * bytes_per_token(cfg)
    # text-only prompts: the reservation is exactly ceil((S + max_new) / page_size)
    r0 = srv.submit(ids[0, 30:50].clamp(min=3), max_new_tokens=12, eos_token_id=None)          # 32 tokens -> 2 pages
    r1 = srv.submit(ids[1, 30:47].clamp(min=3), max_new_tokens=16, eos_token_id=None)          # 33 tokens -> 3 pages
    r2 = srv.submit(ids[2, 30:40].clamp(min=3), max_new_tokens=6, eos_token_id=None)           # 16 tokens -> 1 page
    assert [r.reserve for r in srv._queue] == [2, 3, 1]
    ev = srv.step()
    # max_batch = 2: r0 and r1 run; r2 fits the pool but waits for a row (FIFO, no overtaking)
    assert [e[0] for e in ev] == [r0, r1, r0, r1] and srv.free_pages() == total - 5 and len(srv._queue) == 1
    seen_pages = set(srv._active[0].pages) | set(srv._active[1].pages)
    while srv._active and all(r.rid != r2 for r in srv._active):
        srv.step()
    # r0 retired (12 tokens) first: its pages went back and r2 took the lowest free one
    assert srv._active[0].rid == r1 and srv._active[1].rid == r2 and set(srv._active[1].pages) <= seen_pages
    outs = srv.run()
    assert sorted(outs) == [r0, r1, r2] and [len(outs[r]) for r in (r0, r1, r2)] == [12, 16, 6]
    assert srv.free_pages() == total and srv.pending() == 0                 # idle: every page is free
    # a request that can never fit: more pages than the pool holds
    with pytest.raises(ValueError, match="pages"):
        srv.submit(ids[0, 30:50].clamp(min=3), max_new_tokens=90)
    # a bare <image> indicator reserves for its expansion (image_token_len + sqrt(image_token_len) - 1 extra positions)
    img_ids = torch.cat([ids[0, :5], torch.tensor([-200]), ids[0, 40:50]]).clamp(min=-200)
    rid = srv.submit(img_ids, images=images, image_sizes=[(56, 56)], max_new_tokens=8)
    assert srv._queue[-1].reserve == -(-(16 + 19 + 8) // ps)
    srv.step()
    assert srv._active[0].rid == rid and len(srv._active[0].pages) == -(-(16 + 19 + 8) // ps)  # 35 positions after splice
    srv.run()
    assert srv.free_pages() == total


@needs_no_gpu
def test_failed_prefill_returns_its_pages(monkeypatch):
    """A request whose prefill raises (two <image> indicators, refused by the multimodal preparation) is dropped with the
    prefill's exception; its pages go back to the pool and the requests around it are served."""
    from cambrian_b200.serving import BatchedGenerator
    cfg, model, ids, feats, images = _setup(monkeypatch)
    srv = BatchedGenerator(model, max_batch=2, max_cached_tokens=8 * 16, page_size=16)
    total = srv.free_pages()
    ok = srv.submit(ids[0, 30:50].clamp(min=3), max_new_tokens=4, eos_token_id=None)
    two = torch.cat([ids[0, :5], torch.tensor([-200]), ids[0, 40:44], torch.tensor([-200]), ids[0, 50:54]])
    srv.submit(two, images=images, image_sizes=[(56, 56)], max_new_tokens=4)
    after = srv.submit(ids[1, 30:46].clamp(min=3), max_new_tokens=5, eos_token_id=None)
    with pytest.raises(NotImplementedError, match="one image"):
        srv.step()
    assert srv.free_pages() == total - srv._active[0].reserve and [r.rid for r in srv._active] == [ok]
    outs = srv.run()
    assert sorted(outs) == [ok, after] and len(outs[ok]) == 4 and len(outs[after]) == 5
    assert srv.free_pages() == total and srv.pending() == 0


@needs_no_gpu
def test_refusals(monkeypatch):
    from cambrian_b200.model.language_model.cambrian_phi3 import CambrianPhi3ForCausalLM
    from cambrian_b200.serving import BatchedGenerator
    cfg, model, ids, feats, images = _setup(monkeypatch)
    with pytest.raises(NotImplementedError, match="Phi3"):
        BatchedGenerator(CambrianPhi3ForCausalLM.__new__(CambrianPhi3ForCausalLM))
    model.get_model()._zero3 = object()
    with pytest.raises(NotImplementedError, match="Zero3Inference"):
        BatchedGenerator(model)
    del model.get_model()._zero3
    with pytest.raises(ValueError, match="kv_cache_dtype"):
        BatchedGenerator(model, kv_cache_dtype="int4")
    with pytest.raises(ValueError, match="page_size"):
        BatchedGenerator(model, page_size=24)
    srv = BatchedGenerator(model, max_batch=2, max_cached_tokens=256, page_size=16)
    p = ids[0, 30:40].clamp(min=3)
    for kw, exc, name in ((dict(num_beams=2), NotImplementedError, "num_beams"),
                          (dict(repetition_penalty=1.3), NotImplementedError, "repetition_penalty"),
                          (dict(cache_implementation="quantized"), NotImplementedError, "cache_implementation"),
                          (dict(no_such_keyword=1), TypeError, "no_such_keyword"),
                          (dict(inputs_embeds=torch.zeros(1)), NotImplementedError, "inputs_embeds")):
        with pytest.raises(exc, match=name):
            model.generate(p[None], max_new_tokens=2, **kw)
        with pytest.raises(exc, match=name):
            srv.submit(p, max_new_tokens=2, **kw)
    with pytest.raises(ValueError, match="unpadded"):
        srv.submit(p, attention_mask=torch.tensor([0] + [1] * 9))
    with pytest.raises(ValueError, match="one sequence"):
        srv.submit(torch.stack([p, p]))
    assert srv.pending() == 0


@needs_no_gpu
def test_served_tokens_equal_solo_generate_and_the_oracle(monkeypatch):
    """Seven requests with different prompt lengths, submitted between steps into a server of four rows: one stops at an
    EOS, one by a stopping criterion, the rest at max_new_tokens.  Tokens equal solo generate() and the fp32 oracle."""
    from test_parity_gpu import _oracle_greedy

    from cambrian_b200.serving import BatchedGenerator
    cfg, model, ids, feats, images = _setup(monkeypatch)
    lens = [40, 33, 52, 27, 45, 38, 60]
    news = [12, 7, 10, 12, 5, 9, 6]
    prompts = [ids[i % ids.shape[0], :n].clone() for i, n in enumerate(lens)]
    img = dict(images=images, image_sizes=[(56, 56)])
    solo = [model.generate(p[None], max_new_tokens=n, do_sample=False, **img)[0].tolist() for p, n in zip(prompts, news)]
    sd = {k: v.detach().float() for k, v in model.state_dict().items()}
    ocfg = oracle_cfg(cfg)
    for p, n, want in zip(prompts, news, solo):
        o, margins = _oracle_greedy(sd, cfg, ocfg, [f.float() for f in feats], p[None], n, torch.float32,
                                    torch.device("cpu"))
        assert o[:len(want)] == want, (want, o, margins)
    # request 1 stops at an EOS (its 4th token, absent before), request 4 by a stopping criterion after 3 tokens
    k = next(i for i in range(2, len(solo[1])) if solo[1][i] not in solo[1][:i])
    kw = [dict() for _ in prompts]
    kw[1]["eos_token_id"] = solo[1][k]
    kw[4]["stopping_criteria"] = [lambda toks, scores: toks.shape[1] >= 3]
    want = [s[:k + 1] if i == 1 else s[:3] if i == 4 else s for i, s in enumerate(solo)]
    assert model.generate(prompts[1][None], max_new_tokens=news[1], **img, **kw[1])[0].tolist() == want[1]

    streamed = []

    class Streamer:
        def put(self, t):
            streamed.append(t.tolist())

        def end(self):
            streamed.append("end")

    kw[0]["streamer"] = Streamer()
    srv = BatchedGenerator(model, max_batch=4, max_cached_tokens=64 * 16, page_size=16)
    total = srv.free_pages()
    rid = [srv.submit(prompts[i], max_new_tokens=news[i], **img, **kw[i]) for i in range(3)]
    got = {}
    rows_seen = []

    def step():
        for r, t, fin in srv.step():
            got.setdefault(r, []).append(t)
        rows_seen.append([r.rid for r in srv._active])
        n = len(srv._active)
        if n and not srv._dirty:
            # packed rows [0, n): lens mirror each running request's cached length (the stand-ins run eagerly)
            assert srv._lens[:n].tolist() == [r.length for r in srv._active]

    step()
    rid += [srv.submit(prompts[i], max_new_tokens=news[i], **img, **kw[i]) for i in (3, 4)]
    step()
    step()
    rid += [srv.submit(prompts[i], max_new_tokens=news[i], **img, **kw[i]) for i in (5, 6)]
    while srv.pending():
        step()
    outs = srv.run()
    assert sorted(outs) == sorted(rid)
    for i, r in enumerate(rid):
        assert outs[r].tolist() == want[i] == got[r], (i, outs[r].tolist(), want[i], got[r])
    assert streamed == [[[]]] + [[t] for t in want[0]] + ["end"]
    assert max(len(r) for r in rows_seen) == 4                               # the row limit was reached
    # compaction: a retired request's row is taken by the next one, the others keep their order
    for a, b in zip(rows_seen, rows_seen[1:]):
        kept = [r for r in a if r in b]
        assert b[:len(kept)] == kept, (a, b)
    assert srv.free_pages() == total
