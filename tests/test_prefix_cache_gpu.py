"""GPU checks of the server's prefix cache (BatchedGenerator(prefix_cache=True)): the gather kernel bit for bit against
torch through shuffled block tables, the decoder layer's hit-path attention against an fp64 reference over the same
gathered rows (and against the miss path for bf16 pages), and the server end to end on the peaked tiny model for bf16
and FP8 pages: multi-turn chat and several questions on one image, served tokens equal to solo generate(), graph and
eager serving in agreement, a hit rate above 0, and every page free or evictable at idle."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import attention_reference as AR  # noqa: E402
import kv_fp8_reference as KR  # noqa: E402
import paged_reference as PR  # noqa: E402

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
bf = torch.bfloat16


def _pages(num_pages, ps, nkv, hd, fp8, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(2, num_pages, ps, nkv, hd, generator=g) * 2).to(bf)
    if not fp8:
        return x[0].to(dev), x[1].to(dev), None, None
    qk, sk = KR.quantize_rows(x[0].float())
    qv, sv = KR.quantize_rows(x[1].float())
    return qk.to(dev), qv.to(dev), sk.to(dev), sv.to(dev)


def _torch_gather(pages, scales, row, P):
    ps = pages.shape[1]
    rows = PR.gather(pages.cpu(), row.cpu(), P, ps)
    if scales is None:
        return rows
    return (rows.float() * PR.gather(scales.cpu(), row.cpu(), P, ps)[..., None]).to(bf)


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("ps", [16, 64])
def test_gather_bitwise_through_shuffled_tables(hd, fp8, ps):
    from cambrian_b200 import ops
    nkv, max_pages, num_pages = 8, 9, 23
    kp, vp, ks, vs = _pages(num_pages, ps, nkv, hd, fp8, hd + ps + fp8)
    row = torch.randperm(num_pages, generator=torch.Generator().manual_seed(ps))[:max_pages].to(torch.int32).to(dev)
    for P in (1, ps - 1, 3 * ps + 5, max_pages * ps - 3, max_pages * ps):
        n = 7
        ok = torch.full((1, P + n, nkv, hd), float("nan"), dtype=bf, device=dev)
        ov = ok.clone()
        ops.paged_kv_gather(kp, vp, ks, vs, row, P, ok, ov)
        for got, pages, sc in ((ok, kp, ks), (ov, vp, vs)):
            want = _torch_gather(pages, sc, row, P)
            assert torch.equal(got[0, :P].cpu().view(torch.int16), want.view(torch.int16)), (hd, fp8, ps, P)
            assert got[0, P:].isnan().all(), "rows past P were written"
    # P = 0 writes nothing
    ok = torch.full((1, 4, nkv, hd), float("nan"), dtype=bf, device=dev)
    ops.paged_kv_gather(kp, vp, ks, vs, row, 0, ok, ok.clone())
    assert ok.isnan().all()


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("hd", [64, 128])
def test_layer_hit_attention_against_fp64(fp8, hd):
    """A prefill of S0 positions as a miss (the flash kernel over its own K / V, appended to the pages), then the same
    prompt as a hit after P cached positions: the hit's attention output is the fp64 attention of its queries over the
    gathered prefix rows and its own bf16 rows, within the flash kernel's bound; for bf16 pages it equals the miss's
    output rows within the same bound."""
    from helpers import tiny_cambrian_config

    from cambrian_b200.model.language_model.cambrian_llama import CBLlamaDecoderLayer
    from cambrian_b200.paged_kv import PagedCacheView, PagedKVPool
    cfg = tiny_cambrian_config()
    cfg.num_attention_heads, cfg.num_key_value_heads = 8, 2
    cfg.hidden_size, cfg.head_dim = 8 * hd, hd
    layer = CBLlamaDecoderLayer(cfg, 0)
    ps, S0 = 16, 150
    pool = PagedKVPool(cfg, 24, ps, "fp8" if fp8 else "bf16", 1, 12, dev)
    table = torch.randperm(24, generator=torch.Generator().manual_seed(hd))[:12].to(torch.int32)[None].to(dev)
    g = torch.Generator().manual_seed(7 + hd)
    nh, nkv = 8, 2
    q = (torch.randn(1, S0, nh, hd, generator=g) * 1.5).to(bf).to(dev)
    k = (torch.randn(1, S0, nkv, hd, generator=g) * 1.5).to(bf).to(dev)
    v = torch.randn(1, S0, nkv, hd, generator=g).to(bf).to(dev)
    miss = layer._attn_paged_cache(q, k, v, PagedCacheView(pool, table, None, prefill=True), None)
    for P in (37, 64, 149):
        view = PagedCacheView(pool, table, None, prefill=True, prefix=P)
        hit = layer._attn_paged_cache(q[:, P:], k[:, P:], v[:, P:], view, None)
        kp, vp, ksc, vsc = pool.layer(0)
        kk = torch.cat([_torch_gather(kp, ksc, table[0], P).to(dev)[None], k[:, P:]], 1)
        vv = torch.cat([_torch_gather(vp, vsc, table[0], P).to(dev)[None], v[:, P:]], 1)
        assert torch.equal(view.kv_buf[0], kk) and torch.equal(view.kv_buf[1], vv)
        ref = AR.fwd_ref(q[:, P:], kk, vv, causal=True)
        err = (hit.double() - ref["o"]).abs()
        assert (err <= 2.0 ** -8 * ref["o"].abs() + ref["tol_o"]).all(), (fp8, hd, P, float(err.max()))
        if not fp8:
            # the same keys: the miss's rows P .. S0-1 differ from the hit's only in the kernel's tiling
            d = (hit.double() - miss[:, P:].double()).abs()
            assert (d <= 2.0 ** -7 * ref["o"].abs() + 2 * ref["tol_o"]).all(), (hd, P, float(d.max()))


# ------------------------------------------------------------------------------------------------ end to end
def _bare(cfg, p):
    """A collator-expanded prompt back to a bare <image> indicator (what a tokenizer produces)."""
    q = int(cfg.image_token_len ** 0.5)
    return torch.cat([p[:cfg.image_position + 1], p[cfg.image_position + q * (q + 1):]])


def _mix(cfg):
    """[(prompt, images kwargs, max_new, depends)]: four questions on image 0, three conversation turns on image 1 (turn
    t's prompt is turn t-1's prompt, its answer and a new question: `depends` is the index of the previous turn), and
    two text-only requests sharing a system prompt."""
    from test_modules_gpu import _tiny_batch
    ids, _, _, _, images, _ = _tiny_batch(cfg, B=2, S=96)
    g = torch.Generator().manual_seed(31)
    sys_ids = _bare(cfg, ids[0])[:cfg.image_position + 1]
    tok = lambda n: torch.randint(3, cfg.vocab_size, (n,), generator=g)  # noqa: E731
    img = [dict(images=[t[i:i + 1].to(dev).bfloat16() for t in images], image_sizes=[(56, 56)]) for i in (0, 1)]
    out = [(torch.cat([sys_ids, tok(9 + 4 * i)]), img[0], 6 + 3 * i, None) for i in range(4)]
    out += [(torch.cat([sys_ids, tok(12)]), img[1], 8, None), (tok(7), img[1], 7, 4), (tok(5), img[1], 9, 5)]
    text = tok(40)
    out += [(torch.cat([text, tok(6)]), {}, 10, None), (torch.cat([text, tok(11)]), {}, 5, None)]
    return out


def _prompt(mix, answers, i):
    """Request i's prompt: a later turn is its previous turn's prompt, that turn's answer and its own question."""
    p, _, _, dep = mix[i]
    return p if dep is None else torch.cat([_prompt(mix, answers, dep), torch.tensor(answers[dep]), p])


def _solo(model, mix, kv):
    answers = {}
    for i, (p, img, n, dep) in enumerate(mix):
        prompt = _prompt(mix, answers, i)
        answers[i] = model.generate(prompt[None].to(dev), max_new_tokens=n, eos_token_id=None, kv_cache_dtype=kv,
                                    **img)[0].tolist()
    return answers


def _serve(model, mix, kv, use_graph):
    """The mix through one server: the first three image-0 questions and the text requests arrive together, the fourth
    while they decode; each turn after its previous turn has finished."""
    from cambrian_b200.serving import BatchedGenerator
    srv = BatchedGenerator(model, max_batch=8, max_cached_tokens=4096, page_size=16, kv_cache_dtype=kv,
                           use_graph=use_graph, prefix_cache=True)
    answers, rid = {}, {}

    def submit(i):
        p, img, n, dep = mix[i]
        rid[i] = srv.submit(_prompt(mix, answers, i).to(dev), max_new_tokens=n, eos_token_id=None, **img)

    for i in (0, 1, 2, 4, 7, 8):
        submit(i)
    srv.step()
    srv.step()
    submit(3)
    for turn in (5, 6):
        out = srv.run()
        answers.update({i: out[r].tolist() for i, r in rid.items() if r in out})
        submit(turn)
    out = srv.run()
    answers.update({i: out[r].tolist() for i, r in rid.items() if r in out})
    assert srv.pending() == 0 and srv.free_pages() == srv.pool.num_pages, "a page is neither free nor evictable at idle"
    return answers, srv


@pytest.mark.parametrize("kv", ["bf16", "fp8"])
def test_served_with_prefix_cache_matches_solo_generate(kv):
    from test_fp8_gpu import _peaked_model
    cfg, model = _peaked_model()
    mix = _mix(cfg)
    calls = []
    inner = type(model).encode_images

    def encode(self, imgs):
        calls.append(1)
        return inner(self, imgs)

    solo = _solo(model, mix, kv)
    type(model).encode_images = encode
    try:
        graph, srv = _serve(model, mix, kv, use_graph=True)
        towers = len(calls)
        eager, _ = _serve(model, mix, kv, use_graph=False)
    finally:
        type(model).encode_images = inner
    assert graph == eager, "graph and eager serving differ"
    for i in range(len(mix)):
        assert graph[i] == solo[i], (i, graph[i], solo[i])
    assert towers == 2, f"the towers ran {towers} times for two distinct images"
    assert srv.hit_rate() > 0 and srv.reused_positions > 0 and srv.cached_pages() > 0
