"""GPU checks of the paged KV cache and continuous batching: the append kernel bit for bit (bf16 copy; FP8 against
cb_kv_fp8_append) through shuffled block tables, decode attention against the fp64 reference of tests/paged_reference.py
at hd 64 / 128, G 1 / 4 / 7 / 8 and ragged lengths up to 16k, its run-to-run determinism and batch invariance, and the
server end to end on the peaked tiny model against solo generate()."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import kv_fp8_reference as KR  # noqa: E402
import paged_reference as PR  # noqa: E402
from helpers import ParityCollector  # noqa: E402

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
bf, f8 = torch.bfloat16, torch.float8_e4m3fn


def _pool(num_pages, ps, nkv, hd, fp8):
    shape = (num_pages, ps, nkv, hd)
    if fp8:
        kp = torch.full(shape, 0x7F, dtype=torch.uint8, device=dev).view(f8)     # NaN sentinels: untouched cells stay NaN
        vp = kp.clone()
        ks = torch.full(shape[:3], float("nan"), device=dev)
        return kp, vp, ks, ks.clone()
    kp = torch.full(shape, float("nan"), dtype=bf, device=dev)
    return kp, kp.clone(), None, None


def _tables(counts, max_pages, num_pages, seed):
    """Row b gets counts[b] distinct pages of a shuffled pool (block tables neither contiguous nor ordered); the entries
    past them hold other rows' pages, which the kernels must never touch."""
    perm = torch.randperm(num_pages, generator=torch.Generator().manual_seed(seed))
    table = torch.zeros(len(counts), max_pages, dtype=torch.int32)
    o = 0
    for b, c in enumerate(counts):
        table[b, :c] = perm[o:o + c]
        o += c
        table[b, c:] = perm[(o + torch.arange(max_pages - c)) % num_pages]
    return table


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("fp8", [False, True])
def test_append_bitwise_through_shuffled_tables(hd, fp8):
    from cambrian_b200 import ops
    rows, S, nh, nkv, ps = 3, 37, 4, 2, 16
    max_pages, num_pages = 6, 24
    g = torch.Generator().manual_seed(hd + fp8)
    qkv = (torch.randn(rows, S, (nh + 2 * nkv) * hd, generator=g) * 3).to(bf).to(dev)     # packed post-RoPE rows
    k = qkv[..., nh * hd:(nh + nkv) * hd].view(rows, S, nkv, hd)
    v = qkv[..., (nh + nkv) * hd:].view(rows, S, nkv, hd)
    table = _tables([max_pages] * rows, max_pages, num_pages, 1).to(dev)
    kp, vp, ks, vs = _pool(num_pages, ps, nkv, hd, fp8)
    # a prefill of S rows at host offset 0, then two decode tokens at lens[b]; row 1 is inactive for the second token
    ops.paged_kv_append(k, v, kp, vp, ks, vs, table, offset=0)
    lens = torch.tensor([S, S, S], dtype=torch.int32, device=dev)
    step = [qkv[:, i:i + 1] for i in range(2)]
    for i, st in enumerate(step):
        if i == 1:
            lens[1] = -1
        ops.paged_kv_append(st[..., nh * hd:(nh + nkv) * hd].view(rows, 1, nkv, hd),
                            st[..., (nh + nkv) * hd:].view(rows, 1, nkv, hd), kp, vp, ks, vs, table, lens,
                            offset_from_lens=True)
        lens += (lens >= 0).int()
    want_k = [torch.cat([k[b], k[b, :1], k[b, 1:2]]) if b != 1 else torch.cat([k[b], k[b, :1]]) for b in range(rows)]
    want_v = [torch.cat([v[b], v[b, :1], v[b, 1:2]]) if b != 1 else torch.cat([v[b], v[b, :1]]) for b in range(rows)]
    if fp8:
        # the dense FP8 cache's append of the same rows: bytes and scales bit for bit
        L = S + 2
        dk = torch.zeros(rows, L, nkv, hd, dtype=f8, device=dev)
        dv, dks, dvs = dk.clone(), torch.zeros(rows, L, nkv, device=dev), torch.zeros(rows, L, nkv, device=dev)
        wk = torch.stack([torch.cat([w, w[:1]]) if w.shape[0] < L else w for w in want_k])
        wv = torch.stack([torch.cat([w, w[:1]]) if w.shape[0] < L else w for w in want_v])
        ops.kv_fp8_append(wk.contiguous(), wv.contiguous(), dk, dv, dks, dvs, offset=0)
    for b in range(rows):
        n = want_k[b].shape[0]
        gk, gv = (PR.gather(t.cpu(), table[b].cpu(), n, ps) for t in (kp, vp))
        if fp8:
            gks, gvs = (PR.gather(t.cpu(), table[b].cpu(), n, ps) for t in (ks, vs))
            assert torch.equal(gk.view(torch.uint8), dk[b, :n].cpu().view(torch.uint8)), f"row {b}: K bytes"
            assert torch.equal(gv.view(torch.uint8), dv[b, :n].cpu().view(torch.uint8)), f"row {b}: V bytes"
            assert torch.equal(gks, dks[b, :n].cpu()) and torch.equal(gvs, dvs[b, :n].cpu()), f"row {b}: scales"
        else:
            assert torch.equal(gk.view(torch.int16), want_k[b].cpu().view(torch.int16)), f"row {b}: K"
            assert torch.equal(gv.view(torch.int16), want_v[b].cpu().view(torch.int16)), f"row {b}: V"
    # the inactive row wrote nothing past its first decode token; nothing outside the tables was touched
    used = set(table.flatten().tolist())
    nan_cells = (ks.isnan() if fp8 else kp.isnan().any(-1)).any(-1).cpu()             # [num_pages, ps]
    for p in range(num_pages):
        if p not in used:
            assert nan_cells[p].all(), f"page {p} outside every table was written"
    p1 = int(table[1, (S + 1) // ps])
    assert nan_cells[p1, (S + 1) % ps], "an inactive row wrote its token"


def _decode_case(hd, G, fp8, lengths, ps=64, nkv=2, seed=0):
    """Pages filled for ragged lengths (a shuffled table per row), a query per row: (q, pool, table, lens)."""
    rows = len(lengths)
    nh = G * nkv
    counts = [max(0, -(-(L + 1) // ps)) for L in lengths]          # room for lens + 1 positions
    max_pages = max(counts)
    num_pages = sum(counts) + 3
    g = torch.Generator().manual_seed(seed)
    table = _tables(counts, max_pages, num_pages, seed + 1)
    x = torch.randn(2, num_pages, ps, nkv, hd, generator=g).to(bf)
    x[1] *= 2.5
    if fp8:
        qk, sk = KR.quantize_rows(x[0].float())
        qv, sv = KR.quantize_rows(x[1].float())
        pool = (qk.to(dev), qv.to(dev), sk.to(dev), sv.to(dev))
    else:
        pool = (x[0].to(dev), x[1].to(dev), None, None)
    q = (torch.randn(rows, 1, nh, hd, generator=g) * 1.5).to(bf).to(dev)
    lens = torch.tensor(lengths, dtype=torch.int32)
    return q, pool, table.to(dev), lens.to(dev)


LENGTHS = [0, 1, 63, 64, 65, 255, 256, 257, 511, 1000, 16384]


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("G", [1, 4, 7, 8])
@pytest.mark.parametrize("fp8", [False, True])
def test_decode_against_fp64(hd, G, fp8):
    from cambrian_b200 import ops
    lengths = LENGTHS + [-1]                                                # and one inactive row
    q, (kp, vp, ks, vs), table, lens = _decode_case(hd, G, fp8, lengths, seed=hd + G)
    rows, nh = q.shape[0], q.shape[2]
    ws = ops.attn_decode_paged_workspace(rows, nh, table.shape[1], kp.shape[1], hd, dev)
    got = ops.attn_decode_paged(q, kp, vp, ks, vs, table, lens, ws, len_add=0)
    again = ops.attn_decode_paged(q, kp, vp, ks, vs, table, lens, ws, len_add=0)
    what = f"paged decode hd={hd} G={G} fp8={fp8}"
    assert torch.equal(got, again), what + ": not deterministic"
    assert torch.isfinite(got).all()
    assert not got[0].any() and not got[-1].any(), what + ": empty / inactive rows must be zero"
    ref = PR.decode_attention(q[:, 0], kp, vp, ks, vs, table, lens, len_add=0)
    eag = PR.decode_attention(q[:, 0], kp, vp, ks, vs, table, lens, len_add=0, dtype=bf)
    pc = ParityCollector()
    for b, L in enumerate(lengths):
        if L > 0:
            pc.check(got[b, 0].float(), ref[b], eag[b].float(), f"{what} L={L}")
    pc.done()


@pytest.mark.parametrize("fp8", [False, True])
def test_decode_is_batch_invariant(fp8):
    """One sequence alone equals the same sequence inside a batch of 32 rows (other pages, padding rows, a wider table)
    bit for bit."""
    from cambrian_b200 import ops
    hd, G = 128, 4
    lengths = [700, 3, 1500, 64, 257] * 6 + [-1, -1]
    q, (kp, vp, ks, vs), table, lens = _decode_case(hd, G, fp8, lengths, seed=11)
    rows, nh = q.shape[0], q.shape[2]
    ws = ops.attn_decode_paged_workspace(rows, nh, table.shape[1], kp.shape[1], hd, dev)
    batch = ops.attn_decode_paged(q, kp, vp, ks, vs, table, lens, ws, len_add=1)
    for b in (0, 2, 3, 29):
        n = -(-(int(lens[b]) + 1) // kp.shape[1])
        t1 = table[b:b + 1, :n].contiguous()
        ws1 = ops.attn_decode_paged_workspace(1, nh, n, kp.shape[1], hd, dev)
        alone = ops.attn_decode_paged(q[b:b + 1].contiguous(), kp, vp, ks, vs, t1, lens[b:b + 1].contiguous(), ws1,
                                      len_add=1)
        assert torch.equal(alone, batch[b:b + 1]), f"row {b} alone != in the batch"


# ------------------------------------------------------------------------------------------------ end to end
def _requests(cfg, n=12):
    """n prompts of mixed length: even ones carry an image (the 4th a non-square one, through the dynamic branch)."""
    from test_modules_gpu import _tiny_batch
    ids, _, _, _, images, _ = _tiny_batch(cfg, B=2, S=96)
    g = torch.Generator().manual_seed(21)
    reqs = []
    for i in range(n):
        L = 30 + 7 * i % 50
        if i % 2 == 0:
            p = ids[i % 2, :max(L, 30)].clone()
            img = [t[i % 2:i % 2 + 1].to(dev).bfloat16() for t in images]
            sizes = [(56, 28)] if i == 4 else [(56, 56)]
            if i == 4:                                 # a bare <image> indicator: the dynamic branch expands it per size
                q = int(cfg.image_token_len ** 0.5)
                p = torch.cat([p[:cfg.image_position + 1], p[cfg.image_position + q * (q + 1):]])
            reqs.append((p.to(dev), dict(images=img, image_sizes=sizes)))
        else:
            reqs.append((torch.randint(3, cfg.vocab_size, (L,), generator=g).to(dev), {}))
    return reqs


def _serve(model, reqs, news, kv, use_graph=True, extra=None, capture=None):
    from cambrian_b200.serving import BatchedGenerator
    srv = BatchedGenerator(model, max_batch=8, max_cached_tokens=4096, page_size=16, kv_cache_dtype=kv,
                           use_graph=use_graph)
    total = srv.free_pages()
    rids = []
    for i, ((p, img), n) in enumerate(zip(reqs, news)):
        kw = dict(max_new_tokens=n, eos_token_id=None, **img, **(extra(i) if extra else {}))
        if capture is not None:
            kw["stopping_criteria"] = [lambda toks, scores, _i=i: capture.setdefault(_i, scores.clone()) is None]
        rids.append(srv.submit(p, **kw))
        if i % 3 == 2:
            srv.step()                                 # staggered: requests arrive between decode steps
    outs = srv.run()
    assert srv.free_pages() == total, "pages leaked at idle"
    return [outs[r].tolist() for r in rids]


def _solo(model, reqs, news, kv, capture=None, extra=None):
    out = []
    for i, ((p, img), n) in enumerate(zip(reqs, news)):
        kw = dict(max_new_tokens=n, eos_token_id=None, kv_cache_dtype=kv, **img, **(extra(i) if extra else {}))
        if capture is not None:
            kw["stopping_criteria"] = [lambda toks, scores, _i=i: capture.setdefault(_i, scores.clone()) is None]
        out.append(model.generate(p[None], **kw)[0].tolist())
    return out


@pytest.mark.parametrize("kv", ["bf16", "fp8"])
def test_server_matches_solo_generate(kv):
    from test_fp8_gpu import _peaked_model
    cfg, model = _peaked_model()
    reqs = _requests(cfg)
    news = [6 + (5 * i) % 14 for i in range(len(reqs))]
    cap_solo, cap_srv = {}, {}
    solo = _solo(model, reqs, news, kv, capture=cap_solo)
    graph = _serve(model, reqs, news, kv, capture=cap_srv)
    eager = _serve(model, reqs, news, kv, use_graph=False)
    assert graph == eager, "graph and eager serving differ"
    for i in range(len(reqs)):
        assert graph[i] == solo[i], (i, graph[i], solo[i])
        assert torch.equal(cap_srv[i], cap_solo[i]), f"request {i}: prefill logits differ from generate()'s"
    assert len({t for s in solo for t in s}) >= 8
    # sampling: per-request generators reproduce run to run, and the first token is solo generate()'s
    def samp(i):
        return dict(do_sample=True, top_k=20, temperature=0.8, generator=torch.Generator(device=dev).manual_seed(100 + i))
    s1 = _serve(model, reqs[:6], news[:6], kv, extra=samp)
    s2 = _serve(model, reqs[:6], news[:6], kv, extra=samp)
    assert s1 == s2
    first = _solo(model, reqs[:6], [1] * 6, kv, extra=samp)
    assert [s[0] for s in s1] == [f[0] for f in first]


@pytest.mark.parametrize("fmt", ["fp8", "nf4"])
def test_server_with_quantised_weights(fmt):
    from test_fp8_gpu import _peaked_model

    from cambrian_b200 import quant, quant_fp8
    cfg, model = _peaked_model()
    (quant_fp8.quantize_decoder_fp8_ if fmt == "fp8" else quant.quantize_decoder_nf4_)(model, dev)
    reqs = _requests(cfg, 6)
    news = [8] * 6
    assert _serve(model, reqs, news, "bf16") == _solo(model, reqs, news, "bf16")


def test_server_above_the_gemv_bucket():
    """20 requests at once into 32 rows: the decode step runs at buckets 32 and 16, where every projection and the
    lm_head take the tensor-core GEMM rather than the GEMV (ops.gemm), so per-row logits are not bucket-invariant there.
    On the peaked model the greedy tokens still equal solo generate()'s, and graph and eager steps agree bit for bit."""
    from test_fp8_gpu import _peaked_model

    from cambrian_b200.serving import BatchedGenerator
    cfg, model = _peaked_model()
    reqs = _requests(cfg, 20)
    news = [6 + (7 * i) % 17 for i in range(len(reqs))]
    solo = _solo(model, reqs, news, "bf16")
    runs = []
    for use_graph in (True, False):
        srv = BatchedGenerator(model, max_batch=32, max_cached_tokens=8192, page_size=16, use_graph=use_graph)
        seen = set()
        inner = srv._decode

        def decode(srv=srv, inner=inner, seen=seen):
            seen.add(srv._bucket(len(srv._active)))
            return inner()

        srv._decode = decode
        rids = [srv.submit(p, max_new_tokens=n, eos_token_id=None, **img) for (p, img), n in zip(reqs, news)]
        outs = srv.run()
        assert {32, 16} <= seen, seen
        assert srv.free_pages() == srv.pool.num_pages
        runs.append([outs[r].tolist() for r in rids])
    assert runs[0] == runs[1], "graph and eager serving differ"
    for i in range(len(reqs)):
        assert runs[0][i] == solo[i], (i, runs[0][i], solo[i])

