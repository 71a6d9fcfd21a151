"""GPU checks of token sampling (ops.sample_tokens, csrc/sample.cu; generation.py states the rule): the kernel's token
against the fp64 reference race of tests/sampling_reference.py, the kept set against HF's warpers, the distribution by a
chi-square test, determinism and batch invariance, and `generate(do_sample=True)` and the server, graph against eager."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import sampling_reference as SR  # noqa: E402

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")

# per-row (T, top_k, top_p) mixes: the model worker's defaults, HF's plain top-k, top-p alone, near-greedy, top-1
MIX = [(0.2, 50, 0.7), (1.0, 50, 1.0), (0.7, 0, 0.9), (1e-4, 0, 1.0), (1.0, 1, 1.0), (1.5, 20, 0.95), (1.0, 0, 1.0),
       (0.8, 3000, 0.8)]


def _params(rows, seed0, step, mix=MIX):
    ps = [mix[b % len(mix)] for b in range(rows)]
    return (torch.tensor([p[0] for p in ps], dtype=torch.float32, device=dev),
            torch.tensor([p[1] for p in ps], dtype=torch.int32, device=dev),
            torch.tensor([p[2] for p in ps], dtype=torch.float32, device=dev),
            torch.tensor([SR_seed(seed0 + 7919 * b) for b in range(rows)], dtype=torch.int64, device=dev),
            torch.full((rows,), step, dtype=torch.int64, device=dev)), ps


def SR_seed(v):
    from cambrian_b200.generation import as_int64
    return as_int64(v * 0x9E3779B97F4A7C15)


def _logits(rows, V, ld, gen):
    buf = torch.full((rows, ld), float("nan"), dtype=torch.float32)
    buf[:, :V] = torch.randn(rows, V, generator=gen) * 2.5
    return buf.to(dev)[:, :V]


@pytest.mark.parametrize("V,ld", [(32000, 32000), (32064, 32064), (64000, 64000), (128256, 128256), (1001, 1040)])
def test_token_matches_the_reference_race(V, ld):
    from cambrian_b200 import ops
    g = torch.Generator().manual_seed(V)
    close = boundary = checked = 0
    for rows, pairs in ((1, 2), (7, 2), (32, 3)):
        logits = _logits(rows, V, ld, g)
        lg = logits.cpu().numpy()
        for j in range(pairs):
            step = [0, 1, 1 << 33, 77][j + rows % 2]
            params, ps = _params(rows, 1000 * rows + j, step)
            got = ops.sample_tokens(logits, *params).tolist()
            seeds = params[3].tolist()
            for b in range(rows):
                T, k, p = ps[b]
                tok, gap, margin = SR.race(lg[b], T, k, p, seeds[b], step)
                if gap < 1e-4:
                    close += 1
                elif margin < 1e-5:
                    boundary += 1
                else:
                    checked += 1
                    assert got[b] == tok, (V, rows, b, ps[b], got[b], tok)
    print(f"V={V}: {checked} draws equal the reference; set aside: {close} close races, {boundary} top-p boundaries")
    assert checked >= 0.75 * (close + boundary + checked)


def test_never_outside_the_warped_set():
    from cambrian_b200 import ops
    from cambrian_b200.generation import warp_logits
    g = torch.Generator().manual_seed(3)
    V, rows = 32000, 32
    logits = _logits(rows, V, V, g)
    mix = [(1.5, 50, 1.0), (1.5, 0, 0.9), (1.5, 20, 0.6), (1.5, 200, 0.95)]
    for step in range(20):
        params, ps = _params(rows, 5, step, mix)
        tok = ops.sample_tokens(logits, *params).cpu()
        for b in range(rows):
            T, k, p = ps[b]
            kept = torch.isfinite(warp_logits(logits[b:b + 1].cpu(), T, k, p))[0]
            assert kept[tok[b]], (step, b, ps[b])


@pytest.mark.parametrize("T,k,p", [(1.0, 0, 1.0), (0.7, 20, 0.9), (1.3, 0, 0.8)])
def test_distribution_chi_square(T, k, p):
    from scipy.stats import chi2

    from cambrian_b200 import ops
    from cambrian_b200.generation import warp_logits
    V, n = 64, 200_000
    row = torch.randn(1, V, generator=torch.Generator().manual_seed(8)) * 1.5
    logits = row.expand(n, V).contiguous().to(dev)
    params, _ = _params(n, 12345, 3, [(T, k, p)])
    tok = ops.sample_tokens(logits, *params).cpu()
    counts = torch.bincount(tok, minlength=V).double()
    probs = warp_logits(row.double(), T, k, p).softmax(-1)[0]
    assert counts[probs == 0].sum() == 0
    live = probs > 0
    exp = probs[live] * n
    stat = float(((counts[live] - exp) ** 2 / exp).sum())
    pval = chi2.sf(stat, int(live.sum()) - 1)
    assert pval > 1e-6, (stat, pval)


def test_bitwise_deterministic_and_batch_invariant():
    from cambrian_b200 import ops
    V, ld, rows = 128256, 128264, 32
    logits = _logits(rows, V, ld, torch.Generator().manual_seed(4))
    params, _ = _params(rows, 99, 5)
    a = ops.sample_tokens(logits, *params)
    b = ops.sample_tokens(logits, *params)
    assert torch.equal(a, b)
    for r in range(rows):
        alone = ops.sample_tokens(logits[r:r + 1], *[t[r:r + 1] for t in params])
        assert int(alone) == int(a[r]), r


def _graph_vs_eager(model, ids, **kw):
    outs = []
    for eager in (False, True):
        model.config.disable_decode_graph = eager
        g = torch.Generator(device=dev).manual_seed(31)
        outs.append(model.generate(ids, do_sample=True, generator=g, eos_token_id=None, **kw))
    model.config.disable_decode_graph = False
    return outs


def test_generate_graph_and_eager_agree_llama():
    from test_modules_gpu import _build_tiny_model

    from helpers import tiny_cambrian_config
    cfg = tiny_cambrian_config()
    model = _build_tiny_model(cfg).eval()
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(3, cfg.vocab_size, (3, 20), generator=g).to(dev)
    am = torch.ones_like(ids)
    am[1, :4] = 0
    am[2, :9] = 0                                        # left padding
    for B in (1, 3):
        for T, k, p in ((0.2, 50, 0.7), (1.0, 0, 0.9), (1.5, 50, 1.0)):
            kw = dict(max_new_tokens=12, temperature=T, top_k=k, top_p=p)
            if B == 3:
                kw["attention_mask"] = am
            graph, eager = _graph_vs_eager(model, ids[:B], **kw)
            assert torch.equal(graph, eager), (B, T, k, p)


def test_generate_graph_and_eager_agree_phi3():
    from test_phi3_gpu import tiny_phi3
    cfg, model = tiny_phi3(window=16)
    model = model.to(dev, torch.bfloat16)
    g = torch.Generator().manual_seed(6)
    ids = torch.randint(3, cfg.vocab_size, (3, 30), generator=g).to(dev)
    am = torch.ones_like(ids)
    am[2, :7] = 0
    for B in (1, 3):
        kw = dict(max_new_tokens=24, temperature=1.0, top_k=50, top_p=0.9)
        if B == 3:
            kw["attention_mask"] = am
        graph, eager = _graph_vs_eager(model, ids[:B], **kw)
        assert torch.equal(graph, eager), B


def test_server_sampling():
    """Sampled and greedy requests served together: graph and eager steps give the same tokens, every sampled token is
    the reference race over the logits of its step (as the stopping criteria see them), and the greedy requests get
    solo generate()'s tokens."""
    from test_fp8_gpu import _peaked_model
    from test_paged_gpu import _requests, _serve, _solo

    from cambrian_b200.generation import GenerationArgs, draw_seed
    cfg, model = _peaked_model()
    reqs = _requests(cfg, 8)
    news = [6 + (3 * i) % 9 for i in range(len(reqs))]
    mix = {1: (0.8, 20, 1.0), 2: (1.2, 0, 0.9), 4: (0.2, 50, 0.7), 5: (1.0, 5, 0.95), 7: (1.5, 0, 1.0)}

    def samp(i):
        if i not in mix:
            return dict(do_sample=False)
        T, k, p = mix[i]
        return dict(do_sample=True, temperature=T, top_k=k, top_p=p,
                    generator=torch.Generator(device=dev).manual_seed(500 + i))

    seen = {}

    def capture_all(i):
        kw = samp(i)

        def crit(toks, scores, _i=i):
            seen.setdefault(_i, []).append((toks[0, -1].item(), scores[0].float().cpu().numpy()))
            return False
        kw["stopping_criteria"] = [crit]
        return kw

    graph = _serve(model, reqs, news, "bf16", extra=capture_all)
    eager = _serve(model, reqs, news, "bf16", use_graph=False, extra=samp)
    assert graph == eager
    solo = _solo(model, reqs, news, "bf16", extra=lambda i: dict(do_sample=False))
    checked = skipped = 0
    for i in range(len(reqs)):
        if i not in mix:
            assert graph[i] == solo[i], i
            continue
        S = draw_seed(GenerationArgs(generator=torch.Generator(device=dev).manual_seed(500 + i)), dev)
        T, k, p = mix[i]
        # the criteria run for every token but the last (max_new_tokens ends the request first)
        assert len(seen[i]) == len(graph[i]) - 1 and [t for t, _ in seen[i]] == graph[i][:-1]
        for t, (tok, scores) in enumerate(seen[i]):
            ref, gap, margin = SR.race(scores, T, k, p, S, t)
            if gap < 1e-4 or margin < 1e-5:
                skipped += 1
                continue
            checked += 1
            assert tok == ref, (i, t, tok, ref)
    print(f"server: {checked} sampled tokens equal the reference race, {skipped} set aside")
    assert checked > skipped
