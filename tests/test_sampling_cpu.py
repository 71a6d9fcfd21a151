"""CPU checks of token sampling (ops.sample_tokens; generation.py states the rule): the Philox4x32-10 of the reference
against the Random123 known-answer vectors, the reference keep set against HF's warpers (`warp_logits`), argument
validation of cb_sample_tokens, and the host logic around the kernel over the stand-in of tests/sampling_reference.py:
seed and step numbering, and the server's per-row parameter buffers through admission, retirement and compaction with
greedy and sampled rows mixed.  The kernel itself is covered under `-m gpu` (tests/test_sampling_gpu.py)."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import sampling_reference as SR  # noqa: E402

needs_no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="kernel stand-ins are for GPU-less machines only")


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    got = SR.philox4x32_10(np.array([ctr], dtype=np.uint64), np.array([key], dtype=np.uint64))[0]
    assert [int(w) for w in got] == list(want)


def test_uniforms_inside_the_open_interval():
    u = SR.uniforms(100_003, seed=(1 << 64) - 1, step=(1 << 40) + 7)
    assert u.min() > 0 and u.max() < 1 and abs(u.mean() - 0.5) < 5e-3
    assert np.all(np.float32(u) == u)          # exact in fp32, as the kernel computes it


@pytest.mark.parametrize("T,k,p", [(1.0, 50, 1.0), (0.2, 50, 0.7), (0.7, 0, 0.9), (1.5, 20, 0.95), (1.0, 0, 0.5),
                                   (0.8, 7, 1.0), (1.0, 1, 1.0), (2.0, 0, 0.999)])
def test_keep_set_equals_hf_warpers(T, k, p):
    from cambrian_b200.generation import warp_logits
    g = torch.Generator().manual_seed(7)
    for V in (64, 1001, 32000):
        # distinct values: a random permutation of an evenly spaced grid, with the exponential tail a softmax has
        grid = torch.linspace(-12, 4, V)
        logits = torch.stack([grid[torch.randperm(V, generator=g)] for _ in range(4)])
        want = torch.isfinite(warp_logits(logits, T, k, p))
        for b in range(4):
            s = SR.scores(logits[b].numpy(), T)
            assert np.unique(s).size == V                       # tie-free
            keep, margin = SR.keep_set(s, k, p, with_margin=True)
            if margin < 1e-5:
                continue                                        # the fp32 cumsum of HF may round across the boundary
            assert np.array_equal(keep, want[b].numpy()), (V, b)


def test_top_p_keeps_a_boundary_tie_whole():
    # masses 0.4, 0.2, 0.2, 0.2 (three tied): at top_p 0.5 the first tied token is needed, so all three are kept
    s = np.log(np.array([0.4, 0.2, 0.2, 0.2, 1e-6], dtype=np.float64)).astype(np.float32)
    assert SR.keep_set(s, 0, 0.5).tolist() == [True, True, True, True, False]
    assert SR.keep_set(s, 0, 0.35).tolist() == [True, False, False, False, False]
    assert SR.keep_set(s, 2, 1.0).tolist() == [True, True, True, True, False]   # top-k keeps ties too


def test_argument_validation_without_gpu(lib):
    one = ctypes.c_void_p(16)                   # non-null, aligned dummy pointer (never dereferenced)
    odd = ctypes.c_void_p(18)
    assert lib.cb_sample_tokens_workspace_floats(32, 128256) >= 0

    def smp(logits=one, ld=1000, rows=2, V=1000, temp=one, topk=one, topp=one, seed=one, step=one, out=one):
        return lib.cb_sample_tokens(logits, ld, rows, V, temp, topk, topp, seed, step, out, None, 0, None)

    for kw, msg in ((dict(rows=0), b"rows"), (dict(V=0), b"V="), (dict(V=1 << 23, ld=1 << 23), b"V="),
                    (dict(ld=999), b"stride"), (dict(logits=None), b"null"), (dict(temp=None), b"null"),
                    (dict(topk=None), b"null"), (dict(topp=None), b"null"), (dict(seed=None), b"null"),
                    (dict(step=None), b"null"), (dict(out=None), b"null"), (dict(logits=odd), b"aligned"),
                    (dict(seed=ctypes.c_void_p(20)), b"aligned"), (dict(out=ctypes.c_void_p(20)), b"aligned")):
        assert smp(**kw) == 1 and msg in lib.cb_last_error(), (kw, lib.cb_last_error())


def test_ops_wrapper_checks_operands():
    from cambrian_b200 import _lib, ops
    with pytest.raises(_lib.CambrianB200Error, match="CUDA"):
        ops.sample_tokens(torch.zeros(2, 8), *[torch.zeros(2)] * 5)


def test_seed_and_step_numbering():
    from cambrian_b200.generation import GenerationArgs, as_int64, draw_seed, sampling_params
    g = torch.Generator().manual_seed(11)
    lo, hi = torch.randint(0, 1 << 32, (2,), generator=g).tolist()
    S = lo | hi << 32
    a = GenerationArgs(do_sample=True, temperature=0.2, top_k=50, top_p=0.7,
                       generator=torch.Generator().manual_seed(11))
    assert draw_seed(a, "cpu") == S and draw_seed(a, "cpu") == S          # drawn once per call
    a.step = 5
    t, k, p, seed, step = sampling_params(a, 3, "cpu")
    assert seed.tolist() == [as_int64(S + b) for b in range(3)] and step.tolist() == [5] * 3
    assert t.dtype == torch.float32 and k.dtype == torch.int32 and k.tolist() == [50] * 3
    assert torch.equal(p, torch.full((3,), 0.7))
    assert as_int64((1 << 64) - 1) == -1 and as_int64(1 << 64) == 0 and as_int64(5) == 5
    huge = GenerationArgs(do_sample=True, top_k=1 << 40, generator=torch.Generator().manual_seed(1))
    assert sampling_params(huge, 1, "cpu")[1].tolist() == [(1 << 31) - 1]


def test_cpu_logits_keep_the_torch_warpers():
    from cambrian_b200.generation import GenerationArgs, next_tokens, warp_logits
    logits = torch.randn(3, 100, generator=torch.Generator().manual_seed(3))
    a = GenerationArgs(do_sample=True, temperature=0.7, top_k=20, top_p=0.9, generator=torch.Generator().manual_seed(4))
    want = torch.multinomial(warp_logits(logits, 0.7, 20, 0.9).softmax(-1), 1,
                             generator=torch.Generator().manual_seed(4)).squeeze(-1)
    assert torch.equal(next_tokens(logits, a), want) and a.seed is None and a.step == 0


@needs_no_gpu
def test_server_sampling_buffers(monkeypatch):
    """Mixed greedy and sampled requests through a two-row server: at every decode step each row's parameters, seed and
    step in the device buffers are its request's, and a sampled request's seed is the one a solo generate() with its
    generator draws for row 0."""
    from test_paged_cpu import _setup

    from cambrian_b200 import ops
    from cambrian_b200.generation import GenerationArgs, as_int64, draw_seed
    from cambrian_b200.serving import BatchedGenerator
    cfg, model, ids, feats, images = _setup(monkeypatch)
    SR.install(monkeypatch)
    srv = BatchedGenerator(model, max_batch=2, max_cached_tokens=32 * 16, page_size=16)
    calls = []

    def checked(logits, temperature, top_k, top_p, seed, step, out=None, workspace=None):
        act = srv._active
        assert srv._sample[:len(act)].tolist() == [r.args.do_sample for r in act]
        for i, r in enumerate(act):
            a = r.args
            if a.do_sample:
                assert (temperature[i].item(), top_k[i].item(), top_p[i].item()) == \
                    (np.float32(a.temperature), a.top_k, np.float32(a.top_p))
                assert seed[i].item() == as_int64(a.seed) and step[i].item() == len(r.tokens)
        calls.append(len(act))
        return SR.sample_tokens(logits, temperature, top_k, top_p, seed, step, out)

    monkeypatch.setattr(ops, "sample_tokens", checked)
    samp = [None, dict(temperature=0.8, top_k=5), None, dict(temperature=1.3, top_k=0, top_p=0.9), dict(top_k=3)]
    news = [4, 7, 3, 6, 5]
    rids = []
    for i, (kw, n) in enumerate(zip(samp, news)):
        extra = {} if kw is None else dict(do_sample=True, generator=torch.Generator().manual_seed(40 + i), **kw)
        rids.append(srv.submit(ids[i % ids.shape[0], 20 + i:36 + i].clamp(min=3), max_new_tokens=n, eos_token_id=None,
                               **extra))
    seeds = {}
    while srv.pending():
        srv.step()
        seeds.update({r.rid: r.args.seed for r in srv._active})
    outs = srv.run()
    assert [len(outs[r]) for r in rids] == news and calls
    for i, kw in enumerate(samp):
        if kw is not None:
            want = draw_seed(GenerationArgs(generator=torch.Generator().manual_seed(40 + i)), "cpu")
            assert seeds[rids[i]] == want
        else:
            assert rids[i] not in seeds or seeds[rids[i]] is None
