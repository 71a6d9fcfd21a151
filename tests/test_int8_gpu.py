"""The 8-bit (LLM.int8) inference path on the GPU: both quantisers bitwise against the torch reference of
tests/int8_reference.py and run-to-run deterministic, the int8 tensor-core GEMM and the dp4a GEMV bitwise against the
reference (so against each other), the prefill of int8 decoder layers bitwise against the same model running the
reference stand-ins, greedy decoding token-exact between the CUDA-graph decode, the eager loop and the fp32 oracle whose
projections run the reference int8 linear, and the memory quantisation gives back."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import int8_reference as R  # noqa: E402
from helpers import oracle_cfg, sd_cpu32, tiny_cambrian_config  # noqa: E402

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
bf = torch.bfloat16


def _weight(N, K, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    w = (torch.randn(N, K, generator=g, device=dev) * 0.02).to(bf)
    w[0, : K // 4] *= 8
    if N > 2:
        w[N // 2] = 0                                             # a zero row
    return w


def _act(M, K, n_out, seed):
    """bf16 activations with |x| < 6 except n_out columns that reach >= 6 in one (random) row each."""
    g = torch.Generator(device=dev).manual_seed(seed)
    x = (torch.randn(M, K, generator=g, device=dev) * 0.8).clamp(-5.5, 5.5)
    if n_out:
        cols = torch.randperm(K, generator=g, device=dev)[:n_out]
        rows = torch.randint(0, M, (n_out,), generator=g, device=dev)
        x[rows, cols] = torch.where(torch.rand(n_out, generator=g, device=dev) < 0.5, -1.0, 1.0) * \
            (6.0 + 20 * torch.rand(n_out, generator=g, device=dev))
    if M > 3:
        x[2] = 0                                                  # a zero row
    return x.to(bf)


@pytest.mark.parametrize("N,K", [(3, 16), (5, 4112), (1024, 4096), (6144, 4096), (4096, 14336), (28672, 4096)])
def test_weight_quantizer_bitwise_and_deterministic(N, K):
    from cambrian_b200 import quant_int8
    w = _weight(N, K, N + K)
    a, b = quant_int8.quantize(w), quant_int8.quantize(w)
    cb, scb = R.quantize_weight(w)
    assert torch.equal(a.cb, cb) and torch.equal(a.scb, scb)
    assert torch.equal(a.cb, b.cb) and torch.equal(a.scb, b.scb)


@pytest.mark.parametrize("M", [1, 5, 8, 9, 300, 2048])
@pytest.mark.parametrize("n_out", [0, 3, 300])
def test_activation_quantizer_bitwise_and_deterministic(M, n_out):
    from cambrian_b200 import ops
    K = 4096
    x = _act(M, K, n_out, M * 7 + n_out)
    got = ops.int8_quantize_act(x, 6.0)
    again = ops.int8_quantize_act(x, 6.0)
    xq, sca, idx = R.quantize_act(x, 6.0)
    n = int(got[3].item())
    assert n == idx.numel() and (n_out == 0 or n >= 1)
    assert torch.equal(got[2][:n].long(), idx)
    assert torch.equal(got[0], xq) and torch.equal(got[1], sca)
    for u, v in zip(got, again):
        assert torch.equal(u[:n] if u is got[2] else u, v[:n] if v is again[2] else v)
    off = ops.int8_quantize_act(x, 0.0)                           # tau <= 0: no outliers
    xq0, sca0, _ = R.quantize_act(x, 0.0)
    assert int(off[3].item()) == 0 and torch.equal(off[0], xq0) and torch.equal(off[1], sca0)


def _case(M, N, K, n_out, seed):
    from cambrian_b200 import ops, quant_int8
    x = _act(M, K, n_out, seed)
    qw = quant_int8.Int8Projection(quant_int8.quantize(_weight(N, K, seed + 1)))
    return x, ops.int8_quantize_act(x, 6.0), qw


def _want(x, qa, qw, **kw):
    n = int(qa[3].item())
    return R.linear_q(x, qa[0], qa[1], qa[2][:n].long(), qw.w.cb, qw.w.scb, **kw)


@pytest.mark.parametrize("M,N,K", [(9, 130, 16), (130, 1000, 4096), (600, 6144, 4096), (257, 4096, 14336),
                                   (2048, 4096, 4096)])
@pytest.mark.parametrize("n_out", [0, 4, 300])
def test_gemm_int8_bitwise(M, N, K, n_out):
    from cambrian_b200 import ops
    x, qa, qw = _case(M, N, K, min(n_out, K // 2), M + N + K + n_out)
    g = torch.Generator(device=dev).manual_seed(M)
    res = torch.randn(M, N, generator=g, device=dev).to(bf)
    bias = torch.randn(N, generator=g, device=dev).to(bf)
    for kw in (dict(), dict(residual=res), dict(out_dtype=torch.float32), dict(bias=bias, residual=res),
               dict(residual=res, out_dtype=torch.float32)):
        got = ops.gemm_int8(x, qa, qw, **kw)
        want = _want(x, qa, qw, **kw)
        assert torch.equal(got, want), (M, N, K, n_out, list(kw), (got.float() - want.float()).abs().max().item())


@pytest.mark.parametrize("M", list(range(1, 9)))
def test_gemv_int8_bitwise_and_equal_to_gemm_rows(M):
    from cambrian_b200 import ops
    for N, K, n_out in ((1000, 4096, 0), (517, 4096 + 16, 5), (6144, 4096, 200), (4096, 14336, 3)):
        x, qa, qw = _case(M, N, K, n_out, 31 * M + N)
        g = torch.Generator(device=dev).manual_seed(N)
        res = torch.randn(M, N, generator=g, device=dev).to(bf)
        bias = torch.randn(N, generator=g, device=dev).to(bf)
        for kw in (dict(), dict(residual=res), dict(bias=bias, out_dtype=torch.float32)):
            got = ops.gemv_int8(x, qa, qw, **kw)
            assert torch.equal(got, _want(x, qa, qw, **kw)), (M, N, K, n_out, list(kw))
            assert torch.equal(got, ops.gemm_int8(x, qa, qw, **kw)), (M, N, K, n_out, list(kw))


def _peaked_model():
    from test_modules_gpu import _build_tiny_model
    cfg = tiny_cambrian_config()
    cfg.fused_lm_loss = True
    model = _build_tiny_model(cfg)
    with torch.no_grad():
        emb = model.get_model().embed_tokens.weight
        perm = torch.randperm(emb.shape[0], generator=torch.Generator().manual_seed(9)).to(emb.device)
        model.lm_head.weight.copy_(emb[perm] * 24.0)
        for n_, p in model.named_parameters():
            if ((n_.endswith("o_proj.weight") and "layers." in n_ and "vision_sampler" not in n_)
                    or n_.endswith("down_proj.weight")
                    or ("vision_sampler_layers" in n_ and n_.endswith("proj_out.linear_2.weight"))):
                p.mul_(0.4)
    return cfg, model.eval()


def test_prefill_is_bitwise_the_reference_int8_layers(monkeypatch):
    from cambrian_b200 import quant_int8
    from cambrian_b200.model.language_model.cambrian_llama import KVCache
    cfg, model = _peaked_model()
    quant_int8.quantize_decoder_int8_(model, dev)
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(3, cfg.vocab_size, (2, 48), generator=g).to(dev)

    def run():
        with torch.no_grad():
            cache = KVCache(cfg, 2, 64, dev)
            h = model.get_model()(input_ids=ids, past_key_values=cache, use_cache=True).last_hidden_state
            return h, model(input_ids=ids).logits, cache.k[-1].clone()

    got = run()
    with monkeypatch.context() as mp:
        R.install(mp)                                             # the int8 entry points -> the torch definition
        want = run()
    for a, b, what in zip(got, want, ("prefill hidden states", "cache-less logits", "last layer's K cache")):
        assert torch.equal(a, b), f"{what} differ from the reference int8 layers"


def test_greedy_generate_8bit_token_exact():
    from test_int8_cpu import oracle_int8_functional
    from test_modules_gpu import _tiny_batch
    from test_parity_gpu import _bf, _oracle_greedy

    from cambrian_b200 import quant_int8
    from oracle import cambrian_oracle as O
    cfg, model = _peaked_model()
    quant_int8.quantize_decoder_int8_(model, dev)
    ids, labels, attn, pos, images, masks = _tiny_batch(cfg)
    S0, n_new = 40, 32
    gen_ids = ids[:1, :S0].clone().to(dev)
    imgs = [i[:1].to(dev).bfloat16() for i in images]
    kw = dict(image_sizes=[(56, 56)], max_new_tokens=n_new, do_sample=False)
    new = model.generate(gen_ids, images=imgs, **kw)
    model.config.disable_decode_graph = True
    eager_loop = model.generate(gen_ids, images=imgs, **kw)
    model.config.disable_decode_graph = False
    assert torch.equal(new, eager_loop), (new.tolist(), eager_loop.tolist())
    got = new[0].tolist()
    sd = sd_cpu32(model)
    towers = model.get_model().vision_tower_aux_list
    feats = [_bf(t(i).float().cpu()) for t, i in zip(towers, imgs)]
    shim = oracle_int8_functional(model, cfg, sd)
    real_F = O.F
    O.F = shim
    try:
        t_32, m_32 = _oracle_greedy(sd, cfg, oracle_cfg(cfg), feats, gen_ids.cpu(), n_new, torch.float32,
                                    torch.device("cpu"))
    finally:
        O.F = real_F
    assert shim.hits >= 7 * cfg.num_hidden_layers * n_new
    assert got == t_32, f"8-bit greedy != fp32 oracle with int8 projections:\n{got}\n{t_32}\nmargins {m_32}"
    assert len(set(got)) >= 8
    # a batch of 12: the decode projections take the int8 tensor-core GEMM inside the captured graph
    b_ids = gen_ids.repeat(12, 1)
    b_ids[:, -4:] = torch.randint(3, cfg.vocab_size, (12, 4), generator=torch.Generator().manual_seed(3)).to(dev)
    b_imgs = [i.repeat(12, 1, 1, 1) for i in imgs]
    kw12 = dict(image_sizes=[(56, 56)] * 12, max_new_tokens=16, do_sample=False)
    graphed = model.generate(b_ids, images=b_imgs, **kw12)
    model.config.disable_decode_graph = True
    eager12 = model.generate(b_ids, images=b_imgs, **kw12)
    model.config.disable_decode_graph = False
    assert torch.equal(graphed, eager12), (graphed.tolist(), eager12.tolist())


def test_quantisation_frees_the_bf16_projection_bytes():
    from test_modules_gpu import _build_tiny_model
    from cambrian_b200 import quant_int8
    cfg = tiny_cambrian_config()
    model = _build_tiny_model(cfg).eval()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    stats = quant_int8.quantize_decoder_int8_(model, dev)
    torch.cuda.synchronize()
    after = torch.cuda.memory_allocated()
    L = cfg.num_hidden_layers
    assert stats["int8_bytes"] == L * quant_int8.bytes_per_layer(cfg)
    want = stats["bf16_bytes"] - stats["int8_bytes"]
    slack = 512 * (2 * 4 * L + 7 * L)                             # the caching allocator rounds every block to 512 B
    assert abs((before - after) - want) <= slack, (before - after, want, slack)
