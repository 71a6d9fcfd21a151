"""The FP8 E4M3 inference path on the GPU: the row quantiser bitwise against the torch reference of
tests/fp8_reference.py and run-to-run deterministic; the tensor-core GEMM and the wgmma decode GEMV against an fp64 sum
over the same quantised operands (one bf16 rounding plus an fp32-accumulation term), per-k-block promotion on an
all-positive K = 14336 product, bitwise run-to-run determinism and prefill rows against decode rows; greedy decoding
token-exact against the fp32 oracle on fake-quantised projections and between the CUDA-graph and eager loops; one
Llama-3-8B-shaped decoder layer against the oracle on fake-quantised weights."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import fp8_reference as R  # noqa: E402
from helpers import ParityCollector, both_modes, oracle_cfg, sd_cpu32, tiny_cambrian_config  # noqa: E402

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
bf = torch.bfloat16


def _bits(t):
    return t.view(torch.uint8)


def _weight(N, K, seed, scale=0.02):
    g = torch.Generator(device=dev).manual_seed(seed)
    w = torch.randn(N, K, generator=g, device=dev) * scale
    w[0, : K // 4] *= 8
    if N > 2:
        w[N // 2] = 0                                             # a zero row
    return w.to(bf)


def _act(M, K, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(M, K, generator=g, device=dev)
    x[:, : max(1, K // 512)] *= 40                                # a few large features, as in LLM activations
    if M > 3:
        x[2] = 0                                                  # a zero row
    return x.to(bf)


# ------------------------------------------------------------------------------------------------ quantisers
@pytest.mark.parametrize("N,K", [(3, 16), (5, 4112), (6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336),
                                 (9216, 7168), (7168, 7168), (40960, 7168), (7168, 20480)])
def test_weight_quantizer_bitwise_and_deterministic(N, K):
    from cambrian_b200 import quant_fp8
    w = _weight(N, K, N + K)
    a, b = quant_fp8.quantize(w), quant_fp8.quantize(w)
    q, s = R.quantize_weight(w)
    assert torch.equal(_bits(a.wq), _bits(q)) and torch.equal(a.sw, s)
    assert torch.equal(_bits(a.wq), _bits(b.wq)) and torch.equal(a.sw, b.sw)


def test_quantizer_edge_rows_bitwise():
    from cambrian_b200 import ops
    from test_fp8_cpu import _row_case
    w = torch.cat([_row_case(), torch.zeros(6, 16, dtype=bf)], 1).to(dev)       # K = 48
    w[0, 40] = 1e6                                                               # 1e6 * (448 / 1e6) rounds to 448 or below
    q, s = ops.fp8_quantize_act(w)
    qr, sr = R.quantize_act(w)
    assert torch.equal(_bits(q), _bits(qr)) and torch.equal(s, sr)
    assert not torch.isnan(q.float()).any()


@pytest.mark.parametrize("M", [1, 5, 8, 9, 600, 2048])
@pytest.mark.parametrize("K", [4096, 14336])
def test_activation_quantizer_bitwise_and_deterministic(M, K):
    from cambrian_b200 import ops
    x = _act(M, K, M * 7 + K)
    got, again = ops.fp8_quantize_act(x), ops.fp8_quantize_act(x)
    q, s = R.quantize_act(x)
    assert torch.equal(_bits(got[0]), _bits(q)) and torch.equal(got[1], s)
    assert torch.equal(_bits(got[0]), _bits(again[0])) and torch.equal(got[1], again[1])


# ------------------------------------------------------------------------------------------------ matmuls
def _case(M, Ns, K, seed, act=None):
    """an activation and a projection of len(Ns) stacked weights (q|k|v-style segments)"""
    from cambrian_b200 import ops, quant_fp8
    x = _act(M, K, seed) if act is None else act
    qw = quant_fp8.Fp8Projection(quant_fp8.quantize(*[_weight(n, K, seed + 1 + i) for i, n in enumerate(Ns)]))
    return ops.fp8_quantize_act(x), qw


def _check(got, qa, qw, what, bias=None, residual=None, out_dtype=torch.bfloat16):
    """|got - y| <= one rounding to the output type of |y| + 2^-10 of the absolute product sum, y the epilogue on the
    fp64 sum.  The second term is the accumulation error: the f8 tensor-core MMA rounds its sums inside a k-block more
    coarsely than fp32 (up to about 2^-11 of the absolute sum on an H100 80GB HBM3), the fp32 promotion adds little."""
    xq, sa = qa
    acc = R.acc64(xq, qw.w.wq)
    scale = sa.double()[:, None] * qw.w.sw.double()[None, :]
    y = acc * scale
    if bias is not None:
        y = y + bias.double()[None, :]
    if residual is not None:
        y = y + residual.double()
    mag = (xq.double().abs() @ qw.w.wq.double().abs().t()) * scale
    rnd = 2.0 ** -8 if out_dtype == torch.bfloat16 else 2.0 ** -22
    tol = rnd * y.abs() + 2.0 ** -10 * mag + 1e-30
    err = (got.double() - y).abs()
    assert got.dtype == out_dtype and torch.isfinite(got).all(), what
    bad = err > tol
    assert not bad.any(), (what, int(bad.sum()), (err / tol).max().item())


@pytest.mark.parametrize("M,Ns,K", [(9, [130], 16), (130, [1000], 4096), (600, [4096, 1024, 1024], 4096),
                                    (257, [4096], 14336), (2048, [14336, 14336], 4096), (64, [7168], 20480),
                                    (300, [520, 136], 1040)])
def test_gemm_fp8_against_fp64_and_deterministic(M, Ns, K):
    from cambrian_b200 import ops
    qa, qw = _case(M, Ns, K, M + sum(Ns) + K)
    N = qw.N
    g = torch.Generator(device=dev).manual_seed(M)
    res = torch.randn(M, N, generator=g, device=dev).to(bf)
    bias = torch.randn(N, generator=g, device=dev).to(bf)
    for kw in (dict(), dict(residual=res), dict(out_dtype=torch.float32), dict(bias=bias, residual=res),
               dict(residual=res, out_dtype=torch.float32)):
        got = ops.gemm_fp8(qa, qw, **kw)
        _check(got, qa, qw, ("gemm", M, Ns, K, list(kw)), **kw)
        assert torch.equal(got, ops.gemm_fp8(qa, qw, **kw)), ("gemm not deterministic", M, Ns, K, list(kw))
    # an output view with a row stride TMA cannot address (not a multiple of 8): the register-store epilogue
    wide = torch.zeros(M, N + 3, dtype=bf, device=dev)
    ops.gemm_fp8(qa, qw, out=wide[:, :N])
    assert torch.equal(wide[:, :N], ops.gemm_fp8(qa, qw)) and not wide[:, N:].any()


@pytest.mark.parametrize("M", list(range(1, 9)))
def test_gemv_fp8_against_fp64_deterministic_and_near_gemm_rows(M):
    from cambrian_b200 import ops
    for Ns, K in (([1000], 4096), ([517], 4096 + 16), ([4096, 1024, 1024], 4096), ([4096], 14336),
                  ([14336, 14336], 4096), ([7168], 20480)):
        qa, qw = _case(M, Ns, K, 31 * M + sum(Ns))
        N = qw.N
        g = torch.Generator(device=dev).manual_seed(N)
        res = torch.randn(M, N, generator=g, device=dev).to(bf)
        bias = torch.randn(N, generator=g, device=dev).to(bf)
        for kw in (dict(), dict(residual=res), dict(bias=bias, out_dtype=torch.float32)):
            got = ops.gemv_fp8(qa, qw, **kw)
            _check(got, qa, qw, ("gemv", M, Ns, K, list(kw)), **kw)
            assert torch.equal(got, ops.gemv_fp8(qa, qw, **kw)), ("gemv not deterministic", M, Ns, K, list(kw))
            # the same rows through the prefill GEMM: a different summation order, the same bound
            _check(ops.gemm_fp8(qa, qw, **kw), qa, qw, ("gemm rows", M, Ns, K, list(kw)), **kw)


@pytest.mark.parametrize("M", [4, 600])
def test_all_positive_product_at_k14336_needs_the_promotion(M):
    """Every product positive, K = 14336: the sum grows to ~14336 x the mean product, where a single f8 MMA accumulator
    running over all of K would drop low-order bits on every addition.  With each 128-deep k-block added in fp32 the
    relative error stays near fp32 rounding; the bound is 1e-3."""
    from cambrian_b200 import ops, quant_fp8
    K, N = 14336, 512
    g = torch.Generator(device=dev).manual_seed(11)
    x = (torch.rand(M, K, generator=g, device=dev) + 0.05).to(bf)
    w = (torch.rand(N, K, generator=g, device=dev) + 0.05).to(bf)
    qa = ops.fp8_quantize_act(x)
    qw = quant_fp8.Fp8Projection(quant_fp8.quantize(w))
    want = R.acc64(*[qa[0], qw.w.wq]) * (qa[1].double()[:, None] * qw.w.sw.double()[None, :])
    fn = ops.gemv_fp8 if M <= 8 else ops.gemm_fp8
    got = fn(qa, qw, out_dtype=torch.float32).double()
    rel = ((got - want).abs() / want.abs()).max().item()
    assert rel <= 1e-3, rel


# ------------------------------------------------------------------------------------------------ end to end
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


def test_greedy_generate_fp8_token_exact_and_graph_equals_eager():
    from test_fp8_cpu import oracle_fp8_functional
    from test_modules_gpu import _tiny_batch
    from test_parity_gpu import _bf, _oracle_greedy

    from cambrian_b200 import quant_fp8
    from oracle import cambrian_oracle as O
    cfg, model = _peaked_model()
    quant_fp8.quantize_decoder_fp8_(model, dev)
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
    shim = oracle_fp8_functional(model, cfg, sd)
    real_F = O.F
    O.F = shim
    try:
        t_32, m_32 = _oracle_greedy(sd, cfg, oracle_cfg(cfg), feats, gen_ids.cpu(), n_new, torch.float32,
                                    torch.device("cpu"))
    finally:
        O.F = real_F
    assert shim.hits >= 7 * cfg.num_hidden_layers * n_new
    assert got == t_32, f"FP8 greedy != fp32 oracle with FP8 projections:\n{got}\n{t_32}\nmargins {m_32}"
    assert len(set(got)) >= 8
    assert min(m_32) > 2.0, f"test model lost its margin (min {min(m_32)})"
    # a batch of 12: the decode projections take the FP8 GEMM inside the captured graph
    b_ids = gen_ids.repeat(12, 1)
    b_ids[:, -4:] = torch.randint(3, cfg.vocab_size, (12, 4), generator=torch.Generator().manual_seed(3)).to(dev)
    b_imgs = [i.repeat(12, 1, 1, 1) for i in imgs]
    kw12 = dict(image_sizes=[(56, 56)] * 12, max_new_tokens=16, do_sample=False)
    graphed = model.generate(b_ids, images=b_imgs, **kw12)
    model.config.disable_decode_graph = True
    eager12 = model.generate(b_ids, images=b_imgs, **kw12)
    model.config.disable_decode_graph = False
    assert torch.equal(graphed, eager12), (graphed.tolist(), eager12.tolist())


class _Fp8ById:
    """`torch.nn.functional` for the oracle with each decoder projection weight replaced by a [1, 1] placeholder holding
    a small integer id (exact in fp32 and bf16, so it survives both oracle modes): F.linear on it quantises the
    activation by the reference rule and runs the reference product on that projection's (wq, sw)."""

    def __init__(self):
        self.table = {}

    def __getattr__(self, name):
        return getattr(torch.nn.functional, name)

    def placeholder(self, wq, sw):
        self.table[len(self.table) + 1] = (wq, sw)
        return torch.full((1, 1), float(len(self.table)))

    def linear(self, x, w, b=None):
        if w.shape != (1, 1):
            return torch.nn.functional.linear(x, w, b)
        wq, sw = self.table[int(w.item())]
        xq, sa = R.quantize_act(x.reshape(-1, x.shape[-1]))
        y = R.epilogue(R.acc64(xq, wq).float(), sa, sw, out_dtype=x.dtype)
        return y.view(*x.shape[:-1], wq.shape[0])


def test_llama3_8b_decoder_layer_infer_fp8():
    """One Llama-3-8B-shaped layer (H 4096, 32 q / 8 kv heads x 128, FFN 14336) quantised to FP8 runs the cache-less
    `infer` at S = 2048 within the parity criterion of the fp32 oracle on the same fake-quantised projections (the
    eager-bf16 run of that oracle is the yardstick)."""
    from cambrian_b200 import quant_fp8
    from cambrian_b200.model.language_model.cambrian_llama import CambrianConfig, CBLlamaDecoderLayer, rope_tables
    from oracle import cambrian_oracle as O
    torch.manual_seed(2)
    cfg = CambrianConfig(hidden_size=4096, intermediate_size=14336, num_hidden_layers=1, num_attention_heads=32,
                         num_key_value_heads=8, vocab_size=1024, max_position_embeddings=4096, rope_theta=500000.0,
                         rms_norm_eps=1e-5)
    layer = CBLlamaDecoderLayer(cfg, 0)
    with torch.no_grad():
        for p in layer.parameters():
            if p.dim() == 2:
                p.normal_(0, 0.02)
            else:
                p.copy_(1 + 0.1 * torch.randn_like(p))
    layer = layer.to(device=dev, dtype=bf).eval()

    class _Holder(torch.nn.Module):                     # quantize_decoder_fp8_ walks model.get_model().layers
        def __init__(self, lay):
            super().__init__()
            self.layers = torch.nn.ModuleList([lay])

        def get_model(self):
            return self

    quant_fp8.quantize_decoder_fp8_(_Holder(layer), dev)
    P = "model.layers.0."
    sd = {P + k: v.detach().float() for k, v in layer.state_dict().items() if v.numel()}
    shim = _Fp8ById()
    H, I, kv = 4096, 14336, 8 * 128
    for key, parts in (("qkv", [("self_attn.q_proj", H), ("self_attn.k_proj", kv), ("self_attn.v_proj", kv)]),
                       ("o", [("self_attn.o_proj", H)]), ("gate_up", [("mlp.gate_proj", I), ("mlp.up_proj", I)]),
                       ("down", [("mlp.down_proj", H)])):
        w, r = layer._fp8[key].w, 0
        for name, rows in parts:
            sd[P + name + ".weight"] = shim.placeholder(w.wq[r:r + rows], w.sw[r:r + rows])
            r += rows
    B, S = 1, 2048
    x = torch.randn(B, S, H).bfloat16().float()
    pos = torch.arange(S)[None]
    ocfg = dict(num_attention_heads=32, num_key_value_heads=8, rms_norm_eps=1e-5, hidden_size=H)
    real_F = O.F
    O.F = shim
    try:
        with torch.no_grad():
            ref, eag = both_modes(lambda s, xx, pp: O.llama_layer(s, P, xx, *O.rope_cos_sin(pp, 128, 500000.0), None,
                                                                  ocfg), sd, x, pos, device=dev)
    finally:
        O.F = real_F
    cos_t, sin_t = rope_tables(cfg, dev)
    rt = dict(pos=pos.to(dev).reshape(-1).contiguous(), cos=cos_t, sin=sin_t, kmask=None, hf_cast=False)
    with torch.no_grad():
        out = layer(x.to(dev).bfloat16(), rt)
    pc = ParityCollector()
    pc.check(out.float(), ref.float(), eag.float(), "8B FP8 decoder layer infer S=2048")
    pc.done()


def test_quantisation_frees_the_bf16_projection_bytes():
    from test_modules_gpu import _build_tiny_model
    from cambrian_b200 import quant_fp8
    cfg = tiny_cambrian_config()
    model = _build_tiny_model(cfg).eval()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    stats = quant_fp8.quantize_decoder_fp8_(model, dev)
    torch.cuda.synchronize()
    after = torch.cuda.memory_allocated()
    L = cfg.num_hidden_layers
    assert stats["fp8_bytes"] == L * quant_fp8.bytes_per_layer(cfg)
    want = stats["bf16_bytes"] - stats["fp8_bytes"]
    slack = 512 * (2 * 4 * L + 7 * L)
    assert abs((before - after) - want) <= slack, (before - after, want, slack)
