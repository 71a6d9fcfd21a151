"""The 4-bit (NF4) inference path on the GPU: the quantiser bitwise against the torch reference of tests/nf4_reference.py,
the dequantiser bitwise, the decode GEMV under the parity criterion against the bf16 GEMV on W~, the prefill bitwise
against the bf16 model holding W~, greedy decoding token-exact against the oracles run on W~, and the memory a
quantised model gives back."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import nf4_reference as R  # noqa: E402
from helpers import ParityCollector, oracle_cfg, oracle_device, sd_cpu32, tiny_cambrian_config  # noqa: E402

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")


def _weight(N, K, seed, zero_block=False):
    g = torch.Generator(device=dev).manual_seed(seed)
    w = (torch.randn(N, K, generator=g, device=dev) * 0.02).to(torch.bfloat16)
    w[0, :K // 4] *= 8                                            # uneven block scales
    if zero_block:
        w[N // 2, :64] = 0
    return w


@pytest.mark.parametrize("N,K", [(3, 6400), (5, 64), (1024, 4096), (4096, 14336)])
def test_quantizer_bitwise_and_deterministic(N, K):
    from cambrian_b200 import quant
    w = _weight(N, K, N + K, zero_block=True)
    qw = quant.quantize(w)
    qw2 = quant.quantize(w)
    torch.cuda.synchronize()
    absmax = w.float().reshape(-1, 64).abs().amax(1)
    mean64 = absmax.double().mean().item()
    assert abs(qw.offset.item() - mean64) <= 1e-6 * abs(mean64)
    packed, q, a2, _ = R.quantize(w, offset=qw.offset)
    assert torch.equal(qw.packed, packed), "packed codes differ from the reference"
    assert torch.equal(qw.qabsmax, q), "qabsmax differs from the reference"
    assert torch.equal(qw.absmax2, a2), "absmax2 differs from the reference"
    for a, b in ((qw.packed, qw2.packed), (qw.qabsmax, qw2.qabsmax), (qw.absmax2, qw2.absmax2), (qw.offset, qw2.offset)):
        assert torch.equal(a, b), "quantising twice gave different bytes"


def _projection(rows, K, seed):
    from cambrian_b200 import quant
    parts = [quant.quantize(_weight(n, K, seed + i, zero_block=i == 1)) for i, n in enumerate(rows)]
    scratch = torch.empty(sum(rows) * K, dtype=torch.bfloat16, device=dev)
    return quant.NF4Projection(parts, scratch)


def test_dequant_is_bitwise_w_tilde():
    from cambrian_b200 import ops
    for rows, K in (([520, 264, 264], 1024), ([1000], 320), ([4096, 4096], 512)):
        qw = _projection(rows, K, 7)
        got = ops.nf4_dequant(qw).clone()
        assert torch.equal(got, R.projection_weight(qw)), (rows, K)


@pytest.mark.parametrize("M", list(range(1, 9)))
def test_gemv_nf4_parity_with_bf16_gemv_on_w_tilde(M):
    from cambrian_b200 import ops
    pc = ParityCollector()
    g = torch.Generator(device=dev).manual_seed(M)
    for rows, K in (([1000], 4096), ([520, 264], 2048 + 192), ([517, 130, 130], 1024), ([6144], 4096)):
        qw = _projection(rows, K, 11 * M)
        wt = R.projection_weight(qw)
        N = qw.N
        x = torch.randn(M, K, generator=g, device=dev).to(torch.bfloat16)
        bias = torch.randn(N, generator=g, device=dev).to(torch.bfloat16)
        res = torch.randn(M, N, generator=g, device=dev).to(torch.bfloat16)
        ref = x.double() @ wt.double().t()
        for use_bias, use_res, fp32 in ((False, False, False), (True, False, True), (False, True, False),
                                        (True, True, True)):
            b = bias if use_bias else None
            r = res if use_res else None
            od = torch.float32 if fp32 else torch.bfloat16
            got = ops.gemv_nf4(x, qw, bias=b, residual=r, out_dtype=od)
            eager = ops.gemv(x, wt, bias=b, residual=r, out_dtype=od)
            want = ref + (b.double() if b is not None else 0) + (r.double() if r is not None else 0)
            pc.check(got, want, eager, f"gemv_nf4 M={M} rows={rows} K={K} bias={use_bias} res={use_res} fp32={fp32}")
    pc.done()


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


def _w_tilde_into(model_bf16, model_q):
    """Copy W~ of every quantised projection of model_q into the bf16 weights of model_bf16 (same architecture)."""
    with torch.no_grad():
        for lb, lq in zip(model_bf16.get_model().layers, model_q.get_model().layers):
            nf = lq._nf4
            a, m = lb.self_attn, lb.mlp
            qkv = R.projection_weight(nf["qkv"])
            nq, nk = a.q_proj.weight.shape[0], a.k_proj.weight.shape[0]
            a.q_proj.weight.copy_(qkv[:nq])
            a.k_proj.weight.copy_(qkv[nq:nq + nk])
            a.v_proj.weight.copy_(qkv[nq + nk:])
            a.o_proj.weight.copy_(R.projection_weight(nf["o"]))
            gu = R.projection_weight(nf["gate_up"])
            I = m.gate_proj.weight.shape[0]
            m.gate_proj.weight.copy_(gu[:I])
            m.up_proj.weight.copy_(gu[I:])
            m.down_proj.weight.copy_(R.projection_weight(nf["down"]))


def test_prefill_is_bitwise_the_bf16_model_on_w_tilde():
    from cambrian_b200 import quant
    from cambrian_b200.model.language_model.cambrian_llama import KVCache
    cfg, model = _peaked_model()
    _, ref = _peaked_model()
    quant.quantize_decoder_nf4_(model, dev)
    _w_tilde_into(ref, model)
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(3, cfg.vocab_size, (2, 48), generator=g).to(dev)
    outs = []
    with torch.no_grad():
        for mdl in (model, ref):
            cache = KVCache(cfg, 2, 64, dev)
            outs.append(mdl.get_model()(input_ids=ids, past_key_values=cache, use_cache=True).last_hidden_state)
            outs.append(mdl(input_ids=ids).logits)                   # no cache: the no-grad scoring path
    assert torch.equal(outs[0], outs[2]), "prefill hidden states differ from the bf16 model on W~"
    assert torch.equal(outs[1], outs[3]), "cache-less logits differ from the bf16 model on W~"


def test_greedy_generate_4bit_token_exact():
    from test_modules_gpu import _tiny_batch
    from test_parity_gpu import _bf, _oracle_greedy
    from cambrian_b200 import quant
    cfg, model = _peaked_model()
    _, ref = _peaked_model()
    quant.quantize_decoder_nf4_(model, dev)
    _w_tilde_into(ref, model)
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
    sd = sd_cpu32(ref)
    towers = ref.get_model().vision_tower_aux_list
    feats = [_bf(t(i).float().cpu()) for t, i in zip(towers, imgs)]
    t_bf, m_bf = _oracle_greedy(sd, cfg, oracle_cfg(cfg), feats, gen_ids.cpu(), n_new, torch.bfloat16, oracle_device())
    t_32, m_32 = _oracle_greedy(sd, cfg, oracle_cfg(cfg), feats, gen_ids.cpu(), n_new, torch.float32, oracle_device())
    assert got == t_bf, f"4-bit greedy != eager-bf16 oracle on W~:\n{got}\n{t_bf}\nmargins {m_bf}"
    assert got == t_32, f"4-bit greedy != fp32 oracle on W~:\n{got}\n{t_32}\nmargins {m_32}"
    assert len(set(got)) >= 8
    # a batch of 12: the decode projections take the dequantise + GEMM path inside the captured graph
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
    from cambrian_b200 import quant
    cfg = tiny_cambrian_config()
    model = _build_tiny_model(cfg).eval()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    stats = quant.quantize_decoder_nf4_(model, dev)
    torch.cuda.synchronize()
    after = torch.cuda.memory_allocated()
    L = cfg.num_hidden_layers
    assert stats["nf4_bytes"] == L * quant.bytes_per_layer(cfg)
    want = stats["bf16_bytes"] - stats["nf4_bytes"] - stats["scratch_bytes"]
    slack = 512 * (4 * 7 * L + 7 * L + 2)                          # the caching allocator rounds every block to 512 B
    assert abs((before - after) - want) <= slack, (before - after, want, slack)
