"""The FP8 decode KV cache on the GPU: the append kernel bitwise against the reference quantiser of
tests/kv_fp8_reference.py (host and device slots, strided packed-qkv rows, edge rows); the decode kernel against fp64
attention over the dequantised cache by the parity criterion of tests/helpers.py, run-to-run bitwise, blind to NaN bytes
past the valid length, and equal under CUDA-graph replay; greedy decoding of the tiny model token-exact against the fp32
oracle with fake-quantised K / V, graph == eager, prefill bitwise equal to the bf16-cache run (also at batch 12 and with
FP8 weights); one Llama-3-8B-shaped layer's decode step over a 2k-position cache against the oracle on the same cache."""
import gc
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import kv_fp8_reference as KR  # noqa: E402
from helpers import ParityCollector, oracle_cfg, sd_cpu32  # noqa: E402

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
bf = torch.bfloat16
f8 = torch.float8_e4m3fn


@pytest.fixture(autouse=True)
def _release_memory():
    """collect this module's models and caches (some sit in reference cycles) before the next test measures memory"""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _bits(t):
    return t.view(torch.uint8)


def _qkv(B, S, nh, nkv, hd, seed, edge=True):
    """packed post-RoPE-like qkv rows [B*S, (nh + 2 nkv) hd] and the q / k / v views the decoder layer takes"""
    from test_kv_fp8_cpu import edge_rows
    g = torch.Generator(device=dev).manual_seed(seed)
    qkv = torch.randn(B * S, (nh + 2 * nkv) * hd, generator=g, device=dev)
    qkv[:, : hd // 8] *= 30                                          # a few large channels, as RoPE'd K has
    qkv = qkv.to(bf)
    if edge:
        rows = edge_rows(hd).to(dev)
        for i in range(min(6, B * S)):
            qkv[i, nh * hd:(nh + 1) * hd] = rows[i]                  # K head 0 of the first rows
            qkv[i, (nh + nkv) * hd:(nh + nkv + 1) * hd] = rows[5 - i]
    q = qkv[:, : nh * hd].view(B, S, nh, hd)
    k = qkv[:, nh * hd:(nh + nkv) * hd].view(B, S, nkv, hd)
    v = qkv[:, (nh + nkv) * hd:].view(B, S, nkv, hd)
    return qkv, q, k, v


def _cache(B, S_max, nkv, hd, fill=0x7F):
    kq = torch.full((B, S_max, nkv, hd), fill, dtype=torch.uint8, device=dev).view(f8)
    vq = kq.clone()
    ks = torch.full((B, S_max, nkv), float("nan"), device=dev)
    return kq, vq, ks, ks.clone()


# ------------------------------------------------------------------------------------------------ append
@pytest.mark.parametrize("B,S,nh,nkv,hd", [(1, 1, 4, 2, 64), (3, 37, 4, 2, 64), (2, 9, 32, 8, 128), (4, 5, 40, 40, 128)])
def test_append_bitwise_host_and_device_slot(B, S, nh, nkv, hd):
    from cambrian_b200 import ops
    S_max = S + 20
    _, _, k, v = _qkv(B, S, nh, nkv, hd, B * S + hd)
    assert B * S == 1 or not k.is_contiguous()                       # read in place from the packed rows
    want_k, want_ks = KR.quantize_rows(k.float())
    want_v, want_vs = KR.quantize_rows(v.float())
    for off, dev_off in ((7, None), (0, 7), (3, 4)):
        kq, vq, ks, vs = _cache(B, S_max, nkv, hd)
        od = None if dev_off is None else torch.tensor([dev_off], dtype=torch.long, device=dev)
        ops.kv_fp8_append(k, v, kq, vq, ks, vs, offset=off, offset_dev=od)
        p = off + (dev_off or 0)
        assert torch.equal(_bits(kq[:, p:p + S]), _bits(want_k)) and torch.equal(ks[:, p:p + S], want_ks)
        assert torch.equal(_bits(vq[:, p:p + S]), _bits(want_v)) and torch.equal(vs[:, p:p + S], want_vs)
        untouched = torch.ones(S_max, dtype=torch.bool)
        untouched[p:p + S] = False
        assert (_bits(kq[:, untouched]) == 0x7F).all() and ks[:, untouched].isnan().all()
    # a device slot past the buffer writes nothing
    kq, vq, ks, vs = _cache(B, S_max, nkv, hd)
    ops.kv_fp8_append(k, v, kq, vq, ks, vs, offset=0, offset_dev=torch.tensor([S_max], dtype=torch.long, device=dev))
    assert (_bits(kq) == 0x7F).all() and ks.isnan().all()


# ------------------------------------------------------------------------------------------------ decode attention
SHAPES = [(32, 8, 128), (40, 40, 128), (56, 8, 128), (4, 2, 64)]     # Llama-3-8B, Vicuna-13B (MHA), Yi-34B, tiny


def _filled(B, S_max, nkv, hd, length, seed):
    from cambrian_b200 import ops
    _, _, k, v = _qkv(B, length, 1, nkv, hd, seed, edge=False)
    kq, vq, ks, vs = _cache(B, S_max, nkv, hd)
    ops.kv_fp8_append(k, v, kq, vq, ks, vs, offset=0)
    return kq, vq, ks, vs


def _check_decode(pc, B, nh, nkv, hd, S_max, length, mask_pad, seed):
    from cambrian_b200 import ops
    kq, vq, ks, vs = _filled(B, S_max, nkv, hd, length, seed)
    _, q, _, _ = _qkv(B, 1, nh, nkv, hd, seed + 1, edge=False)
    kmask = torch.ones(B, S_max, dtype=torch.bool, device=dev)
    for b in range(B):
        kmask[b, : (b * mask_pad) % max(length - 1, 1)] = False      # left padding, a different amount per sequence
    ws = ops.attn_decode_fp8_workspace(B, nh, nkv, S_max, hd, dev)
    got = ops.attn_decode_fp8(q, kq, vq, ks, vs, ws, length=length, kmask=kmask)
    again = ops.attn_decode_fp8(q, kq, vq, ks, vs, ws, length=length, kmask=kmask)
    what = f"decode B={B} nh={nh} nkv={nkv} hd={hd} S_max={S_max} L={length}"
    assert torch.equal(got, again), what + ": not deterministic"
    assert torch.isfinite(got).all(), what + ": NaN bytes / scales past the valid length leaked"
    # the same call with zeros past the valid length: unchanged
    z = [t.clone() for t in (kq, vq, ks, vs)]
    for t in z:
        t.view(torch.uint8 if t.dtype == f8 else t.dtype)[:, length:] = 0
    assert torch.equal(got, ops.attn_decode_fp8(q, *z, ws, length=length, kmask=kmask)), what + ": reads past the length"
    ref = KR.decode_attention(q[:, 0], kq, ks, vq, vs, length, kmask)
    eag = KR.decode_attention(q[:, 0], kq, ks, vq, vs, length, kmask, dtype=bf)
    pc.check(got[:, 0].float(), ref, eag.float(), what)


@pytest.mark.parametrize("nh,nkv,hd", SHAPES)
def test_decode_attention_against_fp64(nh, nkv, hd):
    pc = ParityCollector()
    for B, S_max, length in ((1, 4096, 100), (1, 4096, 4096), (2, 1100, 257), (2, 1100, 1099), (8, 16384, 9000),
                             (1, 16384, 16384), (64, 1088, 1088), (64, 1088, 530)):
        if nh == 40 and B == 64 and length == 1088 and S_max > 0:
            B = 16                                                    # keep the MHA case's reference within memory
        _check_decode(pc, B, nh, nkv, hd, S_max, length, 37, B * nh + length)
    pc.done()


def test_decode_graph_replay_equals_eager():
    from cambrian_b200 import ops
    B, nh, nkv, hd, S_max, L0 = 4, 32, 8, 128, 2048, 1500
    kq, vq, ks, vs = _filled(B, S_max, nkv, hd, L0, 5)
    ws = ops.attn_decode_fp8_workspace(B, nh, nkv, S_max, hd, dev)
    kmask = torch.ones(B, S_max, dtype=torch.bool, device=dev)
    kmask[1, :40] = False
    steps = [_qkv(B, 1, nh, nkv, hd, 100 + i, edge=False) for i in range(3)]
    eager_cache = [t.clone() for t in (kq, vq, ks, vs)]
    eager = []
    for i, (_, q, k, v) in enumerate(steps):
        ops.kv_fp8_append(k, v, *eager_cache, offset=L0 + i)
        eager.append(ops.attn_decode_fp8(q, *eager_cache, ws, length=L0 + i + 1, kmask=kmask))
    slot = torch.tensor([L0], dtype=torch.long, device=dev)
    qkv_buf = steps[0][0].clone()
    nq = nh * hd
    q = qkv_buf[:, :nq].view(B, 1, nh, hd)
    k = qkv_buf[:, nq:nq + nkv * hd].view(B, 1, nkv, hd)
    v = qkv_buf[:, nq + nkv * hd:].view(B, 1, nkv, hd)
    out = torch.empty(B, 1, nh, hd, dtype=bf, device=dev)

    def step():
        ops.kv_fp8_append(k, v, kq, vq, ks, vs, offset_dev=slot)
        out.copy_(ops.attn_decode_fp8(q, kq, vq, ks, vs, ws, length=1, length_dev=slot, kmask=kmask))
        slot.add_(1)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()                                                       # warm-up outside capture
    torch.cuda.current_stream().wait_stream(side)
    slot.fill_(L0)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    slot.fill_(L0)
    for i, st in enumerate(steps):
        qkv_buf.copy_(st[0])
        graph.replay()
        assert torch.equal(out, eager[i]), i
    assert torch.equal(_bits(kq[:, L0:L0 + 3]), _bits(eager_cache[0][:, L0:L0 + 3]))


# ------------------------------------------------------------------------------------------------ end to end
def _first_hidden(model):
    """forward hook on the decoder: the last hidden state of its first call (the prefill)"""
    seen = []
    h = model.get_model().register_forward_hook(lambda m, a, o: seen.append(o.last_hidden_state.clone()) if not seen else None)
    return seen, h


def test_greedy_generate_fp8_cache_token_exact_graph_eager_and_prefill_bitwise():
    from test_fp8_gpu import _peaked_model
    from test_modules_gpu import _tiny_batch
    from test_parity_gpu import _bf, _oracle_greedy

    from cambrian_b200 import quant_fp8
    from oracle import cambrian_oracle as O
    cfg, model = _peaked_model()
    ids, labels, attn, pos, images, masks = _tiny_batch(cfg)
    S0, n_new = 40, 32
    gen_ids = ids[:1, :S0].clone().to(dev)
    imgs = [i[:1].to(dev).bfloat16() for i in images]
    kw = dict(image_sizes=[(56, 56)], max_new_tokens=n_new, do_sample=False)

    def run(**extra):
        seen, h = _first_hidden(model)
        try:
            toks = model.generate(gen_ids if "ids" not in extra else extra.pop("ids"),
                                  images=imgs if "imgs" not in extra else extra.pop("imgs"), **{**kw, **extra})
        finally:
            h.remove()
        return toks, seen[0]

    new, pre8 = run(kv_cache_dtype="fp8")
    model.config.disable_decode_graph = True
    eager_loop, _ = run(kv_cache_dtype="fp8")
    model.config.disable_decode_graph = False
    assert torch.equal(new, eager_loop), (new.tolist(), eager_loop.tolist())
    ref16, pre16 = run()
    assert torch.equal(pre8, pre16) and new[0, 0] == ref16[0, 0]                  # prefill bitwise the bf16-cache run's
    sd = sd_cpu32(model)
    towers = model.get_model().vision_tower_aux_list
    feats = [_bf(t(i).float().cpu()) for t, i in zip(towers, imgs)]
    real_layer = O.llama_layer
    O.llama_layer = KR.oracle_layer_kv_fp8(S0)
    try:
        t_32, m_32 = _oracle_greedy(sd, cfg, oracle_cfg(cfg), feats, gen_ids.cpu(), n_new, torch.float32,
                                    torch.device("cpu"))
    finally:
        O.llama_layer = real_layer
    got = new[0].tolist()
    assert got == t_32, f"FP8-cache greedy != fp32 oracle with fake-quantised K/V:\n{got}\n{t_32}\nmargins {m_32}"
    assert len(set(got)) >= 8
    assert min(m_32) > 2.0, f"test model lost its margin (min {min(m_32)})"
    # batch 12, then the same with FP8 weights: graph == eager, prefill bitwise the bf16-cache run's
    b_ids = gen_ids.repeat(12, 1)
    b_ids[:, -4:] = torch.randint(3, cfg.vocab_size, (12, 4), generator=torch.Generator().manual_seed(3)).to(dev)
    b_imgs = [i.repeat(12, 1, 1, 1) for i in imgs]
    for quantise in (False, True):
        if quantise:
            quant_fp8.quantize_decoder_fp8_(model, dev)
        kw12 = dict(ids=b_ids, imgs=b_imgs, image_sizes=[(56, 56)] * 12, max_new_tokens=16)
        graphed, p8 = run(kv_cache_dtype="fp8", **dict(kw12))
        model.config.disable_decode_graph = True
        eager12, _ = run(kv_cache_dtype="fp8", **dict(kw12))
        model.config.disable_decode_graph = False
        b16, p16 = run(**dict(kw12))
        assert torch.equal(graphed, eager12), (quantise, graphed.tolist(), eager12.tolist())
        assert torch.equal(p8, p16) and torch.equal(graphed[:, 0], b16[:, 0]), quantise
        assert (graphed == b16).float().mean().item() > 0.5, (quantise, graphed.tolist(), b16.tolist())


def test_llama3_8b_decoder_layer_decode_step_over_a_2k_fp8_cache():
    """One Llama-3-8B-shaped layer (H 4096, 32 q / 8 kv heads x 128, FFN 14336): a 2047-token prefill into an FP8 cache,
    then one decode step.  The step's output is held to the parity criterion against the fp32 oracle of that step over
    the same quantised cache (dequantised, plus the step's own K / V through the reference quantiser), with the oracle's
    eager-bf16 run as the yardstick."""
    import math

    import torch.nn.functional as F_

    from cambrian_b200.model.language_model.cambrian_llama import CambrianConfig, CBLlamaDecoderLayer, KVCache, rope_tables
    from helpers import both_modes
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
    S0, H, nh, nkv, hd = 2047, 4096, 32, 8, 128
    cos_t, sin_t = rope_tables(cfg, dev)
    cache = KVCache(cfg, 1, S0 + 1, dev, dtype="fp8")
    x0 = torch.randn(1, S0, H, device=dev).to(bf)
    x1 = torch.randn(1, 1, H, device=dev).to(bf)
    with torch.no_grad():
        rt = dict(pos=torch.arange(S0, device=dev), cos=cos_t, sin=sin_t, kmask=None, hf_cast=False)
        layer.infer(x0, rt, cache)
        cache.length = S0
        rt1 = dict(pos=torch.tensor([S0], device=dev), cos=cos_t, sin=sin_t, kmask=None, hf_cast=False)
        out = layer.infer(x1, rt1, cache)
    kq, vq, ks, vs = (t[:, :S0].cpu() for t in cache.fp8.layer(0))
    P = "model.layers.0."
    sd = {P + k: v.detach().float().cpu() for k, v in layer.state_dict().items()}

    def step(s, xx, kd, vd):
        h = O.rms_norm(xx, s[P + "input_layernorm.weight"], 1e-5)
        cos, sin = O.rope_cos_sin(torch.tensor([[S0]], device=xx.device), hd, 500000.0)
        q = O.apply_rope(F_.linear(h, s[P + "self_attn.q_proj.weight"]).view(1, 1, nh, hd).transpose(1, 2), cos, sin)
        k = O.apply_rope(F_.linear(h, s[P + "self_attn.k_proj.weight"]).view(1, 1, nkv, hd).transpose(1, 2), cos, sin)
        v = F_.linear(h, s[P + "self_attn.v_proj.weight"]).view(1, 1, nkv, hd).transpose(1, 2)
        kn, vn = (KR.dequantize(*KR.quantize_rows(t), dtype=xx.dtype) for t in (k, v))
        K = torch.cat([kd.to(xx.dtype), kn], 2).repeat_interleave(nh // nkv, 1)
        V = torch.cat([vd.to(xx.dtype), vn], 2).repeat_interleave(nh // nkv, 1)
        a = torch.softmax(((q @ K.transpose(-1, -2)) / math.sqrt(hd)).float(), -1).to(xx.dtype) @ V
        xx = xx + F_.linear(a.transpose(1, 2).reshape(1, 1, H), s[P + "self_attn.o_proj.weight"])
        h = O.rms_norm(xx, s[P + "post_attention_layernorm.weight"], 1e-5)
        g = F_.silu(F_.linear(h, s[P + "mlp.gate_proj.weight"])) * F_.linear(h, s[P + "mlp.up_proj.weight"])
        return xx + F_.linear(g, s[P + "mlp.down_proj.weight"])

    kd = KR.dequantize(kq, ks, torch.float32).transpose(1, 2)       # [1, nkv, S0, hd]
    vd = KR.dequantize(vq, vs, torch.float32).transpose(1, 2)
    with torch.no_grad():
        ref, eag = both_modes(step, sd, x1.float(), kd, vd, device=dev)
    pc = ParityCollector()
    pc.check(out.float(), ref.float(), eag.float(), "8B decoder layer decode step over a 2k FP8 cache")
    pc.done()
