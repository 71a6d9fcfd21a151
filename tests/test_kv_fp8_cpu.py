"""CPU checks of the FP8 decode KV cache: the reference row rule on edge rows, KVCache sizes, `kv_cache_dtype` resolution
and refusals, argument validation of the two entry points, and the host logic of generate() with the FP8 cache against
the fp32 oracle whose decode steps attend over K / V passed through the reference quantiser.  The kernels are replaced by
the plain-torch stand-ins of tests/kv_fp8_reference.py; their numerics are covered under `-m gpu`
(tests/test_kv_fp8_gpu.py)."""
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import fp8_reference as R  # noqa: E402
import kv_fp8_reference as KR  # noqa: E402
import ops_emulation  # noqa: E402
from helpers import tiny_cambrian_config  # noqa: E402

needs_no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="kernel stand-ins are for GPU-less machines only")
bf = torch.bfloat16


def _bits(t):
    return t.view(torch.uint8).tolist()


def edge_rows(hd):
    """[6, hd] bf16 head rows: saturation at the amax element, a zero row, a row of signed zeros, a row reaching the
    subnormal range, a row of bf16 subnormals (448 / amax overflows fp32) and a negative underflow to -0."""
    w = torch.zeros(6, hd, dtype=bf)
    w[0, :4] = torch.tensor([2.0, -1.0, 0.5, 0.25])
    w[2, 0] = w[2, 1] = -0.0
    w[3, :3] = torch.tensor([3.0, 3.0 * 2 ** -8, 3.0 * 2 ** -11])
    w[4, :2] = torch.tensor([2.0 ** -133, -(2.0 ** -130)], dtype=bf)
    w[5, :2] = torch.tensor([1.0, -1e-6])
    return w


@pytest.mark.parametrize("hd", [64, 128])
def test_reference_row_rule_on_edge_rows(hd):
    rows = edge_rows(hd)
    q, s = KR.quantize_rows(rows.view(1, 6, 1, hd))
    assert q.shape == (1, 6, 1, hd) and s.shape == (1, 6, 1)
    q, s = q.view(6, hd), s.view(6)
    want_q, want_s = R.quantize_rows(rows)
    assert _bits(q) == _bits(want_q) and torch.equal(s, want_s)
    qf = q.float()
    assert qf[0, 0].item() == 448.0 and s[0].item() == (torch.tensor(2.0) / 448).item()      # saturation at amax, exact
    assert s[1].item() == 0.0 and _bits(q[1]) == [0] * hd                                    # zero row
    assert s[2].item() == 0.0 and _bits(q[2])[:3] == [0x80, 0x80, 0]                         # signed zeros survive
    assert s[4].item() > 0 and 0 < qf[4].abs().max().item() < 448                            # bf16 subnormals: no NaN
    assert _bits(q[5, 1:2]) == [0x80]                                                        # -1e-6 * 448 -> -0
    assert not torch.isnan(qf).any()
    deq = KR.dequantize(q, s)
    assert torch.equal(deq[1], torch.zeros(hd, dtype=torch.float64))
    x = rows[0, :4].double()                                 # q exact (448, -224, ...): only s = 2 / 448 is fp32-rounded
    assert ((deq[0, :4] - x).abs() <= 2.0 ** -24 * x.abs()).all()


def test_kv_cache_sizes_and_nbytes(monkeypatch):
    from cambrian_b200.model.language_model.cambrian_llama import KVCache
    KR.install(monkeypatch)
    cfg = tiny_cambrian_config()
    L, nkv, hd, B, S_max = cfg.num_hidden_layers, cfg.num_key_value_heads, cfg.hidden_size // cfg.num_attention_heads, 3, 80
    c16 = KVCache(cfg, B, S_max, "cpu")
    assert c16.dtype == "bf16" and c16.fp8 is None and c16.nbytes() == L * 2 * B * S_max * nkv * hd * 2
    c8 = KVCache(cfg, B, S_max, "cpu", dtype="fp8")
    assert c8.k is None and c8.v is None and c8.fp8 is not None
    kq, vq, ks, vs = c8.fp8.layer(0)
    assert kq.dtype == vq.dtype == torch.float8_e4m3fn and kq.shape == vq.shape == (B, S_max, nkv, hd)
    assert ks.dtype == vs.dtype == torch.float32 and ks.shape == vs.shape == (B, S_max, nkv)
    assert all(not t.any() for i in range(L) for t in (c8.fp8.ks[i], c8.fp8.vs[i]))        # scales start at zero
    from cambrian_b200 import kv_fp8
    assert c8.nbytes() == L * 2 * B * S_max * nkv * (hd + 4) + c8.fp8.ws.numel() * 4
    assert c8.nbytes() - c8.fp8.ws.numel() * 4 == kv_fp8.bytes_per_token(cfg) * B * S_max
    assert (128 + 4) / (2 * 128) == pytest.approx(0.516, abs=1e-3)                          # 51.6 % of bf16 at hd 128
    with pytest.raises(ValueError, match="dtype"):
        KVCache(cfg, B, S_max, "cpu", dtype="int8")


def test_kv_cache_dtype_resolution():
    from cambrian_b200.kv_fp8 import resolve_cache_dtype
    cfg = tiny_cambrian_config()
    assert resolve_cache_dtype(cfg) == "bf16" and resolve_cache_dtype(cfg, "fp8") == "fp8"
    cfg.kv_cache_dtype = "fp8"
    assert resolve_cache_dtype(cfg) == "fp8" and resolve_cache_dtype(cfg, "bf16") == "bf16"
    cfg.kv_cache_dtype = None
    assert resolve_cache_dtype(cfg) == "bf16"
    for bad in ("int8", "fp16", "float8_e4m3fn", 8):
        with pytest.raises(ValueError, match="kv_cache_dtype"):
            resolve_cache_dtype(cfg, bad)


def test_entry_point_argument_validation_without_gpu(lib):
    one = ctypes.c_void_p(16)                                   # non-null, 16-byte aligned dummy pointer (never dereferenced)
    odd = ctypes.c_void_p(20)
    f = ctypes.c_float(0.125)

    def dec(q=one, q_bs=768, B=1, Sq=1, nh=4, nkv=2, S_max=64, hd=64, length=8, kmask=None, kmask_ld=0, ws_floats=1 << 20):
        return lib.cb_attn_decode_fp8(q, q_bs, one, one, one, one, kmask, kmask_ld, one, one, ws_floats, B, Sq, nh, nkv,
                                      S_max, hd, length, None, f, None)

    for kw, msg in ((dict(Sq=2), b"Sq"), (dict(hd=96), b"hd"), (dict(nh=32, nkv=2), b"nh"), (dict(nh=6, nkv=4), b"nh"),
                    (dict(q=odd), b"aligned"), (dict(q_bs=772), b"aligned"), (dict(length=65), b"length"),
                    (dict(kmask=one, kmask_ld=4), b"kmask")):
        assert dec(**kw) == 1 and msg in lib.cb_last_error(), (kw, lib.cb_last_error())
    assert lib.cb_attn_decode_fp8_workspace_floats(0, 4, 2, 64, 64) == 0
    assert lib.cb_attn_decode_fp8_workspace_floats(1, 32, 8, 4096, 128) % (32 * 130) == 0

    def app(k=one, ld=384, S=1, S_max=64, hd=64, offset=0):
        return lib.cb_kv_fp8_append(k, one, ld, one, one, one, one, 1, S, S_max, 2, hd, offset, None, None)

    for kw, msg in ((dict(hd=96), b"hd"), (dict(k=odd), b"aligned"), (dict(ld=100), b"stride"),
                    (dict(S=4, offset=62), b"outside")):
        assert app(**kw) == 1 and msg in lib.cb_last_error(), (kw, lib.cb_last_error())


# ------------------------------------------------------------------------------------------------ generate()
def _peaked(cfg):
    from test_fp8_cpu import _build
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
    return model.eval()


@needs_no_gpu
def test_greedy_generate_fp8_cache_routes_decode_and_matches_the_oracle(monkeypatch):
    from test_model_host_logic_cpu import _batch, _tower_feats
    from test_parity_gpu import _oracle_greedy

    from cambrian_b200 import ops
    from helpers import oracle_cfg
    from oracle import cambrian_oracle as O
    ops_emulation.install(monkeypatch)
    KR.install(monkeypatch)
    calls = []
    for name in ("attn_fwd", "attn_decode_fp8", "kv_fp8_append"):
        fn = getattr(ops, name)
        monkeypatch.setattr(ops, name, lambda *a, _n=name, _f=fn, **k: calls.append(_n) or _f(*a, **k))
    cfg = tiny_cambrian_config()
    cfg.fused_lm_loss = True
    model = _peaked(cfg)
    L = cfg.num_hidden_layers
    ids, _, _, _, _ = _batch(cfg, S=96)
    S0, n_new = 40, 12
    gen_ids = ids[:1, :S0].clone()
    feats = [f[:1] for f in _tower_feats(model, cfg, 2, 31)]
    monkeypatch.setattr(type(model), "encode_images", lambda self, imgs: feats)
    images = [torch.zeros(1, 3, 8, 8, dtype=bf) for _ in feats]
    kw = dict(images=images, image_sizes=[(56, 56)], max_new_tokens=n_new, do_sample=False)
    new = model.generate(gen_ids, kv_cache_dtype="fp8", **kw)
    # prefill: the flash kernel on the prompt's own K / V, then one append per layer; every decode step: append, then
    # the FP8 decode kernel, never the flash kernel
    assert calls[:2 * L] == ["attn_fwd", "kv_fp8_append"] * L
    assert calls[2 * L:] == ["kv_fp8_append", "attn_decode_fp8"] * (L * (n_new - 1))
    calls.clear()
    bf16_run = model.generate(gen_ids, **kw)
    assert "attn_decode_fp8" not in calls and "kv_fp8_append" not in calls           # the default keeps today's path
    assert new[0, 0] == bf16_run[0, 0]                                                   # the first token comes from prefill
    sd = {k: v.detach().float() for k, v in model.state_dict().items()}
    monkeypatch.setattr(O, "llama_layer", KR.oracle_layer_kv_fp8(S0))      # the spliced prompt keeps its length S0
    want, margins = _oracle_greedy(sd, cfg, oracle_cfg(cfg), [f.float() for f in feats], gen_ids, n_new, torch.float32,
                                   torch.device("cpu"))
    assert new[0].tolist() == want, (new[0].tolist(), want, margins)
    assert len(set(want)) >= 4 and min(margins) > 1.0, margins
    cfg.kv_cache_dtype = "fp8"                                                           # the config default
    calls.clear()
    assert torch.equal(model.generate(gen_ids, **kw), new) and "attn_decode_fp8" in calls
    cfg.kv_cache_dtype = "bf16"


@needs_no_gpu
def test_fp8_cache_with_left_padding_sampling_and_stopping(monkeypatch):
    """attention_mask with left padding, sampling, a streamer and stopping criteria run through the FP8 cache's eager loop."""
    from test_model_host_logic_cpu import _batch, _tower_feats
    ops_emulation.install(monkeypatch)
    KR.install(monkeypatch)
    cfg = tiny_cambrian_config()
    model = _peaked(cfg)
    ids, _, _, _, _ = _batch(cfg, S=96)
    gen_ids = ids[:2, :40].clone()
    mask = torch.ones_like(gen_ids)
    gen_ids[1, :3] = 0
    mask[1, :3] = 0
    feats = _tower_feats(model, cfg, 2, 31)
    monkeypatch.setattr(type(model), "encode_images", lambda self, imgs: feats)
    images = [torch.zeros(2, 3, 8, 8, dtype=bf) for _ in feats]
    seen = []

    class Streamer:
        def put(self, t):
            seen.append(t.shape)

        def end(self):
            seen.append("end")

    stop_after = 5
    out = model.generate(gen_ids, images=images, image_sizes=[(56, 56)] * 2, attention_mask=mask, max_new_tokens=9,
                         do_sample=True, top_k=20, generator=torch.Generator().manual_seed(0), streamer=Streamer(),
                         stopping_criteria=[lambda toks, scores: toks.shape[1] >= stop_after], kv_cache_dtype="fp8")
    assert out.shape == (2, stop_after) and seen[-1] == "end" and len(seen) == stop_after + 2


def test_generate_refusals(monkeypatch):
    from cambrian_b200.model.language_model.cambrian_llama import CambrianLlamaForCausalLM
    cfg = tiny_cambrian_config()
    torch.manual_seed(0)
    model = CambrianLlamaForCausalLM(cfg).eval()
    ids = torch.ones(1, 8, dtype=torch.long)
    with pytest.raises(ValueError, match="kv_cache_dtype"):
        model.generate(ids, kv_cache_dtype="int4", max_new_tokens=2)
    model.get_model()._zero3 = object()
    with pytest.raises(NotImplementedError, match="Zero3Inference"):
        model.generate(ids, kv_cache_dtype="fp8", max_new_tokens=2)
    del model.get_model()._zero3
    for kw in (dict(num_beams=2), dict(repetition_penalty=1.3), dict(cache_implementation="quantized")):
        with pytest.raises(NotImplementedError, match=list(kw)[0]):
            model.generate(ids, kv_cache_dtype="fp8", max_new_tokens=2, **kw)


@needs_no_gpu
def test_fp8_cache_refuses_a_multi_token_step_on_a_filled_cache(monkeypatch):
    from test_model_host_logic_cpu import _batch
    from cambrian_b200.model.language_model.cambrian_llama import KVCache
    ops_emulation.install(monkeypatch)
    KR.install(monkeypatch)
    cfg = tiny_cambrian_config()
    from test_fp8_cpu import _build
    model = _build(cfg).eval()
    ids = _batch(cfg, S=96)[0][:1, 20:30].clamp(min=3)
    cache = KVCache(cfg, 1, 32, "cpu", dtype="fp8")
    with torch.no_grad():
        model.get_model()(input_ids=ids[:, :6], past_key_values=cache, use_cache=True)
        assert cache.length == 6 and cache.fp8.ks[0][:, :6].gt(0).all() and not cache.fp8.ks[0][:, 6:].any()
        model.get_model()(input_ids=ids[:, 6:7], past_key_values=cache, use_cache=True)
        assert cache.length == 7 and cache.fp8.ks[0][:, 6].gt(0).all()
        with pytest.raises(NotImplementedError, match="FP8 KV cache"):
            model.get_model()(input_ids=ids[:, 7:9], past_key_values=cache, use_cache=True)
