"""CPU checks of FP8 training (`config.fp8_training`, cambrian_b200/train_fp8.py): argument validation of the three new
entry points, the routing of a decoder layer's GEMMs (forward and input-gradient GEMMs through the FP8 GEMM, every
weight gradient through the bf16 GEMM into main_grad), recompute on / off, generate() untouched by the flag, and the
refusal of widths that are not multiples of 16.  The kernels are replaced by the torch stand-ins of
tests/fp8_train_reference.py; their numerics are covered under `-m gpu` (tests/test_fp8_train_gpu.py)."""
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import fp8_train_reference as T  # noqa: E402
import ops_emulation  # noqa: E402
from helpers import tiny_cambrian_config  # noqa: E402

needs_no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="kernel stand-ins are for GPU-less machines only")
bf = torch.bfloat16


# ------------------------------------------------------------------------------------------------ C ABI
def test_argument_validation_of_the_training_entry_points_without_gpu():
    from cambrian_b200 import _lib
    lib = _lib.load()
    assert lib.cb_fp8_quantize_weight_t_workspace_floats(0, 64) == 0
    # N not a multiple of 16
    rc = lib.cb_fp8_quantize_weight_t(None, 40, 64, 64, None, None, None, 0, None)
    assert rc == 1 and b"fp8_quantize_weight_t" in lib.cb_last_error() and b"N=40" in lib.cb_last_error()
    rc = lib.cb_fp8_quantize_weight_t(None, 64, 64, 64, None, None, None, 0, None)
    assert rc == 1 and b"null" in lib.cb_last_error()
    rc = lib.cb_rmsnorm_fwd_fp8(None, None, None, None, None, 4, 40, ctypes.c_float(1e-5), 0, None)
    assert rc == 1 and b"rmsnorm_fwd_fp8" in lib.cb_last_error() and b"C=40" in lib.cb_last_error()
    rc = lib.cb_rmsnorm_fwd_fp8(None, None, None, None, None, 4, 64, ctypes.c_float(1e-5), 0, None)
    assert rc == 1 and b"null" in lib.cb_last_error()
    rc = lib.cb_swiglu_bwd_fp8(None, None, None, None, None, None, None, 4, 12, 24, 12, 24, None)
    assert rc == 1 and b"swiglu_bwd_fp8" in lib.cb_last_error() and b"I=12" in lib.cb_last_error()
    rc = lib.cb_swiglu_bwd_fp8(None, None, None, None, None, None, None, 4, 16, 32, 16, 32, None)
    assert rc == 1 and b"null" in lib.cb_last_error()


def test_ops_wrappers_refuse_bad_shapes(monkeypatch):
    from cambrian_b200 import ops
    monkeypatch.setattr(ops, "_require_cuda_bf16", lambda *a: None)
    w = torch.zeros(32, 48, dtype=bf)
    with pytest.raises(ValueError, match="fp8_quantize_weight_t"):
        ops.fp8_quantize_weight_t(w, torch.empty(32, 48, dtype=torch.float8_e4m3fn), torch.empty(48))
    g = torch.zeros(4, 32, dtype=bf)
    with pytest.raises(ValueError, match="swiglu_bwd_fp8"):
        ops.swiglu_bwd_fp8(g, g, g[:, :16], g, g)


def test_reference_transposed_and_dual_output_rules():
    """The emulations restate the row rule on the stated rows: W^T's rows, and the whole [dgate | dup] row."""
    import fp8_reference as R
    g = torch.Generator().manual_seed(0)
    w = (torch.randn(48, 32, generator=g) * 0.02).to(bf)
    w[:, 3] = 0                                                   # a zero column of W is a zero row of W^T
    q, s = T.quantize_weight_t(w)
    qr, sr = R.quantize_rows(w.t().contiguous())
    assert torch.equal(q.view(torch.uint8), qr.view(torch.uint8)) and torch.equal(s, sr) and s[3] == 0
    dg, du = torch.randn(5, 16, generator=g).to(bf), (torch.randn(5, 16, generator=g) * 9).to(bf)
    q, s = T.quantize_dgu(dg, du)
    assert q.shape == (5, 32) and torch.equal(s, torch.cat([dg, du], 1).float().abs().amax(1) / 448)


# ------------------------------------------------------------------------------------------------ the decoder layer
def _layer(cfg, seed=0):
    from cambrian_b200.model.language_model.cambrian_llama import CBLlamaDecoderLayer
    torch.manual_seed(seed)
    layer = CBLlamaDecoderLayer(cfg, 0)
    with torch.no_grad():
        for p in layer.parameters():
            p.copy_(torch.randn_like(p) * 0.05 if p.dim() == 2 else 1 + 0.1 * torch.randn_like(p))
    return layer.to(bf)


def _rt(cfg, B, S, recompute, fp8=True):
    from cambrian_b200.model.language_model.cambrian_llama import rope_tables
    cos, sin = rope_tables(cfg, torch.device("cpu"))
    pos = torch.arange(S).repeat(B)
    return dict(pos=pos, cos=cos, sin=sin, kmask=None, hf_cast=False, recompute=recompute, fp8=fp8)


def _with_main_grad(layer):
    """TrainEngine-like buffers: one flat bf16 gradient buffer in named_parameters() order, main_grad views into it."""
    params = [p for _, p in layer.named_parameters()]
    flat = torch.zeros(sum(p.numel() for p in params), dtype=bf)
    o = 0
    for p in params:
        p.main_grad = flat[o:o + p.numel()].view_as(p)
        p._cb_fresh = set()
        o += p.numel()
    return flat


def _run(layer, cfg, recompute, fp8=True, B=2, S=24, seed=1):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, S, cfg.hidden_size, generator=g).to(bf).requires_grad_()
    dout = torch.randn(B, S, cfg.hidden_size, generator=g).to(bf)
    out = layer(x, _rt(cfg, B, S, recompute, fp8))
    out.backward(dout)
    return out.detach(), x.grad


@needs_no_gpu
@pytest.mark.parametrize("recompute", [False, True])
def test_flag_routes_fwd_and_dgrad_through_fp8_and_wgrad_through_bf16_into_main_grad(monkeypatch, recompute):
    from cambrian_b200 import ops
    ops_emulation.install(monkeypatch)
    T.install(monkeypatch)
    calls = dict(fp8=[], bf16=[], wt=0, rows=0, norm_fp8=0, swiglu_fp8=0)
    real_fp8, real_gemm = ops.gemm_fp8, ops.gemm
    real_wt, real_w, real_norm, real_sw = (ops.fp8_quantize_weight_t, ops.fp8_quantize_weight, ops.rmsnorm_fwd_fp8,
                                           ops.swiglu_bwd_fp8)

    def gemm_fp8(qa, qw, **kw):
        calls["fp8"].append((qa[0].shape[0], qw.N, qw.K))
        return real_fp8(qa, qw, **kw)

    def gemm(a, b, **kw):
        calls["bf16"].append((kw.get("a_mn"), kw.get("b_mn"), kw.get("out")))
        return real_gemm(a, b, **kw)

    def count(key, fn):
        def f(*a, **k):
            calls[key] += 1
            return fn(*a, **k)
        return f

    monkeypatch.setattr(ops, "gemm_fp8", gemm_fp8)
    monkeypatch.setattr(ops, "gemm", gemm)
    monkeypatch.setattr(ops, "fp8_quantize_weight_t", count("wt", real_wt))
    monkeypatch.setattr(ops, "fp8_quantize_weight", count("rows", real_w))
    monkeypatch.setattr(ops, "rmsnorm_fwd_fp8", count("norm_fp8", real_norm))
    monkeypatch.setattr(ops, "swiglu_bwd_fp8", count("swiglu_fp8", real_sw))
    monkeypatch.setattr(ops, "mlp_gate_up", lambda *a, **k: pytest.fail("the bf16 gate|up GEMM ran under fp8_training"))
    cfg = tiny_cambrian_config()
    layer = _layer(cfg)
    _with_main_grad(layer)
    B, S = 2, 24
    _run(layer, cfg, recompute, B=B, S=S)
    H, I = cfg.hidden_size, cfg.intermediate_size
    hd = H // cfg.num_attention_heads
    nq = (cfg.num_attention_heads + 2 * cfg.num_key_value_heads) * hd
    M = B * S
    fwd = [(M, nq, H), (M, H, cfg.num_attention_heads * hd), (M, 2 * I, H), (M, H, I)]
    dgrad = [(M, I, H), (M, H, 2 * I), (M, cfg.num_attention_heads * hd, H), (M, H, nq)]
    recomputed = fwd[:3] if recompute else []                  # the recompute stops before the down projection
    assert calls["fp8"] == fwd + recomputed + dgrad
    # every bf16 GEMM is a weight gradient accumulating into main_grad (down, gate|up, o, q|k|v)
    assert len(calls["bf16"]) == 4
    flat = layer.mlp.down_proj.weight.main_grad.untyped_storage().data_ptr()
    for a_mn, b_mn, out in calls["bf16"]:
        assert a_mn and b_mn and out is not None and out.untyped_storage().data_ptr() == flat
    assert all(p.grad is None for p in layer.parameters())     # autograd received None: everything went to main_grad
    assert calls["wt"] == 4 and calls["rows"] == 4 + len(recomputed)
    assert calls["norm_fp8"] == 2 + (2 if recompute else 0) and calls["swiglu_fp8"] == 1
    for n, p in layer.named_parameters():
        assert p.main_grad.float().abs().sum() > 0, n


@needs_no_gpu
def test_recompute_on_and_off_give_identical_gradients(monkeypatch):
    ops_emulation.install(monkeypatch)
    T.install(monkeypatch)
    cfg = tiny_cambrian_config()
    res = {}
    for recompute in (False, True):
        layer = _layer(cfg)
        out, dx = _run(layer, cfg, recompute)
        res[recompute] = (out, dx, {n: p.grad.clone() for n, p in layer.named_parameters()})
    (o0, d0, g0), (o1, d1, g1) = res[False], res[True]
    assert torch.equal(o0, o1) and torch.equal(d0, d1)
    for n in g0:
        assert torch.equal(g0[n], g1[n]), n


@needs_no_gpu
def test_fp8_layer_differs_from_bf16_only_by_quantisation(monkeypatch):
    """With the stand-ins the FP8 layer is the bf16 layer with E4M3 operands: close (E4M3 keeps 4 significant bits), not
    equal."""
    ops_emulation.install(monkeypatch)
    T.install(monkeypatch)
    cfg = tiny_cambrian_config()
    o8, d8 = _run(_layer(cfg), cfg, False, fp8=True)
    o16, d16 = _run(_layer(cfg), cfg, False, fp8=False)
    rel = lambda a, b: ((a.float() - b.float()).norm() / b.float().norm()).item()
    assert 0 < rel(o8, o16) < 2 ** -4 and 0 < rel(d8, d16) < 2 ** -3


@needs_no_gpu
@pytest.mark.parametrize("field,value,name", [("hidden_size", 264, "hidden_size"),
                                              ("intermediate_size", 520, "intermediate_size"),
                                              ("head_dim", 72, "q|k|v width")])
def test_width_not_a_multiple_of_16_is_refused(monkeypatch, field, value, name):
    ops_emulation.install(monkeypatch)
    T.install(monkeypatch)
    cfg = tiny_cambrian_config()
    if field == "hidden_size":
        cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim = 2, 2, 128
    if field == "head_dim":
        cfg.num_attention_heads, cfg.num_key_value_heads = 3, 1              # q|k|v = 5 x 72 = 360 (a multiple of 8 only)
    setattr(cfg, field, value)
    layer = _layer(cfg)
    with pytest.raises(ValueError, match=f"fp8_training: {name}"):
        _run(layer, cfg, False, fp8=True)


@needs_no_gpu
def test_flag_changes_nothing_in_generate(monkeypatch):
    from cambrian_b200 import ops
    from test_fp8_cpu import _build
    from test_model_host_logic_cpu import _batch, _tower_feats
    ops_emulation.install(monkeypatch)
    T.install(monkeypatch)
    for n in ("gemm_fp8", "fp8_quantize_act", "fp8_quantize_weight", "fp8_quantize_weight_t", "rmsnorm_fwd_fp8",
              "swiglu_bwd_fp8"):
        monkeypatch.setattr(ops, n, lambda *a, _n=n, **k: pytest.fail(f"{_n} ran in generate()"))
    cfg = tiny_cambrian_config()
    cfg.fused_lm_loss = True
    model = _build(cfg)
    model.eval()
    ids, _, _, _, _ = _batch(cfg, S=64)
    feats = [f[:1] for f in _tower_feats(model, cfg, 2, 31)]
    monkeypatch.setattr(type(model), "encode_images", lambda self, imgs: feats)
    images = [torch.zeros(1, 3, 8, 8, dtype=bf) for _ in feats]
    gen_ids = ids[:1, :32].clone()
    runs = []
    for flag in (False, True):
        cfg.fp8_training = flag
        runs.append(model.generate(gen_ids, images=images, image_sizes=[(56, 56)], max_new_tokens=6, do_sample=False))
    assert torch.equal(runs[0], runs[1])
