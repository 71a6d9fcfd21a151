"""FP8 training (`config.fp8_training`) on the GPU: the three new kernels bitwise against their emulations at the
Llama-3.2-3B and Llama-3-8B training shapes (stacked q|k|v views, zero / subnormal / saturating rows and columns, row
counts that are not a multiple of the tile); one 3B-shaped decoder layer forward + backward against an fp64 emulation
that quantises at the same points, and against the bf16 layer; TrainEngine steps bitwise reproducible; and a small model
memorising a batch in FP8 as well as in bf16."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import fp8_reference as R  # noqa: E402
import fp8_train_reference as T  # noqa: E402
from helpers import tiny_cambrian_config  # noqa: E402

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
bf = torch.bfloat16
f8 = torch.float8_e4m3fn

# (H, I, nh, nkv, hd) of the shipped training shapes
SHAPES = {"3b": (3072, 8192, 24, 8, 128), "8b": (4096, 14336, 32, 8, 128)}


def _bits(t):
    return t.view(torch.uint8)


def _gen(seed):
    return torch.Generator(device=dev).manual_seed(seed)


# ------------------------------------------------------------------------------------------------ transposed weights
def _fused_weight(N_list, K, seed):
    """len(N_list) weights stacked by rows in one flat buffer (the TrainEngine layout of q|k|v and gate|up), with a zero
    column, a column of bf16 subnormals and columns of large values (the rule scales a column amax to 448 exactly)"""
    g = _gen(seed)
    N = sum(N_list)
    w = (torch.randn(N, K, generator=g, device=dev) * 0.02)
    w[:, 5] = 0
    w[:, 7] = 2.0 ** -130 * torch.sign(torch.randn(N, generator=g, device=dev))
    w[:, 9] *= 5000.0
    w[0, 11] = -1e4
    return w.to(bf)


@pytest.mark.parametrize("shape", list(SHAPES))
def test_weight_t_quantizer_bitwise_at_training_shapes(shape):
    from cambrian_b200 import ops, train_fp8
    H, I, nh, nkv, hd = SHAPES[shape]
    cases = [([nh * hd, nkv * hd, nkv * hd], H), ([H], nh * hd), ([I, I], H), ([H], I)]
    for i, (Ns, K) in enumerate(cases):
        w = _fused_weight(Ns, K, 100 * i + len(shape))
        a, b = train_fp8.weight_t(w), train_fp8.weight_t(w)
        q, s = T.quantize_weight_t(w)
        want_q = torch.empty(K, w.shape[0], dtype=f8, device=dev)
        want_s = torch.empty(K, dtype=torch.float32, device=dev)
        ops.fp8_quantize_weight(w.t().contiguous(), want_q, want_s)
        assert torch.equal(_bits(a.w.wq), _bits(want_q)) and torch.equal(a.w.sw, want_s), (shape, Ns, K)
        assert torch.equal(_bits(a.w.wq), _bits(q)) and torch.equal(a.w.sw, s), (shape, Ns, K)
        assert torch.equal(_bits(a.w.wq), _bits(b.w.wq)) and torch.equal(a.w.sw, b.w.sw)
        assert a.w.sw[5] == 0 and not torch.isnan(a.w.wq.float()).any()


def test_weight_t_quantizer_row_stride_and_tails():
    """A weight seen through a wider row stride (a column block of a larger buffer), N and K not multiples of 64."""
    from cambrian_b200 import ops
    big = _fused_weight([80], 112 + 48, 7)
    w = big[:, :112]
    wtq = torch.empty(112, 80, dtype=f8, device=dev)
    st = torch.empty(112, dtype=torch.float32, device=dev)
    ops.fp8_quantize_weight_t(w, wtq, st)
    q, s = T.quantize_weight_t(w)
    assert torch.equal(_bits(wtq), _bits(q)) and torch.equal(st, s)


# ------------------------------------------------------------------------------------------------ RMSNorm -> E4M3
def _hidden(M, H, seed):
    g = _gen(seed)
    x = torch.randn(M, H, generator=g, device=dev)
    x[:, : H // 256] *= 60                                         # a few large features
    x[3] = 0                                                       # a zero row: y = 0, s = 0
    x[5] *= 1e-30                                                  # a tiny row: rstd = rsqrt(eps), y near bf16 subnormals
    return x.to(bf)


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("hf_cast", [False, True])
def test_rmsnorm_fwd_fp8_bitwise(shape, hf_cast):
    from cambrian_b200 import ops
    H = SHAPES[shape][0]
    M = 4099                                                      # not a multiple of any tile
    x = _hidden(M, H, H + int(hf_cast))
    gamma = (1 + 0.2 * torch.randn(H, generator=_gen(1), device=dev)).to(bf)
    for gm in (gamma, (gamma.float() * 2.0 ** -126).to(bf)):      # the second makes every row bf16 subnormals
        (q, s), rstd = ops.rmsnorm_fwd_fp8(x, gm, 1e-5, hf_cast)
        h, rstd_ref = ops.rmsnorm_fwd(x, gm, 1e-5, hf_cast, save_stats=True)
        wq, ws = ops.fp8_quantize_act(h)
        assert torch.equal(rstd, rstd_ref)
        assert torch.equal(_bits(q), _bits(wq)) and torch.equal(s, ws)
        rq, rs = R.quantize_act(h)
        assert torch.equal(_bits(q), _bits(rq)) and torch.equal(s, rs)
        (q2, s2), _ = ops.rmsnorm_fwd_fp8(x, gm, 1e-5, hf_cast)
        assert torch.equal(_bits(q), _bits(q2)) and torch.equal(s, s2)
        assert s[3] == 0 and not torch.isnan(q.float()).any()


# ------------------------------------------------------------------------------------------------ SwiGLU bwd -> E4M3
@pytest.mark.parametrize("shape", list(SHAPES))
def test_swiglu_bwd_fp8_bitwise(shape):
    from cambrian_b200 import ops
    I = SHAPES[shape][1]
    M = 4099
    g = _gen(I)
    gu = (torch.randn(M, 2 * I, generator=g, device=dev) * 3).to(bf)
    dact = torch.randn(M, I, generator=g, device=dev)
    dact[1] = 0                                                   # a zero row
    dact[2] *= 1e-38                                              # a row of subnormal gradients
    dact[4] *= 1e30                                               # a row of huge gradients
    dact = dact.to(bf)
    dgu = torch.empty(M, 2 * I, dtype=bf, device=dev)
    q, s = ops.swiglu_bwd_fp8(dact, gu[:, :I], gu[:, I:], dgu[:, :I], dgu[:, I:])
    ref = torch.empty_like(dgu)
    ops.swiglu_bwd(dact, gu[:, :I], gu[:, I:], ref[:, :I], ref[:, I:])
    assert torch.equal(dgu, ref)
    wq, ws = ops.fp8_quantize_act(ref)
    assert torch.equal(_bits(q), _bits(wq)) and torch.equal(s, ws)
    rq, rs = T.quantize_dgu(ref[:, :I], ref[:, I:])
    assert torch.equal(_bits(q), _bits(rq)) and torch.equal(s, rs)
    q2, s2 = ops.swiglu_bwd_fp8(dact, gu[:, :I], gu[:, I:], dgu[:, :I], dgu[:, I:])
    assert torch.equal(_bits(q), _bits(q2)) and torch.equal(s, s2)
    assert s[1] == 0 and not torch.isnan(q.float()).any()


# ------------------------------------------------------------------------------------------------ one decoder layer
def _layer_cfg(shape):
    from cambrian_b200.model.language_model.cambrian_llama import CambrianConfig
    H, I, nh, nkv, hd = SHAPES[shape]
    return CambrianConfig(hidden_size=H, intermediate_size=I, num_attention_heads=nh, num_key_value_heads=nkv,
                          num_hidden_layers=1, vocab_size=1024, max_position_embeddings=4096, rope_theta=500000.0,
                          rms_norm_eps=1e-5)


def _layer(cfg, seed=0):
    from cambrian_b200.model.language_model.cambrian_llama import CBLlamaDecoderLayer
    torch.manual_seed(seed)
    layer = CBLlamaDecoderLayer(cfg, 0)
    with torch.no_grad():
        for p in layer.parameters():
            p.copy_(torch.randn_like(p) * 0.02 if p.dim() == 2 else 1 + 0.1 * torch.randn_like(p))
    return layer.to(device=dev, dtype=bf)


def _run_layer(layer, cfg, fp8, recompute=False, B=2, S=300, seed=1):
    from cambrian_b200.model.language_model.cambrian_llama import rope_tables
    cos, sin = rope_tables(cfg, dev)
    g = _gen(seed)
    x = torch.randn(B, S, cfg.hidden_size, generator=g, device=dev).to(bf).requires_grad_()
    dout = (torch.randn(B, S, cfg.hidden_size, generator=g, device=dev) * 0.1).to(bf)
    rt = dict(pos=torch.arange(S, device=dev).repeat(B), cos=cos, sin=sin, kmask=None, hf_cast=False,
              recompute=recompute, fp8=fp8)
    layer.zero_grad()
    out = layer(x, rt)
    out.backward(dout)
    return x.detach(), dout, out.detach(), x.grad


def _fp8_gemm_tol(qa, qw, residual):
    """fp64 value y of the FP8 GEMM on its own quantised operands and the bound of tests/test_fp8_gpu.py::_check: one
    bf16 rounding of |y| plus 2^-10 of the absolute product sum (the f8 MMA's in-block accumulation, about 2^-11 of it on
    an H100, plus the fp32 promotion)."""
    xq, sa = qa
    scale = sa.double()[:, None] * qw.w.sw.double()[None, :]
    y = R.acc64(xq, qw.w.wq) * scale
    if residual is not None:
        y = y + residual.double()
    mag = (xq.double().abs() @ qw.w.wq.double().abs().t()) * scale
    return y, 2.0 ** -8 * y.abs() + 2.0 ** -10 * mag + 1e-30


def _assert_within(got, y, tol, what):
    err = (got.double() - y).abs()
    bad = err > tol
    assert torch.isfinite(got).all() and not bad.any(), (what, int(bad.sum()), (err / tol).max().item())


def test_decoder_layer_fp8_against_fp64_emulation(monkeypatch):
    """Every GEMM of one FP8 forward + backward, checked on the operands the layer actually quantised: the quantised
    weights are the row rule of W (forward) and of W^T (dgrad), the first dgrad's activation that of dout; each FP8 GEMM
    is within _fp8_gemm_tol of its fp64 value (so is the layer output, the down GEMM's); each bf16 wgrad GEMM within one
    bf16 rounding plus the worst-case fp32 summation error K 2^-24 of its absolute product sum (K = tokens); dx is the
    RMSNorm backward of the q|k|v dgrad, checked against the fp64 RMSNorm backward of that GEMM's fp64 value with the
    GEMM's bound carried through the (linear) backward plus one bf16 rounding."""
    from cambrian_b200 import ops
    cfg = _layer_cfg("3b")
    layer = _layer(cfg)
    fp8_calls, bf16_calls = [], []
    real_fp8, real_gemm = ops.gemm_fp8, ops.gemm

    # copies at the call: the layer goes on to modify some results in place (RoPE on the q|k|v output)
    def gemm_fp8(qa, qw, **kw):
        out = real_fp8(qa, qw, **kw)
        res = kw.get("residual")
        fp8_calls.append((qa, qw, None if res is None else res.clone(), out.clone()))
        return out

    def gemm(a, b, **kw):
        out = real_gemm(a, b, **kw)
        bf16_calls.append((a.clone(), b.clone(), kw, out.clone()))
        return out

    act_inputs = []
    real_act = ops.fp8_quantize_act

    def fp8_quantize_act(t):
        act_inputs.append(t.clone())
        return real_act(t)

    monkeypatch.setattr(ops, "gemm_fp8", gemm_fp8)
    monkeypatch.setattr(ops, "gemm", gemm)
    monkeypatch.setattr(ops, "fp8_quantize_act", fp8_quantize_act)
    x, dout, out, dx = _run_layer(layer, cfg, fp8=True)
    monkeypatch.undo()
    torch.cuda.synchronize()
    assert len(fp8_calls) == 8 and len(bf16_calls) == 4 and len(act_inputs) == 5
    assert all(kw.get("a_mn") and kw.get("b_mn") for _, _, kw, _ in bf16_calls)
    # the activations quantised by the row rule: attn, act (forward), dout, dx1, dqkv (dgrad of down, o, q|k|v)
    for t, (qa, _, _, _) in zip(act_inputs, [fp8_calls[1], fp8_calls[3], fp8_calls[4], fp8_calls[6], fp8_calls[7]]):
        q, s = R.quantize_act(t)
        assert torch.equal(_bits(qa[0]), _bits(q)) and torch.equal(qa[1], s)
    a, m = layer.self_attn, layer.mlp
    H, M = cfg.hidden_size, x.shape[0] * x.shape[1]
    qkv_w = torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight])
    gu_w = torch.cat([m.gate_proj.weight, m.up_proj.weight])
    weights = [qkv_w, a.o_proj.weight, gu_w, m.down_proj.weight]
    for (qa, qw, res, got), w, i in zip(fp8_calls[:4], weights, range(4)):          # forward: rows of W
        q, s = R.quantize_rows(w)
        assert torch.equal(_bits(qw.w.wq), _bits(q)) and torch.equal(qw.w.sw, s), ("fwd weight", i)
        _assert_within(got, *_fp8_gemm_tol(qa, qw, res), ("fwd", i))
    assert torch.equal(fp8_calls[3][3].view_as(out), out)                          # the output is the down GEMM's
    for (qa, qw, res, got), w, i in zip(fp8_calls[4:], weights[::-1], range(4)):    # dgrad: rows of W^T
        q, s = T.quantize_weight_t(w)
        assert torch.equal(_bits(qw.w.wq), _bits(q)) and torch.equal(qw.w.sw, s), ("dgrad weight", i)
        _assert_within(got, *_fp8_gemm_tol(qa, qw, res), ("dgrad", i))
    assert torch.equal(act_inputs[2], dout.reshape(M, H))
    for a_, b_, kw, got in bf16_calls:                                             # wgrad: dW = dy^T x, bf16
        y = a_.double().t() @ b_.double()
        mag = a_.double().abs().t() @ b_.double().abs()
        _assert_within(got, y, 2.0 ** -8 * y.abs() + a_.shape[0] * 2.0 ** -24 * mag + 1e-30, ("wgrad", tuple(y.shape)))
    # dx = rmsnorm_bwd(dh) + dx1: dh the q|k|v dgrad's output, dx1 the o dgrad's bf16 input
    qa, qw, _, dh = fp8_calls[7]
    dh64, dh_tol = _fp8_gemm_tol(qa, qw, None)
    x2 = x.reshape(M, H).double()
    rstd = torch.rsqrt(x2.pow(2).mean(-1, keepdim=True) + cfg.rms_norm_eps)
    xh, gm = x2 * rstd, layer.input_layernorm.weight.double()
    dres = act_inputs[3].double()
    want = _rms_bwd(dh64, xh, gm, rstd) + dres
    prop = rstd * gm.abs() * dh_tol + rstd * xh.abs() * (gm.abs() * dh_tol * xh.abs()).mean(-1, keepdim=True)
    fp32 = H * 2.0 ** -24 * rstd * (gm.abs() * dh64.abs() + xh.abs() * (gm.abs() * dh64.abs() * xh.abs()).mean(-1, True))
    _assert_within(dx.reshape(M, H), want, prop + fp32 + 2.0 ** -8 * want.abs() + 2.0 ** -8 * dres.abs() + 1e-30, "dx")


def _rms_bwd(dy, xh, gm, rstd):
    g = dy * gm
    return rstd * (g - xh * (g * xh).mean(-1, keepdim=True))


def test_decoder_layer_fp8_against_bf16():
    """The FP8 layer against the bf16 layer on the same inputs.  E4M3 keeps 4 significant bits (unit roundoff
    u = 2^-4); each FP8 product carries two quantised factors, (1 + u)^2 - 1 = 2u + u^2 relative, and the output and dx
    are sums of such products plus bf16 terms.  The bound on the relative Frobenius error is that 2u + u^2."""
    u = 2.0 ** -4
    bound = 2 * u + u * u
    cfg = _layer_cfg("3b")
    layer = _layer(cfg)
    _, _, out8, dx8 = _run_layer(layer, cfg, fp8=True)
    g8 = {n: p.grad.clone() for n, p in layer.named_parameters()}
    _, _, out16, dx16 = _run_layer(layer, cfg, fp8=False)
    rel = lambda a, b: ((a.double() - b.double()).norm() / b.double().norm()).item()
    e_out, e_dx = rel(out8, out16), rel(dx8, dx16)
    e_w = {n: rel(g8[n], p.grad) for n, p in layer.named_parameters()}
    print(f"\nfp8 vs bf16 relative Frobenius error: out {e_out:.3e}, dx {e_dx:.3e} (bound {bound:.3e}); "
          f"weight gradients {max(e_w.values()):.3e} at most")
    assert 0 < e_out < bound and 0 < e_dx < bound


def test_decoder_layer_fp8_recompute_matches_no_recompute():
    cfg = _layer_cfg("3b")
    layer = _layer(cfg)
    res = []
    for recompute in (False, True):
        _, _, out, dx = _run_layer(layer, cfg, fp8=True, recompute=recompute)
        res.append((out, dx, {n: p.grad.clone() for n, p in layer.named_parameters()}))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
    for n in res[0][2]:
        assert torch.equal(res[0][2][n], res[1][2][n]), n


# ------------------------------------------------------------------------------------------------ training
def _setup(fp8, seed=0):
    import test_modules_gpu as TM
    cfg = tiny_cambrian_config()
    cfg.fused_lm_loss = True
    cfg.fp8_training = fp8
    torch.manual_seed(seed)
    model = TM._build_tiny_model(cfg)
    model.train()
    ids, labels, attn, pos, images, masks = TM._tiny_batch(cfg)
    batch = dict(input_ids=ids.to(dev), labels=labels.to(dev), attention_mask=attn.to(dev), position_ids=pos.to(dev),
                 images=[i.to(dev).bfloat16() for i in images], image_aux_attention_masks_list=[m.to(dev) for m in masks])
    return cfg, model, batch


def test_engine_fp8_steps_are_bitwise_reproducible():
    """Two FP8 runs of three TrainEngine steps (data-parallel engine on one rank, clipping on): losses, main_grad and
    weights bitwise equal."""
    from cambrian_b200.engine import TrainEngine
    runs = []
    for _ in range(2):
        cfg, model, batch = _setup(True)
        eng = TrainEngine(model, lr=1e-3, bucket_mb=8.0, max_grad_norm=0.05)
        losses = []
        for _ in range(3):
            eng.zero_grad()
            loss = model(**batch).loss
            loss.backward()
            eng.step()
            losses.append(loss.detach().clone())
        torch.cuda.synchronize()
        grads = {n: p.main_grad.clone() for n, p in model.named_parameters() if getattr(p, "main_grad", None) is not None}
        runs.append((torch.stack(losses), grads, {n: p.detach().clone() for n, p in model.named_parameters()}))
    (l0, g0, w0), (l1, g1, w1) = runs
    assert torch.equal(l0, l1) and torch.isfinite(l0).all()
    assert g0.keys() == g1.keys() and len(g0) > 0
    for n in g0:
        assert torch.equal(g0[n], g1[n]), n
    for n in w0:
        assert torch.equal(w0[n], w1[n]), n


def test_memorisation_fp8_tracks_bf16():
    """100 steps on one fixed seeded batch: both runs drive the loss well below its start, and the FP8 final loss is
    within 5 % of the bf16 one."""
    from cambrian_b200.engine import TrainEngine
    finals = {}
    for fp8 in (False, True):
        cfg, model, batch = _setup(fp8)
        eng = TrainEngine(model, lr=1e-3, bucket_mb=8.0, max_grad_norm=1.0)
        losses = []
        for _ in range(100):
            eng.zero_grad()
            loss = model(**batch).loss
            loss.backward()
            eng.step()
            losses.append(float(loss.detach()))
        finals[fp8] = (losses[0], losses[-1])
    print(f"\nmemorisation, 100 steps: bf16 {finals[False][0]:.4f} -> {finals[False][1]:.4f}, "
          f"fp8 {finals[True][0]:.4f} -> {finals[True][1]:.4f}")
    for fp8, (first, last) in finals.items():
        assert last < 0.5 * first, (fp8, first, last)
    assert abs(finals[True][1] - finals[False][1]) <= 0.05 * finals[False][1]
