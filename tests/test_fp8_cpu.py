"""CPU checks of the FP8 E4M3 inference path: the format on hand-built cases (torch reference of tests/fp8_reference.py,
itself checked against torch's float8_e4m3fn conversion where the two must agree), the host routing of ops.fp8_linear,
load_pretrained_model(load_fp8=True), greedy generate against the fp32 oracle whose decoder projections run the
reference FP8 linear, and the operations an FP8 model refuses.  The four FP8 kernels are replaced by the reference's CPU
stand-ins; their numerics are covered under `-m gpu` (tests/test_fp8_gpu.py)."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import fp8_reference as R  # noqa: E402
import ops_emulation  # noqa: E402
from helpers import tiny_cambrian_config  # noqa: E402

needs_no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="kernel stand-ins are for GPU-less machines only")
bf = torch.bfloat16
f8 = torch.float8_e4m3fn


def _bits(t):
    return t.view(torch.uint8).tolist()


# ------------------------------------------------------------------------------------------------ the format
def test_e4m3_rounding_ties_subnormals_saturation_and_signed_zero():
    v = torch.tensor([
        1.0, 1.0625, 1.1875,           # ties between 1, 1.125, 1.25: to even mantissa (1.0, 1.25)
        17.0, 19.0,                    # quantum 2 in [16, 32): ties -> 16, 20
        2.0 ** -9, 2.0 ** -10,         # smallest subnormal; half of it ties to +0
        3 * 2.0 ** -10, 2.0 ** -11,    # 1.5 quanta -> 2 quanta; a quarter quantum -> 0
        2.0 ** -6 - 2.0 ** -10,        # between the largest subnormal (7 * 2^-9) and 2^-6: tie -> 2^-6 (even)
        448.0, 460.0, 464.0, 1e6,      # max finite; below the 448/480 midpoint; at it; far above: all 448
        -0.0, -1e-6, -465.0,           # signed zero, negative underflow to -0, negative saturation
    ])
    want = [1.0, 1.0, 1.25, 16.0, 20.0, 2.0 ** -9, 0.0, 2.0 ** -8, 0.0, 2.0 ** -6, 448, 448, 448, 448, -0.0, -0.0, -448]
    got = R.e4m3_rn_satfinite(v)
    assert got.tolist() == want
    assert torch.equal(torch.signbit(got), torch.signbit(torch.tensor(want)))
    assert _bits(R.to_e4m3(v))[-3:] == [0x80, 0x80, 0xFE]


def test_reference_rounding_agrees_with_torch_float8_inside_the_range():
    """torch's float8_e4m3fn conversion is round-to-nearest-even but turns |v| > 464 into NaN instead of saturating:
    the two must agree bit for bit everywhere else, including subnormals and signed zeros."""
    g = torch.Generator().manual_seed(0)
    v = torch.cat([torch.randn(20000, generator=g) * s for s in (1e-3, 0.05, 1.0, 30.0, 150.0)])
    grid = torch.arange(-464.0, 464.0, 2.0 ** -4)                   # every E4M3 midpoint above 2^-2 on the grid
    tiny = torch.arange(-2 ** -5, 2 ** -5, 2.0 ** -12)               # subnormals, their midpoints, -0
    v = torch.cat([v.clamp(-464, 464), grid, tiny, torch.tensor([-0.0, 0.0])])
    assert _bits(R.to_e4m3(v)) == _bits(v.to(f8))


def _row_case():
    w = torch.zeros(6, 32, dtype=bf)
    w[0, :4] = torch.tensor([2.0, -1.0, 0.5, 0.25])    # amax 2: r = 224, 2 -> 448 exactly
    w[1] = 0                                            # zero row
    w[2, 0] = -0.0                                      # a row of +-0
    w[2, 1] = -0.0
    w[3, :3] = torch.tensor([3.0, 3.0 * 2 ** -8, 3.0 * 2 ** -11])   # 448, 448 * 2^-8 = 1.75 (exact), subnormal range
    w[4, :2] = torch.tensor([2.0 ** -133, -(2.0 ** -130)], dtype=bf)   # bf16 subnormals: 448 / amax overflows fp32
    w[5, :2] = torch.tensor([1.0, -1e-6])
    return w


def test_row_quantiser_hand_built_cases():
    w = _row_case()
    q, s = R.quantize_weight(w)
    qf = q.float()
    assert s[0].item() == (torch.tensor(2.0) / 448).item() and qf[0, :4].tolist() == [448.0, -224.0, 112.0, 56.0]
    assert s[1].item() == 0.0 and _bits(q[1]) == [0] * 32
    assert s[2].item() == 0.0 and _bits(q[2])[:3] == [0x80, 0x80, 0]         # -0 survives quantisation
    assert qf[3, :2].tolist() == [448.0, 1.75]
    assert qf[3, 2].item() == R.e4m3_rn_satfinite(torch.tensor(3.0 * 2 ** -11) * (448.0 / 3.0)).item()
    # the subnormal row: r = FLT_MAX, nothing reaches 448, nothing is NaN, the scale is amax / 448 in fp32
    amax = torch.tensor(2.0 ** -130)
    assert s[4].item() == (amax / 448).item() and s[4].item() > 0
    want = R.e4m3_rn_satfinite(torch.tensor([2.0 ** -133, -(2.0 ** -130)]) * R.FLT_MAX)
    assert qf[4, :2].tolist() == want.tolist() and 0 < want.abs().max().item() < 448
    assert not torch.isnan(qf).any()
    # -1e-6 * 448 is below half the smallest subnormal: a signed zero
    assert _bits(q[5, 1:2]) == [0x80]
    # activations follow the same rule
    qa, sa = R.quantize_act(w)
    assert _bits(qa) == _bits(q) and torch.equal(sa, s)


def test_reference_linear_tracks_the_bf16_product():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(16, 512, generator=g).to(bf)
    x[:, 7] *= 30                               # a large feature: per-row scaling copes without outlier columns
    w = (torch.randn(256, 512, generator=g) * 0.02).to(bf)
    wq, sw = R.quantize_weight(w)
    y = R.linear(x, wq, sw, out_dtype=torch.float32)
    ref = x.float() @ w.float().t()
    assert ((y - ref).norm() / ref.norm()).item() < 0.06
    # the epilogue order: acc * (sa * sw), then bias, then residual
    xq, sa = R.quantize_act(x)
    b = torch.randn(256, generator=g).to(bf)
    res = torch.randn(16, 256, generator=g).to(bf)
    acc = (xq.double() @ wq.double().t()).float()
    want = ((acc * (sa[:, None] * sw[None, :])) + b.float()[None]) + res.float()
    assert torch.equal(R.linear(x, wq, sw, bias=b, residual=res, out_dtype=torch.float32), want)


def test_byte_accounting():
    from cambrian_b200 import quant_fp8
    cfg = tiny_cambrian_config()
    qw = quant_fp8.Fp8Weight(512, 256, "cpu")
    assert qw.wq.dtype == f8 and qw.nbytes == quant_fp8.bytes_per_weight(512, 256) == 512 * 256 + 4 * 512
    H, I = cfg.hidden_size, cfg.intermediate_size
    assert quant_fp8.bytes_per_layer(cfg) == sum(quant_fp8.bytes_per_weight(n, k) for n, k in
                                                 [(H, H), (H // 2, H), (H // 2, H), (H, H), (I, H), (I, H), (H, I)])
    with pytest.raises(ValueError):
        quant_fp8.Fp8Weight(4, 40, "cpu")


# ------------------------------------------------------------------------------------------------ host routing
def test_fp8_linear_routes_decode_to_gemv_and_prefill_to_gemm(monkeypatch):
    from cambrian_b200 import _lib, ops, quant_fp8
    calls = []

    class FakeLib:
        def __getattr__(self, name):
            return lambda *a: calls.append(name) or 0

    monkeypatch.setattr(ops, "_require_cuda_bf16", lambda *a: None)
    monkeypatch.setattr(_lib, "load", lambda: FakeLib())
    monkeypatch.setattr(ops, "stream", lambda: 0)
    qkv = quant_fp8.Fp8Projection(quant_fp8.Fp8Weight(512, 256, "cpu"))
    gu = quant_fp8.Fp8Projection(quant_fp8.Fp8Weight(1024, 256, "cpu"))
    for M, mm in ((1, "cb_gemv_fp8"), (8, "cb_gemv_fp8"), (9, "cb_gemm_fp8"), (2048, "cb_gemm_fp8")):
        calls.clear()
        y = qkv.linear(torch.zeros(M, 256, dtype=bf))
        assert calls == ["cb_fp8_quantize_act", mm] and y.shape == (M, 512), (M, calls)
    for M, mm in ((4, "cb_gemv_fp8"), (300, "cb_gemm_fp8")):
        calls.clear()
        g, a = gu.gate_up(torch.zeros(M, 256, dtype=bf))
        assert calls == ["cb_fp8_quantize_act", mm, "cb_swiglu_fwd"] and g.shape == (M, 1024) and a.shape == (M, 512)


# ------------------------------------------------------------------------------------------------ model plumbing
def _build(cfg, seed=3):
    from test_nf4_cpu import _build as build_nf4_test_model
    return build_nf4_test_model(cfg, seed)


@needs_no_gpu
def test_load_fp8_quantises_exactly_the_seven_projections(monkeypatch, tmp_path):
    from cambrian_b200 import checkpoint, quant, quant_fp8
    from cambrian_b200.model.language_model.cambrian_llama import CambrianLlamaForCausalLM
    ops_emulation.install(monkeypatch)
    R.install(monkeypatch)
    cfg = tiny_cambrian_config()
    torch.manual_seed(0)
    src = CambrianLlamaForCausalLM(cfg).to(bf)
    src.save_pretrained(tmp_path / "ckpt")
    ref = src.state_dict()
    _, model, _, _ = checkpoint.load_pretrained_model(str(tmp_path / "ckpt"), load_fp8=True, device="cpu",
                                                      load_tokenizer=False)
    assert quant.is_quantized(model) and quant.quantized_format(model) == "8-bit (FP8)"
    sd = model.state_dict()
    groups = dict(qkv=["q_proj", "k_proj", "v_proj"], o=["o_proj"], gate_up=["gate_proj", "up_proj"], down=["down_proj"])
    nbytes = 0
    for i, layer in enumerate(model.get_model().layers):
        assert layer._nf4 is None and layer._int8 is None and set(layer._fp8) == set(groups)
        assert layer._quantized() is layer._fp8
        for key, names in groups.items():
            ws = [ref[f"model.layers.{i}.{'self_attn' if n[0] in 'qkvo' else 'mlp'}.{n}.weight"] for n in names]
            want_q, want_s = R.quantize_weight(torch.cat(ws, 0))
            got = layer._fp8[key].w
            assert _bits(got.wq) == _bits(want_q) and torch.equal(got.sw, want_s), (i, key)
            nbytes += got.nbytes
    assert nbytes == cfg.num_hidden_layers * quant_fp8.bytes_per_layer(cfg)
    for k, v in sd.items():
        if v.numel():
            assert v.dtype == bf and torch.equal(v, ref[k]), k
    assert sum(1 for v in sd.values() if v.numel() == 0) == 7 * cfg.num_hidden_layers


class _Fp8Functional:
    """Stands in for `torch.nn.functional` inside the oracle module: F.linear on a registered placeholder weight runs
    the reference FP8 linear on that projection's (wq, sw); everything else is torch's."""

    def __init__(self, table):
        self.table = table
        self.hits = 0

    def __getattr__(self, name):
        return getattr(torch.nn.functional, name)

    def linear(self, x, w, b=None):
        q = self.table.get(w.data_ptr())
        if q is None:
            return torch.nn.functional.linear(x, w, b)
        self.hits += 1
        wq, sw = q
        x2 = x.reshape(-1, x.shape[-1])
        xq, sa = R.quantize_act(x2)
        y = R.epilogue(R.acc64(xq, wq.to(x.device)).float(), sa, sw.to(x.device), out_dtype=x.dtype)
        return y.view(*x.shape[:-1], wq.shape[0])


def oracle_fp8_functional(model, cfg, sd):
    """Put one fp32 placeholder per decoder projection of the FP8 `model` into the oracle state dict `sd` (CPU) and
    return the F stand-in that maps each placeholder to the rows of that projection in its stacked (wq, sw)."""
    hd = cfg.hidden_size // cfg.num_attention_heads
    rows_of = {"self_attn.q_proj": cfg.num_attention_heads * hd, "self_attn.k_proj": cfg.num_key_value_heads * hd,
               "self_attn.v_proj": cfg.num_key_value_heads * hd, "self_attn.o_proj": cfg.hidden_size,
               "mlp.gate_proj": cfg.intermediate_size, "mlp.up_proj": cfg.intermediate_size,
               "mlp.down_proj": cfg.hidden_size}
    table = {}
    for i, layer in enumerate(model.get_model().layers):
        for key, names in (("qkv", ["self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj"]),
                           ("o", ["self_attn.o_proj"]), ("gate_up", ["mlp.gate_proj", "mlp.up_proj"]),
                           ("down", ["mlp.down_proj"])):
            w = layer._fp8[key].w
            r = 0
            for n_ in names:
                rows = rows_of[n_]
                placeholder = torch.zeros(rows, w.shape[1])
                sd[f"model.layers.{i}.{n_}.weight"] = placeholder
                table[placeholder.data_ptr()] = (w.wq[r:r + rows].cpu(), w.sw[r:r + rows].cpu())
                r += rows
            assert r == w.shape[0]
    return _Fp8Functional(table)


@needs_no_gpu
def test_greedy_generate_fp8_matches_fp32_oracle_with_fp8_projections(monkeypatch):
    from test_parity_gpu import _oracle_greedy

    from cambrian_b200 import quant_fp8
    from helpers import oracle_cfg
    from oracle import cambrian_oracle as O
    ops_emulation.install(monkeypatch)
    R.install(monkeypatch)
    cfg = tiny_cambrian_config()
    cfg.fused_lm_loss = True
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
    model.eval()
    stats = quant_fp8.quantize_decoder_fp8_(model, "cpu")
    assert stats["fp8_bytes"] == cfg.num_hidden_layers * quant_fp8.bytes_per_layer(cfg)
    sd = {k: v.detach().float() for k, v in model.state_dict().items()}
    shim = oracle_fp8_functional(model, cfg, sd)
    monkeypatch.setattr(O, "F", shim)
    from test_model_host_logic_cpu import _batch, _tower_feats
    ids, labels, attn, pos, masks = _batch(cfg, S=96)
    S0, n_new = 40, 12
    gen_ids = ids[:1, :S0].clone()
    feats = [f[:1] for f in _tower_feats(model, cfg, 2, 31)]
    monkeypatch.setattr(type(model), "encode_images", lambda self, imgs: feats)
    images = [torch.zeros(1, 3, 8, 8, dtype=bf) for _ in feats]
    new = model.generate(gen_ids, images=images, image_sizes=[(56, 56)], max_new_tokens=n_new, do_sample=False)
    want, margins = _oracle_greedy(sd, cfg, oracle_cfg(cfg), [f.float() for f in feats], gen_ids, n_new, torch.float32,
                                   torch.device("cpu"))
    assert shim.hits >= 7 * cfg.num_hidden_layers * n_new      # every decoder projection of every pass was FP8
    assert new[0].tolist() == want, (new[0].tolist(), want, margins)
    assert len(set(want)) >= 4
    with torch.no_grad():
        out = model(input_ids=gen_ids, images=images, image_sizes=[(56, 56)])
    assert torch.isfinite(out.logits).all()
    with pytest.raises(NotImplementedError, match="FP8"):
        model(input_ids=gen_ids, images=images, image_sizes=[(56, 56)])


@needs_no_gpu
def test_fp8_model_refuses_training_sharding_and_saving(monkeypatch, tmp_path):
    from cambrian_b200 import quant_fp8
    from cambrian_b200.engine import TrainEngine
    from cambrian_b200.sharded import Zero3Inference
    ops_emulation.install(monkeypatch)
    R.install(monkeypatch)
    cfg = tiny_cambrian_config()
    model = _build(cfg)
    quant_fp8.quantize_decoder_fp8_(model, "cpu")
    with pytest.raises(ValueError, match="FP8"):
        TrainEngine(model)
    with pytest.raises(ValueError, match="FP8"):
        Zero3Inference(model)
    with pytest.raises(NotImplementedError, match="FP8"):
        model.save_pretrained(tmp_path / "q")
    assert not (tmp_path / "q").exists()


@pytest.mark.parametrize("other", ["load_4bit", "load_8bit"])
def test_load_fp8_rejects_a_second_format_before_reading(tmp_path, other):
    from cambrian_b200 import checkpoint
    with pytest.raises(ValueError, match="load_fp8"):
        checkpoint.load_pretrained_model(str(tmp_path / "missing"), load_fp8=True, device="cpu", load_tokenizer=False,
                                         **{other: True})


@needs_no_gpu
def test_load_fp8_on_cuda_without_cuda_raises_before_reading(tmp_path):
    from cambrian_b200 import checkpoint
    with pytest.raises(NotImplementedError, match="FP8"):
        checkpoint.load_pretrained_model(str(tmp_path / "missing"), load_fp8=True, device="cuda", load_tokenizer=False)
