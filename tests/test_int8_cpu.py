"""CPU checks of the 8-bit (LLM.int8) inference path: the format and the output arithmetic on hand-built cases (torch
reference of tests/int8_reference.py), the host routing of ops.int8_linear, load_pretrained_model(load_8bit=True),
greedy generate against the fp32 oracle whose decoder projections run the reference int8 linear, and the operations an
8-bit model refuses.  The four int8 kernels are replaced by the reference's CPU stand-ins; their numerics are covered
under `-m gpu` (tests/test_int8_gpu.py)."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import int8_reference as R  # noqa: E402
import ops_emulation  # noqa: E402
from helpers import oracle_cfg, tiny_cambrian_config  # noqa: E402

needs_no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="kernel stand-ins are for GPU-less machines only")
bf = torch.bfloat16


# ------------------------------------------------------------------------------------------------ the format
def test_constants_are_the_fp32_quotients():
    assert R.INV127.item() == float(np.float32(1) / np.float32(127))
    assert R.INV16129.item() == float(np.float32(1) / np.float32(16129))


def test_weight_ties_round_half_to_even_and_clamp():
    w = torch.tensor([[127.0, 0.5, 1.5, 2.5, -0.5, -2.5, 3.5, -127.0] + [0.0] * 8], dtype=bf)
    cb, scb = R.quantize_weight(w)
    assert scb.tolist() == [127.0]
    assert cb[0, :8].tolist() == [127, 0, 2, 2, 0, -2, 4, -127]
    # a row whose scale divides unevenly still stays inside +-127
    g = torch.Generator().manual_seed(0)
    w = (torch.randn(64, 256, generator=g) * 0.05).to(bf)
    cb, scb = R.quantize_weight(w)
    assert int(cb.abs().max()) == 127 and int(cb.min()) >= -127
    assert torch.equal(scb, w.float().abs().amax(1))


def test_activation_ties_and_disabled_threshold():
    x = torch.tensor([[127.0, 0.5, 1.5, 2.5, -0.5, -2.5, 3.5, 100.0] + [0.0] * 8], dtype=bf)
    for thr in (0.0, -1.0):                     # tau <= 0: no outliers even at |x| = 127
        xq, sca, idx = R.quantize_act(x, thr)
        assert idx.numel() == 0 and sca.tolist() == [127.0]
        assert xq[0, :8].tolist() == [127, 0, 2, 2, 0, -2, 4, 100]


def test_outlier_at_exactly_tau_and_in_one_row_only():
    x = torch.zeros(3, 32, dtype=bf)
    x[:, :] = 0.25
    x[1, 5] = 6.0                               # exactly tau: an outlier
    x[2, 9] = -7.0                              # one row only: the whole column is an outlier
    x[0, 11] = 5.96875                          # the bf16 just below 6.0: not an outlier
    xq, sca, idx = R.quantize_act(x, 6.0)
    assert idx.tolist() == [5, 9]
    assert xq[:, 5].tolist() == [0, 0, 0] and xq[:, 9].tolist() == [0, 0, 0]
    assert sca.tolist() == [float(x[0, 11]), 0.25, 0.25]
    assert xq[0, 11].item() == 127
    # the outlier columns contribute through the fp32 term, in ascending order
    g = torch.Generator().manual_seed(1)
    w = (torch.randn(8, 32, generator=g) * 0.1).to(bf)
    cb, scb = R.quantize_weight(w)
    y = R.linear(x, cb, scb, out_dtype=torch.float32)
    acc = xq.long() @ cb.long().t()
    v = (acc.float() * (sca[:, None] * scb[None, :])) * R.INV16129
    wsc = scb * R.INV127
    o = x[:, 5:6].float() * (cb[:, 5].float() * wsc)[None]
    o = o + x[:, 9:10].float() * (cb[:, 9].float() * wsc)[None]
    assert torch.equal(y, v + o)
    wt = cb.float() * (scb / 127)[:, None]
    assert torch.allclose(y, x.float() @ wt.t(), rtol=1e-2, atol=2e-2)


def test_all_columns_outliers_and_zero_rows():
    g = torch.Generator().manual_seed(2)
    x = (torch.randn(4, 48, generator=g)).to(bf)
    x[0] = 8.0                                  # every column reaches tau in row 0
    w = (torch.randn(6, 48, generator=g) * 0.1).to(bf)
    w[3] = 0
    cb, scb = R.quantize_weight(w)
    assert scb[3].item() == 0.0 and cb[3].abs().sum().item() == 0
    xq, sca, idx = R.quantize_act(x, 6.0)
    assert idx.tolist() == list(range(48)) and xq.abs().sum().item() == 0 and sca.abs().sum().item() == 0
    y = R.linear(x, cb, scb, out_dtype=torch.float32)
    assert torch.equal(y[:, 3], torch.zeros(4))
    wt = cb.float() * (scb / 127)[:, None]
    assert torch.allclose(y, x.float() @ wt.t(), rtol=1e-4, atol=1e-4)   # all fp32: only the summation order differs
    xz = x.clone()
    xz[2] = 0                                   # a zero activation row quantises to 0 with scale 0
    xq, sca, _ = R.quantize_act(xz, 0.0)
    assert sca[2].item() == 0.0 and xq[2].abs().sum().item() == 0
    assert torch.equal(R.linear(xz, cb, scb, 0.0, out_dtype=torch.float32)[2], torch.zeros(6))


def test_reference_linear_tracks_the_bf16_product():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(16, 512, generator=g).to(bf)
    x[:, 7] *= 10                               # one outlier feature, as in LLM activations
    w = (torch.randn(256, 512, generator=g) * 0.02).to(bf)
    cb, scb = R.quantize_weight(w)
    y = R.linear(x, cb, scb, out_dtype=torch.float32)
    ref = x.float() @ w.float().t()
    assert ((y - ref).norm() / ref.norm()).item() < 0.02


def test_byte_accounting():
    from cambrian_b200 import quant_int8
    cfg = tiny_cambrian_config()
    qw = quant_int8.Int8Weight(512, 256, "cpu")
    assert qw.nbytes == quant_int8.bytes_per_weight(512, 256) == 512 * 256 + 4 * 512
    H, I = cfg.hidden_size, cfg.intermediate_size
    assert quant_int8.bytes_per_layer(cfg) == sum(quant_int8.bytes_per_weight(n, k) for n, k in
                                                  [(H, H), (H // 2, H), (H // 2, H), (H, H), (I, H), (I, H), (H, I)])
    with pytest.raises(ValueError):
        quant_int8.Int8Weight(4, 40, "cpu")


# ------------------------------------------------------------------------------------------------ host routing
def test_int8_linear_routes_decode_to_gemv_and_prefill_to_gemm(monkeypatch):
    from cambrian_b200 import _lib, ops, quant_int8
    calls = []

    class FakeLib:
        def __getattr__(self, name):
            return lambda *a: calls.append(name) or 0

    monkeypatch.setattr(ops, "_require_cuda_bf16", lambda *a: None)
    monkeypatch.setattr(_lib, "load", lambda: FakeLib())
    monkeypatch.setattr(ops, "stream", lambda: 0)
    qkv = quant_int8.Int8Projection(quant_int8.Int8Weight(512, 256, "cpu"))
    gu = quant_int8.Int8Projection(quant_int8.Int8Weight(1024, 256, "cpu"))
    for M, mm in ((1, "cb_gemv_int8"), (8, "cb_gemv_int8"), (9, "cb_gemm_int8"), (2048, "cb_gemm_int8")):
        calls.clear()
        y = qkv.linear(torch.zeros(M, 256, dtype=bf))
        assert calls == ["cb_int8_quantize_act", mm] and y.shape == (M, 512), (M, calls)
    for M, mm in ((4, "cb_gemv_int8"), (300, "cb_gemm_int8")):
        calls.clear()
        g, a = gu.gate_up(torch.zeros(M, 256, dtype=bf))
        assert calls == ["cb_int8_quantize_act", mm, "cb_swiglu_fwd"] and g.shape == (M, 1024) and a.shape == (M, 512)


# ------------------------------------------------------------------------------------------------ model plumbing
def _build(cfg, seed=3):
    from test_nf4_cpu import _build as build_nf4_test_model
    return build_nf4_test_model(cfg, seed)


@needs_no_gpu
@pytest.mark.parametrize("also_4bit", [False, True])
def test_load_8bit_quantises_exactly_the_seven_projections(monkeypatch, tmp_path, also_4bit):
    """load_8bit=True quantises the seven projections to int8; with load_4bit=True as well, 8-bit wins (builder.py)."""
    from cambrian_b200 import checkpoint, quant, quant_int8
    from cambrian_b200.model.language_model.cambrian_llama import CambrianLlamaForCausalLM
    ops_emulation.install(monkeypatch)
    R.install(monkeypatch)
    cfg = tiny_cambrian_config()
    torch.manual_seed(0)
    src = CambrianLlamaForCausalLM(cfg).to(bf)
    src.save_pretrained(tmp_path / "ckpt")
    ref = src.state_dict()
    _, model, _, _ = checkpoint.load_pretrained_model(str(tmp_path / "ckpt"), load_8bit=True, load_4bit=also_4bit,
                                                      device="cpu", load_tokenizer=False)
    assert quant.is_quantized(model) and quant.quantized_format(model) == "8-bit (LLM.int8)"
    sd = model.state_dict()
    groups = dict(qkv=["q_proj", "k_proj", "v_proj"], o=["o_proj"], gate_up=["gate_proj", "up_proj"], down=["down_proj"])
    nbytes = 0
    for i, layer in enumerate(model.get_model().layers):
        assert layer._nf4 is None and set(layer._int8) == set(groups)
        for key, names in groups.items():
            ws = [ref[f"model.layers.{i}.{'self_attn' if n[0] in 'qkvo' else 'mlp'}.{n}.weight"] for n in names]
            want_cb, want_scb = R.quantize_weight(torch.cat(ws, 0))
            got = layer._int8[key].w
            assert torch.equal(got.cb, want_cb) and torch.equal(got.scb, want_scb), (i, key)
            nbytes += got.nbytes
    assert nbytes == cfg.num_hidden_layers * quant_int8.bytes_per_layer(cfg)
    for k, v in sd.items():
        if v.numel():
            assert v.dtype == bf and torch.equal(v, ref[k]), k
    assert sum(1 for v in sd.values() if v.numel() == 0) == 7 * cfg.num_hidden_layers
    assert all(not p.requires_grad for n, p in model.named_parameters() if p.numel() == 0)


class _Int8Functional:
    """Stands in for `torch.nn.functional` inside the oracle module: F.linear on a registered placeholder weight runs
    the reference int8 linear on that projection's (cb, scb); everything else is torch's."""

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
        cb, scb = q
        y = R.linear(x.reshape(-1, x.shape[-1]), cb.to(x.device), scb.to(x.device), out_dtype=x.dtype)
        return y.view(*x.shape[:-1], cb.shape[0])


def oracle_int8_functional(model, cfg, sd):
    """Put one fp32 placeholder per decoder projection of the int8 `model` into the oracle state dict `sd` (CPU) and
    return the F stand-in that maps each placeholder to the rows of that projection in its stacked (cb, scb)."""
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
            w = layer._int8[key].w
            r = 0
            for n_ in names:
                rows = rows_of[n_]
                placeholder = torch.zeros(rows, w.shape[1])
                sd[f"model.layers.{i}.{n_}.weight"] = placeholder
                table[placeholder.data_ptr()] = (w.cb[r:r + rows].cpu(), w.scb[r:r + rows].cpu())
                r += rows
            assert r == w.shape[0]
    return _Int8Functional(table)


@needs_no_gpu
def test_greedy_generate_8bit_matches_fp32_oracle_with_int8_projections(monkeypatch):
    from test_parity_gpu import _oracle_greedy

    from cambrian_b200 import quant_int8
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
    stats = quant_int8.quantize_decoder_int8_(model, "cpu")
    assert stats["int8_bytes"] == cfg.num_hidden_layers * quant_int8.bytes_per_layer(cfg)
    sd = {k: v.detach().float() for k, v in model.state_dict().items()}
    shim = oracle_int8_functional(model, cfg, sd)
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
    assert shim.hits >= 7 * cfg.num_hidden_layers * n_new      # every decoder projection of every pass was int8
    assert new[0].tolist() == want, (new[0].tolist(), want, margins)
    assert len(set(want)) >= 4
    with torch.no_grad():
        out = model(input_ids=gen_ids, images=images, image_sizes=[(56, 56)])
    assert torch.isfinite(out.logits).all()
    with pytest.raises(NotImplementedError, match="8-bit"):
        model(input_ids=gen_ids, images=images, image_sizes=[(56, 56)])


@needs_no_gpu
def test_8bit_model_refuses_training_sharding_and_saving(monkeypatch, tmp_path):
    from cambrian_b200 import checkpoint, quant_int8
    from cambrian_b200.engine import TrainEngine
    from cambrian_b200.sharded import Zero3Inference
    ops_emulation.install(monkeypatch)
    R.install(monkeypatch)
    cfg = tiny_cambrian_config()
    model = _build(cfg)
    quant_int8.quantize_decoder_int8_(model, "cpu")
    with pytest.raises(ValueError, match="8-bit"):
        TrainEngine(model)
    with pytest.raises(ValueError, match="8-bit"):
        Zero3Inference(model)
    with pytest.raises(NotImplementedError, match="8-bit"):
        model.save_pretrained(tmp_path / "q")
    assert not (tmp_path / "q").exists()
    with pytest.raises(NotImplementedError, match="LoRA"):
        checkpoint.load_pretrained_model("x", model_name="cambrian-lora", load_8bit=True, device="cpu",
                                         load_tokenizer=False)
    with pytest.raises(NotImplementedError, match="LLaMA"):
        checkpoint.load_pretrained_model("x", model_name="cambrian-mistral", load_8bit=True, device="cpu",
                                         load_tokenizer=False)
