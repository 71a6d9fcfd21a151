"""CPU checks of the 4-bit (NF4) inference path: the format on hand-built blocks (torch reference of tests/nf4_reference.py),
the host routing of ops.nf4_linear, load_pretrained_model(load_4bit=True), greedy generate against the fp32 oracle run
with the W~ weights, and the operations a 4-bit model refuses.  The three NF4 kernels are replaced by the reference's
CPU stand-ins; their numerics are covered under `-m gpu` (tests/test_nf4_gpu.py)."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import nf4_reference as R  # noqa: E402
import ops_emulation  # noqa: E402
from helpers import oracle_cfg, tiny_cambrian_config  # noqa: E402

needs_no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="kernel stand-ins are for GPU-less machines only")


# ------------------------------------------------------------------------------------------------ the format
def test_dynamic_map_and_tables():
    from cambrian_b200 import quant
    m = R.DMAP
    assert m.numel() == 256 and m.unique().numel() == 256 and bool((m[1:] > m[:-1]).all())
    assert 0.0 in m.tolist() and 1.0 in m.tolist() and -1.0 not in m.tolist()
    assert abs(float(m[0]) + 0.99297) < 1e-5
    assert torch.equal(quant.dynamic_map(), m)
    assert torch.equal(torch.tensor(quant.NF4_CODE, dtype=torch.float32), R.NF4)


def test_codes_at_nf4_points_and_around_midpoints():
    c = R.NF4
    row = torch.zeros(64)
    row[:16] = c                                                   # absmax 1.0: every table point maps to itself
    mids = (c[:-1] + c[1:]) / 2
    for i in range(15):
        row[16 + 2 * i] = torch.nextafter(mids[i], torch.tensor(-2.0))   # just below midpoint i -> code i
        row[17 + 2 * i] = torch.nextafter(mids[i], torch.tensor(2.0))    # just above -> code i + 1
    row[46] = mids[3]                                               # exactly on a midpoint: not strictly less -> code 3
    w = row.to(torch.bfloat16)[None]
    x = w.float()[0]
    packed, q, a2, off = R.quantize(w)
    codes = torch.stack([packed[0].long() >> 4, packed[0].long() & 15], -1).reshape(-1)
    assert codes[:16].tolist() == list(range(16))
    want = [(mids < v).sum().item() for v in x[16:46]]             # bf16 storage moves the probes: recompute from x
    assert codes[16:46].tolist() == want
    assert codes[46].item() == int((mids < x[46]).sum())


def test_packing_is_high_nibble_first():
    w = torch.zeros(1, 64, dtype=torch.bfloat16)
    w[0, 0], w[0, 1] = -1.0, 1.0                                    # codes 0 and 15
    packed, *_ = R.quantize(w)
    assert packed.shape == (1, 32) and packed[0, 0].item() == 0x0F
    assert packed[0, 1:].tolist() == [0x77] * 31                  # zeros are code 7


def test_all_zero_block_and_partial_group():
    g = torch.Generator().manual_seed(0)
    N, K = 5, 64 * 300 // 5 * 1                                     # 300 blocks: one full group of 256 + a partial one
    w = (torch.randn(N, K, generator=g) * 0.02).to(torch.bfloat16)
    w[2, :64] = 0                                                   # one all-zero block
    packed, q, a2, off = R.quantize(w)
    assert a2.numel() == 2 and q.numel() == 300
    wt = R.dequantize(packed, q, a2, off)
    assert not torch.isnan(wt.float()).any()
    assert torch.equal(wt[2, :64].float(), torch.zeros(64))
    err = (wt.float() - w.float()).norm() / w.float().norm()
    assert err < 0.15, err
    # a group whose scales are all equal to the offset stores the index of 0.0 and decodes to the offset exactly
    w1 = torch.ones(1, 64 * 3, dtype=torch.bfloat16) * 0.5
    packed, q, a2, off = R.quantize(w1)
    assert a2.tolist() == [0.0] and q.tolist() == [R.ZERO_INDEX] * 3
    assert torch.equal(R.dequantize(packed, q, a2, off).float(), w1.float())


def test_byte_accounting():
    from cambrian_b200 import quant
    cfg = tiny_cambrian_config()
    qw = quant.NF4Weight(512, 256, "cpu")
    assert qw.nbytes == quant.bytes_per_weight(512, 256) == 512 * 128 + 2048 + 4 * 8 + 4
    H, I = cfg.hidden_size, cfg.intermediate_size
    assert quant.bytes_per_layer(cfg) == sum(quant.bytes_per_weight(n, k) for n, k in
                                             [(H, H), (H // 2, H), (H // 2, H), (H, H), (I, H), (I, H), (H, I)])
    with pytest.raises(ValueError):
        quant.NF4Weight(4, 96, "cpu")


# ------------------------------------------------------------------------------------------------ host routing
def test_nf4_linear_routes_decode_to_gemv_and_prefill_to_dequant_gemm(monkeypatch):
    from cambrian_b200 import _lib, ops, quant
    calls = []

    class FakeLib:
        def __getattr__(self, name):
            return lambda *a: calls.append(name) or 0

    monkeypatch.setattr(ops, "_require_cuda_bf16", lambda *a: None)
    monkeypatch.setattr(_lib, "load", lambda: FakeLib())
    monkeypatch.setattr(ops, "stream", lambda: 0)
    scratch = torch.empty(1024 * 256, dtype=torch.bfloat16)
    parts = [quant.NF4Weight(n, 256, "cpu") for n in (256, 128, 128)]
    qkv = quant.NF4Projection(parts, scratch)
    gu = quant.NF4Projection([quant.NF4Weight(512, 256, "cpu"), quant.NF4Weight(512, 256, "cpu")], scratch)
    for M, want in ((1, ["cb_gemv_nf4"]), (8, ["cb_gemv_nf4"]), (9, ["cb_nf4_dequant", "cb_gemm_bf16"]),
                    (2048, ["cb_nf4_dequant", "cb_gemm_bf16"])):
        calls.clear()
        y = ops.nf4_linear(torch.zeros(M, 256, dtype=torch.bfloat16), qkv)
        assert calls == want and y.shape == (M, 512), (M, calls)
    calls.clear()
    ops.nf4_mlp_gate_up(torch.zeros(4, 256, dtype=torch.bfloat16), gu)
    assert calls == ["cb_gemv_nf4", "cb_swiglu_fwd"]
    calls.clear()
    ops.nf4_mlp_gate_up(torch.zeros(300, 256, dtype=torch.bfloat16), gu)
    calls[:] = [c for c in calls if c != "cb_sm_count"]
    assert calls[0] == "cb_nf4_dequant" and calls[1:] in (["cb_gemm_bf16", "cb_swiglu_fwd"], ["cb_gemm_swiglu_bf16"])


# ------------------------------------------------------------------------------------------------ model plumbing
def _build(cfg, seed=3):
    from cambrian_b200.model.language_model.cambrian_llama import CambrianLlamaForCausalLM
    torch.manual_seed(seed)
    cfg.dino_config_overrides = dict(hidden_size=384, num_hidden_layers=2, num_attention_heads=6, mlp_ratio=4)
    model = CambrianLlamaForCausalLM(cfg)
    for t in model.get_model().vision_tower_aux_list:
        t.load_model()
    with torch.no_grad():
        for n_, p in model.named_parameters():
            if "pos_embed" in n_:
                p.mul_(0.1)
    return model.to(torch.bfloat16)


@needs_no_gpu
def test_load_4bit_quantises_exactly_the_seven_projections(monkeypatch, tmp_path):
    from cambrian_b200 import checkpoint, quant
    from cambrian_b200.model.language_model.cambrian_llama import CambrianLlamaForCausalLM
    ops_emulation.install(monkeypatch)
    R.install(monkeypatch)
    cfg = tiny_cambrian_config()
    torch.manual_seed(0)
    src = CambrianLlamaForCausalLM(cfg).to(torch.bfloat16)
    src.save_pretrained(tmp_path / "ckpt")
    ref = src.state_dict()
    _, model, _, _ = checkpoint.load_pretrained_model(str(tmp_path / "ckpt"), load_4bit=True, device="cpu",
                                                      load_tokenizer=False)
    assert quant.is_quantized(model)
    sd = model.state_dict()
    for i, layer in enumerate(model.get_model().layers):
        assert set(layer._nf4) == {"qkv", "o", "gate_up", "down"}
        parts = dict(zip(quant.PROJECTIONS, layer._nf4["qkv"].parts + layer._nf4["o"].parts +
                         layer._nf4["gate_up"].parts + layer._nf4["down"].parts))
        for name in quant.PROJECTIONS:
            sub = "self_attn" if name in ("q_proj", "k_proj", "v_proj", "o_proj") else "mlp"
            key = f"model.layers.{i}.{sub}.{name}.weight"
            assert sd[key].numel() == 0 and not model.get_parameter(key).requires_grad
            want = R.quantize(ref[key])
            got = parts[name]
            assert got.shape == tuple(ref[key].shape)
            assert torch.equal(got.packed, want[0]) and torch.equal(got.qabsmax, want[1])
    for k, v in sd.items():
        if v.numel():
            assert v.dtype == torch.bfloat16 and torch.equal(v, ref[k]), k
    quantised = sum(1 for k, v in sd.items() if v.numel() == 0)
    assert quantised == 7 * cfg.num_hidden_layers
    assert all(p.numel() == 0 for n, p in model.named_parameters() if "layers." in n and "proj" in n
               and "vision" not in n)


@needs_no_gpu
def test_greedy_generate_4bit_matches_fp32_oracle_on_dequantised_weights(monkeypatch):
    from test_parity_gpu import _oracle_greedy

    from cambrian_b200 import quant
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
    stats = quant.quantize_decoder_nf4_(model, "cpu")
    assert stats["nf4_bytes"] == cfg.num_hidden_layers * quant.bytes_per_layer(cfg)
    sd = {k: v.detach().float() for k, v in model.state_dict().items()}
    for i, layer in enumerate(model.get_model().layers):
        nf = layer._nf4
        qkv = R.projection_weight(nf["qkv"]).float()
        H, hd = cfg.hidden_size, cfg.hidden_size // cfg.num_attention_heads
        nq, nk = cfg.num_attention_heads * hd, cfg.num_key_value_heads * hd
        gu = R.projection_weight(nf["gate_up"]).float()
        I = cfg.intermediate_size
        pre = f"model.layers.{i}."
        sd[pre + "self_attn.q_proj.weight"], sd[pre + "self_attn.k_proj.weight"], sd[pre + "self_attn.v_proj.weight"] = \
            qkv[:nq], qkv[nq:nq + nk], qkv[nq + nk:]
        sd[pre + "self_attn.o_proj.weight"] = R.projection_weight(nf["o"]).float()
        sd[pre + "mlp.gate_proj.weight"], sd[pre + "mlp.up_proj.weight"] = gu[:I], gu[I:]
        sd[pre + "mlp.down_proj.weight"] = R.projection_weight(nf["down"]).float()
    from test_model_host_logic_cpu import _batch, _tower_feats
    ids, labels, attn, pos, masks = _batch(cfg, S=96)
    S0, n_new = 40, 12
    gen_ids = ids[:1, :S0].clone()
    feats = [f[:1] for f in _tower_feats(model, cfg, 2, 31)]
    monkeypatch.setattr(type(model), "encode_images", lambda self, imgs: feats)
    images = [torch.zeros(1, 3, 8, 8, dtype=torch.bfloat16) for _ in feats]
    new = model.generate(gen_ids, images=images, image_sizes=[(56, 56)], max_new_tokens=n_new, do_sample=False)
    want, margins = _oracle_greedy(sd, cfg, oracle_cfg(cfg), [f.float() for f in feats], gen_ids, n_new, torch.float32,
                                   torch.device("cpu"))
    assert new[0].tolist() == want, (new[0].tolist(), want, margins)
    assert len(set(want)) >= 4
    # scoring without a cache (no_grad) runs the same inference body; with grad enabled a 4-bit model refuses
    with torch.no_grad():
        out = model(input_ids=gen_ids, images=images, image_sizes=[(56, 56)])
    assert torch.isfinite(out.logits).all()
    with pytest.raises(NotImplementedError, match="QLoRA"):
        model(input_ids=gen_ids, images=images, image_sizes=[(56, 56)])


@needs_no_gpu
def test_quantised_model_refuses_training_sharding_and_saving(monkeypatch, tmp_path):
    from cambrian_b200 import checkpoint, quant
    from cambrian_b200.engine import TrainEngine
    from cambrian_b200.sharded import Zero3Inference
    ops_emulation.install(monkeypatch)
    R.install(monkeypatch)
    cfg = tiny_cambrian_config()
    model = _build(cfg)
    quant.quantize_decoder_nf4_(model, "cpu")
    with pytest.raises(ValueError, match="NF4"):
        TrainEngine(model)
    with pytest.raises(ValueError, match="NF4"):
        Zero3Inference(model)
    with pytest.raises(NotImplementedError):
        model.save_pretrained(tmp_path / "q")
    assert not (tmp_path / "q").exists()
    with pytest.raises(NotImplementedError, match="8-bit"):
        checkpoint.load_pretrained_model("x", load_8bit=True, load_tokenizer=False)
