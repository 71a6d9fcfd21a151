"""CPU tests of the host-side logic: collator mirror vs golden fixtures from the reference functions, tower-name
parsing / builder dispatch / error conventions, fused-parameter storage, image-token expansion, TrainEngine flat layout,
and the data-parallel gradient reduction on a 2-process gloo group."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
sys.path.insert(0, HERE)
from helpers import ns, tiny_cambrian_config  # noqa: E402


# ------------------------------------------------------------------------------------------------ collator (bit-exact)
def test_prepare_image_info_matches_reference_golden():
    from cambrian_b200.train.collator import prepare_image_info
    z = np.load(os.path.join(GOLD, "collator.npz"))
    n = 0
    for key in z.files:
        if not key.startswith("mask_"):
            continue
        _, wh, tok, nl = key.split("_")
        w, h = map(int, wh.split("x"))
        m, p = prepare_image_info((w, h), int(tok), newline=bool(int(nl)))
        assert np.array_equal(m.numpy(), z[key]), key
        assert np.array_equal(p.numpy(), z["pos_" + key[5:]]), key
        n += 1
    assert n >= 15


def test_prepare_multimodal_data_matches_reference_golden():
    from cambrian_b200.train.collator import prepare_multimodal_data
    z = np.load(os.path.join(GOLD, "collator.npz"))
    ids = torch.from_numpy(z["cm_ids_in"])
    attn = torch.from_numpy(z["cm_attn_in"])
    out = prepare_multimodal_data(ids, ids.clone(), attn, [(640, 480), (336, 336), (200, 1000)], image_token_len=16,
                                  image_aux_token_len_list=[16, 64], max_length=64)
    for got, key in zip(out[:4], ("cm_ids", "cm_labels", "cm_attn", "cm_pos")):
        assert np.array_equal(got.numpy(), z[key]), key
    assert np.array_equal(out[4][0].numpy(), z["cm_aux0"])
    assert np.array_equal(out[4][1].numpy(), z["cm_aux1"])


def test_collator_edge_cases():
    from cambrian_b200.train.collator import get_padding_offset, prepare_multimodal_data
    assert get_padding_offset((24, 24), (336, 336)) == (0, 0, 0, 0)
    l, r, t, b = get_padding_offset((24, 24), (1000, 10))      # extreme aspect ratio: almost everything padded
    assert (l, r) == (0, 0) and t == b == 12                   # int(10 * 24/1000) = 0 visible rows
    ids = torch.tensor([[5, 6, 7]])
    with pytest.raises(AssertionError):                         # exactly one image per sample (train_fsdp.py:1100)
        prepare_multimodal_data(ids, ids, torch.ones_like(ids, dtype=torch.bool), [(10, 10)], 16, [16], 64)
    # truncation to max_length
    ids = torch.full((1, 60), 9)
    ids[0, 50] = -200
    o = prepare_multimodal_data(ids, ids.clone(), torch.ones_like(ids, dtype=torch.bool), [(10, 10)], 16, [16], 64)
    assert o[0].shape == (1, 64) and o[3].shape == (1, 64)


# ------------------------------------------------------------------------------------------------ builders / parsing
def test_tower_name_parsing_and_dispatch():
    from cambrian_b200.model.multimodal_encoder.builder import build_vision_tower_aux_list
    from cambrian_b200.model.multimodal_encoder.towers import (CLIPConvNextTower, ClipVisionTower, DinoVisionTower,
                                                               SiglipVisionTower, _parse_res_interp)
    assert _parse_res_interp("facebook/dinov2-large-res336-interp576") == ("facebook/dinov2-large", 336, 576)
    assert _parse_res_interp("openai/clip-vit-large-patch14-336-interp576") == ("openai/clip-vit-large-patch14-336", None, 576)
    cfg = ns(mm_vision_tower_aux_list=["siglip/CLIP-ViT-SO400M-14-384", "openai/clip-vit-large-patch14-336",
                                       "facebook/dinov2-large-res336", "clip-convnext-XXL-multi-stage"],
             mm_vision_tower_aux_token_len_list=[576, 576, 576, 9216])
    towers = build_vision_tower_aux_list(cfg, delay_load=True)
    assert [type(t) for t in towers] == [SiglipVisionTower, ClipVisionTower, DinoVisionTower, CLIPConvNextTower]
    assert [t.hidden_size for t in towers] == [1152, 1024, 1024, 5760]
    assert [t.num_patches for t in towers] == [576, 576, 576, 9216]
    assert [t.image_size for t in towers] == [384, 336, 336, 1024]
    assert towers[3].is_multi_stage and not towers[0].is_loaded
    with pytest.raises(ValueError, match="Unknown vision tower"):        # builder.py:147
        build_vision_tower_aux_list(ns(mm_vision_tower_aux_list=["acme/unknown"], mm_vision_tower_aux_token_len_list=[576]))


def test_projector_builder_keys_and_errors():
    from cambrian_b200.model.multimodal_projector.builder import build_vision_projector
    p = build_vision_projector(ns(mm_projector_type="mlp2x_gelu", mm_hidden_size=1024, hidden_size=4096))
    assert sorted(p.state_dict()) == ["0.bias", "0.weight", "2.bias", "2.weight"]
    assert p.state_dict()["0.weight"].shape == (4096, 1024)
    assert build_vision_projector(ns(mm_projector_type="linear", mm_hidden_size=8, hidden_size=16)).weight.shape == (16, 8)
    with pytest.raises(ValueError, match="Unknown projector type"):      # multimodal_projector/builder.py:78
        build_vision_projector(ns(mm_projector_type="qformer", mm_hidden_size=8, hidden_size=8))


def test_sampler_rejects_unsupported_configs():
    from cambrian_b200.model.vision_sampler import VisionTokenSampler
    with pytest.raises(NotImplementedError):
        VisionTokenSampler(64, 512, [512], [1], 512, 1)
    with pytest.raises(NotImplementedError):
        VisionTokenSampler(64, 512, [512], [1], 512, 1, layer_type="sep")
    with pytest.raises(AssertionError):
        VisionTokenSampler(64, 1024, [1024], [1], 1024, 1, layer_type="bogus")


def test_sep_sampler_state_dict_follows_the_reference_layout():
    """layer_type="sep" (VisionAggregationLayer, vision_sampler.py:330-405): parameter names and shapes in registration
    order — weight_mlp only with more than one tower, CrossAttention for r > 1, an MLP otherwise; CPU tensors raise."""
    from cambrian_b200.model.vision_sampler import VisionTokenSampler
    m = VisionTokenSampler(256, 1024, [1024] * 3, [2, 1, 3], 1024, 2, layer_type="sep")
    sd = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    p = "layers.1."
    assert sd[p + "weight_mlp.linear_2.weight"] == (3, 1024) and sd[p + "weight_mlp.linear_1.weight"] == (1024, 1280)
    assert sd[p + "aggregate_0.attention_layer.q_proj.0.bias"] == (1024,) and sd[p + "pos_embed_2"] == (9, 1024)
    assert sd[p + "aggregate_1.attention_layer.linear_1.weight"] == (1024, 1024) and p + "pos_embed_1" not in sd
    single = VisionTokenSampler(256, 1024, [1024], [2], 1024, 1, layer_type="sep")
    assert not any("weight_mlp" in k for k in single.state_dict())
    z = np.load(os.path.join(GOLD, "pin_state_dicts.npz"))     # the reference module's layout (tests/golden/make_golden.py)
    assert list(sd.items()) == [(str(k), tuple(int(x) for x in str(sh).split(",") if x))
                                for k, sh in zip(z["sep_sd_keys"], z["sep_sd_shapes"])]
    with pytest.raises(RuntimeError):
        m(torch.zeros(4, 1, 256), torch.zeros(4, 1, 1024), torch.zeros(4, 4, 1024), torch.zeros(4, 1, 1024),
          torch.zeros(4, 9, 1024))


def test_decode_projection_dispatch(monkeypatch):
    """ops.gemm routes decode-shaped projections (M <= 8 rows, plain epilogue) to the weight-streaming GEMV, except 6-8
    rows on wide outputs, which keep the tensor-core tile; training shapes, transposed
    operands and fused epilogues always take the tensor-core kernel.  Host-side routing only: both kernels are faked."""
    from cambrian_b200 import _lib, ops
    calls = []

    class FakeLib:
        def cb_gemm_bf16(self, *a):
            calls.append("gemm")
            return 0

    monkeypatch.setattr(ops, "_require_cuda_bf16", lambda *a: None)
    monkeypatch.setattr(ops, "gemv", lambda a, b, **kw: calls.append("gemv") or torch.empty(a.shape[0], b.shape[0]))
    monkeypatch.setattr(_lib, "load", lambda: FakeLib())
    monkeypatch.setattr(ops, "stream", lambda: 0)

    def route(M, N, K=64, **kw):
        calls.clear()
        ops.gemm(torch.zeros(M, K, dtype=torch.bfloat16), torch.zeros(N, K, dtype=torch.bfloat16), **kw)
        return calls[-1]

    assert route(1, 128256) == "gemv" and route(4, 28672) == "gemv" and route(5, 28672) == "gemv"
    assert route(8, 4096) == "gemv" and route(8, 6144) == "gemv"
    assert route(8, 28672) == "gemm" and route(6, 16384) == "gemm" and route(8, 128256) == "gemm"
    assert route(9, 4096) == "gemm" and route(2048, 4096) == "gemm"
    assert route(1, 4096, act="gelu") == "gemm"
    calls.clear()
    ops.gemm(torch.zeros(64, 8, dtype=torch.bfloat16), torch.zeros(64, 32, dtype=torch.bfloat16), a_mn=True, b_mn=True)
    assert calls == ["gemm"]


# ------------------------------------------------------------------------------------------------ model plumbing
def test_state_dict_keys_follow_the_reference_layout():
    from cambrian_b200.model.language_model.cambrian_llama import CambrianLlamaForCausalLM
    cfg = tiny_cambrian_config()
    m = CambrianLlamaForCausalLM(cfg)
    keys = set(m.state_dict())
    for k in ["model.embed_tokens.weight", "model.layers.0.self_attn.q_proj.weight", "model.layers.3.mlp.down_proj.weight",
              "model.norm.weight", "lm_head.weight", "model.mm_projector.0.weight", "model.mm_projector.2.bias",
              "model.mm_projector_aux_3.3.weight", "model.vision_sampler_0.layers.1.cross_attn.k_proj_2.1.weight",
              "model.vision_sampler_layers.1.layers.0.proj_in.weight", "model.vision_sampler_layers.0.layers.0.pos_embed_3",
              "model.vision_query", "model.image_newline"]:
        assert k in keys, k
    assert not any("vision_tower" in k for k in keys)       # frozen towers are not part of the state dict (cambrian_arch.py:125-128)
    assert m.get_model().vision_sampler_layers[0].layers[0].proj_in.weight.shape == (1024, cfg.hidden_size + 1024)


def test_fuse_rows_repoints_parameters_once():
    from cambrian_b200.model.language_model.cambrian_llama import CBLlamaDecoderLayer, _adjacent
    layer = CBLlamaDecoderLayer(tiny_cambrian_config(), 0)
    a = layer.self_attn
    before = [p.detach().clone() for p in (a.q_proj.weight, a.k_proj.weight, a.v_proj.weight)]
    qkv, gu, _, _ = layer._fused()
    assert qkv.shape == (256 + 128 + 128, 256) and gu.shape == (1024, 256)
    assert _adjacent([a.q_proj.weight.data, a.k_proj.weight.data, a.v_proj.weight.data])
    assert torch.equal(qkv, torch.cat(before, 0))
    ptr = qkv.data_ptr()
    qkv2, *_ = layer._fused()
    assert qkv2.data_ptr() == ptr                           # already adjacent: no new copy
    a.k_proj.weight.data = a.k_proj.weight.data.clone()     # e.g. after load_state_dict / .to(): adjacency broken
    qkv3, *_ = layer._fused()
    assert torch.equal(qkv3, torch.cat(before, 0)) and a.k_proj.weight.data_ptr() != 0


def test_expand_image_tokens_matches_collator():
    from cambrian_b200.model.cambrian_arch import _expand_image_tokens
    from cambrian_b200.train.collator import prepare_multimodal_data
    ids = torch.randint(3, 100, (2, 30))
    ids[0, 4] = -200
    ids[1, 11] = -200
    attn = torch.ones_like(ids, dtype=torch.bool)
    e_ids, e_lab, e_mask, e_pos = _expand_image_tokens(ids, ids.clone(), attn, 20, "cpu")
    c = prepare_multimodal_data(ids, ids.clone(), attn, [(64, 64), (64, 64)], 16, [16], 1000)
    assert torch.equal(e_ids, c[0]) and torch.equal(e_lab, c[1]) and torch.equal(e_mask, c[2]) and torch.equal(e_pos, c[3])


# ------------------------------------------------------------------------------------------------ data parallel
def _dp_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from cambrian_b200 import engine as E
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(16, 24, bias=True), torch.nn.Linear(24, 8, bias=False)).bfloat16()
    eng = E.TrainEngine(model, bucket_mb=0.0005)  # tiny buckets -> several all-reduces
    assert eng.world == world and len(eng.buckets) >= 2
    # flat layout: parameters are views of one buffer in named_parameters() order, 8-element aligned
    off = 0
    for p in eng.params:
        assert p.data_ptr() == eng.flat_p.data_ptr() + 2 * off and p.main_grad.data_ptr() == eng.flat_g.data_ptr() + 2 * off
        off += (p.numel() + 7) // 8 * 8
    eng.zero_grad()
    for i, p in enumerate(eng.params):
        p.main_grad.fill_(float(rank + 1) * (i + 1))
        p._cb_fresh.add("all")
    eng.reduce_gradients()
    ok = all(torch.allclose(p.main_grad.float(), torch.full_like(p.main_grad, 3.0 * (i + 1)).float())
             for i, p in enumerate(eng.params))
    q.put((rank, ok))
    dist.destroy_process_group()


def _zero2_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from cambrian_b200 import engine as E
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(16, 24, bias=True), torch.nn.Linear(24, 9, bias=False)).bfloat16()
    eng = E.TrainEngine(model, zero_stage=2)
    assert eng.total == eng.shard * world and eng.master.numel() == eng.shard   # optimizer state is sharded
    assert all((e - s) % (8 * world) == 0 for s, e, _ in eng.buckets)           # every rank owns an aligned piece of each bucket
    # stand-in for the CUDA AdamW kernel (not available on CPU): plain SGD on the fp32 master slice
    def sgd(master, m, v, g, p16, lr, wd, step, coef):
        master.sub_(0.5 * g.float() / world)
        p16.copy_(master.to(torch.bfloat16))
    eng._adamw = sgd
    before = eng.flat_p.float().clone()
    eng.zero_grad()
    for i, p in enumerate(eng.params):
        p.main_grad.fill_(float(rank + 1) * 0.25 * (i + 1))
        p._cb_fresh.add("all")
    eng.step()
    # expected: every element moved by 0.5 * mean over ranks of its gradient = 0.5 * 0.375 * (i+1)
    ok = True
    for i, (p, o) in enumerate(zip(eng.params, eng.offsets)):
        exp = before[o:o + p.numel()] - 0.5 * 0.375 * (i + 1)
        ok &= torch.allclose(eng.flat_p[o:o + p.numel()].float(), exp.to(torch.bfloat16).float(), atol=2e-2)
        ok &= p.data_ptr() == eng.flat_p.data_ptr() + 2 * o     # parameters still alias the (all-gathered) flat buffer
    q.put((rank, bool(ok)))
    dist.destroy_process_group()


def test_zero2_sharded_optimizer_two_ranks_gloo():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + os.getpid() % 2000
    procs = [ctx.Process(target=_zero2_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=180) for _ in procs)
    for p in procs:
        p.join(60)
    assert res == [(0, True), (1, True)]


def test_gradient_allreduce_two_ranks_gloo():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=180) for _ in procs)
    for p in procs:
        p.join(60)
    assert res == [(0, True), (1, True)]


# ------------------------------------------------------------------------------------------------ checkpoints (§8f rank 2)
def test_hf_checkpoint_roundtrip_and_mm_projector_overlay(tmp_path):
    """save_pretrained -> from_pretrained keeps every tensor (the released checkpoints use this layout); the adapter-only
    file holds exactly the reference's key filter (train_fsdp.py:255) and overlays onto a fresh model."""
    from cambrian_b200 import checkpoint
    from cambrian_b200.model.language_model.cambrian_llama import CambrianLlamaForCausalLM
    cfg = tiny_cambrian_config()
    torch.manual_seed(0)
    m = CambrianLlamaForCausalLM(cfg)
    m.save_pretrained(tmp_path / "full")
    m2 = CambrianLlamaForCausalLM.from_pretrained(tmp_path / "full")
    a, b = m.state_dict(), m2.state_dict()
    assert list(a) == list(b)
    assert all(torch.equal(a[k], b[k]) for k in a)
    assert m2.config.mm_vision_tower_aux_token_len_list == cfg.mm_vision_tower_aux_token_len_list
    # adapter-only checkpoint
    path = checkpoint.save_mm_projector(m, str(tmp_path / "adapter"))
    sd = torch.load(path)
    assert all(any(key in k for key in checkpoint.ADAPTER_KEYS) for k in sd)
    assert "model.vision_query" in sd and "model.image_newline" in sd and "model.mm_projector.0.weight" in sd
    assert not any(k.startswith("model.layers.") or k.startswith("lm_head") or "embed_tokens" in k for k in sd)
    torch.manual_seed(1)
    fresh = CambrianLlamaForCausalLM(cfg)
    assert not torch.equal(fresh.state_dict()["model.vision_query"], a["model.vision_query"])
    unexpected = checkpoint.load_mm_projector(fresh, path, strict_submodules=True)
    assert unexpected == []
    f = fresh.state_dict()
    assert all(torch.equal(f[k], a[k]) for k in sd)
    assert not torch.equal(f["model.layers.0.mlp.up_proj.weight"], a["model.layers.0.mlp.up_proj.weight"])
    # wrapper prefixes of PEFT-era files (builder.py:84-86) and shape errors
    checkpoint.load_mm_projector(fresh, {"base_model.model." + k: v for k, v in sd.items()})
    with pytest.raises(RuntimeError):
        checkpoint.load_mm_projector(fresh, {"model.image_newline": torch.zeros(3)})
    with pytest.raises(RuntimeError):
        checkpoint.load_mm_projector(fresh, {"model.image_newline": a["model.image_newline"]}, strict_submodules=True)
    with pytest.raises(NotImplementedError):
        checkpoint.load_pretrained_model("x", model_name="cambrian-lora", load_tokenizer=False)


def test_state_dict_keys_equal_the_reference_modules():
    """Connector key set == the reference's own modules' (stored by tests/golden/make_golden.py)."""
    from cambrian_b200.model.vision_sampler import VisionTokenSampler
    z = np.load(os.path.join(GOLD, "pin_state_dicts.npz"))
    for i, args in enumerate([(1024, 1024, [1024] * 4, [1, 1, 1, 1], 1024, 3), (256, 1024, [1024] * 3, [1, 2, 3], 1024, 1)]):
        assert [str(k) for k in z[f"keys{i}"]] == list(VisionTokenSampler(*args).state_dict())


# ------------------------------------------------------------------------------------------------ ZeRO-3 inference (§8e, config 5)
def _zero3_worker(rank, world, port, n_layers, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from cambrian_b200.model.language_model.cambrian_llama import CambrianLlamaForCausalLM
        from cambrian_b200.sharded import Zero3Inference
        cfg = tiny_cambrian_config()
        cfg.num_hidden_layers = n_layers
        torch.manual_seed(5)
        m = CambrianLlamaForCausalLM(cfg).to(torch.bfloat16)
        want = [{k: v.clone() for k, v in layer.state_dict().items()} for layer in m.get_model().layers]
        z = Zero3Inference(m)
        assert all(p.numel() == 0 for layer in m.get_model().layers for p in layer.parameters())
        assert z.shards[0].numel() * world >= sum(v.numel() for v in want[0].values())
        ok = True
        for sweep in range(3):                        # prefill + two decode steps: the prefetch wraps around
            for i, layer in enumerate(m.get_model().layers):
                z.before_layer(i)
                got = layer.state_dict()
                ok &= all(torch.equal(got[k], want[i][k]) for k in want[i])
                qkv, gu, _, _ = layer._fused()        # fused views stay zero-copy inside the staging buffer
                ok &= qkv.data_ptr() == layer.self_attn.q_proj.weight.data_ptr()
        done = torch.tensor([rank == 0])
        ok &= z.all_done(done) is False and z.all_done(torch.tensor([True])) is True
        q.put((rank, bool(ok), z.gathers))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("n_layers", [4, 3])
def test_zero3_inference_gathers_every_layer_world2(n_layers):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29650 + n_layers
    procs = [ctx.Process(target=_zero3_worker, args=(r, 2, port, n_layers, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=180) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    assert [r[1] for r in res] == [True, True], res
    assert res[0][2] == 3 * n_layers + 1              # one gather per layer visit + the wrapped prefetch left in flight


# ------------------------------------------------------------------------------------------------ preprocessing (§8f rank 4)
def _pil_equivalent_resize(arr, R, pad):
    """numpy emulation of the two CUDA passes using the library's coefficient tables (host entry point)."""
    from cambrian_b200 import ops
    H, W, _ = arr.shape
    S = max(H, W)
    sq = np.empty((S, S, 3), dtype=np.int64)
    sq[...] = np.array(pad)
    oy, ox = ((W - H) // 2, 0) if W > H else (0, (H - W) // 2)
    sq[oy:oy + H, ox:ox + W] = arr
    bounds, kk = ops.resample_coeffs(S, R)
    bounds, kk = bounds.numpy(), kk.numpy().astype(np.int64)

    def one_pass(src):                                   # resample axis 1
        out = np.empty((src.shape[0], R, 3), dtype=np.int64)
        for xx in range(R):
            x0, n = bounds[xx]
            acc = (src[:, x0:x0 + n, :] * kk[xx, :n, None]).sum(1) + (1 << 21)
            out[:, xx, :] = np.clip(acc >> 22, 0, 255)
        return out
    tmp = one_pass(sq)
    return one_pass(tmp.transpose(1, 0, 2)).transpose(1, 0, 2).astype(np.uint8)


@pytest.mark.parametrize("hw,R", [((480, 640), 336), ((700, 300), 384), ((100, 130), 336), ((336, 336), 336),
                                  ((1500, 1100), 1024)])
def test_resample_coefficients_reproduce_pillow_bit_exact(hw, R):
    """Pins the restated Resample.c arithmetic (third-party: Pillow, the `Image.resize` of mm_utils.py:194) against the
    installed Pillow on the reference's own call chain expand2square -> resize."""
    from PIL import Image
    rng = np.random.default_rng(hw[0] * 7 + R)
    arr = rng.integers(0, 256, size=(hw[0], hw[1], 3), dtype=np.uint8)
    pad = (122, 116, 104)
    img = Image.fromarray(arr)
    w, h = img.size
    if w != h:                                            # expand2square, mm_utils.py:153-164
        s = max(w, h)
        sq = Image.new(img.mode, (s, s), pad)
        sq.paste(img, (0, (w - h) // 2) if w > h else ((h - w) // 2, 0))
        img = sq
    want = np.asarray(img.resize((R, R)))
    got = _pil_equivalent_resize(arr, R, pad)
    assert np.array_equal(got, want)


# ------------------------------------------------------------------------------------------------ dynamic-branch host helpers
def test_product_unmask_and_unpad_match_reference_golden():
    """cambrian_b200.model.cambrian_arch.unmask_attention_mask / unpad_image / unpad_bounds (host code of the dynamic
    branch) against the fixtures generated from the reference's own functions (tests/golden/dynamic.npz)."""
    from cambrian_b200.model import cambrian_arch as A
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "dynamic.npz"))
    n = 0
    for k in z.files:
        if not k.startswith("unmask_"):
            continue
        wh, side = k[len("unmask_"):].rsplit("_", 1)
        w, h = map(int, wh.split("x"))
        side = int(side)
        got = A.unmask_attention_mask(torch.ones(1, side, side, dtype=torch.bool), (w, h))
        assert np.array_equal(got.numpy(), z[k]), k
        y0, y1, x0, x1 = A.unpad_bounds(side, side, (w, h))
        assert (y1 - y0, x1 - x0) == tuple(z["unpad_" + k[len("unmask_"):]]), k
        t = torch.arange(side * side).view(1, side, side, 1)
        assert torch.equal(A.unpad_image(t, (w, h)), t[:, y0:y1, x0:x1])
        n += 1
    assert n == 15


def test_product_unmask_and_unpad_match_live_reference_on_random_sizes():
    """The product's unmask_attention_mask / unpad_image vs the reference's on 300 random image sizes (the reference's
    masks and crops stored by tests/golden/make_golden.py)."""
    sys.path.insert(0, GOLD)
    from make_golden import unpad_cases
    from cambrian_b200.model import cambrian_arch as A
    z = np.load(os.path.join(GOLD, "pin_unpad.npz"))
    offs = np.concatenate([[0], np.cumsum(z["mask_lens"])])
    for i, (w, h, side) in enumerate(unpad_cases()):
        got = A.unmask_attention_mask(torch.ones(1, side, side, dtype=torch.bool), (w, h))
        want = np.unpackbits(z["masks"][offs[i]:offs[i + 1]])[:side * side].reshape(1, side, side).astype(bool)
        assert np.array_equal(got.numpy(), want), (w, h, side)
        y0, y1, x0, x1 = (int(v) for v in z["crops"][i])
        if y0 < 0:
            continue                                   # degenerate aspect ratios crop everything away in the reference too
        t = torch.arange(side * side).view(1, side, side, 1)
        assert torch.equal(A.unpad_image(t, (w, h)), t[:, y0:y1, x0:x1]), (w, h, side)


def test_valid_label_ranges_cover_exactly_the_valid_shifted_labels():
    from cambrian_b200.train.collator import valid_label_ranges
    rng = np.random.default_rng(9)
    for _ in range(50):
        B, S = int(rng.integers(1, 5)), int(rng.integers(2, 40))
        lab = torch.from_numpy(np.where(rng.random((B, S)) < 0.5, -100, rng.integers(0, 100, (B, S))))
        ranges, n = valid_label_ranges(lab)
        shift = torch.full_like(lab, -100)
        shift[:, :-1] = lab[:, 1:]
        mask = torch.zeros(B * S, dtype=torch.bool)
        for a, b in ranges:
            assert a < b
            mask[a:b] = True
        assert torch.equal(mask, (shift != -100).view(-1)) and n == int(mask.sum())
        assert all(ranges[i][1] < ranges[i + 1][0] for i in range(len(ranges) - 1))       # maximal, ordered runs


# ------------------------------------------------------------------------------------------------ generate() policy (A12)
def test_sampling_warpers_match_transformers():
    """temperature / top-k / top-p filtering == HF's LogitsWarpers (what GenerationMixin.generate applies for the
    reference's callers: model_worker.py:177-187 passes do_sample, temperature, top_p)."""
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    from cambrian_b200.generation import warp_logits
    torch.manual_seed(0)
    logits = torch.randn(3, 500) * 3
    for temp, k, p in [(0.7, 50, 0.9), (1.0, 0, 0.5), (1.3, 10, 1.0), (0.2, 50, 0.95)]:
        want = logits.clone()
        if temp != 1.0:
            want = TemperatureLogitsWarper(temp)(None, want)
        if k:
            want = TopKLogitsWarper(k)(None, want)
        if p < 1.0:
            want = TopPLogitsWarper(p)(None, want)
        got = warp_logits(logits, temp, k, p)
        assert torch.equal(torch.isinf(got), torch.isinf(want)), (temp, k, p)
        keep = ~torch.isinf(want)
        torch.testing.assert_close(got[keep], want[keep])


def test_generation_kwargs_are_honoured_or_rejected_never_dropped():
    from cambrian_b200.generation import GenerationArgs
    model = ns(config=ns(eos_token_id=2, pad_token_id=None), generation_config=None)
    a = GenerationArgs.from_kwargs(model, 10, dict(do_sample=True, temperature=0.2, top_p=0.7, max_new_tokens=7, num_beams=1,
                                                   use_cache=True, stopping_criteria=[lambda i, s: False], streamer=None))
    assert (a.do_sample, a.temperature, a.top_p, a.top_k, a.max_new_tokens, a.eos_token_ids, a.pad_token_id) == \
        (True, 0.2, 0.7, 50, 7, [2], 2) and len(a.stopping_criteria) == 1
    a = GenerationArgs.from_kwargs(model, 10, dict(do_sample=False, temperature=0, max_length=30))     # inference.py:77-85
    assert not a.do_sample and a.max_new_tokens == 20
    with pytest.raises(NotImplementedError, match="num_beams"):
        GenerationArgs.from_kwargs(model, 10, dict(num_beams=4))
    with pytest.raises(NotImplementedError, match="repetition_penalty"):
        GenerationArgs.from_kwargs(model, 10, dict(repetition_penalty=1.2))
    with pytest.raises(TypeError, match="frobnicate"):
        GenerationArgs.from_kwargs(model, 10, dict(frobnicate=1))
    with pytest.raises(ValueError, match="top_p"):
        GenerationArgs.from_kwargs(model, 10, dict(do_sample=True, top_p=0.0))


def test_cosine_schedule_equals_transformers():
    from transformers import get_cosine_schedule_with_warmup
    from cambrian_b200.engine import cosine_schedule_with_warmup
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.SGD([p], lr=1.0)
    sched = get_cosine_schedule_with_warmup(opt, 7, 100)
    f = cosine_schedule_with_warmup(7, 100)
    for step in range(100):
        assert abs(sched.get_last_lr()[0] - f(step)) < 1e-12, step
        opt.step()
        sched.step()


def test_module_alias_recipe_from_integration_md():
    """INTEGRATION.md §1: aliasing `cambrian.model` to the drop-in package must make the reference's import statements
    resolve to the drop-in classes (run in a subprocess: it edits sys.modules)."""
    import subprocess
    import sys as _sys
    code = r'''
import sys, cambrian_b200.model as m
sys.modules["cambrian"] = type(sys)("cambrian")
sys.modules["cambrian.model"] = m
for sub in ("vision_sampler", "cambrian_arch", "multimodal_encoder.builder", "multimodal_projector.builder",
            "language_model.cambrian_llama"):
    sys.modules["cambrian.model." + sub] = __import__("cambrian_b200.model." + sub, fromlist=["*"])
from cambrian.model.language_model.cambrian_llama import CambrianLlamaForCausalLM, CambrianConfig
from cambrian.model.vision_sampler import VisionTokenSampler
from cambrian.model.multimodal_encoder.builder import build_vision_tower_aux_list
from cambrian.model.multimodal_projector.builder import build_vision_projector
import cambrian_b200.model.language_model.cambrian_llama as ours
assert CambrianLlamaForCausalLM is ours.CambrianLlamaForCausalLM and CambrianConfig.model_type == "cambrian_llama"
from transformers import AutoConfig
assert type(AutoConfig.for_model("cambrian_llama")).__name__ == "CambrianConfig"
print("alias ok")
'''
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([_sys.executable, "-c", code], capture_output=True, text=True, cwd=root, timeout=300)
    assert r.returncode == 0 and "alias ok" in r.stdout, r.stderr[-2000:]
