"""Pins the CPU oracle (oracle/cambrian_oracle.py) — CPU only, no GPU:
  * against the committed golden fixtures generated from the reference's own modules (tests/golden/make_golden.py);
  * against the installed `transformers` implementations the reference delegates to (CLIPVisionModel, Dinov2Model,
    LlamaDecoderLayer + LlamaRMSNorm + rotary embedding);
  * against stored outputs (and sampled gradients) of the reference modules in the configurations below
    (tests/golden/pin_*.npz, same generator)."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden import (SEP_LIVE_CASES, SVA_CASES, SVA_FULL_CASES, SVA_SEP_CASES, TWO_GROUPS, config1_inputs,  # noqa: E402
                         flat_sample, grad_sample_index, projector_input, sd_from_layout, seeded_fill, seeded_inputs,
                         sep_live_dy, two_groups_inputs)

from oracle import cambrian_oracle as O  # noqa: E402

GOLD = os.path.join(HERE, "golden")


def _sva_shapes(q_dim, rs, layers):
    """state-dict shapes of VisionTokenSampler in the reference's registration order (vision_sampler.py:254-268,170-175)."""
    sd = {}
    for l in range(layers):
        p = f"layers.{l}."
        for i, r in enumerate(rs):
            if r > 1:
                sd[p + f"pos_embed_{i}"] = (r * r, 1024)
        sd[p + "proj_context.weight"] = (1024, 1024)
        sd[p + "proj_in.weight"] = (1024, q_dim + 1024)
        sd[p + "proj_out.linear_1.weight"] = (1024, 1024)
        sd[p + "proj_out.linear_2.weight"] = (q_dim, 1024)
        sd[p + "norm.weight"] = (1024,)
        sd[p + "norm.bias"] = (1024,)
        names = ["q_proj"] + [f"{k}_proj_{i}" for i in range(len(rs)) for k in "kv"]
        for nm in names:
            sd[p + f"cross_attn.{nm}.0.weight"] = (1024,)
            sd[p + f"cross_attn.{nm}.0.bias"] = (1024,)
            sd[p + f"cross_attn.{nm}.1.weight"] = (1024, 1024)
        sd[p + "cross_attn.o_proj.weight"] = (1024, 1024)
    return {k: torch.empty(v) for k, v in sd.items()}


@pytest.mark.parametrize("name", sorted(SVA_CASES))
def test_sva_oracle_matches_reference_golden(name):
    c = SVA_CASES[name]
    sd = seeded_fill(_sva_shapes(c["q_dim"], c["rs"], c["layers"]), c["seed"])
    queries, ctx, feats, masks = seeded_inputs(c["seed"] + 100, c["n"], c["q_dim"], c["rs"])
    with torch.no_grad():
        got = O.sva_sampler(sd, "", queries, ctx, feats, masks, c["layers"])
    ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
    torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-5)


def _sep_state_dict(name):
    """Seeded weights of a layer_type="sep" sampler, regenerated from the parameter names / shapes stored in the golden."""
    z = np.load(os.path.join(GOLD, name + ".npz"))
    shapes = {str(k): tuple(int(x) for x in str(sh).split(",")) for k, sh in zip(z["sd_keys"], z["sd_shapes"])}
    return seeded_fill({k: torch.empty(v) for k, v in shapes.items()}, SVA_SEP_CASES[name]["seed"]), z


@pytest.mark.parametrize("name", sorted(SVA_SEP_CASES))
def test_sva_sep_oracle_matches_reference_golden(name):
    """VisionAggregationLayer restatement (oracle.sva_agg_layer) vs the committed output of the reference's own
    VisionTokenSampler(layer_type="sep") (vision_sampler.py:330-419)."""
    c = SVA_SEP_CASES[name]
    sd, z = _sep_state_dict(name)
    queries, ctx, feats, masks = seeded_inputs(c["seed"] + 100, c["n"], c["q_dim"], c["rs"])
    with torch.no_grad():
        got = O.sva_sampler(sd, "", queries, ctx, feats, masks, c["layers"], layer_type="sep")
    torch.testing.assert_close(got, torch.from_numpy(z["out"]), rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("rs,q_dim,layers", SEP_LIVE_CASES)
def test_sva_sep_oracle_matches_live_reference_fwd_bwd(rs, q_dim, layers):
    """Output AND gradients of the sep restatement against the reference module's (output: a fixed sample plus every row
    sum; gradients: a fixed sample of every tensor plus its norm; tests/golden/pin_sep_fwd_bwd.npz)."""
    case = SEP_LIVE_CASES.index((rs, q_dim, layers))
    z = np.load(os.path.join(GOLD, "pin_sep_fwd_bwd.npz"))
    zc = {k[len(f"c{case}_"):]: z[k] for k in z.files if k.startswith(f"c{case}_")}
    sd = {k: v.requires_grad_() for k, v in sd_from_layout(zc, 71).items()}
    names = [str(k) for k in zc["names"]]
    queries, ctx, feats, masks = seeded_inputs(72, 10, q_dim, rs)
    queries.requires_grad_()
    got = O.sva_sampler(sd, "", queries, ctx, feats, masks, layers, layer_type="sep")
    ggot = torch.autograd.grad(got, [queries] + [sd[k] for k in names], sep_live_dy(got.shape))
    torch.testing.assert_close(flat_sample(got.detach()), torch.from_numpy(zc["out"]), rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(got.detach().sum(-1), torch.from_numpy(zc["outsum"]), rtol=1e-4, atol=1e-4)
    idx = grad_sample_index([g.numel() for g in ggot])
    sample = torch.cat([g.reshape(-1)[torch.from_numpy(ix)] for g, ix in zip(ggot, idx)])
    torch.testing.assert_close(sample, torch.from_numpy(zc["gsample"]), rtol=1e-3, atol=1e-5)
    norms = torch.tensor([g.double().norm().item() for g in ggot], dtype=torch.float64)
    torch.testing.assert_close(norms, torch.from_numpy(zc["gnorm"]), rtol=1e-3, atol=1e-6)


@pytest.mark.parametrize("name", sorted(SVA_FULL_CASES))
def test_sva_oracle_matches_reference_golden_full_size(name):
    """BASELINE config 1 at its real size (576 queries, 4 x 576 x 1024 grids, depth 3), the release grids [1,1,1,4] and one
    in-LLM layer at Llama-3-8B width: oracle vs the reference module's output (subsampled rows + all row sums)."""
    c = SVA_FULL_CASES[name]
    sd = seeded_fill(_sva_shapes(c["q_dim"], c["rs"], c["layers"]), c["seed"])
    queries, ctx, feats, masks = seeded_inputs(c["seed"] + 100, c["n"], c["q_dim"], c["rs"])
    with torch.no_grad():
        got = O.sva_sampler(sd, "", queries, ctx, feats, masks, c["layers"])[:, 0]
    z = np.load(os.path.join(GOLD, name + ".npz"))
    stride = 4 * c["q_dim"] // 1024
    torch.testing.assert_close(got[0::stride], torch.from_numpy(z["rows"]).float(), rtol=2e-3, atol=2e-3)  # fp16 storage
    torch.testing.assert_close(got.sum(1), torch.from_numpy(z["rowsum"]), rtol=1e-4, atol=2e-3)


def test_window_rearrange_matches_reference_golden():
    z = np.load(os.path.join(GOLD, "rearrange.npz"))
    got = O.window_rearrange(torch.from_numpy(z["feat"]), 4)
    assert torch.equal(got, torch.from_numpy(z["out"]))


def test_oracle_clip_matches_transformers():
    from transformers import CLIPVisionConfig, CLIPVisionModel
    torch.manual_seed(0)
    cfg = CLIPVisionConfig(hidden_size=128, intermediate_size=256, num_hidden_layers=3, num_attention_heads=2, patch_size=14,
                           image_size=56, hidden_act="quick_gelu")
    m = CLIPVisionModel(cfg).eval()
    img = torch.randn(2, 3, 56, 56)
    with torch.no_grad():
        ref = m(img, output_hidden_states=True).hidden_states[-2][:, 1:]      # clip_encoder.py:55-68
        got = O.clip_vit({k: v for k, v in m.state_dict().items()},
                         dict(num_hidden_layers=3, patch_size=14, num_attention_heads=2, select_layer=-2), img)
    torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("res,swiglu", [(518 // 37 * 4, False), (14 * 6, False), (14 * 6, True)])
def test_oracle_dinov2_matches_transformers(res, swiglu):
    """swiglu=True is the dinov2-giant FFN (the release tower, finetune_cambrian_8b.sh:17-18)."""
    from transformers import Dinov2Config, Dinov2Model
    torch.manual_seed(0)
    cfg = Dinov2Config(hidden_size=128, num_hidden_layers=2, num_attention_heads=2, mlp_ratio=4, patch_size=14,
                       image_size=56, use_swiglu_ffn=swiglu)
    m = Dinov2Model(cfg).eval()
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if "lambda1" in n_:
                p.copy_(0.5 + torch.rand_like(p))
    img = torch.randn(2, 3, res, res)
    with torch.no_grad():
        ref = m(img).last_hidden_state[:, 1:]                                 # dino_encoder.py:115-126
        got = O.dinov2_vit({k: v for k, v in m.state_dict().items()},
                           dict(num_hidden_layers=2, patch_size=14, num_attention_heads=2), img)
    torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-5)


def test_oracle_llama_layer_matches_transformers():
    from transformers import LlamaConfig
    from transformers.models.llama.modeling_llama import LlamaDecoderLayer, LlamaRotaryEmbedding
    torch.manual_seed(0)
    cfg = LlamaConfig(hidden_size=128, intermediate_size=256, num_hidden_layers=1, num_attention_heads=4,
                      num_key_value_heads=2, rms_norm_eps=1e-5, rope_theta=500000.0, max_position_embeddings=256)
    cfg._attn_implementation = "eager"
    layer = LlamaDecoderLayer(cfg, 0).eval()
    rot = LlamaRotaryEmbedding(cfg)
    B, S = 2, 37
    x = torch.randn(B, S, 128)
    pos = torch.arange(S)[None].expand(B, S)
    keymask = torch.ones(B, S, dtype=torch.bool)
    keymask[1, 30:] = False
    causal = torch.ones(S, S, dtype=torch.bool).tril()
    allow = causal[None, None] & keymask[:, None, None, :]
    add_mask = torch.zeros(B, 1, S, S).masked_fill(~allow, torch.finfo(torch.float32).min)
    with torch.no_grad():
        pe = rot(x, pos)
        ref = layer(x, attention_mask=add_mask, position_ids=pos, position_embeddings=pe)
        ref = ref[0] if isinstance(ref, tuple) else ref
        sd = {"model.layers.0." + k: v for k, v in layer.state_dict().items()}
        cos, sin = O.rope_cos_sin(pos, 32, 500000.0)
        got = O.llama_layer(sd, "model.layers.0.", x, cos, sin, keymask,
                            dict(num_attention_heads=4, num_key_value_heads=2, rms_norm_eps=1e-5))
    torch.testing.assert_close(got[keymask], ref[keymask], rtol=1e-4, atol=1e-5)


# ------------------------------------------------------------------ stored outputs of the reference modules (pin_*.npz)
def test_oracle_sva_config1_full_size_against_reference():
    """BASELINE config 1: SVA projector alone (576 queries, 4 x 24 x 24 x 1024 grids), plus the [1,1,1,4] variant, with
    random window masks: a fixed sample of the output and all row sums of the reference module."""
    z = np.load(os.path.join(GOLD, "pin_config1.npz"))
    for j, rs in enumerate(([1, 1, 1, 1], [1, 1, 1, 4])):
        zc = {k[3:]: z[k] for k in z.files if k.startswith(f"r{j}_")}
        query, ctx, fw, masks = config1_inputs(rs, 82 + j)
        with torch.no_grad():
            got = O.sva_sampler(sd_from_layout(zc, 81 + j), "", query, ctx, fw, masks, 3)[:, 0]
        torch.testing.assert_close(flat_sample(got, 512), torch.from_numpy(zc["sample"]), rtol=1e-4, atol=2e-5)
        torch.testing.assert_close(got.sum(1), torch.from_numpy(zc["rowsum"]), rtol=1e-4, atol=2e-3)


def test_oracle_two_query_groups_static_branch_against_reference():
    """cambrian_arch.py:382-420 with num_query_group = 2 (a 4x4 and a 2x2 group: own sampler each, window masks reused
    through the raw reshape of :284, the small group's output bilinearly resized to the final grid :394-401, channel concat,
    mm_projector, newline column) — the stored result of the reference's own prepare_inputs_labels_for_multimodal on its
    static (XLA) branch vs oracle.connector + splice."""
    c = TWO_GROUPS
    z = np.load(os.path.join(GOLD, "pin_two_groups.npz"))
    sd = {"model." + k: v for k, v in sd_from_layout(z, c["seed"]).items()}
    feats, masks, ids = two_groups_inputs()
    cfg = dict(image_token_len=c["q"] ** 2, query_num_list=[c["q"] ** 2, 4], connector_depth=2)
    with torch.no_grad():
        img, feats_w, ctx_q = O.connector(sd, cfg, feats, masks)
        got = O.splice(sd, ids, img)
    torch.testing.assert_close(flat_sample(got), torch.from_numpy(z["emb"]), rtol=1e-4, atol=2e-5)
    torch.testing.assert_close(got.sum(-1), torch.from_numpy(z["embsum"]), rtol=1e-4, atol=1e-4)
    for i, a in enumerate(feats_w):                 # window-rearranged aux features handed to the in-LLM SVA layers
        torch.testing.assert_close(flat_sample(a), torch.from_numpy(z[f"feat_w{i}"]), rtol=1e-4, atol=2e-5)


def test_oracle_projectors_against_reference():
    z = np.load(os.path.join(GOLD, "pin_projector.npz"))
    sd = {"p." + k: v for k, v in sd_from_layout(z, 95).items()}
    with torch.no_grad():
        torch.testing.assert_close(flat_sample(O.mlp2x_gelu(sd, "p.", projector_input())), torch.from_numpy(z["out"]),
                                   rtol=1e-5, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------------
# dynamic-shape (off-XLA / inference) branch for non-square images — golden generated from the reference's own
# unmask_attention_mask / unpad_image / rearrange_vision_tower_features_inference / prepare_inputs_labels_for_multimodal
# ---------------------------------------------------------------------------------------------------------------
def dynamic_golden():
    from make_golden import DYN, dynamic_inputs
    z = np.load(os.path.join(GOLD, "dynamic.npz"))
    shapes = {k: torch.empty([int(d) for d in sh.split(",")] if sh else [])
              for k, sh in zip(z["sd_keys"].tolist(), z["sd_shapes"].tolist())}
    sd = seeded_fill(shapes, DYN["seed"] + 1)
    return z, sd, DYN, dynamic_inputs()


def test_unmask_and_unpad_match_reference_golden():
    z = np.load(os.path.join(GOLD, "dynamic.npz"))
    n = 0
    for k in z.files:
        if k.startswith("unmask_"):
            wh, side = k[len("unmask_"):].rsplit("_", 1)
            w, h = map(int, wh.split("x"))
            got = O.unmask_attention_mask(torch.ones(1, int(side), int(side), dtype=torch.bool), (w, h))
            assert np.array_equal(got.numpy(), z[k]), k
            shp = O.unpad_image(torch.zeros(1, int(side), int(side), 1), (w, h)).shape[1:3]
            assert tuple(shp) == tuple(z["unpad_" + k[len("unmask_"):]]), k
            n += 1
    assert n == 15


@pytest.mark.parametrize("unpad", [False, True])
def test_rearrange_inference_matches_reference_golden(unpad):
    z, _, d, (feats, _, _, _) = dynamic_golden()
    fr, mr = O.rearrange_inference(feats, d["q"], d["sizes"], unpad=unpad)
    for i, (f, m) in enumerate(zip(fr, mr)):
        assert np.array_equal(f.numpy().astype(np.float16), z[f"re{int(unpad)}_f{i}"])       # pure gather: exact
        assert np.array_equal(m.numpy(), z[f"re{int(unpad)}_m{i}"])


def test_prepare_dynamic_matches_reference_golden():
    z, sd, d, (feats, ids, attn, labels) = dynamic_golden()
    cfg = dict(image_token_len=d["q"] ** 2, connector_depth=2)
    with torch.no_grad():
        emb, lab, am, pos, ff, mf, fs, ctx = O.prepare_dynamic(sd, cfg, feats, ids, attn, labels, d["sizes"])
    assert [tuple(x) for x in z["final_size"].tolist()] == [tuple(x) for x in fs]
    torch.testing.assert_close(emb, torch.from_numpy(z["emb"]), rtol=1e-4, atol=2e-5)
    assert np.array_equal(lab.numpy(), z["labels"]) and np.array_equal(am.numpy(), z["attn"])
    assert (ctx.numpy().astype(np.float32) - z["ctx"].astype(np.float32)).__abs__().max() < 2e-3     # stored as fp16
    for i, (f, m) in enumerate(zip(ff, mf)):
        assert np.abs(f.numpy() - z[f"final_f{i}"].astype(np.float32)).max() < 4e-3               # stored as fp16
        assert np.array_equal(m.numpy(), z[f"final_m{i}"])
    # right-padded position ids of the branch (cambrian_arch.py:582-584) restart at 0 for every sample
    assert pos[0, :5].tolist() == [0, 1, 2, 3, 4]


# ---------------------------------------------------------------------------------------------------------------
# SigLIP ViT and ConvNeXt trunks: the reference takes them from timm 0.9.16 via open_clip (not installed, cannot be
# fetched).  The restatements are pinned instead against the independent `transformers` implementations of the same
# published architectures with the weights mapped name by name — this fixes the block structure, the fused-qkv split,
# LN placement / eps, layer scale, stem / downsample arithmetic; what remains unpinned is only timm's choice of GELU
# flavour for the SigLIP MLP (a config field of the restatement and of the CUDA tower).
# ---------------------------------------------------------------------------------------------------------------
def test_oracle_siglip_matches_transformers_siglip_vision_model():
    from transformers import SiglipVisionConfig, SiglipVisionModel
    cfg = SiglipVisionConfig(hidden_size=96, intermediate_size=160, num_hidden_layers=2, num_attention_heads=4, image_size=56,
                             patch_size=14, layer_norm_eps=1e-6, hidden_act="gelu_pytorch_tanh")
    torch.manual_seed(0)
    m = SiglipVisionModel(cfg).eval()
    hf = m.state_dict()
    sd = {"patch_embed.proj.weight": hf["vision_model.embeddings.patch_embedding.weight"],
          "patch_embed.proj.bias": hf["vision_model.embeddings.patch_embedding.bias"],
          "pos_embed": hf["vision_model.embeddings.position_embedding.weight"][None],
          "norm.weight": hf["vision_model.post_layernorm.weight"], "norm.bias": hf["vision_model.post_layernorm.bias"]}
    for i in range(cfg.num_hidden_layers):
        h, q = f"vision_model.encoder.layers.{i}.", f"blocks.{i}."
        for a, b in (("layer_norm1", "norm1"), ("layer_norm2", "norm2"), ("self_attn.out_proj", "attn.proj"),
                     ("mlp.fc1", "mlp.fc1"), ("mlp.fc2", "mlp.fc2")):
            sd[q + b + ".weight"], sd[q + b + ".bias"] = hf[h + a + ".weight"], hf[h + a + ".bias"]
        sd[q + "attn.qkv.weight"] = torch.cat([hf[h + f"self_attn.{n}_proj.weight"] for n in "qkv"], 0)
        sd[q + "attn.qkv.bias"] = torch.cat([hf[h + f"self_attn.{n}_proj.bias"] for n in "qkv"], 0)
    x = torch.randn(2, 3, 56, 56)
    with torch.no_grad():
        want = m(pixel_values=x).last_hidden_state                        # post-layernorm tokens, no head
        got = O.siglip_vit(sd, dict(patch_size=14, num_attention_heads=4, num_hidden_layers=2, act="gelu_tanh"), x)
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5)


def test_oracle_convnext_matches_transformers_convnext_model():
    from transformers import ConvNextConfig, ConvNextModel
    depths, dims = [1, 1, 2, 1], [16, 32, 64, 128]
    cfg = ConvNextConfig(num_channels=3, patch_size=4, num_stages=4, hidden_sizes=dims, depths=depths, hidden_act="gelu",
                         layer_norm_eps=1e-6, layer_scale_init_value=0.5, drop_path_rate=0.0)
    torch.manual_seed(0)
    m = ConvNextModel(cfg).eval()
    hf = m.state_dict()
    sd = {"stem.0.weight": hf["embeddings.patch_embeddings.weight"], "stem.0.bias": hf["embeddings.patch_embeddings.bias"],
          "stem.1.weight": hf["embeddings.layernorm.weight"], "stem.1.bias": hf["embeddings.layernorm.bias"]}
    for s, depth in enumerate(depths):
        h, p = f"encoder.stages.{s}.", f"stages.{s}."
        if s > 0:
            sd[p + "downsample.0.weight"], sd[p + "downsample.0.bias"] = hf[h + "downsampling_layer.0.weight"], hf[h + "downsampling_layer.0.bias"]
            sd[p + "downsample.1.weight"], sd[p + "downsample.1.bias"] = hf[h + "downsampling_layer.1.weight"], hf[h + "downsampling_layer.1.bias"]
        for b in range(depth):
            hb, q = f"{h}layers.{b}.", f"{p}blocks.{b}."
            sd[q + "conv_dw.weight"], sd[q + "conv_dw.bias"] = hf[hb + "dwconv.weight"], hf[hb + "dwconv.bias"]
            sd[q + "norm.weight"], sd[q + "norm.bias"] = hf[hb + "layernorm.weight"], hf[hb + "layernorm.bias"]
            sd[q + "mlp.fc1.weight"], sd[q + "mlp.fc1.bias"] = hf[hb + "pwconv1.weight"], hf[hb + "pwconv1.bias"]
            sd[q + "mlp.fc2.weight"], sd[q + "mlp.fc2.bias"] = hf[hb + "pwconv2.weight"], hf[hb + "pwconv2.bias"]
            sd[q + "gamma"] = hf[hb + "layer_scale_parameter"]
    x = torch.randn(2, 3, 64, 64)
    with torch.no_grad():
        out = m(pixel_values=x, output_hidden_states=True)
        want = out.hidden_states[-1]                                       # last stage feature map [B, C, 2, 2]
        got = O.convnext_trunk(sd, dict(depths=depths, interp=4), x)       # 2 x 2 grid -> identity resize
    torch.testing.assert_close(got, want.flatten(2).transpose(1, 2), rtol=1e-4, atol=1e-5)
