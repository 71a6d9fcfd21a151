"""Generates the committed golden fixtures from the UNMODIFIED reference modules (run where the reference tree exists;
nothing else in the repository needs it).

    python tests/golden/make_golden.py            (--only-pins: just the pin_*.npz fixtures)

Weights are not stored: every parameter is regenerated from numpy's PCG64 stream (stable across numpy versions) by
`seeded_fill`, in state-dict order, so the fixtures stay a few hundred KB.  Each .npz holds the seeded inputs and the
reference's outputs for:
  sva_*.npz        VisionTokenSampler.forward (vision_sampler.py:407-419) — connector shape (q_dim 1024) and in-LLM
                   shape (q_dim 256), kv sizes with r > 1 and letter-box style masks; sva_sep*.npz: layer_type="sep"
  rearrange.npz    rearrange_vision_tower_features_train (cambrian_arch.py:271-287)
  collator.npz     prepare_image_info / get_padding_offset (train_fsdp.py:1039-1085) for several image sizes
  dynamic.npz      the off-XLA (inference) branch for non-square images: unmask_attention_mask / unpad_image /
                   rearrange_vision_tower_features_inference (cambrian_arch.py:203-330) and the whole
                   prepare_inputs_labels_for_multimodal dynamic path (:340-451, :493-609) run on a stub model that
                   holds reference modules (VisionTokenSampler, nn.Sequential projectors) under the reference's names
  pin_*.npz        what the reference modules compute in the oracle pins of tests/test_oracle_pin.py and
                   tests/test_host_logic_cpu.py: sep sampler output + sampled gradients, config 1 at full size, two query
                   groups through prepare_inputs_labels_for_multimodal, the mlp2x_gelu projector, state-dict layouts,
                   unmask_attention_mask / unpad_image on random sizes
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)


def seeded_fill(module_or_sd, seed):
    """Deterministic parameter values in state-dict order (shared by the generator and the tests)."""
    rng = np.random.default_rng(seed)
    sd = module_or_sd if isinstance(module_or_sd, dict) else module_or_sd.state_dict()
    out = {}
    for k, v in sd.items():
        a = rng.standard_normal(tuple(v.shape)).astype(np.float32)
        if v.dim() >= 2 and "pos_embed" not in k:
            a *= 0.03
        elif "pos_embed" in k:
            a *= 0.1
        elif k.endswith("weight"):      # LayerNorm scale
            a = 1.0 + 0.1 * a
        else:                            # biases
            a *= 0.1
        out[k] = torch.from_numpy(a)
    return out


def seeded_inputs(seed, n, q_dim, rs, mask_p=0.3):
    rng = np.random.default_rng(seed)
    queries = torch.from_numpy(rng.standard_normal((n, 1, q_dim)).astype(np.float32))
    ctx = torch.from_numpy(rng.standard_normal((n, 1, 1024)).astype(np.float32))
    feats = [torch.from_numpy(rng.standard_normal((n, r * r, 1024)).astype(np.float32)) for r in rs]
    masks = []
    for r in rs:
        m = rng.random((n, r * r)) > mask_p
        m[m.sum(1) == 0] = True
        masks.append(torch.from_numpy(m))
    return queries, ctx, feats, masks


SVA_CASES = {
    "sva_connector": dict(q_dim=1024, rs=[1, 1, 1, 1], layers=2, n=32, seed=11),
    "sva_connector_r4": dict(q_dim=1024, rs=[1, 1, 1, 4], layers=1, n=18, seed=12),
    "sva_inllm": dict(q_dim=256, rs=[1, 2, 1, 3], layers=1, n=32, seed=13),
}

# full-size cases (BASELINE config 1: 576 queries over 4 x 24 x 24 x 1024 grids, connector depth 3; the release grids
# [1,1,1,4]; one in-LLM layer at Llama-3-8B width).  Outputs are stored subsampled (rows 0::(4 * q_dim / 1024) as fp16) together with the
# fp32 row sums of ALL rows, so the fixtures stay small while every row is covered.
SVA_FULL_CASES = {
    "sva_config1": dict(q_dim=1024, rs=[1, 1, 1, 1], layers=3, n=576, seed=51),
    "sva_config1_r4": dict(q_dim=1024, rs=[1, 1, 1, 4], layers=3, n=576, seed=52),
    "sva_inllm_4096": dict(q_dim=4096, rs=[1, 1, 1, 4], layers=1, n=576, seed=53),
}

# layer_type="sep" (VisionAggregationLayer, vision_sampler.py:330-405): API surface no reference caller constructs; one
# case with attention towers (r > 1), MLP towers (r = 1) and masks, one single-tower case (no weight_mlp)
SVA_SEP_CASES = {
    "sva_sep": dict(q_dim=256, rs=[2, 1, 3, 1], layers=2, n=24, seed=61),
    "sva_sep_single": dict(q_dim=1024, rs=[2], layers=1, n=16, seed=62),
}

DYN = dict(sizes=[(800, 400), (336, 336), (200, 500)], q=4, tower_dims=[96, 80], tower_sides=[4, 8], H=128, vocab=200,
           seed=41)


def dynamic_stub(arch, vs):
    """A CambrianMetaForCausalLM whose get_model() holds reference modules under the reference's attribute names; the
    'towers' are identities so the seeded tower features are the images."""
    import torch.nn as nn
    d = DYN

    class Inner(nn.Module):
        def __init__(self):
            super().__init__()
            for i, c in enumerate(d["tower_dims"]):
                setattr(self, f"mm_projector_aux_{i}", nn.Sequential(nn.Linear(c, 1024), nn.GELU(), nn.Linear(1024, 1024),
                                                                     nn.LayerNorm(1024)))
            self.vision_sampler_0 = vs.VisionTokenSampler(1024, 1024, [1024, 1024], [s // d["q"] for s in d["tower_sides"]],
                                                          1024, 2)
            self.mm_projector = nn.Sequential(nn.Linear(1024, d["H"]), nn.GELU(), nn.Linear(d["H"], d["H"]))
            self.embed_tokens = nn.Embedding(d["vocab"], d["H"])
            self.vision_query = nn.Parameter(torch.zeros(1, 1024))
            self.image_newline = nn.Parameter(torch.zeros(d["H"]))
            self.config = type("C", (), dict(image_token_len=d["q"] ** 2, query_num_list=[d["q"] ** 2],
                                             mm_projector_type="sva"))()

        def get_vision_tower_aux_list(self):
            return [lambda x: x for _ in d["tower_dims"]]

    class Top(nn.Module, arch.CambrianMetaForCausalLM):
        def __init__(self):
            nn.Module.__init__(self)
            self.model = Inner()
            self.config = self.model.config
            self.device = torch.device("cpu")

        def get_model(self):
            return self.model

    return Top().eval()


def dynamic_inputs():
    d = DYN
    rng = np.random.default_rng(d["seed"])
    B = len(d["sizes"])
    feats = [torch.from_numpy(rng.standard_normal((B, s * s, c)).astype(np.float32))
             for s, c in zip(d["tower_sides"], d["tower_dims"])]
    L = 24
    ids = torch.from_numpy(rng.integers(3, d["vocab"], size=(B, L)))
    for b, p0 in enumerate((5, 5, 5)):
        ids[b, p0] = -200
    attn = torch.ones(B, L, dtype=torch.bool)
    attn[1, 20:] = False
    attn[2, 15:] = False
    labels = ids.clone()
    return feats, ids, attn, labels


def make_dynamic(arch, vs):
    d = DYN
    top = dynamic_stub(arch, vs)
    top.load_state_dict(seeded_fill(top, d["seed"] + 1))
    feats, ids, attn, labels = dynamic_inputs()
    recs = {}
    xla_flag = arch.IS_XLA_AVAILABLE
    arch.IS_XLA_AVAILABLE = False           # the shim's torch_xla stub makes the import succeed; take the GPU/CPU branch
    with torch.no_grad():
        for unpad in (False, True):
            fr, mr = top.rearrange_vision_tower_features_inference(feats, d["q"], d["sizes"], unpad=unpad)
            for i, (f, m) in enumerate(zip(fr, mr)):
                recs[f"re{int(unpad)}_f{i}"] = f.numpy().astype(np.float16)
                recs[f"re{int(unpad)}_m{i}"] = m.numpy()
        out = top.prepare_inputs_labels_for_multimodal(ids, None, attn, None, labels, feats, None, d["sizes"])
    arch.IS_XLA_AVAILABLE = xla_flag
    (_, pos, am, _, emb, lab, ff, mf, fs, ctx) = out
    recs.update(emb=emb.numpy(), labels=lab.numpy(), attn=am.numpy(), final_size=np.array(fs),
                ctx=ctx.numpy().astype(np.float16))
    assert pos is None                                  # position_ids stay None when none were passed (:596-597)
    for i, (f, m) in enumerate(zip(ff, mf)):
        recs[f"final_f{i}"] = f.numpy().astype(np.float16)
        recs[f"final_m{i}"] = m.numpy()
    for (w, h) in [(640, 480), (480, 640), (1000, 200), (123, 457), (336, 336)]:
        for side in (24, 27, 96):
            recs[f"unmask_{w}x{h}_{side}"] = arch.unmask_attention_mask(torch.ones(1, side, side, dtype=torch.bool), (w, h)).numpy()
            recs[f"unpad_{w}x{h}_{side}"] = np.array(arch.unpad_image(torch.zeros(1, side, side, 1), (w, h)).shape[1:3])
    # parameter names / shapes in state-dict order, so the tests can regenerate the weights without the reference
    recs["sd_keys"] = np.array(list(top.state_dict().keys()))
    recs["sd_shapes"] = np.array([",".join(map(str, v.shape)) for v in top.state_dict().values()])
    np.savez_compressed(os.path.join(HERE, "dynamic.npz"), **recs)
    print("dynamic", len(recs), "final sizes", fs, "embeds", tuple(emb.shape))


def make_full(vs):
    for name, c in SVA_FULL_CASES.items():
        T = len(c["rs"])
        m = vs.VisionTokenSampler(c["q_dim"], 1024, [1024] * T, c["rs"], 1024, c["layers"]).eval()
        m.load_state_dict(seeded_fill(m, c["seed"]))
        queries, ctx, feats, masks = seeded_inputs(c["seed"] + 100, c["n"], c["q_dim"], c["rs"])
        with torch.no_grad():
            out = m(queries, ctx, *feats, *masks)[:, 0]
        stride = 4 * c["q_dim"] // 1024
        np.savez_compressed(os.path.join(HERE, name + ".npz"), rows=out[0::stride].numpy().astype(np.float16),
                            rowsum=out.sum(1).numpy().astype(np.float32), absmean=np.float32(out.abs().mean()))
        print(name, tuple(out.shape), float(out.abs().mean()))


def make_sep(vs):
    for name, c in SVA_SEP_CASES.items():
        T = len(c["rs"])
        m = vs.VisionTokenSampler(c["q_dim"], 1024, [1024] * T, c["rs"], 1024, c["layers"], layer_type="sep").eval()
        sd = seeded_fill(m, c["seed"])
        m.load_state_dict(sd)
        queries, ctx, feats, masks = seeded_inputs(c["seed"] + 100, c["n"], c["q_dim"], c["rs"])
        with torch.no_grad():
            out = m(queries, ctx, *feats, *masks)
        # parameter names / shapes in state-dict order, so the tests regenerate the weights without the reference
        np.savez_compressed(os.path.join(HERE, name + ".npz"), out=out.numpy(), sd_keys=np.array(list(sd.keys())),
                            sd_shapes=np.array([",".join(map(str, v.shape)) for v in sd.values()]))
        print(name, tuple(out.shape), float(out.abs().mean()))


# ------------------------------------------------------------------------------------------------------------------
# pins of the oracle against the reference modules: what the reference computed, stored so the comparison needs no
# reference tree (tests/test_oracle_pin.py, tests/test_host_logic_cpu.py)
# ------------------------------------------------------------------------------------------------------------------
SEP_LIVE_CASES = [([1, 2, 1], 256, 2), ([3], 512, 1), ([1], 1024, 1)]
GRAD_SAMPLES = 32
OUT_SAMPLES = 256


def sd_layout(sd):
    """parameter names / shapes in state-dict order: enough to regenerate seeded_fill weights without the module"""
    return dict(sd_keys=np.array(list(sd.keys())), sd_shapes=np.array([",".join(map(str, v.shape)) for v in sd.values()]))


def sd_from_layout(z, seed):
    shapes = {str(k): tuple(int(x) for x in str(sh).split(",") if x) for k, sh in zip(z["sd_keys"], z["sd_shapes"])}
    return seeded_fill({k: torch.empty(v) for k, v in shapes.items()}, seed)


def grad_sample_index(numels, seed=74):
    """fixed sample of GRAD_SAMPLES flat indices per gradient tensor"""
    rng = np.random.default_rng(seed)
    return [rng.integers(0, n, size=min(GRAD_SAMPLES, n)) for n in numels]


def flat_sample(t, k=OUT_SAMPLES, seed=75):
    """a fixed seeded sample of k elements of t (all of them if t is smaller): keeps the pin fixtures a few KB"""
    n = t.numel()
    if n <= k:
        return t.reshape(-1)
    idx = np.random.default_rng(seed).integers(0, n, size=k)
    return t.reshape(-1)[torch.from_numpy(idx)]


def sep_live_dy(shape):
    return torch.from_numpy(np.random.default_rng(73).standard_normal(tuple(shape)).astype(np.float32))


def config1_inputs(rs, seed):
    from oracle import cambrian_oracle as O
    g = torch.Generator().manual_seed(seed)
    feats = [torch.randn(1, (24 * r) ** 2, 1024, generator=g) for r in rs]
    query = (torch.randn(1, 1024, generator=g) / 32).view(1, 1, 1, -1).expand(1, 576, -1, -1).flatten(0, 1)
    ctx = feats[0].mean(1).view(1, 1, 1, -1).expand(-1, 576, 1, -1).flatten(0, 1)
    fw = [O.window_rearrange(f, 24) for f in feats]
    masks = [torch.rand(576, r * r, generator=g) > 0.2 for r in rs]
    for mk in masks:
        mk[mk.sum(1) == 0] = True
    return query, ctx, fw, masks


TWO_GROUPS = dict(H=64, q=4, sides=[4, 8], dims=[48, 40], B=2, seed=91)


def two_groups_inputs():
    c = TWO_GROUPS
    g = torch.Generator().manual_seed(c["seed"] + 1)
    q, B = c["q"], c["B"]
    feats = [torch.randn(B, s * s, d, generator=g) for s, d in zip(c["sides"], c["dims"])]
    masks = [torch.ones(B * q * q, (s // q) ** 2, dtype=torch.bool) for s in c["sides"]]
    masks[1][::5, 1] = False
    span = q * (q + 1)
    ids = torch.randint(3, 100, (B, 5 + span + 6), generator=g)
    ids[:, 5] = -200
    ids[:, 6:5 + span] = 0
    return feats, masks, ids


def projector_input():
    return torch.from_numpy(np.random.default_rng(96).standard_normal((3, 7, 96)).astype(np.float32))


def unpad_cases():
    rng = np.random.default_rng(5)
    cases = []
    for _ in range(300):
        w, h = int(rng.integers(16, 4000)), int(rng.integers(16, 4000))
        cases.append((w, h, int(rng.choice([16, 24, 27, 48, 96]))))
    return cases


def make_pins(vs, arch):
    import torch.nn as nn
    from oracle import ref_shim
    # layer_type="sep": output and every gradient of the reference module (gradients as a fixed sample + their norms)
    recs = {}
    for i, (rs, q_dim, layers) in enumerate(SEP_LIVE_CASES):
        m = vs.VisionTokenSampler(q_dim, 1024, [1024] * len(rs), rs, 1024, layers, layer_type="sep")
        sd = seeded_fill(m, 71)
        m.load_state_dict(sd)
        queries, ctx, feats, masks = seeded_inputs(72, 10, q_dim, rs)
        queries.requires_grad_()
        ref = m(queries, ctx, *feats, *masks)
        params = list(m.named_parameters())
        grads = torch.autograd.grad(ref, [queries] + [p for _, p in params], sep_live_dy(ref.shape))
        idx = grad_sample_index([g.numel() for g in grads])
        recs.update({f"c{i}_" + k: v for k, v in sd_layout(sd).items()})
        recs[f"c{i}_names"] = np.array([k for k, _ in params])
        recs[f"c{i}_out"] = flat_sample(ref.detach()).numpy()
        recs[f"c{i}_outsum"] = ref.detach().sum(-1).numpy()
        recs[f"c{i}_gsample"] = np.concatenate([g.reshape(-1)[torch.from_numpy(ix)].numpy() for g, ix in zip(grads, idx)])
        recs[f"c{i}_gnorm"] = np.array([g.double().norm().item() for g in grads])
    np.savez_compressed(os.path.join(HERE, "pin_sep_fwd_bwd.npz"), **recs)
    # BASELINE config 1 at full size, random masks: a fixed sample of the output + all row sums
    recs = {}
    for j, rs in enumerate(([1, 1, 1, 1], [1, 1, 1, 4])):
        m = vs.VisionTokenSampler(1024, 1024, [1024] * 4, rs, 1024, 3).eval()
        sd = seeded_fill(m, 81 + j)
        m.load_state_dict(sd)
        query, ctx, fw, masks = config1_inputs(rs, 82 + j)
        with torch.no_grad():
            ref = m(query, ctx, *fw, *masks)[:, 0]
        recs.update({f"r{j}_" + k: v for k, v in sd_layout(sd).items()})
        recs[f"r{j}_sample"] = flat_sample(ref, 512).numpy()
        recs[f"r{j}_rowsum"] = ref.sum(1).numpy()
    np.savez_compressed(os.path.join(HERE, "pin_config1.npz"), **recs)
    # two query groups through the reference's static-branch prepare_inputs_labels_for_multimodal
    c = TWO_GROUPS
    H, q, sides, dims = c["H"], c["q"], c["sides"], c["dims"]

    class Inner(nn.Module):
        def __init__(self):
            super().__init__()
            for i, d in enumerate(dims):
                setattr(self, f"mm_projector_aux_{i}", nn.Sequential(nn.Linear(d, 1024), nn.GELU(), nn.Linear(1024, 1024),
                                                                     nn.LayerNorm(1024)))
            self.vision_sampler_0 = vs.VisionTokenSampler(1024, 1024, [1024, 1024], [s // 4 for s in sides], 1024, 2)
            self.vision_sampler_1 = vs.VisionTokenSampler(1024, 1024, [1024, 1024], [s // 2 for s in sides], 1024, 2)
            self.mm_projector = nn.Sequential(nn.Linear(2048, H), nn.GELU(), nn.Linear(H, H))
            self.embed_tokens = nn.Embedding(100, H)
            self.vision_query = nn.Parameter(torch.zeros(2, 1024))
            self.image_newline = nn.Parameter(torch.zeros(H))
            self.config = type("C", (), dict(image_token_len=q * q, query_num_list=[q * q, 4], mm_projector_type="sva"))()

        def get_vision_tower_aux_list(self):
            return [lambda x: x for _ in dims]

    class Top(nn.Module, arch.CambrianMetaForCausalLM):
        def __init__(self):
            nn.Module.__init__(self)
            self.model = Inner()
            self.config = self.model.config
            self.device = torch.device("cpu")

        def get_model(self):
            return self.model

    top = Top().eval()
    sd = seeded_fill(top.model, c["seed"])
    top.model.load_state_dict(sd)
    feats, masks, ids = two_groups_inputs()
    flag = arch.IS_XLA_AVAILABLE
    arch.IS_XLA_AVAILABLE = True
    try:
        with torch.no_grad():
            out = top.prepare_inputs_labels_for_multimodal(ids, None, None, None, None, feats, masks, None)
    finally:
        arch.IS_XLA_AVAILABLE = flag
    recs = dict(sd_layout(sd), emb=flat_sample(out[4]).numpy(), embsum=out[4].sum(-1).numpy())
    for i, f in enumerate(out[6]):          # window-rearranged aux features handed to the in-LLM SVA layers (sampled)
        recs[f"feat_w{i}"] = flat_sample(f).numpy()
    np.savez_compressed(os.path.join(HERE, "pin_two_groups.npz"), **recs)
    # mlp2x_gelu projector
    pb = ref_shim.ref_module("cambrian.model.multimodal_projector.builder")
    from types import SimpleNamespace
    proj = pb.build_vision_projector(SimpleNamespace(mm_projector_type="mlp2x_gelu", mm_hidden_size=96, hidden_size=64)).eval()
    sd = seeded_fill(proj, 95)
    proj.load_state_dict(sd)
    with torch.no_grad():
        y = proj(projector_input())
    np.savez_compressed(os.path.join(HERE, "pin_projector.npz"), **sd_layout(sd), out=flat_sample(y).numpy())
    # state-dict layouts of the reference samplers
    recs = {}
    for i, args in enumerate([(1024, 1024, [1024] * 4, [1, 1, 1, 1], 1024, 3), (256, 1024, [1024] * 3, [1, 2, 3], 1024, 1)]):
        recs[f"keys{i}"] = np.array(list(vs.VisionTokenSampler(*args).state_dict()))
    recs.update({"sep_" + k: v for k, v in sd_layout(vs.VisionTokenSampler(256, 1024, [1024] * 3, [2, 1, 3], 1024, 2,
                                                                          layer_type="sep").state_dict()).items()})
    np.savez_compressed(os.path.join(HERE, "pin_state_dicts.npz"), **recs)
    # unmask_attention_mask / unpad_image on random image sizes: the mask (packed bits) and the crop unpad_image keeps
    masks, crops = [], []
    for (w, h, side) in unpad_cases():
        masks.append(np.packbits(arch.unmask_attention_mask(torch.ones(1, side, side, dtype=torch.bool), (w, h)).numpy()))
        t = torch.arange(side * side).view(1, side, side, 1)
        u = arch.unpad_image(t, (w, h))
        if 0 in u.shape:
            crops.append((-1, -1, -1, -1))
        else:
            v = u[0, :, :, 0]
            crops.append((int(v[0, 0]) // side, int(v[-1, 0]) // side + 1, int(v[0, 0]) % side, int(v[0, -1]) % side + 1))
    np.savez_compressed(os.path.join(HERE, "pin_unpad.npz"), masks=np.concatenate(masks), mask_lens=np.array([len(m) for m in masks]),
                        crops=np.array(crops))
    print("pins written")


def main():
    from oracle import ref_shim
    vs = ref_shim.ref_module("cambrian.model.vision_sampler")
    if "--only-pins" in sys.argv:
        make_pins(vs, ref_shim.ref_module("cambrian.model.cambrian_arch"))
        return
    if "--only-sep" in sys.argv:
        make_sep(vs)
        return
    arch = ref_shim.ref_module("cambrian.model.cambrian_arch")
    if "--only-full" in sys.argv:
        make_full(vs)
        return
    make_full(vs)
    make_sep(vs)
    for name, c in SVA_CASES.items():
        T = len(c["rs"])
        m = vs.VisionTokenSampler(c["q_dim"], 1024, [1024] * T, c["rs"], 1024, c["layers"]).eval()
        m.load_state_dict(seeded_fill(m, c["seed"]))
        queries, ctx, feats, masks = seeded_inputs(c["seed"] + 100, c["n"], c["q_dim"], c["rs"])
        with torch.no_grad():
            out = m(queries, ctx, *feats, *masks)
        np.savez_compressed(os.path.join(HERE, name + ".npz"), out=out.numpy())
        print(name, tuple(out.shape), float(out.abs().mean()))

    # window rearrange
    rng = np.random.default_rng(21)
    feat = torch.from_numpy(rng.standard_normal((2, 64, 8)).astype(np.float32))   # 8x8 grid, q_side 4 -> r = 2
    mask = torch.from_numpy(rng.random((2 * 16, 4)) > 0.5)

    class _Dummy(arch.CambrianMetaForCausalLM):
        def get_model(self):
            return None
    fr, mr = _Dummy().rearrange_vision_tower_features_train([feat], [mask], 4)
    np.savez_compressed(os.path.join(HERE, "rearrange.npz"), feat=feat.numpy(), out=fr[0].numpy(), mask=mr[0].numpy())

    # collator geometry (train_fsdp.py imports torch_xla etc. at module scope -> stubbed by the shim)
    # The TPU harness module cannot be imported (torch_xla, transformers-4.37 trainer symbols), so the three pure
    # functions are lifted out of the reference file by name with `ast` and executed unmodified.
    import ast
    import types
    src = open("/root/reference/cambrian/train/train_fsdp.py").read()
    tree = ast.parse(src)
    want = {"get_padding_offset", "prepare_image_info", "prepare_multimodal_data"}
    code = "\n\n".join(ast.get_source_segment(src, n) for n in tree.body
                       if isinstance(n, ast.FunctionDef) and n.name in want)
    tf = types.SimpleNamespace()
    ns_ = {"torch": torch, "IMAGE_TOKEN_INDEX": -200, "IGNORE_INDEX": -100}
    exec(compile(code, "train_fsdp_extract", "exec"), ns_)
    tf.prepare_image_info = ns_["prepare_image_info"]
    tf.prepare_multimodal_data = ns_["prepare_multimodal_data"]
    sizes = [(640, 480), (480, 640), (336, 336), (1000, 200), (123, 457)]
    recs = {}
    for (w, h) in sizes:
        for tok in (576, 9216):
            for nl in (False, True):
                if nl and tok != 576:
                    continue
                am, pid = tf.prepare_image_info((w, h), tok, newline=nl)
                recs[f"mask_{w}x{h}_{tok}_{int(nl)}"] = am.numpy()
                recs[f"pos_{w}x{h}_{tok}_{int(nl)}"] = pid.numpy()
    # full collator expansion (train_fsdp.py:1089-1165) on a seeded batch with one image per sample
    rng = np.random.default_rng(31)
    B, L = 3, 40
    ids = torch.from_numpy(rng.integers(3, 1000, size=(B, L)))
    for b, p0 in enumerate((5, 9, 0)):
        ids[b, p0] = -200
    labels = ids.clone()
    attn = torch.ones(B, L, dtype=torch.bool)
    attn[2, 30:] = False
    im_sizes = [(640, 480), (336, 336), (200, 1000)]
    out = tf.prepare_multimodal_data(ids, labels, attn, im_sizes, image_token_len=16,
                                     image_aux_token_len_list=[16, 64], max_length=64)
    recs.update(cm_ids_in=ids.numpy(), cm_attn_in=attn.numpy(), cm_ids=out[0].numpy(), cm_labels=out[1].numpy(),
                cm_attn=out[2].numpy(), cm_pos=out[3].numpy(), cm_aux0=out[4][0].numpy(), cm_aux1=out[4][1].numpy())
    np.savez_compressed(os.path.join(HERE, "collator.npz"), **recs)
    print("collator", len(recs))
    make_dynamic(arch, vs)
    make_pins(vs, arch)


if __name__ == "__main__":
    main()
