"""The four Cambrian-1 vision towers, forward-only on hand-written sm_90a kernels.

Mirrors the reference wrappers (cambrian/model/multimodal_encoder/{base,clip,siglip,dino,clip_convnext}_encoder.py):
same class names, name parsing (`-res{N}`, `-interp{N}`), properties and `forward(images) -> [B, N, C]`, and the
parameters keep the names of the third-party modules the reference delegates to (HF CLIPVisionModel / Dinov2Model,
timm VisionTransformer / ConvNeXt), so their state dicts load with `load_state_dict`.

The towers are frozen in every released Cambrian recipe (train_fsdp.py:1655-1659, base_encoder.py:43); only the
forward is implemented and `unfreeze_mm_vision_tower=True` raises NotImplementedError.

There is no network in this environment: `load_model()` builds the architecture with random weights unless a
state dict is supplied (`load_model(state_dict=...)`).
"""
from __future__ import annotations

import math
import re

import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import ops


# ------------------------------------------------------------------------------------------------------------------
# image processor (minimal stand-in for the HF processors the reference instantiates)
# ------------------------------------------------------------------------------------------------------------------
class SimpleImageProcessor:
    """Resize (bicubic, shortest edge) + centre crop + normalise.  Provides the attributes mm_utils.process_images
    uses: crop_size['height'], image_mean, preprocess(img, return_tensors='pt')['pixel_values'] (mm_utils.py:186-199)."""

    def __init__(self, size, mean, std):
        self.crop_size = {"height": size, "width": size}
        self.size = {"shortest_edge": size}
        self.image_mean = list(mean)
        self.image_std = list(std)

    def preprocess(self, image, return_tensors="pt"):
        import numpy as np
        if not torch.is_tensor(image):
            image = torch.from_numpy(np.asarray(image.convert("RGB"))).permute(2, 0, 1)
        x = image.float()[None] / 255.0
        s = self.crop_size["height"]
        h, w = x.shape[-2:]
        sc = s / min(h, w)
        nh, nw = max(s, round(h * sc)), max(s, round(w * sc))
        x = F.interpolate(x, size=(nh, nw), mode="bicubic", align_corners=False).clamp(0, 1)
        t, l = (nh - s) // 2, (nw - s) // 2
        x = x[..., t:t + s, l:l + s]
        mean = torch.tensor(self.image_mean).view(1, 3, 1, 1)
        std = torch.tensor(self.image_std).view(1, 3, 1, 1)
        return {"pixel_values": (x - mean) / std}


CLIP_MEAN, CLIP_STD = (0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711)
IMNET_MEAN, IMNET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def _parse_res_interp(name: str):
    res = interp = None
    base = name
    for part in name.split("-"):
        if re.fullmatch(r"res\d+", part):
            res = int(part[3:])
            base = base.replace("-" + part, "")
        elif re.fullmatch(r"interp\d+", part):
            interp = int(part[6:])
            base = base.replace("-" + part, "")
    return base, res, interp


class BaseVisionTower(nn.Module):
    """base_encoder.py:33-134."""

    def __init__(self, vision_tower_name, args, delay_load=False):
        super().__init__()
        self.is_loaded = False
        self.args = args
        self.vision_tower_name = vision_tower_name
        self.select_layer = getattr(args, "mm_vision_select_layer", -2)
        self.select_feature = getattr(args, "mm_vision_select_feature", "patch")
        self.unfreeze_mm_vision_tower = getattr(args, "unfreeze_mm_vision_tower", False)
        self.delay_load = delay_load
        self._interp_size = None
        self._gpu = None  # prepared (fused / padded / permuted) bf16 weights, built lazily

    def _check_frozen(self):
        if self.unfreeze_mm_vision_tower:
            raise NotImplementedError("cambrian_b200 towers are forward-only (frozen), as in every released Cambrian recipe")

    def load_state_dict(self, *a, **k):
        self._gpu = None
        return super().load_state_dict(*a, **k)

    def _apply(self, fn, *a, **k):
        self._gpu = None
        return super()._apply(fn, *a, **k)

    def forward(self, images):
        self._check_frozen()
        if type(images) is list:
            return [self._forward(im.unsqueeze(0)) for im in images]
        return self._forward(images)

    @torch.no_grad()
    def _forward(self, images):
        if not self.is_loaded:
            raise RuntimeError(f"{type(self).__name__}: call load_model() first")
        if not images.is_cuda:
            raise RuntimeError("cambrian_b200 towers need CUDA inputs (no CPU fallback)")
        with ops.nvtx(f"tower.{type(self).__name__}"):
            return self._run(images.to(device=self.device, dtype=torch.bfloat16)).to(images.dtype)

    @property
    def dummy_feature(self):
        return torch.zeros(1, self.hidden_size, device=self.device, dtype=self.dtype)

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    @property
    def config(self):
        return self.cfg

    @property
    def hidden_size(self):
        return self._hidden_size

    @property
    def image_size(self):
        return self._image_size

    @property
    def patch_size(self):
        return self._patch_size

    @property
    def num_patches_per_side(self):
        if self._interp_size is not None:
            return int(self._interp_size ** 0.5)
        return self._image_size // self._patch_size

    @property
    def num_patches(self):
        if self._interp_size is not None:
            return self._interp_size
        return self.num_patches_per_side ** 2

    def _finish_tokens(self, x, grid, skip_cls):
        """Drop CLS and bilinearly resize the token grid to the interp size (fp32 interpolation, align_corners=False:
        clip_encoder.py:70-96, siglip_encoder.py:67-93, dino_encoder.py:128-154).  Also makes the result contiguous."""
        t = grid if self._interp_size is None else int(self._interp_size ** 0.5)
        src = x[:, 1:] if skip_cls else x
        return ops.bilinear(src, grid, grid, t, t, in_bs=x.stride(0))


def _p(*shape, std=0.02):
    return nn.Parameter(torch.randn(*shape) * std)


def _pad_cols(w2d, mult=8):
    k = w2d.shape[1]
    kp = (k + mult - 1) // mult * mult
    if kp == k:
        return w2d.contiguous()
    out = torch.zeros(w2d.shape[0], kp, dtype=w2d.dtype, device=w2d.device)
    out[:, :k] = w2d
    return out


def _vit_blocks(x, blocks, heads, act, eps):
    """Pre-LN transformer encoder blocks: x [B, T, D] bf16 (contiguous).  Each block dict has ln1_w/b, qkv_w/b (fused),
    proj_w/b, ln2_w/b, fc1_w/b, fc2_w/b and optional ls1 / ls2 (LayerScale)."""
    B, T, D = x.shape
    hd = D // heads
    x2 = x.reshape(B * T, D)
    for blk in blocks:
        h = ops.layernorm_fwd(x2, blk["ln1_w"], blk["ln1_b"], eps)
        qkv = ops.gemm(h, blk["qkv_w"], bias=blk["qkv_b"]).view(B, T, 3, heads, hd)
        a = ops.attn_fwd(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], causal=False)
        x2 = ops.gemm(a.view(B * T, D), blk["proj_w"], bias=blk["proj_b"], colscale=blk.get("ls1"), residual=x2)
        h = ops.layernorm_fwd(x2, blk["ln2_w"], blk["ln2_b"], eps)
        if "win_w" in blk:   # DINOv2-giant: SwiGLU FFN (HF Dinov2SwiGLUFFN: chunk(weights_in(x)) -> silu(x1) * x2 -> weights_out)
            gu = ops.gemm(h, blk["win_w"], bias=blk["win_b"])
            F_ = gu.shape[1] // 2
            m = ops.swiglu_fwd(gu[:, :F_], gu[:, F_:])
        else:
            m = ops.gemm(h, blk["fc1_w"], bias=blk["fc1_b"], act=act)
        x2 = ops.gemm(m, blk["fc2_w"], bias=blk["fc2_b"], colscale=blk.get("ls2"), residual=x2)
    return x2.view(B, T, D)


# ------------------------------------------------------------------------------------------------------------------
# A1 — OpenAI CLIP ViT-L/14@336  (clip_encoder.py; HF CLIPVisionModel parameter names)
# ------------------------------------------------------------------------------------------------------------------
class ClipVisionTower(BaseVisionTower):
    DEFAULT = dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16,
                   patch_size=14, image_size=336, layer_norm_eps=1e-5)

    def __init__(self, vision_tower, args, delay_load=False):
        super().__init__(vision_tower, args, delay_load)
        base, res, interp = _parse_res_interp(vision_tower)
        self.vision_tower_name = base
        self._interp_size = interp
        self.cfg = dict(self.DEFAULT, **getattr(args, "clip_config_overrides", {}) or {})
        self._image_size = res if res is not None else self.cfg["image_size"]
        self._patch_size = self.cfg["patch_size"]
        self._hidden_size = self.cfg["hidden_size"]
        if not delay_load:
            self.load_model()

    def load_model(self, device_map=None, state_dict=None):
        c = self.cfg
        D, I, L, ps = c["hidden_size"], c["intermediate_size"], c["num_hidden_layers"], c["patch_size"]
        n_pos = (self._image_size // ps) ** 2 + 1
        vm = nn.Module()
        vm.embeddings = nn.Module()
        vm.embeddings.class_embedding = _p(D)
        vm.embeddings.patch_embedding = nn.Conv2d(3, D, ps, ps, bias=False)
        vm.embeddings.position_embedding = nn.Embedding(n_pos, D)
        vm.pre_layrnorm = nn.LayerNorm(D, eps=c["layer_norm_eps"])
        vm.encoder = nn.Module()
        layers = []
        for _ in range(L):
            l = nn.Module()
            l.self_attn = nn.Module()
            for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
                setattr(l.self_attn, n, nn.Linear(D, D))
            l.layer_norm1 = nn.LayerNorm(D, eps=c["layer_norm_eps"])
            l.mlp = nn.Module()
            l.mlp.fc1 = nn.Linear(D, I)
            l.mlp.fc2 = nn.Linear(I, D)
            l.layer_norm2 = nn.LayerNorm(D, eps=c["layer_norm_eps"])
            layers.append(l)
        vm.encoder.layers = nn.ModuleList(layers)
        vm.post_layernorm = nn.LayerNorm(D, eps=c["layer_norm_eps"])
        self.vision_tower = nn.Module()
        self.vision_tower.vision_model = vm
        if state_dict is not None:
            self.vision_tower.load_state_dict(state_dict, strict=False)
        self.image_processor = SimpleImageProcessor(self._image_size, CLIP_MEAN, CLIP_STD)
        self.vision_tower.requires_grad_(False)
        self.is_loaded = True
        self._gpu = None

    def _prepare(self):
        vm = self.vision_tower.vision_model
        c = self.cfg
        g = dict(patch_w=_pad_cols(vm.embeddings.patch_embedding.weight.flatten(1)),
                 cls=vm.embeddings.class_embedding.contiguous(), pos=vm.embeddings.position_embedding.weight.contiguous(),
                 pre_w=vm.pre_layrnorm.weight, pre_b=vm.pre_layrnorm.bias, blocks=[])
        n_run = c["num_hidden_layers"] + 1 + self.select_layer if self.select_layer < 0 else self.select_layer
        for l in vm.encoder.layers[:n_run]:  # hidden_states[select_layer]: later layers are never needed
            a = l.self_attn
            g["blocks"].append(dict(
                ln1_w=l.layer_norm1.weight, ln1_b=l.layer_norm1.bias,
                qkv_w=torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], 0).contiguous(),
                qkv_b=torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias], 0).contiguous(),
                proj_w=a.out_proj.weight, proj_b=a.out_proj.bias, ln2_w=l.layer_norm2.weight, ln2_b=l.layer_norm2.bias,
                fc1_w=l.mlp.fc1.weight, fc1_b=l.mlp.fc1.bias, fc2_w=l.mlp.fc2.weight, fc2_b=l.mlp.fc2.bias))
        self._gpu = g

    def _run(self, images):
        if self._gpu is None:
            self._prepare()
        g, c = self._gpu, self.cfg
        B = images.shape[0]
        grid = images.shape[-1] // c["patch_size"]
        patches = ops.gemm(ops.patchify_nchw(images, c["patch_size"]), g["patch_w"]).view(B, grid * grid, -1)
        x = ops.add_pos_tokens(patches, g["cls"], g["pos"])
        x = ops.layernorm_fwd(x, g["pre_w"], g["pre_b"], c["layer_norm_eps"])
        x = _vit_blocks(x, g["blocks"], c["num_attention_heads"], "quick_gelu", c["layer_norm_eps"])
        if self.select_feature not in ("patch", "cls_patch"):
            raise ValueError(f"Unexpected select feature: {self.select_feature}")
        if self.select_feature == "cls_patch":
            return x
        return self._finish_tokens(x, grid, skip_cls=True)


# ------------------------------------------------------------------------------------------------------------------
# A3 — DINOv2 ViT-L/14  (dino_encoder.py; HF Dinov2Model parameter names)
# ------------------------------------------------------------------------------------------------------------------
class DinoVisionTower(BaseVisionTower):
    CONFIGS = {
        "facebook/dinov2-large": dict(hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, mlp_ratio=4),
        "facebook/dinov2-base": dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, mlp_ratio=4),
        "facebook/dinov2-small": dict(hidden_size=384, num_hidden_layers=12, num_attention_heads=6, mlp_ratio=4),
        # the release tower (scripts/cambrian/finetune_cambrian_8b.sh:17-18: facebook/dinov2-giant-res378): SwiGLU FFN
        "facebook/dinov2-giant": dict(hidden_size=1536, num_hidden_layers=40, num_attention_heads=24, mlp_ratio=4,
                                      swiglu=True),
    }

    def __init__(self, vision_tower, args, delay_load=False):
        super().__init__(vision_tower, args, delay_load)
        base, res, interp = _parse_res_interp(vision_tower)
        if "dinov2-giant-imagenet1k" in base:
            raise NotImplementedError("facebook/dinov2-giant-imagenet1k-1-layer (classifier checkpoint) is unused by Cambrian-1")
        key = next((k for k in self.CONFIGS if base.startswith(k)), None)
        if key is None:
            raise ValueError(f"Unknown vision tower: {vision_tower}")
        self.vision_tower_name = key
        self._interp_size = interp
        self.cfg = dict(self.CONFIGS[key], patch_size=14, image_size=518, layer_norm_eps=1e-6)
        self.cfg.update(getattr(args, "dino_config_overrides", {}) or {})
        self._image_size = res if res is not None else 518
        self._patch_size = 14
        self._hidden_size = self.cfg["hidden_size"]
        if not delay_load:
            self.load_model()

    def load_model(self, device_map=None, state_dict=None):
        c = self.cfg
        D, L = c["hidden_size"], c["num_hidden_layers"]
        I = D * c["mlp_ratio"]
        vt = nn.Module()
        vt.embeddings = nn.Module()
        vt.embeddings.cls_token = _p(1, 1, D)
        vt.embeddings.mask_token = nn.Parameter(torch.zeros(1, D))
        vt.embeddings.position_embeddings = _p(1, (518 // 14) ** 2 + 1, D)
        vt.embeddings.patch_embeddings = nn.Module()
        vt.embeddings.patch_embeddings.projection = nn.Conv2d(3, D, 14, 14)
        vt.encoder = nn.Module()
        layers = []
        for _ in range(L):
            l = nn.Module()
            l.norm1 = nn.LayerNorm(D, eps=1e-6)
            l.attention = nn.Module()
            l.attention.attention = nn.Module()
            for n in ("query", "key", "value"):
                setattr(l.attention.attention, n, nn.Linear(D, D))
            l.attention.output = nn.Module()
            l.attention.output.dense = nn.Linear(D, D)
            l.layer_scale1 = nn.Module()
            l.layer_scale1.lambda1 = nn.Parameter(torch.ones(D))
            l.norm2 = nn.LayerNorm(D, eps=1e-6)
            l.mlp = nn.Module()
            if c.get("swiglu", False):      # HF Dinov2SwiGLUFFN parameter names
                Fh = (int(I * 2 / 3) + 7) // 8 * 8
                l.mlp.weights_in = nn.Linear(D, 2 * Fh)
                l.mlp.weights_out = nn.Linear(Fh, D)
            else:
                l.mlp.fc1 = nn.Linear(D, I)
                l.mlp.fc2 = nn.Linear(I, D)
            l.layer_scale2 = nn.Module()
            l.layer_scale2.lambda1 = nn.Parameter(torch.ones(D))
            layers.append(l)
        vt.encoder.layer = nn.ModuleList(layers)
        vt.layernorm = nn.LayerNorm(D, eps=1e-6)
        self.vision_tower = vt
        if state_dict is not None:
            vt.load_state_dict(state_dict, strict=False)
        self.image_processor = SimpleImageProcessor(self._image_size, IMNET_MEAN, IMNET_STD)
        vt.requires_grad_(False)
        self.is_loaded = True
        self._gpu = None

    def _prepare(self):
        vt = self.vision_tower
        grid = self._image_size // 14
        pos = vt.embeddings.position_embeddings
        n = int((pos.shape[1] - 1) ** 0.5)
        if n != grid:  # one-time (load-time) bicubic resize of the learned position table, as HF interpolate_pos_encoding
            pp = pos[:, 1:].reshape(1, n, n, -1).permute(0, 3, 1, 2).float()
            pp = F.interpolate(pp, size=(grid, grid), mode="bicubic", align_corners=False).to(pos.dtype)
            pos = torch.cat([pos[:, :1], pp.permute(0, 2, 3, 1).reshape(1, grid * grid, -1)], 1)
        g = dict(patch_w=_pad_cols(vt.embeddings.patch_embeddings.projection.weight.flatten(1)),
                 patch_b=vt.embeddings.patch_embeddings.projection.bias, cls=vt.embeddings.cls_token.reshape(-1).contiguous(),
                 pos=pos[0].contiguous(), ln_w=vt.layernorm.weight, ln_b=vt.layernorm.bias, blocks=[])
        for l in vt.encoder.layer:
            a = l.attention.attention
            blk = dict(
                ln1_w=l.norm1.weight, ln1_b=l.norm1.bias,
                qkv_w=torch.cat([a.query.weight, a.key.weight, a.value.weight], 0).contiguous(),
                qkv_b=torch.cat([a.query.bias, a.key.bias, a.value.bias], 0).contiguous(),
                proj_w=l.attention.output.dense.weight, proj_b=l.attention.output.dense.bias,
                ls1=l.layer_scale1.lambda1, ln2_w=l.norm2.weight, ln2_b=l.norm2.bias, ls2=l.layer_scale2.lambda1)
            if hasattr(l.mlp, "weights_in"):
                blk.update(win_w=l.mlp.weights_in.weight, win_b=l.mlp.weights_in.bias, fc2_w=l.mlp.weights_out.weight,
                           fc2_b=l.mlp.weights_out.bias)
            else:
                blk.update(fc1_w=l.mlp.fc1.weight, fc1_b=l.mlp.fc1.bias, fc2_w=l.mlp.fc2.weight, fc2_b=l.mlp.fc2.bias)
            g["blocks"].append(blk)
        self._gpu = g

    def _run(self, images):
        if self._gpu is None:
            self._prepare()
        g, c = self._gpu, self.cfg
        B = images.shape[0]
        grid = images.shape[-1] // 14
        patches = ops.gemm(ops.patchify_nchw(images, 14), g["patch_w"], bias=g["patch_b"]).view(B, grid * grid, -1)
        x = ops.add_pos_tokens(patches, g["cls"], g["pos"])
        x = _vit_blocks(x, g["blocks"], c["num_attention_heads"], "gelu", 1e-6)
        x = ops.layernorm_fwd(x, g["ln_w"], g["ln_b"], 1e-6)
        if self.select_feature == "cls_patch":
            return x
        if self.select_feature != "patch":
            raise ValueError(f"Unexpected select feature: {self.select_feature}")
        return self._finish_tokens(x, grid, skip_cls=True)


# ------------------------------------------------------------------------------------------------------------------
# A2 — SigLIP ViT-SO400M/14@384  (siglip_encoder.py; timm VisionTransformer trunk parameter names)
# ------------------------------------------------------------------------------------------------------------------
class SiglipVisionTower(BaseVisionTower):
    DEFAULT = dict(hidden_size=1152, intermediate_size=4304, num_hidden_layers=27, num_attention_heads=16, patch_size=14,
                   image_size=384, act="gelu")

    def __init__(self, vision_tower, args, delay_load=False):
        super().__init__(vision_tower, args, delay_load)
        base, res, interp = _parse_res_interp(vision_tower)
        self.vision_tower_name = base
        self._interp_size = interp
        self.cfg = dict(self.DEFAULT, **getattr(args, "siglip_config_overrides", {}) or {})
        self._image_size = res if res is not None else self.cfg["image_size"]
        self._patch_size = 14
        self._hidden_size = self.cfg["hidden_size"]
        if not delay_load:
            self.load_model()

    def load_model(self, device_map=None, state_dict=None):
        c = self.cfg
        D, I, L = c["hidden_size"], c["intermediate_size"], c["num_hidden_layers"]
        vt = nn.Module()
        vt.patch_embed = nn.Module()
        vt.patch_embed.proj = nn.Conv2d(3, D, 14, 14)
        vt.pos_embed = _p(1, (self._image_size // 14) ** 2, D)
        blocks = []
        for _ in range(L):
            b = nn.Module()
            b.norm1 = nn.LayerNorm(D, eps=1e-6)
            b.attn = nn.Module()
            b.attn.qkv = nn.Linear(D, 3 * D)
            b.attn.proj = nn.Linear(D, D)
            b.norm2 = nn.LayerNorm(D, eps=1e-6)
            b.mlp = nn.Module()
            b.mlp.fc1 = nn.Linear(D, I)
            b.mlp.fc2 = nn.Linear(I, D)
            blocks.append(b)
        vt.blocks = nn.ModuleList(blocks)
        vt.norm = nn.LayerNorm(D, eps=1e-6)
        self.vision_tower = vt
        if state_dict is not None:
            vt.load_state_dict(state_dict, strict=False)
        self.image_processor = SimpleImageProcessor(self._image_size, (0.5, 0.5, 0.5), (0.5, 0.5, 0.5))
        vt.requires_grad_(False)
        self.is_loaded = True
        self._gpu = None

    def _prepare(self):
        vt = self.vision_tower
        g = dict(patch_w=_pad_cols(vt.patch_embed.proj.weight.flatten(1)), patch_b=vt.patch_embed.proj.bias,
                 pos=vt.pos_embed[0].contiguous(), ln_w=vt.norm.weight, ln_b=vt.norm.bias, blocks=[])
        for b in vt.blocks:
            g["blocks"].append(dict(ln1_w=b.norm1.weight, ln1_b=b.norm1.bias, qkv_w=b.attn.qkv.weight, qkv_b=b.attn.qkv.bias,
                                    proj_w=b.attn.proj.weight, proj_b=b.attn.proj.bias, ln2_w=b.norm2.weight,
                                    ln2_b=b.norm2.bias, fc1_w=b.mlp.fc1.weight, fc1_b=b.mlp.fc1.bias,
                                    fc2_w=b.mlp.fc2.weight, fc2_b=b.mlp.fc2.bias))
        self._gpu = g

    def _run(self, images):
        if self._gpu is None:
            self._prepare()
        g, c = self._gpu, self.cfg
        B = images.shape[0]
        grid = images.shape[-1] // 14
        patches = ops.gemm(ops.patchify_nchw(images, 14), g["patch_w"], bias=g["patch_b"]).view(B, grid * grid, -1)
        x = ops.add_pos_tokens(patches, None, g["pos"])
        x = _vit_blocks(x, g["blocks"], c["num_attention_heads"], c["act"], 1e-6)
        x = ops.layernorm_fwd(x, g["ln_w"], g["ln_b"], 1e-6)
        return self._finish_tokens(x, grid, skip_cls=False)


# ------------------------------------------------------------------------------------------------------------------
# A4 — OpenCLIP ConvNeXt-XXL  (clip_convnext_encoder.py; timm ConvNeXt trunk parameter names)
# ------------------------------------------------------------------------------------------------------------------
class CLIPConvNextTower(BaseVisionTower):
    DEFAULT = dict(depths=(3, 4, 30, 3), dims=(384, 768, 1536, 3072), image_size=1024)

    def __init__(self, vision_tower, args, delay_load=False):
        super().__init__(vision_tower, args, delay_load)
        base, res, interp = _parse_res_interp(vision_tower)
        self.is_multi_stage = "multi-stage" in base
        self.vision_tower_name = base
        self._interp_size = interp
        self.cfg = dict(self.DEFAULT, **getattr(args, "convnext_config_overrides", {}) or {})
        self._image_size = res if res is not None else self.cfg["image_size"]
        self._patch_size = 32
        dims = self.cfg["dims"]
        self._hidden_size = sum(dims) if self.is_multi_stage else dims[-1]
        if not delay_load:
            self.load_model()

    def load_model(self, device_map=None, state_dict=None):
        depths, dims = self.cfg["depths"], self.cfg["dims"]
        vt = nn.Module()
        vt.stem = nn.Sequential(nn.Conv2d(3, dims[0], 4, 4), nn.LayerNorm(dims[0], eps=1e-6))
        stages = []
        for s, (depth, C) in enumerate(zip(depths, dims)):
            st = nn.Module()
            if s > 0:
                st.downsample = nn.Sequential(nn.LayerNorm(dims[s - 1], eps=1e-6), nn.Conv2d(dims[s - 1], C, 2, 2))
            blocks = []
            for _ in range(depth):
                b = nn.Module()
                b.conv_dw = nn.Conv2d(C, C, 7, padding=3, groups=C)
                b.norm = nn.LayerNorm(C, eps=1e-6)
                b.mlp = nn.Module()
                b.mlp.fc1 = nn.Linear(C, 4 * C)
                b.mlp.fc2 = nn.Linear(4 * C, C)
                b.gamma = nn.Parameter(torch.ones(C))
                blocks.append(b)
            st.blocks = nn.ModuleList(blocks)
            stages.append(st)
        vt.stages = nn.ModuleList(stages)
        self.vision_tower = vt
        if state_dict is not None:
            vt.load_state_dict(state_dict, strict=False)
        self.image_processor = SimpleImageProcessor(self._image_size, CLIP_MEAN, CLIP_STD)
        vt.requires_grad_(False)
        self.is_loaded = True
        self._gpu = None

    def _prepare(self):
        vt = self.vision_tower
        g = dict(stem_w=_pad_cols(vt.stem[0].weight.flatten(1)), stem_b=vt.stem[0].bias, stem_ln_w=vt.stem[1].weight,
                 stem_ln_b=vt.stem[1].bias, stages=[])
        for s, st in enumerate(vt.stages):
            d = dict(blocks=[])
            if s > 0:
                w = st.downsample[1].weight  # [Cout, Cin, 2, 2] -> [Cout, (py, px, Cin)] to match patchify_nhwc
                d.update(ds_ln_w=st.downsample[0].weight, ds_ln_b=st.downsample[0].bias,
                         ds_w=w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous(), ds_b=st.downsample[1].bias)
            for b in st.blocks:
                C = b.conv_dw.weight.shape[0]
                d["blocks"].append(dict(dw_w=b.conv_dw.weight.view(C, 49).t().contiguous().view(7, 7, C), dw_b=b.conv_dw.bias,
                                        ln_w=b.norm.weight, ln_b=b.norm.bias, fc1_w=b.mlp.fc1.weight, fc1_b=b.mlp.fc1.bias,
                                        fc2_w=b.mlp.fc2.weight, fc2_b=b.mlp.fc2.bias, gamma=b.gamma))
            g["stages"].append(d)
        self._gpu = g

    def _run(self, images):
        if self._gpu is None:
            self._prepare()
        g = self._gpu
        B, _, R, _ = images.shape
        H = W = R // 4
        x = ops.gemm(ops.patchify_nchw(images, 4), g["stem_w"], bias=g["stem_b"])
        x = ops.layernorm_fwd(x, g["stem_ln_w"], g["stem_ln_b"], 1e-6).view(B, H, W, -1)
        outs = []
        for s, st in enumerate(g["stages"]):
            if s > 0:
                x = ops.layernorm_fwd(x, st["ds_ln_w"], st["ds_ln_b"], 1e-6)
                pt = ops.patchify_nhwc(x, 2)
                H, W = H // 2, W // 2
                x = ops.gemm(pt, st["ds_w"], bias=st["ds_b"]).view(B, H, W, -1)
            C = x.shape[-1]
            for b in st["blocks"]:
                h = ops.dwconv7(x, b["dw_w"], b["dw_b"])
                h = ops.layernorm_fwd(h, b["ln_w"], b["ln_b"], 1e-6).view(B * H * W, C)
                m = ops.gemm(h, b["fc1_w"], bias=b["fc1_b"], act="gelu")
                x = ops.gemm(m, b["fc2_w"], bias=b["fc2_b"], colscale=b["gamma"], residual=x.view(B * H * W, C)).view(B, H, W, C)
            outs.append((x, H, W))
        feats = outs if self.is_multi_stage else outs[-1:]
        t = int(self._interp_size ** 0.5) if self._interp_size is not None else feats[-1][1]
        Ctot = sum(f[0].shape[-1] for f in feats)
        out = torch.empty((B, t * t, Ctot), dtype=torch.bfloat16, device=images.device)
        col = 0
        for f, h, w in feats:  # bilinear resize each stage to the interp grid, channel-concatenate in place (:99-119)
            ops.bilinear(f.view(B, h * w, -1), h, w, t, t, out=out, out_ld=Ctot, out_col0=col)
            col += f.shape[-1]
        return out

    @property
    def num_patches_per_side(self):
        if self._interp_size is not None:
            return int(self._interp_size ** 0.5)
        return self._image_size // 32
