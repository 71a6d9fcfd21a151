"""Spatial Vision Aggregator — H100-native mirror of the reference's `cambrian/model/vision_sampler.py`.

Same class names, constructor signatures, attribute / state-dict key names and call conventions as the reference
(`VisionTokenSampler` vision_sampler.py:407-419, `VisionCrossAttentionLayer` :248-327, `MultiKVCrossAttention`
:155-234, `MLP` :237-245), so released checkpoints load unchanged and `cambrian_arch` / `cambrian_llama` call sites work
as they are.  The arithmetic runs in `cambrian_b200.autograd.SVALayerFn` on the hand-written sm_90a kernels
(wgmma GEMMs for the LayerNorm+Linear projections, the fused window-attention kernel for the softmax).

Both layer types are implemented: `joint` (`VisionCrossAttentionLayer`, the one every released model and every reference
caller uses — one hand-scheduled `SVALayerFn` block) and `sep` (`VisionAggregationLayer` :330-405 with `CrossAttention`
:55-121 / `AggregationBlock` :124-153 — API surface only in the reference, composed here from finer-grained Functions
plus the fused softmax-over-towers combine kernel).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import ops
from ..autograd import (ActFn, CatLinearFn, CrossAttnTowerFn, LayerNormFn, LinearFn, LinearResidualFn, NarrowLinearFn,
                        SVALayerFn, TowerCombineFn)


class MultiKVCrossAttention(nn.Module):
    """Parameter container with the reference's names (q_proj / k_proj_i / v_proj_i = LayerNorm+Linear, o_proj)."""

    def __init__(self, q_dim, kv_dim_list, hidden_dim, num_heads, attention_bias=False):
        super().__init__()
        self.hidden_dim = hidden_dim
        self.num_heads = num_heads
        self.head_dim = hidden_dim // num_heads
        if self.head_dim * num_heads != hidden_dim:
            raise ValueError(
                f"hidden_dim must be divisible by num_heads (got `hidden_dim`: {hidden_dim} and `num_heads`: {num_heads}).")
        if attention_bias:
            raise NotImplementedError("attention_bias=True is never used by the reference models")
        self.q_proj = nn.Sequential(nn.LayerNorm(q_dim), nn.Linear(q_dim, hidden_dim, bias=False))
        self.num_of_kvs = len(kv_dim_list)
        for i, kv_dim in enumerate(kv_dim_list):
            setattr(self, f"k_proj_{i}", nn.Sequential(nn.LayerNorm(kv_dim), nn.Linear(kv_dim, hidden_dim, bias=False)))
            setattr(self, f"v_proj_{i}", nn.Sequential(nn.LayerNorm(kv_dim), nn.Linear(kv_dim, hidden_dim, bias=False)))
        self.o_proj = nn.Linear(hidden_dim, q_dim, bias=False)


class MLP(nn.Module):
    def __init__(self, d_in, d_hidden, d_out):
        super().__init__()
        self.linear_1 = nn.Linear(d_in, d_hidden, bias=False)
        self.act = nn.GELU()
        self.linear_2 = nn.Linear(d_hidden, d_out, bias=False)


class VisionCrossAttentionLayer(nn.Module):
    def __init__(self, q_dim, context_dim, kv_dim_list, kv_size_list, hidden_dim=1024, layer_idx=0):
        super().__init__()
        num_heads = 16
        if hidden_dim != 1024 or any(d != hidden_dim for d in kv_dim_list):
            raise NotImplementedError("the SVA kernels are specialised for vision_hidden_size = 1024 (16 x 64)")
        self.num_of_kvs = len(kv_dim_list)
        self.q_dim = q_dim
        self.proj_context = nn.Linear(context_dim, hidden_dim, bias=False)
        self.proj_in = nn.Linear(q_dim + hidden_dim, hidden_dim, bias=False)
        self.proj_out = MLP(hidden_dim, hidden_dim, q_dim)
        self.norm = nn.LayerNorm(hidden_dim)
        self.cross_attn = MultiKVCrossAttention(hidden_dim, kv_dim_list, hidden_dim, num_heads)
        self.kv_size_list = list(kv_size_list)
        for i, kv_size in enumerate(kv_size_list):
            if kv_size > 1:
                setattr(self, f"pos_embed_{i}", nn.Parameter(torch.randn(kv_size ** 2, hidden_dim)))

    def _named_params(self):
        ca = self.cross_attn
        items = [("proj_context", self.proj_context.weight), ("proj_in", self.proj_in.weight),
                 ("out1_w", self.proj_out.linear_1.weight), ("out2_w", self.proj_out.linear_2.weight),
                 ("norm_w", self.norm.weight), ("norm_b", self.norm.bias),
                 ("q_ln_w", ca.q_proj[0].weight), ("q_ln_b", ca.q_proj[0].bias), ("q_w", ca.q_proj[1].weight),
                 ("o_w", ca.o_proj.weight)]
        for i in range(self.num_of_kvs):
            kp, vp = getattr(ca, f"k_proj_{i}"), getattr(ca, f"v_proj_{i}")
            items += [(f"k_ln_w_{i}", kp[0].weight), (f"k_ln_b_{i}", kp[0].bias), (f"k_w_{i}", kp[1].weight),
                      (f"v_ln_w_{i}", vp[0].weight), (f"v_ln_b_{i}", vp[0].bias), (f"v_w_{i}", vp[1].weight)]
            if self.kv_size_list[i] > 1:
                items.append((f"pos_embed_{i}", getattr(self, f"pos_embed_{i}")))
        return items

    def forward(self, queries, context_feature, *vision_latents_attention_mask_list, natural_layout=None):
        """Reference call convention (vision_sampler.py:270-275): queries [N,1,q_dim], context [N,1,ctx_dim], then T
        window-rearranged latents [N, r_i^2, 1024] followed by T bool masks [N, r_i^2].

        natural_layout=(B, q_side): fast path used by our cambrian_arch — latents are the un-rearranged grids
        [B, (r_i q_side)^2, 1024] and the window gather happens inside the kernels (no permute/contiguous copies)."""
        T = self.num_of_kvs
        latents = list(vision_latents_attention_mask_list[:T])
        masks = list(vision_latents_attention_mask_list[T:])
        n = queries.shape[0]
        for i, m in enumerate(masks):
            if m is not None and m.numel() != n * self.kv_size_list[i] ** 2:
                # same failure class as the reference's mask-shape check (vision_sampler.py:202-206)
                raise ValueError(f"Attention mask should be of size {(n, 1, 1, self.kv_size_list[i] ** 2)}, "
                                 f"but is {tuple(m.shape)}")
        masks = [None if m is None else m.reshape(n, -1) for m in masks] if masks else None
        if masks is not None and all(m is None for m in masks):
            masks = None
        items = self._named_params()
        names = [k for k, _ in items]
        params = [p for _, p in items]
        ops.require_cuda_bf16_params(params, "SVA layers")
        meta = dict(T=T, rs=self.kv_size_list, masks=masks, natural=natural_layout, names=names, params=params,
                    feat_shapes=[t.shape for t in latents])
        q2 = queries.reshape(n, -1)
        c2 = context_feature.reshape(n, -1)
        latents = [t.to(torch.bfloat16) for t in latents]
        out = SVALayerFn.apply(meta, q2.contiguous(), c2.contiguous(), *[t.contiguous() for t in latents], *params)
        return out.view(queries.shape)


class CrossAttention(nn.Module):
    """Parameter container of vision_sampler.py:55-121 (q_proj / k_proj / v_proj = LayerNorm + Linear, o_proj)."""

    def __init__(self, q_dim, kv_dim, hidden_dim, num_heads, attention_bias=False):
        super().__init__()
        self.hidden_dim = hidden_dim
        self.num_heads = num_heads
        self.head_dim = hidden_dim // num_heads
        if self.head_dim * num_heads != hidden_dim:
            raise ValueError(
                f"hidden_dim must be divisible by num_heads (got `hidden_dim`: {hidden_dim} and `num_heads`: {num_heads}).")
        if attention_bias:
            raise NotImplementedError("attention_bias=True is never used by the reference models")
        self.q_proj = nn.Sequential(nn.LayerNorm(q_dim), nn.Linear(q_dim, hidden_dim, bias=False))
        self.k_proj = nn.Sequential(nn.LayerNorm(kv_dim), nn.Linear(kv_dim, hidden_dim, bias=False))
        self.v_proj = nn.Sequential(nn.LayerNorm(kv_dim), nn.Linear(kv_dim, hidden_dim, bias=False))
        self.o_proj = nn.Linear(hidden_dim, q_dim, bias=False)


class AggregationBlock(nn.Module):
    """vision_sampler.py:124-153: CrossAttention over the tower's window, or an MLP of its single latent."""

    def __init__(self, attention, q_dim, kv_dim, hidden_dim, num_heads, attention_bias=False):
        super().__init__()
        self.hidden_dim = hidden_dim
        self.num_heads = num_heads
        self.head_dim = hidden_dim // num_heads
        if self.head_dim * num_heads != hidden_dim:
            raise ValueError(
                f"hidden_dim must be divisible by num_heads (got `hidden_dim`: {hidden_dim} and `num_heads`: {num_heads}).")
        self.attention = attention
        if attention:
            self.attention_layer = CrossAttention(q_dim, kv_dim, hidden_dim, num_heads, attention_bias)
        else:
            self.attention_layer = MLP(kv_dim, q_dim, q_dim)


class VisionAggregationLayer(nn.Module):
    """layer_type="sep" (vision_sampler.py:330-405): one aggregate per tower, mixed by a per-query softmax over towers."""

    def __init__(self, q_dim, context_dim, kv_dim_list, kv_size_list, hidden_dim=1024, layer_idx=0):
        super().__init__()
        num_heads = 16
        if hidden_dim != 1024 or any(d != hidden_dim for d in kv_dim_list):
            raise NotImplementedError("the SVA kernels are specialised for vision_hidden_size = 1024 (16 x 64)")
        self.num_of_kvs = len(kv_dim_list)
        if self.num_of_kvs > NarrowLinearFn.PAD:
            raise NotImplementedError(f"at most {NarrowLinearFn.PAD} towers")
        self.q_dim = q_dim
        self.proj_context = nn.Linear(context_dim, hidden_dim, bias=False)
        self.proj_in = nn.Linear(q_dim + hidden_dim, hidden_dim, bias=False)
        self.proj_out = MLP(hidden_dim, hidden_dim, q_dim)
        self.norm = nn.LayerNorm(hidden_dim)
        if self.num_of_kvs > 1:
            self.weight_mlp = MLP(q_dim + hidden_dim, hidden_dim, self.num_of_kvs)
        self.kv_size_list = list(kv_size_list)
        for i, kv_size in enumerate(kv_size_list):
            if kv_size > 1:
                setattr(self, f"pos_embed_{i}", nn.Parameter(torch.randn(kv_size ** 2, hidden_dim)))
                setattr(self, f"aggregate_{i}", AggregationBlock(True, hidden_dim, kv_dim_list[i], hidden_dim, num_heads))
            else:
                setattr(self, f"aggregate_{i}", AggregationBlock(False, hidden_dim, kv_dim_list[i], hidden_dim, num_heads))

    def forward(self, queries, context_feature, *vision_latents_attention_mask_list, natural_layout=None):
        """Same call conventions as VisionCrossAttentionLayer.forward above (reference: vision_sampler.py:352-357)."""
        T = self.num_of_kvs
        latents = list(vision_latents_attention_mask_list[:T])
        masks = list(vision_latents_attention_mask_list[T:]) or [None] * T
        n = queries.shape[0]
        for i, m in enumerate(masks):
            if m is not None and m.numel() != n * self.kv_size_list[i] ** 2:
                raise ValueError(f"Attention mask should be of size {(n, 1, 1, self.kv_size_list[i] ** 2)}, "
                                 f"but is {tuple(m.shape)}")
        ops.require_cuda_bf16_params(list(self.parameters()), "SVA layers")
        q2 = queries.reshape(n, -1).contiguous()
        c2 = context_feature.reshape(n, -1).contiguous()
        ctxp = LinearFn.apply(c2, self.proj_context.weight, None)                                  # :360
        if T > 1:                                                                                  # :364-368
            hid = ActFn.apply(CatLinearFn.apply(q2, ctxp, self.weight_mlp.linear_1.weight), "gelu")
            logits = NarrowLinearFn.apply(hid, self.weight_mlp.linear_2.weight)
        else:
            logits = torch.zeros((n, NarrowLinearFn.PAD), dtype=torch.bfloat16, device=q2.device)  # softmax of one = 1
        q_in = CatLinearFn.apply(q2, ctxp, self.proj_in.weight)                                    # :370
        aggs = []
        for i in range(T):
            r = self.kv_size_list[i]
            blk = getattr(self, f"aggregate_{i}").attention_layer
            lat = latents[i].to(torch.bfloat16).contiguous()
            if r > 1:                                                                              # :382-392
                params = [blk.q_proj[0].weight, blk.q_proj[0].bias, blk.q_proj[1].weight,
                          blk.k_proj[0].weight, blk.k_proj[0].bias, blk.k_proj[1].weight,
                          blk.v_proj[0].weight, blk.v_proj[0].bias, blk.v_proj[1].weight,
                          blk.o_proj.weight, getattr(self, f"pos_embed_{i}")]
                mask = None if masks[i] is None else masks[i].reshape(n, -1)
                meta = dict(r=r, mask=mask, natural=natural_layout, params=params)
                aggs.append(CrossAttnTowerFn.apply(meta, q_in, lat, *params))
            else:
                f2 = lat.reshape(n, -1)
                h = ActFn.apply(LinearFn.apply(f2, blk.linear_1.weight, None), "gelu")
                aggs.append(LinearFn.apply(h, blk.linear_2.weight, None))
        q = TowerCombineFn.apply(logits, q_in, *aggs)                                              # :394-396
        q = LayerNormFn.apply(q, self.norm.weight, self.norm.bias, 1e-5)                           # :398
        h = ActFn.apply(LinearFn.apply(q, self.proj_out.linear_1.weight, None), "gelu")
        out = LinearResidualFn.apply(h, self.proj_out.linear_2.weight, q2)                         # :400-402
        return out.view(queries.shape)


class VisionTokenSampler(nn.Module):
    def __init__(self, q_dim, context_dim, kv_dim_list, kv_size_list, vision_hidden_size, num_of_layers=1,
                 layer_type="joint"):
        super().__init__()
        assert layer_type in ["joint", "sep"]
        layer_cls = VisionCrossAttentionLayer if layer_type == "joint" else VisionAggregationLayer
        self.layers = nn.ModuleList([
            layer_cls(q_dim, context_dim, kv_dim_list, kv_size_list, vision_hidden_size, idx)
            for idx in range(num_of_layers)])

    def forward(self, queries, context_feature, *vision_latents_attention_mask_list, natural_layout=None):
        for layer in self.layers:
            queries = layer(queries, context_feature, *vision_latents_attention_mask_list, natural_layout=natural_layout)
        return queries
