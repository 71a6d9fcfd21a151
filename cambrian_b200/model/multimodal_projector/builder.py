"""`build_vision_projector` — mirror of cambrian/model/multimodal_projector/builder.py:54-78 for the projector types the
hot path uses (`linear`, `mlp{N}x_gelu`, `identity`).  Returns nn.Sequential modules with the reference's state-dict
keys (0.weight, 0.bias, 2.weight, ...), whose Linear / GELU children run on the sm_90a GEMM / activation kernels."""
from __future__ import annotations

import re

import torch.nn as nn

from ...autograd import ActFn, LayerNormFn, LinearFn


class CBLinear(nn.Linear):
    def forward(self, x):
        return LinearFn.apply(x, self.weight, self.bias)


class CBGELU(nn.GELU):
    def forward(self, x):
        return ActFn.apply(x, "gelu")


class CBLayerNorm(nn.LayerNorm):
    def forward(self, x):
        return LayerNormFn.apply(x, self.weight, self.bias, self.eps)


class IdentityMap(nn.Module):
    def forward(self, x, *args, **kwargs):
        return x

    @property
    def config(self):
        return {"mm_projector_type": "identity"}


def build_vision_projector(config, delay_load=False, **kwargs):
    projector_type = getattr(config, "mm_projector_type", "linear")
    config.mm_hidden_size = 256 if getattr(config, "mm_hidden_size", None) is None else config.mm_hidden_size
    if projector_type == "linear":
        return CBLinear(config.mm_hidden_size, config.hidden_size)
    m = re.match(r"^mlp(\d+)x_gelu$", projector_type)
    if m:
        depth = int(m.group(1))
        mods = [CBLinear(config.mm_hidden_size, config.hidden_size)]
        for _ in range(1, depth):
            mods += [CBGELU(), CBLinear(config.hidden_size, config.hidden_size)]
        return nn.Sequential(*mods)
    if projector_type == "identity":
        return IdentityMap()
    raise ValueError(f"Unknown projector type: {projector_type}")  # builder.py:78
