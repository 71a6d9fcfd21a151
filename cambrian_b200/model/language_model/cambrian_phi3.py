"""CambrianPhi3ForCausalLM — H100-native mirror of the reference's `cambrian/model/language_model/cambrian_phi3.py`
(Cambrian-Phi3-3B), for inference and training.

Phi-3-mini is the LLaMA decoder with three differences, and this file adds only those:
  * fused projections under Phi-3's state-dict keys: `self_attn.qkv_proj` ([q | k | v] rows) and `mlp.gate_up_proj`
    ([gate | up] rows) — exactly the layouts `fuse_rows` builds for LLaMA, so they feed the same GEMM / SwiGLU kernels
    as they are, without copies;
  * head dim 96 (hidden 3072 / 32 heads), which the flash-attention forward and backward instantiate;
  * a causal sliding window (`config.sliding_window`, 2047 in the released checkpoints).  The reference loads the model
    with `use_flash_attention_2=False`, so its mask is transformers' `_prepare_4d_causal_attention_mask(...,
    sliding_window=W)` as of the transformers 4.37 it pins: key slot j is visible from query slot i iff 0 <= i - j < W,
    counted in cache slots (left padding included), on top of the padding mask.  flash-attn's window_size=(W, W) —
    and later transformers releases — admit one more key (i - j <= W).  tests/golden/phi3_mask.npz pins the rule.

Everything else is shared with CambrianLlamaForCausalLM: the decoder layer's `infer` (the layer hands it its fused
weights through `_fused()` and its window through `window`), `KVCache`, `generate()` and its CUDA-graph decode loop, and
the multimodal front end of cambrian_arch.py (towers, SVA connector, in-LLM SVA sites).  In training each layer runs
autograd.FusedDecoderLayerFn — DecoderLayerFn's forward and backward with the fused `qkv_proj` / `gate_up_proj` weights
as the leaf parameters (each with its own `main_grad` under TrainEngine) and the window passed to both attention calls,
recompute included.  The reference trains Phi-3 with eager attention (`_supports_sdpa = False`) under the same mask, its
RMSNorm in fp32 (`hf_cast=False` in training, as for LLaMA).

Not supported, each refused with an exception that names it: training on parameters that are not all CUDA bf16 (the
attention backward has no CPU path), non-zero `attention_dropout` / `resid_pdrop` / `embd_pdrop` (dropout is not
implemented; Phi-3-mini's are 0), `fp8_training`, NF4 / LLM.int8 / FP8 weights (the quantisers address the LLaMA
projections by name), the FP8 KV cache (its decode kernel takes head dims 64 and 128), Zero3Inference, and
`rope_scaling` (the 128k `su` / `yarn` variants).
"""
from __future__ import annotations

import torch
import torch.nn as nn
from transformers import AutoConfig, AutoModelForCausalLM, PretrainedConfig

from ...autograd import FusedDecoderLayerFn
from .cambrian_llama import (CambrianLlamaForCausalLM, CambrianLlamaModel, CambrianPreTrainedModel, CBLlamaDecoderLayer,
                             CBRMSNorm)

DROPOUT_FIELDS = ("attention_dropout", "resid_pdrop", "embd_pdrop")


class CambrianPhi3Config(PretrainedConfig):
    """Phi-3's configuration fields (defaults: Phi-3-mini-4k) under model_type "cambrian_phi3"; the Cambrian multimodal
    fields (mm_*, image_token_len, ...) ride along as extra attributes, as in the reference's config.json."""
    model_type = "cambrian_phi3"

    def __init__(self, vocab_size=32064, hidden_size=3072, intermediate_size=8192, num_hidden_layers=32,
                 num_attention_heads=32, num_key_value_heads=None, resid_pdrop=0.0, embd_pdrop=0.0,
                 attention_dropout=0.0, hidden_act="silu", max_position_embeddings=4096,
                 original_max_position_embeddings=4096, initializer_range=0.02, rms_norm_eps=1e-5, use_cache=True,
                 tie_word_embeddings=False, rope_theta=10000.0, rope_scaling=None, bos_token_id=1, eos_token_id=32000,
                 pad_token_id=32000, sliding_window=None, **kwargs):
        self.vocab_size = vocab_size
        self.hidden_size = hidden_size
        self.intermediate_size = intermediate_size
        self.num_hidden_layers = num_hidden_layers
        self.num_attention_heads = num_attention_heads
        self.num_key_value_heads = num_attention_heads if num_key_value_heads is None else num_key_value_heads
        self.resid_pdrop = resid_pdrop
        self.embd_pdrop = embd_pdrop
        self.attention_dropout = attention_dropout
        self.hidden_act = hidden_act
        self.max_position_embeddings = max_position_embeddings
        self.original_max_position_embeddings = original_max_position_embeddings
        self.initializer_range = initializer_range
        self.rms_norm_eps = rms_norm_eps
        self.use_cache = use_cache
        self.rope_theta = rope_theta
        self.rope_scaling = rope_scaling
        self.sliding_window = sliding_window
        super().__init__(bos_token_id=bos_token_id, eos_token_id=eos_token_id, pad_token_id=pad_token_id,
                         tie_word_embeddings=tie_word_embeddings, **kwargs)


def check_supported(config):
    """Refuse the configurations the kernels do not cover, before any weight is allocated."""
    rs = getattr(config, "rope_scaling", None)
    kind = (rs.get("type", rs.get("rope_type")) if isinstance(rs, dict) else rs) if rs is not None else None
    if kind not in (None, "default"):       # newer transformers store plain RoPE as {"rope_type": "default", ...}
        raise NotImplementedError(f"Cambrian-Phi3 with rope_scaling type {kind!r} (the 128k `su` / `yarn` variants) is "
                                  "not supported: only plain RoPE (rope_scaling=None, the 4k models) is implemented")
    if getattr(config, "hidden_act", "silu") != "silu":
        raise NotImplementedError(f"Cambrian-Phi3 with hidden_act={config.hidden_act!r}: the SwiGLU kernel is SiLU only")


def require_cuda_bf16(model):
    """Training runs the CUDA kernels only: refuse parameters that are not all CUDA bf16."""
    if any(p.device.type != "cuda" or p.dtype != torch.bfloat16 for p in model.parameters()):
        raise NotImplementedError("Cambrian-Phi3 trains in bf16 on CUDA only: its head-dim-96 / sliding-window "
                                  "flash-attention backward has no CPU path; move the model to CUDA in bf16, or run "
                                  "it under torch.no_grad()")


def check_trainable(model):
    """Refuse the training configurations that are not implemented, before the first kernel runs."""
    cfg = model.config
    for name in DROPOUT_FIELDS:
        if getattr(cfg, name, 0.0):
            raise NotImplementedError(f"training Cambrian-Phi3 with {name}={getattr(cfg, name)} is not supported: "
                                      "dropout is not implemented (Phi-3-mini's dropouts are 0)")
    if getattr(cfg, "fp8_training", False):
        raise NotImplementedError("Cambrian-Phi3 with fp8_training is not supported: FP8 training is validated for "
                                  "the LLaMA decoder only")
    require_cuda_bf16(model)


class CBPhi3Attention(nn.Module):
    def __init__(self, config):
        super().__init__()
        H, nh, nkv = config.hidden_size, config.num_attention_heads, config.num_key_value_heads
        hd = H // nh
        self.qkv_proj = nn.Linear(H, (nh + 2 * nkv) * hd, bias=False)
        self.o_proj = nn.Linear(nh * hd, H, bias=False)


class CBPhi3MLP(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.gate_up_proj = nn.Linear(config.hidden_size, 2 * config.intermediate_size, bias=False)
        self.down_proj = nn.Linear(config.intermediate_size, config.hidden_size, bias=False)


class CBPhi3DecoderLayer(CBLlamaDecoderLayer):
    """Phi3DecoderLayer under its state-dict keys: FusedDecoderLayerFn under grad, CBLlamaDecoderLayer.infer without."""

    def __init__(self, config, layer_idx):
        nn.Module.__init__(self)
        self.layer_idx = layer_idx
        self.nh, self.nkv = config.num_attention_heads, config.num_key_value_heads
        self.hd = config.hidden_size // self.nh
        self.window = int(getattr(config, "sliding_window", None) or 0)
        self.self_attn = CBPhi3Attention(config)
        self.mlp = CBPhi3MLP(config)
        self.input_layernorm = CBRMSNorm(config.hidden_size, config.rms_norm_eps)
        self.post_attention_layernorm = CBRMSNorm(config.hidden_size, config.rms_norm_eps)
        self._nf4 = self._int8 = self._fp8 = None

    def _fused(self):
        # Phi-3 stores the fused layouts itself: [q | k | v] and [gate | up] rows, used as they are
        return self.self_attn.qkv_proj.weight, self.mlp.gate_up_proj.weight, None, None

    def forward(self, x, rt):
        if not torch.is_grad_enabled():
            return self.infer(x, rt, None)
        a, m = self.self_attn, self.mlp
        ln1, ln2 = self.input_layernorm.weight, self.post_attention_layernorm.weight
        qkv_w, gu_w = a.qkv_proj.weight, m.gate_up_proj.weight
        meta = self._train_meta(rt, qkv_w, gu_w, window=self.window)
        return FusedDecoderLayerFn.apply(meta, x, ln1, qkv_w, a.o_proj.weight, ln2, gu_w, m.down_proj.weight)


class CambrianPhi3Model(CambrianLlamaModel):
    config_class = CambrianPhi3Config
    decoder_layer_cls = CBPhi3DecoderLayer


class CambrianPhi3ForCausalLM(CambrianLlamaForCausalLM):
    config_class = CambrianPhi3Config
    _no_split_modules = ["CBPhi3DecoderLayer"]

    def __init__(self, config):
        check_supported(config)
        CambrianPreTrainedModel.__init__(self, config)
        self.model = CambrianPhi3Model(config)
        self.vocab_size = config.vocab_size
        self.lm_head = nn.Linear(config.hidden_size, config.vocab_size, bias=False)
        self.post_init()

    def attention_window(self) -> int:
        return int(getattr(self.config, "sliding_window", None) or 0)

    def check_trainable(self):
        """TrainEngine's and the grad-mode forward's check: see `check_trainable`."""
        check_trainable(self)

    def forward(self, *args, **kwargs):
        """cambrian_phi3.py's forward (the Phi3ForCausalLM outputs: loss, logits, past_key_values)."""
        if torch.is_grad_enabled():
            check_trainable(self)
        return super().forward(*args, **kwargs)

    @torch.no_grad()
    def generate(self, inputs=None, images=None, image_sizes=None, **kwargs):
        """cambrian_phi3.py's generate(inputs, images, image_sizes, **kw): CambrianLlamaForCausalLM.generate with the
        sliding window applied in prefill and at every decode step."""
        from ...kv_fp8 import resolve_cache_dtype
        if resolve_cache_dtype(self.config, kwargs.get("kv_cache_dtype")) == "fp8":
            raise NotImplementedError("Cambrian-Phi3 with kv_cache_dtype='fp8' is not supported: the FP8 decode attention "
                                      "kernel takes head dims 64 and 128, Phi-3's is 96")
        return super().generate(inputs, images=images, image_sizes=image_sizes, **kwargs)


AutoConfig.register("cambrian_phi3", CambrianPhi3Config)
AutoModelForCausalLM.register(CambrianPhi3Config, CambrianPhi3ForCausalLM)
