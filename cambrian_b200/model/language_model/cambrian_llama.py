"""CambrianLlamaForCausalLM — H100-native mirror of the reference's `cambrian/model/language_model/cambrian_llama.py`.

Same public surface (SURVEY.md §8b): `CambrianConfig` (model_type "cambrian_llama"), `CambrianLlamaModel`,
`CambrianLlamaForCausalLM.forward(input_ids, attention_mask, position_ids, past_key_values, inputs_embeds, labels,
use_cache, output_attentions, output_hidden_states, images, image_aux_attention_masks_list, image_sizes, return_dict,
cache_position)`, `generate(inputs, images, image_sizes, **kw)`, `get_model()`, HF auto-class registration, and the
HF LLaMA state-dict keys (`model.layers.{i}.self_attn.q_proj.weight`, ...), so released checkpoints load unchanged.

Every decoder layer runs as one `DecoderLayerFn` (RMSNorm -> fused QKV wgmma GEMM -> RoPE -> wgmma flash attention
-> o-proj GEMM + residual -> RMSNorm -> fused gate/up GEMM -> SwiGLU -> down GEMM + residual), with the SVA layers
re-inserted on the image span after decoder layers start + k*stride exactly as cambrian_llama.py:168-207 does.
q/k/v (and gate/up) keep their HF parameter names but share one contiguous storage so each pair/triple is one GEMM.
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.nn as nn
from transformers import AutoConfig, AutoModelForCausalLM, LlamaConfig, PreTrainedModel
from transformers.modeling_outputs import BaseModelOutputWithPast, CausalLMOutputWithPast

try:  # transformers >= 5: initialisers that honour the per-parameter `_is_hf_initialized` flag
    from transformers import initialization as _hf_init
except ImportError:  # pragma: no cover - older transformers
    _hf_init = None

from ... import ops, train_fp8
from ...autograd import DecoderLayerFn, LinearFn, LMHeadLossFn, RMSNormFn, SpanMergeFn, SpanSplitFn
from ...paged_kv import PagedCacheView
from ..cambrian_arch import IGNORE_INDEX, CambrianMetaForCausalLM, CambrianMetaModel, WindowedFeatures


_DECODE_GRAPH = __import__("os").environ.get("CB_DECODE_GRAPH", "1") != "0"


class CambrianConfig(LlamaConfig):
    model_type = "cambrian_llama"


# ------------------------------------------------------------------------------------------------------------------
# fused-storage helpers
# ------------------------------------------------------------------------------------------------------------------
def _adjacent(ts) -> bool:
    p = ts[0].data_ptr()
    st = ts[0].untyped_storage().data_ptr()
    for t in ts:
        if not t.is_contiguous() or t.data_ptr() != p or t.untyped_storage().data_ptr() != st:
            return False
        p += t.numel() * t.element_size()
    return True


def fuse_rows(params) -> torch.Tensor:
    """Return one [sum(rows), K] tensor aliasing the given [rows_i, K] parameters, re-pointing their .data into a
    fresh contiguous buffer first if they are not already adjacent in memory (e.g. after .to() / load_state_dict)."""
    datas = [p.data for p in params]
    if not _adjacent(datas):
        fused = torch.cat(datas, 0)
        o = 0
        for p in params:
            n = p.shape[0]
            p.data = fused[o:o + n]
            o += n
    rows = sum(p.shape[0] for p in params)
    K = params[0].shape[1]
    return torch.as_strided(params[0].data, (rows, K), (K, 1))


class _MultiFresh:
    """'gradient already written this step' marker shared by the parameters behind one fused weight."""

    def __init__(self, sets):
        self.sets = sets

    def __contains__(self, key):
        return key in self.sets[0]

    def add(self, key):
        for s in self.sets:
            s.add(key)


class _FusedGrad:
    """Gradient holder for a fused weight: exposes `.main_grad` as one view over the adjacent per-parameter
    main_grad slices (laid out by TrainEngine in named_parameters() order), or None when running under plain autograd."""

    def __init__(self, params):
        mgs = [getattr(p, "main_grad", None) for p in params]
        self.main_grad = None
        self._cb_fresh = None
        self._params = params
        if all(m is not None for m in mgs) and _adjacent(mgs):
            rows = sum(m.shape[0] for m in mgs)
            K = mgs[0].shape[1]
            self.main_grad = torch.as_strided(mgs[0], (rows, K), (K, 1))
            sets = [getattr(p, "_cb_fresh", None) for p in params]
            self._cb_fresh = _MultiFresh(sets) if all(s is not None for s in sets) else None

    def _cb_notify(self):
        for p in self._params:
            n = getattr(p, "_cb_notify", None)
            if n is not None:
                n()


def rope_tables(config, device):
    """HF LlamaRotaryEmbedding (default rope): inv_freq = theta^(-2i/d); cos/sin of pos * inv_freq in fp32."""
    hd = getattr(config, "head_dim", None) or config.hidden_size // config.num_attention_heads
    theta = getattr(config, "rope_theta", None)
    if theta is None:
        rp = getattr(config, "rope_parameters", None) or {}
        theta = rp.get("rope_theta", 10000.0)
    inv = 1.0 / (theta ** (torch.arange(0, hd, 2, dtype=torch.int64).float() / hd))
    t = torch.arange(config.max_position_embeddings, dtype=torch.float32)
    fr = torch.outer(t, inv)
    return fr.cos().contiguous().to(device), fr.sin().contiguous().to(device)


# ------------------------------------------------------------------------------------------------------------------
# LLaMA modules with HF parameter names
# ------------------------------------------------------------------------------------------------------------------
class CBRMSNorm(nn.Module):
    def __init__(self, hidden_size, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.variance_epsilon = eps

    def forward(self, x, hf_cast=False):
        return RMSNormFn.apply(x, self.weight, self.variance_epsilon, hf_cast)


class CBLlamaAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        H, nh, nkv = config.hidden_size, config.num_attention_heads, config.num_key_value_heads
        hd = getattr(config, "head_dim", None) or H // nh
        self.q_proj = nn.Linear(H, nh * hd, bias=False)
        self.k_proj = nn.Linear(H, nkv * hd, bias=False)
        self.v_proj = nn.Linear(H, nkv * hd, bias=False)
        self.o_proj = nn.Linear(nh * hd, H, bias=False)


class CBLlamaMLP(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.gate_proj = nn.Linear(config.hidden_size, config.intermediate_size, bias=False)
        self.up_proj = nn.Linear(config.hidden_size, config.intermediate_size, bias=False)
        self.down_proj = nn.Linear(config.intermediate_size, config.hidden_size, bias=False)


class CBLlamaDecoderLayer(nn.Module):
    window = 0                  # causal sliding window of the attention (0: none); Phi-3's layer sets it

    def __init__(self, config, layer_idx):
        super().__init__()
        self.layer_idx = layer_idx
        self.nh, self.nkv = config.num_attention_heads, config.num_key_value_heads
        self.hd = getattr(config, "head_dim", None) or config.hidden_size // self.nh
        self.self_attn = CBLlamaAttention(config)
        self.mlp = CBLlamaMLP(config)
        self.input_layernorm = CBRMSNorm(config.hidden_size, config.rms_norm_eps)
        self.post_attention_layernorm = CBRMSNorm(config.hidden_size, config.rms_norm_eps)
        self._nf4 = None        # NF4 projections (quant.quantize_decoder_nf4_): the bf16 weights are freed then
        self._int8 = None       # LLM.int8 projections (quant_int8.quantize_decoder_int8_), likewise
        self._fp8 = None        # FP8 E4M3 projections (quant_fp8.quantize_decoder_fp8_), likewise

    def _quantized(self):
        """{qkv, o, gate_up, down} -> projection objects with `linear(x, residual=None)` / `gate_up(x)`, or None."""
        return next((q for q in (self._nf4, self._int8, self._fp8) if q is not None), None)

    def _fused(self):
        a, m = self.self_attn, self.mlp
        qkv = [a.q_proj.weight, a.k_proj.weight, a.v_proj.weight]
        gu = [m.gate_proj.weight, m.up_proj.weight]
        return fuse_rows(qkv), fuse_rows(gu), _FusedGrad(qkv), _FusedGrad(gu)

    def forward(self, x, rt):
        if self._quantized() is not None:
            if torch.is_grad_enabled():
                fmt = ("a 4-bit (NF4)" if self._nf4 is not None else
                       "an 8-bit (LLM.int8)" if self._int8 is not None else "an 8-bit (FP8)")
                raise NotImplementedError(f"{fmt} model is inference-only: training quantised weights (QLoRA) is "
                                          "not supported; run it under torch.no_grad()")
            return self.infer(x, rt, None)
        a, m = self.self_attn, self.mlp
        qkv_w, gu_w, g_qkv, g_gu = self._fused()
        fp8 = bool(rt.get("fp8", False))
        if fp8:
            train_fp8.check_widths(x.shape[-1], gu_w.shape[0] // 2, qkv_w.shape[0])
        meta = self._train_meta(rt, g_qkv, g_gu, fp8=fp8, qkv_w=qkv_w, gu_w=gu_w)
        return DecoderLayerFn.apply(meta, x, self.input_layernorm.weight, a.q_proj.weight, a.k_proj.weight,
                                    a.v_proj.weight, a.o_proj.weight, self.post_attention_layernorm.weight,
                                    m.gate_proj.weight, m.up_proj.weight, m.down_proj.weight)

    def _train_meta(self, rt, qkv_grad, gu_grad, **extra):
        """DecoderLayerFn's meta; qkv_grad / gu_grad: what receives the fused weights' gradients (see `params`)."""
        a, m = self.self_attn, self.mlp
        return dict(nh=self.nh, nkv=self.nkv, hd=self.hd, eps=self.input_layernorm.variance_epsilon,
                    hf_cast=rt["hf_cast"], cos=rt["cos"], sin=rt["sin"], pos=rt["pos"], kmask=rt["kmask"],
                    recompute=rt["recompute"], **extra,
                    params=(self.input_layernorm.weight, qkv_grad, a.o_proj.weight, self.post_attention_layernorm.weight,
                            gu_grad, m.down_proj.weight))

    @torch.no_grad()
    def infer(self, x, rt, cache):
        """KV-cache path (prefill and decode): same kernels, K/V appended to the per-layer cache.  cache=None: causal
        attention over the sequence itself (no-grad forward of a quantised model).  Quantised layers (NF4, int8 or FP8) run
        their projections through the format's projection objects (`linear` / `gate_up`)."""
        a, m = self.self_attn, self.mlp
        qp = self._quantized()
        if qp is None:
            qkv_w, gu_w, _, _ = self._fused()
        B, S, H = x.shape
        nh, nkv, hd = self.nh, self.nkv, self.hd
        rows = B * S
        x2 = x.reshape(rows, H)
        h = ops.rmsnorm_fwd(x2, self.input_layernorm.weight, self.input_layernorm.variance_epsilon, rt["hf_cast"])
        qkv = qp["qkv"].linear(h) if qp is not None else ops.gemm(h, qkv_w)
        ops.rope_(qkv, rt["pos"], rt["cos"], rt["sin"], nh + nkv, hd)
        q = qkv[:, : nh * hd].view(B, S, nh, hd)
        k_new = qkv[:, nh * hd:(nh + nkv) * hd].view(B, S, nkv, hd)
        v_new = qkv[:, (nh + nkv) * hd:].view(B, S, nkv, hd)
        win = {"window": self.window} if self.window else {}
        if cache is None:
            attn = ops.attn_fwd(q, k_new, v_new, causal=True, kmask=rt["kmask"], **win)
        elif isinstance(cache, PagedCacheView):
            attn = self._attn_paged_cache(q, k_new, v_new, cache, rt["kmask"])
        elif cache.fp8 is not None:
            attn = self._attn_fp8_cache(q, k_new, v_new, cache, rt["kmask"])
        elif cache.slot is not None:
            # static-shape decode step (CUDA-graph replay): the write slot is a DEVICE index, attention runs over the whole
            # cache buffer and the validity mask (updated on the device) hides the slots not written yet and, with a
            # sliding window, the ones that have left it
            kc, vc = cache.k[self.layer_idx], cache.v[self.layer_idx]
            kc.index_copy_(1, cache.slot, k_new)
            vc.index_copy_(1, cache.slot, v_new)
            attn = ops.attn_fwd(q, kc, vc, causal=False, kmask=rt["kmask"])
        else:
            kc, vc = cache.k[self.layer_idx], cache.v[self.layer_idx]
            t0 = cache.length
            kc[:, t0:t0 + S].copy_(k_new)   # cache append (memory plumbing)
            vc[:, t0:t0 + S].copy_(v_new)
            attn = ops.attn_fwd(q, kc[:, : t0 + S], vc[:, : t0 + S], causal=True, kmask=rt["kmask"], **win)
        attn2 = attn.view(rows, nh * hd)
        if qp is not None:
            x1 = qp["o"].linear(attn2, residual=x2)
        else:
            x1 = ops.gemm(attn2, a.o_proj.weight, residual=x2)
        h2 = ops.rmsnorm_fwd(x1, self.post_attention_layernorm.weight, self.post_attention_layernorm.variance_epsilon,
                             rt["hf_cast"])
        if qp is not None:
            _, act = qp["gate_up"].gate_up(h2)
            return qp["down"].linear(act, residual=x1).view(B, S, H)
        _, act = ops.mlp_gate_up(h2, gu_w)
        return ops.gemm(act, m.down_proj.weight, residual=x1).view(B, S, H)

    def _attn_fp8_cache(self, q, k_new, v_new, cache, kmask):
        """Attention with the FP8 cache (kv_fp8.py): the prompt attends over its own bf16 K / V and is then appended; a
        decode step appends its row, then attends over the quantised cache up to and including it."""
        kq, vq, ks, vs = cache.fp8.layer(self.layer_idx)
        S = q.shape[1]
        if cache.slot is None and cache.length == 0:
            attn = ops.attn_fwd(q, k_new, v_new, causal=True, kmask=kmask)
            ops.kv_fp8_append(k_new, v_new, kq, vq, ks, vs, offset=0)
            return attn
        if S != 1:
            raise NotImplementedError("an FP8 KV cache takes a prompt into an empty cache or one token per decode step, "
                                      f"not {S} tokens after {cache.length} cached positions")
        if cache.slot is not None:       # graph-replayed step: write slot and valid length come from the device slot
            ops.kv_fp8_append(k_new, v_new, kq, vq, ks, vs, offset=0, offset_dev=cache.slot)
            return ops.attn_decode_fp8(q, kq, vq, ks, vs, cache.fp8.ws, length=1, length_dev=cache.slot, kmask=kmask)
        t0 = cache.length
        ops.kv_fp8_append(k_new, v_new, kq, vq, ks, vs, offset=t0)
        return ops.attn_decode_fp8(q, kq, vq, ks, vs, cache.fp8.ws, length=t0 + 1, kmask=kmask)

    def _attn_paged_cache(self, q, k_new, v_new, cache, kmask):
        """Attention with the paged cache (paged_kv.py): a prefill attends over its own bf16 K / V and is then appended
        into its empty pages; a decode step appends each row's token at lens[b], then attends over its pages.  A prefill
        after a cached prefix of P positions (a prefix-cache hit of the server) gathers [0, P) out of the pages into bf16
        rows, puts its own bf16 K / V after them, attends over both (causal, aligned bottom-right) and appends at P."""
        kp, vp, ksc, vsc = cache.pool.layer(self.layer_idx)
        if cache.prefill:
            P = cache.prefix
            if P:
                kb, vb = cache.prefix_buffers(k_new.shape[1], self.nkv, self.hd, q.device)
                ops.paged_kv_gather(kp, vp, ksc, vsc, cache.table[0], P, kb, vb)
                kb[:, P:].copy_(k_new)
                vb[:, P:].copy_(v_new)
                attn = ops.attn_fwd(q, kb, vb, causal=True, kmask=kmask)
            else:
                attn = ops.attn_fwd(q, k_new, v_new, causal=True, kmask=kmask)
            ops.paged_kv_append(k_new, v_new, kp, vp, ksc, vsc, cache.table, offset=P)
            return attn
        ops.paged_kv_append(k_new, v_new, kp, vp, ksc, vsc, cache.table, cache.lens, offset_from_lens=True)
        return ops.attn_decode_paged(q, kp, vp, ksc, vsc, cache.table, cache.lens, cache.pool.ws, len_add=1)


class KVCache:
    """Per-layer [B, S_max, n_kv, head_dim] bf16 buffers (the layout the attention kernel's TMA maps address), or with
    dtype="fp8" the E4M3 rows and fp32 scales of kv_fp8.py plus the decode workspace (`fp8`)."""

    def __init__(self, config, batch, max_len, device, dtype="bf16"):
        from ...kv_fp8 import CACHE_DTYPES, Fp8KVLayers
        if dtype not in CACHE_DTYPES:
            raise ValueError(f"KVCache dtype {dtype!r} is not supported: use one of {CACHE_DTYPES}")
        nkv = config.num_key_value_heads
        hd = getattr(config, "head_dim", None) or config.hidden_size // config.num_attention_heads
        L = config.num_hidden_layers
        self.dtype = dtype
        self.fp8 = None
        if dtype == "fp8":
            self.k = self.v = None
            self.fp8 = Fp8KVLayers(L, batch, max_len, config.num_attention_heads, nkv, hd, device)
        else:
            # zero-initialised: the static-shape decode step attends over the WHOLE buffer with not-yet-written slots
            # masked out — their probabilities are exactly 0, but 0 x (uninitialised NaN / Inf bit patterns in V) would
            # still be NaN
            self.k = [torch.zeros((batch, max_len, nkv, hd), dtype=torch.bfloat16, device=device) for _ in range(L)]
            self.v = [torch.zeros((batch, max_len, nkv, hd), dtype=torch.bfloat16, device=device) for _ in range(L)]
        self.length = 0
        self.max_len = max_len
        self.kmask = None  # [B, max_len] bool, key validity over the whole cache
        self.slot = None   # device int64 [1]: write position of a static-shape (graph-replayed) decode step

    def get_seq_length(self):
        return self.length

    def nbytes(self) -> int:
        """Device bytes the cache holds (for fp8: rows, scales and the decode workspace)."""
        if self.fp8 is not None:
            return self.fp8.nbytes()
        return sum(t.numel() * t.element_size() for t in self.k + self.v)


class CambrianPreTrainedModel(PreTrainedModel):
    config_class = CambrianConfig
    base_model_prefix = "model"
    supports_gradient_checkpointing = True
    _no_split_modules = ["CBLlamaDecoderLayer"]

    def _init_weights(self, module):
        """HF LlamaPreTrainedModel._init_weights.  transformers >= 5 re-runs this over every module AFTER loading a
        checkpoint and relies on the guarded initialisers (they skip parameters flagged `_is_hf_initialized`); writing
        through `.data` here would overwrite freshly loaded weights."""
        std = getattr(self.config, "initializer_range", 0.02)

        def normal_(p):
            if getattr(p, "_is_hf_initialized", False):
                return
            if _hf_init is not None:
                _hf_init.normal_(p, mean=0.0, std=std)
            else:
                with torch.no_grad():
                    p.normal_(mean=0.0, std=std)

        if isinstance(module, nn.Linear):
            normal_(module.weight)
            if module.bias is not None and not getattr(module.bias, "_is_hf_initialized", False):
                with torch.no_grad():
                    module.bias.zero_()
        elif isinstance(module, nn.Embedding):
            normal_(module.weight)


class CBLlamaModel(CambrianPreTrainedModel):
    decoder_layer_cls = CBLlamaDecoderLayer

    def __init__(self, config):
        super().__init__(config)
        self.padding_idx = getattr(config, "pad_token_id", None)
        self.vocab_size = config.vocab_size
        self.embed_tokens = nn.Embedding(config.vocab_size, config.hidden_size, self.padding_idx)
        self.layers = nn.ModuleList([self.decoder_layer_cls(config, i) for i in range(config.num_hidden_layers)])
        self.norm = CBRMSNorm(config.hidden_size, eps=config.rms_norm_eps)
        self.gradient_checkpointing = False
        self._rope = None


class CambrianLlamaModel(CambrianMetaModel, CBLlamaModel):
    config_class = CambrianConfig

    def __init__(self, config):
        super(CambrianLlamaModel, self).__init__(config)

    def _rope_tables(self, device):
        if self._rope is None or self._rope[0].device != device:
            self._rope = rope_tables(self.config, device)
        return self._rope

    def forward(self, input_ids=None, attention_mask=None, position_ids=None, past_key_values=None, inputs_embeds=None,
                use_cache=None, output_attentions=None, output_hidden_states=None, return_dict=None,
                vision_tower_aux_feature_list=None, vision_tower_aux_attention_masks_list=None,
                final_vision_feature_size=None, global_context_feature=None):
        """cambrian_llama.py:57-277 (static SVA-insertion branch :168-207)."""
        if output_attentions:
            raise NotImplementedError("output_attentions is not available with the fused attention kernel")
        if input_ids is not None and inputs_embeds is not None:
            raise ValueError("You cannot specify both input_ids and inputs_embeds at the same time")
        cfg = self.config
        if inputs_embeds is None:
            if input_ids is None:
                raise ValueError("You have to specify either input_ids or inputs_embeds")
            meta = dict(ids=input_ids.contiguous(), img_start=None, q_side=1, params=(self.embed_tokens.weight, None))
            from ...autograd import EmbedSpliceFn
            inputs_embeds = EmbedSpliceFn.apply(meta, self.embed_tokens.weight, None, None)
        B, S, H = inputs_embeds.shape
        dev = inputs_embeds.device
        cache = past_key_values if isinstance(past_key_values, (KVCache, PagedCacheView)) else None
        if use_cache and cache is None:
            raise ValueError("use_cache=True needs a cambrian_b200 KVCache in past_key_values (see generate())")
        past = cache.length if cache is not None else 0
        if position_ids is None:
            position_ids = torch.arange(past, past + S, dtype=torch.long, device=dev).unsqueeze(0).expand(B, S)
        pos = position_ids.to(torch.long).expand(B, S).contiguous().view(-1)
        cos, sin = self._rope_tables(dev)
        kmask = None
        if cache is not None:
            if cache.slot is not None:
                kmask = cache.kmask                      # whole buffer; the mask itself is advanced on the device
            elif cache.kmask is not None:
                kmask = cache.kmask[:, : past + S].contiguous()
        elif attention_mask is not None:
            kmask = attention_mask.bool().contiguous()
        rt = dict(pos=pos, cos=cos, sin=sin, kmask=kmask, hf_cast=not self.training,
                  recompute=bool(self.gradient_checkpointing and self.training), fp8=train_fp8.enabled(cfg))
        sites = []
        if not getattr(cfg, "connector_only", True) and vision_tower_aux_feature_list is not None:
            sites = [cfg.start_of_vision_sampler_layers + k * cfg.stride_of_vision_sampler_layers
                     for k in range(len(self.vision_sampler_layers))]
        q_num = getattr(cfg, "image_token_len", 576)
        q_side = int(q_num ** 0.5)
        hidden = inputs_embeds.contiguous()
        all_hidden = () if output_hidden_states else None
        z3 = getattr(self, "_zero3", None)
        for i, layer in enumerate(self.layers):
            if output_hidden_states:
                all_hidden += (hidden,)
            if z3 is not None:
                z3.before_layer(i)                      # ZeRO-3 inference: weights of layer i resident, i+1 in flight
            hidden = layer.infer(hidden, rt, cache) if cache is not None else layer(hidden, rt)
            if i in sites and isinstance(vision_tower_aux_feature_list, WindowedFeatures):
                # per-sample unpadded query grids (cambrian_llama.py:208-253), inference only: the latent queries of
                # every sample are gathered into one ragged batch, updated by the SVA layer, scattered back in place
                if torch.is_grad_enabled() and hidden.requires_grad:
                    raise NotImplementedError("the dynamic-shape SVA branch is inference-only")
                start = cfg.image_position
                sizes = [(int(h), int(w)) for (h, w) in final_vision_feature_size]
                lats = [ops.span_gather_hw(hidden[b:b + 1], start, h, w) for b, (h, w) in enumerate(sizes)]
                lat = lats[0] if len(lats) == 1 else torch.cat(lats, 0)
                feats = [f.to(lat.dtype) for f in vision_tower_aux_feature_list]
                masks = vision_tower_aux_attention_masks_list or [None] * len(feats)
                lat = self.vision_sampler_layers[sites.index(i)](
                    lat.view(lat.shape[0], 1, H), global_context_feature, *feats, *masks)
                lat = lat.view(-1, H)
                o = 0
                for b, (h, w) in enumerate(sizes):
                    ops.span_scatter_hw_(hidden[b:b + 1], lat[o:o + h * w], start, h, w)
                    o += h * w
            elif i in sites:
                start = cfg.image_position                                                      # :175
                n = B * q_num
                lat, hidden = SpanSplitFn.apply(hidden, start, q_side)
                feats = [f.to(lat.dtype) for f in vision_tower_aux_feature_list]
                masks = vision_tower_aux_attention_masks_list or [None] * len(feats)
                lat = self.vision_sampler_layers[sites.index(i)](
                    lat.view(n, 1, H), global_context_feature, *feats, *masks, natural_layout=(B, q_side))
                hidden = SpanMergeFn.apply(hidden, lat.view(n, H), start, q_side)
        if cache is not None and cache.slot is None:
            cache.length = past + S
        hidden = self.norm(hidden, hf_cast=not self.training)
        if output_hidden_states:
            all_hidden += (hidden,)
        if return_dict is False:
            return tuple(v for v in [hidden, cache, all_hidden] if v is not None)
        return BaseModelOutputWithPast(last_hidden_state=hidden, past_key_values=cache, hidden_states=all_hidden)


class _CELossFn(torch.autograd.Function):
    """Shifted cross-entropy on materialised bf16 logits (API-compat path; training uses the fused LMHeadLossFn)."""

    @staticmethod
    def forward(ctx, logits2d, shift_labels, n_valid, inv_dev):
        buf = logits2d.clone()
        rows = buf.shape[0]
        loss_rows = torch.empty(rows, dtype=torch.float32, device=buf.device)
        acc = torch.zeros(2, dtype=torch.float32, device=buf.device)
        if n_valid is not None:
            ops.cross_entropy(buf, shift_labels, loss_rows, acc, 1.0 / max(n_valid, 1), True)
            loss = acc[0] / max(n_valid, 1)
        else:       # count of valid labels stays on the device
            ops.cross_entropy(buf, shift_labels, loss_rows, acc, 1.0, True, scale_dev=inv_dev)
            loss = acc[0] * inv_dev[0]
        ctx.save_for_backward(buf)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        return ctx.saved_tensors[0] * dloss.to(ctx.saved_tensors[0].dtype), None, None, None


class CambrianLlamaForCausalLM(CambrianPreTrainedModel, CambrianMetaForCausalLM):
    config_class = CambrianConfig
    _tied_weights_keys = {}

    def __init__(self, config):
        super().__init__(config)
        self.model = CambrianLlamaModel(config)
        self.vocab_size = config.vocab_size
        self.lm_head = nn.Linear(config.hidden_size, config.vocab_size, bias=False)
        self.post_init()

    def get_model(self):
        return self.model

    def attention_window(self) -> int:
        """Causal sliding window of the decoder's attention (0: none)."""
        return 0

    def save_pretrained(self, *args, **kwargs):
        from ...quant import quantized_format
        fmt = quantized_format(self)
        if fmt is not None:
            raise NotImplementedError(f"save_pretrained of a {fmt} model is not supported: its decoder projections "
                                      "hold no bf16 weights; save the bf16 checkpoint it was loaded from instead")
        return super().save_pretrained(*args, **kwargs)

    def get_input_embeddings(self):
        return self.model.embed_tokens

    def get_output_embeddings(self):
        return self.lm_head

    def forward(self, input_ids: torch.LongTensor = None, attention_mask: Optional[torch.Tensor] = None,
                position_ids: Optional[torch.LongTensor] = None, past_key_values=None,
                inputs_embeds: Optional[torch.FloatTensor] = None, labels: Optional[torch.LongTensor] = None,
                use_cache: Optional[bool] = None, output_attentions: Optional[bool] = None,
                output_hidden_states: Optional[bool] = None, images: Optional[List[torch.Tensor]] = None,
                image_aux_attention_masks_list: Optional[List[torch.Tensor]] = None,
                image_sizes: Optional[List[List[int]]] = None, return_dict: Optional[bool] = None,
                cache_position=None, num_valid_labels: Optional[int] = None,
                image_positions: Optional[List[int]] = None, label_ranges=None, **kw):
        """cambrian_llama.py:297-434.  Extensions (host-side hints the collator already has; both avoid a device->host
        sync per step): `num_valid_labels` = number of non-ignored shifted labels, `image_positions` = index of the
        <image> indicator per sample of an already-expanded batch; `label_ranges` = host list of (row_start, row_end) over
        the flattened [B*S] positions outside of which every SHIFTED label is ignore_index (train/collator.py:
        valid_label_ranges) — the fused loss then skips the vocabulary GEMMs of rows that cannot contribute."""
        feats = masks = final_size = ctx_feat = None
        if inputs_embeds is None:
            (input_ids, position_ids, attention_mask, past_key_values, inputs_embeds, labels, feats, masks, final_size,
             ctx_feat) = self.prepare_inputs_labels_for_multimodal(
                input_ids, position_ids, attention_mask, past_key_values, labels, images, image_aux_attention_masks_list,
                image_sizes, image_positions=image_positions)
        out = self.model(input_ids=input_ids, attention_mask=attention_mask, position_ids=position_ids,
                         past_key_values=past_key_values, inputs_embeds=inputs_embeds, use_cache=use_cache,
                         output_attentions=output_attentions, output_hidden_states=output_hidden_states, return_dict=True,
                         vision_tower_aux_feature_list=feats, vision_tower_aux_attention_masks_list=masks,
                         final_vision_feature_size=final_size, global_context_feature=ctx_feat)
        hidden = out.last_hidden_state
        B, S, H = hidden.shape
        loss = logits = None
        fused = bool(getattr(self.config, "fused_lm_loss", False))
        shift = None
        inv_count_dev = None
        if labels is not None:
            shift = torch.full_like(labels, IGNORE_INDEX)
            shift[:, :-1] = labels[:, 1:]
            shift = shift.reshape(-1).contiguous()
            if num_valid_labels is None:
                # mean over non-ignored labels (:411-422): the count stays on the device (no host sync per step)
                cnt = ((shift != IGNORE_INDEX) & (shift >= 0) & (shift < self.vocab_size)).sum()
                inv_count_dev = (1.0 / cnt.clamp(min=1).float()).reshape(1)
        if labels is not None and fused:
            # gradients are formed inside the fused forward: only when something will consume them (training mode, or no
            # TrainEngine buffers to write into) — an eval pass with labels under grad mode must not touch main_grad
            train = torch.is_grad_enabled() and (self.training or getattr(self.lm_head.weight, "main_grad", None) is None)
            meta = dict(shift_labels=shift, n_valid=num_valid_labels, train=train,
                        params=(self.lm_head.weight,), chunk=getattr(self.config, "lm_loss_chunk", 4096),
                        label_ranges=label_ranges, loss_scale=getattr(self, "_cb_loss_scale", 1.0),
                        inv_count_dev=inv_count_dev)
            loss = LMHeadLossFn.apply(meta, hidden, self.lm_head.weight)
        else:
            logits_bf16 = LinearFn.apply(hidden, self.lm_head.weight, None)                     # :408
            if labels is not None:
                loss = _CELossFn.apply(logits_bf16.view(B * S, -1), shift, num_valid_labels, inv_count_dev)   # :411-422
            logits = logits_bf16.float()                                                        # :409
        if return_dict is False:
            return tuple(v for v in (loss, logits, out.past_key_values) if v is not None)
        return CausalLMOutputWithPast(loss=loss, logits=logits, past_key_values=out.past_key_values,
                                      hidden_states=out.hidden_states)

    @torch.no_grad()
    def generate(self, inputs: Optional[torch.Tensor] = None, images: Optional[torch.Tensor] = None,
                 image_sizes: Optional[torch.Tensor] = None, **kwargs):
        """cambrian_llama.py:437-483: multimodal prefill once (towers + connector + SVA sites), then KV-cache decoding.

        The reference hands `inputs_embeds` to HF `GenerationMixin.generate`; the subset of that API its callers use is
        implemented here (cambrian_b200/generation.py): greedy or temperature / top-k / top-p sampling, `eos_token_id`,
        `pad_token_id`, `max_new_tokens` / `max_length`, `stopping_criteria`, `streamer`, `attention_mask`,
        `position_ids`, `generation_config`, `generator`.  Any other keyword is rejected unless it carries its neutral
        value (num_beams=1, use_cache=True, ...).  Returns the newly generated ids [B, T], as HF does when generation
        starts from `inputs_embeds`.

        `kv_cache_dtype` ("bf16" or "fp8", default `config.kv_cache_dtype` or "bf16") selects the decode KV cache:
        "fp8" keeps it in E4M3 with per-row scales (cambrian_b200/kv_fp8.py), about half the bytes of bf16."""
        from ...generation import next_tokens, should_stop
        from ...kv_fp8 import resolve_cache_dtype
        if "inputs_embeds" in kwargs:
            raise NotImplementedError("`inputs_embeds` is not supported")                       # :447-448
        kv_dtype = resolve_cache_dtype(self.config, kwargs.pop("kv_cache_dtype", None))
        z3 = getattr(self.get_model(), "_zero3", None)
        if z3 is not None and kv_dtype == "fp8":
            raise NotImplementedError("kv_cache_dtype='fp8' is not supported with Zero3Inference")
        sync = getattr(self, "_cb_param_sync", None)
        if sync is not None:
            sync()      # a TrainEngine with deferred parameter sync: inference kernels read parameters directly
        attention_mask = kwargs.pop("attention_mask", None)
        position_ids = kwargs.pop("position_ids", None)
        was_training = self.training
        self.eval()
        args, cache, h_last, next_pos, S0 = self._prefill(
            inputs, images, image_sizes, attention_mask, position_ids, kwargs,
            lambda B, S0, max_new: KVCache(self.config, B, S0 + max_new, inputs.device, dtype=kv_dtype))
        B = inputs.shape[0]
        max_new = args.max_new_tokens
        dev = inputs.device
        done = torch.zeros(B, dtype=torch.bool, device=dev)
        check_stop = bool(args.eos_token_ids or args.stopping_criteria)
        if args.streamer is not None:
            args.streamer.put(torch.empty((B, 0), dtype=torch.long))     # HF streams the (here: empty) prompt ids first
        if (_DECODE_GRAPH and z3 is None and max_new > 2 and h_last.is_cuda
                and not getattr(self.config, "disable_decode_graph", False)):
            toks = self._generate_graphed(args, cache, h_last, next_pos, S0, max_new, check_stop)
            self.train(was_training)
            return toks
        tokens = []
        for step in range(max_new):
            logits = ops.gemm(h_last, self.lm_head.weight, out_dtype=torch.float32)             # fp32 logits (:409)
            nxt = next_tokens(logits, args)
            nxt = torch.where(done, torch.full_like(nxt, args.pad_token_id), nxt)
            tokens.append(nxt)
            if args.streamer is not None:
                args.streamer.put(nxt.cpu())
            if check_stop:
                done = should_stop(args, torch.stack(tokens, 1), logits, done)
                if (z3.all_done(done) if z3 is not None else bool(done.all())):
                    break
            if step + 1 == max_new:
                break
            out = self.model(input_ids=nxt.view(B, 1), position_ids=next_pos.view(B, 1), past_key_values=cache,
                             use_cache=True)
            h_last = out.last_hidden_state[:, 0].contiguous()
            next_pos = next_pos + 1
        if args.streamer is not None:
            args.streamer.end()
        self.train(was_training)
        return torch.stack(tokens, 1)

    def _prefill(self, inputs, images, image_sizes, attention_mask, position_ids, kwargs, make_cache, prefix: int = 0):
        """The prefill of generate() and of serving.BatchedGenerator: multimodal preparation (towers, connector, splice),
        the generation keywords (GenerationArgs, which needs the spliced prompt length S0), the cache from
        make_cache(B, S0, max_new_tokens), the prefill forward over it, and each row's last hidden state and next
        position.  Returns (args, cache, h_last [B, H], next_pos [B], S0).

        prefix > 0 (the server's prefix-cache hit): the cache already holds positions [0, prefix) of the one sequence and
        `inputs` are the text ids of positions prefix .. S0-1 (S0 = prefix + n), so no image preparation runs; the
        keywords and the cache mask see the whole S0."""
        from ...generation import GenerationArgs
        if prefix and (images is not None or attention_mask is not None or position_ids is not None
                       or inputs.shape[0] != 1):
            raise ValueError("a prefill after a cached prefix takes one unpadded text-only sequence")
        feats = masks = final_size = ctx_feat = None
        if images is not None:
            (_, position_ids, attention_mask, _, inputs_embeds, _, feats, masks, final_size, ctx_feat) = \
                self.prepare_inputs_labels_for_multimodal(inputs, position_ids, attention_mask, None, None, images,
                                                          image_sizes=image_sizes)
        else:
            inputs_embeds = None
        B = inputs.shape[0]
        n = inputs_embeds.shape[1] if inputs_embeds is not None else inputs.shape[1]
        S0 = prefix + n
        args = GenerationArgs.from_kwargs(self, S0, kwargs)
        max_new = args.max_new_tokens
        dev = inputs.device
        cache = make_cache(B, S0, max_new)
        cache.kmask = torch.ones((B, S0 + max_new), dtype=torch.bool, device=dev)
        if attention_mask is not None:
            cache.kmask[:, :S0] = attention_mask.bool()
            if position_ids is None:
                position_ids = (attention_mask.long().cumsum(1) - 1).clamp_(min=0)
        out = self.model(input_ids=None if inputs_embeds is not None else inputs, inputs_embeds=inputs_embeds,
                         position_ids=position_ids, past_key_values=cache, use_cache=True,
                         vision_tower_aux_feature_list=feats, vision_tower_aux_attention_masks_list=masks,
                         final_vision_feature_size=final_size, global_context_feature=ctx_feat)
        last_idx = (cache.kmask[:, :S0].long().cumsum(1).argmax(1)) if attention_mask is not None else \
            torch.full((B,), n - 1, device=dev)
        h_last = out.last_hidden_state[torch.arange(B, device=dev), last_idx].contiguous()
        next_pos = (position_ids.max(1).values + 1) if position_ids is not None else torch.full((B,), S0, device=dev)
        return args, cache, h_last, next_pos, S0

    def _generate_graphed(self, args, cache, h_last, next_pos, S0, max_new, check_stop):
        """Decoding with ONE CUDA graph per generate() call: a decode step is ~290 kernel launches whose device time
        (weight streaming, a few ms) is far below the cost of enqueueing them one by one from Python, so the step is captured
        once — static shapes: token / position /
        cache-slot / validity mask live in device buffers that the captured kernels advance themselves — and replayed per
        token.  EOS / stopping criteria are evaluated between replays on the host exactly as in the eager loop.  Greedy
        decoding takes the argmax; sampling runs ops.sample_tokens on per-row parameter buffers and a step buffer that
        the graph advances, so it draws the tokens the eager loop's next_tokens draws."""
        from ...generation import sampling_params, should_stop
        B = h_last.shape[0]
        dev = h_last.device
        pad = args.pad_token_id
        h_buf = h_last.clone()
        pos_buf = next_pos.view(B, 1).clone().long()
        done_buf = torch.zeros(B, dtype=torch.bool, device=dev)
        tok_buf = torch.zeros(B, dtype=torch.long, device=dev)
        logits_buf = torch.empty((B, self.lm_head.weight.shape[0]), dtype=torch.float32, device=dev)
        cache.slot = torch.full((1,), cache.length, dtype=torch.long, device=dev)
        window = self.attention_window()
        if args.do_sample:
            *params, step_buf = sampling_params(args, B, dev)
            samp_buf = torch.empty(B, dtype=torch.long, device=dev)

        def pick(logits):
            if not args.do_sample:
                return logits.argmax(-1)
            return ops.sample_tokens(logits, *params, step_buf, out=samp_buf)

        def step():
            ops.gemm(h_buf, self.lm_head.weight, out=logits_buf)                                 # fp32 logits (:409)
            nxt = pick(logits_buf)
            tok_buf.copy_(torch.where(done_buf, torch.full_like(nxt, pad), nxt))
            cache.kmask.index_fill_(1, cache.slot, True)
            if window:
                # the query at slot s sees slots s - window + 1 .. s: slot s - window leaves the window now (nothing
                # leaves while s < window); an index and a select-and-mask on the device, no host sync
                old = (cache.slot - window).clamp_(min=0)
                cache.kmask.index_copy_(1, old, cache.kmask.index_select(1, old) & (cache.slot < window))
            out = self.model(input_ids=tok_buf.view(B, 1), position_ids=pos_buf, past_key_values=cache, use_cache=True)
            h_buf.copy_(out.last_hidden_state[:, 0])
            pos_buf.add_(1)
            cache.slot.add_(1)
            if args.do_sample:
                step_buf.add_(1)

        # slots beyond the prompt start invalid; each step validates the one it writes
        cache.kmask[:, S0:] = False
        if window:
            cache.kmask[:, :max(0, S0 - window)] = False    # already outside the first step's window
        state = (h_buf, pos_buf, cache.slot, cache.kmask) + ((step_buf,) if args.do_sample else ())
        snap = tuple(t.clone() for t in state)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):                      # warm-up outside capture (lazy kernel attributes, allocator)
            step()
        torch.cuda.current_stream().wait_stream(side)
        for buf, s0 in zip(state, snap):
            buf.copy_(s0)                                  # the warm-up step advanced the state: rewind (K/V slot S0 is
        graph = torch.cuda.CUDAGraph()                     # simply rewritten with the same values)
        with torch.cuda.graph(graph):
            step()
        for buf, s0 in zip(state, snap):
            buf.copy_(s0)
        tokens = []
        for i in range(max_new):
            if i + 1 == max_new:
                # the last token needs no further decoder pass: logits -> argmax or a draw at step i (step_buf) only
                logits = ops.gemm(h_buf, self.lm_head.weight, out_dtype=torch.float32)
                nxt = pick(logits)
                tok = torch.where(done_buf, torch.full_like(nxt, pad), nxt)
            else:
                graph.replay()
                tok, logits = tok_buf.clone(), logits_buf
            tokens.append(tok)
            if args.streamer is not None:
                args.streamer.put(tok.cpu())
            if check_stop:
                done_buf.copy_(should_stop(args, torch.stack(tokens, 1), logits, done_buf))
                if bool(done_buf.all()):
                    break
        cache.length = S0 + len(tokens)
        cache.slot = None
        if args.streamer is not None:
            args.streamer.end()
        return torch.stack(tokens, 1)

    def prepare_inputs_for_generation(self, input_ids, past_key_values=None, inputs_embeds=None, **kwargs):
        images = kwargs.pop("images", None)
        image_sizes = kwargs.pop("image_sizes", None)
        d = dict(input_ids=input_ids, past_key_values=past_key_values, inputs_embeds=inputs_embeds, **kwargs)
        if images is not None:
            d["images"] = images
        if image_sizes is not None:
            d["image_sizes"] = image_sizes
        return d


AutoConfig.register("cambrian_llama", CambrianConfig)
AutoModelForCausalLM.register(CambrianConfig, CambrianLlamaForCausalLM)
