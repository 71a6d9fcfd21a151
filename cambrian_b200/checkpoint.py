"""Checkpoint compatibility with the reference (SURVEY.md §8f rank 2).

The modules in `cambrian_b200.model` own their weights under the reference's state-dict keys, so the released
`nyu-visionx/cambrian-*` checkpoints (HF `save_pretrained` layout: config.json + sharded safetensors / .bin) load through
the unchanged `PreTrainedModel.from_pretrained`.  This file adds the three reference-specific pieces around that:

  * `get_mm_adapter_state` / `save_mm_projector` — the adapter-only checkpoint written during connector pre-training
    (`safe_save_model_for_hf_trainer`, train_fsdp.py:249-283; key filter :255);
  * `load_mm_projector` — the `mm_projector.bin` overlay on top of a base LLM (model/builder.py:107-114) and the
    `pretrain_mm_mlp_adapter` path of `initialize_vision_modules` (cambrian_arch.py:183-200, strict per sub-module);
  * `load_pretrained_model` — the loader the eval / serve harness calls (model/builder.py:29-175), bf16 on one GPU, or
    with `load_4bit=True` the decoder projections in NF4 (quant.py), with `load_8bit=True` in LLM.int8
    (quant_int8.py), with `load_fp8=True` in FP8 E4M3 (quant_fp8.py).  LoRA merging raises NotImplementedError.
"""
from __future__ import annotations

import os

import torch

ADAPTER_KEYS = ["mm_projector", "pos_emb", "vision_sampler", "vision_sampler_layers", "vision_query", "image_newline"]


def get_mm_adapter_state(named_params, keys_to_match=ADAPTER_KEYS):
    """train_fsdp.py:218-226 (`get_mm_adapter_state_maybe_zero_3` without the ZeRO-3 gather): detached CPU copies of
    every parameter whose name contains one of the keys."""
    return {k: v.detach().cpu().clone() for k, v in named_params if any(m in k for m in keys_to_match)}


def save_mm_projector(model, output_dir: str, use_im_start_end: bool = False) -> str:
    keys = list(ADAPTER_KEYS) + (["embed_tokens", "embed_in"] if use_im_start_end else [])
    os.makedirs(output_dir, exist_ok=True)
    model.config.save_pretrained(output_dir)
    path = os.path.join(output_dir, "mm_projector.bin")
    torch.save(get_mm_adapter_state(model.named_parameters(), keys), path)
    return path


def _strip_wrappers(sd):
    """model/builder.py:84-86: checkpoints written through PEFT / an extra wrapper carry `base_model.` / `model.model.`"""
    sd = {(k[len("base_model."):] if k.startswith("base_model.") else k): v for k, v in sd.items()}
    if any(k.startswith("model.model.") for k in sd):
        sd = {(k[len("model."):] if k.startswith("model.") else k): v for k, v in sd.items()}
    return sd


def load_mm_projector(model, path_or_state, strict_submodules: bool = False):
    """Overlay adapter weights on an instantiated model.  strict_submodules=False reproduces builder.py:112-114
    (`load_state_dict(strict=False)` of the whole file); True reproduces cambrian_arch.py:183-200 (every connector
    sub-module must be fully covered).  Values are cast to the destination parameter's dtype."""
    sd = torch.load(path_or_state, map_location="cpu") if isinstance(path_or_state, (str, os.PathLike)) else dict(path_or_state)
    sd = _strip_wrappers(sd)
    own = model.state_dict()
    unexpected = [k for k in sd if k not in own]
    if strict_submodules:
        if unexpected:
            raise RuntimeError(f"Unexpected key(s) in adapter state: {unexpected[:8]}")
        needed = [k for k in own if any(m in k for m in ADAPTER_KEYS)]
        missing = [k for k in needed if k not in sd]
        if missing:
            raise RuntimeError(f"Missing key(s) in adapter state: {missing[:8]}")
    with torch.no_grad():
        for k, v in sd.items():
            if k in own:
                if own[k].shape != v.shape:
                    raise RuntimeError(f"size mismatch for {k}: checkpoint {tuple(v.shape)} vs model {tuple(own[k].shape)}")
                own[k].copy_(v.to(own[k].dtype))
    return unexpected


def load_pretrained_model(model_path, model_base=None, model_name="cambrian", load_8bit=False, load_4bit=False,
                          device="cuda", dtype=torch.bfloat16, load_tokenizer=True, load_fp8=False, **kwargs):
    """model/builder.py:29-175 for the LLaMA-family Cambrian checkpoints: returns (tokenizer, model, image_processor list,
    context_len).  `model_base` + `<model_path>/mm_projector.bin` is the connector-only layout (:103-114).
    load_4bit=True (:37-44): the checkpoint loads in bf16 on the CPU, the seven projections of every decoder layer are
    quantised to NF4 layer by layer on `device` (quant.quantize_decoder_nf4_), everything else moves there in bf16.
    load_8bit=True (:35-36) does the same with LLM.int8 weights (quant_int8.quantize_decoder_int8_) and takes precedence
    over load_4bit.  load_fp8=True (no reference counterpart) does the same with FP8 E4M3 weights
    (quant_fp8.quantize_decoder_fp8_); it names one format, so combining it with load_4bit or load_8bit is a ValueError."""
    from transformers import AutoConfig, AutoTokenizer

    from .model.language_model.cambrian_llama import CambrianLlamaForCausalLM
    if load_fp8 and (load_4bit or load_8bit):
        raise ValueError("load_fp8 cannot be combined with load_4bit or load_8bit: choose one weight format")
    if load_fp8 and torch.device(device).type == "cuda" and not torch.cuda.is_available():
        # fail before the bf16 checkpoint is read into host memory: the FP8 kernels exist for the GPU only
        raise NotImplementedError("8-bit (FP8) weights run on CUDA only and no CUDA device is available")
    if load_8bit and torch.device(device).type == "cuda" and not torch.cuda.is_available():
        # fail before the bf16 checkpoint is read into host memory: the int8 kernels exist for the GPU only
        raise NotImplementedError("8-bit (LLM.int8) weights run on CUDA only and no CUDA device is available")
    if "lora" in model_name.lower():
        raise NotImplementedError("LoRA merging (builder.py:56-92) is outside the hot path: merge with the reference tools first")
    if "mistral" in model_name.lower() or "phi3" in model_name.lower():
        raise NotImplementedError("only the LLaMA-family Cambrian models (8B / 13B / 34B) are implemented")
    tok_src = model_base if model_base is not None else model_path
    tokenizer = AutoTokenizer.from_pretrained(tok_src, use_fast=False) if load_tokenizer else None
    if model_base is not None:
        cfg = AutoConfig.from_pretrained(model_path)
        model = CambrianLlamaForCausalLM.from_pretrained(model_base, config=cfg, torch_dtype=dtype, **kwargs)
        load_mm_projector(model, os.path.join(model_path, "mm_projector.bin"))
    else:
        model = CambrianLlamaForCausalLM.from_pretrained(model_path, torch_dtype=dtype, **kwargs)
    if load_fp8:
        from .quant_fp8 import quantize_decoder_fp8_
        quantize_decoder_fp8_(model, device)
    elif load_8bit:                                 # takes precedence over load_4bit, as in builder.py:35-38
        from .quant_int8 import quantize_decoder_int8_
        quantize_decoder_int8_(model, device)
    elif load_4bit:
        from .quant import quantize_decoder_nf4_
        quantize_decoder_nf4_(model, device)
    model.to(device=device, dtype=dtype)
    towers = model.get_vision_tower_aux_list() or []
    for t in towers:
        if not t.is_loaded:
            t.load_model()
        t.to(device=device, dtype=dtype)
    image_processor = [t.image_processor for t in towers]
    context_len = getattr(model.config, "max_sequence_length", 2048)
    return tokenizer, model, image_processor, context_len
