#!/usr/bin/env python
"""bench.py — Cambrian-1 training-step throughput on N x H100 (BASELINE.json metric) + roofline + CPU baseline.

    python bench.py --gpus N --steps K --warmup W                    # this framework (hand-written sm_90a kernels)
    python bench.py --impl reference --gpus N --steps K --warmup W   # the reference algorithm on the host cores
    python bench.py --config {8b-ddp,7b-clip-mlp,13b-zero2} ...      # BASELINE.json configs 3, 2, 4
    python bench.py --config 8b-release                              # the released 8B recipe's towers / grids (not a BASELINE config)
    python bench.py ... --dump-outputs DIR                           # also write the last timed step's results as .npy

Workloads (SURVEY.md §8d):
  3b-ddp       the default: the 8b-ddp vision stack (four towers, SVA connector + 10 in-LLM SVA layers) on a
               Llama-3.2-3B-shaped decoder (28 L, H 3072, 24/8 heads x 128, FFN 8192, vocab 128256), seq 2048, per-layer
               recompute: the largest Cambrian training step whose fp32 master weights + AdamW state (16 B per trainable
               parameter, ~62 GB) fit one 80 GB H100.  The 8B / 7B decoders need ~128 / ~112 GB of such state per GPU
               under DDP, so 8b-ddp and 7b-clip-mlp run on GPUs with more memory than an H100 has.
  8b-ddp       config 3 — Llama-3-8B decoder (32 L, H 4096, 32/8 heads x 128, FFN 14336, vocab 128256), four towers
               (SigLIP-SO400M/14@384, CLIP ViT-L/14@336, DINOv2 ViT-L/14@336, ConvNeXt-XXL@1024 — each interpolated to 576
               tokens), SVA connector depth 3 + 10 in-LLM SVA layers (start 0, stride 3), image_position 91, 576 visual
               tokens + 24 newlines spliced into a 2048-token sequence; DDP: bucketed NCCL all-reduce of the gradients.
  7b-clip-mlp  config 2 — single CLIP ViT-L/14@336 tower + `mlp2x_gelu` projector into a Vicuna-7B-shaped MHA decoder
               (32 L, H 4096, 32 heads x 128, FFN 11008, vocab 32000), seq 1024, no SVA anywhere.
  13b-zero2    config 4 — Vicuna-13B-shaped decoder (40 L, H 5120, 40 heads, FFN 13824), 4 towers, SVA (stride 4),
               ZeRO-2: per-bucket reduce-scatter, sharded fp32 master / Adam state, in-place all-gather (needs >= 2 GPUs).
  8b-release   the released Cambrian-1-8B recipe (scripts/cambrian/finetune_cambrian_8b.sh:17-29): DINOv2-giant@378 (SwiGLU
               FFN) instead of ViT-L, ConvNeXt-XXL multi-stage (4 stages -> 96 x 96 x 5760 = 9216 tokens), SVA grids
               [576, 576, 576, 9216] (16-key windows on the ConvNeXt grid, learned pos_embed), per-layer activation
               recompute as the recipe's `--gradient_checkpointing True`.  Not a BASELINE.json config: no CPU arm.
All: bf16 compute with fp32 master weights + AdamW (lr 4e-5, wd 0) and gradient clipping at max_grad_norm 1.0 (HF
Trainer's default, active in every reference script), random-init weights, synthetic images / ids (no network).
One "step" = towers fwd + (connector + decoder + loss) fwd/bwd + gradient collective + clip + AdamW on one micro-batch per
GPU.  Weak scaling: the per-GPU micro-batch is fixed; `value` is whole-job samples/s.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "train_samples_per_sec"
UNIT = "samples/s"

# algorithmic forward TFLOP per sample of the frozen towers (BASELINE.md §2)
TOWER_TF = {"siglip": 0.665, "clip": 0.381, "dino": 0.381, "convnext1024": 6.335}
TOWER_TF_RELEASE = {"siglip": 0.665, "clip": 0.381, "dino_giant378": 1.78, "convnext1024": 6.335}   # SURVEY.md §8d deltas

LLMS = {
    "llama3-8b": dict(hidden_size=4096, intermediate_size=14336, num_hidden_layers=32, num_attention_heads=32,
                      num_key_value_heads=8, vocab_size=128256, max_position_embeddings=8192, rope_theta=500000.0,
                      rms_norm_eps=1e-5),
    "vicuna-7b": dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32,
                      num_key_value_heads=32, vocab_size=32000, max_position_embeddings=4096, rope_theta=10000.0,
                      rms_norm_eps=1e-5),
    "vicuna-13b": dict(hidden_size=5120, intermediate_size=13824, num_hidden_layers=40, num_attention_heads=40,
                       num_key_value_heads=40, vocab_size=32000, max_position_embeddings=4096, rope_theta=10000.0,
                       rms_norm_eps=1e-5),
    "llama3.2-3b": dict(hidden_size=3072, intermediate_size=8192, num_hidden_layers=28, num_attention_heads=24,
                        num_key_value_heads=8, vocab_size=128256, max_position_embeddings=8192, rope_theta=500000.0,
                        rms_norm_eps=1e-5),
    "small": dict(hidden_size=1024, intermediate_size=2048, num_hidden_layers=4, num_attention_heads=8,
                  num_key_value_heads=2, vocab_size=8192, max_position_embeddings=8192, rope_theta=500000.0,
                  rms_norm_eps=1e-5),
}
FOUR_TOWERS = ["siglip/CLIP-ViT-SO400M-14-384", "openai/clip-vit-large-patch14-336", "facebook/dinov2-large-res336",
               "clip-convnext-XXL"]
RELEASE_TOWERS = ["siglip/CLIP-ViT-SO400M-14-384", "openai/clip-vit-large-patch14-336", "facebook/dinov2-giant-res378",
                  "clip-convnext-XXL-multi-stage"]
CONFIGS = {
    "3b-ddp": dict(llm="llama3.2-3b", towers=FOUR_TOWERS, res=[384, 336, 336, 1024], sva=True, stride=3, n_sva=10,
                   image_position=91, seq=2048, micro_batch=4, zero=0, recompute=1, baseline_config=None,
                   tower_tf=sum(TOWER_TF.values()),
                   workload="Cambrian-1 train step on one H100: 4 towers (SigLIP-SO400M@384, CLIP-L@336, DINOv2-L@336, "
                            "ConvNeXt-XXL@1024) -> SVA (3 + 10 layers) -> Llama-3.2-3B-shaped decoder, 576 vis-tok, seq 2048, "
                            "per-layer recompute"),
    "8b-release": dict(llm="llama3-8b", towers=RELEASE_TOWERS, res=[384, 336, 378, 1024], token_lens=[576, 576, 576, 9216],
                       sva=True, stride=3, n_sva=10, image_position=91, seq=2048, micro_batch=4, zero=0, recompute=1,
                       baseline_config=None, tower_tf=sum(TOWER_TF_RELEASE.values()), aux_tf=0.136,
                       workload="Cambrian-1-8B RELEASE recipe train step (finetune_cambrian_8b.sh): SigLIP-SO400M@384, CLIP-L@336, "
                                "DINOv2-giant@378, ConvNeXt-XXL@1024 multi-stage -> SVA grids [576,576,576,9216] (3 + 10 layers) "
                                "-> Llama-3-8B, 576 vis-tok, seq 2048, per-layer recompute"),
    "8b-ddp": dict(llm="llama3-8b", towers=FOUR_TOWERS, res=[384, 336, 336, 1024], sva=True, stride=3, n_sva=10,
                   image_position=91, seq=2048, micro_batch=4, zero=0, baseline_config=3,
                   tower_tf=sum(TOWER_TF.values()),
                   workload="Cambrian-1-8B train step: 4 towers (SigLIP-SO400M@384, CLIP-L@336, DINOv2-L@336, "
                            "ConvNeXt-XXL@1024) -> SVA (3 + 10 layers) -> Llama-3-8B, 576 vis-tok, seq 2048"),
    "7b-clip-mlp": dict(llm="vicuna-7b", towers=FOUR_TOWERS[1:2], res=[336], sva=False, stride=0, n_sva=0,
                        image_position=35, seq=1024, micro_batch=8, zero=0, baseline_config=2, tower_tf=TOWER_TF["clip"],
                        workload="single-tower train step: CLIP ViT-L/14@336 -> mlp2x_gelu -> Vicuna-7B (MHA), 576 vis-tok, "
                                 "seq 1024"),
    "13b-zero2": dict(llm="vicuna-13b", towers=FOUR_TOWERS, res=[384, 336, 336, 1024], sva=True, stride=4, n_sva=10,
                      image_position=35, seq=2048, micro_batch=2, zero=2, baseline_config=4,
                      tower_tf=sum(TOWER_TF.values()),
                      workload="Cambrian-1-13B train step: 4 towers -> SVA (3 + 10 layers, stride 4) -> Vicuna-13B, 576 "
                               "vis-tok, seq 2048, ZeRO-2"),
}


def build_config(name, small=False):
    from cambrian_b200.model.language_model.cambrian_llama import CambrianConfig
    c = CONFIGS[name]
    cfg = CambrianConfig(**LLMS["small" if small else c["llm"]])
    cfg.mm_vision_tower_aux_list = list(c["towers"])
    cfg.mm_vision_tower_aux_token_len_list = list(c.get("token_lens", [576] * len(c["towers"])))
    cfg.image_token_len = 576
    cfg.image_position = c["image_position"]
    cfg.fused_lm_loss = True
    cfg.lm_loss_chunk = 4096
    cfg.inputs_pre_expanded = True     # training harness: batches come from the collator (the reference's static branch)
    if c["sva"]:
        cfg.mm_projector_type = "sva"
        cfg.vision_hidden_size = 1024
        cfg.num_query_group = 1
        cfg.query_num_list = [576]
        cfg.connector_depth = 3
        cfg.connector_only = False
        cfg.num_of_vision_sampler_layers = c["n_sva"] if not small else 2
        cfg.start_of_vision_sampler_layers = 0
        cfg.stride_of_vision_sampler_layers = c["stride"] if not small else 2
    else:
        cfg.mm_projector_type = "mlp2x_gelu"
        cfg.connector_only = True
    if small:
        cfg.convnext_config_overrides = dict(depths=(1, 1, 2, 1), dims=(96, 192, 384, 768), image_size=256)
    return cfg


def llm_fwd_tflop(cfg, S):
    """Algorithmic forward TFLOP per sample of the decoder + lm_head (2*MAC; causal attention counted at half)."""
    H, I, L, V = cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers, cfg.vocab_size
    nh, nkv = cfg.num_attention_heads, cfg.num_key_value_heads
    hd = H // nh
    lin = L * (2 * H * (nh + 2 * nkv) * hd + 2 * H * nh * hd + 3 * 2 * H * I) + 2 * H * V
    attn = L * 4 * S * nh * hd * 0.5
    return S * (lin + attn) / 1e12


def sva_fwd_tflop(cfg, T, aux_tf=None):
    """SVA connector + in-LLM layers + aux projectors + mm_projector, 576 queries over the towers' grids (BASELINE.md §2:
    0.308 + 0.012 + 0.024 for the 8B config with four 576-token grids; 0.780 + 0.136 for the release grids)."""
    if cfg.mm_projector_type != "sva":
        return 576 * (2 * 1024 * cfg.hidden_size + 2 * cfg.hidden_size ** 2) / 1e12      # mlp2x_gelu on 576 tokens
    q, h, H = 576, 1024, cfg.hidden_size
    kv_tok = sum(cfg.mm_vision_tower_aux_token_len_list)      # the K / V projections run over every grid token

    def layer(D):
        return 2 * (q * (h * h + (D + h) * h + h * h + h * h + h * h + h * D) + 2 * kv_tok * h * h)
    conn = cfg.connector_depth * layer(h)
    inllm = (0 if cfg.connector_only else cfg.num_of_vision_sampler_layers) * layer(H)
    aux = (0.012e12 * T / 4) if aux_tf is None else aux_tf * 1e12
    proj = q * 2 * (h * H + H * H)
    return (conn + inllm + aux + proj) / 1e12


class _Tok:
    """The three tokenizer attributes the collator reads (train_fsdp.py:1186-1199)."""

    def __init__(self, max_len):
        self.model_max_length, self.padding_side, self.pad_token_id = max_len, "right", 0


def make_host_batch(cfg, B, S, seed, res, hints):
    """Synthetic batch on the host (pinned), produced by the collator mirror exactly as the training harness would
    (cambrian_b200.train.collator.DataCollatorForSupervisedDataset == train_fsdp.py:1168-1236): raw samples with one
    <image> indicator at `image_position`, square 336-class images, prompt prefix unlabelled."""
    from cambrian_b200.train.collator import DataCollatorForSupervisedDataset
    g = torch.Generator().manual_seed(seed)
    q = int(cfg.image_token_len ** 0.5)
    span = q * (q + 1)
    p0 = cfg.image_position
    raw = S - (span - 1)
    instances = []
    for _ in range(B):
        ids = torch.randint(3, cfg.vocab_size, (raw,), generator=g)
        ids[p0] = -200
        labels = ids.clone()
        labels[:p0 + 1] = -100
        instances.append(dict(input_ids=ids, labels=labels, image_size=(336, 336),
                              image_aux_list=[torch.randn(3, r, r, generator=g).bfloat16() for r in res]))
    coll = DataCollatorForSupervisedDataset(_Tok(S), cfg.image_token_len, list(cfg.mm_vision_tower_aux_token_len_list), p0,
                                            emit_hints=hints)
    batch = coll(instances)
    assert batch["input_ids"].shape == (B, S)
    if getattr(cfg, "mm_projector_type", "") != "sva":
        batch.pop("image_aux_attention_masks_list")      # no SVA: the window masks have no consumer
    for k, v in batch.items():
        if torch.is_tensor(v):
            batch[k] = v.pin_memory()
        elif isinstance(v, list) and v and torch.is_tensor(v[0]):
            batch[k] = [t.pin_memory() for t in v]
    return batch


def to_device(batch, dev):
    out = {}
    nbytes = 0
    for k, v in batch.items():
        if isinstance(v, list) and v and torch.is_tensor(v[0]):
            out[k] = [t.to(dev, non_blocking=True) for t in v]
            nbytes += sum(t.numel() * t.element_size() for t in v)
        elif torch.is_tensor(v):
            out[k] = v.to(dev, non_blocking=True)
            nbytes += v.numel() * v.element_size()
        else:
            out[k] = v          # host-side collator hints (python ints / lists)
    return out, nbytes


class ClockSampler(threading.Thread):
    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.rows, self.stop_flag = index, [], False

    def run(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
        while not self.stop_flag:
            try:
                o = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", str(self.index)],
                                   capture_output=True, text=True, timeout=5).stdout.strip()
                if o:
                    self.rows.append([x.strip() for x in o.split(",")])
            except Exception:
                pass
            time.sleep(0.2)

    def summary(self):
        if not self.rows:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        sm = [float(r[0]) for r in self.rows if r[0].replace(".", "").isdigit()]
        mx = [float(r[1]) for r in self.rows if r[1].replace(".", "").isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(r[3 + i].lower().startswith("active") for r in self.rows)]
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "power_w_max": max((float(r[2]) for r in self.rows if r[2].replace(".", "").isdigit()), default=None),
                "samples": len(self.rows), "reasons": reasons}


class KernelTimer:
    """CUDA-event timing of individual C-ABI launches on the launching stream (events are recorded on torch's CURRENT
    stream, which is the stream the wrapped op launches on — the optimizer's side stream included)."""

    def __init__(self):
        self.events = []  # (kind, work, start, end)
        self.shapes = []  # per GEMM launch: (out shape, K, a_mn, b_mn, act, bias?, residual?, event index)
        self.enabled = False
        self.main = None  # the stream of the training step: kernels launched on other streams (the four towers run
        #                   concurrently on their own streams, the optimizer on its own) overlap each other, so their event
        #                   intervals are not additive; they are recorded under "<kind>@side" and kept out of the rooflines

    def _kind(self, kind):
        if self.main is not None and torch.cuda.current_stream().cuda_stream != self.main:
            return kind + "@side"
        return kind

    def _timed(self, kind, work_fn, fn):
        timer = self

        def wrapped(*a, **kw):
            if not timer.enabled:
                return fn(*a, **kw)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            out = fn(*a, **kw)
            e.record()
            timer.events.append((timer._kind(kind) if kind != "adamw" else kind, float(work_fn(out, *a, **kw)), s, e))
            return out
        return wrapped

    def wrap(self, ops_mod):
        timer = self
        g0 = ops_mod.gemm

        def gemm(a, b, **kw):
            if not timer.enabled:
                return g0(a, b, **kw)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            out = g0(a, b, **kw)
            e.record()
            K = a.shape[-2] if kw.get("a_mn") else a.shape[-1]
            timer.events.append((timer._kind("gemm"), 2.0 * out.numel() * K, s, e))
            timer.shapes.append((tuple(out.shape), K, bool(kw.get("a_mn")), bool(kw.get("b_mn")), kw.get("act"),
                                 kw.get("bias") is not None, kw.get("residual") is not None, len(timer.events) - 1))
            return out

        gs0 = ops_mod.gemm_swiglu

        def gemm_swiglu(x2d, w_gu, gu_out=None, act_out=None):
            # the decoder's fused gate/up projection + SwiGLU (the dominant launch): 2 * M * 2F * K FLOP
            if not timer.enabled:
                return gs0(x2d, w_gu, gu_out, act_out)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            out = gs0(x2d, w_gu, gu_out, act_out)
            e.record()
            M, K = x2d.shape
            timer.events.append((timer._kind("gemm"), 2.0 * M * w_gu.shape[0] * K, s, e))
            timer.shapes.append(((M, w_gu.shape[0]), K, False, False, "swiglu_pair", False, False, len(timer.events) - 1))
            return out

        def sva_bytes(out, q, ks, vs, masks, *a, **kw):
            return 2 * (2 * sum(k.numel() for k in ks) + 2 * q.numel()) + sum(0 if m is None else m.numel() for m in (masks or []))

        def sva_bwd_bytes(out, q, o_, do, lse, ks, *a, **kw):
            return 2 * (4 * sum(k.numel() for k in ks) + 4 * q.numel())  # read K,V,Q,O,dO; write dK,dV,dQ

        def attn_flop(mult):
            def f(out, q, k, v, *a, causal=False, **kw):
                B, Sq, nh, hd = q.shape
                return mult * B * nh * Sq * k.shape[1] * hd * (0.5 if causal and Sq == k.shape[1] else 1.0)
            return f

        ops_mod.gemm, ops_mod.gemm_swiglu = gemm, gemm_swiglu
        ops_mod.sva_window_attn_fwd = self._timed("sva_fwd", sva_bytes, ops_mod.sva_window_attn_fwd)
        ops_mod.sva_window_attn_bwd = self._timed("sva_bwd", sva_bwd_bytes, ops_mod.sva_window_attn_bwd)
        ops_mod.attn_fwd = self._timed("attn_fwd", attn_flop(4.0), ops_mod.attn_fwd)
        ops_mod.attn_bwd = self._timed("attn_bwd", attn_flop(10.0), ops_mod.attn_bwd)
        # AdamW: read g (2) + p, m, v (12); write p, m, v (12) + bf16 p (2) = 28 B / parameter
        ops_mod.adamw = self._timed("adamw", lambda out, p32, *a, **kw: 28.0 * p32.numel(), ops_mod.adamw)

    def shape_table(self, top=24):
        """Per-shape GEMM time / rate inside the timed step (CB_BENCH_SHAPES=1 prints it to stderr)."""
        agg = {}
        for rec in self.shapes:
            _, work, s, e = self.events[rec[-1]]
            a = agg.setdefault(rec[:-1], [0.0, 0.0, 0])
            a[0] += work
            a[1] += s.elapsed_time(e)
            a[2] += 1
        rows = sorted(agg.items(), key=lambda kv: -kv[1][1])[:top]
        return [f"{ms:9.2f} ms {n:5d}x {fl / ms / 1e9:7.0f} TF/s  out={k[0]} K={k[1]} a_mn={int(k[2])} b_mn={int(k[3])} "
                f"act={k[4]} bias={int(k[5])} res={int(k[6])}" for k, (fl, ms, n) in rows]

    def dominant(self):
        """The fused gate/up + SwiGLU GEMM launches alone: per-launch
        algorithmic FLOP / average CUDA-event duration."""
        fl = ms = 0.0
        n = 0
        shape = None
        for rec in self.shapes:
            if rec[4] != "swiglu_pair":
                continue
            _, work, s, e = self.events[rec[-1]]
            fl += work
            ms += s.elapsed_time(e)
            n += 1
            shape = (rec[0], rec[1])
        if n == 0 or ms <= 0:
            return None
        return dict(kernel="gemm_bf16_wgmma<128,0,0,swiglu_pair> (cb_gemm_swiglu_bf16)",
                    shape=f"M={shape[0][0]} 2F={shape[0][1]} K={shape[1]}", launches_timed=n,
                    flop_per_launch=fl / n, avg_launch_ms=ms / n, achieved=fl / (ms / 1000.0) / 1e12)

    def totals(self):
        agg = {}
        for kind, work, s, e in self.events:
            ms = s.elapsed_time(e)
            a = agg.setdefault(kind, [0.0, 0.0, 0])
            a[0] += work
            a[1] += ms
            a[2] += 1
        return agg


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d.get("hbm_gbs", 3350.0), d.get("bf16_tflops_sustained", 989.0), d.get("bf16_tflops", 989.0), "measured"
    # NVIDIA's H100 SXM data sheet (700 W): 3.35 TB/s HBM3, 989 dense BF16 TFLOP/s — a bound, not a measured rate
    return 3350.0, 989.0, 989.0, "H100 SXM data sheet"


# ------------------------------------------------------------------------------------------------------------------
# CPU arm: the reference algorithm on the host cores (oracle/cpu_arm.py: the reference's own vision_sampler.py from
# oracle/_ref when present, the pinned oracle port for everything the reference delegates to third-party libraries)
# ------------------------------------------------------------------------------------------------------------------
def run_reference(args, rank, world):
    if rank != 0:
        return
    if CONFIGS[args.config]["baseline_config"] is None:
        raise SystemExit(f"--impl reference is defined for the BASELINE.json configs (8b-ddp, 7b-clip-mlp, 13b-zero2), not {args.config}")
    from oracle import cpu_arm
    c = CONFIGS[args.config]
    steps, warm = max(1, args.steps), max(1, args.warmup)
    res = cpu_arm.run(args.config, LLMS[c["llm"]], c, steps=steps, warmup=warm)
    line = dict(metric=METRIC, value=res["value"], unit=UNIT, n_gpus=args.gpus, steps=steps, warmup=warm,
                ms_per_step=res["ms_per_bounded_step"], higher_is_better=True, scaling="weak", vs_baseline=None,
                dtype="fp32", data="synthetic", impl="reference",
                config={"workload": c["workload"] + " — host CPU, one BOUNDED step = every distinct block of the step timed "
                                                    "once (fwd+bwd, B=1); value = 1 / sum(count x measured block time)",
                        "baseline_config": c["baseline_config"]},
                value_basis=res["basis"], est_seconds_per_full_sample=res["est_seconds_per_sample"],
                bounded_step_fraction_of_full_step=res["fraction"], components=res["components"],
                cpu_baseline=dict(value=res["value"], unit=UNIT, cores=res["cores"], kind=res["kind"], sample=res["sample"]),
                e2e=dict(value=res["value"], unit=UNIT, h2d_bytes_per_step=0, d2h_bytes_per_step=0))
    print(json.dumps(line))


DUMP_PER_TENSOR = 4096


def dump_outputs(out_dir, loss, model):
    """What the timed step hands back to its caller: the loss, and the trainable parameters it updated (a fixed, seeded
    sample of DUMP_PER_TENSOR elements per tensor, in named_parameters() order; ~5 MB for 3b-ddp)."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "loss.npy"), np.array([float(loss.detach())], dtype=np.float32))
    g = torch.Generator().manual_seed(0)
    parts = []
    for _, p in model.named_parameters():
        if not p.requires_grad:
            continue
        flat = p.detach().reshape(-1)
        idx = torch.randint(0, flat.numel(), (min(DUMP_PER_TENSOR, flat.numel()),), generator=g)
        parts.append(flat[idx.to(flat.device)].float().cpu())
    np.save(os.path.join(out_dir, "params_sample.npy"), torch.cat(parts).numpy())


# ------------------------------------------------------------------------------------------------------------------
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--config", default=os.environ.get("CB_BENCH_CONFIG", "3b-ddp"), choices=sorted(CONFIGS))
    ap.add_argument("--micro-batch", type=int, default=int(os.environ.get("CB_MICRO_BATCH", "0")))
    ap.add_argument("--seq", type=int, default=0)
    ap.add_argument("--recompute", type=int, default=int(os.environ.get("CB_RECOMPUTE", "-1")),
                    help="per-layer activation recompute (1 / 0); default: the config's own (0, release recipe 1)")
    ap.add_argument("--max-grad-norm", type=float, default=float(os.environ.get("CB_MAX_GRAD_NORM", "1.0")),
                    help="gradient clipping as in the reference recipe (HF Trainer default 1.0); 0 disables it")
    ap.add_argument("--bucket-mb", type=float, default=float(os.environ.get("CB_BUCKET_MB", "256")))
    ap.add_argument("--small", action="store_true", help="tiny shapes for a functional check (not a valid bench)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the last step's loss and a fixed seeded sample of the updated "
                         "trainable parameters to DIR as float32 .npy files (compare two builds output for output)")
    args = ap.parse_args()

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.impl == "reference":
        run_reference(args, rank, world)
        return

    import torch.distributed as dist
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        # NCCL's own tuner picks the LL protocol for the 256 MB gradient buckets; Simple streams large buckets at least as
        # well (measured on an earlier 8-GPU node; not re-measured on H100)
        os.environ.setdefault("NCCL_PROTO", "Simple")
        dist.init_process_group("nccl", device_id=dev)
    from cambrian_b200 import _lib, ops
    from cambrian_b200.engine import TrainEngine
    from cambrian_b200.model.language_model.cambrian_llama import CambrianLlamaForCausalLM
    lib = _lib.load()

    C = CONFIGS[args.config]
    if args.recompute < 0:
        args.recompute = C.get("recompute", 0)
    if C["zero"] == 2 and world < 2 and not args.small:
        raise SystemExit("13b-zero2 needs >= 2 GPUs (16 B/param of training state = 214 GB unsharded): launch with torchrun")
    cfg = build_config(args.config, args.small)
    res = C["res"] if not args.small else [r if r < 1024 else 256 for r in C["res"]]
    torch.manual_seed(1234 + rank)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    with torch.device(dev):
        model = CambrianLlamaForCausalLM(cfg)
        for t in model.get_model().vision_tower_aux_list:
            t.load_model()
    torch.set_default_dtype(prev)
    model.train()
    model.get_model().gradient_checkpointing = bool(args.recompute)
    engine = TrainEngine(model, lr=4e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, zero_stage=C["zero"],
                         max_grad_norm=args.max_grad_norm, bucket_mb=args.bucket_mb,
                         overlap=os.environ.get("CB_OVERLAP", "1") != "0",
                         collective=os.environ.get("CB_COLLECTIVE", "nccl"),
                         background_optimizer=os.environ.get("CB_BACKGROUND_OPT", "0") != "0")
    engine.defer_param_sync = os.environ.get("CB_DEFER_PARAM_SYNC", "1") != "0"   # consumers wait per bucket
    n_train = sum(p.numel() for p in engine.params)
    n_tower = sum(p.numel() for t in model.get_model().vision_tower_aux_list for p in t.parameters())

    B = args.micro_batch or C["micro_batch"]
    S = args.seq or C["seq"]
    if args.small:
        B, S = min(B, 2), min(S, 1024)
    # The batch is what the harness's collator emits and is passed as `model(**batch)`, as HF Trainer does
    # (cambrian_trainer.py:226-227).  Our collator mirror adds three host-side hints to that dict (collator.py; switch them
    # off with CB_BENCH_HINTS=0: the model then counts labels / locates the image span on the device — still no host sync —
    # and the fused loss processes every row like the reference).
    hints = os.environ.get("CB_BENCH_HINTS", "1") != "0"
    host_batch = make_host_batch(cfg, B, S, 1000 * rank, res, hints)
    dev_batch, h2d_bytes = to_device(host_batch, dev)
    label_ranges = host_batch.get("label_ranges")
    torch.cuda.synchronize()

    def step_resident():
        engine.zero_grad()
        out = model(**dev_batch)
        out.loss.backward()
        engine.step()
        return out.loss

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    for _ in range(max(3, args.warmup)):
        loss = step_resident()
    torch.cuda.synchronize()
    if not torch.isfinite(loss):
        raise RuntimeError(f"non-finite loss after warm-up: {loss}")

    timer = KernelTimer()
    timer.main = torch.cuda.current_stream().cuda_stream
    timer.wrap(ops)
    sampler = ClockSampler(local_rank)
    sampler.start()
    # ---- timed region: inputs resident in HBM
    barrier()
    timer.enabled = True
    l0 = lib.cb_launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    t_host0 = time.perf_counter()
    for _ in range(args.steps):
        loss = step_resident()
    host_enqueue_ms = (time.perf_counter() - t_host0) * 1000.0 / args.steps  # CPU time to enqueue one step (no sync)
    engine.wait_for_params()          # the last step's optimizer belongs to the timed region
    e1.record()
    barrier()
    timer.enabled = False
    launches = (lib.cb_launch_count() - l0) // args.steps
    ms = e0.elapsed_time(e1)
    sampler.stop_flag = True
    sampler.join(timeout=3)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, loss, model)
    if world > 1:
        t = torch.tensor([ms], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t[0])
    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return

    ms_step = ms / args.steps
    value = world * B / (ms_step / 1000.0)
    hbm_peak, tf_sustained, tf_burst, peak_src = peaks()
    agg = timer.totals()
    if os.environ.get("CB_BENCH_SHAPES"):
        print("\n".join(timer.shape_table(40)), file=sys.stderr)
    roof = None
    if "gemm" in agg:
        fl, tms, n = agg["gemm"]
        ach = fl / (tms / 1000.0) / 1e12
        roof = dict(bound="tensor", kernel="gemm_bf16_wgmma", achieved=ach, peak=tf_sustained, unit="TFLOP/s",
                    frac=ach / tf_sustained, launches_timed=n, share_of_step=tms / ms,
                    peak_source=f"{peak_src} bf16_tflops_sustained (kernel timed inside a long step)",
                    scope="every GEMM launched on the step's main stream (connector + SVA + decoder + loss, fwd and bwd); the "
                          "frozen towers run concurrently on four side streams where per-launch event times overlap and are "
                          "not additive: " + (f"{agg['gemm@side'][2]} tower GEMM launches, {agg['gemm@side'][0] / 1e12 / args.steps:.1f} "
                                              f"TFLOP per step, excluded" if "gemm@side" in agg else "none this run"))
        try:
            dom = timer.dominant()
            if dom is not None:
                dom["frac"] = dom["achieved"] / tf_sustained
                roof["dominant_launch"] = dom
        except Exception as exc:  # never let optional reporting break the bench line
            roof["dominant_launch"] = {"error": str(exc)}

    def tensor_entry(kind, kernel):
        if kind not in agg:
            return None
        fl, tms, n = agg[kind]
        a = fl / (tms / 1000.0) / 1e12
        return dict(bound="tensor", kernel=kernel, achieved=a, peak=tf_sustained, unit="TFLOP/s", frac=a / tf_sustained,
                    launches_timed=n, share_of_step=tms / ms, peak_source=f"{peak_src} bf16_tflops_sustained")
    roof_attn = dict(fwd=tensor_entry("attn_fwd", "attn_fwd_kernel (causal GQA hd128 + ViT hd64/72)"),
                     bwd=tensor_entry("attn_bwd", "attn_bwd_kernel (causal GQA hd128)"))
    roof_adamw = None
    if "adamw" in agg:
        by, tms, n = agg["adamw"]
        a = by / (tms / 1000.0) / 1e9
        roof_adamw = dict(bound="hbm", kernel="adamw_kernel (side stream, co-running with the next step's tower forward)",
                          achieved=a, peak=hbm_peak, unit="GB/s", frac=a / hbm_peak, launches_timed=n,
                          algorithmic_bytes_per_param=28, busy_ms_per_step=tms / args.steps,
                          note="event time on the optimizer stream while GEMMs of the main stream share the SMs and HBM; "
                               "the exposed part is (step time - main-stream time), not this figure")
    roof_sva = None
    if not args.small and C["sva"]:
        # second headline metric (BASELINE.json "SVA HBM GB/s"): the fused window-attention kernel alone, on inputs larger
        # than L2 (batch 32: 377 MB for the BASELINE grids, 1.51 GB for the release grids), CUDA events, 20 launches
        roof_sva = {}
        for tag, rs in (("baseline_grids_576x4", [1, 1, 1, 1]), ("release_grids_576x3_9216", [1, 1, 1, 4])):
            Bq, qs = 32, 24
            qq = torch.randn(Bq * qs * qs, 1024, device=dev).bfloat16()
            ks = [torch.randn(Bq, (r * qs) ** 2, 1024, device=dev).bfloat16() for r in rs]
            vs = [torch.randn(Bq, (r * qs) ** 2, 1024, device=dev).bfloat16() for r in rs]
            for _ in range(3):
                ops.sva_window_attn_fwd(qq, ks, vs, None, rs, Bq, qs)
            s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s0.record()
            for _ in range(20):
                ops.sva_window_attn_fwd(qq, ks, vs, None, rs, Bq, qs)
            s1.record()
            torch.cuda.synchronize()
            byts = 2.0 * (2 * sum(k.numel() for k in ks) + 2 * qq.numel())
            ach = byts / (s0.elapsed_time(s1) / 20 / 1000.0) / 1e9
            roof_sva[tag] = dict(achieved=ach, frac=ach / hbm_peak, algorithmic_bytes_per_launch=byts,
                                 mb_per_sample_per_layer=byts / Bq / 1e6)
            del qq, ks, vs
        roof_sva.update(bound="hbm", kernel="sva_window_attn_fwd", peak=hbm_peak, unit="GB/s",
                        achieved=roof_sva["baseline_grids_576x4"]["achieved"],
                        frac=roof_sva["baseline_grids_576x4"]["frac"], peak_source=f"{peak_src} hbm_gbs")
        if "sva_fwd" in agg:
            by, tms, n = agg["sva_fwd"]
            roof_sva["in_step_achieved"] = by / (tms / 1000.0) / 1e9  # B=4 inputs (38 MB) are L2-resident in the step
    # executed FLOPs per sample: with the collator's label-range hint the fused loss skips the vocabulary GEMMs
    # (3 x 2*H*V per row) of rows whose shifted label is ignore_index — identical loss / gradients, fewer FLOPs
    step_tf = C["tower_tf"] + 3 * (llm_fwd_tflop(cfg, S) + sva_fwd_tflop(cfg, len(C["towers"]), C.get("aux_tf")))
    rows_done = sum(b - a for a, b in label_ranges) if label_ranges is not None else B * S
    skipped_tf = 3 * 2.0 * cfg.hidden_size * cfg.vocab_size * (B * S - rows_done) / B / 1e12
    model_tf = value * (step_tf - skipped_tf) if not args.small else None
    line = dict(metric=METRIC, value=value, unit=UNIT, n_gpus=world, steps=args.steps, warmup=max(3, args.warmup),
                ms_per_step=ms_step, higher_is_better=True, scaling="weak", vs_baseline=None, dtype="bf16",
                data="synthetic", per_gpu=value / world,
                config={"workload": C["workload"] if not args.small else "SMALL functional check (not the benchmark config)",
                        "baseline_config": C["baseline_config"], "name": args.config,
                        "micro_batch_per_gpu": B, "global_batch": B * world, "seq_len": S,
                        "parallelism": (f"zero2x{world}" if C["zero"] == 2 else f"dp{world}"),
                        "collective": engine.collective if world > 1 else None,
                        "activation_recompute": bool(args.recompute),
                        "optimizer": "AdamW fp32 master + bf16 grads, fused, side stream (overlaps the next step's frozen towers)",
                        "grad_clip": engine.max_grad_norm, "trainable_params": n_train, "frozen_tower_params": n_tower,
                        "algorithmic_tflop_per_sample": round(step_tf, 2),
                        "collator_hints": hints,
                        "lm_head_rows": f"{rows_done} of {B * S}" + (" (rows with an ignored label skip the vocabulary GEMMs; "
                                        "loss and gradients identical; MFU counts executed FLOPs only)" if hints else ""),
                        "l2_policy": "inputs larger than L2 (>= 13 GB of weights streamed per pass)"},
                gpu_launches=int(launches), host_enqueue_ms_per_step=round(host_enqueue_ms, 1), loss=float(loss.detach()),
                peak_mem_gb=round(torch.cuda.max_memory_allocated() / 2 ** 30, 1),
                peak_reserved_gb=round(torch.cuda.max_memory_reserved() / 2 ** 30, 1),
                h2d_bytes_per_batch=int(h2d_bytes),
                clocks=sampler.summary(), roofline=roof, roofline_sva=roof_sva, roofline_attn=roof_attn,
                roofline_adamw=roof_adamw,
                model_tflops_per_gpu=(model_tf / world) if model_tf else None,
                mfu_vs_sustained=(model_tf / world / tf_sustained) if model_tf else None)
    if C["baseline_config"] is None:
        line["cpu_baseline"] = dict(value=None, unit=UNIT, cores=os.cpu_count(), kind="port",
                                    sample="not a BASELINE.json config: the CPU arm is defined for configs 2 / 3 / 4")
    elif world == 1 and not args.no_cpu_baseline:
        try:
            from oracle import cpu_arm
            r = cpu_arm.run(args.config, LLMS[C["llm"]], C, steps=1, warmup=1, budget_s=30.0)
            line["cpu_baseline"] = dict(value=r["value"], unit=UNIT, cores=r["cores"], kind=r["kind"], sample=r["sample"])
        except Exception as ex:  # the baseline leg must never take the GPU number down with it
            line["cpu_baseline"] = dict(value=None, unit=UNIT, cores=os.cpu_count(), kind="port", sample=f"failed: {ex}")
    print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
