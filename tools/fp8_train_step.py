#!/usr/bin/env python
"""What FP8 training (`config.fp8_training`) buys on this GPU, bf16 and FP8 measured in one session.

    python tools/fp8_train_step.py [--config 3b-ddp] [--windows 3] [--steps 5] [--warmup 3] [--loss-batches 4]
                                   [--reps 20] [--out DIR]

1. Builds bench.py's model, batch and engine (bench.build_config / bench.make_host_batch, the same seeds) once.
2. Loss of both formats on the same weights over --loss-batches seeded batches (forward only, before any step).
3. Step time: after --warmup steps of each format, --windows timed windows of --steps steps, bf16 and FP8 alternating
   (the flag is read at every forward, so one model serves both).  ms/step per window and peak device memory per format.
4. Per projection (q|k|v, o, gate|up, down) at the step's token count: the forward GEMM and the input-gradient GEMM in
   bf16, and in FP8 split into the activation quantiser, the per-call weight quantiser (row-wise for forward, transposed
   for dgrad) and the FP8 GEMM; CUDA events over --reps launches each.

The card's name and power limit are printed with the numbers; --out DIR writes them to DIR/fp8_train_step.json too.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception as e:
        out = f"nvidia-smi unavailable: {e}"
    return f"{torch.cuda.get_device_name()} | {out} (name, power limit, max SM clock)"


def set_fp8(model, on):
    model.config.fp8_training = on
    model.get_model().config.fp8_training = on


def time_ms(fn, reps):
    fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def projections(cfg, M, reps, dev):
    """bf16 and FP8 times of each projection's forward and dgrad GEMM at M tokens."""
    from cambrian_b200 import ops, train_fp8
    from cambrian_b200.quant_fp8 import Fp8Weight
    H, I = cfg.hidden_size, cfg.intermediate_size
    nh, nkv = cfg.num_attention_heads, cfg.num_key_value_heads
    hd = getattr(cfg, "head_dim", None) or H // nh
    shapes = dict(qkv=((nh + 2 * nkv) * hd, H), o=(H, nh * hd), gate_up=(2 * I, H), down=(H, I))
    g = torch.Generator(device=dev).manual_seed(0)
    rows = {}
    for name, (N, K) in shapes.items():
        w = (torch.randn(N, K, generator=g, device=dev) * 0.02).bfloat16()
        x = torch.randn(M, K, generator=g, device=dev).bfloat16()
        dy = torch.randn(M, N, generator=g, device=dev).bfloat16()
        qa, qd = ops.fp8_quantize_act(x), ops.fp8_quantize_act(dy)
        pw, pt = train_fp8.weight_rows(w), train_fp8.weight_t(w)
        wr, wt = Fp8Weight(N, K, dev), Fp8Weight(K, N, dev)
        r = dict(N=N, K=K, M=M,
                 fwd_bf16=time_ms(lambda: ops.gemm(x, w), reps),
                 fwd_fp8_quant_act=time_ms(lambda: ops.fp8_quantize_act(x), reps),
                 fwd_fp8_quant_weight=time_ms(lambda: ops.fp8_quantize_weight(w, wr.wq, wr.sw), reps),
                 fwd_fp8_gemm=time_ms(lambda: ops.gemm_fp8(qa, pw), reps),
                 dgrad_bf16=time_ms(lambda: ops.gemm(dy, w, b_mn=True), reps),
                 dgrad_fp8_quant_act=time_ms(lambda: ops.fp8_quantize_act(dy), reps),
                 dgrad_fp8_quant_weight_t=time_ms(lambda: ops.fp8_quantize_weight_t(w, wt.wq, wt.sw), reps),
                 dgrad_fp8_gemm=time_ms(lambda: ops.gemm_fp8(qd, pt), reps))
        r["fwd_fp8"] = r["fwd_fp8_quant_act"] + r["fwd_fp8_quant_weight"] + r["fwd_fp8_gemm"]
        r["dgrad_fp8"] = r["dgrad_fp8_quant_act"] + r["dgrad_fp8_quant_weight_t"] + r["dgrad_fp8_gemm"]
        r["gemm_tflops_bf16_fwd"] = 2 * M * N * K / r["fwd_bf16"] / 1e9
        r["gemm_tflops_fp8_fwd"] = 2 * M * N * K / r["fwd_fp8_gemm"] / 1e9
        rows[name] = r
        del w, x, dy, qa, qd, pw, pt, wr, wt
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="3b-ddp")
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--loss-batches", type=int, default=4)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write DIR/fp8_train_step.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_train_step.py measures on the GPU; none is visible")
    sys.path.insert(0, ROOT)
    import bench
    from cambrian_b200.engine import TrainEngine
    from cambrian_b200.model.language_model.cambrian_llama import CambrianLlamaForCausalLM
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    card = card_info()
    print(f"# {card}")
    C = bench.CONFIGS[args.config]
    cfg = bench.build_config(args.config)
    torch.manual_seed(1234)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    with torch.device(dev):
        model = CambrianLlamaForCausalLM(cfg)
        for t in model.get_model().vision_tower_aux_list:
            t.load_model()
    torch.set_default_dtype(prev)
    model.train()
    model.get_model().gradient_checkpointing = bool(C.get("recompute", 0))
    engine = TrainEngine(model, lr=4e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, zero_stage=C["zero"],
                         max_grad_norm=1.0, bucket_mb=256.0)
    engine.defer_param_sync = True
    res = dict(card=card, config=args.config, micro_batch=C["micro_batch"], seq=C["seq"])

    # 2. loss of both formats, same weights, same seeded batches
    losses = {"bf16": [], "fp8": []}
    with torch.no_grad():
        for seed in range(args.loss_batches):
            b, _ = bench.to_device(bench.make_host_batch(cfg, C["micro_batch"], C["seq"], seed, C["res"], True), dev)
            for mode in ("bf16", "fp8"):
                set_fp8(model, mode == "fp8")
                losses[mode].append(float(model(**b).loss))
            del b
    res["loss_same_weights"] = losses
    print(f"# loss on the same weights, batches 0..{args.loss_batches - 1}: bf16 {losses['bf16']}, fp8 {losses['fp8']}")

    # 3. alternating timed windows
    batch, _ = bench.to_device(bench.make_host_batch(cfg, C["micro_batch"], C["seq"], 0, C["res"], True), dev)

    def step():
        engine.zero_grad()
        out = model(**batch)
        out.loss.backward()
        engine.step()
        return out.loss

    windows = {"bf16": [], "fp8": []}
    peak = {"bf16": 0.0, "fp8": 0.0}
    step_loss = {"bf16": [], "fp8": []}
    for mode in ("bf16", "fp8"):
        set_fp8(model, mode == "fp8")
        for _ in range(args.warmup):
            step()
    torch.cuda.synchronize()
    for _ in range(args.windows):
        for mode in ("bf16", "fp8"):
            set_fp8(model, mode == "fp8")
            torch.cuda.reset_peak_memory_stats()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                loss = step()
            engine.wait_for_params()
            e1.record()
            torch.cuda.synchronize()
            windows[mode].append(e0.elapsed_time(e1) / args.steps)
            peak[mode] = max(peak[mode], torch.cuda.max_memory_allocated() / 2 ** 30)
            step_loss[mode].append(float(loss.detach()))
    set_fp8(model, False)
    res.update(ms_per_step=windows, peak_device_gb=peak, last_step_loss=step_loss, steps=args.steps,
               warmup=args.warmup)
    for mode in ("bf16", "fp8"):
        w = windows[mode]
        print(f"# {mode}: ms/step per window {[round(v, 1) for v in w]} (median {sorted(w)[len(w) // 2]:.1f}), "
              f"peak device {peak[mode]:.1f} GB")
    del batch, engine, model
    torch.cuda.empty_cache()

    # 4. per projection
    rows = projections(cfg, C["micro_batch"] * C["seq"], args.reps, dev)
    res["projections"] = rows
    print(f"# per projection at M = {C['micro_batch'] * C['seq']} tokens, ms (FP8 = act quant + weight quant + GEMM)")
    for name, r in rows.items():
        print(f"  {name:8s} [{r['N']:5d} x {r['K']:5d}]  fwd bf16 {r['fwd_bf16']:.3f}  fp8 {r['fwd_fp8']:.3f} = "
              f"{r['fwd_fp8_quant_act']:.3f} + {r['fwd_fp8_quant_weight']:.3f} + {r['fwd_fp8_gemm']:.3f}   dgrad bf16 "
              f"{r['dgrad_bf16']:.3f}  fp8 {r['dgrad_fp8']:.3f} = {r['dgrad_fp8_quant_act']:.3f} + "
              f"{r['dgrad_fp8_quant_weight_t']:.3f} + {r['dgrad_fp8_gemm']:.3f}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "fp8_train_step.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
