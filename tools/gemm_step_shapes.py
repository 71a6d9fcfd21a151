#!/usr/bin/env python
"""GEMM shapes of one bench.py training step, timed one by one against torch.matmul (cuBLAS) at the same shape.

    python tools/gemm_step_shapes.py [--config 3b-ddp] [--iters 20] [--no-sweep] [--hash] [--json OUT]

The shapes come from bench.CONFIGS / bench.LLMS: every decoder linear (forward, dX, dW with the layout flags and fused
epilogues the model uses), the fused gate/up + SwiGLU launch, the lm_head chunk, and the MLP GEMMs of the frozen towers
(ConvNeXt-XXL stage 3 at 1024 px, SigLIP and CLIP ViT MLPs).  Each shape is warmed up, then timed with CUDA events over
--iters launches whose operands rotate through enough copies to exceed L2, so that operands stream from HBM as in the
step.  `per_step_ms` = launches per step x time per launch.

The K sweep times two shapes at K = 512 .. 8192 and fits t = t0 + K * c: t0 is the fixed cost per wave of tiles (launch,
pipeline fill, epilogue), c the mainloop cost per unit of K; cuBLAS's slope over ours is the mainloop efficiency.

--hash prints a SHA-256 of every output on seeded inputs, so two builds can be compared output for output.
The card's name, power limit and SM clock are printed with the numbers: they belong to them.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

L2_BYTES = 50 * 2 ** 20       # H100 SXM
ROTATE_BYTES = 4 * L2_BYTES   # operand copies cycled per launch


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception as e:
        out = f"nvidia-smi unavailable: {e}"
    return dict(torch_name=torch.cuda.get_device_name(), smi=out, sms=torch.cuda.get_device_properties(0).multi_processor_count)


def step_shapes(config):
    """(name, launches per step, spec) for the config's step.  spec keys: M N K a_mn b_mn act bias colscale residual acc
    swiglu (M rows, N = 2F columns of gate + up)."""
    import bench
    c = bench.CONFIGS[config]
    llm = bench.LLMS[c["llm"]]
    H, I, L, V = llm["hidden_size"], llm["intermediate_size"], llm["num_hidden_layers"], llm["vocab_size"]
    hd = H // llm["num_attention_heads"]
    QKV = (llm["num_attention_heads"] + 2 * llm["num_key_value_heads"]) * hd
    B, S = c["micro_batch"], c["seq"]
    R = B * S
    fwd = L * (2 if c.get("recompute") else 1)   # forward, and again in the backward when layers are recomputed

    def g(M, N, K, **kw):
        d = dict(M=M, N=N, K=K, a_mn=False, b_mn=False, act=None, bias=False, colscale=False, residual=False, acc=False,
                 swiglu=False)
        d.update(kw)
        return d
    # label rows: the collator leaves the prompt (image_position + 1 tokens) and the 600-token image span unlabelled
    span = 24 * 25
    label_rows = B * (S - (span - 1) - c["image_position"] - 1)
    chunk = 4096
    n_chunks = math.ceil(label_rows / chunk)
    rows = [
        ("dec.qkv fwd", fwd, g(R, QKV, H)),
        ("dec.o fwd +res", fwd, g(R, H, H, residual=True)),
        ("dec.gate_up+swiglu fwd", fwd, g(R, 2 * I, H, swiglu=True)),
        ("dec.down fwd +res", L, g(R, H, I, residual=True)),   # the recompute stops before the down projection
        ("dec.down dX", L, g(R, I, H, b_mn=True)),
        ("dec.gate_up dX", L, g(R, H, 2 * I, b_mn=True)),
        ("dec.o dX", L, g(R, H, H, b_mn=True)),
        ("dec.qkv dX", L, g(R, H, QKV, b_mn=True)),
        ("dec.down dW +=", L, g(H, I, R, a_mn=True, b_mn=True, acc=True)),
        ("dec.gate_up dW +=", L, g(2 * I, H, R, a_mn=True, b_mn=True, acc=True)),
        ("dec.o dW +=", L, g(H, H, R, a_mn=True, b_mn=True, acc=True)),
        ("dec.qkv dW +=", L, g(QKV, H, R, a_mn=True, b_mn=True, acc=True)),
        ("lm_head logits", n_chunks, g(chunk, V, H)),
        ("lm_head dX", n_chunks, g(chunk, H, V, b_mn=True)),
        ("lm_head dW +=", n_chunks, g(V, H, chunk, a_mn=True, b_mn=True, acc=True)),
    ]
    if "clip-convnext-XXL" in c["towers"]:
        res = c["res"][c["towers"].index("clip-convnext-XXL")]
        # stages 1-3: stride 4 / 8 / 16, 384 / 768 / 1536 channels, 3 / 4 / 30 blocks (stage 4 is small)
        for st, stride, C, blocks in ((1, 4, 384, 3), (2, 8, 768, 4), (3, 16, 1536, 30)):
            cn_rows = B * (res // stride) ** 2
            rows += [(f"convnext s{st} fc1 gelu", blocks, g(cn_rows, 4 * C, C, act="gelu", bias=True)),
                     (f"convnext s{st} fc2 ls+res", blocks,
                      g(cn_rows, C, 4 * C, bias=True, colscale=True, residual=True))]
    if any("siglip" in t for t in c["towers"]):
        rows += [("siglip fc1 gelu", 27, g(B * 729, 4304, 1152, act="gelu", bias=True))]
    if any("clip-vit-large" in t for t in c["towers"]):
        rows += [("clip fc1 quick_gelu", 24, g(B * 577, 4096, 1024, act="quick_gelu", bias=True)),
                 ("clip fc2 +res", 24, g(B * 577, 1024, 4096, bias=True, residual=True))]
    return rows


def make_operands(s, gen, dev):
    M, N, K = s["M"], s["N"], s["K"]
    a = torch.randn((K, M) if s["a_mn"] else (M, K), generator=gen, device=dev).bfloat16()
    b = (torch.randn((K, N) if s["b_mn"] else (N, K), generator=gen, device=dev) * K ** -0.5).bfloat16()
    extra = {}
    if s["bias"]:
        extra["bias"] = torch.randn(N, generator=gen, device=dev).bfloat16()
    if s["colscale"]:
        extra["colscale"] = torch.rand(N, generator=gen, device=dev).bfloat16()
    if s["residual"]:
        extra["residual"] = torch.randn(M, N, generator=gen, device=dev).bfloat16()
    return a, b, extra


def run_ours(s, a, b, extra, out, out2):
    from cambrian_b200 import ops
    if s["swiglu"]:
        ops.gemm_swiglu(a, b, out, out2)
    else:
        ops.gemm(a, b, a_mn=s["a_mn"], b_mn=s["b_mn"], act=s["act"], out=out, accumulate=s["acc"], **extra)


def run_cublas(s, a, b, out):
    torch.matmul(a.t() if s["a_mn"] else a, b if s["b_mn"] else b.t(), out=out)


def time_launches(fn, sets, iters):
    for i in range(3):
        fn(*sets[i % len(sets)])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(*sets[i % len(sets)])
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def measure(s, iters, want_hash, seed=0):
    dev = "cuda"
    gen = torch.Generator(device=dev).manual_seed(seed)
    M, N, K = s["M"], s["N"], s["K"]
    first = make_operands(s, gen, dev)
    set_bytes = 2 * (first[0].numel() + first[1].numel() + sum(t.numel() for t in first[2].values()))
    sets = [first] + [make_operands(s, gen, dev) for _ in range(min(7, ROTATE_BYTES // max(set_bytes, 1)))]
    out = torch.zeros((M, N), dtype=torch.bfloat16, device=dev)
    out2 = torch.empty((M, N // 2), dtype=torch.bfloat16, device=dev) if s["swiglu"] else None
    digest = None
    if want_hash:
        run_ours(s, *first, out, out2)
        torch.cuda.synchronize()
        h = hashlib.sha256(out.view(torch.int16).cpu().numpy().tobytes())
        if out2 is not None:
            h.update(out2.view(torch.int16).cpu().numpy().tobytes())
        digest = h.hexdigest()[:16]
    ms = time_launches(lambda a, b, extra: run_ours(s, a, b, extra, out, out2), sets, iters)
    ms_cublas = time_launches(lambda a, b, extra: run_cublas(s, a, b, out), sets, iters)
    del sets, out, out2
    torch.cuda.empty_cache()
    fl = 2.0 * M * N * K
    return dict(ms=ms, tflops=fl / ms / 1e9, cublas_ms=ms_cublas, cublas_tflops=fl / ms_cublas / 1e9, sha=digest)


def k_sweep(name, base, iters):
    pts = []
    for K in (512, 1024, 2048, 4096, 8192):
        s = dict(base, K=K)
        r = measure(s, iters, False)
        pts.append((K, r["ms"], r["cublas_ms"]))

    def fit(ys):
        ks = [p[0] for p in pts]
        n, mk, my = len(ks), sum(ks) / len(ks), sum(ys) / len(ys)
        c = sum((k - mk) * (y - my) for k, y in zip(ks, ys)) / sum((k - mk) ** 2 for k in ks)
        return my - c * mk, c
    t0, c = fit([p[1] for p in pts])
    t0c, cc = fit([p[2] for p in pts])
    return dict(shape=name, M=base["M"], N=base["N"], points=pts, t0_ms=t0, slope_us_per_kblock=c * 64 * 1e3,
                cublas_t0_ms=t0c, cublas_slope_us_per_kblock=cc * 64 * 1e3, mainloop_eff_vs_cublas=cc / c)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="3b-ddp")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--no-sweep", action="store_true")
    ap.add_argument("--hash", action="store_true", help="print a SHA-256 prefix of each output on seeded inputs")
    ap.add_argument("--json", default=None, help="also write the results here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gemm_step_shapes.py times kernels on the GPU: no CUDA device is visible")
    torch.cuda.set_device(0)
    card = card_info()
    print(f"# {card['torch_name']} | {card['smi']} (name, power limit, SM clock, max SM clock) | {card['sms']} SMs")
    res = dict(card=card, config=args.config, shapes=[], sweeps=[])
    print(f"{'shape':26s} {'M':>6s} {'N':>6s} {'K':>6s} {'flags':14s} {'n/step':>6s} {'ms':>8s} {'TF/s':>6s} "
          f"{'cuBLAS ms':>9s} {'TF/s':>6s} {'vs cuBLAS':>9s} {'ms/step':>8s}" + ("  sha256" if args.hash else ""))
    total = 0.0
    for name, n, s in step_shapes(args.config):
        r = measure(s, args.iters, args.hash)
        flags = ("A_MN " if s["a_mn"] else "") + ("B_MN " if s["b_mn"] else "") + (s["act"] or "") + \
                (" acc" if s["acc"] else "")
        total += n * r["ms"]
        print(f"{name:26s} {s['M']:6d} {s['N']:6d} {s['K']:6d} {flags.strip():14s} {n:6d} {r['ms']:8.3f} "
              f"{r['tflops']:6.0f} {r['cublas_ms']:9.3f} {r['cublas_tflops']:6.0f} {r['cublas_ms'] / r['ms']:9.2f} "
              f"{n * r['ms']:8.1f}" + (f"  {r['sha']}" if args.hash else ""), flush=True)
        res["shapes"].append(dict(name=name, per_step=n, per_step_ms=n * r["ms"], **s, **r))
    print(f"# sum over the listed shapes: {total:.1f} ms per step (launches run back to back, one stream)")
    res["sum_ms_per_step"] = total
    if not args.no_sweep:
        shapes = dict((nm, s) for nm, _, s in step_shapes(args.config))
        for nm in ("dec.o fwd +res", "dec.gate_up+swiglu fwd"):
            sw = k_sweep(nm, shapes[nm], args.iters)
            res["sweeps"].append(sw)
            print(f"# K sweep {nm} (M={sw['M']} N={sw['N']}): t0 {sw['t0_ms'] * 1e3:.1f} us, "
                  f"{sw['slope_us_per_kblock']:.2f} us per 64-deep k-block | cuBLAS t0 {sw['cublas_t0_ms'] * 1e3:.1f} us, "
                  f"{sw['cublas_slope_us_per_kblock']:.2f} us per k-block | mainloop efficiency vs cuBLAS "
                  f"{sw['mainloop_eff_vs_cublas']:.2f}")
            print("#   K, ms, cuBLAS ms: " + "; ".join(f"{k} {a:.3f} {b:.3f}" for k, a, b in sw["points"]))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
