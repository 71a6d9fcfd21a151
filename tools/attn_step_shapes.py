#!/usr/bin/env python
"""Flash-attention launches of one bench.py training step, timed one by one at their real shapes.

    python tools/attn_step_shapes.py [--config 3b-ddp] [--iters 20] [--hash] [--json OUT]

Shapes: the decoder's causal GQA attention (q / k / v are views of the packed QKV GEMM output, dQ / dK / dV land in a
packed dQKV buffer, as in autograd.py) with the all-True key mask the training step passes and with kmask=None, forward
and backward; and the forward of the ViT towers (CLIP-L and DINOv2-L: 577 tokens x 16 heads x hd 64; SigLIP: 729 x 16 x
72; B = 4).  Each launch is warmed up, then timed with CUDA events over --iters launches.  The backward is also split
into its kernels with torch.profiler in a separate pass.

TF/s uses bench.py's FLOP counts (forward 4 B nh Sq Skv hd, backward 10 B nh Sq Skv hd, halved when causal); the
executed rate counts what the kernels run (the backward's dK / dV kernel runs 4 GEMMs and its dQ kernel 3, so 14 instead
of 10).

--hash prints a SHA-256 prefix of every output (O, lse, dQ, dK, dV) on inputs drawn from a seeded CPU generator, so two
builds can be compared bit for bit.  The card's name, power limit and SM clock are printed with the numbers.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import re
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gemm_step_shapes import card_info  # noqa: E402

TOWERS = {  # name key in bench.CONFIGS[...]["towers"] -> (label, tokens, heads, hd, layers)
    "siglip": ("siglip fwd", 729, 16, 72, 27),
    "clip-vit-large": ("clip-L fwd", 577, 16, 64, 24),
    "dinov2": ("dinov2-L fwd", 577, 16, 64, 24),
}


def step_shapes(config):
    """(name, launches per step, spec) for the config's step."""
    import bench
    c = bench.CONFIGS[config]
    llm = bench.LLMS[c["llm"]]
    nh, nkv, L = llm["num_attention_heads"], llm["num_key_value_heads"], llm["num_hidden_layers"]
    hd = llm["hidden_size"] // nh
    B, S = c["micro_batch"], c["seq"]
    fwd = L * (2 if c.get("recompute") else 1)
    dec = dict(kind="decoder", B=B, S=S, nh=nh, nkv=nkv, hd=hd)
    rows = [("dec fwd kmask", fwd, dict(dec, mask=True, bwd=False)),
            ("dec fwd kmask=None", fwd, dict(dec, mask=False, bwd=False)),
            ("dec bwd kmask", L, dict(dec, mask=True, bwd=True)),
            ("dec bwd kmask=None", L, dict(dec, mask=False, bwd=True))]
    for key, (label, T, heads, thd, layers) in TOWERS.items():
        if any(key in t for t in c["towers"]):
            rows.append((label, layers, dict(kind="tower", B=B, S=T, nh=heads, nkv=heads, hd=thd, mask=False, bwd=False)))
    return rows


def make_inputs(s, seed):
    """Packed operands as the model holds them, from a seeded CPU generator."""
    gen = torch.Generator().manual_seed(seed)
    B, S, nh, nkv, hd = s["B"], s["S"], s["nh"], s["nkv"], s["hd"]
    dev = "cuda"
    if s["kind"] == "tower":
        qkv = torch.randn(B, S, 3, nh, hd, generator=gen).bfloat16().to(dev)
        return dict(q=qkv[:, :, 0], k=qkv[:, :, 1], v=qkv[:, :, 2], kmask=None, causal=False)
    qkv = torch.randn(B * S, (nh + 2 * nkv) * hd, generator=gen).bfloat16().to(dev)
    do = torch.randn(B, S, nh, hd, generator=gen).bfloat16().to(dev)
    kmask = torch.ones(B, S, dtype=torch.bool, device=dev) if s["mask"] else None
    return dict(qkv=qkv, q=qkv[:, : nh * hd].view(B, S, nh, hd), k=qkv[:, nh * hd:(nh + nkv) * hd].view(B, S, nkv, hd),
                v=qkv[:, (nh + nkv) * hd:].view(B, S, nkv, hd), do=do, kmask=kmask, causal=True)


def bwd_views(s, dqkv):
    B, S, nh, nkv, hd = s["B"], s["S"], s["nh"], s["nkv"], s["hd"]
    return dict(dq=dqkv[:, : nh * hd].view(B, S, nh, hd), dk=dqkv[:, nh * hd:(nh + nkv) * hd].view(B, S, nkv, hd),
                dv=dqkv[:, (nh + nkv) * hd:].view(B, S, nkv, hd))


def sha(*ts):
    h = hashlib.sha256()
    for t in ts:
        t = t.contiguous()
        h.update((t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)).cpu().numpy().tobytes())
    return h.hexdigest()[:16]


def time_launches(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def kernel_split(fn, iters):
    """Mean device time per launch of each kernel fn runs, by torch.profiler (a pass of its own)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.events():
        if ev.device_type.name != "CUDA":
            continue
        name = re.sub(r"<.*", "", ev.name).split("(")[0].split("::")[-1]
        out[name] = out.get(name, 0.0) + ev.device_time / 1e3 / iters
    return out


def run_fns(s, x):
    """(forward, backward or None, the backward's outputs or None) on the inputs of make_inputs."""
    from cambrian_b200 import ops
    fwd = lambda: ops.attn_fwd(x["q"], x["k"], x["v"], causal=x["causal"], kmask=x["kmask"], need_lse=True)
    if not s["bwd"]:
        return fwd, None, None
    o, lse = fwd()
    views = bwd_views(s, torch.empty_like(x["qkv"]))
    bwd = lambda: ops.attn_bwd(x["q"], x["k"], x["v"], o, x["do"], lse, causal=True, kmask=x["kmask"], **views)
    return fwd, bwd, views


def fingerprint(s, seed=0):
    """SHA-256 prefixes of every output of the shape on seeded inputs: O and lse, and dQ / dK / dV for a backward."""
    x = make_inputs(s, seed)
    fwd, bwd, views = run_fns(s, x)
    o, lse = fwd()
    if bwd:
        bwd()
    torch.cuda.synchronize()
    out = dict(o=sha(o), lse=sha(lse))
    if bwd:
        out.update(dq=sha(views["dq"]), dk=sha(views["dk"]), dv=sha(views["dv"]))
    return out


def measure(s, iters, want_hash, seed=0):
    B, S, nh, hd = s["B"], s["S"], s["nh"], s["hd"]
    r = dict(sha=fingerprint(s, seed) if want_hash else None, split=None)
    x = make_inputs(s, seed)
    fwd, bwd, _ = run_fns(s, x)
    half = 0.5 if x["causal"] else 1.0
    if not bwd:
        r["ms"] = time_launches(fwd, iters)
        flop = exec_flop = 4.0 * B * nh * S * S * hd * half
    else:
        r["ms"] = time_launches(bwd, iters)
        r["split"] = kernel_split(bwd, max(3, iters // 4))
        flop = 10.0 * B * nh * S * S * hd * half
        exec_flop = 14.0 * B * nh * S * S * hd * half
    r["tflops"] = flop / r["ms"] / 1e9
    r["exec_tflops"] = exec_flop / r["ms"] / 1e9
    del x, fwd, bwd
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="3b-ddp")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--hash", action="store_true", help="print a SHA-256 prefix of each output on seeded inputs")
    ap.add_argument("--json", default=None, help="also write the results here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_step_shapes.py times kernels on the GPU: no CUDA device is visible")
    torch.cuda.set_device(0)
    card = card_info()
    print(f"# {card['torch_name']} | {card['smi']} (name, power limit, SM clock, max SM clock) | {card['sms']} SMs")
    res = dict(card=card, config=args.config, shapes=[])
    print(f"{'shape':20s} {'B':>2s} {'S':>5s} {'nh':>3s} {'nkv':>3s} {'hd':>3s} {'n/step':>6s} {'ms':>8s} {'TF/s':>6s} "
          f"{'exec TF/s':>9s}")
    for name, n, s in step_shapes(args.config):
        r = measure(s, args.iters, args.hash)
        print(f"{name:20s} {s['B']:2d} {s['S']:5d} {s['nh']:3d} {s['nkv']:3d} {s['hd']:3d} {n:6d} {r['ms']:8.3f} "
              f"{r['tflops']:6.0f} {r['exec_tflops']:9.0f}", flush=True)
        if r["split"]:
            print("    kernels (ms / launch): " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(r["split"].items())))
        if r["sha"]:
            print("    sha256: " + " ".join(f"{k}={v}" for k, v in r["sha"].items()))
        res["shapes"].append(dict(name=name, per_step=n, per_step_ms=n * r["ms"], **s, **r))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
