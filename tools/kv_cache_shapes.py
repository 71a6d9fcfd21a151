"""Decode attention of one layer, timed with CUDA events: today's bf16-cache path (ops.attn_fwd with Sq = 1 over the
whole [B, S_max] bf16 buffer and the key mask, as the graph-replayed decode step runs it) against ops.attn_decode_fp8
over the FP8 cache (cambrian_b200/kv_fp8.py), at the head shapes of Cambrian-8B (32 / 8), Cambrian-13B (40 / 40, MHA) and
Cambrian-34B (56 / 8), hd 128, batch 1 / 8 / 64, filled length 1k / 4k / 16k in a buffer of that size.

    python tools/kv_cache_shapes.py [--iters 50] [--out FILE]

GB/s counts the cache bytes each path needs at that length (bf16: 2 * B * L * nkv * hd * 2; FP8: 2 * B * L * nkv *
(hd + 4)) over its time, against the H100 SXM data-sheet 3.35 TB/s.  The card's name, power limit and max SM clock are
read in the same run.  One JSON line per shape.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HEADS = {"8b": (32, 8), "13b": (40, 40), "yi34b": (56, 8)}
HBM_TBPS = 3.35


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def timed(fn, iters):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters                      # us per call


def one(name, B, L, iters, hd=128):
    from cambrian_b200 import ops
    nh, nkv = HEADS[name]
    dev = torch.device("cuda")
    kc = torch.empty(B, L, nkv, hd, dtype=torch.bfloat16, device=dev).normal_()
    vc = torch.empty_like(kc).normal_()
    q = torch.randn(B, 1, nh, hd, device=dev).to(torch.bfloat16)
    kmask = torch.ones(B, L, dtype=torch.bool, device=dev)
    f8 = torch.float8_e4m3fn
    kq, vq = torch.empty(B, L, nkv, hd, dtype=f8, device=dev), torch.empty(B, L, nkv, hd, dtype=f8, device=dev)
    ks, vs = torch.empty(B, L, nkv, device=dev), torch.empty(B, L, nkv, device=dev)
    ops.kv_fp8_append(kc, vc, kq, vq, ks, vs, offset=0)
    ws = ops.attn_decode_fp8_workspace(B, nh, nkv, L, hd, dev)
    t16 = timed(lambda: ops.attn_fwd(q, kc, vc, causal=False, kmask=kmask), iters)
    t8 = timed(lambda: ops.attn_decode_fp8(q, kq, vq, ks, vs, ws, length=L, kmask=kmask), iters)
    b16, b8 = 2 * B * L * nkv * hd * 2, 2 * B * L * nkv * (hd + 4)
    del kc, vc, kq, vq, ks, vs
    torch.cuda.empty_cache()
    return dict(shape=name, nh=nh, nkv=nkv, hd=hd, batch=B, length=L, bf16_attn_fwd_us=round(t16, 2),
                fp8_decode_us=round(t8, 2), speedup=round(t16 / t8, 2), bf16_gbps=round(b16 / t16 / 1e3, 1),
                fp8_gbps=round(b8 / t8 / 1e3, 1), fp8_frac_of_hbm=round(b8 / t8 / 1e3 / (HBM_TBPS * 1e3), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    info = card()
    out = open(args.out, "a") if args.out else None
    for name in HEADS:
        for B in (1, 8, 64):
            for L in (1024, 4096, 16384):
                rec = dict(one(name, B, L, args.iters), card=info)
                line = json.dumps(rec)
                print(line, flush=True)
                if out:
                    out.write(line + "\n")
                    out.flush()


if __name__ == "__main__":
    main()
