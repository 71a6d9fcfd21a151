"""Cambrian-Phi3-3B inference on one GPU: prefill and greedy decode of a random Phi-3-mini-shaped text decoder (hidden
3072, 32 layers, 32 heads of 96, intermediate 8192, vocab 32064, sliding window 2047), and the head-dim-96 flash-attention
forward on its own.

    python tools/phi3_decode.py [--batch 1,8] [--prompt 1024] [--new 64] [--out FILE]

Prints one JSON line per measurement, the first with the card's name, power limit and max SM clock, and with --out also
writes them all to FILE as one JSON list:
  * prefill ms and decode ms / token (CUDA-graph loop) per batch, against the weight-streaming floor (decoder + lm_head
    bf16 bytes / 3.35 TB/s, the H100 SXM data-sheet bandwidth);
  * attention forward TF/s (causal FLOPs: 4 * B * nh * hd * visible (query, key) pairs) at the Phi-3 prefill shape next
    to hd 128 at the Llama-3-8B shape, and the time the window's tile skipping saves at S = 4096.
Times are CUDA-event means over repeated calls after warm-up.
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

HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def timed(fn, reps, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def visible_pairs(S, window):
    if not window or window >= S:
        return S * (S + 1) // 2
    return sum(min(i + 1, window) for i in range(S))


def attention(out):
    from cambrian_b200 import ops
    rows = []
    for name, B, S, nh, nkv, hd, W in (("phi3 prefill", 1, 2048, 32, 32, 96, 2047),
                                       ("phi3 prefill", 1, 4096, 32, 32, 96, 2047),
                                       ("phi3 prefill, no window", 1, 4096, 32, 32, 96, 0),
                                       ("llama3-8b prefill", 1, 2048, 32, 8, 128, 0),
                                       ("phi3 batch 8", 8, 2048, 32, 32, 96, 2047)):
        g = torch.Generator(device="cuda").manual_seed(S)
        q = torch.randn(B, S, nh, hd, device="cuda", generator=g).bfloat16()
        k = torch.randn(B, S, nkv, hd, device="cuda", generator=g).bfloat16()
        v = torch.randn(B, S, nkv, hd, device="cuda", generator=g).bfloat16()
        ms = timed(lambda: ops.attn_fwd(q, k, v, causal=True, window=W), 20)
        flops = 4.0 * B * nh * hd * visible_pairs(S, W)
        r = dict(what="attn_fwd", shape=name, B=B, S=S, nh=nh, nkv=nkv, hd=hd, window=W, ms=round(ms, 4),
                 tflops=round(flops / ms / 1e9, 1))
        rows.append(r)
        print(json.dumps(r), flush=True)
    w = next(r for r in rows if r["S"] == 4096 and r["window"])
    n = next(r for r in rows if r["S"] == 4096 and not r["window"])
    r = dict(what="window tile skipping at S=4096", ms_window=w["ms"], ms_full_causal=n["ms"],
             saved_ms=round(n["ms"] - w["ms"], 4), saved_pct=round(100 * (1 - w["ms"] / n["ms"]), 1))
    print(json.dumps(r), flush=True)
    out.extend(rows + [r])


def decode(out, batches, prompt, new):
    from cambrian_b200.model.language_model.cambrian_phi3 import CambrianPhi3Config, CambrianPhi3ForCausalLM
    cfg = CambrianPhi3Config(sliding_window=2047, pad_token_id=32000, max_position_embeddings=4096)
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = CambrianPhi3ForCausalLM(cfg).to(torch.bfloat16).eval()
    wbytes = sum(p.numel() * p.element_size() for n, p in model.named_parameters() if "embed_tokens" not in n)
    floor_ms = wbytes / HBM_BYTES_PER_S * 1e3
    for B in batches:
        ids = torch.randint(3, 32000, (B, prompt), device="cuda")
        prefill = timed(lambda: model.generate(ids, max_new_tokens=1, do_sample=False, eos_token_id=None), 3)
        total = timed(lambda: model.generate(ids, max_new_tokens=new + 1, do_sample=False, eos_token_id=None), 3, warm=1)
        per_tok = (total - prefill) / new
        r = dict(what="generate", batch=B, prompt=prompt, new=new, prefill_ms=round(prefill, 2),
                 decode_ms_per_token=round(per_tok, 3), weight_stream_floor_ms=round(floor_ms, 3),
                 floor_share=round(floor_ms / per_tok, 3), weight_gb=round(wbytes / 1e9, 2))
        print(json.dumps(r), flush=True)
        out.append(r)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", default="1,8")
    ap.add_argument("--prompt", type=int, default=1024)
    ap.add_argument("--new", type=int, default=64)
    ap.add_argument("--out", default=None, help="also write every measurement to this JSON file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("phi3_decode.py measures on the GPU and needs CUDA")
    out = [dict(card=card())]
    print(json.dumps(out[0]), flush=True)
    attention(out)
    decode(out, [int(b) for b in a.batch.split(",")], a.prompt, a.new)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
