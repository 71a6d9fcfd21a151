"""Kernel time of ops.sample_tokens (csrc/sample.cu) against the torch path it replaces (generation.warp_logits + softmax
+ torch.multinomial, one call over all rows), with CUDA events, over the vocabularies of the supported decoders.

    python tools/sample_shapes.py [--iters 50] [--out FILE]

Grid: V in {32000 (Vicuna), 32064 (Phi-3), 64000 (Yi), 128256 (Llama-3)}, rows in {1, 8, 32, 128}, and (T, top_k, top_p)
in {(1, 50, 1): HF's top-k default, (0.2, 50, 0.7): the model worker's defaults, (0.7, 0, 0.9): top-p alone}.  One JSON
line per shape, with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def timed(fn, iters):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1000.0 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sample_shapes.py measures on a GPU; none is visible")
    from cambrian_b200 import ops
    from cambrian_b200.generation import warp_logits
    dev = torch.device("cuda")
    name = card()
    lines = []
    for V in (32000, 32064, 64000, 128256):
        for rows in (1, 8, 32, 128):
            logits = torch.randn(rows, V, device=dev, generator=torch.Generator(device=dev).manual_seed(V + rows)) * 2.5
            for T, k, p in ((1.0, 50, 1.0), (0.2, 50, 0.7), (0.7, 0, 0.9)):
                prm = (torch.full((rows,), T, device=dev), torch.full((rows,), k, dtype=torch.int32, device=dev),
                       torch.full((rows,), p, device=dev), torch.arange(rows, device=dev) * 7919 + 1,
                       torch.zeros(rows, dtype=torch.long, device=dev))
                out = torch.empty(rows, dtype=torch.long, device=dev)
                gen = torch.Generator(device=dev).manual_seed(0)
                kern = timed(lambda: ops.sample_tokens(logits, *prm, out=out), args.iters)
                ref = timed(lambda: torch.multinomial(warp_logits(logits, T, k, p).softmax(-1), 1, generator=gen),
                            args.iters)
                line = dict(V=V, rows=rows, T=T, top_k=k, top_p=p, kernel_us=round(kern, 2), torch_us=round(ref, 2),
                            speedup=round(ref / kern, 2), card=name)
                print(json.dumps(line), flush=True)
                lines.append(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
