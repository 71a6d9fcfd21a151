"""The LLM.int8 matmuls at the decoder projection shapes of Cambrian-8B (Llama-3-8B) and Cambrian-34B (Yi-34B), next to
the bf16 kernels at the same shapes, timed with CUDA events.

    python tools/int8_shapes.py [--rows 1,8,600,2048] [--outliers 0] [--iters 20] [--json OUT]

Per (model, projection, M): `cb_int8_quantize_act` alone, the int8 product alone (`cb_gemv_int8` for M <= 8,
`cb_gemm_int8` above), and the bf16 product (`ops.gemm`, which is the bf16 GEMV for M <= 8 at these widths and the
wgmma GEMM above).  GEMM rows report TOPS (2 M N K / t), GEMV rows weight GB/s (weight bytes / t).  Weights are cycled
through enough copies to exceed L2, so every launch streams them from HBM.  The activations are N(0, 1) in bf16, with
--outliers columns raised to 8.0 in one row; the outlier count the quantiser found is reported.  The card's name, power
limit and SM clock are printed with the numbers: they belong to them.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gemm_step_shapes import card_info  # noqa: E402

ROTATE_BYTES = 200 * 2 ** 20

MODELS = {
    # hidden, intermediate, heads, kv heads, head_dim
    "8b": (4096, 14336, 32, 8, 128),
    "yi34b": (7168, 20480, 56, 8, 128),
}


def projections(model):
    H, I, nh, nkv, hd = MODELS[model]
    return [("qkv", (nh + 2 * nkv) * hd, H), ("o", H, nh * hd), ("gate_up", 2 * I, H), ("down", H, I)]


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="1,8,600,2048")
    ap.add_argument("--models", default="8b,yi34b")
    ap.add_argument("--outliers", type=int, default=0)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    from cambrian_b200 import ops, quant_int8
    dev = torch.device("cuda")
    card = card_info()
    print(f"# {card['torch_name']} | {card['smi']} (name, power limit, SM clock, max SM clock) | {card['sms']} SMs")
    g = torch.Generator(device=dev).manual_seed(0)
    out = []
    for model in args.models.split(","):
        for name, N, K in projections(model):
            w = (torch.randn(N, K, generator=g, device=dev) * 0.02).to(torch.bfloat16)
            n_copy = max(1, -(-ROTATE_BYTES // (N * K)))
            qws = [quant_int8.Int8Projection(quant_int8.quantize(w)) for _ in range(n_copy)]
            n_copy_bf = max(1, -(-ROTATE_BYTES // (2 * N * K)))
            ws = [w.clone() for _ in range(n_copy_bf)]
            for M in [int(m) for m in args.rows.split(",")]:
                x = torch.randn(M, K, generator=g, device=dev)
                if args.outliers:
                    cols = torch.randperm(K, generator=g, device=dev)[: args.outliers]
                    x[0, cols] = 8.0
                x = x.to(torch.bfloat16)
                qa = ops.int8_quantize_act(x, quant_int8.THRESHOLD)
                n_out = int(qa[3].item())
                mm = ops.gemv_int8 if M <= 8 else ops.gemm_int8
                i = [0]

                def run_int8():
                    i[0] = (i[0] + 1) % n_copy
                    mm(x, qa, qws[i[0]])

                j = [0]

                def run_bf16():
                    j[0] = (j[0] + 1) % n_copy_bf
                    ops.gemm(x, ws[j[0]])

                t_q = timed(lambda: ops.int8_quantize_act(x, quant_int8.THRESHOLD), args.iters)
                t_i8 = timed(run_int8, args.iters)
                t_bf = timed(run_bf16, args.iters)
                row = dict(model=model, proj=name, M=M, N=N, K=K, kernel="cb_gemv_int8" if M <= 8 else "cb_gemm_int8",
                           outliers=n_out, quant_act_ms=round(t_q, 4), int8_ms=round(t_i8, 4), bf16_ms=round(t_bf, 4),
                           int8_vs_bf16=round(t_bf / t_i8, 3))
                if M <= 8:
                    row.update(int8_weight_GBps=round(N * K / t_i8 / 1e6, 1), bf16_weight_GBps=round(2 * N * K / t_bf / 1e6, 1))
                else:
                    row.update(int8_TOPS=round(2 * M * N * K / t_i8 / 1e9, 1), bf16_TFLOPS=round(2 * M * N * K / t_bf / 1e9, 1))
                print(json.dumps(row), flush=True)
                out.append(row)
            del qws, ws
            torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card, rows=out), f, indent=1)


if __name__ == "__main__":
    main()
