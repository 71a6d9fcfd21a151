"""The FP8 E4M3 matmuls at the decoder projection shapes of Cambrian-8B (Llama-3-8B) and Cambrian-34B (Yi-34B), next to
the bf16 and LLM.int8 kernels at the same shapes, timed with CUDA events.

    python tools/fp8_shapes.py [--rows 1,8,600,2048] [--iters 20] [--json OUT]

Per (model, projection, M): `cb_fp8_quantize_act` alone, the FP8 product alone (`cb_gemv_fp8` for M <= 8, `cb_gemm_fp8`
above), the int8 product (`cb_gemv_int8` / `cb_gemm_int8`, no outlier columns) and the bf16 product (`ops.gemm`: the
bf16 GEMV for M <= 8 at these widths, the wgmma GEMM above).  GEMM rows report TFLOP/s (2 M N K / t) and the share of the
1,979 TFLOP/s dense FP8 data-sheet figure of the H100 SXM; GEMV rows report weight GB/s (weight bytes / t) and the share
of its 3.35 TB/s.  Weights are cycled through enough copies to exceed L2, so every launch streams them from HBM.  The
card's name, power limit and SM clock are printed with the numbers: they belong to them.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gemm_step_shapes import card_info  # noqa: E402
from int8_shapes import ROTATE_BYTES, projections, timed  # noqa: E402

FP8_PEAK_TFLOPS = 1979.0
HBM_GBPS = 3350.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="1,8,600,2048")
    ap.add_argument("--models", default="8b,yi34b")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    from cambrian_b200 import ops, quant_fp8, quant_int8
    dev = torch.device("cuda")
    card = card_info()
    print(f"# {card['torch_name']} | {card['smi']} (name, power limit, SM clock, max SM clock) | {card['sms']} SMs")
    g = torch.Generator(device=dev).manual_seed(0)
    out = []
    for model in args.models.split(","):
        for name, N, K in projections(model):
            w = (torch.randn(N, K, generator=g, device=dev) * 0.02).to(torch.bfloat16)
            n_copy = max(1, -(-ROTATE_BYTES // (N * K)))
            f8s = [quant_fp8.Fp8Projection(quant_fp8.quantize(w)) for _ in range(n_copy)]
            i8s = [quant_int8.Int8Projection(quant_int8.quantize(w)) for _ in range(n_copy)]
            n_copy_bf = max(1, -(-ROTATE_BYTES // (2 * N * K)))
            ws = [w.clone() for _ in range(n_copy_bf)]
            for M in [int(m) for m in args.rows.split(",")]:
                x = torch.randn(M, K, generator=g, device=dev).to(torch.bfloat16)
                qa = ops.fp8_quantize_act(x)
                qa8 = ops.int8_quantize_act(x, 0.0)
                f8mm, i8mm = (ops.gemv_fp8, ops.gemv_int8) if M <= 8 else (ops.gemm_fp8, ops.gemm_int8)
                c = [0, 0, 0]

                def run_fp8():
                    c[0] = (c[0] + 1) % n_copy
                    f8mm(qa, f8s[c[0]])

                def run_int8():
                    c[1] = (c[1] + 1) % n_copy
                    i8mm(x, qa8, i8s[c[1]])

                def run_bf16():
                    c[2] = (c[2] + 1) % n_copy_bf
                    ops.gemm(x, ws[c[2]])

                t_q = timed(lambda: ops.fp8_quantize_act(x), args.iters)
                t_f8, t_i8, t_bf = timed(run_fp8, args.iters), timed(run_int8, args.iters), timed(run_bf16, args.iters)
                row = dict(model=model, proj=name, M=M, N=N, K=K, kernel="cb_gemv_fp8" if M <= 8 else "cb_gemm_fp8",
                           quant_act_ms=round(t_q, 4), fp8_ms=round(t_f8, 4), int8_ms=round(t_i8, 4),
                           bf16_ms=round(t_bf, 4), fp8_speedup_vs_bf16=round(t_bf / t_f8, 3))
                if M <= 8:
                    gbps = N * K / t_f8 / 1e6
                    row.update(fp8_weight_GBps=round(gbps, 1), fp8_frac_of_3p35TBps=round(gbps / HBM_GBPS, 3),
                               int8_weight_GBps=round(N * K / t_i8 / 1e6, 1), bf16_weight_GBps=round(2 * N * K / t_bf / 1e6, 1))
                else:
                    tf = 2 * M * N * K / t_f8 / 1e9
                    row.update(fp8_TFLOPS=round(tf, 1), fp8_frac_of_1979=round(tf / FP8_PEAK_TFLOPS, 3),
                               int8_TOPS=round(2 * M * N * K / t_i8 / 1e9, 1), bf16_TFLOPS=round(2 * M * N * K / t_bf / 1e9, 1))
                print(json.dumps(row), flush=True)
                out.append(row)
            del f8s, i8s, ws
            torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card, rows=out), f, indent=1)


if __name__ == "__main__":
    main()
