"""Cambrian-Phi3-3B fine-tuning on one GPU: the head-dim-96 / sliding-window flash-attention backward on its own, and
training steps of a random Phi-3-mini-shaped text decoder (hidden 3072, 32 heads of 96, intermediate 8192, vocab 32064,
sliding window 2047) under TrainEngine with per-layer recompute.

    python tools/phi3_train_step.py [--layers 32] [--seq 4096] [--batch 1] [--steps 5] [--offload] [--out FILE]

Prints one JSON line per measurement, the first with the card's name, power limit and max SM clock, and with --out also
writes them all to FILE as one JSON list:
  * attention backward TF/s (dq + dk + dv: 10 * B * nh * hd FLOPs per visible (query, key) pair, 2.5 x the forward's)
    of hd 96 at S = 2048 and 4096 (W = 2047) next to hd 128 at the Llama-3-8B shape, and the windowed (W = 2047)
    against the plain causal backward at S = 4096;
  * ms / step, tokens / s and peak memory of TrainEngine steps (forward, backward, AdamW) on seeded batches.
    --offload keeps the AdamW state in pinned host memory (`offload_optimizer=True`), for when the device cannot hold
    weights, gradients, fp32 masters and both moments at once.
Times are CUDA-event means after warm-up.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from phi3_decode import card, timed, visible_pairs  # noqa: E402


def attention_bwd(out):
    from cambrian_b200 import ops
    rows = []
    for name, B, S, nh, nkv, hd, W in (("phi3", 1, 2048, 32, 32, 96, 2047),
                                       ("phi3", 1, 4096, 32, 32, 96, 2047),
                                       ("phi3, no window", 1, 4096, 32, 32, 96, 0),
                                       ("llama3-8b", 1, 2048, 32, 8, 128, 0)):
        g = torch.Generator(device="cuda").manual_seed(S + hd)
        q = torch.randn(B, S, nh, hd, device="cuda", generator=g).bfloat16()
        k = torch.randn(B, S, nkv, hd, device="cuda", generator=g).bfloat16()
        v = torch.randn(B, S, nkv, hd, device="cuda", generator=g).bfloat16()
        do = torch.randn(B, S, nh, hd, device="cuda", generator=g).bfloat16()
        win = {"window": W} if W else {}
        o, lse = ops.attn_fwd(q, k, v, causal=True, need_lse=True, **win)
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        ms = timed(lambda: ops.attn_bwd(q, k, v, o, do, lse, causal=True, dq=dq, dk=dk, dv=dv, **win), 20)
        flops = 10.0 * B * nh * hd * visible_pairs(S, W)
        r = dict(what="attn_bwd", shape=name, B=B, S=S, nh=nh, nkv=nkv, hd=hd, window=W, ms=round(ms, 4),
                 tflops=round(flops / ms / 1e9, 1))
        rows.append(r)
        print(json.dumps(r), flush=True)
    w = next(r for r in rows if r["S"] == 4096 and r["window"])
    n = next(r for r in rows if r["S"] == 4096 and not r["window"])
    r = dict(what="windowed vs causal backward at S=4096", ms_window=w["ms"], ms_full_causal=n["ms"],
             pair_share=round(visible_pairs(4096, 2047) / visible_pairs(4096, 0), 3),
             saved_pct=round(100 * (1 - w["ms"] / n["ms"]), 1))
    print(json.dumps(r), flush=True)
    out.extend(rows + [r])


def train_steps(out, layers, seq, batch, steps, offload):
    from cambrian_b200.engine import TrainEngine
    from cambrian_b200.model.language_model.cambrian_phi3 import CambrianPhi3Config, CambrianPhi3ForCausalLM
    cfg = CambrianPhi3Config(num_hidden_layers=layers, sliding_window=2047, pad_token_id=32000,
                             max_position_embeddings=max(4096, seq))
    cfg.fused_lm_loss = True
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = CambrianPhi3ForCausalLM(cfg).to(torch.bfloat16).train()
    model.gradient_checkpointing = model.get_model().gradient_checkpointing = True
    eng = TrainEngine(model, lr=1e-5, offload_optimizer=offload)
    g = torch.Generator(device="cuda").manual_seed(1)
    batches = [torch.randint(3, 32000, (batch, seq), device="cuda", generator=g) for _ in range(2)]
    it = [0]

    def step():
        ids = batches[it[0] % 2]
        it[0] += 1
        eng.zero_grad()
        loss = model(input_ids=ids, labels=ids).loss
        loss.backward()
        eng.step()
        return loss

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ms = timed(step, steps, warm=0)
    r = dict(what="train step", layers=layers, batch=batch, seq=seq, window=2047, recompute=True,
             offload_optimizer=offload, params_b=round(sum(p.numel() for p in model.parameters()) / 1e9, 3),
             ms_per_step=round(ms, 1), tokens_per_s=round(batch * seq / ms * 1e3), peak_gb=round(
                 torch.cuda.max_memory_allocated() / 1e9, 2), final_loss=round(float(step().item()), 4))
    print(json.dumps(r), flush=True)
    out.append(r)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--seq", type=int, default=4096)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--offload", action="store_true", help="AdamW state in pinned host memory (offload_optimizer)")
    ap.add_argument("--skip-attention", action="store_true")
    ap.add_argument("--out", default=None, help="also write every measurement to this JSON file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("phi3_train_step.py measures on the GPU and needs CUDA")
    out = [dict(card=card())]
    print(json.dumps(out[0]), flush=True)
    if not a.skip_attention:
        attention_bwd(out)
    train_steps(out, a.layers, a.seq, a.batch, a.steps, a.offload)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
