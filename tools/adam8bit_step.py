#!/usr/bin/env python
"""What 8-bit Adam moments (`TrainEngine(optim="adamw_bnb_8bit")`, cb_adamw8 / cb_adamw8_host) change on this GPU.

    python tools/adam8bit_step.py [--config 3b-ddp] [--state device,offload] [--steps 5] [--windows 3] [--warmup 3]
                                  [--loss-steps 10] [--skip-8b] [--json FILE]
    python tools/adam8bit_step.py --kernel [--state-gb 2]

--kernel times cb_adamw8_host on --state-gb of 8-bit state (fp32 master, two codes and two scales per 256 elements) for
each ctas of a sweep, as GB/s of PCIe traffic (12 B per element read and written), next to the copy engines.

For --config (bench.py's model, batch and settings) it runs four arms in one session, alternating 32- and 8-bit moments:
device state 32 / 8, then offloaded state 32 / 8.  Per arm: ms/step over --windows windows of --steps steps after
--warmup, peak allocated device memory, device and registered host state bytes, the optimizer kernels' busy time per
step (CUDA events around every launch) with the bytes they move per step, computed from the layout, and the loss of
each of --loss-steps seeded steps from a fresh model.  Device state is set against 3.35 TB/s (H100 SXM HBM3), offloaded
state against 2 x the PCIe copy-engine rate this tool measures (H2D and D2H at once on registered memory).

Then 8b-ddp with offload and 8-bit moments: the host bytes it needs are printed before anything is built, and the arm
runs only when MemAvailable covers them plus a margin; otherwise it is recorded as not measured.  That arm runs 3 seeded
loss steps, 1 warm-up step and windows of 2 steps.
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

from offload_step import MARGIN_GB, card_info  # noqa: E402

HBM_BPS = 3.35e12


def mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def copy_engine_rate(nbytes=1 << 30):
    """Bytes/s of H2D and D2H at once on registered memory (the PCIe ceiling of the offloaded update)."""
    h = torch.empty(nbytes // 2, dtype=torch.uint8, pin_memory=True)
    h2 = torch.empty(nbytes // 2, dtype=torch.uint8, pin_memory=True)
    d = torch.empty(nbytes // 2, dtype=torch.uint8, device="cuda")
    d2 = torch.empty(nbytes // 2, dtype=torch.uint8, device="cuda")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    best = 0.0
    for _ in range(3):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        s1.wait_event(e0), s2.wait_event(e0)
        with torch.cuda.stream(s1):
            d.copy_(h, non_blocking=True)
        with torch.cuda.stream(s2):
            h2.copy_(d2, non_blocking=True)
        torch.cuda.current_stream().wait_stream(s1), torch.cuda.current_stream().wait_stream(s2)
        e1.record()
        torch.cuda.synchronize()
        best = max(best, nbytes / (e0.elapsed_time(e1) / 1e3))
    return best


def build(config, seed=1234):
    import bench
    from cambrian_b200.model.language_model.cambrian_llama import CambrianLlamaForCausalLM
    cfg = bench.build_config(config)
    torch.manual_seed(seed)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    with torch.device("cuda"):
        model = CambrianLlamaForCausalLM(cfg)
        for t in model.get_model().vision_tower_aux_list:
            t.load_model()
    torch.set_default_dtype(prev)
    model.train()
    model.get_model().gradient_checkpointing = bool(bench.CONFIGS[config].get("recompute", 0))
    return cfg, model


def host_bytes_8bit(config):
    """Registered host bytes of 8-bit offloaded state for `config`, from the parameter shapes (meta device)."""
    import bench
    from cambrian_b200 import adam8bit
    from cambrian_b200.model.language_model.cambrian_llama import CambrianLlamaForCausalLM
    cfg = bench.build_config(config)
    with torch.device("meta"):
        model = CambrianLlamaForCausalLM(cfg)
    emb = adam8bit.embedding_params(model)
    total = 0
    for p in model.parameters():
        if not p.requires_grad:
            continue
        if adam8bit.fp32_moments(p, emb):
            n = (p.numel() + 7) // 8 * 8
            total += 12 * n
        else:
            n = (p.numel() + 255) // 256 * 256
            total += 4 * n + 2 * n + 8 * (n // 256)
    return total


def optimizer_bytes(eng):
    """Bytes the update moves per step, from the layout: 8-bit elements 16 B (g 2, master 8, codes 4, p16 2) plus 16 B of
    scales per block; fp32-moment elements 28 B.  Returns (device-side bytes, bytes over PCIe when offloaded)."""
    n8, n32 = (eng._n8, eng._n32) if eng.eight_bit else (0, eng.master.numel())
    state = 8 * n8 + 4 * n8 + 16 * (n8 // 256) + 24 * n32          # master, codes, scales read and written; fp32 moments
    return state + 4 * (n8 + n32), state


def run_arm(config, optim, offload, args, bw):
    import bench
    from cambrian_b200 import ops
    from cambrian_b200.engine import TrainEngine
    C = bench.CONFIGS[config]
    cfg, model = build(config)
    engine = TrainEngine(model, lr=4e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, zero_stage=C["zero"],
                         max_grad_norm=1.0, bucket_mb=256.0, offload_optimizer=offload, optim=optim)
    names = ("adamw", "adamw8", "adamw_host", "adamw8_host")
    saved = {n: getattr(ops, n) for n in names}
    busy, record = [], [False]

    def wrap(fn):
        def timed(*a, **kw):
            if not record[0]:
                return fn(*a, **kw)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn(*a, **kw)
            e.record()
            busy.append((s, e))
        return timed
    try:
        for n in names:
            setattr(ops, n, wrap(saved[n]))
        engine.defer_param_sync = True
        batch, _ = bench.to_device(bench.make_host_batch(cfg, C["micro_batch"], C["seq"], 0, C["res"], True),
                                   torch.device("cuda"))
        losses = []

        def step():
            engine.zero_grad()
            out = model(**batch)
            out.loss.backward()
            engine.step()
            return out.loss
        for _ in range(args.loss_steps):
            losses.append(step())
        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        losses = [float(x) for x in losses]
        torch.cuda.reset_peak_memory_stats()
        windows = []
        record[0] = True
        for _ in range(args.windows):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step()
            engine.wait_for_params()
            e1.record()
            torch.cuda.synchronize()
            windows.append(e0.elapsed_time(e1) / args.steps)
        record[0] = False
        opt_ms = sum(s.elapsed_time(e) for s, e in busy) / (args.steps * args.windows)
        dev_b, pcie_b = optimizer_bytes(engine)
        moved, ceiling = (pcie_b, bw) if offload else (dev_b, HBM_BPS)
        res = dict(config=config, optim=optim, offload=offload, ms_per_step=windows,
                   optimizer_ms_per_step=opt_ms, optimizer_bytes_per_step=moved,
                   optimizer_gbps=moved / (opt_ms / 1e3) / 1e9, optimizer_ceiling_gbps=ceiling / 1e9,
                   peak_allocated_gb=torch.cuda.max_memory_allocated() / 2 ** 30,
                   device_state_gb=engine.state_bytes() / 2 ** 30, host_state_gb=engine.host_state_bytes() / 2 ** 30,
                   losses=losses)
        print(f"# {config} {optim} offload={offload}: ms/step {' / '.join(f'{w:.1f}' for w in windows)}, optimizer "
              f"{opt_ms:.1f} ms/step at {res['optimizer_gbps']:.0f} GB/s (ceiling {ceiling / 1e9:.0f}), peak "
              f"{res['peak_allocated_gb']:.1f} GB, device state {res['device_state_gb']:.1f} GB, host state "
              f"{res['host_state_gb']:.1f} GB, losses {' '.join(f'{x:.5f}' for x in losses)}", flush=True)
        return res
    finally:
        for n in names:
            setattr(ops, n, saved[n])
        engine.close()
        del engine, model
        torch.cuda.empty_cache()


def kernel_sweep(args, bw):
    from cambrian_b200 import ops
    n = int(args.state_gb * 2 ** 30 / 6.03) // 256 * 256
    nb = n // 256
    host = [torch.zeros(n), torch.zeros(n, dtype=torch.uint8), torch.zeros(n, dtype=torch.uint8), torch.zeros(nb),
            torch.zeros(nb)]
    for t in host:
        ops.host_register(t)
    try:
        g = torch.randn(n, device="cuda").bfloat16()
        p16 = torch.empty(n, device="cuda", dtype=torch.bfloat16)
        out = []
        for ctas in (4, 16, 33, 66, 132, 264, 528):
            def run():
                ops.adamw8_host(*host, g, p16, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, ctas=ctas)
            run()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(3):
                run()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 3
            gbps = (12 * n + 16 * nb) / (ms / 1e3) / 1e9
            out.append(dict(ctas=ctas, ms=ms, pcie_gbps=gbps))
            print(f"# cb_adamw8_host n={n}: ctas {ctas:4d}: {ms:8.1f} ms, {gbps:5.1f} GB/s of PCIe traffic "
                  f"({100 * gbps / (bw / 1e9):.0f} % of the copy engines)", flush=True)
        return out
    finally:
        torch.cuda.synchronize()
        for t in host:
            ops.host_unregister(t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kernel", action="store_true")
    ap.add_argument("--state-gb", type=float, default=2.0)
    ap.add_argument("--config", default="3b-ddp")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--loss-steps", type=int, default=10)
    ap.add_argument("--skip-8b", action="store_true")
    ap.add_argument("--state", default="device,offload", help="which arms: device and / or offload state")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    card = card_info()
    print(f"# {card}", flush=True)
    bw = copy_engine_rate()
    print(f"# copy engines, H2D + D2H at once: {bw / 1e9:.1f} GB/s", flush=True)
    out = dict(card=card, copy_engine_gbps=bw / 1e9, arms=[])
    if args.kernel:
        out["kernel"] = kernel_sweep(args, bw)
        if args.json:
            with open(args.json, "w") as f:
                json.dump(out, f, indent=1)
        return
    for offload in [s == "offload" for s in args.state.split(",")]:
        for optim in ("adamw_torch", "adamw_bnb_8bit"):
            out["arms"].append(run_arm(args.config, optim, offload, args, bw))
    if not args.skip_8b:
        try:
            need = host_bytes_8bit("8b-ddp")
        except Exception as e:      # the shapes could not be built on the meta device: nothing is registered blind
            print(f"# 8b-ddp: not measured (host bytes unknown: {e})", flush=True)
            need = float("inf")
        avail = mem_available()
        print(f"# 8b-ddp offload, 8-bit moments: {need / 2 ** 30:.1f} GB of registered host state needed, "
              f"{avail / 2 ** 30:.1f} GB available", flush=True)
        if need + MARGIN_GB * 2 ** 30 > avail:
            out["8b-ddp"] = dict(host_state_gb=need / 2 ** 30, available_gb=avail / 2 ** 30, result="not measured")
            print("# 8b-ddp: not measured (host memory)", flush=True)
        else:
            short = argparse.Namespace(**{**vars(args), "loss_steps": 3, "warmup": 1, "steps": 2})
            try:
                out["8b-ddp"] = run_arm("8b-ddp", "adamw_bnb_8bit", True, short, bw)
            except torch.OutOfMemoryError as e:
                out["8b-ddp"] = dict(host_state_gb=need / 2 ** 30, result="not measured", reason=f"device OOM: {e}"[:300])
                print("# 8b-ddp: not measured (device out of memory)", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
