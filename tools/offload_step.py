#!/usr/bin/env python
"""What keeping the AdamW state in host memory (`TrainEngine(offload_optimizer=True)`, cb_adamw_host) costs on this GPU.

    python tools/offload_step.py --kernel [--state-gb 2]            # kernel GB/s against ctas, next to the copy engines
    python tools/offload_step.py --coresidency                       # GEMM / attention-backward slowdown under the kernel
    python tools/offload_step.py --config 3b-ddp|8b-ddp [--no-offload] [--recompute 0|1] [--steps K] [--warmup W]
                                 [--dump-outputs DIR]

--kernel times cb_adamw_host on a --state-gb state (fp32 master + 2 moments, 12 B per element) for every ctas of the
sweep.  PCIe traffic is 24 B per element (12 read, 12 written); the device adds 4 B (bf16 gradient in, bf16 copy out).
In the same call the copy engines move the same bytes (H2D and D2H at once, registered memory): the ceiling the kernel
is measured against.

--coresidency times the decoder GEMM shapes of 8b-ddp (tools/gemm_step_shapes.py) and the decoder's attention backward
(tools/attn_step_shapes.py) alone, then while the kernel runs on a side stream at the default ctas.

--config builds bench.py's model, batch and engine (same seeds, same settings) with the optimizer state offloaded, and
reports ms/step in steady state, peak device memory, registered host memory and the optimizer kernel's busy time per
step.  --dump-outputs writes loss.npy / params_sample.npy exactly as `bench.py --dump-outputs` does.

Host memory is checked against MemAvailable (plus an 8 GB margin) before anything is registered, and every registration is
undone on the way out.  The card's name, power limit, max SM clock and PCIe link are printed with the numbers.
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

SWEEP_CTAS = (4, 8, 16, 32, 64, 132)
MARGIN_GB = 8.0


def card_info():
    q = "name,power.limit,clocks.max.sm,pcie.link.gen.current,pcie.link.width.current"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception as e:
        out = f"nvidia-smi unavailable: {e}"
    return f"{torch.cuda.get_device_name()} | {out} (name, power limit, max SM clock, PCIe gen, PCIe width)"


def require_host_memory(nbytes):
    avail = 0
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                avail = int(line.split()[1]) * 1024
    if nbytes + MARGIN_GB * 2 ** 30 > avail:
        raise SystemExit(f"offload_step.py: {nbytes / 2 ** 30:.1f} GB of host state + {MARGIN_GB:.0f} GB margin does not fit "
                         f"the {avail / 2 ** 30:.1f} GB this host has available; nothing was registered")
    return avail


def events_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


class HostState:
    """n fp32 elements of master / exp_avg / exp_avg_sq in registered host memory (+ `extra` registered bytes)."""

    def __init__(self, n, extra_bytes=0):
        from cambrian_b200 import ops
        self.ops = ops
        require_host_memory(12 * n + extra_bytes)
        self.tensors = []
        self.p, self.m, self.v = (self._reg(torch.randn(n)), self._reg(torch.randn(n) * 1e-2),
                                  self._reg(torch.rand(n) * 1e-4))
        self.extra = self._reg(torch.empty(extra_bytes, dtype=torch.uint8)) if extra_bytes else None

    def _reg(self, t):
        self.ops.host_register(t)
        self.tensors.append(t)
        return t

    def close(self):
        torch.cuda.synchronize()
        for t in self.tensors:
            self.ops.host_unregister(t)
        self.tensors = []


def kernel_sweep(args):
    from cambrian_b200 import ops
    n = int(args.state_gb * 1e9 / 12) // 1024 * 1024
    g = torch.randn(n, device="cuda").bfloat16()
    p16 = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    st = HostState(n, extra_bytes=12 * n)
    try:
        run = lambda c: ops.adamw_host(st.p, st.m, st.v, g, p16, 1e-5, 0.9, 0.999, 1e-8, 0.0, 5, ctas=c)
        # copy-engine ceiling: the same 12 n bytes up and 12 n bytes down at once, registered memory both ways
        up = torch.empty(3 * n, device="cuda")
        down = torch.empty(3 * n, device="cuda")
        s_up, s_down = torch.cuda.Stream(), torch.cuda.Stream()
        host_down = st.extra.view(torch.float32)

        def copies():
            cur = torch.cuda.current_stream()
            s_up.wait_stream(cur), s_down.wait_stream(cur)
            with torch.cuda.stream(s_up):
                for i, t in enumerate((st.p, st.m, st.v)):
                    up[i * n:(i + 1) * n].copy_(t, non_blocking=True)
            with torch.cuda.stream(s_down):
                host_down.copy_(down, non_blocking=True)
            cur.wait_stream(s_up), cur.wait_stream(s_down)
        copies()
        run(0)
        torch.cuda.synchronize()
        ce_ms = events_ms(copies, args.reps)
        ceiling = 24.0 * n / ce_ms / 1e6
        print(f"# state {12 * n / 1e9:.2f} GB ({n} elements); copy engines, H2D + D2H of {12 * n / 1e9:.2f} GB each at once: "
              f"{ce_ms:.1f} ms = {ceiling:.1f} GB/s over PCIe (the ceiling below)")
        print(f"{'ctas':>5s} {'ms':>9s} {'PCIe GB/s':>10s} {'of ceiling':>10s} {'+device GB/s':>12s}")
        rows = []
        for c in (0,) + SWEEP_CTAS:
            run(c)
            ms = events_ms(lambda: run(c), args.reps)
            pcie = 24.0 * n / ms / 1e6
            rows.append(dict(ctas=c, ms=ms, pcie_gbs=pcie, share_of_ceiling=pcie / ceiling, total_gbs=28.0 * n / ms / 1e6))
            print(f"{c if c else 'def':>5} {ms:9.2f} {pcie:10.1f} {pcie / ceiling:10.2f} {28.0 * n / ms / 1e6:12.1f}", flush=True)
        return dict(state_bytes=12 * n, copy_engine_ms=ce_ms, ceiling_gbs=ceiling, sweep=rows)
    finally:
        st.close()


def coresidency(args):
    """Each operation timed alone, then while the offload kernel streams a state large enough to outlast it."""
    import attn_step_shapes as A
    import gemm_step_shapes as G
    from cambrian_b200 import ops
    n = int(args.state_gb * 1e9 / 12) // 1024 * 1024
    g = torch.randn(n, device="cuda").bfloat16()
    p16 = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    st = HostState(n)
    side = torch.cuda.Stream()
    try:
        def offload():
            ops.adamw_host(st.p, st.m, st.v, g, p16, 1e-5, 0.9, 0.999, 1e-8, 0.0, 5)
        offload()
        torch.cuda.synchronize()
        k_ms = events_ms(offload, 1)
        cases = []
        for name, _, s in G.step_shapes("8b-ddp"):
            if name.startswith("dec."):
                a, b, extra = G.make_operands(s, torch.Generator(device="cuda").manual_seed(0), "cuda")
                out = torch.zeros((s["M"], s["N"]), dtype=torch.bfloat16, device="cuda")
                out2 = torch.empty((s["M"], s["N"] // 2), dtype=torch.bfloat16, device="cuda") if s["swiglu"] else None
                cases.append((name, lambda s=s, a=a, b=b, e=extra, o=out, o2=out2: G.run_ours(s, a, b, e, o, o2)))
        for name, _, s in A.step_shapes("8b-ddp"):
            if name == "dec bwd kmask":
                x = A.make_inputs(s, 0)
                cases.append(("attn " + name, A.run_fns(s, x)[1]))
        print(f"# offload kernel alone at the default ctas: {k_ms:.1f} ms for {12 * n / 1e9:.2f} GB of state")
        print(f"{'operation':28s} {'alone ms':>9s} {'with ms':>9s} {'slowdown':>9s} {'covered':>8s}")
        rows = []
        for name, fn in cases:
            fn()
            torch.cuda.synchronize()
            alone = events_ms(fn, args.iters)
            iters = max(1, min(args.iters, int(0.8 * k_ms / alone)))    # the window must end before the kernel does
            torch.cuda.synchronize()
            k0, k1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(side):
                k0.record()
                offload()
                k1.record()
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            with_ms = e0.elapsed_time(e1) / iters
            covered = k0.elapsed_time(e0) >= 0 and k0.elapsed_time(k1) >= k0.elapsed_time(e1)
            rows.append(dict(op=name, alone_ms=alone, with_ms=with_ms, slowdown=with_ms / alone - 1, iters=iters,
                             covered=covered))
            print(f"{name:28s} {alone:9.3f} {with_ms:9.3f} {100 * (with_ms / alone - 1):8.1f}% {str(covered):>8s}", flush=True)
        return dict(offload_ms=k_ms, state_bytes=12 * n, ops=rows)
    finally:
        st.close()


def train_config(args):
    import bench
    from cambrian_b200 import ops
    from cambrian_b200.engine import TrainEngine
    from cambrian_b200.model.language_model.cambrian_llama import CambrianLlamaForCausalLM
    dev = torch.device("cuda", 0)
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
    recompute = C.get("recompute", 0) if args.recompute < 0 else args.recompute
    model.get_model().gradient_checkpointing = bool(recompute)
    offload = not args.no_offload
    if offload:
        n_state = sum((p.numel() + 7) // 8 * 8 for p in model.parameters() if p.requires_grad)
        require_host_memory(12 * n_state)
    engine = TrainEngine(model, lr=4e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, zero_stage=C["zero"],
                         max_grad_norm=1.0, bucket_mb=256.0, offload_optimizer=offload)
    try:
        engine.defer_param_sync = True
        batch, _ = bench.to_device(bench.make_host_batch(cfg, C["micro_batch"], C["seq"], 0, C["res"], True), dev)
        busy = []
        fn = ops.adamw_host if offload else ops.adamw

        def timed(*a, **kw):
            if record[0]:
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                fn(*a, **kw)
                e.record()
                busy.append((s, e))
            else:
                fn(*a, **kw)
        record = [False]
        setattr(ops, fn.__name__, timed)

        def step():
            engine.zero_grad()
            out = model(**batch)
            out.loss.backward()
            engine.step()
            return out.loss
        for _ in range(max(1, args.warmup)):
            loss = step()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        record[0] = True
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            loss = step()
        engine.wait_for_params()
        e1.record()
        torch.cuda.synchronize()
        record[0] = False
        setattr(ops, fn.__name__, fn)
        ms = e0.elapsed_time(e1) / args.steps
        opt_ms = sum(s.elapsed_time(e) for s, e in busy) / args.steps
        res = dict(config=args.config, offload=offload, ms_per_step=ms, optimizer_ms_per_step=opt_ms,
                   optimizer_share=opt_ms / ms, peak_device_gb=torch.cuda.max_memory_allocated() / 2 ** 30,
                   device_state_gb=engine.state_bytes() / 2 ** 30, host_state_gb=engine.host_state_bytes() / 2 ** 30,
                   trainable_params=sum(p.numel() for p in engine.params), loss=float(loss.detach()),
                   steps=args.steps, warmup=args.warmup, recompute=bool(recompute))
        print(f"# {args.config} offload={offload}: {ms:.1f} ms/step, optimizer kernel {opt_ms:.1f} ms/step "
              f"({100 * opt_ms / ms:.0f} % of the step), peak device {res['peak_device_gb']:.1f} GB, registered host "
              f"{res['host_state_gb']:.1f} GB, loss {res['loss']:.6f}")
        if args.dump_outputs:
            bench.dump_outputs(args.dump_outputs, loss, model)
        return res
    finally:
        engine.close()


def main():
    ap = argparse.ArgumentParser()
    mode = ap.add_mutually_exclusive_group(required=True)
    mode.add_argument("--kernel", action="store_true")
    mode.add_argument("--coresidency", action="store_true")
    mode.add_argument("--config", choices=["3b-ddp", "8b-ddp"])
    ap.add_argument("--no-offload", action="store_true", help="--config with the optimizer state on the device")
    ap.add_argument("--recompute", type=int, default=-1, help="--config per-layer activation recompute 1 / 0 (default: the "
                                                               "config's own, as bench.py)")
    ap.add_argument("--state-gb", type=float, default=2.0, help="--kernel / --coresidency state size (12 B per element)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    ap.add_argument("--json", default=None, help="also write the results here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("offload_step.py measures on the GPU: no CUDA device is visible")
    torch.cuda.set_device(0)
    card = card_info()
    print(f"# {card}")
    res = kernel_sweep(args) if args.kernel else coresidency(args) if args.coresidency else train_config(args)
    res["card"] = card
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
