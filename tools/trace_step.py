"""Per-stream kernel timeline of ONE training step under torchrun (torch.profiler / CUPTI; nsys is not installed):

    python -m torch.distributed.run --nproc-per-node N ... tools/trace_step.py --gpus N [--config 8b-ddp]

Rank 0 writes trace_out/trace_n{N}.json: per stream {kernels, busy ms, first/last}, the NCCL kernels (count, total ms, how
much of that time a compute kernel was running on another stream = overlapped), main-stream idle gaps, and the step wall
time.  This is the evidence for 'the collectives hide under backward' (or not)."""
import argparse
import gzip
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402


def union_len(iv):
    iv = sorted(iv)
    tot, cs, ce = 0.0, None, None
    for s, e in iv:
        if cs is None:
            cs, ce = s, e
        elif s <= ce:
            ce = max(ce, e)
        else:
            tot += ce - cs
            cs, ce = s, e
    if cs is not None:
        tot += ce - cs
    return tot


def overlap_len(a, b):
    """total length of (union of a) intersected with (union of b)"""
    return union_len(a) + union_len(b) - union_len(a + b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--config", default="8b-ddp")
    ap.add_argument("--max-grad-norm", type=float, default=1.0)
    a = ap.parse_args()
    rank, local, world = int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    import torch.distributed as dist
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    from cambrian_b200.engine import TrainEngine
    from cambrian_b200.model.language_model.cambrian_llama import CambrianLlamaForCausalLM
    C = bench.CONFIGS[a.config]
    cfg = bench.build_config(a.config)
    torch.manual_seed(1234 + rank)
    torch.set_default_dtype(torch.bfloat16)
    with torch.device(dev):
        model = CambrianLlamaForCausalLM(cfg)
        for t in model.get_model().vision_tower_aux_list:
            t.load_model()
    torch.set_default_dtype(torch.float32)
    model.train()
    eng = TrainEngine(model, zero_stage=C["zero"], max_grad_norm=a.max_grad_norm)
    eng.defer_param_sync = True
    db, _ = bench.to_device(bench.make_host_batch(cfg, C["micro_batch"], C["seq"], rank, C["res"], True), dev)

    def step():
        eng.zero_grad()
        out = model(**db)
        out.loss.backward()
        eng.step()

    for _ in range(3):
        step()
    eng.wait_for_params()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        step()
        eng.wait_for_params()
        torch.cuda.synchronize()
    if rank != 0:
        if world > 1:
            dist.barrier()
            dist.destroy_process_group()
        return
    os.makedirs("trace_out", exist_ok=True)
    path = f"trace_out/trace_n{world}_raw.json"
    prof.export_chrome_trace(path)
    ev = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel"]
    with gzip.open(path + ".gz", "wt") as f:
        json.dump([dict(name=e["name"][:80], ts=e["ts"], dur=e["dur"], stream=e["args"].get("stream")) for e in ev], f)
    os.remove(path)
    t0 = min(e["ts"] for e in ev)
    t1 = max(e["ts"] + e["dur"] for e in ev)
    streams = {}
    for e in ev:
        streams.setdefault(e["args"].get("stream"), []).append(e)
    main_stream = max(streams, key=lambda s: sum(e["dur"] for e in streams[s] if "nccl" not in e["name"].lower()))
    nccl = [e for e in ev if "nccl" in e["name"].lower()]
    comp_main = [(e["ts"], e["ts"] + e["dur"]) for e in streams[main_stream]]
    niv = [(e["ts"], e["ts"] + e["dur"]) for e in nccl]
    gaps = []
    cm = sorted(comp_main)
    for (s0, e0), (s1, e1) in zip(cm, cm[1:]):
        if s1 - e0 > 20:
            gaps.append(s1 - e0)
    summ = dict(n_gpus=world, config=a.config, two_steps_wall_ms=(t1 - t0) / 1e3, kernels=len(ev),
                main_stream=main_stream, main_busy_ms=union_len(comp_main) / 1e3,
                main_idle_gaps_over_20us=dict(count=len(gaps), total_ms=sum(gaps) / 1e3, max_ms=max(gaps, default=0) / 1e3),
                nccl=dict(kernels=len(nccl), total_ms=sum(e["dur"] for e in nccl) / 1e3, busy_ms=union_len(niv) / 1e3,
                          overlapped_with_main_stream_kernels_ms=overlap_len(niv, comp_main) / 1e3,
                          longest_ms=max((e["dur"] for e in nccl), default=0) / 1e3,
                          names=sorted({e["name"][:60] for e in nccl})[:6]),
                streams={str(s): dict(kernels=len(v), busy_ms=union_len([(e["ts"], e["ts"] + e["dur"]) for e in v]) / 1e3,
                                      first_ms=(min(e["ts"] for e in v) - t0) / 1e3,
                                      last_ms=(max(e["ts"] + e["dur"] for e in v) - t0) / 1e3,
                                      top=sorted({e["name"][:50] for e in v})[:3]) for s, v in streams.items()})
    json.dump(summ, open(f"trace_out/trace_n{world}.json", "w"), indent=1)
    print(json.dumps({k: v for k, v in summ.items() if k != "streams"}))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
