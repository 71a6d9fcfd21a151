"""Single-GPU decode latency of the Cambrian-8B-shaped model (A12): ms/token of the KV-cache greedy loop after a multimodal
prefill, against the weight-streaming floor (bf16 weights / measured HBM bandwidth).

    python tools/decode_bench.py [--batch 1] [--prompt 1024] [--new 64] [--config 8b-ddp | yi34b] [--load-4bit | --load-8bit]

--load-4bit quantises the decoder projections to NF4 (cambrian_b200/quant.py), --load-8bit to LLM.int8
(cambrian_b200/quant_int8.py), layer by layer after building the model on the CPU, so configurations whose bf16 decoder
does not fit one GPU (--config yi34b: Cambrian-34B-shaped, 60 layers) run.  8-bit takes precedence, as in the loader.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", default="1", help="batch size, or a comma-separated list (one JSON line each, one model build)")
    ap.add_argument("--prompt", type=int, default=1024)
    ap.add_argument("--new", type=int, default=64)
    ap.add_argument("--config", default="8b-ddp")
    ap.add_argument("--no-graph", action="store_true", help="eager per-token loop instead of the CUDA-graph replay")
    ap.add_argument("--profile", action="store_true", help="kernel time per token by kernel name (torch.profiler)")
    ap.add_argument("--load-4bit", action="store_true", help="NF4 decoder projections (quant.quantize_decoder_nf4_)")
    ap.add_argument("--load-8bit", action="store_true", help="LLM.int8 decoder projections (quant_int8)")
    ap.add_argument("--layers", type=int, default=60, help="decoder layers of --config yi34b")
    args = ap.parse_args()
    from cambrian_b200 import quant, quant_int8
    from cambrian_b200.model.language_model.cambrian_llama import CambrianLlamaForCausalLM
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    if args.config == "yi34b":
        from zero3_generate import yi34b_config
        cfg = yi34b_config(args.layers)
    else:
        cfg = bench.build_config(args.config)
    cfg.inputs_pre_expanded = False
    cfg.disable_decode_graph = args.no_graph
    torch.manual_seed(0)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    qstats = None
    quantize = (quant_int8.quantize_decoder_int8_ if args.load_8bit else
                quant.quantize_decoder_nf4_ if args.load_4bit else None)
    if quantize is not None and args.config == "yi34b":
        # built on the CPU (a 34B decoder does not fit the GPU in bf16), quantised onto the GPU one layer at a time
        model = CambrianLlamaForCausalLM(cfg)
        qstats = quantize(model, dev)
        model.to(dev)
        with torch.device(dev):
            for t in model.get_model().vision_tower_aux_list:
                t.load_model()
    else:
        with torch.device(dev):
            model = CambrianLlamaForCausalLM(cfg)
            for t in model.get_model().vision_tower_aux_list:
                t.load_model()
        if quantize is not None:
            qstats = quantize(model, dev)
            torch.cuda.empty_cache()
    torch.set_default_dtype(prev)
    model.eval()
    torch.cuda.reset_peak_memory_stats()
    model._bench_qstats = qstats
    for B in [int(b) for b in str(args.batch).split(",")]:
        one_batch(args, model, cfg, dev, B)


def one_batch(args, model, cfg, dev, B):
    from cambrian_b200 import _lib
    C = bench.CONFIGS["8b-ddp"] if args.config == "yi34b" else bench.CONFIGS[args.config]
    ids = torch.randint(3, cfg.vocab_size, (B, args.prompt - 599), device=dev)
    ids[:, cfg.image_position] = -200
    images = [torch.randn(B, 3, r, r, device=dev).bfloat16() for r in C["res"]]
    kw = dict(images=images, image_sizes=[(336, 336)] * B, do_sample=False)

    def run(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        l0 = _lib.load().cb_launch_count()
        e0.record()
        out = model.generate(ids, max_new_tokens=n, **kw)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), _lib.load().cb_launch_count() - l0, out

    run(2)
    run(2)
    t1, l1, _ = run(1)
    tn, ln, out = run(args.new + 1)
    ms_tok = (tn - t1) / args.new
    # weight bytes one decode step streams: decoder layers (bf16, NF4 or int8) + norms + lm_head
    qstats = model._bench_qstats
    n_params = sum(p.numel() for n, p in model.named_parameters() if "vision" not in n and "mm_projector" not in n
                   and "embed_tokens" not in n)
    q_bytes = (qstats.get("nf4_bytes") or qstats.get("int8_bytes")) if qstats else None
    weight_bytes = n_params * 2 + (q_bytes or 0)
    hbm = bench.peaks()[0]
    floor = weight_bytes / (hbm * 1e9) * 1e3
    top = None
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run(args.new + 1)
        agg = {}
        for e in prof.events():
            if e.device_type is not None and "cuda" in str(e.device_type).lower() and e.device_time > 0:
                a_ = agg.setdefault(e.name[:70], [0.0, 0])
                a_[0] += e.device_time
                a_[1] += 1
        top = [dict(kernel=k, ms_per_token=round(v[0] / 1e3 / args.new, 4), launches_per_token=round(v[1] / args.new, 1))
               for k, v in sorted(agg.items(), key=lambda kv: -kv[1][0])[:14]]
    print(json.dumps(dict(metric="decode_ms_per_token", value=ms_tok, unit="ms", config=args.config, load_4bit=args.load_4bit and not args.load_8bit,
                          load_8bit=args.load_8bit,
                          batch=B, prompt=args.prompt, new_tokens=args.new, prefill_ms=t1, tokens_per_s=B * 1000.0 / ms_tok,
                          launches_per_token=(ln - l1) / args.new, decode_graph=not args.no_graph, weight_bytes=weight_bytes,
                          decoder_nf4_bytes=qstats.get("nf4_bytes") if qstats else None,
                          decoder_int8_bytes=qstats.get("int8_bytes") if qstats else None,
                          peak_mem_gb=torch.cuda.max_memory_allocated() / 2 ** 30, gpu=torch.cuda.get_device_name(0),
                          floor_ms=floor, frac_of_floor=floor / ms_tok,
                          note="floor = weight bytes per step (decoder bf16, NF4 or int8, lm_head bf16) / measured HBM copy "
                               "bandwidth", top_kernels=top)),
          flush=True)


if __name__ == "__main__":
    main()
