"""Serving throughput of the Cambrian-8B-shaped random model on one GPU: continuous batching over the paged KV cache
(cambrian_b200/serving.py) against sequential generate() and static batches of generate() with left padding, on the
same seeded request mix, in one session, alternated.

    python tools/serve_bench.py [--requests 64] [--max-batch 32] [--rounds 2] [--load-fp8] [--kv-fp8] [--out FILE]
                                [--prefix-cache] [--mix random|shared]

The mix: every request has one image and a text prompt of 64-448 tokens (at least the config's image position, 91
for the 8B config; plus the 600-position image span), and
max_new_tokens drawn from 16-256; EOS is off, so every request runs to its max_new_tokens and the three ways of serving
do the same work.  Reported per way: generated tokens / s and wall time (host clock around work that ends in a device
synchronise), peak device allocation; for the server also the decode-step latency per bucket, the page pool's bytes and
the paged attention kernel's time at the mix's lengths (CUDA events) with its bytes / s against the 3.35 TB/s HBM3
figure of the H100 SXM data sheet (bytes computed from the lengths).  One server serves the warm-up and every timed run,
so its page pool and its per-bucket CUDA graphs are built before the clock starts, as in a long-running server; each
`generate()` call builds its own cache and graph inside its timed run, as it does in use.  Each request's greedy tokens are compared with the
sequential run's: where they differ, the first differing step and the sequential run's top-1 / top-2 logit margin there.
The card's name, power limit and max SM clock are read in the same call and printed with the numbers.
`--prefix-cache` serves the random mix with BatchedGenerator(prefix_cache=True) (its prompts share nothing, so this
measures the cache's bookkeeping).

`--mix shared` measures the prefix cache on the traffic it is for: per round, 8 images with 6 questions each (one system
prompt up to the image position, the image, a question of 8-64 tokens) and 8 three-turn conversations about their own
image (each turn resends the previous turn, its answer and a new question), arriving in three waves: the first turns
with all questions, then the second turns, then the third.  Two servers, one with the prefix cache and one without,
are each warmed up once on a mix of another seed and then timed alternately, each round on a fresh mix (so no round
hits on pages of an earlier one).  Reported per server: generated tokens / s, mean and p90 time to first token (from a
wave's submit to the request's first token), the hit rate and cached pages; then the gather kernel's time (CUDA events)
at the mix's hit lengths, with its bytes / s against 3.35 TB/s.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def card_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception as e:
        out = f"nvidia-smi unavailable: {e}"
    return f"{torch.cuda.get_device_name()} | {out} (name, power limit, max SM clock)"


def build_model(args, dev):
    from cambrian_b200 import quant_fp8
    from cambrian_b200.model.language_model.cambrian_llama import CambrianLlamaForCausalLM
    cfg = bench.build_config("8b-ddp")
    cfg.inputs_pre_expanded = False
    torch.manual_seed(0)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    with torch.device(dev):
        model = CambrianLlamaForCausalLM(cfg)
        for t in model.get_model().vision_tower_aux_list:
            t.load_model()
    torch.set_default_dtype(prev)
    if args.load_fp8:
        quant_fp8.quantize_decoder_fp8_(model, dev)
        torch.cuda.empty_cache()
    return cfg, model.eval()


def request_mix(cfg, n, seed, dev):
    g = torch.Generator().manual_seed(seed)
    res = bench.CONFIGS["8b-ddp"]["res"]
    reqs = []
    for _ in range(n):
        # T text tokens and the <image> indicator at the config's image position (the in-LLM SVA sites read the image
        # span there), so a prompt holds at least image_position text tokens
        T = max(int(torch.randint(64, 449, (1,), generator=g)), cfg.image_position)
        ids = torch.randint(3, cfg.vocab_size, (T + 1,), generator=g)
        ids[cfg.image_position] = -200
        images = [torch.randn(1, 3, r, r, generator=g).bfloat16().to(dev) for r in res]
        reqs.append(dict(ids=ids.to(dev), images=images, new=int(torch.randint(16, 257, (1,), generator=g))))
    return reqs


def timed(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0, torch.cuda.max_memory_allocated()


def make_server(model, args, kv, prefix_cache=False):
    """One server for the warm-up and every timed run: its page pool and its per-bucket CUDA graphs are built once, in
    the warm-up.  `srv.lat` collects the host time of each decode step by bucket (reset after the warm-up), `srv.hits`
    the positions each prefill reused."""
    from cambrian_b200.serving import BatchedGenerator
    srv = BatchedGenerator(model, max_batch=args.max_batch, max_cached_tokens=args.max_cached_tokens, page_size=64,
                           kv_cache_dtype=kv, prefix_cache=prefix_cache)
    srv.lat, srv.hits = {}, []
    prefill = srv._prefill

    def record(r):
        srv.hits.append(r.prefix)
        return prefill(r)

    srv._prefill = record
    inner = srv._decode

    def decode():
        nb = srv._bucket(len(srv._active))
        t0 = time.perf_counter()
        ev = inner()                                   # ends in a host read of the sampled tokens (a synchronise)
        srv.lat.setdefault(nb, []).append((time.perf_counter() - t0) * 1e3)
        return ev

    srv._decode = decode
    return srv


def run_server(srv, reqs):
    rids = [srv.submit(r["ids"], images=r["images"], image_sizes=[(336, 336)], max_new_tokens=r["new"],
                       do_sample=False, eos_token_id=None) for r in reqs]
    outs = srv.run()
    return [outs[i].tolist() for i in rids]


def run_sequential(model, reqs, kv):
    return [model.generate(r["ids"][None], images=r["images"], image_sizes=[(336, 336)], max_new_tokens=r["new"],
                           do_sample=False, eos_token_id=None, kv_cache_dtype=kv)[0].tolist() for r in reqs]


def run_static(model, reqs, args, kv):
    out = []
    for i in range(0, len(reqs), args.max_batch):
        chunk = reqs[i:i + args.max_batch]
        S = max(r["ids"].shape[0] for r in chunk)
        ids = torch.zeros((len(chunk), S), dtype=torch.long, device=chunk[0]["ids"].device)
        mask = torch.zeros_like(ids)
        for b, r in enumerate(chunk):                  # left padding
            n = r["ids"].shape[0]
            ids[b, S - n:] = r["ids"]
            mask[b, S - n:] = 1
        images = [torch.cat([r["images"][t] for r in chunk]) for t in range(len(chunk[0]["images"]))]
        new = max(r["new"] for r in chunk)
        toks = model.generate(ids, images=images, image_sizes=[(336, 336)] * len(chunk), attention_mask=mask,
                              max_new_tokens=new, do_sample=False, eos_token_id=None, kv_cache_dtype=kv)
        out += [toks[b, :r["new"]].tolist() for b, r in enumerate(chunk)]
    return out


def margin_at(model, r, step, kv):
    """The sequential run's top-1 / top-2 logit margin at `step` of request r (an untimed re-run)."""
    seen = []

    def crit(toks, scores):
        if toks.shape[1] == step + 1:
            top = scores[0].topk(2).values
            seen.append(float(top[0] - top[1]))
        return False

    model.generate(r["ids"][None], images=r["images"], image_sizes=[(336, 336)], max_new_tokens=step + 1,
                   do_sample=False, eos_token_id=None, kv_cache_dtype=kv, stopping_criteria=[crit])
    return seen[0] if seen else None


def attn_kernel(srv, reqs, args, iters=50):
    """One layer's paged decode attention at max_batch rows with lengths from the mix (prompt + half of its new tokens),
    CUDA events; bytes = K + V (+ scales) rows read below each length, plus q and o."""
    from cambrian_b200 import ops
    cfg = srv.model.config
    nh, nkv = cfg.num_attention_heads, cfg.num_key_value_heads
    hd = cfg.hidden_size // nh
    pool = srv.pool
    ps = pool.page_size
    rows = min(args.max_batch, len(reqs))
    span = cfg.image_token_len + int(cfg.image_token_len ** 0.5)
    lens = [r["ids"].shape[0] - 1 + span + r["new"] // 2 for r in reqs[:rows]]
    need = [-(-(L + 1) // ps) for L in lens]
    if sum(need) > pool.num_pages:
        return None
    table = torch.zeros((rows, pool.max_pages_per_seq), dtype=torch.int32)
    o = 0
    for b, n in enumerate(need):
        table[b, :n] = torch.arange(o, o + n)
        o += n
    table = table.to(srv.device)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=srv.device)
    q = torch.randn(rows, 1, nh, hd, device=srv.device).bfloat16()
    kp, vp, ks, vs = pool.layer(0)
    f = lambda: ops.attn_decode_paged(q, kp, vp, ks, vs, table, lens_d, pool.ws, len_add=1)  # noqa: E731
    for _ in range(5):
        f()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        f()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / iters
    per_pos = 2 * nkv * (hd * (1 if pool.fp8 else 2) + (4 if pool.fp8 else 0))
    nbytes = sum(L + 1 for L in lens) * per_pos + 2 * rows * nh * hd * 2
    return dict(rows=rows, mean_len=sum(lens) / rows, us=us, bytes=nbytes, gb_s=nbytes / us / 1e3,
                share_of_3_35_tb_s=nbytes / us / 1e6 / 3.35)


# ------------------------------------------------------------------------------------------------ --mix shared
def shared_mix(cfg, seed, dev, images=8, questions=6, convs=8):
    """[dict(ids, images, new, turn, prev)]: questions on shared images (turn 0) and conversation turns 0..2 (`prev`: the
    index of the previous turn, whose prompt and answer the turn's prompt starts with)."""
    g = torch.Generator().manual_seed(seed)
    res = bench.CONFIGS["8b-ddp"]["res"]
    system = torch.randint(3, cfg.vocab_size, (cfg.image_position,), generator=g)
    tok = lambda lo, hi: torch.randint(3, cfg.vocab_size, (int(torch.randint(lo, hi, (1,), generator=g)),),  # noqa: E731
                                       generator=g)
    new = lambda: int(torch.randint(16, 129, (1,), generator=g))  # noqa: E731
    image = lambda: [torch.randn(1, 3, r, r, generator=g).bfloat16().to(dev) for r in res]  # noqa: E731
    out = []
    for _ in range(images):
        img = image()
        for _ in range(questions):
            out.append(dict(ids=torch.cat([system, torch.tensor([-200]), tok(8, 65)]), images=img, new=new(), turn=0,
                            prev=None))
    for _ in range(convs):
        img = image()
        out.append(dict(ids=torch.cat([system, torch.tensor([-200]), tok(8, 65)]), images=img, new=new(), turn=0,
                        prev=None))
        for t in (1, 2):
            out.append(dict(ids=tok(8, 33), images=img, new=new(), turn=t, prev=len(out) - 1))
    return out


def run_shared(srv, mix):
    """The mix in three waves (turn 0, 1, 2); returns (tokens per request, time to first token per request in s)."""
    answers, prompts, ttft = {}, {}, {}
    for turn in range(3):
        wave = [i for i, r in enumerate(mix) if r["turn"] == turn]
        rid = {}
        t0 = time.perf_counter()
        for i in wave:
            r = mix[i]
            p = r["ids"] if r["prev"] is None else torch.cat([prompts[r["prev"]], torch.tensor(answers[r["prev"]]),
                                                               r["ids"]])
            prompts[i] = p
            rid[srv.submit(p.to(srv.device), images=r["images"], image_sizes=[(336, 336)], max_new_tokens=r["new"],
                           do_sample=False, eos_token_id=None)] = i
        while srv.pending():
            for q, _, _ in srv.step():                 # step() ends in a host read of the tokens (a synchronise)
                if rid.get(q) is not None and rid[q] not in ttft:
                    ttft[rid[q]] = time.perf_counter() - t0
        outs = srv.run()
        answers.update({rid[q]: t.tolist() for q, t in outs.items()})
    return [answers[i] for i in range(len(mix))], [ttft[i] for i in range(len(mix))]


def gather_kernel(srv, lengths, iters=50):
    """One layer's cb_paged_kv_gather at the given prefix lengths, CUDA events around `iters` launches replayed from one
    CUDA graph (so the host's per-call checks do not pace the device); bytes = K + V rows (+ scales) read and the bf16
    rows written."""
    from cambrian_b200 import ops
    cfg = srv.model.config
    pool = srv.pool
    nkv = cfg.num_key_value_heads
    hd = cfg.hidden_size // cfg.num_attention_heads
    row = torch.arange(pool.max_pages_per_seq, dtype=torch.int32, device=srv.device) % pool.num_pages
    kp, vp, ks, vs = pool.layer(0)
    out = []
    for P in lengths:
        ok = torch.empty((1, P, nkv, hd), dtype=torch.bfloat16, device=srv.device)
        ov = torch.empty_like(ok)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            ops.paged_kv_gather(kp, vp, ks, vs, row, P, ok, ov)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(iters):
                ops.paged_kv_gather(kp, vp, ks, vs, row, P, ok, ov)
        graph.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / iters
        nbytes = 2 * P * nkv * (hd * (1 if pool.fp8 else 2) + (4 if pool.fp8 else 0) + hd * 2)
        out.append(dict(P=P, us=us, us_all_layers=us * cfg.num_hidden_layers, bytes=nbytes, gb_s=nbytes / us / 1e3,
                        share_of_3_35_tb_s=nbytes / us / 1e6 / 3.35))
    return out


def main_shared(args, dev, card, cfg, model, kv):
    servers = {pc: make_server(model, args, kv, prefix_cache=pc) for pc in (True, False)}
    for pc, srv in servers.items():
        run_shared(srv, shared_mix(cfg, args.seed + 1000, dev))            # warm-up: pool, graphs, allocator
    lines, tokens = [], {}
    for rnd in range(args.rounds):
        mix = shared_mix(cfg, args.seed + rnd, dev)
        n_tokens = sum(r["new"] for r in mix)
        for pc, srv in servers.items():
            srv.hits = []
            reused, prompt = srv.reused_positions, srv.prompt_positions
            (toks, ttft), wall, peak = timed(lambda: run_shared(srv, mix))
            tokens[pc] = toks
            ttft = sorted(ttft)
            line = dict(way="server", mix="shared", prefix_cache=pc, round=rnd, requests=len(mix),
                        generated_tokens=n_tokens, wall_s=wall, tokens_per_s=n_tokens / wall,
                        ttft_mean_ms=1e3 * sum(ttft) / len(ttft), ttft_p90_ms=1e3 * ttft[int(0.9 * (len(ttft) - 1))],
                        hit_rate=(srv.reused_positions - reused) / max(srv.prompt_positions - prompt, 1),
                        cached_pages=srv.cached_pages(), page_pool_bytes=srv.nbytes(), peak_alloc_bytes=peak,
                        kv_cache_dtype=kv, load_fp8=args.load_fp8, max_batch=args.max_batch, card=card)
            lines.append(line)
            print(json.dumps(line), flush=True)
    hits = sorted(h for h in servers[True].hits if h > 0)
    lengths = sorted({hits[0], hits[len(hits) // 2], hits[-1]}) if hits else []
    same = sum(a == b for a, b in zip(tokens[True], tokens[False]))
    summary = dict(metric="serve_shared_summary", card=card, gather_kernel=gather_kernel(servers[True], lengths),
                   hits=len(hits), requests=len(tokens[True]), equal_tokens_with_and_without_cache=same)
    lines.append(summary)
    print(json.dumps(summary), flush=True)
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=64)
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--max-cached-tokens", type=int, default=65536)
    ap.add_argument("--rounds", type=int, default=2, help="alternations of the three ways (server, sequential, static)")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--load-fp8", action="store_true", help="FP8 E4M3 decoder projections (quant_fp8)")
    ap.add_argument("--kv-fp8", action="store_true", help="FP8 pages / FP8 KV cache instead of bf16")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    ap.add_argument("--prefix-cache", action="store_true", help="serve the random mix with prefix_cache=True")
    ap.add_argument("--mix", choices=("random", "shared"), default="random",
                    help="shared: the prefix cache's workload, with and without the cache (module docstring)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("serve_bench.py measures on a GPU; none is visible")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    card = card_info()
    cfg, model = build_model(args, dev)
    kv = "fp8" if args.kv_fp8 else "bf16"
    if args.mix == "shared":
        lines = main_shared(args, dev, card, cfg, model, kv)
        if args.out:
            with open(args.out, "w") as f:
                for ln in lines:
                    f.write(json.dumps(ln) + "\n")
        return
    reqs = request_mix(cfg, args.requests, args.seed, dev)
    n_tokens = sum(r["new"] for r in reqs)
    # warm-up of every path (kernel attributes, allocator); the server's warm-up fills every bucket from max_batch down to
    # 1 as its requests retire, so the timed runs replay graphs captured here and allocate no pages
    srv = make_server(model, args, kv, prefix_cache=args.prefix_cache)
    warm = reqs[:min(len(reqs), args.max_batch)]
    run_server(srv, warm)
    captured = sorted(srv._graphs)
    srv.lat = {}
    run_sequential(model, warm[:1], kv)
    run_static(model, warm, args, kv)
    lines, results = [], {}
    for rnd in range(args.rounds):
        for way in ("server", "sequential", "static"):
            if way == "server":
                n_graphs = len(srv._graphs)
                toks, wall, peak = timed(lambda: run_server(srv, reqs))
            elif way == "sequential":
                toks, wall, peak = timed(lambda: run_sequential(model, reqs, kv))
            else:
                toks, wall, peak = timed(lambda: run_static(model, reqs, args, kv))
            results[way] = toks
            line = dict(way=way, round=rnd, requests=len(reqs), generated_tokens=n_tokens, wall_s=wall,
                        tokens_per_s=n_tokens / wall, peak_alloc_bytes=peak, kv_cache_dtype=kv, load_fp8=args.load_fp8,
                        max_batch=args.max_batch, card=card)
            if way == "server":
                line["prefix_cache"] = args.prefix_cache
                line["page_pool_bytes"] = srv.nbytes()
                line["graphs_captured_in_timed_run"] = len(srv._graphs) - n_graphs
            lines.append(line)
            print(json.dumps(line), flush=True)
    steps = {nb: dict(steps=len(v), mean_ms=sum(v) / len(v), min_ms=min(v)) for nb, v in sorted(srv.lat.items())}
    kern = attn_kernel(srv, reqs, args)
    diffs = []
    for i, r in enumerate(reqs):
        a, b = results["server"][i], results["sequential"][i]
        if a != b:
            k = next((j for j, (x, y) in enumerate(zip(a, b)) if x != y), min(len(a), len(b)))
            diffs.append(dict(request=i, first_diff_step=k, margin=margin_at(model, r, k, kv)))
    static_diffs = sum(results["static"][i] != results["sequential"][i] for i in range(len(reqs)))
    summary = dict(metric="serve_summary", card=card, buckets_captured_in_warm_up=captured,
                   decode_step_ms_per_bucket=steps, paged_attention_kernel=kern,
                   server_equal_to_sequential=len(reqs) - len(diffs), server_diffs=diffs,
                   static_equal_to_sequential=len(reqs) - static_diffs, requests=len(reqs), generated_tokens=n_tokens)
    lines.append(summary)
    print(json.dumps(summary), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
