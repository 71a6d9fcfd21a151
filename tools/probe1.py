"""GPU probe (development tool, not a test): exercises GEMM / SVA / norm kernels against torch references
and prints one line per case.  Run per group under `timeout` so a deadlocked kernel cannot hang the box."""
import sys
import time

import torch

sys.path.insert(0, ".")
from cambrian_b200 import ops  # noqa: E402

dev = "cuda"
torch.manual_seed(0)


def rel_err(a, b):
    a, b = a.float(), b.float()
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()


def timeit(fn, iters=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def gemm_case(M, N, K, a_mn, b_mn, bn, batch=0, **epi):
    bs = (batch,) if batch else ()
    a = torch.randn(*bs, *((K, M) if a_mn else (M, K)), device=dev).bfloat16()
    b = torch.randn(*bs, *((K, N) if b_mn else (N, K)), device=dev).bfloat16()
    A = a.float().transpose(-1, -2) if a_mn else a.float()
    B = b.float() if b_mn else b.float().transpose(-1, -2)
    ref = A @ B
    kw = {}
    if epi.get("bias"):
        kw["bias"] = torch.randn(N, device=dev).bfloat16()
        ref = ref + kw["bias"].float()
    if epi.get("act"):
        kw["act"] = epi["act"]
        f = {"gelu": torch.nn.functional.gelu, "quick_gelu": lambda x: x * torch.sigmoid(1.702 * x),
             "silu": torch.nn.functional.silu,
             "gelu_tanh": lambda x: torch.nn.functional.gelu(x, approximate="tanh")}[epi["act"]]
        ref = f(ref)
    if epi.get("colscale"):
        kw["colscale"] = torch.randn(N, device=dev).bfloat16()
        ref = ref * kw["colscale"].float()
    if epi.get("residual"):
        kw["residual"] = torch.randn(*bs, M, N, device=dev).bfloat16()
        ref = ref + kw["residual"].float()
    out_dtype = torch.float32 if epi.get("fp32") else torch.bfloat16
    if epi.get("accumulate"):
        out = torch.randn(*bs, M, N, device=dev).to(out_dtype)
        ref = ref + out.float()
        got = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, force_bn=bn, out=out, accumulate=True, **kw)
    else:
        got = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, force_bn=bn, out_dtype=out_dtype, **kw)
    torch.cuda.synchronize()
    e = rel_err(got, ref)
    tol = 2e-5 if epi.get("fp32") and not epi.get("accumulate") else 1e-2
    print(f"gemm M={M} N={N} K={K} a_mn={int(a_mn)} b_mn={int(b_mn)} bn={bn} batch={batch} {epi} "
          f"rel_err={e:.3e} {'OK' if e < tol else 'FAIL'}", flush=True)


def group_gemm_basic():
    for a_mn in (False, True):
        for b_mn in (False, True):
            for bn in (64, 128, 256):
                gemm_case(256, 512, 256, a_mn, b_mn, bn, fp32=True)


def group_gemm_shapes():
    for (M, N, K) in [(128, 64, 64), (100, 72, 40), (577, 1024, 1024), (1000, 4304, 1152), (2304, 1024, 2048),
                      (333, 200, 8), (4096, 4096, 4096), (129, 257, 72)]:
        for a_mn, b_mn in ((False, False), (False, True), (True, False), (True, True)):
            if (a_mn and M % 8) or (b_mn and N % 8):
                continue
            gemm_case(M, N, K, a_mn, b_mn, 0, fp32=True)
    gemm_case(512, 768, 512, False, False, 0, batch=5, fp32=True)
    gemm_case(512, 768, 512, True, True, 0, batch=3, fp32=True)
    gemm_case(300, 200, 128, False, True, 0, batch=4)


def group_gemm_epi():
    gemm_case(512, 1024, 512, False, False, 0, bias=True)
    gemm_case(512, 1024, 512, False, False, 0, bias=True, act="gelu")
    gemm_case(512, 1024, 512, False, False, 0, bias=True, act="quick_gelu")
    gemm_case(512, 1024, 512, False, False, 0, act="silu", fp32=True)
    gemm_case(512, 1024, 512, False, False, 0, act="gelu_tanh", fp32=True)
    gemm_case(512, 1024, 512, False, False, 0, bias=True, colscale=True, residual=True)
    gemm_case(500, 1000, 512, False, False, 0, bias=True, residual=True, fp32=True)
    gemm_case(500, 1001 - 1, 512, False, False, 0, accumulate=True, fp32=True)
    gemm_case(512, 1024, 512, True, False, 0, accumulate=True)
    gemm_case(77, 50, 64, False, False, 0, bias=True, residual=True)  # scalar (non-vector) store path


def group_gemm_swiglu():
    """Fused gate/up projection + SwiGLU (cb_gemm_swiglu_bf16) vs GEMM + the stand-alone SwiGLU kernel and fp32 torch."""
    import torch.nn.functional as F_
    for (M, F, K) in [(256, 128, 64), (512, 256, 256), (300, 1024, 192), (1000, 384, 520), (4096, 2048, 1024)]:
        x = torch.randn(M, K, device=dev).bfloat16()
        w = (torch.randn(2 * F, K, device=dev) * 0.05).bfloat16()
        gu, act = ops.gemm_swiglu(x, w)
        ref_gu = (x.float() @ w.float().t())
        e1 = rel_err(gu, ref_gu)
        g16 = gu.float()
        ref_act = F_.silu(g16[:, :F]) * g16[:, F:]
        e2 = rel_err(act, ref_act)
        gu2 = ops.gemm(x, w)
        act2 = ops.swiglu_fwd(gu2[:, :F], gu2[:, F:])
        same = bool(torch.equal(gu, gu2)) and (act.float() - act2.float()).abs().max().item() <= 2 ** -7 * act2.float().abs().max().item()
        ok = e1 < 1e-2 and e2 < 1e-2 and same
        print(f"gemm_swiglu M={M} F={F} K={K} gu={e1:.2e} act={e2:.2e} same_as_unfused={same} {'OK' if ok else 'FAIL'}", flush=True)
    M, F, K = 8192, 14336, 4096
    x = torch.randn(M, K, device=dev).bfloat16()
    w = (torch.randn(2 * F, K, device=dev) * 0.02).bfloat16()
    gu = torch.empty(M, 2 * F, device=dev, dtype=torch.bfloat16)
    act = torch.empty(M, F, device=dev, dtype=torch.bfloat16)
    t_f = timeit(lambda: ops.gemm_swiglu(x, w, gu, act))

    def unfused():
        ops.gemm(x, w, out=gu)
        ops.swiglu_fwd(gu[:, :F], gu[:, F:])
    t_u = timeit(unfused)
    print(f"perf gate/up+swiglu M={M} F={F} K={K}: fused {t_f:.4f} ms ({4 * M * F * K / t_f / 1e9:.0f} TFLOP/s)  "
          f"unfused {t_u:.4f} ms", flush=True)


def group_gemv():
    """Decode-shaped (M <= 8) projections: the weight-streaming GEMV vs an fp32 reference (bias / residual / fp32 output /
    ragged N and K tails), and the achieved weight bandwidth of GEMV and of the 128-row wgmma tile on the same shapes."""
    for (M, N, K, bias, res, f32) in [(1, 4096, 4096, False, True, False), (3, 520, 1032, True, False, False),
                                      (8, 6144, 4096, False, False, False), (5, 1000, 2056, True, True, True),
                                      (8, 128256, 4096, False, False, True), (2, 4096, 14336, False, True, False)]:
        x = torch.randn(M, K, device=dev).bfloat16()
        w = torch.randn(N, K, device=dev).bfloat16() * 0.05
        b = torch.randn(N, device=dev).bfloat16() if bias else None
        r = torch.randn(M, N, device=dev).bfloat16() if res else None
        ref = x.float() @ w.float().t()
        if bias:
            ref = ref + b.float()
        if res:
            ref = ref + r.float()
        got = ops.gemv(x, w, bias=b, residual=r, out_dtype=torch.float32 if f32 else torch.bfloat16)
        e = rel_err(got, ref)
        tol = 2e-5 if f32 else 1e-2
        print(f"gemv M={M} N={N} K={K} bias={int(bias)} res={int(res)} fp32={int(f32)}: err {e:.2e} {'OK' if e < tol else 'FAIL'}", flush=True)
    for (N, K) in ((6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336), (128256, 4096)):
        w = torch.randn(N, K, device=dev).bfloat16() * 0.02
        for M in (1, 8):
            x = torch.randn(M, K, device=dev).bfloat16()
            t_v = timeit(lambda: ops.gemv(x, w), iters=30)
            ops._GEMV = False
            t_t = timeit(lambda: ops.gemm(x, w), iters=30)
            ops._GEMV = True
            print(f"gemv perf M={M} N={N} K={K}: gemv {t_v * 1e3:7.1f} us {N * K * 2 / t_v / 1e6:6.0f} GB/s | wgmma tile "
                  f"{t_t * 1e3:7.1f} us {N * K * 2 / t_t / 1e6:6.0f} GB/s", flush=True)


def group_gemm_perf():
    for (M, N, K) in [(8192, 8192, 8192), (8192, 14336, 4096), (8192, 4096, 14336), (4096, 4096, 4096),
                      (2304, 1024, 1024)]:
        for a_mn, b_mn in ((False, False), (False, True), (True, True)):
            a = torch.randn((K, M) if a_mn else (M, K), device=dev).bfloat16()
            b = torch.randn((K, N) if b_mn else (N, K), device=dev).bfloat16()
            out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            for bn in (128, 256):
                ms = timeit(lambda: ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out=out, force_bn=bn))
                print(f"perf gemm M={M} N={N} K={K} a_mn={int(a_mn)} b_mn={int(b_mn)} bn={bn}: {ms:.4f} ms "
                      f"{2 * M * N * K / ms / 1e9:.1f} TFLOP/s", flush=True)
            if not a_mn and not b_mn:
                ms = timeit(lambda: torch.matmul(a, b.t(), out=out))
                print(f"perf cublas M={M} N={N} K={K}: {ms:.4f} ms {2 * M * N * K / ms / 1e9:.1f} TFLOP/s", flush=True)


def sva_ref(q, ks, vs, masks, rs, batch, q_side):
    """Straight restatement of cambrian_arch.py:271-287 + vision_sampler.py:191-230 in fp32 torch."""
    n = q.shape[0]
    kk, vv, mm = [], [], []
    for k, v, m, r in zip(ks, vs, masks, rs):
        def win(t):
            t = t.view(batch, q_side, r, q_side, r, -1).permute(0, 1, 3, 2, 4, 5).contiguous()
            return t.flatten(0, 2).flatten(1, 2)
        kk.append(win(k.float()))
        vv.append(win(v.float()))
        mm.append(m if m is not None else torch.ones(n, r * r, dtype=torch.bool, device=q.device))
    K = torch.cat(kk, 1).view(n, -1, 16, 64).transpose(1, 2)
    V = torch.cat(vv, 1).view(n, -1, 16, 64).transpose(1, 2)
    Mk = torch.cat(mm, 1)[:, None, None, :]
    Q = q.float().view(n, 1, 16, 64).transpose(1, 2)
    o = torch.nn.functional.scaled_dot_product_attention(Q, K, V, attn_mask=Mk)
    return o.transpose(1, 2).reshape(n, 1024)


def group_sva():
    for batch, q_side, rs, use_mask in [(1, 24, [1, 1, 1, 1], False), (2, 24, [1, 1, 1, 4], True),
                                        (3, 12, [2, 1, 3], True), (1, 24, [1, 1, 1, 4], False)]:
        n = batch * q_side * q_side
        q = torch.randn(n, 1024, device=dev).bfloat16().requires_grad_()
        ks = [torch.randn(batch, (r * q_side) ** 2, 1024, device=dev).bfloat16().requires_grad_() for r in rs]
        vs = [torch.randn(batch, (r * q_side) ** 2, 1024, device=dev).bfloat16().requires_grad_() for r in rs]
        masks = None
        mref = [None] * len(rs)
        if use_mask:
            masks = []
            for r in rs:
                m = torch.rand(n, r * r, device=dev) > 0.3
                m[m.sum(1) == 0] = True
                masks.append(m)
            mref = masks
        out, lse = ops.sva_window_attn_fwd(q.detach(), [k.detach() for k in ks], [v.detach() for v in vs], masks,
                                           rs, batch, q_side)
        ref = sva_ref(q, ks, vs, mref, rs, batch, q_side)
        do = torch.randn_like(ref)
        ref.backward(do)
        dq, dks, dvs = ops.sva_window_attn_bwd(q.detach(), out, do.bfloat16(), lse, [k.detach() for k in ks],
                                               [v.detach() for v in vs], masks, rs, batch, q_side)
        torch.cuda.synchronize()
        errs = [rel_err(out, ref), rel_err(dq, q.grad)] + [rel_err(a, b.grad) for a, b in zip(dks, ks)] + \
               [rel_err(a, b.grad) for a, b in zip(dvs, vs)]
        ok = all(e < 2e-2 for e in errs)
        print(f"sva batch={batch} q_side={q_side} rs={rs} mask={use_mask} errs={[f'{e:.2e}' for e in errs]} "
              f"{'OK' if ok else 'FAIL'}", flush=True)
    # bandwidth, BASELINE grids [576]x4 and release [576,576,576,9216], batch 8
    for rs in ([1, 1, 1, 1], [1, 1, 1, 4]):
        batch, q_side = 8, 24
        n = batch * 576
        q = torch.randn(n, 1024, device=dev).bfloat16()
        ks = [torch.randn(batch, (r * q_side) ** 2, 1024, device=dev).bfloat16() for r in rs]
        vs = [torch.randn(batch, (r * q_side) ** 2, 1024, device=dev).bfloat16() for r in rs]
        ms = timeit(lambda: ops.sva_window_attn_fwd(q, ks, vs, None, rs, batch, q_side))
        byts = (2 * sum(k.numel() for k in ks) + 2 * q.numel()) * 2
        print(f"perf sva fwd rs={rs} batch={batch}: {ms * 1e3:.1f} us, {byts / ms / 1e6:.1f} GB/s", flush=True)
        out, lse = ops.sva_window_attn_fwd(q, ks, vs, None, rs, batch, q_side)
        ms = timeit(lambda: ops.sva_window_attn_bwd(q, out, out, lse, ks, vs, None, rs, batch, q_side))
        print(f"perf sva bwd rs={rs} batch={batch}: {ms * 1e3:.1f} us, {(2 * byts + 2 * q.numel() * 2) / ms / 1e6:.1f} GB/s",
              flush=True)


def group_norm():
    F = torch.nn.functional
    for rows, C in [(577, 1024), (1000, 1152), (300, 384), (64, 3072), (2048, 4096), (100, 5120), (50, 7168),
                    (10, 16384), (33, 1536)]:
        x = torch.randn(rows, C, device=dev).bfloat16()
        g = (1 + 0.1 * torch.randn(C, device=dev)).bfloat16()
        b = (0.1 * torch.randn(C, device=dev)).bfloat16()
        dy = torch.randn(rows, C, device=dev).bfloat16()
        xf = x.float().requires_grad_()
        gf, bf = g.float().requires_grad_(), b.float().requires_grad_()
        ref = F.layer_norm(xf, (C,), gf, bf, 1e-5)
        ref.backward(dy.float())
        y, mean, rstd = ops.layernorm_fwd(x, g, b, 1e-5, save_stats=True)
        dx, dg, db = ops.layernorm_bwd(dy, x, g, mean, rstd)
        torch.cuda.synchronize()
        errs = [rel_err(y, ref), rel_err(dx, xf.grad), rel_err(dg, gf.grad), rel_err(db, bf.grad)]
        print(f"layernorm rows={rows} C={C} errs={[f'{e:.2e}' for e in errs]} "
              f"{'OK' if all(e < 1.5e-2 for e in errs) else 'FAIL'}", flush=True)
        xf = x.float().requires_grad_()
        gf = g.float().requires_grad_()
        ref = gf * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6))
        ref.backward(dy.float())
        y, rstd = ops.rmsnorm_fwd(x, g, 1e-6, save_stats=True)
        dx, dg = ops.rmsnorm_bwd(dy, x, g, rstd)
        torch.cuda.synchronize()
        errs = [rel_err(y, ref), rel_err(dx, xf.grad), rel_err(dg, gf.grad)]
        print(f"rmsnorm rows={rows} C={C} errs={[f'{e:.2e}' for e in errs]} "
              f"{'OK' if all(e < 1.5e-2 for e in errs) else 'FAIL'}", flush=True)
    # pos-embed fused LN: grid side 8, r=4 (q_side 2), batch 3
    side, r, C, B = 8, 4, 1024, 3
    x = torch.randn(B * side * side, C, device=dev).bfloat16()
    pos = torch.randn(r * r, C, device=dev).bfloat16()
    g = torch.randn(C, device=dev).bfloat16()
    b = torch.randn(C, device=dev).bfloat16()
    idx = torch.arange(side * side, device=dev)
    pidx = ((idx // side) % r) * r + (idx % side) % r
    xin = (x.view(B, side * side, C) + pos[pidx][None]).float()
    ref = F.layer_norm(xin, (C,), g.float(), b.float(), 1e-5).view(-1, C)
    y = ops.layernorm_fwd(x, g, b, 1e-5, pos=pos, side=side, r=r)
    print(f"layernorm+pos err={rel_err(y, ref):.2e} {'OK' if rel_err(y, ref) < 1.5e-2 else 'FAIL'}", flush=True)
    x = torch.randn(8 * 2048, 4096, device=dev).bfloat16()
    g = torch.randn(4096, device=dev).bfloat16()
    ms = timeit(lambda: ops.rmsnorm_fwd(x, g))
    print(f"perf rmsnorm fwd 16384x4096: {ms * 1e3:.1f} us {2 * x.numel() * 2 / ms / 1e6:.1f} GB/s", flush=True)
    y, rstd = ops.rmsnorm_fwd(x, g, save_stats=True)
    ms = timeit(lambda: ops.rmsnorm_bwd(x, x, g, rstd))
    print(f"perf rmsnorm bwd 16384x4096: {ms * 1e3:.1f} us {3 * x.numel() * 2 / ms / 1e6:.1f} GB/s", flush=True)


if __name__ == "__main__":
    t0 = time.time()
    globals()["group_" + sys.argv[1]]()
    print(f"group {sys.argv[1]} done in {time.time() - t0:.1f}s", flush=True)
