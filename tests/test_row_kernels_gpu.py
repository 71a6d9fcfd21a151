"""The row kernels of a training step against float64 references, and the CPU stand-ins of tests/ops_emulation.py against
the same references.

Every case runs three arms on the same seeded inputs: the `cambrian_b200.ops` kernel, a float64 reference written from the
op's definition (tests/row_kernels_reference.py, which also derives each error bound), and the ops_emulation stand-in on
CPU copies.  The kernel is held to the fp64 bound; the stand-in is held to the same bound, or to the kernel's bits where
both specify the same rounding steps; memory the op must not write is compared bitwise with a sentinel.  Shapes are
chosen to reach every template instance, loop and branch the model reaches: every threads-per-row width of the norms,
more rows than one pass of the backward's grid, vocabularies below and above the block's reach, labels in the last
vector, AdamW and sumsq beyond one grid-stride pass.  Each check prints its worst error-to-bound ratio.
"""
from __future__ import annotations

import math

import pytest
import torch

import ops_emulation as emu
from row_kernels_reference import (HALF_ULP, U, assert_bitwise, assert_either, check_abs, check_bf16, norm_bwd_cfg,
                                   norm_bwd_ref, norm_bwd_tols, norm_fwd_cfg, norm_fwd_ref, norm_fwd_tols, norm_input,
                                   rope_fp32_ref, rope_fp64_ref, rope_tables, round_either, sentinel_like, sm_count)

pytestmark = pytest.mark.gpu

DEV = "cuda"


@pytest.fixture(scope="module")
def ops():
    from cambrian_b200 import ops as o
    return o


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(shape, seed, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(shape, generator=_gen(seed), device=DEV) * scale).to(dtype)


def _cpu(*ts):
    return [None if t is None else t.detach().cpu() for t in ts]


# ======================================================================================================= norms (norm.cu)
FWD_WIDTHS = [384, 1024, 1152, 1160, 1536, 3072, 4096, 5120, 7168, 8192, 16384]


def _row_counts(C):
    """1; a count that is not a multiple of the rows per block; and more than 2 x SMs x rows-per-block of the backward, so
    its grid-stride row loop runs three times and the last pass is partial."""
    _, _, rpb = norm_bwd_cfg(C)
    return [1, 8 * 5 + 3, 2 * (2 * sm_count() * rpb) + 3 * rpb + 1]


def _norm_case(ops, C, rows, *, rms, hf_cast=False, pos_mode=None, with_dres=False, seed=0):
    r = 3
    pos = side = None
    sd = 0
    if pos_mode is not None:
        pos = _randn((r * r, C), seed + 7, 0.5)
        if pos_mode == "grid":
            side = 4 * r
            sd = side
            rows = -(-rows // (side * side)) * side * side
        else:
            sd = 0
            rows = -(-rows // (r * r)) * r * r
    x = _randn((rows, C), seed + 1, 1.0) + (0.25 if not rms else 0.0)
    x = x.to(torch.bfloat16)
    gamma = (1 + _randn((C,), seed + 2, 0.25, torch.float32)).to(torch.bfloat16)
    beta = None if rms else _randn((C,), seed + 3, 0.1)
    dy = _randn((rows, C), seed + 4, 1.0)
    dres = _randn((rows, C), seed + 5, 0.5) if with_dres else None
    eps = 1e-6 if rms else 1e-5
    tag = f"C={C} rows={rows}"
    print(f"\n  {'rmsnorm' if rms else 'layernorm'} {tag} hf_cast={hf_cast} pos={pos_mode} dres={with_dres} "
          f"fwd TPR={norm_fwd_cfg(C)[0]} bwd (TPR, VPT)={norm_bwd_cfg(C)[:2]}")

    # ---- kernel
    if rms:
        y, rstd = ops.rmsnorm_fwd(x, gamma, eps, hf_cast=hf_cast, save_stats=True)
        mean = None
        dx, dg = ops.rmsnorm_bwd(dy, x, gamma, rstd, dres=dres)
        db = None
    else:
        y, mean, rstd = ops.layernorm_fwd(x, gamma, beta, eps, pos=pos, side=sd, r=r if pos is not None else 0,
                                          save_stats=True)
        dx, dg, db = ops.layernorm_bwd(dy, x, gamma, mean, rstd, pos=pos, side=sd, r=r if pos is not None else 0,
                                       dres=dres)
    torch.cuda.synchronize()

    # ---- fp64 reference
    xp = norm_input(x, pos, sd, r)
    ref = norm_fwd_ref(xp, gamma, beta, eps, rms)
    tf = norm_fwd_tols(ref, xp, gamma, beta, rms)
    bref = norm_bwd_ref(xp, dy, gamma, dres, ref, rms)
    tb = norm_bwd_tols(xp, ref, bref, dres, rms, rows, C, sm_count())

    def fwd_checks(arm, y_, mean_, rstd_):
        check_abs(f"{arm} rstd", rstd_, ref["rstd"], tf["rstd"])
        if not rms:
            check_abs(f"{arm} mean", mean_, ref["mean"], tf["mean"] + U * ref["mean"].abs())
        if rms and hf_cast:
            # x_hat is rounded to bf16 before gamma multiplies it (HF order): the product of two bf16 values is exact in fp32,
            # so y is the rounding of gamma * (either bf16 neighbour of the fp32 x_hat)
            lo, hi = round_either(ref["xh"], tf["rstd"][:, None] / ref["rstd"][:, None] + 2 * U)
            g = gamma.float()
            assert_either(f"{arm} y (hf_cast)", y_.reshape(rows, C).to(DEV), (g * lo.float()).to(torch.bfloat16),
                          (g * hi.float()).to(torch.bfloat16))
        else:
            check_bf16(f"{arm} y", y_.reshape(rows, C), ref["y"], tf["y"])

    def bwd_checks(arm, dx_, dg_, db_):
        check_bf16(f"{arm} dx", dx_.reshape(rows, C), bref["dx"], tb["dx"])
        check_bf16(f"{arm} dgamma", dg_, bref["dgamma"], tb["dgamma"])
        if not rms:
            check_bf16(f"{arm} dbeta", db_, bref["dbeta"], tb["dbeta"])

    fwd_checks("kernel", y, mean, rstd)
    bwd_checks("kernel", dx, dg, db)

    # ---- stand-in (CPU), fed the kernel's saved statistics in the backward as the product does
    xc, gc, bc, dyc, dresc, posc, meanc, rstdc = _cpu(x, gamma, beta, dy, dres, pos, mean, rstd)
    if rms:
        ye, re_ = emu.rmsnorm_fwd(xc, gc, eps, hf_cast=hf_cast, save_stats=True)
        me = None
        dxe, dge = emu.rmsnorm_bwd(dyc, xc, gc, rstdc, dres=dresc)
        dbe = None
    else:
        ye, me, re_ = emu.layernorm_fwd(xc, gc, bc, eps, pos=posc, side=sd, r=r if pos is not None else 0, save_stats=True)
        dxe, dge, dbe = emu.layernorm_bwd(dyc, xc, gc, meanc, rstdc, pos=posc, side=sd, r=r if pos is not None else 0,
                                          dres=dresc)
    fwd_checks("stand-in", ye, me, re_)
    bwd_checks("stand-in", dxe, dge, dbe)


@pytest.mark.parametrize("C", FWD_WIDTHS)
def test_layernorm_every_width(ops, C):
    for rows in _row_counts(C):
        _norm_case(ops, C, rows, rms=False, seed=C + rows)


@pytest.mark.parametrize("C", FWD_WIDTHS)
def test_rmsnorm_every_width(ops, C):
    for rows in _row_counts(C):
        _norm_case(ops, C, rows, rms=True, seed=C + rows)


@pytest.mark.parametrize("C", [1024, 1160, 4096])
@pytest.mark.parametrize("variant", ["pos_grid", "pos_windowed", "dres", "pos_dres"])
def test_layernorm_pos_and_dres(ops, C, variant):
    pos_mode = {"pos_grid": "grid", "pos_windowed": "windowed", "dres": None, "pos_dres": "grid"}[variant]
    rows = _row_counts(C)[-1]
    _norm_case(ops, C, rows, rms=False, pos_mode=pos_mode, with_dres=variant in ("dres", "pos_dres"), seed=11)
    _norm_case(ops, C, 43, rms=False, pos_mode=pos_mode, with_dres=variant in ("dres", "pos_dres"), seed=12)


@pytest.mark.parametrize("C", [1160, 3072, 4096, 16384])
@pytest.mark.parametrize("hf_cast", [False, True])
@pytest.mark.parametrize("with_dres", [False, True])
def test_rmsnorm_hf_cast_and_dres(ops, C, hf_cast, with_dres):
    _norm_case(ops, C, _row_counts(C)[-1], rms=True, hf_cast=hf_cast, with_dres=with_dres, seed=21)
    _norm_case(ops, C, 43, rms=True, hf_cast=hf_cast, with_dres=with_dres, seed=22)


# ================================================================================================================== RoPE
@pytest.mark.parametrize("hd", [64, 96, 128])
@pytest.mark.parametrize("nh,nkv", [(32, 32), (32, 8)])
def test_rope_forward_inverse_and_adjoint(ops, hd, nh, nkv):
    max_pos = 4096
    cos_t, sin_t = (t.to(DEV) for t in rope_tables(max_pos, hd))
    rows = 300
    width = (nh + 2 * nkv) * hd
    pos = torch.randint(0, max_pos, (rows,), generator=_gen(hd + nh + nkv), device=DEV)
    pos[:6] = torch.tensor([0, max_pos - 1, 1, max_pos - 2, -3, max_pos + 5], device=DEV)   # ends, and the clamp
    buf0 = _randn((rows, width), 31 + hd, 2.0)
    nq = nh + nkv
    for inverse in (False, True):
        buf = buf0.clone()
        ops.rope_(buf, pos, cos_t, sin_t, nq, hd, inverse=inverse)
        torch.cuda.synchronize()
        print(f"\n  rope hd={hd} nh={nh} nkv={nkv} inverse={inverse}")
        want = rope_fp32_ref(buf0, pos, cos_t, sin_t, nq, hd, inverse)
        assert_bitwise("kernel vs fp32 rounding-order reference", buf, want)
        assert_bitwise("V columns untouched", buf[:, nq * hd:], buf0[:, nq * hd:])
        o64, tol = rope_fp64_ref(buf0, pos, cos_t, sin_t, nq, hd, inverse)
        check_bf16("kernel vs unrounded fp64 rotation", buf[:, : nq * hd], o64, tol)
        e = emu.rope_(buf0.cpu().clone(), pos.cpu(), cos_t.cpu(), sin_t.cpu(), nq, hd, inverse=inverse)
        assert_bitwise("stand-in vs kernel", e, buf)
    # <rope(x), y> = <x, rope^-1(y)> per head, within the bounds of the two rotations
    y0 = _randn((rows, width), 41 + hd, 1.0)
    rx, ry = buf0.clone(), y0.clone()
    ops.rope_(rx, pos, cos_t, sin_t, nq, hd)
    ops.rope_(ry, pos, cos_t, sin_t, nq, hd, inverse=True)
    _, tx = rope_fp64_ref(buf0, pos, cos_t, sin_t, nq, hd, False)
    _, ty = rope_fp64_ref(y0, pos, cos_t, sin_t, nq, hd, True)
    n = nq * hd
    sh = (rows, nq, hd)
    lhs = (rx[:, :n].double() * y0[:, :n].double()).reshape(sh).sum(-1)
    rhs = (buf0[:, :n].double() * ry[:, :n].double()).reshape(sh).sum(-1)
    ax, ay = rx[:, :n].double().abs(), ry[:, :n].double().abs()
    bound = ((HALF_ULP * ax + tx) * y0[:, :n].double().abs() + buf0[:, :n].double().abs() * (HALF_ULP * ay + ty)).reshape(sh).sum(-1)
    check_abs("adjoint <rope(x), y> - <x, rope^-1(y)>", lhs - rhs, torch.zeros_like(lhs), bound)


# ============================================================================================ cross-entropy, loss_reduce
def _ce_case(V, seed):
    rows = 12
    g = _gen(seed)
    logits = torch.randn((rows, V), generator=g, device=DEV) * 3
    logits[3] = torch.where(torch.rand(V, generator=g, device=DEV) < 0.5, -80.0, 80.0)      # the online max restarts
    logits[4] = -80.0 + torch.rand(V, generator=g, device=DEV) * 160.0
    logits[5, V - 1] = 60.0                                                                # max in the last vector
    labels = torch.randint(0, V, (rows,), generator=g, device=DEV)
    labels[0] = -100        # ignore_index
    labels[1] = -7          # negative
    labels[2] = V           # >= V
    labels[6] = V + 123
    labels[3] = 0
    labels[5] = V - 1       # last 8-wide vector
    labels[7] = V - 8
    labels[8] = 1
    return logits.to(torch.bfloat16), labels


def _ce_ref(logits, labels, V, gs):
    lf = logits.double()
    valid = (labels != -100) & (labels >= 0) & (labels < V)
    lab = labels.clamp(0, V - 1)
    lse = torch.logsumexp(lf, -1)
    m = lf.amax(-1)
    loss = torch.where(valid, lse - lf.gather(1, lab[:, None])[:, 0], torch.zeros_like(lse))
    p = torch.softmax(lf, -1)
    onehot = torch.zeros_like(p)
    onehot[torch.arange(len(labels), device=lf.device), lab] = 1.0
    grad = torch.where(valid[:, None], (p - onehot) * gs, torch.zeros_like(p))
    # fp32 arithmetic of cross_entropy_kernel: each of the ceil(V / 8 / 1024) loop steps adds 8 terms and rescales
    # (a chain of 8 + 2 per step), a 5-level warp tree, 32 warp partials in order: h.  __expf has <= 2 + 1.16|a| ulp at
    # argument a; terms with a < -20 weigh < 2e-9 each, so each exponential (the terms and the <= steps + 3 rescales) is
    # good to 26 u.  logf adds 1 ulp of log(s), the two subtractions 1 ulp of |lse| and |loss|.
    steps = -(-(V // 8) // 1024)
    h = (8 + 2) * steps + 5 + 32
    e_s = (h + 26 * (steps + 3)) * U
    t_loss = torch.where(valid, e_s + U * (math.log(V) + 2 * lse.abs() + m.abs() + loss.abs()), torch.zeros_like(lse))
    # 2^-126: probabilities below FLT_MIN underflow to 0 in __expf
    t_grad = abs(gs) * (p * (e_s + 30 * U) + U * onehot + 2.0 ** -126) * (1 + HALF_ULP)
    return dict(loss=loss, grad=grad, valid=valid, t_loss=t_loss, t_grad=torch.where(valid[:, None], t_grad, 0 * t_grad))


@pytest.mark.parametrize("V", [1024, 32000, 32064, 64000, 128256])
@pytest.mark.parametrize("mode", ["loss_only", "grad", "grad_scale_dev"])
def test_cross_entropy_and_loss_reduce(ops, V, mode):
    logits, labels = _ce_case(V, V)
    rows = logits.shape[0]
    # logits live in rows [2, 2 + rows) and columns [0, V) of a wider buffer, as one chunk of the chunked loss loop
    big = sentinel_like((rows + 4, V + 16), torch.bfloat16, DEV)
    big[2:2 + rows, :V] = logits
    view = big[2:2 + rows, :V]
    big0 = big.clone()
    loss_rows = sentinel_like((rows,), torch.float32, DEV)
    acc = torch.tensor([1.5, 3.0], device=DEV)      # accumulated over earlier chunks
    write = mode != "loss_only"
    gs_host, scale_dev = (0.25, None) if mode != "grad_scale_dev" else (0.5, torch.tensor([0.125], device=DEV))
    gs = float(torch.tensor(gs_host * (0.125 if scale_dev is not None else 1.0), dtype=torch.float32))
    half = 7      # two calls, as two chunks: loss_acc accumulates over both
    for a, b in ((0, half), (half, rows)):
        ops.cross_entropy(view[a:b], labels[a:b], loss_rows[a:b], acc, gs_host, write, scale_dev=scale_dev)
    torch.cuda.synchronize()
    R = _ce_ref(logits, labels, V, gs)
    print(f"\n  cross_entropy V={V} mode={mode}")
    check_abs("kernel loss rows", loss_rows, R["loss"], R["t_loss"])
    ign = ~R["valid"]
    assert bool((loss_rows[ign] == 0).all()), "ignored rows must have loss 0"
    n_valid = int(R["valid"].sum())
    assert float(acc[1]) == 3.0 + n_valid, f"count {float(acc[1])} != {3.0 + n_valid}"
    # loss_reduce: per call, ceil(rows / 1024) + 5 + 32 ordered additions, then += into acc[0]
    t_sum = (1 + 5 + 32 + 2) * U * (R["loss"].abs().sum() + 1.5) + R["t_loss"].sum()
    check_abs("kernel loss_acc sum", acc[0:1], (R["loss"].sum() + 1.5)[None], t_sum[None])
    assert_bitwise("rows and columns outside the chunk untouched", torch.cat([big[:2].reshape(-1), big[2 + rows:].reshape(-1),
                                                                             big[:, V:].reshape(-1)]),
                   torch.cat([big0[:2].reshape(-1), big0[2 + rows:].reshape(-1), big0[:, V:].reshape(-1)]))
    if write:
        check_bf16("kernel gradient", view, R["grad"], R["t_grad"])
        assert bool((view[ign] == 0).all()), "ignored rows' gradient must be 0"
    else:
        assert_bitwise("logits untouched without write_grad", view, logits)
    # stand-in
    lc = logits.cpu().clone()
    lr_e = torch.empty(rows)
    acc_e = torch.tensor([1.5, 3.0])
    for a, b in ((0, half), (half, rows)):
        emu.cross_entropy(lc[a:b], labels.cpu()[a:b], lr_e[a:b], acc_e, gs_host, write,
                          scale_dev=None if scale_dev is None else scale_dev.cpu())
    check_abs("stand-in loss rows", lr_e, R["loss"], R["t_loss"])
    assert float(acc_e[1]) == 3.0 + n_valid, "stand-in count"
    check_abs("stand-in loss_acc sum", acc_e[0:1], (R["loss"].sum() + 1.5)[None], t_sum[None])
    if write:
        check_bf16("stand-in gradient", lc, R["grad"], R["t_grad"])
    else:
        assert_bitwise("stand-in leaves logits without write_grad", lc, logits)


# ================================================================================================ AdamW, sumsq, clip_coef
def _adamw_ref(p, m, v, g16, lr, b1, b2, eps, wd, step, gs):
    """torch.optim.AdamW (decoupled decay) in float64 at the fp32 values of the hyper-parameters, and its allowance.
    Bias corrections: the host computes b^step with powf (< 1 ulp) and 1 - b^step in fp32: relative error
    (2 u b^step + u bc) / bc, large where bc is small.  m, v: two products and a sum (4-5 u of their terms).  p: the decay
    (3 u |p|), the update's m, sqrt(v) (half of v's), rsqrtf(bc2) (2 ulp), bc1, the divide and the eps add (8 u)."""
    f = lambda x: float(torch.tensor(x, dtype=torch.float32))
    lr, b1, b2, eps, wd, gs = map(f, (lr, b1, b2, eps, wd, gs))
    p, m, v = p.double(), m.double(), v.double()
    g = g16.double() * gs
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    r1 = (2 * U * b1 ** step + U * bc1) / bc1
    r2 = (2 * U * b2 ** step + U * bc2) / bc2
    m2 = b1 * m + (1 - b1) * g
    v2 = b2 * v + (1 - b2) * g * g
    t_m = 5 * U * (b1 * m.abs() + (1 - b1) * g.abs())
    t_v = 6 * U * (b2 * v + (1 - b2) * g * g)
    denom = v2.sqrt() / math.sqrt(bc2) + eps
    upd = (lr / bc1) * m2 / denom
    p2 = p * (1 - lr * wd) - upd
    t_p = (3 * U * p.abs() + (lr / bc1) * t_m / denom
           + upd.abs() * (r1 + 0.5 * r2 + 0.5 * t_v / v2.clamp_min(1e-300) + 8 * U) + U * p2.abs())
    return dict(p=p2, m=m2, v=v2, t_p=t_p, t_m=t_m, t_v=t_v)


@pytest.mark.parametrize("background", [False, True])
@pytest.mark.parametrize("scale", ["grad_scale", "device_coef"])
@pytest.mark.parametrize("wd", [0.0, 0.1])
def test_adamw_steps(ops, background, scale, wd):
    sms = sm_count()
    per_pass = sms * (1 if background else 8) * (128 if background else 256) * 8     # elements per grid-stride pass
    n = 2 * per_pass + 8 * 37
    lr, b1, b2, eps = 1e-3, 0.9, 0.999, 1e-8
    p = torch.randn(n, generator=_gen(1), device=DEV)
    m = torch.zeros(n, device=DEV)
    v = torch.zeros(n, device=DEV)
    coef = torch.tensor([0.37, 1.0], device=DEV) if scale == "device_coef" else None
    gs_used = 0.37 if coef is not None else 0.5
    gs_arg = 123.0 if coef is not None else 0.5       # the device coefficient replaces grad_scale
    for step in (1, 2, 3, 1000):
        if step == 1000:
            m = torch.randn(n, generator=_gen(5), device=DEV) * 1e-3
            v = torch.rand(n, generator=_gen(6), device=DEV) * 1e-6
        g16 = _randn((n,), 10 + step, 0.01)
        g16[:8] = 0
        pre = [t.clone() for t in (p, m, v)]
        p16 = sentinel_like((n,), torch.bfloat16, DEV)
        ops.adamw(p, m, v, g16, p16, lr, b1, b2, eps, wd, step, grad_scale=gs_arg, clip_coef=coef, background=background)
        torch.cuda.synchronize()
        R = _adamw_ref(*pre, g16, lr, b1, b2, eps, wd, step, gs_used)
        print(f"\n  adamw n={n} background={background} {scale} wd={wd} step={step}")
        check_abs("kernel p32", p, R["p"], R["t_p"])
        check_abs("kernel m", m, R["m"], R["t_m"])
        check_abs("kernel v", v, R["v"], R["t_v"])
        assert_bitwise("p16 == p32.to(bf16)", p16, p.to(torch.bfloat16))
        pe, me, ve = _cpu(*pre)
        p16e = torch.empty(n, dtype=torch.bfloat16)
        emu.adamw(pe, me, ve, g16.cpu(), p16e, lr, b1, b2, eps, wd, step, grad_scale=gs_arg,
                  clip_coef=None if coef is None else coef.cpu(), background=background)
        check_abs("stand-in p32", pe, R["p"], R["t_p"])
        check_abs("stand-in m", me, R["m"], R["t_m"])
        check_abs("stand-in v", ve, R["v"], R["t_v"])
        assert_bitwise("stand-in p16 == p32.to(bf16)", p16e, pe.to(torch.bfloat16))


@pytest.mark.parametrize("background", [False, True])
def test_sumsq_and_clip_coef(ops, background):
    sms = sm_count()
    threads, per_sm = (128, 1) if background else (256, 8)
    sizes = [8, 8 * 1000 + 8, 2 * sms * per_sm * threads * 8 + 8 * 13, 40 * threads * 8]
    gs = [_randn((n,), 50 + i, 0.02 * (i + 1)) for i, n in enumerate(sizes)]
    ws = torch.empty(8192, device=DEV)
    acc = torch.zeros(1, device=DEV)
    for g in gs:
        ops.sumsq_accumulate(g, acc, ws, background=background)
    torch.cuda.synchronize()
    ref = sum(float((g.double() ** 2).sum()) for g in gs)
    tol = 0.0
    for n, g in zip(sizes, gs):
        nb = min(max(-(-(n // 8) // threads), 1), sms * per_sm)
        iters = -(-(n // 8) // (nb * threads))
        h = 8 * iters + 5 + threads // 32 + -(-nb // 32) + 5 + 1      # fmaf chain, warp, block, final warp, +=
        tol += h * U * float((g.double() ** 2).sum())
    print(f"\n  sumsq background={background} partial blocks={[min(max(-(-(n // 8) // threads), 1), sms * per_sm) for n in sizes]}")
    check_abs("kernel sumsq", acc, torch.tensor([ref], dtype=torch.float64, device=DEV), tol)
    acc_e = torch.zeros(1)
    for g in gs:
        emu.sumsq_accumulate(g.cpu(), acc_e, None)
    check_abs("stand-in sumsq", acc_e, torch.tensor([ref], dtype=torch.float64), tol)
    for max_norm in (0.01, 100.0):
        for inv_world in (1.0, 0.5):
            s = torch.tensor([float(acc[0])], device=DEV)
            coef = sentinel_like((2,), torch.float32, DEV)
            ops.clip_coef(s, max_norm, inv_world, coef)
            torch.cuda.synchronize()
            s64 = float(acc[0])
            norm = math.sqrt(s64) * inv_world
            want = torch.tensor([inv_world * min(1.0, max_norm / (norm + 1e-6)), norm], dtype=torch.float64)
            # sqrtf, the product, the add, the division, fminf's operand and the product: <= 5 u relative
            print(f"  clip_coef max_norm={max_norm} inv_world={inv_world}")
            check_abs("kernel coef", coef, want.to(DEV), 5 * U * want.abs().to(DEV))
            assert float(s[0]) == 0.0, "clip_coef must reset sumsq"
            se, ce = torch.tensor([s64]), torch.zeros(2)
            emu.clip_coef(se, max_norm, inv_world, ce)
            check_abs("stand-in coef", ce, want, 5 * U * want.abs())
            assert float(se[0]) == 0.0


# ======================================================================================================= SwiGLU, acts
@pytest.mark.parametrize("I", [8192, 14336, 1000])
def test_swiglu_fused_buffer(ops, I):
    rows = 37
    gu = _randn((rows, 2 * I), 60 + I, 3.0)
    gu[0, :64] = torch.linspace(-30, 30, 64, device=DEV).to(torch.bfloat16)     # saturated silu
    gate, up = gu[:, :I], gu[:, I:]
    out = ops.swiglu_fwd(gate, up)
    dout = _randn((rows, I), 61 + I, 1.0)
    dgu = sentinel_like((rows, 2 * I + 64), torch.bfloat16, DEV)
    ops.swiglu_bwd(dout, gate, up, dgu[:, :I], dgu[:, I:2 * I])
    torch.cuda.synchronize()
    print(f"\n  swiglu I={I} rows={rows}")
    g64, u64 = gate.double(), up.double()
    # silu in fp32 on the MUFU (ex2 / rcp approx: 8 u, and the argument's rounding: |x| u) is rounded to bf16, then
    # multiplied by up (exact in fp32) and rounded: out is the rounding of either bf16 neighbour of silu times up
    lo, hi = round_either(g64 * torch.sigmoid(g64), (8 + g64.abs()) * U)
    want_lo, want_hi = (lo.float() * up.float()).to(torch.bfloat16), (hi.float() * up.float()).to(torch.bfloat16)
    assert_either("kernel out", out, want_lo, want_hi)
    assert_either("stand-in out", emu.swiglu_fwd(*_cpu(gate, up)).to(DEV), want_lo, want_hi)
    # backward: sigmoid with __expf (2 + 1.16|g| ulp) + the add and the IEEE division -> e_s relative; 1 - s absolute
    # s e_s + u; the products add 3 u
    s = torch.sigmoid(g64)
    d = dout.double()
    e_s = (4 + 1.16 * g64.abs()) * U
    du = d * g64 * s
    dg = d * u64 * s * (1 + g64 * (1 - s))
    t_du = du.abs() * (e_s + 3 * U) * (1 + HALF_ULP)
    t_dg = ((d * u64 * s).abs() * ((e_s + 3 * U) * (1 + g64 * (1 - s)).abs() + g64.abs() * (s * e_s + U)
            + 2 * U * (1 + (g64 * (1 - s)).abs()))) * (1 + HALF_ULP)
    check_bf16("kernel dgate (strided)", dgu[:, :I], dg, t_dg)
    check_bf16("kernel dup (strided)", dgu[:, I:2 * I], du, t_du)
    assert_bitwise("columns past the two halves untouched", dgu[:, 2 * I:], sentinel_like((rows, 64), torch.bfloat16, DEV))
    dge, due = torch.empty(rows, I, dtype=torch.bfloat16), torch.empty(rows, I, dtype=torch.bfloat16)
    emu.swiglu_bwd(*_cpu(dout, gate, up), dge, due)
    check_bf16("stand-in dgate", dge, dg.cpu(), t_dg.cpu())
    check_bf16("stand-in dup", due, du.cpu(), t_du.cpu())


_ACT64 = {
    "gelu": lambda x: 0.5 * x * (1 + torch.erf(x / math.sqrt(2))),
    "gelu_tanh": lambda x: 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3))),
    "quick_gelu": lambda x: x * torch.sigmoid(1.702 * x),
    "silu": lambda x: x * torch.sigmoid(x),
}


@pytest.mark.parametrize("act", list(_ACT64))
def test_activations(ops, act):
    sms = sm_count()
    n = 2 * sms * 8 * 256 * 8 + 8 * 37           # two grid-stride passes of act_fwd / act_bwd and a partial third
    x = _randn((n,), 70, 3.0)
    sat = torch.linspace(10, 80, 4096, device=DEV)
    x[:4096] = sat.to(torch.bfloat16)
    x[4096:8192] = (-sat).to(torch.bfloat16)
    dy = _randn((n,), 71, 1.0)
    y = ops.act_fwd(x, act)
    dx = ops.act_bwd(dy, x, act)
    torch.cuda.synchronize()
    x64 = x.double().requires_grad_()
    with torch.enable_grad():
        y64 = _ACT64[act](x64)
    (d64,) = torch.autograd.grad(y64, x64, dy.double())
    y64, x64 = y64.detach(), x64.detach()
    ax = x64.abs()
    # fp32 on the MUFU (ex2 / rcp approx, A&S erf with 1.5e-7 absolute error): <= 16 u of |x|, and the rounding of the
    # exponent's argument: 2 u |x| of |x|.  2^-126: the approximate units flush results below FLT_MIN.
    t_y = (16 + 2 * ax) * U * ax + 2.0 ** -126
    # derivative: the same units and the cancellation in 1 - s (sigmoid forms) or 1 - tanh^2 (gelu_tanh, whose inner
    # derivative 0.8 (1 + 0.134 x^2) multiplies it until tanh saturates at |x| ~ 5)
    chain = 1 + 0.134 * ax.clamp(max=5) ** 2 if act == "gelu_tanh" else 1.0
    t_d = dy.double().abs() * (32 + 4 * ax) * U * chain + 2.0 ** -126
    print(f"\n  {act} n={n}")
    check_bf16("kernel fwd", y, y64, t_y)
    check_bf16("kernel bwd", dx, d64, t_d)
    xc, dyc = _cpu(x, dy)
    check_bf16("stand-in fwd", emu.act_fwd(xc, act), y64.cpu(), t_y.cpu())
    check_bf16("stand-in bwd", emu.act_bwd(dyc, xc, act), d64.cpu(), t_d.cpu())


# ================================================================================================== gradient routing
def _splice_inputs(B, S, H, q_side, vocab, starts, seed):
    g = _gen(seed)
    ids = torch.randint(0, 40, (B, S), generator=g, device=DEV)          # many repeats
    ids[0, 0], ids[0, 1], ids[-1, -1], ids[-1, -2] = -1, -100, vocab, vocab + 3   # out of range -> row 0
    img_start = torch.tensor(starts, dtype=torch.int32, device=DEV)
    dout = _randn((B, S, H), seed + 1, 1.0)
    return ids, img_start, dout


def _text_rows(ids, img_start, q_side, vocab):
    """flat positions that carry an embedding gradient, and the row each adds into (out of range -> 0)."""
    B, S = ids.shape
    span = q_side * (q_side + 1)
    pos = torch.arange(S, device=ids.device)[None]
    st = img_start.long()[:, None] if img_start is not None else torch.full((B, 1), -1, device=ids.device)
    text = ~((st >= 0) & (pos >= st) & (pos < st + span))
    row = torch.where((ids < 0) | (ids >= vocab), torch.zeros_like(ids), ids)
    return text.reshape(-1), row.reshape(-1)


def test_embed_splice_bwd(ops):
    B, S, H, q, vocab = 2, 64, 1024, 3, 50
    ids, img_start, dout = _splice_inputs(B, S, H, q, vocab, [5, 40], 80)
    d_embed = torch.zeros(vocab, H, dtype=torch.bfloat16, device=DEV)
    d_img, d_nl = ops.embed_splice_bwd(dout, ids, img_start, d_embed, q, True)
    torch.cuda.synchronize()
    print("\n  embed_splice_bwd")
    e_img, e_nl = emu.embed_splice_bwd(*_cpu(dout, ids, img_start), None, q, True)
    flat = dout.reshape(B * S, H)
    want_img = torch.stack([flat[b * S + img_start[b] + r * (q + 1) + c] for b in range(B) for r in range(q) for c in range(q)])
    want_nl = torch.stack([flat[b * S + img_start[b] + r * (q + 1) + q] for b in range(B) for r in range(q)])
    assert_bitwise("kernel d_img", d_img.reshape(-1, H), want_img)
    assert_bitwise("kernel d_nl rows", d_nl, want_nl)
    assert_bitwise("stand-in d_img", e_img.reshape(-1, H), want_img)
    assert_bitwise("stand-in d_nl rows", e_nl, want_nl)
    text, row = _text_rows(ids, img_start, q, vocab)
    acc = torch.zeros(vocab, H, dtype=torch.float64, device=DEV).index_add_(0, row[text], flat[text].double())
    mag = torch.zeros(vocab, H, dtype=torch.float64, device=DEV).index_add_(0, row[text], flat[text].double().abs())
    cnt = torch.zeros(vocab, dtype=torch.float64, device=DEV).index_add_(0, row[text], torch.ones_like(row[text], dtype=torch.float64))
    # bf16x2 atomics: each of a row's cnt - 1 later additions rounds the running sum to bf16 (<= 2^-8 of the terms so far)
    check_bf16("kernel d_embed (bf16 atomics)", d_embed, acc, (cnt - 1).clamp_min(0)[:, None] * HALF_ULP * mag * (1 + HALF_ULP))


@pytest.mark.parametrize("H", [1024, 1280])
def test_embed_grad_sorted(ops, H):
    B, S, q, vocab = 2, 200, 4, 300
    ids, img_start, dout = _splice_inputs(B, S, H, q, vocab, [10, -1], 90 + H)
    d0 = _randn((vocab, H), 91, 0.5)                     # running sum of an earlier micro-batch: the op adds to it
    d_embed = d0.clone()
    ops.embed_grad_sorted(dout, ids, img_start, d_embed, q)
    torch.cuda.synchronize()
    print(f"\n  embed_grad_sorted H={H} (vectors per row {H // 8}, 128 threads)")
    text, row = _text_rows(ids, img_start, q, vocab)
    flat = dout.reshape(B * S, H)
    acc = torch.zeros(vocab, H, dtype=torch.float64, device=DEV).index_add_(0, row[text], flat[text].double())
    mag = torch.zeros(vocab, H, dtype=torch.float64, device=DEV).index_add_(0, row[text], flat[text].double().abs())
    cnt = torch.zeros(vocab, dtype=torch.long, device=DEV).index_add_(0, row[text], torch.ones_like(row[text]))
    touched = cnt > 0
    assert bool(touched[0]) and int(cnt.max()) > 1
    want = acc + d0.double()
    # a row's cnt terms are added in position order in fp32, then the old value: (cnt + 1) u of the magnitudes
    tol = (cnt[:, None] + 1).double() * U * (mag + d0.double().abs()) * (1 + HALF_ULP)
    check_bf16("kernel touched rows", d_embed[touched], want[touched], tol[touched])
    assert_bitwise("kernel untouched rows", d_embed[~touched], d0[~touched])
    de = d0.cpu().clone()
    emu.embed_grad_sorted(*_cpu(dout, ids, img_start), de, q)
    assert_bitwise("stand-in vs kernel (same fp32 order)", de, d_embed)


@pytest.mark.parametrize("fp32", [False, True])
@pytest.mark.parametrize("accumulate", [False, True])
def test_group_colsum(ops, fp32, accumulate):
    G, R, C = 3, 517, 1000                 # C not a multiple of 32: the last column block is partial
    x = _randn((G * R, C), 100, 1.0)
    scale = 1.0 / R
    old = _randn((G, C), 101, 0.2, torch.float32 if fp32 else torch.bfloat16)
    out = old.clone()
    ops.group_colsum(x, G, scale, out=out, accumulate=accumulate)
    torch.cuda.synchronize()
    xs = x.double().reshape(G, R, C)
    want = xs.sum(1) * float(torch.tensor(scale)) + (old.double() if accumulate else 0.0)
    # 8 row lanes add ceil(R / 8) rows each, then the 8 lanes in order, the scale, the += : h u of the magnitudes
    h = -(-R // 8) + 8 + 2
    tol = h * U * xs.abs().sum(1) * scale + (U * old.double().abs() if accumulate else 0.0)
    print(f"\n  group_colsum fp32={fp32} accumulate={accumulate}")
    chk = check_abs if fp32 else check_bf16
    chk("kernel", out, want, tol * (1 + HALF_ULP) if not fp32 else tol + U * want.abs())
    oute = old.cpu().clone()
    rete = emu.group_colsum(x.cpu(), G, scale, out=oute, accumulate=accumulate, fp32=fp32)
    assert rete is oute, "the stand-in must write `out` like the kernel"
    chk("stand-in", oute, want.cpu(), (tol * (1 + HALF_ULP) if not fp32 else tol + U * want.abs()).cpu())


def test_group_broadcast_accumulate(ops):
    G, R, C = 3, 129, 1024
    dmean = _randn((G, C), 110, 1.0)
    old = _randn((G * R, C), 111, 1.0)
    scale = 1.0 / R
    out = old.clone()
    ops.group_broadcast(dmean, R, scale, out=out, accumulate=True)
    torch.cuda.synchronize()
    # the kernel's dmean * scale + old contracts to one fma: the exact value (dmean * scale has 32 significant bits, so the
    # sum is exact in fp64) rounded to fp32, then to bf16, bit for bit
    s32 = float(torch.tensor(scale, dtype=torch.float32))
    exact = (dmean.double() * s32).repeat_interleave(R, 0) + old.double()
    want = exact.float().to(torch.bfloat16)
    print("\n  group_broadcast accumulate")
    assert_bitwise("kernel", out, want)
    oute = old.cpu().clone()
    assert emu.group_broadcast(dmean.cpu(), R, scale, out=oute, accumulate=True) is oute
    # the stand-in rounds the product before the add: the fp64 bound of two fp32 roundings
    check_bf16("stand-in", oute, exact.cpu(), 2 * U * ((dmean.double() * s32).repeat_interleave(R, 0).abs() + old.double().abs()).cpu()
               * (1 + HALF_ULP))
    out2 = ops.group_broadcast(dmean, R, scale)
    assert_bitwise("kernel without accumulate", out2, (dmean.float() * scale).repeat_interleave(R, 0).to(torch.bfloat16))


@pytest.mark.parametrize("layout", ["grid", "windowed"])
@pytest.mark.parametrize("C", [1024, 1000])
def test_pos_grad(ops, layout, C):
    r = 3
    if layout == "grid":
        B, side = 2, 4 * r
    else:
        B, side = 37, r                                    # side == r: the window-rearranged [N, r*r, C] layout
    dx = _randn((B * side * side, C), 120 + C, 1.0)
    old = _randn((r * r, C), 121, 0.5)
    out = old.clone()
    ops.pos_grad(dx, B, side, r, out=out, accumulate=True)
    torch.cuda.synchronize()
    q = side // r
    x6 = dx.double().reshape(B, q, r, q, r, C)
    want = x6.sum((0, 1, 3)).reshape(r * r, C) + old.double()
    mag = x6.abs().sum((0, 1, 3)).reshape(r * r, C)
    tol = ((B * q * q + 1) * U * (mag + old.double().abs())) * (1 + HALF_ULP)
    print(f"\n  pos_grad {layout} C={C} B={B} side={side}")
    check_bf16("kernel", out, want, tol)
    oute = old.cpu().clone()
    assert emu.pos_grad(dx.cpu(), B, side, r, out=oute, accumulate=True) is oute
    check_bf16("stand-in", oute, want.cpu(), tol.cpu())


def test_f32_to_bf16_into_packed_buffer(ops):
    rows, cols, ld = 2200, 1024, 3 * 1024              # dQ lands in the middle third of a packed dQKV buffer
    src = torch.randn(rows, cols, generator=_gen(130), device=DEV) * 5
    buf = _randn((rows, ld), 131, 1.0)
    buf0 = buf.clone()
    scale = 0.125
    ops.f32_to_bf16(src, buf[:, cols:2 * cols], scale, cols=cols, out_ld=ld)
    torch.cuda.synchronize()
    print("\n  f32_to_bf16")
    want = (src * scale).to(torch.bfloat16)
    assert_bitwise("kernel", buf[:, cols:2 * cols], want)
    assert_bitwise("other columns untouched", torch.cat([buf[:, :cols], buf[:, 2 * cols:]], 1),
                   torch.cat([buf0[:, :cols], buf0[:, 2 * cols:]], 1))
    bufe = buf0.cpu().clone()
    emu.f32_to_bf16(src.cpu(), bufe[:, cols:2 * cols], scale, cols=cols, out_ld=ld)
    assert_bitwise("stand-in", bufe, buf)


def test_span_gather_scatter(ops):
    B, S, H, start, q = 3, 120, 1024, 7, 6
    hidden = _randn((B, S, H), 140, 1.0)
    lat = ops.span_gather(hidden, start, q)
    idx = torch.tensor([b * S + start + r * (q + 1) + c for b in range(B) for r in range(q) for c in range(q)], device=DEV)
    print("\n  span_gather / span_scatter_")
    assert_bitwise("gather", lat, hidden.reshape(B * S, H)[idx])
    assert_bitwise("stand-in gather", emu.span_gather(hidden.cpu(), start, q), lat)
    new = _randn((B * q * q, H), 141, 1.0)
    h2 = hidden.clone()
    ops.span_scatter_(h2, new, start, q)
    torch.cuda.synchronize()
    want = hidden.clone().reshape(B * S, H)
    want[idx] = new
    assert_bitwise("scatter (newline rows and the rest untouched)", h2.reshape(B * S, H), want)
    he = hidden.cpu().clone()
    emu.span_scatter_(he, new.cpu(), start, q)
    assert_bitwise("stand-in scatter", he, h2)
