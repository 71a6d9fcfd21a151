"""Hand-scheduled forward/backward of the hot-path blocks, exposed as torch.autograd.Functions.

Each Function launches only kernels of libcambrian_b200.so (through `ops`); torch supplies tensor storage and the
autograd tape between blocks.  Blocks are coarse on purpose (a whole SVA layer, a whole decoder layer) so that every
gradient fan-in is an explicit fused kernel (`dres` of the norm backward, GEMM residual epilogue) instead of an
autograd-inserted add.

Weight gradients: if a parameter carries a `main_grad` tensor (set by `cambrian_b200.engine.TrainEngine`, a view into
the flat bf16 gradient buffer that the optimizer and the NCCL all-reduce consume), the dW GEMM accumulates straight
into it and autograd receives None; otherwise the gradient tensor is returned to autograd as usual.
"""
from __future__ import annotations

import torch

from . import ops, train_fp8


def _ranged(tag):
    """NVTX range around a Function's forward / backward (ops.nvtx: a no-op unless CB_NVTX=1)."""
    def deco(fn):
        def wrapped(*a, **k):
            with ops.nvtx(tag):
                return fn(*a, **k)
        wrapped.__name__ = fn.__name__
        wrapped.__doc__ = fn.__doc__
        return wrapped
    return deco


def _notify(param):
    """Tell the TrainEngine (if any) that one gradient contribution of `param` has been enqueued on the stream; it uses
    the per-step contribution counts to launch a bucket's all-reduce as soon as the bucket is final."""
    n = getattr(param, "_cb_notify", None)
    if n is not None:
        n()


def _await(*params):
    """Before a block's first kernel reads `params`: make the current stream wait for optimizer updates of their buckets
    that the TrainEngine still has in flight on its side stream (engine.await_bucket; a no-op dictionary miss otherwise).
    Accepts nn.Parameters and the fused-weight holders of cambrian_llama (`_params`)."""
    for p in params:
        if p is None:
            continue
        eng = getattr(p, "_cb_engine", None)
        if eng is not None:
            eng.await_bucket(p._cb_bucket)
        else:
            for q in getattr(p, "_params", ()):
                eng = getattr(q, "_cb_engine", None)
                if eng is not None:
                    eng.await_bucket(q._cb_bucket)


def _frozen(param) -> bool:
    return not getattr(param, "requires_grad", True)


def wgrad(param: torch.Tensor, dy2d: torch.Tensor, x2d: torch.Tensor, out_view=None, notify: bool = True):
    """dW[N_out, K_in] = dy2d[rows, N_out]^T @ x2d[rows, K_in].  `out_view` selects a column slice of the gradient
    (used for proj_in's two halves).  Frozen parameters (stage-1 connector pre-training freezes the LLM) cost nothing."""
    if _frozen(param):
        return None
    mg = getattr(param, "main_grad", None)
    if mg is not None:
        tgt = mg if out_view is None else out_view(mg)
        fresh = getattr(param, "_cb_fresh", None)
        key = "all" if out_view is None else id(out_view)
        first = fresh is not None and key not in fresh
        ops.gemm(dy2d, x2d, a_mn=True, b_mn=True, out=tgt, accumulate=not first)
        if fresh is not None:
            fresh.add(key)
        if notify:
            _notify(param)
        return None
    return ops.gemm(dy2d, x2d, a_mn=True, b_mn=True)


def vgrad(param: torch.Tensor, g: torch.Tensor):
    """Gradient of a vector/small parameter computed by a reduction kernel (bf16)."""
    if _frozen(param):
        return None
    mg = getattr(param, "main_grad", None)
    if mg is not None:
        fresh = getattr(param, "_cb_fresh", None)
        if fresh is not None and "all" not in fresh:
            mg.view(-1).copy_(g.view(-1))  # first write of the step (tiny tensors: LN affine, biases)
            fresh.add("all")
        else:
            ops.add_(mg.view(-1), g.contiguous().view(-1)) if mg.numel() % 8 == 0 else mg.add_(g.view_as(mg))
        _notify(param)
        return None
    return g


def _uniform_stack(tensors):
    """If the given equally-shaped 2-D contiguous tensors sit at one constant positive stride in a common storage (the K/V
    projection weights of an SVA layer inside the TrainEngine's flat buffer do: named_parameters() lays them out as
    ln.weight, ln.bias, linear.weight, repeated), return a [n, rows, cols] view over them — a batched GEMM operand without
    any copy.  None otherwise."""
    t0 = tensors[0]
    if len(tensors) < 2 or any(t.shape != t0.shape or not t.is_contiguous() or t.dtype != t0.dtype for t in tensors):
        return None
    st = t0.untyped_storage().data_ptr()
    if any(t.untyped_storage().data_ptr() != st for t in tensors):
        return None
    es = t0.element_size()
    d = (tensors[1].data_ptr() - t0.data_ptr()) // es
    if d <= 0 or (d * es) % 16 or any((tensors[i + 1].data_ptr() - tensors[i].data_ptr()) != d * es for i in range(len(tensors) - 1)):
        return None
    return torch.as_strided(t0, (len(tensors), t0.shape[0], t0.shape[1]), (d, t0.stride(0), 1))


def _kv_groups(feats):
    """Towers with the same number of feature rows share one batched launch (BASELINE grids: all four; release grids
    [576, 576, 576, 9216]: the three small ones, the ConvNeXt grid alone)."""
    groups = {}
    for i, f in enumerate(feats):
        groups.setdefault(f.shape[0], []).append(i)
    return list(groups.values())


def wgrad_batched(params, dy_stack, x_stack):
    """dW_j = dy_stack[j]^T @ x_stack[j] for a group of equally-shaped weights in ONE batched launch.  With TrainEngine
    buffers the results accumulate straight into the (uniformly strided) main_grad slices; otherwise the list of gradient
    tensors is returned.  Falls back to one launch per weight when the layout / state does not allow batching."""
    n = len(params)
    if all(_frozen(p) for p in params):
        return [None] * n
    mgs = [getattr(p, "main_grad", None) for p in params]
    if all(m is None for m in mgs) and not any(_frozen(p) for p in params):
        dw = ops.gemm(dy_stack, x_stack, a_mn=True, b_mn=True)
        return [dw[j] for j in range(n)]
    if all(m is not None for m in mgs) and not any(_frozen(p) for p in params):
        firsts = [p._cb_fresh is not None and "all" not in p._cb_fresh for p in params]
        mstack = _uniform_stack(mgs)
        if mstack is not None and (all(firsts) or not any(firsts)):
            ops.gemm(dy_stack, x_stack, a_mn=True, b_mn=True, out=mstack, accumulate=not firsts[0])
            for p in params:
                if p._cb_fresh is not None:
                    p._cb_fresh.add("all")
                _notify(p)
            return [None] * n
    return [wgrad(p, dy_stack[j], x_stack[j]) for j, p in enumerate(params)]


def _merge_wgrad(parts):
    """Assemble a full-weight gradient from column blocks when no main_grad buffer exists."""
    return torch.cat(parts, dim=1)


# ------------------------------------------------------------------------------------------------------------------
# Linear (+ bias) and small projector MLPs (mm_projector, mm_projector_aux)
# ------------------------------------------------------------------------------------------------------------------
class LinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias):
        _await(weight, bias)
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        ctx.params = (weight, bias)
        return ops.linear(x, weight, bias)

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        w_param, b_param = ctx.params
        dy2 = dy.reshape(-1, dy.shape[-1]).contiguous()
        x2 = x.reshape(-1, x.shape[-1])
        dx = ops.gemm(dy2, weight, b_mn=True).view(x.shape) if ctx.needs_input_grad[0] else None
        dw = wgrad(w_param, dy2, x2) if ctx.needs_input_grad[1] else None
        db = None
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = vgrad(b_param, ops.group_colsum(dy2, 1).view(-1))
        return dx, dw, db


class ActFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, act):
        ctx.save_for_backward(x)
        ctx.act = act
        return ops.act_fwd(x, act)

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        return ops.act_bwd(dy.contiguous(), x, ctx.act), None


class LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, eps):
        _await(weight, bias)
        y, mean, rstd = ops.layernorm_fwd(x, weight, bias, eps, save_stats=True)
        ctx.save_for_backward(x, weight, mean, rstd)
        ctx.params = (weight, bias)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, mean, rstd = ctx.saved_tensors
        dx, dg, db = ops.layernorm_bwd(dy.contiguous(), x, weight, mean, rstd)
        return dx, vgrad(ctx.params[0], dg), vgrad(ctx.params[1], db), None


class RMSNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, eps, hf_cast):
        _await(weight)
        y, rstd = ops.rmsnorm_fwd(x, weight, eps, hf_cast, save_stats=True)
        ctx.save_for_backward(x, weight, rstd)
        ctx.param = weight
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, rstd = ctx.saved_tensors
        dx, dg = ops.rmsnorm_bwd(dy.contiguous(), x, weight, rstd)
        return dx, vgrad(ctx.param, dg), None, None


class MeanTokensFn(torch.autograd.Function):
    """global context = mean over tokens (cambrian_arch.py:377): [B, N, C] -> [B, C]."""

    @staticmethod
    def forward(ctx, x):
        B, N, C = x.shape
        ctx.shape = (B, N, C)
        return ops.group_colsum(x.contiguous(), B, 1.0 / N)

    @staticmethod
    def backward(ctx, dy):
        B, N, C = ctx.shape
        return ops.group_broadcast(dy.contiguous(), N, 1.0 / N).view(B, N, C)


# ------------------------------------------------------------------------------------------------------------------
# SVA layer (VisionCrossAttentionLayer.forward, vision_sampler.py:270-327)
# ------------------------------------------------------------------------------------------------------------------
class SVALayerFn(torch.autograd.Function):
    _nvtx = "SVALayer"

    """args: meta, queries [N,Dq], ctx [N,Dc], feats_0..T-1, then the layer's parameters in `meta['names']` order.

    meta = dict(T, rs, masks (list of bool tensors or None), natural=(B, q_side) or None (window-rearranged inputs),
                params (list of nn.Parameter in the same order as the tensor args))
    """

    @staticmethod
    @_ranged("sva_layer.fwd")
    def forward(ctx, meta, queries, ctxf, *tensors):
        T, rs = meta["T"], meta["rs"]
        _await(*meta["params"])
        feats = [t.reshape(-1, t.shape[-1]) for t in tensors[:T]]
        P = dict(zip(meta["names"], tensors[T:]))
        N, D = queries.shape
        nat = meta["natural"]
        windowed = nat is None
        B, q_side = (N, 1) if windowed else nat
        masks = meta["masks"]

        ctxp = ops.gemm(ctxf, P["proj_context"])
        t32 = ops.gemm(queries, P["proj_in"][:, :D], out_dtype=torch.float32)
        ops.gemm(ctxp, P["proj_in"][:, D:], out=t32, accumulate=True)
        qin = ops.f32_to_bf16(t32, torch.empty((N, t32.shape[1]), dtype=torch.bfloat16, device=queries.device))
        qn, mq, rq = ops.layernorm_fwd(qin, P["q_ln_w"], P["q_ln_b"], 1e-5, save_stats=True)
        Q = ops.gemm(qn, P["q_w"])
        # K/V projections (vision_sampler.py:187-189: a per-tower list comprehension of LayerNorm + Linear).  Towers with equal
        # row counts are ONE batched GEMM [2g, rows, 1024] x [2g, 1024, 1024]: the 2g LayerNorm outputs are written into one
        # buffer, the 2g weights are read in place through a strided view when they sit at a uniform stride (TrainEngine
        # flat buffer) — 8 sub-wave launches of 144 tiles become one launch of 1152 tiles.
        kins, vins, stats, Ks, Vs = [None] * T, [None] * T, [None] * (2 * T), [None] * T, [None] * T
        kv_w = []          # per group: the stacked-weight view (saved for backward) or None
        for grp in _kv_groups(feats):
            g = len(grp)
            rows = feats[grp[0]].shape[0]
            wstack = _uniform_stack([P[f"{kv}_w_{i}"] for i in grp for kv in ("k", "v")]) if g > 1 else None
            kv_w.append(wstack)
            xin = torch.empty((2 * g, rows, feats[grp[0]].shape[1]), dtype=torch.bfloat16, device=queries.device) \
                if wstack is not None else None
            for j, i in enumerate(grp):
                r = rs[i]
                pos = P.get(f"pos_embed_{i}") if r > 1 else None
                side = 0 if windowed else r * q_side
                kin, mean, rstd = ops.layernorm_fwd(feats[i], P[f"k_ln_w_{i}"], P[f"k_ln_b_{i}"], 1e-5, pos=pos, side=side,
                                                    r=r, save_stats=True, out=None if xin is None else xin[2 * j])
                vin = ops.layernorm_fwd(feats[i], P[f"v_ln_w_{i}"], P[f"v_ln_b_{i}"], 1e-5, pos=pos, side=side, r=r,
                                        out=None if xin is None else xin[2 * j + 1])
                kins[i], vins[i] = kin, vin
                stats[2 * i], stats[2 * i + 1] = mean, rstd
            if wstack is not None:
                kv = ops.gemm(xin, wstack)                       # [2g, rows, 1024]
                for j, i in enumerate(grp):
                    Ks[i], Vs[i] = kv[2 * j], kv[2 * j + 1]
            else:
                for i in grp:
                    Ks[i] = ops.gemm(kins[i], P[f"k_w_{i}"])
                    Vs[i] = ops.gemm(vins[i], P[f"v_w_{i}"])
        A, lse = ops.sva_window_attn_fwd(Q, Ks, Vs, masks, rs, B, q_side, need_lse=True, windowed=windowed)
        q2 = ops.gemm(A, P["o_w"], residual=qin)
        q3, m3, r3 = ops.layernorm_fwd(q2, P["norm_w"], P["norm_b"], 1e-5, save_stats=True)
        h1 = ops.gemm(q3, P["out1_w"])
        h2 = ops.act_fwd(h1, "gelu")
        out = ops.gemm(h2, P["out2_w"], residual=queries)

        ctx.meta = meta
        ctx.dims = (N, D, B, q_side, windowed)
        ctx.nparams = len(meta["names"])
        ctx.save_for_backward(queries, ctxf, ctxp, qin, mq, rq, qn, Q, A, lse, q2, m3, r3, q3, h1, h2,
                              *feats, *kins, *vins, *stats, *Ks, *Vs, *tensors[T:])
        return out

    @staticmethod
    @_ranged("sva_layer.bwd")
    def backward(ctx, dout):
        meta = ctx.meta
        T, rs, masks = meta["T"], meta["rs"], meta["masks"]
        N, D, B, q_side, windowed = ctx.dims
        sv = ctx.saved_tensors
        queries, ctxf, ctxp, qin, mq, rq, qn, Q, A, lse, q2, m3, r3, q3, h1, h2 = sv[:16]
        o = 16
        feats = sv[o:o + T]; o += T
        kins = sv[o:o + T]; o += T
        vins = sv[o:o + T]; o += T
        stats = sv[o:o + 2 * T]; o += 2 * T
        Ks = sv[o:o + T]; o += T
        Vs = sv[o:o + T]; o += T
        P = dict(zip(meta["names"], sv[o:]))
        prm = dict(zip(meta["names"], meta["params"]))
        g = {}
        dout = dout.contiguous()

        dh2 = ops.gemm(dout, P["out2_w"], b_mn=True)
        g["out2_w"] = wgrad(prm["out2_w"], dout, h2)
        dh1 = ops.act_bwd(dh2, h1, "gelu")
        dq3 = ops.gemm(dh1, P["out1_w"], b_mn=True)
        g["out1_w"] = wgrad(prm["out1_w"], dh1, q3)
        dq2, dgn, dbn = ops.layernorm_bwd(dq3, q2, P["norm_w"], m3, r3)
        g["norm_w"], g["norm_b"] = vgrad(prm["norm_w"], dgn), vgrad(prm["norm_b"], dbn)
        dA = ops.gemm(dq2, P["o_w"], b_mn=True)
        g["o_w"] = wgrad(prm["o_w"], dq2, A)
        # dK / dV land in one stacked buffer per equal-row group so that dX = dKV @ W and dW = dKV^T @ X are batched launches
        groups = _kv_groups(feats)
        stacks = {}
        dKs, dVs = [None] * T, [None] * T
        for grp in groups:
            ng = len(grp)
            wstack = _uniform_stack([P[f"{kv}_w_{i}"] for i in grp for kv in ("k", "v")]) if ng > 1 else None
            xstack = _uniform_stack([t for i in grp for t in (kins[i], vins[i])]) if wstack is not None else None
            if wstack is not None and xstack is not None:
                dkv = torch.empty((2 * ng,) + tuple(Ks[grp[0]].shape), dtype=torch.bfloat16, device=dout.device)
                for j, i in enumerate(grp):
                    dKs[i], dVs[i] = dkv[2 * j], dkv[2 * j + 1]
                stacks[grp[0]] = (wstack, xstack, dkv)
            else:
                for i in grp:
                    dKs[i], dVs[i] = torch.empty_like(Ks[i]), torch.empty_like(Vs[i])
        dQ, _, _ = ops.sva_window_attn_bwd(Q, A, dA, lse, list(Ks), list(Vs), masks, rs, B, q_side, windowed=windowed,
                                           dks=dKs, dvs=dVs)
        dqn = ops.gemm(dQ, P["q_w"], b_mn=True)
        g["q_w"] = wgrad(prm["q_w"], dQ, qn)
        dqin, dgq, dbq = ops.layernorm_bwd(dqn, qin, P["q_ln_w"], mq, rq, dres=dq2)
        g["q_ln_w"], g["q_ln_b"] = vgrad(prm["q_ln_w"], dgq), vgrad(prm["q_ln_b"], dbq)
        dfeats = [None] * T
        for grp in groups:
            batched = stacks.get(grp[0])
            if batched is not None:
                wstack, xstack, dkv = batched
                dxin = ops.gemm(dkv, wstack, b_mn=True)                                  # [2g, rows, 1024]
                names = [f"{kv}_w_{i}" for i in grp for kv in ("k", "v")]
                for nme, gw in zip(names, wgrad_batched([prm[nme] for nme in names], dkv, xstack)):
                    g[nme] = gw
            for j, i in enumerate(grp):
                r = rs[i]
                pos = P.get(f"pos_embed_{i}") if r > 1 else None
                side = 0 if windowed else r * q_side
                mean, rstd = stats[2 * i], stats[2 * i + 1]
                if batched is not None:
                    dkin, dvin = dxin[2 * j], dxin[2 * j + 1]
                else:
                    dkin = ops.gemm(dKs[i], P[f"k_w_{i}"], b_mn=True)
                    g[f"k_w_{i}"] = wgrad(prm[f"k_w_{i}"], dKs[i], kins[i])
                    dvin = ops.gemm(dVs[i], P[f"v_w_{i}"], b_mn=True)
                    g[f"v_w_{i}"] = wgrad(prm[f"v_w_{i}"], dVs[i], vins[i])
                dxk, dgk, dbk = ops.layernorm_bwd(dkin, feats[i], P[f"k_ln_w_{i}"], mean, rstd, pos=pos, side=side, r=r)
                dxv, dgv, dbv = ops.layernorm_bwd(dvin, feats[i], P[f"v_ln_w_{i}"], mean, rstd, pos=pos, side=side, r=r,
                                                  dres=dxk)
                g[f"k_ln_w_{i}"], g[f"k_ln_b_{i}"] = vgrad(prm[f"k_ln_w_{i}"], dgk), vgrad(prm[f"k_ln_b_{i}"], dbk)
                g[f"v_ln_w_{i}"], g[f"v_ln_b_{i}"] = vgrad(prm[f"v_ln_w_{i}"], dgv), vgrad(prm[f"v_ln_b_{i}"], dbv)
                if r > 1:
                    if windowed:
                        dp = ops.pos_grad(dxv, dxv.shape[0] // (r * r), r, r)
                    else:
                        dp = ops.pos_grad(dxv, B, r * q_side, r)
                    g[f"pos_embed_{i}"] = vgrad(prm[f"pos_embed_{i}"], dp)
                dfeats[i] = dxv
        dqueries = ops.gemm(dqin, P["proj_in"][:, :D], b_mn=True, residual=dout)
        dctxp = ops.gemm(dqin, P["proj_in"][:, D:], b_mn=True)
        w_in = prm["proj_in"]
        if getattr(w_in, "main_grad", None) is not None:
            wgrad(w_in, dqin, queries, out_view=_slice_a(D))
            wgrad(w_in, dqin, ctxp, out_view=_slice_b(D))
            g["proj_in"] = None
        else:
            g["proj_in"] = torch.cat([ops.gemm(dqin, queries, a_mn=True, b_mn=True),
                                      ops.gemm(dqin, ctxp, a_mn=True, b_mn=True)], 1)
        dctx = ops.gemm(dctxp, P["proj_context"], b_mn=True)
        g["proj_context"] = wgrad(prm["proj_context"], dctxp, ctxf)
        tensors_in = meta["feat_shapes"]
        dfeats = [d.view(s) for d, s in zip(dfeats, tensors_in)]
        return (None, dqueries, dctx, *dfeats, *[g.get(n) for n in meta["names"]])


_slice_cache: dict = {}


def _slice_a(D):
    k = ("a", D)
    if k not in _slice_cache:
        _slice_cache[k] = lambda t: t[:, :D]
    return _slice_cache[k]


def _slice_b(D):
    k = ("b", D)
    if k not in _slice_cache:
        _slice_cache[k] = lambda t: t[:, D:]
    return _slice_cache[k]


# ------------------------------------------------------------------------------------------------------------------
# `sep` SVA layer (VisionAggregationLayer.forward, vision_sampler.py:330-405) — building blocks.  The layer type is API
# surface only (no reference caller constructs it, cambrian_arch.py:60-68 use the default "joint"), so it is composed of
# finer-grained Functions instead of one hand-scheduled block; every kernel is still one of libcambrian_b200.so.
# ------------------------------------------------------------------------------------------------------------------
class CatLinearFn(torch.autograd.Function):
    """y = cat([a, b], -1) @ W^T without materialising the concatenation (vision_sampler.py:362 + :366 / :370): two GEMMs
    over the column halves of W accumulate in fp32, rounded to bf16 once."""

    @staticmethod
    def forward(ctx, a, b, weight):
        _await(weight)
        D = a.shape[1]
        t32 = ops.gemm(a, weight[:, :D], out_dtype=torch.float32)
        ops.gemm(b, weight[:, D:], out=t32, accumulate=True)
        y = ops.f32_to_bf16(t32, torch.empty(t32.shape, dtype=torch.bfloat16, device=a.device))
        ctx.save_for_backward(a, b, weight)
        ctx.param = weight
        return y

    @staticmethod
    def backward(ctx, dy):
        a, b, weight = ctx.saved_tensors
        D = a.shape[1]
        dy = dy.contiguous()
        da = ops.gemm(dy, weight[:, :D], b_mn=True) if ctx.needs_input_grad[0] else None
        db = ops.gemm(dy, weight[:, D:], b_mn=True) if ctx.needs_input_grad[1] else None
        dw = None
        w_param = ctx.param
        if ctx.needs_input_grad[2] and not _frozen(w_param):
            if getattr(w_param, "main_grad", None) is not None:
                wgrad(w_param, dy, a, out_view=_slice_a(D), notify=False)
                wgrad(w_param, dy, b, out_view=_slice_b(D))
            else:
                dw = torch.cat([ops.gemm(dy, a, a_mn=True, b_mn=True), ops.gemm(dy, b, a_mn=True, b_mn=True)], 1)
        return da, db, dw


class LinearResidualFn(torch.autograd.Function):
    """y = x @ W^T + residual (residual add in the GEMM epilogue; vision_sampler.py:400-402)."""

    @staticmethod
    def forward(ctx, x, weight, residual):
        _await(weight)
        ctx.save_for_backward(x, weight)
        ctx.param = weight
        return ops.gemm(x, weight, residual=residual.contiguous())

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dy = dy.contiguous()
        dx = ops.gemm(dy, weight, b_mn=True) if ctx.needs_input_grad[0] else None
        dw = wgrad(ctx.param, dy, x) if ctx.needs_input_grad[1] else None
        return dx, dw, (dy if ctx.needs_input_grad[2] else None)


class NarrowLinearFn(torch.autograd.Function):
    """y[N, 8] = x @ pad8(W)^T for a weight with fewer than 8 output rows (weight_mlp.linear_2: one logit per tower,
    vision_sampler.py:341,367).  The output keeps the 8-column padding (16-byte rows); columns >= W.shape[0] are zero."""

    PAD = 8

    @staticmethod
    def forward(ctx, x, weight):
        _await(weight)
        T, K = weight.shape
        if T > NarrowLinearFn.PAD:
            raise ValueError(f"NarrowLinearFn: {T} output rows > {NarrowLinearFn.PAD}")
        wpad = torch.zeros((NarrowLinearFn.PAD, K), dtype=weight.dtype, device=weight.device)
        wpad[:T].copy_(weight)
        ctx.save_for_backward(x, wpad)
        ctx.param, ctx.T = weight, T
        return ops.gemm(x, wpad)

    @staticmethod
    def backward(ctx, dy):
        x, wpad = ctx.saved_tensors
        dy = dy.contiguous()
        dx = ops.gemm(dy, wpad, b_mn=True) if ctx.needs_input_grad[0] else None
        dw = None
        if ctx.needs_input_grad[1] and not _frozen(ctx.param):
            dw = vgrad(ctx.param, ops.gemm(dy, x, a_mn=True, b_mn=True)[:ctx.T].contiguous())
        return dx, dw


class TowerCombineFn(torch.autograd.Function):
    """q_in + sum_t softmax(logits)[:, t] * agg_t (vision_sampler.py:367-368, :394-396) in one kernel."""

    @staticmethod
    def forward(ctx, logits, q_in, *aggs):
        aggs = [a.contiguous() for a in aggs]
        logits = logits.contiguous()
        ctx.save_for_backward(logits, *aggs)
        return ops.tower_combine_fwd(logits, aggs, q_in.contiguous())

    @staticmethod
    def backward(ctx, dout):
        logits, *aggs = ctx.saved_tensors
        dout = dout.contiguous()
        daggs, dlogits = ops.tower_combine_bwd(logits, aggs, dout)
        return (dlogits if ctx.needs_input_grad[0] else None, dout, *daggs)


class CrossAttnTowerFn(torch.autograd.Function):
    """AggregationBlock with attention (CrossAttention.forward, vision_sampler.py:79-121) for ONE tower whose window has
    r^2 > 1 keys: q_proj / k_proj / v_proj = LayerNorm + Linear, window softmax (the SVA kernel with a single tower),
    o_proj; the layer's pos_embed is added to the latents inside the K/V LayerNorm kernels (:382-387).

    args: meta, q_in [N, 1024], feat (natural [B, (r q)^2, 1024] or windowed [N, r^2, 1024]), then the parameters
    q_ln_w, q_ln_b, q_w, k_ln_w, k_ln_b, k_w, v_ln_w, v_ln_b, v_w, o_w, pos.
    meta = dict(r, mask (bool [N, r^2] or None), natural=(B, q_side) or None, params (the 11 nn.Parameters))"""

    NAMES = ("q_ln_w", "q_ln_b", "q_w", "k_ln_w", "k_ln_b", "k_w", "v_ln_w", "v_ln_b", "v_w", "o_w", "pos")

    @staticmethod
    def forward(ctx, meta, q_in, feat, *tensors):
        _await(*meta["params"])
        P = dict(zip(CrossAttnTowerFn.NAMES, tensors))
        r = meta["r"]
        N = q_in.shape[0]
        nat = meta["natural"]
        windowed = nat is None
        B, q_side = (N, 1) if windowed else nat
        side = 0 if windowed else r * q_side
        masks = None if meta["mask"] is None else [meta["mask"]]
        f2 = feat.reshape(-1, feat.shape[-1])
        qn, mq, rq = ops.layernorm_fwd(q_in, P["q_ln_w"], P["q_ln_b"], 1e-5, save_stats=True)
        Q = ops.gemm(qn, P["q_w"])
        kin, mean, rstd = ops.layernorm_fwd(f2, P["k_ln_w"], P["k_ln_b"], 1e-5, pos=P["pos"], side=side, r=r, save_stats=True)
        vin = ops.layernorm_fwd(f2, P["v_ln_w"], P["v_ln_b"], 1e-5, pos=P["pos"], side=side, r=r)
        K = ops.gemm(kin, P["k_w"])
        V = ops.gemm(vin, P["v_w"])
        A, lse = ops.sva_window_attn_fwd(Q, [K], [V], masks, [r], B, q_side, need_lse=True, windowed=windowed)
        out = ops.gemm(A, P["o_w"])
        ctx.meta = meta
        ctx.dims = (N, B, q_side, windowed, side, feat.shape)
        ctx.save_for_backward(q_in, f2, qn, mq, rq, Q, kin, vin, mean, rstd, K, V, A, lse, *tensors)
        return out

    @staticmethod
    def backward(ctx, dout):
        meta = ctx.meta
        r = meta["r"]
        N, B, q_side, windowed, side, fshape = ctx.dims
        sv = ctx.saved_tensors
        q_in, f2, qn, mq, rq, Q, kin, vin, mean, rstd, K, V, A, lse = sv[:14]
        P = dict(zip(CrossAttnTowerFn.NAMES, sv[14:]))
        prm = dict(zip(CrossAttnTowerFn.NAMES, meta["params"]))
        masks = None if meta["mask"] is None else [meta["mask"]]
        g = {}
        dout = dout.contiguous()
        dA = ops.gemm(dout, P["o_w"], b_mn=True)
        g["o_w"] = wgrad(prm["o_w"], dout, A)
        dQ, (dK,), (dV,) = ops.sva_window_attn_bwd(Q, A, dA, lse, [K], [V], masks, [r], B, q_side, windowed=windowed)
        dqn = ops.gemm(dQ, P["q_w"], b_mn=True)
        g["q_w"] = wgrad(prm["q_w"], dQ, qn)
        dq_in, dgq, dbq = ops.layernorm_bwd(dqn, q_in, P["q_ln_w"], mq, rq)
        g["q_ln_w"], g["q_ln_b"] = vgrad(prm["q_ln_w"], dgq), vgrad(prm["q_ln_b"], dbq)
        dkin = ops.gemm(dK, P["k_w"], b_mn=True)
        g["k_w"] = wgrad(prm["k_w"], dK, kin)
        dvin = ops.gemm(dV, P["v_w"], b_mn=True)
        g["v_w"] = wgrad(prm["v_w"], dV, vin)
        dxk, dgk, dbk = ops.layernorm_bwd(dkin, f2, P["k_ln_w"], mean, rstd, pos=P["pos"], side=side, r=r)
        dxv, dgv, dbv = ops.layernorm_bwd(dvin, f2, P["v_ln_w"], mean, rstd, pos=P["pos"], side=side, r=r, dres=dxk)
        g["k_ln_w"], g["k_ln_b"] = vgrad(prm["k_ln_w"], dgk), vgrad(prm["k_ln_b"], dbk)
        g["v_ln_w"], g["v_ln_b"] = vgrad(prm["v_ln_w"], dgv), vgrad(prm["v_ln_b"], dbv)
        dp = ops.pos_grad(dxv, dxv.shape[0] // (r * r), r, r) if windowed else ops.pos_grad(dxv, B, r * q_side, r)
        g["pos"] = vgrad(prm["pos"], dp)
        return (None, dq_in, dxv.view(fshape), *[g[n] for n in CrossAttnTowerFn.NAMES])


# ------------------------------------------------------------------------------------------------------------------
# LLaMA decoder layer (HF LlamaDecoderLayer as called from cambrian_llama.py:142-166)
# ------------------------------------------------------------------------------------------------------------------
class DecoderLayerFn(torch.autograd.Function):
    _nvtx = "DecoderLayer"

    """x [B,S,H] -> x'.  Parameters: input_ln, qkv_w (fused [ (nh+2nkv)*hd, H ]), o_w, post_ln, gu_w (fused [2I, H]), down_w.

    meta = dict(nh, nkv, hd, eps, hf_cast, cos, sin, pos (int64 [B*S]), kmask (bool [B,S] or None), params (6 Parameters),
                recompute (bool: keep only x and redo the forward in backward — per-layer activation checkpointing),
                fp8 (bool, optional: the four projection GEMMs and their input-gradient GEMMs in E4M3, train_fp8.py),
                window (int, optional: causal sliding window of the attention, 0 = none; Phi-3))
    """

    @staticmethod
    def _forward(meta, x, ln1, qkv_w, o_w, ln2, gu_w, down_w, keep, need_out=True):
        B, S, H = x.shape
        nh, nkv, hd = meta["nh"], meta["nkv"], meta["hd"]
        rows = B * S
        fp8 = meta.get("fp8", False)
        x2 = x.reshape(rows, H)
        if fp8:  # train_fp8.py: each weight quantised row-wise here, per call; activations per token
            hq, rstd1 = ops.rmsnorm_fwd_fp8(x2, ln1, meta["eps"], meta["hf_cast"])
            qkv = ops.gemm_fp8(hq, train_fp8.weight_rows(qkv_w))
            del hq
        else:
            h, rstd1 = ops.rmsnorm_fwd(x2, ln1, meta["eps"], meta["hf_cast"], save_stats=True)
            qkv = ops.gemm(h, qkv_w)
        ops.rope_(qkv, meta["pos"], meta["cos"], meta["sin"], nh + nkv, hd)
        q = qkv[:, : nh * hd].view(B, S, nh, hd)
        k = qkv[:, nh * hd:(nh + nkv) * hd].view(B, S, nkv, hd)
        v = qkv[:, (nh + nkv) * hd:].view(B, S, nkv, hd)
        win = {"window": meta["window"]} if meta.get("window") else {}
        attn, lse = ops.attn_fwd(q, k, v, causal=True, kmask=meta["kmask"], need_lse=True, **win)
        attn2 = attn.view(rows, nh * hd)
        if fp8:
            x1 = ops.gemm_fp8(ops.fp8_quantize_act(attn2), train_fp8.weight_rows(o_w), residual=x2)
            h2q, rstd2 = ops.rmsnorm_fwd_fp8(x1, ln2, meta["eps"], meta["hf_cast"])
            gu = ops.gemm_fp8(h2q, train_fp8.weight_rows(gu_w))
            del h2q
            I = gu_w.shape[0] // 2
            act = ops.swiglu_fwd(gu[:, :I], gu[:, I:])
        else:
            x1 = ops.gemm(attn2, o_w, residual=x2)
            h2, rstd2 = ops.rmsnorm_fwd(x1, ln2, meta["eps"], meta["hf_cast"], save_stats=True)
            gu, act = ops.mlp_gate_up(h2, gu_w)
        saved = (rstd1, qkv, attn, lse, x1, rstd2, gu, act) if keep else None
        if not need_out:  # the backward's recompute needs only the saved activations, not the layer's output
            return None, saved
        if fp8:
            out = ops.gemm_fp8(ops.fp8_quantize_act(act), train_fp8.weight_rows(down_w), residual=x1)
        else:
            out = ops.gemm(act, down_w, residual=x1)
        return out.view(B, S, H), saved

    @staticmethod
    @_ranged("decoder_layer.fwd")
    def forward(ctx, meta, x, ln1, q_w, k_w, v_w, o_w, ln2, gate_w, up_w, down_w):
        # q_w/k_w/v_w and gate_w/up_w are the HF-named leaf parameters (for autograd bookkeeping); the GEMMs use the
        # fused views meta["qkv_w"] / meta["gu_w"] over the same storage (CBLlamaDecoderLayer._fused()).
        return DecoderLayerFn._forward_saving(ctx, meta, x, ln1, meta["qkv_w"], o_w, ln2, meta["gu_w"], down_w)

    @staticmethod
    def _forward_saving(ctx, meta, x, ln1, qkv_w, o_w, ln2, gu_w, down_w):
        keep = not meta["recompute"]
        _await(*meta["params"])
        out, saved = DecoderLayerFn._forward(meta, x, ln1, qkv_w, o_w, ln2, gu_w, down_w, keep)
        ctx.meta = meta
        if keep:
            ctx.save_for_backward(x, ln1, qkv_w, o_w, ln2, gu_w, down_w, *saved)
        else:
            ctx.save_for_backward(x, ln1, qkv_w, o_w, ln2, gu_w, down_w)
        return out

    @staticmethod
    @_ranged("decoder_layer.bwd")
    def backward(ctx, dout):
        nh, nkv, hd = ctx.meta["nh"], ctx.meta["nkv"], ctx.meta["hd"]
        dx, g_ln1, g_qkv, g_o, g_ln2, g_gu, g_down = DecoderLayerFn._backward(ctx, dout)
        gq = gk = gv = gg = gup = None
        if g_qkv is not None:  # no main_grad buffers: hand autograd the per-parameter slices of the fused gradient
            gq, gk, gv = g_qkv[: nh * hd], g_qkv[nh * hd:(nh + nkv) * hd], g_qkv[(nh + nkv) * hd:]
        if g_gu is not None:
            I = g_gu.shape[0] // 2
            gg, gup = g_gu[:I], g_gu[I:]
        return None, dx, g_ln1, gq, gk, gv, g_o, g_ln2, gg, gup, g_down

    @staticmethod
    def _backward(ctx, dout):
        """-> dx, then the gradients of ln1, the fused qkv weight, o, ln2, the fused gate|up weight and down (None where
        they went to main_grad or the parameter is frozen)."""
        meta = ctx.meta
        sv = ctx.saved_tensors
        x, ln1, qkv_w, o_w, ln2, gu_w, down_w = sv[:7]
        if meta["recompute"]:
            _, saved = DecoderLayerFn._forward(meta, x, ln1, qkv_w, o_w, ln2, gu_w, down_w, True, need_out=False)
        else:
            saved = sv[7:]
        rstd1, qkv, attn, lse, x1, rstd2, gu, act = saved
        # p_qkv / p_gu: holders exposing .main_grad (fused view over the three / two adjacent grad slices) or None
        p_ln1, p_qkv, p_o, p_ln2, p_gu, p_down = meta["params"]
        B, S, H = x.shape
        nh, nkv, hd = meta["nh"], meta["nkv"], meta["hd"]
        rows = B * S
        I = gu_w.shape[0] // 2
        x2 = x.reshape(rows, H)
        dx2 = dout.reshape(rows, H).contiguous()
        # dgrad: dX = dY W, either bf16 (W as the MN-major operand) or E4M3 on W^T quantised here, per call (train_fp8.py)
        fp8 = meta.get("fp8", False)
        if fp8:
            _await(*meta["params"])

        def dgrad(dy, w):
            if fp8:
                return ops.gemm_fp8(ops.fp8_quantize_act(dy), train_fp8.weight_t(w))
            return ops.gemm(dy, w, b_mn=True)

        # ---- MLP
        h2 = ops.rmsnorm_fwd(x1, ln2, meta["eps"], meta["hf_cast"])       # cheap recompute (bandwidth only)
        dact = dgrad(dx2, down_w)
        g_down = wgrad(p_down, dx2, act)
        del act
        dgu = torch.empty_like(gu)
        if fp8:  # the bf16 dgu feeds the gate|up wgrad, its E4M3 rows the gate|up dgrad
            dguq = ops.swiglu_bwd_fp8(dact, gu[:, :I], gu[:, I:], dgu[:, :I], dgu[:, I:])
            del dact
            dh2 = ops.gemm_fp8(dguq, train_fp8.weight_t(gu_w))
            del dguq
        else:
            ops.swiglu_bwd(dact, gu[:, :I], gu[:, I:], dgu[:, :I], dgu[:, I:])
            del dact
            dh2 = ops.gemm(dgu, gu_w, b_mn=True)
        g_gu = wgrad(p_gu, dgu, h2)
        del dgu, h2
        dx1, dg2 = ops.rmsnorm_bwd(dh2, x1, ln2, rstd2, dres=dx2)
        g_ln2 = vgrad(p_ln2, dg2)
        # ---- attention
        attn2 = attn.view(rows, nh * hd)
        dattn = dgrad(dx1, o_w)
        g_o = wgrad(p_o, dx1, attn2)
        dqkv = torch.empty_like(qkv)
        q = qkv[:, : nh * hd].view(B, S, nh, hd)
        k = qkv[:, nh * hd:(nh + nkv) * hd].view(B, S, nkv, hd)
        v = qkv[:, (nh + nkv) * hd:].view(B, S, nkv, hd)
        win = {"window": meta["window"]} if meta.get("window") else {}
        ops.attn_bwd(q, k, v, attn, dattn.view(B, S, nh, hd), lse, causal=True, kmask=meta["kmask"],
                     dq=dqkv[:, : nh * hd].view(B, S, nh, hd), dk=dqkv[:, nh * hd:(nh + nkv) * hd].view(B, S, nkv, hd),
                     dv=dqkv[:, (nh + nkv) * hd:].view(B, S, nkv, hd), **win)
        ops.rope_(dqkv, meta["pos"], meta["cos"], meta["sin"], nh + nkv, hd, inverse=True)
        h = ops.rmsnorm_fwd(x2, ln1, meta["eps"], meta["hf_cast"])
        dh = dgrad(dqkv, qkv_w)
        g_qkv = wgrad(p_qkv, dqkv, h)
        del dqkv, h
        dx, dg1 = ops.rmsnorm_bwd(dh, x2, ln1, rstd1, dres=dx1)
        g_ln1 = vgrad(p_ln1, dg1)
        return dx.view(B, S, H), g_ln1, g_qkv, g_o, g_ln2, g_gu, g_down


class FusedDecoderLayerFn(torch.autograd.Function):
    _nvtx = "DecoderLayer"

    """DecoderLayerFn for a layer whose fused weights are themselves the leaf parameters (Phi-3's qkv_proj and
    gate_up_proj): x [B,S,H] -> x'; arguments ln1, qkv_w, o_w, ln2, gu_w, down_w, and the same meta, whose params hold
    the six leaves (each with its own main_grad under TrainEngine)."""

    @staticmethod
    @_ranged("decoder_layer.fwd")
    def forward(ctx, meta, x, ln1, qkv_w, o_w, ln2, gu_w, down_w):
        return DecoderLayerFn._forward_saving(ctx, meta, x, ln1, qkv_w, o_w, ln2, gu_w, down_w)

    @staticmethod
    @_ranged("decoder_layer.bwd")
    def backward(ctx, dout):
        return (None, *DecoderLayerFn._backward(ctx, dout))


# ------------------------------------------------------------------------------------------------------------------
# embedding + image splice, lm_head + loss
# ------------------------------------------------------------------------------------------------------------------
class EmbedSpliceFn(torch.autograd.Function):
    """cambrian_arch.py:413-420 + :457-490 (static branch): embed_tokens gather, image span replace, newline column."""

    @staticmethod
    def forward(ctx, meta, embed_w, img, newline):
        ids, img_start, q_side = meta["ids"], meta["img_start"], meta["q_side"]
        _await(*meta["params"])
        ctx.meta = meta
        ctx.has_img = img is not None
        ctx.vshape = embed_w.shape
        return ops.embed_splice(ids, img_start, embed_w, img, newline, q_side)

    @staticmethod
    def backward(ctx, dout):
        meta = ctx.meta
        p_embed, p_newline = meta["params"]
        dout = dout.contiguous()
        d_embed_ret = None
        tgt = None
        if ctx.needs_input_grad[1]:
            mg = getattr(p_embed, "main_grad", None)
            if mg is not None:
                fresh = getattr(p_embed, "_cb_fresh", None)
                if fresh is not None and "all" not in fresh:
                    mg.zero_()
                    fresh.add("all")
                tgt = mg
            else:
                tgt = torch.zeros(ctx.vshape, dtype=torch.bfloat16, device=dout.device)
                d_embed_ret = tgt
        # image / newline rows are plain gathers; the embedding rows are summed per token id in position order
        # (deterministic: no atomics whose bf16 rounding depends on arrival order)
        d_img, d_nl_rows = ops.embed_splice_bwd(dout, meta["ids"], meta["img_start"], None, meta["q_side"], ctx.has_img)
        if tgt is not None:
            ops.embed_grad_sorted(dout, meta["ids"], meta["img_start"] if ctx.has_img else None, tgt, meta["q_side"])
        if tgt is not None and d_embed_ret is None:
            _notify(p_embed)
        d_nl = None
        if ctx.has_img and ctx.needs_input_grad[3]:
            d_nl = vgrad(p_newline, ops.group_colsum(d_nl_rows, 1).view(-1))
        return None, d_embed_ret, d_img, d_nl


class LMHeadLossFn(torch.autograd.Function):
    _nvtx = "LMHeadLoss"

    """cambrian_llama.py:402-422: lm_head -> logits.float() -> shift -> CrossEntropyLoss(mean over non-ignored), computed
    in row chunks so the [B*S, V] logits are never resident at once; the backward GEMMs run inside the forward (the
    per-chunk (softmax - onehot) overwrites the chunk's logits), so the only saved tensor is dhidden."""

    @staticmethod
    @_ranged("lm_head_loss.fwd")
    def forward(ctx, meta, hidden, weight):
        labels = meta["shift_labels"]  # int64 [B*S]: labels[b, s+1] at row (b, s), -100 on the last position
        rows, H = hidden.reshape(-1, hidden.shape[-1]).shape
        h2 = hidden.reshape(rows, H)
        V = weight.shape[0]
        dev = hidden.device
        chunk = meta.get("chunk", 4096)
        n_valid = meta["n_valid"]  # python int (host-side, from the collator) or None: counted on the device (inv_count_dev)
        inv_dev = meta.get("inv_count_dev")   # fp32 [1] device tensor = 1 / max(#valid labels, 1) when n_valid is None
        train = meta["train"]
        p_w = meta["params"][0]
        _await(p_w)
        need_dw = train and not _frozen(p_w)
        # Rows whose shifted label is ignore_index contribute neither loss nor gradient.  When the collator hands over
        # the row ranges that can hold a valid label (host ints, `label_ranges`), only those rows are pushed through the
        # vocabulary GEMMs: they are packed into one dense buffer (device-to-device copies), dhidden of all other rows
        # is exactly zero.  Without the hint every row is processed, as the reference does.
        ranges = meta.get("label_ranges")
        dh_full = None
        if ranges is not None:
            ranges = [(int(a), int(b)) for a, b in ranges if b > a]
            n_rows = sum(b - a for a, b in ranges)
            hc = torch.empty((max(n_rows, 1), H), dtype=h2.dtype, device=dev)
            lc = torch.full((max(n_rows, 1),), -100, dtype=labels.dtype, device=dev)
            o = 0
            for a, b in ranges:
                hc[o:o + b - a].copy_(h2[a:b])
                lc[o:o + b - a].copy_(labels[a:b])
                o += b - a
            if train:
                dh_full = torch.zeros_like(h2)
            h2, labels, rows = hc, lc, max(n_rows, 1)
        loss_rows = torch.empty(rows, dtype=torch.float32, device=dev)
        acc = torch.zeros(2, dtype=torch.float32, device=dev)
        dh = torch.empty_like(h2) if train else None
        # `loss_scale` (TrainEngine: e.g. 1 / gradient_accumulation_steps) is folded into the gradients formed here; the
        # returned loss value is the unscaled mean.  The gradients are final when forward returns: backward() only hands
        # out dhidden, so `(loss * c).backward()` with c != 1 is NOT supported on this path (use loss_scale).
        gscale = float(meta.get("loss_scale", 1.0)) / (max(n_valid, 1) if n_valid is not None else 1)
        logits = torch.empty((min(chunk, rows), V), dtype=torch.bfloat16, device=dev)
        dw_local = None
        if need_dw and getattr(p_w, "main_grad", None) is None:
            dw_local = torch.empty_like(weight)
        for r0 in range(0, rows, chunk):
            r1 = min(rows, r0 + chunk)
            lg = logits[: r1 - r0]
            ops.gemm(h2[r0:r1], weight, out=lg)
            ops.cross_entropy(lg, labels[r0:r1], loss_rows[r0:r1], acc, gscale, train,
                              scale_dev=inv_dev if n_valid is None else None)
            if train:
                ops.gemm(lg, weight, b_mn=True, out=dh[r0:r1])
                if not need_dw:
                    pass
                elif dw_local is None:
                    wgrad(p_w, lg, h2[r0:r1], notify=False)
                else:
                    ops.gemm(lg, h2[r0:r1], a_mn=True, b_mn=True, out=dw_local, accumulate=r0 > 0)
        if need_dw and dw_local is None:
            _notify(p_w)      # ONE contribution per step however many chunks ran: the count must not depend on the data
        if dh_full is not None:
            o = 0
            for a, b in ranges:
                dh_full[a:b].copy_(dh[o:o + b - a])
                o += b - a
            dh = dh_full
        ctx.train = train
        ctx.hshape = hidden.shape
        ctx.has_dw = dw_local is not None
        if train:
            ctx.save_for_backward(dh, *([dw_local] if dw_local is not None else []))
        loss = acc[0] / max(n_valid, 1) if n_valid is not None else acc[0] * inv_dev[0]
        return loss

    @staticmethod
    @_ranged("lm_head_loss.bwd")
    def backward(ctx, dloss):
        dh = ctx.saved_tensors[0]
        if ctx.has_dw:      # plain-autograd path (no TrainEngine): honour an upstream scale, e.g. (loss / accum).backward()
            return None, (dh * dloss.to(dh.dtype)).view(ctx.hshape), ctx.saved_tensors[1] * dloss.to(dh.dtype)
        # TrainEngine path: dW already sits in main_grad with `loss_scale` folded in (see forward); dloss must be 1
        return None, dh.view(ctx.hshape), None


# ------------------------------------------------------------------------------------------------------------------
# in-LLM SVA site plumbing (cambrian_llama.py:168-207, static branch) and row broadcast
# ------------------------------------------------------------------------------------------------------------------
class SpanSplitFn(torch.autograd.Function):
    """hidden [B,S,H] -> (latent queries [B*q*q, H] copied out of the image span, hidden passed through).

    The pass-through output shares storage with `hidden`; SpanMergeFn later overwrites the latent rows in place, exactly
    like the reference's `hidden_states[:, start:start+600] = ...` assignment.  Backward needs no add: the gradient of
    the overwritten rows is replaced by the gradient that arrived through the latent-query branch."""

    @staticmethod
    def forward(ctx, hidden, start, q_side):
        ctx.start, ctx.q_side = start, q_side
        lat = ops.span_gather(hidden, start, q_side)
        return lat, hidden.detach()

    @staticmethod
    def backward(ctx, d_lat, d_pass):
        d_hidden = d_pass if d_pass.is_contiguous() else d_pass.contiguous()
        ops.span_scatter_(d_hidden, d_lat.contiguous(), ctx.start, ctx.q_side)
        return d_hidden, None, None


class SpanMergeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, passthru, lat_new, start, q_side):
        ctx.start, ctx.q_side = start, q_side
        ops.span_scatter_(passthru, lat_new.contiguous(), start, q_side)
        ctx.mark_dirty(passthru)
        return passthru

    @staticmethod
    def backward(ctx, dout):
        dout = dout.contiguous()
        return dout, ops.span_gather(dout, ctx.start, ctx.q_side), None, None


class ResizeTokenGridFn(torch.autograd.Function):
    """cambrian_arch.py:394-401: a query group whose side differs from the final grid is resized with fp32 bilinear
    interpolation (align_corners=False): [B, q*q, C] -> [B, f*f, C].  Backward = the adjoint gather kernel
    (`cb_bilinear_bwd`, deterministic)."""

    @staticmethod
    def forward(ctx, x, q_side, f_side):
        ctx.sides = (q_side, f_side)
        return ops.bilinear(x.contiguous(), q_side, q_side, f_side, f_side)

    @staticmethod
    def backward(ctx, dy):
        q_side, f_side = ctx.sides
        return ops.bilinear_bwd(dy.contiguous(), q_side, q_side, f_side, f_side), None, None


class ExpandRowsFn(torch.autograd.Function):
    """x [G, C] -> [G*rows, C] (each row repeated `rows` times): the `.expand(...).flatten(0,1)` of the global context
    and of vision_query (cambrian_arch.py:383-385)."""

    @staticmethod
    def forward(ctx, x, rows):
        ctx.rows = rows
        return ops.group_broadcast(x.contiguous(), rows, 1.0)

    @staticmethod
    def backward(ctx, dy):
        G = dy.shape[0] // ctx.rows
        return ops.group_colsum(dy.contiguous(), G, 1.0), None
