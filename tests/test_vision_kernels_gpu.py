"""The SVA window attention, the vision-tower kernels, the token gathers and splices and the bf16 decode GEMV against float64
references, and the CPU stand-ins of tests/ops_emulation.py against the same references.

Every case runs three arms on the same seeded inputs: the `cambrian_b200.ops` kernel, the float64 reference of
tests/vision_kernels_reference.py (computed on the device; the module also derives each error bound), and, where one
exists, the ops_emulation stand-in on CPU copies.  Arithmetic outputs are held to the fp64 bound, copies and gathers
bitwise; memory the op must not write is sentinel-filled and compared bitwise.  Each check prints its worst error-to-bound
ratio.  tests/test_vision_kernels_cpu.py runs the reference and stand-in arms of the same case tables without a GPU.
"""
from __future__ import annotations

import pytest
import torch

import ops_emulation as emu
import vision_kernels_reference as R
from row_kernels_reference import assert_bitwise, check_abs, check_bf16, sentinel_like, sm_count

pytestmark = pytest.mark.gpu

DEV = "cuda"


@pytest.fixture(scope="module")
def ops():
    from cambrian_b200 import ops as o
    return o


def _cpu(*ts):
    return [None if t is None else t.detach().cpu() for t in ts]


def _cpu_list(ts):
    return None if ts is None else [None if t is None else t.cpu() for t in ts]


def _slabs(shapes, guard=8 * 1024):
    """one sentinel-filled buffer holding a contiguous slab per shape, with sentinel guards between and after them."""
    sizes = [int(torch.Size(s).numel()) for s in shapes]
    buf = sentinel_like((sum(sizes) + guard * (len(sizes) + 1),), torch.bfloat16, DEV)
    slabs, guards, off = [], [buf[:guard]], guard
    for s, n in zip(shapes, sizes):
        slabs.append(buf[off:off + n].view(s))
        guards.append(buf[off + n:off + n + guard])
        off += n + guard
    return buf, slabs, guards


# ================================================================================================================== SVA
@pytest.mark.parametrize("case", R.SVA_CASES, ids=R.sva_case_id)
def test_sva_window_attention(ops, case):
    q_side, B, rs, mode, std = case
    q, ks, vs, masks, dout = R.sva_inputs(case, DEV)
    T = len(rs)
    print(f"\n  sva q_side={q_side} B={B} rs={rs} masks={mode} std={std} queries={q.shape[0]}")
    ref = R.sva_ref(q, ks, vs, masks, rs, B, q_side, dout)

    # ---- kernel, natural layout; dK / dV into slabs of one sentinel-filled stacked buffer
    o, lse = ops.sva_window_attn_fwd(q, ks, vs, masks, rs, B, q_side)
    buf, slabs, guards = _slabs([k.shape for k in ks] + [v.shape for v in vs])
    dq, dks, dvs = ops.sva_window_attn_bwd(q, o, dout, lse, ks, vs, masks, rs, B, q_side, dks=slabs[:T], dvs=slabs[T:])
    torch.cuda.synchronize()

    def checks(arm, o_, lse_, dq_, dks_, dvs_):
        check_bf16(f"{arm} O", o_, ref["o"], ref["tol_o"])
        R.check_lse(f"{arm} LSE", lse_, ref, check_abs)
        check_bf16(f"{arm} dQ", dq_, ref["dq"], ref["tol_dq"])
        for t in range(T):
            check_bf16(f"{arm} dK[{t}] (r={rs[t]})", dks_[t], ref["dk"][t], ref["tol_dk"][t])
            check_bf16(f"{arm} dV[{t}] (r={rs[t]})", dvs_[t], ref["dv"][t], ref["tol_dv"][t])

    checks("kernel", o, lse, dq, dks, dvs)
    for i, g in enumerate(guards):
        assert_bitwise(f"dK/dV guard {i}", g, sentinel_like(g.shape, torch.bfloat16, DEV))

    # ---- a second run, into fresh destinations, gives the same bits
    o2, lse2 = ops.sva_window_attn_fwd(q, ks, vs, masks, rs, B, q_side)
    dq2, dks2, dvs2 = ops.sva_window_attn_bwd(q, o2, dout, lse2, ks, vs, masks, rs, B, q_side)
    assert_bitwise("rerun O", o2, o)
    assert_bitwise("rerun LSE", lse2, lse)
    assert_bitwise("rerun dQ", dq2, dq)
    for t in range(T):
        assert_bitwise(f"rerun dK[{t}]", dks2[t], dks[t])
        assert_bitwise(f"rerun dV[{t}]", dvs2[t], dvs[t])

    # ---- windowed layout: K / V gathered by ops.window_gather; identical bits
    kw = [ops.window_gather(k, q_side) for k in ks]
    vw = [ops.window_gather(v, q_side) for v in vs]
    ow, lsew = ops.sva_window_attn_fwd(q, kw, vw, masks, rs, B, q_side, windowed=True)
    _, wslabs, wguards = _slabs([k.shape for k in kw] + [v.shape for v in vw])
    dqw, dkw, dvw = ops.sva_window_attn_bwd(q, ow, dout, lsew, kw, vw, masks, rs, B, q_side, windowed=True,
                                            dks=wslabs[:T], dvs=wslabs[T:])
    assert_bitwise("windowed O", ow, o)
    assert_bitwise("windowed LSE", lsew, lse)
    assert_bitwise("windowed dQ", dqw, dq)
    for t in range(T):
        assert_bitwise(f"windowed dK[{t}]", dkw[t], ops.window_gather(dks[t], q_side))
        assert_bitwise(f"windowed dV[{t}]", dvw[t], ops.window_gather(dvs[t], q_side))
    for i, g in enumerate(wguards):
        assert_bitwise(f"windowed guard {i}", g, sentinel_like(g.shape, torch.bfloat16, DEV))

    # ---- stand-in (CPU); its backward recomputes O in fp32, within the same bounds
    qc, doc = _cpu(q, dout)
    kc, vc, mc = _cpu_list(ks), _cpu_list(vs), _cpu_list(masks)
    oe, lsee = emu.sva_window_attn_fwd(qc, kc, vc, mc, rs, B, q_side)
    dqe, dke, dve = emu.sva_window_attn_bwd(qc, oe, doc, lsee, kc, vc, mc, rs, B, q_side)
    checks("stand-in", oe, lsee, dqe, dke, dve)


# ============================================================================================================== dwconv7
def _dwconv7_case(ops, B, H, W, C):
    cfg = R.dwconv7_cfg(B, H, W, C, sm_count())
    print(f"\n  dwconv7 B={B} H={H} W={W} C={C} {cfg}")
    x, w, b = R.dwconv7_inputs(B, H, W, C, DEV)
    y = ops.dwconv7(x, w, b)
    torch.cuda.synchronize()
    ref, tol = R.dwconv7_ref(x, w, b)
    check_bf16("kernel y", y, ref, tol)
    assert_bitwise("rerun", ops.dwconv7(x, w, b), y)
    return cfg


@pytest.mark.parametrize("B,H,W,C", R.DW_EDGE_CASES + R.DW_STAGE_CASES)
def test_dwconv7(ops, B, H, W, C):
    _dwconv7_case(ops, B, H, W, C)


@pytest.mark.parametrize("B,W,C", R.DW_UNEVEN_CASES)
def test_dwconv7_uneven_ysplit(ops, B, W, C):
    H = R.dwconv7_uneven_height(B, W, C, sm_count())
    cfg = _dwconv7_case(ops, B, H, W, C)
    assert H % 8 and cfg["ysplit"] > 1 and cfg["steps"] % cfg["ysplit"] != 0
    assert cfg["per"] * (cfg["ysplit"] - 1) >= cfg["steps"], "the last y-part should be empty"


# ============================================================================================================= bilinear
def _bilinear_checks(arm, got, ref, tol, coord=None):
    check_bf16(f"{arm} y", got, ref, tol if coord is None else tol + coord)


@pytest.mark.parametrize("cls", [False, True])
@pytest.mark.parametrize("h,w,th,tw", R.BILINEAR_CASES)
def test_bilinear(ops, h, w, th, tw, cls):
    B, C = 2, 64
    full = R.randn((B, h * w + int(cls) + 3, C), 1, DEV)          # spare rows after the grid: in_bs != h * w * C
    x = full[:, int(cls):]
    print(f"\n  bilinear {h}x{w} -> {th}x{tw} cls-view={cls}")
    y = ops.bilinear(x, h, w, th, tw, in_bs=full.stride(0))
    torch.cuda.synchronize()
    ref, tol, coord = R.bilinear_ref(x, h, w, th, tw)
    if (h, w) == (th, tw):
        assert_bitwise("identity", y, x[:, :h * w])
    _bilinear_checks("kernel", y, ref, tol)
    ye = emu.bilinear(full.cpu()[:, int(cls):], h, w, th, tw, in_bs=full.stride(0))
    _bilinear_checks("stand-in", ye, ref, tol, coord)


def test_bilinear_convnext_concat(ops):
    """each ConvNeXt-XXL@1024 stage resized to 96 x 96 into its column slice of one sentinel-filled [B, 96^2, 5760]."""
    B, t = 1, R.CONVNEXT_OUT
    Ctot = sum(c for _, c in R.CONVNEXT_STAGES)
    out = sentinel_like((B, t * t, Ctot), torch.bfloat16, DEV)
    out_e = out.cpu().clone()
    col = 0
    for i, (side, C) in enumerate(R.CONVNEXT_STAGES):
        f = R.randn((B, side * side, C), 10 + i, DEV)
        print(f"\n  bilinear stage {side}^2 x {C} -> {t}^2 into columns [{col}, {col + C})")
        ops.bilinear(f, side, side, t, t, out=out, out_ld=Ctot, out_col0=col)
        emu.bilinear(f.cpu(), side, side, t, t, out=out_e, out_ld=Ctot, out_col0=col)
        torch.cuda.synchronize()
        ref, tol, coord = R.bilinear_ref(f, side, side, t, t)
        _bilinear_checks("kernel", out[..., col:col + C], ref, tol)
        _bilinear_checks("stand-in", out_e[..., col:col + C], ref, tol, coord)
        col += C
        rest = out[..., col:]
        assert_bitwise("columns not yet written", rest, sentinel_like(rest.shape, torch.bfloat16, DEV))
        assert_bitwise("stand-in columns not yet written", out_e[..., col:], sentinel_like(rest.shape, torch.bfloat16, "cpu"))


# ============================================================================================================= patchify
@pytest.mark.parametrize("R_,p", R.PATCHIFY_NCHW_CASES)
def test_patchify_nchw(ops, R_, p):
    B = 2 if R_ < 1024 else 1
    img = R.randn((B, 3, R_, R_), 1, DEV)
    got = ops.patchify_nchw(img, p)
    want = R.patchify_nchw_ref(img, p)
    print(f"\n  patchify_nchw R={R_} p={p} -> {tuple(got.shape)}")
    assert got.shape == want.shape
    assert_bitwise("patches (pad columns zero)", got, want)


@pytest.mark.parametrize("B,H,W,C", R.PATCHIFY_NHWC_CASES)
def test_patchify_nhwc(ops, B, H, W, C):
    x = R.randn((B, H, W, C), 1, DEV)
    got = ops.patchify_nhwc(x, 2)
    print(f"\n  patchify_nhwc {B}x{H}x{W}x{C} p=2")
    assert_bitwise("patches", got, R.patchify_nhwc_ref(x, 2))


@pytest.mark.parametrize("N,cls", R.ADD_POS_CASES)
def test_add_pos_tokens(ops, N, cls):
    B, C = 2, 1024
    patch = R.randn((B, N, C), 1, DEV)
    c = R.randn((C,), 2, DEV) if cls else None
    pos = R.randn((N + int(cls), C), 3, DEV)
    print(f"\n  add_pos_tokens N={N} cls={cls}")
    assert_bitwise("tokens", ops.add_pos_tokens(patch, c, pos), R.add_pos_tokens_ref(patch, c, pos))


# ================================================================================================ gathers and splices
@pytest.mark.parametrize("ci", range(5))
def test_window_gather(ops, ci):
    B, q, r, C = 2, 6, 3, 64
    crop = R.window_gather_crops(q)[ci]
    feat = R.randn((B, (q * r) ** 2, C), 1, DEV)
    print(f"\n  window_gather q={q} r={r} crop={crop}")
    want = R.window_gather_ref(feat, q, crop)
    assert_bitwise("kernel", ops.window_gather(feat, q, crop), want)
    assert_bitwise("stand-in", emu.window_gather(feat.cpu(), q, crop), want)


@pytest.mark.parametrize("B,S,start,q_h,q_w", R.SPAN_CASES)
def test_span_gather_scatter_hw(ops, B, S, start, q_h, q_w):
    H = 64
    hidden = R.randn((B, S, H), 1, DEV)
    lat = R.randn((B * q_h * q_w, H), 2, DEV)
    idx = torch.tensor(R.span_rows(B, S, start, q_h, q_w), device=DEV)
    print(f"\n  span_gather_hw / span_scatter_hw_ B={B} S={S} start={start} {q_h}x{q_w} (ends at {start + q_h * (q_w + 1)})")
    want_g = hidden.reshape(B * S, H)[idx]
    assert_bitwise("gather kernel", ops.span_gather_hw(hidden, start, q_h, q_w), want_g)
    assert_bitwise("gather stand-in", emu.span_gather_hw(hidden.cpu(), start, q_h, q_w), want_g)
    want_s = hidden.clone()
    want_s.view(B * S, H)[idx] = lat
    h_k = ops.span_scatter_hw_(hidden.clone(), lat, start, q_h, q_w)
    assert_bitwise("scatter kernel (newline rows and the rest untouched)", h_k, want_s)
    assert_bitwise("scatter stand-in", emu.span_scatter_hw_(hidden.cpu().clone(), lat.cpu(), start, q_h, q_w), want_s)


@pytest.mark.parametrize("with_img", [True, False])
def test_embed_splice(ops, with_img):
    q_side = 3
    ids, st, embed, img, nl = R.embed_splice_inputs(DEV, q_side)
    img = img if with_img else None
    print(f"\n  embed_splice img={with_img} img_start={st.tolist()}")
    want = R.embed_splice_ref(ids, st, embed, img, nl, q_side)
    assert_bitwise("kernel", ops.embed_splice(ids, st, embed, img, nl, q_side), want)
    assert_bitwise("stand-in", emu.embed_splice(*_cpu(ids, st, embed, img, nl), q_side), want)


@pytest.mark.parametrize("with_img", [True, False])
def test_embed_splice_ragged(ops, with_img):
    batch, max_len, V, H, n_img = 3, 7, 40, 64, 5
    embed = R.randn((V, H), 1, DEV)
    img = R.randn((n_img, H), 2, DEV) if with_img else None
    nl = R.randn((H,), 3, DEV)
    src = R.ragged_src(batch * max_len, V, n_img, DEV, with_img)
    print(f"\n  embed_splice_ragged img={with_img} src={src.tolist()}")
    want = R.embed_splice_ragged_ref(embed, img, nl, src, batch, max_len)
    assert_bitwise("kernel", ops.embed_splice_ragged(embed, img, nl, src, batch, max_len), want)
    assert_bitwise("stand-in", emu.embed_splice_ragged(*_cpu(embed, img, nl, src), batch, max_len), want)


# ================================================================================================================= GEMV
@pytest.mark.parametrize("M", range(1, 9))
def test_gemv_shapes(ops, M):
    print(f"\n  gemv M={M}")
    for K in R.GEMV_K:
        for N in R.GEMV_N:
            x, w, _, _ = R.gemv_inputs(M, N, K, DEV, seed=M * 100 + K + N)
            ref, tol = R.gemv_ref(x, w)
            y = ops.gemv(x, w)
            check_bf16(f"M={M} K={K} N={N}", y, ref, tol)
            if not (M >= 6 and N >= 16384):
                assert_bitwise("  ops.gemm == ops.gemv", ops.gemm(x, w), y)


@pytest.mark.parametrize("bias,residual,fp32", R.GEMV_EPILOGUES)
def test_gemv_epilogues(ops, bias, residual, fp32):
    print(f"\n  gemv bias={bias} residual={residual} fp32 out={fp32}")
    for M in range(1, 9):
        K = R.GEMV_K[M % len(R.GEMV_K)]
        N = R.GEMV_N[(M + 2) % len(R.GEMV_N)]
        x, w, b, r = R.gemv_inputs(M, N, K, DEV, seed=M, bias=bias, residual=residual)
        ref, tol = R.gemv_ref(x, w, b, r)
        dt = torch.float32 if fp32 else torch.bfloat16
        y = ops.gemv(x, w, bias=b, residual=r, out_dtype=dt)
        (check_abs if fp32 else check_bf16)(f"M={M} K={K} N={N}", y, ref, tol)
        assert_bitwise("  ops.gemm == ops.gemv", ops.gemm(x, w, bias=b, residual=r, out_dtype=dt), y)


@pytest.mark.parametrize("fp32", [False, True])
def test_gemv_strided_and_inplace_residual(ops, fp32):
    """x with row stride K + 8, out a row-strided view of a sentinel buffer, and residual aliasing out."""
    dt = torch.float32 if fp32 else torch.bfloat16
    for M, K, N in [(1, 1032, 17), (4, 2056, 520), (6, 8, 15), (7, 14336, 16), (8, 2048, 4104)]:
        xb = R.randn((M, K + 8), M, DEV)
        x = xb[:, :K]
        _, w, b, r = R.gemv_inputs(M, N, K, DEV, seed=M + 7, bias=True, residual=True)
        ob = sentinel_like((M, N + 24), dt, DEV)
        out = ob[:, :N]
        ref, tol = R.gemv_ref(x, w, b)
        ops.gemv(x, w, bias=b, out=out)
        print(f"\n  gemv strided M={M} K={K} N={N} ldx={x.stride(0)} ldy={out.stride(0)} fp32={fp32}")
        (check_abs if fp32 else check_bf16)("strided", out, ref, tol)
        assert_bitwise("columns past N", ob[:, N:], sentinel_like((M, 24), dt, DEV))
        if fp32:   # the residual operand is bf16: alias a bf16 out only
            continue
        out.copy_(r)
        ref, tol = R.gemv_ref(x, w, b, r)
        ops.gemv(x, w, bias=b, residual=out, out=out)
        check_bf16("residual is out", out, ref, tol)
        assert_bitwise("columns past N", ob[:, N:], sentinel_like((M, 24), dt, DEV))


def test_gemv_routing_threshold(ops):
    """ops.gemm sends M <= 8 to the GEMV except M >= 6 with N >= 16384, which keeps the tensor-core tile: both sides."""
    K = 2048
    for M, N in [(5, 16384), (6, 16376), (8, 16376)]:
        x, w, _, _ = R.gemv_inputs(M, N, K, DEV, seed=M)
        y = ops.gemm(x, w)
        ref, tol = R.gemv_ref(x, w)
        print(f"\n  gemm M={M} N={N} (GEMV side)")
        check_bf16("gemv", y, ref, tol)
        assert_bitwise("ops.gemm == ops.gemv", y, ops.gemv(x, w))
    for M in (6, 7, 8):
        x, w, b, r = R.gemv_inputs(M, 16384, K, DEV, seed=M, bias=True, residual=True)
        print(f"\n  gemm M={M} N=16384 (tile side)")
        ref, tol = R.gemv_ref(x, w, tile=True)
        check_bf16("tile", ops.gemm(x, w), ref, tol)
        ref, tol = R.gemv_ref(x, w, b, r, tile=True)
        check_bf16("tile + bias + residual", ops.gemm(x, w, bias=b, residual=r), ref, tol)
        ref, tol = R.gemv_ref(x, w, tile=True)
        check_abs("tile fp32 out", ops.gemm(x, w, out_dtype=torch.float32), ref, tol)
