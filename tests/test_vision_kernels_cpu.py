"""The reference and stand-in arms of tests/test_vision_kernels_gpu.py on CPU: the ops_emulation stand-ins of the SVA window
attention, bilinear resize, window gather, span gather / scatter and embedding splices against the float64 references of
tests/vision_kernels_reference.py, on the same case tables (the smaller shapes where CPU float64 is slow).  The ops with no
stand-in (dwconv7, patchify, add_pos_tokens, GEMV) have their references checked against an independent torch
formulation, so the GPU file holds its kernels to a reference that is itself pinned here.
"""
from __future__ import annotations

import pytest
import torch
import torch.nn.functional as F

import ops_emulation as emu
import vision_kernels_reference as R
from row_kernels_reference import assert_bitwise, check_abs, check_bf16, sentinel_like

DEV = "cpu"

SVA_CPU_CASES = [c for c in R.SVA_CASES if c[0] * c[0] * c[1] <= 144]


# ================================================================================================================== SVA
@pytest.mark.parametrize("case", SVA_CPU_CASES, ids=R.sva_case_id)
def test_sva_stand_in(case):
    q_side, B, rs, mode, std = case
    q, ks, vs, masks, dout = R.sva_inputs(case, DEV)
    T = len(rs)
    print(f"\n  sva q_side={q_side} B={B} rs={rs} masks={mode} std={std}")
    ref = R.sva_ref(q, ks, vs, masks, rs, B, q_side, dout)
    o, lse = emu.sva_window_attn_fwd(q, ks, vs, masks, rs, B, q_side)
    dks = [sentinel_like(k.shape, torch.bfloat16, DEV) for k in ks]
    dvs = [sentinel_like(v.shape, torch.bfloat16, DEV) for v in vs]
    dq, dks, dvs = emu.sva_window_attn_bwd(q, o, dout, lse, ks, vs, masks, rs, B, q_side, dks=dks, dvs=dvs)
    check_bf16("O", o, ref["o"], ref["tol_o"])
    R.check_lse("LSE", lse, ref, check_abs)
    check_bf16("dQ", dq, ref["dq"], ref["tol_dq"])
    for t in range(T):
        check_bf16(f"dK[{t}]", dks[t], ref["dk"][t], ref["tol_dk"][t])
        check_bf16(f"dV[{t}]", dvs[t], ref["dv"][t], ref["tol_dv"][t])
    # the window-rearranged layout gives the same bits
    kw = [emu.window_gather(k, q_side) for k in ks]
    vw = [emu.window_gather(v, q_side) for v in vs]
    ow, lsew = emu.sva_window_attn_fwd(q, kw, vw, masks, rs, B, q_side, windowed=True)
    dqw, dkw, dvw = emu.sva_window_attn_bwd(q, ow, dout, lsew, kw, vw, masks, rs, B, q_side, windowed=True)
    assert_bitwise("windowed O", ow, o)
    assert_bitwise("windowed dQ", dqw, dq)
    for t in range(T):
        assert_bitwise(f"windowed dK[{t}]", dkw[t], emu.window_gather(dks[t], q_side))
        assert_bitwise(f"windowed dV[{t}]", dvw[t], emu.window_gather(dvs[t], q_side))


def test_sva_fully_masked_query_is_zero():
    """a query with every key masked: out 0, LSE +inf, and zero gradients (not NaN)."""
    case = (2, 1, [1, 2], "all_masked", 1.0)
    q, ks, vs, _, dout = R.sva_inputs(case, DEV)
    masks = [torch.zeros(4, 1, dtype=torch.bool), torch.ones(4, 4, dtype=torch.bool)]
    masks[1][2] = False
    o, lse = emu.sva_window_attn_fwd(q, ks, vs, masks, [1, 2], 1, 2)
    dq, dk, dv = emu.sva_window_attn_bwd(q, o, dout, lse, ks, vs, masks, [1, 2], 1, 2)
    assert torch.equal(o[2], torch.zeros_like(o[2])) and torch.isinf(lse[2]).all() and (lse[2] > 0).all()
    assert torch.isfinite(lse[[0, 1, 3]]).all() and torch.isfinite(o.float()).all()
    assert torch.equal(dq[2], torch.zeros_like(dq[2]))
    assert all(torch.isfinite(g.float()).all() for g in [dq, *dk, *dv])


# ============================================================================================================= bilinear
@pytest.mark.parametrize("cls", [False, True])
@pytest.mark.parametrize("h,w,th,tw", R.BILINEAR_CASES)
def test_bilinear_stand_in(h, w, th, tw, cls):
    B, C = 2, 16
    full = R.randn((B, h * w + int(cls) + 3, C), 1, DEV)
    x = full[:, int(cls):]
    ref, tol, coord = R.bilinear_ref(x, h, w, th, tw)
    y = emu.bilinear(x, h, w, th, tw, in_bs=full.stride(0))
    check_bf16("stand-in", y, ref, tol + coord)
    if (h, w) == (th, tw):
        assert_bitwise("identity", y, x[:, :h * w])


def test_bilinear_stand_in_convnext_concat():
    """the ConvNeXt stages (channels / 48) resized into column slices of one sentinel-filled buffer."""
    B, t = 1, R.CONVNEXT_OUT
    stages = [(side, C // 48) for side, C in R.CONVNEXT_STAGES]
    Ctot = sum(c for _, c in stages)
    out = sentinel_like((B, t * t, Ctot), torch.bfloat16, DEV)
    col = 0
    for i, (side, C) in enumerate(stages):
        f = R.randn((B, side * side, C), 10 + i, DEV)
        emu.bilinear(f, side, side, t, t, out=out, out_ld=Ctot, out_col0=col)
        ref, tol, coord = R.bilinear_ref(f, side, side, t, t)
        check_bf16(f"stage {side}", out[..., col:col + C], ref, tol + coord)
        col += C
        assert_bitwise("columns not yet written", out[..., col:], sentinel_like(out[..., col:].shape, torch.bfloat16, DEV))


# ============================================================================================== gathers and splices
@pytest.mark.parametrize("ci", range(5))
def test_window_gather_stand_in(ci):
    B, q, r, C = 2, 6, 3, 16
    crop = R.window_gather_crops(q)[ci]
    feat = R.randn((B, (q * r) ** 2, C), 1, DEV)
    assert_bitwise("stand-in", emu.window_gather(feat, q, crop), R.window_gather_ref(feat, q, crop))


@pytest.mark.parametrize("B,S,start,q_h,q_w", R.SPAN_CASES)
def test_span_gather_scatter_hw_stand_in(B, S, start, q_h, q_w):
    H = 16
    hidden = R.randn((B, S, H), 1, DEV)
    lat = R.randn((B * q_h * q_w, H), 2, DEV)
    idx = torch.tensor(R.span_rows(B, S, start, q_h, q_w))
    assert_bitwise("gather", emu.span_gather_hw(hidden, start, q_h, q_w), hidden.reshape(B * S, H)[idx])
    want = hidden.clone()
    want.view(B * S, H)[idx] = lat
    assert_bitwise("scatter", emu.span_scatter_hw_(hidden.clone(), lat, start, q_h, q_w), want)


@pytest.mark.parametrize("with_img", [True, False])
def test_embed_splice_stand_in(with_img):
    ids, st, embed, img, nl = R.embed_splice_inputs(DEV)
    img = img if with_img else None
    assert_bitwise("stand-in", emu.embed_splice(ids, st, embed, img, nl, 3), R.embed_splice_ref(ids, st, embed, img, nl, 3))


@pytest.mark.parametrize("with_img", [True, False])
def test_embed_splice_ragged_stand_in(with_img):
    batch, max_len, V, H, n_img = 3, 7, 40, 16, 5
    embed = R.randn((V, H), 1, DEV)
    img = R.randn((n_img, H), 2, DEV) if with_img else None
    nl = R.randn((H,), 3, DEV)
    src = R.ragged_src(batch * max_len, V, n_img, DEV, with_img)
    assert {0, V - 1, -1, R.INT32_MIN} <= set(src.tolist())
    want = R.embed_splice_ragged_ref(embed, img, nl, src, batch, max_len)
    assert_bitwise("stand-in", emu.embed_splice_ragged(embed, img, nl, src, batch, max_len), want)


# ================================================================================= references of the ops with no stand-in
@pytest.mark.parametrize("B,H,W,C", R.DW_EDGE_CASES)
def test_dwconv7_reference(B, H, W, C):
    x, w, b = R.dwconv7_inputs(B, H, W, C, DEV)
    ref, tol = R.dwconv7_ref(x, w, b)
    conv = F.conv2d(x.double().permute(0, 3, 1, 2), w.double().permute(2, 0, 1)[:, None], b.double(), padding=3, groups=C)
    torch.testing.assert_close(ref, conv.permute(0, 2, 3, 1), rtol=1e-12, atol=1e-12)
    # an fp32 evaluation in the kernel's order (bias first, taps by row then column) lands within the bound
    xp = F.pad(x.float(), (0, 0, 3, 3, 3, 3))
    y = b.float().expand(B, H, W, C).clone()
    for dy in range(7):
        for dx in range(7):
            y = torch.addcmul(y, xp[:, dy:dy + H, dx:dx + W], w.float()[dy, dx])
    check_bf16("fp32 in kernel order", y.to(torch.bfloat16), ref, tol)


def test_dwconv7_cfg():
    """the launch arithmetic of dwconv7_launch, and the shape dwconv7_uneven_height derives from it (132 SMs here)."""
    assert R.dwconv7_cfg(1, 256, 256, 384, 132) == dict(nchunk=3, strips=32, steps=32, ysplit=17, per=2)
    for B, W, C in R.DW_UNEVEN_CASES:
        H = R.dwconv7_uneven_height(B, W, C, 132)
        cfg = R.dwconv7_cfg(B, H, W, C, 132)
        assert H % 8 and 1 < cfg["ysplit"] < cfg["steps"] and cfg["steps"] % cfg["ysplit"]
        assert cfg["per"] * (cfg["ysplit"] - 1) >= cfg["steps"]


@pytest.mark.parametrize("R_,p", R.PATCHIFY_NCHW_CASES)
def test_patchify_nchw_reference(R_, p):
    img = R.randn((1, 3, R_, R_), 1, DEV)
    ref = R.patchify_nchw_ref(img, p)
    K = 3 * p * p
    un = F.unfold(img.float(), kernel_size=p, stride=p)[0].T.to(torch.bfloat16)
    assert ref.shape == (un.shape[0], -(-K // 8) * 8) and un.shape[0] == (R_ // p) ** 2
    assert_bitwise("patches", ref[:, :K], un)
    assert not ref[:, K:].view(torch.int16).any(), "pad columns must be +0.0"


@pytest.mark.parametrize("B,H,W,C", R.PATCHIFY_NHWC_CASES)
def test_patchify_nhwc_reference(B, H, W, C):
    x = R.randn((B, H, W, C), 1, DEV)
    un = F.unfold(x.float().permute(0, 3, 1, 2), kernel_size=2, stride=2)         # [B, (c, py, px), L]
    L = un.shape[-1]
    un = un.reshape(B, C, 2, 2, L).permute(0, 4, 2, 3, 1).reshape(B * L, 4 * C).to(torch.bfloat16)
    assert_bitwise("patches", R.patchify_nhwc_ref(x, 2), un)


@pytest.mark.parametrize("N,cls", R.ADD_POS_CASES)
def test_add_pos_tokens_reference(N, cls):
    B, C = 2, 16
    patch = R.randn((B, N, C), 1, DEV)
    c = R.randn((C,), 2, DEV) if cls else None
    pos = R.randn((N + int(cls), C), 3, DEV)
    ref = R.add_pos_tokens_ref(patch, c, pos)
    assert ref.shape == (B, N + int(cls), C)
    if cls:
        assert_bitwise("CLS row", ref[:, 0], (c.float() + pos[0].float()).to(torch.bfloat16).expand(B, C))
    assert_bitwise("patch rows", ref[:, int(cls):], (patch.float() + pos[int(cls):].float()).to(torch.bfloat16))


@pytest.mark.parametrize("M", range(1, 9))
def test_gemv_reference(M):
    """the fp64 reference against an fp64 einsum, and an fp32 sequential-per-lane evaluation within the bound."""
    for K in (8, 1032, 2056):
        for N in (1, 17, 520):
            x, w, b, r = R.gemv_inputs(M, N, K, DEV, seed=M, bias=True, residual=True)
            ref, tol = R.gemv_ref(x, w, b, r)
            want = torch.einsum("mk,nk->mn", x.double(), w.double()) + b.double() + r.double()
            torch.testing.assert_close(ref, want, rtol=1e-12, atol=1e-12)
            y = (x.float() @ w.float().T + b.float() + r.float()).to(torch.bfloat16)
            check_bf16(f"fp32 M={M} K={K} N={N}", y, ref, tol)
