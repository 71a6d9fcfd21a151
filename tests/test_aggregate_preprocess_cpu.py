"""The reference, stand-in and model arms of tests/test_aggregate_preprocess_gpu.py on CPU.

The float64 references of tests/aggregate_reference.py are checked against independent fp64 formulations (autograd
through torch.softmax and the mix, and through F.interpolate), the ops_emulation stand-ins of the tower combine and the
bilinear adjoint against the references' bounds, the case tables against the geometries they exist to reach, and the
integer preprocessing model against Pillow at every GPU case geometry.  `ops.resample_coeffs` runs in the built library.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import aggregate_reference as A
import ops_emulation as emu
import vision_kernels_reference as V
from row_kernels_reference import assert_bitwise, check_bf16

DEV = "cpu"
SMS = (132, 114)          # H100 SXM and PCIe
CPU_ROWS = 300            # grid-stride row counts are a GPU matter: the CPU arms run this many rows instead


def _cpu_combine_cases():
    return [(T, ldl, C, N if isinstance(N, int) else CPU_ROWS, regime, cancel)
            for T, ldl, C, N, regime, cancel in A.COMBINE_CASES]


# ======================================================================================================= tower combine
@pytest.mark.parametrize("case", _cpu_combine_cases(), ids=A.combine_case_id)
def test_combine_reference_matches_autograd(case):
    T, ldl, C, N, _, _ = case
    logits, aggs, q_in, dout = A.combine_inputs(case, N, DEV)
    ref = A.combine_ref(logits, aggs, q_in, dout)
    lf = logits.double()[:, :T].requires_grad_()
    af = [a.double().requires_grad_() for a in aggs]
    w = torch.softmax(lf, -1)
    out = q_in.double() + sum(w[:, t:t + 1] * af[t] for t in range(T))
    g = torch.autograd.grad(out, [lf, *af], dout.double())
    close = lambda a, b: torch.testing.assert_close(a, b, rtol=1e-10, atol=1e-10 * float(b.abs().max() + 1e-300))
    close(ref["out"], out.detach())
    close(ref["dl"], g[0])
    for t in range(T):
        close(ref["dagg"][t], g[1 + t])
    assert all(torch.isfinite(x).all() for x in (ref["tol_out"], ref["tol_dl"]))


@pytest.mark.parametrize("case", _cpu_combine_cases(), ids=A.combine_case_id)
def test_combine_stand_in(case):
    T, ldl, C, N, _, _ = case
    logits, aggs, q_in, dout = A.combine_inputs(case, N, DEV)
    ref = A.combine_ref(logits, aggs, q_in, dout)
    check_bf16("out", emu.tower_combine_fwd(logits, aggs, q_in), ref["out"], ref["tol_out"])
    daggs, dl = emu.tower_combine_bwd(logits, aggs, dout)
    for t in range(T):
        check_bf16(f"dagg[{t}]", daggs[t], ref["dagg"][t], ref["tol_dagg"][t])
    check_bf16("dlogits", dl[:, :T], ref["dl"], ref["tol_dl"])
    assert dl.shape == logits.shape
    assert_bitwise("dlogits padding columns are +0", dl[:, T:], torch.zeros(N, ldl - T, dtype=torch.bfloat16))


def test_combine_regimes_do_what_they_say():
    """'cancel' aggregates make dlogits cancel (|w (g - dot)| << w |g|), and at |logits| ~ 100 the weights' bound stays
    small while an unshifted fp32 exp overflows."""
    case = (4, 8, 1024, 64, "large", True)
    logits, aggs, q_in, dout = A.combine_inputs(case, 64, DEV)
    ref = A.combine_ref(logits, aggs, q_in, dout)
    w, dw = A.combine_weights(logits, 4)
    assert float((dw / w.clamp(min=1e-30)).masked_fill(w < 1e-6, 0).max()) < 1e-4
    assert bool(torch.isinf(logits[:, :4].float().exp()).any())
    g = torch.stack([(a.double() * dout.double()).sum(1) for a in aggs], 1)
    assert float((ref["dl"].abs() / (w * g.abs())).median()) < 0.05


# =================================================================================================== bilinear backward
def _cpu_bilinear_cases():
    return [(h, w, th, tw, 1 if B == "grid" else B, min(C, 64)) for h, w, th, tw, B, C in A.BILINEAR_BWD_CASES]


@pytest.mark.parametrize("case", _cpu_bilinear_cases(), ids=A.bilinear_bwd_case_id)
def test_bilinear_bwd_reference(case):
    """against fp64 autograd through F.interpolate (whose fp64 source coordinate is within an fp32 ulp of the kernel's),
    and the exact adjoint identity with the forward reference."""
    h, w, th, tw, B, C = case
    g = V.randn((B, th * tw, C), 2, DEV)
    ref, _ = A.bilinear_bwd_ref(g, h, w, th, tw)
    x = torch.zeros(B, C, h, w, dtype=torch.float64, requires_grad=True)
    y = F.interpolate(x, size=(th, tw), mode="bilinear", align_corners=False)
    (gx,) = torch.autograd.grad(y, x, g.double().reshape(B, th, tw, C).permute(0, 3, 1, 2))
    want = gx.permute(0, 2, 3, 1).reshape(B, h * w, C)
    allow = A.bilinear_bwd_coord_allowance(g, h, w, th, tw) + 1e-12
    assert bool(((ref - want).abs() <= allow).all()), float(((ref - want).abs() / allow).max())
    xs = V.randn((B, h * w, C), 1, DEV)
    yref, _, _ = V.bilinear_ref(xs, h, w, th, tw)
    lhs, rhs = float((yref * g.double()).sum()), float((xs.double() * ref).sum())
    assert abs(lhs - rhs) <= 1e-11 * (float((yref.abs() * g.double().abs()).sum()) + 1e-300)
    if (h, w) == (th, tw):
        assert torch.equal(ref, g.double())


@pytest.mark.parametrize("case", _cpu_bilinear_cases(), ids=A.bilinear_bwd_case_id)
def test_bilinear_bwd_stand_in(case):
    h, w, th, tw, B, C = case
    g = V.randn((B, th * tw, C), 2, DEV)
    ref, tol = A.bilinear_bwd_ref(g, h, w, th, tw)
    got = emu.bilinear_bwd(g, h, w, th, tw)
    assert got.shape == (B, h * w, C) and got.dtype == torch.bfloat16
    check_bf16("stand-in", got, ref, tol + A.bilinear_bwd_coord_allowance(g, h, w, th, tw))


# ===================================================================================================== case tables
@pytest.mark.parametrize("sms", SMS)
def test_case_tables_reach_each_geometry(sms):
    cases = A.COMBINE_CASES
    assert {(T, ldl) for T, ldl, *_ in cases} >= {(T, l) for T in range(1, 9) for l in (T, 8)}
    assert {C for _, _, C, *_ in cases} == set(A.COMBINE_C) and any((C // 8) % 32 for C in A.COMBINE_C)
    assert {r for *_, r, _ in cases} == set(A.COMBINE_REGIMES) and any(c for *_, c in cases)
    rows = [A.combine_rows(N, sms) for _, _, _, N, _, _ in cases]
    cap = A.combine_grid_rows(sms)
    assert min(rows) == 1 and any(cap < n < 2 * cap for n in rows) and any(n > 2 * cap for n in rows)
    assert (8, 8, 264, "2cap+", "large", True) in cases            # grid-stride rows with overflowing unshifted exps

    geo = [(h, w, th, tw) for h, w, th, tw, _, _ in A.BILINEAR_BWD_CASES]
    items = [A.bilinear_bwd_batch(B, h, w, C, sms) * h * w * C // 8 for h, w, _, _, B, C in A.BILINEAR_BWD_CASES]
    assert max(items) > A.bilinear_bwd_cap(sms)
    assert (12, 12, 24, 24) in geo and (2, 2, 96, 96) in geo and (64, 64, 1024, 1024) in geo
    assert any(h == th and w == tw for h, w, th, tw in geo), "identity"
    assert any(h == 1 for h, *_ in geo) and any(w == 1 for _, w, *_ in geo), "1-row and 1-column inputs"
    assert any(h != w for h, w, *_ in geo) and any(th < h for h, _, th, _ in geo), "non-square and down-sampling"

    pre = A.PREPROCESS_CASES
    towers = A.tower_processors()
    assert {t for *_, t in pre} == set(towers)
    assert {towers[t][0] for t in towers} == {336, 378, 384, 518, 1024}
    assert max(A.resample_ksize(max(H, W), towers[t][0]) for H, W, t in pre) >= 49
    assert any(W > H and (W - H) % 2 for H, W, _ in pre) and any(H > W and (H - W) % 2 for H, W, _ in pre), "odd pad offsets"
    assert any(H == 1 for H, *_ in pre) and any(W == 1 for _, W, _ in pre), "1-pixel sides"
    assert any(towers[t][0] > 10 * max(H, W) for H, W, t in pre), "a large up-scale"


def test_kernel_constants_match_the_reference_module():
    """the thresholds the reference module restates, against the sources they come from."""
    import pathlib
    src = (pathlib.Path(A.__file__).resolve().parents[1] / "cambrian_b200" / "csrc" / "aggregate.cu").read_text()
    assert "device_sm_count() * 16" in src and "blockIdx.x * 8 + (threadIdx.x >> 5)" in src
    assert "device_sm_count() * 8" in src and "(total + 255) / 256" in src
    from cambrian_b200 import ops
    for S, R in [(6000, 336), (4000, 336), (1, 384), (336, 336), (16, 1024)]:
        assert ops.resample_coeffs(S, R)[1].shape[1] == A.resample_ksize(S, R)


# ====================================================================================================== preprocessing
@pytest.mark.parametrize("case", A.PREPROCESS_CASES, ids=A.preprocess_case_id)
def test_preprocess_model_matches_pillow(case):
    H, W, tower = case
    R, mean, std = A.tower_processors()[tower]
    pad = tuple(int(x * 255) for x in mean)
    arr = A.preprocess_image_input(H, W)
    want = A.pillow_resize(arr, R, pad)
    got = A.resize_model(arr, R, pad)
    assert got.shape == want.shape == (R, R, 3)
    assert np.array_equal(got, want), f"{int((got != want).sum())} bytes differ from Pillow"
    # the normalisation candidates are one rounding of the fp64 formula
    ref = (torch.from_numpy(np.array(want)).permute(2, 0, 1).double() / 255 - torch.tensor(mean).double().view(3, 1, 1)) / \
        torch.tensor(std).double().view(3, 1, 1)
    for cand in A.normalise_candidates(want, mean, std):
        check_bf16("normalised", cand, ref, 4 * 2.0 ** -24 * (ref.abs() + 1 / 0.2))
