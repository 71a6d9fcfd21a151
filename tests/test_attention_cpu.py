"""The flash-attention references of tests/attention_reference.py and the CPU stand-ins of tests/ops_emulation.py, without a
GPU: the fp64 references against an independent fp64 torch formulation (softmax and autograd) on rows that see a key, the
stand-ins against the references' bounds on the small cases of the GPU tables, the case tables' coverage, and the key-mask
operand check of `ops`."""
from __future__ import annotations

import math

import pytest
import torch

import attention_reference as R
import ops_emulation as emu
from row_kernels_reference import check_abs, check_bf16

SMALL = [c for c in R.FWD_CASES + R.BWD_CASES if c.Sq * c.Skv <= 130 * 300 and c.B * c.nh <= 16]


def test_case_tables_reach_every_geometry():
    f, b = R.FWD_CASES, R.BWD_CASES
    assert {c.hd for c in f} == {32, 64, 72, 80, 88, 96, 104, 128}
    assert {c.hd for c in b} == {64, 96, 128}
    lens = {1, 63, 64, 65, 127, 128, 129, 300, 577, 729, 730, 2048}
    assert lens <= {c.Sq for c in f} | {c.Skv for c in f}
    assert {(1, 4096), (5, 700), (130, 900)} <= {(c.Sq, c.Skv) for c in f if c.causal}
    assert any(c.causal and c.Sq > c.Skv for c in f) and any(c.causal and c.Sq > c.Skv for c in b)
    assert {1, 2, 3, 4, 7, 8} <= {c.nh // c.nkv for c in f}
    assert {1, 3, 4, 8} <= {c.nh // c.nkv for c in b}
    wins = {c.window for c in f if c.window}
    assert {1, 64, 127, 128, 129, 257} <= wins and any(c.window == c.Skv - 1 for c in f)
    assert any(c.window and c.mask != "none" and c.Sq < c.Skv for c in f)
    masks = {"none", "all_true", "left", "right", "hole", "rand20", "row_false"}
    assert masks <= {c.mask for c in f} and masks <= {c.mask for c in b}
    assert any(c.mask not in ("none", "decode") and c.Skv % 2 for c in f)
    assert {"contig", "packed", "padded_batch", "out_slice"} <= {c.layout for c in f}
    assert any(c.mask == "decode" and c.Sq == 1 and not c.causal for c in f)
    assert any(c.scale for c in f) and any(c.scale for c in b)
    assert {"std1", "std3", "ramp", "first"} <= {c.regime for c in f}
    assert {65, 127, 129, 191, 300, 1000} <= {c.Sq for c in b} | {c.Skv for c in b}
    assert any(c.Sq < c.Skv for c in b) and {True, False} == {c.causal for c in b}
    assert any(c.window and c.Sq < c.Skv for c in b)         # key tiles no query's window reaches: n_iter = 0
    assert any(c.hd == 96 and (c.B * c.Sq * c.nh) % 2 for c in b)
    assert any(c.hd == 64 and (c.B * c.Sq * c.nh) % 4 for c in b)
    assert any(c.layout == "packed" for c in b)


def _independent(q, k, v, do, causal, kmask, scale, window):
    """fp64 softmax attention and its autograd gradients; rows that see no key are excluded (their dO is zero)."""
    B, Sq, nh, hd = q.shape
    G = nh // k.shape[2]
    scale = hd ** -0.5 if scale is None else scale
    Q, K, V = (t.double().transpose(1, 2).requires_grad_() for t in (q, k, v))
    vis = R.visible(Sq, Skv := k.shape[1], causal, window, kmask, "cpu")[:, None]
    live = vis.any(-1, keepdim=True)
    s = (Q @ K.repeat_interleave(G, 1).transpose(-1, -2) * scale).masked_fill(~vis, -math.inf).masked_fill(~live, 0.0)
    o = torch.softmax(s, -1) @ V.repeat_interleave(G, 1)
    lse = torch.logsumexp(s, -1) / math.log(2.0)
    dO = do.double().transpose(1, 2) * live
    dq, dk, dv = torch.autograd.grad(o, (Q, K, V), dO)
    return [t.transpose(1, 2).detach() for t in (o, dq, dk, dv)] + [lse.detach(), live[..., 0].expand(B, nh, Sq)]


@pytest.mark.parametrize("c", SMALL, ids=lambda c: c.id)
def test_reference_matches_an_independent_formulation(c):
    q, k, v, do = R.make_inputs(c, "cpu")
    kmask = R.make_kmask(c, "cpu")
    o, dq, dk, dv, lse, live = _independent(q, k, v, do, c.causal, kmask, c.scale, c.window)
    f = R.fwd_ref(q, k, v, causal=c.causal, kmask=kmask, scale=c.scale, window=c.window)
    rows = live.transpose(1, 2)
    torch.testing.assert_close(f["o"][rows], o[rows], rtol=1e-10, atol=1e-12)
    assert torch.equal(f["empty"], ~live) and (f["o"][~rows] == 0).all()
    torch.testing.assert_close(f["lse"][live], lse[live], rtol=1e-10, atol=1e-10)
    b = R.bwd_ref(q, k, v, f["o"], do, f["lse"], causal=c.causal, kmask=kmask, scale=c.scale, window=c.window)
    for name, got, want in (("dq", b["dq"], dq), ("dk", b["dk"], dk), ("dv", b["dv"], dv)):
        torch.testing.assert_close(got, want, rtol=1e-9, atol=1e-10, msg=name)


@pytest.mark.parametrize("c", SMALL, ids=lambda c: c.id)
def test_stand_in_within_the_kernel_bounds(c):
    q, k, v, do = R.make_inputs(c, "cpu")
    kmask = R.make_kmask(c, "cpu")
    out = torch.full((c.B, c.Sq, c.nh + 1, c.hd), 7.0, dtype=torch.bfloat16)
    o, lse = emu.attn_fwd(q, k, v, causal=c.causal, kmask=kmask, scale=c.scale, need_lse=True, out=out[:, :, 1:],
                          window=c.window)
    assert o.data_ptr() == out[:, :, 1:].data_ptr() and (out[:, :, 0] == 7.0).all()
    f = R.fwd_ref(q, k, v, causal=c.causal, kmask=kmask, scale=c.scale, window=c.window)
    check_bf16("stand-in O", o, f["o"], f["tol_o"])
    R.check_lse("stand-in LSE", lse, f, check_abs)
    dqkv = torch.zeros(c.B, c.Sq, c.nh + 2 * c.nkv, c.hd, dtype=torch.bfloat16) if c.Sq == c.Skv else None
    views = (dqkv[:, :, :c.nh], dqkv[:, :, c.nh:c.nh + c.nkv], dqkv[:, :, c.nh + c.nkv:]) if dqkv is not None else (None,) * 3
    dq, dk, dv = emu.attn_bwd(q, k, v, o, do, lse, causal=c.causal, kmask=kmask, scale=c.scale, dq=views[0], dk=views[1],
                              dv=views[2], window=c.window)
    if dqkv is not None:
        assert dq.data_ptr() == dqkv.data_ptr() and dv.data_ptr() == views[2].data_ptr()
    b = R.bwd_ref(q, k, v, o, do, lse, causal=c.causal, kmask=kmask, scale=c.scale, window=c.window)
    check_bf16("stand-in dQ", dq, b["dq"], b["tol_dq"])
    check_bf16("stand-in dK", dk, b["dk"], b["tol_dk"])
    check_bf16("stand-in dV", dv, b["dv"], b["tol_dv"])


def test_kmask_operand_check():
    from cambrian_b200.ops import _kmask_u8
    assert _kmask_u8(None, 2, 5) is None
    m = torch.tensor([[True, False, True], [False, True, True]])
    u = _kmask_u8(m, 2, 3)
    assert u.dtype == torch.uint8 and u.is_contiguous() and u.tolist() == [[1, 0, 1], [0, 1, 1]]
    assert _kmask_u8(m.long(), 2, 3).tolist() == u.tolist()
    assert _kmask_u8(torch.ones(3, 2, dtype=torch.bool).T, 2, 3).is_contiguous()
    for bad in (torch.ones(2, 4, dtype=torch.bool), torch.ones(3, dtype=torch.bool), torch.ones(1, 3, dtype=torch.bool)):
        with pytest.raises(ValueError, match=r"kmask must be \[B, Skv\]"):
            _kmask_u8(bad, 2, 3)
