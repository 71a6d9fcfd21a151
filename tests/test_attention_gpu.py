"""Flash attention (csrc/attention.cu through `ops.attn_fwd` / `ops.attn_bwd`) against the float64 references of
tests/attention_reference.py, which also derives each error bound and holds the case tables.

Every case checks its outputs against the bound and prints the worst error-to-bound ratio, then the bitwise properties:
outputs land in views of sentinel-filled buffers and nothing else changes; a second run gives the same bits; K / V rows
hidden from every query (masked, outside every window, past Skv in the buffer the view comes from) can be overwritten
without changing one bit, and their dK / dV are exactly 0; changing the key at slot t leaves every row that cannot see it
unchanged; each batch element and head run alone equals its slice of the full run.
"""
from __future__ import annotations

import pytest
import torch

import attention_reference as R
from row_kernels_reference import assert_bitwise, check_abs, check_bf16, sentinel_like

pytestmark = pytest.mark.gpu

DEV = "cuda"
PAD = 64          # rows past S in every backing buffer (past the last tile, read by nothing)


@pytest.fixture(scope="module")
def ops():
    from cambrian_b200 import ops as o
    return o


@pytest.fixture(scope="module", autouse=True)
def _release_cache():
    """the module allocates many odd-sized buffers (sentinel views, fp64 references); hand the cached blocks back to the
    device when it ends, so later tests' memory accounting does not start from a fragmented cache"""
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


class View:
    """A [B, S, heads, hd] view into a larger backing buffer; `fill` puts values in it, `guard` checks that nothing
    outside it changed from the sentinel."""

    def __init__(self, B, S, heads, hd, layout, col=0, width=None, sentinel=True):
        width = width or heads
        self.sl = lambda t: t[:, :S, col:col + heads]
        if layout == "contig":
            self.sl = lambda t: t
            shape = (B, S, heads, hd)
        else:
            shape = (B, S + PAD, width, hd)
        self.buf = sentinel_like(shape, torch.bfloat16, DEV) if sentinel else torch.zeros(shape, dtype=torch.bfloat16,
                                                                                          device=DEV)
        self.view = self.sl(self.buf)

    def fill(self, t):
        self.view.copy_(t)
        return self.view

    def guard(self, name):
        t = self.buf.clone()
        self.sl(t).view(torch.int16).fill_(0x7FA5)
        assert_bitwise(f"{name} outside the view", t, sentinel_like(t.shape, torch.bfloat16, DEV))


def operands(c, q, k, v):
    """q / k / v views in the case's layout, with K / V backing buffers that hold rows past Skv."""
    lay = "padded" if c.layout in ("padded_batch", "out_slice") else c.layout
    if lay == "packed":
        w = c.nh + 2 * c.nkv
        qv = View(c.B, c.Sq, c.nh, c.hd, "packed", 0, w, sentinel=False)
        kb = View(c.B, c.Skv, c.nkv, c.hd, "packed", c.nh, w, sentinel=False)
        vb = View(c.B, c.Skv, c.nkv, c.hd, "packed", c.nh + c.nkv, w, sentinel=False)
        vb.buf = kb.buf
        vb.view = vb.sl(kb.buf)
    else:
        qv, kb, vb = (View(c.B, S, hh, c.hd, lay, sentinel=False)
                      for S, hh in ((c.Sq, c.nh), (c.Skv, c.nkv), (c.Skv, c.nkv)))
    return qv.fill(q), kb.fill(k), vb.fill(v), kb, vb


def out_view(c):
    """O's destination: a column slice of a wider buffer (out_slice) or rows of a taller one, sentinel-filled."""
    if c.layout == "out_slice":
        return View(c.B, c.Sq, c.nh, c.hd, "slice", 1, c.nh + 2)
    return View(c.B, c.Sq, c.nh, c.hd, "padded")


def fwd(ops, c, q, k, v, kmask, out=None):
    return ops.attn_fwd(q, k, v, causal=c.causal, kmask=kmask, scale=c.scale, need_lse=True, out=out, window=c.window)


def bwd(ops, c, q, k, v, o, do, lse, kmask, dq=None, dk=None, dv=None):
    return ops.attn_bwd(q, k, v, o, do, lse, causal=c.causal, kmask=kmask, scale=c.scale, dq=dq, dk=dk, dv=dv,
                        window=c.window)


def hide_keys(c, kmask, kb, vb):
    """overwrite every K / V row no query of its batch element sees, and the rows past Skv, with BIG; returns the
    [B, Skv] bool of hidden keys."""
    vis = R.visible(c.Sq, c.Skv, c.causal, c.window, kmask, DEV).expand(c.B, c.Sq, c.Skv)
    hidden = ~vis.any(1)
    for t in (kb, vb):
        if t.buf.shape[1] > c.Skv:
            t.buf[:, c.Skv:] = R.BIG
        t.view.masked_fill_(hidden[:, :, None, None], R.BIG)
    return hidden


def forward_checks(ops, c, q, k, v, kmask):
    """the forward's bound, sentinel, rerun, hidden-key, key-slot and independence checks; returns (o, lse) of the run."""
    qv, kv, vv, kb, vb = operands(c, q, k, v)
    ov = out_view(c)
    o, lse = fwd(ops, c, qv, kv, vv, kmask, out=ov.view)
    torch.cuda.synchronize()
    ref = R.fwd_ref(q, k, v, causal=c.causal, kmask=kmask, scale=c.scale, window=c.window)
    check_bf16("O", o, ref["o"], ref["tol_o"])
    R.check_lse("LSE", lse, ref, check_abs)
    ov.guard("O")
    o2, lse2 = fwd(ops, c, qv, kv, vv, kmask)
    assert_bitwise("rerun O", o2, o)
    assert_bitwise("rerun LSE", lse2, lse)

    # the same problem with every hidden K / V row overwritten
    q2, k2, v2, kb2, vb2 = operands(c, q, k, v)
    hidden = hide_keys(c, kmask, kb2, vb2)
    print(f"    {int(hidden.sum())} hidden keys overwritten")
    o3, lse3 = fwd(ops, c, q2, k2, v2, kmask)
    assert_bitwise("hidden keys overwritten: O", o3, o)
    assert_bitwise("hidden keys overwritten: LSE", lse3, lse)

    # a changed key at slot t: the rows that cannot see it keep their bits
    if c.causal:
        t = c.Skv // 2
        k2[:, t] = -k2[:, t] + 0.5
        v2[:, t] = -v2[:, t] - 0.5
        o4, lse4 = fwd(ops, c, q2, k2, v2, kmask)
        i = torch.arange(c.Sq, device=DEV) + c.Skv - c.Sq
        blind = (i < t) | ((i - t >= c.window) if c.window else torch.zeros_like(i, dtype=torch.bool))
        print(f"    key slot {t} changed: {int(blind.sum())} of {c.Sq} rows cannot see it")
        assert_bitwise("rows blind to the changed key: O", o4[:, blind], o[:, blind])
        assert_bitwise("rows blind to the changed key: LSE", lse4[:, :, blind], lse[:, :, blind])

    # each batch element and head alone
    for b, h in {(0, 0), (c.B - 1, c.nh - 1)}:
        hk = h // (c.nh // c.nkv)
        km = None if kmask is None else kmask[b:b + 1]
        o5, lse5 = fwd(ops, c, qv[b:b + 1, :, h:h + 1], kv[b:b + 1, :, hk:hk + 1], vv[b:b + 1, :, hk:hk + 1], km)
        assert_bitwise(f"batch {b} head {h} alone: O", o5, o[b:b + 1, :, h:h + 1])
        assert_bitwise(f"batch {b} head {h} alone: LSE", lse5, lse[b:b + 1, h:h + 1])
    return o, lse


@pytest.mark.parametrize("c", R.FWD_CASES, ids=lambda c: c.id)
def test_attention_forward(ops, c):
    print(f"\n  {c.id}")
    q, k, v, _ = R.make_inputs(c, DEV)
    forward_checks(ops, c, q, k, v, R.make_kmask(c, DEV))


@pytest.mark.parametrize("c", R.BWD_CASES, ids=lambda c: c.id)
def test_attention_backward(ops, c):
    print(f"\n  {c.id}")
    q, k, v, do = R.make_inputs(c, DEV)
    kmask = R.make_kmask(c, DEV)
    o, lse = forward_checks(ops, c, q, k, v, kmask)
    qv, kv, vv, _, _ = operands(c, q, k, v)
    if c.layout == "packed":          # dQ and dK / dV in the packed column layout of a dQKV buffer
        w = c.nh + 2 * c.nkv
        dqv = View(c.B, c.Sq, c.nh, c.hd, "packed", 0, w)
        dkv = View(c.B, c.Skv, c.nkv, c.hd, "packed", c.nh, w)
        dvv = View(c.B, c.Skv, c.nkv, c.hd, "packed", c.nh + c.nkv, w)
        if c.Sq == c.Skv:
            dkv.buf = dvv.buf = dqv.buf
            dkv.view, dvv.view = dkv.sl(dqv.buf), dvv.sl(dqv.buf)
    else:
        dqv, dkv, dvv = (View(c.B, S, hh, c.hd, "padded") for S, hh in ((c.Sq, c.nh), (c.Skv, c.nkv), (c.Skv, c.nkv)))
    dq, dk, dv = bwd(ops, c, qv, kv, vv, o, do, lse, kmask, dqv.view, dkv.view, dvv.view)
    torch.cuda.synchronize()
    ref = R.bwd_ref(q, k, v, o, do, lse, causal=c.causal, kmask=kmask, scale=c.scale, window=c.window)
    check_bf16("dQ", dq, ref["dq"], ref["tol_dq"])
    check_bf16("dK", dk, ref["dk"], ref["tol_dk"])
    check_bf16("dV", dv, ref["dv"], ref["tol_dv"])
    if c.layout == "packed" and c.Sq == c.Skv:
        t = dqv.buf.clone()
        for vw in (dqv, dkv, dvv):
            vw.sl(t).view(torch.int16).fill_(0x7FA5)
        assert_bitwise("dQKV outside the three views", t, sentinel_like(t.shape, torch.bfloat16, DEV))
    else:
        for name, vw in (("dQ", dqv), ("dK", dkv), ("dV", dvv)):
            vw.guard(name)
    got = [t.clone() for t in (dq, dk, dv)]
    for name, a, b_ in zip(("dQ", "dK", "dV"), bwd(ops, c, qv, kv, vv, o, do, lse, kmask), got):
        assert_bitwise(f"rerun {name}", a, b_)

    q2, k2, v2, kb2, vb2 = operands(c, q, k, v)
    hidden = hide_keys(c, kmask, kb2, vb2)
    dq3, dk3, dv3 = bwd(ops, c, q2, k2, v2, o, do, lse, kmask)
    assert_bitwise("hidden keys overwritten: dQ", dq3, got[0])
    assert_bitwise("hidden keys overwritten: dK", dk3, got[1])
    assert_bitwise("hidden keys overwritten: dV", dv3, got[2])
    for name, t in (("dK", got[1]), ("dV", got[2])):
        assert int((t[hidden] != 0).sum()) == 0, f"{name} of hidden keys is not exactly 0"

    for b in range(c.B):
        km = None if kmask is None else kmask[b:b + 1]
        one = bwd(ops, c, qv[b:b + 1], kv[b:b + 1], vv[b:b + 1], o[b:b + 1], do[b:b + 1], lse[b:b + 1], km)
        for name, a, full in zip(("dQ", "dK", "dV"), one, got):
            assert_bitwise(f"batch {b} alone: {name}", a, full[b:b + 1])


@pytest.mark.parametrize("hdp", sorted(R.HDP_CLASSES))
def test_all_true_mask_equals_no_mask(ops, hdp):
    """every padded head-dim class (a full and a zero-padded head), an odd Skv so that batch row 1 of the mask is not
    4-byte aligned: an all-True mask gives the bits of no mask, causal and not."""
    for hd in R.HDP_CLASSES[hdp]:
        for causal in (False, True):
            c = R.case("fwd", hd, 3, 2, 1, 257, 387, causal)
            q, k, v, _ = R.make_inputs(c, DEV, seed=5)
            ones = torch.ones(c.B, c.Skv, dtype=torch.bool, device=DEV)
            o0, l0 = fwd(ops, c, q, k, v, None)
            o1, l1 = fwd(ops, c, q, k, v, ones)
            assert_bitwise(f"hd {hd} causal={causal}: O", o1, o0)
            assert_bitwise(f"hd {hd} causal={causal}: LSE", l1, l0)


def test_kmask_over_a_longer_buffer_is_refused(ops):
    c = R.case("fwd", 64, 2, 2, 2, 5, 40, True)
    q, k, v, do = R.make_inputs(c, DEV)
    whole = torch.ones(c.B, 64, dtype=torch.bool, device=DEV)
    with pytest.raises(ValueError, match=r"kmask must be \[B, Skv\]"):
        ops.attn_fwd(q, k, v, causal=True, kmask=whole)
    o, lse = ops.attn_fwd(q, k, v, causal=True, kmask=whole[:, :40], need_lse=True)
    with pytest.raises(ValueError, match=r"kmask must be \[B, Skv\]"):
        ops.attn_bwd(q, k, v, o, do, lse, causal=True, kmask=whole)
