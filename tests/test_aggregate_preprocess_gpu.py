"""The tower combine and the bilinear adjoint (aggregate.cu) and the GPU image preprocessing (preprocess.cu) against the
float64 references and bounds of tests/aggregate_reference.py, and the preprocessing bit for bit against Pillow.

Every case calls the C entry point through `_lib.load()` into sentinel-filled slabs with guards between them, so a write
outside an output shows up bitwise, then runs the `cambrian_b200.ops` wrapper into fresh memory and requires the same bits.
Size thresholds (the tower combine's and the adjoint's grid-stride caps) come from `cb_sm_count()`, so the grid-stride
cases reach that loop on any H100.  Each check prints its worst error-to-bound ratio; the module prints the worst per output
at the end.  tests/test_aggregate_preprocess_cpu.py runs the references, the stand-ins and the integer preprocessing model
of the same case tables without a GPU.
"""
from __future__ import annotations

import ctypes

import numpy as np
import pytest
import torch

import aggregate_reference as A
import vision_kernels_reference as V
from row_kernels_reference import HALF_ULP, assert_bitwise, assert_either, check_abs, check_bf16, sentinel_like

pytestmark = pytest.mark.gpu

DEV = "cuda"
GUARD = 4096
WORST: dict = {}


@pytest.fixture(scope="module")
def ops():
    from cambrian_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def sms(lib):
    return lib.cb_sm_count()


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    print("\n  worst |err|/bound per output over all cases:")
    for k, v in sorted(WORST.items()):
        print(f"    {k}: {v:.3g}")


def _note(key, ratio):
    WORST[key] = max(WORST.get(key, 0.0), ratio)


def _bf16(key, name, got, ref, tol):
    _note(key, check_bf16(name, got, ref, tol))


def _slabs(shapes, dtype=torch.bfloat16):
    """one sentinel-filled buffer holding a contiguous slab per shape, with sentinel guards before, between and after."""
    sizes = [int(torch.Size(s).numel()) for s in shapes]
    n = sum(sizes) + GUARD * (len(sizes) + 1)
    if dtype == torch.uint8:
        buf = torch.full((n,), 0xA5, dtype=torch.uint8, device=DEV)
    else:
        buf = sentinel_like((n,), dtype, DEV)
    slabs, guards, off = [], [buf[:GUARD]], GUARD
    for s, k in zip(shapes, sizes):
        slabs.append(buf[off:off + k].view(s))
        guards.append(buf[off + k:off + k + GUARD])
        off += k + GUARD
    return slabs, guards


def _guards_intact(what, guards):
    for i, g in enumerate(guards):
        if g.dtype == torch.uint8:
            bad = int((g != 0xA5).sum())
            print(f"    {what} guard {i}: {bad} of {g.numel()} bytes changed")
            assert bad == 0, f"{what} guard {i}: {bad} bytes changed"
        else:
            assert_bitwise(f"{what} guard {i}", g, sentinel_like(g.shape, g.dtype, DEV))


def _ptrs(ts):
    arr = (ctypes.c_void_p * len(ts))()
    for i, t in enumerate(ts):
        arr[i] = t.data_ptr()
    return arr


def _rc(lib, rc, what):
    assert rc == 0, f"{what}: {lib.cb_last_error().decode()}"


# ======================================================================================================= tower combine
@pytest.mark.parametrize("case", A.COMBINE_CASES, ids=A.combine_case_id)
def test_tower_combine(ops, lib, sms, case):
    T, ldl, C, N_, regime, cancel = case
    N = A.combine_rows(N_, sms)
    logits, aggs, q_in, dout = A.combine_inputs(case, N, DEV)
    print(f"\n  tower_combine T={T} ld={ldl} C={C} N={N} (grid cap {A.combine_grid_rows(sms)} rows) {regime} cancel={cancel}")
    ref = A.combine_ref(logits, aggs, q_in, dout)

    slabs, guards = _slabs([(N, C)] * (T + 1) + [(N, ldl)])
    out, daggs, dl = slabs[0], slabs[1:T + 1], slabs[T + 1]
    st = torch.cuda.current_stream().cuda_stream
    _rc(lib, lib.cb_tower_combine_fwd(logits.data_ptr(), ldl, _ptrs(aggs), q_in.data_ptr(), out.data_ptr(), N, C, T, st),
        "cb_tower_combine_fwd")
    _rc(lib, lib.cb_tower_combine_bwd(logits.data_ptr(), ldl, _ptrs(aggs), dout.data_ptr(), _ptrs(daggs), dl.data_ptr(),
                                      N, C, T, st), "cb_tower_combine_bwd")
    torch.cuda.synchronize()

    _bf16("tower_combine out", "out", out, ref["out"], ref["tol_out"])
    for t in range(T):
        _bf16("tower_combine dagg", f"dagg[{t}]", daggs[t], ref["dagg"][t], ref["tol_dagg"][t])
    _bf16("tower_combine dlogits", "dlogits", dl[:, :T], ref["dl"], ref["tol_dl"])
    if ldl > T:
        assert_bitwise("dlogits padding columns are +0", dl[:, T:], torch.zeros(N, ldl - T, dtype=torch.bfloat16, device=DEV))
    _guards_intact("tower_combine", guards)

    out2 = ops.tower_combine_fwd(logits, aggs, q_in)
    daggs2, dl2 = ops.tower_combine_bwd(logits, aggs, dout)
    assert_bitwise("rerun out", out2, out)
    for t in range(T):
        assert_bitwise(f"rerun dagg[{t}]", daggs2[t], daggs[t])
    assert_bitwise("rerun dlogits", dl2, dl)


def test_tower_combine_operand_checks(ops, lib):
    """each malformed call raises ValueError in the wrapper, before anything is launched."""
    N, C, T = 16, 64, 3
    logits, aggs, q_in, dout = A.combine_inputs((T, 8, C, N, "spread", False), N, DEV)
    wide = torch.zeros(N, 2 * C, dtype=torch.bfloat16, device=DEV)
    calls = [
        ("fwd: q_in a column slice", lambda: ops.tower_combine_fwd(logits, aggs, wide[:, C:])),
        ("fwd: aggregate a column slice", lambda: ops.tower_combine_fwd(logits, [aggs[0], wide[:, :C], aggs[2]], q_in)),
        ("fwd: logits rows != N", lambda: ops.tower_combine_fwd(logits[:-1], aggs, q_in)),
        ("bwd: aggregate a column slice", lambda: ops.tower_combine_bwd(logits, [aggs[0], wide[:, :C], aggs[2]], dout)),
        ("bwd: aggregate with fewer rows", lambda: ops.tower_combine_bwd(logits, [aggs[0], aggs[1][:-1], aggs[2]], dout)),
        ("bwd: aggregate with fewer columns", lambda: ops.tower_combine_bwd(logits, [a[:, :C - 8].contiguous() for a in aggs],
                                                                           dout)),
        ("bwd: logits rows != N", lambda: ops.tower_combine_bwd(logits[:-1], aggs, dout)),
        ("bwd: logits with 40 columns", lambda: ops.tower_combine_bwd(torch.zeros(N, 40, dtype=torch.bfloat16, device=DEV),
                                                                     aggs, dout)),
        ("bwd: logits not contiguous", lambda: ops.tower_combine_bwd(torch.zeros(N, 16, dtype=torch.bfloat16,
                                                                                 device=DEV)[:, :8], aggs, dout)),
    ]
    torch.cuda.synchronize()
    for what, call in calls:
        before = lib.cb_launch_count()
        with pytest.raises(ValueError):
            call()
        assert lib.cb_launch_count() == before, f"{what}: launched before refusing"
        print(f"    {what}: ValueError, nothing launched")


# =================================================================================================== bilinear backward
@pytest.mark.parametrize("case", A.BILINEAR_BWD_CASES, ids=A.bilinear_bwd_case_id)
def test_bilinear_bwd(ops, lib, sms, case):
    h, w, th, tw, B_, C = case
    B = A.bilinear_bwd_batch(B_, h, w, C, sms)
    items, cap = B * h * w * C // 8, A.bilinear_bwd_cap(sms)
    print(f"\n  bilinear_bwd {h}x{w} <- {th}x{tw} B={B} C={C}: {items} work items (grid cap {cap})")
    if B_ == "grid":
        assert items > cap
    g = V.randn((B, th * tw, C), 2, DEV)
    ref, tol = A.bilinear_bwd_ref(g, h, w, th, tw)

    (din,), guards = _slabs([(B, h * w, C)])
    _rc(lib, lib.cb_bilinear_bwd(g.data_ptr(), din.data_ptr(), B, h, w, th, tw, C, torch.cuda.current_stream().cuda_stream),
        "cb_bilinear_bwd")
    torch.cuda.synchronize()
    _bf16("bilinear_bwd din", "din", din, ref, tol)
    if (h, w) == (th, tw):
        assert_bitwise("identity", din, g)
    _guards_intact("bilinear_bwd", guards)
    assert_bitwise("rerun din", ops.bilinear_bwd(g, h, w, th, tw), din)

    # <bilinear(x), g> == <x, bilinear_bwd(g)> on the two kernels' outputs, in fp64, within both kernels' bounds
    x = V.randn((B, h * w, C), 1, DEV)
    y = ops.bilinear(x, h, w, th, tw)
    yref, ytol, _ = V.bilinear_ref(x, h, w, th, tw)
    lhs = (y.double() * g.double()).sum()
    rhs = (x.double() * din.double()).sum()
    bound = ((g.double().abs() * (HALF_ULP * yref.abs() + ytol)).sum()
             + (x.double().abs() * (HALF_ULP * ref.abs() + tol)).sum())
    _note("bilinear adjoint identity", check_abs("adjoint identity", lhs, rhs, bound))


# ====================================================================================================== preprocessing
@pytest.mark.parametrize("case", A.PREPROCESS_CASES, ids=A.preprocess_case_id)
def test_preprocess(ops, lib, case):
    H, W, tower = case
    R, mean, std = A.tower_processors()[tower]
    pad = tuple(int(x * 255) for x in mean)
    S = max(H, W)
    print(f"\n  preprocess {H}x{W} -> {R} ({tower}, pad {pad}) offsets {A.pad_offsets(H, W)} ksize {A.resample_ksize(S, R)}")
    arr = A.preprocess_image_input(H, W)
    want = A.pillow_resize(arr, R, pad)
    model = A.resize_model(arr, R, pad)
    assert np.array_equal(model, want), "the integer model differs from Pillow"
    img = torch.from_numpy(arr).to(DEV)

    (u8,), u8_guards = _slabs([(R, R, 3)], torch.uint8)
    (out,), out_guards = _slabs([(3, R, R)])
    nbytes = lib.cb_preprocess_workspace_bytes(H, W, R)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    padc = (ctypes.c_int32 * 3)(*pad)
    m = (ctypes.c_float * 3)(*mean)
    sd = (ctypes.c_float * 3)(*std)
    _rc(lib, lib.cb_preprocess_image(img.data_ptr(), H, W, R, ctypes.addressof(padc), ctypes.addressof(m),
                                     ctypes.addressof(sd), out.data_ptr(), u8.data_ptr(), ws.data_ptr(), nbytes,
                                     torch.cuda.current_stream().cuda_stream), "cb_preprocess_image")
    torch.cuda.synchronize()
    got = u8.cpu().numpy()
    bad = int((got != want).sum())
    print(f"    uint8 vs Pillow: {bad} of {got.size} bytes differ")
    assert bad == 0, f"uint8 image: {bad} bytes differ from Pillow"
    fused, unfused = A.normalise_candidates(want, mean, std)
    assert_either("bf16 normalised", out.cpu(), fused, unfused)
    _guards_intact("preprocess uint8", u8_guards)
    _guards_intact("preprocess bf16", out_guards)

    out2, u82 = ops.preprocess_image(img, R, pad, mean, std, return_u8=True)
    assert torch.equal(u82, u8), "a second call gave different uint8 bytes"
    assert_bitwise("second call bf16", out2, out)
