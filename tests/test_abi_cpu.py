"""CPU-only checks of the drop-in boundary: the C-ABI library loads, exports every symbol include/cambrian_b200.h
declares (and the ctypes table lists exactly those), and the product path fails loudly without CUDA (no fallback)."""
import ctypes
import re
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent


def _header_symbols():
    text = (ROOT / "include" / "cambrian_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(cb_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol(lib):
    syms = _header_symbols()
    assert len(syms) >= 30
    for s in syms:
        assert hasattr(lib, s), f"libcambrian_b200.so does not export {s}"


def test_ctypes_table_matches_header():
    from cambrian_b200 import _lib
    assert sorted(_lib.SIGNATURES) == _header_symbols()


def test_version_and_error_channel(lib):
    assert lib.cb_version() == 1
    assert isinstance(lib.cb_last_error(), bytes)
    assert lib.cb_launch_count() >= 0


def test_argument_validation_returns_error_code_without_gpu(lib):
    # empty problem -> CB_ERR_INVALID (1) before any CUDA call; message available through cb_last_error
    rc = lib.cb_gemm_bf16(None, None, None, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0, None, None, None, 0, 0,
                          ctypes.c_float(1.0), 0, 0, 0, 0, None)
    assert rc == 1
    assert b"gemm" in lib.cb_last_error()
    rc = lib.cb_sva_window_attn_fwd(None, None, None, 0, None, None, None, None, 1, 24, 1024, 0, None)
    assert rc == 1 and b"num_towers" in lib.cb_last_error()
    rc = lib.cb_sva_window_attn_fwd(None, None, None, 1, None, None, None, None, 1, 24, 512, 0, None)
    assert rc == 1 and b"hidden" in lib.cb_last_error()
    rc = lib.cb_attn_fwd(None, None, None, None, None, None, 1, 6, 4, 8, 8, 64, 0, 0, 0, 0, 0, 0, 0, 0,
                         ctypes.c_float(1.0), 0, None)
    assert rc == 1 and b"nh" in lib.cb_last_error()


def test_no_cpu_fallback():
    from cambrian_b200 import _lib, ops
    a = torch.zeros(8, 8, dtype=torch.bfloat16)
    with pytest.raises(_lib.CambrianB200Error):
        ops.gemm(a, a)
    from cambrian_b200.model.vision_sampler import VisionTokenSampler
    m = VisionTokenSampler(64, 1024, [1024], [1], 1024, 1)
    with pytest.raises(RuntimeError):
        m(torch.zeros(4, 1, 64), torch.zeros(4, 1, 1024), torch.zeros(4, 1, 1024), torch.ones(4, 1, dtype=torch.bool))


def test_product_never_imports_the_oracle():
    for p in (ROOT / "cambrian_b200").rglob("*.py"):
        src = p.read_text()
        assert "oracle" not in re.sub(r'""".*?"""', "", src, flags=re.S).replace("# oracle", ""), \
            f"{p} references the oracle — the product path must not depend on test infrastructure"


def test_argument_validation_of_later_entry_points_without_gpu(lib):
    """Every check below fails before the first CUDA call, so it runs on the CPU-only builder too."""
    one = ctypes.c_void_p(16)                                   # non-null, 16-byte aligned dummy pointer (never dereferenced)
    rc = lib.cb_gemm_swiglu_bf16(one, one, one, one, 256, 100, 64, 64, 64, 200, 100, None)
    assert rc == 1 and b"multiple of 128" in lib.cb_last_error()
    rc = lib.cb_gemm_swiglu_bf16(None, one, one, one, 256, 128, 64, 64, 64, 256, 128, None)
    assert rc == 1 and b"null" in lib.cb_last_error()
    rc = lib.cb_window_gather(one, one, 1, 4, 2, 64, 0, 5, 0, 4, None)        # crop rows [0, 5) of a 4 x 4 query grid
    assert rc == 1 and b"crop" in lib.cb_last_error()
    rc = lib.cb_window_gather(one, one, 1, 4, 2, 60, 0, 4, 0, 4, None)        # channels not a multiple of 8
    assert rc == 1
    rc = lib.cb_span_gather_hw(one, one, 1, 20, 64, 5, 4, 4, None)            # 4 x (4 + 1) = 20 rows from position 5 of 20
    assert rc == 1 and b"outside sequence" in lib.cb_last_error()
    rc = lib.cb_span_scatter_hw(one, one, 1, 64, 64, 5, 0, 4, None)           # empty grid
    assert rc == 1
    rc = lib.cb_embed_splice_ragged(one, one, one, one, one, 0, 64, None)
    assert rc == 1 and b"no rows" in lib.cb_last_error()
    rc = lib.cb_preprocess_image(None, 10, 10, 8, None, None, None, None, None, None, 0, None)
    assert rc == 1 and b"null" in lib.cb_last_error()
    pad = (ctypes.c_int32 * 3)(0, 0, 0)
    f3 = (ctypes.c_float * 3)(0.5, 0.5, 0.5)
    need = lib.cb_preprocess_workspace_bytes(480, 640, 336)
    assert need > 640 * 336 * 3
    rc = lib.cb_preprocess_image(one, 480, 640, 336, ctypes.addressof(pad), ctypes.addressof(f3), ctypes.addressof(f3), one, None,
                                 one, need - 1, None)
    assert rc == 1 and b"workspace" in lib.cb_last_error()
    assert lib.cb_preprocess_workspace_bytes(0, 640, 336) == 0
    assert lib.cb_resample_ksize(640, 336) == 9 and lib.cb_resample_ksize(336, 336) == 5


def test_resample_coefficients_are_normalised(lib):
    """Fixed-point rows sum to 2^22 (+- rounding) and stay inside the source image — host-only entry point."""
    for (src, dst) in ((640, 336), (336, 336), (100, 384), (1500, 1024)):
        ks = lib.cb_resample_ksize(src, dst)
        bounds = (ctypes.c_int32 * (2 * dst))()
        kk = (ctypes.c_int32 * (ks * dst))()
        assert lib.cb_resample_coeffs(src, dst, ctypes.addressof(bounds), ctypes.addressof(kk)) == 0
        for x in range(dst):
            x0, n = bounds[2 * x], bounds[2 * x + 1]
            assert 0 <= x0 and x0 + n <= src and 0 < n <= ks
            row = kk[x * ks:(x + 1) * ks]
            assert abs(sum(row) - (1 << 22)) <= ks and all(v == 0 for v in row[n:])


def test_attention_backward_refuses_misaligned_operands_without_gpu(lib):
    """O and dO are read as 16-byte vectors by the delta kernel, dK and dV stored as bf16 pairs: a misaligned pointer or
    stride is refused before the first launch (fake, never dereferenced pointers)."""
    B, nh, nkv, S, hd = 2, 4, 2, 128, 64
    rs, bs = nh * hd, S * nh * hd                                   # packed heads: row and batch strides of a [B, S, nh, hd]
    ks, kbs = nkv * hd, S * nkv * hd
    base = 1 << 20

    def call(o=base, d_o=base, dk=base, dv=base, o_ss=rs, o_bs=bs, do_ss=rs, do_bs=bs, dk_ss=ks, dk_bs=kbs, dv_ss=ks,
             dv_bs=kbs, Bn=B):
        p = ctypes.c_void_p
        return lib.cb_attn_bwd(p(base), p(base), p(base), p(o), p(d_o), p(base), p(base), p(base), p(dk), p(dv), None,
                               Bn, nh, nkv, S, S, hd, bs, rs, kbs, ks, kbs, ks, o_bs, o_ss, do_bs, do_ss, bs, rs, dk_bs,
                               dk_ss, dv_bs, dv_ss, ctypes.c_float(0.125), 1, None)

    for kw, name in ((dict(o=base + 2), b"o must"), (dict(o=base + 8), b"o must"), (dict(o_ss=rs + 4), b"o must"),
                     (dict(o_bs=bs + 2), b"o must"), (dict(d_o=base + 8), b"d_o must"), (dict(do_ss=rs + 2), b"d_o must"),
                     (dict(do_bs=bs + 4), b"d_o must"), (dict(dk=base + 2), b"dk must"), (dict(dk_ss=ks + 1), b"dk must"),
                     (dict(dk_bs=kbs + 1), b"dk must"), (dict(dv=base + 6), b"dv must"), (dict(dv_ss=ks + 1), b"dv must"),
                     (dict(dv_bs=kbs - 1), b"dv must"), (dict(o=0), b"o must")):
        assert call(**kw) == 1, kw
        assert name in lib.cb_last_error(), (kw, lib.cb_last_error())
    # a single batch element never uses its batch stride
    assert call(Bn=1, o=base + 2) == 1
    rc = lib.cb_attn_bwd_window(*([ctypes.c_void_p(base)] * 4 + [ctypes.c_void_p(base + 8)] + [ctypes.c_void_p(base)] * 5
                                  + [None]), B, nh, nkv, S, S, hd, bs, rs, kbs, ks, kbs, ks, bs, rs, bs, rs, bs, rs, kbs, ks,
                                kbs, ks, ctypes.c_float(0.125), 1, 64, None)
    assert rc == 1 and b"d_o must" in lib.cb_last_error()
