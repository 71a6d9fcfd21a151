"""Torch emulations of the FP8 training entry points (cambrian_b200/train_fp8.py states the format), written on the row
rule of tests/fp8_reference.py, and CPU stand-ins of them for host-logic tests.

  fp8_quantize_weight_t(W)  = the row rule on the rows of W^T (per input column of W);
  rmsnorm_fwd_fp8(x)        = the row rule on rmsnorm_fwd(x), i.e. after its rounding to bf16;
  swiglu_bwd_fp8(...)       = swiglu_bwd, then the row rule on the [rows, 2I] gradient [dgate | dup].
"""
import torch

import fp8_reference as R
import ops_emulation as E


def quantize_weight_t(w):
    """bf16 W [N, K] -> (wtq float8_e4m3fn [K, N], st fp32 [K])."""
    return R.quantize_rows(w.t())


def quantize_dgu(dgate, dup):
    """E4M3 rows of the bf16 gradient [dgate | dup] [rows, 2I]."""
    return R.quantize_act(torch.cat([dgate, dup], 1))


# ---- CPU stand-ins of the three entry points (host-logic tests on machines without a GPU) ----
def fp8_quantize_weight_t(w, wtq, st):
    q, s = quantize_weight_t(w)
    wtq.copy_(q)
    st.copy_(s)


def rmsnorm_fwd_fp8(x, gamma, eps=1e-6, hf_cast=False):
    y, rstd = E.rmsnorm_fwd(x, gamma, eps, hf_cast, save_stats=True)
    return R.quantize_act(y.reshape(-1, x.shape[-1])), rstd


def swiglu_bwd_fp8(dout, gate, up, dgate, dup):
    E.swiglu_bwd(dout, gate, up, dgate, dup)
    return quantize_dgu(dgate, dup)


def install(monkeypatch):
    """The FP8 inference stand-ins of fp8_reference.py plus the three training ones."""
    from cambrian_b200 import ops
    R.install(monkeypatch)
    for n in ("fp8_quantize_weight_t", "rmsnorm_fwd_fp8", "swiglu_bwd_fp8"):
        monkeypatch.setattr(ops, n, globals()[n])
