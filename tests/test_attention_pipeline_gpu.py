"""The flash-attention kernels' tile fast paths, heavy-first tile order and bf16 dQ store.

Tiles whose keys are all valid, inside Skv and below the causal diagonal skip the per-element masking, so an all-True key
mask must give exactly the kmask=None outputs.  Masked holes and padded tails must still match the fp32 reference at
sequence lengths that cut tiles, and with a key cache longer than the queries.  dQ is rounded to bf16 inside the dQ
kernel and stored straight into the caller's view, which may be the Q columns of a packed dQKV buffer.  Every output has
one writer, so two runs agree bit for bit, and the outputs equal the fingerprints that the build before these kernels
produced (tests/golden/attn_fingerprints.json, from tools/attn_step_shapes.py --hash on an H100)."""
import json
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

DEV = "cuda"
B, S, NH, NKV, HD = 4, 2048, 24, 8, 128


def _packed(Sq, Skv, nh, nkv, hd, seed, batch=B):
    g = torch.Generator(device=DEV).manual_seed(seed)
    q = torch.randn(batch, Sq, nh, hd, generator=g, device=DEV).bfloat16()
    k = torch.randn(batch, Skv, nkv, hd, generator=g, device=DEV).bfloat16()
    v = torch.randn(batch, Skv, nkv, hd, generator=g, device=DEV).bfloat16()
    do = torch.randn(batch, Sq, nh, hd, generator=g, device=DEV).bfloat16()
    return q, k, v, do


def _run(q, k, v, do, kmask, causal=True):
    from cambrian_b200 import ops
    o, lse = ops.attn_fwd(q, k, v, causal=causal, kmask=kmask, need_lse=True)
    dq, dk, dv = ops.attn_bwd(q, k, v, o, do, lse, causal=causal, kmask=kmask)
    torch.cuda.synchronize()
    return dict(o=o, lse=lse, dq=dq, dk=dk, dv=dv)


def _bitwise_equal(a, b):
    for name in a:
        assert torch.equal(a[name].view(torch.int16) if a[name].dtype == torch.bfloat16 else a[name].view(torch.int32),
                           b[name].view(torch.int16) if b[name].dtype == torch.bfloat16 else b[name].view(torch.int32)), name


def test_all_true_kmask_equals_no_mask_bitwise():
    q, k, v, do = _packed(S, S, NH, NKV, HD, seed=1)
    ones = torch.ones(B, S, dtype=torch.bool, device=DEV)
    _bitwise_equal(_run(q, k, v, do, ones), _run(q, k, v, do, None))


@pytest.mark.parametrize("Sq,Skv", [(300, 300), (2048, 2048), (300, 428), (200, 2048)])
def test_masked_keys_match_fp32_reference(Sq, Skv):
    from probe2 import attn_ref, rel_err
    q, k, v, do = _packed(Sq, Skv, 8, 2, HD, seed=Sq + Skv, batch=3)
    kmask = torch.ones(3, Skv, dtype=torch.bool, device=DEV)
    kmask[0, Skv - 77:] = False              # padded tail keys
    kmask[1, Skv // 3:Skv // 3 + 150] = False  # a hole spanning a tile boundary
    got = _run(q, k, v, do, kmask)
    qf, kf, vf = (t.detach().float().requires_grad_() for t in (q, k, v))
    ref = attn_ref(qf, kf, vf, True, kmask)
    ref.backward(do.float())
    errs = [rel_err(got["o"], ref), rel_err(got["dq"], qf.grad), rel_err(got["dk"], kf.grad), rel_err(got["dv"], vf.grad)]
    assert all(e < 2e-2 for e in errs), errs


def test_two_runs_bitwise_equal():
    q, k, v, do = _packed(S, S, NH, NKV, HD, seed=2)
    kmask = torch.ones(B, S, dtype=torch.bool, device=DEV)
    kmask[2, 1500:] = False
    _bitwise_equal(_run(q, k, v, do, kmask), _run(q, k, v, do, kmask))


def test_dq_into_packed_view_leaves_kv_columns():
    from cambrian_b200 import ops
    q, k, v, do = _packed(S, S, NH, NKV, HD, seed=3)
    o, lse = ops.attn_fwd(q, k, v, causal=True, need_lse=True)
    dq_ref, _, _ = ops.attn_bwd(q, k, v, o, do, lse, causal=True)
    W = (NH + 2 * NKV) * HD
    sentinel = torch.randn(B * S, W, device=DEV).bfloat16()
    dqkv = sentinel.clone()
    dq = dqkv[:, : NH * HD].view(B, S, NH, HD)
    dk = torch.empty_like(k)
    dv = torch.empty_like(v)
    ops.attn_bwd(q, k, v, o, do, lse, causal=True, dq=dq, dk=dk, dv=dv)
    torch.cuda.synchronize()
    assert torch.equal(dqkv[:, NH * HD:], sentinel[:, NH * HD:])
    assert torch.equal(dq, dq_ref)


def test_outputs_match_fingerprints_of_previous_build():
    import attn_step_shapes as T
    with open(os.path.join(ROOT, "tests", "golden", "attn_fingerprints.json")) as f:
        want = json.load(f)
    rows = {name: s for name, _, s in T.step_shapes(want["config"])}
    assert set(rows) == set(want["shapes"])
    for name, s in rows.items():
        assert T.fingerprint(s, want["seed"]) == want["shapes"][name], name
