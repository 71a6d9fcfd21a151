"""Kernel-level GPU parity tests, called through the C ABI (ctypes): every case compares one hand-written sm_90a kernel
with a plain PyTorch fp32 reference of the same op on seeded inputs.  The case tables live in tools/probe1.py /
tools/probe2.py (they print one line per case, which doubles as the profiling log); a case that misses its tolerance
prints FAIL.  Tolerances: GEMM with fp32 output 2e-5 relative (north_star's rtol 1e-3 / atol 1e-5 with margin); bf16 outputs
1e-2 .. 2e-2 of the tensor's max (one to two bf16 ulps of accumulated rounding)."""
import os
import sys

import pytest

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))


def _run(mod, group, capsys, min_ok):
    m = __import__(mod)
    getattr(m, "group_" + group)()
    out = capsys.readouterr().out
    sys.stdout.write(out)
    assert "FAIL" not in out, out
    assert out.count(" OK") >= min_ok, f"expected at least {min_ok} passing cases\n{out}"


def test_gemm_all_layouts_and_tiles(capsys):
    _run("probe1", "gemm_basic", capsys, 12)


def test_gemm_shapes_tails_batched(capsys):
    _run("probe1", "gemm_shapes", capsys, 25)


def test_gemm_epilogues(capsys):
    _run("probe1", "gemm_epi", capsys, 10)


def test_decode_gemv(capsys):
    _run("probe1", "gemv", capsys, 6)


def test_gemm_fused_gate_up_swiglu(capsys):
    _run("probe1", "gemm_swiglu", capsys, 5)


def test_sva_window_attention_fwd_bwd(capsys):
    _run("probe1", "sva", capsys, 4)


def test_layernorm_rmsnorm_fwd_bwd(capsys):
    _run("probe1", "norm", capsys, 19)


def test_elementwise_family(capsys):
    _run("probe2", "elem", capsys, 23)


def test_flash_attention_forward(capsys):
    _run("probe2", "attn_fwd", capsys, 9)


def test_flash_attention_backward(capsys):
    _run("probe2", "attn_bwd", capsys, 7)


def test_full_size_properties():
    """Size-independent properties at BASELINE's full shapes (no oracle needed):
    linearity of the GEMM, softmax rows of the SVA kernel summing to one (V = 1 -> out = 1), attention with a single
    visible key returning that key's value."""
    import torch
    from cambrian_b200 import ops
    dev = "cuda"
    torch.manual_seed(0)
    a = torch.randn(4608, 4096, device=dev).bfloat16()
    w = torch.randn(14336, 4096, device=dev).bfloat16() * 0.02
    y1 = ops.gemm(a, w, out_dtype=torch.float32)
    y2 = ops.gemm(a, w, out_dtype=torch.float32, alpha=2.0)
    assert torch.allclose(y2, 2 * y1, rtol=1e-6, atol=1e-6)
    y3 = ops.gemm(a, w, out_dtype=torch.float32, out=y1.clone(), accumulate=True)
    assert torch.allclose(y3, 2 * y1, rtol=1e-5, atol=1e-5)
    # SVA, release grids [576,576,576,9216], batch 4
    B, q, rs = 4, 24, [1, 1, 1, 4]
    n = B * q * q
    qq = torch.randn(n, 1024, device=dev).bfloat16()
    ks = [torch.randn(B, (r * q) ** 2, 1024, device=dev).bfloat16() for r in rs]
    ones = [torch.ones_like(k) for k in ks]
    out, _ = ops.sva_window_attn_fwd(qq, ks, ones, None, rs, B, q)
    assert torch.allclose(out.float(), torch.ones_like(out).float(), atol=1e-2)
    # causal attention, S = 2048: the first query sees only key 0
    S, nh, nkv, hd = 2048, 32, 8, 128
    qkv = torch.randn(1, S, (nh + 2 * nkv) * hd, device=dev).bfloat16()
    qv = qkv[..., : nh * hd].view(1, S, nh, hd)
    kv = qkv[..., nh * hd:(nh + nkv) * hd].view(1, S, nkv, hd)
    vv = qkv[..., (nh + nkv) * hd:].view(1, S, nkv, hd)
    o = ops.attn_fwd(qv, kv, vv, causal=True)
    assert torch.equal(o[0, 0], vv[0, 0].repeat_interleave(nh // nkv, 0))


@pytest.mark.parametrize("hw,R", [((480, 640), 336), ((700, 300), 384), ((90, 130), 336), ((336, 336), 336),
                                  ((1500, 1100), 1024)])
def test_gpu_preprocess_matches_pillow_bit_exact(hw, R):
    """cb_preprocess_image vs the reference's host chain (mm_utils.py:186-201): expand2square -> PIL resize (bicubic,
    uint8) is reproduced bit for bit; the normalised bf16 tensor matches (x/255 - mean)/std to bf16 rounding."""
    import numpy as np
    import torch
    from PIL import Image
    from cambrian_b200 import ops
    rng = np.random.default_rng(hw[0] + R)
    arr = rng.integers(0, 256, size=(hw[0], hw[1], 3), dtype=np.uint8)
    mean, std = (0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711)
    pad = tuple(int(x * 255) for x in mean)
    img = Image.fromarray(arr)
    w, h = img.size
    if w != h:
        s = max(w, h)
        sq = Image.new(img.mode, (s, s), pad)
        sq.paste(img, (0, (w - h) // 2) if w > h else ((h - w) // 2, 0))
        img = sq
    want_u8 = np.asarray(img.resize((R, R)))
    out, u8 = ops.preprocess_image(torch.from_numpy(arr).cuda(), R, pad, mean, std, return_u8=True)
    assert np.array_equal(u8.cpu().numpy(), want_u8)
    want = (torch.from_numpy(want_u8).permute(2, 0, 1).float() / 255.0 - torch.tensor(mean).view(3, 1, 1)) / \
        torch.tensor(std).view(3, 1, 1)
    assert (out.float().cpu() - want).abs().max().item() <= 2 ** -7 * want.abs().max().item()


def test_process_images_returns_one_tensor_per_tower():
    import numpy as np
    import torch
    from cambrian_b200.model.multimodal_encoder.towers import SimpleImageProcessor
    from cambrian_b200.preprocess import process_images
    procs = [SimpleImageProcessor(384, (0.5, 0.5, 0.5), (0.5, 0.5, 0.5)),
             SimpleImageProcessor(336, (0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711))]
    rng = np.random.default_rng(0)
    imgs = [rng.integers(0, 256, size=(200, 320, 3), dtype=np.uint8), rng.integers(0, 256, size=(500, 400, 3), dtype=np.uint8)]
    outs = process_images(imgs, procs)
    assert [tuple(o.shape) for o in outs] == [(2, 3, 384, 384), (2, 3, 336, 336)]
    assert all(o.dtype == torch.bfloat16 and o.is_cuda and torch.isfinite(o.float()).all() for o in outs)


@pytest.mark.parametrize("h,th,C", [(2, 4, 256), (12, 24, 1024), (24, 12, 1024), (27, 24, 1152), (5, 3, 64)])
def test_bilinear_backward_is_the_adjoint_of_the_forward(h, th, C):
    """cb_bilinear_bwd (the query-grid resize of cambrian_arch.py:394-401 under training) vs torch autograd through
    F.interpolate(bilinear, align_corners=False), and <bilinear(x), g> == <x, bilinear_bwd(g)> on the kernels themselves."""
    import torch
    import torch.nn.functional as F
    from cambrian_b200 import ops
    torch.manual_seed(0)
    B = 2
    x = torch.randn(B, h * h, C, device="cuda").bfloat16()
    g = torch.randn(B, th * th, C, device="cuda").bfloat16()
    xf = x.float().view(B, h, h, C).permute(0, 3, 1, 2).requires_grad_()
    y = F.interpolate(xf, size=(th, th), mode="bilinear", align_corners=False)
    (gx,) = torch.autograd.grad(y, xf, g.float().view(B, th, th, C).permute(0, 3, 1, 2))
    ref = gx.permute(0, 2, 3, 1).reshape(B, h * h, C)
    got = ops.bilinear_bwd(g, h, h, th, th)
    torch.cuda.synchronize()
    err = ((got.float() - ref).abs().max() / ref.abs().max()).item()
    assert err < 6e-3, err           # one bf16 rounding of the fp32 sum
    fwd = ops.bilinear(x, h, h, th, th)
    lhs, rhs = (fwd.float() * g.float()).sum().item(), (x.float() * got.float()).sum().item()
    assert abs(lhs - rhs) <= 2e-2 * max(abs(lhs), abs(rhs), 1.0), (lhs, rhs)


@pytest.mark.parametrize("T,N,C", [(1, 37, 1024), (4, 300, 1024), (8, 64, 256)])
def test_tower_combine_forward_backward(T, N, C):
    """cb_tower_combine_fwd / _bwd (softmax over towers + weighted sum + residual, vision_sampler.py:367-368, :394-396) vs
    fp32 torch autograd."""
    import torch
    from cambrian_b200 import ops
    torch.manual_seed(0)
    logits = torch.zeros(N, 8, device="cuda").bfloat16()
    logits[:, :T] = (torch.randn(N, T, device="cuda") * 2).bfloat16()
    aggs = [torch.randn(N, C, device="cuda").bfloat16() for _ in range(T)]
    qin = torch.randn(N, C, device="cuda").bfloat16()
    dout = torch.randn(N, C, device="cuda").bfloat16()
    lf = logits.float()[:, :T].clone().requires_grad_()
    af = [a.float().requires_grad_() for a in aggs]
    w = torch.softmax(lf, -1)
    ref = qin.float() + sum(w[:, t:t + 1] * af[t] for t in range(T))
    grads = torch.autograd.grad(ref, [lf, *af], dout.float())
    out = ops.tower_combine_fwd(logits, aggs, qin)
    daggs, dlogits = ops.tower_combine_bwd(logits, aggs, dout)
    torch.cuda.synchronize()

    def e(a, b):
        return ((a.float() - b).abs().max() / (b.abs().max() + 1e-6)).item()

    assert e(out, ref) < 6e-3, e(out, ref)
    for t in range(T):
        assert e(daggs[t], grads[1 + t]) < 6e-3, (t, e(daggs[t], grads[1 + t]))
    if T > 1:
        assert e(dlogits[:, :T], grads[0]) < 1e-2, e(dlogits[:, :T], grads[0])
    else:
        assert float(dlogits.float().abs().max()) < 1e-3
    assert float(dlogits[:, T:].float().abs().max()) == 0.0 if T < 8 else True
