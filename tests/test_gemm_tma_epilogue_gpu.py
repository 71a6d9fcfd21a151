"""The GEMM's two bf16 store paths and its persistent tile loop.

A bf16 output whose base is 16-byte aligned with row / batch strides that are multiples of 8 elements is written by TMA
stores from a shared-memory staging tile; any other bf16 output is written from registers.  Both paths run the same
fp32 epilogue arithmetic, so they must agree bit for bit, including in M and N tails at every tile width.  Each CTA
walks a strided list of tiles, so a batched problem with more than twice as many tiles as SMs has CTAs crossing batch
boundaries; its batches must equal the same problems launched one by one."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _operands(M, N, K, batch=0, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    lead = (batch,) if batch else ()
    a = torch.randn(*lead, M, K, generator=g, device=DEV).bfloat16()
    b = (torch.randn(*lead, N, K, generator=g, device=DEV) * K ** -0.5).bfloat16()
    return a, b


def _register_path_out(M, N, kind):
    """An [M, N] bf16 view that TMA cannot address: base one element past an aligned address, or row stride N + 2."""
    if kind == "offset":
        return torch.zeros(M * N + 1, dtype=torch.bfloat16, device=DEV)[1:].view(M, N)
    return torch.zeros(M, N + 2, dtype=torch.bfloat16, device=DEV)[:, :N]


# M and N tails at every tile width: 1000 = 7 x 128 + 104 rows, 200 = 3 x 64 + 8 = 128 + 72 columns (< 256)
@pytest.mark.parametrize("kind", ["offset", "ldc"])
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_register_path_matches_tma_path_bitwise(bn, kind):
    from cambrian_b200 import ops
    M, N, K = 1000, 200, 320
    a, b = _operands(M, N, K, seed=7)
    bias = torch.randn(N, device=DEV).bfloat16()
    ls = torch.rand(N, device=DEV).bfloat16()
    res = torch.randn(M, N, device=DEV).bfloat16()
    kw = dict(bias=bias, act="gelu", colscale=ls, residual=res, force_bn=bn)
    tma = ops.gemm(a, b, **kw)
    assert tma.data_ptr() % 16 == 0 and tma.stride(0) % 8 == 0
    reg = ops.gemm(a, b, out=_register_path_out(M, N, kind), **kw)
    assert torch.equal(reg, tma)
    z = torch.nn.functional.gelu(a.double() @ b.double().t() + bias.double()) * ls.double() + res.double()
    err = (tma.double() - z).abs().max().item()
    assert err <= 1e-2 * z.abs().max().item()


@pytest.mark.parametrize("kind", ["offset", "ldc"])
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_accumulate_register_path_matches_tma_path_bitwise(bn, kind):
    """dW layout accumulated into a bf16 gradient with M and N tails."""
    from cambrian_b200 import ops
    M, N, K = 1000, 200, 1000
    g = torch.Generator(device=DEV).manual_seed(8)
    a = torch.randn(K, M, generator=g, device=DEV).bfloat16()
    b = (torch.randn(K, N, generator=g, device=DEV) * K ** -0.5).bfloat16()
    c0 = torch.randn(M, N, generator=g, device=DEV).bfloat16()
    tma = ops.gemm(a, b, a_mn=True, b_mn=True, out=c0.clone(), accumulate=True, force_bn=bn)
    reg = _register_path_out(M, N, kind)
    reg.copy_(c0)
    ops.gemm(a, b, a_mn=True, b_mn=True, out=reg, accumulate=True, force_bn=bn)
    assert torch.equal(reg, tma)
    want = c0.double() + a.double().t() @ b.double()
    assert (tma.double() - want).abs().max().item() <= 1e-2 * want.abs().max().item()


@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_batched_tiles_cross_batches(bn, out_dtype):
    """3 batches of 9 m-blocks x 2048 columns: at least 3 x 9 x 8 = 216 tiles, and 864 at BN = 64, against 132 SMs."""
    from cambrian_b200 import ops
    a, b = _operands(1144, 2048, 192, batch=3, seed=9)
    res = torch.randn(3, 1144, 2048, device=DEV).bfloat16()
    full = ops.gemm(a, b, residual=res, out_dtype=out_dtype, force_bn=bn)
    for i in range(3):
        assert torch.equal(ops.gemm(a[i], b[i], residual=res[i], out_dtype=out_dtype, force_bn=bn), full[i]), i


def test_swiglu_more_tiles_than_sms():
    """65 m-blocks (an M tail of 40 rows) x 8 feature tiles = 520 tiles, about 4 per CTA."""
    from cambrian_b200 import ops
    M, F, K = 8192 + 40, 1024, 256
    x, w = _operands(M, 2 * F, K, seed=10)
    gu, act = ops.gemm_swiglu(x, w)
    want = x.double() @ w.double().t()
    assert (gu.double() - want).abs().max().item() <= 1e-2 * want.abs().max().item()
    g, u = gu[:, :F].float(), gu[:, F:].float()
    want_act = (g * torch.sigmoid(g) * u).double()
    assert (act.double() - want_act).abs().max().item() <= 2e-2 * want_act.abs().max().item()
    gu_p, act_p = ops.gemm_swiglu(x[-1000:], w)
    assert torch.equal(gu_p, gu[-1000:]) and torch.equal(act_p, act[-1000:])
