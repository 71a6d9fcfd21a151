"""The GEMM (cb_gemm_bf16 / cb_gemm_swiglu_bf16) against fp64 torch at shapes that exercise its tiling: fewer tiles than
SMs, tile counts that are not a multiple of the SM count, odd m-block counts, batched problems with an odd m-block count
per batch, every operand layout and tile width, the accumulate / residual / activation epilogues, and SwiGLU with an odd
number of 128-feature tiles.

Where a tile sits in the grid must not change any output bit: rows of one large GEMM are compared bitwise with the same
rows computed by smaller GEMMs, whose grids and tile assignments differ."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _operands(M, N, K, a_mn, b_mn, batch=0, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    lead = (batch,) if batch else ()
    a = torch.randn(*lead, *((K, M) if a_mn else (M, K)), generator=g, device=DEV).bfloat16()
    b = (torch.randn(*lead, *((K, N) if b_mn else (N, K)), generator=g, device=DEV) * K ** -0.5).bfloat16()
    return a, b


def _ref(a, b, a_mn, b_mn):
    a64, b64 = a.double(), b.double()
    return (a64.transpose(-1, -2) if a_mn else a64) @ (b64 if b_mn else b64.transpose(-1, -2))


def _close(got, want, rel):
    err = (got.double() - want).abs().max().item()
    scale = want.abs().max().item()
    assert err <= rel * scale, f"max error {err} vs {rel} x {scale}"


# (M, N, K), every row stride a multiple of 8 elements as TMA requires: tiles < SMs (1 and 2 m-blocks); 5, 9 and 33
# m-blocks (odd); tile counts that do not divide by the SM count; N and K tails
SHAPES = [(104, 72, 64), (256, 256, 64), (640, 320, 200), (1144, 520, 136), (4104, 2000, 320)]


@pytest.mark.parametrize("bn", [64, 128, 256])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_layouts_tiles_and_schedules(M, N, K, a_mn, b_mn, bn):
    from cambrian_b200 import ops
    a, b = _operands(M, N, K, a_mn, b_mn)
    want = _ref(a, b, a_mn, b_mn)
    _close(ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_dtype=torch.float32, force_bn=bn), want, 1e-5)
    _close(ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, force_bn=bn), want, 1e-2)


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M", [9 * 128 - 8, 128])
def test_batched_odd_m_blocks_per_batch(M, a_mn, b_mn):
    """9 m-blocks per batch: tiles index the right batch, and the last m-block of one batch stops at its M."""
    from cambrian_b200 import ops
    a, b = _operands(M, 264, 192, a_mn, b_mn, batch=3, seed=1)
    _close(ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_dtype=torch.float32), _ref(a, b, a_mn, b_mn), 1e-5)


@pytest.mark.parametrize("out_dtype,rel", [(torch.bfloat16, 1e-2), (torch.float32, 1e-5)])
@pytest.mark.parametrize("M", [1144, 4096])
def test_accumulate(M, out_dtype, rel):
    """dW layout (both operands MN-major) accumulated into an existing bf16 / fp32 gradient buffer."""
    from cambrian_b200 import ops
    a, b = _operands(M, 768, 1000, True, True, seed=2)
    c0 = torch.randn(M, 768, device=DEV).to(out_dtype)
    got = ops.gemm(a, b, a_mn=True, b_mn=True, out=c0.clone(), accumulate=True)
    _close(got, c0.double() + _ref(a, b, True, True), rel)


@pytest.mark.parametrize("act", [None, "gelu", "quick_gelu"])
@pytest.mark.parametrize("M", [2308, 2916])
def test_bias_activation_layerscale_residual(M, act):
    """The towers' MLP epilogues at their odd m-block counts (2308 rows = 19 m-blocks, 2916 = 23)."""
    from cambrian_b200 import ops
    N, K = 1024, 384
    a, b = _operands(M, N, K, False, False, seed=3)
    bias = torch.randn(N, device=DEV).bfloat16()
    ls = torch.rand(N, device=DEV).bfloat16()
    res = torch.randn(M, N, device=DEV).bfloat16()
    z = _ref(a, b, False, False) + bias.double()
    if act == "gelu":
        z = torch.nn.functional.gelu(z)
    elif act == "quick_gelu":
        z = z * torch.sigmoid(1.702 * z)
    want = z * ls.double() + res.double()
    got = ops.gemm(a, b, bias=bias, act=act, colscale=ls, residual=res, out_dtype=torch.float32)
    _close(got, want, 1e-4)


@pytest.mark.parametrize("M,F", [(1149, 384), (256, 640), (4096, 128 * 9)])
def test_swiglu_odd_feature_tiles(M, F):
    """Fused gate/up + SwiGLU with F / 128 odd: gate and up halves of each 128-feature tile come from rows f and F + f."""
    from cambrian_b200 import ops
    x, w = _operands(M, 2 * F, 512, False, False, seed=4)
    gu, act = ops.gemm_swiglu(x, w)
    want = _ref(x, w, False, False)
    _close(gu, want, 1e-2)
    g, u = gu[:, :F].float(), gu[:, F:].float()
    want_act = (g * torch.sigmoid(g) * u).double()
    _close(act, want_act, 2e-2)


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True)])
def test_rows_do_not_depend_on_the_schedule(a_mn, b_mn):
    """Rows of an M = 8192 GEMM (64 m-blocks, several waves) are bit-identical to the same rows computed by GEMMs of 384
    rows (3 m-blocks, fewer tiles than SMs) and 1152 rows (9 m-blocks)."""
    from cambrian_b200 import ops
    M, N, K = 8192, 1536, 1024
    a, b = _operands(M, N, K, a_mn, b_mn, seed=5)
    for bn in (64, 128, 256):
        full = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, force_bn=bn, out_dtype=torch.float32)
        for r0, m in ((0, 384), (1024, 1152), (8192 - 384, 384)):
            part = a[:, r0:r0 + m] if a_mn else a[r0:r0 + m]
            got = ops.gemm(part, b, a_mn=a_mn, b_mn=b_mn, force_bn=bn, out_dtype=torch.float32)
            assert torch.equal(got, full[r0:r0 + m]), (bn, r0, m)


def test_swiglu_rows_do_not_depend_on_the_schedule():
    from cambrian_b200 import ops
    x, w = _operands(8192, 2 * 1024, 768, False, False, seed=6)
    gu, act = ops.gemm_swiglu(x, w)
    for r0, m in ((0, 384), (2048, 1152)):
        gu_p, act_p = ops.gemm_swiglu(x[r0:r0 + m], w)
        assert torch.equal(gu_p, gu[r0:r0 + m]) and torch.equal(act_p, act[r0:r0 + m]), (r0, m)
