"""The GEMM epilogue (shared-memory slices written back by TMA stores, residual read by TMA loads): the tower's own shapes, outputs
inside larger buffers (nothing outside [M][N] is written), M tails just past a tile boundary for both tile widths, and repeat
launches being bitwise equal."""

from __future__ import annotations

import pytest
import torch

from gpu_helpers import ctx  # noqa: F401

pytestmark = pytest.mark.gpu

EPI_NONE, EPI_QUICK_GELU, EPI_GELU_TANH = 0, 1, 2
M_TOWER = 264 * 257  # 264 frames x 257 tokens


def _act(z, epi):
    if epi == EPI_QUICK_GELU:
        return z * torch.sigmoid(1.702 * z)
    if epi == EPI_GELU_TANH:
        return torch.nn.functional.gelu(z, approximate="tanh")
    return z


def _operands(m, n, k, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = (torch.randn(m, k, device="cuda", generator=g) * 0.5).half()
    w = (torch.randn(n, k, device="cuda", generator=g) * 0.5).half()
    bias = torch.randn(n, device="cuda", generator=g)
    return a, w, bias, g


def _gemm_into(ctx, out, a, w, bias, residual, epi):
    """cb_gemm_f16 writing into `out`, a contiguous [M][N] view that may sit inside a larger buffer."""
    from cosmos_curate_b200.runtime import _stream_ptr, check

    m, k = a.shape
    n = w.shape[0]
    o32, o16 = (out.data_ptr(), None) if out.dtype == torch.float32 else (None, out.data_ptr())
    rc = ctx.lib.cb_gemm_f16(ctx.h, a.data_ptr(), w.data_ptr(), bias.data_ptr() if bias is not None else None,
                             residual.data_ptr() if residual is not None else None, o32, o16, m, n, k, epi, _stream_ptr())  # fmt: skip
    check(rc, "cb_gemm_f16", ctx.h)


def _guarded(ctx, a, w, bias, epi, out_f32, residual=None, seed=0):
    """Run with the output at a row offset inside a sentinel-filled buffer followed by a neighbouring matrix of other width;
    assert nothing outside [M][N] changed and return the output."""
    m, n = a.shape[0], w.shape[0]
    dt = torch.float32 if out_f32 else torch.float16
    pre, post = 3 * n + 8, 37 * 24  # elements before (3 rows and a bit: keeps 16-byte alignment) and after the output
    g = torch.Generator(device="cuda").manual_seed(seed)
    buf = torch.randn(pre + m * n + post, device="cuda", generator=g).to(dt)
    before = buf.clone()
    out = buf[pre : pre + m * n].view(m, n)
    if residual is not None:
        out.copy_(residual)
        before = buf.clone()
    _gemm_into(ctx, out, a, w, bias, out if residual is not None else None, epi)
    torch.cuda.synchronize()
    assert torch.equal(buf[:pre], before[:pre]), "rows before the output were written"
    assert torch.equal(buf[pre + m * n :], before[pre + m * n :]), "the neighbouring matrix after the output was written"
    return out


def _check_f16(got, want):
    err = (got.float() - want).abs().max().item()
    assert err <= 2e-3 * want.abs().max().item() + 1e-2, err  # tolerance of test_gemm_plain


def _check_f32(got, want):
    torch.testing.assert_close(got, want, rtol=1e-4, atol=2e-3)  # tolerance of test_gemm_with_tails


# name, N, K, output, epilogue, residual: every GEMM of a CLIP ViT-L/14 layer and the two of SigLIP's MLP
TOWER = [
    ("qkv", 3072, 1024, "f16", EPI_NONE, False),
    ("out_proj", 1024, 1024, "f32", EPI_NONE, True),
    ("fc1", 4096, 1024, "f16", EPI_QUICK_GELU, False),
    ("fc2", 1024, 4096, "f32", EPI_NONE, True),
    ("siglip_fc1", 4304, 1152, "f16", EPI_GELU_TANH, False),
    ("siglip_fc2", 1152, 4304, "f32", EPI_NONE, True),
]


@pytest.mark.parametrize(("name", "n", "k", "out", "epi", "res"), TOWER, ids=[t[0] for t in TOWER])
def test_gemm_tower_shapes(ctx, name, n, k, out, epi, res):
    m = M_TOWER
    a, w, bias, g = _operands(m, n, k, seed=n + k)
    z = torch.addmm(bias, a.float(), w.float().t())
    if out == "f16":
        _check_f16(_guarded(ctx, a, w, bias, epi, False), _act(z, epi))
    else:
        r = torch.randn(m, n, device="cuda", generator=g) if res else None
        got = _guarded(ctx, a, w, bias, epi, True, residual=r)
        _check_f32(got, z + r if res else z)


@pytest.mark.parametrize("tail", [1, 8, 63, 65])
@pytest.mark.parametrize("n", [640, 1024, 136])  # 640 / 136: 128-wide tiles; 1024 at these M: 256-wide tiles
def test_gemm_m_tails(ctx, n, tail):
    m, k = 128 * 40 + tail, 192
    a, w, bias, g = _operands(m, n, k, seed=tail * 31 + n)
    z = torch.addmm(bias, a.float(), w.float().t())
    _check_f16(_guarded(ctx, a, w, bias, EPI_QUICK_GELU, False, seed=1), _act(z, EPI_QUICK_GELU))
    _check_f16(_guarded(ctx, a, w, None, EPI_NONE, False, seed=2), z - bias)
    r = torch.randn(m, n, device="cuda", generator=g)
    _check_f32(_guarded(ctx, a, w, bias, EPI_NONE, True, residual=r, seed=3), z + r)
    _check_f32(_guarded(ctx, a, w, bias, EPI_NONE, True, seed=4), z)


@pytest.mark.parametrize(("m", "n", "k"), [(M_TOWER, 1024, 1024), (5000, 640, 320), (1000, 1000, 264)])
def test_gemm_repeat_launches_bitwise_equal(ctx, m, n, k):
    a, w, bias, g = _operands(m, n, k, seed=m)
    r = torch.randn(m, n, device="cuda", generator=g)
    first16 = ctx.gemm(a, w, bias=bias, epilogue=EPI_QUICK_GELU)
    first32 = ctx.gemm(a, w, bias=bias, residual=r.clone(), out_f32=True)
    for _ in range(3):
        assert torch.equal(first16, ctx.gemm(a, w, bias=bias, epilogue=EPI_QUICK_GELU))
        assert torch.equal(first32, ctx.gemm(a, w, bias=bias, residual=r.clone(), out_f32=True))


def test_gemm_residual_separate_from_output(ctx):
    """residual and output need not alias: the residual is read from its own tensor and left as it was."""
    m, n, k = 3000, 1024, 256
    a, w, bias, g = _operands(m, n, k, seed=5)
    r = torch.randn(m, n, device="cuda", generator=g)
    r_before = r.clone()
    out = torch.full((m, n), float("nan"), device="cuda")
    _gemm_into(ctx, out, a, w, bias, r, EPI_NONE)
    torch.cuda.synchronize()
    assert torch.equal(r, r_before)
    _check_f32(out, torch.addmm(bias, a.float(), w.float().t()) + r)
