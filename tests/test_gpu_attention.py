"""Attention (cb_attention_f16) against oracle/attention.py at every dispatch boundary of both kernels.

* exact: selection inputs (one-hot softmax) must return V[pi(i)] bit for bit, uniform inputs the per-image constant bit for bit;
* bounded: random inputs (plain, sharp rows, logits ~10^3, exact ties) within the per-element bound of the kernels' own rounding;
* every call runs with the input between NaN rows and the output inside a sentinel-filled buffer: nothing past the input may be
  read, nothing outside [n*T][hidden] written;
* an image's output does not depend on its neighbour, even one full of Inf and NaN;
* the wgmma kernel's persistent grid just under, at and over the SM count; repeat launches; the error codes.

Shapes the wgmma kernel takes run on both kernels (CB_ATTN_KERNEL=mma is read on every call and forces the mma.sync kernel).
"""

from __future__ import annotations

import pytest
import torch

from gpu_helpers import ctx  # noqa: F401
from oracle import attention as A

pytestmark = pytest.mark.gpu

PAD = 3  # NaN rows before and after the input, sentinel rows before and after the output
SENTINEL = -7777.0
KINDS = ("normal", "sharp", "large", "ties")


def _call(ctx, qkv_ptr, out_ptr, n, t, heads, hd) -> int:
    from cosmos_curate_b200.runtime import _stream_ptr

    return ctx.lib.cb_attention_f16(ctx.h, qkv_ptr, out_ptr, n, t, heads, hd, _stream_ptr())


def _run(ctx, qkv: torch.Tensor, heads: int) -> torch.Tensor:
    """cb_attention_f16 on qkv [n][T][3 * hidden] placed between NaN rows, writing into a sentinel-filled buffer; asserts nothing
    outside the output was written and returns the output [n][T][hidden]."""
    from cosmos_curate_b200.runtime import check

    n, t, three_hidden = qkv.shape
    hidden, rows = three_hidden // 3, n * t
    src = torch.full((rows + 2 * PAD, three_hidden), float("nan"), dtype=torch.float16, device="cuda")
    src[PAD : PAD + rows] = qkv.reshape(rows, three_hidden)
    dst = torch.full((rows + 2 * PAD, hidden), SENTINEL, dtype=torch.float16, device="cuda")
    check(_call(ctx, src[PAD:].data_ptr(), dst[PAD:].data_ptr(), n, t, heads, hidden // heads), "cb_attention_f16", ctx.h)
    torch.cuda.synchronize()
    assert (dst[:PAD] == SENTINEL).all() and (dst[PAD + rows :] == SENTINEL).all(), "rows outside [n*T][hidden] were written"
    return dst[PAD : PAD + rows].view(n, t, hidden)


def _kernel(monkeypatch, force_mma: bool) -> None:
    if force_mma:
        monkeypatch.setenv("CB_ATTN_KERNEL", "mma")
    else:
        monkeypatch.delenv("CB_ATTN_KERNEL", raising=False)


def _assert_bitwise(got: torch.Tensor, want: torch.Tensor, what: str) -> None:
    bad = (got.view(torch.int16) != want.view(torch.int16)).nonzero()
    if len(bad):
        img, tok, col = bad[0].tolist()
        pytest.fail(f"{what}: {len(bad)} elements differ; first at image {img} token {tok} column {col}: "
                    f"got {got[img, tok, col].item()} want {want[img, tok, col].item()}")  # fmt: skip


def _selection(ctx, n, t, heads, hd, seed, what):
    qkv, pi = A.selection_inputs(n, t, heads, hd, seed)
    _, _, v = A.split_heads(qkv, heads)
    want = A.merge_heads(torch.gather(v, 2, pi[..., None].expand(-1, -1, -1, hd)))
    _assert_bitwise(_run(ctx, qkv.cuda(), heads), want.cuda(), f"selection {what}")


# every row of the dispatch table gets the swept shapes that land on it; shapes the wgmma kernel takes also run forced onto mma.sync
CASES = sorted({(p.name, t, hd, force) for p in A.PATHS for hd in p.head_dims for t in A.SWEEP_T for force in (False, True)
                if A.table_path(t, hd, force) == p.name and (not force or A.table_path(t, hd, False) != p.name)})  # fmt: skip


def test_cases_cover_every_path():
    assert {c[0] for c in CASES} == {p.name for p in A.PATHS}


@pytest.fixture(scope="module")
def worst():
    """Worst err/bound per path over the random inputs, printed when the module ends."""
    w: dict[str, float] = {}
    yield w
    for name, r in sorted(w.items()):
        print(f"\nattention {name}: worst err/bound {r:.3f}", end="")
    print()


@pytest.mark.parametrize(("path", "t", "hd", "force"), CASES, ids=[f"{c[0]}{'-forced' if c[3] else ''}-T{c[1]}-hd{c[2]}" for c in CASES])
def test_attention_sweep(ctx, monkeypatch, worst, path, t, hd, force):
    _kernel(monkeypatch, force)
    n, heads = (2, 2) if t < 1000 else (1, 2)
    seed = t * 100 + hd
    _selection(ctx, n, t, heads, hd, seed, path)

    qkv, c = A.uniform_inputs(n, t, heads, hd, seed)
    want = A.merge_heads(c[:, :, None, :].expand(n, heads, t, hd)).half()
    _assert_bitwise(_run(ctx, qkv.cuda(), heads), want.cuda(), f"uniform {path}")

    for kind in KINDS:
        qkv = A.random_inputs(n, t, heads, hd, seed, kind=kind).cuda()
        got = _run(ctx, qkv, heads).double()
        ref, s_abs = A.reference(qkv, heads)
        ratio = ((got - ref).abs() / A.bound(ref, s_abs, qkv, heads)).max().item()
        worst[path] = max(worst.get(path, 0.0), ratio)
        assert ratio <= 1.0, f"{kind}: err/bound {ratio:.3f}"


@pytest.mark.parametrize("t", [129, 200, 256, 257])
def test_wgmma_persistent_grid(ctx, monkeypatch, t):
    """n * heads units over min(units, SMs) persistent CTAs: one unit, just under, at and over one and two waves."""
    _kernel(monkeypatch, False)
    s = ctx.device_info()["sm_count"]
    for units in (1, s - 1, s, s + 1, 2 * s, 2 * s + 1):
        heads = 2 if units % 2 == 0 else 1
        _selection(ctx, units // heads, t, heads, 64, seed=units + t, what=f"T={t} units={units}")


POISON = [(t, 64, False) for t in (129, 200, 255, 256, 257)] + [(t, 64, True) for t in (129, 200, 255, 256, 257)] + [
    (50, 64, False), (200, 32, False), (288, 80, False), (600, 64, False), (729, 72, False)]  # fmt: skip


@pytest.mark.parametrize(("t", "hd", "force"), POISON, ids=[f"{A.path_of(t, hd, f)}{'-forced' if f else ''}-T{t}-hd{hd}" for t, hd, f in POISON])
def test_poisoned_neighbour(ctx, monkeypatch, t, hd, force):
    """Image 1 is Inf and NaN in Q, K and V: images 0 and 2 stay finite and equal, bit for bit, to runs of each image alone."""
    _kernel(monkeypatch, force)
    heads = 3
    qkv = A.random_inputs(3, t, heads, hd, seed=t + hd).cuda()
    pattern = torch.tensor([float("inf"), float("nan"), float("-inf")], dtype=torch.float16, device="cuda")
    qkv[1] = pattern[torch.arange(qkv.shape[2], device="cuda") % 3]
    out = _run(ctx, qkv, heads)
    for b in (0, 2):
        assert torch.isfinite(out[b]).all(), f"image {b} has non-finite outputs next to a poisoned image"
        _assert_bitwise(out[b : b + 1], _run(ctx, qkv[b : b + 1].clone(), heads), f"image {b} next to a poisoned image vs alone")


@pytest.mark.parametrize(("n", "t", "heads", "hd"), [(3, 257, 16, 64), (2, 50, 12, 64), (2, 200, 4, 72), (1, 729, 4, 72), (2, 600, 4, 64)])
def test_mma_repeat_launches_bitwise_equal(ctx, monkeypatch, n, t, heads, hd):
    _kernel(monkeypatch, True)
    qkv = A.random_inputs(n, t, heads, hd, seed=n * t, kind="sharp").cuda()
    first = _run(ctx, qkv, heads)
    for _ in range(3):
        assert torch.equal(first, _run(ctx, qkv, heads))


@pytest.mark.parametrize("hd", [8, 12, 88])
def test_unsupported_head_dim(ctx, hd):
    t, heads = 100, 2
    qkv = torch.zeros(t, 3 * heads * hd, dtype=torch.float16, device="cuda")
    out = torch.full((t, heads * hd), SENTINEL, dtype=torch.float16, device="cuda")
    assert _call(ctx, qkv.data_ptr(), out.data_ptr(), 1, t, heads, hd) == -3  # CB_ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert (out == SENTINEL).all()


@pytest.mark.parametrize("t", [50, 257])
def test_zero_images_is_a_no_op(ctx, t):
    heads, hd = 2, 64
    qkv = torch.full((t, 3 * heads * hd), float("nan"), dtype=torch.float16, device="cuda")
    out = torch.full((t, heads * hd), SENTINEL, dtype=torch.float16, device="cuda")
    assert _call(ctx, qkv.data_ptr(), out.data_ptr(), 0, t, heads, hd) == 0
    torch.cuda.synchronize()
    assert (out == SENTINEL).all()
