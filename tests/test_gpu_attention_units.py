"""The wgmma attention kernel (head_dim 64, 129..257 tokens) over many (image, head) units per persistent CTA.

Each CTA loops over its units through a two-stage shared-memory ring whose barriers flip phase every second unit, while the two
consumer warpgroups hand the tensor cores back and forth and three warps share query row 256.  test_gpu_attention.py's persistent
grid test reaches three units per CTA; these run enough units that every stage passes every barrier phase several times.

* selection inputs (one-hot softmax) at 2..9 units per CTA must return V[pi(i)] bit for bit;
* the bench shape (264 images x 257 tokens x 16 heads: 32 units per CTA on 132 SMs) against the mma.sync kernel, both within
  oracle/attention.py's bound of the float64 reference, and bitwise equal over repeat launches.
"""

from __future__ import annotations

import pytest
import torch

from gpu_helpers import ctx  # noqa: F401
from oracle import attention as A
from test_gpu_attention import _kernel, _run, _selection

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("t", [129, 193, 256, 257])
def test_wgmma_selection_many_units_per_cta(ctx, monkeypatch, t):
    _kernel(monkeypatch, False)
    s = ctx.device_info()["sm_count"]
    for per_cta in (2, 4, 5, 9):
        heads = 4
        units = per_cta * s - 1  # the last CTA runs one unit fewer than the others
        n = (units + heads - 1) // heads
        _selection(ctx, n, t, heads, 64, seed=per_cta * 1000 + t, what=f"T={t} ~{per_cta} units per CTA")


def test_wgmma_bench_shape_against_mma(ctx, monkeypatch):
    n, t, heads = 264, 257, 16
    qkv = A.random_inputs(n, t, heads, 64, seed=264).cuda()
    _kernel(monkeypatch, False)
    tc = _run(ctx, qkv, heads)
    for _ in range(2):
        assert torch.equal(tc, _run(ctx, qkv, heads)), "repeat launches differ"
    _kernel(monkeypatch, True)
    mma = _run(ctx, qkv, heads)
    for i in range(0, n, 66):  # the float64 reference in slices of images keeps its memory small
        sl = slice(i, i + 66)
        ref, s_abs = A.reference(qkv[sl], heads)
        bnd = A.bound(ref, s_abs, qkv[sl], heads)
        for name, got in (("wgmma", tc[sl]), ("mma", mma[sl])):
            ratio = ((got.double() - ref).abs() / bnd).max().item()
            assert ratio <= 1.0, f"{name} images {i}..{i + 65}: err/bound {ratio:.3f}"
