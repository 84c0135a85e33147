"""Shared helpers for the GPU parity tests."""

from __future__ import annotations

import numpy as np
import pytest
import torch


@pytest.fixture(scope="module")
def ctx():
    from cosmos_curate_b200.runtime import Context

    c = Context(0)
    yield c
    c.close()


def nv12_pool(ctx, frames_nv12, width: int, height: int, pitch: int, luma_rows: int, colour: str = "opencv"):
    rows = luma_rows + height // 2
    buf = np.zeros((len(frames_nv12), rows, pitch), dtype=np.uint8)
    for i, f in enumerate(frames_nv12):
        buf[i, :height, :width] = f[:height, :width]
        buf[i, luma_rows : luma_rows + height // 2, :width] = f[height:, :width]
    t = torch.from_numpy(buf).cuda()
    return ctx.nv12_pool(t, width, height, luma_rows, colour=colour)


def u8_budget(got: np.ndarray, want: np.ndarray, frac: float = 1e-4):
    d = np.abs(got.astype(np.int16) - want.astype(np.int16))
    assert d.max() <= 1, f"max diff {d.max()}"
    assert (d > 0).mean() <= frac, f"{(d > 0).mean():.2e} of pixels differ"


def assert_typed_outputs_are_lut_of(ctx, pool, res: int, u8: np.ndarray, slots=None, patches=((14, 640), (16, 768))):
    """The typed NCHW output (fp32) and the fp16 / bf16 patch rows of cb_preprocess_clip are exactly LUT(u8) of the u8 image `u8` of the
    same call: both resample kernels share the normalise/pack step."""
    from oracle import preprocess

    lut = preprocess.normalize_lut()
    want32 = np.stack([lut[c][u8[:, c]] for c in range(3)], axis=1)
    np.testing.assert_array_equal(ctx.preprocess_clip(pool, slots=slots, res=res, dtype=torch.float32).cpu().numpy(), want32)
    for patch, k_pad in patches:
        gp = ctx.preprocess_clip(pool, slots=slots, res=res, dtype=torch.float16, layout="patch", patch=patch, k_pad=k_pad).cpu().numpy()
        np.testing.assert_array_equal(gp, preprocess.to_patches(want32.astype(np.float16), patch, k_pad))
        gb = ctx.preprocess_clip(pool, slots=slots, res=res, dtype=torch.bfloat16, layout="patch", patch=patch, k_pad=k_pad).float().cpu().numpy()
        want_bf = torch.from_numpy(want32).to(torch.bfloat16).float().numpy()
        np.testing.assert_array_equal(gb, preprocess.to_patches(want_bf, patch, k_pad))
