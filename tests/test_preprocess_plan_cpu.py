"""The preprocess plan oracle (oracle/preprocess_plan.py) against the sources, the library's own plan query, torchvision's size rules
and the numpy oracle; and proof that the sweep of tests/test_gpu_preprocess_sweep.py reaches every plan class of both kernels."""

from __future__ import annotations

import ctypes as C
from collections import defaultdict

import numpy as np
import pytest
import torch

from oracle import color, preprocess
from oracle import preprocess_plan as PP


def test_constants_read_from_the_sources_equal_the_oracle():
    assert PP.constants_from_source() == PP.K


def test_library_plan_equals_the_oracle_at_every_swept_point():
    """cb_preprocess_plan touches no device: with a null context it runs here, at every point of the sweep and at the refused ones."""
    from cosmos_curate_b200 import _lib

    try:
        lib = _lib.load()
    except _lib.CurateB200Error:
        pytest.skip("libcurate_b200.so is not built")
    cases = PP.sweep_cases() + [(w, h, f, r) for w, h, r in PP.REFUSED for f in PP.FORMATS] + [(854, 481, "opencv", 224), (853, 480, "swscale", 224)]
    for w, h, f, r in cases:
        p = _lib.PreprocessPlan()
        assert lib.cb_preprocess_plan(None, w, h, PP.FMT_CODE[f], r, C.byref(p)) == 0
        want = PP.plan(w, h, f, r)
        assert p.as_dict() == want, (w, h, f, r, {k: (v, want[k]) for k, v in p.as_dict().items() if v != want[k]})
    for args in ((640, 360, 0, 0), (640, 360, 0, 1025), (0, 360, 0, 224), (640, 360, 7, 224)):
        assert lib.cb_preprocess_plan(None, *args, C.byref(_lib.PreprocessPlan())) == -2, args
    assert lib.cb_preprocess_plan(None, 640, 360, 0, 224, None) == -2


def _classes():
    seen = defaultdict(set)
    for case in PP.sweep_cases():
        c = PP.plan_class(*case)
        for k, v in c.items():
            seen[k].add(v)
        seen[("kernel x band", c["kernel"], c["taps_band"])].add(True)
        seen[("kernel x partial ntile", c["kernel"], c.get("tc_partial_ntile"))].add(True)
        if c["kernel"] != "none":
            seen[("tc_nc x partial slab", c["tc_nc"], c["tc_partial_slab"])].add(c["fmt"] != "rgb")
            seen[("simt_tc x partial tile", c["simt_tc"], c["simt_partial_tile"])].add(True)
            seen[("simt_tc x fmt", c["simt_tc"], c["fmt"])].add(True)
            seen[("ru x fmt", c["tc_ru"], c["fmt"])].add(True)
    return seen


def test_the_sweep_reaches_every_plan_class_of_both_kernels():
    s = _classes()
    assert s["kernel"] == {"tc", "simt", "none"}
    assert s["simt_kernel"] == {"simt", "none"}
    assert {"OK", "RGB", "TAPS40", "TAPS64", "UNITS"} <= s["tc_why"], s["tc_why"]
    assert s["taps_band"] == {"<=25", "26-33", "34-40", "41-64", ">64"}
    assert {32, 16} <= s["tc_nc"] and {32, 16, 8} <= s["simt_tc"]
    for band in ("<=25", "26-33", "34-40"):
        assert ("kernel x band", "tc", band) in s, band
    assert ("kernel x band", "simt", "41-64") in s
    for nc in (32, 16):  # full and partial last slab, on NV12 pools the tensor pipe serves
        for partial in (False, True):
            assert True in s[("tc_nc x partial slab", nc, partial)], (nc, partial)
    assert True in s["tc_empty_ntile"]  # a partial 32-column slab whose second N-tile has nk = 0
    assert ("kernel x partial ntile", "tc", True) in s  # ... and one whose second N-tile has 1..15 columns
    for tc in (32, 16, 8):
        for partial in (False, True):
            assert ("simt_tc x partial tile", tc, partial) in s, (tc, partial)
        for fmt in PP.FORMATS:
            assert ("simt_tc x fmt", tc, fmt) in s, (tc, fmt)
    for ru in (40, 32, 24):
        assert ("ru x fmt", ru, "opencv") in s and ("ru x fmt", ru, "swscale") in s, ru
    # torchvision's size rule scales both axes by the short side's factor, so up- and downscale come in pairs
    assert {"up", "down"} <= s["scale_x"] and {"up", "down"} <= s["scale_y"]
    for k in ("top_odd", "left_odd", "src_y_begin_odd", "row_bytes_16"):
        assert s[k] == {False, True}, k
    assert s["orientation"] == {"landscape", "portrait", "square"}
    assert {r % 32 for _, _, _, r in PP.sweep()} >= {0, 8, 16, 26}  # 200, 336 and 250: partial slabs and tiles
    assert any(r % 16 for _, _, _, r in PP.sweep())


def test_every_boundary_has_a_swept_point_on_each_side():
    pts = {(w, h, r) for w, h, _, r in PP.sweep()}
    for name, thr, lo, hi in PP.boundary_points():
        assert lo is not None and hi is not None, name
        assert lo[0] <= thr < hi[0], (name, lo, hi)
        assert (lo[1], lo[2], 224) in pts and (hi[1], hi[2], 224) in pts, name
    names = {b[0] for b in PP.boundary_points()}
    assert {"kw 256/257", "swa 256/257 at 32 columns", "swa 256/257 at 16 columns", "taps 25/26", "taps 40/41", "taps 64/65"} <= names
    for w, h in PP.SOURCES:
        assert (w, h, 224) in pts
    for r in PP.RESES:
        assert any(rr == r for _, _, _, rr in PP.sweep()), r
    assert any((w * 3) % 16 for w, _, fmts, _ in PP.sweep() if fmts == ("rgb",))


def test_size_and_crop_rules_equal_torchvision():
    F = pytest.importorskip("torchvision.transforms.functional")
    from torchvision.transforms import _functional_tensor  # noqa: F401

    try:
        from torchvision.transforms.functional import _compute_resized_output_size
    except ImportError:
        pytest.skip("torchvision has no _compute_resized_output_size")
    sizes = {(w, h) for w, h, _, _ in PP.sweep()} | {(w, h) for w, h, _ in PP.REFUSED} | {(333, 777), (1000, 999), (999, 1000)}
    for w, h in sizes:
        for res in PP.RESES:
            nh, nw = PP.resized_output_size(h, w, res)
            assert [nh, nw] == list(_compute_resized_output_size((h, w), [res])), (w, h, res)
            top, left = PP.center_crop_offsets(nh, nw, res)
            img = torch.arange(nh * nw, dtype=torch.int64).reshape(1, nh, nw)
            assert F.center_crop(img, [res])[0, 0, 0].item() == top * nw + left, (w, h, res)


@pytest.mark.parametrize(("w", "h", "res"), [(96, 64, 224), (224, 224, 224), (226, 226, 200), (854, 480, 336), (1080, 1920, 224)])
def test_constant_frames_through_the_oracle_are_exact(w, h, res):
    for value in ((0, 0, 0), (255, 255, 255), (17, 130, 244)):
        rgb = PP.constant_rgb(h, w, value)[None]
        out = preprocess.clip_resize_crop_u8(rgb, res)
        np.testing.assert_array_equal(out, np.broadcast_to(np.array(value, np.uint8)[None, :, None, None], out.shape))
    for fmt in ("opencv", "swscale"):
        for yuv in ((16, 128, 128), (235, 16, 240), (81, 90, 240)):
            c = PP.constant_nv12_rgb(*yuv, fmt)
            conv = color.nv12_to_rgb_swscale if fmt == "swscale" else color.nv12_to_rgb
            rgb = conv(PP.constant_nv12(h, w, *yuv), h, w)
            assert (rgb == c).all()
            out = preprocess.clip_resize_crop_u8(rgb[None], res)
            assert (out == c[None, :, None, None]).all(), (fmt, yuv)


@pytest.mark.parametrize(("w", "h", "res"), [(96, 64, 224), (854, 480, 200), (1080, 1920, 336), (224, 224, 224), (226, 226, 224), (1920, 1080, 384)])
def test_fast_oracle_equals_the_numpy_oracle(w, h, res):
    """The torch restatement the GPU sweep runs gives the numpy oracle's bytes: colour conversion in both arithmetics and the resize."""
    rng = np.random.default_rng(w * h + res)
    frames = [rng.integers(0, 256, size=(h * 3 // 2, w), dtype=np.uint8) for _ in range(2)]
    for fmt, conv in (("opencv", color.nv12_to_rgb), ("swscale", color.nv12_to_rgb_swscale)):
        rgb = np.stack([conv(f, h, w) for f in frames])
        fast = torch.stack([PP.nv12_to_rgb_fast(torch.from_numpy(f), h, w, fmt) for f in frames]).numpy()
        np.testing.assert_array_equal(fast, rgb)
        np.testing.assert_array_equal(PP.resize_crop_u8_fast(torch.from_numpy(rgb), res).numpy(), preprocess.clip_resize_crop_u8(rgb, res))
