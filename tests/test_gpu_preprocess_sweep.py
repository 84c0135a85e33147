"""Both CLIP resample kernels at every plan class and on both sides of every plan boundary, sources from 96x64 to 6K.

`oracle.preprocess_plan.sweep()` lists the points; `tests/test_preprocess_plan_cpu.py` shows that they reach every class.  At every
point, for NV12 (OpenCV and libswscale colour arithmetic) and RGB pools, with 2 frames of distinct seeds:

* `cb_preprocess_plan` equals the oracle's plan field by field;
* the default and the forced-SIMT u8 images are each within the u8 budget of the oracle (<= 1 LSB on <= 1e-4 of the pixels), within
  2e-4 of each other, and bitwise equal where the plan runs the SIMT kernel by default;
* one-colour frames come out as that colour exactly, on both kernels;
* bytes outside the frames (pitch padding, rows between height and luma_rows, the other slots) do not change the output;
* nothing outside the [n][3][res][res] output is written, and the typed and patch outputs are exactly LUT(u8);
* RGB points also match torchvision's CUDA Resize(antialias) + CenterCrop: within 1 LSB, on no more pixels than the oracle itself
  differs from it on plus the kernels' budget against the oracle.

The oracle images are computed on the GPU by `oracle.preprocess_plan.resize_crop_u8_fast` (separate fp32 torch operations, checked
byte for byte against the numpy oracle on the CPU and once here).  The other resamplers that read the same surfaces are swept over the
NV12 sources too.  Each point's worst LSB and differing fraction are printed when the module ends.
"""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

from cosmos_curate_b200 import _lib
from cosmos_curate_b200.runtime import COLOURS, Pool
from gpu_helpers import assert_typed_outputs_are_lut_of, ctx  # noqa: F401
from oracle import color, preprocess
from oracle import preprocess_plan as PP

pytestmark = pytest.mark.gpu

GUARD = 4096  # sentinel bytes on each side of every u8 output
SENTINEL = 0xA5
ARG, UNSUPPORTED = -2, -3  # CB_ERR_ARG, CB_ERR_UNSUPPORTED
CASES = PP.sweep_cases()
NV12_SOURCES = sorted({(w, h) for w, h, f, _ in CASES if f != "rgb"}, key=lambda s: s[0] * s[1])


@pytest.fixture(scope="module")
def record(pytestconfig):
    """Per point and kernel: worst |LSB| and differing fraction against the oracle; per RGB point: bitwise-equal fraction against
    torchvision.  Written to the terminal (past output capture) when the module ends."""
    r = {"oracle": {}, "tv": {}}
    yield r
    lines = ["preprocess sweep: point (W x H fmt res): kernel worst-LSB/differing-fraction vs the oracle, default | forced SIMT"]
    for key, v in r["oracle"].items():
        lines.append(f"  {key[0]}x{key[1]} {key[2]} {key[3]}: {v['kernel']} {v['default'][0]}/{v['default'][1]:.1e} | simt {v['simt'][0]}/{v['simt'][1]:.1e}")
    if r["tv"]:
        lines.append("RGB points against torchvision CUDA Resize + CenterCrop: bitwise-equal fraction, default | forced SIMT "
                     "(differing fraction of the oracle itself)")
        for key, v in r["tv"].items():
            lines.append(f"  {key[0]}x{key[1]} {key[2]}: {v[0]:.6f} | {v[1]:.6f} (oracle {v[2]:.1e})")
        fr = np.array(list(r["tv"].values()))
        lines.append(f"  all RGB points: bitwise-equal worst {fr[:, :2].min():.6f}, mean {fr[:, :2].mean():.6f}; oracle differs on at most {fr[:, 2].max():.1e}")
    capman = pytestconfig.pluginmanager.get_plugin("capturemanager")
    with capman.global_and_fixture_disabled():
        print("\n" + "\n".join(lines))


# ------------------------------------------------------------------------------------------------ inputs
_FRAMES: dict = {}


def _frames(w: int, h: int):
    """2 frames of (w, h), distinct seeds, on the GPU: NV12 uint8 [2][H * 3 / 2][W] (None for odd sizes) and the RGB of each colour
    arithmetic ({"opencv", "swscale", "rgb"}: the RGB pool holds the OpenCV conversion, or random RGB for odd sizes).  One source is
    kept at a time: the cases come grouped by source."""
    key = (w, h)
    if key not in _FRAMES:
        _FRAMES.clear()
        g = torch.Generator(device="cuda").manual_seed(w * 10007 + h)
        if (w | h) & 1:
            rgb = torch.randint(0, 256, (2, h, w, 3), generator=g, device="cuda", dtype=torch.uint8)
            _FRAMES[key] = (None, {"rgb": rgb})
        else:
            nv12 = torch.randint(0, 256, (2, h * 3 // 2, w), generator=g, device="cuda", dtype=torch.uint8)
            conv = {f: torch.stack([PP.nv12_to_rgb_fast(x, h, w, f) for x in nv12]) for f in ("opencv", "swscale")}
            conv["rgb"] = conv["opencv"]
            _FRAMES[key] = (nv12, conv)
    return _FRAMES[key]


def _pool(frames, w: int, h: int, fmt: str, fill: str = "zero"):
    """A 4-slot pool holding frame 0 in slot 3 and frame 1 in slot 1 (call with slots [3, 1]); pitch padding, the rows between height and
    luma_rows, the rows after the chroma plane and slots 0 and 2 hold `fill`: zeros, 255 or random bytes."""
    n_slots, slot_of = 4, (3, 1)
    if fmt == "rgb":
        row = 3 * w
        pitch, luma_rows, rows = ((row + 15) & ~15) + 48, h, h + 3
    else:
        pitch, luma_rows = ((w + 63) & ~63) + 64, h + 8
        rows = luma_rows + h // 2 + 3
    if fill == "zero":
        buf = torch.zeros((n_slots, rows, pitch), dtype=torch.uint8, device="cuda")
    elif fill == "255":
        buf = torch.full((n_slots, rows, pitch), 255, dtype=torch.uint8, device="cuda")
    else:
        g = torch.Generator(device="cuda").manual_seed(99)
        buf = torch.randint(0, 256, (n_slots, rows, pitch), generator=g, device="cuda", dtype=torch.uint8)
    for i, s in enumerate(slot_of):
        if fmt == "rgb":
            buf[s, :h, : 3 * w] = frames[i].reshape(h, 3 * w)
        else:
            buf[s, :h, :w] = frames[i][:h]
            buf[s, luma_rows : luma_rows + h // 2, :w] = frames[i][h:]
    code = _lib.FMT_RGB24 if fmt == "rgb" else COLOURS[fmt]
    return Pool(buf, _lib.SurfacePool(buf.data_ptr(), rows * pitch, w, h, pitch, luma_rows, code))


SLOTS = np.array([3, 1], np.int32)


def _run_u8(ctx, pool, res: int, slots=SLOTS):
    """cb_preprocess_clip_u8 into a buffer with GUARD sentinel bytes on each side: (rc, output [n][3][res][res] or None, guards intact)."""
    n = len(slots)
    size = n * 3 * res * res
    buf = torch.full((size + 2 * GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
    arr = np.ascontiguousarray(slots, np.int32)
    rc = ctx.lib.cb_preprocess_clip_u8(ctx.h, C.byref(pool.desc), arr.ctypes.data_as(C.POINTER(C.c_int32)), n, res, buf.data_ptr() + GUARD,
                                       torch.cuda.current_stream().cuda_stream)  # fmt: skip
    torch.cuda.synchronize()
    b = buf.cpu().numpy()
    guards = bool((b[:GUARD] == SENTINEL).all() and (b[GUARD + size :] == SENTINEL).all())
    return rc, b[GUARD : GUARD + size].reshape(n, 3, res, res), guards


def _plan(ctx, w: int, h: int, fmt: str, res: int) -> tuple[int, dict]:
    p = _lib.PreprocessPlan()
    rc = ctx.lib.cb_preprocess_plan(ctx.h, w, h, PP.FMT_CODE[fmt], res, C.byref(p))
    return rc, p.as_dict()


def _stats(got: np.ndarray, want: np.ndarray) -> tuple[int, float]:
    d = np.abs(got.astype(np.int16) - want.astype(np.int16))
    return int(d.max()), float((d > 0).mean())


def _both(ctx, monkeypatch, pool, res: int):
    """(default, forced-SIMT) u8 images; each call's sentinel guards must be intact."""
    rc, default, ok = _run_u8(ctx, pool, res)
    assert rc == 0 and ok, f"default kernel: rc {rc}, guard bytes intact {ok}"
    monkeypatch.setenv("CB_PRE_KERNEL", "simt")
    rc, simt, ok = _run_u8(ctx, pool, res)
    monkeypatch.delenv("CB_PRE_KERNEL")
    assert rc == 0 and ok, f"SIMT kernel: rc {rc}, guard bytes intact {ok}"
    return default, simt


# ------------------------------------------------------------------------------------------------ the sweep
def test_fast_oracle_on_the_gpu_equals_the_numpy_oracle():
    """The oracle images of this file come from torch operations on the GPU: the same bytes as the numpy oracle."""
    for w, h, res, fmt in ((854, 480, 200, "swscale"), (1080, 1920, 336, "opencv"), (96, 64, 224, "opencv")):
        nv12 = np.random.default_rng(w).integers(0, 256, size=(h * 3 // 2, w), dtype=np.uint8)
        conv = color.nv12_to_rgb_swscale if fmt == "swscale" else color.nv12_to_rgb
        rgb = conv(nv12, h, w)
        got_rgb = PP.nv12_to_rgb_fast(torch.from_numpy(nv12).cuda(), h, w, fmt)
        np.testing.assert_array_equal(got_rgb.cpu().numpy(), rgb)
        got = PP.resize_crop_u8_fast(got_rgb[None], res).cpu().numpy()
        np.testing.assert_array_equal(got, preprocess.clip_resize_crop_u8(rgb[None], res))


@pytest.mark.parametrize(("w", "h", "fmt", "res"), CASES, ids=[f"{w}x{h}-{f}-{r}" for w, h, f, r in CASES])
def test_sweep_point(ctx, monkeypatch, record, w, h, fmt, res):
    rc, got_plan = _plan(ctx, w, h, fmt, res)
    want_plan = PP.plan(w, h, fmt, res)
    assert rc == 0
    assert got_plan == want_plan, {k: (v, want_plan[k]) for k, v in got_plan.items() if v != want_plan[k]}
    nv12, rgb = _frames(w, h)
    src = rgb["rgb"] if fmt == "rgb" else nv12
    pool = _pool(src, w, h, fmt)
    if want_plan["kernel"] == PP.PRE_NONE:  # more than 64 taps
        rc, out, ok = _run_u8(ctx, pool, res)
        assert rc == UNSUPPORTED and ok and (out == SENTINEL).all()
        return
    want = PP.resize_crop_u8_fast(rgb[fmt][[0, 1]], res).cpu().numpy()
    default, simt = _both(ctx, monkeypatch, pool, res)
    cls = PP.plan_class(w, h, fmt, res)
    record["oracle"][(w, h, fmt, res)] = {"kernel": cls["kernel"], "default": _stats(default, want), "simt": _stats(simt, want)}
    _u8 = lambda got, ref, frac=1e-4: (_stats(got, ref)[0] <= 1 and _stats(got, ref)[1] <= frac)  # noqa: E731
    assert _u8(default, want), f"default kernel ({cls['kernel']}) against the oracle: worst {_stats(default, want)}"
    assert _u8(simt, want), f"SIMT kernel against the oracle: worst {_stats(simt, want)}"
    assert _u8(default, simt, 2e-4), f"default against SIMT: {_stats(default, simt)}"
    if want_plan["kernel"] == PP.PRE_SIMT:
        np.testing.assert_array_equal(default, simt)

    # isolation: other bytes of the pool never reach the output
    for fill in ("255", "random"):
        dirty = _pool(src, w, h, fmt, fill)
        d2, s2 = _both(ctx, monkeypatch, dirty, res)
        np.testing.assert_array_equal(d2, default, err_msg=f"default kernel reads bytes outside the frames ({fill})")
        np.testing.assert_array_equal(s2, simt, err_msg=f"SIMT kernel reads bytes outside the frames ({fill})")

    # typed and patch outputs are LUT(u8) of each kernel's own image
    assert_typed_outputs_are_lut_of(ctx, pool, res, default, slots=SLOTS, patches=((14, 640),) if res >= 14 else ())
    monkeypatch.setenv("CB_PRE_KERNEL", "simt")
    assert_typed_outputs_are_lut_of(ctx, pool, res, simt, slots=SLOTS, patches=((14, 640),) if res >= 14 else ())
    monkeypatch.delenv("CB_PRE_KERNEL")

    # one colour in, that colour out
    k = CASES.index((w, h, fmt, res))
    yuv = (16 + (37 * k) % 220, 16 + (53 * k) % 225, 16 + (71 * k) % 225)
    if fmt == "rgb":
        value = np.array([(29 * k) % 256, (113 * k + 7) % 256, (201 * k + 3) % 256], np.uint8)
        const = torch.from_numpy(PP.constant_rgb(h, w, value)).cuda()[None].expand(2, h, w, 3)
    else:
        value = PP.constant_nv12_rgb(*yuv, fmt)
        const = torch.from_numpy(PP.constant_nv12(h, w, *yuv)).cuda()[None].expand(2, h * 3 // 2, w)
    cd, cs = _both(ctx, monkeypatch, _pool(const, w, h, fmt), res)
    for got, name in ((cd, "default"), (cs, "SIMT")):
        np.testing.assert_array_equal(got, np.broadcast_to(value[None, :, None, None], got.shape), err_msg=f"{name} kernel, constant {value}")

    if fmt == "rgb":  # the reference's actual GPU path
        tv = pytest.importorskip("torchvision.transforms")
        t = tv.Compose([tv.Resize(res, interpolation=tv.InterpolationMode.BICUBIC, antialias=True), tv.CenterCrop(res)])
        ref = t(rgb["rgb"].permute(0, 3, 1, 2)).cpu().numpy()
        # torchvision's CUDA kernel is itself 1 LSB from the oracle (ATen's CPU arithmetic) on a fraction of the pixels; a kernel may
        # differ from it by that fraction plus its own budget against the oracle
        o_max, o_frac = _stats(want, ref)
        assert o_max <= 1
        for got, name in ((default, "default"), (simt, "SIMT")):
            g_max, g_frac = _stats(got, ref)
            assert g_max <= 1 and g_frac <= o_frac + 1e-4, f"{name} kernel against torchvision: {g_max} LSB on {g_frac:.2e} (oracle: {o_frac:.2e})"
        record["tv"][(w, h, res)] = (float((default == ref).mean()), float((simt == ref).mean()), o_frac)


# ------------------------------------------------------------------------------------------------ refusals
def test_refused_requests_leave_the_output_untouched(ctx, monkeypatch):
    """8K -> 224 (78 taps) and odd NV12 sizes are CB_ERR_UNSUPPORTED on both kernels; res 0 and 1025 are CB_ERR_ARG; no output byte
    changes."""
    for w, h, res in PP.REFUSED:
        nv12 = torch.randint(0, 256, (2, h * 3 // 2, w), device="cuda", dtype=torch.uint8)
        for fmt in PP.FORMATS:
            src = torch.stack([PP.nv12_to_rgb_fast(x, h, w, "opencv") for x in nv12]) if fmt == "rgb" else nv12
            pool = _pool(src, w, h, fmt)
            assert _plan(ctx, w, h, fmt, res)[1]["kernel"] == PP.PRE_NONE
            for forced in (False, True):
                if forced:
                    monkeypatch.setenv("CB_PRE_KERNEL", "simt")
                rc, out, ok = _run_u8(ctx, pool, res)
                monkeypatch.delenv("CB_PRE_KERNEL", raising=False)
                assert rc == UNSUPPORTED and ok and (out == SENTINEL).all(), (w, h, fmt, forced, rc)
    for w, h in ((854, 481), (853, 480), (1921, 1081)):
        frames = torch.zeros((2, h + h // 2, w), device="cuda", dtype=torch.uint8)
        for fmt in ("opencv", "swscale"):
            p = _plan(ctx, w, h, fmt, 224)[1]
            assert p["kernel"] == PP.PRE_NONE and PP.WHY[p["tc_why"]] == "ODD"
            rc, out, ok = _run_u8(ctx, _pool(frames, w, h, fmt), 224)
            assert rc == UNSUPPORTED and ok and (out == SENTINEL).all(), (w, h, fmt, rc)
    pool = _pool(_frames(640, 360)[0], 640, 360, "opencv")
    for res in (0, 1025):
        assert _plan(ctx, 640, 360, "opencv", res)[0] == ARG
        rc, out, ok = _run_u8(ctx, pool, res)
        assert rc == ARG and ok and (out == SENTINEL).all(), (res, rc)


# ------------------------------------------------------------------------------------------------ the other resamplers on the same surfaces
@pytest.mark.parametrize(("w", "h"), NV12_SOURCES, ids=[f"{w}x{h}" for w, h in NV12_SOURCES])
def test_other_resamplers_at_every_source(ctx, w, h):
    """27x48 bilinear thumbnails (shot detection decodes whole videos at any size) against the oracle on the existing budget; the
    video tube bit-exact; cv2 INTER_CUBIC (OpenCV arithmetic) bit-exact at sources up to 1080p."""
    from oracle import resize_cubic as R
    from oracle import video_tube as T

    nv12, rgb = _frames(w, h)
    for fmt in ("opencv", "swscale"):
        pool = _pool(nv12, w, h, fmt, "random")
        ref = rgb[fmt].cpu().numpy()
        got = ctx.preprocess_bilinear_u8(pool, 48, 27, slots=SLOTS).cpu().numpy()
        for i in range(2):
            want = preprocess.resize_bilinear_u8(ref[i], 27, 48)
            d = np.abs(got[i].astype(int) - want.astype(int))
            assert d.max() <= 1 and (d > 0).mean() < 1e-3, (fmt, i, d.max(), (d > 0).mean())
        tube = ctx.video_tube(pool, 224, 224, slots=SLOTS).cpu().numpy()
        np.testing.assert_array_equal(tube, T.construct_frames(list(ref), fnum=2)[0], err_msg=f"video tube {fmt}")
        if w * h <= 1920 * 1080:
            cub = ctx.resize_cubic_u8(pool, 224, 224, slots=SLOTS, mode=_lib.CUBIC_OPENCV).cpu().numpy()
            for i in range(2):
                np.testing.assert_array_equal(cub[i], R.resize_cubic_u8(ref[i], 224, 224), err_msg=f"cubic {fmt} frame {i}")
