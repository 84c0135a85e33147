"""GPU parity tests (B200): every call goes through the C ABI of libcurate_b200.so.

Integer / byte stages are compared bit-exactly with the oracle where the arithmetic is pinned
(colour conversion, frame indices), within the stated fp32-summation budget where it is not
(u8 stage of the antialiased resize: <= 1 LSB on <= 1e-4 of the pixels - the same budget the
oracle itself needs against ATen, tests/test_oracle_cpu.py).  Floating-point stages: tolerance in
each test.
"""

from __future__ import annotations

import numpy as np
import pytest
import torch

from conftest import golden_json, load_golden
from gpu_helpers import assert_typed_outputs_are_lut_of, ctx, nv12_pool as _nv12_pool, u8_budget as _u8_budget  # noqa: F401
from oracle import color, preprocess, vit

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------ colour / bilinear
@pytest.mark.parametrize(("h", "w", "pitch", "luma_rows"), [(64, 96, 128, 64), (480, 854, 1024, 480), (1080, 1920, 2048, 1088)])
def test_nv12_to_rgb_bit_exact(ctx, h, w, pitch, luma_rows):
    if w % 2:
        pytest.skip("odd width")
    rng = np.random.default_rng(0)
    frames = [rng.integers(0, 256, size=(h * 3 // 2, w), dtype=np.uint8) for _ in range(2)]
    pool = _nv12_pool(ctx, frames, w, h, pitch, luma_rows)
    got = ctx.nv12_to_rgb(pool).cpu().numpy()
    for i, f in enumerate(frames):
        np.testing.assert_array_equal(got[i], color.nv12_to_rgb(f, h, w))


def test_bilinear_27x48_matches_oracle(ctx):
    frames = [color.synthetic_nv12(1080, 1920, seed=s) for s in range(3)]
    pool = _nv12_pool(ctx, frames, 1920, 1080, 2048, 1088)
    got = ctx.preprocess_bilinear_u8(pool, 48, 27).cpu().numpy()
    assert got.shape == (3, 27, 48, 3)
    for i, f in enumerate(frames):
        want = preprocess.resize_bilinear_u8(color.nv12_to_rgb(f, 1080, 1920), 27, 48)
        d = np.abs(got[i].astype(int) - want.astype(int))
        assert d.max() <= 1 and (d > 0).mean() < 1e-3  # fp32 contraction differences only


# ------------------------------------------------------------------------------------ CLIP preprocess
@pytest.mark.parametrize(("h", "w", "pitch", "luma_rows"), [(1080, 1920, 2048, 1088), (720, 1280, 1280, 720), (480, 854, 1024, 480), (1920, 1080, 1280, 1920)])
def test_clip_preprocess_nv12_u8_stage(ctx, h, w, pitch, luma_rows):
    frames = [color.synthetic_nv12(h, w, seed=s) for s in range(2)]
    pool = _nv12_pool(ctx, frames, w, h, pitch, luma_rows)
    got = ctx.preprocess_clip_u8(pool, res=224).cpu().numpy()
    rgb = np.stack([color.nv12_to_rgb(f, h, w) for f in frames])
    _u8_budget(got, preprocess.clip_resize_crop_u8(rgb, 224))


def test_clip_preprocess_typed_and_patch_layout(ctx):
    h, w = 1080, 1920
    frames = [color.synthetic_nv12(h, w, seed=10 + s) for s in range(3)]
    pool = _nv12_pool(ctx, frames, w, h, 2048, 1088)
    u8 = ctx.preprocess_clip_u8(pool).cpu().numpy()
    lut = preprocess.normalize_lut()
    want32 = np.stack([lut[c][u8[:, c]] for c in range(3)], axis=1)
    # given the u8 stage, normalise + cast must be exact
    got32 = ctx.preprocess_clip(pool, dtype=torch.float32).cpu().numpy()
    np.testing.assert_array_equal(got32, want32)
    got16 = ctx.preprocess_clip(pool, dtype=torch.float16).cpu().numpy()
    np.testing.assert_array_equal(got16, want32.astype(np.float16))
    gotbf = ctx.preprocess_clip(pool, dtype=torch.bfloat16).float().cpu().numpy()
    np.testing.assert_array_equal(gotbf, torch.from_numpy(want32).to(torch.bfloat16).float().numpy())
    for patch, k_pad in ((14, 640), (32, 3072), (16, 768)):
        gp = ctx.preprocess_clip(pool, dtype=torch.float16, layout="patch", patch=patch, k_pad=k_pad).cpu().numpy()
        np.testing.assert_array_equal(gp, preprocess.to_patches(want32.astype(np.float16), patch, k_pad))


def test_clip_preprocess_rgb_frames_vs_reference_golden(ctx):
    """Host RGB frames (the ModelInterface input of clip.py:64-70) against the REFERENCE's own transform output."""
    g = load_golden("clip_preprocess_ref.npz")
    lut = preprocess.normalize_lut()
    for name in sorted(k[:-3] for k in g.files if k.endswith("_in")):
        fr, want = g[name + "_in"], g[name + "_out"]
        pool = ctx.rgb_pool(torch.from_numpy(fr).cuda())
        got = ctx.preprocess_clip(pool, dtype=torch.float32).cpu().numpy()
        assert got.shape == want.shape
        bad = 0
        for c in range(3):
            ref_u8 = np.abs(want[:, c, :, :, None] - lut[c]).argmin(-1)
            got_u8 = np.abs(got[:, c, :, :, None] - lut[c]).argmin(-1)
            assert np.abs(lut[c][got_u8] - got[:, c]).max() == 0.0
            d = np.abs(ref_u8 - got_u8)
            assert d.max() <= 1, name
            bad += int((d > 0).sum())
        assert bad <= 1e-4 * want.size, (name, bad)


def test_clip_preprocess_vs_torchvision_cuda(ctx):
    """The reference's actual CUDA path: torchvision transforms on a CUDA uint8 tensor (clip.py:48-70)."""
    tv = pytest.importorskip("torchvision.transforms")
    t = tv.Compose([tv.Resize(224, interpolation=tv.InterpolationMode.BICUBIC, antialias=True), tv.CenterCrop(224)])
    rng = np.random.default_rng(5)
    fr = rng.integers(0, 256, size=(2, 1080, 1920, 3), dtype=np.uint8)
    x = torch.from_numpy(fr).cuda()
    want = t(x.permute(0, 3, 1, 2)).cpu().numpy()
    got = ctx.preprocess_clip_u8(ctx.rgb_pool(x)).cpu().numpy()
    _u8_budget(got, want)


def test_preprocess_edge_cases(ctx):
    from cosmos_curate_b200._lib import CurateB200Error

    frames = [color.synthetic_nv12(64, 96, seed=1)]
    pool = _nv12_pool(ctx, frames, 96, 64, 128, 64)
    assert ctx.preprocess_clip_u8(pool, slots=np.zeros(0, np.int32)).shape[0] == 0  # empty batch
    out = ctx.preprocess_clip_u8(pool, slots=[0, 0, 0]).cpu().numpy()  # repeated slot (supersampled frame ids)
    np.testing.assert_array_equal(out[0], out[2])
    with pytest.raises(CurateB200Error):
        ctx.preprocess_clip_u8(pool, slots=[-1])
    # upscale (scale < 1) path
    rgb = color.nv12_to_rgb(frames[0], 64, 96)[None]
    _u8_budget(out[:1], preprocess.clip_resize_crop_u8(rgb, 224))




# ------------------------------------------------------------------------------------ mode B: cv2 INTER_CUBIC target_res
def test_resize_cubic_matches_cv2_goldens(ctx):
    """cb_resize_cubic_u8 on RGB frames against cv2.resize(INTER_CUBIC) outputs generated by cv2 itself (extract_frames'
    target_res, decoder_utils.py:666-670): CB_CUBIC_OPENCV bit-exact with OpenCV's own code, CB_CUBIC_IPP within 1 LSB on
    < 1e-4 of the pixels of the x86 wheels' Intel IPP result."""
    from conftest import load_golden
    from cosmos_curate_b200 import _lib

    g = load_golden("resize_cubic_ref.npz")
    for name in sorted(k[:-3] for k in g.files if k.endswith("_in")):
        img, (th, tw) = g[name + "_in"], (int(g[name + "_res"][0]), int(g[name + "_res"][1]))
        pool = ctx.rgb_pool(torch.from_numpy(np.stack([img, img[::-1].copy()])).cuda())
        got = ctx.resize_cubic_u8(pool, tw, th, mode=_lib.CUBIC_OPENCV).cpu().numpy()
        assert got.shape == (2, th, tw, 3)
        np.testing.assert_array_equal(got[0], g[name + "_opencv"], err_msg=name)
        got_f = ctx.resize_cubic_u8(pool, tw, th, mode=_lib.CUBIC_IPP).cpu().numpy()
        _u8_budget(got_f[0], g[name + "_ipp"], frac=1e-4)


def test_resize_cubic_from_nv12_and_into_the_tower(ctx):
    """NV12 surfaces (colour-converted per tap) -> 224x224 cubic -> CLIP transforms (Resize(224) is then the identity):
    u8 frames bit-exact with the oracle chain, embeddings of the mode-B path within 1e-3 of the fp32 oracle."""
    from cosmos_curate_b200 import _lib
    from cosmos_curate_b200.runtime import VitTower
    from oracle import resize_cubic as R

    frames = [color.synthetic_nv12(1080, 1920, seed=80 + s) for s in range(3)]
    pool = _nv12_pool(ctx, frames, 1920, 1080, 2048, 1088)
    rgb = np.stack([color.nv12_to_rgb(f, 1080, 1920) for f in frames])
    got = ctx.resize_cubic_u8(pool, 224, 224, mode=_lib.CUBIC_OPENCV).cpu().numpy()
    want = np.stack([R.resize_cubic_u8(f, 224, 224) for f in rgb])
    np.testing.assert_array_equal(got, want)
    got_f = ctx.resize_cubic_u8(pool, 224, 224, mode=_lib.CUBIC_IPP)
    want_f = np.stack([R.resize_cubic_real_u8(f, 224, 224) for f in rgb])
    _u8_budget(got_f.cpu().numpy(), want_f, frac=1e-4)
    # non-square target, odd source subset through slots
    got2 = ctx.resize_cubic_u8(pool, 48, 27, slots=np.array([2, 0], dtype=np.int32), mode=_lib.CUBIC_OPENCV).cpu().numpy()
    np.testing.assert_array_equal(got2[0], R.resize_cubic_u8(rgb[2], 27, 48))
    np.testing.assert_array_equal(got2[1], R.resize_cubic_u8(rgb[0], 27, 48))
    cfg = vit.CLIP_VIT_B32
    w = vit.random_weights(cfg, seed=6)
    tower = VitTower(ctx, cfg.to_dict(), w, max_batch=4)
    emb, _, _ = tower.embed_pool(ctx.rgb_pool(got_f))
    ref = vit.forward(cfg, w, preprocess.clip_preprocess(want_f))["embedding"]  # 224x224 input: torchvision Resize / CenterCrop are no-ops
    rel = np.linalg.norm(emb.cpu().numpy() - ref, axis=1) / np.linalg.norm(ref, axis=1)
    assert rel.max() < 1e-3


# ------------------------------------------------------------------------------------ tensor-pipe kernel vs SIMT kernel
@pytest.mark.parametrize(("h", "w", "pitch", "res", "colour"), [(1080, 1920, 2048, 224, "opencv"), (1080, 1920, 2048, 224, "swscale"), (2160, 3840, 3840, 384, "swscale"),
                                                                (480, 854, 1024, 224, "swscale"), (720, 1280, 1280, 384, "opencv"), (360, 640, 640, 224, "opencv"),
                                                                (2160, 3840, 3840, 224, "swscale"), (2160, 3840, 3840, 192, "opencv"), (1080, 1920, 0, 224, "rgb")])
def test_tensor_pipe_preprocess_agrees_with_simt_kernel_and_oracle(ctx, monkeypatch, h, w, pitch, res, colour):
    """clip_preprocess_tc_kernel (horizontal pass as a banded fp16 hi/lo GEMM on wgmma, the default) against the SIMT kernel
    (CB_PRE_KERNEL=simt) and the oracle: same u8 image within the fp32-summation-order budget, both colour conversions, 1080p -> 224
    (bench shape), 4K -> 384 (SoViT shape, 24 vertical taps, 256-column windows), widths that are not a multiple of the window.
    4K -> 192 has 45 vertical taps, more than the tensor-pipe kernel takes, and an RGB pool is never served by it: there the default
    call runs the SIMT kernel too.  Both kernels share the normalise/pack step, so typed and patch outputs are exactly LUT(u8) of
    each kernel's own u8 image."""
    frames = [color.synthetic_nv12(h, w, seed=60 + s) for s in range(2)]
    conv = color.nv12_to_rgb_swscale if colour == "swscale" else color.nv12_to_rgb
    rgb = np.stack([conv(f, h, w) for f in frames])
    if colour == "rgb":
        pool = ctx.rgb_pool(torch.from_numpy(rgb).cuda())
    else:
        buf = np.zeros((2, h + h // 2, pitch), dtype=np.uint8)
        for i, f in enumerate(frames):
            buf[i, :, :w] = f
        pool = ctx.nv12_pool(torch.from_numpy(buf).cuda(), w, h, h, colour=colour)
    got_tc = ctx.preprocess_clip_u8(pool, res=res).cpu().numpy()
    monkeypatch.setenv("CB_PRE_KERNEL", "simt")
    got_simt = ctx.preprocess_clip_u8(pool, res=res).cpu().numpy()
    assert_typed_outputs_are_lut_of(ctx, pool, res, got_simt)
    monkeypatch.delenv("CB_PRE_KERNEL")
    want = preprocess.clip_resize_crop_u8(rgb, res)
    _u8_budget(got_tc, want)
    _u8_budget(got_simt, want)
    _u8_budget(got_tc, got_simt, frac=2e-4)  # two fp32 summation orders apart
    if res == 192 or colour == "rgb":  # the default call ran the SIMT kernel too
        np.testing.assert_array_equal(got_tc, got_simt)
    assert_typed_outputs_are_lut_of(ctx, pool, res, got_tc)


def test_clip_preprocess_4k_rgb_frames_strong_downscale(ctx):
    """4K host RGB frames -> 224 (9.6 source pixels per output column, 40 taps): the SIMT kernel halves its column tile so that the
    window still fits one TMA box; against torchvision's own CUDA transform (clip.py:48-70)."""
    tv = pytest.importorskip("torchvision.transforms")
    t = tv.Compose([tv.Resize(224, interpolation=tv.InterpolationMode.BICUBIC, antialias=True), tv.CenterCrop(224)])
    rng = np.random.default_rng(8)
    fr = rng.integers(0, 256, size=(1, 2160, 3840, 3), dtype=np.uint8)
    x = torch.from_numpy(fr).cuda()
    want = t(x.permute(0, 3, 1, 2)).cpu().numpy()
    pool = ctx.rgb_pool(x)
    _u8_budget(ctx.preprocess_clip_u8(pool).cpu().numpy(), want)
    lut = preprocess.normalize_lut()
    want32 = np.stack([lut[c][want[:, c]] for c in range(3)], axis=1)
    gp = ctx.preprocess_clip(pool, dtype=torch.float16, layout="patch", patch=14, k_pad=640).cpu().numpy()
    ref = preprocess.to_patches(want32.astype(np.float16), 14, 640)
    assert (gp != ref).mean() < 2e-4  # the same <= 1e-4 u8 budget seen through the LUT


# ------------------------------------------------------------------------------------ video-tower tubes (InternVideo2 input formulation)
def test_video_tube_matches_the_reference_formulation_bit_for_bit(ctx):
    """cb_video_tube against tubes produced by the reference's own InternVideo2MultiModality._construct_frames
    (internvideo2_mm.py:390-405: cv2.resize + numpy float32 normalise): every float32 bit equal - linear taps, the 2x2
    decimation cv2 reroutes to INTER_AREA, the copy for equal sizes, upscaling, a tall source - and, at the real 224 x 224
    size, a sha256 of the whole tube for SD / HD / 4K sources."""
    import hashlib

    from conftest import load_golden
    from cosmos_curate_b200.models.internvideo2_frames import InternVideo2FrameFormulator, select_frame_ids
    from oracle import video_tube as T

    g = load_golden("video_tube_ref.npz")
    for name in sorted(k[:-3] for k in g.files if k.endswith("_in")):
        fr, (tw, th) = g[name + "_in"], (int(v) for v in g[name + "_size"])
        ids = select_frame_ids(len(fr), 8)
        assert ids == T.select_frames(len(fr), 8)
        pool = ctx.rgb_pool(torch.from_numpy(np.ascontiguousarray(fr[ids])).cuda())
        tube, u8 = ctx.video_tube(pool, tw, th, want_u8=True)
        np.testing.assert_array_equal(tube.cpu().numpy()[None], g[name + "_tube"], err_msg=name)
        np.testing.assert_array_equal(u8.cpu().numpy(), np.stack([T.resize_linear_u8(fr[i], th, tw) for i in ids]), err_msg=name)
    m = InternVideo2FrameFormulator()
    m.setup()
    assert m.get_target_num_frames() == 8 and m.model_id_names == []
    for name in ("sd", "hd", "uhd"):
        n, h, w = (int(v) for v in g[name + "_shape"])
        rng = np.random.default_rng([20250924, h])
        fr = [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for _ in range(n)]
        tube = m.formulate_input_frames(fr)
        assert tube.shape == (1, 8, 3, 224, 224) and tube.dtype == np.float32
        assert hashlib.sha256(np.ascontiguousarray(tube).tobytes()).digest() == g[name + "_sha256"].tobytes(), name
        if name == "sd":
            np.testing.assert_array_equal(m.formulate_input_image(fr[3]), T.construct_image(fr[3]))
            np.testing.assert_array_equal(tube, T.construct_frames(fr))
    assert m.formulate_input_frames(fr[:5]).shape == (0,)  # too few frames: the reference's empty float32 array
    mixed = [np.full((40, 60, 3), 7, np.uint8)] * 4 + [np.full((50, 30, 3), 200, np.uint8)] * 4  # frame-by-frame resize: sizes may differ
    np.testing.assert_array_equal(m.formulate_input_frames(mixed), T.construct_frames(mixed))


@pytest.mark.parametrize("colour", ["swscale", "opencv"])
def test_video_tube_from_nv12_surfaces(ctx, colour):
    """NV12 decode surfaces (colour-converted per tap) -> tube, bit-exact with convert-then-formulate on the CPU."""
    from cosmos_curate_b200._lib import CurateB200Error
    from oracle import video_tube as T

    conv = color.nv12_to_rgb_swscale if colour == "swscale" else color.nv12_to_rgb
    for (h, w, pitch, rows) in [(1080, 1920, 2048, 1088), (360, 640, 640, 360), (448, 448, 512, 448)]:
        frames = [color.synthetic_nv12(h, w, seed=300 + s) for s in range(3)]
        pool = _nv12_pool(ctx, frames, w, h, pitch, rows, colour=colour)
        rgb = [conv(f, h, w) for f in frames]
        slots = np.array([2, 0, 2, 1], dtype=np.int32)
        got = ctx.video_tube(pool, 224, 224, slots=slots).cpu().numpy()
        want = T.construct_frames([rgb[i] for i in slots], fnum=4)[0]
        np.testing.assert_array_equal(got, want)
    with pytest.raises(CurateB200Error):
        ctx.video_tube(pool, 0, 224)
