"""GPU: parity of the REAL input path and of the bench-shape execution (VERDICT r1 "what's weak" 1-2).

* swscale RGB (what the reference feeds CLIP: PyAV `to_ndarray("rgb24")`, decoder_utils.py:439-451; cv2/libavcodec+swscale
  is the stand-in, PyAV is not installable here) -> fp32 oracle embeddings, against NVDEC -> fused NV12 kernel -> fp16 tower,
  on CLIP ViT-L/14.  Round 1 converted with OpenCV / CV-CUDA semantics and claimed the difference to swscale was "absorbed by the
  1e-3 tolerance"; measured here it is NOT (1.2e-2 on the dark title frames), so the fused kernel now has libswscale's own
  arithmetic (CB_FMT_NV12_SWS) and the stages default to it: the RGB is byte-identical, the embeddings within 1e-3.
* batch invariance at the bench shape: 264 frames through the wgmma GEMM + attention_wgmma + chunking vs the same frames at n=3.
* activation outliers: real CLIP-L/14 has a few residual-stream channels two orders of magnitude above the rest; seeded
  Gaussian weights do not.  A stress configuration plants such channels and checks the fp16 qkv / mlp activations survive.
* the reference's real-weight goldens 4.8575 / 3.7989 +- 0.002 (test_aesthetic_filter.py:33-35) - skipped unless the
  checkpoints are present (they are not downloadable here).
"""

from __future__ import annotations

import os
import uuid
from pathlib import Path

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from gpu_helpers import ctx, nv12_pool as _nv12_pool  # noqa: F401
from oracle import color, preprocess, vit

pytestmark = pytest.mark.gpu
os.environ.setdefault("OPENCV_LOG_LEVEL", "ERROR")

SINTEL_IDS = [0, 24, 48, 72, 96, 120, 144, 168, 192, 216, 239]  # sample_closest(1 fps) on the fixture (SURVEY.md V4)


def _rel_rows(got: np.ndarray, want: np.ndarray) -> np.ndarray:
    return np.linalg.norm(got - want, axis=1) / np.linalg.norm(want, axis=1)


def _swscale_frames(path: Path, ids) -> np.ndarray:
    import cv2

    cap = cv2.VideoCapture(str(path))
    out, i, want = [], 0, set(ids)
    while True:
        ok, bgr = cap.read()
        if not ok:
            break
        if i in want:
            out.append(bgr[:, :, ::-1].copy())
        i += 1
    cap.release()
    assert len(out) == len(ids)
    return np.stack(out)


def test_real_input_path_embeddings_swscale_vs_nvdec_l14(ctx):
    from cosmos_curate_b200.runtime import Decoder, VitTower, alloc_nv12_pool

    cfg = vit.CLIP_VIT_L14
    w = vit.random_weights(cfg, seed=3)
    sd = vit.random_aesthetic_mlp(seed=3, in_dim=cfg.proj_dim)
    aw, ab = vit.collapse_aesthetic_mlp(sd)
    path = GOLDEN / "sintel_clip_10s.mp4"
    rgb_sws = _swscale_frames(path, SINTEL_IDS)  # [11, 480, 854, 3] - the reference's CLIP input
    ref = vit.forward(cfg, w, preprocess.clip_preprocess(rgb_sws))  # the reference chain in fp32 on the CPU
    ref_score = vit.aesthetic_mlp_forward(sd, ref["embedding"])

    tower = VitTower(ctx, cfg.to_dict(), w, max_batch=16, aesthetic=(aw, ab))
    # (b) our tower on the SAME swscale RGB frames: isolates fp16-tower + resize error from the colour path
    emb_b, _, score_b = tower.embed_pool(ctx.rgb_pool(torch.from_numpy(rgb_sws).cuda()))
    # (c) the product path: NVDEC surfaces -> fused NV12 kernel with libswscale's colour arithmetic -> tower
    pool = alloc_nv12_pool(ctx, len(SINTEL_IDS), 854, 480, colour="swscale")
    Decoder(ctx).decode(path.read_bytes(), SINTEL_IDS, pool, np.arange(len(SINTEL_IDS)))
    rgb_gpu = ctx.nv12_to_rgb(pool).cpu().numpy()
    assert np.array_equal(rgb_gpu, rgb_sws)  # NVDEC + our conversion == libavcodec + libswscale, every byte of every sampled frame
    emb_c, _, score_c = tower.embed_pool(pool)
    # (d) for the record: the same surfaces through the OpenCV / CV-CUDA conversion (the reference's nvcodec_utils branch)
    pool_cv = ctx.nv12_pool(pool.buf, 854, 480, 480, colour="opencv")
    emb_d, _, _ = tower.embed_pool(pool_cv)
    rgb_cv = ctx.nv12_to_rgb(pool_cv).cpu().numpy()

    rel_b = _rel_rows(emb_b.cpu().numpy(), ref["embedding"])
    rel_c = _rel_rows(emb_c.cpu().numpy(), ref["embedding"])
    rel_d = _rel_rows(emb_d.cpu().numpy(), ref["embedding"])
    px = np.abs(rgb_cv.astype(int) - rgb_sws.astype(int))
    print(f"\n[real-input parity, ViT-L/14 seeded] embedding rel err vs fp32 oracle on swscale RGB: tower on uploaded RGB max {rel_b.max():.2e}, "
          f"product path (NVDEC + swscale-exact fused kernel) max {rel_c.max():.2e} mean {rel_c.mean():.2e}, score |d| max "
          f"{np.abs(score_c.cpu().numpy() - ref_score).max():.2e} | with the OpenCV/CV-CUDA colour instead: pixels mean |d| {px.mean():.3f} max {px.max()}, "
          f"embedding rel err max {rel_d.max():.2e} (dark title frames dominate)")  # fmt: skip
    assert rel_b.max() < 1e-3  # BASELINE.json: fp embeddings within 1e-3 relative, same input frames
    assert rel_c.max() < 1e-3  # ... and on the product path from the compressed clip
    # identical pixels in: the RGB upload goes through the SIMT resize kernel, the NV12 surfaces through the tensor-pipe one - two fp32
    # summation orders, i.e. a handful of u8 pixels one LSB apart (the <= 1e-4 budget), visible only on the near-black title frame
    assert _rel_rows(emb_c.cpu().numpy(), emb_b.cpu().numpy()).max() < 5e-4
    np.testing.assert_allclose(score_c.cpu().numpy(), ref_score, atol=2e-3)  # the reference's own test tolerance


def test_batch_invariance_at_bench_shape_l14(ctx):
    """n=264 (128 x 256 GEMM tiles, attention_wgmma over 4224 units, max_batch chunking) vs n=3: same frames, same embeddings."""
    from cosmos_curate_b200.runtime import VitTower

    cfg = vit.CLIP_VIT_L14
    w = vit.random_weights(cfg, seed=5)
    tower_big = VitTower(ctx, cfg.to_dict(), w, max_batch=264)
    frames = [color.synthetic_nv12(480, 854, seed=200 + s) for s in range(6)]
    pool = _nv12_pool(ctx, frames, 854, 480, 1024, 480)
    slots = np.arange(264, dtype=np.int32) % 6
    emb_big, _, _ = tower_big.embed_pool(pool, slots=slots)
    emb_big2, _, _ = tower_big.embed_pool(pool, slots=slots)
    assert torch.equal(emb_big, emb_big2)  # run-to-run determinism at the bench shape (fixed P.V chunk order)
    e = emb_big.cpu().numpy()
    for r in range(6):  # the same frame at 44 batch positions: bitwise equal rows
        rows = e[r::6]
        assert np.array_equal(rows, np.broadcast_to(rows[0], rows.shape)), r
    emb_small, _, _ = tower_big.embed_pool(pool, slots=np.arange(3, dtype=np.int32))
    rel = _rel_rows(emb_small.cpu().numpy(), e[:3])
    assert rel.max() < 2e-5, rel  # other tile shapes may be picked at n=3; results still agree far inside 1e-3
    # and against the fp32 oracle for those three frames
    u8 = ctx.preprocess_clip_u8(pool, slots=np.arange(3, dtype=np.int32)).cpu().numpy()
    lut = preprocess.normalize_lut()
    x = np.stack([lut[c][u8[:, c]] for c in range(3)], axis=1)
    ref = vit.forward(cfg, w, x)
    assert _rel_rows(e[:3], ref["embedding"]).max() < 1e-3


def outlier_weights(cfg, seed: int, channels=(7, 300, 511), gain: float = 50.0):
    """Seeded weights with planted residual-stream outlier channels, the pattern of real CLIP-L/14 checkpoints ("massive
    activations"): the MLP of layer 1 writes +120 / -90 into three channels and a few fc2 rows of those channels are 12x larger,
    so from layer 2 on the residual stream carries values > 100 on three channels while the rest stays O(1) (max/median ~ 170,
    checked on the CPU oracle) - LayerNorm statistics, the fp16 qkv / mlp activations and the fp16 GEMM operands all see a
    dynamic range that Gaussian weights never produce."""
    w = {k: v.copy() for k, v in vit.random_weights(cfg, seed=seed).items()}
    for j, c in enumerate(channels):
        w["L1.fc2_b"][c] += 120.0 if j % 2 == 0 else -90.0
        for i in (1, 5, 11):
            w[f"L{i}.fc2_w"][c, :] *= gain / 4
    return w


def test_activation_outliers_survive_fp16_storage_l14(ctx):
    from cosmos_curate_b200.runtime import VitTower

    cfg = vit.CLIP_VIT_L14
    w = outlier_weights(cfg, seed=9)
    frames = [color.synthetic_nv12(480, 854, seed=300 + s) for s in range(3)]
    pool = _nv12_pool(ctx, frames, 854, 480, 1024, 480)
    tower = VitTower(ctx, cfg.to_dict(), w, max_batch=4)
    emb, _, _ = tower.embed_pool(pool)
    u8 = ctx.preprocess_clip_u8(pool).cpu().numpy()
    lut = preprocess.normalize_lut()
    x = np.stack([lut[c][u8[:, c]] for c in range(3)], axis=1)
    ref = vit.forward(cfg, w, x, return_hidden=True)
    hid = ref["hidden"] if "hidden" in ref else None
    if hid is not None:
        h_last = np.abs(np.asarray(hid[-1]))
        ratio = h_last.max() / np.median(h_last)
        print(f"\n[outlier stress] residual stream max/median |x| = {ratio:.0f}")
        assert ratio > 100  # the stress really has outliers
    rel = _rel_rows(emb.cpu().numpy(), ref["embedding"])
    print(f"[outlier stress] embedding rel err max {rel.max():.2e}")
    assert rel.max() < 1e-3


def _real_weights():
    clip_dir, aes = os.environ.get("CURATE_B200_CLIP_DIR"), os.environ.get("CURATE_B200_AESTHETIC_CKPT")
    if not clip_dir or not aes or not Path(clip_dir).is_dir() or not Path(aes).is_file():
        pytest.skip("real checkpoints absent: set CURATE_B200_CLIP_DIR (openai/clip-vit-large-patch14 snapshot dir) and "
                    "CURATE_B200_AESTHETIC_CKPT (ttj/sac-logos-ava1-l14-linearMSE model.safetensors)")  # fmt: skip
    return clip_dir, aes


@pytest.mark.parametrize("reduction,expected", [("mean", 4.8575), ("min", 3.7989)])
def test_reference_real_weight_goldens(ctx, reduction, expected):
    """The reference's own regression values (tests/.../test_aesthetic_filter.py:33-35, TOLERANCE 0.002) on its fixture clip,
    through the reference's stage pair on the NVDEC path and through the fused stage."""
    clip_dir, aes = _real_weights()
    from cosmos_curate_b200.data_model import Clip, SplitPipeTask, Video
    from cosmos_curate_b200.interfaces import run_pipeline
    from cosmos_curate_b200.models import weights as W
    from cosmos_curate_b200.models.clip_aesthetics import CLIPAestheticScorer
    from cosmos_curate_b200.runtime import VitTower, get_context
    from cosmos_curate_b200.stages import AestheticFilterStage, ClipFrameExtractionStage, NvdecClipAestheticStage

    cfg, w = W.load_hf_clip_dir(clip_dir)
    head = W.load_aesthetic_mlp(aes)

    class _Real(CLIPAestheticScorer):
        def setup(self_inner):
            from cosmos_curate_b200.models.clip import CLIPImageEmbeddings

            m = CLIPImageEmbeddings()
            m._tower = VitTower(get_context(), cfg.to_dict(), w, max_batch=64, aesthetic=head)
            self_inner._clip_model = m

    data = (GOLDEN / "sintel_clip_10s.mp4").read_bytes()

    def task():
        clip = Clip(uuid=uuid.UUID("12345678-1234-5678-1234-567812345678"), source_video="sample_video.mp4", span=(0.0, 10.0), encoded_data=data)
        return SplitPipeTask(session_id="test-session", video=Video(input_video="sample_video.mp4", clips=[clip]))

    t1 = task()
    run_pipeline([t1], [ClipFrameExtractionStage(target_fps=[1]), AestheticFilterStage(score_threshold=0.0, reduction=reduction, model=_Real())])
    assert t1.video.clips[0].aesthetic_score == pytest.approx(expected, abs=0.002)
    t2 = task()
    run_pipeline([t2], [NvdecClipAestheticStage(score_threshold=0.0, reduction=reduction, num_decoders=2, max_batch=64, model=_Real())])
    assert t2.video.clips[0].aesthetic_score == pytest.approx(expected, abs=0.002)
