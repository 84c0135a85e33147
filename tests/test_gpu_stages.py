"""GPU: the CuratorStage / ModelInterface drop-ins end to end (SequentialRunner, like the reference's stage tests),
scores and embeddings checked against the oracle."""

from __future__ import annotations

import os
import uuid

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from gpu_helpers import ctx  # noqa: F401

pytestmark = pytest.mark.gpu
os.environ.setdefault("OPENCV_LOG_LEVEL", "ERROR")

SIG1 = "FrameExtractionPolicy.sequence-1000"


def _oracle_scores(cfg, w, sd, rgb_frames):
    from oracle import preprocess, vit

    ref = vit.forward(cfg, w, preprocess.clip_preprocess(rgb_frames))
    return ref["embedding"], vit.aesthetic_mlp_forward(sd, ref["embedding"])


def _model(cfg_name="CLIP_TINY", seed=7):
    """CLIPAestheticScorer with oracle-seeded weights so the oracle can reproduce the numbers."""
    from cosmos_curate_b200.models.clip_aesthetics import CLIPAestheticScorer
    from cosmos_curate_b200.runtime import VitTower, get_context
    from oracle import vit

    cfg = getattr(vit, cfg_name)
    w = vit.random_weights(cfg, seed=seed)
    sd = vit.random_aesthetic_mlp(seed=seed, in_dim=cfg.proj_dim)
    aw, ab = vit.collapse_aesthetic_mlp(sd)

    class _Seeded(CLIPAestheticScorer):
        def setup(self_inner):
            from cosmos_curate_b200.models.clip import CLIPImageEmbeddings

            m = CLIPImageEmbeddings()
            m._tower = VitTower(get_context(), cfg.to_dict(), w, max_batch=64, aesthetic=(aw, ab))
            self_inner._clip_model = m

    return _Seeded(), cfg, w, sd


def _clip_task(data: bytes, n_clips=1):
    from cosmos_curate_b200.data_model import Clip, SplitPipeTask, Video

    clips = [Clip(uuid=uuid.uuid4(), source_video="v.mp4", span=(0.0, 10.0), encoded_data=data) for _ in range(n_clips)]
    return SplitPipeTask(session_id="s", video=Video(input_video="v.mp4", clips=clips))


def test_extraction_then_aesthetic_filter_matches_oracle(ctx):
    """ClipFrameExtractionStage (NVDEC) -> AestheticFilterStage, the reference's stage pair, on the reference fixture."""
    from cosmos_curate_b200.interfaces import run_pipeline
    from cosmos_curate_b200.stages import AestheticFilterStage, ClipFrameExtractionStage

    data = (GOLDEN / "sintel_clip_10s.mp4").read_bytes()
    model, cfg, w, sd = _model()
    task = _clip_task(data)
    extract = ClipFrameExtractionStage(target_fps=[1, 2], log_stats=True)
    extract.stage_setup()
    extract.process_data([task])
    clip = task.video.clips[0]
    ef = clip.extracted_frames.resolve()
    assert set(ef) == {SIG1, "FrameExtractionPolicy.sequence-2000"}
    assert ef[SIG1].shape == (11, 480, 854, 3) and ef["FrameExtractionPolicy.sequence-2000"].shape == (21, 480, 854, 3)
    np.testing.assert_array_equal(ef[SIG1], ef["FrameExtractionPolicy.sequence-2000"][::2])  # LCM + stride rule
    frames = ef[SIG1].copy()
    stage = AestheticFilterStage(score_threshold=0.0, reduction="mean", log_stats=True, model=model)
    out = run_pipeline([task], [stage])
    assert out is not None and "AestheticFilterStage" in task.stage_perf and "ClipFrameExtractionStage" in task.stage_perf
    _, want = _oracle_scores(cfg, w, sd, frames)
    assert clip.aesthetic_score == pytest.approx(float(want.mean()), abs=2e-3)  # reference test tolerance (TOLERANCE = 0.002)
    assert SIG1 not in clip.extracted_frames.resolve()  # popped; the 2 fps key stays for the embedding consumer
    stage2 = AestheticFilterStage(score_threshold=float(want.min()) + 0.5, reduction="min", model=model)
    stage2._model = model
    t2 = _clip_task(data)
    t2.video.clips[0].extracted_frames = type(clip.extracted_frames)(value={SIG1: frames}, nbytes=frames.nbytes)
    stage2.stage_setup()
    stage2.process_data([t2])
    assert len(t2.video.filtered_clips) == 1 and t2.video.clip_stats.num_filtered_by_aesthetic == 1


def test_fused_nvdec_stage_matches_oracle_and_error_convention(ctx):
    from cosmos_curate_b200.interfaces import run_pipeline
    from cosmos_curate_b200.runtime import Decoder, alloc_nv12_pool
    from cosmos_curate_b200.stages import NvdecClipAestheticStage
    from oracle import color
    from tools import synth_h264

    sintel = (GOLDEN / "sintel_clip_10s.mp4").read_bytes()
    synth = synth_h264.make_clip(640, 360, 30, 3.0, seed=5, gop=30, pan=(2, 1))
    model, cfg, w, sd = _model()
    task = _clip_task(sintel, n_clips=2)
    from cosmos_curate_b200.data_model import Clip

    task.video.clips.append(Clip(uuid=uuid.uuid4(), source_video="v.mp4", span=(0, 3), encoded_data=synth))
    task.video.clips.append(Clip(uuid=uuid.uuid4(), source_video="v.mp4", span=(0, 1), encoded_data=b"\x00" * 4096))  # garbage
    task.video.clips.append(Clip(uuid=uuid.uuid4(), source_video="v.mp4", span=(0, 1)))  # no data
    stage = NvdecClipAestheticStage(score_threshold=-0.5, reduction="min", write_embedding=True, max_batch=16, num_decoders=3, log_stats=True, model=model)
    out = run_pipeline([task], [stage])
    assert out is not None
    v = task.video
    assert len(v.clips) == 3 and len(v.filtered_clips) == 2 and v.clip_stats.num_filtered_by_aesthetic == 2
    bad, empty = v.filtered_clips
    assert bad.errors["frame_extraction"] == "video_decode_failed" and bad.aesthetic_score == -1.0 and not bad.encoded_data
    assert empty.errors == {"encoded_data": "empty"} and empty.aesthetic_score == -1.0
    assert "NvdecClipAestheticStage" in task.stage_perf
    # oracle: decode the same frames with the (already validated) NVDEC wrapper, then the CPU oracle chain
    dec = Decoder(ctx)
    for clip, data, (wd, h), ids in ((v.clips[0], sintel, (854, 480), [0, 24, 48, 72, 96, 120, 144, 168, 192, 216, 239]), (v.clips[2], synth, (640, 360), [0, 30, 60, 89])):
        pool = alloc_nv12_pool(ctx, len(ids), wd, h)
        dec.decode(data, ids, pool, np.arange(len(ids)))
        nv12 = pool.buf.cpu().numpy()
        rgb = np.stack([color.nv12_to_rgb_swscale(np.ascontiguousarray(f[:, :wd]), h, wd) for f in nv12])  # the stages convert like the reference CPU decode
        emb, scores = _oracle_scores(cfg, w, sd, rgb)
        assert clip.aesthetic_score == pytest.approx(float(scores.min()), abs=3e-3)
        m = emb.mean(axis=0)
        m /= np.linalg.norm(m)
        assert np.linalg.norm(clip.openai_embedding - m) / np.linalg.norm(m) < 2e-3
    assert v.clips[0].aesthetic_score == v.clips[1].aesthetic_score  # identical clips, batch-invariant results


def test_fused_stage_on_source_video_spans(ctx):
    """source="video_span": clips are decoded out of the source video at clip.span (no transcode, SURVEY.md 8f N2)."""
    from cosmos_curate_b200 import sampling
    from cosmos_curate_b200.data_model import Clip, SplitPipeTask, Video
    from cosmos_curate_b200.interfaces import run_pipeline
    from cosmos_curate_b200.runtime import Decoder, alloc_nv12_pool, mp4_index
    from cosmos_curate_b200.stages import NvdecClipAestheticStage
    from oracle import color

    sintel = (GOLDEN / "sintel_clip_10s.mp4").read_bytes()
    model, cfg, w, sd = _model()
    spans = [(0.0, 10.0), (2.5, 7.5), (5.0, 10.0), (20.0, 21.0)]
    video = Video(input_video="v.mp4", encoded_data=sintel, clips=[Clip(uuid=uuid.uuid4(), source_video="v.mp4", span=s) for s in spans])
    task = SplitPipeTask(session_id="s", video=video)
    stage = NvdecClipAestheticStage(score_threshold=-0.5, reduction="mean", write_embedding=True, max_batch=32, num_decoders=2, source="video_span", model=model)
    assert run_pipeline([task], [stage]) is not None
    assert len(video.clips) == 3 and len(video.filtered_clips) == 1
    assert video.filtered_clips[0].errors == {"frame_extraction": "video_decode_failed"} and video.filtered_clips[0].aesthetic_score == -1.0
    assert video.encoded_data  # the source video is never dropped
    # whole-video span == the ordinary clip path on the same bytes
    t2 = _clip_task(sintel)
    run_pipeline([t2], [NvdecClipAestheticStage(score_threshold=-0.5, reduction="mean", write_embedding=True, max_batch=32, num_decoders=2, model=model)])
    assert video.clips[0].aesthetic_score == t2.video.clips[0].aesthetic_score
    assert np.array_equal(video.clips[0].openai_embedding, t2.video.clips[0].openai_embedding)
    # sub-spans against the oracle chain on the frames the span rule selects
    idx = mp4_index(sintel)
    ts = sampling.timestamps_from_index(idx["pts"], idx["timescale"])
    dec = Decoder(ctx)
    for clip in video.clips[1:]:
        ids = sampling.span_frame_ids(ts, clip.span, 1.0)
        pool = alloc_nv12_pool(ctx, len(ids), 854, 480)
        dec.decode(sintel, ids, pool, np.arange(len(ids)))
        rgb = np.stack([color.nv12_to_rgb_swscale(np.ascontiguousarray(f[:, :854]), 480, 854) for f in pool.buf.cpu().numpy()])
        _, scores = _oracle_scores(cfg, w, sd, rgb)
        assert clip.aesthetic_score == pytest.approx(float(scores.mean()), abs=3e-3)


def test_video_frame_extraction_thumbnails(ctx):
    from cosmos_curate_b200.data_model import SplitPipeTask, Video
    from cosmos_curate_b200.runtime import Decoder, alloc_nv12_pool
    from cosmos_curate_b200.stages import VideoFrameExtractionStage
    from oracle import color, preprocess

    data = (GOLDEN / "sintel_clip_10s.mp4").read_bytes()
    task = SplitPipeTask(session_id="s", video=Video(input_video="v.mp4", encoded_data=data))
    stage = VideoFrameExtractionStage(output_hw=(27, 48), log_stats=True)
    stage.stage_setup()
    stage.process_data([task])
    fa = task.video.frame_array.resolve()
    assert fa.shape == (240, 27, 48, 3) and fa.dtype == np.uint8  # TransNetV2 input of the reference (a8/a9)
    ids = [0, 100, 239]
    pool = alloc_nv12_pool(ctx, 3, 854, 480)
    Decoder(ctx).decode(data, ids, pool, [0, 1, 2])
    nv12 = pool.buf.cpu().numpy()
    for k, i in enumerate(ids):
        want = preprocess.resize_bilinear_u8(color.nv12_to_rgb(np.ascontiguousarray(nv12[k][:, :854]), 480, 854), 27, 48)
        d = np.abs(fa[i].astype(int) - want.astype(int))
        assert d.max() <= 1 and (d > 0).mean() < 5e-3
    bad = SplitPipeTask(session_id="b", video=Video(input_video="b.mp4", encoded_data=b"\x01" * 999))
    stage.process_data([bad])
    assert bad.video.errors["frame_extraction"] == "null" and not bad.video.frame_array
    with pytest.raises(ValueError):
        stage.process_data([SplitPipeTask(session_id="n", video=Video(input_video="n.mp4"))])  # "Please load video bytes!"


def test_model_interfaces_direct_calls(ctx):
    from oracle import preprocess, vit

    model, cfg, w, sd = _model()
    model.setup()
    rng = np.random.default_rng(2)
    frames = rng.integers(0, 256, size=(5, 270, 480, 3), dtype=np.uint8)
    scores = model(frames)
    assert isinstance(scores, torch.Tensor) and scores.is_cuda and scores.shape == (5,)
    emb, want = _oracle_scores(cfg, w, sd, frames)
    np.testing.assert_allclose(scores.cpu().numpy(), want, atol=3e-3)
    e2 = model._clip_model(torch.from_numpy(frames).permute(0, 3, 1, 2))  # NCHW tensor input like clip.py:64-70 accepts
    assert np.linalg.norm(e2.cpu().numpy() - emb, axis=1).max() < 2e-3
    assert model._clip_model(frames[:0]).shape == (0, cfg.proj_dim)
    with pytest.raises(ValueError):
        model(frames.astype(np.float32))
    from cosmos_curate_b200.models.aesthetics import AestheticScorer

    a = AestheticScorer(seed=3, dim=cfg.proj_dim)
    a.setup()
    np.testing.assert_allclose(a(emb).cpu().numpy(), emb @ a.w + a.b, rtol=1e-5, atol=1e-5)


def test_image_clip_embedding_stage_on_gpu(ctx):
    """ImageCLIPEmbeddingStage (image_embedding_stages.py:219-283) with the real CLIPImageEmbeddings model on the GPU:
    image.embeddings["clip"] per task against the fp32 oracle; the reference's error convention for missing image data."""
    import types

    from cosmos_curate_b200.models import weights as W
    from cosmos_curate_b200.models.clip import CLIPImageEmbeddings
    from cosmos_curate_b200.stages import ImageCLIPEmbeddingStage
    from oracle import preprocess, vit

    cfg = vit.CLIP_VIT_B32

    class _Seeded(CLIPImageEmbeddings):
        def setup(self_inner):
            from cosmos_curate_b200.runtime import VitTower, get_context

            self_inner._tower = VitTower(get_context(), cfg.to_dict(), vit.random_weights(cfg, seed=11), max_batch=8)

    def task(frame):
        img = types.SimpleNamespace(image_data=None if frame is None else types.SimpleNamespace(frames=[frame]), embeddings={}, errors={})
        return types.SimpleNamespace(image=img, stage_perf={}, session_id="s", get_major_size=lambda: 0 if frame is None else frame.nbytes)

    rng = np.random.default_rng(4)
    frames = [rng.integers(0, 256, size=s, dtype=np.uint8) for s in ((360, 640, 3), (360, 640, 3), (500, 375, 3))]
    tasks = [task(frames[0]), task(None), task(frames[1]), task(frames[2])]
    stage = ImageCLIPEmbeddingStage(model=_Seeded(), log_stats=True, stage_batch_size=4)
    stage.stage_setup()
    out = stage.process_data(tasks)
    assert out == tasks
    assert tasks[1].image.errors == {"clip_embedding": "no image_data"} and "clip" not in tasks[1].image.embeddings
    w = vit.random_weights(cfg, seed=11)
    for t, f in ((tasks[0], frames[0]), (tasks[2], frames[1]), (tasks[3], frames[2])):
        e = t.image.embeddings["clip"]
        assert isinstance(e, np.ndarray) and e.shape == (cfg.proj_dim,) and e.dtype == np.float32
        want = vit.forward(cfg, w, preprocess.clip_preprocess(f[None]))["embedding"][0]
        assert np.linalg.norm(e - want) / np.linalg.norm(want) < 1.5e-3  # 1e-3 tower budget + the <=1 LSB u8 resize budget
        assert "ImageCLIPEmbeddingStage" in t.stage_perf
    # one image per call (the reference's batch of 1) gives the same vector as the shared batch
    solo = task(frames[0])
    stage.process_data([solo])
    assert np.array_equal(solo.image.embeddings["clip"], tasks[0].image.embeddings["clip"])


def test_stage_perf_covers_the_work_and_concurrent_decode_errors(ctx):
    """a17: process_time of the fused stage is the wall time of the call (StageTimer.reinit before the work, as the reference
    does); several corrupt clips failing concurrently on different sessions each get their own error (per-thread messages)."""
    import time

    from cosmos_curate_b200.data_model import Clip
    from cosmos_curate_b200.stages import NvdecClipAestheticStage
    from tools import synth_h264

    model, cfg, w, sd = _model()
    good = synth_h264.make_clip(640, 360, 30, 2.0, seed=9, gop=30)
    task = _clip_task(good, n_clips=6)
    for k in range(6):
        task.video.clips.append(Clip(uuid=uuid.uuid4(), source_video="v.mp4", span=(0, 2), encoded_data=b"\x00" * (512 + 97 * k)))  # not an mp4
    stage = NvdecClipAestheticStage(score_threshold=-0.5, reduction="min", max_batch=16, num_decoders=6, log_stats=True, model=model)
    stage.stage_setup()
    t0 = time.time()
    stage.process_data([task])
    wall = time.time() - t0
    perf = task.stage_perf["NvdecClipAestheticStage"]
    assert 0.5 * wall <= perf.process_time <= wall + 0.05, (perf.process_time, wall)
    assert perf.input_data_size_mb > 0
    v = task.video
    assert len(v.clips) == 6 and len(v.filtered_clips) == 6
    assert all(c.errors == {"frame_extraction": "video_decode_failed"} and c.aesthetic_score == -1.0 for c in v.filtered_clips)
    assert len({c.aesthetic_score for c in v.clips}) == 1  # six identical clips, identical scores whatever batch they landed in
    stage.destroy()


def test_fused_stage_is_deterministic_at_l14_shape(ctx):
    """ADVICE r1: clips near score_threshold must not flip between runs - the L/14 shape (attention_wgmma) through the stage,
    twice, bitwise equal scores and embeddings; identical clips inside one call agree too."""
    from cosmos_curate_b200.models.clip_aesthetics import CLIPAestheticScorer
    from cosmos_curate_b200.runtime import VitTower, get_context
    from cosmos_curate_b200.stages import NvdecClipAestheticStage
    from oracle import vit

    cfg = vit.CLIP_VIT_L14
    w = vit.random_weights(cfg, seed=2)
    aw, ab = vit.collapse_aesthetic_mlp(vit.random_aesthetic_mlp(seed=2, in_dim=cfg.proj_dim))

    class _Seeded(CLIPAestheticScorer):
        def setup(self_inner):
            from cosmos_curate_b200.models.clip import CLIPImageEmbeddings

            m = CLIPImageEmbeddings()
            m._tower = VitTower(get_context(), cfg.to_dict(), w, max_batch=64, aesthetic=(aw, ab))
            self_inner._clip_model = m

    model = _Seeded()
    sintel = (GOLDEN / "sintel_clip_10s.mp4").read_bytes()
    stage = NvdecClipAestheticStage(score_threshold=-100.0, reduction="mean", write_embedding=True, max_batch=64, num_decoders=4, model=model)
    stage.stage_setup()
    runs = []
    for _ in range(2):
        task = _clip_task(sintel, n_clips=7)  # 77 frames: two tower batches
        stage.process_data([task])
        runs.append([(c.aesthetic_score, c.openai_embedding.copy()) for c in task.video.clips])
    for (s0, e0), (s1, e1) in zip(*runs):
        assert s0 == s1 and np.array_equal(e0, e1)
    assert len({s for s, _ in runs[0]}) == 1
    stage.destroy()


def test_clip_frame_extraction_target_res_mode_b(ctx):
    """ClipFrameExtractionStage(target_res=(224, 224)) - the reference benchmark's clip_extraction_target_res - returns the
    cv2 INTER_CUBIC squares (decoder_utils.py:666-670) of the NVDEC frames, and the fused stage scores them like the pair does."""
    from cosmos_curate_b200.interfaces import run_pipeline
    from cosmos_curate_b200.runtime import Decoder, alloc_nv12_pool
    from cosmos_curate_b200.stages import AestheticFilterStage, ClipFrameExtractionStage, NvdecClipAestheticStage
    from oracle import color
    from oracle import resize_cubic as R

    data = (GOLDEN / "sintel_clip_10s.mp4").read_bytes()
    ids = [0, 24, 48, 72, 96, 120, 144, 168, 192, 216, 239]
    pool = alloc_nv12_pool(ctx, len(ids), 854, 480)
    Decoder(ctx).decode(data, ids, pool, np.arange(len(ids)))
    rgb = np.stack([color.nv12_to_rgb_swscale(np.ascontiguousarray(f[:, :854]), 480, 854) for f in pool.buf.cpu().numpy()])
    for mode, fn in (("opencv", R.resize_cubic_u8), ("ipp", R.resize_cubic_real_u8)):
        task = _clip_task(data)
        st = ClipFrameExtractionStage(target_fps=[1], target_res=(224, 224), cubic_mode=mode)
        st.stage_setup()
        st.process_data([task])
        frames = task.video.clips[0].extracted_frames.resolve()[SIG1]
        assert frames.shape == (11, 224, 224, 3) and frames.dtype == np.uint8
        want = np.stack([fn(f, 224, 224) for f in rgb])
        if mode == "opencv":
            np.testing.assert_array_equal(frames, want)
        else:
            d = np.abs(frames.astype(int) - want.astype(int))
            assert d.max() <= 1 and (d > 0).mean() < 1e-4
    model, cfg, w, sd = _model()
    t_pair = _clip_task(data)
    run_pipeline([t_pair], [ClipFrameExtractionStage(target_fps=[1], target_res=(224, 224)), AestheticFilterStage(score_threshold=-9.0, reduction="mean", model=model)])
    t_fused = _clip_task(data)
    run_pipeline([t_fused], [NvdecClipAestheticStage(score_threshold=-9.0, reduction="mean", target_res=(224, 224), num_decoders=2, max_batch=16, model=model)])
    assert t_pair.video.clips[0].aesthetic_score == pytest.approx(t_fused.video.clips[0].aesthetic_score, abs=1e-6)
    _, want_scores = _oracle_scores(cfg, w, sd, want)
    assert t_fused.video.clips[0].aesthetic_score == pytest.approx(float(want_scores.mean()), abs=3e-3)


def test_fused_stage_embedding_only_with_siglip_tower(ctx):
    """score_threshold=None: an embedding-only tower (SigLIP geometry: no CLS, MAP head, mean = std = 0.5) behind the same fused
    stage - clip.openai_embedding is the output, nothing is filtered (BASELINE.json configs[3]'s embed step)."""
    from cosmos_curate_b200.interfaces import run_pipeline
    from cosmos_curate_b200.models import weights as W
    from cosmos_curate_b200.models.siglip import SigLIPImageEmbeddings
    from cosmos_curate_b200.runtime import Decoder, alloc_nv12_pool
    from cosmos_curate_b200.stages import NvdecClipAestheticStage
    from oracle import color, preprocess, vit

    cfg = W.VitConfig(image_size=224, patch=16, hidden=256, layers=2, heads=4, mlp=512, proj_dim=0, act="gelu_tanh", ln_eps=1e-6, arch="siglip")
    model = SigLIPImageEmbeddings(seed=5, max_batch=32, config=cfg)
    data = (GOLDEN / "sintel_clip_10s.mp4").read_bytes()
    task = _clip_task(data, n_clips=2)
    stage = NvdecClipAestheticStage(score_threshold=None, write_embedding=True, max_batch=32, num_decoders=2, model=model)
    assert run_pipeline([task], [stage]) is not None
    assert len(task.video.clips) == 2 and not task.video.filtered_clips and task.video.clips[0].aesthetic_score is None
    ids = [0, 24, 48, 72, 96, 120, 144, 168, 192, 216, 239]
    pool = alloc_nv12_pool(ctx, len(ids), 854, 480)
    Decoder(ctx).decode(data, ids, pool, np.arange(len(ids)))
    rgb = np.stack([color.nv12_to_rgb_swscale(np.ascontiguousarray(f[:, :854]), 480, 854) for f in pool.buf.cpu().numpy()])
    ocfg = vit.VitConfig(**cfg.to_dict())
    ref = vit.forward(ocfg, W.seeded_weights(cfg, 5), preprocess.clip_preprocess(rgb, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5)))["embedding"]
    m = ref.mean(axis=0)
    m /= np.linalg.norm(m)
    e = task.video.clips[0].openai_embedding
    assert e.shape == (256,) and np.linalg.norm(e - m) / np.linalg.norm(m) < 2e-3
    assert np.array_equal(e, task.video.clips[1].openai_embedding)
    with pytest.raises(ValueError):
        NvdecClipAestheticStage(score_threshold=0.5, write_embedding=True, model=SigLIPImageEmbeddings(seed=5, config=cfg)).stage_setup()


def test_fused_stage_keyframe_seek_gives_identical_results(ctx):
    """seek_keyframes=True decodes only the GOPs that hold sampled frames; scores and embeddings are bitwise those of the default
    (every frame decoded, the reference's decode work) - on a multi-GOP residual-coded clip."""
    from cosmos_curate_b200.stages import NvdecClipAestheticStage
    from tools import synth_h264

    clip = synth_h264.make_coded_clip(640, 368, 30, 6.0, seed=17, bitrate=1.5e6)
    model, cfg, w, sd = _model()
    out = {}
    for seek in (False, True):
        task = _clip_task(clip, n_clips=3)
        st = NvdecClipAestheticStage(score_threshold=-100.0, reduction="mean", write_embedding=True, max_batch=32, num_decoders=3, seek_keyframes=seek, model=model)
        st.stage_setup()
        st.process_data([task])
        out[seek] = ([c.aesthetic_score for c in task.video.clips], [c.openai_embedding for c in task.video.clips], st.last_call_stats["frames_decoded"])
        st.destroy()
    assert out[False][0] == out[True][0] and all(np.array_equal(a, b) for a, b in zip(out[False][1], out[True][1]))
    assert out[True][2] < out[False][2] == 3 * 180  # 7 sampled frames per clip: the seek mode skips most of every GOP


def test_fused_stage_mixed_resolutions_in_one_call(ctx):
    """BASELINE.json configs[4] mixes 720p / 1080p / 4K clips in one stream: clips of different sizes inside ONE process_data call go
    through per-resolution surface-pool rings and batches; every clip gets the score it gets when processed alone, also the clips
    that share a batch with a clip whose decode fails."""
    import struct

    from cosmos_curate_b200.data_model import Clip
    from cosmos_curate_b200.stages import NvdecClipAestheticStage
    from tools import synth_h264

    # 640x368 like sources[0], a valid index, every sample's NAL length past the sample: demuxes, fails to decode
    undecodable = synth_h264.mux_mp4([struct.pack(">I", 1 << 20) + bytes(16)] * 60, [i % 30 == 0 for i in range(60)], synth_h264.sps(640, 368, 30),
                                     synth_h264.pps(), 640, 368, 30)  # fmt: skip
    sources = [synth_h264.make_coded_clip(640, 368, 30, 2.0, seed=31, bitrate=1.0e6), synth_h264.make_coded_clip(1280, 720, 30, 2.0, seed=32, bitrate=2.0e6),
               (GOLDEN / "sintel_clip_10s.mp4").read_bytes(), synth_h264.make_coded_clip(1920, 1080, 30, 2.0, seed=33, bitrate=4.0e6), undecodable]
    model, cfg, w, sd = _model()
    stage = NvdecClipAestheticStage(score_threshold=-100.0, reduction="mean", write_embedding=True, max_batch=16, num_decoders=4, model=model)
    stage.stage_setup()
    alone = []
    for s in sources[:4]:
        t = _clip_task(s)
        stage.process_data([t])
        alone.append((t.video.clips[0].aesthetic_score, t.video.clips[0].openai_embedding))
    # interleaved sizes, more frames than one batch holds (max_batch = 16); the undecodable clip (4) shares a batch with two of 0
    order = [0, 1, 4, 2, 3, 1, 0, 3, 2, 2, 1]
    task = _clip_task(sources[0], n_clips=0)
    task.video.clips = [Clip(uuid=uuid.uuid4(), source_video="v.mp4", span=(0.0, 2.0), encoded_data=sources[k]) for k in order]
    stage.process_data([task])
    assert len(task.video.clips) == len(order)
    for clip, k in zip(task.video.clips, order):
        if k == 4:
            assert clip.errors == {"frame_extraction": "video_decode_failed"} and clip.aesthetic_score == -1.0 and clip.openai_embedding is None
            continue
        assert clip.aesthetic_score == alone[k][0] and np.array_equal(clip.openai_embedding, alone[k][1]), k
    assert stage.last_call_stats["batches"] >= 4
    stage.destroy()


def test_internvideo2_frame_creation_stage_matches_the_reference_formulation(ctx):
    """InternVideo2FrameCreationStage (internvideo2_stages.py:43-184): `clip.intern_video_2_frames` bit-equal to the
    reference's _construct_frames arithmetic (oracle/video_tube.py, pinned to the imported reference) on the frames the
    upstream extraction stage delivered; the NVDEC-direct source gives the same tube without host frames; short clips are
    re-sampled at a doubled rate; the reference's error keys."""
    from cosmos_curate_b200.data_model import Clip
    from cosmos_curate_b200.interfaces import run_pipeline
    from cosmos_curate_b200.stages import ClipFrameExtractionStage, InternVideo2FrameCreationStage
    from oracle import video_tube as T
    from tools import synth_h264

    sig2 = "FrameExtractionPolicy.sequence-2000"
    sintel = (GOLDEN / "sintel_clip_10s.mp4").read_bytes()
    short = synth_h264.make_clip(640, 360, 30, 1.5, seed=9, gop=30, pan=(1, 2))  # 45 frames: 2 fps -> 4, 4 fps -> 7, 8 fps -> 13 frames
    task = _clip_task(sintel)
    task.video.clips.append(Clip(uuid=uuid.uuid4(), source_video="v.mp4", span=(0, 1.5), encoded_data=short))
    task.video.clips.append(Clip(uuid=uuid.uuid4(), source_video="v.mp4", span=(0, 1)))  # no data
    task.video.clips.append(Clip(uuid=uuid.uuid4(), source_video="v.mp4", span=(0, 1), encoded_data=sintel))  # data, no frames
    extract = ClipFrameExtractionStage(target_fps=[2])
    extract.stage_setup()
    extract.process_data([task])
    task.video.clips[3].extracted_frames.drop()
    frames = [c.extracted_frames.resolve()[sig2].copy() for c in task.video.clips[:2]]
    assert frames[0].shape == (21, 480, 854, 3) and frames[1].shape[0] < 8
    stage = InternVideo2FrameCreationStage(target_fps=2.0, log_stats=True)
    assert stage.resources.cpus == 1.0 and stage.model.get_target_num_frames() == 8
    out = run_pipeline([task], [stage])
    assert out is not None and "InternVideo2FrameCreationStage" in task.stage_perf
    c0, c1, c2, c3 = task.video.clips
    tube0 = c0.intern_video_2_frames.resolve()
    assert tube0.shape == (1, 8, 3, 224, 224) and tube0.dtype == np.float32
    np.testing.assert_array_equal(tube0, T.construct_frames(list(frames[0])))
    assert not c0.extracted_frames  # last consumer: dropped (internvideo2_stages.py:178)
    assert c2.errors == {"encoded_data": "empty"} and not c2.intern_video_2_frames
    assert c3.errors == {f"frames-{sig2}": "missing"} and not c3.intern_video_2_frames
    # short clip: re-extracted at 8 fps (13 frames), stride 1, first 8 kept
    ext8 = ClipFrameExtractionStage(target_fps=[8])
    ext8.stage_setup()
    t8 = _clip_task(short)
    ext8.process_data([t8])
    f8 = t8.video.clips[0].extracted_frames.resolve()["FrameExtractionPolicy.sequence-8000"]
    assert f8.shape[0] >= 8
    np.testing.assert_array_equal(c1.intern_video_2_frames.resolve(), T.construct_frames(list(f8)))
    # NVDEC-direct source: same tubes, no upstream extraction stage
    t_dir = _clip_task(sintel)
    t_dir.video.clips.append(Clip(uuid=uuid.uuid4(), source_video="v.mp4", span=(0, 1.5), encoded_data=short))
    t_dir.video.clips.append(Clip(uuid=uuid.uuid4(), source_video="v.mp4", span=(0, 1), encoded_data=b"\x00" * 4096))
    tiny = synth_h264.make_clip(320, 192, 30, 0.2, seed=3, gop=30)  # 6 frames: never reaches 8 below 20 fps
    t_dir.video.clips.append(Clip(uuid=uuid.uuid4(), source_video="v.mp4", span=(0, 0.2), encoded_data=tiny))
    run_pipeline([t_dir], [InternVideo2FrameCreationStage(target_fps=2.0, source="nvdec")])
    d0, d1, d2, d3 = t_dir.video.clips
    np.testing.assert_array_equal(d0.intern_video_2_frames.resolve(), tube0)
    np.testing.assert_array_equal(d1.intern_video_2_frames.resolve(), c1.intern_video_2_frames.resolve())
    assert d2.errors["frame_extraction"] == "video_decode_failed" and not d2.intern_video_2_frames
    assert d3.intern_video_2_frames.resolve().shape == (0,) and not d3.errors  # the reference's empty array for too short clips


def test_local_split_pipeline_chain_from_file_to_dedup(ctx, tmp_path):
    """The whole slice a user of the reference's split pipeline would run here, stage classes only: VideoDownloader ->
    FixedStrideExtractorStage -> ClipStreamCopyStage (re-chunking like ClipTranscodingStage) -> NvdecClipAestheticStage ->
    the ClipWriterStage file layout -> the dedup reader -> semdedup_cluster.  Checks the plumbing (tasks multiply at the chunking
    stage, every clip is scored and embedded, files round-trip); the numbers themselves are pinned by the tests above."""
    import shutil

    from cosmos_curate_b200 import dedup as D
    from cosmos_curate_b200 import embedding_io as E
    from cosmos_curate_b200.data_model import SplitPipeTask, Video
    from cosmos_curate_b200.interfaces import run_pipeline
    from cosmos_curate_b200.stages import ClipStreamCopyStage, FixedStrideExtractorStage, NvdecClipAestheticStage, VideoDownloader

    src = tmp_path / "sintel.mp4"
    shutil.copy(GOLDEN / "sintel_clip_10s.mp4", src)
    model, _, _, _ = _model()
    stages = [VideoDownloader(log_stats=True), FixedStrideExtractorStage(clip_len_s=4, clip_stride_s=3, min_clip_length_s=2, log_stats=True),
              ClipStreamCopyStage(num_clips_per_chunk=1, snap_spans=False, log_stats=True),
              NvdecClipAestheticStage(score_threshold=-9.0, reduction="mean", write_embedding=True, max_batch=32, num_decoders=2, log_stats=True, model=model)]
    out = run_pipeline([SplitPipeTask(session_id=str(src), video=Video(input_video=src))], stages)
    assert out is not None and len(out) == 2  # spans (0,4) (3,7) (6,10) (9,10 dropped: < 2 s): 4 + 4 s close a chunk, the third clip forms the next
    clips = [c for t in out for c in t.video.clips]
    assert [c.span for c in clips] == [(0.0, 4.0), (3.0, 7.0), (6.0, 10.0)]
    assert all(c.aesthetic_score is not None and c.aesthetic_score > -1.0 and c.openai_embedding.shape == (model.tower.out_dim,) for c in clips)
    assert all(abs(float(np.linalg.norm(c.openai_embedding)) - 1.0) < 1e-5 for c in clips)
    assert {"VideoDownloader", "FixedStrideExtractorStage", "ClipStreamCopyStage", "NvdecClipAestheticStage"} <= set(out[0].stage_perf)
    assert [t.video.clip_chunk_index for t in out] == [0, 1] and out[0].video.num_total_clips == 3
    for t in out:
        E.write_task_outputs(t, str(tmp_path / "out"), "openai")
    files = sorted((tmp_path / "out" / "openai_embd_parquet").glob("*.parquet"))
    assert len(files) == 2  # one per (video, chunk)
    ids, emb = E.read_embedding_parquets([str(f) for f in files])
    assert sorted(ids.tolist()) == sorted(str(c.uuid) for c in clips) and emb.shape == (3, model.tower.out_dim)
    by_id = {str(c.uuid): c.openai_embedding for c in clips}
    np.testing.assert_array_equal(emb, np.stack([by_id[i] for i in ids.tolist()]))
    r = D.semdedup_cluster(ids, emb, np.zeros(3, np.float32), eps=0.01)
    assert r["total"] == 3 and len(r["id"]) == 3

