"""InternVideo2 from decoded surfaces on the GPU: cb_video_tube_patches against cb_tube_patches(cb_video_tube(...)) in every fp16 bit,
cb_iv2_embed_surfaces against cb_iv2_forward of cb_video_tube's tubes (chunk tail, n_clips = 0, argument and state errors), and
NvdecInternVideo2EmbeddingStage against InternVideo2FrameCreationStage(source="nvdec") -> InternVideo2EmbeddingStage on the same tasks."""

from __future__ import annotations

import ctypes as C
import uuid

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from cosmos_curate_b200.data_model import Clip, SplitPipeTask, Video
from gpu_helpers import ctx  # noqa: F401

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE = -2, -6
VOCAB = GOLDEN / "bert_vocab_synth.txt"


def _stream():
    from cosmos_curate_b200.runtime import _stream_ptr

    return _stream_ptr()


def _pool(ctx, fmt: str, w: int, h: int, n: int, seed: int):
    """n random frames of w x h as an NV12 ("opencv" / "swscale" colour) or RGB24 pool."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if fmt == "rgb":
        return ctx.rgb_pool(torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device="cuda", generator=g))
    pitch = (w + 255) // 256 * 256
    buf = torch.randint(0, 256, (n, h + h // 2, pitch), dtype=torch.uint8, device="cuda", generator=g)
    return ctx.nv12_pool(buf, w, h, h, colour=fmt)


def _slots(arr):
    a = np.ascontiguousarray(arr, dtype=np.int32)
    return a, a.ctypes.data_as(C.POINTER(C.c_int32))


def _f3(v):
    return (C.c_float * 3)(*v)


# ------------------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("fmt", ["opencv", "swscale", "rgb"])
@pytest.mark.parametrize(("w", "h"), [(854, 480), (448, 448), (224, 224), (320, 180)])  # linear, 2x2 area, copy, upscale
@pytest.mark.parametrize(("patch", "k_pad"), [(14, 640), (14, 588), (16, 770)])
def test_video_tube_patches_equals_tube_then_patches(ctx, fmt, w, h, patch, k_pad):
    from cosmos_curate_b200.runtime import IMAGENET_MEAN, IMAGENET_STD, check

    size = 224
    pool = _pool(ctx, fmt, w, h, 5, seed=w + h + k_pad)
    slots, ptr = _slots([3, 0, 3, 4, 1, 1, 2])  # out of order, repeated
    n, g = len(slots), size // patch
    tube = ctx.video_tube(pool, size, size, slots=slots)
    want = torch.full((n * g * g + 1, k_pad), float("nan"), dtype=torch.float16, device="cuda")
    check(ctx.lib.cb_tube_patches(ctx.h, tube.data_ptr(), want.data_ptr(), n, size, patch, k_pad, _stream()), "cb_tube_patches", ctx.h)
    got = torch.full_like(want, float("nan"))
    check(ctx.lib.cb_video_tube_patches(ctx.h, C.byref(pool.desc), ptr, n, size, patch, k_pad, _f3(IMAGENET_MEAN), _f3(IMAGENET_STD),
                                        got.data_ptr(), _stream()), "cb_video_tube_patches", ctx.h)  # fmt: skip
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), f"{fmt} {w}x{h} patch {patch} k_pad {k_pad}"
    assert torch.isnan(got[-1]).all(), "a row past the output was written"
    assert (got[:-1, 3 * patch * patch :].view(torch.int16) == 0).all()  # pad columns are +0


def test_video_tube_patches_argument_errors(ctx):
    from cosmos_curate_b200.runtime import IMAGENET_MEAN, IMAGENET_STD

    pool = _pool(ctx, "opencv", 448, 448, 2, seed=1)
    slots, ptr = _slots([0, 1])
    out = torch.empty((2 * 256, 640), dtype=torch.float16, device="cuda")
    m, s = _f3(IMAGENET_MEAN), _f3(IMAGENET_STD)

    def call(n=2, size=224, patch=14, k_pad=640, mean=m, std=s, o=out.data_ptr(), sl=ptr):
        return ctx.lib.cb_video_tube_patches(ctx.h, C.byref(pool.desc), sl, n, size, patch, k_pad, mean, std, o, _stream())

    assert call(k_pad=587) == ERR_ARG and call(k_pad=586) == ERR_ARG and call(size=12) == ERR_ARG and call(patch=0) == ERR_ARG
    assert call(n=-1) == ERR_ARG and call(o=None) == ERR_ARG and call(mean=None) == ERR_ARG and call(sl=None) == ERR_ARG
    assert call(o=out.data_ptr() + 1) == ERR_ARG
    assert call(n=0, o=None) == 0  # a no-op
    assert call() == 0


# ------------------------------------------------------------------------------------------------------------ entry point
@pytest.fixture(scope="module")
def tower(ctx):
    from cosmos_curate_b200.models.internvideo2 import IV2_1B_CFG, seeded_weights
    from cosmos_curate_b200.runtime import Iv2Tower

    cfg = dict(IV2_1B_CFG, layers=2)
    t = Iv2Tower(ctx, cfg, seeded_weights(cfg, 7), max_clips=2)
    yield t
    t.close()


@pytest.mark.parametrize(("fmt", "w", "h"), [("swscale", 854, 480), ("opencv", 448, 448), ("rgb", 224, 224)])
def test_embed_surfaces_equals_forward_of_the_tube(ctx, tower, fmt, w, h):
    pool = _pool(ctx, fmt, w, h, 9, seed=w)
    slots = np.array([8, 0, 3, 3, 1, 2, 4, 5, 7, 7, 7, 6, 0, 1, 2, 8, 5, 3, 1, 0], dtype=np.int32)  # 5 clips: chunks 2, 2, 1
    got = tower.embed_pool(pool, slots)
    tubes = ctx.video_tube(pool, 224, 224, slots=slots).view(5, 4, 3, 224, 224)
    want = tower.forward(tubes)
    torch.cuda.synchronize()
    assert got.shape == (5, 512) and torch.equal(got, want)
    one = tower.embed_pool(pool, slots[8:12])  # a clip's embedding does not depend on its chunk
    assert torch.equal(one[0], got[2])


def test_embed_surfaces_errors_and_empty_call(ctx, tower):
    from cosmos_curate_b200.models.internvideo2 import IV2_1B_CFG, seeded_weights
    from cosmos_curate_b200.runtime import IMAGENET_MEAN, IMAGENET_STD

    pool = _pool(ctx, "opencv", 448, 448, 4, seed=3)
    slots, ptr = _slots([0, 1, 2, 3])
    emb = torch.full((1, 512), float("nan"), device="cuda")
    m, s = _f3(IMAGENET_MEAN), _f3(IMAGENET_STD)

    def call(n=1, pl=C.byref(pool.desc), sl=ptr, mean=m, std=s, out=emb.data_ptr()):
        return ctx.lib.cb_iv2_embed_surfaces(tower.h, pl, sl, n, mean, std, out, _stream())

    assert call(n=0, sl=None, out=None) == 0 and torch.isnan(emb).all()  # n_clips == 0: nothing written
    for kw in ({"n": -1}, {"pl": None}, {"sl": None}, {"mean": None}, {"std": None}, {"out": None}):
        assert call(**kw) == ERR_ARG, kw
    assert ctx.lib.cb_iv2_embed_surfaces(None, C.byref(pool.desc), ptr, 1, m, s, emb.data_ptr(), _stream()) == ERR_ARG
    assert torch.isnan(emb).all()
    cls = np.ascontiguousarray(seeded_weights(dict(IV2_1B_CFG, layers=2), 7)["cls"])
    assert ctx.lib.cb_iv2_set_tensor(tower.h, b"cls", cls.ctypes.data_as(C.POINTER(C.c_float)), cls.size) == 0
    assert call() == ERR_STATE  # un-finalized by set_tensor
    assert ctx.lib.cb_iv2_finalize(tower.h, 2) == 0
    assert call() == 0
    torch.cuda.synchronize()
    assert torch.equal(emb, tower.forward(ctx.video_tube(pool, 224, 224, slots=slots).view(1, 4, 3, 224, 224)))


# ------------------------------------------------------------------------------------------------------------ stage vs chain
def _task_clips():
    from tools import synth_h264

    sintel = (GOLDEN / "sintel_clip_10s.mp4").read_bytes()
    a = [synth_h264.make_clip(640, 360, 30, 3.0, seed=s, gop=30, pan=(2, 1)) for s in range(4)]
    b = [synth_h264.make_clip(320, 192, 30, 2.0, seed=10 + s, gop=15, pan=(1, 2)) for s in range(3)]
    regen = synth_h264.make_clip(320, 192, 30, 0.4, seed=20, gop=15)  # 12 frames: 4 kept only at a doubled rate
    short = synth_h264.make_clip(640, 360, 30, 0.1, seed=21, gop=15)  # 3 frames: too short at any rate
    return [sintel, a[0], b[0], regen, a[1], None, b[1], short, a[2], b"\x00not an mp4" * 20, b[2], a[3], a[0]]


def _tasks(datas):
    clips = [Clip(uuid=uuid.uuid5(uuid.NAMESPACE_URL, f"iv2f{i}"), source_video="v.mp4", span=(0.0, 3.0), encoded_data=d) for i, d in enumerate(datas)]
    return [SplitPipeTask(session_id="s", video=Video(input_video=f"v{t}.mp4", clips=clips[t::3])) for t in range(3)]


@pytest.fixture(scope="module")
def model(ctx):
    from cosmos_curate_b200.models.bert_tokenizer import BertTokenizer
    from cosmos_curate_b200.models.internvideo2 import IV2_1B_CFG, IV2_TEXT_CFG, InternVideo2MultiModality

    tok = BertTokenizer.from_file(VOCAB)
    vcfg, tcfg = dict(IV2_1B_CFG, layers=2), dict(IV2_TEXT_CFG, layers=2, vocab=len(tok.vocab))
    m = InternVideo2MultiModality(seed=7, config=vcfg, text_config=tcfg, vocab_file=VOCAB, max_clips=8)
    m.setup()
    return m


def test_fused_stage_equals_the_chain(ctx, model, monkeypatch):
    from cosmos_curate_b200.compare import compare_tasks
    from cosmos_curate_b200.models.internvideo2_frames import InternVideo2FrameFormulator
    from cosmos_curate_b200.stages import InternVideo2EmbeddingStage, InternVideo2FrameCreationStage, NvdecInternVideo2EmbeddingStage

    datas = _task_clips()
    texts = ["a red car on a road", "waves on a beach", "a snowy mountain", "people dancing"]
    monkeypatch.setattr(InternVideo2FrameCreationStage, "GROUP", 4)  # several decode groups per resolution
    monkeypatch.setattr(NvdecInternVideo2EmbeddingStage, "GROUP", 4)

    chain = _tasks(datas)
    frames = InternVideo2FrameCreationStage(target_fps=2.0, source="nvdec", num_decoders=3, model=InternVideo2FrameFormulator(num_frames=4))
    frames.stage_setup()
    frames.process_data(chain)
    embed = InternVideo2EmbeddingStage(batch_size=8, texts_to_verify=texts, model=model)
    embed.stage_setup()
    embed.process_data(chain)
    frames.destroy()

    flat = [c for t in chain for c in t.video.clips]
    assert sum(c.intern_video_2_embedding is not None for c in flat) == 10
    assert {tuple(sorted(c.errors.items())) for c in flat if c.errors} == {
        (("encoded_data", "empty"), ("iv2_frames", "none")), (("iv2_frames", "empty"),),
        (("frame_extraction", "video_decode_failed"), ("iv2_frames", "none"))}  # fmt: skip

    for seek in (False, True):
        fused = _tasks(datas)
        stage = NvdecInternVideo2EmbeddingStage(batch_size=3, texts_to_verify=texts, num_decoders=3, seek_keyframes=seek, log_stats=True, model=model)
        stage.stage_setup()
        stage.process_data(fused)
        stats = dict(stage.last_call_stats)
        stage.destroy()
        diffs = compare_tasks(chain, fused, atol=0)
        assert diffs == [], (seek, diffs[:5])
        assert all("NvdecInternVideo2EmbeddingStage" in t.stage_perf for t in fused)
        assert stats["groups"] == 4 and stats["frames_decoded"] > 0, stats
        print(f"\nseek_keyframes={seek}: {stats}")
