"""CPU tests of NvdecInternVideo2EmbeddingStage's host contract, with a fake tower, a fake decoder pool and fake surface pools.

The fakes make each embedding a function of the (clip bytes, frame id) pairs its slots hold, so the same clips run through the pair
InternVideo2FrameCreationStage(source="nvdec") -> InternVideo2EmbeddingStage (whose fake formulator writes those pairs into the tube)
and through the fused stage must leave equal tasks: the error table, the kept frames, the chunking and the text match."""

from __future__ import annotations

import pickle
import types
import uuid
import zlib
from concurrent.futures import Future

import numpy as np
import pytest
import torch

from cosmos_curate_b200 import runtime
from cosmos_curate_b200._lib import CurateB200Error
from cosmos_curate_b200.compare import compare_tasks
from cosmos_curate_b200.data_model import Clip, SplitPipeTask, Video
from cosmos_curate_b200.models.internvideo2 import InternVideo2MultiModality
from tools import synth_h264

CTX = types.SimpleNamespace(device=0)
FRAMES = 4
DIM = 512


class _Pool:
    """A surface pool that remembers which (clip tag, frame id) each slot holds."""

    def __init__(self, slots, width, height):
        self.buf = np.empty((slots, 0, 0), dtype=np.uint8)
        self.size = (width, height)
        self.held: dict[int, tuple[int, int]] = {}


def _tag(data) -> int:
    return zlib.crc32(data if isinstance(data, bytes) else np.asarray(data, dtype=np.uint8).tobytes())


def _embedding(frames) -> np.ndarray:
    """The fake tower: a unit vector from the clip's (tag, frame id) pairs, in order."""
    seed = zlib.crc32(repr([(int(t), int(f)) for t, f in frames]).encode())
    e = np.random.default_rng(seed).standard_normal(DIM)
    return (e / np.linalg.norm(e)).astype(np.float32)


class _Decoders:
    """DecoderPool.submit_group with no decoder: fills the fake pool's slots, fails the clips in `bad`."""

    def __init__(self, bad=()):
        self.bad, self.groups, self.seek = {_tag(b) for b in bad}, [], []

    def submit_group(self, pool, shape, jobs, seek_keyframes=False):
        assert shape == pool.size
        self.groups.append(len(jobs))
        self.seek.append(seek_keyframes)
        out, first = [], 0
        for data, ids in jobs:
            f = Future()
            if _tag(data) in self.bad:
                f.set_exception(CurateB200Error(-4, "cb_decoder_decode", "decode: corrupt slice"))
            else:
                for k, i in enumerate(ids):
                    pool.held[first + k] = (_tag(data), int(i))
                f.set_result({"frames_decoded": int(ids[-1]) + 1, "frames_emitted": len(ids)})
            out.append((first, f))
            first += len(ids)
        return out

    def close(self):
        pass


class _Tower:
    frames, embed_dim = FRAMES, DIM

    def __init__(self):
        self.calls: list[int] = []

    def embed_pool(self, pool, slots, mean=None, std=None):
        assert len(slots) % FRAMES == 0 and (tuple(mean), tuple(std)) == (runtime.IMAGENET_MEAN, runtime.IMAGENET_STD)
        self.calls.append(len(slots) // FRAMES)
        held = [pool.held[int(s)] for s in slots]
        return torch.from_numpy(np.stack([_embedding(held[i : i + FRAMES]) for i in range(0, len(held), FRAMES)]))


class _Model:
    """The InternVideo2 model as both stages use it: tower, frame count, texts and the reference's evaluate."""

    evaluate = staticmethod(InternVideo2MultiModality.evaluate)

    def __init__(self, text=True):
        self._tower = None
        if not text:
            self.encode_texts = None

    def setup(self):
        self._tower = self._tower or _Tower()

    @property
    def tower(self):
        return self._tower

    def get_target_num_frames(self):
        return FRAMES

    def encode_texts(self, texts):
        return np.stack([_embedding([(zlib.crc32(t.encode()), 0)]) for t in texts])

    def encode_batched_videos(self, videos, batch_size):  # the pair's tower: the tube holds the (tag, frame id) pairs
        return [_embedding([tuple(v[0, f, :2, 0, 0].astype(np.int64)) for f in range(FRAMES)])[None] for v in videos]


class _Formulator:
    """The pair's formulator: tube channel 0 / 1 = the slot's (tag, frame id)."""

    def __init__(self):
        self.pool = None

    def setup(self):
        pass

    def get_target_num_frames(self):
        return FRAMES

    def formulate_pool(self, pool, slots):
        out = torch.zeros((len(slots), 3, 1, 1), dtype=torch.float64)
        for i, s in enumerate(slots):
            out[i, 0], out[i, 1] = pool.held[int(s)]
        return out


@pytest.fixture
def fakes(monkeypatch):
    from cosmos_curate_b200.stages import internvideo2_frames, internvideo2_fused

    monkeypatch.setattr(runtime, "alloc_nv12_pool", lambda ctx, slots, w, h, colour="opencv": _Pool(slots, w, h))
    for mod in (internvideo2_frames, internvideo2_fused):
        monkeypatch.setattr(mod, "get_context", lambda: CTX)
    monkeypatch.setattr(internvideo2_fused, "nvdec_available", lambda ctx: True)

    class _Event:
        def record(self, stream):
            pass

        def synchronize(self):
            pass

    monkeypatch.setattr(torch.cuda, "current_stream", lambda: None)
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    return internvideo2_fused


def _clips():
    """Every row of the error table, two resolutions interleaved, a supersampled short clip and more clips than one decode group."""
    from conftest import GOLDEN

    sintel = (GOLDEN / "sintel_clip_10s.mp4").read_bytes()
    small = [synth_h264.make_clip(320, 192, 30, 1.0, seed=s, gop=15) for s in range(3)]
    other = [synth_h264.make_clip(256, 144, 30, 1.0, seed=10 + s, gop=15) for s in range(2)]
    regen = synth_h264.make_clip(320, 192, 30, 0.4, seed=20, gop=15)  # 12 frames: 4 kept only at a doubled rate
    short = synth_h264.make_clip(320, 192, 30, 0.1, seed=21, gop=15)  # 3 frames: too short at any rate
    broken = synth_h264.make_clip(256, 144, 30, 1.0, seed=22, gop=15)  # demuxes, fails to decode
    datas = [sintel, small[0], other[0], regen, None, small[1], short, b"\x00not an mp4" * 9, other[1], broken, small[2]]
    datas += [small[i % 3] for i in range(6)]  # 17 decodable clips with GROUP = 4 below: several groups per resolution
    return datas, broken


def _tasks(datas):
    clips = [Clip(uuid=uuid.uuid5(uuid.NAMESPACE_URL, f"c{i}"), source_video="v.mp4", span=(0.0, 1.0), encoded_data=d) for i, d in enumerate(datas)]
    return [SplitPipeTask(session_id="s", video=Video(input_video=f"v{t}.mp4", clips=clips[t::3])) for t in range(3)]


def test_fused_stage_leaves_the_pairs_state(fakes, monkeypatch):
    from cosmos_curate_b200.stages import InternVideo2EmbeddingStage, InternVideo2FrameCreationStage, NvdecInternVideo2EmbeddingStage

    datas, broken = _clips()
    texts = ["a red car", "a dog on a beach", "snow"]
    monkeypatch.setattr(InternVideo2FrameCreationStage, "GROUP", 4)

    pair_tasks = _tasks(datas)
    frames = InternVideo2FrameCreationStage(source="nvdec", model=_Formulator())
    frames.stage_setup()
    frames._decode_pool = _Decoders(bad=[broken])
    frames.process_data(pair_tasks)
    embed = InternVideo2EmbeddingStage(batch_size=3, texts_to_verify=texts, model=_Model())
    embed.stage_setup()
    embed.process_data(pair_tasks)

    fused_tasks = _tasks(datas)
    monkeypatch.setattr(NvdecInternVideo2EmbeddingStage, "GROUP", 4)
    stage = NvdecInternVideo2EmbeddingStage(batch_size=3, texts_to_verify=texts, log_stats=True, model=_Model())
    monkeypatch.setattr(fakes, "DecoderPool", lambda ctx, n: _Decoders(bad=[broken]))
    stage.stage_setup()
    assert stage.process_data(fused_tasks) is fused_tasks

    assert compare_tasks(pair_tasks, fused_tasks, atol=0) == []
    clips = [c for t in fused_tasks for c in t.video.clips]
    errors = sorted(tuple(sorted(c.errors.items())) for c in clips if c.errors)
    assert errors == sorted([(("encoded_data", "empty"), ("iv2_frames", "none")),
                             (("iv2_frames", "empty"),),
                             (("frame_extraction", "video_decode_failed"), ("iv2_frames", "none")),
                             (("frame_extraction", "video_decode_failed"), ("iv2_frames", "none"))])  # fmt: skip
    done = [c for c in clips if not c.errors]
    assert len(done) == 13 and all(c.intern_video_2_embedding.shape == (1, DIM) and c.intern_video_2_embedding.dtype == np.float32 for c in done)
    assert all(c.intern_video_2_text_match[0] in texts for c in done)
    assert all(c.intern_video_2_frames.resolve() is None for c in clips)
    assert all(c.intern_video_2_embedding is None and c.intern_video_2_text_match is None for c in clips if c.errors)
    assert stage.last_call_stats["groups"] == 5 and stage.last_call_stats["nvdec_sessions"] == 8 and not stage.last_call_stats["host_decode"]
    assert stage.last_call_stats["frames_decoded"] > 0
    assert max(stage._model.tower.calls) <= 3  # tower chunks of batch_size clips
    assert all(t.stage_perf.keys() == {"NvdecInternVideo2EmbeddingStage"} for t in fused_tasks)
    assert stage._decode_pool.seek == [False] * 5


def test_seek_keyframes_passes_through(fakes, monkeypatch):
    from cosmos_curate_b200.stages import NvdecInternVideo2EmbeddingStage

    stage = NvdecInternVideo2EmbeddingStage(seek_keyframes=True, model=_Model())
    decoders = _Decoders()
    monkeypatch.setattr(fakes, "DecoderPool", lambda ctx, n: decoders)
    stage.stage_setup()
    tasks = _tasks([synth_h264.make_clip(320, 192, 30, 1.0, seed=s, gop=15) for s in range(3)])
    stage.process_data(tasks)
    assert decoders.seek == [True]
    assert all(c.intern_video_2_embedding is not None for t in tasks for c in t.video.clips)


def test_refusals_resources_and_pickling():
    from cosmos_curate_b200.stages import NvdecInternVideo2EmbeddingStage

    with pytest.raises(ValueError, match="texts_to_verify is empty"):
        NvdecInternVideo2EmbeddingStage(texts_to_verify=[], model=_Model())
    with pytest.raises(ValueError, match="needs a model that embeds text"):
        NvdecInternVideo2EmbeddingStage(texts_to_verify=["a cat"], model=_Model(text=False))
    with pytest.raises(ValueError, match="colour"):
        NvdecInternVideo2EmbeddingStage(colour="bt709", model=_Model())
    stage = NvdecInternVideo2EmbeddingStage(num_gpus_per_worker=0.5, stage_batch_size=5, texts_to_verify=["a cat"],
                                            model=InternVideo2MultiModality(seed=0))  # fmt: skip
    assert stage.stage_batch_size == 5 and stage.resources.gpus == 0.5
    assert NvdecInternVideo2EmbeddingStage(model=_Model()).resources.gpus == 1.0
    again = pickle.loads(pickle.dumps(stage))  # before setup: no CUDA, NVDEC or weights held
    assert again.stage_batch_size == 5 and again._text_match._texts == ["a cat"] and again._pools is None and again._decode_pool is None
