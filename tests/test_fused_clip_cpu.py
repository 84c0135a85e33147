"""CPU tests of NvdecClipAestheticStage's host contract, with a fake tower, a fake decoder pool and fake surface pools.

The fakes make each frame's embedding and score a function of the (clip bytes, frame id) pair its slot holds, so every clip's
expected score and embedding follow from the sampling rules alone: the batching per resolution, the error table, the reductions,
the filter, the target_res and video_span paths and the write-back are checked without a GPU."""

from __future__ import annotations

import uuid
import zlib
from concurrent.futures import Future

import numpy as np
import pytest
import torch

from cosmos_curate_b200 import runtime, sampling
from cosmos_curate_b200._lib import CurateB200Error
from cosmos_curate_b200.data_model import Clip, SplitPipeTask, Video
from tools import synth_h264

DIM = 16
MAX_BATCH = 8
DECODED, EMPTY = {"frame_extraction": "video_decode_failed"}, {"encoded_data": "empty"}


class _Pool:
    """A surface pool that remembers what each slot holds."""

    def __init__(self, slots, size=None, held=None):
        self.buf = np.empty((slots, 0, 0), dtype=np.uint8)
        self.size = size
        self.held: dict[int, tuple] = held or {}


def _tag(data) -> int:
    return zlib.crc32(data if isinstance(data, bytes) else np.asarray(data, dtype=np.uint8).tobytes())


def _frame(key) -> tuple[np.ndarray, np.float32]:
    """The fake tower on one frame: (embedding, aesthetic score) from what the slot holds; zeros for a slot no decode filled."""
    if key is None:
        return np.zeros(DIM, np.float32), np.float32(0)
    rng = np.random.default_rng(zlib.crc32(repr(key).encode()))
    return rng.standard_normal(DIM).astype(np.float32), np.float32(rng.standard_normal())


class _Ctx:
    """The context calls of the target_res path: the resize keeps (out_w, out_h) and the source slot's content."""

    device = 0

    def resize_cubic_u8(self, pool, out_w, out_h, slots=None, mode=None):
        return [None if pool.held.get(int(s)) is None else (out_w, out_h, *pool.held[int(s)]) for s in slots]

    def rgb_pool(self, frames):
        return _Pool(len(frames), held={i: k for i, k in enumerate(frames) if k is not None})


class _Decoders:
    """DecoderPool.submit_group with no decoder: fills the fake pool's slots with (tag, frame id), fails the clips in `bad`."""

    numa_node, cpus = 1, [2, 3]

    def __init__(self, bad=()):
        self.bad, self.groups, self.seek = {_tag(b) for b in bad}, [], []

    def submit_group(self, pool, shape, jobs, seek_keyframes=False):
        assert shape == pool.size
        self.groups.append((shape, [_tag(data) for data, _ in jobs]))
        self.seek.append(seek_keyframes)
        out, first = [], 0
        for data, ids in jobs:
            assert np.all(np.diff(ids) >= 0) and first + len(ids) <= pool.buf.shape[0]
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
    out_dim = DIM

    def __init__(self, has_aesthetic=True):
        self.has_aesthetic, self.rows, self.norms = has_aesthetic, [], set()

    def embed_pool(self, pool, slots=None, mean=runtime.CLIP_MEAN, std=runtime.CLIP_STD):
        slots = range(pool.buf.shape[0]) if slots is None else [int(s) for s in slots]
        frames = [_frame(pool.held.get(s)) for s in slots]
        self.rows.append(len(frames))
        self.norms.add((tuple(mean), tuple(std)))
        emb = torch.from_numpy(np.stack([e for e, _ in frames]))
        score = torch.from_numpy(np.array([s for _, s in frames], dtype=np.float32)) if self.has_aesthetic else None
        return emb, None, score


class _Model:
    def __init__(self, tower, norm=None):
        self.tower = tower
        if norm is not None:
            self.mean = self.std = norm

    def setup(self):
        pass


@pytest.fixture(autouse=True)
def fakes(monkeypatch):
    from cosmos_curate_b200.stages import fused_clip

    monkeypatch.setattr(runtime, "alloc_nv12_pool", lambda ctx, slots, w, h, colour="opencv": _Pool(slots, (w, h)))
    monkeypatch.setattr(fused_clip, "get_context", _Ctx)

    class _Event:
        def record(self, stream):
            pass

        def synchronize(self):
            pass

    monkeypatch.setattr(torch.cuda, "current_stream", lambda: None)
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)


def _stage(monkeypatch, bad=(), model=None, max_batch=MAX_BATCH, **kw):
    from cosmos_curate_b200.stages import NvdecClipAestheticStage, fused_clip

    decoders = _Decoders(bad)
    monkeypatch.setattr(fused_clip, "DecoderPool", lambda ctx, n: decoders)
    stage = NvdecClipAestheticStage(max_batch=max_batch, num_decoders=5, model=model or _Model(_Tower()), **kw)
    stage.stage_setup()
    return stage, decoders


def _sampled(data, span=None) -> np.ndarray:
    """The frame ids the stage samples at 1 fps, repeats expanded: of the clip, or of a span of the source video."""
    idx = runtime.mp4_index(data)
    ts = sampling.timestamps_from_index(idx["pts"], idx["timescale"])
    if span is not None:
        return sampling.span_frame_ids(ts, span, 1.0)
    ids, counts = sampling.frame_ids(ts, sampling.FrameExtractionPolicy.sequence, 1.0)
    return np.repeat(ids, counts)


def _want(keys, reduce) -> tuple[float, np.ndarray]:
    """(reduced score, L2-normalised mean embedding) of a clip whose frames hold `keys`."""
    frames = [_frame(k) for k in keys]
    m = np.stack([e for e, _ in frames]).mean(axis=0)
    return float(reduce(np.array([s for _, s in frames], dtype=np.float32))), (m / np.linalg.norm(m)).astype(np.float32)


def _groups(planned, max_batch=MAX_BATCH) -> list:
    """[(size, [tag])]: per resolution in first-seen order, whole clips filling each batch up to max_batch frames."""
    by_size: dict = {}
    for size, tag, n in planned:
        by_size.setdefault(size, []).append((tag, n))
    out = []
    for size, clips in by_size.items():
        used = max_batch
        for tag, n in clips:
            if used + n > max_batch:
                out.append((size, []))
                used = 0
            out[-1][1].append(tag)
            used += n
    return out


def _check(tasks, want, threshold, emb=True, score=True):
    """want: {clip uuid: (errors, ((score, embedding) or None), encoded_data kept)}; the filter's split of every video."""
    for task in tasks:
        for video in task.videos:
            clips = video.clips + video.filtered_clips
            for c in clips:
                errors, result, kept = want[c.uuid]
                assert c.errors == errors and bool(c.encoded_data) == kept, c.uuid
                if result is None:
                    assert c.aesthetic_score == -1.0 and c.openai_embedding is None
                    continue
                assert c.aesthetic_score == (result[0] if score else None)
                if emb:
                    assert c.openai_embedding.dtype == np.float32 and np.array_equal(c.openai_embedding, result[1])
                else:
                    assert c.openai_embedding is None
            if threshold is None:
                assert not video.filtered_clips
                continue
            assert all(c.aesthetic_score >= threshold for c in video.clips)
            assert all(c.aesthetic_score < threshold for c in video.filtered_clips)
            assert video.clip_stats.num_filtered_by_aesthetic == len(video.filtered_clips)


def _clips(datas, spans=None):
    return [Clip(uuid=uuid.uuid5(uuid.NAMESPACE_URL, f"c{i}"), source_video="v.mp4", span=(spans or {}).get(i, (0.0, 2.0)), encoded_data=d)
            for i, d in enumerate(datas)]  # fmt: skip


A = [synth_h264.make_clip(320, 192, 30, 2.0, seed=s, gop=15) for s in range(4)]  # 3 sampled frames each
B = [synth_h264.make_clip(256, 144, 30, 1.0, seed=10 + s, gop=15) for s in range(3)]  # 2 sampled frames each
BROKEN = synth_h264.make_clip(320, 192, 30, 1.0, seed=22, gop=15)  # demuxes, fails to decode
GARBAGE = b"\x00not an mp4" * 9


def _mixed():
    """Two resolutions interleaved, a decode failure in a batch with good clips, more frames than one batch, a clip over max_batch
    (the 11 sampled frames of the golden clip), garbage bytes, no data, the same bytes twice."""
    from conftest import GOLDEN

    sintel = (GOLDEN / "sintel_clip_10s.mp4").read_bytes()
    return [A[0], B[0], BROKEN, A[1], None, B[1], sintel, GARBAGE, A[2], B[2], A[3], A[0]]


def _run_mixed(monkeypatch, reduction="min", threshold=None, **kw):
    datas = _mixed()
    clips = _clips(datas)
    tasks = [SplitPipeTask(session_id="s", video=Video(input_video=f"v{t}.mp4", clips=clips[t::2])) for t in range(2)]
    want, planned, decoded = {}, [], 0
    for i in [i for t in range(2) for i in range(t, len(clips), 2)]:  # the stage's order: task by task
        c, d = clips[i], datas[i]
        if d is None:
            want[c.uuid] = (EMPTY, None, False)
            continue
        if d is GARBAGE:
            want[c.uuid] = (DECODED, None, False)
            continue
        ids = _sampled(d)
        if len(ids) > MAX_BATCH or d is BROKEN:
            want[c.uuid] = (DECODED, None, False)
        else:
            decoded += int(ids[-1]) + 1
            want[c.uuid] = ({}, _want([(_tag(d), int(i)) for i in ids], np.mean if reduction == "mean" else np.min), True)
        if len(ids) <= MAX_BATCH:
            idx = runtime.mp4_index(d)
            planned.append((runtime.even_size(idx["width"], idx["height"]), _tag(d), len(ids)))
    if threshold == "median":
        threshold = float(np.median([r[0] for _, r, _ in want.values() if r is not None]))
    stage, decoders = _stage(monkeypatch, bad=[BROKEN], reduction=reduction, score_threshold=threshold, **kw)
    assert stage.process_data(tasks) is tasks
    return stage, decoders, tasks, want, threshold, _groups(planned), decoded


@pytest.mark.parametrize("reduction", ["min", "mean"])
def test_batches_errors_filter_and_write_back(monkeypatch, reduction):
    stage, decoders, tasks, want, threshold, groups, decoded = _run_mixed(monkeypatch, reduction, "median", write_embedding=True, log_stats=True)
    _check(tasks, want, threshold)
    assert sum(len(v.filtered_clips) for t in tasks for v in t.videos) >= 4  # the failures and some low scores
    assert sum(len(v.clips) for t in tasks for v in t.videos) >= 3
    assert decoders.groups == groups and len(groups) == 4  # 320x192: 3 + 2 + 3, 3 + 3, 3 frames; 256x144: 2 + 2 + 2
    assert decoders.seek == [False] * 4
    assert all(n <= MAX_BATCH for n in stage._model.tower.rows) and len(stage._model.tower.rows) == 4
    assert stage._model.tower.norms == {(runtime.CLIP_MEAN, runtime.CLIP_STD)}
    assert stage.last_call_stats == {"frames_decoded": decoded, "batches": 4, "nvdec_sessions": 5, "numa_node": 1, "pinned_cpus": 2}
    assert all(t.stage_perf.keys() == {"NvdecClipAestheticStage"} for t in tasks)


def test_score_only_without_embedding(monkeypatch):
    stage, _, tasks, want, threshold, _, _ = _run_mixed(monkeypatch, "min", -100.0, seek_keyframes=True)
    _check(tasks, want, threshold, emb=False)
    assert stage._decode_pool.seek == [True] * 4  # seek_keyframes reaches every decode group


def test_embedding_only_tower(monkeypatch):
    """score_threshold=None with a tower without an aesthetic head: nothing is filtered, the embedding is the output; the mean / std
    of the model reach the tower."""
    half = (0.5, 0.5, 0.5)
    model = _Model(_Tower(has_aesthetic=False), norm=half)
    stage, _, tasks, want, _, _, _ = _run_mixed(monkeypatch, "min", None, model=model, write_embedding=True)
    _check(tasks, want, None, score=False)
    assert model.tower.norms == {(half, half)}
    from cosmos_curate_b200.stages import NvdecClipAestheticStage

    with pytest.raises(ValueError, match="no aesthetic head"):
        NvdecClipAestheticStage(score_threshold=0.5, write_embedding=True, model=_Model(_Tower(has_aesthetic=False))).stage_setup()
    with pytest.raises(ValueError, match="needs write_embedding=True"):
        NvdecClipAestheticStage(score_threshold=None, model=_Model(_Tower())).stage_setup()


def test_target_res_resizes_the_decoded_frames(monkeypatch):
    """target_res = (h, w): the tower embeds the (w, h) resize of every decoded frame, failed clips in the same batch included."""
    datas = [A[0], BROKEN, B[0], A[1]]
    clips = _clips(datas)
    tasks = [SplitPipeTask(session_id="s", video=Video(input_video="v.mp4", clips=list(clips)))]
    stage, decoders = _stage(monkeypatch, bad=[BROKEN], score_threshold=-100.0, reduction="mean", write_embedding=True, target_res=(96, 128))
    stage.process_data(tasks)
    want = {c.uuid: (DECODED, None, False) if d is BROKEN else ({}, _want([(128, 96, _tag(d), int(i)) for i in _sampled(d)], np.mean), True)
            for c, d in zip(clips, datas)}  # fmt: skip
    _check(tasks, want, -100.0)
    assert len(decoders.groups) == 2


def test_video_span_source(monkeypatch):
    """source="video_span": every clip is a span of the source video, sampled like a clip of its own; the video is indexed once per
    call and never dropped; a span past the video's end and a video without bytes get the error table's entries."""
    from conftest import GOLDEN

    from cosmos_curate_b200.stages import fused_clip

    sintel = (GOLDEN / "sintel_clip_10s.mp4").read_bytes()
    spans = [(0.0, 10.0), (2.5, 7.5), (20.0, 21.0), (5.0, 10.0), (1.0, 3.0)]
    clips = _clips([None] * 5, spans=dict(enumerate(spans)))
    tasks = [SplitPipeTask(session_id="s", video=Video(input_video="v.mp4", encoded_data=sintel, clips=list(clips))),
             SplitPipeTask(session_id="s", video=Video(input_video="w.mp4", clips=[Clip(uuid=uuid.uuid4(), source_video="w.mp4", span=s)
                                                                                   for s in spans[:2]]))]  # fmt: skip
    indexed = []
    real_index = fused_clip.mp4_index
    monkeypatch.setattr(fused_clip, "mp4_index", lambda data: indexed.append(_tag(data)) or real_index(data))
    stage, decoders = _stage(monkeypatch, max_batch=16, score_threshold=-100.0, reduction="mean", write_embedding=True, source="video_span")
    stage.process_data(tasks)
    want = {c.uuid: (DECODED, None, False) if s[0] > 10 else ({}, _want([(_tag(sintel), int(i)) for i in _sampled(sintel, s)], np.mean), False)
            for c, s in zip(clips, spans)}  # fmt: skip
    want.update({c.uuid: (EMPTY, None, False) for c in tasks[1].video.clips})
    _check(tasks, want, -100.0)
    assert tasks[0].video.encoded_data and indexed == [_tag(sintel)]
    assert [len(tags) for _, tags in decoders.groups] == [1, 3]  # 11 frames, then 6 + 6 + 3
    assert stage.last_call_stats["batches"] == 2
