"""Task containers the path reads and mutates.

Inside a cosmos-curate environment the reference's own classes are re-exported.  Otherwise slim stand-ins with
the SAME field names are defined, restating only the fields this path touches:

    LazyData            cosmos_curate/core/utils/data/lazy_data.py:189-405   (inline payloads only; no Ray Plasma here)
    Clip / ClipStats    cosmos_curate/pipelines/video/utils/data_model.py:194-343, 345-390
    Video               :413-600
    SplitPipeTask       :690-800
    StagePerfStats      cosmos_curate/core/utils/infra/performance_utils.py:70-140
    StageTimer          :195-330   (reinit / time_process / log_stats call pattern; no OTel)
"""

from __future__ import annotations

import contextlib
import pathlib
import time
from typing import Any
from uuid import UUID

import attrs
import numpy as np

from .interfaces import PipelineTask

try:  # pragma: no cover - full cosmos-curate environment
    from cosmos_curate.core.utils.data.lazy_data import LazyData
    from cosmos_curate.core.utils.infra.performance_utils import StagePerfStats, StageTimer
    from cosmos_curate.pipelines.video.utils.data_model import Clip, ClipStats, SplitPipeTask, Video

    USING_REFERENCE_DATA_MODEL = True
except Exception:  # noqa: BLE001
    USING_REFERENCE_DATA_MODEL = False

    def bytes_to_numpy(data: bytes) -> np.ndarray:
        return np.frombuffer(data, dtype=np.uint8)

    @attrs.define(eq=False)
    class LazyData:
        value: Any = None
        ref: Any = attrs.field(default=None, repr=False)
        nbytes: int = 0

        @classmethod
        def coerce(cls, val):
            if isinstance(val, LazyData):
                return cls(ref=val.ref, value=val.value, nbytes=val.nbytes)
            if isinstance(val, bytes):
                arr = bytes_to_numpy(val)
                return cls(value=arr, nbytes=arr.nbytes)
            return cls(value=val, nbytes=getattr(val, "nbytes", 0) if val is not None else 0)

        def resolve(self):
            return self.value  # inline only (the reference's .store() calls are disabled, lazy_data.py:49-54)

        def store(self) -> None:
            return

        def release(self) -> None:
            self.value = None

        def drop(self) -> None:
            self.value, self.ref, self.nbytes = None, None, 0

        def __bool__(self) -> bool:
            return self.value is not None or self.ref is not None

    @attrs.define
    class ClipStats:
        num_filtered_by_motion: int = 0
        num_filtered_by_aesthetic: int = 0
        num_filtered_by_qwen_classifier: int = 0
        num_filtered_by_qwen_semantic: int = 0
        num_filtered_by_artificial_text: int = 0
        num_passed: int = 0
        num_transcoded: int = 0
        num_with_embeddings: int = 0
        num_with_caption: int = 0
        num_with_webp: int = 0
        total_clip_duration: float = 0.0
        max_clip_duration: float = 0.0
        total_prompt_tokens: int = 0
        total_output_tokens: int = 0

        def combine(self, other) -> None:  # data_model.py:369-390
            for f in attrs.fields(type(self)):
                a, b = getattr(self, f.name), getattr(other, f.name)
                setattr(self, f.name, max(a, b) if f.name == "max_clip_duration" else a + b)

    @attrs.define
    class Clip:
        uuid: UUID
        source_video: str
        span: tuple[float, float]
        encoded_data: LazyData = attrs.field(factory=LazyData, converter=LazyData.coerce)
        extracted_frames: LazyData = attrs.field(factory=LazyData)
        aesthetic_score: float | None = None
        cosmos_embed1_frames: LazyData = attrs.field(factory=LazyData, converter=LazyData.coerce)
        cosmos_embed1_embedding: np.ndarray | None = None
        intern_video_2_frames: LazyData = attrs.field(factory=LazyData, converter=LazyData.coerce)
        intern_video_2_embedding: np.ndarray | None = None
        intern_video_2_text_match: tuple[str, float] | None = None
        openai_embedding: np.ndarray | None = None
        errors: dict[str, str] = attrs.Factory(dict)

        @property
        def duration(self) -> float:  # data_model.py:310-318
            return self.span[1] - self.span[0]

    @attrs.define
    class VideoMetadata:  # data_model.py:392-410 (not decoder_utils.VideoMetadata: different field names)
        size: int | None = None
        height: int | None = None
        width: int | None = None
        framerate: float | None = None
        num_frames: int | None = None
        duration: float | None = None
        video_codec: str | None = None
        pixel_format: str | None = None
        audio_codec: str | None = None
        bit_rate_k: int | None = None
        format_name: str | None = None

    @attrs.define
    class Video:
        input_video: pathlib.Path | str
        relative_path: str = ""
        metadata: VideoMetadata = attrs.Factory(VideoMetadata)
        encoded_data: LazyData = attrs.field(factory=LazyData, converter=LazyData.coerce)
        frame_array: LazyData = attrs.field(factory=LazyData, converter=LazyData.coerce)
        timestamps: np.ndarray | None = attrs.field(default=None, eq=False)
        clips: list[Clip] = attrs.Factory(list)
        filtered_clips: list[Clip] = attrs.Factory(list)
        num_total_clips: int = 0
        num_clip_chunks: int = 0
        clip_chunk_index: int = 0
        clip_stats: ClipStats = attrs.Factory(ClipStats)
        errors: dict[str, str] = attrs.Factory(dict)

        def has_metadata(self) -> bool:  # data_model.py:536-552
            m = self.metadata
            return all([m.height, m.width, m.duration, m.framerate, m.num_frames, m.video_codec])

        @property
        def fraction(self) -> float:  # data_model.py:496-507
            if self.num_total_clips == 0:
                return 1.0
            return (len(self.clips) + len(self.filtered_clips)) / self.num_total_clips

        @property
        def weight(self) -> float:
            """data_model.py:509-523: duration normalised to 5 minutes x the fraction of its clips this chunk carries
            (what sharding.shard_by_weight balances across ranks)."""
            if self.metadata.size is None:
                return 0
            assert self.metadata.duration is not None
            return self.metadata.duration / 300 * self.fraction

        def nvdec_support(self) -> bool:
            """data_model.py:554-577: h264 with an 8-bit 4:2:0 / nv16 pixel format, hevc 4:2:0 / 4:4:4; everything else goes
            to the CPU decoder in the reference (here: is refused by cb_decoder_decode with CB_ERR_UNSUPPORTED)."""
            codec, pix = self.metadata.video_codec, self.metadata.pixel_format
            if codec is None or pix is None:
                return False
            if codec == "h264" and ("nv16" in pix or "420p" in pix):
                return True
            if codec == "hevc" and ("420p" in pix or "444p" in pix):
                return True
            return False

        def is_10_bit_color(self) -> bool | None:  # data_model.py:579-583
            pix = self.metadata.pixel_format
            if pix is None:
                return None
            return "10le" in pix or "10be" in pix

        def populate_timestamps(self) -> None:
            """data_model.py:449-460: per-frame presentation timestamps (seconds, float32, sorted) - from the moov index here,
            from a PyAV demux of every packet in the reference (decoder_utils.py:230-278)."""
            from .runtime import mp4_index
            from .sampling import timestamps_from_index

            data = self.encoded_data.resolve()
            if data is None:
                error_msg = "No video data available: encoded_data is None"
                raise ValueError(error_msg)
            idx = mp4_index(data)
            self.timestamps = timestamps_from_index(idx["pts"], idx["timescale"])

        def populate_metadata(self) -> None:
            """data_model.py:455-494, with the moov index instead of an ffprobe subprocess."""
            from .runtime import mp4_index
            from .sampling import video_metadata_from_index

            data = self.encoded_data.resolve()
            if data is None:
                error_msg = "No video data available: encoded_data is None"
                raise ValueError(error_msg)
            e = video_metadata_from_index(mp4_index(data))
            m = self.metadata
            m.size = data.nbytes
            m.height, m.width, m.framerate, m.num_frames, m.duration = e.height, e.width, e.fps, e.num_frames, e.video_duration
            m.video_codec, m.pixel_format, m.audio_codec, m.bit_rate_k, m.format_name = e.video_codec, e.pixel_format, e.audio_codec, e.bit_rate_k, e.format_name

    @attrs.define
    class StagePerfStats:
        process_time: float = 0.0
        actor_idle_time: float = 0.0
        input_data_size_mb: float = 0.0
        rss_before_mb: float = 0.0
        rss_after_mb: float = 0.0
        rss_delta_mb: float = 0.0
        wall_start: float = 0.0
        wall_end: float = 0.0

        def reset(self) -> None:  # performance_utils.py:126-135
            self.process_time = self.actor_idle_time = self.input_data_size_mb = 0.0
            self.rss_before_mb = self.rss_after_mb = self.rss_delta_mb = self.wall_start = self.wall_end = 0.0

    @attrs.define
    class SplitPipeTask(PipelineTask):
        session_id: str = ""
        videos: list[Video] = attrs.field(factory=list)
        stage_perf: dict[str, StagePerfStats] = attrs.Factory(dict)
        errors: dict[str, str] = attrs.Factory(dict)
        _init_video: Video | None = attrs.field(default=None, init=True, alias="video")

        def __attrs_post_init__(self) -> None:
            if self._init_video is not None:
                if self.videos:
                    msg = "Cannot specify both 'video' and 'videos' parameters"
                    raise ValueError(msg)
                self.videos = [self._init_video]
                self._init_video = None

        @property
        def video(self) -> Video:
            return self.videos[0]

        @property
        def weight(self) -> float:  # data_model.py:779-790: multi-camera tasks sum their videos
            return sum(v.weight for v in self.videos)

        @property
        def fraction(self) -> float:  # data_model.py:744-758
            total = sum(v.num_total_clips for v in self.videos)
            if total == 0:
                return 1.0
            return sum(len(v.clips) + len(v.filtered_clips) for v in self.videos) / total

        def get_major_size(self) -> int:
            total = 0
            for v in self.videos:
                total += v.encoded_data.nbytes + v.frame_array.nbytes
                for c in v.clips:
                    total += c.encoded_data.nbytes + c.extracted_frames.nbytes
            return total

    def _rss_mb() -> float:
        try:
            import psutil

            return psutil.Process().memory_info().rss / (1024 * 1024)
        except Exception:  # noqa: BLE001
            return 0.0

    class StageTimer:
        """performance_utils.py:195-330: per-process_data timing recorded into task.stage_perf."""

        def __init__(self, stage) -> None:
            self._stage_name = str(stage.__class__.__name__)
            self._last_active_time = time.time()
            self._initialized = False
            self._reset()

        def _reset(self) -> None:
            self._num_samples = 0
            self._durations_s: list[float] = []
            self._input_data_size_b = 0
            self._start = 0.0
            self._idle_time_s = 0.0
            self._rss_before_mb = 0.0

        def reinit(self, stage, stage_input_size: int = 1) -> None:
            self._reset()
            self._input_data_size_b = stage_input_size
            self._rss_before_mb = _rss_mb()
            self._start = time.time()
            if self._initialized:
                self._idle_time_s = self._start - self._last_active_time
            self._initialized = True

        @contextlib.contextmanager
        def time_process(self, num_samples: int = 1, source_video_duration_s: float = 0):
            t0 = time.time()
            yield
            dur = time.time() - t0
            self._num_samples += num_samples
            self._durations_s.extend([dur / max(1, num_samples)] * num_samples)

        def log_stats(self, *, verbose: bool = False):
            end = time.time()
            self._last_active_time = end
            rss_after = _rss_mb()
            return self._stage_name, StagePerfStats(
                process_time=end - self._start, actor_idle_time=self._idle_time_s, input_data_size_mb=self._input_data_size_b / 1024 / 1024,
                rss_before_mb=self._rss_before_mb, rss_after_mb=rss_after, rss_delta_mb=rss_after - self._rss_before_mb,
                wall_start=self._start, wall_end=end,
            )  # fmt: skip
