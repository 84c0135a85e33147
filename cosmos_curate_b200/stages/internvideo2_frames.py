"""InternVideo2FrameCreationStage on the B200 path - same name, constructor and task mutations as the reference stage
(cosmos_curate/pipelines/video/embedding/internvideo2_stages.py:43-184): `clip.intern_video_2_frames` <- float32
[1, 8, 3, 224, 224], the tube the video tower's encode_video_frames consumes (:277-296).

source="frames" (default, drop-in): reads the host RGB frames a ClipFrameExtractionStage left in `clip.extracted_frames`
    under this stage's signature; only the 8 frames the stride keeps cross PCIe.  A clip with fewer sampled frames than the
    model needs is re-extracted at 2x the rate (up to 20 fps) from `encoded_data` (:157-176) - on NVDEC here.
source="nvdec": no upstream frame extraction; the sampled frame ids come from the MP4 index, the re-extraction rule is
    applied to the id lists (no decode needed to know how many frames a rate yields), the 8 kept frames are decoded
    straight into NV12 surfaces and resized / normalised from there.  Host frames never exist; 4.8 MB per clip come back.
"""

from __future__ import annotations

import numpy as np

from .. import sampling
from ..data_model import StageTimer
from ..interfaces import CuratorStage, CuratorStageResource, ModelInterface
from ..models.internvideo2_frames import InternVideo2FrameFormulator, select_frame_ids
from ..runtime import DecoderPool, SurfacePools, check_colour, even_size, get_context, mp4_index, run_decode_groups
from ..sampling import FrameExtractionPolicy, FrameExtractionSignature

try:
    from loguru import logger
except Exception:  # noqa: BLE001
    import logging

    logger = logging.getLogger(__name__)

MAX_FPS = 20  # internvideo2_stages.py:138


def sampled_ids_with_regen(ts: np.ndarray, target_fps: float, target_num_frames: int, max_fps: int = MAX_FPS):
    """Frame ids of the `sequence` policy at target_fps, the rate doubled while it yields fewer than target_num_frames
    frames and stays <= max_fps (internvideo2_stages.py:157-176).  Returns (ids, rate actually used)."""
    def expanded(rate):
        ids, counts = sampling.frame_ids(ts, FrameExtractionPolicy.sequence, rate)
        return np.repeat(ids, counts)

    fps = used = target_fps
    ids = expanded(fps)
    while len(ids) < target_num_frames:
        fps *= 2
        if fps > max_fps:
            break
        ids, used = expanded(fps), fps
    return ids, used


def plan_clip(clip, data, target_fps: float, fn: int, verbose: bool = False):
    """The decode plan of one clip's tube: -> (surface size, distinct frame ids to decode, slot of every kept frame relative to the
    clip's first slot), None when the clip is too short (tube = the reference's empty array), or raises for an unreadable container.
    The sampled ids come from the MP4 index, with the re-extraction rule applied to the id lists (sampled_ids_with_regen)."""
    idx = mp4_index(data)
    ts = sampling.timestamps_from_index(idx["pts"], idx["timescale"])
    ids, fps = sampled_ids_with_regen(ts, target_fps, fn)
    if len(ids) < fn:
        logger.error(f"Clip {clip.uuid} is too short to extract enough frames.")
        logger.error(f"Frame count {len(ids)} is smaller than minimal requirement {fn}")
        return None
    if verbose and fps != target_fps:
        logger.warning(f"Clip {clip.uuid} has <{fn} frames at target_fps={target_fps}; sampled at {fps}.")
    keep = np.asarray(ids)[select_frame_ids(len(ids), fn)]
    uniq, inverse = np.unique(keep, return_inverse=True)  # a frame kept twice (supersampled clip) is decoded once
    return even_size(idx["width"], idx["height"]), uniq.astype(np.int32), inverse.astype(np.int32)


class InternVideo2FrameCreationStage(CuratorStage):
    """Stage for creating InternVideo2 input frames from video clips."""

    # clips per decode group of the nvdec source (32 x 8 surfaces: 0.8 GB of 1080p NV12 per pool, two pools).  A group's device tubes
    # (32 x 8 x 3 x 224 x 224 fp32, 154 MB) are copied to the host only after the next group is queued: two groups' tubes at peak.
    GROUP = 32

    def __init__(self, target_fps: float = 2.0, *, verbose: bool = False, log_stats: bool = False, source: str = "frames",
                 num_gpus_per_worker: float = 0.1, num_decoders: int = 8, stage_batch_size: int = 1, colour: str = "swscale",
                 model: InternVideo2FrameFormulator | None = None) -> None:  # fmt: skip
        if source not in ("frames", "nvdec"):
            msg = f"source={source!r} not in ('frames', 'nvdec')"
            raise ValueError(msg)
        self._timer = StageTimer(self)
        self._target_fps = target_fps
        self._extraction_policy = FrameExtractionPolicy.sequence
        self._frame_extraction_signature = FrameExtractionSignature(extraction_policy=FrameExtractionPolicy.sequence, target_fps=target_fps).to_str()
        self._model = model if model is not None else InternVideo2FrameFormulator()
        self._verbose, self._log_stats = verbose, log_stats
        self._source, self._colour, self._num_gpus = source, check_colour(colour), num_gpus_per_worker
        self._num_decoders, self._stage_batch_size = num_decoders, stage_batch_size
        self._decode_pool = None
        self._pools: SurfacePools | None = None

    @property
    def model(self) -> ModelInterface:
        return self._model

    @property
    def resources(self) -> CuratorStageResource:
        return CuratorStageResource(cpus=1.0, gpus=self._num_gpus)  # the reference stage is CPU-only (cpus=1.0, :93)

    @property
    def stage_batch_size(self) -> int:
        return self._stage_batch_size

    def stage_setup(self) -> None:
        self._model.setup()
        self._ctx = get_context()
        self._pools = SurfacePools(self._ctx, 2, self._model.get_target_num_frames(), self._colour)

    def destroy(self) -> None:
        if self._decode_pool is not None:
            self._decode_pool.close()
            self._decode_pool = None
        if self._pools is not None:
            self._pools.clear()

    # ---- NVDEC side --------------------------------------------------------------------------------
    def _decoders(self) -> DecoderPool:
        if self._decode_pool is None:
            self._decode_pool = DecoderPool(self._ctx, self._num_decoders)
        return self._decode_pool

    def _tubes_from_streams(self, items) -> None:
        """items: [(clip, data)].  Decode groups of GROUP clips on the session pool (group k+1 decodes while group k is
        resized, normalised and copied out), one tube kernel launch per group."""
        fn = self._model.get_target_num_frames()

        def too_short(clip):
            clip.intern_video_2_frames = np.empty(0, dtype=np.float32)

        def compute(k, pool, ok, slots):
            tubes = self._model.formulate_pool(pool, slots)  # [len(ok) * fn, 3, s, s]

            def write():
                host = tubes.cpu().numpy()
                for i, (clip, _) in enumerate(ok):
                    clip.intern_video_2_frames = host[i * fn : (i + 1) * fn][None].copy()

            return write

        run_decode_groups(items, lambda clip, data: plan_clip(clip, data, self._target_fps, fn, self._verbose), self._pools, self._decoders,
                          compute, on_short=too_short, on_error=self._decode_failed, max_frames=self.GROUP * fn)  # fmt: skip

    @staticmethod
    def _decode_failed(clip, e) -> None:
        logger.error(f"Error extracting frames from clip {clip.uuid}: {e}")
        clip.errors["frame_extraction"] = "video_decode_failed"

    # ---- the reference's process_data ----------------------------------------------------------
    def process_data(self, tasks):
        if self._source == "nvdec":
            return self._process_streams(tasks)
        for task in tasks:
            self._timer.reinit(self, task.get_major_size())
            video = task.video
            for clip in video.clips:
                data = clip.encoded_data.resolve() if clip.encoded_data else None
                if data is None:
                    clip.errors["encoded_data"] = "empty"
                    continue
                ef = clip.extracted_frames.resolve()
                if ef is None or self._frame_extraction_signature not in ef:
                    clip.errors[f"frames-{self._frame_extraction_signature}"] = "missing"
                    logger.error(f"Clip {clip.uuid} has buffer but no extracted frames for {self._frame_extraction_signature}")
                    continue
                with self._timer.time_process():
                    frames = ef[self._frame_extraction_signature]
                    if frames.shape[0] < self._model.get_target_num_frames():
                        # re-extract at a higher rate from the stream (internvideo2_stages.py:157-176): the id-list rule lands on
                        # the rate the reference's decode-and-count loop stops at; a clip still too short gets the empty
                        # float32 array `_construct_frames` returns (internvideo2_mm.py:396-398)
                        self._tubes_from_streams([(clip, data)])
                    else:
                        clip.intern_video_2_frames = self._model.formulate_input_frames(list(frames))
                clip.extracted_frames.drop()

            if self._log_stats:
                stage_name, stage_perf_stats = self._timer.log_stats()
                task.stage_perf[stage_name] = stage_perf_stats
        return tasks

    def _process_streams(self, tasks):
        """source="nvdec": clips of all tasks of the call share the decode groups, so the timer window is per call."""
        self._timer.reinit(self, sum(task.get_major_size() for task in tasks))
        items = []
        for task in tasks:
            for clip in task.video.clips:
                data = clip.encoded_data.resolve() if clip.encoded_data else None
                if data is None:
                    clip.errors["encoded_data"] = "empty"
                    continue
                items.append((clip, data))
        with self._timer.time_process(num_samples=max(1, len(items))):
            self._tubes_from_streams(items)
        if self._log_stats:
            stage_name, stats = self._timer.log_stats()
            for task in tasks:
                task.stage_perf[stage_name] = stats
        return tasks
