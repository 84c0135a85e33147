"""NvdecInternVideo2EmbeddingStage: clip mp4 bytes -> NVDEC -> the tube's kept frames as NV12 surfaces -> InternVideo2 tower ->
`clip.intern_video_2_embedding`, in one GPU stage.

Replaces the pair InternVideo2FrameCreationStage(source="nvdec") -> InternVideo2EmbeddingStage, which hands a float32 tube
[1, T, 3, 224, 224] (2.4 MB at T = 4) to the host and back to the GPU between two actors.  Here the decoded frames go straight into
the tower's patch rows (cb_iv2_embed_surfaces: one resize + normalise + patch-row launch per tower chunk, bitwise the tube the pair
computes), and only the [n, 512] embeddings come back, through pinned host buffers.  The tube's frame count is the tower's own
(model.get_target_num_frames(), read from pos_embed), so the formulator / tower frame-count pairing cannot go wrong.

The frame plan (sampled ids from the MP4 index, the reference's re-extraction rule, the kept frames) is the frame-creation stage's own
(plan_clip), and the decode-group loop is runtime.run_decode_groups, which that stage and NvdecClipAestheticStage run too: the kept
frames, the errors and the embeddings are the pair's.  Per clip:

    no encoded_data                    -> errors {"encoded_data": "empty", "iv2_frames": "none"}, no embedding
    unreadable container / decode fail -> errors {"frame_extraction": "video_decode_failed", "iv2_frames": "none"}, no embedding
    too short even at the highest rate -> errors {"iv2_frames": "empty"}, no embedding
    otherwise                          -> clip.intern_video_2_embedding float32 [1, embed_dim] (+ intern_video_2_text_match with texts)

`clip.intern_video_2_frames` is never set.  Clips of all tasks of a call share decode groups and tower chunks; decode of the next
groups overlaps the tower on the current one (a ring of RING surface pools per resolution, one pinned host buffer per ring slot, each
reused only after the loop has waited on the event of the group that last used it).
"""

from __future__ import annotations

import numpy as np
import torch

from ..data_model import StageTimer
from ..interfaces import CuratorStage, CuratorStageResource, ModelInterface
from ..models.internvideo2 import InternVideo2MultiModality
from ..runtime import IMAGENET_MEAN, IMAGENET_STD, DecoderPool, SurfacePools, check_colour, get_context, nvdec_available, run_decode_groups
from .internvideo2_embedding import TextMatch
from .internvideo2_frames import InternVideo2FrameCreationStage, plan_clip

try:
    from loguru import logger
except Exception:  # noqa: BLE001
    import logging

    logger = logging.getLogger(__name__)


class NvdecInternVideo2EmbeddingStage(CuratorStage):
    """InternVideo2 clip embeddings (and text matches) from clip mp4 bytes, decoded and embedded on the GPU."""

    GROUP = InternVideo2FrameCreationStage.GROUP  # clips per decode group
    RING = 3  # surface pools per resolution: the tower on group k, NVDEC filling k+1 and k+2

    def __init__(self, target_fps: float = 2.0, num_gpus_per_worker: float = 1.0, batch_size: int = 8, texts_to_verify: list[str] | None = None,
                 *, num_decoders: int = 8, stage_batch_size: int = 8, seek_keyframes: bool = False, colour: str = "swscale",
                 verbose: bool = False, log_stats: bool = False, model: InternVideo2MultiModality | None = None) -> None:  # fmt: skip
        self._model = model if model is not None else InternVideo2MultiModality(max_clips=batch_size)
        self._text_match = TextMatch(self._model, texts_to_verify)
        self._timer = StageTimer(self)
        self._target_fps, self._num_gpus_per_worker, self._batch_size = target_fps, num_gpus_per_worker, max(1, int(batch_size))
        self._num_decoders, self._stage_batch_size = num_decoders, stage_batch_size
        # True: only the GOPs that hold kept frames are decoded (bit-identical frames); False: every frame up to the last kept one
        self._seek = seek_keyframes
        self._colour = check_colour(colour)
        self._verbose, self._log_stats = verbose, log_stats
        self._decode_pool: DecoderPool | None = None
        self._pools: SurfacePools | None = None
        self._host: list[torch.Tensor] = []
        self.last_call_stats: dict = {}

    @property
    def model(self) -> ModelInterface:
        return self._model

    @property
    def resources(self) -> CuratorStageResource:
        return CuratorStageResource(gpus=self._num_gpus_per_worker)

    @property
    def stage_batch_size(self) -> int:
        return self._stage_batch_size

    def stage_setup(self) -> None:
        self._model.setup()
        self._text_match.embed()
        self._ctx = get_context()
        self._frames = self._model.get_target_num_frames()
        self._decode_pool = DecoderPool(self._ctx, self._num_decoders)
        self._pools = SurfacePools(self._ctx, self.RING, self._frames, self._colour)

    def destroy(self) -> None:
        if self._decode_pool is not None:
            self._decode_pool.close()
            self._decode_pool = None
        if self._pools is not None:
            self._pools.clear()

    def _host_buffer(self, r: int, n: int, dim: int) -> torch.Tensor:
        """Pinned float32 [>= n, dim] of ring slot r (grown when a group has more clips)."""
        while len(self._host) <= r:
            self._host.append(torch.empty((0, dim), dtype=torch.float32))
        if self._host[r].shape[0] < n:
            self._host[r] = torch.empty((max(n, self.GROUP), dim), dtype=torch.float32).pin_memory()
        return self._host[r]

    @staticmethod
    def _decode_failed(clip, e) -> None:
        InternVideo2FrameCreationStage._decode_failed(clip, e)
        clip.errors["iv2_frames"] = "none"

    @staticmethod
    def _too_short(clip) -> None:
        clip.errors["iv2_frames"] = "empty"

    def _embed(self, items) -> None:
        """items: [(clip, mp4 bytes)] -> embeddings on the clips.  Group k's tower work and D2H copy into the pinned buffer of its ring
        slot are queued; the buffer is read once group k's event has fired."""
        tower, fn, bs = self._model.tower, self._frames, self._batch_size

        def compute(k, pool, ok, slots):
            host = self._host_buffer(k % self.RING, len(ok), tower.embed_dim)
            for i in range(0, len(ok), bs):
                m = min(bs, len(ok) - i)
                emb = tower.embed_pool(pool, slots[i * fn : (i + m) * fn], mean=IMAGENET_MEAN, std=IMAGENET_STD)
                host[i : i + m].copy_(emb, non_blocking=True)

            def write():
                for i, (clip, _) in enumerate(ok):
                    clip.intern_video_2_embedding = host[i : i + 1].numpy().copy()

            return write

        decoded, groups = run_decode_groups(items, lambda clip, data: plan_clip(clip, data, self._target_fps, fn, self._verbose), self._pools,
                                            lambda: self._decode_pool, compute, on_short=self._too_short, on_error=self._decode_failed,
                                            max_frames=self.GROUP * fn, depth=self.RING, seek_keyframes=self._seek)  # fmt: skip
        self.last_call_stats = {"frames_decoded": decoded, "groups": groups, "nvdec_sessions": self._num_decoders,
                                "host_decode": not nvdec_available(self._ctx)}  # fmt: skip

    def process_data(self, tasks):
        self._timer.reinit(self, sum(task.get_major_size() for task in tasks))
        clips = [clip for task in tasks for clip in task.video.clips]
        with self._timer.time_process(num_samples=max(1, len(clips))):
            items = []
            for clip in clips:
                data = clip.encoded_data.resolve() if clip.encoded_data else None
                if data is None:
                    clip.errors["encoded_data"] = "empty"
                    clip.errors["iv2_frames"] = "none"
                    continue
                items.append((clip, data))
            self._embed(items)
            for clip in clips:
                self._text_match.verify(clip)
        if self._log_stats:
            stage_name, stats = self._timer.log_stats()  # one batched call -> the same window on every task of the call
            for task in tasks:
                task.stage_perf[stage_name] = stats
        return tasks
