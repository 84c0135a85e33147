"""NvdecClipAestheticStage: clip mp4 bytes -> NVDEC -> sampled NV12 surfaces -> fused preprocess -> tower -> scores.

Replaces the pair ClipFrameExtractionStage (CPU PyAV decode of every frame + RGB frames pickled to the next actor,
clip_frame_extraction_stages.py:102-165) -> AestheticFilterStage (aesthetic_filter_stages.py:120-221) with one GPU
stage that never materialises RGB frames.  Task mutations and the error convention are the reference's:

    clip.aesthetic_score, video.filtered_clips, video.clip_stats.num_filtered_by_aesthetic, task.stage_perf,
    no encoded_data            -> clip.errors["encoded_data"] = "empty", score -1.0
    demux / decode failure     -> clip.errors["frame_extraction"] = "video_decode_failed", encoded_data dropped, score -1.0
    task.stage_perf follows the reference's StageTimer call pattern (reinit BEFORE the work, aesthetic_filter_stages.py:161).
    (optional) clip.openai_embedding = L2-normalised mean of the per-frame embeddings (SURVEY.md 8b: the reference has
    no pooling rule for frame embeddings; this documented choice fills the existing generic clip-embedding slot).

Inside one `process_data` call the work is pipelined by runtime.run_decode_groups, the decode-group loop the InternVideo2 stages
run too (this IS the product path bench.py times as `e2e`): the clips of tower batches k+1 and k+2 are being decoded by the
persistent NVDEC sessions (DecoderPool: one session per worker thread, kept across calls, pinned to the GPU's NUMA node) while
the SMs run preprocess + tower on batch k out of a three-deep ring of surface pools; scores / embeddings come back through
pinned host buffers with one async copy per batch.  A batch holds whole clips of one resolution, at most max_batch frames; a
clip that samples more frames than that fails like a clip that does not decode.
"""

from __future__ import annotations

from typing import Literal

import numpy as np
import torch

from .. import sampling
from ..data_model import StageTimer
from ..interfaces import CuratorStage, CuratorStageResource, ModelInterface
from ..models.clip_aesthetics import CLIPAestheticScorer
from ..runtime import DecoderPool, SurfacePools, check_colour, even_size, get_context, mp4_index, run_decode_groups

try:
    from loguru import logger
except Exception:  # noqa: BLE001
    import logging

    logger = logging.getLogger(__name__)


class NvdecClipAestheticStage(CuratorStage):
    def __init__(  # noqa: PLR0913
        self,
        score_threshold: float | None,
        reduction: Literal["mean", "min"] = "min",
        target_fps: float = 1.0,
        num_gpus_per_worker: float = 1.0,
        *,
        write_embedding: bool = False,
        max_batch: int = 256,
        num_decoders: int = 20,
        stage_batch_size: int = 8,
        seek_keyframes: bool = False,
        source: Literal["clip", "video_span"] = "clip",
        target_res: tuple[int, int] | None = None,
        cubic_mode: str | None = None,
        colour: str = "swscale",
        verbose: bool = False,
        log_stats: bool = False,
        model: CLIPAestheticScorer | None = None,
    ) -> None:
        self._timer = StageTimer(self)
        self._score_threshold, self._reduction, self._target_fps = score_threshold, reduction, target_fps
        self._num_gpus_per_worker = num_gpus_per_worker
        self._write_embedding, self._max_batch, self._num_decoders = write_embedding, max_batch, num_decoders
        self._stage_batch_size, self._verbose, self._log_stats = stage_batch_size, verbose, log_stats
        # False (default): every frame up to the last sampled one is decoded, the reference's decode work (decoder_utils.py:439-455) and
        # what bench.py's headline `e2e` times.  True: only the GOPs that hold sampled frames are decoded - bit-identical frames
        # (tested), 5x the clips/s on 1 fps sampling of GOP-30 clips; recommended in INTEGRATION.md, reported as `e2e_keyframe_seek`.
        self._seek = seek_keyframes
        if source not in ("clip", "video_span"):
            error_msg = f"source={source!r} not in ('clip', 'video_span')"
            raise ValueError(error_msg)
        # "video_span": analysis without the transcode (SURVEY.md 8f N2) - the clip's frames are decoded straight out of the SOURCE
        # video (video.encoded_data) at clip.span, so ClipTranscodingStage's re-encode + this stage's re-decode disappear for runs
        # that only need scores / embeddings.  Pixels are the source's, not the 4 Mb/s re-encode's: not bit-comparable with "clip".
        self._source = source
        # colour conversion of the decoded NV12 surfaces inside the fused kernel: "swscale" = bit-identical to the RGB frames the
        # reference's CPU decode hands to CLIP (libswscale yuv420p -> rgb24, decoder_utils.py:439-451), "opencv" = CV-CUDA semantics
        self._colour = check_colour(colour)
        # clip_extraction_target_res of the reference pipeline (splitting_pipeline -> ClipFrameExtractionStage(target_res=(r, r))):
        # frames are squashed to (h, w) with cv2 INTER_CUBIC before the CLIP transforms (decoder_utils.py:666-670).  None / (-1, -1)
        # = native resolution into the antialiased short-side resize (the reference default).
        from .frame_extraction import CUBIC_MODES, default_cubic_mode

        self._target_res = None if target_res is None or target_res[0] <= 0 or target_res[1] <= 0 else (int(target_res[0]), int(target_res[1]))
        self._cubic_mode = CUBIC_MODES[cubic_mode or default_cubic_mode()]
        self._video_index: dict[int, tuple] = {}
        # Any ModelInterface with a `.tower` works: CLIPAestheticScorer (score + embedding) or an embedding-only tower such as
        # SigLIPImageEmbeddings (score_threshold=None: nothing is filtered, clip.openai_embedding is the output).
        self._model = model if model is not None else CLIPAestheticScorer(max_batch=max_batch)
        self._reduce_fn = np.min
        self._pools: SurfacePools | None = None
        self.last_call_stats: dict = {}

    @property
    def resources(self) -> CuratorStageResource:
        return CuratorStageResource(gpus=self._num_gpus_per_worker)

    @property
    def model(self) -> ModelInterface:
        return self._model

    @property
    def stage_batch_size(self) -> int:
        return self._stage_batch_size

    def stage_setup(self) -> None:
        if self._reduction not in ("mean", "min"):
            error_msg = f"Reduction `{self._reduction}` not implemented."
            raise NotImplementedError(error_msg)
        self._reduce_fn = np.mean if self._reduction == "mean" else np.min
        self._model.setup()
        self._ctx = get_context()
        self._norm = (getattr(self._model, "mean", None), getattr(self._model, "std", None))
        if self._score_threshold is not None and not self._model.tower.has_aesthetic:
            error_msg = "score_threshold given but the model has no aesthetic head (pass score_threshold=None for embedding-only towers)"
            raise ValueError(error_msg)
        if self._score_threshold is None and not self._write_embedding:
            error_msg = "embedding-only mode (score_threshold=None) needs write_embedding=True"
            raise ValueError(error_msg)
        self._decode_pool = DecoderPool(self._ctx, self._num_decoders)  # 7 NVDEC engines need ~20 sessions in flight (DESIGN.md 5)
        self._pools = SurfacePools(self._ctx, self.RING, self._max_batch, self._colour)
        self._host: list[tuple[torch.Tensor, torch.Tensor | None]] = []

    def destroy(self) -> None:
        if getattr(self, "_decode_pool", None):
            self._decode_pool.close()
            self._decode_pool = None
        if self._pools is not None:
            self._pools.clear()

    # ---- helpers ---------------------------------------------------------------------------------
    def _plan(self, clip, data):
        """-> (surface size, sampled frame ids with repeats, slot of each relative to the clip's first), or raises for an unreadable
        container or a span that selects no frame.  source="video_span": the source video's frames inside clip.span, re-timed from
        the clip start and sampled like a clip of its own."""
        cached = self._video_index.get(id(data))  # the clips of a span-sourced video share its bytes: indexed once per call
        if cached is None:  # an entry holds its bytes, so their id names no other object while it exists
            idx = mp4_index(data)
            cached = self._video_index[id(data)] = (data, even_size(idx["width"], idx["height"]),
                                                    sampling.timestamps_from_index(idx["pts"], idx["timescale"]))  # fmt: skip
        _, size, ts = cached
        if self._source == "video_span":
            ids = sampling.span_frame_ids(ts, clip.span, self._target_fps)
        else:
            ids, counts = sampling.frame_ids(ts, sampling.FrameExtractionPolicy.sequence, self._target_fps)
            ids = np.repeat(ids, counts).astype(np.int32)
        return size, ids, np.arange(len(ids), dtype=np.int32)

    def _decode_failed(self, clip, e) -> None:
        logger.error(f"Error extracting frames from clip {clip.uuid}: {e}")
        clip.errors["frame_extraction"] = "video_decode_failed"
        if self._source == "clip":
            clip.encoded_data.drop()
        clip.aesthetic_score = -1.0

    RING = 3  # surface pools per resolution: tower on batch k, NVDEC filling k+1 and k+2

    def _host_buffers(self, r: int):
        while len(self._host) <= r:
            tower = self._model.tower
            score = torch.empty((self._max_batch,), dtype=torch.float32).pin_memory() if tower.has_aesthetic else None
            emb = torch.empty((self._max_batch, tower.out_dim), dtype=torch.float32).pin_memory() if self._write_embedding else None
            self._host.append((score, emb))
        return self._host[r]

    def _compute(self, k, pool, ok, slots):
        """Preprocess + tower on batch k's decoded frames and the D2H copy of the results into ring slot k % RING, queued; -> the
        finisher that writes each clip's reduced score and L2-normalised mean embedding."""
        tower = self._model.tower
        norm = {} if self._norm[0] is None else {"mean": self._norm[0], "std": self._norm[1]}
        if self._target_res is not None:
            th, tw = self._target_res
            small = self._ctx.resize_cubic_u8(pool, tw, th, slots=slots, mode=self._cubic_mode)
            emb, _, score = tower.embed_pool(self._ctx.rgb_pool(small), **norm)
        else:
            emb, _, score = tower.embed_pool(pool, slots=slots, **norm)
        n = len(slots)
        score_h, emb_h = self._host_buffers(k % self.RING)
        if score_h is not None:
            score_h[:n].copy_(score, non_blocking=True)
        if emb_h is not None:
            emb_h[:n].copy_(emb, non_blocking=True)

        def write():
            row = 0
            for clip, m in ok:
                if score_h is not None:
                    clip.aesthetic_score = float(self._reduce_fn(score_h[row : row + m].numpy()))
                if emb_h is not None:
                    e = emb_h[row : row + m].numpy().mean(axis=0)
                    clip.openai_embedding = (e / np.linalg.norm(e)).astype(np.float32)
                row += m

        return write

    # ---- stage entry -----------------------------------------------------------------------------
    def process_data(self, tasks):
        self._timer.reinit(self, sum(task.get_major_size() for task in tasks))
        n_clips = sum(len(video.clips) for task in tasks for video in task.videos)
        with self._timer.time_process(num_samples=max(1, n_clips)):
            items = []
            for task in tasks:
                for video in task.videos:
                    for clip in video.clips:
                        source = video if self._source == "video_span" else clip
                        data = source.encoded_data.resolve() if source.encoded_data else None
                        if data is None:
                            logger.warning(f"Clip {clip.uuid} has no encoded_data (source={self._source}).")
                            clip.errors["encoded_data"] = "empty"
                            clip.aesthetic_score = -1.0
                            continue
                        items.append((clip, data))
            # decode of batches k+1, k+2 (NVDEC + host parsing threads) overlaps preprocess + tower of batch k (SMs)
            decoded, batches = run_decode_groups(items, self._plan, self._pools, lambda: self._decode_pool, self._compute,
                                                 on_error=self._decode_failed, max_frames=self._max_batch, depth=self.RING,
                                                 seek_keyframes=self._seek)  # fmt: skip
            self.last_call_stats = {"frames_decoded": decoded, "batches": batches, "nvdec_sessions": self._num_decoders,
                                    "numa_node": self._decode_pool.numa_node, "pinned_cpus": len(self._decode_pool.cpus)}  # fmt: skip

            for task in tasks:
                for video in task.videos:
                    passed = []
                    if self._score_threshold is None:  # embedding-only tower: nothing to filter on
                        continue
                    for clip in video.clips:
                        if clip.aesthetic_score is None:
                            clip.aesthetic_score = -1.0
                        if clip.aesthetic_score < self._score_threshold:
                            video.filtered_clips.append(clip)
                            video.clip_stats.num_filtered_by_aesthetic += 1
                        else:
                            passed.append(clip)
                    video.clips = passed
        if self._log_stats:
            stage_name, stats = self._timer.log_stats()  # one batched call -> the same window on every task of the call
            for task in tasks:
                task.stage_perf[stage_name] = stats
        self._video_index.clear()
        return tasks
