"""InternVideo2EmbeddingStage on the H100 path - same name, constructor and task mutations as the reference stage
(cosmos_curate/pipelines/video/embedding/internvideo2_stages.py:187-309): `clip.intern_video_2_embedding` <- float32 [1, 512] from
the tube InternVideo2FrameCreationStage left in `clip.intern_video_2_frames`, which is dropped for every clip.

Clips of all tasks of one call share the tower's batches (an embedding does not depend on its batch neighbours).  With
`texts_to_verify`, every clip whose embedding is set also gets `clip.intern_video_2_text_match = (text, probability)`: the most probable
text under softmax(100 * clip . text) (_verify_with_texts, :251-256).  The texts are embedded once per stage, not once per clip as the
reference does (a text's embedding does not depend on the clip).  An empty list, or a model that cannot embed text, is refused at
construction.  Build the pair as
InternVideo2FrameCreationStage(model=InternVideo2FrameFormulator(num_frames=4)) -> InternVideo2EmbeddingStage: a tube of another
frame count raises ValueError naming both counts (the reference fails on the pos_embed add).
"""

from __future__ import annotations

from ..data_model import StageTimer
from ..interfaces import CuratorStage, CuratorStageResource, ModelInterface
from ..models.internvideo2 import InternVideo2MultiModality


class TextMatch:
    """`texts_to_verify` of the InternVideo2 embedding stages: the constructor refuses an empty list and a model that cannot embed text,
    embed() embeds the texts once (stage_setup), verify(clip) sets clip.intern_video_2_text_match on a clip that has an embedding."""

    def __init__(self, model, texts_to_verify: list[str] | None) -> None:
        if texts_to_verify is not None:
            if not texts_to_verify:
                msg = "texts_to_verify is empty: give at least one text, or None"
                raise ValueError(msg)
            if not (callable(getattr(model, "encode_texts", None)) and callable(getattr(model, "evaluate", None))):
                msg = f"texts_to_verify needs a model that embeds text (encode_texts / evaluate); {type(model).__name__} does not"
                raise ValueError(msg)
        self._model = model
        self._texts = list(texts_to_verify) if texts_to_verify is not None else None
        self._text_embeddings = None

    def embed(self):
        if self._texts is not None and self._text_embeddings is None:
            self._text_embeddings = list(self._model.encode_texts(self._texts))
        return self._text_embeddings

    def verify(self, clip) -> None:
        if self._texts is not None and clip.intern_video_2_embedding is not None:
            probs, idxs = self._model.evaluate(clip.intern_video_2_embedding, self.embed())
            clip.intern_video_2_text_match = (self._texts[idxs[0]], probs[0])


class InternVideo2EmbeddingStage(CuratorStage):
    """Stage for generating embeddings from InternVideo2 input frames."""

    def __init__(self, num_gpus_per_worker: float = 0.25, batch_size: int = 8, *, verbose: bool = False, log_stats: bool = False,
                 texts_to_verify: list[str] | None = None, model: InternVideo2MultiModality | None = None) -> None:  # fmt: skip
        self._model = model if model is not None else InternVideo2MultiModality()
        self._text_match = TextMatch(self._model, texts_to_verify)
        self._timer = StageTimer(self)
        self._num_gpus_per_worker, self._batch_size = num_gpus_per_worker, batch_size
        self._verbose, self._log_stats = verbose, log_stats

    def stage_setup(self) -> None:
        self._model.setup()
        self._text_match.embed()

    @property
    def model(self) -> ModelInterface:
        return self._model

    @property
    def resources(self) -> CuratorStageResource:
        return CuratorStageResource(gpus=self._num_gpus_per_worker)

    def process_data(self, tasks):
        self._timer.reinit(self, sum(task.get_major_size() for task in tasks))
        clips = [clip for task in tasks for clip in task.video.clips]
        with self._timer.time_process(num_samples=max(1, len(clips))):
            todo, inputs = [], []
            for clip in clips:
                frames = clip.intern_video_2_frames.resolve()
                if frames is None:
                    clip.errors["iv2_frames"] = "none"
                elif frames.size == 0:
                    clip.errors["iv2_frames"] = "empty"
                else:
                    todo.append(clip)
                    inputs.append(frames)
            try:
                if inputs:
                    embeddings = self._model.encode_batched_videos(inputs, self._batch_size)
                    assert len(embeddings) == len(todo), f"Expected {len(todo)} embeddings, but got {len(embeddings)}"
                    for clip, e in zip(todo, embeddings):
                        clip.intern_video_2_embedding = e
                for clip in clips:
                    self._text_match.verify(clip)
            finally:
                for clip in clips:
                    clip.intern_video_2_frames.drop()
        if self._log_stats:
            stage_name, stats = self._timer.log_stats()
            for task in tasks:
                task.stage_perf[stage_name] = stats
        return tasks
