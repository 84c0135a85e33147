"""CuratorStage implementations of the path.

Same-name drop-ins (constructor arguments, task mutations and error convention of the reference):
    AestheticFilterStage        cosmos_curate/pipelines/video/filtering/aesthetics/aesthetic_filter_stages.py:41-221
    ClipFrameExtractionStage    cosmos_curate/pipelines/video/clipping/clip_frame_extraction_stages.py:43-192
    VideoFrameExtractionStage   cosmos_curate/pipelines/video/clipping/frame_extraction_stages.py:71-204
    ImageCLIPEmbeddingStage     cosmos_curate/pipelines/image/embedding/image_embedding_stages.py:219-283
    TransNetV2ClipExtractionStage  cosmos_curate/pipelines/video/clipping/transnetv2_extraction_stages.py:39-212
    VideoDownloader             cosmos_curate/pipelines/video/read_write/download_stages.py:40-228 (local files only, host only)
    FixedStrideExtractorStage   cosmos_curate/pipelines/video/clipping/clip_extraction_stages.py:664-760 (host only)
    ClipWriterStage             cosmos_curate/pipelines/video/read_write/metadata_writer_stage.py:66-1020 (local output directory, host only)
    InternVideo2FrameCreationStage  cosmos_curate/pipelines/video/embedding/internvideo2_stages.py:43-184 (the tower's input tube)
    InternVideo2EmbeddingStage  cosmos_curate/pipelines/video/embedding/internvideo2_stages.py:187-309 (the 1B vision tower; no text tower)
    ClipFrameEmbeddingStage     local producer of clip.openai_embedding (the slot of embedding/openai_embedding_stage.py:47-190)
New fused stage (replaces ClipFrameExtractionStage -> AestheticFilterStage [-> clip embedding] in one GPU pass):
    NvdecClipAestheticStage
    NvdecShotDetectionStage      (VideoFrameExtractionStage -> TransNetV2ClipExtractionStage, frames stay in HBM)
    ClipStreamCopyStage          (ClipTranscodingStage without the transcode: clip mp4s by stream copy, clip_extraction_stages.py:167-442)
    NvdecInternVideo2EmbeddingStage  (InternVideo2FrameCreationStage(source="nvdec") -> InternVideo2EmbeddingStage, tubes stay in HBM)
"""

from .aesthetic_filter import AestheticFilterStage  # noqa: F401
from .clip_writer import ClipWriterStage  # noqa: F401
from .clip_embedding import ClipFrameEmbeddingStage  # noqa: F401
from .clip_stream_copy import ClipStreamCopyStage  # noqa: F401
from .download import VideoDownloader  # noqa: F401
from .fixed_stride import FixedStrideExtractorStage  # noqa: F401
from .fused_clip import NvdecClipAestheticStage  # noqa: F401
from .frame_extraction import ClipFrameExtractionStage, VideoFrameExtractionStage  # noqa: F401
from .internvideo2_embedding import InternVideo2EmbeddingStage  # noqa: F401
from .internvideo2_frames import InternVideo2FrameCreationStage  # noqa: F401
from .internvideo2_fused import NvdecInternVideo2EmbeddingStage  # noqa: F401
from .image_embedding import ImageCLIPEmbeddingStage  # noqa: F401
from .transnetv2_extraction import NvdecShotDetectionStage, TransNetV2ClipExtractionStage  # noqa: F401
