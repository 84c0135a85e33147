"""Times InternVideo2 clip embedding from mp4 bytes: the two-stage chain against the fused stage, and the two resident-input paths.

    python tools/prof_iv2_stage.py [--clips 16] [--rounds 2] [--out results.json]

Full-depth seeded weights (InternVideo2-1B, 4 frames); synthetic 1080p 10 s clips (bench.make_clips, 30 fps, 4 Mb/s).  Arms, alternated
within each round, each timed as wall time between two device synchronisations:
  * chain:           InternVideo2FrameCreationStage(source="nvdec", 4-frame formulator) -> InternVideo2EmbeddingStage (tubes via the host);
  * fused:           NvdecInternVideo2EmbeddingStage, seek_keyframes=False;
  * fused_seek:      NvdecInternVideo2EmbeddingStage, seek_keyframes=True;
  * resident_fused:  cb_iv2_embed_surfaces on the clips' kept frames, already decoded into one surface pool;
  * resident_tube:   cb_video_tube + cb_iv2_forward on the same pool.
The first line has the card name, power limit and SM clock (nvidia-smi, read only) and whether NVDEC or the host decoder (host_decode.py)
served the decodes: where NVDEC is not usable the e2e arms measure host decode.  Ranges are min..max clips/s over the rounds.  The
embeddings of the arms are compared at the end (they must be bitwise equal).
"""

from __future__ import annotations

import argparse
import json
import sys
import time
import uuid
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import bench  # noqa: E402
from tools.prof_iv2 import card  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--decoders", type=int, default=8)
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    datas = bench.make_clips(args.clips, rank=0)  # before CUDA: the generator forks
    from cosmos_curate_b200.data_model import Clip, SplitPipeTask, Video
    from cosmos_curate_b200.models.internvideo2 import InternVideo2MultiModality
    from cosmos_curate_b200.models.internvideo2_frames import InternVideo2FrameFormulator
    from cosmos_curate_b200.runtime import DecoderPool, SurfacePools, collect_group, get_context, nvdec_available
    from cosmos_curate_b200.stages import InternVideo2EmbeddingStage, InternVideo2FrameCreationStage, NvdecInternVideo2EmbeddingStage
    from cosmos_curate_b200.stages.internvideo2_frames import plan_clip

    ctx = get_context()
    head = {"card": card(), "decode": "host (libavcodec)" if not nvdec_available(ctx) else "nvdec", "clips": args.clips,
            "clip": f"{bench.FRAME_W}x{bench.FRAME_H} {bench.FPS} fps {bench.SECONDS:.0f} s"}  # fmt: skip
    print(json.dumps(head), flush=True)

    model = InternVideo2MultiModality(seed=0, max_clips=8)
    model.setup()
    tower = model.tower

    def tasks():
        clips = [Clip(uuid=uuid.uuid4(), source_video="v.mp4", span=(0.0, bench.SECONDS), encoded_data=d) for d in datas]
        return [SplitPipeTask(session_id="s", video=Video(input_video=f"v{i}.mp4", clips=clips[i::4])) for i in range(4)]

    frames = InternVideo2FrameCreationStage(source="nvdec", num_decoders=args.decoders, model=InternVideo2FrameFormulator(num_frames=4))
    frames.stage_setup()
    embed = InternVideo2EmbeddingStage(batch_size=8, model=model)
    embed.stage_setup()
    fused = {seek: NvdecInternVideo2EmbeddingStage(batch_size=8, num_decoders=args.decoders, seek_keyframes=seek, model=model) for seek in (False, True)}
    for st in fused.values():
        st.stage_setup()

    # the resident pair: every clip's kept frames in one pool, decoded once
    plans = [plan_clip(Clip(uuid=uuid.uuid4(), source_video="v.mp4", span=(0.0, bench.SECONDS)), d, 2.0, 4) for d in datas]
    size = plans[0][0]
    pools = SurfacePools(ctx, 1, 4, "swscale")
    pool = pools.get(size, sum(len(p[1]) for p in plans))
    dp = DecoderPool(ctx, args.decoders)
    jobs = dp.submit_group(pool, size, [(d, p[1]) for d, p in zip(datas, plans)])
    _, errs = collect_group(jobs)
    assert not any(errs), errs
    slots = np.concatenate([first + p[2] for (first, _), p in zip(jobs, plans)]).astype(np.int32)
    n = len(datas)

    out = {}

    def run_chain():
        t = tasks()
        frames.process_data(t)
        embed.process_data(t)
        return t

    def run_fused(seek):
        def f():
            t = tasks()
            fused[seek].process_data(t)
            return t

        return f

    arms = {"chain": run_chain, "fused": run_fused(False), "fused_seek": run_fused(True),
            "resident_fused": lambda: tower.embed_pool(pool, slots),
            "resident_tube": lambda: tower.forward(ctx.video_tube(pool, 224, 224, slots=slots).view(n, 4, 3, 224, 224))}  # fmt: skip
    rates: dict[str, list[float]] = {k: [] for k in arms}
    for name, fn in arms.items():  # warm-up: every shape, every session
        out[name] = fn()
    torch.cuda.synchronize()
    for r in range(args.rounds):
        for name, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = fn()
            torch.cuda.synchronize()
            rates[name].append(n / (time.perf_counter() - t0))
            out[name] = res
        print(json.dumps({"round": r, **{k: round(v[-1], 2) for k, v in rates.items()}}), flush=True)

    def embs(res):
        if isinstance(res, torch.Tensor):
            return res.cpu().numpy()
        return np.concatenate([c.intern_video_2_embedding for t in res for c in t.video.clips])

    order = [i for t in range(4) for i in range(t, n, 4)]  # the stages' clip order -> the clip index
    ref = embs(out["resident_tube"])
    same = {}
    for k, res in out.items():
        e = embs(res)
        if not isinstance(res, torch.Tensor):
            e = e[np.argsort(order)]
        same[k] = bool(np.array_equal(e, ref))
    summary = {"clips_per_s": {k: f"{min(v):.2f}..{max(v):.2f}" for k, v in rates.items()}, "bitwise_equal_to_resident_tube": same,
               "fused_stats": fused[False].last_call_stats, "fused_seek_stats": fused[True].last_call_stats, **head}  # fmt: skip
    print(json.dumps(summary), flush=True)
    if args.out:
        Path(args.out).write_text(json.dumps(summary, indent=1))
    for st in (frames, *fused.values()):
        st.destroy()
    dp.close()


if __name__ == "__main__":
    main()
