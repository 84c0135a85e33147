"""What does a resolution switch cost an NVDEC session?  Alternating 1280x720 / 3840x2160 clips on ONE session (the cuvid decoder is
destroyed and re-created at every switch) against one session per stream shape (runtime.DecoderPool.decoder(shape)).
    python tools/mixed_decode_probe.py   ->  one JSON line (1 GPU)"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cosmos_curate_b200.runtime import Decoder, alloc_nv12_pool, get_context  # noqa: E402
from tools import synth_h264  # noqa: E402

ctx = get_context()
clips = {(1280, 720): synth_h264.make_coded_clip(1280, 720, 30, 1.0, seed=1, gop=30, bitrate=2e6),
         (3840, 2160): synth_h264.make_coded_clip(3840, 2160, 30, 1.0, seed=2, gop=30, bitrate=16e6)}
pools = {k: alloc_nv12_pool(ctx, 2, k[0], k[1], "swscale") for k in clips}
ids, slots = np.array([0, 29], dtype=np.int32), np.arange(2, dtype=np.int32)
order = [k for _ in range(8) for k in clips]  # 720p, 4K, 720p, 4K, ...


def run(decoder_for):
    per = []
    for k in order:
        t0 = time.perf_counter()
        decoder_for(k).decode(clips[k], ids, pools[k], slots)
        per.append(time.perf_counter() - t0)
    return per


one = Decoder(ctx)
run(lambda k: one)  # warm-up (first creation, staging buffers)
shared = run(lambda k: one)
per_shape = {k: Decoder(ctx) for k in clips}
run(lambda k: per_shape[k])
split = run(lambda k: per_shape[k])
same = []
for k in clips:  # same-shape back to back on one session: the decode time itself
    for _ in range(2):
        per_shape[k].decode(clips[k], ids, pools[k], slots)
    t0 = time.perf_counter()
    for _ in range(4):
        per_shape[k].decode(clips[k], ids, pools[k], slots)
    same.append((time.perf_counter() - t0) / 4)
print(json.dumps({"clips": "30-frame 1280x720 and 3840x2160 H.264 clips, alternating, 16 decodes",
                  "one_session_ms_per_clip": 1e3 * float(np.mean(shared)), "session_per_shape_ms_per_clip": 1e3 * float(np.mean(split)),
                  "same_shape_ms_per_clip": {"720p": 1e3 * same[0], "2160p": 1e3 * same[1]},
                  "switch_cost_ms": 1e3 * float(np.mean(shared) - np.mean(split))}))
