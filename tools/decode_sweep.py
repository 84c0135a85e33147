"""NVDEC decode-only rate vs number of concurrent sessions (one GPU): how many sessions the 7 engines of an H100 need.
    python tools/decode_sweep.py [sessions ...]   ->  one JSON line per setting
"""

from __future__ import annotations

import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import bench  # noqa: E402


def main() -> None:
    settings = [int(a) for a in sys.argv[1:]] or [8, 14, 20, 28, 40]
    clips = bench.make_clips(16, 0)
    sintel = (ROOT / "tests" / "golden" / "sintel_clip_10s.mp4").read_bytes()
    import torch  # noqa: F401

    from cosmos_curate_b200.runtime import Context, DecoderPool, decode_discard

    ctx = Context(0)
    for n in settings:
        pool = DecoderPool(ctx, n)
        row = {"sessions": n}
        for name, data, secs in (("synthetic_1080p_4mbps", clips, 4.0), ("sintel_480p_real", [sintel], 3.0)):
            deadline = [0.0]

            def loop(dec, k, data=data):
                c, i = 0, k
                while time.perf_counter() < deadline[0]:
                    c += decode_discard(dec, data[i % len(data)])
                    i += n
                return c

            [f.result() for f in [pool.submit(lambda dec, k=k, data=data: decode_discard(dec, data[k % len(data)])) for k in range(n)]]
            t0 = time.perf_counter()
            deadline[0] = t0 + secs
            frames = sum(f.result() for f in [pool.submit(loop, k) for k in range(n)])
            row[name + "_fps"] = frames / (time.perf_counter() - t0)
        pool.close()
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
