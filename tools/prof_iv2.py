"""Times the InternVideo2-1B clip-embedding tower (cb_iv2_forward) at batch 8 and 4 frames, with a library-path baseline on the same card.

    python tools/prof_iv2.py [--rounds 3] [--steps 5] [--out results.json]

Arms, alternated within each round (seeded weights, gammas ~ U(0.1, 1); 8 random clips):
  * tower:      cb_iv2_forward, clips/s and achieved TFLOP/s against flops_per_clip (2 M N K of the block GEMMs + 4 T^2 d heads
                of attention, 40 layers: 2.31 TFLOP per clip);
  * attention:  cb_attention_stream_f16 alone at the tower's shape (8 clips x 16 heads x 1025 tokens x 88), TFLOP/s of 4 T^2 d heads;
  * baseline:   oracle/internvideo2.py in bf16 (cuBLAS GEMMs + torch SDPA), the precision the reference runs at.
Then one profiled tower call: milliseconds per kernel category (cb_profile_*).  The embeddings of the tower and of the bf16 baseline are
compared in the same run.  The first line has the card name, power limit and SM clock (nvidia-smi, read only); the SM clock is read
again while the tower runs (`clocks_under_load`).  Ranges are min..max over the rounds.
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from cosmos_curate_b200.runtime import Context, Iv2Tower  # noqa: E402
from oracle import internvideo2 as O  # noqa: E402

BATCH = 8


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return dict(zip(q.split(","), [s.strip() for s in out.splitlines()[0].split(",")]))
    except (OSError, subprocess.CalledProcessError) as e:
        return {"error": str(e)}


def timed(fn, steps: int) -> float:
    """Seconds per call: `steps` calls between two synchronises."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_iv2 needs a CUDA device")
    info = card()
    print(json.dumps({"card": info}))
    cfg = O.IV2_1B
    ctx = Context(0)
    w = O.random_weights(cfg, seed=1, gamma=(0.1, 1.0))
    frames = np.random.default_rng(2).integers(0, 256, (BATCH, cfg.frames, 224, 224, 3), dtype=np.uint8)
    tubes = torch.from_numpy(O.tube_from_frames(frames)).cuda()
    tower = Iv2Tower(ctx, cfg.to_dict(), w, max_clips=BATCH)
    wb = {k: torch.from_numpy(v).cuda().bfloat16() for k, v in w.items()}
    qkv = (torch.randn(BATCH, cfg.tokens, 3 * cfg.hidden, device="cuda") * 1.5).half()

    def baseline():
        with torch.no_grad():
            return O.forward(cfg, wb, tubes, dtype=torch.bfloat16, device="cuda")

    arms = {"tower": lambda: tower.forward(tubes), "attention": lambda: ctx.attention_stream(qkv, cfg.heads), "baseline_bf16": baseline}
    for fn in arms.values():  # warm-up: module loads, cuBLAS algorithm choice
        fn()
    res: dict[str, list[float]] = {k: [] for k in arms}
    for _ in range(args.rounds):
        for name, fn in arms.items():
            res[name].append(timed(fn, args.steps))
    flops = O.flops_per_clip(cfg) * BATCH
    attn_flops = 4.0 * cfg.tokens**2 * (cfg.hidden // cfg.heads) * cfg.heads * BATCH
    rows = {
        "tower_clips_per_s": [BATCH / s for s in res["tower"]],
        "tower_tflops": [flops / s / 1e12 for s in res["tower"]],
        "attention_ms": [s * 1e3 for s in res["attention"]],
        "attention_tflops": [attn_flops / s / 1e12 for s in res["attention"]],
        "baseline_bf16_clips_per_s": [BATCH / s for s in res["baseline_bf16"]],
        "baseline_bf16_tflops": [flops / s / 1e12 for s in res["baseline_bf16"]],
    }
    summary = {k: {"min": min(v), "max": max(v), "runs": [round(x, 3) for x in v]} for k, v in rows.items()}
    for _ in range(args.steps):  # queued work keeps the GPU busy while nvidia-smi reads the clock
        tower.forward(tubes)
    under_load = card()
    torch.cuda.synchronize()
    ctx.profile_begin()
    tower.forward(tubes)
    prof = ctx.profile_end()
    emb = tower.forward(tubes)
    ref = baseline()
    cos = torch.nn.functional.cosine_similarity(emb, ref, dim=-1)
    result = {"card": info, "clocks_under_load": {k: under_load.get(k) for k in ("clocks.sm", "clocks.max.sm")}, "batch": BATCH, "frames": cfg.frames, "tflop_per_clip": O.flops_per_clip(cfg) / 1e12, "timing": summary,
              "profile_ms": {k: round(v["ms"], 3) for k, v in prof.items() if v["launches"]},
              "profile_launches": {k: v["launches"] for k, v in prof.items() if v["launches"]},
              "tower_vs_baseline_bf16": {"min_cosine": cos.min().item(), "max_abs": (emb - ref).abs().max().item()}}  # fmt: skip
    print(json.dumps(result))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
