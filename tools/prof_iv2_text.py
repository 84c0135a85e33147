"""Times InternVideo2 text embedding (`InternVideo2MultiModality.encode_texts`: tokenizer + cb_iv2_text_forward, 19 layers of
BERT-large) at 8, 64 and 256 texts of 40 tokens each.

    python tools/prof_iv2_text.py [--rounds 3] [--steps 5] [--out results.json]

Seeded weights at the real shape (vocab 30522) with the synthetic test vocabulary (tests/golden/bert_vocab_synth.txt) for the
tokenizer; every text is long enough to fill all 40 tokens.  Per batch size: texts/s of the whole call (host tokenization and the
copy back included) and of the tower alone on pre-tokenized ids, with achieved TFLOP/s against oracle.internvideo2_text.flops_per_text
(2 M N K of the layer GEMMs + 4 T^2 d of attention: 19.3 GFLOP per 40-token text).  Then one profiled tower call at 256 texts:
milliseconds per kernel category (cb_profile_*).  The first line has the card name, power limit and SM clock (nvidia-smi, read only);
the SM clock is read again while the tower runs.  Ranges are min..max over the rounds.
"""

from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from cosmos_curate_b200.models.internvideo2 import IV2_TEXT_CFG, MAX_TXT_L, InternVideo2MultiModality  # noqa: E402
from oracle import internvideo2_text as O  # noqa: E402
from tools.prof_iv2 import card  # noqa: E402

BATCHES = (8, 64, 256)
VOCAB = ROOT / "tests" / "golden" / "bert_vocab_synth.txt"
WORDS = "a the man woman dog cat car bike walks runs rides plays in on at park street beach red blue green small large video".split()


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
        raise SystemExit("prof_iv2_text needs a CUDA device")
    info = card()
    print(json.dumps({"card": info}))
    rng = np.random.default_rng(0)
    texts = [" ".join(rng.choice(WORDS, 50)) for _ in range(max(BATCHES))]
    model = InternVideo2MultiModality(seed=1, vocab_file=VOCAB, max_texts=max(BATCHES))
    model.setup_text()
    tower = model._text_tower
    ids, lengths = model.tokenizer(texts, MAX_TXT_L)
    assert (lengths == MAX_TXT_L).all()
    arms = {}
    for b in BATCHES:
        arms[f"encode_texts_{b}"] = (b, lambda b=b: model.encode_texts(texts[:b]))
        arms[f"tower_{b}"] = (b, lambda b=b: tower.forward(ids[:b], lengths[:b]))
    for _, fn in arms.values():  # warm-up: module loads, every shape once
        fn()
    res: dict[str, list[float]] = {k: [] for k in arms}
    for _ in range(args.rounds):
        for name, (_, fn) in arms.items():
            res[name].append(timed(fn, args.steps))
    per_text = O.flops_per_text(O.IV2_TEXT, MAX_TXT_L)
    rows = {}
    for name, (b, _) in arms.items():
        rows[f"{name}_texts_per_s"] = [b / s for s in res[name]]
        rows[f"{name}_tflops"] = [per_text * b / s / 1e12 for s in res[name]]
    summary = {k: {"min": min(v), "max": max(v), "runs": [round(x, 3) for x in v]} for k, v in rows.items()}
    for _ in range(args.steps):  # queued work keeps the GPU busy while nvidia-smi reads the clock
        tower.forward(ids, lengths)
    under_load = card()
    torch.cuda.synchronize()
    ctx = tower.ctx
    ctx.profile_begin()
    tower.forward(ids, lengths)
    prof = ctx.profile_end()
    result = {"card": info, "clocks_under_load": {k: under_load.get(k) for k in ("clocks.sm", "clocks.max.sm")}, "tokens": MAX_TXT_L,
              "layers": IV2_TEXT_CFG["layers"], "gflop_per_text": per_text / 1e9, "timing": summary,
              "profile_ms_256": {k: round(v["ms"], 3) for k, v in prof.items() if v["launches"]},
              "profile_launches_256": {k: v["launches"] for k, v in prof.items() if v["launches"]}}  # fmt: skip
    print(json.dumps(result))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
