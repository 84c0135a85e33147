"""Run the reference's own functions on the seeded inputs of oracle/reference_cases.py and store what they returned:

    python -m oracle.make_reference_golden        # needs a checkout of the reference (CURATE_REFERENCE_ROOT)

writes tests/golden/reference_live.json.gz (results as text: float.hex / repr, so every bit is kept; sha256 of each float32
video tube)."""

from __future__ import annotations

import gzip
import hashlib
import json
import sys
from pathlib import Path

import numpy as np

from oracle import ref_import
from oracle import reference_cases as RC

GOLDEN = Path(__file__).resolve().parent.parent / "tests" / "golden"


def main() -> None:
    out: dict = {"n_cases": RC.N_CASES}
    du = ref_import.decoder_utils()
    rows = []
    for seed in range(RC.N_CASES):
        c = RC.sample_closest_case(seed)
        ts = c["ts"]
        want = du.sample_closest(ts, sample_rate=c["rate"], start=ts[0], stop=ts[-1], endpoint=c["endpoint"], dedup=c["dedup"])
        rows.append({"sample": [np.asarray(w).tolist() for w in want], "closest": du.find_closest_indices(ts, c["dst"]).tolist()})
    out["sample_closest"] = rows
    f = ref_import.fixed_stride_functions()
    rows = []
    for seed in range(RC.N_CASES):
        c = RC.fixed_stride_case(seed)
        spans = f["_make_spans_fixed_stride"](0.0, c["end"], c["clip_len"], c["stride"], c["min_len"])
        rows.append({"spans": [(float.hex(a), float.hex(b)) for a, b in spans], "uuids": [str(u) for u in f["_make_clip_uuids"](c["session"], spans[:50])]})
    out["fixed_stride"] = rows
    rows = []
    for seed in range(RC.N_CASES):
        c = RC.chunk_case(seed)
        spans = [(float(i), float(i) + d) for i, d in enumerate(c["durs"])]
        rows.append([len(ch) for ch in ref_import.grouping_module().split_by_chunk_size(spans, c["per_chunk"] * 8, lambda s: int(s[1] - s[0]))])
    out["chunk_sizes"] = rows
    f = ref_import.transnetv2_stage_functions()
    rows = []
    for seed in range(RC.N_CASES):
        c = RC.shot_case(seed)
        want = f["_get_scenes"](c["track"], entire_scene_as_clip=c["entire"])
        row = {"scenes": want.tolist(), "dtype": str(want.dtype), "filtered": None}
        if len(want):
            row["filtered"] = f["_get_filtered_scenes"](want.copy(), min_length=c["min_len"], max_length=c["max_len"], max_length_mode=c["mode"], crop_length=c["crop"]).tolist()
        rows.append(row)
    out["shot_logic"] = rows
    ref = ref_import.stage_compare_functions()["_compare_values"]
    rows = []
    for seed in range(RC.N_CASES):
        c = RC.compare_case(seed)
        rows.append([repr([RC.diff_key(d) for d in ref("t", g, cand, atol=c["atol"])]) for g, cand in ((c["golden"], c["candidate"]), (c["golden"], c["golden"]))])
    out["compare_values"] = rows
    sys.path.insert(0, str(GOLDEN.parent))
    from test_compare_cpu import _cases  # the hand-written case table lives with its test

    out["compare_table"] = {name: repr([RC.diff_key(d) for d in ref("root", g, c, atol=atol)]) for name, g, c, atol in _cases()}
    form = ref_import.internvideo2_formulator()
    rows = []
    for seed in range(RC.N_CASES):
        c = RC.video_tube_case(seed)
        want = form._construct_frames(c["frames"], fnum=8, target_size=c["target"])
        rows.append({"shape": list(want.shape), "dtype": str(want.dtype), "sha256": hashlib.sha256(np.ascontiguousarray(want).tobytes()).hexdigest()})
    out["video_tube"] = rows
    (GOLDEN / "reference_live.json.gz").write_bytes(gzip.compress(json.dumps(out, separators=(",", ":")).encode(), mtime=0))


if __name__ == "__main__":
    main()
