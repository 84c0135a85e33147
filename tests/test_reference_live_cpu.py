"""Differential tests against the reference's OWN functions on randomly generated inputs nobody hand-picked: frame-index math
(decoder_utils.find_closest_indices / sample_closest), fixed-stride spans, chunk sizes, shot logic, the video-tube formulation and
the stage-replay comparator must agree with the reference.

The inputs are rebuilt from seeds (oracle/reference_cases.py); what the reference's functions returned on them was stored in
tests/golden/reference_live.json.gz by `python -m oracle.make_reference_golden`, so the comparison runs without a checkout of the
reference."""

from __future__ import annotations

import gzip
import hashlib
import json

import numpy as np

from conftest import GOLDEN
from cosmos_curate_b200 import compare as C
from cosmos_curate_b200 import sampling as S
from cosmos_curate_b200 import spans as SP
from oracle import reference_cases as RC

WANT = json.loads(gzip.decompress((GOLDEN / "reference_live.json.gz").read_bytes()))
SEEDS = range(RC.N_CASES)
assert WANT["n_cases"] == RC.N_CASES


def _sample_closest_agrees_with_the_reference(seed):
    c, want = RC.sample_closest_case(seed), WANT["sample_closest"][seed]
    ts = c["ts"]
    got = S.sample_closest(ts, c["rate"], start=ts[0], stop=ts[-1], endpoint=c["endpoint"], dedup=c["dedup"])
    assert len(got) == len(want["sample"])
    for g, w in zip(got, want["sample"]):
        assert np.array_equal(np.asarray(g), np.asarray(w))
    assert np.array_equal(S.find_closest_indices(ts, c["dst"]), np.asarray(want["closest"]))


def _fixed_stride_spans_and_uuids_agree_with_the_reference(seed):
    c, want = RC.fixed_stride_case(seed), WANT["fixed_stride"][seed]
    got = SP.make_spans_fixed_stride(0.0, c["end"], c["clip_len"], c["stride"], c["min_len"])
    assert [[float.hex(a), float.hex(b)] for a, b in got] == want["spans"]
    assert [str(u) for u in SP.make_clip_uuids(c["session"], got[:50])] == want["uuids"]


def _chunk_sizes_agree_with_the_reference(seed):
    c = RC.chunk_case(seed)
    spans = [(float(i), float(i) + d) for i, d in enumerate(c["durs"])]
    size = lambda s: int(s[1] - s[0])  # noqa: E731
    assert [len(ch) for ch in SP.split_by_chunk_size(spans, c["per_chunk"] * 8, size)] == WANT["chunk_sizes"][seed]


def _compare_values_agrees_with_the_reference(seed):
    c, want = RC.compare_case(seed), WANT["compare_values"][seed]
    for (g, cand), w in zip(((c["golden"], c["candidate"]), (c["golden"], c["golden"])), want):
        assert repr([RC.diff_key(d) for d in C.compare_values("t", g, cand, atol=c["atol"])]) == w  # repr: NaN-carrying details compare equal as text


def _shot_logic_agrees_with_the_reference(seed):
    """0/1 transition tracks -> scenes -> filtered scenes: transnetv2_extraction_stages._get_scenes / _get_filtered_scenes."""
    from cosmos_curate_b200 import shots

    c, want = RC.shot_case(seed), WANT["shot_logic"][seed]
    got = shots.scenes_from_predictions(c["track"], entire_scene_as_clip=c["entire"])
    assert got.tolist() == want["scenes"] and str(got.dtype) == want["dtype"]
    if want["filtered"] is not None:
        got_f = shots.filter_scenes(got.copy(), min_length=c["min_len"], max_length=c["max_len"], max_length_mode=c["mode"], crop_length=c["crop"])
        assert np.asarray(got_f).tolist() == want["filtered"]


def _video_tube_oracle_agrees_with_the_reference_formulation(seed):
    """oracle/video_tube.py vs InternVideo2MultiModality._construct_frames (cv2.resize + numpy) on arbitrary sizes, every float32 bit:
    up- and down-scaling, 1-pixel sources and targets, the exact-2x INTER_AREA reroute, the copy for equal sizes."""
    from oracle import video_tube as T

    c, want = RC.video_tube_case(seed), WANT["video_tube"][seed]
    got = T.construct_frames(c["frames"], fnum=8, target_size=c["target"])
    assert list(got.shape) == want["shape"] and str(got.dtype) == want["dtype"]
    assert hashlib.sha256(np.ascontiguousarray(got).tobytes()).hexdigest() == want["sha256"]


def _all_seeds(check):
    bad = []
    for seed in SEEDS:
        try:
            check(seed)
        except AssertionError as exc:
            bad.append(f"seed {seed}: {str(exc)[:200]}")
    assert not bad, "\n".join(bad)


def test_sample_closest_agrees_with_the_reference():
    _all_seeds(_sample_closest_agrees_with_the_reference)


def test_fixed_stride_spans_and_uuids_agree_with_the_reference():
    _all_seeds(_fixed_stride_spans_and_uuids_agree_with_the_reference)


def test_chunk_sizes_agree_with_the_reference():
    _all_seeds(_chunk_sizes_agree_with_the_reference)


def test_compare_values_agrees_with_the_reference():
    _all_seeds(_compare_values_agrees_with_the_reference)


def test_shot_logic_agrees_with_the_reference():
    _all_seeds(_shot_logic_agrees_with_the_reference)


def test_video_tube_oracle_agrees_with_the_reference_formulation():
    _all_seeds(_video_tube_oracle_agrees_with_the_reference_formulation)
