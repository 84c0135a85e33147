"""cosmos_curate_b200/compare.py: the reference's stage-output comparison semantics (stage_compare.py `_compare_values`), checked
(a) against what the reference functions themselves returned on a case table (stored in tests/golden/reference_live.json.gz by
`python -m oracle.make_reference_golden`) and (b) against the known answers of the reference's own tests
(tests/cosmos_curate/core/utils/misc/test_stage_compare.py:112-162), then used the way the reference uses it: on task lists."""

from __future__ import annotations

import gzip
import json
import uuid

import attrs
import numpy as np
import pytest

from conftest import GOLDEN
from cosmos_curate_b200 import compare as C
from cosmos_curate_b200.data_model import Clip, SplitPipeTask, Video


@attrs.define
class _Leaf:
    score: float
    vec: np.ndarray
    tags: dict


def _cases():
    a = np.arange(6, dtype=np.float32).reshape(2, 3)
    nan = np.array([1.0, np.nan, 3.0], dtype=np.float32)
    return [
        ("equal", {"a": a, "b": [1, "x", (2, 3)]}, {"a": a.copy(), "b": [1, "x", (2, 3)]}, 0.0),
        ("within", a, a + np.float32(9e-4), 1e-3),
        ("beyond", a, a + np.float32(2e-3), 1e-3),
        ("rtol_zero", np.array([1e6], np.float32), np.array([1e6 + 1], np.float32), 0.5),  # allclose's default rtol would pass this
        ("unsigned", np.array([0, 255], np.uint8), np.array([1, 0], np.uint8), 0.0),
        ("nan_match", nan, nan.copy(), 0.0),
        ("nan_one_side", nan, np.array([1.0, 2.0, 3.0], np.float32), 0.0),
        ("nan_plus_diff", nan, np.array([1.5, np.nan, 3.0], np.float32), 0.1),
        ("shape", a, a.T.copy(), 1.0),
        ("dtype_ok", a, a.astype(np.float64), 0.0),  # both ndarray: dtypes may differ
        ("type", [1, 2], (1, 2), 0.0),
        ("int_float", {"k": 1}, {"k": 1.0}, 0.0),
        ("keys", {"a": 1, "b": 2}, {"a": 1, "c": 2}, 0.0),
        ("length", [1, 2, 3], [1, 2], 0.0),
        ("strings", np.array(["a", "b"]), np.array(["a", "c"]), 0.0),
        ("bytes", b"abc", b"abd", 0.0),
        ("attrs", _Leaf(1.0, a, {"x": [a]}), _Leaf(1.5, a + 1, {"x": [a * 2]}), 0.25),
        ("nested_path", {"v": [{"w": a}]}, {"v": [{"w": a + 1}]}, 0.0),
        ("empty", [], [], 0.0),
    ]


def test_compare_values_equals_the_reference_comparator():
    want = json.loads(gzip.decompress((GOLDEN / "reference_live.json.gz").read_bytes()))["compare_table"]
    cases = _cases()
    assert sorted(want) == sorted(name for name, *_ in cases)
    for name, g, c, atol in cases:
        got = [(d.field, d.detail, d.max_diff_observed, d.shape_mismatch) for d in C.compare_values("root", g, c, atol=atol)]
        assert repr(got) == want[name], name  # repr: NaN-carrying details compare equal as text


def test_reference_known_answers():
    a = np.array([1.0, 2.0], dtype=np.float32)
    assert C.compare_values("", {"x": a}, {"x": a.copy()}, atol=0.0) == []
    assert C.compare_values("", a, a + np.float32(5e-4), atol=1e-3) == []
    d = C.compare_values("arr", np.array([0], np.uint8), np.array([1], np.uint8), atol=0.0)
    assert len(d) == 1 and d[0].max_diff_observed == 1.0  # not 255: the difference is taken in float64
    n = np.array([np.nan, 1.0], np.float32)
    assert C.compare_values("arr", n, n.copy(), atol=0.0) == []
    d = C.compare_values("arr", n, np.array([np.nan, 3.0], np.float32), atol=0.5)
    assert d[0].detail == "max diff 2.0" and d[0].max_diff_observed == 2.0  # the matching NaNs do not poison the maximum
    d = C.compare_values("arr", np.zeros((2, 3)), np.zeros((3, 2)), atol=1.0)
    assert d[0].shape_mismatch and "shape mismatch" in d[0].detail
    assert C.compare_values("v", 1, 1.0, atol=1.0)[0].detail == "type mismatch golden=int new=float"


def test_task_lists_the_way_stage_replay_compares_them():
    """SplitPipeTask semantic fields (session_id, videos, errors): stage_perf and timing never count; an embedding off by more than
    atol, a moved clip or a new error key do."""

    def task(score=4.25, emb_shift=0.0, filtered=False, perf=1.0):
        rng = np.random.default_rng(0)
        e = rng.standard_normal(8).astype(np.float32)
        clip = Clip(uuid=uuid.UUID(int=7), source_video="v.mp4", span=(0.0, 5.0), encoded_data=b"abc")
        clip.aesthetic_score, clip.openai_embedding = score, e + np.float32(emb_shift)
        v = Video(input_video="v.mp4", clips=[] if filtered else [clip], filtered_clips=[clip] if filtered else [])
        t = SplitPipeTask(session_id="s", video=v)
        t.stage_perf["X"] = perf
        return t

    assert C.compare_tasks([task()], [task(perf=9.0)], atol=0.0) == []
    assert C.compare_tasks([task()], [task(emb_shift=5e-4)], atol=1e-3) == []
    bad = C.compare_tasks([task()], [task(emb_shift=5e-3)], atol=1e-3)
    assert [d.field for _, d in bad] == ["videos[0].clips[0].openai_embedding"] and bad[0][1].max_diff_observed == pytest.approx(5e-3, rel=1e-3)
    assert C.compare_tasks([task()], [task(score=4.26)], atol=1e-3)[0][1].field == "videos[0].clips[0].aesthetic_score"  # scalars: exact
    moved = C.compare_tasks([task()], [task(filtered=True)], atol=1e-3)
    assert {d.field for _, d in moved} == {"videos[0].clips", "videos[0].filtered_clips"}
    assert C.compare_tasks([task()], [], atol=0.0)[0][1].field == "tasks"
    assert C.compare_tasks([task()], [task(perf=9.0)], atol=0.0, field_names=None)[0][1].field == "stage_perf.X"  # generic comparator: everything
