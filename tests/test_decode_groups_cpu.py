"""CPU tests of runtime.run_decode_groups, the decode-group loop of the NVDEC stages, with fake decoders, surface pools and CUDA
events that write one trace: the grouping by surface size and frame budget, where failing clips go, and the order of decode
submits, GPU work, event waits and write-backs that lets a surface pool be decoded into again only after its readers are done."""

from __future__ import annotations

import types
from concurrent.futures import Future

import numpy as np
import pytest
import torch

from cosmos_curate_b200 import runtime
from cosmos_curate_b200._lib import CurateB200Error

S, T = (320, 192), (256, 144)
MAX_FRAMES = 4


def _plan(ids, inverse=None, size=S):
    return size, np.asarray(ids, dtype=np.int32), np.arange(len(ids), dtype=np.int32) if inverse is None else np.asarray(inverse, np.int32)


# name -> plan result (None: too short, an exception: unreadable); BAD decodes fail
PLANS = {
    "a": _plan([0, 3, 7]), "b": _plan([1, 2], size=T), "c": _plan([0, 9], inverse=[0, 0, 1]), "d": _plan([0, 1, 2, 3]),
    "e": _plan([4, 5, 6], size=T), "f": _plan([2]), "g": _plan([0, 1, 2, 3, 4]), "h": None, "i": ValueError("span selects no frame"),
    "j": _plan([0, 8], size=T), "k": _plan([5]), "x": _plan([0, 1], size=T), "y": _plan([3, 4, 5], size=T),
}  # fmt: skip
BAD = {"j", "y"}
SCENARIOS = {
    "one group": ("a f", [(S, "a f")]),
    "two groups": ("a b f", [(S, "a f"), (T, "b")]),
    # S: 3 | 3 (on 2 surfaces) | 4 | 1 + 1, T: 2 | 3 | 2 + 2 | 3 (no clip decodes); g keeps 5 > MAX_FRAMES frames, h is too short,
    # i unreadable
    "many groups": ("a b c d e f g h i j k x y", [(S, "a"), (S, "c"), (S, "d"), (S, "f k"), (T, "b"), (T, "e"), (T, "j x"), (T, "y")]),
}


class _Run:
    """One run_decode_groups call on the fakes; `trace` holds ("submit", pool, size, names), ("compute", k, pool), ("wait", k) and
    ("finish", k) in call order."""

    def __init__(self, monkeypatch, names, depth):
        self.trace, self.errors, self.short, self.computed = [], {}, [], {}
        run = self

        class _Event:
            recorded = 0

            def record(self, stream):
                self.k = _Event.recorded
                _Event.recorded += 1

            def synchronize(self):
                run.trace.append(("wait", self.k))

        class _Decoders:
            def submit_group(self, pool, size, jobs, seek_keyframes=False):
                assert seek_keyframes is True
                run.trace.append(("submit", pool, size, " ".join(data for data, _ in jobs)))
                out, first = [], 0
                for data, ids in jobs:
                    assert np.array_equal(ids, PLANS[data][1]) and first + len(ids) <= pool.buf.shape[0]
                    f = Future()
                    if data in BAD:
                        f.set_exception(CurateB200Error(-4, "cb_decoder_decode", "decode: corrupt slice"))
                    else:
                        f.set_result({"frames_decoded": 10})
                    out.append((first, f))
                    first += len(ids)
                return out

        monkeypatch.setattr(torch.cuda, "Event", _Event)
        monkeypatch.setattr(torch.cuda, "current_stream", lambda: None)
        monkeypatch.setattr(runtime, "alloc_nv12_pool", lambda ctx, slots, w, h, colour: types.SimpleNamespace(buf=np.empty((slots, 0, 0))))
        pools = runtime.SurfacePools(types.SimpleNamespace(device=0), depth, MAX_FRAMES, "swscale")  # never outgrown: one object per ring slot
        decoders = _Decoders()

        def plan(clip, data):
            assert clip == data
            p = PLANS[data]
            if isinstance(p, Exception):
                raise p
            return p

        def compute(k, pool, ok, slots):
            run.trace.append(("compute", k, pool))
            run.computed[k] = ([clip for clip, _ in ok], slots)
            assert [n for _, n in ok] == [len(PLANS[clip][2]) for clip, _ in ok]
            return (lambda: run.trace.append(("finish", k))) if k % 3 != 2 else None  # a group may have nothing to write

        self.result = runtime.run_decode_groups([(n, n) for n in names.split()], plan, pools, lambda: decoders, compute,
                                                on_error=lambda clip, e: self.errors.setdefault(clip, e), max_frames=MAX_FRAMES,
                                                on_short=self.short.append, depth=depth, seek_keyframes=True)  # fmt: skip


@pytest.mark.parametrize("depth", [2, 3])
@pytest.mark.parametrize("scenario", list(SCENARIOS))
def test_groups_errors_and_the_order_of_submits_waits_and_write_backs(monkeypatch, depth, scenario):
    names, want_groups = SCENARIOS[scenario]
    run = _Run(monkeypatch, names, depth)
    n = len(want_groups)
    submits = [i for i, e in enumerate(run.trace) if e[0] == "submit"]
    assert [run.trace[i][2:] for i in submits] == want_groups  # per size in first-seen order, whole clips, greedy fill
    ok = [c for c in names.split() if isinstance(PLANS[c], tuple) and c not in BAD and len(PLANS[c][2]) <= MAX_FRAMES]
    assert run.result == (10 * len(ok), n)

    # errors: the unreadable, the over-budget and the undecodable clips; the short one apart
    assert set(run.errors) == {c for c in ("g", "i", "j", "y") if c in names.split()}
    if "g" in run.errors:
        assert isinstance(run.errors["g"], ValueError) and "5 kept frames exceed max_frames=4" in str(run.errors["g"])
        assert run.errors["i"] is PLANS["i"] and isinstance(run.errors["j"], CurateB200Error)
        assert run.short == ["h"]

    # compute gets the decoded clips and their kept frames' surfaces, clip-major; a group with no decoded clip is not computed
    for k, (_, clips) in enumerate(want_groups):
        good = [c for c in clips.split() if c not in BAD]
        if not good:
            assert k not in run.computed
            continue
        got, slots = run.computed[k]
        assert got == good
        firsts = np.cumsum([0] + [len(PLANS[c][1]) for c in clips.split()])
        want_slots = [firsts[i] + PLANS[c][2] for i, c in enumerate(clips.split()) if c not in BAD]
        assert slots.dtype == np.int32 and np.array_equal(slots, np.concatenate(want_slots))

    at = {e[:2]: i for i, e in enumerate(run.trace) if e[0] != "submit"}
    assert submits[: depth - 1] == list(range(min(depth - 1, n)))  # the first depth - 1 groups are submitted up front
    for k in range(n):
        if ("compute", k) in at:
            assert at[("compute", k)] < at[("wait", k)]
            if k >= 1:
                assert at[("compute", k)] < at[("wait", k - 1)]  # the GPU has group k queued before the host waits on k - 1
        if k >= 1 and k + depth - 1 < n:
            assert at[("wait", k - 1)] < submits[k + depth - 1] < at.get(("finish", k - 1), len(run.trace))
        if ("finish", k) in at:
            assert at[("wait", k)] < at[("finish", k)]
    assert [e for e in run.trace if e[0] == "finish"] == [("finish", k) for k in sorted(run.computed) if k % 3 != 2]

    # a pool is decoded into again only after the events of every group that read it were waited on
    for i in submits:
        readers = [e[1] for e in run.trace[:i] if e[0] == "compute" and e[2] is run.trace[i][1]]
        assert all(at[("wait", j)] < i for j in readers), (i, readers)
    # each size's groups go round a ring of `depth` pools: its j-th group decodes into the pool of its (j - depth)-th
    for size in {size for size, _ in want_groups}:
        used = [run.trace[i][1] for i in submits if run.trace[i][2] == size]
        assert all(used[j] is used[j % depth] for j in range(len(used)))
        assert len({id(p) for p in used}) == min(depth, len(used))
