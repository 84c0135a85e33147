"""CPU tests of the decode-side caches and group helpers of runtime.py, with fake decoders, futures and surface pools: the
least-recently-used cache keyed by stream shape, the per-resolution surface-pool rings of the three decoding stages, the
decode-group submit / collect pair, and the stages' colour check."""

from __future__ import annotations

import types
from concurrent.futures import Future

import numpy as np
import pytest

from cosmos_curate_b200 import runtime
from cosmos_curate_b200._lib import CurateB200Error

SHAPES = [(320, 192), (640, 360), (352, 288), (480, 272), (256, 144)]
CTX = types.SimpleNamespace(device=0)


class _FakeDecoder:
    made: list = []

    def __init__(self, ctx):
        self.ctx, self.closed, self.calls = ctx, 0, []
        _FakeDecoder.made.append(self)

    def close(self):
        self.closed += 1

    def decode(self, data, ids, pool, slots, seek_keyframes=False):
        self.calls.append((data, list(ids), pool, list(slots), seek_keyframes))
        if data == "bad":
            raise CurateB200Error(-5, "cb_decoder_decode", "mp4: not an mp4")
        return {"frames_decoded": 10 * len(ids), "frames_emitted": len(ids)}


@pytest.fixture
def fake_decoders(monkeypatch):
    monkeypatch.setattr(_FakeDecoder, "made", [])
    monkeypatch.setattr(runtime, "Decoder", _FakeDecoder)
    return _FakeDecoder.made


@pytest.fixture
def allocs(monkeypatch):
    made = []

    def alloc(ctx, slots, width, height, colour="opencv"):
        made.append((slots, width, height, colour))
        return types.SimpleNamespace(buf=np.empty((slots, 0, 0), dtype=np.uint8))

    monkeypatch.setattr(runtime, "alloc_nv12_pool", alloc)
    return made


def test_shape_cache_refreshes_on_hit_and_closes_the_least_recently_used_once():
    closed = []
    cache = runtime.ShapeCache(lambda shape: [shape], closed.append)
    first = {s: cache.get(s) for s in SHAPES[:4]}
    assert cache.get(SHAPES[0]) is first[SHAPES[0]]  # a hit: now the most recently used
    assert closed == []
    fifth = cache.get(SHAPES[4])
    assert closed == [first[SHAPES[1]]]  # SHAPES[1] was the least recently used, not SHAPES[0] (the oldest inserted)
    assert cache.get(SHAPES[0]) is first[SHAPES[0]]
    again = cache.get(SHAPES[1])  # evicted: made anew, evicting SHAPES[2]
    assert again is not first[SHAPES[1]] and closed == [first[SHAPES[1]], first[SHAPES[2]]]
    cache.close()
    assert sorted(map(id, closed)) == sorted(map(id, [first[SHAPES[1]], first[SHAPES[2]], first[SHAPES[3]], fifth, first[SHAPES[0]], again]))
    assert runtime.ShapeCache.MAX_SHAPES == runtime.SessionTable.MAX_SHAPES == runtime.DecoderPool.MAX_SHAPES == 4


SEQUENCE = [SHAPES[0], SHAPES[1], SHAPES[0], SHAPES[2], SHAPES[3], SHAPES[4], SHAPES[0], SHAPES[1], SHAPES[4]]


def _eviction_pattern(decoders, get):
    """Index of the session each request got, and after the sequence the indices of the sessions closed (each once)."""
    got = [decoders.index(get(s)) for s in SEQUENCE]
    assert all(d.closed <= 1 for d in decoders)
    return got, [i for i, d in enumerate(decoders) if d.closed]


def test_session_table_and_decoder_pool_thread_table_evict_the_same_way(fake_decoders):
    table = runtime.SessionTable(CTX)
    single = _eviction_pattern(fake_decoders, table.get)
    # 0 1 0 2 3 | SHAPES[4] evicts SHAPES[1] (LRU) | SHAPES[0] hit | SHAPES[1] anew, evicting SHAPES[2] | SHAPES[4] hit
    assert single == ([0, 1, 0, 2, 3, 4, 0, 5, 4], [1, 2])
    table.close()
    assert all(d.closed == 1 for d in fake_decoders)

    fake_decoders.clear()
    dp = runtime.DecoderPool(CTX, 1, pin=False)  # one worker thread: one session table
    pooled = _eviction_pattern(fake_decoders, lambda s: dp.submit(lambda dec: dec, shape=s).result())
    assert pooled == single
    assert sorted(map(fake_decoders.index, dp._decoders)) == [0, 3, 4, 5]  # the open sessions: the other two were evicted
    assert dp.submit(lambda dec: dec).result() is fake_decoders[-1]  # shape-less callers get a session of their own
    dp.close()
    assert all(d.closed == 1 for d in fake_decoders) and dp._decoders == []


@pytest.mark.parametrize(("depth", "min_slots"), [(3, 256), (2, 8), (1, 64)])  # fused (max_batch), InternVideo2 (frames per tube), ClipFrameExtraction
def test_surface_pool_capacity_growth_and_ring_positions(allocs, depth, min_slots):
    pools = runtime.SurfacePools(CTX, depth, min_slots, "swscale")
    size = (1920, 1080)
    for n, cap in ((0, min_slots), (1, min_slots), (min_slots, min_slots), (min_slots + 1, 2 * min_slots), (4 * min_slots + 1, 8 * min_slots)):
        assert runtime.SurfacePools(CTX, depth, min_slots, "swscale").get(size, n).buf.shape[0] == cap
    allocs.clear()

    ring = [pools.get(size, min_slots, r) for r in range(depth)]
    assert len({id(p) for p in ring}) == depth and allocs == [(min_slots, 1920, 1080, "swscale")] * depth
    assert all(pools.get(size, n, r) is ring[r] for r in range(depth) for n in (1, min_slots))  # within capacity: reused
    grown = pools.get(size, min_slots + 1, 0)  # past capacity: replaced, the other positions untouched
    assert grown is not ring[0] and grown.buf.shape[0] == 2 * min_slots
    assert all(pools.get(size, min_slots, r) is ring[r] for r in range(1, depth))
    assert pools.get(size, min_slots, 0) is grown  # a larger pool serves smaller requests

    for s in SHAPES[:3]:  # four resolutions resident
        pools.get(s, 1)
    assert pools.get(size, 1, 0) is grown  # a hit: SHAPES[0] is now the least recently used
    pools.get(SHAPES[3], 1)  # a fifth resolution evicts SHAPES[0], not `size` (the oldest inserted)
    n = len(allocs)
    assert pools.get(size, 1, 0) is grown and len(allocs) == n
    pools.get(SHAPES[0], 1)
    assert len(allocs) == n + 1


def _stage_pools(which, monkeypatch):
    from cosmos_curate_b200.stages import ClipFrameExtractionStage, InternVideo2FrameCreationStage, NvdecClipAestheticStage
    from cosmos_curate_b200.stages import frame_extraction, fused_clip, internvideo2_frames

    for mod in (frame_extraction, fused_clip, internvideo2_frames):
        monkeypatch.setattr(mod, "get_context", lambda: CTX)
    if which == "fused":
        monkeypatch.setattr(fused_clip, "DecoderPool", lambda ctx, n: None)
        model = types.SimpleNamespace(setup=lambda: None, tower=types.SimpleNamespace(has_aesthetic=True))
        stage = NvdecClipAestheticStage(score_threshold=0.0, max_batch=48, model=model)
    elif which == "internvideo2":
        stage = InternVideo2FrameCreationStage(source="nvdec")
        monkeypatch.setattr(stage._model, "setup", lambda: None)
    else:
        stage = ClipFrameExtractionStage()
    stage.stage_setup()
    return stage._pools


@pytest.mark.parametrize(("which", "depth", "min_slots"), [("fused", 3, 48), ("internvideo2", 2, 8), ("frames", 1, 64)])
def test_stages_keep_their_ring_depth_and_pool_size(allocs, monkeypatch, which, depth, min_slots):
    pools = _stage_pools(which, monkeypatch)
    assert [pools.get((854, 480), 1, r).buf.shape[0] for r in range(depth)] == [min_slots] * depth
    assert {a[3] for a in allocs} == {"swscale"}
    with pytest.raises(IndexError):
        pools.get((854, 480), 1, depth)


def test_submit_group_slots_are_consecutive_and_pass_seek_and_shape(fake_decoders):
    dp = runtime.DecoderPool(CTX, 3, pin=False)
    asked = []
    dp.decoder = lambda shape=None: asked.append(shape) or _FakeDecoder(CTX)
    pool = object()
    jobs = [("a", [0, 4, 9]), ("b", []), ("c", [1, 2, 3, 5, 8]), ("d", [7, 7])]
    for seek in (False, True):
        fake_decoders.clear()
        asked.clear()
        out = dp.submit_group(pool, (854, 480), jobs, seek_keyframes=seek)
        assert [first for first, _ in out] == [0, 3, 3, 8]
        assert [f.result()["frames_emitted"] for _, f in out] == [3, 0, 5, 2]
        calls = sorted(c for d in fake_decoders for c in d.calls)
        assert [c[0] for c in calls] == ["a", "b", "c", "d"]
        for (data, ids, p, slots, sk), (first, _), (_, want_ids) in zip(calls, out, jobs):
            assert p is pool and sk is seek and ids == want_ids and slots == list(range(first, first + len(ids)))
        assert asked == [(854, 480)] * 4
    dp.close()


def _future(value=None, exc=None) -> Future:
    f = Future()
    if exc is not None:
        f.set_exception(exc)
    else:
        f.set_result(value)
    return f


def test_collect_group_errors_in_order_and_frames_of_the_jobs_that_succeeded():
    e1, e2 = CurateB200Error(-5, "cb_decoder_decode", "one"), CurateB200Error(-4, "cb_decoder_decode", "two")
    jobs = [(0, _future({"frames_decoded": 30})), (4, _future(exc=e1)), (4, _future({"frames_decoded": 12})), (9, _future(exc=e2))]
    decoded, errs = runtime.collect_group(jobs)
    assert decoded == 42
    assert errs[0] is None and errs[1] is e1 and errs[2] is None and errs[3] is e2
    assert runtime.collect_group([]) == (0, [])


def test_stages_reject_an_unknown_colour_at_construction():
    from cosmos_curate_b200.stages import ClipFrameExtractionStage, InternVideo2FrameCreationStage, NvdecClipAestheticStage

    for make in (lambda c: InternVideo2FrameCreationStage(source="nvdec", colour=c), lambda c: ClipFrameExtractionStage(colour=c),
                 lambda c: NvdecClipAestheticStage(score_threshold=None, colour=c)):  # fmt: skip
        with pytest.raises(ValueError, match="colour='bogus' not in"):
            make("bogus")
    assert runtime.check_colour("opencv") == "opencv" and set(runtime.COLOURS) == {"opencv", "swscale"}
    assert runtime.even_size(853, 481) == (854, 482) and runtime.even_size(1920, 1080) == (1920, 1080)
