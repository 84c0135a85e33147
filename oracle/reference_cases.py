"""Seeded random inputs for the differential tests against the reference's own functions (tests/test_reference_live_cpu.py).

The same generators feed `python -m oracle.make_reference_golden` (run where a checkout of the reference exists: it executes the
reference's functions on these inputs and stores what they returned in tests/golden/reference_live.json.gz) and the tests, which
rebuild the inputs from the seeds and compare this project's functions with the stored results.

Test infrastructure only (see oracle/__init__.py)."""

from __future__ import annotations

import numpy as np

N_CASES = 60


def timestamps(rng: np.random.Generator) -> np.ndarray:
    """Sorted float32 presentation times: constant or variable frame rate, optional dropped frames, optional start offset."""
    n = int(rng.integers(2, 401))
    fps = float(rng.choice([10.0, 23.976, 24.0, 25.0, 29.97, 30.0, 50.0, 59.94, 60.0]))
    t = np.arange(n, dtype=np.float64) / fps + float(rng.choice([0.0, 0.0, 0.033, 1.5]))
    if rng.random() < 0.5:
        t = t + np.cumsum(rng.uniform(0.0, 0.02, size=n))  # variable frame rate
    if rng.random() < 0.5 and n > 10:
        keep = np.ones(n, bool)
        keep[rng.integers(1, n - 1, size=int(rng.integers(0, n // 5 + 1)))] = False  # dropped frames
        t = t[keep]
    return np.sort(t.astype(np.float32))


def sample_closest_case(seed: int) -> dict:
    rng = np.random.default_rng(seed)
    ts = timestamps(rng)
    return {"ts": ts, "rate": float(rng.choice([0.5, 1.0, 2.0, 3.0, 4.0, 7.5, 8.0, 16.0, 30.0, 100.0])), "endpoint": bool(rng.random() < 0.5),
            "dedup": bool(rng.random() < 0.5), "dst": np.linspace(float(ts[0]) - 0.3, float(ts[-1]) + 0.3, 57).astype(np.float32)}  # fmt: skip


def fixed_stride_case(seed: int) -> dict:
    rng = np.random.default_rng(seed)
    alphabet = "abcXYZ019-_/ é"
    return {"end": float(rng.uniform(0.0, 400.0)), "clip_len": float(rng.uniform(0.1, 60.0)), "stride": float(rng.uniform(0.05, 90.0)),
            "min_len": float(rng.uniform(0.0, 30.0)), "session": "".join(rng.choice(list(alphabet), size=int(rng.integers(0, 13))))}  # fmt: skip


def chunk_case(seed: int) -> dict:
    rng = np.random.default_rng(seed)
    return {"durs": [float(d) for d in rng.uniform(0.0, 40.0, size=int(rng.integers(0, 121)))], "per_chunk": int(rng.integers(1, 41))}


def shot_case(seed: int) -> dict:
    rng = np.random.default_rng(seed)
    opt = lambda lo, hi: None if rng.random() < 0.3 else int(rng.integers(lo, hi + 1))  # noqa: E731
    return {"track": rng.choice([0, 0, 0, 0, 1], size=int(rng.integers(1, 601))).astype(np.uint8).reshape(-1, 1), "entire": bool(rng.random() < 0.5),
            "min_len": opt(1, 80), "max_len": opt(1, 200), "mode": str(rng.choice(["truncate", "stride"])), "crop": opt(0, 20)}  # fmt: skip


def video_tube_case(seed: int) -> dict:
    rng = np.random.default_rng(seed)
    small = rng.random() < 0.3  # 1-pixel sources and targets, exact-2x and equal sizes are drawn more often than uniformly
    h, w = (int(rng.integers(1, 5)), int(rng.integers(1, 5))) if small else (int(rng.integers(1, 261)), int(rng.integers(1, 261)))
    th, tw = int(rng.integers(1, 73)), int(rng.integers(1, 73))
    kind = rng.random()
    if kind < 0.15:
        h, w = 2 * th, 2 * tw  # the exact-2x INTER_AREA reroute
    elif kind < 0.25:
        h, w = th, tw  # the copy for equal sizes
    n = int(rng.integers(8, 20))
    return {"frames": [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for _ in range(n)], "target": (tw, th)}


def _leaf(rng: np.random.Generator):
    k = int(rng.integers(0, 7))
    if k == 0:
        return int(rng.integers(-5, 6))
    if k == 1:
        return float(rng.uniform(-2, 2))
    if k == 2:
        return "".join(rng.choice(list("ab "), size=int(rng.integers(0, 4))))
    if k == 3:
        return bool(rng.random() < 0.5)
    if k == 4:
        return None
    if k == 5:
        v = rng.uniform(-3, 3, size=int(rng.integers(0, 6))).astype(np.float32)
        v[rng.random(v.shape) < 0.15] = np.nan
        return np.array(v, dtype=str(rng.choice(["float32", "float64"])))
    return rng.integers(0, 256, size=int(rng.integers(0, 6))).astype(np.uint8)


def tree(rng: np.random.Generator, depth: int = 0):
    """A nested list / tuple / dict of leaves, like the task payloads the stage-replay comparator walks."""
    if depth >= 3 or rng.random() < 0.4:
        return _leaf(rng)
    k = int(rng.integers(0, 3))
    if k == 0:
        return [tree(rng, depth + 1) for _ in range(int(rng.integers(0, 5)))]
    if k == 1:
        return (tree(rng, depth + 1), tree(rng, depth + 1))
    keys = ["a", "b", "c", 1]
    return {keys[i]: tree(rng, depth + 1) for i in sorted(set(int(j) for j in rng.integers(0, 4, size=int(rng.integers(0, 4)))))}


def compare_case(seed: int) -> dict:
    rng = np.random.default_rng(seed)
    golden = tree(rng)
    candidate = tree(rng) if rng.random() < 0.5 else tree(np.random.default_rng(seed))  # half the pairs differ in structure, half barely
    return {"golden": golden, "candidate": candidate, "atol": float(rng.choice([0.0, 1e-3, 0.5, 2.0]))}


def diff_key(d) -> tuple:
    return (d.field, d.detail, d.max_diff_observed, d.shape_mismatch)
