"""Oracle: the numeric core of SemanticDedupActor (cosmos_curate/pipelines/video/dedup/dedup_actor.py), in numpy.

  pairwise_max        dedup() :398-470 for one cluster - sort by cosine_dist_to_cent descending, L2-normalise
                      (x / max(|x|, 1e-12)), strict upper-triangular cosine matrix (only earlier rows i < j), clip to
                      [-1, 1], per column the maximum and the FIRST row attaining it (cp.argmax; a later tile only wins
                      with a strictly greater value, :437-440), start values -1.0 / -1, row 0 forced to (0.0, 0),
                      kept = count(max <= 1 - eps)
  assign              nearest centroid as KMeans defines it (argmin squared Euclidean distance) and
                      cosine_dist_to_cent = 1 - clip(x . c/|c|) (:244-249)

Pinned (tests/test_dedup_cpu.py, tests/golden/dedup_ref.npz) against the reference's OWN array code for dedup(): the section
dedup_actor.py:404-466 is executed from its source with numpy standing in for cupy (oracle/ref_import.dedup_core; CuPy mirrors
numpy for every call in it), tiles of 256 and of the default 4096, exact / scaled / near duplicates and sort-key ties.  What stays
unpinned is library behaviour outside that section: cudf's `sort_values` tie order (restated as a stable sort) and KMeansMG
(scalable k-means++ seeding on cuML's RNG is not reproducible outside cuML: only its defining properties are tested - labels are
nearest centroids, centroids are cluster means, multi-rank == single-rank).  The reference's 4096-row tiling does not change
any result (max / first-argmax are tiling-invariant by the `>` rule above).

Test infrastructure only (see oracle/__init__.py).
"""

from __future__ import annotations

import numpy as np


def l2_normalize(x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, dtype=np.float32)
    n = np.linalg.norm(x, axis=1, keepdims=True).astype(np.float32)
    return x / np.maximum(n, np.float32(1e-12))


def pairwise_max(ids, embeddings, cosine_dist_to_cent, eps: float) -> dict:
    ids = np.asarray(ids)
    dist = np.asarray(cosine_dist_to_cent, dtype=np.float32)
    m = len(ids)
    order = np.argsort(-dist, kind="stable")  # descending, ties keep their input order
    e = l2_normalize(np.asarray(embeddings, dtype=np.float32)[order])
    maxv = np.full(m, -1.0, dtype=np.float32)
    argi = np.full(m, -1, dtype=np.int32)
    tile = 512
    for j0 in range(0, m, tile):
        j1 = min(m, j0 + tile)
        s = np.clip(e[:j1] @ e[j0:j1].T, -1.0, 1.0).astype(np.float32)  # rows i < j1, columns j0..j1
        i_idx = np.arange(j1)[:, None]
        j_idx = np.arange(j0, j1)[None, :]
        s = np.where(i_idx < j_idx, s, -np.inf)
        a = np.argmax(s, axis=0)  # first maximum
        v = s[a, np.arange(j1 - j0)]
        better = v > maxv[j0:j1]
        maxv[j0:j1] = np.where(better, v, maxv[j0:j1])
        argi[j0:j1] = np.where(better, a.astype(np.int32), argi[j0:j1])
    if m:
        maxv[0], argi[0] = 0.0, 0
    kept = int(np.count_nonzero(maxv <= np.float32(1 - eps))) if m else 0
    argi = np.where(argi < 0, 0, argi)
    sid = ids[order]
    return {"id": sid, "max_id": sid[argi], "cosine_sim_score": maxv, "kept": kept, "total": m, "sim_matrix_unit": e}


def assign(x_unit: np.ndarray, centroids: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    x = np.asarray(x_unit, dtype=np.float64)
    c = np.asarray(centroids, dtype=np.float64)
    d2 = (x * x).sum(1)[:, None] - 2.0 * x @ c.T + (c * c).sum(1)[None, :]
    labels = np.argmin(d2, axis=1).astype(np.int32)
    cu = c / np.maximum(np.linalg.norm(c, axis=1, keepdims=True), 1e-12)
    sim = (x * cu[labels]).sum(1)
    return labels, (1.0 - np.clip(sim, -1.0, 1.0)).astype(np.float32)


# ------------------------------------------------------------------------------------------------ the CUDA building blocks
# cb_rowdot_argmax, cb_rows_l2_normalize and cb_cluster_sums (csrc/dedup.cu) restated at float64 or in their own fp32 order, with
# inputs whose fp32 arithmetic is exact, for tests/test_gpu_dedup_exact.py.

U32 = 2.0**-24  # fp32 unit roundoff


def rowdot_scores(a, b, bias=None, upper: bool = False, clip: bool = False, prod: np.ndarray | None = None) -> np.ndarray:
    """S[i, j] = a_i . b_j + bias_i in float64, clamped to [-1, 1] with `clip`, -inf where `upper` excludes it (i >= j).  `prod`:
    a @ b.T at float64 when the caller already has it."""
    s = np.asarray(a, np.float64) @ np.asarray(b, np.float64).T if prod is None else prod.copy()
    if bias is not None:
        s += np.asarray(bias, np.float64)[:, None]
    if clip:
        s = np.clip(s, -1.0, 1.0)
    if upper:
        s[np.arange(s.shape[0])[:, None] >= np.arange(s.shape[1])[None, :]] = -np.inf
    return s


def rowdot_pick(s: np.ndarray, init_val: float) -> tuple[np.ndarray, np.ndarray]:
    """Per column of the scores: (maximum, FIRST row attaining it) when the maximum is strictly greater than init_val, else
    (init_val, -1)."""
    na, nb = s.shape
    if na == 0:
        return np.full(nb, init_val, np.float64), np.full(nb, -1, np.int64)
    i = np.argmax(s, axis=0)
    v = s[i, np.arange(nb)]
    ok = v > init_val
    return np.where(ok, v, init_val), np.where(ok, i, -1)


def rowdot_reference(a, b, bias=None, upper: bool = False, clip: bool = False, init_val: float = -np.inf) -> tuple[np.ndarray, np.ndarray]:
    """cb_rowdot_argmax's contract at float64: for every row j of b, the maximum over the rows i of a (i < j with `upper`) of
    a_i . b_j + bias_i (clamped to [-1, 1] with `clip`) and the first i attaining it, if it is strictly greater than init_val;
    (init_val, -1) otherwise."""
    return rowdot_pick(rowdot_scores(a, b, bias, upper, clip), init_val)


def rowdot_bound(a, b, bias=None) -> np.ndarray:
    """B[i, j] bounds |fp32 score - exact score| for the kernel's order: one sequential fma chain over d (d roundings), then one
    add of the bias: (d + 1) u (sum_k |a_ik b_jk| + |bias_i|).  Clamping to [-1, 1] is 1-Lipschitz, so B also bounds clipped scores."""
    a, b = np.abs(np.asarray(a, np.float64)), np.abs(np.asarray(b, np.float64))
    t = a @ b.T
    if bias is not None:
        t += np.abs(np.asarray(bias, np.float64))[:, None]
    return (a.shape[1] + 1) * U32 * t


def dyadic_rows(n: int, d: int, rng: np.random.Generator) -> np.ndarray:
    """Entries k/8 with |k| <= 8: every product is a multiple of 1/64 of magnitude <= 1, so every partial sum of a dot product of
    d <= 4096 terms (and a bias that is a multiple of 1/64) is exact in fp32, whatever the order.  Every third row is dense; the
    others hold ~8 non-zeros, so their scores are small, often 0 and often tied."""
    x = rng.integers(-8, 9, (n, d)).astype(np.float32)
    sparse = np.arange(n) % 3 != 0
    x[sparse] *= rng.random((int(sparse.sum()), d)) < min(1.0, 8.0 / d)
    return x / np.float32(8)


def dyadic_bias(n: int, rng: np.random.Generator) -> np.ndarray:
    return (rng.integers(-128, 129, n) / 64).astype(np.float32)


def tile_slot(i: int) -> tuple[int, int, int]:
    """Where rowdot_argmax_kernel folds candidate row i: (128-row tile, ty = the thread group of 4 rows, r = the register slot of that
    thread, r >> 2 = the 64-row half)."""
    k = i % 128
    return i // 128, (k % 64) // 4, (k % 4) + 4 * (k // 64)


# Rows that hold copies of one row; the first is the index the kernel must report.  Each group puts the first copy somewhere the
# kernel visits LATER than (or in another reduction slot from) a later copy.
TIE_GROUPS = (
    ("same_thread", (2, 66)),  # one thread, r = 2 and r = 6 (the two 64-row halves)
    ("ty_groups", (45, 70)),  # ty 11 and ty 1: the cross-thread combine meets the later row first
    ("halves", (30, 100)),  # ty 7 first half, ty 9 second half
    ("first_tile", (3, 35, 60)),  # ty 0, 8, 15 of one tile, all below row 64
    ("row_tiles", (50, 130, 300, 700)),  # tiles 0, 1, 2, 5; the later tiles' copies in lower ty
)


def tie_groups(n: int) -> list[tuple[str, tuple[int, ...]]]:
    """The TIE_GROUPS that fit n rows (the copies past row n - 1 dropped, groups left with one copy dropped)."""
    out = []
    for name, pos in TIE_GROUPS:
        p = tuple(i for i in pos if i < n)
        if len(p) >= 2:
            out.append((name, p))
    return out


def tie_columns(g: int, nb: int) -> tuple[int, ...]:
    """Columns of b set to tie group g's row: one in each tx half of the first column tile and, while it has room, one in the last
    (partial) tile."""
    last = (nb - 1) // 128 * 128
    return tuple(sorted({j for j in (g, 64 + g, nb - 1 - g) if 0 <= j < nb and (j < 128 or j >= last)}))


def plant_ties(a: np.ndarray, bias: np.ndarray | None, b: np.ndarray | None, rng: np.random.Generator):
    """Copies of one dense +-1 row at each group's positions of a (bias equal on the copies), and - when b is given - at the
    tie_columns of b: such a column's score is d + bias on every copy and below that on every other row, so its maximum is an exact
    tie and the first copy must win.  Returns (a, bias, b, [(name, positions, columns)])."""
    a, b = a.copy(), (None if b is None else b.copy())
    bias = None if bias is None else bias.copy()
    planted = []
    for g, (name, pos) in enumerate(tie_groups(len(a))):
        row = np.where(rng.random(a.shape[1]) < 0.5, -1.0, 1.0).astype(np.float32)
        a[list(pos)] = row
        if bias is not None:
            bias[list(pos)] = bias[pos[0]]
        cols = ()
        if b is not None:
            cols = tie_columns(g, len(b))
            b[list(cols)] = row
        planted.append((name, pos, cols))
    return a, bias, b, planted


UNIT_SCALES = (1.0, 2.5, 0.125)


def unit_exact_rows(n: int, d: int, rng: np.random.Generator) -> np.ndarray:
    """Rows with 4 or 16 non-zeros of +-s, s in UNIT_SCALES: the norm is 2s or 4s, so normalisation gives +-1/2 or +-1/4 exactly and
    every cosine is an exact multiple of 1/16.  Mixed in: zero rows, exact duplicates, duplicates scaled by another s, and rows that
    flip 2 signs of a 16-non-zero row (cosine exactly 3/4 with it)."""
    assert d >= 16
    x = np.zeros((n, d), np.float32)
    for i in range(n):
        kind = i % 8
        if kind == 7:  # zero row (row 7), then duplicates of an earlier row, maybe scaled
            if i >= 8:
                x[i] = x[rng.integers(0, i)] * np.float32(UNIT_SCALES[rng.integers(0, 3)])
            continue
        if kind == 6 and i >= 8:  # zero row, or 3/4-cosine sibling of an earlier 16-non-zero row
            src = [k for k in range(i) if np.count_nonzero(x[k]) == 16]
            if src:
                x[i] = x[src[rng.integers(0, len(src))]]
                nz = np.flatnonzero(x[i])
                x[i, rng.choice(nz, 2, replace=False)] *= -1
            continue
        nnz = 16 if kind % 2 else 4
        x[i, rng.choice(d, nnz, replace=False)] = np.where(rng.random(nnz) < 0.5, -1, 1) * UNIT_SCALES[rng.integers(0, 3)]
    return x


def cluster_sums_sequential(x, order, seg, sums0) -> np.ndarray:
    """cb_cluster_sums in its own fp32 order: per cluster c, 0.0f + x[order[seg[c]]] + x[order[seg[c] + 1]] + ... left to right,
    then added once to sums0[c]."""
    x = np.asarray(x, np.float32)
    order, seg = np.asarray(order, np.int64), np.asarray(seg, np.int64)
    k = len(seg) - 1
    s = np.zeros((k, x.shape[1]), np.float32)
    lens = np.diff(seg)
    for t in range(int(lens.max(initial=0))):  # step t adds every longer cluster's t-th row: the same sequential sum per cluster
        c = np.flatnonzero(lens > t)
        s[c] = s[c] + x[order[seg[c] + t]]
    return (np.asarray(sums0, np.float32) + s).astype(np.float32)


def l2_normalize_bound(x) -> tuple[np.ndarray, np.ndarray]:
    """Bounds on |fp32 - exact| of cb_rows_l2_normalize's outputs (x / |x|, |x|) for its order: a per-thread fma chain of ceil(d / 128)
    terms, 5 shuffle and 2 shared-memory levels (all terms >= 0: relative error L u, L = ceil(d / 128) + 7), then sqrtf (u / 2 more
    for the norm) and one divide (u more for the output, plus the norm's error)."""
    x = np.asarray(x, np.float64)
    lev = -(-x.shape[1] // 128) + 7
    nrm = np.sqrt((x * x).sum(1))
    rel_n = (lev / 2 + 1) * U32
    return (rel_n + 2 * U32) * np.abs(x) / np.maximum(nrm, 1e-12)[:, None], rel_n * nrm
